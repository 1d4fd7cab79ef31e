/*
 * srl_image.h -- C-ABI of the batched JPEG encoder that sits next to srl_sim_render in libsrl_sim_b200.so.
 *
 * A dataset of SRL frames is a folder of .jpg files per episode (the reference's state_representation/episode_saver.py writes one per
 * recorded state with cv2.imwrite).  Rendering a batch of frames on the GPU takes milliseconds; encoding them one by one on the host
 * takes far longer, and copying raw frames to the host moves ~10-30x more bytes than the JPEG files.  This entry point encodes a whole
 * batch of device frames on the device and leaves the finished files in device memory.
 *
 * Output: baseline JFIF, 4:2:0, Annex K Huffman tables, libjpeg's quality rule -- byte for byte what
 * `cv2.imencode('.jpg', frame[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, quality])` returns for an RGB frame (csrc/jpeg_core.h).
 *
 * Conventions are those of srl_sim.h: 0 on success, message from srl_sim_last_error(); for the CUDA library every buffer is a DEVICE
 * pointer and the call is asynchronous on `stream`.  The CPU checker (csrc/libjpeg_ref.so, test infrastructure) exports the same three
 * functions on HOST pointers (workspace unused, may be NULL; stream ignored).
 */
#ifndef SRL_IMAGE_H_
#define SRL_IMAGE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Worst-case size in bytes of one encoded w x h frame, whatever its pixels and quality: the 623 header bytes, 1660 bits per 8 x 8 block
 * (the longest DC code and 63 of the longest AC codes), every entropy-coded byte doubled by 0xFF stuffing, and EOI.  0 for an invalid size. */
size_t srl_jpeg_bound(int width, int height);

/* Device workspace of one srl_jpeg_encode call of n frames (per 8 x 8 block: the coefficients, bit count and offset, and room for its
 * longest code before stuffing). */
size_t srl_jpeg_workspace_bytes(int n, int width, int height);

/* Encode n frames.
 *   rgb            u8[n, height, width, channels]; R G B are the channels channel_offset .. channel_offset + 2 (so one camera of a
 *                  [n, H, W, 6] two-camera frame is encoded without a copy)
 *   quality        1..100 (libjpeg's scale of the Annex K tables; OpenCV's default is 95)
 *   workspace      srl_jpeg_workspace_bytes(n, width, height) bytes; no state is kept between calls
 *   out            out_stride > 0: frame i is written at out + i * out_stride, and out_stride must be >= srl_jpeg_bound(width, height);
 *                  out_stride == 0: the files are packed back to back in frame order (frame i starts at the sum of out_len[0 .. i-1]),
 *                  and out must hold n * srl_jpeg_bound(width, height) bytes in the worst case
 *   out_len        u32[n]: the size of each file
 * The bytes are deterministic: the same input gives the same output on every call. */
int srl_jpeg_encode(const uint8_t* rgb, int n, int height, int width, int channels, int channel_offset, int quality, void* workspace,
                    uint8_t* out, size_t out_stride, uint32_t* out_len, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SRL_IMAGE_H_ */
