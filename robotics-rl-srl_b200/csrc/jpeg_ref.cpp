// CPU checker of the JPEG encoder (include/srl_image.h on host pointers): jpeg_core.h compiled for the host and driven one block at a
// time -- a sequential DC predictor, a sequential run-length loop and a byte writer that stuffs as it goes, where the kernels
// (jpeg_kernels.cu) scan bit counts and scatter.  Test infrastructure, like the oracle: srl_sim.jpeg.encode_jpeg uses it for frames
// of the CPU oracle backend.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <vector>
#include "jpeg_core.h"
#include "../../include/srl_image.h"

namespace {

thread_local char g_err[256] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

struct ByteSink {
    std::vector<uint8_t>& out;
    uint32_t acc = 0;
    int nacc = 0;
    void byte(uint8_t b) { out.push_back(b); if (b == 0xFF) out.push_back(0); }
    void operator()(uint32_t code, int len) {
        for (int i = len - 1; i >= 0; --i) {
            acc = (acc << 1) | ((code >> i) & 1u);
            if (++nacc == 8) { byte((uint8_t)acc); acc = 0; nacc = 0; }
        }
    }
    void pad() { if (nacc) (*this)(0x7Fu, 8 - nacc); }
};

void encode_frame(const JpegFrame& F, size_t f, const JpegQuant& Q, const JpegHuffCodes& H, std::vector<uint8_t>& out) {
    out.resize(JPEG_HEADER_BYTES);
    jpeg_write_header(out.data(), F.w, F.h, Q);
    ByteSink sink{out};
    int pred[3] = {0, 0, 0};                                // DC predictor of Y, Cb, Cr
    const int mw = jpeg_mcus_x(F.w), mh = jpeg_mcus_y(F.h);
    for (int my = 0; my < mh; ++my)
        for (int mx = 0; mx < mw; ++mx)
            for (int b = 0; b < 6; ++b) {
                const int c = b < 4 ? 0 : 1;
                int zz[64];
                if (b < 4 && jpeg_dummy(F.w, F.h, mx, my, b)) {
                    for (int k = 0; k < 64; ++k) zz[k] = 0;
                    zz[0] = pred[0];                        // the DC of the luma block coded before it
                } else {
                    int d[64];
                    for (int i = 0; i < 64; ++i) {
                        const int r = i / 8, col = i % 8;
                        if (b < 4) d[i] = jpeg_luma(F, f, 16 * mx + 8 * (b & 1) + col, 16 * my + 8 * (b >> 1) + r);
                        else { int cb, cr; jpeg_chroma(F, f, 8 * mx + col, 8 * my + r, cb, cr); d[i] = b == 4 ? cb : cr; }
                    }
                    for (int r = 0; r < 8; ++r) jpeg_fdct_pass(d + 8 * r, 1, 0);
                    for (int col = 0; col < 8; ++col) jpeg_fdct_pass(d + col, 8, 1);
                    for (int k = 0; k < 64; ++k) { const int i = Q.zz[k]; zz[k] = jpeg_quantize(d[i], Q.recip[c][i], Q.shift[c][i], Q.q[c][i]); }
                }
                int& p = pred[b < 4 ? 0 : b - 3];
                jpeg_emit_dc(H, c, zz[0] - p, sink);
                p = zz[0];
                int run = 0;
                for (int k = 1; k < 64; ++k) {
                    if (!zz[k]) { ++run; continue; }
                    jpeg_emit_ac(H, 2 + c, run, zz[k], sink);
                    run = 0;
                }
                if (run) jpeg_emit_eob(H, 2 + c, sink);
            }
    sink.pad();
    out.push_back(0xFF);
    out.push_back(0xD9);
}

}  // namespace

extern "C" {

const char* srl_sim_last_error(void) { return g_err; }

size_t srl_jpeg_bound(int width, int height) {
    return jpeg_size_ok(width, height) ? jpeg_bound(width, height) : 0;
}

size_t srl_jpeg_workspace_bytes(int n, int width, int height) { return 0; }

int srl_jpeg_encode(const uint8_t* rgb, int n, int height, int width, int channels, int channel_offset, int quality, void* workspace,
                    uint8_t* out, size_t out_stride, uint32_t* out_len, void* stream) {
    if (!rgb || !out || !out_len) { set_error("jpeg_encode: null argument"); return 1; }
    if (n < 1 || !jpeg_size_ok(width, height)) { set_error("jpeg_encode: bad shape n=%d %dx%d", n, width, height); return 1; }
    if (channels < 3 || channel_offset < 0 || channel_offset > channels - 3) { set_error("jpeg_encode: channels %d / offset %d", channels, channel_offset); return 1; }
    if (quality < 1 || quality > 100) { set_error("jpeg_encode: quality %d outside 1..100", quality); return 1; }
    const size_t bound = jpeg_bound(width, height);
    if (out_stride && out_stride < bound) { set_error("jpeg_encode: out_stride %zu < srl_jpeg_bound %zu", out_stride, bound); return 1; }
    JpegQuant Q; jpeg_build_quant(quality, Q);
    static const JpegHuffCodes H = [] { JpegHuffCodes h; jpeg_build_huff(h); return h; }();
    const JpegFrame F{rgb, width, height, channels, channel_offset};
    std::vector<uint8_t> buf;
    size_t pos = 0;
    for (int f = 0; f < n; ++f) {
        encode_frame(F, (size_t)f, Q, H, buf);
        uint8_t* dst = out_stride ? out + (size_t)f * out_stride : out + pos;
        memcpy(dst, buf.data(), buf.size());
        out_len[f] = (uint32_t)buf.size();
        pos += buf.size();
    }
    return 0;
}

}  // extern "C"
