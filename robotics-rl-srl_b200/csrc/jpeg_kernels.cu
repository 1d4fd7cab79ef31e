// Batched baseline JPEG encoder (include/srl_image.h) on sm_90a.  The per-sample and per-block arithmetic is jpeg_core.h; this file
// lays it out over the GPU so that no stage walks a frame sequentially:
//   1. jpeg_block_kernel    one CTA of 64 threads per MCU row of one frame, looping over the row's MCUs: colour conversion, 2 x 2
//                           downsampling, the two FDCT passes and quantisation of the six blocks of an MCU in shared memory; writes the
//                           zig-zag coefficients, the DC and the number of AC bits of every block (two warps, one ballot per block)
//   2. jpeg_offset_kernel   one CTA per frame: adds each block's DC-difference bits, scans the counts into bit offsets, clears the
//                           frame's bit buffer and sets its 1-bit padding
//   3. jpeg_huff_kernel     one warp per block: every lane codes two coefficients at its own bit offset (a warp scan of the lanes'
//                           counts) and ORs them into the frame's bit buffer; words shared by two lanes or two blocks are merged with
//                           atomicOr, which is order-independent, so the bytes never depend on scheduling
//   4. jpeg_count_kernel    one CTA per frame: counts the 0xFF bytes, i.e. the file size after stuffing
//   5. jpeg_place_kernel    one CTA: the file offsets (packed output: a scan of the sizes)
//   6. jpeg_write_kernel    one CTA per frame: header, the data with a 0x00 after every 0xFF (a scan of the 0xFF counts), EOI
// Bit buffers are big-endian 32-bit words: bit p of a frame's stream is bit 31 - p % 32 of word p / 32.
#include <string.h>
#include "common.cuh"
#include "jpeg_core.h"
#include "../../include/srl_image.h"

namespace {

struct JpegHeader { uint8_t b[JPEG_HEADER_BYTES]; };

struct JpegWs {
    int16_t* coef;      // [n][nb][64] zig-zag order
    int16_t* dc;        // [n][nb]
    uint16_t* acbits;   // [n][nb] AC bits incl. EOB
    uint32_t* off;      // [n][nb] bit offset of the block in its frame
    uint32_t* words;    // [n][wpf] bit buffer
    uint32_t* nbytes;   // [n] entropy-coded bytes before stuffing (incl. padding)
    uint64_t* start;    // [n] file offset in `out`
    size_t nb, wpf;
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

size_t ws_layout(int n, int w, int h, uint8_t* base, JpegWs* ws) {
    const size_t nb = jpeg_blocks(w, h), wpf = jpeg_max_data_bytes(w, h) / 4 + 1, N = (size_t)n;
    size_t p = 0;
    auto take = [&](size_t bytes) { uint8_t* q = base ? base + p : nullptr; p += align256(bytes); return q; };
    JpegWs W;
    W.coef = (int16_t*)take(N * nb * 64 * sizeof(int16_t));
    W.dc = (int16_t*)take(N * nb * sizeof(int16_t));
    W.acbits = (uint16_t*)take(N * nb * sizeof(uint16_t));
    W.off = (uint32_t*)take(N * nb * sizeof(uint32_t));
    W.words = (uint32_t*)take(N * wpf * sizeof(uint32_t));
    W.nbytes = (uint32_t*)take(N * sizeof(uint32_t));
    W.start = (uint64_t*)take(N * sizeof(uint64_t));
    W.nb = nb; W.wpf = wpf;
    if (ws) *ws = W;
    return p;
}

// Code and length of every symbol: the tables do not depend on quality, so they are a constant of the library.
__constant__ JpegHuffCodes c_huff;
bool g_huff_ready[64] = {};

struct CountBits {
    int n = 0;
    __device__ void operator()(uint32_t, int len) { n += len; }
};

struct WriteBits {
    uint32_t* buf;
    uint32_t pos, acc = 0;
    __device__ void operator()(uint32_t code, int len) {          // len <= 16
        while (len > 0) {
            const int room = 32 - (int)(pos & 31), take = len < room ? len : room;
            acc |= ((code >> (len - take)) & ((1u << take) - 1u)) << (room - take);
            pos += take; len -= take;
            if (!(pos & 31)) { if (acc) atomicOr(buf + (pos >> 5) - 1, acc); acc = 0; }
        }
    }
    __device__ void flush() { if ((pos & 31) && acc) atomicOr(buf + (pos >> 5), acc); }
};

// bit k of the result = bit k / 2 of `even` (k even) or of `odd` (k odd)
__device__ __forceinline__ uint64_t interleave(uint32_t even, uint32_t odd) {
    auto spread = [](uint64_t x) {
        x = (x | (x << 16)) & 0x0000FFFF0000FFFFull; x = (x | (x << 8)) & 0x00FF00FF00FF00FFull;
        x = (x | (x << 4)) & 0x0F0F0F0F0F0F0F0Full; x = (x | (x << 2)) & 0x3333333333333333ull;
        return (x | (x << 1)) & 0x5555555555555555ull;
    };
    return spread(even) | (spread(odd) << 1);
}

// The AC codes of zig-zag positions 2 lane and 2 lane + 1 of one block (v0, v1; position 0 is the DC and is skipped), and the EOB if this
// lane holds the block's last non-zero coefficient (lane 0 when there is none).  Every lane of the warp calls it.
template <class Emit>
__device__ int lane_ac(const JpegHuffCodes& H, int table, int lane, int v0, int v1, Emit& emit) {
    const uint32_t ev = __ballot_sync(0xffffffffu, lane > 0 && v0 != 0), od = __ballot_sync(0xffffffffu, v1 != 0);
    const uint64_t nz = interleave(ev, od);
    int bits = 0;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const int k = 2 * lane + j, v = j ? v1 : v0;
        if (k == 0 || v == 0) continue;
        const uint64_t below = nz & ((1ull << k) - 1ull);
        const int prev = below ? 63 - __clzll((long long)below) : 0;
        bits += jpeg_emit_ac(H, table, k - prev - 1, v, emit);
    }
    const int last = nz ? 63 - __clzll((long long)nz) : 0;
    if (last < 63 && lane == last / 2) bits += jpeg_emit_eob(H, table, emit);
    return bits;
}

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int warp_excl_scan(int v, int lane) {
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    return x - v;
}
// Exclusive scan over a CTA of NT threads (NT a multiple of 32, <= 1024); *total = the sum.  Uses `tmp` (33 elements).
template <int NT, class T>
__device__ T cta_excl_scan(T v, T* tmp, T* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    T x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const T y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) tmp[wid] = x;
    __syncthreads();
    if (wid == 0) {
        T s = lane < NT / 32 ? tmp[lane] : T(0), t = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const T y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= o) t += y; }
        tmp[lane] = t - s;
        if (lane == 31) tmp[32] = t;
    }
    __syncthreads();
    const T r = tmp[wid] + x - v;
    *total = tmp[32];
    __syncthreads();
    return r;
}

// index of the block whose DC predicts block j (same component, previous MCU for the first luma block and the chroma blocks), -1: none
__device__ __forceinline__ long pred_block(long j) {
    const long m = j / 6, b = j % 6;
    if (b >= 1 && b <= 3) return j - 1;
    if (m == 0) return -1;
    return b == 0 ? j - 3 : j - 6;
}

__global__ void __launch_bounds__(64) jpeg_block_kernel(JpegFrame F, size_t f0, const __grid_constant__ JpegQuant Qp, JpegWs ws) {
    __shared__ int blk[6][64];
    __shared__ int zz[6][64];
    __shared__ JpegQuant Q;
    __shared__ JpegHuffCodes H;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    for (int i = t; i < (int)(sizeof(JpegQuant) / 4); i += 64) reinterpret_cast<uint32_t*>(&Q)[i] = reinterpret_cast<const uint32_t*>(&Qp)[i];
    for (int i = t; i < (int)(sizeof(JpegHuffCodes) / 4); i += 64) reinterpret_cast<uint32_t*>(&H)[i] = reinterpret_cast<const uint32_t*>(&c_huff)[i];
    const size_t f = f0 + blockIdx.z;
    const int my = blockIdx.x, mw = jpeg_mcus_x(F.w);
    __syncthreads();
    for (int mx = 0; mx < mw; ++mx) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int p = t + 64 * i, ly = p >> 4, lx = p & 15;
            blk[(ly >> 3) * 2 + (lx >> 3)][(ly & 7) * 8 + (lx & 7)] = jpeg_luma(F, f, 16 * mx + lx, 16 * my + ly);
        }
        int cb, cr;
        jpeg_chroma(F, f, 8 * mx + (t & 7), 8 * my + (t >> 3), cb, cr);
        blk[4][t] = cb; blk[5][t] = cr;
        __syncthreads();
        if (t < 48) jpeg_fdct_pass(&blk[t >> 3][(t & 7) * 8], 1, 0);
        __syncthreads();
        if (t < 48) jpeg_fdct_pass(&blk[t >> 3][t & 7], 8, 1);
        __syncthreads();
        const int nat = Q.zz[t];
#pragma unroll
        for (int b = 0; b < 6; ++b) {
            const int c = b < 4 ? 0 : 1;
            const bool dummy = b < 4 && jpeg_dummy(F.w, F.h, mx, my, b);
            zz[b][t] = dummy ? 0 : jpeg_quantize(blk[b][nat], Q.recip[c][nat], Q.shift[c][nat], Q.q[c][nat]);
        }
        __syncthreads();
        if (t == 0)
            for (int b = 1; b < 4; ++b)
                if (jpeg_dummy(F.w, F.h, mx, my, b)) zz[b][0] = zz[b - 1][0];   // a dummy block repeats the DC coded before it
        __syncthreads();
        const size_t j0 = f * ws.nb + (size_t)(my * mw + mx) * 6;
        for (int b = warp; b < 6; b += 2) {
            CountBits cnt;
            const int bits = warp_sum(lane_ac(H, b < 4 ? 2 : 3, lane, zz[b][2 * lane], zz[b][2 * lane + 1], cnt));
            if (lane == 0) ws.acbits[j0 + b] = (uint16_t)bits;
        }
#pragma unroll
        for (int b = 0; b < 6; ++b) ws.coef[(j0 + b) * 64 + t] = (int16_t)zz[b][t];
        if (t < 6) ws.dc[j0 + t] = (int16_t)zz[t][0];
        __syncthreads();
    }
}

constexpr int OFF_NT = 256;
__global__ void __launch_bounds__(OFF_NT) jpeg_offset_kernel(JpegWs ws) {
    __shared__ uint32_t tmp[33];
    __shared__ uint8_t dcsize[2][12];
    if (threadIdx.x < 24) dcsize[threadIdx.x / 12][threadIdx.x % 12] = c_huff.size[threadIdx.x / 12][threadIdx.x % 12];
    __syncthreads();
    const size_t f = blockIdx.x, nb = ws.nb, per = (nb + OFF_NT - 1) / OFF_NT;
    const int16_t* dc = ws.dc + f * nb;
    const uint16_t* ac = ws.acbits + f * nb;
    auto bits_of = [&](long j) {
        const long p = pred_block(j);
        const int n = jpeg_nbits(dc[j] - (p < 0 ? 0 : dc[p]));
        return (uint32_t)ac[j] + dcsize[j % 6 < 4 ? 0 : 1][n] + n;
    };
    const size_t j0 = threadIdx.x * per, j1 = j0 + per < nb ? j0 + per : nb;
    uint32_t mine = 0;
    for (size_t j = j0; j < j1; ++j) mine += bits_of((long)j);
    uint32_t total;
    uint32_t o = cta_excl_scan<OFF_NT, uint32_t>(mine, tmp, &total);
    for (size_t j = j0; j < j1; ++j) { ws.off[f * nb + j] = o; o += bits_of((long)j); }
    const uint32_t pad = (8u - (total & 7u)) & 7u, bytes = (total + pad) / 8u, nw = (bytes + 3u) / 4u;
    uint32_t* words = ws.words + f * ws.wpf;
    for (uint32_t i = threadIdx.x; i < nw; i += OFF_NT) {
        uint32_t v = 0;
        if (pad && i == (total >> 5)) v = ((1u << pad) - 1u) << (32u - (total & 31u) - pad);   // padding: 1 bits up to the byte boundary
        words[i] = v;
    }
    if (threadIdx.x == 0) ws.nbytes[f] = bytes;
}

__global__ void __launch_bounds__(256) jpeg_huff_kernel(JpegWs ws, size_t total_blocks) {
    __shared__ JpegHuffCodes H;
    for (int i = threadIdx.x; i < (int)(sizeof(JpegHuffCodes) / 4); i += 256) reinterpret_cast<uint32_t*>(&H)[i] = reinterpret_cast<const uint32_t*>(&c_huff)[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    // a grid of a few CTAs per SM strides over the blocks, so that the table is copied once per CTA rather than once per 8 blocks
    for (size_t g = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5); g < total_blocks; g += (size_t)gridDim.x * 8) {
        const size_t f = g / ws.nb, j = g % ws.nb;
        const int b = (int)(j % 6), c = b < 4 ? 0 : 1;
        const uint32_t pair = reinterpret_cast<const uint32_t*>(ws.coef + g * 64)[lane];
        const int v0 = (int16_t)(pair & 0xFFFFu), v1 = (int16_t)(pair >> 16);
        int diff = 0;
        if (lane == 0) { const long p = pred_block((long)j); diff = v0 - (p < 0 ? 0 : ws.dc[f * ws.nb + p]); }
        CountBits cnt;
        if (lane == 0) jpeg_emit_dc(H, c, diff, cnt);
        lane_ac(H, 2 + c, lane, v0, v1, cnt);
        WriteBits wr{ws.words + f * ws.wpf, ws.off[g] + (uint32_t)warp_excl_scan(cnt.n, lane)};
        if (lane == 0) jpeg_emit_dc(H, c, diff, wr);
        lane_ac(H, 2 + c, lane, v0, v1, wr);
        wr.flush();
    }
}

__device__ __forceinline__ uint32_t byte_of(const uint32_t* words, uint32_t i) { return (words[i >> 2] >> (24 - 8 * (i & 3))) & 0xFFu; }

constexpr int STUFF_NT = 256, STUFF_PER = 16;   // bytes per thread and pass
__global__ void __launch_bounds__(STUFF_NT) jpeg_count_kernel(JpegWs ws, uint32_t* out_len) {
    __shared__ uint32_t tmp[33];
    const size_t f = blockIdx.x;
    const uint32_t nbytes = ws.nbytes[f];
    const uint32_t* words = ws.words + f * ws.wpf;
    uint32_t ff = 0;
    for (uint32_t i = threadIdx.x; i < nbytes; i += STUFF_NT) ff += byte_of(words, i) == 0xFFu;
    uint32_t total;
    cta_excl_scan<STUFF_NT, uint32_t>(ff, tmp, &total);
    if (threadIdx.x == 0) out_len[f] = JPEG_HEADER_BYTES + nbytes + total + 2;
}

constexpr int PLACE_NT = 1024;
__global__ void __launch_bounds__(PLACE_NT) jpeg_place_kernel(JpegWs ws, const uint32_t* out_len, int n, size_t stride) {
    __shared__ uint64_t tmp[33];
    if (stride) {
        for (int f = threadIdx.x; f < n; f += PLACE_NT) ws.start[f] = (uint64_t)f * stride;
        return;
    }
    uint64_t carry = 0;
    for (int f0 = 0; f0 < n; f0 += PLACE_NT) {
        const int f = f0 + threadIdx.x;
        uint64_t total;     // 64-bit: a chunk of 1024 file sizes can exceed 2^32 bytes
        const uint64_t o = cta_excl_scan<PLACE_NT, uint64_t>(f < n ? (uint64_t)out_len[f] : 0ull, tmp, &total);
        if (f < n) ws.start[f] = carry + o;
        carry += total;
    }
}

__global__ void __launch_bounds__(STUFF_NT) jpeg_write_kernel(JpegWs ws, const __grid_constant__ JpegHeader hdr, uint8_t* out) {
    __shared__ uint32_t tmp[33];
    const size_t f = blockIdx.x;
    uint8_t* o = out + ws.start[f];
    for (int i = threadIdx.x; i < JPEG_HEADER_BYTES; i += STUFF_NT) o[i] = hdr.b[i];
    o += JPEG_HEADER_BYTES;
    const uint32_t nbytes = ws.nbytes[f];
    const uint32_t* words = ws.words + f * ws.wpf;
    uint32_t carry = 0;
    for (uint32_t base = 0; base < nbytes; base += STUFF_NT * STUFF_PER) {
        const uint32_t i0 = base + threadIdx.x * STUFF_PER;
        uint32_t ff = 0;
        for (uint32_t i = i0; i < i0 + STUFF_PER && i < nbytes; ++i) ff += byte_of(words, i) == 0xFFu;
        uint32_t total;
        uint32_t q = carry + i0 + cta_excl_scan<STUFF_NT, uint32_t>(ff, tmp, &total);
        for (uint32_t i = i0; i < i0 + STUFF_PER && i < nbytes; ++i) {
            const uint32_t v = byte_of(words, i);
            o[q++] = (uint8_t)v;
            if (v == 0xFFu) o[q++] = 0;
        }
        carry += total;
    }
    if (threadIdx.x == 0) { const uint32_t end = nbytes + carry; o[end] = 0xFF; o[end + 1] = 0xD9; }
}

int ensure_huff() {
    int dev = 0;
    SRL_CUDA_OK(cudaGetDevice(&dev));
    if (dev >= 0 && dev < 64 && g_huff_ready[dev]) return 0;
    static const JpegHuffCodes H = [] { JpegHuffCodes h; jpeg_build_huff(h); return h; }();
    SRL_CUDA_OK(cudaMemcpyToSymbol(c_huff, &H, sizeof(H)));
    if (dev >= 0 && dev < 64) g_huff_ready[dev] = true;
    return 0;
}

}  // namespace

extern "C" {

size_t srl_jpeg_bound(int width, int height) {
    return jpeg_size_ok(width, height) ? jpeg_bound(width, height) : 0;
}

size_t srl_jpeg_workspace_bytes(int n, int width, int height) {
    if (n < 1 || !jpeg_size_ok(width, height)) return 0;
    return ws_layout(n, width, height, nullptr, nullptr);
}

int srl_jpeg_encode(const uint8_t* rgb, int n, int height, int width, int channels, int channel_offset, int quality, void* workspace,
                    uint8_t* out, size_t out_stride, uint32_t* out_len, void* stream) {
    if (!rgb || !workspace || !out || !out_len) { srl_set_error("jpeg_encode: null argument"); return 1; }
    if (n < 1 || !jpeg_size_ok(width, height)) { srl_set_error("jpeg_encode: bad shape n=%d %dx%d", n, width, height); return 1; }
    if (channels < 3 || channel_offset < 0 || channel_offset > channels - 3) { srl_set_error("jpeg_encode: channels %d / offset %d", channels, channel_offset); return 1; }
    if (quality < 1 || quality > 100) { srl_set_error("jpeg_encode: quality %d outside 1..100", quality); return 1; }
    const size_t bound = jpeg_bound(width, height);
    if (out_stride && out_stride < bound) { srl_set_error("jpeg_encode: out_stride %zu < srl_jpeg_bound %zu", out_stride, bound); return 1; }
    if (ensure_huff()) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    JpegWs ws;
    ws_layout(n, width, height, (uint8_t*)workspace, &ws);
    JpegQuant Q;
    jpeg_build_quant(quality, Q);
    JpegHeader hdr;
    jpeg_write_header(hdr.b, width, height, Q);
    const JpegFrame F{rgb, width, height, channels, channel_offset};
    for (int f0 = 0; f0 < n; f0 += 65535)                                  // grid.z is limited to 65535
        jpeg_block_kernel<<<dim3(jpeg_mcus_y(height), 1, min(65535, n - f0)), 64, 0, st>>>(F, (size_t)f0, Q, ws);
    SRL_CUDA_OK(cudaGetLastError());
    jpeg_offset_kernel<<<n, OFF_NT, 0, st>>>(ws);
    int dev = 0, sms = 0;
    SRL_CUDA_OK(cudaGetDevice(&dev));
    SRL_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const size_t total_blocks = (size_t)n * ws.nb, ctas = (total_blocks + 7) / 8, cap = (size_t)sms * 8;
    jpeg_huff_kernel<<<(unsigned)(ctas < cap ? ctas : cap), 256, 0, st>>>(ws, total_blocks);
    jpeg_count_kernel<<<n, STUFF_NT, 0, st>>>(ws, out_len);
    jpeg_place_kernel<<<1, PLACE_NT, 0, st>>>(ws, out_len, n, out_stride);
    jpeg_write_kernel<<<n, STUFF_NT, 0, st>>>(ws, hdr, out);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
