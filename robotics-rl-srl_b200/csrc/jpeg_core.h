// Baseline JPEG encoding of RGB frames (include/srl_image.h): the per-sample and per-block arithmetic, shared by the sm_90a kernels
// (csrc/jpeg_kernels.cu) and the sequential CPU checker (csrc/jpeg_ref.cpp, test infrastructure).
//
// The target is the byte stream OpenCV writes for `cv2.imencode('.jpg', bgr, [cv2.IMWRITE_JPEG_QUALITY, q])` with its bundled
// libjpeg-turbo: JFIF APP0 1.01 (aspect 1:1), one DQT per table, SOF0 with Y sampled 2x2 and Cb / Cr 1x1 (4:2:0), the four Huffman tables
// of ITU-T T.81 Annex K.3, one interleaved scan over Y0 Y1 Y2 Y3 Cb Cr minimum coded units (MCUs) in raster order, no restart markers.
// Everything below is written from T.81 and from the observable behaviour of that encoder:
//   colour       Y  = (19595 R + 38470 G +  7471 B + 2^15) >> 16
//                Cb = (-11059 R - 21709 G + 32768 B + 2^23 + 2^15 - 1) >> 16,  Cr = (32768 R - 27439 G - 5329 B + 2^23 + 2^15 - 1) >> 16
//   edges        columns past the frame repeat the last column; Y rows past the frame repeat the last row; a chroma row is the 2 x 2 mean
//                of rows (2 cy, min(2 cy + 1, H - 1)), and chroma rows past ceil(H / 2) repeat the last chroma row;
//                8 x 8 luma blocks wholly outside ceil(W / 8) x ceil(H / 8) are "dummy" blocks: zero AC, the DC of the block coded before them
//   downsample   (a + b + c + d + bias) >> 2 with bias 1 on even and 2 on odd chroma columns
//   FDCT         the separable integer "islow" transform (13-bit constants, 2 extra bits between the passes), output scaled by 8
//   quantise     round-half-up division of |c| by 8 q (q from the Annex K.1 / K.2 tables scaled by the quality rule, clamped to 1..255)
//   entropy      DC differences per component, AC run / size symbols with ZRL and EOB, 0xFF -> 0xFF 0x00 stuffing, 1-bit padding, EOI.
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(__CUDACC__)
#define JPEG_HD __host__ __device__ __forceinline__
#else
#define JPEG_HD inline
#endif

#define JPEG_HEADER_BYTES 623          // SOI + APP0 + 2 DQT + SOF0 + 4 DHT + SOS for this layout (independent of size and quality)
#define JPEG_MAX_BLOCK_BITS 1660       // 22 (chroma DC code of category 11 + 11 bits) + 63 x 26 (16-bit AC code + 10 bits)
#define JPEG_BLOCK_WORDS ((JPEG_MAX_BLOCK_BITS + 31) / 32)

// ---- tables (T.81 Annex K) --------------------------------------------------------------------------------------------------------
static const uint8_t JPEG_QUANT_BASE[2][64] = {
    {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
     18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};

// Huffman table specifications: number of codes of length 1..16, then the symbols in code order.  0 = luma DC, 1 = chroma DC,
// 2 = luma AC, 3 = chroma AC.
static const uint8_t JPEG_HUFF_BITS[4][16] = {
    {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
    {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0},
    {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
    {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
static const uint8_t JPEG_HUFF_DC_VALS[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t JPEG_HUFF_AC_VALS[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1,
     0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26,
     0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56,
     0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85,
     0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa,
     0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6,
     0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9,
     0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42,
     0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19,
     0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55,
     0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83,
     0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8,
     0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4,
     0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9,
     0xfa}};

// ---- per-quality tables the encoder is parameterised with (built on the host, passed to the kernels by value) -------------------------
struct JpegHuffCodes { uint16_t code[4][256]; uint8_t size[4][256]; };   // Annex C: code and length of every symbol of the four tables
struct JpegQuant {
    uint8_t zz[64];           // zig-zag index -> natural (row-major) index
    uint16_t q[2][64];        // quantiser (natural order) of the luma / chroma table after the quality rule
    uint32_t recip[2][64];    // round-half-up division of |c| by 8 q as ((|c| + 4 q) * recip) >> shift: exact for |c| < 2^15
    uint8_t shift[2][64];
};

inline void jpeg_zigzag(uint8_t zz[64]) {
    int k = 0;
    for (int s = 0; s <= 14; ++s)                          // anti-diagonals r + c = s, alternating direction
        for (int i = 0; i <= s; ++i) {
            const int r = (s & 1) ? i : s - i, c = s - r;
            if (r < 8 && c < 8) zz[k++] = (uint8_t)(8 * r + c);
        }
}

inline int jpeg_quality_scale(int quality) {
    if (quality < 1) quality = 1;
    if (quality > 100) quality = 100;
    return quality < 50 ? 5000 / quality : 200 - 2 * quality;
}

inline void jpeg_build_quant(int quality, JpegQuant& t) {
    jpeg_zigzag(t.zz);
    const int scale = jpeg_quality_scale(quality);
    for (int c = 0; c < 2; ++c)
        for (int i = 0; i < 64; ++i) {
            long v = ((long)JPEG_QUANT_BASE[c][i] * scale + 50) / 100;
            v = v < 1 ? 1 : v > 255 ? 255 : v;
            t.q[c][i] = (uint16_t)v;
            const uint32_t d = 8u * (uint32_t)v;
            int b = 31; while (!(d >> b)) --b;             // floor(log2 d)
            const int sh = 16 + b;
            t.recip[c][i] = (uint32_t)(((1ull << sh) + d - 1) / d);
            t.shift[c][i] = (uint8_t)sh;
        }
}

inline void jpeg_build_huff(JpegHuffCodes& h) {
    for (int t = 0; t < 4; ++t) {
        const uint8_t* vals = t < 2 ? JPEG_HUFF_DC_VALS : JPEG_HUFF_AC_VALS[t - 2];
        for (int s = 0; s < 256; ++s) { h.code[t][s] = 0; h.size[t][s] = 0; }
        int code = 0, k = 0;
        for (int len = 1; len <= 16; ++len) {
            for (int i = 0; i < JPEG_HUFF_BITS[t][len - 1]; ++i, ++k) { h.code[t][vals[k]] = (uint16_t)code++; h.size[t][vals[k]] = (uint8_t)len; }
            code <<= 1;
        }
    }
}

// ---- sizes --------------------------------------------------------------------------------------------------------------------------
JPEG_HD int jpeg_mcus_x(int w) { return (w + 15) / 16; }
JPEG_HD int jpeg_mcus_y(int h) { return (h + 15) / 16; }
inline size_t jpeg_blocks(int w, int h) { return (size_t)6 * jpeg_mcus_x(w) * jpeg_mcus_y(h); }
// entropy-coded bytes before stuffing, worst case (every block at JPEG_MAX_BLOCK_BITS, plus the padding byte)
inline size_t jpeg_max_data_bytes(int w, int h) { return (jpeg_blocks(w, h) * JPEG_MAX_BLOCK_BITS + 7) / 8; }
// a whole file, worst case: header, every data byte stuffed (0xFF 0x00), EOI
inline size_t jpeg_bound(int w, int h) { return JPEG_HEADER_BYTES + 2 * jpeg_max_data_bytes(w, h) + 2; }
// Sizes the encoder accepts: 1..65535 per side (SOF0), and a worst case that 32-bit bit offsets and file sizes can count
// (about 8800 x 8800 pixels and beyond are refused rather than wrapped).
inline bool jpeg_size_ok(int w, int h) {
    return w >= 1 && h >= 1 && w <= 65535 && h <= 65535 && jpeg_blocks(w, h) * JPEG_MAX_BLOCK_BITS + 32 < (1ull << 32) &&
           jpeg_bound(w, h) < (1ull << 32);
}

// The 623 header bytes for a w x h frame at `quality`.
inline void jpeg_write_header(uint8_t* o, int w, int h, const JpegQuant& t) {
    int p = 0;
    auto b = [&](int v) { o[p++] = (uint8_t)v; };
    auto w16 = [&](int v) { b(v >> 8); b(v & 0xFF); };
    w16(0xFFD8);
    w16(0xFFE0); w16(16); b('J'); b('F'); b('I'); b('F'); b(0); b(1); b(1); b(0); w16(1); w16(1); b(0); b(0);
    for (int c = 0; c < 2; ++c) { w16(0xFFDB); w16(67); b(c); for (int k = 0; k < 64; ++k) b(t.q[c][t.zz[k]]); }
    w16(0xFFC0); w16(17); b(8); w16(h); w16(w); b(3); b(1); b(0x22); b(0); b(2); b(0x11); b(1); b(3); b(0x11); b(1);
    const int order[4] = {0, 2, 1, 3};                    // per component: DC then AC table (luma, then chroma)
    for (int i = 0; i < 4; ++i) {
        const int t2 = order[i], nv = t2 < 2 ? 12 : 162;
        w16(0xFFC4); w16(2 + 1 + 16 + nv); b((t2 >= 2 ? 0x10 : 0) | (t2 & 1));
        for (int l = 0; l < 16; ++l) b(JPEG_HUFF_BITS[t2][l]);
        const uint8_t* vals = t2 < 2 ? JPEG_HUFF_DC_VALS : JPEG_HUFF_AC_VALS[t2 - 2];
        for (int k = 0; k < nv; ++k) b(vals[k]);
    }
    w16(0xFFDA); w16(12); b(3); b(1); b(0x00); b(2); b(0x11); b(3); b(0x11); b(0); b(63); b(0);
}

// ---- samples ------------------------------------------------------------------------------------------------------------------------
// Frame f, pixel (x, y) of an [n, h, w, channels] u8 array; R G B at channel_offset .. channel_offset + 2.
struct JpegFrame { const uint8_t* rgb; int w, h, channels, offset; };
JPEG_HD const uint8_t* jpeg_px(const JpegFrame& F, size_t frame, int x, int y) {
    x = x < F.w ? x : F.w - 1; y = y < F.h ? y : F.h - 1;
    return F.rgb + ((frame * F.h + y) * F.w + x) * F.channels + F.offset;
}
JPEG_HD int jpeg_y(const uint8_t* p) { return (19595 * p[0] + 38470 * p[1] + 7471 * p[2] + 32768) >> 16; }
JPEG_HD int jpeg_cb(const uint8_t* p) { return (-11059 * p[0] - 21709 * p[1] + 32768 * p[2] + (128 << 16) + 32767) >> 16; }
JPEG_HD int jpeg_cr(const uint8_t* p) { return (32768 * p[0] - 27439 * p[1] - 5329 * p[2] + (128 << 16) + 32767) >> 16; }

// Level-shifted luma sample at (x, y) of the padded plane.
JPEG_HD int jpeg_luma(const JpegFrame& F, size_t frame, int x, int y) { return jpeg_y(jpeg_px(F, frame, x, y)) - 128; }

// Level-shifted chroma samples (Cb, Cr) of the 2 x 2 downsampled plane at (cx, cy).
JPEG_HD void jpeg_chroma(const JpegFrame& F, size_t frame, int cx, int cy, int& cb, int& cr) {
    const int last = (F.h + 1) / 2 - 1;                     // chroma rows past the frame repeat the last one
    cy = cy < last ? cy : last;
    const int y0 = 2 * cy, y1 = 2 * cy + 1 < F.h ? 2 * cy + 1 : F.h - 1, x0 = 2 * cx;
    const uint8_t* a = jpeg_px(F, frame, x0, y0); const uint8_t* b = jpeg_px(F, frame, x0 + 1, y0);
    const uint8_t* c = jpeg_px(F, frame, x0, y1); const uint8_t* d = jpeg_px(F, frame, x0 + 1, y1);
    const int bias = 1 + (cx & 1);
    cb = ((jpeg_cb(a) + jpeg_cb(b) + jpeg_cb(c) + jpeg_cb(d) + bias) >> 2) - 128;
    cr = ((jpeg_cr(a) + jpeg_cr(b) + jpeg_cr(c) + jpeg_cr(d) + bias) >> 2) - 128;
}

// Is luma block `j` (0..3, raster order inside the MCU) of MCU (mx, my) a dummy block?
JPEG_HD bool jpeg_dummy(int w, int h, int mx, int my, int j) {
    return 2 * mx + (j & 1) >= (w + 7) / 8 || 2 * my + (j >> 1) >= (h + 7) / 8;
}

// ---- forward DCT: one 8-point pass over d[0], d[s], ..., d[7 s] ------------------------------------------------------------------------
// pass 0 (rows) keeps 2 extra bits of precision, pass 1 (columns) removes them; the 2-D result is 8 x the orthonormal DCT.
JPEG_HD int jpeg_descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }
JPEG_HD void jpeg_fdct_pass(int* d, int s, int pass) {
    const int t0 = d[0] + d[7 * s], t7 = d[0] - d[7 * s], t1 = d[s] + d[6 * s], t6 = d[s] - d[6 * s];
    const int t2 = d[2 * s] + d[5 * s], t5 = d[2 * s] - d[5 * s], t3 = d[3 * s] + d[4 * s], t4 = d[3 * s] - d[4 * s];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    const int sh = pass == 0 ? 13 - 2 : 13 + 2;
    if (pass == 0) { d[0] = (t10 + t11) * 4; d[4 * s] = (t10 - t11) * 4; }
    else { d[0] = jpeg_descale(t10 + t11, 2); d[4 * s] = jpeg_descale(t10 - t11, 2); }
    const int z1 = (t12 + t13) * 4433;
    d[2 * s] = jpeg_descale(z1 + t13 * 6270, sh);
    d[6 * s] = jpeg_descale(z1 - t12 * 15137, sh);
    const int z5 = (t4 + t6 + t5 + t7) * 9633;
    const int a1 = (t4 + t7) * -7373, a2 = (t5 + t6) * -20995, a3 = (t4 + t6) * -16069 + z5, a4 = (t5 + t7) * -3196 + z5;
    d[7 * s] = jpeg_descale(t4 * 2446 + a1 + a3, sh);
    d[5 * s] = jpeg_descale(t5 * 16819 + a2 + a4, sh);
    d[3 * s] = jpeg_descale(t6 * 25172 + a2 + a3, sh);
    d[s] = jpeg_descale(t7 * 12299 + a1 + a4, sh);
}

JPEG_HD int jpeg_quantize(int c, uint32_t recip, int shift, int q) {
    const uint32_t a = (uint32_t)(c < 0 ? -c : c) + 4u * (uint32_t)q;
    const int v = (int)(((uint64_t)a * recip) >> shift);
    return c < 0 ? -v : v;
}

// ---- entropy coding -----------------------------------------------------------------------------------------------------------------
JPEG_HD int jpeg_nbits(int v) {                             // magnitude category: bits of |v|
    unsigned a = (unsigned)(v < 0 ? -v : v);
    int n = 0;
    while (a) { ++n; a >>= 1; }
    return n;
}
// code of a value of category n: v itself if positive, else v - 1 in n bits
JPEG_HD uint32_t jpeg_amp(int v, int n) { return (uint32_t)(v < 0 ? v - 1 : v) & ((1u << n) - 1u); }

// The bits of one DC difference (table 0 luma / 1 chroma), appended through emit(code, length).
template <class Emit>
JPEG_HD int jpeg_emit_dc(const JpegHuffCodes& H, int table, int diff, Emit& emit) {
    const int n = jpeg_nbits(diff);
    emit(H.code[table][n], H.size[table][n]);
    if (n) emit(jpeg_amp(diff, n), n);
    return H.size[table][n] + n;
}
// One non-zero AC coefficient v after `run` zeros (table 2 luma / 3 chroma): ZRLs, the run/size symbol, the amplitude bits.
template <class Emit>
JPEG_HD int jpeg_emit_ac(const JpegHuffCodes& H, int table, int run, int v, Emit& emit) {
    int bits = 0;
    for (; run > 15; run -= 16) { emit(H.code[table][0xF0], H.size[table][0xF0]); bits += H.size[table][0xF0]; }
    const int n = jpeg_nbits(v), sym = (run << 4) | n;
    emit(H.code[table][sym], H.size[table][sym]);
    emit(jpeg_amp(v, n), n);
    return bits + H.size[table][sym] + n;
}
template <class Emit>
JPEG_HD int jpeg_emit_eob(const JpegHuffCodes& H, int table, Emit& emit) {
    emit(H.code[table][0], H.size[table][0]);
    return H.size[table][0];
}
