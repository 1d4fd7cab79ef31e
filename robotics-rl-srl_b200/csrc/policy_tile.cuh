// The register-tiled 64-64 tower of the fused policy step (policy_kernels.cu: srl_policy_act) and its weight staging helpers, shared with the
// dueling Q forward of dqn_kernels.cu (srl_dqn_act, srl_dqn_target), which runs the same tile with ReLU instead of tanh.
#pragma once
#include <cuda_runtime.h>
#include "policy_core.h"

namespace {

constexpr int H = SRL_POLICY_HIDDEN;
constexpr int POLICY_LANES = 4;                   // threads per env in the last layer and for the per-env work
constexpr int POLICY_ENVS = 32;                   // envs per CTA -> 4096 envs = 128 CTAs of 128 threads (round 1: 64 CTAs of 64, one env per thread, slower)
constexpr int POLICY_BLOCK = POLICY_ENVS * POLICY_LANES;
constexpr int WS = H + 4;                         // padded row stride of the 64-wide rows: 16-byte aligned, and the 4 rows the lanes of an env read at
                                                  // the same time (o, o + 1, o + 2, o + 3) start 4 banks apart -- LDS.128 without bank conflicts

// Staging of the weights: every thread first ISSUES all of its global loads (registers), then stores them to shared memory -- one exposed
// L2 latency for the whole set instead of one per array (a load -> store loop per array paid one each, 12 arrays).
template <int PER>
struct RowRegs { float4 v[PER]; };
// 64-wide rows -> padded shared rows, 16 bytes per load; PER = ceil(rows * 16 / POLICY_BLOCK)
template <int PER>
__device__ __forceinline__ void rows_load(RowRegs<PER>& r, const float* __restrict__ src, int rows, bool vec) {
#pragma unroll
    for (int k = 0; k < PER; ++k) {
        const int i = threadIdx.x + k * POLICY_BLOCK;
        r.v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < rows * (H / 4)) {
            if (vec) r.v[k] = __ldg(reinterpret_cast<const float4*>(src) + i);
            else r.v[k] = make_float4(__ldg(src + 4 * i), __ldg(src + 4 * i + 1), __ldg(src + 4 * i + 2), __ldg(src + 4 * i + 3));   // a view at an odd offset
        }
    }
}
template <int PER>
__device__ __forceinline__ void rows_store(const RowRegs<PER>& r, float* dst, int rows) {
#pragma unroll
    for (int k = 0; k < PER; ++k) {
        const int i = threadIdx.x + k * POLICY_BLOCK;
        if (i < rows * (H / 4)) *reinterpret_cast<float4*>(dst + (i >> 4) * WS + 4 * (i & 15)) = r.v[k];
    }
}
template <int PER>
struct VecRegs { float v[PER]; };
template <int PER>
__device__ __forceinline__ void vec_load(VecRegs<PER>& r, const float* __restrict__ src, int count) {
#pragma unroll
    for (int k = 0; k < PER; ++k) {
        const int i = threadIdx.x + k * POLICY_BLOCK;
        r.v[k] = i < count ? __ldg(src + i) : 0.f;
    }
}
template <int PER>
__device__ __forceinline__ void vec_store(const VecRegs<PER>& r, float* dst, int count) {
#pragma unroll
    for (int k = 0; k < PER; ++k) {
        const int i = threadIdx.x + k * POLICY_BLOCK;
        if (i < count) dst[i] = r.v[k];
    }
}

struct TowerSmem { const float *w1, *b1, *w2, *b2, *w3, *b3; };

__device__ __forceinline__ void load_column(const float* h, float (&a)[H]) {
#pragma unroll
    for (int i4 = 0; i4 < H / 4; ++i4) {
        const float4 v = *reinterpret_cast<const float4*>(h + 4 * i4);
        a[4 * i4] = v.x; a[4 * i4 + 1] = v.y; a[4 * i4 + 2] = v.z; a[4 * i4 + 3] = v.w;
    }
}
// one padded 64-wide row against the activations: the four partial sums and their combination of policy_core.h's srl_mlp_tower
__device__ __forceinline__ float dot_row(const float* row, const float (&a)[H], float bias) {
    float s0 = bias, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
    for (int i4 = 0; i4 < H / 4; ++i4) {
        const float4 w = *reinterpret_cast<const float4*>(row + 4 * i4);
        s0 = fmaf(w.x, a[4 * i4 + 0], s0); s1 = fmaf(w.y, a[4 * i4 + 1], s1);
        s2 = fmaf(w.z, a[4 * i4 + 2], s2); s3 = fmaf(w.w, a[4 * i4 + 3], s3);
    }
    return (s0 + s1) + (s2 + s3);
}

// One 64-64 tower for the CTA's 32 envs: same arithmetic, value by value, as srl_mlp_tower (policy_core.h) -- per output the four partial sums
// over i4 = 0..15 in order, then (s0 + s1) + (s2 + s3).  Layers 1 and 2 are REGISTER-TILED: thread t owns 4 envs (4 (t / 16) + 0..3) x 4
// outputs ((t % 16) + 0, 16, 32, 48) -- per 4 inputs it loads 4 weight quads + 4 activation quads (8 LDS.128) for 64 FFMA into 64 independent
// accumulators.  (One env's 16 outputs per thread needed 1 LDS.128 per 4 FFMA and was bound by the shared-memory pipe: ncu: most of the
// stalls on the first FFMA after a weight load.)  The 8 lanes of a quarter-warp read 8 consecutive weight
// rows (stride WS = 68 words: 8 different 4-bank groups) and one common activation quad (broadcast).  `xs` [32][MO] observations, `ha` / `hb`
// [32][WS] activation columns (layer 1 -> ha, layer 2 -> hb), `out` [32][stride] receives the last layer (thread t: env t / 4, outputs t % 4 + 4 k).
// MO = SRL_POLICY_MAX_OBS: W1 is [64][D], one input per step.  MO = SRL_POLICY_WIDE_OBS: W1 rows are padded to w1_stride<MO>() = MO + 4 words and
// both W1 and `xs` rows are zero past D, so layer 1 takes 4 inputs per step (one LDS.128 per weight row and per env) for any D; the FMA chain per
// output is still d = 0, 1, ... in order, and the padded inputs add 0 * 0.
template <int MO>
__host__ __device__ constexpr int w1_stride() { return MO == SRL_POLICY_MAX_OBS ? MO : MO + 4; }
// RELU: max(x, 0) after layers 1 and 2 (the dueling Q towers of dqn_kernels.cu) instead of tanh.
template <int MO, bool RELU = false>
__device__ __forceinline__ void tower_tiled(const TowerSmem& W, int D, int n_out, const float* xs, float* ha, float* hb, float* out, int out_stride) {
    const int t = threadIdx.x, eg = t >> 4, og = t & 15;
    {   // layer 1: obs_dim -> 64
        float acc[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[e][k] = W.b1[og + 16 * k];
        if constexpr (MO == SRL_POLICY_MAX_OBS) {
            for (int d = 0; d < D; ++d) {
                float w[4], x[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) w[k] = W.w1[(og + 16 * k) * D + d];
#pragma unroll
                for (int e = 0; e < 4; ++e) x[e] = xs[(4 * eg + e) * SRL_POLICY_MAX_OBS + d];
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int k = 0; k < 4; ++k) acc[e][k] = fmaf(w[k], x[e], acc[e][k]);
            }
        } else {
            for (int d4 = 0; d4 < D; d4 += 4) {
                float4 w[4], x[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) w[k] = *reinterpret_cast<const float4*>(W.w1 + (og + 16 * k) * w1_stride<MO>() + d4);
#pragma unroll
                for (int e = 0; e < 4; ++e) x[e] = *reinterpret_cast<const float4*>(xs + (4 * eg + e) * MO + d4);
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        acc[e][k] = fmaf(w[k].x, x[e].x, acc[e][k]); acc[e][k] = fmaf(w[k].y, x[e].y, acc[e][k]);
                        acc[e][k] = fmaf(w[k].z, x[e].z, acc[e][k]); acc[e][k] = fmaf(w[k].w, x[e].w, acc[e][k]);
                    }
            }
        }
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int k = 0; k < 4; ++k) ha[(4 * eg + e) * WS + og + 16 * k] = RELU ? fmaxf(acc[e][k], 0.f) : tanhf(acc[e][k]);
    }
    __syncthreads();
    {   // layer 2: 64 -> 64
        float s[4][4][4];
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int k = 0; k < 4; ++k) { s[e][k][0] = W.b2[og + 16 * k]; s[e][k][1] = 0.f; s[e][k][2] = 0.f; s[e][k][3] = 0.f; }
#pragma unroll 2
        for (int i4 = 0; i4 < H / 4; ++i4) {
            float4 w[4], a[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) w[k] = *reinterpret_cast<const float4*>(W.w2 + (og + 16 * k) * WS + 4 * i4);
#pragma unroll
            for (int e = 0; e < 4; ++e) a[e] = *reinterpret_cast<const float4*>(ha + (4 * eg + e) * WS + 4 * i4);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    s[e][k][0] = fmaf(w[k].x, a[e].x, s[e][k][0]); s[e][k][1] = fmaf(w[k].y, a[e].y, s[e][k][1]);
                    s[e][k][2] = fmaf(w[k].z, a[e].z, s[e][k][2]); s[e][k][3] = fmaf(w[k].w, a[e].w, s[e][k][3]);
                }
        }
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float z = (s[e][k][0] + s[e][k][1]) + (s[e][k][2] + s[e][k][3]);
                hb[(4 * eg + e) * WS + og + 16 * k] = RELU ? fmaxf(z, 0.f) : tanhf(z);
            }
    }
    __syncthreads();
    {   // layer 3: 64 -> n_out (<= 8): thread t -> env t / 4, outputs t % 4 and t % 4 + 4
        const int e = t >> 2, u = t & 3;
        if (u < n_out) {
            float a[H];
            load_column(hb + e * WS, a);
            for (int k = u; k < n_out; k += POLICY_LANES) out[e * out_stride + k] = dot_row(W.w3 + k * WS, a, W.b3[k]);
        }
    }
}

}  // namespace
