// PPO2 minibatch gradient in one pass (include/srl_policy.h: srl_ppo2_grad) -- the optimiser phase of the GPU-resident PPO2 consumer
// (SURVEY.md 8(f).1; the reference trains through stable-baselines' PPO2 with MlpPolicy, rl_baselines/rl_algorithm/ppo2.py:58-72).
//
// What it replaces: torch autograd over a 131 072-sample minibatch of config 3 -- ~150 launches, every activation of both 64-64 towers
// written to and read back from HBM / L2 (33 MB per [mb, 64] tensor), the larger part of a PPO2 update even when captured in a CUDA
// graph.  Here a persistent CTA keeps the weights (and W2 transposed) in shared
// memory, walks its share of the minibatch in chunks of 64 samples, and for each chunk runs forward -> PPO2 loss derivative -> backward with
// every activation in shared memory and the weight gradients accumulating in registers; the per-CTA partial gradients are summed in a fixed
// order by a second kernel (deterministic: no atomics).  Gradient clipping and Adam stay with torch (a dozen launches over 9.3 k parameters).
//
// The loss is stable-baselines' PPO2 loss as rl_baselines/ppo2.py states it (its `minibatch_step` is the torch reference of the tests):
//   A_n = (adv_n - mean) / (std + 1e-8) over the minibatch (std unbiased), ratio = exp(logp - old_logp),
//   pg = mean(max(-A ratio, -A clip(ratio, 1 - c, 1 + c))), vf = 0.5 mean(max((v - R)^2, (old_v + clip(v - old_v, -c, c) - R)^2)),
//   loss = pg - ent_coef mean(entropy) + vf_coef vf.
#include <cuda_runtime.h>
#include <math.h>
#include "common.cuh"
#include "../../include/srl_policy.h"

namespace {

constexpr int H = 64, WS = 68, CH = 64, NT = 256, MAXO = 8, MAXD = 8;      // 64 samples per chunk, 8 warps per CTA (two per scheduler)
constexpr int WIDE_D = 32;     // the wide instantiation: observation widths 9..32 (stacked states)
static_assert(NT == 4 * CH && NT == 256, "thread roles: 4 threads per sample in the heads, 128 owners per tower of the W2 gradient patches");

// offsets of the parameter tensors inside a flat gradient vector (the order of the per-CTA partials)
struct Seg { int pw1, pb1, pw2, pb2, pw3, pb3, vw1, vb1, vw2, vb2, vw3, vb3, ls, P; };
__host__ __device__ inline Seg make_seg(int D, int A, int discrete) {
    Seg s; int o = 0;
    s.pw1 = o; o += H * D; s.pb1 = o; o += H; s.pw2 = o; o += H * H; s.pb2 = o; o += H; s.pw3 = o; o += A * H; s.pb3 = o; o += A;
    s.vw1 = o; o += H * D; s.vb1 = o; o += H; s.vw2 = o; o += H * H; s.vb2 = o; o += H; s.vw3 = o; o += H; s.vb3 = o; o += 1;
    s.ls = o; o += discrete ? 0 : A; s.P = o;
    return s;
}

struct GradArgs {
    srl_mlp_policy p;
    int mb;
    const long long* idx; const float* obs; const void* act; const float* adv; const float* ret; const float* old_logp; const float* old_val;
    float clip, ent_coef, vf_coef;
    const double* stats;      // STATS_CTAS x {sum(x - shift), sum((x - shift)^2)}, then the shift: the minibatch's advantages
    float* partial;           // [gridDim.x][P]
    float* td;                // DQN: per-sample TD error out, [mb] in batch order
};

// ---- advantage statistics of the minibatch: STATS_CTAS partial sums (float64, about the first element: no cancellation), combined in a fixed
//      order by every CTA of the gradient kernel (a single CTA gathering 131 072 elements was slow) ----
constexpr int STATS_CTAS = 64, STATS_NT = 256;
__global__ void __launch_bounds__(STATS_NT) adv_stats_kernel(int mb, const long long* __restrict__ idx, const float* __restrict__ adv, double* __restrict__ part) {
    __shared__ double red[STATS_NT / 32][2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double shift = (double)adv[idx ? idx[0] : 0];
    double s1 = 0.0, s2 = 0.0;
    for (int e0 = blockIdx.x * STATS_NT + tid; e0 < mb; e0 += 8 * STATS_CTAS * STATS_NT) {
        float x[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) { const int e = e0 + k * STATS_CTAS * STATS_NT; x[k] = e < mb ? adv[idx ? idx[e] : e] : 0.f; }
#pragma unroll
        for (int k = 0; k < 8; ++k) if (e0 + k * STATS_CTAS * STATS_NT < mb) { const double c = (double)x[k] - shift; s1 += c; s2 = fma(c, c, s2); }
    }
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if (lane == 0) { red[warp][0] = s1; red[warp][1] = s2; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < STATS_NT / 32; ++w) { s1 += red[w][0]; s2 += red[w][1]; }
        part[2 * blockIdx.x] = s1; part[2 * blockIdx.x + 1] = s2;
        if (blockIdx.x == 0) part[2 * STATS_CTAS] = shift;
    }
}

// out[n][o] for the thread's 4 samples (4 eg + e) x 4 units (og + 16 k): bias[o] + sum_i W[o][i] in[n][i], W rows padded to WS words.
// Four partial sums per output over the 16 input quads, as csrc/policy_core.h's tower does.
__device__ __forceinline__ void tile_matvec(const float* W, const float* bias, const float* in, int eg, int og, float (&out)[4][4]) {
    float s[4][4][4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int k = 0; k < 4; ++k) { s[e][k][0] = bias ? bias[og + 16 * k] : 0.f; s[e][k][1] = 0.f; s[e][k][2] = 0.f; s[e][k][3] = 0.f; }
#pragma unroll 2
    for (int i4 = 0; i4 < H / 4; ++i4) {
        float4 w[4], a[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) w[k] = *reinterpret_cast<const float4*>(W + (og + 16 * k) * WS + 4 * i4);
#pragma unroll
        for (int e = 0; e < 4; ++e) a[e] = *reinterpret_cast<const float4*>(in + (4 * eg + e) * WS + 4 * i4);
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
        for (int k = 0; k < 4; ++k) out[e][k] = (s[e][k][0] + s[e][k][1]) + (s[e][k][2] + s[e][k][3]);
}

__device__ __forceinline__ float dot64(const float* row, const float* col) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
    for (int i4 = 0; i4 < H / 4; ++i4) {
        const float4 w = *reinterpret_cast<const float4*>(row + 4 * i4), a = *reinterpret_cast<const float4*>(col + 4 * i4);
        s0 = fmaf(w.x, a.x, s0); s1 = fmaf(w.y, a.y, s1); s2 = fmaf(w.z, a.z, s2); s3 = fmaf(w.w, a.w, s3);
    }
    return (s0 + s1) + (s2 + s3);
}

// the loss a gradient kernel instantiation differentiates (srl_ppo2_grad, srl_a2c_grad, srl_dqn_grad)
enum LossKind { PPO2_LOSS, A2C_LOSS, DQN_LOSS };

struct SampleRegs { float x[MAXD], af[MAXO], adv, ret, olp, ov; int ai, valid; };

template <bool LOAD_X, int L>
__device__ __forceinline__ void load_sample(const GradArgs& a, int s, SampleRegs& r) {
    const int D = a.p.obs_dim, A = a.p.n_out;
    r.valid = s < a.mb;
    const long long g = r.valid ? (a.idx ? a.idx[s] : (long long)s) : 0;
    if constexpr (LOAD_X) {
#pragma unroll
        for (int d = 0; d < MAXD; ++d) r.x[d] = (r.valid && d < D) ? a.obs[g * D + d] : 0.f;
    }
    r.ai = 0;
#pragma unroll
    for (int k = 0; k < MAXO; ++k) r.af[k] = 0.f;
    if (r.valid) {
        if (a.p.discrete) r.ai = (int)reinterpret_cast<const long long*>(a.act)[g];
        else {
#pragma unroll
            for (int k = 0; k < MAXO; ++k) if (k < A) r.af[k] = reinterpret_cast<const float*>(a.act)[g * A + k];
        }
    }
    if constexpr (L == A2C_LOSS) { r.adv = 0.f; r.ret = r.valid ? a.ret[g] : 0.f; r.olp = 0.f; r.ov = r.valid ? a.old_val[g] : 0.f; }   // advantage: ret - old_val
    else if constexpr (L == DQN_LOSS) {    // ret: the target y, ov: the importance weight (NULL: 1); both in batch order, not row order
        r.adv = 0.f; r.ret = r.valid ? a.ret[s] : 0.f; r.olp = 0.f; r.ov = r.valid ? (a.old_val ? a.old_val[s] : 1.f) : 0.f;
    }
    else { r.adv = r.valid ? a.adv[g] : 0.f; r.ret = r.valid ? a.ret[g] : 0.f; r.olp = r.valid ? a.old_logp[g] : 0.f; r.ov = r.valid ? a.old_val[g] : 0.f; }
}

// The wide instantiation (MD = WIDE_D) differs from the narrow one (MD = MAXD) in three places, all to fit shared memory and registers:
//  - W1 rows are padded to MD + 1 words (the 16 units a layer-1 step reads sit in 16 different banks), `xs` rows are MD wide;
//  - a chunk's observation rows are prefetched by all 256 threads (thread t: sample t / 4, columns t % 4 + 4 j), 8 registers each, instead of
//    a [MD] array in the 64 sample threads' SampleRegs (32 more registers there would spill);
//  - the first-layer deltas d1 overwrite the second-layer activations hb, which are dead once the layer-3 gradients are taken: one more barrier
//    per chunk, 34 KB less shared memory (the wider W1 copies and rows need 18 KB more than the narrow kernel's 224 KB leave).
// the wide kernel's observation prefetch: columns u + 4 j (j < XQ) of sample s, zero past D and past the minibatch
template <int XQ>
__device__ __forceinline__ void load_row_part(const GradArgs& a, int s, int u, float (&x)[XQ]) {
    const int D = a.p.obs_dim;
    const bool valid = s < a.mb;
    const long long g = valid ? (a.idx ? a.idx[s] : (long long)s) : 0;
#pragma unroll
    for (int j = 0; j < XQ; ++j) x[j] = (valid && u + 4 * j < D) ? a.obs[g * D + u + 4 * j] : 0.f;
}

// hidden activation of the towers and its derivative from the activation h: tanh (1 - h^2), or ReLU (TF's gradient: 0 where the
// pre-activation is <= 0, i.e. where h = 0)
template <int L>
__device__ __forceinline__ float act_fn(float x) { if constexpr (L == DQN_LOSS) return fmaxf(x, 0.f); else return tanhf(x); }
template <int L>
__device__ __forceinline__ float dact_fn(float d, float h) { if constexpr (L == DQN_LOSS) return h > 0.f ? d : 0.f; else return d * (1.0f - h * h); }

template <int MD>
__host__ __device__ constexpr int grad_w1_stride() { return MD == MAXD ? MAXD : MD + 1; }
// A2C_LOSS: the loss of srl_a2c_grad instead of PPO2's (stage 2 only; no advantage statistics, no clip ratio, no value clip).
// DQN_LOSS: srl_dqn_grad's dueling Q loss (stage 2) and ReLU instead of tanh (forward, and its derivative in stages 3 and 4).
template <int MD, int L>
__device__ __forceinline__ void ppo2_grad_cta(const GradArgs& a) {
    constexpr bool WIDE = MD != MAXD;
    constexpr int W1S = grad_w1_stride<MD>(), XQ = MD / 4;     // XQ: observation columns per thread of the wide prefetch
    constexpr int G1 = WIDE ? (H * MD) / NT : 4;              // W1 gradient entries per thread
    extern __shared__ __align__(16) float sm[];
    const int D = a.p.obs_dim, A = a.p.n_out, t = threadIdx.x;
    const bool discrete = a.p.discrete != 0;
    const Seg seg = make_seg(D, A, a.p.discrete);
    // ---- shared memory map (floats) ----
    float* w2p = sm;                 float* w2v = w2p + H * WS;       float* w2pT = w2v + H * WS;      float* w2vT = w2pT + H * WS;
    float* w3p = w2vT + H * WS;      float* w3v = w3p + MAXO * WS;
    float* hap = w3v + WS;           float* hbp = hap + CH * WS;      float* hav = hbp + CH * WS;      float* hbv = hav + CH * WS;
    float* d2p = hbv + CH * WS;      float* d2v = d2p + CH * WS;
    float* d1p = WIDE ? hbp : d2v + CH * WS;                          float* d1v = WIDE ? hbv : d1p + CH * WS;
    float* w1p = WIDE ? d2v + CH * WS : d1v + CH * WS;                float* w1v = w1p + H * W1S;
    float* b1p = w1v + H * W1S;      float* b1v = b1p + H;            float* b2p = b1v + H;            float* b2v = b2p + H;
    float* b3p = b2v + H;            float* b3v = b3p + MAXO;         float* lsd = b3v + 4;            // logstd
    float* xs = lsd + MAXO;          // [CH][MD]
    float* zo = xs + CH * MD;        // [CH][MAXO + 1]: logits / mean, value at [MAXO]
    float* d3 = zo + CH * (MAXO + 1);   // [CH][MAXO + 1]: d loss / d logits, d loss / d value
    float* dls = d3 + CH * (MAXO + 1);  // [CH][MAXO]: per-sample d loss / d logstd
    float* saf = dls + CH * MAXO;    // [CH][MAXO] actions (Box)
    float* ssc = saf + CH * MAXO;    // [CH][4]: adv, ret, old_logp, old_val
    int* sai = reinterpret_cast<int*>(ssc + CH * 4);   // [CH][2]: action (Discrete), valid
    // ---- weights, once per CTA ----
    for (int e = t; e < H * H; e += NT) {
        const int j = e >> 6, i = e & 63;
        const float wp = a.p.pi_w2[e], wv = a.p.vf_w2[e];
        w2p[j * WS + i] = wp; w2pT[i * WS + j] = wp; w2v[j * WS + i] = wv; w2vT[i * WS + j] = wv;
    }
    for (int e = t; e < A * H; e += NT) w3p[(e >> 6) * WS + (e & 63)] = a.p.pi_w3[e];
    for (int e = t; e < H; e += NT) {
        w3v[e] = a.p.vf_w3[e];
        b1p[e] = a.p.pi_b1[e]; b1v[e] = a.p.vf_b1[e]; b2p[e] = a.p.pi_b2[e]; b2v[e] = a.p.vf_b2[e];
    }
    for (int e = t; e < H * D; e += NT) { w1p[(e / D) * W1S + e % D] = a.p.pi_w1[e]; w1v[(e / D) * W1S + e % D] = a.p.vf_w1[e]; }
    if (t < A) { b3p[t] = a.p.pi_b3[t]; lsd[t] = discrete ? 0.f : a.p.logstd[t]; }
    if (t == 0) b3v[0] = a.p.vf_b3[0];
    __shared__ float s_adv[2];
    if (L == PPO2_LOSS && t < 32) {                  // mean and 1 / (std + 1e-8) (torch.std(): unbiased) from the partial sums, in a fixed order
        double s1 = a.stats[2 * t] + a.stats[2 * (t + 32)], s2 = a.stats[2 * t + 1] + a.stats[2 * (t + 32) + 1];
        for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
        if (t == 0) {
            const double n = (double)a.mb, mean = a.stats[2 * STATS_CTAS] + s1 / n;
            const double var = a.mb > 1 ? fmax((s2 - s1 * s1 / n) / (n - 1.0), 0.0) : 0.0;
            s_adv[0] = (float)mean; s_adv[1] = (float)(1.0 / (sqrt(var) + 1e-8));
        }
    }
    __syncthreads();
    const float amean = L != PPO2_LOSS ? 0.f : s_adv[0], ainv = L != PPO2_LOSS ? 0.f : s_adv[1], inv_mb = 1.0f / (float)a.mb;
    // ---- gradient accumulators (registers; every entry of the flat gradient has exactly one owner thread) ----
    const int eg = t >> 4, og = t & 15;          // forward / delta tiles: samples 4 eg + e, units og + 16 k
    const bool own_pi = t < 128;                 // W2 gradient: threads 0..127 own the policy tower's 4 x 8 patches, 128..255 the value tower's
    const int jq = (t & 127) >> 3, iq = t & 7;   // rows 4 jq + jj, columns 8 iq + ii
    float gw2[4][8];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int ii = 0; ii < 8; ++ii) gw2[jj][ii] = 0.f;
    float gw3p[4] = {0.f, 0.f, 0.f, 0.f}, gw1p[G1], gw1v[G1];
#pragma unroll
    for (int m = 0; m < G1; ++m) { gw1p[m] = 0.f; gw1v[m] = 0.f; }
    float gw3v = 0.f, gb3 = 0.f, gls = 0.f, gb2 = 0.f, gb1 = 0.f;       // gb2 / gb1: t < 64 the policy tower's unit t, t >= 64 the value tower's unit t - 64
    const int nchunks = (a.mb + CH - 1) / CH;
    SampleRegs cur;
    float xr[XQ];                                // wide: this thread's columns t % 4 + 4 j of sample t / 4 of the next chunk
    if (t < CH) load_sample<!WIDE, L>(a, blockIdx.x * CH + t, cur);
    if constexpr (WIDE) load_row_part<XQ>(a, blockIdx.x * CH + (t >> 2), t & 3, xr);
    __syncthreads();
    for (int c = blockIdx.x; c < nchunks; c += gridDim.x) {
        // ---- 0: this chunk's samples -> shared; the next chunk's loads are issued now and consumed an iteration later ----
        if (t < CH) {
            if constexpr (!WIDE) {
#pragma unroll
                for (int d = 0; d < MAXD; ++d) xs[t * MAXD + d] = cur.x[d];
            }
#pragma unroll
            for (int k = 0; k < MAXO; ++k) saf[t * MAXO + k] = cur.af[k];
            ssc[t * 4] = cur.adv; ssc[t * 4 + 1] = cur.ret; ssc[t * 4 + 2] = cur.olp; ssc[t * 4 + 3] = cur.ov;
            sai[t * 2] = cur.ai; sai[t * 2 + 1] = cur.valid;
            load_sample<!WIDE, L>(a, (c + gridDim.x) * CH + t, cur);
        }
        if constexpr (WIDE) {
#pragma unroll
            for (int j = 0; j < XQ; ++j) xs[(t >> 2) * MD + (t & 3) + 4 * j] = xr[j];
            load_row_part<XQ>(a, (c + gridDim.x) * CH + (t >> 2), t & 3, xr);
        }
        __syncthreads();
        // ---- 1: forward, both towers ----
        {
            float accp[4][4], accv[4][4];
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int e = 0; e < 4; ++e) { accp[e][k] = b1p[og + 16 * k]; accv[e][k] = b1v[og + 16 * k]; }
            for (int d = 0; d < D; ++d) {
                float wp[4], wv[4], x[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) { wp[k] = w1p[(og + 16 * k) * W1S + d]; wv[k] = w1v[(og + 16 * k) * W1S + d]; }
#pragma unroll
                for (int e = 0; e < 4; ++e) x[e] = xs[(4 * eg + e) * MD + d];
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int k = 0; k < 4; ++k) { accp[e][k] = fmaf(wp[k], x[e], accp[e][k]); accv[e][k] = fmaf(wv[k], x[e], accv[e][k]); }
            }
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) { hap[(4 * eg + e) * WS + og + 16 * k] = act_fn<L>(accp[e][k]); hav[(4 * eg + e) * WS + og + 16 * k] = act_fn<L>(accv[e][k]); }
        }
        __syncthreads();
        {
            float o[4][4];
            tile_matvec(w2p, b2p, hap, eg, og, o);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) hbp[(4 * eg + e) * WS + og + 16 * k] = act_fn<L>(o[e][k]);
            tile_matvec(w2v, b2v, hav, eg, og, o);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) hbv[(4 * eg + e) * WS + og + 16 * k] = act_fn<L>(o[e][k]);
        }
        __syncthreads();
        {   // heads: thread t -> sample t / 4; outputs t % 4 and t % 4 + 4 of the policy head, the value by lane 3 of the sample's four
            const int n = t >> 2, u = t & 3;
            for (int k = u; k < A; k += 4) zo[n * (MAXO + 1) + k] = b3p[k] + dot64(w3p + k * WS, hbp + n * WS);
            if (u == 3) zo[n * (MAXO + 1) + MAXO] = b3v[0] + dot64(w3v, hbv + n * WS);
        }
        __syncthreads();
        // ---- 2: d loss / d outputs, one thread per sample ----
        if (t < CH) {
            const int n = t, row0 = c * CH;            // row0: the chunk's first sample (`c` is the clip range below)
            float z[MAXO], g[MAXO];
#pragma unroll
            for (int k = 0; k < MAXO; ++k) { z[k] = k < A ? zo[n * (MAXO + 1) + k] : 0.f; g[k] = 0.f; }
            const float v = zo[n * (MAXO + 1) + MAXO];
            const float adv = ssc[n * 4], R = ssc[n * 4 + 1], olp = ssc[n * 4 + 2], ov = ssc[n * 4 + 3];
            const bool valid = sai[n * 2 + 1] != 0;
            const float An = (adv - amean) * ainv, c = a.clip;
            float gv = 0.f, gl[MAXO];
#pragma unroll
            for (int k = 0; k < MAXO; ++k) gl[k] = 0.f;
            if (valid && L != DQN_LOSS) {
                float logp;
                float p[MAXO], lse = 0.f, Hent = 0.f;
                if (discrete) {
                    float m = z[0];
#pragma unroll
                    for (int k = 1; k < MAXO; ++k) if (k < A) m = fmaxf(m, z[k]);
                    float S = 0.f;
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) { p[k] = k < A ? expf(z[k] - m) : 0.f; S += p[k]; }
                    lse = m + logf(S);
                    const float iS = 1.0f / S;
                    float pz = 0.f, za = 0.f;
                    const int ai = sai[n * 2];
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) { p[k] *= iS; pz = fmaf(p[k], z[k], pz); if (k == ai) za = z[k]; }
                    Hent = lse - pz;
                    logp = za - lse;
                } else {
                    logp = 0.f;
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) if (k < A) {
                        const float is = expf(-lsd[k]), u = (saf[n * MAXO + k] - z[k]) * is;
                        logp += -0.5f * u * u - lsd[k] - 0.91893853320467274178f;
                        p[k] = u;                      // (a - mu) / sigma, reused below
                    }
                }
                float dlogp;
                if constexpr (L == A2C_LOSS) {
                    dlogp = -(R - ov) * inv_mb;                                         // pg_loss = mean(-(R - V) logp)
                } else {
                    const float ratio = expf(logp - olp);
                    const float rc = fminf(fmaxf(ratio, 1.0f - c), 1.0f + c);
                    const float unclipped = -An * ratio, clipped = -An * rc;
                    const float dr = (rc == ratio || unclipped > clipped) ? -An : 0.f;  // max(): the live branch (a tie inside the clip range sums to the same)
                    dlogp = dr * ratio * inv_mb;
                }
                if (discrete) {
                    const int ai = sai[n * 2];
                    const float ec = a.ent_coef * inv_mb;
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) if (k < A) g[k] = dlogp * ((k == ai ? 1.f : 0.f) - p[k]) + ec * p[k] * ((z[k] - lse) + Hent);
                } else {
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) if (k < A) {
                        const float is = expf(-lsd[k]);
                        g[k] = dlogp * p[k] * is;                                   // d logp / d mu = (a - mu) / sigma^2
                        gl[k] = dlogp * (p[k] * p[k] - 1.0f) - a.ent_coef * inv_mb;     // d logp / d logstd; entropy = sum(logstd) + const
                    }
                }
                if constexpr (L == A2C_LOSS) {
                    gv = v - R;                                                         // vf_loss = 0.5 mean((v - R)^2)
                } else {
                    const float dv = v - ov, dvc = fminf(fmaxf(dv, -c), c);
                    const float e1 = v - R, e2 = (ov + dvc) - R;
                    const float l1 = e1 * e1, l2 = e2 * e2;
                    gv = (dvc == dv || l1 > l2) ? e1 : (l1 == l2 ? 0.5f * e1 : 0.f);
                }
                gv *= a.vf_coef * inv_mb;
            }
            if constexpr (L == DQN_LOSS) {          // Q = V + A - mean(A), td = Q(s, a) - y, loss = mean(w huber(td)), huber with delta = 1
                if (valid) {
                    const int ai = sai[n * 2];
                    float sa = 0.f, za = 0.f;
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) if (k < A) { sa += z[k]; if (k == ai) za = z[k]; }
                    const float inv_a = 1.0f / (float)A;
                    const float td = (v + (za - sa * inv_a)) - R;
                    a.td[row0 + n] = td;
                    const float gq = ov * fminf(fmaxf(td, -1.0f), 1.0f) * inv_mb;      // d loss / d Q(s, a)
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) if (k < A) g[k] = gq * ((k == ai ? 1.f : 0.f) - inv_a);
                    gv = gq;
                }
            }
#pragma unroll
            for (int k = 0; k < MAXO; ++k) { d3[n * (MAXO + 1) + k] = g[k]; dls[n * MAXO + k] = gl[k]; }
            d3[n * (MAXO + 1) + MAXO] = gv;
        }
        __syncthreads();
        // ---- 3: delta of the second hidden layer (pre-activation), both towers ----
        {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int n = 4 * eg + e;
                float gz[MAXO];
#pragma unroll
                for (int k = 0; k < MAXO; ++k) gz[k] = d3[n * (MAXO + 1) + k];
                const float gvn = d3[n * (MAXO + 1) + MAXO];
#pragma unroll
                for (int k4 = 0; k4 < 4; ++k4) {
                    const int j = og + 16 * k4;
                    float s = 0.f;
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) if (k < A) s = fmaf(w3p[k * WS + j], gz[k], s);
                    const float hp = hbp[n * WS + j], hv = hbv[n * WS + j];
                    d2p[n * WS + j] = dact_fn<L>(s, hp);
                    d2v[n * WS + j] = dact_fn<L>(w3v[j] * gvn, hv);
                }
            }
        }
        __syncthreads();
        // ---- 4: gradients of layers 3 and 2; delta of the first hidden layer ----
        {
            for (int m = 0; m < 4; ++m) {            // policy head weights: entries t + 128 m of [A][64]
                const int e = t + NT * m;
                if (e < A * H) {
                    const int k = e >> 6, j = e & 63;
                    float s = 0.f;
#pragma unroll 8
                    for (int n = 0; n < CH; ++n) s = fmaf(d3[n * (MAXO + 1) + k], hbp[n * WS + j], s);
                    gw3p[m] += s;
                }
            }
            if (t < H) {
                float s = 0.f, sb = 0.f;
#pragma unroll 8
                for (int n = 0; n < CH; ++n) { s = fmaf(d3[n * (MAXO + 1) + MAXO], hbv[n * WS + t], s); sb += d2p[n * WS + t]; }
                gw3v += s; gb2 += sb;
            } else if (t < 2 * H) {
                float sb = 0.f;
#pragma unroll 8
                for (int n = 0; n < CH; ++n) sb += d2v[n * WS + (t - H)];
                gb2 += sb;
            }
            if (t < A || t == MAXO) {                 // head biases: t < A the policy's, t == 8 the value's
                float s = 0.f;
                const int col = t < A ? t : MAXO;
                for (int n = 0; n < CH; ++n) s += d3[n * (MAXO + 1) + col];
                gb3 += s;
            }
            if (!discrete && t >= 16 && t < 16 + A) {
                float s = 0.f;
                for (int n = 0; n < CH; ++n) s += dls[n * MAXO + (t - 16)];
                gls += s;
            }
            // W2 gradient patches: per sample one delta quad and two activation quads
            {
                const float* dsrc = own_pi ? d2p : d2v;
                const float* hsrc = own_pi ? hap : hav;
#pragma unroll 4
                for (int n = 0; n < CH; ++n) {
                    const float4 dq = *reinterpret_cast<const float4*>(dsrc + n * WS + 4 * jq);
                    const float4 h0 = *reinterpret_cast<const float4*>(hsrc + n * WS + 8 * iq), h1 = *reinterpret_cast<const float4*>(hsrc + n * WS + 8 * iq + 4);
                    const float dd[4] = {dq.x, dq.y, dq.z, dq.w}, hh[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                        for (int ii = 0; ii < 8; ++ii) gw2[jj][ii] = fmaf(dd[jj], hh[ii], gw2[jj][ii]);
                }
            }
            if constexpr (WIDE) __syncthreads();        // d1 overwrites hb: every read of hb above comes first
            // delta 1 = (W2^T delta 2) (1 - h1^2): the same tile as the forward pass, on the transposed weights
            float o[4][4];
            tile_matvec(w2pT, nullptr, d2p, eg, og, o);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) { const float h = hap[(4 * eg + e) * WS + og + 16 * k]; d1p[(4 * eg + e) * WS + og + 16 * k] = dact_fn<L>(o[e][k], h); }
            tile_matvec(w2vT, nullptr, d2v, eg, og, o);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) { const float h = hav[(4 * eg + e) * WS + og + 16 * k]; d1v[(4 * eg + e) * WS + og + 16 * k] = dact_fn<L>(o[e][k], h); }
        }
        __syncthreads();
        // ---- 5: gradients of layer 1 ----
        {
            if (t < 2 * H) {
                const float* d1 = t < H ? d1p : d1v;
                const int unit = t < H ? t : t - H;
                float sb = 0.f;
#pragma unroll 8
                for (int n = 0; n < CH; ++n) sb += d1[n * WS + unit];
                gb1 += sb;
            }
#pragma unroll
            for (int m = 0; m < G1; ++m) {
                const int e = t + NT * m;
                if (e < H * D) {
                    const int i = e / D, d = e % D;
                    float sp = 0.f, sv = 0.f;
#pragma unroll 8
                    for (int n = 0; n < CH; ++n) { const float x = xs[n * MD + d]; sp = fmaf(d1p[n * WS + i], x, sp); sv = fmaf(d1v[n * WS + i], x, sv); }
                    gw1p[m] += sp; gw1v[m] += sv;
                }
            }
        }
        __syncthreads();
    }
    // ---- this CTA's partial gradient ----
    float* out = a.partial + (size_t)blockIdx.x * seg.P;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int ii = 0; ii < 8; ++ii) out[(own_pi ? seg.pw2 : seg.vw2) + (4 * jq + jj) * H + 8 * iq + ii] = gw2[jj][ii];
    if constexpr (!WIDE) {
        for (int m = 0; m < 4; ++m) {
            const int e = t + NT * m;
            if (e < A * H) out[seg.pw3 + e] = gw3p[m];
            if (e < H * D) { out[seg.pw1 + e] = gw1p[m]; out[seg.vw1 + e] = gw1v[m]; }
        }
    } else {
        for (int m = 0; m < 4; ++m) {
            const int e = t + NT * m;
            if (e < A * H) out[seg.pw3 + e] = gw3p[m];
        }
#pragma unroll
        for (int m = 0; m < G1; ++m) {
            const int e = t + NT * m;
            if (e < H * D) { out[seg.pw1 + e] = gw1p[m]; out[seg.vw1 + e] = gw1v[m]; }
        }
    }
    if (t < H) { out[seg.vw3 + t] = gw3v; out[seg.pb2 + t] = gb2; out[seg.pb1 + t] = gb1; }
    else if (t < 2 * H) { out[seg.vb2 + (t - H)] = gb2; out[seg.vb1 + (t - H)] = gb1; }
    if (t < A) out[seg.pb3 + t] = gb3;
    if (t == MAXO) out[seg.vb3] = gb3;
    if (!discrete && t >= 16 && t < 16 + A) out[seg.ls + (t - 16)] = gls;
}

__global__ void __launch_bounds__(NT, 1) ppo2_grad_kernel(const __grid_constant__ GradArgs a) { ppo2_grad_cta<MAXD, PPO2_LOSS>(a); }
__global__ void __launch_bounds__(NT, 1) ppo2_grad_wide_kernel(const __grid_constant__ GradArgs a) { ppo2_grad_cta<WIDE_D, PPO2_LOSS>(a); }
__global__ void __launch_bounds__(NT, 1) a2c_grad_kernel(const __grid_constant__ GradArgs a) { ppo2_grad_cta<MAXD, A2C_LOSS>(a); }
__global__ void __launch_bounds__(NT, 1) a2c_grad_wide_kernel(const __grid_constant__ GradArgs a) { ppo2_grad_cta<WIDE_D, A2C_LOSS>(a); }
__global__ void __launch_bounds__(NT, 1) dqn_grad_kernel(const __grid_constant__ GradArgs a) { ppo2_grad_cta<MAXD, DQN_LOSS>(a); }
__global__ void __launch_bounds__(NT, 1) dqn_grad_wide_kernel(const __grid_constant__ GradArgs a) { ppo2_grad_cta<WIDE_D, DQN_LOSS>(a); }

// GAE(lambda) of one rollout, the reference's backward recursion (stable-baselines PPO2 runner): one thread per env, T sequential steps,
// eight steps' loads in flight.  Separate roundings (no FMA contraction): the same bits as the torch recursion of rl_baselines/ppo2.py.
__global__ void __launch_bounds__(128) gae_kernel(int T, int N, const float* __restrict__ rew, const float* __restrict__ val, const float* __restrict__ done,
                                                   const float* __restrict__ last_val, float gamma, float gl, float* __restrict__ adv, float* __restrict__ ret) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float lastgae = 0.f, nextval = last_val[n];
    for (int t0 = T - 1; t0 >= 0; t0 -= 8) {
        float r[8], v[8], d[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int t = t0 - k;
            const size_t o = (size_t)(t >= 0 ? t : 0) * N + n;
            r[k] = rew[o]; v[k] = val[o]; d[k] = done[o];
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int t = t0 - k;
            if (t >= 0) {
                const float nonterminal = __fsub_rn(1.0f, d[k]);
                const float delta = __fsub_rn(__fadd_rn(r[k], __fmul_rn(__fmul_rn(gamma, nextval), nonterminal)), v[k]);
                lastgae = __fadd_rn(delta, __fmul_rn(__fmul_rn(gl, nonterminal), lastgae));
                const size_t o = (size_t)t * N + n;
                adv[o] = lastgae; ret[o] = __fadd_rn(lastgae, v[k]);
                nextval = v[k];
            }
        }
    }
}

struct ReduceArgs { srl_mlp_grads g; Seg seg; int nparts; const float* partial; };

// sum of the per-CTA partials in CTA order (deterministic) -> the parameter's gradient tensor
__global__ void ppo2_reduce_kernel(const __grid_constant__ ReduceArgs r) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= r.seg.P) return;
    float s = 0.f;
    for (int c = 0; c < r.nparts; ++c) s += r.partial[(size_t)c * r.seg.P + e];
    const Seg& q = r.seg;
    float* dst; int off;
    if (e < q.pb1) { dst = r.g.pi_w1; off = e - q.pw1; } else if (e < q.pw2) { dst = r.g.pi_b1; off = e - q.pb1; }
    else if (e < q.pb2) { dst = r.g.pi_w2; off = e - q.pw2; } else if (e < q.pw3) { dst = r.g.pi_b2; off = e - q.pb2; }
    else if (e < q.pb3) { dst = r.g.pi_w3; off = e - q.pw3; } else if (e < q.vw1) { dst = r.g.pi_b3; off = e - q.pb3; }
    else if (e < q.vb1) { dst = r.g.vf_w1; off = e - q.vw1; } else if (e < q.vw2) { dst = r.g.vf_b1; off = e - q.vb1; }
    else if (e < q.vb2) { dst = r.g.vf_w2; off = e - q.vw2; } else if (e < q.vw3) { dst = r.g.vf_b2; off = e - q.vb2; }
    else if (e < q.vb3) { dst = r.g.vf_w3; off = e - q.vw3; } else if (e < q.ls) { dst = r.g.vf_b3; off = e - q.vb3; }
    else { dst = r.g.logstd; off = e - q.ls; }
    dst[off] = s;
}

// TF1 `clip_by_global_norm` then `RMSPropOptimizer(momentum=0)` over every tensor of the policy (include/srl_policy.h: srl_clip_rmsprop).
// One CTA: 9-13 k parameters are one pass of 1024 threads; the squared norm is summed in float64 in a fixed order (thread-strided, then a
// shuffle tree, then the 32 warps in order), so two calls give the same bytes.  The update keeps TF's expression order with separate
// float32 roundings (no FMA contraction), the order rl_baselines/a2c.py's torch restatement evaluates.
constexpr int OPT_NT = 1024;
struct OptArgs { srl_mlp_grads p, g, ms; Seg seg; const float* lr; float max_norm, alpha, eps; };

__device__ __forceinline__ float* seg_elem(const srl_mlp_grads& t, const Seg& q, int e) {
    if (e < q.pb1) return t.pi_w1 + (e - q.pw1); if (e < q.pw2) return t.pi_b1 + (e - q.pb1);
    if (e < q.pb2) return t.pi_w2 + (e - q.pw2); if (e < q.pw3) return t.pi_b2 + (e - q.pb2);
    if (e < q.pb3) return t.pi_w3 + (e - q.pw3); if (e < q.vw1) return t.pi_b3 + (e - q.pb3);
    if (e < q.vb1) return t.vf_w1 + (e - q.vw1); if (e < q.vw2) return t.vf_b1 + (e - q.vb1);
    if (e < q.vb2) return t.vf_w2 + (e - q.vw2); if (e < q.vw3) return t.vf_b2 + (e - q.vb2);
    if (e < q.vb3) return t.vf_w3 + (e - q.vw3); if (e < q.ls) return t.vf_b3 + (e - q.vb3);
    return t.logstd + (e - q.ls);
}

__global__ void __launch_bounds__(OPT_NT, 1) clip_rmsprop_kernel(const __grid_constant__ OptArgs o) {
    __shared__ double red[OPT_NT / 32];
    __shared__ float s_scale;
    const int t = threadIdx.x;
    double s = 0.0;
    for (int e = t; e < o.seg.P; e += OPT_NT) { const double g = (double)*seg_elem(o.g, o.seg, e); s = fma(g, g, s); }
    for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
    if ((t & 31) == 0) red[t >> 5] = s;
    __syncthreads();
    if (t == 0) {
        double tot = 0.0;
        for (int w = 0; w < OPT_NT / 32; ++w) tot += red[w];
        const double norm = sqrt(tot);      // + (norm - norm): NaN for a non-finite norm, so that every tensor becomes NaN, as in TF
        s_scale = (float)((double)o.max_norm / fmax(norm, (double)o.max_norm) + (norm - norm));     // scale = max_norm / max(norm, max_norm)
    }
    __syncthreads();
    const float scale = s_scale, lr = *o.lr, rho1 = __fsub_rn(1.0f, o.alpha);
    for (int e = t; e < o.seg.P; e += OPT_NT) {
        const float g = __fmul_rn(*seg_elem(o.g, o.seg, e), scale);
        float* msp = seg_elem(o.ms, o.seg, e);
        float* wp = seg_elem(o.p, o.seg, e);
        const float ms = __fadd_rn(*msp, __fmul_rn(__fsub_rn(__fmul_rn(g, g), *msp), rho1));        // ms += (g^2 - ms) (1 - alpha)
        *msp = ms;
        *wp = __fsub_rn(*wp, __fdiv_rn(__fmul_rn(g, lr), __fsqrt_rn(__fadd_rn(ms, o.eps))));          // w -= g lr / sqrt(ms + eps)
    }
}

// Per-tensor `tf.clip_by_norm(g, clip_norm)` then one TF1 `AdamOptimizer` step over every tensor of the policy (include/srl_policy.h:
// srl_clip_adam).  One CTA, like clip_rmsprop_kernel: each tensor's squared norm is summed in float64 in a fixed order; the update keeps the
// expression order of TF's ApplyAdam with separate float32 roundings, the order rl_baselines/deepq.py's torch restatement evaluates.
constexpr int NSEG = 13;
struct AdamArgs { srl_mlp_grads p, g, m, v; Seg seg; const float* lr; float* beta_power; float clip_norm, beta1, beta2, eps; };

__global__ void __launch_bounds__(OPT_NT, 1) clip_adam_kernel(const __grid_constant__ AdamArgs o) {
    __shared__ double red[OPT_NT / 32];
    __shared__ float s_norm[NSEG];
    const int t = threadIdx.x;
    const Seg& q = o.seg;
    const int off[NSEG + 1] = {q.pw1, q.pb1, q.pw2, q.pb2, q.pw3, q.pb3, q.vw1, q.vb1, q.vw2, q.vb2, q.vw3, q.vb3, q.ls, q.P};
    for (int k = 0; k < NSEG; ++k) {
        double s = 0.0;
        for (int e = off[k] + t; e < off[k + 1]; e += OPT_NT) { const double g = (double)*seg_elem(o.g, q, e); s = fma(g, g, s); }
        for (int w = 16; w > 0; w >>= 1) s += __shfl_xor_sync(0xffffffffu, s, w);
        if ((t & 31) == 0) red[t >> 5] = s;
        __syncthreads();
        if (t == 0) {
            double tot = 0.0;
            for (int w = 0; w < OPT_NT / 32; ++w) tot += red[w];
            s_norm[k] = (float)sqrt(tot);
        }
        __syncthreads();
    }
    const float lr = *o.lr, b1p = o.beta_power[0], b2p = o.beta_power[1];
    const float lr_t = __fdiv_rn(__fmul_rn(lr, __fsqrt_rn(__fsub_rn(1.0f, b2p))), __fsub_rn(1.0f, b1p));   // lr sqrt(1 - beta2^t) / (1 - beta1^t)
    const float r1 = __fsub_rn(1.0f, o.beta1), r2 = __fsub_rn(1.0f, o.beta2);
    for (int e = t; e < q.P; e += OPT_NT) {
        int k = 0;
        while (e >= off[k + 1]) ++k;
        const float nk = s_norm[k];
        const float den = nk != nk ? nk : fmaxf(nk, o.clip_norm);                          // max(norm, clip_norm), NaN for a NaN norm
        const float g = __fdiv_rn(__fmul_rn(*seg_elem(o.g, q, e), o.clip_norm), den);       // t clip_norm / max(l2norm, clip_norm)
        float* mp = seg_elem(o.m, q, e);
        float* vp = seg_elem(o.v, q, e);
        float* wp = seg_elem(o.p, q, e);
        const float m = __fadd_rn(*mp, __fmul_rn(__fsub_rn(g, *mp), r1));                    // m += (g - m) (1 - beta1)
        const float v = __fadd_rn(*vp, __fmul_rn(__fsub_rn(__fmul_rn(g, g), *vp), r2));      // v += (g^2 - v) (1 - beta2)
        *mp = m; *vp = v;
        *wp = __fsub_rn(*wp, __fdiv_rn(__fmul_rn(m, lr_t), __fadd_rn(__fsqrt_rn(v), o.eps)));   // w -= m lr_t / (sqrt(v) + eps)
    }
    if (t == 0) { o.beta_power[0] = __fmul_rn(b1p, o.beta1); o.beta_power[1] = __fmul_rn(b2p, o.beta2); }   // TF's beta1_power *= beta1 after the step
}

template <int MD>
constexpr size_t grad_smem_bytes() {
    return sizeof(float) * (size_t)(4 * H * WS + MAXO * WS + WS + (MD == MAXD ? 8 : 6) * CH * WS + 2 * H * grad_w1_stride<MD>() + 4 * H + MAXO + 4 + MAXO +
                                    CH * MD + 2 * CH * (MAXO + 1) + 2 * CH * MAXO + CH * 4 + CH * 2);
}
static_assert(grad_smem_bytes<MAXD>() <= 227 * 1024 && grad_smem_bytes<WIDE_D>() <= 227 * 1024, "shared memory of one CTA");

int grid_ctas(int mb) {
    static int sms[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (dev < 0 || dev >= 64) return 0;
    if (!sms[dev]) { if (cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0; }
    const int chunks = (mb + CH - 1) / CH;
    return chunks < sms[dev] ? chunks : sms[dev];
}

// the checks srl_ppo2_grad and srl_a2c_grad share (`who` prefixes the message); the grid size, or 0 after setting the error
int grad_args_ok(const char* who, const srl_mlp_policy* p, const srl_mlp_grads* grads, int minibatch) {
    if (p->struct_size != sizeof(srl_mlp_policy) || grads->struct_size != sizeof(srl_mlp_grads)) { srl_set_error("%s: struct size mismatch", who); return 0; }
    if (p->obs_dim < 1 || p->obs_dim > WIDE_D || p->n_out < 1 || p->n_out > MAXO || (p->discrete && p->n_out < 2) || minibatch < 1) {
        srl_set_error("%s: unsupported shape obs_dim=%d n_out=%d minibatch=%d (obs_dim 1..%d, n_out 1..%d)", who, p->obs_dim, p->n_out, minibatch,
                      WIDE_D, MAXO); return 0;
    }
    if (!p->pi_w1 || !p->pi_b1 || !p->pi_w2 || !p->pi_b2 || !p->pi_w3 || !p->pi_b3 || !p->vf_w1 || !p->vf_b1 || !p->vf_w2 || !p->vf_b2 || !p->vf_w3 ||
        !p->vf_b3 || (!p->discrete && !p->logstd)) { srl_set_error("%s: null weight pointer", who); return 0; }
    if (!grads->pi_w1 || !grads->pi_b1 || !grads->pi_w2 || !grads->pi_b2 || !grads->pi_w3 || !grads->pi_b3 || !grads->vf_w1 || !grads->vf_b1 || !grads->vf_w2 ||
        !grads->vf_b2 || !grads->vf_w3 || !grads->vf_b3 || (!p->discrete && !grads->logstd)) { srl_set_error("%s: null gradient pointer", who); return 0; }
    const int ctas = grid_ctas(minibatch);
    if (ctas <= 0) srl_set_error("%s: no CUDA device", who);
    return ctas;
}

// the gradient kernel of the row width (narrow or wide instantiation), then the CTA-order reduction into the gradient tensors
template <void (*NARROW)(GradArgs), void (*WIDE)(GradArgs)>
int launch_grad(const GradArgs& a, const srl_mlp_grads* grads, int ctas, cudaStream_t st) {
    if (a.p.obs_dim <= MAXD) {
        constexpr size_t smem = grad_smem_bytes<MAXD>();
        SRL_CUDA_OK(srl_smem_opt_in<NARROW>(smem));
        NARROW<<<ctas, NT, smem, st>>>(a);
    } else {
        constexpr size_t smem = grad_smem_bytes<WIDE_D>();
        SRL_CUDA_OK(srl_smem_opt_in<WIDE>(smem));
        WIDE<<<ctas, NT, smem, st>>>(a);
    }
    SRL_CUDA_OK(cudaGetLastError());
    ReduceArgs r;
    r.g = *grads; r.seg = make_seg(a.p.obs_dim, a.p.n_out, a.p.discrete); r.nparts = ctas; r.partial = a.partial;
    ppo2_reduce_kernel<<<(r.seg.P + 255) / 256, 256, 0, st>>>(r);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace

extern "C" {

size_t srl_ppo2_workspace_bytes(int obs_dim, int n_out, int discrete, int minibatch) {
    if (obs_dim < 1 || obs_dim > WIDE_D || n_out < 1 || n_out > MAXO || minibatch < 1) {
        srl_set_error("ppo2_workspace_bytes: unsupported shape obs_dim=%d n_out=%d minibatch=%d (obs_dim 1..%d, n_out 1..%d)", obs_dim, n_out, minibatch,
                      WIDE_D, MAXO);
        return 0;
    }
    const Seg seg = make_seg(obs_dim, n_out, discrete);
    const int ctas = grid_ctas(minibatch);
    return 2048 + sizeof(float) * (size_t)seg.P * (size_t)(ctas > 0 ? ctas : 1);
}

int srl_ppo2_grad(const srl_mlp_policy* p, const srl_mlp_grads* grads, int minibatch, const int64_t* idx, const float* obs, const void* actions,
                  const float* adv, const float* ret, const float* old_logp, const float* old_value, float cliprange, float ent_coef, float vf_coef,
                  void* workspace, size_t workspace_bytes, void* stream) {
    if (!p || !grads || !obs || !actions || !adv || !ret || !old_logp || !old_value || !workspace) { srl_set_error("ppo2_grad: null argument"); return 1; }
    const int ctas = grad_args_ok("ppo2_grad", p, grads, minibatch);
    if (ctas <= 0) return 1;
    const Seg seg = make_seg(p->obs_dim, p->n_out, p->discrete);
    if (workspace_bytes < 2048 + sizeof(float) * (size_t)seg.P * (size_t)ctas) { srl_set_error("ppo2_grad: workspace too small (srl_ppo2_workspace_bytes)"); return 1; }
    cudaStream_t st = (cudaStream_t)stream;
    double* stats = reinterpret_cast<double*>(workspace);
    float* partial = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + 2048);
    adv_stats_kernel<<<STATS_CTAS, STATS_NT, 0, st>>>(minibatch, reinterpret_cast<const long long*>(idx), adv, stats);
    SRL_CUDA_OK(cudaGetLastError());
    GradArgs a;
    a.p = *p; a.mb = minibatch; a.idx = reinterpret_cast<const long long*>(idx); a.obs = obs; a.act = actions; a.adv = adv; a.ret = ret;
    a.old_logp = old_logp; a.old_val = old_value; a.clip = cliprange; a.ent_coef = ent_coef; a.vf_coef = vf_coef; a.stats = stats; a.partial = partial;
    return launch_grad<ppo2_grad_kernel, ppo2_grad_wide_kernel>(a, grads, ctas, st);
}

size_t srl_a2c_workspace_bytes(int obs_dim, int n_out, int discrete, int rows) {
    if (obs_dim < 1 || obs_dim > WIDE_D || n_out < 1 || n_out > MAXO || rows < 1) {
        srl_set_error("a2c_workspace_bytes: unsupported shape obs_dim=%d n_out=%d rows=%d (obs_dim 1..%d, n_out 1..%d)", obs_dim, n_out, rows, WIDE_D, MAXO);
        return 0;
    }
    const int ctas = grid_ctas(rows);
    return sizeof(float) * (size_t)make_seg(obs_dim, n_out, discrete).P * (size_t)(ctas > 0 ? ctas : 1);
}

int srl_a2c_grad(const srl_mlp_policy* p, const srl_mlp_grads* grads, int rows, const int64_t* idx, const float* obs, const void* actions,
                 const float* ret, const float* old_value, float ent_coef, float vf_coef, void* workspace, size_t workspace_bytes, void* stream) {
    if (!p || !grads || !obs || !actions || !ret || !old_value || !workspace) { srl_set_error("a2c_grad: null argument"); return 1; }
    const int ctas = grad_args_ok("a2c_grad", p, grads, rows);
    if (ctas <= 0) return 1;
    const Seg seg = make_seg(p->obs_dim, p->n_out, p->discrete);
    if (workspace_bytes < sizeof(float) * (size_t)seg.P * (size_t)ctas) { srl_set_error("a2c_grad: workspace too small (srl_a2c_workspace_bytes)"); return 1; }
    GradArgs a = {};
    a.p = *p; a.mb = rows; a.idx = reinterpret_cast<const long long*>(idx); a.obs = obs; a.act = actions; a.ret = ret; a.old_val = old_value;
    a.ent_coef = ent_coef; a.vf_coef = vf_coef; a.partial = reinterpret_cast<float*>(workspace);
    return launch_grad<a2c_grad_kernel, a2c_grad_wide_kernel>(a, grads, ctas, (cudaStream_t)stream);
}

int srl_dqn_grad(const srl_mlp_policy* q, const srl_mlp_grads* grads, int batch, const int64_t* idx, const float* obs, const int64_t* actions,
                 const float* y, const float* weights, float* td_out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!q || !grads || !obs || !actions || !y || !td_out || !workspace) { srl_set_error("dqn_grad: null argument"); return 1; }
    if (q->struct_size == sizeof(srl_mlp_policy) && !q->discrete) { srl_set_error("dqn_grad: the Q network needs discrete = 1"); return 1; }
    const int ctas = grad_args_ok("dqn_grad", q, grads, batch);
    if (ctas <= 0) return 1;
    const Seg seg = make_seg(q->obs_dim, q->n_out, 1);
    if (workspace_bytes < sizeof(float) * (size_t)seg.P * (size_t)ctas) { srl_set_error("dqn_grad: workspace too small (srl_a2c_workspace_bytes)"); return 1; }
    GradArgs a = {};
    a.p = *q; a.mb = batch; a.idx = reinterpret_cast<const long long*>(idx); a.obs = obs; a.act = actions; a.ret = y; a.old_val = weights;
    a.partial = reinterpret_cast<float*>(workspace); a.td = td_out;
    return launch_grad<dqn_grad_kernel, dqn_grad_wide_kernel>(a, grads, ctas, (cudaStream_t)stream);
}

int srl_clip_adam(int obs_dim, int n_out, int discrete, const srl_mlp_grads* params, const srl_mlp_grads* grads, const srl_mlp_grads* m,
                  const srl_mlp_grads* v, const float* lr, float* beta_power, float clip_norm, float beta1, float beta2, float epsilon, void* stream) {
    if (!params || !grads || !m || !v || !lr || !beta_power) { srl_set_error("clip_adam: null argument"); return 1; }
    if (!discrete) { srl_set_error("clip_adam: the DQN optimiser step takes a discrete Q network (discrete = 1)"); return 1; }
    if (obs_dim < 1 || obs_dim > WIDE_D || n_out < 1 || n_out > MAXO || (discrete && n_out < 2)) {
        srl_set_error("clip_adam: unsupported shape obs_dim=%d n_out=%d (obs_dim 1..%d, n_out 1..%d)", obs_dim, n_out, WIDE_D, MAXO); return 1;
    }
    if (!(clip_norm > 0.f) || !(beta1 >= 0.f && beta1 < 1.f) || !(beta2 >= 0.f && beta2 < 1.f) || !(epsilon >= 0.f)) {
        srl_set_error("clip_adam: need clip_norm > 0, 0 <= beta1, beta2 < 1, epsilon >= 0 (got %g, %g, %g, %g)", clip_norm, beta1, beta2, epsilon); return 1;
    }
    for (const srl_mlp_grads* t : {params, grads, m, v}) {
        if (t->struct_size != sizeof(srl_mlp_grads)) { srl_set_error("clip_adam: struct size mismatch"); return 1; }
        if (!t->pi_w1 || !t->pi_b1 || !t->pi_w2 || !t->pi_b2 || !t->pi_w3 || !t->pi_b3 || !t->vf_w1 || !t->vf_b1 || !t->vf_w2 || !t->vf_b2 || !t->vf_w3 ||
            !t->vf_b3 || (!discrete && !t->logstd)) { srl_set_error("clip_adam: null tensor pointer"); return 1; }
    }
    AdamArgs o;
    o.p = *params; o.g = *grads; o.m = *m; o.v = *v; o.seg = make_seg(obs_dim, n_out, discrete); o.lr = lr; o.beta_power = beta_power;
    o.clip_norm = clip_norm; o.beta1 = beta1; o.beta2 = beta2; o.eps = epsilon;
    clip_adam_kernel<<<1, OPT_NT, 0, (cudaStream_t)stream>>>(o);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_clip_rmsprop(int obs_dim, int n_out, int discrete, const srl_mlp_grads* params, const srl_mlp_grads* grads, const srl_mlp_grads* ms,
                     const float* lr, float max_grad_norm, float alpha, float epsilon, void* stream) {
    if (!params || !grads || !ms || !lr) { srl_set_error("clip_rmsprop: null argument"); return 1; }
    if (params->struct_size != sizeof(srl_mlp_grads) || grads->struct_size != sizeof(srl_mlp_grads) || ms->struct_size != sizeof(srl_mlp_grads)) {
        srl_set_error("clip_rmsprop: struct size mismatch"); return 1;
    }
    if (obs_dim < 1 || obs_dim > WIDE_D || n_out < 1 || n_out > MAXO || (discrete && n_out < 2)) {
        srl_set_error("clip_rmsprop: unsupported shape obs_dim=%d n_out=%d (obs_dim 1..%d, n_out 1..%d)", obs_dim, n_out, WIDE_D, MAXO); return 1;
    }
    if (!(max_grad_norm > 0.f) || !(alpha >= 0.f && alpha <= 1.f) || !(epsilon >= 0.f)) {
        srl_set_error("clip_rmsprop: need max_grad_norm > 0, 0 <= alpha <= 1, epsilon >= 0 (got %g, %g, %g)", max_grad_norm, alpha, epsilon); return 1;
    }
    for (const srl_mlp_grads* t : {params, grads, ms}) {
        if (!t->pi_w1 || !t->pi_b1 || !t->pi_w2 || !t->pi_b2 || !t->pi_w3 || !t->pi_b3 || !t->vf_w1 || !t->vf_b1 || !t->vf_w2 || !t->vf_b2 || !t->vf_w3 ||
            !t->vf_b3 || (!discrete && !t->logstd)) { srl_set_error("clip_rmsprop: null tensor pointer"); return 1; }
    }
    OptArgs o;
    o.p = *params; o.g = *grads; o.ms = *ms; o.seg = make_seg(obs_dim, n_out, discrete); o.lr = lr; o.max_norm = max_grad_norm; o.alpha = alpha; o.eps = epsilon;
    clip_rmsprop_kernel<<<1, OPT_NT, 0, (cudaStream_t)stream>>>(o);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_ppo2_gae(int n_steps, int n_envs, const float* rew, const float* value, const float* done, const float* last_value, double gamma, double lam,
                 float* adv_out, float* ret_out, void* stream) {
    if (!rew || !value || !done || !last_value || !adv_out || !ret_out) { srl_set_error("ppo2_gae: null argument"); return 1; }
    if (n_steps < 1 || n_envs < 1) { srl_set_error("ppo2_gae: bad shape"); return 1; }
    // the coefficients of the torch recursion: `gamma * nextval` rounds gamma to float32, `gamma * lam * nonterminal` rounds the double product
    gae_kernel<<<(n_envs + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n_steps, n_envs, rew, value, done, last_value, (float)gamma, (float)(gamma * lam), adv_out, ret_out);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
