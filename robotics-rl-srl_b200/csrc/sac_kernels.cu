// SAC consumer kernels (include/srl_policy.h: srl_sac_*): the policy step, the replay ring's store, the per-sample half of a gradient step
// (sampling, target values, the actor's reparameterised action and log-probability, qf1's input gradient, every head derivative), the weight
// gradients of the four trained networks, and TF1 Adam over the parameter arena with the Polyak update of the target value network.
//
// All five networks are in -> 64 -> 64 -> out with ReLU.  Per-sample work (act, prepare) runs one thread per sample with the weights staged in
// shared memory and read by every lane at the same address (broadcast); the hidden layer of 64 values sits in registers and the second layer is
// folded into the head as it is produced, so a forward pass keeps only the two ReLU masks.  The weight gradients (srl_sac_grad) run the chunked
// scheme of ppo2_kernels.cu: a persistent CTA per (chunk stride, network) recomputes the forward pass of 64 samples with every activation in
// shared memory, accumulates its share of the weight gradient in registers, and a second launch sums the per-CTA partials in CTA order.
#include <cuda_runtime.h>
#include <math.h>
#include "common.cuh"
#include "policy_core.h"
#include "../../include/srl_policy.h"

namespace {

constexpr int H = 64, MAXW = 32, MAXA = 8, DINMAX = MAXW + MAXA, OUTMAX = 2 * MAXA;
// counter word 3 of the Philox streams (the simulator uses 0..10, the policy step 16..18, DQN 24 and 25)
enum { SRL_PHILOX_PURPOSE_SAC_ACT = 26, SRL_PHILOX_PURPOSE_SAC_RANDOM = 28, SRL_PHILOX_PURPOSE_SAC_SAMPLE = 30, SRL_PHILOX_PURPOSE_SAC_REPARAM = 31 };
constexpr float LOG_STD_MIN = -20.f, LOG_STD_MAX = 2.f, SQUASH_EPS = 1e-6f, LOG_2PI = 1.83787706640934548356f;

// ---- the arena: actor | qf1 | qf2 | vf | log_ent_coef, each network w1 [64][in], b1, w2 [64][64], b2, w3 [out][64], b3 ----
struct NetOff { int w1, b1, w2, b2, w3, b3, end, in, out; };
__host__ __device__ inline NetOff net_off(int base, int in, int out) {
    NetOff o; o.in = in; o.out = out;
    o.w1 = base; o.b1 = o.w1 + H * in; o.w2 = o.b1 + H; o.b2 = o.w2 + H * H; o.w3 = o.b2 + H; o.b3 = o.w3 + out * H; o.end = o.b3 + out;
    return o;
}
enum { ACTOR = 0, QF1 = 1, QF2 = 2, VF = 3, NNETS = 4 };
struct Layout { NetOff net[NNETS]; int le, P; };
__host__ __device__ inline Layout make_layout(int W, int A) {
    Layout L;
    L.net[ACTOR] = net_off(0, W, 2 * A);
    L.net[QF1] = net_off(L.net[ACTOR].end, W + A, 1);
    L.net[QF2] = net_off(L.net[QF1].end, W + A, 1);
    L.net[VF] = net_off(L.net[QF2].end, W, 1);
    L.le = L.net[VF].end; L.P = L.le + 1;
    return L;
}

__device__ __forceinline__ void philox(unsigned long long seed, unsigned long long stream, uint32_t counter, uint32_t purpose, uint32_t (&r)[4]) {
    srl_philox4x32_10_hd(seed, stream, counter, purpose, r);
}
// the Gaussian of dim k from its block r (srl_sample_gaussian's word use): k % 4 = 0, 1 the cos / sin of words (0, 1), 2, 3 of words (2, 3)
__device__ __forceinline__ float box_muller(const uint32_t (&r)[4], int k) {
    const uint32_t wa = r[k & 2], wb = r[(k & 2) + 1];
    const float u1 = ((float)(wa >> 8) + 0.5f) * (1.0f / 16777216.0f), u2 = ((float)(wb >> 8) + 0.5f) * (1.0f / 16777216.0f);
    const float rad = sqrtf(-2.0f * logf(u1)), ang = 6.28318530717958647692f * u2;
    return (k & 1) ? rad * sinf(ang) : rad * cosf(ang);
}

// the LAST CTA to retire advances the counter of a {seed, counter, arrivals} record (srl_policy_act's rule); returns true in that CTA's thread 0
__device__ __forceinline__ bool last_cta_advance(unsigned long long* rng, unsigned long long counter) {
    __syncthreads();
    bool last = false;
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long arrived = atomicAdd(rng + 2, 1ull);
        if (arrived == (unsigned long long)gridDim.x - 1ull) {
            __threadfence();
            last = true;
            rng[2] = 0ull;
            rng[1] = counter + 1ull;
        }
    }
    return last;
}

// ---- one thread per sample: a network staged as w1T [DINMAX][64], b1 [64], w2 [64][64], b2 [64], w3T [64][OUTMAX], b3 [OUTMAX] ----
constexpr int NET_FLOATS = DINMAX * H + H + H * H + H + H * OUTMAX + OUTMAX;
static_assert(NET_FLOATS % 4 == 0, "16-byte aligned networks");
constexpr int XS = DINMAX + 1;     // per-thread input rows in shared memory: an odd stride, no bank conflicts
struct NetS { const float *w1T, *b1, *w2, *b2, *w3T, *b3; };

__device__ NetS stage_net(const float* arena, const NetOff& o, float* s, int nt) {
    float* w1T = s; float* b1 = w1T + DINMAX * H; float* w2 = b1 + H; float* b2 = w2 + H * H; float* w3T = b2 + H; float* b3 = w3T + H * OUTMAX;
    for (int e = threadIdx.x; e < H * o.in; e += nt) { const int i = e / o.in, d = e % o.in; w1T[d * H + i] = arena[o.w1 + e]; }
    for (int e = threadIdx.x; e < H * H; e += nt) w2[e] = arena[o.w2 + e];
    for (int e = threadIdx.x; e < o.out * H; e += nt) { const int k = e >> 6, j = e & 63; w3T[j * OUTMAX + k] = arena[o.w3 + e]; }
    for (int e = threadIdx.x; e < H; e += nt) { b1[e] = arena[o.b1 + e]; b2[e] = arena[o.b2 + e]; }
    for (int e = threadIdx.x; e < o.out; e += nt) b3[e] = arena[o.b3 + e];
    return NetS{w1T, b1, w2, b2, w3T, b3};
}

// out[k] (k < nout) of the row x[0 .. din); m1 / m2: bit i set where hidden unit i of layer 1 / 2 is positive (ReLU's gradient mask)
template <int NOUT>
__device__ __forceinline__ void mlp_fwd(const NetS& w, int din, int nout, const float* x, float (&out)[NOUT], unsigned long long& m1, unsigned long long& m2) {
    float h[H];
#pragma unroll
    for (int i = 0; i < H; ++i) h[i] = w.b1[i];
    for (int d = 0; d < din; ++d) {
        const float xd = x[d];
#pragma unroll
        for (int i4 = 0; i4 < H / 4; ++i4) {
            const float4 wv = *reinterpret_cast<const float4*>(w.w1T + d * H + 4 * i4);
            h[4 * i4] = fmaf(wv.x, xd, h[4 * i4]); h[4 * i4 + 1] = fmaf(wv.y, xd, h[4 * i4 + 1]);
            h[4 * i4 + 2] = fmaf(wv.z, xd, h[4 * i4 + 2]); h[4 * i4 + 3] = fmaf(wv.w, xd, h[4 * i4 + 3]);
        }
    }
    m1 = 0ull;
#pragma unroll
    for (int i = 0; i < H; ++i) { if (h[i] > 0.f) m1 |= 1ull << i; h[i] = fmaxf(h[i], 0.f); }
#pragma unroll
    for (int k = 0; k < NOUT; ++k) out[k] = k < nout ? w.b3[k] : 0.f;
    m2 = 0ull;
#pragma unroll 2
    for (int j = 0; j < H; ++j) {
        float s0 = w.b2[j], s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int i4 = 0; i4 < H / 4; ++i4) {
            const float4 wv = *reinterpret_cast<const float4*>(w.w2 + j * H + 4 * i4);
            s0 = fmaf(wv.x, h[4 * i4], s0); s1 = fmaf(wv.y, h[4 * i4 + 1], s1); s2 = fmaf(wv.z, h[4 * i4 + 2], s2); s3 = fmaf(wv.w, h[4 * i4 + 3], s3);
        }
        const float z = (s0 + s1) + (s2 + s3);
        if (z > 0.f) m2 |= 1ull << j;
        const float r = fmaxf(z, 0.f);
#pragma unroll
        for (int k = 0; k < NOUT; ++k) if (k < nout) out[k] = fmaf(w.w3T[j * OUTMAX + k], r, out[k]);
    }
}

// d out[0] / d x[first + k] for k < count, of a one-output network whose forward pass left the masks m1, m2
__device__ __forceinline__ void mlp_input_grad(const NetS& w, unsigned long long m1, unsigned long long m2, int first, int count, float (&dx)[MAXA]) {
    float g[H];
#pragma unroll
    for (int i = 0; i < H; ++i) g[i] = 0.f;
#pragma unroll 2
    for (int j = 0; j < H; ++j) {
        const float c = ((m2 >> j) & 1ull) ? w.w3T[j * OUTMAX] : 0.f;
#pragma unroll
        for (int i4 = 0; i4 < H / 4; ++i4) {
            const float4 wv = *reinterpret_cast<const float4*>(w.w2 + j * H + 4 * i4);
            g[4 * i4] = fmaf(wv.x, c, g[4 * i4]); g[4 * i4 + 1] = fmaf(wv.y, c, g[4 * i4 + 1]);
            g[4 * i4 + 2] = fmaf(wv.z, c, g[4 * i4 + 2]); g[4 * i4 + 3] = fmaf(wv.w, c, g[4 * i4 + 3]);
        }
    }
#pragma unroll
    for (int i = 0; i < H; ++i) if (!((m1 >> i) & 1ull)) g[i] = 0.f;
#pragma unroll
    for (int k = 0; k < MAXA; ++k) {
        dx[k] = 0.f;
        if (k < count) {
            float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
            for (int i4 = 0; i4 < H / 4; ++i4) {
                const float4 wv = *reinterpret_cast<const float4*>(w.w1T + (first + k) * H + 4 * i4);
                s0 = fmaf(wv.x, g[4 * i4], s0); s1 = fmaf(wv.y, g[4 * i4 + 1], s1); s2 = fmaf(wv.z, g[4 * i4 + 2], s2); s3 = fmaf(wv.w, g[4 * i4 + 3], s3);
            }
            dx[k] = (s0 + s1) + (s2 + s3);
        }
    }
}

// ---- srl_sac_act ----
constexpr int ACT_NT = 128;
struct ActArgs { Layout L; int W, A, n, mode; const float* arena; const float* obs; unsigned long long* rng; unsigned long long env_offset; float* act; };

__global__ void __launch_bounds__(ACT_NT) sac_act_kernel(const __grid_constant__ ActArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int W = a.W, A = a.A, i = blockIdx.x * ACT_NT + threadIdx.x;
    const unsigned long long seed = a.rng[0], counter = a.rng[1];
    if (a.mode == 2) {
        if (i < a.n) {
            uint32_t r[4] = {0u, 0u, 0u, 0u};
#pragma unroll
            for (int k = 0; k < MAXA; ++k) if (k < A) {
                if ((k & 3) == 0) philox(seed, a.env_offset + (unsigned long long)i, (uint32_t)counter, SRL_PHILOX_PURPOSE_SAC_RANDOM + (k >> 2), r);
                a.act[(size_t)i * A + k] = __fsub_rn(__fmul_rn(2.0f, (float)(r[k & 3] >> 8) * (1.0f / 16777216.0f)), 1.0f);
            }
        }
        last_cta_advance(a.rng, counter);
        return;
    }
    const NetS net = stage_net(a.arena, a.L.net[ACTOR], smem, ACT_NT);
    float* xs = smem + NET_FLOATS + threadIdx.x * XS;
    if (i < a.n) for (int d = 0; d < W; ++d) xs[d] = a.obs[(size_t)i * W + d];
    __syncthreads();
    if (i < a.n) {
        float out[OUTMAX];
        unsigned long long m1, m2;
        mlp_fwd<OUTMAX>(net, W, 2 * A, xs, out, m1, m2);
        uint32_t r[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int k = 0; k < MAXA; ++k) if (k < A) {
            float u = out[k];
            if (a.mode == 0) {
                if ((k & 3) == 0) philox(seed, a.env_offset + (unsigned long long)i, (uint32_t)counter, SRL_PHILOX_PURPOSE_SAC_ACT + (k >> 2), r);
                float raw = 0.f;                                                            // out[A + k], selected in registers
#pragma unroll
                for (int j = 0; j < OUTMAX; ++j) if (j == A + k) raw = out[j];
                const float ls = fminf(fmaxf(raw, LOG_STD_MIN), LOG_STD_MAX);
                u = __fadd_rn(out[k], __fmul_rn(expf(ls), box_muller(r, k)));             // mu + std eps
            }
            a.act[(size_t)i * A + k] = tanhf(u);
        }
    }
    last_cta_advance(a.rng, counter);
}

// ---- srl_sac_store ----
constexpr int STORE_NT = 256;
struct StoreArgs {
    int rows, n, W, A; long long* step; float* obs; const float* act; const float* rew; const uint8_t* done; const float* new_obs;
    float* obs_ring; float* act_ring; float* rew_ring; uint8_t* done_ring; float* next_obs_ring;
};
__global__ void __launch_bounds__(STORE_NT) sac_store_kernel(const __grid_constant__ StoreArgs a) {
    const long long step = a.step[0];
    const size_t row = (size_t)(step % a.rows), n = (size_t)a.n, j = (size_t)blockIdx.x * STORE_NT + threadIdx.x;
    if (j < n * a.W) {
        const float o = a.obs[j], no = a.new_obs[j];
        a.obs_ring[row * n * a.W + j] = o;
        a.next_obs_ring[row * n * a.W + j] = no;
        a.obs[j] = no;
    }
    if (j < n * a.A) a.act_ring[row * n * a.A + j] = a.act[j];
    if (j < n) { a.rew_ring[row * n + j] = a.rew[j]; a.done_ring[row * n + j] = a.done[j]; }
    __syncthreads();
    if (threadIdx.x == 0) {              // the last CTA advances the step: every CTA has read it by then
        __threadfence();
        const unsigned long long arrived = atomicAdd(reinterpret_cast<unsigned long long*>(a.step + 1), 1ull);
        if (arrived == (unsigned long long)gridDim.x - 1ull) { a.step[1] = 0; a.step[0] = step + 1; __threadfence(); }
    }
}

// ---- srl_sac_prepare ----
constexpr int PREP_NT = 128;
struct PrepArgs {
    Layout L; int W, A, rows, n, B, auto_ent; const float* arena; const float* target; const long long* step;
    const float* obs; const float* act; const float* rew; const uint8_t* done; const float* next_obs;
    float gamma, ent_coef, target_entropy;
    unsigned long long* rng; long long* idx; float* qb; float* vb; float* logp; float* dact; float* ent_grad; double* partial;
};

__global__ void __launch_bounds__(PREP_NT) sac_prepare_kernel(const __grid_constant__ PrepArgs a) {
    extern __shared__ __align__(16) float smem[];
    __shared__ double red[PREP_NT / 32];
    const int W = a.W, A = a.A, b = blockIdx.x * PREP_NT + threadIdx.x;
    const unsigned long long seed = a.rng[0], counter = a.rng[1];
    const NetS actor = stage_net(a.arena, a.L.net[ACTOR], smem, PREP_NT);
    const NetS qf1 = stage_net(a.arena, a.L.net[QF1], smem + NET_FLOATS, PREP_NT);
    const NetS qf2 = stage_net(a.arena, a.L.net[QF2], smem + 2 * NET_FLOATS, PREP_NT);
    const NetS vt = stage_net(a.target, net_off(0, W, 1), smem + 3 * NET_FLOATS, PREP_NT);
    float* xs = smem + 4 * NET_FLOATS + threadIdx.x * XS;
    const float alpha = a.auto_ent ? expf(a.arena[a.L.le]) : a.ent_coef;
    __syncthreads();
    double ent_term = 0.0;
    const long long stored = a.step[0] < a.rows ? a.step[0] : (long long)a.rows, size = stored * a.n;
    if (b < a.B && size <= 0) {                // nothing stored yet: no sample, zero outputs (srl_sac_grad skips idx -1)
        a.idx[b] = -1;
        a.qb[b] = 0.f; a.vb[b] = 0.f; a.logp[b] = 0.f;
        for (int k = 0; k < 2 * A; ++k) a.dact[(size_t)b * 2 * A + k] = 0.f;
    }
    if (b < a.B && size > 0) {
        uint32_t r[4];
        philox(seed, (unsigned long long)b, (uint32_t)counter, SRL_PHILOX_PURPOSE_SAC_SAMPLE, r);
        const double u01 = ((double)(r[0] >> 5) * 67108864.0 + (double)(r[1] >> 6)) * (1.0 / 9007199254740992.0);
        long long g = (long long)(u01 * (double)size);
        if (g > size - 1) g = size - 1;
        a.idx[b] = g;
        float o1[1];
        unsigned long long m1, m2;
        // q_backup = r + gamma ((1 - d) V_targ(s'))
        for (int d = 0; d < W; ++d) xs[d] = a.next_obs[g * W + d];
        mlp_fwd<1>(vt, W, 1, xs, o1, m1, m2);
        const float notdone = a.done[g] ? 0.f : 1.f;
        a.qb[b] = __fadd_rn(a.rew[g], __fmul_rn(a.gamma, __fmul_rn(notdone, o1[0])));
        // the actor at s: a_pi = tanh(mu + std eps) and its log-probability
        for (int d = 0; d < W; ++d) xs[d] = a.obs[g * W + d];
        float out[OUTMAX];
        mlp_fwd<OUTMAX>(actor, W, 2 * A, xs, out, m1, m2);
        float std_[MAXA], eps[MAXA], ap[MAXA], lsr[MAXA], zz[MAXA], sd[MAXA];
        float lp1 = 0.f, lp2 = 0.f;
#pragma unroll
        for (int k = 0; k < MAXA; ++k) {
            std_[k] = eps[k] = ap[k] = lsr[k] = zz[k] = sd[k] = 0.f;
            if (k < A) {
                if ((k & 3) == 0) philox(seed, (unsigned long long)b, (uint32_t)counter, SRL_PHILOX_PURPOSE_SAC_REPARAM + (k >> 2), r);
                eps[k] = box_muller(r, k);
                lsr[k] = out[A + k];
                const float ls = fminf(fmaxf(lsr[k], LOG_STD_MIN), LOG_STD_MAX);
                std_[k] = expf(ls);
                const float u = __fadd_rn(out[k], __fmul_rn(std_[k], eps[k]));
                sd[k] = __fadd_rn(std_[k], SQUASH_EPS);
                zz[k] = __fdiv_rn(__fsub_rn(u, out[k]), sd[k]);
                lp1 = __fadd_rn(lp1, __fmul_rn(-0.5f, __fadd_rn(__fadd_rn(__fmul_rn(zz[k], zz[k]), __fmul_rn(2.0f, ls)), LOG_2PI)));
                ap[k] = tanhf(u);
                lp2 = __fadd_rn(lp2, logf(__fadd_rn(__fsub_rn(1.0f, __fmul_rn(ap[k], ap[k])), SQUASH_EPS)));
                xs[W + k] = ap[k];
            }
        }
        const float lp = __fsub_rn(lp1, lp2);
        a.logp[b] = lp;
        // v_backup = min(qf1, qf2)(s, a_pi) - alpha logp, and qf1's input gradient at a_pi
        float q2[1];
        unsigned long long n1, n2;
        mlp_fwd<1>(qf2, W + A, 1, xs, q2, n1, n2);
        mlp_fwd<1>(qf1, W + A, 1, xs, o1, m1, m2);
        a.vb[b] = __fsub_rn(fminf(o1[0], q2[0]), __fmul_rn(alpha, lp));
        float dq[MAXA];
        mlp_input_grad(qf1, m1, m2, W, A, dq);
        // d policy_loss / d (mu, raw log_std) of this sample, policy_loss = mean(alpha logp - qf1(s, a_pi))
        const float invB = 1.0f / (float)a.B;
#pragma unroll
        for (int k = 0; k < MAXA; ++k) if (k < A) {
            const float one_m = 1.0f - ap[k] * ap[k];
            const float T = 2.0f * ap[k] * one_m / (one_m + SQUASH_EPS);      // d(-log(1 - a^2 + 1e-6)) / du
            const float se = std_[k] * eps[k];                                  // du / dls (and d(u - mu) / dls)
            const float dz = se / sd[k] - zz[k] * std_[k] / sd[k];               // d zz / dls
            const float dlp_dls = -zz[k] * dz - 1.0f + T * se;
            const float dq_du = dq[k] * one_m;
            a.dact[(size_t)b * 2 * A + k] = (alpha * T - dq_du) * invB;
            const bool live = lsr[k] >= LOG_STD_MIN && lsr[k] <= LOG_STD_MAX;  // tf.clip_by_value's gradient
            a.dact[(size_t)b * 2 * A + A + k] = live ? (alpha * dlp_dls - dq_du * se) * invB : 0.f;
        }
        ent_term = (double)__fadd_rn(lp, a.target_entropy);
    }
    // -mean(logp + target_entropy): per-CTA float64 sums in a fixed order, combined in CTA order by the last CTA
    for (int o = 16; o > 0; o >>= 1) ent_term += __shfl_xor_sync(0xffffffffu, ent_term, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ent_term;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < PREP_NT / 32; ++w) s += red[w];
        a.partial[blockIdx.x] = s;
    }
    if (last_cta_advance(a.rng, counter)) {
        double s = 0.0;
        for (int c = 0; c < (int)gridDim.x; ++c) s += *(volatile double*)(a.partial + c);
        *a.ent_grad = a.auto_ent && a.step[0] > 0 ? (float)(-s / (double)a.B) : 0.f;
    }
}

// ---- srl_sac_grad: chunks of CH samples, GNT threads; thread tiles as ppo2_kernels.cu's (samples 4 eg + e, units og + 16 k) ----
constexpr int CH = 64, GNT = 256, WS = H + 4, W1S = DINMAX + 1, GS = OUTMAX + 1, G1 = (H * DINMAX + GNT - 1) / GNT;
constexpr int GRAD_FLOATS = H * W1S + 2 * H * WS + OUTMAX * WS + 4 * CH * WS + CH * W1S + CH * GS + 2 * H + OUTMAX;
static_assert((H * W1S) % 4 == 0 && (CH * W1S) % 4 == 0, "16-byte aligned regions");

struct GradArgs {
    Layout L; int W, A, B; const float* arena; const float* obs; const float* act; const long long* idx;
    const float* qb; const float* vb; const float* dact; float* partial;
};

__device__ __forceinline__ void tile_matvec(const float* Wm, const float* bias, const float* in, int eg, int og, float (&out)[4][4]) {
    float s[4][4][4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int k = 0; k < 4; ++k) { s[e][k][0] = bias ? bias[og + 16 * k] : 0.f; s[e][k][1] = 0.f; s[e][k][2] = 0.f; s[e][k][3] = 0.f; }
#pragma unroll 2
    for (int i4 = 0; i4 < H / 4; ++i4) {
        float4 w[4], x[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) w[k] = *reinterpret_cast<const float4*>(Wm + (og + 16 * k) * WS + 4 * i4);
#pragma unroll
        for (int e = 0; e < 4; ++e) x[e] = *reinterpret_cast<const float4*>(in + (4 * eg + e) * WS + 4 * i4);
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                s[e][k][0] = fmaf(w[k].x, x[e].x, s[e][k][0]); s[e][k][1] = fmaf(w[k].y, x[e].y, s[e][k][1]);
                s[e][k][2] = fmaf(w[k].z, x[e].z, s[e][k][2]); s[e][k][3] = fmaf(w[k].w, x[e].w, s[e][k][3]);
            }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int k = 0; k < 4; ++k) out[e][k] = (s[e][k][0] + s[e][k][1]) + (s[e][k][2] + s[e][k][3]);
}

__global__ void __launch_bounds__(GNT, 1) sac_grad_kernel(const __grid_constant__ GradArgs a) {
    extern __shared__ __align__(16) float sm[];
    const int net = blockIdx.y, t = threadIdx.x, W = a.W, A = a.A;
    const NetOff o = a.L.net[net];
    const int din = o.in, dout = o.out;
    float* w1 = sm;                  float* w2 = w1 + H * W1S;        float* w2T = w2 + H * WS;       float* w3 = w2T + H * WS;
    float* h1 = w3 + OUTMAX * WS;    float* h2 = h1 + CH * WS;        float* d2 = h2 + CH * WS;       float* d1 = d2 + CH * WS;
    float* xs = d1 + CH * WS;        float* g3 = xs + CH * W1S;       float* b1 = g3 + CH * GS;       float* b2 = b1 + H;      float* b3 = b2 + H;
    const float* P = a.arena;
    for (int e = t; e < H * din; e += GNT) w1[(e / din) * W1S + e % din] = P[o.w1 + e];
    for (int e = t; e < H * H; e += GNT) { const int j = e >> 6, i = e & 63; const float w = P[o.w2 + e]; w2[j * WS + i] = w; w2T[i * WS + j] = w; }
    for (int e = t; e < dout * H; e += GNT) w3[(e >> 6) * WS + (e & 63)] = P[o.w3 + e];
    for (int e = t; e < H; e += GNT) { b1[e] = P[o.b1 + e]; b2[e] = P[o.b2 + e]; }
    if (t < dout) b3[t] = P[o.b3 + t];
    const float invB = 1.0f / (float)a.B;
    const int eg = t >> 4, og = t & 15, jq = t >> 4, iq = t & 15;
    float gw2[4][4], gw3[4] = {0.f, 0.f, 0.f, 0.f}, gw1[G1], gb = 0.f, gb1 = 0.f;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) gw2[jj][ii] = 0.f;
#pragma unroll
    for (int m = 0; m < G1; ++m) gw1[m] = 0.f;
    const int nchunks = (a.B + CH - 1) / CH;
    for (int c = blockIdx.x; c < nchunks; c += gridDim.x) {
        __syncthreads();                              // the previous chunk's reads are done
        for (int j = t; j < CH * din; j += GNT) {
            const int n = j / din, d = j % din, s = c * CH + n;
            float v = 0.f;
            const long long g = s < a.B ? a.idx[s] : -1;
            if (g >= 0) v = d < W ? a.obs[g * W + d] : a.act[g * A + (d - W)];
            xs[n * W1S + d] = v;
        }
        __syncthreads();
        {   // layer 1
            float acc[4][4];
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[e][k] = b1[og + 16 * k];
            for (int d = 0; d < din; ++d) {
                float w[4], x[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) w[k] = w1[(og + 16 * k) * W1S + d];
#pragma unroll
                for (int e = 0; e < 4; ++e) x[e] = xs[(4 * eg + e) * W1S + d];
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int k = 0; k < 4; ++k) acc[e][k] = fmaf(w[k], x[e], acc[e][k]);
            }
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) h1[(4 * eg + e) * WS + og + 16 * k] = fmaxf(acc[e][k], 0.f);
        }
        __syncthreads();
        {   // layer 2
            float z[4][4];
            tile_matvec(w2, b2, h1, eg, og, z);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) h2[(4 * eg + e) * WS + og + 16 * k] = fmaxf(z[e][k], 0.f);
        }
        __syncthreads();
        if (t < CH) {   // head derivatives: the actor's from srl_sac_prepare, the critics' (out - target) / B
            const int s = c * CH + t;
            const bool live = s < a.B && a.idx[s] >= 0;
            if (net == ACTOR) {
                for (int k = 0; k < dout; ++k) g3[t * GS + k] = live ? a.dact[(size_t)s * dout + k] : 0.f;
            } else {
                float s0 = b3[0], s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
                for (int i4 = 0; i4 < H / 4; ++i4) {
                    const float4 w = *reinterpret_cast<const float4*>(w3 + 4 * i4), x = *reinterpret_cast<const float4*>(h2 + t * WS + 4 * i4);
                    s0 = fmaf(w.x, x.x, s0); s1 = fmaf(w.y, x.y, s1); s2 = fmaf(w.z, x.z, s2); s3 = fmaf(w.w, x.w, s3);
                }
                const float q = (s0 + s1) + (s2 + s3);
                g3[t * GS] = live ? __fmul_rn(__fsub_rn(q, net == VF ? a.vb[s] : a.qb[s]), invB) : 0.f;
            }
        }
        __syncthreads();
#pragma unroll
        for (int e = 0; e < 4; ++e) {    // delta of layer 2
            const int n = 4 * eg + e;
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) {
                const int j = og + 16 * k4;
                float s = 0.f;
                for (int k = 0; k < dout; ++k) s = fmaf(w3[k * WS + j], g3[n * GS + k], s);
                d2[n * WS + j] = h2[n * WS + j] > 0.f ? s : 0.f;
            }
        }
        __syncthreads();
#pragma unroll
        for (int m = 0; m < 4; ++m) {    // layer 3
            const int e = t + GNT * m;
            if (e < dout * H) {
                const int k = e >> 6, j = e & 63;
                float s = 0.f;
#pragma unroll 8
                for (int n = 0; n < CH; ++n) s = fmaf(g3[n * GS + k], h2[n * WS + j], s);
                gw3[m] += s;
            }
        }
        if (t < dout) { float s = 0.f; for (int n = 0; n < CH; ++n) s += g3[n * GS + t]; gb += s; }
        else if (t >= H && t < 2 * H) { float s = 0.f; for (int n = 0; n < CH; ++n) s += d2[n * WS + (t - H)]; gb += s; }
#pragma unroll 4
        for (int n = 0; n < CH; ++n) {   // layer 2: the 4 x 4 patch rows 4 jq + jj, columns 4 iq + ii
            const float4 dq = *reinterpret_cast<const float4*>(d2 + n * WS + 4 * jq), hq = *reinterpret_cast<const float4*>(h1 + n * WS + 4 * iq);
            const float dd[4] = {dq.x, dq.y, dq.z, dq.w}, hh[4] = {hq.x, hq.y, hq.z, hq.w};
#pragma unroll
            for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int ii = 0; ii < 4; ++ii) gw2[jj][ii] = fmaf(dd[jj], hh[ii], gw2[jj][ii]);
        }
        {   // delta of layer 1 = (W2^T delta 2) masked by layer 1's ReLU
            float z[4][4];
            tile_matvec(w2T, nullptr, d2, eg, og, z);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) { const int q = (4 * eg + e) * WS + og + 16 * k; d1[q] = h1[q] > 0.f ? z[e][k] : 0.f; }
        }
        __syncthreads();
        if (t < H) { float s = 0.f; for (int n = 0; n < CH; ++n) s += d1[n * WS + t]; gb1 += s; }
#pragma unroll
        for (int m = 0; m < G1; ++m) {   // layer 1
            const int e = t + GNT * m;
            if (e < H * din) {
                const int i = e / din, d = e % din;
                float s = 0.f;
#pragma unroll 8
                for (int n = 0; n < CH; ++n) s = fmaf(d1[n * WS + i], xs[n * W1S + d], s);
                gw1[m] += s;
            }
        }
    }
    float* out = a.partial + (size_t)blockIdx.x * a.L.P;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) out[o.w2 + (4 * jq + jj) * H + 4 * iq + ii] = gw2[jj][ii];
#pragma unroll
    for (int m = 0; m < 4; ++m) if (t + GNT * m < dout * H) out[o.w3 + t + GNT * m] = gw3[m];
#pragma unroll
    for (int m = 0; m < G1; ++m) if (t + GNT * m < H * din) out[o.w1 + t + GNT * m] = gw1[m];
    if (t < dout) out[o.b3 + t] = gb;
    else if (t >= H && t < 2 * H) out[o.b2 + (t - H)] = gb;
    if (t < H) out[o.b1 + t] = gb1;
}

// grad[e] = sum over CTAs c in order of partial[c][e] (float64), every entry but log_ent_coef's
__global__ void __launch_bounds__(256) sac_grad_reduce_kernel(int P, int ctas, const float* __restrict__ partial, float* __restrict__ grad) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= P - 1) return;
    double s = 0.0;
    for (int c = 0; c < ctas; ++c) s += (double)partial[(size_t)c * P + e];
    grad[e] = (float)s;
}

// ---- srl_sac_adam: one CTA; each thread updates its entries and, inside vf, the target entries they feed ----
constexpr int ADAM_NT = 1024;
struct AdamArgs { Layout L; float* arena; float* target; const float* g; float* m; float* v; const float* lr; float* beta_power; float beta1, beta2, eps, tau; int polyak; };
__global__ void __launch_bounds__(ADAM_NT, 1) sac_adam_kernel(const __grid_constant__ AdamArgs o) {
    const float lr = *o.lr, b1p = o.beta_power[0], b2p = o.beta_power[1];
    const float lr_t = __fdiv_rn(__fmul_rn(lr, __fsqrt_rn(__fsub_rn(1.0f, b2p))), __fsub_rn(1.0f, b1p));   // lr sqrt(1 - beta2^t) / (1 - beta1^t)
    const float r1 = __fsub_rn(1.0f, o.beta1), r2 = __fsub_rn(1.0f, o.beta2), keep = __fsub_rn(1.0f, o.tau);
    const int vlo = o.L.net[VF].w1, vhi = o.L.net[VF].end;
    for (int e = threadIdx.x; e < o.L.P; e += ADAM_NT) {
        const float g = o.g[e];
        const float m = __fadd_rn(o.m[e], __fmul_rn(__fsub_rn(g, o.m[e]), r1));                  // m += (g - m) (1 - beta1)
        const float v = __fadd_rn(o.v[e], __fmul_rn(__fsub_rn(__fmul_rn(g, g), o.v[e]), r2));    // v += (g^2 - v) (1 - beta2)
        o.m[e] = m; o.v[e] = v;
        const float w = __fsub_rn(o.arena[e], __fdiv_rn(__fmul_rn(m, lr_t), __fadd_rn(__fsqrt_rn(v), o.eps)));   // w -= m lr_t / (sqrt(v) + eps)
        o.arena[e] = w;
        if (o.polyak && e >= vlo && e < vhi)
            o.target[e - vlo] = __fadd_rn(__fmul_rn(keep, o.target[e - vlo]), __fmul_rn(o.tau, w));               // (1 - tau) target + tau vf
    }
    __syncthreads();
    if (threadIdx.x == 0) { o.beta_power[0] = __fmul_rn(b1p, o.beta1); o.beta_power[1] = __fmul_rn(b2p, o.beta2); }
}

int nets_ok(const char* who, const srl_sac_nets* s) {
    if (!s) { srl_set_error("%s: null nets", who); return 0; }
    if (s->struct_size != sizeof(srl_sac_nets)) { srl_set_error("%s: srl_sac_nets size mismatch", who); return 0; }
    if (s->obs_dim < 1 || s->obs_dim > MAXW || s->act_dim < 1 || s->act_dim > MAXA) {
        srl_set_error("%s: unsupported shape obs_dim=%d act_dim=%d (obs_dim 1..%d, act_dim 1..%d)", who, s->obs_dim, s->act_dim, MAXW, MAXA);
        return 0;
    }
    if (!s->arena || !s->target) { srl_set_error("%s: null arena or target", who); return 0; }
    return 1;
}

int sms_of_device() {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return sms;
}
int grad_ctas(int batch) {
    const int sms = sms_of_device(), chunks = (batch + CH - 1) / CH;
    return sms <= 0 ? 0 : (chunks < sms ? chunks : sms);
}
int prep_ctas(int batch) { return (batch + PREP_NT - 1) / PREP_NT; }

}  // namespace

extern "C" {

size_t srl_sac_arena_floats(int obs_dim, int act_dim) {
    if (obs_dim < 1 || obs_dim > MAXW || act_dim < 1 || act_dim > MAXA) return 0;
    return (size_t)make_layout(obs_dim, act_dim).P;
}

size_t srl_sac_workspace_bytes(int obs_dim, int act_dim, int batch) {
    if (obs_dim < 1 || obs_dim > MAXW || act_dim < 1 || act_dim > MAXA || batch < 1) {
        srl_set_error("sac_workspace_bytes: unsupported shape obs_dim=%d act_dim=%d batch=%d", obs_dim, act_dim, batch);
        return 0;
    }
    const int ctas = grad_ctas(batch);
    if (ctas <= 0) { srl_set_error("sac_workspace_bytes: no CUDA device"); return 0; }
    const size_t grad = sizeof(float) * (size_t)make_layout(obs_dim, act_dim).P * (size_t)ctas, prep = sizeof(double) * (size_t)prep_ctas(batch);
    return grad > prep ? grad : prep;
}

int srl_sac_act(const srl_sac_nets* nets, int n, const float* obs, int mode, uint64_t* rng, uint64_t env_offset, float* act_out, void* stream) {
    if (!nets_ok("sac_act", nets)) return 1;
    if (!rng || !act_out || (mode != 2 && !obs)) { srl_set_error("sac_act: null argument"); return 1; }
    if (n <= 0) { srl_set_error("sac_act: n must be positive"); return 1; }
    if (mode < 0 || mode > 2) { srl_set_error("sac_act: mode %d is not 0 (sample), 1 (deterministic) or 2 (random)", mode); return 1; }
    ActArgs a;
    a.L = make_layout(nets->obs_dim, nets->act_dim); a.W = nets->obs_dim; a.A = nets->act_dim; a.n = n; a.mode = mode; a.arena = nets->arena;
    a.obs = obs; a.rng = reinterpret_cast<unsigned long long*>(rng); a.env_offset = env_offset; a.act = act_out;
    constexpr size_t smem = sizeof(float) * (NET_FLOATS + ACT_NT * XS);
    SRL_CUDA_OK(srl_smem_opt_in<sac_act_kernel>(smem));
    sac_act_kernel<<<(n + ACT_NT - 1) / ACT_NT, ACT_NT, smem, (cudaStream_t)stream>>>(a);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_sac_store(int rows, int n, int obs_dim, int act_dim, int64_t* step, float* obs, const float* act, const float* rew, const uint8_t* done,
                  const float* new_obs, float* obs_ring, float* act_ring, float* rew_ring, uint8_t* done_ring, float* next_obs_ring, void* stream) {
    if (!step || !obs || !act || !rew || !done || !new_obs || !obs_ring || !act_ring || !rew_ring || !done_ring || !next_obs_ring) {
        srl_set_error("sac_store: null argument"); return 1;
    }
    if (rows < 1 || n < 1 || obs_dim < 1 || obs_dim > MAXW || act_dim < 1 || act_dim > MAXA) {
        srl_set_error("sac_store: unsupported shape rows=%d n=%d obs_dim=%d act_dim=%d", rows, n, obs_dim, act_dim); return 1;
    }
    StoreArgs a;
    a.rows = rows; a.n = n; a.W = obs_dim; a.A = act_dim; a.step = reinterpret_cast<long long*>(step); a.obs = obs; a.act = act; a.rew = rew; a.done = done;
    a.new_obs = new_obs; a.obs_ring = obs_ring; a.act_ring = act_ring; a.rew_ring = rew_ring; a.done_ring = done_ring; a.next_obs_ring = next_obs_ring;
    const size_t widest = (size_t)n * (size_t)(obs_dim > act_dim ? obs_dim : act_dim);
    sac_store_kernel<<<(unsigned)((widest + STORE_NT - 1) / STORE_NT), STORE_NT, 0, (cudaStream_t)stream>>>(a);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_sac_prepare(const srl_sac_nets* nets, int rows, int n, const int64_t* step, const float* obs_ring, const float* act_ring, const float* rew_ring,
                    const uint8_t* done_ring, const float* next_obs_ring, int batch, float gamma, int auto_ent, float ent_coef, float target_entropy,
                    uint64_t* rng, int64_t* idx, float* q_backup, float* v_backup, float* logp, float* d_actor, float* ent_grad, void* workspace,
                    size_t workspace_bytes, void* stream) {
    if (!nets_ok("sac_prepare", nets)) return 1;
    if (!step || !obs_ring || !act_ring || !rew_ring || !done_ring || !next_obs_ring || !rng || !idx || !q_backup || !v_backup || !logp || !d_actor ||
        !ent_grad || !workspace) { srl_set_error("sac_prepare: null argument"); return 1; }
    if (rows < 1 || n < 1 || batch < 1) { srl_set_error("sac_prepare: rows, n and batch must be positive"); return 1; }
    if (workspace_bytes < sizeof(double) * (size_t)prep_ctas(batch)) { srl_set_error("sac_prepare: workspace too small (srl_sac_workspace_bytes)"); return 1; }
    PrepArgs a;
    a.L = make_layout(nets->obs_dim, nets->act_dim); a.W = nets->obs_dim; a.A = nets->act_dim; a.rows = rows; a.n = n; a.B = batch; a.auto_ent = auto_ent ? 1 : 0;
    a.arena = nets->arena; a.target = nets->target; a.step = reinterpret_cast<const long long*>(step);
    a.obs = obs_ring; a.act = act_ring; a.rew = rew_ring; a.done = done_ring; a.next_obs = next_obs_ring;
    a.gamma = gamma; a.ent_coef = ent_coef; a.target_entropy = target_entropy;
    a.rng = reinterpret_cast<unsigned long long*>(rng); a.idx = reinterpret_cast<long long*>(idx); a.qb = q_backup; a.vb = v_backup; a.logp = logp;
    a.dact = d_actor; a.ent_grad = ent_grad; a.partial = reinterpret_cast<double*>(workspace);
    constexpr size_t smem = sizeof(float) * (4 * NET_FLOATS + PREP_NT * XS);
    static_assert(smem <= 227 * 1024, "shared memory of one CTA");
    SRL_CUDA_OK(srl_smem_opt_in<sac_prepare_kernel>(smem));
    sac_prepare_kernel<<<prep_ctas(batch), PREP_NT, smem, (cudaStream_t)stream>>>(a);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_sac_grad(const srl_sac_nets* nets, int n, const float* obs_ring, const float* act_ring, int batch, const int64_t* idx, const float* q_backup,
                 const float* v_backup, const float* d_actor, float* grad, void* workspace, size_t workspace_bytes, void* stream) {
    (void)n;
    if (!nets_ok("sac_grad", nets)) return 1;
    if (!obs_ring || !act_ring || !idx || !q_backup || !v_backup || !d_actor || !grad || !workspace) { srl_set_error("sac_grad: null argument"); return 1; }
    if (batch < 1) { srl_set_error("sac_grad: batch must be positive"); return 1; }
    const int ctas = grad_ctas(batch);
    if (ctas <= 0) { srl_set_error("sac_grad: no CUDA device"); return 1; }
    GradArgs a;
    a.L = make_layout(nets->obs_dim, nets->act_dim); a.W = nets->obs_dim; a.A = nets->act_dim; a.B = batch; a.arena = nets->arena;
    a.obs = obs_ring; a.act = act_ring; a.idx = reinterpret_cast<const long long*>(idx); a.qb = q_backup; a.vb = v_backup; a.dact = d_actor;
    a.partial = reinterpret_cast<float*>(workspace);
    if (workspace_bytes < sizeof(float) * (size_t)a.L.P * (size_t)ctas) { srl_set_error("sac_grad: workspace too small (srl_sac_workspace_bytes)"); return 1; }
    constexpr size_t smem = sizeof(float) * GRAD_FLOATS;
    static_assert(smem <= 227 * 1024, "shared memory of one CTA");
    cudaStream_t st = (cudaStream_t)stream;
    SRL_CUDA_OK(srl_smem_opt_in<sac_grad_kernel>(smem));
    sac_grad_kernel<<<dim3(ctas, NNETS), GNT, smem, st>>>(a);
    SRL_CUDA_OK(cudaGetLastError());
    sac_grad_reduce_kernel<<<(a.L.P + 255) / 256, 256, 0, st>>>(a.L.P, ctas, a.partial, grad);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_sac_adam(const srl_sac_nets* nets, const float* grad, float* m, float* v, const float* lr, float* beta_power, float beta1, float beta2,
                 float epsilon, int polyak, float tau, void* stream) {
    if (!nets_ok("sac_adam", nets)) return 1;
    if (!grad || !m || !v || !lr || !beta_power) { srl_set_error("sac_adam: null argument"); return 1; }
    if (!(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && epsilon >= 0.f && tau >= 0.f && tau <= 1.f)) {
        srl_set_error("sac_adam: need 0 <= beta1, beta2 < 1, epsilon >= 0, 0 <= tau <= 1 (got %g, %g, %g, %g)", beta1, beta2, epsilon, tau); return 1;
    }
    AdamArgs o;
    o.L = make_layout(nets->obs_dim, nets->act_dim); o.arena = nets->arena; o.target = nets->target; o.g = grad; o.m = m; o.v = v; o.lr = lr;
    o.beta_power = beta_power; o.beta1 = beta1; o.beta2 = beta2; o.eps = epsilon; o.tau = tau; o.polyak = polyak ? 1 : 0;
    sac_adam_kernel<<<1, ADAM_NT, 0, (cudaStream_t)stream>>>(o);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
