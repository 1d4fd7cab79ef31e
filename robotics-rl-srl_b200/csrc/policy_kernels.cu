// PPO2 consumer helpers (include/srl_policy.h): the per-step policy forward + sample and the VecNormalize observation filter as ONE
// launch each, so that a captured rollout is three launches per env step (policy, simulator, filter) instead of ~60 small torch
// kernels around the simulator's.  Per-env arithmetic lives in policy_core.h (shared with the CPU checker of the tests).
#include <cuda_runtime.h>
#include "common.cuh"
#include "policy_tile.cuh"
#include "policy_core.h"
#include "../../include/srl_policy.h"

namespace {

struct PolicyArgs {
    srl_mlp_policy p;
    int n;
    const float* obs;
    unsigned long long* rng;
    unsigned long long env_offset;
    float* obs_buf; void* act_env; void* act_buf; float* logp; float* value;
};

// MO: the observation width class (SRL_POLICY_MAX_OBS or SRL_POLICY_WIDE_OBS), which sets the stride of the staged observation rows and of W1
// (tower_tiled); the wide class zero-fills the padding both read.
template <int MO>
__global__ void __launch_bounds__(POLICY_BLOCK) policy_act_kernel(const __grid_constant__ PolicyArgs a) {
    extern __shared__ __align__(16) float smem[];
    constexpr int W1S = w1_stride<MO>();
    const int D = a.p.obs_dim, A = a.p.n_out;
    float* pi_w2 = smem;                 float* vf_w2 = pi_w2 + H * WS;
    float* pi_w3 = vf_w2 + H * WS;       float* vf_w3 = pi_w3 + SRL_POLICY_MAX_OUT * WS;
    float* ha = vf_w3 + WS;              float* hb = ha + POLICY_ENVS * WS;       // [POLICY_ENVS][WS] activation columns (16-byte aligned)
    float* pi_w1 = hb + POLICY_ENVS * WS;            float* vf_w1 = pi_w1 + H * W1S;
    float* pi_b1 = vf_w1 + H * W1S;                  float* vf_b1 = pi_b1 + H;
    float* pi_b2 = vf_b1 + H;            float* vf_b2 = pi_b2 + H;
    float* pi_b3 = vf_b2 + H;            float* vf_b3 = pi_b3 + SRL_POLICY_MAX_OUT;
    float* s_logstd = vf_b3 + 4;         float* outs = s_logstd + SRL_POLICY_MAX_OUT;   // [POLICY_ENVS][SRL_POLICY_MAX_OUT + 1]: logits / mean, value
    float* xs = outs + POLICY_ENVS * (SRL_POLICY_MAX_OUT + 1);                           // [POLICY_ENVS][MO] observations
    {
        constexpr int W2PER = H * (H / 4) / POLICY_BLOCK, W3PER = (SRL_POLICY_MAX_OUT * (H / 4) + POLICY_BLOCK - 1) / POLICY_BLOCK;
        constexpr int W1PER = (H * MO + POLICY_BLOCK - 1) / POLICY_BLOCK, XPER = (POLICY_ENVS * MO + POLICY_BLOCK - 1) / POLICY_BLOCK;
        static_assert(H * (H / 4) % POLICY_BLOCK == 0 && H <= POLICY_BLOCK && SRL_POLICY_MAX_OUT <= POLICY_BLOCK, "staging shape");
        const bool vec = ((reinterpret_cast<uintptr_t>(a.p.pi_w2) | reinterpret_cast<uintptr_t>(a.p.vf_w2) | reinterpret_cast<uintptr_t>(a.p.pi_w3) |
                           reinterpret_cast<uintptr_t>(a.p.vf_w3)) & 15u) == 0;
        RowRegs<W2PER> r_pw2, r_vw2; RowRegs<W3PER> r_pw3; RowRegs<1> r_vw3;
        VecRegs<W1PER> r_pw1, r_vw1; VecRegs<1> r_pb1, r_vb1, r_pb2, r_vb2, r_pb3, r_vb3, r_ls; VecRegs<XPER> r_x;
        rows_load(r_pw2, a.p.pi_w2, H, vec); rows_load(r_vw2, a.p.vf_w2, H, vec); rows_load(r_pw3, a.p.pi_w3, A, vec); rows_load(r_vw3, a.p.vf_w3, 1, vec);
        vec_load(r_pw1, a.p.pi_w1, H * D); vec_load(r_vw1, a.p.vf_w1, H * D);
        vec_load(r_pb1, a.p.pi_b1, H); vec_load(r_vb1, a.p.vf_b1, H); vec_load(r_pb2, a.p.pi_b2, H); vec_load(r_vb2, a.p.vf_b2, H);
        vec_load(r_pb3, a.p.pi_b3, A); vec_load(r_vb3, a.p.vf_b3, 1);
        vec_load(r_ls, a.p.discrete ? a.p.pi_b3 : a.p.logstd, a.p.discrete ? 0 : A);
        // this CTA's observations: a contiguous run of (up to) 32 D floats
        const int first = blockIdx.x * POLICY_ENVS, nx = min(POLICY_ENVS, a.n - first) * D;
        vec_load(r_x, a.obs + (size_t)first * D, nx);
        rows_store(r_pw2, pi_w2, H); rows_store(r_vw2, vf_w2, H); rows_store(r_pw3, pi_w3, A); rows_store(r_vw3, vf_w3, 1);
        if constexpr (MO == SRL_POLICY_MAX_OBS) {
            vec_store(r_pw1, pi_w1, H * D); vec_store(r_vw1, vf_w1, H * D);
        } else {                                             // [64][D] -> [64][W1S], zero past D (disjoint from the weight stores)
#pragma unroll
            for (int k = 0; k < W1PER; ++k) {
                const int i = threadIdx.x + k * POLICY_BLOCK;
                if (i < H * D) { pi_w1[(i / D) * W1S + i % D] = r_pw1.v[k]; vf_w1[(i / D) * W1S + i % D] = r_vw1.v[k]; }
            }
            for (int j = threadIdx.x; j < H * W1S; j += POLICY_BLOCK)
                if (j % W1S >= D) { pi_w1[j] = 0.f; vf_w1[j] = 0.f; }
            for (int j = threadIdx.x; j < POLICY_ENVS * MO; j += POLICY_BLOCK)
                if (j % MO >= D) xs[j] = 0.f;
        }
        vec_store(r_pb1, pi_b1, H); vec_store(r_vb1, vf_b1, H); vec_store(r_pb2, pi_b2, H); vec_store(r_vb2, vf_b2, H);
        vec_store(r_pb3, pi_b3, A); vec_store(r_vb3, vf_b3, 1);
        vec_store(r_ls, s_logstd, a.p.discrete ? 0 : A);
#pragma unroll
        for (int k = 0; k < XPER; ++k) {                     // [env][D] -> [env][8]; envs past n read as zeros (their results are never stored)
            const int j = threadIdx.x + k * POLICY_BLOCK;
            if (j < POLICY_ENVS * D) xs[(j / D) * MO + (j % D)] = r_x.v[k];
            if (a.obs_buf && j < nx) a.obs_buf[(size_t)first * D + j] = r_x.v[k];
        }
    }
    const unsigned long long seed = a.rng[0], counter = a.rng[1];    // read before this CTA arrives: the counter moves only after ALL CTAs arrived
    __syncthreads();
    const TowerSmem Wpi = {pi_w1, pi_b1, pi_w2, pi_b2, pi_w3, pi_b3};
    const TowerSmem Wvf = {vf_w1, vf_b1, vf_w2, vf_b2, vf_w3, vf_b3};
    tower_tiled<MO>(Wpi, D, A, xs, ha, hb, outs, SRL_POLICY_MAX_OUT + 1);
    tower_tiled<MO>(Wvf, D, 1, xs, ha, hb, outs + SRL_POLICY_MAX_OUT, SRL_POLICY_MAX_OUT + 1);   // its layer 1 rewrites `ha`, last read before the previous tower's second barrier
    __syncwarp();                                            // an env's outputs were written by the 4 lanes t / 4 = env of this warp
    const int slot = threadIdx.x >> 2, u = threadIdx.x & 3;
    const int i = blockIdx.x * POLICY_ENVS + slot;
    if (i < a.n && u == 0) {                                 // the lead lane of each env samples and stores
        const float* out = outs + slot * (SRL_POLICY_MAX_OUT + 1);
        float lg[SRL_POLICY_MAX_OUT];
        for (int k = 0; k < A; ++k) lg[k] = out[k];
        a.value[i] = out[SRL_POLICY_MAX_OUT];
        const unsigned long long env = a.env_offset + (unsigned long long)i;
        float lp;
        if (a.p.discrete) {
            const int act = srl_sample_categorical(lg, A, seed, env, (uint32_t)counter, &lp);
            reinterpret_cast<int32_t*>(a.act_env)[i] = act;
            if (a.act_buf) reinterpret_cast<long long*>(a.act_buf)[i] = (long long)act;
        } else {
            float smp[SRL_POLICY_MAX_OUT], clp[SRL_POLICY_MAX_OUT];
            srl_sample_gaussian(lg, s_logstd, A, seed, env, (uint32_t)counter, smp, clp, &lp);
            for (int k = 0; k < A; ++k) {
                reinterpret_cast<float*>(a.act_env)[(size_t)i * A + k] = clp[k];
                if (a.act_buf) reinterpret_cast<float*>(a.act_buf)[(size_t)i * A + k] = smp[k];
            }
        }
        a.logp[i] = lp;
    }
    // the LAST CTA to retire advances the step counter: every CTA has read it by then, and the next launch sees the new value
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long arrived = atomicAdd(a.rng + 2, 1ull);
        if (arrived == (unsigned long long)gridDim.x - 1ull) {
            a.rng[2] = 0ull;
            a.rng[1] = counter + 1ull;
            __threadfence();
        }
    }
}

constexpr int FILTER_BLOCK = 1024;

// One CTA: batch mean and biased variance in float64, Chan's parallel-variance merge into the running state (the update of stable-baselines'
// RunningMeanStd), then the normalisation of the whole batch in float32.  ONE pass over the batch: the sums S1 = sum(x - m0), S2 = sum((x - m0)^2)
// are taken about the running mean m0 (known before the batch is read), so mean = m0 + S1 / n and var = S2 / n - (S1 / n)^2 lose nothing to
// cancellation (|x - m0| is of the order of the standard deviation; float64 throughout: ~1e-13 of numpy's two-pass result at n = 4096), one
// block reduction of 2 D values instead of two of D with a second read in between, the D state updates by D threads.  D is a template
// parameter: every per-dimension array is registers (a run-time D put them in local memory: the first one-pass version was SLOWER than
// two passes), and a thread keeps its envs' observations in registers between the statistics and the normalisation (one read of the batch).
// Every phase of this kernel is a latency; there is no throughput to speak of.
template <int D>
__global__ void __launch_bounds__(FILTER_BLOCK) obs_filter_kernel(int n, const float* __restrict__ obs, double* state, int update,
                                                                   float clip, float eps, float* __restrict__ out) {
    constexpr int KEEP = 4;              // envs per thread held in registers (n <= KEEP * FILTER_BLOCK: the trainer's 4096); beyond that re-read
    __shared__ double red[32][2 * D];
    __shared__ double s_sum[2 * D];
    __shared__ float s_mf[D], s_inv[D];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float x[KEEP][D];
#pragma unroll
    for (int k = 0; k < KEEP; ++k) {
        const int i = tid + k * FILTER_BLOCK;
#pragma unroll
        for (int d = 0; d < D; ++d) x[k][d] = i < n ? obs[(size_t)i * D + d] : 0.f;
    }
    if (update) {
        double m0[D], acc[2 * D];
#pragma unroll
        for (int d = 0; d < D; ++d) { m0[d] = state[d]; acc[d] = 0.0; acc[D + d] = 0.0; }
#pragma unroll
        for (int k = 0; k < KEEP; ++k) {
            if (tid + k * FILTER_BLOCK < n) {
#pragma unroll
                for (int d = 0; d < D; ++d) { const double c = (double)x[k][d] - m0[d]; acc[d] += c; acc[D + d] = fma(c, c, acc[D + d]); }
            }
        }
        for (int i = tid + KEEP * FILTER_BLOCK; i < n; i += FILTER_BLOCK) {
#pragma unroll
            for (int d = 0; d < D; ++d) { const double c = (double)obs[(size_t)i * D + d] - m0[d]; acc[d] += c; acc[D + d] = fma(c, c, acc[D + d]); }
        }
#pragma unroll
        for (int q = 0; q < 2 * D; ++q) {
            double v = acc[q];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) red[warp][q] = v;
        }
        __syncthreads();
        if (warp == 0) {
#pragma unroll
            for (int q = 0; q < 2 * D; ++q) {
                double v = red[lane][q];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                if (lane == 0) s_sum[q] = v;
            }
        }
        __syncthreads();
        if (tid < D) {
            const int d = tid;
            const double count = state[2 * D], bc = (double)n, tot = count + bc;
            const double s1 = s_sum[d] / bc, bmean = state[d] + s1, bvar = s_sum[D + d] / bc - s1 * s1;
            const double mean = state[d], var = state[D + d], delta = bmean - mean;
            const double nm = mean + delta * bc / tot, nv = (var * count + bvar * bc + delta * delta * count * bc / tot) / tot;
            state[d] = nm; state[D + d] = nv;
            s_mf[d] = (float)nm; s_inv[d] = sqrtf((float)nv + eps);
        }
        __syncthreads();                 // every thread d < D has read the count before thread 0 moves it
        if (tid == 0) state[2 * D] += (double)n;
    } else {
        if (tid < D) { s_mf[tid] = (float)state[tid]; s_inv[tid] = sqrtf((float)state[D + tid] + eps); }
        __syncthreads();
    }
    float mf[D], sd[D];
#pragma unroll
    for (int d = 0; d < D; ++d) { mf[d] = s_mf[d]; sd[d] = s_inv[d]; }
#pragma unroll
    for (int k = 0; k < KEEP; ++k) {
        const int i = tid + k * FILTER_BLOCK;
        if (i < n) {
#pragma unroll
            for (int d = 0; d < D; ++d) out[(size_t)i * D + d] = fminf(fmaxf((x[k][d] - mf[d]) / sd[d], -clip), clip);
        }
    }
    for (int i = tid + KEEP * FILTER_BLOCK; i < n; i += FILTER_BLOCK) {
#pragma unroll
        for (int d = 0; d < D; ++d) out[(size_t)i * D + d] = fminf(fmaxf((obs[(size_t)i * D + d] - mf[d]) / sd[d], -clip), clip);
    }
}

// VecFrameStack + VecNormalize in one CTA: advance the caller's [n][W = k D] stack by the new observation, then filter the W-wide rows like
// obs_filter_kernel does (one pass about the running mean m0, float64 sums, the same merge and normalisation).  Thread t owns column t % W of
// rows t / W + R u (R = FILTER_BLOCK / W rows per slot, STACK_ROWS slots per pass): its sums are those of one column, so a column's total is one
// warp's reduction over the R threads of that column (W <= 32 = the number of warps).  The roll reads column c + D of the row it writes, which
// another thread of the same pass overwrites: every load of a pass precedes the barrier, every store follows it.  The second sweep re-reads
// the stack (L2-resident at the trainer's sizes): W <= 32 columns per row do not fit in registers the way obs_filter_kernel's <= 8 do.
constexpr int STACK_ROWS = 8;
__global__ void __launch_bounds__(FILTER_BLOCK) obs_stack_filter_kernel(int n, int D, int K, const float* __restrict__ obs, const uint8_t* __restrict__ done,
                                                                         float* stack, double* state, int update, float clip, float eps,
                                                                         float* __restrict__ out) {
    __shared__ double red[2][FILTER_BLOCK];
    __shared__ float s_mf[SRL_POLICY_WIDE_OBS], s_inv[SRL_POLICY_WIDE_OBS];
    const int W = D * K, keep = W - D, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int R = FILTER_BLOCK / W, r = tid / W, c = tid - r * W;
    const bool active = r < R;
    const double m0 = (update && active) ? state[c] : 0.0;
    double s1 = 0.0, s2 = 0.0;
    for (int base = 0; base < n; base += R * STACK_ROWS) {
        float v[STACK_ROWS];
#pragma unroll
        for (int u = 0; u < STACK_ROWS; ++u) {
            const int i = base + r + R * u;
            v[u] = 0.f;
            if (active && i < n) {
                if (c >= keep) v[u] = obs[(size_t)i * D + (c - keep)];                      // the newest frame: the last D columns
                else if (done && !done[i]) v[u] = stack[(size_t)i * W + c + D];           // roll left by D; a done env (or a reset: done == NULL) starts from zeros
            }
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < STACK_ROWS; ++u) {
            const int i = base + r + R * u;
            if (active && i < n) {
                stack[(size_t)i * W + c] = v[u];
                const double d = (double)v[u] - m0;
                s1 += d; s2 = fma(d, d, s2);
            }
        }
    }
    if (update) {
        red[0][tid] = s1; red[1][tid] = s2;
        __syncthreads();
        if (warp < W) {                  // warp w: column w, summed over the R threads that own it
            double a1 = 0.0, a2 = 0.0;
            for (int q = lane; q < R; q += 32) { a1 += red[0][q * W + warp]; a2 += red[1][q * W + warp]; }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { a1 += __shfl_xor_sync(0xffffffffu, a1, o); a2 += __shfl_xor_sync(0xffffffffu, a2, o); }
            if (lane == 0) {
                const int d = warp;
                const double count = state[2 * W], bc = (double)n, tot = count + bc;
                const double b1 = a1 / bc, bmean = state[d] + b1, bvar = a2 / bc - b1 * b1;
                const double mean = state[d], var = state[W + d], delta = bmean - mean;
                const double nm = mean + delta * bc / tot, nv = (var * count + bvar * bc + delta * delta * count * bc / tot) / tot;
                state[d] = nm; state[W + d] = nv;
                s_mf[d] = (float)nm; s_inv[d] = sqrtf((float)nv + eps);
            }
        }
        __syncthreads();                 // every column's lane 0 has read the count before thread 0 moves it
        if (tid == 0) state[2 * W] += (double)n;
    } else {
        if (tid < W) { s_mf[tid] = (float)state[tid]; s_inv[tid] = sqrtf((float)state[W + tid] + eps); }
        __syncthreads();                 // also orders the stack stores above before the reads below
    }
    const size_t total = (size_t)n * W;
    for (size_t e0 = tid; e0 < total; e0 += (size_t)4 * FILTER_BLOCK) {
        float x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { const size_t e = e0 + (size_t)u * FILTER_BLOCK; x[u] = e < total ? stack[e] : 0.f; }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const size_t e = e0 + (size_t)u * FILTER_BLOCK;
            if (e < total) { const int col = (int)(e % (size_t)W); out[e] = fminf(fmaxf((x[u] - s_mf[col]) / s_inv[col], -clip), clip); }
        }
    }
}

template <int MO>
constexpr size_t policy_smem_bytes() {
    return sizeof(float) * (size_t)(2 * H * WS + SRL_POLICY_MAX_OUT * WS + WS + 2 * POLICY_ENVS * WS + 2 * H * w1_stride<MO>() + 4 * H + SRL_POLICY_MAX_OUT + 4 +
                                    SRL_POLICY_MAX_OUT + POLICY_ENVS * (SRL_POLICY_MAX_OUT + 1) + POLICY_ENVS * MO);
}

}  // namespace

extern "C" {

int srl_policy_act(const srl_mlp_policy* p, int n, const float* obs, uint64_t* rng, uint64_t env_offset, float* obs_buf,
                   void* act_env, void* act_buf, float* logp, float* value, void* stream) {
    if (!p || !obs || !rng || !act_env || !logp || !value) { srl_set_error("policy_act: null argument"); return 1; }
    if (p->struct_size != sizeof(srl_mlp_policy)) { srl_set_error("policy_act: srl_mlp_policy size mismatch (%u != %zu)", p->struct_size, sizeof(srl_mlp_policy)); return 1; }
    if (n <= 0) { srl_set_error("policy_act: n must be positive"); return 1; }
    if (p->obs_dim < 1 || p->obs_dim > SRL_POLICY_WIDE_OBS || p->n_out < 1 || p->n_out > SRL_POLICY_MAX_OUT || (p->discrete && p->n_out < 2)) {
        srl_set_error("policy_act: unsupported shape obs_dim=%d n_out=%d (obs_dim 1..%d, n_out 1..%d)", p->obs_dim, p->n_out, SRL_POLICY_WIDE_OBS,
                      SRL_POLICY_MAX_OUT); return 1;
    }
    if (!p->pi_w1 || !p->pi_b1 || !p->pi_w2 || !p->pi_b2 || !p->pi_w3 || !p->pi_b3 || !p->vf_w1 || !p->vf_b1 || !p->vf_w2 || !p->vf_b2 ||
        !p->vf_w3 || !p->vf_b3 || (!p->discrete && !p->logstd)) { srl_set_error("policy_act: null weight pointer"); return 1; }
    PolicyArgs a;
    a.p = *p; a.n = n; a.obs = obs; a.rng = reinterpret_cast<unsigned long long*>(rng); a.env_offset = env_offset;
    a.obs_buf = obs_buf; a.act_env = act_env; a.act_buf = act_buf; a.logp = logp; a.value = value;
    const int grid = (n + POLICY_ENVS - 1) / POLICY_ENVS;
    if (p->obs_dim <= SRL_POLICY_MAX_OBS) {
        constexpr size_t smem = policy_smem_bytes<SRL_POLICY_MAX_OBS>();
        SRL_CUDA_OK(srl_smem_opt_in<policy_act_kernel<SRL_POLICY_MAX_OBS>>(smem));
        policy_act_kernel<SRL_POLICY_MAX_OBS><<<grid, POLICY_BLOCK, smem, (cudaStream_t)stream>>>(a);
    } else {
        constexpr size_t smem = policy_smem_bytes<SRL_POLICY_WIDE_OBS>();
        SRL_CUDA_OK(srl_smem_opt_in<policy_act_kernel<SRL_POLICY_WIDE_OBS>>(smem));
        policy_act_kernel<SRL_POLICY_WIDE_OBS><<<grid, POLICY_BLOCK, smem, (cudaStream_t)stream>>>(a);
    }
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_obs_filter(int n, int obs_dim, const float* obs_raw, double* state, int update, float clip, float eps, float* obs_norm_out,
                   void* stream) {
    if (!obs_raw || !state || !obs_norm_out) { srl_set_error("obs_filter: null argument"); return 1; }
    if (n <= 0 || obs_dim < 1 || obs_dim > SRL_POLICY_MAX_OBS) { srl_set_error("obs_filter: unsupported shape n=%d obs_dim=%d", n, obs_dim); return 1; }
    switch (obs_dim) {
#define SRL_FILTER_CASE(DD) case DD: obs_filter_kernel<DD><<<1, FILTER_BLOCK, 0, (cudaStream_t)stream>>>(n, obs_raw, state, update, clip, eps, obs_norm_out); break;
        SRL_FILTER_CASE(1) SRL_FILTER_CASE(2) SRL_FILTER_CASE(3) SRL_FILTER_CASE(4) SRL_FILTER_CASE(5) SRL_FILTER_CASE(6) SRL_FILTER_CASE(7) SRL_FILTER_CASE(8)
#undef SRL_FILTER_CASE
        default: srl_set_error("obs_filter: unsupported obs_dim %d", obs_dim); return 1;
    }
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_obs_stack_filter(int n, int obs_dim, int num_stack, const float* obs_raw, const uint8_t* done, float* stack, double* state, int update,
                         float clip, float eps, float* obs_norm_out, void* stream) {
    if (!obs_raw || !stack || !state || !obs_norm_out) { srl_set_error("obs_stack_filter: null argument"); return 1; }
    if (n <= 0 || obs_dim < 1 || num_stack < 1 || obs_dim > SRL_POLICY_WIDE_OBS || num_stack > SRL_POLICY_WIDE_OBS || obs_dim * num_stack > SRL_POLICY_WIDE_OBS) {
        srl_set_error("obs_stack_filter: unsupported shape n=%d obs_dim=%d num_stack=%d (obs_dim * num_stack must be 1..%d)", n, obs_dim, num_stack,
                      SRL_POLICY_WIDE_OBS);
        return 1;
    }
    obs_stack_filter_kernel<<<1, FILTER_BLOCK, 0, (cudaStream_t)stream>>>(n, obs_dim, num_stack, obs_raw, done, stack, state, update, clip, eps, obs_norm_out);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
