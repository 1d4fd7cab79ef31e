// Per-environment arithmetic of the fused PPO2 "policy act" step, shared by the sm_90a kernel (policy_kernels.cu) and by the
// CPU checker the tests build from it (oracle/policy_ref.cpp) -- plain C++, no CUDA types.  The checker takes any obs_dim: the
// tower below reads the observation width at run time, so it covers the narrow (<= 8) and the wide (<= 32) kernels alike.
//
// What it computes is what stable-baselines' PPO2 runner does per env step through `model.step(obs)` with `MlpPolicy`
// (rl_baselines/rl_algorithm/ppo2.py:58-72 of the reference picks that policy): two separate 64-64 tanh towers -- policy logits
// (Discrete) or mean (Box) and the value -- a sample from the resulting distribution, its log-probability and the value estimate.
// Weights use torch.nn.Linear's layout: weight [out][in] row-major, bias [out].
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define SRL_HD __host__ __device__ __forceinline__
#else
#define SRL_HD static inline
#endif

#define SRL_POLICY_HIDDEN 64
#define SRL_POLICY_MAX_OBS 8
#define SRL_POLICY_WIDE_OBS 32     // widest observation of the wide kernel instantiations (stacked states); widths above 8 take those
#define SRL_POLICY_MAX_OUT 8
enum { SRL_PHILOX_PURPOSE_POLICY = 16 };   // counter word 3 of the policy-sampling stream (the simulator uses 0..10, csrc/philox.cuh)

// Philox4x32-10 (Salmon et al., SC'11), same key / counter layout as csrc/philox.cuh: key = seed, counter = (env lo, env hi, index, purpose)
SRL_HD void srl_philox4x32_10_hd(uint64_t seed, uint64_t env, uint32_t index, uint32_t purpose, uint32_t out[4]) {
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    uint32_t c0 = (uint32_t)env, c1 = (uint32_t)(env >> 32), c2 = index, c3 = purpose;
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        c0 = n0; c1 = (uint32_t)p1; c2 = n2; c3 = (uint32_t)p0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

struct alignas(16) srl_f4 { float x, y, z, w; };   // one 16-byte load (LDS.128 in the kernel)

struct SrlTowerWeights {   // one 64-64 tower; pointers into shared memory (kernel) or host arrays (checker)
    const float *w1, *b1, *w2, *b2, *w3, *b3;
};

// One tower for one env.  `h` is this env's private column of SRL_POLICY_HIDDEN activations, element i at h[i * hstride] (a
// shared-memory column in the kernel: the output index of a layer is a run-time loop variable, the input index a compile-time
// one, so a layer is written to the column and read back into registers).  w2 / w3 rows must be 16-byte aligned.
SRL_HD void srl_mlp_tower(const SrlTowerWeights& W, int obs_dim, int n_out, const float* x, float* h, int hstride, float* out) {
    constexpr int H = SRL_POLICY_HIDDEN;
    for (int o = 0; o < H; ++o) {                       // layer 1: obs_dim -> 64
        float acc = W.b1[o];
        for (int d = 0; d < obs_dim; ++d) acc = fmaf(W.w1[o * obs_dim + d], x[d], acc);
        h[o * hstride] = tanhf(acc);
    }
    float a[H];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < H; ++i) a[i] = h[i * hstride];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int o = 0; o < H; ++o) {                       // layer 2: 64 -> 64, four partial sums (independent FMA chains)
        const srl_f4* row = reinterpret_cast<const srl_f4*>(W.w2 + o * H);
        float s0 = W.b2[o], s1 = 0.f, s2 = 0.f, s3 = 0.f;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int i4 = 0; i4 < H / 4; ++i4) {
            const srl_f4 w = row[i4];
            s0 = fmaf(w.x, a[4 * i4 + 0], s0); s1 = fmaf(w.y, a[4 * i4 + 1], s1);
            s2 = fmaf(w.z, a[4 * i4 + 2], s2); s3 = fmaf(w.w, a[4 * i4 + 3], s3);
        }
        h[o * hstride] = tanhf((s0 + s1) + (s2 + s3));
    }
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < H; ++i) a[i] = h[i * hstride];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int k = 0; k < n_out; ++k) {                   // layer 3: 64 -> n_out
        const srl_f4* row = reinterpret_cast<const srl_f4*>(W.w3 + k * H);
        float s0 = W.b3[k], s1 = 0.f, s2 = 0.f, s3 = 0.f;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int i4 = 0; i4 < H / 4; ++i4) {
            const srl_f4 w = row[i4];
            s0 = fmaf(w.x, a[4 * i4 + 0], s0); s1 = fmaf(w.y, a[4 * i4 + 1], s1);
            s2 = fmaf(w.z, a[4 * i4 + 2], s2); s3 = fmaf(w.w, a[4 * i4 + 3], s3);
        }
        out[k] = (s0 + s1) + (s2 + s3);
    }
}

// Categorical(logits).sample() by inverse CDF on one 53-bit uniform of the env's counter-based stream, and its log-probability.
SRL_HD int srl_sample_categorical(const float* logits, int n, uint64_t seed, uint64_t env, uint32_t index, float* logp) {
    float m = logits[0];
    for (int k = 1; k < n; ++k) m = fmaxf(m, logits[k]);
    float p[SRL_POLICY_MAX_OUT], S = 0.f;
    for (int k = 0; k < n; ++k) { p[k] = expf(logits[k] - m); S += p[k]; }
    uint32_t r[4];
    srl_philox4x32_10_hd(seed, env, index, SRL_PHILOX_PURPOSE_POLICY, r);
    const double u = ((double)(r[0] >> 5) * 67108864.0 + (double)(r[1] >> 6)) * (1.0 / 9007199254740992.0);
    const float target = (float)(u * (double)S);
    int a = n - 1;
    float cum = 0.f;
    for (int k = 0; k < n; ++k) {
        cum += p[k];
        if (target < cum) { a = k; break; }
    }
    *logp = (logits[a] - m) - logf(S);
    return a;
}

// Normal(mean, exp(logstd)).sample() (Box-Muller on the env's stream), the summed log-probability of the sample, and the
// action handed to the env: the sample clipped to the Box(-1, 1) bounds (stable-baselines' runner clips before env.step).
SRL_HD void srl_sample_gaussian(const float* mean, const float* logstd, int n, uint64_t seed, uint64_t env, uint32_t index,
                                float* sample, float* clipped, float* logp) {
    float lp = 0.f;
    uint32_t r[4] = {0u, 0u, 0u, 0u};
    for (int k = 0; k < n; ++k) {
        if ((k & 3) == 0) srl_philox4x32_10_hd(seed, env, index, SRL_PHILOX_PURPOSE_POLICY + 1 + (k >> 2), r);
        // words (0, 1) and (2, 3) are two Box-Muller pairs: k % 4 = 0, 1 take the cos / sin of the first, 2, 3 of the second
        const uint32_t wa = r[(k & 2)], wb = r[(k & 2) + 1];
        const float u1 = ((float)(wa >> 8) + 0.5f) * (1.0f / 16777216.0f);    // (0, 1): never 0, the log is finite
        const float u2 = ((float)(wb >> 8) + 0.5f) * (1.0f / 16777216.0f);
        const float rad = sqrtf(-2.0f * logf(u1)), ang = 6.28318530717958647692f * u2;
        const float z = (k & 1) ? rad * sinf(ang) : rad * cosf(ang);
        const float s = fmaf(expf(logstd[k]), z, mean[k]);
        sample[k] = s;
        clipped[k] = fminf(fmaxf(s, -1.0f), 1.0f);
        lp += -0.5f * z * z - logstd[k] - 0.91893853320467274178f;
    }
    *logp = lp;
}
