// TRPO's update on the device (include/srl_policy.h: srl_trpo_*) -- stable-baselines 2.5 `TRPO` with `MlpPolicy`, chosen by
// rl_baselines/rl_algorithm/trpo.py of the reference; rl_baselines/trpo.py is the trainer and the torch statement the tests compare against.
//
// One chunked kernel runs over ONE 64-64 tanh tower (the pi tower with its logstd, or the value tower) in four modes:
//   SURR  the gradient of optimgain = mean(ratio atarg) + ent_coef mean(entropy) at theta_old (ratio = 1), the losses before the step,
//         the standardised advantages and the old head outputs (logits / means) that the trials' KL and ratio start from;
//   FVP   the Fisher-vector product on a strided subsample: forward at theta_old, the tangent forward J v, the output-space metric of the
//         KL's Hessian at theta_old (Categorical diag(p) - p p^T, Gaussian 1 / sigma^2 on the mean) and the backward pass J^T (.);
//   TRIAL the losses at theta_old + s fullstep (s from the device status record), the trial weights formed while they are staged;
//   VGRAD the gradient of mean((v - ret)^2) over an index vector.
// A persistent CTA keeps the weights in shared memory and walks 64-sample chunks with every activation on chip; each thread owns a fixed
// set of gradient entries, so a CTA's partial is written once, and the partials are summed in float64 in CTA order by a second kernel
// (deterministic, no atomics).  A single-CTA vector kernel holds the conjugate-gradient state, the step size and the line-search decision
// on the device, so an update needs no host round trip.
#include <cuda_runtime.h>
#include <math.h>
#include "common.cuh"
#include "../../include/srl_policy.h"

namespace {

constexpr int H = 64, HS = H + 1, CH = 64, NT = 256, MAXO = 8, NARROW_D = 8, WIDE_D = 32;
enum Mode { SURR = 0, FVP = 1, TRIAL = 2, VGRAD = 3 };

// the flat parameter vector of one tower in the order pi_w1, pi_b1, pi_w2, pi_b2, pi_w3, pi_b3, logstd (Box; the value tower has none)
struct Seg { int w1, b1, w2, b2, w3, b3, ls, P; };
__host__ __device__ inline Seg make_seg(int D, int A, int with_ls) {
    Seg s; int o = 0;
    s.w1 = o; o += H * D; s.b1 = o; o += H; s.w2 = o; o += H * H; s.b2 = o; o += H; s.w3 = o; o += A * H; s.b3 = o; o += A;
    s.ls = o; o += with_ls ? A : 0; s.P = o;
    return s;
}

struct TowerArgs {
    int D, A, discrete, rows, group, gstride;     // sample s -> row (s / group) gstride + s % group, or idx[s]
    const float *w1, *b1, *w2, *b2, *w3, *b3, *ls;
    const long long* idx;
    const float* obs; const void* act; const float* adv; const float* ret;
    const float* v;           // FVP: the tangent vector (flat); TRIAL: fullstep (flat)
    const double* stats;      // SURR: STATS_CTAS x {sum(x - shift), sum((x - shift)^2)}, then the shift
    const double* state;      // TRIAL: the status record (scale, and whether the trial runs at all)
    float* atarg; float* old_out;
    float ent_coef;
    float* partial;           // [gridDim.x][P] per-CTA partial gradients
    double* lpart;            // [gridDim.x][4] per-CTA loss sums {surrogate, kl, entropy, 0}
};

constexpr int STATS_CTAS = 64, STATS_NT = 256;
__global__ void __launch_bounds__(STATS_NT) trpo_stats_kernel(int n, const float* __restrict__ x, double* __restrict__ part) {
    __shared__ double red[STATS_NT / 32][2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const double shift = (double)x[0];
    double s1 = 0.0, s2 = 0.0;
    for (int e = blockIdx.x * STATS_NT + tid; e < n; e += STATS_CTAS * STATS_NT) { const double c = (double)x[e] - shift; s1 += c; s2 = fma(c, c, s2); }
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if (lane == 0) { red[warp][0] = s1; red[warp][1] = s2; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < STATS_NT / 32; ++w) { s1 += red[w][0]; s2 += red[w][1]; }
        part[2 * blockIdx.x] = s1; part[2 * blockIdx.x + 1] = s2;
        if (blockIdx.x == 0) part[2 * STATS_CTAS] = shift;
    }
}

// out[e][k] (samples 4 ng + e, units jg + 16 k) = bias + sum_i W[i][unit] in[sample][i]: W stored input-major ([64][64], unit fastest)
__device__ __forceinline__ void tile64(const float* Wt, const float* in, int ng, int jg, float (&o)[4][4]) {
#pragma unroll 4
    for (int i = 0; i < H; ++i) {
        float w[4], a[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) w[k] = Wt[i * H + jg + 16 * k];
#pragma unroll
        for (int e = 0; e < 4; ++e) a[e] = in[(4 * ng + e) * HS + i];
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int k = 0; k < 4; ++k) o[e][k] = fmaf(w[k], a[e], o[e][k]);
    }
}

template <int MD>
__host__ __device__ constexpr size_t tower_smem_floats() {
    // w1t v1t | w2t w2n v2t | w3 v3 | b1 b2 vb1 vb2 | b3 vb3 ls | x | h1 h2 t1 t2 | d3 dls | sact | sc
    return (size_t)2 * MD * H + 3 * H * H + 2 * MAXO * H + 4 * H + 3 * MAXO + CH * MD + 4 * CH * HS + CH * (MAXO + 1) + CH * MAXO + CH * MAXO + 4 * CH;
}

template <int MD, int MODE>
__device__ __forceinline__ void tower_cta(const TowerArgs& a) {
    constexpr int NACC = (H * MD + H + H * H + H + MAXO * H + 2 * MAXO + NT - 1) / NT;     // owned entries of the largest flat vector
    extern __shared__ __align__(16) float sm[];
    const int D = a.D, A = a.A, t = threadIdx.x;
    const bool discrete = a.discrete != 0, box = !discrete && MODE != VGRAD;
    const Seg seg = make_seg(D, A, box);
    float* w1t = sm;              float* v1t = w1t + MD * H;
    float* w2t = v1t + MD * H;    float* w2n = w2t + H * H;     float* v2t = w2n + H * H;
    float* w3 = v2t + H * H;      float* v3 = w3 + MAXO * H;
    float* b1 = v3 + MAXO * H;    float* b2 = b1 + H;           float* vb1 = b2 + H;          float* vb2 = vb1 + H;
    float* b3 = vb2 + H;          float* vb3 = b3 + MAXO;       float* lss = vb3 + MAXO;
    float* xs = lss + MAXO;       // [CH][MD]
    float* h1 = xs + CH * MD;     float* h2 = h1 + CH * HS;     float* t1 = h2 + CH * HS;     float* t2 = t1 + CH * HS;   // t1 / t2: tangents, then d1 / d2
    float* d3 = t2 + CH * HS;     // [CH][MAXO + 1]
    float* dls = d3 + CH * (MAXO + 1);   // [CH][MAXO]
    float* sact = dls + CH * MAXO;       // [CH][MAXO] Box actions
    float* sc = sact + CH * MAXO;        // [CH][4] {atarg or ret, action (Discrete), valid, 0}

    __shared__ double red[NT / 32][4];
    __shared__ float s_norm[2];
    __shared__ int s_run;
    // ---- TRIAL: does this trial run, and at which scale? ----
    float scale = 0.f;
    if constexpr (MODE == TRIAL) {
        if (t == 0) s_run = a.state[SRL_TRPO_SKIP] == 0.0 && a.state[SRL_TRPO_NONFINITE] == 0.0 && a.state[SRL_TRPO_ACCEPTED] < 0.0 &&
                            a.state[SRL_TRPO_TRIALS] < (double)SRL_TRPO_MAX_TRIALS;
        __syncthreads();
        if (!s_run) return;
        scale = (float)a.state[SRL_TRPO_SCALE];
    }
    // ---- weights (TRIAL: theta_old + scale * fullstep, rounded as the update writes them) ----
    auto wt = [&](const float* base, int off, int e) -> float {
        if constexpr (MODE == TRIAL) return __fadd_rn(base[e], __fmul_rn(a.v[off + e], scale));
        else return base[e];
    };
    for (int e = t; e < H * D; e += NT) {
        const int j = e / D, d = e % D;
        w1t[d * H + j] = wt(a.w1, seg.w1, e);
        if constexpr (MODE == FVP) v1t[d * H + j] = a.v[seg.w1 + e];
    }
    for (int e = t; e < H * H; e += NT) {
        const int j = e >> 6, i = e & 63;
        const float w = wt(a.w2, seg.w2, e);
        w2t[i * H + j] = w; w2n[j * H + i] = w;
        if constexpr (MODE == FVP) v2t[i * H + j] = a.v[seg.w2 + e];
    }
    for (int e = t; e < A * H; e += NT) { w3[e] = wt(a.w3, seg.w3, e); if constexpr (MODE == FVP) v3[e] = a.v[seg.w3 + e]; }
    if (t < H) {
        b1[t] = wt(a.b1, seg.b1, t); b2[t] = wt(a.b2, seg.b2, t);
        if constexpr (MODE == FVP) { vb1[t] = a.v[seg.b1 + t]; vb2[t] = a.v[seg.b2 + t]; }
    }
    if (t < A) {
        b3[t] = wt(a.b3, seg.b3, t);
        if constexpr (MODE == FVP) vb3[t] = a.v[seg.b3 + t];
        lss[t] = box ? wt(a.ls, seg.ls, t) : 0.f;
    }
    if (MODE == SURR && t == 0) {     // mean and population std of the advantages (numpy's atarg.std(), no epsilon)
        double s1 = 0.0, s2 = 0.0;
        for (int c = 0; c < STATS_CTAS; ++c) { s1 += a.stats[2 * c]; s2 += a.stats[2 * c + 1]; }
        const double n = (double)a.rows, m1 = s1 / n;
        s_norm[0] = (float)(a.stats[2 * STATS_CTAS] + m1);
        s_norm[1] = (float)sqrt(fmax(s2 / n - m1 * m1, 0.0));
    }
    __syncthreads();
    const float amean = MODE == SURR ? s_norm[0] : 0.f, astd = MODE == SURR ? s_norm[1] : 1.f;
    const float inv_b = 1.0f / (float)a.rows;
    float acc[NACC];
#pragma unroll
    for (int m = 0; m < NACC; ++m) acc[m] = 0.f;
    double l_surr = 0.0, l_kl = 0.0, l_ent = 0.0;
    const int ng = t >> 4, jg = t & 15;
    const int nchunks = (a.rows + CH - 1) / CH;
    for (int c = blockIdx.x; c < nchunks; c += gridDim.x) {
        // ---- 0: the chunk's samples ----
        for (int e = t; e < CH * MD; e += NT) {
            const int n = e / MD, d = e % MD, s = c * CH + n;
            float x = 0.f;
            if (s < a.rows && d < D) {
                const long long g = a.idx ? a.idx[s] : (long long)(s / a.group) * a.gstride + s % a.group;
                x = a.obs[g * D + d];
            }
            xs[e] = x;
        }
        if (t < CH) {
            const int s = c * CH + t;
            const bool valid = s < a.rows;
            const long long g = !valid ? 0 : a.idx ? a.idx[s] : (long long)(s / a.group) * a.gstride + s % a.group;
            float sv = 0.f, ai = 0.f;
            if (valid && MODE != FVP) {
                if constexpr (MODE == VGRAD) sv = a.ret[g];
                else {
                    if (discrete) ai = (float)reinterpret_cast<const long long*>(a.act)[g];
                    else for (int k = 0; k < A; ++k) sact[t * MAXO + k] = reinterpret_cast<const float*>(a.act)[g * A + k];
                    if constexpr (MODE == SURR) { sv = __fdiv_rn(__fsub_rn(a.adv[g], amean), astd); a.atarg[g] = sv; }
                    else sv = a.atarg[g];
                }
            }
            sc[t * 4] = sv; sc[t * 4 + 1] = ai; sc[t * 4 + 2] = valid ? 1.f : 0.f;
            if (valid && MODE == TRIAL)      // the old head outputs into d3 (overwritten by the trial's derivative-free use below)
                for (int k = 0; k < A; ++k) d3[t * (MAXO + 1) + k] = a.old_out[g * A + k];
        }
        __syncthreads();
        // ---- 1: forward (FVP: and the tangent J v) ----
        {
            float o[4][4], q[4][4];
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) { o[e][k] = b1[jg + 16 * k]; q[e][k] = MODE == FVP ? vb1[jg + 16 * k] : 0.f; }
            for (int d = 0; d < D; ++d) {
                float w[4], v[4], x[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) { w[k] = w1t[d * H + jg + 16 * k]; if (MODE == FVP) v[k] = v1t[d * H + jg + 16 * k]; }
#pragma unroll
                for (int e = 0; e < 4; ++e) x[e] = xs[(4 * ng + e) * MD + d];
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int k = 0; k < 4; ++k) { o[e][k] = fmaf(w[k], x[e], o[e][k]); if (MODE == FVP) q[e][k] = fmaf(v[k], x[e], q[e][k]); }
            }
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const int at = (4 * ng + e) * HS + jg + 16 * k;
                    const float h = tanhf(o[e][k]);
                    h1[at] = h;
                    if (MODE == FVP) t1[at] = q[e][k] * (1.0f - h * h);
                }
        }
        __syncthreads();
        {
            float o[4][4];
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) o[e][k] = b2[jg + 16 * k];
            tile64(w2t, h1, ng, jg, o);
            if constexpr (MODE == FVP) {
                float q[4][4];
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int k = 0; k < 4; ++k) q[e][k] = vb2[jg + 16 * k];
                tile64(w2t, t1, ng, jg, q);       // W2 (J1 v)
                tile64(v2t, h1, ng, jg, q);       // + V2 h1
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int k = 0; k < 4; ++k) { const float h = tanhf(o[e][k]); t2[(4 * ng + e) * HS + jg + 16 * k] = q[e][k] * (1.0f - h * h); }
            }
            __syncthreads();                      // FVP: t1 is read above by other threads' tiles before h2 / t2 change
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int k = 0; k < 4; ++k) h2[(4 * ng + e) * HS + jg + 16 * k] = tanhf(o[e][k]);
        }
        __syncthreads();
        // ---- 2: the head, per sample (thread t < 64: sample t); d3 = d objective / d outputs, dls = d objective / d logstd ----
        if (t < CH) {
            const int n = t;
            const bool valid = sc[n * 4 + 2] != 0.f;
            float z[MAXO], dz[MAXO], g[MAXO], gl[MAXO], zo[MAXO];
#pragma unroll
            for (int k = 0; k < MAXO; ++k) {
                z[k] = 0.f; dz[k] = 0.f; g[k] = 0.f; gl[k] = 0.f; zo[k] = 0.f;
                if (k < A) {
                    float s0 = b3[k], s1 = MODE == FVP ? vb3[k] : 0.f;
                    for (int i = 0; i < H; ++i) {
                        s0 = fmaf(w3[k * H + i], h2[n * HS + i], s0);
                        if (MODE == FVP) s1 = fmaf(v3[k * H + i], h2[n * HS + i], fmaf(w3[k * H + i], t2[n * HS + i], s1));
                    }
                    z[k] = s0; dz[k] = s1;
                    if (MODE == TRIAL) zo[k] = d3[n * (MAXO + 1) + k];
                }
            }
            if (valid) {
                if constexpr (MODE == VGRAD) {
                    g[0] = 2.0f * (z[0] - sc[n * 4]) * inv_b;                              // d mean((v - ret)^2) / d v
                } else if (discrete) {
                    // stable-baselines' CategoricalProbabilityDistribution: max-shifted logits
                    const int ai = (int)sc[n * 4 + 1];
                    float m = z[0], mo = zo[0];
#pragma unroll
                    for (int k = 1; k < MAXO; ++k) if (k < A) { m = fmaxf(m, z[k]); mo = fmaxf(mo, zo[k]); }
                    float S = 0.f, So = 0.f, p[MAXO];
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) { p[k] = k < A ? expf(z[k] - m) : 0.f; S += p[k]; if (MODE == TRIAL && k < A) So += expf(zo[k] - mo); }
                    const float lS = logf(S);
                    float ent = 0.f;
#pragma unroll
                    for (int k = 0; k < MAXO; ++k) { p[k] = p[k] / S; if (k < A) ent += p[k] * (lS - (z[k] - m)); }
                    if constexpr (MODE == SURR) {
                        const float at = sc[n * 4];
#pragma unroll
                        for (int k = 0; k < MAXO; ++k) if (k < A) {
                            const float lp = (z[k] - m) - lS;                                   // log p_k
                            g[k] = (at * ((k == ai ? 1.f : 0.f) - p[k]) - a.ent_coef * p[k] * (lp + ent)) * inv_b;
                            zo[k] = z[k];
                        }
                        l_surr += (double)at; l_ent += (double)ent;
                    } else if constexpr (MODE == FVP) {
                        float pd = 0.f;
#pragma unroll
                        for (int k = 0; k < MAXO; ++k) if (k < A) pd = fmaf(p[k], dz[k], pd);
#pragma unroll
                        for (int k = 0; k < MAXO; ++k) if (k < A) g[k] = p[k] * (dz[k] - pd) * inv_b;   // (diag(p) - p p^T) J v
                    } else {   // TRIAL: ratio, KL(old || new), entropy of the new distribution
                        const float lSo = logf(So);
                        float kl = 0.f, lpn = 0.f, lpo = 0.f;
#pragma unroll
                        for (int k = 0; k < MAXO; ++k) if (k < A) {
                            const float po = expf(zo[k] - mo) / So, lo = (zo[k] - mo) - lSo, ln = (z[k] - m) - lS;
                            kl += po * (lo - ln);
                            if (k == ai) { lpn = ln; lpo = lo; }
                        }
                        l_surr += (double)(expf(lpn - lpo) * sc[n * 4]); l_kl += (double)kl; l_ent += (double)ent;
                    }
                } else {       // DiagGaussian: mean z, log std lss
                    if constexpr (MODE == SURR) {
                        const float at = sc[n * 4];
                        float ent = 0.f;
#pragma unroll
                        for (int k = 0; k < MAXO; ++k) if (k < A) {
                            const float is = expf(-lss[k]), u = (sact[n * MAXO + k] - z[k]) * is;
                            g[k] = at * u * is * inv_b;                                          // d logp / d mu = (a - mu) / sigma^2
                            gl[k] = (at * (u * u - 1.0f) + a.ent_coef) * inv_b;                // d logp / d logstd; d entropy / d logstd = 1
                            ent += lss[k] + 1.4189385332046727f;                               // 0.5 log(2 pi e)
                            zo[k] = z[k];
                        }
                        l_surr += (double)at; l_ent += (double)ent;
                    } else if constexpr (MODE == FVP) {
#pragma unroll
                        for (int k = 0; k < MAXO; ++k) if (k < A) { const float is = expf(-lss[k]); g[k] = dz[k] * is * is * inv_b; }
                    } else {
                        float kl = 0.f, ent = 0.f, dl = 0.f;
#pragma unroll
                        for (int k = 0; k < MAXO; ++k) if (k < A) {
                            const float lso = a.ls[k], sn = expf(lss[k]), so = expf(lso), dm = zo[k] - z[k];
                            kl += lss[k] - lso + (so * so + dm * dm) / (2.0f * sn * sn) - 0.5f;
                            ent += lss[k] + 1.4189385332046727f;
                            const float un = (sact[n * MAXO + k] - z[k]) / sn, uo = (sact[n * MAXO + k] - zo[k]) / so;
                            dl += (-0.5f * un * un - lss[k]) - (-0.5f * uo * uo - lso);           // logp_new - logp_old (the 2 pi terms cancel)
                        }
                        l_surr += (double)(expf(dl) * sc[n * 4]); l_kl += (double)kl; l_ent += (double)ent;
                    }
                }
            }
            if (MODE == SURR && valid) {
                const long long s = (long long)c * CH + n;
#pragma unroll
                for (int k = 0; k < MAXO; ++k) if (k < A) a.old_out[s * A + k] = zo[k];
            }
#pragma unroll
            for (int k = 0; k < MAXO; ++k) { d3[n * (MAXO + 1) + k] = g[k]; dls[n * MAXO + k] = gl[k]; }
        }
        __syncthreads();
        if constexpr (MODE != TRIAL) {
            // ---- 3: d2 = (W3^T d3)(1 - h2^2) ----
            for (int e = t; e < CH * H; e += NT) {
                const int n = e >> 6, j = e & 63;
                float s = 0.f;
                for (int k = 0; k < A; ++k) s = fmaf(w3[k * H + j], d3[n * (MAXO + 1) + k], s);
                const float h = h2[n * HS + j];
                t2[n * HS + j] = s * (1.0f - h * h);
            }
            __syncthreads();
            // ---- 4: d1 = (W2^T d2)(1 - h1^2) ----
            {
                float o[4][4];
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int k = 0; k < 4; ++k) o[e][k] = 0.f;
                tile64(w2n, t2, ng, jg, o);
#pragma unroll
                for (int e = 0; e < 4; ++e)
#pragma unroll
                    for (int k = 0; k < 4; ++k) { const int at = (4 * ng + e) * HS + jg + 16 * k; const float h = h1[at]; t1[at] = o[e][k] * (1.0f - h * h); }
            }
            __syncthreads();
            // ---- 5: the owned gradient entries e = t + NT m of the flat vector ----
#pragma unroll
            for (int m = 0; m < NACC; ++m) {
                const int e = t + NT * m;
                if (e >= seg.P) break;
                const float *pa, *pb; int sa, sb;
                if (e < seg.b1)      { const int j = e / D, d = e % D; pa = t1 + j; sa = HS; pb = xs + d; sb = MD; }
                else if (e < seg.w2) { pa = t1 + (e - seg.b1); sa = HS; pb = nullptr; sb = 0; }
                else if (e < seg.b2) { const int j = (e - seg.w2) >> 6, i = (e - seg.w2) & 63; pa = t2 + j; sa = HS; pb = h1 + i; sb = HS; }
                else if (e < seg.w3) { pa = t2 + (e - seg.b2); sa = HS; pb = nullptr; sb = 0; }
                else if (e < seg.b3) { const int k = (e - seg.w3) >> 6, i = (e - seg.w3) & 63; pa = d3 + k; sa = MAXO + 1; pb = h2 + i; sb = HS; }
                else if (e < seg.ls) { pa = d3 + (e - seg.b3); sa = MAXO + 1; pb = nullptr; sb = 0; }
                else                 { pa = dls + (e - seg.ls); sa = MAXO; pb = nullptr; sb = 0; }
                float s = 0.f;
                if (pb) {
#pragma unroll 8
                    for (int n = 0; n < CH; ++n) s = fmaf(pa[n * sa], pb[n * sb], s);
                } else {
#pragma unroll 8
                    for (int n = 0; n < CH; ++n) s += pa[n * sa];
                }
                acc[m] += s;
            }
        }
        __syncthreads();
    }
    if constexpr (MODE != TRIAL) {
        float* out = a.partial + (size_t)blockIdx.x * seg.P;
#pragma unroll
        for (int m = 0; m < NACC; ++m) { const int e = t + NT * m; if (e < seg.P) out[e] = acc[m]; }
    }
    if constexpr (MODE == SURR || MODE == TRIAL) {
        for (int o = 16; o > 0; o >>= 1) {
            l_surr += __shfl_xor_sync(0xffffffffu, l_surr, o); l_kl += __shfl_xor_sync(0xffffffffu, l_kl, o); l_ent += __shfl_xor_sync(0xffffffffu, l_ent, o);
        }
        if ((t & 31) == 0) { red[t >> 5][0] = l_surr; red[t >> 5][1] = l_kl; red[t >> 5][2] = l_ent; }
        __syncthreads();
        if (t == 0) {
            double s0 = 0.0, s1 = 0.0, s2 = 0.0;
            for (int w = 0; w < NT / 32; ++w) { s0 += red[w][0]; s1 += red[w][1]; s2 += red[w][2]; }
            double* lp = a.lpart + 4 * blockIdx.x;
            lp[0] = s0; lp[1] = s1; lp[2] = s2; lp[3] = 0.0;
        }
    }
}

#define TOWER_KERNEL(name, MD, MODE) \
    __global__ void __launch_bounds__(NT, 1) name(const __grid_constant__ TowerArgs a) { tower_cta<MD, MODE>(a); }
TOWER_KERNEL(trpo_surr_kernel, NARROW_D, SURR)
TOWER_KERNEL(trpo_surr_wide_kernel, WIDE_D, SURR)
TOWER_KERNEL(trpo_fvp_kernel, NARROW_D, FVP)
TOWER_KERNEL(trpo_fvp_wide_kernel, WIDE_D, FVP)
TOWER_KERNEL(trpo_trial_kernel, NARROW_D, TRIAL)
TOWER_KERNEL(trpo_trial_wide_kernel, WIDE_D, TRIAL)
TOWER_KERNEL(trpo_vgrad_kernel, NARROW_D, VGRAD)
TOWER_KERNEL(trpo_vgrad_wide_kernel, WIDE_D, VGRAD)

// the per-CTA partials summed in float64 in CTA order.  FVP: + 2 v on logstd (the Gaussian KL's Hessian there), then + damping v in float32.
// Losses: the CTA sums in CTA order, divided by the row count -> {surrgain, meankl, meanent} (float64).
struct ReduceArgs { int P, ls, nparts, rows, fvp; const float* partial; const double* lpart; const float* v; float damping; float* out; double* losses;
                    const double* state; };
__global__ void trpo_reduce_kernel(const __grid_constant__ ReduceArgs r) {
    if (r.state && !(r.state[SRL_TRPO_SKIP] == 0.0 && r.state[SRL_TRPO_NONFINITE] == 0.0 && r.state[SRL_TRPO_ACCEPTED] < 0.0 &&
                     r.state[SRL_TRPO_TRIALS] < (double)SRL_TRPO_MAX_TRIALS)) return;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (r.losses && e == 0) {
        double s[3] = {0.0, 0.0, 0.0};
        for (int c = 0; c < r.nparts; ++c) for (int k = 0; k < 3; ++k) s[k] += r.lpart[4 * c + k];
        for (int k = 0; k < 3; ++k) r.losses[k] = s[k] / (double)r.rows;
    }
    if (e >= r.P) return;
    double s = 0.0;
    for (int c = 0; c < r.nparts; ++c) s += (double)r.partial[(size_t)c * r.P + e];
    if (r.fvp) {
        if (e >= r.ls) s += 2.0 * (double)r.v[e];
        r.out[e] = __fadd_rn((float)s, __fmul_rn(r.damping, r.v[e]));
    } else {
        r.out[e] = (float)s;
    }
}

// ---- the vector kernel: one CTA over the flat vectors g, x, r, p, z, fullstep of the pi tower ----
constexpr int VEC_NT = 1024;
struct VecArgs {
    int op, P;
    float* vecs;              // [6][P]: g, x, r, p, z, fullstep
    double* state;
    const double* losses;     // {surrgain, meankl, meanent}
    float* params[7];         // pi_w1, pi_b1, pi_w2, pi_b2, pi_w3, pi_b3, logstd (Box): theta, written on acceptance
    int seg_off[8];
    float max_kl, ent_coef, residual_tol;
};

__device__ double block_sum(double s, double* red) {
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    double tot = 0.0;
    for (int w = 0; w < VEC_NT / 32; ++w) tot += red[w];
    return tot;
}

__global__ void __launch_bounds__(VEC_NT, 1) trpo_vector_kernel(const __grid_constant__ VecArgs o) {
    __shared__ double red[VEC_NT / 32];
    const int t = threadIdx.x, P = o.P;
    float *g = o.vecs, *x = g + P, *r = x + P, *p = r + P, *z = p + P, *fs = z + P;
    double* st = o.state;
    if (o.op == SRL_TRPO_OP_START) {
        int big = 0;
        double rr = 0.0;
        for (int e = t; e < P; e += VEC_NT) {
            const float ge = g[e];
            big |= !(fabsf(ge) <= 1e-8f);           // np.allclose(g, 0): |g| <= atol = 1e-8 everywhere
            x[e] = 0.f; r[e] = ge; p[e] = ge;
            rr = fma((double)ge, (double)ge, rr);
        }
        big = __syncthreads_or(big);
        rr = block_sum(rr, red);
        if (t == 0) {
            for (int k = 0; k < SRL_TRPO_STATE_DOUBLES; ++k) st[k] = 0.0;
            st[SRL_TRPO_SKIP] = big ? 0.0 : 1.0;
            st[SRL_TRPO_ACCEPTED] = -1.0;
            st[SRL_TRPO_SCALE] = 1.0;
            st[SRL_TRPO_RDOTR] = rr;
            st[SRL_TRPO_GAIN_BEFORE] = o.losses[0] + (double)o.ent_coef * o.losses[2];
            st[SRL_TRPO_SURR_BEFORE] = o.losses[0]; st[SRL_TRPO_ENT_BEFORE] = o.losses[2];
        }
        return;
    }
    if (st[SRL_TRPO_SKIP] != 0.0) return;
    if (o.op == SRL_TRPO_OP_CG) {                   // baselines' cg(): one iteration on z = F p
        if (st[SRL_TRPO_CG_DONE] != 0.0) return;
        double pz = 0.0;
        for (int e = t; e < P; e += VEC_NT) pz = fma((double)p[e], (double)z[e], pz);
        pz = block_sum(pz, red);
        const double rdotr = st[SRL_TRPO_RDOTR];
        const float v = (float)(rdotr / pz);
        double rr = 0.0;
        for (int e = t; e < P; e += VEC_NT) {
            x[e] = __fadd_rn(x[e], __fmul_rn(v, p[e]));
            const float re = __fsub_rn(r[e], __fmul_rn(v, z[e]));
            r[e] = re;
            rr = fma((double)re, (double)re, rr);
        }
        rr = block_sum(rr, red);
        const float mu = (float)(rr / rdotr);
        for (int e = t; e < P; e += VEC_NT) p[e] = __fadd_rn(r[e], __fmul_rn(mu, p[e]));
        if (t == 0) {
            st[SRL_TRPO_RDOTR] = rr;
            st[SRL_TRPO_CG_ITERS] += 1.0;
            if (rr < (double)o.residual_tol) st[SRL_TRPO_CG_DONE] = 1.0;
        }
        return;
    }
    if (o.op == SRL_TRPO_OP_STEP) {                 // z = F x: shs, lm, fullstep; a non-finite stepdir is flagged (the reference asserts)
        int bad = 0;
        double xz = 0.0;
        for (int e = t; e < P; e += VEC_NT) { bad |= !isfinite(x[e]); xz = fma((double)x[e], (double)z[e], xz); }
        bad = __syncthreads_or(bad);
        xz = block_sum(xz, red);
        const double shs = 0.5 * xz, lm = sqrt(fabs(shs) / (double)o.max_kl);
        const float lmf = (float)lm;
        if (!bad) for (int e = t; e < P; e += VEC_NT) fs[e] = __fdiv_rn(x[e], lmf);
        if (t == 0) { st[SRL_TRPO_SHS] = shs; st[SRL_TRPO_LM] = lm; st[SRL_TRPO_NONFINITE] = bad ? 1.0 : 0.0; }
        return;
    }
    // SRL_TRPO_OP_TRIAL: the decision on the losses of the trial at st[SCALE]
    if (st[SRL_TRPO_NONFINITE] != 0.0 || st[SRL_TRPO_ACCEPTED] >= 0.0 || st[SRL_TRPO_TRIALS] >= (double)SRL_TRPO_MAX_TRIALS) return;
    const double surr = o.losses[0], kl = o.losses[1], ent = o.losses[2];
    const double gain = surr + (double)o.ent_coef * ent;
    const int k = (int)st[SRL_TRPO_TRIALS];
    const bool finite = isfinite(gain) && isfinite(kl) && isfinite(surr) && isfinite(ent);
    const bool accept = finite && !(kl > 1.5 * (double)o.max_kl) && !(gain - st[SRL_TRPO_GAIN_BEFORE] < 0.0);
    const float scale = (float)st[SRL_TRPO_SCALE];
    if (accept) {
        for (int s = 0; s < 7; ++s) {
            float* w = o.params[s];
            if (!w) continue;
            for (int e = t; e < o.seg_off[s + 1] - o.seg_off[s]; e += VEC_NT) w[e] = __fadd_rn(w[e], __fmul_rn(fs[o.seg_off[s] + e], scale));
        }
    }
    __syncthreads();
    if (t == 0) {
        st[SRL_TRPO_TRIAL_LOSSES + 3 * k] = gain; st[SRL_TRPO_TRIAL_LOSSES + 3 * k + 1] = kl; st[SRL_TRPO_TRIAL_LOSSES + 3 * k + 2] = ent;
        st[SRL_TRPO_TRIALS] = k + 1;
        if (accept) st[SRL_TRPO_ACCEPTED] = k;
        else {
            st[SRL_TRPO_SCALE] = 0.5 * st[SRL_TRPO_SCALE];
            if (k + 1 == SRL_TRPO_MAX_TRIALS) st[SRL_TRPO_RESTORED] = 1.0;
        }
    }
}

// MpiAdam over the value tower, the statement of srl_ddpg_adam with one learning rate and no target
struct VAdamArgs { int P; float* w[6]; int off[7]; const float* g; float* m; float* v; long long* t; double lr, beta1, beta2; float eps; };
__global__ void __launch_bounds__(VEC_NT, 1) trpo_vf_adam_kernel(const __grid_constant__ VAdamArgs o) {
    const long long t = o.t[0] + 1;
    const double b1t = pow(o.beta1, (double)t), b2t = pow(o.beta2, (double)t);
    const float neg_a = (float)(-((o.lr * sqrt(1.0 - b2t)) / (1.0 - b1t)));
    const float b1 = (float)o.beta1, r1 = (float)(1.0 - o.beta1), b2 = (float)o.beta2, r2 = (float)(1.0 - o.beta2);
    for (int e = threadIdx.x; e < o.P; e += VEC_NT) {
        const float g = o.g[e];
        const float m = __fadd_rn(__fmul_rn(b1, o.m[e]), __fmul_rn(r1, g));
        const float v = __fadd_rn(__fmul_rn(b2, o.v[e]), __fmul_rn(r2, __fmul_rn(g, g)));
        o.m[e] = m; o.v[e] = v;
        int s = 0;
        while (e >= o.off[s + 1]) ++s;
        float* w = o.w[s] + (e - o.off[s]);
        *w = __fadd_rn(*w, __fdiv_rn(__fmul_rn(neg_a, m), __fadd_rn(__fsqrt_rn(v), o.eps)));
    }
    __syncthreads();
    if (threadIdx.x == 0) o.t[0] = t;
}

int sms_count() {
    static int sms[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
    if (!sms[dev] && cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return sms[dev];
}
int tower_ctas(int rows) {
    const int sms = sms_count(), chunks = (rows + CH - 1) / CH;
    return sms <= 0 ? 0 : (chunks < sms ? chunks : sms);
}

bool shape_ok(const char* who, const srl_mlp_policy* p, int rows) {
    if (!p || p->struct_size != sizeof(srl_mlp_policy)) { srl_set_error("%s: null policy or struct size mismatch", who); return false; }
    if (p->obs_dim < 1 || p->obs_dim > WIDE_D || p->n_out < 1 || p->n_out > MAXO || (p->discrete && p->n_out < 2) || rows < 1) {
        srl_set_error("%s: unsupported shape obs_dim=%d n_out=%d rows=%d (obs_dim 1..%d, n_out 1..%d)", who, p->obs_dim, p->n_out, rows, WIDE_D, MAXO);
        return false;
    }
    return true;
}

// workspace: [STATS] doubles, then per-CTA loss sums [ctas][4] doubles, then per-CTA partial gradients [ctas][P] floats
constexpr size_t STATS_BYTES = 2048;
size_t ws_bytes(int D, int A, int rows) {
    const int ctas = tower_ctas(rows);
    const int P = make_seg(D, A, 1).P;
    return STATS_BYTES + (size_t)(ctas > 0 ? ctas : 1) * (32 + sizeof(float) * (size_t)P);
}

template <void (*NARROW)(TowerArgs), void (*WIDEK)(TowerArgs)>
int launch_tower(const TowerArgs& a, int ctas, cudaStream_t st) {
    if (a.D <= NARROW_D) {
        constexpr size_t smem = sizeof(float) * tower_smem_floats<NARROW_D>();
        SRL_CUDA_OK(srl_smem_opt_in<NARROW>(smem));
        NARROW<<<ctas, NT, smem, st>>>(a);
    } else {
        constexpr size_t smem = sizeof(float) * tower_smem_floats<WIDE_D>();
        SRL_CUDA_OK(srl_smem_opt_in<WIDEK>(smem));
        WIDEK<<<ctas, NT, smem, st>>>(a);
    }
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}
static_assert(sizeof(float) * tower_smem_floats<WIDE_D>() <= 227 * 1024, "shared memory of one CTA");

int prepare(const char* who, const srl_mlp_policy* p, int rows, bool value_tower, void* ws, size_t wsb, TowerArgs& a, int& ctas) {
    if (!shape_ok(who, p, rows)) return 1;
    if (!ws) { srl_set_error("%s: null workspace", who); return 1; }
    ctas = tower_ctas(rows);
    if (ctas <= 0) { srl_set_error("%s: no CUDA device", who); return 1; }
    if (wsb < ws_bytes(p->obs_dim, p->n_out, rows)) { srl_set_error("%s: workspace too small (srl_trpo_workspace_bytes)", who); return 1; }
    a = TowerArgs{};
    a.D = p->obs_dim; a.A = value_tower ? 1 : p->n_out; a.discrete = value_tower ? 0 : p->discrete; a.rows = rows; a.group = rows; a.gstride = rows;
    if (value_tower) { a.w1 = p->vf_w1; a.b1 = p->vf_b1; a.w2 = p->vf_w2; a.b2 = p->vf_b2; a.w3 = p->vf_w3; a.b3 = p->vf_b3; a.ls = nullptr; }
    else { a.w1 = p->pi_w1; a.b1 = p->pi_b1; a.w2 = p->pi_w2; a.b2 = p->pi_b2; a.w3 = p->pi_w3; a.b3 = p->pi_b3; a.ls = p->logstd; }
    if (!a.w1 || !a.b1 || !a.w2 || !a.b2 || !a.w3 || !a.b3 || (!value_tower && !p->discrete && !a.ls)) { srl_set_error("%s: null weight pointer", who); return 1; }
    a.stats = reinterpret_cast<double*>(ws);
    a.lpart = reinterpret_cast<double*>(reinterpret_cast<char*>(ws) + STATS_BYTES);
    a.partial = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + STATS_BYTES + 32 * (size_t)ctas);
    return 0;
}

int reduce(const TowerArgs& a, int ctas, int fvp, float damping, float* out, double* losses, const double* state, cudaStream_t st) {
    const Seg seg = make_seg(a.D, a.A, !a.discrete && a.ls != nullptr);
    ReduceArgs r;
    r.P = out ? seg.P : 0; r.ls = seg.ls; r.nparts = ctas; r.rows = a.rows; r.fvp = fvp; r.partial = a.partial; r.lpart = a.lpart; r.v = a.v;
    r.damping = damping; r.out = out; r.losses = losses; r.state = state;
    trpo_reduce_kernel<<<r.P > 0 ? (r.P + 255) / 256 : 1, 256, 0, st>>>(r);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace

extern "C" {

size_t srl_trpo_flat_floats(int obs_dim, int n_out, int discrete) {
    if (obs_dim < 1 || obs_dim > WIDE_D || n_out < 1 || n_out > MAXO) return 0;
    return (size_t)make_seg(obs_dim, n_out, !discrete).P;
}

size_t srl_trpo_workspace_bytes(int obs_dim, int n_out, int rows) {
    if (obs_dim < 1 || obs_dim > WIDE_D || n_out < 1 || n_out > MAXO || rows < 1) {
        srl_set_error("trpo_workspace_bytes: unsupported shape obs_dim=%d n_out=%d rows=%d", obs_dim, n_out, rows);
        return 0;
    }
    if (tower_ctas(rows) <= 0) { srl_set_error("trpo_workspace_bytes: no CUDA device"); return 0; }
    return ws_bytes(obs_dim, n_out, rows);
}

int srl_trpo_surrogate(const srl_mlp_policy* p, int rows, const float* obs, const void* actions, const float* adv, float ent_coef, float* atarg,
                       float* old_out, float* grad, double* losses, void* workspace, size_t workspace_bytes, void* stream) {
    TowerArgs a; int ctas;
    if (prepare("trpo_surrogate", p, rows, false, workspace, workspace_bytes, a, ctas)) return 1;
    if (!obs || !actions || !adv || !atarg || !old_out || !grad || !losses) { srl_set_error("trpo_surrogate: null argument"); return 1; }
    cudaStream_t st = (cudaStream_t)stream;
    trpo_stats_kernel<<<STATS_CTAS, STATS_NT, 0, st>>>(rows, adv, const_cast<double*>(a.stats));
    SRL_CUDA_OK(cudaGetLastError());
    a.obs = obs; a.act = actions; a.adv = adv; a.atarg = atarg; a.old_out = old_out; a.ent_coef = ent_coef;
    if (launch_tower<trpo_surr_kernel, trpo_surr_wide_kernel>(a, ctas, st)) return 1;
    return reduce(a, ctas, 0, 0.f, grad, losses, nullptr, st);
}

int srl_trpo_fvp(const srl_mlp_policy* p, int rows, int group, int group_stride, const float* obs, const float* v, float damping, float* out,
                 void* workspace, size_t workspace_bytes, void* stream) {
    TowerArgs a; int ctas;
    if (prepare("trpo_fvp", p, rows, false, workspace, workspace_bytes, a, ctas)) return 1;
    if (!obs || !v || !out) { srl_set_error("trpo_fvp: null argument"); return 1; }
    if (group < 1 || group_stride < group) { srl_set_error("trpo_fvp: need group >= 1 and group_stride >= group (got %d, %d)", group, group_stride); return 1; }
    a.group = group; a.gstride = group_stride; a.obs = obs; a.v = v;
    cudaStream_t st = (cudaStream_t)stream;
    if (launch_tower<trpo_fvp_kernel, trpo_fvp_wide_kernel>(a, ctas, st)) return 1;
    return reduce(a, ctas, 1, damping, out, nullptr, nullptr, st);
}

int srl_trpo_trial(const srl_mlp_policy* p, int rows, const float* obs, const void* actions, const float* atarg, const float* old_out,
                   const float* fullstep, const double* state, double* losses, void* workspace, size_t workspace_bytes, void* stream) {
    TowerArgs a; int ctas;
    if (prepare("trpo_trial", p, rows, false, workspace, workspace_bytes, a, ctas)) return 1;
    if (!obs || !actions || !atarg || !old_out || !fullstep || !state || !losses) { srl_set_error("trpo_trial: null argument"); return 1; }
    a.obs = obs; a.act = actions; a.atarg = const_cast<float*>(atarg); a.old_out = const_cast<float*>(old_out); a.v = fullstep; a.state = state;
    cudaStream_t st = (cudaStream_t)stream;
    if (launch_tower<trpo_trial_kernel, trpo_trial_wide_kernel>(a, ctas, st)) return 1;
    return reduce(a, ctas, 0, 0.f, nullptr, losses, state, st);
}

int srl_trpo_vf_grad(const srl_mlp_policy* p, int rows, const int64_t* idx, const float* obs, const float* ret, float* grad, void* workspace,
                     size_t workspace_bytes, void* stream) {
    TowerArgs a; int ctas;
    if (prepare("trpo_vf_grad", p, rows, true, workspace, workspace_bytes, a, ctas)) return 1;
    if (!obs || !ret || !grad) { srl_set_error("trpo_vf_grad: null argument"); return 1; }
    a.idx = reinterpret_cast<const long long*>(idx); a.obs = obs; a.ret = ret;
    cudaStream_t st = (cudaStream_t)stream;
    if (launch_tower<trpo_vgrad_kernel, trpo_vgrad_wide_kernel>(a, ctas, st)) return 1;
    return reduce(a, ctas, 0, 0.f, grad, nullptr, nullptr, st);
}

int srl_trpo_vector(int op, int obs_dim, int n_out, int discrete, const srl_mlp_grads* params, float* vecs, double* state, const double* losses,
                    float max_kl, float ent_coef, float residual_tol, void* stream) {
    if (op < SRL_TRPO_OP_START || op > SRL_TRPO_OP_TRIAL) { srl_set_error("trpo_vector: unknown op %d", op); return 1; }
    if (obs_dim < 1 || obs_dim > WIDE_D || n_out < 1 || n_out > MAXO || (discrete && n_out < 2)) {
        srl_set_error("trpo_vector: unsupported shape obs_dim=%d n_out=%d", obs_dim, n_out); return 1;
    }
    if (!vecs || !state || ((op == SRL_TRPO_OP_START || op == SRL_TRPO_OP_TRIAL) && !losses)) { srl_set_error("trpo_vector: null argument"); return 1; }
    if (!(max_kl > 0.f)) { srl_set_error("trpo_vector: max_kl must be positive (got %g)", max_kl); return 1; }
    VecArgs o = {};
    const Seg seg = make_seg(obs_dim, n_out, !discrete);
    o.op = op; o.P = seg.P; o.vecs = vecs; o.state = state; o.losses = losses; o.max_kl = max_kl; o.ent_coef = ent_coef;
    o.residual_tol = residual_tol;
    const int off[8] = {seg.w1, seg.b1, seg.w2, seg.b2, seg.w3, seg.b3, seg.ls, seg.P};
    for (int s = 0; s < 8; ++s) o.seg_off[s] = off[s];
    if (op == SRL_TRPO_OP_TRIAL) {
        if (!params || params->struct_size != sizeof(srl_mlp_grads)) { srl_set_error("trpo_vector: null params or struct size mismatch"); return 1; }
        float* w[7] = {params->pi_w1, params->pi_b1, params->pi_w2, params->pi_b2, params->pi_w3, params->pi_b3, discrete ? nullptr : params->logstd};
        for (int s = 0; s < 7; ++s) {
            if (!w[s] && !(s == 6 && discrete)) { srl_set_error("trpo_vector: null parameter pointer"); return 1; }
            o.params[s] = w[s];
        }
    }
    trpo_vector_kernel<<<1, VEC_NT, 0, (cudaStream_t)stream>>>(o);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_trpo_vf_adam(int obs_dim, const srl_mlp_grads* params, const float* grad, float* m, float* v, int64_t* step, double lr, double beta1, double beta2,
                     double epsilon, void* stream) {
    if (!params || !grad || !m || !v || !step) { srl_set_error("trpo_vf_adam: null argument"); return 1; }
    if (params->struct_size != sizeof(srl_mlp_grads)) { srl_set_error("trpo_vf_adam: struct size mismatch"); return 1; }
    if (obs_dim < 1 || obs_dim > WIDE_D) { srl_set_error("trpo_vf_adam: unsupported obs_dim=%d", obs_dim); return 1; }
    if (!(beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0 && epsilon >= 0.0)) {
        srl_set_error("trpo_vf_adam: need 0 <= beta1, beta2 < 1, epsilon >= 0 (got %g, %g, %g)", beta1, beta2, epsilon); return 1;
    }
    VAdamArgs o;
    float* w[6] = {params->vf_w1, params->vf_b1, params->vf_w2, params->vf_b2, params->vf_w3, params->vf_b3};
    const Seg seg = make_seg(obs_dim, 1, 0);
    const int off[7] = {seg.w1, seg.b1, seg.w2, seg.b2, seg.w3, seg.b3, seg.P};
    for (int s = 0; s < 6; ++s) { if (!w[s]) { srl_set_error("trpo_vf_adam: null parameter pointer"); return 1; } o.w[s] = w[s]; }
    for (int s = 0; s < 7; ++s) o.off[s] = off[s];
    o.P = seg.P; o.g = grad; o.m = m; o.v = v; o.t = reinterpret_cast<long long*>(step); o.lr = lr; o.beta1 = beta1; o.beta2 = beta2; o.eps = (float)epsilon;
    trpo_vf_adam_kernel<<<1, VEC_NT, 0, (cudaStream_t)stream>>>(o);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"
