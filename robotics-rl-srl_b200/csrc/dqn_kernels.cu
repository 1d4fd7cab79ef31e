// DQN consumer kernels (include/srl_policy.h): the epsilon-greedy step of the dueling Q network, the double-Q target, and baselines'
// prioritized replay (a float64 sum tree and min tree over the transitions of the replay ring).  The gradient of the DQN loss is a mode of
// the PPO2 gradient kernel (ppo2_kernels.cu: srl_dqn_grad) and the optimiser step sits next to RMSProp there (srl_clip_adam).
//
// The Q network is an srl_mlp_policy with discrete = 1: the pi tower is the advantage head A (n_out values), the vf tower the state value V,
// both W -> 64 -> 64 with ReLU; Q = V + (A - mean(A)), with mean(A) = (A_0 + ... + A_{n-1}) / n summed in order, the same statement in every
// kernel that forms Q (act, target, gradient).
#include <cuda_runtime.h>
#include <math.h>
#include "common.cuh"
#include "policy_tile.cuh"
#include "../../include/srl_policy.h"

namespace {

constexpr int MAXO = SRL_POLICY_MAX_OUT;
// counter word 3 of the Philox streams (the simulator uses 0..10, the policy step 16..18: csrc/policy_core.h)
enum { SRL_PHILOX_PURPOSE_DQN_ACT = 24, SRL_PHILOX_PURPOSE_REPLAY = 25 };

__device__ __forceinline__ double philox_u53(unsigned long long seed, unsigned long long stream, uint32_t counter, uint32_t purpose, uint32_t (&r)[4]) {
    srl_philox4x32_10_hd(seed, stream, counter, purpose, r);
    return ((double)(r[0] >> 5) * 67108864.0 + (double)(r[1] >> 6)) * (1.0 / 9007199254740992.0);    // [0, 1), 53 bits
}

// the LAST CTA to retire advances the counter of a {seed, counter, arrivals} record: every CTA has read it by then (srl_policy_act's rule)
__device__ __forceinline__ void advance_counter(unsigned long long* rng, unsigned long long counter) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long arrived = atomicAdd(rng + 2, 1ull);
        if (arrived == (unsigned long long)gridDim.x - 1ull) {
            rng[2] = 0ull;
            rng[1] = counter + 1ull;
            __threadfence();
        }
    }
}

// ---- the dueling Q forward: one network staged in shared memory in the layout tower_tiled reads (policy_tile.cuh) ----
template <int MO>
__host__ __device__ constexpr int net_floats() { return 2 * H * WS + MAXO * WS + WS + 2 * H * w1_stride<MO>() + 4 * H + MAXO + 4; }
static_assert(net_floats<SRL_POLICY_MAX_OBS>() % 4 == 0 && net_floats<SRL_POLICY_WIDE_OBS>() % 4 == 0, "16-byte aligned regions");
// after the networks: ha, hb [POLICY_ENVS][WS], outs [POLICY_ENVS][MAXO + 1], xs [POLICY_ENVS][MO]
template <int MO>
constexpr size_t q_smem_bytes(int nets) {
    return sizeof(float) * ((size_t)nets * net_floats<MO>() + 2 * POLICY_ENVS * WS + POLICY_ENVS * (MAXO + 1) + POLICY_ENVS * MO);
}

template <int MO>
__device__ void stage_net(const srl_mlp_policy& p, float* s, TowerSmem& pi, TowerSmem& vf) {
    constexpr int W1S = w1_stride<MO>();
    const int D = p.obs_dim, A = p.n_out, t = threadIdx.x;
    float* w2p = s;               float* w2v = w2p + H * WS;       float* w3p = w2v + H * WS;      float* w3v = w3p + MAXO * WS;
    float* w1p = w3v + WS;        float* w1v = w1p + H * W1S;
    float* b1p = w1v + H * W1S;   float* b1v = b1p + H;            float* b2p = b1v + H;           float* b2v = b2p + H;
    float* b3p = b2v + H;         float* b3v = b3p + MAXO;
    for (int e = t; e < H * H; e += POLICY_BLOCK) { w2p[(e >> 6) * WS + (e & 63)] = p.pi_w2[e]; w2v[(e >> 6) * WS + (e & 63)] = p.vf_w2[e]; }
    for (int e = t; e < A * H; e += POLICY_BLOCK) w3p[(e >> 6) * WS + (e & 63)] = p.pi_w3[e];
    for (int e = t; e < H; e += POLICY_BLOCK) {
        w3v[e] = p.vf_w3[e];
        b1p[e] = p.pi_b1[e]; b1v[e] = p.vf_b1[e]; b2p[e] = p.pi_b2[e]; b2v[e] = p.vf_b2[e];
    }
    if constexpr (MO == SRL_POLICY_MAX_OBS) {          // the narrow tile reads W1 as [64][D]
        for (int e = t; e < H * D; e += POLICY_BLOCK) { w1p[e] = p.pi_w1[e]; w1v[e] = p.vf_w1[e]; }
    } else {                                           // the wide tile: rows of W1S words, zero past D
        for (int e = t; e < H * W1S; e += POLICY_BLOCK) {
            const int o = e / W1S, d = e % W1S;
            w1p[e] = d < D ? p.pi_w1[o * D + d] : 0.f; w1v[e] = d < D ? p.vf_w1[o * D + d] : 0.f;
        }
    }
    if (t < A) b3p[t] = p.pi_b3[t];
    if (t == 0) b3v[0] = p.vf_b3[0];
    pi = {w1p, b1p, w2p, b2p, w3p, b3p};
    vf = {w1v, b1v, w2v, b2v, w3v, b3v};
}

// rows first .. first + 31 of x (row r read from x[idx ? idx[r] : r]) -> xs [POLICY_ENVS][MO], zero past D and past `rows`; optionally copied
// to copy_out[r] (the replay ring's observation row)
template <int MO>
__device__ __forceinline__ void load_rows(const float* x, const long long* idx, int D, int rows, int first, float* xs, float* copy_out) {
    for (int j = threadIdx.x; j < POLICY_ENVS * MO; j += POLICY_BLOCK) {
        const int r = first + j / MO, d = j % MO;
        float v = 0.f;
        if (r < rows && d < D) {
            v = x[(idx ? idx[r] : (long long)r) * D + d];
            if (copy_out) copy_out[(size_t)r * D + d] = v;
        }
        xs[j] = v;
    }
}

// Q of one row from the towers' outputs (A at out[0 .. n), V at out[MAXO]) and its greedy action (ties: the lowest index, as tf.argmax)
__device__ __forceinline__ int dueling_q(const float* out, int A, float (&q)[MAXO]) {
    float sa = 0.f;
    for (int k = 0; k < A; ++k) sa += out[k];
    const float mean = sa * (1.0f / (float)A), v = out[MAXO];
    int best = 0;
    for (int k = 0; k < A; ++k) {
        q[k] = v + (out[k] - mean);
        if (q[k] > q[best]) best = k;
    }
    return best;
}

struct ActArgs {
    srl_mlp_policy q;
    int n;
    const float* obs; const float* eps;
    unsigned long long* rng; unsigned long long env_offset;
    float* obs_buf; int* act_env; long long* act_buf; float* q_out;
};

template <int MO>
__global__ void __launch_bounds__(POLICY_BLOCK) dqn_act_kernel(const __grid_constant__ ActArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int D = a.q.obs_dim, A = a.q.n_out, first = blockIdx.x * POLICY_ENVS;
    TowerSmem pi, vf;
    stage_net<MO>(a.q, smem, pi, vf);
    float* ha = smem + net_floats<MO>();  float* hb = ha + POLICY_ENVS * WS;  float* outs = hb + POLICY_ENVS * WS;  float* xs = outs + POLICY_ENVS * (MAXO + 1);
    load_rows<MO>(a.obs, nullptr, D, a.n, first, xs, a.obs_buf);
    const unsigned long long seed = a.rng[0], counter = a.rng[1];
    const double eps = (double)*a.eps;
    __syncthreads();
    tower_tiled<MO, true>(pi, D, A, xs, ha, hb, outs, MAXO + 1);
    tower_tiled<MO, true>(vf, D, 1, xs, ha, hb, outs + MAXO, MAXO + 1);
    __syncwarp();                                            // an env's outputs were written by the 4 lanes t / 4 = env of this warp
    const int slot = threadIdx.x >> 2, u = threadIdx.x & 3, i = first + slot;
    if (i < a.n && u == 0) {
        float q[MAXO];
        const int best = dueling_q(outs + slot * (MAXO + 1), A, q);
        uint32_t r[4];
        // epsilon-greedy: words 0-1 decide (a 53-bit uniform below eps explores), word 2 picks the uniform action
        const bool explore = philox_u53(seed, a.env_offset + (unsigned long long)i, (uint32_t)counter, SRL_PHILOX_PURPOSE_DQN_ACT, r) < eps;
        const int act = explore ? (int)(((unsigned long long)r[2] * (unsigned long long)A) >> 32) : best;
        a.act_env[i] = act;
        if (a.act_buf) a.act_buf[i] = (long long)act;
        if (a.q_out) for (int k = 0; k < A; ++k) a.q_out[(size_t)i * A + k] = q[k];
    }
    advance_counter(a.rng, counter);
}

struct TargetArgs {
    srl_mlp_policy online, target;
    int B;
    const long long* idx; const float* next_obs; const float* rew; const uint8_t* done;
    float gamma;
    float* y;
};

// persistent CTAs over chunks of 32 sampled rows, both networks staged once per CTA
template <int MO>
__global__ void __launch_bounds__(POLICY_BLOCK) dqn_target_kernel(const __grid_constant__ TargetArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int D = a.online.obs_dim, A = a.online.n_out;
    TowerSmem opi, ovf, tpi, tvf;
    stage_net<MO>(a.online, smem, opi, ovf);
    stage_net<MO>(a.target, smem + net_floats<MO>(), tpi, tvf);
    float* ha = smem + 2 * net_floats<MO>();  float* hb = ha + POLICY_ENVS * WS;  float* outs = hb + POLICY_ENVS * WS;  float* xs = outs + POLICY_ENVS * (MAXO + 1);
    const int slot = threadIdx.x >> 2, u = threadIdx.x & 3, nchunks = (a.B + POLICY_ENVS - 1) / POLICY_ENVS;
    for (int c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const int b = c * POLICY_ENVS + slot;
        __syncthreads();                                     // the previous chunk's reads of xs and outs are done
        load_rows<MO>(a.next_obs, a.idx, D, a.B, c * POLICY_ENVS, xs, nullptr);
        __syncthreads();
        tower_tiled<MO, true>(opi, D, A, xs, ha, hb, outs, MAXO + 1);
        tower_tiled<MO, true>(ovf, D, 1, xs, ha, hb, outs + MAXO, MAXO + 1);
        __syncwarp();
        float q[MAXO];
        const int best = (b < a.B && u == 0) ? dueling_q(outs + slot * (MAXO + 1), A, q) : 0;    // argmax_b Q_online(s', b)
        tower_tiled<MO, true>(tpi, D, A, xs, ha, hb, outs, MAXO + 1);     // its layer 3 writes `outs` after two barriers the lead lanes passed
        tower_tiled<MO, true>(tvf, D, 1, xs, ha, hb, outs + MAXO, MAXO + 1);
        __syncwarp();
        if (b < a.B && u == 0) {
            dueling_q(outs + slot * (MAXO + 1), A, q);
            const long long g = a.idx ? a.idx[b] : (long long)b;
            const float notdone = a.done[g] ? 0.f : 1.f;
            a.y[b] = __fadd_rn(a.rew[g], __fmul_rn(a.gamma, __fmul_rn(notdone, q[best])));      // r + gamma ((1 - d) Q_target(s', best))
        }
    }
}

// ---- prioritized replay: baselines' SegmentTree, node 1 the root, node k's children 2k and 2k + 1, leaf i at cap + i ----
constexpr int TREE_S = 2048, TREE_NT = 1024;     // nodes of one level a CTA rebuilds a subtree from (two per thread at the bottom)
struct TreeArgs {
    double* sum; double* mn;
    long long cap;                 // this pass's bottom level: nodes [cap, 2 cap); CTA b takes nodes cap + (first + b) s .. + s - 1, s = min(cap, TREE_S)
    long long first;
    long long set_lo, set_hi;      // first pass of srl_replay_add: leaves [set_lo, set_hi) become max_priority^alpha in both trees
    const double* max_p; double alpha;
    long long* size; long long new_size;
};

// every node above the CTA's bottom nodes, up to the root of its subtree (the tree's root when cap <= TREE_S), = op(left, right)
__global__ void __launch_bounds__(TREE_NT) tree_rebuild_kernel(const __grid_constant__ TreeArgs a) {
    __shared__ double ss[TREE_S], sm[TREE_S];
    const int t = threadIdx.x;
    const long long s = a.cap < TREE_S ? a.cap : TREE_S, base = a.cap + (a.first + blockIdx.x) * s;
    const double leaf = a.set_hi > a.set_lo ? pow(*a.max_p, a.alpha) : 0.0;
    for (int j = t; j < s; j += TREE_NT) {
        const long long node = base + j, li = node - a.cap;
        if (li >= a.set_lo && li < a.set_hi) { a.sum[node] = leaf; a.mn[node] = leaf; ss[j] = leaf; sm[j] = leaf; }
        else { ss[j] = a.sum[node]; sm[j] = a.mn[node]; }
    }
    if (a.size && blockIdx.x == 0 && t == 0 && *a.size < a.new_size) *a.size = a.new_size;
    __syncthreads();
    long long nb = base;
    for (int w = (int)(s >> 1); w >= 1; w >>= 1) {
        nb >>= 1;
        double vs = 0.0, vm = 0.0;
        if (t < w) { vs = ss[2 * t] + ss[2 * t + 1]; vm = fmin(sm[2 * t], sm[2 * t + 1]); }
        __syncthreads();
        if (t < w) { ss[t] = vs; sm[t] = vm; a.sum[nb + t] = vs; a.mn[nb + t] = vm; }
        __syncthreads();
    }
}

// the passes that make every ancestor of the bottom leaves [lo, hi) consistent: subtrees of TREE_S nodes, then the level of their roots, ...
int rebuild(TreeArgs a, long long lo, long long hi, cudaStream_t st) {
    for (;;) {
        const long long s = a.cap < TREE_S ? a.cap : TREE_S, b0 = lo / s, b1 = (hi - 1) / s;
        a.first = b0;
        tree_rebuild_kernel<<<(unsigned)(b1 - b0 + 1), TREE_NT, 0, st>>>(a);
        SRL_CUDA_OK(cudaGetLastError());
        if (a.cap <= TREE_S) return 0;
        a.cap /= TREE_S; lo = b0; hi = b1 + 1;
        a.set_lo = a.set_hi = 0; a.size = nullptr;
    }
}

struct SampleArgs {
    const double* sum; const double* mn; long long cap; const long long* size;
    int B, prioritized;
    const double* beta;
    unsigned long long* rng;
    long long* idx; float* w;
};

__global__ void __launch_bounds__(256) replay_sample_kernel(const __grid_constant__ SampleArgs a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long seed = a.rng[0], counter = a.rng[1];
    if (b < a.B) {
        uint32_t r[4];
        const double u = philox_u53(seed, (unsigned long long)b, (uint32_t)counter, SRL_PHILOX_PURPOSE_REPLAY, r);
        const long long n = *a.size;
        long long i;
        float w = 1.f;
        if (!a.prioritized) {
            i = (long long)(u * (double)n);
            if (i > n - 1) i = n - 1;
        } else {
            const double total = a.sum[1];
            double mass = u * total;
            long long node = 1;
            while (node < a.cap) {                           // find_prefixsum_idx
                const double left = a.sum[2 * node];
                if (left > mass) node = 2 * node;
                else { mass -= left; node = 2 * node + 1; }
            }
            i = node - a.cap;
            if (i > n - 1) i = n - 1;                        // rounding walked past the stored transitions into an empty leaf
            const double beta = *a.beta, nd = (double)n;
            const double max_w = pow(a.mn[1] / total * nd, -beta);
            w = (float)(pow(a.sum[a.cap + i] / total * nd, -beta) / max_w);
        }
        a.idx[b] = i;
        a.w[b] = w;
    }
    advance_counter(a.rng, counter);
}

// duplicates of a batch: the last occurrence writes its priority (the order baselines' update loop leaves), whatever order threads run in
__global__ void replay_stamp_kernel(int B, const long long* __restrict__ idx, int* stamp) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < B) atomicMax(stamp + idx[b], b);
}

__global__ void replay_priority_kernel(int B, const long long* __restrict__ idx, const float* __restrict__ td, int* stamp, double* sum, double* mn,
                                       long long cap, double* max_p, double alpha, float eps) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const long long i = idx[b];
    const float p = __fadd_rn(fabsf(td[b]), eps);           // priority = |td| + eps in float32
    if (stamp[i] == b) {
        const double leaf = pow((double)p, alpha);
        sum[cap + i] = leaf; mn[cap + i] = leaf;
        stamp[i] = -1;
    }
    // max_priority = max(max_priority, p): positive doubles order as their bit patterns
    atomicMax(reinterpret_cast<unsigned long long*>(max_p), (unsigned long long)__double_as_longlong((double)p));
}

int tree_ok(const char* who, const srl_replay_tree* t) {
    if (!t) { srl_set_error("%s: null tree", who); return 0; }
    if (t->struct_size != sizeof(srl_replay_tree)) { srl_set_error("%s: srl_replay_tree size mismatch", who); return 0; }
    if (t->n_envs < 1 || t->capacity < 1 || t->capacity % t->n_envs || t->tree_cap < t->capacity || (t->tree_cap & (t->tree_cap - 1)) ||
        t->capacity > 0x7FFFFFFFll) {
        srl_set_error("%s: bad tree shape n_envs=%d capacity=%lld tree_cap=%lld (tree_cap: the power of two >= capacity, a multiple of n_envs)", who,
                      t->n_envs, (long long)t->capacity, (long long)t->tree_cap);
        return 0;
    }
    if (!t->sum || !t->min || !t->max_priority || !t->size || !t->stamp) { srl_set_error("%s: null tree pointer", who); return 0; }
    return 1;
}

int q_ok(const char* who, const srl_mlp_policy* q) {
    if (!q) { srl_set_error("%s: null network", who); return 0; }
    if (q->struct_size != sizeof(srl_mlp_policy)) { srl_set_error("%s: srl_mlp_policy size mismatch", who); return 0; }
    if (!q->discrete || q->n_out < 2 || q->n_out > MAXO || q->obs_dim < 1 || q->obs_dim > SRL_POLICY_WIDE_OBS) {
        srl_set_error("%s: unsupported Q network discrete=%d obs_dim=%d n_out=%d (discrete only, obs_dim 1..%d, n_out 2..%d)", who, q->discrete, q->obs_dim,
                      q->n_out, SRL_POLICY_WIDE_OBS, MAXO);
        return 0;
    }
    if (!q->pi_w1 || !q->pi_b1 || !q->pi_w2 || !q->pi_b2 || !q->pi_w3 || !q->pi_b3 || !q->vf_w1 || !q->vf_b1 || !q->vf_w2 || !q->vf_b2 || !q->vf_w3 ||
        !q->vf_b3) { srl_set_error("%s: null weight pointer", who); return 0; }
    return 1;
}

int sm_count() {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return sms;
}

}  // namespace

extern "C" {

int srl_dqn_act(const srl_mlp_policy* q, int n, const float* obs, const float* eps, uint64_t* rng, uint64_t env_offset, float* obs_buf,
                int32_t* act_env, int64_t* act_buf, float* q_out, void* stream) {
    if (!q_ok("dqn_act", q)) return 1;
    if (!obs || !eps || !rng || !act_env) { srl_set_error("dqn_act: null argument"); return 1; }
    if (n <= 0) { srl_set_error("dqn_act: n must be positive"); return 1; }
    ActArgs a;
    a.q = *q; a.n = n; a.obs = obs; a.eps = eps; a.rng = reinterpret_cast<unsigned long long*>(rng); a.env_offset = env_offset;
    a.obs_buf = obs_buf; a.act_env = act_env; a.act_buf = reinterpret_cast<long long*>(act_buf); a.q_out = q_out;
    const int grid = (n + POLICY_ENVS - 1) / POLICY_ENVS;
    cudaStream_t st = (cudaStream_t)stream;
    if (q->obs_dim <= SRL_POLICY_MAX_OBS) {
        constexpr size_t smem = q_smem_bytes<SRL_POLICY_MAX_OBS>(1);
        SRL_CUDA_OK(srl_smem_opt_in<dqn_act_kernel<SRL_POLICY_MAX_OBS>>(smem));
        dqn_act_kernel<SRL_POLICY_MAX_OBS><<<grid, POLICY_BLOCK, smem, st>>>(a);
    } else {
        constexpr size_t smem = q_smem_bytes<SRL_POLICY_WIDE_OBS>(1);
        SRL_CUDA_OK(srl_smem_opt_in<dqn_act_kernel<SRL_POLICY_WIDE_OBS>>(smem));
        dqn_act_kernel<SRL_POLICY_WIDE_OBS><<<grid, POLICY_BLOCK, smem, st>>>(a);
    }
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_dqn_target(const srl_mlp_policy* online, const srl_mlp_policy* target, int batch, const int64_t* idx, const float* next_obs, const float* rew,
                   const uint8_t* done, float gamma, float* y, void* stream) {
    if (!q_ok("dqn_target", online) || !q_ok("dqn_target", target)) return 1;
    if (online->obs_dim != target->obs_dim || online->n_out != target->n_out) { srl_set_error("dqn_target: the two networks differ in shape"); return 1; }
    if (!next_obs || !rew || !done || !y) { srl_set_error("dqn_target: null argument"); return 1; }
    if (batch <= 0) { srl_set_error("dqn_target: batch must be positive"); return 1; }
    TargetArgs a;
    a.online = *online; a.target = *target; a.B = batch; a.idx = reinterpret_cast<const long long*>(idx); a.next_obs = next_obs; a.rew = rew;
    a.done = done; a.gamma = gamma; a.y = y;
    const int sms = sm_count();
    if (sms <= 0) { srl_set_error("dqn_target: no CUDA device"); return 1; }
    const int chunks = (batch + POLICY_ENVS - 1) / POLICY_ENVS, grid = chunks < sms ? chunks : sms;
    cudaStream_t st = (cudaStream_t)stream;
    if (online->obs_dim <= SRL_POLICY_MAX_OBS) {
        constexpr size_t smem = q_smem_bytes<SRL_POLICY_MAX_OBS>(2);
        SRL_CUDA_OK(srl_smem_opt_in<dqn_target_kernel<SRL_POLICY_MAX_OBS>>(smem));
        dqn_target_kernel<SRL_POLICY_MAX_OBS><<<grid, POLICY_BLOCK, smem, st>>>(a);
    } else {
        constexpr size_t smem = q_smem_bytes<SRL_POLICY_WIDE_OBS>(2);
        SRL_CUDA_OK(srl_smem_opt_in<dqn_target_kernel<SRL_POLICY_WIDE_OBS>>(smem));
        dqn_target_kernel<SRL_POLICY_WIDE_OBS><<<grid, POLICY_BLOCK, smem, st>>>(a);
    }
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_replay_add(const srl_replay_tree* t, int64_t row, double alpha, void* stream) {
    if (!tree_ok("replay_add", t)) return 1;
    const long long lo = (long long)row * t->n_envs;
    if (row < 0 || lo + t->n_envs > t->capacity) { srl_set_error("replay_add: row %lld outside the ring", (long long)row); return 1; }
    TreeArgs a = {};
    a.sum = t->sum; a.mn = t->min; a.cap = t->tree_cap; a.set_lo = lo; a.set_hi = lo + t->n_envs; a.max_p = t->max_priority; a.alpha = alpha;
    a.size = reinterpret_cast<long long*>(t->size); a.new_size = lo + t->n_envs;
    return rebuild(a, lo, lo + t->n_envs, (cudaStream_t)stream);
}

int srl_replay_sample(const srl_replay_tree* t, int batch, int prioritized, const double* beta, uint64_t* rng, int64_t* idx_out, float* w_out,
                      void* stream) {
    if (!tree_ok("replay_sample", t)) return 1;
    if (!rng || !idx_out || !w_out || (prioritized && !beta)) { srl_set_error("replay_sample: null argument"); return 1; }
    if (batch <= 0) { srl_set_error("replay_sample: batch must be positive"); return 1; }
    SampleArgs a;
    a.sum = t->sum; a.mn = t->min; a.cap = t->tree_cap; a.size = reinterpret_cast<const long long*>(t->size); a.B = batch; a.prioritized = prioritized;
    a.beta = beta; a.rng = reinterpret_cast<unsigned long long*>(rng); a.idx = reinterpret_cast<long long*>(idx_out); a.w = w_out;
    replay_sample_kernel<<<(batch + 255) / 256, 256, 0, (cudaStream_t)stream>>>(a);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int srl_replay_update(const srl_replay_tree* t, int batch, const int64_t* idx, const float* td, double alpha, float eps, void* stream) {
    if (!tree_ok("replay_update", t)) return 1;
    if (!idx || !td) { srl_set_error("replay_update: null argument"); return 1; }
    if (batch <= 0) { srl_set_error("replay_update: batch must be positive"); return 1; }
    cudaStream_t st = (cudaStream_t)stream;
    const long long* ix = reinterpret_cast<const long long*>(idx);
    replay_stamp_kernel<<<(batch + 255) / 256, 256, 0, st>>>(batch, ix, t->stamp);
    SRL_CUDA_OK(cudaGetLastError());
    replay_priority_kernel<<<(batch + 255) / 256, 256, 0, st>>>(batch, ix, td, t->stamp, t->sum, t->min, t->tree_cap, t->max_priority, alpha, eps);
    SRL_CUDA_OK(cudaGetLastError());
    TreeArgs a = {};
    a.sum = t->sum; a.mn = t->min; a.cap = t->tree_cap;
    return rebuild(a, 0, t->tree_cap, st);          // a full bottom-up rebuild: B samples touch most nodes above the lowest levels anyway
}

}  // extern "C"
