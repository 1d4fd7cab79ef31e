// MobileRobot family -- sm_90a kernels.
//
// Replaces MobileRobotGymEnv.reset/step/_reward/_termination
// (environments/mobile_robot/mobile_robot_env.py:159-222,235-280,336-363) and the three variants
// (mobile_robot_2target_env.py, mobile_robot_1D_env.py, mobile_robot_line_target_env.py) for
// thousands of independent envs held in structure-of-arrays HBM.  The reference teleports a
// fixed-base racecar (`resetBasePositionAndOrientation`, :265); there are no dynamics to integrate,
// so the kernel is the kinematic update + bump revert + reward + fixed-length episodes.
//
// Layout: one thread per env, 16-byte (double2 / int4) coalesced loads and stores of the state
// records; in the fused rollout the state lives in registers for all T steps and only
// action (4 B) in, obs (4-8 B) / reward (4 B) / done (1 B) out touch HBM per env-step.
//
// Arithmetic is float64 like the reference's numpy code, written with the explicit
// round-to-nearest intrinsics (__dadd_rn/__dmul_rn/__dsqrt_rn) so that no multiply-add is fused:
// positions, rewards and done flags are BIT-EXACT against the CPU restatement.
#include <stdio.h>
#include <stdlib.h>
#include <initializer_list>
#include <type_traits>
#include <cuda_pipeline_primitives.h>
#include "common.cuh"
#include "philox.cuh"

namespace {

// module constants, mobile_robot_env.py:13-28,101-104
constexpr double MAX_X = 4.0, MAX_Y = 4.0, MIN_X = 0.0, MIN_Y = 0.0;
constexpr double DELTA_POS = 0.1;
constexpr double ROBOT_WIDTH = 0.2, ROBOT_LENGTH = 0.325 * 2;
constexpr double COLLISION_MARGIN = 0.1;
constexpr double LINE_REWARD_DIST_THRESHOLD = 0.1, LINE_ROBOT_OFFSET = 0.2;  // line_target_env.py:3-4

struct MobileEnvRegs {
    double px, py;
    double t0x, t0y, t1x, t1y;
    int counter, current_target, has_bumped;
    uint32_t episode, total_steps;
    double ep_ret, ep_len;
};

__device__ __forceinline__ double uniform_rn(double low, double high, double u) {
    // numpy RandomState.uniform: low + (high - low) * random_sample()
    return __dadd_rn(low, __dmul_rn(high - low, u));
}

template <int KIND>
__device__ __forceinline__ void mobile_reset_env(MobileEnvRegs& e, const double* __restrict__ d6, bool random_target,
                                                 uint64_t seed, uint64_t genv) {
    double d[6];
    if (d6) {
#pragma unroll
        for (int k = 0; k < 6; ++k) d[k] = d6[k];
    } else {
        uint4 r = philox4x32_10(seed, genv, e.episode, PHILOX_PURPOSE_RESET0 + 0);
        d[0] = __dadd_rn(MAX_X / 2, uniform_rn(-MAX_X / 3, MAX_X / 3, philox_u01(r.x, r.y)));  // :168
        d[1] = __dadd_rn(MAX_Y / 2, uniform_rn(-MAX_Y / 3, MAX_Y / 3, philox_u01(r.z, r.w)));  // :169
        constexpr double margin = 0.1 * MAX_X;                                                  // :176
        d[2] = d[3] = d[4] = d[5] = 0.0;
        if (random_target) {
            r = philox4x32_10(seed, genv, e.episode, PHILOX_PURPOSE_RESET0 + 1);
            d[2] = uniform_rn(MIN_X + margin, MAX_X - margin, philox_u01(r.x, r.y));
            d[3] = uniform_rn(MIN_Y + margin, MAX_Y - margin, philox_u01(r.z, r.w));
            if (KIND == SRL_ENV_MOBILE_2TARGET) {
                r = philox4x32_10(seed, genv, e.episode, PHILOX_PURPOSE_RESET0 + 2);
                d[4] = uniform_rn(MIN_X + margin, MAX_X - margin, philox_u01(r.x, r.y));
                d[5] = uniform_rn(MIN_Y + margin, MAX_Y - margin, philox_u01(r.z, r.w));
            }
        }
    }
    e.px = d[0];
    e.py = (KIND == SRL_ENV_MOBILE_1D) ? 0.0 : d[1];  // 1D_env.py:66
    // fixed targets: mobile_robot_env.py:173-174, 2target_env.py:52-53,62-63, 1D_env.py:69, line_target_env.py:56-57
    double t0x = 0.9 * MAX_X, t0y = MAX_Y * 3 / 4, t1x = 0.1 * MAX_X, t1y = MAX_Y * 3 / 4;
    if (KIND == SRL_ENV_MOBILE_1D) t0y = 0.0;
    if (KIND == SRL_ENV_MOBILE_LINE_TARGET) t0y = MAX_X;
    if (random_target) {
        t0x = d[2];
        if (KIND == SRL_ENV_MOBILE || KIND == SRL_ENV_MOBILE_2TARGET) t0y = d[3];
        if (KIND == SRL_ENV_MOBILE_2TARGET) { t1x = d[4]; t1y = d[5]; }
    }
    e.t0x = t0x; e.t0y = t0y; e.t1x = t1x; e.t1y = t1y;
    e.current_target = 0;
    e.counter = 0;
    e.has_bumped = 0;
    e.ep_ret = 0.0;
    e.ep_len = 0.0;
    e.episode += 1;
}

// getSRLState = getGroundTruth() - getTargetPos()  (srl_env.py:39-42, RELATIVE_POS = True)
template <int KIND>
__device__ __forceinline__ void mobile_store_obs(const MobileEnvRegs& e, float* __restrict__ obs, size_t i) {
    const double tx = e.current_target ? e.t1x : e.t0x;
    const double ty = e.current_target ? e.t1y : e.t0y;
    if (KIND == SRL_ENV_MOBILE_1D) {
        obs[i] = (float)__dsub_rn(e.px, tx);
    } else if (KIND == SRL_ENV_MOBILE_LINE_TARGET) {
        const double lx = __dsub_rn(tx, LINE_ROBOT_OFFSET);  // line_target_env.py:35-40, 1-vector broadcast
        reinterpret_cast<float2*>(obs)[i] = make_float2((float)__dsub_rn(e.px, lx), (float)__dsub_rn(e.py, lx));
    } else {
        reinterpret_cast<float2*>(obs)[i] = make_float2((float)__dsub_rn(e.px, tx), (float)__dsub_rn(e.py, ty));
    }
}

__device__ __forceinline__ void mobile_load(const MobileDev& m, int i, MobileEnvRegs& e, bool two_targets) {
    const double2 p = m.pos[i];
    const double2 t0 = m.tgt0[i];
    const int4 mt = m.meta[i];
    const double2 ep = m.ep[i];
    e.px = p.x; e.py = p.y;
    e.t0x = t0.x; e.t0y = t0.y;
    e.t1x = 0.0; e.t1y = 0.0;
    if (two_targets) { const double2 t1 = m.tgt1[i]; e.t1x = t1.x; e.t1y = t1.y; }
    e.counter = mt.x;
    e.current_target = mt.y & 0xff;
    e.has_bumped = (mt.y >> 8) & 1;
    e.episode = (uint32_t)mt.z;
    e.total_steps = (uint32_t)mt.w;
    e.ep_ret = ep.x; e.ep_len = ep.y;
}

__device__ __forceinline__ void mobile_store(const MobileDev& m, int i, const MobileEnvRegs& e, bool store_targets,
                                             bool two_targets) {
    m.pos[i] = make_double2(e.px, e.py);
    if (store_targets) {
        m.tgt0[i] = make_double2(e.t0x, e.t0y);
        if (two_targets) m.tgt1[i] = make_double2(e.t1x, e.t1y);
    }
    m.meta[i] = make_int4(e.counter, e.current_target | (e.has_bumped << 8), (int)e.episode, (int)e.total_steps);
    m.ep[i] = make_double2(e.ep_ret, e.ep_len);
}

template <int KIND>
__global__ void __launch_bounds__(128) mobile_reset_kernel(MobileDev m, int n, const uint8_t* __restrict__ mask,
                                                           const double* __restrict__ draws,
                                                           float* __restrict__ obs, bool random_target, uint64_t seed,
                                                           uint64_t env_offset) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (mask && !mask[i]) return;
    MobileEnvRegs e;
    mobile_load(m, i, e, KIND == SRL_ENV_MOBILE_2TARGET);
    mobile_reset_env<KIND>(e, draws ? draws + (size_t)i * 6 : nullptr, random_target, seed, env_offset + (uint64_t)i);
    mobile_store(m, i, e, true, KIND == SRL_ENV_MOBILE_2TARGET);
    if (obs) mobile_store_obs<KIND>(e, obs, (size_t)i);
}

// sqrt_rn(s) <= 0.4  <=>  s <= S_THR_04 for every non-negative double s (sqrt is monotone and correctly rounded; the
// constant is the largest double whose rounded square root does not exceed 0.4, found by exact rational arithmetic).
// It lets the unshaped reward test `np.linalg.norm(.) <= REWARD_DIST_THRESHOLD` (:353) skip the square root BIT-EXACTLY.
constexpr double S_THR_04 = 0x1.47ae147ae147cp-3;

// ------------------------------------------------------------------------------------------------------------------
// Fused T-step rollout, EPISODE-PARALLEL.  T = 1 is the plain lockstep step.  Auto-reset on done reproduces the
// SubprocVecEnv worker loop (rl_baselines/utils.py:216-220): the stored obs is the post-reset one.
//
// Why (env, episode) and not (env) is the unit of parallel work.  `terminated` is never set in the reference
// (mobile_robot_env.py:355 is commented out), so an episode ends exactly when `_env_step_counter > max_steps` (:336-343):
// every episode is max_steps + 1 = 251 steps long, and the state an episode starts from is a pure function of the env's
// counter-based RNG stream (seed, global env index, episode index) -- it does not depend on the previous episode.  A
// T-step rollout of env i is therefore a sequence of INDEPENDENT segments whose boundaries are known before the first
// step runs:
//     segment 0   : steps [0, max_steps - counter]              starts from the state in HBM
//     segment s>0 : the next max_steps + 1 steps each           starts from reset(episode0 + s - 1)
// One thread runs one segment (blockIdx.y = segment): an 8192-env x 1024-step rollout becomes ~41 000 threads instead
// of 8192 (round 1: 256 warps for 592 schedulers, a ~600-cycle latency chain per step with nothing to overlap it).  The
// thread of a finished segment also produces the post-reset observation of the next one (it re-derives that reset),
// the thread whose segment reaches step T writes the state back.  State is double-buffered (`in` -> `out`): the
// segment-0 thread of an env may be scheduled after the thread that writes that env's final state.
// Arithmetic per step is the round-1 kernel's (same operations, same order): results stay bit-exact.
//
// Inside a segment (per chunk of MOBILE_PF steps):
//  * the action / noise streams do not depend on the state: PREFETCHED one chunk ahead into registers;
//  * pass 1 is the only serial part -- position += action, bump test, revert -- and records (target - position);
//  * pass 2 turns those into distance, reward, observation and the HBM stores; its steps are independent;
//  * nothing per-step is spent on episode bookkeeping: the step counter, `done`, the episode length follow from t, and
//    the unshaped episode return is an integer sum (rewards are -1 / 0 / 1: the float64 accumulation is exact either way).
constexpr int MOBILE_RING = 4;      // chunks of actions in the shared-memory ring (MOBILE_RING - 1 in flight ahead of the one being stepped; 4 was faster than 3 or 6)
constexpr int MOBILE_PF = 8;        // steps per chunk (8192 envs x 1024 steps: 8 was faster than 2 or 4)

template <bool DISCRETE, bool NOISE, int NS>
struct ActionChunk {
    int a[DISCRETE ? NS : 1];
    float x[DISCRETE ? 1 : NS], y[DISCRETE ? 1 : NS];
    float nz[NOISE ? NS : 1];
};

// actions of steps [t0, t0 + NS) of env i (idx0 = t0 * N + i): from HBM, or (GEN) the env's own stream -- the reference's random agent
template <int KIND, bool DISCRETE, bool GEN, bool NOISE, int NS>
__device__ __forceinline__ void load_chunk(ActionChunk<DISCRETE, NOISE, NS>& c, const void* __restrict__ actions, const float* __restrict__ noise,
                                           size_t N, size_t idx0, uint64_t seed, uint64_t genv, uint32_t total_steps0, int nvalid = NS) {
    constexpr uint32_t NA = (KIND == SRL_ENV_MOBILE_1D) ? 2u : 4u;
    size_t idx = idx0;
#pragma unroll
    for (int k = 0; k < NS; ++k) {
        if (k >= nvalid) {   // past the end of the segment: never stepped, never dereferenced
            c.a[DISCRETE ? k : 0] = 0; c.x[DISCRETE ? 0 : k] = 0.f; c.y[DISCRETE ? 0 : k] = 0.f; if (NOISE) c.nz[NOISE ? k : 0] = 0.f;
        } else if (GEN) {
            const uint4 r = philox4x32_10(seed, genv, total_steps0 + (uint32_t)k, PHILOX_PURPOSE_ACTION);
            if (DISCRETE) c.a[DISCRETE ? k : 0] = (int)__umulhi(r.x, NA);
            else {
                c.x[DISCRETE ? 0 : k] = (float)((double)r.x * (2.0 / 4294967296.0) - 1.0);
                c.y[DISCRETE ? 0 : k] = (float)((double)r.y * (2.0 / 4294967296.0) - 1.0);
            }
        } else if (DISCRETE) {
            c.a[DISCRETE ? k : 0] = __ldg(reinterpret_cast<const int32_t*>(actions) + idx);
        } else {
            const float2 v = __ldg(reinterpret_cast<const float2*>(actions) + idx);
            c.x[DISCRETE ? 0 : k] = v.x; c.y[DISCRETE ? 0 : k] = v.y;
        }
        if (NOISE && k < nvalid) c.nz[NOISE ? k : 0] = noise ? __ldg(noise + idx) : 0.f;
        idx += N;
    }
}

struct SegmentAcc {        // per-segment running values that are not part of the serial position chain
    int ret_i;             // unshaped: integer sum of the -1 / 0 / 1 rewards of this segment
    double ret_d;          // shaped: the float64 episode return, accumulated in step order
};

// NS steps of one env.  FAST = no noise stream and obs / rew / done all present (the rollout a trainer asks for): no per-step
// pointer tests, dv is the constant DELTA_POS.  MAYDONE = false: the caller guarantees that no step of the chunk ends an
// episode (true for every full chunk of a segment: an episode can only end on the segment's last step), so `done` is a
// constant 0 and the episode statistics are not touched.
template <int KIND, bool DISCRETE, bool SHAPED, bool FAST, bool MAYDONE, int NS>
__device__ __forceinline__ void step_chunk(MobileEnvRegs& e, SegmentAcc& acc, const ActionChunk<DISCRETE, !FAST, NS>& cur,
                                           int t0, int t_done, int t_start, size_t N, size_t idx0, double ep_ret0, double ep_len0,
                                           float* __restrict__ obs, float* __restrict__ rew, uint8_t* __restrict__ done,
                                           float* __restrict__ ep_ret, int32_t* __restrict__ ep_len, const double2* delta_table, int nvalid = NS) {
    constexpr bool TWO = (KIND == SRL_ENV_MOBILE_2TARGET);
    constexpr double mx = COLLISION_MARGIN + ROBOT_LENGTH / 2, my = COLLISION_MARGIN + ROBOT_WIDTH / 2;  // :257-258
    // ---------------- pass 1: the serial state chain (mobile_robot_env.py:237-268) ----------------
    // odx / ody = position - target: the observation (getSRLState = getGroundTruth() - getTargetPos(), srl_env.py:39-42) and,
    // up to an exact sign flip, the vector _reward() takes the norm of (:345-353)
    double odx[NS], ody[NS];
    float ox[TWO ? NS : 1], oy[TWO ? NS : 1];   // 2-target: the observation is relative to the target AFTER a switch
    uint32_t bump_mask = 0u, reach_mask = 0u;
#pragma unroll
    for (int k = 0; k < NS; ++k) {
        if (MAYDONE && k >= nvalid) { odx[k] = 0.0; ody[k] = 0.0; if (TWO) { ox[TWO ? k : 0] = 0.f; oy[TWO ? k : 0] = 0.f; } continue; }   // tail chunk: only its first nvalid steps exist
        // dv = DELTA_POS + np_random.normal(0.0, scale=NOISE_STD), NOISE_STD = 0.0 (:239-241)
        const double dv = FAST ? DELTA_POS : __dadd_rn(DELTA_POS, (double)cur.nz[FAST ? 0 : k]);
        double ax = 0.0, ay = 0.0;
        if (DISCRETE) {
            // dx = [-dv, dv, 0, 0][a], dy = [0, 0, -dv, dv][a] (:242-243; 1D_env.py:115), branch-free: even actions flip the
            // sign bit, the axis that does not move gets +0.0
            const int a = cur.a[DISCRETE ? k : 0];
            if (FAST && KIND != SRL_ENV_MOBILE_1D) {
                // the four (dx, dy) pairs of the constant dv = DELTA_POS (one LDS.128 instead of 8 integer instructions);
                // `a & 3` is Python's list index for a in [-4, 3]
                const double2 d = delta_table[a & 3];
                ax = d.x; ay = d.y;
            } else {
            const int hi = __double2hiint(dv) ^ ((a & 1) ? 0 : (int)0x80000000u), lo = __double2loint(dv);
            if (KIND == SRL_ENV_MOBILE_1D) ax = __hiloint2double(hi, lo);
            else {
                const bool along_x = (a & 2) == 0;
                ax = __hiloint2double(along_x ? hi : 0, along_x ? lo : 0);
                ay = __hiloint2double(along_x ? 0 : hi, along_x ? 0 : lo);
            }
            }
        } else {
            // float32 action array * python float -> float32 product, then += into float64 (:250,255)
            const float fdv = (float)dv;
            ax = (double)__fmul_rn(fmaxf(fminf(cur.x[DISCRETE ? 0 : k], 1.0f), -1.0f), fdv);
            ay = (double)__fmul_rn(fmaxf(fminf(cur.y[DISCRETE ? 0 : k], 1.0f), -1.0f), fdv);
        }
        const double nx = __dadd_rn(e.px, ax);                             // :254-255
        const double ny = (KIND != SRL_ENV_MOBILE_1D) ? __dadd_rn(e.py, ay) : e.py;
        bool bumped = (nx < mx) || (nx > MAX_X - mx);                      // :257-263
        if (KIND != SRL_ENV_MOBILE_1D) bumped = bumped || (ny < my) || (ny > MAX_Y - my);
        e.px = bumped ? e.px : nx;                                         // has_bumped: revert the whole position
        e.py = bumped ? e.py : ny;
        bump_mask |= (bumped ? 1u : 0u) << k;
        const double tx = e.current_target ? e.t1x : e.t0x, ty = e.current_target ? e.t1y : e.t0y;
        if (KIND == SRL_ENV_MOBILE_LINE_TARGET) {
            const double lx = __dsub_rn(tx, LINE_ROBOT_OFFSET);      // line_target_env.py:35-40,113: a 1-vector, broadcast
            odx[k] = __dsub_rn(e.px, lx); ody[k] = __dsub_rn(e.py, lx);
        } else {
            odx[k] = __dsub_rn(e.px, tx); ody[k] = (KIND == SRL_ENV_MOBILE_1D) ? 0.0 : __dsub_rn(e.py, ty);
        }
        if (TWO) {  // the target switch feeds later steps: decide it here (2target_env.py:170-173)
            const double sq = __dadd_rn(__dmul_rn(odx[k], odx[k]), __dmul_rn(ody[k], ody[k]));
            if (sq <= S_THR_04) {
                reach_mask |= 1u << k;
                if (e.current_target < 1) e.current_target += 1;   // the observation of THIS step is already relative to the new target
            }
            const double ux = e.current_target ? e.t1x : e.t0x, uy = e.current_target ? e.t1y : e.t0y;
            ox[TWO ? k : 0] = (float)__dsub_rn(e.px, ux); oy[TWO ? k : 0] = (float)__dsub_rn(e.py, uy);
        }
    }
    e.has_bumped = (bump_mask >> ((MAYDONE ? nvalid : NS) - 1)) & 1u;
    // ---------------- pass 2: rewards and outputs, independent across the chunk (:345-363) ----------------
    // Addresses: one 64-bit base per output stream and chunk, plus the 32-bit element offsets k * N (loop-invariant, hoisted): a store
    // address is then a single IMAD.WIDE.U32 instead of a carried 64-bit add (two instructions) per stream and step.
    float chunk_ret = 0.f;
    const uint32_t n32 = (uint32_t)N;                   // the launcher guarantees (NS - 1) * N < 2^32
    float* const rew_c = rew + idx0; uint8_t* const done_c = done + idx0;
    float* const obs1_c = obs + idx0; float2* const obs2_c = reinterpret_cast<float2*>(obs) + idx0;
    float* const ep_ret_c = ep_ret + idx0; int32_t* const ep_len_c = ep_len + idx0;
#pragma unroll
    for (int k = 0; k < NS; ++k) {
        if (MAYDONE && k >= nvalid) break;
        const uint32_t idx = (uint32_t)k * n32;
        const bool bumped = (bump_mask >> k) & 1u;
        float reward_f;
        if (SHAPED) {
            double distance;
            if (KIND == SRL_ENV_MOBILE_LINE_TARGET) distance = fabs(odx[k]);
            else if (KIND == SRL_ENV_MOBILE_1D) distance = __dsqrt_rn(__dmul_rn(odx[k], odx[k]));
            else distance = __dsqrt_rn(__dadd_rn(__dmul_rn(odx[k], odx[k]), __dmul_rn(ody[k], ody[k])));  // np.linalg.norm = sqrt(x.dot(x))
            acc.ret_d = __dadd_rn(acc.ret_d, -distance);
            reward_f = (float)(-distance);
        } else {
            bool reached;
            if (KIND == SRL_ENV_MOBILE_LINE_TARGET) reached = fabs(odx[k]) <= LINE_REWARD_DIST_THRESHOLD;
            else if (TWO) reached = (reach_mask >> k) & 1u;
            else if (KIND == SRL_ENV_MOBILE_1D) reached = __dmul_rn(odx[k], odx[k]) <= S_THR_04;
            else reached = __dadd_rn(__dmul_rn(odx[k], odx[k]), __dmul_rn(ody[k], ody[k])) <= S_THR_04;
            reward_f = bumped ? -1.f : (reached ? 1.f : 0.f);
            chunk_ret += reward_f;              // a sum of at most NS values from {-1, 0, 1}: exact in float32
            if (MAYDONE) { acc.ret_i += (int)chunk_ret; chunk_ret = 0.f; }   // the tail chunk reads the running return at its done step
        }
        if (FAST || rew) rew_c[idx] = reward_f;
        if (MAYDONE) {
            const int t = t0 + k;
            const bool is_done = t >= t_done;   // _termination (:336-343); `terminated` is never set
            if (FAST || done) done_c[idx] = is_done ? 1 : 0;
            if (is_done) {   // Monitor-style episode statistics (environments/utils.py:53-54)
                if (ep_ret) ep_ret_c[idx] = (float)(SHAPED ? acc.ret_d : __dadd_rn(ep_ret0, (double)acc.ret_i));
                if (ep_len) ep_len_c[idx] = (int32_t)ep_len0 + (t - t_start + 1);
            }
        } else if (FAST || done) done_c[idx] = 0;
        if (FAST || obs) {
            if (KIND == SRL_ENV_MOBILE_1D) obs1_c[idx] = (float)odx[k];
            else if (TWO) obs2_c[idx] = make_float2(ox[TWO ? k : 0], oy[TWO ? k : 0]);
            else obs2_c[idx] = make_float2((float)odx[k], (float)ody[k]);
        }
    }
    if (!SHAPED && !MAYDONE) acc.ret_i += (int)chunk_ret;
}

template <int KIND, bool DISCRETE, bool GEN, bool SHAPED, bool FAST>
__global__ void __launch_bounds__(128) mobile_rollout_kernel(MobileDev in, MobileDev out, int n, int T, const void* __restrict__ actions,
                                                             const float* __restrict__ noise, float* __restrict__ obs,
                                                             float* __restrict__ rew, uint8_t* __restrict__ done,
                                                             float* __restrict__ ep_ret, int32_t* __restrict__ ep_len,
                                                             bool random_target, bool auto_reset,
                                                             int max_steps, uint64_t seed, uint64_t env_offset) {
    // dx = [-dv, dv, 0, 0][a], dy = [0, 0, -dv, dv][a] (mobile_robot_env.py:242-243) for the constant dv of the FAST instantiation
    __shared__ double2 s_delta[4];
    if (FAST && DISCRETE && KIND != SRL_ENV_MOBILE_1D) {
        if (threadIdx.x < 4) s_delta[threadIdx.x] = threadIdx.x < 2 ? make_double2(threadIdx.x ? DELTA_POS : -DELTA_POS, 0.0)
                                                                     : make_double2(0.0, threadIdx.x == 3 ? DELTA_POS : -DELTA_POS);
        __syncthreads();   // before any thread leaves
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    constexpr bool TWO = (KIND == SRL_ENV_MOBILE_2TARGET);
    constexpr int D = (KIND == SRL_ENV_MOBILE_1D) ? 1 : 2;
    constexpr int PF = MOBILE_PF;
    const int seg = blockIdx.y;
    const uint64_t genv = env_offset + (uint64_t)i;
    const size_t N = (size_t)n;
    // ---- segment boundaries from the env's step counter alone ----
    const int4 mt = in.meta[i];
    int t_done0 = max_steps - mt.x;                 // step at which `counter > max_steps` first holds
    t_done0 = t_done0 < 0 ? 0 : (t_done0 > T ? T : t_done0);
    int t_start = 0, t_done = t_done0;
    if (seg > 0) {                                  // only launched with auto_reset
        const long long ts = (long long)t_done0 + 1 + (long long)(seg - 1) * ((long long)max_steps + 1);
        if (ts >= T) return;
        t_start = (int)ts;
        t_done = (ts + max_steps > T) ? T : (int)(ts + max_steps);
    }
    if (t_start >= T) return;
    const int t_end = auto_reset ? (t_done + 1 < T ? t_done + 1 : T) : T;
    const int t_plain = t_done < t_end ? t_done : t_end;   // steps [t_start, t_plain) cannot end an episode
    MobileEnvRegs e;
    if (seg == 0) mobile_load(in, i, e, TWO);   // independent of the boundary arithmetic above: these loads overlap the meta load
    else {
        e.episode = (uint32_t)mt.z + (uint32_t)(seg - 1);
        e.total_steps = (uint32_t)mt.w + (uint32_t)t_start;
        mobile_reset_env<KIND>(e, nullptr, random_target, seed, genv);
    }
    const int c_start = e.counter;
    const uint32_t ts_start = e.total_steps;
    const double ep_ret0 = e.ep_ret, ep_len0 = e.ep_len;
    SegmentAcc acc; acc.ret_i = 0; acc.ret_d = e.ep_ret;
    int t0 = t_start;
    size_t idx = (size_t)t_start * N + (size_t)i;          // element index of (t0, env i) in the [T, N] streams
    const size_t idx0 = idx;
    const size_t chunk_stride = (size_t)PF * N;
    // The steps after the last full plain chunk -- at most PF - 1 plain ones and the step that ends the episode -- run as ONE
    // masked chunk; its actions are requested now, so their latency hides behind the whole main loop.
    const int n_full = (t_plain - t_start) / PF;
    const int t_tail = t_start + n_full * PF;
    ActionChunk<DISCRETE, !FAST, PF> tl;
    int tail_valid = t_end - t_tail < PF ? t_end - t_tail : PF;
    if (!GEN) load_chunk<KIND, DISCRETE, GEN, !FAST, PF>(tl, actions, noise, N, idx + (size_t)n_full * chunk_stride, seed, genv, 0u, tail_valid);
    if (n_full > 0) {
        ActionChunk<DISCRETE, !FAST, PF> c0;
        if (GEN) {
#pragma unroll 1
            for (; t0 < t_tail; t0 += PF, idx += chunk_stride) {
                load_chunk<KIND, DISCRETE, GEN, !FAST, PF>(c0, actions, noise, N, idx, seed, genv, ts_start + (uint32_t)(t0 - t_start));
                step_chunk<KIND, DISCRETE, SHAPED, FAST, false, PF>(e, acc, c0, t0, t_done, t_start, N, idx, ep_ret0, ep_len0, obs, rew, done, ep_ret, ep_len, s_delta);
            }
        } else {
            // ACTION RING in shared memory, filled by cp.async (LDGSTS) MOBILE_RING - 1 chunks ahead of the chunk being stepped.
            // Registers cannot carry loads that far: rotating a register ring copies values that are still in flight, and the copy
            // waits for them (ncu: one instruction, the first use of a chunk's first action, held the largest share of the stall
            // samples as `long_sb` with a 2- or 3-deep register ring).  cp.async needs no destination register, each thread
            // reads back only what it wrote itself (no barrier, only wait_group), and slot (stage, step) of the 32 lanes of a warp
            // is one 128-byte row: conflict-free.
            using Elem = typename std::conditional<DISCRETE, int32_t, float2>::type;
            extern __shared__ __align__(16) unsigned char s_ring_raw[];
            Elem* ring = reinterpret_cast<Elem*>(s_ring_raw);
            const Elem* src = reinterpret_cast<const Elem*>(actions);
            const int tid = threadIdx.x;
            constexpr int nthr = 128;     // ring row stride = the largest CTA (compile-time: slots are [base + immediate])
            auto issue = [&](int chunk) {       // chunk index within this segment; an empty group keeps the group count uniform
                if (chunk < n_full) {
                    const Elem* g = src + idx0 + (size_t)chunk * chunk_stride;
                    Elem* dst = ring + (size_t)((chunk % MOBILE_RING) * PF) * nthr + tid;
#pragma unroll
                    for (int k = 0; k < PF; ++k) __pipeline_memcpy_async(dst + (size_t)k * nthr, g + (uint32_t)k * (uint32_t)N, sizeof(Elem));
                }
                __pipeline_commit();
            };
#pragma unroll
            for (int c = 0; c < MOBILE_RING - 1; ++c) issue(c);
            int chunk = 0;
#pragma unroll 1
            for (; t0 < t_tail; t0 += PF, idx += chunk_stride, ++chunk) {
                issue(chunk + MOBILE_RING - 1);
                __pipeline_wait_prior(MOBILE_RING - 1);                   // everything up to and including `chunk` has landed
                const Elem* slot = ring + (size_t)((chunk % MOBILE_RING) * PF) * nthr + tid;
#pragma unroll
                for (int k = 0; k < PF; ++k) {
                    if constexpr (DISCRETE) c0.a[k] = slot[(size_t)k * nthr];
                    else { const float2 v = slot[(size_t)k * nthr]; c0.x[DISCRETE ? 0 : k] = v.x; c0.y[DISCRETE ? 0 : k] = v.y; }
                    if (!FAST) c0.nz[FAST ? 0 : k] = noise ? __ldg(noise + idx + (size_t)k * N) : 0.f;
                }
                step_chunk<KIND, DISCRETE, SHAPED, FAST, false, PF>(e, acc, c0, t0, t_done, t_start, N, idx, ep_ret0, ep_len0, obs, rew, done, ep_ret, ep_len, s_delta);
            }
            __pipeline_wait_prior(0);
        }
    }
#pragma unroll 1
    for (; t0 < t_end; t0 += PF, idx += chunk_stride) {   // one iteration with auto-reset; more only when stepping on past `done`
        tail_valid = t_end - t0 < PF ? t_end - t0 : PF;
        if (GEN || t0 != t_tail) load_chunk<KIND, DISCRETE, GEN, !FAST, PF>(tl, actions, noise, N, idx, seed, genv, ts_start + (uint32_t)(t0 - t_start), tail_valid);
        step_chunk<KIND, DISCRETE, SHAPED, FAST, true, PF>(e, acc, tl, t0, t_done, t_start, N, idx, ep_ret0, ep_len0, obs, rew, done, ep_ret, ep_len, s_delta, tail_valid);
    }
    const int steps = t_end - t_start;
    e.counter = c_start + steps;                                   // :268
    e.total_steps = ts_start + (uint32_t)steps;
    e.ep_ret = SHAPED ? acc.ret_d : __dadd_rn(ep_ret0, (double)acc.ret_i);
    e.ep_len = ep_len0 + (double)steps;
    if (auto_reset && t_end - 1 >= t_done) {
        // the segment ended its episode: SubprocVecEnv resets and returns the POST-RESET observation for that step
        mobile_reset_env<KIND>(e, nullptr, random_target, seed, genv);
        if (obs) mobile_store_obs<KIND>(e, obs + (size_t)(t_end - 1) * N * D, (size_t)i);   // same thread, same address: overwrites the terminal one
    }
    if (t_end == T) mobile_store(out, i, e, true, TWO);
}

template <int KIND, bool DISCRETE, bool GEN, bool SHAPED, bool FAST>
int launch_rollout_variant(srl_sim* s, int T, const void* actions, const float* noise, float* obs, float* rew, uint8_t* done,
                           float* ep_ret, int32_t* ep_len, cudaStream_t st) {
    // segments per env: 1 + the episodes that can start inside T steps (worst case: the first step ends an episode)
    const long long per = (long long)s->max_steps + 1;
    const int nseg = s->auto_reset ? (int)(1 + ((long long)T - 1 + per - 1) / per) : 1;
    // one warp per CTA while the whole launch is a few warps per SM: spreads the (latency-bound) warps over all SMs
    const long long warps = (long long)nseg * ((s->n + 31) / 32);
    const int block = warps <= (long long)s->sms * 4 ? 32 : 128;
    const dim3 grid((unsigned)((s->n + block - 1) / block), (unsigned)nseg);
    const size_t ring_bytes = GEN ? 0 : (size_t)MOBILE_RING * MOBILE_PF * 128 * (DISCRETE ? sizeof(int32_t) : sizeof(float2));   // rows of 128 lanes whatever the CTA size
    mobile_rollout_kernel<KIND, DISCRETE, GEN, SHAPED, FAST><<<grid, block, ring_bytes, st>>>(s->mob, s->mob_alt, s->n, T, actions, noise, obs, rew, done, ep_ret, ep_len,
                                                                                       s->cfg.random_target != 0, s->auto_reset != 0,
                                                                                       s->max_steps, s->seed, s->cfg.global_env_offset);
    SRL_CUDA_OK(cudaGetLastError());
    const MobileDev tmp = s->mob; s->mob = s->mob_alt; s->mob_alt = tmp;   // stream-ordered: later launches read what this one wrote
    return 0;
}

template <int KIND, bool DISCRETE, bool GEN>
int launch_rollout_gen(srl_sim* s, int T, const void* actions, const float* noise, float* obs, float* rew, uint8_t* done,
                       float* ep_ret, int32_t* ep_len, cudaStream_t st) {
    const bool fast = !noise && obs && rew && done;
    if (s->cfg.shape_reward)
        return fast ? launch_rollout_variant<KIND, DISCRETE, GEN, true, true>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st)
                    : launch_rollout_variant<KIND, DISCRETE, GEN, true, false>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st);
    return fast ? launch_rollout_variant<KIND, DISCRETE, GEN, false, true>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st)
                : launch_rollout_variant<KIND, DISCRETE, GEN, false, false>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st);
}

template <int KIND>
int launch_rollout_kind(srl_sim* s, int T, const void* actions, const float* noise, float* obs, float* rew, uint8_t* done,
                        float* ep_ret, int32_t* ep_len, cudaStream_t st) {
    if (s->cfg.is_discrete)
        return actions ? launch_rollout_gen<KIND, true, false>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st)
                       : launch_rollout_gen<KIND, true, true>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st);
    // continuous actions exist for the 2-D kinds only (srl_sim_create rejects them for the others): no kernels for the rest
    if constexpr (KIND == SRL_ENV_MOBILE || KIND == SRL_ENV_MOBILE_LINE_TARGET)
        return actions ? launch_rollout_gen<KIND, false, false>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st)
                       : launch_rollout_gen<KIND, false, true>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st);
    else {
        srl_set_error("rollout: env kind %d has no continuous actions", KIND);
        return 1;
    }
}

}  // namespace

static int mobile_alloc_one(MobileDev& m, size_t N) {
    SRL_CUDA_OK(cudaMalloc(&m.pos, N * sizeof(double2)));
    SRL_CUDA_OK(cudaMalloc(&m.tgt0, N * sizeof(double2)));
    SRL_CUDA_OK(cudaMalloc(&m.tgt1, N * sizeof(double2)));
    SRL_CUDA_OK(cudaMalloc(&m.meta, N * sizeof(int4)));
    SRL_CUDA_OK(cudaMalloc(&m.ep, N * sizeof(double2)));
    SRL_CUDA_OK(cudaMemset(m.pos, 0, N * sizeof(double2)));
    SRL_CUDA_OK(cudaMemset(m.tgt0, 0, N * sizeof(double2)));
    SRL_CUDA_OK(cudaMemset(m.tgt1, 0, N * sizeof(double2)));
    SRL_CUDA_OK(cudaMemset(m.meta, 0, N * sizeof(int4)));
    SRL_CUDA_OK(cudaMemset(m.ep, 0, N * sizeof(double2)));
    return 0;
}

// Two copies of the 80 B/env state: a rollout reads `mob` and writes `mob_alt`, then the two swap (see the kernel header).
int mobile_alloc(srl_sim* s) {
    const size_t N = (size_t)s->n;
    if (mobile_alloc_one(s->mob, N)) return 1;
    if (mobile_alloc_one(s->mob_alt, N)) return 1;
    return 0;
}

void mobile_free(srl_sim* s) {
    for (MobileDev* m : {&s->mob, &s->mob_alt}) {
        cudaFree(m->pos); cudaFree(m->tgt0); cudaFree(m->tgt1); cudaFree(m->meta); cudaFree(m->ep);
        *m = MobileDev{};
    }
}

int mobile_launch_reset(srl_sim* s, const uint8_t* mask, const double* draws, float* obs, cudaStream_t st) {
    const int block = 128, grid = (s->n + block - 1) / block;
    const bool rt = s->cfg.random_target != 0;
    switch (s->kind) {
    case SRL_ENV_MOBILE: mobile_reset_kernel<SRL_ENV_MOBILE><<<grid, block, 0, st>>>(s->mob, s->n, mask, draws, obs, rt, s->seed, s->cfg.global_env_offset); break;
    case SRL_ENV_MOBILE_2TARGET: mobile_reset_kernel<SRL_ENV_MOBILE_2TARGET><<<grid, block, 0, st>>>(s->mob, s->n, mask, draws, obs, rt, s->seed, s->cfg.global_env_offset); break;
    case SRL_ENV_MOBILE_1D: mobile_reset_kernel<SRL_ENV_MOBILE_1D><<<grid, block, 0, st>>>(s->mob, s->n, mask, draws, obs, rt, s->seed, s->cfg.global_env_offset); break;
    default: mobile_reset_kernel<SRL_ENV_MOBILE_LINE_TARGET><<<grid, block, 0, st>>>(s->mob, s->n, mask, draws, obs, rt, s->seed, s->cfg.global_env_offset); break;
    }
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int mobile_launch_rollout(srl_sim* s, int T, const void* actions, const float* noise, float* obs, float* rew, uint8_t* done,
                          float* ep_ret, int32_t* ep_len, cudaStream_t st) {
    switch (s->kind) {
    case SRL_ENV_MOBILE: return launch_rollout_kind<SRL_ENV_MOBILE>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st);
    case SRL_ENV_MOBILE_2TARGET: return launch_rollout_kind<SRL_ENV_MOBILE_2TARGET>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st);
    case SRL_ENV_MOBILE_1D: return launch_rollout_kind<SRL_ENV_MOBILE_1D>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st);
    default: return launch_rollout_kind<SRL_ENV_MOBILE_LINE_TARGET>(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st);
    }
}

// ---- host-side state access (debug / single-env accessors; not on the hot path) -------------
#include <vector>

int mobile_get_state(srl_sim* s, int field, void* dst, size_t bytes) {
    const size_t N = (size_t)s->n;
    std::vector<double2> a(N), b(N);
    std::vector<int4> mt(N);
    SRL_CUDA_OK(cudaDeviceSynchronize());
    SRL_CUDA_OK(cudaMemcpy(mt.data(), s->mob.meta, N * sizeof(int4), cudaMemcpyDeviceToHost));
    switch (field) {
    case SRL_F_ROBOT_POS:
    case SRL_F_TARGET_POS: {
        if (bytes != N * 3 * sizeof(double)) { srl_set_error("get_state: size mismatch"); return 1; }
        double* o = (double*)dst;
        if (field == SRL_F_ROBOT_POS) {
            SRL_CUDA_OK(cudaMemcpy(a.data(), s->mob.pos, N * sizeof(double2), cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < N; ++i) { o[3 * i] = a[i].x; o[3 * i + 1] = a[i].y; o[3 * i + 2] = 0.0; }
        } else {
            SRL_CUDA_OK(cudaMemcpy(a.data(), s->mob.tgt0, N * sizeof(double2), cudaMemcpyDeviceToHost));
            SRL_CUDA_OK(cudaMemcpy(b.data(), s->mob.tgt1, N * sizeof(double2), cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < N; ++i) {
                const double2 t = (mt[i].y & 0xff) ? b[i] : a[i];
                o[3 * i] = t.x; o[3 * i + 1] = t.y; o[3 * i + 2] = 0.0;
            }
        }
        return 0;
    }
    case SRL_F_STEP_COUNTER:
        if (bytes != N * sizeof(int32_t)) { srl_set_error("get_state: size mismatch"); return 1; }
        for (size_t i = 0; i < N; ++i) ((int32_t*)dst)[i] = mt[i].x;
        return 0;
    case SRL_F_COUNTERS:
        if (bytes != N * 4 * sizeof(int32_t)) { srl_set_error("get_state: size mismatch"); return 1; }
        for (size_t i = 0; i < N; ++i) {
            int32_t* o = (int32_t*)dst + 4 * i;
            o[0] = mt[i].y & 0xff; o[1] = (mt[i].y >> 8) & 1; o[2] = 0; o[3] = mt[i].z;
        }
        return 0;
    case SRL_F_EPISODE_STATS:
        if (bytes != N * 2 * sizeof(double)) { srl_set_error("get_state: size mismatch"); return 1; }
        SRL_CUDA_OK(cudaMemcpy(dst, s->mob.ep, N * sizeof(double2), cudaMemcpyDeviceToHost));
        return 0;
    default:
        srl_set_error("get_state: field %d not available for MobileRobot", field);
        return 1;
    }
}

int mobile_set_state(srl_sim* s, int field, const void* src, size_t bytes) {
    const size_t N = (size_t)s->n;
    SRL_CUDA_OK(cudaDeviceSynchronize());
    switch (field) {
    case SRL_F_ROBOT_POS:
    case SRL_F_TARGET_POS: {
        if (bytes != N * 3 * sizeof(double)) { srl_set_error("set_state: size mismatch"); return 1; }
        const double* in = (const double*)src;
        std::vector<double2> a(N);
        for (size_t i = 0; i < N; ++i) a[i] = make_double2(in[3 * i], in[3 * i + 1]);
        if (field == SRL_F_ROBOT_POS) {
            SRL_CUDA_OK(cudaMemcpy(s->mob.pos, a.data(), N * sizeof(double2), cudaMemcpyHostToDevice));
        } else {
            std::vector<int4> mt(N);
            std::vector<double2> t0(N), t1(N);
            SRL_CUDA_OK(cudaMemcpy(mt.data(), s->mob.meta, N * sizeof(int4), cudaMemcpyDeviceToHost));
            SRL_CUDA_OK(cudaMemcpy(t0.data(), s->mob.tgt0, N * sizeof(double2), cudaMemcpyDeviceToHost));
            SRL_CUDA_OK(cudaMemcpy(t1.data(), s->mob.tgt1, N * sizeof(double2), cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < N; ++i) ((mt[i].y & 0xff) ? t1[i] : t0[i]) = a[i];
            SRL_CUDA_OK(cudaMemcpy(s->mob.tgt0, t0.data(), N * sizeof(double2), cudaMemcpyHostToDevice));
            SRL_CUDA_OK(cudaMemcpy(s->mob.tgt1, t1.data(), N * sizeof(double2), cudaMemcpyHostToDevice));
        }
        return 0;
    }
    case SRL_F_STEP_COUNTER: {
        if (bytes != N * sizeof(int32_t)) { srl_set_error("set_state: size mismatch"); return 1; }
        std::vector<int4> mt(N);
        SRL_CUDA_OK(cudaMemcpy(mt.data(), s->mob.meta, N * sizeof(int4), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < N; ++i) mt[i].x = ((const int32_t*)src)[i];
        SRL_CUDA_OK(cudaMemcpy(s->mob.meta, mt.data(), N * sizeof(int4), cudaMemcpyHostToDevice));
        return 0;
    }
    default:
        srl_set_error("set_state: field %d not settable for MobileRobot", field);
        return 1;
    }
}
