// Kuka button-push family -- kernels and host launchers (sm_90a).  KukaRandButton's distractor bodies: distractor_kernels.cu.
//
// Replaces, for thousands of envs in lockstep, KukaButtonGymEnv.reset/step/step2/_reward/_termination
// (environments/kuka_gym/kuka_button_gym_env.py:214-281,293-368,422-463), Kuka.applyAction
// (environments/kuka_gym/kuka.py:118-187) and the PyBullet calls behind them.
//
// Mapping: all dynamic state of an env in registers for the whole fused rollout.  By default an env is a GROUP of 4 lanes
// (kuka_coop.cuh), which share out the once-per-step kinematics and dynamics and run the projected Gauss-Seidel solve (150 sweeps x
// >= 13 strictly sequential rows, a chain no intra-env parallelism shortens) redundantly; `envs_per_warp` <= 8 spreads the batch at one
// warp per warp scheduler.  One thread per env is the layout for batches that need more than 8 envs per warp (above 4 224 envs on
// an H100).  With next-episode records on (KukaNext), 4096 envs run at 7 envs per warp instead of 8, so that every warp keeps the idle
// slot that produces them.  The robot model arrives as a __grid_constant__ parameter block (constant bank, folded into FFMA operands).  HBM traffic
// is the SoA state once per launch (float4 / int4 records, coalesced) plus action + noise in and obs + reward + done out per step.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "common.cuh"
#include "kuka_state.cuh"
#include "kuka_device.cuh"
#include "render_core.h"

// "Next episode" records (opt-in, srl_cfg.prefetch_resets): the post-reset state of every env's NEXT episode -- a pure function of
// (seed, global env index, episode index) -- produced ahead of time, so that a LOCKSTEP step whose env finishes an episode copies a
// record in instead of running reset()'s five random micro-steps inside the launch (measured: every steady-state launch of 4096 envs
// contains such an env, and it made the launch several times longer).
// Who produces them (round 2): the first IDLE SLOT of every warp of every rollout / step launch.  A batch is spread over all warp schedulers, so
// a warp carries fewer envs (7 of 8 groups of 4 lanes, or 7 of 32 lanes, at 4096 envs) than it has slots; the idle slot picks one env of its
// own warp whose record is incomplete and advances that record by (at most T) random micro-steps of reset() -- ONE per lockstep launch, the
// very instructions its warp is executing anyway, so the launch stays one physics step long and costs no extra issue slot; a record is
// complete after five launches.  (Round 1's version ran the whole five-step reset in a separate launch on a side stream: bit-identical, memcheck
// clean, but its long launches shared schedulers with 2-4 following step launches and doubled their duration.  A helper CTA on the
// last SM worked too, but cannot serve enough records once an env takes 4 lanes.)
// op = PREFETCH as a launch of its own (srl_sim_prefetch_resets) remains as the bulk fill after an explicit reset of all envs.
struct KukaNext : KukaState {
    uint8_t* valid;     // [N] 1 = record complete and not yet consumed
    int32_t* episode;   // [N] episode index the record was produced for (a record for another episode is dropped)
    uint8_t* progress;  // [N] random micro-steps of reset() already applied to an incomplete record (0 = not started)
    int helper;         // 1 (rollout launches): the first idle slot of every warp advances an incomplete record of its warp's envs (see kuka_kernel)
};

namespace {

constexpr float DELTA_V = 0.03f, DELTA_V_CONTINUOUS = 0.0035f, DELTA_THETA = 0.1f;   // kuka_button_gym_env.py:27-29
constexpr double NOISE_STD = 0.01, NOISE_STD_CONTINUOUS = 0.0001, NOISE_STD_JOINTS = 0.002;   // :31-33
constexpr int N_CONTACTS_BEFORE_TERMINATION = 5, N_STEPS_OUTSIDE_SAFETY_SPHERE = 5000, N_RANDOM_ACTIONS_AT_INIT = 5;

// CG: read through L2 only (__ldcg) -- for records another kernel may have completed while this one was already running
template <bool CG, class T>
KK_DEV T ld_state(const T* p) { return CG ? __ldcg(p) : *p; }

template <bool TWOB, bool CG = false>
KK_DEV void env_load(const KukaState& d, int i, KukaEnv& e) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float4 a = ld_state<CG>(d.q[k] + i), b = ld_state<CG>(d.qd[k] + i);
        e.q[4 * k] = a.x; e.q[4 * k + 1] = a.y; e.q[4 * k + 2] = a.z; e.q[4 * k + 3] = a.w;
        e.qd[4 * k] = b.x; e.qd[4 * k + 1] = b.y; e.qd[4 * k + 2] = b.z; e.qd[4 * k + 3] = b.w;
    }
    const float4 m0 = ld_state<CG>(d.misc0 + i), m1 = ld_state<CG>(d.misc1 + i), tg = ld_state<CG>(d.tgt + i), gr = ld_state<CG>(d.grip + i),
                 ep = ld_state<CG>(d.eepos + i);
    const int4 c = ld_state<CG>(d.cnt + i), c2 = ld_state<CG>(d.cnt2 + i);
    e.ee[0] = m0.x; e.ee[1] = m0.y; e.ee[2] = m0.z; e.qb = m0.w;
    e.qdb = m1.x; e.bbx = m1.y; e.bby = m1.z; e.ep_ret = m1.w;
    e.tgt[0] = tg.x; e.tgt[1] = tg.y; e.tgt[2] = tg.z; e.bbz = tg.w;
    e.grip[0] = gr.x; e.grip[1] = gr.y; e.grip[2] = gr.z; e.bspeed = gr.w;
    e.eepos[0] = ep.x; e.eepos[1] = ep.y; e.eepos[2] = ep.z;
    e.counter = c.x; e.n_contacts = c.y; e.n_outside = c.z;
    e.terminated = c.w & 1; e.cbutton = (c.w >> 1) & 1; e.ctable = (c.w >> 2) & 1;
    e.episode = (uint32_t)c2.x; e.total_steps = (uint32_t)c2.y; e.ep_len = c2.z;
    e.by64 = __hiloint2double(c2.w, __float_as_int(ep.w));
    e.qb2 = 0.f; e.qdb2 = 0.f; e.bb2x = 0.f; e.bb2y = 0.f; e.n_contacts2 = 0; e.goal_id = 0; e.cany0 = 0; e.cany1 = 0;
    if (TWOB) {
        const float4 b2 = ld_state<CG>(d.btn2 + i);
        e.qb2 = b2.x; e.qdb2 = b2.y; e.bb2x = b2.z; e.bb2y = b2.w;
        e.n_contacts2 = c2.w; e.by64 = 0.0;
        e.cany0 = (c.w >> 3) & 1; e.cany1 = (c.w >> 4) & 1; e.goal_id = (c.w >> 5) & 1;
    }
}

template <bool TWOB>
KK_DEV void env_store(const KukaState& d, int i, const KukaEnv& e) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        d.q[k][i] = make_float4(e.q[4 * k], e.q[4 * k + 1], e.q[4 * k + 2], e.q[4 * k + 3]);
        d.qd[k][i] = make_float4(e.qd[4 * k], e.qd[4 * k + 1], e.qd[4 * k + 2], e.qd[4 * k + 3]);
    }
    d.misc0[i] = make_float4(e.ee[0], e.ee[1], e.ee[2], e.qb);
    d.misc1[i] = make_float4(e.qdb, e.bbx, e.bby, e.ep_ret);
    d.tgt[i] = make_float4(e.tgt[0], e.tgt[1], e.tgt[2], e.bbz);
    d.grip[i] = make_float4(e.grip[0], e.grip[1], e.grip[2], e.bspeed);
    d.eepos[i] = make_float4(e.eepos[0], e.eepos[1], e.eepos[2], __int_as_float(__double2loint(e.by64)));
    int flags = e.terminated | (e.cbutton << 1) | (e.ctable << 2);
    if (TWOB) flags |= (e.cany0 << 3) | (e.cany1 << 4) | (e.goal_id << 5);
    d.cnt[i] = make_int4(e.counter, e.n_contacts, e.n_outside, flags);
    d.cnt2[i] = make_int4((int)e.episode, (int)e.total_steps, e.ep_len, TWOB ? e.n_contacts2 : __double2hiint(e.by64));
    if (TWOB) d.btn2[i] = make_float4(e.qb2, e.qdb2, e.bb2x, e.bb2y);
}

// Kuka.applyAction's accumulate + clip of the commanded end-effector position (kuka.py:134-139)
KK_DEV void apply_ee_delta(const KukaParams& P, KukaEnv& e, float dx, float dy, float dz) {
    e.ee[0] = fminf(fmaxf(e.ee[0] + dx, P.box[0]), P.box[1]);
    e.ee[1] = fminf(fmaxf(e.ee[1] + dy, P.box[2]), P.box[3]);
    e.ee[2] = fminf(fmaxf(e.ee[2] + dz, P.box[4]), P.box[5]);
}

// Decode the reference's random initial action k of reset() (:250-268) from host draws or the env's stream.
KK_DEV void reset_action(const KukaParams& P, const double* __restrict__ d17, uint64_t genv, uint32_t episode, int s,
                         float& dx, float& dy, float& dz) {
    dx = dy = dz = 0.f;
    if (d17) { dx = (float)d17[2 + 3 * s]; dy = (float)d17[3 + 3 * s]; dz = (float)d17[4 + 3 * s]; return; }
    const uint4 r = philox4x32_10(P.seed, genv, episode, PHILOX_PURPOSE_RESET0 + 1 + s);
    if (P.action_joints) {
        // joints += DELTA_THETA * np_random.normal(joints.shape): ONE draw from N(loc=7, 1), broadcast to the 7 joints (:257-260);
        // carried in dx as the common set-point offset
        const double u1 = philox_u01(r.x, r.y), u2 = philox_u01(r.z, r.w);
        dx = (float)(0.1 * (7.0 + sqrt(-2.0 * log(1.0 - u1)) * cos(6.283185307179586 * u2)));
    } else if (P.is_discrete) {
        const float sign = philox_u01(r.x, r.y) > 0.5 ? 1.f : -1.f;     // np_random.rand() > 0.5
        const uint32_t idx = __umulhi(r.z, 3u);                          // np_random.randint(3)
        dx = idx == 0 ? sign * DELTA_V : 0.f; dy = idx == 1 ? sign * DELTA_V : 0.f; dz = idx == 2 ? sign * DELTA_V : 0.f;
    } else {
        // np_random.normal((3,)) is ONE draw from N(loc=3, 1); normalised it is +-1 on all three axes (:263-266)
        const double u1 = philox_u01(r.x, r.y), u2 = philox_u01(r.z, r.w);
        const double z = sqrt(-2.0 * log(1.0 - u1)) * cos(6.283185307179586 * u2);
        const float sign = (3.0 + z) >= 0.0 ? 1.f : -1.f;
        dx = dy = dz = sign * DELTA_V_CONTINUOUS;
    }
}

// reset(), first half: restore the post-settle snapshot and place the button (:214-247)
template <bool TWOB>
KK_DEV void reset_begin(const KukaParams& P, KukaEnv& e, const double* __restrict__ d17, uint64_t genv) {
#pragma unroll
    for (int i = 0; i < KK_NB; ++i) { e.q[i] = P.snap_q[i]; e.qd[i] = P.snap_qd[i]; }
    e.ee[0] = P.snap_ee[0]; e.ee[1] = P.snap_ee[1]; e.ee[2] = P.snap_ee[2];
    e.qb = P.snap_qb; e.qdb = P.snap_qdb;
    e.bbx = P.btn_base[0]; e.bby = P.btn_base[1]; e.bbz = P.btn_base[2];
    e.bspeed = 0.f;
    if (P.moving_button) {   // BUTTON_SPEED * np_random.choice([-1, 1]) (kuka_moving_button_gym_env.py:33)
        if (d17) e.bspeed = (float)d17[17];
        else e.bspeed = (philox4x32_10(P.seed, genv, e.episode, PHILOX_PURPOSE_RESET0 + 6).x & 1u) ? 0.001f : -0.001f;
    }
    e.by64 = (double)P.btn_base[1];
    if (TWOB) {
        // kuka_2button_gym_env.py:49-69: button 1 always sits at (0.5, 0.125) (its random placement is overwritten, :56-57);
        // button 2 at (0.5, -0.125), or x = 0.5 + 0.15 U(-1, 1), y = -0.125 + 0.175 U(-1, 0) with random_target
        e.qb2 = P.snap_qb; e.qdb2 = P.snap_qdb;       // both buttons settle identically (nothing touches them in the 500 steps)
        e.bb2x = P.btn_base[0]; e.bb2y = -P.btn_base[1];
        if (P.random_target) {
            if (d17) { e.bb2x = (float)d17[0]; e.bb2y = (float)d17[1]; }
            else {
                const uint4 r = philox4x32_10(P.seed, genv, e.episode, PHILOX_PURPOSE_RESET0);
                e.bb2x = (float)((double)P.btn_base[0] + (double)P.rand_x * (-1.0 + 2.0 * philox_u01(r.x, r.y)));
                e.bb2y = (float)(-(double)P.btn_base[1] + 0.175 * (-1.0 + philox_u01(r.z, r.w)));
            }
        }
        return;
    }
    if (P.random_target) {
        if (d17) { e.bbx = (float)d17[0]; e.bby = (float)d17[1]; e.by64 = d17[1]; }
        else {
            const uint4 r = philox4x32_10(P.seed, genv, e.episode, PHILOX_PURPOSE_RESET0);
            e.bbx = (float)((double)P.btn_base[0] + (double)P.rand_x * (-1.0 + 2.0 * philox_u01(r.x, r.y)));  // :230
            e.by64 = (double)P.btn_base[1] + (double)P.rand_y * (-1.0 + 2.0 * philox_u01(r.z, r.w));              // :231
            e.bby = (float)e.by64;
        }
    }
}

// reset(), second half: after the random steps, freeze the target and clear the episode counters (:273-274,215-217)
template <bool TWOB>
KK_DEV void reset_end(const KukaParams& P, KukaEnv& e) {
    e.tgt[0] = e.bbx; e.tgt[1] = e.bby;
    e.tgt[2] = e.bbz + P.glider_z + e.qb + P.target_h;  // button link state + BUTTON_DISTANCE_HEIGHT
    if (TWOB) e.tgt[2] = P.two_tgt_z;          // button_all_pos = [x, y, Z_TABLE + BUTTON_DISTANCE_HEIGHT] (kuka_2button_gym_env.py:59,69,72)
    if (TWOB) { e.n_contacts2 = 0; e.goal_id = 0; }
    e.counter = 0; e.n_contacts = 0; e.n_outside = 0; e.terminated = 0;
    e.ep_ret = 0.f; e.ep_len = 0;
    e.episode += 1;
}

enum { KUKA_OP_ROLLOUT = 0, KUKA_OP_RESET = 1, KUKA_OP_SETTLE = 2, KUKA_OP_PREFETCH = 3 };

// ONE kernel for reset, lockstep step and fused T-step rollout.  Every thread runs a single micro-step loop
//     forward kinematics + collision detection  ->  [finish the env step whose physics just ran: reward, done,
//     auto-reset]  ->  pick the next micro action (policy action, or one of reset()'s random actions)  ->  physics
// so that the expensive bodies (FK, dynamics, PGS) exist exactly once in the instruction stream, and an env that is
// inside reset()'s 5 random steps costs its warp 5 extra micro-steps and nothing else.
//   op = ROLLOUT: T env steps (step() + step2() + _reward() + _termination() + VecEnv auto-reset)
//   op = RESET  : reset() of the masked envs with optional host-supplied draws
//   op = SETTLE : the 500 zero-action steps of reset() (:242-247), identical for every episode -> snapshot
//   op = PREFETCH (PREFETCH instantiation only): reset() of the env's NEXT episode into its `nx` record, for the envs whose record is
//                 not valid -- the very instructions of the in-launch reset, so a record and an in-launch reset agree bit for bit
// PREFETCH = false (the default instantiations): `nx` is ignored and the kernel is what it was before the feature existed.
#ifdef KK_TIMING
// diagnostic build (scripts/build_variant.sh timing -DKK_TIMING): per env slot of the LAST launch, cycles from kernel entry to the slot's exit (high word)
// and what its last physics step did (low word: 1 watched loop, 2 general loop, nc << 2, 64 joint limit, general sweeps << 8, 1 << 16 episode finished,
// 1 << 17 record taken, 1 << 18 helper slot)
__device__ unsigned long long kk_timing[1 << 16];
#define KK_TIMING_RECORD() do { if (lead) kk_timing[(warp * (COOP ? 8 : 32) + slot) & 0xFFFF] = ((unsigned long long)(clock64() - kk_t0) << 32) | dbgf | (helper ? 1u << 18 : 0u); } while (0)
#else
#define KK_TIMING_RECORD() do { } while (0)
#endif
#ifdef KK_PHASES
// diagnostic build (scripts/build_variant.sh phases -DKK_PHASES): per env slot of the LAST launch, cycles spent in each phase of the micro-step
// loop (KK_PH_* of kuka_device.cuh), then the number of physics steps the slot ran and how many of them ran the watch copy of the fast loop
__device__ unsigned long long kk_phase[1 << 13][KK_NPH + 2];
#endif
// TRACE (KukaRandButton with distractor bodies only): every micro-step also writes the arm configuration it starts from and what kind
// of micro-step it is to `trace` (layout: kuka_state.cuh), and each env its number of micro-steps to `trace_len`; distractor_kernel
// (distractor_kernels.cu) then advances the bodies through the same micro-steps.  TRACE = false: the kernel is what it was before.
template <bool JOINTS, bool TWOB, bool PREFETCH = false, bool COOP = false, bool TRACE = false>
__global__ void __launch_bounds__(128, 1) kuka_kernel(const __grid_constant__ KukaDev d, int n, int op, int T,
                                                       const void* __restrict__ actions, const float* __restrict__ noise,
                                                       const uint8_t* __restrict__ mask, const double* __restrict__ draws,
                                                       float* __restrict__ obs, float* __restrict__ rew,
                                                       uint8_t* __restrict__ done, float* __restrict__ ep_ret,
                                                       int32_t* __restrict__ ep_len, float* __restrict__ snap, const KukaNext nx,
                                                       float4* __restrict__ trace, int* __restrict__ trace_len) {
    // Thread -> env.  One thread per env (COOP = false: lane l of a warp carries the warp's env l, `epw` live lanes), or a GROUP of 4 adjacent
    // lanes per env (COOP = true: kuka_coop.cuh; group g = lane / 4 carries env g, `epw` <= 8 live groups): all 4 lanes hold identical copies of
    // the env state and run the env logic and the sweeps redundantly; `u` = lane within the group deals out the once-per-step work.
    const int lane = threadIdx.x & 31, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
#ifdef KK_TIMING
    const long long kk_t0 = clock64(); unsigned dbgf = 0u;
#endif
#ifdef KK_PHASES
    KkPhaseClock kk_ph_clk; KkPhaseClock* const ph = &kk_ph_clk; unsigned kk_nphys = 0u;
    kk_ph_clk.last = (unsigned)clock();
#pragma unroll
    for (int k2 = 0; k2 < KK_NPH; ++k2) kk_ph_clk.acc[k2] = 0;
    kk_ph_clk.nwatch = 0u;
#else
    KkPhaseClock* const ph = nullptr;
#endif
    const int slot = COOP ? lane >> 2 : lane;            // env slot within the warp
    const int u = COOP ? lane & 3 : 0;
    const bool lead = !COOP || u == 0;                   // the lane of the group that talks to global memory
    const unsigned gmask = COOP ? 0xFu << (lane & ~3) : 0u;
    extern __shared__ float4 kc_smem[];
    float* const kc_tab = reinterpret_cast<float*>(kc_smem);                                   // per-CTA model tables
    KcScratch sc;                                                                              // this env's scratch area
    sc.b = reinterpret_cast<float*>(kc_smem) + ((KC_CONST_WORDS + 31) / 32) * 32 + (8 * (threadIdx.x >> 5) + (lane >> 2)) * KC_ES;
    if constexpr (COOP) {
        kc_fill_const(d.P, kc_tab, threadIdx.x, blockDim.x);
        __syncthreads();
    }
    int i = -1;
    if (slot < d.epw) { i = warp * d.epw + slot; if (i >= n) i = -1; }
    bool helper = false;         // PREFETCH: this thread (group) advances the next-episode record of one env of its warp
    if constexpr (PREFETCH) {
        // helper slot = the first idle slot of the warp: it runs the same micro-step loop as the warp's envs (SIMT: at no extra issue cost)
        if (nx.helper && op == KUKA_OP_ROLLOUT && slot == d.epw && slot < (COOP ? 8 : 32)) {
            int pick = -1;
            if (lead) {          // first env of this warp whose record is incomplete, a record in progress first
                int best = -1;
                for (int k2 = 0; k2 < d.epw; ++k2) {
                    const int j = warp * d.epw + k2;
                    if (j < n && !reinterpret_cast<volatile const uint8_t*>(nx.valid)[j]) {
                        const int pr = nx.progress[j];
                        if (pr > best) { best = pr; pick = j; }
                    }
                }
            }
            if (COOP) pick = __shfl_sync(gmask, pick, lane & ~3);
            if (pick >= 0) { i = pick; helper = true; op = KUKA_OP_PREFETCH; }
        }
    }
    if (i < 0) return;
    if (op == KUKA_OP_RESET && mask && !mask[i]) return;
    if constexpr (PREFETCH) { if (op == KUKA_OP_PREFETCH && !helper && nx.valid[i]) return; }
    const KukaParams& P = d.P;
    const uint64_t genv = P.env_offset + (uint64_t)i;
    const size_t N = (size_t)n;
    KukaEnv e; KukaKin k; KukaContacts ct;
    env_load<TWOB>(d, i, e);
    int nc_reg = 0;              // COOP: contact rows of the current configuration (the manifold itself lives in the scratch area)
    if constexpr (PREFETCH) {
        // the helper slot has read the live state and the record flags of an env that another slot of this warp is about to step:
        // nobody moves on before everybody has loaded
        __syncwarp();
    }

    int reset_left = 0;          // > 0: inside reset(), this many random micro-steps to go
    bool in_reset = false;       // reset() in progress (finalised when reset_left reaches 0)
    bool pending = false;        // an env step's physics has run; reward / done / obs still to be produced
    int rep = 0, t = 0;
    int saved_cb = 0, saved_ct = 0, saved_a0 = 0, saved_a1 = 0;
    float dx = 0.f, dy = 0.f, dz = 0.f;
    float qj[JOINTS ? 7 : 1];   // joint-space micro action: the 7 arm set-points (action_joints)
#pragma unroll
    for (int j = 0; j < (JOINTS ? 7 : 1); ++j) qj[j] = 0.f;
    const double* d17 = nullptr;
    if (op == KUKA_OP_RESET) {
        d17 = draws ? draws + (size_t)i * (TRACE ? KUKA_DIST_DRAWS : 18) : nullptr;
        reset_begin<TWOB>(P, e, d17, genv);
        in_reset = true; reset_left = N_RANDOM_ACTIONS_AT_INIT;
    } else if (op == KUKA_OP_SETTLE) {
#pragma unroll
        for (int j = 0; j < KK_NB; ++j) { e.q[j] = P.snap_q[j]; e.qd[j] = 0.f; }  // resetJointState (kuka.py:68-69)
        e.ee[0] = P.ee_init[0]; e.ee[1] = P.ee_init[1]; e.ee[2] = P.ee_init[2];
        e.qb = 0.f; e.qdb = 0.f; e.bbx = P.btn_base[0]; e.bby = P.btn_base[1]; e.bbz = P.btn_base[2]; e.bspeed = 0.f; e.by64 = 0.0;
        if (TWOB) { e.qb2 = 0.f; e.qdb2 = 0.f; e.bb2x = P.btn_base[0]; e.bb2y = -P.btn_base[1]; }
        in_reset = true; reset_left = 500;
    }
    int ms = 0;                  // TRACE: micro-steps of this env in this launch
    bool consumed = false;       // PREFETCH: the env just took its next-episode record (reset_end is already part of it)
    bool partial = false;        // helper: the launch ends before the record is complete
    int budget = T;              // helper: random micro-steps this launch may add to the record
    if constexpr (PREFETCH) {
        if (op == KUKA_OP_PREFETCH) {   // e.episode (live state) is the index the env's next reset() will draw with
            const int prog = helper ? (int)nx.progress[i] : 0;
            if (prog > 0 && nx.episode[i] == (int)e.episode) {
                // continue the record where the previous launch left it: the loop-carried state of reset() is all in KukaEnv, the
                // kinematics are recomputed from it -- the same values in the same instructions as an uninterrupted reset
                env_load<TWOB, true>(nx, i, e);
                in_reset = true; reset_left = N_RANDOM_ACTIONS_AT_INIT - prog;
            } else {
                if (helper && lead) nx.episode[i] = (int)e.episode;
                reset_begin<TWOB>(P, e, nullptr, genv);
                in_reset = true; reset_left = N_RANDOM_ACTIONS_AT_INIT;
            }
        }
    }
    // COOP: an env that is done with the loop does not leave it alone: it waits at the loop head until every env of its warp is done.
    // The vote there is the one point where all groups of the warp meet at the start of every micro-step.  Without it, a group that
    // branches off (reset(), a taken record, the end of the rollout) stays off the others' instruction stream for the rest of the launch:
    // a group running its reset micro-steps and the groups running their env steps execute the same code at different times, and the warp
    // issues every instruction of the sweeps once per stream.  (Lanes that returned before the loop have exited, which the vote allows.)
    // what an env does when it leaves the micro-step loop: write its state back (or publish its next-episode record).  With 4 lanes per env
    // this runs where the env leaves, before it waits for the rest of its warp: a record completed by a helper slot is published while the
    // other envs of the launch are still running, so an episode that ends later in the same launch can take it
    auto leave = [&]() {
        e.cbutton = saved_cb; e.ctable = saved_ct;
        if (TWOB) { e.cany0 = saved_a0; e.cany1 = saved_a1; }
        KK_TIMING_RECORD();
        if constexpr (TRACE) { if (lead && op != KUKA_OP_SETTLE) trace_len[i] = ms; }
#ifdef KK_PHASES
        KK_PH(ph, KK_PH_ENV);
        if (lead) {
            unsigned long long* const kp = kk_phase[(warp * (COOP ? 8 : 32) + slot) & ((1 << 13) - 1)];
#pragma unroll
            for (int k2 = 0; k2 < KK_NPH; ++k2) kp[k2] = (unsigned long long)kk_ph_clk.acc[k2];
            kp[KK_NPH] = kk_nphys;
            kp[KK_NPH + 1] = kk_ph_clk.nwatch;
        }
#endif
        if constexpr (PREFETCH) {
            if (op == KUKA_OP_PREFETCH) {
                if (!lead) return;
                env_store<TWOB>(nx, i, e);
                if (partial) { nx.progress[i] = (uint8_t)(N_RANDOM_ACTIONS_AT_INIT - reset_left); return; }   // nx.episode[i] was set when the record was begun
                nx.episode[i] = (int)e.episode - 1;   // record first, then the episode it is for, then the flag
                nx.progress[i] = 0;
                __threadfence();
                reinterpret_cast<volatile uint8_t*>(nx.valid)[i] = 1;
                return;
            }
        }
        if (lead) env_store<TWOB>(d, i, e);
    };
    bool fin = false, settled = false;
#define KK_LEAVE_LOOP() { if (COOP) { leave(); fin = true; continue; } else break; }
    for (;;) {
        if constexpr (COOP) {
            if (__all_sync(0xffffffffu, fin)) break;
            if (fin) continue;
        }
        // link states of the configuration just reached + collision detection for the next step
        if constexpr (COOP) {
            KcKinIn kin;
#pragma unroll
            for (int j = 0; j < KK_NB; ++j) kin.q[j] = e.q[j];
            kin.qb = e.qb; kin.qb2 = e.qb2; kin.bbx = e.bbx; kin.bby = e.bby; kin.bbz = e.bbz; kin.bb2x = e.bb2x; kin.bb2y = e.bb2y;
            KK_PH(ph, KK_PH_ENV);
            __syncwarp(gmask);   // the group is done with the rows / matrices of the previous micro-step (the candidates reuse that storage)
            const bool near = kc_kinematics<TWOB>(sc, kc_tab, P, kin, u, gmask, ph);
            e.grip[0] = sc[8 * KC_BS + KB_C]; e.grip[1] = sc[8 * KC_BS + KB_C + 1]; e.grip[2] = sc[8 * KC_BS + KB_C + 2];   // getLinkState(kuka, 8)[0]: COM of link 8
            e.eepos[0] = sc[6 * KC_BS + KB_P]; e.eepos[1] = sc[6 * KC_BS + KB_P + 1]; e.eepos[2] = sc[6 * KC_BS + KB_P + 2];
            const int fl = near ? (int)sc[KC_OFF_LINK + 6] : 0;
            e.cbutton = fl & 1; e.ctable = (fl >> 1) & 1;
            if (TWOB) { e.cany0 = (fl >> 2) & 1; e.cany1 = (fl >> 3) & 1; }
            nc_reg = near ? (int)sc[KC_OFF_LINK + 7] : 0;
            KK_PH(ph, KK_PH_KIN_COLLECT);
        } else { KK_PH(ph, KK_PH_ENV); kuka_fk<TWOB>(P, e, k, ct); KK_PH(ph, KK_PH_KIN_COLLECT); }
        const int new_cb = e.cbutton, new_ct = e.ctable, new_a0 = TWOB ? e.cany0 : 0, new_a1 = TWOB ? e.cany1 : 0;
        if (pending) {
            // ---- _reward() (:428-463): manifold of the step that just ran, link states after it ----
            pending = false;
            const size_t off = (size_t)t * N + (size_t)i;
            const float ddx = e.tgt[0] - e.grip[0], ddy = e.tgt[1] - e.grip[1], ddz = e.tgt[2] - e.grip[2];
            const float distance = sqrtf(ddx * ddx + ddy * ddy + ddz * ddz);
            float reward;
            if (TWOB) {
                // Kuka2ButtonGymEnv._reward (kuka_2button_gym_env.py:157-214): contact with ANY link of the goal button; the sparse
                // reward only counts on the last button; 5 contacts on button 1 switch the goal (and the target) to button 2
                const int contact = e.goal_id ? saved_a1 : saved_a0;
                reward = 0.f;
                if (e.goal_id) { e.n_contacts2 += contact; reward = contact ? 1.f : 0.f; }
                else {
                    e.n_contacts += contact;
                    if (e.n_contacts >= N_CONTACTS_BEFORE_TERMINATION) { e.goal_id = 1; e.tgt[0] = e.bb2x; e.tgt[1] = e.bb2y; }
                }
                if (distance > P.max_distance || saved_ct) { reward = -1.f; e.n_outside += 1; } else e.n_outside = 0;
                if (saved_ct || e.n_contacts2 >= N_CONTACTS_BEFORE_TERMINATION || e.n_outside >= N_STEPS_OUTSIDE_SAFETY_SPHERE - 1) e.terminated = 1;
                if (P.shape_reward) {
                    const int n_goal = e.goal_id ? e.n_contacts2 : e.n_contacts;   // of the goal AFTER a possible switch (:198)
                    if (e.terminated && reward > 0.f) reward = 50.f;
                    else if (n_goal < N_CONTACTS_BEFORE_TERMINATION && contact) reward = 25.f;
                    else if (saved_ct) reward = -250.f;
                    else if (distance > P.max_distance) reward = -20.f;
                    else reward = -distance;
                }
            } else {
            reward = saved_cb ? 1.f : 0.f;
            e.n_contacts += saved_cb;
            if (distance > P.max_distance || saved_ct) { reward = -1.f; e.n_outside += 1; } else e.n_outside = 0;
            if (saved_ct || e.n_contacts >= N_CONTACTS_BEFORE_TERMINATION || e.n_outside >= N_STEPS_OUTSIDE_SAFETY_SPHERE) e.terminated = 1;
            if (P.shape_reward) {
                if (P.is_discrete) reward = -distance;
                else if (e.terminated && reward > 0.f) reward = 50.f;
                else if (e.terminated && reward < 0.f) reward = -250.f;
                else reward = -distance;
            }
            }
            const bool is_done = e.terminated || e.counter > P.max_steps;  // _termination() (:422-426)
#ifdef KK_TIMING
            if (is_done) dbgf |= 1u << 16;
#endif
            e.ep_ret += reward; e.ep_len += 1;
            if (rew && lead) rew[off] = reward;
            if (done && lead) done[off] = is_done ? 1 : 0;
            if (is_done && lead) {
                if (ep_ret) ep_ret[off] = e.ep_ret;
                if (ep_len) ep_len[off] = e.ep_len;
            }
            if (is_done && P.auto_reset) {   // SubprocVecEnv worker: reset and return the post-reset observation
                if constexpr (PREFETCH) {
                    if (op == KUKA_OP_ROLLOUT) {
                        // 0: no record, 1: a complete record for another episode (explicit reset in between: dropped), 2: the record of this episode.
                        // Read by the group's lead lane and broadcast: the 4 lanes must take the same branch whatever the helper is doing meanwhile
                        int rec = 0;
                        if (lead && reinterpret_cast<volatile const uint8_t*>(nx.valid)[i]) {
                            __threadfence();     // the record was written before the flag (message passing with op = PREFETCH)
                            rec = reinterpret_cast<volatile const int32_t*>(nx.episode)[i] == (int)e.episode ? 2 : 1;
                        }
                        if (COOP) rec = __shfl_sync(gmask, rec, lane & ~3);
#ifdef KK_TIMING
                        if (rec == 2) dbgf |= 1u << 17;
#endif
                        if (rec == 2) {
                            const uint32_t total_steps = e.total_steps;         // the only field that runs across episodes
                            env_load<TWOB, true>(nx, i, e);
                            e.total_steps = total_steps;
                            __threadfence();   // the record is read before the flag is cleared: a PREFETCH thread that sees 0 may overwrite it
                            if (COOP) __syncwarp(gmask);
                        }
                        if (rec && lead) reinterpret_cast<volatile uint8_t*>(nx.valid)[i] = 0;   // consumed or stale: to be produced again
                        if (rec == 2) {
                            saved_cb = e.cbutton; saved_ct = e.ctable;           // what the in-launch reset leaves behind: the manifold flags of its last micro-step
                            if (TWOB) { saved_a0 = e.cany0; saved_a1 = e.cany1; }
                            consumed = true; in_reset = true; reset_left = 0;
                            continue;          // kinematics of the post-reset configuration, then the observation (below)
                        }
                    }
                }
                d17 = nullptr;
                reset_begin<TWOB>(P, e, nullptr, genv);
                in_reset = true; reset_left = N_RANDOM_ACTIONS_AT_INIT;
                continue;                      // the snapshot configuration needs its own kinematics
            }
            if (obs && lead) { float* o = obs + 3 * off; o[0] = e.grip[0] - e.tgt[0]; o[1] = e.grip[1] - e.tgt[1]; o[2] = e.grip[2] - e.tgt[2]; }
            ++t;
        }
        if (in_reset && reset_left == 0) {
            in_reset = false;
            if (op == KUKA_OP_SETTLE) {
                if (lead) {
                    for (int j = 0; j < KK_NB; ++j) { snap[j] = e.q[j]; snap[KK_NB + j] = e.qd[j]; }
                    snap[24] = e.ee[0]; snap[25] = e.ee[1]; snap[26] = e.ee[2]; snap[27] = e.qb; snap[28] = e.qdb;
                }
                settled = true;                 // no state to write back
                if (COOP) { fin = true; continue; } else break;
            }
            if (!(PREFETCH && consumed)) reset_end<TWOB>(P, e);
            consumed = false;
            if (obs && lead && op != KUKA_OP_PREFETCH) {  // getSRLState after reset (:278-279)
                float* o = obs + 3 * (op == KUKA_OP_RESET ? (size_t)i : (size_t)t * N + (size_t)i);
                o[0] = e.grip[0] - e.tgt[0]; o[1] = e.grip[1] - e.tgt[1]; o[2] = e.grip[2] - e.tgt[2];
            }
            if (op == KUKA_OP_ROLLOUT) ++t;
        }
        if (!in_reset && (op != KUKA_OP_ROLLOUT || t >= T)) KK_LEAVE_LOOP()
        // ---- next micro action ----
        bool armed;
        if (in_reset) {
            if (op == KUKA_OP_SETTLE) { dx = dy = dz = 0.f; }
            else reset_action(P, d17, genv, e.episode, N_RANDOM_ACTIONS_AT_INIT - reset_left, dx, dy, dz);
            if (JOINTS) {   // settle: the initial joint vector (:244); random init: the same vector + one common offset (:257-260)
#pragma unroll
                for (int j = 0; j < 7; ++j) qj[JOINTS ? j : 0] = P.qinit[j] + dx;
            }
            --reset_left;
            armed = false;  // the button motor is only commanded from step2() (:347)
        } else {
            if (rep == 0) {
                // ---- step(): action decoding + noise (:293-340) ----
                const size_t off = (size_t)t * N + (size_t)i;
                float nz;
                if (noise) nz = __ldg(noise + off);
                else {
                    const uint4 r = philox4x32_10(P.seed, genv, e.total_steps, PHILOX_PURPOSE_NOISE);
                    const double u1 = philox_u01(r.x, r.y), u2 = philox_u01(r.z, r.w);
                    nz = (float)((JOINTS ? NOISE_STD_JOINTS : P.is_discrete ? NOISE_STD : NOISE_STD_CONTINUOUS) * sqrt(-2.0 * log(1.0 - u1)) * cos(6.283185307179586 * u2));
                }
                dx = dy = dz = 0.f;
                uint4 ra = make_uint4(0, 0, 0, 0);
                if (!actions) ra = philox4x32_10(P.seed, genv, e.total_steps, PHILOX_PURPOSE_ACTION);
                if (JOINTS) {
                    // real_action = action * (DELTA_THETA + N(0, NOISE_STD_JOINTS)) + joint_positions[:7] (:317-323): set-points
                    // relative to the INITIAL joint vector, which the reference never updates (kuka.py:65-66)
                    float a7[7];
                    if (actions) {
                        const float* ap = reinterpret_cast<const float*>(actions) + 7 * off;
#pragma unroll
                        for (int j = 0; j < 7; ++j) a7[j] = __ldg(ap + j);
                    } else {
                        const uint4 rb = philox4x32_10(P.seed, genv, e.total_steps, PHILOX_PURPOSE_ACTION + 1);
                        const uint32_t w[7] = {ra.x, ra.y, ra.z, ra.w, rb.x, rb.y, rb.z};
#pragma unroll
                        for (int j = 0; j < 7; ++j) a7[j] = (float)((double)w[j] * (2.0 / 4294967296.0) - 1.0);
                    }
                    const float d_theta = DELTA_THETA + nz;
#pragma unroll
                    for (int j = 0; j < 7; ++j) qj[JOINTS ? j : 0] = fmaf(a7[j], d_theta, P.qinit[j]);
                } else if (P.is_discrete) {
                    const int a = actions ? __ldg(reinterpret_cast<const int32_t*>(actions) + off) : (int)__umulhi(ra.x, 6u);
                    if (a >= 0) {  // a < 0 is the reference's step(None): zero action (:295-299)
                        const float dv = DELTA_V + nz;
                        const int am = a % 6;
                        dx = am == 0 ? -dv : am == 1 ? dv : 0.f;
                        dy = am == 2 ? -dv : am == 3 ? dv : 0.f;
                        dz = am == 4 ? -dv : am == 5 ? (P.force_down ? -dv : dv) : 0.f;
                    }
                } else {
                    float a0, a1, a2;
                    if (actions) {
                        const float* ap = reinterpret_cast<const float*>(actions) + 3 * off;
                        a0 = __ldg(ap); a1 = __ldg(ap + 1); a2 = __ldg(ap + 2);
                    } else {
                        a0 = (float)((double)ra.x * (2.0 / 4294967296.0) - 1.0);
                        a1 = (float)((double)ra.y * (2.0 / 4294967296.0) - 1.0);
                        a2 = (float)((double)ra.z * (2.0 / 4294967296.0) - 1.0);
                    }
                    const float dv = DELTA_V_CONTINUOUS + nz;
                    dx = a0 * dv; dy = a1 * dv;
                    dz = P.force_down ? -fabsf(a2 * dv) : a2 * dv;
                }
                e.total_steps += 1;
                if (P.moving_button) {
                    // kuka_moving_button_gym_env.py:109-119: bounce at the table edge, slide the target, teleport the button base
                    // to (button_pos - BUTTON_DISTANCE_HEIGHT): x, y follow the target, z becomes the button LINK height of reset
                    if (e.by64 > 0.3 || e.by64 < -0.3) e.bspeed = -e.bspeed;
                    e.by64 = __dadd_rn(e.by64, e.bspeed > 0.f ? 0.001 : -0.001);   // float64, like the reference's numpy array
                    e.tgt[1] = (float)e.by64;
                    e.bbx = e.tgt[0]; e.bby = e.tgt[1]; e.bbz = e.tgt[2] - P.target_h;
                }
            }
            armed = true;
        }
        // ---- applyAction + stepSimulation ----
        if (!JOINTS) apply_ee_delta(P, e, dx, dy, dz);
        saved_cb = new_cb; saved_ct = new_ct; saved_a0 = new_a0; saved_a1 = new_a1;
        if constexpr (TRACE) {
            // the configuration this micro-step starts from (the bodies see the arm where its own contacts are detected) and its kind
            if (lead) {
                int tag = 0;
                if (op == KUKA_OP_SETTLE) tag = 0;
                else if (in_reset) tag = DT_RESET | (reset_left == N_RANDOM_ACTIONS_AT_INIT - 1 ? DT_FIRST | (d17 ? DT_HOST_DRAWS : 0) : 0);
                else if (rep == 0 && e.counter == 10) tag = DT_KICK;
                const size_t base = (size_t)ms * 4 * N + (size_t)i;
                trace[base] = make_float4(e.q[0], e.q[1], e.q[2], e.q[3]);
                trace[base + N] = make_float4(e.q[4], e.q[5], e.q[6], e.q[7]);
                trace[base + 2 * N] = make_float4(e.q[8], e.q[9], e.q[10], e.q[11]);
                trace[base + 3 * N] = make_float4(e.qb, e.bbx, e.bby, __int_as_float(tag | (int)(e.episode << 4)));
            }
            ++ms;
        }
        KK_PH(ph, KK_PH_ENV);
#ifdef KK_PHASES
        ++kk_nphys;
#endif
#ifdef KK_TIMING
        kuka_physics_step<JOINTS, TWOB, COOP>(P, e, k, ct, armed, qj, sc, u, gmask, nc_reg, &dbgf, ph);
#else
        kuka_physics_step<JOINTS, TWOB, COOP>(P, e, k, ct, armed, qj, sc, u, gmask, nc_reg, nullptr, ph);
#endif
        if constexpr (PREFETCH) { if (helper && --budget <= 0 && reset_left > 0) { partial = true; KK_LEAVE_LOOP() } }
        if (!in_reset) {
            // step2()'s repeat loop (:349-354): stop repeating once terminated / past the step limit
            if (e.terminated || e.counter > P.max_steps) { pending = true; rep = 0; }
            else { e.counter += 1; if (++rep == P.action_repeat) { pending = true; rep = 0; } }
        }
    }
#undef KK_LEAVE_LOOP
    if (settled) return;
    if constexpr (!COOP) leave();
}

// Scene primitives of every env for srl_sim_render (render_core.h): one thread per env recomputes the joint frames of the stored
// configuration (the link states in HBM are only the two the env logic reads) and lists the primitives, then the env's distractor bodies
// when the handle has them (`bodies`: [N][DC_NBODY][DC_B_WORDS], written by distractor_kernel earlier on the same stream).
template <bool TWOB>
__global__ void kuka_prims_kernel(const __grid_constant__ KukaDev d, int n, const float* __restrict__ bodies, const __grid_constant__ SrlBodyLooks looks,
                                  float* __restrict__ prims, int* __restrict__ counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const KukaParams& P = d.P;
    KukaEnv e;
    env_load<TWOB>(d, i, e);
    // world rotations are needed for the sphere centres: rerun the chain with the rotations kept (12 bodies, negligible next to the ray-casting)
    float Rb[KK_NB][9]; f3 pb[KK_NB];
    kuka_world_frames(P, e.q, Rb, pb);
    float jp[KK_NB * 3], sph[KM_MAX_SPHERES * 4];
    for (int b = 0; b < KK_NB; ++b) { jp[3 * b] = pb[b].x; jp[3 * b + 1] = pb[b].y; jp[3 * b + 2] = pb[b].z; }
    int ns = 0;
    for (int sidx = 0; sidx < P.nsph; ++sidx) {
        const int b = P.sph_body[sidx];
        if (b < 7) continue;          // the arm links are drawn as capsules; the gripper bodies by their collision spheres
        const float* R = Rb[b];
        sph[4 * ns] = pb[b].x + R[0] * P.sph_c[sidx][0] + R[1] * P.sph_c[sidx][1] + R[2] * P.sph_c[sidx][2];
        sph[4 * ns + 1] = pb[b].y + R[3] * P.sph_c[sidx][0] + R[4] * P.sph_c[sidx][1] + R[5] * P.sph_c[sidx][2];
        sph[4 * ns + 2] = pb[b].z + R[6] * P.sph_c[sidx][0] + R[7] * P.sph_c[sidx][1] + R[8] * P.sph_c[sidx][2];
        sph[4 * ns + 3] = P.sph_r[sidx];
        ++ns;
    }
    SrlKukaSceneConst K;
    K.base[0] = P.base[0]; K.base[1] = P.base[1]; K.base[2] = P.base[2];
    K.table_z = P.table_z; K.txmin = P.txmin; K.txmax = P.txmax; K.tymin = P.tymin; K.tymax = P.tymax;
    K.glider_z = P.glider_z; K.disc_r = P.disc_r; K.disc_z0 = P.disc_z0; K.disc_z1 = P.disc_z1; K.stack_r = P.stack_r; K.stack_top = P.stack_top;
    K.two_buttons = TWOB ? 1 : 0;
    SrlPrim* out = reinterpret_cast<SrlPrim*>(prims + (size_t)i * SRL_MAX_PRIMS * SRL_PRIM_WORDS);
    int np = srl_kuka_scene(K, jp, sph, ns, e.bbx, e.bby, e.bbz, e.qb, e.bb2x, e.bb2y, P.btn_base[2], e.qb2, out);
    if (bodies) np = srl_distractor_prims(looks, bodies + (size_t)i * DC_NBODY * DC_B_WORDS, np, out);
    counts[i] = np;
}

// ---- host side -------------------------------------------------------------------------------
// the model part comes from kuka_params_from_blob (kuka_params.cuh); what depends on the env kind and srl_cfg is set here
bool fill_params(const void* blob, size_t bytes, const srl_sim* s, KukaParams& P) {
    const double* d = (const double*)blob;
    if (const char* err = kuka_params_from_blob(d, bytes, s->cfg.timestep, P)) { srl_set_error("%s", err); return false; }
    const double* sc = d + (int)d[KM_H_SCENE_OFF];
    P.iters = s->cfg.solver_iterations > 0 ? s->cfg.solver_iterations : (int)sc[KM_SC_SOLVER_ITERS];
    const bool two = s->kind == SRL_ENV_KUKA_2BUTTON;
    // small_constraints = not random_target (:239); Kuka2Button always uses the large box (kuka_2button_gym_env.py:78)
    const double* box = sc + ((s->cfg.random_target || two) ? KM_SC_BOX_LARGE : KM_SC_BOX_SMALL);
    for (int a = 0; a < 6; ++a) P.box[a] = (float)box[a];
    P.is_discrete = s->cfg.is_discrete; P.random_target = s->cfg.random_target; P.force_down = s->cfg.force_down;
    P.shape_reward = s->cfg.shape_reward; P.action_repeat = s->cfg.action_repeat; P.max_steps = s->max_steps;
    P.auto_reset = s->auto_reset; P.max_distance = s->cfg.max_distance;
    P.moving_button = s->kind == SRL_ENV_KUKA_MOVING_BUTTON;
    P.action_joints = s->cfg.action_joints != 0;
    P.two_buttons = two;
    if (two) {
        P.btn_base[1] = 0.125f;                               // kuka_2button_gym_env.py:49-57 (button 2 mirrors it at -0.125)
        // `use_null_space = True` (:80) -> calculateInverseKinematics(uid, link, pos, orn, ll, ul, jr, rp) (kuka.py:147-149).  RECALLED
        // pybullet 1.8.6 behaviour: the null-space task needs one list entry per JOINT (14; kuka.py:34-40 gives 7) and is dropped,
        // and without a jointDamping argument the server's default damping 0.5 per DoF applies (DESIGN.md section 4)
        P.ik_damp = 0.5;
    }
    P.seed = s->seed; P.env_offset = s->cfg.global_env_offset;
    return true;
}

int alloc_state(KukaState& a, size_t N) {
    float4** f4[] = {&a.q[0], &a.q[1], &a.q[2], &a.qd[0], &a.qd[1], &a.qd[2], &a.misc0, &a.misc1, &a.tgt, &a.grip, &a.eepos, &a.btn2};
    for (float4** p : f4) { SRL_CUDA_OK(cudaMalloc(p, N * sizeof(float4))); SRL_CUDA_OK(cudaMemset(*p, 0, N * sizeof(float4))); }
    int4** i4[] = {&a.cnt, &a.cnt2};
    for (int4** p : i4) { SRL_CUDA_OK(cudaMalloc(p, N * sizeof(int4))); SRL_CUDA_OK(cudaMemset(*p, 0, N * sizeof(int4))); }
    return 0;
}

void free_state(KukaState& a) {
    for (int k = 0; k < 3; ++k) { cudaFree(a.q[k]); cudaFree(a.qd[k]); }
    cudaFree(a.misc0); cudaFree(a.misc1); cudaFree(a.tgt); cudaFree(a.grip); cudaFree(a.eepos); cudaFree(a.cnt); cudaFree(a.cnt2); cudaFree(a.btn2);
}

#define KUKA_SMEM_BYTES ((size_t)(((KC_CONST_WORDS + 31) / 32) * 32 + 32 * KC_ES) * sizeof(float))   /* 4 warps x 8 env slots */
template <bool J, bool T2, bool PF, bool CO, bool TR>
cudaError_t kuka_launch_inst(const KukaDev& d, const KukaNext& nx, int grid, int block, cudaStream_t st, int n, int op, int T, const void* actions,
                             const float* noise, const uint8_t* mask, const double* draws, float* obs, float* rew, uint8_t* done, float* ep_ret,
                             int32_t* ep_len, float* snap, float4* trace, int* trace_len) {
    const size_t smem = CO ? KUKA_SMEM_BYTES : 0;
    if constexpr (CO) { if (const cudaError_t e = srl_smem_opt_in<kuka_kernel<J, T2, PF, CO, TR>>(smem)) return e; }
    kuka_kernel<J, T2, PF, CO, TR><<<grid, block, smem, st>>>(d, n, op, T, actions, noise, mask, draws, obs, rew, done, ep_ret, ep_len, snap, nx,
                                                              trace, trace_len);
    return cudaGetLastError();
}

// One instantiation per (action_joints, two_buttons, four lanes per env) at inst[action_joints | two_buttons << 1 | coop << 2]: the default
// kernel pays nothing for the variants.  With a trace (distractor bodies: single button, no records; `trace_len` null for the settle) the
// TRACE one at inst[8 + (action_joints | coop << 1)]; with next-episode records (`nx`, single-button IK kinds) PREFETCH at inst[12 + coop].
cudaError_t kuka_launch(const KukaDev& d, const KukaNext* nx, int grid, int block, cudaStream_t st, int n, int op, int T, const void* actions,
                        const float* noise, const uint8_t* mask, const double* draws, float* obs, float* rew, uint8_t* done, float* ep_ret,
                        int32_t* ep_len, float* snap, float4* trace = nullptr, int* trace_len = nullptr) {
    using Launch = decltype(&kuka_launch_inst<false, false, false, false, false>);
    static const Launch inst[14] = {kuka_launch_inst<false, false, false, false, false>, kuka_launch_inst<true, false, false, false, false>,
                                    kuka_launch_inst<false, true, false, false, false>,  kuka_launch_inst<true, true, false, false, false>,
                                    kuka_launch_inst<false, false, false, true, false>,  kuka_launch_inst<true, false, false, true, false>,
                                    kuka_launch_inst<false, true, false, true, false>,   kuka_launch_inst<true, true, false, true, false>,
                                    kuka_launch_inst<false, false, false, false, true>,  kuka_launch_inst<true, false, false, false, true>,
                                    kuka_launch_inst<false, false, false, true, true>,   kuka_launch_inst<true, false, false, true, true>,
                                    kuka_launch_inst<false, false, true, false, false>,  kuka_launch_inst<false, false, true, true, false>};
    const int j = d.P.action_joints ? 1 : 0, co = d.coop ? 1 : 0;
    const Launch launch = nx ? inst[12 + co] : trace ? inst[8 + (j | co << 1)] : inst[j | (d.P.two_buttons ? 2 : 0) | co << 2];
    return launch(d, nx ? *nx : KukaNext{}, grid, block, st, n, op, T, actions, noise, mask, draws, obs, rew, done, ep_ret, ep_len, snap,
                  trace, trace_len);
}

void grid_for(const srl_sim* s, int& grid, int& block) {
    const int warps = (s->n + s->kuka->epw - 1) / s->kuka->epw;
    block = 128;
    grid = (warps * 32 + block - 1) / block;
}

// The 500 zero-action settle steps of reset() for one env, from resetJointState at the initial joint vector: h[0..28] = the reset
// snapshot (q, qd, commanded end effector, glider q, qd).  With `trace`, the traced instantiation also records the arm's trajectory.
int settle(srl_sim* s, float4* trace, float* h) {
    KukaDev one = *s->kuka;
    one.epw = 1;
    for (int k = 0; k < KK_NB; ++k) one.P.snap_q[k] = s->kuka_q0[k];
    float* snap = nullptr;
    SRL_CUDA_OK(cudaMalloc(&snap, 32 * sizeof(float)));
    SRL_CUDA_OK(kuka_launch(one, nullptr, 1, 32, 0, 1, KUKA_OP_SETTLE, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                            nullptr, snap, trace, nullptr));
    SRL_CUDA_OK(cudaMemcpy(h, snap, 29 * sizeof(float), cudaMemcpyDeviceToHost));
    cudaFree(snap);
    return 0;
}

}  // namespace

int kuka_alloc(srl_sim* s, const void* blob, size_t bytes) {
    KukaDev* d = new KukaDev();
    memset(d, 0, sizeof(*d));
    s->kuka = d;
    if (!fill_params(blob, bytes, s, d->P)) return 1;
    const size_t N = (size_t)s->n;
    if (alloc_state(*d, N)) return 1;
    // live lanes per warp: spread a small batch over every warp scheduler (4 per SM), ONE warp each -- the PGS
    // sweep of a single warp already fills its scheduler's issue slots, a second resident warp only adds latency
    const int sms = s->sms;
    int epw = s->cfg.envs_per_warp;
    const bool auto_epw = epw <= 0;
    if (auto_epw) { epw = (int)((N + (size_t)sms * 4 - 1) / ((size_t)sms * 4)); }
    if (epw < 1) epw = 1;
    if (epw > 32) epw = 32;
    // next-episode records are produced by the first idle slot of every warp (kuka_kernel), so a batch that would fill its warps
    // (8 groups of 4 lanes, or 32 lanes: 4096 envs on the 132 SMs of an H100) is spread one env per warp thinner
    const bool records = s->cfg.prefetch_resets && s->auto_reset && !d->P.two_buttons && !d->P.action_joints;
    if (auto_epw && records && (epw == 8 || epw == 32)) epw -= 1;
    d->epw = epw;
    // four lanes per env while a warp carries at most 8 envs (the whole batch still fits one warp per scheduler)
    d->coop = epw <= 8 ? 1 : 0;
    // the 500 settle steps of reset(), once
    for (int k = 0; k < KK_NB; ++k) s->kuka_q0[k] = d->P.snap_q[k];
    float h[29];
    if (settle(s, nullptr, h)) return 1;
    for (int i = 0; i < KK_NB; ++i) { d->P.snap_q[i] = h[i]; d->P.snap_qd[i] = h[KK_NB + i]; }
    d->P.snap_ee[0] = h[24]; d->P.snap_ee[1] = h[25]; d->P.snap_ee[2] = h[26]; d->P.snap_qb = h[27]; d->P.snap_qdb = h[28];
    s->launches += 1;
    // opt-in next-episode records (single-button kinds with IK actions and auto-reset: the instantiation that exists)
    if (records) {
        KukaNext* nx = new KukaNext();
        memset(nx, 0, sizeof(*nx));
        s->kuka_next = nx;
        if (alloc_state(*nx, N)) return 1;
        SRL_CUDA_OK(cudaMalloc(&nx->valid, N)); SRL_CUDA_OK(cudaMemset(nx->valid, 0, N));
        SRL_CUDA_OK(cudaMalloc(&nx->episode, N * sizeof(int32_t))); SRL_CUDA_OK(cudaMemset(nx->episode, 0xff, N * sizeof(int32_t)));
        SRL_CUDA_OK(cudaMalloc(&nx->progress, N)); SRL_CUDA_OK(cudaMemset(nx->progress, 0, N));
        SRL_CUDA_OK(cudaEventCreateWithFlags(&s->pf_ev, cudaEventDisableTiming));
        SRL_CUDA_OK(cudaEventCreateWithFlags(&s->roll_ev, cudaEventDisableTiming));
    }
    return 0;
}

void kuka_free(srl_sim* s) {
    KukaDev* d = s->kuka;
    if (!d) return;
    dist_free(s);
    free_state(*d);
    delete d;
    s->kuka = nullptr;
    if (KukaNext* nx = s->kuka_next) {
        free_state(*nx);
        cudaFree(nx->valid); cudaFree(nx->episode); cudaFree(nx->progress);
        delete nx;
        s->kuka_next = nullptr;
        if (s->pf_ev) cudaEventDestroy(s->pf_ev);
        if (s->roll_ev) cudaEventDestroy(s->roll_ev);
    }
}

int kuka_launch_reset(srl_sim* s, const uint8_t* mask, const double* draws, float* obs, cudaStream_t st) {
    s->kuka_started = true;
    float4* trace = nullptr; int* trace_len = nullptr;
    if (s->dist && dist_trace(s, N_RANDOM_ACTIONS_AT_INIT, st, &trace, &trace_len)) return 1;
    int grid, block; grid_for(s, grid, block);
    SRL_CUDA_OK(kuka_launch(*s->kuka, nullptr, grid, block, st, s->n, KUKA_OP_RESET, 0, nullptr, nullptr, mask, draws, obs, nullptr, nullptr, nullptr, nullptr,
                            nullptr, trace, trace_len));
    return s->dist ? dist_advance(s, draws, st) : 0;
}

int kuka_launch_rollout(srl_sim* s, int T, const void* actions, const float* noise, float* obs, float* rew, uint8_t* done,
                        float* ep_ret, int32_t* ep_len, cudaStream_t st) {
    s->kuka_started = true;
    float4* trace = nullptr; int* trace_len = nullptr;
    // an env step is at most action_repeat micro-steps, a reset() inside the launch 5 more
    if (s->dist && dist_trace(s, (size_t)T * (size_t)(s->cfg.action_repeat + N_RANDOM_ACTIONS_AT_INIT), st, &trace, &trace_len)) return 1;
    int grid, block; grid_for(s, grid, block);
    KukaNext nx{};
    bool capturing = false;
    if (s->kuka_next) {         // the rollout path that takes a ready next-episode record instead of resetting inside the launch
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        cudaStreamIsCapturing(st, &cap);
        capturing = cap != cudaStreamCaptureStatusNone;   // events recorded outside a capture cannot be waited for inside it
        if (s->pf_pending && !capturing) { SRL_CUDA_OK(cudaStreamWaitEvent(st, s->pf_ev, 0)); s->pf_pending = false; }
        nx = *s->kuka_next;
        nx.helper = 1;          // the first idle slot of every warp advances one incomplete record of its warp's envs by up to T micro-steps
    }
    SRL_CUDA_OK(kuka_launch(*s->kuka, s->kuka_next ? &nx : nullptr, grid, block, st, s->n, KUKA_OP_ROLLOUT, T, actions, noise, nullptr, nullptr, obs, rew, done,
                            ep_ret, ep_len, nullptr, trace, trace_len));
    if (s->kuka_next && !capturing) { SRL_CUDA_OK(cudaEventRecord(s->roll_ev, st)); s->roll_ev_valid = true; }
    return s->dist ? dist_advance(s, nullptr, st) : 0;
}

// Refresh the next-episode records of the envs that consumed theirs (or never had one).  Asynchronous on `st`; meant for a side stream, it may
// run concurrently with step / rollout launches of the same handle (flag + fence hand-over, see KukaNext).  A no-op when the feature is off.
int kuka_launch_prefetch(srl_sim* s, cudaStream_t st) {
    if (!s->kuka_next) return 0;
    int grid, block; grid_for(s, grid, block);
    // never concurrent with a rollout launch of the handle: its idle slots advance the same records
    if (s->roll_ev_valid) SRL_CUDA_OK(cudaStreamWaitEvent(st, s->roll_ev, 0));
    SRL_CUDA_OK(kuka_launch(*s->kuka, s->kuka_next, grid, block, st, s->n, KUKA_OP_PREFETCH, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr));
    SRL_CUDA_OK(cudaEventRecord(s->pf_ev, st));
    s->pf_pending = true;
    s->launches += 1;
    return 0;
}

int kuka_set_distractors(srl_sim* s, const void* blob, size_t bytes) {
    float4* trajectory = nullptr;
    if (dist_alloc(s, blob, bytes, &trajectory)) return 1;
    // the arm's settle trajectory: the settle launch of kuka_alloc again, traced (the same instructions, so the same trajectory)
    float h[29];
    if (settle(s, trajectory, h)) return 1;
    // the traced settle must be the trajectory kuka_alloc's settle produced: its end state is the reset snapshot, bit for bit
    const KukaDev* d = s->kuka;
    bool same = memcmp(h + 27, &d->P.snap_qb, sizeof(float)) == 0 && memcmp(h + 28, &d->P.snap_qdb, sizeof(float)) == 0;
    for (int k = 0; k < KK_NB; ++k) same = same && memcmp(h + k, &d->P.snap_q[k], sizeof(float)) == 0 && memcmp(h + KK_NB + k, &d->P.snap_qd[k], sizeof(float)) == 0;
    if (!same) { srl_set_error("set_distractors: the traced settle does not reproduce the reset snapshot"); return 1; }
    s->launches += 1;
    return 0;
}

int kuka_render_prims(srl_sim* s, float* prims, int* counts, cudaStream_t st) {
    KukaDev* d = s->kuka;
    const int grid = (s->n + 63) / 64;
    SrlBodyLooks looks = {};
    const float* bodies = dist_render_bodies(s, &looks);
    if (d->P.two_buttons) kuka_prims_kernel<true><<<grid, 64, 0, st>>>(*d, s->n, bodies, looks, prims, counts);
    else kuka_prims_kernel<false><<<grid, 64, 0, st>>>(*d, s->n, bodies, looks, prims, counts);
    SRL_CUDA_OK(cudaGetLastError());
    return 0;
}

int kuka_get_state(srl_sim* s, int field, void* dst, size_t bytes) {
    KukaDev* d = s->kuka;
    const size_t N = (size_t)s->n;
    SRL_CUDA_OK(cudaDeviceSynchronize());
    auto need = [&](size_t width, size_t elem) { if (bytes != N * width * elem) { srl_set_error("get_state: size mismatch"); return false; } return true; };
    std::vector<float4> a(N), b(N), c(N);
    std::vector<int4> ia(N);
    double* D = (double*)dst; int32_t* I = (int32_t*)dst;
    auto pull = [&](std::vector<float4>& v, const float4* src) { return cudaMemcpy(v.data(), src, N * sizeof(float4), cudaMemcpyDeviceToHost); };
    switch (field) {
    case SRL_F_ROBOT_POS: case SRL_F_TARGET_POS: case SRL_F_EE_POS: {
        if (!need(3, 8)) return 1;
        SRL_CUDA_OK(pull(a, field == SRL_F_ROBOT_POS ? d->grip : field == SRL_F_TARGET_POS ? d->tgt : d->eepos));
        for (size_t i = 0; i < N; ++i) { D[3 * i] = a[i].x; D[3 * i + 1] = a[i].y; D[3 * i + 2] = a[i].z; }
        return 0;
    }
    case SRL_F_JOINT_POS: case SRL_F_JOINT_VEL: {
        if (!need(KK_NB, 8)) return 1;
        float4* const* src = field == SRL_F_JOINT_POS ? d->q : d->qd;
        SRL_CUDA_OK(pull(a, src[0])); SRL_CUDA_OK(pull(b, src[1])); SRL_CUDA_OK(pull(c, src[2]));
        for (size_t i = 0; i < N; ++i) {
            const float4 v[3] = {a[i], b[i], c[i]};
            for (int k = 0; k < 3; ++k) { D[12 * i + 4 * k] = v[k].x; D[12 * i + 4 * k + 1] = v[k].y; D[12 * i + 4 * k + 2] = v[k].z; D[12 * i + 4 * k + 3] = v[k].w; }
        }
        return 0;
    }
    case SRL_F_EE_CMD:
        if (!need(3, 8)) return 1;
        SRL_CUDA_OK(pull(a, d->misc0));
        for (size_t i = 0; i < N; ++i) { D[3 * i] = a[i].x; D[3 * i + 1] = a[i].y; D[3 * i + 2] = a[i].z; }
        return 0;
    case SRL_F_BUTTON_GLIDER:
        if (!need(2, 8)) return 1;
        SRL_CUDA_OK(pull(a, d->misc0)); SRL_CUDA_OK(pull(b, d->misc1));
        for (size_t i = 0; i < N; ++i) { D[2 * i] = a[i].w; D[2 * i + 1] = b[i].x; }
        return 0;
    case SRL_F_BUTTON_BASE:
        if (!need(3, 8)) return 1;
        SRL_CUDA_OK(pull(b, d->misc1));
        SRL_CUDA_OK(pull(a, d->tgt));
        for (size_t i = 0; i < N; ++i) { D[3 * i] = b[i].y; D[3 * i + 1] = b[i].z; D[3 * i + 2] = a[i].w; }
        return 0;
    case SRL_F_STEP_COUNTER:
        if (!need(1, 4)) return 1;
        SRL_CUDA_OK(cudaMemcpy(ia.data(), d->cnt, N * sizeof(int4), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < N; ++i) I[i] = ia[i].x;
        return 0;
    case SRL_F_COUNTERS: {
        if (!need(4, 4)) return 1;
        std::vector<int4> ib(N);
        SRL_CUDA_OK(cudaMemcpy(ia.data(), d->cnt, N * sizeof(int4), cudaMemcpyDeviceToHost));
        SRL_CUDA_OK(cudaMemcpy(ib.data(), d->cnt2, N * sizeof(int4), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < N; ++i) { I[4 * i] = ia[i].y; I[4 * i + 1] = ia[i].z; I[4 * i + 2] = ia[i].w & 1; I[4 * i + 3] = ib[i].x; }
        return 0;
    }
    case SRL_F_TWO_BUTTON: {
        if (!need(8, 8)) return 1;
        std::vector<int4> ib(N);
        SRL_CUDA_OK(pull(a, d->btn2));
        SRL_CUDA_OK(cudaMemcpy(ia.data(), d->cnt, N * sizeof(int4), cudaMemcpyDeviceToHost));
        SRL_CUDA_OK(cudaMemcpy(ib.data(), d->cnt2, N * sizeof(int4), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < N; ++i) {
            D[8 * i] = d->P.two_buttons ? ia[i].y : 0; D[8 * i + 1] = d->P.two_buttons ? ib[i].w : 0; D[8 * i + 2] = (ia[i].w >> 5) & 1;
            D[8 * i + 3] = a[i].z; D[8 * i + 4] = a[i].w; D[8 * i + 5] = d->P.btn_base[2]; D[8 * i + 6] = a[i].x; D[8 * i + 7] = a[i].y;
        }
        return 0;
    }
    case SRL_F_EPISODE_STATS: {
        if (!need(2, 8)) return 1;
        SRL_CUDA_OK(pull(b, d->misc1));
        SRL_CUDA_OK(cudaMemcpy(ia.data(), d->cnt2, N * sizeof(int4), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < N; ++i) { D[2 * i] = b[i].w; D[2 * i + 1] = (double)ia[i].z; }
        return 0;
    }
#ifdef KK_TIMING
    case 99: {   // diagnostic build: the per-slot timing words of the last launch
        if (cudaMemcpyFromSymbol(dst, kk_timing, bytes < sizeof(kk_timing) ? bytes : sizeof(kk_timing)) != cudaSuccess) return 1;
        return 0;
    }
#endif
#ifdef KK_PHASES
    case 98: {   // diagnostic build: the per-slot phase cycles of the last launch, [slot][KK_NPH + 2]
        if (cudaMemcpyFromSymbol(dst, kk_phase, bytes < sizeof(kk_phase) ? bytes : sizeof(kk_phase)) != cudaSuccess) return 1;
        return 0;
    }
#endif
    case SRL_F_DISTRACTORS: case SRL_F_DISTRACTOR_TOUCH:
    case SRL_F_DISTRACTOR_RECORDS: case SRL_F_DISTRACTOR_TRACE_LEN: case SRL_F_DISTRACTOR_TRACE: case SRL_F_DISTRACTOR_SETTLE:
        return dist_get_state(s, field, dst, bytes);
    case SRL_F_NEXT_RECORD: {
        if (!need(3, 4)) return 1;
        const KukaNext* nx = s->kuka_next;
        for (size_t i = 0; i < N; ++i) { I[3 * i] = 0; I[3 * i + 1] = 0; I[3 * i + 2] = -1; }
        if (nx) {
            std::vector<uint8_t> va(N), pr(N); std::vector<int32_t> ep(N);
            SRL_CUDA_OK(cudaMemcpy(va.data(), nx->valid, N, cudaMemcpyDeviceToHost));
            SRL_CUDA_OK(cudaMemcpy(pr.data(), nx->progress, N, cudaMemcpyDeviceToHost));
            SRL_CUDA_OK(cudaMemcpy(ep.data(), nx->episode, N * sizeof(int32_t), cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < N; ++i) { I[3 * i] = va[i]; I[3 * i + 1] = pr[i]; I[3 * i + 2] = ep[i]; }
        }
        return 0;
    }
    default:
        srl_set_error("get_state: unknown field %d", field);
        return 1;
    }
}

int kuka_set_state(srl_sim* s, int field, const void* src, size_t bytes) {
    KukaDev* d = s->kuka;
    const size_t N = (size_t)s->n;
    SRL_CUDA_OK(cudaDeviceSynchronize());
    auto need = [&](size_t width, size_t elem) { if (bytes != N * width * elem) { srl_set_error("set_state: size mismatch"); return false; } return true; };
    const double* D = (const double*)src; const int32_t* I = (const int32_t*)src;
    std::vector<float4> a(N), b(N), c(N);
    auto pull = [&](std::vector<float4>& v, const float4* p) { return cudaMemcpy(v.data(), p, N * sizeof(float4), cudaMemcpyDeviceToHost); };
    auto push = [&](const std::vector<float4>& v, float4* p) { return cudaMemcpy(p, v.data(), N * sizeof(float4), cudaMemcpyHostToDevice); };
    switch (field) {
    case SRL_F_JOINT_POS: case SRL_F_JOINT_VEL: {
        if (!need(KK_NB, 8)) return 1;
        float4* const* dst = field == SRL_F_JOINT_POS ? d->q : d->qd;
        for (size_t i = 0; i < N; ++i) {
            a[i] = make_float4((float)D[12 * i], (float)D[12 * i + 1], (float)D[12 * i + 2], (float)D[12 * i + 3]);
            b[i] = make_float4((float)D[12 * i + 4], (float)D[12 * i + 5], (float)D[12 * i + 6], (float)D[12 * i + 7]);
            c[i] = make_float4((float)D[12 * i + 8], (float)D[12 * i + 9], (float)D[12 * i + 10], (float)D[12 * i + 11]);
        }
        SRL_CUDA_OK(push(a, dst[0])); SRL_CUDA_OK(push(b, dst[1])); SRL_CUDA_OK(push(c, dst[2]));
        return 0;
    }
    case SRL_F_EE_CMD:
        if (!need(3, 8)) return 1;
        SRL_CUDA_OK(pull(a, d->misc0));
        for (size_t i = 0; i < N; ++i) { a[i].x = (float)D[3 * i]; a[i].y = (float)D[3 * i + 1]; a[i].z = (float)D[3 * i + 2]; }
        SRL_CUDA_OK(push(a, d->misc0));
        return 0;
    case SRL_F_TARGET_POS:
        if (!need(3, 8)) return 1;
        SRL_CUDA_OK(pull(a, d->tgt));
        for (size_t i = 0; i < N; ++i) { a[i].x = (float)D[3 * i]; a[i].y = (float)D[3 * i + 1]; a[i].z = (float)D[3 * i + 2]; }
        SRL_CUDA_OK(push(a, d->tgt));
        return 0;
    case SRL_F_BUTTON_GLIDER:
        if (!need(2, 8)) return 1;
        SRL_CUDA_OK(pull(a, d->misc0)); SRL_CUDA_OK(pull(b, d->misc1));
        for (size_t i = 0; i < N; ++i) { a[i].w = (float)D[2 * i]; b[i].x = (float)D[2 * i + 1]; }
        SRL_CUDA_OK(push(a, d->misc0)); SRL_CUDA_OK(push(b, d->misc1));
        return 0;
    case SRL_F_BUTTON_BASE:
        if (!need(3, 8)) return 1;
        SRL_CUDA_OK(pull(b, d->misc1));
        for (size_t i = 0; i < N; ++i) { b[i].y = (float)D[3 * i]; b[i].z = (float)D[3 * i + 1]; }
        SRL_CUDA_OK(push(b, d->misc1));
        return 0;
    case SRL_F_STEP_COUNTER: case SRL_F_COUNTERS: {
        if (!need(field == SRL_F_STEP_COUNTER ? 1 : 4, 4)) return 1;
        std::vector<int4> ia(N);
        SRL_CUDA_OK(cudaMemcpy(ia.data(), d->cnt, N * sizeof(int4), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < N; ++i) {
            if (field == SRL_F_STEP_COUNTER) ia[i].x = I[i];
            else { ia[i].y = I[4 * i]; ia[i].z = I[4 * i + 1]; ia[i].w = (ia[i].w & ~1) | (I[4 * i + 2] & 1); }
        }
        SRL_CUDA_OK(cudaMemcpy(d->cnt, ia.data(), N * sizeof(int4), cudaMemcpyHostToDevice));
        return 0;
    }
    case SRL_F_DISTRACTOR_RECORDS:
        return dist_set_state(s, src, bytes);
    default:
        srl_set_error("set_state: field %d not settable", field);
        return 1;
    }
}
