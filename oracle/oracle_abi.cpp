/*
 * ORACLE (test infrastructure, not product code) -- the C-ABI of include/srl_sim.h implemented
 * on the host in double precision (device must be -1, all pointers are host pointers).
 * Lockstep semantics mirror the SubprocVecEnv worker loop the reference uses
 * (rl_baselines/utils.py:216-220): step every env, auto-reset the finished ones.
 */
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <new>
#include "oracle_sim.h"

static thread_local char g_err[512] = "";

void oracle_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

static bool is_mobile(int kind) { return kind >= SRL_ENV_MOBILE && kind <= SRL_ENV_MOBILE_LINE_TARGET; }
static bool is_kuka(int kind) { return kind >= SRL_ENV_KUKA_BUTTON && kind <= SRL_ENV_KUKA_MOVING_BUTTON; }

extern "C" {

int srl_sim_abi_version(void) { return SRL_SIM_ABI_VERSION; }
const char* srl_sim_last_error(void) { return g_err; }

int srl_sim_create(srl_sim** out, int env_kind, int num_envs, int device, const srl_cfg* cfg,
                   const void* model_blob, size_t model_bytes, uint64_t seed) {
    if (!out || !cfg) { oracle_set_error("create: null argument"); return 1; }
    *out = NULL;
    if (cfg->struct_size != sizeof(srl_cfg)) { oracle_set_error("create: srl_cfg size mismatch (%u != %zu)", cfg->struct_size, sizeof(srl_cfg)); return 1; }
    if (device != -1) { oracle_set_error("create: the oracle library only supports device=-1"); return 1; }
    if (num_envs <= 0) { oracle_set_error("create: num_envs must be positive"); return 1; }
    if (!is_mobile(env_kind) && !is_kuka(env_kind)) { oracle_set_error("create: unknown env kind %d", env_kind); return 1; }
    if (cfg->action_joints && (!is_kuka(env_kind) || cfg->is_discrete)) {
        /* kuka_button_gym_env.py:149-161: the (7,) joint action space only exists for continuous Kuka actions */
        oracle_set_error("create: action_joints needs a Kuka env with is_discrete=0"); return 1;
    }
    if (is_mobile(env_kind) && !cfg->is_discrete && env_kind != SRL_ENV_MOBILE && env_kind != SRL_ENV_MOBILE_LINE_TARGET) {
        /* mobile_robot_2target_env.py:128, mobile_robot_1D_env.py:43,118: ValueError */
        oracle_set_error("Only discrete actions is supported");
        return 2;
    }
    srl_sim* s = new (std::nothrow) srl_sim();
    if (!s) { oracle_set_error("create: out of memory"); return 1; }
    s->kind = env_kind;
    s->n = num_envs;
    s->cfg = *cfg;
    if (s->cfg.action_repeat < 1) s->cfg.action_repeat = 1;
    s->seed = seed;
    s->auto_reset = !cfg->no_auto_reset;
    s->kuka = NULL;
    s->launches = 0;
    if (is_mobile(env_kind)) {
        s->mobile.resize(num_envs);
        memset(s->mobile.data(), 0, sizeof(MobileEnv) * (size_t)num_envs);
    } else {
        s->kuka = oracle_kuka_create(s, model_blob, model_bytes);
        if (!s->kuka) { delete s; return 1; }
    }
    *out = s;
    return 0;
}

void srl_sim_destroy(srl_sim* s) {
    if (!s) return;
    if (s->kuka) oracle_kuka_destroy(s->kuka);
    delete s;
}

int srl_sim_num_envs(const srl_sim* s) { return s ? s->n : 0; }
int srl_sim_obs_dim(const srl_sim* s) { return !s ? 0 : is_mobile(s->kind) ? oracle_mobile_obs_dim(s->kind) : 3; }
int srl_sim_action_dim(const srl_sim* s) {
    if (!s) return 0;
    if (s->cfg.is_discrete) return 1;
    return is_mobile(s->kind) ? 2 : (s->cfg.action_joints ? 7 : 3);
}
uint64_t srl_sim_launch_count(const srl_sim* s) { return s ? s->launches : 0; }
float srl_sim_last_kernel_ms(srl_sim*) { return -1.0f; }

int srl_sim_reset(srl_sim* s, const uint8_t* mask, const double* reset_draws, float* obs_out, void*) {
    if (!s) { oracle_set_error("reset: null handle"); return 1; }
    const int D = srl_sim_obs_dim(s);
    const int R = is_mobile(s->kind) ? 6 : 18;
    for (int i = 0; i < s->n; ++i) {
        if (mask && !mask[i]) continue;
        const double* d = reset_draws ? reset_draws + (size_t)i * R : NULL;
        if (is_mobile(s->kind)) {
            oracle_mobile_reset_env(s, i, d);
            if (obs_out) oracle_mobile_obs(s, i, obs_out + (size_t)i * D);
        } else {
            oracle_kuka_reset_env(s, i, d);
            if (obs_out) oracle_kuka_obs(s, i, obs_out + (size_t)i * D);
        }
    }
    return 0;
}

int srl_sim_step(srl_sim* s, const void* actions, const float* noise, float* obs_out, float* rew_out,
                 uint8_t* done_out, float* ep_ret_out, int32_t* ep_len_out, void*) {
    if (!s) { oracle_set_error("step: null handle"); return 1; }
    for (int i = 0; i < s->n; ++i) {
        if (is_mobile(s->kind))
            oracle_mobile_step_env(s, i, actions, noise, obs_out, rew_out, done_out, ep_ret_out, ep_len_out);
        else
            oracle_kuka_step_env(s, i, actions, noise, obs_out, rew_out, done_out, ep_ret_out, ep_len_out);
    }
    s->launches += 1;
    return 0;
}

int srl_sim_rollout(srl_sim* s, int T, const void* actions, const float* noise, float* obs_out,
                    float* rew_out, uint8_t* done_out, float* ep_ret_out, int32_t* ep_len_out, void* stream) {
    if (!s) { oracle_set_error("rollout: null handle"); return 1; }
    if (T < 0) { oracle_set_error("rollout: negative T"); return 1; }
    const size_t N = (size_t)s->n;
    const size_t D = (size_t)srl_sim_obs_dim(s);
    const size_t A = (size_t)srl_sim_action_dim(s);
    for (int t = 0; t < T; ++t) {
        const void* a = NULL;
        if (actions) a = s->cfg.is_discrete ? (const void*)((const int32_t*)actions + (size_t)t * N)
                                            : (const void*)((const float*)actions + (size_t)t * N * A);
        int rc = srl_sim_step(s, a, noise ? noise + (size_t)t * N : NULL,
                              obs_out ? obs_out + (size_t)t * N * D : NULL,
                              rew_out ? rew_out + (size_t)t * N : NULL,
                              done_out ? done_out + (size_t)t * N : NULL,
                              ep_ret_out ? ep_ret_out + (size_t)t * N : NULL,
                              ep_len_out ? ep_len_out + (size_t)t * N : NULL, stream);
        if (rc) return rc;
    }
    return 0;
}

/* The CPU oracle resets inside the step (there is no launch whose latency a ready record could shorten): the entry point exists so that
 * both libraries export the same symbols; srl_cfg.prefetch_resets is ignored here, which is the behaviour the CUDA library must reproduce. */
int srl_sim_prefetch_resets(srl_sim* s, void* stream) {
    (void)stream;
    if (!s) { oracle_set_error("prefetch_resets: null handle"); return 1; }
    return 0;
}

int srl_sim_rollout_host(srl_sim* s, int T, const void* actions, const float* noise, float* obs_out,
                         float* rew_out, uint8_t* done_out) {
    return srl_sim_rollout(s, T, actions, noise, obs_out, rew_out, done_out, NULL, NULL, NULL);
}

static int mobile_get_state(srl_sim* s, int field, void* dst, size_t bytes) {
    const size_t N = (size_t)s->n;
    switch (field) {
    case SRL_F_ROBOT_POS:
    case SRL_F_TARGET_POS: {
        if (bytes != N * 3 * sizeof(double)) { oracle_set_error("get_state: size mismatch"); return 1; }
        double* o = (double*)dst;
        for (size_t i = 0; i < N; ++i) {
            const MobileEnv& e = s->mobile[i];
            const double* src = field == SRL_F_ROBOT_POS ? e.pos : e.target[e.current_target];
            o[3 * i] = src[0]; o[3 * i + 1] = src[1]; o[3 * i + 2] = src[2];
        }
        return 0;
    }
    case SRL_F_STEP_COUNTER: {
        if (bytes != N * sizeof(int32_t)) { oracle_set_error("get_state: size mismatch"); return 1; }
        for (size_t i = 0; i < N; ++i) ((int32_t*)dst)[i] = s->mobile[i].counter;
        return 0;
    }
    case SRL_F_COUNTERS: {
        if (bytes != N * 4 * sizeof(int32_t)) { oracle_set_error("get_state: size mismatch"); return 1; }
        for (size_t i = 0; i < N; ++i) {
            int32_t* o = (int32_t*)dst + 4 * i;
            o[0] = s->mobile[i].current_target; o[1] = s->mobile[i].has_bumped; o[2] = 0;
            o[3] = (int32_t)s->mobile[i].episode;
        }
        return 0;
    }
    case SRL_F_EPISODE_STATS: {
        if (bytes != N * 2 * sizeof(double)) { oracle_set_error("get_state: size mismatch"); return 1; }
        for (size_t i = 0; i < N; ++i) {
            ((double*)dst)[2 * i] = s->mobile[i].ep_ret;
            ((double*)dst)[2 * i + 1] = (double)s->mobile[i].ep_len;
        }
        return 0;
    }
    default:
        oracle_set_error("get_state: field %d not available for MobileRobot", field);
        return 1;
    }
}

static int mobile_set_state(srl_sim* s, int field, const void* src, size_t bytes) {
    const size_t N = (size_t)s->n;
    switch (field) {
    case SRL_F_ROBOT_POS:
    case SRL_F_TARGET_POS: {
        if (bytes != N * 3 * sizeof(double)) { oracle_set_error("set_state: size mismatch"); return 1; }
        const double* in = (const double*)src;
        for (size_t i = 0; i < N; ++i) {
            MobileEnv& e = s->mobile[i];
            double* d = field == SRL_F_ROBOT_POS ? e.pos : e.target[e.current_target];
            d[0] = in[3 * i]; d[1] = in[3 * i + 1]; d[2] = in[3 * i + 2];
        }
        return 0;
    }
    case SRL_F_STEP_COUNTER: {
        if (bytes != N * sizeof(int32_t)) { oracle_set_error("set_state: size mismatch"); return 1; }
        for (size_t i = 0; i < N; ++i) s->mobile[i].counter = ((const int32_t*)src)[i];
        return 0;
    }
    default:
        oracle_set_error("set_state: field %d not settable for MobileRobot", field);
        return 1;
    }
}

int srl_sim_get_state(srl_sim* s, int field, void* dst, size_t bytes) {
    if (!s || !dst) { oracle_set_error("get_state: null argument"); return 1; }
    return is_mobile(s->kind) ? mobile_get_state(s, field, dst, bytes) : oracle_kuka_get_state(s, field, dst, bytes);
}

int srl_sim_set_state(srl_sim* s, int field, const void* src, size_t bytes) {
    if (!s || !src) { oracle_set_error("set_state: null argument"); return 1; }
    return is_mobile(s->kind) ? mobile_set_state(s, field, src, bytes) : oracle_kuka_set_state(s, field, src, bytes);
}

} /* extern "C" */

/* Test hook: raw Philox block, for the known-answer test against the published vectors. */
#include "philox.h"
extern "C" void oracle_philox4x32(uint64_t seed, uint64_t env, uint32_t index, uint32_t purpose, uint32_t* out4) {
    philox4x32_10(seed, env, index, purpose, out4);
}
