// C-ABI of include/srl_sim.h for the sm_90a library (libsrl_sim_b200.so).
// Plain pointers and sizes only; torch never appears in a signature.  All buffers are DEVICE
// pointers except in srl_sim_rollout_host.  There is no CPU path in this library.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <new>
#include "common.cuh"

static thread_local char g_err[512] = "";

void srl_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

namespace {

struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; }
        if (prev != dev) ok = (cudaSetDevice(dev) == cudaSuccess);
    }
    ~DeviceGuard() {
        int cur = -1;
        if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
    }
};

int ensure_stage(srl_sim* s, int slot, size_t bytes) {
    if (s->stage_cap[slot] >= bytes) return 0;
    if (s->stage[slot]) cudaFree(s->stage[slot]);
    s->stage[slot] = nullptr;
    s->stage_cap[slot] = 0;
    SRL_CUDA_OK(cudaMalloc(&s->stage[slot], bytes));
    s->stage_cap[slot] = bytes;
    return 0;
}

// Streams of the srl_sim_rollout_host pipeline.  They are ordinary (blocking) streams: each one orders itself after work already
// queued on the legacy default stream -- where a preceding reset() / step() of a host-side caller runs -- and they do not
// serialise against each other.
int ensure_host_pipe(srl_sim* s) {
    if (s->host_pipe_ready) return 0;
    for (int k = 0; k < 3; ++k) SRL_CUDA_OK(cudaStreamCreate(&s->host_st[k]));
    for (int k = 0; k < 2 * SRL_HOST_MAX_CHUNKS; ++k) SRL_CUDA_OK(cudaEventCreateWithFlags(&s->host_ev[k], cudaEventDisableTiming));
    const char* env = getenv("SRL_HOST_CHUNKS");
    s->host_chunks = env ? atoi(env) : 0;
    s->host_pipe_ready = true;
    return 0;
}

int launch_rollout(srl_sim* s, int T, const void* actions, const float* noise, float* obs, float* rew, uint8_t* done,
                   float* ep_ret, int32_t* ep_len, cudaStream_t st) {
    SRL_CUDA_OK(cudaEventRecord(s->ev0, st));
    int rc = srl_is_mobile(s->kind) ? mobile_launch_rollout(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st)
                                    : kuka_launch_rollout(s, T, actions, noise, obs, rew, done, ep_ret, ep_len, st);
    if (rc) return rc;
    SRL_CUDA_OK(cudaEventRecord(s->ev1, st));
    s->ev_valid = true;
    s->launches += 1;
    return 0;
}

}  // namespace

extern "C" {

int srl_sim_abi_version(void) { return SRL_SIM_ABI_VERSION; }
const char* srl_sim_last_error(void) { return g_err; }

int srl_sim_create(srl_sim** out, int env_kind, int num_envs, int device, const srl_cfg* cfg, const void* model_blob,
                   size_t model_bytes, uint64_t seed) {
    if (!out || !cfg) { srl_set_error("create: null argument"); return 1; }
    *out = nullptr;
    if (cfg->struct_size != sizeof(srl_cfg)) {
        srl_set_error("create: srl_cfg size mismatch (%u != %zu)", cfg->struct_size, sizeof(srl_cfg));
        return 1;
    }
    if (device < 0) { srl_set_error("create: this library has no CPU path (device=%d)", device); return 1; }
    if (num_envs <= 0) { srl_set_error("create: num_envs must be positive"); return 1; }
    if (!srl_is_mobile(env_kind) && !srl_is_kuka(env_kind)) { srl_set_error("create: unknown env kind %d", env_kind); return 1; }
    if (cfg->action_joints && (!srl_is_kuka(env_kind) || cfg->is_discrete)) {
        // kuka_button_gym_env.py:149-161: the (7,) joint action space only exists for continuous Kuka actions
        srl_set_error("create: action_joints needs a Kuka env with is_discrete=0"); return 1;
    }
    if (srl_is_mobile(env_kind) && !cfg->is_discrete && env_kind != SRL_ENV_MOBILE && env_kind != SRL_ENV_MOBILE_LINE_TARGET) {
        // mobile_robot_2target_env.py:128, mobile_robot_1D_env.py:43,118 raise ValueError
        srl_set_error("Only discrete actions is supported");
        return 2;
    }
    int ndev = 0;
    SRL_CUDA_OK(cudaGetDeviceCount(&ndev));
    if (device >= ndev) { srl_set_error("create: device %d out of range (%d visible)", device, ndev); return 1; }
    DeviceGuard guard(device);
    if (!guard.ok) { srl_set_error("create: cudaSetDevice(%d) failed", device); return 1; }
    cudaDeviceProp prop;
    SRL_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        srl_set_error("create: device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
        return 1;
    }
    srl_sim* s = new (std::nothrow) srl_sim();
    if (!s) { srl_set_error("create: out of memory"); return 1; }
    memset(s, 0, sizeof(*s));
    s->kind = env_kind;
    s->n = num_envs;
    s->device = device;
    s->sms = prop.multiProcessorCount;
    s->cfg = *cfg;
    if (s->cfg.action_repeat < 1) s->cfg.action_repeat = 1;
    if (s->cfg.solver_iterations <= 0) s->cfg.solver_iterations = 150;
    if (s->cfg.timestep <= 0.f) s->cfg.timestep = 1.0f / 240.0f;
    s->seed = seed;
    s->auto_reset = !cfg->no_auto_reset;
    s->max_steps = cfg->max_steps > 0 ? cfg->max_steps : (srl_is_mobile(env_kind) ? 250 : (env_kind == SRL_ENV_KUKA_MOVING_BUTTON || env_kind == SRL_ENV_KUKA_2BUTTON) ? 1500 : 1000);
    if (cudaEventCreate(&s->ev0) != cudaSuccess || cudaEventCreate(&s->ev1) != cudaSuccess) {
        srl_set_error("create: cudaEventCreate failed");
        delete s;
        return 1;
    }
    int rc = srl_is_mobile(env_kind) ? mobile_alloc(s) : kuka_alloc(s, model_blob, model_bytes);
    if (rc) { srl_sim_destroy(s); return rc; }
    *out = s;
    return 0;
}

void srl_sim_destroy(srl_sim* s) {
    if (!s) return;
    DeviceGuard guard(s->device);
    cudaDeviceSynchronize();
    if (srl_is_mobile(s->kind)) mobile_free(s); else kuka_free(s);
    render_free(s);
    for (int k = 0; k < 5; ++k) if (s->stage[k]) cudaFree(s->stage[k]);
    for (int k = 0; k < 3; ++k) if (s->host_st[k]) cudaStreamDestroy(s->host_st[k]);
    for (int k = 0; k < 2 * SRL_HOST_MAX_CHUNKS; ++k) if (s->host_ev[k]) cudaEventDestroy(s->host_ev[k]);
    if (s->ev0) cudaEventDestroy(s->ev0);
    if (s->ev1) cudaEventDestroy(s->ev1);
    delete s;
}

int srl_sim_num_envs(const srl_sim* s) { return s ? s->n : 0; }
int srl_sim_obs_dim(const srl_sim* s) { return !s ? 0 : srl_is_kuka(s->kind) ? 3 : (s->kind == SRL_ENV_MOBILE_1D ? 1 : 2); }
int srl_sim_action_dim(const srl_sim* s) {
    if (!s) return 0;
    if (s->cfg.is_discrete) return 1;
    return srl_is_mobile(s->kind) ? 2 : (s->cfg.action_joints ? 7 : 3);
}
uint64_t srl_sim_launch_count(const srl_sim* s) { return s ? s->launches : 0; }

float srl_sim_last_kernel_ms(srl_sim* s) {
    if (!s || !s->ev_valid) return -1.0f;
    DeviceGuard guard(s->device);
    if (cudaEventSynchronize(s->ev1) != cudaSuccess) return -1.0f;
    float ms = -1.0f;
    if (cudaEventElapsedTime(&ms, s->ev0, s->ev1) != cudaSuccess) return -1.0f;
    return ms;
}

int srl_sim_reset(srl_sim* s, const uint8_t* mask, const double* reset_draws, float* obs_out, void* stream) {
    if (!s) { srl_set_error("reset: null handle"); return 1; }
    DeviceGuard guard(s->device);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = srl_is_mobile(s->kind) ? mobile_launch_reset(s, mask, reset_draws, obs_out, st)
                                    : kuka_launch_reset(s, mask, reset_draws, obs_out, st);
    if (!rc) s->launches += 1;
    return rc;
}

int srl_sim_step(srl_sim* s, const void* actions, const float* noise, float* obs_out, float* rew_out, uint8_t* done_out,
                 float* ep_ret_out, int32_t* ep_len_out, void* stream) {
    if (!s) { srl_set_error("step: null handle"); return 1; }
    if (!actions) { srl_set_error("step: actions must not be NULL (use srl_sim_rollout for in-kernel random actions)"); return 1; }
    DeviceGuard guard(s->device);
    return launch_rollout(s, 1, actions, noise, obs_out, rew_out, done_out, ep_ret_out, ep_len_out, (cudaStream_t)stream);
}

int srl_sim_rollout(srl_sim* s, int T, const void* actions, const float* noise, float* obs_out, float* rew_out,
                    uint8_t* done_out, float* ep_ret_out, int32_t* ep_len_out, void* stream) {
    if (!s) { srl_set_error("rollout: null handle"); return 1; }
    if (T < 0) { srl_set_error("rollout: negative T"); return 1; }
    if (T == 0) return 0;
    DeviceGuard guard(s->device);
    return launch_rollout(s, T, actions, noise, obs_out, rew_out, done_out, ep_ret_out, ep_len_out, (cudaStream_t)stream);
}

int srl_sim_prefetch_resets(srl_sim* s, void* stream) {
    if (!s) { srl_set_error("prefetch_resets: null handle"); return 1; }
    if (!srl_is_kuka(s->kind)) return 0;
    DeviceGuard guard(s->device);
    return kuka_launch_prefetch(s, (cudaStream_t)stream);
}

int srl_sim_rollout_host(srl_sim* s, int T, const void* actions, const float* noise, float* obs_out, float* rew_out,
                         uint8_t* done_out) {
    if (!s) { srl_set_error("rollout_host: null handle"); return 1; }
    if (T <= 0) { srl_set_error("rollout_host: T must be positive"); return 1; }
    DeviceGuard guard(s->device);
    const size_t N = (size_t)s->n, TN = (size_t)T * N;
    const size_t D = (size_t)srl_sim_obs_dim(s), A = (size_t)srl_sim_action_dim(s);
    const size_t act_step = N * A * 4, noise_step = N * 4, obs_step = N * D * 4, rew_step = N * 4, done_step = N;   // bytes per env step
    if (ensure_host_pipe(s)) return 1;
    // The [T, N] streams are time-major, so a range of steps is a contiguous slice of every buffer: the rollout runs as a few
    // T-chunks, chunk c's kernel overlapping the copy-in of chunk c + 1 and the copy-out of chunk c - 1 (PCIe is full duplex).
    // Results do not depend on the chunking (a rollout of T steps == consecutive shorter rollouts; tests/test_*_gpu.py).
    const size_t moved = (actions ? T * act_step : 0) + (noise ? T * noise_step : 0) + (obs_out ? T * obs_step : 0) +
                         (rew_out ? T * rew_step : 0) + (done_out ? TN : 0);
    // Chunk count by bytes moved, one chunk per 32 MB (where it was measured, the 143 MB MobileRobot rollout ran
    // faster in 4 chunks than in 1 and no better in 16; the 13 MB Kuka rollout is fastest unsplit -- every extra launch of its long
    // kernel pays a tail of warps finishing at different times)
    int chunks = s->host_chunks > 0 ? s->host_chunks : (int)(moved / ((size_t)32 << 20));
    if (chunks < 1) chunks = 1;
    if (chunks > SRL_HOST_MAX_CHUNKS) chunks = SRL_HOST_MAX_CHUNKS;
    if (chunks > T) chunks = T;
    // Outputs are always staged in HBM and copied out, also into pinned host buffers: letting the kernel store straight into pinned,
    // device-mapped buffers was measured no faster end to end with the 4096-env x 128-step Kuka rollout (the device->host copy it
    // removes is paid back by the kernel draining its sysmem stores).
    char *d_act = nullptr, *d_noise = nullptr, *d_obs = nullptr, *d_rew = nullptr, *d_done = nullptr;
    if (actions) { if (ensure_stage(s, 0, T * act_step)) return 1; d_act = (char*)s->stage[0]; }
    if (noise) { if (ensure_stage(s, 1, T * noise_step)) return 1; d_noise = (char*)s->stage[1]; }
    if (obs_out) { if (ensure_stage(s, 2, T * obs_step)) return 1; d_obs = (char*)s->stage[2]; }
    if (rew_out) { if (ensure_stage(s, 3, T * rew_step)) return 1; d_rew = (char*)s->stage[3]; }
    if (done_out) { if (ensure_stage(s, 4, TN)) return 1; d_done = (char*)s->stage[4]; }
    const int chunk_T = (T + chunks - 1) / chunks;
    cudaStream_t st_in = s->host_st[0], st_run = s->host_st[1], st_out = s->host_st[2];
    int c = 0;
    for (int t0 = 0; t0 < T; t0 += chunk_T, ++c) {
        const size_t tc = (size_t)(T - t0 < chunk_T ? T - t0 : chunk_T);
        if (actions) SRL_CUDA_OK(cudaMemcpyAsync(d_act + t0 * act_step, (const char*)actions + t0 * act_step, tc * act_step, cudaMemcpyHostToDevice, st_in));
        if (noise) SRL_CUDA_OK(cudaMemcpyAsync(d_noise + t0 * noise_step, (const char*)noise + t0 * noise_step, tc * noise_step, cudaMemcpyHostToDevice, st_in));
        SRL_CUDA_OK(cudaEventRecord(s->host_ev[2 * c], st_in));
    }
    c = 0;
    for (int t0 = 0; t0 < T; t0 += chunk_T, ++c) {
        const int tc = T - t0 < chunk_T ? T - t0 : chunk_T;
        SRL_CUDA_OK(cudaStreamWaitEvent(st_run, s->host_ev[2 * c], 0));
        int rc = launch_rollout(s, tc, d_act ? d_act + t0 * act_step : nullptr, d_noise ? (const float*)(d_noise + t0 * noise_step) : nullptr,
                                d_obs ? (float*)(d_obs + t0 * obs_step) : nullptr, d_rew ? (float*)(d_rew + t0 * rew_step) : nullptr,
                                d_done ? (uint8_t*)(d_done + t0 * done_step) : nullptr, nullptr, nullptr, st_run);
        if (rc) { cudaDeviceSynchronize(); return rc; }
        SRL_CUDA_OK(cudaEventRecord(s->host_ev[2 * c + 1], st_run));
        SRL_CUDA_OK(cudaStreamWaitEvent(st_out, s->host_ev[2 * c + 1], 0));
        if (obs_out) SRL_CUDA_OK(cudaMemcpyAsync((char*)obs_out + t0 * obs_step, d_obs + t0 * obs_step, tc * obs_step, cudaMemcpyDeviceToHost, st_out));
        if (rew_out) SRL_CUDA_OK(cudaMemcpyAsync((char*)rew_out + t0 * rew_step, d_rew + t0 * rew_step, tc * rew_step, cudaMemcpyDeviceToHost, st_out));
        if (done_out) SRL_CUDA_OK(cudaMemcpyAsync((char*)done_out + t0 * done_step, d_done + t0 * done_step, tc * done_step, cudaMemcpyDeviceToHost, st_out));
    }
    SRL_CUDA_OK(cudaStreamSynchronize(st_run));   // the state update is complete even when no output was requested
    SRL_CUDA_OK(cudaStreamSynchronize(st_out));
    return 0;
}

int srl_sim_render(srl_sim* s, const srl_camera* camera, int width, int height, uint8_t* rgb_out, void* stream) {
    if (!s || !camera || !rgb_out) { srl_set_error("render: null argument"); return 1; }
    if (width <= 0 || height <= 0 || width > 4096 || height > 4096) { srl_set_error("render: bad image size %d x %d", width, height); return 1; }
    if (!(camera->distance > 0.f) || !(camera->fov > 0.f && camera->fov < 180.f)) { srl_set_error("render: bad camera (distance %g, fov %g)", camera->distance, camera->fov); return 1; }
    DeviceGuard guard(s->device);
    return render_launch(s, camera, width, height, rgb_out, (cudaStream_t)stream);
}

int srl_sim_render_cameras(srl_sim* s, const srl_camera* cameras, int follow_robot, int width, int height, uint8_t* rgb_out, void* stream) {
    if (!s || !cameras || !rgb_out) { srl_set_error("render_cameras: null argument"); return 1; }
    if (width <= 0 || height <= 0 || width > 4096 || height > 4096) { srl_set_error("render_cameras: bad image size %d x %d", width, height); return 1; }
    if (follow_robot && !srl_is_mobile(s->kind)) { srl_set_error("render_cameras: follow_robot needs a MobileRobot env kind (got kind %d)", s->kind); return 1; }
    for (int i = 0; i < s->n; ++i) {
        const srl_camera& c = cameras[i];
        if (!(c.distance > 0.f) || !(c.fov > 0.f && c.fov < 180.f)) { srl_set_error("render_cameras: bad camera %d (distance %g, fov %g)", i, c.distance, c.fov); return 1; }
    }
    DeviceGuard guard(s->device);
    return render_cams_launch(s, cameras, follow_robot, width, height, rgb_out, (cudaStream_t)stream);
}

int srl_sim_set_distractors(srl_sim* s, const void* assets_blob, size_t bytes) {
    if (!s) { srl_set_error("set_distractors: null handle"); return 1; }
    if (!srl_is_kuka(s->kind)) { srl_set_error("set_distractors: only KukaRandButtonGymEnv-v0 has distractor bodies"); return 1; }
    DeviceGuard guard(s->device);
    return kuka_set_distractors(s, assets_blob, bytes);
}

int srl_sim_get_state(srl_sim* s, int field, void* dst, size_t bytes) {
    if (!s || !dst) { srl_set_error("get_state: null argument"); return 1; }
    DeviceGuard guard(s->device);
    return srl_is_mobile(s->kind) ? mobile_get_state(s, field, dst, bytes) : kuka_get_state(s, field, dst, bytes);
}

int srl_sim_set_state(srl_sim* s, int field, const void* src, size_t bytes) {
    if (!s || !src) { srl_set_error("set_state: null argument"); return 1; }
    DeviceGuard guard(s->device);
    return srl_is_mobile(s->kind) ? mobile_set_state(s, field, src, bytes) : kuka_set_state(s, field, src, bytes);
}

}  // extern "C"
