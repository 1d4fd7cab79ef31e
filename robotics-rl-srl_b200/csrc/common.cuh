// Internal declarations shared by the translation units of libsrl_sim_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <atomic>
#include "../../include/srl_sim.h"

void srl_set_error(const char* fmt, ...);

#define SRL_CUDA_OK(expr)                                                                   \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) {                                                            \
            srl_set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,              \
                          cudaGetErrorString(_e));                                          \
            return 1;                                                                       \
        }                                                                                   \
    } while (0)

// Opt `Kernel` in to `bytes` (> 48 KB) of dynamic shared memory on the current device.  The attribute belongs to the device context,
// so it is set once per kernel and device; a process with handles on several devices sets it on each.
template <auto Kernel>
cudaError_t srl_smem_opt_in(size_t bytes) {
    static std::atomic<uint64_t> devices{0};   // bit d: set on device d (devices from 64 on: set at every call)
    int dev = 0;
    if (const cudaError_t e = cudaGetDevice(&dev)) return e;
    const uint64_t bit = dev >= 0 && dev < 64 ? 1ull << dev : 0ull;
    if (devices.load(std::memory_order_relaxed) & bit) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) devices.fetch_or(bit, std::memory_order_relaxed);
    return e;
}

// ---- MobileRobot family: structure-of-arrays state in HBM, 16-byte records per field -----
struct MobileDev {
    double2* pos;   // [N] robot_pos (x, y); z is identically 0 (mobile_robot_env.py:170)
    double2* tgt0;  // [N] target_pos (x, y)
    double2* tgt1;  // [N] second target (2-target variant only)
    int4*    meta;  // [N] {_env_step_counter, current_target | has_bumped << 8, episode, total_steps}
    double2* ep;    // [N] {running episode return, running episode length}
};

struct KukaDev;   // kuka_state.cuh
struct KukaNext;  // kuka_kernels.cu
struct DistDev;   // distractor_kernels.cu
struct SrlBodyLooks;  // render_core.h
struct SrlCam;        // render_core.h
struct SrlCamFollow;  // render_core.h

#define SRL_HOST_MAX_CHUNKS 16

struct srl_sim {
    int kind;
    int n;
    int device;
    int sms;            // multiprocessors of `device`
    srl_cfg cfg;
    uint64_t seed;
    int auto_reset;
    int max_steps;
    MobileDev mob;      // current state
    MobileDev mob_alt;  // the other half of the double buffer (rollouts write here, then swap)
    KukaDev* kuka;
    KukaNext* kuka_next; // next-episode records, only with srl_cfg.prefetch_resets (nullptr: off)
    DistDev* dist;      // KukaRandButton distractor bodies, only after srl_sim_set_distractors (nullptr: off)
    float kuka_q0[12];  // the initial joint vector the settle starts from
    bool kuka_started;  // a reset / step / rollout has been issued
    cudaEvent_t pf_ev;  // end of the last bulk record fill (srl_sim_prefetch_resets); the next rollout launch waits for it
    bool pf_pending;
    cudaEvent_t roll_ev; // end of the last rollout launch of a handle with records; a bulk fill waits for it
    bool roll_ev_valid;
    uint64_t launches;
    cudaEvent_t ev0, ev1;
    bool ev_valid;
    // device staging buffers for the *_host entry points (grown on demand)
    void* stage[5];
    size_t stage_cap[5];
    // srl_sim_rollout_host pipeline: copy-in / kernel / copy-out streams and one (inputs landed, outputs ready) event pair per T-chunk
    cudaStream_t host_st[3];
    cudaEvent_t host_ev[2 * SRL_HOST_MAX_CHUNKS];
    bool host_pipe_ready;
    int host_chunks;    // SRL_HOST_CHUNKS override (0 = by bytes moved)
    float* render_prims; // [N][SRL_MAX_PRIMS][16] scene primitives of the last srl_sim_render (allocated on first use)
    float* render_prep;  // same shape: their per-camera prepared forms (render_core.h SrlPrep)
    int* render_counts;
    // srl_sim_render_cameras (allocated on first use): every env's camera, the follow_robot inputs, their pinned staging buffer and the event
    // of its last upload, and the camera array, size and follow_robot of the last call (the cameras are rebuilt only when these change)
    SrlCam* render_cams;          // [N]
    SrlCamFollow* render_follow;  // [N]
    void* render_cam_stage;
    cudaEvent_t render_cam_ev;
    srl_camera* render_cam_key;   // [N], host
    int render_cam_follow, render_cam_w, render_cam_h, render_cam_valid;
};

static inline bool srl_is_mobile(int kind) { return kind >= SRL_ENV_MOBILE && kind <= SRL_ENV_MOBILE_LINE_TARGET; }
static inline bool srl_is_kuka(int kind) { return kind >= SRL_ENV_KUKA_BUTTON && kind <= SRL_ENV_KUKA_MOVING_BUTTON; }

// ---- launchers (mobile_kernels.cu) -------------------------------------------------------
int mobile_alloc(srl_sim* s);
void mobile_free(srl_sim* s);
int mobile_launch_reset(srl_sim* s, const uint8_t* mask, const double* draws, float* obs, cudaStream_t st);
int mobile_launch_rollout(srl_sim* s, int T, const void* actions, const float* noise, float* obs, float* rew,
                          uint8_t* done, float* ep_ret, int32_t* ep_len, cudaStream_t st);
int mobile_get_state(srl_sim* s, int field, void* dst, size_t bytes);
int mobile_set_state(srl_sim* s, int field, const void* src, size_t bytes);

// ---- image observations (render_kernels.cu) ------------------------------------------------
int render_launch(srl_sim* s, const srl_camera* cam, int width, int height, uint8_t* rgb, cudaStream_t st);
int render_cams_launch(srl_sim* s, const srl_camera* cams, int follow_robot, int width, int height, uint8_t* rgb, cudaStream_t st);
void render_free(srl_sim* s);

// ---- launchers (kuka_kernels.cu) ---------------------------------------------------------
int kuka_alloc(srl_sim* s, const void* blob, size_t bytes);
void kuka_free(srl_sim* s);
int kuka_launch_reset(srl_sim* s, const uint8_t* mask, const double* draws, float* obs, cudaStream_t st);
int kuka_launch_rollout(srl_sim* s, int T, const void* actions, const float* noise, float* obs, float* rew,
                        uint8_t* done, float* ep_ret, int32_t* ep_len, cudaStream_t st);
int kuka_launch_prefetch(srl_sim* s, cudaStream_t st);
int kuka_render_prims(srl_sim* s, float* prims, int* counts, cudaStream_t st);   // [N][SRL_MAX_PRIMS][16] primitive list of every env's scene
int kuka_set_distractors(srl_sim* s, const void* blob, size_t bytes);
int kuka_get_state(srl_sim* s, int field, void* dst, size_t bytes);
int kuka_set_state(srl_sim* s, int field, const void* src, size_t bytes);

// ---- KukaRandButton's distractor bodies (distractor_kernels.cu), driven by the Kuka launchers ----------------------------------
int dist_alloc(srl_sim* s, const void* blob, size_t bytes, float4** settle);   // checks, assets, buffers; *settle: room for the arm's settle trace
int dist_trace(srl_sim* s, size_t steps, cudaStream_t st, float4** trace, int** trace_len);   // trace buffers for <= `steps` micro-steps per env
int dist_advance(srl_sim* s, const double* draws, cudaStream_t st);   // distractor_kernel through the micro-steps of the last traced launch
void dist_free(srl_sim* s);
int dist_get_state(srl_sim* s, int field, void* dst, size_t bytes);   // SRL_F_DISTRACTORS, SRL_F_DISTRACTOR_TOUCH and the SRL_F_DISTRACTOR_* test hooks
int dist_set_state(srl_sim* s, const void* src, size_t bytes);   // SRL_F_DISTRACTOR_RECORDS
const float* dist_render_bodies(const srl_sim* s, SrlBodyLooks* looks);   // [N][DC_NBODY][DC_B_WORDS] body poses + drawing table; nullptr: no bodies
