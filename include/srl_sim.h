/*
 * srl_sim.h -- C-ABI of the H100-native batched simulator for the robotics-rl-srl
 * PyBullet environments (Kuka button-push family and MobileRobot family, `ground_truth`
 * observation mode).
 *
 * This is the drop-in boundary.  Everything above it is host Python that mirrors the
 * reference's `SRLGymEnv` / `environments.registry` surface; everything below it is
 * hand-written sm_90a CUDA (libsrl_sim_b200.so).  The CPU oracle (oracle/liboracle_sim.so,
 * test infrastructure only) exports the SAME symbols with `device = -1` and host pointers,
 * so parity tests drive both through one binding.
 *
 * Reference interfaces each entry point replaces (paths relative to the reference repo):
 *   srl_sim_create      <- env constructors + world build:
 *                          environments/kuka_gym/kuka_button_gym_env.py:78-173,
 *                          environments/mobile_robot/mobile_robot_env.py:61-145,
 *                          environments/utils.py:36-57 (makeEnv: one env per process, seed+rank)
 *   srl_sim_reset       <- KukaButtonGymEnv.reset (kuka_button_gym_env.py:214-281),
 *                          MobileRobotGymEnv.reset (mobile_robot_env.py:159-222)
 *   srl_sim_step        <- KukaButtonGymEnv.step/step2/_reward/_termination
 *                          (kuka_button_gym_env.py:293-368,422-463), Kuka.applyAction
 *                          (kuka_gym/kuka.py:118-187), pybullet.stepSimulation (:351),
 *                          MobileRobotGymEnv.step/_reward/_termination
 *                          (mobile_robot_env.py:235-280,336-363), plus the SubprocVecEnv
 *                          worker's auto-reset-on-done (rl_baselines/utils.py:216-220)
 *   srl_sim_rollout*    <- the consumer loop `for t in range(n_steps): env.step(actions[t])`
 *                          (rl_baselines/random_agent.py:28-42; PPO2 runner, n_steps=128,
 *                          rl_baselines/rl_algorithm/ppo2.py:58-72), fused into one launch
 *   srl_sim_get/set_state <- getGroundTruth/getTargetPos/getArmPos accessors
 *                          (kuka_button_gym_env.py:191-212, mobile_robot_env.py:147-157)
 *
 * Conventions
 *   - All functions return 0 on success, non-zero on error; the message is available from
 *     srl_sim_last_error() (thread-local).  Nothing throws across the ABI.
 *   - The library owns the per-env structure-of-arrays state.  The caller owns action /
 *     observation / reward / done buffers.  For the CUDA library those are DEVICE pointers
 *     (e.g. torch tensors' data_ptr()) unless the function name ends in `_host`; for the
 *     oracle they are host pointers.
 *   - Calls are stream-ordered and asynchronous on `stream` (a cudaStream_t passed as void*;
 *     NULL = the legacy default stream).  `_host` entry points synchronise before returning.
 *   - One srl_sim per (process, GPU); a handle is not re-entrant.
 *   - Environment `i` of a handle has the GLOBAL index `cfg->global_env_offset + i`; its
 *     counter-based RNG stream is keyed by (seed, global index), so results do not depend on
 *     how a batch is sharded over GPUs.
 */
#ifndef SRL_SIM_H_
#define SRL_SIM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SRL_SIM_ABI_VERSION 1

typedef struct srl_sim srl_sim; /* opaque */

/* environments/registry.py:42-49 -- the eight PyBullet ids */
enum srl_env_kind {
    SRL_ENV_KUKA_BUTTON        = 0, /* KukaButtonGymEnv-v0            */
    SRL_ENV_KUKA_RAND_BUTTON   = 1, /* KukaRandButtonGymEnv-v0        */
    SRL_ENV_KUKA_2BUTTON       = 2, /* Kuka2ButtonGymEnv-v0           */
    SRL_ENV_KUKA_MOVING_BUTTON = 3, /* KukaMovingButtonGymEnv-v0      */
    SRL_ENV_MOBILE             = 4, /* MobileRobotGymEnv-v0           */
    SRL_ENV_MOBILE_2TARGET     = 5, /* MobileRobot2TargetGymEnv-v0    */
    SRL_ENV_MOBILE_1D          = 6, /* MobileRobot1DGymEnv-v0         */
    SRL_ENV_MOBILE_LINE_TARGET = 7  /* MobileRobotLineTargetGymEnv-v0 */
};

/* Constructor keyword arguments of the reference envs that change the arithmetic
 * (kuka_button_gym_env.py:78-81, mobile_robot_env.py:61-64) plus solver parameters the
 * reference sets on the physics client (kuka_button_gym_env.py:218-220,236). */
typedef struct srl_cfg {
    uint32_t struct_size;       /* = sizeof(srl_cfg); checked                                  */
    int32_t  is_discrete;       /* Discrete(6)/Discrete(4) vs Box actions                      */
    int32_t  random_target;     /* randomise button / target position at reset                 */
    int32_t  force_down;        /* Kuka: remove the "up" action                                */
    int32_t  shape_reward;      /* reward = -distance (and 50/-250 on continuous Kuka)         */
    int32_t  action_joints;     /* Kuka joint-space actions f32[N,7] (continuous only)         */
    int32_t  action_repeat;     /* Kuka physics sub-steps per env step (>=1)                   */
    int32_t  max_steps;         /* 0 = reference default for the env kind (1000 / 250)         */
    int32_t  solver_iterations; /* 0 = 150 (setPhysicsEngineParameter)                        */
    int32_t  envs_per_warp;     /* Kuka CUDA kernels: active lanes per warp, 0 = auto          */
    int32_t  no_auto_reset;     /* 0 = VecEnv semantics (reset on done, return post-reset obs);
                                   1 = single-env gym semantics (terminal obs, caller resets)  */
    float    max_distance;      /* Kuka safety-sphere radius (0.8); unused for MobileRobot     */
    float    timestep;          /* 0 = 1/240                                                   */
    uint32_t prefetch_resets;   /* Kuka, opt-in (0 = off): keep a ready post-reset state per env so that a lockstep
                                   step never runs reset() inside the launch; the records are advanced by the idle slot
                                   of every warp of every step / rollout launch (bulk fill: srl_sim_prefetch_resets)   */
    uint64_t global_env_offset; /* global index of local env 0 (multi-GPU sharding)            */
} srl_cfg;

/* Fields addressable through srl_sim_get_state / srl_sim_set_state.  All are dense
 * host-side arrays [num_envs, width] of the listed type (the library converts from its
 * internal layout). */
enum srl_state_field {
    SRL_F_ROBOT_POS     = 0,  /* f64[N,3] Mobile: robot_pos; Kuka: gripper (link 8 COM) world pos */
    SRL_F_TARGET_POS    = 1,  /* f64[N,3] Mobile: target_pos; Kuka: button_pos (target, frozen at reset) */
    SRL_F_STEP_COUNTER  = 2,  /* i32[N,1] _env_step_counter                                    */
    SRL_F_JOINT_POS     = 3,  /* f64[N,12] Kuka q (movable joints in index order 0-8,10,11,13) */
    SRL_F_JOINT_VEL     = 4,  /* f64[N,12] Kuka qd                                             */
    SRL_F_EE_CMD        = 5,  /* f64[N,3] Kuka commanded end-effector position (kuka.py:73,134-139) */
    SRL_F_EE_POS        = 6,  /* f64[N,3] Kuka link-6 frame origin (the IK link)               */
    SRL_F_BUTTON_GLIDER = 7,  /* f64[N,2] button prismatic joint (q, qd)                       */
    SRL_F_COUNTERS      = 8,  /* i32[N,4] Kuka: n_contacts, n_steps_outside, terminated, episode index */
    SRL_F_EPISODE_STATS = 9,  /* f64[N,2] running episode return, length                       */
    SRL_F_BUTTON_BASE   = 10, /* f64[N,3] Kuka: button base link origin (x, y, z)              */
    SRL_F_TWO_BUTTON    = 11, /* f64[N,8] Kuka2Button (read-only): n_contacts[0], n_contacts[1], goal_id, second button base x y z,
                                 second glider q, qd (kuka_2button_gym_env.py:34,40-43)          */
    SRL_F_NEXT_RECORD   = 12, /* i32[N,3] Kuka with srl_cfg.prefetch_resets (read-only, CUDA library): next-episode record
                                 complete (0/1), random reset micro-steps applied to an incomplete record (0-4), episode index
                                 the record is for; all zero / -1 without the feature                         */
    SRL_F_DISTRACTORS   = 13, /* f64[N,11,9] KukaRandButton distractor bodies (read-only): position xyz, orientation quaternion
                                 xyz w, body type (0 duck_vhacd, 1 lego, 2 cube_small, 3 sphere_small), present (0/1); slots 0-9
                                 are the 10 placements of reset() (absent inside the square around the button), slot 10 the
                                 kicked sphere; all zero without srl_sim_set_distractors                       */
    SRL_F_DISTRACTOR_TOUCH = 14, /* i32[N,2] (read-only) bit k set: distractor slot k touched another body / the arm since its
                                 placement                                                                     */
    /* Test hooks of the CUDA library's distractor bodies (copies of device buffers in their own float32 layout; not for
     * applications, and not in the CPU oracle, which refuses them like every field it does not know): */
    SRL_F_DISTRACTOR_RECORDS = 15, /* f32[N,11,16] the full body records (csrc/distractor_core.h, DC_B_*): position, quaternion
                                 xyz w, v, w, type, present, 2 unused words.  Settable, so that a test can start the bodies from a
                                 crafted configuration: every value finite, present 0 or 1, type 0-3, unit quaternion (1e-4), else the
                                 call is refused.  The touch masks are left as they are.                       */
    SRL_F_DISTRACTOR_TRACE_LEN = 16, /* i32[N,1] (read-only) micro-steps the last reset / step / rollout launch recorded per env */
    SRL_F_DISTRACTOR_TRACE = 17, /* f32[N,L,16] (read-only) the first L records of that launch's trace per env, L = bytes / (64 N)
                                 at most the launch's capacity T (action_repeat + 5) (5 for a reset): joint angles q[0-11], glider q,
                                 button base x, y, and the tag word (bits of an int32: tag | episode << 4, csrc/kuka_state.cuh)  */
    SRL_F_DISTRACTOR_SETTLE = 18 /* f32[500,16] (read-only, not per env) the arm's settle trajectory the bodies are settled against,
                                 same record layout                                                            */
};

int srl_sim_abi_version(void);

/* Build `num_envs` environments of one kind on `device` (CUDA ordinal; -1 only in the
 * oracle library).  `model_blob` is the flat robot/scene model produced by the URDF loader
 * (srl_sim/model.py; layout in csrc/kuka_model.h); MobileRobot kinds accept NULL.  The envs
 * are created un-reset: call srl_sim_reset before the first step. */
int srl_sim_create(srl_sim** out, int env_kind, int num_envs, int device, const srl_cfg* cfg,
                   const void* model_blob, size_t model_bytes, uint64_t seed);

/* Reset the envs whose mask byte is non-zero (mask == NULL: all).
 * `reset_draws` (nullable): f64[N, R] values the reference would have drawn from `np_random`
 * during reset(), supplied by the host for exact-seed parity; NULL = generate them from the
 * env's counter-based stream.
 *   MobileRobot R=6: x_start, y_start, x_target, y_target, x_target2, y_target2 -- the final
 *                    values, not the raw uniforms (mobile_robot_env.py:168-181,
 *                    mobile_robot_2target_env.py:52-69); unused slots are ignored
 *   Kuka        R=18: button x_pos, y_pos, then 5 x (dx,dy,dz) random init actions (action_joints: the common joint
 *                     set-point offset DELTA_THETA * normal in the dx slot, kuka_button_gym_env.py:257-260)
 *                     (kuka_button_gym_env.py:227-234,250-268), then the signed button speed of
 *                     KukaMovingButtonGymEnv (kuka_moving_button_gym_env.py:33; 0 for the other kinds)
 * `obs_out` (nullable): f32[N, D] observation after reset (rows of unmasked envs untouched). */
int srl_sim_reset(srl_sim* sim, const uint8_t* mask, const double* reset_draws, float* obs_out,
                  void* stream);

/* One env step for every env (lockstep), with SubprocVecEnv auto-reset semantics: where
 * done, the env is reset and `obs_out` holds the post-reset observation.
 *   actions : i32[N] (discrete) or f32[N, A] (continuous; A = 3 Kuka, 7 Kuka with action_joints, 2 Mobile); a negative
 *             discrete action is the reference's `step(None)` (zero action, Kuka only)
 *   noise   : nullable f32[N], the value of the `np_random.normal(0, NOISE_STD)` draw of this
 *             step (kuka_button_gym_env.py:305,327; mobile_robot_env.py:241,248); NULL =
 *             counter-based stream (Kuka) / exactly 0.0 (Mobile, NOISE_STD = 0.0)
 *   obs_out : f32[N, D];  rew_out : f32[N];  done_out : u8[N]
 *   ep_ret_out / ep_len_out : nullable f32[N] / i32[N], Monitor-style episode return and
 *             length, valid where done (environments/utils.py:53-54) */
int srl_sim_step(srl_sim* sim, const void* actions, const float* noise, float* obs_out,
                 float* rew_out, uint8_t* done_out, float* ep_ret_out, int32_t* ep_len_out,
                 void* stream);

/* T fused lockstep steps in ONE launch (state stays in registers between steps).
 *   actions : i32[T,N] / f32[T,N,A], or NULL = uniform random actions from the env's stream
 *             (the reference's random agent, rl_baselines/random_agent.py:34)
 *   noise   : nullable f32[T,N]
 *   obs/rew/done : nullable [T,N,D] / [T,N] / [T,N] outputs (NULL = not stored)
 *   ep_ret_out / ep_len_out : nullable f32[T,N] / i32[T,N], valid where done */
int srl_sim_rollout(srl_sim* sim, int T, const void* actions, const float* noise, float* obs_out,
                    float* rew_out, uint8_t* done_out, float* ep_ret_out, int32_t* ep_len_out,
                    void* stream);

/* Same as srl_sim_rollout but every buffer is a HOST pointer (pinned for full speed): copies
 * the actions/noise host->device, runs the fused rollout, copies obs/rew/done device->host and
 * synchronises.  This is the call an out-of-process consumer (the reference's VecEnv user)
 * makes; bench.py's `e2e` leg times it. */
int srl_sim_rollout_host(srl_sim* sim, int T, const void* actions, const float* noise,
                         float* obs_out, float* rew_out, uint8_t* done_out);

/* Opt-in (srl_cfg.prefetch_resets): next-episode records.  The post-reset state of an episode is a pure function of (seed, global
 * env index, episode index), so it can be produced ahead of time; a step whose env finishes an episode then copies the record in
 * instead of running reset()'s five random micro-steps inside the launch; if no record is ready it resets in the launch as
 * before -- results never depend on which of the two happened.  With the option on, EVERY srl_sim_step / srl_sim_rollout launch
 * uses the first idle slot of each of its warps (a batch is spread over all warp schedulers, so a warp carries fewer envs than it has
 * slots) to advance one incomplete record of that warp's envs by one random micro-step per env step of the launch -- the helper runs
 * the same instructions as its warp, at no extra cost -- so no call is needed in steady state (and a captured CUDA graph of step
 * launches just works).  This entry point is the BULK
 * fill: it completes the records of all envs that have none, in one launch of its own -- call it once after srl_sim_reset of all
 * envs if the first episodes are short.  Stream-ordered like every other call; when `stream` differs from the stream of the
 * handle's step launches the library orders the two with events (it never overlaps them).  No-op (returns 0) for handles
 * without the feature.  Reference: the reset() a SubprocVecEnv worker runs between two steps
 * (kuka_button_gym_env.py:214-281 via rl_baselines/utils.py:216-220). */
int srl_sim_prefetch_resets(srl_sim* sim, void* stream);

/* Opt-in for SRL_ENV_KUKA_RAND_BUTTON: simulate the reference's distractor objects (kuka_rand_button_gym_env.py:58-68,117-127) --
 * up to 10 objects dropped at random positions around the button and a small sphere that is kicked at env step 10.  The bodies are
 * free rigid bodies pushed by the arm, the button and the table, and by each other; they never push back, so observations, rewards,
 * done flags and episode statistics are the same bytes with and without them.  `assets_blob` = f64[4][32] (srl_sim/model.py
 * distractor_blob; layout in csrc/distractor_core.h).  Valid only between srl_sim_create and the first reset, and not together with
 * srl_cfg.prefetch_resets.  With the bodies on, `reset_draws` rows are 48 wide: the 18 Kuka values, the 10 placements (x, y) as
 * final positions and the 10 object types (0-2); NULL = all from the env's counter-based stream.  The object types and the kick
 * direction come from the env's stream too (the reference draws them from the global, unseeded np.random).  State: SRL_F_DISTRACTORS.
 * The CPU oracle library has no body dynamics: it exports this entry point and always returns 1. */
int srl_sim_set_distractors(srl_sim* sim, const void* assets_blob, size_t bytes);

/* Image observations (`srl_model = "raw_pixels"`): what the reference obtains per env from PyBullet's TinyRenderer in render(mode='rgb_array')
 * (environments/kuka_gym/kuka_button_gym_env.py:370-420, environments/mobile_robot/mobile_robot_env.py:287-334).  The camera is given the way
 * the reference gives it to computeViewMatrixFromYawPitchRoll (upAxisIndex = 2) / computeProjectionMatrixFOV; rows run top to bottom like
 * getCameraImage's.  One frame of `width` x `height` RGB bytes per env: rgb_out is u8[N, height, width, 3] (device pointer for the CUDA
 * library).  The scene is drawn from analytic primitives (the pybullet_data meshes and textures are not available): same camera and
 * layout as the reference, not TinyRenderer's pixels -- see csrc/render_core.h. */
typedef struct srl_camera {
    float target[3];            /* cameraTargetPosition                                         */
    float distance, yaw, pitch, roll;   /* degrees                                              */
    float fov;                  /* vertical field of view in degrees; aspect = width / height   */
} srl_camera;
int srl_sim_render(srl_sim* sim, const srl_camera* camera, int width, int height, uint8_t* rgb_out, void* stream);

/* One camera per env: cameras[i] draws env i (host array of N srl_camera, like srl_sim_render's camera).  follow_robot != 0
 * (MobileRobot kinds only): the x and y of each camera's target are offsets from that env's robot position at the time of the call,
 * computed as float32(float64 robot position + float64(offset)); the target's z stays absolute.  This is the reference's fpv camera
 * (mobile_robot_env.py:316-326) with target offset (-0.25, 0, 0.15).  Output layout and frame contents as srl_sim_render: env i's frame
 * is the bytes srl_sim_render(cameras[i]) gives it (with follow_robot: the camera with the absolute target).  The robot positions are read
 * on the device.  The handle keeps the cameras it built last and reuses them when a call passes the same array (bytes), size and
 * follow_robot again, so a caller that renders through fixed cameras every step pays no per-call host set-up.  The CPU oracle library
 * implements it too, on host arrays. */
int srl_sim_render_cameras(srl_sim* sim, const srl_camera* cameras, int follow_robot, int width, int height,
                           uint8_t* rgb_out, void* stream);

/* Debug / single-env accessors (host arrays, synchronising; not on the hot path).  Derived link-state fields
 * (SRL_F_ROBOT_POS, SRL_F_EE_POS) reflect the last step or reset; they are not recomputed by set_state. */
int srl_sim_get_state(srl_sim* sim, int field, void* dst, size_t bytes);
int srl_sim_set_state(srl_sim* sim, int field, const void* src, size_t bytes);

/* Number of kernel launches issued by this handle so far (bench.py's gpu_launches). */
uint64_t srl_sim_launch_count(const srl_sim* sim);

/* Device time (ms) of the most recent step/rollout kernel, measured with CUDA events on the
 * launching stream; blocks until that kernel has finished.  < 0 on error. */
float srl_sim_last_kernel_ms(srl_sim* sim);

int srl_sim_num_envs(const srl_sim* sim);
int srl_sim_obs_dim(const srl_sim* sim);
int srl_sim_action_dim(const srl_sim* sim); /* 1 for discrete */

const char* srl_sim_last_error(void);
void srl_sim_destroy(srl_sim* sim);

#ifdef __cplusplus
}
#endif
#endif /* SRL_SIM_H_ */
