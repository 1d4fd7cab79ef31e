/*
 * srl_policy.h -- C-ABI of the helpers a GPU-resident PPO2 consumer needs next to srl_sim_step (same shared library,
 * libsrl_sim_b200.so): the policy step and the observation filter of the collection loop, and the minibatch gradient of the update.  They belong to the
 * CONSUMER of the simulator (SURVEY.md 8(f).1), not to the environment boundary of include/srl_sim.h.
 *
 * Reference interfaces they replace (paths relative to the reference repo):
 *   srl_policy_act  <- stable-baselines 2.5 `PPO2` runner's `model.step(obs)` with `MlpPolicy` (two separate 64-64 tanh
 *                      towers), chosen by rl_baselines/rl_algorithm/ppo2.py:58-72; one call per env step:
 *                      policy forward, sample, log-probability, value, rollout-buffer writes
 *   srl_ppo2_grad   <- the loss + `tf.gradients` of stable-baselines 2.5 `PPO2.setup_model`, run once per minibatch by `PPO2._train_step`
 *   srl_obs_filter  <- stable-baselines `VecNormalize._obfilt` (norm_obs=True, clip_obs=10), wrapped around the envs
 *                      by rl_baselines/utils.py:224-227: running mean / variance update + normalisation
 *   srl_obs_stack_filter <- `VecFrameStack(envs, num_stack)` -> `VecNormalize` (rl_baselines/utils.py:222-227): the frame stack
 *                      step and the filter of the stacked rows in one launch
 *   srl_a2c_grad    <- the loss + `tf.gradients` of stable-baselines 2.5 `A2C.setup_model`, run once per update by `A2C._train_step`
 *                      (chosen by rl_baselines/rl_algorithm/a2c.py)
 *   srl_clip_rmsprop <- the same `_train_step`'s `tf.clip_by_global_norm` + `tf.train.RMSPropOptimizer` apply op
 *   srl_dqn_act, srl_replay_add, srl_replay_sample, srl_dqn_target, srl_dqn_grad, srl_replay_update, srl_clip_adam
 *                   <- stable-baselines 2.5 `DQN.learn` with the deepq `MlpPolicy` (chosen by rl_baselines/rl_algorithm/deepq.py): the
 *                      epsilon-greedy `act`, baselines' `PrioritizedReplayBuffer` (add, sample, update_priorities) and `build_train`'s double-Q
 *                      loss, `tf.clip_by_norm` per gradient tensor and `tf.train.AdamOptimizer`
 *   srl_sac_act, srl_sac_store, srl_sac_prepare, srl_sac_grad, srl_sac_adam
 *                   <- stable-baselines 2.5 `SAC.learn` with its `MlpPolicy` (chosen by rl_baselines/rl_algorithm/sac.py): the policy step,
 *                      `ReplayBuffer.add` / `sample`, the losses and `tf.gradients` of `SAC.setup_model`, its three `tf.train.AdamOptimizer`s
 *                      and the Polyak target update
 *
 * Conventions are those of srl_sim.h: 0 on success, message from srl_sim_last_error(); all pointers are DEVICE pointers;
 * calls are asynchronous on `stream` and capturable into a CUDA graph (everything a launch reads that changes between
 * replays -- weights, filter state, RNG counter -- lives in device memory).
 */
#ifndef SRL_POLICY_H_
#define SRL_POLICY_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* stable-baselines MlpPolicy: separate policy / value towers obs_dim -> 64 -> 64 -> n_out / 1, tanh.
 * Weights in torch.nn.Linear layout: weight [out][in] row-major float32, bias [out]. */
typedef struct srl_mlp_policy {
    uint32_t struct_size;   /* = sizeof(srl_mlp_policy); checked                          */
    int32_t  obs_dim;       /* 1..32 (1..8 and 9..32 run separate kernel instantiations)  */
    int32_t  n_out;         /* Discrete: number of actions (2..8); Box: action dim (1..8) */
    int32_t  discrete;      /* 1 = Categorical(logits), 0 = Normal(mean, exp(logstd))     */
    const float *pi_w1, *pi_b1, *pi_w2, *pi_b2, *pi_w3, *pi_b3;
    const float *vf_w1, *vf_b1, *vf_w2, *vf_b2, *vf_w3, *vf_b3;
    const float *logstd;    /* Box only: [n_out]                                          */
} srl_mlp_policy;

/* One policy step for n envs.
 *   obs      : f32[n, obs_dim], already normalised
 *   rng      : u64[3] device words {seed, step counter, 0}; env i samples from the Philox stream
 *              (seed, env_offset + i, counter); the launch advances the counter by one when its last CTA retires
 *   obs_buf  : nullable f32[n, obs_dim], copy of obs (rollout buffer row)
 *   act_env  : i32[n] (Discrete) / f32[n, n_out] clipped to [-1, 1] (Box): the action for srl_sim_step
 *   act_buf  : nullable i64[n] / f32[n, n_out] unclipped sample (rollout buffer row)
 *   logp, value : f32[n] */
int srl_policy_act(const srl_mlp_policy* policy, int n, const float* obs, uint64_t* rng, uint64_t env_offset,
                   float* obs_buf, void* act_env, void* act_buf, float* logp, float* value, void* stream);

/* VecNormalize's observation filter for one batch.
 *   state : f64[2 * obs_dim + 1] device words {mean[obs_dim], var[obs_dim], count}
 *   update != 0: fold the batch moments of `obs_raw` into the state first (parallel-variance merge), then
 *   out = clip((obs_raw - mean) / sqrt(var + eps), -clip, clip) in float32.  obs_dim <= 8. */
int srl_obs_filter(int n, int obs_dim, const float* obs_raw, double* state, int update, float clip, float eps,
                   float* obs_norm_out, void* stream);

/* VecFrameStack (stable-baselines 2.5) followed by VecNormalize's filter of the stacked rows, in one launch.  W = obs_dim * num_stack,
 * 1 <= W <= 32; rows are oldest frame first.
 *   obs_raw : f32[n, obs_dim], the observation of this step (for a done env: the first one of its next episode)
 *   done    : nullable u8[n]; NULL means reset: every row starts from zeros
 *   stack   : f32[n, W], updated in place: roll left by obs_dim, zero the row where done[i] != 0 (every row when done is NULL), write
 *             obs_raw into the last obs_dim columns
 *   state   : f64[2 * W + 1] {mean[W], var[W], count}; update != 0 folds the new stack rows (zeros included) into it first
 *   obs_norm_out : f32[n, W] = clip((stack - mean) / sqrt(var + eps), -clip, clip), as srl_obs_filter computes it */
int srl_obs_stack_filter(int n, int obs_dim, int num_stack, const float* obs_raw, const uint8_t* done, float* stack, double* state, int update,
                         float clip, float eps, float* obs_norm_out, void* stream);

/* Gradient tensors of an MlpPolicy, same shapes and layout as the weights (torch: `param.grad`, contiguous float32). */
typedef struct srl_mlp_grads {
    uint32_t struct_size;   /* = sizeof(srl_mlp_grads); checked */
    uint32_t reserved;
    float *pi_w1, *pi_b1, *pi_w2, *pi_b2, *pi_w3, *pi_b3;
    float *vf_w1, *vf_b1, *vf_w2, *vf_b2, *vf_w3, *vf_b3;
    float *logstd;          /* Box only */
} srl_mlp_grads;

/* The gradient of stable-baselines' PPO2 loss over one minibatch, in one pass: what `loss.backward()` leaves in `param.grad` for
 *   loss = pg_loss - ent_coef * entropy + vf_coef * vf_loss     (PPO2.setup_model of stable-baselines 2.5, chosen by
 *                                                                 rl_baselines/rl_algorithm/ppo2.py:58-72 of the reference)
 *   A = (adv - mean(adv)) / (std(adv) + 1e-8) over the minibatch, ratio = exp(logp - old_logp),
 *   pg_loss = mean(max(-A ratio, -A clip(ratio, 1 - c, 1 + c))),
 *   vf_loss = 0.5 mean(max((v - ret)^2, (old_value + clip(v - old_value, -c, c) - ret)^2)).
 * Gradient clipping and the optimiser step stay with the caller.
 *   idx        : nullable i64[minibatch] row indices into the rollout arrays (NULL: rows 0 .. minibatch - 1)
 *   obs        : f32[rows, obs_dim]; actions : i64[rows] (Discrete) / f32[rows, n_out] (Box, the unclipped samples)
 *   adv, ret, old_logp, old_value : f32[rows]
 *   workspace  : device memory of at least srl_ppo2_workspace_bytes(...) bytes (per-CTA partial gradients; no state between calls)
 * The gradient tensors are OVERWRITTEN (not accumulated).  Deterministic: partial sums are combined in a fixed order. */
size_t srl_ppo2_workspace_bytes(int obs_dim, int n_out, int discrete, int minibatch);   /* 0 for an unsupported shape */
int srl_ppo2_grad(const srl_mlp_policy* policy, const srl_mlp_grads* grads, int minibatch, const int64_t* idx, const float* obs,
                  const void* actions, const float* adv, const float* ret, const float* old_logp, const float* old_value,
                  float cliprange, float ent_coef, float vf_coef, void* workspace, size_t workspace_bytes, void* stream);

/* The gradient of stable-baselines 2.5's A2C loss over `rows` rows, written into `grads` like srl_ppo2_grad (same kernels and chunking, same
 * deterministic CTA-order reduction; only the per-sample loss derivative differs):
 *   ADV = ret - old_value (not normalised), pg_loss = mean(-ADV logp(a)), vf_loss = 0.5 mean((v - ret)^2),
 *   loss = pg_loss - ent_coef * mean(entropy) + vf_coef * vf_loss.
 * RECALLED, not checked against an installed stable-baselines (none can be installed here; re-pin these when one is): the 0.5 of vf_loss
 * (`mse()` of stable_baselines/a2c/utils.py divides by 2), and that A2C clips neither the value nor the probability ratio.
 *   idx : nullable i64[rows] row indices (NULL: rows 0 .. rows - 1); obs, actions, ret, old_value as for srl_ppo2_grad
 *   workspace : at least srl_a2c_workspace_bytes(...) bytes (per-CTA partial gradients; no state between calls) */
size_t srl_a2c_workspace_bytes(int obs_dim, int n_out, int discrete, int rows);   /* 0 for an unsupported shape */
int srl_a2c_grad(const srl_mlp_policy* policy, const srl_mlp_grads* grads, int rows, const int64_t* idx, const float* obs, const void* actions,
                 const float* ret, const float* old_value, float ent_coef, float vf_coef, void* workspace, size_t workspace_bytes, void* stream);

/* One optimiser step of stable-baselines' A2C over every tensor of an MlpPolicy, in one launch:
 *   tf.clip_by_global_norm(grads, max_grad_norm): norm = sqrt(sum of every squared gradient entry), scale = max_grad_norm / max(norm, max_grad_norm);
 *     a NaN or infinite norm makes the scale NaN, so one non-finite gradient entry turns every parameter NaN (TF's behaviour);
 *   tf.train.RMSPropOptimizer(lr, decay=alpha, epsilon, momentum=0) on g = scale * grad:
 *     ms <- ms + (g^2 - ms) (1 - alpha);   param <- param - lr g / sqrt(ms + epsilon).
 * RECALLED from TF 1.x, not checked against an installed TF: the `ms` slot starts at 1.0 (not 0; the caller initialises it), and epsilon sits
 * inside the square root.  This is not torch.optim.RMSprop.
 *   params, grads, ms : the tensors of the policy, its gradients and the RMSProp slot, each in the layout of srl_mlp_grads for this shape
 *                       (logstd only for Box); params and ms are updated in place, grads are read
 *   lr : f32[1] device scalar (a captured call follows a schedule that rewrites it)
 * The squared norm is summed in float64 in a fixed order: two calls on the same inputs give the same bytes.  No host synchronisation. */
int srl_clip_rmsprop(int obs_dim, int n_out, int discrete, const srl_mlp_grads* params, const srl_mlp_grads* grads, const srl_mlp_grads* ms,
                     const float* lr, float max_grad_norm, float alpha, float epsilon, void* stream);

/* GAE(lambda) over one rollout (the backward recursion of stable-baselines' PPO2 runner): rew, value, done (1.0 where the episode ended at that
 * step), adv_out, ret_out are f32[n_steps, n_envs]; last_value f32[n_envs] is the value of the observation after the last step.
 *   delta_t = rew_t + gamma * V_{t+1} * (1 - done_t) - V_t;  adv_t = delta_t + gamma * lam * (1 - done_t) * adv_{t+1};  ret_t = adv_t + V_t
 * gamma and lam are doubles: the float32 recursion uses fl32(gamma) and fl32(gamma * lam), the coefficients a float32 array expression with
 * Python-float hyper-parameters uses (fl32(gamma) * fl32(lam) is another float for e.g. gamma = lam = 0.9).
 * With lam = 1, ret_t = rew_t + gamma (1 - done_t) ret_{t+1} from ret_{n_steps} = last_value: A2C's bootstrapped n-step returns
 * (stable-baselines' `discount_with_dones` over the rewards followed by the last value). */
int srl_ppo2_gae(int n_steps, int n_envs, const float* rew, const float* value, const float* done, const float* last_value, double gamma, double lam,
                 float* adv_out, float* ret_out, void* stream);

/* ---- DQN (rl_baselines/deepq.py) ----
 * The Q network is an srl_mlp_policy with discrete = 1, n_out = the number of actions (2..8), obs_dim 1..32: the pi tower is the advantage head
 * A (n_out values), the vf tower the state value V, both obs_dim -> 64 -> 64 with ReLU (not tanh), and
 *   Q = V + (A - mean(A)),   mean(A) = (A_0 + ... + A_{n-1}) * (1 / n) in float32, summed in order.
 * RECALLED from stable-baselines 2.5 / baselines, not checked against an installed copy (none can be installed here): the dueling head and the
 * ReLU towers of the deepq MlpPolicy (layers [64, 64], no layer norm), double Q in build_train, the Huber loss with delta 1, tf.clip_by_norm
 * per tensor, TF1 Adam's update order, and baselines' PrioritizedReplayBuffer / SegmentTree.  Every entry point refuses discrete = 0. */

/* The epsilon-greedy step for n envs: Q of obs (f32[n, obs_dim]); env i draws from the Philox stream (seed, env_offset + i, counter) with purpose 24:
 * a 53-bit uniform from words 0-1 below *eps explores, and then the action is (word 2 * n_out) >> 32, otherwise argmax Q (ties: the lowest index).
 *   eps     : f32[1] device scalar;  rng : u64[3] {seed, counter, 0}, the counter advances by one per launch as for srl_policy_act
 *   obs_buf : nullable f32[n, obs_dim] copy of obs;  act_env : i32[n];  act_buf : nullable i64[n];  q_out : nullable f32[n, n_out], Q itself */
int srl_dqn_act(const srl_mlp_policy* q, int n, const float* obs, const float* eps, uint64_t* rng, uint64_t env_offset, float* obs_buf,
                int32_t* act_env, int64_t* act_buf, float* q_out, void* stream);

/* The double-Q target of `batch` sampled transitions: for row g = idx[b] (idx NULL: g = b), b* = argmax Q_online(next_obs[g]) and
 *   y[b] = rew[g] + gamma * ((1 - done[g]) * Q_target(next_obs[g], b*))   (float32, in this order of roundings).
 *   next_obs : f32[rows, obs_dim];  rew : f32[rows];  done : u8[rows];  y : f32[batch] */
int srl_dqn_target(const srl_mlp_policy* online, const srl_mlp_policy* target, int batch, const int64_t* idx, const float* next_obs, const float* rew,
                   const uint8_t* done, float gamma, float* y, void* stream);

/* The gradient of loss = mean(w * huber(td)), td = Q(obs[g], act[g]) - y[b], over `batch` samples, written into `grads` like srl_a2c_grad (the same
 * kernels, chunking and deterministic CTA-order reduction; ReLU towers, and per sample the head derivatives g = w clamp(td, -1, 1) / batch,
 * d/dA_k = g ([k = act] - 1 / n), d/dV = g).
 *   idx : nullable i64[batch] rows;  obs : f32[rows, obs_dim];  actions : i64[rows];  y, weights : f32[batch] in batch order (weights NULL: 1)
 *   td_out : f32[batch], td of every sample;  workspace : at least srl_a2c_workspace_bytes(obs_dim, n_out, 1, batch) bytes (no state between calls) */
int srl_dqn_grad(const srl_mlp_policy* q, const srl_mlp_grads* grads, int batch, const int64_t* idx, const float* obs, const int64_t* actions,
                 const float* y, const float* weights, float* td_out, void* workspace, size_t workspace_bytes, void* stream);

/* One optimiser step of stable-baselines' DQN over every tensor of the Q network (discrete = 1; discrete = 0 is refused), in one launch: per tensor g = t * clip_norm / max(l2norm(t), clip_norm)
 * (tf.clip_by_norm; l2norm summed in float64, rounded to float32; an infinite entry makes that entry NaN and the tensor's others 0, a NaN entry
 * makes the whole tensor NaN; other tensors are unaffected), then TF1 Adam with slots m, v from 0:
 *   m += (g - m)(1 - beta1);  v += (g^2 - v)(1 - beta2);  lr_t = lr sqrt(1 - beta2^t) / (1 - beta1^t);  w -= m lr_t / (sqrt(v) + epsilon)
 * (epsilon outside the square root; not torch.optim.Adam's bias correction).
 *   lr : f32[1] device scalar;  beta_power : f32[2] {beta1^t, beta2^t}, TF's accumulators: the caller starts them at {beta1, beta2}, every call
 *   multiplies them by {beta1, beta2} after its step.  Two calls on the same inputs give the same bytes. */
int srl_clip_adam(int obs_dim, int n_out, int discrete, const srl_mlp_grads* params, const srl_mlp_grads* grads, const srl_mlp_grads* m,
                  const srl_mlp_grads* v, const float* lr, float* beta_power, float clip_norm, float beta1, float beta2, float epsilon, void* stream);

/* Prioritized replay over a ring of capacity = rows * n_envs transitions, row r holding transitions r * n_envs .. r * n_envs + n_envs - 1.
 * Two float64 segment trees (baselines' SegmentTree): node 1 is the root, node k has children 2k and 2k + 1, leaf i sits at tree_cap + i, and
 * every internal node is sum(left, right) / min(left, right).  The caller allocates and initialises the device words: sum 0, min +inf,
 * max_priority 1, size 0, stamp -1. */
typedef struct srl_replay_tree {
    uint32_t struct_size;   /* = sizeof(srl_replay_tree); checked                                      */
    int32_t  n_envs;        /* transitions per ring row                                                */
    int64_t  capacity;      /* transitions the ring holds (a multiple of n_envs)                      */
    int64_t  tree_cap;      /* leaves per tree: the power of two >= capacity                          */
    double*  sum;           /* f64[2 tree_cap] (entry 0 unused)                                        */
    double*  min;           /* f64[2 tree_cap]                                                         */
    double*  max_priority;  /* f64[1]                                                                  */
    int64_t* size;          /* i64[1]: transitions stored                                              */
    int32_t* stamp;         /* i32[capacity]: srl_replay_update's scratch, -1 between calls            */
} srl_replay_tree;

/* The leaves of ring row `row` become max_priority^alpha (float64) in both trees, their ancestors are rebuilt and size becomes
 * max(size, (row + 1) n_envs). */
int srl_replay_add(const srl_replay_tree* t, int64_t row, double alpha, void* stream);

/* `batch` i.i.d. samples; sample b draws a 53-bit uniform u from the Philox stream (seed, b, counter) with purpose 25 (rng as for srl_dqn_act).
 *   prioritized: mass = u * sum[root], then find_prefixsum_idx (left child > mass: go left, else mass -= left, go right); a walk that float64
 *                rounding ends in an empty leaf (index >= size) is clamped to size - 1.  w = (p_i size)^-beta / (p_min size)^-beta with
 *                p = leaf / sum[root], p_min = min[root] / sum[root], in float64, rounded to float32.  beta : f64[1] device scalar.
 *   otherwise:   i = min(floor(u size), size - 1), w = 1.
 *   idx_out : i64[batch];  w_out : f32[batch] */
int srl_replay_sample(const srl_replay_tree* t, int batch, int prioritized, const double* beta, uint64_t* rng, int64_t* idx_out, float* w_out,
                      void* stream);

/* After a gradient step: priority p = |td[b]| + eps in float32, leaf idx[b] = p^alpha in float64 in both trees (a leaf sampled twice takes the
 * priority of its LAST occurrence in the batch), max_priority = max(max_priority, p), then every internal node is rebuilt bottom-up.
 * idx entries must be stored transitions (0 <= idx < size). */
int srl_replay_update(const srl_replay_tree* t, int batch, const int64_t* idx, const float* td, double alpha, float eps, void* stream);

/* ---- SAC (rl_baselines/sac.py) ----
 * stable-baselines 2.5 `SAC` with its `MlpPolicy` (chosen by rl_baselines/rl_algorithm/sac.py).  Five 64-64 ReLU networks, each
 * in -> 64 -> 64 -> out in torch.nn.Linear layout (w1 [64][in], b1 [64], w2 [64][64], b2 [64], w3 [out][64], b3 [out]):
 *   actor     W -> 2A: rows 0..A-1 of w3 / b3 are the `mu` head, rows A..2A-1 the `log_std` head, log_std = clip(., -20, 2)
 *   qf1, qf2  W + A -> 1 on concat(obs, action), obs first
 *   vf        W -> 1;  the target vf has vf's layout in a separate array
 * W = obs_dim 1..32, A = act_dim 1..8.  The parameters live in one flat f32 ARENA in the order actor | qf1 | qf2 | vf | log_ent_coef (one
 * float), each network's six tensors in the order above; srl_sac_arena_floats gives its length P.  The gradient and the Adam slots m, v are
 * arrays of the same layout.
 * RECALLED from stable-baselines 2.5, not checked against an installed copy (none can be installed here): the networks and their init, the
 * log_std clip and its gradient (zero strictly outside [-20, 2], passed at the bounds), the log-probability as the TF graph writes it, the
 * losses and which optimiser owns which variables, TF1 Adam, the Polyak update after the Adam steps, and the learn loop's conditions.
 * Philox purposes (counter word 3; DQN uses 24 and 25): 26, 27 the acting noise of dims 0-3 / 4-7; 28, 29 the uniform random action of
 * dims 0-3 / 4-7; 30 the sample index; 31, 32 the reparameterisation noise of dims 0-3 / 4-7 of a sample.  Gaussian words are those of
 * srl_sample_gaussian (Box-Muller on 24-bit uniforms, dims 4j..4j+3 from one block: cos / sin of words (0, 1), then of words (2, 3)).
 * Every entry point is asynchronous on `stream`, capturable (counters, step, learning rate and log_ent_coef live in device memory) and
 * deterministic (fixed-order reductions). */
typedef struct srl_sac_nets {
    uint32_t struct_size;   /* = sizeof(srl_sac_nets); checked            */
    int32_t  obs_dim;       /* W, 1..32                                    */
    int32_t  act_dim;       /* A, 1..8                                     */
    int32_t  reserved;
    float*   arena;         /* f32[P]: actor | qf1 | qf2 | vf | log_ent_coef */
    float*   target;        /* f32[vf's size]: the target value network    */
} srl_sac_nets;

size_t srl_sac_arena_floats(int obs_dim, int act_dim);   /* P; 0 for an unsupported shape */

/* The action of n envs from the observations obs (f32[n, obs_dim]).  mode 0: sample, a = tanh(mu + std z) with std = exp(clip(log_std)),
 * z_k Gaussian from the Philox stream (seed, env_offset + i, counter) with purposes 26 + k / 4;  mode 1: deterministic, a = tanh(mu);
 * mode 2: uniform random, a_k = 2 (word >> 8) / 2^24 - 1 from word k % 4 of purpose 28 + k / 4 (the network is not evaluated).
 *   rng : u64[3] {seed, counter, 0}; the launch advances the counter by one when its last CTA retires (srl_policy_act's rule)
 *   act_out : f32[n, act_dim], the squashed action for srl_sim_step and the replay ring */
int srl_sac_act(const srl_sac_nets* nets, int n, const float* obs, int mode, uint64_t* rng, uint64_t env_offset, float* act_out, void* stream);

/* The replay ring of `rows` rows of n transitions: row r = (*step) % rows receives obs, act, rew, done and new_obs (ring arrays obs_ring,
 * next_obs_ring f32[rows, n, obs_dim], act_ring f32[rows, n, act_dim], rew_ring f32[rows, n], done_ring u8[rows, n]); then obs <- new_obs
 * in place (the next step's observation) and step[0] += 1.  step : i64[2] {lockstep steps stored, 0} (word 1 counts the launch's retired
 * CTAs).  The row comes from device memory, so one captured launch serves every row. */
int srl_sac_store(int rows, int n, int obs_dim, int act_dim, int64_t* step, float* obs, const float* act, const float* rew, const uint8_t* done,
                  const float* new_obs, float* obs_ring, float* act_ring, float* rew_ring, uint8_t* done_ring, float* next_obs_ring, void* stream);

/* The per-sample part of one gradient step over `batch` samples drawn from the size = min(*step, rows) * n stored transitions:
 *   sample b: u a 53-bit uniform of words 0-1 of the stream (seed, b, counter), purpose 30; g = min(floor(u size), size - 1) -> idx[b]
 *   q_backup[b] = rew[g] + gamma ((1 - done[g]) V_targ(next_obs[g]))
 *   actor at obs[g]: mu, ls = clip(log_std, -20, 2), eps_k Gaussian (stream (seed, b, counter), purposes 31 + k / 4), u = mu + exp(ls) eps,
 *     a_pi = tanh(u), logp[b] = sum_k -0.5 (((u - mu) / (exp(ls) + 1e-6))^2 + 2 ls + log 2 pi) - sum_k log(1 - a_pi^2 + 1e-6)
 *   v_backup[b] = min(qf1(obs, a_pi), qf2(obs, a_pi)) - alpha logp[b],  alpha = exp(log_ent_coef) (auto_ent) or ent_coef
 *   d_actor[b] : f32[batch, 2 act_dim], d policy_loss / d (mu, raw log_std) of the sample, policy_loss = mean(alpha logp - qf1(obs, a_pi)),
 *                through qf1's input gradient; the log_std part is 0 where the raw head is outside [-20, 2]
 *   ent_grad : f32[1], d ent_coef_loss / d log_ent_coef = -mean(logp + target_entropy), summed in float64 in a fixed order (0 unless auto_ent);
 *              it may point at log_ent_coef's entry of the gradient arena.  rng as for srl_sac_act (its own record).
 * With nothing stored (step[0] == 0) every idx[b] is -1 and every output is 0; srl_sac_grad then writes a zero gradient. */
int srl_sac_prepare(const srl_sac_nets* nets, int rows, int n, const int64_t* step, const float* obs_ring, const float* act_ring, const float* rew_ring,
                    const uint8_t* done_ring, const float* next_obs_ring, int batch, float gamma, int auto_ent, float ent_coef, float target_entropy,
                    uint64_t* rng, int64_t* idx, float* q_backup, float* v_backup, float* logp, float* d_actor, float* ent_grad, void* workspace,
                    size_t workspace_bytes, void* stream);

/* The weight gradients of one step, written into `grad` (f32[P], every entry but log_ent_coef's, which srl_sac_prepare writes):
 *   actor from d_actor;  qf_i from qf_i_loss = 0.5 mean((q_backup - qf_i(obs, act))^2) at the STORED action;  vf from
 *   value_loss = 0.5 mean((vf(obs) - v_backup)^2).  Each network's forward pass is recomputed in chunks of 64 samples with every activation
 *   in shared memory; per-CTA partial gradients are summed in float64 in CTA order.  idx, q_backup, v_backup, d_actor as srl_sac_prepare left them.
 *   workspace : at least srl_sac_workspace_bytes(obs_dim, act_dim, batch) bytes (shared with srl_sac_prepare; no state between calls) */
size_t srl_sac_workspace_bytes(int obs_dim, int act_dim, int batch);
int srl_sac_grad(const srl_sac_nets* nets, int n, const float* obs_ring, const float* act_ring, int batch, const int64_t* idx, const float* q_backup,
                 const float* v_backup, const float* d_actor, float* grad, void* workspace, size_t workspace_bytes, void* stream);

/* TF1 Adam over the whole arena in srl_clip_adam's statement and order of roundings (no clipping), then, when `polyak`, the target update
 * target = (1 - tau) target + tau vf from the updated vf, in float32:  m += (g - m)(1 - beta1); v += (g^2 - v)(1 - beta2);
 * lr_t = lr sqrt(1 - beta2^t) / (1 - beta1^t); w -= m lr_t / (sqrt(v) + epsilon).  One launch; the three optimisers of stable-baselines'
 * SAC step together, so one beta_power f32[2] {beta1^t, beta2^t} serves them all (multiplied by {beta1, beta2} after the step).  lr : f32[1]. */
int srl_sac_adam(const srl_sac_nets* nets, const float* grad, float* m, float* v, const float* lr, float* beta_power, float beta1, float beta2,
                 float epsilon, int polyak, float tau, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SRL_POLICY_H_ */
