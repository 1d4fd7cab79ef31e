"""
PPO2 consumer of the batched simulator (SURVEY.md section 8(f).1, BASELINE config 3).

The reference trains with stable-baselines' TF-1.8 ``PPO2`` through ``rl_baselines/rl_algorithm/ppo2.py:58-73`` and
``rl_baselines/base_classes.py:214-253``; neither TensorFlow nor stable-baselines exists in this image, so the algorithm is
restated in PyTorch with the reference's hyper-parameters (n_steps=128, nminibatches=4, noptepochs=4, lr=2.5e-4 * f,
ent_coef=0.01, vf_coef=0.5, cliprange=0.2, gamma=0.99, lam=0.95, max_grad_norm=0.5) and stable-baselines' ``MlpPolicy``
(two separate 64-64 tanh networks for policy and value).  Everything -- envs, observation normalisation
(``VecNormalize(norm_obs=True, norm_reward=False)``, rl_baselines/utils.py:224-227), policy, GAE, optimisation -- stays on the
GPU: the env step is ``srl_sim_step`` on torch tensors, no host round trip per step.
This is a CONSUMER of the hot path (library GEMMs via torch are fine here); the product is the simulator underneath.

Data-parallel over GPUs (SURVEY.md section 8(e)): under ``torchrun`` every rank owns ``num_envs`` envs (global env offset
``rank * num_envs``, so env streams do not depend on the GPU count) and a replica of the policy.  Two collectives, none of
them on the env-step path: ONE all-reduce of the flattened ~10^4-parameter gradient per minibatch, and ONE all-reduce of the
observation filter's sufficient statistics ([2 D + 1] float64) per rollout.  NCCL on GPUs, gloo in the CPU tests.
"""
import json
import os
import time

import numpy as np
import torch
import torch.nn as nn

from srl_sim.vec_env import BatchedSRLVecEnv

PPO2_DEFAULTS = dict(n_steps=128, ent_coef=0.01, learning_rate=2.5e-4, vf_coef=0.5, max_grad_norm=0.5, gamma=0.99, lam=0.95,
                     nminibatches=4, noptepochs=4, cliprange=0.2)   # rl_algorithm/ppo2.py:58-72


class MlpPolicy(nn.Module):
    """stable-baselines 2.5 ``MlpPolicy``: separate pi / vf towers, 2 x 64 tanh, orthogonal init."""

    def __init__(self, obs_dim, n_actions=None, action_dim=None):
        super().__init__()
        self.discrete = n_actions is not None
        out = n_actions if self.discrete else action_dim

        def tower(last, gain):
            layers = [nn.Linear(obs_dim, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, last)]
            for m in layers:
                if isinstance(m, nn.Linear):
                    nn.init.orthogonal_(m.weight, np.sqrt(2)); nn.init.zeros_(m.bias)
            nn.init.orthogonal_(layers[-1].weight, gain)
            return nn.Sequential(*layers)
        self.pi, self.vf = tower(out, 0.01), tower(1, 1.0)
        if not self.discrete:
            self.logstd = nn.Parameter(torch.zeros(out))

    def dist(self, obs):
        logits = self.pi(obs)
        if self.discrete:
            return torch.distributions.Categorical(logits=logits, validate_args=False)   # validation synchronises: not allowed in a captured graph
        return torch.distributions.Normal(logits, self.logstd.exp(), validate_args=False)

    def act(self, obs):
        d = self.dist(obs)
        a = d.sample()
        logp = d.log_prob(a) if self.discrete else d.log_prob(a).sum(-1)
        return a, logp, self.vf(obs).squeeze(-1)

    def evaluate(self, obs, actions):
        d = self.dist(obs)
        logp = d.log_prob(actions) if self.discrete else d.log_prob(actions).sum(-1)
        ent = d.entropy() if self.discrete else d.entropy().sum(-1)
        return logp, ent, self.vf(obs).squeeze(-1)


class RunningNorm(object):
    """VecNormalize's observation filter on the device: running mean / var, clip to +-10.  All of its state (the sample
    count included) lives in device tensors and is updated in place, so the update can sit inside a captured CUDA graph."""

    def __init__(self, dim, device, clip=10.0, eps=1e-8):
        # one contiguous float64 record {mean[dim], var[dim], count} (the layout srl_obs_filter updates in place); the attributes are views
        self.state = torch.cat([torch.zeros(dim, dtype=torch.float64), torch.ones(dim, dtype=torch.float64),
                                torch.full((1,), 1e-4, dtype=torch.float64)]).to(device)
        self.mean, self.var, self.count = self.state[:dim], self.state[dim:2 * dim], self.state[2 * dim]
        self.clip, self.eps = clip, eps

    def update(self, x):
        x = x.double()
        bm, bv, bc = x.mean(0), x.var(0, unbiased=False), float(x.shape[0])
        delta, tot = bm - self.mean, self.count + bc
        new_var = (self.var * self.count + bv * bc + delta ** 2 * self.count * bc / tot) / tot
        self.mean.add_(delta * bc / tot)
        self.var.copy_(new_var)
        self.count.copy_(tot)

    def __call__(self, x, update=True):
        if update:
            self.update(x)
        return torch.clamp((x - self.mean.float()) / torch.sqrt(self.var.float() + self.eps), -self.clip, self.clip)


def _dist_world():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist, dist.get_rank(), dist.get_world_size()
    return None, 0, 1


def merge_running_moments(norm, prior, all_reduce_sum, world):
    """Merge the per-rank observation filters after a rollout.  Every rank started the rollout from the same ``prior`` =
    (mean, var, count) and folded its own batches in; the sufficient statistics S = (count, count * mean, count * (var + mean^2))
    are additive, so the filter that saw every rank's batches is  sum_r S_r - (world - 1) * S_prior.  One all-reduce of
    2 D + 1 doubles; the result is identical on every rank."""
    def stats(mean, var, count):
        return torch.cat([count.reshape(1), count * mean, count * (var + mean * mean)])
    d = norm.mean.numel()
    s = stats(norm.mean, norm.var, norm.count)
    all_reduce_sum(s)
    s = s - (world - 1) * stats(*prior)
    count, mean = s[0], s[1:1 + d] / s[0]
    norm.count.copy_(count)
    norm.mean.copy_(mean)
    norm.var.copy_(torch.clamp(s[1 + d:] / count - mean * mean, min=0.0))


def allreduce_mean_gradients(params, dist, world):
    """Average the gradients over ranks with ONE collective: flatten, all-reduce (sum), scale, scatter back."""
    grads = [p.grad for p in params]
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat)
    flat.div_(world)
    off = 0
    for g in grads:
        n = g.numel()
        g.copy_(flat[off:off + n].view_as(g))
        off += n


# ---- pieces shared with rl_baselines/a2c.py: the run's envs, policy and first observation, the collection loop, and the per-update
#      bookkeeping (monitor log, episode statistics, best-model callback, saved model and run files) ----

def make_run(algo, env_id, num_envs, seed, env_kwargs, device, prefetch_resets, num_stack, fused_flags, network=None):
    """The envs of this process (global env offset ``rank * num_envs``) and a policy over rows of ``num_stack * D`` values, identical on
    every rank.  ``fused_flags``: the trainer's fused-path switches (None: on whenever the envs live on a GPU); rows wider than the fused
    kernels take are refused when any is on.  ``network(width, env)``: builds another network than the MlpPolicy (rl_baselines/deepq.py's Q
    network); it becomes ``run.policy``.  Call after ``torch.manual_seed(seed)``; reseeds with ``seed + rank`` when data-parallel."""
    env_kwargs = dict(env_kwargs or {})
    dist, rank, world = _dist_world()
    if prefetch_resets is None:
        from srl_sim.backend import default_backend
        prefetch_resets = default_backend(device).on_gpu
    if prefetch_resets:
        env_kwargs["prefetch_resets"] = True
    if env_kwargs.get("srl_model", "ground_truth") != "ground_truth":
        # the collection loop feeds the simulator's observation buffer (the 3-D / 2-D ground-truth observation) straight to the policy
        raise ValueError("%s.train supports srl_model='ground_truth' only (got %r)" % (algo, env_kwargs["srl_model"]))
    import types
    from rl_baselines.utils import createTensorEnvs
    env = createTensorEnvs(types.SimpleNamespace(env=env_id, num_cpu=num_envs, seed=seed, device=device), env_kwargs=env_kwargs,
                           global_env_offset=rank * num_envs)
    on_gpu = env.backend.on_gpu
    # device -1 is the CPU oracle installed by a test through srl_sim.backend.use_library (its buffers are numpy arrays,
    # shared with torch below); the product backend is always a CUDA device
    dev = env.backend.torch_device if on_gpu else torch.device("cpu")
    e_obs, e_rew, e_done, e_ep_ret, e_ep_len = [x if on_gpu else torch.from_numpy(x) for x in (env._obs, env._rew, env._done, env._ep_ret, env._ep_len)]
    D = env.observation_space.shape[0]
    K = int(num_stack)
    if K < 1:
        raise ValueError("num_stack must be >= 1 (got %d)" % K)
    W = K * D                                  # the width of what the policy sees: the stacked row
    if W > 32 and any(on_gpu if f is None else f for f in fused_flags):
        from srl_sim.policy import MAX_OBS
        raise ValueError("num_stack=%d x %d-wide observations = %d: the fused policy kernels take at most %d values per row" % (K, D, W, MAX_OBS))
    if network is not None:
        policy = network(W, env).to(dev)
    elif env.is_discrete:
        policy = MlpPolicy(W, n_actions=env.action_space.n).to(dev)
    else:
        policy = MlpPolicy(W, action_dim=env.action_space.shape[0]).to(dev)
    if dist is not None:
        for p in policy.parameters():         # same seed => same init; the broadcast makes it independent of library versions
            dist.broadcast(p.data, 0)
        torch.manual_seed(seed + rank)        # action sampling / minibatch permutations differ per rank
    return types.SimpleNamespace(algo=algo, env_id=env_id, num_envs=num_envs, env=env, env_kwargs=env_kwargs, prefetch_resets=prefetch_resets,
                                 on_gpu=on_gpu, dev=dev, e_obs=e_obs, e_rew=e_rew, e_done=e_done, e_ep_ret=e_ep_ret, e_ep_len=e_ep_len,
                                 D=D, K=K, W=W, policy=policy, dist=dist, rank=rank, world=world)


def write_run_files(run, log_dir, num_timesteps, seed, hp):
    """args.json and env_globals.json of the run directory (rank 0; rl_baselines/train.py:282-315 of the reference)."""
    if log_dir and run.rank == 0:
        os.makedirs(log_dir, exist_ok=True)
        with open(os.path.join(log_dir, "args.json"), "w") as f:       # train.py:282-283
            json.dump(dict(env=run.env_id, algo=run.algo, num_cpu=run.num_envs, num_timesteps=num_timesteps, seed=seed, srl_model="ground_truth",
                           num_stack=run.K, **hp), f)
        with open(os.path.join(log_dir, "env_globals.json"), "w") as f:  # train.py:285-315
            json.dump({k: v for k, v in run.env_kwargs.items() if isinstance(v, (int, float, str, bool))}, f)


def first_observation(run, norm):
    """Reset every env; returns (the filtered observation, updated in place by the collection loop; the frame stack or None)."""
    env, N, D, W = run.env, run.num_envs, run.D, run.W
    env.sim.reset(obs_out=env._obs, stream=env.backend.stream())
    row, stack = run.e_obs, None          # what the filter sees: the observation, or the frame stack over it
    if run.K > 1:                         # VecFrameStack.reset: zeros, the first observation in the last D columns
        stack = torch.zeros((N, W), device=run.dev)
        stack[:, W - D:].copy_(run.e_obs)
        row = stack
    if run.dist is not None:              # the reset batch goes through the same merge, so every rank starts from one filter
        prior = (norm.mean.clone(), norm.var.clone(), norm.count.clone())
        norm.update(row)
        merge_running_moments(norm, prior, run.dist.all_reduce, run.world)
        obs = norm(row.clone(), update=False)
    else:
        obs = norm(row.clone())
    return obs, stack


def collect_rollout(run, norm, obs, stack, buf, last_val, fused=None, act_dev=None, done_u8=None):
    """T lockstep env steps under the current policy into the [T, N, ...] rollout buffers ``buf``; everything stays on the device, nothing
    synchronises.  With ``fused`` (srl_sim.policy.FusedPolicy) an env step is three launches -- policy step, simulator step, observation
    filter (the frame stack in the same launch) -- and the simulator writes reward / done / episode return straight into the buffers;
    otherwise the policy and the filter run in torch."""
    env, policy, D, W = run.env, run.policy, run.D, run.W
    T, N = buf["rew"].shape
    with torch.no_grad():
        if fused is not None:
            st = env.backend.stream()          # torch's current stream: the capture's while a graph is captured
            for t in range(T):
                fused.act(N, obs, act_dev, buf["logp"][t], buf["val"][t], obs_buf=buf["obs"][t], act_buf=buf["act"][t], stream=st)
                env.sim.step(act_dev, None, env._obs, buf["rew"][t], done_u8[t], buf["ep_ret"][t], buf["ep_len"][t], stream=st)
                if run.K > 1:
                    fused.stack_filter(N, env._obs, done_u8[t], stack, obs, update=True, stream=st)
                else:
                    fused.filter(N, env._obs, obs, update=True, stream=st)
            buf["done"].copy_(done_u8)
        else:
            for t in range(T):
                a, logp, v = policy.act(obs)
                buf["obs"][t], buf["act"][t], buf["logp"][t], buf["val"][t] = obs, a, logp, v
                a_env = a.to(torch.int32) if env.is_discrete else torch.clamp(a, -1, 1).contiguous()
                env.step_tensors(a_env)                                   # one kernel launch, tensors stay on the GPU
                buf["rew"][t], buf["done"][t], buf["ep_ret"][t], buf["ep_len"][t] = run.e_rew, run.e_done.float(), run.e_ep_ret, run.e_ep_len
                if run.K > 1:                                             # VecFrameStack.step: roll by one frame, zero where done, newest frame last
                    stack.copy_(torch.where(run.e_done.bool()[:, None], 0.0, torch.roll(stack, -D, 1)))
                    stack[:, W - D:].copy_(run.e_obs)
                    obs.copy_(norm(stack))
                else:
                    obs.copy_(norm(run.e_obs))
        last_val.copy_(policy.vf(obs).squeeze(-1))


def phase_timer(phase_times, on_gpu):
    """tick(name, since): with a ``phase_times`` dict, synchronise and add the wall time since ``since`` to ``phase_times[name]``."""
    def tick(name=None, since=0.0):
        if phase_times is None:
            return 0.0
        if on_gpu:
            torch.cuda.synchronize()
        now = time.perf_counter()
        if name is not None:
            phase_times[name] = phase_times.get(name, 0.0) + now - since
        return now
    return tick


class RunLog(object):
    """The bookkeeping of a training run after each update: the monitor log (environments/utils.py:53-54 wraps every env in bench.Monitor;
    rl_baselines/visualize.py:59-107 reads the files back: one ``<rank>.monitor.csv`` per process with the episodes of all its envs, return
    and length straight from the kernel's episode statistics), the history of (steps, mean return of the last episodes, fps), the reference's
    best-model callback (rl_baselines/train.py:132-159: every ``save_interval`` updates the mean return of the last N_EPISODES_EVAL episodes
    of the monitor logs is computed, and when it beats the best so far and MIN_EPISODES_BEFORE_SAVE episodes exist the observation filter
    and the model are saved as ``<algo>_model.pt``) and the files of the finished run."""
    N_EPISODES_EVAL, MIN_EPISODES_BEFORE_SAVE = 100, 100

    def __init__(self, run, norm, log_dir, save_interval, episode_window, verbose):
        self.run, self.norm, self.log_dir, self.save_interval, self.episode_window, self.verbose = run, norm, log_dir, save_interval, episode_window, verbose
        self.history, self.ep_returns = [], []
        self.best_mean_reward, self.n_saved = -10000.0, 0
        self.monitor = None
        if log_dir:
            from srl_sim.monitor import MonitorWriter
            os.makedirs(log_dir, exist_ok=True)
            self.monitor = MonitorWriter(os.path.join(log_dir, str(run.rank)), env_id=run.env_id)
        self.t_start = time.time()

    def start(self):
        self.t_start = time.time()

    def episodes(self, done, ep_ret, ep_len):
        """The episodes that ended in the [steps, N] rows since the last call; their monitor times are spread over the wall time since then."""
        dmask = done.bool()
        new_rets = ep_ret[dmask].tolist()
        self.ep_returns.extend(new_rets)
        if self.monitor is not None and new_rets:
            t_now = time.time() - self.monitor.t_start
            t_idx = dmask.nonzero()[:, 0].float()                          # step index of each finished episode within the rows
            t_prev = getattr(self.monitor, "_t_prev", 0.0)
            self.monitor.write_episodes(new_rets, ep_len[dmask].tolist(), (t_prev + (t_now - t_prev) * (t_idx + 1.0) / done.shape[0]).tolist())
            self.monitor._t_prev = t_now

    def end_update(self, update, n_updates, steps, callback=True, print_every=1):
        """History entry of update ``update`` (1-based) at ``steps`` global env steps, then -- with ``callback`` -- the best-model check when
        the update is a multiple of ``save_interval``, then the progress line every ``print_every`` updates."""
        run = self.run
        fps = steps / (time.time() - self.t_start)
        window = self.ep_returns[-max(self.episode_window, run.num_envs):]   # --episode_window (train.py:182), at least one episode per env
        if run.dist is not None:
            from srl_sim.distributed import allgather_episode_stats
            mean_ret, n_ep = allgather_episode_stats(float(np.sum(window)), len(window), device=run.dev if run.on_gpu else None)
            mean_ret = mean_ret if n_ep else float("nan")
        else:
            mean_ret = float(np.mean(window)) if window else float("nan")
        self.history.append((steps, mean_ret, fps))
        if callback and self.log_dir and update % self.save_interval == 0:
            if run.dist is not None:
                run.dist.barrier()             # every rank's monitor file holds this update's episodes
            if run.rank == 0:
                if run.dist is None:           # one process: the in-memory list is the monitor file (same episodes, same order)
                    ok, n_episodes = len(self.ep_returns) > 0, len(self.ep_returns)
                    eval_reward = float(np.mean(self.ep_returns[-self.N_EPISODES_EVAL:])) if ok else 0.0
                else:
                    from srl_sim.monitor import compute_mean_reward
                    ok, eval_reward, n_episodes = compute_mean_reward(self.log_dir, self.N_EPISODES_EVAL)
                if ok and self.verbose:
                    print("Best mean reward: {:.2f} - Last mean reward per episode: {:.2f}".format(self.best_mean_reward, eval_reward))
                if ok and eval_reward > self.best_mean_reward and n_episodes >= self.MIN_EPISODES_BEFORE_SAVE:
                    self.best_mean_reward = eval_reward
                    if self.verbose:
                        print("Saving new best model")
                    self.save_model(os.path.join(self.log_dir, "%s_model.pt" % run.algo))
                    self.n_saved += 1
        if self.verbose and run.rank == 0 and (update == n_updates or update % print_every == 0):
            print("update %d/%d  steps %d  mean episode return %.3f  episodes %d  fps %.0f" % (update, n_updates, steps, mean_ret, len(self.ep_returns), fps))

    def save_model(self, path):
        from rl_baselines.utils import save_obs_rms
        norm = self.norm
        torch.save(dict(policy=self.run.policy.state_dict(), obs_mean=norm.mean.clone(), obs_var=norm.var.clone(), obs_count=norm.count.clone()), path)
        save_obs_rms(self.log_dir, norm.mean.detach().cpu().numpy(), norm.var.detach().cpu().numpy(), float(norm.count))

    def finish(self):
        """Close the monitor; rank 0 saves ``<algo>_model_final.pt`` (and ``<algo>_model.pt`` if the callback never saved) and best_model.json."""
        if self.monitor is not None:
            self.monitor.close()
        if self.log_dir and self.run.rank == 0:
            algo = self.run.algo
            self.save_model(os.path.join(self.log_dir, "%s_model_final.pt" % algo))
            if self.n_saved == 0:              # a run too short for the callback to fire (fewer than MIN_EPISODES_BEFORE_SAVE episodes): keep the last model
                self.save_model(os.path.join(self.log_dir, "%s_model.pt" % algo))
            with open(os.path.join(self.log_dir, "best_model.json"), "w") as f:
                json.dump(dict(best_mean_reward=self.best_mean_reward if self.n_saved else None, saves=self.n_saved, n_episodes_eval=self.N_EPISODES_EVAL,
                               min_episodes_before_save=self.MIN_EPISODES_BEFORE_SAVE, save_interval_updates=self.save_interval), f)


def train(env_id, num_envs, num_timesteps, seed=0, env_kwargs=None, log_dir=None, device=0, hyperparams=None, verbose=1, cuda_graph=True,
          phase_times=None, fused_act=None, prefetch_resets=None, episode_window=40, fused_update=None, num_stack=1):
    """PPO2.learn on a BatchedSRLVecEnv.  Returns a history of (timesteps, mean episode return, fps).

    ``cuda_graph``: the n_steps-long collection loop (policy forward, action sampling, observation filter, one simulator
    launch per step, buffer writes -- a few dozen small kernels per env step) is captured ONCE into a CUDA graph and replayed
    per update, so a rollout costs one graph launch instead of ~n_steps x 50 kernel launches from Python.
    ``fused_act`` (default: on whenever the envs live on a GPU; faster end to end with the records on):
    run the per-step policy work through the library's own kernels (``srl_policy_act``: both towers, sample, log-prob,
    value and the rollout-buffer writes in one launch; ``srl_obs_filter``: the observation filter in one launch; include/srl_policy.h)
    instead of ~60 small torch kernels: an env step of the collection loop is then three launches.  Sampling then uses the library's
    counter-based streams (keyed by seed and global env index) instead of torch's generator.
    ``prefetch_resets`` (default: on whenever the envs live on a GPU; a no-op for the kinds without records): create the envs with ``srl_cfg.prefetch_resets`` -- every lockstep launch then uses the idle slot of each warp as a helper that
    prepares the next-episode records, so that a step whose env finishes an episode copies a record in instead of running reset() inside
    the launch (include/srl_sim.h: srl_sim_prefetch_resets; validated bit-identical against in-launch resets).
    ``fused_update`` (default: on whenever the envs live on a GPU): the gradient of a minibatch step comes from the library's
    ``srl_ppo2_grad`` (include/srl_policy.h: forward, PPO2 loss derivative and backward of both towers in one pass, every activation on chip)
    instead of torch autograd over [minibatch, 64] tensors; gradient clipping, the data-parallel all-reduce and Adam stay in torch.
    ``num_stack``: ``VecFrameStack(envs, num_stack)`` before the filter, as the reference's ``createEnvs`` wraps every env (rl_baselines/utils.py:222-227):
    the policy, the filter and the rollout buffer see rows of ``num_stack * D`` values, oldest frame first, zeroed where an episode ended.  The
    stack is a static device buffer; the fused path advances it and filters it in one launch (``srl_obs_stack_filter``), so an env step stays
    three launches.  The fused kernels take rows of up to 32 values.
    ``phase_times``: optional dict; when given, every update synchronises between its phases and accumulates the wall time of
    ``collect`` / ``gae`` / ``optimise`` in it (a profiling aid: the synchronisations cost throughput)."""
    hp = dict(PPO2_DEFAULTS); hp.update(hyperparams or {})
    torch.manual_seed(seed)
    run = make_run("ppo2", env_id, num_envs, seed, env_kwargs, device, prefetch_resets, num_stack, [fused_act, fused_update])
    env, on_gpu, dev, policy, dist, rank, world = run.env, run.on_gpu, run.dev, run.policy, run.dist, run.rank, run.world
    prefetch_resets, K, W = run.prefetch_resets, run.K, run.W
    params = list(policy.parameters())
    params0 = [p.detach().clone() for p in params]
    N, T = num_envs, hp["n_steps"]
    # The GAE recursion and the minibatch step (forward, losses, backward, gradient clip, Adam) are captured into CUDA graphs too:
    # ~1000 and ~150 small launches respectively that cost more on the host than on the GPU.  Data-parallel runs keep the eager
    # minibatch step (its gradient all-reduce sits between backward and the optimiser step).
    graph_update = bool(cuda_graph and on_gpu and dist is None and (T * N) % hp["nminibatches"] == 0)
    if graph_update:      # a captured optimiser needs its step counter and its learning rate on the device
        lr_t = torch.tensor(float(hp["learning_rate"]), device=dev, dtype=torch.float32)
        opt = torch.optim.Adam(params, lr=lr_t, eps=1e-5, capturable=True)
    else:
        opt = torch.optim.Adam(params, lr=hp["learning_rate"], eps=1e-5)
    norm = RunningNorm(W, dev)
    n_updates = max(1, int(num_timesteps) // (N * T * world))
    write_run_files(run, log_dir, num_timesteps, seed, hp)
    obs, stack = first_observation(run, norm)    # the current (filtered) observation; updated IN PLACE by the collection loop
    buf = dict(obs=torch.empty((T, N, W), device=dev), act=torch.empty((T, N) if env.is_discrete else (T, N, env.sim.action_dim), device=dev,
                                                                       dtype=torch.int64 if env.is_discrete else torch.float32),
               logp=torch.empty((T, N), device=dev), val=torch.empty((T, N), device=dev), rew=torch.empty((T, N), device=dev),
               done=torch.empty((T, N), device=dev), ep_ret=torch.empty((T, N), device=dev), ep_len=torch.zeros((T, N), device=dev, dtype=torch.int32))
    last_val = torch.empty(N, device=dev)
    fused = None
    if fused_act is None:
        fused_act = on_gpu
    if fused_act:
        if not on_gpu:
            raise ValueError("fused_act=True needs the CUDA library (there is no CPU fallback)")
        from srl_sim.policy import FusedPolicy
        fused = FusedPolicy(env.backend.library, policy, norm.state, seed=seed, env_offset=rank * num_envs, clip=norm.clip, eps=norm.eps)
        act_dev = torch.zeros(N if env.is_discrete else (N, env.sim.action_dim), device=dev, dtype=torch.int32 if env.is_discrete else torch.float32)
        done_u8 = torch.zeros((T, N), device=dev, dtype=torch.uint8)

    if prefetch_resets and on_gpu:
        env.sim.prefetch_resets(stream=env.backend.stream())   # bulk fill of the first records; from here on the helper slots of every step launch keep them up

    def collect():
        """n_steps lockstep env steps under the current policy (three launches per env step on the fused path)."""
        if fused is not None:
            collect_rollout(run, norm, obs, stack, buf, last_val, fused=fused, act_dev=act_dev, done_u8=done_u8)
        else:
            collect_rollout(run, norm, obs, stack, buf, last_val)

    graph = None
    if cuda_graph and on_gpu:
        # an even number of simulator launches per replay keeps the MobileRobot state double buffer (swapped by the host at every
        # launch, so the pointers are baked into the captured kernels) in phase
        if T % 2:
            raise ValueError("cuda_graph=True needs an even n_steps")
        side = torch.cuda.Stream(device=dev)      # library handles / workspaces are created outside the capture
        side.wait_stream(torch.cuda.current_stream(dev))
        # the warm-up must not change what the run draws: the library's sampling counter and torch's generator (the torch policy's samples
        # below) are restored after it, so that a captured run samples actions and minibatch permutations as an eager one does
        rng0, torch_rng0 = fused.rng.clone() if fused is not None else None, torch.cuda.get_rng_state(dev)
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(3):
                policy.act(obs); norm(run.e_obs if stack is None else stack, update=False)
            if fused is not None:         # first launches outside the capture (one-off function attributes); they change nothing that matters:
                fused.act(N, obs, act_dev, buf["logp"][0], buf["val"][0], stream=env.backend.stream())
                if K > 1:                 # a copy of the stack and a scratch output: the stack itself must not advance
                    fused.stack_filter(N, env._obs, done_u8[0], stack.clone(), torch.empty_like(obs), update=False, stream=env.backend.stream())
                else:
                    fused.filter(N, env._obs, obs, update=False, stream=env.backend.stream())               # re-normalises the current observation
                fused.rng.copy_(rng0)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize()
        torch.cuda.set_rng_state(torch_rng0, dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):       # capture only records the launches: neither the envs nor the filter advance
            collect()

    # ---- advantage estimation and the minibatch step on static buffers (so that both can be captured) ----
    adv, ret = torch.zeros((T, N), device=dev), torch.zeros((T, N), device=dev)
    flat = {k: v.reshape((T * N,) + v.shape[2:]) for k, v in buf.items()}
    flat_adv, flat_ret = adv.reshape(-1), ret.reshape(-1)
    mb = max(1, T * N // hp["nminibatches"])
    idx_static = torch.zeros(mb, dtype=torch.int64, device=dev)

    def gae():
        """GAE(lambda), the reference's backward recursion over the rollout."""
        if fused_grad is not None:     # one launch instead of ~6 small kernels per step of the recursion
            fused_grad.gae(buf["rew"], buf["val"], buf["done"], last_val, hp["gamma"], hp["lam"], adv, ret, stream=env.backend.stream())
            return
        with torch.no_grad():
            lastgae = torch.zeros(N, device=dev)
            for t in reversed(range(T)):
                nonterminal = 1.0 - buf["done"][t]
                nextval = last_val if t == T - 1 else buf["val"][t + 1]
                delta = buf["rew"][t] + hp["gamma"] * nextval * nonterminal - buf["val"][t]
                lastgae = delta + hp["gamma"] * hp["lam"] * nonterminal * lastgae
                adv[t].copy_(lastgae)
            torch.add(adv, buf["val"], out=ret)

    fused_grad = None
    if fused_update is None:
        fused_update = on_gpu
    if fused_update:
        if not on_gpu:
            raise ValueError("fused_update=True needs the CUDA library (there is no CPU fallback)")
        if (T * N) % mb:
            raise ValueError("fused_update=True needs n_steps * num_envs divisible by nminibatches")
        from srl_sim.policy import FusedPPO2Grad
        fused_grad = FusedPPO2Grad(env.backend.library, policy, mb)

    def zero_grads():
        if fused_grad is None:         # the fused gradient kernel overwrites its static .grad tensors: nothing to clear
            opt.zero_grad(set_to_none=True)

    def minibatch_step(idx):
        if fused_grad is not None:     # the kernel overwrites the static .grad tensors
            fused_grad(idx, flat["obs"], flat["act"], flat_adv, flat_ret, flat["logp"], flat["val"], hp["cliprange"], hp["ent_coef"], hp["vf_coef"],
                       stream=env.backend.stream())
            if dist is not None:
                allreduce_mean_gradients(params, dist, world)
            nn.utils.clip_grad_norm_(params, hp["max_grad_norm"])
            opt.step()
            return
        logp, ent, v = policy.evaluate(flat["obs"][idx], flat["act"][idx])
        a_mb = flat_adv[idx]
        a_mb = (a_mb - a_mb.mean()) / (a_mb.std() + 1e-8)
        ratio = torch.exp(logp - flat["logp"][idx])
        pg = torch.max(-a_mb * ratio, -a_mb * torch.clamp(ratio, 1 - hp["cliprange"], 1 + hp["cliprange"])).mean()
        vclip = flat["val"][idx] + torch.clamp(v - flat["val"][idx], -hp["cliprange"], hp["cliprange"])
        vf_loss = 0.5 * torch.max((v - flat_ret[idx]) ** 2, (vclip - flat_ret[idx]) ** 2).mean()
        loss = pg - hp["ent_coef"] * ent.mean() + hp["vf_coef"] * vf_loss
        loss.backward()
        if dist is not None:           # one all-reduce of the flattened gradient per minibatch
            allreduce_mean_gradients(params, dist, world)
        nn.utils.clip_grad_norm_(params, hp["max_grad_norm"])
        opt.step()

    gae_graph = None
    if graph is not None:              # same conditions as the collection graph; elementwise work only, nothing to warm up
        gae_graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gae_graph):
            gae()
    mb_graph, mb_warm = None, 0        # the minibatch step is captured after three eager warm-up steps (real ones) on a side stream

    # best-model callback every SAVE_INTERVAL callback calls of the reference: 20 PPO2 updates of 8 envs x 128 steps there, scaled to this batch
    log = RunLog(run, norm, log_dir, max(1, 20 * 8 * 128 // (N * T * world)), episode_window, verbose)
    tick = phase_timer(phase_times, on_gpu)
    log.start()
    for update in range(1, n_updates + 1):
        frac = 1.0 - (update - 1.0) / n_updates
        if graph_update:
            lr_t.fill_(hp["learning_rate"] * frac)                        # learning_rate = lambda f: f * 2.5e-4
        else:
            for g in opt.param_groups:
                g["lr"] = hp["learning_rate"] * frac
        prior = (norm.mean.clone(), norm.var.clone(), norm.count.clone()) if dist is not None else None
        t_ph = tick()
        if graph is not None:
            graph.replay()
        else:
            collect()
        if dist is not None:                   # one all-reduce of 2 D + 1 doubles per rollout
            merge_running_moments(norm, prior, dist.all_reduce, world)
        t_ph = tick("collect", t_ph)
        log.episodes(buf["done"], buf["ep_ret"], buf["ep_len"])
        if gae_graph is not None:
            gae_graph.replay()
        else:
            gae()
        t_ph = tick("gae", t_ph)
        perms = []
        for _ in range(hp["noptepochs"]):
            perm = torch.randperm(T * N, device=dev)
            perms.append(perm)
            for s in range(0, T * N, mb):
                if not graph_update:
                    zero_grads()
                    minibatch_step(perm[s:s + mb])
                    continue
                idx_static.copy_(perm[s:s + mb])
                if mb_graph is not None:
                    mb_graph.replay()
                elif mb_warm < 3:          # warm-up iterations run on a side stream (torch's whole-network capture recipe)
                    cur = torch.cuda.current_stream(dev)
                    side = torch.cuda.Stream(device=dev)
                    side.wait_stream(cur)
                    with torch.cuda.stream(side):
                        zero_grads()
                        minibatch_step(idx_static)
                    cur.wait_stream(side)
                    mb_warm += 1
                else:
                    mb_graph = torch.cuda.CUDAGraph()
                    zero_grads()
                    with torch.cuda.graph(mb_graph):   # gradients are allocated from the graph's pool and re-created by every replay
                        minibatch_step(idx_static)
                    mb_graph.replay()                  # the capture only recorded this minibatch: now run it
        t_ph = tick("optimise", t_ph)
        log.end_update(update, n_updates, update * N * T * world)
    log.finish()
    env.close()
    train.best_mean_reward, train.n_saved = log.best_mean_reward, log.n_saved
    train.last_policy, train.last_norm = policy, norm      # for callers that want the trained objects (tests, enjoy)
    # what the last update started from and left behind, for tests that rebuild it: the initial parameters, the rollout buffers, GAE's
    # inputs and outputs, the epochs' permutations and the optimiser (its Adam state)
    train.last_update = dict(params0=params0, buf=buf, obs=obs, adv=adv, ret=ret, last_val=last_val, perms=perms, opt=opt, mb=mb)
    return log.history
