"""
DQN consumer of the batched simulator: stable-baselines 2.5's ``DQN`` with the deepq ``MlpPolicy`` behind ``VecNormalize``, as the reference
trains it through ``rl_baselines/rl_algorithm/deepq.py`` (learning_rate 1e-4, buffer_size ``--buffer-size``, exploration_fraction 0.1,
exploration_final_eps 0.01, train_freq 4, learning_starts 500, target_network_update_freq 500, gamma 0.99, prioritized_replay
``--prioritized``, prioritized_replay_alpha 0.6; stable-baselines' defaults batch_size 32, prioritized_replay_beta0 0.4,
prioritized_replay_beta_iters = the run's length, prioritized_replay_eps 1e-6).  Restated in PyTorch next to rl_baselines/ppo2.py, whose
env set-up, observation filter, run files and data-parallel collectives it imports.

RECALLED from stable-baselines 2.5 and baselines, not checked against an installed copy (none can be installed here; include/srl_policy.h):
the dueling two-tower network with ReLU and glorot-uniform weights, double Q, the Huber loss, ``tf.clip_by_norm(g, 10)`` per tensor, TF1 Adam,
the learn loop's conditions, baselines' PrioritizedReplayBuffer and SegmentTree, and the default hyper-parameters named above.
``--dueling`` is parsed by the reference and never passed: the deepq MlpPolicy is dueling regardless, and so is this one.

Batched semantics.  The reference steps one env.  Here N envs per rank step in lockstep, and everything the reference counts in env steps is
counted in lockstep steps: ``t``, learning_starts, train_freq, target_network_update_freq, and the epsilon and beta schedules, whose horizon
is ``num_timesteps / (N world)``.  Sizes scale with N: the per-rank replay ring holds ``buffer_size`` lockstep rows (``buffer_size N``
transitions) and a gradient step samples ``batch_size N`` transitions, which keeps the reference's replay ratio and its number of gradient
steps per env step.  Per lockstep step t (from 0):
  act epsilon(t)-greedily, step, store (obs, a, r, new_obs, done) in ring row t % buffer_size, obs = new_obs;
  if t > learning_starts and t % train_freq == 0: one gradient step (sample with beta(t), double-Q target, gradient, clip + Adam, priorities);
  if t > learning_starts and t % target_network_update_freq == 0: target <- online.
Data-parallel (torchrun): every rank keeps its own ring and trees and samples from them only; the gradient is averaged over ranks before the
optimiser; the observation filter is merged once per train_freq steps; importance weights are normalised by the rank's own p_min (a
deviation from one global buffer).

On the GPU (``fused``) every step is the library's kernels: ``srl_dqn_act``, ``srl_sim_step``, ``srl_obs_filter`` /
``srl_obs_stack_filter`` writing straight into ring row t, ``srl_replay_add``; a gradient step is ``srl_replay_sample``, ``srl_dqn_target``,
``srl_dqn_grad``, ``srl_clip_adam``, ``srl_replay_update``; a block of train_freq steps (two when it is odd) with its gradient step is one CUDA
graph replay, one graph per ring phase (:func:`train`).  A gradient step also needs the ring to hold ``batch_size`` rows
(``replay_buffer.can_sample(batch_size)``, RECALLED), so a ``--buffer-size`` below batch_size never trains.  The CPU path (the oracle backend of the tests, and ``fused=False``) runs the same
algorithm in torch and numpy: :class:`DuelingQ`, :func:`dqn_loss`, :func:`clip_adam` and :class:`ReplayTree`.
"""
import numpy as np
import torch
import torch.nn as nn

from rl_baselines.ppo2 import (RunLog, RunningNorm, allreduce_mean_gradients, first_observation, make_run, merge_running_moments, phase_timer,
                               write_run_files)

DQN_DEFAULTS = dict(learning_rate=1e-4, buffer_size=1000, exploration_fraction=0.1, exploration_final_eps=0.01, train_freq=4, learning_starts=500,
                    target_network_update_freq=500, gamma=0.99, prioritized_replay=True, prioritized_replay_alpha=0.6,      # rl_algorithm/deepq.py
                    batch_size=32, prioritized_replay_beta0=0.4, prioritized_replay_eps=1e-6)                               # stable-baselines 2.5
GRAD_CLIP_NORM = 10.0                                   # build_train's grad_norm_clipping in stable-baselines' DQN (RECALLED)
ADAM_BETA1, ADAM_BETA2, ADAM_EPS = 0.9, 0.999, 1e-8     # tf.train.AdamOptimizer's defaults
CONTINUOUS_ERROR = "deepq does not support continuous actions, please remove the '--continuous-actions' (or '-c') flag."


class DuelingQ(nn.Module):
    """The deepq MlpPolicy with layers [64, 64] (RECALLED): an advantage tower ``pi`` (W -> 64 -> 64 -> n, ReLU) and a state-value tower
    ``vf`` (W -> 64 -> 64 -> 1), Q = V + (A - mean(A)).  The towers have the layout of rl_baselines.ppo2.MlpPolicy, so the library's kernels
    read it as an srl_mlp_policy with discrete = 1.  Weights glorot-uniform, biases zero (tf.contrib.layers.fully_connected's defaults)."""
    discrete = True

    def __init__(self, obs_dim, n_actions):
        super().__init__()
        self.n_actions = int(n_actions)

        def tower(last):
            layers = [nn.Linear(obs_dim, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, last)]
            for m in layers:
                if isinstance(m, nn.Linear):
                    nn.init.xavier_uniform_(m.weight); nn.init.zeros_(m.bias)
            return nn.Sequential(*layers)
        self.pi, self.vf = tower(self.n_actions), tower(1)

    def forward(self, obs):
        a = self.pi(obs)
        return self.vf(obs) + (a - a.sum(-1, keepdim=True) * (1.0 / self.n_actions))


def huber(x):
    """tf.losses.huber_loss with delta 1 as baselines' U.huber_loss writes it."""
    return torch.where(x.abs() < 1.0, 0.5 * x * x, x.abs() - 0.5)


def double_q_target(online, target, rew, done, next_obs, gamma):
    """y = r + gamma ((1 - d) Q_target(s', argmax_b Q_online(s', b))) (build_train with double_q=True; argmax ties: the lowest index)."""
    with torch.no_grad():
        best = online(next_obs).argmax(-1, keepdim=True)
        q_t = target(next_obs).gather(-1, best).squeeze(-1)
        return rew + gamma * ((1.0 - done) * q_t)


def dqn_loss(qnet, obs, act, y, weights):
    """mean(w huber(Q(s, a) - y)); returns (loss, td)."""
    td = qnet(obs).gather(-1, act.reshape(-1, 1)).squeeze(-1) - y
    return (weights * huber(td)).mean(), td.detach()


def clip_adam(params, m, v, beta_power, lr, clip_norm, beta1, beta2, eps):
    """``tf.clip_by_norm`` per tensor then TF1 Adam on the ``.grad`` of ``params`` (the torch statement of srl_clip_adam, in its order of float32
    roundings): ``g = t clip / max(norm, clip)``, ``m += (g - m)(1 - b1)``, ``v += (g^2 - v)(1 - b2)``, ``lr_t = lr sqrt(1 - b2^t) / (1 - b1^t)``,
    ``p -= m lr_t / (sqrt(v) + eps)``; ``beta_power`` (float32 [2], from {b1, b2}) is multiplied by {b1, b2} after the step."""
    with torch.no_grad():
        f32 = lambda x: torch.tensor(x, dtype=torch.float32, device=beta_power.device)
        lr_t = (f32(lr) * torch.sqrt(1.0 - beta_power[1])) / (1.0 - beta_power[0])
        r1, r2 = f32(1.0) - f32(beta1), f32(1.0) - f32(beta2)
        for p, mm, vv in zip(params, m, v):
            norm = torch.sqrt((p.grad.double() ** 2).sum()).float()
            den = norm if bool(torch.isnan(norm)) else torch.clamp(norm, min=clip_norm)
            g = (p.grad * clip_norm) / den
            mm.add_((g - mm) * r1)
            vv.add_((g * g - vv) * r2)
            p.sub_((mm * lr_t) / (torch.sqrt(vv) + eps))
        beta_power.mul_(torch.stack([f32(beta1), f32(beta2)]))


class ReplayTree(object):
    """baselines' PrioritizedReplayBuffer bookkeeping over a ring of ``rows`` x ``n_envs`` transitions, vectorised in numpy: float64 sum and
    min trees (root 1, leaf i at tree_cap + i, internal node = op(left, right), unused leaves 0 / inf), ``max_priority`` and ``size``.  The
    statement srl_replay_add / _sample / _update follow (include/srl_policy.h)."""

    def __init__(self, rows, n_envs, alpha):
        self.n_envs, self.capacity, self.alpha = int(n_envs), int(rows) * int(n_envs), float(alpha)
        self.tree_cap = 1
        while self.tree_cap < self.capacity:
            self.tree_cap *= 2
        self.sum = np.zeros(2 * self.tree_cap)
        self.min = np.full(2 * self.tree_cap, np.inf)
        self.max_priority, self.size = 1.0, 0

    def _rebuild(self, lo, hi):
        """op(left, right) for every ancestor of leaves [lo, hi), level by level."""
        lo, hi = lo + self.tree_cap, hi + self.tree_cap
        while lo > 1:
            lo, hi = lo // 2, (hi - 1) // 2 + 1
            k = np.arange(lo, hi)
            self.sum[k] = self.sum[2 * k] + self.sum[2 * k + 1]
            self.min[k] = np.minimum(self.min[2 * k], self.min[2 * k + 1])

    def add(self, row):
        lo = int(row) * self.n_envs
        leaf = self.max_priority ** self.alpha
        self.sum[self.tree_cap + lo:self.tree_cap + lo + self.n_envs] = leaf
        self.min[self.tree_cap + lo:self.tree_cap + lo + self.n_envs] = leaf
        self._rebuild(lo, lo + self.n_envs)
        self.size = max(self.size, lo + self.n_envs)

    def sample(self, u, beta, prioritized=True):
        """Indices and float32 importance weights of the samples whose uniforms in [0, 1) are ``u`` (float64)."""
        u, n = np.asarray(u, np.float64), self.size
        if not prioritized:
            return np.minimum((u * n).astype(np.int64), n - 1), np.ones(len(u), np.float32)
        total = self.sum[1]
        mass, node = u * total, np.ones(len(u), np.int64)
        while node[0] < self.tree_cap:           # find_prefixsum_idx, every walk one level per pass
            left = self.sum[2 * node]
            go_left = left > mass
            mass = np.where(go_left, mass, mass - left)
            node = 2 * node + (~go_left)
        idx = np.minimum(node - self.tree_cap, n - 1)      # rounding into an empty leaf: the last stored transition
        max_w = (self.min[1] / total * n) ** -beta
        return idx, ((self.sum[self.tree_cap + idx] / total * n) ** -beta / max_w).astype(np.float32)

    def update(self, idx, td, eps):
        """priority = |td| + eps in float32; leaf = priority^alpha in float64, the last occurrence of a repeated index wins."""
        idx = np.asarray(idx, np.int64)
        p = np.abs(np.asarray(td, np.float32)) + np.float32(eps)
        uniq, first_rev = np.unique(idx[::-1], return_index=True)
        last = len(idx) - 1 - first_rev
        leaf = np.array([float(x) ** self.alpha for x in p[last]])         # libm's pow, as baselines' Python loop (numpy's vector pow may differ by an ulp)
        self.sum[self.tree_cap + uniq] = leaf
        self.min[self.tree_cap + uniq] = leaf
        self.max_priority = max(self.max_priority, float(p.max()))
        self._rebuild(0, self.tree_cap)


def linear_schedule(schedule_timesteps, initial_p, final_p, t):
    """baselines' LinearSchedule.value(t); a horizon of 0 steps (a run shorter than 1 / exploration_fraction steps) is taken as 1."""
    fraction = min(float(t) / max(1, int(schedule_timesteps)), 1.0)
    return initial_p + fraction * (final_p - initial_p)


def cadence(t, hp):
    """(gradient step at lockstep step t, target copy at t): DQN.learn's conditions."""
    late = t > hp["learning_starts"]
    return late and t % hp["train_freq"] == 0, late and t % hp["target_network_update_freq"] == 0


def can_sample(t, hp, num_envs):
    """stable-baselines' ``replay_buffer.can_sample(batch_size)`` in DQN.learn's condition (RECALLED): after step t the ring stores at least
    ``batch_size`` rows of N transitions, i.e. ``batch_size N`` transitions."""
    return min(t + 1, hp["buffer_size"]) * num_envs >= hp["batch_size"] * num_envs


def train(env_id, num_envs, num_timesteps, seed=0, env_kwargs=None, log_dir=None, device=0, hyperparams=None, verbose=1, fused=None,
          cuda_graph=True, phase_times=None, prefetch_resets=None, episode_window=40, num_stack=1):
    """DQN.learn on a BatchedSRLVecEnv (module docstring).  Returns a history of (timesteps, mean episode return, fps), one entry per
    ``train_freq`` lockstep steps.  ``fused`` (default: on whenever the envs live on a GPU): the library's kernels; off, or on the CPU
    oracle backend, torch and numpy.  ``num_stack``, ``prefetch_resets``, ``episode_window``: as for rl_baselines.ppo2.train.

    The steps run in blocks of G lockstep steps: G = train_freq, or 2 train_freq when train_freq is odd (MobileRobot's state double buffer
    needs an even number of simulator launches per graph replay).  ``cuda_graph`` (fused, single process, no ``phase_times``): a block that
    takes its gradient steps at its offsets 0 (and train_freq) is ONE CUDA graph replay -- per step srl_dqn_act, srl_sim_step, the filter,
    srl_replay_add; per gradient step sample, target, gradient, clip + Adam, priorities.  The ring rows a block writes are baked into its
    graph, so there is one graph per ring phase (``t0 % buffer_size``), captured the first time that phase comes up; epsilon and beta are
    read from device arrays the host rewrites before each block.  Blocks before learning_starts (collection only), the first gradient block
    (it warms every kernel up), blocks whose gradient steps fall elsewhere and a block with a target copy between its two gradient steps run
    the same launches eagerly.  The target copy is a device copy after the step (eager) or after the replay (captured: the target is read by
    gradient steps only, and none follows in the block).  ``phase_times``: a dict that accumulates the wall time of ``collect`` / ``replay``
    (sample, priorities) / ``gradient`` (target, gradient) / ``optimise``, synchronising between them (eager)."""
    hp = dict(DQN_DEFAULTS); hp.update(hyperparams or {})
    if not dict(env_kwargs or {}).get("is_discrete", True):
        raise ValueError(CONTINUOUS_ERROR)
    torch.manual_seed(seed)
    run = make_run("deepq", env_id, num_envs, seed, env_kwargs, device, prefetch_resets, num_stack, [fused],
                   network=lambda width, env: DuelingQ(width, env.action_space.n))
    env, on_gpu, dev, qnet, dist, rank, world, K, W = run.env, run.on_gpu, run.dev, run.policy, run.dist, run.rank, run.world, run.K, run.W
    if fused is None:
        fused = on_gpu
    if fused and not on_gpu:
        raise ValueError("fused=True needs the CUDA library (there is no CPU fallback)")
    N, F, rows = num_envs, hp["train_freq"], hp["buffer_size"]
    G = F if F % 2 == 0 else 2 * F
    B = hp["batch_size"] * N
    n_steps = max(1, int(num_timesteps) // (N * world))          # lockstep steps: the horizon of both schedules
    explore_steps = int(hp["exploration_fraction"] * n_steps)
    prioritized = bool(hp["prioritized_replay"])
    use_graph = bool(cuda_graph and fused and dist is None and phase_times is None)
    target = DuelingQ(W, qnet.n_actions).to(dev)
    target.load_state_dict(qnet.state_dict())
    target.requires_grad_(False)
    norm = RunningNorm(W, dev)
    write_run_files(run, log_dir, num_timesteps, seed, hp)
    obs, stack = first_observation(run, norm)
    z = lambda *shape, dtype=torch.float32: torch.zeros(shape, device=dev, dtype=dtype)
    ring = dict(obs=z(rows, N, W), next_obs=z(rows, N, W), act=z(rows, N, dtype=torch.int64), rew=z(rows, N), done=z(rows, N, dtype=torch.uint8))
    flat = {k: v.reshape((rows * N,) + v.shape[2:]) for k, v in ring.items()}
    block = dict(done=z(G, N), ep_ret=z(G, N), ep_len=z(G, N, dtype=torch.int32))      # the episodes of one block
    eps_blk, beta_blk = z(G), z(G, dtype=torch.float64)                                # epsilon / beta of each step of a block
    params = list(qnet.parameters())
    for p in params:
        p.grad = torch.zeros_like(p)
    if fused:
        from srl_sim.policy import FusedClipAdam, FusedDQNAct, FusedDQNGrad, FusedDQNTarget, FusedObsFilter, FusedReplay
        lib = env.backend.library
        ffilter = FusedObsFilter(lib, norm.state, clip=norm.clip, eps=norm.eps)
        fact = FusedDQNAct(lib, qnet, seed=seed, env_offset=rank * N)
        ftarget = FusedDQNTarget(lib, qnet, target)
        fgrad = FusedDQNGrad(lib, qnet, B)
        fopt = FusedClipAdam(lib, qnet, GRAD_CLIP_NORM, ADAM_BETA1, ADAM_BETA2, ADAM_EPS)
        fopt.lr.fill_(hp["learning_rate"])
        replay = FusedReplay(lib, rows, N, seed + 1 + rank, hp["prioritized_replay_alpha"], dev)
        act_dev, idx, w, y, td = z(N, dtype=torch.int32), z(B, dtype=torch.int64), z(B), z(B), z(B)
        m, v, beta_power = fopt.m, fopt.v, fopt.beta_power
    else:
        replay = ReplayTree(rows, N, hp["prioritized_replay_alpha"])
        m, v = [torch.zeros_like(p) for p in params], [torch.zeros_like(p) for p in params]
        beta_power = torch.tensor([ADAM_BETA1, ADAM_BETA2], dtype=torch.float32, device=dev)
    if run.prefetch_resets and on_gpu:
        env.sim.prefetch_resets(stream=env.backend.stream())
    tick = phase_timer(phase_times, on_gpu)

    def env_step(t, k):
        """Act, step and store ring row t % rows; the new (filtered) observation is a view of the ring's next_obs row."""
        row = t % rows
        st = env.backend.stream()
        new_obs = ring["next_obs"][row]
        with torch.no_grad():
            if fused:
                fact(N, cur[0], act_dev, obs_buf=ring["obs"][row], act_buf=ring["act"][row], eps=eps_blk[k:k + 1], stream=st)
                env.sim.step(act_dev, None, env._obs, ring["rew"][row], ring["done"][row], block["ep_ret"][k], block["ep_len"][k], stream=st)
                if K > 1:
                    ffilter.stack_filter(N, env._obs, ring["done"][row], stack, new_obs, update=True, stream=st)
                else:
                    ffilter.filter(N, env._obs, new_obs, update=True, stream=st)
                block["done"][k].copy_(ring["done"][row])
                replay.add(row, stream=st)
            else:
                o = cur[0]
                greedy = qnet(o).argmax(-1)
                explore = torch.rand(N, device=dev) < float(eps_blk[k])
                a = torch.where(explore, torch.randint(0, qnet.n_actions, (N,), device=dev), greedy)
                ring["obs"][row].copy_(o); ring["act"][row].copy_(a)
                env.step_tensors(a.to(torch.int32))
                ring["rew"][row].copy_(run.e_rew); ring["done"][row].copy_(run.e_done)
                block["done"][k].copy_(run.e_done); block["ep_ret"][k].copy_(run.e_ep_ret); block["ep_len"][k].copy_(run.e_ep_len)
                if K > 1:                                    # VecFrameStack.step
                    stack.copy_(torch.where(run.e_done.bool()[:, None], 0.0, torch.roll(stack, -run.D, 1)))
                    stack[:, W - run.D:].copy_(run.e_obs)
                    new_obs.copy_(norm(stack))
                else:
                    new_obs.copy_(norm(run.e_obs))
                replay.add(row)
        cur[0] = new_obs

    def gradient_step(k):
        st = env.backend.stream()
        if fused:
            t_ph = tick()
            replay.sample(B, idx, w, prioritized=prioritized, beta=beta_blk[k:k + 1], stream=st)
            t_ph = tick("replay", t_ph)
            ftarget(B, idx, flat["next_obs"], flat["rew"], flat["done"], hp["gamma"], y, stream=st)
            fgrad(idx, flat["obs"], flat["act"], y, w if prioritized else None, td, stream=st)
            if dist is not None:
                allreduce_mean_gradients(params, dist, world)
            t_ph = tick("gradient", t_ph)
            fopt(stream=st)
            t_ph = tick("optimise", t_ph)
            if prioritized:
                replay.update(B, idx, td, hp["prioritized_replay_eps"], stream=st)
            tick("replay", t_ph)
            return
        u = torch.rand(B, dtype=torch.float64).numpy()
        ix, wt = replay.sample(u, float(beta_blk[k]), prioritized)
        ix_t = torch.from_numpy(ix).to(dev)
        y_t = double_q_target(qnet, target, flat["rew"][ix_t], flat["done"][ix_t].float(), flat["next_obs"][ix_t], hp["gamma"])
        for p in params:
            p.grad.zero_()
        loss, td_t = dqn_loss(qnet, flat["obs"][ix_t], flat["act"][ix_t], y_t, torch.from_numpy(wt).to(dev))
        loss.backward()
        if dist is not None:
            allreduce_mean_gradients(params, dist, world)
        clip_adam(params, m, v, beta_power, hp["learning_rate"], GRAD_CLIP_NORM, ADAM_BETA1, ADAM_BETA2, ADAM_EPS)
        if prioritized:
            replay.update(ix, td_t.cpu().numpy(), hp["prioritized_replay_eps"])

    def target_copy():
        with torch.no_grad():
            for q_t, q in zip(target.parameters(), params):
                q_t.copy_(q)
        stats["target_copies"] += 1

    def run_block(t0, steps, copies):
        """The block's steps with their gradient steps (the learn loop's conditions); the target copies too when ``copies``."""
        for k in range(steps):
            t_ph = tick()
            env_step(t0 + k, k)
            tick("collect", t_ph)
            do_grad, do_copy = cadence(t0 + k, hp)
            if do_grad and can_sample(t0 + k, hp, N):
                gradient_step(k)
                stats["grad_steps"] += 1
            if do_copy and copies:
                target_copy()

    def graph_block(t0):
        """Whether the block at t0 (G full steps) can be one replay: gradient steps exactly at offsets 0 (and F), no target copy between them."""
        if not (t0 > hp["learning_starts"] and can_sample(t0, hp, N) and t0 + G <= n_steps):
            return False
        return not (G == 2 * F and any(cadence(t, hp)[1] for t in range(t0, t0 + F)))

    cur = [obs]
    graphs, pool, warmed = {}, None, False
    # best-model callback: SAVE_INTERVAL = 200 callback calls of one env step each in the reference, scaled to periods of F x N x world env steps
    log = RunLog(run, norm, log_dir, max(1, 200 // (F * N * world)), episode_window, verbose)
    log.start()
    n_periods = (n_steps + F - 1) // F
    stats = dict(grad_steps=0, target_copies=0, graph_replays=0, graphs=0)
    t0, p_i = 0, 0
    while t0 < n_steps:
        steps = min(G, n_steps - t0)
        prior = (norm.mean.clone(), norm.var.clone(), norm.count.clone()) if dist is not None else None
        eps_blk.copy_(torch.tensor([linear_schedule(explore_steps, 1.0, hp["exploration_final_eps"], t0 + k) for k in range(G)]))
        beta_blk.copy_(torch.tensor([linear_schedule(n_steps, hp["prioritized_replay_beta0"], 1.0, t0 + k) for k in range(G)], dtype=torch.float64))
        if use_graph and graph_block(t0) and warmed:
            key = t0 % rows
            if key not in graphs:
                pool = pool if pool is not None else torch.cuda.graph_pool_handle()
                g, cur0, counts = torch.cuda.CUDAGraph(), cur[0], dict(stats)
                with torch.cuda.graph(g, pool=pool):       # capture records the launches only: nothing advances
                    run_block(t0, G, copies=False)
                cur[0] = cur0
                stats.update(counts, graphs=counts["graphs"] + 1)
                graphs[key] = g
            graphs[key].replay()
            cur[0] = ring["next_obs"][(t0 + G - 1) % rows]
            stats["graph_replays"] += 1
            stats["grad_steps"] += G // F
            for t in range(t0, t0 + G):
                if cadence(t, hp)[1]:
                    target_copy()
        else:
            run_block(t0, steps, copies=True)
            warmed = warmed or (t0 > hp["learning_starts"] and can_sample(t0, hp, N))
        if dist is not None:
            merge_running_moments(norm, prior, dist.all_reduce, world)
        for k0 in range(0, steps, F):                        # one history entry per train_freq steps
            n = min(F, steps - k0)
            log.episodes(block["done"][k0:k0 + n], block["ep_ret"][k0:k0 + n], block["ep_len"][k0:k0 + n])
            p_i += 1
            log.end_update(p_i, n_periods, (t0 + k0 + n) * N * world, print_every=max(1, n_periods // 20))
        t0 += steps
    log.finish()
    env.close()
    train.best_mean_reward, train.n_saved, train.stats = log.best_mean_reward, log.n_saved, stats
    train.last_policy, train.last_target, train.last_norm, train.last_replay = qnet, target, norm, replay
    train.last_ring = ring
    train.last_adam = (m, v, beta_power)
    return log.history
