"""
A2C consumer of the batched simulator: stable-baselines 2.5's ``A2C`` with ``MlpPolicy`` behind ``VecNormalize``, as the reference
trains it through ``rl_baselines/rl_algorithm/a2c.py`` (defaults there: n_steps=5, vf_coef=0.5, ent_coef=0.01, max_grad_norm=0.5,
learning_rate=7e-4, epsilon=1e-5, alpha=0.99, gamma=0.99, ``--lr-schedule``).  Restated in PyTorch next to rl_baselines/ppo2.py, whose
policy, observation filter, env set-up and data-parallel collectives it imports.

One update: ``n_steps`` steps of every env, the bootstrapped n-step returns, ONE gradient of the A2C loss over all n_steps x num_envs
rows, TF1's global-norm clip and one TF1 RMSProp step.  An update is 20 480 samples at 4096 envs (PPO2's is 524 288), so the per-update
launch overhead of torch would cost as much as the collection; on the GPU the whole update is kernels of the library:
3 per env step (``srl_policy_act``, ``srl_sim_step``, ``srl_obs_filter`` / ``srl_obs_stack_filter``), the last value (torch), ``srl_ppo2_gae``
with lambda = 1 for the returns, ``srl_a2c_grad`` and ``srl_clip_rmsprop`` -- captured as ONE CUDA graph in a single process.  The graph
holds TWO updates: MobileRobot's state double buffer needs an even number of simulator launches per replay, and n_steps = 5 is odd.
The learning rates of both updates sit in a device array the host rewrites before each replay.

The CPU path (the oracle backend of the tests) and ``fused=False`` run the same update in torch: autograd of the loss below, and
:func:`clip_rmsprop`, the torch restatement of the optimiser that the kernel tests also use.
"""

import numpy as np
import torch

from rl_baselines.ppo2 import (RunLog, RunningNorm, allreduce_mean_gradients, collect_rollout, first_observation, make_run, merge_running_moments,
                               phase_timer, write_run_files)

A2C_DEFAULTS = dict(n_steps=5, vf_coef=0.5, ent_coef=0.01, max_grad_norm=0.5, learning_rate=7e-4, epsilon=1e-5, alpha=0.99, gamma=0.99,
                    lr_schedule="constant")   # rl_algorithm/a2c.py


def constant(_):
    return 1.0


def linear_schedule(progress):
    return 1.0 - progress


def middle_drop(progress):
    eps = 0.75
    if 1.0 - progress < eps:
        return eps * 0.1
    return 1.0 - progress


def double_linear_con(progress):
    progress *= 2
    eps = 0.125
    if 1.0 - progress < eps:
        return eps
    return 1.0 - progress


def double_middle_drop(progress):
    eps1, eps2 = 0.75, 0.25
    if 1.0 - progress < eps1:
        if 1.0 - progress < eps2:
            return eps2 * 0.5
        return eps1 * 0.1
    return 1.0 - progress


SCHEDULES = {"constant": constant, "linear": linear_schedule, "middle_drop": middle_drop, "double_linear_con": double_linear_con,
             "double_middle_drop": double_middle_drop}


def learning_rate(hp, update, n_batch, total_timesteps):
    """The learning rate of update ``update`` (0-based) under stable-baselines' ``Scheduler``, as recalled from stable_baselines/a2c/utils.py
    (not checked against an installed stable-baselines): ``value()`` returns ``initial * schedule(step / total_timesteps)`` and advances
    ``step`` by one; ``A2C._train_step`` calls it once per sample of the update and uses the last value, so update k trains with
    ``step = (k + 1) n_batch - 1``.  With p = step / total_timesteps the five schedules are
      constant: 1;   linear: 1 - p;   middle_drop: 1 - p, then 0.075 once 1 - p < 0.75;
      double_linear_con: 1 - 2p, then 0.125 once 1 - 2p < 0.125;
      double_middle_drop: 1 - p, then 0.075 once 1 - p < 0.75, then 0.125 once 1 - p < 0.25.
    p is capped at 1 (a run shorter than one batch still makes one update)."""
    progress = min(1.0, ((update + 1) * n_batch - 1) / float(total_timesteps))
    return hp["learning_rate"] * SCHEDULES[hp["lr_schedule"]](progress)


def a2c_loss(policy, obs, actions, ret, old_value, ent_coef, vf_coef):
    """stable-baselines 2.5 ``A2C.setup_model``'s loss (include/srl_policy.h, srl_a2c_grad): advantage ``ret - old_value`` without
    normalisation, ``pg = mean(-adv logp)``, ``vf = 0.5 mean((v - ret)^2)``, ``pg - ent_coef entropy + vf_coef vf``."""
    logp, ent, v = policy.evaluate(obs, actions)
    adv = ret - old_value
    return (-adv * logp).mean() - ent_coef * ent.mean() + vf_coef * (0.5 * ((v - ret) ** 2).mean())


def clip_rmsprop(params, ms, lr, max_grad_norm, alpha, epsilon):
    """TF1 ``clip_by_global_norm`` + ``RMSPropOptimizer(momentum=0)`` on the ``.grad`` of ``params`` (torch statement of srl_clip_rmsprop, in its
    order of float32 roundings): ``scale = max_norm / max(norm, max_norm)``, ``ms += (g^2 - ms) (1 - alpha)``, ``p -= g lr / sqrt(ms + eps)``.
    A non-finite norm makes every parameter NaN.  ``ms`` starts at 1 (TF's slot initialiser) and epsilon sits inside the square root -- both recalled from TF 1.x, see include/srl_policy.h.
    ``lr``: a float32 tensor (or a float)."""
    with torch.no_grad():
        sq = torch.stack([(p.grad.double() ** 2).sum() for p in params]).sum()
        norm = torch.sqrt(sq)
        scale = (max_grad_norm / torch.clamp(norm, min=max_grad_norm) + (norm - norm)).float()     # NaN for a non-finite norm, as in TF
        rho1 = float(np.float32(1.0) - np.float32(alpha))
        for p, m in zip(params, ms):
            g = p.grad * scale
            m.add_((g * g - m) * rho1)
            p.sub_((g * lr) / torch.sqrt(m + epsilon))


def train(env_id, num_envs, num_timesteps, seed=0, env_kwargs=None, log_dir=None, device=0, hyperparams=None, verbose=1, cuda_graph=True,
          phase_times=None, fused=None, prefetch_resets=None, episode_window=40, num_stack=1):
    """A2C.learn on a BatchedSRLVecEnv.  Returns a history of (timesteps, mean episode return, fps), one entry per update.

    ``fused`` (default: on whenever the envs live on a GPU): the update runs on the library's kernels (module docstring); off, or on the
    CPU oracle backend, it runs in torch.  ``cuda_graph`` (fused, single process): two updates per graph replay.  ``phase_times``: a dict
    that accumulates the wall time of ``collect`` / ``grad`` (returns + gradient) / ``optimise`` -- it synchronises between the phases and
    therefore runs the updates eagerly.  ``num_stack``, ``prefetch_resets``, ``episode_window``: as for rl_baselines.ppo2.train."""
    hp = dict(A2C_DEFAULTS); hp.update(hyperparams or {})
    if hp["lr_schedule"] not in SCHEDULES:
        raise ValueError("unknown lr_schedule %r (one of %s)" % (hp["lr_schedule"], ", ".join(sorted(SCHEDULES))))
    torch.manual_seed(seed)
    run = make_run("a2c", env_id, num_envs, seed, env_kwargs, device, prefetch_resets, num_stack, [fused])
    env, on_gpu, dev, policy, dist, rank, world, K, W = run.env, run.on_gpu, run.dev, run.policy, run.dist, run.rank, run.world, run.K, run.W
    if fused is None:
        fused = on_gpu
    if fused and not on_gpu:
        raise ValueError("fused=True needs the CUDA library (there is no CPU fallback)")
    N, T = num_envs, hp["n_steps"]
    n_batch = N * T * world                  # samples of one update over all ranks: the step of the learning-rate schedule
    n_updates = max(1, int(num_timesteps) // n_batch)
    use_graph = bool(cuda_graph and fused and dist is None and phase_times is None)
    H = 2 if use_graph else 1                # rollout halves: one per update of a graph replay
    norm = RunningNorm(W, dev)
    write_run_files(run, log_dir, num_timesteps, seed, hp)
    obs, stack = first_observation(run, norm)
    z = lambda *shape, dtype=torch.float32: torch.zeros(shape, device=dev, dtype=dtype)
    act_shape = (H, T, N) if env.is_discrete else (H, T, N, env.sim.action_dim)
    buf = dict(obs=z(H, T, N, W), act=z(*act_shape, dtype=torch.int64 if env.is_discrete else torch.float32), logp=z(H, T, N), val=z(H, T, N),
               rew=z(H, T, N), done=z(H, T, N), ep_ret=z(H, T, N), ep_len=z(H, T, N, dtype=torch.int32))
    last_val, adv, ret = z(H, N), z(H, T, N), z(H, T, N)
    lr_t = z(H)                              # the learning rate of each update of a replay, rewritten by the host
    params = list(policy.parameters())       # logstd (Box) first, then pi and vf: the CPU path pairs ms with them tensor by tensor
    params0 = [p.detach().clone() for p in params]
    for p in params:
        p.grad = torch.zeros_like(p)         # static gradient tensors
    fpol = None
    if fused:
        from srl_sim.policy import FusedA2CGrad, FusedClipRMSprop, FusedPolicy
        fpol = FusedPolicy(env.backend.library, policy, norm.state, seed=seed, env_offset=rank * num_envs, clip=norm.clip, eps=norm.eps)
        fgrad = FusedA2CGrad(env.backend.library, policy, T * N)
        fopt = FusedClipRMSprop(env.backend.library, policy, hp["max_grad_norm"], hp["alpha"], hp["epsilon"])
        ms = fopt.ms                         # in srl_mlp_grads order (srl_sim.policy.policy_params)
        act_dev = z(N, dtype=torch.int32) if env.is_discrete else z(N, env.sim.action_dim)
        done_u8 = z(H, T, N, dtype=torch.uint8)
    else:
        ms = [torch.ones_like(p) for p in params]
    if run.prefetch_resets and on_gpu:
        env.sim.prefetch_resets(stream=env.backend.stream())

    def collect(h):
        half = {k: v[h] for k, v in buf.items()}
        if fpol is not None:
            collect_rollout(run, norm, obs, stack, half, last_val[h], fused=fpol, act_dev=act_dev, done_u8=done_u8[h])
        else:
            collect_rollout(run, norm, obs, stack, half, last_val[h])

    def gradient(h):
        """Bootstrapped returns, then the loss gradient into the static ``.grad`` tensors."""
        flat = lambda k: buf[k][h].reshape((T * N,) + buf[k].shape[3:])
        st = env.backend.stream()
        if fused:
            fgrad.gae(buf["rew"][h], buf["val"][h], buf["done"][h], last_val[h], hp["gamma"], 1.0, adv[h], ret[h], stream=st)
            fgrad(None, flat("obs"), flat("act"), ret[h].reshape(-1), flat("val"), hp["ent_coef"], hp["vf_coef"], stream=st)
        else:
            with torch.no_grad():            # discount_with_dones over the rewards followed by the last value
                r = last_val[h]
                for t in reversed(range(T)):
                    r = buf["rew"][h, t] + hp["gamma"] * r * (1.0 - buf["done"][h, t])
                    ret[h, t].copy_(r)
            for p in params:
                p.grad.zero_()
            a2c_loss(policy, flat("obs"), flat("act"), ret[h].reshape(-1), flat("val"), hp["ent_coef"], hp["vf_coef"]).backward()
        if dist is not None:
            allreduce_mean_gradients(params, dist, world)

    def optimise(h):
        if fused:
            fopt(lr=lr_t[h:h + 1], stream=env.backend.stream())
        else:
            clip_rmsprop(params, ms, lr_t[h], hp["max_grad_norm"], hp["alpha"], hp["epsilon"])

    graph = None
    if use_graph:
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        rng0 = fpol.rng.clone()
        with torch.cuda.stream(side), torch.no_grad():
            st = env.backend.stream()
            # first launches outside the capture, on scratch outputs or undone after: the policy step (its sampling counter is restored), the
            # filter without an update, the torch value head, returns and gradient (overwritten before use), and the optimiser on zero
            # gradients (parameters unchanged; its slots are reset to 1), so that a captured run draws and computes what an eager one does
            fpol.act(N, obs, act_dev, buf["logp"][0, 0], buf["val"][0, 0], stream=st)
            if K > 1:
                fpol.stack_filter(N, env._obs, done_u8[0, 0], stack.clone(), torch.empty_like(obs), update=False, stream=st)
            else:
                fpol.filter(N, env._obs, obs, update=False, stream=st)
            for _ in range(3):
                policy.vf(obs)
            gradient(0)
            for p in params:
                p.grad.zero_()
            fopt(lr=lr_t[0:1], stream=st)
            for m in ms:
                m.fill_(1.0)
            fpol.rng.copy_(rng0)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):        # capture records the launches only: nothing advances
            for h in range(2):
                collect(h); gradient(h); optimise(h)

    # best-model callback every A2CModel.SAVE_INTERVAL = 10 callback calls of 1 env x 5 steps in the reference, scaled to this batch as for
    # PPO2; evaluated at most once per graph replay, after both of its updates
    log = RunLog(run, norm, log_dir, max(1, 10 * 1 * 5 // n_batch), episode_window, verbose)
    tick = phase_timer(phase_times, on_gpu)
    log.start()
    update = 0
    while update < n_updates:
        pair = 2 if graph is not None and update + 2 <= n_updates else 1
        for h in range(pair):
            lr_t[h].fill_(learning_rate(hp, update + h, n_batch, num_timesteps))
        if pair == 2:
            graph.replay()
        else:                                # eager: also the last, odd update of a graph run (its launches leave the double buffer in any phase)
            prior = (norm.mean.clone(), norm.var.clone(), norm.count.clone()) if dist is not None else None
            t_ph = tick()
            collect(0)
            if dist is not None:
                merge_running_moments(norm, prior, dist.all_reduce, world)
            t_ph = tick("collect", t_ph)
            gradient(0)
            t_ph = tick("grad", t_ph)
            optimise(0)
            tick("optimise", t_ph)
        # the episodes of the replay's rows, then one history entry per update (the first update of a replay already counts the episodes
        # of the second) and the best-model callback once, on the weights after both updates
        log.episodes(*(buf[k][:pair].reshape(pair * T, N) for k in ("done", "ep_ret", "ep_len")))
        for h in range(pair):
            update += 1
            log.end_update(update, n_updates, update * n_batch, callback=h == pair - 1, print_every=max(1, n_updates // 20))
    log.finish()
    env.close()
    train.best_mean_reward, train.n_saved = log.best_mean_reward, log.n_saved
    train.last_policy, train.last_norm, train.last_ms = policy, norm, ms
    # what the last replay (or eager update) started from and left behind, for tests that rebuild it: the initial parameters, the rollout
    # buffers of both halves, the returns and the learning rates
    train.last_update = dict(params0=params0, buf=buf, obs=obs, adv=adv, ret=ret, last_val=last_val, lr_t=lr_t)
    return log.history
