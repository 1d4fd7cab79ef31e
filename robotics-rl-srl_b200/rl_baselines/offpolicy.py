"""
The replay-ring loop that the SAC (rl_baselines/sac.py) and DDPG (rl_baselines/ddpg.py) trainers share.  Both keep a ring of ``buffer_size``
rows of N transitions, written row ``t % buffer_size`` at lockstep step t by ``srl_sac_store`` on the GPU, and run their lockstep steps in
blocks of G steps with ONE captured CUDA graph replayed for every block whose steps do the same work.  :func:`setup` builds the run and its
buffers, :func:`learn` runs the steps; the trainer brings its networks, its action, its gradient step and the schedule of both (``cadence``).
"""
import types

import torch

from rl_baselines.ppo2 import RunLog, RunningNorm, first_observation, make_run, merge_running_moments, phase_timer, write_run_files


def ring_bytes(rows, n_envs, W, A):
    """Device bytes of the replay ring: obs and next_obs f32[rows, N, W], act f32[rows, N, A], rew f32 and done u8 [rows, N]."""
    return int(rows) * int(n_envs) * (4 * (2 * W + A + 1) + 1)


def setup(algo, network, env_id, num_envs, num_timesteps, seed, env_kwargs, log_dir, device, hp, verbose, fused, cuda_graph, phase_times,
          prefetch_resets, episode_window, num_stack, step_bytes):
    """The run of an off-policy trainer, up to its first step: the envs and ``network(W, A)`` (make_run's, the target synchronised), the
    observation filter and the first observation ``obs``, the ring (``ring``, and ``flat``: its [rows N, ...] views), the gradient arena
    ``grad``, the action ``act_dev`` and the done flags ``done_s`` of the current step, and on the GPU (``fused``) the filter and store
    launches.  ``step_bytes(B, W, A, sms)``: the device bytes of one gradient step beside the ring; a ring and step that do not fit in free
    device memory are refused before anything is allocated.  Call after ``torch.manual_seed(seed)``."""
    run = make_run(algo, env_id, num_envs, seed, env_kwargs, device, prefetch_resets, num_stack, [fused],
                   network=lambda width, env: network(width, env.action_space.shape[0]))
    env, on_gpu, dev, nets, W = run.env, run.on_gpu, run.dev, run.policy, run.W
    nets.sync_target()                                        # after make_run's broadcast: every rank starts from one network
    A = nets.act_dim
    if fused is None:
        fused = on_gpu
    if fused and not on_gpu:
        raise ValueError("fused=True needs the CUDA library (there is no CPU fallback)")
    N, rows = num_envs, hp["buffer_size"]
    B = hp["batch_size"] * N
    if on_gpu:                                                # before the ring or any step buffer is allocated
        nbytes = ring_bytes(rows, N, W, A) + step_bytes(B, W, A, torch.cuda.get_device_properties(dev).multi_processor_count)
        free, _ = torch.cuda.mem_get_info(dev)
        if nbytes > free:
            env.close()
            raise ValueError("the replay ring of --buffer-size %d rows x %d envs and the gradient step's buffers need %.2f GB and the device has "
                             "%.2f GB free: lower --buffer-size or --num-cpu" % (rows, N, nbytes / 1e9, free / 1e9))
    norm = RunningNorm(W, dev)
    write_run_files(run, log_dir, num_timesteps, seed, hp)
    obs, stack = first_observation(run, norm)
    z = lambda *shape, dtype=torch.float32: torch.zeros(shape, device=dev, dtype=dtype)
    ring = dict(obs=z(rows, N, W), next_obs=z(rows, N, W), act=z(rows, N, A), rew=z(rows, N), done=z(rows, N, dtype=torch.uint8))
    grad = torch.zeros_like(nets.arena.data)
    nets.arena.grad = grad                                   # the gradient arena, what allreduce_mean_gradients averages
    ctx = types.SimpleNamespace(run=run, env=env, dev=dev, nets=nets, dist=run.dist, rank=run.rank, world=run.world, N=N, W=W, A=A,
                                B=B, rows=rows, n_steps=max(1, int(num_timesteps) // (N * run.world)), fused=fused, norm=norm, obs=obs.contiguous(),
                                stack=stack, ring=ring, flat={k: v.reshape((rows * N,) + v.shape[2:]) for k, v in ring.items()}, grad=grad,
                                act_dev=z(N, A), done_s=z(N, dtype=torch.uint8), fstore=None, before_first_step=None, log_dir=log_dir,
                                episode_window=episode_window, verbose=verbose,
                                use_graph=bool(cuda_graph and fused and run.dist is None and phase_times is None))
    if fused:
        from srl_sim.policy import FusedObsFilter, FusedSACStore
        ctx.ffilter = FusedObsFilter(env.backend.library, norm.state, clip=norm.clip, eps=norm.eps)
        ctx.fstore = FusedSACStore(env.backend.library, ring, dev)
        ctx.rew_s, ctx.new_obs = z(N), z(N, W)
    if run.prefetch_resets and on_gpu:
        env.sim.prefetch_resets(stream=env.backend.stream())
    ctx.tick = phase_timer(phase_times, on_gpu)
    return ctx


def learn(ctx, period, G, cadence, act, gradient_step, adam_state):
    """The lockstep steps of the run, in blocks of G steps.  Step t: ``cadence(t)`` gives (random action, one target-update flag per
    gradient step); ``act(random_action)`` writes the action into ``ctx.act_dev``; then the env step, the filter (with the frame stack) and
    the store into ring row t % rows; then ``gradient_step(t, polyak)`` for each flag.  ``adam_state``: the trainer's optimiser tensors by
    name, copied with the parameters into ``ctx.before_first_step`` before the first gradient step.

    ``ctx.use_graph``: a block is ONE CUDA graph replay when it is full, a gradient step has already run (eagerly: it warmed every kernel
    up), no step takes a random action, and its gradient steps and target updates, step by step, are those of the captured block; the
    first such block is captured.  The ring row, the sampling counters and every optimiser input are read on the device, so one graph
    serves every such block.  Every other block runs the same launches eagerly.  After each block the per-rank filters are merged
    (data-parallel); the log takes one history entry per ``period`` steps.  Returns (the RunLog, the step counts)."""
    env, run, nets, norm, ring, dist, world, N, W, tick = ctx.env, ctx.run, ctx.nets, ctx.norm, ctx.ring, ctx.dist, ctx.world, ctx.N, ctx.W, ctx.tick
    z = lambda *shape, dtype=torch.float32: torch.zeros(shape, device=ctx.dev, dtype=dtype)
    block = dict(done=z(G, N), ep_ret=z(G, N), ep_len=z(G, N, dtype=torch.int32))
    obs, stack, act_dev, done_s = ctx.obs, ctx.stack, ctx.act_dev, ctx.done_s
    stats = dict(grad_steps=0, target_updates=0, graph_replays=0, graphs=0)

    def env_step(t, k, random_action):
        st = env.backend.stream()
        with torch.no_grad():
            act(random_action)
            if ctx.fused:
                env.sim.step(act_dev, None, env._obs, ctx.rew_s, done_s, block["ep_ret"][k], block["ep_len"][k], stream=st)
                if run.K > 1:
                    ctx.ffilter.stack_filter(N, env._obs, done_s, stack, ctx.new_obs, update=True, stream=st)
                else:
                    ctx.ffilter.filter(N, env._obs, ctx.new_obs, update=True, stream=st)
                ctx.fstore(obs, act_dev, ctx.rew_s, done_s, ctx.new_obs, stream=st)          # ring row t % rows, then obs <- new_obs
                block["done"][k].copy_(done_s)
                return
            row = t % ctx.rows
            ring["obs"][row].copy_(obs); ring["act"][row].copy_(act_dev)
            env.step_tensors(act_dev)
            ring["rew"][row].copy_(run.e_rew); ring["done"][row].copy_(run.e_done); done_s.copy_(run.e_done)
            block["done"][k].copy_(run.e_done); block["ep_ret"][k].copy_(run.e_ep_ret); block["ep_len"][k].copy_(run.e_ep_len)
            if run.K > 1:                                    # VecFrameStack.step
                stack.copy_(torch.where(run.e_done.bool()[:, None], 0.0, torch.roll(stack, -run.D, 1)))
                stack[:, W - run.D:].copy_(run.e_obs)
                ring["next_obs"][row].copy_(norm(stack))
            else:
                ring["next_obs"][row].copy_(norm(run.e_obs))
            obs.copy_(ring["next_obs"][row])

    def run_block(t0, steps):
        for k in range(steps):
            t = t0 + k
            random_action, targets = cadence(t)
            t_ph = tick()
            env_step(t, k, random_action)
            tick("collect", t_ph)
            for polyak in targets:
                if stats["grad_steps"] == 0:                 # what a test needs to redo the first gradient step
                    ctx.before_first_step = dict(arena=nets.arena.detach().clone(), target=nets.target.clone(),
                                                 **{name: x.clone() for name, x in adam_state.items()})
                gradient_step(t, polyak)
                stats["grad_steps"] += 1
                stats["target_updates"] += int(polyak)

    graph, graph_targets = None, None
    log = RunLog(run, norm, ctx.log_dir, max(1, 200 // (period * N * world)), ctx.episode_window, ctx.verbose)
    log.start()
    n_periods = (ctx.n_steps + period - 1) // period
    t0, p_i = 0, 0
    while t0 < ctx.n_steps:
        steps = min(G, ctx.n_steps - t0)
        prior = (norm.mean.clone(), norm.var.clone(), norm.count.clone()) if dist is not None else None
        pattern = [cadence(t) for t in range(t0, t0 + G)] if ctx.use_graph and stats["grad_steps"] and steps == G else None
        targets = None if pattern is None or any(r for r, _ in pattern) else [tg for _, tg in pattern]
        if targets is not None and (graph is None or targets == graph_targets):
            if graph is None:
                graph, graph_targets, counts = torch.cuda.CUDAGraph(), targets, dict(stats)
                with torch.cuda.graph(graph):                  # capture records the launches only: nothing advances
                    run_block(t0, G)
                stats.update(counts, graphs=1)
            graph.replay()
            stats["graph_replays"] += 1
            stats["grad_steps"] += sum(len(tg) for tg in targets)
            stats["target_updates"] += sum(sum(tg) for tg in targets)
        else:
            run_block(t0, steps)
        if dist is not None:
            merge_running_moments(norm, prior, dist.all_reduce, world)
        for k0 in range(0, steps, period):
            n = min(period, steps - k0)
            log.episodes(block["done"][k0:k0 + n], block["ep_ret"][k0:k0 + n], block["ep_len"][k0:k0 + n])
            p_i += 1
            log.end_update(p_i, n_periods, (t0 + k0 + n) * N * world, print_every=max(1, n_periods // 20))
        t0 += steps
    log.finish()
    env.close()
    return log, stats
