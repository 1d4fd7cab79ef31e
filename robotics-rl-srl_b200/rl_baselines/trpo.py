"""
TRPO consumer of the batched simulator: stable-baselines 2.5's ``TRPO`` with ``MlpPolicy`` behind ``VecNormalize``, as the reference trains it
through ``rl_baselines/rl_algorithm/trpo.py`` (timesteps_per_batch 128, entcoeff 0.01, vf_stepsize 2.5e-4, gamma 0.99, lam 0.95, cg_iters 4,
cg_damping 0.2, vf_iters 3, max_kl 0.01).  Restated in PyTorch next to rl_baselines/ppo2.py, whose policy, observation filter, env set-up,
collection loop and run bookkeeping it imports.

RECALLED from stable-baselines 2.5 / baselines' trpo_mpi, not checked against an installed copy (none can be installed here; re-pin when one
is): one update is a rollout of ``timesteps_per_batch`` steps, GAE(lambda) with ``tdlamret = adv + vpred``, ``atarg`` standardised with the
population std and no epsilon, ``optimgain = mean(ratio atarg) + entcoeff mean(entropy)`` against a copy of the policy, its gradient ``g`` (no
update when ``np.allclose(g, 0)``), ``stepdir = cg(fvp, g, cg_iters)`` with the Fisher-vector product ``fvp(v) = grad(grad(meankl) . v) +
cg_damping v`` on every 5th sample, ``lm = sqrt(|shs| / max_kl)`` with ``shs = 0.5 stepdir . fvp(stepdir)``, a backtracking line search of
ten trials at ``theta_old + fullstep / 2^k`` (rejected: non-finite losses, ``meankl > 1.5 max_kl`` or a negative improvement of optimgain;
theta_old restored after ten rejections), then ``vf_iters`` epochs of shuffled minibatches of 128 steps (no final partial batch), one MpiAdam
step each on ``mean((v - tdlamret)^2)``.

Batched rule (DESIGN.md section 5.4): every env runs T = timesteps_per_batch lockstep steps, so a batch is T x N rows; the FVP subsample is the
rows with t % 5 == 0 (ceil(T / 5) x N rows, contiguous [t, :] slices); a value minibatch is 128 x N rows, floor(T / 128) of them per epoch -- with
T < 128 the value function is never trained, as in the reference.

On the GPU the update runs on the library's kernels (include/srl_policy.h: srl_trpo_*): the surrogate gradient, cg_iters + 1 products, the
vector kernel that keeps the CG state and the line-search decision on the device, ten trial launches and the value steps -- no host
synchronisation inside an update.  With ``cuda_graph`` (single process, even T, no ``phase_times``) collection and update are ONE graph
replay; the value permutations are drawn into static index buffers before each replay.  The CPU path (the oracle backend of the tests) is
the torch statement below: torch distributions, the FVP by double backprop as TF takes it, float32 CG and line search as in baselines, MpiAdam.
"""
import math

import numpy as np
import torch

from rl_baselines.ppo2 import (RunLog, RunningNorm, collect_rollout, first_observation, make_run, merge_running_moments, phase_timer,
                               write_run_files)

TRPO_DEFAULTS = dict(timesteps_per_batch=128, max_kl=0.01, cg_iters=4, gamma=0.99, lam=0.95, entcoeff=0.01, cg_damping=0.2, vf_stepsize=2.5e-4,
                     vf_iters=3)   # rl_algorithm/trpo.py
VF_BATCH = 128            # dataset.iterbatches(batch_size=128, include_final_partial_batch=False)
FVP_STRIDE = 5            # fvpargs = [arr[::5] for arr in args]
MAX_TRIALS = 10
RESIDUAL_TOL = 1e-10
ADAM_BETA1, ADAM_BETA2, ADAM_EPS = 0.9, 0.999, 1e-8


def pi_params(policy):
    """The policy variables in the flat order of include/srl_policy.h: pi_w1, pi_b1, pi_w2, pi_b2, pi_w3, pi_b3, logstd (Box)."""
    ps = [t for m in policy.pi if hasattr(m, "weight") for t in (m.weight, m.bias)]
    return ps if policy.discrete else ps + [policy.logstd]


def vf_params(policy):
    return [t for m in policy.vf if hasattr(m, "weight") for t in (m.weight, m.bias)]


def flat(tensors):
    return torch.cat([t.reshape(-1) for t in tensors])


def set_flat(tensors, vec):
    off = 0
    with torch.no_grad():
        for t in tensors:
            t.copy_(vec[off:off + t.numel()].view_as(t))
            off += t.numel()


def categorical_kl(old_logits, new_logits):
    """stable-baselines' CategoricalProbabilityDistribution.kl: max-shifted logits."""
    a0 = old_logits - old_logits.max(-1, keepdim=True).values
    a1 = new_logits - new_logits.max(-1, keepdim=True).values
    z0, z1 = a0.exp().sum(-1, keepdim=True), a1.exp().sum(-1, keepdim=True)
    p0 = a0.exp() / z0
    return (p0 * (a0 - z0.log() - a1 + z1.log())).sum(-1)


def gaussian_kl(mu_old, ls_old, mu_new, ls_new):
    """stable-baselines' DiagGaussianProbabilityDistribution.kl."""
    return (ls_new - ls_old + (torch.exp(2 * ls_old) + (mu_old - mu_new) ** 2) / (2.0 * torch.exp(2 * ls_new)) - 0.5).sum(-1)


def trpo_losses(policy, old_out, old_logstd, obs, actions, atarg, entcoeff):
    """(optimgain, meankl, meanent, surrgain) of the policy against the old head outputs (logits or means) and old logstd, torch distributions."""
    z = policy.pi(obs)
    if policy.discrete:
        new, old = torch.distributions.Categorical(logits=z), torch.distributions.Categorical(logits=old_out)
        ratio = torch.exp(new.log_prob(actions) - old.log_prob(actions))
        kl, ent = categorical_kl(old_out, z), new.entropy()
    else:
        new = torch.distributions.Normal(z, policy.logstd.exp())
        old = torch.distributions.Normal(old_out, old_logstd.exp())
        ratio = torch.exp(new.log_prob(actions).sum(-1) - old.log_prob(actions).sum(-1))
        kl, ent = gaussian_kl(old_out, old_logstd, z, policy.logstd), new.entropy().sum(-1)
    surrgain, meankl, meanent = (ratio * atarg).mean(), kl.mean(), ent.mean()
    return surrgain + entcoeff * meanent, meankl, meanent, surrgain


def fvp_double_backprop(policy, obs_sub, v, damping):
    """grad(grad(meankl) . v) + damping v at the policy's weights, as TF takes it (the old distribution is a detached copy)."""
    params = pi_params(policy)
    with torch.no_grad():
        old_out = policy.pi(obs_sub)
        old_ls = None if policy.discrete else policy.logstd.detach().clone()
    z = policy.pi(obs_sub)
    kl = (categorical_kl(old_out, z) if policy.discrete else gaussian_kl(old_out, old_ls, z, policy.logstd)).mean()
    grads = torch.autograd.grad(kl, params, create_graph=True)
    gvp = (flat(grads) * v).sum()
    hvp = torch.autograd.grad(gvp, params)
    return flat(hvp).detach() + damping * v


def conjugate_gradient(f_Ax, b, cg_iters, residual_tol=RESIDUAL_TOL):
    """baselines' common/cg.py, float32: the loop breaks after updating p, once r.r < residual_tol.  Returns (x, iterations run, iterates)."""
    p, r, x = b.clone(), b.clone(), torch.zeros_like(b)
    rdotr = r.dot(r)
    iterates, n = [], 0
    for _ in range(cg_iters):
        z = f_Ax(p)
        v = rdotr / p.dot(z)
        x += v * p
        r -= v * z
        newrdotr = r.dot(r)
        mu = newrdotr / rdotr
        p = r + mu * p
        rdotr = newrdotr
        n += 1
        iterates.append(x.clone())
        if rdotr < residual_tol:
            break
    return x, n, iterates


def line_search(losses_at, surr_before, fullstep, max_kl, max_trials=MAX_TRIALS):
    """baselines' backtracking: trial k at scale 2^-k; ``losses_at(scale)`` -> (optimgain, meankl, *others).  Returns (accepted trial or -1,
    the trial losses)."""
    stepsize, tried = 1.0, []
    for k in range(max_trials):
        losses = [float(x) for x in losses_at(stepsize)]
        tried.append(losses)
        surr, kl = losses[0], losses[1]
        if not np.isfinite(losses).all():
            pass
        elif kl > max_kl * 1.5:
            pass
        elif surr - surr_before < 0:
            pass
        else:
            return k, tried
        stepsize *= 0.5
    return -1, tried


def vf_minibatches(T, N):
    """The value minibatches of one epoch: floor(T / 128) of 128 x N rows (none with T < 128)."""
    return [(b * VF_BATCH * N, (b + 1) * VF_BATCH * N) for b in range(T // VF_BATCH)]


def mpi_adam(params, grad, m, v, t, lr, beta1=ADAM_BETA1, beta2=ADAM_BETA2, eps=ADAM_EPS):
    """MpiAdam.update on the flat value vector (srl_trpo_vf_adam's statement, rl_baselines/ddpg.py's mpi_adam_polyak without targets)."""
    with torch.no_grad():
        f32 = lambda x: torch.tensor(x, dtype=torch.float32, device=grad.device)
        step = int(t[0]) + 1
        a = lr * math.sqrt(1 - beta2 ** step) / (1 - beta1 ** step)
        m.copy_(f32(beta1) * m + f32(1 - beta1) * grad)
        v.copy_(f32(beta2) * v + f32(1 - beta2) * (grad * grad))
        sqrt_v = torch.sqrt(v.double()).float()
        set_flat(params, flat(params) + (f32(-a) * m) / (sqrt_v + f32(eps)))
        t.add_(1)


def gae_torch(buf, last_val, gamma, lam, adv, ret):
    with torch.no_grad():
        T = buf["rew"].shape[0]
        lastgae = torch.zeros_like(last_val)
        for t in reversed(range(T)):
            nonterminal = 1.0 - buf["done"][t]
            nextval = last_val if t == T - 1 else buf["val"][t + 1]
            delta = buf["rew"][t] + gamma * nextval * nonterminal - buf["val"][t]
            lastgae = delta + gamma * lam * nonterminal * lastgae
            adv[t].copy_(lastgae)
        torch.add(adv, buf["val"], out=ret)


def policy_step_torch(policy, obs, actions, adv, obs_sub, hp, all_reduce_mean=None):
    """The policy half of one update in torch (the oracle backend's path): standardise ``adv`` (population std), the gradient of optimgain
    against a copy of the policy, the zero-gradient skip, CG on the double-backprop FVP over ``obs_sub``, the step size and the line search,
    which leaves the accepted point or theta_old in the policy.  ``all_reduce_mean``: a mean over data-parallel ranks, or None.  Returns a record
    of what it did: g, atarg, skip, cg_iters, iterates, stepdir, nonfinite, shs, fullstep, accepted (-1 for none), restored, trials."""
    pis = pi_params(policy)
    atarg = (adv - adv.mean()) / adv.std(unbiased=False)
    with torch.no_grad():
        old_out = policy.pi(obs).detach()
        old_ls = None if policy.discrete else policy.logstd.detach().clone()
    gain, kl, ent, surr = trpo_losses(policy, old_out, old_ls, obs, actions, atarg, hp["entcoeff"])
    g = flat(torch.autograd.grad(gain, pis)).detach()
    losses_before = torch.stack([surr.detach(), ent.detach()]).double()
    if all_reduce_mean is not None:
        all_reduce_mean(g); all_reduce_mean(losses_before)
    gain_before = float(losses_before[0] + hp["entcoeff"] * losses_before[1])
    rec = dict(g=g, atarg=atarg, skip=bool(torch.allclose(g, torch.zeros_like(g), rtol=1e-5, atol=1e-8)), accepted=-1, restored=False, cg_iters=0,
               nonfinite=False, gain_before=gain_before)
    if rec["skip"]:                  # np.allclose(g, 0): "Got zero gradient. not updating"
        return rec

    def fvp(v):
        out = fvp_double_backprop(policy, obs_sub, v, 0.0)
        if all_reduce_mean is not None:
            all_reduce_mean(out)
        return out + hp["cg_damping"] * v
    stepdir, n_it, iterates = conjugate_gradient(fvp, g, hp["cg_iters"])
    rec.update(cg_iters=n_it, iterates=iterates, stepdir=stepdir)
    if not torch.isfinite(stepdir).all():
        rec["nonfinite"] = True
        return rec
    shs = 0.5 * stepdir.dot(fvp(stepdir))
    lm = torch.sqrt(torch.abs(shs) / hp["max_kl"])
    fullstep = stepdir / lm
    th_before = flat(pis).detach().clone()

    def losses_at(scale):
        set_flat(pis, th_before + fullstep * scale)
        with torch.no_grad():
            out = torch.stack([x.detach() for x in trpo_losses(policy, old_out, old_ls, obs, actions, atarg, hp["entcoeff"])]).double()
        if all_reduce_mean is not None:
            all_reduce_mean(out)
        return out.tolist()
    k, tried = line_search(losses_at, gain_before, fullstep, hp["max_kl"])
    set_flat(pis, th_before if k < 0 else th_before + fullstep * 0.5 ** k)
    rec.update(shs=float(shs), fullstep=fullstep, accepted=k, restored=k < 0, trials=tried)
    return rec


def value_steps_torch(policy, obs, ret, perms, mbs, adam, hp, all_reduce_mean=None):
    """The value half of one update in torch: per permutation (one per epoch) and minibatch (``mbs``), one MpiAdam step on mean((v - ret)^2).
    ``adam`` = (m, v, step) over the flat value vector."""
    vfs = vf_params(policy)
    for perm in perms:
        for s, e in mbs:
            idx = perm[s:e]
            loss = ((policy.vf(obs[idx]).squeeze(-1) - ret[idx]) ** 2).mean()
            vg = flat(torch.autograd.grad(loss, vfs)).detach()
            if all_reduce_mean is not None:
                all_reduce_mean(vg)
            mpi_adam(vfs, vg, *adam, hp["vf_stepsize"])


def train(env_id, num_envs, num_timesteps, seed=0, env_kwargs=None, log_dir=None, device=0, hyperparams=None, verbose=1, cuda_graph=True,
          phase_times=None, prefetch_resets=None, episode_window=40, num_stack=1):
    """TRPO.learn on a BatchedSRLVecEnv.  Returns a history of (timesteps, mean episode return, fps), one entry per update.
    ``cuda_graph``, ``phase_times`` (``collect`` / ``policy`` / ``value``, eager), ``num_stack``, ``prefetch_resets``, ``episode_window``: as for
    rl_baselines.ppo2.train.  ``train.last_update`` keeps what the last update started from and left behind, and its status record."""
    hp = dict(TRPO_DEFAULTS); hp.update(hyperparams or {})
    torch.manual_seed(seed)
    run = make_run("trpo", env_id, num_envs, seed, env_kwargs, device, prefetch_resets, num_stack, [None])
    env, on_gpu, dev, policy, dist, rank, world, K, W = run.env, run.on_gpu, run.dev, run.policy, run.dist, run.rank, run.world, run.K, run.W
    N, T = num_envs, int(hp["timesteps_per_batch"])
    rows, sub_rows = T * N, ((T + FVP_STRIDE - 1) // FVP_STRIDE) * N
    n_updates = max(1, int(num_timesteps) // (N * T * world))
    mbs = vf_minibatches(T, N)
    norm = RunningNorm(W, dev)
    write_run_files(run, log_dir, num_timesteps, seed, hp)
    obs, stack = first_observation(run, norm)
    z = lambda *shape, dtype=torch.float32: torch.zeros(shape, device=dev, dtype=dtype)
    buf = dict(obs=z(T, N, W), act=z(T, N, dtype=torch.int64) if env.is_discrete else z(T, N, env.sim.action_dim), logp=z(T, N), val=z(T, N),
               rew=z(T, N), done=z(T, N), ep_ret=z(T, N), ep_len=z(T, N, dtype=torch.int32))
    last_val, adv, ret = z(N), z(T, N), z(T, N)
    flat_obs, flat_act, flat_ret = buf["obs"].reshape(rows, W), buf["act"].reshape((rows,) + buf["act"].shape[2:]), ret.reshape(-1)
    pis, vfs = pi_params(policy), vf_params(policy)
    vidx = z(max(1, hp["vf_iters"] * len(mbs)), VF_BATCH * N, dtype=torch.int64)   # the value minibatches' rows, drawn before each update
    all_reduce_mean = (lambda x: (dist.all_reduce(x), x.div_(world))) if dist is not None else None
    fused = None
    if on_gpu:
        from srl_sim.policy import FusedPolicy, FusedTRPO, ppo2_gae
        fpol = FusedPolicy(env.backend.library, policy, norm.state, seed=seed, env_offset=rank * num_envs, clip=norm.clip, eps=norm.eps)
        fused = FusedTRPO(env.backend.library, policy, rows)
        act_dev = z(N, dtype=torch.int32) if env.is_discrete else z(N, env.sim.action_dim)
        done_u8 = z(T, N, dtype=torch.uint8)
        adam_m, adam_v, adam_t = fused.m, fused.v, fused.step
        if run.prefetch_resets:
            env.sim.prefetch_resets(stream=env.backend.stream())
    else:
        adam_m, adam_v, adam_t = torch.zeros_like(flat(vfs)), torch.zeros_like(flat(vfs)), torch.zeros(1, dtype=torch.int64)

    def collect():
        if fused is not None:
            collect_rollout(run, norm, obs, stack, buf, last_val, fused=fpol, act_dev=act_dev, done_u8=done_u8)
        else:
            collect_rollout(run, norm, obs, stack, buf, last_val)

    def policy_update_gpu():
        st = env.backend.stream()
        ppo2_gae(env.backend.library, buf["rew"], buf["val"], buf["done"], last_val, hp["gamma"], hp["lam"], adv, ret, stream=st)
        fused.surrogate(flat_obs, flat_act, adv.reshape(-1), hp["entcoeff"], stream=st)
        if dist is not None:
            all_reduce_mean(fused.g); all_reduce_mean(fused.losses)
        fused.vector(0, hp["max_kl"], hp["entcoeff"], stream=st)
        for i in range(hp["cg_iters"] + 1):
            fused.fvp(sub_rows, N, FVP_STRIDE * N, flat_obs, fused.p if i < hp["cg_iters"] else fused.x, hp["cg_damping"], fused.z, stream=st)
            if dist is not None:
                all_reduce_mean(fused.z)
            fused.vector(1 if i < hp["cg_iters"] else 2, hp["max_kl"], hp["entcoeff"], stream=st)
        for _ in range(MAX_TRIALS):
            fused.trial(flat_obs, flat_act, stream=st)
            if dist is not None:
                all_reduce_mean(fused.losses)
            fused.vector(3, hp["max_kl"], hp["entcoeff"], stream=st)

    def value_update_gpu():
        st = env.backend.stream()
        for b in range(vidx.shape[0] if mbs else 0):
            fused.vf_grad(VF_BATCH * N, vidx[b], flat_obs, flat_ret, stream=st)
            if dist is not None:
                all_reduce_mean(fused.vgrad)
            fused.vf_adam(hp["vf_stepsize"], stream=st)

    def update_cpu():
        """The torch statement of one update after the rollout (the oracle backend's path); returns its record."""
        gae_torch(buf, last_val, hp["gamma"], hp["lam"], adv, ret)
        rec = policy_step_torch(policy, flat_obs, flat_act, adv.reshape(-1), buf["obs"][::FVP_STRIDE].reshape(-1, W), hp, all_reduce_mean)
        value_steps_torch(policy, flat_obs, flat_ret, [torch.randperm(rows) for _ in range(hp["vf_iters"])], mbs, (adam_m, adam_v, adam_t), hp,
                          all_reduce_mean)
        return rec

    def draw_value_rows():
        if not mbs:
            return
        b = 0
        for _ in range(hp["vf_iters"]):
            perm = torch.randperm(rows, device=dev)
            for s, e in mbs:
                vidx[b].copy_(perm[s:e]); b += 1

    graph = None
    if cuda_graph and on_gpu and dist is None and phase_times is None and T % 2 == 0:
        # first launches outside the capture, undone after: the policy step (its counter restored), the filter without an update, the torch
        # value head, and one update on the current buffers (parameters and value optimiser restored), so that nothing is first called inside it
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        rng0 = fpol.rng.clone()
        saved = [t.detach().clone() for t in pis + vfs + [adam_m, adam_v, adam_t]]
        with torch.cuda.stream(side), torch.no_grad():
            st = env.backend.stream()
            fpol.act(N, obs, act_dev, buf["logp"][0], buf["val"][0], stream=st)
            if K > 1:
                fpol.stack_filter(N, env._obs, done_u8[0], stack.clone(), torch.empty_like(obs), update=False, stream=st)
            else:
                fpol.filter(N, env._obs, obs, update=False, stream=st)
            for _ in range(3):
                policy.vf(obs)
            policy_update_gpu(); value_update_gpu()
            for t, s in zip(pis + vfs + [adam_m, adam_v, adam_t], saved):
                t.copy_(s)
            fpol.rng.copy_(rng0)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph), torch.no_grad():
            collect(); policy_update_gpu(); value_update_gpu()

    log = RunLog(run, norm, log_dir, 1, episode_window, verbose)     # SAVE_INTERVAL = 1: the best-model callback after every update
    tick = phase_timer(phase_times, on_gpu)
    log.start()
    params0, record = None, {}
    for update in range(1, n_updates + 1):
        params0 = [t.detach().clone() for t in pis + vfs]
        adam0 = [t.detach().clone() for t in (adam_m, adam_v, adam_t)]
        if on_gpu:
            draw_value_rows()
        if graph is not None:
            graph.replay()
        else:
            prior = (norm.mean.clone(), norm.var.clone(), norm.count.clone()) if dist is not None else None
            t_ph = tick()
            collect()
            if dist is not None:
                merge_running_moments(norm, prior, dist.all_reduce, world)
            t_ph = tick("collect", t_ph)
            if on_gpu:
                with torch.no_grad():
                    policy_update_gpu()
                t_ph = tick("policy", t_ph)
                with torch.no_grad():
                    value_update_gpu()
            else:
                record = update_cpu()
            tick("value", t_ph)
        log.episodes(buf["done"], buf["ep_ret"], buf["ep_len"])      # synchronises: the status record below is ready
        if on_gpu:
            s = fused.state.cpu().numpy()
            record = dict(skip=bool(s[0]), cg_iters=int(s[1]), nonfinite=bool(s[3]), accepted=int(s[4]), restored=bool(s[5]), state=s)
        if record.get("nonfinite"):
            raise FloatingPointError("TRPO: the conjugate-gradient step direction is not finite (update %d)" % update)
        log.end_update(update, n_updates, update * N * T * world)
    log.finish()
    env.close()
    train.best_mean_reward, train.n_saved = log.best_mean_reward, log.n_saved
    train.last_policy, train.last_norm = policy, norm
    train.last_update = dict(params0=params0, adam0=adam0, adam=(adam_m, adam_v, adam_t), buf=buf, adv=adv, ret=ret, last_val=last_val,
                             vidx=vidx if on_gpu else None, record=record, fused=fused, graph=graph is not None, hp=hp)
    return log.history
