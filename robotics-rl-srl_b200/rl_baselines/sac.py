"""
SAC consumer of the batched simulator: stable-baselines 2.5's ``SAC`` with its ``MlpPolicy`` behind ``VecNormalize``, as the reference trains it
through ``rl_baselines/rl_algorithm/sac.py``.  That file passes only ``--hyperparam`` values to the model (its ``--ent-coef`` and
``--batch-size`` are parsed and never used), so the library's defaults apply: gamma 0.99, learning_rate 3e-4 (constant), buffer_size 50 000,
learning_starts 100, train_freq 1, batch_size 64, tau 0.005, ent_coef 'auto' (log_ent_coef from 0, target_entropy = -action_dim),
target_update_interval 1, gradient_steps 1.  Restated in PyTorch next to rl_baselines/deepq.py, whose batched rule it follows; the replay-ring
loop is rl_baselines/offpolicy.py, shared with DDPG.

RECALLED from stable-baselines 2.5, not checked against an installed copy (none can be installed here; include/srl_policy.h): the defaults
above; the networks (layers [64, 64], ReLU, glorot-uniform weights and zero biases; an actor trunk with separate ``mu`` and ``log_std`` heads,
log_std clipped to [-20, 2]; qf1 and qf2 on concat(obs, action); vf and its target); the squashed Gaussian and its log-probability as the TF
graph writes it; the losses and which of the three Adam optimisers owns which variables; the Polyak update after the Adam steps; and the
learn loop's conditions (:func:`cadence`).

Batched semantics (DQN's, unchanged).  N envs per rank step in lockstep; t, learning_starts, train_freq and target_update_interval count
lockstep steps.  The ring holds ``buffer_size`` rows of N transitions and a gradient step samples ``batch_size N`` transitions uniformly, with
replacement, from the stored ones (``ReplayBuffer.sample``).  Per lockstep step t (from 0):
  act (uniform random while t < learning_starts), step, store (obs, a, r, new_obs, done) in ring row t % buffer_size, obs = new_obs;
  if t % train_freq == 0: up to gradient_steps gradient steps (none while t + 1 < batch_size or t + 1 < learning_starts), each followed by
  the target update when (t + grad_step) % target_update_interval == 0.
Data-parallel (torchrun): every rank keeps its own ring; the gradient arena is all-reduced (mean) before Adam; the observation filter is
merged once per block.

On the GPU (``fused``) every step is the library's kernels: ``srl_sac_act``, ``srl_sim_step``, the filter, ``srl_sac_store``; a gradient step
is ``srl_sac_prepare``, ``srl_sac_grad``, ``srl_sac_adam``.  The parameters live in one flat arena (:class:`SACNets`), so the gradient, the
Adam slots and the all-reduce are single tensors.  The CPU path (the oracle backend of the tests, and ``fused=False``) runs the same algorithm
in torch: :func:`sac_losses`, :func:`adam_polyak` and uniform sampling with torch's generator.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from rl_baselines import offpolicy
from rl_baselines.ppo2 import allreduce_mean_gradients

SAC_DEFAULTS = dict(gamma=0.99, learning_rate=3e-4, buffer_size=50000, learning_starts=100, train_freq=1, batch_size=64, tau=0.005,
                    ent_coef="auto", target_update_interval=1, gradient_steps=1)          # stable-baselines 2.5 SAC (RECALLED)
ADAM_BETA1, ADAM_BETA2, ADAM_EPS = 0.9, 0.999, 1e-8     # tf.train.AdamOptimizer's defaults
LOG_STD_MIN, LOG_STD_MAX, SQUASH_EPS = -20.0, 2.0, 1e-6
DISCRETE_ERROR = "sac does not support discrete actions, please use the '--continuous-actions' (or '-c') flag."
HIDDEN = 64


def net_layout(W, A):
    """Offsets of the arena (include/srl_policy.h: srl_sac_nets): {name: {tensor: (offset, shape)}} for actor, qf1, qf2, vf, and
    ``log_ent_coef`` / ``P``."""
    lay, off = {}, 0
    for name, n_in, n_out in (("actor", W, 2 * A), ("qf1", W + A, 1), ("qf2", W + A, 1), ("vf", W, 1)):
        t = {}
        for key, shape in (("w1", (HIDDEN, n_in)), ("b1", (HIDDEN,)), ("w2", (HIDDEN, HIDDEN)), ("b2", (HIDDEN,)), ("w3", (n_out, HIDDEN)), ("b3", (n_out,))):
            t[key] = (off, shape)
            off += int(np.prod(shape))
        t["end"] = off
        lay[name] = t
    lay["log_ent_coef"], lay["P"] = off, off + 1
    return lay


class SACNets(nn.Module):
    """The five networks of the SAC MlpPolicy in one flat float32 parameter ``arena`` (actor | qf1 | qf2 | vf | log_ent_coef) and the target
    value network in the buffer ``target`` (vf's layout).  Weights glorot-uniform, biases zero (``tf.layers.dense``), log_ent_coef 0, the
    target a copy of vf."""
    discrete = False

    def __init__(self, obs_dim, act_dim):
        super().__init__()
        self.obs_dim, self.act_dim = int(obs_dim), int(act_dim)
        self.layout = net_layout(self.obs_dim, self.act_dim)
        arena = torch.zeros(self.layout["P"])
        for name in ("actor", "qf1", "qf2", "vf"):
            for key in ("w1", "w2", "w3"):
                off, shape = self.layout[name][key]
                if name == "actor" and key == "w3":            # two dense heads, each glorot-uniform over (64, A)
                    for h in range(2):
                        lim = math.sqrt(6.0 / (HIDDEN + self.act_dim))
                        n = self.act_dim * HIDDEN
                        arena[off + h * n:off + (h + 1) * n].uniform_(-lim, lim)
                    continue
                lim = math.sqrt(6.0 / (shape[0] + shape[1]))
                arena[off:off + int(np.prod(shape))].uniform_(-lim, lim)
        self.arena = nn.Parameter(arena)
        lo, hi = self.layout["vf"]["w1"][0], self.layout["vf"]["end"]
        self.register_buffer("target", arena[lo:hi].clone())

    def tensors(self, name, source=None):
        """The six tensors of network ``name`` as views of ``source`` (default: the arena; the target for ``vf_target``)."""
        if name == "vf_target":
            base, lay, src = self.layout["vf"]["w1"][0], self.layout["vf"], self.target if source is None else source
        else:
            base, lay, src = 0, self.layout[name], self.arena if source is None else source
        return [src[off - base:off - base + int(np.prod(shape))].view(shape) for off, shape in (lay[k] for k in ("w1", "b1", "w2", "b2", "w3", "b3"))]

    def mlp(self, name, x, source=None):
        w1, b1, w2, b2, w3, b3 = self.tensors(name, source)
        h = torch.relu(x @ w1.t() + b1)
        h = torch.relu(h @ w2.t() + b2)
        return h @ w3.t() + b3

    def actor(self, obs, source=None):
        """(mu, raw log_std) of the actor's two heads."""
        out = self.mlp("actor", obs, source)
        return out[..., :self.act_dim], out[..., self.act_dim:]

    @property
    def log_ent_coef(self):
        return self.arena[self.layout["log_ent_coef"]]

    def sync_target(self):
        lo, hi = self.layout["vf"]["w1"][0], self.layout["vf"]["end"]
        with torch.no_grad():
            self.target.copy_(self.arena[lo:hi])

    def act(self, obs, deterministic=False):
        """tanh(mu), or tanh(mu + std z) with z from torch's generator."""
        mu, ls = self.actor(obs)
        if deterministic:
            return torch.tanh(mu)
        return torch.tanh(mu + torch.exp(torch.clamp(ls, LOG_STD_MIN, LOG_STD_MAX)) * torch.randn_like(mu))


def squashed_logp(mu, log_std, eps):
    """(a_pi, logp_pi) of the reparameterised sample: u = mu + std eps, a = tanh(u), log-probability as stable-baselines' TF graph writes it."""
    log_std = torch.clamp(log_std, LOG_STD_MIN, LOG_STD_MAX)
    std = torch.exp(log_std)
    u = mu + std * eps
    logp = (-0.5 * (((u - mu) / (std + SQUASH_EPS)) ** 2 + 2 * log_std + math.log(2 * math.pi))).sum(-1)
    a = torch.tanh(u)
    return a, logp - torch.log(1 - a ** 2 + SQUASH_EPS).sum(-1)


def sac_losses(nets, obs, act, rew, next_obs, done, eps, gamma, ent_coef, target_entropy):
    """One step's losses from the parameters as they are (SAC.setup_model; ``ent_coef`` a float, or None for 'auto').  Returns a dict with
    ``total``, whose gradient with respect to the arena is each optimiser's gradient on its own variables: policy_loss on the actor,
    qf1_loss + qf2_loss + value_loss on qf1, qf2 and vf, ent_coef_loss on log_ent_coef; and q_backup, v_backup, logp and the losses."""
    alpha = torch.exp(nets.log_ent_coef) if ent_coef is None else torch.tensor(float(ent_coef), dtype=obs.dtype, device=obs.device)
    frozen = nets.arena.detach()
    with torch.no_grad():
        v_t = nets.mlp("vf_target", next_obs).squeeze(-1)
        q_backup = rew + gamma * ((1 - done) * v_t)
    mu, ls = nets.actor(obs)
    a_pi, logp = squashed_logp(mu, ls, eps)
    x_pi = torch.cat([obs, a_pi], -1)
    qf1_pi = nets.mlp("qf1", x_pi, frozen).squeeze(-1)            # the policy optimiser moves the actor only
    with torch.no_grad():
        qf2_pi = nets.mlp("qf2", x_pi, frozen).squeeze(-1)
        v_backup = torch.min(qf1_pi, qf2_pi) - alpha.detach() * logp
    x = torch.cat([obs, act], -1)
    qf1, qf2, vf = nets.mlp("qf1", x).squeeze(-1), nets.mlp("qf2", x).squeeze(-1), nets.mlp("vf", obs).squeeze(-1)
    qf1_loss, qf2_loss = 0.5 * ((q_backup - qf1) ** 2).mean(), 0.5 * ((q_backup - qf2) ** 2).mean()
    value_loss = 0.5 * ((vf - v_backup) ** 2).mean()
    policy_loss = (alpha.detach() * logp - qf1_pi).mean()
    ent_coef_loss = -(nets.log_ent_coef * (logp.detach() + target_entropy)).mean() if ent_coef is None else torch.zeros((), device=obs.device)
    total = policy_loss + qf1_loss + qf2_loss + value_loss + ent_coef_loss
    return dict(total=total, q_backup=q_backup, v_backup=v_backup.detach(), logp=logp.detach(), policy_loss=policy_loss, qf1_loss=qf1_loss,
                qf2_loss=qf2_loss, value_loss=value_loss, ent_coef_loss=ent_coef_loss)


def adam_polyak(nets, grad, m, v, beta_power, lr, tau, polyak, beta1=ADAM_BETA1, beta2=ADAM_BETA2, eps=ADAM_EPS):
    """TF1 Adam over the arena (the torch statement of srl_sac_adam, in its order of float32 roundings), then ``target = (1 - tau) target
    + tau vf`` from the updated vf when ``polyak``; ``beta_power`` (float32 [2]) is multiplied by {beta1, beta2} after the step."""
    with torch.no_grad():
        f32 = lambda x: torch.tensor(x, dtype=torch.float32, device=beta_power.device)
        lr_t = (f32(lr) * torch.sqrt(1.0 - beta_power[1])) / (1.0 - beta_power[0])
        m.add_((grad - m) * (f32(1.0) - f32(beta1)))
        v.add_((grad * grad - v) * (f32(1.0) - f32(beta2)))
        nets.arena.sub_((m * lr_t) / (torch.sqrt(v) + eps))
        if polyak:
            lo, hi = nets.layout["vf"]["w1"][0], nets.layout["vf"]["end"]
            nets.target.copy_((f32(1.0) - f32(tau)) * nets.target + f32(tau) * nets.arena[lo:hi])
        beta_power.mul_(torch.stack([f32(beta1), f32(beta2)]))


def cadence(t, hp):
    """SAC.learn at lockstep step t (RECALLED): (random action: num_timesteps = t < learning_starts, then after the store num_timesteps =
    t + 1 and, when t % train_freq == 0, the target update after each of the gradient steps taken -- a list of booleans, one per gradient
    step; none while t + 1 < batch_size or t + 1 < learning_starts)."""
    random_action = t < hp["learning_starts"]
    if t % hp["train_freq"] or t + 1 < hp["batch_size"] or t + 1 < hp["learning_starts"]:
        return random_action, []
    return random_action, [(t + g) % hp["target_update_interval"] == 0 for g in range(hp["gradient_steps"])]


def step_bytes(batch, W, A, sms):
    """Device bytes of one gradient step's buffers beside the ring: idx i64, q_backup / v_backup / logp f32 and d_actor f32[2A] per sample,
    and srl_sac_grad's per-CTA partial gradients (at most one CTA per SM)."""
    return int(batch) * (8 + 4 * 3 + 4 * 2 * A) + 4 * net_layout(W, A)["P"] * int(sms)


def train(env_id, num_envs, num_timesteps, seed=0, env_kwargs=None, log_dir=None, device=0, hyperparams=None, verbose=1, fused=None,
          cuda_graph=True, phase_times=None, prefetch_resets=None, episode_window=40, num_stack=1):
    """SAC.learn on a BatchedSRLVecEnv (module docstring); the signature and return value of rl_baselines.deepq.train: a history of
    (timesteps, mean episode return, fps), one entry per ``train_freq`` lockstep steps.

    The steps run in rl_baselines.offpolicy.learn's blocks of G = train_freq lockstep steps, or 2 train_freq when train_freq is odd
    (MobileRobot's state double buffer needs an even number of simulator launches per graph replay).  ``cuda_graph`` (fused, single process,
    no ``phase_times``): a block with no random action and every gradient step taken is one graph replay (the learning rate and log_ent_coef
    are read on the device).  ``phase_times``: a dict that accumulates the wall time of ``collect`` / ``prepare`` / ``gradient`` /
    ``optimise``, synchronising between them (eager)."""
    hp = dict(SAC_DEFAULTS); hp.update(hyperparams or {})
    if dict(env_kwargs or {}).get("is_discrete", True):
        raise ValueError(DISCRETE_ERROR)
    torch.manual_seed(seed)
    ctx = offpolicy.setup("sac", SACNets, env_id, num_envs, num_timesteps, seed, env_kwargs, log_dir, device, hp, verbose, fused, cuda_graph,
                          phase_times, prefetch_resets, episode_window, num_stack, step_bytes)
    env, dev, nets, dist, world, N, A, B, flat, grad, tick = ctx.env, ctx.dev, ctx.nets, ctx.dist, ctx.world, ctx.N, ctx.A, ctx.B, ctx.flat, ctx.grad, ctx.tick
    F = hp["train_freq"]
    ent_coef = None if hp["ent_coef"] == "auto" else float(hp["ent_coef"])
    target_entropy = -float(A)
    if ctx.fused:
        from srl_sim.policy import FusedSACAct, FusedSACAdam, FusedSACGrad, FusedSACPrepare
        lib = env.backend.library
        fact = FusedSACAct(lib, nets, seed=seed, env_offset=ctx.rank * N)
        workspace = FusedSACGrad.workspace(lib, nets, B)
        fprep = FusedSACPrepare(lib, nets, ctx.ring, B, seed + 1 + ctx.rank, grad, workspace)
        fgrad = FusedSACGrad(lib, nets)
        fopt = FusedSACAdam(lib, nets, ADAM_BETA1, ADAM_BETA2, ADAM_EPS, hp["tau"])
        fopt.lr.fill_(hp["learning_rate"])
        m, v, beta_power = fopt.m, fopt.v, fopt.beta_power
    else:
        m, v = torch.zeros_like(grad), torch.zeros_like(grad)
        beta_power = torch.tensor([ADAM_BETA1, ADAM_BETA2], dtype=torch.float32, device=dev)

    def act(random_action):
        if ctx.fused:
            fact(N, ctx.obs, ctx.act_dev, mode=FusedSACAct.RANDOM if random_action else FusedSACAct.SAMPLE, stream=env.backend.stream())
        else:
            ctx.act_dev.copy_(torch.rand(N, A, device=dev) * 2 - 1 if random_action else nets.act(ctx.obs))

    def gradient_step(t, polyak):
        st, t_ph = env.backend.stream(), tick()
        if ctx.fused:
            fprep(ctx.fstore.step, hp["gamma"], ent_coef, target_entropy, stream=st)
        else:
            ix = torch.randint(0, min(t + 1, ctx.rows) * N, (B,), device=dev)
            eps = torch.randn(B, A, device=dev)
            L = sac_losses(nets, flat["obs"][ix], flat["act"][ix], flat["rew"][ix], flat["next_obs"][ix], flat["done"][ix].float(), eps,
                           hp["gamma"], ent_coef, target_entropy)
        t_ph = tick("prepare", t_ph)
        if ctx.fused:
            fgrad(fprep, grad, stream=st)
        else:
            grad.copy_(torch.autograd.grad(L["total"], nets.arena)[0])
        if dist is not None:
            allreduce_mean_gradients([nets.arena], dist, world)
        t_ph = tick("gradient", t_ph)
        if ctx.fused:
            fopt(grad, polyak=polyak, stream=st)
        else:
            adam_polyak(nets, grad, m, v, beta_power, hp["learning_rate"], hp["tau"], polyak)
        tick("optimise", t_ph)

    log, stats = offpolicy.learn(ctx, F, F if F % 2 == 0 else 2 * F, lambda t: cadence(t, hp), act, gradient_step, dict(m=m, v=v, beta_power=beta_power))
    train.best_mean_reward, train.n_saved, train.stats = log.best_mean_reward, log.n_saved, stats
    train.last_nets, train.last_norm, train.last_ring, train.last_grad = nets, ctx.norm, ctx.ring, grad
    train.last_adam, train.last_before_first_step = (m, v, beta_power), ctx.before_first_step
    train.last_fused = dict(store=ctx.fstore, prepare=fprep, act=fact) if ctx.fused else None
    return log.history
