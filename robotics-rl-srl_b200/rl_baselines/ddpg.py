"""
DDPG consumer of the batched simulator: stable-baselines 2.5's ``DDPG`` with its ``MlpPolicy`` behind ``VecNormalize(norm_reward=False)``,
as the reference trains it through ``rl_baselines/rl_algorithm/ddpg.py``.  That file passes (ddpg.py:134-153) critic_l2_reg 1e-2, actor_lr
1e-4, critic_lr 1e-3, gamma 0.99, reward_scale 1, nb_rollout_steps 100, nb_train_steps 100, nb_eval_steps 50 (no eval env: no effect),
batch_size ``--batch-size``, no observation / return normalisation, no popart, clip_norm None, and the action noise of ``--noise-action``
(none, normal or Ornstein-Uhlenbeck, sigma ``--noise-action-sigma``); ``--hyperparam`` overrides them, ``noise_action`` and
``noise_action_sigma`` there taking precedence over the flags.  Restated in PyTorch next to rl_baselines/sac.py, whose batched rule and
replay-ring loop (rl_baselines/offpolicy.py) it shares.

RECALLED from stable-baselines 2.5, not checked against an installed copy (none can be installed here; include/srl_policy.h): tau 0.001;
memory_limit 100 (the ring's default rows; the reference's ``--memory-limit`` is parsed and never passed to the model); observation_range
(-5, 5), clipping every network input; the OU process (theta 0.15, dt 0.01, state from 0, reset when an episode ends); the networks
(glorot-uniform hidden kernels, zero biases, output kernels uniform(+-3e-3); the critic concatenates the action after its first layer); the
critic's L2 term over its two hidden kernels; MpiAdam and its order of float32 roundings; and the Polyak update after every gradient step.

Batched semantics (SAC's, with DDPG's cycle: :func:`cadence`).  N envs per rank step in lockstep.  A cycle is ``nb_rollout_steps`` lockstep
steps (act, step, filter, store in ring row t % buffer_size), then ``nb_train_steps`` gradient steps, each drawing ``batch_size N``
transitions uniformly, with replacement, from the min(t + 1, rows) N stored ones, and each followed by the target update.  Deviation:
``Memory.sample`` draws indices from [1, nb_entries - 1) so that every sampled entry has a following one; an N-wide ring has no such quirk to
reproduce.  Data-parallel (torchrun): every rank keeps its own ring; the gradient arena is all-reduced (mean) before Adam, which is MpiAdam's
sum / size; the observation filter is merged once per cycle.

On the GPU (``fused``) every step is the library's kernels: ``srl_ddpg_act``, ``srl_sim_step``, the filter, ``srl_sac_store``; a gradient
step is ``srl_ddpg_prepare``, ``srl_ddpg_grad``, ``srl_ddpg_adam``.  The parameters live in one flat arena (:class:`DDPGNets`), so the
gradient, the Adam slots and the all-reduce are single tensors.  The CPU path (the oracle backend of the tests, and ``fused=False``) runs the
same algorithm in torch: :func:`ddpg_losses`, :func:`mpi_adam_polyak`, :func:`ou_step` and sampling with torch's generator.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from rl_baselines import offpolicy
from rl_baselines.ppo2 import allreduce_mean_gradients

MEMORY_LIMIT = 100                         # stable-baselines 2.5 DDPG's memory_limit (RECALLED): the default ring rows
DDPG_DEFAULTS = dict(critic_l2_reg=1e-2, actor_lr=1e-4, critic_lr=1e-3, gamma=0.99, reward_scale=1.0, nb_rollout_steps=100, nb_train_steps=100,
                     nb_eval_steps=50, batch_size=64, tau=0.001, buffer_size=MEMORY_LIMIT, noise_action="ou", noise_action_sigma=0.2)
OU_THETA, OU_DT = 0.15, 1e-2               # OrnsteinUhlenbeckActionNoise's defaults (RECALLED)
OBS_RANGE = 5.0                            # observation_range (-5, 5) (RECALLED)
ADAM_BETA1, ADAM_BETA2, ADAM_EPS = 0.9, 0.999, 1e-8     # MpiAdam's defaults
NOISE_MODES = {"none": 0, "normal": 1, "ou": 2}
DISCRETE_ERROR = "ddpg does not support discrete actions, please use the '--continuous-actions' (or '-c') flag."
PARAM_NOISE_ERROR = "--noise-param: adaptive parameter noise is not supported by this DDPG (it needs a perturbed actor per episode)"
HIDDEN = 64


def net_layout(W, A):
    """Offsets of the arena (include/srl_policy.h: srl_ddpg_nets): {name: {tensor: (offset, shape)}} for actor and critic, and ``P``."""
    lay, off = {}, 0
    for name, shapes in (("actor", ((HIDDEN, W), (HIDDEN,), (HIDDEN, HIDDEN), (HIDDEN,), (A, HIDDEN), (A,))),
                         ("critic", ((HIDDEN, W), (HIDDEN,), (HIDDEN, HIDDEN + A), (HIDDEN,), (1, HIDDEN), (1,)))):
        t = {}
        for key, shape in zip(("w1", "b1", "w2", "b2", "w3", "b3"), shapes):
            t[key] = (off, shape)
            off += int(np.prod(shape))
        t["end"] = off
        lay[name] = t
    lay["P"] = off
    return lay


class DDPGNets(nn.Module):
    """The actor and the critic of the DDPG MlpPolicy in one flat float32 parameter ``arena`` (actor | critic), and the target actor and
    critic in the buffer ``target`` (the same layout, a copy at the start).  Hidden kernels glorot-uniform, output kernels uniform(+-3e-3),
    biases zero."""
    discrete = False

    def __init__(self, obs_dim, act_dim):
        super().__init__()
        self.obs_dim, self.act_dim = int(obs_dim), int(act_dim)
        self.layout = net_layout(self.obs_dim, self.act_dim)
        arena = torch.zeros(self.layout["P"])
        for name in ("actor", "critic"):
            for key in ("w1", "w2", "w3"):
                off, shape = self.layout[name][key]
                lim = 3e-3 if key == "w3" else math.sqrt(6.0 / (shape[0] + shape[1]))
                arena[off:off + int(np.prod(shape))].uniform_(-lim, lim)
        self.arena = nn.Parameter(arena)
        self.register_buffer("target", arena.clone())

    def tensors(self, name, source=None):
        """The six tensors of network ``name`` as views of ``source`` (default: the arena)."""
        src = self.arena if source is None else source
        return [src[off:off + int(np.prod(shape))].view(shape) for off, shape in (self.layout[name][k] for k in ("w1", "b1", "w2", "b2", "w3", "b3"))]

    def actor(self, obs, source=None):
        w1, b1, w2, b2, w3, b3 = self.tensors("actor", source)
        h = torch.relu(torch.clamp(obs, -OBS_RANGE, OBS_RANGE) @ w1.t() + b1)
        h = torch.relu(h @ w2.t() + b2)
        return torch.tanh(h @ w3.t() + b3)

    def critic(self, obs, act, source=None):
        w1, b1, w2, b2, w3, b3 = self.tensors("critic", source)
        h = torch.relu(torch.clamp(obs, -OBS_RANGE, OBS_RANGE) @ w1.t() + b1)
        h = torch.relu(torch.cat([h, act], -1) @ w2.t() + b2)
        return (h @ w3.t() + b3).squeeze(-1)

    def sync_target(self):
        with torch.no_grad():
            self.target.copy_(self.arena)

    def act(self, obs):
        """The noise-free action (DDPG.predict)."""
        return self.actor(obs)


def ddpg_losses(nets, obs, act, rew, next_obs, done, gamma, reward_scale, critic_l2_reg):
    """One step's losses from the parameters as they are (DDPG._setup_actor_optimizer / _setup_critic_optimizer).  Returns a dict with
    ``total``, whose gradient with respect to the arena is each optimiser's gradient on its own network: actor_loss on the actor (the critic
    frozen), critic_loss on the critic; and y, the losses."""
    with torch.no_grad():
        q_next = nets.critic(next_obs, nets.actor(next_obs, nets.target), nets.target)
        y = rew * reward_scale + (1 - done) * gamma * q_next
    actor_loss = -nets.critic(obs, nets.actor(obs), nets.arena.detach()).mean()
    w1, _, w2, _, _, _ = nets.tensors("critic")
    critic_loss = ((nets.critic(obs, act) - y) ** 2).mean() + critic_l2_reg * ((w1 ** 2).sum() + (w2 ** 2).sum()) / 2
    return dict(total=actor_loss + critic_loss, y=y, actor_loss=actor_loss, critic_loss=critic_loss)


def mpi_adam_polyak(nets, grad, m, v, t, actor_lr, critic_lr, tau, beta1=ADAM_BETA1, beta2=ADAM_BETA2, eps=ADAM_EPS):
    """MpiAdam over the arena with the actor's and the critic's learning rate (the torch statement of srl_ddpg_adam, in its order of float32
    roundings), then ``target = (1 - tau) target + tau arena``; ``t`` (int64 [1]) counts the steps and is advanced."""
    with torch.no_grad():
        dev = nets.arena.device
        f32 = lambda x: torch.tensor(x, dtype=torch.float32, device=dev)
        step = int(t[0]) + 1
        a = lambda lr: lr * math.sqrt(1 - beta2 ** step) / (1 - beta1 ** step)          # float64, MpiAdam's order
        end = nets.layout["actor"]["end"]
        neg_a = torch.empty_like(nets.arena)
        neg_a[:end], neg_a[end:] = f32(-a(actor_lr)), f32(-a(critic_lr))
        m.copy_(f32(beta1) * m + f32(1 - beta1) * grad)
        v.copy_(f32(beta2) * v + f32(1 - beta2) * (grad * grad))
        sqrt_v = torch.sqrt(v.double()).float()             # the correctly rounded float32 root (numpy's, the kernel's); torch's CPU float one is not
        nets.arena.add_((neg_a * m) / (sqrt_v + f32(eps)))
        nets.target.copy_(f32(1 - tau) * nets.target + f32(tau) * nets.arena)
        t.add_(1)


def ou_step(state, z, prev_done, sigma, theta=OU_THETA, dt=OU_DT):
    """OrnsteinUhlenbeckActionNoise.__call__ per env, after its reset for every env whose previous step ended an episode (float32, in place):
    x = x + (theta (0 - x)) dt + (sigma sqrt(dt)) z.  Returns the new state."""
    f32 = lambda x: torch.tensor(x, dtype=torch.float32, device=state.device)
    state.masked_fill_(prev_done.bool()[:, None], 0.0)
    state.copy_((state + (f32(theta) * -state) * f32(dt)) + (f32(sigma) * torch.sqrt(f32(dt))) * z)
    return state


def cadence(t, hp):
    """The gradient steps after lockstep step t (from 0): ``nb_train_steps`` once every ``nb_rollout_steps`` steps, at the end of a cycle's
    rollout; none after a rollout cut short by the end of training."""
    return hp["nb_train_steps"] if (t + 1) % hp["nb_rollout_steps"] == 0 else 0


def step_bytes(batch, W, A, sms):
    """Device bytes of one gradient step's buffers beside the ring: idx i64, y f32, mu and d_actor f32[A] per sample, and srl_ddpg_grad's
    per-CTA partial gradients (at most one CTA per SM)."""
    return int(batch) * (8 + 4 + 2 * 4 * A) + 4 * net_layout(W, A)["P"] * int(sms)


def train(env_id, num_envs, num_timesteps, seed=0, env_kwargs=None, log_dir=None, device=0, hyperparams=None, verbose=1, fused=None,
          cuda_graph=True, phase_times=None, prefetch_resets=None, episode_window=40, num_stack=1, noise_param=False):
    """DDPG.learn on a BatchedSRLVecEnv (module docstring); the signature and return value of rl_baselines.sac.train: a history of
    (timesteps, mean episode return, fps), one entry per cycle of ``nb_rollout_steps`` lockstep steps.

    The steps run in rl_baselines.offpolicy.learn's blocks of G = nb_rollout_steps lockstep steps, or 2 nb_rollout_steps when that is odd
    and the blocks are captured (MobileRobot's state double buffer needs an even number of simulator launches per graph replay).
    ``cuda_graph`` (fused, single process, no ``phase_times``): every full block after the first is one graph replay (the OU state, the step
    count and the learning rates are read on the device).  ``phase_times``: a dict that accumulates the wall time of ``collect`` /
    ``prepare`` / ``gradient`` / ``optimise``, synchronising between them (eager)."""
    hp = dict(DDPG_DEFAULTS); hp.update(hyperparams or {})
    if dict(env_kwargs or {}).get("is_discrete", True):
        raise ValueError(DISCRETE_ERROR)
    if noise_param:
        raise ValueError(PARAM_NOISE_ERROR)
    if hp["noise_action"] not in NOISE_MODES:
        raise ValueError("noise_action must be one of %s (got %r)" % (sorted(NOISE_MODES), hp["noise_action"]))
    mode, sigma = NOISE_MODES[hp["noise_action"]], float(hp["noise_action_sigma"])
    torch.manual_seed(seed)
    ctx = offpolicy.setup("ddpg", DDPGNets, env_id, num_envs, num_timesteps, seed, env_kwargs, log_dir, device, hp, verbose, fused, cuda_graph,
                          phase_times, prefetch_resets, episode_window, num_stack, step_bytes)
    env, dev, nets, dist, world, N, A, B, flat, grad, tick = ctx.env, ctx.dev, ctx.nets, ctx.dist, ctx.world, ctx.N, ctx.A, ctx.B, ctx.flat, ctx.grad, ctx.tick
    R = hp["nb_rollout_steps"]
    if ctx.fused:
        from srl_sim.policy import FusedDDPGAct, FusedDDPGAdam, FusedDDPGGrad, FusedDDPGPrepare
        lib = env.backend.library
        fact = FusedDDPGAct(lib, nets, N, seed=seed, sigma=sigma, theta=OU_THETA, dt=OU_DT, env_offset=ctx.rank * N)
        fprep = FusedDDPGPrepare(lib, nets, ctx.ring, B, seed + 1 + ctx.rank)
        fgrad = FusedDDPGGrad(lib, nets, B, hp["critic_l2_reg"])
        fopt = FusedDDPGAdam(lib, nets, hp["actor_lr"], hp["critic_lr"], hp["tau"], ADAM_BETA1, ADAM_BETA2, ADAM_EPS)
        m, v, t_adam, ou = fopt.m, fopt.v, fopt.t, fact.ou
    else:
        m, v, t_adam, ou = torch.zeros_like(grad), torch.zeros_like(grad), torch.zeros(1, dtype=torch.int64), torch.zeros(N, A, device=dev)

    def act(random_action):
        if ctx.fused:
            fact(N, ctx.obs, ctx.done_s, ctx.act_dev, mode=mode, stream=env.backend.stream())
            return
        a = nets.act(ctx.obs)
        if mode == NOISE_MODES["normal"]:
            a = a + sigma * torch.randn(N, A, device=dev)
        elif mode == NOISE_MODES["ou"]:
            a = a + ou_step(ou, torch.randn(N, A, device=dev), ctx.done_s, sigma)        # ctx.done_s: the previous step's done flags
        ctx.act_dev.copy_(torch.clamp(a, -1.0, 1.0))

    def gradient_step(t, polyak):                          # polyak is always True: the target update follows every gradient step
        st, t_ph = env.backend.stream(), tick()
        if ctx.fused:
            fprep(ctx.fstore.step, hp["gamma"], hp["reward_scale"], stream=st)
        else:
            ix = torch.randint(0, min(t + 1, ctx.rows) * N, (B,), device=dev)
            L = ddpg_losses(nets, flat["obs"][ix], flat["act"][ix], flat["rew"][ix], flat["next_obs"][ix], flat["done"][ix].float(), hp["gamma"],
                            hp["reward_scale"], hp["critic_l2_reg"])
        t_ph = tick("prepare", t_ph)
        if ctx.fused:
            fgrad(fprep, grad, stream=st)
        else:
            grad.copy_(torch.autograd.grad(L["total"], nets.arena)[0])
        if dist is not None:
            allreduce_mean_gradients([nets.arena], dist, world)
        t_ph = tick("gradient", t_ph)
        if ctx.fused:
            fopt(grad, stream=st)
        else:
            mpi_adam_polyak(nets, grad, m, v, t_adam, hp["actor_lr"], hp["critic_lr"], hp["tau"])
        tick("optimise", t_ph)

    # Every block starts at a multiple of R, so a full block has its gradient steps at its steps R - 1 (and 2 R - 1) and no random action:
    # every full block after the first gradient step is the captured one (tests/test_ddpg_cpu.py::test_cadence).
    log, stats = offpolicy.learn(ctx, R, 2 * R if R % 2 and ctx.use_graph else R, lambda t: (False, [True] * cadence(t, hp)), act, gradient_step,
                                 dict(m=m, v=v, t=t_adam))
    train.best_mean_reward, train.n_saved, train.stats = log.best_mean_reward, log.n_saved, stats
    train.last_nets, train.last_norm, train.last_ring, train.last_grad = nets, ctx.norm, ctx.ring, grad
    train.last_adam, train.last_ou, train.last_before_first_step = (m, v, t_adam), ou, ctx.before_first_step
    train.last_fused = dict(store=ctx.fstore, prepare=fprep, act=fact) if ctx.fused else None
    return log.history
