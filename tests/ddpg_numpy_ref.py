"""
Float64 numpy models of the DDPG trainer (rl_baselines/ddpg.py, include/srl_policy.h: srl_ddpg_*), written from the definitions rather than
from the trainer: the arena layout, the actor and the critic (the action concatenated after the critic's first layer, every input clipped to
[-5, 5]) with a hand-written backward pass, the gradient of one step (critic MSE + L2 on the two hidden critic kernels, actor -mean Q), the
Ornstein-Uhlenbeck step, and a float32 transcription of MpiAdam + the Polyak update.
"""
import math

import numpy as np

H = 64
OBS_RANGE = 5.0


def layout(W, A):
    """{net: {tensor: (offset, shape)}} for actor and critic, and P."""
    lay, off = {}, 0
    for name, shapes in (("actor", ((H, W), (H,), (H, H), (H,), (A, H), (A,))), ("critic", ((H, W), (H,), (H, H + A), (H,), (1, H), (1,)))):
        t = {}
        for key, shape in zip(("w1", "b1", "w2", "b2", "w3", "b3"), shapes):
            t[key] = (off, shape)
            off += int(np.prod(shape))
        t["end"] = off
        lay[name] = t
    return lay, off


def unpack(arena, W, A, name):
    lay, _ = layout(W, A)
    f = np.asarray(arena, np.float64)
    return {k: f[o:o + int(np.prod(s))].reshape(s) for k, (o, s) in ((k, lay[name][k]) for k in ("w1", "b1", "w2", "b2", "w3", "b3"))}


def actor_fwd(p, x):
    """(tanh head, its pre-activation, cache)."""
    xc = np.clip(x, -OBS_RANGE, OBS_RANGE)
    z1 = xc @ p["w1"].T + p["b1"]
    h1 = np.maximum(z1, 0.0)
    z2 = h1 @ p["w2"].T + p["b2"]
    h2 = np.maximum(z2, 0.0)
    out = h2 @ p["w3"].T + p["b3"]
    return np.tanh(out), out, (xc, z1, h1, z2, h2)


def actor_bwd(p, cache, g_out):
    """Flat gradients (layout order) of sum(g_out * pre-tanh head)."""
    xc, z1, h1, z2, h2 = cache
    g = {"w3": g_out.T @ h2, "b3": g_out.sum(0)}
    d2 = (g_out @ p["w3"]) * (z2 > 0)
    g["w2"], g["b2"] = d2.T @ h1, d2.sum(0)
    d1 = (d2 @ p["w2"]) * (z1 > 0)
    g["w1"], g["b1"] = d1.T @ xc, d1.sum(0)
    return np.concatenate([g[k].reshape(-1) for k in ("w1", "b1", "w2", "b2", "w3", "b3")])


def critic_fwd(p, x, a):
    xc = np.clip(x, -OBS_RANGE, OBS_RANGE)
    z1 = xc @ p["w1"].T + p["b1"]
    h1 = np.maximum(z1, 0.0)
    c = np.concatenate([h1, a], 1)
    z2 = c @ p["w2"].T + p["b2"]
    h2 = np.maximum(z2, 0.0)
    return (h2 @ p["w3"].T + p["b3"])[:, 0], (xc, z1, c, z2, h2)


def critic_bwd(p, cache, gq):
    """(flat gradients of sum(gq * Q) in layout order, dQ/da weighted by gq)."""
    xc, z1, c, z2, h2 = cache
    g = {"w3": gq[None, :] @ h2, "b3": np.array([gq.sum()])}
    d2 = (gq[:, None] * p["w3"]) * (z2 > 0)
    g["w2"], g["b2"] = d2.T @ c, d2.sum(0)
    dc = d2 @ p["w2"]
    d1 = dc[:, :H] * (z1 > 0)
    g["w1"], g["b1"] = d1.T @ xc, d1.sum(0)
    return np.concatenate([g[k].reshape(-1) for k in ("w1", "b1", "w2", "b2", "w3", "b3")]), dc[:, H:]


def ddpg_step_model(arena, target, W, A, obs, act, rew, next_obs, done, gamma, reward_scale, critic_l2_reg):
    """One gradient step's gradient arena (float64) and its per-sample values: y, mu and d_actor (d actor_loss / d the actor's pre-tanh head)."""
    lay, P = layout(W, A)
    obs, act, next_obs = (np.asarray(x, np.float64) for x in (obs, act, next_obs))
    rew, done = np.asarray(rew, np.float64), np.asarray(done, np.float64)
    B = obs.shape[0]
    pa, pc = unpack(arena, W, A, "actor"), unpack(arena, W, A, "critic")
    ta, tc = unpack(target, W, A, "actor"), unpack(target, W, A, "critic")
    a_next, _, _ = actor_fwd(ta, next_obs)
    q_next, _ = critic_fwd(tc, next_obs, a_next)
    y = rew * reward_scale + (1.0 - done) * gamma * q_next
    # actor_loss = -mean(Q(s, mu(s))), the critic frozen
    mu, _, c_actor = actor_fwd(pa, obs)
    _, c_pi = critic_fwd(pc, obs, mu)
    _, dq_da = critic_bwd(pc, c_pi, np.ones(B))
    d_actor = -dq_da * (1.0 - mu ** 2) / B
    grad = np.zeros(P)
    grad[:lay["actor"]["end"]] = actor_bwd(pa, c_actor, d_actor)
    # critic_loss = mean((Q(s, a) - y)^2) + critic_l2_reg (|w1|^2 + |w2|^2) / 2
    q, cache = critic_fwd(pc, obs, act)
    g, _ = critic_bwd(pc, cache, 2.0 * (q - y) / B)
    lo = lay["actor"]["end"]
    grad[lo:] = g
    w = np.asarray(arena, np.float64)
    for key in ("w1", "w2"):
        off, shape = lay["critic"][key]
        n = int(np.prod(shape))
        grad[off:off + n] += critic_l2_reg * w[off:off + n]
    return grad, dict(y=y, mu=mu, d_actor=d_actor)


def ou_model(state, z, prev_done, sigma, theta=0.15, dt=1e-2):
    """OrnsteinUhlenbeckActionNoise in float64 after a reset of every env whose previous step ended an episode: the new state."""
    x = np.where(np.asarray(prev_done, bool)[:, None], 0.0, np.asarray(state, np.float64))
    return x + theta * (0.0 - x) * dt + sigma * math.sqrt(dt) * np.asarray(z, np.float64)


def mpi_adam_polyak_f32(arena, target, grads, actor_end, actor_lr, critic_lr, tau, beta1=0.9, beta2=0.999, eps=1e-8, m=None, v=None, steps=0):
    """MpiAdam.update (a in float64, then every array operation in float32, python floats rounded to float32 as numpy 1.x does) for each
    gradient, each step followed by the Polyak update of the targets.  The slots ``m``, ``v`` (default 0) are those left by ``steps``
    earlier updates, so the first update here has MpiAdam's t = steps + 1.  Returns (arena, target, m, v)."""
    f32 = np.float32
    w, tg = np.array(arena, f32), np.array(target, f32)
    m = np.zeros_like(w) if m is None else np.array(m, f32)
    v = np.zeros_like(w) if v is None else np.array(v, f32)
    for t, g in enumerate(grads, int(steps) + 1):
        g = np.asarray(g, f32)
        neg_a = np.empty_like(w)
        for lo, hi, lr in ((0, actor_end, actor_lr), (actor_end, w.size, critic_lr)):
            neg_a[lo:hi] = f32(-(lr * math.sqrt(1 - beta2 ** t) / (1 - beta1 ** t)))
        m = f32(beta1) * m + f32(1 - beta1) * g
        v = f32(beta2) * v + f32(1 - beta2) * (g * g)
        w = w + (neg_a * m) / (np.sqrt(v) + f32(eps))
        tg = f32(1 - tau) * tg + f32(tau) * w
    return w, tg, m, v
