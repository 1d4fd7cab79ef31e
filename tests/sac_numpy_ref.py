"""
Float64 numpy models of the SAC trainer (rl_baselines/sac.py, include/srl_policy.h: srl_sac_*), written from the definitions rather than from
the trainer: the arena layout, the five ReLU networks with a hand-written backward pass, the losses of one gradient step by the chain rule
through u = mu + std eps (not the simplified form the kernel uses), and TF1 Adam + the Polyak update.
"""
import math

import numpy as np

H = 64
LOG_STD_MIN, LOG_STD_MAX, DELTA = -20.0, 2.0, 1e-6


def layout(W, A):
    """{net: (offset, in, out)} and P: actor (W -> 2A), qf1, qf2 (W + A -> 1), vf (W -> 1), then log_ent_coef."""
    nets, off = {}, 0
    for name, n_in, n_out in (("actor", W, 2 * A), ("qf1", W + A, 1), ("qf2", W + A, 1), ("vf", W, 1)):
        nets[name] = (off, n_in, n_out)
        off += H * n_in + H + H * H + H + n_out * H + n_out
    return nets, off + 1


def unpack(flat, off, n_in, n_out):
    f = np.asarray(flat, np.float64)
    sizes = [("w1", (H, n_in)), ("b1", (H,)), ("w2", (H, H)), ("b2", (H,)), ("w3", (n_out, H)), ("b3", (n_out,))]
    out, o = {}, off
    for k, shape in sizes:
        n = int(np.prod(shape))
        out[k] = f[o:o + n].reshape(shape)
        o += n
    return out


def forward(p, x):
    z1 = x @ p["w1"].T + p["b1"]
    h1 = np.maximum(z1, 0.0)
    z2 = h1 @ p["w2"].T + p["b2"]
    h2 = np.maximum(z2, 0.0)
    return h2 @ p["w3"].T + p["b3"], (x, z1, h1, z2, h2)


def backward(p, cache, gout):
    """Gradients of sum(gout * out) for the six tensors (flat, in layout order) and the input; ReLU passes where the pre-activation is > 0."""
    x, z1, h1, z2, h2 = cache
    g = {"w3": gout.T @ h2, "b3": gout.sum(0)}
    d2 = (gout @ p["w3"]) * (z2 > 0)
    g["w2"], g["b2"] = d2.T @ h1, d2.sum(0)
    d1 = (d2 @ p["w2"]) * (z1 > 0)
    g["w1"], g["b1"] = d1.T @ x, d1.sum(0)
    return np.concatenate([g[k].reshape(-1) for k in ("w1", "b1", "w2", "b2", "w3", "b3")]), d1 @ p["w1"]


def sac_step_model(arena, target, W, A, obs, act, rew, next_obs, done, eps, gamma, ent_coef, target_entropy):
    """One gradient step's gradient arena (float64) and its per-sample values: q_backup, v_backup, logp and d_actor (d policy_loss /
    d (mu, raw log_std), [B, 2A]).  ``ent_coef`` None: 'auto', alpha = exp(log_ent_coef)."""
    nets, P = layout(W, A)
    arena = np.asarray(arena, np.float64)
    B = obs.shape[0]
    obs, act, next_obs, eps = (np.asarray(x, np.float64) for x in (obs, act, next_obs, eps))
    rew, done = np.asarray(rew, np.float64), np.asarray(done, np.float64)
    alpha = math.exp(arena[P - 1]) if ent_coef is None else float(ent_coef)
    pr = {k: unpack(arena, *nets[k]) for k in nets}
    vt, _ = forward(unpack(target, 0, W, 1), next_obs)
    q_backup = rew + gamma * (1.0 - done) * vt[:, 0]
    out, c_actor = forward(pr["actor"], obs)
    mu, lsr = out[:, :A], out[:, A:]
    ls = np.clip(lsr, LOG_STD_MIN, LOG_STD_MAX)
    std = np.exp(ls)
    u = mu + std * eps
    z = (u - mu) / (std + DELTA)
    a = np.tanh(u)
    logp = (-0.5 * (z ** 2 + 2 * ls + math.log(2 * math.pi))).sum(1) - np.log(1 - a ** 2 + DELTA).sum(1)
    x_pi = np.concatenate([obs, a], 1)
    q1_pi, c_q1 = forward(pr["qf1"], x_pi)
    q2_pi, _ = forward(pr["qf2"], x_pi)
    v_backup = np.minimum(q1_pi[:, 0], q2_pi[:, 0]) - alpha * logp
    _, dx = backward(pr["qf1"], c_q1, np.ones((B, 1)))
    dq_da = dx[:, W:]
    # policy_loss = mean(alpha logp - qf1(s, a_pi)), chain rule through u = mu + std eps
    T = 2 * a * (1 - a ** 2) / (1 - a ** 2 + DELTA)
    dL_du = alpha * (-z / (std + DELTA) + T) - dq_da * (1 - a ** 2)
    dL_dmu = dL_du + alpha * z / (std + DELTA)
    dL_dls = dL_du * std * eps + alpha * (z * (u - mu) * std / (std + DELTA) ** 2 - 1.0)
    dL_dls = dL_dls * ((lsr >= LOG_STD_MIN) & (lsr <= LOG_STD_MAX))
    d_actor = np.concatenate([dL_dmu, dL_dls], 1) / B
    grad = np.zeros(P)
    off, n_in, n_out = nets["actor"]
    g, _ = backward(pr["actor"], c_actor, d_actor)
    grad[off:off + g.size] = g
    x = np.concatenate([obs, act], 1)
    for name, inp, tgt in (("qf1", x, q_backup), ("qf2", x, q_backup), ("vf", obs, v_backup)):
        o, cache = forward(pr[name], inp)
        g, _ = backward(pr[name], cache, (o - tgt[:, None]) / B)
        grad[nets[name][0]:nets[name][0] + g.size] = g
    grad[P - 1] = -np.mean(logp + target_entropy) if ent_coef is None else 0.0
    return grad, dict(q_backup=q_backup, v_backup=v_backup, logp=logp, d_actor=d_actor)


def adam_polyak_model(arena, target, grads, W, A, lr, tau, beta1=0.9, beta2=0.999, eps=1e-8):
    """TF1 Adam (slots from 0, t from 1) over the arena for each gradient in ``grads``, each step followed by target = (1 - tau) target +
    tau vf.  Float64; returns (arena, target, m, v)."""
    nets, P = layout(W, A)
    w, tg = np.array(arena, np.float64), np.array(target, np.float64)
    m, v = np.zeros(P), np.zeros(P)
    lo = nets["vf"][0]
    for t, g in enumerate(grads, 1):
        g = np.asarray(g, np.float64)
        lr_t = lr * math.sqrt(1 - beta2 ** t) / (1 - beta1 ** t)
        m = beta1 * m + (1 - beta1) * g
        v = beta2 * v + (1 - beta2) * g * g
        w = w - lr_t * m / (np.sqrt(v) + eps)
        tg = (1 - tau) * tg + tau * w[lo:lo + tg.size]
    return w, tg, m, v
