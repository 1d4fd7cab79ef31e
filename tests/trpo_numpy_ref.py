"""
Float64 numpy model of TRPO's update pieces (rl_baselines/trpo.py, include/srl_policy.h: srl_trpo_*), written from the formulas, not from
either implementation: the tanh tower forward and backward by hand, the surrogate gradient and losses of both distributions, the Fisher-vector
product in its Gauss-Newton form, baselines' CG loop, the step size, the line-search decision and MpiAdam.
"""
import numpy as np

H = 64
HALF_LOG_2PI_E = 0.5 * np.log(2 * np.pi * np.e)


def unflat(theta, D, A, box):
    """The flat pi vector (pi_w1, pi_b1, pi_w2, pi_b2, pi_w3, pi_b3, logstd) -> dict of float64 arrays."""
    shapes = [("w1", (H, D)), ("b1", (H,)), ("w2", (H, H)), ("b2", (H,)), ("w3", (A, H)), ("b3", (A,))] + ([("ls", (A,))] if box else [])
    out, o = {}, 0
    for k, s in shapes:
        n = int(np.prod(s))
        out[k] = np.asarray(theta[o:o + n], dtype=np.float64).reshape(s)
        o += n
    return out


def flat_of(grads, keys):
    return np.concatenate([grads[k].reshape(-1) for k in keys])


def forward(w, x):
    h1 = np.tanh(x @ w["w1"].T + w["b1"])
    h2 = np.tanh(h1 @ w["w2"].T + w["b2"])
    return h1, h2, h2 @ w["w3"].T + w["b3"]


def backward(w, x, h1, h2, dz):
    """The weight gradients of sum(dz * z)."""
    d2 = (dz @ w["w3"]) * (1 - h2 ** 2)
    d1 = (d2 @ w["w2"]) * (1 - h1 ** 2)
    return dict(w1=d1.T @ x, b1=d1.sum(0), w2=d2.T @ h1, b2=d2.sum(0), w3=dz.T @ h2, b3=dz.sum(0))


def jvp(w, v, x, h1, h2):
    """d z along the weight direction v (dict of the same shapes)."""
    t1 = (x @ v["w1"].T + v["b1"]) * (1 - h1 ** 2)
    t2 = (t1 @ w["w2"].T + h1 @ v["w2"].T + v["b2"]) * (1 - h2 ** 2)
    return t2 @ w["w3"].T + h2 @ v["w3"].T + v["b3"]


def softmax(z):
    e = np.exp(z - z.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def surrogate(theta, D, A, discrete, x, act, adv, entcoeff, atarg=None):
    """At theta_old: (atarg, the gradient of optimgain (flat), {surrgain, meankl, meanent}, old head outputs).  ``atarg`` given: used as the
    standardised advantages instead of standardising ``adv``."""
    box = not discrete
    w = unflat(theta, D, A, box)
    if atarg is None:
        atarg = (adv - adv.mean()) / adv.std()
    h1, h2, z = forward(w, x)
    B = x.shape[0]
    if discrete:
        p = softmax(z)
        logp = np.log(p)
        ent = -(p * logp).sum(-1)
        onehot = np.eye(A)[act]
        dz = (atarg[:, None] * (onehot - p) - entcoeff * p * (logp + ent[:, None])) / B
        gls = None
    else:
        s = np.exp(w["ls"])
        u = (act - z) / s
        dz = atarg[:, None] * u / s / B
        gls = (atarg[:, None] * (u * u - 1)).sum(0) / B + entcoeff
        ent = np.full(B, (w["ls"] + HALF_LOG_2PI_E).sum())
    g = backward(w, x, h1, h2, dz)
    keys = ["w1", "b1", "w2", "b2", "w3", "b3"]
    if box:
        g["ls"] = gls
        keys.append("ls")
    return atarg, flat_of(g, keys), dict(surrgain=atarg.mean(), meankl=0.0, meanent=ent.mean()), z


def fvp_gauss_newton(theta, D, A, discrete, x, v, damping):
    """J^T M J v / B + damping v with M the KL's Hessian in the outputs at theta_old (Categorical diag(p) - p p^T, Gaussian 1 / sigma^2 on the
    mean, 2 on logstd)."""
    box = not discrete
    w, vv = unflat(theta, D, A, box), unflat(v, D, A, box)
    h1, h2, z = forward(w, x)
    dz = jvp(w, vv, x, h1, h2)
    B = x.shape[0]
    if discrete:
        p = softmax(z)
        m = p * dz - p * (p * dz).sum(-1, keepdims=True)
    else:
        m = dz / np.exp(2 * w["ls"])
    g = backward(w, x, h1, h2, m / B)
    keys = ["w1", "b1", "w2", "b2", "w3", "b3"]
    if box:
        g["ls"] = 2 * vv["ls"]
        keys.append("ls")
    return flat_of(g, keys) + damping * np.asarray(v, dtype=np.float64)


def trial_losses(theta, D, A, discrete, x, act, atarg, old_out, old_ls, entcoeff):
    """{optimgain, meankl, meanent, surrgain} at theta against the old outputs (stable-baselines' KL and entropy)."""
    w = unflat(theta, D, A, not discrete)
    _, _, z = forward(w, x)
    if discrete:
        lp_new, lp_old = np.log(softmax(z)), np.log(softmax(old_out))
        idx = np.arange(len(act))
        ratio = np.exp(lp_new[idx, act] - lp_old[idx, act])
        kl = (np.exp(lp_old) * (lp_old - lp_new)).sum(-1)
        ent = -(np.exp(lp_new) * lp_new).sum(-1)
    else:
        ls = w["ls"]
        sn, so = np.exp(ls), np.exp(old_ls)
        lp = lambda mu, s, l: (-0.5 * ((act - mu) / s) ** 2 - l - 0.5 * np.log(2 * np.pi)).sum(-1)
        ratio = np.exp(lp(z, sn, ls) - lp(old_out, so, old_ls))
        kl = (ls - old_ls + (so ** 2 + (old_out - z) ** 2) / (2 * sn ** 2) - 0.5).sum(-1)
        ent = np.full(len(x), (ls + HALF_LOG_2PI_E).sum())
    surr = (ratio * atarg).mean()
    return dict(optimgain=surr + entcoeff * ent.mean(), meankl=kl.mean(), meanent=ent.mean(), surrgain=surr)


def cg_loop(f_Ax, b, cg_iters, residual_tol=1e-10):
    """baselines' common/cg.py, transcribed loop for loop.  Returns (x, iterations, iterates, the products' inputs)."""
    p, r, x = b.copy(), b.copy(), np.zeros_like(b)
    rdotr = r.dot(r)
    iterates, inputs = [], []
    for i in range(cg_iters):
        inputs.append(p.copy())
        z = f_Ax(p)
        v = rdotr / p.dot(z)
        x += v * p
        r -= v * z
        newrdotr = r.dot(r)
        mu = newrdotr / rdotr
        p = r + mu * p
        rdotr = newrdotr
        iterates.append(x.copy())
        if rdotr < residual_tol:
            break
    return x, len(iterates), iterates, inputs


def step_size(stepdir, fvp_stepdir, max_kl):
    shs = 0.5 * stepdir.dot(fvp_stepdir)
    lm = np.sqrt(abs(shs) / max_kl)
    return shs, lm, stepdir / lm


def decide(losses, gain_before, max_kl):
    """One line-search trial: 'nonfinite', 'kl', 'improve' (rejections) or 'accept'."""
    if not np.all(np.isfinite([losses["optimgain"], losses["meankl"], losses["meanent"]])):
        return "nonfinite"
    if losses["meankl"] > 1.5 * max_kl:
        return "kl"
    if losses["optimgain"] - gain_before < 0:
        return "improve"
    return "accept"


def mpi_adam_f32(w, g, m, v, t, lr, beta1=0.9, beta2=0.999, eps=1e-8):
    """MpiAdam.update in float32 with a float64 step size (srl_trpo_vf_adam's statement); returns (w, m, v, t + 1)."""
    f = np.float32
    t = t + 1
    a = lr * np.sqrt(1 - beta2 ** t) / (1 - beta1 ** t)
    m = f(beta1) * m + f(1 - beta1) * g
    v = f(beta2) * v + f(1 - beta2) * (g * g)
    w = w + (f(-a) * m) / (np.sqrt(v.astype(np.float64)).astype(np.float32) + f(eps))
    return w.astype(np.float32), m.astype(np.float32), v.astype(np.float32), t
