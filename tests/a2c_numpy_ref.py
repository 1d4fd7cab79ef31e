"""
float64 numpy statements of one stable-baselines 2.5 A2C update, written from the formulas (include/srl_policy.h: srl_a2c_grad,
srl_clip_rmsprop) and not from rl_baselines/a2c.py, for the CPU and GPU tests of the A2C path:
  a2c_grads_model     : the gradient of the A2C loss of an MlpPolicy, forward and backward by hand
  clip_rmsprop_model  : tf.clip_by_global_norm followed by TF1's RMSProp (momentum 0) on a list of arrays
  discount_with_dones : stable-baselines' return recursion, bootstrapped from the last value where the rollout did not end
  scheduler_values    : stable-baselines' Scheduler stepped once per sample, the value A2C._train_step trains each update with
"""
import numpy as np
import torch


def _layers(seq):
    return [(m.weight.detach().cpu().double().numpy(), m.bias.detach().cpu().double().numpy()) for m in seq if isinstance(m, torch.nn.Linear)]


def a2c_grads_model(pol, obs, act, ret, old_val, ent_coef, vf_coef):
    """Gradients, in the order of pol.parameters(), of mean(-(ret - old_val) logp) - ent_coef mean(entropy) + vf_coef 0.5 mean((v - ret)^2)."""
    x = np.asarray(obs, np.float64)
    ret, old_val = np.asarray(ret, np.float64), np.asarray(old_val, np.float64)
    B = x.shape[0]
    adv = ret - old_val

    def forward(layers):
        hs = [x]
        for k, (w, b) in enumerate(layers):
            h = hs[-1] @ w.T + b
            hs.append(np.tanh(h) if k < len(layers) - 1 else h)
        return hs

    def backward(layers, hs, dout):
        grads = []
        d = dout
        for k in reversed(range(len(layers))):
            w, _ = layers[k]
            grads = [d.T @ hs[k], d.sum(0)] + grads
            if k:
                d = (d @ w) * (1.0 - hs[k] ** 2)
        return grads

    pi, vf = _layers(pol.pi), _layers(pol.vf)
    hp, hv = forward(pi), forward(vf)
    out, v = hp[-1], hv[-1][:, 0]
    extra = []
    if pol.discrete:
        a = np.asarray(act, np.int64)
        m = out.max(1, keepdims=True)
        lse = m + np.log(np.exp(out - m).sum(1, keepdims=True))
        logp_all = out - lse
        p = np.exp(logp_all)
        ent = -(p * logp_all).sum(1, keepdims=True)
        onehot = np.eye(out.shape[1])[a]
        dout = -(adv[:, None] / B) * (onehot - p) + (ent_coef / B) * p * (logp_all + ent)
    else:
        ls = pol.logstd.detach().cpu().double().numpy()
        u = (np.asarray(act, np.float64) - out) / np.exp(ls)
        dout = -(adv[:, None] / B) * u / np.exp(ls)
        extra = [(-(adv[:, None] / B) * (u * u - 1.0)).sum(0) - ent_coef]
    dv = (vf_coef / B) * (v - ret)
    return extra + backward(pi, hp, dout) + backward(vf, hv, dv[:, None])      # pol.parameters(): logstd (Box) comes first


def clip_rmsprop_model(params, grads, ms, lr, max_grad_norm, alpha, epsilon):
    """One step in float64 on copies: returns (params, ms)."""
    norm = np.sqrt(sum(float((np.asarray(g, np.float64) ** 2).sum()) for g in grads))
    scale = max_grad_norm / max(norm, max_grad_norm)
    new_p, new_ms = [], []
    for p, g, m in zip(params, grads, ms):
        g = np.asarray(g, np.float64) * scale
        m = alpha * np.asarray(m, np.float64) + (1.0 - alpha) * g * g
        new_ms.append(m)
        new_p.append(np.asarray(p, np.float64) - lr * g / np.sqrt(m + epsilon))
    return new_p, new_ms


def discount_with_dones(rewards, dones, gamma):
    r, out = 0.0, []
    for reward, done in zip(rewards[::-1], dones[::-1]):
        r = reward + gamma * r * (1.0 - done)
        out.append(r)
    return out[::-1]


def a2c_returns_model(rew, done, last_val, gamma):
    """[T, N] returns of the A2C runner: per env, discount_with_dones(rewards + [last value], dones + [0])[:-1] when the last step did not end
    an episode, discount_with_dones(rewards, dones) when it did (``done[t]``: the episode ended at step t)."""
    rew, done, last_val = (np.asarray(a, np.float64) for a in (rew, done, last_val))
    T, N = rew.shape
    out = np.zeros((T, N))
    for n in range(N):
        r, d = list(rew[:, n]), list(done[:, n])
        out[:, n] = discount_with_dones(r + [last_val[n]], d + [0.0], gamma)[:-1] if d[-1] == 0 else discount_with_dones(r, d, gamma)
    return out


SCHEDULE_FNS = {
    "constant": lambda p: 1.0,
    "linear": lambda p: 1.0 - p,
    "middle_drop": lambda p: 0.075 if 1.0 - p < 0.75 else 1.0 - p,
    "double_linear_con": lambda p: 0.125 if 1.0 - 2.0 * p < 0.125 else 1.0 - 2.0 * p,
    "double_middle_drop": lambda p: (0.125 if 1.0 - p < 0.25 else 0.075) if 1.0 - p < 0.75 else 1.0 - p,
}


def scheduler_values(initial, total_timesteps, schedule, n_batch, n_updates):
    """The learning rate of each update: Scheduler.value() called once per sample of the update, the last value kept."""
    step, lrs = 0, []
    for _ in range(n_updates):
        for _ in range(n_batch):
            cur = initial * SCHEDULE_FNS[schedule](step / total_timesteps)
            step += 1
        lrs.append(cur)
    return lrs
