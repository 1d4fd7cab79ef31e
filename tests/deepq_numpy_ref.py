"""
float64 / loop-form statements of one stable-baselines 2.5 DQN step, written from the formulas (include/srl_policy.h: srl_dqn_*, srl_replay_*,
srl_clip_adam) and not from rl_baselines/deepq.py, for the CPU and GPU tests of the DQN path:
  dqn_forward_model   : Q of a dueling network, forward by hand
  dqn_grads_model     : the gradient of mean(w huber(Q(s, a) - y)), backward by hand (ReLU: 0 where the pre-activation is <= 0)
  double_q_model      : y = r + gamma (1 - d) Q_target(s', argmax Q_online(s'))
  clip_adam_model     : tf.clip_by_norm per tensor followed by TF1 Adam, on lists of arrays
  SegmentTree / PrioritizedReplay : a direct transcription of baselines' SegmentTree (loop form) and of the prioritized buffer's bookkeeping
  first_sample_model  : the indices of a replay's first batch, while every stored leaf is still 1^alpha (uniform or prioritized)
  tree_sample_model   : the indices and importance weights of a batch drawn from any sum / min trees (find_prefixsum_idx, vectorised)
  dqn_step_model      : one gradient step (double Q with its own online and target networks, gradient, clip, Adam from given slots)
"""
import operator

import numpy as np
import torch


def _layers(seq):
    return [(m.weight.detach().cpu().double().numpy(), m.bias.detach().cpu().double().numpy()) for m in seq if isinstance(m, torch.nn.Linear)]


def _forward(layers, x):
    hs, pre = [x], []
    for k, (w, b) in enumerate(layers):
        h = hs[-1] @ w.T + b
        pre.append(h)
        hs.append(np.maximum(h, 0.0) if k < len(layers) - 1 else h)
    return hs, pre


def dqn_forward_model(qnet, obs):
    x = np.asarray(obs, np.float64)
    a = _forward(_layers(qnet.pi), x)[0][-1]
    v = _forward(_layers(qnet.vf), x)[0][-1]
    return v + a - a.mean(1, keepdims=True)


def dqn_grads_model(qnet, obs, act, y, w):
    """Gradients in the order of qnet.parameters() and the per-sample td."""
    x = np.asarray(obs, np.float64)
    act, y, w = np.asarray(act, np.int64), np.asarray(y, np.float64), np.asarray(w, np.float64)
    B = x.shape[0]
    pi, vf = _layers(qnet.pi), _layers(qnet.vf)
    hp, pp = _forward(pi, x)
    hv, pv = _forward(vf, x)
    a, v = hp[-1], hv[-1][:, 0]
    n = a.shape[1]
    q = v[:, None] + a - a.mean(1, keepdims=True)
    td = q[np.arange(B), act] - y
    gq = w * np.where(np.abs(td) < 1.0, td, np.sign(td)) / B          # d mean(w huber(td)) / d Q(s, a)
    da = gq[:, None] * (np.eye(n)[act] - 1.0 / n)

    def backward(layers, hs, pre, d):
        grads = []
        for k in reversed(range(len(layers))):
            wk, _ = layers[k]
            grads = [d.T @ hs[k], d.sum(0)] + grads
            if k:
                d = (d @ wk) * (pre[k - 1] > 0.0)
        return grads
    return backward(pi, hp, pp, da) + backward(vf, hv, pv, gq[:, None]), td


def double_q_model(online, target, rew, done, next_obs, gamma):
    qo, qt = dqn_forward_model(online, next_obs), dqn_forward_model(target, next_obs)
    best = qo.argmax(1)
    return np.asarray(rew, np.float64) + gamma * (1.0 - np.asarray(done, np.float64)) * qt[np.arange(len(best)), best], qo


def clip_adam_model(params, grads, m, v, step, lr, clip_norm, beta1, beta2, eps):
    """One step (1-based ``step``) in float64 on copies: returns (params, m, v)."""
    lr_t = lr * np.sqrt(1.0 - beta2 ** step) / (1.0 - beta1 ** step)
    out = ([], [], [])
    for p, g, mm, vv in zip(params, grads, m, v):
        g = np.asarray(g, np.float64)
        g = g * clip_norm / max(np.sqrt((g * g).sum()), clip_norm)
        mm = beta1 * mm + (1.0 - beta1) * g
        vv = beta2 * vv + (1.0 - beta2) * g * g
        out[0].append(p - lr_t * mm / (np.sqrt(vv) + eps)); out[1].append(mm); out[2].append(vv)
    return out


class SegmentTree(object):
    """baselines.common.segment_tree.SegmentTree, transcribed loop for loop."""

    def __init__(self, capacity, operation, neutral_element):
        assert capacity > 0 and capacity & (capacity - 1) == 0
        self._capacity = capacity
        self._value = [neutral_element for _ in range(2 * capacity)]
        self._operation = operation

    def __setitem__(self, idx, val):
        idx += self._capacity
        self._value[idx] = val
        idx //= 2
        while idx >= 1:
            self._value[idx] = self._operation(self._value[2 * idx], self._value[2 * idx + 1])
            idx //= 2

    def __getitem__(self, idx):
        return self._value[self._capacity + idx]

    def find_prefixsum_idx(self, prefixsum):
        idx = 1
        while idx < self._capacity:
            if self._value[2 * idx] > prefixsum:
                idx = 2 * idx
            else:
                prefixsum -= self._value[2 * idx]
                idx = 2 * idx + 1
        return idx - self._capacity


class PrioritizedReplay(object):
    """The bookkeeping of baselines' PrioritizedReplayBuffer over a ring of rows x n_envs transitions, with the statement of
    include/srl_policy.h for the float32 priority and the clamp of a walk into an empty leaf."""

    def __init__(self, rows, n_envs, alpha):
        self.n_envs, self.capacity, self.alpha = n_envs, rows * n_envs, alpha
        cap = 1
        while cap < self.capacity:
            cap *= 2
        self.tree_cap = cap
        self.it_sum = SegmentTree(cap, operator.add, 0.0)
        self.it_min = SegmentTree(cap, min, float("inf"))
        self.max_priority, self.size = 1.0, 0

    def add_row(self, row):
        for i in range(row * self.n_envs, (row + 1) * self.n_envs):
            self.it_sum[i] = self.max_priority ** self.alpha
            self.it_min[i] = self.max_priority ** self.alpha
        self.size = max(self.size, (row + 1) * self.n_envs)

    def sample(self, us, beta):
        total = self.it_sum._value[1]
        idxes = []
        for u in us:
            i = self.it_sum.find_prefixsum_idx(float(u) * total)
            idxes.append(min(i, self.size - 1))
        p_min = self.it_min._value[1] / total
        max_weight = (p_min * self.size) ** (-beta)
        weights = [((self.it_sum[i] / total) * self.size) ** (-beta) / max_weight for i in idxes]
        return np.array(idxes, np.int64), np.array(weights, np.float32)

    def update_priorities(self, idxes, td, eps):
        for i, t in zip(idxes, td):
            p = np.float32(abs(np.float32(t))) + np.float32(eps)
            self.it_sum[int(i)] = float(p) ** self.alpha
            self.it_min[int(i)] = float(p) ** self.alpha
            self.max_priority = max(self.max_priority, float(p))

    def trees(self):
        return np.array(self.it_sum._value), np.array(self.it_min._value)


def first_sample_model(u, n, tree_cap, prioritized, boundary=1e-11):
    """Indices of the uniforms ``u`` over ``n`` stored transitions whose leaves all hold 1 (a tree of ``tree_cap`` leaves, zeros past n),
    and the samples whose index may differ by one in a float64 walk (``u n`` within ``boundary n`` of a leaf boundary: the rule of the
    replay tests).  Uniform: min(floor(u n), n - 1), exact.  Prioritized: find_prefixsum_idx walked without building the tree, a node's sum
    being the number of stored leaves under it, and a walk into an empty leaf clamped to n - 1."""
    u = np.asarray(u, np.float64)
    if not prioritized:
        return np.minimum((u * n).astype(np.int64), n - 1), np.zeros(len(u), bool)
    mass, node, span = u * float(n), np.ones(len(u), np.int64), int(tree_cap)
    while span > 1:
        span //= 2
        left = np.clip(n - (2 * node * span - tree_cap), 0, span).astype(np.float64)      # stored leaves under the left child
        go_left = left > mass
        mass = np.where(go_left, mass, mass - left)
        node = 2 * node + (~go_left)
    un = u * float(n)
    return np.minimum(node - tree_cap, n - 1), np.abs(un - np.round(un)) <= boundary * n


def tree_sample_model(sum_tree, min_tree, size, tree_cap, u, beta, prioritized=True):
    """PrioritizedReplayBuffer.sample over the float64 trees ``sum_tree`` / ``min_tree`` (root 1, leaf i at tree_cap + i) holding ``size``
    transitions, for the uniforms ``u``: find_prefixsum_idx at mass u * total, one tree level per pass for every sample at once, a walk into
    an empty leaf clamped to size - 1, and weights (p_i size)^-beta / (p_min size)^-beta.  Uniform replay: min(floor(u size), size - 1) and
    weights 1.  Returns (idx, float32 weights)."""
    u, n = np.asarray(u, np.float64), int(size)
    if not prioritized:
        return np.minimum((u * n).astype(np.int64), n - 1), np.ones(len(u), np.float32)
    s = np.asarray(sum_tree, np.float64)
    total = s[1]
    mass, node = u * total, np.ones(len(u), np.int64)
    while node[0] < tree_cap:
        left = s[2 * node]
        right = left <= mass
        mass = np.where(right, mass - left, mass)
        node = 2 * node + right
    idx = np.minimum(node - tree_cap, n - 1)
    max_weight = (min_tree[1] / total * n) ** (-beta)
    return idx, ((s[tree_cap + idx] / total * n) ** (-beta) / max_weight).astype(np.float32)


def dqn_step_model(qnet, obs, act, rew, done, next_obs, gamma, lr, clip_norm, beta1, beta2, eps, target=None, weights=None, m=None, v=None,
                   step=1):
    """One gradient step of a DQN with online network ``qnet`` and target network ``target`` (default: ``qnet`` itself) over sampled rows
    with importance ``weights`` (default 1), from the Adam slots ``m``, ``v`` (default 0) at TF's step ``step`` (1-based): y (double Q), td
    and the gradients, the per-tensor clip factors, and the parameters and slots after the step."""
    y, _ = double_q_model(qnet, qnet if target is None else target, rew, done, next_obs, gamma)
    grads, td = dqn_grads_model(qnet, obs, act, y, np.ones(len(y)) if weights is None else weights)
    params = [p.detach().cpu().double().numpy() for p in qnet.parameters()]
    zeros = [np.zeros(p.shape) for p in params]
    new, m, v = clip_adam_model(params, grads, zeros if m is None else m, zeros if v is None else v, step, lr, clip_norm, beta1, beta2, eps)
    scale = [clip_norm / max(np.sqrt((g * g).sum()), clip_norm) for g in grads]
    return dict(y=y, td=td, grads=grads, clip_scale=scale, params=params, new_params=new, m=m, v=v)
