"""
The references of tests/test_consumer_kernels_gpu.py, and CPU checks that they compute what they claim.  The GPU file holds the PPO2
consumer kernels (include/srl_policy.h) to these models at the trainer's shapes, so a reader of the CPU suite alone can trust them:
  ppo2_minibatch_grads : rl_baselines.ppo2's minibatch loss through autograd, in the dtype of the policy it is given (float64 = the reference)
  filter_model         : VecNormalize's running moments (RunningNorm.update) as a two-pass float64 numpy merge
  normalise            : the float32 expression RunningNorm applies, on a given filter state
  policy_model         : the two 64-64 tanh towers of MlpPolicy and the log-probability of an action, in float64 numpy
  philox_words         : Philox4x32-10 over many streams at once, in numpy
  sample_model         : the action the policy step draws from a Philox stream, written from the distributions' definitions
  gae_torch, gae_model : the trainer's float32 torch GAE recursion, and the same recursion in float64 numpy
  clip_adam_torch_model: nn.utils.clip_grad_norm_ followed by torch.optim.Adam (PPO2's optimiser), in float64 numpy
"""
import copy

import numpy as np
import pytest
import torch

from rl_baselines.ppo2 import RunningNorm
from test_policy_cpu import _policy, _ref_act, ref  # noqa: F401  (ref: module fixture of the CPU checker)

CLIP, ENT_COEF, VF_COEF = 0.2, 0.01, 0.5           # rl_baselines.ppo2.PPO2_DEFAULTS


# ---- PPO2 minibatch gradient ----

def ppo2_minibatch_grads(pol, idx, d, keep=None):
    """``param.grad`` after rl_baselines.ppo2's ``minibatch_step`` up to ``loss.backward()`` on a COPY of ``pol`` in its own dtype; `d` holds the
    rollout arrays (cast to that dtype).  ``keep`` (0 / 1 per minibatch sample) drops samples from the three loss terms only -- the advantage
    statistics and the 1 / minibatch of the means still see every sample: what a kernel that lost a chunk of its work would return."""
    pol = copy.deepcopy(pol)
    dt = next(pol.parameters()).dtype
    cast = lambda t: t.to(dt)
    obs, adv, ret, old_logp, old_val = (cast(d[k]) for k in ("obs", "adv", "ret", "old_logp", "old_val"))
    act = d["act"] if pol.discrete else cast(d["act"])
    logp, ent, v = pol.evaluate(obs[idx], act[idx])
    a_mb = adv[idx]
    a_mb = (a_mb - a_mb.mean()) / (a_mb.std() + 1e-8)
    ratio = torch.exp(logp - old_logp[idx])
    pg = torch.max(-a_mb * ratio, -a_mb * torch.clamp(ratio, 1 - CLIP, 1 + CLIP))
    vclip = old_val[idx] + torch.clamp(v - old_val[idx], -CLIP, CLIP)
    vf = torch.max((v - ret[idx]) ** 2, (vclip - ret[idx]) ** 2)
    if keep is not None:
        keep = keep.to(dt)
        pg, ent, vf = pg * keep, ent * keep, vf * keep
    loss = pg.mean() - ENT_COEF * ent.mean() + VF_COEF * (0.5 * vf.mean())
    loss.backward()
    return [p.grad.detach().clone() for p in pol.parameters()]


def ppo2_policy(obs_dim, discrete, n_out, device):
    """Trained-looking weights (the default head gain of 0.01 makes every logit ~0) and spread log-stds."""
    pol = _policy(obs_dim, discrete, n_out, seed=7).to(device)
    with torch.no_grad():
        for p in pol.parameters():
            p.mul_(3.0)
        if not discrete:
            pol.logstd.copy_(torch.linspace(-0.5, 0.3, n_out))
    return pol


def ppo2_rollout(pol, rows, seed):
    """Rollout arrays for a minibatch step.  Ratios from ~0.3 to ~3 and value moves up to ~1 reach both sides of both clip ranges; the loss
    gradient is discontinuous at the clip boundaries, so the data stay 5 % away from the four of them (a sample on a boundary to within
    float32 rounding is decided by the last bit of the forward pass).  The advantages trend along the row index, so that a sample missing
    from the advantage statistics moves their mean and std instead of cancelling."""
    dev = next(pol.parameters()).device
    D, A = pol.pi[0].weight.shape[1], pol.pi[-1].weight.shape[0]
    g = torch.Generator(device=dev).manual_seed(seed)
    obs = torch.randn((rows, D), device=dev, generator=g)
    act = torch.randint(0, A, (rows,), device=dev, generator=g) if pol.discrete else torch.randn((rows, A), device=dev, generator=g)
    with torch.no_grad():
        logp0, _, v0 = pol.evaluate(obs, act)
    dl = 0.4 * torch.randn(rows, device=dev, generator=g)
    for edge in (-float(np.log(1.2)), -float(np.log(0.8))):          # logp - old_logp = -dl at log(1 +- clip)
        dl = torch.where((dl - edge).abs() < 0.01, dl * 1.2, dl)
    dvn = 0.3 * torch.randn(rows, device=dev, generator=g)
    dvn = torch.where((dvn.abs() - CLIP).abs() < 0.01, dvn * 1.2, dvn)
    row = torch.arange(rows, device=dev, dtype=torch.float32)
    return dict(obs=obs, act=act, old_logp=(logp0 + dl).contiguous(), old_val=(v0 + dvn).contiguous(),
                adv=(0.5 + 2.0 * torch.randn(rows, device=dev, generator=g) + 3.0 * row / rows).contiguous(),
                ret=(v0 + torch.randn(rows, device=dev, generator=g)).contiguous())


def grad_errors(got, want):
    """Per tensor: (max |got - want|, max |want|)."""
    return [(float((a.double() - b.double()).abs().max()), float(b.abs().max())) for a, b in zip(got, want)]


def grad_bound(scale):
    """The tolerance of a gradient tensor: 2e-4 of its largest entry, + 2e-6 (a bias gradient is a sum of terms that may cancel)."""
    return 2e-4 * scale + 2e-6


# ---- observation filter ----

def filter_model(state, x):
    """RunningNorm.update in float64 numpy, batch moments in two passes.  state = [mean[D], var[D], count]."""
    D = x.shape[1]
    mean, var, count = state[:D], state[D:2 * D], state[2 * D]
    x = np.asarray(x, np.float64)
    bm = x.mean(0)
    bv = ((x - bm) ** 2).mean(0)
    bc = float(x.shape[0])
    delta, tot = bm - mean, count + bc
    return np.concatenate([mean + delta * bc / tot, (var * count + bv * bc + delta ** 2 * count * bc / tot) / tot, [tot]])


def normalise(x, state, clip=10.0, eps=1e-8):
    """RunningNorm's float32 output expression, on the filter state `state` (a float64 tensor on x's device)."""
    D = x.shape[1]
    return torch.clamp((x - state[:D].float()) / torch.sqrt(state[D:2 * D].float() + eps), -clip, clip)


# ---- policy step ----

def policy_model(pol, obs):
    """(logits or Gaussian means [n, n_out], values [n]) of MlpPolicy in float64 numpy."""
    def tower(seq, h):
        lin = [m for m in seq if isinstance(m, torch.nn.Linear)]
        for k, m in enumerate(lin):
            h = h @ m.weight.detach().cpu().double().numpy().T + m.bias.detach().cpu().double().numpy()
            if k < len(lin) - 1:
                h = np.tanh(h)
        return h
    x = np.asarray(obs, np.float64)
    return tower(pol.pi, x), tower(pol.vf, x)[:, 0]


def logp_model(pol, out, act):
    """float64 log-probability of `act` (int [n] / float [n, n_out]) under the distribution with logits / means `out`."""
    if pol.discrete:
        m = out.max(1, keepdims=True)
        lsm = out - m - np.log(np.exp(out - m).sum(1, keepdims=True))
        return lsm[np.arange(out.shape[0]), np.asarray(act, np.int64)]
    ls = pol.logstd.detach().cpu().double().numpy()
    z = (np.asarray(act, np.float64) - out) / np.exp(ls)
    return (-0.5 * z * z - ls - 0.5 * np.log(2.0 * np.pi)).sum(1)


# ---- the policy's draws ----

PURPOSE_POLICY = 16                # counter word 3 of the categorical draw; the Gaussian's block k // 4 uses 17 + k // 4


def philox_words(seed, envs, counter, purpose):
    """Philox4x32-10 (Salmon et al., SC'11) of the streams ``envs`` in numpy: [len(envs), 4] uint32 words.  Key = seed; counter = (env lo,
    env hi, ``counter``, ``purpose``)."""
    M = np.uint64(0xFFFFFFFF)
    env = np.asarray(envs, np.uint64).reshape(-1)
    c0, c1 = env & M, env >> np.uint64(32)
    c2, c3 = np.full_like(c0, int(counter) & 0xFFFFFFFF), np.full_like(c0, int(purpose) & 0xFFFFFFFF)
    k0, k1 = int(seed) & 0xFFFFFFFF, (int(seed) >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = c0 * np.uint64(0xD2511F53), c2 * np.uint64(0xCD9E8D57)        # 32 x 32 -> 64 bits: no wrap in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & M, (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & M
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return np.stack([c0, c1, c2, c3], 1).astype(np.uint32)


def u53(words):
    """The 53-bit uniform in [0, 1) of words 0 and 1 (numpy's random_sample construction)."""
    w = words.astype(np.float64)
    return (np.floor(w[:, 0] / 32.0) * 67108864.0 + np.floor(w[:, 1] / 64.0)) / 9007199254740992.0


def sample_model(out64, sigma, seed, envs, counter, near_tol=None):
    """The action drawn for each env of ``envs`` at sampling counter ``counter``, in float64 from the distributions' definitions.
    ``out64`` [n, n_out]: logits (``sigma`` None) or Gaussian means (``sigma`` [n_out]: the standard deviations).
      Categorical: inverse CDF of softmax(logits) at u = the 53-bit uniform of words 0 and 1 of Philox (seed; env; counter; 16).
      Gaussian:    Box-Muller on 24-bit uniforms (w >> 8 + 1/2) / 2^24.  Dimension k takes block 17 + k // 4; words (0, 1) are the pair of
                   k % 4 = 0 (cos) and 1 (sin), words (2, 3) the pair of k % 4 = 2 (cos) and 3 (sin).
    Returns (action, near, z): ``near`` marks categorical draws whose u lies within ``near_tol`` (per row; default 1e-5 (1 + max |logit|),
    the float32 rounding of logits, exponentials and the running CDF sum) of a CDF boundary, where a float32 computation may take either
    side; ``z`` [n, n_out] are the Gaussian's standard normals (None for a categorical)."""
    out64 = np.asarray(out64, np.float64)
    n, A = out64.shape
    if sigma is None:
        u = u53(philox_words(seed, envs, counter, PURPOSE_POLICY))
        p = np.exp(out64 - out64.max(1, keepdims=True))
        cdf = np.cumsum(p / p.sum(1, keepdims=True), 1)[:, :-1]               # the last boundary is 1: u < 1 always
        act = (cdf <= u[:, None]).sum(1)
        tol = 1e-5 * (1.0 + np.abs(out64).max(1)) if near_tol is None else near_tol
        near = (np.abs(cdf - u[:, None]) <= np.reshape(tol, (-1, 1))).any(1) if A > 1 else np.zeros(n, bool)
        return act, near, None
    z = np.zeros((n, A))
    for k in range(A):
        w = philox_words(seed, envs, counter, PURPOSE_POLICY + 1 + k // 4).astype(np.float64)
        j = k & 2
        u1, u2 = (np.floor(w[:, j] / 256.0) + 0.5) / 16777216.0, (np.floor(w[:, j + 1] / 256.0) + 0.5) / 16777216.0
        rad, ang = np.sqrt(-2.0 * np.log(u1)), 2.0 * np.pi * u2
        z[:, k] = rad * (np.sin(ang) if k & 1 else np.cos(ang))
    return out64 + np.asarray(sigma, np.float64) * z, np.zeros(n, bool), z


def box_sample_bound(out64, sigma, z):
    """How far a float32 draw may sit from mean64 + sigma64 z64: the float32 towers' error on the mean (the value tolerance of the kernel
    tests, 2e-5 + 1e-6 |mean|), float32 logf / sqrtf / sinf / cosf on z (a few ulps: 1e-6 (1 + |z|) with margin) scaled by sigma, and the
    rounding of the final fused multiply-add."""
    return 2e-5 + 2e-6 * np.abs(out64) + 2e-6 * np.asarray(sigma) * (1.0 + np.abs(z))


# ---- GAE ----

def gae_torch(rew, val, done, last_val, gamma, lam):
    """rl_baselines.ppo2's GAE recursion (the torch path of its gae())."""
    T, N = rew.shape
    adv, ret = torch.zeros_like(rew), torch.zeros_like(rew)
    lastgae = torch.zeros(N, device=rew.device)
    for t in reversed(range(T)):
        nonterminal = 1.0 - done[t]
        nextval = last_val if t == T - 1 else val[t + 1]
        delta = rew[t] + gamma * nextval * nonterminal - val[t]
        lastgae = delta + gamma * lam * nonterminal * lastgae
        adv[t].copy_(lastgae)
    torch.add(adv, val, out=ret)
    return adv, ret


def gae_model(rew, val, done, last_val, gamma, lam):
    """The same recursion in float64 numpy."""
    rew, val, done, last_val = (np.asarray(a, np.float64) for a in (rew, val, done, last_val))
    T = rew.shape[0]
    adv = np.zeros_like(rew)
    lastgae, nextval = np.zeros_like(last_val), last_val
    for t in reversed(range(T)):
        nt = 1.0 - done[t]
        lastgae = rew[t] + gamma * nextval * nt - val[t] + gamma * lam * nt * lastgae
        adv[t] = lastgae
        nextval = val[t]
    return adv, adv + val


def gae_rollout(T, N, device, seed):
    """Rewards, values, dones and bootstrap values of a [T, N] rollout; dones at t = 0, at t = T - 1 and on consecutive steps."""
    g = torch.Generator(device=device).manual_seed(seed)
    rew = torch.randn((T, N), device=device, generator=g)
    val = torch.randn((T, N), device=device, generator=g) * 3.0
    done = (torch.rand((T, N), device=device, generator=g) < 0.05).float()
    done[0, ::3] = 1.0
    done[T - 1, 1::2] = 1.0
    if T >= 4:
        done[T // 2:T // 2 + 3, ::4] = 1.0
    return rew, val, done, torch.randn(N, device=device, generator=g) * 3.0


GAE_ULPS = 8       # float32 recursion vs float64, in float32 ulps (2^-23) of the tensor's largest magnitude: up to 3.3 at T = 129


# ---- PPO2's optimiser ----

def clip_grad_norm_model(grads, max_norm):
    """nn.utils.clip_grad_norm_: the global 2-norm over every tensor, coef = max_norm / (norm + 1e-6) clamped at 1.  Returns (clipped grads, coef)."""
    norm = np.sqrt(sum(float((np.asarray(g, np.float64) ** 2).sum()) for g in grads))
    coef = min(1.0, max_norm / (norm + 1e-6))
    return [np.asarray(g, np.float64) * coef for g in grads], coef


def adam_torch_model(params, grads, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-5):
    """Step ``step`` (1-based) of torch.optim.Adam without weight decay or amsgrad: bias-corrected moments, eps added AFTER the square root
    (torch's formula; TF's Adam in tests/deepq_numpy_ref.py adds it to the uncorrected root).  Returns (params, m, v)."""
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    new_p, new_m, new_v = [], [], []
    for p, g, mk, vk in zip(params, grads, m, v):
        mk = beta1 * np.asarray(mk, np.float64) + (1.0 - beta1) * g
        vk = beta2 * np.asarray(vk, np.float64) + (1.0 - beta2) * g * g
        new_p.append(np.asarray(p, np.float64) - (lr / bc1) * mk / (np.sqrt(vk) / np.sqrt(bc2) + eps))
        new_m.append(mk)
        new_v.append(vk)
    return new_p, new_m, new_v


def clip_adam_torch_model(params, grad_steps, lr, max_norm=0.5, eps=1e-5):
    """PPO2's optimiser over a sequence of raw gradients (lists of arrays), from zero Adam slots: clip_grad_norm_(max_norm) then one Adam step
    each.  Returns (params, m, v, clipped gradients of every step)."""
    p = [np.asarray(x, np.float64) for x in params]
    m, v, clipped = [np.zeros_like(x) for x in p], [np.zeros_like(x) for x in p], []
    for s, g in enumerate(grad_steps):
        gc, _ = clip_grad_norm_model(g, max_norm)
        clipped.append(gc)
        p, m, v = adam_torch_model(p, gc, m, v, s + 1, lr, eps=eps)
    return p, m, v, clipped


# ---- CPU checks of the references ----

@pytest.mark.parametrize("discrete,obs_dim,n_out", [(True, 3, 6), (True, 1, 2), (False, 3, 7), (False, 1, 2)])
def test_float64_ppo2_gradient_matches_float32_autograd(discrete, obs_dim, n_out):
    """The float64 reference is the trainer's loss: float32 autograd on the same minibatch agrees with it to float32 accuracy, an all-ones
    `keep` changes nothing, and dropping 64 samples moves it far outside the kernels' tolerance."""
    pol = ppo2_policy(obs_dim, discrete, n_out, "cpu")
    d = ppo2_rollout(pol, 900, seed=1)
    idx = torch.randperm(900, generator=torch.Generator().manual_seed(2))[:640]
    g64 = ppo2_minibatch_grads(copy.deepcopy(pol).double(), idx, d)
    g32 = ppo2_minibatch_grads(pol, idx, d)
    assert [t.dtype for t in g64] == [torch.float64] * len(g64) and [t.dtype for t in g32] == [torch.float32] * len(g32)
    # the value tower's gradients carry v - ret ~ 1 against values of ~50: float32 rounding of v shows up as up to ~1e-4 of the tensor's scale
    for (name, _), (err, scale) in zip(pol.named_parameters(), grad_errors(g32, g64)):
        assert scale > 0 and err <= grad_bound(scale), (name, err, scale)
    ones = ppo2_minibatch_grads(copy.deepcopy(pol).double(), idx, d, keep=torch.ones(640))
    assert all(torch.equal(a, b) for a, b in zip(ones, g64))
    keep = torch.ones(640)
    keep[64:128] = 0.0
    dropped = ppo2_minibatch_grads(copy.deepcopy(pol).double(), idx, d, keep=keep)
    assert max(err / grad_bound(scale) for err, scale in grad_errors(dropped, g64)) > 10.0


def test_ppo2_rollout_keeps_the_clip_boundaries_away():
    pol = ppo2_policy(3, True, 6, "cpu")
    d = ppo2_rollout(pol, 20000, seed=4)
    with torch.no_grad():
        logp, _, v = copy.deepcopy(pol).double().evaluate(d["obs"].double(), d["act"])
    lr = (logp - d["old_logp"].double()).numpy()
    dv = (v - d["old_val"].double()).numpy()
    for edge in (np.log(1.2), np.log(0.8)):
        assert np.abs(lr - edge).min() > 0.009
    assert np.abs(np.abs(dv) - CLIP).min() > 0.009
    assert (lr > np.log(1.2)).mean() > 0.1 and (lr < np.log(0.8)).mean() > 0.1 and (np.abs(dv) > CLIP).mean() > 0.1   # both sides are reached


@pytest.mark.parametrize("D", range(1, 9))
def test_filter_model_matches_running_norm(D):
    rng = np.random.default_rng(D)
    norm = RunningNorm(D, torch.device("cpu"))
    state = norm.state.numpy().copy()
    for it, n in enumerate((1, 33, 4097)):
        x = (rng.normal(0.0, 1.0, (n, D)) * np.linspace(0.3, 9.0, D) + np.linspace(-4.0, 4.0, D) * (it + 1)).astype(np.float32)
        state = filter_model(state, x)
        norm.update(torch.from_numpy(x))
        assert np.allclose(state[:D], norm.mean.numpy(), rtol=0, atol=1e-12)
        assert np.allclose(state[D:2 * D], norm.var.numpy(), rtol=1e-12, atol=1e-12)
        assert state[2 * D] == pytest.approx(float(norm.count), rel=1e-15)
        xt = torch.from_numpy(x)
        assert torch.equal(normalise(xt, norm.state), norm(xt, update=False))


@pytest.mark.parametrize("discrete,obs_dim,n_out", [(True, 3, 6), (True, 1, 2), (False, 3, 7), (False, 1, 1)])
def test_float64_policy_model_matches_torch(discrete, obs_dim, n_out):
    pol = _policy(obs_dim, discrete, n_out, seed=3)
    obs = torch.randn(2000, obs_dim) * 1.5
    out, value = policy_model(pol, obs.numpy())
    pol64, x64 = copy.deepcopy(pol).double(), obs.double()
    with torch.no_grad():
        act = pol.dist(obs).sample()
        t_out, t_val = pol64.pi(x64), pol64.vf(x64).squeeze(-1)
        d = pol64.dist(x64)
        t_logp = d.log_prob(act) if discrete else d.log_prob(act.double()).sum(-1)
    assert np.abs(out - t_out.numpy()).max() < 1e-12 and np.abs(value - t_val.numpy()).max() < 1e-12
    assert np.abs(logp_model(pol, out, act.numpy()) - t_logp.numpy()).max() < 1e-11


@pytest.mark.parametrize("T,N", [(1, 5), (9, 129), (129, 64)])
def test_gae_references_agree(T, N):
    """The float32 torch recursion stays within a few float32 ulps of the float64 one (the GPU tests hold the kernel to both)."""
    rew, val, done, last_val = gae_rollout(T, N, "cpu", seed=T)
    assert done[0].sum() > 0 and done[T - 1].sum() > 0
    for gamma, lam in ((0.99, 0.95), (0.9, 0.9)):
        adv, ret = gae_torch(rew, val, done, last_val, gamma, lam)
        a64, r64 = gae_model(rew.numpy(), val.numpy(), done.numpy(), last_val.numpy(), gamma, lam)
        for got, want in ((adv, a64), (ret, r64)):
            assert np.abs(got.numpy() - want).max() <= GAE_ULPS * 2.0 ** -23 * np.abs(want).max()
        if T == 1:      # no recursion: adv = rew + gamma * last_val * (1 - done) - val
            assert np.allclose(a64[0], (rew[0] + gamma * last_val * (1 - done[0]) - val[0]).numpy(), rtol=1e-6, atol=1e-6)


def test_numpy_philox_matches_the_oracle(oracle_lib):
    """philox_words equals the oracle's Philox4x32-10 (itself held to the published known-answer vectors in tests/test_mobile_cpu.py) word for
    word, over streams that cross 2^32, counters up to 2^32 - 1, every policy purpose and a 64-bit key."""
    import ctypes
    fn = oracle_lib.lib.oracle_philox4x32
    fn.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32)]
    fn.restype = None
    out = (ctypes.c_uint32 * 4)()
    envs = [0, 1, 7, 4095, 4096, 2 ** 32 - 1, 2 ** 32 + 5, 2 ** 63 + 3]
    for seed in (0, 1234, 0x299F31D0A4093822):
        for counter in (0, 1, 31, 2 ** 32 - 1):
            for purpose in (16, 17, 18):
                got = philox_words(seed, envs, counter, purpose)
                for i, e in enumerate(envs):
                    fn(seed, e, counter, purpose, out)
                    assert list(got[i]) == list(out), (seed, e, counter, purpose)
    w = np.array([[0, 0, 0, 0], [0xFFFFFFFF, 0xFFFFFFFF, 0, 0], [0x80000000, 0, 0, 0]], np.uint32)
    assert list(u53(w)) == [0.0, 1.0 - 2.0 ** -53, 0.5]


@pytest.mark.parametrize("discrete,obs_dim,n_out", [(True, 3, 1), (True, 3, 3), (True, 12, 7), (False, 3, 1), (False, 3, 3), (False, 12, 7)])
def test_sample_model_matches_the_checker_draws(ref, discrete, obs_dim, n_out):
    """The host checker (csrc/policy_core.h compiled for the CPU) draws what sample_model says, at the float64 towers' outputs: the same category
    except at the few draws within rounding of a CDF boundary, and Gaussian samples within float32 of mean64 + sigma64 z64.  n_out = 7 is the
    Gaussian's two-block case.  Two counters and an env offset check the stream each draw takes; the models of two natural mistakes (every
    Gaussian dimension from the first word pair, a CDF from half the logits) are far from the checker."""
    pol = _policy(obs_dim, discrete, n_out, seed=60 + obs_dim + n_out)
    n = 6000
    obs = torch.randn(n, obs_dim, generator=torch.Generator().manual_seed(obs_dim)) * 1.5
    out64, _ = policy_model(pol, obs.numpy())
    sigma = None if discrete else np.exp(pol.logstd.detach().double().numpy())
    for seed, counter, off in ((5, 0, 0), (1234, 3, 4096)):
        _, act_buf, _, _, _ = _ref_act(ref, pol, obs, seed=seed, counter=counter, env_offset=off)
        act, near, z = sample_model(out64, sigma, seed, np.arange(n) + off, counter)
        if discrete:
            same = act_buf == act
            print("\n%s n_out=%d counter %d: %d of %d draws near a CDF boundary, %d of them differ" % (discrete, n_out, counter, near.sum(), n,
                                                                                                     (~same[near]).sum()))
            assert same[~near].all(), np.nonzero(~same & ~near)[0][:10]
            assert near.sum() <= 2e-3 * n
            if n_out > 1:
                assert len(np.unique(act)) == n_out
                p = np.exp(0.5 * (out64 - out64.max(1, keepdims=True)))
                u = u53(philox_words(seed, np.arange(n) + off, counter, PURPOSE_POLICY))
                half = (np.cumsum(p / p.sum(1, keepdims=True), 1)[:, :-1] <= u[:, None]).sum(1)
                assert (half != act_buf).mean() > 0.01
        else:
            err = np.abs(act_buf - act)
            assert (err <= box_sample_bound(out64, sigma, z)).all(), err.max()
            assert 0.9 < z.std() < 1.1 and abs(z.mean()) < 0.1
            if n_out > 2:                               # dims 2 and 3 from words (2, 3), not again from words (0, 1)
                assert np.abs(act_buf[:, 2] - (out64[:, 2] + sigma[2] * z[:, 0])).max() > 0.1
            if n_out > 4:                               # dim 4 from a second block, not again from the first
                assert np.abs(act_buf[:, 4] - (out64[:, 4] + sigma[4] * z[:, 0])).max() > 0.1


def test_clip_adam_model_matches_torch():
    """clip_adam_torch_model is nn.utils.clip_grad_norm_(0.5) + torch.optim.Adam(eps=1e-5) in float64 over four steps: one gradient far above the
    clip norm, one below it, one at about twice it, one of zeros (the moments decay, the step stays finite).  torch runs the CPU Adam
    implementation here; the trainer's capturable CUDA Adam states the same formula."""
    g = torch.Generator().manual_seed(3)
    shapes = [(64, 3), (64,), (64, 64), (6,)]
    params = [torch.randn(s, generator=g, dtype=torch.float64, requires_grad=True) for s in shapes]
    p0 = [p.detach().numpy().copy() for p in params]
    opt = torch.optim.Adam(params, lr=2.5e-4, eps=1e-5)
    steps = []
    for scale in (3.0, 0.001, 0.01, 0.0):
        grads = [torch.randn(s, generator=g, dtype=torch.float64) * scale for s in shapes]
        steps.append([x.numpy().copy() for x in grads])
        for p, x in zip(params, grads):
            p.grad = x.clone()
        torch.nn.utils.clip_grad_norm_(params, 0.5)
        opt.step()
    assert np.sqrt(sum((x ** 2).sum() for x in steps[0])) > 10 * 0.5 and np.sqrt(sum((x ** 2).sum() for x in steps[1])) < 0.5
    got_p, got_m, got_v, clipped = clip_adam_torch_model(p0, steps, 2.5e-4)
    for k, p in enumerate(params):
        st = opt.state[p]
        assert float(st["step"]) == 4.0
        assert np.allclose(got_m[k], st["exp_avg"].numpy(), rtol=1e-12, atol=1e-300)
        assert np.allclose(got_v[k], st["exp_avg_sq"].numpy(), rtol=1e-12, atol=1e-300)
        assert np.allclose(got_p[k], p.detach().numpy(), rtol=0, atol=1e-15)
    assert np.allclose(np.sqrt(sum((x ** 2).sum() for x in clipped[0])), 0.5 / (1.0 + 1e-6 / np.sqrt(sum((x ** 2).sum() for x in steps[0]))), rtol=1e-12)
    assert all(np.array_equal(a, b) for a, b in zip(clipped[1], steps[1]))
    # TF's Adam (eps on the uncorrected root) differs visibly after one step at this eps: the model is torch's, not TF's
    _, m1, v1 = adam_torch_model(p0, clipped[1], [np.zeros_like(x) for x in p0], [np.zeros_like(x) for x in p0], 1, 1.0)
    tf_move = np.sqrt(1 - 0.999) / (1 - 0.9) * m1[1] / (np.sqrt(v1[1]) + 1e-5)
    torch_move = m1[1] / (1 - 0.9) / (np.sqrt(v1[1]) / np.sqrt(1 - 0.999) + 1e-5)
    assert np.abs(tf_move - torch_move).max() > 1e-3
