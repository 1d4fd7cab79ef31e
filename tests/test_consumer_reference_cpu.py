"""
The references of tests/test_consumer_kernels_gpu.py, and CPU checks that they compute what they claim.  The GPU file holds the PPO2
consumer kernels (include/srl_policy.h) to these models at the trainer's shapes, so a reader of the CPU suite alone can trust them:
  ppo2_minibatch_grads : rl_baselines.ppo2's minibatch loss through autograd, in the dtype of the policy it is given (float64 = the reference)
  filter_model         : VecNormalize's running moments (RunningNorm.update) as a two-pass float64 numpy merge
  normalise            : the float32 expression RunningNorm applies, on a given filter state
  policy_model         : the two 64-64 tanh towers of MlpPolicy and the log-probability of an action, in float64 numpy
  gae_torch, gae_model : the trainer's float32 torch GAE recursion, and the same recursion in float64 numpy
"""
import copy

import numpy as np
import pytest
import torch

from rl_baselines.ppo2 import RunningNorm
from test_policy_cpu import _policy

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
