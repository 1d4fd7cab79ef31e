"""
GPU tests of the PPO2 consumer kernels (include/srl_policy.h) at the shapes the trainer runs, against the float64 references of
tests/test_consumer_reference_cpu.py:
  srl_ppo2_grad   -- float64 autograd of the trainer's minibatch loss, at minibatches where every CTA walks several chunks (mb = 131 072 is
                     the 4096-env trainer's) and where the advantage statistics loop twice;
  srl_obs_filter  -- a two-pass float64 merge for every obs_dim, on batches on both sides of the 4096 rows a thread block keeps in registers;
  srl_policy_act  -- a float64 model at every registry shape, with weights the kernel cannot load 16 bytes at a time, and sharded over two launches;
  srl_ppo2_gae    -- the trainer's float32 torch recursion bit for bit, and a float64 one, at lengths that are not multiples of 8.
Minibatch sizes are expressed in SMs, so "k chunks per CTA" holds on any device.
"""
import copy
from ctypes import byref

import numpy as np
import pytest
import torch

from test_consumer_reference_cpu import (GAE_ULPS, box_sample_bound, filter_model, gae_model, gae_rollout, gae_torch, grad_bound, grad_errors,
                                         logp_model, normalise, policy_model, ppo2_minibatch_grads, ppo2_policy, ppo2_rollout, sample_model, CLIP,
                                         ENT_COEF, VF_COEF)
from test_policy_cpu import _policy

pytestmark = pytest.mark.gpu

CH = 64                                   # samples per chunk of ppo2_grad_kernel


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def lib(cuda_lib):
    from srl_sim.policy import bind
    bind(cuda_lib.lib)
    return cuda_lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------- srl_ppo2_grad

GRAD_SHAPES = [(True, 3, 6), (True, 2, 4), (True, 1, 2), (False, 3, 3), (False, 3, 7), (False, 2, 2), (False, 1, 2)]
# "3_chunks_per_cta" = SMs * 64 * 3 + 17: every CTA walks at least 3 chunks and the ragged last chunk is the 4th of CTA 0;
# 131072 = T * N / 4 of the 4096-env trainer; 200003 > 131072 = 8 x 64 x 256: adv_stats_kernel's outer loop runs twice.
GRAD_SIZES = ["3_chunks_per_cta", "131072", "200003"]


def _grad_mb(size):
    return _sms() * CH * 3 + 17 if size == "3_chunks_per_cta" else int(size)


@pytest.mark.parametrize("use_idx", [True, False], ids=["idx", "no_idx"])
@pytest.mark.parametrize("size", GRAD_SIZES)
@pytest.mark.parametrize("discrete,obs_dim,n_out", GRAD_SHAPES)
def test_ppo2_grad_matches_float64_autograd(lib, discrete, obs_dim, n_out, size, use_idx):
    """Every parameter gradient within 2e-4 of its tensor's largest entry (+ 2e-6) of float64 autograd; float32 autograd's own error on the
    same data is printed next to the kernel's.  At 131 072 a second call gives the same bytes.  At the 3-chunks size the check is shown to
    see a lost chunk: the float64 gradient without one whole chunk of the minibatch is far outside the tolerance of the kernel's result."""
    from srl_sim.policy import FusedPPO2Grad
    mb = _grad_mb(size)
    rows = mb + mb // 3 if use_idx else mb + 5
    pol = ppo2_policy(obs_dim, discrete, n_out, "cuda")
    d = ppo2_rollout(pol, rows, seed=mb)
    g = torch.Generator(device="cuda").manual_seed(11)
    idx = torch.randperm(rows, device="cuda", generator=g)[:mb].contiguous() if use_idx else None
    ref_idx = idx if use_idx else torch.arange(mb, device="cuda")
    pol64 = copy.deepcopy(pol).double()
    want = ppo2_minibatch_grads(pol64, ref_idx, d)
    f32 = grad_errors(ppo2_minibatch_grads(pol, ref_idx, d), want)

    fused = FusedPPO2Grad(lib, pol, mb)
    fused(idx, d["obs"], d["act"], d["adv"], d["ret"], d["old_logp"], d["old_val"], CLIP, ENT_COEF, VF_COEF, stream=_stream())
    torch.cuda.synchronize()
    got = [p.grad.detach().clone() for p in pol.parameters()]
    kern = grad_errors(got, want)
    names = [n for n, _ in pol.named_parameters()]
    print("\nppo2_grad %s mb=%d %s  max|g - g64| / max|g64|  kernel | float32 autograd:" % ((discrete, obs_dim, n_out), mb, "idx" if use_idx else "no idx"))
    print("  " + "  ".join("%s %.1e|%.1e" % (n, e / s, e32 / s) for n, (e, s), (e32, _) in zip(names, kern, f32)))
    # The bound is 2e-4 of the tensor's scale PLUS 4x float32 autograd's own error on the same data.  The second term matters for the value
    # tower only: its loss derivative is v - ret with |v| up to ~50 and |v - ret| ~ 1, so float32 rounding of v (ulp(50) ~ 4e-6, in torch as in
    # the kernel) is a visible share of it, and that share grows with the minibatch -- the gradient, a mean of noise-dominated v - ret, shrinks
    # while the rounding of correlated values does not average out.  Measured on an H100 for the value tower at (Discrete, 1, 2): float32
    # autograd 1e-4 of the scale at mb = 25 361, 6.6e-4 at 200 003, the kernel within 3x of it; the policy tower stays at ~1e-6 for both.
    for n, (err, scale), (e32, _) in zip(names, kern, f32):
        assert scale > 0 and err <= grad_bound(scale) + 4.0 * e32, (n, err, e32, scale)

    if size == "131072":
        fused(idx, d["obs"], d["act"], d["adv"], d["ret"], d["old_logp"], d["old_val"], CLIP, ENT_COEF, VF_COEF, stream=_stream())
        torch.cuda.synchronize()
        assert all(torch.equal(p.grad, a) for p, a in zip(pol.parameters(), got))
    if size == "3_chunks_per_cta":
        keep = torch.ones(mb, device="cuda")
        lost = _sms() + 1                                   # CTA 1's second chunk
        keep[lost * CH:(lost + 1) * CH] = 0.0
        wrong = grad_errors(got, ppo2_minibatch_grads(pol64, ref_idx, d, keep=keep))
        margin = max(err / grad_bound(scale) for err, scale in wrong)
        print("  without chunk %d of %d the float64 reference is %.0f x the tolerance away from the kernel" % (lost, (mb + CH - 1) // CH, margin))
        assert margin > 10.0


# ---------------------------------------------------------------- srl_obs_filter

FILTER_SCALE = [0.3, 2.0, 9.0, 0.5, 4.0, 1.0, 0.7, 3.0]
FILTER_OFFSET = [1.0, -4.0, 0.5, 3.0, -2.0, 0.0, 2.5, -1.0]
FILTER_DRIFT = [0.0, 1.5, 0.0, -1.0, 0.0, 0.5, 0.0, 2.0]


def _filter(lib, x, state, update, out):
    n, D = x.shape
    rc = lib.lib.srl_obs_filter(n, D, x.data_ptr(), state.data_ptr(), int(update), 10.0, 1e-8, out.data_ptr(), _stream())
    lib.check(rc, "srl_obs_filter")


@pytest.mark.parametrize("n", [1, 33, 4096, 4097, 8192, 50000])
@pytest.mark.parametrize("D", range(1, 9))
def test_obs_filter_matches_a_float64_merge_and_torch_normalisation(lib, D, n):
    """Three updates from RunningNorm's initial state (per-dimension scales and offsets, some dimensions drifting): the state against a
    two-pass float64 merge, the output bit for bit against RunningNorm's float32 expression on the kernel's own state.  Then update=False
    leaves the state alone and clips a far outlier."""
    from rl_baselines.ppo2 import RunningNorm
    state = RunningNorm(D, torch.device("cuda", 0)).state
    model = state.cpu().numpy().copy()
    g = torch.Generator(device="cuda").manual_seed(100 * D + n % 97)
    scale, offset, drift = (torch.tensor(v[:D], device="cuda") for v in (FILTER_SCALE, FILTER_OFFSET, FILTER_DRIFT))
    for it in range(3):
        x = (torch.randn((n, D), device="cuda", generator=g) * scale + offset + drift * it).contiguous()
        out = torch.full_like(x, float("nan"))
        _filter(lib, x, state, True, out)
        torch.cuda.synchronize()
        model = filter_model(model, x.cpu().numpy())
        s = state.cpu().numpy()
        assert np.allclose(s[:D], model[:D], rtol=0, atol=1e-11), (s[:D], model[:D])
        assert np.allclose(s[D:2 * D], model[D:2 * D], rtol=1e-11, atol=1e-11), (s[D:2 * D], model[D:2 * D])
        assert s[2 * D] == pytest.approx(model[2 * D], rel=1e-14)
        assert torch.equal(out, normalise(x, state))
    frozen = state.clone()
    x = (torch.randn((n, D), device="cuda", generator=g) * scale * 40.0 + offset).contiguous()
    x[0] = frozen[:D].float() + 12.0 * frozen[D:2 * D].sqrt().float()        # 12 standard deviations out in every dimension
    out = torch.full_like(x, float("nan"))
    _filter(lib, x, state, False, out)
    torch.cuda.synchronize()
    assert torch.equal(state, frozen)
    assert torch.equal(out, normalise(x, state)) and torch.equal(out[0], torch.full((D,), 10.0, device="cuda"))


# ---------------------------------------------------------------- srl_policy_act

ACT_SHAPES = GRAD_SHAPES + [(False, 1, 1)]


def _act_buffers(n, n_out, discrete, obs_dim):
    z = lambda *shape, dtype=torch.float32: torch.full(shape, -7, dtype=dtype, device="cuda")
    return dict(act_env=z(n, dtype=torch.int32) if discrete else z(n, n_out), act_buf=z(n, dtype=torch.int64) if discrete else z(n, n_out),
                logp=z(n), value=z(n), obs_buf=z(n, obs_dim))


def _act(lib, st, n, obs, rng, env_offset, b, first=0):
    """srl_policy_act over envs [first, first + n) of the buffers in `b`, with the sampling streams env_offset + i."""
    rc = lib.lib.srl_policy_act(byref(st), n, obs[first:].data_ptr(), rng.data_ptr(), env_offset, b["obs_buf"][first:].data_ptr(),
                                b["act_env"][first:].data_ptr(), b["act_buf"][first:].data_ptr(), b["logp"][first:].data_ptr(),
                                b["value"][first:].data_ptr(), _stream())
    lib.check(rc, "srl_policy_act")


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4096, 8192])
@pytest.mark.parametrize("discrete,obs_dim,n_out", ACT_SHAPES)
def test_policy_act_against_a_float64_model(lib, discrete, obs_dim, n_out, n):
    """Value and log-probability OF THE ACTION THE KERNEL DREW against the float64 towers, the draw itself against sample_model at the launch's
    counter, Box actions clipped for the env, the rollout buffer copy of the observations, and the sampling counter advancing by exactly one
    per launch."""
    from srl_sim.policy import policy_struct
    pol = _policy(obs_dim, discrete, n_out, seed=40 + obs_dim * 9 + n_out).cuda()
    st, keep = policy_struct(pol)
    seed = 1234 + n
    rng = torch.tensor([seed, 0, 0], dtype=torch.int64, device="cuda")
    obs = (torch.randn((n, obs_dim), device="cuda", generator=torch.Generator(device="cuda").manual_seed(n)) * 1.5).contiguous()
    out64, v64 = policy_model(pol, obs.cpu().numpy())
    sigma = None if discrete else np.exp(pol.logstd.detach().cpu().double().numpy())
    draws = []
    for launch in range(2):
        b = _act_buffers(n, n_out, discrete, obs_dim)
        _act(lib, st, n, obs, rng, 5, b)
        torch.cuda.synchronize()
        assert rng.tolist() == [seed, launch + 1, 0]
        assert torch.equal(b["obs_buf"], obs)
        v = b["value"].cpu().numpy()
        assert (np.abs(v - v64) <= 2e-5 + 1e-6 * np.abs(v64)).all(), np.abs(v - v64).max()
        lp, lp64 = b["logp"].cpu().numpy(), logp_model(pol, out64, b["act_buf"].cpu().numpy())
        if discrete:
            a = b["act_env"].cpu().numpy()
            assert a.min() >= 0 and a.max() < n_out and np.array_equal(a, b["act_buf"].cpu().numpy())
            tol = 4e-6 + 1e-6 * np.abs(out64).max(1)
        else:
            assert torch.equal(b["act_env"], b["act_buf"].clamp(-1.0, 1.0))
            # float32 ulps of a mean move the standardised sample z = (a - mean) / sigma by ~ulp(mean) / sigma and the log-probability by z times that
            act = b["act_buf"].cpu().numpy().astype(np.float64)
            z = (act - out64) / sigma
            tol = 4e-6 + 4e-7 * (np.abs(z) * (1.0 + np.abs(act)) / sigma).sum(1)
        assert (np.abs(lp - lp64) <= tol).all(), np.abs(lp - lp64).max()
        check_draws(out64, sigma, seed, 5 + np.arange(n), launch, b["act_env"].cpu().numpy(), b["act_buf"].cpu().numpy())
        draws.append(b["act_buf"].clone())
    assert n < 8 or not torch.equal(draws[0], draws[1])                 # a new counter, new samples


def check_draws(out64, sigma, seed, envs, counter, act_env, act_buf, label=""):
    """The kernel's draws are sample_model's at this counter: the exact category except at draws within float32 rounding of a CDF boundary
    (their count is printed and must stay under 0.5 % of the draws: about (n_out - 1) x 2 x 1e-5 (1 + max |logit|) of them are expected); a
    Box sample within box_sample_bound of mean64 + sigma64 z64, and the env's action its clamp to [-1, 1].  Returns the number of near draws."""
    want, near, z = sample_model(out64, sigma, seed, envs, counter)
    if sigma is None:
        bad = (act_buf != want) & ~near
        assert not bad.any(), (label, int(bad.sum()), np.nonzero(bad)[0][:8])
        assert near.sum() <= max(2, 5e-3 * len(want)), (label, int(near.sum()))
        if near.any():
            print("  %s%d of %d draws within rounding of a CDF boundary, %d of them differ" % (label, near.sum(), len(want),
                                                                                        int((act_buf != want)[near].sum())))
    else:
        err = np.abs(act_buf.astype(np.float64) - want)
        assert (err <= box_sample_bound(out64, sigma, z)).all(), (label, err.max())
        assert np.array_equal(act_env, np.clip(act_buf, -1.0, 1.0))
    return int(near.sum())


def _unaligned_struct(pol):
    """srl_mlp_policy whose weight pointers sit in one flat buffer at float offsets = 1 (mod 4): no 16-byte loads of the weights."""
    from srl_sim.policy import SrlMlpPolicy, policy_struct
    st, tensors = policy_struct(pol)
    names = ["pi_w1", "pi_b1", "pi_w2", "pi_b2", "pi_w3", "pi_b3", "vf_w1", "vf_b1", "vf_w2", "vf_b2", "vf_w3", "vf_b3"]
    if not pol.discrete:
        names.append("logstd"); tensors = tensors + [pol.logstd.detach()]
    flat = torch.zeros(sum(t.numel() for t in tensors) + 4 * len(tensors) + 4, device="cuda")
    u = SrlMlpPolicy()
    u.struct_size, u.obs_dim, u.n_out, u.discrete = st.struct_size, st.obs_dim, st.n_out, st.discrete
    off = 1
    for name, t in zip(names, tensors):
        flat[off:off + t.numel()].copy_(t.detach().reshape(-1))
        setattr(u, name, flat.data_ptr() + 4 * off)
        off += t.numel()
        off += (1 - off) % 4
    assert all(getattr(u, name) % 16 == 4 for name in names)
    return u, flat


@pytest.mark.parametrize("discrete,obs_dim,n_out", [(True, 3, 6), (True, 1, 2), (False, 3, 7), (False, 1, 1)])
def test_policy_act_unaligned_weights_give_the_same_bytes(lib, discrete, obs_dim, n_out):
    from srl_sim.policy import policy_struct
    pol = _policy(obs_dim, discrete, n_out, seed=8).cuda()
    st, keep = policy_struct(pol)
    ust, flat = _unaligned_struct(pol)
    n = 1000
    obs = torch.randn((n, obs_dim), device="cuda") * 1.5
    res = []
    for s in (st, ust):
        rng = torch.tensor([77, 3, 0], dtype=torch.int64, device="cuda")
        b = _act_buffers(n, n_out, discrete, obs_dim)
        _act(lib, s, n, obs, rng, 0, b)
        torch.cuda.synchronize()
        res.append(b)
    for k in res[0]:
        assert torch.equal(res[0][k], res[1][k]), k


@pytest.mark.parametrize("discrete,obs_dim,n_out", [(True, 3, 6), (False, 3, 7), (False, 1, 1)])
def test_policy_act_sharded_over_two_launches_gives_the_same_bytes(lib, discrete, obs_dim, n_out):
    """A sample depends only on (seed, env_offset + i, counter): envs [0, k) and [k, n) in two launches with env_offset = k for the second
    (k odd, inside a CTA's 32 envs) equal one launch over [0, n) -- what the data-parallel trainer's env_offset = rank * num_envs relies on."""
    from srl_sim.policy import policy_struct
    pol = _policy(obs_dim, discrete, n_out, seed=9).cuda()
    st, keep = policy_struct(pol)
    n, k = 1000, 333
    obs = torch.randn((n, obs_dim), device="cuda") * 1.5
    one, two = _act_buffers(n, n_out, discrete, obs_dim), _act_buffers(n, n_out, discrete, obs_dim)
    rng = torch.tensor([55, 4, 0], dtype=torch.int64, device="cuda")
    _act(lib, st, n, obs, rng, 0, one)
    rng.copy_(torch.tensor([55, 4, 0]))
    _act(lib, st, k, obs, rng, 0, two)
    rng.copy_(torch.tensor([55, 4, 0]))
    _act(lib, st, n - k, obs, rng, k, two, first=k)
    torch.cuda.synchronize()
    assert rng.tolist() == [55, 5, 0]
    for key in one:
        assert torch.equal(one[key], two[key]), key


# ---------------------------------------------------------------- srl_ppo2_gae

@pytest.mark.parametrize("N", [1, 127, 129, 4096])
@pytest.mark.parametrize("T", [1, 7, 8, 9, 129])
def test_gae_matches_the_trainer_recursion_bit_for_bit(lib, T, N):
    """srl_ppo2_gae equals rl_baselines.ppo2's float32 torch recursion bit for bit (the trainer's gamma / lam and a pair whose float32
    product differs from the rounded double product), and the float64 recursion to a few float32 ulps of the result's scale."""
    rew, val, done, last_val = gae_rollout(T, N, "cuda", seed=T * 10007 + N)
    for gamma, lam in ((0.99, 0.95), (0.9, 0.9)):
        adv, ret = torch.full_like(rew, float("nan")), torch.full_like(rew, float("nan"))
        rc = lib.lib.srl_ppo2_gae(T, N, rew.data_ptr(), val.data_ptr(), done.data_ptr(), last_val.data_ptr(), gamma, lam, adv.data_ptr(), ret.data_ptr(),
                                  _stream())
        lib.check(rc, "srl_ppo2_gae")
        t_adv, t_ret = gae_torch(rew, val, done, last_val, gamma, lam)
        torch.cuda.synchronize()
        diff = int((adv != t_adv).sum()) + int((ret != t_ret).sum())
        assert torch.equal(adv, t_adv) and torch.equal(ret, t_ret), (gamma, lam, diff, float((adv - t_adv).abs().max()))
        a64, r64 = gae_model(*(a.cpu().numpy() for a in (rew, val, done, last_val)), gamma, lam)
        for got, want in ((adv, a64), (ret, r64)):
            assert np.abs(got.cpu().numpy() - want).max() <= GAE_ULPS * 2.0 ** -23 * np.abs(want).max()
