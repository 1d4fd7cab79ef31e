"""
GPU tests of stacked state observations (``--num-stack k``) on the sm_90a kernels:
  srl_obs_stack_filter -- the frame stack against numpy VecFrameStack byte for byte, the filter state against a two-pass float64 merge, the output
                          bit for bit against RunningNorm's float32 expression on the kernel's own state;
  srl_policy_act       -- the wide instantiation (widths 9..32) against a float64 model and the CPU checker's samples;
  srl_ppo2_grad        -- the wide instantiation against float64 autograd, with the tolerance rule of tests/test_consumer_kernels_gpu.py;
  width 33             -- refused by every entry point with a message that names the limit;
  the trainer          -- fused collection (stack filter) against the torch collection on the same raw observations, then a graph-captured run
                          and its replay.
"""
import copy
import ctypes
from ctypes import byref

import numpy as np
import pytest
import torch

from test_consumer_kernels_gpu import CH, _act, _act_buffers, _grad_mb, _sms, _stream, check_draws, lib  # noqa: F401  (lib: module fixture)
from test_consumer_reference_cpu import (filter_model, grad_bound, grad_errors, logp_model, normalise, policy_model, ppo2_minibatch_grads, ppo2_policy,
                                         ppo2_rollout, CLIP, ENT_COEF, VF_COEF)
from test_policy_cpu import _policy, _ref_act, ref  # noqa: F401  (ref: module fixture of the CPU checker)

pytestmark = pytest.mark.gpu

MAX_W = 32


def _stack_ref(stack, obs, done):
    """VecFrameStack.step of rl_baselines/utils.py in numpy (done None: VecFrameStack.reset)."""
    D = obs.shape[1]
    if done is None:
        stack = np.zeros_like(stack)
    else:
        stack = np.roll(stack, shift=-D, axis=-1)
        stack[done.astype(bool)] = 0
    stack[:, -D:] = obs
    return stack


# ---------------------------------------------------------------- srl_obs_stack_filter

@pytest.mark.parametrize("n", [1, 33, 4096, 50000])
@pytest.mark.parametrize("k", [1, 2, 4, "max"])
@pytest.mark.parametrize("D", [1, 2, 3])
def test_stack_filter_matches_vecframestack_and_a_float64_merge(lib, D, k, n):
    """A reset and 40 steps with ~10 % dones: the stack byte for byte, the state within float64 rounding of a two-pass merge of the stacked rows,
    the output bit for bit against RunningNorm's float32 expression on the kernel's state.  Then update=False leaves the state alone."""
    from rl_baselines.ppo2 import RunningNorm
    k = MAX_W // D if k == "max" else k
    W = k * D
    state = RunningNorm(W, torch.device("cuda", 0)).state
    model = state.cpu().numpy().copy()
    g = torch.Generator(device="cuda").manual_seed(1000 * D + 10 * k + n % 97)
    scale = torch.tensor([0.3, 2.0, 9.0][:D], device="cuda")
    offset = torch.tensor([1.0, -4.0, 0.5][:D], device="cuda")
    stack = torch.full((n, W), float("nan"), device="cuda")
    want = np.zeros((n, W), np.float32)
    for it in range(41):
        obs = (torch.randn((n, D), device="cuda", generator=g) * scale + offset + 0.05 * it).contiguous()
        done = None if it == 0 else (torch.rand(n, device="cuda", generator=g) < 0.1).to(torch.uint8)
        out = torch.full((n, W), float("nan"), device="cuda")
        rc = lib.lib.srl_obs_stack_filter(n, D, k, obs.data_ptr(), None if done is None else done.data_ptr(), stack.data_ptr(), state.data_ptr(), 1,
                                          10.0, 1e-8, out.data_ptr(), _stream())
        lib.check(rc, "srl_obs_stack_filter")
        torch.cuda.synchronize()
        want = _stack_ref(want, obs.cpu().numpy(), None if done is None else done.cpu().numpy())
        assert np.array_equal(stack.cpu().numpy().view(np.uint32), want.view(np.uint32)), it
        model = filter_model(model, want)
        s = state.cpu().numpy()
        assert np.allclose(s[:W], model[:W], rtol=0, atol=1e-11), (it, np.abs(s[:W] - model[:W]).max())
        assert np.allclose(s[W:2 * W], model[W:2 * W], rtol=1e-11, atol=1e-11), (it, np.abs(s[W:2 * W] - model[W:2 * W]).max())
        assert s[2 * W] == pytest.approx(model[2 * W], rel=1e-14)
        assert torch.equal(out, normalise(stack, state)), it
    frozen, before = state.clone(), stack.clone()
    obs = (torch.randn((n, D), device="cuda", generator=g) * scale * 40.0).contiguous()
    done = torch.zeros(n, dtype=torch.uint8, device="cuda")
    out = torch.empty((n, W), device="cuda")
    lib.check(lib.lib.srl_obs_stack_filter(n, D, k, obs.data_ptr(), done.data_ptr(), stack.data_ptr(), state.data_ptr(), 0, 10.0, 1e-8, out.data_ptr(),
                                           _stream()), "srl_obs_stack_filter")
    torch.cuda.synchronize()
    assert torch.equal(state, frozen)
    assert torch.equal(stack.cpu(), torch.from_numpy(_stack_ref(before.cpu().numpy(), obs.cpu().numpy(), done.cpu().numpy())))
    assert torch.equal(out, normalise(stack, state))


# ---------------------------------------------------------------- srl_policy_act, wide

WIDE = [9, 12, 17, 32]
WIDE_HEADS = [(True, 6), (False, 3), (False, 7)]


@pytest.mark.parametrize("n", [1, 31, 32, 33, 4096, 8192])
@pytest.mark.parametrize("discrete,n_out", WIDE_HEADS)
@pytest.mark.parametrize("obs_dim", WIDE)
def test_wide_policy_act_against_float64_and_the_checker(lib, ref, obs_dim, discrete, n_out, n):  # noqa: F811
    """Value and log-probability of the drawn action against the float64 towers (the tolerances of test_consumer_kernels_gpu.py), the draws
    against sample_model, the rollout copy of the observations, the counter; the samples against the CPU checker's (an ulp of expf / tanhf may
    move a CDF boundary)."""
    from srl_sim.policy import policy_struct
    pol = _policy(obs_dim, discrete, n_out, seed=500 + obs_dim * 9 + n_out).cuda()
    st, keep = policy_struct(pol)
    seed = 77 + n
    rng = torch.tensor([seed, 0, 0], dtype=torch.int64, device="cuda")
    obs = (torch.randn((n, obs_dim), device="cuda", generator=torch.Generator(device="cuda").manual_seed(n + obs_dim)) * 1.5).contiguous()
    out64, v64 = policy_model(pol, obs.cpu().numpy())
    sigma = None if discrete else np.exp(pol.logstd.detach().cpu().double().numpy())
    b = _act_buffers(n, n_out, discrete, obs_dim)
    _act(lib, st, n, obs, rng, 3, b)
    torch.cuda.synchronize()
    assert rng.tolist() == [seed, 1, 0]
    assert torch.equal(b["obs_buf"], obs)
    v = b["value"].cpu().numpy()
    assert (np.abs(v - v64) <= 2e-5 + 1e-6 * np.abs(v64)).all(), np.abs(v - v64).max()
    lp, lp64 = b["logp"].cpu().numpy(), logp_model(pol, out64, b["act_buf"].cpu().numpy())
    pol_cpu = copy.deepcopy(pol).cpu()
    r_env, r_buf, r_logp, r_val, _ = _ref_act(ref, pol_cpu, obs.cpu(), seed=seed, counter=0, env_offset=3)
    if discrete:
        a = b["act_env"].cpu().numpy()
        assert a.min() >= 0 and a.max() < n_out and np.array_equal(a, b["act_buf"].cpu().numpy())
        assert (a == r_env).mean() > 0.999
        tol = 4e-6 + 1e-6 * np.abs(out64).max(1)
    else:
        assert torch.equal(b["act_env"], b["act_buf"].clamp(-1.0, 1.0))
        assert (np.abs(b["act_buf"].cpu().numpy() - r_buf) <= 1e-4 + 1e-5 * np.abs(r_buf)).all()
        act = b["act_buf"].cpu().numpy().astype(np.float64)
        z = (act - out64) / sigma
        tol = 4e-6 + 4e-7 * (np.abs(z) * (1.0 + np.abs(act)) / sigma).sum(1)
    assert (np.abs(lp - lp64) <= tol).all(), np.abs(lp - lp64).max()
    check_draws(out64, sigma, seed, 3 + np.arange(n), 0, b["act_env"].cpu().numpy(), b["act_buf"].cpu().numpy())


# ---------------------------------------------------------------- srl_ppo2_grad, wide

@pytest.mark.parametrize("use_idx", [True, False], ids=["idx", "no_idx"])
@pytest.mark.parametrize("size", ["3_chunks_per_cta", "131072", "200003"])
@pytest.mark.parametrize("discrete,n_out", [(True, 6), (False, 3)])
@pytest.mark.parametrize("obs_dim", [12, 32])
def test_wide_ppo2_grad_matches_float64_autograd(lib, obs_dim, discrete, n_out, size, use_idx):
    """Every gradient within 2e-4 of its tensor's largest entry (+ 2e-6) plus 4x float32 autograd's own error, as for the narrow kernel; a
    second call gives the same bytes."""
    from srl_sim.policy import FusedPPO2Grad
    mb = _grad_mb(size)
    rows = mb + mb // 3 if use_idx else mb + 5
    pol = ppo2_policy(obs_dim, discrete, n_out, "cuda")
    d = ppo2_rollout(pol, rows, seed=mb + obs_dim)
    g = torch.Generator(device="cuda").manual_seed(12)
    idx = torch.randperm(rows, device="cuda", generator=g)[:mb].contiguous() if use_idx else None
    ref_idx = idx if use_idx else torch.arange(mb, device="cuda")
    want = ppo2_minibatch_grads(copy.deepcopy(pol).double(), ref_idx, d)
    f32 = grad_errors(ppo2_minibatch_grads(pol, ref_idx, d), want)
    fused = FusedPPO2Grad(lib, pol, mb)
    fused(idx, d["obs"], d["act"], d["adv"], d["ret"], d["old_logp"], d["old_val"], CLIP, ENT_COEF, VF_COEF, stream=_stream())
    torch.cuda.synchronize()
    got = [p.grad.detach().clone() for p in pol.parameters()]
    names = [nm for nm, _ in pol.named_parameters()]
    kern = grad_errors(got, want)
    print("\nppo2_grad wide %s mb=%d: " % ((obs_dim, discrete, n_out), mb) + "  ".join("%s %.1e|%.1e" % (nm, e / s, e32 / s)
                                                                                       for nm, (e, s), (e32, _) in zip(names, kern, f32)))
    for nm, (err, scale), (e32, _) in zip(names, kern, f32):
        assert scale > 0 and err <= grad_bound(scale) + 4.0 * e32, (nm, err, e32, scale)
    fused(idx, d["obs"], d["act"], d["adv"], d["ret"], d["old_logp"], d["old_val"], CLIP, ENT_COEF, VF_COEF, stream=_stream())
    torch.cuda.synchronize()
    assert all(torch.equal(p.grad, a) for p, a in zip(pol.parameters(), got))


# ---------------------------------------------------------------- width 33

def test_width_33_is_refused_with_the_limit(lib):
    from srl_sim.policy import policy_struct, SrlMlpGrads
    pol = _policy(32, True, 6, seed=1).cuda()
    st, keep = policy_struct(pol)
    st.obs_dim = 33
    b = _act_buffers(4, 6, True, 33)
    obs = torch.zeros((4, 33), device="cuda")
    rng = torch.zeros(3, dtype=torch.int64, device="cuda")
    rc = lib.lib.srl_policy_act(byref(st), 4, obs.data_ptr(), rng.data_ptr(), 0, None, b["act_env"].data_ptr(), None, b["logp"].data_ptr(),
                                b["value"].data_ptr(), _stream())
    assert rc != 0 and "1..32" in lib.last_error()
    assert lib.lib.srl_ppo2_workspace_bytes(33, 6, 1, 1024) == 0 and "1..32" in lib.last_error()
    gr = SrlMlpGrads()
    gr.struct_size = ctypes.sizeof(SrlMlpGrads)
    for name in ("pi_w1", "pi_b1", "pi_w2", "pi_b2", "pi_w3", "pi_b3", "vf_w1", "vf_b1", "vf_w2", "vf_b2", "vf_w3", "vf_b3"):
        setattr(gr, name, obs.data_ptr())
    rc = lib.lib.srl_ppo2_grad(byref(st), byref(gr), 4, None, obs.data_ptr(), obs.data_ptr(), obs.data_ptr(), obs.data_ptr(), obs.data_ptr(),
                               obs.data_ptr(), 0.2, 0.01, 0.5, obs.data_ptr(), obs.numel() * 4, _stream())
    assert rc != 0 and "1..32" in lib.last_error()
    state = torch.zeros(2 * 33 + 1, dtype=torch.float64, device="cuda")
    rc = lib.lib.srl_obs_stack_filter(4, 3, 11, obs.data_ptr(), None, obs.data_ptr(), state.data_ptr(), 1, 10.0, 1e-8, obs.data_ptr(), _stream())
    assert rc != 0 and "1..32" in lib.last_error()
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        policy_struct(_policy(33, True, 6, seed=1))


# ---------------------------------------------------------------- the trainer

def test_trainer_fused_stack_collection_matches_torch_and_the_captured_run_replays(cuda_lib, monkeypatch, tmp_path):
    """KukaButton (50-step episodes), N = 256, k = 4, two updates with the fused paths and no graph: the rows the policy kernel got are the torch collection's
    (roll / zero / insert + RunningNorm) on the same raw observations and dones.  Then a graph-captured run completes and its model replays."""
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines import ppo2
    from rl_baselines.ppo2 import RunningNorm
    from srl_sim.policy import FusedPolicy
    fed, raw, rows0 = [], [], []
    act, sf, filt = FusedPolicy.act, FusedPolicy.stack_filter, RunningNorm.__call__

    def act_rec(self, n, obs, *a, **kw):
        fed.append(obs.clone())
        return act(self, n, obs, *a, **kw)

    def sf_rec(self, n, obs_raw, done, stack, out, update=True, stream=None):
        if update:
            raw.append((obs_raw.clone(), done.clone()))
        return sf(self, n, obs_raw, done, stack, out, update, stream)

    def filt_rec(self, x, update=True):
        if update:
            rows0.append(x.clone())
        return filt(self, x, update)
    monkeypatch.setattr(FusedPolicy, "act", act_rec)
    monkeypatch.setattr(FusedPolicy, "stack_filter", sf_rec)
    monkeypatch.setattr(RunningNorm, "__call__", filt_rec)
    N, T, K = 256, 128, 4
    hist = ppo2.train("KukaButtonGymEnv-v0", N, N * T * 2, seed=4, env_kwargs=dict(max_steps=50), verbose=0, cuda_graph=False, num_stack=K)
    assert len(hist) == 2 and len(fed) == 2 * T and len(raw) == 2 * T and len(rows0) == 1
    D = raw[0][0].shape[1]
    norm = RunningNorm(K * D, torch.device("cuda", 0))
    stack = rows0[0].clone()
    assert (stack[:, :-D] == 0).all()
    worst = 0.0
    for t in range(2 * T):
        obs = norm(stack)
        worst = max(worst, float((obs - fed[t]).abs().max()))
        o, d = raw[t]
        stack = torch.where(d.bool()[:, None], 0.0, torch.roll(stack, -D, 1))
        stack[:, -D:] = o
    assert sum(int(d.sum()) for _, d in raw) > 0
    print("\nfused vs torch collection, k=%d: max |difference| %.2e" % (K, worst))
    assert worst <= 1e-5
    monkeypatch.undo()
    hist = ppo2.train("KukaButtonGymEnv-v0", N, N * T * 2, seed=4, verbose=0, num_stack=K, log_dir=str(tmp_path))
    assert len(hist) == 2 and all(np.isfinite(h[2]) for h in hist)
    from replay.enjoy_baselines import main
    n_done, mean_reward = main(["--log-dir", str(tmp_path), "--num-cpu", "16", "--num-timesteps", "1100"])
    assert n_done >= 16 and np.isfinite(mean_reward)
