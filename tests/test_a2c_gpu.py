"""
GPU tests of the A2C path (include/srl_policy.h, rl_baselines/a2c.py):
  srl_a2c_grad      -- float64 autograd of rl_baselines.a2c.a2c_loss at every registry shape and the wide widths, with the tolerance rule of
                       tests/test_consumer_kernels_gpu.py, byte-identical on a second call, and shown to see a missing row;
  srl_clip_rmsprop  -- the float64 TF model of tests/a2c_numpy_ref.py over 100 steps, clipped and unclipped, byte-identical when repeated;
  srl_ppo2_gae      -- with lambda = 1, the A2C runner's discount_with_dones returns;
  the trainer       -- learns MobileRobot, gives the same parameters captured and eager, and runs from the entry point for every env id.
"""
import copy

import numpy as np
import pytest
import torch

from a2c_numpy_ref import a2c_returns_model, clip_rmsprop_model
from test_consumer_reference_cpu import GAE_ULPS, gae_rollout, grad_bound, grad_errors, ppo2_policy, ppo2_rollout

pytestmark = pytest.mark.gpu

CH = 64
ENT_COEF, VF_COEF = 0.01, 0.5
# the seven registry shapes (tests/test_consumer_kernels_gpu.py) and two stacked widths of the wide kernel
A2C_SHAPES = [(True, 3, 6), (True, 2, 4), (True, 1, 2), (False, 3, 3), (False, 3, 7), (False, 2, 2), (False, 1, 2), (True, 12, 6), (False, 32, 2)]
A2C_SIZES = ["1", "33", "3_chunks_per_cta", "20480"]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _a2c_grads(pol, idx, d, rows=None):
    from rl_baselines.a2c import a2c_loss
    pol = copy.deepcopy(pol)
    dt = next(pol.parameters()).dtype
    cast = lambda t: t if t.dtype == torch.int64 else t.to(dt)
    sel = idx if rows is None else idx[:rows]
    a2c_loss(pol, *(cast(d[k])[sel] for k in ("obs", "act", "ret", "old_val")), ENT_COEF, VF_COEF).backward()
    return [p.grad.detach().clone() for p in pol.parameters()]


@pytest.mark.parametrize("use_idx", [True, False], ids=["idx", "no_idx"])
@pytest.mark.parametrize("size", A2C_SIZES)
@pytest.mark.parametrize("discrete,obs_dim,n_out", A2C_SHAPES)
def test_a2c_grad_matches_float64_autograd(cuda_lib, discrete, obs_dim, n_out, size, use_idx):
    from srl_sim.policy import FusedA2CGrad
    B = _sms() * CH * 3 + 17 if size == "3_chunks_per_cta" else int(size)
    rows = B + B // 3 + 1 if use_idx else B + 5
    pol = ppo2_policy(obs_dim, discrete, n_out, "cuda")
    d = ppo2_rollout(pol, rows, seed=B + obs_dim)
    g = torch.Generator(device="cuda").manual_seed(12)
    idx = torch.randperm(rows, device="cuda", generator=g)[:B].contiguous() if use_idx else None
    ref_idx = idx if use_idx else torch.arange(B, device="cuda")
    pol64 = copy.deepcopy(pol).double()
    want = _a2c_grads(pol64, ref_idx, d)
    f32 = grad_errors(_a2c_grads(pol, ref_idx, d), want)
    fused = FusedA2CGrad(cuda_lib, pol, B)
    params = list(pol.parameters())
    fused(idx, d["obs"], d["act"], d["ret"], d["old_val"], ENT_COEF, VF_COEF, stream=_stream())
    torch.cuda.synchronize()
    got = [p.grad.detach().clone() for p in params]
    kern = grad_errors(got, want)
    names = [n for n, _ in pol.named_parameters()]
    print("\na2c_grad %s B=%d %s  max|g - g64| / max|g64|  kernel | float32 autograd:" % ((discrete, obs_dim, n_out), B, "idx" if use_idx else "no idx"))
    print("  " + "  ".join("%s %.1e|%.1e" % (n, e / s, e32 / s) for n, (e, s), (e32, _) in zip(names, kern, f32)))
    for n, (err, scale), (e32, _) in zip(names, kern, f32):
        assert scale > 0 and err <= grad_bound(scale) + 4.0 * e32, (n, err, e32, scale)
    if size == "20480":
        fused(idx, d["obs"], d["act"], d["ret"], d["old_val"], ENT_COEF, VF_COEF, stream=_stream())
        torch.cuda.synchronize()
        assert all(torch.equal(p.grad, a) for p, a in zip(params, got))
    if size == "33":
        wrong = grad_errors(got, _a2c_grads(pol64, ref_idx, d, rows=B - 1))
        margin = max(err / grad_bound(scale) for err, scale in wrong)
        print("  without the last row the float64 reference is %.0f x the tolerance away from the kernel" % margin)
        assert margin > 10.0


@pytest.mark.parametrize("max_grad_norm", [0.5, 1e3], ids=["clipped", "unclipped"])
@pytest.mark.parametrize("discrete,obs_dim,n_out", [(True, 3, 6), (False, 3, 7), (False, 32, 2)])
def test_clip_rmsprop_matches_the_float64_tf_model(cuda_lib, discrete, obs_dim, n_out, max_grad_norm):
    """100 steps from ms = 1 on fresh random gradients; then the same 100 steps again from the same start give the same bytes."""
    from srl_sim.policy import FusedClipRMSprop, policy_params
    alpha, eps, lr = 0.99, 1e-5, 7e-4
    pol = ppo2_policy(obs_dim, discrete, n_out, "cuda")
    params = policy_params(pol)
    for p in params:
        p.grad = torch.zeros_like(p)
    start = [p.detach().clone() for p in params]
    runs = []
    for rep in range(2):
        with torch.no_grad():
            for p, s in zip(params, start):
                p.copy_(s)
        opt = FusedClipRMSprop(cuda_lib, pol, max_grad_norm, alpha, eps)
        opt.lr.fill_(lr)
        p64, m64 = [s.double().cpu().numpy() for s in start], [np.ones(s.shape) for s in start]
        g = torch.Generator(device="cuda").manual_seed(21)
        for step in range(100):
            for p in params:
                p.grad.copy_(torch.randn(p.shape, device="cuda", generator=g) * 0.05)
            norm = float(torch.sqrt(sum((p.grad.double() ** 2).sum() for p in params)))
            assert (norm > max_grad_norm) == (max_grad_norm == 0.5)
            if rep == 0:
                p64, m64 = clip_rmsprop_model(p64, [p.grad.cpu().numpy() for p in params], m64, float(np.float32(lr)), max_grad_norm,
                                              float(np.float32(alpha)), float(np.float32(eps)))
            opt(stream=_stream())
        torch.cuda.synchronize()
        runs.append([p.detach().clone() for p in params] + [m.clone() for m in opt.ms])
        if rep == 0:
            for p, w, m, mw in zip(params, p64, opt.ms, m64):
                assert np.abs(m.double().cpu().numpy() - mw).max() <= 100 * 2.0 ** -24 * np.abs(mw).max()
                assert np.abs(p.detach().double().cpu().numpy() - w).max() <= 100 * 2.0 ** -23 * (np.abs(w).max() + 1.0)
            assert max(float((p.detach() - s).abs().max()) for p, s in zip(params, start)) > 1e-4     # the steps moved the parameters
    assert all(torch.equal(a, b) for a, b in zip(*runs))


@pytest.mark.parametrize("bad", [float("inf"), float("nan")], ids=["inf", "nan"])
def test_clip_rmsprop_non_finite_gradient_makes_every_parameter_nan(cuda_lib, bad):
    """tf.clip_by_global_norm's scale is NaN for a non-finite norm: one bad entry in one tensor reaches every tensor, as in the torch statement."""
    from rl_baselines.a2c import clip_rmsprop
    from srl_sim.policy import FusedClipRMSprop, policy_params
    pol = ppo2_policy(3, False, 2, "cuda")
    params = policy_params(pol)
    for p in params:
        p.grad = torch.randn(p.shape, device="cuda") * 0.05
    params[-1].grad[0] = bad
    ref = copy.deepcopy(pol)
    for p, q in zip(params, policy_params(ref)):
        q.grad = p.grad.clone()
    opt = FusedClipRMSprop(cuda_lib, pol, 0.5, 0.99, 1e-5)
    opt.lr.fill_(7e-4)
    opt(stream=_stream())
    clip_rmsprop(policy_params(ref), [torch.ones_like(p) for p in params], opt.lr[0], 0.5, 0.99, 1e-5)
    torch.cuda.synchronize()
    for p, q in zip(params, policy_params(ref)):
        assert torch.isnan(p).all() and torch.isnan(q).all()


def test_clip_rmsprop_refuses_bad_arguments(cuda_lib):
    from srl_sim._abi import SimError
    from srl_sim.policy import FusedClipRMSprop
    pol = ppo2_policy(3, True, 6, "cuda")
    for p in pol.parameters():
        p.grad = torch.zeros_like(p)
    with pytest.raises(SimError, match="max_grad_norm > 0"):
        FusedClipRMSprop(cuda_lib, pol, 0.0, 0.99, 1e-5)(stream=_stream())


@pytest.mark.parametrize("T", [1, 5, 9])
def test_gae_with_lambda_one_gives_the_a2c_returns(cuda_lib, T):
    """srl_ppo2_gae(lam = 1).ret_out equals discount_with_dones over the rewards followed by the last value, per env, in float64 -- with
    dones at the first step, the last step and mid-rollout."""
    from srl_sim.policy import bind
    bind(cuda_lib.lib)
    N = 4096
    rew, val, done, last_val = gae_rollout(T, N, "cuda", seed=T)
    assert done[0].sum() > 0 and done[T - 1].sum() > 0 and (T < 4 or done[T // 2].sum() > 0)
    adv, ret = torch.full_like(rew, float("nan")), torch.full_like(rew, float("nan"))
    rc = cuda_lib.lib.srl_ppo2_gae(T, N, rew.data_ptr(), val.data_ptr(), done.data_ptr(), last_val.data_ptr(), 0.99, 1.0, adv.data_ptr(), ret.data_ptr(),
                                   _stream())
    cuda_lib.check(rc, "srl_ppo2_gae")
    want = a2c_returns_model(*(a.cpu().numpy() for a in (rew, done, last_val)), 0.99)
    torch.cuda.synchronize()
    assert np.abs(ret.cpu().numpy() - want).max() <= GAE_ULPS * 2.0 ** -23 * np.abs(want).max()


def test_a2c_learns_mobile_robot(cuda_lib):
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.a2c import train
    hist = train("MobileRobotGymEnv-v0", 1024, 1024 * 5 * 1600, seed=0, env_kwargs=dict(is_discrete=True, shape_reward=True), verbose=0)
    rets = [h[1] for h in hist if np.isfinite(h[1])]
    print("\nA2C MobileRobot: first window %.1f, last %.1f, fps %.0f" % (rets[0], rets[-1], hist[-1][2]))
    # shaped reward = -distance per step over 251 steps: a random policy scores about -420
    assert rets[-1] > rets[0] + 60, rets[::50]


@pytest.mark.parametrize("env_id,num_stack", [("MobileRobotGymEnv-v0", 1), ("KukaButtonGymEnv-v0", 1), ("MobileRobotGymEnv-v0", 3)])
def test_captured_and_eager_updates_agree(cuda_lib, env_id, num_stack):
    """Two updates replayed from the captured graph and the same two updates launched eagerly: same parameters and RMSProp slots within float32
    rounding (the same kernels in the same order: in practice the same bytes)."""
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.a2c import train
    out = []
    for graph in (True, False):
        train(env_id, 1024, 1024 * 5 * 2, seed=5, env_kwargs=dict(is_discrete=True, shape_reward=True), verbose=0, cuda_graph=graph, num_stack=num_stack)
        out.append([p.detach().clone() for p in train.last_policy.parameters()] + [m.clone() for m in train.last_ms])
    equal = all(torch.equal(a, b) for a, b in zip(*out))
    print("\ncaptured vs eager (%s, num_stack %d): %s" % (env_id, num_stack, "identical bytes" if equal else "differ"))
    for a, b in zip(*out):
        assert float((a - b).abs().max()) <= 4 * 2.0 ** -23 * (float(b.abs().max()) + 1e-3)
    moved = train.last_policy.pi[0].weight.detach()
    assert torch.isfinite(moved).all()


@pytest.mark.parametrize("env_id", ["KukaButtonGymEnv-v0", "KukaRandButtonGymEnv-v0", "Kuka2ButtonGymEnv-v0", "KukaMovingButtonGymEnv-v0",
                                    "MobileRobotGymEnv-v0", "MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0", "MobileRobotLineTargetGymEnv-v0"])
def test_train_entry_point_runs_a2c_for_every_env(env_id, cuda_lib, tmp_path):
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.train import main
    hist = main(["--algo", "a2c", "--env", env_id, "--num-cpu", "4", "--num-timesteps", "1600", "--log-dir", str(tmp_path)])
    assert len(hist) == int(1.1 * 1600) // 20 and all(np.isfinite(h[2]) for h in hist)
