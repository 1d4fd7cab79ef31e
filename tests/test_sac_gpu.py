"""
SAC kernels (include/srl_policy.h: srl_sac_*) on the GPU against float64 models: the policy step and its Philox draws, the per-sample half of
a gradient step, the weight gradients (tolerance rule of tests/test_consumer_reference_cpu.py), Adam + Polyak, and the fused trainer
(captured and eager runs give the same bytes; every registry id through the entry point; an oversized ring is refused before allocating;
learning MobileRobot with shaped reward).
"""
import math

import numpy as np
import pytest
import torch

from sac_numpy_ref import adam_polyak_model, forward, layout, sac_step_model, unpack
from test_consumer_reference_cpu import grad_bound, philox_words, u53

pytestmark = pytest.mark.gpu


def _nets(W, A, seed):
    from rl_baselines.sac import SACNets
    torch.manual_seed(seed)
    nets = SACNets(W, A)
    with torch.no_grad():
        nets.arena.add_(0.05 * torch.randn_like(nets.arena))      # biases too: some ReLU units off for most rows, some on
        nets.arena[-1] = -0.4
        # the actor's samples stay away from tanh's saturation, where float32 (the kernel's and the TF graph's alike) loses
        # log(1 - a^2 + 1e-6): 1 - a^2 is then below float32's resolution near 1 (test_sac_cpu.py covers saturation in float64)
        (w3, _), (b3, _) = nets.layout["actor"]["w3"], nets.layout["actor"]["b3"]
        nets.arena[w3:w3 + A * 64] *= 0.5
        nets.arena[w3 + A * 64:w3 + 2 * A * 64] *= 0.1
        nets.arena[b3 + A:b3 + 2 * A] = -1.5
        nets.target.copy_(nets.target + 0.01 * torch.randn_like(nets.target))
    return nets.cuda()


def _gauss(seed, streams, counter, purpose0, A):
    """Box-Muller of srl_sample_gaussian's word use in float64: [len(streams), A]."""
    z = np.zeros((len(streams), A))
    for k in range(A):
        w = philox_words(seed, streams, counter, purpose0 + k // 4).astype(np.float64)
        j = k & 2
        u1, u2 = (np.floor(w[:, j] / 256.0) + 0.5) / 16777216.0, (np.floor(w[:, j + 1] / 256.0) + 0.5) / 16777216.0
        rad, ang = np.sqrt(-2.0 * np.log(u1)), 2 * math.pi * u2
        z[:, k] = rad * np.sin(ang) if k & 1 else rad * np.cos(ang)
    return z


@pytest.mark.parametrize("W,A,n", [(3, 3, 4096), (2, 2, 1000), (32, 7, 300), (1, 8, 77)])
def test_sac_act_modes_against_float64_and_philox(cuda_lib, W, A, n):
    from srl_sim.policy import FusedSACAct
    nets = _nets(W, A, W + A)
    obs = torch.randn(n, W, device="cuda")
    act = torch.zeros(n, A, device="cuda")
    f = FusedSACAct(cuda_lib, nets, seed=11, env_offset=5)
    out64, _ = forward(unpack(nets.arena.detach().cpu().numpy(), 0, W, 2 * A), obs.cpu().double().numpy())
    mu, ls = out64[:, :A], np.clip(out64[:, A:], -20, 2)
    f(n, obs, act, mode=FusedSACAct.DETERMINISTIC)
    np.testing.assert_allclose(act.cpu().double().numpy(), np.tanh(mu), atol=2e-5)
    f(n, obs, act, mode=FusedSACAct.SAMPLE)                            # counter 1
    z = _gauss(11, np.arange(n) + 5, 1, 26, A)
    np.testing.assert_allclose(act.cpu().double().numpy(), np.tanh(mu + np.exp(ls) * z), atol=5e-5)
    f(n, obs, act, mode=FusedSACAct.RANDOM)                            # counter 2
    want = np.zeros((n, A))
    for k in range(A):
        w = philox_words(11, np.arange(n) + 5, 2, 28 + k // 4)[:, k % 4].astype(np.float64)
        want[:, k] = 2 * (np.floor(w / 256.0) / 16777216.0) - 1
    np.testing.assert_array_equal(act.cpu().double().numpy(), want)
    assert int(f.rng[1]) == 3
    # sharded launches: two halves with env_offset give the bytes of one launch
    g = FusedSACAct(cuda_lib, nets, seed=11, env_offset=5)
    one = torch.zeros_like(act); g(n, obs, one)
    h = n // 2
    a0 = FusedSACAct(cuda_lib, nets, seed=11, env_offset=5); a1 = FusedSACAct(cuda_lib, nets, seed=11, env_offset=5 + h)
    p0, p1 = torch.zeros(h, A, device="cuda"), torch.zeros(n - h, A, device="cuda")
    a0(h, obs[:h].contiguous(), p0); a1(n - h, obs[h:].contiguous(), p1)
    assert torch.equal(torch.cat([p0, p1]), one)


def test_sac_act_random_mode_is_uniform(cuda_lib):
    from scipy.stats import chisquare
    from srl_sim.policy import FusedSACAct
    nets = _nets(3, 3, 0)
    n = 1 << 16
    act = torch.zeros(n, 3, device="cuda")
    FusedSACAct(cuda_lib, nets, seed=2)(n, None, act, mode=FusedSACAct.RANDOM)
    a = act.cpu().numpy()
    assert a.min() >= -1.0 and a.max() < 1.0
    for k in range(3):
        counts, _ = np.histogram(a[:, k], bins=32, range=(-1, 1))
        assert chisquare(counts).pvalue > 1e-4


def _ring(rows, n, W, A, stored, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    ring = dict(obs=r(rows, n, W), next_obs=r(rows, n, W), act=torch.tanh(r(rows, n, A)), rew=r(rows, n),
                done=(torch.rand(rows, n, generator=g) < 0.1).to(torch.uint8))
    ring = {k: v.cuda() for k, v in ring.items()}
    step = torch.tensor([stored, 0], dtype=torch.int64, device="cuda")
    return ring, step


def _prepare_and_grad(cuda_lib, nets, ring, step, B, seed, ent_coef):
    from srl_sim.policy import FusedSACGrad, FusedSACPrepare
    grad = torch.full_like(nets.arena.detach(), float("nan"))
    ws = FusedSACGrad.workspace(cuda_lib, nets, B)
    prep = FusedSACPrepare(cuda_lib, nets, ring, B, seed, grad, ws)
    prep(step, 0.99, ent_coef, -float(nets.act_dim))
    FusedSACGrad(cuda_lib, nets)(prep, grad)
    torch.cuda.synchronize()
    return prep, grad


def _model(nets, ring, prep, seed, ent_coef):
    W, A, B = nets.obs_dim, nets.act_dim, prep.batch
    flat = {k: v.reshape((-1,) + v.shape[2:]).cpu().numpy() for k, v in ring.items()}
    ix = prep.idx.cpu().numpy()
    eps = _gauss(seed, np.arange(B), 0, 31, A)
    return sac_step_model(nets.arena.detach().cpu().numpy(), nets.target.cpu().numpy(), W, A, flat["obs"][ix], flat["act"][ix], flat["rew"][ix],
                          flat["next_obs"][ix], flat["done"][ix].astype(np.float64), eps, 0.99, ent_coef, -float(A))


@pytest.mark.parametrize("W,A,B,ent_coef", [(3, 3, 1, None), (3, 3, 33, None), (3, 7, 64 * 132 * 3 + 5, None), (2, 2, 4000, 0.1), (1, 2, 999, None),
                                            (32, 7, 3000, None), (3, 3, 262144, None)])
def test_sac_prepare_and_grad_against_float64(cuda_lib, W, A, B, ent_coef):
    rows, n, stored = 50, 64, 37
    nets = _nets(W, A, 7 * W + A)
    ring, step = _ring(rows, n, W, A, stored, W * A)
    prep, grad = _prepare_and_grad(cuda_lib, nets, ring, step, B, 9, ent_coef)
    size = stored * n
    want_idx = np.minimum(np.floor(u53(philox_words(9, np.arange(B), 0, 30)) * size), size - 1).astype(np.int64)
    np.testing.assert_array_equal(prep.idx.cpu().numpy(), want_idx)
    assert int(prep.rng[1]) == 1 and int(prep.rng[2]) == 0
    want, ref = _model(nets, ring, prep, 9, ent_coef)
    for k in ("q_backup", "v_backup", "logp"):
        got = getattr(prep, k).cpu().double().numpy()
        assert np.abs(got - ref[k]).max() <= 2e-4 * (1 + np.abs(ref[k]).max()), k
    d = prep.d_actor.cpu().double().numpy()
    assert np.abs(d - ref["d_actor"]).max() <= grad_bound(np.abs(ref["d_actor"]).max())
    g = grad.cpu().double().numpy()
    worst = 0.0
    for name, lo, hi in _tensors(W, A):
        err, scale = np.abs(g[lo:hi] - want[lo:hi]).max(), np.abs(want[lo:hi]).max()
        worst = max(worst, err / grad_bound(scale))
        assert err <= grad_bound(scale), (name, lo, err, scale)
    print("\nB=%d: largest error / grad_bound over the tensors %.3f" % (B, worst))
    assert abs(g[-1] - want[-1]) <= 1e-5 * (1 + abs(want[-1]))
    # the same bytes twice (the prepare counter rewound)
    prep.rng[1] = 0
    first = grad.clone()
    prep(step, 0.99, ent_coef, -float(A))
    from srl_sim.policy import FusedSACGrad
    FusedSACGrad(cuda_lib, nets)(prep, grad)
    assert torch.equal(grad, first)


def _tensors(W, A):
    """(network, first, end) of each of the 24 gradient tensors in the arena."""
    nets_lay, _ = layout(W, A)
    out = []
    for name, (off, n_in, n_out) in nets_lay.items():
        for size in (64 * n_in, 64, 64 * 64, 64, 64 * n_out, n_out):
            out.append((name, off, off + size))
            off += size
    return out


@pytest.mark.parametrize("B,drop", [(130, (129, 130)), (64 * 132 * 3 + 5, (64 * 200, 64 * 201))])
def test_sac_grad_leave_rows_out(cuda_lib, B, drop):
    """A control: the model without one sample (B = 130) or without one 64-sample chunk in the middle of a several-chunks-per-CTA batch
    differs from the kernel beyond the bound the comparison above holds it to, in some tensor of every network: a kernel that skipped those
    rows would fail it."""
    W, A = 3, 3
    nets = _nets(W, A, 3)
    ring, step = _ring(20, 16, W, A, 20, 1)
    prep, grad = _prepare_and_grad(cuda_lib, nets, ring, step, B, 4, None)
    want, _ = _model(nets, ring, prep, 4, None)
    g = grad.cpu().double().numpy()
    flat = {k: v.reshape((-1,) + v.shape[2:]).cpu().numpy() for k, v in ring.items()}
    keep = np.ones(B, bool)
    keep[drop[0]:drop[1]] = False
    ix = prep.idx.cpu().numpy()[keep]
    eps = _gauss(4, np.arange(B), 0, 31, A)[keep]
    short, _ = sac_step_model(nets.arena.detach().cpu().numpy(), nets.target.cpu().numpy(), W, A, flat["obs"][ix], flat["act"][ix], flat["rew"][ix],
                              flat["next_obs"][ix], flat["done"][ix].astype(np.float64), eps, 0.99, None, -3.0)
    short *= keep.sum() / B                                   # the same 1 / B per sample as the full batch
    missed = {}
    for name, lo, hi in _tensors(W, A):
        bound = grad_bound(np.abs(want[lo:hi]).max())
        assert np.abs(g[lo:hi] - want[lo:hi]).max() <= bound, (name, lo)
        missed[name] = missed.get(name, False) or np.abs(g[lo:hi] - short[lo:hi]).max() > bound
    assert all(missed.values()), missed


def test_sac_adam_against_the_float64_tf_model(cuda_lib):
    from srl_sim.policy import FusedSACAdam
    W, A = 3, 3
    nets = _nets(W, A, 5)
    a0, t0 = nets.arena.detach().cpu().numpy().copy(), nets.target.cpu().numpy().copy()
    opt = FusedSACAdam(cuda_lib, nets, tau=0.005)
    opt.lr.fill_(3e-4)
    g = torch.Generator().manual_seed(0)
    grads = [torch.randn(nets.arena.numel(), generator=g).cuda() * (0.1 + k % 5) for k in range(50)]
    for gr in grads:
        opt(gr)
    w, tg, m, v = adam_polyak_model(a0, t0, [x.cpu().numpy() for x in grads], W, A, 3e-4, 0.005)
    assert np.abs(nets.arena.detach().cpu().numpy() - w).max() < 1e-4 * 3e-4 * 50
    assert np.abs(nets.target.cpu().numpy() - tg).max() < 1e-4 * 3e-4 * 50
    np.testing.assert_allclose(opt.m.cpu().numpy(), m, rtol=1e-4, atol=1e-6)
    # the same bytes twice, and the torch statement's bytes
    from rl_baselines.sac import adam_polyak
    state = [x.clone() for x in (nets.arena.detach(), nets.target, opt.m, opt.v, opt.beta_power)]
    opt(grads[0])
    after = [x.clone() for x in (nets.arena.detach(), nets.target, opt.m, opt.v, opt.beta_power)]
    for x, s in zip((nets.arena.data, nets.target, opt.m, opt.v, opt.beta_power), state):
        x.copy_(s)
    opt(grads[0])
    for x, s in zip((nets.arena.detach(), nets.target, opt.m, opt.v, opt.beta_power), after):
        assert torch.equal(x, s)
    for x, s in zip((nets.arena.data, nets.target, opt.m, opt.v, opt.beta_power), state):
        x.copy_(s)
    adam_polyak(nets, grads[0], opt.m, opt.v, opt.beta_power, 3e-4, 0.005, polyak=True)
    assert torch.equal(nets.arena.detach(), after[0]) and torch.equal(nets.target, after[1])


@pytest.mark.parametrize("env_id,stack,hp", [("MobileRobotGymEnv-v0", 1, {}), ("KukaButtonGymEnv-v0", 1, {}), ("KukaButtonGymEnv-v0", 3, {}),
                                             ("MobileRobotGymEnv-v0", 1, dict(train_freq=3)), ("KukaButtonGymEnv-v0", 1, dict(gradient_steps=2))])
def test_captured_and_eager_sac_runs_give_the_same_bytes(cuda_lib, env_id, stack, hp):
    from rl_baselines import sac
    out = []
    for graph in (True, False):
        sac.train(env_id, 512, 512 * 130, seed=2, env_kwargs=dict(is_discrete=False, shape_reward=True), verbose=0, hyperparams=dict(buffer_size=300, **hp),
                  num_stack=stack, cuda_graph=graph)
        t = sac.train
        out.append(dict(arena=t.last_nets.arena.detach().clone(), target=t.last_nets.target.clone(), m=t.last_adam[0].clone(), v=t.last_adam[1].clone(),
                        **{"ring_" + k: v.clone() for k, v in t.last_ring.items()}, stats=dict(t.stats)))
    assert out[0]["stats"]["graph_replays"] > 0 and out[1]["stats"]["graph_replays"] == 0
    assert out[0]["stats"]["grad_steps"] == out[1]["stats"]["grad_steps"] > 0
    for k in out[0]:
        if k != "stats":
            assert torch.equal(out[0][k], out[1][k]), k


def test_train_entry_point_runs_sac_on_every_registry_id(cuda_lib, tmp_path):
    from environments.registry import registered_env
    from rl_baselines.train import main
    refused = []
    for env_id in registered_env:
        argv = ["--algo", "sac", "-c", "--env", env_id, "--num-cpu", "256", "--num-timesteps", str(256 * 120), "--buffer-size", "200",
                "--log-dir", str(tmp_path), "--seed", "1"]
        if env_id in ("MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0"):    # discrete only, as in the reference
            with pytest.raises(ValueError, match="Only discrete actions is supported"):
                main(argv)
            refused.append(env_id)
            continue
        hist = main(argv)
        assert len(hist) == 132 and all(np.isfinite(h[2]) for h in hist), env_id
    assert len(refused) == 2 and len(registered_env) == 8


def test_oversized_ring_is_refused_before_allocating(cuda_lib):
    from rl_baselines import sac
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="--buffer-size"):
        sac.train("KukaButtonGymEnv-v0", 4096, 4096 * 10, env_kwargs=dict(is_discrete=False), verbose=0, hyperparams=dict(buffer_size=10 ** 7))
    assert torch.cuda.memory_allocated() - before < 64 << 20


def test_sac_learns_mobile_robot(cuda_lib):
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.sac import train
    hist = train("MobileRobotGymEnv-v0", 1024, 1024 * 2000, seed=0, env_kwargs=dict(is_discrete=False, shape_reward=True), verbose=0)
    rets = [h[1] for h in hist if np.isfinite(h[1])]
    print("\nSAC MobileRobot: first window %.1f, last %.1f, fps %.0f, %s" % (rets[0], rets[-1], hist[-1][2], train.stats))
    print("  windows:", [round(x, 1) for x in rets[::100]])
    # shaped reward = -distance per step over 251 steps; measured on an H100 80GB HBM3 (700 W): -496.5 in the first window, -122.6 in the
    # last, 1901 gradient steps, 950 graph replays of the one graph
    assert rets[-1] > rets[0] + 200, rets[::100]
    assert train.stats["graph_replays"] > 0
