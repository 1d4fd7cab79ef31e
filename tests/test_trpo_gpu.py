"""
TRPO's kernels (include/srl_policy.h: srl_trpo_*) on the GPU against the float64 model of tests/trpo_numpy_ref.py, the vector kernel's CG,
step and line-search decisions on the kernel's own products, and the trainer (rl_baselines/trpo.py): captured against eager runs, an odd
timesteps_per_batch, and the entry point.
"""
import numpy as np
import pytest
import torch

import trpo_numpy_ref as ref
from test_consumer_reference_cpu import grad_bound

pytestmark = pytest.mark.gpu
THREE_CHUNKS_PER_CTA = -1      # rows = SMs x 64 x 3 + 17, with the device's SM count

# (obs_dim, n_out, discrete): MobileRobot (2-D, 4 actions / 2-D Box), Kuka (3-D, 6 actions / 3-D Box), -joints (7-D Box), stacks of 4 and of 8
SHAPES = [(2, 4, True), (2, 2, False), (3, 6, True), (3, 3, False), (3, 7, False), (12, 6, True), (32, 8, False)]


def _lib():
    from srl_sim._abi import load_cuda_library
    return load_cuda_library()


def _policy(D, A, discrete, seed, wide_sigma=False):
    from rl_baselines.ppo2 import MlpPolicy
    torch.manual_seed(seed)
    pol = MlpPolicy(D, n_actions=A) if discrete else MlpPolicy(D, action_dim=A)
    with torch.no_grad():
        for p in pol.parameters():
            p.add_(0.3 * torch.randn_like(p))
        if discrete:
            pol.pi[4].bias[0] = 12.0                     # a saturated softmax
        else:
            pol.logstd.copy_(torch.linspace(-1.5, 1.2, A))   # sigma far from 1
    return pol.cuda()


def _data(D, A, discrete, rows, seed):
    g = torch.Generator().manual_seed(seed)
    obs = 2 * torch.randn(rows, D, generator=g)
    act = torch.randint(0, A, (rows,), generator=g) if discrete else torch.randn(rows, A, generator=g)
    adv = torch.randn(rows, generator=g) + 0.5
    return obs.cuda(), act.cuda(), adv.cuda()


def _theta(pol):
    from rl_baselines.trpo import flat, pi_params
    return flat(pi_params(pol)).detach().double().cpu().numpy()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _segments(D, A, box):
    names = [("w1", 64 * D), ("b1", 64), ("w2", 64 * 64), ("b2", 64), ("w3", A * 64), ("b3", A)] + ([("ls", A)] if box else [])
    out, o = [], 0
    for n, k in names:
        out.append((n, o, o + k)); o += k
    return out


def _per_tensor(got, want, segs, what):
    """Every tensor of a flat vector within grad_bound of its largest entry; returns the largest error / bound."""
    got, want, worst = np.asarray(got, np.float64), np.asarray(want, np.float64), 0.0
    for name, lo, hi in segs:
        err, bound = np.abs(got[lo:hi] - want[lo:hi]).max(), grad_bound(np.abs(want[lo:hi]).max())
        assert err <= bound, (what, name, err, bound)
        worst = max(worst, err / bound)
    return worst


def _misses(got, want, segs):
    """Some tensor lies beyond grad_bound of ``want`` (a control's shortened model)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return any(np.abs(got[lo:hi] - want[lo:hi]).max() > grad_bound(np.abs(want[lo:hi]).max()) for _, lo, hi in segs)


def _close(got, want, what, rel=2e-4, atol=1e-7):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    bound = rel * np.abs(want).max() + atol
    err = np.abs(got - want).max()
    assert err <= bound, "%s: max error %.3g > %.3g" % (what, err, bound)
    return err


@pytest.mark.parametrize("D,A,discrete", SHAPES)
@pytest.mark.parametrize("rows", [1, 33, THREE_CHUNKS_PER_CTA, 26 * 4096, 128 * 4096])
def test_surrogate_fvp_trial_match_the_float64_model(D, A, discrete, rows):
    """Rows: one, a partial chunk, three chunks per CTA and a tail, the FVP subsample and the full batch of KukaButton at 4096 envs."""
    from srl_sim.policy import FusedTRPO
    lib = _lib()
    if rows == THREE_CHUNKS_PER_CTA:
        rows = _sms() * 64 * 3 + 17
    segs = _segments(D, A, not discrete)
    pol = _policy(D, A, discrete, D * 100 + A)
    obs, act, adv = _data(D, A, discrete, rows, rows + D)
    f = FusedTRPO(lib, pol, rows)
    f.surrogate(obs, act, adv, 0.01)
    th = _theta(pol)
    x64, a64, adv64 = obs.double().cpu().numpy(), act.cpu().numpy(), adv.double().cpu().numpy()
    if rows > 1:
        atarg, g, losses, zold = ref.surrogate(th, D, A, discrete, x64, a64 if discrete else a64.astype(np.float64), adv64, 0.01)
        _close(f.atarg.cpu().numpy(), atarg, "atarg", 1e-5)
        _per_tensor(f.g.cpu().numpy(), g, segs, "gradient")
        _close(f.old_out.cpu().numpy(), zold, "old outputs", 1e-5)
        l = f.losses.cpu().numpy()
        assert abs(l[0] - losses["surrgain"]) < 1e-5 and l[1] == 0.0 and abs(l[2] - losses["meanent"]) < 1e-4 * (1 + abs(losses["meanent"]))
    v = torch.randn(f.P, generator=torch.Generator().manual_seed(rows)).cuda()
    out = torch.empty_like(v)
    f.fvp(rows, rows, rows, obs, v, 0.2, out)
    _per_tensor(out.cpu().numpy(), ref.fvp_gauss_newton(th, D, A, discrete, x64, v.double().cpu().numpy(), 0.2), segs, "fvp")
    # the same bytes twice
    out2 = torch.empty_like(v)
    f.fvp(rows, rows, rows, obs, v, 0.2, out2)
    assert torch.equal(out, out2)
    if rows > 1:
        # one trial at theta_old + fullstep: the state record asks for scale 1 after START
        f.vector(0, 0.01, 0.01)
        f.fullstep.copy_(0.002 * torch.randn(f.P, generator=torch.Generator().manual_seed(7)).cuda())
        f.trial(obs, act)
        th_new = th + f.fullstep.double().cpu().numpy()
        old_ls = None if discrete else pol.logstd.detach().double().cpu().numpy()
        want = ref.trial_losses(th_new, D, A, discrete, x64, a64, f.atarg.double().cpu().numpy(), f.old_out.double().cpu().numpy(), old_ls, 0.01)
        l = f.losses.cpu().numpy()
        # means of O(1) float32 terms: an absolute floor for the cancellation of a mean near 0
        _close(l[0], want["surrgain"], "trial surrgain", 1e-4, 2e-6)
        _close(l[1], want["meankl"], "trial meankl", 1e-3, 2e-6)
        _close(l[2], want["meanent"], "trial meanent", 1e-4, 2e-6)


@pytest.mark.parametrize("D,A,discrete", [(3, 6, True), (3, 3, False)])
@pytest.mark.parametrize("rows,drop", [(130, "row"), (THREE_CHUNKS_PER_CTA, "chunk")])
def test_controls_leave_rows_out(D, A, discrete, rows, drop):
    """Controls: the model without one row (130 rows) or without one 64-row chunk in the middle of a three-chunks-per-CTA batch, at the same
    1 / rows per sample, differs from the kernel beyond the bound the comparisons hold it to, in the surrogate gradient, the FVP and the value
    gradient."""
    from rl_baselines.trpo import flat, vf_params
    from srl_sim.policy import FusedTRPO
    lib = _lib()
    if rows == THREE_CHUNKS_PER_CTA:
        rows = _sms() * 64 * 3 + 5
    keep = np.ones(rows, bool)
    if drop == "row":
        keep[rows - 1] = False
    else:
        keep[64 * 200:64 * 201] = False
    pol = _policy(D, A, discrete, 13)
    obs, act, adv = _data(D, A, discrete, rows, 17)
    ret = torch.randn(rows, generator=torch.Generator().manual_seed(2)).cuda()
    f = FusedTRPO(lib, pol, rows)
    f.surrogate(obs, act, adv, 0.01)
    v = torch.randn(f.P, generator=torch.Generator().manual_seed(3)).cuda()
    f.fvp(rows, rows, rows, obs, v, 0.2, f.z)
    f.vf_grad(rows, None, obs, ret)
    th, segs, scale = _theta(pol), _segments(D, A, not discrete), keep.sum() / rows
    x, a, at, v64 = obs.double().cpu().numpy(), act.cpu().numpy(), f.atarg.double().cpu().numpy(), v.double().cpu().numpy()
    model_g = lambda k: ref.surrogate(th, D, A, discrete, x[k], a[k], None, 0.01, atarg=at[k])[1]
    _per_tensor(f.g.cpu().numpy(), model_g(slice(None)), segs, "gradient")
    assert _misses(f.g.cpu().numpy(), model_g(keep) * scale, segs), "gradient control"
    fv = lambda k: ref.fvp_gauss_newton(th, D, A, discrete, x[k], v64, 0.0)
    _per_tensor(f.z.cpu().numpy() - 0.2 * v.cpu().numpy(), fv(slice(None)), segs, "fvp")
    short = fv(keep)
    if not discrete:                                   # the logstd block 2 v does not depend on the rows
        short[-A:] /= scale
    assert _misses(f.z.cpu().numpy() - 0.2 * v.cpu().numpy(), short * scale, segs), "fvp control"
    wv = ref.unflat(flat(vf_params(pol)).detach().double().cpu().numpy(), D, 1, False)
    r64 = ret.double().cpu().numpy()

    def vgrad(k):
        h1, h2, out = ref.forward(wv, x[k])
        return ref.flat_of(ref.backward(wv, x[k], h1, h2, 2 * (out - r64[k, None]) / rows), ["w1", "b1", "w2", "b2", "w3", "b3"])
    vsegs = _segments(D, 1, False)
    _per_tensor(f.vgrad.cpu().numpy(), vgrad(slice(None)), vsegs, "value gradient")
    assert _misses(f.vgrad.cpu().numpy(), vgrad(keep), vsegs), "value gradient control"


def test_fvp_on_the_strided_subsample_is_symmetric_and_positive():
    from srl_sim.policy import FusedTRPO
    lib = _lib()
    T, N = 128, 832
    for D, A, discrete in [(3, 6, True), (3, 3, False)]:
        pol = _policy(D, A, discrete, 5)
        obs, _, _ = _data(D, A, discrete, T * N, 11)
        f = FusedTRPO(lib, pol, T * N)
        sub = ((T + 4) // 5) * N
        g = torch.Generator().manual_seed(3)
        u, v = torch.randn(f.P, generator=g).cuda(), torch.randn(f.P, generator=g).cuda()
        Fu, Fv = torch.empty_like(u), torch.empty_like(v)
        f.fvp(sub, N, 5 * N, obs, u, 0.2, Fu)
        f.fvp(sub, N, 5 * N, obs, v, 0.2, Fv)
        a, b = float(u.double() @ Fv.double()), float(v.double() @ Fu.double())
        assert abs(a - b) <= 1e-4 * max(abs(a), abs(b))
        assert float(v.double() @ Fv.double()) > 0.2 * float(v.double() @ v.double()) * 0.999
        x_sub = obs.reshape(T, N, D)[::5].reshape(-1, D).double().cpu().numpy()
        _close(Fv.cpu().numpy(), ref.fvp_gauss_newton(_theta(pol), D, A, discrete, x_sub, v.double().cpu().numpy(), 0.2), "strided fvp")


@pytest.mark.parametrize("D,A,discrete", [(3, 6, True), (3, 3, False)])
def test_vector_kernel_cg_step_and_line_search(D, A, discrete):
    from srl_sim.policy import (FusedTRPO, TRPO_ACCEPTED, TRPO_CG_ITERS, TRPO_RESTORED, TRPO_SHS, TRPO_SKIP, TRPO_TRIAL_LOSSES, TRPO_TRIALS)
    lib = _lib()
    rows = 4096
    pol = _policy(D, A, discrete, 9)
    obs, act, adv = _data(D, A, discrete, rows, 2)
    f = FusedTRPO(lib, pol, rows)
    f.surrogate(obs, act, adv, 0.01)
    f.vector(0, 0.01, 0.01)
    assert f.state[TRPO_SKIP].item() == 0
    g = f.g.double().cpu().numpy()
    products = []
    for i in range(4):
        products.append(f.p.double().cpu().numpy())
        f.fvp(rows, rows, rows, obs, f.p, 0.2, f.z)
        zi = f.z.double().cpu().numpy()
        f.vector(1, 0.01, 0.01)
        products[-1] = (products[-1], zi)
    # float64 CG on the kernel's own products: the iterate after 4 iterations
    p, r, x = g.copy(), g.copy(), np.zeros_like(g)
    rdotr, n_it = r @ r, 0
    for pin, z in products:
        _close(pin, p, "cg input", 1e-3)
        vv = rdotr / (pin @ z)
        x += vv * pin; r -= vv * z
        nr = r @ r; p = r + nr / rdotr * p; rdotr = nr
        n_it += 1
        if rdotr < 1e-10:                   # the tolerance break: the kernel's later iterations are no-ops
            break
    _close(f.x.cpu().numpy(), x, "cg iterate", 1e-3)
    assert f.state[TRPO_CG_ITERS].item() == n_it
    f.fvp(rows, rows, rows, obs, f.x, 0.2, f.z)
    f.vector(2, 0.01, 0.01)
    shs, lm, fullstep = ref.step_size(f.x.double().cpu().numpy(), f.z.double().cpu().numpy(), 0.01)
    assert abs(f.state[TRPO_SHS].item() - shs) <= 1e-9 * abs(shs)
    _close(f.fullstep.cpu().numpy(), fullstep, "fullstep", 1e-6)
    before = [t.detach().clone() for t in pol.parameters()]
    th = _theta(pol)
    old_ls = None if discrete else pol.logstd.detach().double().cpu().numpy()
    gain_before = f.state[9].item()
    decisions = []
    for k in range(10):
        f.trial(obs, act)
        f.vector(3, 0.01, 0.01)
        st = f.state.cpu().numpy()
        if st[TRPO_TRIALS] == k:            # a decision was made before: nothing ran
            break
        l = dict(optimgain=st[TRPO_TRIAL_LOSSES + 3 * k], meankl=st[TRPO_TRIAL_LOSSES + 3 * k + 1], meanent=st[TRPO_TRIAL_LOSSES + 3 * k + 2])
        want = ref.trial_losses(th + fullstep * 0.5 ** k, D, A, discrete, obs.double().cpu().numpy(), act.cpu().numpy(),
                                f.atarg.double().cpu().numpy(), f.old_out.double().cpu().numpy(), old_ls, 0.01)
        d, dw = ref.decide(l, gain_before, 0.01), ref.decide(want, gain_before, 0.01)
        margin = min(abs(want["meankl"] - 0.015), abs(want["optimgain"] - gain_before))
        assert d == dw or margin < 1e-5, (k, d, dw, margin)
        decisions.append(d)
        if d == "accept":
            break
    st = f.state.cpu().numpy()
    if decisions[-1] == "accept":
        assert st[TRPO_ACCEPTED] == len(decisions) - 1
        new = _theta(pol)
        want_th = (torch.tensor(th, dtype=torch.float32) + torch.tensor(f.fullstep.cpu().numpy()) * np.float32(0.5 ** (len(decisions) - 1))).numpy()
        np.testing.assert_array_equal(new.astype(np.float32), want_th)
    else:
        assert st[TRPO_RESTORED] == 1
        assert all(torch.equal(a, b) for a, b in zip(before, pol.parameters()))


def test_crafted_trials_reject_everything_and_leave_the_bytes():
    from srl_sim.policy import FusedTRPO, TRPO_ACCEPTED, TRPO_RESTORED, TRPO_TRIALS
    lib = _lib()
    rows = 2048
    pol = _policy(3, 6, True, 1)
    obs, act, adv = _data(3, 6, True, rows, 4)
    f = FusedTRPO(lib, pol, rows)
    f.surrogate(obs, act, adv, 0.01)
    f.vector(0, 0.01, 0.01)
    before = [t.detach().clone() for t in pol.parameters()]
    f.fullstep.copy_(-1e3 * f.g)          # a step against the gradient, far too long: KL violations, then negative improvements
    for _ in range(10):
        f.trial(obs, act); f.vector(3, 0.01, 0.01)
    st = f.state.cpu().numpy()
    assert st[TRPO_TRIALS] == 10 and st[TRPO_ACCEPTED] == -1 and st[TRPO_RESTORED] == 1
    assert all(torch.equal(a, b) for a, b in zip(before, pol.parameters()))
    # a tiny step along the gradient is accepted at the first trial
    f.vector(0, 0.01, 0.01)
    f.fullstep.copy_(1e-4 * f.g / f.g.norm())
    f.trial(obs, act); f.vector(3, 0.01, 0.01)
    assert f.state[TRPO_ACCEPTED].item() == 0
    # a non-finite trial is rejected
    f.vector(0, 0.01, 0.01)
    f.fullstep.fill_(float("nan"))
    f.trial(obs, act); f.vector(3, 0.01, 0.01)
    assert f.state[TRPO_ACCEPTED].item() == -1 and f.state[TRPO_TRIALS].item() == 1
    # a zero gradient skips the update
    f.g.zero_(); f.vector(0, 0.01, 0.01)
    assert f.state[0].item() == 1


def test_value_gradient_and_adam_match_the_model():
    from rl_baselines.trpo import flat, vf_params
    from srl_sim.policy import FusedTRPO
    lib = _lib()
    rows, D = 128 * 40, 3
    pol = _policy(D, 6, True, 3)
    obs, _, _ = _data(D, 6, True, rows, 8)
    ret = torch.randn(rows, generator=torch.Generator().manual_seed(5)).cuda()
    f = FusedTRPO(lib, pol, rows)
    idx = torch.randperm(rows, device="cuda")[:rows // 2]
    f.vf_grad(rows // 2, idx, obs, ret)
    vfs = vf_params(pol)
    w = {k: t.detach().double().cpu().numpy() for k, t in zip(["w1", "b1", "w2", "b2", "w3", "b3"], vfs)}
    x = obs[idx].double().cpu().numpy()
    h1, h2, v = ref.forward(w, x)
    dz = 2 * (v - ret[idx].double().cpu().numpy()[:, None]) / x.shape[0]
    want = ref.flat_of(ref.backward(w, x, h1, h2, dz), ["w1", "b1", "w2", "b2", "w3", "b3"])
    _close(f.vgrad.cpu().numpy(), want, "value gradient")
    w0, g = flat(vfs).detach().cpu().numpy(), f.vgrad.cpu().numpy()
    f.vf_adam(2.5e-4)
    wn, m, vv, t = ref.mpi_adam_f32(w0, g, np.zeros_like(g), np.zeros_like(g), 0, 2.5e-4)
    np.testing.assert_array_equal(flat(vfs).detach().cpu().numpy(), wn)
    np.testing.assert_array_equal(f.m.cpu().numpy(), m)
    np.testing.assert_array_equal(f.v.cpu().numpy(), vv)
    assert int(f.step.item()) == 1


def _run(env_id, N, updates, T, cuda_graph, env_kwargs, num_stack=1):
    from rl_baselines import trpo
    hp = dict(timesteps_per_batch=T)
    hist = trpo.train(env_id, N, N * T * updates, seed=5, env_kwargs=env_kwargs, verbose=0, device=0, hyperparams=hp, cuda_graph=cuda_graph,
                      num_stack=num_stack)
    lu = trpo.train.last_update
    pol = trpo.train.last_policy
    return dict(hist=hist, params=[p.detach().cpu().clone() for p in pol.parameters()], filt=trpo.train.last_norm.state.cpu().clone(),
                adam=[t.cpu().clone() for t in lu["adam"]], state=lu["record"]["state"].copy(), graph=lu["graph"])


@pytest.mark.parametrize("env_id,kw,stack", [("MobileRobotGymEnv-v0", dict(is_discrete=True, shape_reward=True), 1),
                                            ("KukaButtonGymEnv-v0", dict(is_discrete=True), 1),
                                            ("KukaButtonGymEnv-v0", dict(is_discrete=False), 1),
                                            ("KukaButtonGymEnv-v0", dict(is_discrete=True), 3)])
def test_captured_update_equals_eager(env_id, kw, stack):
    a = _run(env_id, 256, 3, 128, True, kw, stack)
    b = _run(env_id, 256, 3, 128, False, kw, stack)
    assert a["graph"] and not b["graph"]
    for x, y in zip(a["params"], b["params"]):
        assert torch.equal(x, y)
    assert torch.equal(a["filt"], b["filt"])
    for x, y in zip(a["adam"], b["adam"]):
        assert torch.equal(x, y)
    np.testing.assert_array_equal(a["state"], b["state"])
    assert a["adam"][2].item() == 9            # 3 updates x 3 epochs x 1 minibatch


def test_odd_batch_trains_eagerly():
    r = _run("MobileRobotGymEnv-v0", 64, 2, 129, True, dict(is_discrete=False))
    assert not r["graph"] and len(r["hist"]) == 2


def test_entry_point_every_registry_id(tmp_path):
    from environments.registry import registered_env
    from rl_baselines.train import main
    for env_id in sorted(registered_env):
        hist = main(["--algo", "trpo", "--env", env_id, "--num-cpu", "64", "--num-timesteps", str(64 * 10 * 2), "--hyperparam",
                     "timesteps_per_batch:10", "--log-dir", str(tmp_path)])
        assert len(hist) == 2, env_id


def test_learning_mobile_robot_shaped():
    from rl_baselines import trpo
    hist = trpo.train("MobileRobotGymEnv-v0", 1024, 1024 * 128 * 30, seed=0, env_kwargs=dict(is_discrete=True, shape_reward=True), verbose=0, device=0)
    first = next(h[1] for h in hist if np.isfinite(h[1]))       # the first update may end no episode
    last = max(h[1] for h in hist[-5:])
    print("TRPO MobileRobot shaped, 1024 envs: windowed return %.3f -> %.3f" % (first, last))
    assert last - first >= 200.0        # measured on an H100: -494.8 -> -52.0 over 30 updates (DESIGN.md section 5.4)
