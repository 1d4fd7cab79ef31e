"""
One TRPO update of the trainer (rl_baselines/trpo.py, captured as one CUDA graph) rebuilt from ``train.last_update``: the advantages, their
standardisation, the gradient, every CG product and iterate, shs and fullstep, each trial's losses and decision against the float64 model of
tests/trpo_numpy_ref.py; the same launches replayed by hand give the trainer's bytes (so the trainer's subsample, product inputs and value rows
are the ones stated here), and the value steps are MpiAdam bit for bit from the kernel's own gradients.
"""
import numpy as np
import pytest
import torch

import trpo_numpy_ref as ref
from test_consumer_reference_cpu import grad_bound

pytestmark = pytest.mark.gpu

CASES = [("KukaButtonGymEnv-v0", 4096, dict(is_discrete=True), 1), ("KukaButtonGymEnv-v0", 4096, dict(is_discrete=False), 1),
         ("KukaButtonGymEnv-v0", 4096, dict(is_discrete=True), 4), ("MobileRobotGymEnv-v0", 8192, dict(is_discrete=True, shape_reward=True), 1)]
DECISION_MARGIN = 1e-5     # a trial decision may differ from float64 only where the float64 value is this close to its threshold


def _segments(D, A, box):
    names = [("w1", H * D), ("b1", H), ("w2", H * H), ("b2", H), ("w3", A * H), ("b3", A)] + ([("ls", A)] if box else [])
    out, o = [], 0
    for n, k in names:
        out.append((n, o, o + k)); o += k
    return out


H = 64


def _per_tensor(got, want, segs, what):
    worst = 0.0
    for name, lo, hi in segs:
        err, bound = np.abs(got[lo:hi] - want[lo:hi]).max(), grad_bound(np.abs(want[lo:hi]).max())
        assert err <= bound, (what, name, err, bound)
        worst = max(worst, err / bound)
    return worst


@pytest.mark.parametrize("env_id,N,kw,stack", CASES)
def test_one_update_rebuilt_in_float64(env_id, N, kw, stack):
    from rl_baselines import trpo
    from srl_sim.policy import TRPO_ACCEPTED, TRPO_GAIN_BEFORE, TRPO_SHS, TRPO_TRIAL_LOSSES, TRPO_TRIALS
    T = 128
    trpo.train(env_id, N, N * T, seed=3, env_kwargs=kw, verbose=0, device=0, num_stack=stack)
    lu, pol = trpo.train.last_update, trpo.train.last_policy
    assert lu["graph"]
    f, hp, buf = lu["fused"], lu["hp"], lu["buf"]
    pis, vfs = trpo.pi_params(pol), trpo.vf_params(pol)
    after = [t.detach().clone() for t in pis + vfs]
    p0 = lu["params0"]
    discrete = pol.discrete
    W, rows = buf["obs"].shape[2], T * N
    A = f.old_out.shape[1]
    segs = _segments(W, A, not discrete)
    flat_obs, flat_act = buf["obs"].reshape(rows, W), buf["act"].reshape((rows,) + buf["act"].shape[2:])
    x64 = flat_obs.double().cpu().numpy()
    a64 = flat_act.cpu().numpy()
    # ---- GAE and the standardised advantages ----
    rew, val, done = (buf[k].double().cpu().numpy() for k in ("rew", "val", "done"))
    last = lu["last_val"].double().cpu().numpy()
    adv_m, lastgae = np.zeros((T, N)), np.zeros(N)
    for t in reversed(range(T)):
        nextval = last if t == T - 1 else val[t + 1]
        delta = rew[t] + hp["gamma"] * nextval * (1 - done[t]) - val[t]
        lastgae = delta + hp["gamma"] * hp["lam"] * (1 - done[t]) * lastgae
        adv_m[t] = lastgae
    adv = lu["adv"].double().cpu().numpy()
    assert np.abs(adv - adv_m).max() <= 1e-4 * np.abs(adv_m).max() + 1e-5
    th0 = trpo.flat(p0[:len(pis)]).double().cpu().numpy()
    atarg_m, g_m, losses_m, z_old = ref.surrogate(th0, W, A, discrete, x64, a64, adv.reshape(-1), hp["entcoeff"])
    assert np.abs(f.atarg.double().cpu().numpy() - atarg_m).max() <= 1e-5 * np.abs(atarg_m).max()
    # ---- the gradient ----
    worst_g = _per_tensor(f.g.double().cpu().numpy(), g_m, segs, "gradient")
    gain_m = losses_m["surrgain"] + hp["entcoeff"] * losses_m["meanent"]
    st_trainer = f.state.cpu().numpy().copy()
    assert abs(st_trainer[TRPO_GAIN_BEFORE] - gain_m) <= 1e-5 * (1 + abs(gain_m))
    x_trainer, fs_trainer, g_trainer = f.x.clone(), f.fullstep.clone(), f.g.clone()
    # ---- the same launches by hand, from the parameters the update started from ----
    with torch.no_grad():
        for t, s in zip(pis + vfs, p0):
            t.copy_(s)
    sub_rows = ((T + 4) // 5) * N
    f.surrogate(flat_obs, flat_act, lu["adv"].reshape(-1), hp["entcoeff"])
    assert torch.equal(f.g, g_trainer)
    f.vector(0, hp["max_kl"], hp["entcoeff"])
    x_sub = buf["obs"][::5].reshape(-1, W).double().cpu().numpy()
    assert x_sub.shape[0] == sub_rows
    fvp_m = lambda v: ref.fvp_gauss_newton(th0, W, A, discrete, x_sub, v, hp["cg_damping"])
    worst_z, iterates = 0.0, []
    for i in range(hp["cg_iters"]):
        p_in = f.p.double().cpu().numpy()
        f.fvp(sub_rows, N, 5 * N, flat_obs, f.p, hp["cg_damping"], f.z)
        worst_z = max(worst_z, _per_tensor(f.z.double().cpu().numpy(), fvp_m(p_in), segs, "product %d" % i))
        f.vector(1, hp["max_kl"], hp["entcoeff"])
        iterates.append(f.x.double().cpu().numpy())
    # float64 CG from the kernel's gradient on the model's products: every iterate the kernel ran
    _, n_it, its_m, _ = ref.cg_loop(fvp_m, f.g.double().cpu().numpy(), hp["cg_iters"])
    assert int(f.state[1].item()) == n_it
    cg_rel = [np.abs(a - b).max() / np.abs(b).max() for a, b in zip(iterates[:n_it], its_m)]
    assert max(cg_rel) <= 2e-3, cg_rel
    x_k = f.x.double().cpu().numpy()
    f.fvp(sub_rows, N, 5 * N, flat_obs, f.x, hp["cg_damping"], f.z)
    f.vector(2, hp["max_kl"], hp["entcoeff"])
    assert torch.equal(f.x, x_trainer) and torch.equal(f.fullstep, fs_trainer)
    shs_m, lm_m, fs_m = ref.step_size(x_k, fvp_m(x_k), hp["max_kl"])
    assert abs(f.state[TRPO_SHS].item() - shs_m) <= 2e-4 * abs(shs_m)
    assert np.abs(f.fullstep.double().cpu().numpy() - fs_m).max() <= 2e-4 * np.abs(fs_m).max()
    for _ in range(10):
        f.trial(flat_obs, flat_act)
        f.vector(3, hp["max_kl"], hp["entcoeff"])
    st = f.state.cpu().numpy()
    np.testing.assert_array_equal(st, st_trainer)
    for a, b in zip(pis, after):
        assert torch.equal(a, b)
    # ---- each trial's losses and decision ----
    fs32, th32 = f.fullstep.cpu(), trpo.flat(p0[:len(pis)]).cpu()
    old_ls = None if discrete else th0[-A:]
    accepted, reported = int(st[TRPO_ACCEPTED]), []
    for k in range(int(st[TRPO_TRIALS])):
        th_k = (th32 + fs32 * np.float32(0.5 ** k)).double().numpy()           # the float32 trial weights the kernel forms
        want = ref.trial_losses(th_k, W, A, discrete, x64, a64, atarg_m, z_old, old_ls, hp["entcoeff"])
        got = dict(optimgain=st[TRPO_TRIAL_LOSSES + 3 * k], meankl=st[TRPO_TRIAL_LOSSES + 3 * k + 1], meanent=st[TRPO_TRIAL_LOSSES + 3 * k + 2])
        assert abs(got["optimgain"] - want["optimgain"]) <= 1e-4 * abs(want["optimgain"]) + 2e-6, (k, got, want)
        assert abs(got["meankl"] - want["meankl"]) <= 1e-3 * abs(want["meankl"]) + 2e-6, (k, got, want)
        d_kernel = "accept" if k == accepted else "reject"
        d_model = ref.decide(want, gain_m, hp["max_kl"])
        if (d_model == "accept") != (d_kernel == "accept"):
            margin = min(abs(want["meankl"] - 1.5 * hp["max_kl"]), abs(want["optimgain"] - gain_m))
            assert margin <= DECISION_MARGIN, (k, d_kernel, d_model, margin)
            reported.append((k, d_kernel, d_model, margin))
    if accepted >= 0:
        want_pi = th32 + fs32 * np.float32(0.5 ** accepted)
        assert torch.equal(trpo.flat(after[:len(pis)]).cpu(), want_pi)
    else:
        assert torch.equal(trpo.flat(after[:len(pis)]).cpu(), th32)
    # ---- the value steps: the kernel's gradients against float64, MpiAdam bit for bit ----
    vidx = lu["vidx"]
    for b in range(vidx.shape[0]):                # T = 128: one minibatch per epoch, a permutation of every row
        assert torch.equal(torch.sort(vidx[b]).values.cpu(), torch.arange(rows))
    m0, v0, t0 = lu["adam0"]
    with torch.no_grad():
        f.m.copy_(m0); f.v.copy_(v0); f.step.copy_(t0)
    w = trpo.flat(vfs).detach().cpu().numpy()
    m, v, tt = m0.cpu().numpy(), v0.cpu().numpy(), int(t0.item())
    vsegs = _segments(W, 1, False)
    ret = lu["ret"].reshape(-1)
    worst_v = 0.0
    for b in range(vidx.shape[0]):
        f.vf_grad(128 * N, vidx[b], flat_obs, ret)
        g = f.vgrad.cpu().numpy()
        ix = vidx[b].cpu().numpy()
        wv = ref.unflat(trpo.flat(vfs).detach().double().cpu().numpy(), W, 1, False)
        h1, h2, vout = ref.forward(wv, x64[ix])
        want = ref.flat_of(ref.backward(wv, x64[ix], h1, h2, 2 * (vout - ret.double().cpu().numpy()[ix, None]) / len(ix)),
                           ["w1", "b1", "w2", "b2", "w3", "b3"])
        worst_v = max(worst_v, _per_tensor(g.astype(np.float64), want, vsegs, "value gradient %d" % b))
        f.vf_adam(hp["vf_stepsize"])
        w, m, v, tt = ref.mpi_adam_f32(w, g, m, v, tt, hp["vf_stepsize"])
        np.testing.assert_array_equal(trpo.flat(vfs).detach().cpu().numpy(), w)
        np.testing.assert_array_equal(f.m.cpu().numpy(), m)
        np.testing.assert_array_equal(f.v.cpu().numpy(), v)
    for a, b in zip(vfs, after[len(pis):]):
        assert torch.equal(a, b)
    print("\n%s N=%d stack=%d %s: error / grad_bound gradient %.3f, products %.3f, value %.3f; CG iterates rel %s; accepted trial %d; "
          "decisions within the margin: %s" % (env_id, N, stack, "discrete" if discrete else "box", worst_g, worst_z, worst_v,
                                               ["%.1e" % r for r in cg_rel], accepted, reported))
