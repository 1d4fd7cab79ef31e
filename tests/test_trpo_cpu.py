"""
TRPO trainer (rl_baselines/trpo.py) without a GPU: the torch statement of the losses, the double-backprop Fisher-vector product, CG, the step
size, the line search and MpiAdam against the float64 model of tests/trpo_numpy_ref.py, the value-minibatch cadence, and the trainer on the
oracle backend (single process, two gloo ranks, the entry point and replay).
"""
import glob
import json
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import trpo_numpy_ref as ref
from conftest import ORACLE_LIB, PKG
from test_ppo2_distributed_cpu import _free_port


def _policy(D, A, discrete, seed):
    from rl_baselines.ppo2 import MlpPolicy
    torch.manual_seed(seed)
    pol = (MlpPolicy(D, n_actions=A) if discrete else MlpPolicy(D, action_dim=A)).double()
    with torch.no_grad():
        for p in pol.parameters():
            p.add_(0.3 * torch.randn_like(p))
        if discrete:
            pol.pi[4].bias[0] = 25.0                         # a saturated softmax
        else:
            pol.logstd.copy_(torch.linspace(-2.0, 1.5, A))   # sigma far from 1
    return pol


def _data(D, A, discrete, B, seed):
    g = torch.Generator().manual_seed(seed)
    obs = 2 * torch.randn(B, D, generator=g, dtype=torch.float64)
    act = torch.randint(0, A, (B,), generator=g) if discrete else torch.randn(B, A, generator=g, dtype=torch.float64)
    return obs, act, torch.randn(B, generator=g, dtype=torch.float64) + 0.3


@pytest.mark.parametrize("D,A,discrete", [(2, 4, True), (3, 6, True), (2, 2, False), (3, 7, False), (12, 6, True), (32, 8, False)])
def test_surrogate_gradient_and_losses_match_the_model(D, A, discrete):
    from rl_baselines.trpo import flat, pi_params, trpo_losses
    pol = _policy(D, A, discrete, D + A)
    obs, act, adv = _data(D, A, discrete, 300, D)
    atarg = (adv - adv.mean()) / adv.std(unbiased=False)
    with torch.no_grad():
        old = pol.pi(obs)
    old_ls = None if discrete else pol.logstd.detach().clone()
    gain, kl, ent, surr = trpo_losses(pol, old, old_ls, obs, act, atarg, 0.01)
    g = flat(torch.autograd.grad(gain, pi_params(pol))).numpy()
    th = flat(pi_params(pol)).detach().numpy()
    atarg_m, g_m, losses, _ = ref.surrogate(th, D, A, discrete, obs.numpy(), act.numpy(), adv.numpy(), 0.01)
    np.testing.assert_allclose(atarg.numpy(), atarg_m, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(g, g_m, rtol=1e-9, atol=1e-12)
    kl, surr, ent = kl.detach(), surr.detach(), ent.detach()
    assert abs(float(kl)) < 1e-15 and abs(float(surr) - losses["surrgain"]) < 1e-12 and abs(float(ent) - losses["meanent"]) < 1e-12
    # a trial point: ratio, KL(old || new) and the new entropy
    step = 0.05 * torch.randn(len(th), generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    from rl_baselines.trpo import set_flat
    set_flat(pi_params(pol), torch.tensor(th) + step)
    with torch.no_grad():
        gain, kl, ent, surr = trpo_losses(pol, old, old_ls, obs, act, atarg, 0.01)
    want = ref.trial_losses(th + step.numpy(), D, A, discrete, obs.numpy(), act.numpy(), atarg.numpy(), old.numpy(), None if discrete else old_ls.numpy(), 0.01)
    for k, got in (("optimgain", gain), ("meankl", kl), ("meanent", ent), ("surrgain", surr)):
        assert abs(float(got) - want[k]) <= 1e-10 * (1 + abs(want[k])), k


@pytest.mark.parametrize("D", [1, 3, 12, 32])
@pytest.mark.parametrize("discrete", [True, False])
def test_double_backprop_fvp_equals_the_gauss_newton_form(D, discrete):
    from rl_baselines.trpo import flat, fvp_double_backprop, pi_params
    A = 6 if discrete else 3
    pol = _policy(D, A, discrete, D)
    obs, _, _ = _data(D, A, discrete, 200, D + 1)
    th = flat(pi_params(pol)).detach()
    v = torch.randn(len(th), generator=torch.Generator().manual_seed(D), dtype=torch.float64)
    got = fvp_double_backprop(pol, obs, v, 0.2).numpy()
    want = ref.fvp_gauss_newton(th.numpy(), D, A, discrete, obs.numpy(), v.numpy(), 0.2)
    np.testing.assert_allclose(got, want, rtol=1e-8, atol=1e-10 * np.abs(want).max())


def test_cg_matches_the_loop_and_breaks_on_the_tolerance():
    from rl_baselines.trpo import conjugate_gradient
    rng = np.random.default_rng(0)
    M = rng.standard_normal((12, 12)); M = M @ M.T + 0.5 * np.eye(12)
    b = rng.standard_normal(12)
    for iters in (1, 4, 10):
        x, n, its = conjugate_gradient(lambda p: torch.tensor(M) @ p, torch.tensor(b), iters)
        xm, nm, itm, _ = ref.cg_loop(lambda p: M @ p, b, iters)
        assert n == nm == iters
        np.testing.assert_allclose(x.numpy(), xm, rtol=1e-9)
    # the tolerance break: an exact solve in 2 iterations on a 2-dimensional problem, later iterations never run
    M2 = np.diag([1.0, 3.0]); b2 = np.array([1.0, 1.0])
    x, n, _ = conjugate_gradient(lambda p: torch.tensor(M2) @ p, torch.tensor(b2), 4)
    xm, nm, _, _ = ref.cg_loop(lambda p: M2 @ p, b2, 4)
    assert n == nm == 2
    np.testing.assert_allclose(x.numpy(), [1.0, 1 / 3.0], rtol=1e-12)
    shs, lm, fullstep = ref.step_size(xm, M2 @ xm, 0.01)
    assert abs(shs - 0.5 * (1 + 1 / 3.0)) < 1e-12 and np.allclose(fullstep, xm / np.sqrt(shs / 0.01))


def test_line_search_branches():
    from rl_baselines.trpo import line_search
    mk = lambda seq: (lambda s, it=iter(seq): next(it))
    # accept at the first trial
    assert line_search(mk([(1.0, 0.001)]), 0.5, None, 0.01)[0] == 0
    # KL violations, then accepted
    assert line_search(mk([(1.0, 0.5), (1.0, 0.016), (1.0, 0.015)]), 0.5, None, 0.01)[0] == 2
    # a negative improvement, then accepted
    assert line_search(mk([(0.4, 0.001), (0.5, 0.001)]), 0.5, None, 0.01)[0] == 1
    # a non-finite trial, then accepted
    assert line_search(mk([(float("nan"), 0.001), (0.6, float("inf")), (0.6, 0.0)]), 0.5, None, 0.01)[0] == 2
    # ten failures
    k, tried = line_search(mk([(0.0, 0.0)] * 10), 0.5, None, 0.01)
    assert k == -1 and len(tried) == 10
    # the model's decisions agree
    assert ref.decide(dict(optimgain=0.4, meankl=0.001, meanent=1.0), 0.5, 0.01) == "improve"
    assert ref.decide(dict(optimgain=0.6, meankl=0.02, meanent=1.0), 0.5, 0.01) == "kl"
    assert ref.decide(dict(optimgain=np.nan, meankl=0.0, meanent=1.0), 0.5, 0.01) == "nonfinite"


def test_mpi_adam_matches_the_ddpg_transcription():
    """The value optimiser against tests/ddpg_numpy_ref.py's MpiAdam (one learning rate: the whole vector is the 'actor'; tau 0)."""
    from ddpg_numpy_ref import mpi_adam_polyak_f32
    from rl_baselines.trpo import flat, mpi_adam
    g = torch.Generator().manual_seed(0)
    ps = [torch.randn(64, 3, generator=g), torch.randn(64, generator=g)]
    w0 = flat(ps).numpy().copy()
    m, v, t = torch.zeros(256), torch.zeros(256), torch.zeros(1, dtype=torch.int64)
    grads = [torch.randn(256, generator=g) for _ in range(5)]
    for gr in grads:
        mpi_adam(ps, gr, m, v, t, 2.5e-4)
    wm, _, mm, vm = mpi_adam_polyak_f32(w0, w0, [gr.numpy() for gr in grads], 256, 2.5e-4, 0.0, 0.0)
    np.testing.assert_array_equal(flat(ps).numpy(), wm)
    np.testing.assert_array_equal(m.numpy(), mm)
    np.testing.assert_array_equal(v.numpy(), vm)
    # and the model of tests/trpo_numpy_ref.py, step by step
    wr, mr, vr, tr = w0.astype(np.float32), np.zeros(256, np.float32), np.zeros(256, np.float32), 0
    for gr in grads:
        wr, mr, vr, tr = ref.mpi_adam_f32(wr, gr.numpy(), mr, vr, tr, 2.5e-4)
    np.testing.assert_array_equal(wr, wm)
    assert int(t) == tr == 5


@pytest.mark.parametrize("discrete", [True, False])
def test_policy_step_restores_theta_after_ten_rejections(discrete):
    from rl_baselines.trpo import TRPO_DEFAULTS, policy_step_torch
    D, A = 3, 6 if discrete else 3
    pol = _policy(D, A, discrete, 4).float()
    obs, act, adv = _data(D, A, discrete, 500, 6)
    obs, adv = obs.float(), adv.float()
    act = act if discrete else act.float()
    before = [p.detach().clone() for p in pol.parameters()]
    hp = dict(TRPO_DEFAULTS, cg_damping=-1e6)       # F - 1e6 I: the step points against the gradient, every trial loses gain
    rec = policy_step_torch(pol, obs, act, adv, obs[::5], hp)
    assert not rec["skip"] and rec["cg_iters"] >= 1 and rec["accepted"] == -1 and rec["restored"] and len(rec["trials"]) == 10
    assert all(torch.equal(a, b) for a, b in zip(before, pol.parameters()))
    # the defaults accept a step, and the policy moves to exactly theta_old + fullstep / 2^k
    from rl_baselines.trpo import flat, pi_params
    th = flat(pi_params(pol)).detach().clone()
    rec = policy_step_torch(pol, obs, act, adv, obs[::5], TRPO_DEFAULTS)
    assert rec["accepted"] >= 0 and not rec["restored"]
    assert torch.equal(flat(pi_params(pol)), th + rec["fullstep"] * 0.5 ** rec["accepted"])


def test_policy_step_skips_a_zero_gradient():
    from rl_baselines.trpo import TRPO_DEFAULTS, policy_step_torch
    pol = _policy(3, 6, True, 2).float()
    with torch.no_grad():
        pol.pi[4].bias[2] = 1e3                          # p = onehot(2) in float32, and every action is 2: d logp / d logits is exactly 0
    obs, _, adv = _data(3, 6, True, 200, 3)
    obs, adv = obs.float(), adv.float()
    before = [p.detach().clone() for p in pol.parameters()]
    rec = policy_step_torch(pol, obs, torch.full((200,), 2), adv, obs[::5], dict(TRPO_DEFAULTS, entcoeff=0.0))
    assert rec["skip"] and not bool(rec["g"].any()) and rec["cg_iters"] == 0 and "trials" not in rec
    assert all(torch.equal(a, b) for a, b in zip(before, pol.parameters()))


def test_value_minibatch_cadence():
    from rl_baselines.trpo import vf_minibatches
    assert vf_minibatches(128, 4) == [(0, 512)]
    assert vf_minibatches(300, 2) == [(0, 256), (256, 512)]
    assert vf_minibatches(127, 4) == []


@pytest.mark.parametrize("env_id,kw,stack", [("MobileRobotGymEnv-v0", dict(is_discrete=True, shape_reward=True), 1),
                                            ("KukaButtonGymEnv-v0", dict(is_discrete=False), 1),
                                            ("KukaButtonGymEnv-v0", dict(is_discrete=False, action_joints=True), 2)])
def test_trainer_on_the_oracle(use_oracle_backend, env_id, kw, stack):
    from rl_baselines import trpo
    T = 130
    hist = trpo.train(env_id, 2, 2 * T * 2, seed=2, env_kwargs=kw, verbose=0, device=None, hyperparams=dict(timesteps_per_batch=T), num_stack=stack)
    assert [h[0] for h in hist] == [2 * T, 4 * T]
    lu = trpo.train.last_update
    rec = lu["record"]
    assert not rec["skip"] and rec["cg_iters"] == 4 and (rec["accepted"] >= 0 or rec["restored"])
    assert int(lu["adam"][2]) == 2 * 3            # two updates x three epochs x one 128-step minibatch
    changed = [not torch.equal(a, b) for a, b in zip(lu["params0"], trpo.pi_params(trpo.train.last_policy) + trpo.vf_params(trpo.train.last_policy))]
    assert any(changed)


def _worker(rank, world, port, outdir):
    import sys
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from srl_sim import backend
    from srl_sim._abi import SimLibrary
    backend.use_library(SimLibrary(ORACLE_LIB), -1)
    from rl_baselines import trpo
    trpo.train("MobileRobotGymEnv-v0", 2, 2 * 128 * 2 * 2, seed=3, env_kwargs=dict(is_discrete=True, shape_reward=True), verbose=0,
               log_dir=os.path.join(outdir, "log"), device=None, hyperparams=dict(timesteps_per_batch=128))
    pol, norm, lu = trpo.train.last_policy, trpo.train.last_norm, trpo.train.last_update
    np.savez(os.path.join(outdir, "rank%d.npz" % rank), params=trpo.flat(list(pol.parameters())).detach().numpy(), mean=norm.mean.numpy(),
             var=norm.var.numpy(), count=norm.count.numpy(), m=lu["adam"][0].numpy(), v=lu["adam"][1].numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_trpo_keeps_replicas_identical(tmp_path, oracle_lib):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    a, b = [np.load(os.path.join(str(tmp_path), "rank%d.npz" % r)) for r in range(world)]
    for k in ("params", "mean", "var", "count", "m", "v"):
        assert np.array_equal(a[k], b[k]), k


def test_train_entry_point_trpo_and_replay(use_oracle_backend, tmp_path):
    from replay.enjoy_baselines import main as enjoy
    from rl_baselines.train import TRPO_OPT_PARAM, main, parserHyperParam
    names = ["timesteps_per_batch:64", "max_kl:0.02", "cg_iters:3", "gamma:0.9", "lam:0.9", "entcoeff:0.0", "cg_damping:0.1", "vf_stepsize:1e-3",
             "vf_iters:2"]
    assert parserHyperParam(names, TRPO_OPT_PARAM) == dict(timesteps_per_batch=64, max_kl=0.02, cg_iters=3, gamma=0.9, lam=0.9, entcoeff=0.0,
                                                           cg_damping=0.1, vf_stepsize=1e-3, vf_iters=2)
    with pytest.raises(AssertionError, match="not in list of valid hyperparameters"):
        parserHyperParam(["learning_rate:0.1"], TRPO_OPT_PARAM)
    log = str(tmp_path)
    hist = main(["--algo", "trpo", "--env", "MobileRobotGymEnv-v0", "--num-cpu", "4", "--num-timesteps", "200", "--hyperparam"] + names[:1] +
                ["--shape-reward", "--log-dir", log, "--device", "-1", "--seed", "4"])
    assert [h[0] for h in hist] == [256]
    run = glob.glob(os.path.join(log, "MobileRobotGymEnv-v0", "ground_truth", "trpo", "*"))[0]
    assert json.load(open(os.path.join(run, "args.json")))["algo"] == "trpo"
    for f in ("0.monitor.csv", "trpo_model.pt", "trpo_model_final.pt", "best_model.json"):
        assert os.path.isfile(os.path.join(run, f)), f
    n_done, _ = enjoy(["--log-dir", run, "--num-cpu", "4", "--num-timesteps", "260", "--device", "-1"])
    assert n_done >= 0
