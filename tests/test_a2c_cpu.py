"""
A2C on CPU (rl_baselines/a2c.py): the torch statement of the update against the float64 numpy model of tests/a2c_numpy_ref.py, the trainer
on the oracle backend (single process, two gloo ranks, the `python -m rl_baselines.train --algo a2c` entry point and replay).
"""
import copy
import glob
import json
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from a2c_numpy_ref import a2c_grads_model, a2c_returns_model, clip_rmsprop_model, scheduler_values
from conftest import ORACLE_LIB, PKG
from test_consumer_reference_cpu import gae_rollout, grad_bound, grad_errors, ppo2_policy, ppo2_rollout
from test_ppo2_distributed_cpu import _free_port

A2C_SHAPES = [(True, 3, 6), (True, 1, 2), (False, 3, 7), (False, 2, 2), (False, 12, 2)]


@pytest.mark.parametrize("discrete,obs_dim,n_out", A2C_SHAPES)
def test_torch_a2c_loss_gradient_matches_the_float64_model(discrete, obs_dim, n_out):
    """Autograd of rl_baselines.a2c.a2c_loss in float64 equals the hand-written numpy backward pass to 1e-10; float32 autograd stays within
    the kernels' tolerance of it; dropping one row moves the model far outside that tolerance."""
    from rl_baselines.a2c import a2c_loss
    pol = ppo2_policy(obs_dim, discrete, n_out, "cpu")
    d = ppo2_rollout(pol, 700, seed=3)
    args = (d["obs"], d["act"], d["ret"], d["old_val"])
    want = a2c_grads_model(pol, *(a.numpy() for a in args), 0.01, 0.5)
    for dt in (torch.float64, torch.float32):
        p = copy.deepcopy(pol).to(dt)
        cast = lambda t: t if t.dtype == torch.int64 else t.to(dt)
        a2c_loss(p, *(cast(a) for a in args), 0.01, 0.5).backward()
        got = [q.grad for q in p.parameters()]
        errs = grad_errors(got, [torch.from_numpy(w) for w in want])
        for (name, _), (err, scale) in zip(p.named_parameters(), errs):
            assert scale > 0 and err <= (1e-10 * scale if dt == torch.float64 else grad_bound(scale)), (dt, name, err, scale)
    keep = [a[:-1] for a in args]
    short = a2c_grads_model(pol, *(a.numpy() for a in keep), 0.01, 0.5)
    assert max(err / grad_bound(scale) for err, scale in grad_errors([torch.from_numpy(w) for w in short],
                                                                     [torch.from_numpy(w) for w in want])) > 10.0


@pytest.mark.parametrize("max_grad_norm", [0.5, 1e3], ids=["clipped", "unclipped"])
def test_torch_clip_rmsprop_matches_the_float64_model(max_grad_norm):
    """rl_baselines.a2c.clip_rmsprop over 100 steps (slots from 1.0) against the float64 TF model, with the norm above max_grad_norm
    (clipped) and below it."""
    from rl_baselines.a2c import clip_rmsprop
    pol = ppo2_policy(3, False, 2, "cpu")
    params = list(pol.parameters())
    ms = [torch.ones_like(p) for p in params]
    p64, m64 = [p.detach().double().numpy().copy() for p in params], [m.double().numpy().copy() for m in ms]
    g = torch.Generator().manual_seed(5)
    lr = torch.tensor(7e-4)
    for step in range(100):
        for p in params:
            p.grad = torch.randn(p.shape, generator=g) * 0.05
        norm = float(torch.sqrt(sum((p.grad.double() ** 2).sum() for p in params)))
        assert (norm > max_grad_norm) == (max_grad_norm == 0.5)
        # the hyper-parameters as the float32 graph holds them (1 - fl32(0.99) is 1e-6 away from 0.01)
        p64, m64 = clip_rmsprop_model(p64, [p.grad.numpy() for p in params], m64, float(lr), max_grad_norm, float(np.float32(0.99)), float(np.float32(1e-5)))
        clip_rmsprop(params, ms, lr, max_grad_norm, 0.99, 1e-5)
    for p, w, m, mw in zip(params, p64, ms, m64):
        # ms rounds once per step and forgets at rate 1 - alpha: up to ~1 / (1 - alpha) float32 ulps of error
        assert np.abs(m.double().numpy() - mw).max() <= 100 * 2.0 ** -24 * np.abs(mw).max()
        # every step adds a float32 rounding of the parameter; a step moves it by about lr
        assert np.abs(p.detach().double().numpy() - w).max() <= 100 * 2.0 ** -23 * (np.abs(w).max() + 1.0)
    assert m64[0].max() < 0.9                  # the slots left their initial 1.0


@pytest.mark.parametrize("bad", [float("inf"), float("nan")], ids=["inf", "nan"])
def test_torch_clip_rmsprop_non_finite_gradient_makes_every_parameter_nan(bad):
    from rl_baselines.a2c import clip_rmsprop
    pol = ppo2_policy(3, True, 6, "cpu")
    params = list(pol.parameters())
    for p in params:
        p.grad = torch.randn(p.shape) * 0.05
    params[0].grad[0, 0] = bad
    clip_rmsprop(params, [torch.ones_like(p) for p in params], torch.tensor(7e-4), 0.5, 0.99, 1e-5)
    assert all(torch.isnan(p).all() for p in params)


@pytest.mark.parametrize("schedule", ["constant", "linear", "middle_drop", "double_linear_con", "double_middle_drop"])
def test_learning_rate_schedules_match_a_per_sample_scheduler(schedule):
    from rl_baselines.a2c import A2C_DEFAULTS, learning_rate
    hp = dict(A2C_DEFAULTS, lr_schedule=schedule)
    n_batch, total = 40, 40 * 23 + 7
    want = scheduler_values(hp["learning_rate"], total, schedule, n_batch, 23)
    got = [learning_rate(hp, k, n_batch, total) for k in range(23)]
    assert np.allclose(got, want, rtol=1e-12, atol=0)
    if schedule != "constant":
        assert len(set(np.round(got, 12))) > 2


def test_returns_recursion_matches_discount_with_dones():
    """The trainer's torch recursion and GAE with lambda = 1 (the recursion srl_ppo2_gae runs) both give the A2C runner's returns."""
    from test_consumer_reference_cpu import gae_model
    rew, val, done, last_val = gae_rollout(9, 64, "cpu", seed=2)
    want = a2c_returns_model(rew.numpy(), done.numpy(), last_val.numpy(), 0.99)
    assert done[0].sum() > 0 and done[-1].sum() > 0
    _, ret = gae_model(rew.numpy(), val.numpy(), done.numpy(), last_val.numpy(), 0.99, 1.0)
    assert np.abs(ret - want).max() <= 1e-12 * np.abs(want).max()


def test_single_process_a2c_runs_on_the_oracle_backend(use_oracle_backend):
    from rl_baselines import a2c
    pt = {}
    hist = a2c.train("MobileRobotGymEnv-v0", 16, 16 * 5 * 30, seed=1, env_kwargs=dict(is_discrete=True, shape_reward=True, max_steps=20),
                     verbose=0, device=None, phase_times=pt)
    assert [h[0] for h in hist] == [80 * k for k in range(1, 31)]
    assert all(np.isfinite(h[1]) and h[1] < 0 for h in hist[6:])
    assert set(pt) == {"collect", "grad", "optimise"}
    ms = a2c.train.last_ms
    assert all(torch.isfinite(m).all() for m in ms) and float(ms[0].max()) < 1.0
    hist_c = a2c.train("MobileRobotGymEnv-v0", 8, 8 * 5 * 2, seed=2, env_kwargs=dict(is_discrete=False, max_steps=20), verbose=0, device=None,
                       num_stack=2, hyperparams=dict(lr_schedule="linear"))
    assert len(hist_c) == 2
    with pytest.raises(ValueError, match="no CPU fallback"):
        a2c.train("MobileRobotGymEnv-v0", 8, 80, verbose=0, device=None, fused=True)
    with pytest.raises(ValueError, match="lr_schedule"):
        a2c.train("MobileRobotGymEnv-v0", 8, 80, verbose=0, device=None, hyperparams=dict(lr_schedule="cosine"))


def _worker(rank, world, port, outdir):
    import sys
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from srl_sim import backend
    from srl_sim._abi import SimLibrary
    backend.use_library(SimLibrary(ORACLE_LIB), -1)
    from rl_baselines import a2c
    hist = a2c.train("MobileRobotGymEnv-v0", 8, 8 * 5 * 2 * 4, seed=3, env_kwargs=dict(is_discrete=True, shape_reward=True, max_steps=20),
                     verbose=0, log_dir=os.path.join(outdir, "log"), device=None)
    policy, norm = a2c.train.last_policy, a2c.train.last_norm
    flat = torch.cat([p.detach().reshape(-1) for p in policy.parameters()]).numpy()
    ms = torch.cat([m.reshape(-1) for m in a2c.train.last_ms]).numpy()
    np.savez(os.path.join(outdir, "rank%d.npz" % rank), params=flat, ms=ms, mean=norm.mean.numpy(), count=norm.count.numpy(),
             steps=[h[0] for h in hist])
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_a2c_keeps_replicas_identical(tmp_path, oracle_lib):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    a, b = [np.load(os.path.join(str(tmp_path), "rank%d.npz" % r)) for r in range(world)]
    for k in ("params", "ms", "mean", "count"):
        assert np.array_equal(a[k], b[k]), k
    assert float(a["count"]) == pytest.approx(4 * 2 * 8 * 5 + 2 * 8 + 1e-4)
    assert list(a["steps"]) == [80, 160, 240, 320]
    assert os.path.isfile(os.path.join(str(tmp_path), "log", "a2c_model.pt"))


def test_train_entry_point_a2c_and_replay(use_oracle_backend, tmp_path):
    from replay.enjoy_baselines import main as enjoy
    from rl_baselines.train import A2C_OPT_PARAM, main, parserHyperParam
    assert parserHyperParam(["alpha:0.9", "lr_schedule:linear"], A2C_OPT_PARAM) == {"alpha": 0.9, "lr_schedule": "linear"}
    with pytest.raises(AssertionError, match="not in list of valid hyperparameters"):
        parserHyperParam(["cliprange:0.1"], A2C_OPT_PARAM)
    hist = main(["--algo", "a2c", "--env", "MobileRobotGymEnv-v0", "--num-cpu", "8", "--num-timesteps", "300", "--hyperparam", "n_steps:4", "alpha:0.95",
                 "--lr-schedule", "middle_drop", "--shape-reward", "--log-dir", str(tmp_path), "--device", "-1", "--seed", "4"])
    assert [h[0] for h in hist] == [32 * k for k in range(1, 11)]       # 1.1 x 300 steps in updates of 8 envs x 4 steps
    run = glob.glob(os.path.join(str(tmp_path), "MobileRobotGymEnv-v0", "ground_truth", "a2c", "*"))[0]
    args = json.load(open(os.path.join(run, "args.json")))
    assert args["algo"] == "a2c" and args["n_steps"] == 4 and args["alpha"] == 0.95 and args["lr_schedule"] == "middle_drop" and args["epsilon"] == 1e-5
    assert os.path.isfile(os.path.join(run, "0.monitor.csv"))
    assert os.path.isfile(os.path.join(run, "a2c_model.pt")) and os.path.isfile(os.path.join(run, "a2c_model_final.pt"))
    n_done, _ = enjoy(["--log-dir", run, "--num-cpu", "4", "--num-timesteps", "260", "--device", "-1"])
    assert n_done >= 4                                                  # every MobileRobot episode lasts 251 steps
