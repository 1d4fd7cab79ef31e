"""
SAC trainer (rl_baselines/sac.py) without a GPU: the torch statement of the losses and of Adam + Polyak against the float64 models of
tests/sac_numpy_ref.py, the learn loop's cadence, and the trainer on the oracle backend (single process, two gloo ranks, the entry point
through replay).
"""
import glob
import json
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ORACLE_LIB, PKG
from sac_numpy_ref import adam_polyak_model, layout, sac_step_model
from test_ppo2_distributed_cpu import _free_port


def _batch(W, A, B, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    return r(B, W), torch.tanh(r(B, A)), r(B), r(B, W), (torch.rand(B, generator=g) < 0.2).double(), r(B, A)


def _torch_step(nets, batch, ent_coef):
    from rl_baselines.sac import sac_losses
    obs, act, rew, next_obs, done, eps = batch
    L = sac_losses(nets, obs, act, rew, next_obs, done, eps, 0.99, ent_coef, -float(nets.act_dim))
    return torch.autograd.grad(L["total"], nets.arena)[0].numpy(), L


@pytest.mark.parametrize("W,A", [(1, 2), (3, 3), (3, 7), (12, 7), (3, 2)])
@pytest.mark.parametrize("ent_coef", [None, 0.05])
def test_sac_losses_gradient_matches_the_float64_model(W, A, ent_coef):
    from rl_baselines.sac import SACNets
    torch.manual_seed(W * 10 + A)
    nets = SACNets(W, A).double()
    with torch.no_grad():
        nets.arena[-1] = 0.3                                   # log_ent_coef away from 0
        nets.target.add_(0.01 * torch.randn_like(nets.target))
        lay = nets.layout["actor"]
        b3 = lay["b3"][0]
        nets.arena[b3 + A] = -25.0                             # log_std of dim 0 below the clip
        nets.arena[b3 + A + 1] = 4.0                           # log_std of dim 1 above it
        nets.arena[b3] = 9.0                                   # mu of dim 0 saturates tanh
        w1, b1 = lay["w1"][0], lay["b1"][0]
        nets.arena[w1:w1 + W] = 0.0; nets.arena[b1] = 0.0       # hidden unit 0 of layer 1: pre-activation exactly 0 (ReLU at 0)
    batch = _batch(W, A, 50, W + A)
    got, L = _torch_step(nets, batch, ent_coef)
    want, ref = sac_step_model(nets.arena.detach().numpy(), nets.target.numpy(), W, A, *[x.numpy() for x in batch], 0.99, ent_coef, -float(A))
    np.testing.assert_allclose(L["q_backup"].numpy(), ref["q_backup"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(L["v_backup"].numpy(), ref["v_backup"], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(L["logp"].numpy(), ref["logp"], rtol=1e-10, atol=1e-10)
    nets_lay, P = layout(W, A)
    assert got.shape == (P,) and nets.layout["P"] == P
    for name, (off, n_in, n_out) in nets_lay.items():            # each group: actor, qf1, qf2, vf
        size = 64 * n_in + 64 + 64 * 64 + 64 + n_out * 64 + n_out
        np.testing.assert_allclose(got[off:off + size], want[off:off + size], rtol=1e-8, atol=1e-9 * np.abs(want[off:off + size]).max(), err_msg=name)
        assert np.abs(want[off:off + size]).max() > 0, name
    np.testing.assert_allclose(got[-1], want[-1], rtol=1e-10, atol=1e-12)
    assert (got[-1] == 0) == (ent_coef is not None)
    ls_head = nets.layout["actor"]["b3"][0] + A
    assert want[ls_head] == 0 and want[ls_head + 1] == 0       # the clipped log_std heads get no gradient


def _adam_polyak_against_the_model(warm):
    """One case of test_torch_adam_polyak_matches_the_float64_tf_model: ``warm`` torch steps before the compared ones."""
    from rl_baselines.sac import SACNets, adam_polyak
    W, A = 3, 3
    torch.manual_seed(0)
    nets = SACNets(W, A)
    m, v = torch.zeros_like(nets.arena), torch.zeros_like(nets.arena)
    beta_power = torch.tensor([0.9, 0.999], dtype=torch.float32)
    g = torch.Generator().manual_seed(1)
    for _ in range(warm):
        adam_polyak(nets, torch.randn(nets.arena.numel(), generator=g), m, v, beta_power, 3e-4, 0.005, polyak=True)
    arena0, target0 = nets.arena.detach().clone().numpy(), nets.target.clone().numpy()
    m0, v0 = m.clone().numpy(), v.clone().numpy()
    assert (np.abs(m0).max() > 0) == (warm > 0)
    grads = [torch.randn(nets.arena.numel(), generator=g) * (0.1 + k % 7) for k in range(100)]
    for k, gr in enumerate(grads):
        adam_polyak(nets, gr, m, v, beta_power, 3e-4, 0.005, polyak=True)
    w, tg, mm, vv = adam_polyak_model(arena0, target0, [x.numpy() for x in grads], W, A, 3e-4, 0.005, m=m0, v=v0, steps=warm)
    scale = 3e-4 * 100
    assert np.abs(nets.arena.detach().numpy() - w).max() < 1e-4 * scale
    assert np.abs(nets.target.numpy() - tg).max() < 1e-4 * scale
    np.testing.assert_allclose(m.numpy(), mm, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(v.numpy(), vv, rtol=1e-4, atol=1e-6)
    assert np.allclose(beta_power.numpy(), [0.9 ** (warm + 101), 0.999 ** (warm + 101)], rtol=1e-5)
    if warm:                                                   # the step count matters: the model one step off misses the first update
        w1, _, _, _ = adam_polyak_model(arena0, target0, [grads[0].numpy()], W, A, 3e-4, 0.005, m=m0, v=v0, steps=warm)
        w_off, _, _, _ = adam_polyak_model(arena0, target0, [grads[0].numpy()], W, A, 3e-4, 0.005, m=m0, v=v0, steps=warm - 1)
        assert np.abs(w_off - w1).max() > 100 * np.abs(w1).max() * 2.0 ** -24
    before = nets.target.clone()
    adam_polyak(nets, grads[0], m, v, beta_power, 3e-4, 0.005, polyak=False)
    assert torch.equal(nets.target, before)


def test_torch_adam_polyak_matches_the_float64_tf_model():
    """100 steps of the torch statement against the float64 model, from zero slots and from the slots, beta powers and target that 37
    earlier steps left (the model told only the slots and the step count)."""
    for warm in (0, 37):
        _adam_polyak_against_the_model(warm)


def test_cadence():
    from rl_baselines.sac import SAC_DEFAULTS, cadence
    hp = dict(SAC_DEFAULTS)
    assert [cadence(t, hp)[0] for t in (0, 99, 100)] == [True, True, False]
    assert [t for t in range(300) if cadence(t, hp)[1]] == list(range(99, 300)) and cadence(99, hp)[1] == [True]
    hp.update(train_freq=3, gradient_steps=2, target_update_interval=2, learning_starts=10, batch_size=20)
    steps = {t: cadence(t, hp)[1] for t in range(40) if cadence(t, hp)[1]}
    assert list(steps) == [21, 24, 27, 30, 33, 36, 39]              # t % 3 == 0 and t + 1 >= max(batch_size, learning_starts)
    assert steps[21] == [False, True] and steps[24] == [True, False]


def test_single_process_sac_runs_on_the_oracle_backend(use_oracle_backend):
    from rl_baselines import sac
    hp = dict(learning_starts=10, batch_size=4, buffer_size=30)
    for env_id, kw, stack in (("MobileRobotGymEnv-v0", dict(shape_reward=True, max_steps=20), 1), ("KukaButtonGymEnv-v0", {}, 1),
                              ("KukaButtonGymEnv-v0", dict(action_joints=True), 2)):
        phases = {}
        hist = sac.train(env_id, 4, 4 * 30, seed=1, env_kwargs=dict(is_discrete=False, **kw), verbose=0, device=None, hyperparams=hp, num_stack=stack,
                         phase_times=phases)
        assert [h[0] for h in hist] == [4 * k for k in range(1, 31)]
        assert sac.train.stats["grad_steps"] == 30 - 9 and sac.train.stats["target_updates"] == 21
        assert set(phases) == {"collect", "prepare", "gradient", "optimise"}
        nets = sac.train.last_nets
        assert bool(torch.isfinite(nets.arena).all()) and float(nets.log_ent_coef.detach()) != 0.0
        first = sac.train.last_before_first_step["arena"]
        assert not torch.equal(first, nets.arena.detach())
        ring = sac.train.last_ring
        assert torch.equal(ring["obs"][1:], ring["next_obs"][:-1]) or bool(ring["done"][:-1].any())
        assert float(ring["act"].abs().max()) <= 1.0
    with pytest.raises(ValueError, match="sac does not support discrete actions"):
        sac.train("MobileRobotGymEnv-v0", 4, 40, verbose=0, device=None, env_kwargs=dict(is_discrete=True))
    with pytest.raises(ValueError, match="no CPU fallback"):
        sac.train("MobileRobotGymEnv-v0", 4, 40, verbose=0, device=None, fused=True, env_kwargs=dict(is_discrete=False))


def _worker(rank, world, port, outdir):
    import sys
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from srl_sim import backend
    from srl_sim._abi import SimLibrary
    backend.use_library(SimLibrary(ORACLE_LIB), -1)
    from rl_baselines import sac
    hp = dict(learning_starts=6, batch_size=4, buffer_size=20, train_freq=2)
    hist = sac.train("MobileRobotGymEnv-v0", 4, 4 * 2 * 24, seed=3, env_kwargs=dict(is_discrete=False, shape_reward=True, max_steps=20),
                     verbose=0, log_dir=os.path.join(outdir, "log"), device=None, hyperparams=hp)
    nets, norm = sac.train.last_nets, sac.train.last_norm
    np.savez(os.path.join(outdir, "rank%d.npz" % rank), arena=nets.arena.detach().numpy(), target=nets.target.numpy(), mean=norm.mean.numpy(),
             count=norm.count.numpy(), steps=[h[0] for h in hist], grad_steps=sac.train.stats["grad_steps"])
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_sac_keeps_replicas_identical(tmp_path, oracle_lib):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    a, b = [np.load(os.path.join(str(tmp_path), "rank%d.npz" % r)) for r in range(world)]
    for k in ("arena", "target", "mean", "count"):
        assert np.array_equal(a[k], b[k]), k
    assert list(a["steps"]) == [16 * k for k in range(1, 13)] and int(a["grad_steps"]) == len(range(6, 24, 2))
    assert os.path.isfile(os.path.join(str(tmp_path), "log", "sac_model.pt"))


def test_train_entry_point_sac_and_replay(use_oracle_backend, tmp_path):
    from replay.enjoy_baselines import main as enjoy
    from rl_baselines.train import SAC_OPT_PARAM, main, parserHyperParam
    assert parserHyperParam(["ent_coef:0.1", "learning_rate:0.001", "gradient_steps:2", "train_freq:3"], SAC_OPT_PARAM) == \
        {"ent_coef": 0.1, "learning_rate": 0.001, "gradient_steps": 2, "train_freq": 3}
    for bad in ("batch_size:10", "tau:0.1", "buffer_size:10"):
        with pytest.raises(AssertionError, match="not in list of valid hyperparameters"):
            parserHyperParam([bad], SAC_OPT_PARAM)
    with pytest.raises(ValueError, match="^sac does not support discrete actions, please use the '--continuous-actions' \\(or '-c'\\) flag.$"):
        main(["--algo", "sac", "--device", "-1"])
    log = str(tmp_path)
    hist = main(["--algo", "sac", "-c", "--env", "MobileRobotGymEnv-v0", "--num-cpu", "4", "--num-timesteps", "200", "--hyperparam", "ent_coef:0.2",
                 "--buffer-size", "40", "--ent-coef", "0.5", "--batch-size", "8", "--shape-reward", "--log-dir", log, "--device", "-1", "--seed", "4"])
    assert [h[0] for h in hist] == [4 * k for k in range(1, 56)]    # 1.1 x 200 steps = 55 lockstep steps of 4 envs
    run = glob.glob(os.path.join(log, "MobileRobotGymEnv-v0", "ground_truth", "sac", "*"))[0]
    args = json.load(open(os.path.join(run, "args.json")))
    assert args["algo"] == "sac" and args["buffer_size"] == 40 and args["ent_coef"] == 0.2 and args["batch_size"] == 64
    for f in ("0.monitor.csv", "env_globals.json", "sac_model.pt", "sac_model_final.pt", "best_model.json"):
        assert os.path.isfile(os.path.join(run, f)), f
    for det in ([], ["--deterministic"]):
        n_done, _ = enjoy(["--log-dir", run, "--num-cpu", "4", "--num-timesteps", "260", "--device", "-1"] + det)
        assert n_done >= 4
