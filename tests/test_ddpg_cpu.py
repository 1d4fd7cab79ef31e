"""
DDPG trainer (rl_baselines/ddpg.py) without a GPU: the torch statement of the losses, of MpiAdam + Polyak and of the Ornstein-Uhlenbeck step
against the models of tests/ddpg_numpy_ref.py, the cycle, and the trainer on the oracle backend (single process, two gloo ranks, the entry
point through replay, the refusals).
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
from ddpg_numpy_ref import ddpg_step_model, layout, mpi_adam_polyak_f32, ou_model
from test_ppo2_distributed_cpu import _free_port


def _batch(W, A, B, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    obs, next_obs = 4 * r(B, W), 4 * r(B, W)                   # many inputs beyond +-5: the clip
    return obs, torch.tanh(r(B, A)), r(B), next_obs, (torch.rand(B, generator=g) < 0.2).double()


@pytest.mark.parametrize("W,A", [(1, 2), (3, 3), (3, 7), (12, 7), (32, 7), (2, 8)])
def test_ddpg_losses_gradient_matches_the_float64_model(W, A):
    from rl_baselines.ddpg import DDPGNets, ddpg_losses
    torch.manual_seed(W * 10 + A)
    nets = DDPGNets(W, A).double()
    lay = nets.layout
    with torch.no_grad():
        nets.arena.add_(0.05 * torch.randn_like(nets.arena))
        nets.target.copy_(nets.arena + 0.02 * torch.randn_like(nets.arena))
        nets.arena[lay["actor"]["b3"][0]] = 40.0                 # the actor's head 0 saturates tanh
        for name in ("actor", "critic"):                         # hidden unit 0 of layer 1: pre-activation exactly 0 (ReLU at 0)
            w1, b1 = lay[name]["w1"][0], lay[name]["b1"][0]
            nets.arena[w1:w1 + W] = 0.0; nets.arena[b1] = 0.0
    obs, act, rew, next_obs, done = _batch(W, A, 60, W + A)
    assert (obs.abs() > 5).any() and (next_obs.abs() > 5).any()
    for l2 in (0.0, 1e-2, 0.5):
        L = ddpg_losses(nets, obs, act, rew, next_obs, done, 0.99, 1.5, l2)
        got = torch.autograd.grad(L["total"], nets.arena)[0].numpy()
        want, ref = ddpg_step_model(nets.arena.detach().numpy(), nets.target.numpy(), W, A, obs.numpy(), act.numpy(), rew.numpy(), next_obs.numpy(),
                                    done.numpy(), 0.99, 1.5, l2)
        np.testing.assert_allclose(L["y"].numpy(), ref["y"], rtol=1e-12, atol=1e-12)
        ref_lay, P = layout(W, A)
        assert got.shape == (P,) and lay["P"] == P
        for name in ("actor", "critic"):
            for key in ("w1", "b1", "w2", "b2", "w3", "b3"):
                off, shape = ref_lay[name][key]
                n = int(np.prod(shape))
                np.testing.assert_allclose(got[off:off + n], want[off:off + n], rtol=1e-9, atol=1e-12 * (1 + np.abs(want[off:off + n]).max()),
                                           err_msg="%s.%s" % (name, key))
        assert np.abs(want[:lay["actor"]["end"]]).max() > 0 and np.abs(want[lay["actor"]["end"]:]).max() > 0
        assert np.all(ref["d_actor"][:, 0] == 0)                 # the saturated head passes no gradient
    # L2 on exactly the critic's two hidden kernels: the gradients at l2 = 0.5 and 0 differ by 0.5 w there and nowhere else
    g = [torch.autograd.grad(ddpg_losses(nets, obs, act, rew, next_obs, done, 0.99, 1.5, l2)["total"], nets.arena)[0].numpy() for l2 in (0.0, 0.5)]
    diff, w = g[1] - g[0], nets.arena.detach().numpy()
    mask = np.zeros(lay["P"], bool)
    for key in ("w1", "w2"):
        off, shape = lay["critic"][key]
        mask[off:off + int(np.prod(shape))] = True
    np.testing.assert_allclose(diff[mask], 0.5 * w[mask], rtol=1e-9, atol=1e-12)
    assert np.all(diff[~mask] == 0)


def _mpi_adam_polyak_against_the_statement(warm):
    """One case of test_torch_mpi_adam_polyak_gives_the_bytes_of_the_numpy_float32_statement: ``warm`` torch steps before the compared ones."""
    from rl_baselines.ddpg import DDPGNets, mpi_adam_polyak
    W, A = 3, 3
    torch.manual_seed(0)
    nets = DDPGNets(W, A)
    with torch.no_grad():
        nets.target.add_(0.01 * torch.randn_like(nets.target))
    m, v, t = torch.zeros_like(nets.arena), torch.zeros_like(nets.arena), torch.zeros(1, dtype=torch.int64)
    g = torch.Generator().manual_seed(1)
    for _ in range(warm):
        mpi_adam_polyak(nets, torch.randn(nets.arena.numel(), generator=g), m, v, t, 1e-4, 1e-3, 0.001)
    arena0, target0, m0, v0 = nets.arena.detach().clone().numpy(), nets.target.clone().numpy(), m.clone().numpy(), v.clone().numpy()
    assert int(t[0]) == warm and (np.abs(m0).max() > 0) == (warm > 0)
    grads = [torch.randn(nets.arena.numel(), generator=g) * (0.1 + k % 7) for k in range(100)]
    for gr in grads:
        mpi_adam_polyak(nets, gr, m, v, t, 1e-4, 1e-3, 0.001)
    w, tg, mm, vv = mpi_adam_polyak_f32(arena0, target0, [x.numpy() for x in grads], nets.layout["actor"]["end"], 1e-4, 1e-3, 0.001, m=m0, v=v0,
                                        steps=warm)
    for got, want in ((nets.arena.detach(), w), (nets.target, tg), (m, mm), (v, vv)):
        assert got.numpy().dtype == want.dtype == np.float32
        assert np.array_equal(got.numpy(), want)
    assert int(t[0]) == warm + 100
    assert not np.array_equal(w, arena0) and not np.array_equal(tg, target0)
    if warm:                                                   # the step count is part of the statement: one off gives other bytes
        w_off, _, _, _ = mpi_adam_polyak_f32(arena0, target0, [grads[0].numpy()], nets.layout["actor"]["end"], 1e-4, 1e-3, 0.001, m=m0, v=v0,
                                             steps=warm - 1)
        w1, _, _, _ = mpi_adam_polyak_f32(arena0, target0, [grads[0].numpy()], nets.layout["actor"]["end"], 1e-4, 1e-3, 0.001, m=m0, v=v0,
                                          steps=warm)
        assert not np.array_equal(w_off, w1)


def test_torch_mpi_adam_polyak_gives_the_bytes_of_the_numpy_float32_statement():
    """100 updates of the torch statement give the bytes of the numpy float32 transcription, from zero slots and from the slots, target
    and step count that 37 earlier updates left."""
    for warm in (0, 37):
        _mpi_adam_polyak_against_the_statement(warm)


def test_ou_step_and_its_reset_match_numpy():
    from rl_baselines.ddpg import OU_DT, OU_THETA, ou_step
    g = torch.Generator().manual_seed(3)
    n, A = 50, 7
    state = torch.zeros(n, A)
    x64 = np.zeros((n, A))
    for k in range(30):
        z = torch.randn(n, A, generator=g)
        prev = (torch.rand(n, generator=g) < 0.1).to(torch.uint8) if k else torch.zeros(n, dtype=torch.uint8)
        ou_step(state, z, prev, 0.2)
        x64 = ou_model(x64, z.double().numpy(), prev.numpy(), 0.2, OU_THETA, OU_DT)
        np.testing.assert_allclose(state.double().numpy(), x64, rtol=1e-5, atol=1e-6)
        if k and prev.any():                                     # a reset env starts from 0: its state is the one noise term
            r = prev.bool().numpy()
            np.testing.assert_allclose(state.numpy()[r], (0.2 * np.sqrt(0.01) * z.double().numpy())[r], rtol=1e-6, atol=1e-7)


def test_cadence():
    from rl_baselines.ddpg import DDPG_DEFAULTS, cadence
    hp = dict(DDPG_DEFAULTS)
    assert [t for t in range(450) if cadence(t, hp)] == [99, 199, 299, 399] and cadence(99, hp) == 100
    hp.update(nb_rollout_steps=3, nb_train_steps=5)
    assert [(t, cadence(t, hp)) for t in range(10) if cadence(t, hp)] == [(2, 5), (5, 5), (8, 5)]
    # the blocks of rl_baselines.offpolicy.learn (G = R, or 2 R for an odd R when captured) start at multiples of G: every full block has
    # one pattern of gradient steps, so the shared graph rule replays every full block after the first gradient step
    for R, G in ((3, 6), (3, 3), (4, 4), (100, 100)):
        hp.update(nb_rollout_steps=R)
        assert len({tuple(cadence(t, hp) for t in range(t0, t0 + G)) for t0 in range(0, 30 * G, G)}) == 1


@pytest.mark.parametrize("noise", ["ou", "normal", "none"])
def test_single_process_ddpg_runs_on_the_oracle_backend(use_oracle_backend, noise):
    from rl_baselines import ddpg
    hp = dict(nb_rollout_steps=5, nb_train_steps=3, batch_size=4, buffer_size=12, noise_action=noise)
    for env_id, kw, stack in (("MobileRobotGymEnv-v0", dict(shape_reward=True, max_steps=8), 1), ("KukaButtonGymEnv-v0", {}, 1),
                              ("KukaButtonGymEnv-v0", dict(action_joints=True), 2)):
        phases = {}
        hist = ddpg.train(env_id, 4, 4 * 23, seed=1, env_kwargs=dict(is_discrete=False, **kw), verbose=0, device=None, hyperparams=hp, num_stack=stack,
                          phase_times=phases)
        assert [h[0] for h in hist] == [4 * 5 * k for k in range(1, 5)] + [4 * 23]
        assert ddpg.train.stats["grad_steps"] == 4 * 3
        assert set(phases) == {"collect", "prepare", "gradient", "optimise"}
        nets = ddpg.train.last_nets
        assert bool(torch.isfinite(nets.arena).all()) and int(ddpg.train.last_adam[2][0]) == 12
        assert not torch.equal(ddpg.train.last_before_first_step["arena"], nets.arena.detach())
        assert not torch.equal(nets.target, nets.arena.detach()) and not torch.equal(nets.target, ddpg.train.last_before_first_step["target"])
        ring = ddpg.train.last_ring
        assert float(ring["act"].abs().max()) <= 1.0
        assert (float(ddpg.train.last_ou.abs().max()) > 0) == (noise == "ou")
        if env_id.startswith("Mobile"):
            assert bool(ring["done"].any())                      # max_steps 8: episodes end, and the OU state restarts there


def test_refusals(use_oracle_backend):
    from rl_baselines import ddpg
    with pytest.raises(ValueError, match="ddpg does not support discrete actions"):
        ddpg.train("MobileRobotGymEnv-v0", 4, 40, verbose=0, device=None, env_kwargs=dict(is_discrete=True))
    with pytest.raises(ValueError, match="--noise-param"):
        ddpg.train("MobileRobotGymEnv-v0", 4, 40, verbose=0, device=None, env_kwargs=dict(is_discrete=False), noise_param=True)
    with pytest.raises(ValueError, match="no CPU fallback"):
        ddpg.train("MobileRobotGymEnv-v0", 4, 40, verbose=0, device=None, fused=True, env_kwargs=dict(is_discrete=False))


def _worker(rank, world, port, outdir):
    import sys
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from srl_sim import backend
    from srl_sim._abi import SimLibrary
    backend.use_library(SimLibrary(ORACLE_LIB), -1)
    from rl_baselines import ddpg
    hp = dict(nb_rollout_steps=4, nb_train_steps=2, batch_size=4, buffer_size=10)
    hist = ddpg.train("MobileRobotGymEnv-v0", 4, 4 * 2 * 20, seed=3, env_kwargs=dict(is_discrete=False, shape_reward=True, max_steps=20),
                      verbose=0, log_dir=os.path.join(outdir, "log"), device=None, hyperparams=hp)
    nets, norm = ddpg.train.last_nets, ddpg.train.last_norm
    np.savez(os.path.join(outdir, "rank%d.npz" % rank), arena=nets.arena.detach().numpy(), target=nets.target.numpy(), mean=norm.mean.numpy(),
             var=norm.var.numpy(), count=norm.count.numpy(), steps=[h[0] for h in hist], grad_steps=ddpg.train.stats["grad_steps"])
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_ddpg_keeps_replicas_identical(tmp_path, oracle_lib):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    a, b = [np.load(os.path.join(str(tmp_path), "rank%d.npz" % r)) for r in range(world)]
    for k in ("arena", "target", "mean", "var", "count"):
        assert np.array_equal(a[k], b[k]), k
    assert list(a["steps"]) == [32 * k for k in range(1, 6)] and int(a["grad_steps"]) == 5 * 2
    assert os.path.isfile(os.path.join(str(tmp_path), "log", "ddpg_model.pt"))


def test_train_entry_point_ddpg_and_replay(use_oracle_backend, tmp_path):
    from replay.enjoy_baselines import main as enjoy
    from rl_baselines.train import DDPG_OPT_PARAM, main, parserHyperParam
    assert parserHyperParam(["noise_action:normal", "noise_action_sigma:0.3", "nb_train_steps:7", "actor_lr:0.001", "tau:0.01"], DDPG_OPT_PARAM) == \
        dict(noise_action="normal", noise_action_sigma=0.3, nb_train_steps=7, actor_lr=0.001, tau=0.01)
    for bad in ("buffer_size:10", "memory_limit:10", "learning_rate:0.1"):
        with pytest.raises(AssertionError, match="not in list of valid hyperparameters"):
            parserHyperParam([bad], DDPG_OPT_PARAM)
    with pytest.raises(ValueError, match="^ddpg does not support discrete actions, please use the '--continuous-actions' \\(or '-c'\\) flag.$"):
        main(["--algo", "ddpg", "--device", "-1"])
    with pytest.raises(ValueError, match="--noise-param"):
        main(["--algo", "ddpg", "-c", "--noise-param", "--env", "MobileRobotGymEnv-v0", "--num-cpu", "4", "--device", "-1", "--log-dir", str(tmp_path)])
    log = str(tmp_path)
    hist = main(["--algo", "ddpg", "-c", "--env", "MobileRobotGymEnv-v0", "--num-cpu", "4", "--num-timesteps", "200", "--memory-limit", "5",
                 "--hyperparam", "nb_rollout_steps:10", "nb_train_steps:2", "noise_action:normal", "--noise-action", "none", "--noise-action-sigma",
                 "0.4", "--batch-size", "8", "--shape-reward", "--log-dir", log, "--device", "-1", "--seed", "4"])
    assert [h[0] for h in hist] == [40 * k for k in range(1, 6)] + [220]   # 1.1 x 200 steps = 55 lockstep steps of 4 envs
    run = glob.glob(os.path.join(log, "MobileRobotGymEnv-v0", "ground_truth", "ddpg", "*"))[0]
    args = json.load(open(os.path.join(run, "args.json")))
    assert args["algo"] == "ddpg" and args["buffer_size"] == 100 and args["batch_size"] == 8 and args["nb_train_steps"] == 2
    assert args["noise_action"] == "normal" and args["noise_action_sigma"] == 0.4          # --hyperparam wins over --noise-action
    for f in ("0.monitor.csv", "env_globals.json", "ddpg_model.pt", "ddpg_model_final.pt", "best_model.json"):
        assert os.path.isfile(os.path.join(run, f)), f
    n_done, _ = enjoy(["--log-dir", run, "--num-cpu", "4", "--num-timesteps", "260", "--device", "-1"])
    assert n_done >= 4
