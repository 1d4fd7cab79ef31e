"""
DQN on CPU (rl_baselines/deepq.py): the torch statement of the update against the float64 / loop-form models of tests/deepq_numpy_ref.py, the
schedules and the learn loop's cadence, and the trainer on the oracle backend (single process, two gloo ranks, the
`python -m rl_baselines.train --algo deepq` entry point and replay).
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

from conftest import ORACLE_LIB, PKG
from deepq_numpy_ref import PrioritizedReplay, SegmentTree, clip_adam_model, double_q_model, dqn_grads_model
from test_consumer_reference_cpu import grad_bound, grad_errors
from test_ppo2_distributed_cpu import _free_port


def _qnet(width, n, seed=3):
    from rl_baselines.deepq import DuelingQ
    torch.manual_seed(seed)
    q = DuelingQ(width, n)
    with torch.no_grad():
        for p in q.parameters():
            p.add_(0.1 * torch.randn_like(p))
    return q


@pytest.mark.parametrize("width,n_act", [(3, 6), (2, 4), (1, 2), (12, 6)])
def test_torch_dqn_loss_gradient_matches_the_float64_model(width, n_act):
    """Autograd of rl_baselines.deepq.dqn_loss in float64 equals the hand-written backward pass to 1e-10 (dueling head, both Huber branches,
    ReLU units on and off, weights away from 1); float32 stays within the kernels' tolerance; dropping one row is far outside it."""
    from rl_baselines.deepq import dqn_loss
    q = _qnet(width, n_act)
    g = torch.Generator().manual_seed(8)
    B = 700
    obs = torch.randn(B, width, generator=g)
    obs[0] = 0.0                                            # first-layer pre-activations equal to the bias
    act = torch.randint(0, n_act, (B,), generator=g)
    with torch.no_grad():
        qa = q(obs).gather(1, act[:, None])[:, 0]
    y = qa + 1.5 * torch.randn(B, generator=g)
    w = 0.2 + torch.rand(B, generator=g)
    want, td = dqn_grads_model(q, obs.numpy(), act.numpy(), y.numpy(), w.numpy())
    assert (np.abs(td) < 1).any() and (np.abs(td) > 1).any()
    for dt in (torch.float64, torch.float32):
        p = copy.deepcopy(q).to(dt)
        loss, td_t = dqn_loss(p, obs.to(dt), act, y.to(dt), w.to(dt))
        loss.backward()
        errs = grad_errors([r.grad for r in p.parameters()], [torch.from_numpy(x) for x in want])
        for (name, _), (err, scale) in zip(p.named_parameters(), errs):
            assert scale > 0 and err <= (1e-10 * scale if dt == torch.float64 else grad_bound(scale)), (dt, name, err, scale)
        assert np.abs(td_t.double().numpy() - td).max() <= (1e-12 if dt == torch.float64 else 1e-5) * (np.abs(td).max() + 1)
    short, _ = dqn_grads_model(q, obs.numpy()[:-1], act.numpy()[:-1], y.numpy()[:-1], w.numpy()[:-1])
    assert max(err / grad_bound(scale) for err, scale in grad_errors([torch.from_numpy(x) for x in short], [torch.from_numpy(x) for x in want])) > 10


def test_relu_gradient_is_zero_at_a_zero_pre_activation():
    """TF's ReLU gradient is 0 where the pre-activation is <= 0: a unit with pre-activation exactly 0 passes nothing back."""
    from rl_baselines.deepq import dqn_loss
    q = _qnet(2, 3)
    with torch.no_grad():
        q.pi[0].bias.zero_(); q.vf[0].bias.zero_()
    obs = torch.zeros(4, 2)                                 # every first-layer pre-activation is exactly 0
    loss, _ = dqn_loss(q, obs, torch.tensor([0, 1, 2, 0]), torch.full((4,), 3.0), torch.ones(4))
    loss.backward()
    assert float(q.pi[0].weight.grad.abs().max()) == 0.0 and float(q.vf[0].bias.grad.abs().max()) == 0.0
    want, _ = dqn_grads_model(q, obs.numpy(), [0, 1, 2, 0], np.full(4, 3.0), np.ones(4))
    assert np.abs(want[0]).max() == 0.0


def test_double_q_target_and_argmax_ties():
    """The torch target against float64, and an exact tie in the online Q going to the lowest action index (tf.argmax)."""
    from rl_baselines.deepq import double_q_target
    online, target = _qnet(3, 4, seed=1), _qnet(3, 4, seed=2)
    g = torch.Generator().manual_seed(3)
    nxt, rew = torch.randn(500, 3, generator=g), torch.randn(500, generator=g)
    done = (torch.rand(500, generator=g) < 0.3).float()
    y = double_q_target(online, target, rew, done, nxt, 0.99)
    want, _ = double_q_model(online, target, rew.numpy(), done.numpy(), nxt.numpy(), 0.99)
    assert np.abs(y.double().numpy() - want).max() <= 1e-5 * (np.abs(want).max() + 1)
    with torch.no_grad():                                   # advantage head that ties actions 1 and 3, above 0 and 2
        for m in online.pi:
            if isinstance(m, torch.nn.Linear):
                m.weight.zero_(); m.bias.zero_()
        online.pi[-1].bias.copy_(torch.tensor([0.0, 1.0, -1.0, 1.0]))
        target.pi[-1].bias.copy_(torch.tensor([0.0, 5.0, 0.0, -5.0]))
    y = double_q_target(online, target, torch.zeros(2), torch.zeros(2), torch.zeros(2, 3), 1.0)
    assert torch.allclose(y, target(torch.zeros(2, 3))[:, 1])


@pytest.mark.parametrize("clip", [0.05, 1e3], ids=["clipped", "unclipped"])
def test_torch_clip_adam_matches_the_float64_tf_model(clip):
    from rl_baselines.deepq import clip_adam
    q = _qnet(3, 6)
    params = list(q.parameters())
    m, v = [torch.zeros_like(p) for p in params], [torch.zeros_like(p) for p in params]
    bp = torch.tensor([0.9, 0.999])
    p64 = [p.detach().double().numpy().copy() for p in params]
    m64, v64 = [np.zeros(p.shape) for p in params], [np.zeros(p.shape) for p in params]
    g = torch.Generator().manual_seed(5)
    for step in range(1, 101):
        for p in params:
            p.grad = torch.randn(p.shape, generator=g) * 0.05
        assert (max(float(torch.sqrt((p.grad.double() ** 2).sum())) for p in params) > clip) == (clip == 0.05)
        p64, m64, v64 = clip_adam_model(p64, [p.grad.numpy() for p in params], m64, v64, step, float(np.float32(1e-3)), clip,
                                        float(np.float32(0.9)), float(np.float32(0.999)), float(np.float32(1e-8)))
        clip_adam(params, m, v, bp, 1e-3, clip, 0.9, 0.999, 1e-8)
    for p, w in zip(params, p64):
        assert np.abs(p.detach().double().numpy() - w).max() <= 1e-3 * 100 * 2e-5 + 100 * 2.0 ** -23 * (np.abs(w).max() + 1.0)
    for mm, w in zip(m, m64):
        assert np.abs(mm.double().numpy() - w).max() <= 1e-5 * (np.abs(w).max() + 1e-6)
    assert abs(float(bp[0]) - 0.9 ** 101) < 1e-6


def test_replay_tree_matches_the_segment_tree_transcription():
    """rl_baselines.deepq.ReplayTree against baselines' SegmentTree loop form: inserts that wrap the ring, duplicates (last wins), max_priority,
    weights, find_prefixsum_idx on masses at and next to node boundaries, and the clamp of a walk into an empty leaf."""
    from rl_baselines.deepq import ReplayTree
    rows, N = 5, 7
    vec, loop = ReplayTree(rows, N, 0.6), PrioritizedReplay(rows, N, 0.6)
    rng = np.random.RandomState(0)
    for step in range(13):
        vec.add(step % rows); loop.add_row(step % rows)
        if step >= 1:
            u = rng.rand(40)
            i1, w1 = vec.sample(u, 0.5)
            i2, w2 = loop.sample(u, 0.5)
            assert np.array_equal(i1, i2) and np.array_equal(w1, w2)
            td = rng.randn(40).astype(np.float32) * 3
            i1[5:9] = i1[0]                              # a repeated index: the last occurrence's priority stays
            vec.update(i1, td, 1e-6); loop.update_priorities(i1, td, 1e-6)
            assert vec.sum[vec.tree_cap + i1[0]] == float(np.float32(abs(td[8])) + np.float32(1e-6)) ** 0.6 or i1[0] in i1[9:]
        s, m = loop.trees()
        assert np.array_equal(vec.sum[1:], s[1:]) and np.array_equal(vec.min[1:], m[1:]) and vec.max_priority == loop.max_priority
        assert vec.size == loop.size == min(step + 1, rows) * N
    # masses at and next to the boundaries between leaves (a total of 8: u = mass / 8 is exact): the walk goes right at equality, as `left > mass` says
    t = SegmentTree(8, lambda a, b: a + b, 0.0)
    for i, x in enumerate([1.0, 2.0, 0.5, 0.25, 4.25]):
        t[i] = x
    tree = ReplayTree(1, 8, 1.0)
    tree.sum[8:13] = [1.0, 2.0, 0.5, 0.25, 4.25]; tree.min[8:] = np.inf; tree.min[8:13] = tree.sum[8:13]
    tree._rebuild(0, 8); tree.size = 5
    cum = np.cumsum([1.0, 2.0, 0.5, 0.25, 4.25])
    masses = np.concatenate([cum[:-1], np.nextafter(cum[:-1], 0), np.nextafter(cum[:-1], 10)])
    want = [t.find_prefixsum_idx(x) for x in masses]
    got, _ = tree.sample(masses / tree.sum[1], 0.4)
    assert list(got) == want and want[:4] == [1, 2, 3, 4]
    # rounding that walks into an empty leaf is clamped to the last stored transition
    tree.sum[1] = np.nextafter(tree.sum[1], 100)          # a root a hair above its children's sum
    got, _ = tree.sample(np.array([1.0 - 2 ** -53]), 0.4)
    assert got[0] == 4


def test_schedules_and_cadence():
    """epsilon and beta follow LinearSchedule; gradient steps at t > learning_starts with t % train_freq == 0, copies at
    t % target_network_update_freq == 0; the trainer counts them so."""
    from rl_baselines.deepq import DQN_DEFAULTS, cadence, linear_schedule
    assert linear_schedule(100, 1.0, 0.01, 0) == 1.0 and linear_schedule(100, 1.0, 0.01, 50) == pytest.approx(0.505)
    assert linear_schedule(100, 1.0, 0.01, 1000) == pytest.approx(0.01) and linear_schedule(1000, 0.4, 1.0, 500) == pytest.approx(0.7)
    hp = dict(DQN_DEFAULTS)
    steps = [t for t in range(2000) if cadence(t, hp)[0]]
    copies = [t for t in range(2000) if cadence(t, hp)[1]]
    assert steps[0] == 504 and all(b - a == 4 for a, b in zip(steps, steps[1:])) and copies == [1000, 1500]


def test_single_process_deepq_runs_on_the_oracle_backend(use_oracle_backend):
    from rl_baselines import deepq
    hp = dict(learning_starts=10, target_network_update_freq=8, buffer_size=50)
    hist = deepq.train("MobileRobotGymEnv-v0", 8, 8 * 60, seed=1, env_kwargs=dict(is_discrete=True, shape_reward=True, max_steps=20), verbose=0,
                       device=None, hyperparams=hp)
    assert [h[0] for h in hist] == [32 * k for k in range(1, 16)]
    assert {k: deepq.train.stats[k] for k in ('grad_steps', 'target_copies')} == dict(grad_steps=len([t for t in range(31, 60) if t % 4 == 0]), target_copies=len([t for t in range(11, 60) if t % 8 == 0]))
    assert all(np.isfinite(h[1]) for h in hist[5:])              # the first episodes end at step 20
    rep = deepq.train.last_replay
    assert rep.max_priority > 1.0 and rep.size == 50 * 8
    hist = deepq.train("KukaButtonGymEnv-v0", 4, 4 * 40, seed=1, env_kwargs=dict(is_discrete=True), verbose=0, device=None,
                       hyperparams=dict(hp, prioritized_replay=False), num_stack=2)
    assert len(hist) == 10 and deepq.train.stats["grad_steps"] == 2
    assert deepq.train.last_replay.max_priority == 1.0
    with pytest.raises(ValueError, match="does not support continuous actions"):
        deepq.train("MobileRobotGymEnv-v0", 8, 80, verbose=0, device=None, env_kwargs=dict(is_discrete=False))
    with pytest.raises(ValueError, match="no CPU fallback"):
        deepq.train("MobileRobotGymEnv-v0", 8, 80, verbose=0, device=None, fused=True)


def _worker(rank, world, port, outdir):
    import sys
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from srl_sim import backend
    from srl_sim._abi import SimLibrary
    backend.use_library(SimLibrary(ORACLE_LIB), -1)
    from rl_baselines import deepq
    hp = dict(learning_starts=10, target_network_update_freq=8, buffer_size=40)
    hist = deepq.train("MobileRobotGymEnv-v0", 8, 8 * 2 * 48, seed=3, env_kwargs=dict(is_discrete=True, shape_reward=True, max_steps=20),
                       verbose=0, log_dir=os.path.join(outdir, "log"), device=None, hyperparams=hp)
    flat = torch.cat([p.detach().reshape(-1) for p in deepq.train.last_policy.parameters()]).numpy()
    tflat = torch.cat([p.detach().reshape(-1) for p in deepq.train.last_target.parameters()]).numpy()
    norm = deepq.train.last_norm
    np.savez(os.path.join(outdir, "rank%d.npz" % rank), params=flat, target=tflat, mean=norm.mean.numpy(), count=norm.count.numpy(),
             steps=[h[0] for h in hist], grad_steps=deepq.train.stats["grad_steps"])
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_deepq_keeps_replicas_identical(tmp_path, oracle_lib):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    a, b = [np.load(os.path.join(str(tmp_path), "rank%d.npz" % r)) for r in range(world)]
    for k in ("params", "target", "mean", "count"):
        assert np.array_equal(a[k], b[k]), k
    assert float(a["count"]) == pytest.approx(2 * 8 * 48 + 2 * 8 + 1e-4)
    assert list(a["steps"]) == [64 * k for k in range(1, 13)] and int(a["grad_steps"]) > 0
    assert os.path.isfile(os.path.join(str(tmp_path), "log", "deepq_model.pt"))


def test_train_entry_point_deepq_and_replay(use_oracle_backend, tmp_path):
    from replay.enjoy_baselines import main as enjoy
    from rl_baselines.train import DQN_OPT_PARAM, main, parserHyperParam
    assert parserHyperParam(["train_freq:2", "exploration_fraction:0.5"], DQN_OPT_PARAM) == {"train_freq": 2, "exploration_fraction": 0.5}
    with pytest.raises(AssertionError, match="not in list of valid hyperparameters"):
        parserHyperParam(["buffer_size:10"], DQN_OPT_PARAM)
    with pytest.raises(ValueError, match="deepq does not support continuous actions, please remove the '--continuous-actions' \\(or '-c'\\) flag."):
        main(["--algo", "deepq", "-c", "--device", "-1"])
    for prioritized, stack in (("1", "1"), ("0", "2")):
        log = os.path.join(str(tmp_path), prioritized)
        hist = main(["--algo", "deepq", "--env", "MobileRobotGymEnv-v0", "--num-cpu", "4", "--num-timesteps", "280", "--hyperparam", "learning_starts:20",
                     "train_freq:2", "--prioritized", prioritized, "--dueling", "0", "--buffer-size", "60", "--num-stack", stack, "--shape-reward",
                     "--log-dir", log, "--device", "-1", "--seed", "4"])
        assert [h[0] for h in hist] == [8 * k for k in range(1, 39)] + [308]      # 1.1 x 280 steps = 77 lockstep steps of 4 envs, periods of 2
        run = glob.glob(os.path.join(log, "MobileRobotGymEnv-v0", "ground_truth", "deepq", "*"))[0]
        args = json.load(open(os.path.join(run, "args.json")))
        assert args["algo"] == "deepq" and args["buffer_size"] == 60 and args["prioritized_replay"] == (prioritized == "1")
        assert args["train_freq"] == 2 and args["num_stack"] == int(stack)
        for f in ("0.monitor.csv", "env_globals.json", "deepq_model.pt", "deepq_model_final.pt", "best_model.json"):
            assert os.path.isfile(os.path.join(run, f)), f
        n_done, _ = enjoy(["--log-dir", run, "--num-cpu", "4", "--num-timesteps", "260", "--device", "-1"])
        assert n_done >= 4
