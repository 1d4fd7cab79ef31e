"""
CPU tests of PPO2 on stacked state observations (``rl_baselines.ppo2.train(..., num_stack=k)``, ``--num-stack k``), on the CPU oracle backend:
  - the rows the trainer feeds the policy are ``VecNormalize(VecFrameStack(...))`` of rl_baselines/utils.py on the same raw observations and dones;
  - ``args.json`` records ``num_stack`` and ``replay.enjoy_baselines`` replays a stacked model;
  - the CPU checker of the policy step (policy_core.h, oracle/libpolicy_ref.so) at the wide widths the sm_90a kernels now take, against float64;
  - data-parallel PPO2 (world size 2, gloo) with a stacked row keeps the replicas and the merged filter identical.
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
from test_consumer_reference_cpu import policy_model
from test_policy_cpu import _policy, _ref_act, ref  # noqa: F401  (ref: the module fixture of the CPU checker)
from test_ppo2_distributed_cpu import _free_port


class _Replay(object):
    """A VecEnv that replays recorded raw observations and dones, to drive the host-side wrappers."""

    def __init__(self, first, steps):
        from srl_sim import spaces
        self.first, self.steps, self.num_envs = first, steps, first.shape[0]
        self.observation_space = spaces.Box(low=-np.inf, high=np.inf, shape=(first.shape[1],), dtype=np.float32)
        self.action_space = None

    def reset(self):
        return self.first.copy()

    def step(self, t):
        obs, done = self.steps[t]
        return obs.copy(), np.zeros(self.num_envs, np.float32), done.astype(bool), [{} for _ in range(self.num_envs)]


def _record_rollout(monkeypatch):
    """Hooks that record what the trainer feeds the policy and what the envs returned, step by step."""
    from rl_baselines.ppo2 import MlpPolicy, RunningNorm
    from srl_sim.vec_env import BatchedSRLVecEnv
    fed, raw, rows = [], [], []
    act, step, filt = MlpPolicy.act, BatchedSRLVecEnv.step_tensors, RunningNorm.__call__

    def filt_rec(self, x, update=True):
        if update:
            rows.append(x.detach().clone().numpy())
        return filt(self, x, update)

    def act_rec(self, obs):
        fed.append(obs.detach().clone().numpy())
        return act(self, obs)

    def step_rec(self, actions, noise=None):
        if not raw:
            raw.append(np.array(self._obs, copy=True))            # the reset observation
        out = step(self, actions, noise)
        raw.append((np.array(self._obs, copy=True), np.array(self._done, copy=True)))
        return out
    monkeypatch.setattr(MlpPolicy, "act", act_rec)
    monkeypatch.setattr(BatchedSRLVecEnv, "step_tensors", step_rec)
    monkeypatch.setattr(RunningNorm, "__call__", filt_rec)
    return fed, raw, rows


@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("env_id,env_kwargs", [("MobileRobotGymEnv-v0", dict(is_discrete=True, max_steps=10)),
                                               ("KukaButtonGymEnv-v0", dict(is_discrete=True, max_steps=12))], ids=["mobile", "kuka"])
def test_trainer_feeds_the_policy_vecnormalize_of_vecframestack(use_oracle_backend, monkeypatch, env_id, env_kwargs, k):
    """One rollout of 24 steps with short episodes (several dones per env), unfused collection on the oracle: the stacked rows the trainer's filter
    folds in are VecFrameStack's byte for byte, and every row the policy saw is the host wrappers' output on the same raw observation and done
    sequence, within 1e-6 (scaled up on columns with a tiny spread, see below)."""
    from rl_baselines import ppo2
    from rl_baselines.utils import VecFrameStack, VecNormalize
    fed, raw, rows = _record_rollout(monkeypatch)
    N, T = 6, 24
    ppo2.train(env_id, N, N * T, seed=5, env_kwargs=env_kwargs, hyperparams=dict(n_steps=T, noptepochs=1), verbose=0, cuda_graph=False, device=None,
               num_stack=k)
    assert len(fed) == T and len(raw) == T + 1
    dones = np.stack([d for _, d in raw[1:]])
    assert dones.sum() >= N and dones[:-1].any(axis=0).all()              # every env finished an episode inside the rollout
    D = raw[0].shape[1]
    host = VecNormalize(VecFrameStack(_Replay(raw[0], raw[1:]), k), norm_obs=True, norm_reward=False)
    assert len(rows) == T + 1                                              # the reset batch and one per step
    for t in range(T):
        want = host.reset() if t == 0 else host.step(t - 1)[0]
        assert np.array_equal(rows[t], host.venv.stackedobs)
        # The host RunningMeanStd takes the batch moments of a float32 array in float32 (numpy) and normalises in float64; the trainer takes them
        # in float64 and normalises in float32.  Either way a float32 rounding of the mean, ~6e-8 |mean|, is divided by the column's spread:
        # 1e-6 holds where the spread is 0.1 or more, and the tolerance grows as 0.1 / std below that (Kuka's z column).
        std = np.sqrt(host.obs_rms.var)
        tol = 1e-6 * np.maximum(1.0, 0.1 / std)
        assert fed[t].shape == (N, k * D)
        assert (np.abs(fed[t] - want) <= tol).all(), (t, (np.abs(fed[t] - want) / tol).max())
    # a done env's row is zero but for its newest frame at the step after the done, in the raw stack the filter saw
    stack = host.venv.stackedobs
    last_done = dones[T - 2].astype(bool)
    if last_done.any():
        assert (stack[last_done, :(k - 1) * D] == 0).all()


def test_args_json_records_num_stack_and_enjoy_replays_a_stacked_model(use_oracle_backend, tmp_path):
    """`python -m rl_baselines.train --num-stack 3` on the oracle: args.json holds num_stack, the saved policy and filter are 3 D wide, and
    replay.enjoy_baselines rebuilds the stack and replays the model."""
    from rl_baselines.train import main
    hist = main(["--algo", "ppo2", "--env", "MobileRobotGymEnv-v0", "--num-cpu", "8", "--num-timesteps", "300", "--hyperparam", "n_steps:16",
                 "noptepochs:1", "--num-stack", "3", "--log-dir", str(tmp_path), "--device", "-1", "--seed", "2"])
    assert [h[0] for h in hist] == [128, 256]
    run = glob.glob(os.path.join(str(tmp_path), "MobileRobotGymEnv-v0", "ground_truth", "ppo2", "*"))[0]
    assert json.load(open(os.path.join(run, "args.json")))["num_stack"] == 3
    saved = torch.load(os.path.join(run, "ppo2_model.pt"))
    assert saved["obs_mean"].numel() == 3 * 2 and saved["policy"]["pi.0.weight"].shape == (64, 6)
    from replay.enjoy_baselines import main as enjoy
    with open(os.path.join(run, "env_globals.json")) as f:
        g = json.load(f)
    g["max_steps"] = 30                                                    # short episodes, so that the replay finishes some
    with open(os.path.join(run, "env_globals.json"), "w") as f:
        json.dump(g, f)
    n_done, mean_reward = enjoy(["--log-dir", run, "--num-cpu", "4", "--num-timesteps", "70", "--device", "-1"])
    assert n_done >= 4 and np.isfinite(mean_reward)
    with pytest.raises(AssertionError, match="num-stack"):
        main(["--env", "MobileRobotGymEnv-v0", "--num-stack", "0", "--device", "-1"])


def test_num_stack_one_records_one_and_wide_rows_need_the_unfused_paths(use_oracle_backend, tmp_path):
    """k = 1 is recorded too; a row wider than 32 is refused up front when a fused path is asked for (the kernels take at most 32 values)."""
    from rl_baselines import ppo2
    ppo2.train("MobileRobotGymEnv-v0", 4, 4 * 16, seed=0, hyperparams=dict(n_steps=16, noptepochs=1), verbose=0, cuda_graph=False, device=None,
               log_dir=str(tmp_path))
    assert json.load(open(str(tmp_path / "args.json")))["num_stack"] == 1
    with pytest.raises(ValueError, match="at most 32"):
        ppo2.train("KukaButtonGymEnv-v0", 4, 4 * 16, seed=0, hyperparams=dict(n_steps=16), verbose=0, device=None, num_stack=11, fused_act=True)


@pytest.mark.parametrize("discrete,n_out", [(True, 6), (False, 3), (False, 7)])
@pytest.mark.parametrize("obs_dim", [9, 12, 17, 32])
def test_checker_policy_step_at_wide_widths_matches_float64(ref, obs_dim, discrete, n_out):  # noqa: F811
    """The CPU checker the GPU tests hold the wide kernels to: value and policy outputs within float32 rounding of a float64 model of the towers."""
    pol = _policy(obs_dim, discrete, n_out, seed=300 + obs_dim)
    obs = torch.randn(2000, obs_dim, generator=torch.Generator().manual_seed(obs_dim)) * 1.5
    act_env, act_buf, logp, val, out = _ref_act(ref, pol, obs, seed=3, counter=1)
    out64, v64 = policy_model(pol, obs.numpy())
    assert np.abs(out - out64).max() <= 2e-5 * max(1.0, np.abs(out64).max())
    assert np.abs(val - v64).max() <= 2e-5 * max(1.0, np.abs(v64).max())
    if discrete:
        assert act_env.min() >= 0 and act_env.max() < n_out and np.array_equal(act_env, act_buf.astype(np.int32))
    else:
        assert np.array_equal(act_env, np.clip(act_buf, -1.0, 1.0))


def _worker(rank, world, port, outdir):
    import sys
    sys.path.insert(0, PKG)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from srl_sim import backend
    from srl_sim._abi import SimLibrary
    backend.use_library(SimLibrary(ORACLE_LIB), -1)
    from rl_baselines import ppo2
    ppo2.train("MobileRobotGymEnv-v0", 8, 8 * 16 * 2 * 2, seed=3, env_kwargs=dict(is_discrete=True, shape_reward=True, max_steps=20),
               hyperparams=dict(n_steps=16), verbose=0, cuda_graph=False, device=None, num_stack=2)
    policy, norm = ppo2.train.last_policy, ppo2.train.last_norm
    flat = torch.cat([p.detach().reshape(-1) for p in policy.parameters()]).numpy()
    np.savez(os.path.join(outdir, "rank%d.npz" % rank), params=flat, mean=norm.mean.numpy(), var=norm.var.numpy(), count=norm.count.numpy(),
             w1=policy.pi[0].weight.shape[1])
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_ppo2_with_stacked_rows_keeps_replicas_identical(tmp_path, oracle_lib):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    a, b = [np.load(os.path.join(str(tmp_path), "rank%d.npz" % r)) for r in range(world)]
    assert int(a["w1"]) == 2 * 2 and a["mean"].shape == (4,)          # MobileRobot's 2-D state, two frames
    assert np.array_equal(a["params"], b["params"])
    for k in ("mean", "var", "count"):
        assert np.array_equal(a[k], b[k]), k
    assert float(a["count"]) == pytest.approx(2 * 2 * 8 * 16 + 2 * 8 + 1e-4)
