"""
GPU parity tests, MobileRobot family: the sm_90a kernels, called through the C-ABI, against
(1) golden vectors produced by the reference classes, (2) the CPU oracle on the same seeded inputs
(bit-exact: positions are float64, rewards/done integer-valued), (3) size-independent properties at
the BASELINE.json size (8192 envs x 1024 fused steps).
"""
import numpy as np
import pytest

from test_mobile_cpu import CASES, replay_golden_case

pytestmark = pytest.mark.gpu

KINDS = ["MobileRobotGymEnv-v0", "MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0",
         "MobileRobotLineTargetGymEnv-v0"]


@pytest.mark.parametrize("tag", sorted(CASES))
def test_reference_golden_through_cuda(tag, cuda_lib):
    from srl_sim import backend
    backend.use_library(None, None)  # product default: the CUDA library
    assert replay_golden_case(tag) in (251, 502)


def _run(backend, kind, n, T, acts, noise=None, stepwise=0, **cfg):
    sim = backend.make_sim(kind, n, **cfg)
    D = sim.obs_dim
    obs0 = backend.zeros((n, D), np.float32)
    sim.reset(obs_out=obs0, stream=backend.stream())
    obs = backend.zeros((T, n, D), np.float32); rew = backend.zeros((T, n), np.float32)
    done = backend.zeros((T, n), np.uint8)
    ep_ret = backend.zeros((T, n), np.float32); ep_len = backend.zeros((T, n), np.int32)
    a = None if acts is None else backend.from_host(acts)
    nz = None if noise is None else backend.from_host(noise)
    if stepwise:
        for t in range(T):
            sim.step(a[t], None if nz is None else nz[t], obs[t], rew[t], done[t], ep_ret[t], ep_len[t],
                     stream=backend.stream())
    else:
        sim.rollout(T, a, nz, obs, rew, done, ep_ret, ep_len, stream=backend.stream())
    out = dict(obs0=backend.to_host(obs0), obs=backend.to_host(obs), rew=backend.to_host(rew),
               done=backend.to_host(done), ep_ret=backend.to_host(ep_ret), ep_len=backend.to_host(ep_len),
               pos=sim.get_state(0), tgt=sim.get_state(1), counter=sim.get_state(2), stats=sim.get_state(9),
               launches=sim.launch_count)
    sim.close()
    return out


def _assert_same(a, b):
    for k in ("obs0", "obs", "rew", "done", "pos", "tgt", "counter", "stats"):
        assert np.array_equal(a[k], b[k]), k
    d = a["done"].astype(bool)
    assert np.array_equal(a["ep_ret"][d], b["ep_ret"][d]) and np.array_equal(a["ep_len"][d], b["ep_len"][d])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("random_target,shape_reward", [(False, False), (True, False), (True, True)])
def test_cuda_matches_oracle_discrete(kind, random_target, shape_reward, cuda_backend, oracle_backend):
    n, T = 1003, 530  # ragged batch (not a multiple of the block size), two auto-resets per env
    na = 2 if "1D" in kind else 4
    acts = np.random.RandomState(1).randint(0, na, size=(T, n)).astype(np.int32)
    cfg = dict(seed=1234, random_target=random_target, shape_reward=shape_reward)
    ref = _run(oracle_backend, kind, n, T, acts, **cfg)
    _assert_same(_run(cuda_backend, kind, n, T, acts, **cfg), ref)
    _assert_same(_run(cuda_backend, kind, n, 60, acts[:60], stepwise=1, **cfg), _run(oracle_backend, kind, n, 60, acts[:60], **cfg))


@pytest.mark.parametrize("kind", ["MobileRobotGymEnv-v0", "MobileRobotLineTargetGymEnv-v0"])
def test_cuda_matches_oracle_continuous(kind, cuda_backend, oracle_backend):
    n, T = 257, 300
    rs = np.random.RandomState(2)
    acts = rs.uniform(-1.5, 1.5, size=(T, n, 2)).astype(np.float32)
    noise = (rs.normal(0, 0.01, size=(T, n))).astype(np.float32)  # exercises the noise pointer (NOISE_STD is 0 in the reference)
    cfg = dict(seed=77, is_discrete=False, random_target=True, shape_reward=True)
    _assert_same(_run(cuda_backend, kind, n, T, acts, noise, **cfg), _run(oracle_backend, kind, n, T, acts, noise, **cfg))


@pytest.mark.parametrize("kind", KINDS)
def test_cuda_in_kernel_random_actions_match_oracle(kind, cuda_backend, oracle_backend):
    """actions=NULL: both sides draw the action from the env's Philox stream (integer-exact)."""
    cfg = dict(seed=99, random_target=True)
    _assert_same(_run(cuda_backend, kind, 300, 520, None, **cfg), _run(oracle_backend, kind, 300, 520, None, **cfg))


def test_cuda_edge_cases(cuda_backend, oracle_backend):
    # single env, single step; masked reset with host-supplied draws
    for n in (1, 2, 65):
        acts = np.zeros((1, n), np.int32)
        _assert_same(_run(cuda_backend, KINDS[0], n, 1, acts, seed=3), _run(oracle_backend, KINDS[0], n, 1, acts, seed=3))
    n = 40
    outs = []
    for be in (cuda_backend, oracle_backend):
        sim = be.make_sim(KINDS[0], n, seed=4, random_target=True)
        sim.reset(stream=be.stream())
        mask = np.zeros(n, np.uint8); mask[::3] = 1
        draws = np.random.RandomState(5).uniform(0.5, 3.5, size=(n, 6))
        obs = be.zeros((n, 2), np.float32)
        sim.reset(mask=be.from_host(mask), reset_draws=be.from_host(draws), obs_out=obs, stream=be.stream())
        outs.append((be.to_host(obs).copy(), sim.get_state(0), sim.get_state(1)))
        sim.close()
    for a, b in zip(outs[0], outs[1]):
        assert np.array_equal(a, b)
    assert np.array_equal(outs[0][1][::3, :2], np.random.RandomState(5).uniform(0.5, 3.5, size=(n, 6))[::3, :2])


def test_cuda_full_size_properties_and_sharding(cuda_backend):
    """BASELINE config 4 size: 8192 envs x 1024 fused steps, in-kernel actions."""
    kind, n, T = KINDS[0], 8192, 1024
    whole = _run(cuda_backend, kind, n, T, None, seed=2024, random_target=True)
    d = whole["done"].astype(bool)
    # every episode is exactly 251 steps: done at t = 250, 501, 752, 1003 for all envs
    expect = np.zeros(T, bool); expect[250::251] = True
    assert np.array_equal(d, np.repeat(expect[:, None], n, axis=1))
    assert (whole["ep_len"][d] == 251).all()
    assert set(np.unique(whole["rew"])) <= {-1.0, 0.0, 1.0}
    # Monitor-style return == sum of rewards of that episode
    assert np.array_equal(whole["ep_ret"][250], whole["rew"][:251].sum(0))
    # robot stays inside the walls minus the collision margin
    assert (whole["pos"][:, 0] >= 0.425).all() and (whole["pos"][:, 0] <= 3.575).all()
    assert (whole["pos"][:, 1] >= 0.2).all() and (whole["pos"][:, 1] <= 3.8).all()
    assert whole["launches"] == 2  # one reset + ONE fused rollout launch
    # sharding invariance: two half batches keyed by global env index == the whole batch
    lo = _run(cuda_backend, kind, n // 2, T, None, seed=2024, random_target=True, global_env_offset=0)
    hi = _run(cuda_backend, kind, n // 2, T, None, seed=2024, random_target=True, global_env_offset=n // 2)
    for k in ("obs", "rew", "done", "pos"):
        assert np.array_equal(whole[k], np.concatenate([lo[k], hi[k]], axis=-2 if k == "obs" else (1 if whole[k].ndim == 2 and k != "pos" else 0))), k


@pytest.mark.parametrize("host_chunks", [0, 3, 7])
def test_rollout_host_matches_device_rollout(cuda_backend, host_chunks, monkeypatch):
    """srl_sim_rollout_host pipelines the rollout in T-chunks (copy-in / kernel / copy-out streams); the chunking
    (here forced through SRL_HOST_CHUNKS, read when the handle first uses the host path) must not change a bit."""
    if host_chunks:
        monkeypatch.setenv("SRL_HOST_CHUNKS", str(host_chunks))
    else:
        monkeypatch.delenv("SRL_HOST_CHUNKS", raising=False)
    kind, n, T = KINDS[0], 512, 300
    acts = np.random.RandomState(8).randint(0, 4, size=(T, n)).astype(np.int32)
    dev = _run(cuda_backend, kind, n, T, acts, seed=6)
    sim = cuda_backend.make_sim(kind, n, seed=6)
    sim.reset(stream=cuda_backend.stream())
    import torch
    torch.cuda.synchronize()
    obs = np.zeros((T, n, 2), np.float32); rew = np.zeros((T, n), np.float32); done = np.zeros((T, n), np.uint8)
    launches0 = sim.launch_count
    sim.rollout_host(T, acts, None, obs, rew, done)
    assert np.array_equal(obs, dev["obs"]) and np.array_equal(rew, dev["rew"]) and np.array_equal(done, dev["done"])
    assert sim.last_kernel_ms() > 0
    assert sim.launch_count - launches0 == max(1, host_chunks)   # one launch per T-chunk


def test_rollout_host_pinned_buffers(cuda_backend, monkeypatch):
    """Pinned host input and output buffers: an unsplit srl_sim_rollout_host stages through HBM and copies out the same bits."""
    import torch
    monkeypatch.delenv("SRL_HOST_CHUNKS", raising=False)
    kind, n, T = KINDS[0], 512, 300
    acts = np.random.RandomState(9).randint(0, 4, size=(T, n)).astype(np.int32)
    dev = _run(cuda_backend, kind, n, T, acts, seed=7)
    sim = cuda_backend.make_sim(kind, n, seed=7)
    sim.reset(stream=cuda_backend.stream())
    torch.cuda.synchronize()
    obs = torch.full((T, n, 2), float("nan")).pin_memory(); rew = torch.full((T, n), float("nan")).pin_memory()
    done = torch.full((T, n), 255, dtype=torch.uint8).pin_memory()
    sim.rollout_host(T, torch.from_numpy(acts).pin_memory(), None, obs, rew, done)
    assert np.array_equal(obs.numpy(), dev["obs"]) and np.array_equal(rew.numpy(), dev["rew"]) and np.array_equal(done.numpy(), dev["done"])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("no_auto_reset", [False, True])
def test_cuda_ragged_counters_and_consecutive_rollouts(kind, no_auto_reset, cuda_backend, oracle_backend):
    """The episode-parallel rollout derives every segment boundary from the env's step counter: give each env a
    different counter (including values at and beyond max_steps), run three back-to-back rollouts whose lengths are
    not multiples of the episode length, and compare everything with the oracle's plain step loop (bit-exact)."""
    n, Ts = 333, (1, 260, 517)
    na = 2 if "1D" in kind else 4
    rs = np.random.RandomState(11)
    counters = rs.randint(0, 251, size=(n, 1)).astype(np.int32)
    counters[:8, 0] = [0, 1, 249, 250, 251, 252, 300, 125]
    outs = []
    for be in (cuda_backend, oracle_backend):
        sim = be.make_sim(kind, n, seed=21, random_target=True, shape_reward=(kind == KINDS[0]), no_auto_reset=no_auto_reset)
        D = sim.obs_dim
        sim.reset(stream=be.stream())
        sim.set_state(2, counters)
        res = []
        for T in Ts:
            acts = np.random.RandomState(T).randint(0, na, size=(T, n)).astype(np.int32)
            obs = be.zeros((T, n, D), np.float32); rew = be.zeros((T, n), np.float32); done = be.zeros((T, n), np.uint8)
            ep_ret = be.zeros((T, n), np.float32); ep_len = be.zeros((T, n), np.int32)
            sim.rollout(T, be.from_host(acts), None, obs, rew, done, ep_ret, ep_len, stream=be.stream())
            res.append([be.to_host(x).copy() for x in (obs, rew, done, ep_ret, ep_len)] +
                       [sim.get_state(f) for f in (0, 1, 2, 8, 9)])
        sim.close()
        outs.append(res)
    for a, b in zip(*outs):
        d = a[2].astype(bool)
        assert np.array_equal(a[2], b[2])
        for k in (0, 1, 5, 6, 7, 8, 9):
            assert np.array_equal(a[k], b[k]), k
        assert np.array_equal(a[3][d], b[3][d]) and np.array_equal(a[4][d], b[4][d])
