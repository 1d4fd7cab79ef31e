"""
GPU parity tests, Kuka button-push family: the fp32 sm_90a kernel, called through the C-ABI, against the
float64 CPU oracle on the same (seed, action, noise) sequences.

Tolerances (BASELINE.json north_star / SURVEY.md section 8(d)): gripper / end-effector position <= 1e-3 m,
joint positions <= 1e-3 rad, joint velocities <= 1e-2 rad/s over 1000 steps; reward and done flags bit-exact.
PARITY UNPINNED at the PyBullet boundary (see oracle/oracle_kuka.cpp header).
"""
import importlib.util
import os

import numpy as np
import pytest

from conftest import GOLDEN
from srl_sim import _abi
from srl_sim.model import load_kuka_scene

pytestmark = pytest.mark.gpu

POS_TOL, Q_TOL, QD_TOL = 1e-3, 1e-3, 1e-2


def _gen():
    spec = importlib.util.spec_from_file_location("gen_kuka_golden", os.path.join(GOLDEN, "gen_kuka_golden.py"))
    gen = importlib.util.module_from_spec(spec); spec.loader.exec_module(gen)
    return gen


def _run(be, kind, n, T, acts, noise, chunk=None, stepwise=False, **cfg):
    sim = be.make_sim(kind, n, model_blob=load_kuka_scene().blob, **cfg)
    obs0 = be.zeros((n, 3), np.float32)
    sim.reset(obs_out=obs0, stream=be.stream())
    obs = be.zeros((T, n, 3), np.float32); rew = be.zeros((T, n), np.float32); done = be.zeros((T, n), np.uint8)
    ep_ret = be.zeros((T, n), np.float32); ep_len = be.zeros((T, n), np.int32)
    a = None if acts is None else be.from_host(acts)
    nz = None if noise is None else be.from_host(noise)
    snaps = []
    chunk = 1 if stepwise else (chunk or T)
    for s in range(0, T, chunk):
        e = min(T, s + chunk)
        if stepwise:
            sim.step(a[s], None if nz is None else nz[s], obs[s], rew[s], done[s], ep_ret[s], ep_len[s], stream=be.stream())
        else:
            sim.rollout(e - s, None if a is None else a[s:e], None if nz is None else nz[s:e], obs[s:e], rew[s:e],
                        done[s:e], ep_ret[s:e], ep_len[s:e], stream=be.stream())
        if chunk != T and not stepwise:
            snaps.append((sim.get_state(_abi.F_JOINT_POS), sim.get_state(_abi.F_JOINT_VEL), sim.get_state(_abi.F_EE_POS)))
    out = dict(obs0=be.to_host(obs0).copy(), obs=be.to_host(obs).copy(), rew=be.to_host(rew).copy(),
               done=be.to_host(done).copy(), ep_ret=be.to_host(ep_ret).copy(), ep_len=be.to_host(ep_len).copy(),
               q=sim.get_state(_abi.F_JOINT_POS), qd=sim.get_state(_abi.F_JOINT_VEL), ee=sim.get_state(_abi.F_EE_POS),
               grip=sim.get_state(_abi.F_ROBOT_POS), target=sim.get_state(_abi.F_TARGET_POS),
               counters=sim.get_state(_abi.F_COUNTERS), counter=sim.get_state(_abi.F_STEP_COUNTER),
               glider=sim.get_state(_abi.F_BUTTON_GLIDER), snaps=snaps, launches=sim.launch_count,
               two=sim.get_state(_abi.F_TWO_BUTTON))
    sim.close()
    return out


def _assert_parity(c, o, flags_exact=True):
    assert np.abs(c["obs0"] - o["obs0"]).max() < POS_TOL
    if flags_exact:
        assert np.array_equal(c["done"], o["done"]), "done flags differ"
        assert np.array_equal(c["rew"] == 1, o["rew"] == 1) and np.array_equal(c["rew"] == -1, o["rew"] == -1)
    d = o["done"].astype(bool)
    assert np.array_equal(c["ep_len"][d], o["ep_len"][d])
    assert np.abs(c["obs"] - o["obs"]).max() < POS_TOL                 # gripper position relative to the target
    assert np.abs(c["grip"] - o["grip"]).max() < POS_TOL and np.abs(c["ee"] - o["ee"]).max() < POS_TOL
    assert np.abs(c["q"] - o["q"]).max() < Q_TOL and np.abs(c["qd"] - o["qd"]).max() < QD_TOL
    assert np.array_equal(c["counters"], o["counters"]) and np.array_equal(c["counter"], o["counter"])
    for (qc, qdc, eec), (qo, qdo, eeo) in zip(c["snaps"], o["snaps"]):
        assert np.abs(qc - qo).max() < Q_TOL and np.abs(qdc - qdo).max() < QD_TOL and np.abs(eec - eeo).max() < POS_TOL


def test_config2_discrete_1000_steps_vs_oracle(cuda_backend, oracle_backend):
    """SURVEY 8(d) config 2 on envs 0..63: 1000 random discrete actions + N(0, 0.01) step noise."""
    n, T = 64, 1000
    acts = np.random.default_rng(0).integers(0, 6, (T, n), dtype=np.int32)
    noise = np.random.default_rng(1).normal(0, 0.01, (T, n)).astype(np.float32)
    cfg = dict(seed=0, is_discrete=True, random_target=False, force_down=True, action_repeat=1, max_distance=0.8)
    c = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, chunk=100, **cfg)
    o = _run(oracle_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, chunk=100, **cfg)
    _assert_parity(c, o)
    assert o["done"].sum() >= n                                          # every env finished at least one episode


def test_config5_continuous_random_target_2000_steps_vs_oracle(cuda_backend, oracle_backend):
    """SURVEY 8(d) config 5 flavour: KukaRandButton, continuous actions, randomised button, 2000 steps."""
    n, T = 32, 2000
    acts = np.random.default_rng(0).uniform(-1, 1, (T, n, 3)).astype(np.float32)
    noise = np.random.default_rng(1).normal(0, 1e-4, (T, n)).astype(np.float32)
    cfg = dict(seed=5, is_discrete=False, random_target=True)
    c = _run(cuda_backend, "KukaRandButtonGymEnv-v0", n, T, acts, noise, chunk=250, **cfg)
    o = _run(oracle_backend, "KukaRandButtonGymEnv-v0", n, T, acts, noise, chunk=250, **cfg)
    _assert_parity(c, o)
    assert o["done"].sum() >= n                                          # >= 1 forced reset per env (1001-step limit)
    assert np.abs(o["target"][:, 0] - 0.5).max() <= 0.15 + 1e-6 and np.abs(o["target"][:, 1]).max() <= 0.3 + 1e-6


@pytest.mark.parametrize("cfg", [
    dict(is_discrete=True, shape_reward=True, action_repeat=2),
    dict(is_discrete=False, shape_reward=True, random_target=True),
    dict(is_discrete=True, force_down=False, max_steps=60),
])
def test_variants_vs_oracle(cfg, cuda_backend, oracle_backend):
    n, T = 16, 300
    rs = np.random.RandomState(3)
    if cfg.get("is_discrete", True):
        acts = rs.randint(-1, 6, size=(T, n)).astype(np.int32)           # includes step(None) (-1)
        noise = rs.normal(0, 0.01, size=(T, n)).astype(np.float32)
    else:
        acts = rs.uniform(-1, 1, size=(T, n, 3)).astype(np.float32)
        noise = rs.normal(0, 1e-4, size=(T, n)).astype(np.float32)
    c = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, seed=9, **cfg)
    o = _run(oracle_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, seed=9, **cfg)
    _assert_parity(c, o, flags_exact=not cfg.get("shape_reward", False))
    assert np.array_equal(c["done"], o["done"])
    if cfg.get("shape_reward", False):
        assert np.abs(c["rew"] - o["rew"]).max() < POS_TOL                # reward = -distance


@pytest.mark.parametrize("in_kernel_actions", [False, True])
def test_action_joints_vs_oracle(in_kernel_actions, cuda_backend, oracle_backend):
    """action_joints=True (kuka_button_gym_env.py:317-323, kuka.py:158-161): 7 joint set-points relative to the initial
    joint vector, no IK; its own 500-step settle snapshot and N(7, 1) random-init offsets.  max_steps=150 forces resets."""
    n, T = 24, 400
    rs = np.random.RandomState(12)
    acts = None if in_kernel_actions else np.clip(np.cumsum(rs.normal(0, 0.2, size=(T, n, 7)), axis=0), -1, 1).astype(np.float32)
    noise = None if in_kernel_actions else rs.normal(0, 0.002, size=(T, n)).astype(np.float32)
    cfg = dict(seed=31, is_discrete=False, action_joints=True, max_steps=150)
    c = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, **cfg)
    o = _run(oracle_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, **cfg)
    _assert_parity(c, o)
    assert o["done"].sum() >= 2 * n
    assert np.abs(o["q"][:, :7] - np.asarray(load_kuka_scene().q_init)[:7]).max() < 0.2   # +-DELTA_THETA around the initial posture


@pytest.mark.parametrize("cfg", [dict(is_discrete=True, force_down=True), dict(is_discrete=True, force_down=True, random_target=True, shape_reward=True)])
def test_two_button_kind_vs_oracle(cfg, cuda_backend, oracle_backend):
    """Kuka2ButtonGymEnv-v0 (kuka_2button_gym_env.py): second button body, goal switching, two-stage reward / termination, IK damping 0.5.
    A greedy controller stepped on the ORACLE produces the action sequence (so both buttons do get pressed); the CUDA kernel then
    replays it as fused rollouts and must agree on everything, including the per-button contact counters and the goal index."""
    n, T = 16, 900
    kind = "Kuka2ButtonGymEnv-v0"
    full = dict(seed=17, max_distance=2.0, **cfg)
    blob = load_kuka_scene().blob
    sim = oracle_backend.make_sim(kind, n, model_blob=blob, **full)
    obs = np.zeros((n, 3), np.float32); rew = np.zeros(n, np.float32); done = np.zeros(n, np.uint8)
    sim.reset(obs_out=obs)
    rs = np.random.RandomState(5)
    acts = np.zeros((T, n), np.int32); noise = rs.normal(0, 0.01, size=(T, n)).astype(np.float32)
    goals = []
    for t in range(T):
        ax, ay = np.abs(obs[:, 0]), np.abs(obs[:, 1])
        a = np.where(np.maximum(ax, ay) < 0.02, 4, np.where(ax > ay, np.where(obs[:, 0] > 0, 0, 1), np.where(obs[:, 1] > 0, 2, 3)))
        rnd = rs.rand(n) < 0.15
        a[rnd] = rs.randint(0, 6, size=rnd.sum())
        acts[t] = a
        sim.step(acts[t], noise[t], obs, rew, done)
        goals.append(sim.get_state(_abi.F_TWO_BUTTON)[:, 2].copy())
    sim.close()
    assert np.max(goals) == 1                                             # the first button was pressed, the goal moved on
    c = _run(cuda_backend, kind, n, T, acts, noise, **full)
    o = _run(oracle_backend, kind, n, T, acts, noise, **full)
    assert o["done"].sum() >= n // 2
    # Per env: identical flags and rewards (1e-3 on the shaped -distance) up to the first difference, if any; a difference must be
    # the documented one-step shift of a contact ONSET (fp32 vs fp64 on the 0.02 m manifold margin, see _parity_until_first_flag_shift):
    # one side reports a contact reward (1 / 25 / 50) that the other side reports one step later.  Few envs may have one.
    contact_rewards = (1.0, 25.0, 50.0, -250.0)    # button contact (sparse / shaped / final) or table contact (shaped)
    shifted = []
    for i in range(n):
        bad = np.nonzero((c["done"][:, i] != o["done"][:, i]) | (np.abs(c["rew"][:, i] - o["rew"][:, i]) > POS_TOL))[0]
        t_end = T if len(bad) == 0 else int(bad[0])
        assert np.abs(c["obs"][:t_end, i] - o["obs"][:t_end, i]).max(initial=0.0) < POS_TOL
        if len(bad):
            shifted.append(i)
            t = t_end
            early, late = (c, o) if float(c["rew"][t, i]) in contact_rewards else (o, c)
            info = (i, t, c["rew"][t - 1:t + 3, i], o["rew"][t - 1:t + 3, i], c["done"][t - 1:t + 3, i], o["done"][t - 1:t + 3, i])
            assert float(early["rew"][t, i]) in contact_rewards and float(late["rew"][t, i]) not in contact_rewards, info
            assert float(late["rew"][t + 1, i]) in contact_rewards, info
    assert len(shifted) <= 2, shifted
    same = np.setdiff1d(np.arange(n), shifted)
    assert np.array_equal(c["two"][same, :3], o["two"][same, :3])               # n_contacts[0], n_contacts[1], goal_id
    assert np.abs(c["two"][same, 3:] - o["two"][same, 3:]).max() < 1e-4         # second button base, second glider q / qd
    assert np.abs(c["target"][same] - o["target"][same]).max() < 1e-6
    assert np.abs(c["q"][same] - o["q"][same]).max() < Q_TOL and np.abs(c["grip"][same] - o["grip"][same]).max() < POS_TOL
    assert np.array_equal(c["counters"][same], o["counters"][same]) and np.array_equal(c["counter"][same], o["counter"][same])


def test_cuda_matches_committed_golden(cuda_backend):
    gen = _gen()
    g = np.load(os.path.join(GOLDEN, "kuka_oracle_golden.npz"))
    blob = load_kuka_scene().blob
    for tag, (env_id, n, T, cfg) in gen.CASES.items():
        acts, noise = gen.inputs(tag, n, T, cfg)
        res = gen.run(cuda_backend, env_id, n, T, cfg, acts, noise, blob)
        assert np.array_equal(res["done"], g[tag + "/done"]), tag
        if not cfg.get("shape_reward", False):
            assert np.array_equal(res["rew"], g[tag + "/rew"]), tag
        for k, tol in (("obs0", POS_TOL), ("obs", POS_TOL), ("grip", POS_TOL), ("ee", POS_TOL), ("q", Q_TOL), ("qd", QD_TOL), ("target", 1e-6)):
            assert np.abs(res[k] - g["%s/%s" % (tag, k)]).max() < tol, (tag, k)


def test_step_equals_rollout_and_lane_packing_invariance(cuda_backend):
    """Lockstep step() x T == fused rollout(T), and the result does not depend on how the envs are packed into warps (bit-exact) -- within
    each of the two layouts the kernel has: four lanes per env (up to 8 envs per warp, the default for batches that fit one warp per
    scheduler) and one thread per env (more envs per warp).  ACROSS the two layouts the once-per-step arithmetic is associated differently,
    so they agree to the float32 tolerances of the oracle comparison, flags included on this seed."""
    n, T = 40, 90
    rs = np.random.RandomState(4)
    acts = rs.randint(0, 6, size=(T, n)).astype(np.int32); noise = rs.normal(0, 0.01, size=(T, n)).astype(np.float32)
    base = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, seed=2, max_steps=40)
    assert base["done"].sum() >= 2 * n
    keys = ("obs0", "obs", "rew", "done", "ep_ret", "ep_len", "q", "qd", "grip", "counters")
    for kw in (dict(stepwise=True), dict(envs_per_warp=1), dict(envs_per_warp=7), dict(envs_per_warp=8), dict(chunk=13)):
        other = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, seed=2, max_steps=40, **kw)
        for k in keys:
            assert np.array_equal(base[k], other[k]), (kw, k)
    wide = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, seed=2, max_steps=40, envs_per_warp=32)      # one thread per env
    for kw in (dict(envs_per_warp=9), dict(envs_per_warp=20, stepwise=True)):
        other = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, seed=2, max_steps=40, **kw)
        for k in keys:
            assert np.array_equal(wide[k], other[k]), (kw, k)
    for k in ("rew", "done", "ep_len", "counters"):
        assert np.array_equal(base[k], wide[k]), k
    for k, tol in (("obs0", POS_TOL), ("obs", POS_TOL), ("grip", POS_TOL), ("q", Q_TOL), ("qd", QD_TOL)):
        assert np.abs(base[k] - wide[k]).max() < tol, k
    assert base["launches"] == 3                                        # settle (create) + reset + ONE fused rollout


def test_in_kernel_streams_and_sharding_invariance(cuda_backend, oracle_backend):
    """actions = noise = NULL: Philox actions/noise/reset draws keyed by the global env index."""
    T = 300
    kind, cfg = "KukaRandButtonGymEnv-v0", dict(seed=21, random_target=True, max_steps=100)
    whole = _run(cuda_backend, kind, 24, T, None, None, **cfg)
    lo = _run(cuda_backend, kind, 10, T, None, None, global_env_offset=0, **cfg)
    hi = _run(cuda_backend, kind, 14, T, None, None, global_env_offset=10, **cfg)
    for k, ax in (("obs", 1), ("rew", 1), ("done", 1), ("q", 0), ("target", 0)):
        assert np.array_equal(whole[k], np.concatenate([lo[k], hi[k]], axis=ax)), k
    # the oracle draws the same integers from the same streams; button placement agrees to float32 rounding
    o = _run(oracle_backend, kind, 24, T, None, None, **cfg)
    assert np.array_equal(whole["done"], o["done"]) and np.abs(whole["obs"] - o["obs"]).max() < POS_TOL
    assert np.abs(whole["target"] - o["target"]).max() < 1e-6


def test_handle_on_every_device(cuda_lib):
    """One process, one Kuka handle per visible device: the four-lane kernel's shared-memory opt-in belongs to a device context, so every
    device must get it, and every device computes the same rollout bit for bit."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible devices")
    from srl_sim.backend import Backend
    runs = [_run(Backend(cuda_lib, dev), "KukaButtonGymEnv-v0", 40, 30, None, None, seed=3, max_steps=20)
            for dev in range(torch.cuda.device_count())]
    for r in runs[1:]:
        for k in ("obs0", "obs", "rew", "done", "ep_len", "q", "qd", "counters"):
            assert np.array_equal(runs[0][k], r[k]), k


def test_full_size_properties_4096_envs(cuda_backend):
    """BASELINE config 2 size: 4096 envs, fused rollouts; size-independent invariants of the env."""
    n, T = 4096, 384
    rs = np.random.default_rng(0)
    acts = rs.integers(0, 6, (T, n), dtype=np.int32); noise = rs.normal(0, 0.01, (T, n)).astype(np.float32)
    r = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, chunk=128, seed=0, max_steps=300)
    assert np.isfinite(r["obs"]).all() and np.isfinite(r["q"]).all() and np.isfinite(r["qd"]).all()
    assert set(np.unique(r["rew"])) <= {-1.0, 0.0, 1.0}
    d = r["done"].astype(bool)
    assert d.any(axis=0).all()                                            # max_steps=300 forces >= 1 episode end per env
    assert r["ep_len"][d].max() <= 301 and r["ep_len"][d].min() >= 1      # counter > max_steps <=> 301 steps
    # Monitor semantics: episode return == sum of the rewards of that episode (first episode of each env)
    first = d.argmax(axis=0)
    csum = np.cumsum(r["rew"], axis=0)
    assert np.allclose(r["ep_ret"][first, np.arange(n)], csum[first, np.arange(n)])
    assert (r["ep_len"][first, np.arange(n)] == first + 1).all()
    # a +1 reward needs the button manifold: the gripper COM is then within reach of the button target
    near = np.linalg.norm(r["obs"][(r["rew"] == 1) & ~d], axis=-1)
    assert near.size > 0 and near.max() < 0.4
    # joints respect their limits (+ solver slop), the commanded pose its box, the glider its travel
    sc = load_kuka_scene()
    lo = np.array([b.lower for b in sc.bodies]); hi = np.array([b.upper for b in sc.bodies])
    assert (r["q"] >= lo - 0.02).all() and (r["q"] <= hi + 0.02).all()
    assert (r["glider"][:, 0] > -1e-4).all() and (r["glider"][:, 0] < 0.0101).all()
    assert np.abs(r["qd"][:, :7]).max() < 2.0


@pytest.mark.parametrize("host_chunks", [0, 3, 7])
def test_rollout_host_matches_device_rollout(cuda_backend, host_chunks, monkeypatch):
    """srl_sim_rollout_host pipelines the rollout in T-chunks (copy-in / kernel / copy-out streams); the chunking
    (here forced through SRL_HOST_CHUNKS, read when the handle first uses the host path) must not change a bit."""
    if host_chunks:
        monkeypatch.setenv("SRL_HOST_CHUNKS", str(host_chunks))
    else:
        monkeypatch.delenv("SRL_HOST_CHUNKS", raising=False)
    n, T = 256, 64
    rs = np.random.RandomState(8)
    acts = rs.randint(0, 6, size=(T, n)).astype(np.int32); noise = rs.normal(0, 0.01, size=(T, n)).astype(np.float32)
    dev = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, seed=6)
    sim = cuda_backend.make_sim("KukaButtonGymEnv-v0", n, model_blob=load_kuka_scene().blob, seed=6)
    sim.reset(stream=cuda_backend.stream())
    import torch
    torch.cuda.synchronize()
    obs = np.zeros((T, n, 3), np.float32); rew = np.zeros((T, n), np.float32); done = np.zeros((T, n), np.uint8)
    launches0 = sim.launch_count
    sim.rollout_host(T, acts, noise, obs, rew, done)
    assert np.array_equal(obs, dev["obs"]) and np.array_equal(rew, dev["rew"]) and np.array_equal(done, dev["done"])
    assert sim.last_kernel_ms() > 0
    assert sim.launch_count - launches0 == max(1, host_chunks)   # one launch per T-chunk


def test_rollout_host_pinned_buffers(cuda_backend, monkeypatch):
    """An unsplit srl_sim_rollout_host into pinned host output buffers gives the same bits as the device rollout; some outputs
    pinned / some pageable is allowed, and so is requesting a single output."""
    import torch
    monkeypatch.delenv("SRL_HOST_CHUNKS", raising=False)
    n, T = 256, 64
    rs = np.random.RandomState(9)
    acts = rs.randint(0, 6, size=(T, n)).astype(np.int32); noise = rs.normal(0, 0.01, size=(T, n)).astype(np.float32)
    dev = _run(cuda_backend, "KukaButtonGymEnv-v0", n, T, acts, noise, seed=7)
    sim = cuda_backend.make_sim("KukaButtonGymEnv-v0", n, model_blob=load_kuka_scene().blob, seed=7)
    sim.reset(stream=cuda_backend.stream())
    torch.cuda.synchronize()
    obs = torch.full((T, n, 3), float("nan")).pin_memory(); rew = torch.full((T, n), float("nan")).pin_memory()
    done = np.full((T, n), 255, np.uint8)                                  # pageable on purpose
    sim.rollout_host(T, torch.from_numpy(acts).pin_memory(), torch.from_numpy(noise).pin_memory(), obs, rew, done)
    assert np.array_equal(obs.numpy(), dev["obs"]) and np.array_equal(rew.numpy(), dev["rew"]) and np.array_equal(done, dev["done"])
    obs.fill_(float("nan"))
    sim2 = cuda_backend.make_sim("KukaButtonGymEnv-v0", n, model_blob=load_kuka_scene().blob, seed=7)
    sim2.reset(stream=cuda_backend.stream())
    sim2.rollout_host(T, acts, noise, obs, None, None)                      # only one output requested
    assert np.array_equal(obs.numpy(), dev["obs"])


def test_single_env_classes_on_cuda(cuda_lib):
    from srl_sim import backend
    backend.use_library(None, None)
    from environments.registry import registered_env
    env = registered_env["KukaButtonGymEnv-v0"][0](srl_model="ground_truth")
    env.seed(5)
    o = env.reset()
    assert o.shape == (3,) and np.allclose(o, np.array(env.getArmPos()) - env.getTargetPos())
    tot = 0
    for t in range(40):
        o, r, d, info = env.step(env.action_space.sample())
        tot += r
        assert isinstance(r, int) and info == {}
    assert np.isfinite(o).all()
    env.close()


@pytest.mark.parametrize("tag", ["disc", "cont", "disc_rep3_none", "rand_button_disc", "disc_rand_shaped", "moving_disc", "moving_cont_rand",
                                 "joints", "joints_shaped_none", "two_disc", "two_disc_rand_shaped", "two_cont_up"])
def test_reference_class_logic_golden_through_cuda(tag, cuda_lib):
    """Trajectories recorded from the REFERENCE Kuka classes (on the oracle's physics, tests/golden/fake_pybullet.py)
    replayed through our env classes -> C-ABI -> the fp32 kernel: flags exact, positions within 1e-3 m."""
    from srl_sim import backend
    from test_kuka_cpu import replay_ref_logic_case
    backend.use_library(None, None)
    # two_disc: after the first button of its third episode is pressed (step 687) the recorded controller drags the gripper sideways
    # ACROSS that button while still pushing down -- a sustained sliding contact over the disc's edge, where the fp32 kernel and the
    # fp64 oracle separate by 8 mm within ten steps (measured; the oracle itself replays the case to 1e-6).  The CUDA replay
    # therefore covers the two complete episodes (both buttons pressed, goal switch, second-button termination) and stops there.
    replay_ref_logic_case(tag, POS_TOL, max_steps={"two_disc": 690}.get(tag))


def _parity_until_first_flag_shift(c, o, max_shifted_envs, max_drift_envs=0, drift_tol=POS_TOL, stats=None):
    """fp32 vs fp64 can move a contact ONSET by one step when the sphere-shape distance lands within float32 rounding
    (~3e-6 m, against ~1.2 mm of approach per step) of the 0.02 m manifold margin.  After such a shift the episode ends one
    step earlier/later and the env legitimately sees different actions, so each env is compared up to its first flag
    difference, which must be exactly such a one-step shift (of a button contact, reward 1, or of a table contact, reward -1 and done);
    only a few envs may have one.  `max_drift_envs` envs may exceed POS_TOL (but not `drift_tol`) before their first flag difference: with
    force_down off and the large workspace box an arm can spend hundreds of steps stretched out towards an unreachable command without an
    episode boundary, where float32 and float64 separate by a few micrometres per step (measured: 2 of 4096 envs pass 1 mm after ~500
    such steps, in the one-thread-per-env kernel of round 1 as well)."""
    T, n = o["rew"].shape
    shifted, drifted, worst = 0, 0, 0.0
    for i in range(n):
        bad = np.nonzero((c["rew"][:, i] != o["rew"][:, i]) | (c["done"][:, i] != o["done"][:, i]))[0]
        t_end = T if len(bad) == 0 else int(bad[0])
        dmax = float(np.abs(c["obs"][:t_end, i] - o["obs"][:t_end, i]).max(initial=0.0))
        worst = max(worst, dmax)
        assert dmax < drift_tol, (i, dmax)
        drifted += dmax >= POS_TOL
        if len(bad):
            shifted += 1
            t = t_end
            rc, ro = float(c["rew"][t, i]), float(o["rew"][t, i])
            flag = -1.0 if -1.0 in (rc, ro) else 1.0          # table contact (-1, ends the episode) or button contact (1): same 0.02 m margin test
            assert {rc, ro} - {flag} <= {0.0, 1.0} and rc != ro                            # a contact flag, on one side only ...
            early, late = (c, o) if rc == flag else (o, c)
            assert late["rew"][t + 1, i] == flag                                           # ... that the other side raises one step later
            if flag == 1.0:                                                                # (a table contact ends the episode: the early side is already past its reset)
                assert early["rew"][t + 1, i] == 1.0
                assert np.abs(c["obs"][t, i] - o["obs"][t, i]).max() < POS_TOL
    assert shifted <= max_shifted_envs, shifted
    assert drifted <= max_drift_envs, drifted
    if stats is not None:
        stats.update(drifted=drifted, worst=worst)
    return shifted


def test_moving_button_kind_vs_oracle(cuda_backend, oracle_backend):
    """KukaMovingButtonGymEnv-v0: the button (and the target) slides +-0.001 per step and bounces at |y| = 0.3."""
    n, T = 24, 900
    rs = np.random.RandomState(6)
    acts = rs.randint(0, 6, size=(T, n)).astype(np.int32); noise = rs.normal(0, 0.01, size=(T, n)).astype(np.float32)
    cfg = dict(seed=4, random_target=True)
    c = _run(cuda_backend, "KukaMovingButtonGymEnv-v0", n, T, acts, noise, **cfg)
    o = _run(oracle_backend, "KukaMovingButtonGymEnv-v0", n, T, acts, noise, **cfg)
    assert np.abs(c["obs0"] - o["obs0"]).max() < POS_TOL
    _parity_until_first_flag_shift(c, o, max_shifted_envs=3)
    assert o["done"].sum() >= n // 2 and np.abs(o["target"][:, 1]).max() <= 0.3011


# BASELINE.json configs at FULL batch: (env id, steps, action kind, cfg, noise std, bound on the envs that may see a one-step contact-onset
# shift = 2 x the count measured on an H100 with this kernel, floor 8)
FULL_BATCH_CASES = {
    # measured on an H100 (four lanes per env): 10 / 26 / 2 / 0 shifted envs
    "config2": ("KukaButtonGymEnv-v0", 1000, "discrete", dict(seed=0, is_discrete=True, random_target=False, force_down=True, action_repeat=1, max_distance=0.8), 0.01, 20),
    "config5": ("KukaRandButtonGymEnv-v0", 2000, "continuous", dict(seed=0, is_discrete=False, random_target=True, force_down=True, action_repeat=1, max_distance=0.8), 1e-4, 52),
    "action_repeat3": ("KukaButtonGymEnv-v0", 400, "discrete", dict(seed=0, is_discrete=True, random_target=False, force_down=True, action_repeat=3, max_distance=0.8), 0.01, 8),
    "no_force_down": ("KukaButtonGymEnv-v0", 600, "discrete", dict(seed=0, is_discrete=True, random_target=True, force_down=False, action_repeat=1, max_distance=0.8), 0.01, 40),
}
FULL_BATCH_DRIFT = {"no_force_down": (6, 6e-3)}     # envs allowed past POS_TOL before their first flag difference, and how far (3 x measured: 2 envs, 3.4 mm)


@pytest.mark.parametrize("case", sorted(FULL_BATCH_CASES))
def test_full_batch_4096_envs_vs_oracle(cuda_backend, oracle_lib, case):
    """BASELINE configs 2 and 5 (and the action_repeat / force_down variants) at FULL size: all 4096 envs, CUDA (float32) vs the oracle
    (float64, sharded over the host threads).  Reward / done flags must agree except for one-step contact-onset shifts (see
    _parity_until_first_flag_shift) in a small, bounded number of envs; positions agree to 1e-3 m up to that point.  The shift statistics
    are printed (pytest -s / the tail of a failing run)."""
    import threading
    from srl_sim.backend import Backend
    env_id, T, kind, cfg, noise_std, bound = FULL_BATCH_CASES[case]
    n = 4096
    if kind == "discrete":
        acts = np.random.default_rng(0).integers(0, 6, (T, n), dtype=np.int32)
    else:
        acts = np.random.default_rng(0).uniform(-1, 1, (T, n, 3)).astype(np.float32)
    noise = np.random.default_rng(1).normal(0, noise_std, (T, n)).astype(np.float32)
    c = _run(cuda_backend, env_id, n, T, acts, noise, **cfg)
    threads = max(1, min(16, os.cpu_count() or 1))
    bounds = np.linspace(0, n, threads + 1).astype(int)
    parts = [None] * threads
    be = Backend(oracle_lib, -1)

    def work(k):
        lo, hi = int(bounds[k]), int(bounds[k + 1])
        parts[k] = _run(be, env_id, hi - lo, T, np.ascontiguousarray(acts[:, lo:hi]), np.ascontiguousarray(noise[:, lo:hi]),
                        global_env_offset=lo, **cfg)
    ths = [threading.Thread(target=work, args=(k,)) for k in range(threads)]
    [t.start() for t in ths]; [t.join() for t in ths]
    o = {k: np.concatenate([p[k] for p in parts], axis=1 if parts[0][k].ndim >= 2 and k in ("obs", "rew", "done", "ep_ret", "ep_len") else 0)
         for k in ("obs0", "obs", "rew", "done")}
    assert np.abs(c["obs0"] - o["obs0"]).max() < POS_TOL
    drift_envs, drift_tol = FULL_BATCH_DRIFT.get(case, (0, POS_TOL))
    st = {}
    shifted = _parity_until_first_flag_shift(c, o, max_shifted_envs=bound, max_drift_envs=drift_envs, drift_tol=drift_tol, stats=st)
    same = (c["rew"] == o["rew"]) & (c["done"] == o["done"])
    print("FULL-BATCH PARITY %s: %d of %d envs with a one-step contact-onset shift (bound %d); %.4f%% of the %d (env, step) flags identical; episodes %d; "
          "largest |obs| difference before an env's first flag difference %.2e m, %d envs above 1e-3 m"
          % (case, shifted, n, bound, 100.0 * same.mean(), same.size, int(o["done"].sum()), st["worst"], st["drifted"]))
    assert o["done"].sum() >= (n if cfg["force_down"] else 100)       # without force_down few arms reach the table / the button within the run
