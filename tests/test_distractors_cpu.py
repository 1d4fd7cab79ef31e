"""KukaRandButtonGymEnv distractor bodies (csrc/distractor_core.h), checked on the CPU: the float64 checker built from the same header
against an independent numpy model of one free body on the table, the placement rule of the reference, and the host plumbing."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "robotics-rl-srl_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)

from srl_sim.model import DISTRACTOR_TYPES, distractor_blob  # noqa: E402

DT = 1.0 / 240.0
G = 10.0
MARGIN = 0.02
TABLE_Z = -0.195
# table top, button far away from the drops below
SCENE = np.array([TABLE_Z, -0.25, 1.25, -0.5, 0.5, 5.0, 5.0, TABLE_Z, 0.03, 0.1, 0.09, 10.0, 10.1], np.float64)


@pytest.fixture(scope="module")
def dref():
    path = os.path.join(PKG, "csrc", "libdistractor_ref.so")
    if not os.path.isfile(path):
        pytest.skip("libdistractor_ref.so not built (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    P = ctypes.c_void_p
    lib.dref_run.argtypes = [P, ctypes.c_size_t, P, ctypes.c_double, ctypes.c_int, ctypes.c_double, P, P, ctypes.c_int, ctypes.c_int, P,
                             ctypes.c_int, P, P]
    lib.dref_run.restype = ctypes.c_int
    lib.dref_place.argtypes = [P, P, ctypes.c_double, ctypes.c_double, P]
    lib.dref_kick.argtypes = [ctypes.c_double, ctypes.c_double, ctypes.c_double, P]
    return lib


def _bodies(type_, pos):
    """11 body slots, only slot 10 present (the kick acts on slot 10)."""
    B = np.zeros((11, 16), np.float64)
    B[:, 6] = 1.0
    B[10, 0:3] = pos
    B[10, 13] = type_
    B[10, 14] = 1.0
    return B


def _run(lib, B, n, iters=150, kick=None, kick_step=0):
    blob = distractor_blob()
    traj = np.zeros((n, 11, 16), np.float64)
    arm = np.zeros((1, 4), np.float64)
    k = None if kick is None else np.ascontiguousarray(kick, np.float64)
    rc = lib.dref_run(blob.ctypes.data, blob.nbytes, SCENE.ctypes.data, DT, iters, MARGIN, B.ctypes.data, arm.ctypes.data, 0, n,
                      None if k is None else k.ctypes.data, kick_step, traj.ctypes.data, None)
    assert rc == 0
    return traj


def _type_row(t):
    return distractor_blob().reshape(4, 32)[t]


def numpy_free_body(t, pos, n, kick=None):
    """Independent model of the restatement for ONE upright body whose spheres are all at the same height (a ball, or the flat
    4-sphere brick) on the table plane: vertical motion only, so each sphere's normal row acts on the COM velocity alone and the
    friction rows carry no load.  A sphere at distance d <= margin constrains the fall speed to at most d / dt (separated) or
    to pushing out at 0.2 |d| / dt (penetrating)."""
    row = _type_row(t)
    m = row[0]
    ns = int(row[5])
    cz = row[6 + 2]
    r = row[6 + 3]
    assert all(row[6 + 4 * k + 2] == cz and row[6 + 4 * k + 3] == r for k in range(ns))
    p = np.array(pos, np.float64)
    v = np.zeros(3)
    out = []
    for s in range(n):
        v[2] -= G * DT
        if kick is not None and s == 0:
            v += np.asarray(kick) / m
        d = p[2] + cz - TABLE_Z - r
        if d <= MARGIN:
            target = -d / DT if d > 0 else -0.2 * d / DT
            v[2] = max(v[2], target)      # normal rows: relative velocity >= target, lambda >= 0
        p = p + DT * v
        out.append((p.copy(), v.copy()))
    return out


@pytest.mark.parametrize("name", ["sphere_small", "lego"])
def test_checker_matches_numpy_model_over_a_drop(dref, name):
    t = DISTRACTOR_TYPES.index(name)
    start = (0.5, 0.0, TABLE_Z + 0.12)
    traj = _run(dref, _bodies(t, start), 100)
    ref = numpy_free_body(t, start, 100)
    for s in range(100):
        np.testing.assert_allclose(traj[s, 10, 0:3], ref[s][0], atol=1e-9, rtol=0)
        np.testing.assert_allclose(traj[s, 10, 7:10], ref[s][1], atol=1e-9, rtol=0)
        np.testing.assert_allclose(traj[s, 10, 3:7], [0, 0, 0, 1], atol=1e-12)


@pytest.mark.parametrize("name", DISTRACTOR_TYPES)
def test_body_comes_to_rest_and_never_gains_energy(dref, name):
    t = DISTRACTOR_TYPES.index(name)
    row = _type_row(t)
    traj = _run(dref, _bodies(t, (0.5, 0.0, TABLE_Z + 0.1)), 600)
    m = row[0]
    I = row[1:4]

    def energy(b):
        from scipy.spatial.transform import Rotation
        R = Rotation.from_quat(b[3:7]).as_matrix()
        w_body = R.T @ b[10:13]
        return 0.5 * m * b[7:10] @ b[7:10] + 0.5 * w_body @ (I * w_body) + m * G * b[2]

    E = np.array([energy(traj[s, 10]) for s in range(600)])
    first = next(s for s in range(1, 600) if traj[s, 10, 9] > traj[s - 1, 10, 9])      # the first contact impulse
    # flat bodies land without penetrating (the separated target stops them exactly on the table); a body that tips over is pushed
    # out of a shallow penetration by the -0.2 dist/dt target, which may add a few 1e-8 J
    tol = 1e-9 if name in ("sphere_small", "lego") else 1e-6
    assert np.max(np.diff(E[first - 1:])) <= tol, (name, np.max(np.diff(E[first - 1:])))
    # at rest: the lowest sphere surface on the table top
    from scipy.spatial.transform import Rotation
    b = traj[-1, 10]
    R = Rotation.from_quat(b[3:7]).as_matrix()
    ns = int(row[5])
    lows = [(b[0:3] + R @ row[6 + 4 * k:9 + 4 * k])[2] - row[9 + 4 * k] for k in range(ns)]
    assert abs(min(lows) - TABLE_Z) < 1e-4, (name, min(lows) - TABLE_Z)
    assert np.linalg.norm(b[7:10]) < 1e-3


def test_kick_gives_impulse_over_mass_towards_plus_x_plus_y(dref):
    t = DISTRACTOR_TYPES.index("sphere_small")
    imp = np.zeros(3)
    dref.dref_kick(-0.6, -1.7, DT, imp.ctypes.data)          # the reference takes the absolute value of each component
    n = np.array([0.6, 1.7]) / np.hypot(0.6, 1.7)
    np.testing.assert_allclose(imp, [10 * n[0] * DT, 10 * n[1] * DT, 1 * DT], rtol=1e-12)
    row = _type_row(t)
    start = (0.5, 0.0, TABLE_Z + row[9])                      # resting on the table
    traj = _run(dref, _bodies(t, start), 1, kick=imp)
    v = traj[0, 10, 7:10]
    np.testing.assert_allclose(v[:2], imp[:2] / row[0], rtol=1e-12)
    assert v[0] > 0 and v[1] > 0


def test_placement_matches_the_reference_class(dref):
    """tests/golden/distractor_placement_golden.npz: where the reference's own KukaRandButtonGymEnv (on fake_pybullet) loads the objects
    and the sphere in 3 consecutive resets, for 6 (seed, random_target, global np.random seed) cases.  Our class, seeded the same way,
    draws the same placement values and types in the same order, and the library's placement rule loads the same bodies at the same
    (x, y, z)."""
    from environments.kuka_gym.kuka_rand_button_gym_env import KukaRandButtonGymEnv
    g = np.load(os.path.join(ROOT, "tests", "golden", "distractor_placement_golden.npz"))
    ncases = len([k for k in g.files if k.endswith("/params")])
    assert ncases == 6
    for c in range(ncases):
        seed, random_target, np_seed = (int(v) for v in g["case%d/params" % c])
        env = KukaRandButtonGymEnv.__new__(KukaRandButtonGymEnv)
        env._random_target = bool(random_target)
        env._is_discrete = True
        env.action_joints = False
        env.distractors = True
        env.seed(seed)
        np.random.seed(np_seed)
        counts = g["case%d/counts" % c]
        ref = np.split(g["case%d/bodies" % c], np.cumsum(counts)[:-1])
        for e in range(len(counts)):
            d = np.asarray(env._reset_draws(), np.float64)
            assert d.shape == (48,)
            np.testing.assert_allclose(d[0:2], g["case%d/button_xy" % c][e], rtol=0, atol=1e-15)
            B = np.zeros((11, 16), np.float64)
            types = d[38:48].astype(np.int32)
            dref.dref_place(np.ascontiguousarray(d[18:38]).ctypes.data, types.ctypes.data, d[0], d[1], B.ctypes.data)
            ours = np.array([[B[k, 13], B[k, 0], B[k, 1], B[k, 2]] for k in range(11) if B[k, 14]], np.float64)
            assert ours.shape == ref[e].shape, (c, e)
            np.testing.assert_allclose(ours, ref[e], rtol=0, atol=1e-12)


def test_placement_follows_the_reference_rule(dref):
    rng = np.random.RandomState(3)
    for _ in range(20):
        bx, by = 0.5 + 0.15 * rng.uniform(-1, 1), 0.3 * rng.uniform(-1, 1)
        xy = np.array([[0.5 + 0.15 * rng.uniform(-1, 1), 0.3 * rng.uniform(-1, 1)] for _ in range(10)], np.float64).reshape(-1)
        types = rng.randint(3, size=10).astype(np.int32)
        B = np.zeros((11, 16), np.float64)
        dref.dref_place(xy.ctypes.data, types.ctypes.data, bx, by, B.ctypes.data)
        for k in range(10):
            x, y = xy[2 * k], xy[2 * k + 1]
            # kuka_rand_button_gym_env.py:65-66
            loaded = (x < bx - 0.1) or (x > bx + 0.1) or (y < by - 0.1) or (y > by + 0.1)
            assert B[k, 14] == (1.0 if loaded else 0.0)
            np.testing.assert_allclose(B[k, 0:3], [x, y, -0.2 + 0.1])
            assert B[k, 13] == types[k]
        np.testing.assert_allclose(B[10, 0:3], [0.25, -0.2, -0.2 + 0.3])
        assert B[10, 13] == 3 and B[10, 14] == 1


def test_both_libraries_export_set_distractors(oracle_lib):
    from srl_sim import _abi
    from srl_sim.model import load_kuka_scene
    path = os.path.join(PKG, "csrc", "libsrl_sim_b200.so")
    if not os.path.isfile(path):
        pytest.fail("%s has not been built (python __graft_entry__.py build)" % path)
    assert "srl_sim_set_distractors" in _abi.EXPORTED_SYMBOLS    # required: SimLibrary refuses a library without it
    assert hasattr(_abi.SimLibrary(path).lib, "srl_sim_set_distractors")
    # the oracle exports it too, and refuses: it has no body dynamics
    sim = _abi.Sim(oracle_lib, "KukaRandButtonGymEnv-v0", 1, -1, model_blob=load_kuka_scene().blob)
    with pytest.raises(_abi.SimError, match="no distractor body dynamics"):
        sim.set_distractors(distractor_blob())
    sim.close()


def test_asset_blob_layout():
    b = distractor_blob().reshape(4, 32)
    assert b.shape == (4, 32)
    assert np.all(b[:, 0] > 0) and np.all(b[:, 1:4] > 0)
    assert list(b[:, 5]) == [3, 4, 4, 1]
    assert b[3, 28] == 1 and b[3, 9] == pytest.approx(0.03)


def test_other_kuka_ids_refuse_distractors():
    from srl_sim.vec_env import BatchedSRLVecEnv
    for env_id in ("KukaButtonGymEnv-v0", "Kuka2ButtonGymEnv-v0", "KukaMovingButtonGymEnv-v0", "MobileRobotGymEnv-v0"):
        with pytest.raises(ValueError):
            BatchedSRLVecEnv(env_id, 2, distractors=True)


def test_rand_button_reset_draws_are_unchanged_when_off():
    """Without the bodies the host class consumes the same env draws as before and leaves the global np.random alone."""
    from environments.kuka_gym.kuka_rand_button_gym_env import KukaRandButtonGymEnv
    env = KukaRandButtonGymEnv.__new__(KukaRandButtonGymEnv)
    env._random_target = True
    env._is_discrete = True
    env.action_joints = False
    from srl_sim import seeding
    env.np_random, _ = seeding.np_random(5)
    np.random.seed(11)
    before = np.random.get_state()[1].copy()
    d = env._reset_draws()
    assert len(d) == 18
    assert np.array_equal(np.random.get_state()[1], before)
    env.distractors = True
    env.np_random, _ = seeding.np_random(5)
    d2 = env._reset_draws()
    assert len(d2) == 48 and d2[:18] == d
    assert all(t in (0.0, 1.0, 2.0) for t in d2[38:])
