"""KukaRandButtonGymEnv distractor bodies on the H100: the CUDA bodies against the float64 checker, the arm's outputs unchanged with the
bodies on, and the ABI's refusals."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "robotics-rl-srl_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)

pytestmark = pytest.mark.gpu

RB = "KukaRandButtonGymEnv-v0"


@pytest.fixture(scope="module")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from srl_sim._abi import load_cuda_library
    from srl_sim.backend import Backend
    return Backend(load_cuda_library(), 0)


def _sim(be, n, kind=RB, seed=0, bodies=True, **cfg):
    from srl_sim.model import distractor_blob, load_kuka_scene
    s = be.make_sim(kind, n, seed=seed, model_blob=load_kuka_scene().blob, **cfg)
    if bodies:
        s.set_distractors(distractor_blob())
    return s


def _bodies(s):
    from srl_sim import _abi
    return s.get_state(_abi.F_DISTRACTORS).reshape(s.num_envs, 11, 9)


def test_abi_refusals(cuda):
    from srl_sim import _abi
    from srl_sim.model import distractor_blob
    for kind in ("KukaButtonGymEnv-v0", "Kuka2ButtonGymEnv-v0", "KukaMovingButtonGymEnv-v0"):
        s = _sim(cuda, 4, kind=kind, bodies=False)
        with pytest.raises(_abi.SimError, match="only KukaRandButton"):
            s.set_distractors(distractor_blob())
    for kind in ("MobileRobotGymEnv-v0", "MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0", "MobileRobotLineTargetGymEnv-v0"):
        s = cuda.make_sim(kind, 4, seed=0)
        with pytest.raises(_abi.SimError, match="only KukaRandButton"):
            s.set_distractors(distractor_blob())
    s = _sim(cuda, 4, bodies=False)
    s.reset(stream=cuda.stream())
    with pytest.raises(_abi.SimError, match="first reset"):
        s.set_distractors(distractor_blob())
    s = _sim(cuda, 4, bodies=False, prefetch_resets=True)
    with pytest.raises(_abi.SimError, match="prefetch_resets"):
        s.set_distractors(distractor_blob())
    s = _sim(cuda, 4, bodies=False)
    with pytest.raises(_abi.SimError, match="wrong size"):
        s.set_distractors(distractor_blob()[:-1])
    # without the bodies the field is all zero
    assert not _bodies(s).any()


def _host_draws(n, seed):
    """48 reset values per env: the button at its default place, zero random init actions, placements and types from a RandomState."""
    rng = np.random.RandomState(seed)
    d = np.zeros((n, 48), np.float64)
    d[:, 0] = 0.5
    d[:, 18:38:2] = 0.5 + 0.15 * rng.uniform(-1, 1, size=(n, 10))
    d[:, 19:38:2] = 0.3 * rng.uniform(-1, 1, size=(n, 10))
    d[:, 38:] = rng.randint(3, size=(n, 10))
    return d


def test_placement_and_settle_against_the_float64_checker(cuda):
    from srl_sim import _abi
    from srl_sim.model import distractor_blob, load_kuka_scene
    n = 64
    draws = _host_draws(n, 1)
    s = _sim(cuda, n, is_discrete=True, no_auto_reset=True)
    obs = cuda.zeros((n, 3), np.float32)
    s.reset(reset_draws=cuda.from_host(draws), obs_out=obs, stream=cuda.stream())
    B = _bodies(s)
    touch = s.get_state(_abi.F_DISTRACTOR_TOUCH)
    # presence: the reference's rule around the button at (0.5, 0)
    for i in range(n):
        for k in range(10):
            x, y = draws[i, 18 + 2 * k], draws[i, 19 + 2 * k]
            assert B[i, k, 8] == float(x < 0.4 or x > 0.6 or y < -0.1 or y > 0.1)
            assert B[i, k, 7] == draws[i, 38 + k]
        assert B[i, 10, 8] == 1 and B[i, 10, 7] == 3
    # float64 checker: the same placement, 505 micro-steps with the arm away (bodies that touched the arm or another body are excluded)
    lib = ctypes.CDLL(os.path.join(PKG, "csrc", "libdistractor_ref.so"))
    P = ctypes.c_void_p
    lib.dref_run.argtypes = [P, ctypes.c_size_t, P, ctypes.c_double, ctypes.c_int, ctypes.c_double, P, P, ctypes.c_int, ctypes.c_int, P,
                             ctypes.c_int, P, P]
    lib.dref_place.argtypes = [P, P, ctypes.c_double, ctypes.c_double, P]
    blob = distractor_blob()
    sc = load_kuka_scene()
    glider = s.get_state(_abi.F_BUTTON_GLIDER)
    errs, compared, skipped = [], 0, 0
    for i in range(n):
        Bd = np.zeros((11, 16), np.float64)
        types = draws[i, 38:].astype(np.int32)
        lib.dref_place(np.ascontiguousarray(draws[i, 18:38]).ctypes.data, types.ctypes.data, 0.5, 0.0, Bd.ctypes.data)
        scene = _button_scene(sc, glider[i, 0])
        touch_d = np.zeros(2, np.uint32)
        arm = np.zeros((1, 4), np.float64)
        lib.dref_run(blob.ctypes.data, blob.nbytes, scene.ctypes.data, 1.0 / 240.0, 150, 0.02, Bd.ctypes.data, arm.ctypes.data, 0, 505, None, 0,
                     None, touch_d.ctypes.data)
        for k in range(11):
            if not B[i, k, 8]:
                continue
            excluded = ((int(touch[i, 0]) | int(touch_d[0])) >> k) & 1 or (int(touch[i, 1]) >> k) & 1
            if excluded:
                skipped += 1
                continue
            compared += 1
            errs.append((int(B[i, k, 7]), np.abs(B[i, k, 0:3] - Bd[k, 0:3]).max()))
    t = np.array([e[0] for e in errs]); errs = np.array([e[1] for e in errs])
    for ty, name in enumerate(("duck", "lego", "cube", "sphere")):
        e = errs[t == ty]
        print("%-6s compared %3d  max |dpos| %.3g m  median %.3g m  > 1 mm: %d" % (name, e.size, e.max(), np.median(e), (e > 1e-3).sum()))
    print("excluded (touched another body or the arm): %d" % skipped)
    assert compared >= n
    # bodies that rest on one face (the flat brick, the ball) agree; the duck and the tetrahedral cube tip over an edge after landing, a
    # tipping direction float32 and float64 may choose differently -- most still agree, the rest are counted
    stable = (t == 1) | (t == 3)
    assert errs[stable].max() < 1e-3
    assert np.median(errs[~stable]) < 1e-3 and (errs[~stable] > 1e-3).mean() < 0.25


def _button_scene(sc, qb):
    """table + button of the loaded model as the library sees them (csrc/kuka_params.cuh)."""
    from srl_sim.model import scene_constants
    c = scene_constants(sc)
    bz = c["button_z"]
    disc0 = bz + c["glider_z"] + qb + c["disc_z0"]
    disc1 = bz + c["glider_z"] + qb + c["disc_z1"]
    return np.array([c["table_z"], c["txmin"], c["txmax"], c["tymin"], c["tymax"], 0.5, 0.0, bz, c["stack_top"], c["stack_r"], c["disc_r"],
                     disc0, disc1], np.float64)


@pytest.mark.parametrize("discrete,repeat,seed", [(True, 1, 0), (False, 1, 3), (True, 3, 7), (False, 3, 11)])
def test_arm_outputs_are_byte_identical_with_bodies(cuda, discrete, repeat, seed):
    import torch
    n, T = 96, 300
    outs = []
    for bodies in (False, True):
        s = _sim(cuda, n, seed=seed, bodies=bodies, is_discrete=discrete, action_repeat=repeat, random_target=True, max_steps=60)
        s.reset(stream=cuda.stream())
        D = 3
        o = [cuda.zeros((T, n, D), np.float32), cuda.zeros((T, n), np.float32), cuda.zeros((T, n), np.uint8),
             cuda.zeros((T, n), np.float32), cuda.zeros((T, n), np.int32)]
        s.rollout(T, obs_out=o[0], rew_out=o[1], done_out=o[2], ep_ret_out=o[3], ep_len_out=o[4], stream=cuda.stream())
        torch.cuda.synchronize()
        outs.append([cuda.to_host(x).copy() for x in o])
        if bodies:
            B = _bodies(s)
            assert np.isfinite(B).all()
    ep = outs[0][2].sum()
    assert ep > n, "expected more than one episode per env"
    for a, b in zip(outs[0], outs[1]):
        assert a.tobytes() == b.tobytes()


def test_bench_size_outputs_identical_and_sphere_kicked(cuda):
    import time
    import torch
    n, T = 4096, 128
    outs = []
    for bodies in (False, True):
        s = _sim(cuda, n, seed=0, bodies=bodies, is_discrete=True)
        s.reset(stream=cuda.stream())
        if bodies:
            before = _bodies(s)[:, 10, 0:3].copy()
        o = [cuda.zeros((T, n, 3), np.float32), cuda.zeros((T, n), np.float32), cuda.zeros((T, n), np.uint8),
             cuda.zeros((T, n), np.float32), cuda.zeros((T, n), np.int32)]
        t0 = time.time()
        s.rollout(T, obs_out=o[0], rew_out=o[1], done_out=o[2], ep_ret_out=o[3], ep_len_out=o[4], stream=cuda.stream())
        torch.cuda.synchronize()
        print("4096 x 128 rollout, bodies %s: %.3f s" % ("on" if bodies else "off", time.time() - t0))
        outs.append([cuda.to_host(x).copy() for x in o])
        if bodies:
            after = _bodies(s)[:, 10, 0:3]
            no_reset = ~outs[1][2].any(axis=0)
            moved = after[no_reset] - before[no_reset]
            print("envs without a reset: %d, sphere moved +x in %d, +y in %d" % (no_reset.sum(), (moved[:, 0] > 0).sum(), (moved[:, 1] > 0).sum()))
    for a, b in zip(outs[0], outs[1]):
        assert a.tobytes() == b.tobytes()
    # the kick at step 10 sends the sphere towards +x, +y; over the remaining 118 steps some run into an object, the button or the arm
    both = ((moved[:, 0] > 1e-3) & (moved[:, 1] > 1e-3)).mean()
    print("sphere moved > 1 mm towards both +x and +y in %.1f %% of the envs" % (100 * both))
    assert no_reset.sum() > 20
    assert both > 0.85


def test_single_env_class_with_bodies(cuda):
    from environments.kuka_gym.kuka_rand_button_gym_env import KukaRandButtonGymEnv
    env = KukaRandButtonGymEnv(srl_model="ground_truth", random_target=True, distractors=True)
    env.seed(2)
    env.reset()
    B = env.getDistractors()
    assert B.shape == (11, 9) and B[10, 8] == 1
    for _ in range(12):
        env.step(0)
    assert np.isfinite(env.getDistractors()).all()
    with pytest.raises(ValueError):
        from environments.kuka_gym.kuka_button_gym_env import KukaButtonGymEnv
        KukaButtonGymEnv(srl_model="ground_truth", distractors=True)
