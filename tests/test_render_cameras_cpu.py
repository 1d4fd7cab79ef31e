"""
One camera per env (srl_sim_render_cameras) on the CPU checker (tests/host/render_cameras_ref.cpp over oracle/liboracle_sim.so): env i's frame is the frame srl_sim_render gives
env i through cameras[i], byte for byte; with follow_robot the MobileRobot cameras are placed from each robot's position (the reference's
first-person camera, mobile_robot_env.py:316-332); and BatchedSRLVecEnv(fpv=True) stacks those frames on the top-down ones.
"""
import numpy as np
import pytest

from srl_sim import _abi
from srl_sim.model import load_kuka_scene
from srl_sim.render import (KUKA_CAMERA, KUKA_CAMERA_2, MOBILE_CAMERA, MOBILE_FPV_FOLLOW, camera, camera_array, mobile_fpv_camera,
                            render_cameras)

MOBILE_IDS = ["MobileRobotGymEnv-v0", "MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0", "MobileRobotLineTargetGymEnv-v0"]


def mid_episode_sim(be, env_id, n, T, seed=7, distractors=False):
    """A handle of n envs (targets randomised) after T random discrete steps."""
    kuka = env_id.startswith("Kuka")
    sim = be.make_sim(env_id, n, model_blob=load_kuka_scene().blob if kuka else None, seed=seed, random_target=True)
    if distractors:
        from srl_sim.model import distractor_blob
        sim.set_distractors(distractor_blob())
    sim.reset(stream=be.stream())
    n_act = 6 if kuka else (2 if env_id == "MobileRobot1DGymEnv-v0" else 4)
    acts = np.random.RandomState(3).randint(0, n_act, size=(T, n)).astype(np.int32)
    obs = be.zeros((T, n, sim.obs_dim), np.float32); rew = be.zeros((T, n), np.float32); done = be.zeros((T, n), np.uint8)
    sim.rollout(T, be.from_host(acts), None, obs, rew, done, stream=be.stream())
    return sim


def mixed_cameras(env_id, n, seed):
    """The env's reference cameras, then random target, yaw, pitch, distance and fov: a different camera for every env."""
    rs = np.random.RandomState(seed)
    kuka = env_id.startswith("Kuka")
    fixed = [KUKA_CAMERA, KUKA_CAMERA_2] if kuka else [MOBILE_CAMERA, mobile_fpv_camera((1.3, 2.6))]
    cams = []
    for i in range(n):
        if i < len(fixed):
            cams.append(dict(fixed[i]))
            continue
        centre = np.array([0.5, 0.0, 0.0]) if kuka else np.array([2.0, 2.0, 0.0])
        target = centre + rs.uniform(-0.6 if kuka else -1.5, 0.6 if kuka else 1.5, 3) * np.array([1.0, 1.0, 0.2])
        cams.append(dict(target=tuple(target), distance=rs.uniform(0.4, 2.0 if kuka else 5.0), yaw=rs.uniform(0, 360),
                         pitch=rs.uniform(-85, -5), roll=0.0, fov=rs.uniform(35, 100)))
    return cams


def single_camera_frames(be, sim, cams, width, height):
    """Frame i of srl_sim_render(cams[i]): what env i must look like through its own camera."""
    n = sim.num_envs
    out = np.zeros((n, height, width, 3), np.uint8)
    for i, c in enumerate(cams):
        buf = be.zeros((n, height, width, 3), np.uint8)
        sim.render(camera(**c), width, height, buf, stream=be.stream())
        out[i] = be.to_host(buf)[i]
    return out


def follow_targets(pos, cams):
    """The absolute cameras of a follow_robot call: target x, y = float32(float64 robot position + float64(float32 offset))."""
    out = []
    for p, c in zip(pos, cams):
        off = np.asarray(c["target"], np.float32).astype(np.float64)
        out.append(dict(c, target=(p[0] + off[0], p[1] + off[1], off[2])))
    return out


@pytest.fixture(scope="module")
def checker_lib():
    import render_cameras_ref
    return render_cameras_ref.library()


@pytest.fixture(scope="module")
def checker_backend(checker_lib):
    from srl_sim.backend import Backend
    return Backend(checker_lib, -1)


@pytest.fixture()
def use_checker_backend(checker_lib):
    """Route BatchedSRLVecEnv to the CPU checker for the duration of one test."""
    from srl_sim import backend
    backend.use_library(checker_lib, -1)
    yield
    backend.use_library(None, None)


def test_export_exists(oracle_lib, checker_lib):
    assert "srl_sim_render_cameras" in _abi.EXPORTED_SYMBOLS
    assert "srl_sim_render_cameras" in _abi.SimLibrary(_abi.CUDA_LIBRARY_PATH).optional
    assert "srl_sim_render_cameras" in checker_lib.optional
    # the oracle library itself has one camera per batch only: the binding refuses instead of calling a missing symbol
    sim = _abi.Sim(oracle_lib, "MobileRobotGymEnv-v0", 2, -1)
    with pytest.raises(_abi.SimError, match="per-env cameras"):
        sim.render_cameras(camera_array([MOBILE_CAMERA] * 2), False, 16, 16, np.zeros((2, 16, 16, 3), np.uint8))
    sim.close()


@pytest.mark.parametrize("env_id", sorted(_abi.ENV_KINDS))
def test_mixed_cameras_match_single_camera_calls(checker_backend, env_id):
    be = checker_backend
    n = 5
    sim = mid_episode_sim(be, env_id, n, 15)
    cams = mixed_cameras(env_id, n, seed=len(env_id))
    for (w, h) in ((224, 224), (50, 33)):
        got = be.to_host(render_cameras(sim, be, cams, width=w, height=h))
        want = single_camera_frames(be, sim, cams, w, h)
        assert np.array_equal(got, want), (env_id, w, h, int((got != want).sum()))
        for k in range(n):
            assert len(np.unique(got[k].reshape(-1, 3), axis=0)) >= 2
    sim.close()


@pytest.mark.parametrize("env_id", MOBILE_IDS)
def test_follow_robot_matches_the_fpv_camera(checker_backend, env_id):
    be = checker_backend
    n = 4
    sim = mid_episode_sim(be, env_id, n, 20, seed=5)
    pos = sim.get_state(_abi.F_ROBOT_POS)
    assert len(np.unique(pos[:, :2], axis=0)) == n                       # the robots have moved apart: every env needs its own camera
    got = be.to_host(render_cameras(sim, be, [MOBILE_FPV_FOLLOW] * n, follow_robot=True))
    want = single_camera_frames(be, sim, [mobile_fpv_camera(p) for p in pos], 224, 224)
    assert np.array_equal(got, want)
    # different offsets and angles per env, an odd size
    rs = np.random.RandomState(2)
    cams = [dict(MOBILE_FPV_FOLLOW, target=(rs.uniform(-0.5, 0.5), rs.uniform(-0.5, 0.5), rs.uniform(0.05, 0.4)), yaw=rs.uniform(0, 360),
                 pitch=rs.uniform(-40, -5), fov=rs.uniform(50, 100)) for _ in range(n)]
    got = be.to_host(render_cameras(sim, be, cams, follow_robot=True, width=50, height=33))
    want = single_camera_frames(be, sim, follow_targets(pos, cams), 50, 33)
    assert np.array_equal(got, want)
    sim.close()


@pytest.mark.parametrize("env_id", MOBILE_IDS)
def test_batched_fpv_observation(use_checker_backend, checker_backend, env_id):
    from srl_sim.vec_env import BatchedSRLVecEnv
    n = 3
    kw = dict(seed=4, srl_model="raw_pixels", random_target=True)
    venv = BatchedSRLVecEnv(env_id, n, fpv=True, **kw)
    top = BatchedSRLVecEnv(env_id, n, **kw)
    assert venv.observation_space.shape == (224, 224, 6)
    o, o_top = venv.reset(), top.reset()
    assert o.shape == (n, 224, 224, 6) and o.dtype == np.uint8
    assert np.array_equal(o[..., :3], o_top)
    n_act = venv.action_space.n
    for t in range(6):
        a = [(t + i) % n_act for i in range(n)]
        o, _, _, _ = venv.step(a)
        o_top, _, _, _ = top.step(a)
    assert o.shape == (n, 224, 224, 6)
    assert np.array_equal(o[..., :3], o_top)
    pos = venv.sim.get_state(_abi.F_ROBOT_POS)
    want = single_camera_frames(checker_backend, venv.sim, [mobile_fpv_camera(p) for p in pos], 224, 224)
    assert np.array_equal(o[..., 3:], want)
    assert np.array_equal(venv.render_tensors(), o)
    assert len(venv.get_images()) == n and venv.get_images()[0].shape == (224, 224, 6)
    venv.close(); top.close()


def test_kuka_ignores_fpv(use_checker_backend):
    from srl_sim.vec_env import BatchedSRLVecEnv
    venv = BatchedSRLVecEnv("KukaButtonGymEnv-v0", 2, srl_model="raw_pixels", fpv=True)
    assert venv.observation_space.shape == (224, 224, 3)
    assert venv.reset().shape == (2, 224, 224, 3)
    venv.close()


def test_refusals_carry_the_library_message(checker_backend):
    be = checker_backend
    kuka = be.make_sim("KukaButtonGymEnv-v0", 2, model_blob=load_kuka_scene().blob)
    kuka.reset()
    buf = np.zeros((2, 16, 16, 3), np.uint8)
    with pytest.raises(_abi.SimError, match="follow_robot"):
        kuka.render_cameras(camera_array([KUKA_CAMERA] * 2), True, 16, 16, buf)
    mob = be.make_sim("MobileRobotGymEnv-v0", 2)
    mob.reset()
    cams = camera_array([MOBILE_CAMERA] * 2)
    with pytest.raises(_abi.SimError, match="null argument"):
        mob.render_cameras(None, False, 16, 16, buf)
    with pytest.raises(_abi.SimError, match="null argument"):
        mob.render_cameras(cams, False, 16, 16, None)
    with pytest.raises(_abi.SimError, match="bad image size"):
        mob.render_cameras(cams, False, 0, 16, buf)
    bad = camera_array([MOBILE_CAMERA, dict(MOBILE_CAMERA, fov=0.0)])
    with pytest.raises(_abi.SimError, match="bad camera 1"):
        mob.render_cameras(bad, False, 16, 16, buf)
    with pytest.raises(ValueError):
        mob.render_cameras(camera_array([MOBILE_CAMERA] * 3), False, 16, 16, buf)
    kuka.close(); mob.close()
