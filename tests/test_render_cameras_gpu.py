"""
One camera per env (srl_sim_render_cameras) on the sm_90a library: the per-env path (prepare_kernel<true>, raster_kernel<..., true> and, with
follow_robot, follow_cams_kernel) gives env i the bytes srl_sim_render(cameras[i]) gives it on the same handle, at every size, batch size and
registry id; the camera cache never serves stale cameras; and BatchedSRLVecEnv(fpv=True) renders the first-person frames of a full batch.
"""
import numpy as np
import pytest

from srl_sim import _abi
from srl_sim.render import MOBILE_FPV_FOLLOW, camera, camera_array, mobile_fpv_camera, render_cameras

from test_render_cameras_cpu import MOBILE_IDS, follow_targets, mid_episode_sim, mixed_cameras

pytestmark = pytest.mark.gpu

SIZES = ((224, 224), (64, 64), (50, 33), (96, 40))


def _pool(env_id, n, seed):
    """n cameras drawn from a pool of at most 16 different ones, the pool's cameras spread over the envs at random; returns (cams, pool, which)."""
    k = min(n, 16)
    pool = mixed_cameras(env_id, k, seed)
    which = np.arange(n) % k
    np.random.RandomState(seed).shuffle(which)
    return [pool[j] for j in which], pool, which


def _expect_single_calls(be, sim, got, pool, which, w, h):
    """got[i] == frame i of srl_sim_render(pool[which[i]]), compared on the device."""
    torch = be.torch
    idx = torch.from_numpy(which).to(got.device)
    for j, c in enumerate(pool):
        ref = be.zeros((sim.num_envs, h, w, 3), np.uint8)
        sim.render(camera(**c), w, h, ref, stream=be.stream())
        sel = idx == j
        diff = int((got[sel] != ref[sel]).sum())
        assert diff == 0, (j, c, w, h, diff)


@pytest.mark.parametrize("n", [1, 33, 4096])
@pytest.mark.parametrize("env_id", sorted(_abi.ENV_KINDS) + ["KukaRandButtonGymEnv-v0+distractors"])
def test_mixed_cameras_match_single_camera_calls(cuda_backend, env_id, n):
    be = cuda_backend
    distractors = env_id.endswith("+distractors")
    env_id = env_id.split("+")[0]
    sim = mid_episode_sim(be, env_id, n, 24 if distractors else 12, distractors=distractors)
    cams, pool, which = _pool(env_id, n, seed=n + len(env_id))
    arr = camera_array(cams)
    for (w, h) in SIZES:
        got = render_cameras(sim, be, arr, width=w, height=h)
        _expect_single_calls(be, sim, got, pool, which, w, h)
    be.torch.cuda.synchronize()
    sim.close()


@pytest.mark.parametrize("n", [1, 33, 4096])
@pytest.mark.parametrize("env_id", MOBILE_IDS)
def test_follow_robot_matches_the_absolute_cameras(cuda_backend, env_id, n):
    """follow_robot frames == the per-env path with the absolute targets (itself == srl_sim_render, above), and for a few envs directly
    == srl_sim_render(mobile_fpv_camera(robot position))."""
    be = cuda_backend
    sim = mid_episode_sim(be, env_id, n, 30, seed=9)
    pos = sim.get_state(_abi.F_ROBOT_POS)
    rs = np.random.RandomState(n)
    cams = [MOBILE_FPV_FOLLOW if i % 2 == 0 else
            dict(MOBILE_FPV_FOLLOW, target=(rs.uniform(-0.5, 0.5), rs.uniform(-0.5, 0.5), rs.uniform(0.05, 0.4)), yaw=rs.uniform(0, 360),
                 pitch=rs.uniform(-40, -5), fov=rs.uniform(50, 100)) for i in range(n)]
    follow, absolute = camera_array(cams), camera_array(follow_targets(pos, cams))
    for (w, h) in SIZES:
        got = render_cameras(sim, be, follow, follow_robot=True, width=w, height=h)
        want = render_cameras(sim, be, absolute, width=w, height=h)
        assert be.torch.equal(got, want), (env_id, n, w, h, int((got != want).sum()))
        for i in sorted({0, n // 2, n - 1}):
            ref_cam = mobile_fpv_camera(pos[i]) if cams[i] is MOBILE_FPV_FOLLOW else follow_targets(pos[i:i + 1], cams[i:i + 1])[0]
            ref = be.zeros((n, h, w, 3), np.uint8)
            sim.render(camera(**ref_cam), w, h, ref, stream=be.stream())
            assert be.torch.equal(got[i], ref[i]), (env_id, n, w, h, i)
    sim.close()


def test_camera_cache_never_serves_stale_cameras(cuda_backend):
    """The handle skips its camera set-up when a call passes the bytes of the previous one: A, B, A (the same array object and a fresh copy),
    a size change, and follow_robot switched on and off with the same bytes must each draw their own cameras."""
    be = cuda_backend
    env_id, n = "MobileRobotGymEnv-v0", 33
    sim = mid_episode_sim(be, env_id, n, 20, seed=2)
    cams_a, pool_a, which_a = _pool(env_id, n, seed=1)
    cams_b, pool_b, which_b = _pool(env_id, n, seed=2)
    a, b = camera_array(cams_a), camera_array(cams_b)
    for arr, pool, which, (w, h) in ((a, pool_a, which_a, (64, 64)), (b, pool_b, which_b, (64, 64)), (a, pool_a, which_a, (64, 64)),
                                     (camera_array(cams_a), pool_a, which_a, (64, 64)), (a, pool_a, which_a, (50, 33)),
                                     (a, pool_a, which_a, (64, 64))):
        got = render_cameras(sim, be, arr, width=w, height=h)
        _expect_single_calls(be, sim, got, pool, which, w, h)
    # the same bytes as offsets (follow_robot) and back
    pos = sim.get_state(_abi.F_ROBOT_POS)
    got = render_cameras(sim, be, a, follow_robot=True, width=64, height=64)
    assert be.torch.equal(got, render_cameras(sim, be, camera_array(follow_targets(pos, cams_a)), width=64, height=64))
    got = render_cameras(sim, be, a, width=64, height=64)
    _expect_single_calls(be, sim, got, pool_a, which_a, 64, 64)
    # follow_robot with cached cameras after the robots have moved
    fpv = camera_array([MOBILE_FPV_FOLLOW] * n)
    render_cameras(sim, be, fpv, follow_robot=True)
    acts = be.from_host(np.full((5, n), 1, np.int32))
    obs = be.zeros((5, n, sim.obs_dim), np.float32); rew = be.zeros((5, n), np.float32); done = be.zeros((5, n), np.uint8)
    sim.rollout(5, acts, None, obs, rew, done, stream=be.stream())
    pos2 = sim.get_state(_abi.F_ROBOT_POS)
    assert not np.array_equal(pos, pos2)
    got = render_cameras(sim, be, fpv, follow_robot=True)
    want = render_cameras(sim, be, camera_array([mobile_fpv_camera(p) for p in pos2]))
    assert be.torch.equal(got, want)
    sim.close()


@pytest.mark.parametrize("env_id", ["KukaButtonGymEnv-v0", "KukaRandButtonGymEnv-v0+distractors", "MobileRobotGymEnv-v0",
                                    "MobileRobotLineTargetGymEnv-v0"])
def test_culling_never_changes_a_byte(cuda_backend, env_id, monkeypatch):
    be = cuda_backend
    distractors = env_id.endswith("+distractors")
    env_id = env_id.split("+")[0]
    n = 64
    sim = mid_episode_sim(be, env_id, n, 40, seed=11, distractors=distractors)
    cams = camera_array(_pool(env_id, n, seed=3)[0])
    follow = camera_array([MOBILE_FPV_FOLLOW] * n) if env_id.startswith("Mobile") else None
    for (w, h) in SIZES:
        out = []
        for no_cull in (False, True):
            if no_cull:
                monkeypatch.setenv("SRL_RENDER_NO_CULL", "1")
            else:
                monkeypatch.delenv("SRL_RENDER_NO_CULL", raising=False)
            frames = [be.to_host(render_cameras(sim, be, cams, width=w, height=h)).copy()]
            if follow is not None:
                frames.append(be.to_host(render_cameras(sim, be, follow, follow_robot=True, width=w, height=h)).copy())
            out.append(frames)
        for x, y in zip(out[0], out[1]):
            assert np.array_equal(x, y), (env_id, w, h, int((x != y).sum()))
    monkeypatch.delenv("SRL_RENDER_NO_CULL", raising=False)
    sim.close()


@pytest.mark.parametrize("env_id", sorted(_abi.ENV_KINDS))
def test_cuda_per_env_cameras_match_the_cpu_checker(cuda_backend, oracle_backend, env_id):
    """float32 kernel state vs float64 oracle state: silhouette pixels may fall on the other side of an edge, so >= 99.5 % of the bytes."""
    n = 6
    cams = mixed_cameras(env_id, n, seed=4)
    frames = {}
    for tag, be in (("cuda", cuda_backend), ("oracle", oracle_backend)):
        sim = mid_episode_sim(be, env_id, n, 12, seed=3)
        out = [be.to_host(render_cameras(sim, be, cams)).copy(), be.to_host(render_cameras(sim, be, cams, width=50, height=33)).copy()]
        if env_id.startswith("Mobile"):
            out.append(be.to_host(render_cameras(sim, be, [MOBILE_FPV_FOLLOW] * n, follow_robot=True)).copy())
        frames[tag] = out
        sim.close()
    for a, b in zip(frames["cuda"], frames["oracle"]):
        same = (a == b).mean()
        assert same > 0.995, (env_id, same)


def test_batched_fpv_vec_env(cuda_lib):
    from srl_sim import backend
    backend.use_library(None, None)
    import torch
    from srl_sim.vec_env import BatchedSRLVecEnv
    n = 4096
    venv = BatchedSRLVecEnv("MobileRobotGymEnv-v0", n, seed=1, srl_model="raw_pixels", fpv=True, random_target=True)
    assert venv.observation_space.shape == (224, 224, 6)
    venv.reset()
    rs = np.random.RandomState(0)
    for _ in range(4):
        venv.step_tensors(torch.from_numpy(rs.randint(0, 4, n).astype(np.int32)).cuda())
    t = venv.render_tensors()
    assert t.is_cuda and t.dtype == torch.uint8 and tuple(t.shape) == (n, 224, 224, 6)
    follow = render_cameras(venv.sim, venv.backend, [MOBILE_FPV_FOLLOW] * n, follow_robot=True)
    assert torch.equal(t[..., 3:], follow)
    top = venv.backend.zeros((n, 224, 224, 3), np.uint8)
    venv.sim.render(camera(**venv._cams[0]), 224, 224, top, stream=venv.backend.stream())
    assert torch.equal(t[..., :3], top)
    for _ in range(2):
        venv.render_tensors()
    torch.cuda.synchronize()
    reps = 5
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        venv.render_tensors()
    e1.record()
    torch.cuda.synchronize()
    print("FPV RENDER: 4096 MobileRobot envs, top-down + first-person frames of 224 x 224 (render_tensors) in %.2f ms"
          % (e0.elapsed_time(e1) / reps))
    venv.close()
