"""
The sm_90a ray caster pixel by pixel against the independent float64 reference (tests/render_numpy_ref.py), both drawing the CUDA handle's
own state (read with get_state from the handle that renders): srl_sim_render, srl_sim_render_cameras with mixed cameras and with
follow_robot, every env id and KukaRandButton with its bodies after they have fallen and been kicked, the env cameras and random ones (roll,
pitch -90 and -89.9, fov 20 to 120), frame sizes from 1 x 1 to 640 x 480, batches of 1, 33 and 4096 envs, and a 65600-env batch past the
65535 grid.z chunk of the raster and JPEG launches.

Tolerance: every channel of a stable pixel within +-1 of the reference, an unstable pixel within +-1 of one of its candidate colours, and
the share of unstable pixels bounded per case at about twice what was measured (UNSTABLE_BOUND; the test prints the measured shares).
"""
import numpy as np
import pytest

import render_numpy_ref as R
from srl_sim import _abi, jpeg
from srl_sim.render import KUKA_CAMERA, MOBILE_CAMERA, MOBILE_FPV_FOLLOW, camera, camera_array
from test_render_cameras_cpu import MOBILE_IDS
from test_render_reference_cpu import check_frames, env_cameras, make_sim

pytestmark = pytest.mark.gpu

ENV_IDS = sorted(_abi.ENV_KINDS)
SIZES = ((1, 1), (7, 5), (32, 16), (33, 17), (320, 96), (48, 200))
# Share of unstable pixels per case, about twice the largest measured on an H100 80GB HBM3 (the test prints them; measured: Kuka env
# cameras 0.012-0.053 with or without bodies, MobileRobot top-down 0.0001-0.0008, sweep and per-env cameras of 1024 pixels or more
# 0.001-0.056, follow_robot 0.011-0.023, frames under 1024 pixels up to 0.29).  Kuka frames have more silhouette and joint pixels than the
# flat MobileRobot ones, and the sides of the button's thin cylinders sit within float32 reach of srl_normal_at's cap band; a sweep camera
# can look along a table edge or at the horizon; a 1 x 1 frame's one pixel may be an edge.
UNSTABLE_BOUND = {"kuka env camera": 0.11, "bodies": 0.08, "mobile env camera": 0.002, "kuka sweep": 0.12, "mobile sweep": 0.12,
                  "follow_robot": 0.045, "small": 0.6, "tiny": 1.0}


def _case(env_id, kind):
    return ("kuka " if env_id.startswith("Kuka") else "mobile ") + kind


def _render(be, sim, cam, w, h):
    buf = be.zeros((sim.num_envs, h, w, 3), np.uint8)
    sim.render(camera(**cam), w, h, buf, stream=be.stream())
    return be.to_host(buf).copy()


def _render_cameras(be, sim, cams, follow, w, h):
    buf = be.zeros((sim.num_envs, h, w, 3), np.uint8)
    sim.render_cameras(camera_array(cams), follow, w, h, buf, stream=be.stream())
    return be.to_host(buf).copy()


def _follow_absolute(pos, offs):
    """The camera a follow_robot call gives env i: target x, y = float32(float64 position + float64(float32 offset)), z as given."""
    return [dict(c, target=(float(np.float32(p[0] + np.float64(np.float32(c["target"][0])))),
                            float(np.float32(p[1] + np.float64(np.float32(c["target"][1])))), c["target"][2])) for p, c in zip(pos, offs)]


def _report(stats, label, share, bound):
    stats.append((label, share, bound))
    print("UNSTABLE %-52s %.5f (bound %.3f)" % (label, share, bound))
    assert share <= bound, (label, share, bound)


def _check(frames, env_id, st, cams, kind, stats, label, **kw):
    """check_frames, then the share of unstable pixels over the checked frames against the case's bound (frames of fewer than 1024 pixels
    are a case of their own: a few edge pixels are a large share of them; a 1 x 1 frame's one pixel may be an edge)."""
    if frames.shape[1] * frames.shape[2] < 16:
        kind = "tiny"
    elif frames.shape[1] * frames.shape[2] < 1024:
        kind = "small"
    bound = UNSTABLE_BOUND[kind] if kind in UNSTABLE_BOUND else UNSTABLE_BOUND[_case(env_id, kind)]
    share = check_frames(frames, env_id, st, cams, label=label, **kw)
    _report(stats, "%s %s %s" % (env_id, label, frames.shape[1:3]), share, bound)


@pytest.mark.parametrize("env_id", ENV_IDS + ["KukaRandButtonGymEnv-v0+distractors"])
def test_cuda_frames_match_the_reference(cuda_backend, env_id):
    """33 envs mid-episode (after an auto-reset, except MobileRobot2Target; with bodies: 30 steps, so they have fallen and the sphere has
    been kicked), srl_sim_render through the env cameras at 224 x 224 and a sweep camera per size; three envs per frame set, first and last
    included."""
    be = cuda_backend
    distractors = env_id.endswith("+distractors")
    env_id = env_id.split("+")[0]
    n = 33
    max_steps = 0 if (distractors or env_id == "MobileRobot2TargetGymEnv-v0") else 9
    sim, targets = make_sim(be, env_id, n, 30 if distractors else 14, seed=17 + len(env_id), max_steps=max_steps, distractors=distractors)
    st = R.read_state(sim, env_id)
    bodies = sim.get_state(_abi.F_DISTRACTORS).reshape(n, 11, 9) if distractors else None
    if distractors:       # the kicked sphere (slot 10) has left its spawn point (0.25, -0.2) in most envs
        assert (np.hypot(bodies[:, 10, 0] - 0.25, bodies[:, 10, 1] + 0.2) > 0.05).mean() > 0.5, bodies[:, 10, :3]
    envs = (0, 16, n - 1)
    stats = []
    kw = dict(bodies=bodies, targets=targets, envs=envs)
    for cam in env_cameras(env_id):
        _check(_render(be, sim, cam, 224, 224), env_id, st, cam, "bodies" if distractors else "env camera", stats, "env camera", **kw)
    sizes = SIZES + (((640, 480),) if env_id in ("KukaButtonGymEnv-v0", "MobileRobotGymEnv-v0") or distractors else ())
    for cam, (w, h) in zip(R.sweep_cameras(env_id, len(sizes), seed=3 + len(env_id)), sizes):
        _check(_render(be, sim, cam, w, h), env_id, st, cam, "sweep", stats, "sweep", **dict(kw, envs=(0, n - 1) if w * h > 20000 else envs))
    sim.close()


@pytest.mark.parametrize("env_id", ENV_IDS + ["KukaRandButtonGymEnv-v0+distractors"])
def test_cuda_per_env_cameras_match_the_reference(cuda_backend, env_id):
    """srl_sim_render_cameras, every env through its own camera (the env cameras and sweep cameras with roll), at 224 x 224 and odd sizes."""
    be = cuda_backend
    distractors = env_id.endswith("+distractors")
    env_id = env_id.split("+")[0]
    n = 33
    sim, targets = make_sim(be, env_id, n, 24 if distractors else 10, seed=29, distractors=distractors)
    st = R.read_state(sim, env_id)
    bodies = sim.get_state(_abi.F_DISTRACTORS).reshape(n, 11, 9) if distractors else None
    cams = (env_cameras(env_id) + R.sweep_cameras(env_id, n, seed=41))[:n]
    stats = []
    for (w, h), envs in (((224, 224), (0, 1, 2, n - 1)), ((33, 17), range(n)), ((7, 5), range(n))):
        frames = _render_cameras(be, sim, cams, False, w, h)
        _check(frames, env_id, st, cams, "sweep", stats, "per-env", bodies=bodies, targets=targets, envs=envs)
    sim.close()


@pytest.mark.parametrize("env_id", MOBILE_IDS)
def test_cuda_follow_robot_matches_the_reference(cuda_backend, env_id):
    """follow_robot: the first-person camera and rolled / wider variants of it, the reference's target float32(float64 position + offset)."""
    be = cuda_backend
    n = 33
    sim, targets = make_sim(be, env_id, n, 12, seed=31)
    st = R.read_state(sim, env_id)
    rs = np.random.RandomState(7)
    offs = [dict(MOBILE_FPV_FOLLOW)] + [dict(MOBILE_FPV_FOLLOW, roll=rs.uniform(-60, 60), fov=rs.uniform(20, 120), yaw=rs.uniform(0, 360))
                                        for _ in range(n - 1)]
    absolute = _follow_absolute(st["robot"], offs)
    stats = []
    for (w, h) in ((224, 224), (48, 200), (33, 17)):
        frames = _render_cameras(be, sim, offs, True, w, h)
        _check(frames, env_id, st, absolute, "follow_robot", stats, "follow_robot", targets=targets, envs=(0, 5, 17, n - 1))
    sim.close()


@pytest.mark.parametrize("env_id", ["KukaButtonGymEnv-v0", "MobileRobotGymEnv-v0"])
@pytest.mark.parametrize("n", [1, 4096])
def test_batch_sizes_match_the_reference(cuda_backend, env_id, n):
    """n = 1 and 4096 (the 33-env cases are above): both entry points, the first and last env and a sample between."""
    be = cuda_backend
    sim, _ = make_sim(be, env_id, n, 12, seed=5, max_steps=9)
    st = R.read_state(sim, env_id)
    envs = sorted({0, n // 3, n // 2, n - 2, n - 1} & set(range(n)))
    stats = []
    cam = env_cameras(env_id)[0]
    _check(_render(be, sim, cam, 224, 224), env_id, st, cam, "env camera", stats, "n=%d" % n, envs=envs)
    cams = R.sweep_cameras(env_id, min(n, 64), seed=n)
    cams = [cams[i % len(cams)] for i in range(n)]
    _check(_render_cameras(be, sim, cams, False, 64, 48), env_id, st, cams, "sweep", stats, "per-env n=%d" % n, envs=envs)
    sim.close()


def test_batch_past_the_grid_z_chunk(cuda_backend):
    """65600 MobileRobot envs (0.4 GB of primitive lists, 50 MB of 16 x 16 frames): the raster launch is split at 65535 envs.  Envs on both
    sides of the split against the reference through both entry points, and the per-env path equal to srl_sim_render on every env."""
    be = cuda_backend
    env_id, n, w, h = "MobileRobotGymEnv-v0", 65600, 16, 16
    sim, _ = make_sim(be, env_id, n, 6, seed=13)
    st = R.read_state(sim, env_id)
    envs = (0, 65534, 65535, 65536, n - 1)
    stats = []
    cam = dict(MOBILE_CAMERA, fov=75.0)
    single = _render(be, sim, cam, w, h)
    _check(single, env_id, st, cam, "env camera", stats, "n=65600", envs=envs)
    same = _render_cameras(be, sim, [cam] * n, False, w, h)
    assert np.array_equal(same, single), int((same != single).any(axis=(1, 2, 3)).sum())
    follow = [dict(MOBILE_FPV_FOLLOW, yaw=float(90 + 10 * (i % 7))) for i in range(n)]
    frames = _render_cameras(be, sim, follow, True, w, h)
    _check(frames, env_id, st, _follow_absolute(st["robot"], follow), "follow_robot", stats, "follow_robot n=65600", envs=envs)
    assert len({frames[i].tobytes() for i in envs}) == len(envs)
    sim.close()


class _Host(object):
    on_gpu = False


def test_jpeg_past_the_grid_z_chunk(cuda_backend):
    """srl_jpeg_encode on 65600 frames of 16 x 16 (its block launch is split at 65535 frames): rendered frames mixed with noise, packed and
    strided output, both byte for byte the CPU checker's files."""
    be = cuda_backend
    torch = be.torch
    n, w, h = 65600, 16, 16
    sim, _ = make_sim(be, "MobileRobotGymEnv-v0", 64, 4, seed=3)
    pool = np.concatenate([_render(be, sim, c, w, h) for c in (MOBILE_CAMERA, dict(MOBILE_CAMERA, distance=2.0, pitch=-40.0, yaw=30.0))])
    sim.close()
    rng = np.random.default_rng(9)
    frames = pool[rng.integers(0, len(pool), n)]
    noisy = rng.random(n) < 0.3
    frames[noisy] = rng.integers(0, 256, (int(noisy.sum()), h, w, 3), dtype=np.uint8)
    frames[65535] = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)        # the first frame of the second launch, and its neighbours differ
    frames[65534] = pool[0]
    want = jpeg.encode_jpeg(_Host(), frames, quality=90)
    dev = torch.from_numpy(frames).to(be.torch_device)
    assert jpeg.encode_jpeg(be, dev, quality=90) == want                 # packed
    lib = jpeg.bind(be.library.lib)
    b = int(lib.srl_jpeg_bound(w, h))
    ws = torch.empty(int(lib.srl_jpeg_workspace_bytes(n, w, h)), dtype=torch.uint8, device=dev.device)
    out = torch.zeros(n * b, dtype=torch.uint8, device=dev.device)
    lens = torch.zeros(n, dtype=torch.int32, device=dev.device)
    rc = lib.srl_jpeg_encode(dev.data_ptr(), n, h, w, 3, 0, 90, ws.data_ptr(), out.data_ptr(), b, lens.data_ptr(), be.stream())
    be.library.check(rc, "srl_jpeg_encode")
    o, k = out.cpu().numpy(), lens.cpu().numpy()
    assert [o[i * b:i * b + k[i]].tobytes() for i in range(n)] == want  # strided
    jpeg.release_buffers()
