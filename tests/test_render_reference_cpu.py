"""
The CPU checker's frames (oracle/liboracle_sim.so, and the two test checkers for per-env cameras and caller-given bodies) pixel by pixel
against the independent float64 ray caster of tests/render_numpy_ref.py, both reading the same oracle handle's state.

The checker and the CUDA kernels compile the same per-pixel arithmetic (csrc/render_core.h), so a stable pixel that disagrees here is a bug
the kernels share.  Tolerance: every channel of a stable pixel within +-1 of the reference, an unstable pixel within +-1 of one of its
candidate colours.  The reference itself is first held to analytic cases, so that it cannot be wrong in the same way as the kernels.
"""
import numpy as np
import pytest

import render_numpy_ref as R
from srl_sim import _abi
from srl_sim.model import distractor_blob, load_kuka_scene
from srl_sim.render import KUKA_CAMERA, KUKA_CAMERA_2, MOBILE_CAMERA, MOBILE_FPV_FOLLOW, camera, camera_array

ENV_IDS = sorted(_abi.ENV_KINDS)
BG = np.floor(R.BACKGROUND * 255 + 0.5)


# ---- the reference on analytic cases ------------------------------------------------------------------------------------------------
def _hits(frame):
    return np.any(frame.astype(int) != BG, axis=-1)


def _shade_bytes(rgb, n):
    n = np.asarray(n, float) / np.linalg.norm(n)
    return np.floor(np.asarray(rgb) * (0.55 + 0.45 * max(n @ R.LIGHT, 0.0)) * 255 + 0.5)


def _pixel_radii(W, H):
    ys, xs = np.mgrid[0:H, 0:W]
    return np.hypot(xs + 0.5 - W / 2, ys + 0.5 - H / 2)


def test_reference_sphere_straight_ahead():
    """A sphere at the camera's target: a disc whose radius in pixels follows from the fov, centre pixel shaded with n = -d."""
    W = H = 101
    for fov, dist, r, yaw, pitch in ((60.0, 3.0, 0.5, 200.0, -30.0), (30.0, 10.0, 0.7, 20.0, -60.0), (100.0, 2.0, 0.3, 120.0, 10.0)):
        c = np.array([0.3, -0.2, 0.4])
        cam = dict(target=tuple(c), distance=dist, yaw=yaw, pitch=pitch, roll=0.0, fov=fov)
        rgb, unstable = R.render([R.sphere(c, r, (0.2, 0.6, 0.9))], cam, W, H)[:2]
        cam32 = {k: np.float32(v) for k, v in cam.items() if k != "target"}
        rpx = np.tan(np.arcsin(r / float(cam32["distance"]))) / np.tan(np.radians(float(cam32["fov"])) / 2) * H / 2
        rad, hit = _pixel_radii(W, H), _hits(rgb)
        assert hit[rad < rpx - 0.6].all() and not hit[rad > rpx + 0.6].any(), (fov, rpx)
        assert not unstable[np.abs(rad - rpx) > 1.0].any()
        _, D = R.camera_rays(cam, W, H)
        assert np.allclose(rgb[H // 2, W // 2], _shade_bytes((0.2, 0.6, 0.9), -D[(H // 2) * W + W // 2]), atol=0)


def test_reference_box_face_on():
    """An axis-aligned box seen from straight above: a rectangle of the top face's projected size, every pixel shaded with n = +z."""
    W, H, fov, dist = 120, 80, 50.0, 4.0
    half = np.array([0.6, 0.3, 0.2])
    cam = dict(target=(0.0, 0.0, 0.0), distance=dist, yaw=0.0, pitch=-90.0, roll=0.0, fov=fov)
    rgb, unstable = R.render([R.box((0, 0, 0), half, 0.0, (0.9, 0.5, 0.1))], cam, W, H)[:2]
    hit = _hits(rgb)
    f = H / 2 / np.tan(np.radians(np.float32(fov)) / 2)
    ys, xs = np.nonzero(hit)
    width, height = xs.max() - xs.min() + 1, ys.max() - ys.min() + 1
    # yaw 0, pitch -90: image right is +x, image up is +y
    assert abs(width - 2 * half[0] / (dist - half[2]) * f) < 1.5 and abs(height - 2 * half[1] / (dist - half[2]) * f) < 1.5, (width, height)
    assert (rgb[hit & ~unstable] == _shade_bytes((0.9, 0.5, 0.1), (0, 0, 1))).all()


def test_reference_capsule_end_on_and_side_on():
    W = H = 81
    e0, e1, r = np.array([0.0, 0.0, 0.0]), np.array([0.0, 1.0, 0.0]), 0.2
    caps = [R.capsule(e0, e1, r, (0.5, 0.5, 0.5))]
    # end-on: the camera looks along +y from y = -3 (yaw 0, pitch 0): a disc of the near end sphere's angular radius
    cam = dict(target=(0.0, 0.0, 0.0), distance=3.0, yaw=0.0, pitch=0.0, roll=0.0, fov=40.0)
    rgb = R.render(caps, cam, W, H)[0]
    rpx = np.tan(np.arcsin(r / 3.0)) / np.tan(np.radians(20.0)) * H / 2
    rad, hit = _pixel_radii(W, H), _hits(rgb)
    assert hit[rad < rpx - 0.6].all() and not hit[rad > rpx + 0.6].any()
    # side-on from +x above the middle: a band 2r wide and |e1 - e0| + 2r long (the ends are hemispheres)
    cam = dict(target=(0.0, 0.5, 0.0), distance=4.0, yaw=90.0, pitch=-89.9, roll=0.0, fov=40.0)
    rgb = R.render(caps, cam, W, H)[0]
    hit = _hits(rgb)
    f = H / 2 / np.tan(np.radians(20.0))
    ys, xs = np.nonzero(hit)
    long_side, short_side = max(np.ptp(xs), np.ptp(ys)) + 1, min(np.ptp(xs), np.ptp(ys)) + 1
    assert abs(long_side - 1.4 / 4.0 * f) < 2.5 and abs(short_side - 0.4 / 4.0 * f) < 2.5, (long_side, short_side)
    # the middle of the band is the side cylinder: its normal there points at the camera (n = +z seen from above)
    assert np.allclose(rgb[H // 2, W // 2], _shade_bytes((0.5, 0.5, 0.5), (0, 0, 1)), atol=1)


def _agree(a, b):
    """Two reference renders give the same bytes wherever both are stable."""
    both = ~a[1] & ~b[1]
    assert both.mean() > 0.95 and np.array_equal(a[0][both], b[0][both]), int((a[0] != b[0]).any(-1)[both].sum())


def test_reference_oriented_box_rotations():
    """OBOX rotated 90 degrees about z is the BOX with swapped half extents; q and -q draw the same frame; a roll of 180 degrees at pitch 0
    turns the frame upside down."""
    half = (0.3, 0.12, 0.2)
    s = np.sqrt(0.5)
    cams = [dict(target=(0.0, 0.0, 0.0), distance=2.0, yaw=35.0, pitch=-40.0, roll=0.0, fov=60.0),
            dict(target=(0.1, 0.0, 0.1), distance=1.5, yaw=250.0, pitch=-70.0, roll=20.0, fov=45.0)]
    for cam in cams:
        a = R.render([R.obox((0, 0, 0), half, (0, 0, s, s), (0.2, 0.8, 0.4))], cam, 64, 48)
        b = R.render([R.box((0, 0, 0), (half[1], half[0], half[2]), 0.0, (0.2, 0.8, 0.4))], cam, 64, 48)
        assert _hits(a[0]).sum() > 60
        _agree(a, b)
        q = np.array([0.3, -0.5, 0.2, 0.7]); q /= np.linalg.norm(q)
        _agree(R.render([R.obox((0, 0, 0), half, q, (0.9, 0.9, 0.1))], cam, 64, 48),
               R.render([R.obox((0, 0, 0), half, -q, (0.9, 0.9, 0.1))], cam, 64, 48))
    prims = [R.plane(-0.5, 1.0, (1, 1, 1)), R.obox((0.2, 0.1, 0.0), half, q, (0.9, 0.9, 0.1)), R.sphere((-0.3, 0.2, 0.1), 0.15, (1, 0, 0))]
    cam = dict(target=(0.0, 0.0, 0.0), distance=2.5, yaw=30.0, pitch=0.0, roll=0.0, fov=60.0)
    up = R.render(prims, cam, 64, 48)
    down = R.render(prims, dict(cam, roll=180.0), 64, 48)
    _agree(up, tuple(x[::-1, ::-1] for x in down))


# ---- the CPU checker against the reference -------------------------------------------------------------------------------------------
def check_frames(frames, env_id, st, cams, scene=None, bodies=None, targets=None, envs=None, label=""):
    """Every env in `envs` (all by default): frame i through cams[i] (or the one camera `cams`) against the reference.  Returns the share of
    unstable pixels over these frames."""
    n, H, W = frames.shape[:3]
    fracs = []
    for i in (range(n) if envs is None else envs):
        cam = cams[i] if isinstance(cams, list) else cams
        prims = R.env_prims(env_id, st, i, scene, None if bodies is None else bodies[i], None if targets is None else targets[i])
        ref = R.render(prims, cam, W, H)
        bad, frac, first = R.compare(frames[i], ref)
        fracs.append(frac)
        assert bad == 0, "%s %s env %d %s %dx%d: %d pixels off, first (y, x) = %s: %s, reference %s, unstable %s, candidates %s" % (
            label, env_id, i, cam, W, H, bad, first, frames[i][first], ref[0][first], ref[1][first], ref[2][first].tolist())
    return float(np.mean(fracs))


def rollout(be, sim, env_id, T, seed):
    n = sim.num_envs
    n_act = 6 if env_id.startswith("Kuka") else (2 if env_id == "MobileRobot1DGymEnv-v0" else 4)
    acts = np.random.RandomState(seed).randint(0, n_act, size=(T, n)).astype(np.int32)
    obs = be.zeros((T, n, sim.obs_dim), np.float32); rew = be.zeros((T, n), np.float32); done = be.zeros((T, n), np.uint8)
    sim.rollout(T, be.from_host(acts), None, obs, rew, done, stream=be.stream())
    return be.to_host(done).copy()


def make_sim(be, env_id, n, T, seed, max_steps=0, distractors=False):
    """A handle of n envs after T random steps; with max_steps every env has auto-reset on the way.  MobileRobot2Target envs start from
    host-supplied reset draws (a masked reset), so both of their targets are known: returns (sim, targets or None)."""
    kuka = env_id.startswith("Kuka")
    sim = be.make_sim(env_id, n, model_blob=load_kuka_scene().blob if kuka else None, seed=seed, random_target=True, max_steps=max_steps)
    if distractors:
        sim.set_distractors(distractor_blob())
    sim.reset(stream=be.stream())
    targets = None
    if env_id == "MobileRobot2TargetGymEnv-v0":
        # oracle_mobile.cpp: draws = robot (x, y), target 0 (x, y), target 1 (x, y)
        draws = np.random.RandomState(seed).uniform(0.5, 3.5, size=(n, _abi.MOBILE_RESET_DRAWS))
        sim.reset(mask=be.from_host(np.ones(n, np.uint8)), reset_draws=be.from_host(draws), stream=be.stream())
        targets = draws[:, 2:6]
    if T:
        done = rollout(be, sim, env_id, T, seed + 1)
        if targets is not None:
            assert not done.any(), "the 2-target envs must not reset: their new targets would be unknown"
        elif max_steps:
            assert done.any(axis=0).all(), "every env should have auto-reset"
    return sim, targets


def env_cameras(env_id):
    return [KUKA_CAMERA, KUKA_CAMERA_2] if env_id.startswith("Kuka") else [MOBILE_CAMERA]


@pytest.fixture(scope="module")
def checker_backend():
    import render_cameras_ref
    from srl_sim.backend import Backend
    return Backend(render_cameras_ref.library(), -1)


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_checker_frames_match_the_reference(oracle_backend, env_id):
    """Mid-episode and (except MobileRobot2Target, whose redrawn targets get_state cannot show) after an auto-reset: the env cameras at
    224 x 224 and a sweep of random cameras with roll at 64 x 48, every pixel."""
    be = oracle_backend
    n = 2
    max_steps = 0 if env_id == "MobileRobot2TargetGymEnv-v0" else 9
    sim, targets = make_sim(be, env_id, n, 14, seed=5 + len(env_id), max_steps=max_steps)
    st = R.read_state(sim, env_id)
    for cam in env_cameras(env_id):
        buf = np.zeros((n, 224, 224, 3), np.uint8)
        sim.render(camera(**cam), 224, 224, buf)
        check_frames(buf, env_id, st, cam, targets=targets, label="env camera")
    for cam in R.sweep_cameras(env_id, 6, seed=len(env_id)):
        buf = np.zeros((n, 48, 64, 3), np.uint8)
        sim.render(camera(**cam), 64, 48, buf)
        check_frames(buf, env_id, st, cam, targets=targets, label="sweep")
    sim.close()


@pytest.mark.parametrize("env_id", ["KukaButtonGymEnv-v0", "Kuka2ButtonGymEnv-v0", "MobileRobotGymEnv-v0", "MobileRobot2TargetGymEnv-v0",
                                    "MobileRobotLineTargetGymEnv-v0"])
def test_per_env_camera_checker_matches_the_reference(checker_backend, env_id):
    """The per-env path's checker (tests/host/render_cameras_ref.cpp): one sweep camera per env, odd sizes; MobileRobot with follow_robot
    (target float32(float64 position + offset))."""
    be = checker_backend
    n = 4
    sim, targets = make_sim(be, env_id, n, 6, seed=2)
    st = R.read_state(sim, env_id)
    cams = R.sweep_cameras(env_id, n, seed=11)
    for (w, h) in ((33, 17), (7, 5)):
        buf = np.zeros((n, h, w, 3), np.uint8)
        sim.render_cameras(camera_array(cams), False, w, h, buf)
        check_frames(buf, env_id, st, cams, targets=targets, label="per-env")
    if not env_id.startswith("Kuka"):
        offs = [dict(MOBILE_FPV_FOLLOW, roll=float(r)) for r in np.linspace(-40, 40, n)]
        buf = np.zeros((n, 40, 96, 3), np.uint8)
        sim.render_cameras(camera_array(offs), True, 96, 40, buf)
        pos = st["robot"]
        absolute = [dict(c, target=(float(np.float32(p[0] + np.float64(np.float32(c["target"][0])))),
                                    float(np.float32(p[1] + np.float64(np.float32(c["target"][1])))), c["target"][2]))
                    for p, c in zip(pos, offs)]
        check_frames(buf, env_id, st, absolute, targets=targets, label="follow_robot")
    sim.close()


def random_bodies(n, seed):
    """Caller-given distractor poses (SRL_F_DISTRACTORS layout): every type, tilted and rotated, resting on or floating above the table."""
    rs = np.random.RandomState(seed)
    B = np.zeros((n, 11, 9))
    for i in range(n):
        for k in range(11):
            q = rs.normal(size=4); q /= np.linalg.norm(q)
            B[i, k, 0:3] = (rs.uniform(0.35, 0.75), rs.uniform(-0.3, 0.3), rs.uniform(-0.17, -0.05))
            B[i, k, 3:7] = q
            B[i, k, 7] = 3 if k == 10 else rs.randint(0, 4)
            B[i, k, 8] = 1.0 if (k == 10 or rs.uniform() < 0.8) else 0.0
    return B


def test_checker_frames_with_bodies_match_the_reference(oracle_backend):
    """KukaRandButton with caller-given bodies (the oracle has no body dynamics: tests/host/distractor_frames_ref.cpp draws them), both env
    cameras and close sweep cameras, mid-episode and after an auto-reset."""
    import distractor_frames_ref as dfr
    env_id = "KukaRandButtonGymEnv-v0"
    n = 2
    sim, _ = make_sim(oracle_backend, env_id, n, 12, seed=4, max_steps=8)
    st = R.read_state(sim, env_id)
    B = random_bodies(n, 9)
    near = [dict(target=(0.55, 0.0, -0.15), distance=0.7, yaw=y, pitch=-35.0, roll=r, fov=70.0) for y, r in ((30.0, 0.0), (200.0, 25.0))]
    for cam, (w, h) in ((KUKA_CAMERA, (224, 224)), (KUKA_CAMERA_2, (224, 224)), (near[0], (160, 120)), (near[1], (160, 120))):
        frames = dfr.render(sim, distractor_blob(), B, cam, w, h)
        check_frames(frames, env_id, st, cam, bodies=B, label="bodies")
    sim.close()
