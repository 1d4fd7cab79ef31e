"""
KukaRandButton frames with the distractor bodies drawn, on the CPU checker (tests/distractor_frames_ref.py: the oracle's scene list plus the
bodies through csrc/render_core.h's srl_distractor_prims, the per-pixel arithmetic of the CUDA kernels).

  * frames of every env id without bodies are the bytes the checker drew before the ray caster learnt the oriented box
    (tests/golden/render_hashes_golden.json, written by tests/golden/gen_render_hashes.py from the checker of the parent revision);
  * absent bodies draw nothing;
  * an oriented box's silhouette lands where an independent numpy restatement of pybullet's view / projection matrices puts its 8 corners,
    q and -q draw the same bytes, and a box turned by 90 degrees about z with its x / y half extents swapped has the same silhouette;
  * a sphere is centred on its projected centre, in the blob's colour;
  * a body behind the button is hidden where the disc covers it.
"""
import json
import os
import sys

import numpy as np
import pytest
from scipy.spatial import Delaunay

import distractor_frames_ref as dfr
from srl_sim import _abi
from srl_sim.model import distractor_blob, load_kuka_scene
from srl_sim.render import KUKA_CAMERA, KUKA_CAMERA_2

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RB = "KukaRandButtonGymEnv-v0"
W = H = 224


def _pybullet_matrices(target, distance, yaw, pitch, roll, fov, aspect, near=0.1, far=100.0):
    """numpy restatement of computeViewMatrixFromYawPitchRoll (upAxisIndex = 2) and computeProjectionMatrixFOV as matrices: eye = target +
    Rz(yaw) Ry(roll) Rx(pitch) (0, -d, 0), up = the same rotation of (0, 0, 1), OpenGL lookAt and perspective."""
    y, p, r = np.radians([yaw, pitch, roll])
    Rz = np.array([[np.cos(y), -np.sin(y), 0], [np.sin(y), np.cos(y), 0], [0, 0, 1]])
    Ry = np.array([[np.cos(r), 0, np.sin(r)], [0, 1, 0], [-np.sin(r), 0, np.cos(r)]])
    Rx = np.array([[1, 0, 0], [0, np.cos(p), -np.sin(p)], [0, np.sin(p), np.cos(p)]])
    R = Rz @ Ry @ Rx
    eye = np.asarray(target, float) + R @ np.array([0.0, -distance, 0.0])
    up = R @ np.array([0.0, 0.0, 1.0])
    f = np.asarray(target, float) - eye
    f /= np.linalg.norm(f)
    s = np.cross(f, up)
    s /= np.linalg.norm(s)
    u = np.cross(s, f)
    view = np.eye(4)
    view[0, :3], view[1, :3], view[2, :3] = s, u, -f
    view[:3, 3] = -view[:3, :3] @ eye
    t = 1.0 / np.tan(np.radians(fov) / 2)
    proj = np.array([[t / aspect, 0, 0, 0], [0, t, 0, 0], [0, 0, (far + near) / (near - far), 2 * far * near / (near - far)], [0, 0, -1, 0]])
    return view, proj, eye


def _project(points, cam, w=W, h=H):
    """pixel coordinates (x right, y down, continuous: pixel k covers [k, k + 1)) of world points [M, 3]."""
    view, proj, _ = _pybullet_matrices(aspect=w / h, **cam)
    P = np.c_[np.asarray(points, float), np.ones(len(points))]
    c = (proj @ view @ P.T).T
    ndc = c[:, :3] / c[:, 3:4]
    return np.c_[(ndc[:, 0] + 1) / 2 * w, (1 - ndc[:, 1]) / 2 * h]


def _rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _corners(p, half, q):
    s = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], float)
    return np.asarray(p, float) + (s * np.asarray(half, float)) @ _rot(q).T


def _quat(axis, deg):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    h = np.radians(deg) / 2
    return np.r_[a * np.sin(h), np.cos(h)]


def _one_body(p, q, btype, n=1):
    """f64[n, 11, 9]: body slot 0 present at pose (p, q) with type `btype`, every other slot absent."""
    b = np.zeros((n, 11, 9))
    b[:, :, 6] = 1.0
    b[:, 0, 0:3] = p
    b[:, 0, 3:7] = q
    b[:, 0, 7] = btype
    b[:, 0, 8] = 1.0
    return b


@pytest.fixture()
def rb(oracle_backend):
    sim = oracle_backend.make_sim(RB, 1, seed=4, model_blob=load_kuka_scene().blob)
    sim.reset()
    yield sim
    sim.close()


def _plain(sim, cam=KUKA_CAMERA, w=W, h=H):
    out = np.zeros((sim.num_envs, h, w, 3), np.uint8)
    from srl_sim.render import camera
    sim.render(camera(**cam), w, h, out)
    return out


def _silhouette(with_body, without):
    return (with_body != without).any(axis=-1)


def test_frames_without_bodies_keep_the_parent_bytes(oracle_backend):
    sys.path.insert(0, GOLDEN)
    try:
        import gen_render_hashes as gen
    finally:
        sys.path.remove(GOLDEN)
    with open(os.path.join(GOLDEN, "render_hashes_golden.json")) as f:
        golden = json.load(f)
    assert sorted(golden) == sorted(_abi.ENV_KINDS)
    for env_id, cfg, acts, cams in gen.cases():
        assert gen.frame_hashes(oracle_backend, env_id, cfg, acts, cams) == golden[env_id], env_id


def test_absent_bodies_draw_nothing(oracle_backend):
    n = 3
    sim = oracle_backend.make_sim(RB, n, seed=9, model_blob=load_kuka_scene().blob, random_target=True)
    sim.reset()
    acts = np.random.RandomState(2).randint(0, 6, size=(6, n)).astype(np.int32)
    sim.rollout(6, acts, None, np.zeros((6, n, 3), np.float32), np.zeros((6, n), np.float32), np.zeros((6, n), np.uint8))
    rng = np.random.RandomState(0)
    bodies = np.zeros((n, 11, 9))
    bodies[:, :, 0:3] = rng.uniform([0.3, -0.3, -0.2], [0.7, 0.3, 0.0], size=(n, 11, 3))
    q = rng.normal(size=(n, 11, 4))
    bodies[:, :, 3:7] = q / np.linalg.norm(q, axis=-1, keepdims=True)
    bodies[:, :, 7] = rng.randint(4, size=(n, 11))
    for cam in (KUKA_CAMERA, KUKA_CAMERA_2):
        for (w, h) in ((W, H), (50, 33)):
            assert np.array_equal(dfr.render(sim, distractor_blob(), bodies, cam, w, h), _plain(sim, cam, w, h))
    sim.close()


def test_checker_refuses_other_handles_and_bad_bodies(oracle_backend):
    sim = oracle_backend.make_sim("KukaButtonGymEnv-v0", 1, seed=0, model_blob=load_kuka_scene().blob)
    sim.reset()
    with pytest.raises(dfr.RenderError, match="only KukaRandButton"):
        dfr.render(sim, distractor_blob(), _one_body((0.5, 0, 0), (0, 0, 0, 1), 2), KUKA_CAMERA, 8, 8)
    sim.close()
    sim = oracle_backend.make_sim(RB, 1, seed=0, model_blob=load_kuka_scene().blob)
    sim.reset()
    with pytest.raises(dfr.RenderError, match="type must be"):
        dfr.render(sim, distractor_blob(), _one_body((0.5, 0, 0), (0, 0, 0, 1), 4), KUKA_CAMERA, 8, 8)
    bad = distractor_blob().reshape(4, 32).copy()
    bad[2, 28] = 3.0
    with pytest.raises(dfr.RenderError, match="DC_A_SHAPE"):
        dfr.render(sim, bad.reshape(-1), _one_body((0.5, 0, 0), (0, 0, 0, 1), 2), KUKA_CAMERA, 8, 8)
    sim.close()


# a place in front of the arm, clear of the table top and the button, that both the cube and the brick can turn in
BOX_AT = (0.42, -0.32, -0.08)
POSES = {"identity": (0.0, 0.0, 0.0, 1.0), "45 deg about z": tuple(_quat((0, 0, 1), 45)), "30 deg about x": tuple(_quat((1, 0, 0), 30)),
         "random": tuple(np.random.RandomState(7).normal(size=4) / np.linalg.norm(np.random.RandomState(7).normal(size=4)))}


@pytest.mark.parametrize("btype", [2, 1], ids=["cube", "lego"])
@pytest.mark.parametrize("pose", sorted(POSES))
def test_oriented_box_against_projected_corners(rb, btype, pose):
    blob = distractor_blob()
    half = blob.reshape(4, 32)[btype, 22:25]
    q = np.array(POSES[pose])
    plain = _plain(rb)
    img = dfr.render(rb, blob, _one_body(BOX_AT, q, btype), KUKA_CAMERA, W, H)
    ys, xs = np.nonzero(_silhouette(img, plain)[0])
    assert len(xs) > 10, pose
    uv = _project(_corners(BOX_AT, half, q), KUKA_CAMERA)
    # a pixel is covered when its centre (k + 0.5) is: the first / last covered pixel of a projected extent [a, b]
    lo, hi = np.ceil(uv.min(axis=0) - 0.5), np.floor(uv.max(axis=0) - 0.5)
    got = np.array([[xs.min(), ys.min()], [xs.max(), ys.max()]], float)
    assert np.abs(got - np.array([lo, hi])).max() <= 1.0, (pose, got, lo, hi)
    # q and -q: the same rotation, the same bytes
    assert np.array_equal(dfr.render(rb, blob, _one_body(BOX_AT, -q, btype), KUKA_CAMERA, W, H), img)


def test_quarter_turn_with_swapped_half_extents_has_the_same_silhouette(rb):
    blob = distractor_blob().reshape(4, 32).copy()           # the duck: an elongated box, 0.09 x 0.06 x 0.08
    swapped = blob.copy()
    swapped[0, 22], swapped[0, 23] = blob[0, 23], blob[0, 22]
    plain = _plain(rb)
    a = _silhouette(dfr.render(rb, blob.reshape(-1), _one_body(BOX_AT, (0, 0, 0, 1), 0), KUKA_CAMERA, W, H), plain)
    b = _silhouette(dfr.render(rb, swapped.reshape(-1), _one_body(BOX_AT, _quat((0, 0, 1), 90), 0), KUKA_CAMERA, W, H), plain)
    assert a.sum() > 100
    # the same box up to rounding in the rotation: at most a few pixels along its outline may fall the other way
    assert (a ^ b).sum() <= max(3, 0.02 * a.sum()), ((a ^ b).sum(), a.sum())


def test_sphere_centred_on_its_projection_in_the_blob_colour(rb):
    blob = distractor_blob()
    r, rgb = blob.reshape(4, 32)[3, 22], blob.reshape(4, 32)[3, 25:28]
    plain = _plain(rb)
    img = dfr.render(rb, blob, _one_body(BOX_AT, (0, 0, 0, 1), 3), KUKA_CAMERA, W, H)
    ys, xs = np.nonzero(_silhouette(img, plain)[0])
    cx, cy = _project([BOX_AT], KUKA_CAMERA)[0]
    assert abs(xs.mean() + 0.5 - cx) < 1.0 and abs(ys.mean() + 0.5 - cy) < 1.0, (xs.mean(), ys.mean(), cx, cy)
    # every pixel of the ball is the blob's colour times one shade factor (ambient + Lambert)
    px = img[0, ys, xs].astype(float)
    shade = px[:, 2] / (255.0 * rgb[2])
    assert shade.min() >= 0.54 and shade.max() <= 1.0
    assert np.abs(px - np.outer(shade, rgb) * 255.0).max() <= 1.5


def test_body_behind_the_button_is_hidden_by_the_disc(rb):
    blob = distractor_blob().reshape(4, 32).copy()
    blob[2, 22:25] = 0.06                                     # a cube larger than the disc, so that it shows around it
    disc_top = rb.get_state(_abi.F_TARGET_POS)[0] - np.array([0, 0, 0.25])
    _, _, eye = _pybullet_matrices(aspect=1.0, **KUKA_CAMERA)
    away = np.r_[(disc_top - eye)[:2], 0.0]
    behind = disc_top + 0.2 * away / np.linalg.norm(away)     # 20 cm beyond the button's centre, seen from the camera: wholly behind it
    plain = _plain(rb)
    img = dfr.render(rb, blob.reshape(-1), _one_body(behind, (0, 0, 0, 1), 2), KUKA_CAMERA, W, H)
    rgb = plain[0].astype(int)
    disc = (rgb[..., 0] > 170) & (rgb[..., 1] > 170) & (rgb[..., 2] < 90)
    # the pixels whose centre lies inside the projected cube (the convex hull of its 8 projected corners)
    hull = Delaunay(_project(_corners(behind, (0.06, 0.06, 0.06), (0, 0, 0, 1)), KUKA_CAMERA))
    yy, xx = np.mgrid[0:H, 0:W] + 0.5
    inside = (hull.find_simplex(np.c_[xx.ravel(), yy.ravel()]) >= 0).reshape(H, W)
    assert (disc & inside).sum() > 20                        # the disc covers part of the cube
    assert np.array_equal(img[0][disc], plain[0][disc])      # ... and there the disc is what is drawn
    assert (_silhouette(img, plain)[0] & inside & ~disc).sum() > 200   # the cube shows around it
