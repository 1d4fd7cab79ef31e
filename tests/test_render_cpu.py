"""
Image observations (SURVEY 8(f).4, `srl_model="raw_pixels"`) on the CPU checker (oracle/liboracle_sim.so; same primitive lists and per-pixel
arithmetic as the CUDA kernels, csrc/render_core.h).

What can be pinned offline: the reference checkout holds exactly two rendered outputs of these envs -- the first frames of its README
animations (imgs/kuka.gif, imgs/mobile_robot.gif; TinyRenderer, 168 x 168), extracted into tests/golden/ref_frame_*.png by
tests/golden/gen_ref_frames.py.  The meshes and textures they were drawn from are not available, so pixels cannot match; the CAMERA
(computeViewMatrixFromYawPitchRoll / computeProjectionMatrixFOV with the parameters of kuka_button_gym_env.py:94-102,385-398 and
mobile_robot_env.py:76-84,297-309) and the LAYOUT (button on the table, the four coloured walls, the target disc) can: the static features of
those frames must land on the same image coordinates here.  A second, independent check projects known world points through a numpy
restatement of pybullet's view / projection matrices.
"""
import os

import cv2
import numpy as np
import pytest

from environments.registry import registered_env
from render_numpy_ref import pybullet_matrices as _pybullet_matrices

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _masks(im):
    r, g, b = [im[..., k].astype(int) for k in range(3)]
    return dict(red=(r > 100) & (g < 60) & (b < 60), green=(g > 110) & (r < 70) & (b < 70), blue=(b > 110) & (r < 60) & (g < 60),
                black=(r < 40) & (g < 40) & (b < 40), yellow=(r > 170) & (g > 170) & (b < 90))


def _blob(mask):
    """(x centre, y centre, width, height) of a mask in image-relative coordinates."""
    ys, xs = np.nonzero(mask)
    H, W = mask.shape
    return np.array([xs.mean() / W, ys.mean() / H, (xs.max() - xs.min() + 1) / W, (ys.max() - ys.min() + 1) / H])


def _line(mask, axis):
    """Image-relative position of a straight wall: the rows (axis 0) / columns (axis 1) it covers for more than 40 % of the other dimension."""
    frac = mask.mean(axis=1 - axis)
    idx = np.nonzero(frac > 0.4)[0]
    return (idx.mean() + 0.5) / mask.shape[axis]


def _ref(name):
    return cv2.cvtColor(cv2.imread(os.path.join(GOLDEN, name)), cv2.COLOR_BGR2RGB)


def test_kuka_frame_layout_matches_the_reference_frame(use_oracle_backend):
    """imgs/kuka.gif, frame 0: the button (yellow disc on its green base, default position (0.5, 0) on the table) seen by the env's fixed
    camera.  Disc and base must appear at the same place and size (1.2 % of the image; the disc's height depends on how far it is pressed)."""
    env = registered_env["KukaButtonGymEnv-v0"][0](srl_model="raw_pixels")
    env.seed(0)
    frame = env.reset()
    assert frame.shape == (224, 224, 3) and frame.dtype == np.uint8 and env.observation_space.shape == (224, 224, 3)
    ours, ref = _masks(frame), _masks(_ref("ref_frame_kuka.png"))
    a, b = _blob(ours["yellow"]), _blob(ref["yellow"])
    assert np.abs(a - b).max() < 0.012, ("yellow", a, b)
    # the green base: x centre, width and lower edge (the 1 cm ring that sticks out left and right of the disc is 1-2 pixels wide: it is
    # blended away in the 168-pixel reference frame, so the blob's upper edge is not comparable)
    (ya, xa), (yb, xb) = np.nonzero(ours["green"]), np.nonzero(ref["green"])
    ga = np.array([xa.mean() / 224, (xa.max() - xa.min() + 1) / 224, (ya.max() + 1) / 224])
    gb = np.array([xb.mean() / 168, (xb.max() - xb.min() + 1) / 168, (yb.max() + 1) / 168])
    assert np.abs(ga - gb).max() < 0.012, ("green", ga, gb)
    # same scene through render(): the observation IS the rendered frame
    assert np.array_equal(frame, env.render("rgb_array"))
    # table in the lower half, checkered plane above it: light wood vs white / light blue
    wood, plane = frame[200, 30].astype(int), frame[10, 10].astype(int)
    assert wood[0] - wood[2] > 30 and plane[2] >= plane[0]            # warm (red > blue) table, white / light-blue plane
    env.close()


def test_mobile_frame_layout_matches_the_reference_frame(use_oracle_backend):
    """imgs/mobile_robot.gif, frame 0: top-down camera (target (2, 2, 0), distance 4.4, yaw 90, pitch -90): the red / green walls are the left /
    right edges, blue / black the top / bottom ones, at the same image coordinates; the target disc has the same size."""
    env = registered_env["MobileRobotGymEnv-v0"][0](srl_model="raw_pixels", random_target=True)
    env.seed(3)
    frame = env.reset()
    ours, ref = _masks(frame), _masks(_ref("ref_frame_mobile.png"))
    for colour, axis in (("red", 1), ("green", 1), ("blue", 0), ("black", 0)):
        a, b = _line(ours[colour], axis), _line(ref[colour], axis)
        assert abs(a - b) < 0.008, (colour, a, b)
    assert _line(ours["red"], 1) < 0.2 < 0.8 < _line(ours["green"], 1) and _line(ours["blue"], 0) < 0.2 < 0.8 < _line(ours["black"], 0)
    assert np.abs(_blob(ours["yellow"])[2:] - _blob(ref["yellow"])[2:]).max() < 0.012      # the disc of urdf/cylinder.urdf: same diameter
    env.close()


def _project(point, view, proj, W, H):
    c = proj @ view @ np.append(np.asarray(point, float), 1.0)
    ndc = c[:3] / c[3]
    return (ndc[0] + 1) / 2 * W, (1 - ndc[1]) / 2 * H          # pixel coordinates, row 0 at the top


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_camera_against_an_independent_view_projection_restatement(use_oracle_backend, seed):
    """Random targets: the centroid of the target disc / the button disc in the frame must be where pybullet-style view and projection MATRICES
    put the disc's top centre (within a pixel and a half; an obliquely seen disc's centroid is not exactly its centre's projection)."""
    from srl_sim.render import KUKA_CAMERA, MOBILE_CAMERA
    env = registered_env["MobileRobotGymEnv-v0"][0](srl_model="raw_pixels", random_target=True)
    env.seed(seed)
    frame = env.reset()
    view, proj = _pybullet_matrices(aspect=1.0, **MOBILE_CAMERA)
    ys, xs = np.nonzero(_masks(frame)["yellow"])
    px, py = _project([env.target_pos[0], env.target_pos[1], 0.03], view, proj, 224, 224)
    assert abs(xs.mean() + 0.5 - px) < 1.5 and abs(ys.mean() + 0.5 - py) < 1.5, (xs.mean(), ys.mean(), px, py)
    env.close()
    env = registered_env["KukaRandButtonGymEnv-v0"][0](srl_model="raw_pixels", random_target=True)
    env.seed(seed)
    frame = env.reset()
    view, proj = _pybullet_matrices(aspect=1.0, **KUKA_CAMERA)
    ys, xs = np.nonzero(_masks(frame)["yellow"])
    top = env.getTargetPos() - np.array([0, 0, 0.28]) + np.array([0, 0, 0.03])     # target = button link origin + 0.28; the disc is 3 cm thick
    px, py = _project(top, view, proj, 224, 224)
    if len(xs) > 200:       # the arm may hide the disc after the random initial moves
        assert abs(xs.mean() + 0.5 - px) < 3.0 and abs(ys.mean() + 0.5 - py) < 3.0, (xs.mean(), ys.mean(), px, py)
    env.close()


def test_second_cameras_batched_frames_and_recorded_images(use_oracle_backend, tmp_path):
    """multi_view (Kuka, kuka_button_gym_env.py:404-418) and fpv (MobileRobot, mobile_robot_env.py:316-332) stack a second camera on the
    channels; the batched VecEnv returns one frame per env; a recording run (record_data=True) writes the frames EpisodeSaver names."""
    from srl_sim.vec_env import BatchedSRLVecEnv
    env = registered_env["KukaButtonGymEnv-v0"][0](srl_model="raw_pixels", multi_view=True)
    env.seed(1)
    f = env.reset()
    assert f.shape == (224, 224, 6) and env.observation_space.shape == (224, 224, 6) and not np.array_equal(f[..., :3], f[..., 3:])
    env.close()
    env = registered_env["MobileRobotGymEnv-v0"][0](srl_model="raw_pixels", fpv=True)
    env.seed(1)
    f = env.reset()
    assert f.shape == (224, 224, 6)
    env.close()
    venv = BatchedSRLVecEnv("MobileRobotGymEnv-v0", 3, seed=2, srl_model="raw_pixels", random_target=True)
    o = venv.reset()
    assert o.shape == (3, 224, 224, 3) and o.dtype == np.uint8 and venv.observation_space.shape == (224, 224, 3)
    o2, r, d, _ = venv.step([0, 1, 2])
    assert o2.shape == o.shape and not np.array_equal(o2, o) and not np.array_equal(o2[0], o2[1])
    assert len(venv.get_images()) == 3
    venv.close()
    env = registered_env["MobileRobotGymEnv-v0"][0](srl_model="raw_pixels", record_data=True, save_path=str(tmp_path) + "/", name="rec")
    env.seed(0)
    env.reset()
    env.step(1)
    env.saver.save()
    assert os.path.isfile(str(tmp_path / "rec" / "record_000" / "frame000000.jpg")) and os.path.isfile(str(tmp_path / "rec" / "record_000" / "frame000001.jpg"))
    env.close()
