"""
Image observations (``srl_model="raw_pixels"``): cameras of the reference envs and the host side of ``srl_sim_render``.

The reference renders every env through ``p.computeViewMatrixFromYawPitchRoll`` / ``p.computeProjectionMatrixFOV`` / ``p.getCameraImage``
(environments/kuka_gym/kuka_button_gym_env.py:370-420, environments/mobile_robot/mobile_robot_env.py:287-334); the camera parameters below
are the ones those files set.  Frames are ``uint8 [N, 224, 224, 3]`` (``RENDER_HEIGHT`` x ``RENDER_WIDTH``), or 6 channels with
``multi_view`` (Kuka, second camera, :404-418) / ``fpv`` (MobileRobot, first-person camera, :316-332).  What is drawn is the analytic-primitive
scene of ``csrc/render_core.h`` -- not TinyRenderer's pixels.
"""
import ctypes

import numpy as np

RENDER_HEIGHT = 224
RENDER_WIDTH = 224


class SrlCamera(ctypes.Structure):
    """struct srl_camera (include/srl_sim.h)."""
    _fields_ = [("target", ctypes.c_float * 3), ("distance", ctypes.c_float), ("yaw", ctypes.c_float), ("pitch", ctypes.c_float),
                ("roll", ctypes.c_float), ("fov", ctypes.c_float)]


def camera(target, distance, yaw, pitch, roll=0.0, fov=60.0):
    c = SrlCamera()
    c.target[0], c.target[1], c.target[2] = [float(x) for x in target]
    c.distance, c.yaw, c.pitch, c.roll, c.fov = float(distance), float(yaw), float(pitch), float(roll), float(fov)
    return c


# kuka_button_gym_env.py:94-102 (main camera), :404-411 (second camera of multi_view)
KUKA_CAMERA = dict(target=(0.316, -0.2, -0.1), distance=1.1, yaw=145, pitch=-36, roll=0, fov=60)
KUKA_CAMERA_2 = dict(target=(0.316, 0.316, -0.105), distance=1.05, yaw=32, pitch=-13, roll=0, fov=60)
# mobile_robot_env.py:88-93 (camera_target_pos (2, 2, 0), distance 4.4, yaw 90, pitch -90)
MOBILE_CAMERA = dict(target=(2.0, 2.0, 0.0), distance=4.4, yaw=90, pitch=-90, roll=0, fov=60)


def mobile_fpv_camera(robot_xy, yaw=90):
    """First-person camera of the MobileRobot envs (mobile_robot_env.py:316-326): fov 90, looking from behind the car."""
    return dict(target=(float(robot_xy[0]) - 0.25, float(robot_xy[1]), 0.15), distance=0.3, yaw=yaw, pitch=-17, roll=0, fov=90)


# the first-person camera as offsets from the robot's position, for srl_sim_render_cameras(follow_robot=1): target (x - 0.25, y, 0.15)
MOBILE_FPV_FOLLOW = mobile_fpv_camera((0.0, 0.0))


def camera_array(cams):
    """A ctypes array of ``SrlCamera``, one per env, from a list of camera dicts (build it once and reuse it: the library skips its
    camera set-up when a call passes the same cameras as the previous one)."""
    arr = (SrlCamera * len(cams))()
    for i, c in enumerate(cams):
        arr[i] = camera(**c)
    return arr


def render_cameras(sim, backend, cams, follow_robot=False, width=RENDER_WIDTH, height=RENDER_HEIGHT, out=None):
    """One frame per env through its own camera: env ``i`` through ``cams[i]`` (a list of camera dicts or a ``camera_array``); with
    ``follow_robot`` (MobileRobot) each target's x and y are offsets from that env's robot position, read on the device.
    ``uint8 [N, H, W, 3]`` in the backend's memory."""
    if not isinstance(cams, ctypes.Array):
        cams = camera_array(cams)
    buf = backend.zeros((sim.num_envs, height, width, 3), np.uint8) if out is None else out
    sim.render_cameras(cams, follow_robot, width, height, buf, stream=backend.stream())
    return buf


def render_batch(sim, backend, cams, width=RENDER_WIDTH, height=RENDER_HEIGHT, out=None):
    """One frame per env and camera: ``uint8 [N, H, W, 3 * len(cams)]`` in the backend's memory (a CUDA tensor for the product library)."""
    n = sim.num_envs
    frames = []
    for c in cams:
        buf = backend.zeros((n, height, width, 3), np.uint8)
        sim.render(camera(**c), width, height, buf, stream=backend.stream())
        frames.append(buf)
    if len(frames) == 1:
        return frames[0]
    if backend.on_gpu:
        return backend.torch.cat(frames, dim=3)
    return np.concatenate(frames, axis=3)
