"""
KukaRandButton frames with the distractor bodies drawn, on the H100: the CUDA list kernel + ray caster against the CPU checker
(tests/distractor_frames_ref.py) fed the CUDA handle's own bodies, culling with bodies, changes confined to the bodies' screen rectangles,
the public surfaces (BatchedSRLVecEnv raw pixels, the single-env class) and the refusal of bad drawing words.
"""
import time

import numpy as np
import pytest

import distractor_frames_ref as dfr
from srl_sim import _abi
from srl_sim.model import distractor_blob, load_kuka_scene
from srl_sim.render import KUKA_CAMERA, KUKA_CAMERA_2, camera

pytestmark = pytest.mark.gpu

RB = "KukaRandButtonGymEnv-v0"


def _sim(be, n, bodies, **cfg):
    s = be.make_sim(RB, n, model_blob=load_kuka_scene().blob, **cfg)
    if bodies:
        s.set_distractors(distractor_blob())
    s.reset(stream=be.stream())
    return s


def _rollout(be, s, acts):
    T, n = acts.shape
    obs = be.zeros((T, n, 3), np.float32); rew = be.zeros((T, n), np.float32); done = be.zeros((T, n), np.uint8)
    s.rollout(T, be.from_host(acts), None, obs, rew, done, stream=be.stream())
    return be.to_host(done).copy()


def _render(be, s, cam, w, h):
    buf = be.zeros((s.num_envs, h, w, 3), np.uint8)
    s.render(camera(**cam), w, h, buf, stream=be.stream())
    return be.to_host(buf).copy()


def _bodies(s):
    return s.get_state(_abi.F_DISTRACTORS).reshape(s.num_envs, 11, 9)


def test_cuda_frames_with_bodies_match_the_cpu_checker(cuda_backend, oracle_backend):
    """Settled (t = 0), after the kick (t = 12) and at t = 60 with max_steps = 25 (every env has auto-reset at least once): the CUDA frames
    against the checker given the CUDA handle's bodies, and the drawn arm / button state of the CUDA handle, so that only the drawing is
    compared."""
    n = 16
    cfg = dict(seed=3, random_target=True, max_steps=25)
    acts = np.random.RandomState(1).randint(0, 6, size=(60, n)).astype(np.int32)
    cu = _sim(cuda_backend, n, True, **cfg)
    plain = _sim(cuda_backend, n, False, **cfg)
    ora = oracle_backend.make_sim(RB, n, model_blob=load_kuka_scene().blob, **cfg)
    ora.reset()
    t, resets = 0, 0
    for t_next in (0, 12, 60):
        if t_next > t:
            done = _rollout(cuda_backend, cu, acts[t:t_next])
            _rollout(cuda_backend, plain, acts[t:t_next])
            resets += int(done.any(axis=0).sum())
            t = t_next
        for f in (_abi.F_JOINT_POS, _abi.F_BUTTON_GLIDER, _abi.F_BUTTON_BASE, _abi.F_TARGET_POS):
            ora.set_state(f, cu.get_state(f))
        B = _bodies(cu)
        assert B[:, 10, 8].all()
        visible = []
        for cam, (w, h) in ((KUKA_CAMERA, (224, 224)), (KUKA_CAMERA_2, (224, 224)), (KUKA_CAMERA, (50, 33))):
            a = _render(cuda_backend, cu, cam, w, h)
            b = dfr.render(ora, distractor_blob(), B, cam, w, h)
            same = (a == b).mean()
            assert same > 0.995, (t, cam, w, h, same)
            assert np.abs(a.astype(int) - b.astype(int)).mean() < 0.5
            visible.append(np.mean([not np.array_equal(a[k], p) for k, p in enumerate(_render(cuda_backend, plain, cam, w, h))]))
        print("t = %d: share of envs whose frame shows bodies, per camera / size: %s" % (t, visible))
        assert visible[0] > 0.5
    assert resets >= n, "expected every env to have auto-reset by t = 60"
    for s in (cu, plain, ora):
        s.close()


def test_tile_culling_with_bodies_never_changes_a_byte(cuda_backend, monkeypatch):
    be = cuda_backend
    n = 64
    s = _sim(be, n, True, seed=11, random_target=True)
    _rollout(be, s, np.random.RandomState(5).randint(0, 6, size=(40, n)).astype(np.int32))
    for c in (KUKA_CAMERA, KUKA_CAMERA_2, dict(KUKA_CAMERA, distance=0.6, pitch=-10.0, yaw=200.0)):
        for (w, h) in ((224, 224), (64, 64), (50, 33), (96, 40)):
            out = []
            for no_cull in (False, True):
                if no_cull:
                    monkeypatch.setenv("SRL_RENDER_NO_CULL", "1")
                else:
                    monkeypatch.delenv("SRL_RENDER_NO_CULL", raising=False)
                out.append(_render(be, s, c, w, h))
            assert np.array_equal(out[0], out[1]), (c, w, h, int((out[0] != out[1]).sum()))
    monkeypatch.delenv("SRL_RENDER_NO_CULL", raising=False)
    s.close()


def _body_rects(B, cam, w, h):
    """per env the union of the bodies' screen rectangles (numpy: each present body's bounding sphere -- a box's half diagonal, a sphere's
    radius -- projected through a pinhole camera restated from the camera parameters), as a boolean [N, h, w] mask."""
    look = distractor_blob().reshape(4, 32)
    y, p = np.radians(cam["yaw"]), np.radians(cam["pitch"])
    Rz = np.array([[np.cos(y), -np.sin(y), 0], [np.sin(y), np.cos(y), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, np.cos(p), -np.sin(p)], [0, np.sin(p), np.cos(p)]])
    R = Rz @ Rx
    eye = np.asarray(cam["target"], float) + R @ np.array([0.0, -cam["distance"], 0.0])
    fwd = np.asarray(cam["target"], float) - eye; fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, R @ np.array([0.0, 0.0, 1.0])); right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    th = np.tan(np.radians(cam["fov"]) / 2)
    fx, fy = w / (2 * th * w / h), h / (2 * th)
    mask = np.zeros((B.shape[0], h, w), bool)
    for i in range(B.shape[0]):
        for k in range(11):
            if not B[i, k, 8]:
                continue
            t = int(B[i, k, 7])
            half = look[t, 22:25]
            rad = (half[0] if look[t, 28] == 1 else np.linalg.norm(half)) + 1e-3
            q = B[i, k, 0:3] - eye
            z = q @ fwd
            if z <= rad:
                mask[i] = True
                continue
            # a sphere of radius rad at depth z spans at most rad / (z - rad) in either screen direction around its centre's projection
            u, v, e = (q @ right) / z, (q @ up) / z, rad / (z - rad) * 1.5
            x0, x1 = int(np.floor(w / 2 + (u - e) * fx)) - 1, int(np.ceil(w / 2 + (u + e) * fx)) + 1
            y0, y1 = int(np.floor(h / 2 - (v + e) * fy)) - 1, int(np.ceil(h / 2 - (v - e) * fy)) + 1
            mask[i, max(y0, 0):max(y1, 0), max(x0, 0):max(x1, 0)] = True
    return mask


def test_frames_change_only_inside_the_bodies_rectangles(cuda_backend):
    be = cuda_backend
    n = 32
    acts = np.random.RandomState(8).randint(0, 6, size=(24, n)).astype(np.int32)
    a = _sim(be, n, True, seed=21, random_target=True)
    b = _sim(be, n, False, seed=21, random_target=True)
    _rollout(be, a, acts)
    _rollout(be, b, acts)
    B = _bodies(a)
    for cam in (KUKA_CAMERA, KUKA_CAMERA_2):
        fa, fb = _render(be, a, cam, 224, 224), _render(be, b, cam, 224, 224)
        diff = (fa != fb).any(axis=-1)
        inside = _body_rects(B, cam, 224, 224)
        assert diff.any()
        assert not (diff & ~inside).any(), int((diff & ~inside).sum())
    a.close(); b.close()


def test_vec_env_and_single_env_show_the_bodies(cuda_lib):
    from srl_sim import backend
    backend.use_library(None, None)
    from srl_sim.vec_env import BatchedSRLVecEnv
    frames = {}
    for bodies in (True, False):
        venv = BatchedSRLVecEnv(RB, 8, seed=1, srl_model="raw_pixels", multi_view=True, distractors=bodies)
        venv.reset()
        o, _, _, _ = venv.step([0] * 8)
        assert o.shape == (8, 224, 224, 6)
        if bodies:
            be = venv.backend
            ref = np.concatenate([_render(be, venv.sim, c, 224, 224) for c in (KUKA_CAMERA, KUKA_CAMERA_2)], axis=3)
            assert np.array_equal(o, ref)
        frames[bodies] = o
        venv.close()
    assert not np.array_equal(frames[True], frames[False])
    from environments.kuka_gym.kuka_rand_button_gym_env import KukaRandButtonGymEnv
    obs = {}
    for bodies in (True, False):
        env = KukaRandButtonGymEnv(srl_model="raw_pixels", random_target=True, distractors=bodies)
        env.seed(2)
        env.reset()
        for _ in range(12):
            o, _, _, _ = env.step(0)
        assert np.array_equal(o, env.render("rgb_array"))
        obs[bodies] = o
        env.close()
    assert not np.array_equal(obs[True], obs[False])


@pytest.mark.parametrize("word,value,message", [(28, 2.0, "DC_A_SHAPE"), (23, 0.0, "DC_A_HALF"), (27, 1.5, "DC_A_RGB"), (25, -0.1, "DC_A_RGB")])
def test_bad_drawing_words_are_refused(cuda_backend, word, value, message):
    blob = distractor_blob().reshape(4, 32).copy()
    blob[1, word] = value
    s = cuda_backend.make_sim(RB, 2, model_blob=load_kuka_scene().blob)
    with pytest.raises(_abi.SimError, match=message):
        s.set_distractors(blob.reshape(-1))
    s.close()


def test_full_batch_with_bodies(cuda_backend):
    import torch
    be = cuda_backend
    n = 4096
    s = _sim(be, n, True, seed=0)
    _rollout(be, s, np.zeros((16, n), np.int32))
    buf = be.zeros((n, 224, 224, 3), np.uint8)
    for _ in range(2):
        s.render(camera(**KUKA_CAMERA), 224, 224, buf, stream=be.stream())
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    reps = 5
    for _ in range(reps):
        s.render(camera(**KUKA_CAMERA), 224, 224, buf, stream=be.stream())
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / reps
    print("RENDER WITH BODIES: 4096 KukaRandButton frames of 224 x 224 in %.2f ms" % (1e3 * dt))
    assert tuple(buf.shape) == (n, 224, 224, 3)
    assert len(np.unique(be.to_host(buf[0]).reshape(-1, 3), axis=0)) >= 3
    s.close()
