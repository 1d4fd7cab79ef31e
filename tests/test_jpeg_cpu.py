"""
The JPEG encoder's CPU checker (csrc/libjpeg_ref.so: csrc/jpeg_core.h compiled for the host, include/srl_image.h on host pointers) against
OpenCV's encoder, and EpisodeSaver's encoded-frame case.  The target is byte equality with
`cv2.imencode('.jpg', rgb[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, q])`: frames the oracle renders for every env id, odd sizes that exercise
edge replication and dummy blocks, and uniform noise (the worst case for the size bound and for 0xFF stuffing).
"""
import os

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from environments.registry import registered_env  # noqa: E402
from srl_sim import jpeg  # noqa: E402

QUALITIES = (1, 50, 75, 95, 100)
ENV_IDS = ["KukaButtonGymEnv-v0", "KukaRandButtonGymEnv-v0", "Kuka2ButtonGymEnv-v0", "KukaMovingButtonGymEnv-v0",
           "MobileRobotGymEnv-v0", "MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0", "MobileRobotLineTargetGymEnv-v0"]


def cv2_jpeg(rgb, quality):
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(rgb[..., ::-1]), [cv2.IMWRITE_JPEG_QUALITY, int(quality)])
    assert ok
    return buf.tobytes()


@pytest.fixture(scope="module")
def ref():
    return jpeg.reference_library()


def _bound(ref, w, h):
    return int(ref.lib.srl_jpeg_bound(w, h))


def _oracle_frames(env_id, n_steps=3):
    env = registered_env[env_id][0](srl_model="raw_pixels", random_target=True)
    env.seed(7)
    env.action_space.seed(7)
    frames = [env.reset()]
    for _ in range(n_steps):
        frames.append(env.step(env.action_space.sample())[0])
    env.close()
    return np.stack(frames)


@pytest.fixture(scope="module")
def env_frames(oracle_lib):
    from srl_sim import backend
    backend.use_library(oracle_lib, -1)
    try:
        return {env_id: _oracle_frames(env_id) for env_id in ENV_IDS}
    finally:
        backend.use_library(None, None)


class _Host(object):
    on_gpu = False


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_rendered_frames_match_cv2(ref, env_frames, env_id):
    frames = env_frames[env_id]
    for q in QUALITIES:
        out = jpeg.encode_jpeg(_Host(), frames, quality=q)
        assert len(out) == len(frames)
        for f, data in zip(frames, out):
            assert data == cv2_jpeg(f, q), (env_id, q)
            assert len(data) <= _bound(ref, 224, 224)


@pytest.mark.parametrize("shape", [(33, 50), (16, 17), (1, 1), (17, 16), (8, 9), (31, 40)])
@pytest.mark.parametrize("kind", ["noise", "gradient"])
def test_odd_sizes_and_noise_match_cv2(ref, shape, kind):
    h, w = shape
    rng = np.random.default_rng(h * 1000 + w)
    if kind == "noise":
        frames = rng.integers(0, 256, (3, h, w, 3), dtype=np.uint8)
    else:
        yy, xx = np.mgrid[0:h, 0:w]
        frames = np.stack([np.stack([(xx * 7 + k * 40) % 256, (yy * 5 + xx) % 256, (yy * 11 + 3 * k) % 256], -1) for k in range(3)]).astype(np.uint8)
    for q in QUALITIES:
        out = jpeg.encode_jpeg(_Host(), frames, quality=q)
        for f, data in zip(frames, out):
            assert data == cv2_jpeg(f, q), (shape, kind, q)
            assert len(data) <= _bound(ref, w, h)


def test_noise_at_full_size_stays_within_the_bound(ref):
    frames = np.random.default_rng(0).integers(0, 256, (2, 224, 224, 3), dtype=np.uint8)
    for q in (95, 100):
        for f, data in zip(frames, jpeg.encode_jpeg(_Host(), frames, quality=q)):
            assert data == cv2_jpeg(f, q)
            assert data.count(b"\xff\x00") > 0 and len(data) <= _bound(ref, 224, 224)


def test_channel_offset_selects_the_camera(ref):
    rng = np.random.default_rng(1)
    two = rng.integers(0, 256, (2, 24, 40, 6), dtype=np.uint8)
    for off in (0, 3):
        out = jpeg.encode_jpeg(_Host(), two, quality=90, channel_offset=off)
        assert out == [cv2_jpeg(f[..., off:off + 3], 90) for f in two]


def test_strided_and_packed_outputs_agree(ref):
    frames = np.random.default_rng(2).integers(0, 256, (3, 20, 30, 3), dtype=np.uint8)
    b = _bound(ref, 30, 20)
    out = np.zeros(3 * b, np.uint8)
    lens = np.zeros(3, np.uint32)
    assert ref.lib.srl_jpeg_encode(frames.ctypes.data, 3, 20, 30, 3, 0, 80, None, out.ctypes.data, b, lens.ctypes.data, None) == 0
    strided = [out[i * b:i * b + lens[i]].tobytes() for i in range(3)]
    assert strided == jpeg.encode_jpeg(_Host(), frames, quality=80)


def test_bad_arguments_are_errors(ref):
    frames = np.zeros((1, 8, 8, 3), np.uint8)
    out = np.zeros(_bound(ref, 8, 8), np.uint8)
    lens = np.zeros(1, np.uint32)
    call = lambda **k: ref.lib.srl_jpeg_encode(frames.ctypes.data, 1, 8, 8, k.get("c", 3), k.get("off", 0), k.get("q", 95), None,
                                               out.ctypes.data, k.get("stride", 0), lens.ctypes.data, None)
    assert call() == 0
    for bad in (dict(q=0), dict(q=101), dict(off=1), dict(c=2), dict(stride=10)):
        assert call(**bad) != 0
    assert ref.lib.srl_jpeg_bound(0, 5) == 0
    with pytest.raises(Exception):
        jpeg.encode_jpeg(_Host(), frames, quality=0)


def test_episode_saver_writes_encoded_frames(tmp_path):
    from state_representation.episode_saver import EpisodeSaver
    saver = EpisodeSaver("ds", 0.28, path=str(tmp_path) + "/")
    a, b, c = b"\xff\xd8one", b"\xff\xd8two", b"\xff\xd8three"
    saver.reset(a, np.zeros(3), np.zeros(3))
    saver.step((b, c), 1, 0, False, np.ones(3))
    saver.step(None, 2, 1, True, np.ones(3))
    rec = os.path.join(str(tmp_path), "ds", "record_000")
    assert open(os.path.join(rec, "frame000000.jpg"), "rb").read() == a
    assert open(os.path.join(rec, "frame000001_1.jpg"), "rb").read() == b
    assert open(os.path.join(rec, "frame000001_2.jpg"), "rb").read() == c
    assert sorted(os.listdir(rec)) == ["frame000000.jpg", "frame000001_1.jpg", "frame000001_2.jpg"]
    gt = np.load(os.path.join(str(tmp_path), "ds", "ground_truth.npz"))
    assert list(gt["images_path"]) == ["ds/record_000/frame000000", "ds/record_000/frame000001"]
