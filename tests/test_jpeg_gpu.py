"""
The sm_90a JPEG encoder (include/srl_image.h in libsrl_sim_b200.so) against its CPU checker (csrc/libjpeg_ref.so, itself held to
cv2.imencode byte for byte by tests/test_jpeg_cpu.py): frames the CUDA library renders for every env id, both Kuka cameras through
channel_offset, odd sizes, uniform noise, every tested quality, batches of 1, 3 and 4096 frames, strided and packed output, and the same
bytes on every call.
"""
import numpy as np
import pytest

from environments.registry import registered_env
from srl_sim import jpeg

pytestmark = pytest.mark.gpu

QUALITIES = (1, 50, 75, 95, 100)
ENV_IDS = ["KukaButtonGymEnv-v0", "KukaRandButtonGymEnv-v0", "Kuka2ButtonGymEnv-v0", "KukaMovingButtonGymEnv-v0",
           "MobileRobotGymEnv-v0", "MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0", "MobileRobotLineTargetGymEnv-v0"]


class _Host(object):
    on_gpu = False


def _checker(frames, quality, channel_offset=0):
    return jpeg.encode_jpeg(_Host(), np.ascontiguousarray(frames), quality=quality, channel_offset=channel_offset)


def _cuda(be, frames, quality, channel_offset=0):
    t = be.torch.from_numpy(np.ascontiguousarray(frames)).to(be.torch_device) if isinstance(frames, np.ndarray) else frames
    return jpeg.encode_jpeg(be, t, quality=quality, channel_offset=channel_offset)


@pytest.fixture(scope="module")
def cuda_frames(cuda_backend):
    """Frames the CUDA library renders: every env id after a reset and three random steps (Kuka with both cameras)."""
    out = {}
    for env_id in ENV_IDS:
        kuka = env_id.startswith("Kuka")
        env = registered_env[env_id][0](srl_model="raw_pixels", random_target=True, **({"multi_view": True} if kuka else {}))
        env.seed(11)
        env.action_space.seed(11)
        frames = [env.reset()]
        for _ in range(3):
            frames.append(env.step(env.action_space.sample())[0])
        env.close()
        out[env_id] = np.stack(frames)
    return out


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_rendered_frames_equal_the_checker(cuda_backend, cuda_frames, env_id):
    frames = cuda_frames[env_id]
    offsets = (0, 3) if frames.shape[-1] == 6 else (0,)
    for off in offsets:
        for q in QUALITIES:
            assert _cuda(cuda_backend, frames, q, off) == _checker(frames, q, off), (env_id, off, q)


@pytest.mark.parametrize("shape", [(33, 50), (16, 17), (1, 1), (17, 16), (8, 9), (31, 40)])
@pytest.mark.parametrize("n", [1, 3])
def test_odd_sizes_and_noise_equal_the_checker(cuda_backend, shape, n):
    h, w = shape
    frames = np.random.default_rng(h * 100 + w + n).integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    for q in QUALITIES:
        assert _cuda(cuda_backend, frames, q) == _checker(frames, q), (shape, n, q)


def test_4096_frames_equal_the_checker_and_repeat(cuda_backend, cuda_frames):
    rng = np.random.default_rng(5)
    pool = np.concatenate([f[..., :3] for f in cuda_frames.values()])
    frames = pool[rng.integers(0, len(pool), 4096)]
    noisy = rng.random(4096) < 0.25                                      # a quarter of uniform noise: long codes and many 0xFF bytes
    frames[noisy] = rng.integers(0, 256, (int(noisy.sum()), 224, 224, 3), dtype=np.uint8)
    first = _cuda(cuda_backend, frames, 95)
    assert first == _checker(frames, 95)
    assert _cuda(cuda_backend, frames, 95) == first                      # deterministic: the same bytes on every call


def test_strided_output_equals_packed(cuda_backend):
    torch = cuda_backend.torch
    frames_np = np.random.default_rng(3).integers(0, 256, (5, 40, 56, 3), dtype=np.uint8)
    frames = torch.from_numpy(frames_np).to(cuda_backend.torch_device)
    lib = jpeg.bind(cuda_backend.library.lib)
    b = int(lib.srl_jpeg_bound(56, 40))
    ws = torch.empty(int(lib.srl_jpeg_workspace_bytes(5, 56, 40)), dtype=torch.uint8, device=frames.device)
    out = torch.zeros(5 * b, dtype=torch.uint8, device=frames.device)
    lens = torch.zeros(5, dtype=torch.int32, device=frames.device)
    rc = lib.srl_jpeg_encode(frames.data_ptr(), 5, 40, 56, 3, 0, 85, ws.data_ptr(), out.data_ptr(), b, lens.data_ptr(), cuda_backend.stream())
    cuda_backend.library.check(rc, "srl_jpeg_encode")
    o, n = out.cpu().numpy(), lens.cpu().numpy()
    assert [o[i * b:i * b + n[i]].tobytes() for i in range(5)] == _cuda(cuda_backend, frames, 85) == _checker(frames_np, 85)


def test_files_decode_back_to_the_frames(cuda_backend, cuda_frames):
    cv2 = pytest.importorskip("cv2")
    frames = cuda_frames["KukaButtonGymEnv-v0"][..., :3]
    for f, data in zip(frames, _cuda(cuda_backend, frames, 95)):
        back = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]
        mse = np.mean((back.astype(float) - f.astype(float)) ** 2)
        psnr = 10 * np.log10(255.0 ** 2 / max(mse, 1e-12))
        # quality 95 with 4:2:0 chroma: the drawn scene's sharp colour edges cost a few levels on average, the frame stays above 30 dB
        assert back.shape == f.shape and psnr > 30.0, psnr


def test_bad_arguments_are_errors(cuda_backend):
    torch = cuda_backend.torch
    frames = torch.zeros((1, 8, 8, 3), dtype=torch.uint8, device=cuda_backend.torch_device)
    with pytest.raises(Exception):
        jpeg.encode_jpeg(cuda_backend, frames, quality=101)
    with pytest.raises(Exception):
        jpeg.encode_jpeg(cuda_backend, frames, channel_offset=1)
