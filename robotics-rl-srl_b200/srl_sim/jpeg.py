"""
ctypes binding of ``include/srl_image.h``: batches of rendered frames encoded as JPEG files where they were rendered.

:func:`encode_jpeg` returns the files as ``bytes`` -- what ``cv2.imencode('.jpg', frame[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, quality])[1]``
holds for each RGB frame, byte for byte.  On the CUDA backend the frames are encoded on the device and packed back to back, and the host
receives one copy of the sizes and one copy of the packed files.  On the CPU oracle backend (test infrastructure) the same entry point of the
CPU checker ``csrc/libjpeg_ref.so`` encodes host arrays.  There is no fallback between the two: a backend without its encoder is an error.
"""
import ctypes
import os
from ctypes import c_int, c_size_t, c_void_p

import numpy as np

from . import _abi

JPEG_EXPORTS = ["srl_jpeg_bound", "srl_jpeg_workspace_bytes", "srl_jpeg_encode"]
JPEG_REF_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "csrc", "libjpeg_ref.so")


def bind(cdll):
    """Declare the argument types of the three entry points on a loaded library (raises AttributeError if one is missing)."""
    cdll.srl_jpeg_bound.restype = c_size_t
    cdll.srl_jpeg_bound.argtypes = [c_int, c_int]
    cdll.srl_jpeg_workspace_bytes.restype = c_size_t
    cdll.srl_jpeg_workspace_bytes.argtypes = [c_int, c_int, c_int]
    cdll.srl_jpeg_encode.restype = c_int
    cdll.srl_jpeg_encode.argtypes = [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p, c_void_p]
    return cdll


_ref_library = None


def reference_library():
    """The CPU checker (host pointers), as an ``srl_sim._abi.SimLibrary``-like object with ``lib`` and ``check``."""
    global _ref_library
    if _ref_library is None:
        if not os.path.isfile(JPEG_REF_PATH):
            raise _abi.SimError("%s is missing: run `python __graft_entry__.py build`" % JPEG_REF_PATH)
        lib = ctypes.CDLL(JPEG_REF_PATH)
        lib.srl_sim_last_error.restype = ctypes.c_char_p
        _ref_library = _RefLibrary(bind(lib))
    return _ref_library


class _RefLibrary(object):
    def __init__(self, lib):
        self.lib = lib

    def check(self, rc, what):
        if rc != 0:
            raise _abi.SimError("%s failed (rc=%d): %s" % (what, rc, self.lib.srl_sim_last_error().decode("utf-8", "replace")))


class _DeviceBuffers(object):
    """Workspace and output of the last call, kept for the next one of the same or a smaller size."""

    def __init__(self):
        self.ws = self.out = self.lens = None

    def get(self, torch, device, ws_bytes, out_bytes, n):
        if self.ws is None or self.ws.device != device or self.ws.numel() < ws_bytes:
            self.ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
        if self.out is None or self.out.device != device or self.out.numel() < out_bytes:
            self.out = torch.empty(out_bytes, dtype=torch.uint8, device=device)
        if self.lens is None or self.lens.device != device or self.lens.numel() < n:
            self.lens = torch.empty(n, dtype=torch.int32, device=device)
        return self.ws, self.out, self.lens


_buffers = _DeviceBuffers()


def release_buffers():
    """Free the device workspace and output kept between :func:`encode_jpeg` calls.  They are sized for the worst case (every block at its
    longest code, every byte stuffed): about 1.7 GB of workspace and 2 GB of output for 4096 frames of 224 x 224, so a caller that is done
    encoding can hand that memory back (the next call allocates again)."""
    _buffers.ws = _buffers.out = _buffers.lens = None


def encode_jpeg(backend, frames, quality=95, channel_offset=0):
    """
    :param backend: (srl_sim.backend.Backend) the CUDA backend (frames: a CUDA uint8 tensor) or the CPU oracle (frames: a numpy array)
    :param frames: uint8 [N, H, W, C] frames, RGB at channels ``channel_offset`` .. ``channel_offset + 2`` (C = 6: two cameras)
    :param quality: (int) 1..100, OpenCV's IMWRITE_JPEG_QUALITY
    :return: ([bytes]) one JPEG file per frame
    """
    n, h, w, c = (int(s) for s in frames.shape)
    if n == 0:
        return []
    if backend.on_gpu:
        torch = backend.torch
        if not frames.is_cuda or frames.dtype != torch.uint8:
            raise ValueError("encode_jpeg on the CUDA backend takes a CUDA uint8 tensor")
        frames = frames.contiguous()
        lib = bind(backend.library.lib)
        bound = int(lib.srl_jpeg_bound(w, h))
        ws, out, lens = _buffers.get(torch, frames.device, int(lib.srl_jpeg_workspace_bytes(n, w, h)), n * bound, n)
        rc = lib.srl_jpeg_encode(frames.data_ptr(), n, h, w, c, int(channel_offset), int(quality), ws.data_ptr(), out.data_ptr(), 0,
                                 lens.data_ptr(), backend.stream())
        backend.library.check(rc, "srl_jpeg_encode")
        sizes = lens[:n].cpu().numpy().astype(np.int64)
        data = out[:int(sizes.sum())].cpu().numpy()
    else:
        frames = np.ascontiguousarray(frames, dtype=np.uint8)
        ref = reference_library()
        bound = int(ref.lib.srl_jpeg_bound(w, h))
        data = np.empty(n * bound, dtype=np.uint8)
        lens = np.empty(n, dtype=np.uint32)
        rc = ref.lib.srl_jpeg_encode(frames.ctypes.data, n, h, w, c, int(channel_offset), int(quality), None, data.ctypes.data, 0,
                                     lens.ctypes.data, None)
        ref.check(rc, "srl_jpeg_encode")
        sizes = lens.astype(np.int64)
    ends = np.cumsum(sizes)
    raw = data.tobytes() if data.size == ends[-1] else data[:ends[-1]].tobytes()
    return [raw[e - s:e] for s, e in zip(sizes, ends)]
