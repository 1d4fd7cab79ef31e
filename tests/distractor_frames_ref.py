"""
CPU checker of KukaRandButton frames with distractor bodies (test-only): tests/host/distractor_frames_ref.cpp compiled once per process into
a temporary directory against oracle/liboracle_sim.so.  `render` draws an oracle handle's scene plus caller-given bodies (the
SRL_F_DISTRACTORS layout, f64[N][11][9]) through the same list builder and per-pixel arithmetic as the CUDA library.
"""
import ctypes
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
_lib = None


def library():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR])
        out = os.path.join(tempfile.mkdtemp(prefix="dfr_"), "libdistractor_frames_ref.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-shared", "-o", out,
                               os.path.join(ROOT, "tests", "host", "distractor_frames_ref.cpp"), os.path.join(ORACLE_DIR, "liboracle_sim.so"),
                               "-Wl,-rpath," + ORACLE_DIR])
        lib = ctypes.CDLL(out)
        P = ctypes.c_void_p
        lib.dfr_render.restype = ctypes.c_int
        lib.dfr_render.argtypes = [P, P, ctypes.c_size_t, P, P, ctypes.c_int, ctypes.c_int, P]
        lib.dfr_last_error.restype = ctypes.c_char_p
        _lib = lib
    return _lib


class RenderError(RuntimeError):
    pass


def render(sim, blob, bodies, cam, width, height):
    """u8[N, H, W, 3]: the frames of oracle handle `sim` with `bodies` (f64[N, 11, 9]) drawn by the drawing words of asset blob `blob`."""
    from srl_sim.render import camera
    lib = library()
    blob = np.ascontiguousarray(blob, np.float64)
    bodies = np.ascontiguousarray(bodies, np.float64).reshape(sim.num_envs, 11, 9)
    out = np.zeros((sim.num_envs, height, width, 3), np.uint8)
    c = camera(**cam)
    rc = lib.dfr_render(sim.handle, blob.ctypes.data, blob.nbytes, bodies.ctypes.data, ctypes.addressof(c), int(width), int(height),
                        out.ctypes.data)
    if rc:
        raise RenderError(lib.dfr_last_error().decode())
    return out
