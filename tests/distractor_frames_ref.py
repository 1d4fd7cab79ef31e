"""
CPU checker of KukaRandButton frames with distractor bodies (test-only): `oracle_render_bodies` of oracle/liboracle_sim.so.  `render` draws
an oracle handle's scene plus caller-given bodies (the SRL_F_DISTRACTORS layout, f64[N][11][9]) through the same list builder and per-pixel
arithmetic as the CUDA library.
"""
import ctypes
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LIB = os.path.join(ROOT, "oracle", "liboracle_sim.so")
_lib = None


def library():
    global _lib
    if _lib is None:
        from srl_sim._abi import SimLibrary
        lib = SimLibrary(ORACLE_LIB).lib
        P = ctypes.c_void_p
        lib.oracle_render_bodies.restype = ctypes.c_int
        lib.oracle_render_bodies.argtypes = [P, P, ctypes.c_size_t, P, P, ctypes.c_int, ctypes.c_int, P]
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
    rc = lib.oracle_render_bodies(sim.handle, blob.ctypes.data, blob.nbytes, bodies.ctypes.data, ctypes.addressof(c), int(width), int(height),
                                  out.ctypes.data)
    if rc:
        raise RenderError(lib.srl_sim_last_error().decode())
    return out
