"""
CPU checker of srl_sim_render_cameras (test-only): tests/host/render_cameras_ref.cpp compiled once per process into a temporary directory
against oracle/liboracle_sim.so.  The library it makes exports srl_sim_render_cameras and resolves every other symbol of the C-ABI from the
oracle library, so ``library()`` is an ``SimLibrary`` that drives oracle handles through the whole binding, per-env cameras included.
"""
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
_lib = None


def library():
    global _lib
    if _lib is None:
        from srl_sim._abi import SimLibrary
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR])
        out = os.path.join(tempfile.mkdtemp(prefix="rcr_"), "librender_cameras_ref.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-shared", "-o", out,
                               os.path.join(ROOT, "tests", "host", "render_cameras_ref.cpp"), os.path.join(ORACLE_DIR, "liboracle_sim.so"),
                               "-Wl,-rpath," + ORACLE_DIR])
        _lib = SimLibrary(out)
    return _lib
