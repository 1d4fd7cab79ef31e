"""
The four-lanes-per-env kinematics / dynamics of the Kuka kernel (csrc/kuka_coop.cuh) compile for the host too: tests/host/coop_host_check.cpp
runs the 4 lanes of a group one after the other, phase by phase, through the same scratch layout, and compares every intermediate the kernel
consumes -- joint frames, axes, world inertias, link states, contact manifold (flags, records, order), bias torques, mass matrix, M^-1,
contact rows -- with the one-thread-per-env functions of csrc/kuka_device.cuh (themselves checked against the float64 oracle and the numpy
Lagrangian reference) on 2 x 300 random configurations of the real model, two thirds of them placed in contact.  The model is the
KukaParams the library itself fills from the blob (csrc/kuka_params.cuh: kuka_params_from_blob), at the blob's own time step.
"""
import os
import subprocess

import numpy as np

from srl_sim.model import load_kuka_scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_four_lane_phases_match_the_one_thread_functions_on_the_library_model(tmp_path):
    blob = tmp_path / "kuka_blob.bin"
    np.ascontiguousarray(load_kuka_scene().blob, dtype=np.float64).tofile(str(blob))
    exe = tmp_path / "coop_host_check"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-ffp-contract=off", "-Wno-unknown-pragmas", "-o", str(exe),
                           os.path.join(ROOT, "tests", "host", "coop_host_check.cpp")])
    out = subprocess.run([str(exe), str(blob), "300"], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "one-button: 300 cases ok" in out.stdout and "two-button: 300 cases ok" in out.stdout
