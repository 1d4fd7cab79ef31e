"""Device time of srl_sim_render_cameras (one camera per env) next to srl_sim_render (one camera for the batch).

    python scripts/render_cameras_timing.py [--runs 5]

4096 MobileRobot frames of 224 x 224, after a 30-step rollout: (a) srl_sim_render with the top-down camera, (b) srl_sim_render_cameras with
that camera for every env, (c) the first-person cameras with follow_robot.  4096 KukaButton frames of 224 x 224, after a 30-step rollout:
(a) srl_sim_render with camera 1, (b) srl_sim_render_cameras with camera 1 for every env.  The camera arrays are built once, so (b) and (c) time
the calls a training loop makes every step (the cameras are cached by the handle; (c) still finishes every camera from the robot positions on
the device).  Each number is the median over runs of the median of 10 calls timed with CUDA events, the L2 flushed before each call; the cases
alternate within a run.  (b) is checked to give the same bytes as (a).
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))


def _gpu():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    import torch
    from srl_sim._abi import load_cuda_library
    from srl_sim.backend import Backend
    from srl_sim.model import load_kuka_scene
    from srl_sim.render import KUKA_CAMERA, MOBILE_CAMERA, MOBILE_FPV_FOLLOW, camera, camera_array

    print("before: name, power limit, SM clock, max SM clock:", _gpu())
    be = Backend(load_cuda_library(), 0)
    st = be.stream()
    n, T = 4096, 30
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    buf = torch.empty((n, 224, 224, 3), dtype=torch.uint8, device="cuda")

    def handle(env_id, blob):
        sim = be.make_sim(env_id, n, model_blob=blob, seed=0, random_target=True)
        sim.reset(stream=st)
        acts = torch.randint(0, 4, (T, n), dtype=torch.int32, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
        o = be.zeros((T, n, sim.obs_dim), np.float32); r = be.zeros((T, n), np.float32); d = be.zeros((T, n), np.uint8)
        sim.rollout(T, acts, None, o, r, d, stream=st)
        return sim

    mob, kuka = handle("MobileRobotGymEnv-v0", None), handle("KukaButtonGymEnv-v0", load_kuka_scene().blob)
    top, k1 = camera(**MOBILE_CAMERA), camera(**KUKA_CAMERA)
    top_n, k1_n, fpv_n = camera_array([MOBILE_CAMERA] * n), camera_array([KUKA_CAMERA] * n), camera_array([MOBILE_FPV_FOLLOW] * n)
    cases = [
        ("MobileRobot (a) srl_sim_render, top-down camera", lambda: mob.render(top, 224, 224, buf, stream=st)),
        ("MobileRobot (b) srl_sim_render_cameras, top-down camera for every env", lambda: mob.render_cameras(top_n, False, 224, 224, buf, stream=st)),
        ("MobileRobot (c) srl_sim_render_cameras, fpv cameras, follow_robot", lambda: mob.render_cameras(fpv_n, True, 224, 224, buf, stream=st)),
        ("KukaButton (a) srl_sim_render, camera 1", lambda: kuka.render(k1, 224, 224, buf, stream=st)),
        ("KukaButton (b) srl_sim_render_cameras, camera 1 for every env", lambda: kuka.render_cameras(k1_n, False, 224, 224, buf, stream=st)),
    ]
    for family, a, b in (("MobileRobot", 0, 1), ("KukaButton", 3, 4)):
        cases[a][1](); ref = buf.clone(); cases[b][1]()
        print("%s: (b) gives the bytes of (a): %s" % (family, bool(torch.equal(ref, buf))))

    def timed(fn, reps=10):
        for _ in range(3):
            fn()
        ms = []
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return float(np.median(ms))

    res = [[] for _ in cases]
    for _ in range(args.runs):
        for k, (_, fn) in enumerate(cases):
            res[k].append(timed(fn))
    print("4096 frames of 224 x 224, device time per call:")
    for (name, _), v in zip(cases, res):
        v = np.array(v)
        print("  %-72s median %.3f ms  min %.3f  max %.3f  runs %s" % (name, np.median(v), v.min(), v.max(), " ".join("%.3f" % x for x in v)))
    print("after: name, power limit, SM clock, max SM clock:", _gpu())


if __name__ == "__main__":
    main()
