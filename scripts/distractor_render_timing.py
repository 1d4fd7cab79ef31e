"""Device time of srl_sim_render with the KukaRandButton distractor bodies drawn, next to the KukaButton frames of the bench's render_kuka
leg, for one or more builds of the library in one process, alternating builds run by run.

    python scripts/distractor_render_timing.py [--lib A.so --lib B.so ...] [--runs 5]

Per run and build: 4096 x 224 x 224 KukaButton frames (camera 1, culled: the render_kuka workload), then 4096 x 224 x 224 KukaRandButton
frames with the bodies simulated, after a 64-step rollout (the sphere has been kicked at step 10), both cameras, with and without the per-tile
culling.  A build that predates body drawing simulates the same bodies but does not draw them, so the difference between two such builds on the
KukaRandButton rows is the cost of drawing them.  Each number is the median of 10 calls timed with CUDA events, the L2 flushed before each.
With two or more builds the script also checks that every env id's frames without bodies are the same bytes under every build.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="library build to time (repeatable; default: the built one)")
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    import subprocess
    import torch
    from srl_sim import _abi
    from srl_sim._abi import CUDA_LIBRARY_PATH, SimLibrary
    from srl_sim.backend import Backend
    from srl_sim.model import distractor_blob, load_kuka_scene
    from srl_sim.render import KUKA_CAMERA, KUKA_CAMERA_2, MOBILE_CAMERA, camera, mobile_fpv_camera

    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    libs = [os.path.abspath(p) for p in (args.lib or [CUDA_LIBRARY_PATH])]
    bes = [Backend(SimLibrary(p), 0) for p in libs]
    n, T = 4096, 64
    blob = load_kuka_scene().blob
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    buf = torch.empty((n, 224, 224, 3), dtype=torch.uint8, device="cuda")

    def timed(be, sim, cam, no_cull, reps=10):
        if no_cull:
            os.environ["SRL_RENDER_NO_CULL"] = "1"
        else:
            os.environ.pop("SRL_RENDER_NO_CULL", None)
        st = be.stream()
        for _ in range(3):
            sim.render(camera(**cam), 224, 224, buf, stream=st)
        ms = []
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); sim.render(camera(**cam), 224, 224, buf, stream=st); e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        os.environ.pop("SRL_RENDER_NO_CULL", None)
        return float(np.median(ms))

    def handles(be):
        st = be.stream()
        kb = be.make_sim("KukaButtonGymEnv-v0", n, model_blob=blob, seed=0, random_target=True)
        kb.reset(stream=st)
        rb = be.make_sim("KukaRandButtonGymEnv-v0", n, model_blob=blob, seed=0, random_target=True)
        rb.set_distractors(distractor_blob())
        rb.reset(stream=st)
        for sim in (kb, rb):
            acts = torch.randint(0, 6, (T, n), dtype=torch.int32, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
            o = be.zeros((T, n, 3), np.float32); r = be.zeros((T, n), np.float32); d = be.zeros((T, n), np.uint8)
            sim.rollout(T, acts, None, o, r, d, stream=st)
        torch.cuda.synchronize()
        return kb, rb

    sims = [handles(be) for be in bes]
    rows = [("render_kuka: KukaButton, camera 1, culled", 0, KUKA_CAMERA, False)] + \
        [("KukaRandButton + bodies, %s, %s" % (cn, "not culled" if nc else "culled"), 1, cam, nc)
         for cn, cam in (("camera 1", KUKA_CAMERA), ("camera 2", KUKA_CAMERA_2)) for nc in (False, True)]
    res = {(li, ri): [] for li in range(len(libs)) for ri in range(len(rows))}
    for run in range(args.runs):
        for li, be in enumerate(bes):
            for ri, (_, which, cam, nc) in enumerate(rows):
                res[(li, ri)].append(timed(be, sims[li][which], cam, nc))
    for ri, (name, _, _, _) in enumerate(rows):
        print(name)
        for li, p in enumerate(libs):
            v = np.array(res[(li, ri)])
            print("  %-60s median %.3f ms  min %.3f  max %.3f  runs %s" % (p[-60:], np.median(v), v.min(), v.max(), " ".join("%.3f" % x for x in v)))

    if len(bes) > 1:
        # frames without bodies: the same bytes under every build, every env id, both cameras of its family
        for env_id in sorted(_abi.ENV_KINDS):
            kuka = env_id.startswith("Kuka")
            cams = [KUKA_CAMERA, KUKA_CAMERA_2] if kuka else [MOBILE_CAMERA, mobile_fpv_camera((2.0, 2.0))]
            cfg = dict(seed=2, random_target=True)
            if env_id in ("MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0"):
                cfg["is_discrete"] = True
            acts = np.random.RandomState(3).randint(0, 6 if kuka else 2, size=(20, 256)).astype(np.int32)
            out = []
            for be in bes:
                sim = be.make_sim(env_id, 256, model_blob=blob if kuka else None, **cfg)
                st = be.stream()
                sim.reset(stream=st)
                o = be.zeros((20, 256, sim.obs_dim), np.float32); r = be.zeros((20, 256), np.float32); d = be.zeros((20, 256), np.uint8)
                sim.rollout(20, be.from_host(acts), None, o, r, d, stream=st)
                frames = []
                for c in cams:
                    for (w, h) in ((224, 224), (50, 33)):
                        f = be.zeros((256, h, w, 3), np.uint8)
                        sim.render(camera(**c), w, h, f, stream=st)
                        frames.append(be.to_host(f).copy())
                out.append(frames)
                sim.close()
            same = all(np.array_equal(a, b) for other in out[1:] for a, b in zip(out[0], other))
            print("frames without bodies, %-32s identical across builds: %s" % (env_id, same))


if __name__ == "__main__":
    main()
