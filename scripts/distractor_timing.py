"""Cost of KukaRandButtonGymEnv's distractor bodies: the fused 128-step rollout of 4096 envs (random actions from the env stream) with
and without them, alternating runs; prints the median and spread of each and the card it ran on (name and power limit read in the
same call).  Usage: python scripts/distractor_timing.py [--runs 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--max-seconds", type=float, default=60.0, help="give up (before the timed runs) when the warm-up rollout with the bodies takes longer")
    args = ap.parse_args()
    import torch
    from srl_sim._abi import load_cuda_library
    from srl_sim.backend import Backend
    from srl_sim.model import distractor_blob, load_kuka_scene
    be = Backend(load_cuda_library(), 0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    n, T = args.envs, args.steps
    sims = {}
    import time
    for bodies in (False, True):
        s = be.make_sim("KukaRandButtonGymEnv-v0", n, seed=0, model_blob=load_kuka_scene().blob, is_discrete=True)
        if bodies:
            s.set_distractors(distractor_blob())
        s.reset(stream=be.stream())
        torch.cuda.synchronize()
        t0 = time.time()
        s.rollout(T, stream=be.stream())          # warm-up
        torch.cuda.synchronize()
        if time.time() - t0 > args.max_seconds:
            print(json.dumps({"card": card, "envs": n, "steps": T, "aborted": "warm-up rollout took %.1f s" % (time.time() - t0)}))
            return
        sims[bodies] = s
    times = {False: [], True: []}
    for _ in range(args.runs):
        for bodies in (False, True):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            sims[bodies].rollout(T, stream=be.stream())
            b.record()
            torch.cuda.synchronize()
            times[bodies].append(a.elapsed_time(b))
    out = {"card": card, "envs": n, "steps": T, "runs": args.runs}
    for bodies, key in ((False, "off"), (True, "on")):
        t = np.array(times[bodies])
        out[key] = {"median_ms": float(np.median(t)), "min_ms": float(t.min()), "max_ms": float(t.max()), "all_ms": [float(x) for x in t]}
    out["ratio"] = out["on"]["median_ms"] / out["off"]["median_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
