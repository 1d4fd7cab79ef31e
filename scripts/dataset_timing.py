"""Cost of turning rendered frames into dataset files at 4096 envs (KukaButtonGymEnv-v0, 224 x 224, quality 95), on the GPU box:
  * device time of srl_jpeg_encode for the 4096 frames and of srl_sim_render for the same frames (CUDA events, median of 10);
  * frames/s of a stand-in per-step loop (render, encode, one copy of the sizes and one of the packed files to the host, one .jpg per
    frame written by a pool of 8 threads into a local temporary directory; no ground truth, no EpisodeSaver), at 4096 envs;
  * frames/s of `python -m environments.dataset_generator --num-envs N` end to end (MobileRobot -r and KukaButton, N envs = N episodes,
    written into a local temporary directory);
  * frames/s of host cv2.imencode on the same frames (1 and 8 threads), for comparison;
  * the card and its power limit, read in the same run.
Usage: python scripts/dataset_timing.py [--envs 4096] [--steps 5]"""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))
import torch  # noqa: E402
from srl_sim._abi import load_cuda_library  # noqa: E402
from srl_sim.backend import Backend  # noqa: E402
from srl_sim.jpeg import encode_jpeg  # noqa: E402
from srl_sim.model import load_kuka_scene  # noqa: E402
from srl_sim.render import KUKA_CAMERA, camera  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except Exception as e:                       # the numbers below still stand; say why the card is not named
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--quality", type=int, default=95)
    ap.add_argument("--gen-envs", type=int, default=256, help="envs (= episodes) of the end-to-end dataset_generator runs")
    args = ap.parse_args()
    n, w, h, q = args.envs, 224, 224, args.quality
    be = Backend(load_cuda_library(), 0)
    st = be.stream()
    lib = be.library.lib
    sim = be.make_sim("KukaButtonGymEnv-v0", n, model_blob=load_kuka_scene().blob, seed=0, random_target=True)
    sim.reset(stream=st)
    acts = torch.randint(0, 6, (32, n), dtype=torch.int32, device=be.torch_device)
    sim.rollout(32, acts, None, None, None, None, stream=st)
    frames = be.zeros((n, h, w, 3), np.uint8)
    obs, rew, done = be.zeros((n, sim.obs_dim), np.float32), be.zeros((n,), np.float32), be.zeros((n,), np.uint8)
    cam = camera(**KUKA_CAMERA)
    encode_jpeg(be, frames, quality=q)                                   # allocates the cached workspace and output
    from srl_sim import jpeg as _jpeg
    ws, out, lens = _jpeg._buffers.ws, _jpeg._buffers.out, _jpeg._buffers.lens

    def events(fn, reps=10):
        ms = []
        for _ in range(3):
            fn()
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(torch.cuda.current_stream()); fn(); e1.record(torch.cuda.current_stream())
            torch.cuda.synchronize(); ms.append(e0.elapsed_time(e1))
        return float(np.median(ms))

    render_ms = events(lambda: sim.render(cam, w, h, frames, stream=st))
    enc = lambda: be.library.check(lib.srl_jpeg_encode(frames.data_ptr(), n, h, w, 3, 0, q, ws.data_ptr(), out.data_ptr(), 0, lens.data_ptr(), st), "encode")
    encode_ms = events(enc)
    files = encode_jpeg(be, frames, quality=q)
    sizes = np.array([len(f) for f in files])
    print("card: %s" % card())
    print("%d frames of %d x %d, quality %d: render %.3f ms, encode %.3f ms (%.2f M frames/s); files %.1f KB mean (%.1f MB per batch, raw %.1f MB)"
          % (n, w, h, q, render_ms, encode_ms, n / encode_ms / 1e3, sizes.mean() / 1e3, sizes.sum() / 1e6, n * w * h * 3 / 1e6))

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            enc()
        torch.cuda.synchronize()
    for evt in prof.key_averages():
        if "jpeg" in evt.key:
            us = getattr(evt, "device_time_total", None) or getattr(evt, "cuda_time_total", 0.0)
            print("  %-22s %.3f ms per encode (torch.profiler)" % (evt.key.split("jpeg_")[-1].split("(")[0].split("<")[0], us / 5 / 1e3))

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for s in range(args.steps):
        sim.step(acts[s % 32], None, obs, rew, done, stream=st)
        sim.render(cam, w, h, frames, stream=st)
        encode_jpeg(be, frames, quality=q)
    dt = time.perf_counter() - t0
    print("step + render + encode + copy of %d files to the host, %d steps: %.1f ms per step, %.0f frames/s"
          % (n, args.steps, dt / args.steps * 1e3, n * args.steps / dt))

    tmp = tempfile.mkdtemp(prefix="dataset_timing_")
    try:
        with ThreadPoolExecutor(8) as pool:
            def write(i, data, step):
                with open(os.path.join(tmp, "s%02d_%05d.jpg" % (step, i)), "wb") as f:
                    f.write(data)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for s in range(args.steps):
                sim.step(acts[s % 32], None, obs, rew, done, stream=st)
                sim.render(cam, w, h, frames, stream=st)
                out_files = encode_jpeg(be, frames, quality=q)
                list(pool.map(lambda a: write(a[0], a[1], s), enumerate(out_files)))
            dt = time.perf_counter() - t0
        print("stand-in loop (no ground truth, no EpisodeSaver): step + render + encode + copy + write %d files per step, %d steps: "
              "%.1f ms per step, %.0f frames/s"
              % (n, args.steps, dt / args.steps * 1e3, n * args.steps / dt))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)

    # the generator itself, end to end: python -m environments.dataset_generator --num-envs N into a local temporary directory
    from environments import dataset_generator
    for env_id, extra, envs in (("MobileRobotGymEnv-v0", ["-r"], args.gen_envs), ("KukaButtonGymEnv-v0", [], args.gen_envs)):
        tmp = tempfile.mkdtemp(prefix="dataset_timing_gen_")
        try:
            t0 = time.perf_counter()
            recorded = dataset_generator.main(["--env", env_id, "--num-episode", str(envs), "--num-envs", str(envs), "--save-path", tmp + "/",
                                               "--name", "ds", "--quality", str(q)] + extra)
            dt = time.perf_counter() - t0
            n_files = sum(len(f) for _, _, f in os.walk(os.path.join(tmp, "ds")))
            print("dataset_generator --env %s --num-envs %d --num-episode %d: %d frames recorded (%d files) in %.1f s, %.0f frames/s end to end"
                  % (env_id, envs, envs, recorded, n_files, dt, recorded / dt))
        finally:
            shutil.rmtree(tmp, ignore_errors=True)

    import cv2
    files = encode_jpeg(be, frames, quality=q)                           # the frames of the last step
    host = frames[:512].cpu().numpy()
    bgr = [np.ascontiguousarray(f[..., ::-1]) for f in host]
    t0 = time.perf_counter()
    for f in bgr:
        cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, q])
    one = len(bgr) / (time.perf_counter() - t0)
    with ThreadPoolExecutor(8) as pool:
        t0 = time.perf_counter()
        list(pool.map(lambda f: cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, q]), bgr))
        eight = len(bgr) / (time.perf_counter() - t0)
    same = all(files[i] == cv2.imencode(".jpg", bgr[i], [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes() for i in range(len(bgr)))
    print("host cv2.imencode of the same frames: %.0f frames/s on 1 thread, %.0f frames/s on 8 threads (%d host cores); GPU bytes equal cv2's: %s"
          % (one, eight, os.cpu_count(), same))
    sim.close()


if __name__ == "__main__":
    main()
