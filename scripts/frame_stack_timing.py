"""
Timings of stacked state observations (``--num-stack k``) on one GPU, in one process: the card and its power limit, CUDA-event times of the policy
step, the observation filter (the stack filter for widths above the raw observation's) and one gradient minibatch at widths 3, 12 and 32 at the
4096-env trainer's shapes (4096 envs, minibatch 131 072), and PPO2 env-steps/s on KukaButton at 4096 envs for k = 1 and k = 4 in alternating runs.

    python scripts/frame_stack_timing.py [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0]


def event_ms(fn, iters=200, warmup=20):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernels(lib, W, N=4096, mb=131072):
    from rl_baselines.ppo2 import MlpPolicy, RunningNorm
    from srl_sim.policy import FusedPolicy, FusedPPO2Grad
    dev = torch.device("cuda", 0)
    torch.manual_seed(W)
    pol = MlpPolicy(W, n_actions=6).to(dev)
    norm = RunningNorm(W, dev)
    fp = FusedPolicy(lib, pol, norm.state, seed=1)
    st = torch.cuda.current_stream().cuda_stream
    obs = torch.randn(N, W, device=dev)
    act, logp, val = torch.zeros(N, dtype=torch.int32, device=dev), torch.empty(N, device=dev), torch.empty(N, device=dev)
    obs_buf, act_buf = torch.empty(N, W, device=dev), torch.empty(N, dtype=torch.int64, device=dev)
    r = {"width": W}
    r["policy_act_ms"] = event_ms(lambda: fp.act(N, obs, act, logp, val, obs_buf=obs_buf, act_buf=act_buf, stream=st))
    out = torch.empty(N, W, device=dev)
    if W <= 8:
        r["filter"] = "srl_obs_filter D=%d" % W
        r["filter_ms"] = event_ms(lambda: fp.filter(N, obs, out, update=True, stream=st))
    else:
        D = 2 if W % 3 else 3                        # Kuka's 3-D ground truth for W = 12 (k = 4), MobileRobot's 2-D one for W = 32 (k = 16)
        raw, done = torch.randn(N, D, device=dev), (torch.rand(N, device=dev) < 0.01).to(torch.uint8)
        stack = torch.zeros(N, W, device=dev)
        r["filter"] = "srl_obs_stack_filter D=%d k=%d" % (D, W // D)
        r["filter_ms"] = event_ms(lambda: fp.stack_filter(N, raw, done, stack, out, update=True, stream=st))
    rows = 128 * N
    grad = FusedPPO2Grad(lib, pol, mb)
    o = torch.randn(rows, W, device=dev)
    a = torch.randint(0, 6, (rows,), device=dev)
    adv, ret, olp, ov = (torch.randn(rows, device=dev) for _ in range(4))
    idx = torch.randperm(rows, device=dev)[:mb].contiguous()
    r["ppo2_grad_ms"] = event_ms(lambda: grad(idx, o, a, adv, ret, olp, ov, 0.2, 0.01, 0.5, stream=st), iters=50, warmup=5)
    return r


def trainer(k, N=4096, updates=6):
    from rl_baselines import ppo2
    hist = ppo2.train("KukaButtonGymEnv-v0", N, N * 128 * updates, seed=0, verbose=0, num_stack=k)
    steps0, _, fps0 = hist[0]
    steps, _, fps = hist[-1]
    t0, t1 = steps0 / fps0, steps / fps
    return (steps - steps0) / (t1 - t0)             # env-steps/s over updates 2.., past the one-off captures of the first


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from srl_sim._abi import load_cuda_library
    lib = load_cuda_library()
    res = {"card": card(), "kernels": [kernels(lib, W) for W in (3, 12, 32)], "ppo2_kuka_4096": []}
    for rnd in range(args.rounds):
        for k in (1, 4):
            res["ppo2_kuka_4096"].append({"round": rnd, "num_stack": k, "env_steps_per_s": trainer(k)})
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
