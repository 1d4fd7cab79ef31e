"""
A2C timings on one GPU, in one process: the card and its power limit; A2C env-steps/s on KukaButton at 4096 envs (captured, two updates per
replay) in runs alternating with PPO2's; the time of one update split into collection / returns + gradient / optimiser (eager, synchronised
between the phases); and CUDA-event times of srl_a2c_grad and srl_clip_rmsprop against the torch code they replace (autograd of the loss;
the global-norm clip + RMSProp step of rl_baselines.a2c.clip_rmsprop, and torch's own clip_grad_norm_ + RMSprop), each launch after an
L2 flush.

    python scripts/a2c_timing.py [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))

import torch  # noqa: E402

ENV, N = "KukaButtonGymEnv-v0", 4096


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return q.strip().splitlines()[0]


def flushed_event_ms(fn, iters=200, warmup=20):
    """Median of per-launch CUDA-event times, a 256 MB write (more than the 50 MB L2) before each launch."""
    scratch = torch.empty(64 * 1024 * 1024, device="cuda")
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        scratch.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def steady_rate(hist, skip):
    """env-steps/s between history entry `skip` and the last (the history's fps is cumulative from the first update)."""
    (s0, _, f0), (s1, _, f1) = hist[skip], hist[-1]
    return (s1 - s0) / (s1 / f1 - s0 / f0)


def optimiser_kernels(lib):
    from rl_baselines.a2c import a2c_loss, clip_rmsprop
    from rl_baselines.ppo2 import MlpPolicy
    from srl_sim.policy import FusedA2CGrad, FusedClipRMSprop, policy_params
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    pol = MlpPolicy(3, n_actions=6).to(dev)
    B = 5 * N
    obs, act = torch.randn(B, 3, device=dev), torch.randint(0, 6, (B,), device=dev)
    ret, val = torch.randn(B, device=dev), torch.randn(B, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    fg = FusedA2CGrad(lib, pol, B)
    fo = FusedClipRMSprop(lib, pol, 0.5, 0.99, 1e-5)
    fo.lr.fill_(1e-9)
    params = policy_params(pol)
    ms = [torch.ones_like(p) for p in params]
    lr = torch.tensor(1e-9, device=dev)
    r = dict(rows=B)
    r["srl_a2c_grad_ms"] = flushed_event_ms(lambda: fg(None, obs, act, ret, val, 0.01, 0.5, stream=st))

    def autograd():
        for p in params:
            p.grad.zero_()
        a2c_loss(pol, obs, act, ret, val, 0.01, 0.5).backward()
    r["torch_autograd_grad_ms"] = flushed_event_ms(autograd)
    r["srl_clip_rmsprop_ms"] = flushed_event_ms(lambda: fo(stream=st))
    r["torch_clip_rmsprop_restatement_ms"] = flushed_event_ms(lambda: clip_rmsprop(params, ms, lr, 0.5, 0.99, 1e-5))
    opt = torch.optim.RMSprop(params, lr=1e-9, alpha=0.99, eps=1e-5)

    def torch_opt():
        torch.nn.utils.clip_grad_norm_(params, 0.5)
        opt.step()
    r["torch_clip_grad_norm_plus_optim_rmsprop_ms"] = flushed_event_ms(torch_opt)
    return r


def a2c_run(updates=600):
    from rl_baselines.a2c import train
    hist = train(ENV, N, N * 5 * updates, seed=0, env_kwargs=dict(is_discrete=True), verbose=0)
    return dict(algo="a2c", updates=len(hist), env_steps_per_s=steady_rate(hist, len(hist) // 4), last_mean_return=hist[-1][1])


def ppo2_run(updates=6):
    from rl_baselines.ppo2 import train
    hist = train(ENV, N, N * 128 * updates, seed=0, env_kwargs=dict(is_discrete=True), verbose=0)
    return dict(algo="ppo2", updates=len(hist), env_steps_per_s=steady_rate(hist, 1), last_mean_return=hist[-1][1])


def phases(updates=200):
    from rl_baselines.a2c import train
    pt = {}
    train(ENV, N, N * 5 * updates, seed=0, env_kwargs=dict(is_discrete=True), verbose=0, phase_times=pt)
    return {k + "_ms_per_update": 1e3 * v / updates for k, v in pt.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r08_a2c_timing.json"))
    args = ap.parse_args()
    from srl_sim._abi import load_cuda_library
    lib = load_cuda_library()
    res = dict(card=card(), env=ENV, num_envs=N)
    res["kernels"] = optimiser_kernels(lib)
    res["update_phases_eager_synchronised"] = phases()
    res["alternating_runs"] = [a2c_run(), ppo2_run(), a2c_run(), ppo2_run()]
    print(json.dumps(res, indent=1))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
