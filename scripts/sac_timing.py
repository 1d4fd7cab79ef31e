"""
SAC timing on one GPU (profiles/r10_sac_timing.json): the card and its power limit; CUDA-event times of each SAC kernel at N = 4096 envs and
B = 64 N = 262 144 samples over the default 50 000-row ring, each launch after an L2 flush; the torch statement of the same gradient step;
the phases of one synchronised eager run; and captured steady-state env-steps/s of the trainer on KukaButton -c and MobileRobot -c, over a
window of graph replays, in runs alternating with DQN on the same envs (discrete).  The card line is nvidia-smi's name, power limit and
maximum SM clock; the SM clock observed while the kernels are timed is sampled separately.

    python scripts/sac_timing.py [--out profiles/r10_sac_timing.json] [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


class ClockSampler(object):
    """The SM clock read through NVML every 10 ms while the kernels are timed (min, median, max MHz)."""

    def __init__(self):
        import threading
        import pynvml
        pynvml.nvmlInit()
        self.nvml, self.h = pynvml, pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        self.samples, self.stop = [], threading.Event()
        self.thread = threading.Thread(target=self._loop, daemon=True)

    def _loop(self):
        while not self.stop.is_set():
            self.samples.append(self.nvml.nvmlDeviceGetClockInfo(self.h, self.nvml.NVML_CLOCK_SM))
            time.sleep(0.01)

    def __enter__(self):
        self.thread.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.thread.join()

    def summary(self):
        s = sorted(self.samples)
        return dict(min=s[0], median=s[len(s) // 2], max=s[-1], samples=len(s)) if s else None


def event_ms(fn, reps, flush):
    """Median CUDA-event time of fn() over reps launches, each after writing a 100 MB buffer (the L2 flush)."""
    times = []
    for _ in range(reps):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    times.sort()
    return times[len(times) // 2]


def kernels(reps):
    from rl_baselines.offpolicy import ring_bytes
    from rl_baselines.sac import SACNets, adam_polyak, sac_losses
    from srl_sim._abi import load_cuda_library
    from srl_sim.policy import FusedSACAct, FusedSACAdam, FusedSACGrad, FusedSACPrepare, FusedSACStore
    lib = load_cuda_library()
    W, A, N, rows = 3, 3, 4096, 50000
    B = 64 * N
    torch.manual_seed(0)
    nets = SACNets(W, A).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    ring = dict(obs=torch.randn(rows, N, W, device="cuda", generator=g), next_obs=torch.randn(rows, N, W, device="cuda", generator=g),
                act=torch.rand(rows, N, A, device="cuda", generator=g) * 2 - 1, rew=torch.randn(rows, N, device="cuda", generator=g),
                done=(torch.rand(rows, N, device="cuda", generator=g) < 0.01).to(torch.uint8))
    flush = torch.empty(25 << 20, device="cuda")
    grad = torch.zeros_like(nets.arena.detach())
    act = FusedSACAct(lib, nets, seed=1)
    store = FusedSACStore(lib, ring, "cuda")
    store.step[0] = rows
    ws = FusedSACGrad.workspace(lib, nets, B)
    prep = FusedSACPrepare(lib, nets, ring, B, 2, grad, ws)
    fgrad, fadam = FusedSACGrad(lib, nets), FusedSACAdam(lib, nets)
    fadam.lr.fill_(3e-4)
    obs, a_out, new_obs = torch.randn(N, W, device="cuda"), torch.zeros(N, A, device="cuda"), torch.randn(N, W, device="cuda")
    rew, done = torch.zeros(N, device="cuda"), torch.zeros(N, dtype=torch.uint8, device="cuda")
    res = dict(W=W, A=A, N=N, B=B, rows=rows, ring_gb=ring_bytes(rows, N, W, A) / 1e9, reps=reps, statistic="median of reps launches")
    res["act_ms"] = event_ms(lambda: act(N, obs, a_out), reps, flush)
    res["store_ms"] = event_ms(lambda: store(obs, a_out, rew, done, new_obs), reps, flush)
    res["prepare_ms"] = event_ms(lambda: prep(store.step, 0.99, None, -3.0), reps, flush)
    res["grad_ms"] = event_ms(lambda: fgrad(prep, grad), reps, flush)
    res["adam_ms"] = event_ms(lambda: fadam(grad), reps, flush)
    res["gradient_step_ms"] = res["prepare_ms"] + res["grad_ms"] + res["adam_ms"]
    # multiply-adds of one sample: forward of vf_targ, actor, qf1, qf2 and qf1's input gradient (prepare); forward + backward of four
    # networks (grad: forward recomputed, then the deltas and the weight gradients, about three times the forward)
    fwd = lambda n_in, n_out: 64 * n_in + 64 * 64 + 64 * n_out
    prep_macs = fwd(W, 1) + fwd(W, 2 * A) + 2 * fwd(W + A, 1) + 64 * 64 + 64 * A
    grad_macs = 3 * (fwd(W, 2 * A) + 2 * fwd(W + A, 1) + fwd(W, 1))
    res["macs_per_sample"] = prep_macs + grad_macs
    flop = 2.0 * res["macs_per_sample"] * B
    res["gflop_per_step"] = flop / 1e9
    res["fp32_bound_ms_at_67_tflops"] = flop / 67e12 * 1e3
    res["share_of_fp32_bound"] = res["fp32_bound_ms_at_67_tflops"] / (res["prepare_ms"] + res["grad_ms"])
    # the torch statement of the same step
    m, v, bp = torch.zeros_like(grad), torch.zeros_like(grad), torch.tensor([0.9, 0.999], device="cuda")
    flat = {k: x.reshape((rows * N,) + x.shape[2:]) for k, x in ring.items()}

    def torch_step():
        ix = torch.randint(0, rows * N, (B,), device="cuda")
        eps = torch.randn(B, A, device="cuda")
        L = sac_losses(nets, flat["obs"][ix], flat["act"][ix], flat["rew"][ix], flat["next_obs"][ix], flat["done"][ix].float(), eps, 0.99, None, -3.0)
        gr = torch.autograd.grad(L["total"], nets.arena)[0]
        adam_polyak(nets, gr, m, v, bp, 3e-4, 0.005, True)
    torch_step()
    res["torch_gradient_step_ms"] = event_ms(torch_step, max(3, reps // 4), flush)
    del ring, flat
    torch.cuda.empty_cache()
    return res


def trainer_rates(n_runs):
    """Captured steady state at 4096 envs with the defaults: SAC over lockstep steps 300-700 (one graph, replayed every block after step
    ~102), DQN over 1600-2600 (its 250 per-phase graphs all captured by step 1000); the runs alternate."""
    from rl_baselines import deepq, sac
    out = dict(sac_kuka=[], sac_mobile=[], dqn_kuka=[], dqn_mobile=[])
    for _ in range(n_runs):
        for name, mod, env_id, disc, steps, first in (("sac_kuka", sac, "KukaButtonGymEnv-v0", False, 700, 300),
                                                      ("dqn_kuka", deepq, "KukaButtonGymEnv-v0", True, 2600, 1600),
                                                      ("sac_mobile", sac, "MobileRobotGymEnv-v0", False, 700, 300),
                                                      ("dqn_mobile", deepq, "MobileRobotGymEnv-v0", True, 2600, 1600)):
            hist = mod.train(env_id, 4096, 4096 * steps, seed=0, env_kwargs=dict(is_discrete=disc), verbose=0)
            assert mod.train.stats["graph_replays"] > 0
            s = [h[0] for h in hist]
            lo = next(i for i, x in enumerate(s) if x >= first * 4096)
            (s0, _, f0), (s1, _, f1) = hist[lo], hist[-1]
            out[name].append((s1 - s0) / (s1 / f1 - s0 / f0))
            torch.cuda.empty_cache()
    return out


def phases():
    from rl_baselines import sac
    ph = {}
    sac.train("KukaButtonGymEnv-v0", 4096, 4096 * 130, seed=0, env_kwargs=dict(is_discrete=False), verbose=0, phase_times=ph)
    return ph


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=os.path.join(ROOT, "profiles", "r10_sac_timing.json"))
    p.add_argument("--reps", type=int, default=20)
    p.add_argument("--runs", type=int, default=2)
    args = p.parse_args()
    assert torch.cuda.is_available(), "sac_timing measures on a GPU"
    with ClockSampler() as clocks:
        k = kernels(args.reps)
    k["sm_clock_mhz_while_timed"] = clocks.summary()
    res = dict(card=card(), kernels=k, eager_phases_s=phases(), captured_env_steps_per_s=trainer_rates(args.runs))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
