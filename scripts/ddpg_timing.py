"""
DDPG timing on one GPU (profiles/r11_ddpg_timing.json): the card and its power limit, read in the same run; CUDA-event times of each DDPG
kernel at N = 4096 envs and B = 64 N = 262 144 samples over the default 100-row ring, each launch after an L2 flush; the FLOP count of a
gradient step from the shapes and its share of the 67 TFLOP/s FP32 data-sheet bound; and captured steady-state env-steps/s of the trainer on
KukaButton -c and MobileRobot -c, over a window of graph replays, in runs alternating with SAC on the same envs.

    python scripts/ddpg_timing.py [--out profiles/r11_ddpg_timing.json] [--reps 20] [--runs 2]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from sac_timing import ClockSampler, card, event_ms  # noqa: E402


def kernels(reps):
    from rl_baselines.ddpg import DDPGNets
    from rl_baselines.offpolicy import ring_bytes
    from srl_sim._abi import load_cuda_library
    from srl_sim.policy import FusedDDPGAct, FusedDDPGAdam, FusedDDPGGrad, FusedDDPGPrepare, FusedSACStore
    lib = load_cuda_library()
    W, A, N, rows = 3, 3, 4096, 100
    B = 64 * N
    torch.manual_seed(0)
    nets = DDPGNets(W, A).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    ring = dict(obs=torch.randn(rows, N, W, device="cuda", generator=g), next_obs=torch.randn(rows, N, W, device="cuda", generator=g),
                act=torch.rand(rows, N, A, device="cuda", generator=g) * 2 - 1, rew=torch.randn(rows, N, device="cuda", generator=g),
                done=(torch.rand(rows, N, device="cuda", generator=g) < 0.01).to(torch.uint8))
    flush = torch.empty(25 << 20, device="cuda")
    grad = torch.zeros_like(nets.arena.detach())
    act = FusedDDPGAct(lib, nets, N, seed=1, sigma=0.2)
    store = FusedSACStore(lib, ring, "cuda")
    store.step[0] = rows
    prep = FusedDDPGPrepare(lib, nets, ring, B, 2)
    fgrad, fadam = FusedDDPGGrad(lib, nets, B, 1e-2), FusedDDPGAdam(lib, nets, 1e-4, 1e-3, 1e-3)
    obs, a_out, new_obs = torch.randn(N, W, device="cuda"), torch.zeros(N, A, device="cuda"), torch.randn(N, W, device="cuda")
    rew, done = torch.zeros(N, device="cuda"), torch.zeros(N, dtype=torch.uint8, device="cuda")
    res = dict(W=W, A=A, N=N, B=B, rows=rows, ring_gb=ring_bytes(rows, N, W, A) / 1e9, reps=reps, statistic="median of reps launches")
    res["act_ou_ms"] = event_ms(lambda: act(N, obs, done, a_out, mode=FusedDDPGAct.OU), reps, flush)
    res["store_ms"] = event_ms(lambda: store(obs, a_out, rew, done, new_obs), reps, flush)
    res["prepare_ms"] = event_ms(lambda: prep(store.step, 0.99, 1.0), reps, flush)
    res["grad_ms"] = event_ms(lambda: fgrad(prep, grad), reps, flush)
    res["adam_ms"] = event_ms(lambda: fadam(grad), reps, flush)
    res["gradient_step_ms"] = res["prepare_ms"] + res["grad_ms"] + res["adam_ms"]
    # multiply-adds of one sample.  prepare: target actor and target critic at s', actor and critic at s, and dQ/da (64 A).  grad: forward
    # and backward of the actor and of the critic (forward recomputed, then the deltas and the weight gradients, about three times the forward)
    actor, critic = 64 * W + 64 * 64 + 64 * A, 64 * W + 64 * (64 + A) + 64
    prep_macs = 2 * actor + 2 * critic + 64 * A
    grad_macs = 3 * (actor + critic)
    res["macs_per_sample"] = prep_macs + grad_macs
    flop = 2.0 * res["macs_per_sample"] * B
    res["gflop_per_step"] = flop / 1e9
    res["fp32_bound_ms_at_67_tflops"] = flop / 67e12 * 1e3
    res["share_of_fp32_bound"] = res["fp32_bound_ms_at_67_tflops"] / (res["prepare_ms"] + res["grad_ms"])
    del ring
    torch.cuda.empty_cache()
    return res


def trainer_rates(n_runs):
    """Captured steady state at 4096 envs with the defaults: DDPG over lockstep steps 300-700 (one graph per 100-step cycle, replayed from
    the second cycle on), SAC over 300-700 (one graph per block after step ~102); the runs alternate."""
    from rl_baselines import ddpg, sac
    out = dict(ddpg_kuka=[], ddpg_mobile=[], sac_kuka=[], sac_mobile=[])
    for _ in range(n_runs):
        for name, mod, env_id in (("ddpg_kuka", ddpg, "KukaButtonGymEnv-v0"), ("sac_kuka", sac, "KukaButtonGymEnv-v0"),
                                  ("ddpg_mobile", ddpg, "MobileRobotGymEnv-v0"), ("sac_mobile", sac, "MobileRobotGymEnv-v0")):
            hist = mod.train(env_id, 4096, 4096 * 700, seed=0, env_kwargs=dict(is_discrete=False), verbose=0)
            assert mod.train.stats["graph_replays"] > 0
            s = [h[0] for h in hist]
            lo = next(i for i, x in enumerate(s) if x >= 300 * 4096)
            (s0, _, f0), (s1, _, f1) = hist[lo], hist[-1]
            out[name].append((s1 - s0) / (s1 / f1 - s0 / f0))
            mod.train.last_ring = mod.train.last_nets = mod.train.last_fused = None
            torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=os.path.join(ROOT, "profiles", "r11_ddpg_timing.json"))
    p.add_argument("--reps", type=int, default=20)
    p.add_argument("--runs", type=int, default=2)
    args = p.parse_args()
    assert torch.cuda.is_available(), "ddpg_timing measures on a GPU"
    with ClockSampler() as clocks:
        k = kernels(args.reps)
    k["sm_clock_mhz_while_timed"] = clocks.summary()
    res = dict(card=card(), kernels=k, captured_env_steps_per_s=trainer_rates(args.runs))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
