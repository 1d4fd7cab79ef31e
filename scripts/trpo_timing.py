"""
TRPO timing on one GPU (profiles/r12_trpo_timing.json): the card and its power limit, read in the same run; CUDA-event times of each TRPO entry
point at KukaButton's shape (obs_dim 3, 6 actions) with N = 4096 envs and T = 128 (524 288 rows, the FVP on the 106 496-row subsample), the
median of --reps launches each after an L2 flush; the FLOP count of each from the shapes and its share of the 67 TFLOP/s FP32 data-sheet
bound; the whole update's launches (surrogate, cg_iters + 1 products, ten trials, three value steps) back to back; the torch statement of the
same update (rl_baselines.trpo.policy_step_torch + value_steps_torch) on the same GPU; and captured steady-state env-steps/s of the trainer on
KukaButton at 4096 envs, in runs alternating with PPO2.

    python scripts/trpo_timing.py [--out profiles/r12_trpo_timing.json] [--reps 200] [--runs 2] [--updates 12]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from sac_timing import ClockSampler, card, event_ms  # noqa: E402

FP32_TFLOPS = 67.0          # H100 SXM data sheet, dense FP32


def fwd_flop(D, A):
    """Multiply-adds x 2 of one tower's forward pass for one row."""
    return 2 * (64 * D + 64 * 64 + 64 * A)


def kernels(reps):
    from rl_baselines.ppo2 import MlpPolicy
    from rl_baselines.trpo import TRPO_DEFAULTS
    from srl_sim._abi import load_cuda_library
    from srl_sim.policy import FusedTRPO
    lib = load_cuda_library()
    D, A, N, T = 3, 6, 4096, 128
    rows, sub = T * N, ((T + 4) // 5) * N
    hp = TRPO_DEFAULTS
    torch.manual_seed(0)
    pol = MlpPolicy(D, n_actions=A).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    obs = torch.randn(rows, D, device="cuda", generator=g)
    act = torch.randint(0, A, (rows,), device="cuda", generator=g)
    adv = torch.randn(rows, device="cuda", generator=g)
    ret = torch.randn(rows, device="cuda", generator=g)
    vidx = torch.randperm(rows, device="cuda")
    flush = torch.empty(64 << 20, device="cuda")         # 256 MB
    f = FusedTRPO(lib, pol, rows)
    saved = [p.detach().clone() for p in pol.parameters()]
    f.surrogate(obs, act, adv, hp["entcoeff"])
    f.vector(0, hp["max_kl"], hp["entcoeff"])            # trials stay runnable: no trial decision is taken while they are timed
    f.fullstep.copy_(1e-3 * f.g)
    res = {}
    res["surrogate_ms"] = event_ms(lambda: f.surrogate(obs, act, adv, hp["entcoeff"]), reps, flush)
    res["fvp_ms"] = event_ms(lambda: f.fvp(sub, N, 5 * N, obs, f.p, hp["cg_damping"], f.z), reps, flush)
    res["trial_ms"] = event_ms(lambda: f.trial(obs, act), reps, flush)
    res["vf_grad_ms"] = event_ms(lambda: f.vf_grad(rows, vidx, obs, ret), reps, flush)
    res["vector_start_ms"] = event_ms(lambda: f.vector(0, hp["max_kl"], hp["entcoeff"]), reps, flush)
    res["vector_step_ms"] = event_ms(lambda: f.vector(2, hp["max_kl"], hp["entcoeff"]), reps, flush)
    res["vf_adam_ms"] = event_ms(lambda: f.vf_adam(hp["vf_stepsize"]), reps, flush)
    flop = dict(surrogate=3 * fwd_flop(D, A) * rows, fvp=5 * fwd_flop(D, A) * sub, trial=fwd_flop(D, A) * rows, vf_grad=3 * fwd_flop(D, 1) * rows)
    res["gflop"] = {k: v / 1e9 for k, v in flop.items()}
    res["share_of_fp32_bound"] = {k: (flop[k] / (FP32_TFLOPS * 1e12)) / (res[k + "_ms"] * 1e-3) for k in flop}

    def update():
        f.surrogate(obs, act, adv, hp["entcoeff"])
        f.vector(0, hp["max_kl"], hp["entcoeff"])
        for i in range(hp["cg_iters"] + 1):
            f.fvp(sub, N, 5 * N, obs, f.p if i < hp["cg_iters"] else f.x, hp["cg_damping"], f.z)
            f.vector(1 if i < hp["cg_iters"] else 2, hp["max_kl"], hp["entcoeff"])
        for _ in range(10):
            f.trial(obs, act)
            f.vector(3, hp["max_kl"], hp["entcoeff"])
        for _ in range(hp["vf_iters"]):
            f.vf_grad(rows, vidx, obs, ret)
            f.vf_adam(hp["vf_stepsize"])

    def restore():
        with torch.no_grad():
            for p, s in zip(pol.parameters(), saved):
                p.copy_(s)
    times = []
    for _ in range(20):
        restore()
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); update(); e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    res["update_kernels_ms"] = sorted(times)[len(times) // 2]
    res["update_trials_run"] = int(f.state[7].item())
    restore()
    res["torch_statement_ms"] = torch_statement(pol, obs, act, adv, ret, T, N, hp)
    return res


def torch_statement(pol, obs, act, adv, ret, T, N, hp, reps=5):
    """Wall time of the torch statement of the same update on the GPU (synchronised), the median of ``reps``."""
    from rl_baselines.trpo import flat, policy_step_torch, value_steps_torch, vf_minibatches, vf_params
    rows = T * N
    obs_sub = obs.reshape(T, N, -1)[::5].reshape(-1, obs.shape[1])
    saved = [p.detach().clone() for p in pol.parameters()]
    nv = flat(vf_params(pol)).numel()
    times = []
    for _ in range(reps):
        with torch.no_grad():
            for p, s in zip(pol.parameters(), saved):
                p.copy_(s)
        adam = (torch.zeros(nv, device="cuda"), torch.zeros(nv, device="cuda"), torch.zeros(1, dtype=torch.int64))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        policy_step_torch(pol, obs, act, adv, obs_sub, hp)
        value_steps_torch(pol, obs, ret, [torch.randperm(rows, device="cuda") for _ in range(hp["vf_iters"])], vf_minibatches(T, N), adam, hp)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return sorted(times)[len(times) // 2]


def trainer_rates(n_runs, updates):
    """Captured steady state at 4096 envs with the defaults on KukaButton (discrete): env-steps/s between the third and the last update,
    TRPO and PPO2 alternating."""
    from rl_baselines import ppo2, trpo
    out = dict(trpo_kuka=[], ppo2_kuka=[])
    N, T = 4096, 128
    for _ in range(n_runs):
        for name, mod in (("trpo_kuka", trpo), ("ppo2_kuka", ppo2)):
            hist = mod.train("KukaButtonGymEnv-v0", N, N * T * updates, seed=0, env_kwargs=dict(is_discrete=True), verbose=0)
            (s0, _, f0), (s1, _, f1) = hist[2], hist[-1]
            out[name].append((s1 - s0) / (s1 / f1 - s0 / f0))
            mod.train.last_update = mod.train.last_policy = mod.train.last_norm = None
            torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default=os.path.join(ROOT, "profiles", "r12_trpo_timing.json"))
    p.add_argument("--reps", type=int, default=200)
    p.add_argument("--runs", type=int, default=2)
    p.add_argument("--updates", type=int, default=12)
    args = p.parse_args()
    assert torch.cuda.is_available(), "trpo_timing measures on a GPU"
    with ClockSampler() as clocks:
        k = kernels(args.reps)
    k["sm_clock_mhz_while_timed"] = clocks.summary()
    res = dict(card=card(), kernels=k, captured_env_steps_per_s=trainer_rates(args.runs, args.updates))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
