"""
DQN timings on one GPU, in one process: the card and its power limit; CUDA-event times of every DQN kernel at 4096 envs, a 1000-row ring
(4 096 000 transitions, 2^22 leaves) and B = 131 072 samples, each launch after an L2 flush; the torch statement of the same gradient step
(target, autograd of the loss, clip + Adam on the GPU, the numpy trees on the host); one eager gradient block split into collection / replay /
gradient / optimiser (synchronised between the phases); and captured env-steps/s of DQN on KukaButton and MobileRobot in runs alternating
with A2C.

    python scripts/deepq_timing.py [--out FILE]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from a2c_timing import a2c_run, card, flushed_event_ms, steady_rate  # noqa: E402

N, ROWS, W, A = 4096, 1000, 3, 6
B = 32 * N


def kernels(lib):
    from rl_baselines.deepq import DuelingQ, ReplayTree, clip_adam, double_q_target, dqn_loss
    from srl_sim.policy import FusedClipAdam, FusedDQNAct, FusedDQNGrad, FusedDQNTarget, FusedReplay
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    q, tq = DuelingQ(W, A).to(dev), DuelingQ(W, A).to(dev)
    st = torch.cuda.current_stream().cuda_stream
    obs_ring, next_ring = torch.randn(ROWS * N, W, device=dev), torch.randn(ROWS * N, W, device=dev)
    act_ring, rew_ring = torch.randint(0, A, (ROWS * N,), device=dev), torch.randn(ROWS * N, device=dev)
    done_ring = (torch.rand(ROWS * N, device=dev) < 0.01).to(torch.uint8)
    rep = FusedReplay(lib, ROWS, N, 1, 0.6, dev)
    for r in range(ROWS):
        rep.add(r, stream=st)
    rep.beta.fill_(0.4)
    idx, w, y, td = torch.zeros(B, dtype=torch.int64, device=dev), torch.zeros(B, device=dev), torch.zeros(B, device=dev), torch.zeros(B, device=dev)
    fact, ftarget, fgrad = FusedDQNAct(lib, q, seed=0), FusedDQNTarget(lib, q, tq), FusedDQNGrad(lib, q, B)
    fopt = FusedClipAdam(lib, q, 10.0)
    fopt.lr.fill_(1e-12)
    act = torch.zeros(N, dtype=torch.int32, device=dev)
    o = torch.randn(N, W, device=dev)
    r = dict(num_envs=N, ring_rows=ROWS, transitions=ROWS * N, tree_leaves=rep.tree_cap, batch=B)
    r["srl_dqn_act_ms"] = flushed_event_ms(lambda: fact(N, o, act, stream=st))
    r["srl_replay_add_ms"] = flushed_event_ms(lambda: rep.add(7, stream=st))
    r["srl_replay_sample_ms"] = flushed_event_ms(lambda: rep.sample(B, idx, w, stream=st))
    r["srl_dqn_target_ms"] = flushed_event_ms(lambda: ftarget(B, idx, next_ring, rew_ring, done_ring, 0.99, y, stream=st))
    r["srl_dqn_grad_ms"] = flushed_event_ms(lambda: fgrad(idx, obs_ring, act_ring, y, w, td, stream=st))
    r["srl_clip_adam_ms"] = flushed_event_ms(lambda: fopt(stream=st))
    td.copy_(torch.randn(B, device=dev))
    r["srl_replay_update_ms"] = flushed_event_ms(lambda: rep.update(B, idx, td, 1e-6, stream=st))
    r["srl_replay_update_note"] = "stamp + priority scatter + the full bottom-up rebuild of both 2^22-leaf trees (two rebuild launches)"
    r["fused_gradient_step_ms"] = r["srl_replay_sample_ms"] + r["srl_dqn_target_ms"] + r["srl_dqn_grad_ms"] + r["srl_clip_adam_ms"] + r["srl_replay_update_ms"]
    # the torch statement of the same gradient step: the torch network on the GPU, the trees in numpy on the host
    tree = ReplayTree(ROWS, N, 0.6)
    for row in range(ROWS):
        tree.add(row)
    params = list(q.parameters())
    m, v = [torch.zeros_like(p) for p in params], [torch.zeros_like(p) for p in params]
    bp = torch.tensor([0.9, 0.999], device=dev)
    ix_t, w_t = idx.clone(), w.clone()

    def torch_gpu_part():
        yy = double_q_target(q, tq, rew_ring[ix_t], done_ring[ix_t].float(), next_ring[ix_t], 0.99)
        for p in params:
            p.grad = None
        loss, _ = dqn_loss(q, obs_ring[ix_t], act_ring[ix_t], yy, w_t)
        loss.backward()
        clip_adam(params, m, v, bp, 1e-12, 10.0, 0.9, 0.999, 1e-8)
    r["torch_target_autograd_clip_adam_ms"] = flushed_event_ms(torch_gpu_part, iters=50, warmup=5)
    u = np.random.RandomState(0).rand(B)
    times = []
    for _ in range(5):
        t0 = time.perf_counter()
        ix, _ = tree.sample(u, 0.4)
        tree.update(ix, td.cpu().numpy(), 1e-6)
        times.append(1e3 * (time.perf_counter() - t0))
    r["numpy_tree_sample_update_ms"] = sorted(times)[2]
    r["torch_statement_gradient_step_ms"] = r["torch_target_autograd_clip_adam_ms"] + r["numpy_tree_sample_update_ms"]
    return r


def phases(env_id="KukaButtonGymEnv-v0"):
    from rl_baselines.deepq import train
    pt = {}
    n = 600
    train(env_id, N, N * n, seed=0, env_kwargs=dict(is_discrete=True), verbose=0, phase_times=pt)
    grads = train.stats["grad_steps"]
    out = dict(env=env_id, lockstep_steps=n, gradient_steps=grads, collect_ms_per_lockstep_step=1e3 * pt["collect"] / n)
    out.update({k + "_ms_per_gradient_step": 1e3 * pt[k] / grads for k in ("replay", "gradient", "optimise")})
    return out


def dqn_run(env_id, n=2600):
    """Defaults (learning_starts 500, train_freq 4, ring of 1000 rows: 250 graphs); the rate over steps 1600..n, after every phase's capture."""
    from rl_baselines.deepq import train
    hist = train(env_id, N, N * n, seed=0, env_kwargs=dict(is_discrete=True, shape_reward=env_id.startswith("Mobile")), verbose=0)
    return dict(algo="deepq", env=env_id, lockstep_steps=n, env_steps_per_s=steady_rate(hist, 1600 // 4), stats=train.stats,
                last_mean_return=hist[-1][1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r09_deepq_timing.json"))
    args = ap.parse_args()
    from srl_sim._abi import load_cuda_library
    lib = load_cuda_library()
    res = dict(card=card())
    res["kernels"] = kernels(lib)
    res["eager_block_phases_synchronised"] = phases()
    res["alternating_runs"] = [dqn_run("KukaButtonGymEnv-v0"), a2c_run(), dqn_run("MobileRobotGymEnv-v0"), dqn_run("KukaButtonGymEnv-v0"), a2c_run(),
                               dqn_run("MobileRobotGymEnv-v0")]
    print(json.dumps(res, indent=1))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
