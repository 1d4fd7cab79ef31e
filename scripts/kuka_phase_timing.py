"""Where the time of the fused Kuka rollout goes, phase by phase.  Needs the -DKK_PHASES build (scripts/build_variant.sh phases -DKK_PHASES,
then SRL_SIM_CUDA_LIB=robotics-rl-srl_b200/csrc/libsrl_variant_phases.so): every env slot accumulates clock64() cycles per phase of the
micro-step loop and stores them at the end of the launch.

Workload = bench.py's headline: KukaButtonGymEnv-v0, 4096 envs, T = 128, bench seeds and inputs, 3 warm-up rollouts, then LAUNCHES measured
rollouts.  Per phase it prints cycles per physics step (median and max over slots), the phase's share of the slowest slot of each launch
(the slot that ends last bounds the launch), and the same for the whole slot.  The fast sweeps are split by the copy of the loop the
warp ran (quiet: no env of the warp watches a contact; watch), with the share of physics steps that ran the watch copy.  The phase clocks add a few registers (more spills) and
one clock read per mark, so the build runs a little slower than the shipped one: the split is the point, not the total."""
import argparse, os, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "robotics-rl-srl_b200"))
import torch
from srl_sim._abi import load_cuda_library
from srl_sim.backend import Backend
from srl_sim.model import load_kuka_scene

# KK_PH_* of kuka_coop.cuh, in order
PHASES = ["kin: local rotations", "kin: transform chain", "kin: body + candidates", "kin: collect + link states",
          "IK: J, error, J^T J, J^T e", "IK: 7x7 solve",
          "dyn D1 velocity terms", "dyn D2 velocity prefix", "dyn D3 acceleration terms", "dyn D4 acceleration prefix", "dyn D5 wrenches",
          "dyn D6 sub-tree sums", "dyn D7 mass rows (+ load M, bias)",
          "Cholesky + M^-1", "v0 + motor / limit set-up", "contact rows + scaling", "Euler",
          "fast sweeps, quiet copy", "fast sweeps, watch copy", "general loop", "env logic / loads / stores"]
NPH = len(PHASES)
FAST_QUIET, FAST_WATCH = PHASES.index("fast sweeps, quiet copy"), PHASES.index("fast sweeps, watch copy")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        print("device:", q.stdout.strip())
    except Exception as ex:  # noqa: BLE001 -- the table is still valid without the card line
        print("device: nvidia-smi unavailable (%r)" % (ex,))
    n, T = 4096, 128
    lib = load_cuda_library()
    be = Backend(lib, 0)
    st = be.stream()
    # bench.py's workload_spec("kuka") / make_inputs / measure_b200 at rank 0
    sim = be.make_sim("KukaButtonGymEnv-v0", n, seed=args.seed, model_blob=load_kuka_scene().blob,
                      is_discrete=True, random_target=False, force_down=True, action_repeat=1, max_distance=0.8)
    sim.reset(stream=st)
    rng = np.random.default_rng(args.seed)
    acts = be.from_host(rng.integers(0, 6, (T, n), dtype=np.int32))
    noise = be.from_host(rng.normal(0, 0.01, (T, n)).astype(np.float32))
    obs = be.zeros((T, n, 3), np.float32); rew = be.zeros((T, n), np.float32); done = be.zeros((T, n), np.uint8)
    ep_ret = be.zeros((T, n), np.float32); ep_len = be.zeros((T, n), np.int32)
    for _ in range(3):
        sim.rollout(T, acts, noise, obs, rew, done, ep_ret, ep_len, stream=st)
    torch.cuda.synchronize()
    words = np.zeros((1 << 13, NPH + 2), np.uint64)
    per_step = []          # [launch] -> (live slots, NPH) cycles per physics step
    slowest = []           # [launch] -> (NPH,) cycles of the slowest slot
    watch_share = []       # [launch] -> (live slots,) share of the slot's physics steps that ran the watch copy of the fast loop
    slowest_watch = []     # [launch] -> that share for the slowest slot
    ms = []
    for _ in range(args.launches):
        words[:] = 0
        sim.rollout(T, acts, noise, obs, rew, done, ep_ret, ep_len, stream=st)
        torch.cuda.synchronize()
        ms.append(sim.last_kernel_ms())
        rc = sim._lib.srl_sim_get_state(sim.handle, 98, words.ctypes.data, words.nbytes)
        assert rc == 0, "srl_sim_get_state(98) failed: not a -DKK_PHASES build?"
        w = words.astype(np.float64)
        live = w[:, NPH] > 0
        cyc, nphys, nwatch = w[live, :NPH], w[live, NPH], w[live, NPH + 1]
        per_step.append(cyc / nphys[:, None])
        k_slow = np.argmax(cyc.sum(axis=1))
        slowest.append(cyc[k_slow])
        watch_share.append(nwatch / nphys)
        slowest_watch.append(nwatch[k_slow] / nphys[k_slow])
    ps = np.concatenate(per_step)
    sl = np.mean(slowest, axis=0)
    print("KukaButtonGymEnv-v0, %d envs x T = %d, %d live slots, %d launches after 3 warm-ups: %s ms per launch (phase-clock build)"
          % (n, T, per_step[0].shape[0], args.launches, " ".join("%.3f" % x for x in ms)))
    print("%-38s %14s %14s %16s" % ("phase", "median cyc/step", "max cyc/step", "slowest slot %"))
    for k in range(NPH):
        print("%-38s %14.0f %14.0f %15.1f%%" % (PHASES[k], np.median(ps[:, k]), np.max(ps[:, k]), 100.0 * sl[k] / sl.sum()))
    tot = ps.sum(axis=1)
    print("%-38s %14.0f %14.0f %15.1f%%" % ("total", np.median(tot), np.max(tot), 100.0))
    print("slowest slot: %.0f cycles per launch = %.3f ms at 1.98 GHz" % (sl.sum(), sl.sum() / 1.98e6))
    ws = np.concatenate(watch_share)
    print("physics steps that ran the watch copy: slowest slot %.1f%% (mean over launches), median slot %.1f%%, all slots %.1f%%"
          % (100.0 * np.mean(slowest_watch), 100.0 * np.median(ws), 100.0 * np.mean(ws)))
    # fast-sweep cycles per physics step of each copy, over the steps that ran it (the table above averages over all steps)
    for name, k, share in (("quiet", FAST_QUIET, 1.0 - ws), ("watch", FAST_WATCH, ws)):
        per = ps[:, k] / np.maximum(share, 1e-12)
        per = per[share > 0]
        if per.size:
            print("fast sweeps, %s copy: median %.0f cycles per physics step that ran it (%d slots)" % (name, np.median(per), per.size))


if __name__ == "__main__":
    main()
