"""
One gradient step of the fused DQN trainer (rl_baselines.deepq.train on the GPU), rebuilt in float64 from the state the run leaves behind.

With learning_starts 32, train_freq 4 and num_timesteps = 37 N, the run's only gradient step is at its last lockstep step, t = 36, and the
target network is never copied.  At that step the ring is the final ring, the online network still equals the target network
(train.last_target), every stored leaf is 1^alpha = 1 and the Adam slots are zero.  So tests/deepq_numpy_ref.py can redo the whole step: the
samples from the replay's own Philox uniforms, y, td and the gradient, the per-tensor clip and one TF Adam step, and the priorities written
back.  That checks the chain srl_replay_sample -> srl_dqn_target -> srl_dqn_grad -> srl_clip_adam -> srl_replay_update as the trainer wires it
(which rows and columns of the ring each kernel reads, gamma, done, the Adam constants), not each kernel alone; and the ring the 37 collection
steps wrote (srl_dqn_act, the filter, srl_replay_add).

Cases: MobileRobot at 8192 envs with the default ring of 1000 rows (8 192 000 transitions, 2^23 leaves: the three-pass tree rebuild inside the
trainer), KukaButton at 4096 envs, and KukaButton with a stack of 4 (width 12: the wide act, target and gradient kernels); prioritized replay
on and off.
"""
import copy

import numpy as np
import pytest
import torch

from deepq_numpy_ref import dqn_forward_model, dqn_step_model, first_sample_model
from test_consumer_reference_cpu import grad_bound, grad_errors
from test_deepq_gpu import PURPOSE_ACT, PURPOSE_REPLAY, philox_u53  # noqa: F401  (philox_u53: the fixture)

pytestmark = pytest.mark.gpu

T, SEED = 37, 7                 # lockstep steps of a run; the gradient step is at t = T - 1
HP = dict(learning_starts=32, train_freq=4, batch_size=32, target_network_update_freq=10 ** 6, buffer_size=1000)
RUNS = [("MobileRobotGymEnv-v0", 8192, 1, dict(is_discrete=True, shape_reward=True)), ("KukaButtonGymEnv-v0", 4096, 1, dict(is_discrete=True)),
        ("KukaButtonGymEnv-v0", 4096, 4, dict(is_discrete=True))]
PARAMS = [(r, p) for r in RUNS for p in (True, False)]
IDS = ["%s_%d_stack%d-%s" % (r[0].split("GymEnv")[0], r[1], r[2], "prioritized" if p else "uniform") for r, p in PARAMS]


@pytest.fixture(scope="module", params=PARAMS, ids=IDS)
def run(request, cuda_lib):
    (env_id, N, K, env_kwargs), prioritized = request.param
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.deepq import train
    hp = dict(HP, prioritized_replay=prioritized)
    train(env_id, N, T * N, seed=SEED, env_kwargs=env_kwargs, verbose=0, hyperparams=hp, num_stack=K)
    assert train.stats["grad_steps"] == 1 and train.stats["target_copies"] == 0, train.stats
    rep, (m, v, beta_power) = train.last_replay, train.last_adam
    net = train.last_policy
    return dict(N=N, K=K, prioritized=prioritized,
                ring={k: t[:T].cpu().numpy() for k, t in train.last_ring.items()},
                before=copy.deepcopy(train.last_target).cpu(),                 # the online network before the step
                after=[p.detach().cpu().double().numpy() for p in net.parameters()],
                grad=[p.grad.detach().cpu().double().numpy() for p in net.parameters()],
                m=[t.cpu().double().numpy() for t in m], v=[t.cpu().double().numpy() for t in v], beta_power=beta_power.cpu().numpy(),
                tree_cap=rep.tree_cap, sum=rep.sum.cpu().numpy(), min=rep.min.cpu().numpy(), max_priority=float(rep.max_priority),
                size=int(rep.size))


def _f32(x):
    return float(np.float32(x))


def test_gradient_step_matches_float64(run, philox_u53):
    from rl_baselines.deepq import ADAM_BETA1, ADAM_BETA2, ADAM_EPS, DQN_DEFAULTS, GRAD_CLIP_NORM, dqn_loss
    N, ring, net = run["N"], run["ring"], run["before"]
    B, n, cap = HP["batch_size"] * N, T * N, run["tree_cap"]
    assert run["size"] == n
    if N == 8192:
        assert cap == 2 ** 23                                    # three passes of srl_replay_add / _update's rebuild
    # the first batch: uniforms from seed + 1 (rank 0), stream b, counter 0; leaf i is ring row i // N, env i % N: the ring's flat layout
    u, _ = philox_u53(SEED + 1, range(B), 0, PURPOSE_REPLAY)
    idx, near = first_sample_model(u, n, cap, run["prioritized"])
    flat = {k: a.reshape((n,) + a.shape[2:]) for k, a in ring.items()}
    lr, b1, b2, eps = _f32(DQN_DEFAULTS["learning_rate"]), _f32(ADAM_BETA1), _f32(ADAM_BETA2), _f32(ADAM_EPS)
    model = dqn_step_model(net, flat["obs"][idx], flat["act"][idx], flat["rew"][idx], flat["done"][idx], flat["next_obs"][idx],
                           _f32(DQN_DEFAULTS["gamma"]), lr, GRAD_CLIP_NORM, b1, b2, eps)
    # float32 autograd's own error on the same rows.  The rows are the simulator's, not drawn away from the ReLU kinks: a pre-activation
    # within rounding of 0 flips one sample's term between float32 and float64, and at B = 32 N one sample's term (at most 1 / B of a
    # weighted, clipped td times an activation) is far below the tolerance; so is one index taken on the other side of a float64 boundary.
    q32 = copy.deepcopy(net).requires_grad_(True)                # a copy of the target network, which the trainer keeps without gradients
    loss, _ = dqn_loss(q32, torch.from_numpy(flat["obs"][idx]), torch.from_numpy(flat["act"][idx]), torch.from_numpy(model["y"]).float(),
                       torch.ones(B))
    loss.backward()
    g64 = [torch.from_numpy(g) for g in model["grads"]]
    e32 = grad_errors([p.grad.cpu() for p in q32.parameters()], g64)
    kern = grad_errors([torch.from_numpy(g) for g in run["grad"]], g64)
    r1, r2 = 1.0 - b1, 1.0 - b2                                  # exact in float32: the kernel's 1 - beta
    lr_t = lr * np.sqrt(r2) / r1
    move = lambda g: lr_t * (r1 * g) / (np.sqrt(r2 * g * g) + eps)        # the first Adam step of a clipped gradient g
    names = [k for k, _ in net.named_parameters()]
    print("\nB=%d  max|g - g64| / max|g64|  kernel | float32 autograd:" % B)
    for k, name in enumerate(names):
        (err, scale), (err32, _) = kern[k], e32[k]
        bound = grad_bound(scale) + 4.0 * err32
        print("  %s %.1e|%.1e" % (name, err / scale, err32 / scale), end="")
        assert scale > 0 and err <= bound, (name, err, err32, scale)
        # m = (1 - beta1) g_clipped: the float64 clipped gradient within the gradient's bound, carried through the clip factor
        c64 = model["clip_scale"][k]
        nk = np.sqrt((run["grad"][k] ** 2).sum())
        dc = abs(GRAD_CLIP_NORM / max(nk, GRAD_CLIP_NORM) - c64)
        gc = c64 * model["grads"][k]
        e = c64 * bound + dc * scale + 4e-7 * c64 * scale
        assert np.abs(run["m"][k] / r1 - gc).max() <= e, (name, np.abs(run["m"][k] / r1 - gc).max(), e)
        assert np.allclose(model["m"][k], r1 * gc, rtol=1e-12, atol=0)
        # v = (1 - beta2) g_clipped^2 under the same bound
        assert np.all(np.abs(run["v"][k] / r2 - gc * gc) <= e * (2.0 * np.abs(gc) + e) + 4e-7 * gc * gc), name
        # the parameters moved by one Adam step (about lr sign(g)): the model's move where the sign of g is clear of the bound, at most lr
        # elsewhere; plus the float32 rounding of the parameter
        p0, p1 = model["params"][k], run["after"][k]
        got, ulp = p0 - p1, np.spacing(np.abs(p0).astype(np.float32)).astype(np.float64)
        clear = np.abs(gc) > e
        assert np.allclose(model["new_params"][k], p0 - move(gc), rtol=0, atol=1e-12)
        spread = np.maximum(np.abs(move(gc + e) - move(gc)), np.abs(move(gc - e) - move(gc)))
        assert np.all(np.abs(got - move(gc))[clear] <= spread[clear] + ulp[clear] + 1e-6 * lr), name
        assert np.all(np.abs(got) <= lr * (1.0 + 1e-6) + ulp), name
        assert clear.mean() > 0.25, (name, clear.mean())           # most entries are compared with the model, not only bounded
    print()
    # exactly one Adam step: TF's beta powers advanced once
    assert np.array_equal(run["beta_power"], np.array([np.float32(b1) * np.float32(b1), np.float32(b2) * np.float32(b2)], np.float32))

    s, mn = run["sum"], run["min"]
    k = np.arange(1, cap)
    assert np.array_equal(s[k], s[2 * k] + s[2 * k + 1]) and np.array_equal(mn[k], np.minimum(mn[2 * k], mn[2 * k + 1]))
    assert np.all(s[cap + n:] == 0.0) and np.all(np.isinf(mn[cap + n:]))
    leaves = s[cap:cap + n]
    assert np.array_equal(leaves, mn[cap:cap + n])
    if not run["prioritized"]:                                   # uniform replay: the gradient step leaves the trees as the adds made them
        assert np.all(leaves == 1.0) and run["max_priority"] == 1.0 and s[1] == float(n)
        return
    # priorities (|td| + 1e-6)^0.6 at the sampled leaves, within the float32 rounding of td; for a sample on a float64 boundary, either leaf
    td64, alpha, peps = model["td"], DQN_DEFAULTS["prioritized_replay_alpha"], DQN_DEFAULTS["prioritized_replay_eps"]
    tol = 2e-5 * (np.abs(td64).max() + 1.0)
    alt = np.clip(np.where(u * n - np.round(u * n) >= 0, idx - 1, idx + 1), 0, n - 1)
    if near.any():
        td_alt = dqn_step_model(net, flat["obs"][alt[near]], flat["act"][alt[near]], flat["rew"][alt[near]], flat["done"][alt[near]],
                                flat["next_obs"][alt[near]], _f32(DQN_DEFAULTS["gamma"]), lr, GRAD_CLIP_NORM, b1, b2, eps)["td"]
    else:
        td_alt = np.zeros(0)
    cand = np.concatenate([idx, alt[near]])
    ctd = np.abs(np.concatenate([td64, td_alt]))
    lo = (np.maximum(ctd - tol, 0.0) + peps) ** alpha * (1.0 - 1e-12)
    hi = (ctd + tol + peps) ** alpha * (1.0 + 1e-12)
    order = np.argsort(cand, kind="stable")
    uniq, start = np.unique(cand[order], return_index=True)
    lo_u, hi_u = np.minimum.reduceat(lo[order], start), np.maximum.reduceat(hi[order], start)
    written = np.nonzero(leaves != 1.0)[0]
    assert np.all(np.isin(written, uniq)), np.setdiff1d(written, uniq)[:10]        # nothing but sampled leaves changed
    sure = idx[~near][(lo[:B][~near] > 1.0) | (hi[:B][~near] < 1.0)]
    assert np.all(np.isin(sure, written)), np.setdiff1d(sure, written)[:10]      # and every sampled leaf did
    at = np.searchsorted(uniq, written)
    assert np.all((leaves[written] >= lo_u[at]) & (leaves[written] <= hi_u[at]))
    p_lo, p_hi = np.maximum(np.abs(td64[~near]) - tol, 0.0) + peps, ctd + tol + peps
    assert max(1.0, p_lo.max()) * (1.0 - 1e-7) <= run["max_priority"] <= max(1.0, p_hi.max()) * (1.0 + 1e-7)
    print("  %d samples, %d distinct leaves written, %d on a float64 boundary" % (B, len(written), int(near.sum())))


def test_ring_holds_the_collected_steps(run, philox_u53):
    """obs[t + 1] is next_obs[t] byte for byte; the envs whose Philox word says explore hold the uniform action of word 2, the rest the
    greedy action of the network before the step (a float64 forward), except where its top two Q values are within float32 rounding."""
    from rl_baselines.deepq import DQN_DEFAULTS, linear_schedule
    N, ring, net = run["N"], run["ring"], run["before"]
    assert np.array_equal(ring["obs"][1:].view(np.uint32), ring["next_obs"][:-1].view(np.uint32))
    A = net.n_actions
    explore_steps = int(DQN_DEFAULTS["exploration_fraction"] * T)
    greedy_checked = 0
    for t in range(T):
        eps = np.float32(linear_schedule(explore_steps, 1.0, DQN_DEFAULTS["exploration_final_eps"], t))
        u, w2 = philox_u53(SEED, range(N), t, PURPOSE_ACT)
        explore = u < float(eps)
        act = ring["act"][t]
        assert np.array_equal(act[explore], ((w2[explore] * np.uint64(A)) >> np.uint64(32)).astype(np.int64)), t
        q = dqn_forward_model(net, ring["obs"][t])
        top2 = np.sort(q, 1)[:, -2:]
        clear = ~explore & (top2[:, 1] - top2[:, 0] > 2e-5 * (np.abs(q).max() + 1.0))
        assert np.array_equal(act[clear], q.argmax(1)[clear]), t
        greedy_checked += int(clear.sum())
    assert greedy_checked > 0.9 * (T - explore_steps) * N
