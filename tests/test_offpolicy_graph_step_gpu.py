"""
The SAC, DDPG and DQN trainers past their first gradient step: the last block of a run, a replayed CUDA graph on a ring that has wrapped,
rebuilt in float64.

After warm-up every gradient step of these trainers runs inside a replayed graph, with a target network that differs from the online one,
optimiser slots that are not zero, sampling counters past 0 and a ring whose stored count is capped at its rows.  A replay shows only its end
state, so the fixture wraps ``torch.cuda.CUDAGraph.replay`` (here only) and, before every replay the trainer issues, clones on the current
stream (the trainers' launch stream, so the clones are ordered before the replay) the state the block reads: the parameters, the target,
the optimiser slots and counters, the sampling and acting records, the stored count, the whole ring and, for DQN, the replay trees.  The
latest snapshot is the state before the run's last block.

From that snapshot the block's gradient steps are launched again by hand with the library's launchers (``FusedSACPrepare`` / ``Grad`` /
``Adam``, their DDPG equivalents, ``FusedReplay`` / ``FusedDQNTarget`` / ``FusedDQNGrad`` / ``FusedClipAdam``), the ring rows the block stored
copied in at their steps; the hand launches must give the trainer's end state byte for byte, and each gradient step's own inputs (the
parameters, the target, the slots and the ring it saw) are then compared with the float64 models of tests/*_numpy_ref.py:
  sampling   : the indices from the trainer's Philox record at counter k = the gradient steps before this one, over min(t + 1, rows) N stored
               transitions (DQN: tree_sample_model on the trees after the block's add);
  gradient   : per tensor within grad_bound (SAC and DQN: + 4x float32 autograd's own error on the same samples);
  optimiser  : bit for bit from the kernel's gradient: TF Adam at the snapshot's beta powers (SAC), MpiAdam at its t (DDPG), clip + Adam (DQN),
               and the Polyak updates;
  ring       : the rows written in the block sit at t % rows, every other row is unchanged, obs[t + 1] == next_obs[t] across the wrap, and the
               stored actions are the trainer's draws from the parameters of the moment;
  controls   : the float64 model with the online network as the target, the sampling counter one step back, or the stored count uncapped
               exceeds the bound the kernel is held to.
"""
import copy
import sys

import numpy as np
import pytest
import torch

from ddpg_numpy_ref import actor_fwd, ddpg_step_model, layout as ddpg_layout, mpi_adam_polyak_f32, ou_model, unpack as ddpg_unpack
from deepq_numpy_ref import dqn_forward_model, dqn_step_model, tree_sample_model
from sac_numpy_ref import forward as sac_forward, layout as sac_layout, unpack as sac_unpack
from test_consumer_reference_cpu import grad_bound, grad_errors, philox_words, u53
from test_ddpg_gpu import _tensors as ddpg_tensors
from test_sac_gpu import _gauss, _tensors as sac_tensors
from test_sac_step_gpu import _float32_autograd as sac_float32_autograd, _model as sac_model

pytestmark = pytest.mark.gpu

SEED = 5
f32 = np.float32


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _np(x):
    if isinstance(x, dict):
        return {k: _np(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_np(v) for v in x]
    return x.detach().cpu().numpy() if torch.is_tensor(x) else x


class Snapshots(object):
    """Wraps torch.cuda.CUDAGraph.replay while a trainer runs: before each replay, ``take(frames)`` (frames: the locals of the calling
    functions up to the trainer's ``train``, by function name) clones what the replay reads, on the current stream.  Only the latest
    snapshot is kept; ``log`` has one ``note(frames)`` per replay."""

    def __init__(self, train, take, note):
        self.code, self.take, self.note, self.last, self.log = train.__code__, take, note, None, []

    def __enter__(self):
        self._mp, orig, snaps = pytest.MonkeyPatch(), torch.cuda.CUDAGraph.replay, self

        def replay(graph):
            frames, f = {}, sys._getframe(1)
            while f is not None:
                frames.setdefault(f.f_code.co_name, f.f_locals)
                if f.f_code is snaps.code:
                    break
                f = f.f_back
            snaps.last = None                                 # free the previous clones first
            snaps.last = snaps.take(frames)
            snaps.log.append(snaps.note(frames))
            return orig(graph)
        self._mp.setattr(torch.cuda.CUDAGraph, "replay", replay)
        return self

    def __exit__(self, *exc):
        self._mp.undo()


def _online(r, arena):
    """What the target network mirrors in the arena: SAC's vf, DDPG's whole arena."""
    if r["algo"] == "ddpg":
        return arena
    lo = sac_layout(r["W"], r["A"])[0]["vf"][0]
    return arena[lo:lo + r["S"]["target"].size]


def _over(g, want, bounds):
    """max over tensors of |g - want| / bound: > 1 where a model misses the bound the kernel is held to."""
    return max(np.abs(g[lo:hi] - want[lo:hi]).max() / b for (lo, hi), b in bounds)


def _ring_checks(S, E, t0, G, rows):
    """Rows outside the block unchanged; obs[t] == next_obs[t - 1] for every step of the block, across the wrap from row rows - 1 to 0."""
    written = sorted({t % rows for t in range(t0, t0 + G)})
    keep = np.setdiff1d(np.arange(rows), written)
    for k in E:
        assert np.array_equal(E[k][keep].view(np.uint8), S[k][keep].view(np.uint8)), k
    for t in range(t0, t0 + G):
        prev = (E if t - 1 >= t0 else S)["next_obs"][(t - 1) % rows]
        assert np.array_equal(E["obs"][t % rows].view(np.uint32), prev.view(np.uint32)), t
    return written


# ---------------------------------------------------------------- SAC and DDPG: the replay-ring loop of rl_baselines/offpolicy.py

def _take_arena(frames):
    L, T = frames["learn"], frames["train"]
    ctx, fopt, fact = T["ctx"], T["fopt"], T["fact"]
    s = dict(t0=L["t0"], stats=dict(L["stats"]), arena=ctx.nets.arena.detach().clone(), target=ctx.nets.target.clone(), m=fopt.m.clone(),
             v=fopt.v.clone(), prep_rng=T["fprep"].rng.clone(), act_rng=fact.rng.clone(), step=ctx.fstore.step.clone(),
             ring={k: x.clone() for k, x in ctx.ring.items()})
    if hasattr(fopt, "beta_power"):
        s.update(beta_power=fopt.beta_power.clone(), lr=fopt.lr.clone())
    else:
        s.update(t=fopt.t.clone(), ou=fact.ou.clone())
    return s


def _note_arena(frames):
    return frames["learn"]["t0"]


def _arena_run(algo, env_id, N, K, kw, hp, T):
    from srl_sim import backend
    backend.use_library(None, None)
    if algo == "sac":
        from rl_baselines.sac import train
    else:
        from rl_baselines.ddpg import train
    with Snapshots(train, _take_arena, _note_arena) as snaps:
        train(env_id, N, T * N, seed=SEED, env_kwargs=dict(is_discrete=False, **kw), verbose=0, num_stack=K, hyperparams=hp)
    torch.cuda.synchronize()
    return train, snaps


def _hand_arena(algo, lib, S, E_ring, hp, W, A, N, t0, G):
    """The block's steps from the snapshot with fresh launchers: each stored row copied in from the end ring at its step, each gradient step
    launched as the trainer does.  Returns (per gradient step: the state it saw and what it left, per env step: the arena it acted with,
    the end state)."""
    rows = E_ring["obs"].shape[0]
    st = _stream()
    ring = {k: x.clone() for k, x in S["ring"].items()}
    if algo == "sac":
        from rl_baselines.sac import ADAM_BETA1, ADAM_BETA2, ADAM_EPS, SACNets, cadence
        from srl_sim.policy import FusedSACAdam, FusedSACGrad, FusedSACPrepare
        nets = SACNets(W, A).cuda()
        grad = torch.zeros_like(nets.arena.data)
        B = hp["batch_size"] * N
        prep = FusedSACPrepare(lib, nets, ring, B, SEED + 1, grad, FusedSACGrad.workspace(lib, nets, B))
        fgrad, fopt = FusedSACGrad(lib, nets), FusedSACAdam(lib, nets, ADAM_BETA1, ADAM_BETA2, ADAM_EPS, hp["tau"])
        fopt.beta_power.copy_(S["beta_power"]); fopt.lr.copy_(S["lr"])
        plan = lambda t: cadence(t, hp)[1]
        launch = lambda step, polyak: (prep(step, hp["gamma"], None, -float(A), stream=st), fgrad(prep, grad, stream=st),
                                       fopt(grad, polyak=polyak, stream=st))
        opt = dict(beta_power=fopt.beta_power)
    else:
        from rl_baselines.ddpg import ADAM_BETA1, ADAM_BETA2, ADAM_EPS, DDPGNets, cadence
        from srl_sim.policy import FusedDDPGAdam, FusedDDPGGrad, FusedDDPGPrepare
        nets = DDPGNets(W, A).cuda()
        grad = torch.zeros_like(nets.arena.data)
        B = hp["batch_size"] * N
        prep = FusedDDPGPrepare(lib, nets, ring, B, SEED + 1)
        fgrad = FusedDDPGGrad(lib, nets, B, hp["critic_l2_reg"])
        fopt = FusedDDPGAdam(lib, nets, hp["actor_lr"], hp["critic_lr"], hp["tau"], ADAM_BETA1, ADAM_BETA2, ADAM_EPS)
        fopt.t.copy_(S["t"])
        plan = lambda t: [True] * cadence(t, hp)
        launch = lambda step, polyak: (prep(step, hp["gamma"], hp["reward_scale"], stream=st), fgrad(prep, grad, stream=st),
                                       fopt(grad, stream=st))
        opt = dict(adam_t=fopt.t)
    with torch.no_grad():
        nets.arena.copy_(S["arena"]); nets.target.copy_(S["target"])
    fopt.m.copy_(S["m"]); fopt.v.copy_(S["v"]); prep.rng.copy_(S["prep_rng"])
    step = S["step"].clone()
    state = lambda: _np(dict(arena=nets.arena, target=nets.target, m=fopt.m, v=fopt.v, **opt))
    steps, actors = [], {}
    for t in range(t0, t0 + G):
        actors[t] = nets.arena.detach().cpu().numpy()
        for k in ring:
            ring[k][t % rows].copy_(E_ring[k][t % rows])
        step[0] += 1
        for polyak in plan(t):
            pre = dict(state(), t=t, rng=int(prep.rng[1]), stored=int(step[0]))
            launch(step, polyak)
            steps.append((pre, dict(state(), idx=prep.idx.cpu().numpy(), grad=grad.cpu().numpy()), polyak))
    torch.cuda.synchronize()
    return steps, actors, dict(state(), ring=_np(ring), rng=prep.rng.cpu().numpy(), grad=grad.cpu().numpy())


def _arena_fixture(algo, param, cuda_lib):
    env_id, N, K, kw, hp_over, T = param
    train, snaps = _arena_run(algo, env_id, N, K, kw, hp_over, T)
    if algo == "sac":
        from rl_baselines.sac import SAC_DEFAULTS as D
        G = 2 if D["train_freq"] % 2 else D["train_freq"]
    else:
        from rl_baselines.ddpg import DDPG_DEFAULTS as D
        G = dict(D, **hp_over)["nb_rollout_steps"]
    hp = dict(D, **hp_over)
    nets, S = train.last_nets, snaps.last
    W, A, rows = nets.obs_dim, nets.act_dim, hp["buffer_size"]
    t0 = int(S["t0"])
    steps, actors, hand = _hand_arena(algo, cuda_lib, S, train.last_ring, hp, W, A, N, t0, G)
    m, v = train.last_adam[0], train.last_adam[1]
    E = _np(dict(arena=nets.arena, target=nets.target, m=m, v=v, ring=train.last_ring, rng=train.last_fused["prepare"].rng,
                 act_rng=train.last_fused["act"].rng, step=train.last_fused["store"].step, grad=train.last_grad))
    if algo == "sac":
        E["beta_power"] = _np(train.last_adam[2])
    else:
        E.update(adam_t=_np(train.last_adam[2]), ou=_np(train.last_ou))
    out = dict(algo=algo, N=N, W=W, A=A, rows=rows, hp=hp, G=G, t0=t0, T=T, S=_np(S), E=E, stats=dict(train.stats), log=list(snaps.log),
               steps=steps, actors=actors, hand=hand, bounds={})
    train.last_ring = train.last_nets = train.last_fused = train.last_adam = train.last_grad = train.last_before_first_step = None
    snaps.last = None
    torch.cuda.empty_cache()
    return out


SAC_RUNS = [("KukaButtonGymEnv-v0", 4096, 1, {}, dict(buffer_size=151), 454),
            ("MobileRobotGymEnv-v0", 8192, 1, dict(shape_reward=True), dict(buffer_size=150), 320),
            ("KukaButtonGymEnv-v0", 4096, 4, {}, dict(buffer_size=151), 454)]
DDPG_RUNS = [("KukaButtonGymEnv-v0", 4096, 1, {}, {}, 300),
             ("MobileRobotGymEnv-v0", 8192, 1, dict(shape_reward=True), dict(buffer_size=130, nb_rollout_steps=20, nb_train_steps=4), 140),
             ("KukaButtonGymEnv-v0", 4096, 4, {}, dict(buffer_size=130, nb_rollout_steps=20, nb_train_steps=4), 140)]
_id = lambda r: "%s_%d_stack%d_rows%d" % (r[0].split("GymEnv")[0], r[1], r[2], r[4].get("buffer_size", 100))


@pytest.fixture(scope="module", params=[("sac", r) for r in SAC_RUNS] + [("ddpg", r) for r in DDPG_RUNS],
                ids=["sac-" + _id(r) for r in SAC_RUNS] + ["ddpg-" + _id(r) for r in DDPG_RUNS])
def arena_run(request, cuda_lib):
    algo, param = request.param
    return _arena_fixture(algo, param, cuda_lib)


def test_arena_block_is_a_graph_replay_on_a_wrapped_ring(arena_run):
    r = arena_run
    S, rows, t0, G, N = r["S"], r["rows"], r["t0"], r["G"], r["N"]
    k0, n = r["S"]["stats"]["grad_steps"], len(r["steps"])
    print("\n%s: last block t0=%d (G=%d), ring phase %d..%d of %d rows, %d rows stored before it, gradient steps k=%d..%d, %d replays" % (
        r["algo"], t0, G, t0 % rows, (t0 + G - 1) % rows, rows, int(S["step"][0]), k0, k0 + n - 1, r["stats"]["graph_replays"]))
    assert t0 + G == r["T"] and r["log"][-1] == t0 and r["stats"]["graphs"] == 1 and r["stats"]["graph_replays"] >= 2
    assert int(S["step"][0]) == t0 and t0 + G > rows and t0 - G > 0    # the block's gradient steps see the stored count capped at rows
    assert r["stats"]["grad_steps"] == k0 + n and n >= 2
    assert int(S["prep_rng"][1]) == k0 and int(S["act_rng"][1]) == t0
    if r["algo"] == "sac" and r["rows"] == 151:
        assert t0 % rows == rows - 1                             # the block stores row 150, then row 0
    if r["algo"] == "ddpg":
        assert int(S["t"][0]) == k0 and (G == rows or (t0 % rows) + G > rows)   # the block rewrites the whole ring, or straddles its wrap
    assert not np.array_equal(S["target"], _online(r, S["arena"]))


def test_arena_hand_launches_give_the_trainers_bytes(arena_run):
    """The block's gradient steps, launched by hand from the snapshot, end in the trainer's parameters, target, slots, counters, gradient and
    ring, byte for byte."""
    r = arena_run
    E, H = r["E"], r["hand"]
    for k in ("arena", "target", "m", "v", "grad", "rng") + (("beta_power",) if r["algo"] == "sac" else ("adam_t",)):
        assert np.array_equal(np.asarray(E[k]).view(np.uint8), np.asarray(H[k]).view(np.uint8)), k
    for k in E["ring"]:
        assert np.array_equal(E["ring"][k].view(np.uint8), H["ring"][k].view(np.uint8)), k
    assert int(E["step"][0]) == r["T"] and int(E["act_rng"][1]) == r["T"]


def test_arena_ring_holds_the_block(arena_run):
    """The rows the block stored sit at t % rows and no other row changed; obs[t] == next_obs[t - 1] across the wrap; each stored action is
    the trainer's draw of step t from the parameters it acted with: SAC tanh(mu + std eps) with eps of (seed, env, t), purposes 26 + k / 4;
    DDPG clip(tanh(actor) + x_t, -1, 1) with the OU state carried on from the snapshot and restarted after a done."""
    r = arena_run
    S, E, N, W, A, rows, t0, G = r["S"]["ring"], r["E"]["ring"], r["N"], r["W"], r["A"], r["rows"], r["t0"], r["G"]
    _ring_checks(S, E, t0, G, rows)
    worst = 0.0
    if r["algo"] == "sac":
        from rl_baselines.sac import LOG_STD_MAX, LOG_STD_MIN
        nets_lay, _ = sac_layout(W, A)
        for t in range(t0, t0 + G):
            out, _ = sac_forward(sac_unpack(r["actors"][t], *nets_lay["actor"]), E["obs"][t % rows].astype(np.float64))
            mu, ls = out[:, :A], np.clip(out[:, A:], LOG_STD_MIN, LOG_STD_MAX)
            want = np.tanh(mu + np.exp(ls) * _gauss(SEED, np.arange(N), t, 26, A))
            worst = max(worst, np.abs(E["act"][t % rows] - want).max())
        assert not np.array_equal(r["actors"][t0], r["actors"][t0 + 1])           # the block's second step acted after a gradient step
    else:
        x, sigma = r["S"]["ou"].astype(np.float64), r["hp"]["noise_action_sigma"]
        pa = ddpg_unpack(r["actors"][t0], W, A, "actor")
        for t in range(t0, t0 + G):
            prev = (E if t - 1 >= t0 else S)["done"][(t - 1) % rows]
            x = ou_model(x, _gauss(SEED, np.arange(N), t, 33, A), prev, sigma)
            mu, _, _ = actor_fwd(pa, E["obs"][t % rows].astype(np.float64))
            worst = max(worst, np.abs(E["act"][t % rows] - np.clip(mu + x, -1, 1)).max())
        assert np.abs(r["E"]["ou"] - x).max() <= 1e-5
        assert np.abs(r["S"]["ou"]).max() > 0                   # the carried state is not the initial zero
    print("\n  stored actions: max |a - a64| = %.1e" % worst)
    assert worst <= 1e-4


def _arena_sample(r, k, stored, uncapped_t=None):
    """The indices of the gradient step at counter k over ``stored`` lockstep rows (min(t + 1, rows)); ``uncapped_t``: over (t + 1) N
    instead, wrapped into the ring (a control)."""
    N, B = r["N"], r["hp"]["batch_size"] * r["N"]
    size = (uncapped_t + 1) * N if uncapped_t is not None else min(stored, r["rows"]) * N
    idx = np.minimum(np.floor(u53(philox_words(SEED + 1, np.arange(B), k, 30 if r["algo"] == "sac" else 35)) * size), size - 1).astype(np.int64)
    return idx % (r["rows"] * N)


def _ring_at(r, j):
    """The ring gradient step j saw: the end ring with the rows the block stores after that step taken from the snapshot."""
    pre = r["steps"][j][0]
    ring = {k: x.copy() for k, x in r["E"]["ring"].items()}
    for t in range(pre["t"] + 1, r["t0"] + r["G"]):
        for k in ring:
            ring[k][t % r["rows"]] = r["S"]["ring"][k][t % r["rows"]]
    return ring


def _arena_model(r, j, idx, target=None, counter=None):
    """(float64 gradient, float32 autograd gradient or None) of gradient step j from the state it saw."""
    pre = r["steps"][j][0]
    W, A, B = r["W"], r["A"], len(idx)
    ring = _ring_at(r, j)
    tg = pre["target"] if target is None else target
    k = pre["rng"] if counter is None else counter
    if r["algo"] == "sac":
        eps = _gauss(SEED + 1, np.arange(B), k, 31, A)
        rr = dict(W=W, A=A, ring=ring, before=dict(arena=pre["arena"], target=tg))
        want, _ = sac_model(rr, idx, eps)
        return want, (sac_float32_autograd(rr, idx, eps) if target is None and counter is None else None)
    flat = {key: a.reshape((-1,) + a.shape[2:]) for key, a in ring.items()}
    hp, want = r["hp"], 0.0
    for lo in range(0, B, 1 << 16):
        ix = idx[lo:lo + (1 << 16)]
        g, _ = ddpg_step_model(pre["arena"], tg, W, A, flat["obs"][ix], flat["act"][ix], flat["rew"][ix], flat["next_obs"][ix],
                               flat["done"][ix].astype(np.float64), hp["gamma"], hp["reward_scale"], 0.0)
        want = want + g * (len(ix) / B)
    w0 = pre["arena"].astype(np.float64)
    for name, lo, hi in ddpg_tensors(W, A):                   # critic_l2_reg w, once over the whole batch
        if name in ("critic.w1", "critic.w2"):
            want[lo:hi] += hp["critic_l2_reg"] * w0[lo:hi]
    return want, None


def _checked(r):
    n = len(r["steps"])
    return sorted({0, 1, n // 2, n - 1})


def _tensor_list(r):
    return sac_tensors(r["W"], r["A"]) if r["algo"] == "sac" else ddpg_tensors(r["W"], r["A"])


def _step_bounds(r, j):
    """Gradient step j against float64: the indices, then each tensor within its bound; returns [((lo, hi), bound)] for the controls."""
    if j in r["bounds"]:
        return r["bounds"][j]
    pre, post, _ = r["steps"][j]
    k = r["S"]["stats"]["grad_steps"] + j
    assert pre["rng"] == k and pre["stored"] == pre["t"] + 1
    idx = _arena_sample(r, k, pre["stored"])
    assert np.array_equal(post["idx"], idx), j
    want, g32 = _arena_model(r, j, idx)
    g = post["grad"].astype(np.float64)
    out, worst = [], 0.0
    for name, lo, hi in _tensor_list(r):
        scale = np.abs(want[lo:hi]).max()
        err = np.abs(g[lo:hi] - want[lo:hi]).max()
        bound = grad_bound(scale) + (4.0 * np.abs(g32[lo:hi] - want[lo:hi]).max() if g32 is not None else 0.0)
        assert scale > 0 and err <= bound, (j, name, lo, err, bound, scale)
        out.append(((lo, hi), bound))
        worst = max(worst, err / bound)
    if r["algo"] == "sac":                                      # d ent_coef_loss / d log_ent_coef
        assert abs(g[-1] - want[-1]) <= 1e-5 * (1.0 + abs(want[-1])) + 4.0 * abs(g32[-1] - want[-1])
    print("  step j=%d (k=%d, t=%d, %d rows stored): worst err/bound %.2f" % (j, k, pre["t"], min(pre["stored"], r["rows"]), worst))
    r["bounds"][j] = out
    return out


def test_arena_gradient_steps_match_float64(arena_run):
    r = arena_run
    print()
    for j in _checked(r):
        _step_bounds(r, j)


def test_arena_optimiser_steps_bit_for_bit(arena_run):
    """Every gradient step of the block: the optimiser and the Polyak update, bit for bit from the kernel's gradient and the slots, beta
    powers or step count that step saw (SAC: TF Adam at beta_power; DDPG: MpiAdam at t = k)."""
    r = arena_run
    hp, W, A = r["hp"], r["W"], r["A"]
    for j, (pre, post, polyak) in enumerate(r["steps"]):
        gk = post["grad"]
        if r["algo"] == "sac":
            from rl_baselines.sac import ADAM_BETA1, ADAM_BETA2, ADAM_EPS
            b1, b2, lr, tau = f32(ADAM_BETA1), f32(ADAM_BETA2), f32(hp["learning_rate"]), f32(hp["tau"])
            bp = pre["beta_power"]
            lr_t = (lr * np.sqrt(f32(1) - bp[1])) / (f32(1) - bp[0])
            m = pre["m"] + (gk - pre["m"]) * (f32(1) - b1)
            v = pre["v"] + (gk * gk - pre["v"]) * (f32(1) - b2)
            p1 = pre["arena"] - (m * lr_t) / (np.sqrt(v) + f32(ADAM_EPS))
            lo = sac_layout(W, A)[0]["vf"][0]
            tg = (f32(1) - tau) * pre["target"] + tau * p1[lo:lo + pre["target"].size] if polyak else pre["target"]
            assert np.array_equal(post["beta_power"], bp * np.array([b1, b2], np.float32)), j
        else:
            steps = int(pre["adam_t"][0])
            assert steps == r["S"]["stats"]["grad_steps"] + j
            p1, tg, m, v = mpi_adam_polyak_f32(pre["arena"], pre["target"], [gk], ddpg_layout(W, A)[0]["actor"]["end"], hp["actor_lr"], hp["critic_lr"], hp["tau"],
                                               m=pre["m"], v=pre["v"], steps=steps)
            assert int(post["adam_t"][0]) == steps + 1
        for key, want in (("m", m), ("v", v), ("arena", p1), ("target", tg)):
            assert np.array_equal(post[key], want), (j, key)
    if r["algo"] == "sac":                                      # the step count matters: beta powers well past their first step
        assert r["S"]["beta_power"][0] < f32(0.9) ** 100
    assert np.abs(r["steps"][0][0]["m"]).max() > 0


def test_arena_controls_exceed_the_bound(arena_run):
    """The float64 model of the block's last gradient step misses the bound the kernel meets when it takes the online network as the
    target, the sampling counter one step back, or the stored count uncapped ((t + 1) N transitions instead of rows N)."""
    r = arena_run
    j = len(r["steps"]) - 1
    bounds = _step_bounds(r, j)
    pre, post, _ = r["steps"][j]
    g = post["grad"].astype(np.float64)
    k = pre["rng"]
    online = _online(r, pre["arena"])
    assert not np.array_equal(online, pre["target"])
    idx = _arena_sample(r, k, pre["stored"])
    ratios = dict(target_is_online=_over(g, _arena_model(r, j, idx, target=online)[0], bounds),
                  counter_minus_one=_over(g, _arena_model(r, j, _arena_sample(r, k - 1, pre["stored"]), counter=k - 1)[0], bounds),
                  uncapped=_over(g, _arena_model(r, j, _arena_sample(r, k, pre["stored"], uncapped_t=pre["t"]))[0], bounds))
    print("\n  controls, max err/bound: " + "  ".join("%s %.1f" % kv for kv in ratios.items()))
    for name, x in ratios.items():
        assert x > 1.0, (name, x)


# ---------------------------------------------------------------- DQN: one graph per ring phase (rl_baselines/deepq.py)

DQN_T = 300
DQN_HP = dict(learning_starts=40, buffer_size=100, train_freq=4, target_network_update_freq=60, batch_size=32)
DQN_RUNS = [("MobileRobotGymEnv-v0", 8192, 1, dict(is_discrete=True, shape_reward=True)), ("KukaButtonGymEnv-v0", 4096, 1, dict(is_discrete=True)),
            ("KukaButtonGymEnv-v0", 4096, 4, dict(is_discrete=True))]
DQN_PARAMS = [(r, p) for r in DQN_RUNS for p in (True, False)]


def _take_dqn(frames):
    T = frames["train"]
    rep, fopt = T["replay"], T["fopt"]
    return dict(t0=T["t0"], key=T["key"], stats=dict(T["stats"]), params=[p.detach().clone() for p in T["params"]],
                target=[p.detach().clone() for p in T["target"].parameters()], m=[x.clone() for x in fopt.m], v=[x.clone() for x in fopt.v],
                beta_power=fopt.beta_power.clone(), lr=fopt.lr.clone(), sum=rep.sum.clone(), min=rep.min.clone(), max_priority=rep.max_priority.clone(),
                size=rep.size.clone(), stamp=rep.stamp.clone(), rng=rep.rng.clone(), act_rng=T["fact"].rng.clone(),
                ring={k: x.clone() for k, x in T["ring"].items()}, eps_blk=T["eps_blk"].clone(), beta_blk=T["beta_blk"].clone())


def _note_dqn(frames):
    T = frames["train"]
    return dict(t0=T["t0"], key=T["key"], size=int(T["replay"].size[0]),
                target_is_online=all(torch.equal(a, b) for a, b in zip(T["params"], T["target"].parameters())))


@pytest.fixture(scope="module", params=DQN_PARAMS, ids=["%s_%d_stack%d-%s" % (r[0].split("GymEnv")[0], r[1], r[2], "prioritized" if p else "uniform")
                                                         for r, p in DQN_PARAMS])
def dqn_run(request, cuda_lib):
    (env_id, N, K, kw), prioritized = request.param
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.deepq import (ADAM_BETA1, ADAM_BETA2, ADAM_EPS, DQN_DEFAULTS, GRAD_CLIP_NORM, DuelingQ, can_sample, cadence, train)
    from srl_sim.policy import FusedClipAdam, FusedDQNGrad, FusedDQNTarget, FusedReplay
    hp = dict(DQN_DEFAULTS, **DQN_HP, prioritized_replay=prioritized)
    with Snapshots(train, _take_dqn, _note_dqn) as snaps:
        train(env_id, N, DQN_T * N, seed=SEED, env_kwargs=kw, verbose=0, hyperparams=hp, num_stack=K)
    torch.cuda.synchronize()
    S, rows, G, B, st = snaps.last, hp["buffer_size"], hp["train_freq"], hp["batch_size"] * N, _stream()
    t0 = int(S["t0"])
    online, W = train.last_policy, train.last_policy.pi[0].weight.shape[1]
    # the block by hand from the snapshot
    qnet, target = DuelingQ(W, online.n_actions).cuda(), DuelingQ(W, online.n_actions).cuda()
    with torch.no_grad():
        for p, x in zip(qnet.parameters(), S["params"]):
            p.copy_(x)
        for p, x in zip(target.parameters(), S["target"]):
            p.copy_(x)
    target.requires_grad_(False)
    params = list(qnet.parameters())
    for p in params:
        p.grad = torch.zeros_like(p)
    ring = {k: x.clone() for k, x in S["ring"].items()}
    flat = {k: x.reshape((rows * N,) + x.shape[2:]) for k, x in ring.items()}
    replay = FusedReplay(cuda_lib, rows, N, SEED + 1, hp["prioritized_replay_alpha"], "cuda")
    for name in ("sum", "min", "max_priority", "size", "stamp", "rng"):
        getattr(replay, name).copy_(S[name])
    ftarget, fgrad = FusedDQNTarget(cuda_lib, qnet, target), FusedDQNGrad(cuda_lib, qnet, B)
    fopt = FusedClipAdam(cuda_lib, qnet, GRAD_CLIP_NORM, ADAM_BETA1, ADAM_BETA2, ADAM_EPS)
    for a, b in zip(fopt.m + fopt.v, S["m"] + S["v"]):
        a.copy_(b)
    fopt.beta_power.copy_(S["beta_power"]); fopt.lr.copy_(S["lr"])
    idx, w, y, td = (torch.zeros(B, dtype=torch.int64, device="cuda"), torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda"),
                     torch.zeros(B, device="cuda"))
    end_ring = train.last_ring
    tree = lambda: _np(dict(sum=replay.sum, min=replay.min, size=replay.size, max_priority=replay.max_priority))
    nets = lambda: _np(dict(params=list(qnet.parameters()), m=fopt.m, v=fopt.v, beta_power=fopt.beta_power))
    steps, actors = [], {}
    for k in range(G):
        t = t0 + k
        actors[t] = [p.detach().cpu().numpy() for p in params]
        for key in ring:
            ring[key][t % rows].copy_(end_ring[key][t % rows])
        replay.add(t % rows, stream=st)
        if cadence(t, hp)[0] and can_sample(t, hp, N):
            pre = dict(tree(), **nets(), t=t, rng=int(replay.rng[1]), target=[p.cpu().numpy() for p in target.parameters()], ring=_np(ring))
            replay.sample(B, idx, w, prioritized=prioritized, beta=S["beta_blk"][k:k + 1], stream=st)
            ftarget(B, idx, flat["next_obs"], flat["rew"], flat["done"], hp["gamma"], y, stream=st)
            fgrad(idx, flat["obs"], flat["act"], y, w if prioritized else None, td, stream=st)
            post = dict(grads=[p.grad.cpu().numpy() for p in params], **_np(dict(idx=idx, w=w, y=y, td=td)))
            fopt(stream=st)
            if prioritized:
                replay.update(B, idx, td, hp["prioritized_replay_eps"], stream=st)
            steps.append((pre, dict(post, **nets(), **tree())))
    torch.cuda.synchronize()
    hand = dict(nets(), **tree(), ring=_np(ring), rng=replay.rng.cpu().numpy(), stamp=replay.stamp.cpu().numpy())
    rep, (m, v, bp) = train.last_replay, train.last_adam
    E = _np(dict(params=list(online.parameters()), target=list(train.last_target.parameters()), m=m, v=v, beta_power=bp, sum=rep.sum, min=rep.min,
                 size=rep.size, max_priority=rep.max_priority, rng=rep.rng, stamp=rep.stamp, ring=end_ring))
    out = dict(N=N, W=W, nA=online.n_actions, rows=rows, hp=hp, G=G, t0=t0, prioritized=prioritized, S=_np(S), E=E, hand=hand, steps=steps,
               actors=actors, stats=dict(train.stats), log=list(snaps.log), cap=rep.tree_cap, bounds=None)
    train.last_ring = train.last_policy = train.last_target = train.last_replay = train.last_adam = None
    snaps.last = None
    torch.cuda.empty_cache()
    return out


def _qnet_of(r, params):
    from rl_baselines.deepq import DuelingQ
    q = DuelingQ(r["W"], r["nA"])
    with torch.no_grad():
        for p, x in zip(q.parameters(), params):
            p.copy_(torch.from_numpy(np.asarray(x)))
    return q


def test_dqn_block_replays_a_graph_captured_during_fill(dqn_run):
    """The last block (t0 = 296) replays the graph of ring phase 96, captured at t0 = 96 while the ring held 96 of its 100 rows, on a ring
    that has wrapped; the target was last copied at t = 240, so it differs from the online network at the block."""
    r = dqn_run
    rows, t0, G, N, log = r["rows"], r["t0"], r["G"], r["N"], r["log"]
    first = {}
    for e in log:
        first.setdefault(e["key"], e)
    fill = sorted(key for key, e in first.items() if e["t0"] < rows)
    later = sorted(key for key, e in first.items() if e["t0"] >= rows)
    print("\nDQN: last block t0=%d phase %d, %d stored before it, gradient step k=%d; phases captured during fill %s, after %s; %d replays" % (
        t0, t0 % rows, int(r["S"]["size"][0]), r["S"]["stats"]["grad_steps"], fill, later, len(log)))
    assert t0 == DQN_T - G and log[-1]["t0"] == t0 and log[-1]["key"] == t0 % rows == 96
    assert first[96]["t0"] == 96 and first[96]["size"] == 96 * N       # captured while the ring was filling ...
    assert log[-1]["size"] == rows * N == int(r["S"]["size"][0])       # ... replayed on the wrapped ring
    assert fill == list(range(48, 100, 4)) and later == list(range(0, 48, 4))
    assert r["stats"]["graphs"] == rows // G and r["stats"]["graph_replays"] == len(log)
    assert any(e["t0"] >= rows and e["key"] in fill for e in log[:-1])
    # target copies at 60, 120, 180, 240: the snapshot after a copy block sees target == online, the last block does not
    assert r["stats"]["target_copies"] == 4
    after_copy = [e for e in log if e["t0"] - G in (60, 120, 180, 240)]
    assert after_copy and all(e["target_is_online"] for e in after_copy) and not log[-1]["target_is_online"]
    assert len(r["steps"]) == 1


def test_dqn_hand_launches_give_the_trainers_bytes(dqn_run):
    r = dqn_run
    E, H = r["E"], r["hand"]
    for k in ("params", "m", "v"):
        for a, b in zip(E[k], H[k]):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), k
    for k in ("beta_power", "sum", "min", "size", "max_priority", "rng", "stamp"):
        assert np.array_equal(np.asarray(E[k]).view(np.uint8), np.asarray(H[k]).view(np.uint8)), k
    for k in E["ring"]:
        assert np.array_equal(E["ring"][k].view(np.uint8), H["ring"][k].view(np.uint8)), k
    for a, b in zip(E["target"], r["S"]["target"]):              # no copy in the block: the target is the one copied at t = 240
        assert np.array_equal(a, b)


def test_dqn_ring_and_trees_hold_the_block(dqn_run):
    """Rows at t % rows, the rest unchanged, obs[t] == next_obs[t - 1]; the actions are the epsilon-greedy draws of the online network of the
    moment; the overwritten leaves hold max_priority^alpha (every leaf 1 for uniform replay)."""
    from rl_baselines.deepq import linear_schedule
    r = dqn_run
    S, E, N, rows, t0, G, A = r["S"]["ring"], r["E"]["ring"], r["N"], r["rows"], r["t0"], r["G"], r["nA"]
    _ring_checks(S, E, t0, G, rows)
    assert int(r["S"]["act_rng"][1]) == t0
    checked = 0
    for t in range(t0, t0 + G):
        eps = np.float32(linear_schedule(int(r["hp"]["exploration_fraction"] * DQN_T), 1.0, r["hp"]["exploration_final_eps"], t))
        assert r["S"]["eps_blk"][t - t0] == eps
        words = philox_words(SEED, np.arange(N), t, 24)
        explore = u53(words) < float(eps)
        act = E["act"][t % rows]
        assert np.array_equal(act[explore], ((words[explore, 2].astype(np.uint64) * np.uint64(A)) >> np.uint64(32)).astype(np.int64)), t
        q = dqn_forward_model(_qnet_of(r, r["actors"][t]), E["obs"][t % rows])
        top2 = np.sort(q, 1)[:, -2:]
        clear = ~explore & (top2[:, 1] - top2[:, 0] > 2e-5 * (np.abs(q).max() + 1.0))
        assert np.array_equal(act[clear], q.argmax(1)[clear]), t
        checked += int(clear.sum())
    assert checked > 0.9 * G * N
    cap, alpha = r["cap"], r["hp"]["prioritized_replay_alpha"]
    pre, post = r["steps"][0]
    lo = (t0 % rows) * N                                          # the block's first add, before its gradient step
    leaf = pre["sum"][cap + lo:cap + lo + N]
    assert np.all(leaf == float(r["S"]["max_priority"][0]) ** alpha) and np.array_equal(pre["min"][cap + lo:cap + lo + N], leaf)
    after = slice(cap + lo + N, cap + (t0 % rows + G) * N)         # the adds after the gradient step, at the max_priority it left
    assert np.all(r["E"]["sum"][after] == float(r["E"]["max_priority"][0]) ** alpha)
    if not r["prioritized"]:
        assert np.all(r["E"]["sum"][cap:cap + rows * N] == 1.0)
    else:
        assert r["E"]["max_priority"][0] > 1.0 and len(np.unique(r["S"]["sum"][cap:cap + rows * N])) > N


def _dqn_sample(r, pre, counter, size=None):
    from rl_baselines.deepq import linear_schedule
    B = r["hp"]["batch_size"] * r["N"]
    beta = linear_schedule(DQN_T, r["hp"]["prioritized_replay_beta0"], 1.0, pre["t"])
    assert r["S"]["beta_blk"][pre["t"] - r["t0"]] == beta
    u = u53(philox_words(SEED + 1, np.arange(B), counter, 25))
    return tree_sample_model(pre["sum"], pre["min"], int(pre["size"][0]) if size is None else size, r["cap"], u, beta, r["prioritized"])


def _dqn_model(r, pre, idx, w, target=None):
    from rl_baselines.deepq import ADAM_BETA1, ADAM_BETA2, ADAM_EPS, GRAD_CLIP_NORM
    flat = {k: a.reshape((-1,) + a.shape[2:]) for k, a in pre["ring"].items()}
    b = lambda x: float(np.float32(x))
    return dqn_step_model(_qnet_of(r, pre["params"]), flat["obs"][idx], flat["act"][idx], flat["rew"][idx], flat["done"][idx], flat["next_obs"][idx],
                          b(r["hp"]["gamma"]), b(r["hp"]["learning_rate"]), GRAD_CLIP_NORM, b(ADAM_BETA1), b(ADAM_BETA2), b(ADAM_EPS),
                          target=_qnet_of(r, pre["target"] if target is None else target), weights=w.astype(np.float64),
                          m=[x.astype(np.float64) for x in pre["m"]], v=[x.astype(np.float64) for x in pre["v"]], step=r["S"]["stats"]["grad_steps"] + 1)


def _dqn_misses(r, chk, model, idx):
    """Each check of the gradient step as (miss / what it allows): the indices off the kernel's (at most 1e-4 of them for prioritized replay,
    where a float64 walk may end on the other side of a leaf boundary; none for uniform), y and td within 2e-5 of their scale, and every
    gradient tensor within its bound.  A ratio above 1 fails the check."""
    post = r["steps"][0][1]
    same = post["idx"] == idx
    out = dict(indices=(~same).sum() / (chk["allowed"] + 0.5))
    for key in ("y", "td"):
        out[key] = np.abs(post[key][same] - model[key][same]).max() / (2e-5 * (np.abs(model[key]).max() + 1.0)) if same.any() else np.inf
    out["gradient"] = max(float(np.abs(g - w).max()) / b for g, w, b in zip(post["grads"], model["grads"], chk["bounds"]))
    return out


def _dqn_bounds(r):
    """The block's gradient step against float64: sampling, y, td and the gradient per tensor (grad_bound + 4x float32 autograd's error)."""
    if r["bounds"] is not None:
        return r["bounds"]
    from rl_baselines.deepq import dqn_loss
    pre, post = r["steps"][0]
    k = r["S"]["stats"]["grad_steps"]
    assert pre["rng"] == k and int(pre["size"][0]) == r["rows"] * r["N"]
    idx, w = _dqn_sample(r, pre, k)
    same = post["idx"] == idx
    assert np.allclose(post["w"][same], w[same], rtol=2e-6, atol=0)
    if r["prioritized"]:
        assert w.min() < 0.9                                       # the leaves differ: the importance weights are not all 1
    model = _dqn_model(r, pre, idx, w)
    flat = {key: a.reshape((-1,) + a.shape[2:]) for key, a in pre["ring"].items()}
    q32 = copy.deepcopy(_qnet_of(r, pre["params"])).requires_grad_(True)
    loss, _ = dqn_loss(q32, torch.from_numpy(flat["obs"][idx]), torch.from_numpy(flat["act"][idx]), torch.from_numpy(model["y"]).float(),
                       torch.from_numpy(w))
    loss.backward()
    g64 = [torch.from_numpy(g) for g in model["grads"]]
    e32 = grad_errors([p.grad for p in q32.parameters()], g64)
    kern = grad_errors([torch.from_numpy(g) for g in post["grads"]], g64)
    assert all(scale > 0 for _, scale in kern)
    chk = dict(bounds=[grad_bound(scale) + 4.0 * err32 for (_, scale), (err32, _) in zip(kern, e32)], allowed=1e-4 * len(idx) if r["prioritized"] else 0)
    miss = _dqn_misses(r, chk, model, idx)
    print("\n  step k=%d (t=%d): %d of %d indices off the float64 walk; miss/allowed: %s" % (
        k, pre["t"], int((~same).sum()), len(idx), "  ".join("%s %.2f" % kv for kv in miss.items())))
    for name, x in miss.items():
        assert x <= 1.0, (name, x)
    r["bounds"] = chk
    return chk


def test_dqn_gradient_step_matches_float64(dqn_run):
    _dqn_bounds(dqn_run)


def test_dqn_optimiser_and_priorities_bit_for_bit(dqn_run):
    """clip + TF Adam at the snapshot's slots and beta powers, bit for bit from the kernel's gradient; the priorities written back are
    (|td| + eps)^alpha of the step's own td (the last occurrence of a repeated index), every other leaf unchanged."""
    from rl_baselines.deepq import ADAM_BETA1, ADAM_BETA2, ADAM_EPS, GRAD_CLIP_NORM
    r = dqn_run
    pre, post = r["steps"][0]
    bp, lr = pre["beta_power"], f32(r["hp"]["learning_rate"])
    assert bp[0] < f32(0.9) ** 10 and np.abs(pre["m"][0]).max() > 0
    lr_t = (lr * np.sqrt(f32(1) - bp[1])) / (f32(1) - bp[0])
    r1, r2, clip = f32(1) - f32(ADAM_BETA1), f32(1) - f32(ADAM_BETA2), f32(GRAD_CLIP_NORM)
    for k, g in enumerate(post["grads"]):
        norm = f32(np.sqrt((g.astype(np.float64) ** 2).sum()))
        gc = (g * clip) / max(norm, clip)
        m = pre["m"][k] + (gc - pre["m"][k]) * r1
        v = pre["v"][k] + (gc * gc - pre["v"][k]) * r2
        p = pre["params"][k] - (m * lr_t) / (np.sqrt(v) + f32(ADAM_EPS))
        assert np.array_equal(post["m"][k], m) and np.array_equal(post["v"][k], v) and np.array_equal(post["params"][k], p), k
    assert np.array_equal(post["beta_power"], bp * np.array([f32(ADAM_BETA1), f32(ADAM_BETA2)], np.float32))
    cap, alpha = r["cap"], r["hp"]["prioritized_replay_alpha"]
    if not r["prioritized"]:
        assert np.array_equal(post["sum"], pre["sum"]) and np.array_equal(post["min"], pre["min"])
        return
    idx, td = post["idx"], post["td"]
    p = np.abs(td.astype(np.float32)) + f32(r["hp"]["prioritized_replay_eps"])
    uniq, first_rev = np.unique(idx[::-1], return_index=True)
    last = len(idx) - 1 - first_rev
    want = np.array([float(x) ** alpha for x in p[last]])
    got = post["sum"][cap + uniq]
    assert np.all(np.abs(got - want) <= 4 * np.spacing(want)) and np.array_equal(post["min"][cap + uniq], got)
    other = np.setdiff1d(np.arange(r["rows"] * r["N"]), uniq)
    assert np.array_equal(post["sum"][cap + other], pre["sum"][cap + other])
    assert post["max_priority"][0] == max(pre["max_priority"][0], float(p.max()))


def test_dqn_controls_exceed_the_bound(dqn_run):
    """The float64 model fails the checks the kernel passes with the online network as the target, with the sampling counter one step back,
    and (uniform replay) with the stored count uncapped, (t + 1) N instead of rows N, wrapped into the ring.  Prioritized replay samples by
    mass, and its stored count enters only the clamp of a walk into an empty leaf and the weights, where it cancels; there the count is held
    to rows N exactly by the tree checks above.  With prioritized replay most of the mass sits on a few leaves, so a batch drawn at another
    counter repeats much the same samples and its gradient may stay within the bound; its indices do not."""
    r = dqn_run
    chk = _dqn_bounds(r)
    pre, post = r["steps"][0]
    k = r["S"]["stats"]["grad_steps"]
    idx, w = _dqn_sample(r, pre, k)
    cases = dict(target_is_online=(idx, w, pre["params"]), counter_minus_one=_dqn_sample(r, pre, k - 1) + (None,))
    if not r["prioritized"]:
        iu, wu = _dqn_sample(r, pre, k, size=(pre["t"] + 1) * r["N"])
        cases["uncapped"] = (iu % (r["rows"] * r["N"]), wu, None)
    print()
    for name, (ix, wx, target) in cases.items():
        miss = _dqn_misses(r, chk, _dqn_model(r, pre, ix, wx, target=target), ix)
        print("  control %s, miss/allowed: %s" % (name, "  ".join("%s %.1f" % kv for kv in miss.items())))
        assert max(miss.values()) > 1.0, (name, miss)
