"""
GPU tests of the DQN path (include/srl_policy.h: srl_dqn_*, srl_replay_*, srl_clip_adam; rl_baselines/deepq.py):
  srl_dqn_act       -- Q against float64, greedy actions at epsilon 0, the exploration rate and uniformity (chi-square), the same bytes twice,
                       two sharded launches (env_offset) give the bytes of one, successive launches draw successive counters;
  srl_replay_*      -- the trees, indices and weights against the loop-form transcription of baselines' SegmentTree (tests/deepq_numpy_ref.py)
                       fed the kernel's own Philox uniforms, and at the trainer's 4096 x 1000 and 8192 x 1000 (two and three rebuild passes)
                       against the vectorised tree of rl_baselines.deepq; prioritized and uniform sampling;
  srl_dqn_target    -- y against float64 double Q, with one chunk and several chunks per CTA, through idx and without;
  srl_dqn_grad      -- float64 autograd of rl_baselines.deepq.dqn_loss with the tolerance rule of tests/test_consumer_kernels_gpu.py, the same
                       bytes twice, no weights (NULL) as all-ones weights, and shown to see a missing row;
  srl_clip_adam     -- the float64 TF model over 100 steps, the same bytes twice, non-finite gradients;
  the trainer       -- learns MobileRobot, captured and eager runs give the same bytes, and the entry point runs for every env id.
One whole gradient step of the trainer against float64: tests/test_deepq_step_gpu.py.
"""
import copy

import numpy as np
import pytest
import torch

from deepq_numpy_ref import PrioritizedReplay, clip_adam_model, double_q_model, dqn_forward_model
from test_consumer_reference_cpu import grad_bound, grad_errors

pytestmark = pytest.mark.gpu

CH = 64
# the discrete registry shapes (width, actions) and the wide kernels' widths
Q_SHAPES = [(3, 6), (2, 4), (1, 2), (12, 6), (32, 2)]
PURPOSE_ACT, PURPOSE_REPLAY = 24, 25


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _qnet(width, n, seed=3):
    from rl_baselines.deepq import DuelingQ
    torch.manual_seed(seed)
    q = DuelingQ(width, n).cuda()
    with torch.no_grad():
        for p in q.parameters():       # biases too: some ReLU units are off for most rows, some on
            p.add_(0.1 * torch.randn_like(p))
    return q


@pytest.fixture(scope="module")
def philox_u53(oracle_lib):
    import ctypes
    fn = oracle_lib.lib.oracle_philox4x32
    fn.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32)]
    fn.restype = None

    def draw(seed, streams, counter, purpose):
        out, u, w2 = (ctypes.c_uint32 * 4)(), [], []
        for s in streams:
            fn(seed, int(s), counter, purpose, out)
            u.append(((out[0] >> 5) * 67108864.0 + (out[1] >> 6)) / 9007199254740992.0)
            w2.append(out[2])
        return np.array(u), np.array(w2, np.uint64)
    return draw


@pytest.mark.parametrize("n", [1, 33, 4096])
@pytest.mark.parametrize("width,n_act", Q_SHAPES)
def test_dqn_act_q_and_greedy_actions(cuda_lib, width, n_act, n):
    from srl_sim.policy import FusedDQNAct
    q = _qnet(width, n_act)
    obs = torch.randn(n, width, device="cuda")
    f = FusedDQNAct(cuda_lib, q, seed=11)
    act, act64, qout, obs_buf = (torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda"),
                                 torch.zeros(n, n_act, device="cuda"), torch.zeros(n, width, device="cuda"))
    f(n, obs, act, obs_buf=obs_buf, act_buf=act64, q_out=qout, stream=_stream())
    torch.cuda.synchronize()
    want = dqn_forward_model(q, obs.cpu().numpy())
    tol = 2e-5 * (np.abs(want).max() + 1.0)
    assert np.abs(qout.cpu().numpy() - want).max() <= tol
    top2 = np.sort(want, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 2 * tol
    assert np.array_equal(act.cpu().numpy()[clear], want.argmax(1)[clear])
    assert clear.mean() > 0.9 and torch.equal(act.long(), act64) and torch.equal(obs_buf, obs)
    assert int(f.rng[1]) == 1


def test_dqn_act_explores_at_the_rate_epsilon_uniformly(cuda_lib, philox_u53):
    """epsilon = 1: the actions are uniform (chi-square); epsilon = 0.3: the envs whose Philox word says explore are the ones that may differ
    from greedy, 30 % of them within 4 sigma, and the rest equal greedy; the same seed and counter give the same bytes."""
    from scipy.stats import chisquare
    from srl_sim.policy import FusedDQNAct
    n, A = 32768, 6
    q = _qnet(3, A)
    obs = torch.randn(n, 3, device="cuda")
    runs = []
    for eps in (1.0, 0.3, 0.3):
        f = FusedDQNAct(cuda_lib, q, seed=5)
        f.eps.fill_(eps)
        act = torch.zeros(n, dtype=torch.int32, device="cuda")
        f(n, obs, act, stream=_stream())
        torch.cuda.synchronize()
        runs.append(act.cpu().numpy())
    counts = np.bincount(runs[0], minlength=A)
    assert chisquare(counts).pvalue > 1e-3, counts
    u, w2 = philox_u53(5, range(n), 0, PURPOSE_ACT)
    explore = u < np.float64(np.float32(0.3))
    assert abs(explore.mean() - 0.3) < 4 * np.sqrt(0.3 * 0.7 / n)
    greedy = dqn_forward_model(q, obs.cpu().numpy()).argmax(1)
    assert np.array_equal(runs[1][explore], ((w2[explore] * A) >> 32).astype(np.int64))
    top2 = np.sort(dqn_forward_model(q, obs.cpu().numpy()), 1)[:, -2:]
    clear = ~explore & (top2[:, 1] - top2[:, 0] > 1e-4)
    assert np.array_equal(runs[1][clear], greedy[clear])
    assert np.array_equal(runs[1], runs[2])


def test_dqn_act_sharded_launches_and_successive_counters(cuda_lib, philox_u53):
    """Envs [0, k) and [k, n) in two launches, the second with env_offset = k (k odd, inside a CTA of 32 envs), as data-parallel ranks launch:
    the actions and Q bytes of one launch over [0, n).  Three successive launches draw with counters 0, 1 and 2."""
    from srl_sim.policy import FusedDQNAct
    n, k, A, seed = 1000, 45, 6, 13
    q = _qnet(3, A)
    obs = torch.randn(n, 3, device="cuda")

    def launch(f, lo, hi, eps):
        act, qout = torch.zeros(hi - lo, dtype=torch.int32, device="cuda"), torch.zeros(hi - lo, A, device="cuda")
        f.eps.fill_(eps)
        f(hi - lo, obs[lo:hi], act, q_out=qout, stream=_stream())
        torch.cuda.synchronize()
        return act, qout
    whole = launch(FusedDQNAct(cuda_lib, q, seed=seed), 0, n, 0.5)
    parts = [launch(FusedDQNAct(cuda_lib, q, seed=seed, env_offset=lo), lo, hi, 0.5) for lo, hi in ((0, k), (k, n))]
    assert torch.equal(torch.cat([p[0] for p in parts]), whole[0]) and torch.equal(torch.cat([p[1] for p in parts]), whole[1])
    greedy = launch(FusedDQNAct(cuda_lib, q, seed=seed), 0, n, 0.0)[0].cpu().numpy()
    f, explored = FusedDQNAct(cuda_lib, q, seed=seed), []
    for counter in range(3):
        act = launch(f, 0, n, 0.5)[0].cpu().numpy()
        assert int(f.rng[1]) == counter + 1
        u, w2 = philox_u53(seed, range(n), counter, PURPOSE_ACT)
        explore = u < 0.5
        assert np.array_equal(act[explore], ((w2[explore] * A) >> 32).astype(np.int64)) and np.array_equal(act[~explore], greedy[~explore])
        explored.append(explore)
    assert not np.array_equal(explored[0], explored[1]) and not np.array_equal(explored[1], explored[2])


def _replay_run(cuda_lib, philox_u53, rows, N, B, n_adds, seed=9, check_loop=True, prioritized=True):
    """Adds (wrapping the ring), then rounds of sample + update with the kernels, mirrored step by step on the numpy statements.  Uniform
    (``prioritized=False``): rounds of sample only, as the trainer runs them; the indices are exact, the weights 1, the trees untouched."""
    from rl_baselines.deepq import ReplayTree
    from srl_sim.policy import FusedReplay
    rep = FusedReplay(cuda_lib, rows, N, seed, 0.6, "cuda")
    loop = PrioritizedReplay(rows, N, 0.6) if check_loop else None
    vec = ReplayTree(rows, N, 0.6)
    idx, w = torch.zeros(B, dtype=torch.int64, device="cuda"), torch.zeros(B, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(seed)
    counter, stats = 0, dict(dup=0, near=0)
    for step in range(n_adds):
        row = step % rows
        rep.add(row, stream=_stream())
        vec.add(row)
        if loop:
            loop.add_row(row)
        if step >= 2:
            beta = 0.4 + 0.05 * step
            rep.beta.fill_(beta)
            trees = (rep.sum.clone(), rep.min.clone(), rep.max_priority.clone(), rep.size.clone())
            rep.sample(B, idx, w, prioritized=prioritized, stream=_stream())
            torch.cuda.synchronize()
            u, _ = philox_u53(seed, range(B), counter, PURPOSE_REPLAY)
            counter += 1
            assert int(rep.rng[1]) == counter and int(rep.rng[2]) == 0
            assert all(torch.equal(a, b) for a, b in zip(trees, (rep.sum, rep.min, rep.max_priority, rep.size)))
            ix, wv = vec.sample(u, beta, prioritized)
            if not prioritized:                      # min(floor(u n), n - 1) exactly, weights exactly 1
                assert np.array_equal(idx.cpu().numpy(), np.minimum(np.floor(u * vec.size).astype(np.int64), vec.size - 1))
                assert bool((w == 1.0).all())
                stats["dup"] += B - len(np.unique(ix))
            else:
                got_i, got_w = idx.cpu().numpy(), w.cpu().numpy()
                # an index may differ only where the mass sits within float64 rounding of the boundary between the two leaves
                bad = got_i != ix
                stats["near"] += int(bad.sum())
                if bad.any():
                    total, cap = vec.sum[1], vec.tree_cap
                    cum = np.cumsum(vec.sum[cap:cap + vec.size])
                    lo = np.minimum(got_i[bad], ix[bad])
                    assert np.all(np.abs(got_i[bad] - ix[bad]) == 1), (got_i[bad], ix[bad])
                    assert np.all(np.abs(u[bad] * total - cum[lo]) <= 1e-11 * total), np.abs(u[bad] * total - cum[lo]).max() / total
                ok = ~bad
                assert np.allclose(got_w[ok], wv[ok], rtol=1e-6, atol=0)
                if loop:
                    li, lw = loop.sample(u, beta)
                    assert np.array_equal(li[ok], ix[ok]) and np.allclose(lw[ok], wv[ok], rtol=1e-6, atol=0)
                # the batch's td: large and small, with repeated indices
                td = torch.randn(B, device="cuda", generator=g) * 2.0
                stats["dup"] += B - len(np.unique(got_i))
                rep.update(B, idx, td, 1e-6, stream=_stream())
                vec.update(got_i, td.cpu().numpy(), 1e-6)
                if loop:
                    loop.update_priorities(got_i, td.cpu().numpy(), 1e-6)
        torch.cuda.synchronize()
        s, m = rep.sum.cpu().numpy(), rep.min.cpu().numpy()
        cap = rep.tree_cap
        # the leaves: p^alpha by the device's pow against numpy's (each within an ulp or two of the exact power)
        assert np.allclose(s[cap:], vec.sum[cap:], rtol=4e-16, atol=0) and np.allclose(m[cap:], vec.min[cap:], rtol=4e-16, atol=0)
        # every internal node is op(left, right) of the kernel's own nodes, bit for bit
        k = np.arange(1, cap)
        assert np.array_equal(s[k], s[2 * k] + s[2 * k + 1]) and np.array_equal(m[k], np.minimum(m[2 * k], m[2 * k + 1]))
        # ... up to the root, which holds the float64 sum and the minimum of the leaves
        assert abs(s[1] - np.sum(s[cap:])) <= 1e-12 * s[1] and m[1] == m[cap:].min()
        assert float(rep.max_priority) == vec.max_priority and int(rep.size) == vec.size
        if loop:
            ls, lm = loop.trees()
            assert np.array_equal(vec.sum[cap:], ls[cap:]) and np.array_equal(vec.min[cap:], lm[cap:])
            assert np.array_equal(vec.sum[1:], ls[1:]) and np.array_equal(vec.min[1:], lm[1:]) and loop.max_priority == vec.max_priority
    return stats


def test_replay_kernels_match_the_segment_tree_transcription(cuda_lib, philox_u53):
    """A ring of 5 rows x 7 envs (a non-power-of-two capacity, 64 leaves), 12 adds (the ring wraps twice), batches with repeated indices;
    prioritized sampling, then uniform sampling."""
    for prioritized in (True, False):
        stats = _replay_run(cuda_lib, philox_u53, rows=5, N=7, B=50, n_adds=12, prioritized=prioritized)
        assert stats["dup"] > 0, prioritized


def test_replay_kernels_at_the_trainers_size(cuda_lib, philox_u53):
    """N envs x 1000 rows, 32 N samples per batch, prioritized then uniform: the vectorised tree of rl_baselines.deepq.  4096 x 1000
    (4 096 000 transitions) is a tree of 2^22 leaves, rebuilt in two passes (subtrees of 2048 leaves, then the level of their 2048 roots);
    8192 x 1000 is 2^23 leaves and three passes, each add (8192 leaves) spanning four 2048-leaf subtrees."""
    for N in (4096, 8192):
        for prioritized in (True, False):
            stats = _replay_run(cuda_lib, philox_u53, rows=1000, N=N, B=32 * N, n_adds=4, check_loop=False, prioritized=prioritized)
            print("\nreplay at %d x 1000 (%s): %d duplicate samples, %d indices on a float64 boundary"
                  % (N, "prioritized" if prioritized else "uniform", stats["dup"], stats["near"]))
            assert stats["dup"] > 0, (N, prioritized)


@pytest.mark.parametrize("width,n_act", Q_SHAPES)
def test_dqn_target_matches_float64_double_q(cuda_lib, width, n_act):
    """Batches of 2049 samples (one chunk of 32 per CTA at most), sms 32 3 + 17 and the trainer's 131 072 (every CTA of the persistent grid
    walks several chunks), read through idx and straight from the first rows (idx = None)."""
    from srl_sim.policy import FusedDQNTarget
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    online, target = _qnet(width, n_act, seed=1), _qnet(width, n_act, seed=2)
    fused = FusedDQNTarget(cuda_lib, online, target)
    for B in (2049, sms * 32 * 3 + 17, 131072):
        rows = 3000 if B == 2049 else B + B // 3 + 1
        g = torch.Generator(device="cuda").manual_seed(4)
        nxt = torch.randn(rows, width, device="cuda", generator=g)
        rew = torch.randn(rows, device="cuda", generator=g)
        done = (torch.rand(rows, device="cuda", generator=g) < 0.2).to(torch.uint8)
        for idx in (torch.randint(0, rows, (B,), device="cuda", generator=g), None):
            y = torch.zeros(B, device="cuda")
            fused(B, idx, nxt, rew, done, 0.99, y, stream=_stream())
            torch.cuda.synchronize()
            ix = np.arange(B) if idx is None else idx.cpu().numpy()
            want, qo = double_q_model(online, target, rew.cpu().numpy()[ix], done.cpu().numpy()[ix], nxt.cpu().numpy()[ix], 0.99)
            got = y.cpu().numpy()
            tol = 2e-5 * (np.abs(want).max() + 1.0)
            bad = np.abs(got - want) > tol
            # a flip of the online argmax is allowed only where its top two are within float32 rounding
            top2 = np.sort(qo, 1)[:, -2:]
            case = (B, "idx" if idx is not None else "no idx", int(bad.sum()), float(np.abs(got - want).max()))
            assert np.all(top2[bad, 1] - top2[bad, 0] < 1e-4 * (np.abs(qo).max() + 1.0)), case
            assert bad.sum() <= max(2, B // 1000), case


def _away_from_relu_kinks(q, obs, g):
    """Redraw the rows with a hidden pre-activation within 1e-4 of 0: there the ReLU derivative of a float32 forward pass (kernel or torch, in
    different orders of summation) may differ from float64's, a difference of a whole sample's term, not of rounding."""
    from deepq_numpy_ref import _forward, _layers
    for _ in range(20):
        x = obs.double().cpu().numpy()
        near = np.zeros(len(x), bool)
        for tower in (q.pi, q.vf):
            for pre in _forward(_layers(tower), x)[1][:2]:
                near |= (np.abs(pre) < 1e-4).any(1)
        if not near.any():
            return obs
        rows = torch.from_numpy(np.nonzero(near)[0]).cuda()
        obs[rows] = torch.randn((len(rows), obs.shape[1]), device="cuda", generator=g)
    raise AssertionError("could not draw rows away from the ReLU kinks")


def _dqn_grads(q, d, idx, rows=None):
    from rl_baselines.deepq import dqn_loss
    q = copy.deepcopy(q)
    dt = next(q.parameters()).dtype
    sel = idx if rows is None else idx[:rows]
    n = len(sel)
    loss, td = dqn_loss(q, d["obs"][sel].to(dt), d["act"][sel], d["y"][:n].to(dt), d["w"][:n].to(dt))
    loss.backward()
    return [p.grad.detach().clone() for p in q.parameters()], td


@pytest.mark.parametrize("use_idx", [True, False], ids=["idx", "no_idx"])
@pytest.mark.parametrize("size", ["1", "33", "3_chunks_per_cta", "131072"])
@pytest.mark.parametrize("width,n_act", Q_SHAPES)
def test_dqn_grad_matches_float64_autograd(cuda_lib, width, n_act, size, use_idx):
    from srl_sim.policy import FusedDQNGrad
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = sms * CH * 3 + 17 if size == "3_chunks_per_cta" else int(size)
    rows = B + B // 3 + 1 if use_idx else B + 5
    q = _qnet(width, n_act)
    g = torch.Generator(device="cuda").manual_seed(B + width)
    obs = _away_from_relu_kinks(q, torch.randn(rows, width, device="cuda", generator=g), g)
    act = torch.randint(0, n_act, (rows,), device="cuda", generator=g)
    idx = torch.randperm(rows, device="cuda", generator=g)[:B].contiguous() if use_idx else None
    ref_idx = idx if use_idx else torch.arange(B, device="cuda")
    with torch.no_grad():
        qa = q(obs[ref_idx]).gather(1, act[ref_idx, None])[:, 0]
    # td spread over both Huber branches; weights away from 1
    y = (qa + 1.5 * torch.randn(B, device="cuda", generator=g)).contiguous()
    w = (0.2 + torch.rand(B, device="cuda", generator=g)).contiguous()
    d = dict(obs=obs, act=act, y=y, w=w)
    want, td64 = _dqn_grads(copy.deepcopy(q).double(), d, ref_idx)
    f32 = grad_errors(_dqn_grads(q, d, ref_idx)[0], want)
    fused = FusedDQNGrad(cuda_lib, q, B)
    td = torch.zeros(B, device="cuda")
    fused(idx, obs, act, y, w, td, stream=_stream())
    torch.cuda.synchronize()
    got = [p.grad.detach().clone() for p in q.parameters()]
    kern = grad_errors(got, want)
    names = [n for n, _ in q.named_parameters()]
    print("\ndqn_grad %s B=%d %s  max|g - g64| / max|g64|  kernel | float32 autograd:" % ((width, n_act), B, "idx" if use_idx else "no idx"))
    print("  " + "  ".join("%s %.1e|%.1e" % (n, e / s, e32 / s) for n, (e, s), (e32, _) in zip(names, kern, f32)))
    for n, (err, scale), (e32, _) in zip(names, kern, f32):
        assert scale > 0 and err <= grad_bound(scale) + 4.0 * e32, (n, err, e32, scale)
    assert float((td.double() - td64).abs().max()) <= 2e-5 * (float(td64.abs().max()) + 1.0)
    if B > 1:
        assert (td64.abs() < 1).any() and (td64.abs() > 1).any()
    if size == "131072":
        td2 = torch.zeros_like(td)
        fused(idx, obs, act, y, w, td2, stream=_stream())
        torch.cuda.synchronize()
        assert all(torch.equal(p.grad, a) for p, a in zip(q.parameters(), got)) and torch.equal(td, td2)
    plain = copy.deepcopy(q)                 # without the kernel's .grad tensors, into which a reference's backward would accumulate
    for p in plain.parameters():
        p.grad = None
    if size in ("33", "3_chunks_per_cta"):
        # weights = NULL, as the trainer passes without prioritized replay: the bytes of all-ones weights, and float64 autograd with w = 1
        ones, out = torch.ones(B, device="cuda"), []
        for wt in (None, ones):
            fused(idx, obs, act, y, wt, td, stream=_stream())
            torch.cuda.synchronize()
            out.append([p.grad.detach().clone() for p in q.parameters()] + [td.clone()])
        assert all(torch.equal(a, b) for a, b in zip(*out))
        d1 = dict(d, w=ones)
        want1, td1 = _dqn_grads(copy.deepcopy(plain).double(), d1, ref_idx)
        f32_1 = grad_errors(_dqn_grads(plain, d1, ref_idx)[0], want1)
        for n, (err, scale), (e32, _) in zip(names, grad_errors(out[0][:-1], want1), f32_1):
            assert scale > 0 and err <= grad_bound(scale) + 4.0 * e32, ("w = None", n, err, e32, scale)
        assert float((out[0][-1].double() - td1).abs().max()) <= 2e-5 * (float(td1.abs().max()) + 1.0)
    if size == "33":
        wrong = grad_errors(got, _dqn_grads(copy.deepcopy(plain).double(), d, ref_idx, rows=B - 1)[0])
        margin = max(err / grad_bound(scale) for err, scale in wrong)
        print("  without the last row the float64 reference is %.0f x the tolerance away from the kernel" % margin)
        assert margin > 10.0


@pytest.mark.parametrize("clip", [0.05, 1e3], ids=["clipped", "unclipped"])
@pytest.mark.parametrize("width,n_act", [(3, 6), (32, 2)])
def test_clip_adam_matches_the_float64_tf_model(cuda_lib, width, n_act, clip):
    from srl_sim.policy import FusedClipAdam, policy_params
    q = _qnet(width, n_act)
    params = policy_params(q)
    for p in params:
        p.grad = torch.zeros_like(p)
    start = [p.detach().clone() for p in params]
    runs = []
    for rep in range(2):
        with torch.no_grad():
            for p, s in zip(params, start):
                p.copy_(s)
        opt = FusedClipAdam(cuda_lib, q, clip)
        opt.lr.fill_(1e-3)
        p64 = [s.double().cpu().numpy() for s in start]
        m64, v64 = [np.zeros(s.shape) for s in start], [np.zeros(s.shape) for s in start]
        g = torch.Generator(device="cuda").manual_seed(21)
        for step in range(1, 101):
            for p in params:
                p.grad.copy_(torch.randn(p.shape, device="cuda", generator=g) * 0.05)
            if rep == 0:
                norms = [float(torch.sqrt((p.grad.double() ** 2).sum())) for p in params]
                assert (max(norms) > clip) == (clip == 0.05)
                p64, m64, v64 = clip_adam_model(p64, [p.grad.cpu().numpy() for p in params], m64, v64, step, float(np.float32(1e-3)), clip,
                                                float(np.float32(0.9)), float(np.float32(0.999)), float(np.float32(1e-8)))
            opt(stream=_stream())
        torch.cuda.synchronize()
        runs.append([p.detach().clone() for p in params] + [t.clone() for t in opt.m + opt.v])
        if rep == 0:
            for p, w in zip(params, p64):
                # 100 steps of about lr each, every one rounded in float32
                assert np.abs(p.detach().double().cpu().numpy() - w).max() <= 1e-3 * 100 * 2e-5 + 100 * 2.0 ** -23 * (np.abs(w).max() + 1.0)
            for mm, w in zip(opt.m, m64):
                assert np.abs(mm.double().cpu().numpy() - w).max() <= 1e-5 * (np.abs(w).max() + 1e-6)
    assert all(torch.equal(a, b) for a, b in zip(*runs))


@pytest.mark.parametrize("bad", [float("inf"), float("nan")], ids=["inf", "nan"])
def test_clip_adam_non_finite_gradient_stays_in_its_tensor(cuda_lib, bad):
    """tf.clip_by_norm of a tensor with an inf entry: that entry NaN, the others 0; with a NaN entry: all NaN.  Other tensors step normally.
    The torch statement of rl_baselines.deepq agrees."""
    from rl_baselines.deepq import clip_adam
    from srl_sim.policy import FusedClipAdam, policy_params
    q = _qnet(3, 6)
    params = policy_params(q)
    for p in params:
        p.grad = torch.randn(p.shape, device="cuda") * 0.05
    params[0].grad[0, 0] = bad
    ref = copy.deepcopy(q)
    rp = policy_params(ref)
    for p, r in zip(params, rp):
        r.grad = p.grad.clone()
    opt = FusedClipAdam(cuda_lib, q, 10.0)
    opt.lr.fill_(1e-4)
    opt(stream=_stream())
    clip_adam(rp, [torch.zeros_like(p) for p in rp], [torch.zeros_like(p) for p in rp], torch.tensor([0.9, 0.999], device="cuda"), 1e-4, 10.0,
              0.9, 0.999, 1e-8)
    torch.cuda.synchronize()
    w0 = params[0].detach()
    if bad == float("inf"):
        assert torch.isnan(w0[0, 0]) and int(torch.isnan(w0).sum()) == 1
    else:
        assert torch.isnan(w0).all()
    for p, r in zip(params, rp):
        assert torch.equal(torch.isnan(p), torch.isnan(r))
        assert torch.isfinite(p).all() or p is params[0]


def test_deepq_learns_mobile_robot(cuda_lib):
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.deepq import train
    hist = train("MobileRobotGymEnv-v0", 1024, 1024 * 4000, seed=0, env_kwargs=dict(is_discrete=True, shape_reward=True), verbose=0)
    rets = [h[1] for h in hist if np.isfinite(h[1])]
    print("\nDQN MobileRobot: first window %.1f, last %.1f, fps %.0f, %s" % (rets[0], rets[-1], hist[-1][2], train.stats))
    # shaped reward = -distance per step over 251 steps; measured on an H100: -699 in the first window, -419 in the last
    assert rets[-1] > rets[0] + 150, rets[::50]
    assert train.stats["graph_replays"] > 0


@pytest.mark.parametrize("env_id,num_stack,train_freq", [("MobileRobotGymEnv-v0", 1, 4), ("KukaButtonGymEnv-v0", 1, 4), ("MobileRobotGymEnv-v0", 3, 4),
                                                       ("MobileRobotGymEnv-v0", 1, 3)])
def test_captured_and_eager_runs_agree(cuda_lib, env_id, num_stack, train_freq):
    """The same run with its blocks replayed from CUDA graphs (one per ring phase) and launched eagerly: the same bytes in the parameters, the
    target network, both trees, max_priority and the Adam slots.  A ring of 12 rows makes the phases repeat; train_freq 3 runs blocks of 6 steps
    (an even number of MobileRobot launches per replay); the target copy falls inside blocks and between the gradient steps of a 6-step block."""
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.deepq import train
    hp = dict(learning_starts=20, target_network_update_freq=25 if train_freq == 3 else 24, buffer_size=12, train_freq=train_freq, batch_size=8)
    out, stats = [], []
    for graph in (True, False):
        train(env_id, 256, 256 * 100, seed=5, env_kwargs=dict(is_discrete=True, shape_reward=True), verbose=0, hyperparams=hp, cuda_graph=graph,
              num_stack=num_stack)
        rep, (m, v, bp) = train.last_replay, train.last_adam
        out.append([p.detach().clone() for p in train.last_policy.parameters()] + [p.detach().clone() for p in train.last_target.parameters()] +
                   [rep.sum.clone(), rep.min.clone(), rep.max_priority.clone(), rep.size.clone(), bp.clone()] + [t.clone() for t in m + v])
        stats.append(dict(train.stats))
    print("\ncaptured %s, eager %s" % (stats[0], stats[1]))
    assert stats[0]["graph_replays"] > 0 and 0 < stats[0]["graphs"] <= 3 and stats[1]["graph_replays"] == 0
    assert stats[0]["grad_steps"] == stats[1]["grad_steps"] > 0 and stats[0]["target_copies"] == stats[1]["target_copies"] > 0
    assert all(torch.equal(a, b) for a, b in zip(*out))
    rep = train.last_replay
    leaves = rep.sum[rep.tree_cap:rep.tree_cap + int(rep.size)]
    assert torch.unique(leaves).numel() > 1                       # the priorities were written back (new transitions all enter at max_priority^alpha)


@pytest.mark.parametrize("env_id", ["KukaButtonGymEnv-v0", "KukaRandButtonGymEnv-v0", "Kuka2ButtonGymEnv-v0", "KukaMovingButtonGymEnv-v0",
                                    "MobileRobotGymEnv-v0", "MobileRobot2TargetGymEnv-v0", "MobileRobot1DGymEnv-v0", "MobileRobotLineTargetGymEnv-v0"])
def test_train_entry_point_runs_deepq_for_every_env(env_id, cuda_lib, tmp_path):
    from srl_sim import backend
    backend.use_library(None, None)
    from rl_baselines.train import main
    hist = main(["--algo", "deepq", "--env", env_id, "--num-cpu", "64", "--num-timesteps", "64000", "--log-dir", str(tmp_path),
                 "--hyperparam", "learning_starts:100", "--buffer-size", "200"])
    assert len(hist) == (int(1.1 * 64000) // 64 + 3) // 4 and all(np.isfinite(h[2]) for h in hist)
