"""distractor_kernel on the H100 against float64 references on the handle's own inputs, and the bodies' structural invariants.

The chain of evidence: tests/test_distractor_reference_cpu.py holds csrc/distractor_core.h in float64 (libdistractor_ref.so) to the
independent numpy model of tests/distractor_numpy_ref.py to 1e-9 in every branch.  Here the kernel is driven through the library, and the
float64 side replays EXACTLY the micro-steps the kernel replayed -- the launch's trace and the handle's settle trajectory, read through the
SRL_F_DISTRACTOR_* test hooks; arm spheres recomputed in float64 from the traced joint angles with srl_sim.model's numpy forward
kinematics; placement and kick from a numpy restatement of the counter-based draws.  All envs are replayed with the float64 header (fast),
a few with the numpy model directly (a pure-Python Gauss-Seidel: ~20 s per settle).

float32 against float64 through contact is not bit-comparable, and errors accumulate along a trajectory, so the step phase is compared
LAUNCH BY LAUNCH from the device's own records: before each lockstep step the float64 side starts from the float32 records the kernel
starts from, and is compared with the records after it.  That keeps the tolerance at float32 rounding through one to three micro-steps
instead of a trajectory's drift; fused rollouts are tied to lockstep steps byte for byte.  A reset's 505 micro-steps are one launch: there
bodies that tip over an edge may fall differently, and the fraction that does is bounded and printed.  The numbers in the asserts are
set from the printed figures of a run on one H100 80GB HBM3 (see DESIGN.md section 3)."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "robotics-rl-srl_b200")
for p in (PKG, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import distractor_numpy_ref as ref  # noqa: E402

pytestmark = pytest.mark.gpu

RB = "KukaRandButtonGymEnv-v0"
DT_FIRST, DT_HOST_DRAWS, DT_KICK = 2, 4, 8
DT = 1.0 / 240.0


@pytest.fixture(scope="module")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from srl_sim._abi import load_cuda_library
    from srl_sim.backend import Backend
    return Backend(load_cuda_library(), 0)


@pytest.fixture(scope="module")
def philox(oracle_lib):
    fn = oracle_lib.lib.oracle_philox4x32
    fn.argtypes = [ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32)]
    fn.restype = None

    def words(seed, env, index, purpose):
        out = (ctypes.c_uint32 * 4)()
        fn(seed, env, index, purpose, out)
        return list(out)
    return words


@pytest.fixture(scope="module")
def checker():
    lib = ctypes.CDLL(os.path.join(PKG, "csrc", "libdistractor_ref.so"))
    P = ctypes.c_void_p
    lib.dref_run_steps.argtypes = [P, ctypes.c_size_t, P, ctypes.c_double, ctypes.c_int, ctypes.c_double, P, P, ctypes.c_int, ctypes.c_int, P, P, P,
                                   P, P]
    lib.dref_run_steps.restype = ctypes.c_int
    return lib


def _sim(be, n, seed=0, bodies=True, **cfg):
    from srl_sim.model import distractor_blob, load_kuka_scene
    s = be.make_sim(RB, n, seed=seed, model_blob=load_kuka_scene().blob, **cfg)
    if bodies:
        s.set_distractors(distractor_blob())
    return s


def _records(s):
    from srl_sim import _abi
    return s.get_state(_abi.F_DISTRACTOR_RECORDS).reshape(s.num_envs, 11, 16)


def _touch(s):
    from srl_sim import _abi
    return s.get_state(_abi.F_DISTRACTOR_TOUCH).astype(np.int64) & 0xFFFFFFFF


class Replayer(object):
    """Float64 replay of trace records for one handle."""

    def __init__(self, checker, philox, seed, offset=0):
        from srl_sim.model import distractor_blob, load_kuka_scene, scene_constants
        self.lib, self.philox, self.seed, self.offset = checker, philox, seed, offset
        self.blob = distractor_blob()
        self.model = load_kuka_scene()
        self.c = scene_constants(self.model)
        assert len(self.model.spheres) <= 16
        self._fk = {}

    def arm(self, rec):
        """f64[narm, 4] world collision spheres of the arm at the traced joint angles."""
        key = rec[:12].tobytes()
        if key not in self._fk:
            P, R = self.model.forward_kinematics(rec[:12].astype(np.float64))
            self._fk[key] = np.array([list(P[bi] + R[bi] @ np.asarray(c, np.float64)) + [rad] for bi, c, rad in self.model.spheres], np.float64)
        return self._fk[key]

    def scene(self, bx, by):
        c = self.c
        return np.array([c["table_z"], c["txmin"], c["txmax"], c["tymin"], c["tymax"], bx, by, c["button_z"], c["stack_top"], c["stack_r"],
                         c["disc_r"], 0.0, 0.0], np.float64)

    def disc(self, qb):
        c = self.c
        z = c["button_z"] + c["glider_z"] + float(qb)
        return [z + c["disc_z0"], z + c["disc_z1"]]

    def segment(self, B, touch, recs, kicks, numpy_model=False):
        """Advance B through the records `recs` (one scene: the same button base) in one call."""
        n = len(recs)
        arm = np.ascontiguousarray(np.stack([self.arm(r) for r in recs]))
        disc = np.array([self.disc(r[12]) for r in recs], np.float64)
        sc = self.scene(float(recs[0][13]), float(recs[0][14]))
        if numpy_model:
            traj, tb, ta, _ = ref.run(self.blob, ref.Scene.from_array(sc, dt=DT, iters=150, margin=0.02), B, n, arm=arm, disc=disc, kicks=kicks)
            B[:] = traj[-1]
            touch[0] |= tb
            touch[1] |= ta
            return
        kv, ko = np.zeros((n, 3)), np.zeros(n, np.uint8)
        for m, j in kicks.items():
            kv[m], ko[m] = j, 1
        t = np.zeros(2, np.uint32)
        rc = self.lib.dref_run_steps(self.blob.ctypes.data, self.blob.nbytes, sc.ctypes.data, DT, 150, 0.02, B.ctypes.data, arm.ctypes.data,
                                     arm.shape[1], n, disc.ctypes.data, kv.ctypes.data, ko.ctypes.data, None, t.ctypes.data)
        assert rc == 0
        touch[0] |= int(t[0])
        touch[1] |= int(t[1])

    def launch(self, env, B, touch, recs, tags, settle, draws=None, numpy_model=False):
        """What distractor_kernel does with one env's trace of one launch.  B f64[11,16] and touch [body, arm] are updated in place.
        Returns the placements made: [(micro-step, records right after placement)]."""
        placed = []
        start = 0
        kicks = {}
        genv = self.offset + env
        for m in range(len(recs)):
            tag = int(tags[m])
            if tag & DT_FIRST:
                if m > start:
                    self.segment(B, touch, recs[start:m], kicks, numpy_model)
                start, kicks = m, {}
                if tag & DT_HOST_DRAWS:
                    xy, types = draws[18:38], draws[38:48].astype(int)
                else:
                    xy, types = ref.stream_placement(self.philox, self.seed, genv, tag >> 4)
                B[:] = ref.place(xy, types, float(recs[m][13]), float(recs[m][14]))
                placed.append((m, B.copy()))
                touch[0] = touch[1] = 0
                srecs = settle.copy()
                srecs[:, 13:15] = recs[m][13:15]
                self.segment(B, touch, srecs, {}, numpy_model)
            if tag & DT_KICK:
                kicks[m - start] = ref.stream_kick(self.philox, self.seed, genv, tag >> 4, DT)
        if len(recs) > start:
            self.segment(B, touch, recs[start:], kicks, numpy_model)
        return placed


def _errors(dev, B):
    """Per body: position error (m), rotation error (rad), v and w error; for present bodies."""
    present = B[:, 14] != 0
    dq = np.abs(np.sum(dev[:, 3:7] * B[:, 3:7], axis=1)).clip(0, 1)
    return present, np.abs(dev[:, 0:3] - B[:, 0:3]).max(axis=1), 2 * np.arccos(dq), np.abs(dev[:, 7:10] - B[:, 7:10]).max(axis=1), \
        np.abs(dev[:, 10:13] - B[:, 10:13]).max(axis=1)


def _physical(rec, table_z, tx, ty):
    """The set no body may leave: finite, unit quaternion, 0/1 flags, not under the table top while over the table."""
    assert np.isfinite(rec).all()
    pres = rec[..., 14] != 0
    assert np.isin(rec[..., 14], (0.0, 1.0)).all() and np.isin(rec[..., 13], (0.0, 1.0, 2.0, 3.0)).all()
    qn = np.linalg.norm(rec[..., 3:7].astype(np.float64), axis=-1)
    assert np.abs(qn[pres] - 1).max() < 1e-5
    over = pres & (rec[..., 0] >= tx[0]) & (rec[..., 0] <= tx[1]) & (rec[..., 1] >= ty[0]) & (rec[..., 1] <= ty[1])
    # the COM of every type is at least its smallest sphere radius (9.5 mm) above what its spheres rest on
    assert (rec[..., 2][over] > table_z - 0.02).all()


def _host_draws(n, seed):
    rng = np.random.RandomState(seed)
    d = np.zeros((n, 48), np.float64)
    d[:, 0] = 0.5
    d[:, 18:38:2] = 0.5 + 0.15 * rng.uniform(-1, 1, size=(n, 10))
    d[:, 19:38:2] = 0.3 * rng.uniform(-1, 1, size=(n, 10))
    d[:, 38:] = rng.randint(3, size=(n, 10))
    return d


def _report(title, types, pos, rot, tol_pos):
    names = ("duck", "lego", "cube", "sphere")
    for t in range(4):
        e, r = pos[types == t], rot[types == t]
        if e.size:
            print("%s %-6s bodies %4d  |dpos| max %.3g median %.3g m  rot max %.3g median %.3g rad  diverged (> %.1g m) %.1f %%"
                  % (title, names[t], e.size, e.max(), np.median(e), r.max(), np.median(r), tol_pos, 100.0 * (e > tol_pos).mean()))


# ---- reset ---------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("host_draws", [False, True])
def test_reset_placement_and_settle_against_float64(cuda, checker, philox, host_draws):
    n, seed = 64, 5
    s = _sim(cuda, n, seed=seed, is_discrete=True, no_auto_reset=True, random_target=not host_draws)
    draws = _host_draws(n, 1) if host_draws else None
    s.reset(reset_draws=None if draws is None else cuda.from_host(draws), stream=cuda.stream())
    dev, touch_dev = _records(s), _touch(s)
    length, trace, tags, settle = s.distractor_trace()
    assert (length == 5).all() and ((tags[:, 0] & DT_FIRST) != 0).all() and (((tags[:, 0] & DT_HOST_DRAWS) != 0) == host_draws).all()
    rp = Replayer(checker, philox, seed)
    pos, rot, types, touched, mism = [], [], [], [], 0
    for i in range(n):
        B, touch = np.zeros((11, 16)), [0, 0]
        placed = rp.launch(i, B, touch, trace[i, :5], tags[i, :5], settle, None if draws is None else draws[i])
        # placement: types and presence exactly, positions as the float32 of the float64 draws
        P0 = placed[0][1]
        assert np.array_equal(dev[i, :, 13:15], P0[:, 13:15].astype(np.float32)), i
        if i < 2:            # the numpy model itself on the same inputs
            Bm, tm = np.zeros((11, 16)), [0, 0]
            rp.launch(i, Bm, tm, trace[i, :5], tags[i, :5], settle, None if draws is None else draws[i], numpy_model=True)
            pm = Bm[:, 14] != 0
            # 505 micro-steps through landings amplify the last-bit differences of the two formulations (1e-9 over the CPU scenarios'
            # <= 260 micro-steps) to ~1e-7; a body that lands balanced on an edge (the cube on two of its spheres) is an unstable
            # equilibrium that grows them by e^(22/s x 2 s), so a body, or a pair in contact, may differ visibly (seen: two touching bodies of one env by 1.5e-3)
            err = np.abs(Bm[pm, :13] - B[pm, :13]).max(axis=1)
            print("env %d, numpy model against the float64 header after 505 micro-steps: per body %s" % (i, np.array2string(err, precision=1)))
            assert np.median(err) < 1e-7 and (err > 1e-5).sum() <= 2 and err.max() < 5e-3, "numpy model and float64 header differ on env %d" % i
            assert tm == touch
        present, ep, er, _, _ = _errors(dev[i].astype(np.float64), B)
        pos += list(ep[present]); rot += list(er[present]); types += list(B[present, 13].astype(int))
        both = (int(touch_dev[i, 0]) | int(touch_dev[i, 1]) | touch[0] | touch[1])
        touched += [bool((both >> k) & 1) for k in np.flatnonzero(present)]
        mism += bin(int(touch_dev[i, 0]) ^ touch[0]).count("1") + bin(int(touch_dev[i, 1]) ^ touch[1]).count("1")
    pos, rot, types, touched = np.array(pos), np.array(rot), np.array(types), np.array(touched)
    _report("reset%s all    " % ("/host" if host_draws else ""), types, pos, rot, 1e-3)
    _report("reset%s touched" % ("/host" if host_draws else ""), types[touched], pos[touched], rot[touched], 1e-3)
    print("touch-mask bits that differ: %d of %d bodies" % (mism, pos.size))
    c = rp.c
    _physical(dev, c["table_z"], (c["txmin"], c["txmax"]), (c["tymin"], c["tymax"]))
    assert touched.sum() >= 20, "too few bodies in contact with another body or the arm to say anything"
    stable = (types == 1) | (types == 3)
    # measured: median 2e-8 ... 5e-7 m per type; beyond 1 mm (a body that tipped or was pushed differently): ball 0 %, brick 0.6 %, duck 4.8 %,
    # the tetrahedral cube 16 %
    assert np.median(pos) < 1e-5
    assert (pos[stable] > 1e-3).mean() < 0.05 and (pos[~stable] > 1e-3).mean() < 0.25
    assert mism <= 0.05 * pos.size


# ---- the step phase, launch by launch ------------------------------------------------------------------------------------------------

def _lockstep_against_float64(cuda, checker, philox, s, seed, T, discrete, crafted=None, label=""):
    import torch
    n = s.num_envs
    rp = Replayer(checker, philox, seed)
    c = rp.c
    rng = np.random.RandomState(seed)
    obs, rew, done = cuda.zeros((n, 3), np.float32), cuda.zeros((n,), np.float32), cuda.zeros((n,), np.uint8)
    before, touch_before = _records(s), _touch(s)
    stats = {"pos": [], "rot": [], "v": [], "w": [], "settle_pos": []}
    kicks = resets = touch_mism = contact_launches = 0
    for t in range(T):
        a = rng.randint(0, 6, size=n).astype(np.int32) if discrete else rng.uniform(-1, 1, size=(n, 3)).astype(np.float32)
        s.step(cuda.from_host(a), obs_out=obs, rew_out=rew, done_out=done, stream=cuda.stream())
        torch.cuda.synchronize()
        after, touch_after = _records(s), _touch(s)
        length, trace, tags, settle = s.distractor_trace()
        assert (length >= 1).all() and (length <= s.cfg.action_repeat + 5).all()
        _physical(after, c["table_z"], (c["txmin"], c["txmax"]), (c["tymin"], c["tymax"]))
        for i in range(n):
            L = int(length[i])
            B = before[i].astype(np.float64)
            touch = [int(touch_before[i, 0]), int(touch_before[i, 1])]
            placed = rp.launch(i, B, touch, trace[i, :L], tags[i, :L], settle)
            kicks += int(((tags[i, :L] & DT_KICK) != 0).sum())
            present, ep, er, ev, ew = _errors(after[i].astype(np.float64), B)
            if placed:
                resets += 1
                assert np.array_equal(after[i, :, 13:15], placed[0][1][:, 13:15].astype(np.float32))
                stats["settle_pos"] += list(ep[present])
            else:
                stats["pos"] += list(ep[present]); stats["rot"] += list(er[present]); stats["v"] += list(ev[present]); stats["w"] += list(ew[present])
                contact_launches += int((touch[0] | touch[1]) != 0)
            touch_mism += bin(int(touch_after[i, 0]) ^ touch[0]).count("1") + bin(int(touch_after[i, 1]) ^ touch[1]).count("1")
        before, touch_before = after, touch_after
    st = {k: np.array(v) for k, v in stats.items()}
    print("%s: %d body-launches, |dpos| max %.3g median %.3g m, rot max %.3g rad, |dv| max %.3g median %.3g m/s, |dw| max %.3g median %.3g rad/s; "
          "%d resets in the rollout (settle |dpos| median %.3g m, > 1 mm %.1f %%), %d kicks, touch bits that differ %d"
          % (label, st["pos"].size, st["pos"].max(), np.median(st["pos"]), st["rot"].max(), st["v"].max(), np.median(st["v"]), st["w"].max(),
             np.median(st["w"]), resets, np.median(st["settle_pos"]) if resets else 0.0, 100.0 * (st["settle_pos"] > 1e-3).mean() if resets else 0.0,
             kicks, touch_mism))
    return st, kicks, resets, touch_mism


@pytest.mark.parametrize("discrete,repeat,n", [(True, 1, 64), (False, 3, 96)])
def test_lockstep_steps_against_float64_launch_by_launch(cuda, checker, philox, discrete, repeat, n):
    seed, T = 3 + repeat, 150
    s = _sim(cuda, n, seed=seed, is_discrete=discrete, action_repeat=repeat, random_target=True, max_steps=60)
    s.reset(stream=cuda.stream())
    st, kicks, resets, touch_mism = _lockstep_against_float64(cuda, checker, philox, s, seed, T, discrete, label="lockstep r%d" % repeat)
    assert resets >= n, "every env should have reset inside the rollout at least once"
    # the kick fires at env step 10 of every episode with action_repeat 1, and never with 3 (the counter is not 10 at a step's start)
    assert (kicks >= n) if repeat == 1 else (kicks == 0)
    # one to three micro-steps from the same float32 state: float32 rounding through the solve
    assert st["pos"].max() < 2e-4 and np.median(st["pos"]) < 1e-6
    assert st["v"].max() < 5e-2 and np.median(st["v"]) < 1e-4
    assert (st["settle_pos"] > 1e-3).mean() < 0.30
    assert touch_mism <= 0.01 * st["pos"].size


def test_crafted_starts_through_the_writable_records(cuda, checker, philox):
    """A stack, a ball beside the button, a ball on the disc, a brick under the gripper, a tight pile: written through
    SRL_F_DISTRACTOR_RECORDS, then stepped and compared launch by launch."""
    from srl_sim import _abi
    n, seed = 16, 9
    s = _sim(cuda, n, seed=seed, is_discrete=True, no_auto_reset=True)
    s.reset(stream=cuda.stream())
    rp = Replayer(checker, philox, seed)
    tz, bz = rp.c["table_z"], rp.c["button_z"]
    ee = s.get_state(_abi.F_EE_POS)
    rec = np.zeros((n, 11, 16), np.float32)
    rec[:, :, 6] = 1.0

    def put(i, slot, t, pos, v=(0, 0, 0)):
        rec[i, slot, 0:3], rec[i, slot, 7:10], rec[i, slot, 13], rec[i, slot, 14] = pos, v, t, 1.0
    for i in range(n):
        k = i % 4
        put(i, 10, 3, (0.25, -0.2, tz + 0.03))
        if k == 0:      # a brick on a brick, and a ball rolling into them
            put(i, 2, 1, (0.3, 0.2, tz + 0.0095)); put(i, 5, 1, (0.302, 0.201, tz + 0.0295)); put(i, 7, 3, (0.22, 0.2, tz + 0.03), (0.5, 0, 0))
        elif k == 1:    # balls against the button's stack and on its disc
            put(i, 0, 3, (0.5 - rp.c["stack_r"] - 0.04, 0.01, tz + 0.03), (0.4, 0, 0)); put(i, 1, 3, (0.52, 0.01, bz + 0.2))
        elif k == 2:    # a brick and a cube right under the gripper, which the arm comes down on
            put(i, 3, 1, (ee[i, 0], ee[i, 1], tz + 0.0095)); put(i, 4, 2, (ee[i, 0] + 0.03, ee[i, 1] + 0.02, tz + 0.025))
        else:           # a tight 3 x 3 pile of bricks with a duck on top: more than 48 contacts in one island
            for j in range(9):
                put(i, j, 1, (0.3 + 0.036 * (j % 3), -0.25 + 0.036 * (j // 3), tz + 0.0105))
            put(i, 9, 0, (0.336, -0.214, tz + 0.06))
    s.set_state(_abi.F_DISTRACTOR_RECORDS, rec.reshape(n, -1))
    assert np.array_equal(_records(s), rec)
    rng = np.random.RandomState(0)
    import torch
    obs, rew, done = cuda.zeros((n, 3), np.float32), cuda.zeros((n,), np.float32), cuda.zeros((n,), np.uint8)
    before, tb = _records(s), _touch(s)
    pos, vel, contact = [], [], 0
    for t in range(120):
        a = np.where(np.arange(n) % 4 == 2, 5, rng.randint(0, 6, size=n)).astype(np.int32)      # action 5: down
        s.step(cuda.from_host(a), obs_out=obs, rew_out=rew, done_out=done, stream=cuda.stream())
        torch.cuda.synchronize()
        after, ta = _records(s), _touch(s)
        length, trace, tags, settle = s.distractor_trace()
        for i in range(n):
            B, touch = before[i].astype(np.float64), [0, 0]
            assert not rp.launch(i, B, touch, trace[i, :int(length[i])], tags[i, :int(length[i])], settle)
            present, ep, er, ev, ew = _errors(after[i].astype(np.float64), B)
            pos += list(ep[present]); vel += list(ev[present])
            contact += int(touch[0] != 0)
        before, tb = after, ta
    pos, vel = np.array(pos), np.array(vel)
    print("crafted starts: %d body-launches (%d env-launches with body-body contact), |dpos| max %.3g median %.3g m, |dv| max %.3g median %.3g m/s"
          % (pos.size, contact, pos.max(), np.median(pos), vel.max(), np.median(vel)))
    assert contact > 200
    print("envs whose bodies touched the arm: %d" % int((ta[:, 1] != 0).sum()))
    assert int(ta[:, 0].max()) != 0
    assert pos.max() < 2e-4 and vel.max() < 5e-2


def test_writable_records_refuse_invalid_input(cuda):
    from srl_sim import _abi
    s = _sim(cuda, 4, is_discrete=True)
    s.reset(stream=cuda.stream())
    good = _records(s).copy()
    for word, value, msg in ((14, 2.0, "present"), (13, 4.0, "type"), (13, 1.5, "type"), (3, 0.5, "quaternion"), (0, np.nan, "non-finite"), (8, np.inf, "non-finite")):
        bad = good.copy()
        bad[1, 3, word] = value
        with pytest.raises(_abi.SimError, match=msg):
            s.set_state(_abi.F_DISTRACTOR_RECORDS, bad.reshape(4, -1))
        assert np.array_equal(_records(s), good)
    plain = _sim(cuda, 4, bodies=False, is_discrete=True)
    with pytest.raises(_abi.SimError, match="set_distractors"):
        plain.get_state(_abi.F_DISTRACTOR_RECORDS)
    with pytest.raises(_abi.SimError, match="set_distractors"):
        plain.set_state(_abi.F_DISTRACTOR_RECORDS, good.reshape(4, -1))


# ---- structural invariants, byte for byte --------------------------------------------------------------------------------------------

def _rollout(cuda, s, T, actions=None):
    import torch
    n = s.num_envs
    o = [cuda.zeros((T, n, 3), np.float32), cuda.zeros((T, n), np.float32), cuda.zeros((T, n), np.uint8)]
    s.rollout(T, actions=actions, obs_out=o[0], rew_out=o[1], done_out=o[2], stream=cuda.stream())
    torch.cuda.synchronize()
    return [cuda.to_host(x).copy() for x in o]


@pytest.mark.parametrize("discrete,repeat", [(True, 1), (False, 3)])
def test_lockstep_steps_equal_one_rollout(cuda, discrete, repeat):
    import torch
    n, T, seed = 96, 300, 2
    rng = np.random.RandomState(1)
    acts = rng.randint(0, 6, size=(T, n)).astype(np.int32) if discrete else rng.uniform(-1, 1, size=(T, n, 3)).astype(np.float32)
    cfg = dict(seed=seed, is_discrete=discrete, action_repeat=repeat, random_target=True, max_steps=60)
    a = _sim(cuda, n, **cfg)
    a.reset(stream=cuda.stream())
    out = _rollout(cuda, a, T, cuda.from_host(acts))
    assert out[2].sum() > 3 * n
    b = _sim(cuda, n, **cfg)
    b.reset(stream=cuda.stream())
    obs, rew, done = cuda.zeros((n, 3), np.float32), cuda.zeros((n,), np.float32), cuda.zeros((n,), np.uint8)
    for t in range(T):
        b.step(cuda.from_host(acts[t]), obs_out=obs, rew_out=rew, done_out=done, stream=cuda.stream())
    torch.cuda.synchronize()
    assert _records(a).tobytes() == _records(b).tobytes()
    assert _touch(a).tobytes() == _touch(b).tobytes()


def test_packing_and_sharding_give_each_env_the_same_bytes(cuda):
    T, seed = 40, 4
    cfg = dict(seed=seed, is_discrete=True, random_target=True, max_steps=25)
    big = _sim(cuda, 4096, **cfg)
    big.reset(stream=cuda.stream())
    _rollout(cuda, big, T)
    R, Tm = _records(big), _touch(big)
    for n in (1, 7, 8, 9, 33, 100):          # 100: a partial last CTA of 8 envs
        s = _sim(cuda, n, **cfg)
        s.reset(stream=cuda.stream())
        _rollout(cuda, s, T)
        assert _records(s).tobytes() == R[:n].tobytes(), n
        assert _touch(s).tobytes() == Tm[:n].tobytes(), n
    n1, n2 = 37, 59
    s2 = _sim(cuda, n2, global_env_offset=n1, **cfg)
    s2.reset(stream=cuda.stream())
    _rollout(cuda, s2, T)
    assert _records(s2).tobytes() == R[n1:n1 + n2].tobytes()
    assert _touch(s2).tobytes() == Tm[n1:n1 + n2].tobytes()
    # beyond 4224 envs the arm runs one thread per env: its outputs do not change with the bodies, and the bodies do not change with it
    outs = []
    for bodies in (False, True):
        s = _sim(cuda, 4352, bodies=bodies, **cfg)
        s.reset(stream=cuda.stream())
        outs.append(_rollout(cuda, s, T))
    for x, y in zip(*outs):
        assert x.tobytes() == y.tobytes()
    assert _records(s)[:4096].tobytes() == R.tobytes() and _touch(s)[:4096].tobytes() == Tm.tobytes()


def test_masked_reset_replaces_only_the_masked_envs(cuda):
    n = 33
    s = _sim(cuda, n, seed=6, is_discrete=True, random_target=True)
    s.reset(stream=cuda.stream())
    _rollout(cuda, s, 30)
    R0, T0 = _records(s), _touch(s)
    mask = (np.arange(n) % 3 == 0).astype(np.uint8)
    s.reset(mask=cuda.from_host(mask), stream=cuda.stream())
    R1, T1 = _records(s), _touch(s)
    keep = mask == 0
    assert R1[keep].tobytes() == R0[keep].tobytes() and T1[keep].tobytes() == T0[keep].tobytes()
    assert all(R1[i].tobytes() != R0[i].tobytes() for i in np.flatnonzero(mask))
    length = s.distractor_trace()[0]
    assert (length[keep] == 0).all() and (length[~keep] == 5).all()


@pytest.mark.parametrize("repeat", [1, 3])
def test_trace_stays_inside_its_capacity(cuda, repeat):
    """Every env resets as often as it can: max_steps = 1 ends every episode at its first step."""
    n, T = 40, 50
    s = _sim(cuda, n, seed=8, is_discrete=True, action_repeat=repeat, max_steps=1)
    s.reset(stream=cuda.stream())
    out = _rollout(cuda, s, T)
    length, trace, tags, _ = s.distractor_trace()
    print("max_steps=1, action_repeat=%d: %d episodes ended, trace_len max %d of capacity %d" % (repeat, out[2].sum(), length.max(), T * (repeat + 5)))
    assert out[2].sum() >= n * T // 3
    assert (length <= T * (repeat + 5)).all() and length.min() > T * repeat
    assert np.isfinite(_records(s)).all()
