"""csrc/distractor_core.h (compiled in float64: csrc/libdistractor_ref.so) against the independent float64 model of
tests/distractor_numpy_ref.py, over whole trajectories, in scenarios built so that every branch of the header runs.

Tolerance.  Both sides are float64 and sweep the same rows in the same order, but they are different formulations (dense Jacobians and
matrix products against the header's cross products, scipy's rotation matrices against dc_rot, a quaternion product against the expanded
update), so they differ in the last bits of every operation: ~1e-16 relative per micro-step.  Contact amplifies that -- a Gauss-Seidel
sweep of a stiff stack multiplies a rounding difference by up to ~1e2, a few hundred micro-steps add up -- which leaves 1e-12 ... 1e-10 at
the end of the longer scenarios.  ATOL = 1e-9 on position (m), quaternion, v (m/s) and w (rad/s) holds for all of them with room, and
is 5 orders below the effect of any wrong sign, swapped tangent or dropped row (>= 1e-4 after one contact micro-step).  Touch masks are
compared exactly."""
import ctypes
import os
import sys

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "robotics-rl-srl_b200")
for p in (PKG, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import distractor_numpy_ref as ref  # noqa: E402
from srl_sim.model import distractor_blob  # noqa: E402

DT, MARGIN, ATOL = 1.0 / 240.0, 0.02, 1e-9
TZ = -0.195
# a table with the button at (0.5, 0): base stack 5 cm high, radius 0.1; the disc (radius 0.09) from 7 to 9 cm above the table
BUTTON = np.array([TZ, -0.25, 1.25, -0.5, 0.5, 0.5, 0.0, TZ, 0.05, 0.1, 0.09, TZ + 0.07, TZ + 0.09], np.float64)
DISC0, DISC1, STACK1 = TZ + 0.07, TZ + 0.09, TZ + 0.05
# the same table with the button far away
PLAIN = BUTTON.copy()
PLAIN[5:7] = 5.0
DUCK, LEGO, CUBE, BALL = range(4)
R_BALL, R_LEGO = 0.03, 0.0095


@pytest.fixture(scope="module")
def dref():
    path = os.path.join(PKG, "csrc", "libdistractor_ref.so")
    if not os.path.isfile(path):
        pytest.skip("libdistractor_ref.so not built (python __graft_entry__.py build)")
    lib = ctypes.CDLL(path)
    P = ctypes.c_void_p
    lib.dref_run_steps.argtypes = [P, ctypes.c_size_t, P, ctypes.c_double, ctypes.c_int, ctypes.c_double, P, P, ctypes.c_int, ctypes.c_int, P, P, P,
                                   P, P]
    lib.dref_run_steps.restype = ctypes.c_int
    lib.dref_island_roots.argtypes = [P, P]
    lib.dref_kick.argtypes = [ctypes.c_double, ctypes.c_double, ctypes.c_double, P]
    return lib


def header_run(lib, blob, scene, B, n, arm, disc, kicks, iters):
    """The header through dref_run_steps.  arm: f64[n, narm, 4]; disc: f64[n, 2] or None; kicks: {micro-step: impulse}."""
    B = np.array(B, np.float64)
    narm = arm.shape[1]
    arm_buf = np.ascontiguousarray(arm if narm else np.zeros((n, 1, 4)), np.float64)
    traj = np.zeros((n, 11, 16), np.float64)
    touch = np.zeros(2, np.uint32)
    kv, ko = np.zeros((n, 3), np.float64), np.zeros(n, np.uint8)
    for s, j in (kicks or {}).items():
        kv[s], ko[s] = j, 1
    d = None if disc is None else np.ascontiguousarray(disc, np.float64)
    rc = lib.dref_run_steps(blob.ctypes.data, blob.nbytes, scene.ctypes.data, DT, iters, MARGIN, B.ctypes.data, arm_buf.ctypes.data, narm, n,
                            None if d is None else d.ctypes.data, kv.ctypes.data, ko.ctypes.data, traj.ctypes.data, touch.ctypes.data)
    assert rc == 0
    return traj, int(touch[0]), int(touch[1])


def both(lib, B, n, scene=PLAIN, arm=None, disc=None, kicks=None, iters=50, blob=None):
    """Run the header and the model on the same input and compare every present body over the whole trajectory.  Returns the header's
    trajectory, the model's contact keys per micro-step and the model's counters of this run."""
    blob = distractor_blob() if blob is None else blob
    arm = np.zeros((n, 0, 4)) if arm is None else np.asarray(arm, np.float64)
    if arm.ndim == 2:
        arm = np.broadcast_to(arm, (n,) + arm.shape).copy()
    th, tb_h, ta_h = header_run(lib, blob, scene, B, n, arm, disc, kicks, iters)
    ref.MODEL_COUNTS.clear()
    sc = ref.Scene.from_array(scene, dt=DT, iters=iters, margin=MARGIN)
    tm, tb_m, ta_m, keys = ref.run(blob, sc, B, n, arm=arm, disc=disc, kicks=kicks)
    counts = dict(ref.MODEL_COUNTS)
    present = np.asarray(B)[:, 14] != 0
    for name, sl in (("position", slice(0, 3)), ("velocity", slice(7, 10)), ("angular velocity", slice(10, 13))):
        err = np.abs(th[:, present, sl] - tm[:, present, sl]).max()
        assert err <= ATOL, "%s differs by %.3g" % (name, err)
    qh, qm = th[:, present, 3:7], tm[:, present, 3:7]
    qerr = np.minimum(np.abs(qh - qm).max(axis=-1), np.abs(qh + qm).max(axis=-1)).max()
    assert qerr <= ATOL, "quaternion differs by %.3g" % qerr
    np.testing.assert_allclose(np.linalg.norm(qh, axis=-1), 1.0, atol=1e-12)
    assert np.array_equal(th[:, ~present], np.broadcast_to(np.asarray(B, np.float64)[~present], th[:, ~present].shape)), "an absent body changed"
    assert (tb_h, ta_h) == (tb_m, ta_m), "touch masks differ: header %x %x, model %x %x" % (tb_h, ta_h, tb_m, ta_m)
    return th, keys, counts


def bodies(*specs):
    """specs: (slot, type, position[, quaternion[, v[, w]]])."""
    B = np.zeros((11, 16), np.float64)
    B[:, 6] = 1.0
    for sp in specs:
        slot, t, pos = sp[:3]
        B[slot, 0:3], B[slot, 13], B[slot, 14] = pos, t, 1.0
        if len(sp) > 3 and sp[3] is not None:
            B[slot, 3:7] = np.asarray(sp[3], np.float64) / np.linalg.norm(sp[3])
        if len(sp) > 4:
            B[slot, 7:10] = sp[4]
        if len(sp) > 5:
            B[slot, 10:13] = sp[5]
    return B


def kinds(keys):
    return {k[2] for s in keys for k in s}


# ---- one body on the table: tilt, spin, loaded friction ----------------------------------------------------------------------------

@pytest.mark.parametrize("t", [DUCK, LEGO, CUBE, BALL])
def test_tilted_drop_with_sideways_velocity(dref, t):
    q = Rotation.random(random_state=10 + t).as_quat()
    B = bodies((4, t, (0.5, 0.0, TZ + 0.08), q, (0.3, -0.2, 0.0), (1.0, -2.0, 0.5)))
    traj, keys, c = both(dref, B, 220)
    assert "table" in kinds(keys)
    assert c.get("integrate_spinning", 0) > 0 and c.get("friction_free", 0) > 0
    assert c.get("friction_clamped", 0) > 0 or t == BALL     # the ball's single contact takes up its rolling without reaching the bound


@pytest.mark.parametrize("name,t,z", [("sphere_small", BALL, TZ + 0.12), ("lego", LEGO, TZ + 0.12)])
def test_upright_drop_lands_on_the_table(dref, name, t, z):
    """The straight drop of test_distractors_cpu.py's one-body model as one more input: no rotation may appear."""
    traj, keys, c = both(dref, bodies((10, t, (0.5, 0.0, z))), 100, iters=150)
    np.testing.assert_allclose(traj[:, 10, 3:7], np.broadcast_to([0, 0, 0, 1], (100, 4)), atol=1e-12)
    assert abs(traj[-1, 10, 2] - (TZ + (R_BALL if t == BALL else R_LEGO))) < 1e-6


def test_brick_slides_until_friction_stops_it(dref):
    B = bodies((0, LEGO, (0.3, 0.1, TZ + R_LEGO), None, (0.5, 0.0, 0.0)))
    traj, keys, c = both(dref, B, 70)
    # mu = 0.5 * 1.0 and g = 10: the Coulomb bound is active while it slides (5 m/s^2 for ~24 micro-steps), then friction holds it
    assert c["friction_clamped"] > 0 and c["friction_free"] > 0
    v = traj[:, 0, 7]
    np.testing.assert_allclose(np.diff(v[2:15]), -5.0 * DT, rtol=0.05)
    assert abs(v[-1]) < 1e-6 and 0.32 < traj[-1, 0, 0] < 0.33


# ---- a ball against the button ------------------------------------------------------------------------------------------------------

BUTTON_CASES = {
    # name: (start position, velocity, branch of the model that must run, contact kind that must appear)
    "disc_top": ((0.53, 0.01, DISC1 + R_BALL + 0.03), (0, 0, 0), "cyl_top", "disc"),
    "stack_top": ((0.5 + 0.097, 0.0, STACK1 + R_BALL + 0.01), (0, 0, 0), "cyl_top", "stack"),
    "disc_side": ((0.5 + 0.09 + R_BALL + 0.02, 0.0, TZ + 0.08), (-0.6, 0.1, 0.4), "cyl_side", "disc"),
    "stack_side": ((0.5 - 0.1 - R_BALL - 0.015, 0.02, TZ + R_BALL), (0.5, 0, 0), "cyl_side", "stack"),
    "disc_rim": ((0.5, 0.09 + 0.012, DISC1 + R_BALL + 0.03), (0, 0, 0), "cyl_rim", "disc"),
    "stack_rim": ((0.5 - 0.1 - 0.01, 0.0, STACK1 + R_BALL + 0.03), (0, 0, 0), "cyl_rim", "stack"),
    "inside_near_top": ((0.53, 0.0, DISC1 - 0.002), (0, 0, 0), "cyl_inside_top", "disc"),
    "inside_near_side": ((0.5, -0.09 + 0.003, TZ + 0.08), (0, 0, 0), "cyl_inside_side", "disc"),
    "below_the_disc": ((0.5 + 0.085, 0.0, STACK1 + 0.005), (0, 0, 0), "cyl_bottom", "disc"),
    "on_the_axis": ((0.5, 0.0, DISC1 + R_BALL + 0.02), (0, 0, 0), "cyl_on_axis", "disc"),
}


@pytest.mark.parametrize("case", sorted(BUTTON_CASES))
def test_ball_against_the_button(dref, case):
    pos, v, branch, kind = BUTTON_CASES[case]
    traj, keys, c = both(dref, bodies((10, BALL, pos, None, v)), 120, scene=BUTTON)
    assert c.get(branch, 0) > 0, (case, c)
    assert kind in kinds(keys)


def test_ball_on_a_disc_that_moves_every_micro_step(dref):
    n = 200
    lift = 0.01 * np.sin(np.arange(n) * 0.15) - 0.005
    disc = np.stack([DISC0 + lift, DISC1 + lift], axis=1)
    traj, keys, c = both(dref, bodies((10, BALL, (0.52, 0.01, DISC1 + R_BALL + 0.001))), n, scene=BUTTON, disc=disc)
    assert all(("disc" in {k[2] for k in s}) for s in keys[:20])
    # the ball is carried: it rises with the disc at some point (a disc frozen at its first range would leave it at rest)
    assert traj[:, 10, 9].max() > 0.01


# ---- the table's edge ----------------------------------------------------------------------------------------------------------------

def test_brick_half_over_the_table_edge_tips_and_ball_falls_off(dref):
    B = bodies((3, LEGO, (1.25 + 0.001, 0.1, TZ + R_LEGO + 0.005)), (10, BALL, (1.25 + 0.05, -0.2, TZ + 0.1)))
    traj, keys, c = both(dref, B, 160)
    first = {k[:3] for k in keys[0]}
    assert {(3, 0, "table"), (3, 1, "table")} <= first and not {(3, 2, "table"), (3, 3, "table")} & first
    assert c["off_table"] > 0
    assert np.abs(traj[-1, 3, 10:13]).max() > 0.1           # it tipped
    assert traj[-1, 10, 2] < TZ - 0.5                       # the ball never met the table


# ---- the arm's spheres ---------------------------------------------------------------------------------------------------------------

def test_ball_rests_against_a_fixed_arm_sphere(dref):
    arm = np.array([[0.5, 0.2, TZ + 0.02, 0.04], [0.9, 0.9, 0.9, 0.01]])
    traj, keys, c = both(dref, bodies((10, BALL, (0.53, 0.2, TZ + 0.13))), 200, arm=arm)
    assert ("arm" in kinds(keys)) and traj[-1, 10, 0] > 0.55


def test_moving_arm_sphere_pushes_a_brick(dref):
    n = 150
    arm = np.zeros((n, 1, 4))
    arm[:, 0] = [0.40, 0.0, TZ + 0.02, 0.02]
    arm[:, 0, 0] += 0.12 * DT * np.arange(n)
    traj, keys, c = both(dref, bodies((6, LEGO, (0.46, 0.004, TZ + R_LEGO))), n, arm=arm)
    assert traj[-1, 6, 0] > 0.47 and "arm" in kinds(keys)


# ---- bodies against bodies -----------------------------------------------------------------------------------------------------------

def test_brick_on_a_brick(dref):
    B = bodies((2, LEGO, (0.4, 0.0, TZ + R_LEGO)), (5, LEGO, (0.403, 0.002, TZ + 3 * R_LEGO + 0.01)))
    traj, keys, c = both(dref, B, 200)
    assert "body" in kinds(keys) and traj[-1, 5, 2] > TZ + 2 * R_LEGO


def test_ball_rolls_into_a_cube(dref):
    B = bodies((3, CUBE, (0.5, 0.0, TZ + 0.025)), (10, BALL, (0.4, 0.004, TZ + R_BALL), None, (0.5, 0, 0), (0, 0.5 / R_BALL, 0)))
    traj, keys, c = both(dref, B, 160)
    assert "body" in kinds(keys) and traj[-1, 3, 0] > 0.5005


def _components_per_step(keys):
    out = []
    for s in keys:
        links = [(k[0], k[3]) for k in s if k[2] == "body"]
        lab = ref.components(links)
        out.append(len({lab[b] for l in links for b in l}))
    return out


def test_chain_of_three_forms_one_island_and_splits_while_another_island_rests(dref):
    # slots in descending order along the chain (7 - 4 - 1), and a brick on a brick elsewhere as a second island
    B = bodies((7, BALL, (0.30, 0.0, TZ + R_BALL), None, (1.5, 0, 0)), (4, BALL, (0.42, 0.003, TZ + R_BALL)), (1, BALL, (0.495, -0.002, TZ + R_BALL)),
               (2, LEGO, (0.7, 0.3, TZ + R_LEGO)), (5, LEGO, (0.702, 0.301, TZ + 3 * R_LEGO)))
    traj, keys, c = both(dref, B, 260)
    groups = _components_per_step(keys)
    pairs = [{(k[0], k[3]) for k in s if k[2] == "body"} for s in keys]
    chain = [{(4, 7), (1, 4)} <= p for p in pairs]
    assert not chain[0] and any(chain), "the three balls never formed one island"
    assert max(groups) == 2 and not all(chain[chain.index(True):]), "the chain never split again"


def test_unequal_friction_coefficients_multiply(dref):
    blob = distractor_blob().reshape(4, 32).copy()
    blob[LEGO, 4], blob[BALL, 4] = 0.9, 0.3
    blob = blob.reshape(-1)
    B = bodies((2, LEGO, (0.4, 0.0, TZ + R_LEGO), None, (0.4, 0, 0)), (10, BALL, (0.404, 0.002, TZ + 2 * R_LEGO + R_BALL + 0.001), None, (-0.3, 0.2, 0)))
    traj, keys, c = both(dref, B, 120, blob=blob)
    assert "body" in kinds(keys) and c["friction_clamped"] > 0


def test_pile_with_more_than_48_contacts_in_one_island(dref):
    spec = [(k, LEGO, (0.4 + 0.036 * (k % 3), 0.036 * (k // 3), TZ + R_LEGO + 0.001)) for k in range(9)]
    spec += [(9, CUBE, (0.436, 0.036, TZ + 2 * R_LEGO + 0.03)), (10, BALL, (0.42, 0.02, TZ + 2 * R_LEGO + R_BALL + 0.005))]
    traj, keys, c = both(dref, bodies(*spec), 60, iters=30)
    assert max(len(s) for s in keys) > ref.MAX_CONTACTS and c["contact_dropped"] > 0


# ---- the kick ------------------------------------------------------------------------------------------------------------------------

def test_kick_away_from_the_origin_gives_linear_and_angular_impulse(dref):
    J = ref.kick_impulse(-0.6, 1.7, DT)
    imp = np.zeros(3)
    dref.dref_kick(-0.6, 1.7, DT, imp.ctypes.data)
    np.testing.assert_allclose(imp, J, rtol=1e-15)
    np.testing.assert_allclose(J, np.array([10 * 0.6, 10 * 1.7, np.hypot(0.6, 1.7)]) / np.hypot(0.6, 1.7) * DT, rtol=1e-14)
    row = distractor_blob().reshape(4, 32)[BALL]
    # in free flight the first micro-step shows the impulse alone: v = J / m - g dt, w = I^-1 ((0 - p) x J)
    p = np.array([0.25, -0.2, 0.3])
    traj, _, _ = both(dref, bodies((10, BALL, p)), 3, kicks={0: J})
    np.testing.assert_allclose(traj[0, 10, 7:10], J / row[0] - [0, 0, 10 * DT], rtol=1e-13)
    np.testing.assert_allclose(traj[0, 10, 10:13], np.cross(-p, J) / row[1], rtol=1e-13)
    # on the table, kicked in micro-step 5, then the roll
    start = (0.25, -0.2, TZ + R_BALL)
    traj, keys, c = both(dref, bodies((10, BALL, start)), 150, kicks={5: J}, iters=150)
    assert traj[-1, 10, 0] > 0.26 and traj[-1, 10, 1] > -0.19 and c["friction_clamped"] > 0


# ---- the tangent basis on both sides of its switch -----------------------------------------------------------------------------------

@pytest.mark.parametrize("deg,branch", [(44.5, "plane_space_z"), (45.5, "plane_space_xy")])
def test_tangent_basis_on_both_sides_of_the_switch(dref, deg, branch):
    a = np.radians(deg)
    n = np.array([np.sin(a) * 0.8, np.sin(a) * 0.6, np.cos(a)])
    centre = np.array([0.5, 0.0, 0.3])
    arm = np.array([[centre[0], centre[1], centre[2], 0.04]])
    # in the air, resting obliquely on the sphere with a tangential velocity: only this contact, its friction rows loaded
    B = bodies((10, BALL, centre + (0.04 + R_BALL + 0.001) * n, None, (0.2, -0.3, -0.2), (3.0, 1.0, -2.0)))
    traj, keys, c = both(dref, B, 1, arm=arm)
    assert c.get(branch, 0) > 0 and c.get("plane_space_xy" if branch == "plane_space_z" else "plane_space_z", 0) == 0, c
    assert kinds(keys[:1]) == {"arm"}


# ---- islands -------------------------------------------------------------------------------------------------------------------------

def _roots(lib, pairs):
    adj = np.zeros(11, np.uint32)
    for k, m in pairs:
        k, m = min(k, m), max(k, m)
        adj[k] |= np.uint32(1 << m)
    root = np.zeros(11, np.int32)
    lib.dref_island_roots(adj.ctypes.data, root.ctypes.data)
    return root


def _expected_roots(pairs):
    i, j = (np.array(pairs).T if pairs else (np.zeros(0, int), np.zeros(0, int)))
    lab = connected_components(csr_matrix((np.ones(len(i)), (i, j)), shape=(11, 11)), directed=False)[1]
    return np.array([np.flatnonzero(lab == lab[k]).min() for k in range(11)], np.int32)


def test_island_roots_against_scipy_connected_components(dref):
    rng = np.random.RandomState(0)
    cases = [[], [(k, k + 1) for k in range(10)], [(k, m) for k in range(11) for m in range(k + 1, 11)]]
    # chains whose links run against the slot order need the most passes: 10-9-...-0 through a permutation, zig-zags, two interleaved chains
    cases.append([(10 - k, 9 - k) for k in range(10)])
    cases.append([(0, 10), (10, 1), (1, 9), (9, 2), (2, 8), (8, 3), (3, 7), (7, 4), (4, 6), (6, 5)])
    cases.append([(5, 10), (10, 4), (4, 9), (9, 3), (3, 8), (8, 2), (2, 7), (7, 1), (1, 6), (6, 0)])
    cases.append([(10, 8), (8, 6), (6, 4), (4, 2), (9, 7), (7, 5), (5, 3), (3, 1)])
    for _ in range(10):
        perm = rng.permutation(11)
        cases.append([(int(perm[k]), int(perm[k + 1])) for k in range(10)])
    for _ in range(300):
        m = rng.randint(0, 12)
        cases.append([tuple(int(x) for x in rng.choice(11, 2, replace=False)) for _ in range(m)])
    for pairs in cases:
        assert np.array_equal(_roots(dref, pairs), _expected_roots(pairs)), pairs
