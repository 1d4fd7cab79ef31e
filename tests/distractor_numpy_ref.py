"""Independent float64 model of KukaRandButton's distractor bodies, written from the specification (DESIGN.md section 4, "Distractor
bodies", and the model comment at the top of csrc/distractor_core.h) and not from the header's code, so that agreement between the two
means something.  Deliberately another formulation:

  * a body is (position, scipy Rotation, v, w); world collision spheres and world inverse inertia come from scipy's rotation matrix;
  * contact geometry is generic closest-point code (a point against a solid cylinder: clamp the point into the cylinder and measure to the
    clamped point; inside, leave through the nearer of the top face and the side wall);
  * every row is a dense 6-DoF Jacobian over the env's 66 velocity coordinates, A_ii = J M^-1 J^T by matrix products on the block
    diagonal M^-1, and ONE projected Gauss-Seidel runs over all rows of the env in the order the specification fixes (bodies in slot order;
    per collision sphere: table, disc, stack, arm spheres, then the spheres of higher-slot bodies; normal, then its two tangents).  There
    are no islands: they are the kernel's device and must not change the result.  Connected components (scipy.sparse.csgraph) serve only
    the rule "at most 48 contacts per group of bodies in contact".

`MODEL_COUNTS` counts which geometric cases ran, so a test can assert that its scenario entered the branch it was built for.
"""
import collections

import numpy as np
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components
from scipy.spatial.transform import Rotation

NBODY = 11
MAX_CONTACTS = 48            # per group of bodies in contact and micro-step
STATIC_MU = 1.0              # table, button, arm
Z_TABLE, DROP_H, SPHERE_XY, SPHERE_H = -0.2, 0.1, (0.25, -0.2), 0.3
BALL_FORCE = 10.0
PURPOSE_PLACE, PURPOSE_KICK, PURPOSE_TYPE = 0x100, 0x10A, 0x10B

MODEL_COUNTS = collections.Counter()


class BodyType(object):
    def __init__(self, row):
        self.mass = float(row[0])
        self.inertia = np.array(row[1:4], np.float64)
        self.mu = float(row[4])
        n = int(row[5])
        sph = np.array(row[6:6 + 4 * n], np.float64).reshape(n, 4)
        self.centres, self.radii = sph[:, :3].copy(), sph[:, 3].copy()


def body_types(blob):
    return [BodyType(r) for r in np.asarray(blob, np.float64).reshape(4, 32)]


class Scene(object):
    """Static table and button, and the disc's absolute z range of the current micro-step."""

    def __init__(self, table_z, txmin, txmax, tymin, tymax, bx, by, bz, stack_top, stack_r, disc_r, disc0, disc1, dt=1.0 / 240.0,
                 iters=150, margin=0.02, g=10.0):
        self.table_z, self.tx, self.ty = table_z, (txmin, txmax), (tymin, tymax)
        self.button_xy = np.array([bx, by], np.float64)
        self.stack = (bz, bz + stack_top, stack_r)
        self.disc_r, self.disc0, self.disc1 = disc_r, disc0, disc1
        self.dt, self.iters, self.margin, self.g = dt, iters, margin, g

    @classmethod
    def from_array(cls, a, **kw):
        return cls(*[float(x) for x in a[:13]], **kw)


class Body(object):
    def __init__(self, rec):
        self.p = np.array(rec[0:3], np.float64)
        self.rot = Rotation.from_quat(np.array(rec[3:7], np.float64))
        self.q = np.array(rec[3:7], np.float64)        # the stored quaternion (x y z w); `rot` is rebuilt from it every micro-step
        self.v = np.array(rec[7:10], np.float64)
        self.w = np.array(rec[10:13], np.float64)
        self.type = int(rec[13])
        self.present = rec[14] != 0

    def record(self):
        out = np.zeros(16, np.float64)
        out[0:3], out[3:7], out[7:10], out[10:13], out[13], out[14] = self.p, self.q, self.v, self.w, self.type, float(self.present)
        return out


def quat_mul(a, b):
    """Hamilton product of quaternions stored (x, y, z, w)."""
    av, aw, bv, bw = a[:3], a[3], b[:3], b[3]
    return np.concatenate([aw * bv + bw * av + np.cross(av, bv), [aw * bw - av @ bv]])


def plane_space(n):
    """Bullet's btPlaneSpace1: two unit tangents p, q with (n, p, q) right-handed."""
    if abs(n[2]) > np.sqrt(0.5):
        MODEL_COUNTS["plane_space_z"] += 1
        a = n[1] * n[1] + n[2] * n[2]
        k = 1.0 / np.sqrt(a)
        p = np.array([0.0, -n[2] * k, n[1] * k])
        q = np.array([a * k, -n[0] * p[2], n[0] * p[1]])
    else:
        MODEL_COUNTS["plane_space_xy"] += 1
        a = n[0] * n[0] + n[1] * n[1]
        k = 1.0 / np.sqrt(a)
        p = np.array([-n[1] * k, n[0] * k, 0.0])
        q = np.array([-n[2] * p[1], n[2] * p[0], a * k])
    return p, q


def point_cylinder(s, axis_xy, z0, z1, rad):
    """Signed distance of point s to the solid upright cylinder and the unit normal from the cylinder towards s."""
    d = s[:2] - axis_xy
    rho = float(np.hypot(d[0], d[1]))
    if rho > 1e-12:
        u = d / rho
    else:
        MODEL_COUNTS["cyl_on_axis"] += 1
        u = np.array([1.0, 0.0])
    inside_z, inside_r = z0 < s[2] < z1, rho <= rad
    if inside_z and inside_r:
        to_top, to_side = z1 - s[2], rad - rho
        if to_top <= to_side:
            MODEL_COUNTS["cyl_inside_top"] += 1
            return -to_top, np.array([0.0, 0.0, 1.0])
        MODEL_COUNTS["cyl_inside_side"] += 1
        return -to_side, np.array([u[0], u[1], 0.0])
    closest = np.array([s[0], s[1], min(max(s[2], z0), z1)])
    if not inside_r:
        closest[:2] = axis_xy + rad * u
    v = s - closest
    if inside_r:
        MODEL_COUNTS["cyl_top" if s[2] >= z1 else "cyl_bottom"] += 1
        return abs(v[2]), np.array([0.0, 0.0, 1.0 if s[2] >= z1 else -1.0])
    dist = float(np.linalg.norm(v))
    MODEL_COUNTS["cyl_side" if inside_z else "cyl_rim"] += 1
    return dist, v / dist


Contact = collections.namedtuple("Contact", "a sa b kind n dist ra rb")


def find_contacts(bodies, types, scene, arm):
    """All contacts of the env within the margin, in the specification's order.  Returns (contacts, touch_body, touch_arm, links)."""
    out, links = [], []
    touch_body = touch_arm = 0
    centres = {}
    for k, b in enumerate(bodies):
        if b.present:
            centres[k] = b.p + b.rot.apply(types[b.type].centres)
    for k in sorted(centres):
        b, T = bodies[k], types[bodies[k].type]
        for s, (c, r) in enumerate(zip(centres[k], T.radii)):
            if scene.tx[0] <= c[0] <= scene.tx[1] and scene.ty[0] <= c[1] <= scene.ty[1]:
                dist = c[2] - scene.table_z - r
                if dist <= scene.margin:
                    n = np.array([0.0, 0.0, 1.0])
                    out.append(Contact(k, s, -1, ("table",), n, dist, c - r * n - b.p, None))
            else:
                MODEL_COUNTS["off_table"] += 1
            for name, (z0, z1, rad) in (("disc", (scene.disc0, scene.disc1, scene.disc_r)), ("stack", scene.stack)):
                d, n = point_cylinder(c, scene.button_xy, z0, z1, rad)
                if d - r <= scene.margin:
                    out.append(Contact(k, s, -1, (name,), n, d - r, c - r * n - b.p, None))
            for j, a in enumerate(arm):
                v = c - a[:3]
                ln = float(np.linalg.norm(v))
                dist = ln - r - a[3]
                if dist <= scene.margin and ln > 1e-9:
                    n = v / ln
                    out.append(Contact(k, s, -1, ("arm", j), n, dist, c - r * n - b.p, None))
                    touch_arm |= 1 << k
            for m in sorted(centres):
                if m <= k:
                    continue
                bm, Tm = bodies[m], types[bodies[m].type]
                for s2, (c2, r2) in enumerate(zip(centres[m], Tm.radii)):
                    v = c - c2
                    ln = float(np.linalg.norm(v))
                    dist = ln - r - r2
                    if dist <= scene.margin:
                        links.append((k, m))
                        if ln > 1e-9:
                            n = v / ln
                            out.append(Contact(k, s, m, ("body", m, s2), n, dist, c - r * n - b.p, c2 + r2 * n - bm.p))
                            touch_body |= (1 << k) | (1 << m)
    return out, touch_body, touch_arm, links


def components(links):
    """Label of the group of bodies in contact each body belongs to."""
    if not links:
        return np.arange(NBODY)
    i, j = np.array(links).T
    g = csr_matrix((np.ones(len(i)), (i, j)), shape=(NBODY, NBODY))
    return connected_components(g, directed=False)[1]


def micro_step(bodies, types, scene, arm=(), kick=None):
    """One micro-step in place.  Returns (touch_body, touch_arm, contact keys)."""
    dt = scene.dt
    Minv = np.zeros((6 * NBODY, 6 * NBODY))
    vel = np.zeros(6 * NBODY)
    for k, b in enumerate(bodies):
        if not b.present:
            continue
        T = types[b.type]
        b.rot = Rotation.from_quat(b.q)
        R = b.rot.as_matrix()
        Iinv = R @ np.diag(1.0 / T.inertia) @ R.T
        Minv[6 * k:6 * k + 3, 6 * k:6 * k + 3] = np.eye(3) / T.mass
        Minv[6 * k + 3:6 * k + 6, 6 * k + 3:6 * k + 6] = Iinv
        b.v[2] -= scene.g * dt
        if kick is not None and k == 10:
            J = np.asarray(kick, np.float64)
            b.v += J / T.mass
            b.w += Iinv @ np.cross(np.zeros(3) - b.p, J)         # the force acts at the world origin
        vel[6 * k:6 * k + 3], vel[6 * k + 3:6 * k + 6] = b.v, b.w
    contacts, touch_body, touch_arm, links = find_contacts(bodies, types, scene, np.asarray(arm, np.float64).reshape(-1, 4))
    label = components(links)
    used = collections.Counter()
    kept = []
    for c in contacts:
        if used[label[c.a]] < MAX_CONTACTS:
            used[label[c.a]] += 1
            kept.append(c)
        else:
            MODEL_COUNTS["contact_dropped"] += 1
    nr = 3 * len(kept)
    if nr:
        J = np.zeros((nr, 6 * NBODY))
        target, mu = np.zeros(nr), np.zeros(nr)
        for i, c in enumerate(kept):
            t1, t2 = plane_space(c.n)
            for j, d in enumerate((c.n, t1, t2)):
                J[3 * i + j, 6 * c.a:6 * c.a + 3] = d
                J[3 * i + j, 6 * c.a + 3:6 * c.a + 6] = np.cross(c.ra, d)
                if c.b >= 0:
                    J[3 * i + j, 6 * c.b:6 * c.b + 3] = -d
                    J[3 * i + j, 6 * c.b + 3:6 * c.b + 6] = -np.cross(c.rb, d)
            target[3 * i] = -c.dist / dt if c.dist > 0 else -0.2 * c.dist / dt
            mu[3 * i:3 * i + 3] = types[bodies[c.a].type].mu * (types[bodies[c.b].type].mu if c.b >= 0 else STATIC_MU)
        MJ = Minv @ J.T
        inv_diag = 1.0 / np.einsum("ij,ji->i", J, MJ)
        MJ = np.ascontiguousarray(MJ.T)
        lam = np.zeros(nr)
        for _ in range(scene.iters):
            moved = False
            for i in range(nr):
                new = lam[i] + inv_diag[i] * (target[i] - J[i] @ vel)
                if i % 3 == 0:
                    new = max(new, 0.0)
                else:
                    bound = mu[i] * lam[i - i % 3]
                    new = min(max(new, -bound), bound)
                    MODEL_COUNTS["friction_clamped" if abs(new) == bound and bound > 0 else "friction_free"] += 1
                dl = new - lam[i]
                if dl != 0.0:
                    lam[i] = new
                    vel += dl * MJ[i]
                    moved = True
            if not moved:        # a sweep that changes nothing repeats itself: the remaining sweeps are the identity
                break
    for k, b in enumerate(bodies):
        if not b.present:
            continue
        b.v, b.w = vel[6 * k:6 * k + 3].copy(), vel[6 * k + 3:6 * k + 6].copy()
        b.p = b.p + dt * b.v
        q = b.q + 0.5 * dt * quat_mul(np.concatenate([b.w, [0.0]]), b.q)
        b.q = q / np.linalg.norm(q)
        if np.any(b.w != 0):
            MODEL_COUNTS["integrate_spinning"] += 1
    keys = frozenset((c.a, c.sa) + c.kind for c in contacts)
    return touch_body, touch_arm, keys


def run(blob, scene, B, n_steps, arm=None, disc=None, kicks=None):
    """Advance the records B (f64[11,16]) by n_steps micro-steps.  arm: None, one f64[narm,4] for all micro-steps or one per micro-step;
    disc: optional (disc0, disc1) per micro-step; kicks: {micro-step: impulse}.  Returns (trajectory f64[n,11,16], touch_body, touch_arm,
    contact keys per micro-step)."""
    types = body_types(blob)
    bodies = [Body(r) for r in np.asarray(B, np.float64).reshape(NBODY, 16)]
    traj = np.zeros((n_steps, NBODY, 16))
    tb = ta = 0
    keys = []
    for s in range(n_steps):
        a = () if arm is None else (arm[s] if np.ndim(arm) == 3 or isinstance(arm, (list, tuple)) else arm)
        if disc is not None:
            scene.disc0, scene.disc1 = disc[s]
        t0, t1, k = micro_step(bodies, types, scene, a, None if not kicks else kicks.get(s))
        tb |= t0
        ta |= t1
        keys.append(k)
        traj[s] = [b.record() for b in bodies]
    return traj, tb, ta, keys


def contact_keys(blob, scene, B, arm=()):
    """The contact set of a configuration (no step taken)."""
    types = body_types(blob)
    bodies = [Body(r) for r in np.asarray(B, np.float64).reshape(NBODY, 16)]
    c = find_contacts(bodies, types, scene, np.asarray(arm, np.float64).reshape(-1, 4))[0]
    return frozenset((x.a, x.sa) + x.kind for x in c)


# ---- reset()'s placement, the kick and the env's counter-based stream -------------------------------------------------------------

def place(xy, types10, btn_x, btn_y):
    """Records after reset()'s loading: object k at (x_k, y_k, Z_TABLE + 0.1) unless inside the +-0.1 square around the button; the
    sphere always at (0.25, -0.2, Z_TABLE + 0.3).  At rest, unrotated."""
    B = np.zeros((NBODY, 16))
    B[:, 6] = 1.0
    xy = np.asarray(xy, np.float64).reshape(10, 2)
    for k in range(10):
        x, y = xy[k]
        B[k, 0:3] = [x, y, Z_TABLE + DROP_H]
        B[k, 13] = types10[k]
        B[k, 14] = 0.0 if (btn_x - 0.1 <= x <= btn_x + 0.1 and btn_y - 0.1 <= y <= btn_y + 0.1) else 1.0
    B[10, 0:3] = [SPHERE_XY[0], SPHERE_XY[1], Z_TABLE + SPHERE_H]
    B[10, 13], B[10, 14] = 3, 1
    return B


def kick_impulse(n0, n1, dt):
    """The force |10 n_x|, |10 n_y|, 1 N of the unit horizontal direction (n0, n1) / |.|, applied for one micro-step."""
    ln = np.hypot(n0, n1)
    f = np.array([abs(n0 / ln) * BALL_FORCE, abs(n1 / ln) * BALL_FORCE, 1.0]) if ln > 0 else np.array([BALL_FORCE, 0.0, 1.0])
    return f * dt


def u01(a, b):
    """53-bit uniform in [0, 1) from two 32-bit words: 27 high bits of a, 26 high bits of b."""
    return ((int(a) >> 5) * 67108864 + (int(b) >> 6)) / 9007199254740992.0


def stream_placement(philox, seed, genv, episode):
    """Placements (x0, y0, ..., x9, y9) and the 10 types of (seed, global env, episode).  philox(seed, env, index, purpose) -> 4 words."""
    xy = np.zeros(20)
    for k in range(10):
        w = philox(seed, genv, episode, PURPOSE_PLACE + k)
        xy[2 * k] = 0.5 + 0.15 * (-1.0 + 2.0 * u01(w[0], w[1]))
        xy[2 * k + 1] = 0.3 * (-1.0 + 2.0 * u01(w[2], w[3]))
    words = [x for b in range(3) for x in philox(seed, genv, episode, PURPOSE_TYPE + b)]
    types10 = [(int(x) * 3) >> 32 for x in words[:10]]           # randint(3): the high word of word * 3
    return xy, types10


def stream_kick(philox, seed, genv, episode, dt):
    """Two Box-Muller normals from one Philox block, then the kick's impulse."""
    w = philox(seed, genv, episode, PURPOSE_KICK)
    u1, u2 = u01(w[0], w[1]), u01(w[2], w[3])
    rad = np.sqrt(-2.0 * np.log(1.0 - u1))
    return kick_impulse(rad * np.cos(2.0 * np.pi * u2), rad * np.sin(2.0 * np.pi * u2), dt)
