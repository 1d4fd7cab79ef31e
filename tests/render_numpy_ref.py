"""
An independent float64 ray caster of the rendered scenes (test-only), written from the geometry rather than from csrc/render_core.h.

What it shares with the kernels is one thing, the documented scene spec: which primitives a scene holds, their sizes, colours and list order.
That spec is restated below (`kuka_prims`, `mobile_prims`) from the comments of srl_kuka_scene, srl_mobile_scene and srl_distractor_prims;
everything else is textbook and computed in float64:

* camera: rays from the eye through the pixel centres (x + 0.5, y + 0.5), row 0 at the top, unprojected through inv(proj @ view) of
  pybullet-style view / projection matrices (`pybullet_matrices`: computeViewMatrixFromYawPitchRoll with upAxisIndex 2, roll included, and
  computeProjectionMatrixFOV).  srl_camera_setup is not used.  The camera's parameters are rounded to float32 first, as the C-ABI passes them;
* intersections: only entry points with t > 1e-4 count (a solid seen from inside is not drawn); the nearest t wins, a tie keeps the earlier
  list index.  Plane z = const (hit by rays going down); sphere by its quadratic; capsule = the minimum over the finite side cylinder and
  the outer halves of both end spheres (its boundary); upright capped cylinder = side quadratic and the two cap discs; boxes = slab tests in
  the box frame, a z-rotation matrix for BOX and the rotation matrix of the unit quaternion for OBOX;
* colour: textbook outward normals, the plane's checker by the parity of floor(x / period) + floor(y / period), shade 0.55 + 0.45 max(n.L, 0)
  with L = (2, 3, 4) / |(2, 3, 4)|, background (0.84, 0.89, 0.95), each byte floor(c shade 255 + 0.5) clamped.

A float32 kernel may disagree with it only where a decision sits within rounding of its boundary, so `render` also returns an *unstable*
mask and, per pixel, the candidate colours.  A pixel is unstable when
* the centre ray and four rays jittered by (+-0.02, +-0.02) px do not all hit the same primitive, part (box face, cylinder side / cap,
  capsule side / end) and checker parity;
* the two nearest hits of different primitives are within 1e-5 of each other (relative) plus what float32 can move each: a quadratic's
  t = (-b - sqrt(h)) / a carries the rounding of h over sqrt(h), so a ray that grazes a surface (at the joints of the arm's capsules) has
  an ill-conditioned t;
* the hit is on a box edge (two slabs entered within 1e-6, relative);
* the hit is a checker point within float32 reach of a cell boundary (near the horizon t = (z - eye_z) / d_z moves by metres, and the
  jittered rays are metres apart);
* the hit lies in the cylinder band render_core.h documents (srl_normal_at takes cap points with r^2 >= 0.9999 R^2 for side points, a
  deliberate approximation).
The candidates are the colours of the five rays, the second-nearest primitive's colour, and at a cylinder band or checker boundary the
colour of the other choice.
"""
import numpy as np

PLANE, SPHERE, CAPSULE, CYL, BOX, OBOX = range(6)
BACKGROUND = np.array([0.84, 0.89, 0.95])
LIGHT = np.array([2.0, 3.0, 4.0]) / np.sqrt(29.0)
CHECKER_2 = (0.68, 0.77, 0.93)
T_MIN = 1e-4
EPS32 = 2.0 ** -24
JITTER = 0.02
N_CAND = 7


# ---- the scene spec (the one part shared with render_core.h) ------------------------------------------------------------------------
def plane(z, period, rgb):
    return dict(type=PLANE, z=float(z), period=float(period), rgb=np.array(rgb, float), rgb2=np.array(CHECKER_2))


def sphere(c, r, rgb):
    return dict(type=SPHERE, c=np.array(c, float), r=float(r), rgb=np.array(rgb, float))


def capsule(e0, e1, r, rgb):
    return dict(type=CAPSULE, e0=np.array(e0, float), e1=np.array(e1, float), r=float(r), rgb=np.array(rgb, float))


def cylinder(cx, cy, z0, z1, r, rgb):
    return dict(type=CYL, cx=float(cx), cy=float(cy), z0=float(z0), z1=float(z1), r=float(r), rgb=np.array(rgb, float))


def box(c, half, yaw, rgb):
    """A box rotated by `yaw` radians about z."""
    cs, sn = np.cos(yaw), np.sin(yaw)
    R = np.array([[cs, -sn, 0.0], [sn, cs, 0.0], [0.0, 0.0, 1.0]])
    return dict(type=BOX, c=np.array(c, float), half=np.array(half, float), R=R, rgb=np.array(rgb, float))


def quat_matrix(q):
    """Rotation matrix of the quaternion (x, y, z, w), normalised first."""
    x, y, z, w = np.asarray(q, float) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def obox(c, half, quat, rgb):
    return dict(type=OBOX, c=np.array(c, float), half=np.array(half, float), R=quat_matrix(quat), rgb=np.array(rgb, float))


def kuka_prims(scene, q, button_base, glider_q, button2=None, bodies=None, looks=None):
    """The Kuka list of srl_kuka_scene (+ srl_distractor_prims): plane at z = -1 with a 1 m checker; the table top (5 cm slab) and four
    10 cm legs down to the plane; per button a green cylinder stack and the yellow disc lifted by the glider; a grey pedestal capsule from
    the base to joint 0, seven link capsules (radius 0.065 for the first four, then 0.055; orange / blue-grey alternating), four gripper
    capsules (0.02 to the finger bases, 0.012 along the fingers), the collision spheres of the gripper bodies (body >= 7); then the present
    bodies (shape 1: a sphere of radius half[0], else an oriented box).

    scene: a KukaScene; q: the 12 joint positions (forward kinematics in float64 here); button_base: (x, y, z); glider_q: the disc's joint
    position; button2: (x, y, q) of the second button (z is the scene constant) or None; bodies: [11, 9] (position, quaternion x y z w,
    type, present) with looks = distractor_blob().reshape(4, 32)."""
    from srl_sim.model import scene_constants
    K = scene_constants(scene)
    P, Rm = scene.forward_kinematics(np.asarray(q, float))
    jp = [np.asarray(p, float) for p in P]
    out =[plane(-1.0, 1.0, (1.0, 1.0, 1.0))]
    tcx, tcy = 0.5 * (K["txmin"] + K["txmax"]), 0.5 * (K["tymin"] + K["tymax"])
    thx, thy = 0.5 * (K["txmax"] - K["txmin"]), 0.5 * (K["tymax"] - K["tymin"])
    tz = K["table_z"]
    out.append(box((tcx, tcy, tz - 0.025), (thx, thy, 0.025), 0.0, (0.92, 0.82, 0.68)))
    for k in range(4):
        sx, sy = (1.0 if k & 1 else -1.0), (1.0 if k & 2 else -1.0)
        out.append(box((tcx + sx * (thx - 0.1), tcy + sy * (thy - 0.1), 0.5 * (tz - 0.05 - 1.0)), (0.05, 0.05, 0.5 * (tz - 0.05 + 1.0)), 0.0,
                       (0.85, 0.75, 0.62)))
    buttons = [(button_base[0], button_base[1], button_base[2], glider_q)]
    if button2 is not None:
        buttons.append((button2[0], button2[1], K["button_z"], button2[2]))
    for (x, y, z, qb) in buttons:
        out.append(cylinder(x, y, z, z + K["stack_top"], K["stack_r"], (0.0, 1.0, 0.0)))
        lift = z + K["glider_z"] + qb
        out.append(cylinder(x, y, lift + K["disc_z0"], lift + K["disc_z1"], K["disc_r"], (1.0, 1.0, 0.0)))
    out.append(capsule(_kuka_base(scene), jp[0], 0.075, (0.3, 0.3, 0.3)))
    for i in range(7):
        orange = i % 2 == 0
        out.append(capsule(jp[i], jp[i + 1], 0.065 if i < 4 else 0.055, (1.0, 0.42, 0.04) if orange else (0.5, 0.7, 1.0)))
    for a, b, r in ((7, 8, 0.02), (8, 9, 0.012), (7, 10, 0.02), (10, 11, 0.012)):
        out.append(capsule(jp[a], jp[b], r, (0.15, 0.15, 0.15)))
    for (body, c, r) in scene.spheres:
        if body >= 7:
            out.append(sphere(jp[body] + Rm[body] @ np.asarray(c, float), r, (0.2, 0.2, 0.2)))
    if bodies is not None:
        for b in np.asarray(bodies, float).reshape(11, 9):
            if b[8] == 0:
                continue
            t = int(b[7])
            half, rgb = looks[t, 22:25], looks[t, 25:28]
            out.append(sphere(b[0:3], half[0], rgb) if looks[t, 28] == 1 else obox(b[0:3], half, b[3:7], rgb))
    return out


def _kuka_base(scene):
    from srl_sim.model import KM
    return np.asarray(scene.scene[KM["KM_SC_BASE_POS"]:KM["KM_SC_BASE_POS"] + 3], float)


# MobileRobot kinds of srl_mobile_scene, by env id
MOBILE_KIND = {"MobileRobotGymEnv-v0": 0, "MobileRobot2TargetGymEnv-v0": 1, "MobileRobotLineTargetGymEnv-v0": 2, "MobileRobot1DGymEnv-v0": 3}


def mobile_prims(kind, robot, target0, target1=None):
    """The MobileRobot list of srl_mobile_scene: plane z = 0 with a 1 m checker; walls 4 x 0.1 x 0.1 centred on z = 0: (2, 0) red, and unless
    the 1-D kind, (4, 2) black and (0, 2) blue (rotated by 90 degrees) and (2, 4) green; the target -- kind 2 a yellow 4 x 0.5 x 0.1 bar at
    (x, 2, -0.045) rotated by 90 degrees, else a yellow disc (r 0.18, z 0 to 0.03) and for kind 1 a second, red one; the robot, a blue box
    0.65 x 0.2 x 0.14 at z 0.09, and a white cabin 0.24 x 0.16 x 0.06 at (x + 0.1, y, 0.17)."""
    out = [plane(0.0, 1.0, (1.0, 1.0, 1.0)), box((2, 0, 0), (2, 0.05, 0.05), 0.0, (0.8, 0, 0))]
    if kind != 3:
        out += [box((4, 2, 0), (2, 0.05, 0.05), np.pi / 2, (0, 0, 0)), box((2, 4, 0), (2, 0.05, 0.05), 0.0, (0, 0.8, 0)),
                box((0, 2, 0), (2, 0.05, 0.05), np.pi / 2, (0, 0, 0.8))]
    if kind == 2:
        out.append(box((target0[0], 2, -0.045), (2, 0.25, 0.05), np.pi / 2, (1, 1, 0)))
    else:
        out.append(cylinder(target0[0], target0[1], 0.0, 0.03, 0.18, (1, 1, 0)))
        if kind == 1:
            out.append(cylinder(target1[0], target1[1], 0.0, 0.03, 0.18, (0.8, 0, 0)))
    rx, ry = float(robot[0]), float(robot[1])
    out.append(box((rx, ry, 0.09), (0.325, 0.1, 0.07), 0.0, (0.1, 0.2, 0.8)))
    out.append(box((rx + 0.1, ry, 0.17), (0.12, 0.08, 0.03), 0.0, (0.95, 0.95, 0.95)))
    return out


# ---- camera ------------------------------------------------------------------------------------------------------------------------
def pybullet_matrices(target, distance, yaw, pitch, roll, fov, aspect, near=0.1, far=100.0):
    """numpy restatement of computeViewMatrixFromYawPitchRoll (upAxisIndex = 2) and computeProjectionMatrixFOV as MATRICES (the renderer uses
    an eye + basis formulation): eye = target + Rz(yaw) Ry(roll) Rx(pitch) (0, -d, 0), up = the same rotation of (0, 0, 1), OpenGL lookAt and
    perspective."""
    y, p, r = np.radians([yaw, pitch, roll])
    Rz = np.array([[np.cos(y), -np.sin(y), 0], [np.sin(y), np.cos(y), 0], [0, 0, 1]])
    Ry = np.array([[np.cos(r), 0, np.sin(r)], [0, 1, 0], [-np.sin(r), 0, np.cos(r)]])
    Rx = np.array([[1, 0, 0], [0, np.cos(p), -np.sin(p)], [0, np.sin(p), np.cos(p)]])
    R = Rz @ Ry @ Rx
    eye = np.asarray(target, float) + R @ np.array([0.0, -distance, 0.0])
    up = R @ np.array([0.0, 0.0, 1.0])
    f = np.asarray(target, float) - eye; f /= np.linalg.norm(f)
    s = np.cross(f, up); s /= np.linalg.norm(s)
    u = np.cross(s, f)
    view = np.eye(4); view[0, :3], view[1, :3], view[2, :3] = s, u, -f
    view[:3, 3] = -view[:3, :3] @ eye
    t = 1.0 / np.tan(np.radians(fov) / 2)
    proj = np.array([[t / aspect, 0, 0, 0], [0, t, 0, 0], [0, 0, (far + near) / (near - far), 2 * far * near / (near - far)], [0, 0, -1, 0]])
    return view, proj


def camera_rays(cam, W, H, dx=0.0, dy=0.0):
    """Eye (3,) and unit directions [H * W, 3] of the rays through (x + 0.5 + dx, y + 0.5 + dy), row 0 at the top."""
    c = {k: (tuple(float(np.float32(v)) for v in cam[k]) if k == "target" else float(np.float32(cam[k])))
         for k in ("target", "distance", "yaw", "pitch", "roll", "fov")}
    view, proj = pybullet_matrices(aspect=float(W) / float(H), **c)
    inv = np.linalg.inv(proj @ view)
    eye = np.linalg.inv(view)[:3, 3]
    xs = (np.arange(W) + 0.5 + dx) / W * 2 - 1
    ys = 1 - (np.arange(H) + 0.5 + dy) / H * 2
    nx, ny = np.meshgrid(xs, ys)
    ndc = np.stack([nx.ravel(), ny.ravel(), np.zeros(W * H), np.ones(W * H)], axis=1)
    w = ndc @ inv.T
    pts = w[:, :3] / w[:, 3:4]
    d = pts - eye
    return eye, d / np.linalg.norm(d, axis=1, keepdims=True)


# ---- intersections: t (inf = no entry point beyond T_MIN), part, for boxes a face-tie flag, and how far float32 may move t ---------------
# A quadratic's t = (-b - sqrt(h)) / a carries the rounding of h (and the rounding / float32 state error `pos_err` of the primitive's
# position) divided by sqrt(h): a ray that grazes a surface has an ill-conditioned t.  Linear hits (plane, caps, slabs) carry a few ulp.
def _entry(t):
    return np.where(t > T_MIN, t, np.inf)


def _quad_err(b, a, o2, r, h, t, pos_err):
    with np.errstate(divide="ignore", invalid="ignore"):
        return (8 * EPS32 * (b * b + a * (o2 + r * r)) + 4 * np.sqrt(a * o2) * pos_err) / (2 * a * np.sqrt(np.maximum(h, 1e-30))) + \
            8 * EPS32 * np.abs(t) + pos_err


def _sphere_t(c, r, eye, D, pos_err):
    oc = eye - c
    b = D @ oc
    h = b * b - (oc @ oc - r * r)
    with np.errstate(invalid="ignore"):
        t = _entry(np.where(h >= 0, -b - np.sqrt(h), np.inf))
    return t, _quad_err(b, 1.0, oc @ oc, r, h, t, pos_err)


def _hit(p, eye, D, pos_err):
    n = D.shape[0]
    part = np.zeros(n, np.int64)
    tie = np.zeros(n, bool)
    ty = p["type"]
    if ty == PLANE:
        with np.errstate(divide="ignore", invalid="ignore"):
            t = _entry(np.where(D[:, 2] < 0, (p["z"] - eye[2]) / D[:, 2], np.inf))
        hit = np.isfinite(t)
        P = eye + np.where(hit, t, 0.0)[:, None] * D
        cells = np.floor(P[:, 0] / p["period"]) + np.floor(P[:, 1] / p["period"])
        part = np.where(hit, np.mod(cells, 2), 0).astype(np.int64)
        return t, part, tie, 8 * EPS32 * np.abs(t) + pos_err
    if ty == SPHERE:
        t, err = _sphere_t(p["c"], p["r"], eye, D, pos_err)
        return t, part, tie, err
    if ty == CAPSULE:
        ax = p["e1"] - p["e0"]
        L = np.linalg.norm(ax)
        (t0, e0), (t1, e1) = _sphere_t(p["e0"], p["r"], eye, D, pos_err), _sphere_t(p["e1"], p["r"], eye, D, pos_err)
        if L > 0:       # the capsule's boundary holds only the outer half of each end sphere: an entry point between the ends is inside it
            with np.errstate(invalid="ignore"):
                t0 = np.where(((eye + np.where(np.isfinite(t0), t0, 0)[:, None] * D) - p["e0"]) @ ax <= 0, t0, np.inf)
                t1 = np.where(((eye + np.where(np.isfinite(t1), t1, 0)[:, None] * D) - p["e1"]) @ ax >= 0, t1, np.inf)
        ts, es = [t0, t1], [e0, e1]
        if L > 0:
            u = ax / L
            oa = eye - p["e0"]
            dperp = D - (D @ u)[:, None] * u
            operp = oa - (oa @ u) * u
            a = np.einsum("ij,ij->i", dperp, dperp)
            b = dperp @ operp
            h = b * b - a * (operp @ operp - p["r"] ** 2)
            with np.errstate(divide="ignore", invalid="ignore"):
                t = (-b - np.sqrt(h)) / a
                s = oa @ u + t * (D @ u)
            ts.append(_entry(np.where((h >= 0) & (a > 0) & (s > 0) & (s < L), t, np.inf)))
            es.append(_quad_err(b, a, oa @ oa, p["r"], h, t, pos_err))
        T = np.stack(ts)
        k = np.argmin(T, axis=0)
        return T[k, np.arange(n)], np.where(k == 2, 0, k + 1), tie, np.stack(es)[k, np.arange(n)]   # part 0 side, 1 end 0, 2 end 1
    if ty == CYL:
        ox, oy = eye[0] - p["cx"], eye[1] - p["cy"]
        a = D[:, 0] ** 2 + D[:, 1] ** 2
        b = ox * D[:, 0] + oy * D[:, 1]
        h = b * b - a * (ox * ox + oy * oy - p["r"] ** 2)
        with np.errstate(divide="ignore", invalid="ignore"):
            ts = (-b - np.sqrt(h)) / a
            zs = eye[2] + ts * D[:, 2]
            side = _entry(np.where((h >= 0) & (a > 0) & (zs >= p["z0"]) & (zs <= p["z1"]), ts, np.inf))
            caps = []
            for z, going in ((p["z1"], D[:, 2] < 0), (p["z0"], D[:, 2] > 0)):
                tc = (z - eye[2]) / D[:, 2]
                x, y = ox + tc * D[:, 0], oy + tc * D[:, 1]
                caps.append(_entry(np.where(going & (x * x + y * y <= p["r"] ** 2), tc, np.inf)))
        T = np.stack([side] + caps)
        k = np.argmin(T, axis=0)
        t = T[k, np.arange(n)]
        err = np.where(k == 0, _quad_err(b, a, ox * ox + oy * oy, p["r"], h, t, pos_err), 8 * EPS32 * np.abs(t) + pos_err)
        return t, k, tie, err                                             # part 0 side, 1 top, 2 bottom
    # BOX / OBOX: slabs in the box frame (world = c + R local)
    R, h = p["R"], p["half"]
    lo = R.T @ (eye - p["c"])
    ld = D @ R
    with np.errstate(divide="ignore", invalid="ignore"):
        t0 = (-h - lo) / ld
        t1 = (h - lo) / ld
    par = ld == 0
    inside = np.abs(lo) <= h
    near = np.where(par, np.where(inside, -np.inf, np.inf), np.minimum(t0, t1))
    far = np.where(par, np.where(inside, np.inf, -np.inf), np.maximum(t0, t1))
    order = np.argsort(near, axis=1)
    axis = order[:, 2]
    tn = near[np.arange(n), axis]
    second = near[np.arange(n), order[:, 1]]
    tf = far.min(axis=1)
    t = _entry(np.where(tn <= tf, tn, np.inf))
    part = axis * 2 + (ld[np.arange(n), axis] < 0)                          # entering through the -side (ld > 0) or the +side
    with np.errstate(invalid="ignore"):
        tie = np.isfinite(t) & (tn - second <= 1e-6 * np.maximum(np.abs(tn), 1.0))
    return t, part, tie, 8 * EPS32 * np.abs(t) + pos_err


def _normal(p, P, part):
    ty = p["type"]
    if ty == SPHERE:
        n = P - p["c"]
    elif ty == CAPSULE:
        ax = p["e1"] - p["e0"]
        L2 = ax @ ax
        s = np.clip(((P - p["e0"]) @ ax) / L2, 0.0, 1.0) if L2 > 0 else np.zeros(len(P))
        n = P - (p["e0"] + s[:, None] * ax)
    elif ty == CYL:
        n = np.stack([P[:, 0] - p["cx"], P[:, 1] - p["cy"], np.zeros(len(P))], axis=1)
        n[part == 1] = (0.0, 0.0, 1.0)
        n[part == 2] = (0.0, 0.0, -1.0)
    elif ty in (BOX, OBOX):
        axis, sign = part // 2, np.where(part % 2 == 1, 1.0, -1.0)
        n = p["R"][:, axis].T * sign[:, None]
    else:
        n = np.tile([0.0, 0.0, 1.0], (len(P), 1))
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def _bytes(col, n):
    shade = 0.55 + 0.45 * np.maximum(n @ LIGHT, 0.0)
    return np.clip(np.floor(col * shade[:, None] * 255.0 + 0.5), 0, 255).astype(np.uint8)


def _trace(prims, eye, D, pos_err):
    """Per ray: colour bytes and feature key (primitive, part) of the nearest hit; the second-nearest primitive's colour and whether it is
    within 1e-5 (relative); and a flag with an alternative colour where the winner's own colour sits on a rounding boundary (a box edge,
    the cylinder band, a checker cell boundary within float32 reach)."""
    n = D.shape[0]
    T = np.full((len(prims) + 1, n), np.inf)                                 # one row of misses: the second hit of a one-primitive list
    parts = np.zeros((len(prims) + 1, n), np.int64)
    ties = np.zeros((len(prims) + 1, n), bool)
    E = np.zeros((len(prims) + 1, n))
    for k, p in enumerate(prims):
        T[k], parts[k], ties[k], E[k] = _hit(p, eye, D, pos_err)
    order = np.argsort(T, axis=0, kind="stable")                            # stable: the earlier list index wins a tie
    idx = np.arange(n)
    background = np.floor(BACKGROUND * 255.0 + 0.5).astype(np.uint8)
    res = []
    for rank in (0, 1):
        win, t = order[rank], T[order[rank], idx]
        part = parts[win, idx]
        hit = np.isfinite(t)
        rgb = np.tile(background, (n, 1))
        alt = rgb.copy()
        flag = hit & ties[win, idx]                                          # box edge: the colour of either face
        for k in np.unique(win[hit]):
            m = np.nonzero(hit & (win == k))[0]
            p = prims[k]
            P = eye + t[m, None] * D[m]
            col = np.tile(p["rgb"], (len(m), 1))
            if p["type"] == PLANE:
                col[part[m] == 1] = p["rgb2"]
            nrm = _normal(p, P, part[m])
            rgb[m] = alt[m] = _bytes(col, nrm)
            if p["type"] == CYL:
                # srl_normal_at takes cap points with r^2 >= 0.9999 R^2 for side points, and side points whose float32 position has moved
                # inside that radius for cap points
                rho2 = (P[:, 0] - p["cx"]) ** 2 + (P[:, 1] - p["cy"]) ** 2
                band = (part[m] > 0) & (rho2 >= 0.9999 * p["r"] ** 2 * (1 - 1e-4))
                alt[m[band]] = _bytes(col[band], _normal(p, P[band], np.zeros(int(band.sum()), np.int64)))
                err_p = E[k, m] - pos_err + 4 * EPS32 * (np.linalg.norm(eye) + t[m])   # where the hit point sits on the cylinder
                inward = (part[m] == 0) & (err_p >= p["r"] * (1 - np.sqrt(0.9999)))
                cap = np.where(P[inward, 2] > 0.5 * (p["z0"] + p["z1"]), 1, 2)
                alt[m[inward]] = _bytes(col[inward], _normal(p, P[inward], cap))
                flag[m[band | inward]] = True
            elif p["type"] == PLANE and p["period"] > 0:
                # t = (z - eye_z) / d_z carries the rounding of d_z (a few 1e-7) relative to d_z itself: near the horizon the point moves
                # by metres, and the jittered rays, metres apart, say nothing about the cell it falls in
                err = 4e-6 * t[m] * (1.0 + 1.0 / np.abs(D[m, 2])) + 1e-6 * np.abs(P[:, :2]).max(axis=1)
                frac = P[:, :2] / p["period"]
                near = np.abs(frac - np.round(frac)).min(axis=1) * p["period"] <= err
                other = np.where(part[m][near, None] == 1, p["rgb"], p["rgb2"])
                alt[m[near]] = _bytes(other, nrm[near])
                flag[m[near]] = True
        res.append((np.where(hit, win, -1), part, t, rgb, alt, flag, E[win, idx]))
    (win, part, t, rgb, alt, flag, err), (_, _, t2, rgb2, _, _, err2) = res
    key = np.where(win >= 0, win * 16 + part, -1)
    with np.errstate(invalid="ignore"):
        close = np.isfinite(t2) & (t2 - t <= 1e-5 * np.abs(t) + err + err2)
    return rgb, key, rgb2, close, flag, alt


def render(prims, cam, W, H, pos_err=1e-6):
    """(frame u8[H, W, 3], unstable bool[H, W], candidates u8[H, W, N_CAND, 3], silhouette bool[H, W], unshaded colours of the primitives
    the centre and jittered rays hit [H, W, 5, 3]) of the primitive list through the camera dict `cam`
    (target, distance, yaw, pitch, roll, fov).  pos_err (m): how far the drawn primitives may sit from these float64 ones (float32
    positions, float32 forward kinematics), for the conditioning of the nearest-hit decision."""
    eye, D = camera_rays(cam, W, H)
    rgb, key, rgb2, close, flag, alt = _trace(prims, eye, D, pos_err)
    unstable = close | flag
    cands = [rgb]
    silhouette = np.zeros(len(key), bool)
    base = [_base_colour(prims, key)]
    for dx, dy in ((-JITTER, -JITTER), (JITTER, -JITTER), (-JITTER, JITTER), (JITTER, JITTER)):
        _, Dj = camera_rays(cam, W, H, dx, dy)
        rj, kj = _trace(prims, eye, Dj, pos_err)[:2]
        silhouette |= (kj != key) & ((kj < 0) | (key < 0) | (kj // 16 != key // 16))
        unstable |= kj != key
        cands.append(rj)
        base.append(_base_colour(prims, kj))
    cands.append(np.where(close[:, None], rgb2, rgb))
    cands.append(alt)
    shape = (H, W, N_CAND - 2, 3)
    return (rgb.reshape(H, W, 3), unstable.reshape(H, W), np.stack(cands, axis=1).reshape(H, W, N_CAND, 3), silhouette.reshape(H, W),
            np.stack(base, axis=1).reshape(shape))


def _base_colour(prims, key):
    """The unshaded colour of the primitive a ray hits (the background's for a miss; -1 for the plane, whose colour is its checker's)."""
    out = np.tile(BACKGROUND, (len(key), 1))
    for k, p in enumerate(prims):
        m = key // 16 == k
        out[m] = -1.0 if p["type"] == PLANE else p["rgb"]
    return out


def compare(frame, ref):
    """Check a rendered frame against render()'s output: every channel of a stable pixel within +-1 of the reference, every unstable pixel
    within +-1 of one of its candidates.  On a silhouette (the jittered rays see different primitives) the surface normal turns fast across
    the pixel, so a candidate primitive's colour is taken at any shade the light allows there (0.55 to 1).  Returns (number of failing pixels,
    unstable fraction, first failing (y, x) or None)."""
    rgb, unstable, cands, silhouette, base = ref
    f = frame.astype(np.int64)
    stable_ok = np.all(np.abs(f - rgb.astype(np.int64)) <= 1, axis=-1)
    cand_ok = np.any(np.all(np.abs(f[:, :, None, :] - cands.astype(np.int64)) <= 1, axis=-1), axis=-1)
    # shade s with |floor(c s 255 + 0.5) - f| <= 1 in every channel: s in [(f - 1.5) / (255 c), (f + 1.5) / (255 c)] where c > 0, f <= 1 where c = 0
    c = base * 255.0
    fb = f[:, :, None, :].astype(float)
    with np.errstate(divide="ignore", invalid="ignore"):
        lo = np.where(c > 0, (fb - 1.5) / c, -np.inf).max(axis=-1)
        hi = np.where(c > 0, (fb + 1.5) / c, np.inf).min(axis=-1)
    zero_ok = np.all((c > 0) | (fb <= 1), axis=-1)
    shaded = (base[..., 0] >= 0) & zero_ok & (np.maximum(lo, 0.55) <= np.minimum(hi, 1.0))
    cand_ok |= silhouette & np.any(shaded, axis=-1)
    ok = np.where(unstable, cand_ok, stable_ok)
    bad = np.argwhere(~ok)
    return int(len(bad)), float(unstable.mean()), (tuple(int(v) for v in bad[0]) if len(bad) else None)


# ---- a handle's state -> primitive lists ---------------------------------------------------------------------------------------------
def read_state(sim, env_id):
    """The fields the scene lists are built from, read with get_state on the handle that renders (float64 arrays, one row per env)."""
    from srl_sim import _abi
    if not env_id.startswith("Kuka"):
        return dict(robot=sim.get_state(_abi.F_ROBOT_POS), target=sim.get_state(_abi.F_TARGET_POS))
    st = dict(q=sim.get_state(_abi.F_JOINT_POS), base=sim.get_state(_abi.F_BUTTON_BASE), glider=sim.get_state(_abi.F_BUTTON_GLIDER)[:, 0])
    if env_id == "Kuka2ButtonGymEnv-v0":
        st["two"] = sim.get_state(_abi.F_TWO_BUTTON)
    return st


def env_prims(env_id, st, i, scene=None, bodies=None, targets=None):
    """Env i's primitive list from read_state()'s `st`.  bodies: [11, 9] of SRL_F_DISTRACTORS (or caller-given poses) for KukaRandButton;
    targets: both targets (t0x, t0y, t1x, t1y) of a MobileRobot2Target env (get_state returns only the current one)."""
    if env_id.startswith("Kuka"):
        from srl_sim.model import distractor_blob, load_kuka_scene
        b2 = None
        if "two" in st:
            b2 = (st["two"][i, 3], st["two"][i, 4], st["two"][i, 6])
        looks = distractor_blob().reshape(4, 32) if bodies is not None else None
        return kuka_prims(scene or load_kuka_scene(), st["q"][i], st["base"][i], st["glider"][i], b2, bodies, looks)
    kind = MOBILE_KIND[env_id]
    if kind == 1:
        return mobile_prims(kind, st["robot"][i], targets[:2], targets[2:4])
    return mobile_prims(kind, st["robot"][i], st["target"][i])


def sweep_cameras(env_id, n, seed):
    """n cameras over the scene: random targets, distances and yaws, roll in [-60, 60], fov 20 to 120, pitch in [-85, -5], and among them
    pitch exactly -90 and -89.9."""
    rs = np.random.RandomState(seed)
    kuka = env_id.startswith("Kuka")
    out = []
    for k in range(n):
        centre = np.array([0.5, 0.0, -0.15]) if kuka else np.array([2.0, 2.0, 0.0])
        target = centre + rs.uniform(-1, 1, 3) * (np.array([0.3, 0.4, 0.1]) if kuka else np.array([1.5, 1.5, 0.1]))
        pitch = (-90.0, -89.9)[k] if k < 2 else rs.uniform(-85, -5)
        out.append(dict(target=tuple(target), distance=rs.uniform(0.5, 1.8) if kuka else rs.uniform(1.5, 6.0), yaw=rs.uniform(0, 360),
                        pitch=pitch, roll=rs.uniform(-60, 60), fov=rs.uniform(20, 120)))
    return out
