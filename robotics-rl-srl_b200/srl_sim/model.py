"""
URDF loader -> flat model blob for the Kuka env kinds.

Replaces what the reference does through PyBullet at every reset -- ``p.loadSDF(kuka_with_gripper2.sdf)``
(environments/kuka_gym/kuka.py:60-71), ``p.loadURDF(table / simple_button)``, ``p.setGravity``
(environments/kuka_gym/kuka_button_gym_env.py:221-239) -- by a one-off, offline parse: links behind
fixed joints are merged into their parent, the 12 movable joints become the 12 bodies of a fixed-topology
tree, and everything the kernels need is packed into one float64 array (layout: csrc/kuka_model.h).
The controller constants of kuka.py (gains, forces, workspace box, initial pose) are packed alongside.
"""
import math
import os
import re
import xml.etree.ElementTree as ET

import numpy as np

ASSETS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "assets")
_HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "csrc", "kuka_model.h")


def _layout():
    """Read the KM_* offsets from csrc/kuka_model.h so loader and kernels cannot drift apart."""
    out = {}
    with open(_HEADER) as f:
        for m in re.finditer(r"#define\s+(KM_\w+)\s+([-0-9.eE]+)", f.read()):
            v = float(m.group(2))
            out[m.group(1)] = int(v) if v == int(v) and "." not in m.group(2) else v
    return out


KM = _layout()


# ---- small rigid-body helpers --------------------------------------------------------------------
def rpy_to_matrix(rpy):
    """URDF fixed-axis roll/pitch/yaw -> rotation matrix R = Rz(yaw) Ry(pitch) Rx(roll)."""
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = math.cos(r), math.sin(r), math.cos(p), math.sin(p), math.cos(y), math.sin(y)
    return np.array([[cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr],
                     [sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr],
                     [-sp, cp * sr, cp * cr]])


def quaternion_from_euler(rpy):
    """pybullet.getQuaternionFromEuler (x, y, z, w), same fixed-axis convention (kuka.py:144)."""
    r, p, y = [0.5 * v for v in rpy]
    cr, sr, cp, sp, cy, sy = math.cos(r), math.sin(r), math.cos(p), math.sin(p), math.cos(y), math.sin(y)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy,
                     cr * cp * cy + sr * sp * sy])


def _vec(s, n=3):
    v = [float(x) for x in s.split()]
    assert len(v) == n, s
    return np.array(v)


def _origin(elem):
    o = elem.find("origin") if elem is not None else None
    if o is None:
        return np.zeros(3), np.eye(3)
    return _vec(o.get("xyz", "0 0 0")), rpy_to_matrix(_vec(o.get("rpy", "0 0 0")))


class Link(object):
    def __init__(self, elem):
        self.name = elem.get("name")
        inertial = elem.find("inertial")
        self.mass = 0.0
        self.com = np.zeros(3)
        self.inertia = np.zeros((3, 3))  # about the COM, link-frame axes
        if inertial is not None:
            self.mass = float(inertial.find("mass").get("value"))
            self.com, R = _origin(inertial)
            i = inertial.find("inertia")
            I = np.array([[float(i.get("ixx")), float(i.get("ixy", 0)), float(i.get("ixz", 0))],
                          [float(i.get("ixy", 0)), float(i.get("iyy")), float(i.get("iyz", 0))],
                          [float(i.get("ixz", 0)), float(i.get("iyz", 0)), float(i.get("izz"))]])
            self.inertia = R @ I @ R.T
        self.collisions = []  # (kind, xyz, R, params)
        for c in elem.findall("collision"):
            xyz, R = _origin(c)
            g = c.find("geometry")
            if g.find("sphere") is not None:
                self.collisions.append(("sphere", xyz, R, (float(g.find("sphere").get("radius")),)))
            elif g.find("cylinder") is not None:
                cyl = g.find("cylinder")
                self.collisions.append(("cylinder", xyz, R, (float(cyl.get("radius")), float(cyl.get("length")))))
            elif g.find("box") is not None:
                self.collisions.append(("box", xyz, R, tuple(_vec(g.find("box").get("size")))))
            else:
                raise ValueError("unsupported collision geometry in link %s (meshes are not supported)" % self.name)


class Joint(object):
    def __init__(self, elem, index):
        self.index = index
        self.name = elem.get("name")
        self.type = elem.get("type")
        self.parent = elem.find("parent").get("link")
        self.child = elem.find("child").get("link")
        self.xyz, self.R = _origin(elem)
        ax = elem.find("axis")
        self.axis = _vec(ax.get("xyz")) if ax is not None else np.array([1.0, 0.0, 0.0])
        lim = elem.find("limit")
        self.lower = float(lim.get("lower", 0)) if lim is not None else 0.0
        self.upper = float(lim.get("upper", 0)) if lim is not None else 0.0
        dyn = elem.find("dynamics")
        self.damping = float(dyn.get("damping", 0)) if dyn is not None else 0.0
        if self.type not in ("revolute", "prismatic", "fixed", "continuous"):
            raise ValueError("unsupported joint type %s (%s)" % (self.type, self.name))


class Urdf(object):
    def __init__(self, path):
        root = ET.parse(path).getroot()
        self.name = root.get("name")
        self.links = {e.get("name"): Link(e) for e in root.findall("link")}
        self.joints = [Joint(e, i) for i, e in enumerate(root.findall("joint"))]
        children = {j.child for j in self.joints}
        roots = [n for n in self.links if n not in children]
        if len(roots) != 1:
            raise ValueError("%s: expected exactly one root link, found %s" % (path, roots))
        self.root = roots[0]
        self.child_joints = {}
        for j in self.joints:
            self.child_joints.setdefault(j.parent, []).append(j)


class Body(object):
    """A movable joint plus the rigid body behind it (its child link and every fixed-attached link)."""

    def __init__(self):
        self.parent = -1
        self.jtype = 0
        self.origin = np.zeros(3)
        self.rot = np.eye(3)
        self.axis = np.array([0.0, 0.0, 1.0])
        self.mass = 0.0
        self.com = np.zeros(3)
        self.inertia = np.zeros((3, 3))
        self.lower = self.upper = self.damping = 0.0
        self.ref_joint = -1
        self.link_names = []
        self.spheres = []  # (center in body frame, radius)
        self.link_frames = {}  # link name -> (p, R) in the body frame


def _merge_rigid(parts):
    """Combine (mass, com, inertia_about_com) triples expressed in one frame."""
    m = sum(p[0] for p in parts)
    if m <= 0.0:
        return 0.0, np.zeros(3), np.zeros((3, 3))
    com = sum(p[0] * p[1] for p in parts) / m
    I = np.zeros((3, 3))
    for mass, c, Ic in parts:
        d = c - com
        I += Ic + mass * (d.dot(d) * np.eye(3) - np.outer(d, d))
    return m, com, I


def build_bodies(urdf):
    """Flatten the link/joint tree into movable bodies, ordered by joint index (PyBullet order)."""
    bodies, body_of_link = [], {}

    def attach(body, link_name, p, R, parts):
        link = urdf.links[link_name]
        body.link_names.append(link_name)
        body.link_frames[link_name] = (p.copy(), R.copy())
        if link.mass > 0.0:
            parts.append((link.mass, p + R @ link.com, R @ link.inertia @ R.T))
        for kind, xyz, Rc, params in link.collisions:
            if kind == "sphere":
                body.spheres.append((p + R @ xyz, params[0]))
        for j in urdf.child_joints.get(link_name, []):
            if j.type == "fixed":
                attach(body, j.child, p + R @ j.xyz, R @ j.R, parts)
            else:
                pending.append((j, body, p + R @ j.xyz, R @ j.R))

    pending = []
    root_body = Body()  # the fixed base: keeps root-attached joints' origins
    attach(root_body, urdf.root, np.zeros(3), np.eye(3), [])
    movable = sorted(pending, key=lambda t: t[0].index)
    # breadth of `pending` grows while we attach children; process in joint-index order
    done = []
    while movable:
        j, pbody, p, R = movable.pop(0)
        b = Body()
        b.parent = -1 if pbody is root_body else bodies.index(pbody)
        b.jtype = 1 if j.type == "prismatic" else 0
        b.origin, b.rot, b.axis = p, R, j.axis / np.linalg.norm(j.axis)
        b.lower, b.upper, b.damping, b.ref_joint = j.lower, j.upper, j.damping, j.index
        bodies.append(b)
        pending = []
        parts = []
        attach(b, j.child, np.zeros(3), np.eye(3), parts)
        b.mass, b.com, b.inertia = _merge_rigid(parts)
        movable = sorted(movable + pending, key=lambda t: t[0].index)
        done.append(j.index)
    for i, b in enumerate(bodies):
        for n in b.link_names:
            body_of_link[n] = i
    if any(b.parent >= i for i, b in enumerate(bodies)):
        raise ValueError("joint order must list parents before children")
    return bodies, body_of_link


# ---- reference controller constants (environments/kuka_gym/kuka.py) -------------------------------
KUKA_INIT_JOINT_POSITIONS = [0.006418, 0.113184, -0.011401, -1.289317, 0.005379, 1.737684, -0.006539, 0.000048,
                             -0.299912, 0.000000, -0.000043, 0.299960, 0.000000, -0.000200]  # kuka.py:65-66
KUKA_MAX_VELOCITY = .35          # kuka.py:22
KUKA_MAX_FORCE = 200.            # kuka.py:23
KUKA_FINGER_A_FORCE = 2          # kuka.py:24
KUKA_FINGER_B_FORCE = 2.5        # kuka.py:25
KUKA_FINGER_TIP_FORCE = 2        # kuka.py:26
KUKA_END_EFFECTOR_INDEX = 6      # kuka.py:31
KUKA_GRIPPER_INDEX = 8           # kuka.py:32
PYBULLET_DEFAULT_KP, PYBULLET_DEFAULT_KD = 0.1, 1.0   # setJointMotorControl2 defaults (SURVEY Appendix B.2)
PYBULLET_DEFAULT_MAX_FORCE = 100000.0


class KukaScene(object):
    """Parsed scene: bodies, spheres, scene/controller constants and the packed ``blob``."""

    EXPECTED_PARENTS = [-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 7, 10]

    def __init__(self, kuka_urdf=None, button_urdf=None, table_urdf=None):
        kuka_urdf = kuka_urdf or os.path.join(ASSETS, "kuka_with_gripper2.urdf")
        button_urdf = button_urdf or os.path.join(ASSETS, "simple_button.urdf")
        table_urdf = table_urdf or os.path.join(ASSETS, "table.urdf")
        self.kuka = Urdf(kuka_urdf)
        self.bodies, self.body_of_link = build_bodies(self.kuka)
        if [b.parent for b in self.bodies] != self.EXPECTED_PARENTS:
            raise ValueError("the kernels are specialised for the 8-chain + two 2-link fingers topology; got parents %s"
                             % [b.parent for b in self.bodies])
        if any(b.jtype != 0 for b in self.bodies):
            raise ValueError("all Kuka joints must be revolute")
        self.ref_joints = [b.ref_joint for b in self.bodies]
        self.q_init = np.array([KUKA_INIT_JOINT_POSITIONS[j] for j in self.ref_joints])
        self.ee_body = self.ref_joints.index(KUKA_END_EFFECTOR_INDEX)
        self.gripper_body = self.ref_joints.index(KUKA_GRIPPER_INDEX)
        self.spheres = [(i, c, r) for i, b in enumerate(self.bodies) for (c, r) in b.spheres]
        if len(self.spheres) > KM["KM_MAX_SPHERES"]:
            raise ValueError("too many collision spheres (%d > %d)" % (len(self.spheres), KM["KM_MAX_SPHERES"]))
        self._controllers()
        self._scene(Urdf(button_urdf), Urdf(table_urdf))
        self.blob = self._pack()

    def _controllers(self):
        """kuka.py:165-187: (kp, kd, max force, max velocity, target selector) per movable joint."""
        ctrl = []
        for j in self.ref_joints:
            if j <= KUKA_END_EFFECTOR_INDEX:    # :167-170
                ctrl.append((0.3, 1.0, KUKA_MAX_FORCE, KUKA_MAX_VELOCITY, 0))
            elif j == 7:                        # :177-178
                ctrl.append((PYBULLET_DEFAULT_KP, PYBULLET_DEFAULT_KD, KUKA_MAX_FORCE, 0.0, 1))
            elif j == 8:                        # :179-180
                ctrl.append((PYBULLET_DEFAULT_KP, PYBULLET_DEFAULT_KD, KUKA_FINGER_A_FORCE, 0.0, 2))
            elif j == 11:                       # :181-182
                ctrl.append((PYBULLET_DEFAULT_KP, PYBULLET_DEFAULT_KD, KUKA_FINGER_B_FORCE, 0.0, 3))
            elif j in (10, 13):                 # :184-187
                ctrl.append((PYBULLET_DEFAULT_KP, PYBULLET_DEFAULT_KD, KUKA_FINGER_TIP_FORCE, 0.0, 4))
            else:
                raise ValueError("unexpected movable joint index %d" % j)
        self.ctrl = ctrl

    def _scene(self, button, table):
        sc = np.zeros(KM["KM_SCENE_SIZE"])
        sc[KM["KM_SC_BASE_POS"]:KM["KM_SC_BASE_POS"] + 3] = [-0.1, 0.0, -0.15]           # kuka.py:63
        sc[KM["KM_SC_GRAVITY_Z"]] = -10.0                                                  # kuka_button_gym_env.py:236
        sc[KM["KM_SC_TIMESTEP"]] = 1. / 240.                                               # :86
        sc[KM["KM_SC_SOLVER_ITERS"]] = 150                                                 # :219
        # table: top slab of table.urdf placed at (0.5, 0, -0.82)  (:223-224)
        table_pos = np.array([0.5, 0.0, -0.82])
        kind, xyz, R, size = [c for c in table.links[table.root].collisions if c[0] == "box"][0]
        sc[KM["KM_SC_TABLE_TOP_Z"]] = table_pos[2] + xyz[2] + size[2] / 2
        sc[KM["KM_SC_TABLE_XMIN"]] = table_pos[0] + xyz[0] - size[0] / 2
        sc[KM["KM_SC_TABLE_XMAX"]] = table_pos[0] + xyz[0] + size[0] / 2
        sc[KM["KM_SC_TABLE_YMIN"]] = table_pos[1] + xyz[1] - size[1] / 2
        sc[KM["KM_SC_TABLE_YMAX"]] = table_pos[1] + xyz[1] + size[1] / 2
        # button: base (+ fixed cylinder) stack and the prismatic button disc
        bbodies, blinks = build_bodies(button)
        if len(bbodies) != 1 or bbodies[0].jtype != 1:
            raise ValueError("the button must have exactly one prismatic joint")
        glider = bbodies[0]
        base_cyls = []  # (z0, z1, r) in the base frame for the base link and links fixed to it
        def collect(link_name, p):
            for kind, xyz, R, params in button.links[link_name].collisions:
                if kind == "cylinder":
                    base_cyls.append((p[2] + xyz[2] - params[1] / 2, p[2] + xyz[2] + params[1] / 2, params[0]))
            for j in button.child_joints.get(link_name, []):
                if j.type == "fixed":
                    collect(j.child, p + j.xyz)
        collect(button.root, np.zeros(3))
        disc = [c for c in button.links[glider.link_names[0]].collisions if c[0] == "cylinder"][0]
        stack_bottom = min(c[0] for c in base_cyls)
        # the button is spawned at Z_TABLE = -0.2 (:23,233), 5 mm inside the table top; it settles with the bottom of
        # its base on the table.  The base (10 kg, free body in Bullet) is treated as static at that rest pose.
        sc[KM["KM_SC_BUTTON_BASE"]:KM["KM_SC_BUTTON_BASE"] + 3] = [0.5, 0.0, sc[KM["KM_SC_TABLE_TOP_Z"]] - stack_bottom]
        sc[KM["KM_SC_GLIDER_Z"]] = glider.origin[2]
        sc[KM["KM_SC_GLIDER_LOWER"]] = glider.lower
        sc[KM["KM_SC_GLIDER_UPPER"]] = glider.upper
        sc[KM["KM_SC_BUTTON_MASS"]] = glider.mass
        sc[KM["KM_SC_DISC_RADIUS"]] = disc[3][0]
        sc[KM["KM_SC_DISC_Z0"]] = disc[1][2] - disc[3][1] / 2
        sc[KM["KM_SC_DISC_Z1"]] = disc[1][2] + disc[3][1] / 2
        sc[KM["KM_SC_STACK_RADIUS"]] = max(c[2] for c in base_cyls)
        sc[KM["KM_SC_STACK_TOP"]] = max(c[1] for c in base_cyls)
        sc[KM["KM_SC_CONTACT_DIST"]] = 0.02
        sc[KM["KM_SC_FRICTION"]] = 0.5 * 0.5
        sc[KM["KM_SC_ERP"]] = 0.2
        sc[KM["KM_SC_LIN_DAMPING"]] = 0.04
        sc[KM["KM_SC_ANG_DAMPING"]] = 0.04
        sc[KM["KM_SC_EE_INIT"]:KM["KM_SC_EE_INIT"] + 3] = [0.537, 0.0, 0.5]                # kuka.py:73
        sc[KM["KM_SC_BOX_SMALL"]:KM["KM_SC_BOX_SMALL"] + 6] = [0.50, 0.65, -0.17, 0.22, 0, 0.5]   # kuka.py:47-49
        sc[KM["KM_SC_BOX_LARGE"]:KM["KM_SC_BOX_LARGE"] + 6] = [0.35, 0.65, -0.30, 0.30, 0, 0.5]   # kuka.py:51-53
        sc[KM["KM_SC_IK_QUAT"]:KM["KM_SC_IK_QUAT"] + 4] = quaternion_from_euler([0, -math.pi, 0])  # kuka.py:144
        sc[KM["KM_SC_IK_DAMPING"]] = 0.00001                                               # kuka.py:42-43
        sc[KM["KM_SC_EE_BODY"]] = self.ee_body
        sc[KM["KM_SC_GRIPPER_BODY"]] = self.gripper_body
        sc[KM["KM_SC_TARGET_HEIGHT"]] = 0.28                                               # kuka_button_gym_env.py:35
        sc[KM["KM_SC_RAND_X"]] = 0.15                                                      # :230
        sc[KM["KM_SC_RAND_Y"]] = 0.3                                                       # :231
        sc[KM["KM_SC_BTN_IDLE_IMPULSE"]] = 1.0
        sc[KM["KM_SC_BTN_KP"]] = PYBULLET_DEFAULT_KP
        sc[KM["KM_SC_BTN_KD"]] = PYBULLET_DEFAULT_KD
        sc[KM["KM_SC_BTN_TARGET"]] = 0.1                                                   # :347
        sc[KM["KM_SC_BTN_MAXFORCE"]] = PYBULLET_DEFAULT_MAX_FORCE
        sc[KM["KM_SC_LIMIT_MAX_IMPULSE"]] = 100.0
        sc[KM["KM_SC_MAX_CONTACTS"]] = 4
        sc[KM["KM_SC_LIMIT_EPS"]] = 1e-6
        self.scene = sc

    def _pack(self):
        nb, ns = len(self.bodies), len(self.spheres)
        body_off = KM["KM_HEADER_SIZE"]
        ctrl_off = body_off + nb * KM["KM_BODY_STRIDE"]
        sph_off = ctrl_off + nb * KM["KM_CTRL_STRIDE"]
        scene_off = sph_off + KM["KM_MAX_SPHERES"] * KM["KM_SPHERE_STRIDE"]
        total = scene_off + KM["KM_SCENE_SIZE"]
        blob = np.zeros(total)
        blob[KM["KM_H_MAGIC"]] = KM["KM_MAGIC"]
        blob[KM["KM_H_VERSION"]] = KM["KM_VERSION"]
        blob[KM["KM_H_NBODY"]] = nb
        blob[KM["KM_H_NSPHERE"]] = ns
        blob[KM["KM_H_BODY_OFF"]] = body_off
        blob[KM["KM_H_CTRL_OFF"]] = ctrl_off
        blob[KM["KM_H_SPHERE_OFF"]] = sph_off
        blob[KM["KM_H_SCENE_OFF"]] = scene_off
        blob[KM["KM_H_TOTAL"]] = total
        for i, b in enumerate(self.bodies):
            r = blob[body_off + i * KM["KM_BODY_STRIDE"]: body_off + (i + 1) * KM["KM_BODY_STRIDE"]]
            r[KM["KM_B_PARENT"]] = b.parent
            r[KM["KM_B_JTYPE"]] = b.jtype
            r[KM["KM_B_ORIGIN"]:KM["KM_B_ORIGIN"] + 3] = b.origin
            r[KM["KM_B_ROT"]:KM["KM_B_ROT"] + 9] = b.rot.reshape(9)
            r[KM["KM_B_AXIS"]:KM["KM_B_AXIS"] + 3] = b.axis
            r[KM["KM_B_MASS"]] = b.mass
            r[KM["KM_B_COM"]:KM["KM_B_COM"] + 3] = b.com
            I = b.inertia
            r[KM["KM_B_INERTIA"]:KM["KM_B_INERTIA"] + 6] = [I[0, 0], I[0, 1], I[0, 2], I[1, 1], I[1, 2], I[2, 2]]
            r[KM["KM_B_LOWER"]] = b.lower
            r[KM["KM_B_UPPER"]] = b.upper
            r[KM["KM_B_DAMPING"]] = b.damping
            r[KM["KM_B_QINIT"]] = self.q_init[i]
            r[KM["KM_B_REFJOINT"]] = b.ref_joint
            c = blob[ctrl_off + i * KM["KM_CTRL_STRIDE"]: ctrl_off + (i + 1) * KM["KM_CTRL_STRIDE"]]
            c[:5] = self.ctrl[i]
        for k, (bi, c, rad) in enumerate(self.spheres):
            s = blob[sph_off + k * KM["KM_SPHERE_STRIDE"]: sph_off + (k + 1) * KM["KM_SPHERE_STRIDE"]]
            s[KM["KM_S_BODY"]] = bi
            s[KM["KM_S_CENTER"]:KM["KM_S_CENTER"] + 3] = c
            s[KM["KM_S_RADIUS"]] = rad
        blob[scene_off:scene_off + KM["KM_SCENE_SIZE"]] = self.scene
        return blob

    # ---- reference-side helpers used by tests / host classes ------------------------------------
    def forward_kinematics(self, q):
        """World pose (p, R) of every body frame for joint vector q[12] (numpy, float64)."""
        base = self.scene[KM["KM_SC_BASE_POS"]:KM["KM_SC_BASE_POS"] + 3]
        P, Rm = [], []
        for i, b in enumerate(self.bodies):
            pp, pr = (base, np.eye(3)) if b.parent < 0 else (P[b.parent], Rm[b.parent])
            a = b.axis
            c, s = math.cos(q[i]), math.sin(q[i])
            K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
            Rq = np.eye(3) + s * K + (1 - c) * (K @ K)
            P.append(pp + pr @ b.origin)
            Rm.append(pr @ b.rot @ Rq)
        return P, Rm


_default_scene = None


def load_kuka_scene():
    """The default scene (assets shipped with the package), cached."""
    global _default_scene
    if _default_scene is None:
        _default_scene = KukaScene()
    return _default_scene


# ---- KukaRandButtonGymEnv distractor bodies (csrc/distractor_core.h) ------------------------------------------------------------
# The reference loads pybullet_data's duck_vhacd.urdf, lego/lego.urdf, cube_small.urdf and sphere_small.urdf
# (kuka_rand_button_gym_env.py:58,68); neither the meshes nor the URDFs are available here.  The values below are RECALLED from
# pybullet_data (mass, size, colour) and unpinned like the rest of the Kuka restatement (SURVEY Appendix C); the collision geometry
# is a compound of at most 4 spheres per body, the way the arm's fingers are modelled.  Inertias are those of the solid shapes.
# name: (mass kg, lateral friction, [(cx, cy, cz, r)] in the link frame = COM frame, half extents for drawing, rgb, 0 box / 1 sphere)
DISTRACTOR_TYPES = ("duck_vhacd", "lego", "cube_small", "sphere_small")
_DISTRACTOR_ASSETS = {
    # a ~0.1 m duck: body and head
    "duck_vhacd": (0.1, 0.5, [(-0.01, 0.0, -0.005, 0.03), (0.025, 0.0, 0.035, 0.02), (-0.03, 0.0, 0.0, 0.025)],
                   (0.045, 0.03, 0.04), (1.0, 0.85, 0.0), 0),
    # a 2 x 2 brick, 32 x 32 x 19 mm: four spheres in a square (rests flat)
    "lego": (0.05, 0.5, [(sx * 0.008, sy * 0.008, 0.0, 0.0095) for sx in (-1, 1) for sy in (-1, 1)],
             (0.016, 0.016, 0.0095), (0.9, 0.1, 0.1), 0),
    # a 5 cm cube: four spheres of radius s/4 on alternate corners of the inner cube (their hull reaches every face)
    "cube_small": (0.1, 0.5, [(0.0125, 0.0125, 0.0125, 0.0125), (0.0125, -0.0125, -0.0125, 0.0125),
                              (-0.0125, 0.0125, -0.0125, 0.0125), (-0.0125, -0.0125, 0.0125, 0.0125)],
                   (0.025, 0.025, 0.025), (0.8, 0.8, 0.8), 0),
    # a 3 cm ball
    "sphere_small": (0.1, 0.5, [(0.0, 0.0, 0.0, 0.03)], (0.03, 0.03, 0.03), (0.3, 0.3, 0.9), 1),
}


def distractor_blob():
    """f64[4][32] asset blob of srl_sim_set_distractors (layout: csrc/distractor_core.h, DC_A_*)."""
    out = np.zeros((len(DISTRACTOR_TYPES), 32), np.float64)
    for t, name in enumerate(DISTRACTOR_TYPES):
        mass, mu, spheres, half, rgb, shape = _DISTRACTOR_ASSETS[name]
        if shape == 1:
            inertia = [0.4 * mass * half[0] ** 2] * 3
        else:
            a, b, c = (2 * h for h in half)
            inertia = [mass / 12.0 * (b * b + c * c), mass / 12.0 * (a * a + c * c), mass / 12.0 * (a * a + b * b)]
        row = out[t]
        row[0] = mass
        row[1:4] = inertia
        row[4] = mu
        row[5] = len(spheres)
        for k, sph in enumerate(spheres):
            row[6 + 4 * k:10 + 4 * k] = sph
        row[22:25] = half
        row[25:28] = rgb
        row[28] = shape
    return out.reshape(-1)


def scene_constants(scene):
    """Table top and button geometry of a loaded KukaScene, as the libraries read them from the blob."""
    g = lambda name: float(scene.scene[KM[name]])   # noqa: E731
    return dict(table_z=g("KM_SC_TABLE_TOP_Z"), txmin=g("KM_SC_TABLE_XMIN"), txmax=g("KM_SC_TABLE_XMAX"), tymin=g("KM_SC_TABLE_YMIN"),
                tymax=g("KM_SC_TABLE_YMAX"), button_z=float(scene.scene[KM["KM_SC_BUTTON_BASE"] + 2]), glider_z=g("KM_SC_GLIDER_Z"),
                disc_z0=g("KM_SC_DISC_Z0"), disc_z1=g("KM_SC_DISC_Z1"), disc_r=g("KM_SC_DISC_RADIUS"), stack_top=g("KM_SC_STACK_TOP"),
                stack_r=g("KM_SC_STACK_RADIUS"))
