"""MJCF-subset model compiler: XML -> flat structure-of-arrays model.

MuJoCo itself is not available offline (SURVEY.md section 0), so the rollout
engine needs its own loader for the handful of MJCF features the BASELINE
configs use.  Field names mirror ``mjModel`` (body_parentid, jnt_qposadr,
dof_invweight0, ...) so that a maintainer who *does* have MuJoCo can fill the
same blob straight from an ``mjModel`` (see INTEGRATION.md).

Host-side, offline: nothing here runs per planning iteration.  The compiled
model is serialised by :mod:`mujoco_mpc_b200.blob` and consumed by the CPU
oracle (``oracle/``) and by the CUDA engine (``csrc/``) through the C ABI.

Reference semantics followed (files of google-deepmind/mujoco_mpc):
  * cost terms from leading ``<sensor><user>`` entries: mjpc/task.cc:147-248
  * ``residual_*`` numerics -> task parameters:        mjpc/task.cc:38-64
  * trace sensors named ``trace%d``:                   mjpc/task.cc:190-198
"""
from __future__ import annotations

import math
import os
import xml.etree.ElementTree as ET

import numpy as np

# geom types (numbering as MuJoCo's mjtGeom)
GEOM_PLANE, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE, GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX = range(7)
GEOM_TYPES = {"plane": 0, "hfield": 1, "sphere": 2, "capsule": 3, "ellipsoid": 4, "cylinder": 5, "box": 6}
# joint types (mjtJoint)
JNT_FREE, JNT_BALL, JNT_SLIDE, JNT_HINGE = range(4)
JNT_TYPES = {"free": 0, "ball": 1, "slide": 2, "hinge": 3}
# sensor types (own enum; only what the residuals / traces read is evaluated)
SENS_USER, SENS_FRAMEPOS, SENS_JOINTPOS, SENS_TOUCH, SENS_SUBTREECOM, SENS_SUBTREELINVEL, \
    SENS_FRAMELINVEL, SENS_FRAMEQUAT, SENS_OTHER, SENS_JOINTVEL, SENS_ACCELEROMETER, SENS_VELOCIMETER, \
    SENS_GYRO = range(13)
SENS_TYPES = {"user": 0, "framepos": 1, "jointpos": 2, "touch": 3, "subtreecom": 4,
              "subtreelinvel": 5, "framelinvel": 6, "framequat": 7, "jointvel": 9, "accelerometer": 10,
              "velocimeter": 11, "gyro": 12}
# what the measurement path (engine step_sensors, estimators) evaluates
SENS_MEASURED = (SENS_FRAMEPOS, SENS_JOINTPOS, SENS_TOUCH, SENS_JOINTVEL, SENS_ACCELEROMETER, SENS_VELOCIMETER,
                 SENS_GYRO)
# the IMU sensors: 3-vectors in the frame of their site
SENS_IMU = (SENS_ACCELEROMETER, SENS_VELOCIMETER, SENS_GYRO)
SENS_DIM = {"framepos": 3, "jointpos": 1, "touch": 1, "subtreecom": 3, "subtreelinvel": 3,
            "framelinvel": 3, "framequat": 4, "jointvel": 1, "frameangvel": 3, "subtreeangmom": 3,
            "actuatorfrc": 1, "framexaxis": 3, "frameyaxis": 3, "framezaxis": 3, "velocimeter": 3,
            "gyro": 3, "accelerometer": 3, "actuatorpos": 1, "actuatorvel": 1, "tendonpos": 1}
OBJ_BODY, OBJ_XBODY, OBJ_GEOM, OBJ_SITE = range(4)

MINVAL = 1e-15
# narrow-phase pairs implemented by oracle and kernels (type1 <= type2)
SUPPORTED_PAIRS = {(GEOM_PLANE, GEOM_SPHERE), (GEOM_PLANE, GEOM_CAPSULE), (GEOM_PLANE, GEOM_BOX),
                   (GEOM_PLANE, GEOM_CYLINDER), (GEOM_SPHERE, GEOM_SPHERE),
                   (GEOM_SPHERE, GEOM_CAPSULE), (GEOM_SPHERE, GEOM_BOX),
                   (GEOM_CAPSULE, GEOM_CAPSULE)}


# ----------------------------------------------------------------------------- math helpers
def _f(s, n=None, default=None):
    if s is None:
        return None if default is None else np.array(default, dtype=float)
    v = np.array([float(x) for x in s.split()], dtype=float)
    if n is not None and len(v) < n and default is not None:
        d = np.array(default, dtype=float)
        d[: len(v)] = v
        v = d
    return v


def quat_mul(a, b):
    return np.array([
        a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
        a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
        a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
        a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def quat2mat(q):
    w, x, y, z = q
    return np.array([
        [w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


def mat2quat(R):
    # robust branch selection
    t = np.trace(R)
    if t > 0:
        s = math.sqrt(t + 1.0) * 2
        q = np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    elif R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = math.sqrt(1.0 + R[0, 0] - R[1, 1] - R[2, 2]) * 2
        q = np.array([(R[2, 1] - R[1, 2]) / s, 0.25 * s, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s])
    elif R[1, 1] > R[2, 2]:
        s = math.sqrt(1.0 + R[1, 1] - R[0, 0] - R[2, 2]) * 2
        q = np.array([(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, 0.25 * s, (R[1, 2] + R[2, 1]) / s])
    else:
        s = math.sqrt(1.0 + R[2, 2] - R[0, 0] - R[1, 1]) * 2
        q = np.array([(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, 0.25 * s])
    q = q / np.linalg.norm(q)
    if q[0] < 0:
        q = -q
    return q


def axisangle2quat(axis, angle):
    axis = np.asarray(axis, float)
    n = np.linalg.norm(axis)
    if n < MINVAL:
        return np.array([1.0, 0, 0, 0])
    axis = axis / n
    return np.concatenate([[math.cos(angle / 2)], math.sin(angle / 2) * axis])


def z2quat(vec):
    """Minimal rotation taking +z onto ``vec``."""
    vec = np.asarray(vec, float)
    n = np.linalg.norm(vec)
    if n < MINVAL:
        return np.array([1.0, 0, 0, 0])
    vec = vec / n
    z = np.array([0.0, 0, 1])
    axis = np.cross(z, vec)
    s = np.linalg.norm(axis)
    if s < 1e-10:
        return np.array([1.0, 0, 0, 0]) if vec[2] > 0 else np.array([0.0, 1, 0, 0])
    ang = math.atan2(s, vec[2])
    return axisangle2quat(axis / s, ang)


# <option><flag> switches the device and the oracle implement; every other flag must keep MuJoCo's default (the enable
# flags below default to "disable"; energy / fwdinv / invdiscrete only add diagnostics, so either value is accepted)
_FLAGS_HANDLED = ("contact", "eulerdamp", "frictionloss", "limit", "refsafe", "warmstart")
_FLAGS_ENABLE = ("override", "multiccd", "island", "sensornoise")
_FLAGS_DIAGNOSTIC = ("energy", "fwdinv", "invdiscrete")

# ----------------------------------------------------------------------------- defaults
_ACT_TAGS = ("general", "motor", "position", "velocity")
_DEF_TAGS = ("geom", "joint", "site", "tendon") + _ACT_TAGS


class _Defaults:
    def __init__(self):
        self.classes = {"main": {t: {} for t in ("geom", "joint", "site", "actuator", "tendon")}}

    def add(self, elem, parent=None):
        """Top-level <default> merges into "main"; a nested <default class=X> inherits its parent."""
        if parent is None:
            name = "main"
            cur = self.classes["main"]
        else:
            name = elem.get("class")
            cur = {k: dict(v) for k, v in self.classes[parent].items()}
        for child in elem:
            if child.tag in _DEF_TAGS:
                key = "actuator" if child.tag in _ACT_TAGS else child.tag
                cur[key].update(dict(child.attrib))
        self.classes[name] = cur
        for child in elem:
            if child.tag == "default":
                self.add(child, parent=name)

    def get(self, tag, cls):
        key = "actuator" if tag in _ACT_TAGS else tag
        return dict(self.classes.get(cls or "main", self.classes["main"]).get(key, {}))


def _expand_includes(root, basedir, files):
    """Splice <include file=.../> children in place (recursively)."""
    out = []
    for child in list(root):
        if child.tag == "include":
            fn = child.get("file")
            if files is not None and fn in files:
                sub = ET.fromstring(files[fn])
                _expand_includes(sub, basedir, files)
            else:
                path = os.path.join(basedir, fn)
                sub = ET.parse(path).getroot()
                _expand_includes(sub, os.path.dirname(path), files)
            out.extend(list(sub))
        else:
            _expand_includes(child, basedir, files)
            out.append(child)
    for c in list(root):
        root.remove(c)
    for c in out:
        root.append(c)


# ----------------------------------------------------------------------------- compiler
class Model(dict):
    """dict of numpy arrays / scalars with attribute access."""
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


def _geom_inertia(gtype, size, density, mass):
    """mass, diagonal inertia (geom frame, about geom centre)."""
    if gtype == GEOM_SPHERE:
        r = size[0]
        vol = 4.0 / 3.0 * math.pi * r ** 3
        m = mass if mass is not None else density * vol
        i = 0.4 * m * r * r
        return m, np.array([i, i, i])
    if gtype == GEOM_CAPSULE:
        r, h = size[0], size[1]
        vc = math.pi * r * r * 2 * h
        vs = 4.0 / 3.0 * math.pi * r ** 3
        rho = density if mass is None else mass / (vc + vs)
        mc, ms = rho * vc, rho * vs
        H = 2 * h
        izz = 0.5 * mc * r * r + 0.4 * ms * r * r
        ixx = mc * (H * H / 12 + r * r / 4) + ms * (0.4 * r * r + H * H / 4 + 3 * H * r / 8)
        return mc + ms, np.array([ixx, ixx, izz])
    if gtype == GEOM_CYLINDER:
        r, h = size[0], size[1]
        vol = math.pi * r * r * 2 * h
        m = mass if mass is not None else density * vol
        return m, np.array([m * (3 * r * r + 4 * h * h) / 12] * 2 + [0.5 * m * r * r])
    if gtype == GEOM_BOX:
        a, b, c = size[:3]
        m = mass if mass is not None else density * 8 * a * b * c
        return m, np.array([m * (b * b + c * c) / 3, m * (a * a + c * c) / 3, m * (a * a + b * b) / 3])
    if gtype == GEOM_ELLIPSOID:
        a, b, c = size[:3]
        m = mass if mass is not None else density * 4.0 / 3.0 * math.pi * a * b * c
        return m, np.array([m * (b * b + c * c) / 5, m * (a * a + c * c) / 5, m * (a * a + b * b) / 5])
    return 0.0, np.zeros(3)


class Compiler:
    def __init__(self, xml_text=None, path=None, files=None):
        if path is not None:
            root = ET.parse(path).getroot()
            basedir = os.path.dirname(os.path.abspath(path))
        else:
            root = ET.fromstring(xml_text)
            basedir = "."
        _expand_includes(root, basedir, files)
        self.root = root
        self.deg = True
        self.autolimits = True
        self.eulerseq = "xyz"
        self.defaults = _Defaults()

    # -------------------------------------------------------- orientation parsing
    def _ang(self, a):
        return a * math.pi / 180.0 if self.deg else a

    def _orient(self, a):
        if "quat" in a:
            q = _f(a["quat"])
            return q / np.linalg.norm(q)
        if "axisangle" in a:
            v = _f(a["axisangle"])
            return axisangle2quat(v[:3], self._ang(v[3]))
        if "euler" in a:
            e = [self._ang(x) for x in _f(a["euler"])]
            q = np.array([1.0, 0, 0, 0])
            for ch, ang in zip(self.eulerseq, e):
                ax = {"x": [1, 0, 0], "y": [0, 1, 0], "z": [0, 0, 1]}[ch.lower()]
                r = axisangle2quat(ax, ang)
                q = quat_mul(q, r) if ch.islower() else quat_mul(r, q)
            return q
        if "xyaxes" in a:
            v = _f(a["xyaxes"])
            x = v[:3] / np.linalg.norm(v[:3])
            y = v[3:] - np.dot(v[3:], x) * x
            y /= np.linalg.norm(y)
            return mat2quat(np.stack([x, y, np.cross(x, y)], axis=1))
        if "zaxis" in a:
            return z2quat(_f(a["zaxis"]))
        return np.array([1.0, 0, 0, 0])

    # -------------------------------------------------------- main entry
    def compile(self) -> Model:
        root = self.root
        for c in root.findall("compiler"):
            if "angle" in c.attrib:
                self.deg = c.get("angle") == "degree"
            if "autolimits" in c.attrib:
                self.autolimits = c.get("autolimits") == "true"
            if "eulerseq" in c.attrib:
                self.eulerseq = c.get("eulerseq")
        for d in root.findall("default"):
            self.defaults.add(d, parent=None)

        m = Model()
        m.model_name = root.get("model", "")
        # ---- options
        opt = dict(timestep=0.002, gravity=[0, 0, -9.81], cone=0, impratio=1.0, tolerance=1e-8,
                   ls_tolerance=0.01, iterations=100, ls_iterations=50, integrator=0,
                   disable_contact=0, disable_eulerdamp=0, disable_frictionloss=0, disable_limit=0,
                   disable_refsafe=0, disable_warmstart=0, o_margin=0.0)
        for o in root.findall("option"):
            for k in ("timestep", "impratio", "tolerance", "ls_tolerance", "o_margin"):
                if k in o.attrib:
                    opt[k] = float(o.get(k))
            for k in ("iterations", "ls_iterations"):
                if k in o.attrib:
                    opt[k] = int(o.get(k))
            if "gravity" in o.attrib:
                opt["gravity"] = list(_f(o.get("gravity")))
            if "cone" in o.attrib:
                opt["cone"] = 1 if o.get("cone") == "elliptic" else 0
            if "integrator" in o.attrib:
                opt["integrator"] = {"Euler": 0, "RK4": 1, "implicit": 2, "implicitfast": 3}[o.get("integrator")]
            for fl in o.findall("flag"):
                for k, v in fl.attrib.items():
                    if k in _FLAGS_HANDLED:
                        opt["disable_" + k] = int(v == "disable")
                    elif k not in _FLAGS_DIAGNOSTIC and v != ("disable" if k in _FLAGS_ENABLE else "enable"):
                        raise NotImplementedError(f'<flag {k}="{v}"/> is not supported (only {", ".join(_FLAGS_HANDLED)} '
                                                  "can be switched)")
        self.opt = opt

        # ---- body tree
        self.bodies, self.joints, self.geoms, self.sites = [], [], [], []
        world = dict(name="world", parent=0, pos=np.zeros(3), quat=np.array([1.0, 0, 0, 0]),
                     mocap=False, inertial=None, joints=[], geoms=[])
        self.bodies.append(world)
        for wb in root.findall("worldbody"):
            self._parse_body_children(wb, 0, None)

        self._finish_bodies(m)
        self._parse_tendons_excludes(m)
        self._parse_actuators(m)
        self._parse_sensors(m)
        self._parse_custom(m)
        self._parse_keys(m)
        for k, v in opt.items():
            m["opt_" + k] = np.array(v, dtype=float) if k == "gravity" else v
        self._constants(m)
        self._pairs(m)
        self._task(m)
        return m

    # -------------------------------------------------------- parsing helpers
    def _attrs(self, elem, tag, childclass):
        cls = elem.get("class", childclass)
        a = self.defaults.get(tag, cls)
        a.update(elem.attrib)
        return a

    def _parse_body_children(self, elem, bid, childclass):
        for ch in elem:
            if ch.tag == "geom":
                a = self._attrs(ch, "geom", childclass)
                a["_body"] = bid
                self.geoms.append(a)
                self.bodies[bid]["geoms"].append(len(self.geoms) - 1)
            elif ch.tag == "site":
                a = self._attrs(ch, "site", childclass)
                a["_body"] = bid
                self.sites.append(a)
            elif ch.tag in ("joint", "freejoint"):
                a = self._attrs(ch, "joint", childclass) if ch.tag == "joint" else dict(ch.attrib)
                if ch.tag == "freejoint":
                    a["type"] = "free"
                a["_body"] = bid
                self.joints.append(a)
                self.bodies[bid]["joints"].append(len(self.joints) - 1)
            elif ch.tag == "inertial":
                self.bodies[bid]["inertial"] = dict(ch.attrib)
            elif ch.tag == "body":
                cc = ch.get("childclass", childclass)
                b = dict(name=ch.get("name", f"body{len(self.bodies)}"), parent=bid,
                         pos=_f(ch.get("pos"), default=[0, 0, 0]), quat=self._orient(ch.attrib),
                         mocap=ch.get("mocap") == "true", inertial=None, joints=[], geoms=[])
                self.bodies.append(b)
                self._parse_body_children(ch, len(self.bodies) - 1, cc)

    def _finish_bodies(self, m):
        nbody = len(self.bodies)
        # ---------------- geoms
        ng = len(self.geoms)
        g_type = np.zeros(ng, np.int32); g_body = np.zeros(ng, np.int32)
        g_contype = np.ones(ng, np.int32); g_conaff = np.ones(ng, np.int32)
        g_condim = np.full(ng, 3, np.int32); g_prio = np.zeros(ng, np.int32); g_group = np.zeros(ng, np.int32)
        g_size = np.zeros((ng, 3)); g_pos = np.zeros((ng, 3)); g_quat = np.zeros((ng, 4))
        g_fric = np.zeros((ng, 3)); g_solmix = np.ones(ng); g_solref = np.zeros((ng, 2)); g_solimp = np.zeros((ng, 5))
        g_margin = np.zeros(ng); g_gap = np.zeros(ng)
        g_massprops = []
        names = []
        for i, a in enumerate(self.geoms):
            names.append(a.get("name", ""))
            t = GEOM_TYPES[a.get("type", "sphere")]
            size = _f(a.get("size"), 3, [0, 0, 0])
            pos = _f(a.get("pos"), default=[0, 0, 0])
            quat = self._orient(a)
            if "fromto" in a:
                ft = _f(a["fromto"])
                vec = ft[:3] - ft[3:]
                pos = 0.5 * (ft[:3] + ft[3:])
                quat = z2quat(vec)
                half = 0.5 * np.linalg.norm(vec)
                if t in (GEOM_CAPSULE, GEOM_CYLINDER):
                    size = np.array([size[0], half, 0.0])
                else:
                    size = np.array([size[0], size[1] if size[1] else size[0], half])
            g_type[i] = t; g_body[i] = a["_body"]; g_size[i] = size; g_pos[i] = pos; g_quat[i] = quat
            g_contype[i] = int(a.get("contype", 1)); g_conaff[i] = int(a.get("conaffinity", 1))
            g_condim[i] = int(a.get("condim", 3)); g_prio[i] = int(a.get("priority", 0))
            g_group[i] = int(a.get("group", 0))
            g_fric[i] = _f(a.get("friction"), 3, [1, 0.005, 0.0001])
            g_solmix[i] = float(a.get("solmix", 1)); g_solref[i] = _f(a.get("solref"), 2, [0.02, 1])
            g_solimp[i] = _f(a.get("solimp"), 5, [0.9, 0.95, 0.001, 0.5, 2])
            g_margin[i] = float(a.get("margin", 0)); g_gap[i] = float(a.get("gap", 0))
            mass = float(a["mass"]) if "mass" in a else None
            g_massprops.append(_geom_inertia(t, size, float(a.get("density", 1000)), mass))
        m.ngeom = ng
        m.geom_type, m.geom_bodyid, m.geom_contype, m.geom_conaffinity = g_type, g_body, g_contype, g_conaff
        m.geom_condim, m.geom_priority, m.geom_group = g_condim, g_prio, g_group
        m.geom_size, m.geom_pos, m.geom_quat, m.geom_friction = g_size, g_pos, g_quat, g_fric
        m.geom_solmix, m.geom_solref, m.geom_solimp, m.geom_margin, m.geom_gap = g_solmix, g_solref, g_solimp, g_margin, g_gap
        rb = np.zeros(ng)
        for i in range(ng):
            s = g_size[i]
            rb[i] = {GEOM_PLANE: 0.0, GEOM_SPHERE: s[0], GEOM_CAPSULE: s[0] + s[1],
                     GEOM_CYLINDER: math.hypot(s[0], s[1]), GEOM_BOX: float(np.linalg.norm(s)),
                     GEOM_ELLIPSOID: float(max(s))}.get(int(g_type[i]), 0.0)
        m.geom_rbound = rb
        m.geom_names = names

        # ---------------- sites
        ns = len(self.sites)
        m.nsite = ns
        m.site_bodyid = np.array([a["_body"] for a in self.sites], np.int32).reshape(ns)
        m.site_pos = np.array([_f(a.get("pos"), default=[0, 0, 0]) for a in self.sites]).reshape(ns, 3)
        m.site_quat = np.array([self._orient(a) for a in self.sites]).reshape(ns, 4)
        # the zone of touch sensors: mjtGeom type and size, MuJoCo's defaults (sphere, 0.005)
        m.site_type = np.array([GEOM_TYPES[a.get("type", "sphere")] for a in self.sites], np.int32).reshape(ns)
        m.site_size = np.array([_f(a.get("size"), 3, [0.005, 0.005, 0.005]) for a in self.sites]).reshape(ns, 3)
        m.site_names = [a.get("name", "") for a in self.sites]

        # ---------------- bodies
        b_parent = np.array([b["parent"] for b in self.bodies], np.int32)
        b_pos = np.array([b["pos"] for b in self.bodies]); b_quat = np.array([b["quat"] for b in self.bodies])
        b_ipos = np.zeros((nbody, 3)); b_iquat = np.tile([1.0, 0, 0, 0], (nbody, 1))
        b_mass = np.zeros(nbody); b_inertia = np.zeros((nbody, 3))
        b_mocapid = np.full(nbody, -1, np.int32)
        nmocap = 0
        for i, b in enumerate(self.bodies):
            if b["mocap"]:
                b_mocapid[i] = nmocap; nmocap += 1
            ine = b["inertial"]
            if ine is not None:
                b_mass[i] = float(ine["mass"]); b_ipos[i] = _f(ine.get("pos"), default=[0, 0, 0])
                if "fullinertia" in ine:
                    f = _f(ine["fullinertia"])
                    I = np.array([[f[0], f[3], f[4]], [f[3], f[1], f[5]], [f[4], f[5], f[2]]])
                    w, V = np.linalg.eigh(I)
                    order = np.argsort(-w); w = w[order]; V = V[:, order]
                    if np.linalg.det(V) < 0:
                        V[:, 2] = -V[:, 2]
                    b_inertia[i] = w; b_iquat[i] = mat2quat(V)
                else:
                    b_inertia[i] = _f(ine["diaginertia"]); b_iquat[i] = self._orient(ine)
            elif i > 0 and b["geoms"]:
                # inertia from geoms (compiler inertiafromgeom="auto")
                ms = [g_massprops[g][0] for g in b["geoms"]]
                M = sum(ms)
                if M > 0:
                    com = sum(mm * g_pos[g] for mm, g in zip(ms, b["geoms"])) / M
                    I = np.zeros((3, 3))
                    for mm, g in zip(ms, b["geoms"]):
                        R = quat2mat(g_quat[g]); d = g_pos[g] - com
                        I += R @ np.diag(g_massprops[g][1]) @ R.T + mm * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
                    w, V = np.linalg.eigh(I)
                    order = np.argsort(-w); w = w[order]; V = V[:, order]
                    if np.linalg.det(V) < 0:
                        V[:, 2] = -V[:, 2]
                    b_mass[i] = M; b_ipos[i] = com; b_inertia[i] = w; b_iquat[i] = mat2quat(V)
        m.nbody, m.nmocap = nbody, nmocap
        m.body_parentid, m.body_pos, m.body_quat, m.body_ipos, m.body_iquat = b_parent, b_pos, b_quat, b_ipos, b_iquat
        m.body_mass, m.body_inertia, m.body_mocapid = b_mass, b_inertia, b_mocapid
        m.body_names = [b["name"] for b in self.bodies]

        # ---------------- joints / dofs
        nj = len(self.joints)
        j_type = np.zeros(nj, np.int32); j_body = np.zeros(nj, np.int32)
        j_qadr = np.zeros(nj, np.int32); j_dadr = np.zeros(nj, np.int32)
        j_pos = np.zeros((nj, 3)); j_axis = np.zeros((nj, 3)); j_limited = np.zeros(nj, np.int32)
        j_range = np.zeros((nj, 2)); j_stiff = np.zeros(nj); j_margin = np.zeros(nj)
        j_solref = np.zeros((nj, 2)); j_solimp = np.zeros((nj, 5))
        qpos0, qspring = [], []
        d_body, d_jnt, d_damp, d_arm, d_floss, d_solref, d_solimp = [], [], [], [], [], [], []
        b_jntnum = np.zeros(nbody, np.int32); b_jntadr = np.full(nbody, -1, np.int32)
        b_dofnum = np.zeros(nbody, np.int32); b_dofadr = np.full(nbody, -1, np.int32)
        for j, a in enumerate(self.joints):
            t = JNT_TYPES[a.get("type", "hinge")]
            bid = a["_body"]
            j_type[j] = t; j_body[j] = bid; j_qadr[j] = len(qpos0); j_dadr[j] = len(d_body)
            if b_jntnum[bid] == 0:
                b_jntadr[bid] = j; b_dofadr[bid] = len(d_body)
            b_jntnum[bid] += 1
            j_pos[j] = _f(a.get("pos"), default=[0, 0, 0])
            ax = _f(a.get("axis"), default=[0, 0, 1])
            j_axis[j] = ax / max(np.linalg.norm(ax), MINVAL)
            rng = _f(a.get("range"), default=[0, 0])
            ref = float(a.get("ref", 0)); sref = float(a.get("springref", 0))
            if t in (JNT_HINGE, JNT_BALL):
                rng = np.array([self._ang(rng[0]), self._ang(rng[1])])
            if t == JNT_HINGE:
                ref, sref = self._ang(ref), self._ang(sref)
            j_range[j] = rng
            if "limited" in a and a["limited"] != "auto":
                j_limited[j] = 1 if a["limited"] == "true" else 0
            else:
                j_limited[j] = 1 if (self.autolimits and "range" in a) else 0
            j_stiff[j] = float(a.get("stiffness", 0)); j_margin[j] = float(a.get("margin", 0))
            if t in (JNT_FREE, JNT_BALL):
                # the limit rows (dev_model.h, oracle make_constraint) and the spring (k_smooth_forces, oracle passive)
                # are implemented for slide and hinge joints only: a quaternion limit or spring would be dropped
                kind = "ball" if t == JNT_BALL else "free"
                if j_limited[j]:
                    raise NotImplementedError(f"joint limits on a {kind} joint ({a.get('name', j)}) are not supported")
                if j_stiff[j] != 0:
                    raise NotImplementedError(f"stiffness on a {kind} joint ({a.get('name', j)}) is not supported")
            if "actuatorfrcrange" in a and a.get("actuatorfrclimited", "auto") != "false":
                raise NotImplementedError(f"actuatorfrcrange on joint {a.get('name', j)} is not supported")
            if a.get("actuatorgravcomp", "false") == "true":
                raise NotImplementedError(f"actuatorgravcomp on joint {a.get('name', j)} is not supported")
            j_solref[j] = _f(a.get("solreflimit"), 2, [0.02, 1])
            j_solimp[j] = _f(a.get("solimplimit"), 5, [0.9, 0.95, 0.001, 0.5, 2])
            ndof = {JNT_FREE: 6, JNT_BALL: 3, JNT_SLIDE: 1, JNT_HINGE: 1}[t]
            if t == JNT_FREE:
                qpos0 += list(self.bodies[bid]["pos"]) + list(self.bodies[bid]["quat"])
                qspring += list(self.bodies[bid]["pos"]) + list(self.bodies[bid]["quat"])
            elif t == JNT_BALL:
                qpos0 += [1, 0, 0, 0]; qspring += [1, 0, 0, 0]
            else:
                qpos0.append(ref); qspring.append(sref)
            for _ in range(ndof):
                d_body.append(bid); d_jnt.append(j)
                d_damp.append(float(a.get("damping", 0))); d_arm.append(float(a.get("armature", 0)))
                d_floss.append(float(a.get("frictionloss", 0)))
                d_solref.append(_f(a.get("solreffriction"), 2, [0.02, 1]))
                d_solimp.append(_f(a.get("solimpfriction"), 5, [0.9, 0.95, 0.001, 0.5, 2]))
            b_dofnum[bid] += ndof
        nv = len(d_body)
        m.njnt, m.nq, m.nv = nj, len(qpos0), nv
        m.jnt_type, m.jnt_bodyid, m.jnt_qposadr, m.jnt_dofadr = j_type, j_body, j_qadr, j_dadr
        m.jnt_pos, m.jnt_axis, m.jnt_limited, m.jnt_range = j_pos, j_axis, j_limited, j_range
        m.jnt_stiffness, m.jnt_margin, m.jnt_solref, m.jnt_solimp = j_stiff, j_margin, j_solref, j_solimp
        m.jnt_names = [a.get("name", "") for a in self.joints]
        m.qpos0 = np.array(qpos0, float); m.qpos_spring = np.array(qspring, float)
        m.body_jntnum, m.body_jntadr, m.body_dofnum, m.body_dofadr = b_jntnum, b_jntadr, b_dofnum, b_dofadr
        m.dof_bodyid = np.array(d_body, np.int32); m.dof_jntid = np.array(d_jnt, np.int32)
        m.dof_damping = np.array(d_damp, float); m.dof_armature = np.array(d_arm, float)
        m.dof_frictionloss = np.array(d_floss, float)
        m.dof_solref = np.array(d_solref, float).reshape(nv, 2); m.dof_solimp = np.array(d_solimp, float).reshape(nv, 5)
        # dof_parentid: previous dof along the kinematic chain
        dpar = np.full(nv, -1, np.int32)
        last_dof_of_body = np.full(nbody, -1, np.int32)  # last dof at or above this body
        for b in range(1, nbody):
            anc = last_dof_of_body[b_parent[b]]
            if b_dofnum[b] > 0:
                for k in range(b_dofnum[b]):
                    d = b_dofadr[b] + k
                    dpar[d] = anc if k == 0 else d - 1
                last_dof_of_body[b] = b_dofadr[b] + b_dofnum[b] - 1
            else:
                last_dof_of_body[b] = anc
        m.dof_parentid = dpar
        # root / weld ids, depth levels, subtree masses
        rootid = np.zeros(nbody, np.int32); weldid = np.zeros(nbody, np.int32); depth = np.zeros(nbody, np.int32)
        for b in range(1, nbody):
            p = b_parent[b]
            rootid[b] = b if p == 0 else rootid[p]
            weldid[b] = b if b_jntnum[b] > 0 else weldid[p]
            depth[b] = depth[p] + 1
        m.body_rootid, m.body_weldid, m.body_depth = rootid, weldid, depth
        sub = b_mass.copy()
        for b in range(nbody - 1, 0, -1):
            sub[b_parent[b]] += sub[b]
        m.body_subtreemass = sub

    def _parse_actuators(self, m):
        acts = []
        for sec in self.root.findall("actuator"):
            for ch in sec:
                if ch.tag not in _ACT_TAGS:
                    raise NotImplementedError(f"<{ch.tag}> actuators are not supported (only {', '.join(_ACT_TAGS)})")
                a = self.defaults.get(ch.tag, ch.get("class"))
                a.update(ch.attrib)
                a["_tag"] = ch.tag
                acts.append(a)
        nu = len(acts)
        m.nu, m.na = nu, 0
        trntype = np.zeros(nu, np.int32)        # 0 joint, 1 fixed tendon (mjTRN_JOINT / mjTRN_TENDON)
        trnid = np.zeros(nu, np.int32); gear = np.zeros(nu); gainprm = np.zeros((nu, 3)); biasprm = np.zeros((nu, 3))
        biastype = np.zeros(nu, np.int32); ctrllim = np.zeros(nu, np.int32); ctrlrange = np.zeros((nu, 2))
        frclim = np.zeros(nu, np.int32); frcrange = np.zeros((nu, 2))
        for i, a in enumerate(acts):
            tag = a["_tag"]
            name = a.get("name", str(i))
            # what the device and the oracle implement: a scalar gear on a slide / hinge joint or a fixed tendon, a
            # fixed gain, no activation dynamics, bias none or affine.  Anything else would simulate a different model.
            if "tendon" in a:
                trntype[i], trnid[i] = 1, m.tendon_names.index(a["tendon"])
            elif "joint" in a:
                trnid[i] = m.jnt_names.index(a["joint"])
                if m.jnt_type[trnid[i]] not in (JNT_SLIDE, JNT_HINGE):
                    raise NotImplementedError(f"actuator {name}: actuation of a ball or free joint is not supported")
            else:
                raise NotImplementedError(f"actuator {name}: only joint and tendon transmissions are supported")
            g = _f(a.get("gear"), default=[1])
            if np.any(g[1:] != 0):
                raise NotImplementedError(f"actuator {name}: a gear vector (gear=\"{a['gear']}\") is not supported, "
                                          "only a scalar gear")
            gear[i] = g[0]
            if tag == "general":
                for key, ok in (("gaintype", "fixed"), ("dyntype", "none")):
                    if a.get(key, ok) != ok:
                        raise NotImplementedError(f"actuator {name}: {key}=\"{a[key]}\" is not supported (only {ok})")
                if a.get("biastype", "none") not in ("none", "affine"):
                    raise NotImplementedError(f"actuator {name}: biastype=\"{a['biastype']}\" is not supported "
                                              "(only none and affine)")
            if tag == "position" and float(a.get("timeconst", 0)) > 0:
                raise NotImplementedError(f"actuator {name}: position timeconst (activation dynamics) is not supported")
            if tag == "position" and "dampratio" in a:
                raise NotImplementedError(f"actuator {name}: position dampratio is not supported")
            if float(a.get("inheritrange", 0)) != 0:
                raise NotImplementedError(f"actuator {name}: inheritrange is not supported (give ctrlrange explicitly)")
            if int(a.get("actdim", 0)) != 0 or a.get("actlimited", "false") == "true":
                raise NotImplementedError(f"actuator {name}: activation state (actdim / actlimited) is not supported")
            gp = _f(a.get("gainprm"), 3, [1, 0, 0]); bp = _f(a.get("biasprm"), 3, [0, 0, 0])
            bt = 1 if a.get("biastype", "none") == "affine" else 0
            if tag == "motor":
                gp, bp, bt = np.array([1.0, 0, 0]), np.zeros(3), 0
            elif tag == "position":
                kp = float(a.get("kp", 1)); kv = float(a.get("kv", 0))
                gp, bp, bt = np.array([kp, 0, 0]), np.array([0, -kp, -kv]), 1
            elif tag == "velocity":
                kv = float(a.get("kv", 1))
                gp, bp, bt = np.array([kv, 0, 0]), np.array([0, 0, -kv]), 1
            gainprm[i], biasprm[i], biastype[i] = gp, bp, bt
            ctrlrange[i] = _f(a.get("ctrlrange"), default=[0, 0])
            if "ctrllimited" in a and a["ctrllimited"] != "auto":
                ctrllim[i] = a["ctrllimited"] == "true"
            else:
                ctrllim[i] = 1 if (self.autolimits and "ctrlrange" in a) else 0
            frcrange[i] = _f(a.get("forcerange"), default=[0, 0])
            if "forcelimited" in a and a["forcelimited"] != "auto":
                frclim[i] = a["forcelimited"] == "true"
            else:
                frclim[i] = 1 if (self.autolimits and "forcerange" in a) else 0
        m.actuator_trnid, m.actuator_gear, m.actuator_gainprm, m.actuator_biasprm = trnid, gear, gainprm, biasprm
        m.actuator_trntype = trntype
        m.actuator_biastype, m.actuator_ctrllimited, m.actuator_ctrlrange = biastype, ctrllim, ctrlrange
        m.actuator_forcelimited, m.actuator_forcerange = frclim, frcrange
        m.actuator_names = [a.get("name", "") for a in acts]

    def _parse_tendons_excludes(self, m):
        excl = []
        for sec in self.root.findall("contact"):
            for ch in sec.findall("exclude"):
                excl.append((m.body_names.index(ch.get("body1")), m.body_names.index(ch.get("body2"))))
        m.exclude = excl
        # fixed tendons (length = sum coef * qpos of scalar joints); spatial tendons are not supported
        t_adr, t_num, w_dof, w_qadr, w_coef = [], [], [], [], []
        t_lim, t_range, t_margin, t_solref, t_solimp, names = [], [], [], [], [], []
        for sec in self.root.findall("tendon"):
            for ch in sec:
                if ch.tag != "fixed":
                    raise NotImplementedError("only <fixed> tendons are supported")
                a = self.defaults.get("tendon", ch.get("class", "main"))
                a.update(ch.attrib)
                if float(a.get("stiffness", 0)) != 0 or float(a.get("damping", 0)) != 0 or float(a.get("frictionloss", 0)) != 0:
                    raise NotImplementedError("tendon stiffness / damping / frictionloss are not supported")
                t_adr.append(len(w_dof)); names.append(ch.get("name", ""))
                for w in ch.findall("joint"):
                    j = m.jnt_names.index(w.get("joint"))
                    if m.jnt_type[j] not in (JNT_SLIDE, JNT_HINGE):
                        raise NotImplementedError("fixed tendons over free/ball joints")
                    w_dof.append(int(m.jnt_dofadr[j])); w_qadr.append(int(m.jnt_qposadr[j])); w_coef.append(float(w.get("coef")))
                t_num.append(len(w_dof) - t_adr[-1])
                rng = _f(a.get("range"), 2, [0, 0])
                lim = a.get("limited", "auto")
                t_lim.append(1 if lim == "true" or (lim == "auto" and "range" in a and self.autolimits) else 0)
                t_range.append(rng); t_margin.append(float(a.get("margin", 0)))
                t_solref.append(_f(a.get("solreflimit"), 2, [0.02, 1]))
                t_solimp.append(_f(a.get("solimplimit"), 5, [0.9, 0.95, 0.001, 0.5, 2]))
        nt = len(t_adr)
        m.ntendon = nt
        m.tendon_names = names
        m.tendon_adr, m.tendon_num = np.array(t_adr, np.int32), np.array(t_num, np.int32)
        m.wrap_dof, m.wrap_qposadr, m.wrap_coef = np.array(w_dof, np.int32), np.array(w_qadr, np.int32), np.array(w_coef, float)
        m.tendon_limited = np.array(t_lim, np.int32)
        m.tendon_range = np.array(t_range, float).reshape(nt, 2)
        m.tendon_margin = np.array(t_margin, float)
        m.tendon_solref = np.array(t_solref, float).reshape(nt, 2)
        m.tendon_solimp = np.array(t_solimp, float).reshape(nt, 5)

    def _parse_sensors(self, m):
        sens = []
        for sec in self.root.findall("sensor"):
            for ch in sec:
                sens.append(ch)
        n = len(sens)
        s_type = np.zeros(n, np.int32); s_dim = np.zeros(n, np.int32); s_adr = np.zeros(n, np.int32)
        s_objtype = np.full(n, -1, np.int32); s_objid = np.full(n, -1, np.int32); cutoff = np.zeros(n)
        users, adr = [], 0
        for i, ch in enumerate(sens):
            tag = ch.tag
            s_type[i] = SENS_TYPES.get(tag, SENS_OTHER)
            dim = int(ch.get("dim")) if tag == "user" else SENS_DIM.get(tag, 1)
            s_dim[i], s_adr[i] = dim, adr
            adr += dim
            users.append(_f(ch.get("user"), default=[]) if ch.get("user") else np.zeros(0))
            if tag in ("framepos", "framelinvel", "framequat"):
                ot = ch.get("objtype")
                nm = ch.get("objname")
                if ot == "site":
                    s_objtype[i], s_objid[i] = OBJ_SITE, m.site_names.index(nm)
                elif ot == "geom":
                    s_objtype[i], s_objid[i] = OBJ_GEOM, m.geom_names.index(nm)
                else:
                    s_objtype[i] = OBJ_XBODY if ot == "xbody" else OBJ_BODY
                    s_objid[i] = m.body_names.index(nm)
            elif tag in ("subtreecom", "subtreelinvel"):
                s_objtype[i], s_objid[i] = OBJ_BODY, m.body_names.index(ch.get("body"))
            elif tag in ("jointpos", "jointvel"):
                s_objid[i] = m.jnt_names.index(ch.get("joint"))
            elif tag in ("touch", "accelerometer", "velocimeter", "gyro"):
                s_objtype[i], s_objid[i] = OBJ_SITE, m.site_names.index(ch.get("site"))
            cutoff[i] = float(ch.get("cutoff", 0))
        nuser = max([len(u) for u in users] + [0])
        s_user = np.zeros((n, max(nuser, 1)))
        for i, u in enumerate(users):
            s_user[i, : len(u)] = u
        m.nsensor, m.nsensordata, m.nuser_sensor = n, adr, nuser
        m.sensor_type, m.sensor_dim, m.sensor_adr, m.sensor_objtype, m.sensor_objid = s_type, s_dim, s_adr, s_objtype, s_objid
        m.sensor_user = s_user
        m.sensor_cutoff = cutoff
        m.sensor_names = [ch.get("name", "") for ch in sens]

    def _parse_custom(self, m):
        num, txt = {}, {}
        order = []
        for sec in self.root.findall("custom"):
            for ch in sec:
                if ch.tag == "numeric":
                    num[ch.get("name")] = _f(ch.get("data"))
                    order.append(ch.get("name"))
                elif ch.tag == "text":
                    txt[ch.get("name")] = ch.get("data")
        m.numeric, m.text, m.numeric_order = num, txt, order
        m.nuserdata = 0
        for sec in self.root.findall("size"):
            if "nuserdata" in sec.attrib:
                m.nuserdata = int(sec.get("nuserdata"))

    def _parse_keys(self, m):
        keys = []
        for sec in self.root.findall("keyframe"):
            keys += list(sec.findall("key"))
        nk = len(keys)
        mp0 = np.array([m.body_pos[b] for b in range(m.nbody) if m.body_mocapid[b] >= 0]).reshape(-1)
        mq0 = np.array([m.body_quat[b] for b in range(m.nbody) if m.body_mocapid[b] >= 0]).reshape(-1)
        m.nkey = nk
        m.key_qpos = np.tile(m.qpos0, (max(nk, 1), 1))[:nk]
        m.key_qvel = np.zeros((nk, m.nv)); m.key_ctrl = np.zeros((nk, m.nu))
        m.key_mpos = np.tile(mp0, (max(nk, 1), 1))[:nk]; m.key_mquat = np.tile(mq0, (max(nk, 1), 1))[:nk]
        m.key_names = []
        for i, k in enumerate(keys):
            m.key_names.append(k.get("name", ""))
            for attr, arr in (("qpos", m.key_qpos), ("qvel", m.key_qvel), ("ctrl", m.key_ctrl),
                              ("mpos", m.key_mpos), ("mquat", m.key_mquat)):
                if k.get(attr) is not None:
                    arr[i] = _f(k.get(attr))
        m.mocap_pos0, m.mocap_quat0 = mp0.reshape(-1, 3), mq0.reshape(-1, 4)

    # -------------------------------------------------------- constants at qpos0 (mj_setConst analogue)
    def _constants(self, m):
        from .refmath import mass_matrix_and_jacobians
        M, Jb = mass_matrix_and_jacobians(m, m.qpos0)
        nv = m.nv
        if nv:
            Minv = np.linalg.inv(M)
            d_inv = np.diag(Minv).copy()
            # free / ball joints: average translational / rotational entries
            for j in range(m.njnt):
                a = m.jnt_dofadr[j]
                if m.jnt_type[j] == JNT_FREE:
                    d_inv[a:a + 3] = d_inv[a:a + 3].mean(); d_inv[a + 3:a + 6] = d_inv[a + 3:a + 6].mean()
                elif m.jnt_type[j] == JNT_BALL:
                    d_inv[a:a + 3] = d_inv[a:a + 3].mean()
            m.dof_invweight0 = d_inv
            biw = np.zeros((m.nbody, 2))
            for b in range(1, m.nbody):
                if m.body_weldid[b] == 0:
                    continue
                A = Jb[b] @ Minv @ Jb[b].T
                biw[b, 0] = max(MINVAL, (A[0, 0] + A[1, 1] + A[2, 2]) / 3)
                biw[b, 1] = max(MINVAL, (A[3, 3] + A[4, 4] + A[5, 5]) / 3)
            m.body_invweight0 = biw
            m.stat_meaninertia = float(np.mean(np.diag(M)))
            # tendon_invweight0 = J M^-1 J^T at qpos0 (set0 in MuJoCo's compiler)
            tiw = np.zeros(m.ntendon)
            for t in range(m.ntendon):
                J = np.zeros(nv)
                for w in range(m.tendon_adr[t], m.tendon_adr[t] + m.tendon_num[t]):
                    J[m.wrap_dof[w]] += m.wrap_coef[w]
                tiw[t] = max(MINVAL, float(J @ Minv @ J))
            m.tendon_invweight0 = tiw
        else:
            m.dof_invweight0 = np.zeros(0); m.body_invweight0 = np.zeros((m.nbody, 2)); m.stat_meaninertia = 1.0
            m.tendon_invweight0 = np.zeros(m.ntendon)
        m.M0 = M

    # -------------------------------------------------------- static candidate pair list
    def _pairs(self, m):
        pairs, dropped = [], []
        if not self.opt["disable_contact"]:
            for i in range(m.ngeom):
                for j in range(i + 1, m.ngeom):
                    b1, b2 = m.geom_bodyid[i], m.geom_bodyid[j]
                    w1, w2 = m.body_weldid[b1], m.body_weldid[b2]
                    if w1 == w2:                       # same body / both static
                        continue
                    if not ((m.geom_contype[i] & m.geom_conaffinity[j]) or (m.geom_contype[j] & m.geom_conaffinity[i])):
                        continue
                    # parent-child filter (unless the parent is the world)
                    if w1 != 0 and w2 != 0 and (m.body_weldid[m.body_parentid[w2]] == w1 or m.body_weldid[m.body_parentid[w1]] == w2):
                        continue
                    if (b1, b2) in m.exclude or (b2, b1) in m.exclude:
                        continue
                    g1, g2 = (i, j) if m.geom_type[i] <= m.geom_type[j] else (j, i)
                    key = (int(m.geom_type[g1]), int(m.geom_type[g2]))
                    if key not in SUPPORTED_PAIRS:
                        dropped.append((g1, g2))
                        continue
                    if self.pair_filter is not None and not self.pair_filter(m, g1, g2):
                        dropped.append((g1, g2))
                        continue
                    pairs.append((g1, g2))
        m.npair = len(pairs)
        m.pair_geom1 = np.array([p[0] for p in pairs], np.int32).reshape(-1)
        m.pair_geom2 = np.array([p[1] for p in pairs], np.int32).reshape(-1)
        m.pairs_dropped = dropped

    pair_filter = None

    # -------------------------------------------------------- task spec (mjpc/task.cc:147-248)
    def _task(self, m):
        num_term = 0
        for i in range(m.nsensor):
            if m.sensor_type[i] != SENS_USER:
                break
            num_term += 1
        from .task import norm_parameter_dimension
        dims, norms, weights, nparams, params = [], [], [], [], []
        for i in range(num_term):
            s = m.sensor_user[i]
            nt = int(s[0])
            npd = norm_parameter_dimension(nt)
            if 4 + npd > m.nuser_sensor and npd > 0:
                raise ValueError("Cost construction from XML: Missing parameter value (sensor %d)" % i)
            for j in range(npd):
                if s[4 + j] <= 0.0:
                    raise ValueError("Cost construction from XML: Missing parameter value (sensor %d)" % i)
            dims.append(int(m.sensor_dim[i])); norms.append(nt); weights.append(float(s[1]))
            nparams.append(npd); params += list(s[4:4 + npd])
        m.task_num_term = num_term
        m.task_num_residual = int(sum(dims))
        m.task_dim_norm_residual = np.array(dims, np.int32).reshape(-1)
        m.task_norm = np.array(norms, np.int32).reshape(-1)
        m.task_weight = np.array(weights, float).reshape(-1)
        m.task_num_norm_parameter = np.array(nparams, np.int32).reshape(-1)
        m.task_norm_parameter = np.array(params, float).reshape(-1)
        m.task_weight_names = m.sensor_names[:num_term]
        if num_term == 0:   # the particle residual (id 0) would write nq + nv entries into an empty residual
            from .task import RESIDUAL_NONE
            m.task_residual_id = RESIDUAL_NONE
        m.task_risk = float(m.numeric.get("task_risk", [0.0])[0])
        # residual parameters: every numeric whose name starts with residual_ (task.cc:38-64)
        pars, pnames = [], []
        for name in m.numeric_order:
            if name.startswith("residual_"):
                pnames.append(name)
                v = m.numeric[name][0]
                if name.startswith("residual_select_"):
                    # selection parameters are ints bit-reinterpreted as doubles in the reference
                    # (utilities.cc:118-124); we keep the integer value as a double.
                    v = float(int(v))
                pars.append(v)
        m.task_parameters = np.array(pars, float).reshape(-1)
        m.task_parameter_names = pnames
        traces = [i for i in range(m.nsensor) if m.sensor_names[i].startswith("trace")]
        m.task_num_trace = len(traces)
        tr_type, tr_id = [], []
        for i in traces:
            tr_type.append(int(m.sensor_objtype[i])); tr_id.append(int(m.sensor_objid[i]))
        m.task_trace_objtype = np.array(tr_type, np.int32).reshape(-1)
        m.task_trace_objid = np.array(tr_id, np.int32).reshape(-1)


def compile_xml(xml_text=None, path=None, files=None, pair_filter=None) -> Model:
    c = Compiler(xml_text=xml_text, path=path, files=files)
    c.pair_filter = pair_filter
    return c.compile()
