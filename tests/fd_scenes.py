"""Scenes whose one-step transition Jacobians are known in closed form, for the finite-difference sweep
(csrc/ilqg_kernels.cuh fd_center_kernel / fd_column_kernel / fd_interp_kernel, oracle/ilqg.h model_derivatives).

Every scene is built from independent root bodies with one joint each and contacts off (joint_scenes.py), and uses the
PARTICLE_COPY residual r = (qpos, qvel).  One semi-implicit Euler step with implicit damping is

    v' = v + h (M + h b)^-1 f(q, v, u),    f = gravity - k (q - springref) - b v + sum gear clamp(u)
    q' = q (+) h v'

so per 1-dof unit, with c = h / (M + h b):  dv'/dq = c f_q,  dv'/dv = 1 - c b,  dv'/du = c gear,  dq'/d. = h dv'/d.
(plus dq'/dq = 1).  A free body (isotropic, centred, zero gravity, no damping) keeps its velocities, and its orientation
Q' = Q exp(h w) (w in the body frame) has, in the tangent space Q (+) d = Q exp(d):

    dtheta'/dtheta = R(h w)^T,    dtheta'/dw = h J_r(h w)      (J_r: the right Jacobian of SO(3))

A ball joint carrying a centred sphere obeys the same rotation law.  C is the derivative of the raw (qpos, qvel) at the
current state: identity on the scalar coordinates, 1/2 Q (x) (0, e_i) on a quaternion's rows; D = 0.

State order: A is [dq (nv); dv (nv)] x [dq; dv], B is [dq; dv] x nu (model_derivatives.cc / mjd_transitionFD).

Shared by tests/test_fd_derivatives_cpu.py and tests/test_gpu_fd_edges.py.
"""
import numpy as np

import joint_scenes as JS

EPS = 2.0 ** -10     # fp32-exact step: u0 +- EPS and the table's limits below are exact in fp32
H = JS.DT
G = JS.G


# ---------------------------------------------------------------------------------------------- SO(3)
def quat_mul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def quat_exp(phi):
    """exp of a rotation vector (the quaternion of a rotation by |phi| about phi)."""
    th = np.linalg.norm(phi)
    if th < 1e-300:
        return np.array([1.0, 0.0, 0.0, 0.0])
    return np.concatenate([[np.cos(th / 2)], np.sin(th / 2) * phi / th])


def quat_log(q):
    """Rotation vector of a unit quaternion (shortest rotation)."""
    q = q if q[0] >= 0 else -q
    s = np.linalg.norm(q[1:])
    if s < 1e-300:
        return np.zeros(3)
    return 2 * np.arctan2(s, q[0]) * q[1:] / s


def quat_conj(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def skew(a):
    return np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])


def rot(phi):
    """Rotation matrix of exp(phi) (Rodrigues)."""
    th = np.linalg.norm(phi)
    K = skew(phi)
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K


def right_jacobian(phi):
    """J_r with exp(phi + d) = exp(phi) exp(J_r(phi) d + O(d^2))."""
    th = np.linalg.norm(phi)
    K = skew(phi)
    if th < 1e-6:
        return np.eye(3) - 0.5 * K + K @ K / 6
    return np.eye(3) - (1 - np.cos(th)) / th ** 2 * K + (th - np.sin(th)) / th ** 3 * K @ K


# ---------------------------------------------------------------------------------------------- scenes
class Body:
    """One root body with one joint.  slide: along world x; hinge: about `axis` with the sphere at (d, 0, 0), so about
    y it is a pendulum under gravity (torque m g d cos q); ball / free: centred isotropic sphere."""

    def __init__(self, kind, m=1.0, r=0.1, d=0.0, axis="1 0 0", stiffness=0.0, springref=0.0, damping=0.0,
                 armature=0.0):
        self.kind, self.m, self.r, self.d, self.axis = kind, m, r, d, axis
        self.k, self.qs, self.b, self.arm = stiffness, springref, damping, armature

    nq = property(lambda s: {"slide": 1, "hinge": 1, "ball": 4, "free": 7}[s.kind])
    nv = property(lambda s: {"slide": 1, "hinge": 1, "ball": 3, "free": 6}[s.kind])

    def inertia(self):
        rot_i = 0.4 * self.m * self.r ** 2
        return {"slide": self.m, "hinge": rot_i + self.m * self.d ** 2, "ball": rot_i}.get(self.kind, None)

    def xml(self, k):
        ax = f' axis="{self.axis}"' if self.kind in ("slide", "hinge") else ""
        attrs = (f' stiffness="{self.k!r}" springref="{self.qs!r}" damping="{self.b!r}" armature="{self.arm!r}"'
                 if self.kind in ("slide", "hinge") else "")
        return (f'<body name="b{k}" pos="0 {0.5 * k} 1"><joint name="j{k}" type="{self.kind}"{ax}{attrs}/>'
                f'<geom type="sphere" size="{self.r}" mass="{self.m}" pos="{self.d} 0 0" contype="0" conaffinity="0"/>'
                f'</body>')


class Motor:
    """A motor on body `body`'s joint; ctrllimited None: MuJoCo's auto rule (limited when ctrlrange is given)."""

    def __init__(self, body, gear=1.0, ctrlrange=(-1.0, 1.0), ctrllimited=None):
        self.body, self.gear, self.lo, self.hi, self.ctrllimited = body, gear, ctrlrange[0], ctrlrange[1], ctrllimited

    @property
    def limited(self):
        return self.ctrllimited != "false"

    def clamp(self, u):
        return min(max(u, self.lo), self.hi) if self.limited else u

    def xml(self):
        a = f'<motor joint="j{self.body}" gear="{self.gear!r}" ctrlrange="{self.lo!r} {self.hi!r}"'
        if self.ctrllimited is not None:
            a += f' ctrllimited="{self.ctrllimited}"'
        return a + "/>"


class FdScene:
    """Bodies, motors, gravity on / off and one pose (q, v, u)."""

    def __init__(self, name, bodies, motors, q, v, u, gravity=True):
        self.name, self.bodies, self.motors, self.gravity = name, bodies, motors, gravity
        self.q, self.v, self.u = (np.asarray(x, float) for x in (q, v, u))
        self.qadr = np.cumsum([0] + [b.nq for b in bodies])[:-1]
        self.dadr = np.cumsum([0] + [b.nv for b in bodies])[:-1]
        self.nq, self.nv, self.nu = sum(b.nq for b in bodies), sum(b.nv for b in bodies), len(motors)

    def text(self):
        body = "".join(b.xml(k) for k, b in enumerate(self.bodies))
        acts = "".join(a.xml() for a in self.motors)
        return JS.scene_xml(self.name, bodies=body, actuator=acts, option="" if self.gravity else ' gravity="0 0 0"')

    def compile(self):
        return JS.compile_scene(self.text())

    @property
    def x(self):
        return np.concatenate([self.q, self.v])

    # ------------------------------------------------------------------ the step in numpy (fp64)
    def _scalar_force(self, k, q, v, u):
        b = self.bodies[k]
        f = -b.k * (q - b.qs) - b.b * v
        if b.kind == "hinge" and self.gravity:
            f += b.m * G * b.d * np.cos(q)
        for a, uu in zip(self.motors, u):
            if a.body == k:
                f += a.gear * a.clamp(uu)
        return f

    def step(self, q, v, u):
        """One semi-implicit Euler step with implicit damping (no ball / free passive forces, zero gravity on them)."""
        q2, v2 = q.copy(), v.copy()
        for k, b in enumerate(self.bodies):
            qa, da = self.qadr[k], self.dadr[k]
            if b.kind in ("slide", "hinge"):
                M = b.inertia() + b.arm
                v2[da] = v[da] + H / (M + H * b.b) * self._scalar_force(k, q[qa], v[da], u)
                q2[qa] = q[qa] + H * v2[da]
            elif b.kind == "ball":
                q2[qa:qa + 4] = quat_mul(q[qa:qa + 4], quat_exp(H * v[da:da + 3]))
            else:
                q2[qa:qa + 3] = q[qa:qa + 3] + H * v[da:da + 3]
                q2[qa + 3:qa + 7] = quat_mul(q[qa + 3:qa + 7], quat_exp(H * v[da + 3:da + 6]))
        return q2, v2

    def plus(self, q, dq):
        """q (+) dq in the tangent space (mj_integratePos with unit time)."""
        out = q.copy()
        for k, b in enumerate(self.bodies):
            qa, da = self.qadr[k], self.dadr[k]
            if b.kind == "ball":
                out[qa:qa + 4] = quat_mul(q[qa:qa + 4], quat_exp(dq[da:da + 3]))
            elif b.kind == "free":
                out[qa:qa + 3] += dq[da:da + 3]
                out[qa + 3:qa + 7] = quat_mul(q[qa + 3:qa + 7], quat_exp(dq[da + 3:da + 6]))
            else:
                out[qa] += dq[da]
        return out

    def minus(self, q1, q0):
        """q1 (-) q0 (mj_differentiatePos with unit time)."""
        out = np.zeros(self.nv)
        for k, b in enumerate(self.bodies):
            qa, da = self.qadr[k], self.dadr[k]
            if b.kind == "ball":
                out[da:da + 3] = quat_log(quat_mul(quat_conj(q0[qa:qa + 4]), q1[qa:qa + 4]))
            elif b.kind == "free":
                out[da:da + 3] = q1[qa:qa + 3] - q0[qa:qa + 3]
                out[da + 3:da + 6] = quat_log(quat_mul(quat_conj(q0[qa + 3:qa + 7]), q1[qa + 3:qa + 7]))
            else:
                out[da] = q1[qa] - q0[qa]
        return out

    # ------------------------------------------------------------------ closed forms
    def jacobians(self):
        """Closed-form A, B, C, D at the scene's pose (B: every control column at its full slope)."""
        nq, nv, nu = self.nq, self.nv, self.nu
        n = 2 * nv
        A, B = np.zeros((n, n)), np.zeros((n, nu))
        C, D = np.zeros((nq + nv, n)), np.zeros((nq + nv, nu))
        q, v = self.q, self.v
        for k, b in enumerate(self.bodies):
            qa, da = self.qadr[k], self.dadr[k]
            if b.kind in ("slide", "hinge"):
                M = b.inertia() + b.arm
                c = H / (M + H * b.b)
                fq = -b.k - (b.m * G * b.d * np.sin(q[qa]) if b.kind == "hinge" and self.gravity else 0.0)
                dvq, dvv = c * fq, 1 - c * b.b
                A[da, da], A[da, nv + da] = 1 + H * dvq, H * dvv
                A[nv + da, da], A[nv + da, nv + da] = dvq, dvv
                for i, a in enumerate(self.motors):
                    if a.body == k:
                        B[da, i], B[nv + da, i] = H * c * a.gear, c * a.gear
                C[qa, da] = 1
                continue
            # rotation block (ball: the whole joint; free: dofs 3..5), translation block (free: dofs 0..2)
            r0, qr = (da, qa) if b.kind == "ball" else (da + 3, qa + 3)
            w = v[r0:r0 + 3]
            A[r0:r0 + 3, r0:r0 + 3] = rot(H * w).T
            A[r0:r0 + 3, nv + r0:nv + r0 + 3] = H * right_jacobian(H * w)
            A[nv + r0:nv + r0 + 3, nv + r0:nv + r0 + 3] = np.eye(3)
            Q = q[qr:qr + 4]
            for i in range(3):
                C[qr:qr + 4, r0 + i] = 0.5 * quat_mul(Q, np.eye(4)[1 + i])
            if b.kind == "free":
                A[da:da + 3, da:da + 3] = np.eye(3)
                A[da:da + 3, nv + da:nv + da + 3] = H * np.eye(3)
                A[nv + da:nv + da + 3, nv + da:nv + da + 3] = np.eye(3)
                C[qa:qa + 3, da:da + 3] = np.eye(3)
        C[nq:, nv:] = np.eye(nv)
        return A, B, C, D

    def numeric_jacobians(self, eps=1e-6):
        """Centred fp64 differences of the numpy step and of r = (q, v) in the tangent space (checks the closed forms'
        sign and ordering conventions; the physics is checked against the oracle)."""
        nq, nv, nu = self.nq, self.nv, self.nu
        n = 2 * nv
        A, B = np.zeros((n, n)), np.zeros((n, nu))
        C = np.zeros((nq + nv, n))
        q0, v0, u0 = self.q, self.v, self.u
        qn, vn = self.step(q0, v0, u0)

        def diff(qa, va, qb, vb):
            return np.concatenate([self.minus(qa, qn) - self.minus(qb, qn), va - vb]) / (2 * eps)
        for j in range(n):
            d = np.zeros(n)
            d[j] = eps
            qp, vp = self.plus(q0, d[:nv]), v0 + d[nv:]
            qm, vm = self.plus(q0, -d[:nv]), v0 - d[nv:]
            A[:, j] = diff(*self.step(qp, vp, u0), *self.step(qm, vm, u0))
            C[:, j] = (np.concatenate([qp, vp]) - np.concatenate([qm, vm])) / (2 * eps)
        for i in range(nu):
            up, um = u0.copy(), u0.copy()
            up[i] += eps
            um[i] -= eps
            B[:, i] = diff(*self.step(q0, v0, up), *self.step(q0, v0, um))
        return A, B, C


def slide_scene():
    """Linear: spring, damping (implicit), armature, gear; a second slide with a negative gear and no ctrl limit."""
    bodies = [Body("slide", m=1.5, stiffness=30.0, springref=0.1, damping=2.0, armature=0.3),
              Body("slide", m=0.7, damping=0.5)]
    motors = [Motor(0, gear=2.5), Motor(1, gear=-1.5, ctrllimited="false")]
    return FdScene("fd_slide", bodies, motors, [0.2, -0.1], [-0.4, 0.7], [0.3, 2.0])


def pendulum_scene():
    """Nonlinear: a hinge about y carrying a sphere at d = 0.3 under gravity, with damping and armature."""
    bodies = [Body("hinge", m=1.0, r=0.05, d=0.3, axis="0 1 0", damping=0.1, armature=0.01)]
    return FdScene("fd_pendulum", bodies, [Motor(0, gear=1.5)], [0.6], [-1.2], [0.2])


W_ROT = np.array([6.0, -9.0, 12.0])     # |h w| = 0.16 rad: R(h w) and J_r(h w) are far from the identity


def free_scene():
    """A free body in zero gravity (plus a motorised slide, so the model has a control)."""
    bodies = [Body("free", m=1.0, r=0.1), Body("slide", m=1.0)]
    q = np.concatenate([[0.1, 0.2, 1.0], JS.QROT, [0.05]])
    v = np.concatenate([[0.3, -0.2, 0.1], W_ROT, [0.2]])
    return FdScene("fd_free", bodies, [Motor(1, gear=1.0)], q, v, [0.4], gravity=False)


def ball_scene():
    """A ball joint carrying a centred sphere in zero gravity (plus a motorised slide)."""
    bodies = [Body("slide", m=1.0), Body("ball", m=2.0, r=0.2)]
    q = np.concatenate([[-0.05], JS.QROT])
    v = np.concatenate([[0.1], -0.8 * W_ROT])
    return FdScene("fd_ball", bodies, [Motor(0, gear=1.0)], q, v, [-0.4], gravity=False)


# the control-limit table: (case, ctrlrange, ctrllimited, u0, expected B column / full slope)
def ctrl_cases(eps=EPS):
    return [
        ("interior", (-1.0, 1.0), None, 0.25, 1.0),
        ("at_hi", (-1.0, 1.0), None, 1.0, 1.0),                    # backward only
        ("hi_minus_half_eps", (-1.0, 1.0), None, 1.0 - eps / 2, 1.0),  # backward only; a clamped forward nudge: 0.5
        ("at_lo", (-1.0, 1.0), None, -1.0, 1.0),                  # forward only
        ("lo_plus_half_eps", (-1.0, 1.0), None, -1.0 + eps / 2, 1.0),
        ("narrower_than_eps", (0.0, eps / 4), None, eps / 8, 0.0),  # neither nudge stays inside
        ("outside", (-1.0, 1.0), None, 1.0 + eps / 2, 0.0),        # u0 itself outside (a backward nudge would give 0.5)
        ("unlimited_far_outside", (-1.0, 1.0), "false", 3.0, 1.0),
    ]


def ctrl_limit_scene(eps=EPS):
    """One slide per case of ctrl_cases, each with its own motor (gear 2, damping 0.5), at rest at q = 0: the next
    state is then the control's effect alone, so its fp32 round-off is relative to that effect."""
    cases = ctrl_cases(eps)
    n = len(cases)
    bodies = [Body("slide", m=1.0 + 0.1 * k, damping=0.5) for k in range(n)]
    motors = [Motor(k, gear=2.0, ctrlrange=c[1], ctrllimited=c[2]) for k, c in enumerate(cases)]
    return FdScene("fd_ctrl_limits", bodies, motors, np.zeros(n), np.zeros(n), [c[3] for c in cases])


def scenes():
    """name -> FdScene; linear scenes first (their secants are exact), then the nonlinear ones."""
    return {s.name: s for s in (slide_scene(), ctrl_limit_scene(), pendulum_scene(), free_scene(), ball_scene())}


LINEAR = ("fd_slide", "fd_ctrl_limits")
