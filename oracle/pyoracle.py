"""TEST INFRASTRUCTURE - ctypes binding of the CPU oracle (oracle/liboracle.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg import this.
The product package (mujoco_mpc_b200) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_dp = C.POINTER(C.c_double)


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".h", ".cc"))]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(so):
            build()
        _LIB = C.CDLL(so)
        _LIB.oracle_create.restype = C.c_void_p
        _LIB.oracle_create.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
        _LIB.oracle_destroy.argtypes = [C.c_void_p]
        _LIB.oracle_norm.restype = C.c_double
        _LIB.oracle_cost_value.restype = C.c_double
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _d(a):
    return None if a is None else np.ascontiguousarray(a, np.float64)


class Oracle:
    def __init__(self, blob: bytes, model, precision=64):
        self.m = model
        self.precision = precision
        self._blob = blob
        self.h = C.c_void_p(lib().oracle_create(blob, len(blob), precision))
        if not self.h:
            raise RuntimeError("oracle_create failed")
        self.ds = model.nq + model.nv
        self.n = 2 * model.nv

    def __del__(self):
        if getattr(self, "h", None):
            lib().oracle_destroy(self.h)
            self.h = None

    def set_task(self, weight=None, parameters=None, task_state=None, risk=None):
        w, p, s = _d(weight), _d(parameters), _d(task_state)
        lib().oracle_set_task(self.h, _p(w), _p(p), _p(s), C.c_double(self.m.task_risk if risk is None else risk))

    def _alloc(self, N, H, full):
        m = self.m
        out = dict(returns=np.zeros(N), failure=np.zeros(N, np.uint8))
        if full:
            out.update(states=np.zeros((N, H, self.ds)), actions=np.zeros((N, H, m.nu)), times=np.zeros((N, H)),
                       residual=np.zeros((N, H, m.task_num_residual)), costs=np.zeros((N, H)),
                       trace=np.zeros((N, H, 3 * m.task_num_trace)))
        return out

    def set_differentiable(self, on=True):
        """MakeDifferentiable (utilities.cc:60-75) on the oracle's model copy."""
        lib().oracle_set_differentiable(self.h, int(bool(on)))

    def set_xfrc_noise(self, std, rate=1.0, seed=0):
        """NoisyRollout perturbation (trajectory.cc:147-155) for the following rollout_spline calls; std 0 = off."""
        lib().oracle_set_xfrc_noise(self.h, C.c_double(std), C.c_double(rate), C.c_uint32(seed))

    def rollout_spline(self, state, time, mocap, knots, knot_times, interp, H, nthreads=1, full=True, userdata=None):
        knots = _d(knots)
        N, P, nu = knots.shape
        o = self._alloc(N, H, full)
        st, mc, kt = _d(state), _d(mocap), _d(knot_times)
        ud = _d(np.zeros(max(self.m.nuserdata, 1)) if userdata is None else userdata)
        g = lambda k: _p(o.get(k))
        lib().oracle_rollout_spline(self.h, _p(st), C.c_double(time), _p(mc), _p(ud), _p(knots), _p(kt), interp, P, N,
                                    H, nthreads, _p(o["returns"]), o["failure"].ctypes.data_as(C.POINTER(C.c_uint8)),
                                    g("states"), g("actions"), g("times"), g("residual"), g("costs"), g("trace"))
        return o

    def rollout_feedback(self, state, time, mocap, u_nom, x_nom, t_nom, gains, du, step_sizes, mode, nthreads=1,
                         full=True, userdata=None):
        u_nom, x_nom, t_nom, gains = _d(u_nom), _d(x_nom), _d(t_nom), _d(gains)
        du = _d(du) if du is not None else None
        step_sizes = _d(step_sizes)
        K, H = len(step_sizes), u_nom.shape[0]
        o = self._alloc(K, H, full)
        st, mc = _d(state), _d(mocap)
        ud = _d(np.zeros(max(self.m.nuserdata, 1)) if userdata is None else userdata)
        g = lambda k: _p(o.get(k))
        lib().oracle_rollout_feedback(self.h, _p(st), C.c_double(time), _p(mc), _p(ud), _p(u_nom), _p(x_nom),
                                      _p(t_nom), _p(gains), _p(du), _p(step_sizes), mode, K, H, nthreads,
                                      _p(o["returns"]), o["failure"].ctypes.data_as(C.POINTER(C.c_uint8)),
                                      g("states"), g("actions"), g("times"), g("residual"), g("costs"), g("trace"))
        return o

    def step_batch(self, qpos, qvel, ctrl, mocap, times, warmstart=None, nthreads=1):
        """B independent mj_steps from given states (teacher-forced per-step parity)."""
        m = self.m
        q, v, u, mc, t, ws = _d(qpos), _d(qvel), _d(ctrl), _d(mocap), _d(times), _d(warmstart)
        B = q.shape[0]
        o = dict(qacc=np.zeros((B, m.nv)), next_qpos=np.zeros((B, m.nq)), next_qvel=np.zeros((B, m.nv)),
                 residual=np.zeros((B, max(m.task_num_residual, 1))), cost=np.zeros(B))
        counts = np.zeros((B, 4), np.int32)
        lib().oracle_step_batch(self.h, B, _p(q), _p(v), _p(u), _p(ws), _p(mc), _p(t), int(nthreads), _p(o["qacc"]),
                                _p(o["next_qpos"]), _p(o["next_qvel"]), _p(o["residual"]), _p(o["cost"]),
                                counts.ctypes.data_as(C.POINTER(C.c_int)))
        o.update(ncon=counts[:, 0], nefc=counts[:, 1], niter=counts[:, 2], warning=counts[:, 3])
        return o

    def solver_hist(self, reset=True):
        h = (C.c_long * 64)()
        lib().oracle_solver_hist(h, int(reset))
        return np.array(h[:])

    def forward_debug(self, qpos, qvel, ctrl, mocap, time=0.0, warmstart=None):
        m = self.m
        o = dict(qacc=np.zeros(m.nv), qM=np.zeros((m.nv, m.nv)), qfrc_bias=np.zeros(m.nv), qfrc_smooth=np.zeros(m.nv),
                 residual=np.zeros(max(m.task_num_residual, 1)), efc_force=np.zeros(256), xpos=np.zeros((m.nbody, 3)),
                 subtree_com=np.zeros((m.nbody, 3)), contact=np.zeros((64, 8)), qfrc_constraint=np.zeros(m.nv),
                 next_qpos=np.zeros(m.nq), next_qvel=np.zeros(m.nv))
        nefc, ncon, niter = C.c_int(), C.c_int(), C.c_int()
        q, v, u, mc, ws = _d(qpos), _d(qvel), _d(ctrl), _d(mocap), _d(warmstart)
        rc = lib().oracle_forward_debug(self.h, _p(q), _p(v), _p(u), _p(mc), C.c_double(time), _p(ws), _p(o["qacc"]),
                                        _p(o["qM"]), _p(o["qfrc_bias"]), _p(o["qfrc_smooth"]), _p(o["residual"]),
                                        _p(o["efc_force"]), C.byref(nefc), C.byref(ncon), C.byref(niter),
                                        _p(o["xpos"]), _p(o["subtree_com"]), _p(o["contact"]),
                                        _p(o["qfrc_constraint"]), _p(o["next_qpos"]), _p(o["next_qvel"]))
        o.update(nefc=nefc.value, ncon=ncon.value, niter=niter.value, warning=rc)
        o["efc_force"] = o["efc_force"][: nefc.value]
        o["contact"] = o["contact"][: ncon.value]
        return o

    def efc_debug(self, qpos, qvel, ctrl, mocap, time=0.0, warmstart=None, cap_efc=256, cap_con=64):
        """The constraint problem of one mj_forward and the solver's answer.  Per row: efc_J [nefc, nv], efc_type,
        efc_id, efc_pos, efc_margin, efc_diagApprox, efc_R, efc_D, efc_aref, efc_force, efc_state, efc_frictionloss,
        efc_vel; per contact: efc_address, dim, geom1, geom2, mu, friction [5], frame [3, 3] (rows: normal, t1, t2),
        dist, pos; and qacc, qacc_smooth, qfrc_smooth, qM, nefc, ncon, niter, warning."""
        m = self.m
        nv = m.nv
        o = dict(qacc=np.zeros(nv), qacc_smooth=np.zeros(nv), qfrc_smooth=np.zeros(nv), qM=np.zeros((nv, nv)))
        J, ty, idx = np.zeros((cap_efc, nv)), np.zeros(cap_efc, np.int32), np.zeros(cap_efc, np.int32)
        row, ci, cr, counts = np.zeros((cap_efc, 10)), np.zeros((cap_con, 4), np.int32), np.zeros((cap_con, 19)), \
            np.zeros(4, np.int32)
        q, v, u, mc, ws = _d(qpos), _d(qvel), _d(ctrl), _d(mocap), _d(warmstart)
        ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))
        lib().oracle_forward_debug_efc(self.h, _p(q), _p(v), _p(u), _p(mc), C.c_double(time), _p(ws), int(cap_efc),
                                       int(cap_con), _p(o["qacc"]), _p(o["qacc_smooth"]), _p(o["qfrc_smooth"]),
                                       _p(o["qM"]), _p(J), ip(ty), ip(idx), _p(row), ip(ci), _p(cr), ip(counts))
        ne, nc = int(counts[0]), int(counts[1])
        assert ne <= cap_efc and nc <= cap_con, (ne, nc)
        o.update(nefc=ne, ncon=nc, niter=int(counts[2]), warning=int(counts[3]), efc_J=J[:ne], efc_type=ty[:ne],
                 efc_id=idx[:ne])
        for k, name in enumerate(("pos", "margin", "diagApprox", "R", "D", "aref", "force", "state", "frictionloss",
                                  "vel")):
            o["efc_" + name] = row[:ne, k]
        o["efc_state"] = o["efc_state"].astype(int)
        o.update(efc_address=ci[:nc, 0], dim=ci[:nc, 1], geom1=ci[:nc, 2], geom2=ci[:nc, 3], mu=cr[:nc, 0],
                 friction=cr[:nc, 1:6], frame=cr[:nc, 6:15].reshape(nc, 3, 3), dist=cr[:nc, 15], pos=cr[:nc, 16:19])
        return o

    def ilqg_policy_action(self, u_nom, x_nom, t_nom, gains, mode, step, state, time):
        """iLQGPolicy::Action of the oracle (fp64 handle only)."""
        assert self.precision == 64
        u, x, t, K, s = _d(u_nom), _d(x_nom), _d(t_nom), _d(gains), _d(state)
        out = np.zeros(self.m.nu)
        lib().oracle_ilqg_policy_action(self.h, _p(u), _p(x), _p(t), _p(K), len(t), int(mode), C.c_double(step), _p(s),
                                        C.c_double(time), _p(out))
        return out

    def cost_value(self, residual, terms=False):
        r = _d(residual)
        t = np.zeros(max(self.m.task_num_term, 1))
        v = lib().oracle_cost_value(self.h, _p(r), _p(t))
        return (v, t[: self.m.task_num_term]) if terms else v

    def model_derivatives(self, states, actions, times, mocap, tol=1e-6, skip=0, mode=0, nthreads=1):
        m = self.m
        H = states.shape[0]
        n, nu, nr = self.n, m.nu, m.task_num_residual
        A, B = np.zeros((H, n, n)), np.zeros((H, n, nu))
        Cm, D = np.zeros((H, nr, n)), np.zeros((H, nr, nu))
        s, a, t, mc = _d(states), _d(actions), _d(times), _d(mocap)
        lib().oracle_model_derivatives(self.h, _p(s), _p(a), _p(t), _p(mc), H, C.c_double(tol), _p(A), _p(B), _p(Cm), _p(D),
                                       int(skip), int(mode), int(nthreads))
        return A, B, Cm, D

    def cost_derivatives(self, residual, Cm, D):
        H, nr, n = Cm.shape
        nu = D.shape[2]
        cx, cu = np.zeros((H, n)), np.zeros((H, nu))
        cxx, cuu, cxu = np.zeros((H, n, n)), np.zeros((H, nu, nu)), np.zeros((H, n, nu))
        r, c, d = _d(residual), _d(Cm), _d(D)
        rc = lib().oracle_cost_derivatives(self.h, _p(r), _p(c), _p(d), H, n, nu, _p(cx), _p(cu), _p(cxx), _p(cuu), _p(cxu))
        assert rc == 0
        return cx, cu, cxx, cuu, cxu


def norm(x, params, ntype, grad=False, hess=False):
    x = _d(x)
    n = len(x)
    p = _d(np.zeros(3) if params is None else np.concatenate([params, np.zeros(3)]))
    g = np.zeros(n) if (grad or hess) else None
    H = np.zeros((n, n)) if hess else None
    y = lib().oracle_norm(_p(g), _p(H), _p(x), _p(p), n, int(ntype))
    return y, g, H


def spline_sample(times, values, interp, t):
    times, values = _d(times), _d(values)
    P, dim = values.shape
    out = np.zeros(dim)
    lib().oracle_spline_sample(_p(out), _p(times), _p(values), P, dim, int(interp), C.c_double(t))
    return out


def backward_pass(A, B, cx, cu, cxx, cxu, cuu, actions, ctrlrange, mu=0.0, reg_type=0, limits=1):
    H, n, m = B.shape[0], B.shape[1], B.shape[2]
    o = dict(Vx=np.zeros((H, n)), Vxx=np.zeros((H, n, n)), du=np.zeros((H, m)), K=np.zeros((H, m, n)), dV=np.zeros(2),
             Qx=np.zeros((H, n)), Qu=np.zeros((H, m)), Qxx=np.zeros((H, n, n)), Qxu=np.zeros((H, n, m)),
             Quu=np.zeros((H, m, m)))
    a = [_d(x) for x in (A, B, cx, cu, cxx, cxu, cuu, actions, ctrlrange)]
    lib().oracle_backward_pass.restype = C.c_int
    status = lib().oracle_backward_pass(*[_p(x) for x in a], n, m, H, C.c_double(mu), reg_type, limits, _p(o["Vx"]),
                                        _p(o["Vxx"]), _p(o["du"]), _p(o["K"]), _p(o["dV"]), _p(o["Qx"]), _p(o["Qu"]),
                                        _p(o["Qxx"]), _p(o["Qxu"]), _p(o["Quu"]))
    o["status"] = status
    return o


def count_flops(blob: bytes, state, time, mocap, knots, knot_times, interp, H):
    """Exact arithmetic-operation count per simulated env-step (instrumented scalar, oracle/counted.h)."""
    knots = _d(knots)
    N, P, nu = knots.shape
    st, mc, kt = _d(state), _d(mocap), _d(knot_times)
    ret = np.zeros(N)
    lib().oracle_count_flops.restype = C.c_double
    f = lib().oracle_count_flops(blob, C.c_size_t(len(blob)), _p(st), C.c_double(time), _p(mc), _p(knots), _p(kt),
                                 int(interp), P, N, int(H), _p(ret))
    return float(f), ret


def find_interval(seq, value):
    seq = _d(seq)
    b = (C.c_int * 2)()
    lib().oracle_find_interval(_p(seq), C.c_double(value), len(seq), b)
    return int(b[0]), int(b[1])


def interpolate(x, xs, ys, rep):
    xs, ys = _d(xs), _d(np.atleast_2d(np.asarray(ys, float).T).T if np.ndim(ys) == 1 else ys)
    dim = ys.shape[1]
    out = np.zeros(dim)
    lib().oracle_interpolate(_p(out), C.c_double(x), _p(xs), _p(ys), dim, len(xs), int(rep))
    return out
