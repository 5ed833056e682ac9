"""ctypes binding of libmjpc_b200.so - the reference-facing call a user makes.

Every method goes through the C ABI in include/mjpc_b200.h; there is no Python/NumPy compute path and no
CPU fallback: if the library is missing or no CUDA device is visible, construction raises.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import re

import numpy as np

from .blob import to_blob
from .build import HERE, SO

HEADER = os.path.join(HERE, "..", "include", "mjpc_b200.h")

_fp = C.POINTER(C.c_float)
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_bp = C.POINTER(C.c_uint8)


class ModelBlob(C.Structure):
    _fields_ = [("data", C.c_void_p), ("nbytes", C.c_size_t)]


class TaskDesc(C.Structure):
    _fields_ = [("weight", _dp), ("parameters", _dp), ("task_state", _dp), ("risk", C.c_double)]


class Info(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("nq", "nv", "nu", "na", "nmocap", "nuserdata", "dim_state", "dim_dstate",
                                       "num_residual", "num_term", "num_trace", "num_parameters", "task_state_size",
                                       "max_candidates", "max_horizon", "device", "smem_bytes_per_warp")]


_SCALARS = {"int": C.c_int, "double": C.c_double, "float": C.c_float, "uint32_t": C.c_uint32, "size_t": C.c_size_t,
            "int64_t": C.c_int64, "uint8_t": C.c_uint8}
_STRUCTS = {"mjpc_model_blob": ModelBlob, "mjpc_task_desc": TaskDesc, "mjpc_b200_info": Info}
_HANDLES = {"mjpc_b200_t", "mjpc_b200_planner_t", "mjpc_b200_batch_planner_t", "mjpc_b200_estimator_t", "void"}


def _ctype(decl, text, is_return):
    """The ctypes type of one C type as the header writes it (`const` ignored, any spacing around `*`)."""
    words = text.replace("*", " * ").split()
    stars = words.count("*")
    base = " ".join(w for w in words if w not in ("const", "*"))
    if is_return and base == "void" and not stars:
        return None
    if is_return and stars:   # raw addresses, strings aside
        return C.c_char_p if (base, stars) == ("char", 1) else C.c_void_p
    if not stars and base in _SCALARS:
        return _SCALARS[base]
    if stars == 1 and base in _SCALARS:
        return C.POINTER(_SCALARS[base])
    if stars == 1 and base in _STRUCTS:
        return C.POINTER(_STRUCTS[base])
    if base in _HANDLES and stars in (1, 2):
        return C.c_void_p if stars == 1 else C.POINTER(C.c_void_p)
    raise TypeError(f"include/mjpc_b200.h: no ctypes type for '{text.strip()}' in `{decl}`")


def parse_header(text):
    """{name: (restype, argtypes)} of every `<return type> mjpc_b200_<name>(<parameters>);` the header text declares.
    A type the binding has no ctypes type for raises TypeError naming the declaration."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^\s*#[^\n]*", " ", text, flags=re.M)
    protos = {}
    for m in re.finditer(r"([A-Za-z_][\w\s*]*?)\b(mjpc_b200_\w+)\s*\(([^()]*)\)\s*;", text):
        decl = " ".join(m.group(0).split())
        params = [p for p in m.group(3).split(",") if p.split() != ["void"]]
        argtypes = [_ctype(decl, re.sub(r"\w+\s*$", "", p), False) for p in params]   # `<type> <name>`
        protos[m.group(2)] = (_ctype(decl, m.group(1), True), argtypes)
    return protos


_LIB = None


def load_library():
    """libmjpc_b200.so with every entry point's argtypes / restype from include/mjpc_b200.h."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(SO):
            raise RuntimeError(f"{SO} not built: run `python -m mujoco_mpc_b200.build` (no fallback path exists)")
        lib = C.CDLL(SO)
        with open(HEADER) as f:
            for name, (restype, argtypes) in parse_header(f.read()).items():
                fn = getattr(lib, name)
                fn.restype, fn.argtypes = restype, argtypes
        _LIB = lib
    return _LIB


def sensor_dim(m, sensor_start, nsensor):
    """Total dimension of the model's sensors [sensor_start, sensor_start + nsensor) (0 for a range outside them: the
    engine refuses it)."""
    if sensor_start < 0 or nsensor < 1 or sensor_start + nsensor > m.nsensor:
        return 0
    return int(np.sum(m.sensor_dim[sensor_start:sensor_start + nsensor]))


class EngineError(RuntimeError):
    pass


def _model_blob(model):
    """The model's blob in a ctypes buffer and the ModelBlob that points at it: keep the buffer while C reads it."""
    blob = to_blob(model)
    buf = C.create_string_buffer(blob, len(blob))
    return buf, ModelBlob(C.cast(buf, C.c_void_p), len(blob))


def _model_blobs(models):
    """The blobs of a list of models as (buffers, ModelBlob array, count); (None, None, 0) for None or an empty list.
    Keep the buffers while C reads them."""
    if not models:
        return None, None, 0
    pairs = [_model_blob(m) for m in models]
    arr = (ModelBlob * len(pairs))(*[mb for _, mb in pairs])
    return [b for b, _ in pairs], arr, len(pairs)


def host_ensemble_score(member_returns, member_failure, worst):
    """The score of one candidate from its K member returns and failure flags on the host
    (mjpc_b200_host_ensemble_score, no device): (score, failure), bitwise what an ensemble launch computes."""
    lib = load_library()
    r = np.ascontiguousarray(member_returns, np.float32)
    f = np.ascontiguousarray(member_failure, np.uint8)
    score, fail = np.zeros(1, np.float32), np.zeros(1, np.uint8)
    lib.mjpc_b200_host_ensemble_score(_pf(r), f.ctypes.data_as(_bp), len(r), int(worst), _pf(score),
                                      fail.ctypes.data_as(_bp))
    return score[0], fail[0]


def host_state_member(model, state, covariance, seed, iteration, problem, member):
    """Member `member` of problem `problem` of a belief launch (Engine.rollout_spline_belief_batched) on the host, in
    fp64 (mjpc_b200_host_state_member, no device): state (+) L z, L the Cholesky factor of (P + P') / 2.  The device's
    member states are this rounded to float."""
    lib = load_library()
    buf, mb = _model_blob(model)
    x, P = _d(state), _d(covariance)
    out = np.zeros(model.nq + model.nv)
    rc = lib.mjpc_b200_host_state_member(C.byref(mb), _pd(x), _pd(P), C.c_uint32(seed), C.c_uint32(iteration),
                                         int(problem), int(member), _pd(out))
    if rc != 0:
        raise EngineError(f"host_state_member failed ({rc}): {lib.mjpc_b200_last_error().decode()}")
    return out


def _ensemble_args(models, worst):
    """(buffers, ModelBlob array, K, worst) of set_ensemble: worst None is K (the expected return)."""
    bufs, arr, n = _model_blobs(models)
    return bufs, arr, n, n if worst is None else int(worst)


def _set_batch_models(obj, models):
    """mjpc_b200_batch_planner_set_models on a batch planner of any kind."""
    bufs, arr, n = _model_blobs(models)
    rc = obj.lib.mjpc_b200_batch_planner_set_models(obj.h, arr, n)
    if rc != 0:
        raise EngineError(f"batch_planner_set_models failed ({rc}): {obj.lib.mjpc_b200_last_error().decode()}")


class _CppObject:
    """A C++ host object created from the model blob by `<prefix>_create` and destroyed by close() through
    `<prefix>_destroy` (the planners and estimators through their family's generic destroy)."""

    def _create(self, prefix, model, *args):
        self.lib = load_library()
        self.m = model
        self._prefix = prefix
        self._buf, mb = _model_blob(model)
        h = C.c_void_p()
        rc = getattr(self.lib, f"{prefix}_create")(C.byref(mb), *args, C.byref(h))
        if rc != 0:
            raise EngineError(f"{prefix}_create failed ({rc}): {self.lib.mjpc_b200_last_error().decode()}")
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            getattr(self.lib, f"{self._prefix}_destroy")(self.h)
            self.h = None

    __del__ = close


class _CppPlanner(_CppObject):
    """A C++ host planner (csrc/host/planner.h): `<prefix>_create` makes it and `<prefix>_get_result` reads result();
    every other call is one of the generic mjpc_b200_planner_* entry points.  The sampling-based planners'
    optimize_policy returns result() and raises on any non-zero code; those with _RETURNS_CODE (Gradient, iLQG, iLQS)
    return the code (1 improved / updated, 0 not) and raise on a negative one."""
    _RETURNS_CODE = False

    def _start(self, model, horizon, device, args):
        """mjpc_b200_<kind>_planner_create(model, *args, horizon, device), args from the kind's _args."""
        self.horizon, self.nu = int(horizon), model.nu
        self._create(f"mjpc_b200_{self._KIND}_planner", model, *args, self.horizon, int(device))

    def result(self):
        return self._result(functools.partial(getattr(self.lib, f"{self._prefix}_get_result"), self.h))

    def close(self):
        if getattr(self, "h", None):
            self.lib.mjpc_b200_planner_destroy(self.h)
            self.h = None

    __del__ = close

    def _fail(self, what):
        raise EngineError(f"{self._prefix}_{what} failed: {self.lib.mjpc_b200_last_error().decode()}")

    def _set_fd(self, tolerance, mode, derivative_skip):
        if self.lib.mjpc_b200_planner_set_fd(self.h, tolerance, mode, derivative_skip):
            self._fail("set_fd")

    def reset(self, initial_repeated_action=None):
        a = _d(initial_repeated_action)
        self.lib.mjpc_b200_planner_reset(self.h, self.horizon, _pd(a))

    def set_state(self, state, time, mocap):
        s, mc = _d(state), _d(mocap)
        self.lib.mjpc_b200_planner_set_state(self.h, _pd(s), time, _pd(mc))

    def optimize_policy(self):
        rc = self.lib.mjpc_b200_planner_optimize_policy(self.h, self.horizon)
        if rc < 0 or (rc and not self._RETURNS_CODE):
            self._fail("optimize_policy")
        return rc if self._RETURNS_CODE else self.result()

    def nominal_trajectory(self):
        """NominalTrajectory: what planning does while it is disabled.  The code is returned (iLQG: 1 / 0 / < 0) or,
        for the sampling-based planners, raises when it is not 0."""
        rc = self.lib.mjpc_b200_planner_nominal_trajectory(self.h, self.horizon)
        if self._RETURNS_CODE:
            return rc
        if rc:
            self._fail("nominal_trajectory")

    def _action(self, time, state, use_previous):
        a, s = np.zeros(self.nu), _d(state)
        self.lib.mjpc_b200_planner_action_from_policy(self.h, _pd(a), _pd(s), time, int(use_previous))
        return a

    def action_from_policy(self, time, use_previous=False):
        return self._action(time, None, use_previous)

    def set_ensemble(self, models, worst=None):
        """Plan on a model ensemble (mjpc_b200_planner_set_ensemble; Engine.set_model_ensemble gives the score):
        Sampling, Cross-Entropy and Sample Gradient.  None or [] clears it."""
        bufs, arr, K, worst = _ensemble_args(models, worst)
        rc = self.lib.mjpc_b200_planner_set_ensemble(self.h, arr, K, worst)
        if rc:
            raise EngineError(f"{self._prefix}_set_ensemble failed ({rc}): {self.lib.mjpc_b200_last_error().decode()}")

    def set_state_ensemble(self, K, worst=None, seed=0):
        """Plan over the state covariance (mjpc_b200_planner_set_state_ensemble): every candidate is scored over K
        initial states drawn from set_state_covariance's covariance, the mean of its `worst` largest member returns
        (None: K).  Sampling, Cross-Entropy and Sample Gradient.  K = 0 clears it."""
        K = int(K)
        rc = self.lib.mjpc_b200_planner_set_state_ensemble(self.h, K, K if worst is None else int(worst), C.c_uint32(seed))
        if rc:
            raise EngineError(f"{self._prefix}_set_state_ensemble failed ({rc})")
        self.state_members = K

    def set_state_covariance(self, covariance):
        """The state covariance [2 nv][2 nv] the state-ensemble launches draw from (None: zero)."""
        P = _d(covariance)
        rc = self.lib.mjpc_b200_planner_set_state_covariance(self.h, _pd(P))
        if rc:
            raise EngineError(f"{self._prefix}_set_state_covariance failed ({rc})")

    def set_task(self, weight=None, parameters=None, task_state=None, risk=None):
        """The task snapshot of every engine handle the planner plans on (mjpc_b200_planner_set_task)."""
        w, p, s = _d(weight), _d(parameters), _d(task_state)
        td = TaskDesc(_pd(w), _pd(p), _pd(s), float(self.m.task_risk if risk is None else risk))
        if self.lib.mjpc_b200_planner_set_task(self.h, C.byref(td)):
            self._fail("set_task")


class _CppFeedbackPlanner(_CppPlanner):
    """iLQG and iLQS: the policy reads the state (time-varying feedback); the code of optimize_policy is returned."""
    _RETURNS_CODE = True

    def action_from_policy(self, time, state=None, use_previous=False):
        return self._action(time, state, use_previous)


def host_ilqg_policy_action(model, u_nom, x_nom, t_nom, gains, representation, feedback_scaling, state, time):
    """iLQGPolicy::Action (ilqg/policy.cc:82-161) on the host through mjpc_b200_host_ilqg_policy_action (no device)."""
    lib = load_library()
    buf, mb = _model_blob(model)
    u, x, t, g = _f(u_nom), _f(x_nom), _d(t_nom), _f(gains)
    st = _d(state)
    out = np.zeros(model.nu)
    rc = lib.mjpc_b200_host_ilqg_policy_action(C.byref(mb), _pf(u), _pf(x), _pd(t), _pf(g), int(u.shape[0]), int(representation),
                                               C.c_double(feedback_scaling), _pd(st), C.c_double(time), _pd(out))
    if rc != 0:
        raise EngineError(f"host_ilqg_policy_action failed ({rc})")
    return out


def host_policy_intervals(nodes, time0, timestep, H):
    """The step table a rollout launch builds per problem (mjpc_b200_host_policy_intervals, no device): the rollout times
    accumulated in double from time0, each step's upper_bound among the absolute node times, and the interval fraction."""
    lib = load_library()
    x = _d(nodes)
    times, upper, frac = np.zeros(H), np.zeros(H, np.int32), np.zeros(H, np.float32)
    lib.mjpc_b200_host_policy_intervals(_pd(x), len(x), C.c_double(time0), C.c_double(timestep), int(H), _pd(times),
                                        upper.ctypes.data_as(C.POINTER(C.c_int)), _pf(frac))
    return times, upper, frac


def _f(a):
    return None if a is None else np.ascontiguousarray(a, np.float32)


def _d(a):
    return None if a is None else np.ascontiguousarray(a, np.float64)


def _pf(a):
    return None if a is None else a.ctypes.data_as(_fp)


def _pd(a):
    return None if a is None else a.ctypes.data_as(_dp)


class Engine:
    """One handle = one GPU's share of the candidates (Planner::Initialize/Allocate analogue)."""

    def __init__(self, model, max_candidates=256, max_horizon=64, device=0):
        self.lib = load_library()
        self.m = model
        self._buf, mb = _model_blob(model)
        h = C.c_void_p()
        rc = self.lib.mjpc_b200_create(C.byref(mb), int(max_candidates), int(max_horizon), int(device), C.byref(h))
        if rc != 0:
            raise EngineError(f"mjpc_b200_create failed ({rc}): {self.lib.mjpc_b200_last_error().decode()}")
        self.h = h
        info = Info()
        self._check(self.lib.mjpc_b200_get_info(self.h, C.byref(info)))
        self.info = info
        self.ds, self.n, self.nu, self.nr = info.dim_state, info.dim_dstate, info.nu, info.num_residual
        self.ntr = 3 * info.num_trace
        self.lastN = self.lastH = 0
        self.members = 0       # K of the model ensemble (set_model_ensemble), 0: none
        self.last_members = 0  # ... of the last launch
        self.lastB = 0

    def close(self):
        if getattr(self, "h", None):
            self.lib.mjpc_b200_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc != 0:
            raise EngineError(f"mjpc_b200 error {rc}: {self.lib.mjpc_b200_last_error().decode()}")

    # ---- task snapshot (Agent::PlanIteration, agent.cc:316-319)
    def set_task(self, weight=None, parameters=None, task_state=None, risk=None):
        w, p, s = _d(weight), _d(parameters), _d(task_state)
        td = TaskDesc(_pd(w), _pd(p), _pd(s), float(self.m.task_risk if risk is None else risk))
        self._check(self.lib.mjpc_b200_set_task(self.h, C.byref(td)))

    def set_model_variants(self, models):
        """Problem b of the following batched launches runs on compiled model models[b] (mjpc_b200_set_model_variants):
        bitwise what an Engine of models[b] computes.  The variants may differ from this engine's model only in its
        physical parameters (include/mjpc_b200.h gives the rule); a launch must then hold len(models) problems, and the
        single-problem, sharded and step calls are refused.  None or [] clears them."""
        bufs, arr, n = _model_blobs(models)
        self._check(self.lib.mjpc_b200_set_model_variants(self.h, arr, n))

    def set_model_ensemble(self, models, worst=None):
        """Score every candidate of the following spline launches on the K = len(models) member models
        (mjpc_b200_set_model_ensemble): the mean of its `worst` largest member returns (None: K, the expected return;
        1: the worst case), 1e6 and failed if any member fails.  Members follow the rule of set_model_variants.  None or
        [] clears the ensemble."""
        bufs, arr, K, worst = _ensemble_args(models, worst)
        self._check(self.lib.mjpc_b200_set_model_ensemble(self.h, arr, K, worst))
        self.members = K

    def set_options(self, timestep, integrator=0):
        """Agent::PlanIteration's planning-model overrides (agent.cc:288-289)."""
        self._check(self.lib.mjpc_b200_set_options(self.h, C.c_double(timestep), int(integrator)))

    def set_differentiable(self, on=True):
        """MakeDifferentiable (utilities.cc:60-75): solimp[0] = 0 for joints and geoms while planning with gradients."""
        self._check(self.lib.mjpc_b200_set_differentiable(self.h, int(bool(on))))

    # ---- SamplingPlanner::Rollouts
    def rollout_spline(self, state, time, mocap, knots, knot_times, interp, H, want_order=True):
        knots = _f(knots)
        N, P, nu = knots.shape
        st, mc, kt = _f(state), _f(mocap), _d(knot_times)
        ret = np.zeros(N, np.float32); fail = np.zeros(N, np.uint8); order = np.zeros(N, np.int32)
        self._check(self.lib.mjpc_b200_rollout_spline(self.h, _pf(st), C.c_double(time), _pf(mc), None, _pf(knots),
                                                      _pd(kt), int(interp), P, N, int(H), _pf(ret),
                                                      fail.ctypes.data_as(_bp), order.ctypes.data_as(_ip)))
        self.lastN, self.lastH, self.lastB, self.last_members = N, H, 1, self.members
        return ret, fail, order

    def rollout_spline_batched(self, states, times, mocaps, knots, knot_times, interp, H, weights=None, parameters=None,
                               task_states=None):
        """B independent problems in one launch (mjpc_b200_rollout_spline_batched): states [B, dim_state], times [B]
        (absolute), mocaps [B, 7 nmocap], knots [B, N, P, nu], knot_times [B, P] (absolute); weights [B, num_term],
        parameters [B, num_parameters], task_states [B, task_state_size] or None for the set_task values.  Returns
        returns [B, N], failure [B, N] and order [B, N] (indices local to each problem); fetch_* then take the flat
        index b * N + i."""
        knots = _f(knots)
        B, N, P, nu = knots.shape
        st, t, mc, kt = _f(states), _d(times), _f(mocaps), _d(knot_times)
        w, p, s = _d(weights), _d(parameters), _d(task_states)
        ret = np.zeros((B, N), np.float32); fail = np.zeros((B, N), np.uint8); order = np.zeros((B, N), np.int32)
        self._check(self.lib.mjpc_b200_rollout_spline_batched(self.h, int(B), _pf(st), _pd(t), _pf(mc), _pd(w), _pd(p), _pd(s),
                                                              _pf(knots), _pd(kt), int(interp), int(P), int(N), int(H),
                                                              _pf(ret), fail.ctypes.data_as(_bp), order.ctypes.data_as(_ip)))
        self.lastN, self.lastH, self.lastB, self.last_members = B * N, H, B, self.members
        return ret, fail, order

    def rollout_spline_belief_batched(self, states, covariances, times, mocaps, knots, knot_times, interp, H, K,
                                      worst=None, seed=0, iteration=0, weights=None, parameters=None, task_states=None):
        """rollout_spline_batched with every candidate scored over K initial states per problem
        (mjpc_b200_rollout_spline_belief_batched): member 0 the state itself, member k states[b] (+) L_b z drawn from
        covariances [B, 2 nv, 2 nv]; the score is the mean of the `worst` largest member returns (None: K).  Returns the
        scores, failure and order [B, N]; fetch_ensemble / fetch_trajectory_member then give the members."""
        knots = _f(knots)
        B, N, P, nu = knots.shape
        K = int(K)
        st, P_, t, mc, kt = _f(states), _d(covariances), _d(times), _f(mocaps), _d(knot_times)
        w, p, s = _d(weights), _d(parameters), _d(task_states)
        ret = np.zeros((B, N), np.float32); fail = np.zeros((B, N), np.uint8); order = np.zeros((B, N), np.int32)
        self._check(self.lib.mjpc_b200_rollout_spline_belief_batched(
            self.h, int(B), K, K if worst is None else int(worst), C.c_uint32(seed), C.c_uint32(iteration), _pf(st),
            _pd(P_), _pd(t), _pf(mc), _pd(w), _pd(p), _pd(s), _pf(knots), _pd(kt), int(interp), int(P), int(N), int(H),
            _pf(ret), fail.ctypes.data_as(_bp), order.ctypes.data_as(_ip)))
        self.lastN, self.lastH, self.lastB, self.last_members = B * N, H, B, K
        return ret, fail, order

    # ---- multi-GPU: one planning problem sharded over an NCCL communicator owned by the handle
    @staticmethod
    def comm_unique_id():
        buf = (C.c_uint8 * 128)()
        lib = load_library()
        rc = lib.mjpc_b200_comm_unique_id(buf, C.c_size_t(128))
        if rc != 0:
            raise EngineError(f"comm_unique_id failed ({rc}): {lib.mjpc_b200_last_error().decode()}")
        return bytes(buf)

    def comm_init(self, nranks, rank, unique_id: bytes):
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self._check(self.lib.mjpc_b200_comm_init(self.h, int(nranks), int(rank), buf, C.c_size_t(128)))
        self.nranks, self.rank = int(nranks), int(rank)

    def comm_init_torch(self, dist):
        """Distribute rank 0's ncclUniqueId over an existing torch.distributed group, then ncclCommInitRank."""
        import torch
        world, rank = dist.get_world_size(), dist.get_rank()
        t = torch.zeros(128, dtype=torch.uint8)
        if rank == 0:
            t = torch.tensor(list(self.comm_unique_id()), dtype=torch.uint8)
        if dist.get_backend() == "nccl":
            t = t.cuda()
        dist.broadcast(t, 0)
        self.comm_init(world, rank, bytes(t.cpu().numpy().tobytes()))

    def rollout_spline_sharded(self, state, time, mocap, knots, knot_times, interp, H):
        knots = _f(knots)
        N, P, nu = knots.shape
        st, mc, kt = _f(state), _f(mocap), _d(knot_times)
        ret = np.zeros(N, np.float32); fail = np.zeros(N, np.uint8); order = np.zeros(N, np.int32)
        self._check(self.lib.mjpc_b200_rollout_spline_sharded(self.h, _pf(st), C.c_double(time), _pf(mc), None, _pf(knots),
                                                              _pd(kt), int(interp), P, N, int(H), _pf(ret),
                                                              fail.ctypes.data_as(_bp), order.ctypes.data_as(_ip)))
        nr, rk = getattr(self, "nranks", 1), getattr(self, "rank", 0)
        self.last_members = 0
        self.lastN, self.lastH = N // nr + (1 if rk < N % nr else 0), H     # fetch_all / fetch_stats are per shard
        return ret, fail, order

    def fetch_trajectory_sharded(self, i):
        return self._fetch(functools.partial(self.lib.mjpc_b200_fetch_trajectory_sharded, self.h, int(i)))

    def upload_spline_inputs(self, state, time, mocap, knots, knot_times, interp, H):
        knots = _f(knots)
        N, P, nu = knots.shape
        st, mc, kt = _f(state), _f(mocap), _d(knot_times)
        self._check(self.lib.mjpc_b200_upload_spline_inputs(self.h, _pf(st), C.c_double(time), _pf(mc), None,
                                                            _pf(knots), _pd(kt), int(interp), P, N, int(H)))
        self.lastN, self.lastH, self.lastB, self.last_members = N, H, 1, self.members

    def launch_resident(self):
        self._check(self.lib.mjpc_b200_launch_resident(self.h))

    def sync(self):
        self._check(self.lib.mjpc_b200_sync(self.h))

    def read_returns(self):
        N = self.lastN
        ret = np.zeros(N, np.float32); fail = np.zeros(N, np.uint8); order = np.zeros(N, np.int32)
        self._check(self.lib.mjpc_b200_read_returns(self.h, _pf(ret), fail.ctypes.data_as(_bp), order.ctypes.data_as(_ip)))
        return ret, fail, order

    # ---- iLQGPlanner::FeedbackRollouts / ActionRollouts
    def rollout_feedback(self, state, time, mocap, u_nom, x_nom, t_nom, gains, du, step_sizes, mode):
        u, x, t, g = _f(u_nom), _f(x_nom), _d(t_nom), _f(gains)
        dd = _f(du)
        ss = _f(step_sizes)
        K, H = len(ss), u.shape[0]
        st, mc = _f(state), _f(mocap)
        ret = np.zeros(K, np.float32); fail = np.zeros(K, np.uint8); order = np.zeros(K, np.int32)
        self._check(self.lib.mjpc_b200_rollout_feedback(self.h, _pf(st), C.c_double(time), _pf(mc), None, _pf(u), _pf(x),
                                                        _pd(t), _pf(g), _pf(dd), _pf(ss), int(mode), K, H, _pf(ret),
                                                        fail.ctypes.data_as(_bp), order.ctypes.data_as(_ip)))
        self.last_members = 0
        self.lastN, self.lastH = K, H
        return ret, fail, order

    def rollout_feedback_batched(self, states, times, mocaps, u_nom, x_nom, t_nom, gains, du, step_sizes, mode,
                                 weights=None, parameters=None, task_states=None):
        """B problems of K feedback rollouts in one launch (mjpc_b200_rollout_feedback_batched): states [B, dim_state],
        times [B] (absolute), mocaps [B, 7 nmocap], u_nom [B, H, nu], x_nom [B, H, dim_state], t_nom [B, H] (absolute),
        gains [B, H, nu, n], du [B, H, nu] or None, step_sizes [B, K]; task arrays [B, ..] or None for the set_task
        values.  Returns returns / failure / order [B, K] (order local to each problem); fetch_* then take b * K + i."""
        u, x, t, g, dd, ss = _f(u_nom), _f(x_nom), _d(t_nom), _f(gains), _f(du), _f(step_sizes)
        B, K = ss.shape
        H = u.shape[1]
        st, tm, mc = _f(states), _d(times), _f(mocaps)
        w, p, s = _d(weights), _d(parameters), _d(task_states)
        ret = np.zeros((B, K), np.float32); fail = np.zeros((B, K), np.uint8); order = np.zeros((B, K), np.int32)
        self._check(self.lib.mjpc_b200_rollout_feedback_batched(self.h, int(B), _pf(st), _pd(tm), _pf(mc), _pd(w), _pd(p), _pd(s),
                                                                _pf(u), _pf(x), _pd(t), _pf(g), _pf(dd), _pf(ss), int(mode),
                                                                int(K), int(H), _pf(ret), fail.ctypes.data_as(_bp),
                                                                order.ctypes.data_as(_ip)))
        self.last_members = 0
        self.lastN, self.lastH = B * K, H
        return ret, fail, order

    def _fetch(self, fetch, *lead):
        """Trajectory-shaped arrays [*lead][lastH][..] filled by fetch(states, actions, times, residual, costs, trace)."""
        s = (*lead, self.lastH)
        o = dict(states=np.zeros((*s, self.ds), np.float32), actions=np.zeros((*s, self.nu), np.float32),
                 times=np.zeros(s), residual=np.zeros((*s, self.nr), np.float32), costs=np.zeros(s, np.float32),
                 trace=np.zeros((*s, self.ntr), np.float32))
        self._check(fetch(_pf(o["states"]), _pf(o["actions"]), _pd(o["times"]), _pf(o["residual"]), _pf(o["costs"]),
                          _pf(o["trace"])))
        return o

    def fetch_trajectory(self, i):
        return self._fetch(functools.partial(self.lib.mjpc_b200_fetch_trajectory, self.h, int(i)))

    def fetch_trajectory_member(self, i, member):
        """Candidate i (flat b * N + i) of the last launch as ensemble member `member` rolled it out."""
        return self._fetch(functools.partial(self.lib.mjpc_b200_fetch_trajectory_member, self.h, int(i), int(member)))

    def fetch_ensemble(self):
        """(member returns [B, K, N], member failure [B, K, N]) of the last launch, an ensemble launch."""
        B, K = max(self.lastB, 1), max(self.last_members, 1)
        shape = (B, K, self.lastN // B)
        ret, fail = np.zeros(shape, np.float32), np.zeros(shape, np.uint8)
        self._check(self.lib.mjpc_b200_fetch_ensemble(self.h, _pf(ret), fail.ctypes.data_as(_bp)))
        return ret, fail

    def fetch_all(self):
        return self._fetch(functools.partial(self.lib.mjpc_b200_fetch_all, self.h), self.lastN)

    def step_debug(self, qpos, qvel, ctrl, mocap, time=0.0, warmstart=None):
        nv, nq = self.info.nv, self.info.nq
        o = dict(qacc=np.zeros(nv, np.float32), residual=np.zeros(max(self.nr, 1), np.float32),
                 next_qpos=np.zeros(nq, np.float32), next_qvel=np.zeros(nv, np.float32),
                 qM=np.zeros((nv, nv), np.float32), efc_force=np.zeros(256, np.float32))
        counts = np.zeros(4, np.int32)
        q, v, u, mc, ws = _f(qpos), _f(qvel), _f(ctrl), _f(mocap), _f(warmstart)
        self._check(self.lib.mjpc_b200_step_debug(self.h, _pf(q), _pf(v), _pf(u), _pf(mc), C.c_double(time), _pf(ws),
                                                  _pf(o["qacc"]), _pf(o["residual"]), _pf(o["next_qpos"]),
                                                  _pf(o["next_qvel"]), _pf(o["qM"]), _pf(o["efc_force"]),
                                                  counts.ctypes.data_as(_ip)))
        o.update(ncon=int(counts[0]), nefc=int(counts[1]), niter=int(counts[2]), warning=int(counts[3]))
        o["efc_force"] = o["efc_force"][: o["nefc"]]
        # geometric contacts [ncon][8] = dist, pos, normal, dim (the oracle's forward_debug()["contact"] layout)
        con, n = np.zeros((64, 8), np.float32), C.c_int()
        self._check(self.lib.mjpc_b200_step_debug_contacts(self.h, 64, _pf(con), C.byref(n)))
        o["contact"] = con[: min(n.value, 64)]
        return o

    def debug_rank(self, returns):
        """The device ranking of returns [nseg, N] (mjpc_b200_debug_rank): order [nseg, N], -1 where no index landed."""
        r = np.ascontiguousarray(np.atleast_2d(returns), np.float32)
        nseg, N = r.shape
        order = np.zeros((nseg, N), np.int32)
        self._check(self.lib.mjpc_b200_debug_rank(self.h, _pf(r), int(nseg), int(N), order.ctypes.data_as(_ip)))
        return order

    def debug_ensemble_score(self, member_returns, member_failure, worst):
        """The device ensemble score of member returns / failure flags [B, K, N] (mjpc_b200_debug_ensemble_score):
        (returns [B, N], failure [B, N])."""
        r = np.ascontiguousarray(member_returns, np.float32)
        f = np.ascontiguousarray(member_failure, np.uint8)
        B, K, N = r.shape
        ret, fail = np.zeros((B, N), np.float32), np.zeros((B, N), np.uint8)
        self._check(self.lib.mjpc_b200_debug_ensemble_score(self.h, _pf(r), f.ctypes.data_as(_bp), int(B), int(K), int(N),
                                                            int(worst), _pf(ret), fail.ctypes.data_as(_bp)))
        return ret, fail

    def step_batch(self, qpos, qvel, ctrl, mocap, times, time0=0.0, warmstart=None):
        """B independent single steps (mjpc_b200_step_batch): teacher-forced per-step parity at planner sizes."""
        q, v, u, mc, ws, t = _f(qpos), _f(qvel), _f(ctrl), _f(mocap), _f(warmstart), _d(times)
        B, nv, nq = q.shape[0], self.info.nv, self.info.nq
        o = dict(qacc=np.zeros((B, nv), np.float32), next_qpos=np.zeros((B, nq), np.float32),
                 next_qvel=np.zeros((B, nv), np.float32), residual=np.zeros((B, max(self.nr, 1)), np.float32),
                 cost=np.zeros(B, np.float32))
        counts = np.zeros((B, 4), np.int32)
        self._check(self.lib.mjpc_b200_step_batch(self.h, B, _pf(q), _pf(v), _pf(u), _pf(ws), _pf(mc), C.c_double(time0),
                                                  _pd(t), _pf(o["qacc"]), _pf(o["next_qpos"]), _pf(o["next_qvel"]),
                                                  _pf(o["residual"]), _pf(o["cost"]), counts.ctypes.data_as(_ip)))
        o.update(ncon=counts[:, 0], nefc=counts[:, 1], niter=counts[:, 2], warning=counts[:, 3])
        return o

    def step_sensors(self, states, ctrl, mocap, time, sensor_start, nsensor, warmstart=None):
        """One step of each of B states from one (ctrl, mocap, time) with the measurement sensors
        [sensor_start, sensor_start + nsensor) of each pre-step state (mjpc_b200_step_sensors): the sigma-point step
        of the Unscented filter (mujoco_mpc_b200.estimator).  Returns dict(next_states [B][nq+nv],
        sensordata [B][dim], qacc [B][nv], ncon, nefc, niter, warning [B])."""
        x, u, mc, ws = _f(np.atleast_2d(states)), _f(ctrl), _f(mocap), _f(warmstart)
        B, nv = x.shape[0], self.info.nv
        dim = sensor_dim(self.m, sensor_start, nsensor)
        o = dict(next_states=np.zeros((B, self.info.dim_state), np.float32), sensordata=np.zeros((B, dim), np.float32),
                 qacc=np.zeros((B, nv), np.float32))
        counts = np.zeros((B, 4), np.int32)
        self._check(self.lib.mjpc_b200_step_sensors(self.h, B, _pf(x), _pf(u), _pf(ws), _pf(mc), C.c_double(time),
                                                    int(sensor_start), int(nsensor), _pf(o["next_states"]),
                                                    _pf(o["sensordata"]), _pf(o["qacc"]), counts.ctypes.data_as(_ip)))
        o.update(ncon=counts[:, 0], nefc=counts[:, 1], niter=counts[:, 2], warning=counts[:, 3])
        return o

    # ---- iLQG sweeps
    def model_derivatives(self, x, u, t, mocap, tol, skip=0, mode=0):
        x, u, t, mc = _f(x), _f(u), _d(t), _f(mocap)
        H = x.shape[0]
        n, nu, nr = self.n, self.nu, self.nr
        A = np.zeros((H, n, n), np.float32); B = np.zeros((H, n, nu), np.float32)
        Cm = np.zeros((H, nr, n), np.float32); D = np.zeros((H, nr, nu), np.float32)
        self._check(self.lib.mjpc_b200_model_derivatives(self.h, _pf(x), _pf(u), _pd(t), _pf(mc), H, int(skip), C.c_float(tol), int(mode),
                                                         _pf(A), _pf(B), _pf(Cm), _pf(D)))
        return A, B, Cm, D

    def cost_derivatives(self, residual, Cm, D):
        r, c, d = _f(residual), _f(Cm), _f(D)
        H = r.shape[0]
        n, nu = self.n, self.nu
        cx = np.zeros((H, n), np.float32); cu = np.zeros((H, nu), np.float32)
        cxx = np.zeros((H, n, n), np.float32); cuu = np.zeros((H, nu, nu), np.float32)
        cxu = np.zeros((H, n, nu), np.float32)
        self._check(self.lib.mjpc_b200_cost_derivatives(self.h, _pf(r), _pf(c), _pf(d), H, _pf(cx), _pf(cu), _pf(cxx),
                                                        _pf(cuu), _pf(cxu)))
        return cx, cu, cxx, cuu, cxu

    def backward_pass(self, A, B, cx, cu, cxx, cxu, cuu, actions, mu=0.0, reg_type=0, limits=1):
        a = [_f(v) for v in (A, B, cx, cu, cxx, cxu, cuu, actions)]
        H, n, nu = a[1].shape
        K = np.zeros((H, nu, n), np.float32); du = np.zeros((H, nu), np.float32); dV = np.zeros(2, np.float32)
        Vx = np.zeros((H, n), np.float32); Vxx = np.zeros((H, n, n), np.float32)
        status = C.c_int(0)
        self._check(self.lib.mjpc_b200_backward_pass(self.h, *[_pf(v) for v in a], H, C.c_float(mu), int(reg_type),
                                                     int(limits), _pf(K), _pf(du), _pf(dV), _pf(Vx), _pf(Vxx),
                                                     C.byref(status)))
        return dict(K=K, du=du, dV=dV, Vx=Vx, Vxx=Vxx, status=status.value)

    def model_derivatives_batched(self, x, u, t, mocaps, tol, skip=0, mode=0, weights=None, parameters=None,
                                  task_states=None):
        """B problems in one sweep (mjpc_b200_model_derivatives_batched): x [B, H, dim_state], u [B, H, nu], t [B, H]
        (absolute), mocaps [B, 7 nmocap]; task arrays [B, ..] or None.  Returns A, B, C, D with a leading [B]."""
        x, u, t, mc = _f(x), _f(u), _d(t), _f(mocaps)
        w, p, s = _d(weights), _d(parameters), _d(task_states)
        Bn, H = x.shape[:2]
        n, nu, nr = self.n, self.nu, self.nr
        A = np.zeros((Bn, H, n, n), np.float32); B = np.zeros((Bn, H, n, nu), np.float32)
        Cm = np.zeros((Bn, H, nr, n), np.float32); D = np.zeros((Bn, H, nr, nu), np.float32)
        self._check(self.lib.mjpc_b200_model_derivatives_batched(self.h, int(Bn), _pf(x), _pf(u), _pd(t), _pf(mc), _pd(w), _pd(p),
                                                                 _pd(s), int(H), int(skip), C.c_float(tol), int(mode),
                                                                 _pf(A), _pf(B), _pf(Cm), _pf(D)))
        return A, B, Cm, D

    def cost_derivatives_batched(self, residual, Cm, D, weights=None):
        """B problems in one launch: residual [B, H, nr], C, D [B, H, ..]; weights [B, num_term] or None."""
        r, c, d, w = _f(residual), _f(Cm), _f(D), _d(weights)
        Bn, H = r.shape[:2]
        n, nu = self.n, self.nu
        cx = np.zeros((Bn, H, n), np.float32); cu = np.zeros((Bn, H, nu), np.float32)
        cxx = np.zeros((Bn, H, n, n), np.float32); cuu = np.zeros((Bn, H, nu, nu), np.float32)
        cxu = np.zeros((Bn, H, n, nu), np.float32)
        self._check(self.lib.mjpc_b200_cost_derivatives_batched(self.h, int(Bn), _pd(w), _pf(r), _pf(c), _pf(d), int(H), _pf(cx),
                                                                _pf(cu), _pf(cxx), _pf(cuu), _pf(cxu)))
        return cx, cu, cxx, cuu, cxu

    def backward_pass_batched(self, A, B, cx, cu, cxx, cxu, cuu, actions, mu, reg_type=0, limits=1):
        """B problems, one CTA each (mjpc_b200_backward_pass_batched): every array [B, H, ..], mu [B].  Returns the
        backward_pass dict with a leading [B] on every entry (status [B])."""
        a = [_f(v) for v in (A, B, cx, cu, cxx, cxu, cuu, actions)]
        Bn, H, n, nu = a[1].shape
        mus = _f(np.broadcast_to(np.asarray(mu, np.float32), (Bn,)))
        K = np.zeros((Bn, H, nu, n), np.float32); du = np.zeros((Bn, H, nu), np.float32); dV = np.zeros((Bn, 2), np.float32)
        Vx = np.zeros((Bn, H, n), np.float32); Vxx = np.zeros((Bn, H, n, n), np.float32)
        status = np.zeros(Bn, np.int32)
        self._check(self.lib.mjpc_b200_backward_pass_batched(self.h, int(Bn), *[_pf(v) for v in a], int(H), _pf(mus),
                                                             int(reg_type), int(limits), _pf(K), _pf(du), _pf(dV), _pf(Vx),
                                                             _pf(Vxx), status.ctypes.data_as(_ip)))
        return dict(K=K, du=du, dV=dV, Vx=Vx, Vxx=Vxx, status=status)

    def gradient_batched(self, x, u, t, mocaps, residual, tol, skip=0, mode=0, weights=None, parameters=None,
                         task_states=None):
        """Gradient::Compute for B problems on the device (mjpc_b200_gradient_batched): the inputs of
        model_derivatives_batched plus residual [B, H, nr].  Returns k [B, H, nu] and dV0 [B] (double)."""
        x, u, t, mc, r = _f(x), _f(u), _d(t), _f(mocaps), _f(residual)
        w, p, s = _d(weights), _d(parameters), _d(task_states)
        Bn, H = x.shape[:2]
        k = np.zeros((Bn, H, self.nu)); dV0 = np.zeros(Bn)
        self._check(self.lib.mjpc_b200_gradient_batched(self.h, int(Bn), _pf(x), _pf(u), _pd(t), _pf(mc), _pd(w), _pd(p),
                                                        _pd(s), _pf(r), int(H), int(skip), C.c_float(tol), int(mode),
                                                        _pd(k), _pd(dV0)))
        return k, dV0

    def fetch_stats(self):
        st = np.zeros((self.lastN * max(self.last_members, 1), 12), np.int64)   # every launched trajectory
        self._check(self.lib.mjpc_b200_fetch_stats(self.h, st.ctypes.data_as(C.POINTER(C.c_int64))))
        return st

    @property
    def launch_count(self):
        return int(self.lib.mjpc_b200_launch_count(self.h))

    def set_xfrc_noise(self, std, rate=1.0, seed=0):
        """NoisyRollout perturbation for the following rollouts (mjpc_b200_set_xfrc_noise); std 0 = off."""
        self._check(self.lib.mjpc_b200_set_xfrc_noise(self.h, C.c_double(std), C.c_double(rate), C.c_uint32(seed)))

    def set_xfrc_noise_batched(self, std, rate, seeds):
        """The same noise with one key per problem (mjpc_b200_set_xfrc_noise_batched): the following launches must
        hold len(seeds) problems, and problem b draws as a launch of it alone after set_xfrc_noise(std, rate, seeds[b])."""
        sd = np.ascontiguousarray(seeds, np.uint32)
        self._check(self.lib.mjpc_b200_set_xfrc_noise_batched(self.h, C.c_double(std), C.c_double(rate), len(sd),
                                                              sd.ctypes.data_as(C.POINTER(C.c_uint32))))

    @property
    def last_kernel_ms(self):
        return float(self.lib.mjpc_b200_last_kernel_ms(self.h))

    @property
    def last_kernel_static(self):
        """True if the last rollout launch ran a statically specialised kernel instance (csrc/spec_*.h)."""
        return bool(self.lib.mjpc_b200_last_kernel_static(self.h))

    @property
    def last_kernel_shape(self):
        """0 generic kernel, 1 static helper-warp instance (shipped), 2 its one-warp twin (MJPC_B200_SHAPE=plain);
        include/mjpc_b200.h."""
        return int(self.lib.mjpc_b200_last_kernel_static(self.h))


PLANT_RUNNING, PLANT_DIVERGED, PLANT_IDLE = 0, 1, 2   # MJPC_B200_PLANT_*


class CppPlantBank:
    """num_plants closed-loop plants whose state stays in device memory (mjpc_b200_plant_*): step() advances every
    running plant by one mj_step in one launch, each on its own model once set_models gave it one.  A plant is idle
    until reset(); a plant whose step would leave a non-finite state becomes PLANT_DIVERGED, keeps its last state and
    is skipped until reset() (MuJoCo would reset it silently).  sensor_start / nsensor (0: none) choose the measurement
    sensors step() returns for each pre-step state.  set_disturbance() and set_xfrc() disturb a plant with the
    reference app's Ornstein-Uhlenbeck control noise, body-force noise and a held wrench."""

    def __init__(self, model, num_plants, sensor_start=None, nsensor=0, device=0):
        self.lib = load_library()
        self.m = model
        self.num_plants = int(num_plants)
        self.nsensor = int(nsensor)
        self.sensor_start = 0 if sensor_start is None else int(sensor_start)
        self.nsensordata = sensor_dim(model, self.sensor_start, self.nsensor) if self.nsensor else 0
        self._buf, mb = _model_blob(model)
        h = C.c_void_p()
        rc = self.lib.mjpc_b200_create(C.byref(mb), self.num_plants, 1, int(device), C.byref(h))
        if rc != 0:
            raise EngineError(f"mjpc_b200_create failed ({rc}): {self.lib.mjpc_b200_last_error().decode()}")
        self.h = h
        self._check(self.lib.mjpc_b200_plant_init(self.h, self.num_plants, self.sensor_start, self.nsensor))
        # each plant's mocap poses as the bank holds them (float), for the planner's set_state
        self.mocap = np.zeros((self.num_plants, 7 * model.nmocap), np.float32)

    def close(self):
        if getattr(self, "h", None):
            self.lib.mjpc_b200_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc != 0:
            raise EngineError(f"mjpc_b200 plant error {rc}: {self.lib.mjpc_b200_last_error().decode()}")

    def reset(self, plant, qpos, qvel, time=0.0, mocap=None):
        """Start an episode: the state and time given, warm start, cost sum and counts 0, running.  mocap None: the
        model's mocap poses."""
        q, v = _f(qpos), _f(qvel)
        mc = _f(self._mocap0() if mocap is None else mocap)
        self._check(self.lib.mjpc_b200_plant_reset(self.h, int(plant), _pf(q), _pf(v), float(time), _pf(mc)))
        if mc is not None:
            self.mocap[plant] = mc

    def _mocap0(self):
        m = self.m
        if not m.nmocap:
            return None
        return np.concatenate([np.asarray(m.mocap_pos0, float).reshape(-1, 3),
                               np.asarray(m.mocap_quat0, float).reshape(-1, 4)], 1).reshape(-1)

    def set(self, plant, qpos=None, qvel=None, mocap=None):
        """What a Task::Transition writes between steps; None keeps the current value."""
        q, v, mc = _f(qpos), _f(qvel), _f(mocap)
        self._check(self.lib.mjpc_b200_plant_set(self.h, int(plant), _pf(q), _pf(v), _pf(mc)))
        if mc is not None:
            self.mocap[plant] = mc

    def set_task(self, plant, weight=None, parameters=None, task_state=None):
        """The plant's task rows for the following steps (task state in absolute time); None keeps the current row."""
        w, p, s = _d(weight), _d(parameters), _d(task_state)
        self._check(self.lib.mjpc_b200_plant_set_task(self.h, int(plant), _pd(w), _pd(p), _pd(s)))

    def set_models(self, models):
        """Plant b steps on compiled model models[b] from now on (len(models) == num_plants; the rule of
        Engine.set_model_variants); None or [] steps every plant on the bank's model again.  The plants are kept."""
        bufs, arr, n = _model_blobs(models)
        self._check(self.lib.mjpc_b200_set_model_variants(self.h, arr, n))

    def set_disturbance(self, plant, ctrl_std=0.0, ctrl_rate=1.0, xfrc_std=0.0, xfrc_rate=1.0, seed=0):
        """Plant `plant`'s OU control noise and body-force noise (std 0: off; rate: the time constant in seconds) and
        the seed of its noise stream; its noise states restart from zero."""
        self._check(self.lib.mjpc_b200_plant_set_disturbance(self.h, int(plant), C.c_double(ctrl_std),
                                                             C.c_double(ctrl_rate), C.c_double(xfrc_std),
                                                             C.c_double(xfrc_rate), C.c_uint32(seed)))

    def set_xfrc(self, plant, xfrc=None):
        """The wrench [nbody][6] (force, torque; world frame, at each body's centre of mass) held on plant `plant` from
        the next step until changed; None clears it."""
        w = None if xfrc is None else np.ascontiguousarray(np.asarray(xfrc, np.float32).reshape(self.m.nbody * 6))
        self._check(self.lib.mjpc_b200_plant_set_xfrc(self.h, int(plant), _pf(w)))

    def set_sensor_noise(self, plant, std=None):
        """Measurement noise of plant `plant`: std [nsensordata] (a scalar is every element's; None clears it).  step()
        then returns sensordata + std z, z white Gaussian noise of the plant's seed (set_disturbance) and step count; the
        plant itself is unaffected."""
        s = None
        if std is not None:
            s = np.ascontiguousarray(np.broadcast_to(np.asarray(std, np.float32), (self.nsensordata,)))
        self._check(self.lib.mjpc_b200_plant_set_sensor_noise(self.h, int(plant), _pf(s)))

    def disturbance(self, plant):
        """dict(ctrl_noise [nu], xfrc_noise [nbody][6]): the plant's OU states after its last committed step."""
        m = self.m
        u, x = np.zeros(m.nu, np.float32), np.zeros((m.nbody, 6), np.float32)
        self._check(self.lib.mjpc_b200_plant_get_disturbance(self.h, int(plant), _pf(u), _pf(x)))
        return dict(ctrl_noise=u, xfrc_noise=x)

    def step(self, ctrl):
        """One step of every running plant from ctrl [num_plants][nu]: dict(state [B][nq+nv], time [B], cost [B] (the
        pre-step residual's cost; 0 where the plant did not step), sensordata [B][dim], status [B], ctrl [B][nu] (the
        ctrl each plant applied: commanded + control noise))."""
        B, m = self.num_plants, self.m
        u = np.ascontiguousarray(np.asarray(ctrl, np.float32).reshape(B, m.nu))
        o = dict(state=np.zeros((B, m.nq + m.nv), np.float32), time=np.zeros(B), cost=np.zeros(B, np.float32),
                 sensordata=np.zeros((B, self.nsensordata), np.float32), status=np.zeros(B, np.int32))
        self._check(self.lib.mjpc_b200_plant_step(self.h, _pf(u), _pf(o["state"]), _pd(o["time"]), _pf(o["cost"]),
                                                  _pf(o["sensordata"]) if self.nsensordata else None,
                                                  o["status"].ctypes.data_as(_ip)))
        o["ctrl"] = np.zeros((B, m.nu), np.float32)
        self._check(self.lib.mjpc_b200_plant_last_ctrl(self.h, _pf(o["ctrl"])))
        return o

    def get(self, plant):
        """dict(state, warmstart, time, cost_sum, steps, warnings, status) of one plant."""
        m = self.m
        x, w = np.zeros(m.nq + m.nv, np.float32), np.zeros(m.nv, np.float32)
        t, cs = C.c_double(), C.c_double()
        st, wn, ss = C.c_int(), C.c_int(), C.c_int()
        self._check(self.lib.mjpc_b200_plant_get(self.h, int(plant), _pf(x), _pf(w), C.byref(t), C.byref(cs),
                                                 C.byref(st), C.byref(wn), C.byref(ss)))
        return dict(state=x, warmstart=w, time=t.value, cost_sum=cs.value, steps=st.value, warnings=wn.value,
                    status=ss.value)

    def last_kernel_ms(self):
        """Device time of the last step's launch (CUDA events)."""
        return float(self.lib.mjpc_b200_last_kernel_ms(self.h))

    def last_kernel_static(self):
        return int(self.lib.mjpc_b200_last_kernel_static(self.h))


def _numeric(model, name, default):
    """The first value of the model's custom numeric `name`, else `default`, as the default's type."""
    return type(default)(model.numeric.get(name, [default])[0])


def _ctrlrange(model):
    """The model's ctrlrange [nu][2] as a create argument (the pointer keeps its array alive through the call)."""
    return _pd(_d(np.asarray(model.actuator_ctrlrange, float).reshape(-1)))


def _seeds(num_problems, seeds):
    """The seeds [num_problems] of a batch planner's create, as _ctrlrange: problem b's is 0x5EED + b unless given."""
    sd = np.ascontiguousarray([0x5EED + b for b in range(int(num_problems))] if seeds is None else seeds, np.uint32)
    return sd.ctypes.data_as(C.POINTER(C.c_uint32))


# ---- The planner kinds, each shared by its single planner and its batch planner.  _args returns the kind's create
# arguments after the model (and the batch's num_problems) and before (max_horizon, device), with `seed` in the seed's
# place: the single planner's seed or the batch's seeds.  _result allocates the kind's get_result outputs, calls
# get_result(*outputs) (bound to the planner, and to the problem of a batch) and decodes them into the result dict.
def _sampling_args(planner, model, num_trajectory, seed):
    """The create arguments of the sampling planner, which those of the Robust and iLQS planners begin with."""
    planner.N, planner.P = int(num_trajectory), _numeric(model, "sampling_spline_points", 3)
    return (planner.N, planner.P, _numeric(model, "sampling_representation", 2),
            _numeric(model, "sampling_exploration", 0.1), float(model.opt_timestep), _ctrlrange(model), seed)


class _Sampling:
    _KIND = "sampling"

    def _args(self, model, num_trajectory, seed):
        return _sampling_args(self, model, num_trajectory, seed)

    def _result(self, get_result):
        winner, imp = C.c_int(), C.c_double()
        ret = np.zeros(self.N, np.float32); knots = np.zeros((self.P, self.nu)); kt = np.zeros(self.P)
        get_result(C.byref(winner), C.byref(imp), _pf(ret), _pd(knots), _pd(kt))
        return dict(winner=winner.value, improvement=imp.value, returns=ret, knots=knots, knot_times=kt)


class _CrossEntropy:
    _KIND = "ce"

    def _args(self, model, num_trajectory, seed, n_elite):
        self.N, self.P = int(num_trajectory), _numeric(model, "sampling_spline_points", 3)
        return (self.N, int(n_elite), self.P, _numeric(model, "sampling_representation", 2),
                _numeric(model, "sampling_exploration", 0.1), _numeric(model, "std_min", 0.01),
                _numeric(model, "explore_fraction", 0.0), float(model.opt_timestep), _ctrlrange(model), seed)

    def _result(self, get_result):
        imp = C.c_double()
        ret = np.zeros(self.N + 1, np.float32); order = np.zeros(self.N, np.int32)
        knots = np.zeros((self.P, self.nu)); kt = np.zeros(self.P); var = np.zeros((self.P, self.nu))
        get_result(C.byref(imp), _pf(ret), order.ctypes.data_as(_ip), _pd(knots), _pd(kt), _pd(var))
        return dict(improvement=imp.value, returns=ret, order=order, knots=knots, knot_times=kt, variance=var)


class _SampleGradient:
    _KIND = "sg"

    def _args(self, model, num_trajectory, seed, num_gradient, gradient_filter):
        self.N, self.P = int(num_trajectory), _numeric(model, "sampling_spline_points", 3)
        G = int(num_gradient if num_gradient is not None else _numeric(model, "sample_gradient_trajectories", 0))
        self.G = max(min(G, self.N - 1), 0)                  # the clamp OptimizePolicy applies
        f = float(gradient_filter if gradient_filter is not None else _numeric(model, "sample_gradient_filter", 1.0))
        return (self.N, G, self.P, _numeric(model, "sampling_representation", 2),
                _numeric(model, "sampling_exploration", 0.1), f, float(model.opt_timestep), _ctrlrange(model), seed)

    def _result(self, get_result):
        winner, wtype, imp = C.c_int(), C.c_int(), C.c_double()
        ret = np.zeros(self.N, np.float32); order = np.zeros(self.N, np.int32)
        knots = np.zeros((self.P, self.nu)); kt = np.zeros(self.P)
        gk = np.zeros((self.G, self.P, self.nu)); grad = np.zeros((self.P, self.nu))
        n = get_result(C.byref(winner), C.byref(wtype), C.byref(imp), _pf(ret), order.ctypes.data_as(_ip), _pd(knots),
                       _pd(kt), _pd(gk) if self.G else None, _pd(grad))
        return dict(winner=winner.value, winner_type=wtype.value, improvement=imp.value, returns=ret, order=order,
                    knots=knots[:n], knot_times=kt[:n], gradient_knots=gk, gradient=grad)


class _Robust:
    _KIND = "robust"

    def _args(self, model, num_trajectory, seed, ncandidates, nrepetitions, xfrc_std, xfrc_rate):
        self.nc = int(ncandidates if ncandidates != -1 else num_trajectory // nrepetitions)
        return _sampling_args(self, model, num_trajectory, seed) + (int(ncandidates), int(nrepetitions), xfrc_std,
                                                                    xfrc_rate)

    def _result(self, get_result):
        winner = C.c_int()
        scores = np.zeros(max(self.nc, 1)); ret = np.zeros(self.N, np.float32)
        knots = np.zeros((self.P, self.nu)); kt = np.zeros(self.P)
        n = get_result(C.byref(winner), _pd(scores), _pf(ret), _pd(knots), _pd(kt))
        return dict(winner=winner.value, scores=scores[:n], returns=ret, knots=knots, knot_times=kt)


class _Gradient:
    _KIND = "gradient"

    def _args(self, model, num_trajectory, num_spline_points, representation, fd_tolerance):
        self.P = int(num_spline_points)
        return (int(num_trajectory), self.P, int(representation), fd_tolerance, float(model.opt_timestep),
                _ctrlrange(model))

    def _result(self, get_result):
        sc = np.zeros(6); p = np.zeros((self.P, self.nu)); t = np.zeros(self.P)
        get_result(_pd(sc), _pd(p), _pd(t))
        return dict(total_return=sc[0], winner=int(sc[1]), action_step=sc[2], expected=sc[3], improvement=sc[4],
                    surprise=sc[5], parameters=p, times=t)


class _ILQG:
    _KIND = "ilqg"

    def _args(self, model, horizon, num_rollouts, representation, fd_tolerance):
        self.H, self.ds = int(horizon), model.nq + model.nv
        return int(num_rollouts), int(representation), fd_tolerance

    def _result(self, get_result):
        sc = np.zeros(6); st = np.zeros((self.H, self.ds), np.float32); ac = np.zeros((self.H, self.nu), np.float32)
        tm = np.zeros(self.H)
        get_result(_pd(sc), _pf(st), _pf(ac), _pd(tm))
        return dict(total_return=sc[0], regularization=sc[1], improvement=sc[2], expected=sc[3], surprise=sc[4],
                    winner=int(sc[5]), states=st, actions=ac, times=tm)


class _ILQS:
    _KIND = "ilqs"

    def _args(self, model, num_trajectory, seed, num_rollouts, fd_tolerance):
        return _sampling_args(self, model, num_trajectory, seed) + (
            int(num_rollouts), _numeric(model, "ilqg_representation", 1), fd_tolerance)

    def _result(self, get_result):
        sc = np.zeros(4)
        get_result(_pd(sc))
        return dict(active_policy=int(sc[0]), sampling_return=sc[1], ilqg_return=sc[2], sampling_winner=int(sc[3]))


class CppSamplingPlanner(_Sampling, _CppPlanner):
    """The C++ host planner (csrc/host/sampling_planner.cc) through its C wrappers."""

    def __init__(self, model, num_trajectory, horizon, seed=0x5EED, device=0):
        self._start(model, horizon, device, self._args(model, num_trajectory, seed))

    def set_exploration(self, exploration, exploration2=0.0):
        self.lib.mjpc_b200_sampling_planner_set_exploration(self.h, C.c_double(exploration), C.c_double(exploration2))


class CppCrossEntropyPlanner(_CrossEntropy, _CppPlanner):
    """The C++ Cross-Entropy planner (csrc/host/cross_entropy_planner.cc) through its C wrappers."""

    def __init__(self, model, num_trajectory, horizon, n_elite=0, seed=0x5EED, device=0):
        self._start(model, horizon, device, self._args(model, num_trajectory, seed, n_elite))


class CppSampleGradientPlanner(_SampleGradient, _CppPlanner):
    """The C++ Sample Gradient planner (csrc/host/sample_gradient_planner.cc) through its C wrappers."""

    def __init__(self, model, num_trajectory, horizon, num_gradient=None, gradient_filter=None, seed=0x5EED, device=0):
        self._start(model, horizon, device, self._args(model, num_trajectory, seed, num_gradient, gradient_filter))


class CppRobustPlanner(_Robust, _CppPlanner):
    """The C++ Robust planner (csrc/host/robust_planner.cc) through its C wrappers."""

    def __init__(self, model, num_trajectory, horizon, ncandidates=-1, nrepetitions=5, xfrc_std=0.1, xfrc_rate=0.1,
                 seed=0x5EED, device=0):
        self._start(model, horizon, device,
                    self._args(model, num_trajectory, seed, ncandidates, nrepetitions, xfrc_std, xfrc_rate))


class CppGradientPlanner(_Gradient, _CppPlanner):
    """The C++ GradientPlanner (csrc/host/gradient_planner.cc) through its C wrappers."""
    _RETURNS_CODE = True

    def __init__(self, model, horizon, num_trajectory=8, num_spline_points=5, representation=1, fd_tolerance=3e-4, device=0, fd_mode=1):
        self._start(model, horizon, device,
                    self._args(model, num_trajectory, num_spline_points, representation, fd_tolerance))
        self._set_fd(fd_tolerance, fd_mode, -1)


class CppILQGPlanner(_ILQG, _CppFeedbackPlanner):
    """The C++ iLQG planner (csrc/host/ilqg_planner.cc) through its C wrappers."""

    def __init__(self, model, horizon, num_rollouts=10, representation=1, fd_tolerance=3e-4, device=0, fd_mode=1, derivative_skip=0):
        self._start(model, horizon, device, self._args(model, horizon, num_rollouts, representation, fd_tolerance))
        self._set_fd(fd_tolerance, fd_mode, derivative_skip)


class CppILQSPlanner(_ILQS, _CppFeedbackPlanner):
    """The C++ iLQSPlanner (csrc/host/gradient_planner.cc) through its C wrappers."""

    def __init__(self, model, horizon, num_trajectory=8, num_rollouts=6, fd_tolerance=3e-4, seed=0x5EED, device=0, fd_mode=1):
        self._start(model, horizon, device, self._args(model, num_trajectory, seed, num_rollouts, fd_tolerance))
        self._set_fd(fd_tolerance, fd_mode, -1)

    def set_exploration(self, sigma):
        self.lib.mjpc_b200_ilqs_planner_set_exploration(self.h, C.c_double(sigma))


class _CppBatchPlanner(_CppObject):
    """A batch of num_problems independent planners of one kind (csrc/host/batch_planner.h): `<prefix>_create` makes it
    and result(problem) reads one problem; every other call is one of the generic mjpc_b200_batch_planner_* entry
    points, and each method that concerns one problem takes its index.  The sampling-based batches' optimize_policy
    returns every problem's result(); those with _RETURNS_CODE (Gradient, iLQG, iLQS) return each problem's code
    (1 improved / updated, 0 not), as their single planners do."""
    _RETURNS_CODE = False

    def _start(self, model, num_problems, horizon, device, args):
        """mjpc_b200_batch_<kind>_planner_create(model, num_problems, *args, horizon, device), args from the kind's
        _args."""
        self.B, self.horizon, self.nu = int(num_problems), int(horizon), model.nu
        self._create(f"mjpc_b200_batch_{self._KIND}_planner", model, self.B, *args, self.horizon, int(device))
        self._codes = np.zeros(self.B, np.int32)   # of the last optimize_policy

    def result(self, problem):
        get_result = getattr(self.lib, f"{self._prefix}_get_result")
        return self._result(lambda *out: self._check(get_result(self.h, int(problem), *out), "get_result"))

    def close(self):
        if getattr(self, "h", None):
            self.lib.mjpc_b200_batch_planner_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc, what):
        if rc < 0:
            raise EngineError(f"batch_planner_{what} failed ({rc}): {self.lib.mjpc_b200_last_error().decode()}")
        return rc

    def reset(self, problem, initial_repeated_action=None):
        a = _d(initial_repeated_action)
        self._check(self.lib.mjpc_b200_batch_planner_reset(self.h, int(problem), self.horizon, _pd(a)), "reset")

    def set_state(self, problem, state, time, mocap):
        s, mc = _d(state), _d(mocap)
        self._check(self.lib.mjpc_b200_batch_planner_set_state(self.h, int(problem), _pd(s), C.c_double(time), _pd(mc)),
                    "set_state")

    def set_task(self, problem, weight=None, parameters=None, task_state=None):
        w, p, s = _d(weight), _d(parameters), _d(task_state)
        self._check(self.lib.mjpc_b200_batch_planner_set_task(self.h, int(problem), _pd(w), _pd(p), _pd(s)), "set_task")

    def set_models(self, models):
        """Problem b plans on compiled model models[b] from now on (len(models) == num_problems), on every engine
        handle the batch owns; None or [] plans every problem on the batch's model again."""
        _set_batch_models(self, models)

    def set_ensemble(self, models, worst=None):
        """Every problem plans on one model ensemble (mjpc_b200_batch_planner_set_ensemble); None or [] clears it."""
        bufs, arr, K, worst = _ensemble_args(models, worst)
        rc = self.lib.mjpc_b200_batch_planner_set_ensemble(self.h, arr, K, worst)
        if rc != 0:
            raise EngineError(f"batch_planner_set_ensemble failed ({rc}): {self.lib.mjpc_b200_last_error().decode()}")

    def set_state_ensemble(self, K, worst=None, seed=0):
        """Every problem plans over its own state covariance with K members (mjpc_b200_batch_planner_set_state_ensemble;
        problem b draws as a single planner with seed + b).  K = 0 clears it."""
        K = int(K)
        rc = self.lib.mjpc_b200_batch_planner_set_state_ensemble(self.h, K, K if worst is None else int(worst),
                                                                 C.c_uint32(seed))
        if rc:
            raise EngineError(f"batch_planner_set_state_ensemble failed ({rc})")
        self.state_members = K

    def set_state_covariance(self, problem, covariance):
        """Problem `problem`'s state covariance [2 nv][2 nv] (None: zero)."""
        P = _d(covariance)
        self._check(self.lib.mjpc_b200_batch_planner_set_state_covariance(self.h, int(problem), _pd(P)),
                    "set_state_covariance")

    def set_fd(self, tolerance, mode=-1, derivative_skip=-1):
        self._check(self.lib.mjpc_b200_batch_planner_set_fd(self.h, C.c_double(tolerance), int(mode), int(derivative_skip)),
                    "set_fd")

    def optimize_policy(self):
        """One planning iteration of every problem; returns the per-problem results or codes."""
        self._check(self.lib.mjpc_b200_batch_planner_optimize_policy(self.h, self.horizon, self._codes.ctypes.data_as(_ip)),
                    "optimize_policy")
        return self._codes.tolist() if self._RETURNS_CODE else [self.result(b) for b in range(self.B)]

    def _action(self, problem, time, state, use_previous):
        a, s = np.zeros(self.nu), _d(state)
        self._check(self.lib.mjpc_b200_batch_planner_action_from_policy(self.h, int(problem), _pd(a), _pd(s),
                                                                        C.c_double(time), int(use_previous)),
                    "action_from_policy")
        return a

    def action_from_policy(self, problem, time, use_previous=False):
        return self._action(problem, time, None, use_previous)


class _CppBatchFeedbackPlanner(_CppBatchPlanner):
    """iLQG and iLQS batches: the policy reads the state (time-varying feedback); optimize_policy returns the codes."""
    _RETURNS_CODE = True
    action_reads_state = True

    def action_from_policy(self, problem, time, state=None, use_previous=False):
        return self._action(problem, time, state, use_previous)


class CppBatchSamplingPlanner(_Sampling, _CppBatchPlanner):
    """num_problems independent Predictive Sampling problems planned with one rollout launch per iteration
    (csrc/host/batch_planner.cc)."""

    def __init__(self, model, num_problems, num_trajectory, horizon, seeds=None, device=0):
        self._start(model, num_problems, horizon, device, self._args(model, num_trajectory, _seeds(num_problems, seeds)))


class CppBatchCrossEntropyPlanner(_CrossEntropy, _CppBatchPlanner):
    """num_problems independent Cross-Entropy problems, one rollout launch of B x (N + 1) per iteration
    (csrc/host/batch_planner.cc).  Mirrors CppCrossEntropyPlanner with a problem argument."""

    def __init__(self, model, num_problems, num_trajectory, horizon, n_elite=0, seeds=None, device=0):
        self._start(model, num_problems, horizon, device,
                    self._args(model, num_trajectory, _seeds(num_problems, seeds), n_elite))


class CppBatchSampleGradientPlanner(_SampleGradient, _CppBatchPlanner):
    """num_problems independent Sample Gradient problems, one rollout launch of B x N per iteration
    (csrc/host/batch_planner.cc).  Mirrors CppSampleGradientPlanner with a problem argument."""

    def __init__(self, model, num_problems, num_trajectory, horizon, num_gradient=None, gradient_filter=None, seeds=None,
                 device=0):
        self._start(model, num_problems, horizon, device,
                    self._args(model, num_trajectory, _seeds(num_problems, seeds), num_gradient, gradient_filter))


class CppBatchRobustPlanner(_Robust, _CppBatchPlanner):
    """num_problems independent Robust problems (csrc/host/batch_planner.cc): per iteration one clean launch of B x N
    and one noisy launch of B x ncandidates x nrepetitions, each problem with its own noise key.  Mirrors
    CppRobustPlanner with a problem argument."""

    def __init__(self, model, num_problems, num_trajectory, horizon, ncandidates=-1, nrepetitions=5, xfrc_std=0.1,
                 xfrc_rate=0.1, seeds=None, device=0):
        self._start(model, num_problems, horizon, device,
                    self._args(model, num_trajectory, _seeds(num_problems, seeds), ncandidates, nrepetitions, xfrc_std,
                               xfrc_rate))


class CppBatchGradientPlanner(_Gradient, _CppBatchPlanner):
    """num_problems independent Gradient problems (csrc/host/batch_planner.cc): per iteration one launch of the B
    nominals, one mjpc_b200_gradient_batched and one launch of the B x num_trajectory line-search candidates.  Mirrors
    CppGradientPlanner with a problem argument; optimize_policy returns each problem's 1/0."""
    _RETURNS_CODE = True

    def __init__(self, model, num_problems, horizon, num_trajectory=8, num_spline_points=5, representation=1,
                 fd_tolerance=3e-4, device=0, fd_mode=1):
        self._start(model, num_problems, horizon, device,
                    self._args(model, num_trajectory, num_spline_points, representation, fd_tolerance))
        self.set_fd(fd_tolerance, fd_mode, -1)

    def result(self, problem):
        return dict(super().result(problem), improved=int(self._codes[problem]))


class CppBatchILQGPlanner(_ILQG, _CppBatchFeedbackPlanner):
    """The batched C++ iLQG planner (csrc/host/batch_planner.cc): B problems, one launch per sweep.  Mirrors
    CppILQGPlanner with a problem argument."""

    def __init__(self, model, num_problems, horizon, num_rollouts=10, representation=1, fd_tolerance=3e-4, device=0,
                 fd_mode=1, derivative_skip=0):
        self._start(model, num_problems, horizon, device,
                    self._args(model, horizon, num_rollouts, representation, fd_tolerance))
        self.set_fd(fd_tolerance, fd_mode, derivative_skip)

    def nominal_trajectory(self):
        return self._check(self.lib.mjpc_b200_batch_ilqg_planner_nominal_trajectory(self.h, self.H), "nominal_trajectory")

    def optimize_policy(self):
        """Every problem's iLQGPlanner::OptimizePolicy; returns updated [B] (1: the policy was updated)."""
        return np.array(super().optimize_policy(), np.int32)


class CppBatchILQSPlanner(_ILQS, _CppBatchFeedbackPlanner):
    """num_problems independent iLQS problems (csrc/host/batch_planner.cc) on two handles: per iteration one feedback
    launch of the iLQG nominals that need converting, one sampling launch of B x num_trajectory, and one batched iLQG
    iteration of the problems sampling did not settle.  Mirrors CppILQSPlanner with a problem argument;
    optimize_policy returns each problem's 1/0."""

    def __init__(self, model, num_problems, horizon, num_trajectory=8, num_rollouts=6, fd_tolerance=3e-4, seeds=None,
                 device=0, fd_mode=1):
        self._start(model, num_problems, horizon, device,
                    self._args(model, num_trajectory, _seeds(num_problems, seeds), num_rollouts, fd_tolerance))
        self.set_fd(fd_tolerance, fd_mode, -1)

    def set_exploration(self, sigma):
        self._check(self.lib.mjpc_b200_batch_ilqs_planner_set_exploration(self.h, C.c_double(sigma)), "set_exploration")

    def result(self, problem):
        return dict(super().result(problem), improved=int(self._codes[problem]))


def host_spline_mapping(representation, input_times, output_times):
    """SplineMapping::Compute (gradient/spline_mapping.cc) as scalar weights W [num_output][num_input]."""
    lib = load_library()
    ti, to = _d(input_times), _d(output_times)
    W = np.zeros((len(to), len(ti)))
    lib.mjpc_b200_host_spline_mapping(int(representation), _pd(ti), len(ti), _pd(to), len(to), _pd(W))
    return W


def host_gradient_sweep(A, B, cx, cu):
    """Gradient::Compute's recursion on the host in fp64 (mjpc_b200_host_gradient_sweep, no device): A [T, n, n],
    B [T, n, m], cx [T, n], cu [T, m] (float32) -> k [T, m], dV0."""
    lib = load_library()
    a, b, x, u = _f(A), _f(B), _f(cx), _f(cu)
    T, n, m = b.shape
    k, dV0 = np.zeros((T, m)), C.c_double()
    lib.mjpc_b200_host_gradient_sweep(_pf(a), _pf(b), _pf(x), _pf(u), int(n), int(m), int(T), _pd(k), C.byref(dV0))
    return k, dV0.value


class CppAgent(_CppObject):
    """Agent::PlanIteration glue (csrc/host/agent.cc) through its C wrappers; settings mirror the task XML numerics."""
    PLANNERS = {"sampling": 0, "gradient": 1, "ilqg": 2, "ilqs": 3, "robust": 4, "cross_entropy": 5, "sample_gradient": 6}

    def __init__(self, model, planner="sampling", horizon=None, timestep=None, integrator=0, differentiable=-1, num_trajectory=None,
                 num_spline_points=None, representation=None, exploration=None, ilqg_num_rollouts=10, ilqg_representation=1,
                 fd_tolerance=3e-4, seed=0x5EED, device=0, num_gradient=None, gradient_filter=None):
        m, num = model, model.numeric
        g = lambda k, d: float(num.get(k, [d])[0])
        st = np.array([self.PLANNERS[planner] if isinstance(planner, str) else planner,
                       g("agent_horizon", 0.5) if horizon is None else horizon,
                       g("agent_timestep", 0.01) if timestep is None else timestep, integrator, differentiable,
                       g("sampling_trajectories", 10) if num_trajectory is None else num_trajectory,
                       g("sampling_spline_points", 3) if num_spline_points is None else num_spline_points,
                       g("sampling_representation", 2) if representation is None else representation,
                       g("sampling_exploration", 0.1) if exploration is None else exploration,
                       ilqg_num_rollouts, ilqg_representation, fd_tolerance, 0, g("std_min", 0.01), g("explore_fraction", 0.0),
                       g("robust_candidates", -1), g("robust_repetitions", 5), g("robust_xfrc", 0.1), g("robust_xfrc_rate", 0.1),
                       seed,
                       g("sample_gradient_trajectories", 0) if num_gradient is None else num_gradient,
                       g("sample_gradient_filter", 1.0) if gradient_filter is None else gradient_filter], float)
        cr = _d(np.asarray(m.actuator_ctrlrange, float).reshape(-1))
        self._create("mjpc_b200_agent", m, _pd(st), _pd(cr), int(device))
        self.nu = m.nu

    @property
    def steps(self):
        return int(self.lib.mjpc_b200_agent_get_steps(self.h))

    def reset(self, initial_repeated_action=None):
        a = _d(initial_repeated_action)
        self.lib.mjpc_b200_agent_reset(self.h, _pd(a))

    def set_state(self, state, time, mocap):
        s, mc = _d(state), _d(mocap)
        self.lib.mjpc_b200_agent_set_state(self.h, _pd(s), C.c_double(time), _pd(mc))

    def set_task(self, weight=None, parameters=None, task_state=None, risk=None):
        w, p, s = _d(weight), _d(parameters), _d(task_state)
        td = TaskDesc(_pd(w), _pd(p), _pd(s), float(self.m.task_risk if risk is None else risk))
        self.lib.mjpc_b200_agent_set_task(self.h, C.byref(td))

    def set_plan_enabled(self, on):
        self.lib.mjpc_b200_agent_set_plan_enabled(self.h, int(bool(on)))

    def plan_iteration(self):
        rc = self.lib.mjpc_b200_agent_plan_iteration(self.h)
        if rc < 0:
            raise EngineError(f"agent_plan_iteration failed ({rc}): {self.lib.mjpc_b200_last_error().decode()}")
        return rc

    def action_from_policy(self, time, state=None, use_previous=False):
        a = np.zeros(self.nu); st = _d(state)
        self.lib.mjpc_b200_agent_action_from_policy(self.h, _pd(a), _pd(st), C.c_double(time), int(use_previous))
        return a
