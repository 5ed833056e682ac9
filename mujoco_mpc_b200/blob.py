"""Binary model blob shared by the CPU oracle and the CUDA engine.

Layout (little endian):
    char[8]  magic  "MJPCB200"
    int32    version (=1), int32 n_entries
    n_entries x { char[40] name, int32 dtype (0=int32, 1=float64), int32 count, int64 byte offset }
    payload, every array 8-byte aligned

The names are ``mjModel`` field names (plus ``opt_*``, ``task_*``, ``pair_*``),
so a maintainer with MuJoCo can emit the same blob from an ``mjModel*``
(INTEGRATION.md shows the C++ for it).  ``include/mjpc_b200.h`` declares the
C view (``mjpc_model_blob``).
"""
from __future__ import annotations

import struct

import numpy as np

MAGIC = b"MJPCB200"
VERSION = 1

_INT_SCALARS = ["nq", "nv", "nu", "na", "nbody", "njnt", "ngeom", "nsite", "nmocap", "nkey", "nuserdata",
                "nsensordata", "npair", "ntendon", "opt_cone", "opt_iterations", "opt_ls_iterations", "opt_integrator",
                "opt_disable_contact", "opt_disable_eulerdamp", "opt_disable_frictionloss", "opt_disable_limit",
                "opt_disable_refsafe", "opt_disable_warmstart", "task_num_term", "task_num_residual",
                "task_num_trace", "task_residual_id", "nsensor"]
_F_SCALARS = ["opt_timestep", "opt_impratio", "opt_tolerance", "opt_ls_tolerance", "stat_meaninertia", "task_risk"]
_INT_ARRAYS = ["body_parentid", "body_rootid", "body_weldid", "body_jntnum", "body_jntadr", "body_dofnum",
               "body_dofadr", "body_mocapid", "body_depth", "jnt_type", "jnt_qposadr", "jnt_dofadr", "jnt_bodyid",
               "jnt_limited", "dof_bodyid", "dof_jntid", "dof_parentid", "geom_type", "geom_bodyid",
               "geom_condim", "geom_priority", "geom_group", "site_bodyid", "actuator_trnid", "actuator_trntype",
               "actuator_biastype", "actuator_ctrllimited", "actuator_forcelimited", "pair_geom1", "pair_geom2",
               "task_dim_norm_residual", "task_norm", "task_num_norm_parameter", "task_trace_objtype",
               "task_trace_objid", "task_ids", "ray_geoms", "tendon_adr", "tendon_num", "tendon_limited", "wrap_dof",
               "wrap_qposadr", "sensor_type", "sensor_objtype", "sensor_objid", "sensor_dim", "sensor_adr", "site_type"]
_F_ARRAYS = ["opt_gravity", "body_pos", "body_quat", "body_ipos", "body_iquat", "body_mass", "body_inertia",
             "body_subtreemass", "body_invweight0", "jnt_pos", "jnt_axis", "jnt_range", "jnt_stiffness",
             "jnt_margin", "jnt_solref", "jnt_solimp", "qpos0", "qpos_spring", "dof_damping", "dof_armature",
             "dof_frictionloss", "dof_solref", "dof_solimp", "dof_invweight0", "geom_size", "geom_pos",
             "geom_quat", "geom_friction", "geom_solmix", "geom_solref", "geom_solimp", "geom_margin", "geom_gap",
             "geom_rbound", "site_pos", "site_quat", "actuator_gear", "actuator_gainprm", "actuator_biasprm",
             "actuator_ctrlrange", "actuator_forcerange", "key_qpos", "key_qvel", "key_ctrl", "key_mpos",
             "key_mquat", "task_weight", "task_norm_parameter", "task_parameters", "task_state", "wrap_coef",
             "tendon_range", "tendon_margin", "tendon_solref", "tendon_solimp", "tendon_invweight0", "site_size", "sensor_cutoff"]


# written only for a model with a magnetometer or a rangefinder, so that every other model's blob stays as it was:
# opt.magnetic, and the alpha mj_ray reads per geom (its material's when it has one, else its rgba's)
_F_RAY_FIELD = ["opt_magnetic", "geom_alpha"]


def to_blob(model) -> bytes:
    from .mjcf import SENS_RAY_FIELD
    entries = []
    for k in _INT_SCALARS:
        entries.append((k, 0, np.array([int(model.get(k, 0))], np.int32)))
    for k in _F_SCALARS:
        entries.append((k, 1, np.array([float(model.get(k, 0.0))], np.float64)))
    for k in _INT_ARRAYS:
        entries.append((k, 0, np.ascontiguousarray(np.asarray(model.get(k, np.zeros(0)), np.int32).reshape(-1))))
    for k in _F_ARRAYS:
        entries.append((k, 1, np.ascontiguousarray(np.asarray(model.get(k, np.zeros(0)), np.float64).reshape(-1))))
    if np.isin(np.asarray(model.get("sensor_type", np.zeros(0))), SENS_RAY_FIELD).any():
        for k in _F_RAY_FIELD:
            entries.append((k, 1, np.ascontiguousarray(np.asarray(model[k], np.float64).reshape(-1))))
    header_size = 16 + len(entries) * 56
    payload = bytearray()
    table = bytearray()
    off = header_size
    for name, dt, arr in entries:
        raw = arr.tobytes()
        pad = (-len(raw)) % 8
        table += struct.pack("<40siiq", name.encode(), dt, arr.size, off)
        payload += raw + b"\0" * pad
        off += len(raw) + pad
    return MAGIC + struct.pack("<ii", VERSION, len(entries)) + bytes(table) + bytes(payload)


def from_blob(buf: bytes) -> dict:
    assert buf[:8] == MAGIC
    ver, n = struct.unpack_from("<ii", buf, 8)
    out = {}
    for i in range(n):
        name, dt, cnt, off = struct.unpack_from("<40siiq", buf, 16 + 56 * i)
        name = name.rstrip(b"\0").decode()
        out[name] = np.frombuffer(buf, np.int32 if dt == 0 else np.float64, cnt, off).copy()
    return out
