"""Small numpy rigid-body routines used only by the offline model compiler.

They compute the configuration-independent constants MuJoCo's ``mj_setConst``
would store in ``mjModel`` (dof_invweight0, body_invweight0, stat.meaninertia)
from the joint-space inertia at ``qpos0``.  The formulation here (world-frame
Jacobians, M = sum_b J_b^T I_b J_b) is deliberately different from the
composite-rigid-body recursion in ``oracle/`` and in the CUDA kernels, so the
tests can cross-check the two.
"""
from __future__ import annotations

import numpy as np

from .mjcf import JNT_BALL, JNT_FREE, JNT_HINGE, JNT_SLIDE, axisangle2quat, quat2mat, quat_mul


def kinematics(m, qpos, mocap_pos=None, mocap_quat=None):
    nb = m.nbody
    xpos = np.zeros((nb, 3)); xquat = np.zeros((nb, 4)); xquat[0, 0] = 1
    xanchor = np.zeros((m.njnt, 3)); xaxis = np.zeros((m.njnt, 3))
    for b in range(1, nb):
        p = m.body_parentid[b]
        if m.body_mocapid[b] >= 0:
            k = m.body_mocapid[b]
            pos = (m.mocap_pos0 if mocap_pos is None else mocap_pos)[k].copy()
            quat = (m.mocap_quat0 if mocap_quat is None else mocap_quat)[k].copy()
        else:
            pos = xpos[p] + quat2mat(xquat[p]) @ m.body_pos[b]
            quat = quat_mul(xquat[p], m.body_quat[b])
        for j in range(m.body_jntadr[b], m.body_jntadr[b] + m.body_jntnum[b]):
            qa = m.jnt_qposadr[j]
            t = m.jnt_type[j]
            if t == JNT_FREE:
                pos = qpos[qa:qa + 3].copy(); quat = qpos[qa + 3:qa + 7] / np.linalg.norm(qpos[qa + 3:qa + 7])
                xanchor[j] = pos; xaxis[j] = [0, 0, 1]
                continue
            R = quat2mat(quat)
            xanchor[j] = pos + R @ m.jnt_pos[j]
            xaxis[j] = R @ m.jnt_axis[j]
            if t == JNT_SLIDE:
                pos = pos + xaxis[j] * (qpos[qa] - m.qpos0[qa])
            elif t == JNT_HINGE:
                quat = quat_mul(quat, axisangle2quat(m.jnt_axis[j], qpos[qa] - m.qpos0[qa]))
                pos = xanchor[j] - quat2mat(quat) @ m.jnt_pos[j]
            elif t == JNT_BALL:
                quat = quat_mul(quat, qpos[qa:qa + 4] / np.linalg.norm(qpos[qa:qa + 4]))
                pos = xanchor[j] - quat2mat(quat) @ m.jnt_pos[j]
        xpos[b] = pos; xquat[b] = quat / np.linalg.norm(quat)
    xmat = np.array([quat2mat(q) for q in xquat])
    xipos = np.array([xpos[b] + xmat[b] @ m.body_ipos[b] for b in range(nb)])
    ximat = np.array([quat2mat(quat_mul(xquat[b], m.body_iquat[b])) for b in range(nb)])
    return dict(xpos=xpos, xquat=xquat, xmat=xmat, xipos=xipos, ximat=ximat, xanchor=xanchor, xaxis=xaxis)


def body_jacobian(m, kin, b, point):
    """6 x nv Jacobian (rows 0-2 translational at ``point``, 3-5 rotational) of body b."""
    J = np.zeros((6, m.nv))
    bb = b
    while bb > 0:
        for j in range(m.body_jntadr[bb], m.body_jntadr[bb] + m.body_jntnum[bb]):
            d = m.jnt_dofadr[j]
            t = m.jnt_type[j]
            if t == JNT_FREE:
                J[0:3, d:d + 3] = np.eye(3)
                R = kin["xmat"][bb]
                for k in range(3):
                    J[3:6, d + 3 + k] = R[:, k]
                    J[0:3, d + 3 + k] = np.cross(R[:, k], point - kin["xpos"][bb])
            elif t == JNT_BALL:
                R = kin["xmat"][bb]
                for k in range(3):
                    J[3:6, d + k] = R[:, k]
                    J[0:3, d + k] = np.cross(R[:, k], point - kin["xanchor"][j])
            elif t == JNT_SLIDE:
                J[0:3, d] = kin["xaxis"][j]
            else:
                J[3:6, d] = kin["xaxis"][j]
                J[0:3, d] = np.cross(kin["xaxis"][j], point - kin["xanchor"][j])
        bb = m.body_parentid[bb]
    return J


def mass_matrix_and_jacobians(m, qpos, mocap_pos=None, mocap_quat=None):
    kin = kinematics(m, qpos, mocap_pos, mocap_quat)
    M = np.diag(m.dof_armature.astype(float)) if m.nv else np.zeros((0, 0))
    Jb = {}
    for b in range(1, m.nbody):
        J = body_jacobian(m, kin, b, kin["xipos"][b])
        Jb[b] = J
        Iw = kin["ximat"][b] @ np.diag(m.body_inertia[b]) @ kin["ximat"][b].T
        M = M + m.body_mass[b] * J[0:3].T @ J[0:3] + J[3:6].T @ Iw @ J[3:6]
    return M, Jb
