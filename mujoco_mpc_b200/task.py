"""Host-side task helpers: norm table, residual registry, per-task state blocks.

Mirrors mjpc/norm.h:27-37 (NormType numbering), mjpc/norm.cc:27-50
(NormParameterDimension) and the name -> residual id registry that replaces
``GetTasks()`` (mjpc/tasks/tasks.cc:46-73) on the device side.
"""
from __future__ import annotations

import math

import numpy as np

# NormType (mjpc/norm.h:27-37)
NORM_NULL, NORM_QUADRATIC, NORM_L22, NORM_L2, NORM_COSH = -1, 0, 1, 2, 3
NORM_POWER_LOSS, NORM_SMOOTH_ABS, NORM_SMOOTH_ABS2, NORM_RECTIFY = 5, 6, 7, 8

# residual registry (device function selected by id)
RESIDUAL_PARTICLE = 0        # mjpc/test/testdata/particle_residual.h:22-52
RESIDUAL_PARTICLE_COPY = 1   # mjpc/test/agent/rollout_test.cc:25-50
RESIDUAL_CARTPOLE = 2        # mjpc/tasks/cartpole/cartpole.cc:36-49
RESIDUAL_QUADRUPED_FLAT = 3  # mjpc/tasks/quadruped/quadruped.cc:33-226
RESIDUAL_HUMANOID_STAND = 4  # mjpc/tasks/humanoid/stand/stand.cc:30-97
# task_ids layout of the humanoid stand residual
HI_TORSO_BODY, HI_HEAD_BODY, HI_SITE_SP0, HI_SIZE = 0, 1, 2, 6
RESIDUAL_HUMANOID_TRACK = 5  # mjpc/tasks/humanoid/tracking/tracking.cc:94-216
# tracking: task_ids = 16 tracking-site ids then the 16 mocap ids, both in tracking.cc:71-75 body order;
# task_state = [current_mode, reference_time] (reference_time is time-like: rebased per rollout)
TRACK_BODIES = ("pelvis", "head", "ltoe", "rtoe", "lheel", "rheel", "lknee", "rknee", "lhand", "rhand", "lelbow",
                "relbow", "lshoulder", "rshoulder", "lhip", "rhip")
RESIDUAL_SHADOW_REORIENT = 6 # mjpc/tasks/shadow_reorient/hand.cc:37-84
SI_GRASP_SITE, SI_CUBE_BODY, SI_GOAL_BODY, SI_KEY_GRASP, SI_SIZE = 0, 1, 2, 3, 4
TRACK_MOTION_LENGTHS = (121, 154, 115, 78, 145, 188, 260, 279, 39, 510)   # tracking.cc:43-54
TRACK_FPS = 30.0
TS_MODE, TS_REFERENCE_TIME, TS_SIZE = 0, 1, 2
RESIDUAL_NONE = 7            # a model without cost terms (the reference's estimator test models): no residual is evaluated

# quadruped task-state block layout (doubles); ResidualFn members, quadruped.h:160-225
QS_MODE, QS_MODE_START_TIME, QS_POSITION, QS_HEADING, QS_SPEED, QS_ANGVEL, QS_GROUND = 0, 1, 2, 5, 7, 8, 9
QS_ORIENTATION, QS_GAIT, QS_PHASE_START, QS_PHASE_START_TIME, QS_PHASE_VELOCITY = 10, 14, 15, 16, 17
QS_JUMP_VEL, QS_FLIGHT_TIME, QS_JUMP_ACC, QS_CROUCH_TIME, QS_LEAP_TIME, QS_JUMP_TIME = 18, 19, 20, 21, 22, 23
QS_CROUCH_VEL, QS_LAND_TIME, QS_LAND_ACC, QS_FLIGHT_ROT_VEL, QS_JUMP_ROT_VEL = 24, 25, 26, 27, 28
QS_JUMP_ROT_ACC, QS_LAND_ROT_ACC, QS_SIZE = 29, 30, 31
# quadruped task_ids layout (ints)
QI_TORSO_BODY, QI_HEAD_SITE, QI_GOAL_MOCAP, QI_FOOT_GEOM, QI_PARAM_GAIT, QI_PARAM_BIPED_TYPE = 0, 1, 2, 3, 7, 8
QI_PARAM_CADENCE, QI_PARAM_AMPLITUDE, QI_PARAM_DUTY, QI_PARAM_ARM_POSTURE, QI_PARAM_HEADING = 9, 10, 11, 12, 13
QI_PARAM_FLIP_DIR, QI_KEY_HOME, QI_KEY_CROUCH, QI_SIZE = 14, 15, 16, 17


def norm_parameter_dimension(t: int) -> int:
    return {NORM_NULL: 0, NORM_QUADRATIC: 0, NORM_L22: 2, NORM_L2: 1, NORM_COSH: 1, NORM_POWER_LOSS: 1,
            NORM_SMOOTH_ABS: 1, NORM_SMOOTH_ABS2: 2, NORM_RECTIFY: 1}.get(int(t), 0)


def quadruped_state_block(gravity_norm=9.81, cadence=2.0):
    """Initial task-state block: QuadrupedFlat::ResetLocked (quadruped.cc:540-606) + member defaults."""
    k_height_quadruped, k_crouch, k_leap, k_max = 0.25, 0.15, 0.5, 0.8
    s = np.zeros(QS_SIZE)
    g = gravity_norm
    jump_vel = math.sqrt(2 * g * (k_max - k_leap))
    flight_time = 2 * jump_vel / g
    jump_acc = jump_vel * jump_vel / (2 * (k_leap - k_crouch))
    crouch_time = math.sqrt(2 * (k_height_quadruped - k_crouch) / jump_acc)
    leap_time = jump_vel / jump_acc
    jump_time = crouch_time + leap_time
    crouch_vel = -jump_acc * crouch_time
    land_time = 2 * (k_leap - k_height_quadruped) / jump_vel
    land_acc = jump_vel / land_time
    flight_rot_vel = 1.25 * math.pi / flight_time
    jump_rot_vel = math.pi / leap_time - flight_rot_vel
    jump_rot_acc = (flight_rot_vel - jump_rot_vel) / leap_time
    land_rot_acc = 2 * (flight_rot_vel * land_time - math.pi / 4) / (land_time * land_time)
    s[QS_JUMP_VEL], s[QS_FLIGHT_TIME], s[QS_JUMP_ACC], s[QS_CROUCH_TIME] = jump_vel, flight_time, jump_acc, crouch_time
    s[QS_LEAP_TIME], s[QS_JUMP_TIME], s[QS_CROUCH_VEL], s[QS_LAND_TIME] = leap_time, jump_time, crouch_vel, land_time
    s[QS_LAND_ACC], s[QS_FLIGHT_ROT_VEL], s[QS_JUMP_ROT_VEL] = land_acc, flight_rot_vel, jump_rot_vel
    s[QS_JUMP_ROT_ACC], s[QS_LAND_ROT_ACC] = jump_rot_acc, land_rot_acc
    # phase velocity is set by the first Transition: 2*pi*cadence (quadruped.cc:256-262)
    s[QS_PHASE_VELOCITY] = 2 * math.pi * cadence
    return s
