"""Model/task definitions for the BASELINE configs, generated as MJCF text.

The reference builds its robot XMLs at configure time by patching Menagerie /
dm_control files that are NOT vendored (SURVEY.md section 0, finding 2), so the
models are restated here programmatically from the numbers that *are* in the
reference tree (the ``.patch`` hunks and the task XMLs); every number that had
to be filled in from outside the tree is marked ``[GUESS]``.

  particle  : mjpc/test/testdata/particle.xml:30-63, particle_task.xml:6-33 (fully in tree)
  cartpole  : mjpc/tasks/cartpole/cartpole.xml.patch:4-31, task.xml:8-47 (pole default class and
              actuator are outside the patch context -> [GUESS] = dm_control suite values)
  quadruped : mjpc/tasks/quadruped/a1.xml.patch:4-205, task_flat.xml:6-161 (collision default
              classes hip/thigh/calf and 4 trunk collision geoms are outside the patch context
              -> [GUESS] = Menagerie unitree_a1 values)
"""
from __future__ import annotations

import numpy as np

from .. import task as T
from ..mjcf import GEOM_PLANE, compile_xml


# ----------------------------------------------------------------------------- particle
def particle_xml(copy_task=False) -> str:
    return """
<mujoco model="Particle Control">
  <option timestep="0.01"><flag contact="disable"/></option>
  <default>
    <joint type="hinge" axis="0 0 1" limited="true" range="-.29 .29" damping="1"/>
    <motor gear=".1" ctrlrange="-1 1" ctrllimited="true"/>
  </default>
  <custom>
    <numeric name="task_risk" data="1.0"/>
    <numeric name="agent_planner" data="0"/>
    <numeric name="agent_horizon" data="1"/>
    <numeric name="agent_timestep" data="0.1"/>
    <numeric name="sampling_spline_points" data="11"/>
    <numeric name="sampling_exploration" data="0.01"/>
    <numeric name="residual_dummy1" data="0.05"/>
    <numeric name="residual_dummy2" data="-0.1"/>
  </custom>
  <worldbody>
    <body name="goal" mocap="true" pos="0.25 0 0.01" quat="1 0 0 0">
      <geom type="sphere" size=".01" contype="0" conaffinity="0"/>
    </body>
    <geom name="ground" type="plane" pos="0 0 0" size=".3 .3 .1"/>
    <body name="pointmass" pos="0 0 .01">
      <joint name="root_x" type="slide" pos="0 0 0" axis="1 0 0"/>
      <joint name="root_y" type="slide" pos="0 0 0" axis="0 1 0"/>
      <geom name="pointmass" type="sphere" size=".01" mass=".3"/>
      <site name="tip" pos="0 0 0" size="0.01"/>
    </body>
  </worldbody>
  <actuator>
    <motor name="x_motor" joint="root_x" gear="1" ctrllimited="true" ctrlrange="-1 1"/>
    <motor name="y_motor" joint="root_y" gear="1" ctrllimited="true" ctrlrange="-1 1"/>
  </actuator>
  <sensor>
    <user name="Position" dim="2" user="0 5.0 0.0 10.0"/>
    <user name="Velocity" dim="2" user="0 0.1 0.0 1.0"/>
    <framepos name="trace0" objtype="site" objname="tip"/>
    <framepos name="position" objtype="site" objname="tip"/>
    <framelinvel name="velocity" objtype="site" objname="tip"/>
    <framepos name="goal" objtype="body" objname="goal"/>
  </sensor>
  <keyframe>
    <key name="home" qpos="1.0 2.0" qvel="-1.0 -2.0"/>
    <key name="ctrl_test" ctrl="0.1 0.2"/>
  </keyframe>
</mujoco>
"""


# ----------------------------------------------------------------------------- cartpole
def cartpole_xml() -> str:
    # pole class + actuator: [GUESS] dm_control suite/cartpole.xml (hinge axis 0 1 0, damping 2e-6
    # overridden to 1e-4 by the patch; capsule 0..1 m, r=.045, mass .1; motor gear 10, ctrl +-1)
    return """
<mujoco model="Cart-Pole Swing-Up">
  <option timestep="0.001"><flag contact="disable"/></option>
  <default>
    <default class="pole">
      <joint type="hinge" axis="0 1 0" damping="2e-6"/>
      <geom type="capsule" fromto="0 0 0 0 0 1" size="0.045" mass=".1"/>
    </default>
  </default>
  <custom>
    <numeric name="agent_planner" data="0"/>
    <numeric name="agent_horizon" data="0.31"/>
    <numeric name="agent_timestep" data="0.01"/>
    <numeric name="sampling_spline_points" data="10"/>
    <numeric name="sampling_exploration" data="0.5"/>
    <numeric name="sampling_trajectories" data="8"/>
    <numeric name="residual_Goal" data="0.0 -1.5 1.5"/>
  </custom>
  <worldbody>
    <geom name="floor" pos="0 0 -.05" size="4 4 .2" type="plane"/>
    <body name="cart" pos="0 0 1">
      <joint name="slider" type="slide" limited="true" axis="1 0 0" range="-1.8 1.8" solreflimit=".08 1" damping="1.0e-4"/>
      <geom name="cart" type="box" size="0.2 0.15 0.1" mass="1"/>
      <body name="pole_1" childclass="pole">
        <joint name="hinge_1" damping="1.0e-4"/>
        <geom name="pole_1"/>
        <site name="tip" pos="0 0 1"/>
      </body>
    </body>
  </worldbody>
  <actuator>
    <motor name="slide" joint="slider" gear="10" ctrllimited="true" ctrlrange="-1 1"/>
  </actuator>
  <sensor>
    <user name="Vertical" dim="1" user="6 10.0 0 100.0 0.01"/>
    <user name="Centered" dim="1" user="6 10.0 0 100.0 0.1"/>
    <user name="Velocity" dim="1" user="0 0.1 0.0 1.0"/>
    <user name="Control" dim="1" user="0 0.1 0.0 1.0"/>
    <jointpos name="slider_pos" joint="slider"/>
    <jointpos name="hinge_pos" joint="hinge_1"/>
    <framepos name="trace0" objtype="site" objname="tip"/>
    <framepos name="position" objtype="site" objname="tip"/>
    <framelinvel name="velocity" objtype="site" objname="tip"/>
  </sensor>
  <keyframe>
    <key name="home" qpos="1 0"/>
  </keyframe>
</mujoco>
"""


# ----------------------------------------------------------------------------- quadruped (A1, flat)
_LEGS = (  # name, hip body name, x sign, y sign, joint prefix, foot geom name, site name
    ("FR", "FR_hip", +1, -1, "FR", "FR", "FR"),
    ("FL", "FL_hip", +1, +1, "FL", "FL", "FL"),
    ("RR", "HR_hip", -1, -1, "RR", "HR", "RR"),
    ("RL", "HL_hip", -1, +1, "RL", "HL", "RL"),
)
# hip inertial quaternions per leg (a1.xml.patch:87-190)
_HIP_IQUAT = {"FR": "0.507528 0.506268 0.491507 0.494499", "FL": "0.494499 0.491507 0.506268 0.507528",
              "RR": "0.491507 0.494499 0.507528 0.506268", "RL": "0.506268 0.507528 0.494499 0.491507"}


def _leg_xml(name, hipbody, sx, sy, jp, footgeom, sitename):
    side = "hip_left" if sy > 0 else "hip_right"
    thigh_q = "0.999125 %g -0.0409531 %g" % (0.00256393 * sy, 0.00806091 * sy)
    extra = ('<geom class="collision" size="0.04 0.04" pos="0 0.055 0" quat="1 1 0 0" type="cylinder"/>'
             if name == "FL" else "")  # a1.xml.patch:121 (only FL has the explicit extra cylinder)
    return f"""
      <body name="{hipbody}" pos="{0.183 * sx:g} {0.047 * sy:g} 0">
        <inertial mass="0.696" pos="{-0.003311 * sx:g} {0.000635 * sy:g} 3.1e-05" quat="{_HIP_IQUAT[name]}"
            diaginertia="0.000807752 0.00055293 0.000468983"/>
        <joint class="abduction" name="{jp}_hip_joint"/>
        <geom class="{side}"/>
        {extra}
        <body name="{jp}_thigh" pos="0 {0.08505 * sy:g} 0">
          <inertial mass="1.013" pos="-0.003237 {-0.022327 * sy:g} -0.027326" quat="{thigh_q}"
              diaginertia="0.00555739 0.00513936 0.00133944"/>
          <joint class="hip" name="{jp}_thigh_joint"/>
          <geom class="thigh1"/><geom class="thigh2"/><geom class="thigh3"/>
          <body name="{jp}_calf" pos="0 0 -0.2">
            <inertial mass="0.226" pos="0.00472659 0 -0.131975" quat="0.706886 0.017653 0.017653 0.706886"
                diaginertia="0.00340344 0.00339393 3.54834e-05"/>
            <joint class="knee" name="{jp}_calf_joint"/>
            <geom class="calf1"/><geom class="calf2"/>
            <geom name="{footgeom}" class="foot"/>
            <site name="{sitename}" pos="0 0 -0.2" type="sphere" size=".015"/>
          </body>
        </body>
      </body>"""


def quadruped_flat_xml(horizon=0.63, trajectories=256) -> str:
    legs = "".join(_leg_xml(*leg) for leg in _LEGS)
    acts = "".join(f'<general class="torque" name="{p}_{j}" joint="{p}_{j}_joint"/>'
                   for p in ("FR", "FL", "RR", "RL") for j in ("hip", "thigh", "calf"))
    return f"""
<mujoco model="Quadruped">
  <compiler angle="radian"/>
  <option cone="elliptic" impratio="10"/>
  <custom>
    <numeric name="agent_planner" data="0"/>
    <numeric name="agent_horizon" data="{horizon}"/>
    <numeric name="agent_timestep" data="0.01"/>
    <numeric name="sampling_spline_points" data="3"/>
    <numeric name="sampling_trajectories" data="{trajectories}"/>
    <numeric name="sampling_exploration" data="0.04"/>
    <numeric name="residual_select_Gait" data="0"/>
    <numeric name="residual_select_Gait switch" data="1"/>
    <numeric name="residual_Cadence" data="2 0 4"/>
    <numeric name="residual_Amplitude" data=".06 0 0.2"/>
    <numeric name="residual_Duty ratio" data="0 0 1"/>
    <numeric name="residual_Walk speed" data="0 0 4"/>
    <numeric name="residual_Walk turn" data="0 -2 2"/>
    <numeric name="residual_select_Flip dir" data="0"/>
    <numeric name="residual_select_Biped type" data="0"/>
    <numeric name="residual_Heading" data="0 -3.14 3.14"/>
    <numeric name="residual_Arm posture" data=".03 0 1"/>
  </custom>
  <default>
    <default class="torque">
      <general gainprm="40" ctrllimited="true" ctrlrange="-1 1"/>
    </default>
    <default class="task"><site size=".02" group="5"/></default>
    <default class="prop"><geom type="box"/></default>
    <default class="a1">
      <geom friction="0.6" margin="0.001" condim="1"/>
      <joint axis="0 1 0" damping="2" armature="0.01" frictionloss="0.2" limited="true"/>
      <default class="abduction"><joint axis="1 0 0" damping="1" range="-0.802851 0.802851"/></default>
      <default class="hip"><joint range="-1.9472 3.28879" ref="-0.9"/></default>
      <default class="knee"><joint range="-0.89653 0.883702" ref="1.8"/></default>
      <default class="collision">
        <geom group="3" type="capsule"/>  <!-- [GUESS] Menagerie unitree_a1 collision classes below -->
        <default class="hip_left"><geom size="0.04 0.04" quat="1 1 0 0" type="cylinder" pos="0 0.055 0"/></default>
        <default class="hip_right"><geom size="0.04 0.04" quat="1 1 0 0" type="cylinder" pos="0 -0.055 0"/></default>
        <default class="thigh1"><geom size="0.015" fromto="-0.02 0 0 -0.02 0 -0.16"/></default>
        <default class="thigh2"><geom size="0.015" fromto="0 0 0 -0.02 0 -0.1"/></default>
        <default class="thigh3"><geom size="0.015" fromto="-0.02 0 -0.16 0 0 -0.2"/></default>
        <default class="calf1"><geom size="0.01" fromto="0 0 0 0.02 0 -0.13"/></default>
        <default class="calf2"><geom size="0.01" fromto="0.02 0 -0.13 0 0 -0.2"/></default>
        <default class="foot">
          <geom type="sphere" size="0.02" pos="0 0 -0.2" priority="1" solimp="0.015 1 0.031" condim="6"
                friction="0.8 0.02 0.01"/>
        </default>
      </default>
    </default>
  </default>
  <worldbody>
    <geom name="floor" size="0 0 0.1" pos="0 0 -0.01" type="plane"/>
    <body name="goal" mocap="true" pos=".3 0 0.26">
      <geom size="0.12" contype="0" conaffinity="0" group="2"/>
    </body>
    <body name="box" mocap="true" pos="-2.5 0 0">
      <geom name="box" class="prop" size="1 1 0.3"/>
    </body>
    <geom name="ramp" class="prop" pos="3.13 2.5 -.18" size="1.6 1 .5" euler="0 -0.2 0"/>
    <geom name="hill" class="prop" pos="6 6 -5.5" size="6" type="sphere"/>
    <body name="trunk" pos="0.0 0.0 0.5" quat="1 0 0 0" childclass="a1">
      <site name="torso"/>
      <site name="head" class="task" pos=".3 0 0"/>
      <freejoint/>
      <inertial mass="4.713" pos="0 0.0041 -0.0005"
          fullinertia="0.0158533 0.0377999 0.0456542 -3.66e-05 -6.11e-05 -2.75e-05"/>
      <geom class="collision" size="0.125 0.04 0.057" type="box"/>
      <geom class="collision" quat="1 0 1 0" pos="0 -0.04 0" size="0.058 0.125" type="cylinder"/>
      <!-- [GUESS] 4 trunk geoms outside the patch context (Menagerie unitree_a1) -->
      <geom class="collision" quat="1 0 1 0" pos="0 0.04 0" size="0.058 0.125" type="cylinder"/>
      <geom class="collision" pos="0.25 0 0" size="0.005 0.06 0.05" type="box"/>
      <geom class="collision" pos="0.25 0.06 -0.01" size="0.009 0.035"/>
      <geom class="collision" pos="0.25 -0.06 -0.01" size="0.009 0.035"/>
      <geom class="collision" pos="0.25 0 -0.05" size="0.005 0.06" quat="1 1 0 0"/>
      <geom class="collision" pos="0.255 0 0.0355" size="0.021 0.052" quat="1 1 0 0"/>
      {legs}
    </body>
  </worldbody>
  <actuator>{acts}</actuator>
  <sensor>
    <user name="Upright" dim="3" user="6 1 0 3 0.05"/>
    <user name="Height" dim="1" user="6 1 0 3 0.04"/>
    <user name="Position" dim="3" user="2 0.2 0 0.5 0.1"/>
    <user name="Gait" dim="4" user="6 2 0 10 0.03"/>
    <user name="Balance" dim="2" user="2 0.2 0 0.3 0.1"/>
    <user name="Effort" dim="12" user="0 0.03 0.0 0.1"/>
    <user name="Posture" dim="12" user="0 0.02 0.0 0.1"/>
    <user name="Orientation" dim="2" user="0 0 0 .03"/>
    <user name="Angmom" dim="3" user="0 0 0 .03"/>
    <framepos name="torso_pos" objtype="site" objname="torso"/>
    <framepos name="FR_pos" objtype="site" objname="FR"/>
    <framepos name="FL_pos" objtype="site" objname="FL"/>
    <framepos name="RR_pos" objtype="site" objname="RR"/>
    <framepos name="RL_pos" objtype="site" objname="RL"/>
    {"".join(f'<jointpos name="pos_{p}_{j}_joint" joint="{p}_{j}_joint"/>' for p in ("FR", "FL", "RR", "RL") for j in ("hip", "thigh", "calf"))}
    <touch name="FR_touch" site="FR"/><touch name="FL_touch" site="FL"/>
    <touch name="RR_touch" site="RR"/><touch name="RL_touch" site="RL"/>
    <framepos name="trace0" objtype="site" objname="head"/>
    <subtreecom name="torso_subtreecom" body="trunk"/>
    <subtreelinvel name="torso_subtreelinvel" body="trunk"/>
    <subtreelinvel name="torso_angmom" body="trunk"/>
  </sensor>
  <keyframe>
    <key name="home" qpos="0 0 0.26 1 0 0 0
         -0.000341931 0.0181576 -0.0268335 0.00160968 0.0247957 -0.0270045
         0.00191398 -0.033048 -0.0675298 -0.00199489 -0.0374747 -0.0681862"/>
    <key name="crouch" qpos="-0.0501827 0.00107117 0.143925 1 0 0 0 0 0 -0.5 0 0 -0.5 0 0 -0.5 0 0 -0.5"/>
  </keyframe>
</mujoco>
"""


def _humanoid_leg(side: str, sy: int) -> str:
    """One leg of the MJPC humanoid (mjpc/tasks/humanoid/humanoid.xml.patch:147-201); sy = -1 right, +1 left."""
    s = "right" if side == "r" else "left"
    ax_x = "1 0 0" if sy < 0 else "-1 0 0"
    ax_z = "0 0 1" if sy < 0 else "0 0 -1"
    ankle_x = "1 0 .5" if sy < 0 else "-1 0 -.5"
    sp_a, sp_b = ("sp2", "sp3") if sy < 0 else ("sp0", "sp1")
    return f"""
          <body name="thigh_{s}" pos="0 {0.1 * sy} -.04">
            <site name="tracking[{side}hip]" class="tracking_site" pos="0 {-0.025 * sy} 0.025"/>
            <joint name="hip_x_{s}" axis="{ax_x}" class="hip_x"/>
            <joint name="hip_z_{s}" axis="{ax_z}" class="hip_z"/>
            <joint name="hip_y_{s}" class="hip_y"/>
            <geom name="thigh_{s}" fromto="0 0 0 0 {-0.01 * sy} -.34" class="thigh"/>
            <body name="shin_{s}" pos="0 {-0.01 * sy} -.4">
              <joint name="knee_{s}" class="knee"/>
              <site name="tracking[{side}knee]" class="tracking_site" pos="0 0 0.05"/>
              <geom name="shin_{s}" class="shin"/>
              <body name="foot_{s}" pos="0 0 -.39">
                <joint name="ankle_y_{s}" class="ankle_y"/>
                <joint name="ankle_x_{s}" class="ankle_x" axis="{ankle_x}"/>
                <geom name="foot1_{s}" class="foot1"/>
                <geom name="foot2_{s}" class="foot2"/>
                <site name="foot_{s}" pos=".05 {-0.03 * sy} 0" type="sphere" size=".027"/>
                <site name="{sp_a}" pos="-.07 0 0" type="sphere" size=".027"/>
                <site name="{sp_b}" pos=".14 0 0" type="sphere" size=".027"/>
                <body name="heel_{s}" pos="-0.05 0 0.04">
                  <site name="tracking[{side}heel]" class="tracking_site"/>
                </body>
                <body name="toe_{s}" pos="0.07 0 -0.01">
                  <site name="tracking[{side}toe]" class="tracking_site"/>
                </body>
              </body>
            </body>
          </body>"""


def _humanoid_arm(side: str, sy: int) -> str:
    """One arm (humanoid.xml.patch:258-287); sy = -1 right, +1 left."""
    s = "right" if side == "r" else "left"
    sh1 = "2 1 1" if sy < 0 else "-2 1 -1"
    sh2 = "0 -1 1" if sy < 0 else "0 -1 -1"
    elb = "0 -1 1" if sy < 0 else "0 -1 -1"
    y = -sy   # right arm extends towards -y
    return f"""
      <body name="upper_arm_{s}" pos="0 {0.17 * sy} .06">
        <site name="tracking[{side}shoulder]" class="tracking_site"/>
        <joint name="shoulder1_{s}" axis="{sh1}" class="shoulder"/>
        <joint name="shoulder2_{s}" axis="{sh2}" class="shoulder"/>
        <geom name="upper_arm_{s}" fromto="0 0 0 .16 {0.16 * sy} -.16" class="arm_upper"/>
        <body name="lower_arm_{s}" pos=".18 {0.18 * sy} -.18">
          <joint name="elbow_{s}" axis="{elb}" class="elbow"/>
          <site name="tracking[{side}elbow]" class="tracking_site"/>
          <site name="tracking[{side}hand]" class="tracking_site" pos="0.13 {0.13 * y} 0.13"/>
          <geom name="lower_arm_{s}" fromto=".01 {0.01 * y} .01 .17 {0.17 * y} .17" class="arm_lower"/>
          <body name="hand_{s}" pos=".18 {0.18 * y} .18">
            <geom name="hand_{s}" class="hand"/>
          </body>
        </body>
      </body>"""


_HUMANOID_ACTUATORS = (("abdomen_y", 40), ("abdomen_z", 40), ("abdomen_x", 40),
                       ("hip_x_right", 40), ("hip_z_right", 40), ("hip_y_right", 120), ("knee_right", 100),
                       ("ankle_x_right", 20), ("ankle_y_right", 20),
                       ("hip_x_left", 40), ("hip_z_left", 40), ("hip_y_left", 120), ("knee_left", 100),
                       ("ankle_x_left", 20), ("ankle_y_left", 20),
                       ("shoulder1_right", 20), ("shoulder2_right", 20), ("elbow_right", 40),
                       ("shoulder1_left", 20), ("shoulder2_left", 20), ("elbow_left", 40))


def humanoid_stand_xml(horizon=0.35, trajectories=10) -> str:
    """MJPC "Humanoid Stand": the modified dm_control humanoid (every body, joint, geom, tendon and actuator is
    spelled out by mjpc/tasks/humanoid/humanoid.xml.patch) + mjpc/tasks/humanoid/stand/task.xml.
    Physics features beyond the A1: pyramidal friction cones (MuJoCo's default cone), joint springs, several
    hinges per body, two fixed tendons with limits, motors with gears 20-120."""
    acts = "".join(f'<motor name="{n}" gear="{g}" joint="{n}"/>' for n, g in _HUMANOID_ACTUATORS)
    return f"""
<mujoco model="Humanoid">
  <custom>
    <numeric name="agent_planner" data="0"/>
    <numeric name="agent_horizon" data="{horizon}"/>
    <numeric name="agent_timestep" data="0.015"/>
    <numeric name="sampling_spline_points" data="3"/>
    <numeric name="sampling_exploration" data="0.05"/>
    <numeric name="sampling_trajectories" data="{trajectories}"/>
    <numeric name="gradient_spline_points" data="5"/>
    <numeric name="residual_Height Goal" data="1.4 0.0 1.5"/>
  </custom>
  <default>
    <motor ctrlrange="-1 1" ctrllimited="true"/>
    <site size=".04" group="3"/>
    <default class="body">
      <geom type="capsule" condim="1" friction=".7" solimp=".9 .99 .003" solref=".015 1"/>
      <default class="thigh"><geom size=".06"/></default>
      <default class="shin"><geom fromto="0 0 0 0 0 -.3" size=".049"/></default>
      <default class="foot">
        <geom size=".027"/>
        <default class="foot1"><geom fromto="-.07 -.01 0 .14 -.03 0"/></default>
        <default class="foot2"><geom fromto="-.07 .01 0 .14 .03 0"/></default>
      </default>
      <default class="arm_upper"><geom size=".04"/></default>
      <default class="arm_lower"><geom size=".031"/></default>
      <default class="hand"><geom type="sphere" size=".04"/></default>
      <joint type="hinge" damping=".2" stiffness="1" armature=".01" limited="true" solimplimit="0 .99 .01"/>
      <default class="joint_big">
        <joint damping="5" stiffness="10"/>
        <default class="hip_x"><joint range="-30 10"/></default>
        <default class="hip_z"><joint range="-60 35"/></default>
        <default class="hip_y"><joint axis="0 1 0" range="-150 20"/></default>
        <default class="joint_big_stiff"><joint stiffness="20"/></default>
      </default>
      <default class="knee"><joint pos="0 0 .02" axis="0 -1 0" range="-160 2"/></default>
      <default class="ankle">
        <joint range="-50 50"/>
        <default class="ankle_y"><joint pos="0 0 .08" axis="0 1 0" stiffness="6"/></default>
        <default class="ankle_x"><joint pos="0 0 .04" stiffness="3"/></default>
      </default>
      <default class="shoulder"><joint range="-85 60"/></default>
      <default class="elbow"><joint range="-100 50" stiffness="0"/></default>
      <default class="tracking_site"><site type="sphere" size="0.027" group="3"/></default>
    </default>
  </default>
  <worldbody>
    <geom name="floor" type="plane" conaffinity="1" size="50 50 .05"/>
    <body name="torso" pos="0 0 1.282" childclass="body">
      <freejoint name="root"/>
      <geom name="torso" fromto="0 -.07 0 0 .07 0" size=".07"/>
      <geom name="waist_upper" fromto="-.01 -.06 -.12 -.01 .06 -.12" size=".06"/>
      <body name="head" pos="0 0 .19">
        <geom name="head" type="sphere" size=".09"/>
        <site name="tracking[head]" class="tracking_site" pos="0.09 0 0"/>
      </body>
      <body name="waist_lower" pos="-.01 0 -.26">
        <geom name="waist_lower" fromto="0 -.06 0 0 .06 0" size=".06"/>
        <joint name="abdomen_z" pos="0 0 .065" axis="0 0 1" range="-45 45" class="joint_big_stiff"/>
        <joint name="abdomen_y" pos="0 0 .065" axis="0 1 0" range="-75 30" class="joint_big"/>
        <body name="pelvis" pos="0 0 -.165">
          <site name="tracking[pelvis]" class="tracking_site" pos="0 0 0.075" size=".05"/>
          <joint name="abdomen_x" pos="0 0 .1" axis="1 0 0" range="-35 35" class="joint_big"/>
          <geom name="butt" fromto="-.02 -.07 0 -.02 .07 0" size=".09"/>{_humanoid_leg("r", -1)}{_humanoid_leg("l", 1)}
        </body>
      </body>{_humanoid_arm("r", -1)}{_humanoid_arm("l", 1)}
    </body>
  </worldbody>
  <contact>
    <exclude body1="waist_lower" body2="thigh_right"/>
    <exclude body1="waist_lower" body2="thigh_left"/>
  </contact>
  <tendon>
    <fixed name="hamstring_right" limited="true" range="-0.3 2">
      <joint joint="hip_y_right" coef=".5"/>
      <joint joint="knee_right" coef="-.5"/>
    </fixed>
    <fixed name="hamstring_left" limited="true" range="-0.3 2">
      <joint joint="hip_y_left" coef=".5"/>
      <joint joint="knee_left" coef="-.5"/>
    </fixed>
  </tendon>
  <actuator>{acts}</actuator>
  <sensor>
    <user name="Height" dim="1" user="6 100.0 0.0 100.0 0.1"/>
    <user name="Balance" dim="1" user="6 50.0 0.0 100.0 0.1"/>
    <user name="CoM Vel." dim="2" user="0 10.0 0.0 100.0"/>
    <user name="Joint Vel." dim="21" user="0 0.01 0.0 0.1"/>
    <user name="Control" dim="21" user="3 0.025 0.0 0.1 0.3"/>
    <framepos name="trace0" objtype="body" objname="torso"/>
    <framepos name="torso_position" objtype="body" objname="torso"/>
    <framepos name="head_position" objtype="body" objname="head"/>
    <subtreelinvel name="torso_subtreelinvel" body="torso"/>
    <subtreecom name="torso_subtreecom" body="torso"/>
    <framepos name="sp0" objtype="site" objname="sp0"/>
    <framepos name="sp1" objtype="site" objname="sp1"/>
    <framepos name="sp2" objtype="site" objname="sp2"/>
    <framepos name="sp3" objtype="site" objname="sp3"/>
  </sensor>
</mujoco>
"""


def humanoid_track_xml(horizon=0.5, trajectories=32) -> str:
    """MJPC "Humanoid Track" (mjpc/tasks/humanoid/tracking/task.xml): the same humanoid, dt 0.005, 16 mocap bodies,
    21 cost terms over 141 residuals.  The 1889 CMU keyframes the reference vendors are replaced by synthetic clips
    of the same lengths (synth_mocap below): they are data of the reference, not part of the path."""
    base = humanoid_stand_xml()
    custom = f"""
  <custom>
    <numeric name="sampling_representation" data="2"/>
    <numeric name="agent_planner" data="2"/>
    <numeric name="agent_horizon" data="{horizon}"/>
    <numeric name="agent_timestep" data="0.005"/>
    <numeric name="sampling_spline_points" data="16"/>
    <numeric name="sampling_exploration" data="0.15"/>
    <numeric name="sampling_trajectories" data="{trajectories}"/>
    <numeric name="gradient_spline_points" data="5"/>
    <numeric name="ilqg_num_rollouts" data="16"/>
    <numeric name="ilqg_regularization_type" data="1"/>
    <numeric name="ilqg_representation" data="2"/>
  </custom>
  <option timestep="0.005"/>"""
    mocap = "".join(f'<body name="mocap[{b}]" mocap="true"><site name="mocap[{b}]" type="sphere" size="0.027" group="3"/></body>'
                    for b in T.TRACK_BODIES)
    terms = [("Joint Vel.", 21, "0 0.001 0.0 0.01"), ("Control", 21, "3 0.1 0 1.0 0.3"),
             ("Pos[avg]", 3, "6 100.0 0.0 100.0 0.1"), ("Pos[pelvis]", 3, "6 30.0 0.0 100.0 0.1"),
             ("Pos[head]", 3, "6 0.0 0.0 100.0 0.1"), ("Pos[toe]", 6, "7 30.0 0.0 100.0 0.2 4"),
             ("Pos[heel]", 6, "7 30.0 0.0 100.0 0.2 4"), ("Pos[knee]", 6, "6 30.0 0.0 100.0 0.1"),
             ("Pos[hand]", 6, "6 30.0 0.0 100.0 0.1"), ("Pos[elbow]", 6, "7 30.0 0.0 100.0 0.2 4"),
             ("Pos[shoulder]", 6, "6 30.0 0.0 100.0 0.1"), ("Pos[hip]", 6, "6 30.0 0.0 100.0 0.1"),
             ("Vel[root]", 3, "6 0.1 0 1.0 0.3"), ("Vel[head]", 3, "6 0.0 0 1.0 0.3"), ("Vel[toe]", 6, "6 0.1 0 1.0 0.3"),
             ("Vel[heel]", 6, "6 0.1 0 1.0 0.3"), ("Vel[knee]", 6, "6 0.1 0 1.0 0.3"), ("Vel[hand]", 6, "6 0.1 0 1.0 0.3"),
             ("Vel[elbow]", 6, "6 0.1 0 1.0 0.3"), ("Vel[shoulder]", 6, "6 0.1 0 1.0 0.3"), ("Vel[hip]", 6, "6 0.1 0 1.0 0.3")]
    sensors = "".join(f'<user name="{n}" dim="{d}" user="{u}"/>' for n, d, u in terms)
    sensors += '<framepos name="trace0" objtype="body" objname="torso"/>'
    a = base.index("<custom>"); b = base.index("</custom>") + len("</custom>")
    base = base[:a] + custom.strip() + base[b:]
    base = base.replace("  </worldbody>", mocap + "\n  </worldbody>")
    a = base.index("<sensor>"); b = base.index("</sensor>")
    base = base[:a] + "<sensor>" + sensors + base[b:]
    return base.replace('<mujoco model="Humanoid">', '<mujoco model="Humanoid Track">')


# ----------------------------------------------------------------------------------------------- Shadow Hand stand-in
_HAND_KEY = ("1 0 0 0 0.33326 -0.00362331 0.0375343 0.707635 0.70405 0.0500937 -0.0325089 5.55212e-10 -0.235248 -0.178041 "
             "0.480484 0.730515 0.6284 -0.059347 0.535468 0.746225 0.56556 -0.03491 0.544632 0.53414 0.793355 0.384846 "
             "-0.254843 0.178072 0.761935 0.746225 -0.90042 0.06721 0.01047 0.6981 0.4255")   # shadow_reorient/task.xml:60


def _hand_finger(name: str, y: float, metacarpal: bool = False) -> str:
    """One finger of the stand-in: knuckle J4 (abduction, about z), J3 / J2 / J1 flexion about -y (positive angles curl
    the finger towards +z, the palm side); the little finger has the extra metacarpal joint J5.  Collision = two
    spheres per link (sphere-box is the narrow phase the engine implements for the cube)."""
    def link(j, length, jrange, inner):
        return (f'<body name="rh_{name}{j}" pos="{{pos}}"><joint name="rh_{name}J{j}" axis="0 -1 0" range="{jrange}"/>'
                f'<geom class="link" fromto="0 0 0 {length} 0 0"/>'
                f'<geom class="pad" pos="{0.3 * length:.4f} 0 0"/><geom class="pad" pos="{0.8 * length:.4f} 0 0"/>{inner}</body>')
    distal = link(1, 0.026, "0 1.5708", "").format(pos="0.025 0 0")
    middle = link(2, 0.025, "0 1.5708", distal).format(pos="0.045 0 0")
    prox = link(3, 0.045, "-0.2618 1.5708", middle).format(pos="0 0 0")
    knuckle = (f'<body name="rh_{name}knuckle" pos="{{pos}}"><joint name="rh_{name}J4" axis="0 0 1" range="-0.349 0.349"/>'
               f'<geom class="link" fromto="0 0 0 0.005 0 0"/>{prox}</body>')
    if metacarpal:
        return (f'<body name="rh_{name}metacarpal" pos="0.07 {y} 0.0236"><joint name="rh_{name}J5" axis="0.571 0 0.821" range="0 0.785"/>'
                f'<geom class="link" fromto="0 0 0 0.04 0 0"/><geom class="pad" pos="0.02 0 0.004"/>'
                + knuckle.format(pos="0.04 0 0") + "</body>")
    return knuckle.format(pos=f"0.11 {y} 0.0236")


def shadow_reorient_xml(horizon=0.25, trajectories=60) -> str:
    """MJPC "In-Hand Manipulation" (mjpc/tasks/shadow_reorient/task.xml + hand.cc) on a STAND-IN hand.

    The reference includes Menagerie's shadow_hand/right_hand.xml with its mesh assets (CMakeLists.txt fetches them at
    configure time; not vendored, not available offline), so the hand below is a primitive-geom stand-in [GUESS: every
    hand length, mass, joint range and gain]: the same kinematic layout and order - 2 wrist + 4 + 4 + 4 + 5 (little)
    + 5 (thumb) = 24 hinges, 20 position actuators of which five act on fixed tendons coupling the two distal joints
    (rh_*J0 = J2 + J1), a grasp_site on the palm - so nq / nv / nu = 35 / 33 / 20 and the qpos layout the residual's
    literal `qpos + 7` / `qvel + 6` offsets assume.  What IS the reference's: the goal body and the cube
    (common_assets/reorientation_cube.xml + cube.xml.patch), the cost terms, the custom numerics, the 35-value grasp
    keyframe.  Collisions: cube (box) vs two spheres per finger link + a 4 x 3 grid on the palm (sphere-box), cube vs
    floor (plane-box); finger-finger collisions are switched off by contype / conaffinity."""
    fingers = "".join(_hand_finger(n, y) for n, y in (("FF", 0.033), ("MF", 0.011), ("RF", -0.011)))
    little = _hand_finger("LF", -0.033, metacarpal=True)
    palm_pads = "".join(f'<geom class="palmpad" pos="{0.035 + 0.022 * i:.3f} {-0.022 + 0.022 * j:.3f} 0.0271"/>'
                        for i in range(4) for j in range(3))
    thumb = """
          <body name="rh_thbase" pos="0.049 0.034 0.0236">
            <joint name="rh_THJ5" axis="0 0 -1" range="-1.047 1.047"/>
            <geom class="link" fromto="0 0 0 0 0.005 0"/>
            <body name="rh_thproximal" pos="0 0 0">
              <joint name="rh_THJ4" axis="1 0 0" range="0 1.222"/>
              <geom class="thlink" fromto="0 0 0 0 0.038 0"/><geom class="thpad" pos="0 0.012 0"/><geom class="thpad" pos="0 0.03 0"/>
              <body name="rh_thhub" pos="0 0.038 0">
                <joint name="rh_THJ3" axis="1 0 0" range="-0.209 0.209"/>
                <geom class="thlink" fromto="0 0 0 0 0.002 0"/>
                <body name="rh_thmiddle" pos="0 0 0">
                  <joint name="rh_THJ2" axis="0 0 1" range="-0.698 0.698"/>
                  <geom class="thlink" fromto="0 0 0 0 0.032 0"/><geom class="thpad" pos="0 0.01 0"/><geom class="thpad" pos="0 0.026 0"/>
                  <body name="rh_thdistal" pos="0 0.032 0">
                    <joint name="rh_THJ1" axis="0 0 1" range="-0.262 1.571"/>
                    <geom class="thlink" fromto="0 0 0 0 0.0275 0"/><geom class="thpad" pos="0 0.008 0"/><geom class="thpad" pos="0 0.022 0"/>
                  </body>
                </body>
              </body>
            </body>
          </body>"""
    def pos_act(j, lo, hi, kp=1.0):
        return f'<position name="rh_A_{j}" joint="rh_{j}" kp="{kp}" ctrlrange="{lo} {hi}" forcerange="-2 2"/>'
    acts = pos_act("WRJ2", -0.523, 0.174, 10) + pos_act("WRJ1", -0.698, 0.489, 10)
    for f in ("FF", "MF", "RF"):
        acts += pos_act(f + "J4", -0.349, 0.349) + pos_act(f + "J3", -0.262, 1.571)
        acts += f'<position name="rh_A_{f}J0" tendon="rh_{f}J0" kp="1" ctrlrange="0 3.1415" forcerange="-2 2"/>'
    acts += pos_act("LFJ5", 0, 0.785) + pos_act("LFJ4", -0.349, 0.349) + pos_act("LFJ3", -0.262, 1.571)
    acts += '<position name="rh_A_LFJ0" tendon="rh_LFJ0" kp="1" ctrlrange="0 3.1415" forcerange="-2 2"/>'
    acts += (pos_act("THJ5", -1.047, 1.047) + pos_act("THJ4", 0, 1.222) + pos_act("THJ3", -0.209, 0.209)
             + pos_act("THJ2", -0.698, 0.698) + pos_act("THJ1", -0.262, 1.571))
    tendons = "".join(f'<fixed name="rh_{f}J0"><joint joint="rh_{f}J2" coef="1"/><joint joint="rh_{f}J1" coef="1"/></fixed>'
                      for f in ("FF", "MF", "RF", "LF"))
    return f"""
<mujoco model="In-Hand Manipulation">
  <compiler angle="radian" autolimits="true"/>
  <option timestep="0.01"/>
  <custom>
    <numeric name="agent_planner" data="5"/>
    <numeric name="agent_horizon" data="{horizon}"/>
    <numeric name="agent_timestep" data="0.01"/>
    <numeric name="agent_policy_width" data="0.0035"/>
    <numeric name="sampling_spline_points" data="5"/>
    <numeric name="sampling_exploration" data="0.2"/>
    <numeric name="sampling_representation" data="0"/>
    <numeric name="sampling_trajectories" data="{trajectories}"/>
    <numeric name="n_elite" data="8"/>
    <numeric name="explore_fraction" data="0.5"/>
    <numeric name="robust_xfrc" data="0.004"/>
  </custom>
  <default>
    <geom friction=".6"/>
    <joint type="hinge" damping="0.05" armature="0.0002"/>
    <default class="link"><geom type="capsule" size="0.008" mass="0.012" contype="0" conaffinity="0" group="2"/></default>
    <default class="thlink"><geom type="capsule" size="0.010" mass="0.016" contype="0" conaffinity="0" group="2"/></default>
    <default class="pad"><geom type="sphere" size="0.009" mass="0.002" contype="2" conaffinity="0" group="3"/></default>
    <default class="thpad"><geom type="sphere" size="0.011" mass="0.003" contype="2" conaffinity="0" group="3"/></default>
    <default class="palmpad"><geom type="sphere" size="0.012" mass="0.02" contype="2" conaffinity="0" group="3"/></default>
  </default>
  <worldbody>
    <geom name="floor" pos="0 0 -0.2" size="0 0 0.05" type="plane"/>
    <body name="goal" pos="0.325 0.17 0.0475">
      <joint type="ball" damping="0.01"/>
      <geom type="box" size=".022 .022 .022" mass=".126" contype="0" conaffinity="0"/>
    </body>
    <body name="cube" pos="0.325 0.0 0.075" quat="0.707 0.707 0 0">
      <freejoint/>
      <geom name="cube" type="box" size=".022 .022 .022" mass=".126" contype="1" conaffinity="3"/>
    </body>
    <body name="rh_forearm" pos="0 0 0">
      <geom class="link" type="capsule" size="0.03" fromto="0.08 0 -0.01 0.21 0 -0.01" mass="1"/>
      <body name="rh_wrist" pos="0.235 0 0">
        <joint name="rh_WRJ2" axis="0 0 1" range="-0.523 0.174"/>
        <geom class="link" fromto="0 0 0 0.01 0 0"/>
        <body name="rh_palm" pos="0 0 0">
          <joint name="rh_WRJ1" axis="0 -1 0" range="-0.698 0.489"/>
          <geom name="rh_palm_box" type="box" size="0.05 0.042 0.006" pos="0.065 0 0.0196" mass="0.3" contype="0" conaffinity="0" group="2"/>
          <site name="grasp_site" pos="0.098 0 0.0636" size="0.005"/>
          {palm_pads}
          {fingers}
          {little}
          {thumb}
        </body>
      </body>
    </body>
  </worldbody>
  <tendon>{tendons}</tendon>
  <actuator>{acts}</actuator>
  <sensor>
    <user name="In Hand" dim="3" user="1 20 0 100 0.02 2"/>
    <user name="Orientation" dim="3" user="0 5 0 10"/>
    <user name="Cube Vel." dim="3" user="0 10 0 20"/>
    <user name="Actuator" dim="20" user="0 0.1 0.0 1.0"/>
    <user name="Grasp" dim="26" user="0 2.5 0.0 10.0"/>
    <user name="Joint Vel." dim="26" user="0 1.0e-4 0.0 1.0e-1"/>
    <framepos name="palm_position" objtype="site" objname="grasp_site"/>
    <framequat name="cube_goal_orientation" objtype="body" objname="goal"/>
    <framepos name="trace0" objtype="body" objname="cube"/>
    <framepos name="cube_position" objtype="body" objname="cube"/>
    <framequat name="cube_orientation" objtype="body" objname="cube"/>
    <framelinvel name="cube_linear_velocity" objtype="body" objname="cube"/>
  </sensor>
  <keyframe><key name="grasp" qpos="{_HAND_KEY}"/></keyframe>
</mujoco>"""


def synth_mocap(m, seed=0):
    """Synthetic stand-in for the reference's CMU keyframes: 10 clips with the reference's lengths (tracking.cc:43-54),
    30 fps.  Each clip is a smooth band-limited joint-angle motion inside 35 % of the joint ranges around the standing
    pose (different frequencies / phases per clip and joint) with the root lowered so the lowest foot marker stays at
    its standing height; the 16 tracked site positions of that pose are the frame's mocap positions.
    Returns key_qpos [K][nq], key_mpos [K][16*3]."""
    from ..refmath import kinematics
    from ..mjcf import quat2mat
    rng = np.random.default_rng(seed)
    sites = [m.site_names.index("tracking[%s]" % b) for b in T.TRACK_BODIES]
    foot = [T.TRACK_BODIES.index(b) for b in ("ltoe", "rtoe", "lheel", "rheel")]
    hinge = [j for j in range(m.njnt) if m.jnt_type[j] == 3]
    lo = np.array([m.jnt_range[j][0] for j in hinge]); hi = np.array([m.jnt_range[j][1] for j in hinge])
    qadr = np.array([m.jnt_qposadr[j] for j in hinge])

    def markers(q):
        kin = kinematics(m, q)
        return np.array([kin["xpos"][m.site_bodyid[s]] + kin["xmat"][m.site_bodyid[s]] @ m.site_pos[s] for s in sites])
    stand = markers(m.qpos0)
    z_foot = stand[foot, 2].min()
    kq, km = [], []
    for clip, length in enumerate(T.TRACK_MOTION_LENGTHS):
        f = rng.uniform(0.3, 1.2, len(hinge)); ph = rng.uniform(0, 2 * np.pi, len(hinge))
        amp = 0.35 * rng.uniform(0.2, 1.0, len(hinge))
        for k in range(length):
            t = k / T.TRACK_FPS
            env = min(1.0, t / 0.5)                       # every clip starts from the standing pose
            q = m.qpos0.copy()
            s = np.sin(2 * np.pi * f * t + ph) - np.sin(ph)
            q[qadr] = np.clip(env * amp * s * 0.5 * (hi - lo), 0.9 * lo, 0.9 * hi)
            q[0] = 0.15 * env * np.sin(2 * np.pi * 0.2 * t + clip)          # slow drift of the root in x
            mk = markers(q)
            dz = z_foot - mk[foot, 2].min()
            q[2] += dz; mk[:, 2] += dz
            kq.append(q); km.append(mk.reshape(-1))
    return np.array(kq), np.array(km)


def track_keyframes(keyframes_dir=None, synthetic=False):
    """The Humanoid Track mocap clips (mjpc/tasks/humanoid/tracking/keyframes/*.xml, tracking.cc:43-54).  Order of
    preference: an explicit directory (or $MJPC_B200_TRACK_KEYFRAMES) holding the reference's XML files, parsed here;
    the committed fixture tests/golden/humanoid_track_keyframes.npz (the same data parsed by make_track_keyframes.py, so
    that the task runs without the reference tree); None -> the caller falls back to synth_mocap.
    Returns (dict(mpos, qpos, qvel) | None, source string)."""
    import os
    if synthetic:
        return None, "synthetic clips (synth_mocap)"
    d = keyframes_dir or os.environ.get("MJPC_B200_TRACK_KEYFRAMES")
    if d:
        from .make_track_keyframes import parse_keyframes
        return parse_keyframes(d), "reference keyframes parsed from " + d
    fx = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "tests", "golden",
                      "humanoid_track_keyframes.npz")
    if os.path.exists(fx):
        z = np.load(fx)
        return dict(mpos=z["mpos"].astype(float), qpos=z["qpos"].astype(float), qvel=z["qvel"].astype(float)), \
            "reference keyframes (1889 CMU frames, fixture tests/golden/humanoid_track_keyframes.npz)"
    return None, "synthetic clips (synth_mocap): fixture missing"


def _robot_vs_world_only(m, g1, g2):
    """Pair filter of `self_collision=False`: keep only pairs with exactly one static (world-welded) geom.  The default
    (self_collision=True) keeps every pair MuJoCo's filters keep and the narrow phase implements (capsule-capsule,
    sphere-capsule, sphere-sphere, sphere-box between robot bodies); pairs that need MuJoCo's general convex collider
    (cylinder / box against capsule, box-box) are listed in Model.pairs_dropped."""
    s1 = m.body_weldid[m.geom_bodyid[g1]] == 0
    s2 = m.body_weldid[m.geom_bodyid[g2]] == 0
    return bool(s1) != bool(s2)


def _ray_geoms(m):
    """Group-0 geoms are what mjpc::Ground ray-casts against (utilities.cc:556-574)."""
    return np.array([g for g in range(m.ngeom) if m.geom_group[g] == 0], np.int32)


def load(name: str, agent_timestep: bool = True, self_collision: bool = True, **kw):
    """Compile one of the built-in tasks. Returns the Model with task ids / state filled in.

    agent_timestep=True applies Agent's override of opt.timestep by the ``agent_timestep`` numeric
    (mjpc/agent.cc:288); False keeps the model's own <option timestep> (as mjpc/test/agent/rollout_test.cc does)."""
    if name in ("particle", "particle_copy"):
        m = compile_xml(particle_xml())
        m.task_residual_id = T.RESIDUAL_PARTICLE if name == "particle" else T.RESIDUAL_PARTICLE_COPY
        m.task_ids = np.zeros(1, np.int32)
        m.task_state = np.zeros(1)
    elif name == "cartpole":
        m = compile_xml(cartpole_xml())
        m.task_residual_id = T.RESIDUAL_CARTPOLE
        m.task_ids = np.zeros(1, np.int32)
        m.task_state = np.zeros(1)
    elif name == "quadruped":
        m = compile_xml(quadruped_flat_xml(**kw), pair_filter=None if self_collision else _robot_vs_world_only)
        m.task_residual_id = T.RESIDUAL_QUADRUPED_FLAT
        ids = np.zeros(T.QI_SIZE, np.int32)
        ids[T.QI_TORSO_BODY] = m.body_names.index("trunk")
        ids[T.QI_HEAD_SITE] = m.site_names.index("head")
        ids[T.QI_GOAL_MOCAP] = m.body_mocapid[m.body_names.index("goal")]
        for k, f in enumerate(("FL", "HL", "FR", "HR")):  # quadruped.cc:560-566
            ids[T.QI_FOOT_GEOM + k] = m.geom_names.index(f)
        pn = [p[len("residual_"):] for p in m.task_parameter_names]
        ids[T.QI_PARAM_GAIT] = pn.index("select_Gait")
        ids[T.QI_PARAM_BIPED_TYPE] = pn.index("select_Biped type")
        ids[T.QI_PARAM_CADENCE] = pn.index("Cadence")
        ids[T.QI_PARAM_AMPLITUDE] = pn.index("Amplitude")
        ids[T.QI_PARAM_DUTY] = pn.index("Duty ratio")
        ids[T.QI_PARAM_ARM_POSTURE] = pn.index("Arm posture")
        ids[T.QI_PARAM_HEADING] = pn.index("Heading")
        ids[T.QI_PARAM_FLIP_DIR] = pn.index("select_Flip dir")
        ids[T.QI_KEY_HOME] = m.key_names.index("home")
        ids[T.QI_KEY_CROUCH] = m.key_names.index("crouch")
        m.task_ids = ids
        m.task_state = T.quadruped_state_block(float(np.linalg.norm(m.opt_gravity)),
                                               float(m.task_parameters[pn.index("Cadence")]))
    elif name == "humanoid":
        m = compile_xml(humanoid_stand_xml(**kw), pair_filter=None if self_collision else _robot_vs_world_only)
        m.task_residual_id = T.RESIDUAL_HUMANOID_STAND
        ids = np.zeros(T.HI_SIZE, np.int32)
        ids[T.HI_TORSO_BODY] = m.body_names.index("torso")
        ids[T.HI_HEAD_BODY] = m.body_names.index("head")
        for k in range(4):
            ids[T.HI_SITE_SP0 + k] = m.site_names.index("sp%d" % k)
        m.task_ids = ids
        m.task_state = np.zeros(1)
    elif name == "humanoid_track":
        keyframes_dir, synthetic = kw.pop("keyframes_dir", None), kw.pop("synthetic_keyframes", False)
        m = compile_xml(humanoid_track_xml(**kw), pair_filter=None if self_collision else _robot_vs_world_only)
        m.task_residual_id = T.RESIDUAL_HUMANOID_TRACK
        ids = [m.site_names.index("tracking[%s]" % b) for b in T.TRACK_BODIES]
        ids += [int(m.body_mocapid[m.body_names.index("mocap[%s]" % b)]) for b in T.TRACK_BODIES]
        m.task_ids = np.array(ids, np.int32)
        m.task_state = np.zeros(T.TS_SIZE)               # mode 0 (first clip), reference_time 0
        kf, m.key_source = track_keyframes(keyframes_dir, synthetic)
        if kf is not None:
            # the reference's 1889 CMU frames (tracking.cc:43-54); a <key> without qpos / qvel takes the model defaults
            km = np.asarray(kf["mpos"], float)
            kq = np.where(np.isnan(kf["qpos"]), m.qpos0[None, :], kf["qpos"]).astype(float)
            kv = np.asarray(kf["qvel"], float)
            if kq.shape[1] != m.nq or km.shape[1] != 3 * m.nmocap:
                raise ValueError("keyframes do not match the humanoid model (nq %d, nmocap %d)" % (m.nq, m.nmocap))
        else:
            kq, km = synth_mocap(m)
            kv = np.zeros((len(kq), m.nv))
        m.nkey = len(kq)
        m.key_qpos, m.key_mpos = kq, km
        m.key_qvel = kv; m.key_ctrl = np.zeros((m.nkey, m.nu))
        m.key_mquat = np.tile(np.array([1.0, 0, 0, 0]), (m.nkey, m.nmocap))
        m.key_names = ["frame%d" % i for i in range(m.nkey)]
        m.mocap_pos0 = km[0].reshape(-1, 3).copy()
    elif name == "shadow_reorient":
        m = compile_xml(shadow_reorient_xml(**kw))
        m.task_residual_id = T.RESIDUAL_SHADOW_REORIENT
        ids = np.zeros(T.SI_SIZE, np.int32)
        ids[T.SI_GRASP_SITE] = m.site_names.index("grasp_site")
        ids[T.SI_CUBE_BODY] = m.body_names.index("cube")
        ids[T.SI_GOAL_BODY] = m.body_names.index("goal")
        ids[T.SI_KEY_GRASP] = m.key_names.index("grasp")
        m.task_ids = ids
        m.task_state = np.zeros(1)
        m.model_note = "Shadow Hand STAND-IN (primitive geoms, [GUESS] dimensions): Menagerie's right_hand.xml is not vendored"
    else:
        raise KeyError(name)
    m.task_name = name
    # agent settings (mjpc/agent.cc:90-107): planning timestep / integrator / horizon
    if agent_timestep and "agent_timestep" in m.numeric:
        m.opt_timestep = float(m.numeric["agent_timestep"][0])
    m.ray_geoms = _ray_geoms(m)
    return m
