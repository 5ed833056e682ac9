"""testspeed-style closed loop (mjpc/testspeed.cc:44-128): plan, act, step the plant, report wall time, x realtime and
the average cost per step.  The plant is the fp64 oracle (test infrastructure - which is why this tool lives under
profiles/ and not in the product package); the planner runs on the CUDA engine (--backend b200) or on the oracle
ThreadPool path (--backend oracle, CPU only).

  python profiles/testspeed.py --task quadruped --planner sampling --steps 200 --backend b200
"""
import argparse, os, sys, time
import numpy as np
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, R); sys.path.insert(0, os.path.join(R, "tests"))
from conftest import OracleBackend, get_model, mocap_of


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", default="quadruped", choices=["quadruped", "humanoid", "humanoid_track", "cartpole", "particle"])
    ap.add_argument("--planner", default="sampling", choices=["sampling", "cross_entropy", "robust", "sample_gradient"])
    ap.add_argument("--backend", default="b200", choices=["b200", "oracle"])
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--candidates", type=int, default=0)
    ap.add_argument("--horizon", type=int, default=0)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    a = ap.parse_args(argv)
    from mujoco_mpc_b200.blob import to_blob
    from mujoco_mpc_b200 import planner as P
    from oracle import pyoracle
    m = get_model(a.task)
    plant = pyoracle.Oracle(to_blob(m), m, 64)
    N = a.candidates or int(m.numeric.get("sampling_trajectories", [10])[0])
    H = a.horizon or int(max(min(m.numeric.get("agent_horizon", [0.5])[0] / m.opt_timestep + 1, 512), 1))
    extra = 1 if a.planner == "cross_entropy" else 0
    if a.backend == "b200":
        from mujoco_mpc_b200.engine import Engine
        backend = Engine(m, N + extra, H)
    else:
        backend = OracleBackend(m, threads=a.threads)
    cls = {"sampling": P.SamplingPlanner, "cross_entropy": P.CrossEntropyPlanner, "robust": P.RobustPlanner,
           "sample_gradient": P.SampleGradientPlanner}[a.planner]
    pl = cls(m, backend, num_trajectory=N, horizon=H)
    pl.reset(np.zeros(m.nu)) if a.planner != "cross_entropy" else pl.reset()
    transition = None
    if a.task == "humanoid_track":
        from mujoco_mpc_b200.transition import HumanoidTrackTransition
        transition = HumanoidTrackTransition(m)
    q = (m.key_qpos[0] if m.nkey else m.qpos0).copy(); v = np.zeros(m.nv)
    mocap = mocap_of(m) if m.nmocap else np.zeros(0)
    t, warm, total_cost, plan_s = 0.0, None, 0.0, 0.0
    t0 = time.perf_counter()
    for k in range(a.steps):
        if transition is not None:
            q, v, mocap = transition.transition(t, q, v)
            plant.set_task(task_state=transition.task_state())
            if hasattr(backend, "set_task"):
                backend.set_task(task_state=transition.task_state())
            else:
                backend.o.set_task(task_state=transition.task_state())
        p0 = time.perf_counter()
        pl.set_state(np.concatenate([q, v]), t, mocap)
        pl.optimize_policy()
        u = pl.action_from_policy(t)
        plan_s += time.perf_counter() - p0
        r = plant.forward_debug(q, v, u, mocap, time=t, warmstart=warm)
        total_cost += plant.cost_value(r["residual"][: m.task_num_residual])
        q, v, warm = r["next_qpos"], r["next_qvel"], r["qacc"]
        t += m.opt_timestep
    wall = time.perf_counter() - t0
    out = dict(task=a.task, planner=a.planner, backend=a.backend, candidates=N, horizon=H, steps=a.steps, wall_s=wall,
               plan_ms_per_step=1e3 * plan_s / a.steps, x_realtime=a.steps * m.opt_timestep / wall,
               average_cost=total_cost / a.steps)
    print("Total wall time (%d steps): %.3f s (%.2fx realtime), planning %.2f ms/step\nAverage cost per step (lower is better): %.4f" % (
        a.steps, wall, out["x_realtime"], out["plan_ms_per_step"], out["average_cost"]))
    return out


if __name__ == "__main__":
    main()
