"""GPU, 2 ranks on 2 GPUs (skipped with fewer): ONE planning problem sharded inside libmjpc_b200.so - contiguous candidate
ranges, one ncclAllGather of (return, failure) per iteration on the engine stream, ranking on the device, winner
trajectory ncclBroadcast from its owner (SURVEY.md 8e).  Checks: identical returns / order on both ranks, BIT-identical
to the single-GPU run of the same problem, ragged shards, identical installed policy after planner iterations."""
import os
import socket

import numpy as np
import pytest

from conftest import get_model, quadruped_inputs

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)      # plumbing only: carries the ncclUniqueId
    from mujoco_mpc_b200.engine import Engine
    from mujoco_mpc_b200.planner import SamplingPlanner
    from mujoco_mpc_b200.sharding import ShardedRollouts
    m = get_model("quadruped")
    N, H = 25, 16                                                       # ragged: 13 + 12
    e = Engine(m, 16, H, device=rank)
    e.comm_init_torch(dist)
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    ret, fail, order = e.rollout_spline_sharded(state, 0.0, mocap, knots, kt, 2, H)
    win = e.fetch_trajectory_sharded(int(order[0]))
    last = e.fetch_trajectory_sharded(N - 1)                            # owned by the last rank
    sh = ShardedRollouts(e, dist)
    pl = SamplingPlanner(m, sh, num_trajectory=N, horizon=H)
    pl.reset(); pl.set_state(state, 0.0, mocap)
    pl.optimize_policy(); pl.optimize_policy()
    q.put((rank, ret, fail, order, win["states"], last["states"], pl.values, pl.winner, e.launch_count))
    dist.barrier()
    e.close()
    dist.destroy_process_group()


def test_two_gpu_sharded_rollouts_match_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in range(2)], key=lambda x: x[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    from mujoco_mpc_b200.engine import Engine
    m = get_model("quadruped")
    N, H = 25, 16
    state, mocap, knots, kt = quadruped_inputs(m, N=N, H=H)
    e = Engine(m, N, H, device=0)
    ref_ret, ref_fail, ref_order = e.rollout_spline(state, 0.0, mocap, knots, kt, 2, H)
    ref_win = e.fetch_trajectory(int(ref_order[0]))["states"]; ref_last = e.fetch_trajectory(N - 1)["states"]
    e.close()
    for rank, ret, fail, order, win, last, values, winner, launches in res:
        assert np.array_equal(ret.view(np.uint32), ref_ret.view(np.uint32))      # bit-identical to the 1-GPU run
        assert np.array_equal(order, ref_order) and not fail.any()
        assert np.array_equal(win, ref_win) and np.array_equal(last, ref_last)
        assert launches > 0
    np.testing.assert_array_equal(res[0][6], res[1][6])                             # same installed policy
    assert res[0][7] == res[1][7]
