"""The drop-in classes on a costmap-sized scene, driven through their test program
teb_local_planner_b200/host/test/test_dropin_large: TebOptimalPlanner::plan with 3000 PointObstacles returns true and
its band equals tebgpu_optimize_batch on the same inputs; HomotopyClassPlanner::plan refuses the scene (its
H-signature stops at 1024 obstacles)."""
import os
import subprocess

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "teb_local_planner_b200", "host", "test", "test_dropin_large")


@pytest.fixture(scope="module")
def exe():
    from teb_local_planner_b200 import build as b
    try:
        b.build()
        b.build_host()
    except Exception:
        if not os.path.exists(EXE):
            raise
    return EXE


def _costmap_points(count):
    """the scene of test_dropin_large.cpp: cell k at column k % 160, row k // 160 alternating above / below the band"""
    o = np.zeros(count, abi.OBST_DTYPE)
    k = np.arange(count)
    row = k // 160
    o["x"] = -4.0 + 0.05 * (k % 160)
    o["y"] = np.where(row % 2 == 1, -1.0, 1.0) * (1.0 + 0.05 * (row // 2))
    return o


@pytest.mark.gpu
def test_dropin_plan_with_3000_point_obstacles(exe, oracle):
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "RESULT DONE" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
    lines = [ln.split() for ln in out.stdout.splitlines() if ln.strip()]
    vals = {f[0]: f[1:] for f in lines if not f[0].endswith("_POSE")}
    got = np.array([[float(x) for x in f[2:6]] for f in lines if f[0] == "LARGE_POSE"])
    assert vals["LARGE_OK"][0] == "1" and int(vals["LARGE_STATUS"][0]) & abi.TEB_STATUS_OPTIMIZED
    assert vals["LARGE_HCP_OK"][0] == "0"
    # the same request through the C-ABI: cold start of plan(start, goal), the drop-in's capacity (max_samples + 1)
    p = abi.default_params()
    obst = _costmap_points(3000)
    rec0 = oracle.init_trajectory([-4, 0, 0], [4, 0, 0], 0.0, p.max_vel_x, p.min_samples)
    n_cap = p.max_samples + 1
    poses = np.zeros((1, n_cap, 4))
    poses[0, :len(rec0)] = rec0
    hb = abi.HostBatch(poses, np.array([len(rec0)], np.int32), obst, np.array([3000], np.int32))
    g = T.TebGpu(1, n_cap, 1, 3000, 0)
    g.set_params(p)
    g.optimize(hb, abi.make_args(p.no_inner_iterations, p.no_outer_iterations, False))
    g.close()
    assert len(got) == hb.n[0] and len(got) > 20
    assert np.array_equal(got, hb.poses[0, :hb.n[0]])
    # and the oracle on the same inputs
    ref, _, _ = oracle.optimize_band(p, rec0, len(rec0), obst, args=abi.make_args(5, 4, False), jac_mode=oracle.JAC_ANALYTIC,
                                     n_cap=512)
    assert len(ref) == len(got) and np.abs(got - ref).max() < 1e-6
