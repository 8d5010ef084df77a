"""The drop-in C++ classes (TebOptimalPlanner / HomotopyClassPlanner / TimedElasticBand) driven by their C++ test
program teb_local_planner_b200/host/test/test_dropin: CPU checks always, the GPU scenes under -m gpu, where the printed
bands are compared with the CPU oracle fed with the same initialisation logic restated in Python."""
import math
import os
import subprocess

import numpy as np
import pytest

from teb_local_planner_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "teb_local_planner_b200", "host", "test", "test_dropin")


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


def test_dropin_cpu_checks(exe):
    """test/teb_basics.cpp gtests on the drop-in TimedElasticBand, cold/warm start plumbing, config defaults"""
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "RESULT PASS" in out.stdout, out.stdout + out.stderr


def _parse(stdout):
    vals, bands = {}, {}
    for ln in stdout.splitlines():
        f = ln.split()
        if not f:
            continue
        if f[0].endswith("_POSE"):
            bands.setdefault(f[0][:-5], []).append([float(x) for x in f[2:6]])
        else:
            vals.setdefault(f[0], []).append(f[1:])
    return vals, {k: np.array(v) for k, v in bands.items()}


def _nt(t):
    return (t + math.pi) % (2 * math.pi) - math.pi if not (-math.pi <= t < math.pi) else t


def _init_from_plan(plan, max_vel_x, max_vel_theta):
    """initTrajectoryToGoal(plan, ..., estimate_orient=True) (timed_elastic_band.cpp:389-452)"""
    def est(a, b):
        dt = math.hypot(b[0] - a[0], b[1] - a[1]) / max_vel_x
        return max(dt, abs(_nt(b[2] - a[2])) / max_vel_theta)
    rec = [[plan[0][0], plan[0][1], plan[0][2], 0.0]]
    for i in range(1, len(plan) - 1):
        yaw = math.atan2(plan[i + 1][1] - plan[i][1], plan[i + 1][0] - plan[i][0])
        p = [plan[i][0], plan[i][1], yaw, 0.0]
        rec[-1][3] = est(rec[-1], p)
        rec.append(p)
    g = [plan[-1][0], plan[-1][1], plan[-1][2], 0.0]
    rec[-1][3] = est(rec[-1], g)
    rec.append(g)
    return np.array(rec)


def _prune(rec, new_start, new_goal, min_samples=3):
    """updateAndPruneTEB (timed_elastic_band.cpp:555-597)"""
    rec = rec.copy()
    n = len(rec)
    d_cache = math.hypot(new_start[0] - rec[0, 0], new_start[1] - rec[0, 1])
    nearest = 0
    for i in range(1, min(n - min_samples, 10) + 1):
        d = math.hypot(new_start[0] - rec[i, 0], new_start[1] - rec[i, 1])
        if d < d_cache:
            d_cache, nearest = d, i
        else:
            break
    if nearest > 0:
        # deletePoses(1, nearest) / deleteTimeDiffs(1, nearest): pose 0 keeps timediff 0
        keep = np.concatenate([rec[:1], rec[1 + nearest:]])
        rec = keep
    rec[0, :3] = new_start
    rec[-1, :3] = new_goal
    return rec


@pytest.mark.gpu
def test_dropin_gpu_scenes_match_oracle(exe, oracle):
    out = subprocess.run([exe, "gpu"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "RESULT PASS" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
    vals, bands = _parse(out.stdout)
    # optimizeAllTEBs sharded over two device contexts = the single-context run (costs bitwise, same winner)
    assert vals["SHARDED_OK"][0][0] == "1"
    # ---- test_optim_node scene through TebOptimalPlanner::plan(start, goal) (cold start + autoResize from 3 poses)
    p = abi.default_params()
    obst = np.zeros(3, abi.OBST_DTYPE)
    obst["x"], obst["y"] = [-3.0, 6.0, 0.0], [1.0, 2.0, 0.1]
    obst["vx"], obst["vy"] = [0.1, -0.3, 0.0], [-0.3, -0.2, 0.0]
    obst["dynamic"] = [1, 1, 0]
    rec0 = oracle.init_trajectory([-4, 0, 0], [4, 0, 0], 0.0, p.max_vel_x, p.min_samples)
    ref, _, st = oracle.optimize_band(p, rec0, len(rec0), obst, args=abi.make_args(5, 4, False), jac_mode=oracle.JAC_ANALYTIC,
                                      n_cap=512)
    got = bands["SINGLE"]
    assert vals["SINGLE_OK"][0][0] == "1" and int(vals["SINGLE_STATUS"][0][0]) & abi.TEB_STATUS_OPTIMIZED
    assert len(got) == len(ref) and len(got) > 20          # autoResize grew the 3-pose cold start
    assert np.abs(got - ref).max() < 1e-6
    # computeCurrentCost outside optimizeTEB = chi2 of the freshly built graph at the final state, multiplier 1
    _, _, chi2 = oracle.build_system(p, ref, len(ref), obst, weight_multiplier=1.0, jac_mode=oracle.JAC_ANALYTIC)
    assert abs(float(vals["SINGLE_COST"][0][0]) - chi2) <= 1e-6 * max(chi2, 1.0)
    # getVelocityCommand (optimal_planner.cpp:1136-1172) on the optimised band
    vx, vy, om = (float(x) for x in vals["SINGLE_CMD"][0])
    dt0 = ref[0, 3]
    dx, dy = ref[1, 0] - ref[0, 0], ref[1, 1] - ref[0, 1]
    sgn = np.sign(dx * math.cos(ref[0, 2]) + dy * math.sin(ref[0, 2]))
    assert abs(vx - sgn * math.hypot(dx, dy) / dt0) < 1e-6 and vy == 0 and abs(om - _nt(ref[1, 2] - ref[0, 2]) / dt0) < 1e-6
    # warm start: prune + new start + start velocity
    w0 = _prune(ref, [-3.9, 0.01, 0.02], [4, 0, 0])
    wref, _, _ = oracle.optimize_band(p, w0, len(w0), obst, vel_start=[vx, 0, om, 1.0], args=abi.make_args(5, 4, False),
                                      jac_mode=oracle.JAC_ANALYTIC, n_cap=512)
    wgot = bands["WARM"]
    assert len(wgot) == len(wref) and np.abs(wgot - wref).max() < 1e-6
    # optimizeTEB(5, 0) returns true with isOptimized() false; optimizeTEB(0, 3) returns false (optimal_planner.cpp:230, :393)
    assert vals["EDGES"][0] == ["1", "0", "0"]
    # ---- HomotopyClassPlanner: 3 candidates optimised in one batch, costs with the selection scales, selectBestTeb
    hp = abi.default_params()
    hp.include_dynamic_obstacles = 0
    hob = np.zeros(3, abi.OBST_DTYPE)
    hob["x"], hob["y"], hob["radius"] = [0.0, -1.5, 2.0], [0.1, -0.4, 0.6], [0.0, 0.0, 0.2]
    hob["type"] = [0, 0, 1]
    plans = []
    for amp in (1.2, -1.0, 0.0):     # candidate order in the container: two seeded, then the initial plan
        s = np.linspace(0, 1, 21)
        plans.append(np.stack([-4 + 8 * s, amp * np.sin(np.pi * s), np.zeros(21)], axis=1))
    args = abi.make_args(5, 4, True, hp.selection_obst_cost_scale, hp.selection_viapoint_cost_scale, False)
    costs = []
    assert vals["HCP_NUM"][0][0] == "3" and vals["HCP_DUP_REJECTED"][0][0] == "1"
    hp2d = abi.default_params()
    hp2d.include_dynamic_obstacles = 0
    for k, plan in enumerate(plans):        # equivalence classes: H-signatures of the bands as initialised from the plans
        r0 = _init_from_plan(plan, hp.max_vel_x, hp.max_vel_theta)
        href = oracle.h_signature(hp2d, r0, len(r0), hob)
        hk = [v for v in vals["HCP_H"] if int(v[0]) == k][0]
        assert abs(complex(float(hk[1]), float(hk[2])) - href) <= 1e-9 * abs(href)
    dup = np.stack([-4 + 8 * np.linspace(0, 1, 21), 0.9 * np.sin(np.pi * np.linspace(0, 1, 21)), np.zeros(21)], axis=1)
    rd = _init_from_plan(dup, hp.max_vel_x, hp.max_vel_theta)
    r1 = _init_from_plan(plans[0], hp.max_vel_x, hp.max_vel_theta)
    hd, h1 = oracle.h_signature(hp2d, rd, len(rd), hob), oracle.h_signature(hp2d, r1, len(r1), hob)
    assert abs(hd.real - h1.real) <= hp.h_signature_threshold and abs(hd.imag - h1.imag) <= hp.h_signature_threshold
    assert vals["HCP2_NUM"][0][0] == "3"
    for k, plan in enumerate(plans):
        r0 = _init_from_plan(plan, hp.max_vel_x, hp.max_vel_theta)
        ref_k, cost_k, _ = oracle.optimize_band(hp, r0, len(r0), hob, args=args, jac_mode=oracle.JAC_ANALYTIC, n_cap=512)
        got_k = bands[f"HCP{k}"]
        assert len(got_k) == len(ref_k) and np.abs(got_k - ref_k).max() < 1e-6
        gcost = float([v for v in vals["HCP_COST"] if int(v[0]) == k][0][1])
        assert abs(gcost - cost_k) <= 1e-6 * max(abs(cost_k), 1.0)
        costs.append(cost_k)
    from teb_local_planner_b200 import distributed as D
    assert int(vals["HCP_BEST"][0][0]) == D.select_best(costs, -1, 2, hp.selection_cost_hysteresis, hp.selection_prefer_initial_plan)
    assert vals["HCP2_OK"][0][0] == "1" and int(vals["HCP2_BEST"][0][0]) in (0, 1, 2)
    # ---- nothing seeded: key-point graph exploration -> batched optimisation -> selection
    from oracle import hcp_explore as X
    ap = abi.default_params()
    ap.include_dynamic_obstacles = 0
    arows = np.zeros(3, abi.OBST_DTYPE)
    arows["x"], arows["y"], arows["radius"] = [-1.5, 0.5, 2.0], [0.3, -0.4, 0.5], [0, 0.3, 0]
    arows["type"] = [abi.TEB_OBST_POINT, abi.TEB_OBST_CIRCULAR, abi.TEB_OBST_POINT]
    ex = X.Explorer(ap, {"max_number_classes": 4, "obstacle_heading_threshold": 0.45}, oracle, arows,
                    [X.Obst("point", (-1.5, 0.3)), X.Obst("circle", (0.5, -0.4), 0.3), X.Obst("point", (2.0, 0.5))])
    ex.lr_key_point_graph([-4, 0, 0.1], [4, 0.2, -0.2], ap.min_obstacle_dist)
    assert vals["AUTO_OK"][0][0] == "1" and int(vals["AUTO_NUM"][0][0]) == len(ex.tebs) and len(ex.tebs) >= 3
    aargs = abi.make_args(5, 4, True, ap.selection_obst_cost_scale, ap.selection_viapoint_cost_scale, False)
    acosts = []
    for k, r0 in enumerate(ex.tebs):
        ref_k, cost_k, _ = oracle.optimize_band(ap, r0, len(r0), arows, args=aargs, jac_mode=oracle.JAC_ANALYTIC, n_cap=512)
        got_k = bands[f"AUTO{k}"]
        assert len(got_k) == len(ref_k) and np.abs(got_k - ref_k).max() < 1e-6, k
        acosts.append(cost_k)
    assert int(vals["AUTO_BEST"][0][0]) == int(np.argmin(acosts))
    # ---- polygon footprint among a line, a moving pill and a polygon obstacle
    from teb_local_planner_b200 import scenes
    sp = abi.default_params()
    scenes.set_polygon_footprint(sp, ((-0.25, -0.2), (0.35, -0.2), (0.35, 0.2), (-0.25, 0.2)))
    pool = np.array([[-1.0, 0.6], [0.5, 1.4], [1.0, -1.2], [2.0, -0.5], [-0.3, -0.6], [0.4, -0.7], [0.2, -0.1]])
    sob = np.zeros(3, abi.OBST_DTYPE)
    sob["type"] = [abi.TEB_OBST_LINE, abi.TEB_OBST_PILL, abi.TEB_OBST_POLYGON]
    sob["vertex_begin"], sob["vertex_count"] = [0, 2, 4], [2, 2, 3]
    sob["radius"] = [0.0, 0.15, 0.0]
    sob["vx"], sob["vy"], sob["dynamic"] = [0, -0.1, 0], [0, 0.1, 0], [0, 1, 0]
    ctr = [scenes.polygon_centroid(pool[b:b + c]) for b, c in zip(sob["vertex_begin"], sob["vertex_count"])]
    sob["x"], sob["y"] = [c[0] for c in ctr], [c[1] for c in ctr]
    rec0 = oracle.init_trajectory([-4, 0, 0], [4, 0, 0], 0.0, sp.max_vel_x, sp.min_samples)
    sref, _, _ = oracle.optimize_band(sp, rec0, len(rec0), sob, args=abi.make_args(5, 4, False), jac_mode=oracle.JAC_ANALYTIC,
                                      n_cap=512, obst_vertices=pool)
    sgot = bands["SHAPES"]
    assert vals["SHAPES_OK"][0][0] == "1" and len(sgot) == len(sref)
    assert np.abs(sgot - sref).max() < 1e-6


@pytest.mark.gpu
def test_dropin_exploration_matches_sequential_restatement(exe, oracle):
    """HomotopyClassPlanner::exploreEquivalenceClassesAndInitTebs with both graph searches (graph_search.cpp) and both
    signature kinds: the chunked, batched C++ exploration proposes exactly the bands of the sequential restatement in
    oracle/hcp_explore.py (same paths, same order, same initial trajectories)"""
    from oracle import hcp_explore as X
    out = subprocess.run([exe, "explore"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "RESULT PASS" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
    vals, bands = _parse(out.stdout)
    for variant in range(4):
        p = abi.default_params()
        p.include_dynamic_obstacles = 1 if variant & 2 else 0
        rows = np.zeros(4, abi.OBST_DTYPE)
        rows["x"], rows["y"] = [-1.5, 0.5, 2.0, -2.75], [0.3, -0.4, 0.5, -1.15]
        rows["radius"] = [0, 0.3, 0, 0]
        rows["type"] = [abi.TEB_OBST_POINT, abi.TEB_OBST_CIRCULAR, abi.TEB_OBST_POINT, abi.TEB_OBST_LINE]
        if variant & 2:
            rows["vx"][2], rows["vy"][2], rows["dynamic"][2] = -0.1, 0.05, 1
        obstacles = [X.Obst("point", (-1.5, 0.3)), X.Obst("circle", (0.5, -0.4), 0.3), X.Obst("point", (2.0, 0.5)),
                     X.Obst("line", (-2.75, -1.15), vertices=[(-3.0, -1.5), (-2.5, -0.8)])]
        hcp = {"max_number_classes": 6, "obstacle_heading_threshold": 0.45, "roadmap_graph_area_width": 6.0,
               "roadmap_graph_area_length_scale": 1.0, "roadmap_graph_no_samples": 15}
        ex = X.Explorer(p, hcp, oracle, rows, obstacles)
        for cycle in range(2):
            ex.classes, ex.tebs = [], []
            if variant & 1:
                ex.lr_key_point_graph([-4, 0, 0.1], [4, 0.2, -0.2], p.min_obstacle_dist)
            else:
                ex.prob_roadmap_graph([-4, 0, 0.1], [4, 0.2, -0.2], p.min_obstacle_dist)
            num = int(vals[f"EXPLORE{variant}_{cycle}_NUM"][0][0])
            assert num == len(ex.tebs) and num >= 2, (variant, cycle, num, len(ex.tebs))
            for k, ref in enumerate(ex.tebs):
                got = bands[f"EXPLORE{variant}_{cycle}_{k}"]
                assert got.shape == ref.shape and np.abs(got - ref).max() < 1e-12, (variant, cycle, k)
