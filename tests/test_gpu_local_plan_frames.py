"""Every robot's local plan from a global plan in its own frame on the device (tebgpu_local_plan_tf / _tf_device,
k_local_plan<true>), held to tests/frame_cases.py's restatement: with no transform it is the identity path bit for bit;
with the identity transform every decision, count and position is the identity path's and the yaws are within 1e-15; on
fleets with per-robot planar and tilted transforms every decision, count, position and via-point is the restatement's
and the yaws are within 1e-12 (the device's trig). Also host bits == device bits, batch-position invariance, argument
errors, and a 20-cycle fleet loop on one stream with each robot's map -> odom drifting."""
import ctypes as C
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import frame_cases as fc
from tests import local_plan_cases as lp
from tests import test_gpu_local_plan as base

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
IDENTITY = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])


@pytest.fixture(scope="module", params=[True, False], ids=["overwrite", "stored_yaw"])
def gpu(request):
    g = base._ctx(request.param)
    g.overwrite = request.param
    yield g
    g.close()


def _frames(ptr, c2p, p2c):
    return abi.make_frame_args(costmap_to_plan=ptr(c2p), plan_to_costmap=ptr(p2c))


def run_host_tf(g, f, a, P_cap, V_cap, c2p, p2c, null_struct=False):
    ins, outs = base._inputs(f), base._outs(f.B, P_cap, V_cap, True)
    la = base._args(f, a, P_cap, V_cap, abi.ptr, ins, outs)
    fr = None if null_struct else _frames(abi.ptr, c2p, p2c)
    rc = g.lib.tebgpu_local_plan_tf(g.ctx, C.byref(base._batch(f, abi.ptr, f.sid)), C.byref(la),
                                    None if fr is None else C.byref(fr))
    assert rc == 0, g.lib.tebgpu_last_error_string(g.ctx)
    outs["plan_begin"] = ins["begin"]
    return outs


def run_device_tf(g, f, a, P_cap, V_cap, c2p, p2c):
    ins_h, outs_h = base._inputs(f), base._outs(f.B, P_cap, V_cap, True)
    ins = {k: base._dev(v) for k, v in ins_h.items()}
    outs = {k: base._dev(v) for k, v in outs_h.items()}
    ptr = lambda t: None if t is None else t.data_ptr()
    la = base._args(f, a, P_cap, V_cap, ptr, ins, outs)
    tc, tp = base._dev(c2p), base._dev(p2c)
    g.local_plan_device(base._batch(f, ptr, base._dev(f.sid)), la, stream=torch.cuda.current_stream().cuda_stream,
                        frames=_frames(ptr, tc, tp))
    torch.cuda.synchronize()
    back = {k: None if v is None else v.cpu().numpy().view(outs_h[k].dtype).reshape(outs_h[k].shape)
            for k, v in outs.items()}
    back["plan_begin"] = ins["begin"].cpu().numpy().view(np.int32)
    return back


def both_tf(g, f, a, P_cap, V_cap, c2p, p2c):
    h = run_host_tf(g, f, a, P_cap, V_cap, c2p, p2c)
    d = run_device_tf(g, f, a, P_cap, V_cap, c2p, p2c)
    for k in h:
        if h[k] is not None:
            assert base._bytes(h[k]) == base._bytes(d[k]), k                     # host bits == device bits
    return d


def assert_close_to(out, want, tol, label=""):
    """decisions, counts, positions and via-points bit equal; every stored yaw within tol (mod 2 pi)"""
    for b, w in enumerate(want):
        lab = (label, b, w.result)
        assert out["result"][b] == w.result and out["plan_begin"][b] == w.plan_begin, lab
        if w.result != lp.EMPTY:
            assert out["goal_idx"][b] == w.goal_idx and tuple(out["needed"][b]) == w.needed, lab
        k = len(w.plan)
        assert out["plan_count"][b] == k, lab
        if k:
            got, ref = out["plan"][b, :k], np.array(w.plan)
            assert base._bytes(got[:, :2]) == base._bytes(ref[:, :2]), lab
            for r in range(k):
                assert base._ang(got[r, 2], ref[r, 2]) <= tol, (lab, r, got[r, 2], ref[r, 2])
        assert (out["plan"][b, k:].view(np.uint8) == base.SENTINEL).all(), lab
        nv = 0 if w.via is None else len(w.via)
        if w.via is not None:
            assert out["via_count"][b] == nv, lab
            if nv:
                assert base._bytes(out["via"][b, :nv]) == base._bytes(np.array(w.via)), lab
        assert (out["via"][b, nv:].view(np.uint8) == base.SENTINEL).all(), lab


def test_null_frames_are_the_identity_path(gpu):
    d = scenes.global_plans(128, 512, S=4, seed=31)
    f = base.Fleet.of(d, inf=np.arange(128) % 12, since=np.linspace(0, 20, 128))
    a = base._args_for(gpu, viapoint_sep=0.25)
    ref = base.run_host(gpu, f, a, 513, 64)
    for null_struct in (True, False):
        out = run_host_tf(gpu, f, a, 513, 64, None, None, null_struct)
        for k in ref:
            assert base._bytes(ref[k]) == base._bytes(out[k]), k
    out = run_device_tf(gpu, f, a, 513, 64, None, None)
    for k in ref:
        assert base._bytes(ref[k]) == base._bytes(out[k]), k


@pytest.mark.parametrize("j", range(len(base.ARGSETS)))
def test_explicit_identity(gpu, j):
    d = scenes.global_plans(128, 512, S=4, seed=40 + j)
    f = base.Fleet.of(d)
    a = base._args_for(gpu, **base.ARGSETS[j])
    ref = base.run_host(gpu, f, a, 513, 64)
    ident = np.tile(IDENTITY, (128, 1))
    out = both_tf(gpu, f, a, 513, 64, ident, ident)
    for k in ("plan_begin", "plan_count", "goal_idx", "result", "needed", "via_count", "via"):
        assert base._bytes(ref[k]) == base._bytes(out[k]), k
    assert base._bytes(ref["plan"][..., :2]) == base._bytes(out["plan"][..., :2])
    for b in range(128):
        for r in range(ref["plan_count"][b]):
            assert base._ang(ref["plan"][b, r, 2], out["plan"][b, r, 2]) <= 1e-15, (b, r)


def _inverse(t):
    """the inverse of a transform, in float64 (only to build test fleets; the device never inverts)"""
    q = np.array(t[3:7])
    m = np.array(fc.tf2_basis(list(q))).reshape(3, 3)
    ti = -m.T @ np.array(t[:3])
    return np.concatenate([ti, [-q[0], -q[1], -q[2], q[3]]])


def framed_fleet(B, G_cap, S, seed, tilted):
    """scenes.global_plans moved into per-robot plan frames: rows_plan = doTransform(row, costmap_to_plan) with
    plan_to_costmap drawn at random (planar or, for odd robots, tilted) and costmap_to_plan its inverse"""
    d = scenes.global_plans(B, G_cap, S=S, seed=seed)
    rng = np.random.default_rng(seed + 1000)
    p2c = np.array([fc.random_transform(rng, tilted=tilted and b % 2 == 1) for b in range(B)])
    c2p = np.array([_inverse(t) for t in p2c])
    gp = d["global_plan"].copy()
    for b in range(B):
        for k in range(int(d["plan_end"][b])):
            gp[b, k] = fc.transform_row(list(c2p[b]), gp[b, k])[0]
    d["global_plan"] = gp
    return d, c2p, p2c


def _margins_ok(f, a, c2p, p2c, want):
    """no band within 1e-9 of the goal-reached yaw test's tie or of getYaw's gimbal threshold"""
    for b, w in enumerate(want):
        if w.result == lp.EMPTY:
            continue
        g = f.gp[b, int(w.plan_begin):int(f.end[b])]
        (_, _, yaw), q = fc.transform_row(list(p2c[b]), g[-1])
        if abs(abs(lp.normalize_theta(yaw - f.robot[b, 2])) - a.yaw_goal_tolerance) < 1e-9:
            return False
        if abs(abs(fc.yaw_sarg(q)) - fc.GIMBAL) < 1e-9:
            return False
    return True


def expect_tf(f, a, c2p, p2c, P_cap, V_cap):
    out = []
    for b in range(f.B):
        s = f.sid[b]
        out.append(fc.restate_tf(f.gp[b], int(f.begin[b]), int(f.end[b]), f.robot[b], f.vel[b],
                                 tuple(int(v) for v in f.grid[s]), float(f.origin[s, 2]), a, c2p[b], p2c[b],
                                 None, None if f.inf is None else int(f.inf[b]),
                                 None if f.since is None else float(f.since[b]), P_cap, V_cap))
    return out


@pytest.mark.parametrize("tilted", [False, True], ids=["planar", "tilted"])
@pytest.mark.parametrize("j", range(len(base.ARGSETS)))
def test_random_fleets_match_the_restatement(gpu, tilted, j):
    d, c2p, p2c = framed_fleet(128, 512, 4, 50 + j, tilted)
    f = base.Fleet.of(d)
    a = base._args_for(gpu, **base.ARGSETS[j])
    want = expect_tf(f, a, c2p, p2c, 513, 64)
    assert _margins_ok(f, a, c2p, p2c, want)
    out = both_tf(gpu, f, a, 513, 64, c2p, p2c)
    assert_close_to(out, want, 1e-12, (tilted, j))
    res = np.array([w.result for w in want])
    assert (res == lp.PLANNED).any()


def test_goal_reached_under_tilted_transforms(gpu):
    """robots standing at their transformed global goal: the goal-reached test reads getYaw of a tilted orientation"""
    d, c2p, p2c = framed_fleet(64, 512, 4, 60, True)
    at_goal = np.arange(64) % 4 < 2                      # b % 4 == 1: tilted, b % 4 == 0: planar
    for b in np.flatnonzero(at_goal):
        (gx, gy, gyaw), _ = fc.transform_row(list(p2c[b]), d["global_plan"][b, int(d["plan_end"][b]) - 1])
        d["robot"][b] = (gx + 0.01, gy - 0.01, lp.normalize_theta(gyaw + 0.05))
        d["robot_vel"][b] = 0.0
    f = base.Fleet.of(d)
    a = base._args_for(gpu)
    want = expect_tf(f, a, c2p, p2c, 513, 64)
    assert _margins_ok(f, a, c2p, p2c, want)
    out = both_tf(gpu, f, a, 513, 64, c2p, p2c)
    assert_close_to(out, want, 1e-12)
    res = np.array([w.result for w in want])
    tilted = np.arange(64) % 2 == 1
    assert (res[at_goal & tilted] == lp.GOAL_REACHED).sum() >= 12
    assert (res[at_goal & ~tilted] == lp.GOAL_REACHED).sum() >= 12
    assert (res[~at_goal] == lp.PLANNED).any()


def test_results_do_not_depend_on_the_band_position(gpu):
    d, c2p, p2c = framed_fleet(96, 1024, 4, 5, True)
    f = base.Fleet.of(d, inf=np.arange(96) % 12, since=np.linspace(0, 20, 96))
    a = base._args_for(gpu, viapoint_sep=0.25)
    ref = run_device_tf(gpu, f, a, 1025, 64, c2p, p2c)
    perm = np.random.default_rng(2).permutation(96)
    out = run_device_tf(gpu, f.subset(perm), a, 1025, 64, c2p[perm], p2c[perm])
    for k in ref:
        assert base._bytes(ref[k][perm]) == base._bytes(out[k]), k
    one = run_host_tf(gpu, f.subset([perm[0]]), a, 1025, 64, c2p[perm[:1]], p2c[perm[:1]])
    for k in ref:
        assert base._bytes(ref[k][perm[:1]]) == base._bytes(one[k]), k


def test_only_one_plan_transform_is_an_argument_error(gpu):
    d = scenes.global_plans(8, 64, S=2, seed=1)
    f = base.Fleet.of(d)
    a = base._args_for(gpu)
    base.run_host(gpu, f, a, 65, 8)
    grid = gpu.last_local_plan_grid()
    ident = np.tile(IDENTITY, (8, 1))
    for c2p, p2c in ((ident, None), (None, ident)):
        for host in (True, False):
            ins, outs = base._inputs(f), base._outs(f.B, 65, 8, True)
            la = base._args(f, a, 65, 8, abi.ptr, ins, outs)
            fr = _frames(abi.ptr, c2p, p2c)
            bs = base._batch(f, abi.ptr, f.sid)
            rc = gpu.lib.tebgpu_local_plan_tf(gpu.ctx, C.byref(bs), C.byref(la), C.byref(fr)) if host else \
                gpu.lib.tebgpu_local_plan_tf_device(gpu.ctx, C.byref(bs), C.byref(la), C.byref(fr), None)
            assert rc == abi.TEBGPU_ERR_INVALID_ARG
            assert (outs["result"] == 77).all()
    assert gpu.last_local_plan_grid() == grid


# ---- the fleet loop with drifting map -> odom
def _drift(B, k):
    """each robot's map -> odom pose at cycle k: (costmap_to_plan, plan_to_costmap) [B][7] each"""
    c2p, p2c = np.zeros((B, 7)), np.zeros((B, 7))
    for b in range(B):
        c2p[b], p2c[b] = abi.transform_from_se2(0.3 * b - 2.0 + 0.01 * k, 1.0 - 0.1 * b - 0.004 * k,
                                                0.2 * b - 2.0 + 0.003 * k)
    return c2p, p2c


def _custom(B, PV):
    """per scene, in the map frame: a point, a circle, a line and a square with a repeated closing vertex"""
    rows = np.zeros((B, 4), abi.OBST_DTYPE)
    verts = np.zeros((B, PV, 2))
    rng = np.random.default_rng(77)
    for s in range(B):
        cx, cy = rng.uniform(-1, 1, 2)
        rows[s]["type"] = [fc.TEB_OBST_POINT, fc.TEB_OBST_CIRCULAR, fc.TEB_OBST_LINE, fc.TEB_OBST_POLYGON]
        rows[s]["x"], rows[s]["y"] = [cx, cx + 0.5, 0, 0], [cy, cy - 0.5, 0, 0]
        rows[s]["radius"] = [0, 0.1, 0, 0]
        rows[s]["vertex_begin"], rows[s]["vertex_count"] = [0, 0, 0, 2], [0, 0, 2, 5]
        verts[s, :2] = [(cx - 0.3, cy + 0.8), (cx + 0.3, cy + 0.8)]
        verts[s, 2:7] = [(cx - 1, cy - 1), (cx - 0.8, cy - 1), (cx - 0.8, cy - 0.8), (cx - 1, cy - 0.8), (cx - 1, cy - 1)]
    return rows, verts


def _fleet_loop(restated, cycles=20, B=16, P_cap=160, M_cap=2048, n_cap=96, Lb=10, PV=8, dev_trace=None):
    """restated=False: costmap_tf -> local_plan_tf -> backup modes -> plan -> check -> finish on one stream. True: the
    same loop with the custom obstacles moved on the host by the restatement (fed through the verbatim path) and the
    local plans restated on the host (fed to plan as rows); a restated yaw within 1e-12 of the device's at the same
    cycle is replaced by the device's bits, so both loops see the same inputs wherever the bars hold."""
    d = scenes.global_plans(B, 1024, S=B, seed=21)
    c0, _ = _drift(B, 0)
    gp_odom = d["global_plan"]
    gp = gp_odom.copy()
    for b in range(B):                                   # the plans in the map frame of cycle 0
        for k in range(int(d["plan_end"][b])):
            gp[b, k] = fc.transform_row(list(c0[b]), gp_odom[b, k])[0]
    r = scenes.costmap_raster(B, 60, 60, 0.05, 0.03, seed=22)
    r["origin"][:, 0] = d["robot"][:, 0] - 1.5
    r["origin"][:, 1] = d["robot"][:, 1] - 1.5
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 0
    p.max_vel_trans = p.max_vel_x
    p.global_plan_overwrite_orientation = 1
    g = T.TebGpu(B, n_cap, B, M_cap, 0, max_obst_vertices=PV)
    g.set_params(p)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=DEV)
    f64, i32 = torch.float64, torch.int32
    cost, grid, origin = t(r["cost"]), t(r["grid"]), t(r["origin"])
    robot = t(d["robot"].copy())
    rows_map, verts_map = _custom(B, PV)
    custom, ccount = t(rows_map.view(np.uint8)), t(np.full(B, 4, np.int32))
    cverts, overts = t(verts_map), z((B, PV, 2), f64)
    obst, ocount = z(B * M_cap * 64, torch.uint8), z(B, i32)
    gpd, begin, end = t(gp), t(d["plan_begin"].copy()), t(d["plan_end"])
    plan, pcount, result = z((B, P_cap, 3), f64), z(B, i32), z(B, i32)
    gidx, needed = z(B, i32), z((B, 2), i32)
    state = {k: t(v) for k, v in abi.make_cycle_state(B, Lb).items()}
    vel, since = z((B, 3), f64), z(B, f64)
    poses, n, sid = z((B, n_cap, 4), f64), z(B, i32), t(np.arange(B, dtype=np.int32))
    vs = np.zeros((B, 4))
    vs[:, 3] = 1.0
    vstart, vgoal = t(vs), t(vs)
    costo, chi2, status, iters = z(B, f64), z(B, f64), z(B, i32), z(B, i32)
    cmd, path, feas, qc = z((B, 4), f64), z(B, i32), z(B, i32), z(B, i32)
    cmd_vel, outcome, osc = z((B, 3), f64), z(B, i32), z(B, i32)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, B, M_cap, 0, PV
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count, bs.obst_vertices = obst.data_ptr(), ocount.data_ptr(), overts.data_ptr()
    bs.vel_start, bs.vel_goal, bs.prefer_rotdir = vstart.data_ptr(), vgoal.data_ptr(), state["prefer_rotdir"].data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = costo.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = B, r["cost"].shape[1], M_cap, 4, 1
    ca.behind_robot_dist = 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.custom, ca.custom_count = custom.data_ptr(), ccount.data_ptr()
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    scal = dict(max_lookahead_dist=2.0)
    la = abi.make_local_plan_args(1024, P_cap, 0, **scal, global_plan=gpd.data_ptr(),
                                  plan_begin=begin.data_ptr(), plan_end=end.data_ptr(), robot=robot.data_ptr(),
                                  robot_vel=vel.data_ptr(), grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  infeasible_count=state["infeasible_count"].data_ptr(), since_infeasible=since.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), goal_idx=gidx.data_ptr(),
                                  result=result.data_ptr(), needed=needed.data_ptr())
    a = lp.Args(overwrite_orientation=True, **scal)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    fa = abi.make_feasibility_args(0.1, max_queries=512, collision_distance=0.05, feasible=feas.data_ptr(),
                                   query_count=qc.data_ptr())
    sc = dict(buffer_length=Lb, oscillation_recovery_min_duration=2.0)
    dt, now = 0.2, 1000.0
    s = torch.cuda.Stream()
    trace = []
    for k in range(cycles):
        c2p, p2c = _drift(B, k)
        tc, tp = t(c2p), t(p2c)
        cy = abi.make_cycle_args(now, L_cap=Lb, **sc, local_plan_result=result.data_ptr(), robot_vel=vel.data_ptr(),
                                 cmd=cmd.data_ptr(), feasible=feas.data_ptr(), cmd_vel=cmd_vel.data_ptr(),
                                 outcome=outcome.data_ptr(), oscillating=osc.data_ptr(),
                                 **{kk: state[kk].data_ptr() for kk in abi.CYCLE_STATE})
        with torch.cuda.stream(s):
            since.copy_(now - state["last_infeasible"])
            if restated:
                s.synchronize()
                moved, ov = np.zeros_like(rows_map), np.zeros((B, PV, 2))
                for sc_i in range(B):
                    moved[sc_i] = fc.move_custom(rows_map[sc_i], verts_map[sc_i], list(p2c[sc_i]), ov[sc_i])
                custom_h = t(moved.view(np.uint8))
                overts.copy_(t(ov))
                ca.custom = custom_h.data_ptr()
                g.costmap_obstacles_device(ca, stream=s.cuda_stream)
                rb, bg = robot.cpu().numpy(), begin.cpu().numpy()
                inf, sn = state["infeasible_count"].cpu().numpy(), since.cpu().numpy()
                hp = np.zeros((B, P_cap, 3))
                hres, hcnt, hbeg = np.zeros(B, np.int32), np.zeros(B, np.int32), bg.copy()
                for b in range(B):
                    w = fc.restate_tf(gp[b], int(bg[b]), int(d["plan_end"][b]), rb[b], vel.cpu().numpy()[b],
                                      (60, 60), 0.05, a, c2p[b], p2c[b], 0, int(inf[b]), float(sn[b]), P_cap, 0)
                    hres[b], hcnt[b], hbeg[b] = w.result, len(w.plan), w.plan_begin
                    if w.plan:
                        hp[b, :len(w.plan)] = w.plan
                        dc = dev_trace[k]["pcount"]
                        dv = dev_trace[k]["plan"][int(dc[:b].sum()):]
                        for rr in range(len(w.plan)):
                            assert base._ang(hp[b, rr, 2], dv[rr, 2]) <= 1e-12, (k, b, rr)
                            hp[b, rr, 2] = dv[rr, 2]
                plan.copy_(t(hp))
                pcount.copy_(t(hcnt))
                result.copy_(t(hres))
                begin.copy_(t(hbeg))
            else:
                fr = abi.make_frame_args(custom_to_costmap=tp.data_ptr(), custom_vertices=cverts.data_ptr(),
                                         obst_vertices=overts.data_ptr(), PV_cap=PV)
                g.costmap_obstacles_device(ca, stream=s.cuda_stream, frames=fr)
                g.local_plan_device(bs, la, stream=s.cuda_stream,
                                    frames=abi.make_frame_args(costmap_to_plan=tc.data_ptr(), plan_to_costmap=tp.data_ptr()))
            g.backup_modes_device(bs, cy, stream=s.cuda_stream)
            g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, path=path,
                          stream=s.cuda_stream)
            g.check_feasible_device(bs, fa, stream=s.cuda_stream)
            g.finish_cycle_device(bs, cy, stream=s.cuda_stream)
            th = robot[:, 2]
            robot[:, 0] += (cmd_vel[:, 0] * torch.cos(th) - cmd_vel[:, 1] * torch.sin(th)) * dt
            robot[:, 1] += (cmd_vel[:, 0] * torch.sin(th) + cmd_vel[:, 1] * torch.cos(th)) * dt
            robot[:, 2] += cmd_vel[:, 2] * dt
            vel.copy_(cmd_vel)
        s.synchronize()
        rec = dict(obst=obst, ocount=ocount, overts=overts, plan=plan, pcount=pcount, result=result, begin=begin,
                   n=n, poses=poses, status=status, path=path, cmd=cmd, cmd_vel=cmd_vel, outcome=outcome,
                   oscillating=osc, feasible=feas, **state)
        rec = {kk: v.cpu().numpy().copy() for kk, v in rec.items()}
        rec["plan"] = np.concatenate([rec["plan"][b, :rec["pcount"][b]] for b in range(B)])   # the rows written
        trace.append(rec)
        now += dt
    g.close()
    return trace


def test_fleet_loop_with_drifting_frames_matches_the_host_transformed_loop():
    dev = _fleet_loop(False)
    ref = _fleet_loop(True, dev_trace=dev)
    for k, (x, y) in enumerate(zip(dev, ref)):
        for key in x:
            assert x[key].tobytes() == y[key].tobytes(), (k, key)
    res = np.concatenate([c["result"] for c in dev])
    assert (res == lp.PLANNED).sum() >= len(res) // 2
    assert (np.concatenate([c["ocount"] for c in dev]) > 4).all()
