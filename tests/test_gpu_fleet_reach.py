"""The footprints' neighbour rule on the device (TebFleetShapes.select = TEB_FLEET_SELECT_FOOTPRINTS: the FleetFootprints
policy of k_fleet_obstacles and k_fleet_obstacles_grid), held to tests/fleet_reach_cases.py: the hand cases bit for bit;
random fleets of mixed kinds up to 8192 robots under each of the five footprint models, every count, status, type, order
and vertex range the restatement's and positions within 1e-12, except robots with a pair whose restated gap lies within
1e-9 of range or of the next gap (counted and reported); the grid and all pairs write the same bytes up to 32768 robots;
uneven shards through the table equal one array call; select = 0 writes the centre rule's bytes."""
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from teb_local_planner_b200 import distributed as D
from tests import fleet_reach_cases as frc
from tests import fleet_shape_cases as fsc
from tests import fleet_table_cases as ftc
from tests.test_fleet_reach_cases import LONG, SMALL, params
from tests.test_gpu_fleet_obstacles import IDENTITY, _raster, _straight_plans
from tests.test_gpu_fleet_shapes import CLOSE, KINDS, PV_CAP, assert_matches, dev, mixed_fleet, outputs, t

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
MAX_R = 32768
FOOT = abi.TEB_FLEET_SELECT_FOOTPRINTS
MODELS = ["point", "circular", "two_circles", "line", "polygon"]


@pytest.fixture(scope="module")
def g():
    ctx = T.TebGpu(MAX_R, 8, MAX_R + 64, 64)
    yield ctx
    ctx.close()


def run(g, f, rng, max_rows, select=FOOT, search=abi.TEBGPU_FLEET_SEARCH_AUTO):
    d = dev(f)
    R, C_cap = f["custom"].shape
    fa = abi.make_fleet_args(R, R, C_cap, max_rows, rng, pose=d["pose"], last_cmd=d["cmd"], world=d["world"],
                             own_count=d["own"], custom=d["custom"], custom_count=d["cc"], needed=d["need"],
                             status=d["st"])
    sh = abi.make_fleet_shapes(KINDS, PV_CAP, select, kind=d["kind"], own_vertex_count=d["ownv"], custom_vertices=d["cv"])
    g.set_fleet_search(search)
    g.fleet_obstacles_shaped_device(fa, sh)
    torch.cuda.synchronize()
    g.set_fleet_search(abi.TEBGPU_FLEET_SEARCH_AUTO)
    return outputs(d, f)


def restated(prm, f, rng, max_rows, gaps=None):
    return frc.restate(prm, f["pose"], f["last_cmd"], KINDS, f["kind"], rng, max_rows, f["custom"], f["cv"],
                       f["own_count"], own_vertex_count=f["own_v"], world=f["world"], gaps=gaps)


def boundary_robots(prm, f, rng, gaps, tol=1e-9):
    """robots with a pair whose restated gap lies within tol of rng, or within tol of the next gap of its list"""
    out = {r for r, _ in frc.near(gaps, rng, tol)}
    pose, kind = f["pose"], f["kind"]
    R = len(pose)
    for r in range(R):
        lo = frc.neighbours(prm, KINDS, pose[:, :2], pose[:, 2], f["world"], np.ones(R, bool), kind, r, pose[r],
                            max(rng - tol, 0.0))[0]
        hi = frc.neighbours(prm, KINDS, pose[:, :2], pose[:, 2], f["world"], np.ones(R, bool), kind, r, pose[r],
                            rng + tol)[0]
        if len(lo) != len(hi):
            out.add(r)
    return out


def test_hand_cases_match_the_restatement(g):
    cases = [("polygon", [[0.0, 0.0, 0.0], [4.5, 0.0, 0.0]], [LONG], [0, 0], 3.0, 8),
             ("polygon", [[0.0, 0.0, math.pi / 2], [0.0, 4.5, math.pi / 2]], [LONG], [0, 0], 3.0, 8),
             ("circular", [[0.0, 0.0, 0.0], [2.0, 0.0, 0.0], [0.0, 2.5, math.pi / 2]],
              [[(fsc.CIRCULAR, [[0.0, 0.0]], 0.2)], LONG], [0, 0, 1], 3.0, 1),
             ("point", [[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, -0.4, 0.0]],
              [[(fsc.POINT, [[0.0, 0.0]])], LONG, SMALL], [0, 0, 1, 2], 3.0, 2),
             ("polygon", [[0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [4.0, 0.0, 0.0], [100.0, 0.0, 1.0]], [LONG], [0] * 4, 0.0, 8),
             ("polygon", [[0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [4.0, 0.0, 0.0], [100.0, 0.0, 1.0]], [LONG], [0] * 4,
              math.inf, 8)]
    for model, pose, kinds, kind, rng, max_rows in cases:
        prm = params(model, radius=0.2)
        g.set_params(prm)
        pose = np.asarray(pose)
        R = len(pose)
        custom = np.zeros((R, 16), abi.OBST_DTYPE)
        got = g.fleet_obstacles_shaped(kinds, kind, pose, np.zeros((R, 3)), custom, rng, max_rows,
                                       custom_vertices=np.zeros((R, 64, 2)), select=FOOT)
        want = frc.restate(prm, pose, np.zeros((R, 3)), kinds, kind, rng, max_rows, custom, np.zeros((R, 64, 2)))
        for a, b in zip(got, want):
            assert a.tobytes() == b.tobytes(), (model, pose.tolist(), rng)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("R,clustered", [(1, True), (700, True), (3000, False), (8192, False)])
def test_random_mixed_fleets_match_the_restatement(g, model, R, clustered):
    prm = params(model, radius=0.3)
    g.set_params(prm)
    f = mixed_fleet(R, 24, 40 + R, clustered)
    rng, max_rows = 1.5, 6
    got = run(g, f, rng, max_rows)
    gaps = {}
    want = restated(prm, f, rng, max_rows, gaps)
    # the exceptions: robots with two restated gaps within 1e-9 (the device may order them the other way) or a gap within
    # 1e-9 of range (searched only when a count differs); every other robot is held to assert_matches
    allowed = {r for r, _ in frc.near(gaps, rng)}
    differ = set(np.nonzero((got[1] != want[1]) | (got[2] != want[2]) | (got[3] != want[3]))[0].tolist())
    if differ - allowed:
        allowed |= boundary_robots(prm, f, rng, gaps)
    assert differ <= allowed, sorted(differ - allowed)[:10]
    keep = np.ones(R, bool)
    keep[sorted(allowed)] = False
    sub = lambda out: tuple(x[keep] for x in out)
    assert_matches(sub(got), sub(want), {k: (v[keep] if k in ("custom", "own_count", "own_v", "cv") else v)
                                         for k, v in f.items()})
    print(f"{model} R={R}: {len(differ)} robots differ, {len(allowed)} robots excepted (a gap within 1e-9 of a "
          f"decision), {int(keep.sum())} compared")


@pytest.mark.parametrize("R", [4096, 16384, MAX_R])
def test_grid_and_all_pairs_write_the_same_bytes(g, R):
    g.set_params(params("two_circles"))
    f = mixed_fleet(R, 16, 90 + R, clustered=True)
    grid = run(g, f, 1.0, 8, search=abi.TEBGPU_FLEET_SEARCH_GRID)
    assert g.last_fleet_search() == "grid"
    pairs = run(g, f, 1.0, 8, search=abi.TEBGPU_FLEET_SEARCH_ALL_PAIRS)
    assert g.last_fleet_search() == "all_pairs"
    for a, b in zip(grid, pairs):
        assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("counts", [(2000,), (700, 0, 1300), (1, 999, 500, 500), (250, 250, 250, 250, 250, 250, 250, 250)])
def test_uneven_shards_through_the_table_equal_one_array_call(g, counts):
    g.set_params(params("polygon", verts=SMALL[0][1]))
    R = sum(counts)
    f = mixed_fleet(R, 24, 7 + len(counts), clustered=True)
    want = run(g, f, 1.5, 6)
    d = dev(f)
    parts = ftc.split(R, counts)
    cap = max(counts)
    T_ = cap * len(counts)
    rows = torch.zeros(T_ * abi.FLEET_ROW_DTYPE.itemsize, dtype=torch.uint8, device=DEV)
    head = torch.zeros(T_, dtype=torch.float64, device=DEV)
    rk = torch.zeros(T_, dtype=torch.int32, device=DEV)
    radius = torch.zeros(R, dtype=torch.float64, device=DEV)
    sl = lambda x, lo, hi: x[lo:hi]
    for s, (lo, hi) in enumerate(parts):
        if hi == lo:
            continue
        fa = abi.make_fleet_args(hi - lo, 1, 0, 0, 0.0, pose=sl(d["pose"], lo, hi), last_cmd=sl(d["cmd"], lo, hi),
                                 radius=sl(radius, lo, hi), world=sl(d["world"], lo, hi))
        sh = abi.make_fleet_shapes(KINDS, PV_CAP, kind=sl(d["kind"], lo, hi), heading=head, row_kind=rk)
        g.fleet_publish_shaped_device(fa, sh, abi.make_fleet_table(T_, s * cap, rows.data_ptr()))
    for s, (lo, hi) in enumerate(parts):
        if hi == lo:
            continue
        fa = abi.make_fleet_args(hi - lo, hi - lo, 24, 6, 1.5, own_count=sl(d["own"], lo, hi),
                                 custom=sl(d["custom"], lo, hi), custom_count=sl(d["cc"], lo, hi),
                                 needed=sl(d["need"], lo, hi), status=sl(d["st"], lo, hi))
        sh = abi.make_fleet_shapes(KINDS, PV_CAP, FOOT, own_vertex_count=sl(d["ownv"], lo, hi),
                                   custom_vertices=sl(d["cv"], lo, hi), heading=head, row_kind=rk)
        g.fleet_obstacles_table_shaped_device(fa, sh, abi.make_fleet_table(T_, s * cap, rows.data_ptr()))
    torch.cuda.synchronize()
    for a, b in zip(outputs(d, f), want):
        assert a.tobytes() == b.tobytes(), counts


def test_select_centres_is_the_centre_rule(g):
    g.set_params(params("polygon"))
    f = mixed_fleet(3000, 24, 5, clustered=True)
    got = run(g, f, 1.5, 6, select=abi.TEB_FLEET_SELECT_CENTRES)
    want = fsc.restate(f["pose"], f["last_cmd"], KINDS, f["kind"], 1.5, 6, f["custom"], f["cv"], f["own_count"],
                       own_vertex_count=f["own_v"], world=f["world"])
    assert_matches(got, want, f)


def test_bad_select_is_refused(g):
    f = mixed_fleet(4, 8, 1)
    for sel in (2, -1):
        with pytest.raises(T.TebGpuError):
            run(g, f, 1.0, 4, select=sel)
    g.set_params(params("circular", radius=math.inf))
    with pytest.raises(T.TebGpuError):
        run(g, f, 1.0, 4)                  # the footprints' rule needs a finite footprint
    g.set_params(params("circular", radius=0.3))
    run(g, f, 1.0, 4)


# ---- a C3 robot and a 4 m polygon robot on one stream, neighbours by their footprints
LOOP_PV = 16


def _reach_kind_params(k):
    """kind 0: C3, the car-like robot with its TwoCircles footprint; kind 1: a 4 x 1 m polygon robot"""
    if k == 0:
        p = scenes.config_params("C3")
        p.footprint_type = abi.TEB_FOOTPRINT_TWO_CIRCLES
        p.footprint_front_offset, p.footprint_front_radius = 0.2, 0.2
        p.footprint_rear_offset, p.footprint_rear_radius = 0.2, 0.2
    else:
        p = scenes.config_params("C2")
        p.footprint_type, p.footprint_vertex_count = abi.TEB_FOOTPRINT_POLYGON, 4
        p.footprint_vertices[:8] = [2.0, 0.5, -2.0, 0.5, -2.0, -0.5, 2.0, -0.5]
    p.include_dynamic_obstacles = 1
    p.max_vel_trans = p.max_vel_x
    p.global_plan_overwrite_orientation = 1
    return p


def _reach_scenario(kind):
    """corridor: the C3 robot and the long robot head-on, centres 5 m apart (bodies 2.6 m); junction: the C3 robot along
    x, the long robot along y, centres 4.3 m apart. The C3 robot first, so each kind is one contiguous shard."""
    if kind == "corridor":
        start, goal = np.array([[-2.5, 0.05], [2.5, -0.05]]), np.array([[4.0, 0.05], [-4.0, -0.05]])
    else:
        start, goal = np.array([[-1.5, 0.1], [0.1, 4.0]]), np.array([[3.0, 0.1], [0.1, -3.0]])
    gp, begin, end = _straight_plans(start, goal, 256)
    return dict(gp=gp, begin=begin, end=end, robot=np.column_stack([start, gp[:, 0, 2]]), G_cap=256, counts=(1, 1),
                raster=_raster(len(start), start, kind))


def _reach_loop(scenario, restated, cycles=20, n_cap=96, P_cap=128, M_cap=2048, Lb=10, max_rows=8, rng=3.0,
                dev_trace=None, graph_at=()):
    """test_gpu_fleet_shapes' two-kind loop under the footprints' rule: restated=False, every kind's context publishes
    its robots into one table and steps them against it with select = TEB_FLEET_SELECT_FOOTPRINTS, then costmap_tf ->
    local_plan_tf -> backup modes -> plan -> costmap check -> finish, all on one stream. True: the fleet steps replaced
    by fleet_reach_cases.restate (each robot measured with its own kind's footprint), uploaded in their place, a
    restated position, vertex or velocity within the bars of assert_matches taking the device's bits. graph_at: the
    cycles after which tebgpu_build_system_graph runs on the long robots' bands."""
    sc = _reach_scenario(scenario)
    B = len(sc["robot"])
    C_cap, PV = 1 + 2 * max_rows, LOOP_PV
    kinds = [abi.fleet_shape_from_params(_reach_kind_params(k)) for k in range(2)]
    prms = [_reach_kind_params(k) for k in range(2)]
    kind_of = np.repeat(np.arange(2), sc["counts"]).astype(np.int32)
    r = sc["raster"]
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    z = lambda shape, dtp: torch.zeros(shape, dtype=dtp, device=DEV)
    f64, i32 = torch.float64, torch.int32
    cost, grid, origin = t(r["cost"]), t(r["grid"]), t(r["origin"])
    robot = t(sc["robot"].copy())
    radius, kindt = t(np.zeros(B)), t(kind_of)
    own_rows = np.zeros((B, C_cap), abi.OBST_DTYPE)     # one static point of the caller's own per scene, far behind
    own_rows[:, 0]["x"], own_rows[:, 0]["y"] = sc["robot"][:, 0] - 5.0, sc["robot"][:, 1] + 5.0
    custom, ccount, own = t(own_rows.view(np.uint8)), t(np.ones(B, np.int32)), t(np.ones(B, np.int32))
    cv, ov = z((B, PV, 2), f64), z((B, PV, 2), f64)
    last_cmd, fneed, fstat = z((B, 3), f64), z(B, i32), z(B, i32)
    gpd, begin, end = t(sc["gp"]), t(sc["begin"]), t(sc["end"])
    vel, cmd_vel = z((B, 3), f64), z((B, 3), f64)
    cap, first = D.fleet_layout(list(sc["counts"]), 2)
    rows = t(ftc.padding(2 * cap).view(np.uint8))
    head, rkind = z(2 * cap, f64), z(2 * cap, i32)
    ctx = []
    lo = 0
    for k, n in enumerate(sc["counts"]):
        hi = lo + n
        sl = slice(lo, hi)
        p = prms[k]
        g = T.TebGpu(n, n_cap, n, M_cap, 0, max_obst_vertices=PV)
        g.set_params(p)
        state = {kk: t(v) for kk, v in abi.make_cycle_state(n, Lb).items()}
        state["last_cmd"] = last_cmd[sl]
        K = dict(g=g, p=p, sl=sl, n=n, state=state, plan=z((n, P_cap, 3), f64), pcount=z(n, i32), result=z(n, i32),
                 gidx=z(n, i32), needed=z((n, 2), i32), since=z(n, f64), poses=z((n, n_cap, 4), f64), nn=z(n, i32),
                 sid=t(np.arange(n, dtype=np.int32)), obst=z(n * M_cap * 64, torch.uint8), ocount=z(n, i32),
                 costo=z(n, f64), chi2=z(n, f64), status=z(n, i32), iters=z(n, i32), cmd=z((n, 4), f64),
                 path=z(n, i32), feas=z(n, i32), qc=z(n, i32), outcome=z(n, i32), osc=z(n, i32),
                 ident=t(np.tile(IDENTITY, (n, 1))))
        vs = np.zeros((n, 4))
        vs[:, 3] = 1.0
        K["vs"], K["vstart"], K["vgoal"] = vs, t(vs), t(vs)
        bs = abi.TebBatch()
        bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = n, n_cap, n, M_cap, 0, PV
        bs.poses, bs.n, bs.scene_id = K["poses"].data_ptr(), K["nn"].data_ptr(), K["sid"].data_ptr()
        bs.obstacles, bs.obst_count, bs.obst_vertices = K["obst"].data_ptr(), K["ocount"].data_ptr(), ov[sl].data_ptr()
        bs.vel_start, bs.vel_goal, bs.prefer_rotdir = K["vstart"].data_ptr(), K["vgoal"].data_ptr(), state["prefer_rotdir"].data_ptr()
        bs.cost, bs.chi2, bs.status, bs.lm_iters = (K["costo"].data_ptr(), K["chi2"].data_ptr(), K["status"].data_ptr(),
                                                     K["iters"].data_ptr())
        K["bs"] = bs
        ca = abi.TebCostmapArgs()
        ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = n, r["cost"].shape[1], M_cap, C_cap, 1
        ca.behind_robot_dist = 1.5
        ca.cost, ca.grid, ca.origin, ca.robot = cost[sl].data_ptr(), grid[sl].data_ptr(), origin[sl].data_ptr(), robot[sl].data_ptr()
        ca.custom, ca.custom_count = custom[sl].data_ptr(), ccount[sl].data_ptr()
        ca.obstacles, ca.obst_count = K["obst"].data_ptr(), K["ocount"].data_ptr()
        K["ca"] = ca
        K["cframes"] = abi.make_frame_args(custom_to_costmap=K["ident"].data_ptr(), custom_vertices=cv[sl].data_ptr(),
                                           obst_vertices=ov[sl].data_ptr(), PV_cap=PV)
        K["pframes"] = abi.make_frame_args(costmap_to_plan=K["ident"].data_ptr(), plan_to_costmap=K["ident"].data_ptr())
        K["la"] = abi.make_local_plan_args(sc["G_cap"], P_cap, 0, max_lookahead_dist=2.0, global_plan=gpd[sl].data_ptr(),
                                           plan_begin=begin[sl].data_ptr(), plan_end=end[sl].data_ptr(),
                                           robot=robot[sl].data_ptr(), robot_vel=vel[sl].data_ptr(),
                                           grid=grid[sl].data_ptr(), origin=origin[sl].data_ptr(),
                                           infeasible_count=state["infeasible_count"].data_ptr(),
                                           since_infeasible=K["since"].data_ptr(), plan=K["plan"].data_ptr(),
                                           plan_count=K["pcount"].data_ptr(), goal_idx=K["gidx"].data_ptr(),
                                           result=K["result"].data_ptr(), needed=K["needed"].data_ptr())
        K["args"] = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0,
                                  False)
        K["fa"] = abi.make_feasibility_args(0.1, max_queries=512, feasible=K["feas"].data_ptr(),
                                            query_count=K["qc"].data_ptr())
        K["world"] = abi.make_costmap_world(r["cost"].shape[1], cost[sl].data_ptr(), grid[sl].data_ptr(),
                                            origin[sl].data_ptr())
        K["fl"] = abi.make_fleet_args(n, n, C_cap, max_rows, rng, pose=robot[sl], last_cmd=last_cmd[sl],
                                      radius=radius[sl], own_count=own[sl], custom=custom[sl], custom_count=ccount[sl],
                                      needed=fneed[sl], status=fstat[sl])
        K["sh"] = abi.make_fleet_shapes(kinds, PV, FOOT, kind=kindt[sl], custom_vertices=cv[sl], heading=head,
                                        row_kind=rkind)
        K["tb"] = abi.make_fleet_table(2 * cap, first[k], rows)
        ctx.append(K)
        lo = hi
    cs = dict(buffer_length=Lb, oscillation_recovery_min_duration=2.0)
    dt, now = 0.2, 1000.0
    s = torch.cuda.Stream()
    trace, graphs = [], []
    for c in range(cycles):
        robot_in = robot.clone()
        with torch.cuda.stream(s):
            if restated:
                s.synchronize()
                cur = custom.cpu().numpy().view(abi.OBST_DTYPE).reshape(B, C_cap).copy()
                outs = [frc.restate(prms[k], robot.cpu().numpy(), last_cmd.cpu().numpy(), kinds, kind_of, rng, max_rows,
                                    cur, cv.cpu().numpy(), np.ones(B, np.int32)) for k in range(2)]
                hc, hcc, hn, hs, hv = (np.stack([outs[kind_of[b]][i][b] for b in range(B)]) for i in range(5))
                d = dev_trace[c]
                dc = d["custom"].view(abi.OBST_DTYPE).reshape(B, C_cap)
                assert_matches((dc, d["ccount"], d["fneed"], d["fstat"], d["cv"]), (hc, hcc, hn, hs, hv),
                               dict(custom=cur, own_count=np.ones(B, np.int32), own_v=np.zeros(B, np.int32),
                                    cv=cv.cpu().numpy()))
                for key in CLOSE:          # within the bars: take the device's bits
                    hc[key] = dc[key]
                hv = d["cv"]
                custom.copy_(t(hc.view(np.uint8).reshape(B, -1)))
                cv.copy_(t(hv))
                ccount.copy_(t(hcc))
                fneed.copy_(t(hn))
                fstat.copy_(t(hs))
            else:
                for K in ctx:
                    K["g"].fleet_publish_shaped_device(K["fl"], K["sh"], K["tb"], stream=s.cuda_stream)
                for K in ctx:
                    K["g"].fleet_obstacles_table_shaped_device(K["fl"], K["sh"], K["tb"], stream=s.cuda_stream)
            for K in ctx:
                g, st, sl = K["g"], K["state"], K["sl"]
                cy = abi.make_cycle_args(now, L_cap=Lb, **cs, local_plan_result=K["result"].data_ptr(),
                                         robot_vel=vel[sl].data_ptr(), cmd=K["cmd"].data_ptr(),
                                         feasible=K["feas"].data_ptr(), cmd_vel=cmd_vel[sl].data_ptr(),
                                         outcome=K["outcome"].data_ptr(), oscillating=K["osc"].data_ptr(),
                                         **{kk: st[kk].data_ptr() for kk in abi.CYCLE_STATE})
                K["since"].copy_(now - st["last_infeasible"])
                g.costmap_obstacles_device(K["ca"], stream=s.cuda_stream, frames=K["cframes"])
                g.local_plan_device(K["bs"], K["la"], stream=s.cuda_stream, frames=K["pframes"])
                g.backup_modes_device(K["bs"], cy, stream=s.cuda_stream)
                g.plan_device(K["bs"], K["args"], K["cmd"], initial_plan=K["plan"], plan_count=K["pcount"],
                              P_cap=P_cap, path=K["path"], stream=s.cuda_stream)
                g.check_feasible_costmap_device(K["bs"], K["fa"], K["world"], stream=s.cuda_stream)
                g.finish_cycle_device(K["bs"], cy, stream=s.cuda_stream)
        s.synchronize()
        if c in graph_at:                  # on contexts of their own, so the loop's contexts are the restated loop's
            for k, K in enumerate(ctx[1:], 1):
                n = K["n"]
                hb = abi.HostBatch(K["poses"].cpu().numpy(), K["nn"].cpu().numpy(),
                                   K["obst"].cpu().numpy().view(abi.OBST_DTYPE).reshape(n, M_cap),
                                   K["ocount"].cpu().numpy(), scene_id=np.arange(n, dtype=np.int32), vel_start=K["vs"],
                                   vel_goal=K["vs"], prefer_rotdir=K["state"]["prefer_rotdir"].cpu().numpy(),
                                   obst_vertices=ov[K["sl"]].cpu().numpy())
                g2 = T.TebGpu(n, n_cap, n, M_cap, 0, max_obst_vertices=PV)
                g2.set_params(K["p"])
                graphs.append((c, k, hb, g2.build_system(hb, graph=True)))
                g2.close()
        with torch.cuda.stream(s):
            th = robot[:, 2].clone()
            robot[:, 0] += (cmd_vel[:, 0] * torch.cos(th) - cmd_vel[:, 1] * torch.sin(th)) * dt
            robot[:, 1] += (cmd_vel[:, 0] * torch.sin(th) + cmd_vel[:, 1] * torch.cos(th)) * dt
            robot[:, 2] += cmd_vel[:, 2] * dt
            vel.copy_(cmd_vel)
        s.synchronize()
        rec = dict(robot_in=robot_in, custom=custom, ccount=ccount, fneed=fneed, fstat=fstat, cv=cv, ov=ov, robot=robot, cmd_vel=cmd_vel,
                   last_cmd=last_cmd)
        for k, K in enumerate(ctx):
            for key in ("obst", "ocount", "pcount", "result", "nn", "poses", "status", "path", "cmd", "outcome", "osc",
                        "feas"):
                rec[f"{key}{k}"] = K[key]
            for key, v in K["state"].items():
                rec[f"{key}{k}"] = v
        rec = {key: v.cpu().numpy().copy() for key, v in rec.items()}
        for k, K in enumerate(ctx):
            pc, pl = rec[f"pcount{k}"], K["plan"].cpu().numpy()
            rec[f"plan{k}"] = np.concatenate([pl[b, :pc[b]] for b in range(K["n"])])
        trace.append(rec)
        now += dt
    for K in ctx:
        K["g"].close()
    return trace, graphs



@pytest.mark.parametrize("scenario", ["corridor", "junction"])
def test_a_long_robot_loop_matches_the_restated_loop_and_sees_its_neighbour_early(scenario):
    cycles = 20
    dev_, graphs = _reach_loop(scenario, False, cycles=cycles, graph_at=range(cycles))
    ref, _ = _reach_loop(scenario, True, cycles=cycles, dev_trace=dev_)
    for c, (x, y) in enumerate(zip(dev_, ref)):
        assert x.keys() == y.keys()
        for key in x:
            assert x[key].tobytes() == y[key].tobytes(), (scenario, c, key)
    assert sum((c[f"outcome{k}"] == abi.TEB_CYCLE_COMMAND).sum() for c in dev_ for k in (0, 1)) > 0
    # cycles where the centres are out of range (the centre rule gives the long robot no row) and the footprints' gap
    # is not: the long robot has the C3 robot's rows, and once they move, its band has dynamic-obstacle edges
    early, edges = 0, 0
    for c, k, hb, gr in graphs:
        pos = dev_[c]["robot_in"]
        d2 = float(((pos[0, :2] - pos[1, :2]) ** 2).sum())
        if d2 <= 3.0 ** 2:
            continue
        rows = dev_[c]["custom"].view(abi.OBST_DTYPE).reshape(2, -1)[1, 1:dev_[c]["ccount"][1]]
        if not len(rows):
            continue
        assert len(rows) == 2 and set(rows["type"].tolist()) == {abi.TEB_OBST_CIRCULAR}, (scenario, c)
        early += 1
        nb, cnt = int(hb.n[0]), int(hb.obst_count[0])
        dyn = np.nonzero(hb.obstacles[0, :cnt]["dynamic"] == 1)[0]
        if nb < 3 or not len(dyn):
            continue
        edges += 1
        assert np.isfinite(gr["dyn_t"][0, 1:nb - 1]).all(), (scenario, c)
        words = gr["assoc"][0, :nb]
        for l in dyn:
            assert not ((words[:, l // 64] >> np.uint64(l % 64)) & np.uint64(1)).any(), (scenario, c, l)
    print(f"{scenario}: {early} cycles with the neighbour out of the centres' range, {edges} with dynamic edges")
    assert early > 0 and edges > 0
