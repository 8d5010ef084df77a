"""tebgpu_costmap_window(_device): every robot's rolling-window costmap cut out of the static maps on the device, held
byte for byte to tests/costmap_window_cases.py's restatement on the hand cases and on random fleets (maps of several
sizes and resolutions, one larger than L2; windows of 60 x 60 to 400 x 400; strides that are and are not multiples of
16; with and without transforms; robots moving for 20 cycles); NULL transforms against explicit identity rows; bad
robots; and a 20-cycle fleet loop fed by the window step against the same loop fed the restatement's rasters."""
import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import costmap_window_cases as cw
from tests import frame_cases as fc

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = "cuda:0"
IDENTITY = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(64, 64, 8192, 64, 0)
    g.set_params(abi.default_params())
    yield g
    g.close()


def host_maps(maps, p=cw.DEFAULTS):
    return abi.make_static_maps([m["data"] for m in maps], [(m["mox"], m["moy"], m["mr"]) for m in maps],
                                unknown_cost_value=p["unknown_cost_value"], lethal_threshold=p["lethal_threshold"],
                                track_unknown_space=p["track_unknown_space"], trinary_costmap=p["trinary_costmap"])


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def device_maps(maps, p=cw.DEFAULTS):
    """(TebStaticMaps of device arrays, the tensors behind it)"""
    m, arrays = host_maps(maps, p)
    keep = {k: t(v) for k, v in arrays.items()}
    m.data, m.offset, m.size, m.origin = (keep[k].data_ptr() for k in ("data", "offset", "size", "origin"))
    return m, keep


def run_device(g, dm, robot, map_id, origin, grid, cap, tf=None, row_shift=0):
    """the device entry point; row_shift moves the raster off a 16-byte boundary by that many bytes"""
    S = len(robot)
    buf = torch.full((S * cap + 16,), 0x5A, dtype=torch.uint8, device=DEV)
    cost = buf[row_shift:row_shift + S * cap]
    org, st = t(np.array(origin, np.float64)), torch.full((S,), -7, dtype=torch.int32, device=DEV)
    ins = dict(robot=t(np.asarray(robot, np.float64)), map_id=t(np.asarray(map_id, np.int32)),
               grid=t(np.asarray(grid, np.int32)), tf=None if tf is None else t(np.asarray(tf, np.float64)))
    wa = abi.TebCostmapWindowArgs()
    wa.S, wa.cell_cap = S, cap
    wa.robot, wa.map_id, wa.grid = ins["robot"].data_ptr(), ins["map_id"].data_ptr(), ins["grid"].data_ptr()
    wa.costmap_to_map = None if tf is None else ins["tf"].data_ptr()
    wa.origin, wa.cost, wa.status = org.data_ptr(), cost.data_ptr(), st.data_ptr()
    g.costmap_window_device(dm, wa, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    assert (b[:row_shift] == 0x5A).all() and (b[row_shift + S * cap:] == 0x5A).all()     # nothing outside the rows
    return cost.cpu().numpy().reshape(S, cap), org.cpu().numpy(), st.cpu().numpy()


def check(g, maps, robot, map_id, origin, grid, cap, tf=None, p=cw.DEFAULTS, host=True, row_shift=0):
    want = cw.window_np(maps, robot, map_id, origin, grid, cap, tf, p)
    dm, keep = device_maps(maps, p)
    got = run_device(g, dm, robot, map_id, origin, grid, cap, tf, row_shift)
    for a, b, name in zip(got, want, ("cost", "origin", "status")):
        assert a.tobytes() == b.tobytes(), name
    if host:
        hm, _ = host_maps(maps, p)
        h = g.costmap_window(hm, robot, map_id, origin, grid, cap, tf)
        for a, b, name in zip(h, want, ("cost", "origin", "status")):
            assert a.tobytes() == b.tobytes(), name
    return want


def test_hand_cases(gpu):
    R = 0.25
    edge = np.zeros((8, 8), np.uint8)
    edge[:, 1] = 100
    grid_map = (10 * np.arange(8)[:, None] + np.arange(8)[None, :]).astype(np.uint8)
    graded = (np.arange(8, dtype=np.uint8) + 1)[None, :].repeat(8, axis=0)
    maps = [dict(data=edge, mox=0.0, moy=0.0, mr=0.125), dict(data=np.full((2, 2), 100, np.uint8), mox=0.125, moy=0.125, mr=R),
            dict(data=grid_map, mox=-1.0, moy=-1.0, mr=R)] + [dict(data=graded, mox=0.0, moy=0.0, mr=mr) for mr in (0.025, 0.05, 0.1)]
    s4, c4 = np.sin(np.pi / 4), np.cos(np.pi / 4)
    a = np.pi / 3
    rows = [  # map, robot, origin, grid, transform
        (0, (0.1875, 0.1875, 0), (0, 0, R), (2, 2), IDENTITY), (1, (0.3125, 0, 0), (0, 0, R), (3, 1), IDENTITY),
        (1, (0.3125, -0.25, 0), (0, 0, R), (3, 1), IDENTITY), (2, (0.1875, 0.1875, 0), (0, 0, R), (2, 2), IDENTITY),
        (2, (0.1875, 0.1875, 0), (0, 0, R), (2, 2), [0.5, -0.25, 0, 0, 0, 0, 1]),
        (2, (0.1875, 0.1875, 0), (0, 0, R), (2, 2), [0, 0, 0, 0, 0, s4, c4]),
        (2, (0.1875, 0.1875, 0), (0, 0, R), (2, 2), [0, 0, 0, 0, 0, 1, np.cos(np.pi / 2)]),
        (2, (0.1875, 0.1875, 0), (0, 0, R), (2, 2), [0, 0, 0, 0, 0, 3 * s4, 3 * c4]),
        (2, (0.1875, 0.1875, 0), (0, 0, R), (2, 2), [0, 0, 0, np.sin(a / 2), 0, 0, np.cos(a / 2)]),
        (2, (1.0, 0.0, 0), (0, 0, R), (4, 1), IDENTITY), (2, (-1.0, 0.0, 0), (0, 0, R), (4, 1), IDENTITY),
        (2, (0.9375, 0.0, 0), (0, 0, R), (4, 1), IDENTITY)] + [
        (3 + k, (0.0875, 0.025, 0), (0, 0, 0.05), (4, 1), IDENTITY) for k in range(3)]
    mid = [r[0] for r in rows]
    robot, origin, grid, tf = (np.array([r[k] for r in rows], float) for k in (1, 2, 3, 4))
    grid = grid.astype(np.int32)
    for p in (cw.DEFAULTS, dict(cw.DEFAULTS, trinary_costmap=False, lethal_threshold=254),
              dict(cw.DEFAULTS, track_unknown_space=False, trinary_costmap=False)):
        want = check(gpu, maps, robot, mid, origin, grid, 4, tf, p)
        check(gpu, maps, robot, mid, origin, grid, 4, None, p)
    assert want[1][9:12, 0].tolist() == [0.5, -1.25, 0.5]                 # the snapped origins of the hand cases


def fleet(seed, S, sx, sy, big=False):
    rng = np.random.default_rng(seed)
    maps = [cw.random_map(rng, 900, 700, -20.0, -15.0, 0.05), cw.random_map(rng, 300, 500, -10.0, -30.0, 0.1),
            cw.random_map(rng, 1600, 1200, -25.0, -12.0, 0.025)]
    if big:   # 8000 x 8000 bytes: more than the 50 MB of the H100's L2
        maps.append(cw.random_map(rng, 8000, 8000, -200.0, -200.0, 0.05))
    map_id = rng.integers(0, len(maps), S).astype(np.int32)
    lo = np.array([[m["mox"], m["moy"]] for m in maps])[map_id]
    hi = lo + np.array([[m["data"].shape[1] * m["mr"], m["data"].shape[0] * m["mr"]] for m in maps])[map_id]
    xy = rng.uniform(lo - 2.0, hi + 2.0)                                 # some windows reach past the map
    robot = np.column_stack([xy, rng.uniform(-np.pi, np.pi, S)])
    res = rng.choice([0.05, 0.05, 0.1, 0.025], S)
    origin = np.column_stack([xy[:, 0] + rng.uniform(-3, 3, S), xy[:, 1] + rng.uniform(-3, 3, S), res])
    grid = np.tile(np.array([sx, sy], np.int32), (S, 1))
    grid[::7] = (max(sx - 5, 1), max(sy - 3, 1))                         # smaller windows in the same stride
    return rng, maps, robot, map_id, origin, grid


@pytest.mark.parametrize("S,sx,sy,extra,tf,big", [
    (1, 60, 60, 0, False, False), (5, 60, 60, 7, True, True), (37, 121, 97, 3, True, False),
    (1024, 120, 120, 0, False, True), (64, 400, 400, 0, False, False), (24, 400, 400, 5, True, True),
    (8192, 60, 60, 0, False, False), (8192, 60, 60, 0, True, True)])
def test_random_fleets_match_the_restatement(gpu, S, sx, sy, extra, tf, big):
    rng, maps, robot, map_id, origin, grid = fleet(S + sx + extra, S, sx, sy, big)
    cap = sx * sy + extra
    trans = np.array([fc.random_transform(rng, tilted=k % 3 == 0, unit=k % 2 == 0) for k in range(S)]) if tf else None
    if tf:   # keep the transformed windows near the maps: a small translation
        trans[:, :3] *= 0.05
    want = check(gpu, maps, robot, map_id, origin, grid, cap, trans, host=S <= 1024, row_shift=S % 16)
    if S > 1:     # the fleet meets the map and leaves it, and meets lethal cells
        on = want[0] != cw.NO_INFORMATION
        assert on.any() and (~on).any() and (want[0] == cw.LETHAL_OBSTACLE).any()


def test_null_transforms_equal_explicit_identity_rows(gpu):
    rng, maps, robot, map_id, origin, grid = fleet(3, 200, 120, 120)
    dm, keep = device_maps(maps)
    a = run_device(gpu, dm, robot, map_id, origin, grid, 120 * 120)
    b = run_device(gpu, dm, robot, map_id, origin, grid, 120 * 120, np.tile(IDENTITY, (200, 1)))
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()


def test_moving_robots_carry_their_origins_for_20_cycles(gpu):
    rng, maps, robot, map_id, origin, grid = fleet(4, 256, 120, 120, big=True)
    S, cap = 256, 120 * 120
    trans = np.array([fc.random_transform(rng) for _ in range(S)])
    trans[:, :2] *= 0.02
    dm, keep = device_maps(maps)
    ins = dict(map_id=t(map_id), grid=t(grid), tf=t(trans))
    org, rob = t(origin), t(robot)
    cost, st = torch.zeros((S, cap), dtype=torch.uint8, device=DEV), torch.zeros(S, dtype=torch.int32, device=DEV)
    wa = abi.TebCostmapWindowArgs()
    wa.S, wa.cell_cap = S, cap
    wa.robot, wa.map_id, wa.grid, wa.costmap_to_map = rob.data_ptr(), ins["map_id"].data_ptr(), ins["grid"].data_ptr(), ins["tf"].data_ptr()
    wa.origin, wa.cost, wa.status = org.data_ptr(), cost.data_ptr(), st.data_ptr()
    h_org, h_rob = origin.copy(), robot.copy()
    vel = np.column_stack([rng.uniform(-0.6, 0.6, S), rng.uniform(-0.6, 0.6, S)])
    for k in range(20):
        gpu.costmap_window_device(dm, wa, stream=torch.cuda.current_stream().cuda_stream)
        want = cw.window_np(maps, h_rob, map_id, h_org, grid, cap, trans)
        torch.cuda.synchronize()
        assert cost.cpu().numpy().tobytes() == want[0].tobytes(), k
        assert org.cpu().numpy().tobytes() == want[1].tobytes(), k
        h_org = want[1]
        h_rob[:, :2] += vel * 0.2
        rob.copy_(t(h_rob))
    assert (h_org[:, :2] != origin[:, :2]).all()


def test_bad_robots_get_the_default_on_the_device_and_are_refused_on_the_host(gpu):
    rng, maps, robot, map_id, origin, grid = fleet(5, 16, 60, 60)
    cap = 60 * 60
    map_id[1], map_id[2] = -1, len(maps)
    grid[3], grid[4], grid[5] = (0, 60), (60, 0), (61, 60)
    origin[6, 2], origin[7, 2], origin[8, 2] = 0.0, -0.05, np.nan
    origin[9, 2] = np.inf
    for p in (cw.DEFAULTS, dict(cw.DEFAULTS, track_unknown_space=False)):
        cost, org, st = check(gpu, maps, robot, map_id, origin, grid, cap, p=p, host=False)
        assert st[1:3].tolist() == [cw.BAD_MAP] * 2 and st[3:10].tolist() == [cw.BAD_GRID] * 7
        assert (st[10:] == cw.OK).all() and st[0] == cw.OK
        assert (cost[1:10] == cw.default_cost(p)).all()
        assert org[1:10].tobytes() == origin[1:10].tobytes()
    hm, _ = host_maps(maps)
    for s in range(1, 10):
        keep = [0, s]
        with pytest.raises(T.TebGpuError):
            gpu.costmap_window(hm, robot[keep], map_id[keep], origin[keep], grid[keep], cap)
    # a map whose bytes lie past the pool is a bad map on the device
    dm, keep_t = device_maps(maps)
    dm.pool_bytes = dm.pool_bytes - 1
    _, _, st = run_device(gpu, dm, robot, np.full(16, len(maps) - 1, np.int32), np.tile([0.0, 0.0, 0.05], (16, 1)), np.full((16, 2), 60, np.int32), cap)
    assert (st == cw.BAD_MAP).all()


def test_argument_errors(gpu):
    rng, maps, robot, map_id, origin, grid = fleet(6, 4, 60, 60)
    hm, _ = host_maps(maps)
    for field, value in (("W", 0), ("unknown_cost_value", 256), ("lethal_threshold", -1), ("pool_bytes", -1)):
        m, _ = host_maps(maps)
        setattr(m, field, value)
        with pytest.raises(T.TebGpuError):
            gpu.costmap_window(m, robot, map_id, origin, grid, 3600)
    with pytest.raises(T.TebGpuError):
        gpu.costmap_window(hm, robot, map_id, origin, grid, 0)
    big = np.zeros((8193, 3))
    with pytest.raises(T.TebGpuError):       # more robots than max_scenes
        gpu.costmap_window(hm, big, np.zeros(8193, np.int32), big + [0, 0, 0.05], np.full((8193, 2), 4, np.int32), 16)


# ---- the fleet cycle on one stream: window -> costmap conversion (custom rows moved) -> local plan -> backup modes
# ---- -> plan -> costmap check -> finish, against the same loop fed the restatement's rasters

FOOTPRINT = np.array([(-0.1, -0.1), (0.1, -0.1), (0.1, 0.1), (-0.1, 0.1)])


def _loop_map(d, tf):
    """a 0.05 m map over the robots and their plans: free, with lethal squares under robots 4 .. 7 (placed through
    the transform) and at random, and an unknown patch"""
    pts = d["global_plan"][:, :, :2].reshape(-1, 2)
    pts = np.vstack([pts[np.isfinite(pts).all(1)], d["robot"][:, :2]])
    lo, hi = pts.min(0) - 6.0, pts.max(0) + 6.0
    mr = 0.05
    msx, msy = (int(v) for v in np.ceil((hi - lo) / mr))
    data = np.zeros((msy, msx), np.uint8)
    rng = np.random.default_rng(23)
    for _ in range(6000):
        x, y = rng.integers(0, msx - 4), rng.integers(0, msy - 4)
        data[y:y + rng.integers(1, 4), x:x + rng.integers(1, 4)] = 100
    data[:40, :40] = 255
    b = fc.tf2_basis(list(tf[3:7]))
    for s in range(4, 8):
        px, py = fc.apply(b, tf[:2], d["robot"][s, 0], d["robot"][s, 1])
        cx, cy = int((px - lo[0]) / mr), int((py - lo[1]) / mr)
        data[cy - 3:cy + 3, cx - 3:cx + 3] = 100
    return dict(data=data, mox=float(lo[0]), moy=float(lo[1]), mr=mr)


def _fleet_loop(restated, cycles=20, B=16, P_cap=160, M_cap=2048, n_cap=96, Lb=10, sx=60):
    d = scenes.global_plans(B, 1024, S=B, seed=21)
    tf_row = np.array(fc.random_transform(np.random.default_rng(3)))
    tf_row[2:] = [0.0, 0.0, 0.0, np.sin(0.05 / 2), np.cos(0.05 / 2)]
    tf_row[:2] = [0.3, -0.2]
    trans = np.tile(tf_row, (B, 1))
    maps = [_loop_map(d, tf_row)]
    cap = sx * sx
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 0
    p.max_vel_trans = p.max_vel_x
    g = T.TebGpu(B, n_cap, B, M_cap, 0)
    g.set_params(p)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=DEV)
    f64, i32 = torch.float64, torch.int32
    dm, keep = device_maps(maps)
    h_org = np.column_stack([d["robot"][:, :2] - 1.5, np.full(B, 0.05)])
    cost, grid, origin = z((B, cap), torch.uint8), t(np.full((B, 2), sx, np.int32)), t(h_org)
    map_id, win_tf, wst = z(B, i32), t(trans), z(B, i32)
    robot = t(d["robot"].copy())
    custom = np.zeros((B, 1), abi.OBST_DTYPE)
    custom["x"], custom["y"], custom["type"] = 0.4, -0.3, abi.TEB_OBST_POINT
    cu, cc, cu_tf = t(custom.view(np.uint8)), t(np.ones(B, np.int32)), t(trans)
    obst, ocount = z(B * M_cap * 64, torch.uint8), z(B, i32)
    gp, begin, end = t(d["global_plan"]), t(d["plan_begin"].copy()), t(d["plan_end"])
    plan, pcount, result = z((B, P_cap, 3), f64), z(B, i32), z(B, i32)
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
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, B, M_cap, 0, 0
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
    bs.vel_start, bs.vel_goal, bs.prefer_rotdir = vstart.data_ptr(), vgoal.data_ptr(), state["prefer_rotdir"].data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = costo.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    wa = abi.TebCostmapWindowArgs()
    wa.S, wa.cell_cap = B, cap
    wa.robot, wa.map_id, wa.costmap_to_map = robot.data_ptr(), map_id.data_ptr(), win_tf.data_ptr()
    wa.origin, wa.grid, wa.cost, wa.status = origin.data_ptr(), grid.data_ptr(), cost.data_ptr(), wst.data_ptr()
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles, ca.behind_robot_dist = B, cap, M_cap, 1, 1, 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.custom, ca.custom_count = cu.data_ptr(), cc.data_ptr()
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    fr = abi.make_frame_args(custom_to_costmap=cu_tf.data_ptr())
    la = abi.make_local_plan_args(1024, P_cap, 0, max_lookahead_dist=2.0, global_plan=gp.data_ptr(),
                                  plan_begin=begin.data_ptr(), plan_end=end.data_ptr(), robot=robot.data_ptr(),
                                  robot_vel=vel.data_ptr(), grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  infeasible_count=state["infeasible_count"].data_ptr(), since_infeasible=since.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), result=result.data_ptr())
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    fa = abi.make_feasibility_args(0.1, max_queries=512, feasible=feas.data_ptr(), query_count=qc.data_ptr())
    world = abi.make_costmap_world(cap, cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), FOOTPRINT)
    sc = dict(buffer_length=Lb, oscillation_recovery_min_duration=2.0)
    dt, now = 0.2, 1000.0
    s = torch.cuda.Stream()
    trace = []
    for k in range(cycles):
        cy = abi.make_cycle_args(now, L_cap=Lb, **sc, local_plan_result=result.data_ptr(), robot_vel=vel.data_ptr(),
                                 cmd=cmd.data_ptr(), feasible=feas.data_ptr(), cmd_vel=cmd_vel.data_ptr(),
                                 outcome=outcome.data_ptr(), oscillating=osc.data_ptr(),
                                 **{kk: state[kk].data_ptr() for kk in abi.CYCLE_STATE})
        with torch.cuda.stream(s):
            since.copy_(now - state["last_infeasible"])
            if restated:
                s.synchronize()
                c, h_org, _ = cw.window_np(maps, robot.cpu().numpy(), np.zeros(B, np.int32), h_org, grid.cpu().numpy(),
                                           cap, trans)
                cost.copy_(t(c))
                origin.copy_(t(h_org))
            else:
                g.costmap_window_device(dm, wa, stream=s.cuda_stream)
            g.costmap_obstacles_device(ca, stream=s.cuda_stream, frames=fr)
            g.local_plan_device(bs, la, stream=s.cuda_stream)
            g.backup_modes_device(bs, cy, stream=s.cuda_stream)
            g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, path=path,
                          stream=s.cuda_stream)
            g.check_feasible_costmap_device(bs, fa, world, stream=s.cuda_stream)
            g.finish_cycle_device(bs, cy, stream=s.cuda_stream)
            th = robot[:, 2]
            robot[:, 0] += (cmd_vel[:, 0] * torch.cos(th) - cmd_vel[:, 1] * torch.sin(th)) * dt
            robot[:, 1] += (cmd_vel[:, 0] * torch.sin(th) + cmd_vel[:, 1] * torch.cos(th)) * dt
            robot[:, 2] += cmd_vel[:, 2] * dt
            vel.copy_(cmd_vel)
        s.synchronize()
        oc = ocount.cpu().numpy()
        rows = obst.cpu().numpy().reshape(B, M_cap * 64)
        rec = dict(n=n, status=status, path=path, cmd=cmd, cmd_vel=cmd_vel, outcome=outcome, feasible=feas,
                   query_count=qc, poses=poses, obst_count=ocount, cost=cost, origin=origin, **state)
        c = {kk: v.cpu().numpy().copy() for kk, v in rec.items()}
        c["rows"] = [rows[b, :max(int(oc[b]), 0) * 64].tobytes() for b in range(B)]
        trace.append(c)
        now += dt
    g.close()
    return trace


def test_fleet_loop_with_the_window_step_matches_the_loop_fed_the_restated_rasters():
    dev = _fleet_loop(False)
    ref = _fleet_loop(True)
    for k, (a, b) in enumerate(zip(dev, ref)):
        for key in a:
            assert (a[key] == b[key]) if key == "rows" else (a[key].tobytes() == b[key].tobytes()), (k, key)
    feas = np.concatenate([c["feasible"] for c in dev])
    cnt = np.concatenate([c["obst_count"] for c in dev])
    assert (feas == 1).any() and (feas == 0).any() and (cnt > 1).any()
    assert (dev[0]["origin"] != dev[-1]["origin"]).any()
