"""The other robots of a fleet as custom obstacle rows on the device (tebgpu_fleet_obstacles / _device,
k_fleet_obstacles), held to tests/fleet_cases.py's restatement: needed, statuses, counts, row order, positions, radii and
dynamic flags bit for bit, velocities within 1e-12 (the device's sin / cos), the caller's own rows and every row past
the ones written untouched, the same bytes from a second call and from the host entry point. Then a fleet loop on one
stream (fleet obstacles -> costmap_tf -> local_plan_tf -> backup modes -> plan with dynamic obstacles -> costmap check
-> finish) against the same loop fed neighbour rows built on the host, for two robots meeting head-on in a corridor,
four crossing at a junction and a random fleet."""
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import fleet_cases as fc

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
IDENTITY = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
MAX_R = 8192


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(MAX_R, 8, MAX_R + 64, 64)
    yield g
    g.close()


def random_fleet(R, S, C_cap, seed, worlds=3, clustered=True):
    """R robots over `worlds` worlds, clustered (a few dense groups) or sparse, some coincident, some still, some
    creeping at the 0.001 boundary; each scene's own rows are random bytes, own_count in 0 .. C_cap"""
    rng = np.random.default_rng(seed)
    if clustered:
        centres = rng.uniform(-20, 20, (max(1, R // 50), 2))
        xy = centres[rng.integers(0, len(centres), R)] + rng.normal(0, 1.0, (R, 2))
    else:
        xy = rng.uniform(-100, 100, (R, 2))
    pose = np.column_stack([xy, rng.uniform(-math.pi, math.pi, R)])
    dup = rng.integers(0, R, R // 20)
    pose[dup[1:]] = pose[dup[:-1]]                       # coincident robots
    cmd = np.column_stack([rng.uniform(-0.4, 0.4, R), rng.uniform(-0.1, 0.1, R), rng.uniform(-0.3, 0.3, R)])
    still = rng.random(R) < 0.2
    cmd[still, :2] = 0.0
    slow = rng.random(R) < 0.05
    cmd[slow, 0], cmd[slow, 1] = rng.choice([0.001, math.nextafter(0.001, 0), 0.0011, 0.0009], slow.sum()), 0.0
    radius = rng.uniform(0.1, 0.6, R)
    world = rng.integers(0, worlds, R).astype(np.int32)
    custom = np.zeros((S, C_cap), abi.OBST_DTYPE)
    custom.view(np.uint8)[:] = rng.integers(0, 256, custom.nbytes, dtype=np.uint8).reshape(S, -1)
    own = rng.integers(0, C_cap + 1, S).astype(np.int32)
    return dict(pose=pose, last_cmd=cmd, radius=radius, world=world, custom=custom, own_count=own)


def run_device(g, f, rng, max_rows, scene=None, S=None, custom_count=None, twice=False, stream=None):
    """the device entry point on torch copies of f; returns (custom, custom_count, needed, status) as numpy"""
    t = lambda x: None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    R = len(f["pose"])
    S = R if S is None else S
    custom = t(f["custom"].view(np.uint8))
    cc = t(np.full(S, -7, np.int32) if custom_count is None else custom_count)
    need, st = torch.full((R,), -9, dtype=torch.int32, device=DEV), torch.full((R,), -9, dtype=torch.int32, device=DEV)
    keep = dict(pose=t(f["pose"]), cmd=t(f["last_cmd"]), rad=t(np.broadcast_to(f["radius"], (R,))),
                world=t(f.get("world")), scene=t(scene), own=t(f.get("own_count")))
    fa = abi.make_fleet_args(R, S, f["custom"].shape[1], max_rows, rng, pose=keep["pose"], last_cmd=keep["cmd"],
                             radius=keep["rad"], world=keep["world"], scene=keep["scene"], own_count=keep["own"],
                             custom=custom if custom.numel() else None, custom_count=cc, needed=need, status=st)
    outs = []
    for _ in range(2 if twice else 1):
        g.fleet_obstacles_device(fa, stream=stream)
        torch.cuda.synchronize()
        outs.append((custom.cpu().numpy().copy().view(abi.OBST_DTYPE).reshape(f["custom"].shape), cc.cpu().numpy().copy(),
                     need.cpu().numpy().copy(), st.cpu().numpy().copy()))
    if twice:
        for a, b in zip(*outs):
            assert a.tobytes() == b.tobytes(), "a second call changed the rows"
    return outs[-1]


def assert_like_restatement(got, f, rng, max_rows, scene=None, custom_count=None, label=""):
    want = fc.restate(f["pose"], f["last_cmd"], f["radius"], rng, max_rows, f["custom"], f.get("own_count"),
                      custom_count, f.get("world"), scene)
    (gc, gcc, gn, gs), (wc, wcc, wn, ws) = got, want
    assert np.array_equal(gn, wn), f"{label}: needed"
    assert np.array_equal(gs, ws), f"{label}: status"
    assert np.array_equal(gcc, wcc), f"{label}: custom_count"
    # everything but the velocities bit for bit (own rows and rows past the written ones included)
    a, b = gc.copy(), wc.copy()
    for key in ("vx", "vy"):
        same = a[key].view(np.uint64) == b[key].view(np.uint64)
        with np.errstate(invalid="ignore"):
            assert (same | (np.abs(a[key] - b[key]) <= 1e-12)).all(), f"{label}: {key}"
        a[key], b[key] = 0, 0
    assert a.tobytes() == b.tobytes(), f"{label}: rows"
    return want


@pytest.mark.parametrize("R,max_rows,clustered", [(1, 8, True), (33, 1, True), (700, 8, True), (700, 32, False),
                                                  (2000, 0, True), (MAX_R, 8, True), (MAX_R, 32, False)])
def test_random_fleets_match_the_restatement(gpu, R, max_rows, clustered):
    f = random_fleet(R, R, 24, seed=R + max_rows, clustered=clustered)
    seen = set()
    for rng in (0.0, 1.5, 6.0):
        got = run_device(gpu, f, rng, max_rows, twice=True)
        want = assert_like_restatement(got, f, rng, max_rows, label=f"R={R} range={rng}")
        seen |= set(want[3].tolist())
        if R > 1 and rng == 6.0:
            assert (want[2] > 0).any()
    if R >= 700 and max_rows:
        assert {fc.TRUNCATED, fc.WRITTEN} <= seen


def test_scenes_given_and_the_scenes_no_robot_writes(gpu):
    R, S = 1500, 1600
    f = random_fleet(R, S, 12, seed=5)
    rng = np.random.default_rng(6)
    scene = rng.permutation(S)[:R].astype(np.int32)
    cc0 = np.full(S, 77, np.int32)
    got = run_device(gpu, f, 4.0, 8, scene=scene, S=S, custom_count=cc0, twice=True)
    assert_like_restatement(got, f, 4.0, 8, scene=scene, custom_count=cc0, label="scenes")
    assert (got[1][np.setdiff1d(np.arange(S), scene)] == 77).all()


def test_bad_and_shared_scenes_on_the_device(gpu):
    R, S = 300, 300
    f = random_fleet(R, S, 10, seed=8)
    scene = np.arange(R, dtype=np.int32)
    scene[5] = -1
    scene[6] = S
    scene[7] = scene[8] = 20                           # robots 7 and 8 share scene 20; robot 20 takes scene 7
    scene[20] = 7
    f["own_count"][30] = 11                            # outside 0 .. C_cap
    cc0 = np.full(S, 5, np.int32)
    got = run_device(gpu, f, 5.0, 8, scene=scene, S=S, custom_count=cc0)
    want = assert_like_restatement(got, f, 5.0, 8, scene=scene, custom_count=cc0, label="bad scenes")
    st = want[3]
    assert st[5] == st[6] == st[30] == fc.BAD_INPUT and st[7] == st[8] == fc.SHARED_SCENE
    assert (got[2][[5, 6, 7, 8, 30]] == -1).all()


def test_the_hand_cases_on_the_device(gpu):
    below = math.nextafter(0.001, 0.0)
    cases = [
        dict(pose=[(0.0, 0.0, 0.0), (3.0, 4.0, 0.0), (3.0, 4.000000000001, 0.0)], rng=5.0, max_rows=8, C=4),
        dict(pose=[(0.0, 0.0, 0.0), (0.0, 1.0, 0.0), (-1.0, 0.0, 0.0), (1.0, 0.0, 0.0), (0.0, -1.0, 0.0)], rng=1.0,
             max_rows=2, C=8),
        dict(pose=[(1.5, -2.0, 0.3), (1.5, -2.0, 2.0)], rng=0.0, max_rows=4, C=4),
        dict(pose=[(0.0, 0.0, 0.0), (0.1, 0.0, 0.0), (0.05, 0.0, 0.0)], rng=10.0, max_rows=8, C=4, world=[7, 7, 3],
             own=[1, 0, 2]),
        dict(pose=[(0.0, 0.0, 0.0)] + [(0.5 * k, 0.0, 0.0) for k in range(1, 7)], rng=100.0, max_rows=4, C=5,
             own=[3, 0, 0, 0, 0, 0, 0]),
        dict(pose=[(0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (2.0, 0.0, 0.0)], rng=10.0, max_rows=8, C=4,
             cmd=[(0.0, 0.0, 0.0), (0.001, 0.0, 0.5), (below, 0.0, 0.0)]),
        dict(pose=[(0.0, 0.0, 0.0), (1.0, 1.0, math.pi / 2)], rng=10.0, max_rows=8, C=1,
             cmd=[(0.0, 0.0, 0.0), (0.4, 0.1, 0.0)]),
    ]
    for k, c in enumerate(cases):
        R = len(c["pose"])
        custom = np.zeros((R, c["C"]), abi.OBST_DTYPE)
        custom.view(np.uint8)[:] = 0xAB
        f = dict(pose=np.array(c["pose"]), last_cmd=np.array(c.get("cmd", np.zeros((R, 3)))), radius=np.full(R, 0.2),
                 custom=custom, world=None if "world" not in c else np.array(c["world"], np.int32),
                 own_count=None if "own" not in c else np.array(c["own"], np.int32))
        got = run_device(gpu, f, c["rng"], c["max_rows"], twice=True)
        want = assert_like_restatement(got, f, c["rng"], c["max_rows"], label=f"case {k}")
        if k == 5:
            assert got[0][0, 0]["dynamic"] == 1 and got[0][0, 0]["vx"] == 0.001 and got[0][0, 1]["dynamic"] == 0
        if k == 6:
            assert abs(got[0][0, 0]["vx"] + 0.1) <= 1e-16 and got[0][0, 0]["vy"] == 0.4


def test_host_and_device_entry_points_give_the_same_bits(gpu):
    R, S = 900, 950
    f = random_fleet(R, S, 16, seed=11)
    scene = np.random.default_rng(12).permutation(S)[:R].astype(np.int32)
    cc0 = np.full(S, 3, np.int32)
    dev = run_device(gpu, f, 3.0, 8, scene=scene, S=S, custom_count=cc0)
    host = gpu.fleet_obstacles(f["pose"], f["last_cmd"], f["radius"], f["custom"], 3.0, 8, own_count=f["own_count"],
                               custom_count=cc0, world=f["world"], scene=scene)
    for a, b, name in zip(dev, host, ("custom", "custom_count", "needed", "status")):
        assert a.tobytes() == b.tobytes(), name
    assert gpu.last_fleet_grid() == (R + 15) // 16


def test_argument_errors_launch_nothing(gpu):
    f = random_fleet(10, 10, 4, seed=2)
    call = lambda **kw: gpu.fleet_obstacles(**{**dict(pose=f["pose"], last_cmd=f["last_cmd"], radius=f["radius"],
                                                      custom=f["custom"], range=1.0, max_rows=8), **kw})
    call()
    bad_pose = f["pose"].copy()
    bad_pose[3, 1] = np.nan
    for kw in (dict(max_rows=33), dict(max_rows=-1), dict(range=-1.0), dict(range=float("nan")), dict(pose=bad_pose),
               dict(radius=-0.1), dict(scene=np.full(10, 2, np.int32)), dict(scene=np.arange(1, 11, dtype=np.int32)),
               dict(own_count=np.full(10, 5, np.int32)), dict(custom=f["custom"][:5])):
        with pytest.raises(T.TebGpuError):
            call(**kw)


# ---- the fleet loop on one stream
def _raster(B, centre, kind):
    """each robot's 60 x 60 costmap (0.05 m) centred at `centre`: one-cell LETHAL walls 0.8 m either side of a corridor
    along x (kind "corridor"), or around a cross of two such corridors (kind "junction"); kind "random": the scenes
    module's rasters"""
    if kind == "random":
        r = scenes.costmap_raster(B, 60, 60, 0.05, 0.02, seed=31)
        r["origin"][:, :2] = centre - 1.5
        return r
    sx = sy = 60
    res = 0.05
    cost = np.zeros((B, sx * sy), np.uint8)
    origin = np.zeros((B, 3))
    for b in range(B):
        ox, oy = centre[b] - 1.5
        origin[b] = (ox, oy, res)
        wx = ox + (np.arange(sx) + 0.5) * res
        wy = oy + (np.arange(sy) + 0.5) * res
        X, Y = np.meshgrid(wx, wy)                          # row my, column mx
        line = lambda v: (np.abs(v) >= 0.8) & (np.abs(v) < 0.85)
        wall = line(Y)
        if kind == "junction":
            wall = (line(Y) & (np.abs(X) >= 0.8)) | (line(X) & (np.abs(Y) >= 0.8))
        cost[b] = np.where(wall, abi.COSTMAP_LETHAL, 0).astype(np.uint8).ravel()
    return dict(cost=cost, grid=np.tile(np.array([sx, sy], np.int32), (B, 1)), origin=origin)


def _straight_plans(start, goal, G_cap, spacing=0.05):
    B = len(start)
    gp = np.full((B, G_cap, 3), np.nan)
    end = np.zeros(B, np.int32)
    for b in range(B):
        d = goal[b] - start[b]
        L = float(np.hypot(*d))
        k = min(G_cap, int(L / spacing) + 1)
        s = np.linspace(0.0, 1.0, k)
        gp[b, :k, 0] = start[b, 0] + s * d[0]
        gp[b, :k, 1] = start[b, 1] + s * d[1]
        gp[b, :k, 2] = math.atan2(d[1], d[0])
        end[b] = k
    return gp, np.zeros(B, np.int32), end


def _scenario(kind):
    if kind == "corridor":              # two robots head-on, 3 m apart
        start, goal = np.array([[-1.5, 0.05], [1.5, -0.05]]), np.array([[3.0, 0.05], [-3.0, -0.05]])
    elif kind == "junction":            # four robots crossing at the centre
        start = np.array([[-1.5, 0.1], [1.5, -0.1], [0.1, 1.5], [-0.1, -1.5]])
        goal = -3.0 * start / 1.5
    else:                               # 24 robots on a 6 x 4 grid, goals across the block
        rng = np.random.default_rng(41)
        start = np.array([[0.9 * i - 2.25, 0.9 * j - 1.35] for i in range(6) for j in range(4)])
        start += rng.uniform(-0.1, 0.1, start.shape)
        goal = -start + rng.uniform(-0.3, 0.3, start.shape)
    G_cap = 256
    gp, begin, end = _straight_plans(start, goal, G_cap)
    robot = np.column_stack([start, gp[:, 0, 2]])
    return dict(gp=gp, begin=begin, end=end, robot=robot, G_cap=G_cap, raster=_raster(len(start), start, kind))


def _fleet_loop(kind, restated, cycles=20, n_cap=96, P_cap=128, M_cap=2048, Lb=10, max_rows=8, rng=3.0,
                dev_trace=None, graph_at=None):
    """restated=False: fleet obstacles -> costmap_tf -> local_plan_tf -> backup modes -> plan -> costmap check ->
    finish on one stream. True: the same loop with the neighbour rows built on the host by the restatement from the
    device's poses and last_cmd, uploaded in the fleet step's place; a restated velocity within 1e-12 of the device's
    at the same cycle is replaced by the device's bits, so both loops see the same inputs wherever the bars hold."""
    sc = _scenario(kind)
    B = len(sc["robot"])
    C_cap = 1 + max_rows
    r = sc["raster"]
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 1
    p.max_vel_trans = p.max_vel_x
    p.global_plan_overwrite_orientation = 1
    g = T.TebGpu(B, n_cap, B, M_cap, 0)
    g.set_params(p)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=DEV)
    f64, i32 = torch.float64, torch.int32
    cost, grid, origin = t(r["cost"]), t(r["grid"]), t(r["origin"])
    robot = t(sc["robot"].copy())
    radius = t(np.full(B, 0.25))
    own_rows = np.zeros((B, C_cap), abi.OBST_DTYPE)     # one static point of the caller's own per scene, far behind
    own_rows[:, 0]["x"], own_rows[:, 0]["y"] = sc["robot"][:, 0] - 5.0, sc["robot"][:, 1] + 5.0
    custom, ccount, own = t(own_rows.view(np.uint8)), t(np.ones(B, np.int32)), t(np.ones(B, np.int32))
    ident = t(np.tile(IDENTITY, (B, 1)))
    obst, ocount = z(B * M_cap * 64, torch.uint8), z(B, i32)
    gpd, begin, end = t(sc["gp"]), t(sc["begin"]), t(sc["end"])
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
    fneed, fstat = z(B, i32), z(B, i32)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, B, M_cap, 0, 0
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
    bs.vel_start, bs.vel_goal, bs.prefer_rotdir = vstart.data_ptr(), vgoal.data_ptr(), state["prefer_rotdir"].data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = costo.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = B, r["cost"].shape[1], M_cap, C_cap, 1
    ca.behind_robot_dist = 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.custom, ca.custom_count = custom.data_ptr(), ccount.data_ptr()
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    cframes = abi.make_frame_args(custom_to_costmap=ident.data_ptr())
    pframes = abi.make_frame_args(costmap_to_plan=ident.data_ptr(), plan_to_costmap=ident.data_ptr())
    la = abi.make_local_plan_args(sc["G_cap"], P_cap, 0, max_lookahead_dist=2.0, global_plan=gpd.data_ptr(),
                                  plan_begin=begin.data_ptr(), plan_end=end.data_ptr(), robot=robot.data_ptr(),
                                  robot_vel=vel.data_ptr(), grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  infeasible_count=state["infeasible_count"].data_ptr(), since_infeasible=since.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), goal_idx=gidx.data_ptr(),
                                  result=result.data_ptr(), needed=needed.data_ptr())
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    fa = abi.make_feasibility_args(0.1, max_queries=512, feasible=feas.data_ptr(), query_count=qc.data_ptr())
    world = abi.make_costmap_world(r["cost"].shape[1], cost.data_ptr(), grid.data_ptr(), origin.data_ptr())
    fl = abi.make_fleet_args(B, B, C_cap, max_rows, rng, pose=robot, last_cmd=state["last_cmd"], radius=radius,
                             own_count=own, custom=custom, custom_count=ccount, needed=fneed, status=fstat)
    cs = dict(buffer_length=Lb, oscillation_recovery_min_duration=2.0)
    dt, now = 0.2, 1000.0
    s = torch.cuda.Stream()
    trace, graph = [], None
    for k in range(cycles):
        cy = abi.make_cycle_args(now, L_cap=Lb, **cs, local_plan_result=result.data_ptr(), robot_vel=vel.data_ptr(),
                                 cmd=cmd.data_ptr(), feasible=feas.data_ptr(), cmd_vel=cmd_vel.data_ptr(),
                                 outcome=outcome.data_ptr(), oscillating=osc.data_ptr(),
                                 **{kk: state[kk].data_ptr() for kk in abi.CYCLE_STATE})
        with torch.cuda.stream(s):
            since.copy_(now - state["last_infeasible"])
            if restated:
                s.synchronize()
                cur = custom.cpu().numpy().view(abi.OBST_DTYPE).reshape(B, C_cap).copy()
                hc, hcc, hn, hs = fc.restate(robot.cpu().numpy(), state["last_cmd"].cpu().numpy(), np.full(B, 0.25), rng,
                                             max_rows, cur, np.ones(B, np.int32))
                dc = dev_trace[k]["custom"].view(abi.OBST_DTYPE).reshape(B, C_cap)
                for key in ("vx", "vy"):
                    assert np.abs(hc[key] - dc[key]).max() <= 1e-12, (k, key)
                    hc[key] = dc[key]
                custom.copy_(t(hc.view(np.uint8).reshape(B, -1)))
                ccount.copy_(t(hcc))
                fneed.copy_(t(hn))
                fstat.copy_(t(hs))
            else:
                g.fleet_obstacles_device(fl, stream=s.cuda_stream)
            g.costmap_obstacles_device(ca, stream=s.cuda_stream, frames=cframes)
            g.local_plan_device(bs, la, stream=s.cuda_stream, frames=pframes)
            g.backup_modes_device(bs, cy, stream=s.cuda_stream)
            g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, path=path,
                          stream=s.cuda_stream)
            g.check_feasible_costmap_device(bs, fa, world, stream=s.cuda_stream)
            g.finish_cycle_device(bs, cy, stream=s.cuda_stream)
        s.synchronize()
        if graph_at == k:                              # on a context of its own, so the loop's context is the restated one's
            hb = abi.HostBatch(poses.cpu().numpy(), n.cpu().numpy(),
                               obst.cpu().numpy().view(abi.OBST_DTYPE).reshape(B, M_cap), ocount.cpu().numpy(),
                               scene_id=np.arange(B, dtype=np.int32), vel_start=vs, vel_goal=vs,
                               prefer_rotdir=state["prefer_rotdir"].cpu().numpy())
            g2 = T.TebGpu(B, n_cap, B, M_cap, 0)
            g2.set_params(p)
            graph = (hb, g2.build_system(hb, graph=True))
            g2.close()
        with torch.cuda.stream(s):
            th = robot[:, 2].clone()
            robot[:, 0] += (cmd_vel[:, 0] * torch.cos(th) - cmd_vel[:, 1] * torch.sin(th)) * dt
            robot[:, 1] += (cmd_vel[:, 0] * torch.sin(th) + cmd_vel[:, 1] * torch.cos(th)) * dt
            robot[:, 2] += cmd_vel[:, 2] * dt
            vel.copy_(cmd_vel)
        s.synchronize()
        rec = dict(custom=custom, ccount=ccount, fneed=fneed, fstat=fstat, obst=obst, ocount=ocount, plan=plan,
                   pcount=pcount, result=result, begin=begin, n=n, poses=poses, status=status, path=path, cmd=cmd,
                   cmd_vel=cmd_vel, outcome=outcome, oscillating=osc, feasible=feas, robot=robot, **state)
        rec = {kk: v.cpu().numpy().copy() for kk, v in rec.items()}
        rec["plan"] = np.concatenate([rec["plan"][b, :rec["pcount"][b]] for b in range(B)])   # the rows written
        trace.append(rec)
        now += dt
    g.close()
    return trace, graph, own_rows


@pytest.mark.parametrize("kind", ["corridor", "junction", "random"])
def test_fleet_loop_matches_the_loop_fed_host_neighbour_rows(kind):
    dev, graph, own_rows = _fleet_loop(kind, False, graph_at=3)
    ref, _, _ = _fleet_loop(kind, True, dev_trace=dev)
    for k, (x, y) in enumerate(zip(dev, ref)):
        for key in x:
            assert x[key].tobytes() == y[key].tobytes(), (kind, k, key)
    B = len(own_rows)
    for c in dev:                                       # the caller's own row stays, the robots see each other
        rows = c["custom"].view(abi.OBST_DTYPE).reshape(B, -1)
        assert rows[:, 0].tobytes() == own_rows[:, 0].tobytes()
        assert (c["ccount"] >= 1).all() and (c["fstat"] >= 0).all() and (c["fstat"] <= 1).all()
    assert any((c["ccount"] > 1).all() for c in dev)
    moving = [c for c in dev if (c["custom"].view(abi.OBST_DTYPE).reshape(B, -1)[:, 1:]["dynamic"] == 1).any()]
    assert moving, "no neighbour row was ever dynamic"
    assert sum((c["outcome"] == abi.TEB_CYCLE_COMMAND).sum() for c in dev) > 0

    # the dynamic neighbour rows give dynamic-obstacle edges: every interior pose of a band whose scene holds one has a
    # time (one edge per dynamic row), and the dynamic rows take no static association bit
    hb, gr = graph
    seen = 0
    for b in range(B):
        nb, cnt = int(hb.n[b]), int(hb.obst_count[b])
        if nb < 3:
            continue
        rows = hb.obstacles[b, :cnt]
        dyn = np.nonzero(rows["dynamic"] == 1)[0]
        inner = gr["dyn_t"][b, 1:nb - 1]
        if len(dyn):
            seen += 1
            assert np.isfinite(inner).all(), (kind, b)
            words = gr["assoc"][b, :nb]
            for l in dyn:
                assert not ((words[:, l // 64] >> np.uint64(l % 64)) & np.uint64(1)).any(), (kind, b, l)
    assert seen > 0, "no band of the graph cycle had a dynamic neighbour row"
