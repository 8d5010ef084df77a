"""Every robot's local plan, goal and via-points from its global plan on the device (tebgpu_local_plan / _device,
teb_local_plan.cuh), held to the restatement of tests/local_plan_cases.py: plan_begin, goal_idx, plan_count, result,
needed, every x / y and stored yaw, and the via rows and counts bit equal; a goal heading that passes through the
device's trig within 1e-12. Also host bits == device bits, batch-position invariance, untouched rows past the counts, the
capacity and bad-input codes, argument errors that launch nothing, and a costmap -> local plan -> plan -> check cycle on
one stream."""
import ctypes as C
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import local_plan_cases as lp

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
SENTINEL = 0xA5
SCALARS = ("prune_distance", "max_lookahead_dist", "viapoint_sep", "xy_goal_tolerance", "yaw_goal_tolerance",
           "trans_stopped_vel", "theta_stopped_vel", "shrink_horizon_min_duration", "free_goal_vel",
           "complete_global_plan", "shrink_horizon_backup")


def _ctx(overwrite, B=256, S=64, V=64):
    g = T.TebGpu(B, 64, S, 64, V)
    p = abi.default_params()
    p.global_plan_overwrite_orientation = int(overwrite)
    g.set_params(p)
    return g


@pytest.fixture(scope="module", params=[True, False], ids=["overwrite", "stored_yaw"])
def gpu(request):
    g = _ctx(request.param)
    g.overwrite = request.param
    yield g
    g.close()


class Fleet:
    """B bands packed as TebLocalPlanArgs wants them"""

    def __init__(self, gp, begin, end, robot, vel, grid, origin, sid, inf=None, since=None, custom_via=None):
        self.gp = np.ascontiguousarray(gp, np.float64)
        self.B, self.G = self.gp.shape[:2]
        self.begin, self.end = np.asarray(begin, np.int32), np.asarray(end, np.int32)
        self.robot, self.vel = np.asarray(robot, np.float64).reshape(-1, 3), np.asarray(vel, np.float64).reshape(-1, 3)
        self.grid, self.origin = np.asarray(grid, np.int32).reshape(-1, 2), np.asarray(origin, np.float64).reshape(-1, 3)
        self.sid = np.asarray(sid, np.int32)
        self.inf = None if inf is None else np.asarray(inf, np.int32)
        self.since = None if since is None else np.asarray(since, np.float64)
        self.custom_via = None if custom_via is None else np.asarray(custom_via, np.int32)

    @staticmethod
    def of(d, **kw):
        return Fleet(d["global_plan"], d["plan_begin"], d["plan_end"], d["robot"], d["robot_vel"], d["grid"],
                     d["origin"], d["scene_id"], **kw)

    def expect(self, a, P_cap, V_cap, own_via):
        out = []
        for b in range(self.B):
            s = self.sid[b]
            cv = None if own_via else (0 if self.custom_via is None else int(self.custom_via[b]))
            out.append(lp.restate(self.gp[b], int(self.begin[b]), int(self.end[b]), self.robot[b], self.vel[b],
                                  tuple(int(v) for v in self.grid[s]), float(self.origin[s, 2]), a, cv,
                                  None if self.inf is None else int(self.inf[b]),
                                  None if self.since is None else float(self.since[b]), P_cap, V_cap))
        return out

    def subset(self, idx):
        idx = np.asarray(idx)
        pick = lambda x: None if x is None else x[idx]
        return Fleet(self.gp[idx], self.begin[idx], self.end[idx], self.robot[idx], self.vel[idx], self.grid,
                     self.origin, self.sid[idx], pick(self.inf), pick(self.since), pick(self.custom_via))


def _outs(B, P_cap, V_cap, own_via, custom_via=None):
    plan = np.zeros((B, P_cap, 3))
    plan.view(np.uint8)[...] = SENTINEL
    via = None
    if own_via:
        via = np.zeros((B, max(V_cap, 1), 2))
        via.view(np.uint8)[...] = SENTINEL
    vc = np.full(B, 77, np.int32) if custom_via is None else custom_via.copy()
    return dict(plan=plan, plan_count=np.full(B, 77, np.int32), goal_idx=np.full(B, 77, np.int32), via=via,
                via_count=vc, result=np.full(B, 77, np.int32), needed=np.full((B, 2), 77, np.int32))


def _args(f, a, P_cap, V_cap, ptr, ins, outs):
    la = abi.make_local_plan_args(f.G, P_cap, V_cap, **{k: getattr(a, k) for k in SCALARS})
    la.global_plan, la.plan_begin, la.plan_end = ptr(ins["gp"]), ptr(ins["begin"]), ptr(ins["end"])
    la.robot, la.robot_vel, la.grid, la.origin = ptr(ins["robot"]), ptr(ins["vel"]), ptr(ins["grid"]), ptr(ins["origin"])
    la.infeasible_count, la.since_infeasible = ptr(ins["inf"]), ptr(ins["since"])
    for k in ("plan", "plan_count", "goal_idx", "via", "via_count", "result", "needed"):
        setattr(la, k, ptr(outs[k]))
    return la


def _batch(f, ptr, sid):
    bs = abi.TebBatch()
    bs.B, bs.S, bs.scene_id = f.B, f.grid.shape[0], ptr(sid)
    return bs


def _inputs(f):
    return dict(gp=f.gp, begin=f.begin.copy(), end=f.end, robot=f.robot, vel=f.vel, grid=f.grid, origin=f.origin,
                inf=f.inf, since=f.since)


def run_host(g, f, a, P_cap, V_cap, own_via=True):
    ins, outs = _inputs(f), _outs(f.B, P_cap, V_cap, own_via, f.custom_via)
    la = _args(f, a, P_cap, V_cap, abi.ptr, ins, outs)
    if not own_via and f.custom_via is None:
        la.via_count = None
    rc = g.lib.tebgpu_local_plan(g.ctx, C.byref(_batch(f, abi.ptr, f.sid)), C.byref(la))
    assert rc == 0, g.lib.tebgpu_last_error_string(g.ctx)
    outs["plan_begin"] = ins["begin"]
    return outs


def _dev(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).to(DEV)


def run_device(g, f, a, P_cap, V_cap, own_via=True, stream=None):
    ins_h, outs_h = _inputs(f), _outs(f.B, P_cap, V_cap, own_via, f.custom_via)
    ins = {k: _dev(v) for k, v in ins_h.items()}
    outs = {k: _dev(v) for k, v in outs_h.items()}
    ptr = lambda t: None if t is None else t.data_ptr()
    la = _args(f, a, P_cap, V_cap, ptr, ins, outs)
    if not own_via and f.custom_via is None:
        la.via_count = None
    sid = _dev(f.sid)
    g.local_plan_device(_batch(f, ptr, sid), la, stream=torch.cuda.current_stream().cuda_stream if stream is None else stream)
    torch.cuda.synchronize()
    back = {k: None if v is None else v.cpu().numpy().view(outs_h[k].dtype).reshape(outs_h[k].shape)
            for k, v in outs.items()}
    back["plan_begin"] = ins["begin"].cpu().numpy().view(np.int32)
    return back


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def _ang(a, b):
    return abs(math.remainder(a - b, 2 * math.pi))


def assert_outputs(out, want, a, overwrite, own_via, label=""):
    """out: one entry point's arrays; want: the restatement's rows, band by band"""
    for b, w in enumerate(want):
        lab = (label, b, w.result)
        assert out["result"][b] == w.result, lab
        assert out["plan_begin"][b] == w.plan_begin, lab
        if w.result in (lp.EMPTY, lp.BAD_INPUT):
            assert out["plan_count"][b] == 0 and out["goal_idx"][b] == 77 and (out["needed"][b] == 77).all(), lab
        else:
            assert out["goal_idx"][b] == w.goal_idx and tuple(out["needed"][b]) == w.needed, lab
        k = len(w.plan)
        assert out["plan_count"][b] == k, lab
        if k:
            got, ref = out["plan"][b, :k], np.array(w.plan)
            if overwrite:   # the goal heading may pass through trig: the device's, not glibc's
                assert _ang(got[-1, 2], ref[-1, 2]) <= 1e-12, (lab, got[-1, 2], ref[-1, 2])
                got, ref = got.copy(), ref.copy()
                got[-1, 2] = ref[-1, 2] = 0.0
            assert _bytes(got) == _bytes(ref), lab
        assert (out["plan"][b, k:].view(np.uint8) == SENTINEL).all(), lab
        if own_via:
            if w.via is None:
                assert out["via_count"][b] == 77, lab
                nv = 0
            else:
                nv = len(w.via)
                assert out["via_count"][b] == nv, lab
                if nv:
                    assert _bytes(out["via"][b, :nv]) == _bytes(np.array(w.via)), lab
            assert (out["via"][b, nv:].view(np.uint8) == SENTINEL).all(), lab


def both(g, f, a, P_cap, V_cap, own_via=True):
    h = run_host(g, f, a, P_cap, V_cap, own_via)
    d = run_device(g, f, a, P_cap, V_cap, own_via)
    for k in h:
        if h[k] is not None:
            assert _bytes(h[k]) == _bytes(d[k]), k                               # host bits == device bits
    return d


def _args_for(g, **kw):
    return lp.Args(**{"overwrite_orientation": g.overwrite, **kw})


HAND = [  # (rows, robot, begin, vel, Args overrides) one band each, the CPU cases' boundaries
    ([(float(x), 0.0, 0.0) for x in range(7)], (0.0, 0.0, 0.0), 0, (1.0, 0, 0), dict(max_lookahead_dist=0.0)),
    ([(float(x), 0.0, 0.0) for x in (0, 1, 2, 3, 4.25, 5, 6)], (0.0, 0.0, 0.0), 0, (1.0, 0, 0), dict(max_lookahead_dist=0.0)),
    ([(float(x), 0.0, 0.1 * x) for x in range(6)], (2.0, 0.0, 0.0), 0, (1.0, 0, 0), dict(prune_distance=2.5)),
    ([(float(x), 0.0, 0.0) for x in range(4)], (1.0, 0.0, 0.0), 0, (1.0, 0, 0), dict()),
    ([(0.1, 0.0, 0.0), (0.5, 0.0, 0.0), (1.0, 0.0, 0.0), (1.0, 1.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 0.0)], (0.0, 0.0, 0.0), 0,
     (1.0, 0, 0), dict(max_lookahead_dist=0.0)),
    ([(0.152, 0.164, 0.0), (1.0, 0.0, 0.0), (0.3, 0.0, 0.0), (0.2, 0.0, 0.0), (2.0, 0.0, 0.0)], (0.0, 0.0, 0.0), 0, (1.0, 0, 0),
     dict(prune_distance=2.0, max_lookahead_dist=0.0)),
    ([(0.1, 0.0, 0.0), (-0.1, 0.0, 0.0), (0.05, 0.0, 0.0), (1.0, 0.0, 0.0), (0.0, 0.0, 0.0)], (0.0, 0.0, 0.0), 0, (1.0, 0, 0),
     dict(max_lookahead_dist=0.0)),
    ([(2e5, 0.0, 0.0), (3e5, 0.0, 0.0)], (0.0, 0.0, 0.0), 0, (1.0, 0, 0), dict()),
    ([(float(x) * 0.5, 0.0, 0.0) for x in range(5)], (0.0, 0.0, 0.0), 0, (1.0, 0, 0), dict(viapoint_sep=0.5, max_lookahead_dist=0)),
    ([(-0.5, 0.0, 0.0), (0.25, 0.0, 0.0)], (0.0, 0.0, 0.0), 0, (0.0, 0, 0), dict(xy_goal_tolerance=0.25)),
    ([(-0.5, 0.0, 0.0), (0.25, 0.0, 0.0)], (0.0, 0.0, 0.0), 0, (0.1, -0.1, 0.1), dict(xy_goal_tolerance=0.2500001)),
    ([(-0.5, 0.0, 0.0), (0.25, 0.0, 0.0)], (0.0, 0.0, -0.2), 0, (0.0, 0, 0), dict(xy_goal_tolerance=1.0)),
    ([(-0.5, 0.0, 0.0), (0.0, 0.0, 0.0), (0.25, 0.0, 0.0)], (0.0, 0.0, 0.0), 0, (0.0, 0, 0),
     dict(xy_goal_tolerance=1.0, viapoint_sep=0.1, complete_global_plan=False)),
    ([(float(x), 0.0, 0.1 * x) for x in range(8)], (0.0, 0.0, 0.0), 0, (1.0, 0, 0), dict(max_lookahead_dist=4.0)),
    ([(0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (2.0, 0.0, 0.0), (2.0, 1.0, 0.0), (3.0, 2.0, 0.0), (3.0, 4.0, 0.0), (9.0, 9.0, 0.0)],
     (0.0, 0.0, 0.0), 0, (1.0, 0, 0), dict()),
    ([(0.5, 0.5, 0.25)], (0.0, 0.1, -1.0), 0, (1.0, 0, 0), dict()),
    ([(0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (math.nan, 0.0, 0.0), (3.0, 0.0, 0.0)], (0.0, 0.0, 0.0), 0, (1.0, 0, 0),
     dict(max_lookahead_dist=0.0)),
    ([(0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (2.0, 0.0, 0.0)], (math.nan, 0.0, 0.0), 1, (1.0, 0, 0), dict()),
    ([(0.0, 0.0, 0.0), (1.0, 0.0, 0.0)], (0.0, 0.0, 0.0), 2, (1.0, 0, 0), dict()),
]


@pytest.mark.parametrize("k", range(len(HAND)))
def test_hand_cases(gpu, k):
    rows, robot, begin, vel, kw = HAND[k]
    G = 8
    gp = np.full((1, G, 3), np.nan)
    gp[0, :len(rows)] = rows
    f = Fleet(gp, [begin], [len(rows)], [robot], [vel], [(40, 40)], [(0.0, 0.0, 0.25)], [0], inf=[3], since=[0.0])
    a = _args_for(gpu, **kw)
    out = both(gpu, f, a, 8, 8)
    assert_outputs(out, f.expect(a, 8, 8, True), a, gpu.overwrite, True, k)
    assert gpu.last_local_plan_grid() == 1


ARGSETS = [dict(), dict(viapoint_sep=0.3), dict(max_lookahead_dist=0.0, viapoint_sep=0.05),
           dict(max_lookahead_dist=3.0, prune_distance=0.5), dict(xy_goal_tolerance=0.6, yaw_goal_tolerance=0.5),
           dict(xy_goal_tolerance=0.6, yaw_goal_tolerance=0.5, free_goal_vel=True, viapoint_sep=0.2,
                complete_global_plan=False)]


@pytest.mark.parametrize("G_cap", [64, 512, 4096])
@pytest.mark.parametrize("j", range(len(ARGSETS)))
def test_random_fleets_match_the_restatement(gpu, G_cap, j):
    B = 64 if G_cap == 4096 else 128
    d = scenes.global_plans(B, G_cap, S=4, seed=G_cap + j)
    f = Fleet.of(d)
    a = _args_for(gpu, **ARGSETS[j])
    P_cap, V_cap = G_cap + 1, 64
    out = both(gpu, f, a, P_cap, V_cap)
    want = f.expect(a, P_cap, V_cap, True)
    assert_outputs(out, want, a, gpu.overwrite, True, (G_cap, j))
    res = np.array([w.result for w in want])
    print(G_cap, j, {r: int((res == r).sum()) for r in range(5)})
    assert (res == lp.PLANNED).any()


def test_results_do_not_depend_on_the_band_position(gpu):
    d = scenes.global_plans(96, 1024, S=4, seed=5)
    f = Fleet.of(d, inf=np.arange(96) % 12, since=np.linspace(0, 20, 96))
    a = _args_for(gpu, viapoint_sep=0.25)
    ref = run_device(gpu, f, a, 1025, 64)
    perm = np.random.default_rng(2).permutation(96)
    out = run_device(gpu, f.subset(perm), a, 1025, 64)
    for k in ref:
        assert _bytes(ref[k][perm]) == _bytes(out[k]), k
    one = run_host(gpu, f.subset([perm[0]]), a, 1025, 64)
    for k in ref:
        assert _bytes(ref[k][perm[:1]]) == _bytes(one[k]), k


def test_custom_via_points(gpu):
    d = scenes.global_plans(64, 256, S=2, seed=9)
    cv = (np.arange(64) % 3).astype(np.int32)
    a = _args_for(gpu, xy_goal_tolerance=0.6, yaw_goal_tolerance=0.5, free_goal_vel=True, viapoint_sep=0.2)
    for custom in (cv, None):
        f = Fleet.of(d, custom_via=custom)
        out = both(gpu, f, a, 257, 0, own_via=False)
        want = f.expect(a, 257, 0, False)
        assert_outputs(out, want, a, gpu.overwrite, False)
        if custom is not None:
            assert (out["via_count"] == cv).all()                                # read, never written


def test_capacity_and_bad_input_on_the_device(gpu):
    d = scenes.global_plans(32, 512, S=2, seed=3)
    f = Fleet.of(d)
    a = _args_for(gpu, max_lookahead_dist=0.0, viapoint_sep=0.05)
    want = f.expect(a, 40, 8, True)
    assert any(w.result == lp.CAPACITY for w in want) and any(w.result == lp.PLANNED for w in want)
    out = both(gpu, f, a, 40, 8)
    assert_outputs(out, want, a, gpu.overwrite, True)
    bad = Fleet.of(d)
    bad.begin[1], bad.end[2], bad.sid[3] = 600, 513, 2
    bad.begin[4], bad.end[4] = 10, 9
    bad.begin[5] = -1
    out = run_device(gpu, bad, a, 40, 8)
    for b in range(32):
        if b in (1, 2, 3, 4, 5):
            assert out["result"][b] == lp.BAD_INPUT and out["plan_count"][b] == 0
            assert out["goal_idx"][b] == 77 and (out["needed"][b] == 77).all() and out["via_count"][b] == 77
            assert (out["plan"][b].view(np.uint8) == SENTINEL).all() and out["plan_begin"][b] == bad.begin[b]
        else:
            assert out["result"][b] == want[b].result and out["goal_idx"][b] == want[b].goal_idx


def test_argument_errors_launch_nothing(gpu):
    d = scenes.global_plans(8, 64, S=2, seed=1)
    f = Fleet.of(d)
    a = _args_for(gpu)
    run_host(gpu, f, a, 65, 8)
    grid = gpu.last_local_plan_grid()
    L = gpu.lib

    def rc(mod, host=True, bmod=None):
        ins, outs = _inputs(f), _outs(f.B, 65, 8, True)
        la = _args(f, a, 65, 8, abi.ptr, ins, outs)
        bs = _batch(f, abi.ptr, f.sid)
        mod(la)
        if bmod:
            bmod(bs)
        r = L.tebgpu_local_plan(gpu.ctx, C.byref(bs), C.byref(la)) if host else \
            L.tebgpu_local_plan_device(gpu.ctx, C.byref(bs), C.byref(la), None)
        assert (outs["result"] == 77).all() and (ins["begin"] == f.begin).all()
        return r

    def setter(**kw):
        return lambda s: [setattr(s, k, v) for k, v in kw.items()]

    nothing = setter()
    bad = [setter(G_cap=0), setter(P_cap=1), setter(V_cap=-1), setter(global_plan=None), setter(plan_begin=None),
           setter(plan_end=None), setter(robot=None), setter(robot_vel=None), setter(grid=None), setter(origin=None),
           setter(plan=None), setter(plan_count=None), setter(result=None), setter(via_count=None)]
    for m in bad:
        for host in (True, False):
            assert rc(m, host) == abi.TEBGPU_ERR_INVALID_ARG
    for host in (True, False):
        assert rc(nothing, host, setter(B=0)) == abi.TEBGPU_ERR_INVALID_ARG
        assert rc(nothing, host, setter(scene_id=None)) == abi.TEBGPU_ERR_INVALID_ARG
        assert rc(nothing, host, setter(B=257)) == abi.TEBGPU_ERR_CAPACITY
        assert rc(nothing, host, setter(S=65)) == abi.TEBGPU_ERR_CAPACITY
    for what in ("begin", "end", "order", "sid"):       # the host entry point refuses what the device answers per band
        g = Fleet.of(d)
        if what == "begin":
            g.begin[3] = -1
        elif what == "end":
            g.end[3] = 65
        elif what == "order":
            g.begin[3], g.end[3] = 5, 4
        else:
            g.sid[3] = 2
        ins, outs = _inputs(g), _outs(g.B, 65, 8, True)
        la = _args(g, a, 65, 8, abi.ptr, ins, outs)
        assert L.tebgpu_local_plan(gpu.ctx, C.byref(_batch(g, abi.ptr, g.sid)), C.byref(la)) == abi.TEBGPU_ERR_INVALID_ARG
    assert L.tebgpu_local_plan(gpu.ctx, None, None) == abi.TEBGPU_ERR_INVALID_ARG
    assert gpu.last_local_plan_grid() == grid


# ---- a costmap -> local plan -> plan -> check cycle on one stream
def _cycle_fleet(B):
    d = scenes.global_plans(B, 1024, S=B, seed=21)
    r = scenes.costmap_raster(B, 60, 60, 0.05, 0.03, seed=22)
    r["robot"] = d["robot"].copy()
    r["origin"][:, 0] = d["robot"][:, 0] - 1.5
    r["origin"][:, 1] = d["robot"][:, 1] - 1.5
    d["scene_id"] = np.arange(B, dtype=np.int32)
    d["grid"], d["origin"] = r["grid"], r["origin"]
    return d, r


def _plan_params(overwrite):
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 0
    p.global_plan_overwrite_orientation = int(overwrite)
    return p


def _run_cycle(d, r, p, a, source, P_cap=160, V_cap=32, M_cap=2048, n_cap=96):
    """source: 'device' (local_plan_device on the stream), 'host' (rows from tebgpu_local_plan uploaded) or 'restated'"""
    B = d["robot"].shape[0]
    g = T.TebGpu(B, n_cap, B, M_cap, V_cap)
    g.set_params(p)
    f = Fleet.of(d)
    t = lambda x: _dev(x)
    cost, grid, origin, robot = t(r["cost"]), t(r["grid"]), t(r["origin"]), t(r["robot"])
    obst, ocount = torch.zeros(B * M_cap * 64, dtype=torch.uint8, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV)
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.include_costmap_obstacles, ca.behind_robot_dist = B, r["cost"].shape[1], M_cap, 1, 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    if source == "host":
        h = run_host(g, f, a, P_cap, V_cap)
        h["via_count"][(h["result"] != lp.PLANNED) & (h["result"] != lp.GOAL_REACHED)] = 0   # not written there
        plan, pcount, via, vcount = t(h["plan"]), t(h["plan_count"]), t(h["via"]), t(h["via_count"])
    elif source == "restated":
        want = f.expect(a, P_cap, V_cap, True)
        hp, hv = np.zeros((B, P_cap, 3)), np.zeros((B, V_cap, 2))
        for b, w in enumerate(want):
            if w.plan:
                hp[b, :len(w.plan)] = w.plan
            if w.via:
                hv[b, :len(w.via)] = w.via
        plan, via = t(hp), t(hv)
        pcount = t(np.array([len(w.plan) for w in want], np.int32))
        vcount = t(np.array([len(w.via or []) for w in want], np.int32))
    else:
        plan, pcount = torch.zeros(B * P_cap * 3, dtype=torch.float64, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV)
        via, vcount = torch.zeros(B * V_cap * 2, dtype=torch.float64, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=DEV)
    poses, n, sid = z((B, n_cap, 4), torch.float64), z((B,), torch.int32), t(d["scene_id"])
    vs = np.zeros((B, 4))
    vs[:, 3] = 1.0
    vstart, vgoal = t(vs), t(vs)
    costo, chi2, status, iters = z((B,), torch.float64), z((B,), torch.float64), z((B,), torch.int32), z((B,), torch.int32)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, B, M_cap, V_cap, 0
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count, bs.via, bs.via_count = obst.data_ptr(), ocount.data_ptr(), via.data_ptr(), vcount.data_ptr()
    bs.vel_start, bs.vel_goal = vstart.data_ptr(), vgoal.data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = costo.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    cmd = z((B, 4), torch.float64)
    feas, qc = torch.full((B,), 77, dtype=torch.int32, device=DEV), torch.full((B,), 77, dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g.costmap_obstacles_device(ca, stream=s.cuda_stream)
        if source == "device":
            ins = {k: t(v) for k, v in _inputs(f).items()}
            outs = dict(plan=plan, plan_count=pcount, goal_idx=None, via=via, via_count=vcount,
                        result=torch.zeros(B, dtype=torch.int32, device=DEV), needed=None)
            la = _args(f, a, P_cap, V_cap, lambda x: None if x is None else x.data_ptr(), ins, outs)
            g.local_plan_device(bs, la, stream=s.cuda_stream)
        g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, stream=s.cuda_stream)
        fa = abi.make_feasibility_args(0.1, max_queries=512, collision_distance=0.05, feasible=feas.data_ptr(),
                                       query_count=qc.data_ptr())
        g.check_feasible_device(bs, fa, stream=s.cuda_stream)
    s.synchronize()
    res = [x.cpu().numpy().copy() for x in (poses, n, costo, status, cmd, feas, qc, plan, pcount, via, vcount)]
    g.close()
    return res


@pytest.mark.parametrize("overwrite", [True, False])
def test_costmap_local_plan_plan_check_on_one_stream(overwrite):
    B = 24
    d, r = _cycle_fleet(B)
    p = _plan_params(overwrite)
    a = lp.Args(overwrite_orientation=overwrite, viapoint_sep=0.3, max_lookahead_dist=2.0)
    dev = _run_cycle(d, r, p, a, "device")
    host = _run_cycle(d, r, p, a, "host")
    sources = [host] + ([_run_cycle(d, r, p, a, "restated")] if not overwrite else [])
    rows = lambda x: x.view(np.uint8).view(np.float64).reshape(B, 160, 3)
    counts = lambda x: x.view(np.uint8).view(np.int32)
    pc = counts(dev[8])
    for other in sources:
        for k in range(7):
            assert _bytes(dev[k]) == _bytes(other[k]), k
        assert (counts(other[8]) == pc).all()
        for b in range(B):
            assert _bytes(rows(dev[7])[b, :pc[b]]) == _bytes(rows(other[7])[b, :pc[b]]), b
    assert (pc >= 2).sum() >= B // 2 and (dev[3] & abi.TEB_STATUS_BAD_INPUT == 0)[pc >= 2].all()
