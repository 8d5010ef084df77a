"""Each scene's obstacle table from its local costmap on the device (tebgpu_costmap_obstacles / _device,
teb_costmap.cuh), held to the restatement of tests/costmap_cases.py: rows memcmp-equal, counts equal, through both entry
points. Also the overflow contract and how the optimize, feasibility and H-signature entry points answer it, the custom
rows, a convert / plan / check cycle on one stream, and the invariants (scene order, untouched inputs and rows, host
bits == device bits, argument errors that launch nothing)."""
import ctypes as C
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import costmap_cases as cm

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(16, 32, 64, 16384, 0)
    g.set_params(abi.default_params())
    yield g
    g.close()


class Fleet:
    """S scenes of possibly different sizes packed as TebCostmapArgs wants them, plus custom rows"""

    def __init__(self, rasters, origin, robot, custom=None, custom_count=None):
        S = len(rasters)
        self.grid = np.array([[r.shape[1], r.shape[0]] for r in rasters], np.int32).reshape(S, 2)
        cap = max([r.size for r in rasters] + [1])
        self.cell_cap = (cap + 15) // 16 * 16
        self.cost = np.zeros((S, self.cell_cap), np.uint8)
        for s, r in enumerate(rasters):
            self.cost[s, :r.size] = r.reshape(-1)
        self.origin = np.ascontiguousarray(origin, np.float64).reshape(S, 3)
        self.robot = np.ascontiguousarray(robot, np.float64).reshape(S, 3)
        self.custom = None if custom is None else np.ascontiguousarray(custom, abi.OBST_DTYPE).reshape(S, -1)
        self.custom_count = None if custom_count is None else np.ascontiguousarray(custom_count, np.int32)
        self.S = S

    def scene(self, s):
        sx, sy = (int(v) for v in self.grid[s])
        return self.cost[s], sx, sy, self.origin[s], self.robot[s]

    def custom_of(self, s):
        if self.custom is None or self.custom_count is None:
            return np.zeros(0, abi.OBST_DTYPE)
        return self.custom[s, :self.custom_count[s]]

    def expect(self, behind, include, cs=None, s_list=None):
        out = []
        for s in (range(self.S) if s_list is None else s_list):
            cost, sx, sy, o, r = self.scene(s)
            out.append(cm.restate_np(cost, sx, sy, o, r, behind, include, self.custom_of(s),
                                     cs=None if cs is None else cs[s]))
        return out

    def args(self, M_cap, behind, include, ptr, outs):
        ca = abi.TebCostmapArgs()
        ca.S, ca.cell_cap, ca.M_cap = self.S, self.cell_cap, int(M_cap)
        ca.include_costmap_obstacles, ca.behind_robot_dist = int(bool(include)), float(behind)
        ca.cost, ca.grid, ca.origin, ca.robot = ptr(self.cost), ptr(self.grid), ptr(self.origin), ptr(self.robot)
        if self.custom is not None and self.custom_count is not None:
            ca.C_cap, ca.custom, ca.custom_count = self.custom.shape[1], ptr(self.custom), ptr(self.custom_count)
        ca.obstacles, ca.obst_count, ca.needed = (ptr(x) for x in outs)
        return ca


def _out_arrays(S, M_cap):
    obst = np.full((S, M_cap), 0, abi.OBST_DTYPE)
    obst.view(np.uint8)[...] = SENTINEL
    return obst, np.full(S, 77, np.int32), np.full(S, 77, np.int32)


def run_host(g, f, M_cap, behind=1.5, include=True):
    """the host entry point with sentinel-filled outputs"""
    outs = _out_arrays(f.S, M_cap)
    ca = f.args(M_cap, behind, include, abi.ptr, outs)
    rc = g.lib.tebgpu_costmap_obstacles(g.ctx, C.byref(ca))
    assert rc == 0, g.lib.tebgpu_last_error_string(g.ctx)
    return outs


class DevFleet:
    """torch copies of a Fleet's inputs and sentinel-filled outputs"""

    def __init__(self, f, M_cap):
        t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(DEV)
        self.f = f
        self.inp = {k: t(getattr(f, k)) for k in ("cost", "grid", "origin", "robot", "custom", "custom_count")}
        o = _out_arrays(f.S, M_cap)
        self.out = [t(x) for x in o]
        self.M_cap = M_cap

    def args(self, behind, include):
        addr = {id(getattr(self.f, k)): v for k, v in self.inp.items() if v is not None}
        ptr = lambda a: None if a is None else addr[id(a)].data_ptr()
        ca = self.f.args(self.M_cap, behind, include, ptr, [None, None, None])
        ca.obstacles, ca.obst_count, ca.needed = (x.data_ptr() for x in self.out)
        return ca

    def read(self):
        obst = self.out[0].cpu().numpy().view(abi.OBST_DTYPE).reshape(self.f.S, self.M_cap)
        return obst, self.out[1].cpu().numpy().view(np.int32), self.out[2].cpu().numpy().view(np.int32)

    def inputs(self):
        return {k: v.cpu().numpy().copy() for k, v in self.inp.items() if v is not None}


def run_device(g, f, M_cap, behind=1.5, include=True, stream=None):
    d = DevFleet(f, M_cap)
    g.costmap_obstacles_device(d.args(behind, include),
                               stream=torch.cuda.current_stream().cuda_stream if stream is None else stream)
    torch.cuda.synchronize()
    return d.read()


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def assert_table(out, want, M_cap, label=""):
    obst, cnt, need = out
    for s, rows in enumerate(want):
        k = len(rows)
        assert need[s] == k, (label, s, need[s], k)
        assert cnt[s] == (k if k <= M_cap else -1), (label, s)
        w = min(k, M_cap)
        assert _bytes(obst[s, :w]) == _bytes(rows[:w]), (label, s)
        assert (obst[s, w:].view(np.uint8) == SENTINEL).all(), (label, s)      # rows past the count are not written


def both(g, f, M_cap, behind=1.5, include=True):
    h = run_host(g, f, M_cap, behind, include)
    d = run_device(g, f, M_cap, behind, include)
    for x, y in zip(h, d):
        assert _bytes(x) == _bytes(y)                                          # host bits == device bits
    return h


@pytest.mark.parametrize("case", cm.cases(), ids=lambda c: c.name)
def test_hand_cases(gpu, case):
    cc = len(case.custom)
    f = Fleet([case.cost.reshape(case.sy, case.sx)], [case.origin], [case.robot],
              custom=case.custom[None] if cc else None, custom_count=[cc] if cc else None)
    out = both(gpu, f, 64, case.behind, case.include)
    assert_table(out, [cm.expected_rows(case)], 64, case.name)
    assert gpu.last_costmap_grid() == 1


def _random_fleet(seed):
    """the sizes of the issue, robots inside and outside their maps, yaws across +-pi"""
    rng = np.random.default_rng(seed)
    shapes = [(0, 0), (1, 37), (37, 1), (2, 2), (3, 5), (120, 120), (127, 129), (128, 128), (300, 60), (400, 150),
              (3, 7000)]
    rasters, origin, robot = [], [], []
    yaws = [math.pi, -math.pi, math.pi / 2, -math.pi / 2, 0.0, 3 * math.pi / 4, -math.pi / 4, math.pi / 3]
    for k, (sx, sy) in enumerate(shapes):
        res = 0.05
        if (sx, sy) == (128, 128):
            c = np.full((sy, sx), 254, np.uint8)                                  # all lethal: 127 x 127 = 16129 rows
        else:
            lethal = 0.01 if (sx, sy) == (300, 60) else 0.15
            c = scenes.costmap_raster(1, sx, sy, res, lethal, seed=seed * 100 + k)["cost"][0, :sx * sy].reshape(sy, sx)
        ox, oy = rng.uniform(-5, 5, 2)
        inside = k % 2 == 0
        rx = ox + (0.5 * sx * res if inside else -3.0)
        ry = oy + (0.4 * sy * res if inside else sy * res + 2.0)
        rasters.append(c)
        origin.append((ox, oy, res))
        robot.append((rx, ry, yaws[k % len(yaws)] if k < len(yaws) else rng.uniform(-math.pi, math.pi)))
    return Fleet(rasters, origin, robot)


def _device_trig(yaws):
    t = torch.tensor(np.asarray(yaws, np.float64), device=DEV)
    return torch.cos(t).cpu().numpy(), torch.sin(t).cpu().numpy()


@pytest.mark.parametrize("behind", [0.0, 1.5, math.inf, -1.0, math.nan])
def test_random_rasters_match_the_restatement(gpu, behind):
    f = _random_fleet(11)
    M_cap = 16384
    assert max(len(r) for r in f.expect(math.inf, True)) == 16129
    out = both(gpu, f, M_cap, behind)
    dc, ds = _device_trig(f.robot[:, 2])
    exact = [dc[s] == math.cos(f.robot[s, 2]) and ds[s] == math.sin(f.robot[s, 2]) for s in range(f.S)]
    want = f.expect(behind, True)
    want_dev = f.expect(behind, True, cs=list(zip(dc, ds)))
    assert_table(out, want_dev, M_cap, "device trig")
    flipped = 0
    for s in range(f.S):
        if exact[s]:
            assert _bytes(want[s]) == _bytes(want_dev[s])
            continue
        # the device's cos / sin differ from glibc's in the last bit: only cells whose projection on the heading is
        # within rounding of 0 may change side
        cost, sx, sy, o, r = f.scene(s)
        allr, dot, norm = cm.restate_np(cost, sx, sy, o, r, math.inf, True, with_dot=True)
        a = set(map(tuple, np.stack([want[s]["x"], want[s]["y"]], 1).tolist()))
        b = set(map(tuple, np.stack([want_dev[s]["x"], want_dev[s]["y"]], 1).tolist()))
        key = {(x, y): k for k, (x, y) in enumerate(zip(allr["x"].tolist(), allr["y"].tolist()))}
        for cell in a ^ b:
            k = key[cell]
            assert abs(dot[k]) <= 2.0 ** -50 * norm[k], (s, cell, dot[k], norm[k])
            flipped += 1
    print(f"behind {behind}: {sum(exact)} / {f.S} yaws with bit-equal device trig, {flipped} cells changed side")


def _overflow_fleet():
    r = scenes.costmap_raster(3, 60, 60, 0.1, 0.1, seed=4)
    rasters = [r["cost"][s, :3600].reshape(60, 60) for s in range(3)]
    rasters[1] = np.where(np.arange(3600).reshape(60, 60) % 3 == 0, 254, rasters[1]).astype(np.uint8)   # > M_cap rows
    return Fleet(rasters, r["origin"], r["robot"])


def test_overflow_writes_the_first_rows_and_minus_one(gpu):
    f = _overflow_fleet()
    M_cap = 500
    want = f.expect(math.inf, True)
    assert len(want[0]) <= M_cap < len(want[1]) and len(want[2]) <= M_cap
    out = both(gpu, f, M_cap, math.inf)
    assert_table(out, want, M_cap)
    assert out[1][1] == -1 and out[1][0] != -1 and out[1][2] != -1


def _bands_on(f, B, n_cap, dist=2.5):
    """cold-start requests: band b on scene b % S from its robot towards a goal `dist` ahead"""
    sid = np.arange(B, dtype=np.int32) % f.S
    start = f.robot[sid].copy()
    goal = start.copy()
    goal[:, 0] += dist * np.cos(start[:, 2])
    goal[:, 1] += dist * np.sin(start[:, 2])
    return sid, start, goal


class DevBatch:
    """a device TebBatch of B bands (n = 0: cold start) whose obstacle table is `obst` / `ocount` (device tensors)"""

    def __init__(self, B, n_cap, S, M_cap, sid, obst, ocount):
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=DEV)
        self.poses, self.n = z((B, n_cap, 4), torch.float64), z((B,), torch.int32)
        self.sid = torch.from_numpy(sid).to(DEV)
        vs = np.zeros((B, 4))
        vs[:, 3] = 1.0
        self.vs, self.vg = torch.from_numpy(vs).to(DEV), torch.from_numpy(vs.copy()).to(DEV)
        self.cost, self.chi2 = z((B,), torch.float64), z((B,), torch.float64)
        self.status, self.iters = z((B,), torch.int32), z((B,), torch.int32)
        self.obst, self.ocount = obst, ocount
        bs = abi.TebBatch()
        bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, S, M_cap, 0, 0
        bs.poses, bs.n, bs.scene_id = self.poses.data_ptr(), self.n.data_ptr(), self.sid.data_ptr()
        bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
        bs.vel_start, bs.vel_goal = self.vs.data_ptr(), self.vg.data_ptr()
        bs.cost, bs.chi2, bs.status, bs.lm_iters = (self.cost.data_ptr(), self.chi2.data_ptr(), self.status.data_ptr(),
                                                    self.iters.data_ptr())
        self.bs = bs

    def result(self):
        return [x.cpu().numpy().copy() for x in (self.poses, self.n, self.cost, self.chi2, self.status, self.iters)]


def _plan_params():
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 0
    return p


def _cycle(g, db, start, goal, args, stream, fa_mq=512):
    """two plan cycles and a feasibility check on one stream"""
    B = start.shape[0]
    st, gl = torch.from_numpy(start).to(DEV), torch.from_numpy(goal).to(DEV)
    cmd = torch.zeros((2, B, 4), dtype=torch.float64, device=DEV)
    feas = torch.full((B,), 77, dtype=torch.int32, device=DEV)
    qc = torch.full((B,), 77, dtype=torch.int32, device=DEV)
    g.plan_device(db.bs, args, cmd[0], start=st, goal=gl, stream=stream)
    g.plan_device(db.bs, args, cmd[1], start=st, goal=gl, stream=stream)
    fa = abi.make_feasibility_args(0.1, max_queries=fa_mq, collision_distance=0.05, feasible=feas.data_ptr(),
                                   query_count=qc.data_ptr())
    g.check_feasible_device(db.bs, fa, stream=stream)
    return cmd, feas, qc


def test_overflowing_scene_is_refused_by_every_consumer():
    f = _overflow_fleet()
    M_cap = 500
    B, n_cap = 12, 64
    for dyn in (0, 1):
        p = _plan_params()
        p.include_dynamic_obstacles = dyn
        g = T.TebGpu(B, n_cap, f.S, M_cap, 0)
        g.set_params(p)
        d = DevFleet(f, M_cap)
        sid, start, goal = _bands_on(f, B, n_cap)
        obst = d.out[0]
        ocount = d.out[1].view(torch.int32)
        db = DevBatch(B, n_cap, f.S, M_cap, sid, obst, ocount)
        s = torch.cuda.Stream()
        args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
        with torch.cuda.stream(s):
            g.costmap_obstacles_device(d.args(math.inf, True), stream=s.cuda_stream)
            cmd, feas, qc = _cycle(g, db, start, goal, args, s.cuda_stream)
            h = torch.full((B, M_cap if dyn else 2), 7.0, dtype=torch.float64, device=DEV)
            s.synchronize()
            rc = g.lib.tebgpu_h_signature(g.ctx, C.byref(db.bs), 1, h.data_ptr(), 1)
            assert rc == 0
        torch.cuda.synchronize()
        status = db.status.cpu().numpy()
        fe, hs = feas.cpu().numpy(), h.cpu().numpy()
        bad = sid == 1
        assert (status[bad] & abi.TEB_STATUS_BAD_INPUT).all() and not (status[~bad] & abi.TEB_STATUS_BAD_INPUT).any()
        assert (fe[bad] == -1).all() and (fe[~bad] >= 0).all()
        assert np.isnan(hs[bad]).all() and np.isfinite(hs[~bad]).all()
        assert_table(d.read(), f.expect(math.inf, True), M_cap)
        g.close()


def test_custom_rows_come_through_verbatim(gpu):
    r = scenes.costmap_raster(4, 50, 40, 0.05, 0.1, seed=8)
    cu = np.zeros((4, 6), abi.OBST_DTYPE)
    base = cm.custom_rows()
    for s in range(4):
        cu[s, :5] = base
        cu[s]["x"] += s
    cu.view(np.uint8).reshape(4, 6, 64)[:, 5] = 0x3C                      # past custom_count: never copied
    cc = np.array([0, 5, 3, 1], np.int32)
    f = Fleet([r["cost"][s, :2000].reshape(40, 50) for s in range(4)], r["origin"], r["robot"], cu, cc)
    for include in (True, False):
        out = both(gpu, f, 2048, 1.5, include)
        want = f.expect(1.5, include)
        assert_table(out, want, 2048)
        if not include:
            assert [len(w) for w in want] == list(cc)


@pytest.mark.parametrize("M_cap,res", [(1024, 0.1), (4096, 0.05)])
def test_convert_plan_check_on_one_stream_equals_the_uploaded_table(M_cap, res):
    side = 60 if res == 0.1 else 120
    r = scenes.costmap_raster(4, side, side, res, 0.08 if M_cap <= 1024 else 0.3, seed=int(M_cap))
    f = Fleet([r["cost"][s, :side * side].reshape(side, side) for s in range(4)], r["origin"], r["robot"])
    want = f.expect(1.5, True)
    counts = [len(w) for w in want]
    assert max(counts) <= M_cap and (max(counts) > 1024) == (M_cap > 1024), counts
    p = _plan_params()
    B, n_cap = 16, 96
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    sid, start, goal = _bands_on(f, B, n_cap)
    results = []
    for from_device in (True, False):
        g = T.TebGpu(B, n_cap, f.S, M_cap, 0)
        g.set_params(p)
        if from_device:
            d = DevFleet(f, M_cap)
            obst, ocount = d.out[0], d.out[1]
        else:
            table = np.zeros((f.S, M_cap), abi.OBST_DTYPE)
            table.view(np.uint8)[...] = SENTINEL
            for s, w in enumerate(want):
                table[s, :len(w)] = w
            obst = torch.from_numpy(table.view(np.uint8).reshape(-1).copy()).to(DEV)
            ocount = torch.from_numpy(np.array(counts, np.int32)).to(DEV)
        db = DevBatch(B, n_cap, f.S, M_cap, sid, obst, ocount.view(torch.int32))
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            if from_device:
                g.costmap_obstacles_device(d.args(1.5, True), stream=s.cuda_stream)
            cmd, feas, qc = _cycle(g, db, start, goal, args, s.cuda_stream)
        s.synchronize()
        results.append(db.result() + [cmd.cpu().numpy(), feas.cpu().numpy(), qc.cpu().numpy(),
                                      obst.cpu().numpy(), ocount.cpu().numpy()])
        g.close()
    for k, (x, y) in enumerate(zip(*results)):
        assert _bytes(x) == _bytes(y), k
    assert (results[0][4] & abi.TEB_STATUS_BAD_INPUT == 0).all() and (results[0][7] >= 0).all()


def test_scene_order_does_not_matter_and_inputs_stay_untouched(gpu):
    f = _random_fleet(12)
    M_cap = 16384
    d = DevFleet(f, M_cap)
    before = d.inputs()
    gpu.costmap_obstacles_device(d.args(1.5, True))
    torch.cuda.synchronize()
    after = d.inputs()
    assert all(np.array_equal(before[k], after[k]) for k in before)
    a = d.read()
    perm = np.random.default_rng(1).permutation(f.S)
    rasters = [f.cost[s, :f.grid[s, 0] * f.grid[s, 1]].reshape(f.grid[s, 1], f.grid[s, 0]) for s in perm]
    pf = Fleet(rasters, f.origin[perm], f.robot[perm])
    b = run_device(gpu, pf, M_cap)
    for x, y in zip(a, b):
        assert _bytes(x[perm]) == _bytes(y)
    one = Fleet([rasters[0]], pf.origin[:1], pf.robot[:1])
    c = run_host(gpu, one, M_cap)
    for x, y in zip(b, c):
        assert _bytes(x[:1]) == _bytes(y)


def test_argument_errors_launch_nothing(gpu):
    f = _random_fleet(13)
    run_host(gpu, Fleet(*[[x] for x in (np.full((4, 4), 254, np.uint8), (0, 0, 0.1), (0, 0, 0))]), 16)
    assert gpu.last_costmap_grid() == 1
    L = gpu.lib
    outs = _out_arrays(f.S, 64)

    def rc(mod, host=True):
        ca = f.args(64, 1.5, True, abi.ptr, outs)
        mod(ca)
        return L.tebgpu_costmap_obstacles(gpu.ctx, C.byref(ca)) if host else L.tebgpu_costmap_obstacles_device(gpu.ctx, C.byref(ca), None)

    def setter(**kw):
        return lambda ca: [setattr(ca, k, v) for k, v in kw.items()]

    bad = [setter(M_cap=0), setter(S=0), setter(cell_cap=-1), setter(C_cap=-1), setter(grid=None), setter(origin=None),
           setter(robot=None), setter(obstacles=None), setter(obst_count=None), setter(cost=None),
           setter(obstacles=outs[0].ctypes.data + 8)]
    for m in bad:
        for host in (True, False):
            assert rc(m, host) == abi.TEBGPU_ERR_INVALID_ARG
    for m in (setter(S=65), setter(M_cap=16385)):
        for host in (True, False):
            assert rc(m, host) == abi.TEBGPU_ERR_CAPACITY
    assert L.tebgpu_costmap_obstacles(gpu.ctx, None) == abi.TEBGPU_ERR_INVALID_ARG
    # per-scene errors: refused by the host entry point, -1 from the device one
    cu = np.zeros((f.S, 2), abi.OBST_DTYPE)
    for what in ("neg", "cap", "cc_hi", "cc_lo"):
        g2 = f.grid.copy()
        cc = np.zeros(f.S, np.int32)
        if what == "neg":
            g2[2, 0] = -1
        elif what == "cap":
            g2[2] = (f.cell_cap, 2)
        else:
            cc[2] = 3 if what == "cc_hi" else -1
        bf = Fleet([np.zeros((1, 1), np.uint8)] * f.S, f.origin, f.robot, cu, cc)
        bf.cost, bf.grid, bf.cell_cap = f.cost, g2, f.cell_cap
        o = _out_arrays(f.S, 64)
        ca = bf.args(64, 1.5, True, abi.ptr, o)
        assert L.tebgpu_costmap_obstacles(gpu.ctx, C.byref(ca)) == abi.TEBGPU_ERR_INVALID_ARG, what
        assert gpu.last_costmap_grid() == 1, what
        dobst, dcnt, dneed = run_device(gpu, bf, 64)
        assert dcnt[2] == -1 and dneed[2] == -1, what
        assert (dobst[2].view(np.uint8) == SENTINEL).all()
        good = [s for s in range(f.S) if s != 2]
        want = bf.expect(1.5, True, s_list=good)
        for k, s in enumerate(good):
            n = len(want[k])
            assert dneed[s] == n and _bytes(dobst[s, :min(n, 64)]) == _bytes(want[k][:64]), (what, s)
        assert gpu.last_costmap_grid() == f.S
        run_host(gpu, Fleet([np.full((4, 4), 254, np.uint8)], [(0, 0, 0.1)], [(0, 0, 0)]), 16)
