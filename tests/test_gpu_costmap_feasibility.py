"""tebgpu_check_feasible_costmap(_device): isTrajectoryFeasible against each scene's costmap, held bit for bit to the
restatement of CostmapModel::footprintCost in tests/costmap_feasibility_cases.py, and to tebgpu_check_feasible's
queries; the host and device entry points, band positions, max_queries, bad bands and argument errors; and the fleet
cycle on one stream with the costmap check in it."""
import ctypes as C
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import costmap_feasibility_cases as cf
from tests import cycle_cases as cc
from tests import feasibility_cases as fc

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = "cuda:0"


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(256, fc.N_CAP, 64, 64, 0)
    g.set_params(abi.default_params())
    yield g
    g.close()


def _stack(rasters):
    """[S][cell_cap] cost, grid, origin of a list of cf.Raster"""
    cap = max(m.sx * m.sy for m in rasters)
    cost = np.zeros((len(rasters), cap), np.uint8)
    for s, m in enumerate(rasters):
        cost[s, :m.sx * m.sy] = m.cost[:m.sx * m.sy]
    grid = np.array([(m.sx, m.sy) for m in rasters], np.int32)
    origin = np.array([(m.ox, m.oy, m.r) for m in rasters])
    return cost, grid, origin


def _batch(rec, n, sid, S):
    obst = np.zeros((S, 1), abi.OBST_DTYPE)
    return abi.HostBatch(np.ascontiguousarray(rec), np.asarray(n, np.int32), obst, np.zeros(S, np.int32),
                         scene_id=np.asarray(sid, np.int32))


def test_hand_cases(gpu):
    cases = cf.hand_cases()
    groups = {}
    for c in cases:          # one band per case; footprints differ, so one call per footprint
        groups.setdefault(tuple(map(tuple, c[3])), []).append(c)
    for fp, cs in groups.items():
        cost, grid, origin = _stack([c[1] for c in cs])
        rec = np.zeros((len(cs), fc.N_CAP, 4))
        for b, c in enumerate(cs):
            rec[b, 0, :3] = c[2]
        hb = _batch(rec, np.ones(len(cs)), np.arange(len(cs)), len(cs))
        f, k, q, qc = gpu.check_feasible_costmap(hb, cost, grid, origin, np.array(fp).reshape(-1, 2), 0.1, max_queries=4,
                                                 queries=True, query_cost=True)
        for b, c in enumerate(cs):
            want = cf.footprint_cost(c[1], *c[2], list(fp))
            assert c[4] is None or want == c[4]
            assert qc[b, 0] == want and k[b] == 1 and f[b] == (0 if want == -1 else 1), c[0]
            assert np.array_equal(q[b, 0], np.array(c[2])) and np.isnan(qc[b, 1:]).all()


def _check_fleet(g, ras, rec, n, sid, fp, inscribed=0.1, mq=600, **kw):
    hb = _batch(rec, n, sid, ras["cost"].shape[0])
    f, k, q, qc = g.check_feasible_costmap(hb, ras["cost"], ras["grid"], ras["origin"], fp, inscribed, max_queries=mq,
                                           queries=True, query_cost=True, **kw)
    return hb, f, k, q, qc


@pytest.mark.parametrize("F", [0, 1, 2, 3, 4, 16])
@pytest.mark.parametrize("size", [120, 400])
def test_random_fleets_match_the_restatement(gpu, F, size):
    ras, rec, n, sid, fp = cf.random_fleet(8, size, size, 0.05, seed=10 * F + size, F=F)
    hb, f, k, q, qc = _check_fleet(gpu, ras, rec, n, sid, fp)
    near, seen = 0, set()
    for b in range(hb.B):
        m = cf.raster_of(ras, sid[b])
        wf, wk, wqc = cf.band_verdict(m, rec[b], n[b], [tuple(p) for p in fp], 0.1, max_queries=600)
        rows = min(wk, 600)
        assert np.array_equal(q[b, :rows], fc.ref_queries(rec[b], n[b], 0.1)[:rows])
        seen.update(wqc)
        if (f[b], k[b]) == (wf, wk) and np.array_equal(qc[b, :len(wqc)], np.array(wqc, float)):
            continue
        # a difference is allowed only where the device's cos / sin can move a vertex across a cell edge
        j = next(i for i in range(len(wqc)) if i >= rows or qc[b, i] != wqc[i])
        assert cf.near_cell_edge(m, *q[b, j], [tuple(p) for p in fp]), (b, j)
        near += 1
    print(f"F={F} size={size}: {near} bands differ at a cell edge")
    assert near == 0
    assert -1 in seen and max(seen) > 0
    assert F < 3 or size > 120 or -2 in seen or -3 in seen       # the larger maps' robots rarely reach an edge or the 255s
    assert set(f) <= {-1, 0, 1} and (f == 0).any() and (f == 1).any()
    assert gpu.last_feasibility_check() == ("costmap", hb.B)


def test_queries_equal_the_table_checks_where_neither_collides(gpu):
    ras, rec, n, sid, fp = cf.random_fleet(6, 120, 120, 0.05, seed=7, F=4)
    hb, f, k, q, _ = _check_fleet(gpu, ras, rec, n, sid, fp, look_ahead_idx=-1, lookahead_distance=1.0)
    tf, tk, tq = gpu.check_feasible(hb, 0.1, lookahead_distance=1.0, max_queries=600, queries=True)
    assert (tf == 1).all()                     # no obstacle rows: the table check finds nothing
    free = f != 0
    assert free.any()
    assert np.array_equal(k[free], tk[free])
    assert np.array_equal(q[free], tq[free], equal_nan=True)


class _Dev:
    """device copies of a fleet's batch and rasters, and the world / args structs over them"""

    def __init__(self, hb, ras, fp, mq, pad=4):
        t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
        self.t = dict(poses=t(hb.poses), n=t(hb.n), scene_id=t(hb.scene_id), cost=t(ras["cost"]), grid=t(ras["grid"]),
                      origin=t(ras["origin"]))
        self.f = torch.full((hb.B + pad,), 77, dtype=torch.int32, device=DEV)
        self.k = torch.full((hb.B + pad,), 77, dtype=torch.int32, device=DEV)
        self.q = torch.full((hb.B, mq, 3), 7.5, dtype=torch.float64, device=DEV)
        self.qc = torch.full((hb.B, mq), 7.5, dtype=torch.float64, device=DEV)
        bs = abi.TebBatch()
        bs.B, bs.n_cap, bs.S = hb.B, hb.n_cap, hb.S
        bs.poses, bs.n, bs.scene_id = (self.t[x].data_ptr() for x in ("poses", "n", "scene_id"))
        self.bs = bs
        self.world = abi.make_costmap_world(ras["cost"].shape[1], self.t["cost"].data_ptr(), self.t["grid"].data_ptr(),
                                            self.t["origin"].data_ptr(), fp, self.qc.data_ptr())
        self.mq = mq

    def run(self, g, inscribed=0.1, stream=None, **kw):
        fa = abi.make_feasibility_args(inscribed, max_queries=self.mq, feasible=self.f.data_ptr(),
                                       query_count=self.k.data_ptr(), queries=self.q.data_ptr(), **kw)
        g.check_feasible_costmap_device(self.bs, fa, self.world, stream=stream)
        torch.cuda.synchronize()
        return self.f.cpu().numpy(), self.k.cpu().numpy(), self.q.cpu().numpy(), self.qc.cpu().numpy()

    def snapshot(self):
        return {k: v.cpu().numpy().copy() for k, v in self.t.items()}


def test_host_and_device_entry_points_give_the_same_bits_and_leave_the_batch_alone(gpu):
    ras, rec, n, sid, fp = cf.random_fleet(6, 120, 120, 0.05, seed=3, F=16)
    for lai, ld in ((-1, -1.0), (5, -1.0), (-1, 1.5)):
        hb, f, k, q, qc = _check_fleet(gpu, ras, rec, n, sid, fp, mq=300, look_ahead_idx=lai, lookahead_distance=ld)
        d = _Dev(hb, ras, fp, 300)
        before = d.snapshot()
        df, dk, dq, dqc = d.run(gpu, look_ahead_idx=lai, lookahead_distance=ld)
        after = d.snapshot()
        assert all(np.array_equal(before[x], after[x]) for x in before)
        assert np.array_equal(df[:hb.B], f) and np.array_equal(dk[:hb.B], k)
        assert (df[hb.B:] == 77).all() and (dk[hb.B:] == 77).all()
        for b in range(hb.B):
            rows = min(k[b], 300)
            assert np.array_equal(dq[b, :rows], q[b, :rows]) and (dq[b, rows:] == 7.5).all()
            assert np.array_equal(dqc[b, :rows], qc[b, :rows]) and (dqc[b, rows:] == 7.5).all()
            assert np.isnan(qc[b, rows:]).all()


def test_bits_do_not_depend_on_the_band_position(gpu):
    ras, rec, n, sid, fp = cf.random_fleet(6, 120, 120, 0.05, seed=4, F=4)
    a = _check_fleet(gpu, ras, rec, n, sid, fp)[1:]
    perm = np.random.default_rng(0).permutation(len(n))
    b = _check_fleet(gpu, ras, rec[perm], n[perm], sid[perm], fp)[1:]
    for x, y in zip(a, b):
        assert np.array_equal(x[perm], y, equal_nan=True)
    c = _check_fleet(gpu, ras, rec[5:6], n[5:6], sid[5:6], fp)[1:]
    for x, y in zip(a, c):
        assert np.array_equal(x[5:6], y, equal_nan=True)


def test_max_queries_below_at_and_above_the_count(gpu):
    ras, rec, n, sid, fp = cf.random_fleet(2, 120, 120, 0.05, seed=5, F=4)
    hb, f, k, _, _ = _check_fleet(gpu, ras, rec, n, sid, fp, inscribed=0.02, mq=4096)
    b = int(np.argmax(np.where(f == 1, k, -1)))
    assert f[b] == 1 and k[b] > 2
    total = k[b]
    for mq, want in ((total - 1, -1), (total, 1), (total + 1, 1)):
        _, ff, kk, qq, qc = _check_fleet(gpu, ras, rec[b:b + 1], n[b:b + 1], sid[b:b + 1], fp, inscribed=0.02, mq=mq)
        assert ff[0] == want and kk[0] == total
        assert not np.isnan(qc[0, :min(total, mq)]).any()
    m = cf.raster_of(ras, sid[b])
    assert cf.band_verdict(m, rec[b], n[b], [tuple(p) for p in fp], 0.02, max_queries=total - 1)[:2] == (-1, total)


def test_bad_bands_give_minus_one_on_the_device_and_are_refused_on_the_host(gpu):
    ras, rec, n, sid, fp = cf.random_fleet(4, 60, 60, 0.05, seed=6, F=4)
    ras["grid"][1] = (0, 60)                                   # sx < 1
    ras["origin"][2, 2] = 0.0                                  # resolution 0
    ras["origin"][3, 0] = np.inf                               # non-finite origin
    hb = _batch(rec, n, sid, 4)
    hb.n[0] = hb.n_cap + 1
    d = _Dev(hb, ras, fp, 64)
    df, dk, _, _ = d.run(gpu)
    bad = (np.arange(hb.B) == 0) | (sid != 0)
    assert (df[:hb.B][bad] == -1).all() and (dk[:hb.B][bad] == 0).all()
    good = np.flatnonzero(~bad)
    assert len(good)
    ok = _check_fleet(gpu, {k: v[:1] for k, v in ras.items()}, rec[good], n[good], sid[good], fp, mq=64)
    assert np.array_equal(df[good], ok[1]) and np.array_equal(dk[good], ok[2])
    for s, b in ((None, 0), (1, None), (2, None), (3, None)):
        h = _batch(rec, n, sid, 4)
        if b is not None:
            h.n[b] = h.n_cap + 1
            h.scene_id[:] = 0
        else:
            h.scene_id[:] = s
        with pytest.raises(T.TebGpuError):
            gpu.check_feasible_costmap(h, ras["cost"], ras["grid"], ras["origin"], fp, 0.1)
    h = _batch(rec, n, sid, 4)
    h.scene_id[3] = 4
    with pytest.raises(T.TebGpuError):
        gpu.check_feasible_costmap(h, ras["cost"], ras["grid"], ras["origin"], fp, 0.1)


def test_argument_errors_launch_nothing(gpu):
    ras, rec, n, sid, fp = cf.random_fleet(2, 60, 60, 0.05, seed=8, F=4)
    hb = _batch(rec, n, sid, 2)
    gpu.check_feasible(hb, 0.1)
    d = _Dev(hb, ras, fp, 64)
    d.run(gpu)
    launches = gpu.launch_count()
    assert launches == 1
    gpu.set_params(abi.default_params())
    L = gpu.lib
    cost = np.ascontiguousarray(ras["cost"])
    f, k = np.zeros(hb.B, np.int32), np.zeros(hb.B, np.int32)
    good_fa = dict(inscribed_radius=0.1, feasible=abi.ptr(f), query_count=abi.ptr(k), max_queries=64)
    good_w = dict(cell_cap=cost.shape[1], cost=abi.ptr(cost), grid=abi.ptr(ras["grid"]), origin=abi.ptr(ras["origin"]),
                  footprint=fp)
    bad = [({"inscribed_radius": 0.0}, {}), ({"inscribed_radius": math.nan}, {}), ({"angular_resolution": 0.0}, {}),
           ({"max_queries": 0}, {}), ({"feasible": None}, {}), ({"query_count": None}, {}),
           ({}, {"cell_cap": 0}), ({}, {"cost": None}), ({}, {"grid": None}), ({}, {"origin": None}),
           ({}, {"footprint": np.zeros((65, 2))}), ({}, {"footprint": np.array([[0.0, math.nan]] * 3)}),
           ({}, {"footprint": np.array([[math.inf, 0.0]] * 3)})]
    for fkw, wkw in bad:
        fa = abi.make_feasibility_args(**{**good_fa, **fkw})
        w = abi.make_costmap_world(**{**good_w, **wkw})
        bs = hb.struct()
        assert L.tebgpu_check_feasible_costmap(gpu.ctx, C.byref(bs), C.byref(fa), C.byref(w)) == abi.TEBGPU_ERR_INVALID_ARG
        assert L.tebgpu_check_feasible_costmap_device(gpu.ctx, C.byref(d.bs), C.byref(fa), C.byref(w), None) == \
            abi.TEBGPU_ERR_INVALID_ARG
        assert gpu.launch_count() == launches, (fkw, wkw)
    fa, w = abi.make_feasibility_args(**good_fa), abi.make_costmap_world(**good_w)
    assert L.tebgpu_check_feasible_costmap(gpu.ctx, C.byref(hb.struct()), C.byref(fa), None) == abi.TEBGPU_ERR_INVALID_ARG
    assert L.tebgpu_check_feasible_costmap(gpu.ctx, None, C.byref(fa), C.byref(w)) == abi.TEBGPU_ERR_INVALID_ARG
    for field in ("poses", "n", "scene_id"):
        bs = hb.struct()
        setattr(bs, field, None)
        assert L.tebgpu_check_feasible_costmap(gpu.ctx, C.byref(bs), C.byref(fa), C.byref(w)) == abi.TEBGPU_ERR_INVALID_ARG
    # collision_distance and the batch's obstacle arrays are not read
    bs = hb.struct()
    bs.obstacles, bs.obst_count = None, None
    fa.collision_distance = -1.0
    assert L.tebgpu_check_feasible_costmap(gpu.ctx, C.byref(bs), C.byref(fa), C.byref(w)) == 0


# ---- the fleet cycle on one stream: costmap -> local plan -> backup modes -> plan -> costmap check -> finish

FOOTPRINT = np.array([(-0.1, -0.1), (0.1, -0.1), (0.1, 0.1), (-0.1, 0.1)])


def _closed_loop(restated, cycles=12, B=16, P_cap=160, M_cap=2048, n_cap=96, Lb=10):
    d = scenes.global_plans(B, 1024, S=B, seed=21)
    r = scenes.costmap_raster(B, 60, 60, 0.05, 0.03, seed=22)
    r["origin"][:, 0] = d["robot"][:, 0] - 1.5
    r["origin"][:, 1] = d["robot"][:, 1] - 1.5
    sx = 60
    for s in range(4, 8):          # a lethal blob under robots 4 .. 7: their bands collide at pose 0
        for my in range(27, 33):
            r["cost"][s, my * sx + 27: my * sx + 33] = 254
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 0
    p.max_vel_trans = p.max_vel_x
    g = T.TebGpu(B, n_cap, B, M_cap, 0)
    g.set_params(p)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=DEV)
    f64, i32 = torch.float64, torch.int32
    cost, grid, origin = t(r["cost"]), t(r["grid"]), t(r["origin"])
    robot = t(d["robot"].copy())
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
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.include_costmap_obstacles, ca.behind_robot_dist = B, r["cost"].shape[1], M_cap, 1, 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    la = abi.make_local_plan_args(1024, P_cap, 0, max_lookahead_dist=2.0, global_plan=gp.data_ptr(),
                                  plan_begin=begin.data_ptr(), plan_end=end.data_ptr(), robot=robot.data_ptr(),
                                  robot_vel=vel.data_ptr(), grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  infeasible_count=state["infeasible_count"].data_ptr(), since_infeasible=since.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), result=result.data_ptr())
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    fa = abi.make_feasibility_args(0.1, max_queries=512, feasible=feas.data_ptr(), query_count=qc.data_ptr())
    world = abi.make_costmap_world(r["cost"].shape[1], cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), FOOTPRINT)
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
            g.costmap_obstacles_device(ca, stream=s.cuda_stream)
            g.local_plan_device(bs, la, stream=s.cuda_stream)
            g.backup_modes_device(bs, cy, stream=s.cuda_stream)
            g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, path=path,
                          stream=s.cuda_stream)
            if restated:
                s.synchronize()
                P, N = poses.cpu().numpy(), n.cpu().numpy()
                out_f, out_k = np.zeros(B, np.int32), np.zeros(B, np.int32)
                for b in range(B):
                    m = cf.raster_of(r, b)
                    out_f[b], out_k[b], _ = cf.band_verdict(m, P[b], N[b], [tuple(v) for v in FOOTPRINT], 0.1,
                                                            max_queries=512)
                feas.copy_(t(out_f))
                qc.copy_(t(out_k))
            else:
                g.check_feasible_costmap_device(bs, fa, world, stream=s.cuda_stream)
            g.finish_cycle_device(bs, cy, stream=s.cuda_stream)
            th = robot[:, 2]
            robot[:, 0] += (cmd_vel[:, 0] * torch.cos(th) - cmd_vel[:, 1] * torch.sin(th)) * dt
            robot[:, 1] += (cmd_vel[:, 0] * torch.sin(th) + cmd_vel[:, 1] * torch.cos(th)) * dt
            robot[:, 2] += cmd_vel[:, 2] * dt
            vel.copy_(cmd_vel)
        s.synchronize()
        rec = dict(n=n, status=status, path=path, cmd_vel=cmd_vel, outcome=outcome, feasible=feas, query_count=qc,
                   poses=poses, **state)
        trace.append({kk: v.cpu().numpy().copy() for kk, v in rec.items()})
        now += dt
    g.close()
    return trace


def test_closed_loop_with_the_costmap_check_matches_the_restated_check():
    dev = _closed_loop(False)
    ref = _closed_loop(True)
    for k, (a, b) in enumerate(zip(dev, ref)):
        for key in a:
            assert a[key].tobytes() == b[key].tobytes(), (k, key)
    feas = np.concatenate([c["feasible"] for c in dev])
    outs = np.concatenate([c["outcome"] for c in dev])
    assert (feas == 1).any() and (feas == 0).any()
    assert (outs == cc.COMMAND).any() and (outs == cc.INFEASIBLE).any()
