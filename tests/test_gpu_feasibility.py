"""isTrajectoryFeasible on the device (tebgpu_check_feasible / _device, teb_feasible.cuh).

Query poses and verdicts are compared with op 12 of the drop-in layer (teb_host_band_op, pinned bit for bit against the
reference by tests/test_host_pin.py) and of the reference itself where oracle/_ref is built, on the cases of
tests/feasibility_cases.py. There op 12's recording costmap (a query collides inside a disc) is the device world of a
Point footprint, circular obstacles of the discs' radii and collision_distance 0. The world model itself is compared
with the oracle's footprint-to-obstacle distance on the scenes of tests/distance_cases.py and on costmap scenes."""
import ctypes as C
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import distance_cases as dc
from tests import feasibility_cases as fc
from tests import oracle_binding as ob
from tests import ref_binding as rb

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def host_op12():
    from teb_local_planner_b200 import build as b
    b.build()
    b.build_host()
    fn = C.CDLL(b.HOST_PIN).teb_host_band_op
    fn.restype = C.c_int32
    fn.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]

    def run(case, with_discs=True):
        rec = np.ascontiguousarray(case.rec[:max(case.n, 1)])
        a = np.ascontiguousarray(case.op12_args(with_discs), dtype=np.float64)
        cap = case.op12_cap()
        out = np.full(cap, np.nan)
        k = fn(12, rec.ctypes.data, case.n, a.ctypes.data, len(a), out.ctypes.data, cap)
        assert k >= 0, case
        return out[:k].copy()
    return run


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(64, fc.N_CAP, 64, 2048, 0, max_obst_vertices=256)
    g.set_params(abi.default_params())
    yield g
    g.close()


def _disc_batch(cases, with_discs=True):
    """one band per case, each on its own scene of circular obstacles (the case's discs)"""
    B = len(cases)
    M = max([len(c.discs) for c in cases] + [1])
    obst = np.zeros((B, M), abi.OBST_DTYPE)
    cnt = np.zeros(B, np.int32)
    for b, c in enumerate(cases):
        if with_discs:
            for k, (x, y, r) in enumerate(c.discs):
                obst[b, k]["type"], obst[b, k]["x"], obst[b, k]["y"], obst[b, k]["radius"] = abi.TEB_OBST_CIRCULAR, x, y, r
            cnt[b] = len(c.discs)
    poses = np.stack([c.rec for c in cases])
    return abi.HostBatch(poses, np.array([c.n for c in cases], np.int32), obst, cnt, scene_id=np.arange(B, dtype=np.int32))


def _check_case(g, c, with_discs=True):
    hb = _disc_batch([c], with_discs)
    mq = len(c.queries) + 8
    return g.check_feasible(hb, c.inscribed, c.look_ahead_idx, c.lookahead_distance, c.ang_res, 0.0, mq, queries=True)


def _same_as_op12(out, feas, cnt, q):
    n = int(out[1])
    assert feas == out[0] and cnt == n
    assert np.array_equal(q[:n], out[2:].reshape(-1, 3))
    assert np.isnan(q[n:]).all()                      # the rows behind the count are not written


def test_query_poses_equal_op12(gpu, host_op12):
    for c in fc.band_cases() + fc.random_cases():
        f, k, q = _check_case(gpu, c, with_discs=False)
        _same_as_op12(host_op12(c, with_discs=False), f[0], k[0], q[0])
        if rb.live():
            _same_as_op12(rb.band_op(12, c.rec[:c.n] if c.n else None, c.op12_args(False), cap=c.op12_cap()), f[0], k[0], q[0])


def test_verdict_and_count_equal_op12_with_discs(gpu, host_op12):
    cases = fc.disc_cases()
    assert any("inter" in c.name and c.feasible == 0 for c in cases) and any(c.name.startswith("contact") for c in cases)
    for c in cases:
        f, k, q = _check_case(gpu, c)
        _same_as_op12(host_op12(c), f[0], k[0], q[0])
        if rb.live():
            _same_as_op12(rb.band_op(12, c.rec[:c.n], c.op12_args(), cap=c.op12_cap()), f[0], k[0], q[0])


def _world_batch(cases, pool):
    """one single-pose band per distance case, each on its own scene (the case's obstacle)"""
    B = len(cases)
    PV = max([len(c.verts) for c in cases if c.verts is not None] + [0]) if pool else 0
    obst = np.zeros((B, 1), abi.OBST_DTYPE)
    verts = np.zeros((B, max(PV, 1), 2))
    poses = np.zeros((B, 1, 4))
    for b, c in enumerate(cases):
        obst[b, 0] = c.obst[0] if c.obst.ndim else c.obst
        if c.verts is not None:
            verts[b, :len(c.verts)] = c.verts
        poses[b, 0, :2] = c.pose
    return abi.HostBatch(poses, np.ones(B, np.int32), obst, np.ones(B, np.int32), scene_id=np.arange(B, dtype=np.int32),
                         obst_vertices=verts if PV else None)


@pytest.mark.parametrize("pool", [True, False])
def test_world_model_on_the_distance_cases(pool):
    """verdict == (oracle distance <= collision_distance) for every footprint x obstacle type, away from ties; exact
    contacts collide at 0 and exact distances collide with collision_distance set to them. pool=False: the Point /
    Circular cases without a vertex pool (the fast-path builds)"""
    cases = dc.all_cases() if pool else dc.path_cases()
    by_fp = {}
    for c in cases:
        by_fp.setdefault(c.fp, []).append(c)
    checked = exact = 0
    for fp, cs in by_fp.items():
        for lo in range(0, len(cs), 64):
            part = cs[lo:lo + 64]
            hb = _world_batch(part, pool)
            p = part[0].params()
            g = T.TebGpu(hb.B, 3, hb.S, 1, 0, max_obst_vertices=hb.PV_cap)
            g.set_params(p)
            d_or = np.array([ob.distance(p, c.pose3(), c.obst, c.verts, 0.0) for c in part])
            exact_d = [float(c.d) if c.d is not None and c.t is None and float(c.d) == c.d else None for c in part]
            for cd in (0.0, dc.MIN_D, dc.FORCE_D, dc.CUT_D, 0.3):
                f, k = g.check_feasible(hb, 1.0, collision_distance=cd)
                assert (k == 1).all()
                for b, c in enumerate(part):
                    if exact_d[b] is not None:
                        assert f[b] == (0 if exact_d[b] <= cd else 1), (c, cd)
                        exact += 1
                    elif abs(d_or[b] - cd) >= 1e-12:
                        assert f[b] == (0 if d_or[b] <= cd else 1), (c, cd, d_or[b])
                        checked += 1
            hit = [b for b, e in enumerate(exact_d) if e is not None and e >= 0]
            for b in hit:                                      # collision_distance set to the exact distance
                f, _ = g.check_feasible(hb, 1.0, collision_distance=exact_d[b])
                assert f[b] == 0, part[b]
            g.close()
    assert checked + exact > 100


def test_nan_distance_is_undecidable_and_collision_dominates(gpu):
    c = fc.Case("nan", fc._line(4, dx=0.25), 4, 1.0)
    hb = _disc_batch([c, c, c], with_discs=False)
    o = np.zeros((3, 2), abi.OBST_DTYPE)
    o["type"] = abi.TEB_OBST_CIRCULAR
    o["x"][0, 0] = o["x"][1, 0] = np.nan                   # band 0: a NaN row; band 1: a NaN row and a disc over pose 0
    o["x"][1, 1], o["radius"][1, 1] = 0.0, 0.01
    o["x"][2, :] = 100.0
    hb2 = abi.HostBatch(hb.poses, hb.n, o, np.array([1, 2, 2], np.int32), scene_id=np.arange(3, dtype=np.int32))
    f, k = gpu.check_feasible(hb2, 1.0)
    assert list(f) == [-1, 0, 1] and list(k) == [1, 1, 4]
    bad = hb2.copy()
    bad.poses[1, 2, 2] = np.inf                            # a non-finite heading among the checked poses
    bad.poses[2, 3, 0] = np.nan
    f, k = gpu.check_feasible(bad, 1.0)
    assert list(f) == [-1, -1, -1] and list(k) == [1, 0, 0]
    f, k = gpu.check_feasible(bad, 1.0, look_ahead_idx=2)   # band 2's NaN pose lies beyond the look-ahead index
    assert f[2] == 1 and k[2] == 3


def test_max_queries_below_at_and_above_the_count(gpu):
    c = fc.Case("cap", fc._line(6, dx=0.5), 6, 0.2)           # 2 extra samples per segment: 16 queries
    T_ = len(c.queries)
    assert T_ == 16
    free = _disc_batch([c], with_discs=False)
    for mq, (ef, ek) in ((T_ - 1, (-1, T_)), (T_, (1, T_)), (T_ + 1, (1, T_)), (1, (-1, T_))):
        f, k, q = gpu.check_feasible(free, 0.2, max_queries=mq, queries=True)
        assert (f[0], k[0]) == (ef, ek), mq
        assert np.array_equal(q[0, :min(T_, mq)], c.queries[:mq]) and np.isnan(q[0, min(T_, mq):]).all()
    j = 7                                                    # a disc over query 7 (an interpolated pose)
    hit = fc.Case("cap_hit", c.rec[:6], 6, 0.2, discs=[(c.queries[j][0], c.queries[j][1] + 1e-3, 0.01)])
    hb = _disc_batch([hit])
    for mq, (ef, ek) in ((j, (-1, T_)), (j + 1, (0, j + 1)), (T_ + 5, (0, j + 1))):
        f, k, q = gpu.check_feasible(hb, 0.2, max_queries=mq, queries=True)
        assert (f[0], k[0]) == (ef, ek), mq
        rows = min(ek, mq)
        assert np.array_equal(q[0, :rows], c.queries[:rows]) and np.isnan(q[0, rows:]).all()


def _pad(hb, M_cap):
    """the scene padded with far points up to M_cap rows (they are never within reach)"""
    o = np.zeros((hb.S, M_cap), abi.OBST_DTYPE)
    o[:, :hb.M_cap] = hb.obstacles
    o["x"][:, hb.M_cap:] = 1e4 + np.arange(M_cap - hb.M_cap)
    o["y"][:, hb.M_cap:] = -1e4
    return abi.HostBatch(hb.poses, hb.n, o, hb.obst_count + (M_cap - hb.M_cap), scene_id=hb.scene_id,
                         obst_vertices=hb.obst_vertices if hb.PV_cap else None)


def test_global_table_path_gives_the_staged_bits():
    p, hb = scenes.costmap_scene(64, n=80, candidates=24, seed=3)
    hb.obst_count[:] = 64
    p.footprint_type = abi.TEB_FOOTPRINT_CIRCULAR
    p.footprint_radius = 0.2
    big = _pad(hb, 1100)
    g = T.TebGpu(hb.B, hb.n_cap, 1, 1100, 0, max_obst_vertices=hb.PV_cap)
    g.set_params(p)
    for cd in (0.0, 0.05, 0.3):
        a = g.check_feasible(hb, 0.1, collision_distance=cd, max_queries=2048, queries=True)
        assert g.last_feasibility_check() == ("staged", hb.B)
        b = g.check_feasible(big, 0.1, collision_distance=cd, max_queries=2048, queries=True)
        assert g.last_feasibility_check() == ("global", hb.B)
        for x, y in zip(a, b):
            assert np.array_equal(x, y, equal_nan=True)
    g.close()


def _oracle_verdicts(p, hb, b, queries, cd):
    """(feasible, count) of band b from the oracle's distance over every row; None where a distance is within 1e-9
    of collision_distance"""
    o = hb.obstacles[hb.scene_id[b], :hb.obst_count[hb.scene_id[b]]]
    verts = hb.obst_vertices[hb.scene_id[b]] if hb.PV_cap else None
    pts = (o["type"] <= abi.TEB_OBST_CIRCULAR)
    fr = p.footprint_radius if p.footprint_type == abi.TEB_FOOTPRINT_CIRCULAR else 0.0
    assert p.footprint_type in (abi.TEB_FOOTPRINT_POINT, abi.TEB_FOOTPRINT_CIRCULAR)
    for k, qp in enumerate(queries):
        d = np.hypot(qp[0] - o["x"][pts], qp[1] - o["y"][pts]) - np.where(o["type"][pts] == abi.TEB_OBST_CIRCULAR, o["radius"][pts], 0) - fr
        d = list(d) + [ob.distance(p, qp, o[m], verts, 0.0) for m in np.nonzero(~pts)[0]]
        if min(abs(x - cd) for x in d) < 1e-9:
            return None
        if min(d) <= cd:
            return 0, k + 1
    return 1, len(queries)


@pytest.mark.parametrize("M", [1500, 4096, 16384])
def test_costmap_scenes_match_the_oracle(M):
    p, hb = scenes.costmap_scene(M, n=100, candidates=12, seed=M)
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.15
    g = T.TebGpu(hb.B, hb.n_cap, 1, M, 0, max_obst_vertices=hb.PV_cap)
    g.set_params(p)
    compared = 0
    for lai, cd in ((-1, 0.0), (5, 0.05), (-1, 0.4)):
        f, k, q = g.check_feasible(hb, 0.1, look_ahead_idx=lai, collision_distance=cd, max_queries=4096, queries=True)
        assert g.last_feasibility_check() == ("global", hb.B)
        for b in range(0, hb.B, 3):
            c = fc.Case("cm", hb.poses[b, :hb.n[b]], int(hb.n[b]), 0.1, look_ahead_idx=lai)
            assert np.array_equal(q[b, :min(k[b], 4096)], c.queries[:k[b]])
            want = _oracle_verdicts(p, hb, b, c.queries, cd)
            if want is not None:
                assert (f[b], k[b]) == want, (b, lai, cd)
                compared += 1
    assert compared >= 6
    g.close()


DEV_FIELDS = ("poses", "n", "scene_id", "obstacles", "obst_count", "obst_vertices", "via", "via_count", "vel_start",
              "vel_goal", "prefer_rotdir", "cost", "chi2", "status", "lm_iters")


class DeviceBatch:
    """torch copies of a HostBatch's arrays and the TebBatch of their device pointers"""

    def __init__(self, hb):
        dev = torch.device("cuda:0")
        self.hb = hb
        self.t = {k: torch.from_numpy(np.ascontiguousarray(getattr(hb, k)).view(np.uint8).reshape(-1).copy()).to(dev)
                  for k in DEV_FIELDS}
        bs = abi.TebBatch()
        bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap, hb.PV_cap
        for k, v in self.t.items():
            setattr(bs, k, v.data_ptr() if v.numel() else None)
        if hb.V_cap == 0:
            bs.via = None
        self.bs = bs

    def snapshot(self):
        return {k: v.cpu().numpy().copy() for k, v in self.t.items()}

    def read(self):
        h = self.hb.copy()
        for k in ("poses", "n", "cost", "chi2", "status", "lm_iters"):
            like = getattr(h, k)
            like[...] = self.t[k].cpu().numpy().view(like.dtype).reshape(like.shape)
        return h


def _device_check(g, db, B, inscribed, mq, pad=4, stream=None, **kw):
    dev = torch.device("cuda:0")
    f = torch.full((B + pad,), 77, dtype=torch.int32, device=dev)
    k = torch.full((B + pad,), 77, dtype=torch.int32, device=dev)
    q = torch.full((B, mq, 3), 7.5, dtype=torch.float64, device=dev)
    fa = abi.make_feasibility_args(inscribed, max_queries=mq, feasible=f.data_ptr(), query_count=k.data_ptr(),
                                   queries=q.data_ptr(), **kw)
    g.check_feasible_device(db.bs, fa, stream=torch.cuda.current_stream().cuda_stream if stream is None else stream)
    torch.cuda.synchronize()
    return f.cpu().numpy(), k.cpu().numpy(), q.cpu().numpy()


def _c3_batch(B=24, seed=5):
    p, hb = scenes.make_config_batch("C3", candidates=B, seed=seed)
    return p, hb


def test_host_and_device_entry_points_give_the_same_bits_and_leave_the_batch_alone():
    p, hb = _c3_batch()
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
    g.set_params(p)
    db = DeviceBatch(hb)
    for lai, ld, cd in ((-1, -1.0, 0.0), (5, -1.0, 0.45), (-1, 2.0, 0.6)):
        before = db.snapshot()
        f, k, q = g.check_feasible(hb, 0.1, look_ahead_idx=lai, lookahead_distance=ld, collision_distance=cd,
                                   max_queries=600, queries=True)
        df, dk, dq = _device_check(g, db, hb.B, 0.1, 600, look_ahead_idx=lai, lookahead_distance=ld, collision_distance=cd)
        after = db.snapshot()
        assert all(np.array_equal(before[x], after[x]) for x in before)          # TebBatch untouched
        assert np.array_equal(df[:hb.B], f) and np.array_equal(dk[:hb.B], k)
        assert (df[hb.B:] == 77).all() and (dk[hb.B:] == 77).all()               # nothing past B
        for b in range(hb.B):
            rows = min(k[b], 600)
            assert np.array_equal(dq[b, :rows], q[b, :rows]) and (dq[b, rows:] == 7.5).all()
        assert set(f) <= {-1, 0, 1}
    g.close()


def test_bits_do_not_depend_on_the_batch_position():
    p, hb = _c3_batch(B=32, seed=6)
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
    g.set_params(p)
    a = g.check_feasible(hb, 0.1, collision_distance=0.45, max_queries=600, queries=True)
    perm = np.random.default_rng(0).permutation(hb.B)
    ph = abi.HostBatch(hb.poses[perm], hb.n[perm], hb.obstacles, hb.obst_count, scene_id=hb.scene_id[perm])
    b = g.check_feasible(ph, 0.1, collision_distance=0.45, max_queries=600, queries=True)
    for x, y in zip(a, b):
        assert np.array_equal(x[perm], y, equal_nan=True)
    one = abi.HostBatch(hb.poses[7:8], hb.n[7:8], hb.obstacles, hb.obst_count, scene_id=hb.scene_id[7:8])
    c = g.check_feasible(one, 0.1, collision_distance=0.45, max_queries=600, queries=True)
    for x, y in zip(a, c):
        assert np.array_equal(x[7:8], y, equal_nan=True)
    g.close()


def test_optimize_and_plan_after_a_check_give_the_same_bits():
    p, hb = _c3_batch(B=16, seed=7)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    outs = []
    for check_first in (False, True):
        g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
        g.set_params(p)
        if check_first:
            g.check_feasible(hb, 0.1, max_queries=50, queries=True)
        h = hb.copy()
        g.optimize(h, args)
        if check_first:
            g.check_feasible(h, 0.05, collision_distance=0.2)
        h2 = h.copy()
        start, goal = h2.poses[:, 2, :3].copy(), h2.poses[np.arange(h2.B), h2.n - 1, :3].copy()
        cmd, path = g.plan(h2, start, goal, args)
        outs.append((h, h2, cmd, path))
        g.close()
    for x, y in zip(outs[0][:2], outs[1][:2]):
        for k in ("poses", "n", "cost", "chi2", "status", "lm_iters"):
            assert np.array_equal(getattr(x, k), getattr(y, k), equal_nan=True), k
    assert np.array_equal(outs[0][2], outs[1][2]) and np.array_equal(outs[0][3], outs[1][3])


def test_argument_errors_launch_nothing():
    p, hb = _c3_batch(B=4, seed=8)
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
    g.set_params(p)
    g.optimize(hb.copy(), abi.make_args(1, 1))
    launches = g.launch_count()
    assert launches > 1
    f, k = np.zeros(hb.B, np.int32), np.zeros(hb.B, np.int32)
    L = g.lib
    good = dict(inscribed_radius=0.1, feasible=abi.ptr(f), query_count=abi.ptr(k))
    bad_args = [dict(inscribed_radius=0.0), dict(inscribed_radius=-1.0), dict(inscribed_radius=math.inf),
                dict(inscribed_radius=math.nan), dict(angular_resolution=0.0), dict(angular_resolution=math.nan),
                dict(collision_distance=-1e-300), dict(collision_distance=math.inf), dict(max_queries=0),
                dict(feasible=None), dict(query_count=None)]
    db = DeviceBatch(hb)
    for kw in bad_args:
        a = dict(good)
        a.update(kw)
        fa = abi.make_feasibility_args(**a)
        bs = hb.struct()
        assert L.tebgpu_check_feasible(g.ctx, C.byref(bs), C.byref(fa)) == abi.TEBGPU_ERR_INVALID_ARG, kw
        assert L.tebgpu_check_feasible_device(g.ctx, C.byref(db.bs), C.byref(fa), None) == abi.TEBGPU_ERR_INVALID_ARG, kw
        assert g.launch_count() == launches, kw
    fa = abi.make_feasibility_args(**good)
    assert L.tebgpu_check_feasible(g.ctx, None, C.byref(fa)) == abi.TEBGPU_ERR_INVALID_ARG
    assert L.tebgpu_check_feasible(g.ctx, C.byref(hb.struct()), None) == abi.TEBGPU_ERR_INVALID_ARG
    for field in ("poses", "n", "scene_id", "obst_count"):
        bs = hb.struct()
        setattr(bs, field, None)
        assert L.tebgpu_check_feasible(g.ctx, C.byref(bs), C.byref(fa)) == abi.TEBGPU_ERR_INVALID_ARG, field
    for field, v in (("n", hb.n_cap + 1), ("scene_id", 1)):          # host entry point: per-band ranges
        h = hb.copy()
        getattr(h, field)[1] = v
        assert L.tebgpu_check_feasible(g.ctx, C.byref(h.struct()), C.byref(fa)) == abi.TEBGPU_ERR_INVALID_ARG, field
    assert g.launch_count() == launches
    # the device entry point answers such a band with -1 and checks the others
    h = hb.copy()
    h.n[1] = hb.n_cap + 1
    h.scene_id[2] = 5
    db = DeviceBatch(h)
    df, dk, _ = _device_check(g, db, hb.B, 0.1, 64)
    hf, hk = g.check_feasible(hb, 0.1, max_queries=64)
    assert g.launch_count() == 1
    assert df[1] == -1 and df[2] == -1 and dk[1] == 0 and dk[2] == 0
    assert df[0] == hf[0] and df[3] == hf[3] and dk[0] == hk[0] and dk[3] == hk[3]
    g.close()


def test_plan_then_check_on_one_stream_matches_the_host_check():
    p, hb = _c3_batch(B=16, seed=9)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
    g.set_params(p)
    db = DeviceBatch(hb)
    dev = torch.device("cuda:0")
    start = torch.from_numpy(hb.poses[:, 1, :3].copy()).to(dev)
    goal = torch.from_numpy(hb.poses[np.arange(hb.B), hb.n - 1, :3].copy()).to(dev)
    cmd = torch.zeros((hb.B, 4), dtype=torch.float64, device=dev)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g.plan_device(db.bs, args, cmd, start=start, goal=goal, stream=s.cuda_stream)
        df, dk, dq = _device_check(g, db, hb.B, 0.1, 800, stream=s.cuda_stream, look_ahead_idx=-1, collision_distance=0.45)
    h = db.read()
    hf, hk, hq = g.check_feasible(h, 0.1, collision_distance=0.45, max_queries=800, queries=True)
    assert np.array_equal(df[:hb.B], hf) and np.array_equal(dk[:hb.B], hk)
    for b in range(hb.B):
        rows = min(hk[b], 800)
        assert np.array_equal(dq[b, :rows], hq[b, :rows])
    # the node's reaction: clear the infeasible bands, the next plan cold-starts them
    n = db.t["n"].view(torch.int32)
    n[torch.from_numpy(df[:hb.B] == 0).to(dev)] = 0
    torch.cuda.synchronize()
    assert (n.cpu().numpy()[df[:hb.B] == 0] == 0).all()
    g.close()
