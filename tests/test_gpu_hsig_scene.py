"""tebgpu_h_signature_scenes / tebgpu_hsig_factors (k_hsig_factors, k_hsig2d_scene, k_hsig3d_scene) against the long
double signature, on scenes of 1025 to 16384 obstacles (tests/hsig_scene_cases.py) and on every case of
tests/hsig_cases.py.

Bars, as tests/test_gpu_hsig.py:
  * 2-D: |H_gpu - H_oracle| <= 1e-12 sum_{k,l} |A_l| |L_kl|; +-inf, NaN and exact zeros equal;
  * x-y-t: 1e-12 max(1, |H|) per obstacle, the rows past M exactly 0;
  * the isEqual partition and isValid of each bundle equal the oracle's, and at M <= 1024 tebgpu_h_signature's.
Factor tables: Q_l against 1 / prod_j (o_l - o_j) of the long double restatement, within 8 M 2^-53, at up to 16384
rows (several parts of the product). Bits: host against device entry, a band alone against a mixed batch (forward and reversed), a scene at index 0 against
index 5 of 8, a table built in the call against one built beforehand and reused, a scene's table whatever S."""
import ctypes as C
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import hsig_cases as hc
from tests import hsig_scene_cases as sc
from tests.test_gpu_hsig import _as_values, _check_3d, _classes, _same_bits

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = torch.device("cuda:0")
SCENE_2D = {c.name: c for c in sc.cases_2d()}
SMALL_2D = {c.name: c for c in hc.cases_2d()}
SCENE_3D = {c.name: c for c in sc.cases_3d()}
_want, _prod = {}, {}


def _products(case):
    if case.name not in _prod:
        _prod[case.name] = sc.scene_products(case.obst)
    return _prod[case.name]


def _oracle_2d(case):
    if case.name not in _want:
        p = case.params()
        pr = _products(case) if len(case.obst) else None
        _want[case.name] = [sc.oracle_2d(p, rec, case.obst, pr) for rec in case.bands]
    return _want[case.name]


def _ctx(B, n_cap, S, M_cap, p):
    g = T.TebGpu(B, n_cap, S, max(M_cap, 1), 0)
    g.set_params(p)
    return g


def _rows(case, out):
    return np.stack([out.real, out.imag], 1) if case.dim == 2 else out


def _check_2d(case, got, want):
    p = case.params()
    for i, rec in enumerate(case.bands):
        w = np.array([want[i].real, want[i].imag])
        where = (case.name, i, got[i], w)
        for q in range(2):
            if not np.isfinite(w[q]):
                assert (np.isnan(w[q]) and np.isnan(got[i, q])) or got[i, q] == w[q], where
        if not np.all(np.isfinite(w)):
            continue
        if w[0] == 0 and w[1] == 0:
            assert got[i, 0] == 0 and got[i, 1] == 0, where
            continue
        scale = sc.error_scale(p, rec, case.obst)
        err = np.hypot(sc.LD(got[i, 0]) - sc.LD(w[0]), sc.LD(got[i, 1]) - sc.LD(w[1]))
        assert np.isfinite(got[i]).all() and err <= max(sc.LD(1e-12) * scale, sc.LD(5e-324)), where + (float(err),)


class Dev:
    """device copies of a HostBatch and a TebBatch of their addresses"""

    def __init__(self, hb):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(DEV)
        self.keep = dict(poses=t(hb.poses), n=t(hb.n), sid=t(hb.scene_id), ob=t(hb.obstacles), oc=t(hb.obst_count),
                         vs=t(hb.vel_start), vg=t(hb.vel_goal))
        bs = abi.TebBatch()
        bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap = hb.B, hb.n_cap, hb.S, hb.M_cap, 0
        k = self.keep
        bs.poses, bs.n, bs.scene_id = k["poses"].data_ptr(), k["n"].data_ptr(), k["sid"].data_ptr()
        bs.obstacles = k["ob"].data_ptr() if hb.M_cap > 0 else None
        bs.obst_count, bs.vel_start, bs.vel_goal = k["oc"].data_ptr(), k["vs"].data_ptr(), k["vg"].data_ptr()
        self.bs, self.hb = bs, hb

    def factors(self):
        S, Mc = self.hb.S, self.hb.M_cap
        self.f = (torch.full((max(S * Mc * 2, 1),), 7.0, dtype=torch.float64, device=DEV),
                  torch.full((max(S * Mc, 1),), 77, dtype=torch.int32, device=DEV),
                  torch.full((S,), 77, dtype=torch.int32, device=DEV))
        return abi.make_hsig_factors(*(x.data_ptr() for x in self.f))

    def read_factors(self):
        S, Mc = self.hb.S, self.hb.M_cap
        return (self.f[0].cpu().numpy()[:S * Mc * 2].reshape(S, Mc, 2), self.f[1].cpu().numpy()[:S * Mc].reshape(S, Mc),
                self.f[2].cpu().numpy())


def _device(g, hb, dim, use_dt=True, factors=None, d=None):
    d = d or Dev(hb)
    stride = max(hb.M_cap, 1) if dim == 3 else 2
    out = torch.full((hb.B, stride), float("nan"), dtype=torch.float64, device=DEV)
    g.h_signature_scenes_device(d.bs, out, factors=factors, use_timediffs=use_dt)
    g.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("name", list(SCENE_2D) + list(SMALL_2D))
def test_hsig2d_scenes_match_oracle(name):
    case = SCENE_2D.get(name) or SMALL_2D[name]
    want = _oracle_2d(case)
    hb, _ = hc.batch([case])
    p = case.params()
    g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, p)
    got = _rows(case, g.h_signature_scenes(hb))
    dev = _device(g, hb, 2)
    assert _same_bits(got, dev)
    _check_2d(case, got, want)
    thr = p.h_signature_threshold
    sc.assert_class_margins(case, want, thr)
    assert _classes(case, _as_values(case, got), thr) == _classes(case, want, thr)
    if hb.M_cap <= 1024:                                     # the same classes as the first entry point
        old = _rows(case, g.h_signature(hb))
        assert _classes(case, _as_values(case, old), thr) == _classes(case, _as_values(case, got), thr)
    g.close()


@pytest.mark.parametrize("name", list(SCENE_3D))
def test_hsig3d_scenes_match_oracle(oracle, name):
    case = SCENE_3D[name]
    p = case.params()
    want = [oracle.h_signature(p, rec, len(rec), case.obst, use_timediffs=True) for rec in case.bands]
    M_cap = len(case.obst) + 3 if len(case.obst) < 16384 else len(case.obst)
    hb, _ = hc.batch([case], M_cap=M_cap)
    g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, p)
    got = g.h_signature_scenes(hb)
    assert _same_bits(got, _device(g, hb, 3))
    _check_3d(case, got, want, M_cap)
    thr = p.h_signature_threshold
    assert _classes(case, _as_values(case, got), thr) == _classes(case, want, thr)
    g.close()


@pytest.mark.parametrize("name", ["costmap_4096", "costmap_16384", "ring_4096", "ring_16384", "grid_64x32",
                                  "far_before_near_1100"])
def test_factor_table_matches_long_double_products(name):
    """Q_l of every row against 1 / P_l of the long double restatement, as mantissa x 2^exponent (which never
    underflows, unlike the costmap signatures themselves). Above 2048 rows the product runs in parts of 2048 rows
    (k_hsig_factors) multiplied by k_hsig_factors_combine, so this holds the split and the combine to the product.
    Bound: each of the M - 1 factors costs at most about 6 units of roundoff u = 2^-53 in norm (the rounded difference
    o_l - o_j: 1; the complex product's numerator: sqrt(5); the rounded modulus and the two divisions: 3), the
    combine at most 8 more products of the same kind, and first-order error terms add: |Q / Q_ld - 1| <= 8 M u."""
    case = SCENE_2D[name]
    M = len(case.obst)
    hb, _ = hc.batch([case])
    g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, case.params())
    f, fe, fc = g.hsig_factors(hb)
    g.close()
    assert fc[0] == M
    err = sc.factor_rel_errors(f[0], fe[0], _products(case))
    bound = 8 * M * 2.0 ** -53
    assert float(err.max()) <= bound, (name, float(err.max()), int(np.argmax(err)), bound)


def test_hsig3d_scenes_equal_first_entry_at_small_scenes():
    """at M <= 1024 the x-y-t kernel does the first kernel's arithmetic per obstacle: the same bits"""
    for c in hc.cases_3d():
        hb, _ = hc.batch([c], M_cap=len(c.obst) + 2)
        g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, c.params())
        a, b = g.h_signature(hb, use_timediffs=c.use_dt), g.h_signature_scenes(hb, use_timediffs=c.use_dt)
        g.close()
        assert _same_bits(a, b), c.name


def test_band_alone_equals_mixed_batch_and_scene_index():
    """every band of several scenes alone and in one batch (forward, reversed); a scene at index 0 alone and at 5 of 8"""
    cases = [SCENE_2D["grid_64x32"], SCENE_2D["costmap_1025"], SMALL_2D["blob_1024"], SMALL_2D["skip_grid_origin"],
             SMALL_2D["range_far_first"], SMALL_2D["m0"], SMALL_2D["short_and_closed"], SCENE_2D["duplicates_1372"]]
    alone = {}
    for c in cases:
        hb, _ = hc.batch([c])
        g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, c.params())
        alone[c.name] = _rows(c, g.h_signature_scenes(hb))
        g.close()
    for reverse in (False, True):
        hb, where = hc.batch(cases, M_cap=2100, reverse=reverse)
        g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, cases[0].params())
        host = _rows(cases[0], g.h_signature_scenes(hb))
        assert _same_bits(host, _device(g, hb, 2))
        g.close()
        for c, i, r in where:
            assert _same_bits(host[r], alone[c.name][i]), (c.name, i, r, reverse)
    # scene index: the grid block at index 0 of 1 and at index 5 of 8 (the reversed batch puts the first case last)
    hb, where = hc.batch(cases[3:] + cases[:3], M_cap=2048)
    assert hb.S == 8
    g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, cases[0].params())
    f8 = g.hsig_factors(hb)
    h8 = _rows(cases[0], g.h_signature_scenes(hb))
    g.close()
    s5 = [c.name for c in cases[3:] + cases[:3]].index("grid_64x32")
    assert s5 == 5
    hb1, _ = hc.batch([cases[0]], M_cap=2048)
    g = _ctx(hb1.B, hb1.n_cap, hb1.S, hb1.M_cap, cases[0].params())
    f1 = g.hsig_factors(hb1)
    g.close()
    M = len(cases[0].obst)
    assert _same_bits(f8[0][5, :M], f1[0][0, :M]) and np.array_equal(f8[1][5, :M], f1[1][0, :M])
    assert f8[2][5] == f1[2][0] == M
    for c, i, r in where:
        assert _same_bits(h8[r], alone[c.name][i]), (c.name, i, r)


def test_factor_table_whatever_S_and_M_cap():
    """Q_l of a scene: the same bits alone (S = 1, M_cap = M) and as scene 2 of 3 at a larger M_cap; rows past the
    count 0 with exponent INT32_MIN; host and device tables equal"""
    c = SCENE_2D["costmap_4096"]
    M = len(c.obst)
    hb1, _ = hc.batch([c], M_cap=M)
    others = [SMALL_2D["blob_1024"], SCENE_2D["far_before_near_1100"]]
    hb3b, _ = hc.batch(others + [c], M_cap=M + 300)
    assert hb3b.S == 3
    g = _ctx(max(hb1.B, hb3b.B), hb1.n_cap, 3, M + 300, c.params())
    a = g.hsig_factors(hb1)
    b = g.hsig_factors(hb3b)
    d = Dev(hb3b)
    fs = d.factors()
    g.hsig_factors_device(d.bs, fs)
    g.synchronize()
    dv = d.read_factors()
    g.close()
    assert _same_bits(a[0][0], b[0][2, :M]) and np.array_equal(a[1][0], b[1][2, :M]) and a[2][0] == b[2][2] == M
    assert np.all(b[0][2, M:] == 0) and np.all(b[1][2, M:] == np.iinfo(np.int32).min)
    for x, y in zip(b, dv):
        assert np.ascontiguousarray(x).tobytes() == np.ascontiguousarray(y).tobytes()


def test_prebuilt_table_reused_equals_built_in_call():
    cases = [SCENE_2D["grid_64x32"], SMALL_2D["skip_grid_origin"], SCENE_2D["costmap_1025"]]
    hb, _ = hc.batch(cases)
    g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, cases[0].params())
    inline = g.h_signature_scenes(hb)
    f = g.hsig_factors(hb)
    a, b = g.h_signature_scenes(hb, factors=f), g.h_signature_scenes(hb, factors=f)
    d = Dev(hb)
    fs = d.factors()
    g.hsig_factors_device(d.bs, fs)
    dev1 = _device(g, hb, 2, factors=fs, d=d)
    dev2 = _device(g, hb, 2, factors=fs, d=d)
    g.close()
    for x in (a, b):
        assert _same_bits(inline, x)
    want = np.stack([inline.real, inline.imag], 1)
    assert _same_bits(dev1, want) and _same_bits(dev2, want)


def test_stale_table_and_out_of_range_rows_give_nan():
    """a table built at another count: NaN for that scene's bands only. Device rows with scene_id, n or obst_count out
    of range (-1 as an overflowing tebgpu_costmap_obstacles_device writes) give NaN; x-y-t too"""
    cases = [SCENE_2D["grid_64x32"], SMALL_2D["skip_exact"], SMALL_2D["blob_1024"]]
    hb, where = hc.batch(cases)
    g = _ctx(hb.B + 4, hb.n_cap, hb.S, hb.M_cap, cases[0].params())
    good = g.h_signature_scenes(hb)
    f = g.hsig_factors(hb)
    f[2][1] -= 1                                             # scene 1's table claims another count
    got = g.h_signature_scenes(hb, factors=f)
    for c, i, r in where:
        if c is cases[1]:
            assert np.isnan(got[r].real) and np.isnan(got[r].imag)
        else:
            assert _same_bits(np.array([got[r]]), np.array([good[r]]))
    bad = hb.copy()
    bad.scene_id[0] = hb.S                                   # scene_id out of range
    bad.n[1] = hb.n_cap + 1                                  # n out of range
    r_sc0 = [r for c, i, r in where if c is cases[2]]
    bad.obst_count[2] = -1                                   # an overflowing costmap conversion
    for dim in (2, 3):
        p = cases[0].params()
        p.include_dynamic_obstacles = int(dim == 3)
        g.set_params(p)
        out = _device(g, bad, dim)
        assert np.isnan(out[0]).all() and np.isnan(out[1]).all()
        for r in r_sc0:
            assert np.isnan(out[r]).all()
        ok = [r for r in range(hb.B) if r not in (0, 1) and r not in r_sc0]
        assert np.isfinite(out[ok, :2]).all(), dim
    g.close()


def test_costmap_cycle_on_one_stream_equals_host_table():
    """costmap rasters -> tebgpu_costmap_obstacles_device -> tebgpu_hsig_factors_device -> signatures on one stream, at
    more than 1024 rows per scene, against the same signatures from the host-uploaded table"""
    S, M_cap, B, n = 2, 3000, 6, 40
    r = scenes.costmap_raster(S, 120, 100, 0.05, 0.12, seed=11)
    cost, grid, origin, robot = r[:4] if isinstance(r, tuple) else (r["cost"], r["grid"], r["origin"], r["robot"])
    p = abi.default_params()
    p.include_dynamic_obstacles = 0
    g = _ctx(B, 64, S, M_cap, p)
    obst_h, cnt_h, _ = g.costmap_obstacles(cost, grid, origin, robot, M_cap, behind_robot_dist=math.inf)
    assert (cnt_h > 1024).all(), cnt_h
    rng = np.random.default_rng(3)
    poses = np.zeros((B, 64, 4))
    for b in range(B):
        s = b % S
        x0, y0, res = origin[s]
        start = (x0 + 0.5, y0 + 0.5)
        goal = (x0 + grid[s][0] * res - 0.5, y0 + grid[s][1] * res - 0.5)
        poses[b, :n] = hc.bent(start, goal, n, rng.uniform(-1.5, 1.5))
    hb = abi.HostBatch(poses, np.full(B, n, np.int32), obst_h, cnt_h, scene_id=np.arange(B, dtype=np.int32) % S)
    want = g.h_signature_scenes(hb)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(DEV)
    inp = [t(x) for x in (cost, grid, origin, robot)]
    ob = torch.zeros(S * M_cap * abi.OBST_DTYPE.itemsize, dtype=torch.uint8, device=DEV)
    oc = torch.zeros(S, dtype=torch.int32, device=DEV)
    ne = torch.zeros(S, dtype=torch.int32, device=DEV)
    ca = abi.TebCostmapArgs()
    cst = np.ascontiguousarray(cost, np.uint8).reshape(S, -1)
    ca.S, ca.cell_cap, ca.M_cap = S, cst.shape[1], M_cap
    ca.include_costmap_obstacles, ca.behind_robot_dist = 1, math.inf
    ca.cost, ca.grid, ca.origin, ca.robot = (x.data_ptr() for x in inp)
    ca.obstacles, ca.obst_count, ca.needed = ob.data_ptr(), oc.data_ptr(), ne.data_ptr()
    d = Dev(hb)
    d.bs.obstacles, d.bs.obst_count = ob.data_ptr(), oc.data_ptr()
    fs = d.factors()
    out = torch.full((B, 2), float("nan"), dtype=torch.float64, device=DEV)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g.costmap_obstacles_device(ca, stream=s.cuda_stream)
        g.hsig_factors_device(d.bs, fs, stream=s.cuda_stream)
        g.h_signature_scenes_device(d.bs, out, factors=fs, stream=s.cuda_stream)
    s.synchronize()
    host_f = g.hsig_factors(hb)
    g.close()
    got = out.cpu().numpy()
    assert _same_bits(got, np.stack([want.real, want.imag], 1))
    dev_f = d.read_factors()                                 # the tables themselves: they do not underflow
    assert np.array_equal(dev_f[2], cnt_h)
    for x, y in zip(host_f, dev_f):
        assert np.ascontiguousarray(x).tobytes() == np.ascontiguousarray(y).tobytes()
