"""Kernel A and the graph build, band by band, through tebgpu_build_system_graph (TebGpu.build_system(graph=True /
bands=...)), against the oracle (run on an H100: pytest -m gpu).

tests/test_gpu_parity.py holds kernel A's H|b and total chi2 to the oracle on smooth random bands. Here:
  a. every scenario at outer 0 and 3: H|b against the oracle's closed-form system with test_gpu_parity's bars, chi2
     by family (obstacles, via, time-optimal, other) against teb_oracle_trial_chi2 at dx = 0 within 1e-12 relative
     per family, and the graph k_build_graph made (association and legacy multiplicity-3 words, via-point poses,
     dynamic-obstacle times) bit-equal to teb_oracle_graph;
  b. shapes: n at every 29-pose warp tile, 116-pose CTA and 120-slot staging edge of k_linearize2 (and the 32-pose
     tiles of variant 1) up to 512, n_cap = n, n + 1, n + 3 and 512, all-ones (NaN) records past n, ragged batches
     over two scenes, one of them empty; every tile holds obstacle, via-point and dynamic-obstacle terms. Rows from 4 n
     on and association words of poses >= n keep the all-ones pattern the entry point fills in;
  c. the branch points of the penalties and edges, on dyadic axis-aligned bands where both sides compute the branch
     variable exactly (each case asserts the variable equals the boundary on the host);
  d. association and via-point edge cases on the staged path and, padded past 1024 rows, on the global-table path,
     whose occupancy words must mark exactly the non-zero association words;
  e. the same bits wherever and however it runs: staged and direct-store (TEBGPU_KA_STAGED=0) output, any batch
     position, and listed launches (the retry side stream's form) in any order, empty and full, which leave every
     unlisted band's rows, words and chi2 all-ones.
The worst errors per family and per build go to the parity report (tests/test_gpu_parity._report).
The legacy association also sets bits on poses 0 and n-1 whose edges g2o drops (every vertex fixed) and no kernel reads;
those two poses are compared only in the non-legacy association.
"""
import os

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi
from tests import oracle_binding as O
from tests import scenarios
from tests.param_cases import weight_multiplier
from tests.test_gpu_parity import _report as _write_report
from tests.test_oracle_graph import _line, _obst, _params

pytestmark = pytest.mark.gpu

H_BAR = 1e-12         # H and b relative to their largest entry (test_gpu_parity)
FAM_BAR = 1e-12       # chi2 per family, relative
ALL_ONES = np.uint64(0xFFFFFFFFFFFFFFFF)
FAMS = ("obst", "via", "time", "other")
_worst = {}


def _report(key, value):
    _worst[key] = max(_worst.get(key, value), value)
    _write_report("linearize", dict(sorted(_worst.items())))


def _ctx(hb, p, staged=True, variant=0, max_bands=None, max_obstacles=None):
    old = os.environ.get("TEBGPU_KA_STAGED")
    os.environ["TEBGPU_KA_STAGED"] = "1" if staged else "0"
    try:
        g = T.TebGpu(max_bands or hb.B, hb.n_cap, hb.S, max_obstacles or max(hb.M_cap, 1), hb.V_cap,
                     max_obst_vertices=hb.PV_cap)
    finally:
        if old is None:
            del os.environ["TEBGPU_KA_STAGED"]
        else:
            os.environ["TEBGPU_KA_STAGED"] = old
    g.set_params(p)
    if variant:
        g.set_linearize_variant(variant)
    return g


def _ones(a):
    a = np.ascontiguousarray(a)
    return (a.view(np.uint8) == 0xFF).all()


def _same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def _padded_from_dense(Hd, bd, n):
    N = 4 * n - 7
    Hb = np.zeros((4 * n, 12))
    Hb[:, 0] = 1.0
    for k in range(11):
        r = np.arange(k, N)
        Hb[r + 3, k] = Hd[r, r - k]
    Hb[3:3 + N, 11] = bd
    return Hb


_oracle_cache = {}


def _oracle(p, hb, b, outer):
    """(H|b in the device layout [4n][12], chi2 by family [4], graph) of band b"""
    n = int(hb.n[b])
    kw = scenarios.band_kwargs(hb, b)
    key = (id(p), bytes(p), hb.poses[b, :n].tobytes(), kw["obstacles"].tobytes(),
           None if kw["via"] is None else kw["via"].tobytes(), hb.vel_start[b].tobytes(), hb.vel_goal[b].tobytes(),
           kw["rotdir"], None if kw["obst_vertices"] is None else kw["obst_vertices"].tobytes(), outer,
           max(1, (hb.M_cap + 63) // 64))
    if key not in _oracle_cache:
        mult = weight_multiplier(p, outer)
        Hd, bd, _ = O.build_system(p, hb.poses[b], n, weight_multiplier=mult, jac_mode=O.JAC_ANALYTIC, **kw)
        fam = O.trial_chi2(p, hb.poses[b], n, hb.poses[b][None, :n], weight_multiplier=mult, **kw)[0]
        gr = O.graph(p, hb.poses[b], n, weight_multiplier=mult, MW=max(1, (hb.M_cap + 63) // 64), **kw)
        _oracle_cache[key] = (_padded_from_dense(Hd, bd, n), fam, gr)
    return _oracle_cache[key]


def check_band(p, hb, out, b, outer, build):
    """H|b, chi2 by family and the structure of band b against the oracle; untouched scratch past n"""
    n, n_cap = int(hb.n[b]), hb.n_cap
    ref, fam, gr = _oracle(p, hb, b, outer)
    got = out["Hb"][b, :4 * n]
    sH = np.abs(ref[:, :11]).max()
    eH = np.abs(got[:, :11] - ref[:, :11]).max() / sH
    eb = np.abs(got[:, 11] - ref[:, 11]).max() / max(np.abs(ref[:, 11]).max(), 1.0)
    _report(f"{build}/H_rel", float(eH))
    _report(f"{build}/b_rel", float(eb))
    assert eH <= H_BAR and eb <= H_BAR, f"{build} band {b} (n {n}): H {eH:.3e} b {eb:.3e}"
    assert _ones(out["Hb"][b, 4 * n:]), f"{build} band {b}: rows from 4 n written"
    cf = out["chi_fam"][b]
    for f, nm in enumerate(FAMS):
        e = 0.0 if cf[f] == fam[f] else abs(cf[f] - fam[f]) / max(abs(fam[f]), 1e-300)
        _report(f"{build}/chi2_{nm}_rel", float(e))
        assert e <= FAM_BAR, f"{build} band {b}: chi2 {nm} {cf[f]!r} vs oracle {fam[f]!r}"
    check_structure(p, hb, out, b, gr, build)


def check_structure(p, hb, out, b, gr, build):
    n = int(hb.n[b])
    lo, hi = (1, n - 1) if p.legacy_obstacle_association else (0, n)
    assert np.array_equal(out["assoc"][b, lo:hi], gr["assoc"][lo:hi]), f"{build} band {b}: association words"
    if p.legacy_obstacle_association:
        assert np.array_equal(out["assoc3"][b, 1:n - 1], gr["assoc3"][1:n - 1]), f"{build} band {b}: assoc3 words"
    assert (out["assoc"][b, n:] == ALL_ONES).all(), f"{build} band {b}: association words of poses >= n written"
    V = int(hb.via_count[b]) if hb.V_cap else 0
    if hb.V_cap:
        assert np.array_equal(out["via_idx"][b, :V], gr["via_idx"]), f"{build} band {b}: via {out['via_idx'][b]}"
        assert (out["via_idx"][b, V:] == -1).all()
    t = np.isfinite(gr["dyn_t"])
    assert _same(out["dyn_t"][b, :n][t], gr["dyn_t"][t]), f"{build} band {b}: dynamic-obstacle times"


def _run(g, hb, outer, bands=None):
    return g.build_system(hb, outer, bands=bands, graph=True)


# ------------------------------------------------------------------ a. every scenario (+ e. staged = direct stores)
@pytest.mark.parametrize("name", scenarios.ALL)
def test_every_scenario_against_oracle(name):
    p, hb = scenarios.scenario(name)
    g, gd = _ctx(hb, p), _ctx(hb, p, staged=False)
    try:
        for outer in (0, 3):
            out = _run(g, hb, outer)
            for b in range(hb.B):
                check_band(p, hb, out, b, outer, "ka2")
            direct = _run(gd, hb, outer)
            for k in out:
                assert _same(out[k], direct[k]), f"TEBGPU_KA_STAGED=0: {k} differs"
            # the existing readout gives the same system
            Hb, _ = g.build_system(hb, outer)
            for b in range(hb.B):
                assert _same(Hb[b, :4 * hb.n[b]], out["Hb"][b, :4 * hb.n[b]])
    finally:
        g.close()
        gd.close()


# ------------------------------------------------------------------ b. shapes
NS = [3, 4, 5, 28, 29, 30, 31, 32, 33, 57, 58, 59, 115, 116, 117, 118, 119, 120, 121, 232, 233, 463, 464, 465, 511, 512]
DX, DT = 0.25, 0.25


def _shape_params():
    p = abi.default_params()
    p.weight_viapoint = 1.0
    p.include_dynamic_obstacles = 1
    p.max_vel_x = 0.8
    return p


def _shape_scene(length):
    """static points every 2 m alternately 0.35 m left / right of the x axis, and one dynamic point that travels with
    the bands 0.3 m to their left (close to every pose at its frozen time)"""
    xs = np.arange(1.0, length + 2.0, 2.0)
    rows = [(x, 0.35 if k % 2 else -0.35) for k, x in enumerate(xs)] + [(0.0, 0.3)]
    ob = _obst(*rows, dynamic=(len(rows) - 1,))
    ob[-1]["vx"] = DX / DT
    return ob


def _shape_band(n, n_cap, seed):
    rng = np.random.default_rng(seed)
    rec = np.full((n_cap, 4), np.nan).view(np.uint64)
    rec[:] = ALL_ONES
    rec = rec.view(np.float64)
    x = DX * np.arange(n) + rng.uniform(-0.02, 0.02, n)
    y = rng.uniform(-0.05, 0.05, n)
    rec[:n, 0], rec[:n, 1] = x, y
    rec[:n, 2] = rng.uniform(-0.2, 0.2, n)
    rec[:n, 3] = DT * rng.uniform(0.9, 1.1, n)
    rec[0, :3] = 0.0
    rec[n - 1, 3] = 0.0
    via = np.stack([np.arange(2.5, DX * n, 5.0), np.full(len(np.arange(2.5, DX * n, 5.0)), 0.1)], axis=1)
    if len(via) == 0:
        via = np.array([[DX * (n - 1) / 2, 0.1]])
    return rec, via


def _shape_batch(ns, n_cap, two_scenes=False, seed=0):
    B = len(ns)
    length = DX * max(ns) + 4
    scene = _shape_scene(length)
    S = 2 if two_scenes else 1
    ob = np.zeros((S, len(scene)), abi.OBST_DTYPE)
    ob[0] = scene
    cnt = np.array([len(scene)] + [0] * (S - 1), np.int32)
    poses = np.zeros((B, n_cap, 4))
    vias = []
    for b, n in enumerate(ns):
        poses[b], v = _shape_band(n, n_cap, seed + 7 * n)
        vias.append(v)
    V_cap = max(len(v) for v in vias) + 2              # V_cap > via_count
    via = np.zeros((B, V_cap, 2))
    vc = np.zeros(B, np.int32)
    for b, v in enumerate(vias):
        via[b, :len(v)] = v
        vc[b] = len(v)
    sid = (np.arange(B) % S).astype(np.int32)
    return abi.HostBatch(poses, np.array(ns, np.int32), ob, cnt, sid, via, vc)


def _shape_runs(variant):
    p = _shape_params()
    for delta in (0, 1, 3):
        for n in NS:
            if n + delta <= 512:                        # the context limit of max_poses
                yield p, _shape_batch([n], n + delta), f"n_cap=n+{delta}"
    yield p, _shape_batch(NS, 512, two_scenes=True), "ragged_n_cap=512"


@pytest.mark.parametrize("variant", [0, 1])
def test_shapes_against_oracle(variant):
    build = "ka2" if variant == 0 else "ka1"
    for p, hb, what in _shape_runs(variant):
        g = _ctx(hb, p, variant=variant)
        try:
            out = _run(g, hb, 1)
        finally:
            g.close()
        for b in range(hb.B):
            n = int(hb.n[b])
            if hb.obst_count[hb.scene_id[b]]:
                assert out["chi_fam"][b, 0] > 0 and out["chi_fam"][b, 1] > 0, (what, n)
            check_band(p, hb, out, b, 1, f"{build}/shapes")


def test_every_tile_holds_unary_terms():
    """the shape bands put obstacle, via-point and dynamic-obstacle terms on every 29-pose tile (else an unwritten
    tile's rows would match the oracle's chain rows by luck)"""
    p = _shape_params()
    hb = _shape_batch([512], 512)
    n = 512
    kw = scenarios.band_kwargs(hb, 0)
    gr = O.graph(p, hb.poses[0], n, **kw)
    for t0 in range(0, n, 29):               # warp w of CTA c produces poses 116 c + 29 w ..
        sl = slice(max(t0, 1), min(t0 + 29, n - 1))
        assert gr["assoc"][sl].any() and np.isin(gr["via_idx"], np.arange(sl.start, sl.stop)).any(), t0
        assert np.isfinite(gr["dyn_t"][sl]).all()


# ------------------------------------------------------------------ c. branch points
EPS = 0.125


def _kink_params(**kw):
    p = _params(min_obstacle_dist=0.5, inflation_dist=0.75, penalty_epsilon=EPS, max_vel_x=1.0, max_vel_x_backwards=EPS,
                max_vel_theta=0.625, acc_lim_x=0.5, acc_lim_theta=1.125, weight_viapoint=1.0,
                obstacle_association_force_inclusion_factor=1.5, obstacle_association_cutoff_factor=4.0)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _batch(recs, obstacles, via=None, rotdir=None):
    n_cap = max(len(r) for r in recs)
    B = len(recs)
    poses = np.zeros((B, n_cap, 4))
    for b, r in enumerate(recs):
        poses[b, :len(r)] = r
    ob = np.asarray(obstacles, abi.OBST_DTYPE)
    if len(ob) == 0:
        ob = np.zeros(1, abi.OBST_DTYPE)
        cnt = 0
    else:
        cnt = len(ob)
    kw = {}
    if via is not None:
        kw = dict(via=np.broadcast_to(via, (B,) + np.shape(via)).copy(), via_count=np.full(B, len(via), np.int32))
    hb = abi.HostBatch(poses, np.array([len(r) for r in recs], np.int32), ob[None], np.array([cnt], np.int32),
                       prefer_rotdir=rotdir, **kw)
    return hb


def _kink_case(case):
    n = 12
    base = _line(n)
    if case == "omega_and_rot_acc":            # omega = +-(max_vel_theta - eps), rotational acceleration acc_lim_theta - eps
        p = _kink_params()
        up, down = base.copy(), base.copy()
        up[2:7, 2] = 0.25 * np.arange(1, 6)
        down[2:7, 2] = -0.25 * np.arange(1, 6)
        w0, w1 = (up[1, 2] - up[0, 2]) / up[0, 3], (up[2, 2] - up[1, 2]) / up[1, 3]
        assert w1 == p.max_vel_theta - p.penalty_epsilon and (down[2, 2] - down[1, 2]) / down[1, 3] == -w1
        assert (w1 - w0) * 2 / (up[0, 3] + up[1, 3]) == p.acc_lim_theta - p.penalty_epsilon
        return p, _batch([up, down], [])
    if case == "zero_segment":                 # v = 0 at pen_interval2's lower bound, proj = 0 for pen_below, sp on 0 length
        p = _kink_params(weight_shortest_path=1.0)
        r = base.copy()
        r[6:, 0] -= 0.5                        # poses 5 and 6 coincide
        assert r[6, 0] == r[5, 0] and -p.max_vel_x_backwards + p.penalty_epsilon == 0.0
        return p, _batch([r, base], [])
    if case == "carlike":                      # dtheta 0, zero length, r exactly min_turning_radius
        p = _kink_params(min_turning_radius=2.0, weight_kinematics_turning_radius=1.0)
        r = base.copy()
        r[3:7, 2] = 0.25 * np.arange(1, 5)
        r[7:, 2] = r[6, 2]
        z = base.copy()
        z[6:, 0] -= 0.5
        z[6:, 2] = 0.25
        assert (r[4, 0] - r[3, 0]) / (r[4, 2] - r[3, 2]) == p.min_turning_radius
        return p, _batch([r, z, base], [])
    if case == "rotdir":                       # prefer-rotdir with dtheta = 0
        p = _kink_params(weight_prefer_rotdir=2.0)
        return p, _batch([base, base, base], [], rotdir=np.array([abi.TEB_ROTDIR_LEFT, abi.TEB_ROTDIR_RIGHT, 0], np.int32))
    if case == "obstacle_distances":           # min_obstacle_dist + eps and inflation_dist, point and circular
        p = _kink_params()
        ob = _obst((2.0, 0.625), (3.5, -0.75), (1.0, -1.0))
        ob[2]["type"], ob[2]["radius"] = abi.TEB_OBST_CIRCULAR, 0.375
        assert 0.625 == p.min_obstacle_dist + p.penalty_epsilon and 0.75 == p.inflation_dist and 1.0 - 0.375 == 0.625
        return p, _batch([base], ob)
    if case == "via_on_pose":                  # e = 0
        p = _kink_params()
        return p, _batch([base], [], via=np.array([[2.0, 0.0], [3.0, 0.0]]))
    if case == "theta_cut":                    # headings of exactly +-pi, steps across the cut, theta outside [-pi, pi)
        p = _kink_params()
        a, c, d = base.copy(), base.copy(), base.copy()
        a[1:-1, 2] = np.where(np.arange(1, n - 1) % 2, np.pi, -np.pi)
        c[1:-1, 2] = np.where(np.arange(1, n - 1) % 2, np.pi - 0.125, -np.pi + 0.125)
        d[1:-1, 2] = np.linspace(3.0, 9.5, n - 2)
        d[3, 2] = -7.0
        return p, _batch([a, c, d], _obst((2.0, 0.25)))
    if case == "dt_extremes":                  # dt of 1e-9 and 1e3
        p = _kink_params()
        s, l = base.copy(), base.copy()
        s[:-1, 3] = 1e-9
        l[:-1, 3] = 1e3
        return p, _batch([s, l], _obst((2.0, 0.25)))
    raise KeyError(case)


KINKS = ["omega_and_rot_acc", "zero_segment", "carlike", "rotdir", "obstacle_distances", "via_on_pose", "theta_cut",
         "dt_extremes"]


@pytest.mark.parametrize("case", KINKS)
def test_branch_points_against_oracle(case):
    p, hb = _kink_case(case)
    for variant in (0, 1):
        g = _ctx(hb, p, variant=variant)
        try:
            for outer in (0, 2):
                out = _run(g, hb, outer)
                for b in range(hb.B):
                    check_band(p, hb, out, b, outer, f"{'ka2' if variant == 0 else 'ka1'}/kinks")
        finally:
            g.close()


# ------------------------------------------------------------------ d. association and via-point edge cases
def _graph_cases():
    n = 12
    rec = _line(n)
    cases = []
    p = _params(min_obstacle_dist=0.5, obstacle_association_force_inclusion_factor=2.0,
                obstacle_association_cutoff_factor=4.0)
    # equal distances (lowest index), exactly at force_d, a right-side candidate further away, exactly at cut_d, just
    # past cut_d, just inside force_d, dead ahead of pose 1
    ob = _obst((2.0 - 0.75, 1.0), (2.0 + 0.75, 1.0), (2.0, -1.0), (2.75, -1.0), (3.5, 2.0), (4.0, 2.0 + 2.0 ** -20),
               (4.5, 1.0 - 2.0 ** -20), (0.5 + 1.5, 0.0))
    cases.append(("nonlegacy", p, [rec], ob, None))
    pd = _params(min_obstacle_dist=0.5, obstacle_association_force_inclusion_factor=2.0,
                 obstacle_association_cutoff_factor=4.0, include_dynamic_obstacles=1)
    obd = _obst((2.0, 0.25), (2.0, -0.25), (4.0, 0.75), dynamic=(0,))
    cases.append(("dynamic_skipped", pd, [rec], obd, None))
    pv = _params(min_obstacle_dist=0.5, weight_velocity_obstacle_ratio=1.0, obstacle_proximity_lower_bound=0.2,
                 obstacle_proximity_upper_bound=1.0)
    cases.append(("vor_pose0", pv, [rec], _obst((0.0, 0.25), (1.0, -0.5)), None))
    for opa in (1, 2, 3, 10, n, n + 5):
        pl = _params(legacy_obstacle_association=1, obstacle_poses_affected=opa)
        obl = _obst((2.5, 0.3), (2.25, 0.0), (0.0, 0.1), (0.5, 0.2), (5.5, 0.0), (5.0, 0.2), (9.0, 0.0))
        cases.append((f"legacy_{opa}", pl, [rec], obl, None))
    # Line and Polygon obstacles: closest-pose search over the vertex list
    pg = _params(legacy_obstacle_association=1, obstacle_poses_affected=4)
    obg = _obst((0.0, 0.0), (0.0, 0.0))
    obg[0]["type"], obg[0]["vertex_begin"], obg[0]["vertex_count"] = abi.TEB_OBST_LINE, 0, 2
    obg[1]["type"], obg[1]["vertex_begin"], obg[1]["vertex_count"] = abi.TEB_OBST_POLYGON, 2, 3
    verts = np.array([[1.75, 0.5], [2.25, 1.0], [3.5, -0.5], [4.0, -1.0], [3.25, -1.5]])
    cases.append(("legacy_line_polygon", pg, [rec], (obg, verts), None))
    via = np.array([[-3.0, 0.0], [100.0, 0.0], [1.25, 0.5], [1.0, 0.25], [2.0, 0.0]])
    for ordered in (0, 1):
        pw = _params(weight_viapoint=1.0, via_points_ordered=ordered)
        cases.append((f"via_{'ordered' if ordered else 'unordered'}", pw, [rec, _line(8)], _obst((2.0, 0.25)), via))
    return cases


def _case_batch(recs, ob, via):
    verts = None
    if isinstance(ob, tuple):
        ob, verts = ob
    n_cap = max(len(r) for r in recs)
    B = len(recs)
    poses = np.zeros((B, n_cap, 4))
    poses.view(np.uint64)[:] = ALL_ONES
    for b, r in enumerate(recs):
        poses[b, :len(r)] = r
    kw = {}
    if via is not None:
        V_cap = len(via) + 3
        v = np.zeros((B, V_cap, 2))
        v[:, :len(via)] = via
        kw = dict(via=v, via_count=np.full(B, len(via), np.int32))
    return abi.HostBatch(poses, np.array([len(r) for r in recs], np.int32), np.asarray(ob, abi.OBST_DTYPE)[None],
                         np.array([len(ob)], np.int32), obst_vertices=None if verts is None else verts[None], **kw)


def _padded(hb, M_cap):
    from tests.test_gpu_large_scenes import _padded as pad
    return pad(hb, M_cap, 0)


def _occ_consistent(out, hb):
    MW = out["assoc"].shape[2]
    for b in range(hb.B):
        for i in range(int(hb.n[b])):
            bits = 0
            for w in range(MW):
                if out["assoc"][b, i, w]:
                    bits |= 1 << w
            words = [int(x) for x in out["occ"][b, i]]
            want = [(bits >> (64 * o)) & 0xFFFFFFFFFFFFFFFF for o in range(len(words))]
            assert words == want, (b, i)


@pytest.mark.parametrize("case", [c[0] for c in _graph_cases()])
def test_association_and_via_cases_on_both_paths(case):
    name, p, recs, ob, via = next(c for c in _graph_cases() if c[0] == case)
    hb = _case_batch(recs, ob, via)
    g = _ctx(hb, p)
    try:
        out = _run(g, hb, 1)
    finally:
        g.close()
    for b in range(hb.B):
        check_band(p, hb, out, b, 1, "ka2/graph_cases")
    # the same scene padded past 1024 rows with points 1000 m away: the global-table association gives the same bits
    big = _padded(hb, 1100)
    gg = _ctx(big, p)
    try:
        outg = _run(gg, big, 1)
    finally:
        gg.close()
    assert big.M_cap > 1024
    _occ_consistent(outg, big)
    for b in range(hb.B):
        n = int(hb.n[b])
        kw = scenarios.band_kwargs(big, b)
        gr = O.graph(p, big.poses[b], n, weight_multiplier=2.0, MW=outg["assoc"].shape[2], **kw)
        check_structure(p, big, outg, b, gr, "ka2_global_table/graph_cases")
        # the far rows add exactly zero terms (they are associated only where obstacle_poses_affected >= n)
        for k in ("Hb", "chi_fam", "via_idx"):
            assert _same(outg[k][b], out[k][b]), f"band {b}: {k} differs on the global-table path"
        t = np.isfinite(_oracle(p, hb, b, 1)[2]["dyn_t"])
        assert _same(outg["dyn_t"][b, :n][t], out["dyn_t"][b, :n][t])


# ------------------------------------------------------------------ e. same bits wherever and however it runs
def test_band_gives_the_same_bits_at_any_batch_position():
    p = _shape_params()
    ns = [30, 3, 121, 59, 116, 5, 233]
    hb = _shape_batch(ns, 240, two_scenes=True)
    g = _ctx(hb, p, max_bands=2 * len(ns))
    try:
        ref = _run(g, hb, 2)
        rng = np.random.default_rng(4)
        for _ in range(3):
            perm = rng.permutation(len(ns))
            moved = _batch_subset(hb, np.concatenate([perm, perm[:2]]))
            out = _run(g, moved, 2)
            for pos, b in enumerate(np.concatenate([perm, perm[:2]])):
                n = int(hb.n[b])
                for k in ("Hb", "chi_fam", "assoc", "via_idx", "dyn_t"):
                    a, c = out[k][pos], ref[k][b]
                    if k in ("assoc", "dyn_t"):
                        a, c = a[:n], c[:n]
                    assert _same(a, c), f"band {b} at position {pos}: {k}"
    finally:
        g.close()


def _batch_subset(hb, idx):
    idx = np.asarray(idx)
    return abi.HostBatch(hb.poses[idx], hb.n[idx], hb.obstacles, hb.obst_count, hb.scene_id[idx], hb.via[idx],
                         hb.via_count[idx], hb.vel_start[idx], hb.vel_goal[idx], hb.prefer_rotdir[idx])


def _check_listed(full, out, hb, listed, what):
    for b in range(hb.B):
        if b in listed:
            for k in ("Hb", "chi_fam", "assoc", "assoc3", "via_idx", "dyn_t", "occ"):
                assert _same(out[k][b], full[k][b]), f"{what}: listed band {b}: {k}"
        else:
            for k in ("Hb", "chi_fam", "assoc", "assoc3", "dyn_t"):
                assert _ones(out[k][b]), f"{what}: unlisted band {b}: {k} written"
            if hb.V_cap:
                assert (out["via_idx"][b] == -1).all()


@pytest.mark.parametrize("name", ["C2", "legacy", "via_ordered", "shapes_polygon", "holonomic"])
def test_listed_launch_touches_only_its_bands(name):
    p, hb = scenarios.scenario(name, candidates=6)
    g = _ctx(hb, p)
    rng = np.random.default_rng(len(name))
    try:
        full = _run(g, hb, 1)
        lists = [[], list(range(hb.B)), list(range(hb.B))[::-1], [int(hb.B - 1), 0], list(rng.permutation(hb.B)[:3])]
        for lst in lists:
            out = _run(g, hb, 1, bands=lst)
            _check_listed(full, out, hb, set(lst), f"{name} list {lst}")
    finally:
        g.close()


def test_listed_launch_on_the_global_table_path():
    p, hb = scenarios.scenario("C3", candidates=5)
    big = _padded(hb, 1100)
    g = _ctx(big, p)
    try:
        full = _run(g, big, 1)
        for lst in ([3, 1], [], [4, 3, 2, 1, 0]):
            _check_listed(full, _run(g, big, 1, bands=lst), big, set(lst), f"global table, list {lst}")
    finally:
        g.close()


def test_band_list_refused_with_the_velocity_obstacle_ratio():
    p, hb = scenarios.scenario("vor")
    g = _ctx(hb, p)
    try:
        with pytest.raises(T.TebGpuError, match="velocity-obstacle ratio"):
            _run(g, hb, 0, bands=[0])
        _run(g, hb, 0)
    finally:
        g.close()
