"""Pins the oracle restatement (oracle/teb_oracle.c) against the REFERENCE'S OWN CODE: oracle/_ref/libteb_ref.so is
src/optimal_planner.cpp + src/timed_elastic_band.cpp + src/obstacles.cpp and their headers compiled where they lie,
with stand-ins only for the absent third-party code (Eigen, boost, ROS messages, the g2o optimizer; oracle/ref_shims/).

What is compared: TebConfig() defaults, penalties.h, every footprint x obstacle distance, the graph buildGraph() builds
edge by edge (errors, information, Jacobians incl. the two analytic overrides), H / b / chi2, whole optimizeTEB calls
(poses, n, cost, number of LM trials), computeCurrentCost outside optimizeTEB, autoResize, initTrajectoryToGoal,
updateAndPruneTEB. The bar is BIT EQUALITY (both sides are fp64, compiled without FMA contraction); where a libm call
order differs the tolerance is written at the assertion.

Runs against the library wherever it exists, and everywhere else against the calls recorded from it
(tests/golden/golden_ref_calls_v1.npz, see tests/ref_binding.py): bit-equal comparisons hold against the digests of the
reference's arrays, tolerances against its stored values."""
import ctypes as C
import os

import numpy as np
import pytest

from teb_local_planner_b200 import abi, scenes
from tests import ref_binding as rb
from tests import scenarios

pytestmark = pytest.mark.skipif(not rb.available(), reason="neither oracle/_ref/libteb_ref.so nor its recorded calls exist")
GOLDEN_REF = os.path.join(os.path.dirname(__file__), "golden", "golden_ref_v1.npz")


def test_default_params_are_the_reference_constructor_defaults(teblib):
    ref = rb.default_params()
    mine = abi.default_params()
    lib = abi.TebParams()
    teblib.tebgpu_default_params(C.byref(lib))
    for name, _ in abi.TebParams._fields_:
        if name.startswith("_"):
            continue
        a, b, c = getattr(ref, name), getattr(mine, name), getattr(lib, name)
        if isinstance(a, C.Array):
            assert list(a) == list(b) == list(c), name
        else:
            assert a == b == c, name


def test_penalties_bit_equal(oracle):
    L = oracle.lib()
    rng = np.random.default_rng(0)
    vals = np.concatenate([rng.normal(0, 1, 4000), [0.0, 0.35, -0.35, 0.4, -0.4, 0.45, 0.05, -0.05, 0.5, 0.55, 0.6]])
    calls, mine = [], []
    for v in vals:
        for a, eps in ((0.4, 0.05), (0.3, 0.0), (0.5, 0.05)):
            calls += [(0, v, a, 0.0, eps), (1, v, -0.2, a, eps), (2, v, a, 0.0, eps)]
            mine += [L.teb_oracle_penalty_interval(v, a, eps), L.teb_oracle_penalty_interval2(v, -0.2, a, eps),
                     L.teb_oracle_penalty_below(v, a, eps)]
    assert rb.same(np.array(mine), rb.penalties(calls))


@pytest.mark.parametrize("footprint", ["point", "circular", "two_circles", "line", "polygon"])
def test_distances_every_footprint_and_obstacle_type(oracle, footprint):
    p, hb = scenarios.scenario("shapes_" + footprint, candidates=2)
    obst = hb.obstacles[0][:hb.obst_count[0]]
    kinds = set(int(o["type"]) for o in obst)
    assert kinds >= {abi.TEB_OBST_POINT, abi.TEB_OBST_LINE, abi.TEB_OBST_PILL, abi.TEB_OBST_POLYGON}
    circ = obst[0].copy()
    circ["type"], circ["radius"] = abi.TEB_OBST_CIRCULAR, 0.3
    rng = np.random.default_rng(5)
    poses, obsts, ts, d_orc = [], [], [], []
    for o in list(obst) + [circ]:
        if not o["dynamic"]:            # a static obstacle has no velocity in the reference (obstacles.h:206 sets both)
            o = o.copy()
            o["vx"], o["vy"] = 0.0, 0.0
        for _ in range(12):
            pose = np.array([o["x"] + rng.normal(0, 1.0), o["y"] + rng.normal(0, 1.0), rng.uniform(-np.pi, np.pi)])
            for t in (None, 0.0, 1.7):
                poses.append(pose)
                obsts.append(o)
                ts.append(-1.0 if t is None else t)
                d_orc.append(oracle.distance(p, pose, o, hb.obst_vertices[0], 0.0 if t is None else t) if (t is not None) else
                             _static_distance(oracle, p, pose, o, hb.obst_vertices[0]))
    d_ref = rb.distances(p, np.array(poses), np.array(obsts), hb.obst_vertices[0], ts)
    worst = np.abs(d_ref - np.array(d_orc)).max()
    assert worst <= 1e-15, worst


def _static_distance(oracle, p, pose, o, verts):
    """calculateDistance ignores the obstacle's velocity: evaluate the oracle on a static copy"""
    s = o.copy()
    s["dynamic"], s["vx"], s["vy"] = 0, 0.0, 0.0
    return oracle.distance(p, pose, s, verts, 0.0)


@pytest.mark.parametrize("name", scenarios.ALL)
def test_graph_edges_and_normal_equations_bit_equal(oracle, name):
    """buildGraph + computeActiveErrors + buildSystem: every active edge (dimension, vertex ids, error, information,
    Jacobian) and the assembled H / b / chi2, for obstacle weight multipliers 1 and 4"""
    p, hb = scenarios.scenario(name)
    for b in range(hb.B):
        n = int(hb.n[b])
        kw = scenarios.band_kwargs(hb, b)
        for wm in (1.0, 4.0):
            Ho, bo, co = oracle.build_system(p, hb.poses[b], n, weight_multiplier=wm, jac_mode=oracle.JAC_G2O, **kw)
            Hr, br, cr, er = rb.build_system(p, hb.poses[b], n, weight_multiplier=wm, want_edges=True, **kw)
            eo = oracle.dump_edges(p, hb.poses[b], n, weight_multiplier=wm, jac_mode=oracle.JAC_G2O, **kw)
            assert eo.shape == er.shape, (name, b, eo.shape, er.shape)
            if isinstance(er, np.ndarray):      # the library itself: name the part that differs
                assert np.array_equal(eo[:, :8], er[:, :8]), "errors / information differ"
                assert np.array_equal(eo[:, 53:], er[:, 53:]), "graph structure differs"
            assert rb.same(eo, er), "Jacobians differ"
            assert rb.same(Ho, Hr) and rb.same(bo, br) and co == cr


@pytest.mark.parametrize("name", scenarios.ALL)
def test_optimize_teb_bit_equal(oracle, name):
    """whole optimizeTEB calls (outer x inner LM iterations, autoResize, weight adaptation, cost): poses, n, cost and
    the number of LM trials of the reference's code and of the restatement are identical"""
    p, hb = scenarios.scenario(name)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale,
                         p.selection_viapoint_cost_scale, False)
    for b in range(hb.B):
        n = int(hb.n[b])
        kw = scenarios.band_kwargs(hb, b)
        ro, co, so = oracle.optimize_band(p, hb.poses[b], n, args=args, jac_mode=oracle.JAC_G2O, n_cap=hb.n_cap, **kw)
        rr, cr, sr, ok = rb.optimize_band(p, hb.poses[b], n, args=args, n_cap=hb.n_cap, **kw)
        assert ok and len(ro) == len(rr), (name, b, len(ro), len(rr))
        assert rb.same(ro, rr), (name, b)
        assert co == cr
        assert so.lm_trials == sr["lm_trials"] and so.rejected == sr["rejected"]
        assert bool(so.status & abi.TEB_STATUS_TERMINATED) == sr["terminated"]


def test_optimize_teb_alternative_time_cost_and_disabled(oracle):
    p, hb = scenarios.scenario("C2")
    kw = scenarios.band_kwargs(hb, 0)
    args = abi.make_args(3, 2, True, 7.0, 3.0, True)
    ro, co, so = oracle.optimize_band(p, hb.poses[0], int(hb.n[0]), args=args, jac_mode=oracle.JAC_G2O, **kw)
    rr, cr, sr, ok = rb.optimize_band(p, hb.poses[0], int(hb.n[0]), args=args, **kw)
    assert ok and rb.same(ro, rr) and co == cr
    p.optimization_activate = 0        # optimizeTEB returns false before touching anything (optimal_planner.cpp:185)
    rr, cr, sr, ok = rb.optimize_band(p, hb.poses[0], int(hb.n[0]), args=args, **kw)
    ro, co, so = oracle.optimize_band(p, hb.poses[0], int(hb.n[0]), args=args, jac_mode=oracle.JAC_G2O, **kw)
    # (isOptimized() is not checked: the constructor used here leaves optimized_ uninitialised, optimal_planner.cpp:67-70)
    assert not ok and rb.same(hb.poses[0][:hb.n[0]], rr) and rb.same(ro, rr)
    assert not (so.status & abi.TEB_STATUS_OPTIMIZED)


def test_divergence_detection_matches(oracle):
    """hasDiverged (optimal_planner.cpp:1023-1039): chi2 of the final state vs divergence_detection_max_chi_squared"""
    p, hb = scenarios.scenario("divergence")
    args = abi.make_args(5, 4, True, 100.0, 1.0, False)
    seen = set()
    for thr in (10, 100000):
        p.divergence_detection_max_chi_squared = thr
        for b in range(hb.B):
            kw = scenarios.band_kwargs(hb, b)
            ro, co, so = oracle.optimize_band(p, hb.poses[b], int(hb.n[b]), args=args, jac_mode=oracle.JAC_G2O, **kw)
            rr, cr, sr, ok = rb.optimize_band(p, hb.poses[b], int(hb.n[b]), args=args, **kw)
            assert rb.same(ro, rr) and co == cr
            assert sr["diverged"] == (so.chi2_final > thr)
            seen.add(sr["diverged"])
    assert seen == {True, False}


def test_compute_cost_outside_optimize_is_undefined_in_the_reference(oracle):
    """computeCurrentCost on a FRESH graph (optimal_planner.cpp:1045-1051, the path HomotopyClassPlanner::
    computeCurrentCost takes): buildGraph + initializeOptimization never evaluate an edge and computeInitialGuess does
    nothing for TEB edges, so edge->chi2() reads the `_error` members as constructed. Upstream g2o leaves them
    uninitialised (Eigen does not zero): the reference's value is undefined. With the zero-initialising stand-in the
    reference code returns exactly 0 (only the alternative time cost survives) - which documents that nothing on that
    path computes errors. tebgpu_compute_cost defines the call as the scaled chi2 AT the current state instead
    (DESIGN.md); that value is what the restatement below computes, and the GPU test checks the C-ABI against it."""
    p, hb = scenarios.scenario("C2")
    kw = scenarios.band_kwargs(hb, 0)
    n = int(hb.n[0])
    assert rb.compute_cost(p, hb.poses[0], n, args=abi.make_args(5, 4, True, 50.0, 2.5, False), **kw) == 0.0
    alt = rb.compute_cost(p, hb.poses[0], n, args=abi.make_args(5, 4, True, 50.0, 2.5, True), **kw)
    t = 0.0
    for i in range(n - 1):              # getSumOfAllTimeDiffs (timed_elastic_band.cpp:184-192), same summation order
        t += hb.poses[0][i, 3]
    assert alt == t
    assert _cost_from_oracle(oracle, p, hb, 0, abi.make_args(5, 4, True, 50.0, 2.5, False)) > 0


def _cost_from_oracle(oracle, p, hb, b, args):
    """scaled chi2 by family at the current state: chi2 is linear in the information weights and a zero weight removes
    the family's edges (optimal_planner.cpp:337, :342, :677), so differences of oracle builds isolate the families. A
    zero obstacle weight also removes the velocity-obstacle ratio edges (obstacles_per_vertex_ stays empty), which
    computeCurrentCost does not scale: the obstacle part is taken with the ratio edges switched off on both sides"""
    kw = scenarios.band_kwargs(hb, b)
    n = int(hb.n[b])

    def chi(q):
        return oracle.build_system(q, hb.poses[b], n, jac_mode=oracle.JAC_G2O, **kw)[2]
    base = chi(p)
    q = type(p).from_buffer_copy(p)
    q.weight_velocity_obstacle_ratio = 0
    no_ratio = chi(q)
    q.weight_obstacle, q.weight_inflation, q.weight_dynamic_obstacle, q.weight_dynamic_obstacle_inflation = 0, 0, 0, 0
    obst = no_ratio - chi(q)
    q = type(p).from_buffer_copy(p)
    q.weight_viapoint = 0
    via = base - chi(q)
    return args.obst_cost_scale * obst + args.viapoint_cost_scale * via + (base - obst - via)


@pytest.mark.parametrize("case", ["large_at_end", "small_at_end", "middle_and_end"])
def test_autoresize_reference_gtests_on_reference_code(oracle, teblib, case):
    """test/teb_basics.cpp:5-68 (the reference's own gtests): same inputs, same assertions, executed on the reference's
    TimedElasticBand; the restatement and the product's host routine must return the identical band"""
    dt, hyst = 0.1, 0.1 / 3.0
    dts = [dt] * 9
    if case == "large_at_end":
        dts.append(dt + 2 * hyst)
    elif case == "small_at_end":
        dts.append(dt - 2 * hyst)
    else:
        dts[5] = dt + 2 * hyst
        dts.append(dt - 2 * hyst)
    n = len(dts) + 1
    rec = np.zeros((64, 4))
    rec[:n, 0] = np.arange(n)
    rec[:n - 1, 3] = dts
    out = rb.auto_resize(rec, n, dt, hyst, 3, 100, False, n_cap=64)
    restated = oracle.auto_resize(rec, n, dt, hyst, 3, 100, False, n_cap=64)
    assert rb.same(restated, out)
    d = restated[:-1, 3]                # == the reference's band, bit for bit
    assert np.all(d <= dt + hyst + 1e-3) and np.all(dt - hyst - 1e-3 <= d)     # ASSERT_LE pairs of the gtest
    mine = rec.copy()
    nn = teblib.tebgpu_auto_resize_host(mine.ctypes.data, n, 64, dt, hyst, 3, 100, 0)
    assert nn == len(out) and rb.same(mine[:nn], out)


def test_autoresize_random_bit_equal(oracle):
    rng = np.random.default_rng(2)
    for k in range(300):
        n = int(rng.integers(3, 40))
        rec = np.zeros((n, 4))
        rec[:, 0] = np.cumsum(rng.uniform(0.0, 0.3, n))
        rec[:, 1] = rng.normal(0, 0.5, n)
        rec[:, 2] = rng.uniform(-3.2, 3.2, n)
        rec[:n - 1, 3] = rng.choice([0.05, 0.1, 0.29, 0.3, 0.41, 0.8, 1.5], n - 1) * rng.uniform(0.9, 1.1, n - 1)
        fast = bool(k % 2)
        a = rb.auto_resize(rec, n, 0.3, 0.1, int(rng.integers(3, 6)) if k % 3 else 3, int(rng.choice([12, 50, 500])), fast, n_cap=1024)
    # the same sequence again for both implementations (rng consumed identically above would hide argument differences)
    rng = np.random.default_rng(2)
    for k in range(300):
        n = int(rng.integers(3, 40))
        rec = np.zeros((n, 4))
        rec[:, 0] = np.cumsum(rng.uniform(0.0, 0.3, n))
        rec[:, 1] = rng.normal(0, 0.5, n)
        rec[:, 2] = rng.uniform(-3.2, 3.2, n)
        rec[:n - 1, 3] = rng.choice([0.05, 0.1, 0.29, 0.3, 0.41, 0.8, 1.5], n - 1) * rng.uniform(0.9, 1.1, n - 1)
        fast = bool(k % 2)
        mn = int(rng.integers(3, 6)) if k % 3 else 3
        mx = int(rng.choice([12, 50, 500]))
        a = rb.auto_resize(rec, n, 0.3, 0.1, mn, mx, fast, n_cap=1024)
        c = oracle.auto_resize(rec, n, 0.3, 0.1, mn, mx, fast, n_cap=1024)
        assert a.shape == c.shape and rb.same(c, a), k


def test_init_trajectory_bit_equal(oracle):
    rng = np.random.default_rng(4)
    for k in range(100):
        start = np.array([rng.normal(0, 2), rng.normal(0, 2), rng.uniform(-3, 3)])
        goal = start + np.array([rng.normal(0, 3), rng.normal(0, 3), rng.uniform(-1, 1)])
        diststep = float(rng.choice([0.0, 0.1, 0.35]))
        back = bool(k % 4 == 0)
        a = rb.init_trajectory(start, goal, diststep, 0.4, int(rng.integers(3, 8)) if k % 2 else 3, back, n_cap=2048)
    rng = np.random.default_rng(4)
    for k in range(100):
        start = np.array([rng.normal(0, 2), rng.normal(0, 2), rng.uniform(-3, 3)])
        goal = start + np.array([rng.normal(0, 3), rng.normal(0, 3), rng.uniform(-1, 1)])
        diststep = float(rng.choice([0.0, 0.1, 0.35]))
        back = bool(k % 4 == 0)
        ms = int(rng.integers(3, 8)) if k % 2 else 3
        a = rb.init_trajectory(start, goal, diststep, 0.4, ms, back, n_cap=2048)
        c = oracle.init_trajectory(start, goal, diststep, 0.4, ms, back, n_cap=2048)
        assert a.shape == c.shape and rb.same(c, a), k


def test_golden_reference_vectors_are_current():
    """the committed fixture was generated from THIS reference build: regenerate a slice and compare"""
    from tests.golden import make_golden_ref
    z = np.load(GOLDEN_REF, allow_pickle=False)
    names = ("C1", "via_ordered")
    keys = sorted(k for k in z.files if k.split("/")[0] in names)
    fresh = rb.recorded("golden_ref_slice", keys, lambda: [make_golden_ref.generate(only=names)[k] for k in keys])
    assert len(fresh) == len(keys)
    for k, v in zip(keys, fresh):
        assert rb.same(z[k], v), k


@pytest.mark.parametrize("cfg", ["C1", "C2", "C3", "C4"])
def test_h_signatures_match_the_reference_header(oracle, cfg):
    """calculateEquivalenceClass executed by the reference's own h_signature.h (HSignature: long double complex
    accumulation; HSignature3d: numeric integration over the x-y-t obstacle 'conductors', with and without the band's
    time differences) against the oracle restatement, plus isValid / isReasonable and the class comparison the planner
    derives from them. 2-D: relative 1e-15 of the long double result; 3-D: bit equal."""
    from tests.golden import make_golden
    p, hb = scenes.make_config_batch(cfg, candidates=6, seed=17)
    obst = hb.obstacles[0][:hb.obst_count[0]]
    sig2 = []
    for b in range(hb.B):
        rec, n = hb.poses[b], int(hb.n[b])
        p.include_dynamic_obstacles = 0
        want, valid, reasonable = rb.h_signature(p, rec, n, obst)
        got = oracle.h_signature(p, rec, n, obst)
        assert valid and np.isfinite(want.real) and np.isfinite(want.imag)
        assert abs(got - want) <= 1e-15 * max(1.0, abs(want)), (cfg, b, got, want)
        sig2.append((got, want))
        p.include_dynamic_obstacles = 1
        for use_dt in (True, False):
            want3, valid3, reasonable3 = rb.h_signature(p, rec, n, obst, use_timediffs=use_dt)
            got3 = oracle.h_signature(p, rec, n, obst, use_timediffs=use_dt)
            assert valid3
            assert np.array_equal(got3, want3), (cfg, b, use_dt, np.abs(got3 - want3).max())
            assert reasonable3 == bool(np.all(want3 <= 1.0))
    # HSignature::isEqual (h_signature.h:195-206): both parts within h_signature_threshold - same partition either way
    thr = p.h_signature_threshold
    eq = lambda x, y: abs(x.real - y.real) <= thr and abs(x.imag - y.imag) <= thr
    for i in range(hb.B):
        for j in range(hb.B):
            assert eq(sig2[i][0], sig2[j][0]) == eq(sig2[i][1], sig2[j][1])
    # the committed H-signature fixtures (tests/golden/golden_v2.npz) agree with the reference header as well
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_v2.npz"), allow_pickle=False)
    for name, pp, hbb in make_golden.hsig_cases():
        ob = hbb.obstacles[0][:hbb.obst_count[0]]
        for b in range(hbb.B):
            want, _, _ = rb.h_signature(pp, hbb.poses[b], hbb.n[b], ob)
            have = g[name][b]
            if pp.include_dynamic_obstacles:
                assert np.array_equal(want, have[:len(ob)])
            else:
                assert abs(want - complex(have[0], have[1])) <= 1e-15 * max(1.0, abs(want))


def _explorer_inputs(rng, n_obst, dynamic):
    from oracle import hcp_explore as X
    rows = np.zeros(n_obst, abi.OBST_DTYPE)
    obstacles, pool = [], []
    for m in range(n_obst):
        kind = ["point", "circle", "line"][int(rng.integers(3))]
        c = np.array([rng.uniform(-3.2, 3.2), rng.uniform(-1.6, 1.6)])
        if kind == "point":
            rows[m]["type"], rows[m]["x"], rows[m]["y"] = abi.TEB_OBST_POINT, c[0], c[1]
            obstacles.append(X.Obst("point", tuple(c)))
        elif kind == "circle":
            r = rng.uniform(0.1, 0.4)
            rows[m]["type"], rows[m]["x"], rows[m]["y"], rows[m]["radius"] = abi.TEB_OBST_CIRCULAR, c[0], c[1], r
            obstacles.append(X.Obst("circle", tuple(c), r))
        else:
            d = rng.normal(0, 0.35, 2)
            a, b = c - d, c + d
            rows[m]["type"], rows[m]["vertex_begin"], rows[m]["vertex_count"] = abi.TEB_OBST_LINE, len(pool), 2
            pool += [a, b]
            ctr = 0.5 * (a + b)
            rows[m]["x"], rows[m]["y"] = ctr[0], ctr[1]
            obstacles.append(X.Obst("line", tuple(ctr), vertices=[tuple(a), tuple(b)]))
        if dynamic and rng.random() < 0.4:
            rows[m]["vx"], rows[m]["vy"], rows[m]["dynamic"] = rng.normal(0, 0.1), rng.normal(0, 0.1), 1
    return rows, obstacles, (np.array(pool) if pool else None)


@pytest.mark.parametrize("prm", [False, True])
@pytest.mark.parametrize("dynamic", [0, 1])
def test_candidate_exploration_matches_the_reference_planner(oracle, prm, dynamic):
    """exploreEquivalenceClassesAndInitTebs of the reference's own HomotopyClassPlanner / graph_search.cpp (key-point graph
    and probabilistic roadmap, DepthFirst enumeration order, addAndInitNewTeb with the path variant of
    initTrajectoryToGoal, H-signature filtering with both signature kinds, class budget) against the sequential
    restatement oracle/hcp_explore.py - the one the GPU test of the drop-in planner is compared with. Same candidates, same
    order, initial bands equal to 1e-12 (the restatement evaluates atan2 / hypot in Python). The roadmap's random stream is
    boost's (absent from the image): both sides restate the same published generator, so that part pins consistency only."""
    from oracle import hcp_explore as X
    rng = np.random.default_rng(100 + 2 * int(prm) + dynamic)
    for case in range(12):
        p = abi.default_params()
        p.include_dynamic_obstacles = dynamic
        rows, obstacles, pool = _explorer_inputs(rng, int(rng.integers(2, 7)), dynamic)
        hcp = {"max_number_classes": int(rng.integers(2, 8)), "obstacle_heading_threshold": [0.0, 0.45, 0.7][int(rng.integers(3))],
               "roadmap_graph_area_width": rng.uniform(3, 7), "roadmap_graph_area_length_scale": [1.0, 0.8][int(rng.integers(2))],
               "roadmap_graph_no_samples": int(rng.integers(5, 16))}
        start = [-4.0, rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4)]
        goal = [4.0, rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4)]
        cycles = 2
        want = rb.hcp_explore(p, hcp, start, goal, rows, pool, cycles=cycles, prm=prm)
        ex = X.Explorer(p, hcp, oracle, rows, obstacles)
        for c in range(cycles):
            ex.classes, ex.tebs = [], []
            (ex.prob_roadmap_graph if prm else ex.lr_key_point_graph)(start, goal, p.min_obstacle_dist)
            assert len(ex.tebs) == len(want[c]), (case, c, len(ex.tebs), len(want[c]))
            for k, (got, ref) in enumerate(zip(ex.tebs, want[c])):
                assert got.shape == ref.shape, (case, c, k, got.shape, ref.shape)
                assert np.abs(got - ref).max() < 1e-12, (case, c, k, np.abs(got - ref).max())


@pytest.mark.parametrize("prm", [False, True])
def test_planning_cycles_match_the_reference_planner(oracle, teblib, prm):
    """consecutive HomotopyClassPlanner::plan(start, goal) calls of the reference's own planner (updateAllTEBs,
    renewAndAnalyzeOldTebs, deletePlansDetouringBackwards, graph exploration, optimizeAllTEBs, selectBestTeb) against the
    sequential restatement oracle/hcp_explore.py::Planner with the start pose moving along: same number of candidates,
    same order, same pose counts, same selected candidate in every cycle. The reference optimises with numeric Jacobians
    (the restatement is switched to that mode); initial bands that differ in the last bit (Python vs C atan2 / hypot) come
    out ~1e-7 apart after 20 LM iterations, hence 1e-5 on poses (less the rounding of recorded bands, which are stored
    in fixed point) and 1e-6 relative on costs.
    The reference's TebConfig constructor leaves hcp.max_number_plans_in_current_class uninitialised (candidate counts
    varied from process to process until oracle/ref_driver.cpp set the dynamic_reconfigure default 1)."""
    from oracle import hcp_explore as X
    rng = np.random.default_rng(300 + int(prm))
    for case in range(5):
        p = abi.default_params()
        p.include_dynamic_obstacles = 0
        p.selection_cost_hysteresis = [1.0, 0.9, 0.8][case % 3]
        carried_best = False
        rows, obstacles, pool = _explorer_inputs(rng, int(rng.integers(2, 5)), 0)
        hcp = {"max_number_classes": int(rng.integers(2, 5)), "obstacle_heading_threshold": 0.45,
               "roadmap_graph_area_width": 5.0, "roadmap_graph_area_length_scale": 1.0, "roadmap_graph_no_samples": 10}
        goal = [4.0, rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2)]
        starts = [[-4.0 + 0.2 * c, 0.03 * c + rng.normal(0, 0.01), 0.05] for c in range(4)]
        want = rb.hcp_plan(p, hcp, starts, goal, rows, pool, prm=prm)
        pl = X.Planner(p, hcp, oracle, rows, obstacles, simple_exploration=not prm)
        pl.jac_mode = oracle.JAC_G2O
        pl.obst_vertices = pool
        args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, p.selection_viapoint_cost_scale,
                             bool(p.selection_alternative_time_cost))
        for c, (ok, best, cands) in enumerate(want):
            got_best = pl.plan(starts[c], goal, args, abi)
            assert ok and len(pl.tebs) == len(cands), (case, c, len(pl.tebs), len(cands))
            assert (got_best if got_best is not None else -1) == best, (case, c, got_best, best)
            # tebgpu_select_best (the C-ABI's selectBestTeb, a pure host function) on the REFERENCE's own costs: the band the
            # planner carried over as its best one sits at index 0 after renewAndAnalyzeOldTebs
            costs_ref = np.array([x for x, _ in cands])
            last = 0 if (c > 0 and carried_best) else -1
            assert teblib.tebgpu_select_best(costs_ref.ctypes.data, len(costs_ref), last, -1, float(p.selection_cost_hysteresis),
                                             float(p.selection_prefer_initial_plan)) == best, (case, c)
            carried_best = best >= 0
            for k, ((cost, band), rec) in enumerate(zip(cands, pl.tebs)):
                assert band.shape == rec.shape, (case, c, k, band.shape, rec.shape)
                assert np.abs(band - rec).max() < 1e-5 - rb.storage_error(), (case, c, k, np.abs(band - rec).max())
                assert abs(cost - pl.costs[k]) <= 1e-6 * max(1.0, abs(cost)), (case, c, k, cost, pl.costs[k])
