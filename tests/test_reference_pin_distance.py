"""The oracle's footprint-to-obstacle distances (oracle/teb_oracle.c: footprint_dist / footprint_grad and the vertex-list
generic_distance) against the reference's own calculateDistance / estimateSpatioTemporalDistance
(oracle/_ref/libteb_ref.so, see tests/ref_binding.py) on every case of tests/distance_cases.py: contacts, parallel and
collinear edges, closest-point clamps, zero-length segments, ties, containment, distances exactly at the penalty and
association thresholds, polygons of 65 and 70 vertices and moving vertex lists.

  * distance: within 1e-15 of the reference, and equal to the case's exact distance where it claims one (both sides);
  * gradient: off the kinks, the oracle's closed form within 1e-5 (O(h) at a clamp) of a central difference (h = 2^-20) of the
    reference's distance;
  * the whole buildGraph / buildSystem of each case's band (tests/distance_cases.Case.band) in the oracle's numeric
    mode, bit for bit: every edge and H / b / chi2, with the legacy and the non-legacy association, moving obstacles as
    dynamic obstacles and as static ones.

Where the library cannot be built the calls are answered from tests/golden/golden_ref_dist_v1.npz (recorded by
tests/golden/make_golden_ref_dist.py). test_oracle_matches_the_exact_distances needs neither."""
import os
from fractions import Fraction

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import distance_cases as dc
from tests import ref_binding as rb

GOLDEN_DIST = os.path.join(os.path.dirname(__file__), "golden", "golden_ref_dist_v1.npz")
REF_AVAILABLE = rb.live() or os.path.exists(GOLDEN_DIST)
needs_ref = pytest.mark.skipif(not REF_AVAILABLE, reason="neither oracle/_ref/libteb_ref.so nor its recorded distance calls exist")
CASES = {c.name: c for c in dc.all_cases()}
H = 2.0 ** -20
GRAD_BAR = 1e-5       # O(h): at a clamp the distance is only once differentiable


@pytest.fixture(scope="module")
def ref():
    rb.add_recording(GOLDEN_DIST)
    return rb


def _oracle_distance(oracle, case, p, pose=None):
    return oracle.distance(p, case.pose3() if pose is None else pose, case.obst[0], case.verts,
                           0.0 if case.t is None else case.t, want_grad=True)


def _ts(case, k):
    return np.full(k, -1.0 if case.t is None else case.t)


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_distance_and_gradient_match_the_reference(oracle, ref, name):
    case = CASES[name]
    p = case.params()
    d, g = _oracle_distance(oracle, case, p)
    poses = [case.pose3()]
    if case.smooth:
        for k in range(3):
            for s in (1.0, -1.0):
                q = case.pose3()
                q[k] += s * H
                poses.append(q)
    want = ref.distances(p, np.array(poses), np.repeat(case.obst, len(poses)), case.verts, _ts(case, len(poses)))
    assert abs(d - want[0]) <= 1e-15, (name, d, want[0])
    if case.d is not None:
        assert d == float(case.d) and want[0] == float(case.d), (name, d, want[0], case.d)
    if case.smooth:
        fd = np.array([(want[1 + 2 * k] - want[2 + 2 * k]) / (2 * H) for k in range(3)])
        assert np.abs(g - fd).max() <= GRAD_BAR, (name, g, fd)


def test_oracle_matches_the_exact_distances(oracle):
    """without the reference: the oracle returns every claimed exact distance exactly, and on the large polygons the
    correctly rounded distance to the nearest of all their edges (not only of the first 64 vertices)"""
    for case in CASES.values():
        d, _ = _oracle_distance(oracle, case, case.params())
        if case.d is not None:
            assert d == float(case.d), (case.name, d, case.d)
        if case.verts is not None and len(case.verts) > 64:
            tr = dc.trace(case.fp, case.obst, case.verts, case.pose, case.t)
            q = min(tr.parts[0][0])
            assert abs(d - float(q) ** 0.5) <= 1e-15, (case.name, d, float(q) ** 0.5)


def _band_kwargs(case):
    return dict(obstacles=case.obst, obst_vertices=case.verts)


def _modes(case):
    """(legacy association, include_dynamic_obstacles) of the case's band runs"""
    return [(leg, dyn) for leg in (0, 1) for dyn in ((0, 1) if case.t is not None else (0,))]


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_band_graph_and_normal_equations_bit_equal(oracle, ref, name):
    """buildGraph + computeActiveErrors + buildSystem of the case's band: every edge and H / b / chi2"""
    case = CASES[name]
    rec = case.band()
    n = len(rec)
    for leg, dyn in _modes(case):
        p = case.params(legacy_obstacle_association=leg, include_dynamic_obstacles=dyn)
        kw = _band_kwargs(case)
        Ho, bo, co = oracle.build_system(p, rec, n, jac_mode=oracle.JAC_G2O, **kw)
        Hr, br, cr, er = ref.build_system(p, rec, n, want_edges=True, **kw)
        eo = oracle.dump_edges(p, rec, n, jac_mode=oracle.JAC_G2O, **kw)
        assert eo.shape == er.shape, (name, leg, dyn, eo.shape, er.shape)
        if isinstance(er, np.ndarray):
            assert np.array_equal(eo[:, :8], er[:, :8]), (name, leg, dyn, "errors / information differ")
            assert np.array_equal(eo[:, 53:], er[:, 53:]), (name, leg, dyn, "graph structure differs")
        assert rb.same(eo, er), (name, leg, dyn, "Jacobians differ")
        assert rb.same(Ho, Hr) and rb.same(bo, br) and co == cr, (name, leg, dyn)


def test_cases_cover_every_shape_and_edge():
    """every footprint, every obstacle kind and vertex count, static and moving vertex lists, and the named edges"""
    cases = list(CASES.values())
    assert {c.fp for c in cases} == set(dc.FOOTPRINTS)
    kinds = {(int(c.obst["type"][0]), int(c.obst["vertex_count"][0])) for c in cases}
    for want in [(abi.TEB_OBST_POINT, 0), (abi.TEB_OBST_CIRCULAR, 0), (abi.TEB_OBST_LINE, 2), (abi.TEB_OBST_PILL, 2)] + \
            [(abi.TEB_OBST_POLYGON, k) for k in (1, 2, 3, 4, 65, 70)]:
        assert want in kinds, want
    moving = [c for c in cases if c.t is not None]
    assert {int(c.obst["type"][0]) for c in moving} >= {abi.TEB_OBST_POINT, abi.TEB_OBST_LINE, abi.TEB_OBST_PILL,
                                                        abi.TEB_OBST_POLYGON}
    assert any(c.d == 0 for c in moving)
    for prefix in ("cross_", "touch_endpoint_denom_pos", "touch_endpoint_denom_neg", "vertex_on_edge", "collinear_overlap",
                   "pose_on_point", "parallel_tie", "clamp_u0", "clamp_u1", "zero_line", "zero_footprint_line",
                   "corner_bisector", "robot_edges_tie", "tc_tie_point", "tc_tie_circular", "tc_tie_line", "tc_uneq_tie",
                   "robot_inside", "obstacle_inside", "thr_min_eps", "thr_inflation", "thr_dyn_inflation", "thr_force_d",
                   "thr_cut_d", "centroid_dead_ahead", "polygon65_", "polygon70_"):
        assert any(c.name.startswith(prefix) for c in cases), prefix
    thresholds = {c.d for c in cases}
    assert {Fraction(v) for v in (dc.MIN_D + dc.EPS, dc.INFL, dc.DYN_INFL, dc.FORCE_D, dc.CUT_D, 0.0)} <= thresholds
