"""Kernel A, the trial evaluation and whole optimize calls at every parameter switch of buildGraph (run on an H100:
pytest -m gpu). The configurations of tests/param_cases.py take each predicate of make_kparams (csrc/teb_cabi.cu) to
both sides and to its boundary; tests/test_reference_pin_params.py holds the oracle to the reference's own code there.
For every configuration:
  a. build_system(graph=True) at outer 0 and 3 against the oracle with test_gpu_linearize.check_band (H|b within
     1e-12, chi2 per family, association / assoc3 / via / dynamic-time words bit-equal), staged and, with the scene
     padded past 1024 rows, on the global-table path; the generic (GEOM) build wherever the footprint or the obstacle
     rows need it. The worst errors per configuration go to the parity report;
  b. one round of trial evaluation on real LM steps against the oracle's trial chi2 and g2o's accept / reject
     (test_gpu_trial_eval.check_chi2 / check_decisions);
  c. optimize against the oracle in closed-form mode: n, LM iterations and status (failed factorisations included)
     identical, poses within 1e-6, cost within 1e-6 relative; in the latency regime with graph replay and in the
     throughput regime (the batch replicated past 2 x SMs, so k_trial_eval2p and k_solve_tpb_rc run). Against the
     reference's results the per-band rule of DESIGN.md §3: within 1e-4, or the band is one where the CPU
     implementation's two Jacobian modes part ways by more than 1e-5 (the oracle's g2o mode stands for the reference:
     tests/test_reference_pin_params.py holds the two bit-equal at these configurations);
  d. one context stepped through every configuration with set_params, graph replay on: each call gives the bits of a
     fresh context with that configuration (params_version in the graph key, the footprint copy);
  e. compute_cost and the finalize cost with non-default selection scales and the alternative time cost."""
import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi
from tests import param_cases as pc
from tests import scenarios
from tests import test_gpu_linearize as LZ
from tests import test_gpu_trial_eval as TE

pytestmark = pytest.mark.gpu
POSE_TOL = 1e-6
REF_TOL, SPREAD = 1e-4, 1e-5


def _gpu(hb, p, B=None, graph=None):
    g = T.TebGpu(B or hb.B, hb.n_cap, hb.S, max(hb.M_cap, 1), hb.V_cap, max_obst_vertices=hb.PV_cap)
    g.set_params(p)
    if graph is not None:
        g.set_graph(graph)
    return g


def _tile(hb, B):
    """the batch's bands repeated to B bands (same scene)"""
    idx = np.arange(B) % hb.B
    return abi.HostBatch(hb.poses[idx], hb.n[idx], hb.obstacles, hb.obst_count, hb.scene_id[idx], hb.via[idx],
                         hb.via_count[idx], hb.vel_start[idx], hb.vel_goal[idx], hb.prefer_rotdir[idx],
                         hb.obst_vertices if hb.PV_cap else None)


def _optimize(hb, p, a, B=None, graph=None):
    g = _gpu(hb, p, B, graph)
    try:
        h = hb.copy()
        g.optimize(h, a)
    finally:
        g.close()
    return h


def _oracle_runs(oracle, p, hb, a, jac):
    return [oracle.optimize_band(p, hb.poses[b], int(hb.n[b]), args=a, jac_mode=jac, n_cap=hb.n_cap,
                                 **scenarios.band_kwargs(hb, b)) for b in range(hb.B)]


def _check_against_oracle(h, runs, nb, what):
    for q in range(h.B):
        ro, co, so = runs[q % nb]
        where = (what, q)
        assert h.n[q] == len(ro), where
        d = np.abs(h.poses[q, :h.n[q]] - ro)
        assert np.array_equal(np.isnan(h.poses[q, :h.n[q]]), np.isnan(ro)), where
        assert np.nanmax(d, initial=0.0) <= POSE_TOL, (where, np.nanmax(d, initial=0.0))
        assert h.status[q] == so.status and h.lm_iters[q] == so.lm_iters, (where, h.status[q], so.status, h.lm_iters[q], so.lm_iters)
        assert (np.isnan(h.cost[q]) and np.isnan(co)) or h.cost[q] == co or abs(h.cost[q] - co) <= 1e-6 * abs(co) + 1e-12, \
            (where, h.cost[q], co)


# ------------------------------------------------------------------ a. kernel A and the graph build
@pytest.mark.parametrize("name", pc.ALL)
def test_graph_build_against_oracle(name):
    p, hb = pc.case(name)
    big = LZ._padded(hb, 1100)
    g, gg = LZ._ctx(hb, p), LZ._ctx(big, p)
    try:
        for outer in (0, 3):
            out = LZ._run(g, hb, outer)
            for b in range(hb.B):
                LZ.check_band(p, hb, out, b, outer, f"params/{name}")
            outg = LZ._run(gg, big, outer)
            for b in range(hb.B):
                LZ.check_band(p, big, outg, b, outer, f"params_global_table/{name}")
    finally:
        g.close()
        gg.close()


# ------------------------------------------------------------------ b. one round of trial evaluation
@pytest.mark.parametrize("name", pc.ALL)
def test_trial_round_against_oracle(name):
    p, hb = pc.case(name)
    g = TE._ctx(hb, p)
    try:
        for outer in (0, 3):
            g.build_system(hb, outer)
            dx, ok, lam = g.solve_system(hb.n.copy(), 4, n_cap=hb.n_cap)
            rd = TE.Round(g, p, hb, 4, dx, ok, lam, TE._state(hb.B), outer, iteration=0)
            list(TE.check_chi2(rd, f"params/{name}"))
            TE.check_decisions(rd, f"params/{name}")
    finally:
        g.close()


# ------------------------------------------------------------------ c. whole optimize calls
@pytest.mark.parametrize("name", pc.ALL)
def test_optimize_against_oracle_and_reference(oracle, name):
    p, hb = pc.case(name)
    a = pc.args(p)
    runs = _oracle_runs(oracle, p, hb, a, oracle.JAC_ANALYTIC)
    lat = _optimize(hb, p, a, graph=1)
    _check_against_oracle(lat, runs, hb.B, "latency")
    B = 2 * TE._sms() + 2 * hb.B
    thr = _optimize(_tile(hb, B), p, a)
    _check_against_oracle(thr, runs, hb.B, "throughput")
    # the reference's results (oracle g2o mode = the reference, bit for bit), per band
    ref = _oracle_runs(oracle, p, hb, a, oracle.JAC_G2O)
    for b in range(hb.B):
        rr, ra = ref[b][0], runs[b][0]
        dn = np.nanmax(np.abs(lat.poses[b, :lat.n[b]] - rr)) if lat.n[b] == len(rr) else np.inf
        spread = np.nanmax(np.abs(ra - rr)) if len(ra) == len(rr) else np.inf
        assert dn <= REF_TOL or spread > SPREAD or np.isnan(spread), (name, b, dn, spread)


# ------------------------------------------------------------------ d. one context through every configuration
def test_set_params_steps_through_every_configuration():
    cases = [(name,) + pc.case(name) for name in pc.ALL]
    pv = max(hb.PV_cap for _, _, hb in cases)
    hb0 = cases[0][2]
    g = T.TebGpu(hb0.B, hb0.n_cap, 1, max(hb.M_cap for _, _, hb in cases), hb0.V_cap, max_obst_vertices=pv)
    g.set_graph(1)
    try:
        for name, p, hb in cases + cases[:3]:
            g.set_params(p)
            h = hb.copy()
            g.optimize(h, pc.args(p))
            fresh = _optimize(hb, p, pc.args(p), graph=1)
            for f in ("poses", "n", "cost", "chi2", "status", "lm_iters"):
                assert np.array_equal(getattr(h, f), getattr(fresh, f), equal_nan=True), (name, f)
    finally:
        g.close()


# ------------------------------------------------------------------ e. costs
COST_CASES = [n for n in pc.ALL if not n.startswith("random_")] + [f"random_{k}" for k in range(8)]


@pytest.mark.parametrize("name", COST_CASES)
def test_costs_with_selection_scales(oracle, name):
    from tests.test_reference_pin import _cost_from_oracle
    p, hb = pc.case(name)
    for alt in (False, True):
        a = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, 37.0, 2.5, alt)
        h = _optimize(hb, p, a, graph=0)
        _check_against_oracle(h, _oracle_runs(oracle, p, hb, a, oracle.JAC_ANALYTIC), hb.B, f"finalize alt={alt}")
    a = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, 37.0, 2.5, False)
    g = _gpu(hb, p)
    try:
        h = hb.copy()
        g.compute_cost(h, a)
    finally:
        g.close()
    for b in range(hb.B):
        want = _cost_from_oracle(oracle, p, hb, b, a)
        assert abs(h.cost[b] - want) <= 1e-9 * max(1.0, abs(want)), (name, b, h.cost[b], want)
