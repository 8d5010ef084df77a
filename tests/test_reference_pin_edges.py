"""The oracle's optimizeTEB against the reference's own code (oracle/_ref/libteb_ref.so, see tests/ref_binding.py) at the
argument edges of optimizeTEB and on bands built to take one exit of its loops (tests/control_flow_bands.py): no outer
iteration, no inner iteration (optimizeGraph's `if (!iter) return false`, optimal_planner.cpp:393), one of each, and the
defaults; autosize on and off; cost computed or not, with and without the alternative time cost; max_vel_x < 0.01.
Where the library cannot be built the calls are answered from tests/golden/golden_ref_edges_v1.npz (recorded by
tests/golden/make_golden_ref_edges.py)."""
import os

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import control_flow_bands as cf
from tests import ref_binding as rb

GOLDEN_EDGES = os.path.join(os.path.dirname(__file__), "golden", "golden_ref_edges_v1.npz")
pytestmark = pytest.mark.skipif(not (rb.live() or os.path.exists(GOLDEN_EDGES)),
                                reason="neither oracle/_ref/libteb_ref.so nor its recorded argument-edge calls exist")


@pytest.fixture(scope="module")
def ref():
    rb.add_recording(GOLDEN_EDGES)
    return rb


def _bands(oracle, p):
    """(name, rec, n, kwargs): two ordinary bands, Z, S, and a band a second autoResize pass still changes"""
    hb = cf.mixed_batch(["O", "O", "Z", "S"], s_band=cf.shifting_band(p, oracle))
    out = [(k if k in "ZS" else f"{k}{b}", hb.poses[b], int(hb.n[b]), cf.band_kwargs(hb, b)) for b, k in enumerate("OOZS")]
    rec, n = cf.resize_twice_band(p, oracle.auto_resize)
    buf = np.zeros((hb.n_cap, 4))
    buf[:n] = rec
    out.append(("R", buf, n, cf.band_kwargs(hb, 0)))
    return out


def _pin(oracle, ref, p, rec, n, a, kw, n_cap):
    ro, co, so = oracle.optimize_band(p, rec, n, args=a, jac_mode=oracle.JAC_G2O, n_cap=n_cap, **kw)
    rr, cr, sr, ok = ref.optimize_band(p, rec, n, args=a, n_cap=n_cap, **kw)
    assert len(ro) == len(rr) and ref.same(ro, rr)
    assert bool(so.status & abi.TEB_STATUS_OPTIMIZED) == ok
    assert co == cr or (np.isnan(co) and np.isnan(cr))
    assert bool(so.status & abi.TEB_STATUS_TERMINATED) == sr["terminated"]
    assert bool(so.status & abi.TEB_STATUS_CHOL_FAILED) == sr["chol_failed"]
    assert so.lm_trials == sr["lm_trials"] and so.rejected == sr["rejected"]
    return ro, co, so, sr, ok


def test_zero_chi2_band_is_exactly_zero(oracle, ref):
    """Z's defining property: chi2, b and H are exactly 0 in the oracle and in the reference"""
    p = cf.params()
    hb = cf.mixed_batch(["Z"])
    kw = cf.band_kwargs(hb, 0)
    H, b, chi2 = oracle.build_system(p, hb.poses[0], int(hb.n[0]), jac_mode=oracle.JAC_G2O, **kw)
    assert chi2 == 0.0 and not b.any() and not H.any()
    Hr, br, cr = ref.build_system(p, hb.poses[0], int(hb.n[0]), **kw)
    assert cr == 0.0 and ref.same(H, Hr) and ref.same(b, br)


@pytest.mark.parametrize("autosize", [True, False])
@pytest.mark.parametrize("outer,inner", cf.EDGES)
def test_optimize_teb_argument_edges(oracle, ref, outer, inner, autosize):
    """n, poses, optimizeTEB's return value, cost, Terminate and the failed-factorisation flag of the oracle equal the
    reference's for every cost switch; the exits are the ones the construction predicts"""
    p = cf.params(autosize)
    for name, rec, n, kw in _bands(oracle, p):
        for cost, alt in ((True, False), (True, True), (False, False), (False, True)):
            a = cf.args(inner, outer, cost, alt)
            ro, co, so, sr, ok = _pin(oracle, ref, p, rec, n, a, kw, len(rec))
            where = (name, cost, alt)
            if outer == 0:
                # optimizeTEB returns true, optimized_ stays false, no cost
                assert ok and not sr["optimized"] and co == np.inf and so.lm_iters == 0, where
                assert len(ro) == n and np.array_equal(ro, rec[:n]), where
            elif inner == 0:
                # the first outer iteration's autoResize / buildGraph, then optimizeGraph fails: nothing else runs
                assert not ok and not sr["optimized"] and co == np.inf and so.lm_iters == 0, where
                once = oracle.auto_resize(rec, n, p.dt_ref, p.dt_hysteresis, p.min_samples, p.max_samples, 1) if autosize else rec[:n]
                twice = oracle.auto_resize(once, len(once), p.dt_ref, p.dt_hysteresis, p.min_samples, p.max_samples, 1)
                assert name != "R" or not autosize or not np.array_equal(once, twice)   # R's defining property
                assert np.array_equal(ro, once), where
            else:
                assert ok and sr["optimized"] and so.lm_iters <= outer * inner, where
                assert (co == np.inf) == (not cost), where
            if name == "S" and outer == 1 and inner > 0:
                # Z's exit in the first outer iteration: carried into the second, where autoResize changes it again
                assert so.lm_iters == 1 and so.nu_final == 2.0 ** 11 and so.lambda_final == 0.0, where
            if name == "Z" and outer > 0 and inner > 0:
                # ten failed factorisations in the first LM iteration of every outer iteration, Terminate
                assert so.lm_iters == outer and so.nu_final == 2.0 ** 11 and so.lambda_final == 0.0, where
                assert so.status & abi.TEB_STATUS_TERMINATED and so.status & abi.TEB_STATUS_CHOL_FAILED, where
                assert so.lm_trials == 10 * outer and (co == 0.0 or not cost or alt), where
                assert np.array_equal(ro, rec[:n]), where


@pytest.mark.parametrize("outer,inner", cf.EDGES)
def test_nan_band_takes_one_trial_per_iteration(oracle, outer, inner):
    """N: every trial's factorisation fails on a NaN system, rho is NaN, so each LM iteration takes one trial and none
    terminates (oracle only: the reference asserts on the non-finite edge error)"""
    p = cf.params()
    hb = cf.mixed_batch(["N"])
    n = int(hb.n[0])
    H, b, chi2 = oracle.build_system(p, hb.poses[0], n, jac_mode=oracle.JAC_G2O, **cf.band_kwargs(hb, 0))
    assert np.isnan(chi2) and np.isnan(H).any() and np.nanmax(np.abs(np.diag(H))) == 0.0
    ro, co, so = oracle.optimize_band(p, hb.poses[0], n, args=cf.args(inner, outer), n_cap=hb.n_cap, **cf.band_kwargs(hb, 0))
    assert np.array_equal(ro, hb.poses[0][:n], equal_nan=True)
    iters = outer * inner if inner else 0
    assert so.lm_iters == iters and so.lm_trials == iters
    assert bool(so.status & abi.TEB_STATUS_OPTIMIZED) == (outer == 0 or inner > 0)
    assert not so.status & abi.TEB_STATUS_TERMINATED
    assert bool(so.status & abi.TEB_STATUS_CHOL_FAILED) == (iters > 0)
    if iters:
        assert np.isnan(co) and np.isnan(so.chi2_final) and so.lambda_final == 0.0 and so.nu_final == 2.0 ** (inner + 1)


@pytest.mark.parametrize("outer,inner", cf.EDGES)
def test_max_vel_below_threshold_resizes_once_then_disables(oracle, ref, outer, inner):
    """D: autoResize runs in the first outer iteration, optimizeGraph refuses (max_vel_x < 0.01), optimizeTEB returns
    false with no cost"""
    p = cf.params()
    p.max_vel_x = 0.005
    hb = cf.mixed_batch(["O"])
    rec = cf.d_band(20, hb.n_cap)
    kw = cf.band_kwargs(hb, 0)
    for cost in (True, False):
        ro, co, so, sr, ok = _pin(oracle, ref, p, rec, 20, cf.args(inner, outer, cost), kw, hb.n_cap)
        assert co == np.inf and so.lm_iters == 0
        if outer == 0:
            assert ok and len(ro) == 20 and not so.status & abi.TEB_STATUS_DISABLED
        else:
            assert not ok and so.status & abi.TEB_STATUS_DISABLED and len(ro) > 20


@pytest.mark.parametrize("outer,inner", cf.EDGES)
def test_rho_zero_band_terminates_after_one_trial(oracle, ref, outer, inner):
    """P: H != 0 and b = 0 exactly, so the first trial leaves the state bit-identical, rho == 0 and LM returns
    Terminate - g2o's third exit - in every outer iteration"""
    p = cf.params(shortest_path=True)
    hb = cf.mixed_batch(["P"])
    n, kw = int(hb.n[0]), cf.band_kwargs(hb, 0)
    H, b, chi2 = oracle.build_system(p, hb.poses[0], n, jac_mode=oracle.JAC_G2O, **kw)
    assert chi2 > 0 and not b.any() and H.any()
    for cost in (True, False):
        ro, co, so, sr, ok = _pin(oracle, ref, p, hb.poses[0], n, cf.args(inner, outer, cost), kw, hb.n_cap)
        assert np.array_equal(ro, hb.poses[0][:n])
        if outer and inner:
            assert so.lm_iters == outer and so.lm_trials == outer and so.nu_final == 4.0 and so.lambda_final > 0
            assert so.status == abi.TEB_STATUS_OPTIMIZED | abi.TEB_STATUS_TERMINATED and (co == chi2 or not cost)
