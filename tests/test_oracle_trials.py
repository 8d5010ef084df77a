"""CPU tests of the oracle's two trial-level functions, the references of tests/test_gpu_trial_eval.py:
  teb_oracle_trial_chi2  chi2 by family of LM trial states on a graph frozen at the linearisation point;
  teb_oracle_lm_decide   g2o's accept / reject chain, the function the oracle's own LM loop runs (so the bit-equality
                         pins of whole optimizeTEB calls against the reference hold it), one hand-worked case per branch."""
import sys

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import scenarios

CHOL_FAILED, NONFINITE = abi.TEB_STATUS_CHOL_FAILED, abi.TEB_STATUS_NONFINITE
DBL_MAX = sys.float_info.max


@pytest.mark.parametrize("name", scenarios.ALL)
def test_trial_chi2_at_the_graph_state_is_the_system_chi2(oracle, name):
    """at trial == linearisation point the families add up to teb_oracle_build_system's chi2 (fp64 against long double
    accumulation), every family is a sum of non-negative squares, and a state moved off the graph changes the sum"""
    p, hb = scenarios.scenario(name)
    for outer in (0, 3):
        for b in range(hb.B):
            n = int(hb.n[b])
            kw = scenarios.band_kwargs(hb, b)
            _, _, chi2 = oracle.build_system(p, hb.poses[b], n, weight_multiplier=2.0 ** outer, **kw)
            moved = hb.poses[b, :n].copy()
            moved[1:n - 1, :2] += 0.05
            fam = oracle.trial_chi2(p, hb.poses[b], n, np.stack([hb.poses[b, :n], moved]),
                                    weight_multiplier=2.0 ** outer, **kw)
            assert (fam >= 0).all()
            assert abs(fam[0].sum() - chi2) <= 1e-13 * chi2, f"{name} band {b} outer {outer}: {fam[0]} vs {chi2}"
            assert fam[1].sum() != fam[0].sum()
            if hb.V_cap and hb.via_count[b] > 0 and p.weight_viapoint > 0:
                assert fam[0, 1] > 0
            assert fam[0, 2] > 0   # time-optimal: weight_optimaltime * sum dt^2


def _decide(oracle, chi, lam, nu, q0, seq):
    t = [s[0] for s in seq]
    sc = [s[1] for s in seq]
    ok = [s[2] if len(s) > 2 else 1 for s in seq]
    return oracle.lm_decide(chi, lam, nu, q0, t, sc, ok)


def test_lm_decide_accepts_and_scales_lambda(oracle):
    """rho = 0.75: alpha = 1 - 0.5^3 = 0.875, clamped to 2/3; rho = 1.0: alpha = 0, floored at 1/3"""
    d = _decide(oracle, 10.0, 1.0, 8.0, 0, [(4.0, 8.0 - 1e-3)])
    assert (d["accepted"], d["used"], d["terminate"], d["need"], d["status"], d["q"]) == (0, 1, False, False, 0, 1)
    assert d["lam"] == 1.0 * (2.0 / 3.0) and d["nu"] == 2.0 and d["current_chi"] == 4.0
    d = _decide(oracle, 10.0, 3.0, 2.0, 0, [(2.0, 8.0 - 1e-3)])
    assert d["accepted"] == 0 and d["lam"] == 3.0 * (1.0 / 3.0)


def test_lm_decide_rejects_then_accepts(oracle):
    d = _decide(oracle, 10.0, 1.0, 2.0, 0, [(12.0, 1.0), (11.0, 1.0), (9.0, 1.0), (1.0, 1.0)])
    assert (d["accepted"], d["used"], d["need"], d["q"]) == (2, 3, False, 3)
    rho = (10.0 - 9.0) / (1.0 + 1e-3)
    alpha = max(1.0 / 3.0, min(1.0 - (2 * rho - 1) ** 3, 2.0 / 3.0))
    assert d["lam"] == 1.0 * 2.0 * 4.0 * alpha and d["nu"] == 2.0 and d["current_chi"] == 9.0


def test_lm_decide_all_rejected_needs_another_round(oracle):
    d = _decide(oracle, 10.0, 1.0, 2.0, 2, [(12.0, 1.0)] * 4)
    assert (d["accepted"], d["used"], d["terminate"], d["need"], d["q"]) == (-1, 4, False, True, 6)
    assert d["lam"] == 2.0 * 4.0 * 8.0 * 16.0 and d["nu"] == 32.0 and d["current_chi"] == 10.0


@pytest.mark.parametrize("q0", [4, 6, 8, 9])
def test_lm_decide_ten_trial_cap(oracle, q0):
    """a retry round starting at trial q0 consumes at most 10 - q0 trials; the tenth rejection terminates"""
    d = _decide(oracle, 10.0, 1.0, 2.0, q0, [(12.0, 1.0)] * 8)
    assert (d["used"], d["q"], d["terminate"], d["need"], d["accepted"]) == (10 - q0, 10, True, False, -1)


def test_lm_decide_failed_factorisation(oracle):
    """ok = 0: tempChi = DBL_MAX whatever the trial's chi2, CHOL_FAILED, rejected"""
    d = _decide(oracle, 10.0, 1.0, 2.0, 0, [(1.0, 1.0, 0), (1.0, 1.0, 1)])
    assert (d["accepted"], d["used"], d["status"]) == (1, 2, CHOL_FAILED)


def test_lm_decide_non_finite_trial_chi2(oracle):
    """NaN: rho is NaN, neither accepted nor < 0, so the iteration ends without Terminate; +inf: rho = -inf, a plain
    rejection"""
    d = _decide(oracle, 10.0, 1.0, 2.0, 0, [(np.nan, 1.0), (1.0, 1.0)])
    assert (d["accepted"], d["used"], d["terminate"], d["need"], d["q"]) == (-1, 1, False, False, 1)
    assert d["lam"] == 2.0 and d["nu"] == 4.0
    d = _decide(oracle, 10.0, 1.0, 2.0, 0, [(np.inf, 1.0), (1.0, 1.0)])
    assert (d["accepted"], d["used"], d["terminate"]) == (1, 2, False)


def test_lm_decide_rho_zero_terminates(oracle):
    """a band whose chi2 is exactly 0 (or unchanged): rho == 0 ends the iteration and terminates after one trial"""
    d = _decide(oracle, 0.0, 1.0, 2.0, 0, [(0.0, 5.0), (0.0, 5.0)])
    assert (d["accepted"], d["used"], d["terminate"], d["need"], d["q"]) == (-1, 1, True, False, 1)
    assert d["lam"] == 2.0 and d["nu"] == 4.0


def test_lm_decide_lambda_overflow(oracle):
    """lambda nu overflows: NONFINITE, the trial is not counted, Terminate"""
    d = _decide(oracle, 10.0, DBL_MAX / 3, 2.0, 0, [(12.0, 1.0), (12.0, 1.0), (1.0, 1.0)])
    assert (d["accepted"], d["used"], d["q"], d["terminate"], d["need"], d["status"]) == (-1, 2, 1, True, False, NONFINITE)
    assert np.isinf(d["lam"])
