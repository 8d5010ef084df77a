"""The restated oscillation detector (tests/cycle_cases.detector_update, which the device's teb_cycle_detector_update
follows) against the reference's own FailureDetector (recovery_behaviors.cpp compiled into
oracle/_ref/libteb_ref_recovery.so by oracle/ref_recovery.mk, with a deque-backed boost::circular_buffer stand-in, driven
by teb_ref_failure_detector in oracle/ref_recovery_driver.cpp).

Seeded random twist sequences with capacities 0 .. 64, three times the capacity long so that every ring wraps, mixing
oscillating runs around zero, signed zeros, NaNs, large values and limits of 0 and below. isOscillating() after every
update must be the same, step for step. Where the library cannot be built the reference's answers come from
tests/golden/golden_ref_recovery_v1.npz (recorded by tests/golden/make_golden_ref_recovery.py); where it exists, the
recording is checked against it too."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import cycle_cases as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libteb_ref_recovery.so")
REFERENCE_TREE = "/root/reference"
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "golden_ref_recovery_v1.npz")
SEED = 20261017
_live = None


def live():
    """True where the reference's FailureDetector answers: built here from the reference sources, or built elsewhere"""
    global _live
    if _live is None:
        if os.path.isdir(REFERENCE_TREE):
            try:
                subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "-f", "ref_recovery.mk"])
            except Exception:
                pass
        _live = os.path.exists(REF_SO)
    return _live


def make_cases(seed=SEED):
    """list of (capacity, twists [T][2], (v_max, v_backwards_max, omega_max, v_eps, omega_eps))"""
    rng = np.random.default_rng(seed)
    caps = list(range(65)) + [int(c) for c in rng.integers(1, 65, 31)]
    cases = []
    for i, cap in enumerate(caps):
        T = 3 * cap + 7
        kind = i % 4
        if kind == 0:    # a robot rocking on the spot: small v, omega alternating in sign
            v = rng.normal(0.0, 0.02, T)
            w = np.where(rng.random(T) < 0.8, np.resize([1.0, -1.0], T), 1.0) * rng.uniform(0.0, 0.05, T)
        elif kind == 1:  # moving: no oscillation expected
            v = rng.uniform(-0.2, 0.4, T)
            w = rng.uniform(-0.3, 0.3, T)
        elif kind == 2:  # quantised: exact zeros, signed zeros and ties at the thresholds
            v = rng.choice([0.0, -0.0, 0.01, -0.01, 0.04, 0.4], T)
            w = rng.choice([0.0, -0.0, 0.03, -0.03, 0.3, -0.3], T)
        else:            # NaN and inf sprinkled into an oscillating run
            v = rng.normal(0.0, 0.01, T)
            w = np.resize([0.02, -0.02], T) * rng.uniform(0.5, 1.5, T)
            m = rng.random((T, 2))
            v[m[:, 0] < 0.05], w[m[:, 1] < 0.05] = np.nan, np.nan
            v[(m[:, 0] > 0.97)] = np.inf
        tw = np.stack([v, w], 1).astype(np.float64)
        lims = rng.choice([[0.4, 0.2, 0.3, 0.1, 0.1], [0.4, 0.0, 0.3, 0.1, 0.1], [0.0, 0.2, 0.0, 0.1, 0.1],
                           [1.0, 1.0, 1.0, 0.05, 0.2], [0.4, -0.2, -1.0, 0.1, 0.1], [0.4, 0.2, 0.3, 0.0, 1.0]])
        cases.append((cap, tw, tuple(float(x) for x in lims)))
    return cases


def restated(case):
    cap, tw, lim = case
    return np.array(cc.detector_sequence([(float(a), float(b)) for a, b in tw], cap, *lim), np.int32)


def reference(case):
    """the reference library's answers (needs oracle/_ref/libteb_ref_recovery.so)"""
    lib = C.CDLL(REF_SO)
    f = lib.teb_ref_failure_detector
    f.restype = None
    f.argtypes = [C.c_int32, C.c_void_p, C.c_int32] + [C.c_double] * 5 + [C.c_void_p]
    cap, tw, lim = case
    tw = np.ascontiguousarray(tw)
    out = np.full(len(tw), -1, np.int32)
    f(cap, tw.ctypes.data, len(tw), *lim, out.ctypes.data)
    return out


def recorded():
    """the reference's answers, concatenated over the cases, from the golden file"""
    z = np.load(GOLDEN)
    assert int(z["seed"]) == SEED
    return z["flags"]


def _answers():
    cases = make_cases()
    if live():
        return cases, np.concatenate([reference(c) for c in cases])
    if os.path.exists(GOLDEN):
        return cases, recorded()
    pytest.skip("neither oracle/_ref/libteb_ref_recovery.so nor tests/golden/golden_ref_recovery_v1.npz exists")


def test_restated_detector_matches_the_reference_step_for_step():
    cases, ref = _answers()
    got = np.concatenate([restated(c) for c in cases])
    assert got.shape == ref.shape
    bad = np.flatnonzero(got != ref)
    assert bad.size == 0, f"{bad.size} steps differ, first at flat index {bad[0]}"
    # the sequences exercise both answers, at every capacity that can oscillate
    assert 0.05 < ref.mean() < 0.95


def test_cases_cover_wraps_signed_zeros_and_nans():
    cases = make_cases()
    assert sorted({c[0] for c in cases}) == list(range(65))
    assert all(len(c[1]) > 2 * c[0] for c in cases)
    tw = np.concatenate([c[1] for c in cases])
    assert np.isnan(tw).any() and np.isinf(tw).any()
    assert (np.signbit(tw) & (tw == 0)).any() and (~np.signbit(tw) & (tw == 0)).any()


@pytest.mark.skipif(not (live() and os.path.exists(GOLDEN)), reason="needs both the reference library and the recording")
def test_recording_is_the_reference_libraries_answer():
    cases = make_cases()
    assert np.array_equal(np.concatenate([reference(c) for c in cases]), recorded())
