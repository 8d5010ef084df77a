"""The long double restatement of tests/hsig_scene_cases.py (per-scene products, then f0 and the sum over segments) against
the reference's own h_signature.h (oracle/_ref/libteb_ref.so, see tests/ref_binding.py) on scenes of 1025 to 2048
obstacles: costmap cells, a 5 cm grid block, duplicate rows and far rows listed before near ones. Short bands (6 poses),
so that the reference's O(n M^2) loop stays affordable.

  * 2-D value within 1e-15 sum_{k,l} |A_l| |L_kl|; +-inf, NaN and exact zeros equal.

Where the library cannot be built the calls are answered from tests/golden/golden_ref_hsig_large_v1.npz (recorded by
tests/golden/make_golden_ref_hsig_large.py)."""
import os

import numpy as np
import pytest

from tests import hsig_cases as hc
from tests import hsig_scene_cases as sc
from tests import ref_binding as rb

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "golden_ref_hsig_large_v1.npz")
pytestmark = pytest.mark.skipif(not (rb.live() or os.path.exists(GOLDEN)),
                                reason="neither oracle/_ref/libteb_ref.so nor its recorded H-signature calls exist")


def _short(case):
    """the case's scene with 6-pose bands between the ends of its first band"""
    rec = case.bands[0]
    a, b = rec[0, :2], rec[-1, :2]
    return hc.Case(case.name, 2, case.obst, [hc.bent(a, b, 6, u) for u in (0.0, 0.9, -0.9)])


CASES = [_short(c) for c in sc.cases_2d(large=False) if len(c.obst) <= 2048]


@pytest.fixture(scope="module")
def ref():
    rb.add_recording(GOLDEN)
    return rb


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_restatement_matches_reference(ref, case):
    assert 1024 < len(case.obst) <= 2048
    p = case.params()
    pr = sc.scene_products(case.obst)
    for rec in case.bands:
        w = complex(ref.h_signature(p, rec, len(rec), case.obst)[0])
        got = sc.oracle_2d(p, rec, case.obst, pr)
        for g, x in ((got.real, w.real), (got.imag, w.imag)):
            if not np.isfinite(x):
                assert g == x or (np.isnan(g) and np.isnan(x)), (case.name, got, w)
        if not (np.isfinite(w.real) and np.isfinite(w.imag)):
            continue
        s = sc.error_scale(p, rec, case.obst)
        if w == 0 or s == 0:
            assert got == w, (case.name, got, w)
            continue
        assert abs(got - w) <= 1e-15 * float(s), (case.name, got, w, float(s))
