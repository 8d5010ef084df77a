"""The oracle's H-signatures (oracle/teb_oracle.c) against the reference's own h_signature.h (oracle/_ref/libteb_ref.so,
see tests/ref_binding.py) on every case of tests/hsig_cases.py: the 2-D skip rule at and around 0.05, partial
products that leave the fp64 range, a signature past it, the angle branch cut and its tie, poses on obstacles, the two
map rectangles, n = 1 / 2, M = 0 / 1 / 1024, and the x-y-t signature's edges.

  * 2-D value: 1e-15 relative to max(1, |H|), +-inf and NaN equal;
  * x-y-t values: bit equal (NaN where the reference has NaN);
  * isValid / isReasonable equal, and the isEqual partition of each case's candidates equal. The one exception is the
    case whose long double signature is past the fp64 range: the reference keeps the long double and says valid, the
    oracle (and the C-ABI, which returns double) hold +-inf and say invalid - asserted as that difference.

Where the library cannot be built the calls are answered from tests/golden/golden_ref_hsig_v1.npz (recorded by
tests/golden/make_golden_ref_hsig.py)."""
import os

import numpy as np
import pytest

from tests import hsig_cases as hc
from tests import ref_binding as rb

GOLDEN_HSIG = os.path.join(os.path.dirname(__file__), "golden", "golden_ref_hsig_v1.npz")
pytestmark = pytest.mark.skipif(not (rb.live() or os.path.exists(GOLDEN_HSIG)),
                                reason="neither oracle/_ref/libteb_ref.so nor its recorded H-signature calls exist")
CASES = {c.name: c for c in hc.all_cases()}


@pytest.fixture(scope="module")
def ref():
    rb.add_recording(GOLDEN_HSIG)
    return rb


def _same_2d(got, want):
    for g, w in ((got.real, want.real), (got.imag, want.imag)):
        if not np.isfinite(w):
            if not ((np.isnan(w) and np.isnan(g)) or g == w):
                return False
    if not (np.isfinite(want.real) and np.isfinite(want.imag)):
        return True
    return abs(got - want) <= 1e-15 * max(1.0, abs(want))


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_h_signature_matches_reference_header(oracle, ref, name):
    case = CASES[name]
    p = case.params()
    mine, theirs = [], []
    for i, rec in enumerate(case.bands):
        want, valid, reasonable = ref.h_signature(p, rec, len(rec), case.obst, use_timediffs=case.use_dt)
        got = oracle.h_signature(p, rec, len(rec), case.obst, use_timediffs=case.use_dt)
        if case.dim == 2:
            assert _same_2d(got, want), (name, i, got, want)
        else:
            assert np.array_equal(got, want, equal_nan=True), (name, i, got, want)
        if case.beyond_range:
            # the documented difference: +-inf in the double both return, valid only for the reference's long double
            assert not np.isfinite(got.real) and not np.isfinite(got.imag), (name, i, got)
            assert valid and not hc.is_valid(got), (name, i)
        else:
            assert hc.is_valid(got) == valid, (name, i, got)
        assert hc.is_reasonable(got, case.dim) == reasonable, (name, i)
        mine.append(got)
        theirs.append(want)
    thr = p.h_signature_threshold
    assert hc.partition(mine, case.dim, thr) == hc.partition(theirs, case.dim, thr)


def test_cases_cover_the_edges():
    """the case set holds what the GPU tests rely on: both signs of the rounded skip decision, both orders of the range
    scene and the past-range signature, M = 0 / 1 / 1024, n = 1 / 2, both time-difference modes"""
    names = set(CASES)
    for n in ("skip_exact", "skip_fp64_skips_0", "skip_fp64_keeps_0", "skip_fp64_keeps_1d", "skip_duplicates",
              "range_far_first", "range_near_first", "range_beyond", "blob_1024", "angle_branch_cut",
              "angle_through_centre", "pose_on_obstacle", "rect_exactly_3", "rect_below_3", "m0", "m1",
              "xyt_coincident_dt0", "xyt_coincident_dt1", "xyt_loop", "xyt_world_line_through_pose"):
        assert n in names, n
    assert {len(c.obst) for c in CASES.values()} >= {0, 1, 1024}
    assert {len(b) for b in CASES["short_and_closed"].bands} >= {1, 2}
    assert [c.name for c in CASES.values() if c.beyond_range] == ["range_beyond"]
