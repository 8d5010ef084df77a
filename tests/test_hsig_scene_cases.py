"""The long double restatement of tests/hsig_scene_cases.py, which checks tebgpu_h_signature_scenes above 1024
obstacles: its signature against the oracle's own h_signature_2d (oracle/teb_oracle.c) on every 2-D case of
tests/hsig_cases.py, its row-chunked error scale against hsig_cases.error_scale, and the properties its cases claim."""
import numpy as np
import pytest

from tests import hsig_cases as hc
from tests import hsig_scene_cases as sc

CASES_2D = hc.cases_2d()


@pytest.mark.parametrize("case", CASES_2D, ids=lambda c: c.name)
def test_restatement_matches_oracle(oracle, case):
    """within 1e-15 of sum |A_l| |L_kl| (the oracle divides its running product, the restatement multiplies chunk
    products; both in long double), infinities, NaNs and zeros equal"""
    p = case.params()
    pr = sc.scene_products(case.obst) if len(case.obst) else None
    for rec in case.bands:
        o = oracle.h_signature(p, rec, len(rec), case.obst)
        r = sc.oracle_2d(p, rec, case.obst, pr)
        for a, b in ((o.real, r.real), (o.imag, r.imag)):
            if not np.isfinite(a):
                assert a == b or (np.isnan(a) and np.isnan(b)), (case.name, o, r)
        if not (np.isfinite(o.real) and np.isfinite(o.imag)):
            continue
        s = sc.error_scale(p, rec, case.obst)
        if s == 0:
            assert o == r, (case.name, o, r)
            continue
        assert abs(complex(o) - complex(r)) <= 1e-15 * float(s), (case.name, o, r, float(s))


@pytest.mark.parametrize("case", CASES_2D, ids=lambda c: c.name)
def test_chunked_error_scale_equals_the_full_one(case):
    p = case.params()
    for rec in case.bands:
        a, b = hc.error_scale(p, rec, case.obst), sc.error_scale(p, rec, case.obst, rows=3)
        assert a == b or (np.isnan(a) and np.isnan(b)), (case.name, a, b)


def test_scene_cases_keep_their_margins():
    """every case up to 4096 rows (the 16384-row cases take the same checks in tests/test_gpu_hsig_scene.py, next to
    their long double values): no pair within the double-double band of the skip threshold, no angle tie, the isEqual
    partition of each bundle away from h_signature_threshold, and at least one scene above 2048 rows whose bundle has
    finite, non-zero signatures in more than one class"""
    nontrivial = []
    for case in sc.cases_2d(large=False):
        assert len(case.obst) > 1024
        hc.assert_skip_margin(case.obst)
        p = case.params()
        pr = sc.scene_products(case.obst)
        vals = []
        for rec in case.bands:
            hc.assert_no_near_tie(rec, case.obst)
            vals.append(sc.oracle_2d(p, rec, case.obst, pr))
        thr = p.h_signature_threshold
        sc.assert_class_margins(case, vals, thr)
        part = hc.partition(vals, 2, thr)
        if len(case.obst) > 2048 and all(np.isfinite(v.real) and np.isfinite(v.imag) and v != 0 for v in vals) and \
                not all(all(row) for row in part):
            nontrivial.append(case.name)
    assert nontrivial, "no case above 2048 rows has distinct finite signatures"
    names = [c.name for c in sc.cases_2d(large=False)]
    assert any(n.startswith("grid_") for n in names) and any(n.startswith("duplicates") for n in names)
