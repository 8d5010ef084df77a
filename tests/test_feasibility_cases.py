"""The isTrajectoryFeasible cases of tests/feasibility_cases.py against the drop-in layer's op 12 (teb_host_band_op) and,
where oracle/_ref is built, the reference's own op 12 (teb_ref_band_op): same verdict, same number of queries and
bit-identical query poses. This pins the case builders' transcription, which the GPU tests read their claims from. Also
the C-ABI size of TebFeasibilityArgs."""
import ctypes as C
import os

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import feasibility_cases as fc
from tests import ref_binding as rb


@pytest.fixture(scope="module")
def host_op12():
    from teb_local_planner_b200 import build as b
    b.build()
    b.build_host()
    fn = C.CDLL(b.HOST_PIN).teb_host_band_op
    fn.restype = C.c_int32
    fn.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]

    def run(case, with_discs=True):
        rec = np.ascontiguousarray(case.rec[:max(case.n, 1)])
        a = np.ascontiguousarray(case.op12_args(with_discs), dtype=np.float64)
        cap = case.op12_cap()
        out = np.full(cap, np.nan)
        k = fn(12, rec.ctypes.data, case.n, a.ctypes.data, len(a), out.ctypes.data, cap)
        assert k >= 0, case
        return out[:k].copy()
    return run


def _expect(case, out, with_discs=True):
    feas, cnt = (case.feasible, case.count) if with_discs else (1, len(case.queries))
    assert out[0] == feas and out[1] == cnt, (case, out[:2], feas, cnt)
    q = out[2:].reshape(-1, 3)
    assert np.array_equal(q, case.queries[:cnt]), case


def test_sizeof_matches_the_library():
    from teb_local_planner_b200 import load_library
    from teb_local_planner_b200 import build as b
    b.build()
    assert load_library().tebgpu_sizeof(6) == C.sizeof(abi.TebFeasibilityArgs) == 64


def test_band_cases_on_the_host_layer(host_op12):
    for c in fc.band_cases() + fc.random_cases():
        _expect(c, host_op12(c, with_discs=False), with_discs=False)


def test_disc_cases_on_the_host_layer(host_op12):
    for c in fc.disc_cases():
        _expect(c, host_op12(c))


@pytest.mark.skipif(not rb.live(), reason="oracle/_ref/libteb_ref.so is not built (the reference sources are absent)")
def test_cases_on_the_reference():
    for c in fc.band_cases() + fc.random_cases():
        _expect(c, rb.band_op(12, c.rec[:c.n] if c.n else None, c.op12_args(False), cap=c.op12_cap()), with_discs=False)
    for c in fc.disc_cases():
        _expect(c, rb.band_op(12, c.rec[:c.n], c.op12_args(), cap=c.op12_cap()))
