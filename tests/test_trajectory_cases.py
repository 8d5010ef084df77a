"""The trajectory read-out cases of tests/trajectory_cases.py on the CPU: the tie cases sit on the tie, the random bands
stay away from it, and op 9 / op 10 (getVelocityProfile / getFullTrajectory) of the drop-in layer and of the reference
agree bit for bit on every case the reference can answer (at least two poses, every time difference positive). The GPU tests read both answers as the device's yardsticks. Also
the C-ABI size of TebTrajectoryArgs."""
import ctypes as C

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import trajectory_cases as tc


def test_sizeof_matches_the_library():
    from teb_local_planner_b200 import load_library
    from teb_local_planner_b200 import build as b
    b.build()
    assert load_library().tebgpu_sizeof(7) == C.sizeof(abi.TebTrajectoryArgs) == 40


def test_tie_cases_sit_on_the_tie_and_random_bands_keep_away():
    cases = {c.name: c for c in tc.all_cases()}
    tie = cases["tie_pure_y"]
    along, length = tc.segment_geometry(tie.rec)
    ties = tc.exact_ties(tie.rec)
    assert ties.sum() == 3 and (along[ties] == 0).all() and (length[ties] > 0).all()
    assert (tie.rec[:-1, 2][ties] == 0).all()                  # heading 0: cos and sin are exact everywhere
    for c in cases.values():
        assert not tc.near_ties(c.rec).any(), c.name
    for c in tc.random_cases():
        along, length = tc.segment_geometry(c.rec)
        assert (np.abs(along) > tc.RANDOM_TIE_MARGIN * length).all(), c.name
    co = tc.segment_geometry(cases["coincident"].rec)[1]
    assert (co == 0).sum() == 3
    assert (cases["inactive_boundaries"].vs[3] == 0) and (cases["inactive_boundaries"].vg[3] == 0)
    assert (cases["zero_dt"].rec[:-1, 3] == 0).any() and (cases["negative_dt"].rec[:-1, 3] < 0).any()
    assert cases["n_cap"].n == tc.N_CAP


def test_host_layer_shapes_and_boundary_rows():
    op = tc.host_band_op()
    for c in tc.all_cases():
        for mvy in tc.MAX_VEL_Y:
            prof = op(9, c, mvy).reshape(-1, 3)
            traj = op(10, c, mvy).reshape(-1, 7)
            assert len(prof) == c.n + 1 and len(traj) == c.n, c.name
            assert np.array_equal(prof[-1], c.vg[:3]), c.name
            if c.n >= 1:
                assert np.array_equal(prof[0], c.vs[:3]) and np.array_equal(traj[0, 3:6], c.vs[:3]) and traj[0, 6] == 0
            if c.n >= 2:
                assert np.array_equal(traj[-1, 3:6], c.vg[:3]), c.name


@pytest.mark.skipif(not tc.reference_available(), reason="neither oracle/_ref/libteb_ref.so nor its recorded calls exist")
def test_host_layer_and_reference_agree():
    tc.use_recording()
    op = tc.host_band_op()
    compared = 0
    for c in tc.all_cases():
        if not c.on_reference:
            continue
        for mvy in tc.MAX_VEL_Y:
            for k in (9, 10):
                assert np.array_equal(op(k, c, mvy), tc.ref_band_op(k, c, mvy)), (c.name, mvy, k)
                compared += 1
    assert compared == 4 * (len(tc.all_cases()) - 4)              # all but n = 0, n = 1, zero_dt and negative_dt
