"""Records tests/golden/golden_ref_traj_v1.npz: every call tests/test_trajectory_cases.py makes into
oracle/_ref/libteb_ref.so (the reference's own getVelocityProfile / getFullTrajectory, ops 9 / 10, see
tests/trajectory_cases.py), with what it returned. The CPU and GPU trajectory tests answer from this file wherever the
library cannot be built. Run where the reference library exists:

    python -m tests.golden.make_golden_ref_traj
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytest  # noqa: E402

from tests import ref_binding as rb  # noqa: E402

OUT = os.path.join(HERE, "golden_ref_traj_v1.npz")

if __name__ == "__main__":
    if not rb.live():
        raise SystemExit("oracle/_ref/libteb_ref.so is missing: the calls can only be recorded from the reference library")
    rb.start_recording()
    rc = pytest.main(["-q", "-p", "no:cacheprovider", os.path.join(ROOT, "tests", "test_trajectory_cases.py")])
    if rc != 0:
        raise SystemExit(f"the trajectory case tests failed (rc={rc}): nothing recorded")
    rb.save_recording(OUT)
    print(OUT, os.path.getsize(OUT), "bytes,", len(rb._recording), "calls")
