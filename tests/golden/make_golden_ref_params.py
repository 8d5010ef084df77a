"""Records tests/golden/golden_ref_params_v1.npz: every call tests/test_reference_pin_params.py makes into
oracle/_ref/libteb_ref.so (the reference's own code, see tests/ref_binding.py), with what it returned. The test answers
from this file wherever the library cannot be built. Run where the reference library exists:

    python -m tests.golden.make_golden_ref_params
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import pytest  # noqa: E402

from tests import ref_binding as rb  # noqa: E402

OUT = os.path.join(HERE, "golden_ref_params_v1.npz")

if __name__ == "__main__":
    if not rb.live():
        raise SystemExit("oracle/_ref/libteb_ref.so is missing: the calls can only be recorded from the reference library")
    rb.start_recording()
    rc = pytest.main(["-q", "-p", "no:cacheprovider", os.path.join(ROOT, "tests", "test_reference_pin_params.py")])
    if rc != 0:
        raise SystemExit(f"the reference-pinned parameter-switch tests failed (rc={rc}): nothing recorded")
    rb.save_recording(OUT)
    print(OUT, os.path.getsize(OUT), "bytes,", len(rb._recording), "calls")
