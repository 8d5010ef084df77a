"""Records tests/golden/golden_ref_recovery_v1.npz: the reference FailureDetector's isOscillating() after every update
of the seeded sequences of tests/test_reference_pin_recovery.py (recovery_behaviors.cpp compiled into
oracle/_ref/libteb_ref_recovery.so by oracle/ref_recovery.mk). The test answers from this file wherever the library
cannot be built. Run where the reference sources exist:

    python -m tests.golden.make_golden_ref_recovery
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from tests import test_reference_pin_recovery as pin  # noqa: E402

OUT = os.path.join(HERE, "golden_ref_recovery_v1.npz")

if __name__ == "__main__":
    if not pin.live():
        raise SystemExit("oracle/_ref/libteb_ref_recovery.so is missing: the answers can only be recorded from the reference library")
    flags = np.concatenate([pin.reference(c) for c in pin.make_cases()]).astype(np.int8)
    np.savez_compressed(OUT, seed=np.int64(pin.SEED), flags=flags)
    print(OUT, os.path.getsize(OUT), "bytes,", flags.size, "steps,", int(flags.sum()), "oscillating")
