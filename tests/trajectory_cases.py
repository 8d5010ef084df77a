"""Bands for the trajectory read-out (tebgpu_read_trajectory: getVelocityProfile / getFullTrajectory,
optimal_planner.cpp:1170-1248) and the operations that answer them on the CPU: op 9 / op 10 of the drop-in layer
(teb_host_band_op) and of the reference (teb_ref_band_op, or its recorded answers in tests/golden/golden_ref_traj_v1.npz,
recorded by tests/golden/make_golden_ref_traj.py).

Named cases: n = 0, 1, 2, 3 and n = N_CAP; a zero and a negative time difference (the drop-in layer answers these,
the reference asserts dt > 0 when it loads a band); heading steps across +-pi and stored
headings outside [-pi, pi); backwards segments; coincident poses; pure-y steps from heading 0 (the sign tie of the
non-holonomic vx, exact on both sides because cos(0) and sin(0) are); boundary velocities whose active flag is 0. Random
bands keep every step's projection on its heading at least RANDOM_TIE_MARGIN of the step length away from zero, so
that device and glibc trigonometry cannot disagree on a sign. Every case is run with both MAX_VEL_Y values."""
import ctypes as C
import math
import os
from dataclasses import dataclass

import numpy as np

from tests import ref_binding as rb

N_CAP = 512
MAX_VEL_Y = (0.0, 0.3)       # non-holonomic, holonomic extractVelocity
TIE = 1e-12                  # |along| <= TIE |step|: the sign of the non-holonomic vx may differ between device and glibc
RANDOM_TIE_MARGIN = 1e-6
GOLDEN_TRAJ = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_ref_traj_v1.npz")


@dataclass
class Case:
    name: str
    rec: np.ndarray          # [n][4] x, y, theta, dt
    vs: np.ndarray           # [4] vx, vy, omega, active as stored in the batch
    vg: np.ndarray

    @property
    def n(self):
        return len(self.rec)

    def padded(self):
        out = np.zeros((N_CAP, 4))
        out[:self.n] = self.rec
        return out

    def op_args(self, max_vel_y):
        """args of op 9 / 10. The boundary velocities are always set (active), because the read-out reports them as
        stored whatever their flag, and the reference reports what setVelocityStart / setVelocityGoal stored."""
        return np.array([max_vel_y, *self.vs[:3], 1.0, *self.vg[:3], 1.0])

    def op_rec(self):
        return self.rec if self.n else None

    @property
    def on_reference(self):
        """whether the reference can answer: at n < 2 getFullTrajectory reads a time difference the band does not have,
        and TimedElasticBand::addTimeDiff asserts dt > 0, so a band with a zero or negative one cannot be loaded there"""
        return self.n >= 2 and bool((self.rec[:-1, 3] > 0).all())


def segment_geometry(rec):
    """per segment k = 1 .. n - 1 (index k - 1): the step's projection on the heading of pose k - 1 and its length"""
    d = rec[1:, :2] - rec[:-1, :2]
    along = np.cos(rec[:-1, 2]) * d[:, 0] + np.sin(rec[:-1, 2]) * d[:, 1]
    return along, np.hypot(d[:, 0], d[:, 1])


def exact_ties(rec):
    """segments that sit on the sign tie where the trigonometry is exact: heading 0, a pure-y step (along == 0)"""
    d = rec[1:, :2] - rec[:-1, :2]
    return (rec[:-1, 2] == 0) & (d[:, 0] == 0) & (d[:, 1] != 0)


def near_ties(rec):
    """segments within TIE of the sign tie that are not exact ties (coincident poses have no sign to get wrong)"""
    along, length = segment_geometry(rec)
    return (np.abs(along) <= TIE * length) & (length > 0) & ~exact_ties(rec)


def _vel(rng, active):
    return np.array([rng.normal(), rng.normal(), rng.normal(), float(active)])


def _walk(rng, n, heading_noise=0.05, wild=False):
    x = np.cumsum(rng.uniform(0.05, 0.3, n))
    y = np.cumsum(rng.normal(0, 0.04, n))
    th = rng.uniform(-math.pi, math.pi, n) if wild else np.arctan2(np.gradient(y), np.gradient(x)) + rng.normal(0, heading_noise, n)
    dt = rng.uniform(0.05, 0.6, n)
    dt[-1] = 0.0
    return np.stack([x, y, th, dt], 1)


def band_cases():
    rng = np.random.default_rng(11)
    cs = []
    add = lambda name, rec, vs=None, vg=None: cs.append(Case(name, np.asarray(rec, np.float64).reshape(-1, 4),
                                                             _vel(rng, 1) if vs is None else vs, _vel(rng, 1) if vg is None else vg))
    add("n0", np.zeros((0, 4)))
    add("n1", [[0.5, -0.25, 0.75, 0.0]])
    add("n2", [[0.0, 0.0, 0.1, 0.4], [0.3, 0.05, 0.2, 0.0]])
    add("n3", [[0.0, 0.0, 0.0, 0.25], [0.2, 0.1, 0.5, 0.5], [0.3, 0.4, 1.2, 0.0]])
    add("n_cap", _walk(rng, N_CAP))
    add("zero_dt", [[0.0, 0.0, 0.1, 0.3], [0.2, 0.0, 0.1, 0.0], [0.4, 0.1, 0.4, 0.2], [0.5, 0.2, 0.6, 0.0]])
    add("negative_dt", [[0.0, 0.0, 0.1, 0.3], [0.2, 0.0, 0.1, -0.25], [0.4, 0.1, 0.4, 0.2], [0.5, 0.2, 0.6, 0.0]])
    add("across_pi", [[0.0, 0.0, 3.1, 0.3], [-0.2, 0.01, -3.1, 0.3], [-0.4, -0.01, 3.0, 0.2], [-0.6, 0.0, -3.05, 0.25],
                      [-0.8, 0.02, math.pi, 0.3], [-1.0, 0.0, -math.pi, 0.0]])
    add("unnormalised_headings", [[0.0, 0.0, 7.0, 0.3], [0.2, 0.1, -9.5, 0.3], [0.3, 0.3, 12.0, 0.3], [0.1, 0.4, 0.0, 0.0]])
    add("backwards", [[0.0, 0.0, 0.0, 0.3], [-0.2, 0.01, 0.05, 0.3], [-0.4, 0.0, 0.0, 0.2], [-0.3, 0.0, 0.0, 0.2],
                      [-0.5, -0.1, 0.1, 0.0]])
    add("coincident", [[0.1, 0.2, 0.3, 0.2], [0.1, 0.2, 0.3, 0.4], [0.1, 0.2, 0.9, 0.1], [0.4, 0.2, 0.9, 0.3],
                       [0.4, 0.2, 0.9, 0.0]])
    add("tie_pure_y", [[0.0, 0.0, 0.0, 0.25], [0.0, 0.5, 0.0, 0.5], [0.0, -0.25, 0.0, 0.125], [0.25, -0.25, 0.0, 0.5],
                       [0.25, 0.75, 0.0, 0.0]])
    add("inactive_boundaries", _walk(rng, 7), vs=np.array([0.3, -0.2, 0.7, 0.0]), vg=np.array([-0.4, 0.1, -0.9, 0.0]))
    return cs


def random_cases(count=24):
    rng = np.random.default_rng(12)
    cs = []
    while len(cs) < count:
        n = int(rng.integers(2, 80))
        rec = _walk(rng, n, wild=rng.random() < 0.3)
        along, length = segment_geometry(rec)
        if (np.abs(along) <= RANDOM_TIE_MARGIN * length).any():
            continue
        cs.append(Case(f"random{len(cs)}", rec, _vel(rng, rng.integers(2)), _vel(rng, rng.integers(2))))
    return cs


def all_cases():
    return band_cases() + random_cases()


# --------------------------------------------------------------------------------------------------- ops 9 / 10
def host_band_op():
    """op(k, case, max_vel_y) -> op k of the drop-in layer (teb_host_band_op) on the case"""
    from teb_local_planner_b200 import build as b
    b.build()
    b.build_host()
    fn = C.CDLL(b.HOST_PIN).teb_host_band_op
    fn.restype = C.c_int32
    fn.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]

    def run(op, case, max_vel_y):
        rec = case.op_rec()
        rec = None if rec is None else np.ascontiguousarray(rec)
        a = case.op_args(max_vel_y)
        cap = 7 * (case.n + 1)
        out = np.full(cap, np.nan)
        k = fn(op, None if rec is None else rec.ctypes.data, case.n, a.ctypes.data, len(a), out.ctypes.data, cap)
        assert k >= 0, (op, case.name)
        return out[:k].copy()
    return run


def reference_available():
    return rb.live() or os.path.exists(GOLDEN_TRAJ)


def use_recording():
    """answer ref_band_op from GOLDEN_TRAJ where the reference library itself does not"""
    if os.path.exists(GOLDEN_TRAJ):
        rb.add_recording(GOLDEN_TRAJ)


def ref_band_op(op, case, max_vel_y):
    """op 9 / 10 of the reference on a case it can answer (Case.on_reference). The answer is kept in full, not as a
    digest, since the holonomic velocities are compared with a tolerance."""
    assert case.on_reference
    rec = np.ascontiguousarray(case.rec)
    a = case.op_args(max_vel_y)
    cap = 7 * (case.n + 1)

    def compute():
        out = np.full(cap, np.nan)
        k = rb.lib().teb_ref_band_op(op, rec.ctypes.data, case.n, a.ctypes.data, len(a), out.ctypes.data, cap)
        assert k >= 0, (op, case.name)
        return (out[:k].copy(),)
    return rb._call("band_op_traj", (op, rec, a, cap), compute)[0]
