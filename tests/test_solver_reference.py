"""CPU checks of tests/banded_reference.py, the extended-precision restatement of the LM step's linear solve that
tests/test_gpu_solver.py holds every solve kernel to: the longdouble solve against mpmath, the synthetic systems against
the solver's profile, and the CPU model of k_solve_lat's index arithmetic (tools/twisted_model.py) against the same
backward-error bound the kernels must meet."""
import importlib.util
import os

import numpy as np
import pytest

from tests import banded_reference as R
from tests.test_band_profile import _assert_in_profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("twisted_model", os.path.join(ROOT, "tools", "twisted_model.py"))
tm = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(tm)

BACKWARD_BOUND = 64 * R.U


@pytest.mark.parametrize("n", [3, 4, 5, 7, 10, 15])
def test_longdouble_solve_matches_mpmath(n):
    mp = pytest.importorskip("mpmath")
    rng = np.random.default_rng(100 + n)
    Hb = R.synthetic_systems(rng, [n] * 2, n, w_lo=1e-3, w_hi=1e3)
    lam = 1e-5 * R.max_real_diag(Hb, [n] * 2)
    x, ok = R.ldl_solve(Hb, [n] * 2, lam)
    assert ok.all()
    with mp.workdps(40):
        for s in range(2):
            A, b = R.dense(Hb[s], n, lam[s])
            xs = mp.lu_solve(mp.matrix(A.tolist()), mp.matrix(b.tolist()))
            ref = np.array([float(v) for v in xs])
            err = np.abs(x[s].astype(np.float64) - ref).max() / np.abs(ref).max()
            kappa = np.linalg.cond(A, np.inf)
            # longdouble has a 64-bit significand: the solve is accurate to a few 2^-64 times the condition number
            assert err <= 64 * 2.0 ** -64 * kappa + 1e-300, (n, s, err, kappa)


def test_residual_and_backward_error_of_the_exact_solution_are_tiny():
    rng = np.random.default_rng(3)
    n = [3, 9, 30]
    Hb = R.synthetic_systems(rng, n, 30)
    lam = 1e-5 * R.max_real_diag(Hb, n)
    x, ok = R.ldl_solve(Hb, n, lam)
    assert ok.all()
    assert (R.backward_error(Hb, n, lam, x) <= 4 * 2.0 ** -64).all()
    # a double solution perturbed by one part in 1e10 is far outside the bound the kernels are held to
    xp = x.astype(np.float64) * (1 + 1e-10 * rng.standard_normal(x.shape))
    assert (R.backward_error(Hb, n, lam, xp) > 100 * BACKWARD_BOUND).all()


def test_synthetic_systems_lie_inside_the_solver_profile():
    rng = np.random.default_rng(7)
    n = list(range(3, 31)) + [64, 129]
    Hb = R.synthetic_systems(rng, n, 129)
    for s, ns in enumerate(n):
        band = Hb[s, :4 * ns, :11]
        r, k = np.nonzero(band)
        _assert_in_profile(r, r - k, f"synthetic band n = {ns}")
        assert (band[R.row_is_real(np.arange(4 * ns), ns), 0] > 0).all()
    lam = 1e-5 * R.max_real_diag(Hb, n)
    Hi = R.make_indefinite(Hb, n, lam, [4 * ns // 2 for ns in n], rng)
    for s, ns in enumerate(n):
        r, k = np.nonzero(Hi[s, :4 * ns, :11])
        _assert_in_profile(r, r - k, f"indefinite band n = {ns}")


def test_indefinite_systems_fail_and_spd_systems_do_not():
    rng = np.random.default_rng(11)
    n = [3, 6, 12, 40]
    Hb = R.synthetic_systems(rng, n, 40)
    lam = 1e-5 * R.max_real_diag(Hb, n)
    assert R.ldl_solve(Hb, n, lam)[1].all()
    for rows in ([3] * 4, [10] * 4, [21] * 4, [4 * ns - 5 for ns in n]):
        Hi = R.make_indefinite(Hb, n, lam, rows, rng)
        assert not R.ldl_solve(Hi, n, lam)[1].any()
        for s, ns in enumerate(n):
            A, _ = R.dense(Hi[s], ns, lam[s])
            assert np.linalg.eigvalsh(A).min() < 0


@pytest.mark.parametrize("n", [3, 4, 5, 6, 7, 8, 11, 17, 30, 61])
def test_twisted_model_meets_the_backward_error_bound(n):
    """k_solve_lat's elimination order on the synthetic systems, executed on the CPU: held to the threshold of the GPU
    tests before any kernel runs"""
    rng = np.random.default_rng(200 + n)
    S = 3
    Hb = R.synthetic_systems(rng, [n] * S, n)
    base = 1e-5 * R.max_real_diag(Hb, [n] * S)
    N = 4 * n
    for scale in (1.0, 2.0 ** 20, 2.0 ** 45):
        lam = base * scale
        xs = np.zeros((S, N))
        for s in range(S):
            Hs = Hb[s, :N].copy()
            real = R.row_is_real(np.arange(N), n)
            Hs[real, 0] += lam[s]                       # solve_lat takes a plain band
            xs[s] = tm.solve_lat(Hs, N)
        be = R.backward_error(Hb, [n] * S, lam, xs)
        assert (be <= BACKWARD_BOUND).all(), (n, scale, be / R.U)
