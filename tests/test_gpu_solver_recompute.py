"""k_solve_tpb in its two forms, through tebgpu_solve_system with the form forced (tebgpu_set_solve_form):
  streamed   the LDL^T factor written to device memory and read back by the back substitution (form 1);
  recompute  the factor not stored: window checkpoints every C rows, each segment refactored and back-substituted from
             shared memory (k_solve_tpb_rc, C = 11, 22, 33).
Both run the same pivot step, so every form gives the same bits as the streamed one and as k_solve_warp: dx, ok and the
lambda of each trial. Checked on kernel A's systems of every scenario, on short bands at every residue of N mod 11 / 22 /
33, on n around 128 / 256 / 512, in ragged warps and retry lists in any order, with the failure contract (NaN in b
included); every accepted solution has a backward error <= 64 u against tests/banded_reference.py and leaves the
scratch past its N untouched."""
import numpy as np
import pytest

import teb_local_planner_b200 as T
from tests import banded_reference as R
from tests import scenarios
from tests.test_gpu_solver import _check_solution, _lambda_replay, _same_bits, _state_after, _synthetic, _untouched

pytestmark = pytest.mark.gpu

FORMS = [1, 11, 22, 33]   # streamed, recompute with C = 11, 22, 33
_contexts = {}


def _ctx(n_cap):
    if n_cap not in _contexts:
        _contexts[n_cap] = T.TebGpu(96, n_cap, 1, 1)
    return _contexts[n_cap]


def _solve(g, form, n, K, **kw):
    """solver 2, thread-per-system mapping (k_solve_tpb) in the given form; form None: k_solve_warp"""
    g.set_solver(2)
    g.set_warp_solver(1 if form is None else 0)
    g.set_solve_form(1 if form is None else form)
    try:
        return g.solve_system(n, K, **kw)
    finally:
        g.set_warp_solver(4)
        g.set_solve_form(0)


def _all_forms(g, n, K, warp=True, **kw):
    """{form: (dx, ok, lambda)} for every form and k_solve_warp (key None); asserts they are the same bits"""
    out = {f: _solve(g, f, n, K, **kw) for f in FORMS + ([None] if warp else [])}
    ref = out[1]
    for f, res in out.items():
        for name, a, b in zip(("dx", "ok", "lambda"), res, ref):
            assert _same_bits(a, b), f"form {f}: {name} differs from the streamed form"
    return out


@pytest.mark.parametrize("name", scenarios.ALL)
def test_kernel_a_systems_every_form(name):
    p, hb = scenarios.scenario(name)
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, max(hb.M_cap, 1), hb.V_cap, max_obst_vertices=hb.PV_cap)
    g.set_params(p)
    try:
        for outer in (0, 2):
            Hb, _ = g.build_system(hb, outer)
            n = hb.n.copy()
            for K in (2, 8):
                dx, ok, lam = _all_forms(g, n, K, n_cap=hb.n_cap)[1]   # the system kernel A just built, LM iteration 0
                base = 1e-5 * R.max_real_diag(Hb, n)
                assert np.array_equal(lam, _lambda_replay(base, np.full(hb.B, 2.0), K))
                _check_solution("tpb_recompute", Hb, n, dx, ok, lam, f"{name} outer {outer} K {K}")
    finally:
        g.close()


@pytest.mark.parametrize("K", [2, 4, 6, 8])
def test_short_bands_every_segment_residue(K):
    """n = 3 .. 36: N = 4n takes every residue mod 11 and mod 33 and every even residue mod 22 (N is a multiple of 4);
    34 bands, so the last warp is partly empty at every K"""
    n = np.arange(3, 37)
    g = _ctx(40)
    Hb = _synthetic(100 + K, n, 40)
    lam0 = 1e-5 * R.max_real_diag(Hb, n) * np.random.default_rng(K).uniform(0.5, 2.0, n.size)
    nu0 = np.full(n.size, 2.0)
    dx, ok, lam = _all_forms(g, n, K, Hb=Hb, lam=lam0, nu=nu0)[1]
    assert np.array_equal(lam, _lambda_replay(lam0, nu0, K))
    _check_solution("tpb_recompute", Hb, n, dx, ok, lam, f"n 3..36 K {K}")


def test_long_bands_every_form():
    """n around the 128 / 256 / 512 boundaries at n_cap 512, lambda from 1e-5 max diag to far past the tenth trial"""
    n = np.array([127, 128, 129, 255, 256, 257, 511, 512])
    g = _ctx(512)
    Hb = _synthetic(3, n, 512)
    base = 1e-5 * R.max_real_diag(Hb, n)
    for q in (0, 20):
        lam0, nu0 = _state_after(base, np.full(n.size, 2.0), [q] * n.size)
        dx, ok, lam = _all_forms(g, n, 4, Hb=Hb, lam=lam0, nu=nu0)[1]
        _check_solution("tpb_recompute", Hb, n, dx, ok, lam, f"long bands, trials {q} ..")


def test_ragged_warps_and_retry_lists():
    """bands of any n with inactive bands in between, and retry rounds over lists in any order: every form gives the
    bits of the streamed form; what no system owns keeps the scratch untouched"""
    n_cap = 256
    rng = np.random.default_rng(31)
    n = np.array([3, 256, 7, 129, 4, 255, 30, 200, 12, 64, 5, 100, 41, 88])
    Hb = _synthetic(31, n, n_cap)
    lam0 = 1e-5 * R.max_real_diag(Hb, n) * rng.uniform(0.5, 4.0, n.size)
    nu0 = np.full(n.size, 2.0)
    g = _ctx(n_cap)
    # inactive bands between the real ones
    B = 2 * n.size + 3
    pos = np.sort(rng.choice(B, n.size, replace=False))
    Hb2 = np.repeat(Hb[:1], B, axis=0)
    n2 = rng.integers(3, n_cap + 1, B)
    lam2, nu2 = np.full(B, 1.0), np.full(B, 2.0)
    act = np.zeros(B, np.int32)
    Hb2[pos], n2[pos], lam2[pos], nu2[pos], act[pos] = Hb, n, lam0, nu0, 1
    for K in (2, 4, 6):
        dx, ok, lam = _all_forms(g, n2, K, Hb=Hb2, lam=lam2, nu=nu2, active=act)[1]
        filler = act == 0
        assert _untouched(dx[filler]).all() and _untouched(ok[filler]).all() and _untouched(lam[filler]).all()
        _check_solution("tpb_recompute", Hb2[pos], n2[pos], dx[pos], ok[pos], lam[pos], f"ragged K {K}")
    for K in (2, 4, 8):
        for rep in range(2):
            order = rng.permutation(n.size)[:rng.integers(1, n.size + 1)]
            qmax = rng.integers(0, 10, n.size).astype(np.int32)
            lam, nu = _state_after(lam0, nu0, qmax)
            dx, ok, lam_used = _all_forms(g, n, K, Hb=Hb, lam=lam, nu=nu, qmax=qmax, order=order)[1]
            listed = np.zeros(n.size, bool)
            listed[order] = True
            runs = np.array([[listed[b] and qmax[b] + k < 10 for k in range(K)] for b in range(n.size)])
            assert _untouched(dx[~runs]).all() and _untouched(ok[~runs]).all() and _untouched(lam_used[~runs]).all()
            if runs.any():
                _check_solution("tpb_recompute", Hb, n, dx, ok, lam_used, f"retry list K {K}", trials=runs)


def test_failure_contract_every_form():
    """indefinite systems (a negative direction at several rows, on both sides of segment boundaries), a NaN in b and a
    +inf diagonal entry fail in every form with the same ok / lambda bits; the positive definite originals succeed"""
    n_cap = 128
    g = _ctx(n_cap)
    rng = np.random.default_rng(12)
    n0 = np.array([3, 5, 12, 30, 64, 128])
    Hb0 = _synthetic(21, n0, n_cap)
    lam0 = 1e-5 * R.max_real_diag(Hb0, n0)
    lam_last = 2.0 * lam0
    parts = []
    for where in (3, 10, 11, 21, 22, 23, 33, 44, "N-5"):
        rows = [min(4 * nb - 5, where) if where != "N-5" else 4 * nb - 5 for nb in n0]
        parts.append(R.make_indefinite(Hb0, n0, lam_last, rows, rng))
    nan_b = Hb0.copy()
    inf_d = Hb0.copy()
    for b, nb in enumerate(n0):
        nan_b[b, 2 * nb + 1, 11] = np.nan
        inf_d[b, 2 * nb, 0] = np.inf
    Hb = np.concatenate(parts + [nan_b, inf_d, Hb0])
    n = np.tile(n0, len(parts) + 3)
    lam = np.tile(lam0, len(parts) + 3)
    # k_solve_warp is left out: what it leaves in dx of a failed system is not part of the contract
    dx, ok, lam_used = _all_forms(g, n, 2, warp=False, Hb=Hb, lam=lam, nu=np.full(n.size, 2.0))[1]
    bad = n.size - n0.size
    assert (ok[:bad] == 0).all(), f"ok = 1 for failing systems {np.argwhere(ok[:bad] != 0).ravel()[:10]}"
    assert (ok[bad:] == 1).all()
    _check_solution("tpb_recompute", Hb[bad:], n[bad:], dx[bad:], ok[bad:], lam_used[bad:], "positive definite originals")
