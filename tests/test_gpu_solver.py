"""Every solve kernel of the LM step against a known system, through tebgpu_solve_system (TebGpu.solve_system).

The end-to-end tests compare whole optimizeTEB runs, which LM tolerates inexact steps in: a step that is slightly wrong
but still lowers chi2 is accepted and the band converges to the same minimum. Here the solve alone is pinned, for the
six mappings of (H + lambda I_real) x = b:
  tpb   k_solve_tpb (solver 2, mapping 0)      warp  k_solve_warp (mapping 1)     lat  k_solve_lat (mapping 3)
  auto  mapping 4 (the default: lat or tpb by size, both at once in retry rounds)
  seq   warp_band_solve (solver 0)             bcr   bcr_solve (solver 1, n_cap <= 256)
  a. accuracy against tests/banded_reference.py (longdouble): normwise backward error <= 64 u and, for N <= 512,
     forward error <= 16 u kappa_inf, on kernel A's systems of every scenario and on synthetic systems with weights
     over twelve decades, lambda from 1e-5 max diag to far past g2o's tenth trial;
  b. shapes: n = 3 .. 30, n around 128 / 256 / 512, K = 2 .. 8, partly empty last warps;
  c. placement invariance, bit for bit: batch position, warp neighbours (ragged n, inactive bands), K, round 0 or a
     retry list in any order; tpb and warp bit-identical;
  d. lambda: the replay of spec_lambda exactly, and 1e-5 max |diag| in LM iteration 0;
  e. scratch hygiene: what no kernel should write keeps the all-ones NaN pattern; NaN past N in the input is not read;
  f. failure: indefinite systems (Sylvester: every elimination order meets a non-positive pivot), a NaN in b and a
     +inf diagonal fail in every mapping, positive definite systems succeed in every mapping.
The largest backward error per mapping goes to the parity report that tests/test_gpu_parity.py writes."""
import hashlib

import numpy as np
import pytest

import teb_local_planner_b200 as T
from tests import banded_reference as R
from tests import scenarios
from tests.test_gpu_parity import _report as _write_report

pytestmark = pytest.mark.gpu

U = R.U
BACKWARD_BOUND = 64 * U
MAPPINGS = ["tpb", "warp", "lat", "auto", "seq", "bcr"]
_SELECT = {"tpb": (2, 0), "warp": (2, 1), "lat": (2, 3), "auto": (2, 4), "seq": (0, 4), "bcr": (1, 4)}
ALL_ONES = np.uint64(0xFFFFFFFFFFFFFFFF)
_worst = {}
_contexts = {}
_refs = {}


def _report(mapping, be):
    """largest measured backward error per mapping, in units of u"""
    _worst[mapping] = max(_worst.get(mapping, 0.0), float(np.max(be, initial=0.0)) / U)
    _write_report("solver_backward_error_in_u", dict(sorted(_worst.items())))


def _untouched(a):
    return np.asarray(a).view(np.uint64) == ALL_ONES


def _ctx(n_cap):
    if n_cap not in _contexts:
        _contexts[n_cap] = T.TebGpu(96, n_cap, 1, 1)
    return _contexts[n_cap]


def _cap(mapping, n_cap=512):
    return min(n_cap, 256) if mapping == "bcr" else n_cap


def _select(g, mapping):
    solver, mode = _SELECT[mapping]
    g.set_solver(solver)
    g.set_warp_solver(mode)


def _solve(g, mapping, n, K, **kw):
    _select(g, mapping)
    try:
        return g.solve_system(n, K, **kw)
    finally:
        g.set_solver(2)
        g.set_warp_solver(4)


def _synthetic(seed, n, n_cap, **kw):
    """synthetic systems with NaN in the rows 4n .. 4 n_cap: a kernel that reads past N cannot stay finite"""
    Hb = R.synthetic_systems(np.random.default_rng(seed), n, n_cap, **kw)
    for b, nb in enumerate(n):
        Hb[b, 4 * nb:] = np.nan
    return Hb


def _check_solution(mapping, Hb, n, dx, ok, lam_used, what, trials=None):
    """a. accuracy of every solved (band, trial) system; e. rows >= 4n untouched"""
    n = np.asarray(n)
    B, K = ok.shape
    sel = [(b, k) for b in range(B) for k in range(K) if trials is None or trials[b, k]]
    assert all(ok[b, k] == 1.0 for b, k in sel), f"{mapping} {what}: ok = {ok}"
    bs = np.array([b for b, _ in sel])
    ks = np.array([k for _, k in sel])
    Hs, ns, lams, xs = Hb[bs], n[bs], lam_used[bs, ks], dx[bs, ks]
    for s in range(len(sel)):
        assert _untouched(xs[s, 4 * ns[s]:]).all(), f"{mapping} {what}: rows past N written (band {bs[s]})"
        assert np.isfinite(xs[s, :4 * ns[s]]).all(), f"{mapping} {what}: non-finite solution (band {bs[s]})"
    key = hashlib.sha1(b"".join(np.ascontiguousarray(a).tobytes() for a in (Hs, ns, lams))).hexdigest()
    if key not in _refs:   # the mappings solve the same systems: one reference for all of them
        if len(_refs) >= 32:
            _refs.pop(next(iter(_refs)))
        _refs[key] =(R.ldl_norm(Hs, ns, lams), R.ldl_solve(Hs, ns, lams))
    norm, (xref, okref) = _refs[key]
    be = R.backward_error(Hs, ns, lams, xs, norm)
    _report(mapping, be)
    assert (be <= BACKWARD_BOUND).all(), f"{mapping} {what}: backward error {be.max() / U:.1f} u > 64 u"
    assert okref.all()
    for s in range(len(sel)):
        N = 4 * int(ns[s])
        if N > 512:
            continue
        ref = xref[s, :N].astype(np.float64)
        err = np.abs(xs[s, :N] - ref).max() / np.abs(ref).max()
        if err > 16 * U:   # kappa >= 1: only then is the condition number needed
            A, _ = R.dense(Hs[s], ns[s], lams[s])
            kappa = np.linalg.cond(A, np.inf)
            assert err <= 16 * U * kappa, f"{mapping} {what}: band {bs[s]} forward error {err:.3g} > 16 u kappa ({kappa:.3g})"


def _lambda_replay(lam0, nu0, K, q0=None):
    """lambda of trial q0 + k from the round's (lambda, nu) by the device's sequence of multiplications"""
    lam0 = np.broadcast_to(lam0, (len(lam0),))
    return np.array([[R.spec_lambda(lam0[b], nu0[b], k) for k in range(K)] for b in range(len(lam0))])


def _state_after(lam0, nu0, q):
    """(lambda, nu) after q rejections"""
    lam = np.array([R.spec_lambda(l, v, qq) for l, v, qq in zip(lam0, nu0, q)])
    nu = np.array([v * 2.0 ** qq for v, qq in zip(nu0, q)])
    return lam, nu


# ------------------------------------------------------------------ a. kernel A's systems of every scenario
@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("name", scenarios.ALL)
def test_kernel_a_systems_against_reference(name, mapping):
    p, hb = scenarios.scenario(name)
    if mapping == "bcr" and hb.n_cap > 256:
        pytest.skip("block cyclic reduction runs for n_cap <= 256 only")
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, max(hb.M_cap, 1), hb.V_cap, max_obst_vertices=hb.PV_cap)
    g.set_params(p)
    try:
        for outer in (0, 2):
            Hb, _ = g.build_system(hb, outer)
            n = hb.n.copy()
            base = 1e-5 * R.max_real_diag(Hb, n)
            # LM iteration 0: lambda from kernel A's partials, 1e-5 max |diag| over the real rows (d.)
            dx, ok, lam = _solve(g, mapping, n, 8, n_cap=hb.n_cap)
            assert np.array_equal(lam, _lambda_replay(base, np.full(hb.B, 2.0), 8)), f"{mapping} {name}: lambda init"
            _check_solution(mapping, Hb, n, dx, ok, lam, f"{name} outer {outer} iteration 0")
            # the same system from host memory, lambda from trial 8 (after 8 rejections) onwards: the tenth trial of g2o
            # is 1e-5 max diag 2^45, and lambda carries over between LM iterations, so go past it
            lam8, nu8 = _state_after(base, np.full(hb.B, 2.0), [8] * hb.B)
            dx, ok, lam = _solve(g, mapping, n, 8, Hb=Hb, lam=lam8, nu=nu8)
            assert np.array_equal(lam, _lambda_replay(lam8, nu8, 8))
            assert lam[0, 1] == base[0] * 2.0 ** 45
            _check_solution(mapping, Hb, n, dx, ok, lam, f"{name} outer {outer} lambda x 2^36 .. 2^120")
    finally:
        g.close()


# ------------------------------------------------------------------ a. / b. synthetic systems, shapes
@pytest.mark.parametrize("mapping", MAPPINGS)
@pytest.mark.parametrize("K", [2, 4, 6, 8])
def test_short_bands_every_residue(mapping, K):
    """n = 3 .. 30 (N mod the 10-row chunk and the 11-row window, k_solve_lat's middle block of short systems),
    28 bands: the last warp is partly empty at every K"""
    n = np.arange(3, 31)
    g = _ctx(32)
    Hb = _synthetic(K, n, 32)
    scale = np.random.default_rng(K).uniform(0.5, 2.0, n.size)
    lam0 = 1e-5 * R.max_real_diag(Hb, n) * scale
    nu0 = np.full(n.size, 2.0)
    dx, ok, lam = _solve(g, mapping, n, K, Hb=Hb, lam=lam0, nu=nu0)
    assert np.array_equal(lam, _lambda_replay(lam0, nu0, K))
    _check_solution(mapping, Hb, n, dx, ok, lam, f"n 3..30 K {K}")


@pytest.mark.parametrize("mapping", MAPPINGS)
def test_long_bands_and_weight_spread(mapping):
    """n around the 128 / 256 / 512 boundaries at n_cap 512 (256 for BCR), weights over twelve decades, lambda from
    1e-5 max diag to far past the tenth trial"""
    n_cap = _cap(mapping)
    n = np.array([v for v in (127, 128, 129, 255, 256, 257, 511, 512) if v <= n_cap])
    g = _ctx(n_cap)
    Hb = _synthetic(1, n, n_cap)
    base = 1e-5 * R.max_real_diag(Hb, n)
    for q in (0, 8, 20):
        lam0, nu0 = _state_after(base, np.full(n.size, 2.0), [q] * n.size)
        dx, ok, lam = _solve(g, mapping, n, 8, Hb=Hb, lam=lam0, nu=nu0)
        assert np.array_equal(lam, _lambda_replay(lam0, nu0, 8))
        _check_solution(mapping, Hb, n, dx, ok, lam, f"long bands, trials {q} .. {q + 7}")


def test_lambda_zero_padded_rows_identity():
    """identity rows take no lambda: with lambda huge the real unknowns are ~b / lambda, the identity rows solve to 0"""
    n = np.array([3, 17])
    g = _ctx(32)
    Hb = _synthetic(5, n, 32)
    for mapping in MAPPINGS:
        dx, ok, lam = _solve(g, mapping, n, 2, Hb=Hb, lam=np.full(2, 1e30), nu=np.full(2, 2.0))
        assert (ok == 1).all()
        for b, nb in enumerate(n):
            fixed = ~R.row_is_real(np.arange(4 * nb), nb)
            assert (dx[b, :, :4 * nb][:, fixed] == 0).all(), mapping


# ------------------------------------------------------------------ c. / e. placement invariance, hygiene
def _placement_systems(n_cap):
    n = np.array([3, n_cap, 7, 129, 4, 255, 30, n_cap - 1, 12, 64, 5, 200])
    n = np.minimum(n, n_cap)
    Hb = _synthetic(17, n, n_cap)
    lam0 = 1e-5 * R.max_real_diag(Hb, n) * np.random.default_rng(2).uniform(0.5, 4.0, n.size)
    return n, Hb, lam0, np.full(n.size, 2.0)


_placement_ref = {}


def _placement_reference(mapping):
    n_cap = _cap(mapping)
    n, Hb, lam0, nu0 = _placement_systems(n_cap)
    if mapping not in _placement_ref:
        dx, ok, lam = _solve(_ctx(n_cap), mapping, n, 8, Hb=Hb, lam=lam0, nu=nu0)
        _check_solution(mapping, Hb, n, dx, ok, lam, "placement reference")
        _placement_ref[mapping] = dx
    return n_cap, n, Hb, lam0, nu0, _placement_ref[mapping]


def _same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


@pytest.mark.parametrize("mapping", MAPPINGS)
def test_placement_in_batch_and_neighbours(mapping):
    """the same (band, trial) system gives the same bits wherever its band sits, whoever its warp neighbours are
    (ragged n, inactive bands in between); inactive bands leave the scratch untouched"""
    n_cap, n, Hb, lam0, nu0, ref = _placement_reference(mapping)
    nb = n.size
    rng = np.random.default_rng(9)
    perm = rng.permutation(nb)
    pos = np.sort(rng.choice(2 * nb + 3, nb, replace=False))   # positions of the real bands, inactive ones in between
    B = 2 * nb + 3
    Hb2 = np.repeat(Hb[:1], B, axis=0)
    n2 = np.full(B, 3)
    lam2, nu2 = np.full(B, 1.0), np.full(B, 2.0)
    act = np.zeros(B, np.int32)
    for p, b in zip(pos, perm):
        Hb2[p], n2[p], lam2[p], nu2[p], act[p] = Hb[b], n[b], lam0[b], nu0[b], 1
    filler = np.flatnonzero(act == 0)
    n2[filler] = rng.integers(3, n_cap + 1, filler.size)   # inactive bands with any n
    dx, ok, lam = _solve(_ctx(n_cap), mapping, n2, 8, Hb=Hb2, lam=lam2, nu=nu2, active=act)
    for p, b in zip(pos, perm):
        assert _same_bits(dx[p], ref[b]), f"{mapping}: band {b} at position {p} differs"
    assert _untouched(dx[filler]).all() and _untouched(ok[filler]).all() and _untouched(lam[filler]).all()


@pytest.mark.parametrize("mapping", MAPPINGS)
def test_placement_across_widths(mapping):
    """trial k at width K = 2, 4, 6 with the round started at trial k0 gives the bits of trial k0 + j at K = 8"""
    n_cap, n, Hb, lam0, nu0, ref = _placement_reference(mapping)
    g = _ctx(n_cap)
    for K in (2, 4, 6):
        for k0 in range(0, 8 - K + 1, 2):
            lam, nu = _state_after(lam0, nu0, [k0] * n.size)
            dx, ok, lam_used = _solve(g, mapping, n, K, Hb=Hb, lam=lam, nu=nu)
            assert (ok == 1).all()
            assert _same_bits(dx, ref[:, k0:k0 + K]), f"{mapping}: K {K} from trial {k0}"


@pytest.mark.parametrize("mapping", MAPPINGS)
def test_placement_in_retry_lists(mapping):
    """a retry round over a list in any order: listed bands give the bits of round 0 for trial q0 + k; trials past
    g2o's tenth and the bands not listed keep the scratch untouched"""
    n_cap, n, Hb, lam0, nu0, ref = _placement_reference(mapping)
    g = _ctx(n_cap)
    rng = np.random.default_rng(4)
    for K in (2, 4, 8):
        for rep in range(2):
            order = rng.permutation(n.size)[:rng.integers(1, n.size + 1)]
            qmax = rng.integers(0, 10, n.size).astype(np.int32)
            lam, nu = _state_after(lam0, nu0, qmax)
            dx, ok, lam_used = _solve(g, mapping, n, K, Hb=Hb, lam=lam, nu=nu, qmax=qmax, order=order)
            listed = np.zeros(n.size, bool)
            listed[order] = True
            for b in range(n.size):
                for k in range(K):
                    q = qmax[b] + k
                    if not listed[b] or q >= 10:
                        assert _untouched(dx[b, k]).all() and _untouched(ok[b, k]) and _untouched(lam_used[b, k]), \
                            f"{mapping}: band {b} trial {q} should not run"
                        continue
                    assert ok[b, k] == 1 and lam_used[b, k] == R.spec_lambda(lam0[b], nu0[b], q)
                    if q < 8:
                        assert _same_bits(dx[b, k], ref[b, q]), f"{mapping}: band {b} trial {q} at list position"


def test_tpb_and_warp_bit_identical():
    """k_solve_tpb and k_solve_warp share the algorithm and the operation order: same bits on every system"""
    n_cap, n, Hb, lam0, nu0, ref_tpb = _placement_reference("tpb")
    _, _, _, _, _, ref_warp = _placement_reference("warp")
    assert _same_bits(ref_tpb, ref_warp)
    n = np.arange(3, 31)
    Hb = _synthetic(8, n, 32)
    lam0 = 1e-5 * R.max_real_diag(Hb, n)
    out = [_solve(_ctx(32), m, n, 8, Hb=Hb, lam=lam0, nu=np.full(n.size, 2.0))[0] for m in ("tpb", "warp")]
    assert _same_bits(out[0], out[1])


def test_dual_retry_launch_takes_the_mapping_the_list_length_selects():
    """mapping 4 in a retry round launches k_solve_lat (lat_cap systems) and k_solve_tpb; a list of up to lat_cap / K
    bands is solved by k_solve_lat, a longer one by k_solve_tpb, with exactly their bits"""
    n_cap, n, Hb, lam0, nu0, _ = _placement_reference("tpb")
    g = _ctx(n_cap)
    K = 4
    qmax = np.zeros(n.size, np.int32)
    order = np.arange(n.size)[::-1].copy()
    kw = dict(Hb=Hb, lam=lam0, nu=nu0, qmax=qmax, order=order)
    want = {m: _solve(g, m, n, K, **kw)[0] for m in ("tpb", "lat")}
    assert not _same_bits(want["tpb"], want["lat"])
    for cap, m in ((n.size * K, "lat"), (n.size * K - 1, "tpb"), (1, "tpb")):
        dx = _solve(g, "auto", n, K, lat_cap=cap, **kw)[0]
        assert _same_bits(dx, want[m]), f"lat_cap {cap}: expected the {m} bits"


# ------------------------------------------------------------------ f. failure contract
@pytest.mark.parametrize("mapping", MAPPINGS)
def test_failure_contract(mapping):
    """indefinite systems (the negative direction at rows 3, 10, 11, 20, 21, N-5 and across k_solve_lat's middle block),
    a NaN in b only and a +inf diagonal entry fail (ok = 0) in every mapping; the positive definite originals succeed"""
    n_cap = _cap(mapping, 128)
    g = _ctx(n_cap)
    rng = np.random.default_rng(12)
    n0 = np.array([3, 5, 12, 30, 64, 128])
    Hb0 = _synthetic(21, n0, n_cap)
    lam0 = 1e-5 * R.max_real_diag(Hb0, n0)
    K = 2
    lam_last = 2.0 * lam0    # trial 1; make_indefinite keeps v^T A v < 0 up to that lambda
    parts, ns, lams = [], [], []
    for where in ("3", "10", "11", "20", "21", "N-5", "m-2", "m+4", "m+9"):
        rows = []
        for nb in n0:
            N, m = 4 * nb, (4 * nb - 10) // 2
            rows.append({"N-5": N - 5, "m-2": m - 2, "m+4": m + 4, "m+9": m + 9}.get(where, None)
                        if where.startswith(("N", "m")) else int(where))
        parts.append(R.make_indefinite(Hb0, n0, lam_last, rows, rng))
        ns.append(n0)
        lams.append(lam0)
    nan_b = Hb0.copy()
    inf_d = Hb0.copy()
    for b, nb in enumerate(n0):
        nan_b[b, 2 * nb + 1, 11] = np.nan
        inf_d[b, 2 * nb, 0] = np.inf
    Hb = np.concatenate(parts + [nan_b, inf_d, Hb0])
    n = np.concatenate(ns + [n0, n0, n0])
    lam = np.concatenate(lams + [lam0, lam0, lam0])
    dx, ok, lam_used = _solve(g, mapping, n, K, Hb=Hb, lam=lam, nu=np.full(n.size, 2.0))
    bad = n.size - n0.size
    assert (ok[:bad] == 0).all(), f"{mapping}: ok = 1 for failing systems {np.argwhere(ok[:bad] != 0).ravel()[:10]}"
    assert (ok[bad:] == 1).all()
    _check_solution(mapping, Hb[bad:], n[bad:], dx[bad:], ok[bad:], lam_used[bad:], "positive definite originals")
