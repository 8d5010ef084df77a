"""k_hsig2d / k_hsig3d (tebgpu_h_signature) against the long double oracle (oracle.h_signature) on every case of
tests/hsig_cases.py: the 2-D skip rule at and around 0.05, partial products that leave the fp64 range, a signature
past it, the angle branch cut and its tie, poses on obstacles, the two map rectangles, n = 1 / 2, M = 0 / 1 / 1024;
x-y-t signatures of static and moving obstacles with and without the band's time differences, coincident poses, a
looping band, a world line through a pose.

Bars:
  * 2-D: |H_gpu - H_oracle| <= 1e-12 sum_{k,l} |A_l| |L_kl| (long double restatement in hsig_cases.error_scale: a bar
    on the terms, so that a single wrong term shows even where the terms cancel); +-inf, NaN and exact zeros equal;
  * x-y-t: 1e-12 max(1, |H|) per obstacle, NaN where the oracle has NaN, the rows past M exactly 0;
  * the isEqual partition of each case's candidates and isValid equal the oracle's;
  * every band gives the same bits through the host-buffer and the device-pointer entry points, alone and in a batch
    holding every case (any position, next to any scene; the 2-D batch at M_cap 1024 and the largest n_cap a context
    accepts there).
The worst errors per case go to the parity report (test_gpu_parity._report)."""
import ctypes as C

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi
from tests import hsig_cases as hc
from tests.test_gpu_parity import _report

pytestmark = pytest.mark.gpu
CASES = {c.name: c for c in hc.all_cases()}
NAMES_2D = [c.name for c in CASES.values() if c.dim == 2]
NAMES_3D = [c.name for c in CASES.values() if c.dim == 3]
_want = {}


def _oracle(oracle, case):
    if case.name not in _want:
        p = case.params()
        _want[case.name] = [oracle.h_signature(p, rec, len(rec), case.obst, use_timediffs=case.use_dt) for rec in case.bands]
    return _want[case.name]


def _ctx(B, n_cap, S, M_cap, p):
    g = T.TebGpu(B, n_cap, S, max(M_cap, 1), 0)
    g.set_params(p)
    return g


def _run_host(g, hb, case):
    """host-buffer entry point -> [B][2] (2-D) or [B][max(M_cap, 1)] float64"""
    out = g.h_signature(hb, use_timediffs=case.use_dt)
    return np.stack([out.real, out.imag], 1) if case.dim == 2 else out


def _run_device(g, hb, case):
    """device-pointer entry point into an output prefilled with NaN (a row the kernel leaves unwritten shows)"""
    import torch
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).to(dev)
    keep = dict(poses=t(hb.poses), n=t(hb.n), sid=t(hb.scene_id), ob=t(hb.obstacles), oc=t(hb.obst_count),
                vs=t(hb.vel_start), vg=t(hb.vel_goal))
    stride = max(hb.M_cap, 1) if case.dim == 3 else 2
    out = torch.full((hb.B * stride,), float("nan"), dtype=torch.float64, device=dev)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap = hb.B, hb.n_cap, hb.S, hb.M_cap, 0
    bs.poses, bs.n, bs.scene_id = keep["poses"].data_ptr(), keep["n"].data_ptr(), keep["sid"].data_ptr()
    bs.obstacles = keep["ob"].data_ptr() if hb.M_cap > 0 else None
    bs.obst_count, bs.vel_start, bs.vel_goal = keep["oc"].data_ptr(), keep["vs"].data_ptr(), keep["vg"].data_ptr()
    g._check(g.lib.tebgpu_h_signature(g.ctx, C.byref(bs), int(case.use_dt), out.data_ptr(), 1), "tebgpu_h_signature")
    g.synchronize()
    return out.cpu().numpy().reshape(hb.B, stride)


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint64), np.ascontiguousarray(b).view(np.uint64))


def _check_2d(case, got, want):
    """got [bands][2], want [bands] complex -> worst error over the bar"""
    p = case.params()
    worst = 0.0
    for i, rec in enumerate(case.bands):
        w = np.array([want[i].real, want[i].imag])
        where = (case.name, i, got[i], w)
        for q in range(2):
            if not np.isfinite(w[q]):
                assert (np.isnan(w[q]) and np.isnan(got[i, q])) or got[i, q] == w[q], where
        if not np.all(np.isfinite(w)):
            continue
        if w[0] == 0 and w[1] == 0:
            assert got[i, 0] == 0 and got[i, 1] == 0, where
            continue
        scale = hc.error_scale(p, rec, case.obst)
        err = np.hypot(hc.LD(got[i, 0]) - hc.LD(w[0]), hc.LD(got[i, 1]) - hc.LD(w[1]))
        bar = max(hc.LD(1e-12) * scale, hc.LD(5e-324))
        assert np.isfinite(got[i]).all() and err <= bar, where + (float(err), float(scale))
        worst = max(worst, float(err / scale) if scale > 0 else 0.0)
    return worst


def _check_3d(case, got, want, M_cap):
    M = len(case.obst)
    worst = 0.0
    for i in range(len(case.bands)):
        g, w = got[i, :M], want[i]
        assert np.array_equal(np.isnan(g), np.isnan(w)), (case.name, i)
        ok = ~np.isnan(w)
        err = np.abs(g[ok] - w[ok]) / np.maximum(1.0, np.abs(w[ok]))
        assert np.all(err <= 1e-12), (case.name, i, err.max(initial=0))
        worst = max(worst, float(err.max(initial=0)))
        assert np.all(got[i, M:max(M_cap, 1)] == 0), (case.name, i, got[i, M:])     # padding written as 0
    return worst


def _classes(case, vals, thr):
    valid = [hc.is_valid(v) for v in vals]
    return hc.partition(vals, case.dim, thr), valid


def _as_values(case, rows):
    M = len(case.obst)
    return [complex(r[0], r[1]) for r in rows] if case.dim == 2 else [r[:M] for r in rows]


@pytest.mark.parametrize("name", NAMES_2D)
def test_hsig2d_case_matches_oracle(oracle, name):
    case = CASES[name]
    want = _oracle(oracle, case)
    hb, _ = hc.batch([case])
    g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, case.params())
    got = _run_host(g, hb, case)
    dev = _run_device(g, hb, case)
    g.close()
    assert _same_bits(got, dev)
    worst = _check_2d(case, got, want)
    thr = case.params().h_signature_threshold
    assert _classes(case, _as_values(case, got), thr) == _classes(case, want, thr)
    _report(f"hsig/{name}", {"bands": len(case.bands), "M": len(case.obst),
                             "max_err_over_sum_abs_terms": worst, "bar": 1e-12})


@pytest.mark.parametrize("name", NAMES_3D)
def test_hsig3d_case_matches_oracle(oracle, name):
    """M_cap = M + 3: the rows past M must come back as 0. The context's output buffer holds a 2-D result of the same
    batch first, so a row the kernel does not write shows on the host-buffer path as well"""
    case = CASES[name]
    want = _oracle(oracle, case)
    M_cap = len(case.obst) + 3 if len(case.obst) else 0
    hb, _ = hc.batch([case], M_cap=M_cap)
    p2 = case.params()
    p2.include_dynamic_obstacles = 0
    g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, p2)
    g.h_signature(hb)
    g.set_params(case.params())
    got = _run_host(g, hb, case)
    dev = _run_device(g, hb, case)
    g.close()
    assert _same_bits(got, dev)
    worst = _check_3d(case, got, want, M_cap)
    thr = case.params().h_signature_threshold
    assert _classes(case, _as_values(case, got), thr) == _classes(case, want, thr)
    _report(f"hsig/{name}", {"bands": len(case.bands), "M": len(case.obst), "use_timediffs": bool(case.use_dt),
                             "max_err_rel_max1": worst, "bar": 1e-12})


def _largest_n_cap(B, S, M_cap):
    """the largest pose capacity (a multiple of 32, at most 512) for which a context with M_cap obstacles is created: the
    optimisation kernels' shared memory bounds it, not the signature kernels'"""
    for n_cap in range(512, 31, -32):
        try:
            T.TebGpu(B, n_cap, S, M_cap, 0).close()
            return n_cap
        except T.TebGpuError:
            continue
    raise AssertionError(f"no context accepts M_cap = {M_cap}")


@pytest.mark.parametrize("dim", [2, 3])
def test_hsig_batch_position_and_entry_points(dim):
    """every band of every case alone, in one batch with all the others (one scene per case) and in that batch reversed,
    through both entry points: the same bits everywhere. The 2-D batch runs at M_cap 1024 and the largest n_cap a
    context accepts there; the x-y-t batch at M_cap past every scene's M. The x-y-t cases with and without time
    differences run in separate batches (use_timediffs is per call)."""
    groups = [[c for c in CASES.values() if c.dim == 2]] if dim == 2 else \
        [[c for c in CASES.values() if c.dim == 3 and c.use_dt == u] for u in (True, False)]
    for cases in groups:
        alone = {}
        for c in cases:
            hb, _ = hc.batch([c], M_cap=len(c.obst) + (2 if dim == 3 else 0))
            g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, c.params())
            alone[c.name] = _run_host(g, hb, c)
            g.close()
        M_cap = 1024 if dim == 2 else max(len(c.obst) for c in cases) + 5
        n_cap = _largest_n_cap(sum(len(c.bands) for c in cases), len(cases), M_cap) if dim == 2 else None
        for reverse in (False, True):
            hb, where = hc.batch(cases, n_cap=n_cap, M_cap=M_cap, reverse=reverse)
            g = _ctx(hb.B, hb.n_cap, hb.S, hb.M_cap, cases[0].params())
            host, dev = _run_host(g, hb, cases[0]), _run_device(g, hb, cases[0])
            g.close()
            assert _same_bits(host, dev)
            for c, i, r in where:
                M = len(c.obst)
                a, b = host[r, :2] if dim == 2 else host[r, :M], alone[c.name][i, :2] if dim == 2 else alone[c.name][i, :M]
                assert _same_bits(a, b), (c.name, i, r, reverse)
                if dim == 3:
                    assert np.all(host[r, M:] == 0), (c.name, i, r)
