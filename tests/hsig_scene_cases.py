"""H-signature cases above 1024 obstacles per scene, for tebgpu_h_signature_scenes (tests/test_gpu_hsig_scene.py), and
the long double restatement they are checked against.

The 2-D signature (h_signature.h:97-186) recomputes A_l = f0(o_l) / prod_{j != l} (o_l - o_j) inside its segment loop:
O(n M^2) long double divisions per band, some 2.7e10 at M = 16384 and n = 100. Here the product over j is formed once
per scene (scene_products), in long double on chunks of 256 factors with a binary exponent carried between chunks, so
that no partial product leaves the long double range; the band then needs only f0 and the sum over (k, l). The skip
rule is the reference's cabsl(o_l - o_j) < 0.05 in long double. tests/test_hsig_scene_cases.py holds this restatement
to the oracle's own h_signature_2d (oracle/teb_oracle.c) on every 2-D case of tests/hsig_cases.py.

error_scale is hsig_cases.error_scale computed row chunk by row chunk (the existing one builds an M x M matrix, 4 GB at
16384 rows): the same per-row sums, so the same value.
"""
import math

import numpy as np

from teb_local_planner_b200 import abi, scenes
from tests import hsig_cases as hc

LD = np.longdouble
SKIP = hc.SKIP
_CH = 256


def _frexp_ld(z):
    """complex long double array -> (mantissa with |.| in [0.5, 1), exponent); 0 stays 0 with exponent 0"""
    e = np.frexp(np.maximum(np.abs(z.real), np.abs(z.imag)))[1]
    return np.ldexp(z.real, -e) + 1j * np.ldexp(z.imag, -e), e.astype(np.int64)


def scene_products(ob, rows=128):
    """P_l = prod_{j != l, cabsl(o_l - o_j) >= 0.05} (o_l - o_j) in long double as (mantissa [M] clongdouble, exponent [M])"""
    M = len(ob)
    x, y = ob["x"].astype(LD), ob["y"].astype(LD)
    mant = np.ones(M, np.clongdouble)
    expo = np.zeros(M, np.int64)
    for l0 in range(0, M, rows):
        l1 = min(M, l0 + rows)
        dx = x[l0:l1, None] - x[None, :]
        dy = y[l0:l1, None] - y[None, :]
        q = dx * dx + dy * dy
        c2 = LD(SKIP) * LD(SKIP)
        keep = q >= c2
        near = np.abs(q - c2) <= LD(1e-12) * c2            # decide these on the modulus, as cabsl does
        if near.any():
            keep[near] = np.hypot(dx[near], dy[near]) >= LD(SKIP)
        keep[np.arange(l1 - l0), np.arange(l0, l1)] = False
        f = np.where(keep, dx + 1j * dy, 1).astype(np.clongdouble)
        m, e = np.ones(l1 - l0, np.clongdouble), np.zeros(l1 - l0, np.int64)
        for j0 in range(0, M, _CH):                          # |chunk product| within 0.05^256 .. (range)^256
            cm, ce = _frexp_ld(np.prod(f[:, j0:j0 + _CH], axis=1))
            m, e2 = _frexp_ld(m * cm)
            e = e + ce + e2
        mant[l0:l1], expo[l0:l1] = m, e
    return mant, expo


def _f0(p, rec, ob):
    """f0(o_l) of the band in long double, as the oracle forms it"""
    M, n = len(ob), len(rec)
    m = max(M - 1, 5)
    a = int(math.ceil(m / 2.0))
    b = m - a
    start = LD(rec[0, 0]) + 1j * LD(rec[0, 1])
    end = LD(rec[n - 1, 0]) + 1j * LD(rec[n - 1, 1])
    delta = (end - start).astype(np.clongdouble)
    normal = -delta.imag + 1j * delta.real
    if np.abs(delta) < 3.0:
        bl, tr = start + (0 - 3j), start + (3 + 3j)
    else:
        bl, tr = start - normal, start + delta + normal
    ol = ob["x"].astype(LD) + 1j * ob["y"].astype(LD)
    return LD(p.h_signature_prescaler) * LD(a) * (ol - bl) * LD(b) * (ol - tr)


def _L(rec, ob):
    """L_kl = ln|z2 - o| - ln|z1 - o| + i * smallest-magnitude angle difference, as the oracle forms it ([n-1][M]
    complex128, 0 where the term is skipped)"""
    n = len(rec)
    ox, oy = ob["x"].astype(LD), ob["y"].astype(LD)
    zx, zy = rec[:, 0].astype(LD), rec[:, 1].astype(LD)
    wx, wy = zx[:, None] - ox[None, :], zy[:, None] - oy[None, :]
    d = np.hypot(wx, wy).astype(np.float64)
    ang = np.arctan2(wy, wx)
    with np.errstate(divide="ignore", invalid="ignore"):
        lr = np.log(d[1:]) - np.log(d[:-1])
    ad = (ang[1:] - ang[:-1]).astype(np.float64)
    prop = np.stack([ad, ad + 2 * math.pi, ad - 2 * math.pi, ad + 4 * math.pi, ad - 4 * math.pi])
    li = np.take_along_axis(prop, np.argmin(np.abs(prop), axis=0)[None], 0)[0]
    ok = (d[1:] != 0) & (d[:-1] != 0)
    return np.where(ok, lr + 1j * li, 0).reshape(n - 1, len(ob))


def oracle_2d(p, rec, ob, products=None):
    """the long double 2-D signature as a complex128 (inf / 0 where the long double value lies past the fp64 range)"""
    M, n = len(ob), len(rec)
    if M == 0 or n < 1:
        return 0j
    if n < 2:
        return 0j
    pm, pe = scene_products(ob) if products is None else products
    am, ae = _frexp_ld(_f0(p, rec, ob) / pm)
    ae = ae - pe
    nz = (am.real != 0) | (am.imag != 0)
    if not nz.any():
        return 0j
    emax = int(ae[nz].max())
    scale = np.where(nz, np.ldexp(np.ones(M, LD), np.clip(ae - emax, -20000, 0)), 0)
    A = am * scale
    Ls = _L(rec, ob).astype(np.clongdouble).sum(axis=0)
    H = (A * Ls).sum()
    e = min(max(emax, -20000), 20000)
    r, i = np.ldexp(H.real, e), np.ldexp(H.imag, e)
    return complex(float(r), float(i))


def error_scale(p, rec, ob, rows=256):
    """hsig_cases.error_scale, row chunk by row chunk: sum_{k,l} |A_l| |L_kl| in long double"""
    M, n = len(ob), len(rec)
    if M == 0 or n < 2:
        return LD(0)
    z = rec[:, 0] + 1j * rec[:, 1]
    o = ob["x"].astype(np.float64) + 1j * ob["y"].astype(np.float64)
    m = max(M - 1, 5)
    a = int(math.ceil(m / 2.0))
    b = m - a
    delta = z[-1] - z[0]
    if abs(delta) < 3.0:
        bl, tr = z[0] - 3j, z[0] + 3 + 3j
    else:
        nrm = complex(-delta.imag, delta.real)
        bl, tr = z[0] - nrm, z[0] + delta + nrm
    f0 = p.h_signature_prescaler * a * (o - bl) * b * (o - tr)
    x, y = ob["x"].astype(np.float64), ob["y"].astype(np.float64)
    logA = np.empty(M)
    for l0 in range(0, M, rows):
        l1 = min(M, l0 + rows)
        dif = o[l0:l1, None] - o[None, :]
        keep = np.abs(dif) >= SKIP
        keep[np.arange(l1 - l0), np.arange(l0, l1)] = False
        d = np.hypot(x[l0:l1, None] - x[None, :], y[l0:l1, None] - y[None, :])
        for li, j in zip(*np.nonzero(np.abs(d - SKIP) <= 1e-9 * SKIP)):
            if l0 + li != j:
                keep[li, j] = not hc.skip_decisions(ob, l0 + li, j)[0]
        with np.errstate(divide="ignore"):
            logd = np.where(keep, np.log(np.where(keep, dif, 1.0)), 0.0)
            logA[l0:l1] = (np.log(f0[l0:l1].astype(np.complex128)) - logd.sum(axis=1)).real
    L = np.zeros((max(n - 1, 0), M), np.complex128)
    for k in range(n - 1):
        w1, w2 = z[k] - o, z[k + 1] - o
        d1, d2 = np.abs(w1), np.abs(w2)
        ok = (d1 != 0) & (d2 != 0)
        ad = np.angle(w2) - np.angle(w1)
        prop = np.stack([ad, ad + 2 * np.pi, ad - 2 * np.pi, ad + 4 * np.pi, ad - 4 * np.pi])
        li = prop[np.argmin(np.abs(prop), axis=0), np.arange(M)]
        with np.errstate(divide="ignore", invalid="ignore"):
            L[k] = np.where(ok, (np.log(d2) - np.log(d1)) + 1j * li, 0)
    return (np.exp(LD(1) * logA)[None, :] * np.abs(L).astype(LD)).sum()


# ------------------------------------------------------------------------------------------------ cases
def _costmap(M, seed):
    """scenes.costmap_scene's rows (one point per occupied 5 cm cell, walls and blobs) and a bundle of candidates
    through the corridor, around the blobs"""
    p, hb = scenes.costmap_scene(M, n=100, candidates=4, seed=seed, shapes=False)   # n = 100: room for 16384 cells
    ob = hb.obstacles[0, :M].copy()
    L = 0.4 * 0.3 * 99
    bands = hc.bundle((-L / 2, 0.0), (L / 2, 0.3), 60, [0.0, 0.5, -0.5, 1.1])
    return hc.Case(f"costmap_{M}", 2, ob, bands)


def _grid_block(nx, ny):
    """an nx x ny block of 5 cm costmap cells, row-major: every row / column neighbour pair at the skip threshold"""
    ob = hc.obstacles(hc.grid_cells(nx, ny, -0.05 * nx / 2, -0.05 * ny / 2))
    # one band on each side: |H| ~ 1e162, where two bands of one class would differ by rounding noise far above 0.1
    bands = hc.bundle((-0.05 * nx, -0.05 * ny), (0.05 * nx, 0.05 * ny + 0.4), 40, [1.2, -1.2])
    return hc.Case(f"grid_{nx}x{ny}", 2, ob, bands)


def _duplicates():
    """a 40 x 30 block with every 7th cell listed twice (diff == 0: skipped by every formula)"""
    cells = hc.grid_cells(40, 30, -1.0, -0.75)
    cells = cells + cells[::7]
    ob = hc.obstacles(cells)
    bands = hc.bundle((-2.0, -1.2), (2.0, 1.4), 40, [1.0, -1.0])
    return hc.Case(f"duplicates_{len(ob)}", 2, ob, bands)


def _far_before_near(M=1100):
    """target T, far rows about 10 m away listed before near duplicates 0.06 m from T: the fp64 running product of A_T
    underflows on the far rows, while the long double value is moderate"""
    T, P = (0.2, 0.1), (0.26, 0.1)
    near = 511
    far = [(6.0 + 0.25 * (i % 30), 7.0 + 0.25 * (i // 30)) for i in range(M - 1 - near)]
    ob = hc.obstacles([T] + far + [P] * near)
    assert len(ob) == M
    pp = hc.fp64_partial_products(abi.default_params(), hc.bent((-2.0, -0.8), (2.0, 1.0), 30, 0.0), ob, 0)
    assert np.any(pp == 0)                                   # a plain fp64 running product leaves the range
    return hc.Case(f"far_before_near_{M}", 2, ob, [hc.bent((-2.0, -0.8), (2.0, 1.0), 30, b) for b in (0.0, 0.5, -0.5)])


def _ring(M, K=4, seed=0):
    """M rows at K positions on a circle of radius r, in random order. The product of the distances from one vertex of a
    regular K-gon to the others is K r^(K-1), and the duplicates of a row's own position are skipped (diff == 0), so
    |Q_l| = (K r^(K-1))^(-M/K): r is chosen for |Q_l| ~ 2^-(3 log2 M + 5), which keeps |H| of order 1 however many
    rows there are. The signature stays inside the fp64 range above 2048 rows, where the product runs in several
    parts, and far enough from 1e12 that fp64 rounding cannot cross h_signature_threshold between equal classes"""
    g = 3 * math.log2(M) + 5                                 # |Q_l| ~ 2^-g: |H| of order 1 against f0 ~ M^2 over M rows
    r = (2.0 ** (g / (M // K)) / K) ** (1.0 / (K - 1))
    c, th = (0.3, -0.2), 0.37
    pos = [(c[0] + r * math.cos(2 * math.pi * k / K + th), c[1] + r * math.sin(2 * math.pi * k / K + th)) for k in range(K)]
    order = np.random.default_rng(seed).permutation(np.arange(M) % K)
    ob = hc.obstacles([pos[k] for k in order])
    bands = hc.bundle((-3.0, -1.0), (3.0, 1.2), 40, [1.6, 0.0, -1.6, 0.8])
    return hc.Case(f"ring_{M}", 2, ob, bands)


def cases_2d(large=True):
    """the 2-D cases; large=False leaves out the 16384-row scenes (some tens of seconds of long double each)"""
    out = [_costmap(1025, 3), _costmap(2048, 4), _costmap(4096, 5), _grid_block(64, 32), _duplicates(),
           _far_before_near(), _ring(4096, seed=1)]
    if large:
        out += [_costmap(16384, 6), _ring(16384, seed=2)]
    return out


def assert_class_margins(case, vals, thr):
    """isEqual compares component differences of two bands with thr: every finite one at least 1e-9 max(1, thr) and
    1e-10 of the larger |H| away from it, so that an fp64 error within the 2-D bar cannot move a band to another class"""
    for i, a in enumerate(vals):
        for b in vals[i + 1:]:
            for d in (abs(a.real - b.real), abs(a.imag - b.imag)):
                assert not np.isfinite(d) or abs(d - thr) > max(1e-9 * max(1.0, thr), 1e-10 * max(abs(a), abs(b))), \
                    (case.name, a, b)


def factor_rel_errors(factor, factor_exp, products):
    """|Q_gpu / Q_ld - 1| per row, Q_gpu = (factor[l][0] + i factor[l][1]) 2^factor_exp[l] from the device table and
    Q_ld = 1 / P_l from scene_products (mantissa and exponent, so that neither underflows)"""
    pm, pe = products
    M = len(pm)
    q = factor[:M, 0].astype(LD) + 1j * factor[:M, 1].astype(LD)
    ratio = q * pm.astype(np.clongdouble)
    ratio = np.ldexp(ratio.real, (factor_exp[:M].astype(np.int64) + pe)) + 1j * np.ldexp(ratio.imag, (factor_exp[:M].astype(np.int64) + pe))
    return np.abs(ratio - 1)


def cases_3d():
    """costmap scenes with moving rows (scenes.costmap_scene's shapes: four moving points) for the x-y-t signature"""
    out = []
    for M, seed in ((2048, 7), (16384, 8)):
        p, hb = scenes.costmap_scene(M, n=100, candidates=3, seed=seed)
        ob = hb.obstacles[0, :M].copy()
        ob["type"][ob["type"] == abi.TEB_OBST_LINE] = abi.TEB_OBST_POINT   # no vertex pool: the signature reads x, y only
        ob["vertex_begin"], ob["vertex_count"] = 0, 0
        assert (ob["dynamic"] != 0).sum() >= 4
        out.append(hc.Case(f"xyt_costmap_{M}", 3, ob, [hb.poses[b, :hb.n[b]].copy() for b in range(hb.B)]))
    return out
