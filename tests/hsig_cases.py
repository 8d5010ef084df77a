"""H-signature cases at the edges of HSignature / HSignature3d::calculateHSignature (h_signature.h:97-186, :282-353),
shared by tests/test_reference_pin_hsig.py (oracle against the reference's own header) and tests/test_gpu_hsig.py
(k_hsig2d / k_hsig3d against the oracle). Plain numpy; every builder asserts on the host the property its case claims.

Skip rule. The 2-D signature leaves obstacle j out of A_l when |o_l - o_j| < 0.05, decided in long double on the exact
difference of the two centroids. A decision taken on rounded fp64 differences (hypot of o_l.x - o_j.x, ...) parts from
it where a difference of two coordinates is not exact in fp64: centroids of smaller magnitude than their difference, or
on both sides of the origin. The builders keep every obstacle pair away from the threshold except where the pair is the
point of the case, and there the exact (rational) decision, the long double decision and the intended fp64 decision
are asserted here; no pair lies within 1e-17 relative of the threshold unless its modulus is exactly 0.05, so a decision
taken on a double-double modulus (about 1e-30 relative) agrees with the long double one on every case.

Range. A_l = f0 / prod_j (o_l - o_j) is a running product of up to M - 1 factors. Long double keeps exponents to about
1e+-4932, fp64 to 1e+-308: far obstacles listed before near ones take an fp64 partial product to 0, the reverse order
to inf, while the long double value is O(1). Where the final long double signature itself is past the fp64 range the
double the C-ABI returns is +-inf, so isValid is false for the oracle and the kernels while the reference, which keeps
the long double, says true: the one documented difference (Case.beyond_range).
"""
import math
from fractions import Fraction

import numpy as np

from teb_local_planner_b200 import abi

SKIP = 0.05
LD = np.longdouble
_H = float.fromhex


class Case:
    """dim 2 or 3; obst: OBST_DTYPE rows of the scene; bands: list of [n][4] arrays (x, y, theta, dt to the next pose)"""

    def __init__(self, name, dim, obst, bands, use_dt=True, beyond_range=False):
        self.name, self.dim, self.obst, self.bands, self.use_dt = name, dim, obst, bands, use_dt
        self.beyond_range = beyond_range

    def params(self):
        p = abi.default_params()
        p.include_dynamic_obstacles = int(self.dim == 3)
        return p

    def __repr__(self):
        return f"Case({self.name})"


def obstacles(xy, v=None):
    xy = np.asarray(xy, np.float64).reshape(-1, 2)
    ob = np.zeros(len(xy), abi.OBST_DTYPE)
    ob["type"] = abi.TEB_OBST_POINT
    ob["x"], ob["y"] = xy[:, 0], xy[:, 1]
    if v is not None:
        v = np.asarray(v, np.float64).reshape(-1, 2)
        ob["vx"], ob["vy"] = v[:, 0], v[:, 1]
        ob["dynamic"] = (v[:, 0] != 0) | (v[:, 1] != 0)
    return ob


def band(xy, dt=0.3):
    xy = np.asarray(xy, np.float64).reshape(-1, 2)
    rec = np.zeros((len(xy), 4))
    rec[:, :2] = xy
    if len(xy) > 1:
        d = np.diff(xy, axis=0)
        rec[:-1, 2] = np.arctan2(d[:, 1], d[:, 0])
        rec[-1, 2] = rec[-2, 2]
    rec[:-1, 3] = dt
    return rec


def bent(start, goal, n, bump):
    """n poses from start to goal, pushed sideways by bump * sin(pi s) (left of the direction of travel for bump > 0)"""
    s = np.linspace(0.0, 1.0, n)
    a, g = np.asarray(start, float), np.asarray(goal, float)
    d = g - a
    nrm = np.array([-d[1], d[0]]) / np.hypot(*d)
    return band(a + s[:, None] * d + bump * np.sin(np.pi * s)[:, None] * nrm)


def bundle(start, goal, n, bumps):
    return [bent(start, goal, n, b) for b in bumps]


# ------------------------------------------------------------------------------------------------ host-side checks
def skip_decisions(ob, l, j):
    """(exact, long double, fp64 hypot) answers to |o_l - o_j| < 0.05 (exact: rationals)"""
    ax, ay, bx, by = float(ob["x"][l]), float(ob["y"][l]), float(ob["x"][j]), float(ob["y"][j])
    dx, dy = Fraction(ax) - Fraction(bx), Fraction(ay) - Fraction(by)
    exact = dx * dx + dy * dy < Fraction(SKIP) ** 2
    ld = bool(np.hypot(LD(ax) - LD(bx), LD(ay) - LD(by)) < LD(SKIP))
    return exact, ld, bool(np.hypot(ax - bx, ay - by) < SKIP)


def near_pairs(ob, rel=1e-9):
    """index pairs l < j with an fp64 modulus within rel of the threshold"""
    x, y = ob["x"].astype(np.float64), ob["y"].astype(np.float64)
    d = np.hypot(x[:, None] - x[None, :], y[:, None] - y[None, :])
    li, ji = np.nonzero(np.triu(np.abs(d - SKIP) <= rel * SKIP, 1))
    return list(zip(li.tolist(), ji.tolist()))


def assert_skip_margin(ob):
    """every near-threshold pair: the long double decision is the exact one, and the exact squared modulus is either
    exactly 0.05^2 or more than 1e-17 relative away from it (outside the band where a double-double decision and the
    long double one could part)"""
    c2 = Fraction(SKIP) ** 2
    for l, j in near_pairs(ob):
        exact, ld, _ = skip_decisions(ob, l, j)
        assert ld == exact, (l, j)
        dx = Fraction(float(ob["x"][l])) - Fraction(float(ob["x"][j]))
        dy = Fraction(float(ob["y"][l])) - Fraction(float(ob["y"][j]))
        q = dx * dx + dy * dy
        assert q == c2 or abs(q - c2) > Fraction(1, 10 ** 17) * c2, (l, j)


def disagreements(ob):
    """near-threshold pairs whose fp64 hypot decision differs from the exact one: [(l, j, exact)]"""
    out = []
    for l, j in near_pairs(ob):
        exact, _, f64 = skip_decisions(ob, l, j)
        if exact != f64:
            out.append((l, j, exact))
    return out


def ld_terms(p, rec, ob):
    """long double restatement for the error bar: log|A_l| (float64 is enough for a bar), the complex A_l as long
    double from its logarithm, and L_kl (complex128, 0 where the term is skipped); skip decisions exact"""
    M, n = len(ob), len(rec)
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
    dif = o[:, None] - o[None, :]
    keep = np.abs(dif) >= SKIP
    np.fill_diagonal(keep, False)
    for l, j in near_pairs(ob):
        keep[l, j] = keep[j, l] = not skip_decisions(ob, l, j)[0]
    with np.errstate(divide="ignore"):
        logd = np.where(keep, np.log(np.where(keep, dif, 1.0)), 0.0)
        logA = np.log(f0.astype(np.complex128)) - logd.sum(axis=1)
    A = np.exp(LD(1) * logA.real) * (np.cos(LD(1) * logA.imag) + 1j * np.sin(LD(1) * logA.imag).astype(LD))
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
    return logA.real, A, L


def error_scale(p, rec, ob):
    """sum_{k,l} |A_l| |L_kl| in long double: the 2-D error bar is 1e-12 of it"""
    if len(ob) == 0 or len(rec) < 2:
        return LD(0)
    logA, _, L = ld_terms(p, rec, ob)
    return (np.exp(LD(1) * logA)[None, :] * np.abs(L).astype(LD)).sum()


def fp64_partial_products(p, rec, ob, l):
    """|A_l| after every division of the fp64 running product the way a plain fp64 kernel forms it"""
    M = len(ob)
    m = max(M - 1, 5)
    a = int(math.ceil(m / 2.0))
    b = m - a
    z0, z1 = complex(rec[0, 0], rec[0, 1]), complex(rec[-1, 0], rec[-1, 1])
    d = z1 - z0
    bl, tr = (z0 - 3j, z0 + 3 + 3j) if abs(d) < 3.0 else (z0 - complex(-d.imag, d.real), z0 + d + complex(-d.imag, d.real))
    o = complex(ob["x"][l], ob["y"][l])
    A = p.h_signature_prescaler * a * (o - bl) * b * (o - tr)
    out = []
    for j in range(M):
        if j == l:
            continue
        c = o - complex(ob["x"][j], ob["y"][j])
        if abs(c) < SKIP:
            continue
        den = c.real * c.real + c.imag * c.imag
        with np.errstate(all="ignore"):
            A = complex((A.real * c.real + A.imag * c.imag) / den, (A.imag * c.real - A.real * c.imag) / den)
        out.append(abs(A) if math.isfinite(A.real) and math.isfinite(A.imag) else math.inf)
    return np.array(out)


def arg_diffs(rec, ob):
    """raw atan2 differences [(n-1)][M] of every (segment, obstacle) term"""
    o = ob["x"] + 1j * ob["y"]
    z = rec[:, 0] + 1j * rec[:, 1]
    return np.array([np.angle(z[k + 1] - o) - np.angle(z[k] - o) for k in range(len(z) - 1)])


def assert_no_near_tie(rec, ob):
    """|arg diff| is pi exactly or away from it: a rounding at the tie would select another proposal"""
    ad = np.abs(arg_diffs(rec, ob))
    assert np.all((ad == np.pi) | (np.abs(ad - np.pi) > 1e-9))


# ------------------------------------------------------------------------------------------------ 2-D cases
def _skip_exact():
    """pairs at exactly 0.05 (kept: 0.05 < 0.05 is false) and at the double just below (skipped) - every formula agrees"""
    c = SKIP
    ob = obstacles([(0.0, 0.0), (c, 0.0), (2 * c, 0.0), (0.0, 1.0), (float(np.nextafter(c, 0)), 1.0), (1.0, 0.5)])
    assert float(ob["x"][1]) - 0.0 == c and float(ob["x"][2]) - float(ob["x"][1]) == c
    for l, j, want in ((0, 1, False), (1, 2, False), (3, 4, True)):
        assert skip_decisions(ob, l, j) == (want, want, want)
    return Case("skip_exact", 2, ob, bundle((-1.0, -0.6), (1.6, 1.4), 24, [0.9, -0.9, 0.1]))


_FP64_SKIPS = [  # exact modulus >= 0.05, fp64 hypot of the rounded differences < 0.05
    (("0x1.cdb496747fb27p-6", "0x1.81b8de3215747p-6"), ("0x1.0fffbe363952dp-4", "0x1.c8e448cd77078p-5")),
    (("0x1.f95b1b1f4e7d7p-6", "0x1.6624d8792de37p-6"), ("0x1.08ab3e63d76fep-4", "0x1.e11e0f790e5cap-5"))]
_FP64_KEEPS = [  # exact modulus < 0.05, fp64 hypot of the rounded differences >= 0.05
    (("0x1.a1940d97cdfb0p-7", "0x1.6c9b443991c8dp-6"), ("0x1.889898769d248p-5", "0x1.d95b4b36b4416p-5")),
    (("0x1.582215f480bb7p-5", "0x1.7054c52dfe627p-8"), ("0x1.2a56ea4dd47e6p-4", "0x1.70853bdbdae61p-5"))]
_FP64_KEEPS_1D = [("0x1.e142247d10747p-6", "-0x1.51f10eb622becp-6"), ("0x1.90db438c3953ep-7", "-0x1.3562c8b68b44ap-5")]


def _skip_pair_case(name, pair, exact_skips, mirror):
    """one pair from a search (kept for both signs), mirrored through the origin for the second pair of a case, plus two
    obstacles a metre away"""
    (ax, ay), (bx, by) = [(_H(u), _H(v)) for u, v in pair]
    s = -1.0 if mirror else 1.0
    ob = obstacles([(s * ax, s * ay), (s * bx, s * by), (1.1, -0.4), (-0.9, 0.7)])
    exact, ld, f64 = skip_decisions(ob, 0, 1)
    assert exact == ld == exact_skips and f64 != exact_skips
    return ob


def _skip_rounded():
    cases = []
    for sign, pairs in (("fp64_skips", _FP64_SKIPS), ("fp64_keeps", _FP64_KEEPS)):
        for i, pair in enumerate(pairs):
            ob = _skip_pair_case(sign, pair, sign == "fp64_keeps", mirror=bool(i))
            cases.append(Case(f"skip_{sign}_{i}", 2, ob, bundle((-1.5, -0.3), (1.5, 0.4), 20, [0.8, -0.8, 0.05])))
    # dy = 0: the rounding of one subtraction alone decides, whatever the hypot: x1 - x2 < 0.05 exactly, == 0.05 in fp64
    xy = []
    for i, (u, v) in enumerate(_FP64_KEEPS_1D):
        x1, x2 = _H(u), _H(v)
        assert Fraction(x1) - Fraction(x2) < Fraction(SKIP) and x1 - x2 == SKIP
        xy += [(x1, 0.8 * i), (x2, 0.8 * i)]
    ob = obstacles(xy + [(1.2, 0.3)])
    for i in range(len(_FP64_KEEPS_1D)):
        assert skip_decisions(ob, 2 * i, 2 * i + 1) == (True, True, False)
    cases.append(Case("skip_fp64_keeps_1d", 2, ob, bundle((-1.5, -0.4), (1.5, 1.2), 20, [0.7, -0.7])))
    return cases


def _skip_duplicates():
    """two obstacles at the same point: diff == 0, skipped by every formula"""
    ob = obstacles([(0.2, 0.1), (0.2, 0.1), (-0.5, 0.6), (0.9, -0.3)])
    assert skip_decisions(ob, 0, 1) == (True, True, True)
    return Case("skip_duplicates", 2, ob, bundle((-1.5, -0.5), (1.5, 0.5), 20, [0.6, -0.6, 0.0]))


def grid_cells(nx, ny, x0, y0, res=0.05):
    """cell centres of a costmap grid (origin (x0, y0), resolution res) listed row-major, as a costmap converts them"""
    return [(x0 + (i + 0.5) * res, y0 + (j + 0.5) * res) for j in range(ny) for i in range(nx)]


def _skip_grid():
    """an 8 x 8 block of 0.05 m cells straddling the origin: every row / column neighbour pair lies at the threshold.
    On cell centres computed as a costmap does (origin + (i + 0.5) res) the neighbour differences come out exact and the
    rounded and exact decisions coincide - here and on 20000 random origins tried when this case was written - so the
    grid holds the kernels to the threshold itself, while the searched pairs above are the ones where rounding decides."""
    ob = obstacles(grid_cells(8, 8, -0.2, -0.2))
    assert len(near_pairs(ob)) == 2 * 8 * 7 and not disagreements(ob)
    return Case("skip_grid_origin", 2, ob, bundle((-1.5, -0.6), (1.5, 0.7), 24, [0.9, -0.9]))


def _range_scene(order):
    """target T, far obstacles about 10 m away and near duplicates 0.06 m from T. The count of near ones is chosen so
    that the long double A_T is O(1); order 'far_first' / 'near_first' lists them after T in that order, 'beyond' has
    only the near ones (A_T and the signature past 1e308)"""
    T = (0.2, 0.1)
    far = [(6.0 + 0.25 * (i % 18), 7.0 + 0.25 * (i // 18)) for i in range(330)]
    P = (0.26, 0.1)
    p = abi.default_params()
    rec0 = bent((-2.0, -0.8), (2.0, 1.0), 30, 0.0)

    def scene(nn, with_far=True):
        rows = [T] + ((far + [P] * nn) if order == "far_first" else ([P] * nn + far) if with_far else [P] * nn)
        return obstacles(rows)
    if order == "beyond":
        nn = 265
        ob = scene(nn, with_far=False)
        logA, _, _ = ld_terms(p, rec0, ob)
        assert logA[0] / math.log(10) > 310
        return ob
    best = min(range(220, 330, 1), key=lambda nn: abs(ld_terms(p, rec0, scene(nn))[0][0]))
    ob = scene(best)
    logA, _, _ = ld_terms(p, rec0, ob)
    assert abs(logA[0]) < math.log(10)                       # long double A_T within [0.1, 10]
    pp = fp64_partial_products(p, rec0, ob, 0)
    if order == "far_first":
        assert pp[-1] == 0 and np.any(pp == 0)              # fp64 partial product underflows to 0 and stays there
    else:
        assert not np.isfinite(pp[-1]) or pp.max() == math.inf   # ... overflows to inf (or NaN)
    return ob


def _range_cases():
    cases = []
    for order in ("far_first", "near_first"):
        ob = _range_scene(order)
        cases.append(Case(f"range_{order}", 2, ob, [bent((-2.0, -0.8), (2.0, 1.0), 30, b) for b in (0.0, 0.5, -0.5)]))
    ob = _range_scene("beyond")
    bands = [bent((-2.0, -0.8), (2.0, 1.0), 30, b) for b in (0.0, 0.5)]
    p = abi.default_params()
    for rec in bands:                                       # the signature itself is past the double range
        _, A, L = ld_terms(p, rec, ob)
        H = (A[None, :] * L.astype(np.clongdouble)).sum()
        assert abs(H) > LD(1e308) * 1000 and np.isfinite(H)
    cases.append(Case("range_beyond", 2, ob, bands, beyond_range=True))
    return cases


def _blob_1024():
    """M = 1024: a 64 x 16 block of 0.05 m costmap cells straddling the origin, row-major (every A_l inside the fp64
    range, spread over some 1000 binary orders of magnitude)"""
    ob = obstacles(grid_cells(64, 16, -1.6, -0.4))
    assert len(ob) == 1024
    p = abi.default_params()
    bands = [bent((-4.0, -2.0), (4.0, 2.5), 40, b) for b in (1.5, -1.5)]
    for rec in bands:
        logA, _, _ = ld_terms(p, rec, ob)
        assert np.all(np.abs(logA) < 1000 * math.log(2)) and logA.max() - logA.min() > 900 * math.log(2)
    return Case("blob_1024", 2, ob, bands)


def _angles():
    cases = []
    # branch cut: segments pass behind obstacle 0 (x < 0 of it), atan2 jumps by ~2 pi and the +-2 pi proposal wins
    ob = obstacles([(0.0, 0.0), (1.3, 0.9), (-0.2, 1.5)])
    rec = band([(0.5, 1.0), (-0.4, 0.7), (-0.8, 0.15), (-0.8, -0.15), (-0.4, -0.7), (0.5, -1.0), (1.5, -1.2)])
    ad = arg_diffs(rec, ob)
    assert np.any(np.abs(ad) > np.pi + 0.1)
    cases.append(Case("angle_branch_cut", 2, ob, [rec, band(rec[::-1, :2]), bent((-1.5, -0.5), (1.5, 0.5), 16, 0.9)]))
    # a segment through obstacle 0's centre: arg diff = -pi exactly, the +2 pi proposal ties at |pi| and the first
    # proposal is kept
    ob = obstacles([(0.5, 0.0), (0.0, 0.8)])
    rec = band([(-1.0, 0.0), (0.0, 0.0), (1.0, 0.0), (2.0, 0.0)])
    ad = arg_diffs(rec, ob)
    assert ad[1, 0] == -np.pi and np.pi == -np.pi + 2 * np.pi
    cases.append(Case("angle_through_centre", 2, ob, [rec, band(rec[::-1, :2])]))
    # a pose exactly on obstacle 0: d1 or d2 == 0, the term is skipped
    ob = obstacles([(0.25, 0.5), (-0.6, -0.2), (1.0, 1.0)])
    rec = band([(-1.0, 0.0), (-0.25, 0.25), (0.25, 0.5), (0.75, 0.75), (1.5, 0.5)])
    z = rec[:, 0] + 1j * rec[:, 1]
    assert np.any(z == complex(ob["x"][0], ob["y"][0]))
    cases.append(Case("pose_on_obstacle", 2, ob, [rec, band(rec[::-1, :2])]))
    # |end - start| exactly 3.0 (map rectangle from the normal) and the double below (the fixed 3 m rectangle); along y,
    # where the two rectangles differ (along +x they coincide)
    for name, start, end in (("rect_exactly_3", (0.0, 0.0), (0.0, 3.0)),
                             ("rect_below_3", (0.0, 0.0), (0.0, float(np.nextafter(3.0, 0)))),
                             ("rect_exactly_3_offset", (1.0, 2.0), (1.0, 5.0))):
        ob = obstacles([(start[0] + 0.3, start[1] + 1.1), (start[0] - 0.4, start[1] + 2.0), (start[0] - 0.6, start[1] + 0.7)])
        bands = bundle(start, end, 12, [0.6, -0.6, 0.0])
        d = np.hypot(LD(end[0]) - LD(start[0]), LD(end[1]) - LD(start[1]))
        assert (d == 3) if "exactly" in name else (d < 3)
        assert float(np.hypot(end[0] - start[0], end[1] - start[1])) == float(d)
        cases.append(Case(name, 2, ob, bands))
    # n = 1 and 2, start == end (a closed loop around obstacle 0)
    ob = obstacles([(0.0, 0.0), (1.2, 0.4), (-0.7, 0.9)])
    loop = band([(0.5 * math.cos(t), 0.5 * math.sin(t)) for t in np.linspace(0, 2 * np.pi, 17)])
    loop[-1, :2] = loop[0, :2]
    cases.append(Case("short_and_closed", 2, ob, [band([(0.3, 0.2)]), band([(-1.0, -0.3), (1.0, 0.4)]), loop]))
    # M = 0 (the signature is 0) and M = 1
    cases.append(Case("m0", 2, obstacles(np.zeros((0, 2))), bundle((-1.0, 0.0), (1.0, 0.0), 8, [0.4, -0.4])))
    cases.append(Case("m1", 2, obstacles([(0.1, 0.05)]), bundle((-1.0, 0.0), (1.0, 0.0), 8, [0.4, -0.4])))
    return cases


# ------------------------------------------------------------------------------------------------ 3-D cases
def _xyt():
    from oracle import teb_oracle_np as npo
    cases = []
    ob = obstacles([(0.0, 0.0), (1.0, 0.6), (-0.8, -0.5), (0.4, -1.2)], v=[(0, 0), (-0.2, 0.05), (0.15, 0.1), (0, 0)])
    bands = bundle((-2.0, -0.4), (2.0, 0.6), 30, [0.8, -0.8, 0.2])
    for use_dt in (1, 0):
        cases.append(Case(f"xyt_static_moving_dt{use_dt}", 3, ob, bands, use_dt=bool(use_dt)))
    # coincident poses (same x, y, dt = 1e-16; the reference's band refuses dt <= 0): the direction is below 1e-15 with
    # and without the time differences - the skip of h_signature.h:328
    rec = bent((-2.0, -0.4), (2.0, 0.6), 20, 0.7)
    rec = np.insert(rec, 7, rec[7], axis=0)
    rec[7, 3] = 1e-16
    assert np.array_equal(rec[7, :2], rec[8, :2]) and 0 < rec[7, 3] < 1e-15
    for use_dt in (1, 0):
        cases.append(Case(f"xyt_coincident_dt{use_dt}", 3, ob, [rec, bands[1]], use_dt=bool(use_dt)))
    # a band looping twice around obstacle 0: |H| >= 1 (isReasonable false)
    t = np.linspace(0, 4 * np.pi, 60)
    helix = band(np.stack([0.6 * np.cos(t), 0.6 * np.sin(t)], 1), dt=0.2)
    p = abi.default_params()
    p.include_dynamic_obstacles = 1
    assert abs(npo.h_signature_3d(p, helix, ob, True)[0]) >= 1.0
    cases.append(Case("xyt_loop", 3, ob, [helix, bands[0]]))
    # obstacle 0's world line through an interior pose: NaN
    rec = bent((-2.0, 0.0), (2.0, 0.0), 21, 0.0)
    assert rec[10, 0] == 0.0 and rec[10, 1] == 0.0
    with np.errstate(all="ignore"):
        assert np.isnan(npo.h_signature_3d(p, rec, ob, True)[0])
    cases.append(Case("xyt_world_line_through_pose", 3, ob, [rec, bands[2]]))
    cases.append(Case("xyt_m0", 3, obstacles(np.zeros((0, 2))), [bands[0]]))
    return cases


def cases_2d():
    out = [_skip_exact()] + _skip_rounded() + [_skip_duplicates(), _skip_grid()] + _range_cases() + [_blob_1024()] + _angles()
    for c in out:
        assert_skip_margin(c.obst)
        for rec in c.bands:
            if len(c.obst):
                assert_no_near_tie(rec, c.obst)
    return out


def cases_3d():
    return _xyt()


_ALL = None


def all_cases():
    global _ALL
    if _ALL is None:
        _ALL = cases_2d() + cases_3d()
    return _ALL


def batch(cases, n_cap=None, M_cap=None, reverse=False):
    """one HostBatch holding every band of the cases, one scene per case. Returns (hb, [(case, band index, row)])"""
    cs = list(cases)[::-1] if reverse else list(cases)
    rows = [(c, i) for c in cs for i in range(len(c.bands))]
    if reverse:
        rows = rows[::-1]
    n_cap = max(3, max(len(c.bands[i]) for c, i in rows)) if n_cap is None else n_cap
    M_cap = max(len(c.obst) for c in cs) if M_cap is None else M_cap
    poses = np.zeros((len(rows), n_cap, 4))
    ns = np.zeros(len(rows), np.int32)
    sid = np.zeros(len(rows), np.int32)
    obst = np.zeros((len(cs), M_cap), abi.OBST_DTYPE)
    cnt = np.zeros(len(cs), np.int32)
    for s, c in enumerate(cs):
        obst[s, :len(c.obst)] = c.obst
        cnt[s] = len(c.obst)
    where = []
    for r, (c, i) in enumerate(rows):
        rec = c.bands[i]
        poses[r, :len(rec)] = rec
        ns[r] = len(rec)
        sid[r] = cs.index(c)
        where.append((c, i, r))
    return abi.HostBatch(poses, ns, obst, cnt, scene_id=sid), where


# ------------------------------------------------------------------------------------------------ class rules
def is_valid(val):
    """isValid: every value finite (both parts of the 2-D one)"""
    return bool(np.all(np.isfinite(np.atleast_1d(np.asarray(val)))))


def is_reasonable(val, dim):
    return True if dim == 2 else not bool(np.any(np.asarray(val) > 1.0))


def is_equal(x, y, dim, thr):
    """HSignature::isEqual (h_signature.h:195-206) / HSignature3d::isEqual (:359-383)"""
    if dim == 2:
        return abs(x.real - y.real) <= thr and abs(x.imag - y.imag) <= thr
    x, y = np.asarray(x), np.asarray(y)
    for a, b in zip(x, y):
        if abs(a) < thr or abs(b) < thr:
            continue
        if np.sign(a) != np.sign(b):
            return False
    return True


def partition(vals, dim, thr):
    return [[is_equal(a, b, dim, thr) for b in vals] for a in vals]
