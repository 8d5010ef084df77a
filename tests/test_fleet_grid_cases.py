"""The 3 x 3 claim of the fleet grid, on the CPU restatement of its cells (tests/fleet_grid_cases.py): two binned points
whose distance passes the step's rule, as rounded, lie in cells whose coordinates differ by at most 1 on each axis. So a
robot that scans the buckets of its 3 x 3 cells and the far list meets every neighbour, and each candidate once."""
import math

import numpy as np
import pytest

from tests import fleet_cases as fc
from tests import fleet_grid_cases as gc

UP, DOWN = math.inf, -math.inf
BOUND = gc.FLEET_CELL_BOUND


def assert_claim(xr, yr, xq, yq, rng):
    """every pair in range whose two points are binned: cell coordinates within 1 on each axis. Returns the pairs in
    range."""
    xr, yr, xq, yq = (np.atleast_1d(np.asarray(v, np.float64)) for v in (xr, yr, xq, yq))
    h = gc.cell_side(rng)
    fin2 = bool(gc.range2(rng) < np.inf)
    ok = gc.in_range(xr, yr, xq, yq, rng)
    kr, cxr, cyr = gc.cells(xr, yr, h, fin2)
    kq, cxq, cyq = gc.cells(xq, yq, h, fin2)
    both = ok & (kr == gc.BINNED) & (kq == gc.BINNED)
    bad = both & ((np.abs(cxr - cxq) > 1) | (np.abs(cyr - cyq) > 1))
    assert not bad.any(), (rng, xr[bad][:3], xq[bad][:3], yr[bad][:3], yq[bad][:3])
    # a point never in range is never in range of anything
    never = (kr == gc.NEVER) | (kq == gc.NEVER)
    assert not (ok & never).any()
    return ok


@pytest.mark.parametrize("rng", [3.0, 0.7, 1e-3, 123.456, 1e6, 2.0 ** -400, 1e150])
def test_pairs_at_exactly_range_across_a_cell_edge(rng):
    h = gc.cell_side(rng)
    xs = []
    for k in (-1000003, -7, -1, 0, 1, 2, 5, 999983):
        e = k * h
        for x in (e, np.nextafter(e, UP), np.nextafter(e, DOWN)):
            xs.append(x)
    xs = np.array(xs)
    # the partner at +- range along x, along y, and on the diagonal, with the sum rounded as it falls
    for sgn in (1.0, -1.0):
        ok = assert_claim(xs, 0.0, xs + sgn * rng, 0.0, rng)
        assert ok.any()
        assert_claim(0.0, xs, 0.0, xs + sgn * rng, rng)
        d = rng / math.sqrt(2.0)
        assert_claim(xs, xs, xs + sgn * d, xs + sgn * d, rng)
        # one ulp beyond range either way
        assert_claim(xs, 0.0, np.nextafter(xs + sgn * rng, sgn * UP), 0.0, rng)
        assert_claim(xs, 0.0, np.nextafter(xs + sgn * rng, -sgn * UP), 0.0, rng)


@pytest.mark.parametrize("rng", [3.0, 1e-9, 2.0 ** -500, 7e-300])
def test_coordinates_one_ulp_either_side_of_a_cell_edge(rng):
    h = gc.cell_side(rng)
    for k in (-(2 ** 23), -3, -1, 1, 3, 2 ** 23 - 2):
        e = np.float64(k) * h
        lo, hi = np.nextafter(e, DOWN), np.nextafter(e, UP)
        pts = np.array([np.nextafter(lo, DOWN), lo, e, hi, np.nextafter(hi, UP)])
        for a in pts:
            assert_claim(a, 0.0, pts, 0.0, rng)
            assert_claim(a - rng, 0.0, pts, 0.0, rng)
            assert_claim(a + rng, 0.0, pts, 0.0, rng)


@pytest.mark.parametrize("rng", [3.0, 1e-6])
def test_negative_coordinates_and_the_far_bound(rng):
    h = gc.cell_side(rng)
    fin2 = True
    for s in (1.0, -1.0):
        edge = s * BOUND * h
        for x in (np.nextafter(edge, 0.0), edge, np.nextafter(edge, s * UP)):
            kind, _, _ = gc.cells(x, 0.0, h, fin2)
            fx = x / h
            assert kind[0] == (gc.BINNED if abs(fx) < BOUND else gc.FAR)
        # pairs straddling the bound: the binned one keeps the claim against its binned partners
        xs = np.array([np.nextafter(edge, 0.0) - k * rng / 3 for k in range(6)] + [edge, np.nextafter(edge, s * UP)])
        for a in xs:
            assert_claim(a, -17.0, xs, -17.0 + rng / 2, rng)
    kind, cx, cy = gc.cells(-0.0, -1e-300, h, fin2)
    assert kind[0] == gc.BINNED and cx[0] == 0 and cy[0] == -1


def test_range_zero_subnormal_and_underflowing_squares():
    tiny = 5e-324
    for rng in (0.0, tiny, 2.0 ** -1030, 1e-200, 2.0 ** -537, 2.0 ** -536):
        h = gc.cell_side(rng)
        assert h == max(rng * gc.FLEET_H_MARGIN, gc.FLEET_H_FLOOR)
        base = np.array([0.0, 1.0, -1.0, 2.0 ** -500, -(2.0 ** -500), 3.0 * 2.0 ** -500, 1e-300, 123.5])
        for b in base:
            # dx whose square underflows to 0 or to a subnormal: d2 <= range2 holds for range 0 too
            for dx in (tiny, 1e-170, 2.0 ** -537, 2.0 ** -536, 1e-162, -1e-170, 2.0 ** -510):
                xq = b + dx
                ok = assert_claim(b, 0.0, xq, 0.0, rng)
                assert_claim(b, b, xq, b + dx, rng)
                if dx * dx == 0.0 and xq != b and (xq - b) * (xq - b) == 0.0:
                    assert ok[0]


def test_overflowing_range_squared_puts_every_finite_point_in_one_cell():
    for rng in (1e155, 1e300, np.finfo(np.float64).max):
        assert gc.cell_side(rng) == np.inf
        xs = np.array([0.0, -1e308, 1e308, 5e-324, -3.0])
        kind, cx, cy = gc.cells(xs, xs[::-1], np.inf, False)
        assert (kind == gc.BINNED).all() and (cx == 0).all() and (cy == 0).all()
        kind, _, _ = gc.cells(np.array([np.nan, np.inf]), 0.0, np.inf, False)
        assert (kind == gc.FAR).all()
    kind, _, _ = gc.cells(np.array([np.nan, np.inf, -np.inf, 0.0]), np.array([0.0, 0.0, 0.0, np.nan]), 3.0, True)
    assert (kind == gc.NEVER).all()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_millions_of_random_pairs_near_the_boundary(seed):
    rng_ = np.random.default_rng(seed)
    n = 1_000_000
    for scale in (1.0, 1e-12, 1e9, 2.0 ** -490):
        rng = float(scale * rng_.uniform(0.5, 5.0))
        h = gc.cell_side(rng)
        # robots near cell edges, partners at range * (1 +- a few ulps) in a random direction
        k = rng_.integers(-(2 ** 22), 2 ** 22, (n, 2)).astype(np.float64)
        xr = k[:, 0] * h + rng_.uniform(-1e-3, 1e-3, n) * h
        yr = k[:, 1] * h + rng_.uniform(-1e-3, 1e-3, n) * h
        th = rng_.uniform(0, 2 * np.pi, n)
        d = rng * (1.0 + rng_.integers(-8, 9, n) * 2.0 ** -52)
        xq, yq = xr + d * np.cos(th), yr + d * np.sin(th)
        axis = rng_.random(n) < 0.25
        xq[axis], yq[axis] = xr[axis] + d[axis], yr[axis]
        ok = assert_claim(xr, yr, xq, yq, rng)
        assert 0.05 < ok.mean() < 0.95


def test_bucket_function_and_the_met_candidates():
    w = np.array([0, 0, 1, -1, 2 ** 31 - 1, -(2 ** 31)])
    b = gc.bucket(w, np.array([0, 1, 0, 0, 5, -5]), np.array([0, 0, 0, 7, -(2 ** 24), 2 ** 24 - 1]), 1023)
    assert b.dtype == np.uint32 and (b <= 1023).all()
    assert (gc.bucket(w, w, w, 0) == 0).all()
    assert gc.buckets_of(1) == 2 and gc.buckets_of(5) == 16 and gc.buckets_of(8) == 16
    # every neighbour is met, and met once, in random fleets with several worlds, padding, far and non-finite points
    r_ = np.random.default_rng(7)
    for trial in range(6):
        N = int(r_.integers(2, 300))
        xy = r_.uniform(-20, 20, (N, 2))
        if trial % 2:
            xy[r_.integers(0, N, 3)] = xy[r_.integers(0, N, 3)]      # coincident
        xy[r_.integers(0, N, 2), 0] = 1e30                             # far from the grid
        xy[r_.integers(0, N, 1), 1] = np.nan
        world = r_.integers(-1, 2, N)
        live = r_.random(N) < 0.9
        for rng in (0.0, 0.5, 3.0, 40.0):
            for one in (False, True):
                for r in range(N):
                    m = gc.met(xy, world, live, r, rng, one_bucket=one)
                    assert len(m) == len(set(m)), (trial, rng, r)
                    idx, _ = fc.neighbours(np.column_stack([xy, np.zeros(N)]), r, rng, world)
                    idx = [q for q in idx if live[q]]
                    assert set(idx) <= set(m), (trial, rng, r)
