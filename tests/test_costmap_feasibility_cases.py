"""The costmap feasibility restatement (tests/costmap_feasibility_cases.py) pinned on hand-computed cases: the
LineIterator walk in every octant and at its ties, worldToMap at the map's edges, pointCost / footprintCost's codes
and their order along the outline, and the verdict loop."""
import math

import numpy as np
import pytest

from tests import costmap_feasibility_cases as cf
from tests import feasibility_cases as fc

# ---- LineIterator


@pytest.mark.parametrize("end, want", [
    # the eight octants from (0, 0), each walked by hand with num starting at den // 2
    ((5, 2), [(0, 0), (1, 0), (2, 1), (3, 1), (4, 2), (5, 2)]),          # x major, +x +y
    ((2, 5), [(0, 0), (0, 1), (1, 2), (1, 3), (2, 4), (2, 5)]),          # y major, +x +y
    ((-2, 5), [(0, 0), (0, 1), (-1, 2), (-1, 3), (-2, 4), (-2, 5)]),     # y major, -x +y
    ((-5, 2), [(0, 0), (-1, 0), (-2, 1), (-3, 1), (-4, 2), (-5, 2)]),    # x major, -x +y
    ((-5, -2), [(0, 0), (-1, 0), (-2, -1), (-3, -1), (-4, -2), (-5, -2)]),
    ((-2, -5), [(0, 0), (0, -1), (-1, -2), (-1, -3), (-2, -4), (-2, -5)]),
    ((2, -5), [(0, 0), (0, -1), (1, -2), (1, -3), (2, -4), (2, -5)]),
    ((5, -2), [(0, 0), (1, 0), (2, -1), (3, -1), (4, -2), (5, -2)]),
    # ties: num reaches den exactly (den = 4, num = 2, numadd = 2: the minor step at k = 1, 3)
    ((4, 2), [(0, 0), (1, 1), (2, 1), (3, 2), (4, 2)]),
    ((-4, -2), [(0, 0), (-1, -1), (-2, -1), (-3, -2), (-4, -2)]),
    # odd den: num = 1 of 3
    ((3, 1), [(0, 0), (1, 0), (2, 1), (3, 1)]),
    # diagonal (dx == dy picks x major), axis-aligned, zero-length
    ((3, 3), [(0, 0), (1, 1), (2, 2), (3, 3)]),
    ((-3, 3), [(0, 0), (-1, 1), (-2, 2), (-3, 3)]),
    ((0, 3), [(0, 0), (0, 1), (0, 2), (0, 3)]),
    ((-3, 0), [(0, 0), (-1, 0), (-2, 0), (-3, 0)]),
    ((0, 0), [(0, 0)]),
])
def test_line_iterator_by_hand(end, want):
    got = cf.line_cells(0, 0, *end)
    assert got == want
    assert [cf.line_cell(0, 0, *end, k) for k in range(len(want))] == want


def test_closed_form_cells_equal_the_walk():
    rng = np.random.default_rng(3)
    for _ in range(3000):
        x0, y0, x1, y1 = (int(v) for v in rng.integers(-40, 40, 4))
        walk = cf.line_cells(x0, y0, x1, y1)
        assert walk[0] == (x0, y0) and walk[-1] == (x1, y1)
        assert [cf.line_cell(x0, y0, x1, y1, k) for k in range(len(walk))] == walk


# ---- worldToMap


def test_world_to_map_edges():
    m = cf.Raster.filled(8, 4, ox=1.0, oy=-2.0, r=0.125)
    assert cf.world_to_map(m, 1.0, -2.0) == (0, 0)                                  # wx == ox: cell 0
    assert cf.world_to_map(m, math.nextafter(1.0, 0.0), -1.5) is None              # just below ox
    assert cf.world_to_map(m, 1.5, math.nextafter(-2.0, -3.0)) is None
    assert cf.world_to_map(m, 1.0 + 8 * 0.125, -1.5) is None                        # ox + sx r: off
    assert cf.world_to_map(m, math.nextafter(2.0, 0.0), math.nextafter(-1.5, -2.0)) == (7, 3)
    assert cf.world_to_map(m, 1.125, -1.875) == (1, 1)                              # on a cell edge: the upper cell
    assert cf.world_to_map(m, 1e300, -1.5) is None                                  # quotient past the int range
    assert cf.world_to_map(m, 1.0 + 2.0 ** 31 * 0.125, -1.5) is None


# ---- footprintCost and its codes


@pytest.mark.parametrize("case", cf.hand_cases(), ids=lambda c: c[0])
def test_footprint_cost_hand_cases(case):
    name, m, (x, y, th), fp, want = case
    got = cf.footprint_cost(m, x, y, th, fp)
    if want is None:          # the 16-gon turned by 0.7 rad: a cost from the ring of 3s, the lethal cell off its outline
        assert got == 3
        cells = set()
        v = cf.transform(x, y, th, fp)
        for i in range(len(v)):
            a, b = cf.world_to_map(m, *v[i]), cf.world_to_map(m, *v[(i + 1) % len(v)])
            cells.update(cf.line_cells(a[0], a[1], b[0], b[1]))
        assert (10, 8) not in cells
    else:
        assert got == want, name


def test_outline_walk_order_by_hand():
    """the square of hand_cases at (1.5, 1.5): vertices (1, 1), (2, 1), (2, 2), (1, 2) fall on cells (4, 4), (8, 4),
    (8, 8), (4, 8); edge 0 walks (4, 4) .. (8, 4), edge 3 (the closing one) walks (4, 8) .. (4, 4)"""
    m = cf.Raster.filled(12, 12)
    sq = [(-0.5, -0.5), (0.5, -0.5), (0.5, 0.5), (-0.5, 0.5)]
    v = cf.transform(1.5, 1.5, 0.0, sq)
    assert [cf.world_to_map(m, *p) for p in v] == [(4, 4), (8, 4), (8, 8), (4, 8)]
    assert cf.line_cells(4, 8, 4, 4) == [(4, 8), (4, 7), (4, 6), (4, 5), (4, 4)]


def test_point_cost_codes():
    m = cf.Raster.filled(4, 1, cells=[(0, 0, 253), (1, 0, 254), (2, 0, 255), (3, 0, 252)])
    assert [cf.point_cost(m, i, 0) for i in range(4)] == [253, -1, -2, 252]
    assert cf.line_cost(m, 3, 0, 0, 0) == -2            # walked 3, 2: the 255 first
    assert cf.line_cost(m, 0, 1, 0, 0) == -1
    assert cf.line_cost(m, 3, 3, 0, 0) == 252
    assert cf.line_cost(m, 0, 0, 0, 0) == 253


# ---- the verdict over the reference's queries


def test_verdict_first_lethal_query_decides_and_minus_two_three_are_free():
    m = cf.Raster.filled(16, 4, r=0.25, cells=[(3, 1, 255), (9, 1, 254), (12, 1, 254)])
    rec = fc._line(5, dx=0.75, x0=0.125, y0=0.375)               # cells x = 0, 3, 6, 9, 12 on row 1
    q = fc.ref_queries(rec, 5, 1.0)
    assert len(q) == 5
    f, k, qc = cf.verdict(m, q, [])
    assert (f, k) == (0, 4) and qc == [0, -2, 0, -1]
    f, k, qc = cf.verdict(m, q, [], max_queries=3)
    assert (f, k) == (-1, 5) and qc == [0, -2, 0]
    f, k, qc = cf.verdict(m, q[:3], [])
    assert (f, k) == (1, 3)
    off = fc._line(3, dx=10.0)                                    # poses 1 and 2 off the map: free
    f, k, qc = cf.verdict(m, fc.ref_queries(off, 3, 100.0), [])
    assert (f, k, qc) == (1, 3, [0, -3, -3])


def test_band_verdict_nonfinite_pose_gives_minus_one_without_query():
    m = cf.Raster.filled(8, 8)
    rec = fc._line(4, dx=0.1)
    rec[2, 1] = np.nan
    assert cf.band_verdict(m, rec, 4, [], 0.2) == (-1, 0, [])
    assert cf.band_verdict(m, rec, 4, [], 0.2, look_ahead_idx=1)[0] == 1


def test_random_fleet_reaches_every_code():
    ras, rec, n, sid, fp = cf.random_fleet(3, 120, 120, 0.05, seed=1, F=4)
    codes = set()
    for b in range(len(n)):
        m = cf.raster_of(ras, sid[b])
        for x, y, th in fc.ref_queries(rec[b], n[b], 0.1):
            codes.add(cf.footprint_cost(m, x, y, th, fp))
    assert {-1, -2, -3} & codes and -1 in codes and max(codes) > 0
