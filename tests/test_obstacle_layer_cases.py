"""tests/obstacle_layer_cases.py pinned on hand-computed cases: rays in every octant and on both axes, Bresenham's
error_b at even and odd abs_da, max_length truncation and a zero-length ray, the four clamps with the - .001 quirk, a
sensor off the map, the obstacle range and height bounds, a mark over a cleared cell, shifts over several cycles, the
combination methods over static 0 / 254 / 255 cells, and footprint clearing of a square, a rotated rectangle, a
triangle, a diamond, a footprint partly off the map and a 2-point footprint; then the numpy form held bit equal to the
literal one, and convexFillCells' column spans to its literal form, on random inputs.

In the grids below row y = 0 comes first; '.' is FREE_SPACE, '#' LETHAL_OBSTACLE, '?' NO_INFORMATION."""
import math

import numpy as np
import pytest

from tests import costmap_window_cases as cw
from tests import obstacle_layer_cases as ol

SYM = {".": ol.FREE_SPACE, "#": ol.LETHAL_OBSTACLE, "?": ol.NO_INFORMATION}


def rows(layer, sx, sy):
    inv = {v: k for k, v in SYM.items()}
    return [("".join(inv.get(int(v), "x") for v in layer[j * sx:(j + 1) * sx])) for j in range(sy)]


def grid_of(text_rows):
    return [SYM[c] for row in text_rows for c in row]


def run(points, sensor, robot=(1.0, 1.0, 0.0), sx=8, sy=8, r=0.25, layer=None, footprint=(), **kw):
    """one standalone call on a layer at origin (0, 0) that the robot does not move; returns (layer, flags, result)"""
    p = dict(ol.PARAMS, mode=ol.STANDALONE, obstacle_range=10.0, raytrace_range=10.0)
    p.update(kw)
    cap = sx * sy
    layer = [ol.NO_INFORMATION] * cap if layer is None else layer
    pts = [tuple(float(np.float32(v)) for v in q) for q in points]
    res = ol.obstacle_layer(p, pts, sensor, robot, (sx, sy), cap, layer, (0.0, 0.0), [0] * cap, (0.0, 0.0, r), footprint)
    assert res[4] == ol.OK and res[1] == (0.0, 0.0)
    return res[0], res[5], res


def centre(i, j, r=0.25, z=0.0):
    return ((i + 0.5) * r, (j + 0.5) * r, z)


def test_rays_in_every_octant_and_on_both_axes():
    ends = [(7, 5), (5, 7), (3, 7), (1, 5), (1, 3), (3, 1), (5, 1), (7, 3), (7, 4), (1, 4), (4, 7), (4, 1)]
    layer, flags, _ = run([centre(i, j) for i, j in ends], centre(4, 4))
    assert flags == 0
    assert rows(layer, 8, 8) == ["????????",
                                 "???###??",
                                 "???...??",
                                 "?#.?.?.#",
                                 "?#.....#",
                                 "?#.?.?.#",
                                 "???...??",
                                 "???###??"]


def test_bresenham_error_starts_at_half_the_major_delta():
    # (+4, +1): abs_da 4, error_b 2 -> the minor step after the second cell; (+5, +2): abs_da 5, error_b 2
    layer, _, _ = run([centre(4, 1), centre(5, 2)], centre(0, 0))
    assert rows(layer, 8, 8)[:3] == ["..??????",
                                     "??..#???",
                                     "????.#??"]
    assert set(rows(layer, 8, 8)[3:]) == {"????????"}


def test_max_length_truncates_the_ray():
    # cellDistance(0.5) at r 0.25 is 2; hypot(3, 1) = 3.1623, scale 0.632, (unsigned)(0.632 * 3) = 1 step
    layer, _, _ = run([centre(7, 5)], centre(4, 4), raytrace_range=0.5)
    assert rows(layer, 8, 8)[4:6] == ["????..??", "???????#"]
    # 2.1 / 0.3 rounds to 7.000000000000001: ceil gives 8 cells, and the ray along x stops after 8 steps
    assert ol.cell_distance(2.1, 0.3) == 8 and ol.cell_distance(3.0, 0.05) == 60
    layer, _, _ = run([(3.45, 0.45, 0.0)], (0.15, 0.45, 0.0), robot=(1.8, 0.45, 0.0), sx=12, sy=3, r=0.3, raytrace_range=2.1)
    assert rows(layer, 12, 3)[1] == ".........??#"
    # 3.0 / 0.05 is 60 exactly: 60 steps of a 69-cell ray, 61 cells
    layer, _, _ = run([(3.475, 0.025, 0.0)], (0.025, 0.025, 0.0), robot=(1.75, 0.02, 0.0), sx=70, sy=1, r=0.05,
                      raytrace_range=3.0)
    assert rows(layer, 70, 1)[0] == "." * 61 + "?" * 8 + "#"
    # a zero-length ray clears the sensor's own cell, which the mark then takes
    layer, _, _ = run([(1.2, 1.2, 0.0)], centre(4, 4), marking=False)
    assert rows(layer, 8, 8)[4] == "????.???"
    layer, _, _ = run([(1.2, 1.2, 0.0)], centre(4, 4))
    assert rows(layer, 8, 8)[4] == "????#???"


def test_the_four_clamps_and_the_shifted_end():
    # left, below, right and above the map; then (2.875, 1.875): t = 0.875 / 1.75 = 0.5 puts y at 1.5, the edge of
    # row 6, where the moved x (map_end - .001) would have put it in row 5
    pts = [(-1.125, 1.125, 0.0), (1.125, -1.0, 0.0), (3.0, 1.125, 0.0), (1.125, 3.0, 0.0), (2.875, 1.875, 0.0)]
    layer, flags, _ = run(pts, centre(4, 4))
    assert flags == 0
    assert ol.clamp_to_map(2.875, 1.875, 1.125, 1.125, 0.0, 0.0, 2.0, 2.0) == (2.0 - .001, 1.5)
    assert rows(layer, 8, 8) == ["????.???",
                                 "????.???",
                                 "????.???",
                                 "????.???",
                                 "........",
                                 "????...?",
                                 "????.??.",
                                 "????.???"]


def test_sensor_off_the_map_still_marks():
    layer, flags, _ = run([centre(2, 2), centre(5, 5)], (-1.0, -1.0, 0.0), obstacle_range=2.5)
    assert flags == ol.SENSOR_OFF_MAP
    # (2, 2) lies at 2.30 m from the sensor, (5, 5) at 3.36 m
    assert rows(layer, 8, 8)[2] == "??#?????" and rows(layer, 8, 8)[5] == "????????"


def test_obstacle_range_bound_is_excluded_and_height_bounds_are_included():
    layer, _, _ = run([(1.625, 1.125, 0.0), (1.375, 1.125, 0.0)], centre(4, 4), obstacle_range=0.5, clearing=False)
    assert rows(layer, 8, 8)[4] == "?????#??" and layer.count(ol.LETHAL_OBSTACLE) == 1
    pts = [(0.125, 1.125, 0.25), (1.125, 0.125, 0.75), (1.875, 1.125, 0.2499), (1.125, 1.875, 0.7501)]
    layer, _, _ = run(pts, centre(4, 4, z=0.5), min_obstacle_height=0.25, max_obstacle_height=0.75,
                      layer_max_obstacle_height=0.5)
    assert rows(layer, 8, 8) == ["????.???", "????.???", "????.???", "????.???", "#....???",
                                 "????????", "????????", "????????"]


def test_a_mark_wins_over_a_cell_another_ray_cleared():
    layer, _, _ = run([centre(7, 4), centre(6, 4)], centre(4, 4))
    assert rows(layer, 8, 8)[4] == "????..##"


def test_shifts_over_several_cycles():
    p = dict(ol.PARAMS, mode=ol.STANDALONE, clearing=False, marking=False)
    layer = [10 * j + i for j in range(3) for i in range(4)]
    lo = (0.0, 0.0)
    want = [((3.0, 2.0), (1.0, 0.0), [1, 2, 3, 255, 11, 12, 13, 255, 21, 22, 23, 255]),
            ((1.0, 0.0), (0.0, -1.0), [255, 255, 255, 255, 255, 1, 2, 3, 255, 11, 12, 13]),
            ((1.0, 0.0), (0.0, -1.0), [255, 255, 255, 255, 255, 1, 2, 3, 255, 11, 12, 13]),
            ((20.0, 20.0), (18.0, 18.0), [255] * 12)]
    for (rx, ry), org, cells in want:
        layer, lo, master, mo, st, _ = ol.obstacle_layer(p, [], (0, 0, 0), (rx, ry, 0.0), (4, 3), 12, layer, lo,
                                                         [0] * 12, (9.0, 9.0, 1.0))
        assert st == ol.OK and lo == org and mo == (org[0], org[1], 1.0)
        assert layer == cells and master == cells
    # without track_unknown_space the cells shifted in are FREE_SPACE
    layer, lo, *_ = ol.obstacle_layer(dict(p, track_unknown_space=False), [], (0, 0, 0), (3.0, 2.0, 0.0), (4, 3), 12,
                                      [254] * 12, (0.0, 0.0), [0] * 12, (0.0, 0.0, 1.0))
    assert layer == [254, 254, 254, 0] * 3


def test_combination_methods_over_static_cells():
    M, L = [0, 254, 255, 100], [0, 254, 255, 50]          # master by column, layer by row
    master = M * 4
    layer = [L[j] for j in range(4) for _ in range(4)]
    want = {1: [0, 254, 0, 100, 254, 254, 254, 254, 0, 254, 255, 100, 50, 254, 50, 100],
            0: [0, 0, 0, 0, 254, 254, 254, 254, 0, 254, 255, 100, 50, 50, 50, 50],
            2: master}
    for method, cells in want.items():
        p = dict(ol.PARAMS, mode=ol.COMBINE, combination_method=method, clearing=False, marking=False)
        out = ol.obstacle_layer(p, [], (0, 0, 0), (1.75, 1.75, 0.0), (4, 4), 16, layer, (0.0, 0.0), master,
                                (0.0, 0.0, 1.0))
        assert out[4] == ol.OK and out[2] == cells and out[0] == layer
    # a layer without track_unknown_space erases the static unknown cells, shifted-in cells included
    p = dict(ol.PARAMS, mode=ol.COMBINE, track_unknown_space=False, clearing=False, marking=False)
    out = ol.obstacle_layer(p, [], (0, 0, 0), (2.75, 1.75, 0.0), (4, 4), 16, [254] * 16, (0.0, 0.0), [255] * 16,
                            (1.0, 0.0, 1.0))
    assert out[4] == ol.OK and out[2] == [254, 254, 254, 0] * 4
    # the snapped origin differs from the master's: nothing is written
    out = ol.obstacle_layer(p, [], (0, 0, 0), (2.75, 1.75, 0.0), (4, 4), 16, [254] * 16, (0.0, 0.0), [255] * 16,
                            (0.0, 0.0, 1.0))
    assert out[4] == ol.ORIGIN_MISMATCH and out[2] == [255] * 16 and out[0] == [254] * 16 and out[1] == (0.0, 0.0)


FOOTPRINTS = {
    "square": ([(-1.5, -1.5), (1.5, -1.5), (1.5, 1.5), (-1.5, 1.5)], 0.0, (4.0, 4.0),
               ["########", "########", "##....##", "##....##", "##....##", "##....##", "########", "########"]),
    "rotated rectangle": ([(-2, -1), (2, -1), (2, 1), (-2, 1)], math.pi / 6, (4.25, 4.25),
                          ["########", "########", "###.####", "###...##", "##.....#", "###...##", "#####.##", "########"]),
    "triangle": ([(-3, -3), (2, -2), (-1, 2)], 0.0, (4.25, 4.25),
                 ["########", "#...####", "#......#", "##....##", "##...###", "###..###", "###.####", "########"]),
    # the tips x = 2 and x = 6 are one-cell columns: their two outline cells are the same vertex, filled from y to y
    "diamond": ([(0, -3), (2, -1), (0, 1), (-2, -1)], 0.0, (4.25, 4.25),
                ["########", "####.###", "###...##", "##.....#", "###...##", "####.###", "########", "########"]),
}


@pytest.mark.parametrize("name", list(FOOTPRINTS))
def test_footprint_clearing(name):
    fp, yaw, (x, y), want = FOOTPRINTS[name]
    layer, flags, _ = run([], (0, 0, 0), robot=(x, y, yaw), r=1.0, layer=[ol.LETHAL_OBSTACLE] * 64, footprint=fp)
    assert flags == 0 and rows(layer, 8, 8) == want


def test_convex_fill_pairs_stay_in_their_column():
    cells = ol.convex_fill_cells([(4, 1), (6, 3), (4, 5), (2, 3)], 8)
    # 12 outline cells sorted by x, then the fills of columns 3, 4 and 5 (the tips add nothing)
    assert cells[:12] == [(2, 3), (2, 3), (3, 4), (3, 2), (4, 1), (4, 5), (4, 5), (4, 1), (5, 2), (5, 4), (6, 3), (6, 3)]
    assert cells[12:] == [(3, 2), (3, 3), (4, 1), (4, 2), (4, 3), (4, 4), (5, 2), (5, 3)]
    assert ol.column_spans([(4, 1), (6, 3), (4, 5), (2, 3)]) == {2: (3, 3), 3: (2, 4), 4: (1, 5), 5: (2, 4), 6: (3, 3)}


def test_footprint_partly_off_the_map_and_two_point_footprints_clear_nothing():
    fp = [(-1.5, -1.5), (1.5, -1.5), (1.5, 1.5), (-1.5, 1.5)]
    layer, flags, _ = run([], (0, 0, 0), robot=(4.0, 4.0, 0.0), r=1.0, layer=[ol.LETHAL_OBSTACLE] * 64,
                          footprint=[(-4.5, -1.5)] + fp[1:])
    assert flags == ol.FOOTPRINT_OFF_MAP and layer == [ol.LETHAL_OBSTACLE] * 64
    layer, flags, _ = run([], (0, 0, 0), robot=(4.0, 4.0, 0.0), r=1.0, layer=[ol.LETHAL_OBSTACLE] * 64,
                          footprint=fp[:2])
    assert flags == 0 and layer == [ol.LETHAL_OBSTACLE] * 64


def test_bad_robots():
    p = dict(ol.PARAMS, mode=ol.STANDALONE)
    ok = (1.75, 1.75, 0)
    for grid, lo, r, pts, rb, want in (((0, 4), (0.0, 0.0), 1.0, [], ok, ol.BAD_GRID),
                                       ((4, 5), (0.0, 0.0), 1.0, [], ok, ol.BAD_GRID),
                                       ((4, 4), (0.0, 0.0), 0.0, [], ok, ol.BAD_GRID),
                                       ((4, 4), (math.nan, 0.0), 1.0, [], ok, ol.BAD_GRID),
                                       ((4, 4), (0.0, 0.0), math.inf, [], ok, ol.BAD_GRID),
                                       ((4, 4), (0.0, 0.0), 1.0, [], (math.nan, 1.75, 0), ol.BAD_GRID),
                                       ((4, 4), (0.0, 0.0), 1.0, [], (1.75, -math.inf, 0), ol.BAD_GRID),
                                       ((4, 4), (0.0, 0.0), 1.0, [(0, 0, 0)] * 3, ok, ol.BAD_POINTS)):
        out = ol.obstacle_layer(p, pts, (0, 0, 0), rb, grid, 16, [7] * 16, lo, [9] * 16, (5.0, 5.0, r), P_cap=2)
        assert out[4] == want and out[0] == [7] * 16 and out[2] == [255] * 16 and out[3] == (5.0, 5.0, r)


# ---- the numpy form against the literal one, and the column spans against convexFillCells

def random_case(rng, S, sx, sy, P, mode, footprint):
    r = float(rng.choice([0.05, 0.1, 0.25]))
    robot = np.column_stack([rng.uniform(-3, 3, (S, 2)), rng.uniform(-np.pi, np.pi, S)])
    layer_origin = robot[:, :2] - np.array([sx, sy]) * r / 2 + rng.uniform(-3, 3, (S, 2)) * r
    grid = np.tile([sx, sy], (S, 1)).astype(np.int32)
    cap = sx * sy + 5
    if mode == ol.COMBINE:
        org = np.array([[cw.snap(layer_origin[s, 0], robot[s, 0], sx, r), cw.snap(layer_origin[s, 1], robot[s, 1], sy, r), r]
                        for s in range(S)])
        org[::5, 0] += r                                                      # some mismatches
    else:
        org = np.column_stack([rng.uniform(-9, 9, (S, 2)), np.full(S, r)])
    sensor = np.column_stack([robot[:, :2] + rng.normal(0, 0.1, (S, 2)), rng.uniform(0, 0.5, S)])
    sensor[::7, :2] += 50.0                                                   # some sensors off the map
    ang = rng.uniform(-np.pi, np.pi, (S, P))
    dist = rng.uniform(0, max(sx, sy) * r, (S, P))
    pts = np.stack([sensor[:, None, 0] + dist * np.cos(ang), sensor[:, None, 1] + dist * np.sin(ang),
                    rng.uniform(-0.3, 2.3, (S, P))], -1).astype(np.float32)
    pts.reshape(-1, 3)[rng.integers(0, S * P, S * P // 20)] = [np.nan, np.inf, 0.5]
    pts.reshape(-1, 3)[rng.integers(0, S * P, S * P // 20)] = [-np.inf, 0.3, 0.5]
    count = rng.integers(0, P + 1, S)
    layer = rng.choice(np.array([0, 254, 255], np.uint8), (S, cap))
    master = rng.choice(np.array([0, 254, 255, 90], np.uint8), (S, cap))
    return pts, count, sensor, robot, grid, cap, layer, layer_origin, master, org


@pytest.mark.parametrize("mode,method,track,fp", [(ol.COMBINE, 1, True, 4), (ol.COMBINE, 0, False, 3),
                                                  (ol.STANDALONE, 1, True, 6), (ol.STANDALONE, 2, False, 0)])
def test_numpy_form_equals_the_literal_one(mode, method, track, fp):
    rng = np.random.default_rng(11 + mode + 3 * method)
    pts, count, sensor, robot, grid, cap, layer, lo, master, org = random_case(rng, 24, 23, 17, 40, mode, fp)
    angles = np.sort(rng.uniform(0, 2 * np.pi, fp))
    footprint = [(0.3 * math.cos(a), 0.2 * math.sin(a)) for a in angles]
    p = dict(ol.PARAMS, mode=mode, combination_method=method, track_unknown_space=track, raytrace_range=1.1,
             obstacle_range=0.9, min_obstacle_height=0.0, max_obstacle_height=2.0, layer_max_obstacle_height=1.5)
    got = ol.obstacle_layer_np(p, pts, count, sensor, robot, grid, cap, layer, lo, master, org, footprint)
    sts, flags = [], []
    for s in range(24):
        want = ol.obstacle_layer(p, [tuple(map(float, q)) for q in pts[s, :count[s]]], sensor[s], robot[s], grid[s], cap,
                                 layer[s].tolist(), lo[s], master[s].tolist(), org[s], footprint, P_cap=40)
        assert got[0][s].tolist() == want[0] and got[2][s].tolist() == want[2], s
        assert got[1][s].tobytes() == np.array(want[1]).tobytes() and got[3][s].tobytes() == np.array(want[3]).tobytes()
        assert got[4][s] == want[4] and got[5][s] == want[5]
        sts.append(want[4])
        flags.append(want[5])
    assert ol.OK in sts and (mode == ol.STANDALONE or ol.ORIGIN_MISMATCH in sts) and ol.SENSOR_OFF_MAP in flags


def test_column_spans_equal_convex_fill_cells():
    rng = np.random.default_rng(5)
    for k in range(400):
        n = int(rng.integers(3, 9))
        if k % 4 == 0:       # convex, as footprints are
            a = np.sort(rng.uniform(0, 2 * np.pi, n))
            rad = rng.uniform(0.5, 12)
            poly = [(int(20 + rad * math.cos(t)), int(20 + rad * math.sin(t))) for t in a]
        else:                # any vertex list: the equivalence does not need convexity
            poly = [tuple(int(v) for v in rng.integers(0, 40, 2)) for _ in range(n)]
        lit = set(ol.convex_fill_cells(poly, 64))
        spans = {(x, y) for x, (lo, hi) in ol.column_spans(poly).items() for y in range(lo, hi + 1)}
        assert lit == spans, poly
