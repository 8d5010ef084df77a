"""tests/costmap_window_cases.py pinned on hand-computed cases: costmap_2d's rolling-window origin, the static layer's
copy with worldToMap and interpretValue, and the tf2 transform into the map frame; and the numpy form held bit equal to
the plain-Python one."""
import ctypes as C
import math

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import costmap_window_cases as cw

R = 0.25    # window resolution of the hand cases: binary fractions, so every centre and quotient below is exact


def one_map(data, mox=0.0, moy=0.0, mr=R):
    return dict(data=np.asarray(data, np.uint8), mox=mox, moy=moy, mr=mr)


def test_origin_snaps_toward_zero_for_positive_and_negative_offsets():
    # sx = 4: size_m = 3.5 * 0.25 = 0.875, half 0.4375
    assert cw.snap(0.0, 1.0, 4, R) == 0.5          # new 0.5625: 2.25 cells -> 2
    assert cw.snap(0.0, -1.0, 4, R) == -1.25       # new -1.4375: -5.75 cells -> -5 (toward zero, not -6)
    assert cw.snap(0.0, 0.4375, 4, R) == 0.0       # exactly on the old origin
    assert cw.snap(0.1, 0.4375, 4, R) == 0.1       # -0.4 cells -> 0: a small move keeps the origin


def test_origin_is_carried_across_cycles():
    o, seen = 0.0, []
    for rx in (1.0, 1.3125, 0.0, 0.0):
        o = cw.snap(o, rx, 4, R)
        seen.append(o)
    # 0.5625 -> 2 cells: 0.5; 0.875 - 0.5 = 1.5 cells -> 1: 0.75; -0.4375 - 0.75 = -4.75 -> -4: -0.25; then 0 cells
    assert seen == [0.5, 0.75, -0.25, -0.25]


def test_size_in_meters_has_the_half_cell():
    assert cw.size_in_meters(4, R) == 0.875
    # with the half cell the robot at 0.9375 gives 0.5 (2 cells); sx * r would give 0.4375 (1.75 -> 1 cell: 0.25)
    assert cw.snap(0.0, 0.9375, 4, R) == 0.5
    assert math.trunc((0.9375 - 4 * R / 2) / R) * R == 0.25


def test_cell_centres_on_map_cell_edges_take_the_upper_cell():
    # window cells of 0.25 from origin 0: centres 0.125, 0.375, ...; a map of 0.125 cells puts them on cell edges
    data = np.zeros((8, 8), np.uint8)
    data[:, 1] = 100                                                   # lethal in map column 1 only
    m = one_map(data, mr=0.125)
    row, org, st = cw.window([m], (0.1875, 0.1875, 0.0), 0, (0.0, 0.0, R), (2, 2), 4)
    assert st == cw.OK and org == (0.0, 0.0, R)
    # centre 0.125 / 0.125 = 1.0 -> cell 1; 0.375 / 0.125 = 3.0 -> cell 3
    assert row == [cw.interpret_value(int(data[1, 1])), cw.interpret_value(int(data[1, 3])),
                   cw.interpret_value(int(data[3, 1])), cw.interpret_value(int(data[3, 3]))]
    assert row == [254, 0, 254, 0]


def test_low_side_is_strict_and_high_side_is_off_at_the_size():
    m = one_map(np.full((2, 2), 100, np.uint8), mox=0.125, moy=0.125)
    assert cw.world_to_map(0.125, 0.125, R, 2) == 0           # on the origin: on the map
    assert cw.world_to_map(np.nextafter(0.125, 0), 0.125, R, 2) is None
    assert cw.world_to_map(0.625 - 1e-12, 0.125, R, 2) == 1
    assert cw.world_to_map(0.625, 0.125, R, 2) is None        # quotient 2.0 == size: off
    assert cw.world_to_map(float("nan"), 0.125, R, 2) is None
    # window origin 0, 3 x 1 cells: centres 0.125 (on the map's origin), 0.375, 0.625 (the map's far edge)
    row, _, _ = cw.window([m], (0.3125, 0.0, 0.0), 0, (0.0, 0.0, R), (3, 1), 3)
    assert cw.snap(0.0, 0.3125, 3, R) == 0.0
    assert row == [254, 254, 255]                             # x 0.625 is off; y 0.125 is on the map's origin
    row, _, _ = cw.window([m], (0.3125, -0.25, 0.0), 0, (0.0, 0.0, R), (3, 1), 3)
    assert cw.snap(0.0, -0.25, 1, R) == -0.25
    assert row == [255, 255, 255]                             # y -0.125 < 0.125: below the map


@pytest.mark.parametrize("v,track,trinary,want", [
    (255, True, True, 255), (255, False, True, 0), (255, True, False, 255), (255, False, False, 0),
    (0, True, True, 0), (0, True, False, 0), (50, True, True, 0), (50, True, False, 127), (99, True, False, 251),
    (99, True, True, 0), (100, True, True, 254), (100, True, False, 254), (101, True, False, 254), (1, True, False, 2),
])
def test_interpret_value(v, track, trinary, want):
    p = dict(cw.DEFAULTS, track_unknown_space=track, trinary_costmap=trinary)
    assert cw.interpret_value(v, p) == want
    assert cw.default_cost(p) == (255 if track else 0)


def test_interpret_value_of_the_int8_minus_one():
    assert np.array([-1], np.int8).view(np.uint8)[0] == 255 == cw.DEFAULTS["unknown_cost_value"]
    m, arrays = abi.make_static_maps([np.array([[-1, 100]], np.int8)], [(0.0, 0.0, 0.05)])
    assert m.unknown_cost_value == 255 and list(arrays["data"]) == [255, 100]


@pytest.mark.parametrize("mr,want", [(0.025, [1, 3, 5, 7]), (0.05, [0, 1, 2, 3]), (0.1, [0, 0, 1, 1])])
def test_map_resolutions_against_a_005_window(mr, want):
    # window cells of 0.05 from origin 0: centres 0.025, 0.075, 0.125, 0.175; map cell k holds the value k + 1 (graded)
    data = (np.arange(8, dtype=np.uint8) + 1)[None, :].repeat(8, axis=0)
    m = one_map(data, mr=mr)
    p = dict(cw.DEFAULTS, trinary_costmap=False, lethal_threshold=254)
    row, _, st = cw.window([m], (0.0875, 0.025, 0.0), 0, (0.0, 0.0, 0.05), (4, 1), 4, p=p)
    assert st == cw.OK and cw.snap(0.0, 0.0875, 4, 0.05) == 0.0
    assert row == [cw.interpret_value(k + 1, p) for k in want] == [k + 1 for k in want]


def _grid_map():
    """8 x 8 map of 0.25 cells centred on the origin, value 10 * my + mx (trinary off, threshold 254: kept as is)"""
    data = (10 * np.arange(8)[:, None] + np.arange(8)[None, :]).astype(np.uint8)
    return one_map(data, mox=-1.0, moy=-1.0), dict(cw.DEFAULTS, trinary_costmap=False, lethal_threshold=254)


def _cells(tf):
    m, p = _grid_map()
    # a 2 x 2 window whose origin stays at 0: centres (0.125, 0.125), (0.375, 0.125), (0.125, 0.375), (0.375, 0.375)
    row, _, st = cw.window([m], (0.1875, 0.1875, 0.0), 0, (0.0, 0.0, R), (2, 2), 4, tf, p)
    assert st == cw.OK
    return [(v // 10, v % 10) for v in row]                       # (my, mx) of each cell


def test_transforms():
    assert _cells(None) == [(4, 4), (4, 5), (5, 4), (5, 5)]
    assert _cells([0, 0, 0, 0, 0, 0, 1]) == _cells(None)
    # pure translation (0.5, -0.25): x + 2 cells, y - 1 cell
    assert _cells([0.5, -0.25, 0, 0, 0, 0, 1]) == [(3, 6), (3, 7), (4, 6), (4, 7)]
    # yaw pi/2: (x, y) -> (-y, x)
    s, c = math.sin(math.pi / 4), math.cos(math.pi / 4)
    assert _cells([0, 0, 0, 0, 0, s, c]) == [(4, 3), (5, 3), (4, 2), (5, 2)]
    # yaw pi: (x, y) -> (-x, -y)
    assert _cells([0, 0, 0, 0, 0, 1, math.cos(math.pi / 2)]) == [(3, 3), (3, 2), (2, 3), (2, 2)]
    # a non-unit quaternion: setRotation divides by |q|^2, so 3 q turns as q does
    assert _cells([0, 0, 0, 0, 0, 3 * s, 3 * c]) == _cells([0, 0, 0, 0, 0, s, c])
    # roll of 60 degrees: y shrinks to cos(60) y = 0.0625 / 0.1875 (the z row is not read)
    a = math.pi / 3
    assert _cells([0, 0, 0, math.sin(a / 2), 0, 0, math.cos(a / 2)]) == [(4, 4), (4, 5), (4, 4), (4, 5)]


def test_bad_robots_get_the_default_and_keep_their_origin():
    m, p = _grid_map()
    for mid, grid, r, st in ((1, (2, 2), R, cw.BAD_MAP), (-1, (2, 2), R, cw.BAD_MAP), (0, (0, 2), R, cw.BAD_GRID),
                             (0, (3, 2), R, cw.BAD_GRID), (0, (2, 2), 0.0, cw.BAD_GRID),
                             (0, (2, 2), float("inf"), cw.BAD_GRID), (0, (2, 2), float("nan"), cw.BAD_GRID)):
        row, org, got = cw.window([m], (5.0, 5.0, 0.0), mid, (0.5, 0.5, r), grid, 5, p=p)
        assert got == st and row == [255] * 5 and org[:2] == (0.5, 0.5)


@pytest.mark.parametrize("tf", [False, True])
def test_numpy_form_is_bit_equal_to_the_plain_one(tf):
    rng = np.random.default_rng(5 + tf)
    maps = [cw.random_map(rng, 90, 70, -2.0, -1.5, 0.05), cw.random_map(rng, 40, 60, -1.0, -2.0, 0.1),
            cw.random_map(rng, 160, 120, -2.5, -2.5, 0.025)]
    S, cap = 12, 23 * 19 + 5
    robot = np.column_stack([rng.uniform(-3, 3, S), rng.uniform(-3, 3, S), rng.uniform(-3, 3, S)])
    map_id = rng.integers(0, 3, S).astype(np.int32)
    map_id[3] = 7                                                       # a bad map id
    grid = np.column_stack([rng.integers(1, 24, S), rng.integers(1, 20, S)]).astype(np.int32)
    origin = np.column_stack([rng.uniform(-2, 2, S), rng.uniform(-2, 2, S), np.full(S, 0.05)])
    t = None
    if tf:
        t = np.array([fcase for fcase in (_random_tf(rng) for _ in range(S))])
    for p in (cw.DEFAULTS, dict(cw.DEFAULTS, track_unknown_space=False, trinary_costmap=False)):
        cost, org, st = cw.window_np(maps, robot, map_id, origin, grid, cap, t, p)
        for s in range(S):
            row, o, k = cw.window(maps, robot[s], int(map_id[s]), origin[s], grid[s], cap,
                                  None if t is None else t[s], p)
            assert k == st[s] and bytes(row) == cost[s].tobytes() and np.array(o).tobytes() == org[s].tobytes(), s
        assert st[3] == cw.BAD_MAP


def _random_tf(rng):
    from tests import frame_cases as fc
    return fc.random_transform(rng, tilted=bool(rng.integers(2)), unit=bool(rng.integers(2)))


def test_abi_mirrors():
    from teb_local_planner_b200 import load_library
    lib = load_library()
    assert lib.tebgpu_sizeof(18) == C.sizeof(abi.TebStaticMaps) == 6 * 4 + 8 + 4 * 8
    assert lib.tebgpu_sizeof(19) == C.sizeof(abi.TebCostmapWindowArgs) == 2 * 4 + 7 * 8
