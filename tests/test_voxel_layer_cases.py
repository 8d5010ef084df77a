"""tests/voxel_layer_cases.py pinned on hand-computed grids: bitsBelowThreshold, the reset column and reconfigureCB's
unknown threshold, mark_threshold, an overhang a ray passes under, rays dominant in every axis with ZOffset up and down,
the 2 r pull-back, the z and map-edge clamps, sensors off the grid, raytrace_range over the float distance, marks below
origin_z, two sources in one call against two calls, shifts over cycles, footprint clearing, both combinations and both
modes; and the numpy form held bit equal to the literal one on random fleets."""
import numpy as np
import pytest

from tests import obstacle_layer_cases as ol
from tests import voxel_layer_cases as vl

U = vl.UNKNOWN_COLUMN


def voxel(z):
    return (1 << z << 16) | (1 << z)


def strip(sources, points, sensors, sx=12, sy=1, r=1.0, voxels=None, layer=None, footprint=(), robot=None, **kw):
    """one robot on an sx x sy grid at the origin (robot at the centre, so nothing shifts), z_resolution 0.1"""
    p = dict(vl.PARAMS, mode=vl.STANDALONE, z_resolution=0.1)
    p.update(kw)
    n = sx * sy
    voxels = [U] * n if voxels is None else voxels
    layer = [vl.NO_INFORMATION] * n if layer is None else layer
    robot = (sx * r / 2, sy * r / 2, 0.0) if robot is None else robot
    return vl.voxel_layer(p, sources, points, sensors, robot, (sx, sy), n, voxels, layer, (0.0, 0.0), [0] * n,
                          (0.0, 0.0, r), footprint)


def test_bits_below_threshold_at_its_edges():
    assert vl.bits_below_threshold(0, 0) and not vl.bits_below_threshold(1, 0)
    assert vl.bits_below_threshold(0b1011, 3) and not vl.bits_below_threshold(0b1111, 3)
    assert vl.bits_below_threshold(0xFFFF, 16) and not vl.bits_below_threshold(0xFFFF, 15)
    assert vl.unknown_bits(U) == 0xFFFF and vl.marked_bits(U) == 0
    assert vl.unknown_bits(U & ~voxel(3)) == 0xFFFF & ~(1 << 3) and vl.unknown_bits(U | voxel(3)) == 0xFFFF & ~(1 << 3)


RAY = ([vl.source(obstacle_range=0.5)], [[(5.5, 0.5, 0.25)]], [(0.5, 0.5, 0.25)])   # clears cells 0 .. 3 at voxel 2


@pytest.mark.parametrize("Z,ut,column,want", [
    (10, 15, U, vl.FREE_SPACE), (10, 5, U, vl.NO_INFORMATION),              # 15 unknown bits against 21 and 11
    (10, 15, 0xFC00, vl.FREE_SPACE), (10, 5, 0xFC00, vl.FREE_SPACE),        # a cleared column: 6 unused bits
    (10, 0, 0xFC00, vl.FREE_SPACE),                                          # reconfigureCB adds the 6 back
    (1, 0, U, vl.FREE_SPACE),                                                # 15 unused bits, 15 added back
    (16, 15, U, vl.FREE_SPACE), (16, 14, U, vl.NO_INFORMATION), (16, 0, 0x0004, vl.FREE_SPACE)])
def test_reset_column_and_the_unknown_threshold(Z, ut, column, want):
    z = 0 if Z == 1 else 2
    sensors = [(0.5, 0.5, 0.05 if Z == 1 else 0.25)]
    pts = [[(5.5, 0.5, sensors[0][2])]]
    vox, lay, *_ = strip(RAY[0], pts, sensors, voxels=[column] * 12, z_voxels=Z, unknown_threshold=ut,
                         z_resolution=0.1)
    assert vox[:4] == [column & ~voxel(z) & 0xFFFFFFFF] * 4 and vox[4:] == [column] * 8
    assert lay[:4] == [want] * 4 and lay[4:] == [vl.NO_INFORMATION] * 8


@pytest.mark.parametrize("mt,want", [(0, vl.LETHAL_OBSTACLE), (1, vl.LETHAL_OBSTACLE), (2, vl.NO_INFORMATION)])
def test_mark_threshold_with_two_points_in_one_column(mt, want):
    src = [vl.source(clearing=False, obstacle_range=10.0)]
    vox, lay, *_ = strip(src, [[(3.5, 0.5, 0.25), (3.5, 0.5, 0.75)]], [(0.5, 0.5, 0.25)], mark_threshold=mt)
    assert vox[3] == U | voxel(2) | voxel(7)
    assert lay[3] == want
    # one mark alone passes only mark_threshold 0
    vox, lay, *_ = strip(src, [[(3.5, 0.5, 0.25)]], [(0.5, 0.5, 0.25)], mark_threshold=mt)
    assert lay[3] == (vl.LETHAL_OBSTACLE if mt == 0 else vl.NO_INFORMATION)


def test_a_ray_under_a_table_top_leaves_it_lethal_and_a_ray_through_it_clears_it():
    top = U | voxel(7)                                          # the top at z 0.7 over cell 5, marked in an earlier cycle
    voxels, layer = [U] * 12, [vl.NO_INFORMATION] * 12
    voxels[5], layer[5] = top, vl.LETHAL_OBSTACLE
    src = [vl.source(obstacle_range=0.5, raytrace_range=10.0)]
    under = [[(8.5, 0.5, 0.25)]]                                 # a leg past the table, seen under the top
    vox, lay, *_ = strip(src, under, [(0.5, 0.5, 0.25)], voxels=voxels, layer=layer)
    assert vox[5] == top & ~voxel(2) and lay[5] == vl.LETHAL_OBSTACLE
    assert lay[:5] == [vl.FREE_SPACE] * 5 and lay[6] == vl.FREE_SPACE
    # the 2-D obstacle layer fed the same point clears the cell
    p2 = dict(ol.PARAMS, mode=ol.STANDALONE, obstacle_range=0.5, raytrace_range=10.0)
    l2 = ol.obstacle_layer(p2, under[0], (0.5, 0.5, 0.25), (6.0, 0.5, 0.0), (12, 1), 12, layer, (0.0, 0.0), [0] * 12,
                           (0.0, 0.0, 1.0))[0]
    assert l2[5] == ol.FREE_SPACE
    # a ray at the top's height clears its voxel, and with it the cell
    vox, lay, *_ = strip(src, [[(8.5, 0.5, 0.75)]], [(0.5, 0.5, 0.75)], voxels=voxels, layer=layer)
    assert vox[5] == top & ~voxel(7) and lay[5] == vl.FREE_SPACE


def cells(visits, sx):
    return [(o % sx, o // sx, m.bit_length() - 17) for o, m in visits]


def test_rays_dominant_in_x_y_and_z_with_zoffset_up_and_down():
    assert cells(vl.raytrace_line_3d(0.5, 0.5, 0.5, 4.5, 2.5, 1.5, 8), 8) == \
        [(0, 0, 0), (1, 1, 0), (2, 1, 1), (3, 2, 1), (4, 2, 1)]
    assert cells(vl.raytrace_line_3d(0.5, 0.5, 0.5, 1.5, 3.5, 0.5, 8), 8) == [(0, 0, 0), (0, 1, 0), (1, 2, 0), (1, 3, 0)]
    assert cells(vl.raytrace_line_3d(0.5, 0.5, 0.5, 1.5, 0.5, 4.5, 8), 8) == \
        [(0, 0, 0), (0, 0, 1), (1, 0, 2), (1, 0, 3), (1, 0, 4)]
    assert cells(vl.raytrace_line_3d(2.5, 1.5, 4.5, 0.5, 0.5, 0.5, 8), 8) == \
        [(2, 1, 4), (1, 1, 3), (1, 0, 2), (0, 0, 1), (0, 0, 0)]
    assert cells(vl.raytrace_line_3d(4.5, 0.5, 3.5, 0.5, 2.5, 0.5, 8), 8) == \
        [(4, 0, 3), (3, 1, 2), (2, 1, 1), (1, 2, 1), (0, 2, 0)]


def test_raytrace_range_over_the_float_distance_and_a_zero_distance():
    # integer deltas (4, 0, 0) but a float distance of 4.4: 3 / 4.4 of 4 steps is 2 steps, not 3
    assert cells(vl.raytrace_line_3d(0.5, 0.5, 0.5, 4.9, 0.5, 0.5, 8, 3), 8) == [(0, 0, 0), (1, 0, 0), (2, 0, 0)]
    assert cells(vl.raytrace_line_3d(0.5, 0.5, 0.5, 4.5, 0.5, 0.5, 8, 3), 8) == [(k, 0, 0) for k in range(4)]
    # 0 / 0 and n / 0 both give scale 1: the one cell
    assert cells(vl.raytrace_line_3d(0.5, 0.5, 0.5, 0.5, 0.5, 0.5, 8, 0), 8) == [(0, 0, 0)]
    assert cells(vl.raytrace_line_3d(0.5, 0.5, 0.5, 0.5, 0.5, 0.5, 8, 3), 8) == [(0, 0, 0)]
    # max_length 0 over a positive distance: only the start
    assert cells(vl.raytrace_line_3d(0.5, 0.5, 0.5, 3.5, 0.5, 0.5, 8, 0), 8) == [(0, 0, 0)]


def test_the_pull_back_of_two_cells():
    p = dict(vl.PARAMS, max_obstacle_height=5.0)
    assert vl.clearing_end(10.0, 0.5, 0.5, (0.0, 0.5, 0.5), 0.0, 0.0, 1.0, 12, 1, p) == (8.0, 0.5, 0.5)
    assert vl.clearing_end(1.5, 0.5, 0.5, (0.0, 0.5, 0.5), 0.0, 0.0, 1.0, 12, 1, p) == (0.0, 0.5, 0.5)   # f = 0
    assert vl.clearing_end(0.0, 0.5, 0.5, (0.0, 0.5, 0.5), 0.0, 0.0, 1.0, 12, 1, p) == (0.0, 0.5, 0.5)   # dist 0
    # on the grid: a point 6 cells out clears 4 cells past the sensor's
    vox, lay, *_ = strip([vl.source(marking=False, raytrace_range=10.0)], [[(6.5, 0.5, 0.25)]], [(0.5, 0.5, 0.25)])
    assert lay[:5] == [vl.FREE_SPACE] * 5 and lay[5:] == [vl.NO_INFORMATION] * 7


def test_the_z_clamps_and_the_four_map_edge_clamps():
    p = dict(vl.PARAMS, max_obstacle_height=2.0, origin_z=0.0)
    x, _, z = vl.clearing_end(12.0, 0.5, 4.0, (0.0, 0.5, 0.0), 0.0, 0.0, 1.0, 40, 1, p)
    assert abs(z - 1.99) < 1e-12 and abs(x - 1.99 * 3) < 1e-12                     # t from max_obstacle_height - 0.01
    x, _, z = vl.clearing_end(12.0, 0.5, -4.0, (0.0, 0.5, 1.0), 0.0, 0.0, 1.0, 40, 1, p)
    assert z == 0.0 and abs(x - 2.4) < 1e-12                                         # t from origin_z
    x, _, z = vl.clearing_end(12.0, 0.5, 4.0, (0.0, 0.5, 3.0), 0.0, 0.0, 1.0, 40, 1, p)
    assert (x, z) == (0.0, 3.0)                                                      # above H: t = max(0, negative) = 0
    ex = 0.0 + (12 - 1 + 0.5) * 1.0                                                  # getSizeInMetersX
    assert vl.clearing_end(30.0, 0.5, 0.5, (6.0, 0.5, 0.5), 0.0, 0.0, 1.0, 12, 4, p)[0] == ex
    assert vl.clearing_end(-30.0, 0.5, 0.5, (6.0, 0.5, 0.5), 0.0, 0.0, 1.0, 12, 4, p)[0] == 0.0
    assert vl.clearing_end(6.0, 30.0, 0.5, (6.0, 0.5, 0.5), 0.0, 0.0, 1.0, 12, 4, p)[1] == 0.0 + 3.5
    assert vl.clearing_end(6.0, -30.0, 0.5, (6.0, 0.5, 0.5), 0.0, 0.0, 1.0, 12, 4, p)[1] == 0.0
    # two clamps at once take the smaller t
    w = vl.clearing_end(30.0, 30.0, 0.5, (6.0, 0.5, 0.5), 0.0, 0.0, 1.0, 12, 4, p)
    assert w[1] == 3.5 and w[0] < ex
    # on the grid: the right edge clamp ends in the last cell
    vox, lay, *_ = strip([vl.source(marking=False, raytrace_range=50.0)], [[(30.5, 0.5, 0.25)]], [(0.5, 0.5, 0.25)])
    assert lay == [vl.FREE_SPACE] * 12


@pytest.mark.parametrize("sensor", [(0.5, 0.5, 1.0), (0.5, 0.5, 5.0), (-0.5, 0.5, 0.25), (0.5, 0.5, -0.1)])
def test_a_sensor_off_the_grid_clears_nothing_and_sets_its_flag(sensor):
    src = [vl.source(clearing=False), vl.source(obstacle_range=50.0)]
    vox, lay, _, _, _, st, fl = strip(src, [[], [(5.5, 0.5, 0.25)]], [(0.5, 0.5, 0.25), sensor])
    assert st == vl.OK and fl == vl.sensor_off_map(1)
    assert lay[5] == vl.LETHAL_OBSTACLE and lay.count(vl.NO_INFORMATION) == 11        # marked, nothing cleared


def test_a_point_below_origin_z_is_marked_in_voxel_0():
    vox, lay, *_ = strip([vl.source(clearing=False, obstacle_range=10.0, min_obstacle_height=-1.0)], [[(3.5, 0.5, -0.3)]],
                         [(0.5, 0.5, 0.25)], origin_z=0.1)
    assert vox[3] == U | voxel(0) and lay[3] == vl.LETHAL_OBSTACLE


def test_height_bounds_and_obstacle_range():
    src = [vl.source(clearing=False, obstacle_range=3.0, min_obstacle_height=0.2, max_obstacle_height=0.6)]
    pts = [[(1.5, 0.5, 0.2), (2.5, 0.5, 0.6), (3.5, 0.5, 0.1999), (4.5, 0.5, 0.6001), (3.5, 0.5, 0.3)]]
    vox, lay, *_ = strip(src, pts, [(0.5, 0.5, 0.3)], max_obstacle_height=0.5)
    # 1.5: kept and marked; 2.5: above the layer's 0.5; 3.5 (z 0.3): distance 3 is not < 3; the other two filtered
    assert [i for i, v in enumerate(lay) if v == vl.LETHAL_OBSTACLE] == [1]


LASER = vl.source(obstacle_range=20.0, raytrace_range=20.0)
CAMERA = vl.source(obstacle_range=20.0, raytrace_range=20.0)
LASER_PTS, CAMERA_PTS = [(10.5, 0.5, 0.25)], [(3.5, 0.5, 0.25), (20.0, 0.5, 0.25)]
SENSOR = (0.5, 0.5, 0.25)


def test_two_sources_clear_before_either_marks_and_two_calls_differ():
    vox, lay, *_ = strip([LASER, CAMERA], [LASER_PTS, CAMERA_PTS], [SENSOR, SENSOR])
    want = [vl.FREE_SPACE] * 12
    want[3] = want[10] = vl.LETHAL_OBSTACLE
    assert lay == want
    for first, second in (((LASER, LASER_PTS), (CAMERA, CAMERA_PTS)), ((CAMERA, CAMERA_PTS), (LASER, LASER_PTS))):
        v1, l1, *_ = strip([first[0]], [first[1]], [SENSOR])
        v2, l2, *_ = strip([second[0]], [second[1]], [SENSOR], voxels=v1, layer=l1)
        assert l2 != lay
        assert (l2[3], l2[10]) == ((vl.LETHAL_OBSTACLE, vl.FREE_SPACE) if first[0] is LASER else
                                   (vl.FREE_SPACE, vl.LETHAL_OBSTACLE))


def test_shifts_by_one_cell_both_ways_and_past_the_window():
    p = dict(vl.PARAMS, mode=vl.STANDALONE)
    off = [vl.source(clearing=False, marking=False)]
    vox = [1000 + c for c in range(12)]
    lay = [c for c in range(12)]
    lo = (0.0, 0.0)
    for rx, want in ((3.0, lambda i, j: 1000 + (j + 1) * 4 + i + 1 if i < 3 and j < 2 else None),):
        out = vl.voxel_layer(p, off, [[]], [(0, 0, 0)], (rx, 3.0, 0.0), (4, 3), 12, vox, lay, lo, [0] * 12,
                             (9.0, 9.0, 1.0))
        assert out[2] == (1.0, 1.0)
        assert out[0] == [want(i, j) if want(i, j) is not None else U for j in range(3) for i in range(4)]
        assert out[1] == [v - 1000 if v != U else vl.NO_INFORMATION for v in out[0]]
    back = vl.voxel_layer(p, off, [[]], [(0, 0, 0)], (1.0, 1.0, 0.0), (4, 3), 12, out[0], out[1], out[2], [0] * 12,
                          (9.0, 9.0, 1.0))
    assert back[2] == (0.0, 0.0)
    assert back[0][5:7] == [1005, 1006] and back[0][:4] == [U] * 4 and back[0][4] == U
    far = vl.voxel_layer(p, off, [[]], [(0, 0, 0)], (40.0, 1.0, 0.0), (4, 3), 12, back[0], back[1], back[2], [0] * 12,
                         (9.0, 9.0, 1.0))
    assert far[0] == [U] * 12 and far[1] == [vl.NO_INFORMATION] * 12


def test_footprint_clearing_touches_only_the_2d_layer():
    sq = [(-1.5, -1.5), (1.5, -1.5), (1.5, 1.5), (-1.5, 1.5)]
    vox, lay, _, _, _, st, fl = strip([vl.source(clearing=False, marking=False)], [[]], [(0, 0, 0)], sx=8, sy=8,
                                      voxels=[U | voxel(4)] * 64, layer=[vl.LETHAL_OBSTACLE] * 64, footprint=sq,
                                      robot=(4.0, 4.0, 0.0))
    assert st == vl.OK and fl == 0 and vox == [U | voxel(4)] * 64
    free = {j * 8 + i for j in range(2, 6) for i in range(2, 6)}
    assert [c for c in range(64) if lay[c] == vl.FREE_SPACE] == sorted(free)
    _, lay, _, _, _, _, fl = strip([vl.source(clearing=False, marking=False)], [[]], [(0, 0, 0)], sx=8, sy=8,
                                   layer=[vl.LETHAL_OBSTACLE] * 64, footprint=[(-4.5, -1.5)] + sq[1:],
                                   robot=(4.0, 4.0, 0.0))
    assert fl == vl.FOOTPRINT_OFF_MAP and lay == [vl.LETHAL_OBSTACLE] * 64


@pytest.mark.parametrize("mode", [vl.COMBINE, vl.STANDALONE])
@pytest.mark.parametrize("method,want", [(0, [0, 254, 100, 50]), (1, [100, 254, 100, 100]), (2, [100] * 4)])
def test_combination_methods_and_modes(mode, method, want):
    p = dict(vl.PARAMS, mode=mode, combination_method=method, master_default=100)
    off = [vl.source(clearing=False, marking=False)]
    layer = [0, 254, 255, 50] * 4
    master = [100] * 16
    out = vl.voxel_layer(p, off, [[]], [(0, 0, 0)], (1.75, 1.75, 0.0), (4, 4), 16, [U] * 16, layer, (0.0, 0.0), master,
                         (0.0, 0.0, 1.0))
    assert out[5] == vl.OK and out[3] == want * 4
    if mode == vl.COMBINE:
        out = vl.voxel_layer(p, off, [[]], [(0, 0, 0)], (1.75, 1.75, 0.0), (4, 4), 16, [U] * 16, layer, (0.0, 0.0),
                             master, (1.0, 0.0, 1.0))
        assert out[5] == vl.ORIGIN_MISMATCH and out[3] == master and out[1] == layer


def test_bad_robots():
    p = dict(vl.PARAMS, mode=vl.STANDALONE, master_default=7)
    src = [vl.source(), vl.source()]
    out = vl.voxel_layer(p, src, [[], [(0, 0, 0)] * 3], [(0, 0, 0)] * 2, (1.0, 1.0, 0.0), (4, 4), 16, [U] * 16,
                         [1] * 16, (0.0, 0.0), [0] * 16, (0.0, 0.0, 1.0), P_cap=2)
    assert out[5] == vl.BAD_POINTS and out[3] == [7] * 16 and out[1] == [1] * 16
    out = vl.voxel_layer(p, src, [[], []], [(0, 0, 0)] * 2, (1.0, 1.0, 0.0), (5, 4), 16, [U] * 16, [1] * 16,
                         (0.0, 0.0), [0] * 16, (0.0, 0.0, 1.0))
    assert out[5] == vl.BAD_GRID


def random_case(rng, S, sx, sy, K, P, mode, footprint):
    r = rng.choice([0.05, 0.1])
    robot = np.column_stack([rng.uniform(-3, 3, (S, 2)), rng.uniform(-np.pi, np.pi, S)])
    lo = robot[:, :2] - np.array([sx, sy]) * r / 2 + rng.uniform(-3, 3, (S, 2)) * r
    grid = np.tile([sx, sy], (S, 1))
    org = np.column_stack([rng.uniform(-9, 9, (S, 2)), np.full(S, r)]) if mode == vl.STANDALONE else \
        np.column_stack([[ol.cw.snap(lo[s, 0], robot[s, 0], sx, r) for s in range(S)],
                         [ol.cw.snap(lo[s, 1], robot[s, 1], sy, r) for s in range(S)], np.full(S, r)])
    sensors = np.concatenate([robot[:, None, :2] + rng.normal(0, 0.05, (S, K, 2)), rng.uniform(-0.1, 1.2, (S, K, 1))], -1)
    reach = max(sx, sy) * r * 0.8
    ang, dist = rng.uniform(-np.pi, np.pi, (S, K, P)), rng.uniform(0, reach, (S, K, P))
    pts = np.stack([sensors[..., None, 0] + dist * np.cos(ang), sensors[..., None, 1] + dist * np.sin(ang),
                    rng.uniform(-0.4, 2.4, (S, K, P))], -1).astype(np.float32)
    flat = pts.reshape(-1, 3)
    k = rng.integers(0, len(flat), max(len(flat) // 40, 1))
    flat[k[0::3], 0], flat[k[1::3], 1], flat[k[2::3], 2] = np.nan, np.inf, -np.inf
    count = rng.integers(0, P + 1, (S, K))
    vox = rng.choice(np.array([U, U | voxel(3), U & ~voxel(2), 0, voxel(1) | voxel(5)], np.uint32), (S, sx * sy))
    lay = rng.choice(np.array([0, 254, 255], np.uint8), (S, sx * sy))
    master = rng.choice(np.array([0, 254, 255, 90], np.uint8), (S, sx * sy))
    return pts, count, sensors, robot, grid, vox, lay, lo, master, org


@pytest.mark.parametrize("K,Z,ut,mt,mode,method,fp", [
    (1, 10, 15, 0, vl.STANDALONE, 1, ()), (2, 10, 5, 1, vl.COMBINE, 0, [(-0.2, -0.15), (0.2, -0.15), (0.2, 0.15)]),
    (3, 16, 0, 2, vl.STANDALONE, 0, [(-0.2, -0.2), (0.2, -0.2), (0.2, 0.2), (-0.2, 0.2)]), (4, 1, 16, 0, vl.COMBINE, 1, ())])
def test_numpy_form_equals_the_literal_one(K, Z, ut, mt, mode, method, fp):
    rng = np.random.default_rng(K * 100 + Z)
    S, sx, sy, P = 6, 23, 17, 40
    pts, count, sensors, robot, grid, vox, lay, lo, master, org = random_case(rng, S, sx, sy, K, P, mode, fp)
    p = dict(vl.PARAMS, mode=mode, combination_method=method, z_voxels=Z, unknown_threshold=ut, mark_threshold=mt,
             z_resolution=0.12, origin_z=0.05, max_obstacle_height=1.5, track_unknown_space=K % 2 == 1)
    sources = [vl.source(clearing=k != 2, marking=k != 1, obstacle_range=1.0 + k * 0.3, raytrace_range=1.5 - k * 0.2,
                         min_obstacle_height=-0.5 + 0.1 * k, max_obstacle_height=2.0) for k in range(K)]
    want = vl.voxel_layer_np(p, sources, pts, count, sensors, robot, grid, sx * sy, vox, lay, lo, master, org, fp)
    for s in range(S):
        got = vl.voxel_layer(p, sources, [pts[s, k, :count[s, k]].tolist() for k in range(K)], sensors[s], robot[s],
                             grid[s], sx * sy, vox[s], lay[s], lo[s], master[s], org[s], fp, P_cap=P)
        assert got[0] == want[0][s].tolist() and got[1] == want[1][s].tolist()
        assert np.float64(got[2]).tobytes() == want[2][s].tobytes() and got[3] == want[3][s].tolist()
        assert np.float64(got[4]).tobytes() == want[4][s].tobytes()
        assert (got[5], got[6]) == (want[5][s], want[6][s])
    assert (want[5] == vl.OK).any()
