"""tebgpu_costmap_obstacle_layer(_device): every robot's obstacle layer marked and cleared on the device, held byte for
byte to tests/obstacle_layer_cases.py on layer, cost, both origins, status and flags: on the hand cases; on random fleets
of 1 to 8192 robots with windows of 60 x 60 to 400 x 400 and one at the shared-memory limit, 0 to 4096 points per robot
(off the map, NaN and inf among them), in both modes and both combination methods, with strides that are and are not
multiples of 16 and misaligned rows, nothing written outside the rows; over 20 cycles of moving robots; bad robots and
argument errors; and a 20-cycle fleet loop (window, obstacle layer, conversion, local plan, backup modes, plan, costmap
check, finish) fed by a beam scanner, against the same loop fed the restatement's rasters."""
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import costmap_window_cases as cw
from tests import obstacle_layer_cases as ol
from tests import test_gpu_costmap_window as tw
from tests import test_obstacle_layer_cases as hand

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = "cuda:0"


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(64, 64, 8192, 64, 0)
    g.set_params(abi.default_params())
    yield g
    g.close()


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def run_device(g, p, pts, count, sensor, robot, grid, cap, layer, lo, master, org, footprint, row_shift=0):
    """the device entry point; row_shift moves both rasters off a 16-byte boundary by that many bytes"""
    S = len(robot)
    bufs = []
    for rows in (layer, master):
        b = torch.full((S * cap + 16,), 0x5A, dtype=torch.uint8, device=DEV)
        b[row_shift:row_shift + S * cap] = t(np.asarray(rows, np.uint8).reshape(-1))
        bufs.append(b)
    ins = dict(points=t(np.asarray(pts, np.float32)), point_count=t(np.asarray(count, np.int32)),
               sensor_origin=t(np.asarray(sensor, np.float64)), robot=t(np.asarray(robot, np.float64)),
               grid=t(np.asarray(grid, np.int32)), layer_origin=t(np.asarray(lo, np.float64)),
               origin=t(np.asarray(org, np.float64)), status=torch.full((S,), -7, dtype=torch.int32, device=DEV),
               flags=torch.full((S,), -7, dtype=torch.int32, device=DEV))
    fp = np.asarray(footprint, np.float64).reshape(-1, 2) if len(footprint) else None
    a = abi.make_obstacle_layer_args(S, cap, np.asarray(pts).shape[1], fp, **p,
                                     layer=bufs[0].data_ptr() + row_shift, cost=bufs[1].data_ptr() + row_shift,
                                     **{k: v.data_ptr() for k, v in ins.items()})
    g.costmap_obstacle_layer_device(a, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    out = []
    for b in bufs:
        h = b.cpu().numpy()
        assert (h[:row_shift] == 0x5A).all() and (h[row_shift + S * cap:] == 0x5A).all()   # nothing outside the rows
        out.append(h[row_shift:row_shift + S * cap].reshape(S, cap))
    return (out[0], ins["layer_origin"].cpu().numpy(), out[1], ins["origin"].cpu().numpy(), ins["status"].cpu().numpy(),
            ins["flags"].cpu().numpy())


NAMES = ("layer", "layer_origin", "cost", "origin", "status", "flags")


def check(g, p, pts, count, sensor, robot, grid, cap, layer, lo, master, org, footprint=(), host=True, row_shift=0):
    """both entry points against the numpy restatement; robots with a placed footprint vertex within 1e-9 of a cell
    edge (where the device's sin / cos may put it in the next cell) are left out of the byte comparison and counted"""
    pts = np.asarray(pts, np.float32)
    want = ol.obstacle_layer_np(p, pts, count, sensor, robot, grid, cap, layer, lo, master, org, footprint)
    S = len(robot)
    keep = np.ones(S, bool)
    if len(footprint) >= 3:
        for s in range(S):
            if want[4][s] == ol.OK and ol.footprint_near_cell_edge(robot[s], footprint, want[1][s], float(org[s][2])):
                keep[s] = False
    got = run_device(g, p, pts, count, sensor, robot, grid, cap, layer, lo, master, org, footprint, row_shift)
    for a, b, name in zip(got, want, NAMES):
        assert a[keep].tobytes() == b[keep].tobytes(), name
    if host and (want[4][keep] == ol.OK).all():
        h = g.costmap_obstacle_layer(pts[keep], np.asarray(count)[keep], np.asarray(sensor)[keep], np.asarray(robot)[keep],
                                     np.asarray(grid)[keep], np.asarray(layer)[keep], np.asarray(lo)[keep],
                                     np.asarray(org)[keep], np.asarray(master)[keep],
                                     footprint=np.asarray(footprint, np.float64).reshape(-1, 2) if len(footprint) else None,
                                     **p)
        for a, b, name in zip(h, want, NAMES):
            assert a.tobytes() == b[keep].tobytes(), name
    return want, int((~keep).sum())


def test_hand_cases(gpu):
    """every hand case of tests/test_obstacle_layer_cases.py through both entry points"""
    sq = [(-1.5, -1.5), (1.5, -1.5), (1.5, 1.5), (-1.5, 1.5)]
    lethal = [ol.LETHAL_OBSTACLE] * 64
    cases = [dict(robot=(x, y, yaw), r=1.0, layer=lethal, fp=fp) for fp, yaw, (x, y), _ in hand.FOOTPRINTS.values()]
    ends = [(7, 5), (5, 7), (3, 7), (1, 5), (1, 3), (3, 1), (5, 1), (7, 3), (7, 4), (1, 4), (4, 7), (4, 1)]
    cases += [dict(robot=(4.0, 4.0, 0.0), r=1.0, layer=lethal, fp=[(-4.5, -1.5)] + sq[1:], flags=ol.FOOTPRINT_OFF_MAP),
              dict(robot=(4.0, 4.0, 0.0), r=1.0, layer=lethal, fp=sq[:2]),
              dict(pts=[hand.centre(i, j) for i, j in ends], sensor=hand.centre(4, 4)),
              dict(pts=[hand.centre(4, 1), hand.centre(5, 2)], sensor=hand.centre(0, 0)),
              dict(kw=dict(raytrace_range=0.5), pts=[hand.centre(7, 5)], sensor=hand.centre(4, 4)),
              dict(kw=dict(raytrace_range=2.1), pts=[(3.45, 0.45, 0.0)], sensor=(0.15, 0.45, 0.0), robot=(1.8, 0.45, 0.0),
                   grid=(12, 3), r=0.3),
              dict(kw=dict(raytrace_range=3.0), pts=[(3.475, 0.025, 0.0)], sensor=(0.025, 0.025, 0.0),
                   robot=(1.75, 0.02, 0.0), grid=(70, 1), r=0.05),
              dict(pts=[(-1.125, 1.125, 0.0), (1.125, -1.0, 0.0), (3.0, 1.125, 0.0), (1.125, 3.0, 0.0), (2.875, 1.875, 0.0)],
                   sensor=hand.centre(4, 4)),
              dict(kw=dict(obstacle_range=2.5), pts=[hand.centre(2, 2), hand.centre(5, 5)], sensor=(-1.0, -1.0, 0.0),
                   flags=ol.SENSOR_OFF_MAP),
              dict(kw=dict(obstacle_range=0.5, clearing=False), pts=[(1.625, 1.125, 0.0), (1.375, 1.125, 0.0)],
                   sensor=hand.centre(4, 4)),
              dict(kw=dict(min_obstacle_height=0.25, max_obstacle_height=0.75, layer_max_obstacle_height=0.5),
                   pts=[(0.125, 1.125, 0.25), (1.125, 0.125, 0.75), (1.875, 1.125, 0.2499), (1.125, 1.875, 0.7501)],
                   sensor=hand.centre(4, 4, z=0.5)),
              dict(pts=[hand.centre(7, 4), hand.centre(6, 4)], sensor=hand.centre(4, 4)),
              dict(kw=dict(marking=False), pts=[(1.2, 1.2, 0.0)], sensor=hand.centre(4, 4)),
              dict(pts=[(1.2, 1.2, 0.0)], sensor=hand.centre(4, 4))]
    for c in cases:
        p = dict(ol.PARAMS, mode=ol.STANDALONE, obstacle_range=10.0, raytrace_range=10.0)
        p.update(c.get("kw", {}))
        pts, (sx, sy) = c.get("pts", []), c.get("grid", (8, 8))
        arr = np.zeros((1, max(len(pts), 1), 3), np.float32)
        if pts:
            arr[0, :len(pts)] = pts
        layer = c.get("layer", [ol.NO_INFORMATION] * (sx * sy))
        want, excluded = check(gpu, p, arr, [len(pts)], [c.get("sensor", (0, 0, 0))], [c.get("robot", (1.0, 1.0, 0.0))],
                               [(sx, sy)], sx * sy, [layer], [(0.0, 0.0)], [[0] * (sx * sy)], [(0.0, 0.0, c.get("r", 0.25))],
                               c.get("fp", ()))
        assert excluded == 0 and want[4][0] == ol.OK and want[5][0] == c.get("flags", 0)
        if c.get("flags") == ol.FOOTPRINT_OFF_MAP or len(c.get("fp", ())) == 2:
            assert want[0][0].tolist() == lethal                    # nothing cleared
    # the shifts over several cycles, and the combinations over static cells
    p = dict(ol.PARAMS, mode=ol.STANDALONE, clearing=False, marking=False)
    layer, lo = np.array([[10 * j + i for j in range(3) for i in range(4)]], np.uint8), np.zeros((1, 2))
    for rx, ry in ((3.0, 2.0), (1.0, 0.0), (20.0, 20.0)):
        want, _ = check(gpu, p, np.zeros((1, 1, 3)), [0], [(0, 0, 0)], [(rx, ry, 0.0)], [(4, 3)], 12, layer, lo,
                        [[0] * 12], [(9.0, 9.0, 1.0)])
        layer, lo = want[0], want[1]
    assert (layer == 255).all()
    M, L = [0, 254, 255, 100], [0, 254, 255, 50]
    for method in (0, 1, 2):
        p = dict(ol.PARAMS, mode=ol.COMBINE, combination_method=method, clearing=False, marking=False)
        check(gpu, p, np.zeros((1, 1, 3)), [0], [(0, 0, 0)], [(1.75, 1.75, 0.0)], [(4, 4)], 16,
              [[L[j] for j in range(4) for _ in range(4)]], [(0.0, 0.0)], [M * 4], [(0.0, 0.0, 1.0)])
    # a layer without track_unknown_space over static unknown cells, one shifted-in column; then out of step
    p = dict(ol.PARAMS, mode=ol.COMBINE, track_unknown_space=False, clearing=False, marking=False)
    want, _ = check(gpu, p, np.zeros((1, 1, 3)), [0], [(0, 0, 0)], [(2.75, 1.75, 0.0)], [(4, 4)], 16, [[254] * 16],
                    [(0.0, 0.0)], [[255] * 16], [(1.0, 0.0, 1.0)])
    assert want[2][0].tolist() == [254, 254, 254, 0] * 4
    want, _ = check(gpu, p, np.zeros((1, 1, 3)), [0], [(0, 0, 0)], [(2.75, 1.75, 0.0)], [(4, 4)], 16, [[254] * 16],
                    [(0.0, 0.0)], [[255] * 16], [(0.0, 0.0, 1.0)])
    assert want[4][0] == ol.ORIGIN_MISMATCH and want[2][0].tolist() == [255] * 16


def fleet(seed, S, sx, sy, P, mode, extra=0):
    rng = np.random.default_rng(seed)
    r = rng.choice([0.05, 0.05, 0.1, 0.025], S)
    robot = np.column_stack([rng.uniform(-20, 20, (S, 2)), rng.uniform(-np.pi, np.pi, S)])
    lo = robot[:, :2] - np.column_stack([sx * r, sy * r]) / 2 + rng.uniform(-4, 4, (S, 2)) * r[:, None]
    grid = np.tile(np.array([sx, sy], np.int32), (S, 1))
    grid[::7] = (max(sx - 5, 1), max(sy - 3, 1))
    cap = sx * sy + extra
    if mode == ol.COMBINE:
        org = np.column_stack([[cw.snap(lo[s, 0], robot[s, 0], grid[s, 0], r[s]) for s in range(S)],
                               [cw.snap(lo[s, 1], robot[s, 1], grid[s, 1], r[s]) for s in range(S)], r])
        org[5::11, 1] += r[5::11]                                              # some robots out of step with the window
    else:
        org = np.column_stack([rng.uniform(-9, 9, (S, 2)), r])
    sensor = np.column_stack([robot[:, :2] + rng.normal(0, 0.05, (S, 2)), rng.uniform(0.1, 0.4, S)])
    sensor[3::13, :2] += 100.0                                                 # sensors off the layer
    reach = max(sx, sy) * r[:, None] * 0.8
    ang = rng.uniform(-np.pi, np.pi, (S, P))
    dist = rng.uniform(0, 1, (S, P)) * reach
    pts = np.stack([sensor[:, None, 0] + dist * np.cos(ang), sensor[:, None, 1] + dist * np.sin(ang),
                    rng.uniform(-0.2, 2.2, (S, P))], -1).astype(np.float32)
    if P:
        flat = pts.reshape(-1, 3)
        k = rng.integers(0, S * P, max(S * P // 50, 1))
        flat[k[0::3], 0] = np.nan
        flat[k[1::3], 1] = np.inf
        flat[k[2::3], 0] = -np.inf
    count = rng.integers(0, P + 1, S)
    count[::4] = P
    layer = rng.choice(np.array([0, 254, 255], np.uint8), (S, cap), p=[0.5, 0.1, 0.4])
    master = rng.choice(np.array([0, 254, 255, 90], np.uint8), (S, cap))
    return pts, count, sensor, robot, grid, cap, layer, lo, master, org


SQUARE = [(-0.3, -0.25), (0.3, -0.25), (0.3, 0.25), (-0.3, 0.25)]
HEX = [(0.35 * math.cos(a), 0.25 * math.sin(a)) for a in np.arange(6) * np.pi / 3]
# 4 m long: off the layer for the 1.5 m and 3 m windows (r 0.025, 0.05), inside for most 6 m ones (r 0.1)
LONG = [(-2.0, -0.2), (2.0, -0.2), (2.0, 0.2), (-2.0, 0.2)]


@pytest.mark.parametrize("S,sx,sy,P,mode,method,extra,fp", [
    (1, 60, 60, 0, ol.COMBINE, 1, 0, SQUARE), (5, 60, 60, 7, ol.STANDALONE, 0, 7, HEX),
    (37, 121, 97, 4096, ol.STANDALONE, 1, 3, SQUARE), (37, 121, 97, 360, ol.COMBINE, 0, 0, ()),
    (1024, 120, 120, 360, ol.COMBINE, 1, 0, SQUARE), (1024, 120, 120, 720, ol.STANDALONE, 0, 5, HEX),
    (64, 400, 400, 1440, ol.COMBINE, 0, 5, HEX), (24, 400, 400, 360, ol.STANDALONE, 1, 0, SQUARE),
    (8192, 60, 60, 64, ol.STANDALONE, 1, 0, SQUARE), (8192, 60, 60, 32, ol.COMBINE, 0, 9, ()),
    (300, 60, 60, 100, ol.STANDALONE, 1, 3, LONG), (1024, 120, 120, 360, ol.COMBINE, 0, 0, LONG)])
def test_random_fleets_match_the_restatement(gpu, S, sx, sy, P, mode, method, extra, fp):
    pts, count, sensor, robot, grid, cap, layer, lo, master, org = fleet(S + sx + P + mode, S, sx, sy, P, mode, extra)
    p = dict(ol.PARAMS, mode=mode, combination_method=method, track_unknown_space=(S % 2 == 1), master_default=255,
             obstacle_range=2.5, raytrace_range=3.0, min_obstacle_height=0.0, max_obstacle_height=2.0,
             layer_max_obstacle_height=1.8)
    want, excluded = check(gpu, p, pts, count, sensor, robot, grid, cap, layer, lo, master, org, fp, host=False,
                           row_shift=S % 16)
    print(f"S={S}: {excluded} robots with a footprint vertex within 1e-9 of a cell edge left out")
    assert excluded <= max(1, S // 100)
    st = want[4]
    assert (st == ol.OK).sum() > S // 2
    if S > 20:
        assert (want[5] & ol.SENSOR_OFF_MAP).any() and (want[0] == ol.LETHAL_OBSTACLE).any()
        if mode == ol.COMBINE:
            assert (st == ol.ORIGIN_MISMATCH).any()
    if fp is LONG:            # both sides of the footprint-off-map gate, on the robots that ran
        off = (want[5][st == ol.OK] & ol.FOOTPRINT_OFF_MAP) != 0
        assert off.any() and (~off).any()


def test_host_entry_point_on_a_fleet(gpu):
    pts, count, sensor, robot, grid, cap, layer, lo, master, org = fleet(7, 300, 90, 70, 500, ol.STANDALONE, 3)
    p = dict(ol.PARAMS, mode=ol.STANDALONE)
    check(gpu, p, pts, count, sensor, robot, grid, cap, layer, lo, master, org, SQUARE, host=True, row_shift=3)


def test_a_window_at_the_shared_memory_limit(gpu):
    cap = gpu.obstacle_layer_max_cell_cap()
    print(f"tebgpu_get_info key 21: {cap} bytes")
    side = int(math.isqrt(cap))
    assert 450 <= side and side * side <= cap < 232448
    pts, count, sensor, robot, grid, _, layer, lo, master, org = fleet(8, 4, side, side, 2048, ol.STANDALONE)
    grid[:] = (side, side)
    layer = np.full((4, cap), 254, np.uint8)
    master = np.zeros((4, cap), np.uint8)
    check(gpu, dict(ol.PARAMS, mode=ol.STANDALONE), pts, count, sensor, robot, grid, cap, layer, lo, master, org, HEX,
          host=True, row_shift=1)
    with pytest.raises(T.TebGpuError):        # one byte past the limit
        gpu.costmap_obstacle_layer(pts[:1], count[:1], sensor[:1], robot[:1], grid[:1], np.zeros((1, cap + 1), np.uint8),
                                   lo[:1], org[:1], np.zeros((1, cap + 1), np.uint8))


def test_moving_robots_for_20_cycles(gpu):
    S, side, P = 256, 120, 360
    pts, count, sensor, robot, grid, cap, layer, lo, master, org = fleet(9, S, side, side, P, ol.STANDALONE)
    p = dict(ol.PARAMS, mode=ol.STANDALONE, combination_method=1, track_unknown_space=True)
    rng = np.random.default_rng(10)
    d = dict(points=t(pts), point_count=t(count.astype(np.int32)), sensor_origin=t(sensor), robot=t(robot), grid=t(grid),
             layer=t(layer), layer_origin=t(lo), origin=t(org), cost=t(master),
             status=torch.zeros(S, dtype=torch.int32, device=DEV), flags=torch.zeros(S, dtype=torch.int32, device=DEV))
    a = abi.make_obstacle_layer_args(S, cap, P, np.array(SQUARE), **p, **{k: v.data_ptr() for k, v in d.items()})
    h = [layer, lo, master, org]
    vel = rng.uniform(-0.6, 0.6, (S, 2))
    excluded = 0
    for k in range(20):
        gpu.costmap_obstacle_layer_device(a, stream=torch.cuda.current_stream().cuda_stream)
        want = ol.obstacle_layer_np(p, pts, count, sensor, robot, grid, cap, h[0], h[1], h[2], h[3], SQUARE)
        torch.cuda.synchronize()
        keep = np.array([not ol.footprint_near_cell_edge(robot[s], SQUARE, want[1][s], org[s, 2]) for s in range(S)])
        excluded += int((~keep).sum())
        got = [d[n].cpu().numpy() for n in ("layer", "layer_origin", "cost", "origin", "status", "flags")]
        for x, y, name in zip(got, want, NAMES):
            assert x[keep].tobytes() == y[keep].tobytes(), (k, name)
        h = [got[0], got[1], got[2], got[3]]      # a left-out robot carries the device's bytes on
        robot[:, :2] += vel * 0.2
        sensor[:, :2] += vel * 0.2
        pts[:, :, :2] += (vel * 0.2)[:, None, :].astype(np.float32)
        for n, v in (("robot", robot), ("sensor_origin", sensor), ("points", pts)):
            d[n].copy_(t(v))
    print(f"{excluded} robot-cycles left out of 20 x {S} (a footprint vertex within 1e-9 of a cell edge)")
    assert excluded <= 20 * S // 100
    assert (h[1] != lo).any(1).mean() > 0.9


def test_bad_robots_and_argument_errors(gpu):
    pts, count, sensor, robot, grid, cap, layer, lo, master, org = fleet(12, 16, 60, 60, 40, ol.COMBINE)
    org[:, :2] = [[cw.snap(lo[s, 0], robot[s, 0], grid[s, 0], org[s, 2]), cw.snap(lo[s, 1], robot[s, 1], grid[s, 1], org[s, 2])]
                  for s in range(16)]
    grid[1], grid[2], grid[3] = (0, 60), (61, 60), (60, -1)
    org[4, 2], org[5, 2] = 0.0, np.nan
    lo[6, 0] = np.inf
    count[7], count[8] = -1, 41
    org[9, 0] += 1e-12                                          # out of step with the window
    for mode in (ol.COMBINE, ol.STANDALONE):
        p = dict(ol.PARAMS, mode=mode, master_default=77)
        want, _ = check(gpu, p, pts, count, sensor, robot, grid, cap, layer, lo, master, org, host=False)
        st = want[4]
        assert st[1:7].tolist() == [ol.BAD_GRID] * 6 and st[7:9].tolist() == [ol.BAD_POINTS] * 2
        assert st[9] == (ol.ORIGIN_MISMATCH if mode == ol.COMBINE else ol.OK) and st[0] == ol.OK
        assert want[0][1:9].tobytes() == layer[1:9].tobytes() and want[1][1:9].tobytes() == lo[1:9].tobytes()
        assert (want[2][1:9] == 77).all() if mode == ol.STANDALONE else want[2][1:10].tobytes() == master[1:10].tobytes()
        for s in range(1, 10 if mode == ol.COMBINE else 9):
            keep = [0, s]
            with pytest.raises(T.TebGpuError):
                gpu.costmap_obstacle_layer(pts[keep], count[keep], sensor[keep], robot[keep], grid[keep], layer[keep],
                                           lo[keep], org[keep], master[keep], **p)
    ok = [0]
    base = (pts[ok], count[ok], sensor[ok], robot[ok], grid[ok], layer[ok], lo[ok], org[ok], master[ok])
    gpu.costmap_obstacle_layer(*base, mode=ol.COMBINE)
    for kw in (dict(footprint=np.zeros((65, 2))), dict(footprint=np.array([[0, 0], [np.nan, 0], [1, 1]])),
               dict(obstacle_range=-1.0), dict(raytrace_range=np.nan), dict(mode=2), dict(master_default=256)):
        with pytest.raises(T.TebGpuError):
            gpu.costmap_obstacle_layer(*base, **kw)
    big = np.zeros((8193, 3))
    with pytest.raises(T.TebGpuError):       # more robots than max_scenes
        gpu.costmap_obstacle_layer(np.zeros((8193, 1, 3)), np.zeros(8193), big, big, np.full((8193, 2), 4), np.zeros((8193, 16)),
                                   np.zeros((8193, 2)), big + [0, 0, 0.05], np.zeros((8193, 16)), mode=ol.STANDALONE)


# ---- the fleet cycle on one stream: window -> obstacle layer -> costmap conversion -> local plan -> backup modes ->
# ---- plan -> costmap check -> finish, fed by a beam scanner, against the same loop fed the restatement's rasters

FOOTPRINT = np.array([(-0.1, -0.1), (0.1, -0.1), (0.1, 0.1), (-0.1, 0.1)])
BEAMS, BEAM_RANGE, BOX_HALF = 120, 3.0, 0.3


def _scan(robot, static, box, radius=0.2):
    """each robot's laser: BEAMS beams from its centre, the first hit on a lethal static cell, the unmapped box or another
    robot's disc, else the point at BEAM_RANGE (which clears and does not mark); [B][BEAMS][3] float32 at z = 0.2"""
    B = len(robot)
    ang = robot[:, 2:3] + np.linspace(-np.pi, np.pi, BEAMS, endpoint=False)[None, :]
    steps = np.arange(1, int(BEAM_RANGE / 0.02) + 1) * 0.02
    X = robot[:, None, None, 0] + np.cos(ang)[:, :, None] * steps
    Y = robot[:, None, None, 1] + np.sin(ang)[:, :, None] * steps
    mx = np.floor((X - static["mox"]) / static["mr"]).astype(np.int64)
    my = np.floor((Y - static["moy"]) / static["mr"]).astype(np.int64)
    msy, msx = static["data"].shape
    on = (mx >= 0) & (my >= 0) & (mx < msx) & (my < msy)
    hit = np.zeros(X.shape, bool)
    hit[on] = static["data"][my[on], mx[on]] == 100
    hit |= (np.abs(X - box[0]) <= BOX_HALF) & (np.abs(Y - box[1]) <= BOX_HALF)
    for o in range(B):
        d2 = (X - robot[o, 0]) ** 2 + (Y - robot[o, 1]) ** 2 <= radius ** 2
        d2[o] = False
        hit |= d2
    first = np.where(hit.any(-1), hit.argmax(-1), len(steps) - 1)
    px = np.take_along_axis(X, first[..., None], -1)[..., 0]
    py = np.take_along_axis(Y, first[..., None], -1)[..., 0]
    return np.stack([px, py, np.full(px.shape, 0.2)], -1).astype(np.float32)


def _loop_params():
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 0
    p.max_vel_trans = p.max_vel_x
    return p


def _box_start(d):
    """the box's first centre: on robot 0's global plan, the first row 1 m or more ahead of the robot's nearest row"""
    pl, r0 = d["global_plan"][0], d["robot"][0]
    b, e = int(d["plan_begin"][0]), int(d["plan_end"][0])
    dist = np.hypot(pl[b:e, 0] - r0[0], pl[b:e, 1] - r0[1])
    k = int(np.argmin(dist))
    ahead = k + int(np.argmax(dist[k:] >= 1.0))
    return pl[b + ahead, :2].copy()


def _fleet_loop(restated, cycles=20, B=16, P_cap=160, M_cap=2048, n_cap=96, Lb=10, side=60):
    d = scenes.global_plans(B, 1024, S=B, seed=21)
    ident = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
    trans = np.tile(ident, (B, 1))
    static = tw._loop_map(d, ident)
    box0 = _box_start(d)
    cap = side * side
    p = _loop_params()
    lp = dict(ol.PARAMS, mode=ol.COMBINE, combination_method=1, obstacle_range=2.5, raytrace_range=3.0)
    g = T.TebGpu(B, n_cap, B, M_cap, 0)
    g.set_params(p)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=DEV)
    f64, i32 = torch.float64, torch.int32
    dm, keep = tw.device_maps([static])
    h_org = np.column_stack([d["robot"][:, :2] - 1.5, np.full(B, 0.05)])
    h_lo, h_layer = h_org[:, :2].copy(), np.full((B, cap), 255, np.uint8)
    cost, grid, origin = z((B, cap), torch.uint8), t(np.full((B, 2), side, np.int32)), t(h_org)
    layer, lorg = t(h_layer), t(h_lo)
    map_id, wst = z(B, i32), z(B, i32)
    lst, lfl = z(B, i32), z(B, i32)
    pts, pcnt, sensor = z((B, BEAMS, 3), torch.float32), t(np.full(B, BEAMS, np.int32)), z((B, 3), f64)
    robot = t(d["robot"].copy())
    custom = np.zeros((B, 1), abi.OBST_DTYPE)
    custom["x"], custom["y"], custom["type"] = 0.4, -0.3, abi.TEB_OBST_POINT
    cu, cc, cu_tf = t(custom.view(np.uint8)), t(np.ones(B, np.int32)), t(trans)
    obst, ocount = z(B * M_cap * 64, torch.uint8), z(B, i32)
    gp, begin, end = t(d["global_plan"]), t(d["plan_begin"].copy()), t(d["plan_end"])
    plan, pcount, result = z((B, P_cap, 3), f64), z(B, i32), z(B, i32)
    state = {k: t(v) for k, v in abi.make_cycle_state(B, Lb).items()}
    vel, since = z((B, 3), f64), z(B, f64)
    poses, n, sid = z((B, n_cap, 4), f64), z(B, i32), t(np.arange(B, dtype=np.int32))
    vs = np.zeros((B, 4))
    vs[:, 3] = 1.0
    vstart, vgoal = t(vs), t(vs)
    costo, chi2, status, iters = z(B, f64), z(B, f64), z(B, i32), z(B, i32)
    cmd, path, feas, qc = z((B, 4), f64), z(B, i32), z(B, i32), z(B, i32)
    cmd_vel, outcome, osc = z((B, 3), f64), z(B, i32), z(B, i32)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, B, M_cap, 0, 0
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
    bs.vel_start, bs.vel_goal, bs.prefer_rotdir = vstart.data_ptr(), vgoal.data_ptr(), state["prefer_rotdir"].data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = costo.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    wa = abi.TebCostmapWindowArgs()
    wa.S, wa.cell_cap = B, cap
    wa.robot, wa.map_id, wa.costmap_to_map = robot.data_ptr(), map_id.data_ptr(), None
    wa.origin, wa.grid, wa.cost, wa.status = origin.data_ptr(), grid.data_ptr(), cost.data_ptr(), wst.data_ptr()
    la_args = abi.make_obstacle_layer_args(B, cap, BEAMS, FOOTPRINT, **lp, points=pts.data_ptr(),
                                           point_count=pcnt.data_ptr(), sensor_origin=sensor.data_ptr(),
                                           robot=robot.data_ptr(), grid=grid.data_ptr(), layer=layer.data_ptr(),
                                           layer_origin=lorg.data_ptr(), origin=origin.data_ptr(), cost=cost.data_ptr(),
                                           status=lst.data_ptr(), flags=lfl.data_ptr())
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles, ca.behind_robot_dist = B, cap, M_cap, 1, 1, 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.custom, ca.custom_count = cu.data_ptr(), cc.data_ptr()
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    fr = abi.make_frame_args(custom_to_costmap=cu_tf.data_ptr())
    la = abi.make_local_plan_args(1024, P_cap, 0, max_lookahead_dist=2.0, global_plan=gp.data_ptr(),
                                  plan_begin=begin.data_ptr(), plan_end=end.data_ptr(), robot=robot.data_ptr(),
                                  robot_vel=vel.data_ptr(), grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  infeasible_count=state["infeasible_count"].data_ptr(), since_infeasible=since.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), result=result.data_ptr())
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    fa = abi.make_feasibility_args(0.1, max_queries=512, feasible=feas.data_ptr(), query_count=qc.data_ptr())
    world = abi.make_costmap_world(cap, cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), FOOTPRINT)
    sc = dict(buffer_length=Lb, oscillation_recovery_min_duration=2.0)
    dt, now = 0.2, 1000.0
    s = torch.cuda.Stream()
    trace = []
    for k in range(cycles):
        box = box0 + np.array([0.01, -0.01]) * k
        cy = abi.make_cycle_args(now, L_cap=Lb, **sc, local_plan_result=result.data_ptr(), robot_vel=vel.data_ptr(),
                                 cmd=cmd.data_ptr(), feasible=feas.data_ptr(), cmd_vel=cmd_vel.data_ptr(),
                                 outcome=outcome.data_ptr(), oscillating=osc.data_ptr(),
                                 **{kk: state[kk].data_ptr() for kk in abi.CYCLE_STATE})
        s.synchronize()
        h_robot = robot.cpu().numpy()
        scan = _scan(h_robot, static, box)
        h_sensor = np.column_stack([h_robot[:, :2], np.full(B, 0.2)])
        with torch.cuda.stream(s):
            pts.copy_(t(scan))
            sensor.copy_(t(h_sensor))
            since.copy_(now - state["last_infeasible"])
            if restated:
                s.synchronize()
                c, h_org, _ = cw.window_np([static], h_robot, np.zeros(B, np.int32), h_org, np.full((B, 2), side), cap)
                h_layer, h_lo, c, h_org, lst_h, _ = ol.obstacle_layer_np(lp, scan, np.full(B, BEAMS), h_sensor, h_robot,
                                                                         np.full((B, 2), side), cap, h_layer, h_lo, c,
                                                                         h_org, FOOTPRINT)
                assert (lst_h == ol.OK).all()
                cost.copy_(t(c))
                origin.copy_(t(h_org))
            else:
                g.costmap_window_device(dm, wa, stream=s.cuda_stream)
                g.costmap_obstacle_layer_device(la_args, stream=s.cuda_stream)
            g.costmap_obstacles_device(ca, stream=s.cuda_stream, frames=fr)
            g.local_plan_device(bs, la, stream=s.cuda_stream)
            g.backup_modes_device(bs, cy, stream=s.cuda_stream)
            g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, path=path,
                          stream=s.cuda_stream)
            g.check_feasible_costmap_device(bs, fa, world, stream=s.cuda_stream)
            g.finish_cycle_device(bs, cy, stream=s.cuda_stream)
            th = robot[:, 2]
            robot[:, 0] += (cmd_vel[:, 0] * torch.cos(th) - cmd_vel[:, 1] * torch.sin(th)) * dt
            robot[:, 1] += (cmd_vel[:, 0] * torch.sin(th) + cmd_vel[:, 1] * torch.cos(th)) * dt
            robot[:, 2] += cmd_vel[:, 2] * dt
            vel.copy_(cmd_vel)
        s.synchronize()
        if not restated:
            assert (lst.cpu().numpy() == ol.OK).all()
        oc = ocount.cpu().numpy()
        rows = obst.cpu().numpy().reshape(B, M_cap * 64)
        rec = dict(n=n, status=status, path=path, cmd=cmd, cmd_vel=cmd_vel, outcome=outcome, feasible=feas,
                   query_count=qc, poses=poses, obst_count=ocount, cost=cost, origin=origin, **state)
        c = {kk: v.cpu().numpy().copy() for kk, v in rec.items()}
        c["rows"] = [rows[b, :max(int(oc[b]), 0) * 64].tobytes() for b in range(B)]
        c["box"] = box
        c["obstacles"] = rows[0].view(abi.OBST_DTYPE).copy()
        trace.append(c)
        now += dt
    g.close()
    return trace


def test_fleet_loop_with_the_obstacle_layer_matches_the_loop_fed_the_restated_rasters():
    dev = _fleet_loop(False)
    ref = _fleet_loop(True)
    for k, (a, b) in enumerate(zip(dev, ref)):
        for key in a:
            assert (a[key] == b[key]) if key == "rows" else (np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes()), (k, key)
    # robot 0 sees the box: rows inside it whose cell the static window does not hold as lethal, and its band
    # associates at least one of them with a pose (tebgpu_build_system_graph on that cycle's band and table)
    d = scenes.global_plans(16, 1024, S=16, seed=21)
    static = tw._loop_map(d, np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]))
    msy, msx = static["data"].shape
    g2 = T.TebGpu(1, 96, 1, 2048, 0)
    g2.set_params(_loop_params())
    seen, associated = 0, 0
    for c in dev:
        cnt, ox, oy, r = int(c["obst_count"][0]), *c["origin"][0]
        rows = c["obstacles"][:cnt]
        new = []
        for l in np.nonzero((np.abs(rows["x"] - c["box"][0]) <= BOX_HALF + 0.05) &
                            (np.abs(rows["y"] - c["box"][1]) <= BOX_HALF + 0.05))[0]:
            i, j = (int(round((v - o) / r - 0.5)) for v, o in ((rows["x"][l], ox), (rows["y"][l], oy)))
            cell = cw.world_to_map(ox + (i + 0.5) * r, static["mox"], static["mr"], msx), \
                cw.world_to_map(oy + (j + 0.5) * r, static["moy"], static["mr"], msy)
            if None in cell or static["data"][cell[1], cell[0]] != 100:
                new.append(l)
        nb = int(c["n"][0])
        if not new or nb < 3:
            continue
        seen += 1
        obst = np.zeros((1, 2048), abi.OBST_DTYPE)
        obst[0, :cnt] = rows
        vs = np.array([[0.0, 0.0, 0.0, 1.0]])
        hb = abi.HostBatch(c["poses"][:1], c["n"][:1], obst, c["obst_count"][:1], scene_id=np.zeros(1, np.int32),
                           vel_start=vs, vel_goal=vs, prefer_rotdir=c["prefer_rotdir"][:1])
        words = g2.build_system(hb, graph=True)["assoc"][0, :nb]
        associated += int(any(((words[:, l // 64] >> np.uint64(l % 64)) & np.uint64(1)).any() for l in new))
    g2.close()
    print(f"robot 0: {seen} cycles with box rows the static map lacks, {associated} with one associated to a pose")
    assert seen > 0 and associated > 0
    feas = np.concatenate([c["feasible"] for c in dev])
    assert (feas == 1).any()
