"""tebgpu_costmap_voxel_layer(_device): every robot's voxel layer marked and cleared on the device, held byte for byte
to tests/voxel_layer_cases.py on voxels, layer, both origins, cost, status and flags: on the hand cases; on random
fleets of 1 to 8192 robots with windows of 60 x 60 up to the shared-memory limit, 1 to 4 sources of 0 to 4096 points
(NaN, inf, off the grid, above and below it), z_voxels 1 / 10 / 16 and varied thresholds, with strides that are and are
not multiples of 16 and misaligned rows, nothing written outside them; over 20 cycles of moving robots; bad robots and
argument errors; a 20-cycle fleet loop (window, voxel layer, conversion, local plan, backup modes, plan, costmap check,
finish) fed by a laser ring and a depth camera, robot 0 driving at an unmapped table, against the same loop fed the
restatement's rasters; and one cycle of window, obstacle layer and voxel layer combined."""
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import costmap_window_cases as cw
from tests import obstacle_layer_cases as ol
from tests import voxel_layer_cases as vl
from tests import test_gpu_costmap_obstacle_layer as tol
from tests import test_gpu_costmap_window as tw
from tests import test_voxel_layer_cases as hand

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
DEV = "cuda:0"
t = tol.t
U = vl.UNKNOWN_COLUMN


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(64, 64, 8192, 64, 0)
    g.set_params(abi.default_params())
    yield g
    g.close()


def src_structs(sources):
    return [abi.make_observation_source(**s) for s in sources]


def run_device(g, p, sources, pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org, footprint, shift=0):
    """the device entry point; shift moves the three rows off a 16-byte boundary by that many cells"""
    S = len(robot)
    bufs = []
    for rows, dt, fill in ((vox, torch.int32, 0x5A5A5A5A), (layer, torch.uint8, 0x5A), (master, torch.uint8, 0x5A)):
        b = torch.full((S * cap + 16,), fill, dtype=dt, device=DEV)
        h = np.asarray(rows, np.uint32 if dt == torch.int32 else np.uint8).reshape(-1)
        b[shift:shift + S * cap] = t(h.view(np.int32) if dt == torch.int32 else h)
        bufs.append(b)
    ins = dict(points=t(np.asarray(pts, np.float32)), point_count=t(np.asarray(count, np.int32)),
               sensor_origin=t(np.asarray(sensor, np.float64)), robot=t(np.asarray(robot, np.float64)),
               grid=t(np.asarray(grid, np.int32)), layer_origin=t(np.asarray(lo, np.float64)),
               origin=t(np.asarray(org, np.float64)), status=torch.full((S,), -7, dtype=torch.int32, device=DEV),
               flags=torch.full((S,), -7, dtype=torch.int32, device=DEV))
    fp = np.asarray(footprint, np.float64).reshape(-1, 2) if len(footprint) else None
    a = abi.make_voxel_layer_args(S, cap, np.asarray(pts).shape[2], src_structs(sources), fp, **p,
                                  voxels=bufs[0].data_ptr() + 4 * shift, layer=bufs[1].data_ptr() + shift,
                                  cost=bufs[2].data_ptr() + shift, **{k: v.data_ptr() for k, v in ins.items()})
    g.costmap_voxel_layer_device(a, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    out = []
    for b, fill in zip(bufs, (0x5A5A5A5A, 0x5A, 0x5A)):
        h = b.cpu().numpy()
        assert (h[:shift] == fill).all() and (h[shift + S * cap:] == fill).all()     # nothing outside the rows
        h = h[shift:shift + S * cap].reshape(S, cap)
        out.append(h.view(np.uint32) if h.dtype == np.int32 else h)
    return (out[0], out[1], ins["layer_origin"].cpu().numpy(), out[2], ins["origin"].cpu().numpy(),
            ins["status"].cpu().numpy(), ins["flags"].cpu().numpy())


NAMES = ("voxels", "layer", "layer_origin", "cost", "origin", "status", "flags")


def check(g, p, sources, pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org, footprint=(), host=True,
          shift=0):
    """both entry points against the numpy restatement; robots with a placed footprint vertex within 1e-9 of a cell
    edge (where the device's sin / cos may put it in the next cell) are left out of the byte comparison and counted"""
    pts = np.asarray(pts, np.float32)
    want = vl.voxel_layer_np(p, sources, pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org, footprint)
    S = len(robot)
    keep = np.ones(S, bool)
    if len(footprint) >= 3:
        for s in range(S):
            if want[5][s] == vl.OK and ol.footprint_near_cell_edge(robot[s], footprint, want[2][s], float(org[s][2])):
                keep[s] = False
    got = run_device(g, p, sources, pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org, footprint, shift)
    for a, b, name in zip(got, want, NAMES):
        assert a[keep].tobytes() == b[keep].tobytes(), name
    if host and (want[5][keep] == vl.OK).all():
        h = g.costmap_voxel_layer(pts[keep], np.asarray(count)[keep], np.asarray(sensor)[keep], np.asarray(robot)[keep],
                                  np.asarray(grid)[keep], np.asarray(vox)[keep], np.asarray(layer)[keep],
                                  np.asarray(lo)[keep], np.asarray(org)[keep], np.asarray(master)[keep],
                                  src_structs(sources),
                                  footprint=np.asarray(footprint, np.float64).reshape(-1, 2) if len(footprint) else None,
                                  **p)
        for a, b, name in zip(h, want, NAMES):
            assert a.tobytes() == b[keep].tobytes(), name
    return want, int((~keep).sum())


def one(g, sources, points, sensors, sx=12, sy=1, r=1.0, voxels=None, layer=None, footprint=(), robot=None, **kw):
    """hand.strip through both entry points; returns the literal restatement's result"""
    want = hand.strip(sources, points, sensors, sx, sy, r, voxels, layer, footprint, robot, **kw)
    p = dict(vl.PARAMS, mode=vl.STANDALONE, z_resolution=0.1)
    p.update(kw)
    n, K = sx * sy, len(sources)
    P = max(1, max(len(v) for v in points))
    arr = np.zeros((1, K, P, 3), np.float32)
    for k, v in enumerate(points):
        if v:
            arr[0, k, :len(v)] = v
    robot = (sx * r / 2, sy * r / 2, 0.0) if robot is None else robot
    got, _ = check(g, p, sources, arr, [[len(v) for v in points]], [sensors], [robot], [(sx, sy)], n,
                   [[U] * n if voxels is None else voxels], [[255] * n if layer is None else layer], [(0.0, 0.0)],
                   [[0] * n], [(0.0, 0.0, r)], footprint)
    assert got[0][0].tolist() == want[0] and got[1][0].tolist() == want[1] and got[3][0].tolist() == want[3]
    assert (got[5][0], got[6][0]) == (want[5], want[6])
    return want


def test_hand_cases(gpu):
    """the hand cases of tests/test_voxel_layer_cases.py through both entry points"""
    for Z, ut, column, want in [(10, 15, U, 0), (10, 5, U, 255), (10, 0, 0xFC00, 0), (1, 0, U, 0), (16, 14, U, 255)]:
        s = [(0.5, 0.5, 0.05 if Z == 1 else 0.25)]
        got = one(gpu, hand.RAY[0], [[(5.5, 0.5, s[0][2])]], s, voxels=[column] * 12, z_voxels=Z, unknown_threshold=ut)
        assert got[1][:4] == [want] * 4
    for mt in (0, 1, 2):
        one(gpu, [vl.source(clearing=False, obstacle_range=10.0)], [[(3.5, 0.5, 0.25), (3.5, 0.5, 0.75)]],
            [(0.5, 0.5, 0.25)], mark_threshold=mt)
    top = [U] * 12
    top[5] = U | hand.voxel(7)
    lay = [255] * 12
    lay[5] = 254
    src = [vl.source(obstacle_range=0.5, raytrace_range=10.0)]
    assert one(gpu, src, [[(8.5, 0.5, 0.25)]], [(0.5, 0.5, 0.25)], voxels=top, layer=lay)[1][5] == 254
    assert one(gpu, src, [[(8.5, 0.5, 0.75)]], [(0.5, 0.5, 0.75)], voxels=top, layer=lay)[1][5] == 0
    one(gpu, [vl.source(marking=False, raytrace_range=50.0)], [[(30.5, 0.5, 0.25)]], [(0.5, 0.5, 0.25)])
    one(gpu, [vl.source(marking=False, raytrace_range=10.0)], [[(6.5, 0.5, 0.25)]], [(0.5, 0.5, 0.25)])
    for sensor in [(0.5, 0.5, 1.0), (0.5, 0.5, 5.0), (-0.5, 0.5, 0.25), (0.5, 0.5, -0.1)]:
        got = one(gpu, [vl.source(clearing=False), vl.source(obstacle_range=50.0)], [[], [(5.5, 0.5, 0.25)]],
                  [(0.5, 0.5, 0.25), sensor])
        assert got[6] == vl.sensor_off_map(1)
    one(gpu, [vl.source(clearing=False, obstacle_range=10.0, min_obstacle_height=-1.0)], [[(3.5, 0.5, -0.3)]],
        [(0.5, 0.5, 0.25)], origin_z=0.1)
    # 3-D rays in every octant from the centre of an 8 x 8 x 10 block
    ends = [(x + 0.5, y + 0.5, z * 0.1 + 0.05) for x in (0, 7) for y in (0, 7) for z in (0, 9)] + \
        [(4.5, 0.5, 0.95), (0.5, 4.5, 0.05), (7.5, 4.5, 0.55), (4.5, 7.5, 0.35)]
    one(gpu, [vl.source(obstacle_range=0.1, raytrace_range=20.0)], [ends], [(4.5, 4.5, 0.45)], sx=8, sy=8,
        robot=(4.0, 4.0, 0.0), r=1.0)
    # two sources in one call: the mark of each survives the other's clearing
    got = one(gpu, [hand.LASER, hand.CAMERA], [hand.LASER_PTS, hand.CAMERA_PTS], [hand.SENSOR, hand.SENSOR])
    assert got[1][3] == got[1][10] == 254
    # two calls, either order, differ; the device matches the single call above
    for first, second in (((hand.LASER, hand.LASER_PTS), (hand.CAMERA, hand.CAMERA_PTS)),
                          ((hand.CAMERA, hand.CAMERA_PTS), (hand.LASER, hand.LASER_PTS))):
        a = one(gpu, [first[0]], [first[1]], [hand.SENSOR])
        b = one(gpu, [second[0]], [second[1]], [hand.SENSOR], voxels=a[0], layer=a[1])
        assert b[1] != got[1]
    sq = [(-1.5, -1.5), (1.5, -1.5), (1.5, 1.5), (-1.5, 1.5)]
    off = [vl.source(clearing=False, marking=False)]
    one(gpu, off, [[]], [(0, 0, 0)], sx=8, sy=8, voxels=[U | hand.voxel(4)] * 64, layer=[254] * 64, footprint=sq,
        robot=(4.0, 4.0, 0.0))
    one(gpu, off, [[]], [(0, 0, 0)], sx=8, sy=8, layer=[254] * 64, footprint=[(-4.5, -1.5)] + sq[1:],
        robot=(4.0, 4.0, 0.0))


def fleet(seed, S, sx, sy, K, P, mode, extra=0):
    rng = np.random.default_rng(seed)
    r = rng.choice([0.05, 0.05, 0.1, 0.025], S)
    robot = np.column_stack([rng.uniform(-20, 20, (S, 2)), rng.uniform(-np.pi, np.pi, S)])
    lo = robot[:, :2] - np.column_stack([sx * r, sy * r]) / 2 + rng.uniform(-4, 4, (S, 2)) * r[:, None]
    grid = np.tile(np.array([sx, sy], np.int32), (S, 1))
    grid[::7] = (max(sx - 5, 1), max(sy - 3, 1))
    cap = sx * sy + extra
    if mode == vl.COMBINE:
        org = np.column_stack([[cw.snap(lo[s, 0], robot[s, 0], grid[s, 0], r[s]) for s in range(S)],
                               [cw.snap(lo[s, 1], robot[s, 1], grid[s, 1], r[s]) for s in range(S)], r])
        org[5::11, 1] += r[5::11]                                              # some robots out of step with the window
    else:
        org = np.column_stack([rng.uniform(-9, 9, (S, 2)), r])
    sensor = np.concatenate([robot[:, None, :2] + rng.normal(0, 0.05, (S, K, 2)), rng.uniform(0.1, 0.9, (S, K, 1))], -1)
    sensor[3::13, 0, :2] += 100.0                                              # sensors off the grid
    sensor[4::13, -1, 2] = 5.0                                                 # and above it
    reach = max(sx, sy) * r[:, None, None] * 0.8
    ang, el = rng.uniform(-np.pi, np.pi, (S, K, P)), rng.uniform(-0.6, 0.6, (S, K, P))
    dist = rng.uniform(0, 1, (S, K, P)) * reach
    pts = np.stack([sensor[..., None, 0] + dist * np.cos(ang), sensor[..., None, 1] + dist * np.sin(ang),
                    sensor[..., None, 2] + dist * np.tan(el)], -1).astype(np.float32)
    if P:
        flat = pts.reshape(-1, 3)
        k = rng.integers(0, S * K * P, max(S * K * P // 50, 1))
        flat[k[0::4], 0] = np.nan
        flat[k[1::4], 1] = np.inf
        flat[k[2::4], 0] = -np.inf
        flat[k[3::4], 2] = np.nan
    count = rng.integers(0, P + 1, (S, K))
    count[::4] = P
    vox = rng.choice(np.array([U, U, U | hand.voxel(3), U & ~hand.voxel(2), 0xFC00, hand.voxel(1) | hand.voxel(5)],
                              np.uint32), (S, cap))
    layer = rng.choice(np.array([0, 254, 255], np.uint8), (S, cap), p=[0.5, 0.1, 0.4])
    master = rng.choice(np.array([0, 254, 255, 90], np.uint8), (S, cap))
    return pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org


def sources_for(K, seed):
    rng = np.random.default_rng(seed)
    return [vl.source(clearing=bool(k != 2 or K < 3), marking=bool(k != 1 or K < 2),
                      obstacle_range=float(rng.uniform(1.0, 3.0)), raytrace_range=float(rng.uniform(1.5, 4.0)),
                      min_obstacle_height=float(rng.uniform(-0.2, 0.1)), max_obstacle_height=float(rng.uniform(1.0, 2.5)))
            for k in range(K)]


SQUARE = tol.SQUARE
HEX = tol.HEX


@pytest.mark.parametrize("S,sx,sy,K,P,Z,ut,mt,mode,method,extra,fp", [
    (1, 60, 60, 1, 0, 10, 15, 0, vl.COMBINE, 1, 0, SQUARE), (5, 60, 60, 2, 7, 16, 0, 1, vl.STANDALONE, 0, 7, HEX),
    (37, 121, 97, 4, 4096, 10, 15, 0, vl.STANDALONE, 1, 3, SQUARE), (37, 121, 97, 3, 360, 1, 16, 2, vl.COMBINE, 0, 0, ()),
    (1024, 120, 120, 2, 360, 10, 15, 0, vl.COMBINE, 1, 0, SQUARE), (1024, 120, 120, 1, 720, 16, 8, 1, vl.STANDALONE, 0, 5, HEX),
    (64, 200, 200, 2, 1440, 10, 5, 0, vl.COMBINE, 0, 5, HEX), (8192, 60, 60, 2, 64, 10, 15, 0, vl.STANDALONE, 1, 0, SQUARE),
    (8192, 60, 60, 1, 32, 1, 0, 0, vl.COMBINE, 0, 9, ()), (300, 60, 60, 4, 100, 16, 15, 3, vl.STANDALONE, 1, 3, tol.LONG)])
def test_random_fleets_match_the_restatement(gpu, S, sx, sy, K, P, Z, ut, mt, mode, method, extra, fp):
    pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org = fleet(S + sx + P + K, S, sx, sy, K, P, mode, extra)
    p = dict(vl.PARAMS, mode=mode, combination_method=method, track_unknown_space=(S % 2 == 1), z_voxels=Z,
             unknown_threshold=ut, mark_threshold=mt, z_resolution=1.0 / Z, origin_z=0.05, max_obstacle_height=1.2)
    sources = sources_for(K, S + K)
    want, excluded = check(gpu, p, sources, pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org, fp,
                           host=False, shift=S % 16)
    print(f"S={S}: {excluded} robots with a footprint vertex within 1e-9 of a cell edge left out")
    assert excluded <= max(1, S // 100)
    st = want[5]
    assert (st == vl.OK).sum() > S // 2
    if S > 20:
        assert (want[6] & 15).any() and (want[1] == vl.LETHAL_OBSTACLE).any()
        if mode == vl.COMBINE:
            assert (st == vl.ORIGIN_MISMATCH).any()


def test_host_entry_point_on_a_fleet(gpu):
    pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org = fleet(7, 300, 90, 70, 3, 500, vl.STANDALONE, 3)
    p = dict(vl.PARAMS, mode=vl.STANDALONE)
    check(gpu, p, sources_for(3, 7), pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org, SQUARE,
          host=True, shift=3)


def test_a_window_at_the_shared_memory_limit(gpu):
    cap = gpu.voxel_layer_max_cell_cap()
    print(f"tebgpu_get_info key 22: {cap} cells")
    side = int(math.isqrt(cap))
    assert 200 <= side and side * side <= cap and cap % 32 == 0 and vl_smem(cap) <= 232448
    pts, count, sensor, robot, grid, _, vox, layer, lo, master, org = fleet(8, 4, side, side, 2, 2048, vl.STANDALONE)
    grid[:] = (side, side)
    vox = np.full((4, cap), U | hand.voxel(2), np.uint32)
    layer = np.full((4, cap), 254, np.uint8)
    master = np.zeros((4, cap), np.uint8)
    check(gpu, dict(vl.PARAMS, mode=vl.STANDALONE), sources_for(2, 8), pts, count, sensor, robot, grid, cap, vox, layer,
          lo, master, org, HEX, host=True, shift=1)
    with pytest.raises(T.TebGpuError):        # one cell past the limit
        gpu.costmap_voxel_layer(pts[:1], count[:1], sensor[:1], robot[:1], grid[:1], np.zeros((1, cap + 1), np.uint32),
                                np.zeros((1, cap + 1), np.uint8), lo[:1], org[:1], np.zeros((1, cap + 1), np.uint8),
                                src_structs(sources_for(2, 8)))


def vl_smem(cap):
    c = (cap + 31) // 32 * 32
    return c * 5 + c // 8


def test_moving_robots_for_20_cycles(gpu):
    S, side, K, P = 256, 120, 2, 360
    pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org = fleet(9, S, side, side, K, P, vl.STANDALONE)
    p = dict(vl.PARAMS, mode=vl.STANDALONE, combination_method=1, track_unknown_space=True, mark_threshold=1)
    sources = sources_for(K, 9)
    rng = np.random.default_rng(10)
    d = dict(points=t(pts), point_count=t(count.astype(np.int32)), sensor_origin=t(sensor), robot=t(robot), grid=t(grid),
             voxels=t(vox.view(np.int32)), layer=t(layer), layer_origin=t(lo), origin=t(org), cost=t(master),
             status=torch.zeros(S, dtype=torch.int32, device=DEV), flags=torch.zeros(S, dtype=torch.int32, device=DEV))
    a = abi.make_voxel_layer_args(S, cap, P, src_structs(sources), np.array(SQUARE), **p,
                                  **{k: v.data_ptr() for k, v in d.items()})
    h = [vox, layer, lo, master, org]
    vel = rng.uniform(-0.6, 0.6, (S, 2))
    excluded = 0
    for k in range(20):
        gpu.costmap_voxel_layer_device(a, stream=torch.cuda.current_stream().cuda_stream)
        want = vl.voxel_layer_np(p, sources, pts, count, sensor, robot, grid, cap, *h, SQUARE)
        torch.cuda.synchronize()
        keep = np.array([not ol.footprint_near_cell_edge(robot[s], SQUARE, want[2][s], org[s, 2]) for s in range(S)])
        excluded += int((~keep).sum())
        got = [d[n].cpu().numpy() for n in ("voxels", "layer", "layer_origin", "cost", "origin", "status", "flags")]
        got[0] = got[0].view(np.uint32)
        for x, y, name in zip(got, want, NAMES):
            assert x[keep].tobytes() == y[keep].tobytes(), (k, name)
        h = got[:5]                                  # a left-out robot carries the device's bytes on
        robot[:, :2] += vel * 0.2
        sensor[:, :, :2] += (vel * 0.2)[:, None, :]
        pts[..., :2] += (vel * 0.2)[:, None, None, :].astype(np.float32)
        for n, v in (("robot", robot), ("sensor_origin", sensor), ("points", pts)):
            d[n].copy_(t(v))
    print(f"{excluded} robot-cycles left out of 20 x {S} (a footprint vertex within 1e-9 of a cell edge)")
    assert excluded <= 20 * S // 100
    assert (h[2] != lo).any(1).mean() > 0.9


def test_bad_robots_and_argument_errors(gpu):
    pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org = fleet(12, 16, 60, 60, 2, 40, vl.COMBINE)
    org[:, :2] = [[cw.snap(lo[s, 0], robot[s, 0], grid[s, 0], org[s, 2]), cw.snap(lo[s, 1], robot[s, 1], grid[s, 1], org[s, 2])]
                  for s in range(16)]
    grid[1], grid[2], grid[3] = (0, 60), (61, 60), (60, -1)
    org[4, 2], org[5, 2] = 0.0, np.nan
    lo[6, 0] = np.inf
    count[7, 1], count[8, 0] = -1, 41
    org[9, 0] += 1e-12                                          # out of step with the window
    sources = sources_for(2, 12)
    for mode in (vl.COMBINE, vl.STANDALONE):
        p = dict(vl.PARAMS, mode=mode, master_default=77)
        want, _ = check(gpu, p, sources, pts, count, sensor, robot, grid, cap, vox, layer, lo, master, org, host=False)
        st = want[5]
        assert st[1:7].tolist() == [vl.BAD_GRID] * 6 and st[7:9].tolist() == [vl.BAD_POINTS] * 2
        assert st[9] == (vl.ORIGIN_MISMATCH if mode == vl.COMBINE else vl.OK) and st[0] == vl.OK
        assert want[0][1:9].tobytes() == vox[1:9].tobytes() and want[1][1:9].tobytes() == layer[1:9].tobytes()
        assert (want[3][1:9] == 77).all() if mode == vl.STANDALONE else want[3][1:10].tobytes() == master[1:10].tobytes()
        for s in range(1, 10 if mode == vl.COMBINE else 9):
            keep = [0, s]
            with pytest.raises(T.TebGpuError):
                gpu.costmap_voxel_layer(pts[keep], count[keep], sensor[keep], robot[keep], grid[keep], vox[keep],
                                        layer[keep], lo[keep], org[keep], master[keep], src_structs(sources), **p)
    ok = [0]
    base = (pts[ok], count[ok], sensor[ok], robot[ok], grid[ok], vox[ok], layer[ok], lo[ok], org[ok], master[ok])
    gpu.costmap_voxel_layer(*base, src_structs(sources), mode=vl.COMBINE)
    bad_src = [dict(vl.SOURCE, obstacle_range=-1.0), dict(vl.SOURCE, raytrace_range=np.nan)]
    for kw in (dict(footprint=np.zeros((65, 2))), dict(footprint=np.array([[0, 0], [np.nan, 0], [1, 1]])),
               dict(mode=2), dict(master_default=256), dict(z_voxels=0), dict(z_voxels=17), dict(unknown_threshold=-1),
               dict(unknown_threshold=17), dict(mark_threshold=17), dict(z_resolution=0.0), dict(z_resolution=np.inf),
               dict(origin_z=np.nan)):
        with pytest.raises(T.TebGpuError):
            gpu.costmap_voxel_layer(*base, src_structs(sources), **kw)
    for srcs in ([bad_src[0], vl.SOURCE], [vl.SOURCE, bad_src[1]]):
        with pytest.raises(T.TebGpuError):
            K = len(srcs)
            gpu.costmap_voxel_layer(np.zeros((1, max(K, 1), 1, 3)), np.zeros((1, max(K, 1))), np.zeros((1, max(K, 1), 3)),
                                    *base[3:], src_structs(srcs), mode=vl.COMBINE)
    a = abi.make_voxel_layer_args(1, 16, 1, src_structs([vl.SOURCE]))
    with pytest.raises(T.TebGpuError, match="missing required"):       # NULL arrays
        gpu.costmap_voxel_layer_device(a)
    for K in (0, 5):
        a = abi.make_voxel_layer_args(1, 16, 1, src_structs([vl.SOURCE] * K))
        with pytest.raises(T.TebGpuError, match="K outside"):
            gpu.costmap_voxel_layer_device(a)
    big = np.zeros((8193, 3))
    with pytest.raises(T.TebGpuError):       # more robots than max_scenes
        gpu.costmap_voxel_layer(np.zeros((8193, 1, 1, 3)), np.zeros((8193, 1)), np.zeros((8193, 1, 3)), big,
                                np.full((8193, 2), 4), np.zeros((8193, 16)), np.zeros((8193, 16)), np.zeros((8193, 2)),
                                big + [0, 0, 0.05], np.zeros((8193, 16)), src_structs([vl.SOURCE]), mode=vl.STANDALONE)


# ---- the fleet cycle on one stream: window -> voxel layer -> costmap conversion -> local plan -> backup modes ->
# ---- plan -> costmap check -> finish, fed by a laser ring and a depth camera; robot 0 drives at an unmapped table

BEAMS, BEAM_RANGE = 360, 3.0
TABLE_HALF, TABLE_TOP, LEG_HALF = 0.3, 0.7, 0.03
CAM_Z, CAM_AZ, CAM_EL = 0.3, 48, 17                     # camera height, azimuth and elevation rays
CAM_HFOV, CAM_VFOV = math.radians(35), math.radians(12)  # half angles
APPROACH = 0.05                                          # robot 0's step toward the table per cycle, m
VOXEL_PARAMS = dict(vl.PARAMS, mode=vl.COMBINE, combination_method=1, z_voxels=10, z_resolution=0.1, origin_z=0.0,
                    max_obstacle_height=1.0)
LASER_SRC = vl.source(obstacle_range=2.5, raytrace_range=3.0, min_obstacle_height=0.0, max_obstacle_height=2.0)
CAMERA_SRC = vl.source(obstacle_range=2.5, raytrace_range=3.0, min_obstacle_height=0.05, max_obstacle_height=2.0)


def _solid(X, Y, Z, static, table, wall):
    """True where (X, Y, Z) is inside something: a lethal static cell (to 1 m), a table leg, the table top, the wall
    behind the table, or the floor"""
    mx = np.floor((X - static["mox"]) / static["mr"]).astype(np.int64)
    my = np.floor((Y - static["moy"]) / static["mr"]).astype(np.int64)
    msy, msx = static["data"].shape
    on = (mx >= 0) & (my >= 0) & (mx < msx) & (my < msy)
    hit = np.zeros(X.shape, bool)
    hit[on] = static["data"][my[on], mx[on]] == 100
    hit &= Z <= 1.0
    dx, dy = X - table[0], Y - table[1]
    hit |= (np.abs(dx) <= TABLE_HALF) & (np.abs(dy) <= TABLE_HALF) & (Z >= TABLE_TOP) & (Z <= TABLE_TOP + 0.04)
    for cx in (-1, 1):
        for cy in (-1, 1):
            hit |= (np.abs(dx - cx * (TABLE_HALF - LEG_HALF)) <= LEG_HALF) & \
                (np.abs(dy - cy * (TABLE_HALF - LEG_HALF)) <= LEG_HALF) & (Z <= TABLE_TOP)
    (wx, wy), (nx, ny) = wall
    hit |= (np.abs((X - wx) * nx + (Y - wy) * ny) <= 0.03) & (np.abs(-(X - wx) * ny + (Y - wy) * nx) <= 1.0) & (Z <= 1.2)
    return hit | (Z <= 0.0)


def _cast(origin, dirs, static, table, wall):
    """the first hit of each ray from origin [B][3] along dirs [B][R][3] in 0.02 m steps, else the point at BEAM_RANGE"""
    steps = np.arange(1, int(BEAM_RANGE / 0.02) + 1) * 0.02
    P = origin[:, None, None, :] + dirs[:, :, None, :] * steps[None, None, :, None]
    hit = _solid(P[..., 0], P[..., 1], P[..., 2], static, table, wall)
    first = np.where(hit.any(-1), hit.argmax(-1), len(steps) - 1)
    return np.take_along_axis(P, first[..., None, None], 2)[:, :, 0, :].astype(np.float32)


def _sense(robot, static, table, wall):
    """(points [B][2][P][3], sensor [B][2][3]): the laser ring at 0.2 m and the depth camera at CAM_Z looking ahead"""
    B = len(robot)
    ang = robot[:, 2:3] + np.linspace(-np.pi, np.pi, BEAMS, endpoint=False)[None, :]
    ldir = np.stack([np.cos(ang), np.sin(ang), np.zeros_like(ang)], -1)
    az = robot[:, 2:3, None] + np.linspace(-CAM_HFOV, CAM_HFOV, CAM_AZ)[None, :, None]
    el = np.broadcast_to(np.linspace(-CAM_VFOV, CAM_VFOV, CAM_EL)[None, None, :], az.shape[:2] + (CAM_EL,))
    az = np.broadcast_to(az, el.shape)
    cdir = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], -1).reshape(B, -1, 3)
    lo = np.column_stack([robot[:, :2], np.full(B, 0.2)])
    co = np.column_stack([robot[:, :2], np.full(B, CAM_Z)])
    pts = np.zeros((B, 2, max(BEAMS, CAM_AZ * CAM_EL), 3), np.float32)
    pts[:, 0, :BEAMS] = _cast(lo, ldir, static, table, wall)
    pts[:, 1, :CAM_AZ * CAM_EL] = _cast(co, cdir, static, table, wall)
    return pts, np.stack([lo, co], 1)


def _table_start(d):
    """the table: on robot 0's global plan, the first row 2 m or more ahead of the robot's nearest row; the wall 0.8 m
    past it, across the plan"""
    pl, r0 = d["global_plan"][0], d["robot"][0]
    b, e = int(d["plan_begin"][0]), int(d["plan_end"][0])
    dist = np.hypot(pl[b:e, 0] - r0[0], pl[b:e, 1] - r0[1])
    k = int(np.argmin(dist))
    ahead = k + int(np.argmax(dist[k:] >= 2.0))
    c = pl[b + ahead, :2].copy()
    n = c - r0[:2]
    n /= np.linalg.norm(n)
    return c, (c + 0.8 * n, n)


def _table_loop(restated, cycles=20, B=16, P_cap=160, M_cap=2048, n_cap=96, Lb=10, side=60, with_obstacle_layer=False):
    d = scenes.global_plans(B, 1024, S=B, seed=21)
    ident = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
    trans = np.tile(ident, (B, 1))
    static = tw._loop_map(d, ident)
    table, wall = _table_start(d)
    r0 = d["robot"][0].copy()
    ahead = (table - r0[:2]) / np.linalg.norm(table - r0[:2])
    cap = side * side
    p = tol._loop_params()
    g = T.TebGpu(B, n_cap, B, M_cap, 0)
    g.set_params(p)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=DEV)
    f64, i32 = torch.float64, torch.int32
    dm, keep = tw.device_maps([static])
    h_org = np.column_stack([d["robot"][:, :2] - 1.5, np.full(B, 0.05)])
    h_lo = h_org[:, :2].copy()
    h_vox, h_layer = vl.reset_rows(B, cap)
    h_olo, h_olayer = h_lo.copy(), np.full((B, cap), 255, np.uint8)
    cost, grid, origin = z((B, cap), torch.uint8), t(np.full((B, 2), side, np.int32)), t(h_org)
    vox, layer, lorg = t(h_vox.view(np.int32)), t(h_layer), t(h_lo)
    olayer, olorg = t(h_olayer), t(h_olo)
    map_id, wst = z(B, i32), z(B, i32)
    lst, lfl, ost = z(B, i32), z(B, i32), z(B, i32)
    P = max(BEAMS, CAM_AZ * CAM_EL)
    pts, pcnt, sensor = z((B, 2, P, 3), torch.float32), t(np.tile([BEAMS, CAM_AZ * CAM_EL], (B, 1)).astype(np.int32)), \
        z((B, 2, 3), f64)
    lcnt, lsensor = t(np.full(B, BEAMS, np.int32)), z((B, 3), f64)      # the obstacle layer's laser
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
    va = abi.make_voxel_layer_args(B, cap, P, src_structs([LASER_SRC, CAMERA_SRC]), tol.FOOTPRINT, **VOXEL_PARAMS,
                                   points=pts.data_ptr(), point_count=pcnt.data_ptr(), sensor_origin=sensor.data_ptr(),
                                   robot=robot.data_ptr(), grid=grid.data_ptr(), voxels=vox.data_ptr(),
                                   layer=layer.data_ptr(), layer_origin=lorg.data_ptr(), origin=origin.data_ptr(),
                                   cost=cost.data_ptr(), status=lst.data_ptr(), flags=lfl.data_ptr())
    olp = dict(ol.PARAMS, mode=ol.COMBINE, combination_method=1, obstacle_range=2.5, raytrace_range=3.0)
    # the obstacle layer of the combined cycle: the laser alone, before the voxel layer
    oa = abi.make_obstacle_layer_args(B, cap, P, tol.FOOTPRINT, **olp, points=pts.data_ptr(),
                                      point_count=lcnt.data_ptr(), sensor_origin=lsensor.data_ptr(),
                                      robot=robot.data_ptr(), grid=grid.data_ptr(), layer=olayer.data_ptr(),
                                      layer_origin=olorg.data_ptr(), origin=origin.data_ptr(), cost=cost.data_ptr(),
                                      status=ost.data_ptr(), flags=None)
    oa.P_cap = 2 * P                                             # robot b's laser row starts at points[b][0]
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
    world = abi.make_costmap_world(cap, cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), tol.FOOTPRINT)
    sc = dict(buffer_length=Lb, oscillation_recovery_min_duration=2.0)
    dt, now = 0.2, 1000.0
    s = torch.cuda.Stream()
    trace = []
    for k in range(cycles):
        cy = abi.make_cycle_args(now, L_cap=Lb, **sc, local_plan_result=result.data_ptr(), robot_vel=vel.data_ptr(),
                                 cmd=cmd.data_ptr(), feasible=feas.data_ptr(), cmd_vel=cmd_vel.data_ptr(),
                                 outcome=outcome.data_ptr(), oscillating=osc.data_ptr(),
                                 **{kk: state[kk].data_ptr() for kk in abi.CYCLE_STATE})
        s.synchronize()
        # robot 0 drives straight at the table, 5 cm a cycle, whatever its plan says; the others follow their plans
        robot[0] = t(np.array([*(r0[:2] + ahead * APPROACH * k), math.atan2(ahead[1], ahead[0])]))
        h_robot = robot.cpu().numpy()
        h_pts, h_sensor = _sense(h_robot, static, table, wall)
        counts = np.tile([BEAMS, CAM_AZ * CAM_EL], (B, 1))
        with torch.cuda.stream(s):
            pts.copy_(t(h_pts))
            sensor.copy_(t(h_sensor))
            lsensor.copy_(t(np.ascontiguousarray(h_sensor[:, 0])))
            since.copy_(now - state["last_infeasible"])
            if restated:
                s.synchronize()
                c, h_org, _ = cw.window_np([static], h_robot, np.zeros(B, np.int32), h_org, np.full((B, 2), side), cap)
                if with_obstacle_layer:
                    h_olayer, h_olo, c, h_org, st_o, _ = ol.obstacle_layer_np(
                        olp, h_pts[:, 0, :BEAMS], np.full(B, BEAMS), h_sensor[:, 0], h_robot, np.full((B, 2), side),
                        cap, h_olayer, h_olo, c, h_org, tol.FOOTPRINT)
                    assert (st_o == ol.OK).all()
                h_vox, h_layer, h_lo, c, h_org, st_v, _ = vl.voxel_layer_np(
                    VOXEL_PARAMS, [LASER_SRC, CAMERA_SRC], h_pts, counts, h_sensor, h_robot, np.full((B, 2), side), cap,
                    h_vox, h_layer, h_lo, c, h_org, tol.FOOTPRINT)
                assert (st_v == vl.OK).all()
                cost.copy_(t(c))
                origin.copy_(t(h_org))
            else:
                g.costmap_window_device(dm, wa, stream=s.cuda_stream)
                if with_obstacle_layer:
                    g.costmap_obstacle_layer_device(oa, stream=s.cuda_stream)
                g.costmap_voxel_layer_device(va, stream=s.cuda_stream)
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
            assert (lst.cpu().numpy() == vl.OK).all()
            if with_obstacle_layer:
                assert (ost.cpu().numpy() == ol.OK).all()
        oc = ocount.cpu().numpy()
        rows = obst.cpu().numpy().reshape(B, M_cap * 64)
        rec = dict(n=n, status=status, path=path, cmd=cmd, cmd_vel=cmd_vel, outcome=outcome, feasible=feas,
                   query_count=qc, poses=poses, obst_count=ocount, cost=cost, origin=origin, **state)
        c = {kk: v.cpu().numpy().copy() for kk, v in rec.items()}
        c["rows"] = [rows[b, :max(int(oc[b]), 0) * 64].tobytes() for b in range(B)]
        c["obstacles"] = rows[0].view(abi.OBST_DTYPE).copy()
        c["robot0"], c["points0"], c["sensor0"] = h_robot[0].copy(), h_pts[0].copy(), h_sensor[0].copy()
        if restated:
            c["vox0"], c["layer0"], c["lo0"] = h_vox[0].copy(), h_layer[0].copy(), h_lo[0].copy()
        else:
            c["vox0"] = vox[0].cpu().numpy().view(np.uint32).copy()
            c["layer0"], c["lo0"] = layer[0].cpu().numpy().copy(), lorg[0].cpu().numpy().copy()
        trace.append(c)
        now += dt
    g.close()
    return trace, table


def _top_seen(c, table):
    """camera points of robot 0 on the table top this cycle"""
    cam = c["points0"][1, :CAM_AZ * CAM_EL]
    return int(((np.abs(cam[:, 0] - table[0]) <= TABLE_HALF) & (np.abs(cam[:, 1] - table[1]) <= TABLE_HALF) &
                (np.abs(cam[:, 2] - TABLE_TOP) <= 0.03)).sum())


def _top_only(vox, layer, lo, side, table, r=0.05):
    """cells under the table top whose only marked voxels are at the top's height (0.7 .. 0.8 m: voxel 7) and whose
    layer byte is lethal: cells nothing but the top made lethal"""
    ii, jj = np.meshgrid(np.arange(side), np.arange(side))
    cx, cy = lo[0] + (ii.ravel() + 0.5) * r, lo[1] + (jj.ravel() + 0.5) * r
    marked = vox[:side * side].astype(np.int64) >> 16
    under = (np.abs(cx - table[0]) <= TABLE_HALF) & (np.abs(cy - table[1]) <= TABLE_HALF)
    return np.nonzero(under & (marked == 1 << 7) & (layer[:side * side] == vl.LETHAL_OBSTACLE))[0]


def test_table_loop_with_the_voxel_layer_matches_the_loop_fed_the_restated_rasters():
    dev, table = _table_loop(False)
    ref, _ = _table_loop(True)
    for k, (a, b) in enumerate(zip(dev, ref)):
        for key in a:
            assert (a[key] == b[key]) if key == "rows" else (np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes()), (k, key)
    seen = [_top_seen(c, table) for c in dev]
    first = next(k for k, v in enumerate(seen) if v)
    gone = [k for k in range(first, len(dev)) if seen[k] == 0]
    assert gone, "the table top never left the camera's view"
    # after the top left the view, cells only the top made lethal stay lethal, their rows stay in robot 0's obstacle
    # table, and a band from robot 0 straight through the table associates one of them with a pose
    # (tebgpu_build_system_graph on that band and the cycle's table; robot 0's own band follows a pose it did not plan)
    side = 60
    g2 = T.TebGpu(1, 96, 1, 2048, 0)
    g2.set_params(tol._loop_params())
    kept, associated, tops = 0, 0, {}
    for k in gone:
        c = dev[k]
        top = _top_only(c["vox0"], c["layer0"], c["lo0"], side, table)
        tops[k] = top
        cnt, ox, oy, r = int(c["obst_count"][0]), *c["origin"][0]
        rows = c["obstacles"][:cnt]
        ij = np.rint((rows["x"] - ox) / r - 0.5).astype(np.int64) + side * np.rint((rows["y"] - oy) / r - 0.5).astype(np.int64)
        in_top = np.nonzero(np.isin(ij, top))[0]
        kept += bool(len(top)) and len(in_top) == len(top)
        if not len(in_top):
            continue
        nb = 25
        start, heading = c["robot0"][:2], c["robot0"][2]
        end = table + 1.2 * np.array([math.cos(heading), math.sin(heading)])
        band = np.zeros((1, 96, 4))
        band[0, :nb, :2] = start + np.linspace(0, 1, nb)[:, None] * (end - start)
        band[0, :nb, 2], band[0, :nb, 3] = heading, 0.1
        obst = np.zeros((1, 2048), abi.OBST_DTYPE)
        obst[0, :cnt] = rows
        vs = np.array([[0.0, 0.0, 0.0, 1.0]])
        hb = abi.HostBatch(band, np.array([nb], np.int32), obst, c["obst_count"][:1], scene_id=np.zeros(1, np.int32),
                           vel_start=vs, vel_goal=vs, prefer_rotdir=np.zeros(1, np.int32))
        words = g2.build_system(hb, graph=True)["assoc"][0, :nb]
        associated += int(any(((words[:, l // 64] >> np.uint64(l % 64)) & np.uint64(1)).any() for l in in_top))
    g2.close()
    # the 2-D obstacle layer fed the same points at the same poses (laser, then camera) clears those cells
    cap = side * side
    lay = np.full((1, cap), 255, np.uint8)
    lo = dev[0]["lo0"][None].copy()
    org = np.array([[lo[0, 0], lo[0, 1], 0.05]])
    cleared = []
    for k, c in enumerate(dev):
        for src, npts, hmin in ((0, BEAMS, 0.0), (1, CAM_AZ * CAM_EL, 0.05)):
            pp = dict(ol.PARAMS, mode=ol.STANDALONE, obstacle_range=2.5, raytrace_range=3.0, min_obstacle_height=hmin)
            lay, lo, _, org, st, _ = ol.obstacle_layer_np(pp, c["points0"][None, src, :npts], [npts],
                                                         c["sensor0"][None, src], c["robot0"][None], [(side, side)],
                                                         cap, lay, lo, np.zeros((1, cap), np.uint8), org)
            assert st[0] == ol.OK
        if k in gone:
            assert lo[0].tobytes() == c["lo0"].tobytes()
            cleared.append(bool(len(tops[k])) and not (lay[0][tops[k]] == ol.LETHAL_OBSTACLE).any())
    print(f"robot 0: camera points on the top per cycle {seen}; top out of view in {len(gone)} cycles; top-only cells "
          f"{[len(tops[k]) for k in gone]}, their rows kept in {kept} cycles, associated in {associated}; the obstacle "
          f"layer cleared them in {sum(cleared)}")
    assert kept == len(gone) and associated > 0 and all(cleared)


def test_window_obstacle_layer_and_voxel_layer_combined_match_the_restatement():
    dev, _ = _table_loop(False, cycles=2, with_obstacle_layer=True)
    ref, _ = _table_loop(True, cycles=2, with_obstacle_layer=True)
    for k, (a, b) in enumerate(zip(dev, ref)):
        for key in a:
            assert (a[key] == b[key]) if key == "rows" else (np.asarray(a[key]).tobytes() == np.asarray(b[key]).tobytes()), (k, key)
