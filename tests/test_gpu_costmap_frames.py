"""Each scene's custom obstacles moved from their own frame into the costmap's on the device
(tebgpu_costmap_obstacles_tf / _tf_device, k_costmap_obstacles<true>), held to tests/frame_cases.py's restatement of
updateObstacleContainerWithCustomObstacles: with no transform the table is the verbatim path's bit for bit; with the
identity transform the rows are memcmp-equal except the recomputed polygon centroids; under random planar, tilted and
non-unit transforms every row and vertex is the restatement's bit for bit. Also host bits == device bits and the
argument errors."""
import ctypes as C

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import frame_cases as fc

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
S, C_CAP, PV, M_CAP = 12, 9, 40, 4096
IDENTITY = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(64, 64, S, M_CAP, 0, max_obst_vertices=PV)
    g.set_params(abi.default_params())
    yield g
    g.close()


def custom_scenes(seed, closing=True):
    """per scene: points, circles (some dynamic), lines, a pill, polygons (one with a repeated closing vertex when
    closing, one with collinear vertices) over a pool of PV vertices; custom_count drawn per scene"""
    rng = np.random.default_rng(seed)
    rows = np.zeros((S, C_CAP), abi.OBST_DTYPE)
    verts = np.zeros((S, PV, 2))
    count = rng.integers(3, C_CAP + 1, S).astype(np.int32)
    for s in range(S):
        nv = 0
        for k in range(C_CAP):
            r = rows[s, k]
            typ = [fc.TEB_OBST_POINT, fc.TEB_OBST_CIRCULAR, fc.TEB_OBST_LINE, fc.TEB_OBST_POLYGON, fc.TEB_OBST_PILL,
                   fc.TEB_OBST_POLYGON, fc.TEB_OBST_CIRCULAR, fc.TEB_OBST_POLYGON, fc.TEB_OBST_POINT][k]
            r["type"] = typ
            r["x"], r["y"] = rng.uniform(-3, 3, 2)
            r["vx"], r["vy"] = (rng.uniform(-0.5, 0.5, 2) if k % 3 == 1 else (0.0, 0.0))
            r["dynamic"] = int(k % 3 == 1)
            r["radius"] = 0.2 if typ in (fc.TEB_OBST_CIRCULAR, fc.TEB_OBST_PILL) else 0.0
            if typ in (fc.TEB_OBST_LINE, fc.TEB_OBST_PILL, fc.TEB_OBST_POLYGON):
                if typ != fc.TEB_OBST_POLYGON:
                    v = rng.uniform(-3, 3, (2, 2))
                elif k == 3:
                    v = rng.uniform(-3, 3, (5, 2))
                    if closing:
                        v = np.vstack([v, v[:1]])
                elif k == 5:
                    v = np.outer(np.linspace(0, 1, 4), rng.uniform(-3, 3, 2)) + rng.uniform(-1, 1, 2)
                else:
                    v = rng.uniform(-3, 3, (3, 2))
                r["vertex_begin"], r["vertex_count"] = nv, len(v)
                verts[s, nv:nv + len(v)] = v
                if typ == fc.TEB_OBST_POLYGON:
                    r["x"], r["y"] = fc.polygon_centroid([tuple(p) for p in v])
                else:
                    r["x"], r["y"] = 0.5 * (v[0, 0] + v[1, 0]), 0.5 * (v[0, 1] + v[1, 1])
                nv += len(v)
    return rows, verts, count


def transforms(seed, kind):
    rng = np.random.default_rng(seed)
    if kind == "identity":
        return np.tile(IDENTITY, (S, 1))
    return np.array([fc.random_transform(rng, tilted=kind == "tilted", unit=kind != "nonunit") for _ in range(S)])


def raster():
    return scenes.costmap_raster(S, 40, 40, 0.05, 0.03, seed=3)


def expect(rows, verts, count, tf):
    out_rows, out_verts = [], np.zeros_like(verts)
    for s in range(S):
        out_rows.append(fc.move_custom(rows[s, :count[s]], verts[s], list(tf[s]), out_verts[s]))
    return out_rows, out_verts


def run_device(g, r, rows, count, tf=None, verts=None):
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).to(DEV)
    cost, grid, origin, robot = t(r["cost"]), t(r["grid"]), t(r["origin"]), t(r["robot"])
    cu, cc = t(rows), t(count)
    obst = torch.zeros(S * M_CAP * 64, dtype=torch.uint8, device=DEV)
    ocount, need = torch.zeros(S, dtype=torch.int32, device=DEV), torch.zeros(S, dtype=torch.int32, device=DEV)
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = S, r["cost"].shape[1], M_CAP, C_CAP, 1
    ca.behind_robot_dist = 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.custom, ca.custom_count = cu.data_ptr(), cc.data_ptr()
    ca.obstacles, ca.obst_count, ca.needed = obst.data_ptr(), ocount.data_ptr(), need.data_ptr()
    ov = torch.zeros(S * PV * 2, dtype=torch.float64, device=DEV)
    fr = None
    if tf is not None:
        ttf = t(tf)
        tv = None if verts is None else t(verts)
        fr = abi.make_frame_args(custom_to_costmap=ttf.data_ptr(), custom_vertices=None if tv is None else tv.data_ptr(),
                                 obst_vertices=ov.data_ptr(), PV_cap=PV)
    g.costmap_obstacles_device(ca, stream=torch.cuda.current_stream().cuda_stream, frames=fr)
    torch.cuda.synchronize()
    o = obst.cpu().numpy().view(abi.OBST_DTYPE).reshape(S, M_CAP)
    return o, ocount.cpu().numpy(), need.cpu().numpy(), ov.cpu().numpy().reshape(S, PV, 2)


def _rows(o, cnt, count):
    """each scene's custom rows: the last count[s] rows of its table"""
    return [o[s, cnt[s] - count[s]:cnt[s]] for s in range(S)]


def test_null_frames_are_the_verbatim_path(gpu):
    r = raster()
    rows, verts, count = custom_scenes(1)
    ref = gpu.costmap_obstacles(r["cost"], r["grid"], r["origin"], r["robot"], M_CAP, custom=rows, custom_count=count)
    d = run_device(gpu, r, rows, count)
    fr = abi.make_frame_args()
    o = np.zeros((S, M_CAP), abi.OBST_DTYPE)
    cnt, need = np.zeros(S, np.int32), np.zeros(S, np.int32)
    ca = abi.TebCostmapArgs()
    cost = np.ascontiguousarray(r["cost"])
    ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles, ca.behind_robot_dist = \
        S, cost.shape[1], M_CAP, C_CAP, 1, 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = abi.ptr(cost), abi.ptr(r["grid"]), abi.ptr(r["origin"]), abi.ptr(r["robot"])
    ca.custom, ca.custom_count = abi.ptr(rows), abi.ptr(count)
    ca.obstacles, ca.obst_count, ca.needed = abi.ptr(o), abi.ptr(cnt), abi.ptr(need)
    assert gpu.lib.tebgpu_costmap_obstacles_tf(gpu.ctx, C.byref(ca), C.byref(fr)) == 0
    for s in range(S):
        k = ref[1][s]
        assert k > count[s] and d[1][s] == k == cnt[s]
        assert ref[0][s, :k].tobytes() == d[0][s, :k].tobytes() == o[s, :k].tobytes()


def test_explicit_identity(gpu):
    r = raster()
    rows, verts, count = custom_scenes(2, closing=False)
    ref = gpu.costmap_obstacles(r["cost"], r["grid"], r["origin"], r["robot"], M_CAP, custom=rows, custom_count=count)
    tf = transforms(0, "identity")
    o, cnt, need, ov = gpu.costmap_obstacles(r["cost"], r["grid"], r["origin"], r["robot"], M_CAP, custom=rows,
                                             custom_count=count, custom_to_costmap=tf, custom_vertices=verts)
    want_rows, want_verts = expect(rows, verts, count, tf)
    for s in range(S):
        k = cnt[s]
        assert k == ref[1][s]
        got, base = o[s, :k].copy(), ref[0][s, :k].copy()
        poly = got["type"] == fc.TEB_OBST_POLYGON
        assert got[~poly].tobytes() == base[~poly].tobytes()
        for field in ("vx", "vy", "radius", "dynamic", "type", "vertex_begin", "vertex_count", "_pad"):
            assert got[poly][field].tobytes() == base[poly][field].tobytes(), field
        assert o[s, k - count[s]:k].tobytes() == want_rows[s].tobytes()          # centroids recomputed as restated
    used = want_verts != 0
    assert (ov[used] == verts[used]).all() and ov.tobytes() == want_verts.tobytes()


@pytest.mark.parametrize("kind", ["planar", "tilted", "nonunit"])
def test_random_transforms_match_the_restatement(gpu, kind):
    r = raster()
    rows, verts, count = custom_scenes(10 + len(kind))
    tf = transforms(20 + len(kind), kind)
    o, cnt, need, ov = gpu.costmap_obstacles(r["cost"], r["grid"], r["origin"], r["robot"], M_CAP, custom=rows,
                                             custom_count=count, custom_to_costmap=tf, custom_vertices=verts)
    d = run_device(gpu, r, rows, count, tf, verts)
    want_rows, want_verts = expect(rows, verts, count, tf)
    for s in range(S):
        assert cnt[s] == d[1][s] == need[s] and o[s, :cnt[s]].tobytes() == d[0][s, :cnt[s]].tobytes()
        assert o[s, cnt[s] - count[s]:cnt[s]].tobytes() == want_rows[s].tobytes(), s
    assert ov.tobytes() == d[3].tobytes() == want_verts.tobytes()
    closed = [w[3]["vertex_count"] for w in want_rows if len(w) > 3]
    assert closed and all(c == 5 for c in closed)                               # the closing vertex dropped


def test_argument_errors(gpu):
    r = raster()
    rows, verts, count = custom_scenes(3)
    tf = transforms(1, "planar")
    with pytest.raises(RuntimeError):      # Line / Polygon rows and no vertices
        gpu.costmap_obstacles(r["cost"], r["grid"], r["origin"], r["robot"], M_CAP, custom=rows, custom_count=count,
                              custom_to_costmap=tf)
    with pytest.raises(RuntimeError):      # vertices and no transform
        gpu.costmap_obstacles(r["cost"], r["grid"], r["origin"], r["robot"], M_CAP, custom=rows, custom_count=count,
                              custom_vertices=verts)
    # the device answers the scenes that need vertices with -1 and converts the others
    pts = rows.copy()
    only_points = np.zeros(S, bool)
    only_points[::3] = True
    for s in np.flatnonzero(only_points):
        pts[s]["type"] = fc.TEB_OBST_POINT
    o, cnt, need, _ = run_device(gpu, r, pts, count, tf, None)
    ref = gpu.costmap_obstacles(r["cost"], r["grid"], r["origin"], r["robot"], M_CAP, custom=pts, custom_count=count)
    for s in range(S):
        if only_points[s]:
            assert cnt[s] == need[s] == ref[1][s]
        else:
            assert cnt[s] == need[s] == -1
