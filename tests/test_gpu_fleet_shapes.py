"""The shaped fleet steps on the device (tebgpu_fleet_obstacles_shaped / _publish_shaped / _gather_shaped /
_obstacles_table_shaped, the FleetShaped writer of k_fleet_obstacles and k_fleet_obstacles_grid), held to
tests/fleet_shape_cases.py: on random fleets of mixed kinds, clustered and sparse, up to 8192 robots, every type, row
order, count, vertex range, needed, status and dynamic flag is the restatement's bit for bit, positions, vertices,
centroids and velocities within 1e-12 (the device's sincos); a kind of one circle at the origin writes the circle step's
bytes under every search; host and device forms and a second call give the same bytes; the caller's own rows and
vertices are untouched; uneven shards through the table equal one array call; argument errors write nothing. Then a fleet of two kinds (C3
TwoCircles robots and polygon robots) in two contexts, head-on in a corridor and at a junction, runs 20 control cycles
on one stream against the same loop fed host-restated rows, and the graph shows dynamic-obstacle edges for the moving
Polygon rows."""
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from teb_local_planner_b200 import distributed as D
from tests import fleet_shape_cases as fsc
from tests import fleet_table_cases as ftc
from tests.test_fleet_shape_cases import KINDS as HAND_KINDS
from tests.test_gpu_fleet_obstacles import IDENTITY, _raster, _straight_plans, random_fleet

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
MAX_R = 8192
SHARDS = 8
PV_CAP = 48
# the hand-computed kinds, a 40-point polygon (the writer's lanes place points 32 .. 39 in a second pass) and a kind of
# TEB_FLEET_MAX_PARTS parts
KINDS = HAND_KINDS + [
    [(abi.TEB_OBST_POLYGON, [[0.3 * math.cos(a), 0.2 * math.sin(a)] for a in np.arange(40) * (2 * math.pi / 40)])],
    [(abi.TEB_OBST_CIRCULAR, [[0.1 * i - 0.35, 0.05 * (i % 2)]], 0.05 + 0.01 * i) for i in range(7)]
    + [(abi.TEB_OBST_LINE, [[0.4, -0.2], [0.4, 0.2]])]]
EXACT = ("type", "dynamic", "vertex_begin", "vertex_count", "radius", "_pad")
CLOSE = ("x", "y", "vx", "vy")


@pytest.fixture(scope="module")
def ctxs():
    gs = [T.TebGpu(MAX_R, 8, MAX_R + 64, 64) for _ in range(SHARDS)]
    yield gs
    for g in gs:
        g.close()


def t(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def mixed_fleet(R, C_cap, seed, clustered=True):
    f = random_fleet(R, R, C_cap, seed, clustered=clustered)
    rng = np.random.default_rng(seed + 1)
    f["kind"] = rng.integers(0, len(KINDS), R).astype(np.int32)
    f["own_v"] = rng.integers(0, PV_CAP + 1, R).astype(np.int32)
    f["cv"] = rng.uniform(-9, 9, (R, PV_CAP, 2))
    return f


def dev(f):
    R = len(f["pose"])
    return dict(pose=t(f["pose"]), cmd=t(f["last_cmd"]), world=t(f["world"]), own=t(f["own_count"]),
                custom=t(f["custom"].view(np.uint8)), cc=torch.full((R,), -7, dtype=torch.int32, device=DEV),
                need=torch.full((R,), -9, dtype=torch.int32, device=DEV),
                st=torch.full((R,), -9, dtype=torch.int32, device=DEV), kind=t(f["kind"]), ownv=t(f["own_v"]),
                cv=t(f["cv"]))


def outputs(d, f):
    return (d["custom"].cpu().numpy().view(abi.OBST_DTYPE).reshape(f["custom"].shape), d["cc"].cpu().numpy(),
            d["need"].cpu().numpy(), d["st"].cpu().numpy(), d["cv"].cpu().numpy())


def args(d, lo, hi, C_cap, max_rows, rng, table=False):
    sl = lambda x: None if x is None else x[lo:hi]
    n = hi - lo
    fa = abi.make_fleet_args(n, n, C_cap, max_rows, rng, pose=None if table else sl(d["pose"]),
                             last_cmd=None if table else sl(d["cmd"]), world=None if table else sl(d["world"]),
                             own_count=sl(d["own"]), custom=sl(d["custom"]), custom_count=sl(d["cc"]),
                             needed=sl(d["need"]), status=sl(d["st"]))
    return fa


def shapes(d, lo, hi, **kw):
    sl = lambda x: None if x is None else x[lo:hi]
    return abi.make_fleet_shapes(KINDS, PV_CAP, kind=sl(d["kind"]), own_vertex_count=sl(d["ownv"]),
                                 custom_vertices=sl(d["cv"]), **kw)


def run_array(g, f, rng, max_rows, twice=False):
    d = dev(f)
    R, C_cap = f["custom"].shape
    fa, sh = args(d, 0, R, C_cap, max_rows, rng), shapes(d, 0, R)
    g.fleet_obstacles_shaped_device(fa, sh)
    torch.cuda.synchronize()
    out = outputs(d, f)
    if twice:
        g.fleet_obstacles_shaped_device(fa, sh)
        torch.cuda.synchronize()
        again = outputs(d, f)
        for a, b in zip(out, again):
            assert a.tobytes() == b.tobytes()
    return out


def assert_matches(got, want, f):
    custom, cc, need, st, cv = got
    wc, wcc, wneed, wst, wcv = want
    assert cc.tobytes() == wcc.tobytes() and need.tobytes() == wneed.tobytes() and st.tobytes() == wst.tobytes()
    for k in EXACT:
        assert custom[k].tobytes() == wc[k].tobytes(), k
    # the caller's own rows and vertices, and everything past the written ones, are the input's bytes
    R, C = custom.shape
    col = np.arange(C)[None, :]
    untouched = (col < f["own_count"][:, None]) | (col >= np.maximum(cc, f["own_count"])[:, None])
    assert custom[untouched].tobytes() == f["custom"][untouched].tobytes()
    assert np.abs(cv - wcv).max(initial=0.0) <= 1e-12
    # positions and velocities within 1e-12 (the device's sincos), except the polygon centroids: calcCentroid's cross
    # products of coordinates tens of metres from the origin cancel, so a last-bit difference of the placed points grows;
    # each centroid is instead exactly the restatement's calcCentroid of the points the device placed
    written = ~untouched
    poly = written & (custom["type"] == fsc.POLYGON)
    for k in CLOSE:
        sel = written & ~poly if k in ("x", "y") else written
        assert np.abs(custom[k][sel] - wc[k][sel]).max(initial=0.0) <= 1e-12, k
    for r, i in zip(*np.nonzero(poly)):
        o = custom[r, i]
        b = int(o["vertex_begin"])
        pts = [tuple(v) for v in cv[r, b:b + int(o["vertex_count"])]]
        assert (o["x"], o["y"]) == fsc.polygon_centroid(pts), (r, i)
        assert abs(o["x"] - wc[r, i]["x"]) <= 1e-9 and abs(o["y"] - wc[r, i]["y"]) <= 1e-9
    mine = np.arange(cv.shape[1])[None, :] < f["own_v"][:, None]
    assert cv[mine].tobytes() == f["cv"][mine].tobytes()


@pytest.mark.parametrize("R,clustered", [(1, True), (700, True), (3000, False), (MAX_R, True), (MAX_R, False)])
def test_random_mixed_fleets_match_the_restatement(ctxs, R, clustered):
    C_cap = 24
    f = mixed_fleet(R, C_cap, seed=R + clustered, clustered=clustered)
    g = ctxs[0]
    for k, (rng, max_rows) in enumerate(((3.0, 8), (6.0, 32), (math.inf, 4))):
        g.set_fleet_search((abi.TEBGPU_FLEET_SEARCH_AUTO, abi.TEBGPU_FLEET_SEARCH_ALL_PAIRS,
                            abi.TEBGPU_FLEET_SEARCH_GRID)[k])
        got = run_array(g, f, rng, max_rows, twice=k == 0)
        want = fsc.restate(f["pose"], f["last_cmd"], KINDS, f["kind"], rng, max_rows, f["custom"], f["cv"],
                           f["own_count"], None, f["own_v"], f["world"])
        assert_matches(got, want, f)
        if R > 1 and rng == 6.0:
            assert (got[3] == abi.TEB_FLEET_TRUNCATED).any() and (got[0]["type"] == abi.TEB_OBST_POLYGON).any()
            if R >= 700:                # the 40-point and the 8-part kinds were written
                assert (got[0]["vertex_count"] == 40).any() and (got[0]["type"] == abi.TEB_OBST_LINE).any()
    g.set_fleet_search(abi.TEBGPU_FLEET_SEARCH_AUTO)


def test_host_and_device_forms_give_the_same_bits(ctxs):
    R, C_cap = 900, 16
    f = mixed_fleet(R, C_cap, seed=4)
    g = ctxs[1]
    dv = run_array(g, f, 3.0, 8)
    host = g.fleet_obstacles_shaped(KINDS, f["kind"], f["pose"], f["last_cmd"], f["custom"], 3.0, 8,
                                    own_count=f["own_count"], world=f["world"], custom_vertices=f["cv"],
                                    own_vertex_count=f["own_v"])
    for a, b in zip(host, dv):
        assert a.tobytes() == b.tobytes()
    counts = [300, 1, 599]
    cap, first = D.fleet_layout(counts, 3)
    rows, head, rk = ftc.padding(3 * cap), np.zeros(3 * cap), np.zeros(3 * cap, np.int32)
    for k, (lo, hi) in enumerate(ftc.split(R, counts)):
        rows, head, rk = g.fleet_publish_shaped(KINDS, f["kind"][lo:hi], f["pose"][lo:hi], f["last_cmd"][lo:hi], 0.0,
                                                rows, head, rk, first[k], world=f["world"][lo:hi])
    rows, head, rk = g.fleet_gather_shaped(KINDS, rows, head, rk, 3 * cap)     # one rank: unchanged
    outs = [g.fleet_obstacles_table_shaped(KINDS, rows, head, rk, first[k], hi - lo, f["custom"][lo:hi], 3.0, 8,
                                           own_count=f["own_count"][lo:hi], custom_vertices=f["cv"][lo:hi],
                                           own_vertex_count=f["own_v"][lo:hi])
            for k, (lo, hi) in enumerate(ftc.split(R, counts))]
    for i in range(5):
        assert np.concatenate([o[i] for o in outs]).tobytes() == dv[i].tobytes(), i


@pytest.mark.parametrize("table", [False, True])
def test_one_circle_at_the_origin_writes_the_circle_steps_bytes(ctxs, table):
    R, C_cap, rho = 5000, 12, 0.35
    f = random_fleet(R, R, C_cap, seed=11)
    g = ctxs[2]
    kinds = [[(abi.TEB_OBST_CIRCULAR, [[0.0, 0.0]], rho)]]
    for mode in (abi.TEBGPU_FLEET_SEARCH_ALL_PAIRS, abi.TEBGPU_FLEET_SEARCH_GRID, abi.TEBGPU_FLEET_SEARCH_ONE_BUCKET):
        g.set_fleet_search(mode)
        outs = []
        for shaped in (False, True):
            custom, cc = t(f["custom"].view(np.uint8)), torch.full((R,), -7, dtype=torch.int32, device=DEV)
            need, st = (torch.full((R,), -9, dtype=torch.int32, device=DEV) for _ in range(2))
            keep = dict(pose=t(f["pose"]), cmd=t(f["last_cmd"]), rad=t(np.full(R, rho)), world=t(f["world"]),
                        own=t(f["own_count"]))       # held: the args keep only their addresses
            fa = abi.make_fleet_args(R, R, C_cap, 8, 4.0, pose=keep["pose"], last_cmd=keep["cmd"], radius=keep["rad"],
                                     world=keep["world"], own_count=keep["own"], custom=custom, custom_count=cc,
                                     needed=need, status=st)
            kind = torch.zeros(R, dtype=torch.int32, device=DEV)
            head, rk = torch.zeros(R, dtype=torch.float64, device=DEV), torch.zeros(R, dtype=torch.int32, device=DEV)
            sh = abi.make_fleet_shapes(kinds, 0, kind=kind, heading=head, row_kind=rk)
            rows = torch.zeros(R * 64, dtype=torch.uint8, device=DEV)
            tb = abi.make_fleet_table(R, 0, rows)
            if table:
                (g.fleet_publish_shaped_device(fa, sh, tb) if shaped else g.fleet_publish_device(fa, tb))
                (g.fleet_obstacles_table_shaped_device(fa, sh, tb) if shaped else g.fleet_obstacles_table_device(fa, tb))
            else:
                (g.fleet_obstacles_shaped_device(fa, sh) if shaped else g.fleet_obstacles_device(fa))
            torch.cuda.synchronize()
            assert g.last_fleet_search() == T.TebGpu.FLEET_SEARCHES[mode]
            outs.append([x.cpu().numpy().tobytes() for x in (custom, cc, need, st)])
        assert outs[0] == outs[1], mode
    g.set_fleet_search(abi.TEBGPU_FLEET_SEARCH_AUTO)


@pytest.mark.parametrize("R,clustered", [(700, True), (MAX_R, True), (MAX_R, False)])
def test_sharded_tables_equal_the_array_call(ctxs, R, clustered):
    C_cap = 20
    f = mixed_fleet(R, C_cap, seed=R + 2 * clustered, clustered=clustered)
    want = run_array(ctxs[0], f, 5.0, 8)
    for n in (1, 2, 3, 5, 8):
        cuts = np.sort(np.random.default_rng(n).integers(0, R + 1, n - 1))
        counts = np.diff(np.concatenate([[0], cuts, [R]])).astype(int).tolist()
        cap, first = D.fleet_layout(counts, n)
        Tn = n * cap
        d = dev(f)
        rows = t(ftc.padding(Tn).view(np.uint8))
        head = torch.full((Tn,), 7.0, dtype=torch.float64, device=DEV)
        rk = torch.full((Tn,), -1, dtype=torch.int32, device=DEV)
        parts = ftc.split(R, counts)
        zero = torch.zeros(R, dtype=torch.float64, device=DEV)
        for k, (lo, hi) in enumerate(parts):
            if hi > lo:
                fa = args(d, lo, hi, C_cap, 8, 5.0)
                fa.radius = zero.data_ptr()
                ctxs[k].fleet_publish_shaped_device(fa, shapes(d, lo, hi, heading=head, row_kind=rk),
                                                    abi.make_fleet_table(Tn, first[k], rows))
        for k, (lo, hi) in enumerate(parts):
            if hi > lo:
                ctxs[k].fleet_obstacles_table_shaped_device(args(d, lo, hi, C_cap, 8, 5.0, table=True),
                                                            shapes(d, lo, hi, heading=head, row_kind=rk),
                                                            abi.make_fleet_table(Tn, first[k], rows))
        torch.cuda.synchronize()
        for a, b in zip(outputs(d, f), want):
            assert a.tobytes() == b.tobytes(), counts


def test_argument_errors_write_nothing(ctxs):
    R, C_cap = 30, 6
    f = mixed_fleet(R, C_cap, seed=2)
    g = ctxs[0]
    d = dev(f)
    before = {k: v.clone() for k, v in d.items() if v is not None}
    fa = args(d, 0, R, C_cap, 8, 3.0)
    bad_libraries = [[], [[]], [[(abi.TEB_OBST_POLYGON, [[0, 0], [1, 0]])]],
                     [[(abi.TEB_OBST_POLYGON, [[0, 0], [1, 0], [1, 1], [0, 0]])]],
                     [[(abi.TEB_OBST_CIRCULAR, [[0, 0]], 0.0)]], [[(abi.TEB_OBST_LINE, [[0, 0], [1, 0], [2, 0]])]],
                     [[(abi.TEB_OBST_PILL, [[0, 0], [1, 0]])]], [[(abi.TEB_OBST_POINT, [[0.0, 0.0]])] * 9],
                     [[(abi.TEB_OBST_POINT, [[math.nan, 0.0]])]],
                     [[(abi.TEB_OBST_POLYGON, [[math.cos(a), math.sin(a)] for a in np.linspace(0, 6, 65)])]],
                     [[(abi.TEB_OBST_POINT, [[0.0, 0.0]])]] * 257]
    for lib in bad_libraries:
        sh = abi.make_fleet_shapes(lib, PV_CAP, kind=d["kind"], own_vertex_count=d["ownv"], custom_vertices=d["cv"])
        with pytest.raises(T.TebGpuError):
            g.fleet_obstacles_shaped_device(fa, sh)
    small = abi.make_fleet_shapes(KINDS, 5, kind=d["kind"], custom_vertices=d["cv"])       # a 6-point polygon
    with pytest.raises(T.TebGpuError):
        g.fleet_obstacles_shaped_device(fa, small)
    with pytest.raises(T.TebGpuError):                                                     # no kind array
        g.fleet_obstacles_shaped_device(fa, abi.make_fleet_shapes(KINDS, PV_CAP, custom_vertices=d["cv"]))
    with pytest.raises(T.TebGpuError):                                                     # no vertex pool
        g.fleet_obstacles_shaped_device(fa, abi.make_fleet_shapes(KINDS, PV_CAP, kind=d["kind"]))
    torch.cuda.synchronize()
    for k, v in before.items():
        assert torch.equal(v, d[k]), k
    kind = f["kind"].copy()
    kind[3] = len(KINDS)                                                                   # a kind out of range
    with pytest.raises(T.TebGpuError):
        g.fleet_obstacles_shaped(KINDS, kind, f["pose"], f["last_cmd"], f["custom"], 3.0, 8, custom_vertices=f["cv"])
    # the host forms check scenes before they read own_vertex_count through them
    for bad in (-1, R):
        scene = np.arange(R, dtype=np.int32)
        scene[5] = bad
        with pytest.raises(T.TebGpuError):
            g.fleet_obstacles_shaped(KINDS, f["kind"], f["pose"], f["last_cmd"], f["custom"], 3.0, 8, scene=scene,
                                     custom_vertices=f["cv"], own_vertex_count=f["own_v"])
        rows = ftc.table([ftc.publish(f["pose"], f["last_cmd"], 0.0, f["world"])], R)
        with pytest.raises(T.TebGpuError):
            g.fleet_obstacles_table_shaped(KINDS, rows, f["pose"][:, 2], f["kind"], 0, R, f["custom"], 3.0, 8,
                                           scene=scene, custom_vertices=f["cv"], own_vertex_count=f["own_v"])
    # on the device a neighbour of an unknown kind ends its robot's list
    d["kind"][3] = len(KINDS)
    g.fleet_obstacles_shaped_device(fa, shapes(d, 0, R))
    torch.cuda.synchronize()
    f2 = dict(f, kind=d["kind"].cpu().numpy())
    want = fsc.restate(f["pose"], f["last_cmd"], KINDS, f2["kind"], 3.0, 8, f["custom"], f["cv"], f["own_count"], None,
                       f["own_v"], f["world"])
    assert_matches(outputs(d, f), want, f)


# ---- two ranks over NCCL, one GPU each
NCCL_R, NCCL_C = 2000, 12


def _nccl_worker(rank, world, port, out_dir, counts):
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch
    import torch.distributed as dist
    import teb_local_planner_b200 as T
    from teb_local_planner_b200 import abi
    from teb_local_planner_b200 import distributed as D
    from tests import fleet_table_cases as ftc
    from tests.test_gpu_fleet_shapes import KINDS
    from tests.test_gpu_fleet_shapes import PV_CAP, mixed_fleet
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("gloo", rank=rank, world_size=world)
    f = mixed_fleet(NCCL_R, NCCL_C, seed=21)
    g = T.TebGpu(NCCL_R, 8, NCCL_R, 8, device=rank)
    D.init_comm(g, rank, world)
    cap, first = D.fleet_layout(counts, world)
    lo, hi = ftc.split(NCCL_R, counts)[rank]
    n = hi - lo
    tt = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    rows = tt(ftc.padding(world * cap).view(np.uint8))
    head = torch.zeros(world * cap, dtype=torch.float64, device=dev)
    rk = torch.zeros(world * cap, dtype=torch.int32, device=dev)
    out = dict(custom=tt(f["custom"][lo:hi].view(np.uint8)), cv=tt(f["cv"][lo:hi]))
    out.update({k: torch.full((n,), -7, dtype=torch.int32, device=dev) for k in ("cc", "need", "st")})
    keep = {k: tt(f[k][lo:hi]) for k in ("pose", "last_cmd", "world", "own_count", "kind", "own_v")}
    keep["radius"] = tt(np.zeros(n))
    fa = abi.make_fleet_args(n, n, NCCL_C, 8, 4.0, pose=keep["pose"], last_cmd=keep["last_cmd"], radius=keep["radius"],
                             world=keep["world"], own_count=keep["own_count"], custom=out["custom"],
                             custom_count=out["cc"], needed=out["need"], status=out["st"])
    sh = abi.make_fleet_shapes(KINDS, PV_CAP, kind=keep["kind"], own_vertex_count=keep["own_v"],
                               custom_vertices=out["cv"], heading=head, row_kind=rk)
    tb = abi.make_fleet_table(world * cap, first[rank], rows)
    g.fleet_publish_shaped_device(fa, sh, tb)
    g.fleet_gather_shaped_device(sh, tb, cap)
    g.fleet_obstacles_table_shaped_device(fa, sh, tb)
    torch.cuda.synchronize()
    for name, x in out.items():
        np.save(os.path.join(out_dir, f"{name}_{rank}.npy"), x.cpu().numpy())
    g.comm_destroy()
    g.close()
    dist.destroy_process_group()


def test_two_ranks_gather_over_nccl_and_equal_the_array_call(ctxs, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("the two-rank NCCL gather of the shaped table needs 2 GPUs; this machine has fewer")
    import multiprocessing
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    world, counts = 2, [1200, 800]
    mpc = multiprocessing.get_context("spawn")
    procs = [mpc.Process(target=_nccl_worker, args=(r, world, port, str(tmp_path), counts)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=240)
    alive = [p for p in procs if p.is_alive()]
    for p in alive:
        p.terminate()
        p.join()
    assert not alive and all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    f = mixed_fleet(NCCL_R, NCCL_C, seed=21)
    want = run_array(ctxs[0], f, 4.0, 8)
    got = [np.concatenate([np.load(tmp_path / f"{k}_{r}.npy") for r in range(world)]) for k in ("custom", "cc", "need",
                                                                                                 "st", "cv")]
    for a, b in zip(got, want):
        assert a.tobytes() == np.asarray(b).view(a.dtype).reshape(a.shape).tobytes()


# ---- a fleet of two kinds on one stream, each kind published as its footprint
LOOP_PV = 16


def _loop_kind_params(k):
    """kind 0: C3, the car-like robot with its TwoCircles footprint; kind 1: a robot with a 0.5 x 0.3 m polygon"""
    if k == 0:
        p = scenes.config_params("C3")
        p.footprint_type = abi.TEB_FOOTPRINT_TWO_CIRCLES
        p.footprint_front_offset, p.footprint_front_radius = 0.2, 0.2
        p.footprint_rear_offset, p.footprint_rear_radius = 0.2, 0.2
    else:
        p = scenes.config_params("C2")
        p.footprint_type, p.footprint_vertex_count = abi.TEB_FOOTPRINT_POLYGON, 4
        p.footprint_vertices[:8] = [0.25, 0.15, -0.25, 0.15, -0.25, -0.15, 0.25, -0.15]
    p.include_dynamic_obstacles = 1
    p.max_vel_trans = p.max_vel_x
    p.global_plan_overwrite_orientation = 1
    return p


def _loop_scenario(kind):
    """corridor: a C3 robot and a polygon robot head-on; junction: two C3 robots crossing along x, two polygon robots
    along y. Robots of kind 0 first, so each kind's robots are one contiguous shard."""
    if kind == "corridor":
        start, goal, counts = np.array([[-1.5, 0.05], [1.5, -0.05]]), np.array([[3.0, 0.05], [-3.0, -0.05]]), (1, 1)
    else:
        start = np.array([[-1.5, 0.1], [1.5, -0.1], [0.1, 1.5], [-0.1, -1.5]])
        goal, counts = -3.0 * start / 1.5, (2, 2)
    gp, begin, end = _straight_plans(start, goal, 256)
    return dict(gp=gp, begin=begin, end=end, robot=np.column_stack([start, gp[:, 0, 2]]), G_cap=256, counts=counts,
                raster=_raster(len(start), start, kind))


def _shaped_loop(scenario, restated, cycles=20, n_cap=96, P_cap=128, M_cap=2048, Lb=10, max_rows=8, rng=3.0,
                 dev_trace=None, graph_at=None):
    """restated=False: every kind's context publishes its robots with their footprints into one table, then steps its
    robots against it; then each context runs costmap_tf (rows and vertices moved) -> local_plan_tf -> backup modes ->
    plan -> costmap check -> finish, all on one stream. True: the fleet steps replaced by the host restatement over the
    whole fleet, uploaded in their place; a restated position, vertex or velocity within the bars of assert_matches of
    the device's at the same cycle is replaced by the device's bits, so both loops see the same inputs."""
    sc = _loop_scenario(scenario)
    B = len(sc["robot"])
    C_cap, PV = 1 + 2 * max_rows, LOOP_PV
    kinds = [abi.fleet_shape_from_params(_loop_kind_params(k)) for k in range(2)]
    kind_of = np.repeat(np.arange(2), sc["counts"]).astype(np.int32)
    r = sc["raster"]
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    z = lambda shape, dtp: torch.zeros(shape, dtype=dtp, device=DEV)
    f64, i32 = torch.float64, torch.int32
    cost, grid, origin = t(r["cost"]), t(r["grid"]), t(r["origin"])
    robot = t(sc["robot"].copy())
    radius, kindt = t(np.zeros(B)), t(kind_of)
    own_rows = np.zeros((B, C_cap), abi.OBST_DTYPE)     # one static point of the caller's own per scene, far behind
    own_rows[:, 0]["x"], own_rows[:, 0]["y"] = sc["robot"][:, 0] - 5.0, sc["robot"][:, 1] + 5.0
    custom, ccount, own = t(own_rows.view(np.uint8)), t(np.ones(B, np.int32)), t(np.ones(B, np.int32))
    cv, ov = z((B, PV, 2), f64), z((B, PV, 2), f64)
    last_cmd, fneed, fstat = z((B, 3), f64), z(B, i32), z(B, i32)
    gpd, begin, end = t(sc["gp"]), t(sc["begin"]), t(sc["end"])
    vel, cmd_vel = z((B, 3), f64), z((B, 3), f64)
    cap, first = D.fleet_layout(list(sc["counts"]), 2)
    rows = t(ftc.padding(2 * cap).view(np.uint8))
    head, rkind = z(2 * cap, f64), z(2 * cap, i32)
    ctx = []
    lo = 0
    for k, n in enumerate(sc["counts"]):
        hi = lo + n
        sl = slice(lo, hi)
        p = _loop_kind_params(k)
        g = T.TebGpu(n, n_cap, n, M_cap, 0, max_obst_vertices=PV)
        g.set_params(p)
        state = {kk: t(v) for kk, v in abi.make_cycle_state(n, Lb).items()}
        state["last_cmd"] = last_cmd[sl]
        K = dict(g=g, p=p, sl=sl, n=n, state=state, plan=z((n, P_cap, 3), f64), pcount=z(n, i32), result=z(n, i32),
                 gidx=z(n, i32), needed=z((n, 2), i32), since=z(n, f64), poses=z((n, n_cap, 4), f64), nn=z(n, i32),
                 sid=t(np.arange(n, dtype=np.int32)), obst=z(n * M_cap * 64, torch.uint8), ocount=z(n, i32),
                 costo=z(n, f64), chi2=z(n, f64), status=z(n, i32), iters=z(n, i32), cmd=z((n, 4), f64),
                 path=z(n, i32), feas=z(n, i32), qc=z(n, i32), outcome=z(n, i32), osc=z(n, i32),
                 ident=t(np.tile(IDENTITY, (n, 1))))
        vs = np.zeros((n, 4))
        vs[:, 3] = 1.0
        K["vs"], K["vstart"], K["vgoal"] = vs, t(vs), t(vs)
        bs = abi.TebBatch()
        bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = n, n_cap, n, M_cap, 0, PV
        bs.poses, bs.n, bs.scene_id = K["poses"].data_ptr(), K["nn"].data_ptr(), K["sid"].data_ptr()
        bs.obstacles, bs.obst_count, bs.obst_vertices = K["obst"].data_ptr(), K["ocount"].data_ptr(), ov[sl].data_ptr()
        bs.vel_start, bs.vel_goal, bs.prefer_rotdir = K["vstart"].data_ptr(), K["vgoal"].data_ptr(), state["prefer_rotdir"].data_ptr()
        bs.cost, bs.chi2, bs.status, bs.lm_iters = (K["costo"].data_ptr(), K["chi2"].data_ptr(), K["status"].data_ptr(),
                                                     K["iters"].data_ptr())
        K["bs"] = bs
        ca = abi.TebCostmapArgs()
        ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = n, r["cost"].shape[1], M_cap, C_cap, 1
        ca.behind_robot_dist = 1.5
        ca.cost, ca.grid, ca.origin, ca.robot = cost[sl].data_ptr(), grid[sl].data_ptr(), origin[sl].data_ptr(), robot[sl].data_ptr()
        ca.custom, ca.custom_count = custom[sl].data_ptr(), ccount[sl].data_ptr()
        ca.obstacles, ca.obst_count = K["obst"].data_ptr(), K["ocount"].data_ptr()
        K["ca"] = ca
        K["cframes"] = abi.make_frame_args(custom_to_costmap=K["ident"].data_ptr(), custom_vertices=cv[sl].data_ptr(),
                                           obst_vertices=ov[sl].data_ptr(), PV_cap=PV)
        K["pframes"] = abi.make_frame_args(costmap_to_plan=K["ident"].data_ptr(), plan_to_costmap=K["ident"].data_ptr())
        K["la"] = abi.make_local_plan_args(sc["G_cap"], P_cap, 0, max_lookahead_dist=2.0, global_plan=gpd[sl].data_ptr(),
                                           plan_begin=begin[sl].data_ptr(), plan_end=end[sl].data_ptr(),
                                           robot=robot[sl].data_ptr(), robot_vel=vel[sl].data_ptr(),
                                           grid=grid[sl].data_ptr(), origin=origin[sl].data_ptr(),
                                           infeasible_count=state["infeasible_count"].data_ptr(),
                                           since_infeasible=K["since"].data_ptr(), plan=K["plan"].data_ptr(),
                                           plan_count=K["pcount"].data_ptr(), goal_idx=K["gidx"].data_ptr(),
                                           result=K["result"].data_ptr(), needed=K["needed"].data_ptr())
        K["args"] = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0,
                                  False)
        K["fa"] = abi.make_feasibility_args(0.1, max_queries=512, feasible=K["feas"].data_ptr(),
                                            query_count=K["qc"].data_ptr())
        K["world"] = abi.make_costmap_world(r["cost"].shape[1], cost[sl].data_ptr(), grid[sl].data_ptr(),
                                            origin[sl].data_ptr())
        K["fl"] = abi.make_fleet_args(n, n, C_cap, max_rows, rng, pose=robot[sl], last_cmd=last_cmd[sl],
                                      radius=radius[sl], own_count=own[sl], custom=custom[sl], custom_count=ccount[sl],
                                      needed=fneed[sl], status=fstat[sl])
        K["sh"] = abi.make_fleet_shapes(kinds, PV, kind=kindt[sl], custom_vertices=cv[sl], heading=head, row_kind=rkind)
        K["tb"] = abi.make_fleet_table(2 * cap, first[k], rows)
        ctx.append(K)
        lo = hi
    cs = dict(buffer_length=Lb, oscillation_recovery_min_duration=2.0)
    dt, now = 0.2, 1000.0
    s = torch.cuda.Stream()
    trace, graphs = [], []
    for c in range(cycles):
        with torch.cuda.stream(s):
            if restated:
                s.synchronize()
                cur = custom.cpu().numpy().view(abi.OBST_DTYPE).reshape(B, C_cap).copy()
                hc, hcc, hn, hs, hv = fsc.restate(robot.cpu().numpy(), last_cmd.cpu().numpy(), kinds, kind_of, rng,
                                                  max_rows, cur, cv.cpu().numpy(), np.ones(B, np.int32))
                d = dev_trace[c]
                dc = d["custom"].view(abi.OBST_DTYPE).reshape(B, C_cap)
                assert_matches((dc, d["ccount"], d["fneed"], d["fstat"], d["cv"]), (hc, hcc, hn, hs, hv),
                               dict(custom=cur, own_count=np.ones(B, np.int32), own_v=np.zeros(B, np.int32),
                                    cv=cv.cpu().numpy()))
                for key in CLOSE:          # within the bars: take the device's bits
                    hc[key] = dc[key]
                hv = d["cv"]
                custom.copy_(t(hc.view(np.uint8).reshape(B, -1)))
                cv.copy_(t(hv))
                ccount.copy_(t(hcc))
                fneed.copy_(t(hn))
                fstat.copy_(t(hs))
            else:
                for K in ctx:
                    K["g"].fleet_publish_shaped_device(K["fl"], K["sh"], K["tb"], stream=s.cuda_stream)
                for K in ctx:
                    K["g"].fleet_obstacles_table_shaped_device(K["fl"], K["sh"], K["tb"], stream=s.cuda_stream)
            for K in ctx:
                g, st, sl = K["g"], K["state"], K["sl"]
                cy = abi.make_cycle_args(now, L_cap=Lb, **cs, local_plan_result=K["result"].data_ptr(),
                                         robot_vel=vel[sl].data_ptr(), cmd=K["cmd"].data_ptr(),
                                         feasible=K["feas"].data_ptr(), cmd_vel=cmd_vel[sl].data_ptr(),
                                         outcome=K["outcome"].data_ptr(), oscillating=K["osc"].data_ptr(),
                                         **{kk: st[kk].data_ptr() for kk in abi.CYCLE_STATE})
                K["since"].copy_(now - st["last_infeasible"])
                g.costmap_obstacles_device(K["ca"], stream=s.cuda_stream, frames=K["cframes"])
                g.local_plan_device(K["bs"], K["la"], stream=s.cuda_stream, frames=K["pframes"])
                g.backup_modes_device(K["bs"], cy, stream=s.cuda_stream)
                g.plan_device(K["bs"], K["args"], K["cmd"], initial_plan=K["plan"], plan_count=K["pcount"],
                              P_cap=P_cap, path=K["path"], stream=s.cuda_stream)
                g.check_feasible_costmap_device(K["bs"], K["fa"], K["world"], stream=s.cuda_stream)
                g.finish_cycle_device(K["bs"], cy, stream=s.cuda_stream)
        s.synchronize()
        if graph_at == c:                  # on contexts of their own, so the loop's contexts are the restated loop's
            for k, K in enumerate(ctx):
                n = K["n"]
                hb = abi.HostBatch(K["poses"].cpu().numpy(), K["nn"].cpu().numpy(),
                                   K["obst"].cpu().numpy().view(abi.OBST_DTYPE).reshape(n, M_cap),
                                   K["ocount"].cpu().numpy(), scene_id=np.arange(n, dtype=np.int32), vel_start=K["vs"],
                                   vel_goal=K["vs"], prefer_rotdir=K["state"]["prefer_rotdir"].cpu().numpy(),
                                   obst_vertices=ov[K["sl"]].cpu().numpy())
                g2 = T.TebGpu(n, n_cap, n, M_cap, 0, max_obst_vertices=PV)
                g2.set_params(K["p"])
                graphs.append((k, hb, g2.build_system(hb, graph=True)))
                g2.close()
        with torch.cuda.stream(s):
            th = robot[:, 2].clone()
            robot[:, 0] += (cmd_vel[:, 0] * torch.cos(th) - cmd_vel[:, 1] * torch.sin(th)) * dt
            robot[:, 1] += (cmd_vel[:, 0] * torch.sin(th) + cmd_vel[:, 1] * torch.cos(th)) * dt
            robot[:, 2] += cmd_vel[:, 2] * dt
            vel.copy_(cmd_vel)
        s.synchronize()
        rec = dict(custom=custom, ccount=ccount, fneed=fneed, fstat=fstat, cv=cv, ov=ov, robot=robot, cmd_vel=cmd_vel,
                   last_cmd=last_cmd)
        for k, K in enumerate(ctx):
            for key in ("obst", "ocount", "pcount", "result", "nn", "poses", "status", "path", "cmd", "outcome", "osc",
                        "feas"):
                rec[f"{key}{k}"] = K[key]
            for key, v in K["state"].items():
                rec[f"{key}{k}"] = v
        rec = {key: v.cpu().numpy().copy() for key, v in rec.items()}
        for k, K in enumerate(ctx):
            pc, pl = rec[f"pcount{k}"], K["plan"].cpu().numpy()
            rec[f"plan{k}"] = np.concatenate([pl[b, :pc[b]] for b in range(K["n"])])
        trace.append(rec)
        now += dt
    for K in ctx:
        K["g"].close()
    return trace, graphs


@pytest.mark.parametrize("scenario", ["corridor", "junction"])
def test_a_two_kind_footprint_loop_matches_the_loop_fed_host_restated_rows(scenario):
    dev, graphs = _shaped_loop(scenario, False, graph_at=3)
    ref, _ = _shaped_loop(scenario, True, dev_trace=dev)
    for c, (x, y) in enumerate(zip(dev, ref)):
        assert x.keys() == y.keys()
        for key in x:
            assert x[key].tobytes() == y[key].tobytes(), (scenario, c, key)
    B = len(dev[0]["ccount"])
    counts = _loop_scenario(scenario)["counts"]
    kind_of = np.repeat(np.arange(2), counts)
    # every robot sees the other kind as its footprint: the C3 robots as two circles, the polygon robots as a polygon
    seen = set()
    for c in dev:
        rows = c["custom"].view(abi.OBST_DTYPE).reshape(B, -1)
        for b in range(B):
            types = set(rows[b, 1:c["ccount"][b]]["type"].tolist())
            seen |= {(int(kind_of[b]), ty) for ty in types}
    assert (0, abi.TEB_OBST_POLYGON) in seen and (1, abi.TEB_OBST_CIRCULAR) in seen, seen
    assert sum((c[f"outcome{k}"] == abi.TEB_CYCLE_COMMAND).sum() for c in dev for k in (0, 1)) > 0
    # the moving polygon rows give dynamic-obstacle edges in the graph of the C3 robots: every interior pose of a band
    # whose table holds one has a time, and the dynamic rows take no static association bit
    hit = 0
    for k, hb, gr in graphs:
        for b in range(len(hb.n)):
            nb, cnt = int(hb.n[b]), int(hb.obst_count[b])
            rows = hb.obstacles[b, :cnt]
            dyn = np.nonzero(rows["dynamic"] == 1)[0]
            vertex_rows = [l for l in dyn if rows[l]["type"] in (abi.TEB_OBST_LINE, abi.TEB_OBST_POLYGON)]
            if nb < 3 or not vertex_rows:
                continue
            hit += 1
            assert np.isfinite(gr["dyn_t"][b, 1:nb - 1]).all(), (scenario, k, b)
            words = gr["assoc"][b, :nb]
            for l in dyn:
                assert not ((words[:, l // 64] >> np.uint64(l % 64)) & np.uint64(1)).any(), (scenario, k, b, l)
    assert hit > 0, "no band of the graph cycle had a dynamic Polygon row"
