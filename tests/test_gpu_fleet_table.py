"""The fleet table on the device (tebgpu_fleet_publish / _gather / _obstacles_table, k_fleet_publish and the table build
of k_fleet_obstacles), held to tebgpu_fleet_obstacles on the whole fleet: a fleet split into contiguous uneven shards,
each shard in a context of its own, all publishing into one padded table and stepping against it, writes the same
bytes as one call over the union; the host and device forms give the same bits; a robot whose own row is padding gets
BAD_INPUT and argument errors write nothing; the gather leaves the table as it is with one rank and joins two ranks'
shards over NCCL. Then a fleet of two robot kinds in two contexts (a circular robot and a car-like TwoCircles robot)
runs 20 control cycles on one stream against the same loop fed by one union tebgpu_fleet_obstacles call."""
import math
import multiprocessing
import os
import sys

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from teb_local_planner_b200 import distributed as D
from tests import fleet_cases as fc
from tests import fleet_table_cases as ftc
from tests.test_gpu_fleet_obstacles import IDENTITY, _raster, _straight_plans, random_fleet

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
MAX_R = 8192
SHARDS = 8
ROW_BYTES = abi.FLEET_ROW_DTYPE.itemsize


@pytest.fixture(scope="module")
def ctxs():
    gs = [T.TebGpu(MAX_R, 8, MAX_R + 64, 64) for _ in range(SHARDS)]
    yield gs
    for g in gs:
        g.close()


def t(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def uneven_counts(R, n, seed):
    """n contiguous shards of R robots, sizes uneven (a shard may hold one robot or none)"""
    if n == 1:
        return [R]
    cuts = np.sort(np.random.default_rng(seed).integers(0, R + 1, n - 1))
    return np.diff(np.concatenate([[0], cuts, [R]])).astype(int).tolist()


def padded_table(T_rows, f, seed):
    """a device table whose rows are padding (live 0) on top of random robots of f, in their worlds"""
    rng = np.random.default_rng(seed)
    pad = np.zeros(T_rows, abi.FLEET_ROW_DTYPE)
    pick = rng.integers(0, len(f["pose"]), T_rows)
    pad["x"], pad["y"] = f["pose"][pick, 0], f["pose"][pick, 1]
    pad["radius"], pad["dynamic"] = 0.3, 1
    pad["world"] = 0 if f.get("world") is None else f["world"][pick]
    return t(pad.view(np.uint8))


def dev_fleet(f, S=None):
    R = len(f["pose"])
    S = R if S is None else S
    return dict(pose=t(f["pose"]), cmd=t(f["last_cmd"]), rad=t(np.broadcast_to(f["radius"], (R,))), world=t(f.get("world")),
                own=t(f.get("own_count")), custom=t(f["custom"].view(np.uint8)),
                cc=torch.full((S,), -7, dtype=torch.int32, device=DEV),
                need=torch.full((R,), -9, dtype=torch.int32, device=DEV),
                st=torch.full((R,), -9, dtype=torch.int32, device=DEV))


def outputs(d, f):
    return (d["custom"].cpu().numpy().view(abi.OBST_DTYPE).reshape(f["custom"].shape), d["cc"].cpu().numpy(),
            d["need"].cpu().numpy(), d["st"].cpu().numpy())


def run_union(g, f, rng, max_rows, stream=None):
    d = dev_fleet(f)
    R, C_cap = f["custom"].shape
    fa = abi.make_fleet_args(R, R, C_cap, max_rows, rng, pose=d["pose"], last_cmd=d["cmd"], radius=d["rad"],
                             world=d["world"], own_count=d["own"], custom=d["custom"], custom_count=d["cc"],
                             needed=d["need"], status=d["st"])
    g.fleet_obstacles_device(fa, stream=stream)
    torch.cuda.synchronize()
    return outputs(d, f)


def shard_args(d, lo, hi, C_cap, max_rows, rng):
    """TebFleetArgs of the robots [lo, hi) of the device fleet d, each writing its own scene"""
    n = hi - lo
    sl = lambda x: None if x is None else x[lo:hi]
    return abi.make_fleet_args(n, n, C_cap, max_rows, rng, pose=sl(d["pose"]), last_cmd=sl(d["cmd"]), radius=sl(d["rad"]),
                               world=sl(d["world"]), own_count=sl(d["own"]), custom=sl(d["custom"]),
                               custom_count=sl(d["cc"]), needed=sl(d["need"]), status=sl(d["st"]))


def run_sharded(gs, f, counts, rng, max_rows, seed=0, stream=None):
    """every shard publishes into one padded device table on its own context, then every shard steps against it, on
    one stream. Returns (outputs, table rows as FLEET_ROW_DTYPE, first per shard)."""
    R, C_cap = f["custom"].shape
    cap, first = D.fleet_layout(counts, len(counts))
    rows = padded_table(len(counts) * cap, f, seed)
    d = dev_fleet(f)
    parts = ftc.split(R, counts)
    for g, (lo, hi) in enumerate(parts):
        if hi > lo:
            gs[g].fleet_publish_device(shard_args(d, lo, hi, C_cap, max_rows, rng),
                                       abi.make_fleet_table(len(counts) * cap, first[g], rows), stream=stream)
    for g, (lo, hi) in enumerate(parts):
        if hi > lo:
            gs[g].fleet_obstacles_table_device(shard_args(d, lo, hi, C_cap, max_rows, rng),
                                               abi.make_fleet_table(len(counts) * cap, first[g], rows), stream=stream)
    torch.cuda.synchronize()
    return outputs(d, f), rows.cpu().numpy().view(abi.FLEET_ROW_DTYPE), first


ROW_KEYS = ("x", "y", "vx", "vy", "radius", "dynamic")


def assert_rows_are_published_rows(union, f, rng, max_rows, tab, counts, first, sample=300):
    """the rows the union step wrote for a sample of robots are, field by field, the published rows of their robots"""
    custom, cc, need, _ = union
    own = np.zeros(len(f["pose"]), np.int64) if f.get("own_count") is None else f["own_count"]
    row_of = np.concatenate([first[g] + np.arange(n) for g, n in enumerate(counts)]).astype(int)
    for r in np.random.default_rng(1).permutation(len(f["pose"]))[:sample]:
        idx, _ = fc.neighbours(f["pose"], r, rng, f.get("world"))
        for i in range(int(cc[r] - own[r])):
            o, w = custom[r, own[r] + i], tab[row_of[idx[i]]]
            for k in ROW_KEYS:
                assert np.asarray(o[k]).tobytes() == np.asarray(w[k]).astype(o[k].dtype).tobytes(), (r, i, k)


@pytest.mark.parametrize("R,clustered", [(1, True), (700, True), (3000, False), (MAX_R, True), (MAX_R, False)])
def test_sharded_fleets_write_what_the_union_call_writes(ctxs, R, clustered):
    C_cap = 24
    f = random_fleet(R, R, C_cap, seed=R + clustered, worlds=3, clustered=clustered)
    s = torch.cuda.Stream()
    for k, n in enumerate((1, 2, 3, 5, 8)):
        counts = uneven_counts(R, n, seed=R + k)
        for max_rows in (0, 8, 32):
            rng = (1.5, 6.0, math.inf)[k % 3]
            want = run_union(ctxs[0], f, rng, max_rows, stream=s.cuda_stream)
            got, tab, first = run_sharded(ctxs, f, counts, rng, max_rows, seed=k, stream=s.cuda_stream)
            for a, b, name in zip(got, want, ("custom", "custom_count", "needed", "status")):
                assert a.tobytes() == b.tobytes(), (name, R, counts, max_rows, rng)
            live = np.concatenate([np.arange(first[g], first[g] + c) for g, c in enumerate(counts)]).astype(int)
            assert (tab["live"][live] == 1).all() and tab["live"].sum() == R
            if max_rows and R > 1:
                assert_rows_are_published_rows(want, f, rng, max_rows, tab, counts, first)
            if R > 1 and rng == 6.0:
                assert (want[2] > 0).any()
            for g, cnt in enumerate(counts):
                if cnt:
                    assert ctxs[g].last_fleet_grid() == (cnt + 15) // 16


def test_host_and_device_forms_give_the_same_bits(ctxs):
    R, C_cap = 900, 16
    f = random_fleet(R, R, C_cap, seed=4)
    counts = [300, 1, 599]
    (dev, tab, first) = run_sharded(ctxs, f, counts, 3.0, 8)
    g = ctxs[1]
    host_tab = ftc.padding(len(tab))
    host_tab[:] = tab
    host_tab["live"] = 0
    for k, (lo, hi) in enumerate(ftc.split(R, counts)):
        host_tab = g.fleet_publish(f["pose"][lo:hi], f["last_cmd"][lo:hi], f["radius"][lo:hi], host_tab, first[k],
                                   world=f["world"][lo:hi])
    assert host_tab.tobytes() == tab.tobytes()
    for k, (lo, hi) in enumerate(ftc.split(R, counts)):
        out = g.fleet_obstacles_table(host_tab, first[k], hi - lo, f["custom"][lo:hi], 3.0, 8,
                                      own_count=f["own_count"][lo:hi])
        for a, b, name in zip(out, (dev[0][lo:hi], dev[1][lo:hi], dev[2][lo:hi], dev[3][lo:hi]), ("custom", "cc", "need", "st")):
            assert a.tobytes() == b.tobytes(), name
    # the restatement agrees too, and the published rows are the restatement's rows bit for bit
    want = ftc.restate(tab, first[2], 599, 3.0, 8, f["custom"][301:], f["own_count"][301:])
    assert want[2].tobytes() == dev[2][301:].tobytes() and want[3].tobytes() == dev[3][301:].tobytes()
    pub = ftc.publish(f["pose"], f["last_cmd"], f["radius"], f["world"])
    for k in ("x", "y", "radius", "dynamic", "world", "live"):
        assert np.array_equal(tab[first[2]:first[2] + 599][k], pub[301:][k]), k


def test_a_robot_whose_own_row_is_padding_gets_bad_input(ctxs):
    R, C_cap = 40, 6
    f = random_fleet(R, R, C_cap, seed=7, worlds=1)
    g = ctxs[0]
    rows = ftc.table([ftc.publish(f["pose"], f["last_cmd"], f["radius"])], R)
    rows["live"][[3, 17]] = 0
    d = dev_fleet(f)
    dt = t(rows.view(np.uint8))
    g.fleet_obstacles_table_device(shard_args(d, 0, R, C_cap, 8, 5.0), abi.make_fleet_table(R, 0, dt))
    torch.cuda.synchronize()
    got = outputs(d, f)
    want = ftc.restate(rows, 0, R, 5.0, 8, f["custom"], f["own_count"], np.full(R, -7, np.int32))
    for a, b in zip(got, want):
        assert a.tobytes() == b.tobytes()
    assert got[3][3] == got[3][17] == fc.BAD_INPUT and got[2][3] == got[2][17] == -1
    assert got[1][3] == -7 and (got[0][3] == f["custom"][3]).all()
    with pytest.raises(T.TebGpuError):
        g.fleet_obstacles_table(rows, 0, R, f["custom"], 5.0, 8, own_count=f["own_count"])
    bad = rows.copy()
    bad["live"][:] = 1
    bad["vx"][30] = np.nan
    with pytest.raises(T.TebGpuError):
        g.fleet_obstacles_table(bad, 0, R, f["custom"], 5.0, 8)


def test_argument_errors_write_nothing(ctxs):
    R, C_cap = 20, 4
    f = random_fleet(R, R, C_cap, seed=2)
    g = ctxs[0]
    d = dev_fleet(f)
    rows = t(ftc.table([ftc.publish(f["pose"], f["last_cmd"], f["radius"], f["world"])], R + 4).view(np.uint8))
    before = [x.clone() for x in (rows, d["custom"], d["cc"], d["need"], d["st"])]
    fa = shard_args(d, 0, R, C_cap, 8, 3.0)
    tables = [abi.make_fleet_table(R + 4, -1, rows), abi.make_fleet_table(R + 4, 5, rows),
              abi.make_fleet_table(R - 1, 0, rows), abi.make_fleet_table(0, 0, rows),
              abi.make_fleet_table(R + 4, 0, rows.data_ptr() + 8), abi.make_fleet_table(R + 4, 0, None)]
    for tb in tables:
        with pytest.raises(T.TebGpuError):
            g.fleet_obstacles_table_device(fa, tb)
        with pytest.raises(T.TebGpuError):
            g.fleet_publish_device(fa, tb)
    nopose = shard_args(d, 0, R, C_cap, 8, 3.0)
    nopose.pose = None
    with pytest.raises(T.TebGpuError):
        g.fleet_publish_device(nopose, abi.make_fleet_table(R + 4, 0, rows))
    for kw in (dict(max_rows=33), dict(range=-1.0)):
        bad = shard_args(d, 0, R, C_cap, kw.get("max_rows", 8), kw.get("range", 3.0))
        with pytest.raises(T.TebGpuError):
            g.fleet_obstacles_table_device(bad, abi.make_fleet_table(R + 4, 0, rows))
    for cap in (0, R + 3, R + 5):                       # one rank: T must be cap
        with pytest.raises(T.TebGpuError):
            g.fleet_gather_device(abi.make_fleet_table(R + 4, 0, rows), cap)
    torch.cuda.synchronize()
    for a, b in zip(before, (rows, d["custom"], d["cc"], d["need"], d["st"])):
        assert torch.equal(a, b)
    # the same table without errors is taken
    g.fleet_obstacles_table_device(fa, abi.make_fleet_table(R + 4, 0, rows))
    torch.cuda.synchronize()
    assert (d["st"] >= 0).all()


def test_the_gather_of_one_rank_leaves_the_table_unchanged(ctxs):
    R = 50
    f = random_fleet(R, R, 4, seed=3)
    host = ftc.table([ftc.publish(f["pose"], f["last_cmd"], f["radius"], f["world"])], R + 6)
    rows = t(host.view(np.uint8))
    g = ctxs[0]
    g.fleet_gather_device(abi.make_fleet_table(R + 6, 0, rows), R + 6)            # no communicator
    assert g.fleet_gather(host, R + 6).tobytes() == host.tobytes()
    g1 = T.TebGpu(64, 8, 64, 8)
    try:
        ident = np.zeros(128, np.uint8)
        g1.comm_get_unique_id(ident)
        g1.comm_init(ident, 1, 0)
        assert g1.info(3) == 1
        g1.fleet_gather_device(abi.make_fleet_table(R + 6, 0, rows), R + 6)
        torch.cuda.synchronize()
        assert rows.cpu().numpy().tobytes() == host.tobytes()
        assert g1.fleet_gather(host, R + 6).tobytes() == host.tobytes()
        g1.comm_destroy()
    finally:
        g1.close()


# ---- two ranks over NCCL, one GPU each
NCCL_R, NCCL_C = 2000, 12


def _nccl_worker(rank, world, port, out_dir, counts):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    import teb_local_planner_b200 as T
    from teb_local_planner_b200 import abi
    from teb_local_planner_b200 import distributed as D
    from tests import fleet_table_cases as ftc
    from tests.test_gpu_fleet_obstacles import random_fleet
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("gloo", rank=rank, world_size=world)
    f = random_fleet(NCCL_R, NCCL_R, NCCL_C, seed=21)
    g = T.TebGpu(NCCL_R, 8, NCCL_R, 8, device=rank)
    D.init_comm(g, rank, world)
    cap, first = D.fleet_layout(counts, world)
    lo, hi = ftc.split(NCCL_R, counts)[rank]
    tt = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    rows = tt(ftc.padding(world * cap).view(np.uint8))
    custom = tt(f["custom"][lo:hi].view(np.uint8))
    own = tt(f["own_count"][lo:hi])
    cc, need, st = (torch.full((hi - lo,), -7, dtype=torch.int32, device=dev) for _ in range(3))
    n = hi - lo
    fa = abi.make_fleet_args(n, n, NCCL_C, 8, 4.0, pose=tt(f["pose"][lo:hi]), last_cmd=tt(f["last_cmd"][lo:hi]),
                             radius=tt(f["radius"][lo:hi]), world=tt(f["world"][lo:hi]), own_count=own, custom=custom,
                             custom_count=cc, needed=need, status=st)
    tb = abi.make_fleet_table(world * cap, first[rank], rows)
    g.fleet_publish_device(fa, tb)
    g.fleet_gather_device(tb, cap)
    g.fleet_obstacles_table_device(fa, tb)
    torch.cuda.synchronize()
    np.save(os.path.join(out_dir, f"table_{rank}.npy"), rows.cpu().numpy())
    for name, x in (("custom", custom), ("cc", cc), ("need", need), ("st", st)):
        np.save(os.path.join(out_dir, f"{name}_{rank}.npy"), x.cpu().numpy())
    g.comm_destroy()
    g.close()
    dist.destroy_process_group()


def test_two_ranks_gather_over_nccl_and_equal_the_union(ctxs, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("the two-rank NCCL fleet gather needs 2 GPUs; this machine has fewer")
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
    assert not alive, "a rank did not finish within 240 s"
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    f = random_fleet(NCCL_R, NCCL_R, NCCL_C, seed=21)
    want = run_union(ctxs[0], f, 4.0, 8)
    tabs = [np.load(tmp_path / f"table_{r}.npy") for r in range(world)]
    assert tabs[0].tobytes() == tabs[1].tobytes()
    got = [np.concatenate([np.load(tmp_path / f"{name}_{r}.npy") for r in range(world)])
           for name in ("custom", "cc", "need", "st")]
    assert got[0].tobytes() == want[0].view(np.uint8).tobytes()
    for a, b in zip(got[1:], want[1:]):
        assert a.tobytes() == b.tobytes()


# ---- a fleet of two robot kinds in two contexts, on one stream
B_KIND = (12, 10)               # circular robots 0 .. 11, car-like robots 12 .. 21 of the fleet
RADIUS = (0.25, 0.4)            # the circle each kind is published as


def _kind_params(k):
    if k == 0:
        p = scenes.config_params("C2")
        p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    else:
        p = scenes.config_params("C3")
        p.footprint_type = abi.TEB_FOOTPRINT_TWO_CIRCLES
        p.footprint_front_offset, p.footprint_front_radius = 0.2, 0.2
        p.footprint_rear_offset, p.footprint_rear_radius = 0.2, 0.2
    p.include_dynamic_obstacles = 1
    p.max_vel_trans = p.max_vel_x
    p.global_plan_overwrite_orientation = 1
    return p


def _mixed_scenario():
    rng = np.random.default_rng(43)
    start = np.array([[0.9 * i - 2.25, 0.9 * j - 1.35] for i in range(6) for j in range(4)])[:sum(B_KIND)]
    start = start[rng.permutation(len(start))] + rng.uniform(-0.1, 0.1, (len(start), 2))   # the kinds mixed in space
    goal = -start + rng.uniform(-0.3, 0.3, start.shape)
    G_cap = 256
    gp, begin, end = _straight_plans(start, goal, G_cap)
    robot = np.column_stack([start, gp[:, 0, 2]])
    return dict(gp=gp, begin=begin, end=end, robot=robot, G_cap=G_cap, raster=_raster(len(start), start, "random"))


def _mixed_loop(union, cycles=20, n_cap=96, P_cap=128, M_cap=512, Lb=10, max_rows=8, rng=3.0, graph_at=(3, 8)):
    """union=False: each kind's context publishes its robots into one padded table, then steps its robots against it;
    True: one tebgpu_fleet_obstacles call over both kinds' robots on a third context. Then every kind's context runs
    costmap_tf -> local_plan_tf -> backup modes -> plan -> costmap check -> finish, all on one stream."""
    sc = _mixed_scenario()
    B = len(sc["robot"])
    C_cap = 1 + max_rows
    r = sc["raster"]
    dt, now = 0.2, 1000.0
    z = lambda shape, dtp: torch.zeros(shape, dtype=dtp, device=DEV)
    f64, i32 = torch.float64, torch.int32
    # the fleet's arrays, one row per robot of either kind; each kind's context works on its rows
    cost, grid, origin = t(r["cost"]), t(r["grid"]), t(r["origin"])
    robot = t(sc["robot"].copy())
    radius = t(np.concatenate([np.full(n, RADIUS[k]) for k, n in enumerate(B_KIND)]))
    own_rows = np.zeros((B, C_cap), abi.OBST_DTYPE)
    own_rows[:, 0]["x"], own_rows[:, 0]["y"] = sc["robot"][:, 0] - 5.0, sc["robot"][:, 1] + 5.0
    custom, ccount, own = t(own_rows.view(np.uint8)), t(np.ones(B, np.int32)), t(np.ones(B, np.int32))
    last_cmd = z((B, 3), f64)
    fneed, fstat = z(B, i32), z(B, i32)
    gpd, begin, end = t(sc["gp"]), t(sc["begin"]), t(sc["end"])
    cmd_vel, vel = z((B, 3), f64), z((B, 3), f64)
    cap, first = D.fleet_layout(list(B_KIND), 2)
    table = padded_table(2 * cap, dict(pose=sc["robot"]), seed=5)
    # the union call's context first, with the kinds' limits: a kernel's shared-memory attribute is set per process by the
    # last context created, so a context with smaller limits created after the kinds' would cut their launches short
    gu = T.TebGpu(B, n_cap, B, M_cap, 0) if union else None
    kinds = []
    lo = 0
    for k, n in enumerate(B_KIND):
        hi = lo + n
        p = _kind_params(k)
        g = T.TebGpu(n, n_cap, n, M_cap, 0)
        g.set_params(p)
        sl = slice(lo, hi)
        state = {kk: t(v) for kk, v in abi.make_cycle_state(n, Lb).items()}
        state["last_cmd"] = last_cmd[sl]
        kk = dict(g=g, p=p, lo=lo, hi=hi, n=n, state=state, plan=z((n, P_cap, 3), f64), pcount=z(n, i32),
                  result=z(n, i32), gidx=z(n, i32), needed=z((n, 2), i32), since=z(n, f64),
                  poses=z((n, n_cap, 4), f64), nn=z(n, i32), sid=t(np.arange(n, dtype=np.int32)),
                  obst=z(n * M_cap * 64, torch.uint8), ocount=z(n, i32), costo=z(n, f64), chi2=z(n, f64),
                  status=z(n, i32), iters=z(n, i32), cmd=z((n, 4), f64), path=z(n, i32), feas=z(n, i32), qc=z(n, i32),
                  outcome=z(n, i32), osc=z(n, i32))
        vs = np.zeros((n, 4))
        vs[:, 3] = 1.0
        kk["vs"], kk["vstart"], kk["vgoal"] = vs, t(vs), t(vs)
        bs = abi.TebBatch()
        bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = n, n_cap, n, M_cap, 0, 0
        bs.poses, bs.n, bs.scene_id = kk["poses"].data_ptr(), kk["nn"].data_ptr(), kk["sid"].data_ptr()
        bs.obstacles, bs.obst_count = kk["obst"].data_ptr(), kk["ocount"].data_ptr()
        bs.vel_start, bs.vel_goal = kk["vstart"].data_ptr(), kk["vgoal"].data_ptr()
        bs.prefer_rotdir = state["prefer_rotdir"].data_ptr()
        bs.cost, bs.chi2, bs.status, bs.lm_iters = (kk["costo"].data_ptr(), kk["chi2"].data_ptr(), kk["status"].data_ptr(),
                                                     kk["iters"].data_ptr())
        kk["bs"] = bs
        ca = abi.TebCostmapArgs()
        ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = n, r["cost"].shape[1], M_cap, C_cap, 1
        ca.behind_robot_dist = 1.5
        ca.cost, ca.grid, ca.origin, ca.robot = cost[sl].data_ptr(), grid[sl].data_ptr(), origin[sl].data_ptr(), robot[sl].data_ptr()
        ca.custom, ca.custom_count = custom[sl].data_ptr(), ccount[sl].data_ptr()
        ca.obstacles, ca.obst_count = kk["obst"].data_ptr(), kk["ocount"].data_ptr()
        kk["ca"] = ca
        kk["ident"] = t(np.tile(IDENTITY, (n, 1)))
        kk["cframes"] = abi.make_frame_args(custom_to_costmap=kk["ident"].data_ptr())
        kk["pframes"] = abi.make_frame_args(costmap_to_plan=kk["ident"].data_ptr(), plan_to_costmap=kk["ident"].data_ptr())
        kk["la"] = abi.make_local_plan_args(sc["G_cap"], P_cap, 0, max_lookahead_dist=2.0, global_plan=gpd[sl].data_ptr(),
                                            plan_begin=begin[sl].data_ptr(), plan_end=end[sl].data_ptr(),
                                            robot=robot[sl].data_ptr(), robot_vel=vel[sl].data_ptr(),
                                            grid=grid[sl].data_ptr(), origin=origin[sl].data_ptr(),
                                            infeasible_count=state["infeasible_count"].data_ptr(),
                                            since_infeasible=kk["since"].data_ptr(), plan=kk["plan"].data_ptr(),
                                            plan_count=kk["pcount"].data_ptr(), goal_idx=kk["gidx"].data_ptr(),
                                            result=kk["result"].data_ptr(), needed=kk["needed"].data_ptr())
        kk["args"] = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0,
                                   False)
        kk["fa"] = abi.make_feasibility_args(0.1, max_queries=512, feasible=kk["feas"].data_ptr(),
                                             query_count=kk["qc"].data_ptr())
        kk["world"] = abi.make_costmap_world(r["cost"].shape[1], cost[sl].data_ptr(), grid[sl].data_ptr(),
                                             origin[sl].data_ptr())
        kk["fl"] = abi.make_fleet_args(n, n, C_cap, max_rows, rng, pose=robot[sl], last_cmd=last_cmd[sl],
                                       radius=radius[sl], own_count=own[sl], custom=custom[sl], custom_count=ccount[sl],
                                       needed=fneed[sl], status=fstat[sl])
        kk["tb"] = abi.make_fleet_table(2 * cap, first[k], table)
        kinds.append(kk)
        lo = hi
    fu = abi.make_fleet_args(B, B, C_cap, max_rows, rng, pose=robot, last_cmd=last_cmd, radius=radius, own_count=own,
                             custom=custom, custom_count=ccount, needed=fneed, status=fstat)
    cs = dict(buffer_length=Lb, oscillation_recovery_min_duration=2.0)
    s = torch.cuda.Stream()
    trace, graphs = [], []
    for c in range(cycles):
        with torch.cuda.stream(s):
            if union:
                gu.fleet_obstacles_device(fu, stream=s.cuda_stream)
            else:
                for kk in kinds:
                    kk["g"].fleet_publish_device(kk["fl"], kk["tb"], stream=s.cuda_stream)
                for kk in kinds:
                    kk["g"].fleet_obstacles_table_device(kk["fl"], kk["tb"], stream=s.cuda_stream)
            for kk in kinds:
                g, st = kk["g"], kk["state"]
                cy = abi.make_cycle_args(now, L_cap=Lb, **cs, local_plan_result=kk["result"].data_ptr(),
                                         robot_vel=vel[kk["lo"]:kk["hi"]].data_ptr(), cmd=kk["cmd"].data_ptr(),
                                         feasible=kk["feas"].data_ptr(), cmd_vel=cmd_vel[kk["lo"]:kk["hi"]].data_ptr(),
                                         outcome=kk["outcome"].data_ptr(), oscillating=kk["osc"].data_ptr(),
                                         **{key: st[key].data_ptr() for key in abi.CYCLE_STATE})
                kk["since"].copy_(now - st["last_infeasible"])
                g.costmap_obstacles_device(kk["ca"], stream=s.cuda_stream, frames=kk["cframes"])
                g.local_plan_device(kk["bs"], kk["la"], stream=s.cuda_stream, frames=kk["pframes"])
                g.backup_modes_device(kk["bs"], cy, stream=s.cuda_stream)
                g.plan_device(kk["bs"], kk["args"], kk["cmd"], initial_plan=kk["plan"], plan_count=kk["pcount"],
                              P_cap=P_cap, path=kk["path"], stream=s.cuda_stream)
                g.check_feasible_costmap_device(kk["bs"], kk["fa"], kk["world"], stream=s.cuda_stream)
                g.finish_cycle_device(kk["bs"], cy, stream=s.cuda_stream)
        s.synchronize()
        if c in graph_at and not union:
            for k, kk in enumerate(kinds):
                n = kk["n"]
                hb = abi.HostBatch(kk["poses"].cpu().numpy(), kk["nn"].cpu().numpy(),
                                   kk["obst"].cpu().numpy().view(abi.OBST_DTYPE).reshape(n, M_cap),
                                   kk["ocount"].cpu().numpy(), scene_id=np.arange(n, dtype=np.int32), vel_start=kk["vs"],
                                   vel_goal=kk["vs"], prefer_rotdir=kk["state"]["prefer_rotdir"].cpu().numpy())
                g2 = T.TebGpu(n, n_cap, n, M_cap, 0)
                g2.set_params(kk["p"])
                graphs.append((k, hb, g2.build_system(hb, graph=True)))
                g2.close()
        with torch.cuda.stream(s):
            th = robot[:, 2].clone()
            robot[:, 0] += (cmd_vel[:, 0] * torch.cos(th) - cmd_vel[:, 1] * torch.sin(th)) * dt
            robot[:, 1] += (cmd_vel[:, 0] * torch.sin(th) + cmd_vel[:, 1] * torch.cos(th)) * dt
            robot[:, 2] += cmd_vel[:, 2] * dt
            vel.copy_(cmd_vel)
        s.synchronize()
        rec = dict(custom=custom, ccount=ccount, fneed=fneed, fstat=fstat, robot=robot, cmd_vel=cmd_vel, last_cmd=last_cmd)
        for k, kk in enumerate(kinds):
            for key in ("obst", "ocount", "pcount", "result", "nn", "poses", "status", "path", "cmd", "outcome", "osc",
                        "feas"):
                rec[f"{key}{k}"] = kk[key]
            for key, v in kk["state"].items():
                rec[f"{key}{k}"] = v
        rec = {key: v.cpu().numpy().copy() for key, v in rec.items()}
        for k, kk in enumerate(kinds):
            pc = kk["pcount"].cpu().numpy()
            pl = kk["plan"].cpu().numpy()
            rec[f"plan{k}"] = np.concatenate([pl[b, :pc[b]] for b in range(kk["n"])])
        trace.append(rec)
        now += dt
    for kk in kinds:
        kk["g"].close()
    if gu is not None:
        gu.close()
    return trace, graphs


def test_a_fleet_of_two_kinds_in_two_contexts_matches_the_union_call():
    tab, graphs = _mixed_loop(False)
    ref, _ = _mixed_loop(True)
    for c, (x, y) in enumerate(zip(tab, ref)):
        assert x.keys() == y.keys()
        for key in x:
            assert x[key].tobytes() == y[key].tobytes(), (c, key)
    B = sum(B_KIND)
    assert any((c["ccount"] > 1).all() for c in tab)
    assert sum((c[f"outcome{k}"] == abi.TEB_CYCLE_COMMAND).sum() for c in tab for k in (0, 1)) > 0
    # each kind sees robots of the other kind: the rows of the other kind's radius, and dynamic-obstacle edges for them
    other_rows = [0, 0]
    for c in tab:
        rows = c["custom"].view(abi.OBST_DTYPE).reshape(B, -1)
        cc = c["ccount"]
        for b in range(B):
            k = 0 if b < B_KIND[0] else 1
            other_rows[k] += int((rows[b, 1:cc[b]]["radius"] == RADIUS[1 - k]).sum())
    assert min(other_rows) > 0, other_rows
    seen = [0, 0]
    for k, hb, gr in graphs:
        for b in range(len(hb.n)):
            nb, cnt = int(hb.n[b]), int(hb.obst_count[b])
            if nb < 3:
                continue
            rows = hb.obstacles[b, :cnt]
            dyn = np.nonzero((rows["dynamic"] == 1) & (rows["radius"] == RADIUS[1 - k]))[0]
            if len(dyn):
                seen[k] += 1
                assert np.isfinite(gr["dyn_t"][b, 1:nb - 1]).all(), (k, b)
                words = gr["assoc"][b, :nb]
                for l in dyn:
                    assert not ((words[:, l // 64] >> np.uint64(l % 64)) & np.uint64(1)).any(), (k, b, l)
    assert sum(seen) > 0, "no band had a dynamic row of the other kind at the graph cycles"
