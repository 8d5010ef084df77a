"""The fleet steps' grid search (k_fleet_bin, the scan, k_fleet_scatter, k_fleet_obstacles_grid) against their all-pairs
search (k_fleet_obstacles), which stays the reference: on the same inputs the grid (tebgpu_set_fleet_search 2), the grid
with every cell in one bucket (3) and the automatic choice (0) write the bytes all pairs (1) writes - custom rows,
custom_count, needed and status - for the array step and the table step, including non-finite and far robots, range 0,
tiny and overflowing ranges, cuts and bad scenes. Two grid calls write the same bytes, and so do the host and device
forms; key 19 reports the search the automatic choice took; the 20-cycle fleet loop is the same with either search."""
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi
from tests import fleet_cases as fc
from tests import test_gpu_fleet_obstacles as tfo
from tests import test_gpu_fleet_table as tft
from tests.test_gpu_fleet_obstacles import random_fleet, run_device

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BIG = 32768
ALL_PAIRS, GRID, ONE_BUCKET, AUTO = (abi.TEBGPU_FLEET_SEARCH_ALL_PAIRS, abi.TEBGPU_FLEET_SEARCH_GRID,
                                     abi.TEBGPU_FLEET_SEARCH_ONE_BUCKET, abi.TEBGPU_FLEET_SEARCH_AUTO)
NAMES = ("custom", "custom_count", "needed", "status")


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(BIG, 8, BIG + 64, 64)
    yield g
    g.set_fleet_search(AUTO)
    g.close()


def run_mode(g, mode, f, rng, max_rows, **kw):
    g.set_fleet_search(mode)
    try:
        return run_device(g, f, rng, max_rows, twice=True, **kw)
    finally:
        g.set_fleet_search(AUTO)


def assert_modes_equal(g, f, rng, max_rows, modes=(GRID, ONE_BUCKET, AUTO), label="", **kw):
    """every mode writes the bytes all pairs writes (each mode twice: the same bytes again); returns all pairs' outputs"""
    want = run_mode(g, ALL_PAIRS, f, rng, max_rows, **kw)
    for mode in modes:
        got = run_mode(g, mode, f, rng, max_rows, **kw)
        for a, b, name in zip(got, want, NAMES):
            assert a.tobytes() == b.tobytes(), (label, mode, name, rng)
    return want


@pytest.mark.parametrize("R,clustered", [(1, True), (700, True), (8192, True), (8192, False), (BIG, True),
                                         (BIG, False)])
def test_random_fleets(gpu, R, clustered):
    f = random_fleet(R, R, 12, seed=R + clustered, worlds=3, clustered=clustered)
    for rng, max_rows in ((1.5, 8), (6.0, 32), (0.25, 1)):
        # the one-bucket grid scans every candidate of a world from every robot: kept to the smaller fleets
        modes = (GRID, ONE_BUCKET, AUTO) if R <= 8192 else (GRID, AUTO)
        want = assert_modes_equal(gpu, f, rng, max_rows, modes=modes, label=f"R={R}")
        if R > 1 and rng == 6.0:
            assert (want[2] > 0).any()


def test_the_restatement_agrees_on_a_grid_fleet(gpu):
    f = random_fleet(3000, 3000, 16, seed=3)
    got = run_mode(gpu, GRID, f, 2.0, 8)
    tfo.assert_like_restatement(got, f, 2.0, 8, label="grid")


@pytest.mark.parametrize("worlds,per", [(4096, 8), (512, 16)])
def test_many_worlds(gpu, worlds, per):
    """many independent worlds over one small square: every world's robots overlap every other world's"""
    R = worlds * per
    rng_ = np.random.default_rng(worlds)
    f = random_fleet(R, R, 10, seed=worlds, worlds=1)
    f["pose"][:, :2] = rng_.uniform(0, 12, (R, 2))
    f["world"] = np.repeat(np.arange(worlds, dtype=np.int32) * 7919 - 2 ** 30, per)
    f["world"][:per] = np.iinfo(np.int32).min
    f["world"][per:2 * per] = np.iinfo(np.int32).max
    want = assert_modes_equal(gpu, f, 3.0, 8, modes=(GRID, AUTO), label="worlds")
    assert (want[2] > 0).any() and (want[2] < per).all()


def test_hand_cases(gpu):
    below = math.nextafter(0.001, 0.0)
    cases = [
        dict(pose=[(0.0, 0.0, 0.0), (3.0, 4.0, 0.0), (3.0, 4.000000000001, 0.0)], rng=5.0, max_rows=8, C=4),
        dict(pose=[(0.0, 0.0, 0.0), (0.0, 1.0, 0.0), (-1.0, 0.0, 0.0), (1.0, 0.0, 0.0), (0.0, -1.0, 0.0)], rng=1.0,
             max_rows=2, C=8),
        dict(pose=[(1.5, -2.0, 0.3), (1.5, -2.0, 2.0)], rng=0.0, max_rows=4, C=4),
        dict(pose=[(0.0, 0.0, 0.0), (0.1, 0.0, 0.0), (0.05, 0.0, 0.0)], rng=10.0, max_rows=8, C=4, world=[7, 7, 3],
             own=[1, 0, 2]),
        dict(pose=[(0.0, 0.0, 0.0)] + [(0.5 * k, 0.0, 0.0) for k in range(1, 7)], rng=100.0, max_rows=4, C=5,
             own=[3, 0, 0, 0, 0, 0, 0]),
        dict(pose=[(0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (2.0, 0.0, 0.0)], rng=10.0, max_rows=8, C=4,
             cmd=[(0.0, 0.0, 0.0), (0.001, 0.0, 0.5), (below, 0.0, 0.0)]),
        dict(pose=[(0.0, 0.0, 0.0), (1.0, 1.0, math.pi / 2)], rng=10.0, max_rows=8, C=1,
             cmd=[(0.0, 0.0, 0.0), (0.4, 0.1, 0.0)]),
        # a neighbour exactly at range across a cell edge, and index ties at equal distance either side
        dict(pose=[(3.0000457763671875, 0.0, 0.0), (0.0, 0.0, 0.0), (6.000091552734375, 0.0, 0.0),
                   (3.0000457763671875, 3.0, 0.0), (3.0000457763671875, -3.0, 0.0)], rng=3.0000457763671875,
             max_rows=3, C=4),
    ]
    for k, c in enumerate(cases):
        R = len(c["pose"])
        custom = np.zeros((R, c["C"]), abi.OBST_DTYPE)
        custom.view(np.uint8)[:] = 0xAB
        f = dict(pose=np.array(c["pose"]), last_cmd=np.array(c.get("cmd", np.zeros((R, 3)))), radius=np.full(R, 0.2),
                 custom=custom, world=None if "world" not in c else np.array(c["world"], np.int32),
                 own_count=None if "own" not in c else np.array(c["own"], np.int32))
        assert_modes_equal(gpu, f, c["rng"], c["max_rows"], label=f"case {k}")


def test_bad_shared_and_given_scenes(gpu):
    R, S = 300, 320
    f = random_fleet(R, S, 10, seed=8)
    scene = np.arange(R, dtype=np.int32)
    scene[5], scene[6] = -1, S
    scene[7] = scene[8] = 20
    scene[20] = 7
    f["own_count"][30] = 11
    want = assert_modes_equal(gpu, f, 5.0, 8, scene=scene, S=S, custom_count=np.full(S, 5, np.int32), label="scenes")
    assert want[3][5] == want[3][6] == want[3][30] == fc.BAD_INPUT and want[3][7] == fc.SHARED_SCENE


def test_non_finite_far_and_coincident_robots(gpu):
    R = 2000
    f = random_fleet(R, R, 8, seed=21, worlds=2)
    p = f["pose"]
    p[3, 0], p[4, 1], p[5, 0], p[6, 1] = np.nan, np.inf, -np.inf, np.nan
    p[7, :2] = (np.inf, -np.inf)
    p[10:20, 0] = 1e30                                   # past the coordinate bound for any range here
    p[20:25, :2] = (-4e29, 4e29)
    p[25:30, :2] = p[10, :2]                             # coincident far robots
    p[30:40, :2] = p[31, :2]                             # coincident robots on the grid
    f["world"][30:40] = 1
    for rng in (0.0, 5e-324, 1e-300, 2.0 ** -500, 1e-9, 2.5, 1e25, 1e200, math.inf):
        want = assert_modes_equal(gpu, f, rng, 8, modes=(GRID, ONE_BUCKET), label="non-finite")
        assert (want[2][[3, 4, 5, 6, 7]] == (0 if rng < 1e154 else want[2][[3, 4, 5, 6, 7]])).all()
        if rng > 0:
            assert want[2][30] >= 9


def test_every_robot_in_one_cell(gpu):
    R = 4096
    f = random_fleet(R, R, 8, seed=9, worlds=1)
    f["pose"][:, :2] = np.random.default_rng(9).uniform(0.0, 1.0, (R, 2))
    want = assert_modes_equal(gpu, f, 3.0, 8, label="one cell")
    assert (want[2] == R - 1).all()


def test_table_step_padded_and_sharded(gpu):
    """1 to 8 uneven shards in as many contexts on a padded table write the bytes of the union all-pairs call"""
    gs = [T.TebGpu(tft.MAX_R, 8, tft.MAX_R + 64, 64) for _ in range(tft.SHARDS)]
    try:
        for R, clustered in ((700, True), (tft.MAX_R, True), (tft.MAX_R, False)):
            f = random_fleet(R, R, 16, seed=R + 5, worlds=3, clustered=clustered)
            s = torch.cuda.Stream()
            for k, n in enumerate((1, 2, 3, 5, 8)):
                counts = tft.uneven_counts(R, n, seed=R + 2 * k)
                rng = (1.5, 6.0, 0.0, 3.0, math.inf)[k]
                gs[0].set_fleet_search(ALL_PAIRS)
                want = tft.run_union(gs[0], f, rng, 8, stream=s.cuda_stream)
                for mode in (GRID, ONE_BUCKET, AUTO) if R <= 700 else (GRID, AUTO):
                    for g in gs:
                        g.set_fleet_search(mode)
                    got, _, _ = tft.run_sharded(gs, f, counts, rng, 8, seed=k, stream=s.cuda_stream)
                    for a, b, name in zip(got, want, NAMES):
                        assert a.tobytes() == b.tobytes(), (name, R, counts, mode, rng)
    finally:
        for g in gs:
            g.close()


def test_host_and_device_forms_give_the_same_bits(gpu):
    R, S = 9000, 9100
    f = random_fleet(R, S, 16, seed=11)
    scene = np.random.default_rng(12).permutation(S)[:R].astype(np.int32)
    cc0 = np.full(S, 3, np.int32)
    dev = run_mode(gpu, GRID, f, 3.0, 8, scene=scene, S=S, custom_count=cc0)
    for mode in (GRID, AUTO):
        gpu.set_fleet_search(mode)
        host = gpu.fleet_obstacles(f["pose"], f["last_cmd"], f["radius"], f["custom"], 3.0, 8, own_count=f["own_count"],
                                   custom_count=cc0, world=f["world"], scene=scene)
        assert gpu.last_fleet_search() == "grid" and gpu.last_fleet_grid() == (R + 15) // 16
        for a, b, name in zip(dev, host, NAMES):
            assert a.tobytes() == b.tobytes(), name
    gpu.set_fleet_search(AUTO)
    # the table step's host form
    rows = tft.ftc.table([tft.ftc.publish(f["pose"], f["last_cmd"], f["radius"], f["world"])], R)
    outs = []
    for mode in (ALL_PAIRS, GRID):
        gpu.set_fleet_search(mode)
        outs.append(gpu.fleet_obstacles_table(rows, 0, R, f["custom"][:R], 3.0, 8, own_count=f["own_count"][:R]))
        assert gpu.last_fleet_search() == ("all_pairs" if mode == ALL_PAIRS else "grid")
    gpu.set_fleet_search(AUTO)
    for a, b, name in zip(*outs, NAMES):
        assert a.tobytes() == b.tobytes(), name


def test_the_automatic_choice(gpu):
    N0 = abi.FLEET_GRID_N0
    for R, rng, search in ((N0 - 1, 3.0, "all_pairs"), (N0, 3.0, "grid"), (N0, math.inf, "all_pairs"),
                           (N0, 0.0, "all_pairs"), (N0, 2.0 ** -500, "all_pairs"), (N0, 1e-9, "grid"),
                           (N0, 1e160, "all_pairs"), (BIG, 3.0, "grid"), (100, 3.0, "all_pairs")):
        f = random_fleet(R, R, 4, seed=R)
        run_device(gpu, f, rng, 4)
        assert gpu.last_fleet_search() == search, (R, rng)
        assert gpu.info(abi.TEBGPU_INFO_FLEET_SEARCH) == {"all_pairs": ALL_PAIRS, "grid": GRID}[search]
        assert gpu.last_fleet_grid() == (R + 15) // 16
    # the table step counts the table's rows: 100 robots against N0 rows take the grid
    f = random_fleet(N0, N0, 4, seed=1)
    rows = tft.ftc.table([tft.ftc.publish(f["pose"], f["last_cmd"], f["radius"], f["world"])], N0)
    for T_rows, search in ((N0, "grid"), (N0 - 1, "all_pairs")):
        gpu.fleet_obstacles_table(rows[:T_rows], T_rows - 100, 100, f["custom"][:100], 3.0, 4)
        assert gpu.last_fleet_search() == search, T_rows


def test_a_new_context_reports_no_search_and_bad_modes_are_refused():
    g = T.TebGpu(16, 8, 16, 8)
    try:
        assert g.last_fleet_search() is None and g.info(abi.TEBGPU_INFO_FLEET_SEARCH) == -1
        for bad in (-1, 4, 100):
            with pytest.raises(T.TebGpuError):
                g.set_fleet_search(bad)
        for mode in (AUTO, ALL_PAIRS, GRID, ONE_BUCKET):
            g.set_fleet_search(mode)
    finally:
        g.close()


def test_argument_errors_write_nothing(gpu):
    R = 9000
    f = random_fleet(R, R, 4, seed=2)
    for mode in (GRID, AUTO):
        gpu.set_fleet_search(mode)
        t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(tfo.DEV)
        custom, cc = t(f["custom"].view(np.uint8)), torch.full((R,), -7, dtype=torch.int32, device=tfo.DEV)
        need = torch.full((R,), -9, dtype=torch.int32, device=tfo.DEV)
        keep = dict(pose=t(f["pose"]), cmd=t(f["last_cmd"]), rad=t(f["radius"]))
        for kw in (dict(max_rows=33), dict(rng=-1.0), dict(rng=math.nan), dict(R=R, S=R - 1), dict(pose=None)):
            fa = abi.make_fleet_args(kw.get("R", R), kw.get("S", R), 4, kw.get("max_rows", 8), kw.get("rng", 3.0),
                                     pose=kw.get("pose", keep["pose"]), last_cmd=keep["cmd"], radius=keep["rad"],
                                     custom=custom, custom_count=cc, needed=need)
            with pytest.raises(T.TebGpuError):
                gpu.fleet_obstacles_device(fa)
        torch.cuda.synchronize()
        assert (cc == -7).all() and (need == -9).all()
        assert custom.cpu().numpy().tobytes() == f["custom"].tobytes()
        bad_pose = f["pose"].copy()
        bad_pose[3, 1] = np.nan
        with pytest.raises(T.TebGpuError):
            gpu.fleet_obstacles(bad_pose, f["last_cmd"], f["radius"], f["custom"], 3.0, 8)
    gpu.set_fleet_search(AUTO)


@pytest.mark.parametrize("kind", ["junction", "random"])
def test_the_fleet_loop_is_the_same_with_the_grid(kind, monkeypatch):
    traces = []
    for mode in (ALL_PAIRS, GRID):
        class Ctx(T.TebGpu):
            def __init__(self, *a, **kw):
                super().__init__(*a, **kw)
                self.set_fleet_search(mode)
        monkeypatch.setattr(T, "TebGpu", Ctx)
        traces.append(tfo._fleet_loop(kind, False)[0])
        monkeypatch.undo()
    for k, (x, y) in enumerate(zip(*traces)):
        for key in x:
            assert x[key].tobytes() == y[key].tobytes(), (kind, k, key)
