"""tests/fleet_table_cases.py, the restatement the fleet table steps are held to: a fleet split into contiguous shards,
each shard published into one padded table and stepped against the whole table, gives exactly what
fleet_cases.restate gives on the whole fleet, on random fleets and on hand cases (equal distances across shards, a
neighbour exactly at range in another shard, coincident robots in different shards, padding rows on top of robots, an
uneven split and a one-robot shard). Then the same over gloo with two and three ranks: every rank publishes its shard,
gathers the table with distributed.gather_fleet_table_torch and steps its robots."""
import math
import os
import socket
import sys

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from teb_local_planner_b200 import distributed as D
from tests import fleet_cases as fc
from tests import fleet_table_cases as ftc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fleet(R, C_cap, seed, worlds=2, clustered=True):
    rng = np.random.default_rng(seed)
    if clustered:
        centres = rng.uniform(-5, 5, (max(1, R // 20), 2))
        xy = centres[rng.integers(0, len(centres), R)] + rng.normal(0, 0.8, (R, 2))
    else:
        xy = rng.uniform(-30, 30, (R, 2))
    pose = np.column_stack([xy, rng.uniform(-math.pi, math.pi, R)])
    dup = rng.integers(0, R, max(2, R // 15))
    pose[dup[1:]] = pose[dup[:-1]]
    cmd = np.column_stack([rng.uniform(-0.4, 0.4, R), rng.uniform(-0.1, 0.1, R), rng.uniform(-0.3, 0.3, R)])
    cmd[rng.random(R) < 0.2, :2] = 0.0
    custom = np.zeros((R, C_cap), abi.OBST_DTYPE)
    custom.view(np.uint8)[:] = rng.integers(0, 256, custom.nbytes, dtype=np.uint8).reshape(R, -1)
    return dict(pose=pose, last_cmd=cmd, radius=rng.uniform(0.1, 0.6, R), world=rng.integers(0, worlds, R).astype(np.int32),
                custom=custom, own_count=rng.integers(0, C_cap + 1, R).astype(np.int32))


def _check(f, rng, max_rows, counts, pad_like=False):
    want = fc.restate(f["pose"], f["last_cmd"], f["radius"], rng, max_rows, f["custom"], f.get("own_count"), None,
                      f.get("world"))
    got, tab = ftc.sharded(f["pose"], f["last_cmd"], f["radius"], rng, max_rows, f["custom"], counts,
                           f.get("own_count"), None, f.get("world"), pad_like=pad_like)
    for a, b, name in zip(got, want, ("custom", "custom_count", "needed", "status")):
        assert a.tobytes() == b.tobytes(), (name, counts, rng, max_rows)
    return want, tab


@pytest.mark.parametrize("R,counts", [(1, [1]), (40, [40]), (40, [13, 27]), (97, [30, 1, 40, 26]),
                                      (120, [17, 0, 33, 20, 50]), (64, [8] * 8)])
@pytest.mark.parametrize("clustered", [True, False])
def test_random_sharded_fleets_equal_the_union(R, counts, clustered):
    f = _fleet(R, 10, seed=R + len(counts), clustered=clustered)
    for rng in (0.0, 1.0, 4.0, math.inf):
        for max_rows in (0, 3, 8):
            _check(f, rng, max_rows, counts)
            _check(f, rng, max_rows, counts, pad_like=True)


def _hand(pose, cmd=None, world=None, C=4, own=None):
    R = len(pose)
    custom = np.zeros((R, C), abi.OBST_DTYPE)
    custom.view(np.uint8)[:] = 0xAB
    return dict(pose=np.array(pose, np.float64), last_cmd=np.zeros((R, 3)) if cmd is None else np.array(cmd, np.float64),
                radius=np.linspace(0.2, 0.5, R), world=None if world is None else np.array(world, np.int32),
                custom=custom, own_count=None if own is None else np.array(own, np.int32))


def test_equal_distances_with_one_neighbour_in_each_shard():
    f = _hand([(0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (-1.0, 0.0, 0.0), (0.0, 1.0, 0.0)])
    want, _ = _check(f, 1.0, 2, [2, 2])
    # robot 0: d2 = 1 to all three, the lower index first, whichever shard it is in
    assert want[2][0] == 3 and [o["x"] for o in want[0][0, :2]] == [1.0, -1.0]
    _check(f, 1.0, 2, [1, 3])
    _check(f, 1.0, 2, [3, 1])


def test_a_neighbour_exactly_at_range_in_another_shard():
    f = _hand([(0.0, 0.0, 0.0), (3.0, 4.000000000001, 0.0), (3.0, 4.0, 0.0)])
    want, _ = _check(f, 5.0, 8, [1, 2])
    assert want[2][0] == 1 and (want[0][0, 0]["x"], want[0][0, 0]["y"]) == (3.0, 4.0)


def test_coincident_robots_in_different_shards():
    f = _hand([(1.5, -2.0, 0.3), (0.0, 0.0, 0.0), (1.5, -2.0, 2.0)], cmd=[(0.3, 0.0, 0.0), (0.0, 0.0, 0.0),
                                                                        (0.0, 0.2, 0.0)])
    want, _ = _check(f, 0.0, 4, [2, 1])
    assert list(want[2]) == [1, 0, 1] and want[0][0, 0]["dynamic"] == 1 and want[0][2, 0]["radius"] == 0.2


def test_padding_rows_on_top_of_robots_are_never_chosen():
    f = _hand([(0.0, 0.0, 0.0), (0.5, 0.0, 0.0), (1.0, 0.0, 0.0)])
    want, tab = _check(f, 10.0, 8, [1, 2], pad_like=True)
    assert len(tab) == 4 and tab["live"].tolist() == [1, 0, 1, 1]
    assert (tab[1]["x"], tab[1]["y"]) == (0.0, 0.0)                 # the padding row sits on robot 0
    assert list(want[2]) == [2, 2, 2]
    # and on top of the robot itself: robot 0's own position copied into every padding row of a wider table
    rows = ftc.table([ftc.publish(f["pose"][:1], f["last_cmd"][:1], f["radius"][:1]),
                      ftc.publish(f["pose"][1:], f["last_cmd"][1:], f["radius"][1:])], 4, pad_like=True)
    out = ftc.restate(rows, 0, 1, 10.0, 8, f["custom"][:1])
    assert out[2][0] == 2 and [o["x"] for o in out[0][0, :2]] == [0.5, 1.0]


def test_an_uneven_split_and_a_one_robot_shard():
    f = _fleet(23, 6, seed=3)
    for counts in ([1, 22], [22, 1], [5, 1, 17], [1, 1, 1, 20]):
        _check(f, 2.0, 4, counts)


def test_a_robot_whose_own_row_is_padding_gets_bad_input():
    rows = ftc.table([ftc.publish([(0.0, 0.0, 0.0)], np.zeros((1, 3)), 0.2)], 3)
    out = ftc.restate(rows, 1, 2, 5.0, 8, np.zeros((2, 2), abi.OBST_DTYPE), custom_count=[7, 7])
    assert list(out[3]) == [fc.BAD_INPUT] * 2 and list(out[2]) == [-1, -1] and list(out[1]) == [7, 7]


def test_fleet_layout_pads_every_shard_to_one_cap():
    assert D.fleet_layout([3, 5, 1], 3) == (5, [0, 5, 10])
    assert D.fleet_layout([0, 0], 2) == (1, [0, 1])
    with pytest.raises(ValueError):
        D.fleet_layout([1, 2], 3)


# ---- over gloo, one process per rank
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


GLOO_R, GLOO_C = 37, 6


def _gloo_worker(rank, world, port, out_dir, counts):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from teb_local_planner_b200 import distributed as D
    from tests import fleet_table_cases as ftc
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    f = _fleet(GLOO_R, GLOO_C, seed=9)
    cap, first = D.fleet_layout(counts, world)
    lo, hi = ftc.split(GLOO_R, counts)[rank]
    rows = ftc.padding(world * cap)
    rows[first[rank]:first[rank] + hi - lo] = ftc.publish(f["pose"][lo:hi], f["last_cmd"][lo:hi], f["radius"][lo:hi],
                                                          f["world"][lo:hi])
    tab = D.gather_fleet_table_torch(rows, cap, rank, world)
    out = ftc.restate(tab, first[rank], hi - lo, 2.5, 8, f["custom"][lo:hi], f["own_count"][lo:hi])
    for k, name in enumerate(("custom", "ccount", "needed", "status")):
        np.save(os.path.join(out_dir, f"{name}_{rank}.npy"), out[k])
    np.save(os.path.join(out_dir, f"table_{rank}.npy"), tab)
    dist.destroy_process_group()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("world,counts", [(2, [20, 17]), (3, [12, 1, 24])])
def test_gloo_ranks_gather_the_table_and_equal_the_single_process_run(tmp_path, world, counts):
    import torch.multiprocessing as mp
    mp.spawn(_gloo_worker, args=(world, _free_port(), str(tmp_path), counts), nprocs=world, join=True)
    f = _fleet(GLOO_R, GLOO_C, seed=9)
    want = fc.restate(f["pose"], f["last_cmd"], f["radius"], 2.5, 8, f["custom"], f["own_count"], None, f["world"])
    tabs = [np.load(tmp_path / f"table_{r}.npy") for r in range(world)]
    assert all(t.tobytes() == tabs[0].tobytes() for t in tabs)
    for k, name in enumerate(("custom", "ccount", "needed", "status")):
        got = np.concatenate([np.load(tmp_path / f"{name}_{r}.npy") for r in range(world)])
        assert got.tobytes() == want[k].tobytes(), name
    assert (want[2] > 0).any() and (want[3] == fc.TRUNCATED).any()
