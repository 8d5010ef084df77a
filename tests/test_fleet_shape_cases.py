"""tests/fleet_shape_cases.py, the restatement the shaped fleet steps are held to, pinned on hand-computed fleets: a kind
of one circle at the body origin gives fleet_cases.restate's bytes; TwoCircles, square and L-shaped polygons at headings
0, pi / 2 and pi, and a line, are placed where they are computed by hand; the cut by rows and by vertices ends the list
at the first neighbour that does not fit; own vertices at the pool's end; the 0.001 rule; split tables equal the union,
in one process and over gloo with two and three ranks."""
import math
import os
import socket
import sys

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from teb_local_planner_b200 import distributed as D
from tests import fleet_cases as fc
from tests import fleet_shape_cases as fsc
from tests import fleet_table_cases as ftc
from tests.test_fleet_table_cases import _fleet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, CI, LI, PO = fsc.POINT, fsc.CIRCULAR, fsc.LINE, fsc.POLYGON
TWO_CIRCLES = [(CI, [[0.3, 0.0]], 0.25), (CI, [[-0.2, 0.0]], 0.2)]
SQUARE = [(PO, [[0.5, 0.5], [-0.5, 0.5], [-0.5, -0.5], [0.5, -0.5]])]
L_SHAPE = [(PO, [[0, 0], [2, 0], [2, 1], [1, 1], [1, 2], [0, 2]])]
LINE = [(LI, [[0.4, 0.0], [-0.4, 0.0]])]
KINDS = [[(CI, [[0.0, 0.0]], 0.3)], TWO_CIRCLES, SQUARE, L_SHAPE, LINE, [(P, [[0.0, 0.0]])]]


def _two(theta, kind, cmd=(0.3, 0.0), C_cap=8, PV_cap=16, kinds=KINDS):
    """robot 0 at the origin, robot 1 at (1, 2, theta) of the given kind: robot 0's rows"""
    pose = np.array([[0.0, 0.0, 0.0], [1.0, 2.0, theta]])
    cmds = np.array([[0.0, 0.0, 0.0], [cmd[0], cmd[1], 0.0]])
    out = fsc.restate(pose, cmds, kinds, [0, kind], 5.0, 8, np.zeros((2, C_cap), abi.OBST_DTYPE),
                      np.zeros((2, PV_cap, 2)))
    return out[0][0, :out[1][0]], out[4][0], out


def test_one_circle_at_the_origin_is_the_circle_step():
    for R, seed in ((1, 0), (40, 1), (97, 2)):
        f = _fleet(R, 10, seed)
        for rng in (0.0, 1.0, 4.0, math.inf):
            for max_rows in (0, 3, 8):
                for rho in (0.0, 0.35):
                    kinds = [[(CI, [[0.0, 0.0]], rho)]] if rho > 0 else [[(P, [[0.0, 0.0]])]]
                    want = fc.restate(f["pose"], f["last_cmd"], rho, rng, max_rows, f["custom"], f["own_count"], None,
                                      f["world"])
                    if rho == 0.0:      # a Point part: the circle row of radius 0 with type Point
                        written = np.arange(want[0].shape[1])[None, :] >= np.asarray(f["own_count"])[:, None]
                        written &= np.arange(want[0].shape[1])[None, :] < want[1][:, None]
                        want[0]["type"][written] = P
                    got = fsc.restate(f["pose"], f["last_cmd"], kinds, 0, rng, max_rows, f["custom"],
                                      own_count=f["own_count"], world=f["world"], PV_cap=0)
                    for a, b in zip(got[:4], want):
                        assert a.tobytes() == b.tobytes(), (R, rng, max_rows, rho)


@pytest.mark.parametrize("theta,c,s", [(0.0, 1.0, 0.0), (math.pi / 2, math.cos(math.pi / 2), 1.0),
                                       (math.pi, -1.0, math.sin(math.pi))])
def test_two_circles_square_and_l_shape_are_placed_by_hand(theta, c, s):
    place = lambda ux, uy: (1.0 + (c * ux - s * uy), 2.0 + (s * ux + c * uy))
    rows, _, _ = _two(theta, 1)
    assert list(rows["type"]) == [CI, CI] and list(rows["radius"]) == [0.25, 0.2]
    assert (rows["x"][0], rows["y"][0]) == place(0.3, 0.0) and (rows["x"][1], rows["y"][1]) == place(-0.2, 0.0)
    assert (rows["vertex_count"] == 0).all() and (rows["dynamic"] == 1).all()
    assert np.allclose(rows["vx"], 0.3 * c, atol=1e-15) and np.allclose(rows["vy"], 0.3 * s, atol=1e-15)
    rows, cv, _ = _two(theta, 2)
    assert rows["type"][0] == PO and rows["vertex_begin"][0] == 0 and rows["vertex_count"][0] == 4
    assert [tuple(v) for v in cv[:4]] == [place(0.5, 0.5), place(-0.5, 0.5), place(-0.5, -0.5), place(0.5, -0.5)]
    assert abs(rows["x"][0] - 1.0) < 1e-15 and abs(rows["y"][0] - 2.0) < 1e-15
    rows, cv, _ = _two(theta, 3)
    assert rows["vertex_count"][0] == 6
    # the L of area 3: a 2 x 1 rectangle centred at (1, 0.5) and a unit square at (0.5, 1.5), centroid (5/6, 5/6)
    gx, gy = place(5 / 6, 5 / 6)
    assert abs(rows["x"][0] - gx) < 1e-14 and abs(rows["y"][0] - gy) < 1e-14
    assert tuple(cv[0]) == (1.0, 2.0)           # the body origin is the position, unchanged


def test_a_line_and_the_point_kind():
    rows, cv, _ = _two(math.pi / 2, 4)
    assert rows["type"][0] == LI and rows["vertex_count"][0] == 2 and rows["vertex_begin"][0] == 0
    assert tuple(cv[0]) == (1.0 + (math.cos(math.pi / 2) * 0.4), 2.0 + 0.4)
    assert rows["x"][0] == 0.5 * (cv[0][0] + cv[1][0]) and rows["y"][0] == 0.5 * (cv[0][1] + cv[1][1])
    rows, cv, _ = _two(0.3, 5)
    assert rows["type"][0] == P and (rows["x"][0], rows["y"][0]) == (1.0, 2.0) and rows["radius"][0] == 0.0


def test_the_0001_rule():
    for cmd, dyn in (((0.0009, 0.0), 0), ((0.0, 0.001), 1), ((0.0006, 0.0008), 1), ((0.0, 0.0), 0)):
        rows, _, _ = _two(1.0, 1, cmd=cmd)
        assert (rows["dynamic"] == dyn).all()
        if not dyn:
            assert (rows["vx"] == 0).all() and (rows["vy"] == 0).all()


def _line_fleet(kinds_of):
    """robot 0 at the origin; robots 1 .. n on the x axis at 1, 2, ... with the given kinds"""
    n = len(kinds_of)
    pose = np.array([[float(i), 0.0, 0.0] for i in range(n + 1)])
    return pose, np.zeros((n + 1, 3)), [0] + list(kinds_of)


def test_the_cut_by_rows_and_by_vertices_ends_the_list():
    # rows: circle (1), two circles (2), circle (1) with 3 rows free: the two circles fit (1 + 2 = 3), the last does not
    pose, cmd, kind = _line_fleet([0, 1, 0])
    out = fsc.restate(pose, cmd, KINDS, kind, 10.0, 8, np.zeros((4, 4), abi.OBST_DTYPE), np.zeros((4, 16, 2)),
                      own_count=[1, 0, 0, 0])
    assert out[1][0] == 4 and out[2][0] == 3 and out[3][0] == fc.TRUNCATED
    # a large neighbour stops the list though a smaller one behind it would fit: square (4 points) then line (2) in 5
    pose, cmd, kind = _line_fleet([4, 2, 4])
    out = fsc.restate(pose, cmd, KINDS, kind, 10.0, 8, np.zeros((4, 8), abi.OBST_DTYPE), np.zeros((4, 5, 2)))
    assert out[1][0] == 1 and out[0][0]["type"][0] == LI and out[3][0] == fc.TRUNCATED
    assert (out[4][0][2:] == 0).all()
    # rows: two circles (2) behind a circle, with 2 rows free: the circle only, the point behind is not taken
    pose, cmd, kind = _line_fleet([0, 1, 5])
    out = fsc.restate(pose, cmd, KINDS, kind, 10.0, 8, np.zeros((4, 2), abi.OBST_DTYPE), np.zeros((4, 0, 2)), PV_cap=0)
    assert out[1][0] == 1 and out[3][0] == fc.TRUNCATED and out[2][0] == 3


def test_own_vertices_at_the_pools_end():
    pose, cmd, kind = _line_fleet([2, 4])
    cv = np.full((3, 8, 2), 7.0)
    for ownv, rows_written in ((4, 1), (5, 0), (8, 0), (2, 2)):
        out = fsc.restate(pose, cmd, KINDS, kind, 10.0, 8, np.zeros((3, 4), abi.OBST_DTYPE), cv,
                          own_vertex_count=[ownv, 0, 0])
        assert out[1][0] == rows_written, ownv
        assert (out[4][0][:ownv] == 7.0).all()
        if rows_written:
            assert out[0][0]["vertex_begin"][0] == ownv
    out = fsc.restate(pose, cmd, KINDS, kind, 10.0, 8, np.zeros((3, 4), abi.OBST_DTYPE), cv, own_vertex_count=[9, 0, 0])
    assert out[2][0] == -1 and out[3][0] == fc.BAD_INPUT


def _mixed(R, seed):
    f = _fleet(R, 12, seed)
    return f, np.random.default_rng(seed).integers(0, len(KINDS), R).astype(np.int32)


@pytest.mark.parametrize("R,counts", [(40, [40]), (40, [13, 27]), (97, [30, 1, 40, 26]), (64, [8] * 8)])
def test_split_tables_equal_the_union(R, counts):
    f, kind = _mixed(R, R + len(counts))
    cv = np.zeros((R, 24, 2))
    ownv = np.random.default_rng(3).integers(0, 25, R).astype(np.int32)
    for rng in (1.0, 4.0, math.inf):
        for max_rows in (0, 3, 8):
            want = fsc.restate(f["pose"], f["last_cmd"], KINDS, kind, rng, max_rows, f["custom"], cv, f["own_count"],
                               None, ownv, f["world"])
            got, _ = fsc.sharded(f["pose"], f["last_cmd"], KINDS, kind, rng, max_rows, f["custom"], cv, counts,
                                 f["own_count"], ownv, f["world"])
            for a, b in zip(got, want):
                assert a.tobytes() == b.tobytes(), (counts, rng, max_rows)
    assert (want[3] == fc.TRUNCATED).any()


def test_fleet_shape_from_params():
    p = abi.default_params()
    p.footprint_type = abi.TEB_FOOTPRINT_TWO_CIRCLES
    p.footprint_front_offset, p.footprint_front_radius, p.footprint_rear_offset, p.footprint_rear_radius = 0.3, 0.2, 0.1, 0.0
    assert abi.fleet_shape_from_params(p) == [(CI, [[0.3, 0.0]], 0.2), (P, [[-0.1, 0.0]])]
    p.footprint_type, p.footprint_vertex_count = abi.TEB_FOOTPRINT_POLYGON, 3
    p.footprint_vertices[:6] = [1, 0, 0, 1, -1, 0]
    assert abi.fleet_shape_from_params(p) == [(PO, [[1, 0], [0, 1], [-1, 0]])]
    sh = abi.make_fleet_shapes(KINDS, PV_cap=16)
    assert sh.K == len(KINDS) and list(sh._keep["kind_parts"]) == [0, 1, 3, 4, 5, 6, 7]
    assert list(sh._keep["part_vertices"]) == [0, 1, 2, 3, 7, 13, 15, 16]


# ---- over gloo, one process per rank
GLOO_R = 37


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _gloo_worker(rank, world, port, out_dir, counts):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from teb_local_planner_b200 import distributed as D
    from tests import fleet_shape_cases as fsc
    from tests import fleet_table_cases as ftc
    from tests.test_fleet_shape_cases import KINDS, _mixed
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    f, kind = _mixed(GLOO_R, 9)
    cap, first = D.fleet_layout(counts, world)
    lo, hi = ftc.split(GLOO_R, counts)[rank]
    rows, head, rk = ftc.padding(world * cap), np.zeros(world * cap), np.zeros(world * cap, np.int32)
    pub = fsc.publish(f["pose"][lo:hi], f["last_cmd"][lo:hi], 0.0, kind[lo:hi], f["world"][lo:hi])
    sl = slice(first[rank], first[rank] + hi - lo)
    rows[sl], head[sl], rk[sl] = pub
    tab, head, rk = D.gather_fleet_table_torch(rows, cap, rank, world, heading=head, row_kind=rk)
    out = fsc.restate_table(tab, head, rk, KINDS, first[rank], hi - lo, 2.5, 8, f["custom"][lo:hi],
                            np.zeros((hi - lo, 24, 2)), f["own_count"][lo:hi])
    for k in range(5):
        np.save(os.path.join(out_dir, f"out{k}_{rank}.npy"), out[k])
    dist.destroy_process_group()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("world,counts", [(2, [20, 17]), (3, [12, 1, 24])])
def test_gloo_ranks_gather_the_table_and_its_companions(tmp_path, world, counts):
    import torch.multiprocessing as mp
    mp.spawn(_gloo_worker, args=(world, _free_port(), str(tmp_path), counts), nprocs=world, join=True)
    f, kind = _mixed(GLOO_R, 9)
    want = fsc.restate(f["pose"], f["last_cmd"], KINDS, kind, 2.5, 8, f["custom"], np.zeros((GLOO_R, 24, 2)),
                       f["own_count"], None, None, f["world"])
    for k in range(5):
        got = np.concatenate([np.load(tmp_path / f"out{k}_{r}.npy") for r in range(world)])
        assert got.tobytes() == want[k].tobytes(), k
    assert (want[2] > 0).any()
