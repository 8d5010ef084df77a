"""tests/fleet_reach_cases.py, the restatement the footprints' neighbour rule (TEB_FLEET_SELECT_FOOTPRINTS) is held to,
pinned on hand-computed fleets: two 4 m robots nose to tail are neighbours by their footprints and not by their centres;
a small robot and a truck swap places in the kept list; a Circular model and one-circle kinds give d - a - b; a Point
model and point kinds give the centres' neighbours; the row, C_cap and vertex cuts on the new order; range 0 and inf,
coincident robots and NaN; split tables equal the union. Then the prefilter: no pair whose gap is within range fails
it, at the R' bound and over millions of random circle / point pairs."""
import math
import os
import socket
import sys

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import fleet_cases as fc
from tests import fleet_reach_cases as frc
from tests import fleet_shape_cases as fsc
from tests import fleet_table_cases as ftc
from tests.test_fleet_table_cases import _fleet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

P, CI, LI, PO = fsc.POINT, fsc.CIRCULAR, fsc.LINE, fsc.POLYGON
LONG = [(PO, [[2.0, 0.5], [-2.0, 0.5], [-2.0, -0.5], [2.0, -0.5]])]          # 4 x 1 m
SMALL = [(PO, [[0.25, 0.15], [-0.25, 0.15], [-0.25, -0.15], [0.25, -0.15]])]  # 0.5 x 0.3 m


def params(kind="polygon", **kw):
    p = abi.default_params()
    if kind == "polygon":
        verts = kw.get("verts", LONG[0][1])
        p.footprint_type = abi.TEB_FOOTPRINT_POLYGON
        p.footprint_vertex_count = len(verts)
        for i, (x, y) in enumerate(verts):
            p.footprint_vertices[2 * i], p.footprint_vertices[2 * i + 1] = x, y
    elif kind == "circular":
        p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, kw["radius"]
    elif kind == "two_circles":
        p.footprint_type = abi.TEB_FOOTPRINT_TWO_CIRCLES
        p.footprint_front_offset, p.footprint_front_radius = 0.2, 0.25
        p.footprint_rear_offset, p.footprint_rear_radius = 0.2, 0.25
    elif kind == "line":
        p.footprint_type = abi.TEB_FOOTPRINT_LINE
        p.footprint_line[:] = [0.3, 0.0, -0.3, 0.0]
    else:
        p.footprint_type = abi.TEB_FOOTPRINT_POINT
    return p


def _run(prm, pose, kinds, kind, rng, max_rows=8, C_cap=16, PV_cap=64, own_count=None, own_vertex_count=None):
    pose = np.asarray(pose, np.float64)
    R = len(pose)
    gaps = {}
    out = frc.restate(prm, pose, np.zeros((R, 3)), kinds, kind, rng, max_rows, np.zeros((R, C_cap), abi.OBST_DTYPE),
                      np.zeros((R, PV_cap, 2)), own_count=own_count, own_vertex_count=own_vertex_count, gaps=gaps)
    return out, gaps


@pytest.mark.parametrize("theta", [0.0, math.pi / 2, math.pi])
def test_nose_to_tail_long_robots_are_footprint_neighbours(theta):
    c, s = round(math.cos(theta)), round(math.sin(theta))
    pose = [[0.0, 0.0, theta], [4.5 * c, 4.5 * s, theta]]
    out, gaps = _run(params(), pose, [LONG], 0, 3.0)
    assert list(out[2]) == [1, 1] and list(out[3]) == [fc.WRITTEN] * 2
    for r in (0, 1):
        assert list(gaps[r][0]) == [1 - r] and abs(gaps[r][1][0] - 0.5) < 1e-12
    centres = fsc.restate(pose, np.zeros((2, 3)), [LONG], 0, 3.0, 8, np.zeros((2, 16), abi.OBST_DTYPE), np.zeros((2, 64, 2)))
    assert list(centres[2]) == [0, 0]
    # the rows are the shaped writer's: the same bytes as the centre rule writes for a neighbour it keeps
    wide = fsc.restate(pose, np.zeros((2, 3)), [LONG], 0, 5.0, 8, np.zeros((2, 16), abi.OBST_DTYPE), np.zeros((2, 64, 2)))
    for a, b in zip(out, wide):
        assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("theta", [0.0, math.pi / 2, math.pi])
def test_truck_corner_comes_before_a_nearer_small_centre(theta):
    c, s = round(math.cos(theta)), round(math.sin(theta))
    rot = lambda x, y: [c * x - s * y, s * x + c * y]
    # robot 0 a circle of 0.2 at the origin; robot 1 a circle of 0.2, centre 2 m away (body 1.6 m); robot 2 a 4 x 1 m
    # truck, centre 2.5 m away, across the line to it, its near side 0.5 m away (body 0.3 m)
    kinds = [[(CI, [[0.0, 0.0]], 0.2)], LONG]
    pose = [[0.0, 0.0, theta], rot(2.0, 0.0) + [theta], rot(0.0, 2.5) + [theta + math.pi / 2]]
    prm = params("circular", radius=0.2)
    out, gaps = _run(prm, pose, kinds, [0, 0, 1], 3.0, max_rows=1)
    assert list(gaps[0][0]) == [2, 1]
    assert abs(gaps[0][1][0] - 0.3) < 1e-12 and abs(gaps[0][1][1] - 1.6) < 1e-12
    assert out[2][0] == 2 and out[3][0] == fc.TRUNCATED and out[0][0, 0]["type"] == PO
    centres = fsc.restate(pose, np.zeros((3, 3)), kinds, [0, 0, 1], 3.0, 1, np.zeros((3, 16), abi.OBST_DTYPE),
                          np.zeros((3, 64, 2)))
    assert centres[0][0, 0]["type"] == CI


def test_circular_model_and_circle_kinds_give_d_minus_a_minus_b():
    a, b = 0.5, 0.25
    prm = params("circular", radius=a)
    for d, th in ((3.0, 0.0), (1.5, math.pi / 2), (0.75, math.pi), (4.0, 1.0)):
        pose = [[1.0, -2.0, th], [1.0 + d, -2.0, -th]]
        out, gaps = _run(prm, pose, [[(CI, [[0.0, 0.0]], b)]], 0, 3.0)
        want = d - b - a
        if want <= 3.0:
            assert gaps[0][1][0] == want and gaps[1][1][0] == want
        else:
            assert out[2][0] == 0


def test_point_model_and_point_kinds_agree_with_the_centres():
    prm = params("point")
    f = _fleet(60, 8, 3, worlds=1)
    for rng in (0.5, 1.5, 3.0):
        out, gaps = _run(prm, f["pose"], [[(P, [[0.0, 0.0]])]], 0, rng, max_rows=5, C_cap=8, PV_cap=0)
        want = fsc.restate(f["pose"], np.zeros((60, 3)), [[(P, [[0.0, 0.0]])]], 0, rng, 5,
                           np.zeros((60, 8), abi.OBST_DTYPE), np.zeros((60, 0, 2)))
        d = np.hypot(f["pose"][:, None, 0] - f["pose"][None, :, 0], f["pose"][:, None, 1] - f["pose"][None, :, 1])
        assert np.all(np.abs(d - rng) > 1e-9)       # no pair at the boundary
        for r in range(60):
            idx, _ = fc.neighbours(f["pose"], r, rng)
            assert list(gaps[r][0]) == list(idx)
        for a, b in zip(out[:4], want[:4]):
            # the order of coincident robots is (0, q) either way, so the rows agree byte for byte
            assert a.tobytes() == b.tobytes()


def test_cuts_follow_the_gap_order():
    prm = params("point")
    # robot 0 at the origin; robot 1 a point 1.0 away; robot 2 a long robot whose side is 0.5 away; robot 3 a small
    # robot whose side is 0.25 away: the gap order is 3, 2, 1 (the centre order 1, 3, 2)
    kinds = [[(P, [[0.0, 0.0]])], LONG, SMALL]
    pose = [[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, -0.4, 0.0]]
    kind = [0, 0, 1, 2]
    out, gaps = _run(prm, pose, kinds, kind, 3.0)
    assert list(gaps[0][0]) == [3, 2, 1] and list(out[2][:1]) == [3]
    rows = lambda o: [int(t) for t in o[0][0, :o[1][0]]["type"]]
    assert rows(out) == [PO, PO, P]
    out, _ = _run(prm, pose, kinds, kind, 3.0, max_rows=2)
    assert rows(out) == [PO, PO] and out[3][0] == fc.TRUNCATED
    out, _ = _run(prm, pose, kinds, kind, 3.0, C_cap=3, own_count=[1, 0, 0, 0])
    assert rows(out)[1:] == [PO, PO] and out[1][0] == 3
    out, _ = _run(prm, pose, kinds, kind, 3.0, PV_cap=7)    # 4 + 4 points do not fit: the list ends at the second
    assert rows(out) == [PO] and out[3][0] == fc.TRUNCATED and out[2][0] == 3
    out, _ = _run(prm, pose, kinds, kind, 3.0, PV_cap=8, own_vertex_count=[1, 0, 0, 0])
    assert rows(out) == [PO] and out[0][0, 0]["vertex_begin"] == 1


def test_range_zero_inf_coincident_and_nan():
    prm = params()
    pose = [[0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [4.0, 0.0, 0.0], [100.0, 0.0, 1.0]]
    out, gaps = _run(prm, pose, [LONG], 0, 0.0)
    assert list(gaps[0][0]) == [1, 2] and list(gaps[0][1]) == [0.0, 0.0]    # coincident, and touching end to end
    assert out[2][3] == 0
    out, gaps = _run(prm, pose, [LONG], 0, math.inf)
    assert list(out[2]) == [3, 3, 3, 3] and list(gaps[3][0]) == [2, 0, 1]
    nan = [[0.0, 0.0, 0.0], [math.nan, 0.0, 0.0], [1.0, 0.0, math.nan]]
    out, gaps = _run(prm, nan, [LONG], 0, 5.0)
    assert list(out[2]) == [0, 0, 0]             # a NaN centre fails the prefilter, a NaN heading gives a NaN gap
    out, gaps = _run(prm, nan, [LONG], 0, math.inf)
    # at range inf R' is inf, and still a NaN centre fails it; a NaN heading leaves the distance code with no edge
    # closer than its start value, which range inf takes
    assert list(out[2]) == [1, 0, 1] and list(gaps[0][0]) == [2]


@pytest.mark.parametrize("model", ["point", "circular", "two_circles", "line", "polygon"])
def test_split_tables_equal_the_union(model):
    prm = params(model, radius=0.3)
    f = _fleet(36, 12, 5)
    kinds = [SMALL, LONG, [(CI, [[0.3, 0.0]], 0.25), (CI, [[-0.3, 0.0]], 0.25)], [(LI, [[0.5, 0.0], [-0.5, 0.0]])]]
    kind = np.arange(36) % 4
    cv = np.zeros((36, 24, 2))
    want = frc.restate(prm, f["pose"], f["last_cmd"], kinds, kind, 1.5, 4, f["custom"], cv, f["own_count"],
                       world=f["world"])
    for counts in ((36,), (10, 0, 26), (5, 7, 11, 13)):
        got, _ = frc.sharded(prm, f["pose"], f["last_cmd"], kinds, kind, 1.5, 4, f["custom"], cv, counts,
                             f["own_count"], world=f["world"])
        for a, b in zip(got, want):
            assert a.tobytes() == b.tobytes(), counts


def _assert_prefilter(xr, yr, xq, yq, a, b, rng):
    """gap <= range implies d2 <= R'^2, the circle / point gap in closed form as the distance code computes it"""
    dx, dy = xr - xq, yr - yq
    g = np.sqrt(dx * dx + dy * dy) - b - a
    pre = (rng + a + b) * frc.MARGIN
    ex, ey = xq - xr, yq - yr
    d2 = ex * ex + ey * ey
    bad = (g <= rng) & ~(d2 <= pre * pre)
    assert not bad.any(), np.nonzero(bad)


def test_prefilter_keeps_every_pair_at_the_bound():
    gen = np.random.default_rng(11)
    n = 200000
    for scale in (1e-6, 1.0, 1e3, 1e6):
        rng = gen.uniform(0, 3, n) * scale
        rng[:100] = 0.0
        a = gen.uniform(0, 1, n) * scale * (gen.random(n) < 0.7)
        b = gen.uniform(0, 1, n) * scale * (gen.random(n) < 0.7)
        h = (rng + a + b) * frc.MARGIN
        # centres near the cell bound 2^24 h, the pair at the largest distance the gap allows and a few ulps either side
        xr = gen.uniform(-1, 1, n) * h * 2.0 ** 23
        yr = gen.uniform(-1, 1, n) * h * 2.0 ** 23
        phi = gen.uniform(0, 2 * math.pi, n)
        d = (rng + a + b) * (1 + gen.integers(-8, 9, n) * 2.0 ** -52)
        _assert_prefilter(xr, yr, xr + d * np.cos(phi), yr + d * np.sin(phi), a, b, rng)


def test_prefilter_keeps_off_centre_parts_near_the_cell_bound():
    """the footprint's front circle and the candidate's front part face each other across the centre line, so the gap
    is D - E_r - E_lib: pairs at the R' bound, centres near the cell bound, the gap through the oracle's distance code
    (placed points, rotation and the distance code's rounding)"""
    prm = params("two_circles")                              # circles of 0.25 at +-0.2: E_r = 0.45
    kind = [(CI, [[0.3, 0.0]], 0.25), (CI, [[-0.3, 0.0]], 0.25)]   # E_lib = 0.55
    gen = np.random.default_rng(13)
    checked = 0
    for rng in (0.0, 1e-3, 0.7, 3.0):
        pre = frc.prefilter(prm, [kind], rng)
        assert frc.footprint_reach(prm) == 0.45 and frc.library_reach([kind]) == 0.55
        for _ in range(300):
            phi = gen.uniform(-math.pi, math.pi)
            xr, yr = gen.uniform(-1, 1, 2) * pre * 2.0 ** 23
            d = (rng + 1.0) * (1 + int(gen.integers(-64, 65)) * 2.0 ** -52)
            xq, yq = xr + d * math.cos(phi), yr + d * math.sin(phi)
            g = frc.gap(prm, [xr, yr, phi], xq, yq, phi + math.pi, kind)
            assert abs(g - (d - 1.0)) <= 1e-6 * pre
            if g <= rng:
                ex, ey = xq - xr, yq - yr
                assert ex * ex + ey * ey <= pre * pre, (rng, xr, yr, phi, d, g)
                checked += 1
    assert checked > 100


def test_prefilter_keeps_every_pair_of_random_circles_and_points():
    gen = np.random.default_rng(12)
    for _ in range(20):
        n = 200000
        scale = 10.0 ** gen.uniform(-3, 3)
        rng = gen.uniform(0, 3, n) * scale
        a = gen.uniform(0, 1, n) * scale * (gen.random(n) < 0.5)
        b = gen.uniform(0, 1, n) * scale * (gen.random(n) < 0.5)
        xr, yr = gen.uniform(-1e4, 1e4, (2, n)) * scale
        xq, yq = xr + gen.normal(0, 2, n) * scale, yr + gen.normal(0, 2, n) * scale
        _assert_prefilter(xr, yr, xq, yq, a, b, rng)


# ---- over gloo, one process per rank, each rank measuring with its own context's footprint
GLOO_R = 37
GLOO_MODELS = ["polygon", "two_circles", "circular"]
GLOO_KINDS = [SMALL, LONG, [(CI, [[0.3, 0.0]], 0.25), (CI, [[-0.3, 0.0]], 0.25)], [(LI, [[0.5, 0.0], [-0.5, 0.0]])]]


def _gloo_fleet():
    f = _fleet(GLOO_R, 12, 9)
    return f, (np.arange(GLOO_R) % len(GLOO_KINDS)).astype(np.int32)


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
    from tests import fleet_reach_cases as frc
    from tests import fleet_shape_cases as fsc
    from tests import fleet_table_cases as ftc
    from tests.test_fleet_reach_cases import GLOO_KINDS, GLOO_MODELS, _gloo_fleet, params
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    f, kind = _gloo_fleet()
    cap, first = D.fleet_layout(counts, world)
    lo, hi = ftc.split(GLOO_R, counts)[rank]
    rows, head, rk = ftc.padding(world * cap), np.zeros(world * cap), np.zeros(world * cap, np.int32)
    pub = fsc.publish(f["pose"][lo:hi], f["last_cmd"][lo:hi], 0.0, kind[lo:hi], f["world"][lo:hi])
    sl = slice(first[rank], first[rank] + hi - lo)
    rows[sl], head[sl], rk[sl] = pub
    tab, head, rk = D.gather_fleet_table_torch(rows, cap, rank, world, heading=head, row_kind=rk)
    out = frc.restate_table(params(GLOO_MODELS[rank], radius=0.3), tab, head, rk, GLOO_KINDS, first[rank], hi - lo,
                            1.5, 8, f["custom"][lo:hi], np.zeros((hi - lo, 24, 2)), f["own_count"][lo:hi])
    for k in range(5):
        np.save(os.path.join(out_dir, f"out{k}_{rank}.npy"), out[k])
    dist.destroy_process_group()


@pytest.mark.timeout(180)
@pytest.mark.parametrize("world,counts", [(2, [20, 17]), (3, [12, 1, 24])])
def test_gloo_ranks_equal_one_call_on_the_union(tmp_path, world, counts):
    import torch.multiprocessing as mp
    mp.spawn(_gloo_worker, args=(world, _free_port(), str(tmp_path), counts), nprocs=world, join=True)
    f, kind = _gloo_fleet()
    parts = ftc.split(GLOO_R, counts)
    # rank g's robots are measured with rank g's footprint: one array call per footprint on the union, each rank's
    # robots taken from its own
    whole = [frc.restate(params(GLOO_MODELS[g], radius=0.3), f["pose"], f["last_cmd"], GLOO_KINDS, kind, 1.5, 8,
                         f["custom"], np.zeros((GLOO_R, 24, 2)), f["own_count"], world=f["world"]) for g in range(world)]
    for k in range(5):
        want = np.concatenate([whole[g][k][lo:hi] for g, (lo, hi) in enumerate(parts)])
        got = np.concatenate([np.load(tmp_path / f"out{k}_{r}.npy") for r in range(world)])
        assert got.tobytes() == want.tobytes(), k
    assert (np.concatenate([whole[g][2][lo:hi] for g, (lo, hi) in enumerate(parts)]) > 0).any()
