"""tests/fleet_cases.py, the restatement tebgpu_fleet_obstacles is held to, pinned on hand-computed fleets: a neighbour
exactly at range, equal distances, coincident robots, a robot alone in its world, max_rows and C_cap cutting the list
behind the caller's own rows, the 0.001 speed rule on both sides of the boundary, a heading of pi / 2, shared and
out-of-range scenes, and the scenes no robot writes."""
import math

import numpy as np

from teb_local_planner_b200 import abi
from tests import fleet_cases as fc


def _empty(S, C_cap, fill=0):
    c = np.zeros((S, C_cap), abi.OBST_DTYPE)
    c.view(np.uint8)[:] = fill
    return c


def test_a_neighbour_exactly_at_range_counts():
    pose = [(0.0, 0.0, 0.0), (3.0, 4.0, 0.0), (3.0, 4.000000000001, 0.0)]
    idx, d2 = fc.neighbours(pose, 0, 5.0)
    assert list(idx) == [1] and d2[0] == 25.0
    out, cc, need, st = fc.restate(pose, np.zeros((3, 3)), 0.2, 5.0, 8, _empty(3, 4))
    assert list(need) == [1, 2, 1] and list(st) == [fc.WRITTEN] * 3 and list(cc) == [1, 2, 1]
    assert (out[0, 0]["x"], out[0, 0]["y"]) == (3.0, 4.0)
    assert list(fc.neighbours(pose, 2, 5.0)[0]) == [1]       # (3, 4.000000000001) is 5.000000000001 from the origin


def test_equal_distances_go_to_the_lower_index():
    pose = [(0.0, 0.0, 0.0), (0.0, 1.0, 0.0), (-1.0, 0.0, 0.0), (1.0, 0.0, 0.0), (0.0, -1.0, 0.0)]
    idx, d2 = fc.neighbours(pose, 0, 1.0)
    assert list(idx) == [1, 2, 3, 4] and list(d2) == [1.0] * 4
    out, cc, need, st = fc.restate(pose, np.zeros((5, 3)), 0.3, 1.0, 2, _empty(5, 8))
    assert need[0] == 4 and st[0] == fc.TRUNCATED and cc[0] == 2
    assert [(o["x"], o["y"]) for o in out[0, :2]] == [(0.0, 1.0), (-1.0, 0.0)]
    # from robot 1: robot 0 at d2 = 1, then robots 2 and 3 both at d2 = 2 (range 2 takes them), robot 4 at 4
    idx, d2 = fc.neighbours(pose, 1, 2.0)
    assert list(idx) == [0, 2, 3, 4] and list(d2) == [1.0, 2.0, 2.0, 4.0]


def test_coincident_robots_are_neighbours():
    pose = [(1.5, -2.0, 0.3), (1.5, -2.0, 2.0)]
    out, cc, need, st = fc.restate(pose, np.zeros((2, 3)), [0.25, 0.5], 0.0, 4, _empty(2, 4))
    assert list(need) == [1, 1] and list(cc) == [1, 1]
    assert out[0, 0]["radius"] == 0.5 and out[1, 0]["radius"] == 0.25
    assert out[0, 0]["x"] == 1.5 and out[0, 0]["type"] == fc.TEB_OBST_CIRCULAR


def test_a_robot_alone_in_its_world():
    pose = [(0.0, 0.0, 0.0), (0.1, 0.0, 0.0), (0.05, 0.0, 0.0)]
    out, cc, need, st = fc.restate(pose, np.zeros((3, 3)), 0.2, 10.0, 8, _empty(3, 4), own_count=[1, 0, 2],
                                   world=[7, 7, 3])
    assert list(need) == [1, 1, 0] and list(st) == [fc.WRITTEN] * 3
    assert list(cc) == [2, 1, 2]
    assert out[0, 1]["x"] == 0.1 and out[1, 0]["x"] == 0.0


def test_max_rows_and_c_cap_cut_behind_the_own_rows():
    pose = [(0.0, 0.0, 0.0)] + [(0.5 * k, 0.0, 0.0) for k in range(1, 7)]
    R = len(pose)
    mine = _empty(R, 5, fill=0xAB)
    own = np.zeros(R, np.int32)
    own[0] = 3
    out, cc, need, st = fc.restate(pose, np.zeros((R, 3)), 0.1, 100.0, 4, mine, own_count=own)
    # robot 0: 6 neighbours, max_rows 4, but C_cap - own = 2 rows left: the two nearest follow the own rows
    assert need[0] == 6 and st[0] == fc.TRUNCATED and cc[0] == 5
    assert [o["x"] for o in out[0, 3:5]] == [0.5, 1.0]
    assert out[0, :3].tobytes() == mine[0, :3].tobytes()
    # robot 6 (own 0): max_rows 4 of its 6
    assert cc[6] == 4 and [o["x"] for o in out[6, :4]] == [2.5, 2.0, 1.5, 1.0]
    assert out[6, 4].tobytes() == mine[6, 4].tobytes()
    # max_rows 0: nothing written, the count is still reported
    out, cc, need, st = fc.restate(pose, np.zeros((R, 3)), 0.1, 100.0, 0, mine, own_count=own)
    assert list(cc) == list(own) and list(need) == [6] * R and (st == fc.TRUNCATED).all()
    assert out.tobytes() == mine.tobytes()


def test_the_speed_rule_at_its_boundary():
    below = math.nextafter(0.001, 0.0)
    pose = [(0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (2.0, 0.0, 0.0)]
    cmd = [(0.0, 0.0, 0.0), (0.001, 0.0, 0.5), (below, 0.0, 0.0)]
    out, cc, need, st = fc.restate(pose, cmd, 0.2, 10.0, 8, _empty(3, 4))
    rows = {float(o["x"]): o for o in out[0, :2]}
    assert rows[1.0]["dynamic"] == 1 and rows[1.0]["vx"] == 0.001 and rows[1.0]["vy"] == 0.0
    assert rows[2.0]["dynamic"] == 0 and rows[2.0]["vx"] == 0.0 and rows[2.0]["vy"] == 0.0
    # a still robot is a static circle, and omega is not read
    assert out[1, 0]["dynamic"] == 0 and out[1, 0]["x"] == 0.0


def test_a_heading_of_half_pi_rotates_the_command():
    pose = [(0.0, 0.0, 0.0), (1.0, 1.0, math.pi / 2)]
    cmd = [(0.0, 0.0, 0.0), (0.4, 0.1, 0.0)]
    out, *_ = fc.restate(pose, cmd, 0.2, 10.0, 8, _empty(2, 1))
    o = out[0, 0]
    assert o["dynamic"] == 1
    assert abs(o["vx"] - (-0.1)) <= 1e-16 and abs(o["vy"] - 0.4) <= 1e-16
    assert o["vx"] == math.cos(math.pi / 2) * 0.4 - 1.0 * 0.1 and o["vy"] == 1.0 * 0.4 + math.cos(math.pi / 2) * 0.1


def test_shared_and_out_of_range_scenes():
    pose = [(0.0, 0.0, 0.0), (0.5, 0.0, 0.0), (1.0, 0.0, 0.0), (1.5, 0.0, 0.0)]
    start = _empty(5, 3, fill=0x11)
    out, cc, need, st = fc.restate(pose, np.zeros((4, 3)), 0.2, 10.0, 8, start, own_count=[0, 4, 0, 1, 0],
                                   custom_count=[9, 9, 9, 9, 9], scene=[2, 2, 5, 1])
    assert list(st) == [fc.SHARED_SCENE, fc.SHARED_SCENE, fc.BAD_INPUT, fc.BAD_INPUT]
    assert list(need) == [-1] * 4 and list(cc) == [9] * 5 and out.tobytes() == start.tobytes()
    out, cc, need, st = fc.restate(pose, np.zeros((4, 3)), 0.2, 10.0, 8, start, own_count=[0, 1, 0, 1, 0],
                                   custom_count=[9, 9, 9, 9, 9], scene=[4, 0, 2, 1])
    assert list(st) == [fc.WRITTEN, fc.WRITTEN, fc.WRITTEN, fc.TRUNCATED] and list(need) == [3] * 4
    assert list(cc) == [3, 3, 3, 9, 3]
    assert [o["x"] for o in out[4]] == [0.5, 1.0, 1.5] and [o["x"] for o in out[1, 1:]] == [1.0, 0.5]
