"""The local-plan restatement of tests/local_plan_cases.py pinned on hand-computed cases, one boundary of the reference's
loops at a time (teb_local_planner_ros.cpp:268-340). CPU only.

Unless a case says otherwise the costmap is 40 x 40 cells at 0.25 m, so the window is (40 * 0.25 / 2 * 0.85)^2 = 4.25^2 =
18.0625 exactly, the length limit is off, the robot moves (so the goal is never reached) and the orientation is not
overwritten, so no trig touches a row."""
import ctypes as C
import math

import pytest

from teb_local_planner_b200 import abi
from tests import local_plan_cases as lp

NAN = math.nan
MOVING = (1.0, 0.0, 0.0)


def run(rows, robot=(0.0, 0.0, 0.0), begin=0, vel=MOVING, grid=(40, 40), res=0.25, **kw):
    extra = {k: kw.pop(k) for k in ("custom_via_count", "infeasible_count", "since", "P_cap", "V_cap") if k in kw}
    a = lp.Args(**{"max_lookahead_dist": 0.0, "overwrite_orientation": False, **kw})
    rows = [(float(r[0]), float(r[1]), float(r[2]) if len(r) > 2 else 0.0) for r in rows]
    return lp.restate(rows, begin, len(rows), robot, vel, grid, res, a, **extra)


def line(xs, y=0.0):
    return [(x, y, 0.0) for x in xs]


def xs(out):
    return [r[0] for r in out.plan[1:]]


def test_window_is_the_dyadic_one():
    assert (40.0 * 0.25 / 2.0) * 0.85 == 4.25


# ---- 1. prune
def test_prune_distance_tie_is_not_pruned():
    o = run(line([0, 1, 2, 3]), robot=(1.0, 0.0, 0.0), prune_distance=1.0)   # row 0 at exactly 1 m: 1 < 1 is false
    assert o.plan_begin == 1


def test_nothing_to_prune_leaves_the_begin():
    o = run(line([0, 1, 2, 3]), robot=(0.0, 10.0, 0.0), begin=2, prune_distance=1.0)
    assert o.plan_begin == 2 and o.result == lp.PLANNED


def test_first_row_already_close():
    o = run(line([0, 1, 2, 3]), robot=(0.0, 0.0, 0.0), begin=0)
    assert o.plan_begin == 0 and o.goal_idx == 3 and xs(o) == [1, 2, 3]


def test_empty_plan():
    o = run(line([0, 1]), begin=2)
    assert o.result == lp.EMPTY and o.plan == [] and o.goal_idx is None and o.needed is None


# ---- 3. closest row
def test_loop_past_the_robot_takes_the_first_minimum_below_005():
    rows = line([0.1, 0.5, 1.0]) + [(1.0, 1.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 0.0), (-1.0, 0.0, 0.0)]
    o = run(rows)
    assert o.plan_begin == 0 and o.needed[0] == 7                          # from row 0, not the exact hit at row 5


def test_without_a_row_below_005_the_global_minimum_wins():
    o = run(line([1.0, 0.5, 2.0, 0.2, 3.0, 0.3]), prune_distance=1.5)
    assert o.plan_begin == 0 and xs(o) == [3.0, 0.3]                     # rows 3 .. 5


def test_exactly_005_does_not_stop_the_search():
    e = (0.152, 0.164, 0.0)
    assert 0.152 * 0.152 + 0.164 * 0.164 == 0.05
    o = run([e, (1.0, 0.0, 0.0), (0.3, 0.0, 0.0), (0.2, 0.0, 0.0), (2.0, 0.0, 0.0)], prune_distance=2.0)
    assert xs(o) == [2.0] and o.needed[0] == 2                              # closest: row 3 (0.04)
    o = run([(0.15, 0.164, 0.0), (1.0, 0.0, 0.0), (0.3, 0.0, 0.0), (0.2, 0.0, 0.0), (2.0, 0.0, 0.0)], prune_distance=2.0)
    assert o.needed[0] == 5                                                 # 0.0494 < 0.05: row 0, break at row 1


def test_equal_minima_keep_the_first():
    o = run(line([1.0, -1.0, 2.0]), prune_distance=3.0)
    assert o.needed[0] == 3                                                 # closest row 0, not row 1


def test_break_is_strictly_greater():
    # after the robot is reached an equal distance does not break, a later smaller one is taken, then > breaks
    o = run(line([0.1, -0.1, 0.05, 1.0, 0.0]))
    assert o.needed[0] == 3 and xs(o) == [1.0, 0.0]                         # closest row 2 (0.0025), row 4 never seen


# ---- 3. walk
def test_first_row_outside_the_window_is_still_taken():
    o = run(line([0, 1, 2, 3, 4, 5, 6]))
    assert o.goal_idx == 5 and xs(o)[-1] == 5                              # 16 <= 18.0625 takes x = 5 (25)


def test_squared_distance_equal_to_the_window():
    o = run(line([0, 1, 2, 3, 4.25, 5, 6]))
    assert 4.25 * 4.25 == 18.0625 and o.goal_idx == 5                       # <=: the row after 4.25 is taken
    o = run(line([0, 1, 2, 3, 4.26, 5, 6]))
    assert o.goal_idx == 4


def test_the_closest_rows_incoming_segment_counts_and_length_tie():
    rows = line([0, 1, 2, 3, 4, 5])
    o = run(rows, robot=(2.0, 0.0, 0.0), prune_distance=2.5, max_lookahead_dist=1.0)
    assert o.plan_begin == 0 and o.goal_idx == 3                            # row 2 adds 1 -> 1 <= 1 takes row 3 -> 2
    o = run(rows, robot=(2.0, 0.0, 0.0), prune_distance=2.5, max_lookahead_dist=0.9999)
    assert o.goal_idx == 2


@pytest.mark.parametrize("mx", [0.0, -1.0])
def test_non_positive_length_limit_is_off(mx):
    o = run(line([0, 1, 2, 3, 4, 5, 6]), max_lookahead_dist=mx)
    assert o.goal_idx == 5


def test_nan_length_limit_takes_no_row():
    o = run(line([0, 1, 2, 3]), max_lookahead_dist=NAN)
    assert o.goal_idx == 3 and o.plan == [(0.0, 0.0, 0.0), (3.0, 0.0, 0.0)]


def test_rows_beyond_1e10_inject_the_goal():
    o = run(line([2e5, 3e5, 4e5]), prune_distance=1.0)
    assert o.goal_idx == 2 and o.plan == [(0.0, 0.0, 0.0), (4e5, 0.0, 0.0)] and o.needed == (2, 0)


def test_rows_outside_the_window_inject_the_goal():
    o = run(line([10, 11, 12]), robot=(0.0, 0.0, 0.5))
    assert o.goal_idx == 2 and o.plan == [(0.0, 0.0, 0.5), (12.0, 0.0, 0.0)]


def test_window_uses_the_larger_side():
    o = run(line([0, 1, 2, 3, 4, 5, 6]), grid=(2, 40))
    assert o.goal_idx == 5
    o = run(line([0, 1, 2, 3, 4, 5, 6]), grid=(40, 2))
    assert o.goal_idx == 5
    o = run(line([0, 1, 2, 3, 4, 5, 6]), grid=(8, 8))                      # w = 0.85: rows 0, 1 (1 > 0.7225 stops)
    assert o.goal_idx == 1


# ---- 4. via-points
def test_via_point_tie_at_sep_is_taken():
    o = run(line([0, 0.5, 1.0, 1.5, 2.0]), viapoint_sep=0.5)
    assert o.via == [(0.5, 0.0), (1.0, 0.0), (1.5, 0.0), (2.0, 0.0)]
    o = run(line([0, 0.5, 1.0, 1.5, 2.0]), viapoint_sep=0.6)
    assert o.via == [(1.0, 0.0), (2.0, 0.0)] and o.needed == (5, 2)


@pytest.mark.parametrize("sep", [0.0, -1.0])
def test_non_positive_sep_gives_none(sep):
    assert run(line([0, 0.5, 1.0]), viapoint_sep=sep).via == []


def test_via_points_come_from_the_rows_before_the_start_row():
    o = run(line([0.1, 1.0, 2.0]), viapoint_sep=0.95)                   # row 0 is (0.1, 0), not the robot
    assert o.via == [(2.0, 0.0)]


def test_custom_via_points_are_not_written():
    o = run(line([0, 1, 2]), viapoint_sep=0.5, custom_via_count=4)
    assert o.via is None and o.needed == (3, 0)


def test_via_capacity():
    o = run(line([0, 1, 2, 3]), viapoint_sep=0.5, V_cap=2)
    assert o.result == lp.CAPACITY and o.needed == (4, 3) and o.plan == [] and o.via is None
    o = run(line([0, 1, 2, 3]), P_cap=3)
    assert o.result == lp.CAPACITY and o.needed == (4, 0)
    assert run(line([0, 1, 2, 3]), P_cap=4).result == lp.PLANNED


# ---- 5. goal reached (rows at yaw 0, where teb_plan_yaw is exact)
STOP = (0.0, 0.0, 0.0)


def goal(**kw):
    base = dict(robot=(0.0, 0.0, 0.0), vel=STOP, xy_goal_tolerance=0.25)
    base.update(kw)
    rows = base.pop("rows", [(-0.5, 0.0, 0.0), (0.25, 0.0, 0.0)])
    return run(rows, **base)


def test_goal_reached_writes_no_plan():
    o = goal(xy_goal_tolerance=0.2500001, viapoint_sep=0.5)
    assert o.result == lp.GOAL_REACHED and o.plan == [] and o.via == [] and o.needed == (0, 0)


def test_goal_xy_boundary():
    assert goal().result == lp.PLANNED                                      # 0.25 < 0.25 is false
    assert goal(xy_goal_tolerance=0.2500001).result == lp.GOAL_REACHED


def test_goal_yaw_boundary():
    assert lp.plan_yaw(0.0) == 0.0
    assert goal(xy_goal_tolerance=1, robot=(0.0, 0.0, -0.2)).result == lp.PLANNED
    assert goal(xy_goal_tolerance=1, robot=(0.0, 0.0, -0.19999)).result == lp.GOAL_REACHED
    assert goal(xy_goal_tolerance=1, robot=(0.0, 0.0, 2 * math.pi)).result == lp.GOAL_REACHED   # normalize_theta


def test_goal_needs_no_via_points_with_complete_global_plan():
    rows = [(-0.5, 0.0, 0.0), (0.0, 0.0, 0.0), (0.25, 0.0, 0.0)]
    assert goal(rows=rows, xy_goal_tolerance=1, viapoint_sep=0.1).result == lp.PLANNED
    o = goal(rows=rows, xy_goal_tolerance=1, viapoint_sep=0.1, complete_global_plan=False)
    assert o.result == lp.GOAL_REACHED and o.via == [(0.25, 0.0)]
    assert goal(xy_goal_tolerance=1, custom_via_count=1).result == lp.PLANNED
    assert goal(xy_goal_tolerance=1, custom_via_count=0).result == lp.GOAL_REACHED


@pytest.mark.parametrize("vel,stopped", [((0.1, 0.0, 0.0), True), ((0.1000001, 0.0, 0.0), False),
                                         ((0.0, -0.1, 0.0), True), ((0.0, -0.1000001, 0.0), False),
                                         ((0.0, 0.0, 0.1), True), ((0.0, 0.0, -0.1000001), False)])
def test_goal_needs_a_stopped_robot_or_a_free_goal_velocity(vel, stopped):
    assert goal(xy_goal_tolerance=1, vel=vel).result == (lp.GOAL_REACHED if stopped else lp.PLANNED)
    assert goal(xy_goal_tolerance=1, vel=vel, free_goal_vel=True).result == lp.GOAL_REACHED


# ---- 6. horizon shrink
def test_shrink_boundaries():
    S = lp.shrink_horizon
    assert S(10, 4, 1, math.inf, 10.0, True) == (7, 2)                    # reduction 2, one more row dropped
    assert S(30, 8, 9, math.inf, 10.0, True) == (25, 4)                   # count 9: 8 / 2
    assert S(30, 8, 10, math.inf, 10.0, True) == (27, 6)                  # count 10: halved again
    assert S(10, 4, 0, 10.0, 10.0, True) == (10, 4)                       # since == min_duration: no shrink
    assert S(10, 4, 0, 9.999, 10.0, True) == (7, 2)
    assert S(10, 4, 0, NAN, 10.0, True) == (10, 4)
    assert S(10, 4, 1, math.inf, 10.0, False) == (10, 4)
    assert S(10, 9, 1, math.inf, 10.0, True) == (10, 9)                   # the goal row already selected
    assert S(4, -3, 1, math.inf, 10.0, True) == (4, -3)                   # reduced goal_idx < 0: restored
    assert S(1, -4, 1, math.inf, 10.0, True) == (1, -4)                   # new index <= 0: restored


def test_shrink_does_not_fire_on_a_transformed_plan():
    # goal_idx counts from the pruned plan's first row, size from the closest row: goal_idx >= size - 1
    for rob in ((0.0, 0.0, 0.0), (3.0, 0.0, 0.0), (50.0, 0.0, 0.0)):
        a = run(line(range(12)), robot=rob, prune_distance=10.0, infeasible_count=5, since=0.0)
        b = run(line(range(12)), robot=rob, prune_distance=10.0)
        assert a == b


# ---- 7. goal heading
def test_heading_without_overwrite_is_the_stored_yaw():
    o = run([(0.0, 0.0, 0.3), (1.0, 0.0, 0.7)])
    assert o.plan[-1] == (1.0, 0.0, 0.7)


def test_heading_at_the_global_goal():
    o = run([(0.0, 0.0, 0.3), (1.0, 0.0, 0.7)], overwrite_orientation=True)
    assert o.goal_idx == 1 and o.plan[-1][2] == lp.plan_yaw(0.7)


def test_heading_near_the_global_goal_is_the_last_rows():
    rows = [(float(x), 0.0, 0.1 * x) for x in range(8)]
    for mx, gi in ((4.0, 5), (3.0, 4)):                                     # goal_idx n - 3, n - 4 (> n - 5)
        o = run(rows, max_lookahead_dist=mx, overwrite_orientation=True)
        assert o.goal_idx == gi and o.plan[-1] == (float(gi), 0.0, lp.plan_yaw(rows[-1][2]))


def test_heading_moving_average():
    rows = [(0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (2.0, 0.0, 0.0), (2.0, 1.0, 0.0), (3.0, 2.0, 0.0), (3.0, 4.0, 0.0),
            (9.0, 9.0, 0.0)]
    o = run(rows, max_lookahead_dist=1.0, overwrite_orientation=True)      # goal_idx 2 == n - 5
    c = [math.atan2(1.0, 0.0), math.atan2(1.0, 1.0), math.atan2(2.0, 0.0)]
    want = math.atan2(math.sin(c[0]) + math.sin(c[1]) + math.sin(c[2]), math.cos(c[0]) + math.cos(c[1]) + math.cos(c[2]))
    assert o.goal_idx == 2 and o.plan[-1] == (2.0, 0.0, want)
    assert lp.average_angles([]) == 0.0 and lp.average_angles([0.0, math.pi / 2]) == math.atan2(1.0, 1.0 + math.cos(math.pi / 2))


# ---- 8. start row
def test_one_row_plan_gets_the_robot_in_front():
    o = run([(0.5, 0.5, 0.25)], robot=(0.0, 0.1, -1.0))
    assert o.goal_idx == 0 and o.plan == [(0.0, 0.1, -1.0), (0.5, 0.5, 0.25)] and o.needed == (2, 0)


def test_row_0_becomes_the_robot():
    o = run(line([0.0, 1.0, 2.0]), robot=(0.01, 0.02, 3.0))
    assert o.plan == [(0.01, 0.02, 3.0), (1.0, 0.0, 0.0), (2.0, 0.0, 0.0)]


# ---- NaN
def test_nan_rows_are_never_closest_and_stop_the_walk():
    o = run([(0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (NAN, 0.0, 0.0), (3.0, 0.0, 0.0)])
    assert o.goal_idx == 2 and o.plan[-1][0] != o.plan[-1][0]               # the NaN row is taken, then NaN <= w fails
    o = run([(NAN, 0.0, 0.0), (NAN, 1.0, 0.0), (2.0, 0.0, 0.0), (3.0, 0.0, 0.0)], prune_distance=2.5)
    assert o.plan_begin == 2 and xs(o) == [3.0]


def test_nan_robot():
    o = run(line([0, 1, 2]), robot=(NAN, 0.0, 0.0), begin=1)
    assert o.plan_begin == 1 and o.goal_idx == 1 and o.result == lp.PLANNED      # no prune, injection (n = 2)
    assert math.isnan(o.plan[0][0]) and o.plan[1] == (2.0, 0.0, 0.0)


def test_sizeof_local_plan_args(teblib):
    assert teblib.tebgpu_sizeof(9) == C.sizeof(abi.TebLocalPlanArgs) == 6 * 4 + 8 * 8 + 16 * 8
