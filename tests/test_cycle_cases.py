"""The restated controller steps (tests/cycle_cases.py) on hand-computed cases at every boundary of the contract at
TebCycleArgs in include/teb_b200.h: each saturation branch in both modes, the trans cut, signed zeros and NaNs, the
steering angle's sign and minimum radius, the detector's capacity, half-full start, ring wrap and zero-crossing rule,
`recently` at exactly min_duration, the failure counter at INT32_MAX and each outcome's effect on the state."""
import math

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import cycle_cases as cc

LIM = dict(max_vel_x=0.4, max_vel_x_backwards=0.2, max_vel_y=0.0, max_vel_trans=0.4, max_vel_theta=0.3,
           min_turning_radius=0.0, divergence_detection_enable=0, divergence_detection_max_chi_squared=10.0)


def lim(**kw):
    return LIM | kw


def bits(x):
    return np.float64(x).tobytes()


# ---- saturateVelocity

def test_saturation_leaves_a_twist_inside_the_limits():
    assert cc.saturate(0.3, 0.0, -0.2, LIM) == (0.3, 0.0, -0.2)


@pytest.mark.parametrize("prop", [False, True])
def test_forward_and_rotation_limits(prop):
    vx, vy, w = cc.saturate(0.8, 0.0, 0.15, LIM, prop)
    assert vx == 0.4 and vy == 0.0
    assert w == (0.15 * 0.5 if prop else 0.15)
    vx, vy, w = cc.saturate(0.2, 0.0, -0.6, LIM, prop)
    assert w == -0.3 and vx == (0.2 * 0.5 if prop else 0.2)


@pytest.mark.parametrize("prop", [False, True])
def test_backwards_limit_replaces_ratio_x_only_when_positive(prop):
    assert cc.saturate(-0.4, 0.0, 0.0, LIM, prop)[0] == -0.2
    # max_vel_x_backwards <= 0: no backwards limit at all
    assert cc.saturate(-0.4, 0.0, 0.0, lim(max_vel_x_backwards=0.0), prop)[0] == -0.4
    assert cc.saturate(-0.3, 0.0, 0.0, lim(max_vel_x_backwards=-1.0), prop)[0] == -0.3


def test_max_vel_y_zero_zeroes_vy_and_with_proportional_saturation_the_twist():
    assert cc.saturate(0.2, 0.1, 0.1, LIM, False) == (0.2, 0.0, 0.1)
    assert cc.saturate(0.2, -0.1, 0.1, LIM, True) == (0.0, -0.0, 0.0)
    # vy == 0 and vy == -0.0 leave ratio_y at 1
    assert cc.saturate(0.2, -0.0, 0.1, LIM, True) == (0.2, -0.0, 0.1)


def test_holonomic_y_ratio_is_absolute():
    L = lim(max_vel_y=0.2, max_vel_trans=10.0)
    assert cc.saturate(0.1, -0.4, 0.0, L, False) == (0.1, -0.2, 0.0)
    assert cc.saturate(0.1, -0.4, 0.0, L, True) == (0.05, -0.2, 0.0)


def test_proportional_takes_the_smallest_ratio():
    L = lim(max_vel_y=0.2, max_vel_trans=10.0)
    # rx = 0.5, ry = 0.5, ro = 0.25
    vx, vy, w = cc.saturate(0.8, 0.4, 1.2, L, True)
    assert (vx, vy, w) == (0.8 * 0.25, 0.4 * 0.25, 1.2 * 0.25)


def test_trans_cut_at_exactly_max_vel_trans_and_above():
    L = lim(max_vel_x=10.0, max_vel_y=10.0, max_vel_trans=5.0, max_vel_theta=10.0)
    assert cc.saturate(3.0, 4.0, 0.0, L) == (3.0, 4.0, 0.0)          # hypot == 5 is not > 5
    vx, vy, _ = cc.saturate(6.0, 8.0, 0.0, L)                        # hypot 10: times 0.5
    assert (vx, vy) == (3.0, 4.0)


def test_max_vel_trans_zero_is_used_as_it_is():
    assert cc.saturate(0.3, 0.0, 0.2, lim(max_vel_trans=0.0)) == (0.0, 0.0, 0.2)


def test_make_cycle_args_replaces_max_vel_trans_zero_as_reconfigure_does():
    p = abi.default_params()
    assert p.max_vel_trans == 0.0
    abi.make_cycle_args(0.0, params=p)
    assert p.max_vel_trans == p.max_vel_x
    p.max_vel_trans = 0.7
    abi.make_cycle_args(0.0, params=p)
    assert p.max_vel_trans == 0.7


def test_negative_zero_and_nan_components():
    vx, vy, w = cc.saturate(-0.0, -0.0, -0.0, LIM)
    assert bits(vx) == bits(-0.0) and bits(w) == bits(-0.0)
    vx, vy, w = cc.saturate(math.nan, 0.0, 0.1, LIM)                  # NaN fails every test: passes through
    assert math.isnan(vx) and w == 0.1
    vx, vy, w = cc.saturate(0.1, 0.0, math.nan, LIM)
    assert vx == 0.1 and math.isnan(w)


# ---- convertTransRotVelToSteeringAngle

def test_steering_zero_cases():
    assert cc.steering(0.0, 0.5, 1.0, 0.5) == 0.0
    assert cc.steering(0.3, 0.0, 1.0, 0.5) == 0.0
    assert cc.steering(-0.0, 0.5, 1.0, 0.5) == 0.0


def test_steering_sign_and_minimum_radius():
    # radius 2 >= 0.95 * 1: atan(wheelbase / 2)
    assert cc.steering(0.4, 0.2, 1.0, 1.0) == math.atan(0.5)
    assert cc.steering(0.4, -0.2, 1.0, 1.0) == math.atan(-0.5)
    assert cc.steering(-0.4, -0.2, 1.0, 1.0) == math.atan(0.5)
    # radius 0.5 < 0.95: replaced by sign(radius) * 0.95
    m = 0.95 * 1.0
    assert cc.steering(0.1, 0.2, 1.0, 1.0) == math.atan(1.0 / m)
    assert cc.steering(0.1, -0.2, 1.0, 1.0) == math.atan(1.0 / -m)
    # negative wheelbase (back-wheeled robots) flips the angle
    assert cc.steering(0.1, 0.2, -1.0, 1.0) == math.atan(-1.0 / m)
    # radius exactly 0.95 * r is not replaced
    assert cc.steering(0.95, 1.0, 1.0, 1.0) == math.atan(1.0 / 0.95)


def test_steering_without_minimum_radius_and_non_finite():
    assert cc.steering(0.2, 0.4, 1.0, 0.0) == math.atan(1.0 / 0.5)
    assert math.isnan(cc.steering(math.nan, 0.4, 1.0, 1.0))
    # v tiny against omega: radius 0 is not < 0 with min_turning_radius 0: atan(1 / 0) = pi / 2
    assert cc.steering(5e-324, 1e300, 1.0, 0.0) == math.pi / 2


# ---- FailureDetector

def run(twists, cap, lims=(0.4, 0.2, 0.3, 0.1, 0.1)):
    return cc.detector_sequence(twists, cap, *lims)


def test_capacity_zero_never_oscillates_and_keeps_nothing():
    st = cc.band_state(0)
    assert not cc.detector_update(st, 0, 0.0, 0.1, 0.4, 0.2, 0.3, 0.1, 0.1)
    assert st["size"] == 0 and st["head"] == 0


def test_detection_starts_at_half_capacity_in_integer_division():
    rock = [(0.0, 0.01), (0.0, -0.01), (0.0, 0.01), (0.0, -0.01), (0.0, 0.01)]
    # capacity 5: starts at size 2 (5 // 2); crossings > 1 needs 3 entries
    assert run(rock, 5) == [False, False, True, True, True]
    # capacity 4: starts at 2; capacity 7: at 3; capacity 1: at 0 but one entry has no crossing
    assert run(rock, 4) == [False, False, True, True, True]
    assert run(rock, 7) == [False, False, True, True, True]
    assert run(rock, 1) == [False] * 5
    # capacity 8 starts at 4
    assert run(rock, 8) == [False, False, False, True, True]


def test_ring_wrap_drops_the_oldest_entry():
    cap = 3
    st = cc.band_state(cap)
    seq = [(0.1, 0.1), (0.2, 0.2), (0.3, 0.3), (0.4, 0.4)]
    for v, w in seq:
        cc.detector_update(st, cap, v, w, 1.0, 1.0, 1.0, 0.1, 0.1)
    assert st["size"] == 3 and st["head"] == 1
    assert st["ring"] == [(0.4, 0.4), (0.2, 0.2), (0.3, 0.3)]
    # means from the oldest entry on: a rock of three after the wrap oscillates, a stale entry no longer counts
    cap = 3
    seq = [(0.9, 0.9), (0.0, 0.01), (0.0, -0.01), (0.0, 0.01)]
    assert run(seq, cap, (1.0, 1.0, 1.0, 0.1, 0.1)) == [False, False, False, True]


def test_zero_crossings_use_g2o_sign_with_zero_and_nan():
    # 0.01, 0, -0.01: two sign changes (1 -> 0 -> -1)
    assert run([(0.0, 0.01), (0.0, 0.0), (0.0, -0.01)], 3)[-1]
    # NaN has sign 0 like 0, but poisons the mean: never oscillating
    assert not run([(0.0, 0.01), (0.0, math.nan), (0.0, -0.01)], 3)[-1]
    # -0.0 has sign 0: 0.01, -0.0, 0.01 are two crossings
    assert run([(0.0, 0.01), (0.0, -0.0), (0.0, 0.01)], 3)[-1]
    # one crossing is not enough
    assert not run([(0.0, 0.01), (0.0, 0.01), (0.0, -0.01)], 3)[-1]


def test_thresholds_are_strict_and_normalised():
    # v normalised by max_vel_x 0.5: 0.05 -> 0.1, mean not < 0.1
    lims = (0.5, 0.2, 0.3, 0.1, 0.1)
    assert not run([(0.05, 0.01), (0.05, -0.01), (0.05, 0.01)], 3, lims)[-1]
    assert run([(0.049, 0.01), (0.049, -0.01), (0.049, 0.01)], 3, lims)[-1]
    # backwards by max_vel_x_backwards 0.2
    lims = (0.4, 0.5, 0.3, 0.1, 0.1)
    assert not run([(-0.05, 0.01), (-0.05, -0.01), (-0.05, 0.01)], 3, lims)[-1]
    assert run([(-0.049, 0.01), (-0.049, -0.01), (-0.049, 0.01)], 3, lims)[-1]
    # omega normalised by omega_max 0.3: mean of (0.09, -0.03, 0.09) / 0.3 = 0.1666 -> not < 0.1
    assert not run([(0.0, 0.09), (0.0, -0.03), (0.0, 0.09)], 3)[-1]
    # omega_max <= 0: omega as it is
    assert run([(0.0, 0.09), (0.0, -0.09), (0.0, 0.09)], 3, (0.4, 0.2, 0.0, 0.1, 0.1))[-1]


def test_recovery_max_vel_theta():
    assert cc.recovery_max_vel_theta(0.1, LIM) == 0.3
    L = lim(min_turning_radius=-0.5)
    assert cc.recovery_max_vel_theta(0.1, L) == 0.4 / 0.5                # max(0.8, 0.3)
    assert cc.recovery_max_vel_theta(-0.1, L) == 0.2 / 0.5               # backwards: max(0.4, 0.3)
    assert cc.recovery_max_vel_theta(math.nan, L) == cc.cmax(0.2 / 0.5, 0.3)
    assert cc.recovery_max_vel_theta(-0.1, lim(min_turning_radius=0.5, max_vel_x_backwards=0.0)) == 0.3


# ---- backup modes

SC = cc.DEFAULT_SCALARS | dict(buffer_length=3)


def rocking_state(**kw):
    """a band whose ring holds two entries of a rock, so that the next rocking last_cmd makes it oscillate"""
    st = cc.band_state(3, last_cmd=(0.0, 0.0, 0.003), ring=[(0.0, 0.01), (0.0, -0.01), (0.0, 0.0)], size=2, head=0)
    st.update(kw)
    return st


@pytest.mark.parametrize("omega,rot", [(0.2, cc.ROT_LEFT), (0.0, cc.ROT_RIGHT), (-0.1, cc.ROT_RIGHT),
                                       (math.nan, cc.ROT_RIGHT), (-0.0, cc.ROT_RIGHT)])
def test_oscillation_sets_the_turning_direction_from_the_odometry(omega, rot):
    st = rocking_state()
    assert cc.backup_band(st, omega, 100.0, LIM, SC) == 1
    assert st["prefer_rotdir"] == rot and st["last_oscillation"] == 100.0


def test_recently_at_exactly_min_duration_is_not_recent():
    # now - last == 10 is not < 10: the direction is chosen again
    st = rocking_state(last_oscillation=90.0, prefer_rotdir=cc.ROT_RIGHT)
    assert cc.backup_band(st, 0.5, 100.0, LIM, SC) == 1
    assert st["prefer_rotdir"] == cc.ROT_LEFT and st["last_oscillation"] == 100.0
    # 9.5 s ago is recent: the direction is kept, the stamp moves
    st = rocking_state(last_oscillation=90.5, prefer_rotdir=cc.ROT_RIGHT)
    assert cc.backup_band(st, 0.5, 100.0, LIM, SC) == 1
    assert st["prefer_rotdir"] == cc.ROT_RIGHT and st["last_oscillation"] == 100.0


def test_direction_resets_only_when_not_oscillating_not_recent_and_set():
    calm = dict(last_cmd=(0.3, 0.0, 0.0))
    st = rocking_state(prefer_rotdir=cc.ROT_LEFT, last_oscillation=90.0, **calm)
    assert cc.backup_band(st, 0.0, 100.0, LIM, SC) == 0
    assert st["prefer_rotdir"] == cc.ROT_NONE and st["last_oscillation"] == 90.0
    st = rocking_state(prefer_rotdir=cc.ROT_LEFT, last_oscillation=90.5, **calm)
    assert cc.backup_band(st, 0.0, 100.0, LIM, SC) == 0
    assert st["prefer_rotdir"] == cc.ROT_LEFT


@pytest.mark.parametrize("result,runs", [(cc.PLANNED, True), (cc.CAPACITY, True), (cc.GOAL_REACHED, False),
                                         (cc.EMPTY, False), (cc.BAD_INPUT, False)])
def test_backup_runs_for_planned_and_capacity_only(result, runs):
    st = rocking_state()
    before = dict(st)
    o = cc.backup_band(st, 0.2, 100.0, LIM, SC, result)
    if runs:
        assert o == 1 and st["size"] == 3
    else:
        assert o is None and st == before


def test_backup_off_and_out_of_range_state():
    st = rocking_state()
    before = dict(st)
    assert cc.backup_band(st, 0.2, 100.0, LIM, SC | dict(oscillation_recovery=False)) == 0 and st == before
    for bad in (dict(size=4), dict(size=-1), dict(head=3), dict(head=-1), dict(prefer_rotdir=3)):
        st = rocking_state(**bad)
        before = dict(st)
        assert cc.backup_band(st, 0.2, 100.0, LIM, SC) == -1 and st == before
    assert cc.backup_band(rocking_state(), 0.2, 100.0, LIM, SC, 5) == -1
    st = cc.band_state(0, head=1)
    assert cc.backup_band(st, 0.2, 100.0, LIM, SC | dict(buffer_length=0)) == -1


# ---- finish cycle

def finish(st=None, n=12, status=1, chi2=1.0, cmd=(0.3, 0.0, 0.1, 1.0), now=50.0, L=LIM, sc=cc.DEFAULT_SCALARS,
           feasible=1, result=cc.PLANNED):
    st = cc.band_state(0, infeasible_count=3, last_infeasible=20.0, last_cmd=(0.1, 0.0, 0.1)) if st is None else st
    return st, cc.finish_band(st, n, status, chi2, cmd, now, L, sc, feasible, result)


def test_command_resets_the_counter_and_stores_last_cmd():
    st, (o, cv, n) = finish(cmd=(0.8, 0.0, 0.1, 1.0))
    assert o == cc.COMMAND and cv == (0.4, 0.0, 0.1) and n == 12
    assert st["infeasible_count"] == 0 and st["last_cmd"] == cv and st["last_infeasible"] == 20.0


def test_steering_angle_goes_into_cmd_vel_and_last_cmd():
    sc = cc.DEFAULT_SCALARS | dict(cmd_angle_instead_rotvel=True, wheelbase=0.5)
    st, (o, cv, n) = finish(cmd=(0.2, 0.0, 0.1, 1.0), sc=sc, L=lim(min_turning_radius=1.0))
    assert o == cc.COMMAND and cv == (0.2, 0.0, math.atan(0.5 / 2.0)) and st["last_cmd"] == cv


@pytest.mark.parametrize("kw,outcome", [
    (dict(status=0), cc.PLAN_FAILED), (dict(status=1 | 64), cc.PLAN_FAILED), (dict(status=1 | 128), cc.PLAN_FAILED),
    (dict(chi2=11.0, L=lim(divergence_detection_enable=1)), cc.DIVERGED),
    (dict(feasible=0), cc.INFEASIBLE), (dict(feasible=-1), cc.UNDECIDABLE),
    (dict(cmd=(0.3, 0.0, 0.1, 0.0)), cc.INVALID_COMMAND),
    (dict(cmd=(math.nan, 0.0, 0.1, 1.0), sc=cc.DEFAULT_SCALARS | dict(cmd_angle_instead_rotvel=True)),
     cc.STEERING_NOT_FINITE)])
def test_failures_zero_clear_count_and_stamp(kw, outcome):
    st, (o, cv, n) = finish(**kw)
    assert o == outcome and cv == (0.0, 0.0, 0.0) and n == 0
    assert st["infeasible_count"] == 4 and st["last_infeasible"] == 50.0 and st["last_cmd"] == (0.0, 0.0, 0.0)


def test_divergence_is_strict_and_off_by_default():
    assert finish(chi2=10.0, L=lim(divergence_detection_enable=1))[1][0] == cc.COMMAND
    assert finish(chi2=1e9)[1][0] == cc.COMMAND
    assert finish(chi2=math.nan, L=lim(divergence_detection_enable=1))[1][0] == cc.COMMAND


def test_order_of_the_checks():
    # plan failure before divergence before feasibility before the command
    assert finish(status=0, chi2=11.0, L=lim(divergence_detection_enable=1), feasible=0)[1][0] == cc.PLAN_FAILED
    assert finish(chi2=11.0, L=lim(divergence_detection_enable=1), feasible=0)[1][0] == cc.DIVERGED
    assert finish(feasible=0, cmd=(0, 0, 0, 0.0))[1][0] == cc.INFEASIBLE
    assert finish(feasible=None)[1][0] == cc.COMMAND


def test_counter_stops_at_int32_max():
    st = cc.band_state(0, infeasible_count=cc.INT32_MAX)
    _, (o, _, _) = finish(st=st, feasible=0)
    assert st["infeasible_count"] == cc.INT32_MAX
    st = cc.band_state(0, infeasible_count=cc.INT32_MAX - 1)
    finish(st=st, feasible=0)
    assert st["infeasible_count"] == cc.INT32_MAX


@pytest.mark.parametrize("result,outcome,n", [(cc.GOAL_REACHED, cc.CYCLE_GOAL_REACHED, 0), (cc.EMPTY, cc.NO_PLAN, 12),
                                              (cc.CAPACITY, cc.NO_PLAN, 12), (cc.BAD_INPUT, cc.NO_PLAN, 12)])
def test_goal_reached_and_no_plan_leave_counters_and_last_cmd(result, outcome, n):
    st, (o, cv, nn) = finish(result=result, feasible=0, status=0)
    assert o == outcome and cv == (0.0, 0.0, 0.0) and nn == n
    assert st["infeasible_count"] == 3 and st["last_infeasible"] == 20.0 and st["last_cmd"] == (0.1, 0.0, 0.1)


@pytest.mark.parametrize("kw", [dict(result=5), dict(result=-1), dict(feasible=2), dict(feasible=-2)])
def test_out_of_range_codes_give_no_plan(kw):
    st, (o, cv, n) = finish(**kw)
    assert o == cc.NO_PLAN and n == 12 and st["infeasible_count"] == 3


def test_fleet_form_matches_the_band_form():
    p = abi.default_params()
    p.max_vel_trans = p.max_vel_x
    B, L = 5, 4
    state = abi.make_cycle_state(B, L)
    state["last_cmd"][:] = [[0.0, 0.0, 0.003]] * B
    n = np.full(B, 10, np.int32)
    status = np.array([1, 0, 1, 1, 1], np.int32)
    cmd = np.array([[0.5, 0, 0.1, 1]] * B, float)
    feas = np.array([1, 1, 0, -1, 1], np.int32)
    out = cc.finish_cycle(state, n, status, np.zeros(B), cmd, 3.0, p, feasible=feas,
                          local_plan_result=np.array([0, 0, 0, 0, 1]))
    assert list(out["outcome"]) == [cc.COMMAND, cc.PLAN_FAILED, cc.INFEASIBLE, cc.UNDECIDABLE, cc.CYCLE_GOAL_REACHED]
    assert list(out["n"]) == [10, 0, 0, 0, 0]
    assert list(out["infeasible_count"]) == [0, 1, 1, 1, 0]
    assert out["cmd_vel"][0].tolist() == [0.4, 0.0, 0.1]
    bk = cc.backup_modes(out, np.zeros((B, 3)), 3.0, p)
    assert list(bk["osc_fill"][:, 0]) == [1] * B and list(bk["oscillating"]) == [0] * B
