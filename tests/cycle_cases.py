"""The controller steps around plan(), restated in plain Python.

`backup_band` follows the oscillation half of TebLocalPlannerROS::configureBackupModes (teb_local_planner_ros.cpp:980-1016)
with FailureDetector::update / detect (recovery_behaviors.cpp); `finish_band` follows computeVelocityCommands from plan()
on (:360-454) with saturateVelocity (:874-919) and convertTransRotVelToSteeringAngle (:922-933), step by step as
include/teb_b200.h defines them at TebCycleArgs. TebLocalPlannerROS is not compiled into oracle/_ref: its headers pull in
the navigation stack. So this restatement is the reference for the device; its detector is held to the reference's own
FailureDetector by tests/test_reference_pin_recovery.py. Python floats are IEEE doubles and Python never contracts
a * b + c into an FMA, so every product and sum is rounded on its own, as in the reference's x86 build. math.atan is
glibc's; math.hypot is correctly rounded, as glibc's is.

A band's state is a dict of Python values (see `band_state`); `backup_modes` / `finish_cycle` run a step over the numpy
arrays of abi.make_cycle_state and return new arrays.
"""
import math

import numpy as np

# TEB_LOCAL_PLAN_*
PLANNED, GOAL_REACHED, EMPTY, CAPACITY, BAD_INPUT = 0, 1, 2, 3, 4
# TEB_CYCLE_*
COMMAND, CYCLE_GOAL_REACHED, NO_PLAN, PLAN_FAILED, DIVERGED, INFEASIBLE, UNDECIDABLE, INVALID_COMMAND, \
    STEERING_NOT_FINITE = range(9)
ROT_NONE, ROT_LEFT, ROT_RIGHT = 0, 1, 2
STATUS_OPTIMIZED, STATUS_CAPACITY, STATUS_BAD_INPUT = 1, 64, 128
INT32_MAX = 2 ** 31 - 1


def sign(x):
    """g2o::sign: 0 for 0 and NaN"""
    return 1 if x > 0 else (-1 if x < 0 else 0)


def div(a, b):
    """a / b in IEEE arithmetic: +-inf or NaN where Python raises"""
    try:
        return a / b
    except ZeroDivisionError:
        return math.nan if a == 0 or a != a else math.copysign(math.inf, a) * math.copysign(1.0, b)


def cmin(a, b):
    """std::min"""
    return b if b < a else a


def cmax(a, b):
    """std::max"""
    return b if a < b else a


def saturate(vx, vy, omega, lim, proportional=False):
    """saturateVelocity. lim: dict with max_vel_x, max_vel_x_backwards, max_vel_y, max_vel_trans, max_vel_theta"""
    rx = ry = ro = 1.0
    if vx > lim["max_vel_x"]:
        rx = div(lim["max_vel_x"], vx)
    if vy > lim["max_vel_y"] or vy < -lim["max_vel_y"]:
        ry = abs(div(lim["max_vel_y"], vy))
    if omega > lim["max_vel_theta"] or omega < -lim["max_vel_theta"]:
        ro = abs(div(lim["max_vel_theta"], omega))
    if lim["max_vel_x_backwards"] <= 0:
        pass
    elif vx < -lim["max_vel_x_backwards"]:
        rx = div(-lim["max_vel_x_backwards"], vx)
    if proportional:
        r = cmin(cmin(rx, ry), ro)
        vx, vy, omega = vx * r, vy * r, omega * r
    else:
        vx, vy, omega = vx * rx, vy * ry, omega * ro
    vel_linear = math.hypot(vx, vy)
    if vel_linear > lim["max_vel_trans"]:
        r = div(lim["max_vel_trans"], vel_linear)
        vx, vy = vx * r, vy * r
    return vx, vy, omega


def steering(v, omega, wheelbase, min_turning_radius):
    """convertTransRotVelToSteeringAngle(v, omega, wheelbase, 0.95 * min_turning_radius)"""
    if omega == 0 or v == 0:
        return 0.0
    m = 0.95 * min_turning_radius
    radius = div(v, omega)
    if abs(radius) < m:
        radius = float(sign(radius)) * m
    return math.atan(div(wheelbase, radius))


def recovery_max_vel_theta(last_vx, lim):
    """configureBackupModes' max_vel_theta for the detector"""
    mvc = lim["max_vel_x"] if last_vx >= 0 else lim["max_vel_x_backwards"]
    if lim["min_turning_radius"] != 0 and mvc > 0:
        return cmax(div(mvc, abs(lim["min_turning_radius"])), lim["max_vel_theta"])
    return lim["max_vel_theta"]


def detector_update(st, cap, v, omega, v_max, v_backwards_max, omega_max, v_eps, omega_eps):
    """FailureDetector::update then isOscillating(), on st['ring'] (cap slots of (v, omega)), st['size'], st['head']"""
    if cap == 0:
        return False
    if v > 0 and v_max > 0:
        v = v / v_max
    elif v < 0 and v_backwards_max > 0:
        v = v / v_backwards_max
    if omega_max > 0:
        omega = omega / omega_max     # the divisors are > 0 here
    size, head = st["size"], st["head"]
    if size < cap:
        slot = (head + size) % cap
        size += 1
    else:
        slot, head = head, (head + 1) % cap
    st["ring"][slot] = (v, omega)
    st["size"], st["head"] = size, head
    if size < cap // 2:
        return False
    entries = [st["ring"][(head + k) % cap] for k in range(size)]
    v_mean = omega_mean = 0.0
    crossings = 0
    for i, (ev, eo) in enumerate(entries):
        v_mean += ev
        omega_mean += eo
        if i > 0 and sign(eo) != sign(entries[i - 1][1]):
            crossings += 1
    v_mean /= size
    omega_mean /= size
    return abs(v_mean) < v_eps and abs(omega_mean) < omega_eps and crossings > 1


def detector_sequence(twists, cap, v_max, v_backwards_max, omega_max, v_eps, omega_eps):
    """isOscillating() after each FailureDetector::update of the (v, omega) sequence, from an empty ring"""
    st = dict(ring=[(0.0, 0.0)] * max(cap, 1), size=0, head=0)
    return [detector_update(st, cap, v, w, v_max, v_backwards_max, omega_max, v_eps, omega_eps) for v, w in twists]


DEFAULT_SCALARS = dict(use_proportional_saturation=False, cmd_angle_instead_rotvel=False, wheelbase=1.0,
                       oscillation_recovery=True, oscillation_v_eps=0.1, oscillation_omega_eps=0.1,
                       oscillation_recovery_min_duration=10.0, buffer_length=50)


def limits(params):
    """the TebParams fields the two steps read"""
    return {k: float(getattr(params, k)) for k in ("max_vel_x", "max_vel_x_backwards", "max_vel_y", "max_vel_trans",
                                                    "max_vel_theta", "min_turning_radius",
                                                    "divergence_detection_max_chi_squared")} | \
        dict(divergence_detection_enable=int(params.divergence_detection_enable))


def band_state(cap=0, **kw):
    """one band's controller state before its first cycle (the node's constructor), with overrides"""
    st = dict(infeasible_count=0, last_infeasible=-math.inf, last_oscillation=-math.inf, last_cmd=(0.0, 0.0, 0.0),
              prefer_rotdir=ROT_NONE, ring=[(0.0, 0.0)] * max(cap, 1), size=0, head=0)
    st.update(kw)
    return st


def backup_valid(st, result, cap):
    if not PLANNED <= result <= BAD_INPUT:
        return False
    if result not in (PLANNED, CAPACITY):
        return True
    if not ROT_NONE <= st["prefer_rotdir"] <= ROT_RIGHT:
        return False
    return 0 <= st["size"] <= cap and st["head"] >= 0 and (st["head"] == 0 if cap == 0 else st["head"] < cap)


def backup_band(st, robot_omega, now, lim, sc, result=PLANNED):
    """the oscillation half of configureBackupModes on band state `st` (changed in place). Returns oscillating: 1 / 0,
    -1 for an out-of-range state (nothing changed), None for a band the step skips (nothing changed)"""
    cap = sc["buffer_length"]
    if not backup_valid(st, result, cap):
        return -1
    if result not in (PLANNED, CAPACITY):
        return None
    if not sc["oscillation_recovery"]:
        return 0
    lvx, lom = st["last_cmd"][0], st["last_cmd"][2]
    osc = detector_update(st, cap, lvx, lom, lim["max_vel_x"], lim["max_vel_x_backwards"],
                          recovery_max_vel_theta(lvx, lim), sc["oscillation_v_eps"], sc["oscillation_omega_eps"])
    recently = now - st["last_oscillation"] < sc["oscillation_recovery_min_duration"]
    if osc:
        if not recently:
            st["prefer_rotdir"] = ROT_LEFT if robot_omega > 0 else ROT_RIGHT
        st["last_oscillation"] = now
    elif not recently and st["prefer_rotdir"] != ROT_NONE:
        st["prefer_rotdir"] = ROT_NONE
    return 1 if osc else 0


def finish_band(st, n, status, chi2, cmd, now, lim, sc, feasible=None, result=PLANNED):
    """computeVelocityCommands from plan() on for band state `st` (changed in place). cmd: (vx, vy, omega, ok);
    feasible: 1 / 0 / -1 or None (not checked). Returns (outcome, cmd_vel, n)"""
    zero = (0.0, 0.0, 0.0)
    if not PLANNED <= result <= BAD_INPUT or (feasible is not None and not -1 <= feasible <= 1):
        return NO_PLAN, zero, n
    if result == GOAL_REACHED:
        return CYCLE_GOAL_REACHED, zero, 0
    if result in (EMPTY, CAPACITY, BAD_INPUT):
        return NO_PLAN, zero, n
    if not status & STATUS_OPTIMIZED or status & (STATUS_CAPACITY | STATUS_BAD_INPUT):
        outcome = PLAN_FAILED
    elif lim["divergence_detection_enable"] and chi2 > lim["divergence_detection_max_chi_squared"]:
        outcome = DIVERGED
    elif feasible == 0:
        outcome = INFEASIBLE
    elif feasible == -1:
        outcome = UNDECIDABLE
    elif cmd[3] == 0:
        outcome = INVALID_COMMAND
    else:
        outcome = COMMAND
        vx, vy, om = saturate(cmd[0], cmd[1], cmd[2], lim, sc["use_proportional_saturation"])
        if sc["cmd_angle_instead_rotvel"]:
            om = steering(vx, om, sc["wheelbase"], lim["min_turning_radius"])
            if not math.isfinite(om):
                outcome = STEERING_NOT_FINITE
    if outcome == COMMAND:
        st["infeasible_count"] = 0
        st["last_cmd"] = (vx, vy, om)
        return COMMAND, (vx, vy, om), n
    if st["infeasible_count"] < INT32_MAX:
        st["infeasible_count"] += 1
    st["last_infeasible"] = now
    st["last_cmd"] = zero
    return outcome, zero, 0


# ---- fleet form, over the arrays of abi.make_cycle_state

def _band(state, b):
    cap = state["osc_ring"].shape[0]
    return dict(infeasible_count=int(state["infeasible_count"][b]), last_infeasible=float(state["last_infeasible"][b]),
                last_oscillation=float(state["last_oscillation"][b]),
                last_cmd=tuple(float(x) for x in state["last_cmd"][b]), prefer_rotdir=int(state["prefer_rotdir"][b]),
                ring=[(float(state["osc_ring"][k, b, 0]), float(state["osc_ring"][k, b, 1])) for k in range(cap)],
                size=int(state["osc_fill"][b, 0]), head=int(state["osc_fill"][b, 1]))


def _store(out, b, st):
    out["infeasible_count"][b] = st["infeasible_count"]
    out["last_infeasible"][b] = st["last_infeasible"]
    out["last_oscillation"][b] = st["last_oscillation"]
    out["last_cmd"][b] = st["last_cmd"]
    out["prefer_rotdir"][b] = st["prefer_rotdir"]
    for k in range(out["osc_ring"].shape[0]):
        out["osc_ring"][k, b] = st["ring"][k]
    out["osc_fill"][b] = (st["size"], st["head"])


def copy_state(state):
    return {k: np.array(v, copy=True) for k, v in state.items()}


def backup_modes(state, robot_vel, now, params, local_plan_result=None, **scalars):
    """backup_band for every band: returns a new state dict plus oscillating [B] (-2 where the step writes nothing)"""
    sc = DEFAULT_SCALARS | dict(buffer_length=state["osc_ring"].shape[0]) | scalars
    lim = limits(params)
    out = copy_state(state)
    B = len(state["prefer_rotdir"])
    osc = np.full(B, -2, np.int32)
    for b in range(B):
        r = PLANNED if local_plan_result is None else int(local_plan_result[b])
        st = _band(state, b)
        o = backup_band(st, float(robot_vel[b][2]), float(now), lim, sc, r)
        if o is not None:
            osc[b] = o
        if o not in (None, -1):
            _store(out, b, st)
    out["oscillating"] = osc
    return out


def finish_cycle(state, n, status, chi2, cmd, now, params, feasible=None, local_plan_result=None, **scalars):
    """finish_band for every band: returns a new state dict plus n, cmd_vel [B][3] and outcome [B]"""
    sc = DEFAULT_SCALARS | dict(buffer_length=state["osc_ring"].shape[0]) | scalars
    lim = limits(params)
    out = copy_state(state)
    B = len(state["prefer_rotdir"])
    n_out, cmd_vel, outcome = np.array(n, np.int32, copy=True), np.zeros((B, 3)), np.zeros(B, np.int32)
    for b in range(B):
        r = PLANNED if local_plan_result is None else int(local_plan_result[b])
        st = _band(state, b)
        o, cv, nb = finish_band(st, int(n[b]), int(status[b]), float(chi2[b]), tuple(float(x) for x in cmd[b]),
                                float(now), lim, sc, None if feasible is None else int(feasible[b]), r)
        outcome[b], cmd_vel[b], n_out[b] = o, cv, nb
        _store(out, b, st)
    out.update(n=n_out, cmd_vel=cmd_vel, outcome=outcome)
    return out
