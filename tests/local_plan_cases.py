"""The step that turns a robot's global plan into its local plan, goal and via-points, restated in plain Python.

`restate` follows TebLocalPlannerROS::computeVelocityCommands from pruneGlobalPlan up to the start row
(teb_local_planner_ros.cpp:268-340), with pruneGlobalPlan (:657-698), transformGlobalPlan (:701-822) under the identity
transform, updateViaPointsContainer (:627-646), the goal-reached test (:290-304), configureBackupModes' horizon shrink
(:950-977) and estimateLocalGoalOrientation (:827-871, average_angles misc.h:72-84), step by step as include/teb_b200.h
defines it at TebLocalPlanArgs. TebLocalPlannerROS is not compiled into oracle/_ref: its headers pull in the navigation
stack. So this restatement is the reference for the device's rows. It uses Python floats: math's trig is glibc's, as in
the reference's x86 build, and Python does not contract a * b + c into an FMA, so every product and sum is rounded on its
own as there.
"""
import math
from dataclasses import dataclass, field

PLANNED, GOAL_REACHED, EMPTY, CAPACITY, BAD_INPUT = 0, 1, 2, 3, 4   # TEB_LOCAL_PLAN_*
MOVING_AVERAGE_LENGTH = 3                                           # estimateLocalGoalOrientation's default argument


def normalize_theta(t):
    """g2o::normalize_theta, as teb_normalize_theta evaluates it"""
    if -math.pi <= t < math.pi:
        return t
    m = math.floor(t / (2 * math.pi))
    t = t + -(m * 2.0 * math.pi)
    if t >= math.pi:
        t -= 2 * math.pi
    if t < -math.pi:
        t += 2 * math.pi
    return t


def plan_yaw(yaw):
    """tf::createQuaternionFromYaw followed by tf::getYaw (teb_plan_yaw)"""
    qz, qw = math.sin(yaw / 2), math.cos(yaw / 2)
    return math.atan2(2.0 * (qw * qz + 0.0 * 0.0), 1.0 - 2.0 * (0.0 * 0.0 + qz * qz))


def sq_dist(ax, ay, bx, by):
    dx, dy = ax - bx, ay - by
    return dx * dx + dy * dy


def distance_points2d(p1, p2):
    dx, dy = p2[0] - p1[0], p2[1] - p1[1]
    return math.sqrt(dx * dx + dy * dy)


def _cdiv(a, b):
    """C's int division, truncating towards zero"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def shrink_horizon(size, goal_idx, count, since, min_duration, enabled):
    """configureBackupModes' reduced horizon (:950-977): (new size of the transformed plan, new goal_idx)"""
    if enabled and goal_idx < size - 1 and (count > 0 or since < min_duration):
        reduction = _cdiv(goal_idx, 2)
        if count > 9:
            reduction = _cdiv(reduction, 2)
        new_size = size - reduction - 1
        goal_idx -= reduction
        if new_size > 0 and goal_idx >= 0:
            size = new_size
        else:
            goal_idx += reduction
    return size, goal_idx


def average_angles(angles):
    x = y = 0.0
    for a in angles:
        x += math.cos(a)
        y += math.sin(a)
    return 0.0 if x == 0 and y == 0 else math.atan2(y, x)


def goal_heading(g, n, goal_idx, local_goal, overwrite, mal=MOVING_AVERAGE_LENGTH):
    """the yaw stored in the local goal row: estimateLocalGoalOrientation, or the row's own yaw"""
    if not overwrite:
        return local_goal[2]
    if goal_idx > n - mal - 2:
        if goal_idx >= n - 1:
            return plan_yaw(local_goal[2])
        return plan_yaw(g[n - 1][2])                    # the identity rotation times the last row's quaternion
    mal = min(mal, n - goal_idx - 1)
    cands = []
    k = local_goal
    for i in range(goal_idx, goal_idx + mal):
        kp1 = g[i + 1]
        cands.append(math.atan2(kp1[1] - k[1], kp1[0] - k[0]))
        k = kp1
    return average_angles(cands)


@dataclass
class Args:
    """the scalars of TebLocalPlanArgs, the reference's defaults (teb_config.h:259-298, :381-382)"""
    prune_distance: float = 1.0
    max_lookahead_dist: float = 1.0
    viapoint_sep: float = -1.0
    xy_goal_tolerance: float = 0.2
    yaw_goal_tolerance: float = 0.2
    trans_stopped_vel: float = 0.1
    theta_stopped_vel: float = 0.1
    shrink_horizon_min_duration: float = 10.0
    free_goal_vel: bool = False
    complete_global_plan: bool = True
    shrink_horizon_backup: bool = True
    overwrite_orientation: bool = True           # TebParams.global_plan_overwrite_orientation


@dataclass
class Out:
    result: int
    plan_begin: int
    goal_idx: int = None                         # None: not written
    plan: list = field(default_factory=list)     # rows (x, y, yaw); [] with plan_count 0
    via: list = None                             # None: not written
    needed: tuple = None


def restate(rows, begin, end, robot, vel, grid, res, a, custom_via_count=None, infeasible_count=None, since=None,
            P_cap=1 << 30, V_cap=1 << 30):
    """One band. rows: the global plan (x, y, yaw) indexable up to `end`; begin / end: its live rows; robot (x, y, yaw);
    vel (vx, vy, omega); grid (sx, sy) and res of its costmap; a: Args. custom_via_count: None to extract via-points from
    the plan (TebLocalPlanArgs.via != NULL), else the caller's via-point count. infeasible_count / since: None for NULL."""
    rx, ry, rt = (float(v) for v in robot)
    # 1. prune
    d2 = a.prune_distance * a.prune_distance
    for k in range(begin, end):
        if sq_dist(rx, ry, rows[k][0], rows[k][1]) < d2:
            begin = k
            break
    g = [tuple(float(v) for v in rows[k]) for k in range(begin, end)]
    n = len(g)
    # 2. no live rows
    if n == 0:
        return Out(EMPTY, begin)
    # 3. transform
    sx, sy = grid
    ax, ay = float(sx) * res / 2.0, float(sy) * res / 2.0
    thr = (ay if ax < ay else ax) * 0.85                 # std::max(a, b) is (a < b) ? b : a
    thr = thr * thr
    i, sq, reached = 0, 1e10, False
    for j in range(n):
        new = sq_dist(rx, ry, g[j][0], g[j][1])
        if reached and new > sq:
            break
        if new < sq:
            sq, i = new, j
            if sq < 0.05:
                reached = True
    first, length, mx = i, 0.0, a.max_lookahead_dist
    while i < n and sq <= thr and (mx <= 0 or length <= mx):
        sq = sq_dist(rx, ry, g[i][0], g[i][1])
        if i > 0 and mx > 0:
            length += distance_points2d(g[i - 1], g[i])
        i += 1
    if i == first:
        first, size, goal_idx = n - 1, 1, n - 1          # the global goal injected
    else:
        size, goal_idx = i - first, i - 1
    t = g[first:first + size]
    # 4. via-points
    via = None
    if custom_via_count is None:
        via = []
        if not a.viapoint_sep <= 0:                       # a NaN separation extracts every row
            prev = 0
            for k in range(1, size):
                if distance_points2d(t[prev], t[k]) < a.viapoint_sep:
                    continue
                via.append((t[k][0], t[k][1]))
                prev = k
    vcount = len(via) if via is not None else int(custom_via_count)
    # 5. goal reached
    gx, gy, gyaw = g[n - 1]
    dx, dy = gx - rx, gy - ry
    vx, vy, om = (float(v) for v in vel)
    stopped = abs(om) <= a.theta_stopped_vel and abs(vx) <= a.trans_stopped_vel and abs(vy) <= a.trans_stopped_vel
    if (abs(math.sqrt(dx * dx + dy * dy)) < a.xy_goal_tolerance
            and abs(normalize_theta(plan_yaw(gyaw) - rt)) < a.yaw_goal_tolerance
            and (not a.complete_global_plan or vcount == 0) and (stopped or a.free_goal_vel)):
        if via is not None and len(via) > V_cap:
            return Out(CAPACITY, begin, goal_idx, needed=(0, len(via)))
        return Out(GOAL_REACHED, begin, goal_idx, via=via, needed=(0, vcount if via is not None else 0))
    # 6. horizon shrink
    enabled = a.shrink_horizon_backup and not (infeasible_count is None and since is None)
    size, goal_idx = shrink_horizon(size, goal_idx, 0 if infeasible_count is None else int(infeasible_count),
                                    math.inf if since is None else float(since), a.shrink_horizon_min_duration, enabled)
    t = t[:size]
    # 7. goal heading
    lg = t[-1]
    heading = goal_heading(g, n, goal_idx, lg, a.overwrite_orientation)
    # 8. start row
    out = [(rx, ry, rt)] + [tuple(r) for r in t[1:-1]] + [(lg[0], lg[1], heading)]
    needed = (len(out), len(via) if via is not None else 0)
    # 9. capacity
    if len(out) > P_cap or (via is not None and len(via) > V_cap):
        return Out(CAPACITY, begin, goal_idx, needed=needed)
    return Out(PLANNED, begin, goal_idx, out, via, needed)
