"""CPU restatement of the shaped fleet steps under TEB_FLEET_SELECT_FOOTPRINTS (include/teb_b200.h, TebFleetShapes):
candidate q of robot r passes the centres' prefilter d2 <= R'^2 (R' = (range + E_r + E_lib)(1 + 2^-16)), then its gap,
the least optimizer distance (oracle_binding.distance, teb_oracle_distance at t = 0) from r's footprint at r's pose to
q's parts placed as the shaped writer places them; q is a neighbour when gap <= range, the list is ordered by (gap, q)
and written by fleet_shape_cases' writer.

The prefilter and the order are exact here as on the device. The gap rests on sin / cos (the C library's here, the
device's there) and on the distance code's rounding (the oracle's, compiled without FMA contraction, against the
device's), so decisions within rounding of range, or of a tie of two gaps, may go either way; `near` reports them."""
import math

import numpy as np

from teb_local_planner_b200 import abi
from tests import fleet_cases as fc
from tests import fleet_shape_cases as fsc
from tests import oracle_binding as ob

MARGIN = 1.0 + 2.0 ** -16


def footprint_reach(params):
    """E_r: the largest distance from the robot's position of a point of its footprint model"""
    t = params.footprint_type
    if t == abi.TEB_FOOTPRINT_CIRCULAR:
        return abs(params.footprint_radius)
    if t == abi.TEB_FOOTPRINT_TWO_CIRCLES:
        return max(abs(params.footprint_front_offset) + abs(params.footprint_front_radius),
                   abs(params.footprint_rear_offset) + abs(params.footprint_rear_radius))
    if t == abi.TEB_FOOTPRINT_LINE:
        ln = list(params.footprint_line)
        return max(math.sqrt(ln[0] * ln[0] + ln[1] * ln[1]), math.sqrt(ln[2] * ln[2] + ln[3] * ln[3]))
    if t == abi.TEB_FOOTPRINT_POLYGON:
        v = list(params.footprint_vertices)
        return max(math.sqrt(v[2 * i] * v[2 * i] + v[2 * i + 1] * v[2 * i + 1])
                   for i in range(params.footprint_vertex_count))
    return 0.0


def library_reach(kinds):
    """E_lib: the largest |u| + radius of a part point u of the library"""
    e = 0.0
    for parts in kinds:
        for p in parts:
            rad = float(p[2]) if p[0] == fsc.CIRCULAR else 0.0
            for u in np.asarray(p[1], np.float64).reshape(-1, 2):
                e = max(e, math.sqrt(u[0] * u[0] + u[1] * u[1]) + rad)
    return e


def prefilter(params, kinds, rng):
    """R' of a step of range rng"""
    return (rng + footprint_reach(params) + library_reach(kinds)) * MARGIN


def gap(params, pose_r, x, y, th, parts):
    """the least distance from the footprint of params at pose_r to the parts placed at (x, y, th)"""
    nv = fsc.kind_size(parts)[1]
    out = np.zeros((1, len(parts)), abi.OBST_DTYPE)
    cv = np.zeros((1, max(nv, 1), 2))
    fsc.write_kind(out, cv, 0, 0, 0, parts, x, y, th, 0.0, 0.0, 0)
    ds = [ob.distance(params, np.asarray(pose_r, np.float64), o, cv[0] if o["type"] in (fsc.LINE, fsc.POLYGON) else None)
          for o in out[0]]
    return min(ds)


def neighbours(params, kinds, xy, th, world, live, kind, me, pose_me, rng):
    """(candidates, gaps) of robot `me` at pose_me in (gap, q) order, and the (q, gap) pairs that passed the prefilter"""
    pre = prefilter(params, kinds, rng)
    dx = xy[:, 0] - xy[me, 0]
    dy = xy[:, 1] - xy[me, 1]
    d2 = dx * dx + dy * dy
    ok = (d2 <= pre * pre) & live & (world == world[me])
    ok[me] = False
    keys = []
    for q in np.nonzero(ok)[0]:
        k = int(kind[q])
        g = -math.inf if not 0 <= k < len(kinds) else gap(params, pose_me, xy[q, 0], xy[q, 1], th[q], kinds[k])
        if g <= rng:
            keys.append((g, int(q)))
    keys.sort()
    return np.array([q for _, q in keys], np.int64), np.array([g for g, _ in keys])


def restate(params, pose, last_cmd, kinds, kind, rng, max_rows, custom, custom_vertices=None, own_count=None,
            custom_count=None, own_vertex_count=None, world=None, scene=None, PV_cap=None, gaps=None):
    """tebgpu_fleet_obstacles_shaped_device with select = TEB_FLEET_SELECT_FOOTPRINTS on the host, params the context's
    TebParams. Returns (custom, custom_count, needed, status, custom_vertices); gaps (a dict or None) gets each robot's
    (list, gaps)."""
    pose = np.asarray(pose, np.float64).reshape(-1, 3)
    R = len(pose)
    cmd = np.asarray(last_cmd, np.float64).reshape(R, 3)
    kind = np.broadcast_to(np.asarray(kind, np.int64), (R,))
    wld = np.zeros(R, np.int64) if world is None else np.asarray(world, np.int64)
    S, C_cap = np.asarray(custom).shape
    PV = (0 if custom_vertices is None else np.asarray(custom_vertices).shape[1]) if PV_cap is None else PV_cap

    def listing(r):
        idx, g = neighbours(params, kinds, pose[:, :2], pose[:, 2], wld, np.ones(R, bool), kind, r, pose[r], rng)
        if gaps is not None:
            gaps[r] = (idx, g)
        return True, max_rows, idx

    def neighbour(q):
        o = fc.row(pose[q], cmd[q], 0.0)
        return pose[q, 0], pose[q, 1], pose[q, 2], o["vx"], o["vy"], int(o["dynamic"]), int(kind[q])

    return fsc._shaped(S, R, C_cap, PV, custom, custom_vertices, own_count, custom_count, own_vertex_count, scene,
                       listing, neighbour, kinds)


def restate_table(params, rows, heading, row_kind, kinds, first, R, rng, max_rows, custom, custom_vertices=None,
                  own_count=None, custom_count=None, own_vertex_count=None, scene=None, PV_cap=None, gaps=None):
    """tebgpu_fleet_obstacles_table_shaped_device with select = TEB_FLEET_SELECT_FOOTPRINTS on the host for robots
    first .. first + R - 1 of the table: robot r's footprint at its row's position and heading[first + r]"""
    S, C_cap = np.asarray(custom).shape
    PV = (0 if custom_vertices is None else np.asarray(custom_vertices).shape[1]) if PV_cap is None else PV_cap
    xy = np.stack([rows["x"], rows["y"]], 1)
    heading = np.asarray(heading, np.float64)

    def listing(r):
        me = first + r
        if not rows["live"][me]:
            return False, 0, None
        idx, g = neighbours(params, kinds, xy, heading, rows["world"], rows["live"] != 0, row_kind, me,
                            [xy[me, 0], xy[me, 1], heading[me]], rng)
        if gaps is not None:
            gaps[r] = (idx, g)
        return True, max_rows, idx

    def neighbour(q):
        w = rows[q]
        return w["x"], w["y"], heading[q], w["vx"], w["vy"], int(w["dynamic"]), int(row_kind[q])

    return fsc._shaped(S, R, C_cap, PV, custom, custom_vertices, own_count, custom_count, own_vertex_count, scene,
                       listing, neighbour, kinds)


def sharded(params, pose, last_cmd, kinds, kind, rng, max_rows, custom, custom_vertices, counts, own_count=None,
            own_vertex_count=None, world=None):
    """fleet_shape_cases.sharded under the footprints' rule: publish per shard, then the table step per shard"""
    from tests import fleet_table_cases as ftc
    pose = np.asarray(pose, np.float64).reshape(-1, 3)
    R = len(pose)
    kind = np.broadcast_to(np.asarray(kind, np.int32), (R,))
    world = None if world is None else np.asarray(world, np.int32)
    parts = ftc.split(R, counts)
    cap = max(1, max(counts))
    pubs = [fsc.publish(pose[lo:hi], np.asarray(last_cmd)[lo:hi], 0.0, kind[lo:hi],
                        None if world is None else world[lo:hi]) for lo, hi in parts]
    tab = ftc.table([p[0] for p in pubs], cap)
    head = np.zeros(len(tab))
    rk = np.zeros(len(tab), np.int32)
    for g, p in enumerate(pubs):
        head[g * cap:g * cap + len(p[1])], rk[g * cap:g * cap + len(p[2])] = p[1], p[2]
    outs = []
    for g, (lo, hi) in enumerate(parts):
        if hi == lo:
            continue
        outs.append(restate_table(params, tab, head, rk, kinds, g * cap, hi - lo, rng, max_rows, custom[lo:hi],
                                  custom_vertices[lo:hi], None if own_count is None else own_count[lo:hi], None,
                                  None if own_vertex_count is None else own_vertex_count[lo:hi]))
    return tuple(np.concatenate([o[k] for o in outs]) for k in range(5)), (tab, head, rk)


def near(gaps, rng, tol=1e-9):
    """the (robot, position) pairs whose gap lies within tol of rng or of the next gap of the list, where the device and
    this restatement may part ways"""
    out = []
    for r, (idx, g) in gaps.items():
        for i in range(len(g)):
            if abs(g[i] - rng) <= tol or (i + 1 < len(g) and g[i + 1] - g[i] <= tol):
                out.append((r, i))
    return out
