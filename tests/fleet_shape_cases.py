"""CPU restatement of the shaped fleet steps (include/teb_b200.h, TebFleetShapes): the neighbours and the kept list of
fleet_cases.restate / fleet_table_cases.restate, each neighbour then written as its kind's parts (Point, Circular, Line,
Polygon) placed at its pose, as a multi-robot publisher's footprint message is read by
updateObstacleContainerWithCustomObstacles (teb_local_planner_ros.cpp:574-623).

Every product and sum is one IEEE double operation rounded on its own, so the order, the cut, every count and flag are
what the device computes; the placed points take sin / cos from the C library and the device its own, so positions,
vertices and centroids agree to ~1e-15 relative."""
import math

import numpy as np

from teb_local_planner_b200 import abi
from tests import fleet_cases as fc
from tests import fleet_table_cases as ftc

POINT, CIRCULAR, LINE, POLYGON = abi.TEB_OBST_POINT, abi.TEB_OBST_CIRCULAR, abi.TEB_OBST_LINE, abi.TEB_OBST_POLYGON


def is_approx(a, b):
    """Eigen's a.isApprox(b) of 2-vectors at 1e-12 (teb_frame.h teb_eigen_is_approx)"""
    dx, dy = a[0] - b[0], a[1] - b[1]
    na, nb = a[0] * a[0] + a[1] * a[1], b[0] * b[0] + b[1] * b[1]
    return dx * dx + dy * dy <= (1e-12 * 1e-12) * min(na, nb)


def polygon_centroid(v):
    """PolygonObstacle::calcCentroid of the points v (teb_frame.h teb_polygon_centroid)"""
    n = len(v)
    if n == 1:
        return v[0][0], v[0][1]
    if n == 2:
        return 0.5 * (v[0][0] + v[1][0]), 0.5 * (v[0][1] + v[1][1])
    cross = lambda i, j: v[i][0] * v[j][1] - v[j][0] * v[i][1]
    A = 0.0
    for i in range(n - 1):
        A = A + cross(i, i + 1)
    A = (A + cross(n - 1, 0)) * 0.5
    if A != 0:
        cx = cy = 0.0
        for i in range(n):
            j = i + 1 if i + 1 < n else 0
            aux = cross(i, j)
            cx = cx + (v[i][0] + v[j][0]) * aux
            cy = cy + (v[i][1] + v[j][1]) * aux
        return cx / (6.0 * A), cy / (6.0 * A)
    best, ic, jc = 0.0, 0, 0
    for i in range(n):
        for j in range(i + 1, n):
            dx, dy = v[j][0] - v[i][0], v[j][1] - v[i][1]
            d = math.sqrt(dx * dx + dy * dy)
            if d > best:
                best, ic, jc = d, i, j
    return 0.5 * (v[ic][0] + v[jc][0]), 0.5 * (v[ic][1] + v[jc][1])


def place(x, y, th, u):
    """body point u of a robot at (x, y, th): p + R(th) u, each operation rounded on its own; (0, 0) gives p"""
    ux, uy = float(u[0]), float(u[1])
    if ux == 0.0 and uy == 0.0:
        return x, y
    c, s = math.cos(th), math.sin(th)
    return x + (c * ux - s * uy), y + (s * ux + c * uy)


def kind_size(parts):
    """(rows, written points) of a kind"""
    return len(parts), sum(len(p[1]) for p in parts if p[0] in (LINE, POLYGON))


def write_kind(out, cv, s, row, vtx, parts, x, y, th, vx, vy, dyn):
    """neighbour at (x, y, th) with velocity (vx, vy, dyn) as rows out[s, row ..] and points cv[s, vtx ..]"""
    for p in parts:
        typ, pts = p[0], np.asarray(p[1], np.float64).reshape(-1, 2)
        o = np.zeros((), abi.OBST_DTYPE)
        o["vx"], o["vy"], o["dynamic"], o["type"] = vx, vy, dyn, typ
        if typ in (POINT, CIRCULAR):
            o["x"], o["y"] = place(x, y, th, pts[0])
            if typ == CIRCULAR:
                o["radius"] = float(p[2])
        else:
            placed = [place(x, y, th, u) for u in pts]
            cv[s, vtx:vtx + len(placed)] = placed
            n = len(placed)
            if typ == LINE:
                o["x"], o["y"] = 0.5 * (placed[0][0] + placed[1][0]), 0.5 * (placed[0][1] + placed[1][1])
            else:
                if is_approx(placed[0], placed[-1]):
                    n -= 1
                o["x"], o["y"] = polygon_centroid(placed[:n])
            o["vertex_begin"], o["vertex_count"] = vtx, n
            vtx += len(placed)
        out[s, row] = o
        row += 1
    return row, vtx


def _shaped(S, R, C_cap, PV_cap, custom, cv, own_count, custom_count, own_vertex_count, scene, listing, neighbour, kinds):
    """the common step: listing(r) -> (ok, status if not ok, kept list, needed) for robot r; neighbour(q) -> (x, y, th,
    vx, vy, dyn, kind)"""
    out = np.array(custom, dtype=abi.OBST_DTYPE).reshape(S, C_cap)
    cv = np.zeros((S, PV_cap, 2)) if cv is None else np.array(cv, np.float64).reshape(S, PV_cap, 2)
    own = np.zeros(S, np.int64) if own_count is None else np.asarray(own_count, np.int64)
    vown = np.zeros(S, np.int64) if own_vertex_count is None else np.asarray(own_vertex_count, np.int64)
    cc = own.astype(np.int32) if custom_count is None else np.array(custom_count, np.int32)
    sc = np.arange(R) if scene is None else np.asarray(scene, np.int64)
    claims = np.bincount(sc[(sc >= 0) & (sc < S)], minlength=S)
    needed, status = np.zeros(R, np.int32), np.zeros(R, np.int32)
    for r in range(R):
        s = int(sc[r])
        ok, st, idx = listing(r)
        if not ok or s < 0 or s >= S or own[s] < 0 or own[s] > C_cap:
            needed[r], status[r] = -1, fc.BAD_INPUT
            continue
        if scene is not None and claims[s] != 1:
            needed[r], status[r] = -1, fc.SHARED_SCENE
            continue
        if vown[s] < 0 or vown[s] > PV_cap:
            needed[r], status[r] = -1, fc.BAD_INPUT
            continue
        kept = idx[:min(len(idx), int(st), C_cap - int(own[s]))]
        row, vtx, written = int(own[s]), int(vown[s]), 0
        for q in kept:
            x, y, th, vx, vy, dyn, k = neighbour(q)
            if not 0 <= k < len(kinds):
                break
            nr, nv = kind_size(kinds[k])
            if row + nr > C_cap or vtx + nv > PV_cap:
                break                              # it does not fit: the list ends here
            row, vtx = write_kind(out, cv, s, row, vtx, kinds[k], x, y, th, vx, vy, dyn)
            written += 1
        cc[s] = row
        needed[r] = len(idx)
        status[r] = fc.TRUNCATED if written < len(idx) else fc.WRITTEN
    return out, cc, needed, status, cv


def restate(pose, last_cmd, kinds, kind, rng, max_rows, custom, custom_vertices=None, own_count=None, custom_count=None,
            own_vertex_count=None, world=None, scene=None, PV_cap=None):
    """tebgpu_fleet_obstacles_shaped_device on the host. kinds: abi.make_fleet_shapes' library, kind [R]. Returns
    (custom, custom_count, needed, status, custom_vertices) as the device leaves them."""
    pose = np.asarray(pose, np.float64).reshape(-1, 3)
    R = len(pose)
    cmd = np.asarray(last_cmd, np.float64).reshape(R, 3)
    kind = np.broadcast_to(np.asarray(kind, np.int64), (R,))
    S, C_cap = np.asarray(custom).shape
    PV = (0 if custom_vertices is None else np.asarray(custom_vertices).shape[1]) if PV_cap is None else PV_cap

    def listing(r):
        idx, _ = fc.neighbours(pose, r, rng, world)
        return True, max_rows, idx

    def neighbour(q):
        o = fc.row(pose[q], cmd[q], 0.0)
        return pose[q, 0], pose[q, 1], pose[q, 2], o["vx"], o["vy"], int(o["dynamic"]), int(kind[q])

    return _shaped(S, R, C_cap, PV, custom, custom_vertices, own_count, custom_count, own_vertex_count, scene, listing,
                   neighbour, kinds)


def publish(pose, last_cmd, radius, kind, world=None):
    """tebgpu_fleet_publish_shaped of robots 0 .. R - 1: (rows, heading, row_kind)"""
    pose = np.asarray(pose, np.float64).reshape(-1, 3)
    return (ftc.publish(pose, last_cmd, radius, world), pose[:, 2].copy(),
            np.broadcast_to(np.asarray(kind, np.int32), (len(pose),)).copy())


def restate_table(rows, heading, row_kind, kinds, first, R, rng, max_rows, custom, custom_vertices=None, own_count=None,
                  custom_count=None, own_vertex_count=None, scene=None, PV_cap=None):
    """tebgpu_fleet_obstacles_table_shaped_device on the host for robots first .. first + R - 1 of the table"""
    S, C_cap = np.asarray(custom).shape
    PV = (0 if custom_vertices is None else np.asarray(custom_vertices).shape[1]) if PV_cap is None else PV_cap

    def listing(r):
        me = first + r
        if not rows["live"][me]:
            return False, 0, None
        idx, _ = ftc.neighbours(rows, me, rng)
        return True, max_rows, idx

    def neighbour(q):
        w = rows[q]
        return w["x"], w["y"], heading[q], w["vx"], w["vy"], int(w["dynamic"]), int(row_kind[q])

    return _shaped(S, R, C_cap, PV, custom, custom_vertices, own_count, custom_count, own_vertex_count, scene, listing,
                   neighbour, kinds)


def sharded(pose, last_cmd, kinds, kind, rng, max_rows, custom, custom_vertices, counts, own_count=None,
            own_vertex_count=None, world=None):
    """publish per shard into one padded table with its companions, then the table step per shard (robot r of a shard
    writes its own scene). Returns the concatenated (custom, custom_count, needed, status, custom_vertices) and the
    table (rows, heading, row_kind)."""
    pose = np.asarray(pose, np.float64).reshape(-1, 3)
    R = len(pose)
    kind = np.broadcast_to(np.asarray(kind, np.int32), (R,))
    world = None if world is None else np.asarray(world, np.int32)
    parts = ftc.split(R, counts)
    cap = max(1, max(counts))
    pubs = [publish(pose[lo:hi], np.asarray(last_cmd)[lo:hi], 0.0, kind[lo:hi], None if world is None else world[lo:hi])
            for lo, hi in parts]
    tab = ftc.table([p[0] for p in pubs], cap)
    head = np.zeros(len(tab))
    rk = np.zeros(len(tab), np.int32)
    for g, p in enumerate(pubs):
        head[g * cap:g * cap + len(p[1])], rk[g * cap:g * cap + len(p[2])] = p[1], p[2]
    outs = []
    for g, (lo, hi) in enumerate(parts):
        if hi == lo:
            continue
        outs.append(restate_table(tab, head, rk, kinds, g * cap, hi - lo, rng, max_rows, custom[lo:hi],
                                  custom_vertices[lo:hi], None if own_count is None else own_count[lo:hi],
                                  None, None if own_vertex_count is None else own_vertex_count[lo:hi]))
    return tuple(np.concatenate([o[k] for o in outs]) for k in range(5)), (tab, head, rk)
