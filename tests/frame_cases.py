"""The arithmetic the node does with a transform it has looked up, restated in plain Python: tf2's doTransform of a plan
pose and getYaw, and the Eigen isometry of the custom obstacles with PolygonObstacle::finalizePolygon; and on top of it
the local-plan step of tests/local_plan_cases.py with the global plan in its own frame (TebFrameArgs in
include/teb_b200.h).

tf2, tf2_geometry_msgs, tf2_eigen and Eigen are not part of the reference checkout, so this restates ROS Noetic's code
(tf2 LinearMath Matrix3x3::setRotation / operator* / getRotation, Quaternion operator*, Transform::operator(),
tf2/impl/utils.h getYaw, tf2_eigen transformToEigen) and Eigen 3.3's QuaternionBase::toRotationMatrix and fixed-size
matrix-vector product as an x86-64 SSE2 build evaluates them (rows 0 and 1 of the product summed (m0 v0 + m1 v1) + m2 v2
by the packet path). Python floats round every product and sum on its own, as that build does, and math's trig is
glibc's. A transform is 7 floats: tx, ty, tz, qx, qy, qz, qw. A basis is a row-major list of 9.
"""
import math

from tests import local_plan_cases as lp

TEB_OBST_POINT, TEB_OBST_CIRCULAR, TEB_OBST_LINE, TEB_OBST_PILL, TEB_OBST_POLYGON = range(5)


def tf2_basis(q):
    """tf2::Matrix3x3::setRotation: s = 2 / |q|^2"""
    x, y, z, w = q
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    return [1.0 - (yy + zz), xy - wz, xz + wy,
            xy + wz, 1.0 - (xx + zz), yz - wx,
            xz - wy, yz + wx, 1.0 - (xx + yy)]


def eigen_basis(q):
    """Eigen::QuaternionBase::toRotationMatrix of Quaterniond(w, x, y, z): no division by |q|^2"""
    x, y, z, w = q
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [1.0 - (tyy + tzz), txy - twz, txz + twy,
            txy + twz, 1.0 - (txx + tzz), tyz - twx,
            txz - twy, tyz + twx, 1.0 - (txx + tyy)]


def apply(m, o, vx, vy, vz=0.0):
    """x, y of basis * v + origin, each row summed ((m0 vx + m1 vy) + m2 vz) + o"""
    return tuple(m[3 * i] * vx + m[3 * i + 1] * vy + m[3 * i + 2] * vz + o[i] for i in range(2))


def basis_product(a, b):
    """tf2 Matrix3x3 operator*(a, b)"""
    return [b[j] * a[3 * i] + b[3 + j] * a[3 * i + 1] + b[6 + j] * a[3 * i + 2] for i in range(3) for j in range(3)]


def get_rotation(m):
    """tf2::Matrix3x3::getRotation -> (x, y, z, w)"""
    trace = m[0] + m[4] + m[8]
    q = [0.0] * 4
    if trace > 0.0:
        s = math.sqrt(trace + 1.0)
        q[3] = s * 0.5
        s = 0.5 / s
        q[0] = (m[7] - m[5]) * s
        q[1] = (m[2] - m[6]) * s
        q[2] = (m[3] - m[1]) * s
    else:
        i = (2 if m[4] < m[8] else 1) if m[0] < m[4] else (2 if m[0] < m[8] else 0)
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(m[4 * i] - m[4 * j] - m[4 * k] + 1.0)
        q[i] = s * 0.5
        s = 0.5 / s
        q[3] = (m[3 * k + j] - m[3 * j + k]) * s
        q[j] = (m[3 * j + i] + m[3 * i + j]) * s
        q[k] = (m[3 * k + i] + m[3 * i + k]) * s
    return tuple(q)


def rotation_branch(m):
    """which branch getRotation takes: 'trace', or the index 0 / 1 / 2 of the largest diagonal element"""
    if m[0] + m[4] + m[8] > 0.0:
        return "trace"
    return (2 if m[4] < m[8] else 1) if m[0] < m[4] else (2 if m[0] < m[8] else 0)


GIMBAL = 0.99999


def get_yaw(q):
    """tf2::getYaw (tf2/impl/utils.h)"""
    x, y, z, w = q
    sqx, sqy, sqz, sqw = x * x, y * y, z * z, w * w
    sarg = -2.0 * (x * z - w * y) / (sqx + sqy + sqz + sqw)
    if sarg <= -GIMBAL:
        return -2.0 * math.atan2(y, x)
    if sarg >= GIMBAL:
        return 2.0 * math.atan2(y, x)
    return math.atan2(2.0 * (x * y + w * z), sqw + sqx - sqy - sqz)


def yaw_sarg(q):
    x, y, z, w = q
    return -2.0 * (x * z - w * y) / (x * x + y * y + z * z + w * w)


def quat_mul(a, b):
    """tf2 Quaternion operator*, the raw product"""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return (aw * bx + ax * bw + ay * bz - az * by,
            aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx,
            aw * bw - ax * bx - ay * by - az * bz)


def yaw_quat(yaw):
    return (0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2))


def transform_row(t, row):
    """tf2::doTransform of a plan row (x, y, yaw) under t: (x, y, stored yaw) and the orientation quaternion"""
    tb = tf2_basis(t[3:7])
    x, y = apply(tb, t[:3], row[0], row[1])
    q = get_rotation(basis_product(tb, tf2_basis(yaw_quat(row[2]))))
    return (x, y, get_yaw(q)), q


def row_xy(t, row):
    return apply(tf2_basis(t[3:7]), t[:3], row[0], row[1])


def goal_yaw(t, yaw):
    """estimateLocalGoalOrientation's near-goal heading: getYaw(rotation * global_orientation)"""
    return get_yaw(quat_mul(tuple(t[3:7]), yaw_quat(yaw)))


# ---- custom obstacles
def eigen_point(t, x, y):
    """Isometry3d(Translation3d(t) * Quaterniond(q)) * (x, y, 0), x and y"""
    return apply(eigen_basis(t[3:7]), (0.0 + t[0], 0.0 + t[1]), x, y)


def is_approx(a, b):
    """Eigen's isApprox of two 2-vectors at 1e-12"""
    dx, dy = a[0] - b[0], a[1] - b[1]
    na, nb = a[0] * a[0] + a[1] * a[1], b[0] * b[0] + b[1] * b[1]
    return dx * dx + dy * dy <= 1e-12 * 1e-12 * (nb if nb < na else na)


def polygon_centroid(v):
    """PolygonObstacle::calcCentroid (obstacles.cpp:57-126)"""
    n = len(v)
    if n == 0:
        return (math.nan, math.nan)
    if n == 1:
        return tuple(v[0])
    if n == 2:
        return (0.5 * (v[0][0] + v[1][0]), 0.5 * (v[0][1] + v[1][1]))
    cross = lambda i, j: v[i][0] * v[j][1] - v[j][0] * v[i][1]
    A = 0.0
    for i in range(n - 1):
        A += cross(i, i + 1)
    A += cross(n - 1, 0)
    A *= 0.5
    if A != 0:
        cx = cy = 0.0
        for i in range(n):
            j = (i + 1) % n
            aux = cross(i, j)
            cx += (v[i][0] + v[j][0]) * aux
            cy += (v[i][1] + v[j][1]) * aux
        return (cx / (6.0 * A), cy / (6.0 * A))
    ic = jc = 0
    best = 0.0
    for i in range(n):
        for j in range(i + 1, n):
            dx, dy = v[j][0] - v[i][0], v[j][1] - v[i][1]
            d = math.sqrt(dx * dx + dy * dy)
            if d > best:
                best, ic, jc = d, i, j
    return (0.5 * (v[ic][0] + v[jc][0]), 0.5 * (v[ic][1] + v[jc][1]))


def finalize_polygon(v):
    """fixPolygonClosure (obstacles.cpp:48-55), then calcCentroid: (vertices kept, centroid)"""
    v = [tuple(p) for p in v]
    if len(v) >= 2 and is_approx(v[0], v[-1]):
        v = v[:-1]
    return v, polygon_centroid(v)


def move_custom(rows, vertices, t, out_vertices):
    """updateObstacleContainerWithCustomObstacles on one scene's custom rows (a numpy abi.OBST_DTYPE array, copied) and
    its vertex pool vertices [PV_cap][2] under t; the moved vertices go to out_vertices (modified in place). Returns
    the moved rows."""
    rows = rows.copy()
    for r in rows:
        typ = int(r["type"])
        if typ in (TEB_OBST_POINT, TEB_OBST_CIRCULAR):
            r["x"], r["y"] = eigen_point(t, float(r["x"]), float(r["y"]))
        elif typ in (TEB_OBST_LINE, TEB_OBST_PILL, TEB_OBST_POLYGON):
            vb, vc = int(r["vertex_begin"]), int(r["vertex_count"])
            moved = [eigen_point(t, float(vertices[vb + i][0]), float(vertices[vb + i][1])) for i in range(vc)]
            for i, p in enumerate(moved):
                out_vertices[vb + i] = p
            if typ == TEB_OBST_POLYGON:
                kept, c = finalize_polygon(moved)
                r["vertex_count"] = len(kept)
            else:
                c = (0.5 * (moved[0][0] + moved[1][0]), 0.5 * (moved[0][1] + moved[1][1]))
            r["x"], r["y"] = c
    return rows


# ---- the local plan with the global plan in its own frame
def restate_tf(rows, begin, end, robot, vel, grid, res, a, c2p, p2c, custom_via_count=None, infeasible_count=None,
               since=None, P_cap=1 << 30, V_cap=1 << 30):
    """lp.restate with the global plan in its own frame: c2p / p2c the band's costmap_to_plan / plan_to_costmap. Rows
    stay in the plan frame for the prune and the closest-row search, which compare them with the robot moved by c2p;
    the rows taken, the goal of the goal-reached test and the rows estimateLocalGoalOrientation reads move by p2c."""
    c2p, p2c = [float(v) for v in c2p], [float(v) for v in p2c]
    rx, ry, rt = (float(v) for v in robot)
    px, py = apply(tf2_basis(c2p[3:7]), c2p[:3], rx, ry)
    # 1. prune
    d2 = a.prune_distance * a.prune_distance
    for k in range(begin, end):
        if lp.sq_dist(px, py, rows[k][0], rows[k][1]) < d2:
            begin = k
            break
    g = [tuple(float(v) for v in rows[k]) for k in range(begin, end)]
    n = len(g)
    if n == 0:
        return lp.Out(lp.EMPTY, begin)
    # 3. the window, in the plan frame
    sx, sy = grid
    ax, ay = float(sx) * res / 2.0, float(sy) * res / 2.0
    thr = (ay if ax < ay else ax) * 0.85
    thr = thr * thr
    i, sq, reached = 0, 1e10, False
    for j in range(n):
        new = lp.sq_dist(px, py, g[j][0], g[j][1])
        if reached and new > sq:
            break
        if new < sq:
            sq, i = new, j
            if sq < 0.05:
                reached = True
    first, length, mx = i, 0.0, a.max_lookahead_dist
    while i < n and sq <= thr and (mx <= 0 or length <= mx):
        sq = lp.sq_dist(px, py, g[i][0], g[i][1])
        if i > 0 and mx > 0:
            length += lp.distance_points2d(g[i - 1], g[i])
        i += 1
    if i == first:
        first, size, goal_idx = n - 1, 1, n - 1
    else:
        size, goal_idx = i - first, i - 1
    t = [transform_row(p2c, r)[0] for r in g[first:first + size]]     # the rows taken, in the costmap frame
    # 4. via-points from the transformed rows
    via = None
    if custom_via_count is None:
        via = []
        if not a.viapoint_sep <= 0:
            prev = 0
            for k in range(1, size):
                if lp.distance_points2d(t[prev], t[k]) < a.viapoint_sep:
                    continue
                via.append((t[k][0], t[k][1]))
                prev = k
    vcount = len(via) if via is not None else int(custom_via_count)
    # 5. goal reached, against the transformed global goal
    gx, gy, gyaw = transform_row(p2c, g[n - 1])[0]
    dx, dy = gx - rx, gy - ry
    vx, vy, om = (float(v) for v in vel)
    stopped = abs(om) <= a.theta_stopped_vel and abs(vx) <= a.trans_stopped_vel and abs(vy) <= a.trans_stopped_vel
    if (abs(math.sqrt(dx * dx + dy * dy)) < a.xy_goal_tolerance
            and abs(lp.normalize_theta(gyaw - rt)) < a.yaw_goal_tolerance
            and (not a.complete_global_plan or vcount == 0) and (stopped or a.free_goal_vel)):
        if via is not None and len(via) > V_cap:
            return lp.Out(lp.CAPACITY, begin, goal_idx, needed=(0, len(via)))
        return lp.Out(lp.GOAL_REACHED, begin, goal_idx, via=via, needed=(0, vcount if via is not None else 0))
    # 6. horizon shrink
    enabled = a.shrink_horizon_backup and not (infeasible_count is None and since is None)
    size, goal_idx = lp.shrink_horizon(size, goal_idx, 0 if infeasible_count is None else int(infeasible_count),
                                       math.inf if since is None else float(since), a.shrink_horizon_min_duration, enabled)
    t = t[:size]
    # 7. goal heading (:827-871 with tf_plan_to_global)
    lg = t[-1]
    if not a.overwrite_orientation:
        heading = lg[2]
    elif goal_idx > n - lp.MOVING_AVERAGE_LENGTH - 2:
        heading = lg[2] if goal_idx >= n - 1 else goal_yaw(p2c, g[n - 1][2])
    else:
        m = min(lp.MOVING_AVERAGE_LENGTH, n - goal_idx - 1)
        cands, k = [], lg
        for j in range(goal_idx, goal_idx + m):
            kp1 = row_xy(p2c, g[j + 1])
            cands.append(math.atan2(kp1[1] - k[1], kp1[0] - k[0]))
            k = kp1
        heading = lp.average_angles(cands)
    # 8. start row
    out = [(rx, ry, rt)] + [tuple(r) for r in t[1:-1]] + [(lg[0], lg[1], heading)]
    needed = (len(out), len(via) if via is not None else 0)
    if len(out) > P_cap or (via is not None and len(via) > V_cap):
        return lp.Out(lp.CAPACITY, begin, goal_idx, needed=needed)
    return lp.Out(lp.PLANNED, begin, goal_idx, out, via, needed)


# ---- random transforms
def random_transform(rng, tilted=False, unit=True):
    """a transform with a planar (yaw only) or a tilted rotation; unit=False scales the quaternion"""
    t = [float(v) for v in rng.uniform(-20, 20, 3)]
    if not tilted:
        t[2] = 0.0
        yaw = float(rng.uniform(-math.pi, math.pi))
        q = [0.0, 0.0, math.sin(yaw / 2), math.cos(yaw / 2)]
    else:
        q = [float(v) for v in rng.normal(size=4)]
        nq = math.sqrt(sum(v * v for v in q))
        q = [v / nq for v in q]
    if not unit:
        s = float(rng.uniform(0.8, 1.25))
        q = [v * s for v in q]
    return t + q
