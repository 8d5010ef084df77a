"""Every robot's obstacle layer marked and cleared from its sensor points, restated in plain Python
(TebObstacleLayerArgs in include/teb_b200.h), plus a numpy form for fleets held bit equal to it.

costmap_2d is not part of the reference checkout, so this restates ROS Noetic navigation's ObstacleLayer::updateBounds /
raytraceFreespace / updateFootprint / updateCosts, Costmap2D::updateOrigin / worldToMap / cellDistance / raytraceLine /
bresenham2D / setConvexPolygonCost / convexFillCells / polygonOutlineCells, costmap_2d::transformFootprint,
CostmapLayer::updateWithOverwrite / updateWithMax and the height filter of ObservationBuffer::bufferCloud. Python floats
round every product and sum on its own, as an x86-64 build of costmap_2d does; divisions by zero follow IEEE (_div).

A robot's state is (layer [cell_cap] ints, layer_origin (ox, oy)); the master raster is TebCostmapArgs' row and origin
(ox, oy, r). The parameters are a dict (PARAMS gives every key).
"""
import math

import numpy as np

from tests import costmap_window_cases as cw

OK, BAD_GRID, BAD_POINTS, ORIGIN_MISMATCH = 0, 1, 2, 3
SENSOR_OFF_MAP, FOOTPRINT_OFF_MAP = 1, 2
COMBINE, STANDALONE = 0, 1
FREE_SPACE, LETHAL_OBSTACLE, NO_INFORMATION = 0, 254, 255
UINT_MAX = 2 ** 32 - 1
PARAMS = dict(mode=COMBINE, combination_method=1, track_unknown_space=True, master_default=NO_INFORMATION,
              clearing=True, marking=True, obstacle_range=2.5, raytrace_range=3.0, min_obstacle_height=0.0,
              max_obstacle_height=2.0, layer_max_obstacle_height=2.0)


def _div(a, b):
    """IEEE double division, a / b with b == 0 allowed"""
    if b != 0.0 or math.isnan(b):
        return a / b
    if a == 0.0 or math.isnan(a):
        return math.nan
    return math.copysign(math.inf, a) * math.copysign(1.0, b)


def layer_default(p):
    return NO_INFORMATION if p["track_unknown_space"] else FREE_SPACE


def world_to_map(wx, wy, ox, oy, r, sx, sy):
    """Costmap2D::worldToMap: (mx, my), or None off the map; a quotient that is NaN or at least the size (where C's
    (int) would be undefined or give a cell past the map) is off the map"""
    if wx < ox or wy < oy:
        return None
    qx, qy = (wx - ox) / r, (wy - oy) / r
    if not (qx < sx and qy < sy):
        return None
    return int(qx), int(qy)


def cell_distance(d, r):
    """Costmap2D::cellDistance: (unsigned)max(0, ceil(d / r)), saturated at UINT_MAX"""
    c = max(0.0, math.ceil(d / r)) if math.isfinite(d / r) else math.inf
    return UINT_MAX if c >= UINT_MAX else int(c)


def bresenham(abs_da, abs_db, error_b, offset_a, offset_b, offset, max_length):
    """Costmap2D::bresenham2D: the offsets the action is applied to, in order"""
    out = []
    for _ in range(min(max_length, abs_da)):
        out.append(offset)
        offset += offset_a
        error_b += abs_db
        if error_b >= abs_da:
            offset += offset_b
            error_b -= abs_da
    out.append(offset)
    return out


def raytrace_line(x0, y0, x1, y1, sx, max_length=UINT_MAX):
    """Costmap2D::raytraceLine: the offsets visited from (x0, y0) toward (x1, y1). hypot of the integer deltas is the
    square root of their exact sum of squares, which is the correctly rounded hypot"""
    dx, dy = x1 - x0, y1 - y0
    abs_dx, abs_dy = abs(dx), abs(dy)
    offset_dx = 1 if dx > 0 else -1                  # costmap_2d's sign(): sign(0) is -1
    offset_dy = (1 if dy > 0 else -1) * sx
    offset = y0 * sx + x0
    dist = math.sqrt(dx * dx + dy * dy)
    scale = 1.0 if dist == 0.0 else min(1.0, float(max_length) / dist)
    if abs_dx >= abs_dy:
        return bresenham(abs_dx, abs_dy, abs_dx // 2, offset_dx, offset_dy, offset, int(scale * abs_dx))
    return bresenham(abs_dy, abs_dx, abs_dy // 2, offset_dy, offset_dx, offset, int(scale * abs_dy))


def clamp_to_map(wx, wy, ox, oy, mox, moy, mex, mey):
    """raytraceFreespace's four clamps of the end point (wx, wy) of a ray from the sensor at (ox, oy)"""
    a, b = wx - ox, wy - oy
    if wx < mox:
        t = _div(mox - ox, a)
        wx, wy = mox, oy + b * t
    if wy < moy:
        t = _div(moy - oy, b)
        wx, wy = ox + a * t, moy
    if wx > mex:
        t = _div(mex - ox, a)
        wx, wy = mex - .001, oy + b * t
    if wy > mey:
        t = _div(mey - oy, b)
        wx, wy = ox + a * t, mey - .001
    return wx, wy


def transform_footprint(x, y, yaw, footprint):
    """costmap_2d::transformFootprint"""
    c, s = math.cos(yaw), math.sin(yaw)
    return [(x + (px * c - py * s), y + (px * s + py * c)) for px, py in footprint]


def convex_fill_cells(polygon, sx):
    """Costmap2D::convexFillCells, literally: the outline of polygonOutlineCells (every edge and the closing edge through
    raytraceLine, both ends and duplicates kept), the swap sort by x, then the column loop that takes the cells in pairs
    and appends each column's fill to the vector it reads. Returns the cells as (x, y)."""
    if len(polygon) < 3:
        return []
    cells = []
    edges = [(polygon[k], polygon[k + 1]) for k in range(len(polygon) - 1)] + [(polygon[-1], polygon[0])]
    for (x0, y0), (x1, y1) in edges:
        cells += [(o % sx, o // sx) for o in raytrace_line(x0, y0, x1, y1, sx)]
    i = 0
    while i < len(cells) - 1:
        if cells[i][0] > cells[i + 1][0]:
            cells[i], cells[i + 1] = cells[i + 1], cells[i]
            if i > 0:
                i -= 1
        else:
            i += 1
    i = 0
    min_x, max_x = cells[0][0], cells[-1][0]
    for x in range(min_x, max_x + 1):
        if i >= len(cells) - 1:
            break
        if cells[i][1] < cells[i + 1][1]:
            lo, hi = cells[i], cells[i + 1]
        else:
            lo, hi = cells[i + 1], cells[i]
        i += 2
        while i < len(cells) and cells[i][0] == x:
            if cells[i][1] < lo[1]:
                lo = cells[i]
            elif cells[i][1] > hi[1]:
                hi = cells[i]
            i += 1
        for y in range(lo[1], hi[1]):
            cells.append((x, y))
    return cells


def column_spans(polygon):
    """The cells convexFillCells gives, as a span per column: {x: (y_lo, y_hi)} with every cell y_lo .. y_hi of column x
    filled. Every column from the least to the greatest vertex x holds at least two outline cells (each vertex ends one
    edge and starts the next; a column between is crossed on the way there and back), so the pairing never leaves the
    column it is in, never reads the cells it appended, and fills from the column's least outline y to its greatest.
    Each edge's cells in column x come from bresenham2D in closed form: after k steps the minor axis has moved
    floor((da / 2 + k db) / da) times."""
    if len(polygon) < 3:
        return {}
    spans = {}
    edges = [(polygon[k], polygon[k + 1]) for k in range(len(polygon) - 1)] + [(polygon[-1], polygon[0])]
    for (x0, y0), (x1, y1) in edges:
        for x, ylo, yhi in edge_columns(x0, y0, x1, y1):
            lo, hi = spans.get(x, (ylo, yhi))
            spans[x] = (min(lo, ylo), max(hi, yhi))
    return spans


def edge_columns(x0, y0, x1, y1):
    """(x, least y, greatest y) of the cells raytraceLine visits from (x0, y0) to (x1, y1), per column"""
    dx, dy = x1 - x0, y1 - y0
    sgx, sgy = (1 if dx > 0 else -1), (1 if dy > 0 else -1)
    adx, ady = abs(dx), abs(dy)
    out = []
    if adx >= ady:      # one cell per column
        for k in range(adx + 1):
            y = y0 + sgy * ((adx // 2 + k * ady) // adx) if adx else y0
            out.append((x0 + sgx * k, y, y))
        return out
    e0 = ady // 2
    for m in range(adx + 1):
        if adx == 0:
            klo, khi = 0, ady
        else:
            klo = max(0, -((e0 - m * ady) // adx))                  # ceil((m ady - e0) / adx)
            khi = min(ady, ((m + 1) * ady - e0 - 1) // adx)
        ya, yb = y0 + sgy * klo, y0 + sgy * khi
        out.append((x0 + sgx * m, min(ya, yb), max(ya, yb)))
    return out


def status(grid, cell_cap, layer_origin, r, count, P_cap, robot):
    sx, sy = int(grid[0]), int(grid[1])
    if (sx < 1 or sy < 1 or sx * sy > cell_cap or not (r > 0) or not math.isfinite(r)
            or not math.isfinite(layer_origin[0]) or not math.isfinite(layer_origin[1])
            or not math.isfinite(float(robot[0])) or not math.isfinite(float(robot[1]))):
        return BAD_GRID
    if not 0 <= count <= P_cap:
        return BAD_POINTS
    return OK


def shift_cells(o, p, n, r):
    """updateOrigin's whole-cell move along one axis (a float: NaN or beyond the grid moves every cell out)"""
    q = (p - (cw.size_in_meters(n, r) / 2) - o) / r
    return float(math.trunc(q)) if math.isfinite(q) else q


def combine(method, master, layer):
    """updateWithOverwrite (0) / updateWithMax (1) of one cell; anything else leaves the master"""
    if layer == NO_INFORMATION or method not in (0, 1):
        return master
    if method == 0:
        return layer
    return layer if (master == NO_INFORMATION or master < layer) else master


def obstacle_layer(p, points, sensor, robot, grid, cell_cap, layer, layer_origin, master, origin, footprint=(), P_cap=None):
    """One robot's step. points: list of (x, y, z) float32 values (the first point_count rows), sensor (x, y, z),
    robot (x, y, yaw), layer [cell_cap], layer_origin (ox, oy), master [cell_cap], origin (ox, oy, r). Returns (layer,
    layer_origin, master, origin, status, flags), all new."""
    layer, master = list(layer), list(master)
    lox, loy = float(layer_origin[0]), float(layer_origin[1])
    mox, moy, r = (float(v) for v in origin)
    P_cap = len(points) if P_cap is None else P_cap
    st = status(grid, cell_cap, (lox, loy), r, len(points), P_cap, robot)
    md = p["master_default"]
    if st == OK:
        sx, sy = int(grid[0]), int(grid[1])
        cx, cy = shift_cells(lox, float(robot[0]), sx, r), shift_cells(loy, float(robot[1]), sy, r)
        nox, noy = lox + cx * r, loy + cy * r
        if p["mode"] == COMBINE and (np.float64(nox).tobytes() != np.float64(mox).tobytes()
                                     or np.float64(noy).tobytes() != np.float64(moy).tobytes()):
            st = ORIGIN_MISMATCH
    if st != OK:
        if p["mode"] == STANDALONE:
            master = [md] * cell_cap
        return layer, (lox, loy), master, (mox, moy, r), st, 0
    d = layer_default(p)
    # 1. the shift (updateOrigin), the bytes past sx * sy at the default
    new = [d] * cell_cap
    if abs(cx) < sx and abs(cy) < sy:
        cx, cy = int(cx), int(cy)
        for j in range(sy):
            for i in range(sx):
                if 0 <= i + cx < sx and 0 <= j + cy < sy:
                    new[j * sx + i] = layer[(j + cy) * sx + i + cx]
    layer = new
    if p["mode"] == STANDALONE:
        mox, moy = nox, noy
        master = [md] * cell_cap
    flags = 0
    # 2. the height filter of the observation source
    kept = [(float(x), float(y), float(z)) for x, y, z in points
            if p["min_obstacle_height"] <= float(z) <= p["max_obstacle_height"]]
    ox, oy, oz = (float(v) for v in sensor)
    # 3. clearing
    if p["clearing"]:
        c0 = world_to_map(ox, oy, nox, noy, r, sx, sy)
        if c0 is None:
            flags |= SENSOR_OFF_MAP
        else:
            mex, mey = nox + sx * r, noy + sy * r
            max_length = cell_distance(p["raytrace_range"], r)
            for wx, wy, _ in kept:
                wx, wy = clamp_to_map(wx, wy, ox, oy, nox, noy, mex, mey)
                c1 = world_to_map(wx, wy, nox, noy, r, sx, sy)
                if c1 is None:
                    continue
                for o in raytrace_line(c0[0], c0[1], c1[0], c1[1], sx, max_length):
                    layer[o] = FREE_SPACE
    # 4. marking
    if p["marking"]:
        sq_range = p["obstacle_range"] * p["obstacle_range"]
        for px, py, pz in kept:
            if pz > p["layer_max_obstacle_height"]:
                continue
            if ((px - ox) * (px - ox) + (py - oy) * (py - oy)) + (pz - oz) * (pz - oz) >= sq_range:
                continue
            c = world_to_map(px, py, nox, noy, r, sx, sy)
            if c is not None:
                layer[c[1] * sx + c[0]] = LETHAL_OBSTACLE
    # 5. footprint clearing
    if len(footprint) >= 3:
        placed = transform_footprint(float(robot[0]), float(robot[1]), float(robot[2]), footprint)
        poly = [world_to_map(x, y, nox, noy, r, sx, sy) for x, y in placed]
        if any(c is None for c in poly):
            flags |= FOOTPRINT_OFF_MAP
        else:
            for x, y in convex_fill_cells(poly, sx):
                layer[y * sx + x] = FREE_SPACE
    # 6. combination over the window
    for c in range(sx * sy):
        master[c] = combine(p["combination_method"], master[c], layer[c])
    return layer, (nox, noy), master, (mox, moy, r), st, flags


# ---- the numpy form for fleets

def _ray_cells(x0, y0, x1, y1, max_length, sx):
    """every (ray, offset) raytraceLine visits, for arrays of rays (int64), through bresenham2D in closed form"""
    dx, dy = x1 - x0, y1 - y0
    adx, ady = np.abs(dx), np.abs(dy)
    xdom = adx >= ady
    da, db = np.where(xdom, adx, ady), np.where(xdom, ady, adx)
    sgx, sgy = np.where(dx > 0, 1, -1), np.where(dy > 0, 1, -1)
    dist = np.sqrt((dx * dx + dy * dy).astype(np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = np.where(dist == 0.0, 1.0, np.minimum(1.0, max_length / dist))
    end = np.minimum((scale * da).astype(np.int64), da)
    ray = np.repeat(np.arange(len(x0)), end + 1)
    start = np.cumsum(end + 1) - (end + 1)
    k = np.arange(len(ray)) - np.repeat(start, end + 1)
    dar, dbr = da[ray], db[ray]
    moves = np.where(dar > 0, (dar // 2 + k * dbr) // np.maximum(dar, 1), 0)
    xd = xdom[ray]
    x = x0[ray] + sgx[ray] * np.where(xd, k, moves)
    y = y0[ray] + sgy[ray] * np.where(xd, moves, k)
    return ray, y * sx + x


def _to_map_np(wx, wy, ox, oy, r, sx, sy):
    with np.errstate(invalid="ignore"):
        qx, qy = (wx - ox) / r, (wy - oy) / r
        on = ~(wx < ox) & ~(wy < oy) & (qx < sx) & (qy < sy)
    return on, np.where(on, qx, 0).astype(np.int64), np.where(on, qy, 0).astype(np.int64)


def obstacle_layer_np(p, points, point_count, sensor, robot, grid, cell_cap, layer, layer_origin, master, origin,
                      footprint=()):
    """The whole fleet, bit equal to obstacle_layer(): points [S][P_cap][3] float32, point_count [S], sensor [S][3],
    robot [S][3], grid [S][2], layer / master [S][cell_cap] uint8, layer_origin [S][2], origin [S][3]. Returns (layer,
    layer_origin, master, origin, status, flags), all new arrays."""
    S, P_cap = points.shape[0], points.shape[1]
    layer, master = np.array(layer, np.uint8).copy(), np.array(master, np.uint8).copy()
    lorg, org = np.array(layer_origin, np.float64).copy(), np.array(origin, np.float64).copy()
    st, fl = np.zeros(S, np.int32), np.zeros(S, np.int32)
    d, md, meth = layer_default(p), p["master_default"], p["combination_method"]
    lut = np.array([[combine(meth, m, l) for l in range(256)] for m in range(256)], np.uint8)
    fp = [tuple(map(float, v)) for v in footprint]
    max_length = None
    for s in range(S):
        lox, loy = float(lorg[s, 0]), float(lorg[s, 1])
        mox, moy, r = (float(v) for v in org[s])
        st[s] = status(grid[s], cell_cap, (lox, loy), r, int(point_count[s]), P_cap, robot[s])
        if st[s] == OK:
            sx, sy = int(grid[s][0]), int(grid[s][1])
            cx, cy = shift_cells(lox, float(robot[s][0]), sx, r), shift_cells(loy, float(robot[s][1]), sy, r)
            nox, noy = lox + cx * r, loy + cy * r
            if p["mode"] == COMBINE and (np.float64(nox).tobytes() != np.float64(mox).tobytes()
                                         or np.float64(noy).tobytes() != np.float64(moy).tobytes()):
                st[s] = ORIGIN_MISMATCH
        if st[s] != OK:
            if p["mode"] == STANDALONE:
                master[s] = md
            continue
        old = layer[s, :sx * sy].reshape(sy, sx).copy()
        win = np.full((sy, sx), d, np.uint8)
        if abs(cx) < sx and abs(cy) < sy:
            cx, cy = int(cx), int(cy)
            win[max(0, -cy):sy - max(0, cy), max(0, -cx):sx - max(0, cx)] = \
                old[max(0, cy):sy + min(0, cy), max(0, cx):sx + min(0, cx)]
        lorg[s] = (nox, noy)
        if p["mode"] == STANDALONE:
            org[s, 0], org[s, 1] = nox, noy
            master[s] = md
        pts = points[s, :int(point_count[s])]
        z = pts[:, 2].astype(np.float64)
        with np.errstate(invalid="ignore"):
            keep = (p["min_obstacle_height"] <= z) & (z <= p["max_obstacle_height"])
        px, py, pz = (pts[keep, k].astype(np.float64) for k in range(3))
        ox, oy, oz = (float(v) for v in sensor[s])
        flat = win.reshape(-1)
        if p["clearing"]:
            c0 = world_to_map(ox, oy, nox, noy, r, sx, sy)
            if c0 is None:
                fl[s] |= SENSOR_OFF_MAP
            elif len(px):
                mex, mey = nox + sx * r, noy + sy * r
                max_length = cell_distance(p["raytrace_range"], r)
                wx, wy = px.copy(), py.copy()
                a, b = wx - ox, wy - oy
                with np.errstate(divide="ignore", invalid="ignore"):
                    m = wx < nox
                    t = (nox - ox) / a
                    wx, wy = np.where(m, nox, wx), np.where(m, oy + b * t, wy)
                    m = wy < noy
                    t = (noy - oy) / b
                    wx, wy = np.where(m, ox + a * t, wx), np.where(m, noy, wy)
                    m = wx > mex
                    t = (mex - ox) / a
                    wx, wy = np.where(m, mex - .001, wx), np.where(m, oy + b * t, wy)
                    m = wy > mey
                    t = (mey - oy) / b
                    wx, wy = np.where(m, ox + a * t, wx), np.where(m, mey - .001, wy)
                on, x1, y1 = _to_map_np(wx, wy, nox, noy, r, sx, sy)
                n = int(on.sum())
                if n:
                    _, offs = _ray_cells(np.full(n, c0[0], np.int64), np.full(n, c0[1], np.int64), x1[on], y1[on],
                                         float(max_length), sx)
                    flat[offs] = FREE_SPACE
        if p["marking"] and len(px):
            with np.errstate(invalid="ignore"):
                near = ~(pz > p["layer_max_obstacle_height"])
                sq = ((px - ox) * (px - ox) + (py - oy) * (py - oy)) + (pz - oz) * (pz - oz)
                near &= ~(sq >= p["obstacle_range"] * p["obstacle_range"])
            on, mx, my = _to_map_np(px, py, nox, noy, r, sx, sy)
            on &= near
            flat[my[on] * sx + mx[on]] = LETHAL_OBSTACLE
        if len(fp) >= 3:
            placed = transform_footprint(float(robot[s][0]), float(robot[s][1]), float(robot[s][2]), fp)
            poly = [world_to_map(x, y, nox, noy, r, sx, sy) for x, y in placed]
            if any(c is None for c in poly):
                fl[s] |= FOOTPRINT_OFF_MAP
            else:
                for x, (ylo, yhi) in column_spans(poly).items():
                    win[ylo:yhi + 1, x] = FREE_SPACE
        layer[s] = d
        layer[s, :sx * sy] = flat
        master[s, :sx * sy] = lut[master[s, :sx * sy], flat]
    return layer, lorg, master, org, st, fl


def footprint_near_cell_edge(p_robot, footprint, layer_origin, r, tol=1e-9):
    """True when a placed footprint vertex lies within tol of a cell edge of the layer ((p - o) / r near an integer),
    where the device's sin / cos may put it in the neighbouring cell"""
    for x, y in transform_footprint(float(p_robot[0]), float(p_robot[1]), float(p_robot[2]), footprint):
        for v, o in ((x, layer_origin[0]), (y, layer_origin[1])):
            q = (v - o) / r
            if math.isfinite(q) and abs(q - round(q)) < tol:
                return True
    return False
