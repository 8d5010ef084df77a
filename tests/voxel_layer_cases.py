"""Every robot's voxel layer marked and cleared in 3-D from several observation sources, restated in plain Python
(TebVoxelLayerArgs in include/teb_b200.h), plus a numpy form for fleets held bit equal to it.

costmap_2d is not part of the reference checkout, so this restates ROS Noetic navigation's VoxelLayer::updateBounds /
raytraceFreespace / updateOrigin / resetMaps / worldToMap3D / worldToMap3DFloat / reconfigureCB and voxel_grid's
VoxelGrid::reset / markVoxelInMap / clearVoxelLineInMap / raytraceLine / bresenham3D with ClearVoxelInMap, GridOffset
and ZOffset, and bitsBelowThreshold. The height filter, the shift, footprint clearing and the combination come from the
obstacle layer's restatement. Python floats round every product and sum on its own; divisions by zero follow IEEE.

The literal form is sequential: it walks every ray voxel by voxel in costmap_2d's order, clearing every source before
marking any, with the column bit operations spelled out. The numpy form uses the argument at TebVoxelLayerArgs (the
last visit to a column sees its final state), so holding the two equal checks that argument.

A robot's state is (voxels [cell_cap] ints, layer [cell_cap] ints, layer_origin (ox, oy)); the master raster is
TebCostmapArgs' row and origin (ox, oy, r). The layer's parameters are a dict (PARAMS gives every key); each source is
a dict (SOURCE gives every key).
"""
import math

import numpy as np

from tests import costmap_window_cases as cw
from tests import obstacle_layer_cases as ol
from tests.obstacle_layer_cases import _div, world_to_map, cell_distance, shift_cells, combine

OK, BAD_GRID, BAD_POINTS, ORIGIN_MISMATCH = 0, 1, 2, 3
FOOTPRINT_OFF_MAP = 16
COMBINE, STANDALONE = 0, 1
FREE_SPACE, LETHAL_OBSTACLE, NO_INFORMATION = 0, 254, 255
UNKNOWN_COLUMN = 0x0000FFFF
VOXEL_BITS = 16
MAX_SOURCES = 4
UINT_MAX = 2 ** 32 - 1
PARAMS = dict(mode=COMBINE, combination_method=1, track_unknown_space=True, master_default=NO_INFORMATION,
              z_voxels=10, unknown_threshold=15, mark_threshold=0, origin_z=0.0, z_resolution=0.2,
              max_obstacle_height=2.0)
SOURCE = dict(clearing=True, marking=True, obstacle_range=2.5, raytrace_range=3.0, min_obstacle_height=0.0,
              max_obstacle_height=2.0)


def sensor_off_map(k):
    return 1 << k


def source(**kw):
    return dict(SOURCE, **kw)


def _min(a, b):
    """std::min(a, b): b < a ? b : a"""
    return b if b < a else a


def _max(a, b):
    """std::max(a, b): a < b ? b : a"""
    return b if a < b else a


def bits_below_threshold(n, bit_threshold):
    """VoxelGrid::bitsBelowThreshold, literally: clear the lowest set bit until n is 0 or the count passes the bound"""
    bit_count = 0
    while n:
        bit_count += 1
        if bit_count > bit_threshold:
            return False
        n &= n - 1
    return True


def marked_bits(col):
    return col >> 16


def unknown_bits(col):
    return ((col >> 16) & 0xFFFF) ^ (col & 0xFFFF)


def layer_unknown_threshold(p):
    """reconfigureCB: unknown_threshold_ = unknown_threshold + (VOXEL_BITS - size_z_)"""
    return p["unknown_threshold"] + (VOXEL_BITS - p["z_voxels"])


def world_to_map3_float(wx, wy, wz, ox, oy, r, p, sx, sy):
    """VoxelLayer::worldToMap3DFloat: (mx, my, mz) as floats, or None off the grid"""
    oz = p["origin_z"]
    if wx < ox or wy < oy or wz < oz:
        return None
    mx, my, mz = (wx - ox) / r, (wy - oy) / r, (wz - oz) / p["z_resolution"]
    if mx < sx and my < sy and mz < p["z_voxels"]:
        return mx, my, mz
    return None


def world_to_map3(wx, wy, wz, ox, oy, r, p, sx, sy):
    """VoxelLayer::worldToMap3D: (mx, my, mz) as ints, or None off the grid"""
    q = world_to_map3_float(wx, wy, wz, ox, oy, r, p, sx, sy)
    return None if q is None else (int(q[0]), int(q[1]), int(q[2]))


def clear_voxel_in_map(vox, layer, offset, z_mask, unknown_threshold, mark_threshold):
    """ClearVoxelInMap::operator()"""
    vox[offset] &= ~z_mask & 0xFFFFFFFF
    col = vox[offset]
    if bits_below_threshold(marked_bits(col), mark_threshold):
        if bits_below_threshold(unknown_bits(col), unknown_threshold):
            layer[offset] = FREE_SPACE
        else:
            layer[offset] = NO_INFORMATION


def raytrace_line_3d(x0, y0, z0, x1, y1, z1, sx, max_length=UINT_MAX):
    """VoxelGrid::raytraceLine with bresenham3D, GridOffset and ZOffset: the (offset, z_mask) pairs the action is applied
    to, in order"""
    dx, dy, dz = int(x1) - int(x0), int(y1) - int(y0), int(z1) - int(z0)
    abs_dx, abs_dy, abs_dz = abs(dx), abs(dy), abs(dz)
    sign = lambda i: 1 if i > 0 else -1
    offset_dx, offset_dy, offset_dz = sign(dx), sign(dy) * sx, sign(dz)
    z_mask = ((1 << 16) | 1) << int(z0)
    offset = int(y0) * sx + int(x0)
    dist = math.sqrt((x0 - x1) * (x0 - x1) + (y0 - y1) * (y0 - y1) + (z0 - z1) * (z0 - z1))
    scale = _min(1.0, _div(float(max_length), dist))
    state = dict(offset=offset, z_mask=z_mask)

    def grid_off(v):
        state["offset"] += v

    def z_off(v):
        state["z_mask"] = (state["z_mask"] << 1) if v > 0 else (state["z_mask"] >> 1)

    def bresenham3d(off_a, off_b, off_c, abs_da, abs_db, abs_dc, error_b, error_c, offset_a, offset_b, offset_c, length):
        out = []
        for _ in range(min(length, abs_da)):
            out.append((state["offset"], state["z_mask"]))
            off_a(offset_a)
            error_b += abs_db
            error_c += abs_dc
            if error_b >= abs_da:
                off_b(offset_b)
                error_b -= abs_da
            if error_c >= abs_da:
                off_c(offset_c)
                error_c -= abs_da
        out.append((state["offset"], state["z_mask"]))
        return out

    if abs_dx >= max(abs_dy, abs_dz):
        return bresenham3d(grid_off, grid_off, z_off, abs_dx, abs_dy, abs_dz, abs_dx // 2, abs_dx // 2,
                           offset_dx, offset_dy, offset_dz, int(scale * abs_dx))
    if abs_dy >= abs_dz:
        return bresenham3d(grid_off, grid_off, z_off, abs_dy, abs_dx, abs_dz, abs_dy // 2, abs_dy // 2,
                           offset_dy, offset_dx, offset_dz, int(scale * abs_dy))
    return bresenham3d(z_off, grid_off, grid_off, abs_dz, abs_dx, abs_dy, abs_dz // 2, abs_dz // 2,
                       offset_dz, offset_dx, offset_dy, int(scale * abs_dz))


def clearing_end(px, py, pz, so, ox, oy, r, sx, sy, p):
    """raytraceFreespace's end point for one point: the 2 r pull-back, then one t from the z clamps and the four map-edge
    clamps"""
    sox, soy, soz = so
    distance = math.sqrt((px - sox) * (px - sox) + (py - soy) * (py - soy) + (pz - soz) * (pz - soz))
    scaling_fact = _max(_min(1.0, _div(distance - 2 * r, distance)), 0.0)
    wpx = scaling_fact * (px - sox) + sox
    wpy = scaling_fact * (py - soy) + soy
    wpz = scaling_fact * (pz - soz) + soz
    a, b, c = wpx - sox, wpy - soy, wpz - soz
    t = 1.0
    H, oz = p["max_obstacle_height"], p["origin_z"]
    if wpz > H:
        t = _max(0.0, _min(t, _div(H - 0.01 - soz, c)))
    elif wpz < oz:
        t = _min(t, _div(oz - soz, c))
    map_end_x, map_end_y = ox + cw.size_in_meters(sx, r), oy + cw.size_in_meters(sy, r)
    if wpx < ox:
        t = _min(t, _div(ox - sox, a))
    if wpy < oy:
        t = _min(t, _div(oy - soy, b))
    if wpx > map_end_x:
        t = _min(t, _div(map_end_x - sox, a))
    if wpy > map_end_y:
        t = _min(t, _div(map_end_y - soy, b))
    return sox + a * t, soy + b * t, soz + c * t


def status(grid, cell_cap, layer_origin, r, counts, P_cap, robot):
    sx, sy = int(grid[0]), int(grid[1])
    if (sx < 1 or sy < 1 or sx * sy > cell_cap or not (r > 0) or not math.isfinite(r)
            or not math.isfinite(layer_origin[0]) or not math.isfinite(layer_origin[1])
            or not math.isfinite(float(robot[0])) or not math.isfinite(float(robot[1]))):
        return BAD_GRID
    if any(not 0 <= n <= P_cap for n in counts):
        return BAD_POINTS
    return OK


def _kept(src, points):
    return [(float(x), float(y), float(z)) for x, y, z in points
            if src["min_obstacle_height"] <= float(z) <= src["max_obstacle_height"]]


def voxel_layer(p, sources, points, sensors, robot, grid, cell_cap, voxels, layer, layer_origin, master, origin,
                footprint=(), P_cap=None):
    """One robot's step. sources: K dicts; points: K lists of (x, y, z) float32 values (the first point_count rows of
    each source); sensors: K (x, y, z); robot (x, y, yaw); voxels / layer / master [cell_cap]; layer_origin (ox, oy);
    origin (ox, oy, r). Returns (voxels, layer, layer_origin, master, origin, status, flags), all new."""
    voxels, layer, master = [int(v) for v in voxels], list(layer), list(master)
    lox, loy = float(layer_origin[0]), float(layer_origin[1])
    mox, moy, r = (float(v) for v in origin)
    P_cap = max((len(v) for v in points), default=0) if P_cap is None else P_cap
    st = status(grid, cell_cap, (lox, loy), r, [len(v) for v in points], P_cap, robot)
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
        return voxels, layer, (lox, loy), master, (mox, moy, r), st, 0
    d = ol.layer_default(p)
    # 1. updateOrigin: both grids shifted together, resetMaps' values shifted in
    new_l, new_v = [d] * cell_cap, [UNKNOWN_COLUMN] * cell_cap
    if abs(cx) < sx and abs(cy) < sy:
        cx, cy = int(cx), int(cy)
        for j in range(sy):
            for i in range(sx):
                if 0 <= i + cx < sx and 0 <= j + cy < sy:
                    new_l[j * sx + i] = layer[(j + cy) * sx + i + cx]
                    new_v[j * sx + i] = voxels[(j + cy) * sx + i + cx]
    layer, voxels = new_l, new_v
    if p["mode"] == STANDALONE:
        mox, moy = nox, noy
        master = [md] * cell_cap
    flags = 0
    ut, mt = layer_unknown_threshold(p), p["mark_threshold"]
    # 2. the height filter of every source
    kept = [_kept(src, pts) for src, pts in zip(sources, points)]
    # 3. raytraceFreespace for every clearing source, before any marking
    for k, src in enumerate(sources):
        if not src["clearing"]:
            continue
        so = tuple(float(v) for v in sensors[k])
        s0 = world_to_map3_float(*so, nox, noy, r, p, sx, sy)
        if s0 is None:
            flags |= sensor_off_map(k)
            continue
        max_length = cell_distance(src["raytrace_range"], r)
        for px, py, pz in kept[k]:
            w = clearing_end(px, py, pz, so, nox, noy, r, sx, sy, p)
            e = world_to_map3_float(*w, nox, noy, r, p, sx, sy)
            if e is None:
                continue
            # clearVoxelLineInMap's endpoint bounds
            if (s0[0] >= sx or s0[1] >= sy or s0[2] >= p["z_voxels"] or e[0] >= sx or e[1] >= sy
                    or e[2] >= p["z_voxels"]):
                continue
            for offset, z_mask in raytrace_line_3d(*s0, *e, sx, max_length):
                clear_voxel_in_map(voxels, layer, offset, z_mask, ut, mt)
    # 4. marking for every marking source
    for k, src in enumerate(sources):
        if not src["marking"]:
            continue
        ox, oy, oz = (float(v) for v in sensors[k])
        sq_range = src["obstacle_range"] * src["obstacle_range"]
        for px, py, pz in kept[k]:
            if pz > p["max_obstacle_height"]:
                continue
            if (px - ox) * (px - ox) + (py - oy) * (py - oy) + (pz - oz) * (pz - oz) >= sq_range:
                continue
            c = world_to_map3(px, py, p["origin_z"] if pz < p["origin_z"] else pz, nox, noy, r, p, sx, sy)
            if c is None:
                continue
            mx, my, mz = c
            index = my * sx + mx
            voxels[index] |= ((1 << mz) << 16) | (1 << mz)         # markVoxelInMap
            if not bits_below_threshold(marked_bits(voxels[index]), mt):
                layer[index] = LETHAL_OBSTACLE
    # 5. footprint clearing, the 2-D layer only
    if len(footprint) >= 3:
        placed = ol.transform_footprint(float(robot[0]), float(robot[1]), float(robot[2]), footprint)
        poly = [world_to_map(x, y, nox, noy, r, sx, sy) for x, y in placed]
        if any(c is None for c in poly):
            flags |= FOOTPRINT_OFF_MAP
        else:
            for x, y in ol.convex_fill_cells(poly, sx):
                layer[y * sx + x] = FREE_SPACE
    # 6. combination over the window
    for c in range(sx * sy):
        master[c] = combine(p["combination_method"], master[c], layer[c])
    return voxels, layer, (nox, noy), master, (mox, moy, r), st, flags


# ---- the numpy form for fleets

_POPC = np.array([bin(v).count("1") for v in range(1 << 16)], np.int64)


def popcount16(a):
    return _POPC[np.asarray(a, np.int64) & 0xFFFF]


def _ray_voxels(x0, y0, z0, x1, y1, z1, max_length, sx):
    """every (cell, z) raytrace_line_3d visits for arrays of rays (float map coordinates), through bresenham3D in closed
    form: after k steps of the major axis each minor axis has moved floor((da / 2 + k d) / da) times"""
    ix0, iy0, iz0 = x0.astype(np.int64), y0.astype(np.int64), z0.astype(np.int64)
    dx, dy, dz = x1.astype(np.int64) - ix0, y1.astype(np.int64) - iy0, z1.astype(np.int64) - iz0
    adx, ady, adz = np.abs(dx), np.abs(dy), np.abs(dz)
    dist = np.sqrt((x0 - x1) * (x0 - x1) + (y0 - y1) * (y0 - y1) + (z0 - z1) * (z0 - z1))
    with np.errstate(divide="ignore", invalid="ignore"):
        q = max_length / dist
    scale = np.where(q < 1.0, q, 1.0)
    xdom = adx >= np.maximum(ady, adz)
    ydom = ~xdom & (ady >= adz)
    da = np.where(xdom, adx, np.where(ydom, ady, adz))
    end = np.minimum((scale * da).astype(np.int64), da)
    ray = np.repeat(np.arange(len(x0)), end + 1)
    start = np.cumsum(end + 1) - (end + 1)
    k = np.arange(len(ray)) - np.repeat(start, end + 1)
    dar = da[ray]
    out = []
    for d_, i0, dom in ((dx, ix0, xdom), (dy, iy0, ydom), (dz, iz0, ~xdom & ~ydom)):
        ad, sg = np.abs(d_)[ray], np.where(d_ > 0, 1, -1)[ray]
        moves = np.where(dom[ray], k, np.where(dar > 0, (dar // 2 + k * ad) // np.maximum(dar, 1), 0))
        out.append(i0[ray] + sg * moves)
    return out[1] * sx + out[0], out[2]


def voxel_layer_np(p, sources, points, point_count, sensors, robot, grid, cell_cap, voxels, layer, layer_origin, master,
                   origin, footprint=()):
    """The whole fleet, bit equal to voxel_layer(): points [S][K][P_cap][3] float32, point_count [S][K], sensors
    [S][K][3], robot [S][3], grid [S][2], voxels [S][cell_cap] uint32, layer / master [S][cell_cap] uint8,
    layer_origin [S][2], origin [S][3]. Returns (voxels, layer, layer_origin, master, origin, status, flags), all new
    arrays."""
    S, K, P_cap = points.shape[0], points.shape[1], points.shape[2]
    vox = np.array(voxels, np.uint32).copy()
    layer, master = np.array(layer, np.uint8).copy(), np.array(master, np.uint8).copy()
    lorg, org = np.array(layer_origin, np.float64).copy(), np.array(origin, np.float64).copy()
    st, fl = np.zeros(S, np.int32), np.zeros(S, np.int32)
    d, md, meth = ol.layer_default(p), p["master_default"], p["combination_method"]
    ut, mt, Z, oz, zr, H = (layer_unknown_threshold(p), p["mark_threshold"], p["z_voxels"], p["origin_z"],
                            p["z_resolution"], p["max_obstacle_height"])
    lut = np.array([[combine(meth, m, l) for l in range(256)] for m in range(256)], np.uint8)
    fp = [tuple(map(float, v)) for v in footprint]
    for s in range(S):
        lox, loy = float(lorg[s, 0]), float(lorg[s, 1])
        mox, moy, r = (float(v) for v in org[s])
        st[s] = status(grid[s], cell_cap, (lox, loy), r, [int(v) for v in point_count[s]], P_cap, robot[s])
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
        win = np.full((sy, sx), d, np.uint8)
        col = np.full((sy, sx), UNKNOWN_COLUMN, np.uint32)
        if abs(cx) < sx and abs(cy) < sy:
            cx, cy = int(cx), int(cy)
            dst = (slice(max(0, -cy), sy - max(0, cy)), slice(max(0, -cx), sx - max(0, cx)))
            src_ = (slice(max(0, cy), sy + min(0, cy)), slice(max(0, cx), sx + min(0, cx)))
            win[dst] = layer[s, :sx * sy].reshape(sy, sx)[src_]
            col[dst] = vox[s, :sx * sy].reshape(sy, sx)[src_]
        lorg[s] = (nox, noy)
        if p["mode"] == STANDALONE:
            org[s, 0], org[s, 1] = nox, noy
            master[s] = md
        flat, cflat = win.reshape(-1), col.reshape(-1).astype(np.int64)
        kept = []
        for k in range(K):
            pts = points[s, k, :int(point_count[s][k])]
            z = pts[:, 2].astype(np.float64)
            with np.errstate(invalid="ignore"):
                keep = (sources[k]["min_obstacle_height"] <= z) & (z <= sources[k]["max_obstacle_height"])
            kept.append(tuple(pts[keep, j].astype(np.float64) for j in range(3)))
        # clearing: the union of every ray's masks per cell, then the visited cells' bytes from the final columns
        cleared = np.zeros(sx * sy, np.int64)
        visited = np.zeros(sx * sy, bool)
        for k in range(K):
            if not sources[k]["clearing"]:
                continue
            so = tuple(float(v) for v in sensors[s][k])
            s0 = world_to_map3_float(*so, nox, noy, r, p, sx, sy)
            if s0 is None:
                fl[s] |= sensor_off_map(k)
                continue
            px, py, pz = kept[k]
            if not len(px):
                continue
            sox, soy, soz = so
            with np.errstate(divide="ignore", invalid="ignore"):
                dist = np.sqrt((px - sox) * (px - sox) + (py - soy) * (py - soy) + (pz - soz) * (pz - soz))
                f = (dist - 2 * r) / dist
                f = np.where(f < 1.0, f, 1.0)
                f = np.where(f < 0.0, 0.0, f)
                wx, wy, wz = f * (px - sox) + sox, f * (py - soy) + soy, f * (pz - soz) + soz
                a, b, c = wx - sox, wy - soy, wz - soz
                t = np.ones(len(px))
                hi, lo = wz > H, ~(wz > H) & (wz < oz)
                u = (H - 0.01 - soz) / c
                th = np.where(u < t, u, t)
                th = np.where(0.0 < th, th, 0.0)
                u = (oz - soz) / c
                tl = np.where(u < t, u, t)
                t = np.where(hi, th, np.where(lo, tl, t))
                mex, mey = nox + cw.size_in_meters(sx, r), noy + cw.size_in_meters(sy, r)
                for m, num, den in ((wx < nox, nox - sox, a), (wy < noy, noy - soy, b), (wx > mex, mex - sox, a),
                                    (wy > mey, mey - soy, b)):
                    u = num / den
                    t = np.where(m & (u < t), u, t)
                ex, ey, ez = sox + a * t, soy + b * t, soz + c * t
                on = ~(ex < nox) & ~(ey < noy) & ~(ez < oz)
                qx, qy, qz = (ex - nox) / r, (ey - noy) / r, (ez - oz) / zr
                on &= (qx < sx) & (qy < sy) & (qz < Z)
            if not on.any():
                continue
            n = int(on.sum())
            cells, zs = _ray_voxels(np.full(n, s0[0]), np.full(n, s0[1]), np.full(n, s0[2]), qx[on], qy[on], qz[on],
                                    float(cell_distance(sources[k]["raytrace_range"], r)), sx)
            np.bitwise_or.at(cleared, cells, (1 << 16 | 1) << zs)
            visited[cells] = True
        cflat &= ~cleared
        vis = np.nonzero(visited)[0]
        cv = cflat[vis]
        write = popcount16(cv >> 16) <= mt
        byte = np.where(popcount16((cv >> 16) ^ cv) <= ut, FREE_SPACE, NO_INFORMATION)
        flat[vis[write]] = byte[write]
        # marking: the union of the marks per cell, then 254 where the final column passes mark_threshold
        marks = np.zeros(sx * sy, np.int64)
        hit = np.zeros(sx * sy, bool)
        for k in range(K):
            if not sources[k]["marking"]:
                continue
            px, py, pz = kept[k]
            if not len(px):
                continue
            ox_, oy_, oz_ = (float(v) for v in sensors[s][k])
            with np.errstate(invalid="ignore"):
                near = ~(pz > H)
                sq = (px - ox_) * (px - ox_) + (py - oy_) * (py - oy_) + (pz - oz_) * (pz - oz_)
                near &= ~(sq >= sources[k]["obstacle_range"] * sources[k]["obstacle_range"])
                wz = np.where(pz < oz, oz, pz)
                on = near & ~(px < nox) & ~(py < noy) & ~(wz < oz)
                qx, qy, qz = (px - nox) / r, (py - noy) / r, (wz - oz) / zr
                on &= (qx < sx) & (qy < sy) & (qz < Z)
            cells = qy[on].astype(np.int64) * sx + qx[on].astype(np.int64)
            np.bitwise_or.at(marks, cells, (1 << 16 | 1) << qz[on].astype(np.int64))
            hit[cells] = True
        cflat |= marks
        flat[hit & (popcount16(cflat >> 16) > mt)] = LETHAL_OBSTACLE
        if len(fp) >= 3:
            placed = ol.transform_footprint(float(robot[s][0]), float(robot[s][1]), float(robot[s][2]), fp)
            poly = [world_to_map(x, y, nox, noy, r, sx, sy) for x, y in placed]
            if any(c is None for c in poly):
                fl[s] |= FOOTPRINT_OFF_MAP
            else:
                for x, (ylo, yhi) in ol.column_spans(poly).items():
                    win[ylo:yhi + 1, x] = FREE_SPACE
        layer[s] = d
        layer[s, :sx * sy] = flat
        vox[s] = UNKNOWN_COLUMN
        vox[s, :sx * sy] = cflat.astype(np.uint32)
        master[s, :sx * sy] = lut[master[s, :sx * sy], flat]
    return vox, layer, lorg, master, org, st, fl


def reset_rows(S, cell_cap, track_unknown_space=True):
    """resetMaps for S robots: (voxels, layer) at 0x0000FFFF and the layer default"""
    return (np.full((S, cell_cap), UNKNOWN_COLUMN, np.uint32),
            np.full((S, cell_cap), NO_INFORMATION if track_unknown_space else FREE_SPACE, np.uint8))
