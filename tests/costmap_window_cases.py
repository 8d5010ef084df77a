"""Every robot's rolling-window local costmap cut out of a static map, restated in plain Python (TebStaticMaps in
include/teb_b200.h), plus a numpy form held bit equal to it for fleets.

costmap_2d is not part of the reference checkout, so this restates ROS Noetic navigation's Costmap2D::mapToWorld /
worldToMap / getSizeInMetersX / updateOrigin, the rolling branch of LayeredCostmap::updateMap and the rolling branch of
StaticLayer::updateCosts with interpretValue. Python floats and numpy float64 round every product and sum on its own, as
an x86-64 build of costmap_2d does; the transform is tf2's (tests/frame_cases.py).

A map is a dict: data [msy][msx] uint8 (the OccupancyGrid's int8 bytes as unsigned char), mox, moy, mr. The
interpretValue parameters are a dict: unknown_cost_value (the byte, 0 .. 255), lethal_threshold, track_unknown_space,
trinary_costmap.
"""
import math

import numpy as np

from tests import frame_cases as fc

OK, BAD_MAP, BAD_GRID = 0, 1, 2
FREE_SPACE, LETHAL_OBSTACLE, NO_INFORMATION = 0, 254, 255
DEFAULTS = dict(unknown_cost_value=255, lethal_threshold=100, track_unknown_space=True, trinary_costmap=True)


def interpret_value(v, p=DEFAULTS):
    """StaticLayer::interpretValue of the byte v (0 .. 255)"""
    if v == p["unknown_cost_value"]:
        return NO_INFORMATION if p["track_unknown_space"] else FREE_SPACE
    if v >= p["lethal_threshold"]:
        return LETHAL_OBSTACLE
    if p["trinary_costmap"]:
        return FREE_SPACE
    return int(v / p["lethal_threshold"] * 254)      # (unsigned char)(scale * LETHAL_OBSTACLE): truncation


def default_cost(p=DEFAULTS):
    return NO_INFORMATION if p["track_unknown_space"] else FREE_SPACE


def size_in_meters(n, r):
    """Costmap2D::getSizeInMetersX: (size - 1 + 0.5) * resolution"""
    return (float(n - 1) + 0.5) * r


def snap(o, p, n, r):
    """LayeredCostmap::updateMap's rolling branch and Costmap2D::updateOrigin along one axis: the new origin of a window
    of n cells whose previous origin is o, for the robot at p"""
    target = p - size_in_meters(n, r) / 2
    q = (target - o) / r
    cells = float(math.trunc(q)) if math.isfinite(q) else q
    return o + cells * r


def world_to_map(p, o, r, n):
    """worldToMap along one axis: the cell, or None off the map"""
    if p < o:
        return None
    q = (p - o) / r
    return int(q) if q < n else None


def status(maps, map_id, grid, r, cell_cap):
    if not 0 <= map_id < len(maps):
        return BAD_MAP
    m = maps[map_id]
    msy, msx = m["data"].shape
    if msx < 1 or msy < 1 or not (m["mr"] > 0) or not math.isfinite(m["mr"]):
        return BAD_MAP
    sx, sy = int(grid[0]), int(grid[1])
    if sx < 1 or sy < 1 or sx * sy > cell_cap or not (r > 0) or not math.isfinite(r):
        return BAD_GRID
    return OK


def window(maps, robot, map_id, origin, grid, cell_cap, tf=None, p=DEFAULTS):
    """One robot's step: (row [cell_cap] list of ints, origin (ox', oy', r), status). tf: 7 floats or None."""
    d = default_cost(p)
    ox, oy, r = (float(v) for v in origin)
    st = status(maps, map_id, grid, r, cell_cap)
    if st != OK:
        return [d] * cell_cap, (ox, oy, r), st
    sx, sy = int(grid[0]), int(grid[1])
    ox, oy = snap(ox, float(robot[0]), sx, r), snap(oy, float(robot[1]), sy, r)
    m = maps[map_id]
    msy, msx = m["data"].shape
    basis = None if tf is None else fc.tf2_basis([float(v) for v in tf[3:7]])
    row = [d] * cell_cap
    for j in range(sy):
        wy = oy + (j + 0.5) * r
        for i in range(sx):
            wx = ox + (i + 0.5) * r
            px, py = (wx, wy) if basis is None else fc.apply(basis, (float(tf[0]), float(tf[1])), wx, wy, 0.0)
            mx, my = world_to_map(px, m["mox"], m["mr"], msx), world_to_map(py, m["moy"], m["mr"], msy)
            if mx is not None and my is not None:
                row[j * sx + i] = interpret_value(int(m["data"][my, mx]), p)
    return row, (ox, oy, r), st


def _axis_np(pv, o, r, n):
    q = (pv - o) / r
    on = ~(pv < o) & (q < n)
    return on, np.where(on, q, 0.0).astype(np.int64)


def window_np(maps, robot, map_id, origin, grid, cell_cap, tf=None, p=DEFAULTS):
    """The whole fleet, numpy per robot, bit equal to window(): (cost [S][cell_cap] uint8, origin [S][3], status [S])"""
    S = len(robot)
    lut = np.array([interpret_value(v, p) for v in range(256)], np.uint8)
    cost = np.full((S, cell_cap), default_cost(p), np.uint8)
    out = np.array(origin, dtype=np.float64).reshape(S, 3).copy()
    st = np.zeros(S, np.int32)
    for s in range(S):
        ox, oy, r = (float(v) for v in out[s])
        st[s] = status(maps, int(map_id[s]), grid[s], r, cell_cap)
        if st[s] != OK:
            continue
        sx, sy = int(grid[s][0]), int(grid[s][1])
        ox, oy = snap(ox, float(robot[s][0]), sx, r), snap(oy, float(robot[s][1]), sy, r)
        out[s, 0], out[s, 1] = ox, oy
        m = maps[int(map_id[s])]
        msy, msx = m["data"].shape
        wx = ox + (np.arange(sx, dtype=np.float64) + 0.5) * r
        wy = oy + (np.arange(sy, dtype=np.float64) + 0.5) * r
        WX, WY = np.broadcast_to(wx[None, :], (sy, sx)), np.broadcast_to(wy[:, None], (sy, sx))
        if tf is None:
            PX, PY = WX, WY
        else:
            t = [float(v) for v in tf[s]]
            b = fc.tf2_basis(t[3:7])
            PX = b[0] * WX + b[1] * WY + b[2] * 0.0 + t[0]
            PY = b[3] * WX + b[4] * WY + b[5] * 0.0 + t[1]
        onx, mx = _axis_np(PX, m["mox"], m["mr"], msx)
        ony, my = _axis_np(PY, m["moy"], m["mr"], msy)
        on = onx & ony
        win = np.full((sy, sx), default_cost(p), np.uint8)
        win[on] = lut[m["data"][my[on], mx[on]]]
        cost[s, :sx * sy] = win.reshape(-1)
    return cost, out, st


def random_map(rng, msx, msy, mox, moy, mr):
    """an OccupancyGrid of free (0), unknown (-1 -> 255), lethal (100) and graded (1 .. 99) cells in blocks, so windows
    meet runs of equal cells and their edges"""
    bx, by = max(msx // 8, 1), max(msy // 8, 1)
    coarse = rng.choice(np.array([0, 0, 0, 255, 100, 50, 99, 101, 7], np.uint8), size=((msy + by - 1) // by, (msx + bx - 1) // bx))
    data = np.repeat(np.repeat(coarse, by, axis=0), bx, axis=1)[:msy, :msx].copy()
    noise = rng.integers(0, 20, (msy, msx), dtype=np.uint8) == 0
    data[noise] = rng.integers(0, 256, int(noise.sum()), dtype=np.uint8)
    return dict(data=data, mox=float(mox), moy=float(moy), mr=float(mr))
