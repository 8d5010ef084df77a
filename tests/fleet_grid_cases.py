"""The fleet grid (csrc/teb_fleet.cuh: k_fleet_bin, k_fleet_obstacles_grid) restated on the CPU with the same fp64
operations: the cell side, a point's cell, the bucket of a cell, and the candidates a robot meets. Every operation is
one IEEE double operation rounded on its own, as numpy performs it, so the cells are the device's."""
import numpy as np

from teb_local_planner_b200.abi import FLEET_CELL_BOUND, FLEET_H_FLOOR, FLEET_H_MARGIN

BINNED, FAR, NEVER = 0, 1, 2


def range2(rng):
    with np.errstate(over="ignore"):
        return np.float64(rng) * np.float64(rng)


def cell_side(rng):
    """h = max(range (1 + 2^-16), 2^-500); inf when range * range overflows (every finite pair is then in range)"""
    if not range2(rng) < np.inf:
        return np.inf
    return max(np.float64(rng) * np.float64(FLEET_H_MARGIN), np.float64(FLEET_H_FLOOR))


def cells(x, y, h, fin2):
    """(kind, cx, cy) of points (x, y): kind BINNED with the cell, FAR past the coordinate bound, NEVER for a non-finite
    x or y when range * range is finite"""
    x, y = np.broadcast_arrays(np.atleast_1d(np.asarray(x, np.float64)), np.atleast_1d(np.asarray(y, np.float64)))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        fx, fy = x / np.float64(h), y / np.float64(h)
        binned = (np.abs(fx) < FLEET_CELL_BOUND) & (np.abs(fy) < FLEET_CELL_BOUND)
    kind = np.where(binned, BINNED, np.where(fin2 & ~(np.isfinite(x) & np.isfinite(y)), NEVER, FAR))
    cx = np.where(binned, np.floor(np.where(binned, fx, 0.0)), 0).astype(np.int64)
    cy = np.where(binned, np.floor(np.where(binned, fy, 0.0)), 0).astype(np.int64)
    return kind, cx, cy


def bucket(w, cx, cy, mask):
    """fleet_bucket: the three words as uint32, a multiplicative mix, a 32-bit avalanche, masked"""
    u = lambda v: np.asarray(v, np.int64).astype(np.uint32)
    with np.errstate(over="ignore"):
        k = (u(cx) * np.uint32(0x9E3779B1)) ^ (u(cy) * np.uint32(0x85EBCA77)) ^ (u(w) * np.uint32(0xC2B2AE3D))
        k ^= k >> np.uint32(16)
        k *= np.uint32(0x7FEB352D)
        k ^= k >> np.uint32(15)
        k *= np.uint32(0x846CA68B)
        k ^= k >> np.uint32(16)
    return k & np.uint32(mask)


def in_range(xr, yr, xq, yq, rng):
    """the step's distance rule: dx * dx + dy * dy <= range * range, each operation rounded on its own"""
    with np.errstate(invalid="ignore", over="ignore"):
        f = lambda v: np.asarray(v, np.float64)
        dx, dy = f(xq) - f(xr), f(yq) - f(yr)
        return dx * dx + dy * dy <= range2(rng)


def buckets_of(N):
    """H: the power of two >= 2 N"""
    H = 1
    while H < 2 * N:
        H <<= 1
    return H


def met(xy, world, live, r, rng, one_bucket=False):
    """the candidates robot r meets in k_fleet_obstacles_grid, as a list with repetitions (it must have none): the
    buckets of its 3 x 3 cells, each bucket once, then the far list; every candidate when r is far, none when r is
    never in range"""
    xy = np.asarray(xy, np.float64)
    N = len(xy)
    world = np.zeros(N, np.int64) if world is None else np.asarray(world, np.int64)
    live = np.ones(N, bool) if live is None else np.asarray(live, bool)
    h = cell_side(rng)
    fin2 = bool(range2(rng) < np.inf)
    kind, cx, cy = cells(xy[:, 0], xy[:, 1], h, fin2)
    mask = 0 if one_bucket else buckets_of(N) - 1
    b = np.where(live & (kind == BINNED), bucket(world, cx, cy, mask).astype(np.int64), -1)
    far = np.nonzero(live & (kind == FAR))[0]
    if kind[r] == NEVER:
        return []
    if kind[r] == FAR:
        return list(range(N))
    out, seen = [], []
    for i in range(9):
        bb = int(bucket(world[r], cx[r] + i % 3 - 1, cy[r] + i // 3 - 1, mask))
        if bb in seen:
            continue
        seen.append(bb)
        out += np.nonzero(b == bb)[0].tolist()
    return out + far.tolist()
