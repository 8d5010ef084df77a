"""CPU restatement of the fleet table steps (include/teb_b200.h, TebFleetTable): tebgpu_fleet_publish writes every
robot as the row fleet_cases.row makes of it, the shards are padded to one cap and concatenated as
tebgpu_fleet_gather leaves them, and tebgpu_fleet_obstacles_table runs TebFleetArgs' step for one shard's robots with
the candidates taken from every live row. `sharded` does the three steps for a fleet split into contiguous shards; its
concatenated outputs are what fleet_cases.restate gives on the whole fleet."""
import numpy as np

from teb_local_planner_b200 import abi
from tests import fleet_cases as fc


def publish(pose, last_cmd, radius, world=None):
    """[R] abi.FLEET_ROW_DTYPE: the rows robots 0 .. R - 1 are published as"""
    pose = np.asarray(pose, np.float64).reshape(-1, 3)
    R = len(pose)
    cmd = np.asarray(last_cmd, np.float64).reshape(R, 3)
    radius = np.broadcast_to(np.asarray(radius, np.float64), (R,))
    rows = np.zeros(R, abi.FLEET_ROW_DTYPE)
    for q in range(R):
        o = fc.row(pose[q], cmd[q], radius[q])
        for k in ("x", "y", "vx", "vy", "radius", "dynamic"):
            rows[q][k] = o[k]
    rows["world"] = 0 if world is None else np.asarray(world, np.int32)
    rows["live"] = 1
    return rows


def padding(n, like=None):
    """n padding rows (live 0); like: rows whose every other field they copy (padding on top of robots)"""
    rows = np.zeros(n, abi.FLEET_ROW_DTYPE)
    if like is not None and len(like):
        rows[:] = like[np.arange(n) % len(like)]
    rows["live"] = 0
    return rows


def table(shards, cap, pad_like=None):
    """the gathered table: shard g's rows at [g cap, g cap + len), the rest of each shard padding"""
    out = []
    for rows in shards:
        out += [rows, padding(cap - len(rows), rows if pad_like else None)]
    return np.concatenate(out)


def neighbours(rows, me, rng):
    """(table rows, d2) of row me's neighbours in (d2, row) order: live, q != me, the same world, d2 <= rng * rng"""
    dx = rows["x"] - rows["x"][me]
    dy = rows["y"] - rows["y"][me]
    d2 = dx * dx + dy * dy
    ok = (d2 <= rng * rng) & (rows["live"] != 0) & (rows["world"] == rows["world"][me])
    ok[me] = False
    idx = np.nonzero(ok)[0]
    order = np.argsort(d2[idx], kind="stable")
    return idx[order], d2[idx[order]]


def restate(rows, first, R, rng, max_rows, custom, own_count=None, custom_count=None, scene=None):
    """tebgpu_fleet_obstacles_table_device on the host for robots first .. first + R - 1 of the table `rows`. custom,
    own_count, custom_count and scene as fleet_cases.restate. Returns (custom, custom_count, needed, status)."""
    out = np.array(custom, dtype=abi.OBST_DTYPE)
    S, C_cap = out.shape
    own = np.zeros(S, np.int64) if own_count is None else np.asarray(own_count, np.int64)
    cc = own.astype(np.int32) if custom_count is None else np.array(custom_count, np.int32)
    sc = np.arange(R) if scene is None else np.asarray(scene, np.int64)
    claims = np.bincount(sc[(sc >= 0) & (sc < S)], minlength=S)
    needed, status = np.zeros(R, np.int32), np.zeros(R, np.int32)
    for r in range(R):
        s, me = int(sc[r]), first + r
        if not rows["live"][me] or s < 0 or s >= S or own[s] < 0 or own[s] > C_cap:
            needed[r], status[r] = -1, fc.BAD_INPUT
            continue
        if scene is not None and claims[s] != 1:
            needed[r], status[r] = -1, fc.SHARED_SCENE
            continue
        idx, _ = neighbours(rows, me, rng)
        written = min(len(idx), int(max_rows), C_cap - int(own[s]))
        for i in range(written):
            w = rows[idx[i]]
            o = np.zeros((), abi.OBST_DTYPE)
            for k in ("x", "y", "vx", "vy", "radius", "dynamic"):
                o[k] = w[k]
            o["type"] = fc.TEB_OBST_CIRCULAR
            out[s, own[s] + i] = o
        cc[s] = own[s] + written
        needed[r] = len(idx)
        status[r] = fc.TRUNCATED if written < len(idx) else fc.WRITTEN
    return out, cc, needed, status


def split(R, counts):
    """the contiguous shards [lo, hi) of robots 0 .. R - 1 with the given sizes"""
    assert sum(counts) == R
    bounds = np.concatenate([[0], np.cumsum(counts)]).astype(int)
    return [(int(bounds[g]), int(bounds[g + 1])) for g in range(len(counts))]


def sharded(pose, last_cmd, radius, rng, max_rows, custom, counts, own_count=None, custom_count=None, world=None,
            pad_like=False):
    """publish per shard, concatenate with padding, then the step per shard (robot r of a shard writes its own scene,
    scene = None). Returns the concatenated (custom, custom_count, needed, status) and the table."""
    pose = np.asarray(pose, np.float64).reshape(-1, 3)
    R = len(pose)
    cmd = np.asarray(last_cmd, np.float64).reshape(R, 3)
    radius = np.broadcast_to(np.asarray(radius, np.float64), (R,))
    world = None if world is None else np.asarray(world, np.int32)
    custom = np.asarray(custom, abi.OBST_DTYPE)
    own = None if own_count is None else np.asarray(own_count, np.int32)
    ccin = None if custom_count is None else np.asarray(custom_count, np.int32)
    parts = split(R, counts)
    cap = max(1, max(counts))
    shards = [publish(pose[lo:hi], cmd[lo:hi], radius[lo:hi], None if world is None else world[lo:hi]) for lo, hi in parts]
    tab = table(shards, cap, pad_like)
    outs = []
    for g, (lo, hi) in enumerate(parts):
        if hi == lo:
            continue
        outs.append(restate(tab, g * cap, hi - lo, rng, max_rows, custom[lo:hi], None if own is None else own[lo:hi],
                            None if ccin is None else ccin[lo:hi]))
    return tuple(np.concatenate([o[k] for o in outs]) for k in range(4)), tab
