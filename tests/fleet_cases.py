"""CPU restatement of tebgpu_fleet_obstacles (include/teb_b200.h, TebFleetArgs): every robot's neighbours as the custom
Circular rows a multi-robot publisher would send, read the way updateObstacleContainerWithCustomObstacles reads a circle
message (teb_local_planner_ros.cpp:576-581) with setCentroidVelocity's 0.001 rule (obstacles.h:214-233).

Every product and sum below is one IEEE double operation, rounded on its own (numpy ufuncs and Python floats do not
contract to FMA), so every decision, position and the order are what the device computes; the velocities take sin / cos
from the C library, the device its own, so they agree to ~1e-16 relative. The 0.001 rule is taken of the body command's norm, which the rotation keeps,
so the dynamic flag does not depend on sin / cos either."""
import math

import numpy as np

from teb_local_planner_b200 import abi

TEB_OBST_CIRCULAR = 1
WRITTEN, TRUNCATED, BAD_INPUT, SHARED_SCENE = range(4)
MAX_ROWS = 32


def neighbours(pose, r, rng, world=None):
    """(indices, d2) of robot r's neighbours in (d2, index) order: q != r, the same world, dx * dx + dy * dy <= rng * rng"""
    pose = np.asarray(pose, np.float64)
    dx = pose[:, 0] - pose[r, 0]
    dy = pose[:, 1] - pose[r, 1]
    d2 = dx * dx + dy * dy
    ok = d2 <= rng * rng
    ok[r] = False
    if world is not None:
        world = np.asarray(world)
        ok &= world == world[r]
    idx = np.nonzero(ok)[0]
    order = np.argsort(d2[idx], kind="stable")          # ties keep the ascending index order
    return idx[order], d2[idx[order]]


def row(pose_q, cmd_q, radius_q):
    """the custom row a robot is published as: a circle at its position, its body command rotated into the map frame
    by its heading, static below a speed of 0.001"""
    x, y, th = (float(v) for v in pose_q[:3])
    bx, by = float(cmd_q[0]), float(cmd_q[1])
    c, s = math.cos(th), math.sin(th)
    vx, vy = c * bx - s * by, s * bx + c * by
    moving = not (math.sqrt(bx * bx + by * by) < 0.001)      # the body command's norm, which the rotation keeps
    o = np.zeros((), abi.OBST_DTYPE)
    o["x"], o["y"], o["radius"] = x, y, float(radius_q)
    o["vx"], o["vy"] = (vx, vy) if moving else (0.0, 0.0)
    o["dynamic"], o["type"] = int(moving), TEB_OBST_CIRCULAR
    return o


def restate(pose, last_cmd, radius, rng, max_rows, custom, own_count=None, custom_count=None, world=None, scene=None):
    """tebgpu_fleet_obstacles_device on the host. custom [S][C_cap] OBST_DTYPE (the caller's rows), own_count [S] or
    None (0), custom_count [S] or None (own_count): the values of the scenes no robot writes. Returns (custom,
    custom_count, needed, status) as the device leaves them, BAD_INPUT / SHARED_SCENE robots included."""
    pose = np.asarray(pose, np.float64).reshape(-1, 3)
    R = len(pose)
    cmd = np.asarray(last_cmd, np.float64).reshape(R, 3)
    radius = np.broadcast_to(np.asarray(radius, np.float64), (R,))
    out = np.array(custom, dtype=abi.OBST_DTYPE)
    S, C_cap = out.shape
    own = np.zeros(S, np.int64) if own_count is None else np.asarray(own_count, np.int64)
    cc = own.astype(np.int32) if custom_count is None else np.array(custom_count, np.int32)
    sc = np.arange(R) if scene is None else np.asarray(scene, np.int64)
    claims = np.bincount(sc[(sc >= 0) & (sc < S)], minlength=S)
    needed, status = np.zeros(R, np.int32), np.zeros(R, np.int32)
    for r in range(R):
        s = int(sc[r])
        if s < 0 or s >= S or own[s] < 0 or own[s] > C_cap:
            needed[r], status[r] = -1, BAD_INPUT
            continue
        if scene is not None and claims[s] != 1:
            needed[r], status[r] = -1, SHARED_SCENE
            continue
        idx, _ = neighbours(pose, r, rng, world)
        K = min(int(max_rows), C_cap - int(own[s]))
        written = min(len(idx), K)
        for i in range(written):
            out[s, own[s] + i] = row(pose[idx[i]], cmd[idx[i]], radius[idx[i]])
        cc[s] = own[s] + written
        needed[r] = len(idx)
        status[r] = TRUNCATED if written < len(idx) else WRITTEN
    return out, cc, needed, status
