"""The obstacle table of a scene built from its local costmap, restated in plain Python, and hand-computed cases for it.

`restate` follows TebLocalPlannerROS::updateObstacleContainerWithCostmap without a costmap_converter plugin
(teb_local_planner_ros.cpp:478-504) and then appends the custom obstacles (:552-625), step by step as include/teb_b200.h
defines it at TebCostmapArgs. TebLocalPlannerROS is not compiled into oracle/_ref: its headers pull in the navigation
stack (costmap_2d, tf, the ROS node). So this restatement is the reference for the device's table. It uses Python floats:
math.cos / math.sin are glibc's, as in the reference's x86 build, and Python does not contract a * b + c into an FMA,
so every product and sum is rounded on its own as there. `restate_np` is the same loop written with numpy's element-wise
float64 operations (each one rounded on its own, in the same order), fast enough for fleets of 120 x 120 maps; the CPU
test holds it bit equal to `restate`.
"""
import math
from dataclasses import dataclass, field

import numpy as np

from teb_local_planner_b200 import abi

LETHAL = abi.COSTMAP_LETHAL


def _rows(xy, custom):
    out = np.zeros(len(xy) + len(custom), abi.OBST_DTYPE)
    if len(xy):
        xy = np.asarray(xy, np.float64).reshape(-1, 2)
        out["x"][:len(xy)], out["y"][:len(xy)] = xy[:, 0], xy[:, 1]
    if len(custom):
        out[len(xy):] = custom
    return out


def restate(cost, sx, sy, origin, robot, behind=1.5, include=True, custom=(), cs=None):
    """The rows of one scene, in order, as an abi.OBST_DTYPE array. cost: the char map (at least sx * sy bytes, cell
    (mx, my) at my * sx + mx); origin (ox, oy, r); robot (x, y, yaw); custom: rows appended verbatim. cs: (cos, sin) of
    the yaw to use instead of math's (to follow a device whose trig differs in the last bit)."""
    ox, oy, r = (float(v) for v in origin)
    rx, ry, rt = (float(v) for v in robot)
    c, s = (math.cos(rt), math.sin(rt)) if cs is None else (float(cs[0]), float(cs[1]))
    behind = float(behind)
    xy = []
    if include and sx >= 2 and sy >= 2:
        for i in range(sx - 1):
            for j in range(sy - 1):
                if int(cost[j * sx + i]) != LETHAL:
                    continue
                wx = ox + (i + 0.5) * r
                wy = oy + (j + 0.5) * r
                dx, dy = wx - rx, wy - ry
                if dx * c + dy * s < 0 and math.sqrt(dx * dx + dy * dy) > behind:
                    continue
                xy.append((wx, wy))
    return _rows(xy, custom)


def restate_np(cost, sx, sy, origin, robot, behind=1.5, include=True, custom=(), cs=None, with_dot=False):
    """restate with numpy's element-wise float64 operations, in the same order; with_dot=True also returns the
    projection dx * c + dy * s and the distance of every row that comes from a cell (in row order)"""
    ox, oy, r = (float(v) for v in origin)
    rx, ry, rt = (float(v) for v in robot)
    c, s = (math.cos(rt), math.sin(rt)) if cs is None else (float(cs[0]), float(cs[1]))
    dot = norm = np.zeros(0)
    xy = np.zeros((0, 2))
    if include and sx >= 2 and sy >= 2:
        grid = np.asarray(cost[:sx * sy], np.uint8).reshape(sy, sx)[:sy - 1, :sx - 1]
        i, j = np.nonzero(grid.T == LETHAL)                         # i outer, j inner: the reference's order
        wx = np.float64(ox) + (i.astype(np.float64) + 0.5) * np.float64(r)
        wy = np.float64(oy) + (j.astype(np.float64) + 0.5) * np.float64(r)
        dx, dy = wx - np.float64(rx), wy - np.float64(ry)
        dot = dx * np.float64(c) + dy * np.float64(s)
        norm = np.sqrt(dx * dx + dy * dy)
        with np.errstate(invalid="ignore"):
            keep = ~((dot < 0) & (norm > np.float64(behind)))
        xy = np.stack([wx[keep], wy[keep]], 1)
        dot, norm = dot[keep], norm[keep]
    rows = _rows(xy, custom)
    return (rows, dot, norm) if with_dot else rows


@dataclass
class Case:
    name: str
    sx: int
    sy: int
    cost: np.ndarray                  # [sy][sx] uint8
    origin: tuple
    robot: tuple
    behind: float
    expect: list                      # hand-computed cell centres, in order
    include: bool = True
    custom: np.ndarray = field(default_factory=lambda: np.zeros(0, abi.OBST_DTYPE))

    def flat(self):
        return np.ascontiguousarray(self.cost, np.uint8).reshape(-1)


def _lethal(sy, sx):
    return np.full((sy, sx), LETHAL, np.uint8)


def custom_rows():
    """one row of every kind the custom list carries: a Circular, a moving Point, a Line and a Polygon on the batch's
    vertex pool, a Pill"""
    o = np.zeros(5, abi.OBST_DTYPE)
    o[0]["type"], o[0]["x"], o[0]["y"], o[0]["radius"] = abi.TEB_OBST_CIRCULAR, 1.5, -0.25, 0.3
    o[1]["type"], o[1]["x"], o[1]["y"], o[1]["vx"], o[1]["vy"], o[1]["dynamic"] = abi.TEB_OBST_POINT, -2.0, 1.0, 0.3, -0.1, 1
    o[2]["type"], o[2]["x"], o[2]["y"], o[2]["vertex_begin"], o[2]["vertex_count"] = abi.TEB_OBST_LINE, 0.5, 0.5, 3, 2
    o[3]["type"], o[3]["x"], o[3]["y"], o[3]["vertex_begin"], o[3]["vertex_count"] = abi.TEB_OBST_POLYGON, 2.0, 2.0, 5, 4
    o[4]["type"], o[4]["x"], o[4]["y"], o[4]["radius"], o[4]["vertex_begin"], o[4]["vertex_count"] = abi.TEB_OBST_PILL, -1.0, -1.0, 0.2, 9, 2
    o[4]["_pad"] = 0.0
    return o


def cases():
    """hand-computed cases; resolution 0.25 and origins on the quarter grid, so every centre is exact"""
    out = []
    # the last column and the last row are never visited; order: i (x) outer, j (y) inner
    out.append(Case("last_row_and_column", 3, 3, _lethal(3, 3), (0.0, 0.0, 0.25), (-10.0, -10.0, 0.0), 1.5,
                    [(0.125, 0.125), (0.125, 0.375), (0.375, 0.125), (0.375, 0.375)]))
    # only 254 counts: 253, 255, 0 and 252 do not; the 254 in the last column and in the last row are not visited
    c = np.array([[253, 254, 255, 0, 254], [254, 254, 254, 254, 254]], np.uint8)
    out.append(Case("only_254", 5, 2, c, (0.0, 0.0, 0.25), (-10.0, 0.0, 0.0), 1.5, [(0.375, 0.125)]))
    c = np.array([[252, 1, 254], [254, 254, 254]], np.uint8)
    out.append(Case("only_254_b", 3, 2, c, (0.0, 0.0, 0.25), (-10.0, 0.0, 0.0), 1.5, []))
    # behind the robot (yaw 0: cos 1, sin 0 exactly), norm == behind_robot_dist is kept, norm > it dropped
    out.append(Case("norm_equal_kept", 5, 2, _lethal(2, 5), (-1.0, -0.125, 0.25), (0.0, 0.0, 0.0), 0.625,
                    [(-0.625, 0.0), (-0.375, 0.0), (-0.125, 0.0)]))
    # straight to the side: dot == 0 is kept however far the cell is
    out.append(Case("dot_zero_kept", 2, 2, _lethal(2, 2), (-0.125, -2.125, 0.25), (0.0, 0.0, 0.0), 0.5, [(0.0, -2.0)]))
    # both conditions are needed: behind and near, ahead and far are kept; behind and far is dropped
    c = np.zeros((2, 18), np.uint8)
    c[0, [0, 2, 4, 8, 12, 16]] = LETHAL
    out.append(Case("both_conditions", 18, 2, c, (-2.125, -0.125, 0.25), (0.0, 0.0, 0.0), 1.0,
                    [(-1.0, 0.0), (0.0, 0.0), (1.0, 0.0), (2.0, 0.0)]))
    # behind_robot_dist -1: every cell behind is dropped; NaN and inf: none is
    out.append(Case("behind_negative", 18, 2, c, (-2.125, -0.125, 0.25), (0.0, 0.0, 0.0), -1.0, [(0.0, 0.0), (1.0, 0.0), (2.0, 0.0)]))
    for b in (math.nan, math.inf):
        out.append(Case(f"behind_{b}", 18, 2, c, (-2.125, -0.125, 0.25), (0.0, 0.0, 0.0), b,
                        [(-2.0, 0.0), (-1.5, 0.0), (-1.0, 0.0), (0.0, 0.0), (1.0, 0.0), (2.0, 0.0)]))
    # sizes 0, 1, 2: only 2 x 2 visits a cell
    for sx in (0, 1, 2):
        for sy in (0, 1, 2):
            out.append(Case(f"size_{sx}x{sy}", sx, sy, _lethal(sy, sx), (0.0, 0.0, 0.25), (0.0, 0.0, 0.0), 1.5,
                            [(0.125, 0.125)] if sx == 2 and sy == 2 else []))
    # a NaN robot keeps every cell: every comparison with NaN is false
    for name, rob in (("nan_x", (math.nan, 0.0, 0.0)), ("nan_yaw", (5.0, 0.0, math.nan))):
        out.append(Case(f"robot_{name}", 3, 2, _lethal(2, 3), (0.0, 0.0, 0.25), rob, 0.0, [(0.125, 0.125), (0.375, 0.125)]))
    # custom rows follow the points, verbatim; without costmap obstacles only they remain
    out.append(Case("custom_after_points", 3, 2, _lethal(2, 3), (0.0, 0.0, 0.25), (0.0, 0.0, 0.0), 1.5,
                    [(0.125, 0.125), (0.375, 0.125)], custom=custom_rows()))
    out.append(Case("custom_only", 3, 2, _lethal(2, 3), (0.0, 0.0, 0.25), (0.0, 0.0, 0.0), 1.5, [], include=False,
                    custom=custom_rows()))
    return out


def expected_rows(case):
    return _rows(case.expect, case.custom)
