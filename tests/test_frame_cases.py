"""The restatement of tests/frame_cases.py (tf2's doTransform / getYaw and Eigen's isometry as the node uses them) pinned
on hand-computed transforms, on extended-precision rigid-body transforms, and, with the identity transform, on the
local-plan restatement of tests/local_plan_cases.py. Also the ABI mirror of TebFrameArgs and abi.transform_from_se2."""
import ctypes as C
import math

import numpy as np
import pytest

from teb_local_planner_b200 import abi, scenes
from tests import frame_cases as fc
from tests import local_plan_cases as lp

IDENTITY = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]


def test_identity_moves_nothing():
    for x, y, yaw in [(1.5, -2.25, 0.3), (0.0, 0.0, -3.0), (-7.0, 1e-9, 2.9)]:
        (tx, ty, tyaw), q = fc.transform_row(IDENTITY, (x, y, yaw))
        assert (tx, ty) == (x, y)
        assert abs(tyaw - yaw) <= 1e-15
        assert fc.eigen_point(IDENTITY, x, y) == (x, y)
    assert fc.tf2_basis(IDENTITY[3:]) == [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    assert fc.eigen_basis(IDENTITY[3:]) == [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]


def test_pure_translation():
    t = [3.0, -2.0, 0.5, 0.0, 0.0, 0.0, 1.0]
    (x, y, yaw), _ = fc.transform_row(t, (1.25, 0.5, -1.0))
    assert (x, y) == (4.25, -1.5) and abs(yaw + 1.0) <= 1e-15
    assert fc.eigen_point(t, 1.25, 0.5) == (4.25, -1.5)


def test_yaw_pi():
    t = [1.0, 2.0, 0.0, 0.0, 0.0, 1.0, 0.0]
    assert fc.tf2_basis(t[3:]) == [-1.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.0, 0.0, 1.0]
    (x, y, yaw), _ = fc.transform_row(t, (0.5, -0.25, 0.5))
    assert (x, y) == (0.5, 2.25)
    assert abs(math.remainder(yaw - (0.5 + math.pi), 2 * math.pi)) <= 1e-15
    assert fc.eigen_point(t, 0.5, -0.25) == (0.5, 2.25)


def test_roll_pi_mirrors_y_and_the_heading():
    t = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
    assert fc.tf2_basis(t[3:]) == [1.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.0, 0.0, -1.0]
    for yaw in (0.3, -1.2, 2.5):
        (x, y, tyaw), _ = fc.transform_row(t, (1.0, 2.0, yaw))
        assert (x, y) == (1.0, -2.0)
        assert abs(math.remainder(tyaw + yaw, 2 * math.pi)) <= 1e-15
    assert fc.eigen_point(t, 1.0, 2.0) == (1.0, -2.0)


@pytest.mark.parametrize("q, branch", [((0.0, 0.0, 0.0, 1.0), "trace"), ((1.0, 0.0, 0.0, 0.0), 0),
                                       ((0.0, 1.0, 0.0, 0.0), 1), ((0.0, 0.0, 1.0, 0.0), 2)])
def test_get_rotation_branches(q, branch):
    m = fc.tf2_basis(q)
    assert fc.rotation_branch(m) == branch
    assert fc.get_rotation(m) == q                       # a half-turn or the identity comes back exactly


def test_get_rotation_branches_of_turned_rows():
    """every branch taken by a basis product, and the quaternion it gives rotates like the product"""
    seen = set()
    rng = np.random.default_rng(4)
    for _ in range(400):
        t = fc.random_transform(rng, tilted=True)
        m = fc.basis_product(fc.tf2_basis(t[3:]), fc.tf2_basis(fc.yaw_quat(float(rng.uniform(-3, 3)))))
        seen.add(fc.rotation_branch(m))
        back = fc.tf2_basis(fc.get_rotation(m))
        assert max(abs(a - b) for a, b in zip(back, m)) <= 1e-14
    assert seen == {"trace", 0, 1, 2}


def test_get_yaw_gimbal_branches():
    q = (0.5, 0.5, -0.5, 0.5)
    assert fc.yaw_sarg(q) == 1.0 and fc.get_yaw(q) == 2 * math.atan2(0.5, 0.5) == math.pi / 2
    q = (0.5, -0.5, 0.5, 0.5)
    assert fc.yaw_sarg(q) == -1.0 and fc.get_yaw(q) == -2 * math.atan2(-0.5, 0.5) == math.pi / 2
    # just inside the threshold the ordinary branch answers
    a = math.asin(0.99998) / 2
    q = (0.0, math.sin(a), 0.0, math.cos(a))
    assert abs(fc.yaw_sarg(q)) < fc.GIMBAL and fc.get_yaw(q) == math.atan2(2.0 * (0.0 + q[3] * 0.0),
                                                                            q[3] ** 2 + 0.0 - q[1] ** 2 - 0.0)


def test_non_unit_quaternion_tf2_normalises_and_eigen_scales():
    t = [0.0, 0.0, 0.0, 0.0, 0.0, 2.0, 0.0]              # yaw pi, |q| = 2
    assert fc.tf2_basis(t[3:]) == [-1.0, 0.0, 0.0, 0.0, -1.0, 0.0, 0.0, 0.0, 1.0]
    assert fc.eigen_basis(t[3:]) == [-7.0, 0.0, 0.0, 0.0, -7.0, 0.0, 0.0, 0.0, 1.0]
    assert fc.row_xy(t, (1.0, 2.0, 0.0)) == (-1.0, -2.0)
    assert fc.eigen_point(t, 1.0, 2.0) == (-7.0, -14.0)


def test_quaternion_product_near_goal():
    # rotation yaw pi/2 times a row of yaw pi/4: yaw 3 pi / 4
    t = [0.0, 0.0, 0.0, 0.0, 0.0, math.sin(math.pi / 4), math.cos(math.pi / 4)]
    assert abs(fc.goal_yaw(t, math.pi / 4) - 3 * math.pi / 4) <= 1e-15
    assert fc.quat_mul((0.0, 0.0, 0.0, 1.0), (1.0, 2.0, 3.0, 4.0)) == (1.0, 2.0, 3.0, 4.0)


def test_polygon_with_a_repeated_closing_vertex():
    t = [1.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0]
    rows = np.zeros(1, abi.OBST_DTYPE)
    rows[0]["type"], rows[0]["vertex_begin"], rows[0]["vertex_count"] = fc.TEB_OBST_POLYGON, 1, 5
    rows[0]["x"], rows[0]["y"] = 99.0, 99.0
    verts = np.array([[9, 9], [0, 0], [2, 0], [2, 2], [0, 2], [0, 0], [9, 9]], np.float64)
    out = np.full_like(verts, -1.0)
    moved = fc.move_custom(rows, verts, t, out)
    assert moved[0]["vertex_count"] == 4 and (moved[0]["x"], moved[0]["y"]) == (2.0, 2.0)
    assert (out[1:6] == verts[1:6] + 1.0).all() and (out[[0, 6]] == -1.0).all()
    assert fc.polygon_centroid([(0.0, 0.0), (1.0, 1.0), (3.0, 3.0)]) == (1.5, 1.5)   # area 0: the farthest pair


def test_line_and_point_rows():
    t = [0.5, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0]              # yaw pi, then x + 0.5
    rows = np.zeros(3, abi.OBST_DTYPE)
    rows["type"] = [fc.TEB_OBST_POINT, fc.TEB_OBST_CIRCULAR, fc.TEB_OBST_LINE]
    rows["x"], rows["y"], rows["radius"] = [1.0, 2.0, 0.0], [1.0, -1.0, 0.0], [0.0, 0.3, 0.0]
    rows["vx"], rows["vy"], rows["dynamic"] = [0.0, 0.2, 0.0], [0.0, 0.1, 0.0], [0, 1, 0]
    rows[2]["vertex_begin"], rows[2]["vertex_count"] = 0, 2
    verts = np.array([[1.0, 0.0], [3.0, 2.0]])
    out = np.zeros_like(verts)
    m = fc.move_custom(rows, verts, t, out)
    assert (m[0]["x"], m[0]["y"]) == (-0.5, -1.0) and (m[1]["x"], m[1]["y"]) == (-1.5, 1.0)
    assert (m[1]["vx"], m[1]["vy"], m[1]["radius"], m[1]["dynamic"]) == (0.2, 0.1, 0.3, 1)   # the twist is not rotated
    assert (out == [[-0.5, 0.0], [-2.5, -2.0]]).all() and (m[2]["x"], m[2]["y"]) == (-1.5, -1.0)


def _longdouble_rigid(t, x, y, normalise):
    ld = np.longdouble
    tx, ty = ld(t[0]), ld(t[1])
    qx, qy, qz, qw = (ld(v) for v in t[3:7])
    n2 = qx * qx + qy * qy + qz * qz + qw * qw
    s = ld(2) / n2 if normalise else ld(2)
    r00, r01 = 1 - s * (qy * qy + qz * qz), s * (qx * qy - qw * qz)
    r10, r11 = s * (qx * qy + qw * qz), 1 - s * (qx * qx + qz * qz)
    return r00 * ld(x) + r01 * ld(y) + tx, r10 * ld(x) + r11 * ld(y) + ty


@pytest.mark.parametrize("tilted", [False, True], ids=["planar", "tilted"])
def test_random_transforms_against_extended_precision(tilted):
    rng = np.random.default_rng(11 + tilted)
    worst = 0.0
    for _ in range(2000):
        t = fc.random_transform(rng, tilted=tilted)
        x, y = (float(v) for v in rng.uniform(-50, 50, 2))
        scale = abs(t[0]) + abs(t[1]) + abs(x) + abs(y)
        for got, normalise in ((fc.row_xy(t, (x, y, 0.0)), True), (fc.eigen_point(t, x, y), False)):
            want = _longdouble_rigid(t, x, y, normalise)
            for g, w in zip(got, want):
                err = float(abs(np.longdouble(g) - w)) / scale
                worst = max(worst, err)
    assert worst <= 1e-15, worst


def test_identity_transform_restates_the_identity_path():
    """restate_tf under the identity takes every decision lp.restate takes, with the same rows and via-points"""
    d = scenes.global_plans(96, 256, S=4, seed=8)
    for kw in (dict(), dict(viapoint_sep=0.3), dict(max_lookahead_dist=0.0, viapoint_sep=0.05),
               dict(xy_goal_tolerance=0.6, yaw_goal_tolerance=0.5, free_goal_vel=True)):
        for overwrite in (True, False):
            a = lp.Args(overwrite_orientation=overwrite, **kw)
            for b in range(96):
                s = int(d["scene_id"][b])
                args = (d["global_plan"][b], int(d["plan_begin"][b]), int(d["plan_end"][b]), d["robot"][b],
                        d["robot_vel"][b], tuple(int(v) for v in d["grid"][s]), float(d["origin"][s, 2]), a)
                w = lp.restate(*args)
                f = fc.restate_tf(*args, IDENTITY, IDENTITY)
                assert (f.result, f.plan_begin, f.goal_idx, f.needed, f.via) == (w.result, w.plan_begin, w.goal_idx,
                                                                                 w.needed, w.via)
                assert len(f.plan) == len(w.plan)
                for r, (p, q) in enumerate(zip(f.plan, w.plan)):
                    assert p[:2] == q[:2]
                    assert abs(math.remainder(p[2] - q[2], 2 * math.pi)) <= 1e-15, (b, r)


def test_transform_from_se2_is_a_pair_of_inverses():
    c2p, p2c = abi.transform_from_se2(3.0, -1.5, 0.7)
    assert c2p.shape == p2c.shape == (7,)
    for x, y in [(0.0, 0.0), (1.0, 2.0), (-4.0, 0.5)]:
        mx, my = fc.row_xy(list(c2p), (x, y, 0.0))      # odom -> map
        bx, by = fc.row_xy(list(p2c), (mx, my, 0.0))    # and back
        assert abs(bx - x) <= 1e-14 and abs(by - y) <= 1e-14
    assert abs(fc.transform_row(list(c2p), (0.0, 0.0, 0.2))[0][2] - 0.9) <= 1e-15


def test_frame_args_mirror(teblib):
    assert teblib.tebgpu_sizeof(12) == C.sizeof(abi.TebFrameArgs) == 2 * 4 + 5 * 8
    a = abi.make_local_plan_args(8, 8)
    assert a.frames is None
    a = abi.make_local_plan_args(8, 8, costmap_to_plan=16, plan_to_costmap=32)
    assert (a.frames.costmap_to_plan, a.frames.plan_to_costmap, a.frames.custom_to_costmap) == (16, 32, None)
