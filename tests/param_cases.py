"""Parameter configurations that take every edge-family switch of buildGraph (optimal_planner.cpp:323-366, 444-1021),
as restated by make_kparams (csrc/teb_cabi.cu), to both sides and to its boundary: a named table and seeded random
configurations drawn within the ranges of the reference's cfg/TebLocalPlannerReconfigure.cfg. Each configuration is a
(TebParams, HostBatch) pair whose batch exercises the family being switched: static point and circular obstacles within
the association and penalty distances of the bands, moving obstacles, via-points, prefer_rotdir on two of the bands,
start and goal velocities, perturbed headings and time differences short enough that the velocity and acceleration
penalties are active. Shared by tests/test_reference_pin_params.py (oracle = reference) and tests/test_gpu_params.py
(device = oracle)."""
import math

import numpy as np

from teb_local_planner_b200 import abi, scenes

N_POSES = 24
BANDS = 3


def _batch(seed, shapes=False, n=N_POSES, bands=BANDS):
    """bands along x through a scene of 10 rows near them (4 points, 3 circles, 3 moving points), 3 via-points per band;
    shapes: every second row a Line / Pill / Polygon (the generic distance path)"""
    rng = np.random.default_rng(1000 + seed)
    L = 0.4 * 0.3 * (n - 1)
    poses = np.zeros((bands, n, 4))
    for b in range(bands):
        rec = scenes.make_band(n, rng.uniform(-0.5, 0.5), 0.4, 0.3)
        rec[1:n - 1, 2] += rng.normal(0, 0.25, n - 2)
        rec[:n - 1, 3] *= rng.uniform(0.7, 0.9)              # faster than max_vel_x: velocity penalties active
        poses[b] = rec
    ob = np.zeros(10, abi.OBST_DTYPE)
    ob["x"] = np.linspace(-L / 2 + 0.6, L / 2 - 0.6, 10) + rng.uniform(-0.1, 0.1, 10)
    ob["y"] = rng.choice([-1.0, 1.0], 10) * rng.uniform(0.25, 0.9, 10)
    ob["type"][4:7], ob["radius"][4:7] = abi.TEB_OBST_CIRCULAR, rng.uniform(0.05, 0.2, 3)
    ob["dynamic"][7:] = 1
    ob["vx"][7:], ob["vy"][7:] = rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.2, 0.2, 3)
    sv = np.array([0.25, 0.5, 0.75])
    via = np.zeros((bands, 3, 2))
    for b in range(bands):
        via[b, :, 0] = -L / 2 + L * sv
        via[b, :, 1] = poses[b, (sv * (n - 1)).astype(int), 1] + rng.uniform(-0.3, 0.3, 3)
    vs = np.zeros((bands, 4))
    vs[:, 0], vs[:, 1], vs[:, 2], vs[:, 3] = 0.2, 0.05, -0.1, 1.0
    vg = np.zeros((bands, 4))
    vg[:, 3] = 1.0
    vg[1 % bands, 3] = 0.0                                    # free goal velocity on band 1
    vg[2 % bands, 0] = 0.15
    rot = np.array([abi.TEB_ROTDIR_LEFT, abi.TEB_ROTDIR_RIGHT, abi.TEB_ROTDIR_NONE] * bands, np.int32)[:bands]
    hb = abi.HostBatch(poses, np.full(bands, n, np.int32), ob, np.array([len(ob)], np.int32), None, via,
                       np.full(bands, 3, np.int32), vs, vg, rot)
    if shapes:
        hb = scenes.add_shape_obstacles(hb, seed=seed)
    return hb


def _base():
    p = abi.default_params()
    p.no_inner_iterations, p.no_outer_iterations = 3, 3
    p.teb_autosize = 0
    p.weight_shortest_path = 0.3
    p.weight_velocity_obstacle_ratio = 0.0
    p.obstacle_proximity_lower_bound, p.obstacle_proximity_upper_bound = 0.2, 1.0
    return p


HOLO = dict(max_vel_y=0.3, acc_lim_y=0.4)
CAR = dict(min_turning_radius=0.6)
UP, DOWN = math.nextafter(1.0, math.inf), math.nextafter(1.0, -math.inf)

# name: (overrides, batch) - batch "plain" (points, circles, moving points) or "shapes" (+ Line / Pill / Polygon rows)
NAMED = {
    # the velocity, acceleration, kinematics, time, shortest-path, rotdir and via-point families at 0 / non-zero
    "vel_x0": (dict(weight_max_vel_x=0.0), "plain"),
    "vel_theta0": (dict(weight_max_vel_theta=0.0), "plain"),
    "vel_both0": (dict(weight_max_vel_x=0.0, weight_max_vel_theta=0.0), "plain"),
    "holo_vel_y0": (dict(HOLO, weight_max_vel_y=0.0), "plain"),
    "holo_vel_x_theta0": (dict(HOLO, weight_max_vel_x=0.0, weight_max_vel_theta=0.0), "plain"),
    "holo_vel_all0": (dict(HOLO, weight_max_vel_x=0.0, weight_max_vel_y=0.0, weight_max_vel_theta=0.0), "plain"),
    "holo_acc_y_limit0": (dict(max_vel_y=0.3, acc_lim_y=0.0), "plain"),
    "acc_x0": (dict(weight_acc_lim_x=0.0), "plain"),
    "acc_theta0": (dict(weight_acc_lim_theta=0.0), "plain"),
    "acc_both0": (dict(weight_acc_lim_x=0.0, weight_acc_lim_theta=0.0), "plain"),
    "holo_acc_x_theta0": (dict(HOLO, weight_acc_lim_x=0.0, weight_acc_lim_theta=0.0), "plain"),
    "holo_acc_y0": (dict(HOLO, weight_acc_lim_y=0.0), "plain"),
    "time0": (dict(weight_optimaltime=0.0), "plain"),
    "shortest_path0": (dict(weight_shortest_path=0.0), "plain"),
    "diff_nh0": (dict(weight_kinematics_nh=0.0), "plain"),
    "diff_forward0": (dict(weight_kinematics_forward_drive=0.0), "plain"),
    "diff_both0": (dict(weight_kinematics_nh=0.0, weight_kinematics_forward_drive=0.0), "plain"),
    "car": (dict(CAR), "plain"),
    "car_nh0": (dict(CAR, weight_kinematics_nh=0.0), "plain"),
    "car_forward0": (dict(CAR, weight_kinematics_forward_drive=0.0), "plain"),
    "car_nh0_forward0": (dict(CAR, weight_kinematics_nh=0.0, weight_kinematics_forward_drive=0.0), "plain"),
    "car_radius_weight0": (dict(CAR, weight_kinematics_turning_radius=0.0), "plain"),
    "car_radius_weight0_nh0": (dict(CAR, weight_kinematics_turning_radius=0.0, weight_kinematics_nh=0.0), "plain"),
    "radius0_weight_on": (dict(min_turning_radius=0.0, weight_kinematics_turning_radius=5.0,
                               weight_kinematics_forward_drive=0.0), "plain"),
    "rotdir0": (dict(weight_prefer_rotdir=0.0), "plain"),
    "via0": (dict(weight_viapoint=0.0), "plain"),
    "via_ordered": (dict(via_points_ordered=1), "plain"),
    # the obstacle families
    "obstacle0_dynamic": (dict(weight_obstacle=0.0), "plain"),
    "obstacle0_ratio": (dict(weight_obstacle=0.0, weight_velocity_obstacle_ratio=2.0), "plain"),
    "obstacle0_ratio_static": (dict(weight_obstacle=0.0, weight_velocity_obstacle_ratio=2.0, include_dynamic_obstacles=0),
                               "plain"),
    "ratio": (dict(weight_velocity_obstacle_ratio=2.0), "plain"),
    "ratio_legacy": (dict(weight_velocity_obstacle_ratio=2.0, legacy_obstacle_association=1, obstacle_poses_affected=5),
                     "plain"),
    "dynamic_off": (dict(include_dynamic_obstacles=0), "plain"),
    "inflation_below": (dict(inflation_dist=0.4), "plain"),
    "inflation_equal": (dict(inflation_dist=0.5), "plain"),
    "inflation_above": (dict(inflation_dist=0.7), "plain"),
    "inflation_equal_legacy": (dict(inflation_dist=0.5, legacy_obstacle_association=1, obstacle_poses_affected=5), "plain"),
    "dyn_inflation_below": (dict(dynamic_obstacle_inflation_dist=0.4), "plain"),
    "dyn_inflation_equal": (dict(dynamic_obstacle_inflation_dist=0.5), "plain"),
    "dyn_inflation_above": (dict(dynamic_obstacle_inflation_dist=0.8), "plain"),
    "penalty_epsilon0": (dict(penalty_epsilon=0.0), "plain"),
    "adapt1": (dict(weight_adapt_factor=1.0), "plain"),
    "adapt100": (dict(weight_adapt_factor=100.0), "plain"),
    "force0": (dict(obstacle_association_force_inclusion_factor=0.0), "plain"),
    "cutoff1": (dict(obstacle_association_cutoff_factor=1.0), "plain"),
    "force_above_cutoff": (dict(obstacle_association_force_inclusion_factor=3.0, obstacle_association_cutoff_factor=1.5),
                           "plain"),
    "legacy_affected0": (dict(legacy_obstacle_association=1, obstacle_poses_affected=0), "plain"),
    "legacy_affected1": (dict(legacy_obstacle_association=1, obstacle_poses_affected=1), "plain"),
    "legacy_affected7": (dict(legacy_obstacle_association=1, obstacle_poses_affected=7), "plain"),
    "legacy_affected_n": (dict(legacy_obstacle_association=1, obstacle_poses_affected=N_POSES), "plain"),
    "legacy_affected_above_n": (dict(legacy_obstacle_association=1, obstacle_poses_affected=N_POSES + 7), "plain"),
    "exact_arc_point": (dict(exact_arc_length=1), "plain"),
    "exact_arc_polygon": (dict(exact_arc_length=1, footprint="polygon"), "shapes"),
    "shapes_line_inflation_equal": (dict(inflation_dist=0.5, footprint="line"), "shapes"),
    "shapes_two_circles_ratio": (dict(weight_velocity_obstacle_ratio=1.5, footprint="two_circles"), "shapes"),
}
# obstacle_cost_exponent at 1, the doubles next to 1, below and above 1; each also with min_obstacle_dist = 0
for _name, _e in (("1", 1.0), ("1_up", UP), ("1_down", DOWN), ("0.01", 0.01), ("0.5", 0.5), ("3", 3.0), ("100", 100.0)):
    NAMED[f"exponent_{_name}"] = (dict(obstacle_cost_exponent=_e), "plain")
    NAMED[f"exponent_{_name}_dist0"] = (dict(obstacle_cost_exponent=_e, min_obstacle_dist=0.0), "plain")


def _footprint(p, kind):
    if kind == "point":
        p.footprint_type = abi.TEB_FOOTPRINT_POINT
    elif kind == "circular":
        p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    elif kind == "two_circles":
        p.footprint_type = abi.TEB_FOOTPRINT_TWO_CIRCLES
        p.footprint_front_offset, p.footprint_front_radius = 0.25, 0.15
        p.footprint_rear_offset, p.footprint_rear_radius = 0.2, 0.2
    elif kind == "line":
        scenes.set_line_footprint(p)
    elif kind == "polygon":
        scenes.set_polygon_footprint(p)
    else:
        raise KeyError(kind)


def named(name):
    """-> (TebParams, HostBatch)"""
    over, kind = NAMED[name]
    p = _base()
    for k, v in over.items():
        if k == "footprint":
            _footprint(p, v)
        else:
            setattr(p, k, v)
    return p, _batch(sum(map(ord, name)) % 97, shapes=kind == "shapes")


# --------------------------------------------------------------------------------------------- seeded random draws
WEIGHTS = {  # name: cfg maximum
    "weight_max_vel_x": 1000, "weight_max_vel_y": 1000, "weight_max_vel_theta": 1000, "weight_acc_lim_x": 1000,
    "weight_acc_lim_y": 1000, "weight_acc_lim_theta": 1000, "weight_kinematics_nh": 10000,
    "weight_kinematics_forward_drive": 10000, "weight_kinematics_turning_radius": 1000, "weight_optimaltime": 1000,
    "weight_shortest_path": 100, "weight_obstacle": 1000, "weight_inflation": 10, "weight_dynamic_obstacle": 1000,
    "weight_dynamic_obstacle_inflation": 10, "weight_velocity_obstacle_ratio": 1000, "weight_viapoint": 1000,
    "weight_prefer_rotdir": 1000}
N_RANDOM = 48


def _weight(rng, top):
    u = rng.random()
    if u < 0.3:
        return 0.0
    return float(np.exp(rng.uniform(np.log(1e-2), np.log(top))))


def random_case(k):
    """-> (TebParams, HostBatch): random configuration k; every switch drawn independently, with probability mass on 0
    and on each boundary of a make_kparams predicate"""
    rng = np.random.default_rng(5000 + k)
    p = _base()
    for w, top in WEIGHTS.items():
        setattr(p, w, _weight(rng, top))
    p.min_obstacle_dist = float(rng.choice([0.0, 0.2, 0.5, rng.uniform(0.05, 1.0)]))
    pick = lambda: float(rng.choice([p.min_obstacle_dist, rng.uniform(0.0, 1.5), p.min_obstacle_dist + 0.2]))
    p.inflation_dist, p.dynamic_obstacle_inflation_dist = pick(), pick()
    p.obstacle_cost_exponent = float(rng.choice([1.0, UP, DOWN, 0.01, rng.uniform(0.3, 1.0), rng.uniform(1.0, 4.0), 100.0]))
    p.penalty_epsilon = float(rng.choice([0.0, 0.05, rng.uniform(0.0, 0.2)]))
    p.weight_adapt_factor = float(rng.choice([1.0, 2.0, 100.0, rng.uniform(1.0, 5.0)]))
    p.max_vel_y = float(rng.choice([0.0, 0.0, rng.uniform(0.1, 0.5)]))
    p.acc_lim_y = float(rng.choice([0.0, rng.uniform(0.1, 1.0)]))   # 0 is below the cfg range but reachable by C++ users
    p.max_vel_trans = float(rng.choice([0.0, rng.uniform(0.3, 0.6)]))
    p.min_turning_radius = float(rng.choice([0.0, 0.0, rng.uniform(0.2, 1.5)]))
    p.legacy_obstacle_association = int(rng.random() < 0.3)
    p.obstacle_poses_affected = int(rng.choice([0, 1, int(rng.integers(2, 30)), N_POSES, N_POSES + 5]))
    p.obstacle_association_force_inclusion_factor = float(rng.choice([0.0, 1.5, rng.uniform(0.0, 4.0)]))
    p.obstacle_association_cutoff_factor = float(rng.choice([1.0, 5.0, rng.uniform(1.0, 8.0)]))
    p.include_dynamic_obstacles = int(rng.random() < 0.7)
    p.exact_arc_length = int(rng.random() < 0.3)
    p.via_points_ordered = int(rng.random() < 0.3)
    p.obstacle_proximity_ratio_max_vel = float(rng.uniform(0.0, 1.0))
    p.obstacle_proximity_lower_bound = float(rng.uniform(0.0, 0.4))
    p.obstacle_proximity_upper_bound = float(p.obstacle_proximity_lower_bound + rng.uniform(0.1, 1.0))
    p.no_inner_iterations, p.no_outer_iterations = int(rng.integers(1, 5)), int(rng.integers(1, 4))
    fp = ["point", "circular", "two_circles", "line", "polygon"][int(rng.integers(5))]
    _footprint(p, fp)
    return p, _batch(k, shapes=bool(rng.random() < 0.3))


ALL = list(NAMED) + [f"random_{k}" for k in range(N_RANDOM)]


def case(name):
    if name.startswith("random_"):
        return random_case(int(name[len("random_"):]))
    return named(name)


def args(p):
    return abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale,
                         p.selection_viapoint_cost_scale, bool(p.selection_alternative_time_cost))


def weight_multiplier(p, outer):
    """the obstacle weight multiplier of outer iteration `outer`: weight_adapt_factor applied `outer` times, product by
    product as optimizeTEB does (optimal_planner.cpp:227)"""
    m = 1.0
    for _ in range(outer):
        m *= p.weight_adapt_factor
    return m
