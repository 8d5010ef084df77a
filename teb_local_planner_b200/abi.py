"""ctypes mirror of include/teb_b200.h (the C-ABI of the H100-native TEB optimizer).

Field order and types must match the header exactly; `check_sizes(lib)` compares against
`tebgpu_sizeof()` exported by the library.
"""
import ctypes as C

import numpy as np

TEBGPU_OK = 0
TEBGPU_ERR_INVALID_ARG = -1
TEBGPU_ERR_CUDA = -2
TEBGPU_ERR_UNSUPPORTED = -3
TEBGPU_ERR_CAPACITY = -4
TEBGPU_ERR_NO_DEVICE = -5

TEB_STATUS_OPTIMIZED = 1
TEB_STATUS_TOO_FEW_POSES = 2
TEB_STATUS_CHOL_FAILED = 4
TEB_STATUS_NONFINITE = 8
TEB_STATUS_TERMINATED = 16
TEB_STATUS_DISABLED = 32
TEB_STATUS_CAPACITY = 64
TEB_STATUS_BAD_INPUT = 128

TEB_FOOTPRINT_POINT, TEB_FOOTPRINT_CIRCULAR, TEB_FOOTPRINT_TWO_CIRCLES, TEB_FOOTPRINT_LINE, TEB_FOOTPRINT_POLYGON = range(5)
TEB_OBST_POINT, TEB_OBST_CIRCULAR, TEB_OBST_LINE, TEB_OBST_PILL, TEB_OBST_POLYGON = range(5)
TEB_MAX_FOOTPRINT_VERTICES = 16
TEB_ROTDIR_NONE, TEB_ROTDIR_LEFT, TEB_ROTDIR_RIGHT = 0, 1, 2

_d, _i = C.c_double, C.c_int32


class TebParams(C.Structure):
    _fields_ = [
        # trajectory
        ("dt_ref", _d), ("dt_hysteresis", _d),
        ("force_reinit_new_goal_dist", _d), ("force_reinit_new_goal_angular", _d),
        ("teb_autosize", _i), ("min_samples", _i), ("max_samples", _i), ("exact_arc_length", _i),
        ("via_points_ordered", _i), ("allow_init_with_backwards_motion", _i),
        ("global_plan_overwrite_orientation", _i), ("_pad0", _i),
        # robot
        ("max_vel_x", _d), ("max_vel_x_backwards", _d), ("max_vel_y", _d), ("max_vel_trans", _d),
        ("max_vel_theta", _d), ("acc_lim_x", _d), ("acc_lim_y", _d), ("acc_lim_theta", _d),
        ("min_turning_radius", _d),
        # footprint
        ("footprint_radius", _d), ("footprint_front_offset", _d), ("footprint_front_radius", _d),
        ("footprint_rear_offset", _d), ("footprint_rear_radius", _d),
        ("footprint_type", _i), ("footprint_vertex_count", _i),
        ("footprint_line", _d * 4), ("footprint_vertices", _d * (2 * 16)),
        # obstacles
        ("min_obstacle_dist", _d), ("inflation_dist", _d), ("dynamic_obstacle_inflation_dist", _d),
        ("obstacle_association_force_inclusion_factor", _d), ("obstacle_association_cutoff_factor", _d),
        ("obstacle_proximity_ratio_max_vel", _d), ("obstacle_proximity_lower_bound", _d),
        ("obstacle_proximity_upper_bound", _d),
        ("include_dynamic_obstacles", _i), ("legacy_obstacle_association", _i),
        ("obstacle_poses_affected", _i), ("_pad2", _i),
        # optim
        ("penalty_epsilon", _d), ("weight_max_vel_x", _d), ("weight_max_vel_y", _d),
        ("weight_max_vel_theta", _d), ("weight_acc_lim_x", _d), ("weight_acc_lim_y", _d),
        ("weight_acc_lim_theta", _d), ("weight_kinematics_nh", _d),
        ("weight_kinematics_forward_drive", _d), ("weight_kinematics_turning_radius", _d),
        ("weight_optimaltime", _d), ("weight_shortest_path", _d), ("weight_obstacle", _d),
        ("weight_inflation", _d), ("weight_dynamic_obstacle", _d),
        ("weight_dynamic_obstacle_inflation", _d), ("weight_velocity_obstacle_ratio", _d),
        ("weight_viapoint", _d), ("weight_prefer_rotdir", _d), ("weight_adapt_factor", _d),
        ("obstacle_cost_exponent", _d),
        ("no_inner_iterations", _i), ("no_outer_iterations", _i), ("optimization_activate", _i), ("_pad3", _i),
        # hcp
        ("selection_cost_hysteresis", _d), ("selection_prefer_initial_plan", _d),
        ("selection_obst_cost_scale", _d), ("selection_viapoint_cost_scale", _d),
        ("selection_alternative_time_cost", _i), ("enable_multithreading", _i),
        ("h_signature_prescaler", _d), ("h_signature_threshold", _d),
        # recovery
        ("divergence_detection_enable", _i), ("_pad4", _i),
        ("divergence_detection_max_chi_squared", _d),
    ]


class TebObstacle(C.Structure):
    _fields_ = [("x", _d), ("y", _d), ("vx", _d), ("vy", _d), ("radius", _d), ("dynamic", _i), ("type", _i),
                ("vertex_begin", _i), ("vertex_count", _i), ("_pad", _d)]


OBST_DTYPE = np.dtype([("x", "f8"), ("y", "f8"), ("vx", "f8"), ("vy", "f8"), ("radius", "f8"),
                       ("dynamic", "i4"), ("type", "i4"), ("vertex_begin", "i4"), ("vertex_count", "i4"), ("_pad", "f8")])
assert OBST_DTYPE.itemsize == C.sizeof(TebObstacle) == 64


class TebBatch(C.Structure):
    _fields_ = [
        ("B", _i), ("n_cap", _i), ("S", _i), ("M_cap", _i), ("V_cap", _i), ("PV_cap", _i),
        ("poses", C.c_void_p), ("n", C.c_void_p), ("scene_id", C.c_void_p),
        ("obstacles", C.c_void_p), ("obst_count", C.c_void_p), ("obst_vertices", C.c_void_p),
        ("via", C.c_void_p), ("via_count", C.c_void_p),
        ("vel_start", C.c_void_p), ("vel_goal", C.c_void_p), ("prefer_rotdir", C.c_void_p),
        ("cost", C.c_void_p), ("chi2", C.c_void_p), ("status", C.c_void_p), ("lm_iters", C.c_void_p),
    ]


class TebOptimizeArgs(C.Structure):
    _fields_ = [("iterations_innerloop", _i), ("iterations_outerloop", _i),
                ("compute_cost_afterwards", _i), ("alternative_time_cost", _i),
                ("obst_cost_scale", _d), ("viapoint_cost_scale", _d)]


class TebPlanInput(C.Structure):
    """TebOptimalPlanner::plan + getVelocityCommand per band (tebgpu_plan_batch): host or device pointers"""
    _fields_ = [("start", C.c_void_p), ("goal", C.c_void_p), ("initial_plan", C.c_void_p), ("plan_count", C.c_void_p),
                ("P_cap", _i), ("look_ahead_poses", _i), ("prevent_look_ahead_poses_near_goal", _i), ("_pad", _i),
                ("cmd", C.c_void_p), ("path", C.c_void_p)]


TEB_PLAN_PATH_NONE, TEB_PLAN_PATH_COLD, TEB_PLAN_PATH_WARM, TEB_PLAN_PATH_REINIT = -1, 0, 1, 2


class TebFeasibilityArgs(C.Structure):
    """TebOptimalPlanner::isTrajectoryFeasible per band (tebgpu_check_feasible): arguments, and host or device output
    pointers"""
    _fields_ = [("look_ahead_idx", _i), ("max_queries", _i), ("lookahead_distance", _d), ("inscribed_radius", _d),
                ("angular_resolution", _d), ("collision_distance", _d),
                ("feasible", C.c_void_p), ("query_count", C.c_void_p), ("queries", C.c_void_p)]


TEBGPU_FEAS_BUILD_STAGED, TEBGPU_FEAS_BUILD_GLOBAL = 0, 1


def make_feasibility_args(inscribed_radius, look_ahead_idx=-1, lookahead_distance=-1.0, angular_resolution=np.pi,
                          collision_distance=0.0, max_queries=1024, feasible=None, query_count=None,
                          queries=None) -> TebFeasibilityArgs:
    """TebFeasibilityArgs with the outputs given as addresses (ints, or None for NULL). The defaults are the
    reference's: the whole band, no look-ahead distance, min_resolution_collision_check_angular = pi."""
    f = TebFeasibilityArgs()
    f.look_ahead_idx, f.max_queries = int(look_ahead_idx), int(max_queries)
    f.lookahead_distance, f.inscribed_radius = float(lookahead_distance), float(inscribed_radius)
    f.angular_resolution, f.collision_distance = float(angular_resolution), float(collision_distance)
    f.feasible, f.query_count, f.queries = feasible, query_count, queries
    return f


class TebCostmapWorld(C.Structure):
    """The costmap world of tebgpu_check_feasible_costmap: each scene's raster (TebCostmapArgs' layout), the footprint
    (a host array, copied into the launch) and an optional query_cost output (host or device pointer)"""
    _fields_ = [("cell_cap", _i), ("footprint_count", _i), ("cost", C.c_void_p), ("grid", C.c_void_p),
                ("origin", C.c_void_p), ("footprint", C.c_void_p), ("query_cost", C.c_void_p)]


TEBGPU_FEAS_BUILD_COSTMAP = 2
TEB_COSTMAP_FOOTPRINT_MAX = 64
COSTMAP_INSCRIBED, COSTMAP_NO_INFORMATION = 253, 255   # costmap_2d::INSCRIBED_INFLATED_OBSTACLE, NO_INFORMATION


def make_costmap_world(cell_cap, cost, grid, origin, footprint=None, query_cost=None):
    """TebCostmapWorld: cost / grid / origin / query_cost as addresses (ints, or None for NULL), footprint a [F][2]
    array of the robot-frame points (None or empty: F = 0). The returned struct keeps the footprint array alive."""
    w = TebCostmapWorld()
    fp = np.ascontiguousarray(np.zeros((0, 2)) if footprint is None else footprint, dtype=np.float64).reshape(-1, 2)
    w.cell_cap, w.footprint_count = int(cell_cap), len(fp)
    w.cost, w.grid, w.origin, w.query_cost = cost, grid, origin, query_cost
    w.footprint = fp.ctypes.data if len(fp) else None
    w._keep = fp
    return w


class TebTrajectoryArgs(C.Structure):
    """getVelocityProfile / getFullTrajectory read-out (tebgpu_read_trajectory): the bands to read (NULL: all B) and
    host or device output pointers"""
    _fields_ = [("bands", C.c_void_p), ("count", _i), ("_pad", _i), ("profile", C.c_void_p), ("trajectory", C.c_void_p),
                ("points", C.c_void_p)]


class TebCostmapArgs(C.Structure):
    """Each scene's obstacle table from its local costmap (tebgpu_costmap_obstacles): the rasters, their geometry, the
    robot poses, optional custom rows, and host or device output pointers"""
    _fields_ = [("S", _i), ("cell_cap", _i), ("M_cap", _i), ("C_cap", _i), ("include_costmap_obstacles", _i), ("_pad", _i),
                ("behind_robot_dist", _d), ("cost", C.c_void_p), ("grid", C.c_void_p), ("origin", C.c_void_p),
                ("robot", C.c_void_p), ("custom", C.c_void_p), ("custom_count", C.c_void_p), ("obstacles", C.c_void_p),
                ("obst_count", C.c_void_p), ("needed", C.c_void_p)]


COSTMAP_LETHAL = 254   # costmap_2d::LETHAL_OBSTACLE, the one cost that gives a row


class TebLocalPlanArgs(C.Structure):
    """Each robot's global plan cut into its local plan, goal and via-points (tebgpu_local_plan): the global plans, the
    robots, the costmap sizes, the step's parameters, and host or device output pointers"""
    _fields_ = [("G_cap", _i), ("P_cap", _i), ("V_cap", _i), ("free_goal_vel", _i), ("complete_global_plan", _i),
                ("shrink_horizon_backup", _i), ("prune_distance", _d), ("max_lookahead_dist", _d), ("viapoint_sep", _d),
                ("xy_goal_tolerance", _d), ("yaw_goal_tolerance", _d), ("trans_stopped_vel", _d),
                ("theta_stopped_vel", _d), ("shrink_horizon_min_duration", _d),
                ("global_plan", C.c_void_p), ("plan_begin", C.c_void_p), ("plan_end", C.c_void_p), ("robot", C.c_void_p),
                ("robot_vel", C.c_void_p), ("grid", C.c_void_p), ("origin", C.c_void_p),
                ("infeasible_count", C.c_void_p), ("since_infeasible", C.c_void_p), ("plan", C.c_void_p),
                ("plan_count", C.c_void_p), ("goal_idx", C.c_void_p), ("via", C.c_void_p), ("via_count", C.c_void_p),
                ("result", C.c_void_p), ("needed", C.c_void_p)]


# TEB_LOCAL_PLAN_*: the result of a band's local plan
TEB_LOCAL_PLAN_PLANNED, TEB_LOCAL_PLAN_GOAL_REACHED, TEB_LOCAL_PLAN_EMPTY, TEB_LOCAL_PLAN_CAPACITY, \
    TEB_LOCAL_PLAN_BAD_INPUT = range(5)


def make_local_plan_args(G_cap, P_cap, V_cap=0, prune_distance=1.0, max_lookahead_dist=1.0, viapoint_sep=-1.0,
                         xy_goal_tolerance=0.2, yaw_goal_tolerance=0.2, trans_stopped_vel=0.1, theta_stopped_vel=0.1,
                         shrink_horizon_min_duration=10.0, free_goal_vel=False, complete_global_plan=True,
                         shrink_horizon_backup=True, costmap_to_plan=None, plan_to_costmap=None,
                         **arrays) -> TebLocalPlanArgs:
    """TebLocalPlanArgs with the scalars set (the defaults are the reference's, teb_config.h:259-298, :381-382) and the
    arrays given by keyword as addresses (ints, or None for NULL): global_plan=..., plan_begin=..., ...
    costmap_to_plan / plan_to_costmap (addresses of [B][7] transforms, see TebFrameArgs) are kept on the returned struct
    as its `frames` (an abi.TebFrameArgs, None when both are None) for the _tf entry points."""
    a = TebLocalPlanArgs()
    a.frames = (None if costmap_to_plan is None and plan_to_costmap is None
                else make_frame_args(costmap_to_plan=costmap_to_plan, plan_to_costmap=plan_to_costmap))
    a.G_cap, a.P_cap, a.V_cap = int(G_cap), int(P_cap), int(V_cap)
    a.free_goal_vel, a.complete_global_plan = int(bool(free_goal_vel)), int(bool(complete_global_plan))
    a.shrink_horizon_backup = int(bool(shrink_horizon_backup))
    a.prune_distance, a.max_lookahead_dist, a.viapoint_sep = float(prune_distance), float(max_lookahead_dist), float(viapoint_sep)
    a.xy_goal_tolerance, a.yaw_goal_tolerance = float(xy_goal_tolerance), float(yaw_goal_tolerance)
    a.trans_stopped_vel, a.theta_stopped_vel = float(trans_stopped_vel), float(theta_stopped_vel)
    a.shrink_horizon_min_duration = float(shrink_horizon_min_duration)
    names = {f[0] for f in TebLocalPlanArgs._fields_[14:]}
    for k, v in arrays.items():
        if k not in names:
            raise TypeError(f"unknown TebLocalPlanArgs array {k}")
        setattr(a, k, v)
    return a


class TebFrameArgs(C.Structure):
    """The frames of tebgpu_local_plan_tf / tebgpu_costmap_obstacles_tf: per-robot plan transforms [B][7], per-scene
    custom-obstacle transforms [S][7] (tx, ty, tz, qx, qy, qz, qw) and the custom vertex pools [S][PV_cap][2], as host
    or device pointers; NULL everywhere is the identity"""
    _fields_ = [("PV_cap", _i), ("_pad", _i), ("costmap_to_plan", C.c_void_p), ("plan_to_costmap", C.c_void_p),
                ("custom_to_costmap", C.c_void_p), ("custom_vertices", C.c_void_p), ("obst_vertices", C.c_void_p)]


class TebHsigFactors(C.Structure):
    """Every scene's factor table of the 2-D H-signature (tebgpu_hsig_factors): factor [S][M_cap][2] float64, the
    mantissa of Q_l = 1 / prod_j (o_l - o_j); factor_exp [S][M_cap] int32, its binary exponent (INT32_MIN for 0);
    factor_count [S] int32, the obst_count the table was built at, or -1. Host or device pointers."""
    _fields_ = [("factor", C.c_void_p), ("factor_exp", C.c_void_p), ("factor_count", C.c_void_p)]


def make_hsig_factors(factor, factor_exp, factor_count) -> TebHsigFactors:
    """TebHsigFactors with the arrays given as addresses (ints)"""
    f = TebHsigFactors()
    f.factor, f.factor_exp, f.factor_count = factor, factor_exp, factor_count
    return f


def make_frame_args(costmap_to_plan=None, plan_to_costmap=None, custom_to_costmap=None, custom_vertices=None,
                    obst_vertices=None, PV_cap=0) -> TebFrameArgs:
    """TebFrameArgs with the arrays given as addresses (ints, or None for NULL)"""
    f = TebFrameArgs()
    f.PV_cap = int(PV_cap)
    f.costmap_to_plan, f.plan_to_costmap = costmap_to_plan, plan_to_costmap
    f.custom_to_costmap, f.custom_vertices, f.obst_vertices = custom_to_costmap, custom_vertices, obst_vertices
    return f


def transform_from_se2(x, y, yaw):
    """The pair of transforms a planar parent -> child pose (x, y, yaw) gives, as the node looks them up for a plan in
    the parent frame (map) and a costmap in the child frame (odom): (costmap_to_plan, plan_to_costmap), 7 doubles each
    (tx, ty, tz, qx, qy, qz, qw). costmap_to_plan is the pose itself; plan_to_costmap its inverse, formed in closed form
    (the device never inverts a transform)."""
    x, y, yaw = float(x), float(y), float(yaw)
    c, s = np.cos(yaw), np.sin(yaw)
    qz, qw = np.sin(yaw / 2), np.cos(yaw / 2)
    fwd = np.array([x, y, 0.0, 0.0, 0.0, qz, qw])
    inv = np.array([-(c * x + s * y), s * x - c * y, 0.0, 0.0, 0.0, -qz, qw])
    return fwd, inv


class TebCycleArgs(C.Structure):
    """The controller steps around plan() (tebgpu_backup_modes / tebgpu_finish_cycle): their scalars, the per-band
    inputs, the controller state carried between cycles and the outputs, as host or device pointers"""
    _fields_ = [("use_proportional_saturation", _i), ("cmd_angle_instead_rotvel", _i), ("oscillation_recovery", _i),
                ("buffer_length", _i), ("L_cap", _i), ("_pad", _i), ("wheelbase", _d), ("oscillation_v_eps", _d),
                ("oscillation_omega_eps", _d), ("oscillation_recovery_min_duration", _d), ("now", _d),
                ("local_plan_result", C.c_void_p), ("robot_vel", C.c_void_p), ("cmd", C.c_void_p),
                ("feasible", C.c_void_p), ("infeasible_count", C.c_void_p), ("last_infeasible", C.c_void_p),
                ("last_oscillation", C.c_void_p), ("last_cmd", C.c_void_p), ("prefer_rotdir", C.c_void_p),
                ("osc_ring", C.c_void_p), ("osc_fill", C.c_void_p), ("cmd_vel", C.c_void_p), ("outcome", C.c_void_p),
                ("oscillating", C.c_void_p)]


# TEB_CYCLE_*: what tebgpu_finish_cycle did with a band
TEB_CYCLE_COMMAND, TEB_CYCLE_GOAL_REACHED, TEB_CYCLE_NO_PLAN, TEB_CYCLE_PLAN_FAILED, TEB_CYCLE_DIVERGED, \
    TEB_CYCLE_INFEASIBLE, TEB_CYCLE_UNDECIDABLE, TEB_CYCLE_INVALID_COMMAND, TEB_CYCLE_STEERING_NOT_FINITE = range(9)


def make_cycle_args(now, buffer_length=50, L_cap=None, use_proportional_saturation=False,
                    cmd_angle_instead_rotvel=False, wheelbase=1.0, oscillation_recovery=True, oscillation_v_eps=0.1,
                    oscillation_omega_eps=0.1, oscillation_recovery_min_duration=10.0, params=None,
                    **arrays) -> TebCycleArgs:
    """TebCycleArgs with the scalars set and the arrays given by keyword as addresses (ints, or None for NULL). The
    defaults are the reference's (teb_config.h:286-289, :383-386); buffer_length 50 is the node's
    round(oscillation_filter_duration * controller_frequency) = round(10 * 5) (teb_local_planner_ros.cpp:188); L_cap
    None: buffer_length. params: a TebParams whose max_vel_trans 0 is replaced by max_vel_x here, as the node's
    reconfigure does (teb_config.cpp:219-224); pass it to set_params afterwards."""
    if params is not None and params.max_vel_trans == 0.0:
        params.max_vel_trans = params.max_vel_x
    a = TebCycleArgs()
    a.buffer_length = int(buffer_length)
    a.L_cap = int(buffer_length if L_cap is None else L_cap)
    a.use_proportional_saturation = int(bool(use_proportional_saturation))
    a.cmd_angle_instead_rotvel = int(bool(cmd_angle_instead_rotvel))
    a.oscillation_recovery = int(bool(oscillation_recovery))
    a.wheelbase, a.now = float(wheelbase), float(now)
    a.oscillation_v_eps, a.oscillation_omega_eps = float(oscillation_v_eps), float(oscillation_omega_eps)
    a.oscillation_recovery_min_duration = float(oscillation_recovery_min_duration)
    names = {f[0] for f in TebCycleArgs._fields_[11:]}
    for k, v in arrays.items():
        if k not in names:
            raise TypeError(f"unknown TebCycleArgs array {k}")
        setattr(a, k, v)
    return a


# the controller state a robot carries between cycles (TebCycleArgs' in/out arrays), and which of it is int32
CYCLE_STATE = ("infeasible_count", "last_infeasible", "last_oscillation", "last_cmd", "prefer_rotdir", "osc_ring",
               "osc_fill")
CYCLE_STATE_INT = ("infeasible_count", "prefer_rotdir", "osc_fill")


def make_cycle_state(B, L_cap=50):
    """The state of B robots that have not run a cycle yet (the node's constructor): no infeasible plan, never
    infeasible or oscillating (-inf), last_cmd 0, no preferred turning direction, empty detector rings [L_cap][B][2]"""
    return dict(infeasible_count=np.zeros(B, np.int32), last_infeasible=np.full(B, -np.inf),
                last_oscillation=np.full(B, -np.inf), last_cmd=np.zeros((B, 3)),
                prefer_rotdir=np.full(B, TEB_ROTDIR_NONE, np.int32), osc_ring=np.zeros((int(L_cap), B, 2)),
                osc_fill=np.zeros((B, 2), np.int32))


class TebFleetArgs(C.Structure):
    """The other robots of a fleet as custom obstacle rows of every robot's scene (tebgpu_fleet_obstacles): the robots'
    poses [R][3], body commands [R][3] (TebCycleArgs.last_cmd), radii [R], optional worlds / scenes [R], each scene's
    own custom rows [S], and the custom rows / counts written, as host or device pointers"""
    _fields_ = [("R", _i), ("S", _i), ("C_cap", _i), ("max_rows", _i), ("range", _d), ("pose", C.c_void_p),
                ("last_cmd", C.c_void_p), ("radius", C.c_void_p), ("world", C.c_void_p), ("scene", C.c_void_p),
                ("own_count", C.c_void_p), ("custom", C.c_void_p), ("custom_count", C.c_void_p), ("needed", C.c_void_p),
                ("status", C.c_void_p)]


TEB_FLEET_MAX_ROWS = 32
# TEBGPU_FLEET_SEARCH_*: tebgpu_set_fleet_search's modes, and tebgpu_get_info key 19's values (-1 before the first step)
(TEBGPU_FLEET_SEARCH_AUTO, TEBGPU_FLEET_SEARCH_ALL_PAIRS, TEBGPU_FLEET_SEARCH_GRID,
 TEBGPU_FLEET_SEARCH_ONE_BUCKET) = range(4)
TEBGPU_INFO_FLEET_GRID, TEBGPU_INFO_FLEET_SEARCH = 18, 19
# the automatic search takes the grid from this many candidates on (FLEET_GRID_N0 in csrc/teb_cabi.cu) ...
FLEET_GRID_N0 = 4096
# ... when range is above the cell side's floor and range * range is finite (csrc/teb_fleet.cuh)
FLEET_H_MARGIN, FLEET_H_FLOOR, FLEET_CELL_BOUND = 1.0 + 2.0 ** -16, 2.0 ** -500, 2.0 ** 24
# TEB_FLEET_*: what tebgpu_fleet_obstacles did for a robot
TEB_FLEET_WRITTEN, TEB_FLEET_TRUNCATED, TEB_FLEET_BAD_INPUT, TEB_FLEET_SHARED_SCENE = range(4)


def make_fleet_args(R, S, C_cap, max_rows, range, **arrays) -> TebFleetArgs:
    """TebFleetArgs with the sizes set and the arrays given by keyword (pose=..., last_cmd=..., ...) as addresses (ints),
    torch tensors (their data_ptr()), numpy arrays (their buffer; keep them alive) or None for NULL"""
    a = TebFleetArgs()
    a.R, a.S, a.C_cap, a.max_rows, a.range = int(R), int(S), int(C_cap), int(max_rows), float(range)
    names = {f[0] for f in TebFleetArgs._fields_[5:]}
    for k, v in arrays.items():
        if k not in names:
            raise TypeError(f"unknown TebFleetArgs array {k}")
        if hasattr(v, "data_ptr"):
            v = v.data_ptr()
        elif isinstance(v, np.ndarray):
            v = ptr(v)
        setattr(a, k, v)
    return a


# TebFleetRow: one robot of a fleet table as it is published (include/teb_b200.h), 64 bytes
FLEET_ROW_DTYPE = np.dtype([("x", "f8"), ("y", "f8"), ("vx", "f8"), ("vy", "f8"), ("radius", "f8"), ("world", "i4"),
                            ("dynamic", "i4"), ("live", "i4"), ("_pad", "i4", (3,))])
assert FLEET_ROW_DTYPE.itemsize == 64


class TebFleetTable(C.Structure):
    """The fleet table of tebgpu_fleet_publish / _gather / _obstacles_table: T rows (FLEET_ROW_DTYPE), this call's robots
    at rows first .. first + R - 1, as a host or device pointer"""
    _fields_ = [("T", _i), ("first", _i), ("rows", C.c_void_p)]


def make_fleet_table(T, first, rows) -> TebFleetTable:
    """TebFleetTable of T rows with the call's robots from row `first`; rows: an address (int), a torch tensor (its
    data_ptr()), a numpy array (its buffer; keep it alive) or None for NULL"""
    t = TebFleetTable()
    t.T, t.first = int(T), int(first)
    if hasattr(rows, "data_ptr"):
        rows = rows.data_ptr()
    elif isinstance(rows, np.ndarray):
        rows = ptr(rows)
    t.rows = rows
    return t


class TebGpuLimits(C.Structure):
    _fields_ = [("max_bands", _i), ("max_poses", _i), ("max_scenes", _i), ("max_obstacles", _i),
                ("max_viapoints", _i), ("max_obst_vertices", _i)]


def default_params() -> TebParams:
    """TebConfig() constructor defaults (reference include/teb_local_planner/teb_config.h:245-390).

    Kept in Python as well so host-side tests do not need the CUDA library; the C-ABI's
    tebgpu_default_params() must return the same values (tests compare them).
    """
    p = TebParams()
    p.dt_ref, p.dt_hysteresis = 0.3, 0.1
    p.force_reinit_new_goal_dist, p.force_reinit_new_goal_angular = 1.0, 0.5 * np.pi
    p.teb_autosize, p.min_samples, p.max_samples, p.exact_arc_length = 1, 3, 500, 0
    p.via_points_ordered, p.allow_init_with_backwards_motion, p.global_plan_overwrite_orientation = 0, 0, 1
    p.max_vel_x, p.max_vel_x_backwards, p.max_vel_y, p.max_vel_trans, p.max_vel_theta = 0.4, 0.2, 0.0, 0.0, 0.3
    p.acc_lim_x, p.acc_lim_y, p.acc_lim_theta, p.min_turning_radius = 0.5, 0.5, 0.5, 0.0
    p.footprint_type = TEB_FOOTPRINT_POINT
    p.min_obstacle_dist, p.inflation_dist, p.dynamic_obstacle_inflation_dist = 0.5, 0.6, 0.6
    p.obstacle_association_force_inclusion_factor, p.obstacle_association_cutoff_factor = 1.5, 5.0
    p.obstacle_proximity_ratio_max_vel, p.obstacle_proximity_lower_bound, p.obstacle_proximity_upper_bound = 1.0, 0.0, 0.5
    p.include_dynamic_obstacles, p.legacy_obstacle_association, p.obstacle_poses_affected = 1, 0, 25
    p.penalty_epsilon = 0.05
    p.weight_max_vel_x, p.weight_max_vel_y, p.weight_max_vel_theta = 2.0, 2.0, 1.0
    p.weight_acc_lim_x, p.weight_acc_lim_y, p.weight_acc_lim_theta = 1.0, 1.0, 1.0
    p.weight_kinematics_nh, p.weight_kinematics_forward_drive, p.weight_kinematics_turning_radius = 1000.0, 1.0, 1.0
    p.weight_optimaltime, p.weight_shortest_path = 1.0, 0.0
    p.weight_obstacle, p.weight_inflation = 50.0, 0.1
    p.weight_dynamic_obstacle, p.weight_dynamic_obstacle_inflation = 50.0, 0.1
    p.weight_velocity_obstacle_ratio, p.weight_viapoint, p.weight_prefer_rotdir = 0.0, 1.0, 50.0
    p.weight_adapt_factor, p.obstacle_cost_exponent = 2.0, 1.0
    p.no_inner_iterations, p.no_outer_iterations, p.optimization_activate = 5, 4, 1
    p.selection_cost_hysteresis, p.selection_prefer_initial_plan = 1.0, 0.95
    p.selection_obst_cost_scale, p.selection_viapoint_cost_scale = 100.0, 1.0
    p.selection_alternative_time_cost, p.enable_multithreading = 0, 1
    p.h_signature_prescaler, p.h_signature_threshold = 1.0, 0.1
    p.divergence_detection_enable, p.divergence_detection_max_chi_squared = 0, 10.0
    return p


def ptr(a):
    """Address of a numpy array (or None), as c_void_p value."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data


class HostBatch:
    """Owns the numpy arrays behind a host TebBatch (keeps them alive while the struct is in use)."""

    def __init__(self, poses, n, obstacles, obst_count, scene_id=None, via=None, via_count=None,
                 vel_start=None, vel_goal=None, prefer_rotdir=None, obst_vertices=None):
        self.poses = np.ascontiguousarray(poses, dtype=np.float64)
        B, n_cap, four = self.poses.shape
        assert four == 4
        self.n = np.ascontiguousarray(n, dtype=np.int32)
        self.obstacles = np.ascontiguousarray(obstacles, dtype=OBST_DTYPE)
        if self.obstacles.ndim == 1:
            self.obstacles = self.obstacles[None, :]
        S, M_cap = self.obstacles.shape
        self.obst_count = np.ascontiguousarray(obst_count, dtype=np.int32).reshape(S)
        # vertex pool of the Line / Pill / Polygon obstacles: [S][PV_cap][2]
        if obst_vertices is None:
            self.obst_vertices = np.zeros((S, 0, 2), np.float64)
        else:
            self.obst_vertices = np.ascontiguousarray(obst_vertices, dtype=np.float64)
            if self.obst_vertices.ndim == 2:
                self.obst_vertices = self.obst_vertices[None]
        assert self.obst_vertices.shape[0] == S and self.obst_vertices.shape[2] == 2
        self.PV_cap = self.obst_vertices.shape[1]
        self.scene_id = (np.zeros(B, np.int32) if scene_id is None
                         else np.ascontiguousarray(scene_id, dtype=np.int32))
        if via is None:
            self.via = np.zeros((B, 0, 2), np.float64)
            self.via_count = np.zeros(B, np.int32)
        else:
            self.via = np.ascontiguousarray(via, dtype=np.float64)
            self.via_count = np.ascontiguousarray(via_count, dtype=np.int32)
        V_cap = self.via.shape[1]
        z = np.zeros((B, 4), np.float64)
        z[:, 3] = 1.0  # vel_start_.first = vel_goal_.first = true (optimal_planner.cpp:94-102)
        self.vel_start = z.copy() if vel_start is None else np.ascontiguousarray(vel_start, dtype=np.float64)
        self.vel_goal = z.copy() if vel_goal is None else np.ascontiguousarray(vel_goal, dtype=np.float64)
        self.prefer_rotdir = (np.zeros(B, np.int32) if prefer_rotdir is None
                              else np.ascontiguousarray(prefer_rotdir, dtype=np.int32))
        self.cost = np.full(B, np.inf)
        self.chi2 = np.zeros(B)
        self.status = np.zeros(B, np.int32)
        self.lm_iters = np.zeros(B, np.int32)
        self.B, self.n_cap, self.S, self.M_cap, self.V_cap = B, n_cap, S, M_cap, V_cap

    def struct(self) -> TebBatch:
        b = TebBatch()
        b.B, b.n_cap, b.S, b.M_cap, b.V_cap = self.B, self.n_cap, self.S, self.M_cap, self.V_cap
        b.poses, b.n, b.scene_id = ptr(self.poses), ptr(self.n), ptr(self.scene_id)
        b.obstacles, b.obst_count = ptr(self.obstacles), ptr(self.obst_count)
        b.PV_cap = self.PV_cap
        b.obst_vertices = ptr(self.obst_vertices) if self.PV_cap > 0 else None
        b.via = ptr(self.via) if self.V_cap > 0 else None
        b.via_count = ptr(self.via_count)
        b.vel_start, b.vel_goal, b.prefer_rotdir = ptr(self.vel_start), ptr(self.vel_goal), ptr(self.prefer_rotdir)
        b.cost, b.chi2, b.status, b.lm_iters = ptr(self.cost), ptr(self.chi2), ptr(self.status), ptr(self.lm_iters)
        return b

    def copy(self):
        h = HostBatch(self.poses.copy(), self.n.copy(), self.obstacles.copy(), self.obst_count.copy(),
                      self.scene_id.copy(), self.via.copy() if self.V_cap > 0 else None,
                      self.via_count.copy() if self.V_cap > 0 else None,
                      self.vel_start.copy(), self.vel_goal.copy(), self.prefer_rotdir.copy(),
                      self.obst_vertices.copy() if self.PV_cap > 0 else None)
        return h


def make_args(inner=5, outer=4, compute_cost=True, obst_scale=1.0, via_scale=1.0, alt_time=False) -> TebOptimizeArgs:
    a = TebOptimizeArgs()
    a.iterations_innerloop, a.iterations_outerloop = inner, outer
    a.compute_cost_afterwards, a.alternative_time_cost = int(compute_cost), int(alt_time)
    a.obst_cost_scale, a.viapoint_cost_scale = obst_scale, via_scale
    return a
