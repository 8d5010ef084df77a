/*
 * teb_b200.h — C-ABI of the H100-native Timed-Elastic-Band optimizer.
 *
 * This is the drop-in boundary for the hot path of rst-tu-dortmund/teb_local_planner:
 *   TebOptimalPlanner::optimizeTEB            src/optimal_planner.cpp:182-231
 *   TebOptimalPlanner::buildGraph/optimizeGraph/computeCurrentCost
 *                                             src/optimal_planner.cpp:323-366, 368-402, 1041-1094
 *   g2o SparseOptimizer + LM + CSparse        call sites src/optimal_planner.cpp:161-179, 385-387
 *   HomotopyClassPlanner::optimizeAllTEBs     src/homotopy_class_planner.cpp:466-493
 *   HomotopyClassPlanner::selectBestTeb       src/homotopy_class_planner.cpp:564-667
 *   TimedElasticBand::autoResize              src/timed_elastic_band.cpp:227-286
 *   HomotopyClassPlanner::calculateEquivalenceClass (HSignature / HSignature3d)
 *                                             include/teb_local_planner/homotopy_class_planner.hpp:46-63, h_signature.h
 *
 * Plain C, plain pointers and sizes, no torch / CUDA types in any signature.
 * All state is fp64 (the reference is fp64 throughout).
 *
 * Band storage ("pose records"): one band = n_cap records of 4 doubles
 *   rec[i] = { x_i, y_i, theta_i, dt_i }      dt_i = TimeDiff(i) connects pose i -> i+1
 * the last valid record (i = n-1) carries dt = 0.  Pose 0 and pose n-1 are fixed
 * during optimisation (timed_elastic_band.cpp:330,377), every dt is free.
 */
#ifndef TEB_B200_H
#define TEB_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TEBGPU_OK                  0
#define TEBGPU_ERR_INVALID_ARG    -1
#define TEBGPU_ERR_CUDA           -2
#define TEBGPU_ERR_UNSUPPORTED    -3   /* an option outside what the kernels cover (e.g. unknown footprint model): fail loudly */
#define TEBGPU_ERR_CAPACITY       -4
#define TEBGPU_ERR_NO_DEVICE      -5

/* per-band status bits written to status[] */
#define TEB_STATUS_OPTIMIZED       1   /* optimizeTEB returned true (optimal_planner.cpp:230): every outer iteration
                                          optimised the band, or iterations_outerloop == 0 (cost stays HUGE_VAL). Never
                                          with iterations_innerloop == 0 and iterations_outerloop > 0: optimizeGraph
                                          fails when optimize() runs no iteration (:393), so only the first outer
                                          iteration's autoResize / buildGraph run */
#define TEB_STATUS_TOO_FEW_POSES   2   /* sizePoses < min_samples guard (optimal_planner.cpp:377)   */
#define TEB_STATUS_CHOL_FAILED     4   /* at least one trial factorisation hit a non-positive pivot */
#define TEB_STATUS_NONFINITE       8   /* non-finite chi2 / lambda encountered                      */
#define TEB_STATUS_TERMINATED     16   /* LM returned Terminate in the last optimizeGraph call      */
#define TEB_STATUS_DISABLED       32   /* optimization_activate == false / max_vel_x < 0.01          */
#define TEB_STATUS_CAPACITY       64   /* autoResize needed more than n_cap poses: band left unoptimised */
#define TEB_STATUS_BAD_INPUT     128   /* the band's scene holds an obstacle row the batch cannot describe (vertex range
                                          outside obst_vertices, unknown type): band left unoptimised */

/* robot_footprint_model.h: PointRobotFootprint :131, CircularRobotFootprint :205, TwoCirclesRobotFootprint :303,
 * LineRobotFootprint :439, PolygonRobotFootprint :635 */
enum { TEB_FOOTPRINT_POINT = 0, TEB_FOOTPRINT_CIRCULAR = 1, TEB_FOOTPRINT_TWO_CIRCLES = 2, TEB_FOOTPRINT_LINE = 3,
       TEB_FOOTPRINT_POLYGON = 4 };
/* obstacles.h: PointObstacle :305, CircularObstacle :447, LineObstacle :597, PillObstacle :746, PolygonObstacle :893 */
enum { TEB_OBST_POINT = 0, TEB_OBST_CIRCULAR = 1, TEB_OBST_LINE = 2, TEB_OBST_PILL = 3, TEB_OBST_POLYGON = 4 };
#define TEB_MAX_FOOTPRINT_VERTICES 16
enum { TEB_ROTDIR_NONE = 0, TEB_ROTDIR_LEFT = 1, TEB_ROTDIR_RIGHT = 2 };

/* POD mirror of the TebConfig fields read on the hot path
 * (include/teb_local_planner/teb_config.h:72-229, defaults :245-390). */
typedef struct TebParams {
  /* trajectory */
  double  dt_ref;
  double  dt_hysteresis;
  double  force_reinit_new_goal_dist;
  double  force_reinit_new_goal_angular;
  int32_t teb_autosize;
  int32_t min_samples;
  int32_t max_samples;
  int32_t exact_arc_length;
  int32_t via_points_ordered;
  int32_t allow_init_with_backwards_motion;
  int32_t global_plan_overwrite_orientation;
  int32_t _pad0;
  /* robot */
  double  max_vel_x;
  double  max_vel_x_backwards;
  double  max_vel_y;
  double  max_vel_trans;
  double  max_vel_theta;
  double  acc_lim_x;
  double  acc_lim_y;
  double  acc_lim_theta;
  double  min_turning_radius;
  /* footprint model (robot_footprint_model.h) */
  double  footprint_radius;        /* circular  */
  double  footprint_front_offset;  /* two circles */
  double  footprint_front_radius;
  double  footprint_rear_offset;
  double  footprint_rear_radius;
  int32_t footprint_type;
  int32_t footprint_vertex_count;  /* polygon: 1 .. TEB_MAX_FOOTPRINT_VERTICES (robot frame, not closed) */
  double  footprint_line[4];       /* line: start x, y, end x, y in the robot frame (robot_footprint_model.h:439) */
  double  footprint_vertices[2 * TEB_MAX_FOOTPRINT_VERTICES]; /* polygon: x0, y0, x1, y1, ... (:635) */
  /* obstacles */
  double  min_obstacle_dist;
  double  inflation_dist;
  double  dynamic_obstacle_inflation_dist;
  double  obstacle_association_force_inclusion_factor;
  double  obstacle_association_cutoff_factor;
  double  obstacle_proximity_ratio_max_vel;
  double  obstacle_proximity_lower_bound;
  double  obstacle_proximity_upper_bound;
  int32_t include_dynamic_obstacles;
  int32_t legacy_obstacle_association;
  int32_t obstacle_poses_affected;
  int32_t _pad2;
  /* optim */
  double  penalty_epsilon;
  double  weight_max_vel_x;
  double  weight_max_vel_y;
  double  weight_max_vel_theta;
  double  weight_acc_lim_x;
  double  weight_acc_lim_y;
  double  weight_acc_lim_theta;
  double  weight_kinematics_nh;
  double  weight_kinematics_forward_drive;
  double  weight_kinematics_turning_radius;
  double  weight_optimaltime;
  double  weight_shortest_path;
  double  weight_obstacle;
  double  weight_inflation;
  double  weight_dynamic_obstacle;
  double  weight_dynamic_obstacle_inflation;
  double  weight_velocity_obstacle_ratio;
  double  weight_viapoint;
  double  weight_prefer_rotdir;
  double  weight_adapt_factor;
  double  obstacle_cost_exponent;
  int32_t no_inner_iterations;
  int32_t no_outer_iterations;
  int32_t optimization_activate;
  int32_t _pad3;
  /* hcp (selection only) */
  double  selection_cost_hysteresis;
  double  selection_prefer_initial_plan;
  double  selection_obst_cost_scale;
  double  selection_viapoint_cost_scale;
  int32_t selection_alternative_time_cost;
  int32_t enable_multithreading;
  double  h_signature_prescaler;   /* teb_config.h:201, default 1   */
  double  h_signature_threshold;   /* teb_config.h:202, default 0.1 */
  /* recovery */
  int32_t divergence_detection_enable;
  int32_t _pad4;
  double  divergence_detection_max_chi_squared;
} TebParams;

/* Obstacle table row (64 bytes), constant-velocity model (obstacles.h:190-206).
 * Point / Circular (obstacles.h:305-445, :447-595): (x, y) is the position, radius the circle radius.
 * Line / Pill / Polygon (:597-740, :746-890, :893-1045): the shape is the vertex list
 * obst_vertices[scene][vertex_begin .. vertex_begin + vertex_count) (2 vertices for Line / Pill; a polygon is closed
 * implicitly when it has more than 2 vertices, distance_calculations.h:172-199), radius is the pill radius and (x, y)
 * must hold getCentroid() (line midpoint :734; polygon centroid obstacles.cpp:47-97) — the obstacle association uses
 * it to tell left from right (optimal_planner.cpp:503). */
typedef struct TebObstacle {
  double  x, y;          /* position / centroid */
  double  vx, vy;        /* centroid velocity (obstacles.h:206) */
  double  radius;        /* Circular, Pill; 0 otherwise */
  int32_t dynamic;       /* isDynamic() (obstacles.h:199) */
  int32_t type;          /* TEB_OBST_* */
  int32_t vertex_begin;  /* Line / Pill / Polygon: first vertex in the scene's vertex pool */
  int32_t vertex_count;
  double  _pad;
} TebObstacle;

/* A batch of bands (homotopy candidates x planning requests). All pointers are HOST pointers for
 * tebgpu_optimize_batch and DEVICE pointers for tebgpu_optimize_batch_device. */
typedef struct TebBatch {
  int32_t B;          /* number of bands                                   */
  int32_t n_cap;      /* records per band (stride); >= every n[b]           */
  int32_t S;          /* number of scenes (obstacle tables)                 */
  int32_t M_cap;      /* obstacle rows per scene (stride)                   */
  int32_t V_cap;      /* via-points per band (stride); may be 0             */
  int32_t PV_cap;     /* obstacle vertices per scene (stride); 0 <=> only Point / Circular obstacles */
  double*            poses;       /* [B][n_cap][4]  in/out                              */
  int32_t*           n;           /* [B]            in/out (autoResize changes it)      */
  const int32_t*     scene_id;    /* [B]                                                */
  const TebObstacle* obstacles;   /* [S][M_cap]                                         */
  const int32_t*     obst_count;  /* [S]                                                */
  const double*      obst_vertices; /* [S][PV_cap][2] vertex pool of the Line / Pill / Polygon obstacles, or NULL   */
  const double*      via;         /* [B][V_cap][2] or NULL                              */
  const int32_t*     via_count;   /* [B] or NULL                                        */
  const double*      vel_start;   /* [B][4] = vx, vy, omega, active(0/1)  (optimal_planner.cpp:233-245) */
  const double*      vel_goal;    /* [B][4] = vx, vy, omega, active(0/1); active=0 <=> free_goal_vel     */
  const int32_t*     prefer_rotdir; /* [B] TEB_ROTDIR_* or NULL (optimal_planner.cpp:961-997)           */
  double*            cost;        /* [B] out: getCurrentCost() (optimal_planner.h:437)  */
  double*            chi2;        /* [B] out: chi2 of the final state of the last LM iteration (hasDiverged) */
  int32_t*           status;      /* [B] out: TEB_STATUS_* bits                          */
  int32_t*           lm_iters;    /* [B] out: inner LM iterations executed (all outer iterations) */
} TebBatch;

/* Arguments of TebOptimalPlanner::optimizeTEB (optimal_planner.h:231). */
typedef struct TebOptimizeArgs {
  int32_t iterations_innerloop;
  int32_t iterations_outerloop;
  int32_t compute_cost_afterwards;
  int32_t alternative_time_cost;
  double  obst_cost_scale;
  double  viapoint_cost_scale;
} TebOptimizeArgs;

typedef struct TebGpuLimits {
  int32_t max_bands;      /* B capacity */
  int32_t max_poses;      /* n_cap capacity (<= 512) */
  int32_t max_scenes;
  int32_t max_obstacles;  /* M_cap capacity, <= 16384. Batches of M_cap <= 1024 stage the scene's table in shared memory;
                             1025 .. 16384 read it from global memory (L2), chosen per call. The association buffers
                             take B x n_cap x (2 MW + ceil(MW / 64)) x 8 bytes of device memory, MW = ceil(max_obstacles / 64)
                             (16384 obstacles: 4.1 KB per pose). Beyond 1024 obstacles solvers 0 / 1, kernel-A variant 1,
                             TEBGPU_EVAL_V1 and tebgpu_h_signature return TEBGPU_ERR_UNSUPPORTED. */
  int32_t max_viapoints;  /* V_cap capacity */
  int32_t max_obst_vertices; /* PV_cap capacity (0: Point / Circular obstacles only) */
} TebGpuLimits;

typedef struct tebgpu_ctx tebgpu_ctx;

/* Fill `p` with the TebConfig() constructor defaults (teb_config.h:245-390). The three fields the
 * reference leaves uninitialised in the ctor get their dynamic_reconfigure defaults
 * (divergence_detection_enable=0, divergence_detection_max_chi_squared=10). */
void tebgpu_default_params(TebParams* p);

/* Per-band inputs and outputs of TebOptimalPlanner::plan followed by getVelocityCommand (tebgpu_plan_batch). HOST
 * pointers for tebgpu_plan_batch, DEVICE pointers for tebgpu_plan_batch_device, like the TebBatch they go with. */
typedef struct TebPlanInput {
  const double*  start;          /* [B][3] x, y, theta: plan(start, goal, ...) (optimal_planner.cpp:290); unused with a plan */
  const double*  goal;           /* [B][3] */
  const double*  initial_plan;   /* [B][P_cap][3] x, y, yaw, or NULL: plan(initial_plan, ...) (:247); start and goal are
                                    then the plan's first and last point (:257-258) */
  const int32_t* plan_count;     /* [B] points of each band's plan, 1 .. P_cap, or NULL: P_cap points each */
  int32_t        P_cap;          /* plan rows per band (stride) */
  int32_t        look_ahead_poses;                   /* getVelocityCommand argument (control_look_ahead_poses) */
  int32_t        prevent_look_ahead_poses_near_goal; /* trajectory.prevent_look_ahead_poses_near_goal (:1145) */
  int32_t        _pad;
  double*        cmd;            /* [B][4] out: vx, vy, omega, ok (getVelocityCommand's return value, 1 / 0) */
  int32_t*       path;           /* [B] out or NULL: TEB_PLAN_PATH_* */
} TebPlanInput;
#define TEB_PLAN_PATH_NONE  -1   /* band left as it was: TEB_STATUS_BAD_INPUT or TEB_STATUS_CAPACITY */
#define TEB_PLAN_PATH_COLD   0   /* n == 0 (!teb_.isInit()): initTrajectoryToGoal */
#define TEB_PLAN_PATH_WARM   1   /* goal moved < force_reinit_new_goal_dist and turned < _angular: updateAndPruneTEB */
#define TEB_PLAN_PATH_REINIT 2   /* otherwise: clearTimedElasticBand + initTrajectoryToGoal */

/* Arguments and outputs of TebOptimalPlanner::isTrajectoryFeasible (optimal_planner.cpp:1250-1310) for every band of a
 * batch (tebgpu_check_feasible). HOST output pointers for tebgpu_check_feasible, DEVICE pointers for
 * tebgpu_check_feasible_device.
 *
 * World model of tebgpu_check_feasible, which differs from the reference. The reference asks
 * base_local_planner::CostmapModel::footprintCost of the costmap, which tebgpu_check_feasible_costmap does (see
 * TebCostmapWorld, with the same arguments and outputs); here footprintCost(x, y, theta) == -1 means: the context's footprint model (TebParams.footprint_type and
 * its geometry) placed at (x, y, theta) has a distance <= collision_distance to some obstacle of the band's scene. The
 * distance is the optimizer's own footprint-to-obstacle distance (the one the obstacle edges use); all obst_count rows of
 * the scene are tested, not the association; dynamic obstacles at their current position (a snapshot, no time
 * prediction). With collision_distance = 0, contact, overlap and containment (distance exactly 0) are collisions. It does
 * not rasterise the footprint outline over costmap cells and has no inscribed-cost band. A query whose distances are all
 * > collision_distance except for some NaN ones is undecidable. */
typedef struct TebFeasibilityArgs {
  int32_t  look_ahead_idx;      /* feasibility_check_no_poses; < 0 or >= n: the whole band */
  int32_t  max_queries;         /* footprint queries tested (and stored) per band, >= 1 */
  double   lookahead_distance;  /* feasibility_check_lookahead_distance; <= 0: off */
  double   inscribed_radius;    /* the interpolation step between poses, > 0 and finite */
  double   angular_resolution;  /* trajectory.min_resolution_collision_check_angular, > 0 and finite */
  double   collision_distance;  /* >= 0 and finite */
  int32_t* feasible;            /* [B] out: 1 feasible, 0 a query collides, -1 undecidable (see tebgpu_check_feasible) */
  int32_t* query_count;         /* [B] out: footprint queries the reference makes */
  double*  queries;             /* [B][max_queries][3] out or NULL: the first min(query_count, max_queries) query poses */
} TebFeasibilityArgs;

/* The costmap world model of tebgpu_check_feasible_costmap(_device): the reference's own check,
 * base_local_planner::CostmapModel::footprintCost on each scene's local costmap. base_local_planner and costmap_2d are
 * not part of the reference checkout; this definition restates navigation's ROS Noetic code (costmap_model.cpp,
 * line_iterator.h, world_model.h, Costmap2D::worldToMap). HOST pointers for tebgpu_check_feasible_costmap, DEVICE pointers
 * for tebgpu_check_feasible_costmap_device, except footprint, which is always a host array copied into the launch.
 *
 * Scene s's raster is TebCostmapArgs' layout: cost[s][my * sx + mx], (sx, sy) = grid[s], (ox, oy, r) = origin[s]; band b
 * reads scene scene_id[b], so the rasters uploaded for tebgpu_costmap_obstacles_device feed this check unchanged. The
 * queries, their order, the look-ahead rule and max_queries are tebgpu_check_feasible's (TebFeasibilityArgs; its
 * collision_distance is not read). footprintCost(x, y, theta) with F = footprint_count points (robot frame):
 *   vertices  c = cos theta, s = sin theta once per query; vertex k = (x + (fx c - fy s), y + (fx s + fy c)), every
 *             product and sum rounded on its own (no FMA contraction).
 *   worldToMap(wx, wy)  off the map when wx < ox or wy < oy; otherwise mx = (int)((wx - ox) / r), my likewise
 *             (truncation), on the map when mx < sx and my < sy. A quotient past the int range is off the map.
 *   1. the centre (x, y) off the map: -3.
 *   2. F < 3: the centre cell alone: 255 (NO_INFORMATION) -2, 254 (LETHAL) or 253 (INSCRIBED_INFLATED) -1, otherwise
 *      its cost.
 *   3. F >= 3: the outline only, never the interior. Edges 0 -> 1, ..., F - 2 -> F - 1, then F - 1 -> 0: an endpoint
 *      off the map gives -3; otherwise the cells of the integer Bresenham walk (LineIterator) from the start vertex's
 *      cell to the end vertex's, both included, in walk order: 255 -2, 254 -1, otherwise the cost (253 is not
 *      negative here). The first negative value met is returned at once.
 *   4. otherwise the largest cost seen (0 for none).
 * LineIterator: dx = |x1 - x0|, dy = |y1 - y0|, the increments by sign (x1 >= x0 gives +1). x is the major axis when
 * dx >= dy: den = dx, num = dx / 2 (integer), numadd = dy, numpixels = dx (y the same with x and y swapped). advance:
 * num += numadd; if num >= den { num -= den; step the minor axis }; step the major axis. Cells 0 .. numpixels.
 * Verdict: the first query whose footprintCost is exactly -1 makes the band infeasible (feasible 0, query_count its
 * index + 1). -2 and -3 are free, as in the reference, so a -2 met earlier on an outline hides a later 254.
 *
 * Defined here where the reference is not: a non-finite pose among the checked ones gives feasible -1 and no query (as
 * tebgpu_check_feasible); more than max_queries queries, the first max_queries free: -1 and the full count (as there).
 * The device entry point answers a band with feasible -1 and query_count 0 when its n or scene_id is out of range, or
 * its scene has sx or sy < 1, sx * sy > cell_cap, a non-finite or non-positive resolution or a non-finite origin; the
 * host entry point refuses the same inputs with TEBGPU_ERR_INVALID_ARG. A caller who wants -2 / -3 to count as
 * collisions reads query_cost. */
#define TEB_COSTMAP_FOOTPRINT_MAX  64
#define TEB_COSTMAP_INSCRIBED      253   /* costmap_2d::INSCRIBED_INFLATED_OBSTACLE */
#define TEB_COSTMAP_LETHAL         254   /* costmap_2d::LETHAL_OBSTACLE */
#define TEB_COSTMAP_NO_INFORMATION 255   /* costmap_2d::NO_INFORMATION */
typedef struct TebCostmapWorld {
  int32_t        cell_cap;        /* raster bytes per scene (stride of cost), >= 1 */
  int32_t        footprint_count; /* F, 0 .. TEB_COSTMAP_FOOTPRINT_MAX */
  const uint8_t* cost;            /* [S][cell_cap] */
  const int32_t* grid;            /* [S][2] sx, sy */
  const double*  origin;          /* [S][3] ox, oy, r */
  const double*  footprint;       /* [F][2] HOST (both entry points), finite: footprint_spec_ in the robot frame */
  double*        query_cost;      /* [B][max_queries] out or NULL: footprintCost of each query tested, the rows
                                     TebFeasibilityArgs.queries gets; the rows behind them are not written */
} TebCostmapWorld;

/* Which bands tebgpu_read_trajectory reads out, and its outputs: TebOptimalPlanner::getVelocityProfile
 * (optimal_planner.cpp:1170-1188) and getFullTrajectory (:1190-1248) of every band read out. HOST pointers for
 * tebgpu_read_trajectory, DEVICE pointers for tebgpu_read_trajectory_device. R is the number of rows read out: count
 * when bands != NULL, B otherwise. Output row r holds band bands[r] (or r).
 *
 * Segment k (1 <= k <= n - 1) is extractVelocity(Pose(k - 1), Pose(k), TimeDiff(k - 1)) with the context's max_vel_y
 * (0: non-holonomic, vx signed by the step's projection on pose k - 1's heading, sign(0) = 0, vy = 0); TimeDiff == 0
 * gives a zero twist. Definitions:
 *   Boundary rows: (vx, vy, omega) of vel_start[b] / vel_goal[b] as stored, whatever their active flag. The reference
 *     reports vel_start_.second / vel_goal_.second and ignores .first (setVelocityGoalFree only clears .first,
 *     optimal_planner.h:260).
 *   Profile, n + 1 rows: the start velocity, segments 1 .. n - 1, the goal velocity. n = 0: one row, the goal velocity
 *     (the reference resizes to 1, and back() overwrites front()).
 *   Trajectory, n rows: pose i; velocity: the start velocity for i = 0, the goal velocity for i = n - 1 >= 1,
 *     otherwise 0.5 * (segment i + segment i + 1); time_from_start: TimeDiff(0) + ... + TimeDiff(i - 1), summed in
 *     that order from 0. n = 0: no row. n = 1: pose 0, the start velocity, t = 0 (the reference reads TimeDiff(0),
 *     which does not exist there; its answer is undefined).
 *   theta: the band's stored yaw. Formatting it as the message's quaternion is left to the caller. */
typedef struct TebTrajectoryArgs {
  const int32_t* bands;      /* [count] band indices, in output order (repeats and any order allowed), or NULL: all B bands */
  int32_t        count;      /* rows read out when bands != NULL (>= 0); ignored when bands == NULL */
  int32_t        _pad;
  double*        profile;    /* [R][n_cap + 1][3] out or NULL: vx, vy, omega */
  double*        trajectory; /* [R][n_cap][7] out or NULL: x, y, theta, vx, vy, omega, time_from_start */
  int32_t*       points;     /* [R] out: n of the band read out; -1 for a row the device entry point could not read (a band
                                index outside 0 .. B - 1 or n outside 0 .. n_cap). Rows past n + 1 (profile) and n
                                (trajectory) are not written. */
} TebTrajectoryArgs;

/* Each scene's obstacle table built from its local costmap (tebgpu_costmap_obstacles): the branch of
 * TebLocalPlannerROS::updateObstacleContainerWithCostmap without a costmap_converter plugin, the reference's default
 * (teb_local_planner_ros.cpp:343-352, :478-504), followed by the custom obstacles (:552-625). HOST pointers for
 * tebgpu_costmap_obstacles, DEVICE pointers for tebgpu_costmap_obstacles_device.
 *
 * Inputs of scene s: the costmap's size (sx, sy) = grid[s] in cells, its origin (ox, oy) and resolution r = origin[s],
 * the robot pose (rx, ry, rt) = robot[s] in the costmap's global frame (robot_pose_), and the char map
 * cost[s][my * sx + mx], costmap_2d's getCharMap() as it is (getCost(mx, my) reads my * size_x + mx). The rows, in order:
 *   1. If include_costmap_obstacles != 0, for i = 0 .. sx - 2 (outer) and j = 0 .. sy - 2 (inner): the last column and
 *      the last row are never visited (the reference's < getSizeInCellsX() - 1); sx < 2 or sy < 2 gives no row (at 0 the
 *      reference's unsigned size - 1 wraps around). A cell with cost == 254 (LETHAL_OBSTACLE exactly; 253 and 255 do
 *      not count) has the centre wx = ox + (i + 0.5) * r, wy = oy + (j + 0.5) * r (costmap_2d mapToWorld). With
 *      dx = wx - rx, dy = wy - ry, c = cos(rt), s = sin(rt) (pose_se2.h:215) it is skipped when
 *      dx * c + dy * s < 0 && sqrt(dx * dx + dy * dy) > behind_robot_dist (a NaN anywhere keeps it, as in the reference),
 *      otherwise it gives the row {wx, wy, 0, 0, 0, dynamic 0, TEB_OBST_POINT, 0, 0, _pad 0}: every byte is defined.
 *      Every product and sum is rounded on its own (no FMA contraction), as in the reference's x86 build.
 *   2. Then custom[s][0 .. custom_count[s]) verbatim (tebgpu_costmap_obstacles_tf moves them, see TebFrameArgs).
 *      Their vertex_begin refers to the batch's obst_vertices, which the caller fills; Point rows use no vertex, so nothing is rebased.
 *   3. needed[s] = the number of rows. If it is <= M_cap, obst_count[s] = needed[s]; otherwise the first M_cap rows are
 *      written and obst_count[s] = -1, which every consumer refuses (TEB_STATUS_BAD_INPUT from the optimize and plan
 *      entry points, -1 from the feasibility check, NaN from the device H-signature): no obstacle is dropped silently.
 *      Rows past obst_count (past M_cap on overflow) are not written. */
typedef struct TebCostmapArgs {
  int32_t  S;                  /* scenes, 1 .. max_scenes */
  int32_t  cell_cap;           /* raster bytes per scene (stride of cost), >= sx * sy; a multiple of 16 with a 16-byte
                                  aligned cost lets the device read the raster with 16-byte loads */
  int32_t  M_cap;              /* output rows per scene (stride of obstacles), 1 .. max_obstacles */
  int32_t  C_cap;              /* custom rows per scene (stride of custom), >= 0 */
  int32_t  include_costmap_obstacles; /* obstacles.include_costmap_obstacles (teb_config.h:133, default true) */
  int32_t  _pad;
  double   behind_robot_dist;  /* obstacles.costmap_obstacles_behind_robot_dist (teb_config.h:134, default 1.5) */
  const uint8_t*     cost;     /* [S][cell_cap] */
  const int32_t*     grid;     /* [S][2] sx, sy */
  const double*      origin;   /* [S][3] ox, oy, r */
  const double*      robot;    /* [S][3] rx, ry, rt */
  const TebObstacle* custom;   /* [S][C_cap] or NULL (C_cap == 0) */
  const int32_t*     custom_count; /* [S] or NULL: no custom rows */
  TebObstacle*       obstacles;    /* [S][M_cap] out, 16-byte aligned */
  int32_t*           obst_count;   /* [S] out */
  int32_t*           needed;       /* [S] out or NULL; saturates at INT32_MAX */
} TebCostmapArgs;

/* Each robot's global plan cut into its local plan, goal and via-points (tebgpu_local_plan): the front of
 * TebLocalPlannerROS::computeVelocityCommands from pruneGlobalPlan up to the start row (teb_local_planner_ros.cpp:268-340),
 * under the identity transform: the global plan is given in the frame of the costmap and of the obstacle tables
 * (tebgpu_local_plan_tf takes it in its own frame, see TebFrameArgs). HOST
 * pointers for tebgpu_local_plan, DEVICE pointers for tebgpu_local_plan_device. Of the batch only B, S and scene_id are
 * read. One output row per band b; plan / plan_count and via / via_count have the layout of TebPlanInput.initial_plan /
 * plan_count and TebBatch.via / via_count, so they feed tebgpu_plan_batch(_device) on the same stream.
 *
 * Band b's global plan is global_plan[b][plan_begin[b] .. plan_end[b]) (x, y, yaw); g[k] below is its row plan_begin + k
 * after step 1, n = plan_end - plan_begin its live rows. (rx, ry, rt) = robot[b]. Every product and sum is rounded on its
 * own (no FMA contraction), pow(d, 2) is d * d, and a NaN goes through every comparison as in the reference (false).
 *   1. Prune (:657-698): plan_begin moves to the first live row with dx * dx + dy * dy < prune_distance * prune_distance
 *      (dx = rx - x, dy = ry - y); none: nothing moves. No row is moved in memory.
 *   2. n == 0: result TEB_LOCAL_PLAN_EMPTY, plan_count = 0, nothing else is written (the reference reads
 *      global_plan[0] before its empty check).
 *   3. Transform (:701-822). The window is w * w with w = max((double)sx * r / 2.0, (double)sy * r / 2.0) * 0.85
 *      ((sx, sy) = grid[scene_id[b]], r = origin[scene_id[b]][2]; max(a, b) = a < b ? b : a). The closest row: from
 *      sq = 1e10, i = 0, over j = 0 .. n - 1: stop when some earlier row set sq < 0.05 and d_j > sq; take j (sq = d_j,
 *      i = j) when d_j < sq (strict), d_j the squared distance from the robot. Then rows are taken from i while i < n,
 *      the squared distance of the row taken last (at first the search's sq) is <= the window, and max_lookahead_dist
 *      <= 0 or plan_length <= max_lookahead_dist; taking row i > 0 adds distance_points2d(g[i - 1], g[i]) to
 *      plan_length (only when max_lookahead_dist > 0), in order, so the segment into the closest row counts. The row
 *      that first leaves the window is still taken. goal_idx = (one past the last row taken) - 1; when no row is taken
 *      the plan is the one row g[n - 1] and goal_idx = n - 1.
 *   4. Via-points (:627-646), when via != NULL, from the rows of step 3: none if viapoint_sep <= 0; otherwise rows 1 ..
 *      in order, each taken when distance_points2d(last via-point or row 0, row) < viapoint_sep is false.
 *   5. Goal reached (:290-304) when sqrt(dx * dx + dy * dy) < xy_goal_tolerance (dx = g[n - 1].x - rx, ...),
 *      |normalize_theta(teb_plan_yaw(g[n - 1].yaw) - rt)| < yaw_goal_tolerance, (!complete_global_plan || via count == 0)
 *      (via == NULL: via_count[b] as given, 0 for NULL) and (stopped || free_goal_vel), stopped =
 *      |omega| <= theta_stopped_vel && |vx| <= trans_stopped_vel && |vy| <= trans_stopped_vel of robot_vel[b]
 *      (base_local_planner::stopped). Result TEB_LOCAL_PLAN_GOAL_REACHED: the via-points and goal_idx are written,
 *      plan_count = 0, so a following tebgpu_plan_batch_device leaves the band as it was; the reference returns a zero
 *      command there, which is the caller's to apply.
 *   6. Horizon shrink (:950-977), when shrink_horizon_backup, infeasible_count or since_infeasible is given (NULL counts
 *      as 0 / inf), goal_idx < size - 1 (size: rows of step 3) and (count > 0 || since < shrink_horizon_min_duration):
 *      reduction = goal_idx / 2, halved again when count > 9; if size - reduction - 1 > 0 and goal_idx - reduction >= 0
 *      the rows from size - reduction - 1 on are dropped and goal_idx -= reduction. As in the reference, goal_idx indexes
 *      the global plan and size counts the rows taken from its closest row on, so goal_idx >= size - 1 and the shrink
 *      does not fire on a plan from step 3; it is kept so the inputs mean what they mean there.
 *   7. Goal heading (:318-333, :827-871) of the last row: its stored yaw when TebParams.global_plan_overwrite_orientation
 *      is 0 (read from the context). Otherwise, with n and goal_idx: goal_idx >= n - 1: teb_plan_yaw(its yaw);
 *      goal_idx > n - 5: teb_plan_yaw(g[n - 1].yaw); else atan2(sum sin, sum cos) (0 when both sums are 0; sums from 0,
 *      in order) of the min(3, n - goal_idx - 1) headings atan2(dy, dx) from the last row to g[goal_idx + 1], then
 *      g[goal_idx + 1] to g[goal_idx + 2], ...
 *   8. Start row (:335-340): a one-row plan gets a row in front of it; row 0 becomes (rx, ry, rt).
 *   9. Capacity: more than P_cap rows, or more than V_cap via-points (via != NULL): result TEB_LOCAL_PLAN_CAPACITY,
 *      plan_count = 0, goal_idx and needed written, no row and no via-point written. No goal is moved silently.
 * Otherwise result TEB_LOCAL_PLAN_PLANNED with plan_count rows, goal_idx after step 6 and the via-points. needed[b] =
 * (plan rows, via-points extracted) for every band that reached step 3 (plan rows 0 when the goal is reached). Rows past
 * plan_count and via_count are not written. tebgpu_local_plan_device answers a band whose plan_begin / plan_end is not
 * 0 <= plan_begin <= plan_end <= G_cap, or whose scene_id is outside 0 .. S - 1, with TEB_LOCAL_PLAN_BAD_INPUT and
 * plan_count = 0, and writes nothing else for it. */
typedef struct TebLocalPlanArgs {
  int32_t  G_cap;                /* global plan rows per band (stride of global_plan), >= 1 */
  int32_t  P_cap;                /* local plan rows per band (stride of plan), >= 2 */
  int32_t  V_cap;                /* via-points per band (stride of via), >= 0 */
  int32_t  free_goal_vel;        /* goal_tolerance.free_goal_vel (teb_config.h:295, default false) */
  int32_t  complete_global_plan; /* goal_tolerance.complete_global_plan (:298, default true) */
  int32_t  shrink_horizon_backup;/* recovery.shrink_horizon_backup (:381, default true) */
  double   prune_distance;       /* trajectory.global_plan_prune_distance (:264, default 1) */
  double   max_lookahead_dist;   /* trajectory.max_global_plan_lookahead_dist (:263, default 1); <= 0: no length limit */
  double   viapoint_sep;         /* trajectory.global_plan_viapoint_sep (:261, default -1: no via-points) */
  double   xy_goal_tolerance;    /* goal_tolerance (:293, default 0.2) */
  double   yaw_goal_tolerance;   /* (:294, default 0.2) */
  double   trans_stopped_vel;    /* (:296, default 0.1) */
  double   theta_stopped_vel;    /* (:297, default 0.1) */
  double   shrink_horizon_min_duration; /* recovery (:382, default 10) */
  const double*  global_plan;    /* [B][G_cap][3] x, y, yaw */
  int32_t*       plan_begin;     /* [B] in/out: the first live row, moved forward by pruning */
  const int32_t* plan_end;       /* [B] one past the last live row */
  const double*  robot;          /* [B][3] x, y, yaw (robot_pose_) */
  const double*  robot_vel;      /* [B][3] odometry vx, vy, omega */
  const int32_t* grid;           /* [S][2] sx, sy: the costmap's size in cells (as TebCostmapArgs) */
  const double*  origin;         /* [S][3] ox, oy, resolution (as TebCostmapArgs; only the resolution is read) */
  const int32_t* infeasible_count; /* [B] or NULL: no_infeasible_plans_ */
  const double*  since_infeasible; /* [B] or NULL: seconds since the last infeasible plan, inf: never */
  double*        plan;           /* [B][P_cap][3] out: x, y, yaw */
  int32_t*       plan_count;     /* [B] out */
  int32_t*       goal_idx;       /* [B] out or NULL: the reference's goal_idx, an index into the pruned plan */
  double*        via;            /* [B][V_cap][2] out, or NULL: the band's via-points are the caller's own
                                    (custom_via_points_active_); nothing is written and via_count is read */
  int32_t*       via_count;      /* [B] out (in when via == NULL, NULL there counts 0) */
  int32_t*       result;         /* [B] out: TEB_LOCAL_PLAN_* */
  int32_t*       needed;         /* [B][2] out or NULL: plan rows, via-points the band needed */
} TebLocalPlanArgs;
#define TEB_LOCAL_PLAN_PLANNED      0  /* plan, goal_idx and via-points written */
#define TEB_LOCAL_PLAN_GOAL_REACHED 1  /* the global goal is reached: plan_count = 0 */
#define TEB_LOCAL_PLAN_EMPTY        2  /* no live row in the global plan: plan_count = 0 */
#define TEB_LOCAL_PLAN_CAPACITY     3  /* more rows than P_cap or via-points than V_cap: plan_count = 0, see needed */
#define TEB_LOCAL_PLAN_BAD_INPUT    4  /* device entry point only: plan_begin / plan_end / scene_id out of range */

/* The frames of tebgpu_local_plan_tf and tebgpu_costmap_obstacles_tf (and their _device forms): the transforms the node
 * has looked up, so that the global plans and the custom obstacles stay in their own frames (usually map) while the
 * costmap, the robot pose and the obstacle tables are in the costmap's global frame (usually odom). The tf tree and its
 * lookups (time, transform_tolerance) stay the caller's. A transform is 7 doubles in geometry_msgs/Transform order
 * tx, ty, tz, qx, qy, qz, qw; the quaternion is taken as given, not normalised. HOST pointers for the synchronous entry
 * points, DEVICE pointers for the _device ones. Every NULL: the identity transform of TebLocalPlanArgs / TebCostmapArgs.
 *
 * The arithmetic is ROS Noetic's (tf2 LinearMath, tf2_geometry_msgs' doTransform, tf2/impl/utils.h getYaw, tf2_eigen's
 * transformToEigen) and Eigen 3.3's (toRotationMatrix, the fixed-size matrix-vector product of an x86-64 SSE2 build),
 * none of which is in the reference checkout; csrc/teb_frame.h holds it once for the host and the device. Every product
 * and sum is rounded on its own (no FMA contraction).
 *
 * tf2::doTransform of a plan row (x, y, yaw) under a transform T = (t, q): the row's orientation is r = (0, 0,
 * sin(yaw / 2), cos(yaw / 2)) (teb_plan_yaw's model) and z = 0. basis(q) is Matrix3x3::setRotation (s = 2 / |q|^2);
 * the position is basis(T) * (x, y, 0) + t, each row of the basis summed ((b0 x + b1 y) + b2 0) + t_i; the orientation
 * is getRotation() of basis(T) * basis(r) (the trace branch, else the largest diagonal element's); the yaw stored is
 * tf2::getYaw of it (sarg = -2 (xz - wy) / |q|^2; sarg <= -0.99999: -2 atan2(y, x); >= 0.99999: 2 atan2(y, x); else
 * atan2(2 (xy + wz), w^2 + x^2 - y^2 - z^2)). In TebLocalPlanArgs' steps:
 *   1, 3  compare the rows, still in the plan frame, with doTransform(robot, costmap_to_plan)'s position; the window,
 *         plan_length and every decision are the plan frame's, as in the reference.
 *   3     every row taken, and the injected global goal, is doTransform(row, plan_to_costmap); only rows taken are
 *         transformed: the plan write moves each once, and the via-point count and write (when via-points are
 *         extracted) move each row they scan once more per pass.
 *   4     via-points from the transformed rows.
 *   5     the goal-reached test reads doTransform(g[n - 1], plan_to_costmap): its position, and getYaw of its orientation
 *         in place of teb_plan_yaw(g[n - 1].yaw).
 *   7     the stored yaw is the transformed row's; goal_idx >= n - 1: getYaw of the transformed local goal's
 *         orientation; goal_idx > n - 5: getYaw(q * r(g[n - 1].yaw)), the raw tf2 quaternion product with
 *         plan_to_costmap's q; else the moving average over the transformed positions of the local goal and g[goal_idx
 *         + 1 ..].
 *   8     row 0 is the robot pose as given (the costmap frame).
 * Custom rows (TebCostmapArgs step 2) under custom_to_costmap: Eigen::Isometry3d(Translation3d(t) * Quaterniond(q)),
 * whose linear part is toRotationMatrix (no division by |q|^2, so a non-unit quaternion scales here where setRotation
 * does not, as in the node) and whose translation is 0 + t; a point p moves to linear * (p.x, p.y, 0) + translation,
 * rows summed as above.
 *   Point, Circular  (x, y) moves; radius, velocities (not rotated: the reference passes setCentroidVelocity the
 *                    message's twist as it is), dynamic and the rest verbatim.
 *   Line, Pill       custom_vertices[s][vertex_begin .. + 2) move into obst_vertices at the same index (vertex_count
 *                    must be 2); (x, y) = 0.5 * (start + end) of the moved ends.
 *   Polygon          custom_vertices[s][vertex_begin .. + vertex_count) move into obst_vertices; then finalizePolygon:
 *                    the last vertex is dropped (fixPolygonClosure, obstacles.cpp:48-55) when Eigen's isApprox (1e-12)
 *                    finds it equal to the first (vertex_count - 1 in the row), and (x, y) = calcCentroid
 *                    (obstacles.cpp:57-126) of the moved vertices.
 *   other types      verbatim.
 * Where the device and the reference part ways: sin, cos, atan2 and sqrt are the device's (the yaws and the goal
 * heading, not the positions: those are bit for bit); a stored yaw that came from a tilted transform is read back
 * downstream through teb_plan_yaw, where the reference keeps the tilted quaternion; an angle the two sides round to
 * opposite ends of +-pi differs by 2 pi. */
typedef struct TebFrameArgs {
  int32_t PV_cap;                  /* vertices per scene (stride of custom_vertices and obst_vertices), >= 0 */
  int32_t _pad;
  const double* costmap_to_plan;   /* [B][7] or NULL: lookupTransform(plan_frame, global_frame), moves the robot pose */
  const double* plan_to_costmap;   /* [B][7] or NULL: plan_to_global_transform, moves the rows taken */
  const double* custom_to_costmap; /* [S][7] or NULL: obstacle_to_map of each scene's custom obstacles */
  const double* custom_vertices;   /* [S][PV_cap][2] or NULL: the custom Line / Pill / Polygon vertices in their frame */
  double*       obst_vertices;     /* [S][PV_cap][2] out (the batch's vertex pool): the moved vertices of the rows written */
} TebFrameArgs;

/* The controller state of every robot between cycles, and the two steps of TebLocalPlannerROS::computeVelocityCommands
 * around plan() that read and write it: tebgpu_backup_modes, the oscillation half of configureBackupModes
 * (teb_local_planner_ros.cpp:980-1016, with FailureDetector of recovery_behaviors.cpp), after tebgpu_local_plan and
 * before tebgpu_plan_batch; and tebgpu_finish_cycle, the back half of the cycle (:360-454 with saturateVelocity :874-919
 * and convertTransRotVelToSteeringAngle :922-933), after the plan and the feasibility check. HOST pointers for the
 * synchronous entry points, DEVICE pointers for the _device ones. The velocity limits (max_vel_x, max_vel_x_backwards,
 * max_vel_y, max_vel_trans, max_vel_theta), min_turning_radius and the divergence settings are the context's
 * parameters (tebgpu_set_params). Of the batch, B is read by both steps and n, status and chi2 by tebgpu_finish_cycle.
 * `now` stands for every ros::Time::now() of the step; the stamps last_infeasible / last_oscillation are in its clock,
 * -inf meaning never, and the caller forms the next local plan's since_infeasible = now - last_infeasible. Every
 * product and sum is rounded on its own (no FMA contraction); min(a, b) = b < a ? b : a, max(a, b) = a < b ? b : a;
 * sign(x) = x > 0 ? 1 : x < 0 ? -1 : 0 (g2o::sign, 0 for 0 and NaN); a NaN fails every comparison.
 *
 * tebgpu_backup_modes, per band b whose local_plan_result is PLANNED or CAPACITY (the results with which the reference
 * reaches configureBackupModes; GOAL_REACHED and EMPTY return before it, :296-304, :713-717; the other bands are not
 * touched), when oscillation_recovery != 0 (else oscillating[b] = 0 and nothing else is written):
 *   1. The recovery's max_vel_theta: mvc = last_cmd[b].vx >= 0 ? max_vel_x : max_vel_x_backwards; if
 *      min_turning_radius != 0 && mvc > 0 it is max(mvc / |min_turning_radius|, max_vel_theta), else max_vel_theta.
 *   2. FailureDetector::update(last_cmd[b]), skipped when buffer_length == 0 (the detector is off, oscillating 0):
 *      v = last_cmd vx divided by max_vel_x when v > 0 && max_vel_x > 0, else by max_vel_x_backwards when v < 0 && that
 *      limit is > 0; omega = last_cmd omega divided by step 1's value when it is > 0. (v, omega) is pushed into the
 *      band's ring of capacity buffer_length; a push into a full ring drops the oldest entry. The ring's k-th oldest
 *      entry is osc_ring[(head + k) % buffer_length][b], (size, head) = osc_fill[b].
 *   3. detect: oscillating when size >= buffer_length / 2 (integer division), |v_mean| < oscillation_v_eps,
 *      |omega_mean| < oscillation_omega_eps and crossings > 1 (all strict), the means summed from 0 over the entries
 *      from the oldest, in order, then divided by size; crossings counts the entries k >= 1 with sign(omega_k) !=
 *      sign(omega_{k-1}).
 *   4. recently = now - last_oscillation[b] < oscillation_recovery_min_duration. Oscillating: if not recently,
 *      prefer_rotdir[b] = robot_vel[b].omega > 0 ? TEB_ROTDIR_LEFT : TEB_ROTDIR_RIGHT (0 and NaN give RIGHT); then
 *      last_oscillation[b] = now. Not oscillating, not recently and prefer_rotdir[b] != NONE: prefer_rotdir[b] = NONE.
 *   oscillating[b] = isOscillating() after the update. Pass prefer_rotdir as TebBatch.prefer_rotdir of the plan.
 *
 * tebgpu_finish_cycle, per band b, with r = local_plan_result[b]; outcome[b] is the first that applies. "Failure"
 * means: cmd_vel[b] = 0, n[b] = 0 (clearPlanner), infeasible_count[b] += 1 (it stops at INT32_MAX), last_infeasible[b]
 * = now, last_cmd[b] = 0.
 *   TEB_CYCLE_GOAL_REACHED     r == GOAL_REACHED (:290-304): cmd_vel 0, n = 0 (isGoalReached's clearPlanner); the
 *                              counters and last_cmd are not touched.
 *   TEB_CYCLE_NO_PLAN          r == EMPTY, CAPACITY or BAD_INPUT: cmd_vel 0, nothing else is written.
 *   TEB_CYCLE_PLAN_FAILED      !(status & OPTIMIZED) || status & (CAPACITY | BAD_INPUT) (:361-371): failure.
 *   TEB_CYCLE_DIVERGED         divergence_detection_enable && chi2 > divergence_detection_max_chi_squared (:374-386,
 *                              hasDiverged): failure.
 *   TEB_CYCLE_INFEASIBLE       feasible[b] == 0 (:396-410): failure.
 *   TEB_CYCLE_UNDECIDABLE      feasible[b] == -1: failure (the safe, infeasible case).
 *   TEB_CYCLE_INVALID_COMMAND  cmd[b][3] == 0, getVelocityCommand returned false (:413-423): failure.
 *   TEB_CYCLE_STEERING_NOT_FINITE  cmd_angle_instead_rotvel and a non-finite steering angle (:433-448): failure.
 *   TEB_CYCLE_COMMAND          otherwise (:425-454): cmd_vel = the saturated (vx, vy, omega) of cmd[b], omega replaced by
 *                              the steering angle when cmd_angle_instead_rotvel; infeasible_count = 0; last_cmd = cmd_vel
 *                              (with the steering angle, as in the reference).
 * saturateVelocity(vx, vy, omega): ratios rx = ry = ro = 1; vx > max_vel_x: rx = max_vel_x / vx; vy > max_vel_y ||
 *   vy < -max_vel_y: ry = |max_vel_y / vy| (so max_vel_y = 0 zeroes vy, and with proportional saturation the whole
 *   twist); omega > max_vel_theta || omega < -max_vel_theta: ro = |max_vel_theta / omega|; when max_vel_x_backwards > 0
 *   and vx < -max_vel_x_backwards, rx = -max_vel_x_backwards / vx. use_proportional_saturation: each component times
 *   min(min(rx, ry), ro); otherwise vx * rx, vy * ry, omega * ro. Then with l = hypot(vx, vy), l > max_vel_trans: vx
 *   and vy times max_vel_trans / l. max_vel_trans = 0 is used as it is and zeroes vx and vy: the node never sees 0,
 *   because its reconfigure replaces it with max_vel_x (teb_config.cpp:219-224); abi.make_cycle_args does the same.
 * Steering angle of (v, omega) = (vx, omega) after saturation: 0 when omega == 0 || v == 0; else radius = v / omega,
 *   replaced by sign(radius) * m when |radius| < m, m = 0.95 * min_turning_radius (one rounded product); atan(wheelbase
 *   / radius).
 *
 * Argument errors return TEBGPU_ERR_INVALID_ARG before anything is launched: NULL batch or required array, B outside
 * 1 .. max_bands, L_cap < 0, buffer_length outside 0 .. L_cap, a non-finite now. The host entry points also refuse a
 * band with local_plan_result outside 0 .. 4, prefer_rotdir outside 0 .. 2, feasible outside -1 .. 1 or osc_fill
 * outside 0 .. buffer_length (head 0 when buffer_length is 0), whichever the step reads. The device entry points answer
 * such a band with outcome TEB_CYCLE_NO_PLAN (cmd_vel 0, nothing else written) or oscillating = -1 (its state not
 * touched). */
typedef struct TebCycleArgs {
  int32_t  use_proportional_saturation; /* robot.use_proportional_saturation (teb_config.h:289, default false) */
  int32_t  cmd_angle_instead_rotvel;    /* robot.cmd_angle_instead_rotvel (:287, default false) */
  int32_t  oscillation_recovery;        /* recovery.oscillation_recovery (:383, default true) */
  int32_t  buffer_length;  /* the detector's capacity: round(oscillation_filter_duration * controller_frequency), the
                              node's setBufferLength (teb_local_planner_ros.cpp:188); 0: the detector is off */
  int32_t  L_cap;          /* ring entries per band (stride of osc_ring), >= buffer_length */
  int32_t  _pad;
  double   wheelbase;                   /* robot.wheelbase (:286, default 1; may be negative) */
  double   oscillation_v_eps;           /* recovery (:384, default 0.1) */
  double   oscillation_omega_eps;       /* (:385, default 0.1) */
  double   oscillation_recovery_min_duration; /* (:386, default 10) */
  double   now;                         /* the cycle's ros::Time::now() in seconds, finite */
  const int32_t* local_plan_result; /* [B] TEB_LOCAL_PLAN_* of tebgpu_local_plan, or NULL: every band PLANNED */
  const double*  robot_vel;         /* [B][3] odometry vx, vy, omega (robot_vel_); backup modes */
  const double*  cmd;               /* [B][4] TebPlanInput.cmd: vx, vy, omega, ok; finish */
  const int32_t* feasible;          /* [B] tebgpu_check_feasible's answer, or NULL: not checked, every band feasible */
  int32_t*       infeasible_count;  /* [B] in/out: no_infeasible_plans_ (tebgpu_local_plan reads it) */
  double*        last_infeasible;   /* [B] in/out: time_last_infeasible_plan_, -inf: never */
  double*        last_oscillation;  /* [B] in/out: time_last_oscillation_, -inf: never */
  double*        last_cmd;          /* [B][3] in/out: last_cmd_ vx, vy, omega */
  int32_t*       prefer_rotdir;     /* [B] in/out: last_preferred_rotdir_, TEB_ROTDIR_* (TebBatch.prefer_rotdir) */
  double*        osc_ring;          /* [L_cap][B][2] in/out: normalised (v, omega), band-minor; may be NULL when buffer_length == 0 */
  int32_t*       osc_fill;          /* [B][2] in/out: the ring's size and head (slot of its oldest entry) */
  double*        cmd_vel;           /* [B][3] out: the twist published (finish) */
  int32_t*       outcome;           /* [B] out: TEB_CYCLE_* (finish) */
  int32_t*       oscillating;       /* [B] out or NULL: 1 / 0, -1 for out-of-range ring state (backup modes) */
} TebCycleArgs;
#define TEB_CYCLE_COMMAND              0
#define TEB_CYCLE_GOAL_REACHED         1
#define TEB_CYCLE_NO_PLAN              2
#define TEB_CYCLE_PLAN_FAILED          3
#define TEB_CYCLE_DIVERGED             4
#define TEB_CYCLE_INFEASIBLE           5
#define TEB_CYCLE_UNDECIDABLE          6
#define TEB_CYCLE_INVALID_COMMAND      7
#define TEB_CYCLE_STEERING_NOT_FINITE  8

/* sizeof() of the ABI structs, for binding sanity checks. which: 0 TebParams, 1 TebObstacle, 2 TebBatch,
 * 3 TebOptimizeArgs, 4 TebGpuLimits, 5 TebPlanInput, 6 TebFeasibilityArgs, 7 TebTrajectoryArgs, 8 TebCostmapArgs,
 * 9 TebLocalPlanArgs, 10 TebCycleArgs, 11 TebCostmapWorld, 12 TebFrameArgs, 13 TebHsigFactors, 14 TebFleetArgs,
 * 15 TebFleetRow, 16 TebFleetTable. */
int32_t tebgpu_sizeof(int32_t which);

/* Context life cycle. One context = one device + one stream + its device workspaces.
 * Replaces initOptimizer()/SparseOptimizer ownership (optimal_planner.cpp:161-179). */
int32_t tebgpu_create(const TebGpuLimits* limits, int32_t device, tebgpu_ctx** out);
int32_t tebgpu_destroy(tebgpu_ctx* ctx);
const char* tebgpu_last_error_string(const tebgpu_ctx* ctx);

/* cfg_ pointer equivalent (optimal_planner.h:675): parameters are copied, call again after changes. */
int32_t tebgpu_set_params(tebgpu_ctx* ctx, const TebParams* params);

/* optimizeTEB over a whole batch, HOST buffers: H2D copy, all outer x inner LM iterations on the
 * device, D2H copy of poses / n / cost / chi2 / status / lm_iters, synchronous.
 * Replaces HomotopyClassPlanner::optimizeAllTEBs' thread fan-out (homotopy_class_planner.cpp:466-493). */
int32_t tebgpu_optimize_batch(tebgpu_ctx* ctx, const TebBatch* batch, const TebOptimizeArgs* args);

/* Same, every pointer in `batch` is a DEVICE pointer on the context's device. Stream-ordered on the
 * context stream (or `cuda_stream` if non-NULL, a cudaStream_t passed as void*; NULL means the context's own
 * stream, so pass cudaStreamLegacy / cudaStreamPerThread explicitly to target a default stream); does NOT
 * synchronise. */
int32_t tebgpu_optimize_batch_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebOptimizeArgs* args,
                                     void* cuda_stream);
int32_t tebgpu_synchronize(tebgpu_ctx* ctx);

/* TebOptimalPlanner::plan (optimal_planner.cpp:247-321) followed by getVelocityCommand (:1135-1168) for every band of
 * the batch, the per-cycle work of a controller:
 *   1. n[b] == 0: cold start, initTrajectoryToGoal(start, goal, 0, max_vel_x, min_samples, ...) or, with a plan,
 *      initTrajectoryToGoal(plan, max_vel_x, max_vel_theta, global_plan_overwrite_orientation, min_samples,
 *      allow_init_with_backwards_motion). n[b] > 0: warm start, updateAndPruneTEB(start, goal, min_samples), when the goal
 *      lies closer than force_reinit_new_goal_dist to the band's last pose and its heading differs by less than
 *      force_reinit_new_goal_angular (both strict); otherwise the band is cleared and initialised again.
 *   2. optimizeTEB(no_inner_iterations, no_outer_iterations) exactly as tebgpu_optimize_batch runs it with `args`
 *      (pass the parameter block's iteration counts for plan()); vel_start / vel_goal are read from the batch as there,
 *      so start_vel == NULL and free_goal_vel are expressed through their active flags. cost, chi2, status and
 *      lm_iters mean what they mean for tebgpu_optimize_batch.
 *   3. cmd[b] = getVelocityCommand(look_ahead_poses) on the optimised band.
 * A band whose initialisation needs more than n_cap poses is left as it was and gets TEB_STATUS_CAPACITY; its command
 * is read from the band as it was. tebgpu_plan_batch: HOST buffers, synchronous; a non-finite start, goal or plan row,
 * or a plan_count outside 1 .. P_cap, returns TEBGPU_ERR_INVALID_ARG before anything runs. It keeps a device copy of
 * the plans sized by the largest P_cap it has been called with (allocated by the first call that needs more; there is
 * no P_cap limit to set). tebgpu_plan_batch_device: DEVICE buffers, stream ordered as tebgpu_optimize_batch_device,
 * does not synchronise; such a band is left as it was and gets TEB_STATUS_BAD_INPUT, the other bands are planned. In
 * the CUDA-graph replay of tebgpu_set_graph the whole cycle (plan, optimize, command) is one captured sequence. */
int32_t tebgpu_plan_batch(tebgpu_ctx* ctx, TebBatch* batch, const TebPlanInput* plan, const TebOptimizeArgs* args);
int32_t tebgpu_plan_batch_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebPlanInput* plan,
                                 const TebOptimizeArgs* args, void* cuda_stream);

/* isTrajectoryFeasible (optimal_planner.cpp:1250-1310) for every band of the batch, against the world model described at
 * TebFeasibilityArgs. Per band:
 *   1. look_ahead_idx is clamped to n - 1, then, with lookahead_distance > 0, set to i - 1 for the first pose i whose
 *      std::hypot distance from pose 0 is > lookahead_distance.
 *   2. The queries, in order: pose i, then for i < look_ahead_idx the reference's intermediate poses towards pose i + 1
 *      (sequential accumulation, strict > tests against angular_resolution and inscribed_radius). Sample counts beyond
 *      the int range, where the reference is undefined, saturate at INT_MAX - 1 per segment.
 *   3. feasible is decided by the first query that is not free: 0 if it collides, -1 if it is undecidable. If every
 *      query is free: 1, unless the band has more than max_queries queries (then only the first max_queries are
 *      tested) and none of those is non-free: -1. A non-finite x / y / theta among the checked poses gives -1 with no
 *      query; so does, in the device entry point, a band whose n or scene_id is out of range or whose scene holds an
 *      obstacle row the batch cannot describe.
 *   4. query_count: the queries the reference makes, up to and including the first non-free one. When the band has more
 *      than max_queries queries and the first max_queries are free, it is the band's total number of queries (what the
 *      reference makes when all are free), so that a retry can be sized; it saturates at INT32_MAX. n == 0 gives
 *      feasible 1 and no query.
 *   5. queries (if not NULL): the first min(query_count, max_queries) query poses; the rows behind them are not written.
 * Reads only poses, n, scene_id, obstacles, obst_count and obst_vertices of the batch and writes only the outputs in
 * `args`; nothing the optimize or plan entry points read changes. Argument errors (NULL batch arrays or outputs, a bad
 * inscribed_radius / angular_resolution / collision_distance / max_queries) return TEBGPU_ERR_INVALID_ARG before anything
 * is launched. tebgpu_check_feasible: HOST buffers, synchronous; n, scene_id, obst_count or obstacle rows out of range
 * are refused with TEBGPU_ERR_INVALID_ARG too; the device copies of the outputs are allocated by the first call that
 * needs them. tebgpu_check_feasible_device: DEVICE buffers, stream ordered as tebgpu_optimize_batch_device, does not
 * synchronise. M_cap <= 1024 stages the scene's table in shared memory, above that the rows are read from global
 * memory (tebgpu_get_info keys 12 / 13). */
int32_t tebgpu_check_feasible(tebgpu_ctx* ctx, const TebBatch* batch, const TebFeasibilityArgs* args);
int32_t tebgpu_check_feasible_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebFeasibilityArgs* args,
                                     void* cuda_stream);

/* isTrajectoryFeasible for every band of the batch against its scene's costmap, the reference's own check, as defined
 * at TebCostmapWorld. Same queries and outputs as tebgpu_check_feasible; reads only poses, n and scene_id of the batch
 * (obstacles, obst_count and obst_vertices are not read) and writes only the outputs in `args` and world->query_cost.
 * One CTA per band, a warp per query, its lanes over the cells of one outline edge; the raster is read through the
 * read-only cache (tebgpu_get_info keys 12 / 13: B CTAs, TEBGPU_FEAS_BUILD_COSTMAP). Argument errors (NULL batch arrays,
 * outputs, world or its arrays, a bad inscribed_radius / angular_resolution / max_queries, cell_cap < 1,
 * footprint_count outside 0 .. TEB_COSTMAP_FOOTPRINT_MAX, a non-finite footprint coordinate) return
 * TEBGPU_ERR_INVALID_ARG before anything is launched. tebgpu_check_feasible_costmap: HOST buffers, synchronous; the
 * bands the device entry point answers with -1 are refused with TEBGPU_ERR_INVALID_ARG too; the device copies are
 * allocated by the first call that needs them. tebgpu_check_feasible_costmap_device: DEVICE buffers, stream ordered as
 * tebgpu_optimize_batch_device, does not synchronise. */
int32_t tebgpu_check_feasible_costmap(tebgpu_ctx* ctx, const TebBatch* batch, const TebFeasibilityArgs* args,
                                      const TebCostmapWorld* world);
int32_t tebgpu_check_feasible_costmap_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebFeasibilityArgs* args,
                                             const TebCostmapWorld* world, void* cuda_stream);

/* getVelocityProfile and getFullTrajectory (optimal_planner.cpp:1170-1248) of the bands listed in `args`, as defined at
 * TebTrajectoryArgs: what a controller publishes as its local plan every cycle. Reads only poses, n, vel_start and
 * vel_goal of the batch and writes only the outputs in `args`. The holonomic / non-holonomic choice is the context's
 * max_vel_y != 0 (tebgpu_set_params; the TebConfig default 0 until then), as in extractVelocity. Argument errors (NULL
 * poses / n / vel_start / vel_goal or points, profile and trajectory both NULL, count < 0 with bands) return
 * TEBGPU_ERR_INVALID_ARG before anything is launched; count == 0 launches nothing. tebgpu_read_trajectory: HOST buffers, synchronous; a band index outside
 * 0 .. B - 1 or a band read out whose n is outside 0 .. n_cap is refused with TEBGPU_ERR_INVALID_ARG too; the device
 * copies of the outputs are allocated by the first call that needs them. tebgpu_read_trajectory_device: DEVICE buffers,
 * stream ordered as tebgpu_optimize_batch_device, does not synchronise; such a row gets points = -1 and nothing else,
 * the other rows are read. One warp per row (tebgpu_get_info key 14). */
int32_t tebgpu_read_trajectory(tebgpu_ctx* ctx, const TebBatch* batch, const TebTrajectoryArgs* args);
int32_t tebgpu_read_trajectory_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebTrajectoryArgs* args,
                                      void* cuda_stream);

/* The obstacle table of every scene from its local costmap, as defined at TebCostmapArgs, written where a TebBatch reads
 * it (obstacles, obst_count): convert, then plan and check on the same stream. One CTA per scene stages the raster in
 * shared memory and enumerates it in the reference's order (tebgpu_get_info key 15). Argument errors (NULL required
 * arrays, S outside 1 .. max_scenes, M_cap outside 1 .. max_obstacles, cell_cap or C_cap < 0, C_cap > 0 with custom ==
 * NULL, a misaligned obstacles or custom pointer) return TEBGPU_ERR_INVALID_ARG (TEBGPU_ERR_CAPACITY past a limit)
 * before anything is launched. tebgpu_costmap_obstacles: HOST buffers, synchronous; a negative size, sx * sy > cell_cap
 * or a custom_count outside 0 .. C_cap is refused with TEBGPU_ERR_INVALID_ARG too; its device copies are allocated by
 * the first call that needs them. tebgpu_costmap_obstacles_device: DEVICE buffers, stream ordered as
 * tebgpu_optimize_batch_device, does not synchronise; such a scene gets obst_count = needed = -1 and nothing else, the
 * other scenes are converted. */
int32_t tebgpu_costmap_obstacles(tebgpu_ctx* ctx, const TebCostmapArgs* args);
int32_t tebgpu_costmap_obstacles_device(tebgpu_ctx* ctx, const TebCostmapArgs* args, void* cuda_stream);

/* Every band's local plan, goal and via-points from its global plan, as defined at TebLocalPlanArgs: cut, then plan on
 * the same stream. One warp per band walks the global plan in 32-row chunks, 4 bands per CTA (tebgpu_get_info key 16).
 * Argument errors (NULL batch, scene_id or required array, B outside 1 .. max_bands, S outside 1 .. max_scenes, G_cap
 * < 1, P_cap < 2, V_cap < 0) return TEBGPU_ERR_INVALID_ARG (TEBGPU_ERR_CAPACITY past a limit) before anything is
 * launched; so does tebgpu_local_plan for a band the device entry point would answer with TEB_LOCAL_PLAN_BAD_INPUT.
 * tebgpu_local_plan: HOST buffers, synchronous; its device copies are allocated by the first call that needs them.
 * tebgpu_local_plan_device: DEVICE buffers, stream ordered as tebgpu_optimize_batch_device, does not synchronise. */
int32_t tebgpu_local_plan(tebgpu_ctx* ctx, const TebBatch* batch, const TebLocalPlanArgs* args);
int32_t tebgpu_local_plan_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebLocalPlanArgs* args, void* cuda_stream);

/* The same two steps with each robot's global plan and each scene's custom obstacles in their own frames, as defined at
 * TebFrameArgs. frames == NULL, or all four of its transform / vertex pointers NULL, is the call without _tf, bit for
 * bit. Argument errors of TebFrameArgs (only one of costmap_to_plan / plan_to_costmap; custom_vertices without
 * custom_to_costmap; custom_vertices without obst_vertices or PV_cap; PV_cap < 0; a misaligned custom array) return
 * TEBGPU_ERR_INVALID_ARG before anything is launched. tebgpu_costmap_obstacles_tf also refuses a custom Line / Pill /
 * Polygon row whose vertices lie outside 0 .. PV_cap or are not given (custom_vertices == NULL); the _device form answers
 * that scene with obst_count = needed = -1 instead. tebgpu_costmap_obstacles_tf copies back the moved vertices of every
 * row it wrote, into frames->obst_vertices (HOST). */
int32_t tebgpu_local_plan_tf(tebgpu_ctx* ctx, const TebBatch* batch, const TebLocalPlanArgs* args,
                             const TebFrameArgs* frames);
int32_t tebgpu_local_plan_tf_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebLocalPlanArgs* args,
                                    const TebFrameArgs* frames, void* cuda_stream);
int32_t tebgpu_costmap_obstacles_tf(tebgpu_ctx* ctx, const TebCostmapArgs* args, const TebFrameArgs* frames);
int32_t tebgpu_costmap_obstacles_tf_device(tebgpu_ctx* ctx, const TebCostmapArgs* args, const TebFrameArgs* frames,
                                           void* cuda_stream);

/* The two controller steps around plan(), as defined at TebCycleArgs. One thread per band, so that the detector's sums
 * run in the reference's order (tebgpu_get_info key 17). A fleet cycle on one stream: tebgpu_costmap_obstacles_device,
 * tebgpu_local_plan_device, tebgpu_backup_modes_device, tebgpu_plan_batch_device, tebgpu_check_feasible_device,
 * tebgpu_finish_cycle_device. tebgpu_backup_modes / tebgpu_finish_cycle: HOST buffers, synchronous; their device copies
 * are allocated by the first call that needs them. The _device forms: DEVICE buffers, stream ordered as
 * tebgpu_optimize_batch_device, do not synchronise. */
int32_t tebgpu_backup_modes(tebgpu_ctx* ctx, const TebBatch* batch, const TebCycleArgs* args);
int32_t tebgpu_backup_modes_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebCycleArgs* args, void* cuda_stream);
int32_t tebgpu_finish_cycle(tebgpu_ctx* ctx, TebBatch* batch, const TebCycleArgs* args);
int32_t tebgpu_finish_cycle_device(tebgpu_ctx* ctx, TebBatch* batch, const TebCycleArgs* args, void* cuda_stream);

/* The other robots of a fleet as custom obstacle rows of every robot's scene (tebgpu_fleet_obstacles): what a
 * multi-robot publisher sends on the custom obstacle topic, one circle with a velocity per robot, read the way
 * TebLocalPlannerROS::updateObstacleContainerWithCustomObstacles reads a circle message (teb_local_planner_ros.cpp:576-581,
 * setCentroidVelocity obstacles.h:214-233). It runs between tebgpu_finish_cycle of one cycle and
 * tebgpu_costmap_obstacles(_tf) of the next, so custom and custom_count are the TebCostmapArgs arrays of the next
 * conversion. HOST pointers for tebgpu_fleet_obstacles, DEVICE pointers for tebgpu_fleet_obstacles_device.
 *
 * Robot r has the pose (x, y, theta) = pose[r] in one common frame, the frame of the custom obstacles (usually map);
 * the body-frame command (vx, vy) = last_cmd[r] (TebCycleArgs.last_cmd, whose omega is not read); radius rho = radius[r];
 * world w = world[r] (NULL: one world); scene s = scene[r] (NULL: s = r). Every product and sum is rounded on its own
 * (no FMA contraction).
 *   1. Neighbours (defined here): q is a neighbour of r when q != r, world[q] == world[r] and dx * dx + dy * dy <=
 *      range * range (dx = x_q - x_r, dy = y_q - y_r). Coincident robots are neighbours; a NaN distance is not.
 *      needed[r] = the number of neighbours. They are ordered by (d2, q): nearest first, a tie to the lower index.
 *   2. Rows: the first written = min(needed, max_rows, C_cap - own) neighbours (own = own_count[s], 0 for NULL) go to
 *      custom[s][own .. own + written), in order. Neighbour q gives {x_q, y_q, vx, vy, rho_q, dynamic, TEB_OBST_CIRCULAR,
 *      0, 0, _pad 0}: the publisher's map-frame velocity (vx, vy) = R(theta_q) (cmd vx, cmd vy), i.e. (c vx - s vy,
 *      s vx + c vy) with c = cos(theta_q), s = sin(theta_q); then setCentroidVelocity's rule, taken of the body command
 *      whose norm the rotation keeps (so that no decision depends on sin / cos): sqrt(cmd vx * cmd vx + cmd vy * cmd vy)
 *      < 0.001 gives dynamic 0 and velocity (0, 0), otherwise dynamic 1 with (vx, vy). The rows move with the other custom
 *      rows under TebFrameArgs.custom_to_costmap; velocities are not rotated there (TebFrameArgs).
 *   3. custom_count[s] = own + written. Rows custom[s][0 .. own) and past own + written are not touched, so a second
 *      call with the same inputs writes the same bytes: own_count holds the caller's own rows and must not be
 *      custom_count.
 *   4. status[r] = TEB_FLEET_WRITTEN, or TEB_FLEET_TRUNCATED when written < needed[r] (max_rows or C_cap cut the list;
 *      the nearest neighbours are the ones kept).
 * sin and cos are the device's (velocities within ~1e-16 relative of the correctly rounded ones); every decision,
 * position, radius and the order are exact.
 *
 * Argument errors return TEBGPU_ERR_INVALID_ARG (TEBGPU_ERR_CAPACITY past a limit) before anything is launched: NULL
 * args or a required array (pose, last_cmd, radius, custom_count; custom when C_cap > 0), R outside 1 .. max_bands, S
 * outside 1 .. max_scenes, C_cap < 0, max_rows outside 0 .. TEB_FLEET_MAX_ROWS, a NaN or negative range, scene == NULL
 * with R > S, own_count == custom_count, a custom pointer that is not 16-byte aligned. tebgpu_fleet_obstacles: HOST
 * buffers, synchronous; it also refuses a non-finite pose or command, a radius that is negative or not finite, a scene
 * outside 0 .. S - 1, an own_count outside 0 .. C_cap, and two robots in one scene; its device copies are allocated by
 * the first call that needs them. tebgpu_fleet_obstacles_device: DEVICE buffers, stream ordered as
 * tebgpu_optimize_batch_device, does not synchronise; a robot whose scene is outside 0 .. S - 1 or whose own_count is
 * outside 0 .. C_cap gets TEB_FLEET_BAD_INPUT, one whose scene another robot also maps to gets TEB_FLEET_SHARED_SCENE;
 * either has needed = -1 and nothing written to its scene. Such robots are still neighbours of the others. The shared
 * scene check takes context scratch of S int32, and the grid search (below) bucket counts and starts, the candidate
 * indices and the far list, sized to the largest candidate count seen; each is allocated by the first call that needs
 * it, which synchronises the stream. Calls of one context share this scratch, so issue them on one stream.
 *
 * One warp per robot, FLEET_WARPS robots per CTA, keeps its top-max_rows list in registers, one slot per lane
 * (tebgpu_get_info key 18: the grid in CTAs). The candidates come from one of two searches (tebgpu_set_fleet_search;
 * key 19 reports the one the last step ran), which write the same bytes on every input:
 *   all pairs  the CTA stages the fleet's (x, y, world) in shared-memory tiles and the lanes test every candidate:
 *              O(R^2);
 *   grid       the candidates are binned into square cells of side h = max(range (1 + 2^-16), 2^-500) per world,
 *              hashed into buckets; each robot tests the candidates of its 3 x 3 cells, and those past the cell
 *              coordinate bound 2^24 (a far list): O(R) for a fleet of bounded density.
 * The automatic search takes the grid from 4096 candidates on when range is above 2^-500 and range * range is finite;
 * below that, and at range inf, all pairs. The kept list is ordered by (d2, index), a total order, so it does not depend
 * on the order the candidates are met in, and both searches are exact and deterministic. */
#define TEB_FLEET_MAX_ROWS 32
#define TEB_FLEET_WRITTEN       0  /* every neighbour in range written */
#define TEB_FLEET_TRUNCATED     1  /* written < needed: max_rows or C_cap - own_count kept the nearest ones */
#define TEB_FLEET_BAD_INPUT     2  /* device entry point only: scene or own_count out of range; nothing written */
#define TEB_FLEET_SHARED_SCENE  3  /* device entry point only: another robot maps to the same scene; nothing written */
typedef struct TebFleetArgs {
  int32_t  R;                 /* robots, 1 .. max_bands */
  int32_t  S;                 /* scenes (rows of custom_count), 1 .. max_scenes */
  int32_t  C_cap;             /* custom rows per scene (stride of custom, as TebCostmapArgs.C_cap), >= 0 */
  int32_t  max_rows;          /* neighbour rows per robot, 0 .. TEB_FLEET_MAX_ROWS */
  double   range;             /* neighbour distance, >= 0 (inf: every robot of the world) */
  const double*  pose;        /* [R][3] x, y, theta in the custom obstacles' frame */
  const double*  last_cmd;    /* [R][3] body-frame vx, vy, omega (TebCycleArgs.last_cmd); omega is not read */
  const double*  radius;      /* [R] the circle each robot is published as */
  const int32_t* world;       /* [R] or NULL: one world */
  const int32_t* scene;       /* [R] or NULL: robot r writes scene r */
  const int32_t* own_count;   /* [S] or NULL: the caller's own custom rows of each scene (0 for NULL) */
  TebObstacle*   custom;      /* [S][C_cap] in/out: TebCostmapArgs.custom, 16-byte aligned */
  int32_t*       custom_count;/* [S] out: TebCostmapArgs.custom_count; only the scenes of valid robots are written */
  int32_t*       needed;      /* [R] out or NULL: neighbours in range, -1 for a robot answered with BAD_INPUT / SHARED */
  int32_t*       status;      /* [R] out or NULL: TEB_FLEET_* */
} TebFleetArgs;
int32_t tebgpu_fleet_obstacles(tebgpu_ctx* ctx, const TebFleetArgs* args);
int32_t tebgpu_fleet_obstacles_device(tebgpu_ctx* ctx, const TebFleetArgs* args, void* cuda_stream);

/* The fleet table: every robot of a fleet as the row it is published as, shared by the contexts and ranks that hold the
 * fleet's robots, so that each robot gets the robots of other contexts (another robot kind, another TebParams) and of
 * other GPUs as neighbour rows. A cycle runs, between tebgpu_finish_cycle and tebgpu_costmap_obstacles(_tf):
 *   1. tebgpu_fleet_publish: every owner writes its R robots as rows first .. first + R - 1 of the table;
 *   2. sharing: one table in one GPU's memory that every context writes (contexts ordered by one stream or by events),
 *      or tebgpu_fleet_gather across the ranks of a communicator (tebgpu_comm_init), one ncclAllGather of 64 T bytes;
 *   3. tebgpu_fleet_obstacles_table: every owner runs TebFleetArgs' step for its R robots with the candidates taken from
 *      all T rows of the table.
 * When the owners' robots are contiguous shards of one global robot order (owner g's robot i is global robot
 * first_g + i - pad_g, padding rows only between shards), the key (d2, table row) orders the candidates as (d2, global
 * index) does, so the outputs are bit for bit those of one tebgpu_fleet_obstacles call over the whole fleet.
 *
 * TebFleetRow: robot q as published. The position, velocity, dynamic flag and radius are those of the custom row
 * TebFleetArgs step 2 writes for q: (vx, vy) = R(theta_q) (cmd vx, cmd vy), (0, 0) with dynamic 0 when the body command's
 * norm is below 0.001. live == 0 marks padding, which is never a neighbour; _pad is written as 0. 64 bytes. */
typedef struct TebFleetRow {
  double  x, y;               /* position in the custom obstacles' frame */
  double  vx, vy;             /* map-frame velocity after the 0.001 rule */
  double  radius;             /* the circle the robot is published as */
  int32_t world;              /* TebFleetArgs.world (0 when that is NULL) */
  int32_t dynamic;            /* 1 moving, 0 still */
  int32_t live;               /* 1 a robot, 0 padding */
  int32_t _pad[3];
} TebFleetRow;

typedef struct TebFleetTable {
  int32_t      T;             /* rows of the table, >= 1 */
  int32_t      first;         /* this call's robots are rows first .. first + R - 1 */
  TebFleetRow* rows;          /* [T], 16-byte aligned; HOST or DEVICE as the entry point says */
} TebFleetTable;

/* tebgpu_fleet_publish(_device): rows[first + r] = robot r, r < args->R, from args->pose, last_cmd, radius and world
 * (NULL: world 0), with live = 1; no other field of args is read and no other row is written. The velocity and the
 * dynamic flag come from the same device function as tebgpu_fleet_obstacles' rows. One thread per robot.
 *
 * tebgpu_fleet_gather(_device): the in-place all-gather of a table of T = world * cap rows over the context's
 * communicator: rank g contributes rows [g cap, (g + 1) cap) and every rank ends with all T rows. NCCL has no
 * all-gather-v, so shards of fewer robots are padded to cap with live = 0 rows (the caller's, written once). Without a
 * communicator (one rank) it does nothing. table->first is not read. Stream ordered on the context's stream (_device,
 * or cuda_stream when given), or synchronous on host rows.
 *
 * tebgpu_fleet_obstacles_table(_device): TebFleetArgs' step for the call's R robots (robot r is table row first + r),
 * the candidates being all T rows of the table: q is a neighbour of r when q != first + r, rows[q].live, rows[q].world
 * == rows[first + r].world and the distance rule holds; they are ordered by (d2, q) and each is written as its row
 * ({x, y, vx, vy, radius, dynamic} of the row, TEB_OBST_CIRCULAR, 0, 0, _pad 0}). The robot's position and world are
 * those of its own row; pose, last_cmd, radius and world of args are not read (may be NULL). scene, own_count, custom,
 * custom_count, needed, status, the cuts and the shared-scene check are TebFleetArgs'. On the device, a robot whose own
 * row is not live gets TEB_FLEET_BAD_INPUT (needed -1, nothing written); the host entry point refuses it, and refuses a
 * live row whose x, y, vx, vy or radius is not finite or whose radius is negative. The candidates are the T rows, found
 * by all pairs or by the grid as in TebFleetArgs' step (4096 rows and up: the grid), so each owner pays O(R T) or
 * O(R + T); tebgpu_get_info keys 18 / 19 report the launch's grid and search.
 *
 * Argument errors return TEBGPU_ERR_INVALID_ARG (TEBGPU_ERR_CAPACITY past a limit) before anything is launched: those
 * of TebFleetArgs for the arrays each step reads, NULL table or rows, T < 1, first < 0, first + R > T, rows not 16-byte
 * aligned; in the gather cap < 1 or T != world * cap. The host forms take HOST rows (and HOST args arrays) and
 * synchronise; their device copies are allocated by the first call that needs them. The _device forms take DEVICE
 * pointers, are stream ordered as tebgpu_optimize_batch_device and do not synchronise. */
int32_t tebgpu_fleet_publish(tebgpu_ctx* ctx, const TebFleetArgs* args, const TebFleetTable* table);
int32_t tebgpu_fleet_publish_device(tebgpu_ctx* ctx, const TebFleetArgs* args, const TebFleetTable* table,
                                    void* cuda_stream);
int32_t tebgpu_fleet_gather(tebgpu_ctx* ctx, const TebFleetTable* table, int32_t cap);
int32_t tebgpu_fleet_gather_device(tebgpu_ctx* ctx, const TebFleetTable* table, int32_t cap, void* cuda_stream);
int32_t tebgpu_fleet_obstacles_table(tebgpu_ctx* ctx, const TebFleetArgs* args, const TebFleetTable* table);
int32_t tebgpu_fleet_obstacles_table_device(tebgpu_ctx* ctx, const TebFleetArgs* args, const TebFleetTable* table,
                                            void* cuda_stream);

/* Linear solver / scheduling of the LM step (replaces LinearSolverCSparse, optimal_planner.h:75-79):
 * 2 (default) speculative: the next 4 damping trials are solved concurrently, one thread per (band, trial), banded
 *   LDL^T with the active window in registers, and the accept / reject chain is replayed in order;
 * 1 block cyclic reduction on 8x8 blocks in shared memory (max_poses <= 256), one CTA per band;
 * 0 sequential banded LDL^T in shared memory, one CTA per band.  All three give the same results up to round-off. */
int32_t tebgpu_set_solver(tebgpu_ctx* ctx, int32_t solver);
/* Thread mapping of kernel A: 0 (default) k_linearize2: one thread per pose, 125-pose tiles, band rows accumulated in
 * registers; 1 the first-generation kernel: one 128-thread CTA per 32-pose tile, one thread per band row. Same
 * arithmetic, different summation order (results agree to round-off); variant 1 is kept as an independent cross-check. */
int32_t tebgpu_set_linearize_variant(tebgpu_ctx* ctx, int32_t variant);
/* The neighbour search of the fleet steps (tebgpu_fleet_obstacles(_device), tebgpu_fleet_obstacles_table(_device)):
 * TEBGPU_FLEET_SEARCH_AUTO (default) the grid from 4096 candidates on with a finite range above 2^-500, else all pairs;
 * _ALL_PAIRS always all pairs; _GRID always the grid; _ONE_BUCKET the grid with every cell hashed to one bucket (a test
 * of the bucket collisions). Every mode writes the same bytes. Another mode returns TEBGPU_ERR_INVALID_ARG. */
#define TEBGPU_FLEET_SEARCH_AUTO 0
#define TEBGPU_FLEET_SEARCH_ALL_PAIRS 1
#define TEBGPU_FLEET_SEARCH_GRID 2
#define TEBGPU_FLEET_SEARCH_ONE_BUCKET 3
int32_t tebgpu_set_fleet_search(tebgpu_ctx* ctx, int32_t mode);
/* Speculation width of solver 2: how many consecutive LM damping trials are solved per round (2, 4, 6 or 8; 0 = auto).
 * Results do not depend on it (the accept / reject chain is replayed in order), only latency and traffic do. */
int32_t tebgpu_set_speculation(tebgpu_ctx* ctx, int32_t k);

/* Mapping of the default solver's solve kernel (replaces LinearSolverCSparse::solve, optimal_planner.cpp:169-172):
 *   0  one THREAD per (band, trial) system (k_solve_tpb) always - the throughput mapping;
 *   1  one WARP per system (k_solve_warp: window spread over the lanes, pivot column through shared memory, axpy back
 *      substitution), 2 the same only while a round has at most (SMs x 8) systems. Bit-identical to mode 0, slower per
 *      solve; kept as an independent cross-check of the factorisation;
 *   3  k_solve_lat always: one warp per system, the system resident in shared memory, TWISTED factorisation (the two
 *      half-warps eliminate from both ends towards an 11-unknown middle block), faster per solve than mode 0 when
 *      the machine is not full; another elimination order, so results agree with mode 0 to rounding, not bit for bit;
 *   4  (default) k_solve_lat while the systems of a round fit three waves of resident CTAs - the latency regime of a
 *      single planning request - and k_solve_tpb above that. */
int32_t tebgpu_set_warp_solver(tebgpu_ctx* ctx, int32_t mode);

/* Form of k_solve_tpb (the thread-per-system mapping above): 0 (default) automatic by speculation width, 1 the LDL^T
 * factor streamed through device memory and read back by the back substitution, 11 / 22 / 33 the factor not stored but
 * recomputed from window checkpoints in segments of that many rows (k_solve_tpb_rc). Same bits in every form; only
 * memory traffic and time differ. The environment variable TEBGPU_SOLVE_FORM sets the initial value. */
int32_t tebgpu_set_solve_form(tebgpu_ctx* ctx, int32_t form);

/* CUDA-graph replay of the launch sequence of tebgpu_optimize_batch(_device): 0 never, 1 always, 2 (default) in the
 * latency regime only (a batch of at most ~2300 bands, e.g. one planning request of 32 candidates, where the 130-170
 * kernel launches of one optimizeTEB are comparable to the kernels themselves). A sequence is captured once per distinct
 * (batch description incl. buffer addresses, optimize arguments, parameters, switches, stream) and replayed afterwards;
 * the context keeps the 8 most recently used graphs. Results are identical to direct launches. */
int32_t tebgpu_set_graph(tebgpu_ctx* ctx, int32_t mode);

/* Per-kernel device timing (CUDA events on the launching stream around every launch) for roofline reporting.
 * enable != 0 -> subsequent optimize calls record events. tebgpu_get_kernel_times synchronises, then returns for
 * kernel kind k (0 begin, 1 auto_resize, 2 build_graph, 3 linearize ["kernel A"], 4 lm_step [fused "kernel B" of
 * solvers 0/1; for solver 2: the solve/eval launches of the retry rounds >= 1], 5 finalize, 6 solve_tpb round 0,
 * 7 trial_eval round 0 (includes the accept / reject replay), 8 unused since the replay was fused into trial_eval
 * ["kernel B" of the default speculative solver])
 * the accumulated milliseconds and launch count since profiling was enabled, and resets the accumulators. */
int32_t tebgpu_set_profiling(tebgpu_ctx* ctx, int32_t enable);
int32_t tebgpu_get_kernel_times(tebgpu_ctx* ctx, double ms_out[9], int64_t count_out[9]);
/* Same for the two launches only the plan entry points issue: 0 k_plan_begin, 1 k_velocity_command. */
int32_t tebgpu_get_plan_kernel_times(tebgpu_ctx* ctx, double ms_out[2], int64_t count_out[2]);

/* HomotopyClassPlanner::calculateEquivalenceClass (homotopy_class_planner.hpp:46-63) for every band of the batch, i.e.
 * the step that decides which candidates are kept before they are optimised (renewAndAnalyzeOldTebs,
 * homotopy_class_planner.cpp:214-256). include_dynamic_obstacles == 0: HSignature (h_signature.h:97-186), h_out[b] =
 * (Re H, Im H), stride 2; otherwise HSignature3d (h_signature.h:282-353), h_out[b][l] for the M obstacles of the band's
 * scene, stride M_cap. The path is the band's pose positions; use_timediffs != 0 takes the transition times from the
 * band's dt, 0 approximates them by |z2 - z1| / max_vel_x (h_signature.h:307-315, graph-search candidates have no time
 * information yet). The reference accumulates the 2-D signature in long double; the device uses fp64 (|dH| <= 1e-9 |H|
 * against the long double oracle, far below h_signature_threshold). device_ptrs as in tebgpu_build_system. The host
 * buffers are checked before anything runs; with device pointers a band whose scene_id is outside 0 .. S - 1, whose
 * scene's obst_count is outside 0 .. M_cap (-1 from an overflowing tebgpu_costmap_obstacles_device) or whose n is
 * outside 0 .. n_cap gets NaN in every output of its row. */
int32_t tebgpu_h_signature(tebgpu_ctx* ctx, const TebBatch* batch, int32_t use_timediffs, double* h_out, int32_t device_ptrs);

/* The scene half of the 2-D signature, for scenes of up to 16384 obstacles (tebgpu_sizeof(13)). HSignature's pole
 * residue A_l = f0(o_l) / prod_{j != l, |o_l - o_j| >= 0.05} (o_l - o_j) (h_signature.h:149-163) splits into the band's
 * f0 (its map rectangle) and
 *     Q_l = 1 / prod_{j != l, |o_l - o_j| >= 0.05} (o_l - o_j),
 * which depends on the scene's rows only. Q_l = (factor[s][l][0] + i factor[s][l][1]) * 2^factor_exp[s][l], exponent
 * INT32_MIN for 0; factor_count[s] is the obst_count the table was built at, -1 for a count outside 0 .. M_cap. Rows past
 * factor_count[s] are 0 / INT32_MIN. The table is the caller's to rebuild whenever a scene's rows change, e.g. after
 * every tebgpu_costmap_obstacles: factor_count only catches a changed count, not moved rows. */
typedef struct TebHsigFactors {
  double*  factor;        /* [S][M_cap][2] mantissa (Re, Im) of Q_l */
  int32_t* factor_exp;    /* [S][M_cap] binary exponent of Q_l */
  int32_t* factor_count;  /* [S] obst_count the scene's table was built at, or -1 */
} TebHsigFactors;

/* Builds every scene's factor table; only S, M_cap, obstacles and obst_count of the batch are read. A scene's table
 * depends on its own rows only (the same bits whatever S, M_cap or the scene's index). NULL arrays, S outside 1 ..
 * max_scenes or M_cap outside 0 .. max_obstacles return TEBGPU_ERR_INVALID_ARG (TEBGPU_ERR_CAPACITY past a limit) before
 * anything is launched. tebgpu_hsig_factors: HOST buffers, synchronous, an obst_count outside 0 .. M_cap is refused.
 * tebgpu_hsig_factors_device: DEVICE buffers, stream ordered as tebgpu_optimize_batch_device, does not synchronise;
 * such a scene gets factor_count = -1. Partial products live in context scratch, allocated by the first call that needs
 * it (it synchronises the stream when it grows) and freed by tebgpu_destroy. */
int32_t tebgpu_hsig_factors(tebgpu_ctx* ctx, const TebBatch* batch, const TebHsigFactors* factors);
int32_t tebgpu_hsig_factors_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebHsigFactors* factors, void* cuda_stream);

/* The output of tebgpu_h_signature (stride 2 for 2-D, stride max(M_cap, 1) for x-y-t, chosen by
 * include_dynamic_obstacles) for every M_cap from 0 to max_obstacles (<= 16384). 2-D: A_l = f0(o_l) * Q_l from the
 * factor table, factors == NULL builds the table in the same call (context scratch); x-y-t does not read factors. The
 * per-band work is O(n M) and a band is split over CTAs of 256 obstacles; its sum does not depend on the batch around it.
 * f0 is applied after the product instead of before it, so the 2-D values are not the bits of tebgpu_h_signature; both
 * stay within 1e-12 sum_{k,l} |A_l| |L_kl| of the long double signature. tebgpu_h_signature_scenes: HOST buffers
 * (factors too), checked as tebgpu_h_signature's, synchronous. tebgpu_h_signature_scenes_device: DEVICE buffers, stream
 * ordered, does not synchronise; a band whose scene_id, n or scene obst_count is out of range (obst_count -1 from an
 * overflowing tebgpu_costmap_obstacles_device) gets NaN in every output of its row, and so does a 2-D band whose
 * scene's factor_count differs from obst_count (a table built for other rows). Calls of one context share its scratch:
 * issue them on one stream. */
int32_t tebgpu_h_signature_scenes(tebgpu_ctx* ctx, const TebBatch* batch, const TebHsigFactors* factors,
                                  int32_t use_timediffs, double* h_out);
int32_t tebgpu_h_signature_scenes_device(tebgpu_ctx* ctx, const TebBatch* batch, const TebHsigFactors* factors,
                                         int32_t use_timediffs, double* h_out, void* cuda_stream);

/* Number of kernels launched by the last optimize call (for bench.py's gpu_launches). */
int64_t tebgpu_last_launch_count(const tebgpu_ctx* ctx);
/* Introspection for measurement scripts. which: 0 speculation width used by the last optimize call, 1 kernel-A variant,
 * 2 solver, 3 communicator size (1 without tebgpu_comm_init), 4 communicator rank, 5 CUDA-graph replay enabled,
 * 6 number of captured graphs held by the context, 7 speculation width of the first LM iteration after a graph rebuild
 * (key 0 reports the width of the later iterations), 8 grid in CTAs of the last trial-evaluation launch the context
 * issued (0 before the first; a replayed CUDA graph issues none), 9 which build that launch ran (TEBGPU_EVAL_BUILD_*,
 * -1 before the first), 10 grid in CTAs of the last kernel-A launch the context issued (0 before the first; a replayed
 * CUDA graph issues none), 11 which build that launch ran (TEBGPU_KA_BUILD_*, -1 before the first), 12 grid in CTAs of
 * the last feasibility-check launch (0 before the first), 13 which build that launch ran (TEBGPU_FEAS_BUILD_*, -1 before
 * the first), 14 grid in CTAs of the last trajectory read-out launch (k_read_trajectory, 4 rows per CTA; 0 before the
 * first), 15 grid in CTAs of the last costmap conversion (k_costmap_obstacles, one CTA per scene; 0 before the first),
 * 16 grid in CTAs of the last local-plan launch (k_local_plan, 4 bands per CTA; 0 before the first), 17 grid in CTAs
 * of the last backup-modes or finish-cycle launch (k_backup_modes / k_finish_cycle, 128 bands per CTA; 0 before the
 * first), 18 grid in CTAs of the last fleet-obstacle launch (k_fleet_obstacles or k_fleet_obstacles_grid, FLEET_WARPS
 * robots per CTA; 0 before the first), 19 the search that launch ran (TEBGPU_FLEET_SEARCH_ALL_PAIRS, _GRID or
 * _ONE_BUCKET; -1 before the first).
 * Returns -1 for an unknown key. */
#define TEBGPU_EVAL_BUILD_V1 0          /* k_trial_eval, first generation (TEBGPU_EVAL_V1=1): B CTAs */
#define TEBGPU_EVAL_BUILD_EVAL2_WIDE 1  /* k_trial_eval2, up to 16 warps per band (2 B <= SMs): B CTAs */
#define TEBGPU_EVAL_BUILD_EVAL2 2       /* k_trial_eval2 (B <= 2 x SMs): B CTAs */
#define TEBGPU_EVAL_BUILD_EVAL2P 3      /* k_trial_eval2p, persistent (B > 2 x SMs): resident CTAs per SM x SMs */
#define TEBGPU_EVAL_BUILD_EVAL3 4       /* k_trial_eval3 (latency regime or TEBGPU_EVAL3=1): K x B CTAs */
#define TEBGPU_KA_BUILD_V1 0       /* k_linearize, first generation (tebgpu_set_linearize_variant(1)): chunks x B CTAs */
#define TEBGPU_KA_BUILD_ONESHOT 1  /* k_linearize2, staged output (TEBGPU_KA_PERSIST=0): ceil(chunks / 4) x B CTAs */
#define TEBGPU_KA_BUILD_DIRECT 2   /* k_linearize2, direct stores (TEBGPU_KA_STAGED=0): ceil(chunks / 4) x B CTAs */
#define TEBGPU_KA_BUILD_PERSIST 3  /* k_linearize2p (default): resident one-warp CTAs per SM x SMs, at most chunks x B */
#define TEBGPU_FEAS_BUILD_STAGED 0  /* k_feasible, the scene's table staged in shared memory (M_cap <= 1024): B CTAs */
#define TEBGPU_FEAS_BUILD_GLOBAL 1  /* k_feasible, the table read from global memory / L2 (M_cap > 1024): B CTAs */
#define TEBGPU_FEAS_BUILD_COSTMAP 2 /* k_feasible, the costmap world (tebgpu_check_feasible_costmap): B CTAs */
int64_t tebgpu_get_info(const tebgpu_ctx* ctx, int32_t which);

/* Linearise only: build the padded banded normal equations of every band at its current state for
 * outer iteration `outer_index` (obstacle weight multiplier = weight_adapt_factor^outer_index).
 * Hb_out [B][4*n_cap][12] (device or host per `device_ptrs`): row r = 11 lower-band entries
 * H[r][r-k], k=0..10, then b[r]; chi2_out[B]. Test / profiling entry point for kernel A
 * (BlockSolver::buildSystem, SURVEY §3.3 step 2). */
int32_t tebgpu_build_system(tebgpu_ctx* ctx, const TebBatch* batch, int32_t outer_index,
                            double* Hb_out, double* chi2_out, int32_t device_ptrs);

/* Solve only: the linear solve of the LM step, (H + lambda_k I_real) x = b for bands 0 .. B-1 and trials k = 0 .. K-1,
 * through the kernel the context's solver selects (tebgpu_set_solver; for solver 2 the mapping of
 * tebgpu_set_warp_solver, launched by the same code as in tebgpu_optimize_batch). Test / profiling entry point of the
 * solve kernels. HOST buffers:
 *   Hb [B][4 n_cap][12]  system in kernel A's layout; NULL: the one the last tebgpu_build_system left in the context
 *                        (n and n_cap must then be the ones of that call);
 *   n [B]                poses per band, 3 .. n_cap;
 *   lambda, nu [B]       damping at the first trial of the round; trial k uses lambda nu (2 nu) ... (k factors), as
 *                        g2o's retries do. NULL: LM iteration 0, lambda = 1e-5 max |H_rr| over the real rows from kernel
 *                        A's partials (only valid after tebgpu_build_system);
 *   active [B]           or NULL (every band active); an inactive band solves nothing;
 *   K                    trials per band: 2, 4, 6 or 8;
 *   qmax [B], list       NULL / 0: round 0 over all bands. Otherwise a retry round over the list_len bands of `list`
 *                        (in that order) whose first qmax[b] trials were already used: trials with qmax[b] + k >= 10 are
 *                        not solved. Needs lambda;
 *   lat_cap              retry rounds with solve mapping 4: > 0 launches both k_solve_lat (lat_cap systems) and
 *                        k_solve_tpb, the list length decides on the device which one works; 0: automatic.
 * Outputs: dx_out [B][K][4 n_cap], ok_out [B][K] (1 solved, 0 not positive definite or not finite), lambda_out [B][K].
 * The solver scratch is filled with all-ones bytes (a NaN) before the launch, and what a kernel did not write is
 * returned as that pattern: the rows >= 4 n of a band, the systems that did not run, dx of a failed solve. */
int32_t tebgpu_solve_system(tebgpu_ctx* ctx, int32_t B, int32_t n_cap, const double* Hb, const int32_t* n,
                            const double* lambda, const double* nu, const int32_t* active, int32_t K, const int32_t* qmax,
                            const int32_t* list, int32_t list_len, int32_t lat_cap, double* dx_out, double* ok_out,
                            double* lambda_out);

/* Graph build + kernel A readout: the launches of tebgpu_build_system (k_begin, k_build_graph, kernel A, k_vor) with
 * the graph structure exposed. Test / profiling entry point of the graph build and of kernel A. HOST buffers.
 *   list, list_len       NULL: every band. Otherwise k_build_graph and kernel A run over the bands of `list` as the
 *                        retry side stream launches them (DevBatch::a_list / a_cnt, grids over the whole batch);
 *                        k_begin still runs for every band. Refused with a velocity-obstacle ratio weight (k_vor has no
 *                        list form).
 * Before the launches, Hb, rhs, the association, multiplicity-3 and occupancy words, via_idx, dyn_t and the tile
 * partials are filled with all-ones bytes (a NaN); what no kernel wrote comes back as that pattern.
 * Outputs (any may be NULL): Hb_out [B][4 n_cap][12]; chi_fam_out [B][4] kernel A's chi2 by family (obstacles, via,
 * time-optimal, other) folded as tebgpu_eval_trials folds its chi_lin, all-ones for a band not listed;
 * assoc_out, assoc3_out [B][n_cap][MW] (MW = max(1, ceil(M_cap / 64))); occ_out [B][n_cap][ceil(MW / 64)] (written
 * on the global-table path only, M_cap > 1024); via_idx_out [B][V_cap] (pose of each via-point, -1 skipped);
 * dyn_t_out [B][n_cap] (frozen dynamic-obstacle time of each pose). */
int32_t tebgpu_build_system_graph(tebgpu_ctx* ctx, const TebBatch* bt, int32_t outer_index, const int32_t* list,
                                  int32_t list_len, double* Hb_out, double* chi_fam_out, uint64_t* assoc_out,
                                  uint64_t* assoc3_out, uint64_t* occ_out, int32_t* via_idx_out, double* dyn_t_out);
/* Kernel A's other outputs of the last tebgpu_build_system(_graph) call on a batch of B bands and n_cap poses, HOST
 * buffers (any may be NULL): rhs_out [B][4 n_cap]; chi_parts_out [B][T][4] the tile partials of chi2 by family;
 * dmax_parts_out [B][T] the tile partials of the largest diagonal entry. T = ceil(n_cap / 29), ceil(n_cap / 32) under
 * linearize variant 1. */
int32_t tebgpu_read_linearize_outputs(tebgpu_ctx* ctx, int32_t B, int32_t n_cap, double* rhs_out, double* chi_parts_out,
                                      double* dmax_parts_out);

/* Trial evaluation only: one round of the speculative LM step's trial evaluation and accept / reject chain, launched by
 * the same code as in tebgpu_optimize_batch (the kernel TEBGPU_EVAL_V1 / TEBGPU_EVAL3 and the batch size select). Test /
 * profiling entry point of the trial-evaluation kernels. The graph, right-hand side and kernel A's chi2 / max-diagonal
 * partials are made as tebgpu_build_system makes them for outer_index. HOST buffers:
 *   bt                   the batch; bt->poses is the band state before the round and receives the state after it;
 *   iteration            LM iteration (0: round 0 takes lambda = 1e-5 max |H_rr| from kernel A, nu = 2), K: 2 .. 8 even;
 *   dx [B][K][4 n_cap], ok [B][K], lambda_k [B][K]   the trials as the solve left them (ok 0: failed factorisation,
 *                        the trial is x + b); a retry round reads the trials of band list[s] from row list[s];
 *   state [B][TEBGPU_EVAL_STATE]   band state before the round: lambda, nu, currentChi, chi2 by family at the current
 *                        state (4), at the last evaluated trial (4), status bits, active (1 / 0), LM iterations;
 *   qmax [B], list       NULL / 0: round 0 over all bands. Otherwise a retry round over the list_len bands of `list`
 *                        whose first qmax[b] trials were already used.
 * Outputs (any may be NULL): res_out [B][K][5] each trial's chi2 by family (obstacles, via, time-optimal, other) and
 * computeScale() sum, all-ones bytes (a NaN) where no trial was evaluated; chi_lin [B][4] kernel A's chi2 by family
 * (the sum of the band's tile partials); state_out [B][TEBGPU_EVAL_STATE]; qmax_out [B] trials of the iteration;
 * need_out [B] 1 when the band is queued for another round, 0 when its iteration ended, -1 where no band decided;
 * next_list [B] and *next_len the bands queued, in queue order. */
#define TEBGPU_EVAL_STATE 14
/* The state every band was left in by the context's last tebgpu_optimize_batch(_device) call (a CUDA-graph replay
 * included; tebgpu_build_system(_graph) and tebgpu_eval_trials overwrite it), in the TEBGPU_EVAL_STATE layout: lambda
 * and nu of the last LM iteration, currentChi, chi2 by family at the current state (4) and at the last evaluated trial
 * (4), status bits (without TEB_STATUS_OPTIMIZED, which only the outputs carry), active (0 once the band's last LM
 * iteration returned Terminate, or the band failed), LM iterations. out [B][TEBGPU_EVAL_STATE], HOST buffer. Test entry
 * point: it tells which exit each band's last LM iteration took (nu = 2^11 after ten rejected trials). Synchronises the
 * context's stream; after tebgpu_optimize_batch_device on another stream, synchronise that stream first. */
int32_t tebgpu_read_band_state(tebgpu_ctx* ctx, int32_t B, double* out);
int32_t tebgpu_eval_trials(tebgpu_ctx* ctx, TebBatch* bt, int32_t outer_index, int32_t iteration, int32_t K, const double* dx,
                           const double* ok, const double* lambda_k, const double* state, const int32_t* qmax,
                           const int32_t* list, int32_t list_len, double* res_out, double* chi_lin, double* state_out,
                           int32_t* qmax_out, int32_t* need_out, int32_t* next_list, int32_t* next_len);

/* TebOptimalPlanner::computeCurrentCost called OUTSIDE optimizeTEB (optimal_planner.cpp:1041-1094, graph rebuilt with
 * weight multiplier 1, errors evaluated at the current state): HOST buffers; writes cost[], chi2[], status[]. */
int32_t tebgpu_compute_cost(tebgpu_ctx* ctx, const TebBatch* batch, const TebOptimizeArgs* args);

/* HomotopyClassPlanner::selectBestTeb (homotopy_class_planner.cpp:564-667) on gathered costs:
 * argmin over cost[i], with cost[last_best] * selection_cost_hysteresis and
 * cost[initial_plan] * selection_prefer_initial_plan (pass -1 for none). Strict '<', first wins.
 * Host-side, pure function. Returns the index or -1 if count == 0. */
int32_t tebgpu_select_best(const double* cost, int32_t count, int32_t last_best, int32_t initial_plan,
                           double selection_cost_hysteresis, double selection_prefer_initial_plan);

/* ---- multi-GPU: one process (or thread) per GPU, each with its own context; the batch axis is sharded and bands never
 * exchange anything while they are optimised. What replaces the join of HomotopyClassPlanner::optimizeAllTEBs' thread
 * fan-out (homotopy_class_planner.cpp:466-493) before selectBestTeb (:564-616) is ONE all-gather of the per-candidate
 * costs over NCCL on the context's stream. NCCL is resolved at run time (dlopen); single-GPU users never load it.
 *   tebgpu_comm_get_unique_id  rank 0 creates the 128-byte id and distributes it out of band (MPI, a store, a file)
 *   tebgpu_comm_init           every rank, collectively: ncclCommInitRank on the context's device
 *   tebgpu_gather_costs        cost_all[r * count_local + k] = cost_local of rank r (same count on every rank);
 *                              device_ptrs != 0: both pointers are device memory, stream ordered on `cuda_stream` (a
 *                              cudaStream_t as void*; NULL = the context's stream, as in tebgpu_optimize_batch_device), no
 *                              synchronisation; 0: host memory, synchronous. Without a communicator (one rank): a copy.
 *   tebgpu_optimize_batch_gather  tebgpu_optimize_batch followed by the gather of batch->cost: cost_all [world * B] (host)
 * Errors: TEBGPU_ERR_UNSUPPORTED when NCCL cannot be loaded, TEBGPU_ERR_CUDA for NCCL / CUDA failures (see
 * tebgpu_last_error_string). */
#define TEBGPU_COMM_ID_BYTES 128
int32_t tebgpu_comm_get_unique_id(void* id_out);
int32_t tebgpu_comm_init(tebgpu_ctx* ctx, const void* id, int32_t world_size, int32_t rank);
int32_t tebgpu_comm_destroy(tebgpu_ctx* ctx);
int32_t tebgpu_gather_costs(tebgpu_ctx* ctx, const double* cost_local, int32_t count_local, double* cost_all, int32_t device_ptrs,
                            void* cuda_stream);
int32_t tebgpu_optimize_batch_gather(tebgpu_ctx* ctx, const TebBatch* batch, const TebOptimizeArgs* args, double* cost_all);

/* TimedElasticBand::autoResize (timed_elastic_band.cpp:227-286) on one host band; same routine the
 * device kernel runs. rec: [n_cap][4] in/out, returns the new n (or <0 on error). */
int32_t tebgpu_auto_resize_host(double* rec, int32_t n, int32_t n_cap, double dt_ref, double dt_hysteresis,
                                int32_t min_samples, int32_t max_samples, int32_t fast_mode);

#ifdef __cplusplus
}
#endif
#endif /* TEB_B200_H */
