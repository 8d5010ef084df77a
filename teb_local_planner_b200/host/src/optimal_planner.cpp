/* optimal_planner.cpp — see include/teb_local_planner/optimal_planner.h. Line references: src/optimal_planner.cpp of
 * the reference. The optimisation itself is ONE tebgpu_optimize_batch call (no CPU fallback: it fails if no GPU). */
#include "teb_local_planner/optimal_planner.h"

#include <algorithm>
#include <cstdio>
#include <mutex>

namespace teb_local_planner {

/* ------------------------------------------------------------------ GPU context */
TebGpuContext::TebGpuContext(int max_bands, int max_poses, int max_obstacles, int max_viapoints, int device,
                             int max_obst_vertices) {
  lim_.max_bands = max_bands;
  lim_.max_poses = max_poses;
  lim_.max_scenes = 1;
  lim_.max_obstacles = max_obstacles;
  lim_.max_viapoints = max_viapoints;
  lim_.max_obst_vertices = max_obst_vertices;
  int rc = tebgpu_create(&lim_, device, &ctx_);
  if (rc != TEBGPU_OK) {
    std::fprintf(stderr, "TebGpuContext: tebgpu_create failed rc=%d (%s)\n", rc, ctx_ ? tebgpu_last_error_string(ctx_) : "");
    if (ctx_) tebgpu_destroy(ctx_);
    ctx_ = nullptr;
  }
}
TebGpuContext::~TebGpuContext() {
  if (ctx_) tebgpu_destroy(ctx_);
}
std::shared_ptr<TebGpuContext> TebGpuContext::shared(int min_bands, int min_poses, int min_obstacles, int min_viapoints,
                                                     int min_obst_vertices) {
  static std::mutex mu;
  static std::shared_ptr<TebGpuContext> inst;
  std::lock_guard<std::mutex> lock(mu);
  if (!inst || !inst->get() || inst->limits().max_bands < min_bands || inst->limits().max_poses < min_poses ||
      inst->limits().max_obstacles < min_obstacles || inst->limits().max_viapoints < min_viapoints ||
      inst->limits().max_obst_vertices < min_obst_vertices) {
    int mb = std::max(min_bands, inst ? inst->limits().max_bands : 0);
    int mp = std::max(min_poses, inst ? inst->limits().max_poses : 0);
    int mo = std::max(min_obstacles, inst ? inst->limits().max_obstacles : 0);
    int mv = std::max(min_viapoints, inst ? inst->limits().max_viapoints : 0);
    int mpv = std::max(min_obst_vertices, inst ? inst->limits().max_obst_vertices : 0);
    inst.reset();
    inst = std::make_shared<TebGpuContext>(mb, mp, mo, mv, 0, mpv);
  }
  return inst;
}

/* ------------------------------------------------------------------ TebOptimalPlanner */
TebOptimalPlanner::TebOptimalPlanner() {
  vel_start_.first = true;
  vel_goal_.first = true;
}
TebOptimalPlanner::TebOptimalPlanner(const TebConfig& cfg, ObstContainer* obstacles, TebVisualizationPtr visual,
                                     const ViaPointContainer* via_points) {
  initialize(cfg, obstacles, visual, via_points);
}
TebOptimalPlanner::~TebOptimalPlanner() {}

/* :80-103 */
void TebOptimalPlanner::initialize(const TebConfig& cfg, ObstContainer* obstacles, TebVisualizationPtr visual,
                                   const ViaPointContainer* via_points) {
  cfg_ = &cfg;
  obstacles_ = obstacles;
  via_points_ = via_points;
  cost_ = HUGE_VAL;
  prefer_rotdir_ = RotType::none;
  setVisualization(visual);
  vel_start_.first = true;
  vel_start_.second = geometry_msgs::Twist();
  vel_goal_.first = true;
  vel_goal_.second = geometry_msgs::Twist();
  initialized_ = true;
}

/* :233-245 */
void TebOptimalPlanner::setVelocityStart(const geometry_msgs::Twist& vel_start) {
  vel_start_.first = true;
  vel_start_.second.linear.x = vel_start.linear.x;
  vel_start_.second.linear.y = vel_start.linear.y;
  vel_start_.second.angular.z = vel_start.angular.z;
}
void TebOptimalPlanner::setVelocityGoal(const geometry_msgs::Twist& vel_goal) {
  vel_goal_.first = true;
  vel_goal_.second = vel_goal;
}

/* :247-281 */
bool TebOptimalPlanner::plan(const std::vector<geometry_msgs::PoseStamped>& initial_plan, const geometry_msgs::Twist* start_vel,
                             bool free_goal_vel) {
  if (!initialized_ || initial_plan.empty()) return false;
  if (!teb_.isInit()) {
    teb_.initTrajectoryToGoal(initial_plan, cfg_->robot.max_vel_x, cfg_->robot.max_vel_theta,
                              cfg_->trajectory.global_plan_overwrite_orientation, cfg_->trajectory.min_samples,
                              cfg_->trajectory.allow_init_with_backwards_motion);
  } else {
    PoseSE2 start_(initial_plan.front().pose);
    PoseSE2 goal_(initial_plan.back().pose);
    if (teb_.sizePoses() > 0 &&
        (goal_.position() - teb_.BackPose().position()).norm() < cfg_->trajectory.force_reinit_new_goal_dist &&
        std::fabs(g2o::normalize_theta(goal_.theta() - teb_.BackPose().theta())) < cfg_->trajectory.force_reinit_new_goal_angular) {
      teb_.updateAndPruneTEB(start_, goal_, cfg_->trajectory.min_samples);
    } else {
      teb_.clearTimedElasticBand();
      teb_.initTrajectoryToGoal(initial_plan, cfg_->robot.max_vel_x, cfg_->robot.max_vel_theta,
                                cfg_->trajectory.global_plan_overwrite_orientation, cfg_->trajectory.min_samples,
                                cfg_->trajectory.allow_init_with_backwards_motion);
    }
  }
  if (start_vel) setVelocityStart(*start_vel);
  if (free_goal_vel) setVelocityGoalFree();
  else vel_goal_.first = true;
  return optimizeTEB(cfg_->optim.no_inner_iterations, cfg_->optim.no_outer_iterations);
}

/* :283-288 (the reference drops free_goal_vel here as well) */
bool TebOptimalPlanner::plan(const tf::Pose& start, const tf::Pose& goal, const geometry_msgs::Twist* start_vel, bool free_goal_vel) {
  (void)free_goal_vel;
  PoseSE2 start_(start);
  PoseSE2 goal_(goal);
  return plan(start_, goal_, start_vel);
}

/* :290-321 */
bool TebOptimalPlanner::plan(const PoseSE2& start, const PoseSE2& goal, const geometry_msgs::Twist* start_vel, bool free_goal_vel) {
  if (!initialized_) return false;
  if (!teb_.isInit()) {
    teb_.initTrajectoryToGoal(start, goal, 0, cfg_->robot.max_vel_x, cfg_->trajectory.min_samples,
                              cfg_->trajectory.allow_init_with_backwards_motion);
  } else {
    if (teb_.sizePoses() > 0 &&
        (goal.position() - teb_.BackPose().position()).norm() < cfg_->trajectory.force_reinit_new_goal_dist &&
        std::fabs(g2o::normalize_theta(goal.theta() - teb_.BackPose().theta())) < cfg_->trajectory.force_reinit_new_goal_angular) {
      teb_.updateAndPruneTEB(start, goal, cfg_->trajectory.min_samples);
    } else {
      teb_.clearTimedElasticBand();
      teb_.initTrajectoryToGoal(start, goal, 0, cfg_->robot.max_vel_x, cfg_->trajectory.min_samples,
                                cfg_->trajectory.allow_init_with_backwards_motion);
    }
  }
  if (start_vel) setVelocityStart(*start_vel);
  if (free_goal_vel) setVelocityGoalFree();
  else vel_goal_.first = true;
  return optimizeTEB(cfg_->optim.no_inner_iterations, cfg_->optim.no_outer_iterations);
}

/* :182-231 — the whole loop runs on the device */
bool TebOptimalPlanner::optimizeTEB(int iterations_innerloop, int iterations_outerloop, bool compute_cost_afterwards,
                                    double obst_cost_scale, double viapoint_cost_scale, bool alternative_time_cost) {
  if (!cfg_ || cfg_->optim.optimization_activate == false) return false;
  optimized_ = false;
  std::vector<TebOptimalPlanner*> one(1, this);
  if (!optimizeTebBatch(*cfg_, one, iterations_innerloop, iterations_outerloop, compute_cost_afterwards, obst_cost_scale,
                        viapoint_cost_scale, alternative_time_cost, gpu_))
    return false;
  return (status_ & TEB_STATUS_OPTIMIZED) != 0; /* optimizeTEB's return value; optimized_ may still be false (:230) */
}

static int rotdir_code(RotType r) { return r == RotType::left ? TEB_ROTDIR_LEFT : (r == RotType::right ? TEB_ROTDIR_RIGHT : TEB_ROTDIR_NONE); }

bool TebOptimalPlanner::runBatch(const TebConfig& cfg, const std::vector<TebOptimalPlanner*>& planners, int iterations_innerloop,
                                 int iterations_outerloop, bool compute_cost_afterwards, double obst_cost_scale,
                                 double viapoint_cost_scale, bool alternative_time_cost, TebGpuContextPtr gpu, bool cost_only, std::vector<std::vector<double>>* hsig_out) {
  const int B = (int)planners.size();
  if (B == 0) return true;
  /* capacities: autoResize may grow a band up to max_samples + 1 poses (timed_elastic_band.cpp:239) */
  int n_max = 0, V_max = 0;
  for (auto* pl : planners) {
    n_max = std::max(n_max, pl->teb().sizePoses());
    if (pl->via_points_) V_max = std::max(V_max, (int)pl->via_points_->size());
  }
  int n_cap = n_max;
  if (cfg.trajectory.teb_autosize && !cost_only) n_cap = std::min(512, std::max(cfg.trajectory.max_samples + 1, n_max));
  n_cap = std::max(n_cap, 3);
  if (n_max > 512) { std::fprintf(stderr, "optimizeTEB: band longer than 512 poses is not supported\n"); return false; }
  /* every planner may carry its own obstacle container: one scene per distinct container */
  std::vector<const ObstContainer*> scenes;
  std::vector<int32_t> scene_id(B);
  for (int b = 0; b < B; ++b) {
    const ObstContainer* oc = planners[b]->obstacles_;
    int s = -1;
    for (size_t k = 0; k < scenes.size(); ++k)
      if (scenes[k] == oc) s = (int)k;
    if (s < 0) { scenes.push_back(oc); s = (int)scenes.size() - 1; }
    scene_id[b] = s;
  }
  const int S = (int)scenes.size();
  int M_cap = 1;
  for (auto* oc : scenes)
    if (oc) M_cap = std::max(M_cap, (int)oc->size());
  if (M_cap > 16384) { std::fprintf(stderr, "optimizeTEB: more than 16384 obstacles per scene is not supported\n"); return false; }
  /* the H-signature kernels stage a scene of at most 1024 obstacles in shared memory and form the 2-D signature's
   * product over the M - 1 obstacle differences, O(M^2) per band, in one CTA */
  if (hsig_out && M_cap > 1024) {
    std::fprintf(stderr, "H-signature: more than 1024 obstacles per scene is not supported (the obstacle table is staged "
                         "in shared memory)\n");
    return false;
  }
  std::vector<TebObstacle> obst((size_t)S * M_cap);
  std::vector<int32_t> obst_count(S, 0);
  std::vector<std::vector<double>> pools(S);
  for (int s = 0; s < S; ++s) {
    if (!scenes[s]) continue;
    obst_count[s] = (int)scenes[s]->size();
    for (size_t m = 0; m < scenes[s]->size(); ++m) {
      TebObstacle& row = obst[(size_t)s * M_cap + m];
      row = (*scenes[s])[m]->toRow();
      (*scenes[s])[m]->appendVertices(pools[s], row); /* Line / Pill / Polygon: vertex range in the scene's pool */
    }
  }
  int PV_cap = 0;
  for (const std::vector<double>& pool : pools) PV_cap = std::max(PV_cap, (int)(pool.size() / 2));
  std::vector<double> obst_vertices((size_t)S * std::max(PV_cap, 1) * 2, 0.0);
  for (int s = 0; s < S; ++s) std::copy(pools[s].begin(), pools[s].end(), obst_vertices.begin() + (size_t)s * PV_cap * 2);
  if (!gpu) gpu = TebGpuContext::shared(B, n_cap, M_cap, V_max, PV_cap);
  if (!gpu || !gpu->get()) return false;
  const TebGpuLimits& lim = gpu->limits();
  if (lim.max_bands < B || lim.max_poses < n_cap || lim.max_obstacles < M_cap || lim.max_viapoints < V_max || lim.max_scenes < S ||
      lim.max_obst_vertices < PV_cap) {
    /* a caller-provided context that is too small: fall back to the (growing) shared one */
    gpu = TebGpuContext::shared(B, n_cap, M_cap, V_max, PV_cap);
    if (!gpu || !gpu->get() || gpu->limits().max_scenes < S) {
      std::fprintf(stderr, "optimizeTEB: GPU context limits exceeded (scenes=%d)\n", S);
      return false;
    }
  }
  /* one context = one stream + one parameter block: set_params .. optimize of two planners on different threads must
   * not interleave on a shared context (the reference gives every planner its own optimizer) */
  std::lock_guard<std::mutex> context_guard(gpu->mutex());
  TebParams params = cfg.toParams();
  if (planners[0]->robot_model_) planners[0]->robot_model_->fillParams(params);
  int rc = tebgpu_set_params(gpu->get(), &params);
  if (rc != TEBGPU_OK) {
    std::fprintf(stderr, "optimizeTEB: %s\n", tebgpu_last_error_string(gpu->get()));
    return false;
  }
  std::vector<double> poses((size_t)B * n_cap * 4, 0.0), via((size_t)B * std::max(V_max, 1) * 2, 0.0);
  std::vector<double> vel_start((size_t)B * 4), vel_goal((size_t)B * 4), cost(B), chi2(B);
  std::vector<int32_t> n(B), via_count(B, 0), rotdir(B), status(B), iters(B);
  for (int b = 0; b < B; ++b) {
    TebOptimalPlanner* pl = planners[b];
    n[b] = pl->teb().sizePoses();
    pl->teb().toRecords(&poses[(size_t)b * n_cap * 4]);
    if (pl->via_points_) {
      via_count[b] = (int)pl->via_points_->size();
      for (int v = 0; v < via_count[b]; ++v) {
        via[((size_t)b * V_max + v) * 2] = (*pl->via_points_)[v].x();
        via[((size_t)b * V_max + v) * 2 + 1] = (*pl->via_points_)[v].y();
      }
    }
    vel_start[4 * b] = pl->vel_start_.second.linear.x; vel_start[4 * b + 1] = pl->vel_start_.second.linear.y;
    vel_start[4 * b + 2] = pl->vel_start_.second.angular.z; vel_start[4 * b + 3] = pl->vel_start_.first ? 1.0 : 0.0;
    vel_goal[4 * b] = pl->vel_goal_.second.linear.x; vel_goal[4 * b + 1] = pl->vel_goal_.second.linear.y;
    vel_goal[4 * b + 2] = pl->vel_goal_.second.angular.z; vel_goal[4 * b + 3] = pl->vel_goal_.first ? 1.0 : 0.0;
    rotdir[b] = rotdir_code(pl->prefer_rotdir_);
    if (!cost_only && !hsig_out) pl->optimized_ = false;
  }
  TebBatch bt{};
  bt.B = B; bt.n_cap = n_cap; bt.S = S; bt.M_cap = M_cap; bt.V_cap = V_max;
  bt.PV_cap = PV_cap; bt.obst_vertices = PV_cap > 0 ? obst_vertices.data() : nullptr;
  bt.poses = poses.data(); bt.n = n.data(); bt.scene_id = scene_id.data(); bt.obstacles = obst.data();
  bt.obst_count = obst_count.data(); bt.via = V_max > 0 ? via.data() : nullptr; bt.via_count = V_max > 0 ? via_count.data() : nullptr;
  bt.vel_start = vel_start.data(); bt.vel_goal = vel_goal.data(); bt.prefer_rotdir = rotdir.data();
  bt.cost = cost.data(); bt.chi2 = chi2.data(); bt.status = status.data(); bt.lm_iters = iters.data();
  TebOptimizeArgs args{};
  args.iterations_innerloop = iterations_innerloop; args.iterations_outerloop = iterations_outerloop;
  args.compute_cost_afterwards = compute_cost_afterwards; args.alternative_time_cost = alternative_time_cost;
  args.obst_cost_scale = obst_cost_scale; args.viapoint_cost_scale = viapoint_cost_scale;
  if (hsig_out) { /* calculateEquivalenceClass for every planner: one device call */
    const bool three_d = cfg.obstacles.include_dynamic_obstacles;
    const size_t stride = three_d ? (size_t)M_cap : 2;
    std::vector<double> h((size_t)B * stride, 0.0);
    rc = tebgpu_h_signature(gpu->get(), &bt, /*use_timediffs=*/1, h.data(), 0);
    if (rc != TEBGPU_OK) {
      std::fprintf(stderr, "calculateEquivalenceClass: tebgpu_h_signature rc=%d (%s)\n", rc, tebgpu_last_error_string(gpu->get()));
      return false;
    }
    hsig_out->assign(B, std::vector<double>());
    for (int b = 0; b < B; ++b) {
      const size_t cnt = three_d ? (size_t)obst_count[scene_id[b]] : 2;
      (*hsig_out)[b].assign(h.begin() + (size_t)b * stride, h.begin() + (size_t)b * stride + cnt);
    }
    return true;
  }
  if (cost_only) {
    rc = tebgpu_compute_cost(gpu->get(), &bt, &args);
    if (rc != TEBGPU_OK) {
      std::fprintf(stderr, "computeCurrentCost: tebgpu_compute_cost rc=%d (%s)\n", rc, tebgpu_last_error_string(gpu->get()));
      return false;
    }
    for (int b = 0; b < B; ++b) planners[b]->cost_ = cost[b];
    return true;
  }
  rc = tebgpu_optimize_batch(gpu->get(), &bt, &args);
  if (rc != TEBGPU_OK) {
    std::fprintf(stderr, "optimizeTEB: tebgpu_optimize_batch rc=%d (%s)\n", rc, tebgpu_last_error_string(gpu->get()));
    return false;
  }
  for (int b = 0; b < B; ++b) {
    TebOptimalPlanner* pl = planners[b];
    pl->status_ = status[b];
    pl->chi2_ = chi2[b];
    /* OPTIMIZED is optimizeTEB's return value (returned by optimizeTEB above); with no outer iteration optimizeTEB
     * returns true with optimized_ still false */
    pl->optimized_ = (status[b] & TEB_STATUS_OPTIMIZED) != 0 && iterations_outerloop > 0;
    if (pl->optimized_ || cfg.trajectory.teb_autosize) pl->teb().fromRecords(&poses[(size_t)b * n_cap * 4], n[b]);
    if (pl->optimized_ && compute_cost_afterwards) pl->cost_ = cost[b];
  }
  return true;
}

bool TebOptimalPlanner::hSignatureBatch(const TebConfig& cfg, const std::vector<TebOptimalPlanner*>& planners,
                                        std::shared_ptr<TebGpuContext> gpu, std::vector<std::vector<double>>& values) {
  return runBatch(cfg, planners, 0, 0, false, 1.0, 1.0, false, gpu, true, &values);
}

bool optimizeTebBatch(const TebConfig& cfg, const std::vector<TebOptimalPlanner*>& planners, int iterations_innerloop,
                      int iterations_outerloop, bool compute_cost_afterwards, double obst_cost_scale,
                      double viapoint_cost_scale, bool alternative_time_cost, TebGpuContextPtr gpu) {
  return TebOptimalPlanner::runBatch(cfg, planners, iterations_innerloop, iterations_outerloop, compute_cost_afterwards, obst_cost_scale,
                     viapoint_cost_scale, alternative_time_cost, gpu, false);
}

/* :1041-1094 outside optimizeTEB: the graph is rebuilt at the current state (weight multiplier 1), fresh errors */
void TebOptimalPlanner::computeCurrentCost(double obst_cost_scale, double viapoint_cost_scale, bool alternative_time_cost) {
  if (!cfg_) return;
  std::vector<TebOptimalPlanner*> one(1, this);
  runBatch(*cfg_, one, 0, 0, true, obst_cost_scale, viapoint_cost_scale, alternative_time_cost, gpu_, true);
}

/* :1023-1039 */
bool TebOptimalPlanner::hasDiverged() const {
  if (!cfg_ || !cfg_->recovery.divergence_detection_enable) return false;
  return chi2_ > cfg_->recovery.divergence_detection_max_chi_squared;
}

/* Mean velocity that carries the robot from pose1 to pose2 in dt (reference :1097-1134). Non-holonomic robots
 * (max_vel_y == 0) move along their heading: the speed is the segment length, signed by whether the displacement points
 * forwards or backwards; holonomic robots get the displacement expressed in the frame of pose1. dt == 0 yields zero. */
inline void TebOptimalPlanner::extractVelocity(const PoseSE2& pose1, const PoseSE2& pose2, double dt, double& vx, double& vy,
                                               double& omega) const {
  vx = vy = omega = 0;
  if (dt == 0) return;
  const Eigen::Vector2d step = pose2.position() - pose1.position();
  const double c = std::cos(pose1.theta()), s = std::sin(pose1.theta());
  const double along = c * step.x() + s * step.y(), across = -s * step.x() + c * step.y();
  if (cfg_->robot.max_vel_y == 0) {
    vx = (double)g2o::sign(along) * step.norm() / dt;
  } else {
    vx = along / dt;
    vy = across / dt;
  }
  omega = g2o::normalize_theta(pose2.theta() - pose1.theta()) / dt;
}

/* Velocity command for the controller (reference :1136-1172): the mean velocity from the first pose to the pose
 * `look_ahead_poses` ahead - clamped so that it stays prevent_look_ahead_poses_near_goal poses away from the goal, and cut
 * short as soon as the accumulated time reaches dt_ref x look_ahead_poses. */
bool TebOptimalPlanner::getVelocityCommand(double& vx, double& vy, double& omega, int look_ahead_poses) const {
  vx = vy = omega = 0;
  const int poses = teb_.sizePoses();
  if (poses < 2) return false;
  int target = std::max(1, std::min(look_ahead_poses, poses - 1 - cfg_->trajectory.prevent_look_ahead_poses_near_goal));
  const double horizon = cfg_->trajectory.dt_ref * target;
  double elapsed = 0.0;
  for (int k = 0; k < target; ++k) {
    elapsed += teb_.TimeDiff(k);
    if (elapsed >= horizon) { target = k + 1; break; }
  }
  if (elapsed <= 0) return false;
  extractVelocity(teb_.Pose(0), teb_.Pose(target), elapsed, vx, vy, omega);
  return true;
}

/* n + 1 twists for n poses (reference :1174-1200): the start velocity, the mean velocity of every segment, the goal velocity */
void TebOptimalPlanner::getVelocityProfile(std::vector<geometry_msgs::Twist>& velocity_profile) const {
  const int poses = teb_.sizePoses();
  velocity_profile.assign(poses + 1, geometry_msgs::Twist());
  auto boundary = [](geometry_msgs::Twist& out, const geometry_msgs::Twist& given) {
    out.linear.x = given.linear.x;
    out.linear.y = given.linear.y;
    out.angular.z = given.angular.z;
  };
  boundary(velocity_profile.front(), vel_start_.second);
  for (int k = 1; k < poses; ++k) {
    geometry_msgs::Twist& t = velocity_profile[k];
    extractVelocity(teb_.Pose(k - 1), teb_.Pose(k), teb_.TimeDiff(k - 1), t.linear.x, t.linear.y, t.angular.z);
  }
  boundary(velocity_profile.back(), vel_goal_.second);
}

}  // namespace teb_local_planner

namespace teb_local_planner {

/* optimal_planner.cpp:1197-1244 */
void TebOptimalPlanner::getFullTrajectory(std::vector<TrajectoryPointMsg>& trajectory) const {
  const int n = teb_.sizePoses();
  trajectory.resize(n);
  if (n == 0) return;
  auto fill_pose = [](const PoseSE2& p, geometry_msgs::Pose& out) {
    out.position.x = p.x(); out.position.y = p.y(); out.position.z = 0;
    out.orientation = tf::createQuaternionFromYaw(p.theta());
  };
  double curr_time = 0;
  fill_pose(teb_.Pose(0), trajectory.front().pose);
  trajectory.front().velocity = geometry_msgs::Twist();
  trajectory.front().velocity.linear.x = vel_start_.second.linear.x;
  trajectory.front().velocity.linear.y = vel_start_.second.linear.y;
  trajectory.front().velocity.angular.z = vel_start_.second.angular.z;
  trajectory.front().time_from_start = curr_time;
  if (n == 1) return;
  curr_time += teb_.TimeDiff(0);
  for (int i = 1; i < n - 1; ++i) { /* mean of the velocities of the two adjacent segments */
    TrajectoryPointMsg& point = trajectory[i];
    fill_pose(teb_.Pose(i), point.pose);
    double v1x, v1y, w1, v2x, v2y, w2;
    extractVelocity(teb_.Pose(i - 1), teb_.Pose(i), teb_.TimeDiff(i - 1), v1x, v1y, w1);
    extractVelocity(teb_.Pose(i), teb_.Pose(i + 1), teb_.TimeDiff(i), v2x, v2y, w2);
    point.velocity = geometry_msgs::Twist();
    point.velocity.linear.x = 0.5 * (v1x + v2x);
    point.velocity.linear.y = 0.5 * (v1y + v2y);
    point.velocity.angular.z = 0.5 * (w1 + w2);
    point.time_from_start = curr_time;
    curr_time += teb_.TimeDiff(i);
  }
  fill_pose(teb_.BackPose(), trajectory.back().pose);
  trajectory.back().velocity = geometry_msgs::Twist();
  trajectory.back().velocity.linear.x = vel_goal_.second.linear.x;
  trajectory.back().velocity.linear.y = vel_goal_.second.linear.y;
  trajectory.back().velocity.angular.z = vel_goal_.second.angular.z;
  trajectory.back().time_from_start = curr_time;
}

/* optimal_planner.cpp:1247-1306 */
bool TebOptimalPlanner::isTrajectoryFeasible(base_local_planner::CostmapModel* costmap_model,
                                             const std::vector<geometry_msgs::Point>& footprint_spec, double inscribed_radius,
                                             double circumscribed_radius, int look_ahead_idx,
                                             double feasibility_check_lookahead_distance) {
  if (!costmap_model || !cfg_) return false;
  if (look_ahead_idx < 0 || look_ahead_idx >= teb().sizePoses()) look_ahead_idx = teb().sizePoses() - 1;
  if (feasibility_check_lookahead_distance > 0) {
    for (int i = 1; i < teb().sizePoses(); ++i) {
      const double d = std::hypot(teb().Pose(i).x() - teb().Pose(0).x(), teb().Pose(i).y() - teb().Pose(0).y());
      if (d > feasibility_check_lookahead_distance) { look_ahead_idx = i - 1; break; }
    }
  }
  for (int i = 0; i <= look_ahead_idx; ++i) {
    const PoseSE2& pi = teb().Pose(i);
    if (costmap_model->footprintCost(pi.x(), pi.y(), pi.theta(), footprint_spec, inscribed_radius, circumscribed_radius) == -1) return false;
    if (i == look_ahead_idx) break;
    /* two consecutive poses pushed apart by an obstacle may straddle it: sample in between */
    const PoseSE2& pn = teb().Pose(i + 1);
    const double delta_rot = g2o::normalize_theta(g2o::normalize_theta(pn.theta()) - g2o::normalize_theta(pi.theta()));
    const Eigen::Vector2d delta_dist = pn.position() - pi.position();
    const double ang_res = cfg_->trajectory.min_resolution_collision_check_angular;
    if (std::fabs(delta_rot) > ang_res || delta_dist.norm() > inscribed_radius) {
      const int n_additional_samples =
          (int)std::max(std::ceil(std::fabs(delta_rot) / ang_res), std::ceil(delta_dist.norm() / inscribed_radius)) - 1;
      PoseSE2 mid = pi;
      for (int step = 0; step < n_additional_samples; ++step) {
        mid.position() = mid.position() + delta_dist / (n_additional_samples + 1.0);
        mid.theta() = g2o::normalize_theta(mid.theta() + delta_rot / (n_additional_samples + 1.0));
        if (costmap_model->footprintCost(mid.x(), mid.y(), mid.theta(), footprint_spec, inscribed_radius, circumscribed_radius) == -1)
          return false;
      }
    }
  }
  return true;
}

}  // namespace teb_local_planner
