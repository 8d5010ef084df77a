/* homotopy_class_planner.cpp — see include/teb_local_planner/homotopy_class_planner.h. Line references:
 * src/homotopy_class_planner.cpp of the reference. */
#include "teb_local_planner/homotopy_class_planner.h"

#include <algorithm>
#include <limits>
#include <thread>

namespace teb_local_planner {

HomotopyClassPlanner::HomotopyClassPlanner() {}
HomotopyClassPlanner::HomotopyClassPlanner(const TebConfig& cfg, ObstContainer* obstacles, TebVisualizationPtr visual,
                                           const ViaPointContainer* via_points) {
  initialize(cfg, obstacles, visual, via_points);
}

/* :61-78 */
void HomotopyClassPlanner::initialize(const TebConfig& cfg, ObstContainer* obstacles, TebVisualizationPtr visual,
                                      const ViaPointContainer* via_points) {
  cfg_ = &cfg;
  obstacles_ = obstacles;
  via_points_ = via_points;
  visualization_ = visual;
  last_eq_class_switching_time_ = std::chrono::steady_clock::now();
  std::random_device rd; /* :73 */
  random_.seed(rd());
  /* :69-72 */
  if (cfg_->hcp.simple_exploration) graph_search_ = std::shared_ptr<GraphSearchInterface>(new lrKeyPointGraph(*cfg_, this));
  else graph_search_ = std::shared_ptr<GraphSearchInterface>(new ProbRoadmapGraph(*cfg_, this));
  initialized_ = true;
}

/* :85-96 */
bool HomotopyClassPlanner::plan(const std::vector<geometry_msgs::PoseStamped>& initial_plan, const geometry_msgs::Twist* start_vel,
                                bool free_goal_vel) {
  if (!initialized_ || initial_plan.empty()) return false;
  initial_plan_ = &initial_plan;
  PoseSE2 start(initial_plan.front().pose);
  PoseSE2 goal(initial_plan.back().pose);
  return plan(start, goal, start_vel, free_goal_vel);
}
bool HomotopyClassPlanner::plan(const tf::Pose& start, const tf::Pose& goal, const geometry_msgs::Twist* start_vel, bool free_goal_vel) {
  PoseSE2 start_pose(start);
  PoseSE2 goal_pose(goal);
  return plan(start_pose, goal_pose, start_vel, free_goal_vel);
}

/* :107-125 */
bool HomotopyClassPlanner::plan(const PoseSE2& start, const PoseSE2& goal, const geometry_msgs::Twist* start_vel, bool free_goal_vel) {
  if (!initialized_) return false;
  if (obstacles_ && obstacles_->size() > 1024) { /* the H-signature's product over the obstacles leaves the double range */
    std::fprintf(stderr, "HomotopyClassPlanner: more than 1024 obstacles per scene is not supported (H-signature)\n");
    return false;
  }
  updateAllTEBs(&start, &goal, start_vel);
  exploreEquivalenceClassesAndInitTebs(start, goal, cfg_->obstacles.min_obstacle_dist, start_vel, free_goal_vel);
  updateReferenceTrajectoryViaPoints(cfg_->hcp.viapoints_all_candidates);
  optimizeAllTEBs(cfg_->optim.no_inner_iterations, cfg_->optim.no_outer_iterations);
  selectBestTeb();
  initial_plan_ = nullptr;
  return true;
}

/* Which candidates are pulled towards the via-points (reference :304-335). Nothing changes when there is nothing to
 * attach (no via-points, weight <= 0) or - in the "initial plan only" mode - when this cycle has no initial plan. Otherwise
 * every candidate gets them, or exactly those whose equivalence class equals the class of the initial plan: the class is
 * compared, not the band object, because from the second cycle on an older band usually holds that class already. */
void HomotopyClassPlanner::updateReferenceTrajectoryViaPoints(bool all_trajectories) {
  const bool nothing_to_attach = !via_points_ || via_points_->empty() || cfg_->optim.weight_viapoint <= 0;
  if (nothing_to_attach || (!all_trajectories && !initial_plan_)) return;
  if (equivalence_classes_.size() < tebs_.size()) return; /* classes and bands out of step: leave the assignment alone */
  for (size_t k = 0; k < tebs_.size(); ++k) {
    bool attach = all_trajectories;
    if (!attach && initial_plan_eq_class_ && equivalence_classes_[k].first)
      attach = initial_plan_eq_class_->isEqual(*equivalence_classes_[k].first);
    tebs_[k]->setViaPoints(attach ? via_points_ : NULL);
  }
}

bool HomotopyClassPlanner::getVelocityCommand(double& vx, double& vy, double& omega, int look_ahead_poses) const {
  TebOptimalPlannerConstPtr best_teb = bestTeb();
  if (!best_teb) { vx = 0; vy = 0; omega = 0; return false; }
  return best_teb->getVelocityCommand(vx, vy, omega, look_ahead_poses);
}

/* ------------------------------------------------------------------ equivalence classes
 * calculateEquivalenceClass (homotopy_class_planner.hpp:46-63) for a set of candidates = ONE tebgpu_h_signature call */
std::vector<EquivalenceClassPtr> HomotopyClassPlanner::calculateEquivalenceClasses(const std::vector<TebOptimalPlanner*>& planners) {
  std::vector<EquivalenceClassPtr> out(planners.size());
  if (planners.empty()) return out;
  std::vector<std::vector<double>> values;
  if (!TebOptimalPlanner::hSignatureBatch(*cfg_, planners, gpu_, values)) return out; /* null classes: never "new" (:191) */
  for (size_t k = 0; k < planners.size(); ++k) {
    if (cfg_->obstacles.include_dynamic_obstacles) out[k] = EquivalenceClassPtr(new HSignature3d(*cfg_, values[k]));
    else out[k] = EquivalenceClassPtr(new HSignature(*cfg_, std::complex<double>(values[k][0], values[k][1])));
  }
  return out;
}
EquivalenceClassPtr HomotopyClassPlanner::calculateEquivalenceClass(TebOptimalPlanner* planner) {
  return calculateEquivalenceClasses(std::vector<TebOptimalPlanner*>(1, planner))[0];
}

/* :178-187 */
bool HomotopyClassPlanner::hasEquivalenceClass(const EquivalenceClassPtr& eq_class) const {
  for (const std::pair<EquivalenceClassPtr, bool>& eqrel : equivalence_classes_)
    if (eq_class->isEqual(*eqrel.first)) return true;
  return false;
}
/* :387-412 */
bool HomotopyClassPlanner::isInBestTebClass(const EquivalenceClassPtr& eq_class) const {
  return best_teb_eq_class_ ? best_teb_eq_class_->isEqual(*eq_class) : false;
}
int HomotopyClassPlanner::numTebsInClass(const EquivalenceClassPtr& eq_class) const {
  int count = 0;
  for (const std::pair<EquivalenceClassPtr, bool>& eqrel : equivalence_classes_)
    if (eq_class->isEqual(*eqrel.first)) ++count;
  return count;
}
int HomotopyClassPlanner::numTebsInBestTebClass() const { return best_teb_eq_class_ ? numTebsInClass(best_teb_eq_class_) : 0; }

/* :189-211 */
bool HomotopyClassPlanner::addEquivalenceClassIfNew(const EquivalenceClassPtr& eq_class, bool lock) {
  if (!eq_class) return false;
  if (!eq_class->isValid()) return false; /* invalid H-signature: ignored */
  if (hasEquivalenceClass(eq_class)) {
    /* up to max_number_plans_in_current_class bands may share the class of the current best band */
    if (!isInBestTebClass(eq_class) || numTebsInBestTebClass() >= cfg_->hcp.max_number_plans_in_current_class) return false;
  }
  equivalence_classes_.push_back(std::make_pair(eq_class, lock));
  return true;
}

/* :214-256: signatures of all existing bands (one device call), then first come first serve with the last best band
 * first; bands whose class is already taken are dropped */
void HomotopyClassPlanner::renewAndAnalyzeOldTebs(bool delete_detours) {
  equivalence_classes_.clear();
  if (tebs_.empty()) return;
  auto it_best_teb = best_teb_ ? std::find(tebs_.begin(), tebs_.end(), best_teb_) : tebs_.end();
  const bool has_best_teb = it_best_teb != tebs_.end();
  if (has_best_teb) std::iter_swap(tebs_.begin(), it_best_teb);
  std::vector<TebOptimalPlanner*> all;
  for (auto& teb : tebs_) all.push_back(teb.get());
  std::vector<EquivalenceClassPtr> classes = calculateEquivalenceClasses(all);
  size_t k = 0;
  auto it_teb = tebs_.begin();
  if (has_best_teb) {
    best_teb_eq_class_ = classes[0];
    addEquivalenceClassIfNew(best_teb_eq_class_);
    ++it_teb; ++k;
  }
  while (it_teb != tebs_.end()) {
    if (!addEquivalenceClassIfNew(classes[k++])) { it_teb = tebs_.erase(it_teb); continue; }
    ++it_teb;
  }
  if (delete_detours)
    deletePlansDetouringBackwards(cfg_->hcp.detours_orientation_tolerance, cfg_->hcp.length_start_orientation_vector);
}

/* :803-838: direction from the first pose that is farther than len_orientation_vector from the start, to the start */
bool HomotopyClassPlanner::computeStartOrientation(const TebOptimalPlannerPtr plan, const double len_orientation_vector,
                                                   double& orientation) {
  const PoseSE2 start_pose = plan->teb().Pose(0);
  Eigen::Vector2d start_vector;
  bool second_pose_found = false;
  for (int i = 0; i < plan->teb().sizePoses(); ++i) {
    start_vector = start_pose.position() - plan->teb().Pose(i).position();
    if (start_vector.norm() > len_orientation_vector) { second_pose_found = true; break; }
  }
  if (!second_pose_found) return false; /* too short to tell */
  orientation = std::atan2(start_vector[1], start_vector[0]);
  return true;
}

/* :766-801 */
void HomotopyClassPlanner::deletePlansDetouringBackwards(const double orient_threshold, const double len_orientation_vector) {
  if (tebs_.size() < 2 || !best_teb_ || std::find(tebs_.begin(), tebs_.end(), best_teb_) == tebs_.end() ||
      best_teb_->teb().sizePoses() < 2)
    return; /* no direction of motion chosen yet */
  double current_movement_orientation;
  const double best_plan_duration = std::max(best_teb_->teb().getSumOfAllTimeDiffs(), 1.0);
  if (!computeStartOrientation(best_teb_, len_orientation_vector, current_movement_orientation)) return;
  for (auto it_teb = tebs_.begin(); it_teb != tebs_.end();) {
    if (*it_teb == best_teb_) { ++it_teb; continue; }
    double plan_orientation;
    const bool drop = (*it_teb)->teb().sizePoses() < 2 || !computeStartOrientation(*it_teb, len_orientation_vector, plan_orientation) ||
                      std::fabs(g2o::normalize_theta(plan_orientation - current_movement_orientation)) > orient_threshold ||
                      !(*it_teb)->isOptimized() ||
                      (*it_teb)->teb().getSumOfAllTimeDiffs() / best_plan_duration > cfg_->hcp.max_ratio_detours_duration_best_duration;
    if (drop) { TebOptimalPlannerPtr victim = *it_teb; it_teb = removeTeb(victim); continue; }
    ++it_teb;
  }
}

/* :539-562 */
void HomotopyClassPlanner::randomlyDropTebs() {
  if (cfg_->hcp.selection_dropping_probability == 0.0) return;
  auto it_eqrel = equivalence_classes_.begin();
  auto it_teb = tebs_.begin();
  while (it_teb != tebs_.end() && it_eqrel != equivalence_classes_.end()) {
    if (it_teb->get() != best_teb_.get() &&
        (double)random_() <= cfg_->hcp.selection_dropping_probability * (double)random_.max()) {
      it_teb = tebs_.erase(it_teb);
      it_eqrel = equivalence_classes_.erase(it_eqrel);
    } else {
      ++it_teb;
      ++it_eqrel;
    }
  }
}

/* :337-357 — renew the classes of the existing bands, inject the initial plan, explore further classes */
void HomotopyClassPlanner::exploreEquivalenceClassesAndInitTebs(const PoseSE2& start, const PoseSE2& goal, double dist_to_obst,
                                                                const geometry_msgs::Twist* start_vel, bool free_goal_vel) {
  (void)dist_to_obst;
  renewAndAnalyzeOldTebs(cfg_->hcp.delete_detours_backwards);
  randomlyDropTebs();
  if (initial_plan_) {
    initial_plan_teb_ = addAndInitNewTeb(*initial_plan_, start_vel, free_goal_vel);
  } else {
    initial_plan_teb_.reset();
    initial_plan_teb_ = getInitialPlanTEB();
  }
  graph_search_->createGraph(start, goal, dist_to_obst, cfg_->hcp.obstacle_heading_threshold, start_vel, free_goal_vel);
}

/* homotopy_class_planner.hpp:67-100, chunked */
bool HomotopyClassPlanner::addAndInitNewTebs(const std::vector<std::vector<Eigen::Vector2d>>& paths, double start_orientation,
                                             double goal_orientation, const geometry_msgs::Twist* start_velocity, bool free_goal_vel) {
  if ((int)tebs_.size() >= cfg_->hcp.max_number_classes) return true;
  std::vector<TebOptimalPlannerPtr> cands;
  std::vector<TebOptimalPlanner*> raw;
  for (const std::vector<Eigen::Vector2d>& path : paths) {
    TebOptimalPlannerPtr candidate(new TebOptimalPlanner(*cfg_, obstacles_));
    candidate->setGpuContext(gpu_);
    if (robot_model_) candidate->updateRobotModel(robot_model_);
    candidate->teb().initTrajectoryToGoal(path, cfg_->robot.max_vel_x, cfg_->robot.max_vel_theta, &cfg_->robot.acc_lim_x,
                                          &cfg_->robot.acc_lim_theta, &start_orientation, &goal_orientation,
                                          cfg_->trajectory.min_samples, cfg_->trajectory.allow_init_with_backwards_motion);
    if (start_velocity) candidate->setVelocityStart(*start_velocity);
    if (free_goal_vel) candidate->setVelocityGoalFree();
    cands.push_back(candidate);
    raw.push_back(candidate.get());
  }
  std::vector<EquivalenceClassPtr> classes = calculateEquivalenceClasses(raw);
  bool ok = true;
  for (size_t k = 0; k < cands.size(); ++k) {
    if ((int)tebs_.size() >= cfg_->hcp.max_number_classes) break;
    if (!classes[k]) { ok = false; break; }
    if (addEquivalenceClassIfNew(classes[k])) tebs_.push_back(cands[k]);
  }
  return ok;
}

/* :359-386 */
TebOptimalPlannerPtr HomotopyClassPlanner::addAndInitNewTeb(const PoseSE2& start, const PoseSE2& goal,
                                                            const geometry_msgs::Twist* start_velocity, bool free_goal_vel) {
  if ((int)tebs_.size() >= cfg_->hcp.max_number_classes) return TebOptimalPlannerPtr();
  TebOptimalPlannerPtr candidate(new TebOptimalPlanner(*cfg_, obstacles_, visualization_));
  candidate->setGpuContext(gpu_);
  if (robot_model_) candidate->updateRobotModel(robot_model_);
  candidate->teb().initTrajectoryToGoal(start, goal, 0, cfg_->robot.max_vel_x, cfg_->trajectory.min_samples,
                                        cfg_->trajectory.allow_init_with_backwards_motion);
  if (start_velocity) candidate->setVelocityStart(*start_velocity);
  if (free_goal_vel) candidate->setVelocityGoalFree();
  /* keep the candidate only if it opens a new class (:370-385) */
  EquivalenceClassPtr H = calculateEquivalenceClass(candidate.get());
  if (addEquivalenceClassIfNew(H)) {
    tebs_.push_back(candidate);
    return tebs_.back();
  }
  return TebOptimalPlannerPtr();
}

/* :414-441 */
TebOptimalPlannerPtr HomotopyClassPlanner::addAndInitNewTeb(const std::vector<geometry_msgs::PoseStamped>& initial_plan,
                                                            const geometry_msgs::Twist* start_velocity, bool free_goal_vel) {
  if ((int)tebs_.size() >= cfg_->hcp.max_number_classes) return TebOptimalPlannerPtr();
  TebOptimalPlannerPtr candidate(new TebOptimalPlanner(*cfg_, obstacles_, visualization_));
  candidate->setGpuContext(gpu_);
  if (robot_model_) candidate->updateRobotModel(robot_model_);
  candidate->teb().initTrajectoryToGoal(initial_plan, cfg_->robot.max_vel_x, cfg_->robot.max_vel_theta,
                                        cfg_->trajectory.global_plan_overwrite_orientation, cfg_->trajectory.min_samples,
                                        cfg_->trajectory.allow_init_with_backwards_motion);
  if (start_velocity) candidate->setVelocityStart(*start_velocity);
  if (free_goal_vel) candidate->setVelocityGoalFree();
  /* the class of the initial plan is stored and locked (:430-440) */
  initial_plan_eq_class_ = calculateEquivalenceClass(candidate.get());
  if (addEquivalenceClassIfNew(initial_plan_eq_class_, true)) {
    tebs_.push_back(candidate);
    return tebs_.back();
  }
  return TebOptimalPlannerPtr();
}

/* :443-463 */
void HomotopyClassPlanner::updateAllTEBs(const PoseSE2* start, const PoseSE2* goal, const geometry_msgs::Twist* start_velocity) {
  if (!tebs_.empty() &&
      ((goal->position() - tebs_.front()->teb().BackPose().position()).norm() >= cfg_->trajectory.force_reinit_new_goal_dist ||
       std::fabs(g2o::normalize_theta(goal->theta() - tebs_.front()->teb().BackPose().theta())) >=
           cfg_->trajectory.force_reinit_new_goal_angular)) {
    tebs_.clear();
    equivalence_classes_.clear();
    initial_plan_teb_.reset();
  }
  for (auto& teb : tebs_) {
    teb->teb().updateAndPruneTEB(*start, *goal);
    if (start_velocity) teb->setVelocityStart(*start_velocity);
  }
}

/* :466-493 — the per-candidate boost::thread fan-out becomes ONE batched launch sequence over all candidates. With
 * several device contexts (setGpuContexts) the candidates are split contiguously over the devices, one host thread per
 * device drives its shard, and the join of those threads is the point where every cost is known - the in-process
 * counterpart of the NCCL all-gather that separate processes use (tebgpu_gather_costs). */
void HomotopyClassPlanner::optimizeAllTEBs(int iter_innerloop, int iter_outerloop) {
  if (tebs_.empty() || !cfg_->optim.optimization_activate) return;
  std::vector<TebOptimalPlanner*> all;
  for (auto& teb : tebs_) all.push_back(teb.get());
  const size_t devices = std::min(gpus_.size(), all.size());
  if (devices <= 1) {
    optimizeTebBatch(*cfg_, all, iter_innerloop, iter_outerloop, true, cfg_->hcp.selection_obst_cost_scale,
                     cfg_->hcp.selection_viapoint_cost_scale, cfg_->hcp.selection_alternative_time_cost,
                     gpus_.empty() ? gpu_ : gpus_.front());
    return;
  }
  std::vector<std::thread> workers;
  for (size_t d = 0; d < devices; ++d) {
    const size_t lo = all.size() * d / devices, hi = all.size() * (d + 1) / devices;
    workers.emplace_back([this, &all, lo, hi, d, iter_innerloop, iter_outerloop]() {
      const std::vector<TebOptimalPlanner*> shard(all.begin() + lo, all.begin() + hi);
      optimizeTebBatch(*cfg_, shard, iter_innerloop, iter_outerloop, true, cfg_->hcp.selection_obst_cost_scale,
                       cfg_->hcp.selection_viapoint_cost_scale, cfg_->hcp.selection_alternative_time_cost, gpus_[d]);
    });
  }
  for (std::thread& w : workers) w.join();
}

namespace {
/* position of a band in the container, -1 when it is not (or no longer) part of it */
int index_of(const TebOptPlannerContainer& bands, const TebOptimalPlannerPtr& band) {
  if (!band) return -1;
  for (size_t k = 0; k < bands.size(); ++k)
    if (bands[k] == band) return (int)k;
  return -1;
}
}  // namespace

/* The candidate that follows the initial plan (reference :495-537): the band created from it in this cycle if it
 * survived the filtering, otherwise the first band whose equivalence class is the plan's class. */
TebOptimalPlannerPtr HomotopyClassPlanner::getInitialPlanTEB() {
  if (index_of(tebs_, initial_plan_teb_) >= 0) return initial_plan_teb_;
  initial_plan_teb_.reset();
  const bool comparable = initial_plan_eq_class_ && equivalence_classes_.size() == tebs_.size();
  if (!comparable) return TebOptimalPlannerPtr();
  for (size_t k = 0; k < tebs_.size(); ++k)
    if (equivalence_classes_[k].first->isEqual(*initial_plan_eq_class_)) return tebs_[k];
  return TebOptimalPlannerPtr();
}

/* Best candidate of the cycle (reference :564-667). The comparison itself is the boundary function tebgpu_select_best on
 * the candidates' costs: the previous winner competes with cost x selection_cost_hysteresis, the initial-plan candidate
 * with cost x selection_prefer_initial_plan, strict '<', first minimum wins. A change of winner is only honoured once
 * switching_blocking_period seconds have passed since the last change. */
TebOptimalPlannerPtr HomotopyClassPlanner::selectBestTeb() {
  const int previous = index_of(tebs_, best_teb_);
  last_best_teb_ = previous >= 0 ? best_teb_ : TebOptimalPlannerPtr();
  const int from_plan = index_of(tebs_, getInitialPlanTEB());
  std::vector<double> cost(tebs_.size());
  for (size_t k = 0; k < tebs_.size(); ++k) cost[k] = tebs_[k]->getCurrentCost();
  const int winner = tebgpu_select_best(cost.data(), (int32_t)cost.size(), previous, from_plan, cfg_->hcp.selection_cost_hysteresis,
                                        cfg_->hcp.selection_prefer_initial_plan);
  best_teb_ = winner >= 0 ? tebs_[winner] : TebOptimalPlannerPtr();
  if (last_best_teb_ && best_teb_ != last_best_teb_) {
    const auto now = std::chrono::steady_clock::now();
    const double since_last_switch = std::chrono::duration<double>(now - last_eq_class_switching_time_).count();
    if (since_last_switch > cfg_->hcp.switching_blocking_period) last_eq_class_switching_time_ = now;
    else best_teb_ = last_best_teb_; /* still blocked: keep the previous winner */
  }
  return best_teb_;
}

/* index of the current winner; a single candidate always wins (reference :669-683) */
int HomotopyClassPlanner::bestTebIdx() const {
  return tebs_.size() == 1 ? 0 : index_of(tebs_, best_teb_);
}

TebOptPlannerContainer::iterator HomotopyClassPlanner::removeTeb(TebOptimalPlannerPtr& teb) {
  /* classes and bands are parallel containers (:686-707) */
  size_t idx = 0;
  for (auto it = tebs_.begin(); it != tebs_.end(); ++it, ++idx)
    if (*it == teb) {
      if (equivalence_classes_.size() == tebs_.size()) equivalence_classes_.erase(equivalence_classes_.begin() + idx);
      return tebs_.erase(it);
    }
  return tebs_.end();
}

void HomotopyClassPlanner::clearPlanner() {
  tebs_.clear();
  equivalence_classes_.clear();
  best_teb_eq_class_.reset();
  initial_plan_eq_class_.reset();
  best_teb_.reset();
  last_best_teb_.reset();
  initial_plan_teb_.reset();
  initial_plan_ = nullptr;
}

void HomotopyClassPlanner::setPreferredTurningDir(RotType dir) {
  for (auto& teb : tebs_) teb->setPreferredTurningDir(dir);
}

/* the stored winner while it is still a candidate, otherwise a fresh selection (reference :709-714) */
TebOptimalPlannerPtr HomotopyClassPlanner::findBestTeb() {
  if (tebs_.empty()) return TebOptimalPlannerPtr();
  if (index_of(tebs_, best_teb_) < 0) best_teb_ = selectBestTeb();
  return best_teb_;
}

/* Feasibility of the plan that will be executed (reference :686-707): the winner is checked against the costmap; an
 * infeasible winner is discarded and the next best candidate takes its place - unless the discarded one was already the
 * previous cycle's winner: then the call fails instead of letting the robot flip between plans. */
bool HomotopyClassPlanner::isTrajectoryFeasible(base_local_planner::CostmapModel* costmap_model,
                                                const std::vector<geometry_msgs::Point>& footprint_spec, double inscribed_radius,
                                                double circumscribed_radius, int look_ahead_idx,
                                                double feasibility_check_lookahead_distance) {
  while (!tebs_.empty()) {
    TebOptimalPlannerPtr candidate = findBestTeb();
    if (!candidate) return false;
    if (candidate->isTrajectoryFeasible(costmap_model, footprint_spec, inscribed_radius, circumscribed_radius, look_ahead_idx,
                                        feasibility_check_lookahead_distance))
      return true;
    const bool was_previous_winner = last_best_teb_ && last_best_teb_ == candidate;
    removeTeb(candidate);
    if (was_previous_winner) return false;
  }
  return false;
}

bool HomotopyClassPlanner::hasDiverged() const {
  if (!best_teb_) return false;
  return best_teb_->hasDiverged();
}

void HomotopyClassPlanner::computeCurrentCost(std::vector<double>& cost, double obst_cost_scale, double viapoint_cost_scale,
                                              bool alternative_time_cost) {
  for (auto& teb : tebs_) {
    teb->computeCurrentCost(obst_cost_scale, viapoint_cost_scale, alternative_time_cost);
    cost.push_back(teb->getCurrentCost());
  }
}

}  // namespace teb_local_planner
