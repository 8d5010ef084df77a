/*
 * teb_plan.h — the band bookkeeping TebOptimalPlanner::plan does around optimizeTEB, and getVelocityCommand, on packed
 * pose records. One routine compiled for the host and for the device (k_plan_begin / k_velocity_command in
 * teb_plan.cuh), like teb_resize.h.
 *
 * Reference behaviour:
 *   plan(start, goal) / plan(initial_plan)     src/optimal_planner.cpp:247-321 (path decision :259-269, :300-309)
 *   initTrajectoryToGoal(start, goal, 0, ...)  src/timed_elastic_band.cpp:325-387
 *   initTrajectoryToGoal(plan, ...)            src/timed_elastic_band.cpp:389-452
 *   updateAndPruneTEB                          src/timed_elastic_band.cpp:555-597 (the search and the shift are
 *                                              spread over a warp in k_plan_begin; the distance is teb_plan_dist)
 *   getVelocityCommand / extractVelocity       src/optimal_planner.cpp:1097-1168
 *   getVelocityProfile / getFullTrajectory     src/optimal_planner.cpp:1170-1248 (teb_extract_velocity per segment,
 *                                              spread over a warp in k_read_trajectory)
 *
 * Record layout as in teb_resize.h: rec[4*i+0..3] = x_i, y_i, theta_i, dt_i; record n-1 has dt = 0.
 *
 * The host layer is compiled without FMA contraction. Every product and sum a decision depends on (goal distance and
 * angle of the re-initialisation test, the prune distances, the backwards-motion guess) is written with explicit
 * round-to-nearest operations, so contraction cannot move a decision on the device either.
 */
#ifndef TEB_PLAN_H
#define TEB_PLAN_H

#include <math.h>

#include "../../include/teb_b200.h" /* TEB_PLAN_PATH_* */
#include "teb_resize.h"             /* TEB_HD, teb_average_angle */

TEB_HD inline double teb_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
TEB_HD inline double teb_add(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

/* g2o::normalize_theta */
TEB_HD inline double teb_normalize_theta(double theta) {
  if (theta >= -M_PI && theta < M_PI) return theta;
  const double multiplier = floor(theta / (2 * M_PI));
  theta = teb_add(theta, -teb_mul(teb_mul(multiplier, 2.0), M_PI));
  if (theta >= M_PI) theta -= 2 * M_PI;
  if (theta < -M_PI) theta += 2 * M_PI;
  return theta;
}

/* (a - b).norm() of two positions */
TEB_HD inline double teb_plan_dist(double ax, double ay, double bx, double by) {
  const double dx = ax - bx, dy = ay - by;
  return sqrt(teb_add(teb_mul(dx, dx), teb_mul(dy, dy)));
}

/* the heading a plan point carries: tf::createQuaternionFromYaw followed by tf::getYaw, as PoseSE2(PoseStamped.pose)
 * reads it back (qx = qy = 0) */
TEB_HD inline double teb_plan_yaw(double yaw) {
  const double qz = sin(yaw / 2), qw = cos(yaw / 2);
  return atan2(2.0 * teb_add(teb_mul(qw, qz), teb_mul(0.0, 0.0)), 1.0 - 2.0 * teb_add(teb_mul(0.0, 0.0), teb_mul(qz, qz)));
}

/* which branch plan() takes for a band of n poses and the new goal g[3]: cold start when the band is empty, warm start
 * when the goal moved less than force_reinit_new_goal_dist and turned less than force_reinit_new_goal_angular (both
 * strict), otherwise re-initialisation */
TEB_HD inline int teb_plan_path(const double* rec, int n, const double* g, double reinit_dist, double reinit_angular) {
  if (n <= 0) return TEB_PLAN_PATH_COLD;
  const double* back = rec + 4 * (n - 1);
  const bool near = teb_plan_dist(g[0], g[1], back[0], back[1]) < reinit_dist &&
                    fabs(teb_normalize_theta(g[2] - back[2])) < reinit_angular;
  return near ? TEB_PLAN_PATH_WARM : TEB_PLAN_PATH_REINIT;
}

/* initTrajectoryToGoal(start, goal, diststep = 0, max_vel_x, min_samples, ...): the start, midpoints towards the goal
 * until min_samples - 1 poses, the goal. With diststep = 0 the backwards-motion guess plays no part. Returns the new n,
 * or -1 (nothing written) when the band would need more than n_cap records. */
TEB_HD inline int teb_init_to_goal_records(double* rec, int n_cap, const double* s, const double* g, double max_vel_x,
                                           int min_samples) {
  const int n = (min_samples - 1 > 1 ? min_samples - 1 : 1) + 1;
  if (n > n_cap) return -1;
  double bx = s[0], by = s[1], bt = s[2], step = 0.1;
  rec[0] = bx; rec[1] = by; rec[2] = bt;
  int k = 1;
  for (; k < min_samples - 1; ++k) {
    const double mx = (bx + g[0]) / 2, my = (by + g[1]) / 2, mt = teb_average_angle(bt, g[2]);
    if (max_vel_x > 0) step = teb_plan_dist(mx, my, bx, by) / max_vel_x;
    rec[4 * (k - 1) + 3] = step;
    rec[4 * k] = mx; rec[4 * k + 1] = my; rec[4 * k + 2] = mt;
    bx = mx; by = my; bt = mt;
  }
  if (max_vel_x > 0) step = teb_plan_dist(g[0], g[1], bx, by) / max_vel_x;
  rec[4 * (k - 1) + 3] = step;
  rec[4 * k] = g[0]; rec[4 * k + 1] = g[1]; rec[4 * k + 2] = g[2]; rec[4 * k + 3] = 0.0;
  return k + 1;
}

/* time to go from pose a to pose b at (v_max, w_max), translation and rotation concurrently (estimateDeltaT) */
TEB_HD inline double teb_travel_time(const double* a, const double* b, double v_max, double w_max) {
  double t = 0.1;
  if (v_max > 0) t = teb_plan_dist(b[0], b[1], a[0], a[1]) / v_max;
  if (w_max > 0) {
    const double tw = fabs(teb_normalize_theta(b[2] - a[2])) / w_max;
    if (t < tw) t = tw;
  }
  return t;
}

/* initTrajectoryToGoal(plan, max_vel_x, max_vel_theta, estimate_orient, min_samples, guess_backwards_motion) over the
 * P rows (x, y, yaw) of `plan`: the first point, every inner point (heading from the plan, or towards the next point
 * and turned by pi for a guessed backwards motion), midpoints towards the last point up to min_samples - 1 poses, the
 * last point. Returns the new n, or -1 (nothing written) when the band would need more than n_cap records. */
TEB_HD inline int teb_init_from_plan_records(double* rec, int n_cap, const double* plan, int P, double max_vel_x,
                                             double max_vel_theta, int estimate_orient, int min_samples,
                                             int guess_backwards_motion) {
  const int head = P - 1 > 1 ? P - 1 : 1; /* the first point and the inner points */
  const int n = (head > min_samples - 1 ? head : min_samples - 1) + 1;
  if (n > n_cap) return -1;
  const double first[3] = {plan[0], plan[1], teb_plan_yaw(plan[2])};
  const double* lp = plan + 3 * (P - 1);
  const double last[3] = {lp[0], lp[1], teb_plan_yaw(lp[2])};
  const double fx = last[0] - first[0], fy = last[1] - first[1];
  const bool reversed = guess_backwards_motion && teb_add(teb_mul(fx, cos(first[2])), teb_mul(fy, sin(first[2]))) < 0;
  rec[0] = first[0]; rec[1] = first[1]; rec[2] = first[2];
  int k = 1;
  auto append = [&](double x, double y, double th) {
    double* r = rec + 4 * k;
    r[0] = x; r[1] = y; r[2] = th;
    r[-1] = teb_travel_time(r - 4, r, max_vel_x, max_vel_theta);
    ++k;
  };
  for (int i = 1; i < P - 1; ++i) {
    const double* here = plan + 3 * i;
    double heading = teb_plan_yaw(here[2]);
    if (estimate_orient) {
      heading = atan2(here[4] - here[1], here[3] - here[0]);
      if (reversed) heading = teb_normalize_theta(heading + M_PI);
    }
    append(here[0], here[1], heading);
  }
  while (k < min_samples - 1) {
    const double* back = rec + 4 * (k - 1);
    append((back[0] + last[0]) / 2, (back[1] + last[1]) / 2, teb_average_angle(back[2], last[2]));
  }
  append(last[0], last[1], last[2]);
  rec[4 * (k - 1) + 3] = 0.0;
  return k;
}

/* extractVelocity(pose1, pose2, dt) (optimal_planner.cpp:1097-1133) of the records p1, p2: v[0..2] = vx, vy, omega.
 * dt == 0 gives zeros. max_vel_y == 0 (non-holonomic): vx is the step length signed by the step's projection on p1's
 * heading (g2o::sign(0) == 0), vy = 0; otherwise the step in p1's frame over dt. */
TEB_HD inline void teb_extract_velocity(const double* p1, const double* p2, double dt, double max_vel_y, double* v) {
  v[0] = v[1] = v[2] = 0;
  if (dt == 0) return;
  const double sx = p2[0] - p1[0], sy = p2[1] - p1[1];
  const double c = cos(p1[2]), s = sin(p1[2]);
  const double along = teb_add(teb_mul(c, sx), teb_mul(s, sy));
  if (max_vel_y == 0) {
    const double sign = along > 0 ? 1.0 : (along < 0 ? -1.0 : 0.0);
    v[0] = teb_mul(sign, sqrt(teb_add(teb_mul(sx, sx), teb_mul(sy, sy)))) / dt;
  } else {
    v[0] = along / dt;
    v[1] = teb_add(teb_mul(-s, sx), teb_mul(c, sy)) / dt;
  }
  v[2] = teb_normalize_theta(p2[2] - p1[2]) / dt;
}

/* getVelocityCommand(vx, vy, omega, look_ahead_poses) on a band of n poses: v[0..2] = vx, vy, omega; returns the
 * command's validity (0 with zeros for fewer than 2 poses or a non-positive accumulated time) */
TEB_HD inline int teb_velocity_command(const double* rec, int n, int look_ahead_poses, int prevent_near_goal, double dt_ref,
                                       double max_vel_y, double* v) {
  v[0] = v[1] = v[2] = 0;
  if (n < 2) return 0;
  int target = look_ahead_poses < n - 1 - prevent_near_goal ? look_ahead_poses : n - 1 - prevent_near_goal;
  if (target < 1) target = 1;
  double dt = 0.0;
  for (int k = 0; k < target; ++k) {
    dt += rec[4 * k + 3];
    if (dt >= dt_ref * target) { target = k + 1; break; }
  }
  if (dt <= 0) return 0;
  teb_extract_velocity(rec, rec + 4 * target, dt, max_vel_y, v);
  return 1;
}

#endif
