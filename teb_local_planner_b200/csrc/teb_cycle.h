/*
 * teb_cycle.h — the controller steps around plan() for one band: the oscillation half of configureBackupModes with
 * FailureDetector, and the back half of computeVelocityCommands with saturateVelocity and
 * convertTransRotVelToSteeringAngle. One routine compiled for the host and for the device (k_backup_modes /
 * k_finish_cycle in teb_cycle.cuh), like teb_plan.h; the host entry points use the range checks below to refuse the
 * bands the device answers with TEB_CYCLE_NO_PLAN / oscillating = -1.
 *
 * Reference behaviour (the contract is at TebCycleArgs in include/teb_b200.h):
 *   configureBackupModes, oscillation half      src/teb_local_planner_ros.cpp:980-1016
 *   FailureDetector::update / detect            src/recovery_behaviors.cpp
 *   computeVelocityCommands after plan()        src/teb_local_planner_ros.cpp:360-454
 *   saturateVelocity                            src/teb_local_planner_ros.cpp:874-919
 *   convertTransRotVelToSteeringAngle           src/teb_local_planner_ros.cpp:922-933
 *
 * The detector's means are sums in the ring's order, so one thread walks a band's ring; the ring is band-minor
 * ([L_cap][B][2]) so that the threads of a warp read entry k of neighbouring bands together. Products and sums go
 * through teb_mul / teb_add, so FMA contraction cannot change a bit on the device.
 */
#ifndef TEB_CYCLE_H
#define TEB_CYCLE_H

#include <math.h>
#include <stdint.h>

#include "teb_plan.h" /* TEB_HD, teb_mul, teb_add, TEB_* codes */

/* the context parameters the two steps read */
struct TebCycleLimits {
  double max_vel_x, max_vel_x_backwards, max_vel_y, max_vel_trans, max_vel_theta, min_turning_radius;
  double divergence_max_chi2;
  int32_t divergence_enable;
};

/* g2o::sign: 0 for 0 and NaN */
TEB_HD inline int teb_cycle_sign(double x) { return x > 0 ? 1 : (x < 0 ? -1 : 0); }
/* std::min / std::max */
TEB_HD inline double teb_cycle_min(double a, double b) { return b < a ? b : a; }
TEB_HD inline double teb_cycle_max(double a, double b) { return a < b ? b : a; }

/* TebLocalPlannerROS::saturateVelocity */
TEB_HD inline void teb_cycle_saturate(double& vx, double& vy, double& omega, const TebCycleLimits& L, bool proportional) {
  double ratio_x = 1, ratio_omega = 1, ratio_y = 1;
  if (vx > L.max_vel_x) ratio_x = L.max_vel_x / vx;
  if (vy > L.max_vel_y || vy < -L.max_vel_y) ratio_y = fabs(L.max_vel_y / vy);
  if (omega > L.max_vel_theta || omega < -L.max_vel_theta) ratio_omega = fabs(L.max_vel_theta / omega);
  if (L.max_vel_x_backwards <= 0) {
  } else if (vx < -L.max_vel_x_backwards) {
    ratio_x = -L.max_vel_x_backwards / vx;
  }
  if (proportional) {
    const double ratio = teb_cycle_min(teb_cycle_min(ratio_x, ratio_y), ratio_omega);
    vx = teb_mul(vx, ratio); vy = teb_mul(vy, ratio); omega = teb_mul(omega, ratio);
  } else {
    vx = teb_mul(vx, ratio_x); vy = teb_mul(vy, ratio_y); omega = teb_mul(omega, ratio_omega);
  }
  const double vel_linear = hypot(vx, vy);
  if (vel_linear > L.max_vel_trans) {
    const double r = L.max_vel_trans / vel_linear;
    vx = teb_mul(vx, r); vy = teb_mul(vy, r);
  }
}

/* TebLocalPlannerROS::convertTransRotVelToSteeringAngle; min_radius = 0.95 * min_turning_radius */
TEB_HD inline double teb_cycle_steering(double v, double omega, double wheelbase, double min_radius) {
  if (omega == 0 || v == 0) return 0;
  double radius = v / omega;
  if (fabs(radius) < min_radius) radius = teb_mul((double)teb_cycle_sign(radius), min_radius);
  return atan(wheelbase / radius);
}

TEB_HD inline int teb_cycle_plan_result(const TebCycleArgs& a, int b) {
  return a.local_plan_result ? a.local_plan_result[b] : TEB_LOCAL_PLAN_PLANNED;
}

/* the band's inputs the backup step reads are in range (else oscillating = -1, nothing else written) */
TEB_HD inline bool teb_cycle_backup_valid(const TebCycleArgs& a, int b) {
  const int r = teb_cycle_plan_result(a, b);
  if (r < TEB_LOCAL_PLAN_PLANNED || r > TEB_LOCAL_PLAN_BAD_INPUT) return false;
  if (r != TEB_LOCAL_PLAN_PLANNED && r != TEB_LOCAL_PLAN_CAPACITY) return true; /* skipped, nothing else is read */
  const int rot = a.prefer_rotdir[b];
  if (rot < TEB_ROTDIR_NONE || rot > TEB_ROTDIR_RIGHT) return false;
  const int size = a.osc_fill[2 * b], head = a.osc_fill[2 * b + 1];
  return size >= 0 && size <= a.buffer_length && head >= 0 && (a.buffer_length == 0 ? head == 0 : head < a.buffer_length);
}

/* the band's inputs the finish step reads are in range (else TEB_CYCLE_NO_PLAN, nothing else written) */
TEB_HD inline bool teb_cycle_finish_valid(const TebCycleArgs& a, int b) {
  const int r = teb_cycle_plan_result(a, b);
  if (r < TEB_LOCAL_PLAN_PLANNED || r > TEB_LOCAL_PLAN_BAD_INPUT) return false;
  return !a.feasible || (a.feasible[b] >= -1 && a.feasible[b] <= 1);
}

/* FailureDetector::update + detect on band b's ring; returns isOscillating() */
TEB_HD inline bool teb_cycle_detector_update(const TebCycleArgs& a, int b, int B, double v, double omega, double v_max,
                                             double v_backwards_max, double omega_max) {
  const int cap = a.buffer_length;
  if (cap == 0) return false;
  if (v > 0 && v_max > 0)
    v /= v_max;
  else if (v < 0 && v_backwards_max > 0)
    v /= v_backwards_max;
  if (omega_max > 0) omega /= omega_max;
  int size = a.osc_fill[2 * b], head = a.osc_fill[2 * b + 1];
  int slot;
  if (size < cap) {
    slot = head + size; if (slot >= cap) slot -= cap;
    ++size;
  } else { /* full: the oldest entry is overwritten */
    slot = head;
    if (++head == cap) head = 0;
  }
  a.osc_ring[2 * ((size_t)slot * B + b)] = v;
  a.osc_ring[2 * ((size_t)slot * B + b) + 1] = omega;
  a.osc_fill[2 * b] = size; a.osc_fill[2 * b + 1] = head;
  if (size < cap / 2) return false;
  double v_mean = 0, omega_mean = 0, prev = 0;
  int crossings = 0;
  for (int i = 0, s = head; i < size; ++i) {
    const double* e = a.osc_ring + 2 * ((size_t)s * B + b);
    const double ev = e[0], eo = e[1];
    v_mean = teb_add(v_mean, ev);
    omega_mean = teb_add(omega_mean, eo);
    if (i > 0 && teb_cycle_sign(eo) != teb_cycle_sign(prev)) ++crossings;
    prev = eo;
    if (++s == cap) s = 0;
  }
  v_mean /= (double)size;
  omega_mean /= (double)size;
  return fabs(v_mean) < a.oscillation_v_eps && fabs(omega_mean) < a.oscillation_omega_eps && crossings > 1;
}

/* configureBackupModes' oscillation half for band b */
TEB_HD inline void teb_cycle_backup_band(const TebCycleArgs& a, const TebCycleLimits& L, int b, int B) {
  if (!teb_cycle_backup_valid(a, b)) {
    if (a.oscillating) a.oscillating[b] = -1;
    return;
  }
  const int r = teb_cycle_plan_result(a, b);
  if (r != TEB_LOCAL_PLAN_PLANNED && r != TEB_LOCAL_PLAN_CAPACITY) return;
  if (!a.oscillation_recovery) {
    if (a.oscillating) a.oscillating[b] = 0;
    return;
  }
  const double lvx = a.last_cmd[3 * (size_t)b], lom = a.last_cmd[3 * (size_t)b + 2];
  const double mvc = lvx >= 0 ? L.max_vel_x : L.max_vel_x_backwards;
  const double max_vel_theta = (L.min_turning_radius != 0 && mvc > 0)
                                   ? teb_cycle_max(mvc / fabs(L.min_turning_radius), L.max_vel_theta)
                                   : L.max_vel_theta;
  const bool osc = teb_cycle_detector_update(a, b, B, lvx, lom, L.max_vel_x, L.max_vel_x_backwards, max_vel_theta);
  const bool recently = teb_add(a.now, -a.last_oscillation[b]) < a.oscillation_recovery_min_duration;
  if (osc) {
    if (!recently) a.prefer_rotdir[b] = a.robot_vel[3 * (size_t)b + 2] > 0 ? TEB_ROTDIR_LEFT : TEB_ROTDIR_RIGHT;
    a.last_oscillation[b] = a.now;
  } else if (!recently && a.prefer_rotdir[b] != TEB_ROTDIR_NONE) {
    a.prefer_rotdir[b] = TEB_ROTDIR_NONE;
  }
  if (a.oscillating) a.oscillating[b] = osc ? 1 : 0;
}

/* computeVelocityCommands from plan() on, for band b */
TEB_HD inline void teb_cycle_finish_band(const TebCycleArgs& a, const TebCycleLimits& L, int32_t* n,
                                         const int32_t* status, const double* chi2, int b) {
  double* out = a.cmd_vel + 3 * (size_t)b;
  const int r = teb_cycle_plan_result(a, b);
  int outcome;
  double vx = 0, vy = 0, omega = 0;
  if (!teb_cycle_finish_valid(a, b) || r == TEB_LOCAL_PLAN_EMPTY || r == TEB_LOCAL_PLAN_CAPACITY ||
      r == TEB_LOCAL_PLAN_BAD_INPUT) {
    outcome = TEB_CYCLE_NO_PLAN;
  } else if (r == TEB_LOCAL_PLAN_GOAL_REACHED) {
    outcome = TEB_CYCLE_GOAL_REACHED;
    n[b] = 0;
  } else {
    const int st = status[b];
    const int fz = a.feasible ? a.feasible[b] : 1;
    const double* c = a.cmd + 4 * (size_t)b;
    if (!(st & TEB_STATUS_OPTIMIZED) || (st & (TEB_STATUS_CAPACITY | TEB_STATUS_BAD_INPUT)))
      outcome = TEB_CYCLE_PLAN_FAILED;
    else if (L.divergence_enable && chi2[b] > L.divergence_max_chi2)
      outcome = TEB_CYCLE_DIVERGED;
    else if (fz == 0)
      outcome = TEB_CYCLE_INFEASIBLE;
    else if (fz == -1)
      outcome = TEB_CYCLE_UNDECIDABLE;
    else if (c[3] == 0)
      outcome = TEB_CYCLE_INVALID_COMMAND;
    else {
      outcome = TEB_CYCLE_COMMAND;
      vx = c[0]; vy = c[1]; omega = c[2];
      teb_cycle_saturate(vx, vy, omega, L, a.use_proportional_saturation != 0);
      if (a.cmd_angle_instead_rotvel) {
        omega = teb_cycle_steering(vx, omega, a.wheelbase, teb_mul(0.95, L.min_turning_radius));
        if (!isfinite(omega)) { outcome = TEB_CYCLE_STEERING_NOT_FINITE; vx = vy = omega = 0; }
      }
    }
    if (outcome == TEB_CYCLE_COMMAND) {
      a.infeasible_count[b] = 0;
    } else {
      n[b] = 0;
      if (a.infeasible_count[b] < INT32_MAX) ++a.infeasible_count[b];
      a.last_infeasible[b] = a.now;
    }
    a.last_cmd[3 * (size_t)b] = vx; a.last_cmd[3 * (size_t)b + 1] = vy; a.last_cmd[3 * (size_t)b + 2] = omega;
  }
  out[0] = vx; out[1] = vy; out[2] = omega;
  a.outcome[b] = outcome;
}

#endif /* TEB_CYCLE_H */
