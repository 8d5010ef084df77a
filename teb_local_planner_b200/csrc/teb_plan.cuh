/*
 * teb_plan.cuh — the launches that turn one optimizeTEB over a batch into TebOptimalPlanner::plan followed by
 * getVelocityCommand for every band (tebgpu_plan_batch / tebgpu_plan_batch_device):
 *
 *   k_plan_begin        warp per band, before k_begin: input check, cold start / warm start / re-initialisation
 *                       decision, initTrajectoryToGoal or updateAndPruneTEB            (optimal_planner.cpp:247-321)
 *   k_velocity_command  thread per band, after k_finalize: getVelocityCommand       (optimal_planner.cpp:1135-1168)
 *
 * and, on its own (tebgpu_read_trajectory / tebgpu_read_trajectory_device):
 *
 *   k_read_trajectory   warp per band read out: getVelocityProfile, getFullTrajectory (optimal_planner.cpp:1170-1248)
 *
 * The band routines are in teb_plan.h. k_plan_begin leaves a band it could not plan untouched and hands the reason
 * (TEB_STATUS_BAD_INPUT, TEB_STATUS_CAPACITY) to k_begin through DevBatch::pre_status, so the optimize sequence skips
 * it and k_finalize reports it, as it does for a band autoResize could not grow.
 */
#pragma once

#include "teb_kernels.cuh"
#include "teb_plan.h"

namespace tebgpu {

constexpr int PLAN_PRUNE_MAX = 10; /* updateAndPruneTEB drops at most 10 poses (timed_elastic_band.cpp:563) */

__global__ void __launch_bounds__(128) k_plan_begin(DevBatch db, const __grid_constant__ TebParams p, TebPlanInput pi,
                                                    int32_t* pre_status) {
  const int b = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= db.B) return; /* whole warps leave together: B is the same for every lane of a warp */
  double* rec = db.poses + (size_t)b * db.n_cap * 4;
  const int n = db.n[b];
  const double* plan = pi.initial_plan ? pi.initial_plan + (size_t)b * pi.P_cap * 3 : nullptr;
  const int P = plan ? (pi.plan_count ? pi.plan_count[b] : pi.P_cap) : 0;
  /* inputs the host entry point rejects with TEBGPU_ERR_INVALID_ARG: a band length outside 0 .. n_cap, a plan length
   * outside 1 .. P_cap, a non-finite start, goal or plan row */
  bool bad = n < 0 || n > db.n_cap || (plan && (P < 1 || P > pi.P_cap));
  if (!bad) {
    if (plan) {
      for (int r = lane; r < P; r += 32)
        bad |= !(isfinite(plan[3 * r]) && isfinite(plan[3 * r + 1]) && isfinite(plan[3 * r + 2]));
    } else if (lane < 6) {
      const double v = lane < 3 ? pi.start[3 * b + lane] : pi.goal[3 * b + lane - 3];
      bad = !isfinite(v);
    }
  }
  bad = __any_sync(0xffffffffu, bad);
  if (bad) {
    if (lane == 0) {
      pre_status[b] = TEB_STATUS_BAD_INPUT;
      if (pi.path) pi.path[b] = TEB_PLAN_PATH_NONE;
    }
    return;
  }
  /* start and goal: the given poses, or the plan's first and last point (optimal_planner.cpp:257-258) */
  double s[3], g[3];
  if (plan) {
    const double* lp = plan + 3 * (P - 1);
    s[0] = plan[0]; s[1] = plan[1]; s[2] = teb_plan_yaw(plan[2]);
    g[0] = lp[0]; g[1] = lp[1]; g[2] = teb_plan_yaw(lp[2]);
  } else {
    for (int c = 0; c < 3; ++c) { s[c] = pi.start[3 * b + c]; g[c] = pi.goal[3 * b + c]; }
  }
  const int path = teb_plan_path(rec, n, g, p.force_reinit_new_goal_dist, p.force_reinit_new_goal_angular);
  int status = 0, code = path;
  if (path == TEB_PLAN_PATH_WARM) {
    /* updateAndPruneTEB(start, goal, min_samples): poses 1 .. k go while each is strictly nearer to the new start than
     * the one before it, k <= lookahead = min(n - min_samples, 10). Lane j holds the distance of pose j. */
    const int lookahead = min(min(n - p.min_samples, PLAN_PRUNE_MAX), n - 1); /* n - 1: min_samples < 1 */
    const double d = lane < n && lane <= PLAN_PRUNE_MAX ? teb_plan_dist(s[0], s[1], rec[4 * lane], rec[4 * lane + 1]) : 0.0;
    const double d_prev = __shfl_up_sync(0xffffffffu, d, 1);
    const unsigned stop = __ballot_sync(0xffffffffu, lane >= 1 && lane <= lookahead && !(d < d_prev));
    const int k = lookahead <= 0 ? 0 : (stop ? __ffs(stop) - 2 : lookahead);
    const int m = n - k;
    if (k > 0) { /* deletePoses(1, k), deleteTimeDiffs(1, k): record j >= 1 takes record j + k, record 0 keeps dt_0 */
      for (int base = 1; base < m; base += 32) {
        const int j = base + lane;
        double v[4];
        if (j < m)
          for (int c = 0; c < 4; ++c) v[c] = rec[4 * (j + k) + c];
        __syncwarp(); /* every lane holds its source record before any lane overwrites one */
        if (j < m)
          for (int c = 0; c < 4; ++c) rec[4 * j + c] = v[c];
        __syncwarp();
      }
    }
    if (lane == 0) {
      rec[0] = s[0]; rec[1] = s[1]; rec[2] = s[2];
      double* back = rec + 4 * (m - 1);
      back[0] = g[0]; back[1] = g[1]; back[2] = g[2];
      db.n[b] = m;
    }
  } else if (lane == 0) { /* cold start, or clearTimedElasticBand + initTrajectoryToGoal: sequential, one lane */
    const int m = plan ? teb_init_from_plan_records(rec, db.n_cap, plan, P, p.max_vel_x, p.max_vel_theta,
                                                    p.global_plan_overwrite_orientation, p.min_samples,
                                                    p.allow_init_with_backwards_motion)
                       : teb_init_to_goal_records(rec, db.n_cap, s, g, p.max_vel_x, p.min_samples);
    if (m < 0) { status = TEB_STATUS_CAPACITY; code = TEB_PLAN_PATH_NONE; }
    else db.n[b] = m;
  }
  if (lane == 0) {
    pre_status[b] = status;
    if (pi.path) pi.path[b] = code;
  }
}

__global__ void k_velocity_command(DevBatch db, const __grid_constant__ TebParams p, TebPlanInput pi) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= db.B) return;
  const int n = db.n[b];
  double v[3] = {0, 0, 0};
  const int ok = n >= 0 && n <= db.n_cap
                     ? teb_velocity_command(db.poses + (size_t)b * db.n_cap * 4, n, pi.look_ahead_poses,
                                            pi.prevent_look_ahead_poses_near_goal, p.dt_ref, p.max_vel_y, v)
                     : 0;
  double* c = pi.cmd + 4 * (size_t)b;
  c[0] = v[0]; c[1] = v[1]; c[2] = v[2]; c[3] = ok;
}

constexpr int TRAJ_THREADS = 128; /* k_read_trajectory: 4 output rows per CTA */

/* getVelocityProfile / getFullTrajectory (optimal_planner.cpp:1170-1248) of band bands[r] (or r) into output row r, one
 * warp per row (tebgpu_read_trajectory). Lane l takes poses l, l + 32, ...; pose i recomputes its two adjacent segments
 * (i - 1 -> i and i -> i + 1) as the reference does. time_from_start is the reference's sequential sum: the warp walks
 * the 32 time differences of a step one shuffle at a time, in order, so the sum is never reassociated. */
__global__ void __launch_bounds__(TRAJ_THREADS) k_read_trajectory(TebBatch bt, TebTrajectoryArgs a, int R, double max_vel_y) {
  const int r = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= R) return; /* whole warps leave together */
  const int b = a.bands ? a.bands[r] : r;
  const int n = b >= 0 && b < bt.B ? bt.n[b] : -1;
  if (n < 0 || n > bt.n_cap) {
    if (lane == 0) a.points[r] = -1;
    return;
  }
  if (lane == 0) a.points[r] = n;
  const double* rec = bt.poses + (size_t)b * bt.n_cap * 4;
  const double* vs = bt.vel_start + 4 * (size_t)b;
  const double* vg = bt.vel_goal + 4 * (size_t)b;
  double* prof = a.profile ? a.profile + (size_t)r * (bt.n_cap + 1) * 3 : nullptr;
  double* traj = a.trajectory ? a.trajectory + (size_t)r * bt.n_cap * 7 : nullptr;
  double carry = 0.0; /* time_from_start of the next step's first pose, the same on every lane */
  for (int base = 0; base <= n; base += 32) {
    const int i = base + lane;
    double v1[3] = {0, 0, 0}, v2[3] = {0, 0, 0};
    if (i >= 1 && i <= n - 1) teb_extract_velocity(rec + 4 * (i - 1), rec + 4 * i, rec[4 * (i - 1) + 3], max_vel_y, v1);
    if (prof && i <= n) { /* n == 0: the one row is the goal velocity */
      const double* v = i == n ? vg : (i == 0 ? vs : v1);
      for (int c = 0; c < 3; ++c) prof[3 * i + c] = v[c];
    }
    if (!traj) continue;
    const double dt = i < n ? rec[4 * i + 3] : 0.0;
    double t = 0.0;
    for (int j = 0; j < 32; ++j) {
      if (lane == j) t = carry;
      carry = teb_add(carry, __shfl_sync(0xffffffffu, dt, j));
    }
    if (i >= n) continue;
    double* o = traj + 7 * (size_t)i;
    o[0] = rec[4 * i]; o[1] = rec[4 * i + 1]; o[2] = rec[4 * i + 2];
    if (i == 0 || i == n - 1) { /* n == 1: the start velocity */
      const double* v = i == 0 ? vs : vg;
      o[3] = v[0]; o[4] = v[1]; o[5] = v[2];
    } else {
      teb_extract_velocity(rec + 4 * i, rec + 4 * (i + 1), dt, max_vel_y, v2);
      for (int c = 0; c < 3; ++c) o[3 + c] = teb_mul(0.5, teb_add(v1[c], v2[c]));
    }
    o[6] = t;
  }
}

}  // namespace tebgpu
