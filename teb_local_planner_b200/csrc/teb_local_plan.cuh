/*
 * teb_local_plan.cuh — every band's local plan, goal and via-points from its global plan (tebgpu_local_plan / _device):
 * the front of TebLocalPlannerROS::computeVelocityCommands (teb_local_planner_ros.cpp:268-340) with pruneGlobalPlan
 * (:657-698), transformGlobalPlan (:701-822), updateViaPointsContainer (:627-646), the goal-reached test (:290-304),
 * configureBackupModes' horizon shrink (:950-977) and estimateLocalGoalOrientation (:827-871). The contract is at
 * TebLocalPlanArgs in include/teb_b200.h.
 *
 *   k_local_plan<false>  one warp per band, LPLAN_THREADS / 32 bands per CTA, the plan in the costmap's frame
 *   k_local_plan<true>   the same with the plan in its own frame (TebFrameArgs): the robot is moved into the plan frame
 *                        once and the walk compares plan-frame rows with it. Only rows taken are moved into the costmap
 *                        frame (teb_frame.h, tf2's doTransform), once per pass that reads them: the plan write (position
 *                        and orientation, one row per lane), and, when via-points are extracted, the via-point count
 *                        and the via-point write (position only, a sliding window of moved rows, lp_via_points_tf)
 *
 * The warp walks the global plan in 32-row chunks, lane l on row base + l. Every loop of the reference is a sequence of
 * exact comparisons, so the warp takes the same decisions as the loop:
 *   prune        a ballot of dist_sq < d^2; the lowest set lane is the loop's first hit.
 *   closest row  an inclusive prefix minimum over the chunk (Kogge-Stone, the left element wins ties, NaN never wins),
 *                seeded with the running (sq, i). The exclusive prefix at lane j is the loop's state before row j, so the
 *                loop's break test (sq < 0.05 && d_j > sq) is evaluated on every lane at once; the lowest breaking lane
 *                ends the search with its exclusive state.
 *   walk         squared distances and segment lengths in parallel; plan_length is added one lane at a time, in order,
 *                as k_read_trajectory adds time_from_start, so the sum is never reassociated; a ballot finds the first
 *                row the loop does not take.
 *   via-points   from the last via-point the lanes test the next 32 rows and a ballot picks the first at >= sep; the
 *                indices found are kept one per lane and written 32 via-points at a time.
 * Output rows are written as consecutive doubles across the warp. Every product and sum is a round-to-nearest helper of
 * teb_plan.h, so FMA contraction cannot move a row or flip a decision.
 */
#pragma once

#include <cstdint>

#include "teb_frame.h"
#include "teb_plan.h"

namespace tebgpu {

constexpr int LPLAN_THREADS = 128; /* k_local_plan: 4 bands per CTA */

/* squared distance from (rx, ry) to a plan row, as the reference forms it (robot - row) */
__device__ __forceinline__ double lp_sq(double rx, double ry, const double* row) {
  const double dx = rx - row[0], dy = ry - row[1];
  return teb_add(teb_mul(dx, dx), teb_mul(dy, dy));
}

/* distance_points2d(p1, p2) = sqrt(pow(p2.x - p1.x, 2) + pow(p2.y - p1.y, 2)) */
__device__ __forceinline__ double lp_dist(const double* p1, const double* p2) {
  const double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
  return sqrt(teb_add(teb_mul(dx, dx), teb_mul(dy, dy)));
}

/* updateViaPointsContainer over the T rows t[0 .. T) (stride 3): returns the number of via-points; with out != NULL it
 * also writes them, (x, y) each */
__device__ int lp_via_points(const double* t, int T, double sep, double* out, int lane) {
  const unsigned full = 0xffffffffu;
  int count = 0, prev = 0, cur = 1, held = -1; /* held: this lane's via-point row of the current group of 32 */
  auto flush = [&](int rows) {                 /* the group's rows as 2 * rows consecutive doubles */
    for (int e0 = 0; e0 < 2 * rows; e0 += 32) {
      const int e = e0 + lane;
      const int k = __shfl_sync(full, held, e >> 1);
      if (e < 2 * rows) out[2 * (size_t)(count - rows) + e] = t[3 * k + (e & 1)];
    }
  };
  while (cur < T) {
    const int k = cur + lane;
    const bool take = k < T && !(lp_dist(t + 3 * prev, t + 3 * k) < sep);
    const unsigned m = __ballot_sync(full, take);
    if (!m) { cur += 32; continue; }
    prev = cur + __ffs(m) - 1;
    cur = prev + 1;
    if (lane == (count & 31)) held = prev;
    ++count;
    if (out && (count & 31) == 0) flush(32);
  }
  if (out && (count & 31)) flush(count & 31);
  return count;
}

/* lp_via_points over rows whose positions cost a rigid transform each, xy(k, x, y): the same decisions, with every row
 * moved once. Lane l keeps row cur + l of the window; after a via-point at lane l the window slides by l + 1 with a
 * shuffle, and only the lanes that run past the old window move a new row. The last via-point's position and this
 * lane's via-point of the current group of 32 are kept as values, so the write reads no row again. */
template <class XY>
__device__ int lp_via_points_tf(const XY& xy, int T, double sep, double* out, int lane) {
  const unsigned full = 0xffffffffu;
  int count = 0, cur = 1;
  double px, py, hx = 0.0, hy = 0.0, wx = 0.0, wy = 0.0; /* the last via-point (row 0 first), this lane's held one */
  xy(0, px, py);
  if (cur + lane < T) xy(cur + lane, wx, wy);
  auto flush = [&](int rows) {
    for (int e0 = 0; e0 < 2 * rows; e0 += 32) {
      const int e = e0 + lane;
      const double vx = __shfl_sync(full, hx, e >> 1), vy = __shfl_sync(full, hy, e >> 1);
      if (e < 2 * rows) out[2 * (size_t)(count - rows) + e] = (e & 1) ? vy : vx;
    }
  };
  while (cur < T) {
    const int k = cur + lane;
    bool take = false;
    if (k < T) {
      const double dx = wx - px, dy = wy - py; /* distance_points2d(last via-point, row k) */
      take = !(sqrt(teb_add(teb_mul(dx, dx), teb_mul(dy, dy))) < sep);
    }
    const unsigned m = __ballot_sync(full, take);
    if (!m) {
      cur += 32;
      if (cur + lane < T) xy(cur + lane, wx, wy);
      continue;
    }
    const int l = __ffs(m) - 1;
    px = __shfl_sync(full, wx, l);
    py = __shfl_sync(full, wy, l);
    if (lane == (count & 31)) { hx = px; hy = py; }
    ++count;
    if (out && (count & 31) == 0) flush(32);
    const unsigned sh = (unsigned)l + 1; /* the window slides to start at the via-point's next row */
    double nx = __shfl_down_sync(full, wx, sh), ny = __shfl_down_sync(full, wy, sh);
    cur += l + 1;
    if (lane + (int)sh >= 32 && cur + lane < T) xy(cur + lane, nx, ny);
    wx = nx; wy = ny;
  }
  if (out && (count & 31)) flush(count & 31);
  return count;
}

/* configureBackupModes' reduced horizon: the new size of the transformed plan, goal_idx updated in place */
__device__ __forceinline__ int lp_shrink_horizon(int size, int& goal_idx, int count, double since, double min_duration,
                                                 bool enabled) {
  if (enabled && goal_idx < size - 1 && (count > 0 || since < min_duration)) {
    int reduction = goal_idx / 2;
    if (count > 9) reduction /= 2;
    const int new_size = size - reduction - 1;
    goal_idx -= reduction;
    if (new_size > 0 && goal_idx >= 0) size = new_size;
    else goal_idx += reduction;
  }
  return size;
}

/* TF: the global plan in its own frame (TebFrameArgs' costmap_to_plan / plan_to_costmap); otherwise f is not read */
template <bool TF>
__global__ void __launch_bounds__(LPLAN_THREADS, 1) k_local_plan(const __grid_constant__ TebLocalPlanArgs a,
                                                              const __grid_constant__ TebFrameArgs f,
                                                              const int32_t* __restrict__ scene_id,
                                                              int B, int S, int overwrite_orientation) {
  const unsigned full = 0xffffffffu;
  const int b = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return; /* whole warps leave together */
  int begin = a.plan_begin[b];
  const int end = a.plan_end[b], sid = scene_id[b];
  if (begin < 0 || begin > end || end > a.G_cap || sid < 0 || sid >= S) {
    if (lane == 0) { a.result[b] = TEB_LOCAL_PLAN_BAD_INPUT; a.plan_count[b] = 0; }
    return;
  }
  const double* gp = a.global_plan + (size_t)b * a.G_cap * 3;
  const double rx = a.robot[3 * (size_t)b], ry = a.robot[3 * (size_t)b + 1], rt = a.robot[3 * (size_t)b + 2];
  /* the robot in the plan frame, which steps 1 and 3 compare the rows with; tb: the basis of plan_to_costmap */
  double px = rx, py = ry, tb[9];
  const double* p2c = nullptr;
  if constexpr (TF) {
    const double* c2p = f.costmap_to_plan + 7 * (size_t)b;
    double cb[9], o[2];
    teb_tf2_basis(c2p + 3, cb);
    teb_frame_point(cb, c2p, rx, ry, 0.0, o);
    px = o[0]; py = o[1];
    p2c = f.plan_to_costmap + 7 * (size_t)b;
    teb_tf2_basis(p2c + 3, tb);
  }
  /* a plan row's position as the local plan holds it: TF, one rigid transform into the costmap frame */
  auto xy = [&](const double* row, double& x, double& y) {
    if constexpr (TF) {
      double o[2];
      teb_frame_point(tb, p2c, row[0], row[1], 0.0, o);
      x = o[0]; y = o[1];
    } else {
      x = row[0]; y = row[1];
    }
  };

  /* 1. prune: the first live row closer than prune_distance */
  const double d2 = teb_mul(a.prune_distance, a.prune_distance);
  for (int base = begin; base < end; base += 32) {
    const int k = base + lane;
    const unsigned m = __ballot_sync(full, k < end && lp_sq(px, py, gp + 3 * k) < d2);
    if (m) { begin = base + __ffs(m) - 1; break; }
  }
  if (lane == 0) a.plan_begin[b] = begin;
  const double* g = gp + 3 * (size_t)begin;
  const int n = end - begin;
  if (n == 0) { /* 2. */
    if (lane == 0) { a.result[b] = TEB_LOCAL_PLAN_EMPTY; a.plan_count[b] = 0; }
    return;
  }

  /* 3. transform: the window, the closest row, the walk */
  const int sx = a.grid[2 * sid], sy = a.grid[2 * sid + 1];
  const double res = a.origin[3 * sid + 2];
  const double wx = teb_mul((double)sx, res) / 2.0, wy = teb_mul((double)sy, res) / 2.0;
  const double w = teb_mul(wx < wy ? wy : wx, 0.85), thr = teb_mul(w, w);
  double sq = 1e10;
  int closest = 0;
  for (int base = 0; base < n; base += 32) {
    const int j = base + lane;
    const double d = j < n ? lp_sq(px, py, g + 3 * j) : __longlong_as_double(0x7ff8000000000000ll);
    double v = d != d ? __longlong_as_double(0x7ff0000000000000ll) : d; /* NaN never becomes the minimum */
    int vi = j;
    for (int off = 1; off < 32; off <<= 1) {
      const double ov = __shfl_up_sync(full, v, off);
      const int oi = __shfl_up_sync(full, vi, off);
      if (lane >= off && !(v < ov)) { v = ov; vi = oi; }
    }
    if (!(v < sq)) { v = sq; vi = closest; }    /* seeded with the state before the chunk */
    double ev = __shfl_up_sync(full, v, 1);     /* the loop's state before row j */
    int ei = __shfl_up_sync(full, vi, 1);
    if (lane == 0) { ev = sq; ei = closest; }
    const unsigned brk = __ballot_sync(full, ev < 0.05 && d > ev);
    if (brk) {
      const int l = __ffs(brk) - 1;
      sq = __shfl_sync(full, ev, l);
      closest = __shfl_sync(full, ei, l);
      break;
    }
    sq = __shfl_sync(full, v, 31);
    closest = __shfl_sync(full, vi, 31);
  }
  const double mx = a.max_lookahead_dist;
  int stop = closest; /* one past the last row taken */
  double prev_sq = sq, len = 0.0;
  for (int base = closest; base < n; base += 32) {
    const int i = base + lane;
    const bool in = i < n;
    const double di = in ? lp_sq(px, py, g + 3 * i) : 0.0;
    const double seg = in && i > 0 && mx > 0 ? lp_dist(g + 3 * (i - 1), g + 3 * i) : 0.0;
    double pq = __shfl_up_sync(full, di, 1);
    if (lane == 0) pq = prev_sq;
    double before = 0.0; /* plan_length before row i: the rows taken so far, summed in order */
    for (int l = 0; l < 32; ++l) {
      if (lane == l) before = len;
      len = teb_add(len, __shfl_sync(full, seg, l));
    }
    const unsigned no = __ballot_sync(full, !(in && pq <= thr && (mx <= 0 || before <= mx)));
    if (no) { stop = base + __ffs(no) - 1; break; }
    prev_sq = __shfl_sync(full, di, 31);
    stop = base + 32;
  }
  int first = closest, size = stop - closest, goal_idx = stop - 1;
  if (size == 0) { first = n - 1; size = 1; goal_idx = n - 1; } /* the global goal injected */
  const double* t = g + 3 * (size_t)first;
  const int taken = size; /* the rows the via-points come from, before the shrink */

  /* 4. via-points (counted here, written once the band's result is known) */
  const bool own_via = a.via != nullptr;
  const bool extract = own_via && !(a.viapoint_sep <= 0);
  const auto txy = [&](int k, double& x, double& y) { xy(t + 3 * k, x, y); };
  int vcount;
  if constexpr (TF) vcount = extract ? lp_via_points_tf(txy, size, a.viapoint_sep, nullptr, lane) : 0;
  else vcount = extract ? lp_via_points(t, size, a.viapoint_sep, nullptr, lane) : 0;
  const int vtest = own_via ? vcount : (a.via_count ? a.via_count[b] : 0);

  /* 5. goal reached */
  const double* gl = g + 3 * (size_t)(n - 1);
  double gx, gy;
  xy(gl, gx, gy);
  const double gdx = gx - rx, gdy = gy - ry;
  const double* vel = a.robot_vel + 3 * (size_t)b;
  const bool stopped = fabs(vel[2]) <= a.theta_stopped_vel && fabs(vel[0]) <= a.trans_stopped_vel &&
                       fabs(vel[1]) <= a.trans_stopped_vel;
  double gyaw;
  if constexpr (TF) gyaw = teb_frame_row_yaw(tb, gl[2]);
  else gyaw = teb_plan_yaw(gl[2]);
  const bool reached = fabs(sqrt(teb_add(teb_mul(gdx, gdx), teb_mul(gdy, gdy)))) < a.xy_goal_tolerance &&
                       fabs(teb_normalize_theta(gyaw - rt)) < a.yaw_goal_tolerance &&
                       (!a.complete_global_plan || vtest == 0) && (stopped || a.free_goal_vel);
  int rows = 0;
  double head = 0.0;
  if (!reached) {
    /* 6. horizon shrink */
    const bool shrink = a.shrink_horizon_backup && (a.infeasible_count || a.since_infeasible);
    const int cnt = a.infeasible_count ? a.infeasible_count[b] : 0;
    const double since = a.since_infeasible ? a.since_infeasible[b] : __longlong_as_double(0x7ff0000000000000ll);
    size = lp_shrink_horizon(size, goal_idx, cnt, since, a.shrink_horizon_min_duration, shrink);
    /* 7. goal heading of the local goal row t[size - 1] */
    const double* lg = t + 3 * (size - 1);
    if (!overwrite_orientation) {
      if constexpr (TF) head = teb_frame_row_yaw(tb, lg[2]);
      else head = lg[2];
    } else if (goal_idx > n - 5) {
      if constexpr (TF) head = goal_idx >= n - 1 ? teb_frame_row_yaw(tb, lg[2]) : teb_frame_goal_yaw(p2c, gl[2]);
      else head = goal_idx >= n - 1 ? teb_plan_yaw(lg[2]) : gyaw;
    } else {
      const int m = n - goal_idx - 1 < 3 ? n - goal_idx - 1 : 3;
      double cx = 0.0, cy = 0.0, kx, ky;
      xy(lg, kx, ky);
#pragma unroll 1
      for (int i = goal_idx; i < goal_idx + m; ++i) {
        const double* k1 = g + 3 * (size_t)(i + 1);
        double k1x, k1y;
        xy(k1, k1x, k1y);
        const double c = atan2(k1y - ky, k1x - kx);
        cx = teb_add(cx, cos(c));
        cy = teb_add(cy, sin(c));
        kx = k1x; ky = k1y;
      }
      head = cx == 0 && cy == 0 ? 0.0 : atan2(cy, cx);
    }
    rows = size < 2 ? 2 : size; /* 8. */
  }

  /* 9. capacity, then the outputs */
  const bool cap = rows > a.P_cap || (own_via && vcount > a.V_cap);
  const int code = cap ? TEB_LOCAL_PLAN_CAPACITY : (reached ? TEB_LOCAL_PLAN_GOAL_REACHED : TEB_LOCAL_PLAN_PLANNED);
  if (code == TEB_LOCAL_PLAN_PLANNED) {
    double* o = a.plan + (size_t)b * a.P_cap * 3;
    if constexpr (TF) { /* one row per lane: each row taken moved once, position and orientation */
      for (int r = lane; r < rows; r += 32) {
        double* out = o + 3 * r;
        if (r == 0) {
          out[0] = rx; out[1] = ry; out[2] = rt;
        } else {
          const double* src = t + 3 * (r == rows - 1 ? size - 1 : r);
          xy(src, out[0], out[1]);
          out[2] = r == rows - 1 ? head : teb_frame_row_yaw(tb, src[2]);
        }
      }
    } else {
      for (int e = lane; e < 3 * rows; e += 32) {
        const int r = e / 3, c = e - 3 * r;
        double v;
        if (r == 0) v = c == 0 ? rx : (c == 1 ? ry : rt);
        else if (r == rows - 1) v = c == 2 ? head : t[3 * (size - 1) + c];
        else v = t[3 * r + c];
        o[e] = v;
      }
    }
  }
  if (extract && !cap) {
    if constexpr (TF) lp_via_points_tf(txy, taken, a.viapoint_sep, a.via + (size_t)b * a.V_cap * 2, lane);
    else lp_via_points(t, taken, a.viapoint_sep, a.via + (size_t)b * a.V_cap * 2, lane);
  }
  if (lane == 0) {
    a.result[b] = code;
    a.plan_count[b] = code == TEB_LOCAL_PLAN_PLANNED ? rows : 0;
    if (a.goal_idx) a.goal_idx[b] = goal_idx;
    if (own_via && !cap) a.via_count[b] = vcount;
    if (a.needed) { a.needed[2 * (size_t)b] = rows; a.needed[2 * (size_t)b + 1] = vcount; }
  }
}

}  // namespace tebgpu
