/*
 * teb_fleet.cuh — the other robots of a fleet as custom obstacle rows of every robot's scene (tebgpu_fleet_obstacles /
 * _device). The contract is at TebFleetArgs in include/teb_b200.h.
 *
 *   k_fleet_claim      one thread per robot: counts the robots of every scene (only when TebFleetArgs.scene is given)
 *   k_fleet_obstacles  one warp per robot, FLEET_WARPS robots per CTA: all pairs, tiled through shared memory; TABLE
 *                      false takes the candidates from the caller's arrays (tebgpu_fleet_obstacles), true from the
 *                      rows of a TebFleetTable (tebgpu_fleet_obstacles_table)
 *   k_fleet_publish    one thread per robot: the robot's TebFleetRow (tebgpu_fleet_publish)
 *
 * The CTA stages FLEET_TILE robots' (x, y, world) at a time (the table build (x, y, world, live)); lane l of a warp tests candidates l, l + 32, ... of the
 * tile against its robot, and the warp keeps the nearest min(max_rows, C_cap - own) neighbours as a list sorted by
 * (d2, index), slot i in lane i. A candidate enters the list only when it is below the list's last slot, so after the
 * first few tiles almost every ballot is empty and the scan costs the distance test alone. The list is a total order
 * on distinct keys, so the rows do not depend on the tiling or on the order the candidates are met in.
 */
#pragma once

#include <climits>
#include <cmath>

namespace tebgpu {

constexpr int FLEET_WARPS = 16;                    /* robots per CTA */
constexpr int FLEET_THREADS = FLEET_WARPS * 32;
constexpr int FLEET_TILE = FLEET_THREADS;          /* robots staged per tile: one load per thread */
constexpr int CLAIM_THREADS = 256;

/* (d2, q) order: nearest first, a tie to the lower index */
__device__ __forceinline__ bool fleet_less(double da, int qa, double db, int qb) {
  return da < db || (da == db && qa < qb);
}

/* the row robot q is published as, from its pose (x, y, theta), body command (vx, vy) and radius: the publisher's
 * map-frame velocity R(theta) (vx, vy), then setCentroidVelocity's rule (obstacles.h:214-233), Eigen's norm() =
 * sqrt(squaredNorm()), of the body command: the rotation keeps the norm, and so the decision does not depend on the last
 * bits of sin / cos. Both the array build of k_fleet_obstacles and k_fleet_publish write their rows from here. */
__device__ __forceinline__ TebFleetRow fleet_row(const double* pose, const double* cmd, const double* radius, int world) {
  const double th = pose[2], bx = cmd[0], by = cmd[1];
  double sn, cs;
  sincos(th, &sn, &cs);
  double vx = __dsub_rn(__dmul_rn(cs, bx), __dmul_rn(sn, by));
  double vy = __dadd_rn(__dmul_rn(sn, bx), __dmul_rn(cs, by));
  const bool moving = !(sqrt(__dadd_rn(__dmul_rn(bx, bx), __dmul_rn(by, by))) < 0.001);
  if (!moving) vx = vy = 0.0;
  TebFleetRow w;
  w.x = pose[0];
  w.y = pose[1];
  w.vx = vx;
  w.vy = vy;
  w.radius = *radius;
  w.world = world;
  w.dynamic = moving ? 1 : 0;
  w.live = 1;
  w._pad[0] = w._pad[1] = w._pad[2] = 0;
  return w;
}

__global__ void __launch_bounds__(CLAIM_THREADS) k_fleet_claim(const TebFleetArgs a, int32_t* claims) {
  const int r = blockIdx.x * CLAIM_THREADS + threadIdx.x;
  if (r >= a.R) return;
  const int s = a.scene[r];
  if (s >= 0 && s < a.S) atomicAdd(&claims[s], 1);
}

/* claims: [S] robots per scene from k_fleet_claim, or NULL when TebFleetArgs.scene is NULL (scene r, never shared).
 * TABLE: robot r is row t.first + r of t and the candidates are its T rows; otherwise t is not read. */
template <bool TABLE>
__global__ void __launch_bounds__(FLEET_THREADS) k_fleet_obstacles(const TebFleetArgs a, const int32_t* claims,
                                                                   const TebFleetTable t) {
  __shared__ double sx[FLEET_TILE], sy[FLEET_TILE];
  __shared__ int sw[FLEET_TILE];
  __shared__ int sl[TABLE ? FLEET_TILE : 1];
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * FLEET_WARPS + (threadIdx.x >> 5);
  const bool live = r < a.R;
  const int self = TABLE ? t.first + r : r;    /* the robot's own candidate index */
  const int N = TABLE ? t.T : a.R;             /* candidates */

  double xr = 0.0, yr = 0.0;
  int wr = 0, s = -1, own = 0, K = 0, st = TEB_FLEET_BAD_INPUT;
  bool valid = false;
  if (live) {
    bool ok = true;
    if constexpr (TABLE) {
      const TebFleetRow& me = t.rows[self];
      xr = me.x;
      yr = me.y;
      wr = me.world;
      ok = me.live != 0;
    } else {
      xr = a.pose[3 * (size_t)r];
      yr = a.pose[3 * (size_t)r + 1];
      wr = a.world ? a.world[r] : 0;
    }
    s = a.scene ? a.scene[r] : r;
    if (ok && s >= 0 && s < a.S) {
      own = a.own_count ? a.own_count[s] : 0;
      if (own >= 0 && own <= a.C_cap) {
        if (claims && claims[s] != 1) st = TEB_FLEET_SHARED_SCENE;
        else valid = true;
      }
    }
    if (valid) K = min(a.max_rows, a.C_cap - own);
  }
  const double range2 = __dmul_rn(a.range, a.range);
  /* slot `lane` of the list (empty: +inf / INT_MAX, above every real key) and the key of slot K - 1 */
  double kd = INFINITY, td = INFINITY;
  int kq = INT_MAX, tq = INT_MAX;
  int needed = 0;

  for (int base = 0; base < N; base += FLEET_TILE) {
    const int nt = min(FLEET_TILE, N - base);
    __syncthreads();
    if ((int)threadIdx.x < nt) {
      const size_t q = (size_t)base + threadIdx.x;
      if constexpr (TABLE) {
        const TebFleetRow& w = t.rows[q];
        sx[threadIdx.x] = w.x;
        sy[threadIdx.x] = w.y;
        sw[threadIdx.x] = w.world;
        sl[threadIdx.x] = w.live;
      } else {
        sx[threadIdx.x] = a.pose[3 * q];
        sy[threadIdx.x] = a.pose[3 * q + 1];
        sw[threadIdx.x] = a.world ? a.world[q] : 0;
      }
    }
    __syncthreads();
    if (!valid) continue;                 /* warp-uniform: one robot per warp */
    for (int j0 = 0; j0 < nt; j0 += 32) {
      const int j = j0 + lane, q = base + j;
      bool in = false;
      double d2 = 0.0;
      if (j < nt && q != self && sw[j] == wr && (!TABLE || sl[j] != 0)) {
        const double dx = __dsub_rn(sx[j], xr), dy = __dsub_rn(sy[j], yr);
        d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
        in = d2 <= range2;
      }
      needed += __popc(__ballot_sync(FULL, in));
      bool pass = in && K > 0 && fleet_less(d2, q, td, tq);
      unsigned pm = __ballot_sync(FULL, pass);
      while (pm) {                        /* insert the passing candidates one at a time, lowest lane first */
        const int src = __ffs(pm) - 1;
        const double cd = __shfl_sync(FULL, d2, src);
        const int cq = __shfl_sync(FULL, q, src);
        const int pos = __popc(__ballot_sync(FULL, lane < K && fleet_less(kd, kq, cd, cq)));
        const double ud = __shfl_up_sync(FULL, kd, 1);
        const int uq = __shfl_up_sync(FULL, kq, 1);
        if (lane < K) {
          if (lane == pos) { kd = cd; kq = cq; }
          else if (lane > pos) { kd = ud; kq = uq; }
        }
        td = __shfl_sync(FULL, kd, K - 1);
        tq = __shfl_sync(FULL, kq, K - 1);
        pass = pass && lane != src && fleet_less(d2, q, td, tq);
        pm = __ballot_sync(FULL, pass);
      }
    }
  }
  if (!live) return;
  if (!valid) {
    if (lane == 0) {
      if (a.needed) a.needed[r] = -1;
      if (a.status) a.status[r] = st;
    }
    return;
  }
  const int written = min(needed, K);
  if (lane < written) {
    const size_t q = (size_t)kq;
    /* the neighbour's row: copied from the table as it was published, or made here from the caller's arrays */
    const TebFleetRow w = TABLE ? t.rows[q] : fleet_row(a.pose + 3 * q, a.last_cmd + 3 * q, a.radius + q, 0);
    TebObstacle o;
    o.x = w.x;
    o.y = w.y;
    o.vx = w.vx;
    o.vy = w.vy;
    o.radius = w.radius;
    o.dynamic = w.dynamic;
    o.type = TEB_OBST_CIRCULAR;
    o.vertex_begin = 0;
    o.vertex_count = 0;
    o._pad = 0.0;
    a.custom[(size_t)s * a.C_cap + own + lane] = o;
  }
  if (lane == 0) {
    a.custom_count[s] = own + written;
    if (a.needed) a.needed[r] = needed;
    if (a.status) a.status[r] = written < needed ? TEB_FLEET_TRUNCATED : TEB_FLEET_WRITTEN;
  }
}

__global__ void __launch_bounds__(CLAIM_THREADS) k_fleet_publish(const TebFleetArgs a, const TebFleetTable t) {
  const int r = blockIdx.x * CLAIM_THREADS + threadIdx.x;
  if (r >= a.R) return;
  t.rows[(size_t)t.first + r] = fleet_row(a.pose + 3 * (size_t)r, a.last_cmd + 3 * (size_t)r, a.radius + r,
                                          a.world ? a.world[r] : 0);
}

}  // namespace tebgpu
