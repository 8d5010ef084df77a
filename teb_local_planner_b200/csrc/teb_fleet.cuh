/*
 * teb_fleet.cuh — the other robots of a fleet as custom obstacle rows of every robot's scene (tebgpu_fleet_obstacles /
 * _device). The contract is at TebFleetArgs in include/teb_b200.h.
 *
 *   k_fleet_claim      one thread per robot: counts the robots of every scene (only when TebFleetArgs.scene is given)
 *   k_fleet_obstacles  one warp per robot, FLEET_WARPS robots per CTA: all pairs, tiled through shared memory
 *
 * The CTA stages FLEET_TILE robots' (x, y, world) at a time; lane l of a warp tests candidates l, l + 32, ... of the
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

__global__ void __launch_bounds__(CLAIM_THREADS) k_fleet_claim(const TebFleetArgs a, int32_t* claims) {
  const int r = blockIdx.x * CLAIM_THREADS + threadIdx.x;
  if (r >= a.R) return;
  const int s = a.scene[r];
  if (s >= 0 && s < a.S) atomicAdd(&claims[s], 1);
}

/* claims: [S] robots per scene from k_fleet_claim, or NULL when TebFleetArgs.scene is NULL (scene r, never shared) */
__global__ void __launch_bounds__(FLEET_THREADS) k_fleet_obstacles(const TebFleetArgs a, const int32_t* claims) {
  __shared__ double sx[FLEET_TILE], sy[FLEET_TILE];
  __shared__ int sw[FLEET_TILE];
  constexpr unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * FLEET_WARPS + (threadIdx.x >> 5);
  const bool live = r < a.R;

  double xr = 0.0, yr = 0.0;
  int wr = 0, s = -1, own = 0, K = 0, st = TEB_FLEET_BAD_INPUT;
  bool valid = false;
  if (live) {
    xr = a.pose[3 * (size_t)r];
    yr = a.pose[3 * (size_t)r + 1];
    wr = a.world ? a.world[r] : 0;
    s = a.scene ? a.scene[r] : r;
    if (s >= 0 && s < a.S) {
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

  for (int base = 0; base < a.R; base += FLEET_TILE) {
    const int nt = min(FLEET_TILE, a.R - base);
    __syncthreads();
    if ((int)threadIdx.x < nt) {
      const size_t q = (size_t)base + threadIdx.x;
      sx[threadIdx.x] = a.pose[3 * q];
      sy[threadIdx.x] = a.pose[3 * q + 1];
      sw[threadIdx.x] = a.world ? a.world[q] : 0;
    }
    __syncthreads();
    if (!valid) continue;                 /* warp-uniform: one robot per warp */
    for (int j0 = 0; j0 < nt; j0 += 32) {
      const int j = j0 + lane, q = base + j;
      bool in = false;
      double d2 = 0.0;
      if (j < nt && q != r && sw[j] == wr) {
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
    const double th = a.pose[3 * q + 2], bx = a.last_cmd[3 * q], by = a.last_cmd[3 * q + 1];
    double sn, cs;
    sincos(th, &sn, &cs);
    double vx = __dsub_rn(__dmul_rn(cs, bx), __dmul_rn(sn, by));
    double vy = __dadd_rn(__dmul_rn(sn, bx), __dmul_rn(cs, by));
    /* setCentroidVelocity (obstacles.h:214-233), Eigen's norm() = sqrt(squaredNorm()), of the body command: the rotation
     * keeps the norm, and so the decision does not depend on the last bits of sin / cos */
    const bool moving = !(sqrt(__dadd_rn(__dmul_rn(bx, bx), __dmul_rn(by, by))) < 0.001);
    if (!moving) vx = vy = 0.0;
    TebObstacle o;
    o.x = a.pose[3 * q];
    o.y = a.pose[3 * q + 1];
    o.vx = vx;
    o.vy = vy;
    o.radius = a.radius[q];
    o.dynamic = moving ? 1 : 0;
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

}  // namespace tebgpu
