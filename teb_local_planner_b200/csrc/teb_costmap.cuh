/*
 * teb_costmap.cuh — every scene's obstacle table from its local costmap (tebgpu_costmap_obstacles / _device): the
 * converter-less branch of TebLocalPlannerROS::updateObstacleContainerWithCostmap (teb_local_planner_ros.cpp:478-504)
 * followed by the custom obstacles (:552-625). The contract is at TebCostmapArgs in include/teb_b200.h.
 *
 *   k_costmap_obstacles<false>  one CTA per scene, custom rows verbatim
 *   k_costmap_obstacles<true>   the same with the custom rows moved from their own frame (TebFrameArgs, teb_frame.h's
 *                               Eigen isometry), one thread per row, a polygon finalised again by its thread
 *
 * The reference runs down the columns of a row-major raster (i over x outer, j over y inner), so 32 consecutive cells of
 * its order lie in 32 different rows: read straight from global memory, one sector each. The CTA therefore stages the
 * visited part of the raster (columns 0 .. sx - 2, rows 0 .. sy - 2) in shared memory, in tiles of at most COSTMAP_SMEM
 * bytes: the whole of it when it fits (read with 16-byte loads when the scene's raster is 16-byte aligned), else strips
 * of columns, else (a map taller than COSTMAP_SMEM / 4 rows) single columns in blocks of rows, so the order is kept. The
 * shared row pitch is a multiple of 4 bytes with an odd word count: the 32 cells a warp reads down a column fall into 32
 * banks. Each tile is enumerated in reference order with an ordered block compaction (ballot and popc per warp, warp
 * offsets in shared memory, a running base), and each kept cell is written as one 64-byte row of four 16-byte stores.
 * The centre, the projection on the heading and the distance use the round-to-nearest helpers of teb_plan.h, so FMA
 * contraction cannot move a centre or flip a decision.
 */
#pragma once

#include <climits>
#include <cstdint>

#include "teb_frame.h"
#include "teb_plan.h"

namespace tebgpu {

constexpr int COSTMAP_THREADS = 256;
constexpr int COSTMAP_SMEM = 24576; /* raster bytes staged per tile: a 128 x 128 map (its 127 x 127 visited cells) in one */
constexpr uint8_t COSTMAP_LETHAL = 254; /* costmap_2d::LETHAL_OBSTACLE */

/* shared row pitch of a tile w columns wide: a multiple of 4 bytes whose word count is odd */
__host__ __device__ inline int costmap_pitch(int w) {
  int p = (w + 3) & ~3;
  if (((p >> 2) & 1) == 0) p += 4;
  return p;
}

__device__ __forceinline__ void costmap_store_row(TebObstacle* dst, const uint4 (&q)[4]) {
  uint4* d = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int k = 0; k < 4; ++k) d[k] = q[k];
}

/* custom row o of scene s moved by custom_to_costmap (TebFrameArgs), its vertices written to obst_vertices; false for a
 * Line / Pill / Polygon row whose vertices are not given or lie outside 0 .. PV_cap */
__device__ bool costmap_move_custom(TebObstacle& o, const TebFrameArgs& f, int s) {
  const double* t = f.custom_to_costmap + 7 * (size_t)s;
  double m[9];
  teb_eigen_basis(t + 3, m);
  const double org[2] = {teb_add(0.0, t[0]), teb_add(0.0, t[1])}; /* Translation3d * Isometry3d: pretranslate of 0 */
  double p[2];
  if (o.type == TEB_OBST_POINT || o.type == TEB_OBST_CIRCULAR) {
    teb_frame_point(m, org, o.x, o.y, 0.0, p);
    o.x = p[0]; o.y = p[1];
    return true;
  }
  if (o.type != TEB_OBST_LINE && o.type != TEB_OBST_PILL && o.type != TEB_OBST_POLYGON) return true;
  const int vb = o.vertex_begin, vc = o.vertex_count;
  if (!f.custom_vertices || vb < 0 || vc < 1 || vb > f.PV_cap - vc || (o.type != TEB_OBST_POLYGON && vc != 2)) return false;
  const double* src = f.custom_vertices + ((size_t)s * f.PV_cap + vb) * 2;
  double* dst = f.obst_vertices + ((size_t)s * f.PV_cap + vb) * 2;
  for (int i = 0; i < vc; ++i) {
    teb_frame_point(m, org, src[2 * i], src[2 * i + 1], 0.0, p);
    dst[2 * i] = p[0]; dst[2 * i + 1] = p[1];
  }
  if (o.type != TEB_OBST_POLYGON) {
    o.x = teb_mul(0.5, teb_add(dst[0], dst[2]));
    o.y = teb_mul(0.5, teb_add(dst[1], dst[3]));
    return true;
  }
  int n = vc; /* finalizePolygon: fixPolygonClosure, then calcCentroid */
  if (n >= 2 && teb_eigen_is_approx(dst[0], dst[1], dst[2 * n - 2], dst[2 * n - 1])) --n;
  o.vertex_count = n;
  teb_polygon_centroid(dst, n, p);
  o.x = p[0]; o.y = p[1];
  return true;
}

/* TF: the custom rows in their own frame (TebFrameArgs' custom_to_costmap != NULL); otherwise f is not read */
template <bool TF>
__global__ void __launch_bounds__(COSTMAP_THREADS) k_costmap_obstacles(TebCostmapArgs a, TebFrameArgs f) {
  __shared__ __align__(16) uint8_t sr[COSTMAP_SMEM];
  __shared__ int swarp[COSTMAP_THREADS / 32];
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int sx = a.grid[2 * s], sy = a.grid[2 * s + 1];
  const int cc = a.custom_count ? a.custom_count[s] : 0;
  /* inputs the host entry point refuses with TEBGPU_ERR_INVALID_ARG */
  if (sx < 0 || sy < 0 || (long long)sx * sy > a.cell_cap || cc < 0 || cc > a.C_cap) {
    if (tid == 0) {
      a.obst_count[s] = -1;
      if (a.needed) a.needed[s] = -1;
    }
    return;
  }
  TebObstacle* out = a.obstacles + (size_t)s * a.M_cap;
  const uint8_t* cost = a.cost + (size_t)s * a.cell_cap;
  const int ncols = a.include_costmap_obstacles ? sx - 1 : 0, nrows = sy - 1;
  int base = 0; /* rows found so far: the next kept cell's row */
  if (ncols > 0 && nrows > 0) {
    const double ox = a.origin[3 * s], oy = a.origin[3 * s + 1], r = a.origin[3 * s + 2];
    const double rx = a.robot[3 * s], ry = a.robot[3 * s + 1], rt = a.robot[3 * s + 2];
    const double c = cos(rt), sn = sin(rt), behind = a.behind_robot_dist;
    /* tile shape: all visited rows of w columns, or one column and h rows when even one column does not fit */
    const int h = min(nrows, COSTMAP_SMEM / 4);
    int w = 1;
    if (h == nrows) {
      w = min(ncols, COSTMAP_SMEM / nrows);
      while (w > 1 && costmap_pitch(w) * nrows > COSTMAP_SMEM) --w;
    }
    const bool vec = w == ncols && h == nrows && (reinterpret_cast<uintptr_t>(cost) & 15) == 0;
    for (int c0 = 0; c0 < ncols; c0 += w) {
      const int wt = min(w, ncols - c0);
      const int P = costmap_pitch(wt);
      for (int r0 = 0; r0 < nrows; r0 += h) {
        const int ht = min(h, nrows - r0);
        __syncthreads(); /* the previous tile has been enumerated */
        if (vec) { /* the whole visited part: rows 0 .. sy - 2 are the contiguous bytes [0, nrows * sx) */
          const int bytes = nrows * sx, chunks = bytes >> 4;
          const uint4* g = reinterpret_cast<const uint4*>(cost);
          for (int q = tid; q < chunks; q += COSTMAP_THREADS) {
            const uint4 v = __ldg(g + q);
            const uint32_t wd[4] = {v.x, v.y, v.z, v.w};
            const int p0 = q << 4;
            int j = p0 / sx, i = p0 - j * sx;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
              if (i < ncols) sr[j * P + i] = (uint8_t)(wd[k >> 2] >> (8 * (k & 3)));
              if (++i == sx) { i = 0; ++j; }
            }
          }
          for (int p = (chunks << 4) + tid; p < bytes; p += COSTMAP_THREADS) {
            const int j = p / sx, i = p - j * sx;
            if (i < ncols) sr[j * P + i] = cost[p];
          }
        } else {
          for (int k = tid; k < wt * ht; k += COSTMAP_THREADS) {
            const int j = k / wt, i = k - j * wt;
            sr[j * P + i] = cost[(size_t)(r0 + j) * sx + c0 + i];
          }
        }
        __syncthreads();
        const int cnt = wt * ht;
        for (int e0 = 0; e0 < cnt; e0 += COSTMAP_THREADS) {
          const int e = e0 + tid;
          bool keep = false;
          double wx = 0, wy = 0;
          if (e < cnt) {
            const int ci = e / ht, rj = e - ci * ht;
            if (sr[rj * P + ci] == COSTMAP_LETHAL) {
              wx = teb_add(ox, teb_mul(teb_add((double)(c0 + ci), 0.5), r)); /* mapToWorld */
              wy = teb_add(oy, teb_mul(teb_add((double)(r0 + rj), 0.5), r));
              const double dx = teb_add(wx, -rx), dy = teb_add(wy, -ry);
              const double dot = teb_add(teb_mul(dx, c), teb_mul(dy, sn));
              const double norm = sqrt(teb_add(teb_mul(dx, dx), teb_mul(dy, dy)));
              keep = !(dot < 0 && norm > behind);
            }
          }
          const unsigned m = __ballot_sync(0xffffffffu, keep);
          if (lane == 0) swarp[warp] = __popc(m);
          __syncthreads();
          int off = base, tot = 0;
#pragma unroll
          for (int q = 0; q < COSTMAP_THREADS / 32; ++q) {
            const int k = swarp[q];
            off += q < warp ? k : 0;
            tot += k;
          }
          off += __popc(m & ((1u << lane) - 1u));
          if (keep && off < a.M_cap) {
            const uint4 z = make_uint4(0, 0, 0, 0); /* vx, vy, radius, dynamic, type TEB_OBST_POINT, vertices, _pad: 0 */
            const uint4 row[4] = {make_uint4(__double2loint(wx), __double2hiint(wx), __double2loint(wy), __double2hiint(wy)),
                                  z, z, z};
            costmap_store_row(out + off, row);
          }
          base += tot;
          __syncthreads(); /* swarp is rewritten by the next step */
        }
      }
    }
  }
  /* the custom rows, verbatim, or moved into the costmap frame */
  const TebObstacle* cu = a.custom ? a.custom + (size_t)s * a.C_cap : nullptr;
  bool bad = false;
  for (int k = tid; k < cc && (long long)base + k < a.M_cap; k += COSTMAP_THREADS) {
    const uint4* src = reinterpret_cast<const uint4*>(cu + k);
    uint4 row[4] = {__ldg(src), __ldg(src + 1), __ldg(src + 2), __ldg(src + 3)};
    if constexpr (TF) {
      TebObstacle o;
      memcpy(&o, row, sizeof(o));
      bad |= !costmap_move_custom(o, f, s);
      memcpy(row, &o, sizeof(o));
    }
    costmap_store_row(out + base + k, row);
  }
  if constexpr (TF) {
    if (__syncthreads_or(bad)) {
      if (tid == 0) {
        a.obst_count[s] = -1;
        if (a.needed) a.needed[s] = -1;
      }
      return;
    }
  }
  if (tid == 0) {
    const long long need = (long long)base + cc;
    a.obst_count[s] = need <= a.M_cap ? (int)need : -1;
    if (a.needed) a.needed[s] = need > INT_MAX ? INT_MAX : (int)need;
  }
}

}  // namespace tebgpu
