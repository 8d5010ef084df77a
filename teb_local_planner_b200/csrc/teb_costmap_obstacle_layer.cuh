/*
 * teb_costmap_obstacle_layer.cuh — every robot's obstacle layer marked and cleared from its sensor points
 * (tebgpu_costmap_obstacle_layer / _device): costmap_2d's ObstacleLayer, as defined at TebObstacleLayerArgs in
 * include/teb_b200.h.
 *
 *   k_costmap_obstacle_layer   one CTA of OL_THREADS per robot, the robot's layer row in dynamic shared memory:
 *                              thread 0 decides the status and the origins; the row is filled with the default and the
 *                              previous row scattered into it shifted (16-byte loads); each thread walks the rays of its
 *                              points; each thread marks its points; warp 0 clears the footprint's column spans; then
 *                              the layer row is stored in place and the master row combined, in 16-byte stores
 *
 * A CTA reads its whole layer row before it writes any of it, so the layer is updated in place. Each phase writes one
 * value (the default and the shifted cells, 0 for the rays, 254 for the marks, 0 for the footprint), so the order of the
 * byte stores inside a phase does not matter and __syncthreads at the phase boundaries gives costmap_2d's bytes. Every
 * product and sum is a round-to-nearest helper of teb_plan.h, so FMA contraction cannot move a point across a cell edge.
 */
#pragma once

#include <climits>
#include <cstdint>
#include <cstring>

#include "teb_costmap_window.cuh"

namespace tebgpu {

constexpr int OL_THREADS = 256;

/* the launch's parameter block: the arguments, and the footprint copied from the host */
struct ObstacleLayerDev {
  TebObstacleLayerArgs a;
  double fp[TEB_COSTMAP_FOOTPRINT_MAX][2];
};

TEB_HD inline bool ol_same_bits(double x, double y) {
#if defined(__CUDA_ARCH__)
  return __double_as_longlong(x) == __double_as_longlong(y);
#else
  long long u, v;
  std::memcpy(&u, &x, 8);
  std::memcpy(&v, &y, 8);
  return u == v;
#endif
}

/* TEB_OBSTACLE_LAYER_* of robot s; on OK or ORIGIN_MISMATCH also the snapped layer origin and the whole-cell move */
TEB_HD inline int obstacle_layer_status(const TebObstacleLayerArgs& a, int s, double* nox, double* noy, double* cx,
                                        double* cy) {
  const long long sx = a.grid[2 * s], sy = a.grid[2 * s + 1];
  const double r = a.origin[3 * (size_t)s + 2];
  const double lox = a.layer_origin[2 * (size_t)s], loy = a.layer_origin[2 * (size_t)s + 1];
  const double rx = a.robot[3 * (size_t)s], ry = a.robot[3 * (size_t)s + 1];
  if (sx < 1 || sy < 1 || sx * sy > a.cell_cap || !(r > 0.0) || !isfinite(r) || !isfinite(lox) || !isfinite(loy) ||
      !isfinite(rx) || !isfinite(ry))
    return TEB_OBSTACLE_LAYER_BAD_GRID;
  const int n = a.point_count[s];
  if (n < 0 || n > a.P_cap) return TEB_OBSTACLE_LAYER_BAD_POINTS;
  *cx = costmap_window_cells(lox, rx, (int)sx, r);
  *cy = costmap_window_cells(loy, ry, (int)sy, r);
  *nox = teb_add(lox, teb_mul(*cx, r));
  *noy = teb_add(loy, teb_mul(*cy, r));
  if (a.mode == TEB_OBSTACLE_LAYER_COMBINE &&
      (!ol_same_bits(*nox, a.origin[3 * (size_t)s]) || !ol_same_bits(*noy, a.origin[3 * (size_t)s + 1])))
    return TEB_OBSTACLE_LAYER_ORIGIN_MISMATCH;
  return TEB_OBSTACLE_LAYER_OK;
}

/* Costmap2D::worldToMap; a NaN quotient or one not below the size is off the map */
__device__ __forceinline__ bool ol_world_to_map(double wx, double wy, double ox, double oy, double r, int sx, int sy,
                                                int* mx, int* my) {
  if (wx < ox || wy < oy) return false;
  const double qx = teb_add(wx, -ox) / r, qy = teb_add(wy, -oy) / r;
  if (!(qx < (double)sx && qy < (double)sy)) return false;
  *mx = (int)qx;
  *my = (int)qy;
  return true;
}

/* Costmap2D::raytraceLine with bresenham2D, the action writing v to every cell visited */
__device__ __forceinline__ void ol_raytrace(uint8_t* row, int x0, int y0, int x1, int y1, int sx, unsigned max_length,
                                            uint8_t v) {
  const int dx = x1 - x0, dy = y1 - y0;
  const unsigned adx = (unsigned)abs(dx), ady = (unsigned)abs(dy);
  const int odx = dx > 0 ? 1 : -1, ody = (dy > 0 ? 1 : -1) * sx; /* costmap_2d's sign(): sign(0) is -1 */
  /* hypot of the integer deltas: the square root of their exact sum of squares is the correctly rounded hypot */
  const double dist = sqrt((double)((long long)dx * dx + (long long)dy * dy));
  const double scale = dist == 0.0 ? 1.0 : fmin(1.0, (double)max_length / dist);
  const bool xdom = adx >= ady;
  const unsigned da = xdom ? adx : ady, db = xdom ? ady : adx;
  const int oa = xdom ? odx : ody, ob = xdom ? ody : odx;
  const unsigned end = min((unsigned)teb_mul(scale, (double)da), da);
  int offset = y0 * sx + x0, err = (int)(da / 2);
  for (unsigned i = 0; i < end; ++i) {
    row[offset] = v;
    offset += oa;
    err += (int)db;
    if ((unsigned)err >= da) {
      offset += ob;
      err -= (int)da;
    }
  }
  row[offset] = v;
}

/* the least and greatest y of the cells raytraceLine visits in column x on the edge (x0, y0) -> (x1, y1), merged into
 * lo / hi: bresenham2D in closed form, the minor axis moved floor((da / 2 + k db) / da) times after k steps */
__device__ __forceinline__ void ol_edge_span(int x0, int y0, int x1, int y1, int x, int& lo, int& hi) {
  const int dx = x1 - x0, dy = y1 - y0, sgx = dx > 0 ? 1 : -1, sgy = dy > 0 ? 1 : -1;
  const int adx = abs(dx), ady = abs(dy), m = (x - x0) * sgx;
  if (m < 0 || m > adx) return;
  int ya, yb;
  if (adx >= ady) {
    ya = yb = adx ? y0 + sgy * (int)(((long long)(adx / 2) + (long long)m * ady) / adx) : y0;
  } else {
    const int e0 = ady / 2;
    int klo = 0, khi = ady;
    if (adx) {
      const long long num = (long long)m * ady - e0;
      klo = num <= 0 ? 0 : (int)((num + adx - 1) / adx);
      khi = min(ady, (int)(((long long)(m + 1) * ady - e0 - 1) / adx));
    }
    ya = y0 + sgy * klo;
    yb = y0 + sgy * khi;
  }
  lo = min(lo, min(ya, yb));
  hi = max(hi, max(ya, yb));
}

/* row[c] = f(c, row[c]) for c < cap, in 16-byte stores where the row is aligned and single bytes at its ends */
template <bool READ, class Fn>
__device__ __forceinline__ void ol_store_row(uint8_t* row, int cap, Fn f) {
  const int tid = threadIdx.x;
  const int head = min(cap, (int)((16 - (reinterpret_cast<uintptr_t>(row) & 15)) & 15));
  const int groups = (cap - head) >> 4, tail = head + (groups << 4);
  for (int c = tid; c < head; c += OL_THREADS) row[c] = f(c, READ ? row[c] : (uint8_t)0);
  for (int c = tail + tid; c < cap; c += OL_THREADS) row[c] = f(c, READ ? row[c] : (uint8_t)0);
  for (int g = tid; g < groups; g += OL_THREADS) {
    const int c0 = head + (g << 4);
    uint4 in = make_uint4(0, 0, 0, 0);
    if (READ) in = *reinterpret_cast<const uint4*>(row + c0);
    const uint32_t iw[4] = {in.x, in.y, in.z, in.w};
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 16; ++k)
      w[k >> 2] |= (uint32_t)f(c0 + k, (uint8_t)(iw[k >> 2] >> (8 * (k & 3)))) << (8 * (k & 3));
    *reinterpret_cast<uint4*>(row + c0) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

/* f(c, row[c]) for every c < cap, read in 16-byte loads where the row is aligned and single bytes at its ends */
template <class Fn>
__device__ __forceinline__ void ol_load_row(const uint8_t* row, int cap, Fn f) {
  const int tid = threadIdx.x;
  const int head = min(cap, (int)((16 - (reinterpret_cast<uintptr_t>(row) & 15)) & 15));
  const int groups = (cap - head) >> 4, tail = head + (groups << 4);
  for (int c = tid; c < head; c += OL_THREADS) f(c, row[c]);
  for (int c = tail + tid; c < cap; c += OL_THREADS) f(c, row[c]);
  for (int g = tid; g < groups; g += OL_THREADS) {
    const int c0 = head + (g << 4);
    const uint4 in = *reinterpret_cast<const uint4*>(row + c0);
    const uint32_t iw[4] = {in.x, in.y, in.z, in.w};
#pragma unroll
    for (int k = 0; k < 16; ++k) f(c0 + k, (uint8_t)(iw[k >> 2] >> (8 * (k & 3))));
  }
}

/* updateWithOverwrite (0) / updateWithMax (1) of one cell, master m and layer l; anything else leaves the master */
__device__ __forceinline__ uint8_t ol_combine(int method, uint8_t m, uint8_t l) {
  if (l == TEB_COSTMAP_NO_INFORMATION || (method != 0 && method != 1)) return m;
  if (method == 0) return l;
  return (m == TEB_COSTMAP_NO_INFORMATION || m < l) ? l : m;
}

/* footprint clearing by the calling warp (lanes 0 .. 31): the footprint fp[F] placed at rb (x, y, yaw), its vertices'
 * cells into vx / vy, then one column span per lane of row set to FREE_SPACE; when a placed vertex is off the map
 * nothing is cleared and lane 0 ors off_bit into *flags */
__device__ __forceinline__ void ol_clear_footprint(const double (*fp)[2], int F, const double* rb, double ox, double oy,
                                                   double r, int sx, int sy, int* vx, int* vy, uint8_t* row, int* flags,
                                                   int off_bit) {
  const int lane = threadIdx.x;
  const double c = cos(rb[2]), sn = sin(rb[2]);
  bool off = false;
  for (int k = lane; k < F; k += 32) {
    const double px = fp[k][0], py = fp[k][1];
    const double wx = teb_add(rb[0], teb_add(teb_mul(px, c), -teb_mul(py, sn)));
    const double wy = teb_add(rb[1], teb_add(teb_mul(px, sn), teb_mul(py, c)));
    off |= !ol_world_to_map(wx, wy, ox, oy, r, sx, sy, &vx[k], &vy[k]);
  }
  off = __any_sync(0xffffffffu, off);
  __syncwarp();
  if (off) {
    if (lane == 0) *flags |= off_bit;
  } else {
    int xmin = INT_MAX, xmax = INT_MIN;
    for (int k = 0; k < F; ++k) {
      xmin = min(xmin, vx[k]);
      xmax = max(xmax, vx[k]);
    }
    for (int x = xmin + lane; x <= xmax; x += 32) {
      int lo = INT_MAX, hi = INT_MIN;
      for (int k = 0; k < F; ++k) {
        const int k1 = k + 1 < F ? k + 1 : 0;
        ol_edge_span(vx[k], vy[k], vx[k1], vy[k1], x, lo, hi);
      }
      for (int y = lo; y <= hi; ++y) row[y * sx + x] = 0;
    }
  }
}

__global__ void __launch_bounds__(OL_THREADS) k_costmap_obstacle_layer(const __grid_constant__ ObstacleLayerDev d) {
  extern __shared__ __align__(16) uint8_t srow[];
  __shared__ int s_st, s_cx, s_cy, s_flags;
  __shared__ double s_o[2];
  __shared__ int s_vx[TEB_COSTMAP_FOOTPRINT_MAX], s_vy[TEB_COSTMAP_FOOTPRINT_MAX];
  const TebObstacleLayerArgs& a = d.a;
  const int s = blockIdx.x, tid = threadIdx.x, cap = a.cell_cap;
  const bool standalone = a.mode == TEB_OBSTACLE_LAYER_STANDALONE;
  const uint8_t mdef = (uint8_t)a.master_default, ldef = a.track_unknown_space ? 255 : 0;
  uint8_t* lrow = a.layer + (size_t)s * cap;
  uint8_t* mrow = a.cost + (size_t)s * cap;
  if (tid == 0) {
    double nox = 0, noy = 0, cx = 0, cy = 0;
    const int st = obstacle_layer_status(a, s, &nox, &noy, &cx, &cy);
    s_st = st;
    s_flags = 0;
    a.status[s] = st;
    if (st == TEB_OBSTACLE_LAYER_OK) {
      const int sx = a.grid[2 * s], sy = a.grid[2 * s + 1];
      const bool in = fabs(cx) < (double)sx && fabs(cy) < (double)sy; /* otherwise every cell moves out (NaN too) */
      s_cx = in ? (int)cx : INT_MAX;
      s_cy = in ? (int)cy : 0;
      s_o[0] = nox;
      s_o[1] = noy;
      a.layer_origin[2 * (size_t)s] = nox;
      a.layer_origin[2 * (size_t)s + 1] = noy;
      if (standalone) {
        a.origin[3 * (size_t)s] = nox;
        a.origin[3 * (size_t)s + 1] = noy;
      }
    } else if (a.flags) {
      a.flags[s] = 0;
    }
  }
  __syncthreads();
  if (s_st != TEB_OBSTACLE_LAYER_OK) {
    if (standalone) ol_store_row<false>(mrow, cap, [&](int, uint8_t) { return mdef; });
    return;
  }
  const int sx = a.grid[2 * s], sy = a.grid[2 * s + 1], ncell = sx * sy;
  const double r = a.origin[3 * (size_t)s + 2], ox = s_o[0], oy = s_o[1];

  /* 1. the row at the default, then the previous row's cells moved by (-cx, -cy) */
  const uint32_t dw = ldef * 0x01010101u;
  for (int g = tid; g < (cap + 15) >> 4; g += OL_THREADS) reinterpret_cast<uint4*>(srow)[g] = make_uint4(dw, dw, dw, dw);
  __syncthreads();
  if (s_cx != INT_MAX) {
    const int cx = s_cx, cy = s_cy;
    ol_load_row(lrow, cap, [&](int c, uint8_t v) {
      if (c >= ncell) return;
      const int j = c / sx, i = c - j * sx, ni = i - cx, nj = j - cy;
      if (ni >= 0 && ni < sx && nj >= 0 && nj < sy) srow[nj * sx + ni] = v;
    });
  }
  __syncthreads();

  const int n = a.point_count[s];
  const float* pts = a.points + (size_t)s * a.P_cap * 3;
  const double* so = a.sensor_origin + 3 * (size_t)s;
  const double sox = so[0], soy = so[1], soz = so[2];
  /* 2. + 3. clearing: every kept point's ray, clamped to the map */
  if (a.clearing) {
    int x0, y0;
    if (!ol_world_to_map(sox, soy, ox, oy, r, sx, sy, &x0, &y0)) {
      if (tid == 0) s_flags |= TEB_OBSTACLE_LAYER_SENSOR_OFF_MAP;
    } else {
      const double ex = teb_add(ox, teb_mul((double)sx, r)), ey = teb_add(oy, teb_mul((double)sy, r));
      const double cells = fmax(0.0, ceil(a.raytrace_range / r));
      const unsigned max_length = cells >= 4294967295.0 ? 4294967295u : (unsigned)cells;
      for (int k = tid; k < n; k += OL_THREADS) {
        const double z = pts[3 * k + 2];
        if (!(a.min_obstacle_height <= z && z <= a.max_obstacle_height)) continue;
        double wx = pts[3 * k], wy = pts[3 * k + 1];
        const double ea = teb_add(wx, -sox), eb = teb_add(wy, -soy);
        if (wx < ox) {
          const double t = teb_add(ox, -sox) / ea;
          wx = ox;
          wy = teb_add(soy, teb_mul(eb, t));
        }
        if (wy < oy) {
          const double t = teb_add(oy, -soy) / eb;
          wx = teb_add(sox, teb_mul(ea, t));
          wy = oy;
        }
        if (wx > ex) {
          const double t = teb_add(ex, -sox) / ea;
          wx = teb_add(ex, -.001);
          wy = teb_add(soy, teb_mul(eb, t));
        }
        if (wy > ey) {
          const double t = teb_add(ey, -soy) / eb;
          wx = teb_add(sox, teb_mul(ea, t));
          wy = teb_add(ey, -.001);
        }
        int x1, y1;
        if (ol_world_to_map(wx, wy, ox, oy, r, sx, sy, &x1, &y1)) ol_raytrace(srow, x0, y0, x1, y1, sx, max_length, 0);
      }
    }
  }
  __syncthreads();

  /* 4. marking */
  if (a.marking) {
    const double sq_range = teb_mul(a.obstacle_range, a.obstacle_range);
    for (int k = tid; k < n; k += OL_THREADS) {
      const double pz = pts[3 * k + 2];
      if (!(a.min_obstacle_height <= pz && pz <= a.max_obstacle_height)) continue;
      if (pz > a.layer_max_obstacle_height) continue;
      const double px = pts[3 * k], py = pts[3 * k + 1];
      const double ddx = teb_add(px, -sox), ddy = teb_add(py, -soy), ddz = teb_add(pz, -soz);
      if (teb_add(teb_add(teb_mul(ddx, ddx), teb_mul(ddy, ddy)), teb_mul(ddz, ddz)) >= sq_range) continue;
      int mx, my;
      if (ol_world_to_map(px, py, ox, oy, r, sx, sy, &mx, &my)) srow[my * sx + mx] = TEB_COSTMAP_LETHAL;
    }
  }
  __syncthreads();

  /* 5. footprint clearing by warp 0 */
  if (a.F >= 3 && tid < 32)
    ol_clear_footprint(d.fp, a.F, a.robot + 3 * (size_t)s, ox, oy, r, sx, sy, s_vx, s_vy, srow, &s_flags,
                       TEB_OBSTACLE_LAYER_FOOTPRINT_OFF_MAP);
  __syncthreads();

  /* 6. the layer row in place, then the master row combined over the window */
  ol_store_row<false>(lrow, cap, [&](int c, uint8_t) { return srow[c]; });
  const int method = a.combination_method;
  auto combine = [&](int c, uint8_t m) -> uint8_t {
    if (standalone) m = mdef;
    if (c >= ncell) return m;
    return ol_combine(method, m, srow[c]);
  };
  if (standalone) ol_store_row<false>(mrow, cap, combine);
  else ol_store_row<true>(mrow, cap, combine);
  if (tid == 0 && a.flags) a.flags[s] = s_flags;
}

}  // namespace tebgpu
