/*
 * teb_costmap_window.cuh — every robot's local costmap cut out of the shared static maps (tebgpu_costmap_window /
 * _device): costmap_2d's rolling window with a static layer, as defined at TebStaticMaps in include/teb_b200.h.
 *
 *   k_costmap_window_origin   one thread per robot: the status, and updateOrigin's grid-snapped origin written back
 *   k_costmap_window<TF>      grid (S, strips): each robot's row of cell_cap bytes in 16-byte stores, lane l of a CTA
 *                             taking the 16 consecutive cells of one store, the CTAs of a robot taking every strips-th
 *                             group of 256 stores; TF: the cell centres moved by costmap_to_map (teb_frame.h's tf2
 *                             arithmetic), otherwise taken as they are
 *
 * The origin is snapped by its own launch because every CTA of a robot reads it: a CTA that wrote it back could not know
 * that the others had read the previous cycle's value. interpretValue depends on the byte alone, so each CTA tabulates
 * it once in shared memory; the map bytes are gathered through the read-only cache. In the identity path a cell's map
 * row depends on its window row alone and is computed once per row a lane meets. Every product and sum is a
 * round-to-nearest helper of teb_plan.h, so FMA contraction cannot move a centre.
 */
#pragma once

#include <cstdint>

#include "teb_frame.h"

namespace tebgpu {

constexpr int WINDOW_THREADS = 256;        /* one thread per interpretValue entry when the table is built */
constexpr int WINDOW_STRIP_BYTES = 16384;  /* bytes of a robot's row per CTA: 120 x 120 windows take one CTA each */

/* TEB_COSTMAP_WINDOW_* of robot s: the inputs the device answers with a default row and the host refuses */
TEB_HD inline int costmap_window_status(const TebStaticMaps& m, const TebCostmapWindowArgs& a, int s) {
  const int id = a.map_id[s];
  if (id < 0 || id >= m.W) return TEB_COSTMAP_WINDOW_BAD_MAP;
  const long long msx = m.size[2 * id], msy = m.size[2 * id + 1], off = m.offset[id];
  const double mr = m.origin[3 * id + 2];
  if (msx < 1 || msy < 1 || !(mr > 0.0) || !isfinite(mr) || off < 0 || off > m.pool_bytes - msx * msy)
    return TEB_COSTMAP_WINDOW_BAD_MAP;
  const long long sx = a.grid[2 * s], sy = a.grid[2 * s + 1];
  const double r = a.origin[3 * (size_t)s + 2];
  if (sx < 1 || sy < 1 || sx * sy > a.cell_cap || !(r > 0.0) || !isfinite(r)) return TEB_COSTMAP_WINDOW_BAD_GRID;
  return TEB_COSTMAP_WINDOW_OK;
}

/* updateOrigin's whole-cell move along one axis (a double: NaN or past the int range where the origin is): o the previous
 * origin, p the robot's coordinate, n the window's cells */
TEB_HD inline double costmap_window_cells(double o, double p, int n, double r) {
  const double size_m = teb_mul(teb_add((double)(n - 1), 0.5), r); /* getSizeInMetersX */
  const double target = teb_add(p, -(size_m / 2));
  return trunc(teb_add(target, -o) / r);
}

/* updateOrigin along one axis: the new origin */
TEB_HD inline double costmap_window_snap(double o, double p, int n, double r) {
  return teb_add(o, teb_mul(costmap_window_cells(o, p, n, r), r));
}

/* StaticLayer::interpretValue of the byte v */
TEB_HD inline uint8_t costmap_window_interpret(const TebStaticMaps& m, int v) {
  if (v == m.unknown_cost_value) return m.track_unknown_space ? 255 : 0;
  if (v >= m.lethal_threshold) return 254;
  if (m.trinary_costmap) return 0;
  return (uint8_t)((double)v / m.lethal_threshold * 254);
}

__global__ void k_costmap_window_origin(TebStaticMaps m, TebCostmapWindowArgs a) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= a.S) return;
  const int st = costmap_window_status(m, a, s);
  a.status[s] = st;
  if (st != TEB_COSTMAP_WINDOW_OK) return;
  double* o = a.origin + 3 * (size_t)s;
  const double r = o[2];
  o[0] = costmap_window_snap(o[0], a.robot[3 * (size_t)s], a.grid[2 * s], r);
  o[1] = costmap_window_snap(o[1], a.robot[3 * (size_t)s + 1], a.grid[2 * s + 1], r);
}

/* worldToMap along one axis: the cell, or -1 off the map (below the origin, at or past n cells, NaN) */
__device__ __forceinline__ int costmap_window_cell(double p, double o, double r, int n) {
  if (p < o) return -1;
  const double q = teb_add(p, -o) / r;
  return q < (double)n ? (int)q : -1;
}

template <bool TF>
__global__ void __launch_bounds__(WINDOW_THREADS) k_costmap_window(TebStaticMaps m, TebCostmapWindowArgs a) {
  __shared__ uint8_t lut[256];
  const int s = blockIdx.x, tid = threadIdx.x;
  lut[tid] = costmap_window_interpret(m, tid);
  __syncthreads();
  const uint8_t def = m.track_unknown_space ? 255 : 0;
  uint8_t* row = a.cost + (size_t)s * a.cell_cap;
  const bool ok = a.status[s] == TEB_COSTMAP_WINDOW_OK;
  int sx = 1, ncell = 0, msx = 1, msy = 1;
  double ox = 0, oy = 0, r = 1, mox = 0, moy = 0, mr = 1;
  const uint8_t* map = m.data;
  double b[9], t[2];
  if (ok) {
    const int id = a.map_id[s];
    sx = a.grid[2 * s];
    ncell = sx * a.grid[2 * s + 1];
    ox = a.origin[3 * (size_t)s]; oy = a.origin[3 * (size_t)s + 1]; r = a.origin[3 * (size_t)s + 2];
    msx = m.size[2 * id]; msy = m.size[2 * id + 1];
    mox = m.origin[3 * id]; moy = m.origin[3 * id + 1]; mr = m.origin[3 * id + 2];
    map += m.offset[id];
    if constexpr (TF) {
      const double* tf = a.costmap_to_map + 7 * (size_t)s;
      teb_tf2_basis(tf + 3, b);
      t[0] = tf[0]; t[1] = tf[1];
    }
  }
  int jc = -1, myc = -1; /* identity path: the window row met last and its map row */
  double wyc = 0;
  auto cell = [&](int c, int i, int j) -> uint8_t {
    if (c >= ncell) return def;
    if (j != jc) {
      jc = j;
      wyc = teb_add(oy, teb_mul(teb_add((double)j, 0.5), r));
      if constexpr (!TF) myc = costmap_window_cell(wyc, moy, mr, msy);
    }
    const double wx = teb_add(ox, teb_mul(teb_add((double)i, 0.5), r));
    int mx, my;
    if constexpr (TF) {
      double p[2];
      teb_frame_point(b, t, wx, wyc, 0.0, p);
      mx = costmap_window_cell(p[0], mox, mr, msx);
      my = costmap_window_cell(p[1], moy, mr, msy);
    } else {
      if (myc < 0) return def;
      mx = costmap_window_cell(wx, mox, mr, msx);
      my = myc;
    }
    if (mx < 0 || my < 0) return def;
    return lut[__ldg(map + (size_t)my * msx + mx)];
  };
  /* bytes before the first 16-byte boundary of the row and after the last one: single stores by the first strip */
  const int head = min(a.cell_cap, (int)((16 - (reinterpret_cast<uintptr_t>(row) & 15)) & 15));
  const int groups = (a.cell_cap - head) >> 4, tail = head + (groups << 4);
  if (blockIdx.y == 0) {
    for (int c = tid; c < head; c += WINDOW_THREADS) row[c] = cell(c, c % sx, c / sx);
    for (int c = tail + tid; c < a.cell_cap; c += WINDOW_THREADS) row[c] = cell(c, c % sx, c / sx);
  }
  for (int g = blockIdx.y * WINDOW_THREADS + tid; g < groups; g += gridDim.y * WINDOW_THREADS) {
    const int c0 = head + (g << 4);
    int j = c0 / sx, i = c0 - j * sx;
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      w[k >> 2] |= (uint32_t)cell(c0 + k, i, j) << (8 * (k & 3));
      if (++i == sx) { i = 0; ++j; }
    }
    *reinterpret_cast<uint4*>(row + c0) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

}  // namespace tebgpu
