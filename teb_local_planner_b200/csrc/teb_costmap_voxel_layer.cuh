/*
 * teb_costmap_voxel_layer.cuh — every robot's voxel layer marked and cleared in 3-D from up to
 * TEB_VOXEL_LAYER_MAX_SOURCES observation sources (tebgpu_costmap_voxel_layer / _device): costmap_2d's VoxelLayer, as
 * defined at TebVoxelLayerArgs in include/teb_b200.h.
 *
 *   k_costmap_voxel_layer   one CTA of VL_THREADS per robot; the robot's voxel row (4 B per cell), its layer row and a
 *                           visited bitmap in dynamic shared memory: thread 0 decides the status and the origins; both
 *                           rows are filled with their defaults and the previous rows scattered into them shifted
 *                           (16-byte loads); each thread walks the rays of its points with atomicAnd on the columns and
 *                           sets the visited bits; one pass writes the visited cells' bytes from their final columns;
 *                           each thread marks its points with atomicOr; warp 0 clears the footprint's column spans; then
 *                           both rows are stored in place and the master row combined, in 16-byte stores
 *
 * Clearing only removes bits from a column and marking only adds them, so the last atomic on a column sees its final
 * state (the argument at TebVoxelLayerArgs): a mark writes 254 when the column it leaves has more marked bits than
 * mark_threshold, which every later mark of the column then also writes, and the clearing bytes are written after a
 * barrier from the final columns. __syncthreads at the phase boundaries is the only order kept.
 */
#pragma once

#include <climits>
#include <cstdint>

#include "teb_costmap_obstacle_layer.cuh"

namespace tebgpu {

constexpr int VL_THREADS = OL_THREADS;   /* ol_load_row / ol_store_row stride by OL_THREADS */

/* the launch's parameter block: the arguments, the sources and the footprint copied from the host */
struct VoxelLayerDev {
  TebVoxelLayerArgs a;
  TebObservationSource src[TEB_VOXEL_LAYER_MAX_SOURCES];
  double fp[TEB_COSTMAP_FOOTPRINT_MAX][2];
};

/* dynamic shared memory of a row of cap cells: the column words, the layer bytes and the visited bits, each of cap
 * rounded up to 32 cells (164 bytes per 32 cells) */
TEB_HD inline long long voxel_layer_smem(long long cap) {
  const long long c = (cap + 31) & ~31LL;
  return c * 4 + c + c / 8;
}

/* TEB_VOXEL_LAYER_* of robot s; on OK or ORIGIN_MISMATCH also the snapped layer origin and the whole-cell move */
TEB_HD inline int voxel_layer_status(const TebVoxelLayerArgs& a, int s, double* nox, double* noy, double* cx,
                                     double* cy) {
  const long long sx = a.grid[2 * s], sy = a.grid[2 * s + 1];
  const double r = a.origin[3 * (size_t)s + 2];
  const double lox = a.layer_origin[2 * (size_t)s], loy = a.layer_origin[2 * (size_t)s + 1];
  const double rx = a.robot[3 * (size_t)s], ry = a.robot[3 * (size_t)s + 1];
  if (sx < 1 || sy < 1 || sx * sy > a.cell_cap || !(r > 0.0) || !isfinite(r) || !isfinite(lox) || !isfinite(loy) ||
      !isfinite(rx) || !isfinite(ry))
    return TEB_VOXEL_LAYER_BAD_GRID;
  for (int k = 0; k < a.K; ++k) {
    const int n = a.point_count[(size_t)s * a.K + k];
    if (n < 0 || n > a.P_cap) return TEB_VOXEL_LAYER_BAD_POINTS;
  }
  *cx = costmap_window_cells(lox, rx, (int)sx, r);
  *cy = costmap_window_cells(loy, ry, (int)sy, r);
  *nox = teb_add(lox, teb_mul(*cx, r));
  *noy = teb_add(loy, teb_mul(*cy, r));
  if (a.mode == TEB_VOXEL_LAYER_COMBINE &&
      (!ol_same_bits(*nox, a.origin[3 * (size_t)s]) || !ol_same_bits(*noy, a.origin[3 * (size_t)s + 1])))
    return TEB_VOXEL_LAYER_ORIGIN_MISMATCH;
  return TEB_VOXEL_LAYER_OK;
}

/* VoxelLayer::worldToMap3DFloat; a NaN quotient or one not below the size is off the grid */
__device__ __forceinline__ bool vl_world_to_map3(double wx, double wy, double wz, double ox, double oy, double oz,
                                                 double r, double zr, int sx, int sy, int Z, double* mx, double* my,
                                                 double* mz) {
  if (wx < ox || wy < oy || wz < oz) return false;
  *mx = teb_add(wx, -ox) / r;
  *my = teb_add(wy, -oy) / r;
  *mz = teb_add(wz, -oz) / zr;
  return *mx < (double)sx && *my < (double)sy && *mz < (double)Z;
}

/* VoxelGrid::raytraceLine with bresenham3D and ClearVoxelInMap's column update: every voxel visited loses its two bits
 * (shared-memory atomicAnd) and its cell's visited bit is set; the layer bytes are written after the phase */
__device__ __forceinline__ void vl_clear_ray(uint32_t* vox, uint32_t* vis, double x0, double y0, double z0, double x1,
                                             double y1, double z1, int sx, unsigned max_length) {
  const int ix0 = (int)x0, iy0 = (int)y0, iz0 = (int)z0;
  const int dx = (int)x1 - ix0, dy = (int)y1 - iy0, dz = (int)z1 - iz0;
  const unsigned adx = (unsigned)abs(dx), ady = (unsigned)abs(dy), adz = (unsigned)abs(dz);
  const int odx = dx > 0 ? 1 : -1, ody = (dy > 0 ? 1 : -1) * sx, odz = dz > 0 ? 1 : -1; /* sign(0) is -1 */
  const double ex = teb_add(x0, -x1), ey = teb_add(y0, -y1), ez = teb_add(z0, -z1);
  const double dist = sqrt(teb_add(teb_add(teb_mul(ex, ex), teb_mul(ey, ey)), teb_mul(ez, ez)));
  const double q = (double)max_length / dist;
  const double scale = q < 1.0 ? q : 1.0;                         /* std::min(1.0, q): 1 for NaN */
  /* the major axis a and the minors b, c; z is c unless z dominates, then it is a (and c is y) */
  const bool xdom = adx >= max(ady, adz), ydom = !xdom && ady >= adz, zdom = !xdom && !ydom;
  const unsigned da = xdom ? adx : ydom ? ady : adz;
  const unsigned db = xdom ? ady : adx;
  const unsigned dc = zdom ? ady : adz;
  const int oa = xdom ? odx : ydom ? ody : odz, ob = xdom ? ody : odx, oc = zdom ? ody : odz;
  const unsigned end = min((unsigned)teb_mul(scale, (double)da), da);
  unsigned offset = (unsigned)(iy0 * sx + ix0);
  uint32_t zmask = 0x10001u << iz0;
  int eb = (int)(da / 2), ec = (int)(da / 2);
  auto visit = [&]() {
    atomicAnd(&vox[offset], ~zmask);
    const uint32_t bit = 1u << (offset & 31);
    if (!(vis[offset >> 5] & bit)) atomicOr(&vis[offset >> 5], bit);
  };
  for (unsigned i = 0; i < end; ++i) {
    visit();
    if (zdom) zmask = oa > 0 ? zmask << 1 : zmask >> 1;
    else offset += oa;
    eb += (int)db;
    ec += (int)dc;
    if ((unsigned)eb >= da) {
      offset += ob;
      eb -= (int)da;
    }
    if ((unsigned)ec >= da) {
      if (zdom) offset += oc;
      else zmask = oc > 0 ? zmask << 1 : zmask >> 1;
      ec -= (int)da;
    }
  }
  visit();
}

/* f(c, row[c]) for every c < cap of a word row, in 16-byte loads where the row is aligned and single words at its ends */
template <class Fn>
__device__ __forceinline__ void vl_load_words(const uint32_t* row, int cap, Fn f) {
  const int tid = threadIdx.x;
  const int head = min(cap, (int)(((16 - (reinterpret_cast<uintptr_t>(row) & 15)) & 15) >> 2));
  const int groups = (cap - head) >> 2, tail = head + (groups << 2);
  for (int c = tid; c < head; c += VL_THREADS) f(c, row[c]);
  for (int c = tail + tid; c < cap; c += VL_THREADS) f(c, row[c]);
  for (int g = tid; g < groups; g += VL_THREADS) {
    const int c0 = head + (g << 2);
    const uint4 in = *reinterpret_cast<const uint4*>(row + c0);
    f(c0, in.x);
    f(c0 + 1, in.y);
    f(c0 + 2, in.z);
    f(c0 + 3, in.w);
  }
}

/* row[c] = src[c] for every c < cap of a word row, in 16-byte stores where the row is aligned */
__device__ __forceinline__ void vl_store_words(uint32_t* row, int cap, const uint32_t* src) {
  const int tid = threadIdx.x;
  const int head = min(cap, (int)(((16 - (reinterpret_cast<uintptr_t>(row) & 15)) & 15) >> 2));
  const int groups = (cap - head) >> 2, tail = head + (groups << 2);
  for (int c = tid; c < head; c += VL_THREADS) row[c] = src[c];
  for (int c = tail + tid; c < cap; c += VL_THREADS) row[c] = src[c];
  for (int g = tid; g < groups; g += VL_THREADS) {
    const int c0 = head + (g << 2);
    *reinterpret_cast<uint4*>(row + c0) = make_uint4(src[c0], src[c0 + 1], src[c0 + 2], src[c0 + 3]);
  }
}

__global__ void __launch_bounds__(VL_THREADS) k_costmap_voxel_layer(const __grid_constant__ VoxelLayerDev d) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ int s_st, s_cx, s_cy, s_flags;
  __shared__ double s_o[2];
  __shared__ int s_vx[TEB_COSTMAP_FOOTPRINT_MAX], s_vy[TEB_COSTMAP_FOOTPRINT_MAX];
  const TebVoxelLayerArgs& a = d.a;
  const int s = blockIdx.x, tid = threadIdx.x, cap = a.cell_cap, cap32 = (cap + 31) & ~31;
  uint32_t* svox = reinterpret_cast<uint32_t*>(smem);
  uint8_t* slay = smem + 4 * (size_t)cap32;
  uint32_t* svis = reinterpret_cast<uint32_t*>(slay + cap32);
  const bool standalone = a.mode == TEB_VOXEL_LAYER_STANDALONE;
  const uint8_t mdef = (uint8_t)a.master_default, ldef = a.track_unknown_space ? 255 : 0;
  uint32_t* vrow = a.voxels + (size_t)s * cap;
  uint8_t* lrow = a.layer + (size_t)s * cap;
  uint8_t* mrow = a.cost + (size_t)s * cap;
  if (tid == 0) {
    double nox = 0, noy = 0, cx = 0, cy = 0;
    const int st = voxel_layer_status(a, s, &nox, &noy, &cx, &cy);
    s_st = st;
    s_flags = 0;
    a.status[s] = st;
    if (st == TEB_VOXEL_LAYER_OK) {
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
  if (s_st != TEB_VOXEL_LAYER_OK) {
    if (standalone) ol_store_row<false>(mrow, cap, [&](int, uint8_t) { return mdef; });
    return;
  }
  const int sx = a.grid[2 * s], sy = a.grid[2 * s + 1], ncell = sx * sy, Z = a.z_voxels;
  const double r = a.origin[3 * (size_t)s + 2], ox = s_o[0], oy = s_o[1], oz = a.origin_z, zr = a.z_resolution;
  const double H = a.max_obstacle_height;
  const int mt = a.mark_threshold, ut = a.unknown_threshold + (16 - Z);

  /* 1. both rows at their defaults and no cell visited, then the previous rows' cells moved by (-cx, -cy) */
  const uint32_t dw = ldef * 0x01010101u, uw = TEB_VOXEL_LAYER_UNKNOWN_COLUMN;
  for (int g = tid; g < cap32 >> 2; g += VL_THREADS) reinterpret_cast<uint4*>(svox)[g] = make_uint4(uw, uw, uw, uw);
  for (int g = tid; g < cap32 >> 4; g += VL_THREADS) reinterpret_cast<uint4*>(slay)[g] = make_uint4(dw, dw, dw, dw);
  for (int g = tid; g < cap32 >> 5; g += VL_THREADS) svis[g] = 0;
  __syncthreads();
  if (s_cx != INT_MAX) {
    const int cx = s_cx, cy = s_cy;
    auto moved = [&](int c) {
      if (c >= ncell) return -1;
      const int j = c / sx, i = c - j * sx, ni = i - cx, nj = j - cy;
      return (ni >= 0 && ni < sx && nj >= 0 && nj < sy) ? nj * sx + ni : -1;
    };
    vl_load_words(vrow, cap, [&](int c, uint32_t v) {
      const int n = moved(c);
      if (n >= 0) svox[n] = v;
    });
    ol_load_row(lrow, cap, [&](int c, uint8_t v) {
      const int n = moved(c);
      if (n >= 0) slay[n] = v;
    });
  }
  __syncthreads();

  /* 2. + 3. clearing from every clearing source: the rays' columns, then the visited cells' bytes */
  const double ex = teb_add(ox, teb_mul(teb_add((double)(sx - 1), 0.5), r));   /* getSizeInMetersX */
  const double ey = teb_add(oy, teb_mul(teb_add((double)(sy - 1), 0.5), r));
  for (int k = 0; k < a.K; ++k) {
    const TebObservationSource& src = d.src[k];
    if (!src.clearing) continue;
    const size_t sk = (size_t)s * a.K + k;
    const double* so = a.sensor_origin + 3 * sk;
    const double sox = so[0], soy = so[1], soz = so[2];
    double x0, y0, z0;
    if (!vl_world_to_map3(sox, soy, soz, ox, oy, oz, r, zr, sx, sy, Z, &x0, &y0, &z0)) {
      if (tid == 0) s_flags |= TEB_VOXEL_LAYER_SENSOR_OFF_MAP(k);
      continue;
    }
    const double rc = fmax(0.0, ceil(src.raytrace_range / r));
    const unsigned max_length = rc >= 4294967295.0 ? 4294967295u : (unsigned)rc;
    const int n = a.point_count[sk];
    const float* pts = a.points + sk * a.P_cap * 3;
    for (int p = tid; p < n; p += VL_THREADS) {
      const double pz = pts[3 * p + 2];
      if (!(src.min_obstacle_height <= pz && pz <= src.max_obstacle_height)) continue;
      const double px = pts[3 * p], py = pts[3 * p + 1];
      const double da = teb_add(px, -sox), db = teb_add(py, -soy), dc = teb_add(pz, -soz);
      const double dist = sqrt(teb_add(teb_add(teb_mul(da, da), teb_mul(db, db)), teb_mul(dc, dc)));
      double f = teb_add(dist, -teb_mul(2.0, r)) / dist;
      f = f < 1.0 ? f : 1.0;
      f = f < 0.0 ? 0.0 : f;
      const double wx = teb_add(teb_mul(f, da), sox), wy = teb_add(teb_mul(f, db), soy), wz = teb_add(teb_mul(f, dc), soz);
      const double ea = teb_add(wx, -sox), eb = teb_add(wy, -soy), ec = teb_add(wz, -soz);
      double t = 1.0, u;
      if (wz > H) {
        u = teb_add(teb_add(H, -0.01), -soz) / ec;
        t = u < t ? u : t;
        t = 0.0 < t ? t : 0.0;
      } else if (wz < oz) {
        u = teb_add(oz, -soz) / ec;
        t = u < t ? u : t;
      }
      if (wx < ox) { u = teb_add(ox, -sox) / ea; t = u < t ? u : t; }
      if (wy < oy) { u = teb_add(oy, -soy) / eb; t = u < t ? u : t; }
      if (wx > ex) { u = teb_add(ex, -sox) / ea; t = u < t ? u : t; }
      if (wy > ey) { u = teb_add(ey, -soy) / eb; t = u < t ? u : t; }
      double x1, y1, z1;
      if (vl_world_to_map3(teb_add(sox, teb_mul(ea, t)), teb_add(soy, teb_mul(eb, t)), teb_add(soz, teb_mul(ec, t)), ox,
                           oy, oz, r, zr, sx, sy, Z, &x1, &y1, &z1))
        vl_clear_ray(svox, svis, x0, y0, z0, x1, y1, z1, sx, max_length);
    }
  }
  __syncthreads();
  for (int c = tid; c < ncell; c += VL_THREADS) {
    if (!((svis[c >> 5] >> (c & 31)) & 1u)) continue;
    const uint32_t col = svox[c];
    if (__popc(col >> 16) > mt) continue;                                  /* ClearVoxelInMap leaves the cell */
    slay[c] = __popc(((col >> 16) ^ col) & 0xFFFFu) <= ut ? 0 : TEB_COSTMAP_NO_INFORMATION;
  }
  __syncthreads();

  /* 4. marking from every marking source */
  for (int k = 0; k < a.K; ++k) {
    const TebObservationSource& src = d.src[k];
    if (!src.marking) continue;
    const size_t sk = (size_t)s * a.K + k;
    const double* so = a.sensor_origin + 3 * sk;
    const double sox = so[0], soy = so[1], soz = so[2];
    const double sq_range = teb_mul(src.obstacle_range, src.obstacle_range);
    const int n = a.point_count[sk];
    const float* pts = a.points + sk * a.P_cap * 3;
    for (int p = tid; p < n; p += VL_THREADS) {
      const double pz = pts[3 * p + 2];
      if (!(src.min_obstacle_height <= pz && pz <= src.max_obstacle_height)) continue;
      if (pz > H) continue;
      const double px = pts[3 * p], py = pts[3 * p + 1];
      const double ddx = teb_add(px, -sox), ddy = teb_add(py, -soy), ddz = teb_add(pz, -soz);
      if (teb_add(teb_add(teb_mul(ddx, ddx), teb_mul(ddy, ddy)), teb_mul(ddz, ddz)) >= sq_range) continue;
      double qx, qy, qz;
      if (!vl_world_to_map3(px, py, pz < oz ? oz : pz, ox, oy, oz, r, zr, sx, sy, Z, &qx, &qy, &qz)) continue;
      const int c = (int)qy * sx + (int)qx;
      const uint32_t m = 0x10001u << (int)qz;
      const uint32_t col = atomicOr(&svox[c], m) | m;
      if (__popc(col >> 16) > mt) slay[c] = TEB_COSTMAP_LETHAL;
    }
  }
  __syncthreads();

  /* 5. footprint clearing by warp 0, on the layer row only */
  if (a.F >= 3 && tid < 32)
    ol_clear_footprint(d.fp, a.F, a.robot + 3 * (size_t)s, ox, oy, r, sx, sy, s_vx, s_vy, slay, &s_flags,
                       TEB_VOXEL_LAYER_FOOTPRINT_OFF_MAP);
  __syncthreads();

  /* 6. both rows in place, then the master row combined over the window */
  vl_store_words(vrow, cap, svox);
  ol_store_row<false>(lrow, cap, [&](int c, uint8_t) { return slay[c]; });
  const int method = a.combination_method;
  auto combine = [&](int c, uint8_t m) -> uint8_t {
    if (standalone) m = mdef;
    if (c >= ncell) return m;
    return ol_combine(method, m, slay[c]);
  };
  if (standalone) ol_store_row<false>(mrow, cap, combine);
  else ol_store_row<true>(mrow, cap, combine);
  if (tid == 0 && a.flags) a.flags[s] = s_flags;
}

}  // namespace tebgpu
