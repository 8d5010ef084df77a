/*
 * teb_fleet.cuh — the other robots of a fleet as custom obstacle rows of every robot's scene (tebgpu_fleet_obstacles /
 * _device). The contract is at TebFleetArgs in include/teb_b200.h.
 *
 *   k_fleet_claim           one thread per robot: counts the robots of every scene (only when TebFleetArgs.scene is given)
 *   k_fleet_obstacles       one warp per robot, FLEET_WARPS robots per CTA: all pairs, tiled through shared memory; TABLE
 *                           false takes the candidates from the caller's arrays (tebgpu_fleet_obstacles), true from the
 *                           rows of a TebFleetTable (tebgpu_fleet_obstacles_table)
 *   k_fleet_bin             one thread per candidate: its cell's bucket and its rank there, or the far list
 *   k_fleet_scatter         one thread per candidate: its index at its bucket's start (after the scan of the counts)
 *   k_fleet_obstacles_grid  one warp per robot, as k_fleet_obstacles: the candidates of the buckets of the robot's 3 x 3
 *                           cells and of the far list
 *   k_fleet_publish         one thread per robot: the robot's TebFleetRow (tebgpu_fleet_publish)
 *   k_fleet_publish_shaped  the same, and the row's heading and kind in the table's companions
 *
 * Both search kernels take a writer, what the kept list becomes: FleetCircles, one TEB_OBST_CIRCULAR row per neighbour
 * (the circle steps), or FleetShaped, each neighbour as its kind's parts from a TebFleetShapes library (the _shaped
 * steps). The contract is at TebFleetShapes in include/teb_b200.h. Beside the writer they take a selection rule:
 * FleetCentres, d2 <= range^2 on the centres (the circle steps and TebFleetShapes.select 0), or FleetFootprints, the
 * centres' prefilter at R' and then the gap from the context's footprint to the candidate's placed parts (fleet_gap, one
 * out-of-line routine both searches call), the gap taking d2's place as the list's key (DESIGN §4).
 *
 * The CTA stages FLEET_TILE robots' (x, y, world) at a time (the table build (x, y, world, live)); lane l of a warp tests candidates l, l + 32, ... of the
 * tile against its robot, and the warp keeps the nearest min(max_rows, C_cap - own) neighbours as a list sorted by
 * (d2, index), slot i in lane i. A candidate enters the list only when it is below the list's last slot, so after the
 * first few tiles almost every ballot is empty and the scan costs the distance test alone. The list is a total order
 * on distinct keys, so the rows do not depend on the tiling or on the order the candidates are met in: the grid kernel
 * meets them in bucket order, which the atomics of k_fleet_bin make differ from run to run, and writes the same bytes.
 *
 * The grid (DESIGN §4): a candidate at (x, y) of world w lies in the cell (w, floor(x / h), floor(y / h)), h =
 * max(range (1 + 2^-16), 2^-500), each operation rounded on its own; d2 <= range^2 as rounded implies cell coordinates
 * that differ by at most 1 on each axis while both |x / h|, |y / h| < 2^24. Cells hash to H buckets (H a power of two
 * >= 2 N, or one bucket), counted, scanned (cub::DeviceScan) and scattered. A candidate past the coordinate bound goes
 * to the far list, which every robot scans; a robot past it scans every candidate. When range^2 overflows every finite
 * pair is in range: h is then inf and every finite candidate is in the cell (w, 0, 0). Otherwise a candidate or robot
 * with a non-finite x or y is never in range (its d2 is NaN or inf) and takes no part.
 */
#pragma once

#include <climits>
#include <cmath>

#include "teb_device.cuh"
#include "teb_frame.h"

namespace tebgpu {

constexpr int FLEET_WARPS = 16;                    /* robots per CTA */
constexpr int FLEET_THREADS = FLEET_WARPS * 32;
constexpr int FLEET_TILE = FLEET_THREADS;          /* robots staged per tile: one load per thread */
constexpr int CLAIM_THREADS = 256;
constexpr double FLEET_H_MARGIN = 1.0 + 0x1p-16;   /* h = range * FLEET_H_MARGIN ... */
constexpr double FLEET_H_FLOOR = 0x1p-500;         /* ... at least FLEET_H_FLOOR */
constexpr double FLEET_CELL_BOUND = 0x1p24;        /* |x / h| or |y / h| at or past it: the far list */

/* (d2, q) order: nearest first, a tie to the lower index */
__device__ __forceinline__ bool fleet_less(double da, int qa, double db, int qb) {
  return da < db || (da == db && qa < qb);
}

/* the map-frame velocity a robot is published with, from its body command (bx, by) and sn, cs = sin, cos of its
 * heading: R(theta) (bx, by), then setCentroidVelocity's rule (obstacles.h:214-233), Eigen's norm() =
 * sqrt(squaredNorm()), of the body command: the rotation keeps the norm, and so the decision does not depend on the last
 * bits of sin / cos. dyn: 1 moving, 0 still with (0, 0). */
__device__ __forceinline__ void fleet_velocity(double bx, double by, double sn, double cs, double& vx, double& vy,
                                               int& dyn) {
  vx = __dsub_rn(__dmul_rn(cs, bx), __dmul_rn(sn, by));
  vy = __dadd_rn(__dmul_rn(sn, bx), __dmul_rn(cs, by));
  const bool moving = !(sqrt(__dadd_rn(__dmul_rn(bx, bx), __dmul_rn(by, by))) < 0.001);
  if (!moving) vx = vy = 0.0;
  dyn = moving ? 1 : 0;
}

/* the row robot q is published as, from its pose (x, y, theta), body command (vx, vy) and radius, with fleet_velocity.
 * The array build of k_fleet_obstacles, k_fleet_publish and k_fleet_publish_shaped write their rows from here, and the
 * shaped writer takes its velocities from fleet_velocity with the same sincos. */
__device__ __forceinline__ TebFleetRow fleet_row(const double* pose, const double* cmd, const double* radius, int world) {
  const double th = pose[2], bx = cmd[0], by = cmd[1];
  double sn, cs;
  sincos(th, &sn, &cs);
  TebFleetRow w;
  fleet_velocity(bx, by, sn, cs, w.vx, w.vy, w.dynamic);
  w.x = pose[0];
  w.y = pose[1];
  w.radius = *radius;
  w.world = world;
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

/* the warp's robot r (live: r < R): its position and world, scene, own rows, list length K and whether it writes. The
 * grid kernel's; k_fleet_obstacles keeps the same lines inline, since through this call its table build compiles to 8
 * more instructions. */
struct FleetRobot {
  double x, y;
  int w, s, own, K, st;
  bool valid;
};

template <bool TABLE>
__device__ __forceinline__ FleetRobot fleet_robot(const TebFleetArgs& a, const int32_t* claims, const TebFleetTable& t,
                                                  int r, bool live) {
  FleetRobot m;
  m.x = 0.0;
  m.y = 0.0;
  m.w = 0;
  m.s = -1;
  m.own = 0;
  m.K = 0;
  m.st = TEB_FLEET_BAD_INPUT;
  m.valid = false;
  if (live) {
    bool ok = true;
    if constexpr (TABLE) {
      const TebFleetRow& me = t.rows[t.first + r];
      m.x = me.x;
      m.y = me.y;
      m.w = me.world;
      ok = me.live != 0;
    } else {
      m.x = a.pose[3 * (size_t)r];
      m.y = a.pose[3 * (size_t)r + 1];
      m.w = a.world ? a.world[r] : 0;
    }
    m.s = a.scene ? a.scene[r] : r;
    if (ok && m.s >= 0 && m.s < a.S) {
      m.own = a.own_count ? a.own_count[m.s] : 0;
      if (m.own >= 0 && m.own <= a.C_cap) {
        if (claims && claims[m.s] != 1) m.st = TEB_FLEET_SHARED_SCENE;
        else m.valid = true;
      }
    }
    if (m.valid) m.K = min(a.max_rows, a.C_cap - m.own);
  }
  return m;
}

/* one candidate per lane met by the warp's robot: `in` is the exact test (world, live, q != self, d2 <= range2). needed
 * counts it; when it is below the list's last slot (td, tq) it is inserted into the list (kd, kq), the passing
 * candidates one at a time, lowest lane first. Warp-uniform: every lane runs it. Both kernels run this one text: a
 * macro, because the same code as a __forceinline__ function compiles k_fleet_obstacles to 16 (array) and 24 (table)
 * more instructions than it is inline. */
#define FLEET_TAKE(in, d2, q, K, lane, kd, kq, td, tq, needed)                               \
  do {                                                                                       \
    constexpr unsigned FULL_ = 0xffffffffu;                                                  \
    needed += __popc(__ballot_sync(FULL_, in));                                              \
    bool pass_ = in && K > 0 && fleet_less(d2, q, td, tq);                                   \
    unsigned pm_ = __ballot_sync(FULL_, pass_);                                              \
    while (pm_) {                                                                            \
      const int src_ = __ffs(pm_) - 1;                                                       \
      const double cd_ = __shfl_sync(FULL_, d2, src_);                                       \
      const int cq_ = __shfl_sync(FULL_, q, src_);                                           \
      const int pos_ = __popc(__ballot_sync(FULL_, lane < K && fleet_less(kd, kq, cd_, cq_))); \
      const double ud_ = __shfl_up_sync(FULL_, kd, 1);                                       \
      const int uq_ = __shfl_up_sync(FULL_, kq, 1);                                          \
      if (lane < K) {                                                                        \
        if (lane == pos_) { kd = cd_; kq = cq_; }                                            \
        else if (lane > pos_) { kd = ud_; kq = uq_; }                                        \
      }                                                                                      \
      td = __shfl_sync(FULL_, kd, K - 1);                                                    \
      tq = __shfl_sync(FULL_, kq, K - 1);                                                    \
      pass_ = pass_ && lane != src_ && fleet_less(d2, q, td, tq);                            \
      pm_ = __ballot_sync(FULL_, pass_);                                                     \
    }                                                                                        \
  } while (0)

/* the writers of fleet_finish: what a kept list becomes. FleetCircles: each neighbour one TEB_OBST_CIRCULAR row of its
 * radius (the circle steps); FleetShaped: each neighbour its kind's parts (the _shaped steps). */
struct FleetCircles {
  static constexpr int MIN_CTAS = 0;   /* __launch_bounds__' minimum CTAs per SM: 0 leaves it to ptxas (40 registers) */
  /* the first min(needed, K) slots of the list (kq, slot `lane`) as rows of the robot's scene, custom_count, needed and
   * status */
  template <bool TABLE>
  __device__ __forceinline__ void write(const TebFleetArgs& a, const TebFleetTable& t, const FleetRobot& m, int r,
                                        int lane, int kq, int needed) const {
    const int written = min(needed, m.K);
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
      a.custom[(size_t)m.s * a.C_cap + m.own + lane] = o;
    }
    if (lane == 0) {
      a.custom_count[m.s] = m.own + written;
      if (a.needed) a.needed[r] = needed;
      if (a.status) a.status[r] = written < needed ? TEB_FLEET_TRUNCATED : TEB_FLEET_WRITTEN;
    }
  }
};

/* one part of a shape library as the device reads it: its type, the radius (Circular), the body point (Point, Circular),
 * and for Line / Polygon its point count and offset among its kind's written points */
struct FleetPart {
  double cx, cy, radius;
  int32_t type, nv, woff, _pad;
};

/* a TebFleetShapes library on the device (the context's copy, built by the launcher in teb_cabi.cu) and the call's
 * per-robot arrays */
struct FleetLib {
  const FleetPart* part;       /* [P] */
  const int32_t* kpart;        /* [K + 1] kind k is parts kpart[k] .. kpart[k + 1] - 1 */
  const int32_t* kvert;        /* [K + 1] kind k writes the points wv[kvert[k] .. kvert[k + 1]) */
  const double* wv;            /* [.][2] the Line / Polygon points of every kind, kind by kind, part by part */
  int K, PV_cap;
  const int32_t* kind;         /* TebFleetShapes' per-robot arrays */
  const int32_t* own_v;
  double* cv;
  double* heading;
  int32_t* row_kind;
};

constexpr int FLEET_NO_FIT = 1 << 20;   /* the parts of a neighbour of an unknown kind: more than any scene holds */

/* body point (ux, uy) of a robot at (x, y) with sin / cos (sn, cs) of its heading: p + R(theta) u, every operation
 * rounded on its own; (0, 0) gives p unchanged */
__device__ __forceinline__ void fleet_place(double x, double y, double sn, double cs, double ux, double uy, double& px,
                                            double& py) {
  if (ux == 0.0 && uy == 0.0) {
    px = x;
    py = y;
    return;
  }
  px = __dadd_rn(x, __dsub_rn(__dmul_rn(cs, ux), __dmul_rn(sn, uy)));
  py = __dadd_rn(y, __dadd_rn(__dmul_rn(sn, ux), __dmul_rn(cs, uy)));
}

struct FleetShaped {
  /* one CTA per SM: under ptxas' default bound of 64 registers for 512 threads the writer spills; with one CTA the
   * instantiations take 118 / 120 registers and spill nothing */
  static constexpr int MIN_CTAS = 1;
  FleetLib L;
  /* lane i holds slot i: its kind's part and point counts, inclusive warp scans of both, and the longest prefix of the
   * kept list that fits the scene's rows and vertices; then neighbour by neighbour, the lanes place its points (lane v
   * point v) and write its parts (lane p part p); then the Line / Polygon rows take their centroids from the points */
  template <bool TABLE>
  __device__ __forceinline__ void write(const TebFleetArgs& a, const TebFleetTable& t, const FleetRobot& m, int r,
                                        int lane, int kq, int needed) const {
    constexpr unsigned FULL = 0xffffffffu;
    const int vown = L.own_v ? L.own_v[m.s] : 0;
    if (vown < 0 || vown > L.PV_cap) {
      if (lane == 0) {
        if (a.needed) a.needed[r] = -1;
        if (a.status) a.status[r] = TEB_FLEET_BAD_INPUT;
      }
      return;
    }
    const int listed = min(needed, m.K);
    /* lane i < listed: its neighbour's kind and the sin / cos of its heading, taken first, while little else is live
     * across sincos' call to its slow path */
    int kd = 0, np = 0, nv = 0;
    double sn = 0.0, cs = 1.0;
    if (lane < listed) {
      kd = TABLE ? L.row_kind[kq] : L.kind[kq];
      sincos(TABLE ? L.heading[kq] : a.pose[3 * (size_t)kq + 2], &sn, &cs);
      if (kd >= 0 && kd < L.K) {
        np = __ldg(L.kpart + kd + 1) - __ldg(L.kpart + kd);
        nv = __ldg(L.kvert + kd + 1) - __ldg(L.kvert + kd);
      } else {
        np = FLEET_NO_FIT;
      }
    }
    int sp = np, sv = nv;
    for (int o = 1; o < 32; o <<= 1) {
      const int up = __shfl_up_sync(FULL, sp, o), uv = __shfl_up_sync(FULL, sv, o);
      if (lane >= o) {
        sp += up;
        sv += uv;
      }
    }
    /* sp and sv grow with the lane, so the lanes that fit are a prefix */
    const bool fits = lane < listed && sp <= a.C_cap - m.own && sv <= L.PV_cap - vown;
    const int n = __popc(__ballot_sync(FULL, fits));
    /* lane i < n: its neighbour's position and velocity, the circle row's */
    double x = 0.0, y = 0.0, vx = 0.0, vy = 0.0;
    int dyn = 0;
    if (lane < n) {
      const size_t q = (size_t)kq;
      if constexpr (TABLE) {
        const TebFleetRow& w = t.rows[q];
        x = w.x;
        y = w.y;
        vx = w.vx;
        vy = w.vy;
        dyn = w.dynamic;
      } else {
        x = a.pose[3 * q];
        y = a.pose[3 * q + 1];
        fleet_velocity(a.last_cmd[3 * q], a.last_cmd[3 * q + 1], sn, cs, vx, vy, dyn);
      }
    }
    const int rb = m.own + sp - np, vb = vown + sv - nv;
    const size_t srow = (size_t)m.s * a.C_cap;
    double* const cv = L.cv + (size_t)m.s * L.PV_cap * 2;
    for (int j = 0; j < n; ++j) {
      const double jx = __shfl_sync(FULL, x, j), jy = __shfl_sync(FULL, y, j);
      const double jsn = __shfl_sync(FULL, sn, j), jcs = __shfl_sync(FULL, cs, j);
      const int jk = __shfl_sync(FULL, kd, j), jnv = __shfl_sync(FULL, nv, j), jvb = __shfl_sync(FULL, vb, j);
      const int w0 = __ldg(L.kvert + jk);
      for (int v = lane; v < jnv; v += 32) {
        const double2 u = __ldg(reinterpret_cast<const double2*>(L.wv) + w0 + v);
        double px, py;
        fleet_place(jx, jy, jsn, jcs, u.x, u.y, px, py);
        cv[2 * (size_t)(jvb + v)] = px;
        cv[2 * (size_t)(jvb + v) + 1] = py;
      }
      const double jvx = __shfl_sync(FULL, vx, j), jvy = __shfl_sync(FULL, vy, j);
      const int jdyn = __shfl_sync(FULL, dyn, j), jnp = __shfl_sync(FULL, np, j), jrb = __shfl_sync(FULL, rb, j);
      if (lane < jnp) {
        const FleetPart& P = L.part[__ldg(L.kpart + jk) + lane];
        TebObstacle o;
        o.vx = jvx;
        o.vy = jvy;
        o.radius = 0.0;
        o.dynamic = jdyn;
        o.type = __ldg(&P.type);
        o.vertex_begin = 0;
        o.vertex_count = 0;
        o._pad = 0.0;
        if (o.type == TEB_OBST_POINT || o.type == TEB_OBST_CIRCULAR) {
          if (o.type == TEB_OBST_CIRCULAR) o.radius = __ldg(&P.radius);
          fleet_place(jx, jy, jsn, jcs, __ldg(&P.cx), __ldg(&P.cy), o.x, o.y);
        } else {
          o.x = o.y = 0.0;   /* the centroid, below */
          o.vertex_begin = jvb + __ldg(&P.woff);
          o.vertex_count = __ldg(&P.nv);
        }
        a.custom[srow + jrb + lane] = o;
      }
    }
    const int total = n ? __shfl_sync(FULL, sp, n - 1) : 0;
    /* the Line / Polygon rows' centroids from their placed points, row by row over the lanes: apart from the loop above,
     * where the calls of the division and the square root would have its state live across them */
    __syncwarp();
    for (int i = lane; i < total; i += 32) {
      TebObstacle& o = a.custom[srow + m.own + i];
      if (o.type != TEB_OBST_LINE && o.type != TEB_OBST_POLYGON) continue;
      const double* d = cv + 2 * (size_t)o.vertex_begin;
      if (o.type == TEB_OBST_LINE) {
        o.x = teb_mul(0.5, teb_add(d[0], d[2]));
        o.y = teb_mul(0.5, teb_add(d[1], d[3]));
        continue;
      }
      int k = o.vertex_count;   /* finalizePolygon, as TebFrameArgs' step finalises a moved polygon */
      if (teb_eigen_is_approx(d[0], d[1], d[2 * k - 2], d[2 * k - 1])) --k;
      double c[2];
      teb_polygon_centroid(d, k, c);
      o.x = c[0];
      o.y = c[1];
      o.vertex_count = k;
    }
    if (lane == 0) {
      a.custom_count[m.s] = m.own + total;
      if (a.needed) a.needed[r] = needed;
      if (a.status) a.status[r] = n < needed ? TEB_FLEET_TRUNCATED : TEB_FLEET_WRITTEN;
    }
  }
};

/* the selection rules of the search kernels (TebFleetShapes.select), beside the writer. FleetCentres: d2 <= range^2 on
 * the centres, key d2 (the circle steps and select = TEB_FLEET_SELECT_CENTRES). FleetFootprints: the centres' prefilter
 * d2 <= pre^2, then the exact test gap <= range, key gap, the gap from fleet_gap (only with the FleetShaped writer,
 * whose library places the candidate's parts). reach(a): the distance of the centres' test. */
struct FleetCentres {
  static constexpr bool EXACT = false;
  __device__ __forceinline__ double reach(const TebFleetArgs& a) const { return a.range; }
};

struct FleetFootprints {
  static constexpr bool EXACT = true;
  /* the grid builds keep 512 threads per CTA, and so ptxas' cap of 128 registers, with 28 bytes of spill stores and 84
   * of loads: 256 threads spill nothing (140 registers) but run one CTA of 8 warps per SM and took 1.6x the time at
   * 8192 and 32768 robots (DESIGN §8) */
  double pre;            /* R' = (range + E_r + E_lib)(1 + 2^-16), on the host (DESIGN §4) */
  const double* fp;      /* KParams.fp_geom of the context: its footprint definition (FP_*) */
  int fp_type;           /* TebParams.footprint_type of the context */
  __device__ __forceinline__ double reach(const TebFleetArgs&) const { return pre; }
};

/* the distance from the footprint (fp_type, fp) of a robot at (px, py) with cos / sin (c, s) of its heading to one
 * placed part: the points ov[0 .. ok) (Line, Polygon) or the point (ox, oy) (Point, Circular of radius orad). The pair
 * loop of generic_distance, value only, over the same inline pair routines (closest_on_segment, seg_seg_dist), so that
 * it is the optimizer's static distance (robot_obstacle_distance_only at t = 0) without passing the local point buffer
 * into the optimizer's out-of-line routine, whose loads would then no longer all be global. */
__device__ __forceinline__ double fleet_part_distance(int fp_type, const double* __restrict__ fp, double px, double py,
                                                      double c, double s, const double* ov, int ok, double ox,
                                                      double oy, double orad, int otype) {
  const bool olist = ov != nullptr;
  const bool obst_first = otype == TEB_OBST_LINE;
  const int oe = ok <= 2 ? 1 : ok;
  double best = 1.7976931348623157e308;
  const int nsub = fp_type == TEB_FOOTPRINT_TWO_CIRCLES ? 2 : 1;
  for (int sub = 0; sub < nsub; ++sub) {
    int rk = 1;
    double rrad = 0;
    if (fp_type == TEB_FOOTPRINT_CIRCULAR) rrad = fp[FP_RADIUS];
    else if (fp_type == TEB_FOOTPRINT_TWO_CIRCLES) rrad = sub == 0 ? fp[FP_FRONT_RAD] : fp[FP_REAR_RAD];
    else if (fp_type == TEB_FOOTPRINT_LINE) rk = 2;
    else if (fp_type == TEB_FOOTPRINT_POLYGON) rk = (int)fp[FP_COUNT];
    const int re = rk <= 2 ? 1 : rk;
    double sbest = 1.7976931348623157e308;
    for (int i = 0; i < re; ++i) {
      double r0x, r0y, r1x, r1y;
      if (fp_type == TEB_FOOTPRINT_LINE || fp_type == TEB_FOOTPRINT_POLYGON) {
        const double* lv = fp + (fp_type == TEB_FOOTPRINT_LINE ? FP_LINE : FP_VERTS);
        const int i1 = (i + 1) % rk;
        const double ax = lv[2 * i], ay = lv[2 * i + 1], bx = lv[2 * i1], by = lv[2 * i1 + 1];
        r0x = px + c * ax - s * ay; r0y = py + s * ax + c * ay;
        r1x = px + c * bx - s * by; r1y = py + s * bx + c * by;
      } else {
        double off = 0;
        if (fp_type == TEB_FOOTPRINT_TWO_CIRCLES) off = sub == 0 ? fp[FP_FRONT_OFF] : -fp[FP_REAR_OFF];
        r0x = r1x = px + off * c; r0y = r1y = py + off * s;
      }
      for (int j = 0; j < oe; ++j) {
        double o0x, o0y, o1x, o1y;
        if (olist) {
          const int j1 = (j + 1) % ok;
          o0x = ov[2 * j]; o0y = ov[2 * j + 1];
          o1x = ov[2 * j1]; o1y = ov[2 * j1 + 1];
        } else { o0x = o1x = ox; o0y = o1y = oy; }
        const int pk = olist ? ok : 1;
        double ax, ay, bx, by, d;
        if (rk == 1 && pk == 1) {
          d = sqrt((r0x - o0x) * (r0x - o0x) + (r0y - o0y) * (r0y - o0y));
        } else if (rk == 1) {
          closest_on_segment(r0x, r0y, o0x, o0y, o1x, o1y, bx, by);
          d = sqrt((r0x - bx) * (r0x - bx) + (r0y - by) * (r0y - by));
        } else if (pk == 1) {
          closest_on_segment(o0x, o0y, r0x, r0y, r1x, r1y, ax, ay);
          d = sqrt((o0x - ax) * (o0x - ax) + (o0y - ay) * (o0y - ay));
        } else if (obst_first) {
          d = seg_seg_dist(o0x, o0y, o1x, o1y, r0x, r0y, r1x, r1y, bx, by, ax, ay);
        } else {
          d = seg_seg_dist(r0x, r0y, r1x, r1y, o0x, o0y, o1x, o1y, ax, ay, bx, by);
        }
        if (d < sbest) sbest = d;
      }
    }
    const double dsub = sbest - orad - rrad;
    if (dsub <= best) best = dsub;
  }
  return best;
}

/* the gap from the footprint (fp_type, fp) of a robot at (rx, ry, rth) to the parts
 * of kind `kind` of a candidate at (qx, qy, qth): the minimum over the parts of fleet_part_distance, each part placed as
 * FleetShaped::write places and writes it (fleet_place with the same sincos, a Polygon finalised by the same closure
 * check). NaN pair values are skipped inside fleet_part_distance as generic_distance skips them, so with finite radii
 * no part's distance is NaN; -inf for a kind outside 0 .. K - 1, so that such a neighbour is kept first and ends its list
 * as the writer ends it. Out of line: both searches run this one routine, so they write the same
 * bytes; the robot's sin / cos are taken here, so that the searches keep one double live across their scans, not two. */
__device__ __noinline__ double fleet_gap(int fp_type, const double* fp, double rx, double ry, double rth,
                                         const FleetPart* part, const int32_t* kpart, const int32_t* kvert,
                                         const double* wv, int K, int kind, double qx, double qy, double qth) {
  if (kind < 0 || kind >= K) return -INFINITY;
  double rs, rc, sn, cs;
  sincos(rth, &rs, &rc);
  sincos(qth, &sn, &cs);
  double pts[2 * TEB_FLEET_MAX_KIND_VERTICES];
  const int p1 = __ldg(kpart + kind + 1), w0 = __ldg(kvert + kind);
  double g = INFINITY;
  for (int p = __ldg(kpart + kind); p < p1; ++p) {
    const FleetPart& P = part[p];
    const int type = __ldg(&P.type);
    double d;
    if (type == TEB_OBST_POINT || type == TEB_OBST_CIRCULAR) {
      double ox, oy;
      fleet_place(qx, qy, sn, cs, __ldg(&P.cx), __ldg(&P.cy), ox, oy);
      d = fleet_part_distance(fp_type, fp, rx, ry, rc, rs, nullptr, 1, ox, oy,
                              type == TEB_OBST_CIRCULAR ? __ldg(&P.radius) : 0.0, type);
    } else {
      int n = __ldg(&P.nv);
      const double2* u = reinterpret_cast<const double2*>(wv) + w0 + __ldg(&P.woff);
      for (int v = 0; v < n; ++v) {
        const double2 b = __ldg(u + v);
        fleet_place(qx, qy, sn, cs, b.x, b.y, pts[2 * v], pts[2 * v + 1]);
      }
      if (type == TEB_OBST_POLYGON && teb_eigen_is_approx(pts[0], pts[1], pts[2 * n - 2], pts[2 * n - 1])) --n;
      d = fleet_part_distance(fp_type, fp, rx, ry, rc, rs, pts, n, 0.0, 0.0, 0.0, type);
    }
    if (d < g) g = d;
  }
  return g;
}

/* the gap of candidate q (at (qx, qy)) of the warp's robot under FleetFootprints: its kind and heading from the
 * caller's arrays or the table's companions */
template <bool TABLE>
__device__ __forceinline__ double fleet_gap_of(const TebFleetArgs& a, const FleetLib& L, const FleetFootprints& f,
                                               double rx, double ry, double rth, size_t q, double qx, double qy) {
  const int kind = TABLE ? L.row_kind[q] : L.kind[q];
  const double th = TABLE ? L.heading[q] : a.pose[3 * q + 2];
  return fleet_gap(f.fp_type, f.fp, rx, ry, rth, L.part, L.kpart, L.kvert, L.wv, L.K, kind, qx, qy, th);
}

/* the warp's robot's heading (FleetFootprints): pose[r] of the array step, heading[first + r] of the table step */
template <bool TABLE>
__device__ __forceinline__ double fleet_robot_heading(const TebFleetArgs& a, const FleetLib& L, int r, int self) {
  return TABLE ? L.heading[self] : a.pose[3 * (size_t)r + 2];
}

/* the outputs of the warp's robot r < R through the writer w; a robot that does not write gets needed -1 and its status */
template <bool TABLE, class W>
__device__ __forceinline__ void fleet_finish(const TebFleetArgs& a, const TebFleetTable& t, const FleetRobot& m, int r,
                                             int lane, int kq, int needed, const W& w) {
  if (!m.valid) {
    if (lane == 0) {
      if (a.needed) a.needed[r] = -1;
      if (a.status) a.status[r] = m.st;
    }
    return;
  }
  w.template write<TABLE>(a, t, m, r, lane, kq, needed);
}

/* claims: [S] robots per scene from k_fleet_claim, or NULL when TebFleetArgs.scene is NULL (scene r, never shared).
 * TABLE: robot r is row t.first + r of t and the candidates are its T rows; otherwise t is not read. */
template <bool TABLE, class W = FleetCircles, class S = FleetCentres>
__global__ void __launch_bounds__(FLEET_THREADS, W::MIN_CTAS) k_fleet_obstacles(const TebFleetArgs a, const int32_t* claims,
                                                                   const TebFleetTable t, const W writer, const S sel) {
  __shared__ double sx[FLEET_TILE], sy[FLEET_TILE];
  __shared__ int sw[FLEET_TILE];
  __shared__ int sl[TABLE ? FLEET_TILE : 1];
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
  const double range2 = __dmul_rn(sel.reach(a), sel.reach(a));
  /* slot `lane` of the list (empty: +inf / INT_MAX, above every real key) and the key of slot K - 1 */
  double kd = INFINITY, td = INFINITY;
  int kq = INT_MAX, tq = INT_MAX;
  int needed = 0;
  double rth = 0.0;
  if constexpr (S::EXACT)
    if (valid) rth = fleet_robot_heading<TABLE>(a, writer.L, r, self);

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
      if constexpr (S::EXACT) {
        if (in) {
          d2 = fleet_gap_of<TABLE>(a, writer.L, sel, xr, yr, rth, (size_t)q, sx[j], sy[j]);
          in = d2 <= a.range;
        }
      }
      FLEET_TAKE(in, d2, q, K, lane, kd, kq, td, tq, needed);
    }
  }
  if (!live) return;
  fleet_finish<TABLE>(a, t, FleetRobot{xr, yr, wr, s, own, K, st, valid}, r, lane, kq, needed, writer);
}

/* the grid of one fleet step: context scratch sized by the launcher (teb_cabi.cu issue_fleet_grid) */
struct FleetGrid {
  int32_t* count;      /* [H + 1] candidates per bucket (count[H] stays 0), then nfar */
  int32_t* nfar;       /* [1] candidates in the far list */
  int32_t* start;      /* [H + 1] exclusive scan of count: bucket b is idx[start[b] .. start[b + 1]) */
  int32_t* key;        /* [N] the candidate's bucket, -1 when it is not binned */
  int32_t* rank;       /* [N] its place in its bucket */
  int32_t* idx;        /* [N] the binned candidates, bucket by bucket */
  int32_t* far;        /* [N] the far list, nfar entries */
  unsigned mask;       /* H - 1, 0 for one bucket */
  double h;            /* the cell side */
  bool fin2;           /* range^2 is finite */
};

/* the cell side of a step of range `range` (DESIGN §4), on the host */
inline double fleet_cell_side(double range) {
  const double range2 = range * range;
  if (!(range2 < INFINITY)) return INFINITY;
  const double h = range * FLEET_H_MARGIN;
  return h > FLEET_H_FLOOR ? h : FLEET_H_FLOOR;
}

/* the cell of a point: 0 binned at (cx, cy), 1 the far list, 2 never in range (a non-finite x or y with a finite
 * range^2) */
__device__ __forceinline__ int fleet_cell(double x, double y, const FleetGrid& g, int& cx, int& cy) {
  const double fx = __ddiv_rn(x, g.h), fy = __ddiv_rn(y, g.h);
  if (fabs(fx) < FLEET_CELL_BOUND && fabs(fy) < FLEET_CELL_BOUND) {
    cx = (int)floor(fx);
    cy = (int)floor(fy);
    return 0;
  }
  return g.fin2 && !(isfinite(x) && isfinite(y)) ? 2 : 1;
}

/* the bucket of the cell (w, cx, cy): a multiplicative mix of the three words, finished by a 32-bit avalanche */
__device__ __forceinline__ unsigned fleet_bucket(int w, int cx, int cy, unsigned mask) {
  unsigned k = (unsigned)cx * 0x9E3779B1u ^ (unsigned)cy * 0x85EBCA77u ^ (unsigned)w * 0xC2B2AE3Du;
  k ^= k >> 16;
  k *= 0x7FEB352Du;
  k ^= k >> 15;
  k *= 0x846CA68Bu;
  k ^= k >> 16;
  return k & mask;
}

/* candidate q's position, world and live flag */
template <bool TABLE>
__device__ __forceinline__ void fleet_candidate(const TebFleetArgs& a, const TebFleetTable& t, size_t q, double& x,
                                                double& y, int& w, bool& live) {
  if constexpr (TABLE) {
    const TebFleetRow& row = t.rows[q];
    x = row.x;
    y = row.y;
    w = row.world;
    live = row.live != 0;
  } else {
    x = a.pose[3 * q];
    y = a.pose[3 * q + 1];
    w = a.world ? a.world[q] : 0;
    live = true;
  }
}

template <bool TABLE>
__global__ void __launch_bounds__(CLAIM_THREADS) k_fleet_bin(const TebFleetArgs a, const TebFleetTable t,
                                                             const FleetGrid g) {
  const int q = blockIdx.x * CLAIM_THREADS + threadIdx.x;
  if (q >= (TABLE ? t.T : a.R)) return;
  double x, y;
  int w, b = -1, cx = 0, cy = 0;
  bool live;
  fleet_candidate<TABLE>(a, t, q, x, y, w, live);
  if (live) {                              /* padding is never a neighbour: not binned */
    const int c = fleet_cell(x, y, g, cx, cy);
    if (c == 0) {
      b = (int)fleet_bucket(w, cx, cy, g.mask);
      g.rank[q] = atomicAdd(&g.count[b], 1);
    } else if (c == 1) {
      g.far[atomicAdd(g.nfar, 1)] = q;
    }
  }
  g.key[q] = b;
}

__global__ void __launch_bounds__(CLAIM_THREADS) k_fleet_scatter(const int N, const FleetGrid g) {
  const int q = blockIdx.x * CLAIM_THREADS + threadIdx.x;
  if (q >= N) return;
  const int b = g.key[q];
  if (b >= 0) g.idx[g.start[b] + g.rank[q]] = q;
}

/* k_fleet_obstacles' step with the candidates taken from the grid: the buckets of the robot's 3 x 3 cells (a bucket two
 * cells share is scanned once, so no candidate is met twice) and the far list; a robot in the far list meets every
 * candidate, one never in range none. Every candidate met takes k_fleet_obstacles' exact test and list. */
template <bool TABLE, class W = FleetCircles, class S = FleetCentres>
__global__ void __launch_bounds__(FLEET_THREADS, W::MIN_CTAS) k_fleet_obstacles_grid(const TebFleetArgs a, const int32_t* claims,
                                                                        const TebFleetTable t, const FleetGrid g,
                                                                        const W writer, const S sel) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * FLEET_WARPS + (threadIdx.x >> 5);
  if (r >= a.R) return;                    /* warp-uniform */
  const int self = TABLE ? t.first + r : r;
  const int N = TABLE ? t.T : a.R;
  const FleetRobot m = fleet_robot<TABLE>(a, claims, t, r, true);
  const double range2 = __dmul_rn(sel.reach(a), sel.reach(a));
  double kd = INFINITY, td = INFINITY;
  int kq = INT_MAX, tq = INT_MAX;
  int needed = 0;
  double rth = 0.0;
  if constexpr (S::EXACT)
    if (m.valid) rth = fleet_robot_heading<TABLE>(a, writer.L, r, self);
  /* lane's candidate q (-1: none) through the exact test into the list */
  auto meet = [&](int q) {
    bool in = false;
    double d2 = 0.0;
    if (q >= 0 && q != self) {
      double x, y;
      int w;
      bool live;
      fleet_candidate<TABLE>(a, t, q, x, y, w, live);
      if (w == m.w && live) {
        const double dx = __dsub_rn(x, m.x), dy = __dsub_rn(y, m.y);
        d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
        in = d2 <= range2;
        if constexpr (S::EXACT) {
          if (in) {
            d2 = fleet_gap_of<TABLE>(a, writer.L, sel, m.x, m.y, rth, (size_t)q, x, y);
            in = d2 <= a.range;
          }
        }
      }
    }
    FLEET_TAKE(in, d2, q, m.K, lane, kd, kq, td, tq, needed);
  };
  if (m.valid) {
    int cx = 0, cy = 0;
    const int c = fleet_cell(m.x, m.y, g, cx, cy);
    if (c == 0) {
      for (int i = 0; i < 9; ++i) {
        const unsigned b = fleet_bucket(m.w, cx + i % 3 - 1, cy + i / 3 - 1, g.mask);
        bool seen = false;
        for (int k = 0; k < i; ++k) seen |= fleet_bucket(m.w, cx + k % 3 - 1, cy + k / 3 - 1, g.mask) == b;
        if (seen) continue;
        const int lo = g.start[b], hi = g.start[b + 1];
        for (int j = lo + lane; j - lane < hi; j += 32) meet(j < hi ? g.idx[j] : -1);
      }
      const int nf = *g.nfar;
      for (int j = lane; j - lane < nf; j += 32) meet(j < nf ? g.far[j] : -1);
    } else if (c == 1) {
      for (int q = lane; q - lane < N; q += 32) meet(q < N ? q : -1);
    }
  }
  fleet_finish<TABLE>(a, t, m, r, lane, kq, needed, writer);
}

__global__ void __launch_bounds__(CLAIM_THREADS) k_fleet_publish(const TebFleetArgs a, const TebFleetTable t) {
  const int r = blockIdx.x * CLAIM_THREADS + threadIdx.x;
  if (r >= a.R) return;
  t.rows[(size_t)t.first + r] = fleet_row(a.pose + 3 * (size_t)r, a.last_cmd + 3 * (size_t)r, a.radius + r,
                                          a.world ? a.world[r] : 0);
}

/* k_fleet_publish's row, and the row's heading and kind in the table's companions (tebgpu_fleet_publish_shaped) */
__global__ void __launch_bounds__(CLAIM_THREADS) k_fleet_publish_shaped(const TebFleetArgs a, const TebFleetTable t,
                                                                        const FleetLib L) {
  const int r = blockIdx.x * CLAIM_THREADS + threadIdx.x;
  if (r >= a.R) return;
  const size_t i = (size_t)t.first + r;
  t.rows[i] = fleet_row(a.pose + 3 * (size_t)r, a.last_cmd + 3 * (size_t)r, a.radius + r, a.world ? a.world[r] : 0);
  L.heading[i] = a.pose[3 * (size_t)r + 2];
  L.row_kind[i] = L.kind[r];
}

}  // namespace tebgpu
