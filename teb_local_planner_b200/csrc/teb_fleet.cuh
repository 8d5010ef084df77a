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

/* the outputs of the warp's robot r < R: the first min(needed, K) slots of its list (kq, slot `lane`) as rows of its
 * scene, custom_count, needed and status; a robot that does not write gets needed -1 and its status */
template <bool TABLE>
__device__ __forceinline__ void fleet_finish(const TebFleetArgs& a, const TebFleetTable& t, const FleetRobot& m, int r,
                                             int lane, int kq, int needed) {
  if (!m.valid) {
    if (lane == 0) {
      if (a.needed) a.needed[r] = -1;
      if (a.status) a.status[r] = m.st;
    }
    return;
  }
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

/* claims: [S] robots per scene from k_fleet_claim, or NULL when TebFleetArgs.scene is NULL (scene r, never shared).
 * TABLE: robot r is row t.first + r of t and the candidates are its T rows; otherwise t is not read. */
template <bool TABLE>
__global__ void __launch_bounds__(FLEET_THREADS) k_fleet_obstacles(const TebFleetArgs a, const int32_t* claims,
                                                                   const TebFleetTable t) {
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
      FLEET_TAKE(in, d2, q, K, lane, kd, kq, td, tq, needed);
    }
  }
  if (!live) return;
  fleet_finish<TABLE>(a, t, FleetRobot{xr, yr, wr, s, own, K, st, valid}, r, lane, kq, needed);
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
template <bool TABLE>
__global__ void __launch_bounds__(FLEET_THREADS) k_fleet_obstacles_grid(const TebFleetArgs a, const int32_t* claims,
                                                                        const TebFleetTable t, const FleetGrid g) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * FLEET_WARPS + (threadIdx.x >> 5);
  if (r >= a.R) return;                    /* warp-uniform */
  const int self = TABLE ? t.first + r : r;
  const int N = TABLE ? t.T : a.R;
  const FleetRobot m = fleet_robot<TABLE>(a, claims, t, r, true);
  const double range2 = __dmul_rn(a.range, a.range);
  double kd = INFINITY, td = INFINITY;
  int kq = INT_MAX, tq = INT_MAX;
  int needed = 0;
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
  fleet_finish<TABLE>(a, t, m, r, lane, kq, needed);
}

__global__ void __launch_bounds__(CLAIM_THREADS) k_fleet_publish(const TebFleetArgs a, const TebFleetTable t) {
  const int r = blockIdx.x * CLAIM_THREADS + threadIdx.x;
  if (r >= a.R) return;
  t.rows[(size_t)t.first + r] = fleet_row(a.pose + 3 * (size_t)r, a.last_cmd + 3 * (size_t)r, a.radius + r,
                                          a.world ? a.world[r] : 0);
}

}  // namespace tebgpu
