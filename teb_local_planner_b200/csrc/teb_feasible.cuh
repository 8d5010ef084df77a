/*
 * teb_feasible.cuh — TebOptimalPlanner::isTrajectoryFeasible (optimal_planner.cpp:1250-1310) for every band of a batch,
 * against one of two world models:
 *
 *   k_feasible<GEOM, GT>             the obstacle table of the band's scene (tebgpu_check_feasible(_device));
 *   k_feasible_costmap                the scene's costmap raster, CostmapModel::footprintCost
 *                                     (tebgpu_check_feasible_costmap(_device)).
 *
 *   k_feasible   one CTA per band. Warp 0 clamps the look-ahead index, cuts it at the look-ahead distance (ballot over
 *                the poses), counts the samples of every segment (lane per segment, 64-bit) and scans them into query
 *                offsets. The CTA then generates the queries in blocks of FEAS_QB, every segment of a block on one
 *                thread with the reference's sequential accumulation, and tests them: a warp per query, in order; the
 *                world model decides the query with the warp's lanes. The first block that holds a non-free query is
 *                the last one. The world model only validates the band's scene and answers a query: look-ahead,
 *                offsets and generation are the same code for both.
 *
 * The table world. footprintCost(x, y, theta) == -1 of the reference means here: the context's footprint model placed at
 * (x, y, theta) has a distance <= collision_distance to some obstacle of the band's scene. The distance is
 * robot_obstacle_distance_only, the optimizer's own code (fast path, and the vertex-list path in the GEOM builds); every
 * one of the scene's obst_count rows is tested (lanes over the rows, __any_sync decides), dynamic obstacles at their
 * current position (a snapshot, no time prediction). A query none of whose distances is <= collision_distance but some
 * of whose distances are NaN is undecidable.
 *
 * The raster world. footprintCost as TebCostmapWorld defines it: the footprint outline walked cell by cell with
 * LineIterator, lanes over the cells of one edge in closed form (cell k steps the minor axis
 * (den / 2 + k numadd) / den times), a ballot finds the first negative code in walk order and the edges run in order,
 * so the first negative code of the reference's walk is the one returned. A thread per query would walk a few hundred
 * cells of a 16-vertex outline one dependent load at a time with lane-divergent lengths; the lanes over the cells keep
 * the loads of a warp independent and the kernel's warp-per-query structure unchanged. The raster is read through the
 * read-only path (__ldg), not staged: an outline touches a few hundred cells of a map of 10^4 - 10^5.
 *
 * Every product and sum that feeds a sample count, a query pose or a footprint vertex uses teb_mul / teb_add /
 * teb_normalize_theta of teb_plan.h, so FMA contraction cannot move a sample or a cell. The outputs do not depend on the
 * grid or the batch position.
 */
#pragma once

#include "teb_kernels.cuh"
#include "teb_plan.h"

namespace tebgpu {

constexpr int FEAS_THREADS = 256;      /* 8 warps per band */
constexpr int FEAS_QB = 256;           /* queries generated and tested per block */
constexpr int FEAS_MAX_POSES = 512;    /* n_cap limit of a context */
constexpr long long FEAS_INT_MAX = 2147483647LL;

struct FeasDev {
  int32_t B, n_cap, S, M_cap, PV_cap;
  const double* poses;
  const int32_t* n;
  const int32_t* scene_id;
  const TebObstacle* obstacles;
  const int32_t* obst_count;
  const double* obst_vertices;
  TebFeasibilityArgs a;
};

/* one segment i -> i+1 of the check (optimal_planner.cpp:1282-1291): delta_rot, delta_dist and the number of
 * intermediate poses. The reference converts the sample count to int; beyond that range it is undefined, here the
 * count saturates at INT_MAX - 1. */
struct FeasSeg { double dx, dy, dr; long long extra; };
__device__ __forceinline__ FeasSeg feas_segment(const double* p, const double* q, double inscribed, double ang_res) {
  FeasSeg s;
  s.dr = teb_normalize_theta(teb_normalize_theta(q[2]) - teb_normalize_theta(p[2]));
  s.dx = q[0] - p[0];
  s.dy = q[1] - p[1];
  const double norm = sqrt(teb_add(teb_mul(s.dx, s.dx), teb_mul(s.dy, s.dy)));
  s.extra = 0;
  if (fabs(s.dr) > ang_res || norm > inscribed) {
    const double ca = ceil(fabs(s.dr) / ang_res), cd = ceil(norm / inscribed);
    const double c = ca < cd ? cd : ca; /* std::max */
    s.extra = (c >= (double)FEAS_INT_MAX ? FEAS_INT_MAX : (long long)c) - 1;
  }
  return s;
}

/* the verdict of one query: 0 free, 1 colliding, 2 undecidable; one warp, lanes over the scene's M obstacles */
template <bool GEOM, bool GT>
__device__ __forceinline__ int feas_query(const KParams& kp, const TebObstacle* tab, const double* pool, int M, double x,
                                          double y, double th, double cdist, int lane) {
  const double c = cos(th), s = sin(th);
  bool hit = false, nan = false;
  for (int base = 0; base < M; base += 32) {
    const int m = base + lane;
    if (m < M) {
      const TebObstacle ob = tab[m];
      const double d = robot_obstacle_distance_only<GEOM>(kp, pool, x, y, c, s, ob, ob.x, ob.y, 0.0, 0.0);
      hit |= d <= cdist;
      nan |= d != d;
    }
    if (__any_sync(0xffffffffu, hit)) return 1;
  }
  return __any_sync(0xffffffffu, nan) ? 2 : 0;
}

/* The obstacle-table world (tebgpu_check_feasible): the scene's rows, staged in shared memory unless GT */
template <bool GEOM, bool GT>
struct FeasTable {
  using Param = KParams;
  const TebObstacle* tab;
  const double* pool;
  int M;
  /* this thread's part of the scene's validation (and staging); true: the band is answered with -1 */
  __device__ __forceinline__ bool begin(const FeasDev& fd, const KParams&, int sc, bool bad, unsigned char* smem, int tid) {
    M = bad ? 0 : fd.obst_count[sc];
    if (M < 0 || M > fd.M_cap) { bad = true; M = 0; }
    const TebObstacle* gtab = fd.obstacles + (size_t)(bad ? 0 : sc) * fd.M_cap;
    pool = fd.obst_vertices ? fd.obst_vertices + (size_t)(bad ? 0 : sc) * fd.PV_cap * 2 : nullptr;
    /* obstacle rows the batch cannot describe (as k_begin): staged into shared memory on the way */
    TebObstacle* stab = reinterpret_cast<TebObstacle*>(smem);
    bool bad_row = false;
    for (int m = tid; m < M; m += FEAS_THREADS) {
      const TebObstacle ob = gtab[m];
      if (!GT) stab[m] = ob;
      if (ob.type < TEB_OBST_POINT || ob.type > TEB_OBST_POLYGON) bad_row = true;
      else if (ob.type >= TEB_OBST_LINE && (ob.vertex_count < 1 || (ob.type != TEB_OBST_POLYGON && ob.vertex_count != 2) ||
                                            ob.vertex_begin < 0 || (long long)ob.vertex_begin + ob.vertex_count > fd.PV_cap))
        bad_row = true;
    }
    tab = GT ? gtab : stab;
    return bad || bad_row;
  }
  /* query j of the current block: 0 free, 1 colliding, 2 undecidable (one warp) */
  __device__ __forceinline__ int query(const FeasDev& fd, const KParams& kp, int, double x, double y, double th, int lane) const {
    return feas_query<GEOM, GT>(kp, tab, pool, M, x, y, th, fd.a.collision_distance, lane);
  }
  __device__ __forceinline__ void store(const FeasDev&, const KParams&, int, long long, int, int) const {}
};

/* The raster world (tebgpu_check_feasible_costmap): the launch's copy of TebCostmapWorld */
struct FeasRasterDev {
  int32_t cell_cap, F;
  const uint8_t* cost;
  const int32_t* grid;
  const double* origin;
  double* query_cost;
  double fp[TEB_COSTMAP_FOOTPRINT_MAX][2];
};

struct FeasRaster {
  using Param = FeasRasterDev;
  const uint8_t* map;
  const double (*fp)[2];
  double* s_cost;
  double ox, oy, r;
  int sx, sy;
  __device__ __forceinline__ bool begin(const FeasDev&, const FeasRasterDev& w, int sc, bool bad, unsigned char*, int tid) {
    __shared__ double s_fp[TEB_COSTMAP_FOOTPRINT_MAX][2];
    __shared__ double s_qcost[FEAS_QB];
    if (tid == 0) { /* constant offsets into the parameter block: no local copy of it */
#pragma unroll
      for (int i = 0; i < TEB_COSTMAP_FOOTPRINT_MAX; ++i)
        if (i < w.F) { s_fp[i][0] = w.fp[i][0]; s_fp[i][1] = w.fp[i][1]; }
    }
    fp = s_fp;
    s_cost = s_qcost;
    map = nullptr;
    if (bad) return true;
    sx = w.grid[2 * sc]; sy = w.grid[2 * sc + 1];
    ox = w.origin[3 * sc]; oy = w.origin[3 * sc + 1]; r = w.origin[3 * sc + 2];
    if (sx < 1 || sy < 1 || (long long)sx * sy > w.cell_cap) return true;
    if (!(isfinite(r) && r > 0) || !isfinite(ox) || !isfinite(oy)) return true;
    map = w.cost + (size_t)sc * w.cell_cap;
    return false;
  }
  /* Costmap2D::worldToMap; a quotient past the int range (or >= the size) is off the map */
  __device__ __forceinline__ bool to_map(double wx, double wy, int& mx, int& my) const {
    if (wx < ox || wy < oy) return false;
    const double qx = __ddiv_rn(teb_add(wx, -ox), r), qy = __ddiv_rn(teb_add(wy, -oy), r);
    if (!(qx < (double)sx && qy < (double)sy)) return false;
    mx = (int)qx; my = (int)qy;
    return true;
  }
  /* WorldModel::footprintCost's vertex k at (x, y) with c = cos theta, s = sin theta, then worldToMap */
  __device__ __forceinline__ bool vertex(int k, double x, double y, double c, double s, int& mx, int& my) const {
    const double fx = fp[k][0], fy = fp[k][1];
    return to_map(teb_add(x, teb_add(teb_mul(fx, c), -teb_mul(fy, s))), teb_add(y, teb_add(teb_mul(fx, s), teb_mul(fy, c))), mx, my);
  }
  /* CostmapModel::footprintCost (one warp): -3 off the map, -2 / -1 as pointCost, otherwise the largest cost */
  __device__ __forceinline__ int footprint_cost(int F, double x, double y, double th, int lane) const {
    int cx, cy;
    if (!to_map(x, y, cx, cy)) return -3;
    if (F < 3) { /* the centre cell only; 253 counts as a collision here */
      const int v = __ldg(map + (size_t)cy * sx + cx);
      return v == TEB_COSTMAP_NO_INFORMATION ? -2 : v >= TEB_COSTMAP_INSCRIBED ? -1 : v;
    }
    const double c = cos(th), s = sin(th);
    int x0, y0, xf, yf;
    bool on0 = vertex(0, x, y, c, s, x0, y0);
    const bool onf = on0;
    xf = x0; yf = y0;
    int hi = 0;
    for (int e = 0; e < F; ++e) { /* edges 0 -> 1, ..., F - 2 -> F - 1, then the closing edge F - 1 -> 0 */
      int x1 = xf, y1 = yf;
      const bool on1 = e + 1 < F ? vertex(e + 1, x, y, c, s, x1, y1) : onf;
      if (!on0 || !on1) return -3;
      /* LineIterator (x0, y0) -> (x1, y1): cells 0 .. den, cell k on the major axis k steps, on the minor axis
       * (den / 2 + k numadd) / den steps */
      const int dx = abs(x1 - x0), dy = abs(y1 - y0);
      const int ix = x1 >= x0 ? 1 : -1, iy = y1 >= y0 ? 1 : -1;
      const bool xmaj = dx >= dy;
      const int den = xmaj ? dx : dy, numadd = xmaj ? dy : dx;
      for (int base = 0; base <= den; base += 32) {
        const int k = base + lane;
        int v = 0;
        if (k <= den) {
          const int m = den ? (int)(((long long)(den >> 1) + (long long)k * numadd) / den) : 0;
          const int mx = x0 + ix * (xmaj ? k : m), my = y0 + iy * (xmaj ? m : k);
          const int raw = __ldg(map + (size_t)my * sx + mx);
          v = raw == TEB_COSTMAP_NO_INFORMATION ? -2 : raw == TEB_COSTMAP_LETHAL ? -1 : raw;
        }
        const unsigned neg = __ballot_sync(0xffffffffu, v < 0);
        if (neg) return __shfl_sync(0xffffffffu, v, __ffs(neg) - 1);
        hi = v > hi ? v : hi;
      }
      x0 = x1; y0 = y1; on0 = on1;
    }
    for (int o = 16; o; o >>= 1) {
      const int u = __shfl_xor_sync(0xffffffffu, hi, o);
      hi = u > hi ? u : hi;
    }
    return hi;
  }
  __device__ __forceinline__ int query(const FeasDev&, const FeasRasterDev& w, int j, double x, double y, double th, int lane) const {
    const int v = footprint_cost(w.F, x, y, th, lane);
    if (lane == 0) s_cost[j] = (double)v;
    return v == -1 ? 1 : 0;
  }
  /* query_cost of the block's tested queries, the rows `queries` gets */
  __device__ __forceinline__ void store(const FeasDev& fd, const FeasRasterDev& w, int b, long long q0, int last, int tid) const {
    if (!w.query_cost) return;
    double* o = w.query_cost + (size_t)b * fd.a.max_queries + q0;
    for (int j = tid; j <= last; j += FEAS_THREADS) o[j] = s_cost[j];
  }
};

/* the check of band blockIdx.x against world W; one CTA of FEAS_THREADS */
template <class W>
__device__ __forceinline__ void feasible_band(const FeasDev& fd, const typename W::Param& wp) {
  extern __shared__ __align__(16) unsigned char feas_smem[];
  __shared__ long long s_off[FEAS_MAX_POSES + 1]; /* s_off[i]: index of pose i's query; s_off[L + 1]: the total */
  __shared__ double s_q[FEAS_QB][3];
  __shared__ double s_carry[2][3];                /* accumulation state of a segment that continues in the next block */
  __shared__ int s_cls[FEAS_QB];
  __shared__ int s_L, s_bad;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x;
  const TebFeasibilityArgs& a = fd.a;
  const double* rec = fd.poses + (size_t)b * fd.n_cap * 4;
  const int n = fd.n[b];
  const int sc = fd.scene_id[b];
  /* inputs the host entry point rejects with TEBGPU_ERR_INVALID_ARG */
  const bool bad_band = n < 0 || n > fd.n_cap || sc < 0 || sc >= fd.S;
  W w;
  const bool bad = __syncthreads_or(w.begin(fd, wp, sc, bad_band, feas_smem, tid));
  if (warp == 0 && !bad) {
    /* the look-ahead index (:1253-1264): clamped, then cut at the first pose farther than the look-ahead distance */
    int L = a.look_ahead_idx;
    if (L < 0 || L >= n) L = n - 1;
    if (a.lookahead_distance > 0) {
      for (int base = 1; base < n; base += 32) {
        const int i = base + lane;
        const bool far = i < n && hypot(rec[4 * i] - rec[0], rec[4 * i + 1] - rec[1]) > a.lookahead_distance;
        const unsigned f = __ballot_sync(0xffffffffu, far);
        if (f) { L = base + __ffs(f) - 2; break; }
      }
    }
    /* a non-finite pose among the checked ones: undecidable */
    bool nf = false;
    for (int i = lane; i <= L; i += 32) nf |= !(isfinite(rec[4 * i]) && isfinite(rec[4 * i + 1]) && isfinite(rec[4 * i + 2]));
    nf = __any_sync(0xffffffffu, nf);
    /* query offsets: pose i, then the extra samples of segment i for i < L */
    long long carry = 0;
    for (int base = 0; base <= L && !nf; base += 32) {
      const int i = base + lane;
      long long c = 0;
      if (i <= L) c = 1 + (i < L ? feas_segment(rec + 4 * i, rec + 4 * (i + 1), a.inscribed_radius, a.angular_resolution).extra : 0);
      long long inc = c;
      for (int o = 1; o < 32; o <<= 1) {
        const long long v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
      }
      if (i <= L) s_off[i + 1] = carry + inc;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) { s_off[0] = 0; s_L = nf ? -2 : L; }
  }
  __syncthreads();
  int32_t* out_f = a.feasible + b;
  int32_t* out_c = a.query_count + b;
  if (bad || s_L == -2) {
    if (tid == 0) { *out_f = -1; *out_c = 0; }
    return;
  }
  const int L = s_L;
  const long long total = L < 0 ? 0 : s_off[L + 1];
  const long long limit = total < (long long)a.max_queries ? total : (long long)a.max_queries;
  double* qout = a.queries ? a.queries + (size_t)b * a.max_queries * 3 : nullptr;
  long long first = -1;
  int cls = 0;
  for (long long q0 = 0; q0 < limit; q0 += FEAS_QB) {
    const int cnt = (int)(limit - q0 < FEAS_QB ? limit - q0 : FEAS_QB);
    const int par = (int)((q0 / FEAS_QB) & 1);
    /* generation: the segments (pose i and its extra samples) that overlap [q0, q0 + cnt), one thread per segment */
    int lo = 0, hi = L; /* first pose whose queries reach past q0: largest i with s_off[i] <= q0 */
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_off[mid] <= q0) lo = mid; else hi = mid - 1;
    }
    for (int i = lo + tid; i <= L && s_off[i] < q0 + cnt; i += FEAS_THREADS) {
      const double* p = rec + 4 * i;
      const long long beg = s_off[i], end = s_off[i + 1];
      const long long ka = q0 > beg ? q0 - beg : 0, kb = (q0 + cnt < end ? q0 + cnt : end) - beg;
      if (ka == 0) { s_q[beg - q0][0] = p[0]; s_q[beg - q0][1] = p[1]; s_q[beg - q0][2] = p[2]; }
      if (kb > 1) {
        const FeasSeg sg = feas_segment(p, p + 4, a.inscribed_radius, a.angular_resolution);
        const double div = (double)sg.extra + 1.0;
        const double sx = sg.dx / div, sy = sg.dy / div, sr = sg.dr / div;
        double x = p[0], y = p[1], t = p[2];
        if (ka > 1) { x = s_carry[par ^ 1][0]; y = s_carry[par ^ 1][1]; t = s_carry[par ^ 1][2]; }
        for (long long k = ka > 1 ? ka : 1; k < kb; ++k) {
          x = teb_add(x, sx);
          y = teb_add(y, sy);
          t = teb_normalize_theta(teb_add(t, sr));
          const long long slot = beg + k - q0;
          s_q[slot][0] = x; s_q[slot][1] = y; s_q[slot][2] = t;
        }
        if (end > q0 + cnt) { s_carry[par][0] = x; s_carry[par][1] = y; s_carry[par][2] = t; }
      }
    }
    if (tid == 0) s_bad = FEAS_QB;
    __syncthreads();
    /* test: a warp per query, in order; a warp skips the queries behind a non-free one already found */
    for (int j = warp; j < cnt; j += FEAS_THREADS / 32) {
      if (j > *(volatile int*)&s_bad) break;
      const int v = w.query(fd, wp, j, s_q[j][0], s_q[j][1], s_q[j][2], lane);
      if (v && lane == 0) { s_cls[j] = v; atomicMin(&s_bad, j); }
    }
    __syncthreads();
    const int jb = s_bad;
    if (qout)
      for (int j = tid; j < cnt && j <= jb; j += FEAS_THREADS) {
        double* o = qout + 3 * (size_t)(q0 + j);
        o[0] = s_q[j][0]; o[1] = s_q[j][1]; o[2] = s_q[j][2];
      }
    w.store(fd, wp, b, q0, (jb < cnt ? jb : cnt - 1), tid);
    if (jb < FEAS_QB) { first = q0 + jb; cls = s_cls[jb]; break; }
    __syncthreads(); /* s_q and s_bad are rewritten by the next block */
  }
  if (tid == 0) {
    long long count;
    int f;
    if (first >= 0) { f = cls == 1 ? 0 : -1; count = first + 1; }
    else { f = total > (long long)a.max_queries ? -1 : 1; count = total; }
    *out_f = f;
    *out_c = (int32_t)(count < FEAS_INT_MAX ? count : FEAS_INT_MAX);
  }
}

template <bool GEOM, bool GT>
__global__ void __launch_bounds__(FEAS_THREADS) k_feasible(FeasDev fd, const KParams kp) {
  feasible_band<FeasTable<GEOM, GT>>(fd, kp);
}

/* two resident CTAs per SM asked for: ptxas then keeps the block loop's live values in registers (98, no spill) instead
 * of holding the kernel to 80 registers with 60 bytes of spill stores */
__global__ void __launch_bounds__(FEAS_THREADS, 2) k_feasible_costmap(FeasDev fd, const FeasRasterDev wp) {
  feasible_band<FeasRaster>(fd, wp);
}

}  // namespace tebgpu
