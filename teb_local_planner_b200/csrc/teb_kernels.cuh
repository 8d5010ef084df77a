/*
 * teb_kernels.cuh — sm_90a kernels of the batched Timed-Elastic-Band optimizer.
 *
 *   k_begin          per-call state reset, optimizeTEB guards                (optimal_planner.cpp:185)
 *   k_auto_resize    TimedElasticBand::autoResize per band                  (timed_elastic_band.cpp:227-286)
 *   k_build_graph    buildGraph: obstacle association, dynamic-obstacle times, via-point assignment
 *                                                                            (optimal_planner.cpp:323-366, 444-548, 646-718)
 *   k_linearize      "kernel A", first generation (variant 1 of tebgpu_set_linearize_variant, kept as an independent
 *                    second mapping): CTA of 128 threads per 32-pose tile, Jacobian blocks in shared memory, one thread
 *                    per band row gathers J^T J. The default kernel A is k_linearize2 in teb_linearize.cuh.
 *                                                                            (g2o buildSystem, SURVEY §3.3 step 2)
 *   k_vor            EdgeVelocityObstacleRatio rows added to the assembled band (only when that weight is > 0)
 *   k_lm_step_t      "kernel B", solvers 0 / 1: one Levenberg-Marquardt iteration per band in one CTA: banded LDL^T
 *                    (sequential warp solver or block cyclic reduction), update, trial chi2, rho / lambda
 *                    accept-reject loop (SURVEY App. A.4). The default solver 2 lives in teb_spec.cuh.
 *   k_finalize       computeCurrentCost with the selection scales, outputs   (optimal_planner.cpp:1041-1094)
 *   k_cost_only      computeCurrentCost outside optimizeTEB
 * Template flags: HOLO = holonomic rows (vy, acc y), GEOM = vertex-list shapes reachable (generic_distance compiled in).
 *
 * Unknown layout ("padded group layout"): scalar index 4*i + c, c = 0,1,2 -> (x,y,theta) of pose i, c = 3 -> dt_i.
 * It equals the g2o vertex-id order (dt_0, pose_1, dt_1, ...) shifted by 3; the fixed start/goal pose and the
 * non-existent dt_{n-1} are identity rows. H is SPD banded with half bandwidth 10 (an acceleration edge spans the 11
 * consecutive scalars 4i .. 4i+10). Storage per band: Hb[4*n_cap][12], row r = H[r][r-k] for k = 0..10, then b[r].
 */
#pragma once

#include "teb_device.cuh"
#include "teb_resize.h"

namespace tebgpu {

constexpr int TP = 32;                 /* poses per kernel-A tile */
constexpr int KA_P1OFF = ((TP + 2 + 31) / 32) * 32; /* first thread of the acceleration-row group */
constexpr int KA_THREADS = 4 * TP;     /* one thread per band row of the tile */
constexpr int JSTRIDE = 83;            /* doubles per anchor Jacobian block: 7 rows x 7 columns + 3 rows x 11 (+1 pad) */
constexpr int J_ACC = 49;              /* offset of the acceleration rows (x, theta, y) inside a block */
constexpr int ESTR = 10;               /* residual slots per anchor: vx|v, omega, kin0, kin1, sp, rot, vy, acc x, acc theta, acc y */
constexpr int START_E = 21;            /* start-edge block: 3 rows x 7 columns, then its 3 residuals */
constexpr int HROW = 12;               /* doubles per band row: 11 band entries + rhs */
constexpr int KB_THREADS = 128;
constexpr int MAX_MW = 16;             /* association bitmask words per pose of the staged path (<= 1024 obstacles per scene) */
constexpr int STAGED_MAX_OBST = 64 * MAX_MW; /* largest M_cap whose table the staged kernels copy into shared memory */
constexpr int GT_MAX_MW = 256;         /* association words per pose of the global-table path (<= 16384 obstacles per scene) */

struct BandState {
  double lambda, ni, current_chi, chi2_final;
  double parts_last[4];  /* chi2 by family at the last evaluated LM trial: obstacles, via, time-optimal, other */
  double parts_cur[4];   /* same at the current (accepted) state */
  int32_t active;        /* optimizeGraph still iterating (no Terminate yet) */
  int32_t failed;        /* optimizeTEB returned false */
  int32_t status;
  int32_t lm_iters;
};

/* Device view of one batch + workspaces. */
struct DevBatch {
  int32_t B, n_cap, S, M_cap, V_cap, MW;
  double* poses;
  int32_t* n;
  const int32_t* scene_id;
  const TebObstacle* obstacles;
  const int32_t* obst_count;
  const double* via;
  const int32_t* via_count;
  const double* vel_start;
  const double* vel_goal;
  const int32_t* prefer_rotdir;
  double* cost;
  double* chi2;
  int32_t* status;
  int32_t* lm_iters;
  /* workspaces */
  double* Hb;                 /* [B][4*n_cap][12] */
  unsigned long long* assoc;  /* [B][n_cap][MW]   */
  unsigned long long* assoc3; /* [B][n_cap][MW] legacy association: edges with multiplicity 3 (centre pose) */
  double* dyn_t;              /* [B][n_cap]       */
  int32_t* via_idx;           /* [B][V_cap]       */
  double* chi_parts;          /* [B][chunks][4]   */
  int32_t* dyn_idx;           /* [S][M_cap] indices of the dynamic obstacles of a scene (built once per call) */
  int32_t* dyn_cnt;           /* [S] */
  double* rhs;                /* [B][4*n_cap] compact copy of b (coalesced reads in the trial evaluation) */
  double* dmax_parts;         /* [B][chunks] max |H_rr| over the real rows of the tile (LM lambda init) */
  BandState* state;           /* [B]              */
  int32_t chunks;             /* tiles per band of the kernel-A mapping in use = ceil(n_cap / tile) */
  int32_t tile;               /* poses per kernel-A tile (chi2 / max-diagonal partials are per tile) */
  const double* obst_vertices; /* [S][PV_cap][2] vertex pool of the Line / Pill / Polygon obstacles (or NULL) */
  int32_t PV_cap;
  /* kernel A band selection (speculative solver, retry rounds overlapped with the next linearisation):
   * a_list != NULL: blockIdx.y indexes the list (a_cnt entries); else bands with defer[b] == skip_tag are skipped */
  const int32_t* a_list;
  const int32_t* a_cnt;
  int32_t* defer;             /* [B] tag of the inner iteration in which the band was queued for a retry round */
  int32_t skip_tag;
  /* global-table path (M_cap > STAGED_MAX_OBST): occupancy words of the association, bit w of word w >> 6 set iff
   * association word w of the pose is non-zero, so that per-iteration kernels read only the words that hold bits */
  unsigned long long* occ;    /* [B][n_cap][OW] */
  int32_t OW;                 /* ceil(MW / 64) */
  /* [B] or NULL: status bits k_plan_begin left for a band it could not plan (teb_plan.cuh); k_begin marks such a band
   * failed, so the optimize sequence leaves it as it is */
  const int32_t* pre_status;
};

/* Global-table path: the obstacles associated with pose row pr = b * n_cap + i, in increasing index order (the order
 * of the staged kernels' walk over all MW words): visit(w, m) for obstacle m of association word w. Only the words the
 * pose's occupancy words mark non-zero are read. */
template <class F>
__device__ __forceinline__ void walk_assoc_occ(const DevBatch& db, size_t pr, F&& visit) {
  const unsigned long long* am = db.assoc + pr * db.MW;
  const unsigned long long* oc = db.occ + pr * db.OW;
  for (int o = 0; o < db.OW; ++o) {
    unsigned long long ow = oc[o];
    while (ow) {
      const int w = (o << 6) + __ffsll((long long)ow) - 1;
      ow &= ow - 1;
      unsigned long long mask = am[w];
      while (mask) {
        const int m = (w << 6) + __ffsll((long long)mask) - 1;
        mask &= mask - 1;
        visit(w, m);
      }
    }
  }
}

/* A band belongs to the side stream's share when it was queued for retry rounds in the iteration with tag `skip_tag` -
 * or, meanwhile, AGAIN in the following one: the side stream's own round 0 of the current iteration may re-queue it
 * (defer = skip_tag + 1) while main-stream kernels of the same iteration are still deciding what to skip. */
__device__ __forceinline__ bool deferred_since(int32_t defer_tag, int32_t skip_tag) {
  return (uint32_t)(defer_tag - skip_tag) <= 1u;
}
/* band handled by this CTA of kernel A, or -1 */
__device__ __forceinline__ int linearize_band(const DevBatch& db, int y) {
  if (db.a_list) return (y < *db.a_cnt) ? db.a_list[y] : -1;
  if (db.skip_tag != 0 && deferred_since(db.defer[y], db.skip_tag)) return -1;
  return y;
}

/* ------------------------------------------------------------------ small block utilities */
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
  return v;
}
/* deterministic block sum of NV values per thread; result valid in thread 0 (and written to out[]) */
template <int NV, int NWARPS>
__device__ __forceinline__ void block_sum(double (&v)[NV], double* scratch /* NV*NWARPS */, double* out /* NV, smem */) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double s = warp_sum(v[k]);
    if (lane == 0) scratch[k * NWARPS + wid] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      double s = 0;
      for (int w = 0; w < NWARPS; ++w) s += scratch[k * NWARPS + w];
      out[k] = s;
    }
  }
  __syncthreads();
}

__device__ __forceinline__ bool row_is_real(int r, int n) {
  const int i = r >> 2, c = r & 3;
  return c == 3 ? (i <= n - 2) : (i >= 1 && i <= n - 2);
}

/* ------------------------------------------------------------------ k_begin */
__global__ void k_begin(DevBatch db, KParams kp) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < db.S) { /* compact list of the scene's dynamic obstacles (AddEdgesDynamicObstacles iterates only those) */
    const TebObstacle* go = db.obstacles + (size_t)b * db.M_cap;
    int cnt = 0;
    const int M = min(max(db.obst_count[b], 0), db.M_cap);
    for (int m = 0; m < M; ++m)
      if (go[m].dynamic) db.dyn_idx[(size_t)b * db.M_cap + cnt++] = m;
    db.dyn_cnt[b] = cnt;
  }
  if (b >= db.B) return;
  BandState st;
  st.lambda = 0; st.ni = 2; st.current_chi = 0; st.chi2_final = 0;
  for (int k = 0; k < 4; ++k) { st.parts_last[k] = 0; st.parts_cur[k] = 0; }
  st.active = 0; st.failed = 0; st.status = 0; st.lm_iters = 0;
  if (!kp.p.optimization_activate) { st.failed = 1; st.status |= TEB_STATUS_DISABLED; }
  { /* inputs the batch cannot describe (the device entry point cannot check them on the host): band length, scene
     * index, obstacle / via-point counts, obstacle rows. Such a band is left untouched and reported. */
    int sc = db.scene_id[b];
    bool bad = false;
    if (sc < 0 || sc >= db.S) { bad = true; sc = 0; }
    if (db.n[b] < 1 || db.n[b] > db.n_cap) bad = true;
    if (db.V_cap > 0 && db.via_count && (db.via_count[b] < 0 || db.via_count[b] > db.V_cap)) bad = true;
    int M = db.obst_count[sc];
    if (M < 0 || M > db.M_cap) { bad = true; M = 0; }
    const TebObstacle* go = db.obstacles + (size_t)sc * db.M_cap;
    for (int m = 0; m < M; ++m) {
      const int type = go[m].type, vb = go[m].vertex_begin, vc = go[m].vertex_count;
      if (type < TEB_OBST_POINT || type > TEB_OBST_POLYGON) bad = true;
      else if (type >= TEB_OBST_LINE &&
               (vc < 1 || (type != TEB_OBST_POLYGON && vc != 2) || vb < 0 || (long long)vb + vc > db.PV_cap))
        bad = true;
    }
    if (bad) { st.failed = 1; st.status |= TEB_STATUS_BAD_INPUT; }
  }
  if (db.pre_status && db.pre_status[b]) { st.failed = 1; st.status |= db.pre_status[b]; }
  db.state[b] = st;
}

/* ------------------------------------------------------------------ k_auto_resize (thread per band) */
__global__ void k_auto_resize(DevBatch db, KParams kp) {
  const int y = blockIdx.x * blockDim.x + threadIdx.x;
  if (y >= db.B) return;
  const int b = linearize_band(db, y); /* all bands, or the deferred list / everything but the deferred bands */
  if (b < 0) return;
  if (db.state[b].failed) return;
  const int fast_mode = !kp.p.include_dynamic_obstacles; /* optimal_planner.cpp:197 */
  int n = db.n[b];
  int nn = teb_auto_resize_records(db.poses + (size_t)b * db.n_cap * 4, n, db.n_cap, kp.p.dt_ref, kp.p.dt_hysteresis,
                                   kp.p.min_samples, kp.p.max_samples, fast_mode);
  if (nn < 0) { db.state[b].failed = 1; db.state[b].status |= TEB_STATUS_CAPACITY; return; }
  db.n[b] = nn;
}

/* ------------------------------------------------------------------ k_build_graph (CTA per band)
 * GT = global-table path (M_cap > STAGED_MAX_OBST): obstacle rows are read from global memory (L2) instead of a
 * shared-memory copy of the scene's table, the non-legacy association runs one warp per pose with the obstacles across
 * the lanes, and the occupancy words of every pose are written at the end. */
template <bool GEOM, bool GT = false>
__global__ void __launch_bounds__(256) k_build_graph(DevBatch db, KParams kp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TebObstacle* so_s = reinterpret_cast<TebObstacle*>(smem_raw);
  const int b = linearize_band(db, blockIdx.x);
  if (b < 0) return;
  BandState* st = &db.state[b];
  const int n = db.n[b];
  if (threadIdx.x == 0) {
    /* optimizeGraph guards (optimal_planner.cpp:370-382) */
    int failed = st->failed;
    if (!failed && kp.p.max_vel_x < 0.01) { failed = 1; st->status |= TEB_STATUS_DISABLED; }
    if (!failed && (n < kp.p.min_samples || n < 3)) { failed = 1; st->status |= TEB_STATUS_TOO_FEW_POSES; }
    st->failed = failed;
    st->active = !failed;
    st->lambda = 0;
    st->ni = 2;
  }
  __syncthreads();
  if (st->failed) return;
  const int s = db.scene_id[b];
  const int M = db.obst_count[s];
  const TebObstacle* go = db.obstacles + (size_t)s * db.M_cap;
  if constexpr (!GT)
    for (int m = threadIdx.x; m < M; m += blockDim.x) so_s[m] = go[m];
  __syncthreads();
  const TebObstacle* so = GT ? go : so_s;
  const double* P = db.poses + (size_t)b * db.n_cap * 4;
  const double* pool = db.obst_vertices + (size_t)s * db.PV_cap * 2; /* only dereferenced for vertex-list obstacles */
  unsigned long long* assoc = db.assoc + (size_t)b * db.n_cap * db.MW;

  unsigned long long* assoc3 = db.assoc3 + (size_t)b * db.n_cap * db.MW;
  if (GT && !kp.p.legacy_obstacle_association) {
    /* the same association, one warp per pose: the force-inclusion bits of each 64-obstacle word are two ballots; the
     * closest left / right obstacle within the cutoff is a warp argmin over (dist, m) taken lexicographically, i.e. the
     * lowest index among equal distances - what the sequential strict-< scan keeps. A NaN distance fails every
     * comparison and never becomes a candidate, as in the scan. */
    const int first_vertex = kp.has_vor ? 0 : 1;
    const int lane = threadIdx.x & 31;
    const double force_d = kp.p.min_obstacle_dist * kp.p.obstacle_association_force_inclusion_factor;
    const double cut_d = kp.p.min_obstacle_dist * kp.p.obstacle_association_cutoff_factor;
    for (int i = threadIdx.x >> 5; i < n; i += blockDim.x >> 5) {
      unsigned long long* am = assoc + (size_t)i * db.MW;
      if (!(kp.has_obst && i >= first_vertex && i <= n - 2)) {
        for (int w = lane; w < db.MW; w += 32) am[w] = 0ull;
        continue;
      }
      const double px = P[4 * i], py = P[4 * i + 1], th = P[4 * i + 2];
      double sn, cs;
      sincos(th, &sn, &cs);
      double left_min = 1.7976931348623157e308, right_min = 1.7976931348623157e308;
      int left = INT_MAX, right = INT_MAX; /* INT_MAX: none (sorts after every index) */
      for (int w = 0; w < db.MW; ++w) {
        unsigned half[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = (w << 6) + (h << 5) + lane;
          bool force = false;
          if (m < M) {
            const TebObstacle ob = go[m];
            if (!(kp.p.include_dynamic_obstacles && ob.dynamic)) {
              const double dist = robot_obstacle_distance_only<GEOM>(kp, pool, px, py, cs, sn, ob, ob.x, ob.y, 0.0, 0.0);
              if (dist < force_d) {
                force = true;
              } else if (!(dist > cut_d)) {
                const double cx = ob.x - px, cy = ob.y - py;
                if (cs * cy - cx * sn > 0) {
                  if (dist < left_min) { left_min = dist; left = m; }
                } else {
                  if (dist < right_min) { right_min = dist; right = m; }
                }
              }
            }
          }
          half[h] = __ballot_sync(0xffffffffu, force);
        }
        if (lane == 0) am[w] = ((unsigned long long)half[1] << 32) | half[0];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ld = __shfl_xor_sync(0xffffffffu, left_min, o), rd = __shfl_xor_sync(0xffffffffu, right_min, o);
        const int lm = __shfl_xor_sync(0xffffffffu, left, o), rm = __shfl_xor_sync(0xffffffffu, right, o);
        if (ld < left_min || (ld == left_min && lm < left)) { left_min = ld; left = lm; }
        if (rd < right_min || (rd == right_min && rm < right)) { right_min = rd; right = rm; }
      }
      if (lane == 0) {
        if (left != INT_MAX) am[left >> 6] |= 1ull << (left & 63);
        if (right != INT_MAX) am[right >> 6] |= 1ull << (right & 63);
      }
    }
  } else if (!kp.p.legacy_obstacle_association) {
    /* AddEdgesObstacles association (optimal_planner.cpp:484-547); pose 0 takes part only to feed
     * EdgeVelocityObstacleRatio (first_vertex, :482) */
    const int first_vertex = kp.has_vor ? 0 : 1;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      unsigned long long mask[MAX_MW] = {0};
      if (kp.has_obst && i >= first_vertex && i <= n - 2) {
        const double px = P[4 * i], py = P[4 * i + 1], th = P[4 * i + 2];
        double sn, cs;
        sincos(th, &sn, &cs);
        double left_min = 1.7976931348623157e308, right_min = 1.7976931348623157e308;
        int left = -1, right = -1;
        const double force_d = kp.p.min_obstacle_dist * kp.p.obstacle_association_force_inclusion_factor;
        const double cut_d = kp.p.min_obstacle_dist * kp.p.obstacle_association_cutoff_factor;
        for (int m = 0; m < M; ++m) {
          const TebObstacle ob = so[m];
          if (kp.p.include_dynamic_obstacles && ob.dynamic) continue;
          const double dist = robot_obstacle_distance_only<GEOM>(kp, pool, px, py, cs, sn, ob, ob.x, ob.y, 0.0, 0.0);
          if (dist < force_d) { mask[m >> 6] |= 1ull << (m & 63); continue; }
          if (dist > cut_d) continue;
          const double cx = ob.x - px, cy = ob.y - py;
          if (cs * cy - cx * sn > 0) {
            if (dist < left_min) { left_min = dist; left = m; }
          } else {
            if (dist < right_min) { right_min = dist; right = m; }
          }
        }
        if (left >= 0) mask[left >> 6] |= 1ull << (left & 63);
        if (right >= 0) mask[right >> 6] |= 1ull << (right & 63);
      }
      for (int w = 0; w < db.MW; ++w) assoc[(size_t)i * db.MW + w] = mask[w];
    }
  } else {
    /* AddEdgesObstaclesLegacy (optimal_planner.cpp:551-643): per obstacle the closest pose and its
     * obstacle_poses_affected/2 neighbours on both sides; the centre pose carries three identical edges */
    for (int k = threadIdx.x; k < n * db.MW; k += blockDim.x) { assoc[k] = 0ull; assoc3[k] = 0ull; }
    __syncthreads();
    if (kp.has_obst) {
      for (int m = threadIdx.x; m < M; m += blockDim.x) {
        const TebObstacle ob = so[m];
        if (kp.p.include_dynamic_obstacles && ob.dynamic) continue;
        int index = -1;
        if (kp.p.obstacle_poses_affected >= n) {
          index = n / 2;
        } else if (GEOM && (ob.type == TEB_OBST_LINE || (ob.type == TEB_OBST_POLYGON && ob.vertex_count >= 2))) {
          /* findClosestTrajectoryPose(line) / (polygon) timed_elastic_band.cpp:480-530: distance of the pose
           * POSITION to the vertex list (no footprint, no radius) */
          double best = 1.7976931348623157e308;
          for (int i = 0; i < n; ++i) {
            const double d = generic_distance(TEB_FOOTPRINT_POINT, kp.fp_geom, pool, P[4 * i], P[4 * i + 1], 1.0, 0.0, ob.x, ob.y,
                                              0.0, TEB_OBST_POLYGON, ob.vertex_begin, ob.vertex_count, 0.0, 0.0).d;
            if (d < best) { best = d; index = i; }
          }
        } else { /* findClosestTrajectoryPose(point) :455-478; Circular and Pill obstacles: centroid (:545) */
          double cx = ob.x, cy = ob.y;
          if (GEOM && ob.type == TEB_OBST_POLYGON && ob.vertex_count == 1) { cx = pool[2 * ob.vertex_begin]; cy = pool[2 * ob.vertex_begin + 1]; }
          double best = 1.7976931348623157e308;
          for (int i = 0; i < n; ++i) {
            const double dx = cx - P[4 * i], dy = cy - P[4 * i + 1];
            const double d2 = dx * dx + dy * dy;
            if (d2 < best) { best = d2; index = i; }
          }
        }
        if (index <= 1 || index > n - 2) continue;
        const unsigned long long bit = 1ull << (m & 63);
        const int w = m >> 6;
        atomicOr(&assoc[(size_t)index * db.MW + w], bit);
        const int half = kp.p.obstacle_poses_affected / 2;
        if (half >= 1) atomicOr(&assoc3[(size_t)index * db.MW + w], bit); /* explicit edge + neighbourIdx 0 twice */
        for (int nb = 1; nb < half; ++nb) {
          if (index + nb < n) atomicOr(&assoc[(size_t)(index + nb) * db.MW + w], bit);
          if (index - nb >= 0) atomicOr(&assoc[(size_t)(index - nb) * db.MW + w], bit);
        }
      }
    }
  }
  /* EdgeDynamicObstacle times: t_1 = dt_0, t_{i+1} = t_i + dt_i, frozen at build (optimal_planner.cpp:662-670);
   * sequential like the reference so the sums are bitwise identical. */
  if (kp.has_dyn && threadIdx.x == 32) {
    double* T = db.dyn_t + (size_t)b * db.n_cap;
    double time = P[3];
    for (int i = 1; i < n - 1; ++i) { T[i] = time; time += P[4 * i + 3]; }
  }
  /* AddEdgesViaPoints (optimal_planner.cpp:675-718), findClosestTrajectoryPose (timed_elastic_band.cpp:455-478) */
  if (kp.has_via && db.V_cap > 0) {
    const int V = db.via_count[b];
    const double* via = db.via + (size_t)b * db.V_cap * 2;
    int32_t* vidx = db.via_idx + (size_t)b * db.V_cap;
    if (!kp.p.via_points_ordered) {
      for (int v = threadIdx.x; v < db.V_cap; v += blockDim.x) {
        int index = -1;
        if (v < V && n >= 3) {
          double best = 1.7976931348623157e308;
          for (int i = 0; i < n; ++i) {
            const double dx = via[2 * v] - P[4 * i], dy = via[2 * v + 1] - P[4 * i + 1];
            const double d2 = dx * dx + dy * dy;
            if (d2 < best) { best = d2; index = i; }
          }
          if (index > n - 2) index = n - 2;
          if (index < 1) index = -1; /* skipped: too close to / behind the robot */
        }
        vidx[v] = index;
      }
    } else if (threadIdx.x == 64) {
      int start_pose_idx = 0;
      for (int v = 0; v < db.V_cap; ++v) {
        int index = -1;
        if (v < V && n >= 3) {
          if (start_pose_idx >= 0 && start_pose_idx < n) {
            double best = 1.7976931348623157e308;
            for (int i = start_pose_idx; i < n; ++i) {
              const double dx = via[2 * v] - P[4 * i], dy = via[2 * v + 1] - P[4 * i + 1];
              const double d2 = dx * dx + dy * dy;
              if (d2 < best) { best = d2; index = i; }
            }
          }
          start_pose_idx = index + 2;
          if (index > n - 2) index = n - 2;
          if (index < 1) index = 1;
        }
        vidx[v] = index;
      }
    }
  }
  if constexpr (GT) { /* occupancy words: bit w of the pose's word w >> 6 iff association word w is non-zero */
    __syncthreads();
    unsigned long long* occ = db.occ + (size_t)b * db.n_cap * db.OW;
    for (int k = threadIdx.x; k < n * db.OW; k += blockDim.x) {
      const int i = k / db.OW, o = k - i * db.OW;
      const unsigned long long* am = assoc + (size_t)i * db.MW + 64 * o;
      const int nw = min(db.MW - 64 * o, 64);
      unsigned long long bits = 0ull;
      for (int w = 0; w < nw; ++w)
        if (am[w]) bits |= 1ull << w;
      occ[k] = bits;
    }
  }
}

/* ------------------------------------------------------------------ unary terms of one pose (obstacles, dynamic
 * obstacles, via-points): accumulates U = sum kappa g g^T (xx,xy,yy,xt,yt,tt), ub = -sum beta g, chi2 by family */
template <bool GEOM, bool GT = false> /* GT: so is the scene's table in global memory, walk via the occupancy words */
__device__ __forceinline__ void unary_terms(const KParams& kp, const DevBatch& db, int b, int sc, int i, int n, double px,
                                            double py, double cs, double sn, const TebObstacle* so, int M,
                                            bool want_grad, double U[6], double ub[3], double& chi_obst,
                                            double& chi_via) {
  if (i < 1 || i > n - 2) return;
  const double* pool = db.obst_vertices + (size_t)sc * db.PV_cap * 2; /* only dereferenced for vertex-list obstacles */
  if (GT && kp.has_obst) {
    walk_assoc_occ(db, (size_t)b * db.n_cap + i, [&](int w, int m) {
      const TebObstacle ob = so[m];
      double g[3], kappa, beta;
      const double d = robot_obstacle_distance<GEOM>(kp, pool, px, py, cs, sn, ob, ob.x, ob.y, 0.0, 0.0, g);
      double cterm = obstacle_terms(kp, d, kappa, beta);
      if (kp.p.legacy_obstacle_association &&
          ((db.assoc3[((size_t)b * db.n_cap + i) * db.MW + w] >> (m & 63)) & 1ull)) {
        cterm *= 3; kappa *= 3; beta *= 3;
      }
      chi_obst += cterm;
      if (want_grad && (kappa != 0 || beta != 0)) {
        U[0] += kappa * g[0] * g[0]; U[1] += kappa * g[0] * g[1]; U[2] += kappa * g[1] * g[1];
        U[3] += kappa * g[0] * g[2]; U[4] += kappa * g[1] * g[2]; U[5] += kappa * g[2] * g[2];
        ub[0] -= beta * g[0]; ub[1] -= beta * g[1]; ub[2] -= beta * g[2];
      }
    });
  } else if (kp.has_obst) {
    const unsigned long long* assoc = db.assoc + ((size_t)b * db.n_cap + i) * db.MW;
    for (int w = 0; w < db.MW; ++w) {
      unsigned long long mask = assoc[w];
      while (mask) {
        const int m = (w << 6) + __ffsll((long long)mask) - 1;
        mask &= mask - 1;
        const TebObstacle ob = so[m];
        double g[3], kappa, beta;
        const double d = robot_obstacle_distance<GEOM>(kp, pool, px, py, cs, sn, ob, ob.x, ob.y, 0.0, 0.0, g);
        double cterm = obstacle_terms(kp, d, kappa, beta);
        if (kp.p.legacy_obstacle_association &&
            ((db.assoc3[((size_t)b * db.n_cap + i) * db.MW + w] >> (m & 63)) & 1ull)) {
          cterm *= 3; kappa *= 3; beta *= 3; /* three identical edges on the centre pose */
        }
        chi_obst += cterm;
        if (want_grad && (kappa != 0 || beta != 0)) {
          U[0] += kappa * g[0] * g[0]; U[1] += kappa * g[0] * g[1]; U[2] += kappa * g[1] * g[1];
          U[3] += kappa * g[0] * g[2]; U[4] += kappa * g[1] * g[2]; U[5] += kappa * g[2] * g[2];
          ub[0] -= beta * g[0]; ub[1] -= beta * g[1]; ub[2] -= beta * g[2];
        }
      }
    }
  }
  if (kp.has_dyn) {
    const double t = db.dyn_t[(size_t)b * db.n_cap + i];
    const int nd = db.dyn_cnt[sc];
    const int32_t* di = db.dyn_idx + (size_t)sc * db.M_cap;
    for (int q = 0; q < nd; ++q) {
      const TebObstacle ob = so[di[q]];
      double g[3], kappa, beta;
      const double d = robot_obstacle_distance<GEOM>(kp, pool, px, py, cs, sn, ob, ob.x + t * ob.vx, ob.y + t * ob.vy, t * ob.vx,
                                               t * ob.vy, g);
      chi_obst += dynamic_terms(kp, d, kappa, beta);
      if (want_grad && (kappa != 0 || beta != 0)) {
        U[0] += kappa * g[0] * g[0]; U[1] += kappa * g[0] * g[1]; U[2] += kappa * g[1] * g[1];
        U[3] += kappa * g[0] * g[2]; U[4] += kappa * g[1] * g[2]; U[5] += kappa * g[2] * g[2];
        ub[0] -= beta * g[0]; ub[1] -= beta * g[1]; ub[2] -= beta * g[2];
      }
    }
  }
  if (kp.has_via && db.V_cap > 0) {
    const int32_t* vidx = db.via_idx + (size_t)b * db.V_cap;
    const double* via = db.via + (size_t)b * db.V_cap * 2;
    const double wv = kp.p.weight_viapoint;
    for (int v = 0; v < db.V_cap; ++v) {
      if (vidx[v] != i) continue;
      const double dx = px - via[2 * v], dy = py - via[2 * v + 1];
      const double e = sqrt(dx * dx + dy * dy); /* EdgeViaPoint edge_via_point.h:86 */
      chi_via += wv * e * e;
      if (want_grad && e > 0) {
        const double gx = dx / e, gy = dy / e;
        U[0] += wv * gx * gx; U[1] += wv * gx * gy; U[2] += wv * gy * gy;
        ub[0] -= wv * e * gx; ub[1] -= wv * e * gy;
      }
    }
  }
}

/* Jacobian rows of the chain edges anchored at a = p0-2+at (sqrt(weight)-scaled, columns 4a .. 4a+10).
 * part 0: EdgeVelocity, EdgeKinematics*, EdgeShortestPath, EdgePreferRotDir rows; part 1: EdgeAcceleration / Start / Goal
 * rows. Returns this part's chi2 contribution if the anchor belongs to the tile (a >= p0), else 0. */
template <bool HOLO>
__device__ __forceinline__ double anchor_rows(const KParams& kp, const DevBatch& db, int b, int part, int at, int p0, int n,
                                              const double* sP, const double* sSC, const double* sSeg, double* sJ,
                                              double* sE, double* sStart) {
  double chi3 = 0;
    const int a = p0 - 2 + at;
    if (a >= 0 && a <= n - 2) {
      double* J = sJ + (size_t)at * JSTRIDE; /* rows 0..6: 7 columns (v|vx, omega, kin0, kin1, sp, rot, vy); rows at J_ACC: 11 columns (acc x, theta, y) */
      double* eh = sE + ESTR * at;
      const double* pa = sP + 4 * at;
      const double* pb = pa + 4;
      const double ca = sSC[2 * at], sa = sSC[2 * at + 1], cb = sSC[2 * at + 2], sb = sSC[2 * at + 3];
      const double* q1 = sSeg + 9 * at;
      const double v1 = q1[0], w1 = q1[1], idt1 = q1[2];
      const double dx = pb[0] - pa[0], dy = pb[1] - pa[1];
      const bool fa = (a == 0), fb = (a + 1 == n - 1);
      double csum = 0;
      if (HOLO && part == 0 && kp.has_vel && kp.holo_vel) { /* EdgeVelocityHolonomic edge_velocity.h:236-273 */
        const HoloDer h = holo_derivs(pa[0], pa[1], pa[2], ca, sa, pb[0], pb[1], pb[2], pa[3]);
        double e[3], sl[3], c0, c1;
        holo_velocity_terms(kp, h.vx, h.vy, h.w, e, sl, c0, c1);
        const double kx = kp.sw_vel_x, ky = kp.sw_vel_y, kw = kp.sw_vel_th * sl[2];
        double* Rx = J;       /* row 0: vx */
        double* Ry = J + 42;  /* row 6: vy */
        /* columns: x_a, y_a, th_a, dt_a, x_b, y_b, th_b */
        Rx[0] = kx * (sl[0] * h.dvx[0] - c0 * h.dvy[0]); Rx[1] = kx * (sl[0] * h.dvx[1] - c0 * h.dvy[1]);
        Rx[2] = kx * (sl[0] * h.dvx[2] - c0 * h.dvy[2]); Rx[3] = kx * (-sl[0] * h.vx + c0 * h.vy) * h.idt;
        Rx[4] = kx * (sl[0] * h.dvx[3] - c0 * h.dvy[3]); Rx[5] = kx * (sl[0] * h.dvx[4] - c0 * h.dvy[4]); Rx[6] = 0;
        Ry[0] = ky * (sl[1] * h.dvy[0] - c1 * h.dvx[0]); Ry[1] = ky * (sl[1] * h.dvy[1] - c1 * h.dvx[1]);
        Ry[2] = ky * (sl[1] * h.dvy[2] - c1 * h.dvx[2]); Ry[3] = ky * (-sl[1] * h.vy + c1 * h.vx) * h.idt;
        Ry[4] = ky * (sl[1] * h.dvy[3] - c1 * h.dvx[3]); Ry[5] = ky * (sl[1] * h.dvy[4] - c1 * h.dvx[4]); Ry[6] = 0;
        J[7 + 0] = J[7 + 1] = J[7 + 4] = J[7 + 5] = 0;
        J[7 + 2] = -kw * h.idt; J[7 + 3] = -kw * h.w * h.idt; J[7 + 6] = kw * h.idt;
        eh[0] = kx * e[0]; eh[6] = ky * e[1]; eh[1] = kp.sw_vel_th * e[2];
      } else if (part == 0 && kp.has_vel) { /* EdgeVelocity edge_velocity.h:113-114 */
        double s0, s1;
        const double e0 = pen_interval2(v1, -kp.p.max_vel_x_backwards, kp.p.max_vel_x, kp.p.penalty_epsilon, s0);
        const double e1 = pen_interval(w1, kp.p.max_vel_theta, kp.p.penalty_epsilon, s1);
        const double k0 = kp.sw_vel_x * s0, k1 = kp.sw_vel_th * s1;
        J[0] = k0 * q1[3]; J[1] = k0 * q1[4]; J[2] = k0 * q1[5]; J[3] = -k0 * v1 * idt1;
        J[4] = k0 * q1[6]; J[5] = k0 * q1[7]; J[6] = k0 * q1[8];
        J[7 + 2] = -k1 * idt1; J[7 + 3] = -k1 * w1 * idt1; J[7 + 6] = k1 * idt1;
        eh[0] = kp.sw_vel_x * e0; eh[1] = kp.sw_vel_th * e1;
      }
      if (part == 0 && kp.has_kin) { /* EdgeKinematicsDiffDrive / Carlike edge_kinematics.h:94-101, :118-148, :203-215 */
        const double A = (ca + cb) * dy - (sa + sb) * dx;
        const double sA = sgn(A) * kp.sw_kin_nh;
        double* R = J + 14;
        R[0] = (sa + sb) * sA; R[1] = -(ca + cb) * sA; R[2] = (-sa * dy - ca * dx) * sA;
        R[4] = -(sa + sb) * sA; R[5] = (ca + cb) * sA; R[6] = (-sb * dy - cb * dx) * sA;
        eh[2] = kp.sw_kin_nh * fabs(A);
        double* R2 = J + 21;
        if (!kp.carlike) {
          double dd;
          const double e1 = pen_below(dx * ca + dy * sa, 0, 0, dd);
          dd *= kp.sw_kin_2;
          R2[0] = -ca * dd; R2[1] = -sa * dd; R2[2] = (-sa * dx + ca * dy) * dd;
          R2[4] = ca * dd; R2[5] = sa * dd;
          eh[3] = kp.sw_kin_2 * e1;
        } else {
          const double ad = normalize_theta(pb[2] - pa[2]);
          if (ad != 0) {
            const double nrm = sqrt(dx * dx + dy * dy);
            const double inr = nrm > 0 ? 1.0 / nrm : 0.0;
            const double ux = dx * inr, uy = dy * inr;
            double r, dr_dn, dr_dad;
            if (kp.p.exact_arc_length) {
              const double h = ad / 2, sh = sin(h);
              const double qq = nrm / (2 * sh);
              r = fabs(qq);
              dr_dn = sgn(qq) / (2 * sh);
              dr_dad = sgn(qq) * (-nrm * cos(h) / (4 * sh * sh));
            } else {
              r = nrm / fabs(ad);
              dr_dn = 1 / fabs(ad);
              dr_dad = -nrm * sgn(ad) / (ad * ad);
            }
            double s1;
            const double e1 = pen_below(r, kp.p.min_turning_radius, 0.0, s1);
            s1 *= kp.sw_kin_2;
            R2[0] = -s1 * dr_dn * ux; R2[1] = -s1 * dr_dn * uy; R2[2] = -s1 * dr_dad;
            R2[4] = s1 * dr_dn * ux; R2[5] = s1 * dr_dn * uy; R2[6] = s1 * dr_dad;
            eh[3] = kp.sw_kin_2 * e1;
          }
        }
      }
      if (part == 0 && kp.has_sp) { /* EdgeShortestPath edge_shortest_path.h:78 */
        const double nrm = sqrt(dx * dx + dy * dy);
        const double inr = nrm > 0 ? 1.0 / nrm : 0.0;
        double* R = J + 28;
        R[0] = -kp.sw_sp * dx * inr; R[1] = -kp.sw_sp * dy * inr;
        R[4] = kp.sw_sp * dx * inr; R[5] = kp.sw_sp * dy * inr;
        eh[4] = kp.sw_sp * nrm;
      }
      if (part == 0 && kp.has_rot && a < 3) { /* EdgePreferRotDir edge_prefer_rotdir.h:85, first three pairs optimal_planner.cpp:983 */
        const int rd = db.prefer_rotdir ? db.prefer_rotdir[b] : 0;
        if (rd == TEB_ROTDIR_LEFT || rd == TEB_ROTDIR_RIGHT) {
          const double meas = (rd == TEB_ROTDIR_LEFT) ? 1.0 : -1.0;
          double s0;
          const double e0 = pen_below(meas * normalize_theta(pb[2] - pa[2]), 0, 0, s0);
          double* R = J + 35;
          R[2] = -kp.sw_rot * s0 * meas;
          R[6] = kp.sw_rot * s0 * meas;
          eh[5] = kp.sw_rot * e0;
        }
      }
      if (HOLO && part == 1 && kp.has_acc && kp.holo_acc) {
        /* EdgeAccelerationHolonomic / Start / Goal edge_acceleration.h:487-540, :580-620, :672-712 */
        const HoloDer h1 = holo_derivs(pa[0], pa[1], pa[2], ca, sa, pb[0], pb[1], pb[2], pa[3]);
        const double sw[3] = {kp.sw_acc_x, kp.sw_acc_th, kp.sw_acc_y};
        const double lim[3] = {kp.p.acc_lim_x, kp.p.acc_lim_theta, kp.p.acc_lim_y};
        /* value / derivative tables in row order x, theta, y */
        const double v1r[3] = {h1.vx, h1.w, h1.vy};
        double d1[3][6];
#pragma unroll
        for (int k = 0; k < 6; ++k) { d1[0][k] = h1.dvx[k]; d1[2][k] = h1.dvy[k]; d1[1][k] = 0; }
        d1[1][2] = -h1.idt; d1[1][5] = h1.idt;
        if (a <= n - 3) {
          const double* pc = pb + 4;
          const HoloDer h2 = holo_derivs(pb[0], pb[1], pb[2], cb, sb, pc[0], pc[1], pc[2], pb[3]);
          const double v2r[3] = {h2.vx, h2.w, h2.vy};
          double d2[3][6];
#pragma unroll
          for (int k = 0; k < 6; ++k) { d2[0][k] = h2.dvx[k]; d2[2][k] = h2.dvy[k]; d2[1][k] = 0; }
          d2[1][2] = -h2.idt; d2[1][5] = h2.idt;
          const double iT = 1.0 / (pa[3] + pb[3]);
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            const double acc = (v2r[r] - v1r[r]) * 2 * iT;
            double sl;
            const double e = pen_interval(acc, lim[r], kp.p.penalty_epsilon, sl);
            const double kk = sw[r] * sl * iT;
            double* R = J + J_ACC + 11 * r;
            R[0] = -2 * kk * d1[r][0]; R[1] = -2 * kk * d1[r][1]; R[2] = -2 * kk * d1[r][2];
            R[3] = kk * (2 * v1r[r] * h1.idt - acc);
            R[4] = 2 * kk * (d2[r][0] - d1[r][3]); R[5] = 2 * kk * (d2[r][1] - d1[r][4]); R[6] = 2 * kk * (d2[r][2] - d1[r][5]);
            R[7] = kk * (-2 * v2r[r] * h2.idt - acc);
            R[8] = 2 * kk * d2[r][3]; R[9] = 2 * kk * d2[r][4]; R[10] = 2 * kk * d2[r][5];
            if (a + 2 == n - 1) { R[8] = R[9] = R[10] = 0; }
            eh[7 + r] = sw[r] * e;
          }
        } else { /* a == n-2: goal edge */
          const double* vg = db.vel_goal + 4 * (size_t)b;
          if (vg[3] != 0) {
            const double tw[3] = {vg[0], vg[2], vg[1]};
#pragma unroll
            for (int r = 0; r < 3; ++r) {
              const double acc = (tw[r] - v1r[r]) * h1.idt;
              double sl;
              const double e = pen_interval(acc, lim[r], kp.p.penalty_epsilon, sl);
              const double kk = sw[r] * sl * h1.idt;
              double* R = J + J_ACC + 11 * r;
              R[0] = -kk * d1[r][0]; R[1] = -kk * d1[r][1]; R[2] = -kk * d1[r][2];
              R[3] = kk * (v1r[r] * h1.idt - acc);
              R[4] = -kk * d1[r][3]; R[5] = -kk * d1[r][4]; R[6] = -kk * d1[r][5];
              eh[7 + r] = sw[r] * e;
            }
          }
        }
        if (a == 0) { /* start edge */
          const double* vs = db.vel_start + 4 * (size_t)b;
          if (vs[3] != 0) {
            const double tw[3] = {vs[0], vs[2], vs[1]};
#pragma unroll
            for (int r = 0; r < 3; ++r) {
              const double acc = (v1r[r] - tw[r]) * h1.idt;
              double sl;
              const double e = pen_interval(acc, lim[r], kp.p.penalty_epsilon, sl);
              const double kk = sw[r] * sl * h1.idt;
              double* S = sStart + 7 * r;
              S[0] = S[1] = S[2] = 0; /* pose 0 is fixed */
              S[3] = kk * (-v1r[r] * h1.idt - acc);
              S[4] = kk * d1[r][3]; S[5] = kk * d1[r][4]; S[6] = kk * d1[r][5];
              if (fb) { S[4] = S[5] = S[6] = 0; }
              sStart[START_E + r] = sw[r] * e;
              if (a >= p0) csum += sStart[START_E + r] * sStart[START_E + r];
            }
          }
        }
      } else if (part == 1 && kp.has_acc) {
        double* R0 = J + J_ACC;
        double* R1 = J + J_ACC + 11;
        if (a <= n - 3) { /* EdgeAcceleration edge_acceleration.h:134-145 */
          const double* q2 = q1 + 9;
          const double v2 = q2[0], w2 = q2[1], idt2 = q2[2];
          const double dt1 = pa[3], dt2 = pb[3];
          const double iT = 1.0 / (dt1 + dt2);
          const double acc = (v2 - v1) * 2 * iT;
          const double accr = (w2 - w1) * 2 * iT;
          double s0, s1;
          const double e0 = pen_interval(acc, kp.p.acc_lim_x, kp.p.penalty_epsilon, s0);
          const double e1 = pen_interval(accr, kp.p.acc_lim_theta, kp.p.penalty_epsilon, s1);
          const double k0 = kp.sw_acc_x * s0 * iT, k1 = kp.sw_acc_th * s1 * iT;
          R0[0] = -2 * k0 * q1[3]; R0[1] = -2 * k0 * q1[4]; R0[2] = -2 * k0 * q1[5];
          R0[3] = k0 * (2 * v1 * idt1 - acc);
          R0[4] = 2 * k0 * (q2[3] - q1[6]); R0[5] = 2 * k0 * (q2[4] - q1[7]); R0[6] = 2 * k0 * (q2[5] - q1[8]);
          R0[7] = k0 * (-2 * v2 * idt2 - acc);
          R0[8] = 2 * k0 * q2[6]; R0[9] = 2 * k0 * q2[7]; R0[10] = 2 * k0 * q2[8];
          R1[2] = 2 * k1 * idt1;
          R1[3] = k1 * (2 * w1 * idt1 - accr);
          R1[6] = 2 * k1 * (-idt2 - idt1);
          R1[7] = k1 * (-2 * w2 * idt2 - accr);
          R1[10] = 2 * k1 * idt2;
          eh[7] = kp.sw_acc_x * e0; eh[8] = kp.sw_acc_th * e1;
          if (a + 2 == n - 1) { R0[8] = R0[9] = R0[10] = 0; R1[10] = 0; }
        } else { /* a == n-2: EdgeAccelerationGoal edge_acceleration.h:420-433 */
          const double* vg = db.vel_goal + 4 * (size_t)b;
          if (vg[3] != 0) {
            const double acc = (vg[0] - v1) * idt1;
            const double accr = (vg[2] - w1) * idt1;
            double s0, s1;
            const double e0 = pen_interval(acc, kp.p.acc_lim_x, kp.p.penalty_epsilon, s0);
            const double e1 = pen_interval(accr, kp.p.acc_lim_theta, kp.p.penalty_epsilon, s1);
            const double k0 = kp.sw_acc_x * s0 * idt1, k1 = kp.sw_acc_th * s1 * idt1;
            R0[0] = -k0 * q1[3]; R0[1] = -k0 * q1[4]; R0[2] = -k0 * q1[5];
            R0[3] = k0 * (v1 * idt1 - acc);
            R0[4] = -k0 * q1[6]; R0[5] = -k0 * q1[7]; R0[6] = -k0 * q1[8];
            R1[2] = k1 * idt1; R1[3] = k1 * (w1 * idt1 - accr); R1[6] = -k1 * idt1;
            eh[7] = kp.sw_acc_x * e0; eh[8] = kp.sw_acc_th * e1;
          }
        }
        if (a == 0) { /* EdgeAccelerationStart edge_acceleration.h:328-341 */
          const double* vs = db.vel_start + 4 * (size_t)b;
          if (vs[3] != 0) {
            const double acc = (v1 - vs[0]) * idt1;
            const double accr = (w1 - vs[2]) * idt1;
            double s0, s1;
            const double e0 = pen_interval(acc, kp.p.acc_lim_x, kp.p.penalty_epsilon, s0);
            const double e1 = pen_interval(accr, kp.p.acc_lim_theta, kp.p.penalty_epsilon, s1);
            const double k0 = kp.sw_acc_x * s0 * idt1, k1 = kp.sw_acc_th * s1 * idt1;
            double* S0 = sStart;
            double* S1 = sStart + 7;
            S0[0] = 0; S0[1] = 0; S0[2] = 0; /* pose 0 is fixed */
            S0[3] = k0 * (-v1 * idt1 - acc);
            S0[4] = k0 * q1[6]; S0[5] = k0 * q1[7]; S0[6] = k0 * q1[8];
            S1[0] = S1[1] = S1[2] = S1[4] = S1[5] = 0;
            S1[3] = k1 * (-w1 * idt1 - accr);
            S1[6] = k1 * idt1;
            if (fb) { S0[4] = S0[5] = S0[6] = 0; S1[6] = 0; }
            sStart[START_E] = kp.sw_acc_x * e0; sStart[START_E + 1] = kp.sw_acc_th * e1;
            if (a >= p0) csum += sStart[START_E] * sStart[START_E] + sStart[START_E + 1] * sStart[START_E + 1];
          }
        }
      }
      /* columns of fixed poses carry no unknowns (g2o skips fixed vertices, SURVEY App. A.3) */
      if (fa) {
        if (part == 0) {
#pragma unroll
          for (int k = 0; k < (HOLO ? 7 : 6); ++k) { J[7 * k] = 0; J[7 * k + 1] = 0; J[7 * k + 2] = 0; }
        } else {
#pragma unroll
          for (int k = 0; k < (HOLO ? 3 : 2); ++k) { J[J_ACC + 11 * k] = 0; J[J_ACC + 11 * k + 1] = 0; J[J_ACC + 11 * k + 2] = 0; }
        }
      }
      if (fb) {
        if (part == 0) {
#pragma unroll
          for (int k = 0; k < (HOLO ? 7 : 6); ++k) { J[7 * k + 4] = 0; J[7 * k + 5] = 0; J[7 * k + 6] = 0; }
        } else {
#pragma unroll
          for (int k = 0; k < (HOLO ? 3 : 2); ++k) { J[J_ACC + 11 * k + 4] = 0; J[J_ACC + 11 * k + 5] = 0; J[J_ACC + 11 * k + 6] = 0; }
        }
      }
      if (a >= p0) {
        if (part == 0) {
#pragma unroll
          for (int k = 0; k < (HOLO ? 7 : 6); ++k) csum += eh[k] * eh[k];
        } else {
          csum += eh[7] * eh[7] + eh[8] * eh[8];
          if (HOLO) csum += eh[9] * eh[9];
        }
        chi3 += csum;
      }
    }
  return chi3;
}

/* One band row r = 4(p0 + t/4) + t%4: gathers J^T J over the (<= 3) anchors that touch it, adds the unary block and
 * the time-optimal term. acc[k] = H[r][r-k], brow = b[r]. */
template <bool HOLO>
__device__ __forceinline__ void gather_row(const KParams& kp, int t, int p0, int n, const double* sP, const double* sJ,
                                           const double* sE, const double* sStart, const double* sU, double (&acc)[11],
                                           double& brow) {
#pragma unroll
  for (int k = 0; k < 11; ++k) acc[k] = 0;
  brow = 0;
  const int tid = t;
  {
    const int il = tid >> 2, c = tid & 3;
    const int i = p0 + il;
    const int r = 4 * i + c;
    if (i < n) {
      if (!row_is_real(r, n)) {
        acc[0] = 1.0;
      } else {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          const int a = i - d;
          const int l = c + 4 * d;
          if (a < 0 || a > n - 2 || l > 10) continue;
          const int slot = a - (p0 - 2);
          const double* J = sJ + (size_t)slot * JSTRIDE;
          const double* eh = sE + ESTR * slot;
          if (l <= 6) {
#pragma unroll
            for (int k = 0; k < (HOLO ? 7 : 6); ++k) {
              if ((k == 4 && !kp.has_sp) || (k == 5 && !kp.has_rot)) continue; /* family switched off: rows are zero */
              const double jl = J[7 * k + l];
              if (jl != 0) {
                brow -= jl * eh[k];
#pragma unroll
                for (int o = 0; o <= 6; ++o)
                  if (o <= l) acc[o] += jl * J[7 * k + l - o];
              }
            }
            if (a == 0) {
#pragma unroll
              for (int k = 0; k < (HOLO ? 3 : 2); ++k) {
                const double jl = sStart[7 * k + l];
                if (jl != 0) {
                  brow -= jl * sStart[START_E + k];
#pragma unroll
                  for (int o = 0; o <= 6; ++o)
                    if (o <= l) acc[o] += jl * sStart[7 * k + l - o];
                }
              }
            }
          }
#pragma unroll
          for (int k = 0; k < (HOLO ? 3 : 2); ++k) {
            const double* R = J + J_ACC + 11 * k;
            const double jl = R[l];
            if (jl != 0) {
              brow -= jl * eh[7 + k];
#pragma unroll
              for (int o = 0; o <= 10; ++o)
                if (o <= l) acc[o] += jl * R[l - o];
            }
          }
        }
        if (c < 3) {
          const double* u = sU + 9 * il;
          if (c == 0) { acc[0] += u[0]; brow += u[6]; }
          else if (c == 1) { acc[0] += u[2]; acc[1] += u[1]; brow += u[7]; }
          else { acc[0] += u[5]; acc[1] += u[4]; acc[2] += u[3]; brow += u[8]; }
        } else if (kp.has_time) {
          acc[0] += kp.p.weight_optimaltime;
          brow -= kp.p.weight_optimaltime * sP[4 * (il + 2) + 3];
        }
      }
    }
  }
}

/* ------------------------------------------------------------------ k_linearize ("kernel A") */
struct KASmem {
  /* sizes in doubles */
  static constexpr int POSES = (TP + 4) * 4;
  static constexpr int SC = (TP + 4) * 2;
  static constexpr int SEG = (TP + 3) * 9;
  static constexpr int JB = (TP + 2) * JSTRIDE;
  static constexpr int EH = (TP + 2) * ESTR;
  static constexpr int START = 3 * 7 + 3;
  static constexpr int UN = TP * 9;
  static constexpr int RED = 4 * (KA_THREADS / 32) + 8 + (KA_THREADS / 32);
  static constexpr int STAGE = KA_THREADS * HROW; /* output stage of the tile (128 rows x 12); reuses the Jacobian region */
};

__host__ __device__ inline size_t ka_smem_bytes(int M_cap) {
  size_t d = KASmem::POSES + KASmem::SC + KASmem::SEG + KASmem::EH + KASmem::START + KASmem::UN + KASmem::RED + 2;
  size_t jb = KASmem::JB > KASmem::STAGE ? KASmem::JB : KASmem::STAGE;
  return (d + jb) * sizeof(double) + (size_t)M_cap * sizeof(TebObstacle) + 64;
}

template <bool HOLO, bool GEOM>
__global__ void __launch_bounds__(KA_THREADS, 6) k_linearize(DevBatch db, KParams kp) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int b = linearize_band(db, blockIdx.y);
  if (b < 0) return;
  const BandState* st = &db.state[b];
  if (!st->active) return;
  const int n = db.n[b];
  const int p0 = blockIdx.x * TP;
  if (p0 >= n) return;
  const int tid = threadIdx.x;

  double* sP = reinterpret_cast<double*>(smem_raw);             /* poses tile, slot j <-> pose p0-2+j */
  double* sJ = sP + KASmem::POSES;                              /* Jacobian blocks, later the output stage */
  constexpr int JBMAX = KASmem::JB > KASmem::STAGE ? KASmem::JB : KASmem::STAGE;
  double* sSC = sJ + JBMAX;
  double* sSeg = sSC + KASmem::SC;
  double* sE = sSeg + KASmem::SEG;
  double* sStart = sE + KASmem::EH;
  double* sU = sStart + KASmem::START;
  double* sRed = sU + KASmem::UN;
  uint64_t* bar = reinterpret_cast<uint64_t*>(sRed + KASmem::RED);
  TebObstacle* so = reinterpret_cast<TebObstacle*>(
      (reinterpret_cast<uintptr_t>(bar) + 16 + 15) & ~static_cast<uintptr_t>(15)); /* TMA destination: 16-byte aligned */

  const int s = db.scene_id[b];
  const int M = db.obst_count[s];
  const int lo = max(p0 - 2, 0), hi = min(p0 + TP + 2, n); /* poses staged */
  const double* gP = db.poses + (size_t)b * db.n_cap * 4;

  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    const uint32_t bytesP = (uint32_t)(hi - lo) * 32u;
    const uint32_t bytesO = (uint32_t)M * (uint32_t)sizeof(TebObstacle);
    mbar_expect_tx(bar, bytesP + bytesO);
    tma_load_1d(sP + (size_t)(lo - (p0 - 2)) * 4, gP + (size_t)lo * 4, bytesP, bar);
    if (bytesO) tma_load_1d(so, db.obstacles + (size_t)s * db.M_cap, bytesO, bar);
  }
  /* zero the Jacobian blocks while the copies are in flight */
  {
    double2* z2 = reinterpret_cast<double2*>(sJ); /* sJ is 16-byte aligned, JB is even */
    constexpr int NZ2 = KASmem::JB / 2, NZE = KASmem::EH + KASmem::START;
    /* fully unrolled: only the last store of each group needs a bounds test */
#pragma unroll
    for (int q = 0; q < (NZ2 + KA_THREADS - 1) / KA_THREADS; ++q) {
      const int k = tid + q * KA_THREADS;
      if ((q + 1) * KA_THREADS <= NZ2 || k < NZ2) z2[k] = make_double2(0.0, 0.0);
    }
#pragma unroll
    for (int q = 0; q < (NZE + KA_THREADS - 1) / KA_THREADS; ++q) {
      const int k = tid + q * KA_THREADS;
      if ((q + 1) * KA_THREADS <= NZE || k < NZE) sE[k] = 0.0;
    }
  }
  mbar_wait(bar, 0);

  double chi[4] = {0, 0, 0, 0}; /* obstacles, via, time-optimal, other */

  /* stage 1 (warps 0-2): sin/cos of every staged pose and the derivative bundle of the segment that starts there
   * (slot j <-> pose / segment p0-2+j); stage 1' (warps 6-7, concurrently): unary terms of the tile's poses */
  if (tid < TP + 4) {
    const int i = p0 - 2 + tid;
    if (i >= lo && i < hi) {
      double sn, cs;
      sincos(sP[4 * tid + 2], &sn, &cs);
      sSC[2 * tid] = cs;
      sSC[2 * tid + 1] = sn;
      if (tid < TP + 3 && i + 1 < hi && i <= n - 2) {
        const double* pa = sP + 4 * tid;
        const double* pb = pa + 4;
        SegDer sd = seg_derivs(kp, pa[0], pa[1], pa[2], cs, sn, pb[0], pb[1], pb[2], pa[3]);
        double* q = sSeg + 9 * tid;
        q[0] = sd.v; q[1] = sd.w; q[2] = sd.idt;
#pragma unroll
        for (int k = 0; k < 6; ++k) q[3 + k] = sd.dv[k];
      }
    }
  }
  {
    const int il = tid - (KA_THREADS - TP); /* last TP threads */
    if (il >= 0) {
      const int i = p0 + il;
      double U[6] = {0, 0, 0, 0, 0, 0}, ub[3] = {0, 0, 0};
      if (i < n) {
        const int j = il + 2;
        double sn = 0, cs = 1;
        if (kp.p.footprint_type >= TEB_FOOTPRINT_TWO_CIRCLES) sincos(sP[4 * j + 2], &sn, &cs);
        unary_terms<GEOM>(kp, db, b, s, i, n, sP[4 * j], sP[4 * j + 1], cs, sn, so, M, true, U, ub, chi[0], chi[1]);
        if (kp.has_time && i <= n - 2) { /* EdgeTimeOptimal edge_time_optimal.h:93 */
          const double dt = sP[4 * j + 3];
          chi[2] += kp.p.weight_optimaltime * dt * dt;
        }
      }
      double* u = sU + 9 * il;
#pragma unroll
      for (int k = 0; k < 6; ++k) u[k] = U[k];
      u[6] = ub[0]; u[7] = ub[1]; u[8] = ub[2];
    }
  }
  __syncthreads();


  /* stage 3a: chain edges anchored at a (EdgeVelocity, EdgeKinematics*, EdgeShortestPath, EdgePreferRotDir,
   * EdgeAcceleration / Start / Goal) -> sqrt(weight)-scaled Jacobian rows over the columns 4a .. 4a+10 */
  /* group 0 (warps 0-2): velocity / kinematics / shortest-path / rotdir rows; group 1 (warps 3-5): acceleration rows */
  const int part = (tid < TP + 2) ? 0 : ((tid >= KA_P1OFF && tid < KA_P1OFF + TP + 2) ? 1 : -1);
  if (part >= 0) {
    const int at = part == 0 ? tid : tid - KA_P1OFF; /* anchor slot */
    chi[3] += anchor_rows<HOLO>(kp, db, b, part, at, p0, n, sP, sSC, sSeg, sJ, sE, sStart);
  }

  __syncthreads();

  /* stage 4: one thread per band row r = 4i + c gathers J^T J over the (<= 3) anchors that touch it */
  double acc[11];
  double brow;
  gather_row<HOLO>(kp, tid, p0, n, sP, sJ, sE, sStart, sU, acc, brow);
  __syncthreads(); /* every thread is done reading sJ: reuse it as the output stage */
  {
    double* o = sJ + (size_t)tid * HROW;
#pragma unroll
    for (int k = 0; k < 11; ++k) o[k] = acc[k];
    o[11] = brow;
    if (p0 + (tid >> 2) < n) db.rhs[(size_t)b * 4 * db.n_cap + 4 * p0 + tid] = brow;
  }
  fence_proxy_async();
  __syncthreads();
  if (tid == 0) {
    const int rows = 4 * (min(p0 + TP, n) - p0);
    double* gH = db.Hb + ((size_t)b * 4 * db.n_cap + (size_t)4 * p0) * HROW;
    tma_store_1d(gH, sJ, (uint32_t)rows * HROW * 8u);
    tma_store_commit_wait();
  }
  /* tile partials: chi2 by family and the max diagonal of the real rows (computeLambdaInit). Every thread parks its
   * five values in shared memory (the dead Jacobian region behind the output stage), then ONE warp folds them in a
   * fixed order - a quarter of the shuffle traffic of a per-warp tree reduction. */
  {
    const int il = tid >> 2, c = tid & 3;
    const int r = 4 * (p0 + il) + c;
    const double dm = (p0 + il < n && row_is_real(r, n)) ? fabs(acc[0]) : 0.0;
    static_assert((KASmem::JB > KASmem::STAGE ? KASmem::JB : KASmem::STAGE) >= KA_THREADS * HROW + 5 * KA_THREADS,
                  "partials do not fit behind the output stage");
    double* park = sJ + KA_THREADS * HROW; /* stage uses KA_THREADS*HROW doubles of the JBMAX region */
    park[0 * KA_THREADS + tid] = chi[0];
    park[1 * KA_THREADS + tid] = chi[1];
    park[2 * KA_THREADS + tid] = chi[2];
    park[3 * KA_THREADS + tid] = chi[3];
    park[4 * KA_THREADS + tid] = dm;
    __syncthreads();
    if (tid < 32) {
      double v[5];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        double sacc = 0;
#pragma unroll
        for (int w = 0; w < KA_THREADS / 32; ++w) sacc += park[k * KA_THREADS + w * 32 + tid];
        v[k] = warp_sum(sacc);
      }
      double m = 0;
#pragma unroll
      for (int w = 0; w < KA_THREADS / 32; ++w) m = fmax(m, park[4 * KA_THREADS + w * 32 + tid]);
      v[4] = warp_max(m);
      if (tid == 0) {
        double* cp = db.chi_parts + ((size_t)b * db.chunks + blockIdx.x) * 4;
        cp[0] = v[0]; cp[1] = v[1]; cp[2] = v[2]; cp[3] = v[3];
        db.dmax_parts[(size_t)b * db.chunks + blockIdx.x] = v[4];
      }
    }
  }
}

/* ------------------------------------------------------------------ trial chi2 (residuals only) on a band held in
 * shared memory: sT[n][4]; block-wide, result in out[4] (shared) after the call */
/* chi2 contributions (residuals only) of everything anchored at pose i of the band stored at sT[n][4]
 * (shared or global memory): chain edges of segment i, time-optimal edge i, unary edges of pose i */
/* Carry between consecutive poses of one thread's chunk: sin/cos of the next pose and the (v, omega) of the next
 * segment are produced while evaluating pose i and are exactly what pose i+1 needs first. */
struct ChainCarry {
  double ca, sa;
  SegVal s;
  bool has_cs, has_seg;
};

template <bool GEOM>
__device__ __forceinline__ void pose_chi2(const KParams& kp, const DevBatch& db, int b, int sc, int i, int n, const double* sT,
                                          const TebObstacle* so, int M, const double* vs, const double* vg,
                                          double (&chi)[4], ChainCarry& cy) {
    const double* pa = sT + 4 * i;
    double sa, ca;
    if (cy.has_cs) { sa = cy.sa; ca = cy.ca; }
    else sincos(pa[2], &sa, &ca);
    cy.has_cs = false;
    const bool had_seg = cy.has_seg;
    cy.has_seg = false;
    if (i <= n - 2) {
      const double* pb = pa + 4;
      double sb, cb;
      sincos(pb[2], &sb, &cb);
      cy.ca = cb; cy.sa = sb; cy.has_cs = true;
      const SegVal s1 = had_seg ? cy.s : seg_value(kp, pa[0], pa[1], pa[2], ca, sa, pb[0], pb[1], pb[2], pa[3]);
      const double dx = pb[0] - pa[0], dy = pb[1] - pa[1];
      double sl, csum = 0;
      if (kp.has_vel && kp.holo_vel) {
        double e[3], s3[3], c0, c1;
        holo_velocity_terms(kp, s1.vx, s1.vy, s1.w, e, s3, c0, c1);
        const double e0 = kp.sw_vel_x * e[0], e1 = kp.sw_vel_y * e[1], e2 = kp.sw_vel_th * e[2];
        csum += e0 * e0 + e1 * e1 + e2 * e2;
      } else if (kp.has_vel) {
        const double e0 = kp.sw_vel_x * pen_interval2(s1.v, -kp.p.max_vel_x_backwards, kp.p.max_vel_x, kp.p.penalty_epsilon, sl);
        const double e1 = kp.sw_vel_th * pen_interval(s1.w, kp.p.max_vel_theta, kp.p.penalty_epsilon, sl);
        csum += e0 * e0 + e1 * e1;
      }
      if (kp.has_kin) {
        const double e0 = kp.sw_kin_nh * fabs((ca + cb) * dy - (sa + sb) * dx);
        double e1 = 0;
        if (!kp.carlike) {
          e1 = pen_below(dx * ca + dy * sa, 0, 0, sl);
        } else {
          const double ad = normalize_theta(pb[2] - pa[2]);
          if (ad != 0) {
            const double nrm = sqrt(dx * dx + dy * dy);
            const double r = kp.p.exact_arc_length ? fabs(nrm / (2 * sin(ad / 2))) : nrm / fabs(ad);
            e1 = pen_below(r, kp.p.min_turning_radius, 0.0, sl);
          }
        }
        e1 *= kp.sw_kin_2;
        csum += e0 * e0 + e1 * e1;
      }
      if (kp.has_sp) {
        const double e = kp.sw_sp * sqrt(dx * dx + dy * dy);
        csum += e * e;
      }
      if (kp.has_rot && i < 3) {
        const int rd = db.prefer_rotdir ? db.prefer_rotdir[b] : 0;
        if (rd == TEB_ROTDIR_LEFT || rd == TEB_ROTDIR_RIGHT) {
          const double meas = (rd == TEB_ROTDIR_LEFT) ? 1.0 : -1.0;
          const double e = kp.sw_rot * pen_below(meas * normalize_theta(pb[2] - pa[2]), 0, 0, sl);
          csum += e * e;
        }
      }
      if (kp.has_acc && kp.holo_acc) {
        const double idt1 = 1.0 / pa[3];
        const double lim[3] = {kp.p.acc_lim_x, kp.p.acc_lim_y, kp.p.acc_lim_theta};
        const double sw[3] = {kp.sw_acc_x, kp.sw_acc_y, kp.sw_acc_th};
        const double u1[3] = {s1.vx, s1.vy, s1.w};
        if (i <= n - 3) {
          const double* pc = pb + 4;
          const SegVal s2 = seg_value(kp, pb[0], pb[1], pb[2], cb, sb, pc[0], pc[1], pc[2], pb[3]);
          cy.s = s2; cy.has_seg = true;
          const double iT = 1.0 / (pa[3] + pb[3]);
          const double u2[3] = {s2.vx, s2.vy, s2.w};
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            const double e = sw[r] * pen_interval((u2[r] - u1[r]) * 2 * iT, lim[r], kp.p.penalty_epsilon, sl);
            csum += e * e;
          }
        } else if (vg[3] != 0) {
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            const double e = sw[r] * pen_interval((vg[r] - u1[r]) * idt1, lim[r], kp.p.penalty_epsilon, sl);
            csum += e * e;
          }
        }
        if (i == 0 && vs[3] != 0) {
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            const double e = sw[r] * pen_interval((u1[r] - vs[r]) * idt1, lim[r], kp.p.penalty_epsilon, sl);
            csum += e * e;
          }
        }
      } else if (kp.has_acc) {
        const double idt1 = 1.0 / pa[3];
        if (i <= n - 3) {
          const double* pc = pb + 4;
          const SegVal s2 = seg_value(kp, pb[0], pb[1], pb[2], cb, sb, pc[0], pc[1], pc[2], pb[3]);
          cy.s = s2; cy.has_seg = true;
          const double iT = 1.0 / (pa[3] + pb[3]);
          const double e0 = kp.sw_acc_x * pen_interval((s2.v - s1.v) * 2 * iT, kp.p.acc_lim_x, kp.p.penalty_epsilon, sl);
          const double e1 = kp.sw_acc_th * pen_interval((s2.w - s1.w) * 2 * iT, kp.p.acc_lim_theta, kp.p.penalty_epsilon, sl);
          csum += e0 * e0 + e1 * e1;
        } else if (vg[3] != 0) {
          const double e0 = kp.sw_acc_x * pen_interval((vg[0] - s1.v) * idt1, kp.p.acc_lim_x, kp.p.penalty_epsilon, sl);
          const double e1 = kp.sw_acc_th * pen_interval((vg[2] - s1.w) * idt1, kp.p.acc_lim_theta, kp.p.penalty_epsilon, sl);
          csum += e0 * e0 + e1 * e1;
        }
        if (i == 0 && vs[3] != 0) {
          const double e0 = kp.sw_acc_x * pen_interval((s1.v - vs[0]) * idt1, kp.p.acc_lim_x, kp.p.penalty_epsilon, sl);
          const double e1 = kp.sw_acc_th * pen_interval((s1.w - vs[2]) * idt1, kp.p.acc_lim_theta, kp.p.penalty_epsilon, sl);
          csum += e0 * e0 + e1 * e1;
        }
      }
      if (kp.has_vor) { /* EdgeVelocityObstacleRatio: obstacles associated with pose i (pose 0 included) */
        const unsigned long long* am = db.assoc + ((size_t)b * db.n_cap + i) * db.MW;
        for (int w = 0; w < db.MW; ++w) {
          unsigned long long mask = am[w];
          while (mask) {
            const int m = (w << 6) + __ffsll((long long)mask) - 1;
            mask &= mask - 1;
            const TebObstacle ob = so[m];
            double dratio;
            const double d = robot_obstacle_distance_only<GEOM>(kp, db.obst_vertices + (size_t)sc * db.PV_cap * 2, pa[0], pa[1], ca, sa, ob,
                                                          ob.x, ob.y, 0.0, 0.0);
            const double ratio = proximity_ratio(kp, d, dratio);
            const double e0 = pen_interval(s1.v, ratio * kp.p.max_vel_x, 0, sl);
            const double e1 = pen_interval(s1.w, ratio * kp.p.max_vel_theta, 0, sl);
            csum += kp.p.weight_velocity_obstacle_ratio * (e0 * e0 + e1 * e1);
          }
        }
      }
      chi[3] += csum;
      if (kp.has_time) chi[2] += kp.p.weight_optimaltime * pa[3] * pa[3];
    }
    double U[6], ub[3];
    unary_terms<GEOM>(kp, db, b, sc, i, n, pa[0], pa[1], ca, sa, so, M, false, U, ub, chi[0], chi[1]);
}

template <int NTHREADS, bool GEOM>
__device__ __forceinline__ void eval_chi2_parts(const KParams& kp, const DevBatch& db, int b, int n, const double* sT,
                                                const TebObstacle* so, int M, double* scratch, double* out) {
  double chi[4] = {0, 0, 0, 0};
  const double* vs = db.vel_start + 4 * (size_t)b;
  const double* vg = db.vel_goal + 4 * (size_t)b;
  const int sc = db.scene_id[b];
  for (int i = threadIdx.x; i < n; i += NTHREADS) {
    ChainCarry cy;
    cy.has_cs = false; cy.has_seg = false;
    pose_chi2<GEOM>(kp, db, b, sc, i, n, sT, so, M, vs, vg, chi, cy);
  }
  block_sum<4, NTHREADS / 32>(chi, scratch, out);
}

/* ------------------------------------------------------------------ banded LDL^T + substitutions, one warp, in
 * shared memory. Hs[N][12]: on entry band + rhs, on exit L (unit lower, offsets 1..10), 1/d (offset 0) and the
 * solution (offset 11). Returns false on a non-positive / non-finite pivot (LinearSolverCSparse would fail) or a
 * non-finite solution. */
__device__ __forceinline__ bool warp_band_solve(double* Hs, int N, int n, double lambda) {
  const int lane = threadIdx.x & 31;
  /* trailing-window entries handled by this lane: e in {lane, lane+32, lane+64}; e < 55 -> (u,q), 1<=q<=u<=10;
   * 55 <= e < 65 -> rhs of row j+u, u = e-54 */
  int eu[3], eq[3];
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    const int e = lane + 32 * t;
    if (e < 55) {
      int u = 1;
      while ((u * (u + 1)) / 2 <= e) ++u;
      eu[t] = u;
      eq[t] = e - (u * (u - 1)) / 2 + 1;
    } else if (e < 65) {
      eu[t] = e - 54;
      eq[t] = 0; /* rhs */
    } else {
      eu[t] = 0;
      eq[t] = 0;
    }
  }
  bool ok = true;
  for (int j = 0; j < N; ++j) {
    const double d = Hs[j * HROW] + (row_is_real(j, n) ? lambda : 0.0);
    if (!(d > 0) || !isfinite(d)) { ok = false; break; }
    const double inv = 1.0 / d;
    const double yj = Hs[j * HROW + 11];
#pragma unroll
    for (int t = 0; t < 3; ++t) {
      const int u = eu[t];
      if (u == 0 || j + u >= N) continue;
      const double cu = Hs[(j + u) * HROW + u];
      if (eq[t] == 0) {
        Hs[(j + u) * HROW + 11] -= cu * inv * yj;
      } else {
        const int q = eq[t];
        const double cq = Hs[(j + q) * HROW + q];
        Hs[(j + u) * HROW + (u - q)] -= cu * inv * cq;
      }
    }
    __syncwarp();
    if (lane >= 1 && lane <= 10 && j + lane < N) Hs[(j + lane) * HROW + lane] *= inv;
    if (lane == 0) Hs[j * HROW] = inv;
    __syncwarp();
  }
  if (!ok) return false;
  /* z = D^-1 y */
  for (int j = lane; j < N; j += 32) Hs[j * HROW + 11] *= Hs[j * HROW];
  __syncwarp();
  /* L^T x = z, column-oriented */
  for (int j = N - 1; j >= 1; --j) {
    const double xj = Hs[j * HROW + 11];
    if (lane >= 1 && lane <= 10 && j - lane >= 0) Hs[(j - lane) * HROW + 11] -= Hs[j * HROW + lane] * xj;
    __syncwarp();
  }
  /* and every component of the solution finite (a NaN in b leaves the pivots alone): the rule of every solve kernel */
  for (int j = lane; j < N; j += 32) ok = ok && isfinite(Hs[j * HROW + 11]);
  return __all_sync(0xffffffffu, ok);
}

/* ------------------------------------------------------------------ block cyclic reduction (BCR) solver
 * The padded normal matrix is block tridiagonal with 8x8 blocks (two pose groups per block; an acceleration edge spans
 * the scalars 4i..4i+10, i.e. at most two adjacent blocks). BCR eliminates every other block per level: log2(m)
 * dependent levels instead of 4n dependent pivots. SPD Schur complements stay SPD, so every pivot block has a Cholesky
 * factor unless H + lambda I is not numerically positive definite (the LinearSolverCSparse failure condition).
 *
 * Per eliminated block i (neighbours p = i-s, q = i+s at stride s): D_i = C C^T,
 *   W^L = C^-1 A_ip, W^R = C^-1 A_iq (stored transposed in q's coupling slot), w = C^-1 b_i,
 *   D_p -= W^L^T W^L, D_q -= W^R^T W^R, A_qp(new) = -W^R^T W^L, b_p -= W^L^T w, b_q -= W^R^T w,
 *   back-substitution x_i = C^-T (w - W^L x_p - W^R x_q). Only C^-1 (packed lower) is stored. */
__host__ __device__ inline int bcr_blocks(int n_cap) { return (4 * n_cap + 7) / 8; }
struct BcrSmem {
  double* Dp;     /* [m][36] packed lower diagonal blocks -> C^-1 after elimination */
  double* L0;     /* [m][64] level-0 left couplings A_{i,i-1}, row major             */
  double* Lpool;  /* couplings created at levels >= 1                                 */
  double* bs;     /* [m][8] rhs -> w                                                  */
  double* xs;     /* [m][8] solution                                                  */
  int off[12];    /* pool offset (in blocks) of level l                               */
};
__device__ __forceinline__ double* bcr_L(const BcrSmem& S, int lvl, int i) {
  return lvl == 0 ? S.L0 + 64 * i : S.Lpool + 64 * (S.off[lvl] + (i >> lvl));
}
#define PIDX(a, c) (((a) * ((a) + 1)) / 2 + (c))

/* in-register Cholesky of a packed 8x8 SPD block and inverse of its factor; in-place safe. */
__device__ __forceinline__ bool chol8_inverse(const double* din, double* cinv_out) {
  double c[36], rinv[8];
#pragma unroll
  for (int k = 0; k < 36; ++k) c[k] = din[k];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const double d = c[PIDX(j, j)];
    if (!(d > 0) || !isfinite(d)) ok = false;
    const double r = rsqrt(d);
    rinv[j] = r;
#pragma unroll
    for (int a = j + 1; a < 8; ++a) c[PIDX(a, j)] *= r;
#pragma unroll
    for (int a = j + 1; a < 8; ++a)
#pragma unroll
      for (int b2 = j + 1; b2 <= a; ++b2) c[PIDX(a, b2)] -= c[PIDX(a, j)] * c[PIDX(b2, j)];
  }
  /* in-place inverse of the lower-triangular factor, column by column (column j of C is dead once X(:,j) is known) */
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    c[PIDX(j, j)] = rinv[j];
#pragma unroll
    for (int a = j + 1; a < 8; ++a) {
      double sacc = c[PIDX(a, j)] * rinv[j];
#pragma unroll
      for (int k = j + 1; k < a; ++k) sacc += c[PIDX(a, k)] * c[PIDX(k, j)];
      c[PIDX(a, j)] = -sacc * rinv[a];
    }
  }
#pragma unroll
  for (int k = 0; k < 36; ++k) cinv_out[k] = c[k];
  return ok;
}
/* z = Cinv v (lower-triangular mat-vec), Cinv packed in shared memory */
__device__ __forceinline__ void tri_mv(const double* ci, const double (&v)[8], double (&z)[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    double sacc = 0;
#pragma unroll
    for (int c = 0; c <= k; ++c) sacc += ci[PIDX(k, c)] * v[c];
    z[k] = sacc;
  }
}

template <int NT>
__device__ __forceinline__ void bcr_solve(const BcrSmem& S, int m, int* s_fail) {
  const int tid = threadIdx.x;
  int Lmax = 0;
  while ((1 << Lmax) < m) ++Lmax;
  for (int lvl = 0; lvl < Lmax; ++lvl) {
    const int s = 1 << lvl;
    const int E = (m > s) ? ((m - s - 1) / (2 * s) + 1) : 0;
    /* phase 1a: C^-1 of every eliminated diagonal block */
    for (int t = tid; t < E; t += NT) {
      const int i = s * (2 * t + 1);
      if (!chol8_inverse(S.Dp + 36 * i, S.Dp + 36 * i)) *s_fail = 1;
    }
    __syncthreads();
    /* phase 1b: W^L (columns of A_ip), W^R^T (rows of A_qi), w */
    for (int t = tid; t < 17 * E; t += NT) {
      const int e = t / 17, r = t - 17 * e;
      const int i = s * (2 * e + 1), q = i + s;
      const double* ci = S.Dp + 36 * i;
      double v[8], z[8];
      if (r < 8) {
        double* L = bcr_L(S, lvl, i);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = L[8 * k + r];
        tri_mv(ci, v, z);
#pragma unroll
        for (int k = 0; k < 8; ++k) L[8 * k + r] = z[k];
      } else if (r < 16) {
        if (q < m) {
          double* L = bcr_L(S, lvl, q) + 8 * (r - 8);
#pragma unroll
          for (int k = 0; k < 8; ++k) v[k] = L[k];
          tri_mv(ci, v, z);
#pragma unroll
          for (int k = 0; k < 8; ++k) L[k] = z[k];
        }
      } else {
        double* bb = S.bs + 8 * i;
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = bb[k];
        tri_mv(ci, v, z);
#pragma unroll
        for (int k = 0; k < 8; ++k) bb[k] = z[k];
      }
    }
    __syncthreads();
    /* phase 2: Schur updates of the surviving blocks e = 2s*u, one thread per block row */
    const int SC = (m + 2 * s - 1) / (2 * s);
    for (int t = tid; t < 8 * SC; t += NT) {
      const int u = t >> 3, a = t & 7;
      const int e = 2 * s * u, iR = e + s, iL = e - s;
      const bool hasR = iR < m, hasL = u > 0;
      double dacc[8], lacc[8], bacc = 0;
#pragma unroll
      for (int c = 0; c < 8; ++c) { dacc[c] = 0; lacc[c] = 0; }
      if (hasR) {
        const double* WL = bcr_L(S, lvl, iR);
        const double* w = S.bs + 8 * iR;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const double wa = WL[8 * k + a];
          bacc += wa * w[k];
#pragma unroll
          for (int c = 0; c < 8; ++c)
            if (c <= a) dacc[c] += wa * WL[8 * k + c];
        }
      }
      if (hasL) {
        const double* Z = bcr_L(S, lvl, e);
        const double* WLl = bcr_L(S, lvl, iL);
        const double* w = S.bs + 8 * iL;
        double za[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) za[k] = Z[8 * a + k];
#pragma unroll
        for (int k = 0; k < 8; ++k) bacc += za[k] * w[k];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          if (c <= a) {
            double sacc = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) sacc += za[k] * Z[8 * c + k];
            dacc[c] += sacc;
          }
        }
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
          for (int c = 0; c < 8; ++c) lacc[c] += za[k] * WLl[8 * k + c];
        double* Ln = bcr_L(S, lvl + 1, e) + 8 * a;
#pragma unroll
        for (int c = 0; c < 8; ++c) Ln[c] = -lacc[c];
      }
      double* De = S.Dp + 36 * e;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c <= a) De[PIDX(a, c)] -= dacc[c];
      S.bs[8 * e + a] -= bacc;
    }
    __syncthreads();
  }
  /* top: block 0 */
  if (tid == 0) {
    if (!chol8_inverse(S.Dp, S.Dp)) *s_fail = 1;
    double v[8], z[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = S.bs[k];
    tri_mv(S.Dp, v, z);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      double sacc = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (k >= c) sacc += S.Dp[PIDX(k, c)] * z[k];
      S.xs[c] = sacc;
    }
  }
  __syncthreads();
  for (int lvl = Lmax - 1; lvl >= 0; --lvl) {
    const int s = 1 << lvl;
    const int E = (m > s) ? ((m - s - 1) / (2 * s) + 1) : 0;
    for (int t = tid; t < 8 * E; t += NT) {
      const int e = t >> 3, k = t & 7;
      const int i = s * (2 * e + 1), p = i - s, q = i + s;
      const double* WL = bcr_L(S, lvl, i);
      double acc = S.bs[8 * i + k];
#pragma unroll
      for (int c = 0; c < 8; ++c) acc -= WL[8 * k + c] * S.xs[8 * p + c];
      if (q < m) {
        const double* Z = bcr_L(S, lvl, q);
#pragma unroll
        for (int a = 0; a < 8; ++a) acc -= Z[8 * a + k] * S.xs[8 * q + a];
      }
      S.bs[8 * i + k] = acc;
    }
    __syncthreads();
    for (int t = tid; t < 8 * E; t += NT) {
      const int e = t >> 3, c = t & 7;
      const int i = s * (2 * e + 1);
      const double* ci = S.Dp + 36 * i;
      double sacc = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (k >= c) sacc += ci[PIDX(k, c)] * S.bs[8 * i + k];
      S.xs[8 * i + c] = sacc;
    }
    __syncthreads();
  }
  /* a solve also fails on a non-finite solution (a NaN in b leaves the pivots alone): the rule of every solve kernel */
  for (int r = tid; r < 8 * m; r += NT)
    if (!isfinite(S.xs[r])) *s_fail = 1;
  __syncthreads();
}

/* BCR staging: the band rows [N][12] (+ lambda on the real diagonals) expanded into the 8x8 blocks of S (coalesced
 * 16-byte loads of each 96-byte row); rows N .. 8m - 1 are identity rows. b0 receives the right-hand side. */
template <int NT>
__device__ __forceinline__ void bcr_stage(const BcrSmem& S, double* b0, const double* gH, int N, int n, int m, double lambda) {
  for (int r = threadIdx.x; r < 8 * m; r += NT) {
    const int i = r >> 3, a = r & 7;
    double* Lrow = S.L0 + 64 * i + 8 * a;
#pragma unroll
    for (int c = 0; c < 8; ++c) Lrow[c] = 0.0;
    double* Dblk = S.Dp + 36 * i;
    if (r < N) {
      const double2* src = reinterpret_cast<const double2*>(gH + (size_t)r * HROW);
      double h[12];
#pragma unroll
      for (int k = 0; k < 6; ++k) { const double2 v2 = src[k]; h[2 * k] = v2.x; h[2 * k + 1] = v2.y; }
      if (row_is_real(r, n)) h[0] += lambda;
#pragma unroll
      for (int k = 0; k < 11; ++k) {
        const int c = a - k;
        if (c >= 0) Dblk[PIDX(a, c)] = h[k];
        else if (c >= -8) Lrow[8 + c] = h[k];
      }
      S.bs[r] = h[11];
      b0[r] = h[11];
    } else {
#pragma unroll
      for (int c = 0; c < 8; ++c)
        if (c <= a) Dblk[PIDX(a, c)] = (c == a) ? 1.0 : 0.0;
      S.bs[r] = 0.0;
      b0[r] = 0.0;
    }
  }
}

/* shared-memory carve-up of the BCR solver for n_cap poses (kb_bcr_smem_bytes) and a system of m blocks; b0: [8 m] */
__device__ __forceinline__ BcrSmem bcr_carve(double* base, int n_cap, int m, double*& b0) {
  const int mc = bcr_blocks(n_cap);
  BcrSmem S;
  S.Dp = base;
  S.L0 = S.Dp + 36 * mc;
  S.Lpool = S.L0 + 64 * mc;
  S.bs = S.Lpool + 64 * (mc + 12);
  S.xs = S.bs + 8 * mc;
  b0 = S.xs + 8 * mc;
  S.off[0] = 0;
  S.off[1] = 0;
  for (int l = 1; l < 11; ++l) S.off[l + 1] = S.off[l] + ((m + (1 << l) - 1) >> l);
  return S;
}

/* ------------------------------------------------------------------ k_lm_step ("kernel B"), CTA per band.
 * SOLVER 0: sequential banded LDL^T by one warp on the TMA-loaded band (any n_cap <= 512);
 * SOLVER 1: block cyclic reduction on the expanded 8x8 block-tridiagonal form (n_cap <= BCR_MAX_POSES). */
constexpr int BCR_MAX_POSES = 256;
constexpr int KB_BCR_THREADS = 256;

__host__ __device__ inline size_t kb_smem_bytes(int n_cap, int M_cap) {
  return ((size_t)4 * n_cap * HROW + (size_t)4 * n_cap + 64) * sizeof(double) + (size_t)M_cap * sizeof(TebObstacle) + 64;
}
__host__ __device__ inline size_t kb_bcr_smem_bytes(int n_cap, int M_cap) {
  const size_t m = bcr_blocks(n_cap);
  /* Dp 36m + L0 64m + Lpool 64(m + 12) + bs 8m + xs 8m + b0 8m + trial poses 4 n_cap + scratch 64 */
  return ((36 + 64 + 64 + 8 + 8 + 8) * m + 64 * 12 + (size_t)4 * n_cap + 64) * sizeof(double) +
         (size_t)M_cap * sizeof(TebObstacle) + 64;
}

template <int SOLVER, int NT, bool GEOM>
__global__ void __launch_bounds__(NT, SOLVER == 1 ? 2 : 1) k_lm_step_t(DevBatch db, KParams kp, int iteration) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int b = blockIdx.x;
  BandState* st = &db.state[b];
  if (!st->active) return;
  const int n = db.n[b];
  const int N = 4 * n;
  const int tid = threadIdx.x;
  __shared__ int s_flag[4];

  /* ---- shared memory carve-up */
  double* Hs = nullptr;   /* SOLVER 0: band [N][12] */
  BcrSmem S;              /* SOLVER 1 */
  double* b0 = nullptr;
  double* sT;
  double* sRed;
  int m = 0;
  if constexpr (SOLVER == 0) {
    Hs = reinterpret_cast<double*>(smem_raw);
    sT = Hs + (size_t)4 * db.n_cap * HROW;
  } else {
    m = (N + 7) / 8;
    S = bcr_carve(reinterpret_cast<double*>(smem_raw), db.n_cap, m, b0);
    sT = b0 + 8 * bcr_blocks(db.n_cap);
  }
  sRed = sT + (size_t)4 * db.n_cap; /* 64 doubles scratch */
  uint64_t* bar = reinterpret_cast<uint64_t*>(sRed + 56);
  TebObstacle* so = reinterpret_cast<TebObstacle*>(sRed + 64);

  const int s = db.scene_id[b];
  const int M = db.obst_count[s];
  double* gP = db.poses + (size_t)b * db.n_cap * 4;
  const double* gH = db.Hb + (size_t)b * 4 * db.n_cap * HROW;

  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
    s_flag[1] = 0;
  }
  __syncthreads();
  uint32_t parity = 0;
  const uint32_t bytesH = (uint32_t)N * HROW * 8u;
  if (tid == 0) {
    const uint32_t bytesO = (uint32_t)M * (uint32_t)sizeof(TebObstacle);
    mbar_expect_tx(bar, (SOLVER == 0 ? bytesH : 0u) + bytesO);
    if constexpr (SOLVER == 0) tma_load_1d(Hs, gH, bytesH, bar);
    if (bytesO) tma_load_1d(so, db.obstacles + (size_t)s * db.M_cap, bytesO, bar);
  }
  /* chi2 at the linearisation point = sum of the kernel-A tile partials (computeActiveErrors, App. A.4) */
  double cur_parts[4] = {0, 0, 0, 0};
  {
    const int chunks_used = (n + db.tile - 1) / db.tile;
    const double* cp = db.chi_parts + (size_t)b * db.chunks * 4;
    for (int c = 0; c < chunks_used; ++c)
      for (int k = 0; k < 4; ++k) cur_parts[k] += cp[4 * c + k];
  }
  double currentChi = cur_parts[0] + cur_parts[1] + cur_parts[2] + cur_parts[3];
  mbar_wait(bar, parity);
  parity ^= 1;

  double lambda = st->lambda, ni = st->ni;
  if (iteration == 0) { /* computeLambdaInit: tau * max diagonal (App. A.4) */
    double mx = 0;
    for (int r = tid; r < N; r += NT)
      if (row_is_real(r, n)) mx = fmax(mx, fabs(SOLVER == 0 ? Hs[r * HROW] : gH[(size_t)r * HROW]));
    mx = warp_max(mx);
    if ((tid & 31) == 0) sRed[tid >> 5] = mx;
    __syncthreads();
    mx = 0;
    for (int w = 0; w < NT / 32; ++w) mx = fmax(mx, sRed[w]);
    __syncthreads();
    lambda = 1e-5 * mx;
    ni = 2;
  }

  double rho = 0;
  int qmax = 0;
  int status_add = 0;
  double last_parts[4] = {cur_parts[0], cur_parts[1], cur_parts[2], cur_parts[3]};
  while (true) {
    /* (H + lambda I) dx = b */
    bool ok2;
    if constexpr (SOLVER == 0) {
      if (tid < 32) {
        const bool ok = warp_band_solve(Hs, N, n, lambda);
        if (tid == 0) s_flag[0] = ok ? 1 : 0;
      }
      __syncthreads();
      ok2 = s_flag[0] != 0;
    } else {
      bcr_stage<NT>(S, b0, gH, N, n, m, lambda);
      if (tid == 0) s_flag[1] = 0;
      __syncthreads();
      bcr_solve<NT>(S, m, &s_flag[1]);
      ok2 = s_flag[1] == 0;
    }
    /* trial state x [+] dx (VertexPose::oplusImpl / VertexTimeDiff::oplusImpl) and computeScale() */
    double sc = 0;
    for (int r = tid; r < N; r += NT) {
      const int i = r >> 2, c = r & 3;
      double xv = gP[r];
      if (row_is_real(r, n)) {
        const double bb = (SOLVER == 0) ? gH[(size_t)r * HROW + 11] : b0[r];
        const double dx = ok2 ? ((SOLVER == 0) ? Hs[r * HROW + 11] : S.xs[r]) : bb; /* CSparse leaves x = b on failure */
        sc += dx * (lambda * dx + bb);
        xv = (c == 2) ? normalize_theta(xv + dx) : xv + dx;
      }
      sT[4 * i + c] = xv;
    }
    __syncthreads();
    double red[1] = {sc};
    block_sum<1, NT / 32>(red, sRed, sRed + 40);
    const double scale = sRed[40] + 1e-3;
    __syncthreads();
    eval_chi2_parts<NT, GEOM>(kp, db, b, n, sT, so, M, sRed, sRed + 40);
    for (int k = 0; k < 4; ++k) last_parts[k] = sRed[40 + k];
    __syncthreads();
    double tempChi = last_parts[0] + last_parts[1] + last_parts[2] + last_parts[3];
    if (!ok2) { tempChi = 1.7976931348623157e308; status_add |= TEB_STATUS_CHOL_FAILED; }
    rho = (currentChi - tempChi) / scale;
    if (rho > 0 && isfinite(tempChi)) {
      double alpha = 1. - pow((2 * rho - 1), 3);
      alpha = fmin(alpha, 2. / 3.);
      const double scaleFactor = fmax(1. / 3., alpha);
      lambda *= scaleFactor;
      ni = 2;
      currentChi = tempChi;
      for (int k = 0; k < 4; ++k) cur_parts[k] = last_parts[k];
      for (int r = tid; r < N; r += NT) gP[r] = sT[r]; /* discardTop(): keep the new state */
    } else {
      lambda *= ni;
      ni *= 2;
      if (!isfinite(lambda)) { status_add |= TEB_STATUS_NONFINITE; break; }
    }
    qmax++;
    if (!(rho < 0 && qmax < 10)) break;
    /* rejected: retry with the larger lambda (SOLVER 0 factorised in place: restore H first) */
    __syncthreads();
    if constexpr (SOLVER == 0) {
      if (tid == 0) {
        mbar_expect_tx(bar, bytesH);
        tma_load_1d(Hs, gH, bytesH, bar);
      }
      mbar_wait(bar, parity);
      parity ^= 1;
    }
  }
  if (tid == 0) {
    const bool terminate = (qmax == 10 || rho == 0 || !isfinite(lambda));
    st->lambda = lambda;
    st->ni = ni;
    st->current_chi = currentChi;
    st->chi2_final = currentChi;
    for (int k = 0; k < 4; ++k) { st->parts_last[k] = last_parts[k]; st->parts_cur[k] = cur_parts[k]; }
    st->lm_iters += 1;
    int stt = st->status | status_add;
    if (terminate) { stt |= TEB_STATUS_TERMINATED; st->active = 0; }
    else stt &= ~TEB_STATUS_TERMINATED;
    st->status = stt;
  }
}

/* ------------------------------------------------------------------ k_finalize (thread per band) */
__global__ void k_finalize(DevBatch db, KParams kp, TebOptimizeArgs args) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= db.B) return;
  const BandState st = db.state[b];
  int status = st.status;
  if (!st.failed && args.iterations_outerloop > 0 && args.iterations_innerloop > 0) status |= TEB_STATUS_OPTIMIZED;
  double cost = __longlong_as_double(0x7ff0000000000000LL); /* cost_ = HUGE_VAL until computed (optimal_planner.cpp:90) */
  if ((status & TEB_STATUS_OPTIMIZED) && args.compute_cost_afterwards) {
    /* computeCurrentCost (optimal_planner.cpp:1041-1094): chi2 of the cached edge errors = last evaluated LM
     * trial, unless batch statistics (divergence detection) refreshed them at the final state */
    const double* parts = kp.p.divergence_detection_enable ? st.parts_cur : st.parts_last;
    cost = 0;
    if (args.alternative_time_cost) {
      const int n = db.n[b];
      const double* P = db.poses + (size_t)b * db.n_cap * 4;
      for (int i = 0; i < n - 1; ++i) cost += P[4 * i + 3];
    }
    cost += args.obst_cost_scale * parts[0] + args.viapoint_cost_scale * parts[1] + parts[3];
    if (!args.alternative_time_cost) cost += parts[2];
  }
  if (db.cost) db.cost[b] = cost;
  if (db.chi2) db.chi2[b] = st.chi2_final;
  if (db.status) db.status[b] = status;
  if (db.lm_iters) db.lm_iters[b] = st.lm_iters;
}

/* ------------------------------------------------------------------ k_vor (CTA per band; launched only when
 * weight_velocity_obstacle_ratio > 0): EdgeVelocityObstacleRatio (edge_velocity_obstacle_ratio.h:82-122,
 * optimal_planner.cpp:999-1021). One edge per obstacle associated with pose a over (pose a, pose a+1, dt_a); the
 * 7x7 J^T Omega J of every anchor is added to the band written by kernel A. Even anchors first, then odd ones, so
 * that overlapping rows are updated in a fixed order (deterministic, no atomics). */
template <bool GEOM, bool GT = false> /* GT: obstacle rows read from global memory, associations via the occupancy words */
__global__ void __launch_bounds__(256) k_vor(const __grid_constant__ DevBatch db, const __grid_constant__ KParams kp) {
  extern __shared__ __align__(16) unsigned char vor_raw[];
  TebObstacle* so_s = reinterpret_cast<TebObstacle*>(vor_raw);
  __shared__ double s_red[8];
  const int b = blockIdx.x;
  if (!db.state[b].active) return;
  const int n = db.n[b];
  const int sc = db.scene_id[b];
  const int M = db.obst_count[sc];
  if constexpr (!GT)
    for (int m = threadIdx.x; m < M; m += blockDim.x) so_s[m] = db.obstacles[(size_t)sc * db.M_cap + m];
  __syncthreads();
  const TebObstacle* so = GT ? db.obstacles + (size_t)sc * db.M_cap : so_s;
  const double* P = db.poses + (size_t)b * db.n_cap * 4;
  const double* pool = db.obst_vertices + (size_t)sc * db.PV_cap * 2;
  double* H = db.Hb + (size_t)b * 4 * db.n_cap * HROW;
  double* rhs = db.rhs + (size_t)b * 4 * db.n_cap;
  const double wv = kp.p.weight_velocity_obstacle_ratio;
  double csum = 0, dmax = 0;
  for (int parity = 0; parity < 2; ++parity) {
    for (int a = 2 * threadIdx.x + parity; a <= n - 2; a += 2 * blockDim.x) {
      const double* pa = P + 4 * a;
      const double* pb = pa + 4;
      double sn, cs;
      sincos(pa[2], &sn, &cs);
      const SegDer sd = seg_derivs(kp, pa[0], pa[1], pa[2], cs, sn, pb[0], pb[1], pb[2], pa[3]);
      const bool fa = (a == 0), fb = (a + 1 == n - 1);
      double G[28], gb[7];
#pragma unroll
      for (int k = 0; k < 28; ++k) G[k] = 0;
#pragma unroll
      for (int k = 0; k < 7; ++k) gb[k] = 0;
      const unsigned long long* am = db.assoc + ((size_t)b * db.n_cap + a) * db.MW;
      /* GT: one pass over the occupancy words yields the non-zero words in increasing order */
      const unsigned long long* oc = db.occ + ((size_t)b * db.n_cap + a) * db.OW;
      unsigned long long ow = 0ull;
      int o = 0;
      for (int w = 0; GT ? true : w < db.MW; ++w) {
        if constexpr (GT) {
          while (ow == 0ull && o < db.OW) ow = oc[o++];
          if (ow == 0ull) break;
          w = ((o - 1) << 6) + __ffsll((long long)ow) - 1;
          ow &= ow - 1;
        }
        unsigned long long mask = am[w];
        while (mask) {
          const int m = (w << 6) + __ffsll((long long)mask) - 1;
          mask &= mask - 1;
          const TebObstacle ob = so[m];
          double g[3], dratio;
          const double d = robot_obstacle_distance<GEOM>(kp, pool, pa[0], pa[1], cs, sn, ob, ob.x, ob.y, 0.0, 0.0, g);
          const double ratio = proximity_ratio(kp, d, dratio);
          double s0, s1;
          const double e0 = pen_interval(sd.v, ratio * kp.p.max_vel_x, 0, s0);
          const double e1 = pen_interval(sd.w, ratio * kp.p.max_vel_theta, 0, s1);
          /* e = |var| - a outside the interval: d e / d a = -1 whenever the penalty is active */
          const double a0 = (s0 != 0) ? -kp.p.max_vel_x * dratio : 0.0, a1 = (s1 != 0) ? -kp.p.max_vel_theta * dratio : 0.0;
          double r0[7], r1[7];
          r0[0] = s0 * sd.dv[0] + a0 * g[0]; r0[1] = s0 * sd.dv[1] + a0 * g[1]; r0[2] = s0 * sd.dv[2] + a0 * g[2];
          r0[3] = -s0 * sd.v * sd.idt; r0[4] = s0 * sd.dv[3]; r0[5] = s0 * sd.dv[4]; r0[6] = s0 * sd.dv[5];
          r1[0] = a1 * g[0]; r1[1] = a1 * g[1]; r1[2] = -s1 * sd.idt + a1 * g[2];
          r1[3] = -s1 * sd.w * sd.idt; r1[4] = 0; r1[5] = 0; r1[6] = s1 * sd.idt;
          if (fa) { r0[0] = r0[1] = r0[2] = 0; r1[0] = r1[1] = r1[2] = 0; }
          if (fb) { r0[4] = r0[5] = r0[6] = 0; r1[4] = r1[5] = r1[6] = 0; }
#pragma unroll
          for (int l = 0; l < 7; ++l) {
#pragma unroll
            for (int mm = 0; mm <= l; ++mm) G[(l * (l + 1)) / 2 + mm] += wv * (r0[l] * r0[mm] + r1[l] * r1[mm]);
            gb[l] -= wv * (r0[l] * e0 + r1[l] * e1);
          }
          csum += wv * (e0 * e0 + e1 * e1);
        }
      }
#pragma unroll
      for (int l = 0; l < 7; ++l) {
        const int r = 4 * a + l;
        if (!row_is_real(r, n)) continue; /* fixed rows stay identity (their Gram entries are zero anyway) */
#pragma unroll
        for (int mm = 0; mm <= l; ++mm) H[(size_t)r * HROW + (l - mm)] += G[(l * (l + 1)) / 2 + mm];
        dmax = fmax(dmax, fabs(H[(size_t)r * HROW]));
        H[(size_t)r * HROW + 11] += gb[l];
        rhs[r] += gb[l];
      }
    }
    __syncthreads();
  }
  /* chi2 of these edges belongs to the "other" family (computeCurrentCost does not scale them): chunk 0's partial */
  csum = warp_sum(csum);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = csum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_red[w];
    db.chi_parts[(size_t)b * db.chunks * 4 + 3] += t;
  }
  __syncthreads();
  /* the diagonal grew: keep the band's max diagonal (LM lambda init) up to date */
  dmax = warp_max(dmax);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = dmax;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = db.dmax_parts[(size_t)b * db.chunks];
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t = fmax(t, s_red[w]);
    db.dmax_parts[(size_t)b * db.chunks] = t;
  }
}

/* ------------------------------------------------------------------ k_cost_only (thread per band):
 * computeCurrentCost on a freshly built graph (optimal_planner.cpp:1045-1051): chi2 at the current state from the
 * kernel-A tile partials, with the selection scales. */
__global__ void k_cost_only(DevBatch db, KParams kp, TebOptimizeArgs args) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= db.B) return;
  const BandState st = db.state[b];
  double cost = __longlong_as_double(0x7ff0000000000000LL);
  double chi = 0;
  if (!st.failed) {
    const int n = db.n[b];
    const int chunks_used = (n + db.tile - 1) / db.tile;
    const double* cp = db.chi_parts + (size_t)b * db.chunks * 4;
    double parts[4] = {0, 0, 0, 0};
    for (int c = 0; c < chunks_used; ++c)
      for (int k = 0; k < 4; ++k) parts[k] += cp[4 * c + k];
    chi = parts[0] + parts[1] + parts[2] + parts[3];
    cost = 0;
    if (args.alternative_time_cost) {
      const double* P = db.poses + (size_t)b * db.n_cap * 4;
      for (int i = 0; i < n - 1; ++i) cost += P[4 * i + 3];
    }
    cost += args.obst_cost_scale * parts[0] + args.viapoint_cost_scale * parts[1] + parts[3];
    if (!args.alternative_time_cost) cost += parts[2];
  }
  if (db.cost) db.cost[b] = cost;
  if (db.chi2) db.chi2[b] = chi;
  if (db.status) db.status[b] = st.status;
  if (db.lm_iters) db.lm_iters[b] = 0;
}

}  // namespace tebgpu
