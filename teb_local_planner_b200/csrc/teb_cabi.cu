/*
 * teb_cabi.cu — C-ABI (include/teb_b200.h) over the sm_90a kernels in teb_kernels.cuh.
 * No CPU fallback: every entry point that optimises needs a CUDA device and fails loudly otherwise.
 */
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "teb_kernels.cuh"
#include "teb_linearize.cuh"
#include "teb_spec.cuh"
#include "teb_solve_warp.cuh"
#include "teb_solve_lat.cuh"
#include "teb_hsig.cuh"
#include "teb_hsig_scene.cuh"
#include "teb_plan.cuh"
#include "teb_feasible.cuh"
#include "teb_costmap.cuh"
#include "teb_local_plan.cuh"
#include "teb_cycle.cuh"
#include "teb_fleet.cuh"
#include "teb_comm.h"
#include <cstdlib>

using namespace tebgpu;

struct tebgpu_ctx {
  int device = 0;
  int sms = 0;                        /* multiprocessors of the device: sizes the latency / throughput regimes below */
  cudaStream_t stream = nullptr;
  cudaStream_t side = nullptr;        /* retry rounds of the speculative solver, overlapped with the next kernel A */
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_s0 = nullptr;
  double* Lf2 = nullptr;              /* scratch of the side stream's solver launches (they overlap the main stream's) */
  double* dx2 = nullptr;
  int split = 1;                      /* throughput regime: the side stream also runs round 0 for its bands (TEBGPU_SPLIT) */
  int overlap = 2;                    /* retry rounds on the side stream: 0 never (one stream), 1 always, 2 (default) only in the
                                         latency regime - at 8192 bands the retry rounds move as many factor bytes as round 0,
                                         so the machine is resource bound either way (TEBGPU_OVERLAP) */
  int32_t* defer = nullptr;           /* [B] */
  double* d_fp = nullptr;             /* footprint definition for the vertex-list distance path (FP_DOUBLES) */
  double* d_pverts = nullptr;         /* [S][max_obst_vertices][2] mirror of TebBatch.obst_vertices */
  double* d_hsig = nullptr;           /* [max_bands][max(min(max_obstacles, 1024), 2)] H-signature output of the host-buffer entry point */
  TebGpuLimits lim{};
  TebParams params{};
  bool have_params = false;
  std::string err;
  int64_t launches = 0;
  int linearize_variant = 0;  /* 0: k_linearize2, one thread per pose, 125-pose tiles (default);
                                 1: k_linearize, first generation: 128-thread CTA per 32-pose tile, thread per band row */
  ncclComm_t comm = nullptr;          /* cost all-gather across the ranks of a sharded batch (tebgpu_comm_init) */
  int world = 1, rank = 0;
  int32_t* arrive = nullptr;          /* [max_bands] k_trial_eval3: CTAs of a band that have published their trial (0 between rounds) */
  int eval_mode = 2;                  /* 2 automatic (k_trial_eval3 in the latency regime), 0 k_trial_eval2 always, 1 k_trial_eval3 always (TEBGPU_EVAL3) */
  double* d_gather = nullptr;         /* [world][max_bands] gathered costs of the host-buffer entry point */
  struct GraphEntry { uint64_t key = 0; cudaGraphExec_t exec = nullptr; int64_t launches = 0; uint64_t stamp = 0; int spec_k = 0, spec_first = 0; };
  std::vector<GraphEntry> graphs;     /* captured launch sequences (tebgpu_set_graph) */
  uint64_t graph_clock = 0;
  uint64_t params_version = 0;        /* bumped by tebgpu_set_params: part of the graph key */
  int graph_mode = 2;                 /* 0 never, 1 always, 2 automatic (latency regime only) */
  int warp_solver = 4; /* solver 2, solve kernel (TEBGPU_WARP_SOLVER / tebgpu_set_warp_solver):
                          0 thread per system (k_solve_tpb) always,
                          1 / 2 k_solve_warp always / in the latency regime - slower per solve than k_solve_tpb,
                            kept as an independently mapped, bit-identical implementation,
                          3 / 4 k_solve_lat (twisted factorisation, system resident in shared memory) always / while the
                            systems of a round fit LAT_WAVES waves of resident CTAs (the latency regime; DEFAULT) */
  int solve_form = 0;  /* k_solve_tpb's factor (TEBGPU_SOLVE_FORM / tebgpu_set_solve_form): 0 automatic (tpb_form),
                          1 streamed through HBM, 11 / 22 / 33 recomputed in segments of that many rows */
  int eval_v1 = 0;     /* TEBGPU_EVAL_V1=1: first-generation trial evaluation (warp per trial, chunk per lane) */
  int ka_staged = 1;   /* kernel A output: 1 (default) shared-memory slot + TMA bulk store per lane, 0 direct 128-bit global stores */
  int ka_persist = 1;  /* kernel A with the staged output: 1 (default) persistent k_linearize2p, 0 one-shot k_linearize2 (TEBGPU_KA_PERSIST) */
  int last_ka_build = -1;      /* the last kernel-A launch this context issued: its build (TEBGPU_KA_BUILD_*) */
  long long last_ka_grid = 0;  /* ... and its grid in CTAs */
  int last_spec_k = 0; /* round-0 width of the later LM iterations of the last optimize call */
  int last_spec_first = 0; /* round-0 width of the first LM iteration after a graph rebuild */
  int last_eval_build = -1;      /* the last trial-evaluation launch this context issued: its build (TEBGPU_EVAL_BUILD_*) */
  long long last_eval_grid = 0;  /* ... and its grid in CTAs */
  int spec_k = 0;  /* speculation width: 0 = auto (6 when B*6 systems fit one warp per SM sub-partition, else 4) */
  int solver = 2;  /* 2: speculative thread-per-(band,trial) LDL^T (default), 1: block cyclic reduction, 0: sequential */
  int MW = 1;
  int chunks = 1;
  /* device workspaces */
  double* Hb = nullptr;
  unsigned long long* assoc = nullptr;
  unsigned long long* assoc3 = nullptr;
  unsigned long long* occ = nullptr;  /* [max_bands][max_poses][ceil(MW / 64)] occupancy words (global-table path) */
  double* dyn_t = nullptr;
  int32_t* via_idx = nullptr;
  double* chi_parts = nullptr;
  double* dmax_parts = nullptr;
  double* rhs = nullptr;
  int32_t* dyn_idx = nullptr;
  int32_t* dyn_cnt = nullptr;
  SpecBufs spec{};
  int eval_minb = 3; /* k_trial_eval register budget: 3 -> 6 CTAs/SM at the price of some spills, 2 -> 4 CTAs/SM without;
                        TEBGPU_EVAL_MINB=2 selects the other build */
  BandState* state = nullptr;
  /* device mirrors for the host-buffer entry point */
  double* d_poses = nullptr; int32_t* d_n = nullptr; int32_t* d_scene = nullptr; TebObstacle* d_obst = nullptr;
  int32_t* d_ocount = nullptr; double* d_via = nullptr; int32_t* d_vcount = nullptr; double* d_vs = nullptr;
  double* d_vg = nullptr; int32_t* d_rot = nullptr; double* d_cost = nullptr; double* d_chi2 = nullptr;
  int32_t* d_status = nullptr; int32_t* d_iters = nullptr;
  /* plan entry points: k_plan_begin's per-band status for k_begin, and the host-buffer entry point's mirrors */
  int32_t* plan_status = nullptr;     /* [max_bands] */
  double* d_start = nullptr; double* d_goal = nullptr; int32_t* d_pcount = nullptr; double* d_cmd = nullptr;
  int32_t* d_path = nullptr;
  double* d_plan = nullptr;           /* [max_bands][plan_rows][3], grown to the largest P_cap tebgpu_plan_batch has seen */
  size_t plan_rows = 0;
  /* feasibility check: the host-buffer entry point's output mirrors, allocated by the first call that needs them */
  int32_t* d_feas = nullptr; int32_t* d_qcount = nullptr;
  double* d_queries = nullptr;        /* [max_bands][feas_rows][3] */
  size_t feas_rows = 0;
  bool feas_ready = false;            /* k_feasible's shared-memory attributes set */
  int last_feas_build = -1;           /* the last k_feasible launch: its build (TEBGPU_FEAS_BUILD_*) */
  long long last_feas_grid = 0;       /* ... and its grid in CTAs */
  double* d_qcost = nullptr;          /* the costmap check's query_cost mirror, grown by the first call that needs more */
  size_t qcost_bytes = 0;
  /* trajectory read-out: the host-buffer entry point's band list and output mirrors, grown by the first call that needs more */
  int32_t* d_tbands = nullptr; int32_t* d_tpoints = nullptr; double* d_tprof = nullptr; double* d_ttraj = nullptr;
  size_t tbands_bytes = 0, tpoints_bytes = 0, tprof_bytes = 0, ttraj_bytes = 0;
  long long last_traj_grid = 0;       /* grid in CTAs of the last k_read_trajectory launch */
  /* costmap conversion: the host-buffer entry point's input and output mirrors, grown by the first call that needs more */
  uint8_t* d_ccost = nullptr; int32_t* d_cgrid = nullptr; double* d_corigin = nullptr; double* d_crobot = nullptr;
  TebObstacle* d_ccustom = nullptr; int32_t* d_ccount = nullptr; TebObstacle* d_cobst = nullptr; int32_t* d_cocount = nullptr;
  int32_t* d_cneeded = nullptr;
  char* d_cframe = nullptr; size_t cframe_bytes = 0; /* tebgpu_costmap_obstacles_tf: transforms and vertex pools */
  size_t ccost_bytes = 0, cgrid_bytes = 0, corigin_bytes = 0, crobot_bytes = 0, ccustom_bytes = 0, ccount_bytes = 0,
         cobst_bytes = 0, cocount_bytes = 0, cneeded_bytes = 0;
  long long last_costmap_grid = 0;    /* grid in CTAs of the last k_costmap_obstacles launch */
  /* local plan: the host-buffer entry point's inputs and outputs, staged in one buffer grown by the first call that
   * needs more */
  char* d_lplan = nullptr; size_t lplan_bytes = 0;
  long long last_lplan_grid = 0;      /* grid in CTAs of the last k_local_plan launch */
  /* backup modes / finish cycle: the host-buffer entry points' arrays, staged in one buffer grown as above */
  char* d_cycle = nullptr; size_t cycle_bytes = 0;
  long long last_cycle_grid = 0;      /* grid in CTAs of the last k_backup_modes / k_finish_cycle launch */
  /* fleet obstacles: the robots per scene of the shared-scene check, and the host-buffer entry point's arrays, staged in
   * one buffer; each grown by the first call that needs more */
  int32_t* d_fclaim = nullptr; size_t fclaim_bytes = 0;
  char* d_fleet = nullptr; size_t fleet_bytes = 0;
  TebFleetRow* d_ftable = nullptr; size_t ftable_bytes = 0;   /* the host-buffer table entry points' table */
  long long last_fleet_grid = 0;      /* grid in CTAs of the last k_fleet_obstacles(_grid) launch */
  int fleet_search = TEBGPU_FLEET_SEARCH_AUTO; /* tebgpu_set_fleet_search */
  int last_fleet_search = -1;         /* the search the last fleet step ran (TEBGPU_FLEET_SEARCH_*), -1 before the first */
  /* the fleet grid: bucket counts and starts, candidate keys, ranks and indices, the far list and the scan's
   * temporary storage, in one buffer grown by the first call that needs more */
  char* d_fgrid = nullptr; size_t fgrid_bytes = 0;
  /* scene H-signatures: the factor table's partial products, the in-call / uploaded factor table, the bands' chunk sums
   * and the host-buffer entry point's output, each grown by the first call that needs more */
  char* d_hsf_part = nullptr; char* d_hsf_tab = nullptr; double* d_hs_part = nullptr; double* d_hs_out = nullptr;
  size_t hsf_part_bytes = 0, hsf_tab_bytes = 0, hs_part_bytes = 0, hs_out_bytes = 0;
  size_t smem_a = 0, smem_b = 0, smem_g = 0;
  /* profiling */
  bool profiling = false;
  std::vector<cudaEvent_t> ev;      /* pairs */
  std::vector<int> ev_kind;
  size_t ev_used = 0;
  double prof_ms[11] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; /* 9 k_plan_begin, 10 k_velocity_command */
  int64_t prof_cnt[11] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
};

static void prof_begin(tebgpu_ctx* c, cudaStream_t st, int kind) {
  if (!c->profiling) return;
  if (c->ev_used + 2 > c->ev.size()) {
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    c->ev.push_back(a);
    c->ev.push_back(b);
    c->ev_kind.push_back(kind);
  }
  c->ev_kind[c->ev_used / 2] = kind;
  cudaEventRecord(c->ev[c->ev_used], st);
}
static void prof_end(tebgpu_ctx* c, cudaStream_t st) {
  if (!c->profiling) return;
  cudaEventRecord(c->ev[c->ev_used + 1], st);
  c->ev_used += 2;
}
static void prof_collect(tebgpu_ctx* c) {
  for (size_t k = 0; k + 1 < c->ev_used + 1 && k < c->ev_used; k += 2) {
    float ms = 0;
    cudaEventSynchronize(c->ev[k + 1]);
    cudaEventElapsedTime(&ms, c->ev[k], c->ev[k + 1]);
    c->prof_ms[c->ev_kind[k / 2]] += ms;
    c->prof_cnt[c->ev_kind[k / 2]] += 1;
  }
  c->ev_used = 0;
}

#define CUDA_TRY(ctx, expr)                                                                      \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      (ctx)->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                           \
      return TEBGPU_ERR_CUDA;                                                                    \
    }                                                                                            \
  } while (0)

extern "C" {

void tebgpu_default_params(TebParams* p) {
  /* TebConfig::TebConfig() teb_config.h:245-390 */
  std::memset(p, 0, sizeof(*p));
  p->dt_ref = 0.3; p->dt_hysteresis = 0.1;
  p->force_reinit_new_goal_dist = 1; p->force_reinit_new_goal_angular = 0.5 * M_PI;
  p->teb_autosize = 1; p->min_samples = 3; p->max_samples = 500; p->exact_arc_length = 0;
  p->via_points_ordered = 0; p->allow_init_with_backwards_motion = 0; p->global_plan_overwrite_orientation = 1;
  p->max_vel_x = 0.4; p->max_vel_x_backwards = 0.2; p->max_vel_y = 0.0; p->max_vel_trans = 0.0; p->max_vel_theta = 0.3;
  p->acc_lim_x = 0.5; p->acc_lim_y = 0.5; p->acc_lim_theta = 0.5; p->min_turning_radius = 0;
  p->footprint_type = TEB_FOOTPRINT_POINT;
  p->min_obstacle_dist = 0.5; p->inflation_dist = 0.6; p->dynamic_obstacle_inflation_dist = 0.6;
  p->obstacle_association_force_inclusion_factor = 1.5; p->obstacle_association_cutoff_factor = 5;
  p->obstacle_proximity_ratio_max_vel = 1; p->obstacle_proximity_lower_bound = 0; p->obstacle_proximity_upper_bound = 0.5;
  p->include_dynamic_obstacles = 1; p->legacy_obstacle_association = 0; p->obstacle_poses_affected = 25;
  p->penalty_epsilon = 0.05;
  p->weight_max_vel_x = 2; p->weight_max_vel_y = 2; p->weight_max_vel_theta = 1;
  p->weight_acc_lim_x = 1; p->weight_acc_lim_y = 1; p->weight_acc_lim_theta = 1;
  p->weight_kinematics_nh = 1000; p->weight_kinematics_forward_drive = 1; p->weight_kinematics_turning_radius = 1;
  p->weight_optimaltime = 1; p->weight_shortest_path = 0;
  p->weight_obstacle = 50; p->weight_inflation = 0.1;
  p->weight_dynamic_obstacle = 50; p->weight_dynamic_obstacle_inflation = 0.1;
  p->weight_velocity_obstacle_ratio = 0; p->weight_viapoint = 1; p->weight_prefer_rotdir = 50;
  p->weight_adapt_factor = 2.0; p->obstacle_cost_exponent = 1.0;
  p->no_inner_iterations = 5; p->no_outer_iterations = 4; p->optimization_activate = 1;
  p->selection_cost_hysteresis = 1.0; p->selection_prefer_initial_plan = 0.95;
  p->selection_obst_cost_scale = 100.0; p->selection_viapoint_cost_scale = 1.0;
  p->selection_alternative_time_cost = 0; p->enable_multithreading = 1;
  p->h_signature_prescaler = 1; p->h_signature_threshold = 0.1;
  p->divergence_detection_enable = 0; p->divergence_detection_max_chi_squared = 10;
}

int32_t tebgpu_sizeof(int32_t which) {
  switch (which) {
    case 0: return (int32_t)sizeof(TebParams);
    case 1: return (int32_t)sizeof(TebObstacle);
    case 2: return (int32_t)sizeof(TebBatch);
    case 3: return (int32_t)sizeof(TebOptimizeArgs);
    case 4: return (int32_t)sizeof(TebGpuLimits);
    case 5: return (int32_t)sizeof(TebPlanInput);
    case 6: return (int32_t)sizeof(TebFeasibilityArgs);
    case 7: return (int32_t)sizeof(TebTrajectoryArgs);
    case 8: return (int32_t)sizeof(TebCostmapArgs);
    case 9: return (int32_t)sizeof(TebLocalPlanArgs);
    case 10: return (int32_t)sizeof(TebCycleArgs);
    case 11: return (int32_t)sizeof(TebCostmapWorld);
    case 12: return (int32_t)sizeof(TebFrameArgs);
    case 13: return (int32_t)sizeof(TebHsigFactors);
    case 14: return (int32_t)sizeof(TebFleetArgs);
    case 15: return (int32_t)sizeof(TebFleetRow);
    case 16: return (int32_t)sizeof(TebFleetTable);
    default: return -1;
  }
}

const char* tebgpu_last_error_string(const tebgpu_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int64_t tebgpu_last_launch_count(const tebgpu_ctx* ctx) { return ctx ? ctx->launches : 0; }
int64_t tebgpu_get_info(const tebgpu_ctx* ctx, int32_t which) {
  if (!ctx) return -1;
  switch (which) {
    case 0: return ctx->last_spec_k;
    case 1: return ctx->linearize_variant;
    case 2: return ctx->solver;
    case 3: return ctx->world;
    case 4: return ctx->rank;
    case 5: return ctx->graph_mode;
    case 6: return (int64_t)ctx->graphs.size();
    case 7: return ctx->last_spec_first;
    case 8: return ctx->last_eval_grid;
    case 9: return ctx->last_eval_build;
    case 10: return ctx->last_ka_grid;
    case 11: return ctx->last_ka_build;
    case 12: return ctx->last_feas_grid;
    case 13: return ctx->last_feas_build;
    case 14: return ctx->last_traj_grid;
    case 15: return ctx->last_costmap_grid;
    case 16: return ctx->last_lplan_grid;
    case 17: return ctx->last_cycle_grid;
    case 18: return ctx->last_fleet_grid;
    case 19: return ctx->last_fleet_search;
    default: return -1;
  }
}

static void free_all(tebgpu_ctx* c) {
  void* ptrs[] = {c->Lf2, c->dx2, c->arrive, c->d_gather, c->d_hsig, c->assoc3, c->occ, c->dyn_idx, c->dyn_cnt, c->rhs, c->dmax_parts, c->spec.Lf, c->spec.dx, c->spec.res, c->spec.need, c->spec.qmax, c->spec.cnt, c->spec.list, c->defer, c->d_fp, c->d_pverts, c->Hb, c->assoc, c->dyn_t, c->via_idx, c->chi_parts, c->state, c->d_poses, c->d_n, c->d_scene,
                  c->d_obst, c->d_ocount, c->d_via, c->d_vcount, c->d_vs, c->d_vg, c->d_rot, c->d_cost, c->d_chi2,
                  c->d_status, c->d_iters, c->plan_status, c->d_start, c->d_goal, c->d_pcount, c->d_cmd, c->d_path,
                  c->d_plan, c->d_feas, c->d_qcount, c->d_queries, c->d_tbands, c->d_tpoints, c->d_tprof, c->d_ttraj,
                  c->d_ccost, c->d_cgrid, c->d_corigin, c->d_crobot, c->d_ccustom, c->d_ccount, c->d_cobst, c->d_cocount,
                  c->d_cneeded, c->d_lplan, c->d_cycle, c->d_qcost, c->d_cframe, c->d_hsf_part, c->d_hsf_tab,
                  c->d_hs_part, c->d_hs_out, c->d_fclaim, c->d_fleet, c->d_ftable, c->d_fgrid};
  for (void* p : ptrs)
    if (p) cudaFree(p);
}

int32_t tebgpu_create(const TebGpuLimits* lim, int32_t device, tebgpu_ctx** out) {
  if (!lim || !out) return TEBGPU_ERR_INVALID_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= device || device < 0) {
    std::fprintf(stderr, "tebgpu_create: no CUDA device %d available (this library has no CPU fallback)\n", device);
    return TEBGPU_ERR_NO_DEVICE;
  }
  if (lim->max_bands < 1 || lim->max_poses < 3 || lim->max_poses > 512 || lim->max_scenes < 1 || lim->max_obstacles < 0 ||
      lim->max_obstacles > 64 * GT_MAX_MW || lim->max_viapoints < 0 || lim->max_obst_vertices < 0)
    return TEBGPU_ERR_INVALID_ARG;
  tebgpu_ctx* c = new (std::nothrow) tebgpu_ctx();
  if (!c) return TEBGPU_ERR_CUDA;
  c->device = device;
  c->lim = *lim;
  if (c->lim.max_obstacles < 1) c->lim.max_obstacles = 1;
  c->MW = (c->lim.max_obstacles + 63) / 64;
  c->chunks = (c->lim.max_poses + KA2_TP - 1) / KA2_TP; /* capacity for the smaller of the two tile sizes */
  *out = c;
  CUDA_TRY(c, cudaSetDevice(device));
  CUDA_TRY(c, cudaDeviceGetAttribute(&c->sms, cudaDevAttrMultiProcessorCount, device));
  CUDA_TRY(c, cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  {
    int lo = 0, hi = 0; /* the latency-bound retry chain should never queue behind the bulk kernels */
    CUDA_TRY(c, cudaDeviceGetStreamPriorityRange(&lo, &hi));
    CUDA_TRY(c, cudaStreamCreateWithPriority(&c->side, cudaStreamNonBlocking, hi));
  }
  CUDA_TRY(c, cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
  CUDA_TRY(c, cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
  CUDA_TRY(c, cudaEventCreateWithFlags(&c->ev_s0, cudaEventDisableTiming));
  if (const char* e = std::getenv("TEBGPU_OVERLAP")) { const int m = std::atoi(e); if (m >= 0 && m <= 2) c->overlap = m; }
  if (const char* e = std::getenv("TEBGPU_SPEC_K")) { const int k = std::atoi(e); if (k == 2 || k == 4 || k == 6 || k == 8) c->spec_k = k; }
  const size_t B = c->lim.max_bands, nc = c->lim.max_poses, S = c->lim.max_scenes, M = c->lim.max_obstacles,
               V = c->lim.max_viapoints > 0 ? c->lim.max_viapoints : 1;
  /* the staged kernels (whole table in shared memory) only ever see batches of M_cap <= 1024: larger batches take the
   * global-table instantiations, whose shared memory does not depend on M_cap */
  const size_t Ms = M < (size_t)STAGED_MAX_OBST ? M : (size_t)STAGED_MAX_OBST;
  CUDA_TRY(c, cudaMalloc(&c->Hb, B * 4 * nc * HROW * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->assoc, B * nc * c->MW * sizeof(unsigned long long)));
  CUDA_TRY(c, cudaMalloc(&c->assoc3, B * nc * c->MW * sizeof(unsigned long long)));
  CUDA_TRY(c, cudaMalloc(&c->occ, B * nc * ((c->MW + 63) / 64) * sizeof(unsigned long long)));
  CUDA_TRY(c, cudaMalloc(&c->dyn_t, B * nc * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->via_idx, B * V * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->chi_parts, B * c->chunks * 4 * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->state, B * sizeof(BandState)));
  CUDA_TRY(c, cudaMalloc(&c->dmax_parts, B * c->chunks * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->rhs, B * 4 * nc * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->dyn_idx, S * M * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->dyn_cnt, S * sizeof(int32_t)));
  {
    size_t ev = eval_smem_bytes((int)nc, (int)Ms, SPEC_K_MAX);
    if (ev > 232448) ev = 232448; /* wide speculation is only chosen when its staging fits (tebgpu_optimize_batch_device) */
    CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ev));
    CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ev));
    CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval<3, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ev));
    if (const char* e = std::getenv("TEBGPU_EVAL3")) { const int m = std::atoi(e); if (m >= 0 && m <= 2) c->eval_mode = m; }
    if (const char* e = std::getenv("TEBGPU_EVAL_MINB")) c->eval_minb = std::atoi(e) == 3 ? 3 : 2;
    if (const char* e = std::getenv("TEBGPU_EVAL_V1")) c->eval_v1 = std::atoi(e) != 0;
    size_t ev2 = eval2_smem_bytes((int)nc, (int)Ms, SPEC_K_MAX);
    if (ev2 > 232448) ev2 = 232448;
#define EV2_ATTR(G)                                                                                                  \
  CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval2<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ev2));          \
  CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval2<G>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    EV2_ATTR(false) EV2_ATTR(true)
    size_t ev2g = eval2_smem_bytes((int)nc, 0, SPEC_K_MAX);
    if (ev2g > 232448) ev2g = 232448;
#define EV2G_ATTR(G)                                                                                                 \
  CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval2<G, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ev2g));   \
  CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval2<G, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    EV2G_ATTR(false) EV2G_ATTR(true)
#undef EV2G_ATTR
#undef EV2_ATTR
    /* the persistent build: the same shared memory as k_trial_eval2 */
#define EVP_ATTR(G, T, BYTES)                                                                                           \
  CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval2p<G, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BYTES)));      \
  CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval2p<G, T>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    EVP_ATTR(false, false, ev2) EVP_ATTR(true, false, ev2) EVP_ATTR(false, true, ev2g) EVP_ATTR(true, true, ev2g)
#undef EVP_ATTR
    size_t ev3 = eval3_smem_bytes((int)nc, (int)Ms, SPEC_K_MAX);
    if (ev3 > 232448) ev3 = 232448;
    CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval3<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ev3));
    CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval3<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ev3));
    size_t ev3g = eval3_smem_bytes((int)nc, 0, SPEC_K_MAX);
    if (ev3g > 232448) ev3g = 232448;
    CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval3<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ev3g));
    CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval3<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ev3g));
  }
  const size_t spec_sys = ((B * SPEC_K_MAX + 31) / 32) * 32; /* whole warps of (band, trial) systems */
  CUDA_TRY(c, cudaMalloc(&c->spec.Lf, spec_sys * 4 * nc * HROW * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->spec.dx, spec_sys * 4 * nc * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->Lf2, spec_sys * 4 * nc * HROW * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->dx2, spec_sys * 4 * nc * sizeof(double)));
  c->spec.sel_list = nullptr; c->spec.sel_cnt = nullptr; c->spec.defer = nullptr; c->spec.skip_tag = 0; c->spec.lat_cap = 0;
  if (const char* e = std::getenv("TEBGPU_SPLIT")) c->split = std::atoi(e) != 0;
  CUDA_TRY(c, cudaMalloc(&c->spec.cnt, SPEC_CNT_CAP * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->spec.list, SPEC_LISTS * B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->defer, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->spec.res, B * SPEC_K_MAX * RES_STRIDE * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->arrive, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMemset(c->arrive, 0, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->spec.need, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->spec.qmax, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->d_poses, B * nc * 4 * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_n, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->d_scene, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->d_obst, S * M * sizeof(TebObstacle)));
  CUDA_TRY(c, cudaMalloc(&c->d_ocount, S * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->d_via, B * V * 2 * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_fp, FP_DOUBLES * sizeof(double)));
  CUDA_TRY(c, cudaMemset(c->d_fp, 0, FP_DOUBLES * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_pverts, (S * (size_t)(lim->max_obst_vertices > 0 ? lim->max_obst_vertices : 1)) * 2 * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_hsig, B * (Ms > 2 ? Ms : 2) * sizeof(double))); /* tebgpu_h_signature: M_cap <= 1024 */
  CUDA_TRY(c, cudaMalloc(&c->d_vcount, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->plan_status, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->d_start, B * 3 * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_goal, B * 3 * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_pcount, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->d_cmd, B * 4 * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_path, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->d_vs, B * 4 * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_vg, B * 4 * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_rot, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->d_cost, B * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_chi2, B * sizeof(double)));
  CUDA_TRY(c, cudaMalloc(&c->d_status, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMalloc(&c->d_iters, B * sizeof(int32_t)));
  CUDA_TRY(c, cudaMemsetAsync(c->dyn_t, 0, B * nc * sizeof(double), c->stream));
  CUDA_TRY(c, cudaMemsetAsync(c->via_idx, 0xff, B * V * sizeof(int32_t), c->stream));
  c->smem_a = ka_smem_bytes((int)Ms);
  c->smem_b = kb_smem_bytes((int)nc, (int)Ms);
  c->smem_g = Ms * sizeof(TebObstacle);
  if (c->smem_b > 232448 || c->smem_a > 232448) {
    if (M <= (size_t)STAGED_MAX_OBST) {
      c->err = "shared-memory footprint exceeds 227 KB for these limits (max_poses / max_obstacles too large)";
      return TEBGPU_ERR_CAPACITY;
    }
    /* a large-scene context: the default path never needs these; solvers 0 / 1 and kernel-A variant 1 take only the
     * staged batches that fit (check_path) */
    auto cap = [c](size_t& bytes, const void* f) -> int32_t { /* what is left beside the static shared memory */
      cudaFuncAttributes fa{};
      CUDA_TRY(c, cudaFuncGetAttributes(&fa, f));
      if (bytes > 232448 - fa.sharedSizeBytes) bytes = 232448 - fa.sharedSizeBytes;
      return TEBGPU_OK;
    };
    const void* ka[] = {(const void*)k_linearize<false, false>, (const void*)k_linearize<false, true>,
                        (const void*)k_linearize<true, false>, (const void*)k_linearize<true, true>};
    const void* kb[] = {(const void*)k_lm_step_t<0, KB_THREADS, false>, (const void*)k_lm_step_t<0, KB_THREADS, true>};
    for (const void* f : ka)
      if (int32_t rc = cap(c->smem_a, f)) return rc;
    for (const void* f : kb)
      if (int32_t rc = cap(c->smem_b, f)) return rc;
  }
  if (ka2_smem_bytes<true>((int)Ms) > 232448) {
    c->err = "kernel A staging exceeds 227 KB for these limits (max_obstacles too large)";
    return TEBGPU_ERR_CAPACITY;
  }
#define KA2_ATTR(H, G, O)                                                                                                    \
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize2<H, G, O>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ka2_smem_bytes<H>((int)Ms))); \
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize2<H, G, O>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  KA2_ATTR(false, false, true) KA2_ATTR(false, true, true) KA2_ATTR(true, false, true) KA2_ATTR(true, true, true)
  KA2_ATTR(false, false, false) KA2_ATTR(false, true, false) KA2_ATTR(true, false, false) KA2_ATTR(true, true, false)
#undef KA2_ATTR
#define KA2G_ATTR(H, G)                                                                                                      \
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize2<H, G, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ka2_smem_bytes<H>(0))); \
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize2<H, G, false, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  KA2G_ATTR(false, false) KA2G_ATTR(false, true) KA2G_ATTR(true, false) KA2G_ATTR(true, true)
#undef KA2G_ATTR
#define KA2P_ATTR(H, G, T) \
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize2p<H, G, T>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  KA2P_ATTR(false, false, false) KA2P_ATTR(false, true, false) KA2P_ATTR(true, false, false) KA2P_ATTR(true, true, false)
  KA2P_ATTR(false, false, true) KA2P_ATTR(false, true, true) KA2P_ATTR(true, false, true) KA2P_ATTR(true, true, true)
#undef KA2P_ATTR
  c->ka_staged = 1; /* TMA bulk store per lane: direct 128-bit stores fill only half of each 32-byte sector */
  if (const char* e = std::getenv("TEBGPU_KA_STAGED")) c->ka_staged = std::atoi(e) != 0; /* staged path (M_cap <= 1024) only */
  if (const char* e = std::getenv("TEBGPU_KA_PERSIST")) c->ka_persist = std::atoi(e) != 0;
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_a));
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_a));
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_a));
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_a));
  CUDA_TRY(c, cudaFuncSetAttribute(k_lm_step_t<0, KB_THREADS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_b));
  CUDA_TRY(c, cudaFuncSetAttribute(k_lm_step_t<0, KB_THREADS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_b));
  if ((int)nc <= BCR_MAX_POSES && kb_bcr_smem_bytes((int)nc, (int)Ms) <= 232448) {
    CUDA_TRY(c, cudaFuncSetAttribute(k_lm_step_t<1, KB_BCR_THREADS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)kb_bcr_smem_bytes((int)nc, (int)Ms)));
    CUDA_TRY(c, cudaFuncSetAttribute(k_lm_step_t<1, KB_BCR_THREADS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)kb_bcr_smem_bytes((int)nc, (int)Ms)));
  }
  CUDA_TRY(c, cudaFuncSetAttribute(k_build_graph<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_g));
  CUDA_TRY(c, cudaFuncSetAttribute(k_build_graph<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->smem_g));
  /* ask for the full shared-memory carveout: occupancy of the tile kernels is shared-memory bound */
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize<false, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize<false, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize<true, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_linearize<true, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_solve_tpb, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
#define RC_ATTR(C)                                                                                                         \
  CUDA_TRY(c, cudaFuncSetAttribute(k_solve_tpb_rc<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, tpb_rc_smem_bytes(C, 2))); \
  CUDA_TRY(c, cudaFuncSetAttribute(k_solve_tpb_rc<C>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  RC_ATTR(11) RC_ATTR(22) RC_ATTR(33)
#undef RC_ATTR
  if (const char* e = std::getenv("TEBGPU_SOLVE_FORM")) { const int m = std::atoi(e); if (m == 0 || m == 1 || m == 11 || m == 22 || m == 33) c->solve_form = m; }
  CUDA_TRY(c, cudaFuncSetAttribute(k_solve_lat, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
  if (const char* e = std::getenv("TEBGPU_LAT_TIMING")) { const int v = std::atoi(e); CUDA_TRY(c, cudaMemcpyToSymbol(g_lat_timing, &v, sizeof(int))); }
  if (const char* e = std::getenv("TEBGPU_WARP_SOLVER")) { const int m = std::atoi(e); if (m >= 0 && m <= 4) c->warp_solver = m; }
  if (const char* e = std::getenv("TEBGPU_GRAPH")) { const int m = std::atoi(e); if (m >= 0 && m <= 2) c->graph_mode = m; }
  CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval<2, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval<2, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_trial_eval<3, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_lm_step_t<0, KB_THREADS, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_lm_step_t<0, KB_THREADS, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_lm_step_t<1, KB_BCR_THREADS, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CUDA_TRY(c, cudaFuncSetAttribute(k_lm_step_t<1, KB_BCR_THREADS, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  tebgpu_default_params(&c->params);
  c->have_params = true;
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  return TEBGPU_OK;
}

int32_t tebgpu_destroy(tebgpu_ctx* ctx) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  if (ctx->stream) { cudaStreamSynchronize(ctx->stream); }
  if (ctx->comm) { nccl_api().CommDestroy(ctx->comm); ctx->comm = nullptr; }
  for (auto& e : ctx->graphs) cudaGraphExecDestroy(e.exec);
  ctx->graphs.clear();
  free_all(ctx);
  for (cudaEvent_t e : ctx->ev) cudaEventDestroy(e);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->side) cudaStreamDestroy(ctx->side);
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
  if (ctx->ev_s0) cudaEventDestroy(ctx->ev_s0);
  delete ctx;
  return TEBGPU_OK;
}

int32_t tebgpu_set_params(tebgpu_ctx* ctx, const TebParams* p) {
  if (!ctx || !p) return TEBGPU_ERR_INVALID_ARG;
  if (p->footprint_type < 0 || p->footprint_type > TEB_FOOTPRINT_POLYGON) { ctx->err = "unknown footprint model"; return TEBGPU_ERR_UNSUPPORTED; }
  if (p->footprint_type == TEB_FOOTPRINT_POLYGON &&
      (p->footprint_vertex_count < 1 || p->footprint_vertex_count > TEB_MAX_FOOTPRINT_VERTICES)) {
    ctx->err = "polygon footprint needs 1 .. TEB_MAX_FOOTPRINT_VERTICES vertices";
    return TEBGPU_ERR_INVALID_ARG;
  }
  /* footprint definition for the vertex-list distance path: a small device array, read by generic_distance */
  double fp[FP_DOUBLES];
  std::memset(fp, 0, sizeof(fp));
  fp[FP_RADIUS] = p->footprint_radius;
  fp[FP_FRONT_OFF] = p->footprint_front_offset; fp[FP_FRONT_RAD] = p->footprint_front_radius;
  fp[FP_REAR_OFF] = p->footprint_rear_offset; fp[FP_REAR_RAD] = p->footprint_rear_radius;
  for (int k = 0; k < 4; ++k) fp[FP_LINE + k] = p->footprint_line[k];
  fp[FP_COUNT] = (double)p->footprint_vertex_count;
  for (int k = 0; k < 2 * TEB_MAX_FOOTPRINT_VERTICES; ++k) fp[FP_VERTS + k] = p->footprint_vertices[k];
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream)); /* no optimize call of this context may still read the old copy */
  CUDA_TRY(ctx, cudaMemcpy(ctx->d_fp, fp, sizeof(fp), cudaMemcpyHostToDevice));
  ctx->params = *p;
  ctx->have_params = true;
  ++ctx->params_version;
  return TEBGPU_OK;
}

/* Kernel instantiations: HOLO = holonomic rows (vy, acc y); GEOM = vertex-list shapes (Line / Polygon footprint,
 * Line / Pill / Polygon obstacles) reachable, i.e. the out-of-line generic_distance call is compiled in. The default
 * diff-drive / car-like + Point / Circular configuration runs <false, false>: no extra rows, no call. */
/* Path of a batch: M_cap <= 1024 runs the staged kernels (the scene's obstacle table copied into shared memory),
 * 1025 .. 16384 their global-table instantiations (GT: rows read from global memory / L2, association walked via the
 * occupancy words). Chosen per call; the CUDA-graph key holds M_cap, so it covers the path. */
static bool global_table(int M_cap) { return M_cap > STAGED_MAX_OBST; }

/* the kernels without a global-table instantiation: TEBGPU_ERR_UNSUPPORTED for such a batch */
static int32_t check_path(tebgpu_ctx* ctx, const TebBatch* bt, bool solves) {
  if (!global_table(bt->M_cap)) {
    /* staged batch in a large-scene context whose staged shared-memory attributes had to be capped */
    if ((ctx->linearize_variant == 1 && ka_smem_bytes(bt->M_cap) > ctx->smem_a) ||
        (solves && ctx->solver != 2 && kb_smem_bytes(bt->n_cap, bt->M_cap) > ctx->smem_b)) {
      ctx->err = "shared-memory footprint exceeds 227 KB for this batch (n_cap / M_cap too large)";
      return TEBGPU_ERR_CAPACITY;
    }
    return TEBGPU_OK;
  }
  if (ctx->linearize_variant == 1) { ctx->err = "kernel-A variant 1 supports at most 1024 obstacles per scene"; return TEBGPU_ERR_UNSUPPORTED; }
  if (solves && ctx->solver != 2) { ctx->err = "solvers 0 and 1 support at most 1024 obstacles per scene"; return TEBGPU_ERR_UNSUPPORTED; }
  if (solves && ctx->eval_v1) { ctx->err = "TEBGPU_EVAL_V1 supports at most 1024 obstacles per scene"; return TEBGPU_ERR_UNSUPPORTED; }
  return TEBGPU_OK;
}

static void launch_linearize(tebgpu_ctx* ctx, const DevBatch& db, const KParams& kp, int B, int M_cap, cudaStream_t st) {
  const bool holo = kp.holo_vel || kp.holo_acc;
  const bool geom = kp.generic != 0;
  if (ctx->ka_persist && ctx->linearize_variant == 0 && (ctx->ka_staged || global_table(M_cap))) {
    /* persistent one-warp CTAs, as many as are resident, never more than the launch has units */
    const size_t sm = holo ? ka2p_smem_bytes<true>() : ka2p_smem_bytes<false>();
    auto go = [&](auto kern) {
      int per_sm = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 32, sm) != cudaSuccess || per_sm < 1) per_sm = 1;
      long long grid = (long long)per_sm * ctx->sms;
      if (grid > (long long)B * db.chunks) grid = (long long)B * db.chunks;
      ctx->last_ka_build = TEBGPU_KA_BUILD_PERSIST; ctx->last_ka_grid = grid;
      kern<<<(unsigned)grid, 32, sm, st>>>(db, kp, B);
    };
    const bool gt = global_table(M_cap);
    if (gt && holo && geom) go(k_linearize2p<true, true, true>);
    else if (gt && holo) go(k_linearize2p<true, false, true>);
    else if (gt && geom) go(k_linearize2p<false, true, true>);
    else if (gt) go(k_linearize2p<false, false, true>);
    else if (holo && geom) go(k_linearize2p<true, true, false>);
    else if (holo) go(k_linearize2p<true, false, false>);
    else if (geom) go(k_linearize2p<false, true, false>);
    else go(k_linearize2p<false, false, false>);
    return;
  }
  if (global_table(M_cap)) { /* output through the staged slot, the default form: TEBGPU_KA_STAGED=0 (direct stores,
                                same results) applies to the staged path only */
    const dim3 g2((db.chunks + KA2_W - 1) / KA2_W, B);
    const size_t sm = holo ? ka2_smem_bytes<true>(0) : ka2_smem_bytes<false>(0);
    ctx->last_ka_build = TEBGPU_KA_BUILD_ONESHOT; ctx->last_ka_grid = (long long)g2.x * B;
    if (holo && geom) k_linearize2<true, true, false, true><<<g2, KA2_THREADS, sm, st>>>(db, kp);
    else if (holo) k_linearize2<true, false, false, true><<<g2, KA2_THREADS, sm, st>>>(db, kp);
    else if (geom) k_linearize2<false, true, false, true><<<g2, KA2_THREADS, sm, st>>>(db, kp);
    else k_linearize2<false, false, false, true><<<g2, KA2_THREADS, sm, st>>>(db, kp);
  } else if (ctx->linearize_variant == 1) {
    const dim3 grid(db.chunks, B);
    const size_t sm = ka_smem_bytes(M_cap);
    ctx->last_ka_build = TEBGPU_KA_BUILD_V1; ctx->last_ka_grid = (long long)grid.x * B;
    if (holo && geom) k_linearize<true, true><<<grid, KA_THREADS, sm, st>>>(db, kp);
    else if (holo) k_linearize<true, false><<<grid, KA_THREADS, sm, st>>>(db, kp);
    else if (geom) k_linearize<false, true><<<grid, KA_THREADS, sm, st>>>(db, kp);
    else k_linearize<false, false><<<grid, KA_THREADS, sm, st>>>(db, kp);
  } else {
    const dim3 g2((db.chunks + KA2_W - 1) / KA2_W, B);
    const size_t sm = holo ? ka2_smem_bytes<true>(M_cap) : ka2_smem_bytes<false>(M_cap);
    ctx->last_ka_build = ctx->ka_staged ? TEBGPU_KA_BUILD_ONESHOT : TEBGPU_KA_BUILD_DIRECT; ctx->last_ka_grid = (long long)g2.x * B;
#define KA2_LAUNCH(H, G)                                                                      \
  do {                                                                                        \
    if (ctx->ka_staged) k_linearize2<H, G, false><<<g2, KA2_THREADS, sm, st>>>(db, kp);       \
    else k_linearize2<H, G, true><<<g2, KA2_THREADS, sm, st>>>(db, kp);                       \
  } while (0)
    if (holo && geom) KA2_LAUNCH(true, true);
    else if (holo) KA2_LAUNCH(true, false);
    else if (geom) KA2_LAUNCH(false, true);
    else KA2_LAUNCH(false, false);
#undef KA2_LAUNCH
  }
}
static void launch_build_graph(const DevBatch& db, const KParams& kp, int B, size_t smem, cudaStream_t st) {
  if (global_table(db.M_cap)) {
    if (kp.generic) k_build_graph<true, true><<<B, 256, 0, st>>>(db, kp);
    else k_build_graph<false, true><<<B, 256, 0, st>>>(db, kp);
  } else if (kp.generic) k_build_graph<true><<<B, 256, smem, st>>>(db, kp);
  else k_build_graph<false><<<B, 256, smem, st>>>(db, kp);
}
static void launch_vor(const DevBatch& db, const KParams& kp, int B, size_t smem, cudaStream_t st) {
  if (global_table(db.M_cap)) {
    if (kp.generic) k_vor<true, true><<<B, 256, 0, st>>>(db, kp);
    else k_vor<false, true><<<B, 256, 0, st>>>(db, kp);
  } else if (kp.generic) k_vor<true><<<B, 256, smem, st>>>(db, kp);
  else k_vor<false><<<B, 256, smem, st>>>(db, kp);
}
static size_t eval_bytes(const tebgpu_ctx* ctx, int n_cap, int M_cap, int K) {
  if (global_table(M_cap)) M_cap = 0; /* no copy of the table: the trial width is not limited by M_cap */
  return ctx->eval_v1 ? eval_smem_bytes(n_cap, M_cap, K) : eval2_smem_bytes(n_cap, M_cap, K);
}
static void launch_trial_eval(tebgpu_ctx* ctx, const SpecBufs& spec, const DevBatch& db, const KParams& kp, int B, int K,
                              size_t smem, int it, int round, int g, int tag, cudaStream_t st) {
  /* latency regime: a CTA per (band, trial) instead of a CTA per band while that still fits ~3 CTAs per SM */
  const bool gt = global_table(db.M_cap);
  const size_t smem3 = eval3_smem_bytes(db.n_cap, gt ? 0 : db.M_cap, K);
  if (!ctx->eval_v1 && smem3 <= 232448 && (ctx->eval_mode == 1 || (ctx->eval_mode == 2 && (long long)B * K <= ctx->sms * 3))) {
    int warps = ev2_tiles(db.n_cap);
    warps = warps < 1 ? 1 : (warps > 16 ? 16 : warps);
    const dim3 grid(K, B);
    ctx->last_eval_build = TEBGPU_EVAL_BUILD_EVAL3; ctx->last_eval_grid = (long long)K * B;
    if (gt && kp.generic) k_trial_eval3<true, true><<<grid, 32 * warps, smem3, st>>>(db, kp, spec, it, round, g, tag, ctx->arrive);
    else if (gt) k_trial_eval3<false, true><<<grid, 32 * warps, smem3, st>>>(db, kp, spec, it, round, g, tag, ctx->arrive);
    else if (kp.generic) k_trial_eval3<true><<<grid, 32 * warps, smem3, st>>>(db, kp, spec, it, round, g, tag, ctx->arrive);
    else k_trial_eval3<false><<<grid, 32 * warps, smem3, st>>>(db, kp, spec, it, round, g, tag, ctx->arrive);
    return;
  }
  if (!ctx->eval_v1) { /* second generation: one lane per pose */
    /* one warp per 30-pose tile of the longest band (2 .. 8 warps; 4 .. 16 in the wide variant: two trials side by side),
     * so that the K x tiles warp tasks split evenly and nobody idles at the barrier */
    int warps = ev2_tiles(db.n_cap);
    warps = warps < 2 ? 2 : (warps > 8 ? 8 : warps);
    const bool wide = (long long)B * 2 <= ctx->sms; /* a CTA per band leaves SMs idle: give each band up to 16 warps */
    if (wide || B <= 2 * ctx->sms) {
      /* a CTA per band, compiled for 1 CTA per SM (all registers): right while every CTA is resident anyway */
      if (wide) warps = 2 * warps;
      const int nt = 32 * warps;
      ctx->last_eval_build = wide ? TEBGPU_EVAL_BUILD_EVAL2_WIDE : TEBGPU_EVAL_BUILD_EVAL2; ctx->last_eval_grid = B;
      if (gt && kp.generic) k_trial_eval2<true, true><<<B, nt, smem, st>>>(db, kp, spec, it, round, g, tag);
      else if (gt) k_trial_eval2<false, true><<<B, nt, smem, st>>>(db, kp, spec, it, round, g, tag);
      else if (kp.generic) k_trial_eval2<true><<<B, nt, smem, st>>>(db, kp, spec, it, round, g, tag);
      else k_trial_eval2<false><<<B, nt, smem, st>>>(db, kp, spec, it, round, g, tag);
      return;
    }
    /* throughput regime: the persistent build, as many CTAs as are resident (same shared memory as k_trial_eval2) */
    const int nt = 32 * warps;
    auto go = [&](auto kern) {
      int per_sm = 0;
      if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, nt, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
      ctx->last_eval_build = TEBGPU_EVAL_BUILD_EVAL2P; ctx->last_eval_grid = (long long)per_sm * ctx->sms;
      kern<<<per_sm * ctx->sms, nt, smem, st>>>(db, kp, spec, it, round, g, tag);
    };
    if (gt && kp.generic) go(k_trial_eval2p<true, true>);
    else if (gt) go(k_trial_eval2p<false, true>);
    else if (kp.generic) go(k_trial_eval2p<true, false>);
    else go(k_trial_eval2p<false, false>);
    return;
  }
  ctx->last_eval_build = TEBGPU_EVAL_BUILD_V1; ctx->last_eval_grid = B;
  if (kp.generic) k_trial_eval<2, true><<<B, 32 * K, smem, st>>>(db, kp, spec, it, round, g, tag);
  else if (ctx->eval_minb == 3) k_trial_eval<3, false><<<B, 32 * K, smem, st>>>(db, kp, spec, it, round, g, tag);
  else k_trial_eval<2, false><<<B, 32 * K, smem, st>>>(db, kp, spec, it, round, g, tag);
}

static KParams make_kparams(const tebgpu_ctx* ctx, const TebBatch* bt, double weight_multiplier) {
  const TebParams& p = ctx->params;
  KParams k;
  std::memset(&k, 0, sizeof(k));
  k.p = p;
  k.generic = p.footprint_type >= TEB_FOOTPRINT_LINE || bt->PV_cap > 0;
  k.fp_geom = ctx->d_fp;
  k.w_obst = p.weight_obstacle * weight_multiplier;
  k.sw_vel_x = std::sqrt(p.weight_max_vel_x); k.sw_vel_th = std::sqrt(p.weight_max_vel_theta);
  k.sw_acc_x = std::sqrt(p.weight_acc_lim_x); k.sw_acc_th = std::sqrt(p.weight_acc_lim_theta);
  k.inflated = p.inflation_dist > p.min_obstacle_dist;
  k.carlike = !(p.min_turning_radius == 0 || p.weight_kinematics_turning_radius == 0);
  k.sw_kin_nh = std::sqrt(p.weight_kinematics_nh);
  k.sw_kin_2 = std::sqrt(k.carlike ? p.weight_kinematics_turning_radius : p.weight_kinematics_forward_drive);
  k.sw_sp = std::sqrt(p.weight_shortest_path);
  k.sw_rot = std::sqrt(p.weight_prefer_rotdir);
  /* holonomic edge families: optimal_planner.cpp:722 / :745 (velocity), :778 / :824 (acceleration) */
  k.holo_vel = p.max_vel_y != 0;
  k.holo_acc = p.max_vel_y != 0 && p.acc_lim_y != 0;
  k.sw_vel_y = std::sqrt(p.weight_max_vel_y); k.sw_acc_y = std::sqrt(p.weight_acc_lim_y);
  k.has_vel = k.holo_vel ? !(p.weight_max_vel_x == 0 && p.weight_max_vel_y == 0 && p.weight_max_vel_theta == 0)
                         : !(p.weight_max_vel_x == 0 && p.weight_max_vel_theta == 0);
  k.has_acc = !(p.weight_acc_lim_x == 0 && p.weight_acc_lim_theta == 0); /* weight_acc_lim_y is not consulted (:768) */
  k.has_kin = k.carlike ? !(p.weight_kinematics_nh == 0 && p.weight_kinematics_turning_radius == 0)
                        : !(p.weight_kinematics_nh == 0 && p.weight_kinematics_forward_drive == 0);
  k.has_sp = p.weight_shortest_path != 0;
  k.has_rot = p.weight_prefer_rotdir != 0;
  k.has_time = p.weight_optimaltime != 0;
  k.has_obst = !(p.weight_obstacle == 0 || weight_multiplier == 0);
  k.has_dyn = p.include_dynamic_obstacles && p.weight_obstacle != 0; /* optimal_planner.cpp:342, :648 */
  k.has_via = p.weight_viapoint != 0;
  k.pow_exponent = (p.obstacle_cost_exponent != 1.0 && p.min_obstacle_dist > 0.0);
  /* optimal_planner.cpp:362; with the legacy association obstacles_per_vertex_ stays empty -> no ratio edges */
  k.has_vor = p.weight_velocity_obstacle_ratio > 0 && !p.legacy_obstacle_association;
  return k;
}

static int32_t check_batch(tebgpu_ctx* ctx, const TebBatch* bt) {
  if (!ctx || !bt) return TEBGPU_ERR_INVALID_ARG;
  if (bt->B < 1 || bt->n_cap < 3 || bt->S < 1 || bt->M_cap < 0 || bt->V_cap < 0) { ctx->err = "bad batch dimensions"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->B > ctx->lim.max_bands || bt->n_cap > ctx->lim.max_poses || bt->S > ctx->lim.max_scenes ||
      bt->M_cap > ctx->lim.max_obstacles || bt->V_cap > ctx->lim.max_viapoints) { ctx->err = "batch exceeds the context limits"; return TEBGPU_ERR_CAPACITY; }
  if (!bt->poses || !bt->n || !bt->scene_id || !bt->obst_count || !bt->vel_start || !bt->vel_goal) { ctx->err = "missing required batch array"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->M_cap > 0 && !bt->obstacles) { ctx->err = "obstacles == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->V_cap > 0 && (!bt->via || !bt->via_count)) { ctx->err = "via == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->PV_cap < 0 || bt->PV_cap > ctx->lim.max_obst_vertices) { ctx->err = "PV_cap exceeds max_obst_vertices"; return TEBGPU_ERR_CAPACITY; }
  if (bt->PV_cap > 0 && !bt->obst_vertices) { ctx->err = "obst_vertices == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (!ctx->have_params) { ctx->err = "tebgpu_set_params has not been called"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

static DevBatch make_devbatch(tebgpu_ctx* ctx, const TebBatch* bt) {
  DevBatch d;
  std::memset(&d, 0, sizeof(d));
  d.B = bt->B; d.n_cap = bt->n_cap; d.S = bt->S; d.M_cap = bt->M_cap; d.V_cap = bt->V_cap;
  d.MW = (bt->M_cap + 63) / 64; if (d.MW < 1) d.MW = 1;
  d.poses = bt->poses; d.n = bt->n; d.scene_id = bt->scene_id; d.obstacles = bt->obstacles; d.obst_count = bt->obst_count;
  d.via = bt->via; d.via_count = bt->via_count; d.vel_start = bt->vel_start; d.vel_goal = bt->vel_goal;
  d.prefer_rotdir = bt->prefer_rotdir;
  d.cost = bt->cost; d.chi2 = bt->chi2; d.status = bt->status; d.lm_iters = bt->lm_iters;
  d.Hb = ctx->Hb; d.assoc = ctx->assoc; d.assoc3 = ctx->assoc3; d.dyn_t = ctx->dyn_t; d.via_idx = ctx->via_idx; d.chi_parts = ctx->chi_parts; d.dmax_parts = ctx->dmax_parts; d.rhs = ctx->rhs; d.dyn_idx = ctx->dyn_idx; d.dyn_cnt = ctx->dyn_cnt;
  d.state = ctx->state;
  d.tile = ctx->linearize_variant == 1 ? TP : KA2_TP;
  d.chunks = (bt->n_cap + d.tile - 1) / d.tile;
  d.obst_vertices = bt->PV_cap > 0 ? bt->obst_vertices : nullptr; d.PV_cap = bt->PV_cap;
  d.defer = ctx->defer; d.a_list = nullptr; d.a_cnt = nullptr; d.skip_tag = 0;
  d.occ = ctx->occ; d.OW = (d.MW + 63) / 64;
  return d;
}

/* Form of k_solve_tpb: 0 the factor streamed through HBM (k_solve_tpb), else the segment length C of the recompute form
 * (k_solve_tpb_rc<C>). Automatic: C = 22, the fastest form at every width measured (K = 2, 4, 6; DESIGN §8). The
 * checkpoints of the recompute form must fit the factor scratch of a warp (only very short bands at C = 11 would not). */
constexpr int TPB_RC_AUTO_C = 22;
static int tpb_form(const tebgpu_ctx* ctx, int n_cap) {
  int C = ctx->solve_form;
  if (C == 0) C = TPB_RC_AUTO_C;
  if (C == 1) return 0;
  const long long segs = (4LL * n_cap + C - 1) / C;
  return segs * TPB_RC_CKPT_PAIRS <= 4LL * n_cap * (HROW / 2) ? C : 0;
}

/* The solve launch of one round of the speculative solver (solver 2) over the db.B bands, K trials each, on stream s:
 * the kernel tebgpu_set_warp_solver selects, its grid and shared memory. Shared by issue_optimize and
 * tebgpu_solve_system. lat_cap > 0 (retry rounds, mode 4) forces the dual launch with that many k_solve_lat systems;
 * 0 sizes it automatically. Returns the number of kernels launched. */
static int launch_spec_solve(const tebgpu_ctx* ctx, const DevBatch& db, const SpecBufs& spec, int K, int it, int round, int g,
                             cudaStream_t s, int lat_cap) {
  const int bk = db.B * K;
  const int warps = (bk + 31) / 32;
  /* k_solve_warp: the sequential order spread over a warp (cross-check only) */
  const bool warp_solver = ctx->warp_solver == 1 || (ctx->warp_solver == 2 && bk <= ctx->sms * 8);
  const size_t smem_lat = solve_lat_smem_bytes(db.n_cap);
  /* automatic: while the round's systems fit LAT_WAVES waves of resident CTAs (one warp + its whole system per CTA)
   * the twisted solver's short per-wave chain beats the fixed time a thread-per-system solve takes
   * regardless of the count */
  const long long lat_wave = smem_lat <= 232448 ? (long long)ctx->sms * (232448 / smem_lat > 16 ? 16 : 232448 / smem_lat) : 0;
  const bool dual = round > 0 && ctx->warp_solver == 4 && lat_wave > 0;
  const bool lat_solver = lat_wave > 0 && (ctx->warp_solver == 3 || (ctx->warp_solver == 4 && bk <= LAT_WAVES * lat_wave && lat_cap == 0));
  /* k_solve_tpb in the form tebgpu_set_solve_form selects: the factor streamed through HBM, or recomputed per
   * segment of C rows (k_solve_tpb_rc) */
  auto launch_tpb = [&](const SpecBufs& sb) {
    switch (tpb_form(ctx, db.n_cap)) {
      case 11: k_solve_tpb_rc<11><<<warps, 32, tpb_rc_smem_bytes(11, K), s>>>(db, sb, it, round, g); break;
      case 22: k_solve_tpb_rc<22><<<warps, 32, tpb_rc_smem_bytes(22, K), s>>>(db, sb, it, round, g); break;
      case 33: k_solve_tpb_rc<33><<<warps, 32, tpb_rc_smem_bytes(33, K), s>>>(db, sb, it, round, g); break;
      default: k_solve_tpb<<<warps, 32, TPB_SMEM_BYTES, s>>>(db, sb, it, round, g);
    }
  };
  if (lat_solver) k_solve_lat<<<bk, 32, smem_lat, s>>>(db, spec, it, round, g);
  else if (dual) {
    /* retry round of the throughput regime: both mappings are launched, the list length decides on the device */
    SpecBufs sl = spec;
    long long cap = lat_cap > 0 ? lat_cap : LAT_WAVES * lat_wave;
    cap = cap < bk ? cap : bk;
    sl.lat_cap = (int32_t)cap;
    k_solve_lat<<<(unsigned)cap, 32, smem_lat, s>>>(db, sl, it, round, g);
    launch_tpb(sl);
    return 2;
  }
  else if (warp_solver) k_solve_warp<<<(bk + SW_WARPS - 1) / SW_WARPS, 32 * SW_WARPS, 0, s>>>(db, spec, it, round, g);
  else launch_tpb(spec);
  return 1;
}

/* the launch sequence of one optimizeTEB over the batch, issued on `st` (directly, or into a stream capture);
 * pre_status: k_plan_begin's per-band status (plan entry points), or NULL */
static int32_t issue_optimize(tebgpu_ctx* ctx, const TebBatch* bt, const TebOptimizeArgs* args, cudaStream_t st,
                              const int32_t* pre_status = nullptr) {
  DevBatch db = make_devbatch(ctx, bt);
  db.pre_status = pre_status;
  const TebParams& p = ctx->params;
  const int B = bt->B;
  const int tb = 128, gb = ((B > bt->S ? B : bt->S) + tb - 1) / tb;
  int64_t launches = 0;
  const size_t smem_a = ka_smem_bytes(bt->M_cap);
  const size_t smem_b = kb_smem_bytes(bt->n_cap, bt->M_cap);
  const size_t smem_bcr = kb_bcr_smem_bytes(bt->n_cap, bt->M_cap);
  const bool use_bcr = ctx->solver == 1 && bt->n_cap <= BCR_MAX_POSES && smem_bcr <= 232448 &&
                       ctx->lim.max_poses <= BCR_MAX_POSES;
  const size_t smem_g = (size_t)(bt->M_cap > 0 ? bt->M_cap : 1) * sizeof(TebObstacle); /* staged path only */
  /* speculation width: one solver warp per SM sub-partition is the latency-optimal regime (SMs x 4 x 32 lanes);
   * below it the wider speculation is free and removes the second round, above it the factor traffic dominates */
  /* Speculation schedule: widths of the rounds of one LM iteration (they add up to g2o's 10 trials).
   *   fixed width (tebgpu_set_speculation / TEBGPU_SPEC_K): K, K, ... as before;
   *   automatic: the first LM iteration after every graph rebuild restarts at lambda = 1e-5 max diag and needs 4-5
   *   damping escalations on 90 % of the bands, later iterations accept the first trial on 60 % (counted on C2-C4).
   *   Latency regime (all B x 8 systems fit one solver warp per SM sub-partition): {8, 2} -
   *   the retry round practically never runs. Throughput regime: {6, 4} for the first iteration, {2, 4, 4} afterwards
   *   - factor traffic and trial evaluations follow the width. */
  int sched_first[5] = {0, 0, 0, 0, 0}, sched_later[5] = {0, 0, 0, 0, 0};
  int n_first = 0, n_later = 0;
  {
    int kmax = SPEC_K_MAX;
    while (kmax > 2 && eval_bytes(ctx, bt->n_cap, bt->M_cap, kmax) > 232448) kmax -= 2;
    if (eval_bytes(ctx, bt->n_cap, bt->M_cap, kmax) > 232448) { ctx->err = "trial-evaluation staging exceeds shared memory"; return TEBGPU_ERR_CAPACITY; }
    auto fill = [&](int* dst, int& cnt, std::initializer_list<int> want) {
      int left = 10;
      cnt = 0;
      for (int w : want) {
        if (left <= 0) break;
        int k = w < kmax ? w : kmax;
        dst[cnt++] = k;
        left -= k;
      }
      while (left > 0) { dst[cnt++] = kmax < 4 ? kmax : 4; left -= dst[cnt - 1]; }
    };
    if (ctx->spec_k != 0) {
      const int k = ctx->spec_k;
      fill(sched_first, n_first, {k, k, k, k, k});
      fill(sched_later, n_later, {k, k, k, k, k});
    } else if ((long long)B * 8 <= (long long)ctx->sms * 4 * 32) {
      fill(sched_first, n_first, {8, 2});
      fill(sched_later, n_later, {8, 2});
    } else {
      fill(sched_first, n_first, {6, 4});
      fill(sched_later, n_later, {2, 4, 4});
    }
  }
  const int rounds_max = n_first > n_later ? n_first : n_later;
  ctx->last_spec_k = ctx->solver == 2 ? sched_later[0] : 1;
  ctx->last_spec_first = ctx->solver == 2 ? sched_first[0] : 1;
  int g = 0; /* running index of the speculative rounds of this call: selects the retry-list counter / buffer */
  if (ctx->solver == 2) {
    const long long need_cnt = (long long)args->iterations_outerloop * args->iterations_innerloop * rounds_max + 2;
    if (need_cnt > SPEC_CNT_CAP) { ctx->err = "outer x inner iterations exceed the retry-list counters"; return TEBGPU_ERR_CAPACITY; }
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->spec.cnt, 0, (size_t)need_cnt * sizeof(int32_t), st));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->defer, 0, (size_t)B * sizeof(int32_t), st));
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->arrive, 0, (size_t)B * sizeof(int32_t), st)); /* k_trial_eval3's arrival counters: a call that
                                                                                    was cut short must not leak into the next */
  }
  /* Retry rounds (bands that rejected all trials of a round) can run on a side stream, followed by kernel A of the next
   * inner iteration for exactly those bands - and, with TEBGPU_SPLIT, by ROUND 0 of that iteration for them - while the
   * main stream works on all other bands. Bands never share data, so this is only a re-ordering of independent work
   * (bit-identical results, tested). It pays when the retry rounds are nearly empty (fixed K = 4: ~5 % of the bands; the
   * latency regime, where it is the default). With the width schedule {2, 4, 4} of the throughput regime 30-40 % of the
   * bands retry, the retry solves move as many factor bytes as round 0, and the machine is resource bound whichever stream
   * runs them, so one stream is the
   * default there. */
  const bool latency_regime_b = (long long)B * 8 <= (long long)ctx->sms * 4 * 32;
  const bool overlap = ctx->solver == 2 && (ctx->overlap == 1 || (ctx->overlap == 2 && latency_regime_b)) && !ctx->profiling;
  int tag = 0; /* running inner-iteration number (1-based) */
  double weight_multiplier = 1.0;
  KParams kp = make_kparams(ctx, bt, weight_multiplier);
  prof_begin(ctx, st, 0); k_begin<<<gb, tb, 0, st>>>(db, kp); ++launches; prof_end(ctx, st);
  const bool split_ok = overlap && ctx->split && !latency_regime_b;
  bool side_share = false;
  int last_r1 = 0;      /* index g of round 1 of the latest LM iteration: its list = the side stream's bands */
  bool carried = false; /* the side stream already ran autoResize / buildGraph / kernel A of this outer iteration for the
                           bands that were still in a retry round when the previous outer iteration ended */
  /* optimizeGraph returns false when optimize() ran no iteration (optimal_planner.cpp:393), so with no inner iterations
   * optimizeTEB stops after the first outer iteration's autoResize / buildGraph, unoptimised */
  const int outer = args->iterations_innerloop == 0 && args->iterations_outerloop > 1 ? 1 : args->iterations_outerloop;
  for (int o = 0; o < outer; ++o) {
    kp = make_kparams(ctx, bt, weight_multiplier);
    {
      DevBatch dm = db;
      if (carried) dm.skip_tag = tag;
      if (p.teb_autosize) { prof_begin(ctx, st, 1); k_auto_resize<<<gb, tb, 0, st>>>(dm, kp); ++launches; prof_end(ctx, st); }
      prof_begin(ctx, st, 2); launch_build_graph(dm, kp, B, smem_g, st); ++launches; prof_end(ctx, st);
    }
    bool deferred_done = carried; /* kernel A of this iteration already ran for the deferred bands (side stream) */
    carried = false;
    for (int it = 0; it < args->iterations_innerloop; ++it) {
      ++tag;
      {
        DevBatch da = db;
        if (deferred_done) da.skip_tag = tag - 1; /* bands queued during the previous iteration were linearised on the side stream */
        prof_begin(ctx, st, 3); launch_linearize(ctx, da, kp, B, bt->M_cap, st); ++launches; prof_end(ctx, st);
        if (kp.has_vor) { prof_begin(ctx, st, 3); launch_vor(db, kp, B, smem_g, st); ++launches; prof_end(ctx, st); }
        /* Split round 0 (throughput regime): the bands that needed retry rounds in the previous iteration were linearised
         * on the side stream; instead of joining here, the side stream also solves / evaluates ROUND 0 for exactly those
         * bands (list of the previous round 1, own scratch) while the main stream does it for all others. Both append to
         * the same retry list; the main stream waits for the side stream's evaluation only before it needs the deferral
         * tags again. Bands never share data: only the schedule changes, the results do not. */
        side_share = deferred_done && split_ok;
        if (deferred_done && !side_share) CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_join, 0));
        deferred_done = false;
      }
      if (ctx->solver == 2) {
        const int* sched = (it == 0) ? sched_first : sched_later;
        const int rounds = (it == 0) ? n_first : n_later; /* widths add up to g2o's maxTrialsAfterFailure = 10 */
        const bool fork = overlap && rounds > 1 && !kp.has_vor;
        cudaStream_t rs = st;
        auto launch_solve = [&](const SpecBufs& spec, int K, int round, cudaStream_t s) {
          launches += launch_spec_solve(ctx, db, spec, K, it, round, g, s, 0);
        };
        for (int round = 0; round < rounds; ++round, ++g) {
          const int K = sched[round];
          ctx->spec.K = K;
          const size_t smem_e = eval_bytes(ctx, bt->n_cap, bt->M_cap, K);
          SpecBufs spec = ctx->spec; /* main-stream launch: every band, or every band but the side stream's share */
          if (round == 0 && side_share) { spec.defer = ctx->defer; spec.skip_tag = tag - 1; }
          if (round == 1 && fork) { /* retry rounds go to the side stream */
            CUDA_TRY(ctx, cudaEventRecord(ctx->ev_fork, st));
            CUDA_TRY(ctx, cudaStreamWaitEvent(ctx->side, ctx->ev_fork, 0));
            rs = ctx->side;
          }
          if (rs == ctx->side) { spec.Lf = ctx->Lf2; spec.dx = ctx->dx2; } /* the side stream's own scratch */
          if (round == 0 && side_share) { /* the side stream's share of round 0, issued before its retry rounds */
            SpecBufs ss = ctx->spec;
            ss.Lf = ctx->Lf2; ss.dx = ctx->dx2;
            ss.sel_list = ctx->spec.list + (size_t)(last_r1 % SPEC_LISTS) * B;
            ss.sel_cnt = ctx->spec.cnt + last_r1;
            launch_solve(ss, K, 0, ctx->side);
            launch_trial_eval(ctx, ss, db, kp, B, K, smem_e, it, 0, g, tag, ctx->side); ++launches;
            CUDA_TRY(ctx, cudaEventRecord(ctx->ev_s0, ctx->side));
          }
          prof_begin(ctx, st, round == 0 ? 6 : 4);
          launch_solve(spec, K, round, rs);
          prof_end(ctx, st);
          prof_begin(ctx, st, round == 0 ? 7 : 4);
          launch_trial_eval(ctx, spec, db, kp, B, K, smem_e, it, round, g, tag, rs);
          ++launches; prof_end(ctx, st);
          /* the deferral tags / the retry list of this iteration are complete once both halves of round 0 are done */
          if (round == 0 && side_share) CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_s0, 0));
        }
        last_r1 = g - rounds + 1;
        if (fork) {
          if (it + 1 < args->iterations_innerloop) { /* next kernel A for the bands of the round-1 list, then join */
            DevBatch dl = db;
            dl.a_list = ctx->spec.list + (size_t)(last_r1 % SPEC_LISTS) * B;
            dl.a_cnt = ctx->spec.cnt + last_r1;
            launch_linearize(ctx, dl, kp, B, bt->M_cap, ctx->side); ++launches;
            deferred_done = true;
            CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->side));
          } else if (o + 1 < outer) {
            /* last inner iteration: the side stream goes on with the next outer iteration's autoResize / buildGraph /
             * first kernel A for its bands (next weight multiplier), the main stream does the same for all others */
            const KParams kn = make_kparams(ctx, bt, weight_multiplier * p.weight_adapt_factor);
            DevBatch dl = db;
            dl.a_list = ctx->spec.list + (size_t)(last_r1 % SPEC_LISTS) * B;
            dl.a_cnt = ctx->spec.cnt + last_r1;
            if (p.teb_autosize) { k_auto_resize<<<gb, tb, 0, ctx->side>>>(dl, kn); ++launches; }
            launch_build_graph(dl, kn, B, smem_g, ctx->side); ++launches;
            launch_linearize(ctx, dl, kn, B, bt->M_cap, ctx->side); ++launches;
            carried = true;
            CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->side));
          } else {
            CUDA_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->side));
            CUDA_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_join, 0));
          }
        }
      } else {
        prof_begin(ctx, st, 4);
        if (use_bcr && kp.generic) k_lm_step_t<1, KB_BCR_THREADS, true><<<B, KB_BCR_THREADS, smem_bcr, st>>>(db, kp, it);
        else if (use_bcr) k_lm_step_t<1, KB_BCR_THREADS, false><<<B, KB_BCR_THREADS, smem_bcr, st>>>(db, kp, it);
        else if (kp.generic) k_lm_step_t<0, KB_THREADS, true><<<B, KB_THREADS, smem_b, st>>>(db, kp, it);
        else k_lm_step_t<0, KB_THREADS, false><<<B, KB_THREADS, smem_b, st>>>(db, kp, it);
        ++launches; prof_end(ctx, st);
      }
    }
    weight_multiplier *= p.weight_adapt_factor; /* optimal_planner.cpp:227 */
  }
  /* With no outer iteration optimizeTEB returns true without computing a cost (optimal_planner.cpp:230): k_finalize
   * sets OPTIMIZED for a band that has not failed and leaves cost = HUGE_VAL when told of one iteration, no cost. */
  TebOptimizeArgs fa = *args;
  if (fa.iterations_outerloop == 0) { fa.iterations_outerloop = 1; fa.iterations_innerloop = 1; fa.compute_cost_afterwards = 0; }
  prof_begin(ctx, st, 5); k_finalize<<<gb, tb, 0, st>>>(db, kp, fa); ++launches; prof_end(ctx, st);
  ctx->launches = launches;
  if (ctx->profiling && ctx->ev_used > 4096) { cudaStreamSynchronize(st); prof_collect(ctx); }
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

/* CUDA-graph replay of the launch sequence. The sequence is a pure function of the batch description (dimensions and
 * buffer addresses), the optimize arguments, the parameter block and the context switches, so it is captured once per
 * distinct key (fork / join of the retry side stream included) and replayed afterwards: one graph launch instead of
 * ~130-170 kernel launches. That only matters in the latency regime (a single planning request: kernels of 10-50 us), so
 * graphs are used there by default (tebgpu_set_graph: 0 never, 1 always, 2 automatic). */
static uint64_t graph_key(const tebgpu_ctx* ctx, const TebBatch* bt, const TebOptimizeArgs* a, cudaStream_t st,
                          const TebPlanInput* plan) {
  uint64_t h = 1469598103934665603ull;
  auto mix = [&](const void* p, size_t nbytes) {
    const unsigned char* c = static_cast<const unsigned char*>(p);
    for (size_t k = 0; k < nbytes; ++k) { h ^= c[k]; h *= 1099511628211ull; }
  };
  mix(bt, sizeof(*bt));
  mix(a, sizeof(*a));
  mix(&ctx->params_version, sizeof(ctx->params_version));
  const int sw[12] = {ctx->solver, ctx->spec_k, ctx->linearize_variant, ctx->ka_staged, ctx->eval_v1, ctx->overlap, ctx->eval_minb, ctx->warp_solver, ctx->eval_mode, ctx->split, ctx->solve_form, ctx->ka_persist};
  mix(sw, sizeof(sw));
  mix(&st, sizeof(st));
  if (plan) mix(plan, sizeof(*plan)); /* the plan entry points' cycle: its buffers and read-out arguments */
  return h;
}

/* the launch sequence of the plan entry points: plan / warm start, the optimize sequence, the velocity command */
static int32_t issue_plan(tebgpu_ctx* ctx, const TebBatch* bt, const TebPlanInput* plan, const TebOptimizeArgs* args,
                          cudaStream_t st) {
  const DevBatch db = make_devbatch(ctx, bt);
  const int B = bt->B;
  prof_begin(ctx, st, 9);
  k_plan_begin<<<(B + 3) / 4, 128, 0, st>>>(db, ctx->params, *plan, ctx->plan_status);
  prof_end(ctx, st);
  const int32_t rc = issue_optimize(ctx, bt, args, st, ctx->plan_status);
  if (rc) return rc;
  prof_begin(ctx, st, 10);
  k_velocity_command<<<(B + 127) / 128, 128, 0, st>>>(db, ctx->params, *plan);
  prof_end(ctx, st);
  ctx->launches += 2;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

/* one optimize call (plan == NULL) or plan cycle, launched directly or through a captured CUDA graph */
static int32_t run_sequence(tebgpu_ctx* ctx, const TebBatch* bt, const TebOptimizeArgs* args, cudaStream_t st,
                            const TebPlanInput* plan) {
  auto issue = [&]() { return plan ? issue_plan(ctx, bt, plan, args, st) : issue_optimize(ctx, bt, args, st); };
  const bool latency_regime = (long long)bt->B * 8 <= (long long)ctx->sms * 4 * 32;
  const bool use_graph = !ctx->profiling && (ctx->graph_mode == 1 || (ctx->graph_mode == 2 && latency_regime));
  if (!use_graph) return issue();
  const uint64_t key = graph_key(ctx, bt, args, st, plan);
  for (auto& e : ctx->graphs)
    if (e.key == key) {
      e.stamp = ++ctx->graph_clock;
      ctx->launches = e.launches;
      ctx->last_spec_k = e.spec_k; ctx->last_spec_first = e.spec_first;
      CUDA_TRY(ctx, cudaGraphLaunch(e.exec, st));
      return TEBGPU_OK;
    }
  CUDA_TRY(ctx, cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  int32_t rc = issue();
  cudaGraph_t graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(st, &graph);
  if (rc != TEBGPU_OK || ce != cudaSuccess || !graph) {
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    if (rc == TEBGPU_OK) { /* capture itself failed: run the sequence directly */
      ctx->graph_mode = 0;
      return issue();
    }
    return rc;
  }
  tebgpu_ctx::GraphEntry ent;
  ent.key = key; ent.launches = ctx->launches; ent.stamp = ++ctx->graph_clock;
  ent.spec_k = ctx->last_spec_k; ent.spec_first = ctx->last_spec_first;
  const cudaError_t ie = cudaGraphInstantiate(&ent.exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ie != cudaSuccess) { cudaGetLastError(); ctx->graph_mode = 0; return issue(); }
  if (ctx->graphs.size() >= 8) { /* drop the least recently used graph */
    size_t old = 0;
    for (size_t k = 1; k < ctx->graphs.size(); ++k)
      if (ctx->graphs[k].stamp < ctx->graphs[old].stamp) old = k;
    cudaGraphExecDestroy(ctx->graphs[old].exec);
    ctx->graphs.erase(ctx->graphs.begin() + old);
  }
  ctx->graphs.push_back(ent);
  CUDA_TRY(ctx, cudaGraphLaunch(ent.exec, st));
  return TEBGPU_OK;
}

int32_t tebgpu_optimize_batch_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebOptimizeArgs* args, void* cuda_stream) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  rc = check_path(ctx, bt, true);
  if (rc) return rc;
  if (!args || args->iterations_innerloop < 0 || args->iterations_outerloop < 0) { ctx->err = "bad optimize args"; return TEBGPU_ERR_INVALID_ARG; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
  return run_sequence(ctx, bt, args, st, nullptr);
}

int32_t tebgpu_set_warp_solver(tebgpu_ctx* ctx, int32_t mode) {
  if (!ctx || mode < 0 || mode > 4) return TEBGPU_ERR_INVALID_ARG;
  ctx->warp_solver = mode;
  return TEBGPU_OK;
}

int32_t tebgpu_set_solve_form(tebgpu_ctx* ctx, int32_t form) {
  if (!ctx || !(form == 0 || form == 1 || form == 11 || form == 22 || form == 33)) return TEBGPU_ERR_INVALID_ARG;
  ctx->solve_form = form;
  return TEBGPU_OK;
}

int32_t tebgpu_set_graph(tebgpu_ctx* ctx, int32_t mode) {
  if (!ctx || mode < 0 || mode > 2) return TEBGPU_ERR_INVALID_ARG;
  ctx->graph_mode = mode;
  return TEBGPU_OK;
}

int32_t tebgpu_set_profiling(tebgpu_ctx* ctx, int32_t enable) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  prof_collect(ctx);
  ctx->profiling = enable != 0;
  for (int k = 0; k < 11; ++k) { ctx->prof_ms[k] = 0; ctx->prof_cnt[k] = 0; }
  return TEBGPU_OK;
}

int32_t tebgpu_get_kernel_times(tebgpu_ctx* ctx, double ms_out[9], int64_t count_out[9]) {
  if (!ctx || !ms_out || !count_out) return TEBGPU_ERR_INVALID_ARG;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  CUDA_TRY(ctx, cudaDeviceSynchronize());
  prof_collect(ctx);
  for (int k = 0; k < 9; ++k) { ms_out[k] = ctx->prof_ms[k]; count_out[k] = ctx->prof_cnt[k]; ctx->prof_ms[k] = 0; ctx->prof_cnt[k] = 0; }
  return TEBGPU_OK;
}

int32_t tebgpu_get_plan_kernel_times(tebgpu_ctx* ctx, double ms_out[2], int64_t count_out[2]) {
  if (!ctx || !ms_out || !count_out) return TEBGPU_ERR_INVALID_ARG;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  CUDA_TRY(ctx, cudaDeviceSynchronize());
  prof_collect(ctx);
  for (int k = 0; k < 2; ++k) { ms_out[k] = ctx->prof_ms[9 + k]; count_out[k] = ctx->prof_cnt[9 + k]; ctx->prof_ms[9 + k] = 0; ctx->prof_cnt[9 + k] = 0; }
  return TEBGPU_OK;
}

int32_t tebgpu_set_linearize_variant(tebgpu_ctx* ctx, int32_t v) {
  if (!ctx || v < 0 || v > 1) return TEBGPU_ERR_INVALID_ARG;
  ctx->linearize_variant = v;
  return TEBGPU_OK;
}

int32_t tebgpu_set_fleet_search(tebgpu_ctx* ctx, int32_t mode) {
  if (!ctx || mode < TEBGPU_FLEET_SEARCH_AUTO || mode > TEBGPU_FLEET_SEARCH_ONE_BUCKET) return TEBGPU_ERR_INVALID_ARG;
  ctx->fleet_search = mode;
  return TEBGPU_OK;
}

int32_t tebgpu_set_speculation(tebgpu_ctx* ctx, int32_t k) {
  if (!ctx || !(k == 0 || k == 2 || k == 4 || k == 6 || k == 8)) return TEBGPU_ERR_INVALID_ARG;
  ctx->spec_k = k;
  return TEBGPU_OK;
}

int32_t tebgpu_set_solver(tebgpu_ctx* ctx, int32_t solver) {
  if (!ctx || solver < 0 || solver > 2) return TEBGPU_ERR_INVALID_ARG;
  ctx->solver = solver;
  return TEBGPU_OK;
}

int32_t tebgpu_synchronize(tebgpu_ctx* ctx) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return TEBGPU_OK;
}

static TebBatch mirror_batch(tebgpu_ctx* ctx, const TebBatch* bt) {
  TebBatch d = *bt;
  d.poses = ctx->d_poses; d.n = ctx->d_n; d.scene_id = ctx->d_scene; d.obstacles = ctx->d_obst; d.obst_count = ctx->d_ocount;
  d.via = bt->V_cap > 0 ? ctx->d_via : nullptr; d.via_count = bt->V_cap > 0 ? ctx->d_vcount : nullptr;
  d.vel_start = ctx->d_vs; d.vel_goal = ctx->d_vg; d.prefer_rotdir = bt->prefer_rotdir ? ctx->d_rot : nullptr;
  d.cost = ctx->d_cost; d.chi2 = ctx->d_chi2; d.status = ctx->d_status; d.lm_iters = ctx->d_iters;
  d.obst_vertices = bt->PV_cap > 0 ? ctx->d_pverts : nullptr;
  return d;
}

static int32_t upload_batch(tebgpu_ctx* ctx, const TebBatch* bt) {
  cudaStream_t st = ctx->stream;
  const size_t B = bt->B, nc = bt->n_cap;
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_poses, bt->poses, B * nc * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_n, bt->n, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_scene, bt->scene_id, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (bt->M_cap > 0)
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_obst, bt->obstacles, (size_t)bt->S * bt->M_cap * sizeof(TebObstacle), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_ocount, bt->obst_count, (size_t)bt->S * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (bt->PV_cap > 0)
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_pverts, bt->obst_vertices, (size_t)bt->S * bt->PV_cap * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
  /* host entry points can check every per-element input before the device indexes with it */
  for (int sc = 0; sc < bt->S; ++sc)
    if (bt->obst_count[sc] < 0 || bt->obst_count[sc] > bt->M_cap) { ctx->err = "obst_count[s] outside 0 .. M_cap"; return TEBGPU_ERR_INVALID_ARG; }
  for (int b = 0; b < bt->B; ++b) {
    if (bt->scene_id[b] < 0 || bt->scene_id[b] >= bt->S) { ctx->err = "scene_id[b] outside 0 .. S-1"; return TEBGPU_ERR_INVALID_ARG; }
    if (bt->n[b] < 0 || bt->n[b] > bt->n_cap) { ctx->err = "n[b] outside 0 .. n_cap"; return TEBGPU_ERR_INVALID_ARG; }
    if (bt->V_cap > 0 && (bt->via_count[b] < 0 || bt->via_count[b] > bt->V_cap)) { ctx->err = "via_count[b] outside 0 .. V_cap"; return TEBGPU_ERR_INVALID_ARG; }
  }
  for (int sc = 0; sc < bt->S; ++sc)
    for (int m = 0; m < bt->obst_count[sc] && m < bt->M_cap; ++m) {
      const TebObstacle& o = bt->obstacles[(size_t)sc * bt->M_cap + m];
      if (o.type < TEB_OBST_POINT || o.type > TEB_OBST_POLYGON) { ctx->err = "unknown obstacle type"; return TEBGPU_ERR_INVALID_ARG; }
      if (o.type >= TEB_OBST_LINE) {
        const int need = o.type == TEB_OBST_POLYGON ? 1 : 2;
        if (o.vertex_count < need || (o.type != TEB_OBST_POLYGON && o.vertex_count != 2) || o.vertex_begin < 0 ||
            (long long)o.vertex_begin + o.vertex_count > bt->PV_cap) {
          ctx->err = "obstacle vertex range outside obst_vertices";
          return TEBGPU_ERR_INVALID_ARG;
        }
      }
    }
  if (bt->V_cap > 0) {
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_via, bt->via, B * bt->V_cap * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_vcount, bt->via_count, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_vs, bt->vel_start, B * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_vg, bt->vel_goal, B * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
  if (bt->prefer_rotdir)
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_rot, bt->prefer_rotdir, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  return TEBGPU_OK;
}

int32_t tebgpu_optimize_batch(tebgpu_ctx* ctx, const TebBatch* bt, const TebOptimizeArgs* args) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rc = upload_batch(ctx, bt);
  if (rc) return rc;
  TebBatch d = mirror_batch(ctx, bt);
  rc = tebgpu_optimize_batch_device(ctx, &d, args, nullptr);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  const size_t B = bt->B, nc = bt->n_cap;
  CUDA_TRY(ctx, cudaMemcpyAsync(bt->poses, ctx->d_poses, B * nc * 4 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(bt->n, ctx->d_n, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (bt->cost) CUDA_TRY(ctx, cudaMemcpyAsync(bt->cost, ctx->d_cost, B * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (bt->chi2) CUDA_TRY(ctx, cudaMemcpyAsync(bt->chi2, ctx->d_chi2, B * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (bt->status) CUDA_TRY(ctx, cudaMemcpyAsync(bt->status, ctx->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (bt->lm_iters) CUDA_TRY(ctx, cudaMemcpyAsync(bt->lm_iters, ctx->d_iters, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

static int32_t check_plan(tebgpu_ctx* ctx, const TebPlanInput* pi) {
  if (!pi || !pi->cmd) { ctx->err = "plan input or cmd == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (pi->initial_plan ? pi->P_cap < 1 : (!pi->start || !pi->goal)) {
    ctx->err = "plan input needs start and goal, or initial_plan with P_cap >= 1";
    return TEBGPU_ERR_INVALID_ARG;
  }
  return TEBGPU_OK;
}

int32_t tebgpu_plan_batch_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebPlanInput* plan, const TebOptimizeArgs* args,
                                 void* cuda_stream) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  rc = check_plan(ctx, plan);
  if (rc) return rc;
  rc = check_path(ctx, bt, true);
  if (rc) return rc;
  if (!args || args->iterations_innerloop < 0 || args->iterations_outerloop < 0) { ctx->err = "bad optimize args"; return TEBGPU_ERR_INVALID_ARG; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
  return run_sequence(ctx, bt, args, st, plan);
}

int32_t tebgpu_plan_batch(tebgpu_ctx* ctx, TebBatch* bt, const TebPlanInput* plan, const TebOptimizeArgs* args) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  rc = check_plan(ctx, plan);
  if (rc) return rc;
  const size_t B = bt->B, nc = bt->n_cap;
  /* the rows the device entry point would report as TEB_STATUS_BAD_INPUT are refused here, before anything runs */
  for (size_t b = 0; b < B; ++b) {
    if (plan->initial_plan) {
      const int P = plan->plan_count ? plan->plan_count[b] : plan->P_cap;
      if (P < 1 || P > plan->P_cap) { ctx->err = "plan_count[b] outside 1 .. P_cap"; return TEBGPU_ERR_INVALID_ARG; }
      for (int k = 0; k < 3 * P; ++k)
        if (!std::isfinite(plan->initial_plan[b * plan->P_cap * 3 + k])) { ctx->err = "non-finite plan row"; return TEBGPU_ERR_INVALID_ARG; }
    } else {
      for (int k = 0; k < 3; ++k)
        if (!std::isfinite(plan->start[3 * b + k]) || !std::isfinite(plan->goal[3 * b + k])) {
          ctx->err = "non-finite start or goal";
          return TEBGPU_ERR_INVALID_ARG;
        }
    }
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rc = upload_batch(ctx, bt);
  if (rc) return rc;
  cudaStream_t st = ctx->stream;
  TebPlanInput dp = *plan;
  dp.cmd = ctx->d_cmd;
  dp.path = plan->path ? ctx->d_path : nullptr;
  if (plan->initial_plan) {
    if ((size_t)plan->P_cap > ctx->plan_rows) { /* the first call with a longer plan grows the mirror */
      CUDA_TRY(ctx, cudaStreamSynchronize(st));
      if (ctx->d_plan) CUDA_TRY(ctx, cudaFree(ctx->d_plan));
      ctx->d_plan = nullptr;
      ctx->plan_rows = 0;
      CUDA_TRY(ctx, cudaMalloc(&ctx->d_plan, (size_t)ctx->lim.max_bands * plan->P_cap * 3 * sizeof(double)));
      ctx->plan_rows = plan->P_cap;
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_plan, plan->initial_plan, B * plan->P_cap * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    dp.initial_plan = ctx->d_plan;
    dp.start = dp.goal = nullptr;
    if (plan->plan_count) {
      CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_pcount, plan->plan_count, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
      dp.plan_count = ctx->d_pcount;
    }
  } else {
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_start, plan->start, B * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_goal, plan->goal, B * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
    dp.start = ctx->d_start; dp.goal = ctx->d_goal;
    dp.plan_count = nullptr;
  }
  TebBatch d = mirror_batch(ctx, bt);
  rc = tebgpu_plan_batch_device(ctx, &d, &dp, args, nullptr);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(bt->poses, ctx->d_poses, B * nc * 4 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(bt->n, ctx->d_n, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (bt->cost) CUDA_TRY(ctx, cudaMemcpyAsync(bt->cost, ctx->d_cost, B * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (bt->chi2) CUDA_TRY(ctx, cudaMemcpyAsync(bt->chi2, ctx->d_chi2, B * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (bt->status) CUDA_TRY(ctx, cudaMemcpyAsync(bt->status, ctx->d_status, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (bt->lm_iters) CUDA_TRY(ctx, cudaMemcpyAsync(bt->lm_iters, ctx->d_iters, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(plan->cmd, ctx->d_cmd, B * 4 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (plan->path) CUDA_TRY(ctx, cudaMemcpyAsync(plan->path, ctx->d_path, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

/* argument checks of every feasibility entry point: nothing is launched when one fails. table: the obstacle-table
 * check, which also reads the batch's obstacle arrays and collision_distance */
static int32_t check_feasible_args(tebgpu_ctx* ctx, const TebBatch* bt, const TebFeasibilityArgs* fa, bool table = true) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  if (!bt || !fa) { ctx->err = "batch or feasibility args == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (table) {
    if (bt->B < 1 || bt->n_cap < 1 || bt->S < 1 || bt->M_cap < 0 || bt->PV_cap < 0) { ctx->err = "bad batch dimensions"; return TEBGPU_ERR_INVALID_ARG; }
    if (bt->B > ctx->lim.max_bands || bt->n_cap > ctx->lim.max_poses || bt->S > ctx->lim.max_scenes ||
        bt->M_cap > ctx->lim.max_obstacles || bt->PV_cap > ctx->lim.max_obst_vertices) { ctx->err = "batch exceeds the context limits"; return TEBGPU_ERR_CAPACITY; }
    if (!bt->poses || !bt->n || !bt->scene_id || !bt->obst_count) { ctx->err = "missing required batch array"; return TEBGPU_ERR_INVALID_ARG; }
    if (bt->M_cap > 0 && !bt->obstacles) { ctx->err = "obstacles == NULL"; return TEBGPU_ERR_INVALID_ARG; }
    if (bt->PV_cap > 0 && !bt->obst_vertices) { ctx->err = "obst_vertices == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  } else {
    if (bt->B < 1 || bt->n_cap < 1 || bt->S < 1) { ctx->err = "bad batch dimensions"; return TEBGPU_ERR_INVALID_ARG; }
    if (bt->B > ctx->lim.max_bands || bt->n_cap > ctx->lim.max_poses || bt->S > ctx->lim.max_scenes) { ctx->err = "batch exceeds the context limits"; return TEBGPU_ERR_CAPACITY; }
    if (!bt->poses || !bt->n || !bt->scene_id) { ctx->err = "missing required batch array"; return TEBGPU_ERR_INVALID_ARG; }
  }
  if (!fa->feasible || !fa->query_count) { ctx->err = "feasible or query_count == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (!(std::isfinite(fa->inscribed_radius) && fa->inscribed_radius > 0)) { ctx->err = "inscribed_radius must be > 0 and finite"; return TEBGPU_ERR_INVALID_ARG; }
  if (!(std::isfinite(fa->angular_resolution) && fa->angular_resolution > 0)) { ctx->err = "angular_resolution must be > 0 and finite"; return TEBGPU_ERR_INVALID_ARG; }
  if (table && !(std::isfinite(fa->collision_distance) && fa->collision_distance >= 0)) { ctx->err = "collision_distance must be >= 0 and finite"; return TEBGPU_ERR_INVALID_ARG; }
  if (fa->max_queries < 1) { ctx->err = "max_queries must be >= 1"; return TEBGPU_ERR_INVALID_ARG; }
  if (!ctx->have_params) { ctx->err = "tebgpu_set_params has not been called"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

/* k_feasible on arguments already checked; the path (staged / global table) follows M_cap like every default kernel */
static int32_t issue_feasible(tebgpu_ctx* ctx, const TebBatch* bt, const TebFeasibilityArgs* fa, cudaStream_t st) {
  if (!ctx->feas_ready) { /* the staged builds take up to 64 KB of obstacle rows beyond the static shared memory */
    const int smax = STAGED_MAX_OBST * (int)sizeof(TebObstacle);
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_feasible<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smax));
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_feasible<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smax));
    ctx->feas_ready = true;
  }
  KParams kp = make_kparams(ctx, bt, 1.0);
  FeasDev fd;
  std::memset(&fd, 0, sizeof(fd));
  fd.B = bt->B; fd.n_cap = bt->n_cap; fd.S = bt->S; fd.M_cap = bt->M_cap; fd.PV_cap = bt->PV_cap;
  fd.poses = bt->poses; fd.n = bt->n; fd.scene_id = bt->scene_id; fd.obstacles = bt->obstacles; fd.obst_count = bt->obst_count;
  fd.obst_vertices = bt->PV_cap > 0 ? bt->obst_vertices : nullptr;
  fd.a = *fa;
  const bool gt = global_table(bt->M_cap);
  const size_t smem = gt ? 0 : (size_t)bt->M_cap * sizeof(TebObstacle);
  const int B = bt->B;
  if (gt && kp.generic) k_feasible<true, true><<<B, FEAS_THREADS, 0, st>>>(fd, kp);
  else if (gt) k_feasible<false, true><<<B, FEAS_THREADS, 0, st>>>(fd, kp);
  else if (kp.generic) k_feasible<true, false><<<B, FEAS_THREADS, smem, st>>>(fd, kp);
  else k_feasible<false, false><<<B, FEAS_THREADS, smem, st>>>(fd, kp);
  ctx->last_feas_build = gt ? TEBGPU_FEAS_BUILD_GLOBAL : TEBGPU_FEAS_BUILD_STAGED;
  ctx->last_feas_grid = B;
  ctx->launches = 1;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

int32_t tebgpu_check_feasible_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebFeasibilityArgs* fa, void* cuda_stream) {
  const int32_t rc = check_feasible_args(ctx, bt, fa);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_feasible(ctx, bt, fa, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

int32_t tebgpu_check_feasible(tebgpu_ctx* ctx, const TebBatch* bt, const TebFeasibilityArgs* fa) {
  int32_t rc = check_feasible_args(ctx, bt, fa);
  if (rc) return rc;
  /* the rows the device entry point would answer with -1 are refused here, before anything runs */
  for (int sc = 0; sc < bt->S; ++sc)
    if (bt->obst_count[sc] < 0 || bt->obst_count[sc] > bt->M_cap) { ctx->err = "obst_count[s] outside 0 .. M_cap"; return TEBGPU_ERR_INVALID_ARG; }
  for (int b = 0; b < bt->B; ++b) {
    if (bt->scene_id[b] < 0 || bt->scene_id[b] >= bt->S) { ctx->err = "scene_id[b] outside 0 .. S-1"; return TEBGPU_ERR_INVALID_ARG; }
    if (bt->n[b] < 0 || bt->n[b] > bt->n_cap) { ctx->err = "n[b] outside 0 .. n_cap"; return TEBGPU_ERR_INVALID_ARG; }
  }
  for (int sc = 0; sc < bt->S; ++sc)
    for (int m = 0; m < bt->obst_count[sc]; ++m) {
      const TebObstacle& o = bt->obstacles[(size_t)sc * bt->M_cap + m];
      if (o.type < TEB_OBST_POINT || o.type > TEB_OBST_POLYGON) { ctx->err = "unknown obstacle type"; return TEBGPU_ERR_INVALID_ARG; }
      if (o.type >= TEB_OBST_LINE && (o.vertex_count < 1 || (o.type != TEB_OBST_POLYGON && o.vertex_count != 2) ||
                                      o.vertex_begin < 0 || (long long)o.vertex_begin + o.vertex_count > bt->PV_cap)) {
        ctx->err = "obstacle vertex range outside obst_vertices";
        return TEBGPU_ERR_INVALID_ARG;
      }
    }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t B = bt->B, nc = bt->n_cap, mq = fa->max_queries;
  if (!ctx->d_feas) {
    CUDA_TRY(ctx, cudaMalloc(&ctx->d_feas, ctx->lim.max_bands * sizeof(int32_t)));
    CUDA_TRY(ctx, cudaMalloc(&ctx->d_qcount, ctx->lim.max_bands * sizeof(int32_t)));
  }
  if (fa->queries && mq > ctx->feas_rows) { /* the first call with more query rows grows the mirror */
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    if (ctx->d_queries) CUDA_TRY(ctx, cudaFree(ctx->d_queries));
    ctx->d_queries = nullptr;
    ctx->feas_rows = 0;
    CUDA_TRY(ctx, cudaMalloc(&ctx->d_queries, (size_t)ctx->lim.max_bands * mq * 3 * sizeof(double)));
    ctx->feas_rows = mq;
  }
  /* the poses / obstacle mirrors of the host-buffer entry points: every host optimize / plan call uploads them anew */
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_poses, bt->poses, B * nc * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_n, bt->n, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_scene, bt->scene_id, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (bt->M_cap > 0)
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_obst, bt->obstacles, (size_t)bt->S * bt->M_cap * sizeof(TebObstacle), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_ocount, bt->obst_count, (size_t)bt->S * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (bt->PV_cap > 0)
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_pverts, bt->obst_vertices, (size_t)bt->S * bt->PV_cap * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
  TebBatch d = *bt;
  d.poses = ctx->d_poses; d.n = ctx->d_n; d.scene_id = ctx->d_scene; d.obstacles = ctx->d_obst; d.obst_count = ctx->d_ocount;
  d.obst_vertices = bt->PV_cap > 0 ? ctx->d_pverts : nullptr;
  TebFeasibilityArgs da = *fa;
  da.feasible = ctx->d_feas; da.query_count = ctx->d_qcount;
  da.queries = fa->queries ? ctx->d_queries : nullptr;
  rc = issue_feasible(ctx, &d, &da, st);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(fa->feasible, ctx->d_feas, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(fa->query_count, ctx->d_qcount, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  if (fa->queries) { /* only the rows the kernel wrote reach the caller: min(query_count, max_queries) per band */
    std::vector<double> q(B * mq * 3);
    CUDA_TRY(ctx, cudaMemcpy(q.data(), ctx->d_queries, q.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t b = 0; b < B; ++b) {
      const size_t rows = std::min<size_t>((size_t)std::max(fa->query_count[b], 0), mq);
      std::memcpy(fa->queries + b * mq * 3, q.data() + b * mq * 3, rows * 3 * sizeof(double));
    }
  }
  return TEBGPU_OK;
}

static int32_t grow_mirror(tebgpu_ctx* ctx, void** p, size_t* have, size_t bytes, cudaStream_t st);

/* argument checks of both costmap feasibility entry points: nothing is launched when one fails */
static int32_t check_feasible_costmap_args(tebgpu_ctx* ctx, const TebBatch* bt, const TebFeasibilityArgs* fa,
                                           const TebCostmapWorld* w) {
  const int32_t rc = check_feasible_args(ctx, bt, fa, false);
  if (rc) return rc;
  if (!w) { ctx->err = "costmap world == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (w->cell_cap < 1) { ctx->err = "cell_cap must be >= 1"; return TEBGPU_ERR_INVALID_ARG; }
  if (!w->cost || !w->grid || !w->origin) { ctx->err = "missing required costmap array"; return TEBGPU_ERR_INVALID_ARG; }
  if (w->footprint_count < 0 || w->footprint_count > TEB_COSTMAP_FOOTPRINT_MAX) { ctx->err = "footprint_count outside 0 .. TEB_COSTMAP_FOOTPRINT_MAX"; return TEBGPU_ERR_INVALID_ARG; }
  if (w->footprint_count > 0 && !w->footprint) { ctx->err = "footprint == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  for (int k = 0; k < 2 * w->footprint_count; ++k)
    if (!std::isfinite(w->footprint[k])) { ctx->err = "non-finite footprint point"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

/* k_feasible_costmap on arguments already checked: the footprint travels in the launch's parameter block */
static int32_t issue_feasible_costmap(tebgpu_ctx* ctx, const TebBatch* bt, const TebFeasibilityArgs* fa,
                                      const TebCostmapWorld* w, cudaStream_t st) {
  FeasDev fd;
  std::memset(&fd, 0, sizeof(fd));
  fd.B = bt->B; fd.n_cap = bt->n_cap; fd.S = bt->S;
  fd.poses = bt->poses; fd.n = bt->n; fd.scene_id = bt->scene_id;
  fd.a = *fa;
  FeasRasterDev rd;
  std::memset(&rd, 0, sizeof(rd));
  rd.cell_cap = w->cell_cap; rd.F = w->footprint_count;
  rd.cost = w->cost; rd.grid = w->grid; rd.origin = w->origin; rd.query_cost = w->query_cost;
  if (rd.F) std::memcpy(rd.fp, w->footprint, (size_t)rd.F * 2 * sizeof(double));
  const int B = bt->B;
  k_feasible_costmap<<<B, FEAS_THREADS, 0, st>>>(fd, rd);
  ctx->last_feas_build = TEBGPU_FEAS_BUILD_COSTMAP;
  ctx->last_feas_grid = B;
  ctx->launches = 1;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

int32_t tebgpu_check_feasible_costmap_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebFeasibilityArgs* fa,
                                             const TebCostmapWorld* w, void* cuda_stream) {
  const int32_t rc = check_feasible_costmap_args(ctx, bt, fa, w);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_feasible_costmap(ctx, bt, fa, w, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

int32_t tebgpu_check_feasible_costmap(tebgpu_ctx* ctx, const TebBatch* bt, const TebFeasibilityArgs* fa,
                                      const TebCostmapWorld* w) {
  int32_t rc = check_feasible_costmap_args(ctx, bt, fa, w);
  if (rc) return rc;
  /* the bands the device entry point would answer with -1 are refused here, before anything runs */
  for (int b = 0; b < bt->B; ++b) {
    const int sc = bt->scene_id[b];
    if (sc < 0 || sc >= bt->S) { ctx->err = "scene_id[b] outside 0 .. S-1"; return TEBGPU_ERR_INVALID_ARG; }
    if (bt->n[b] < 0 || bt->n[b] > bt->n_cap) { ctx->err = "n[b] outside 0 .. n_cap"; return TEBGPU_ERR_INVALID_ARG; }
    const int32_t sx = w->grid[2 * sc], sy = w->grid[2 * sc + 1];
    const double* o = w->origin + 3 * sc;
    if (sx < 1 || sy < 1) { ctx->err = "costmap size < 1"; return TEBGPU_ERR_INVALID_ARG; }
    if ((long long)sx * sy > w->cell_cap) { ctx->err = "sx * sy > cell_cap"; return TEBGPU_ERR_INVALID_ARG; }
    if (!(std::isfinite(o[2]) && o[2] > 0)) { ctx->err = "costmap resolution must be > 0 and finite"; return TEBGPU_ERR_INVALID_ARG; }
    if (!std::isfinite(o[0]) || !std::isfinite(o[1])) { ctx->err = "non-finite costmap origin"; return TEBGPU_ERR_INVALID_ARG; }
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t B = bt->B, nc = bt->n_cap, mq = fa->max_queries, S = bt->S, cells = S * (size_t)w->cell_cap;
  if (!ctx->d_feas) {
    CUDA_TRY(ctx, cudaMalloc(&ctx->d_feas, ctx->lim.max_bands * sizeof(int32_t)));
    CUDA_TRY(ctx, cudaMalloc(&ctx->d_qcount, ctx->lim.max_bands * sizeof(int32_t)));
  }
  if (fa->queries && mq > ctx->feas_rows) { /* the first call with more query rows grows the mirror */
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
    if (ctx->d_queries) CUDA_TRY(ctx, cudaFree(ctx->d_queries));
    ctx->d_queries = nullptr;
    ctx->feas_rows = 0;
    CUDA_TRY(ctx, cudaMalloc(&ctx->d_queries, (size_t)ctx->lim.max_bands * mq * 3 * sizeof(double)));
    ctx->feas_rows = mq;
  }
  /* the rasters share the costmap conversion's input mirrors */
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_ccost, &ctx->ccost_bytes, cells, st))) return rc;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_cgrid, &ctx->cgrid_bytes, S * 2 * sizeof(int32_t), st))) return rc;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_corigin, &ctx->corigin_bytes, S * 3 * sizeof(double), st))) return rc;
  if (w->query_cost && (rc = grow_mirror(ctx, (void**)&ctx->d_qcost, &ctx->qcost_bytes, B * mq * sizeof(double), st))) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_poses, bt->poses, B * nc * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_n, bt->n, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_scene, bt->scene_id, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_ccost, w->cost, cells, cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_cgrid, w->grid, S * 2 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_corigin, w->origin, S * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
  TebBatch d = *bt;
  d.poses = ctx->d_poses; d.n = ctx->d_n; d.scene_id = ctx->d_scene;
  TebFeasibilityArgs da = *fa;
  da.feasible = ctx->d_feas; da.query_count = ctx->d_qcount;
  da.queries = fa->queries ? ctx->d_queries : nullptr;
  TebCostmapWorld dw = *w;
  dw.cost = ctx->d_ccost; dw.grid = ctx->d_cgrid; dw.origin = ctx->d_corigin;
  dw.query_cost = w->query_cost ? ctx->d_qcost : nullptr;
  rc = issue_feasible_costmap(ctx, &d, &da, &dw, st);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(fa->feasible, ctx->d_feas, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(fa->query_count, ctx->d_qcount, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  /* only the rows the kernel wrote reach the caller: min(query_count, max_queries) per band */
  if (fa->queries) {
    std::vector<double> q(B * mq * 3);
    CUDA_TRY(ctx, cudaMemcpy(q.data(), ctx->d_queries, q.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t b = 0; b < B; ++b) {
      const size_t rows = std::min<size_t>((size_t)std::max(fa->query_count[b], 0), mq);
      std::memcpy(fa->queries + b * mq * 3, q.data() + b * mq * 3, rows * 3 * sizeof(double));
    }
  }
  if (w->query_cost) {
    std::vector<double> c(B * mq);
    CUDA_TRY(ctx, cudaMemcpy(c.data(), ctx->d_qcost, c.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t b = 0; b < B; ++b) {
      const size_t rows = std::min<size_t>((size_t)std::max(fa->query_count[b], 0), mq);
      std::memcpy(w->query_cost + b * mq, c.data() + b * mq, rows * sizeof(double));
    }
  }
  return TEBGPU_OK;
}

/* argument checks of both trajectory read-out entry points: nothing is launched when one fails */
static int32_t check_trajectory_args(tebgpu_ctx* ctx, const TebBatch* bt, const TebTrajectoryArgs* ta) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  if (!bt || !ta) { ctx->err = "batch or trajectory args == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->B < 1 || bt->n_cap < 1) { ctx->err = "bad batch dimensions"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->B > ctx->lim.max_bands || bt->n_cap > ctx->lim.max_poses) { ctx->err = "batch exceeds the context limits"; return TEBGPU_ERR_CAPACITY; }
  if (!bt->poses || !bt->n || !bt->vel_start || !bt->vel_goal) { ctx->err = "missing required batch array"; return TEBGPU_ERR_INVALID_ARG; }
  if (!ta->points) { ctx->err = "points == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (!ta->profile && !ta->trajectory) { ctx->err = "profile and trajectory both NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (ta->bands && ta->count < 0) { ctx->err = "count < 0"; return TEBGPU_ERR_INVALID_ARG; }
  if (!ctx->have_params) { ctx->err = "tebgpu_set_params has not been called"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

/* k_read_trajectory on arguments already checked */
static int32_t issue_read_trajectory(tebgpu_ctx* ctx, const TebBatch* bt, const TebTrajectoryArgs* ta, cudaStream_t st) {
  const int R = ta->bands ? ta->count : bt->B;
  ctx->launches = 0;
  if (R == 0) return TEBGPU_OK;
  const long long grid = ((long long)R * 32 + TRAJ_THREADS - 1) / TRAJ_THREADS;
  k_read_trajectory<<<(unsigned)grid, TRAJ_THREADS, 0, st>>>(*bt, *ta, R, ctx->params.max_vel_y);
  ctx->last_traj_grid = grid;
  ctx->launches = 1;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

int32_t tebgpu_read_trajectory_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebTrajectoryArgs* ta, void* cuda_stream) {
  const int32_t rc = check_trajectory_args(ctx, bt, ta);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_read_trajectory(ctx, bt, ta, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

/* grows one of the read-out's device mirrors to at least `bytes` */
static int32_t grow_mirror(tebgpu_ctx* ctx, void** p, size_t* have, size_t bytes, cudaStream_t st) {
  if (bytes <= *have) return TEBGPU_OK;
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  if (*p) CUDA_TRY(ctx, cudaFree(*p));
  *p = nullptr;
  *have = 0;
  CUDA_TRY(ctx, cudaMalloc(p, bytes));
  *have = bytes;
  return TEBGPU_OK;
}

int32_t tebgpu_read_trajectory(tebgpu_ctx* ctx, const TebBatch* bt, const TebTrajectoryArgs* ta) {
  int32_t rc = check_trajectory_args(ctx, bt, ta);
  if (rc) return rc;
  const size_t R = ta->bands ? ta->count : bt->B;
  /* the rows the device entry point would answer with -1 are refused here, before anything runs */
  for (size_t r = 0; r < R; ++r) {
    const int b = ta->bands ? ta->bands[r] : (int)r;
    if (b < 0 || b >= bt->B) { ctx->err = "bands[r] outside 0 .. B-1"; return TEBGPU_ERR_INVALID_ARG; }
    if (bt->n[b] < 0 || bt->n[b] > bt->n_cap) { ctx->err = "n[b] outside 0 .. n_cap"; return TEBGPU_ERR_INVALID_ARG; }
  }
  if (R == 0) { ctx->launches = 0; return TEBGPU_OK; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t B = bt->B, nc = bt->n_cap, prow = (nc + 1) * 3, trow = nc * 7;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_tpoints, &ctx->tpoints_bytes, R * sizeof(int32_t), st))) return rc;
  if (ta->bands && (rc = grow_mirror(ctx, (void**)&ctx->d_tbands, &ctx->tbands_bytes, R * sizeof(int32_t), st))) return rc;
  if (ta->profile && (rc = grow_mirror(ctx, (void**)&ctx->d_tprof, &ctx->tprof_bytes, R * prow * sizeof(double), st))) return rc;
  if (ta->trajectory && (rc = grow_mirror(ctx, (void**)&ctx->d_ttraj, &ctx->ttraj_bytes, R * trow * sizeof(double), st))) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_poses, bt->poses, B * nc * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_n, bt->n, B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_vs, bt->vel_start, B * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_vg, bt->vel_goal, B * 4 * sizeof(double), cudaMemcpyHostToDevice, st));
  if (ta->bands) CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_tbands, ta->bands, R * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  TebBatch d = *bt;
  d.poses = ctx->d_poses; d.n = ctx->d_n; d.vel_start = ctx->d_vs; d.vel_goal = ctx->d_vg;
  TebTrajectoryArgs da = *ta;
  da.bands = ta->bands ? ctx->d_tbands : nullptr;
  da.points = ctx->d_tpoints;
  da.profile = ta->profile ? ctx->d_tprof : nullptr;
  da.trajectory = ta->trajectory ? ctx->d_ttraj : nullptr;
  rc = issue_read_trajectory(ctx, &d, &da, st);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(ta->points, ctx->d_tpoints, R * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  /* only the rows the kernel wrote reach the caller: n + 1 profile rows and n trajectory rows per band read out */
  auto rows_back = [&](double* dst, const double* src, size_t width, int extra) -> int32_t {
    const size_t row = (nc + extra) * width;
    std::vector<double> h(R * row);
    CUDA_TRY(ctx, cudaMemcpy(h.data(), src, h.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t r = 0; r < R; ++r)
      std::memcpy(dst + r * row, h.data() + r * row, (size_t)(ta->points[r] + extra) * width * sizeof(double));
    return TEBGPU_OK;
  };
  if (ta->profile && (rc = rows_back(ta->profile, ctx->d_tprof, 3, 1))) return rc;
  if (ta->trajectory && (rc = rows_back(ta->trajectory, ctx->d_ttraj, 7, 0))) return rc;
  return TEBGPU_OK;
}

/* argument checks of both costmap conversion entry points: nothing is launched when one fails */
static int32_t check_costmap_args(tebgpu_ctx* ctx, const TebCostmapArgs* ca) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  if (!ca) { ctx->err = "costmap args == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (ca->S < 1 || ca->M_cap < 1 || ca->cell_cap < 0 || ca->C_cap < 0) { ctx->err = "bad costmap dimensions"; return TEBGPU_ERR_INVALID_ARG; }
  if (ca->S > ctx->lim.max_scenes || ca->M_cap > ctx->lim.max_obstacles) { ctx->err = "costmap scenes exceed the context limits"; return TEBGPU_ERR_CAPACITY; }
  if (!ca->grid || !ca->origin || !ca->robot || !ca->obstacles || !ca->obst_count) { ctx->err = "missing required costmap array"; return TEBGPU_ERR_INVALID_ARG; }
  if (ca->cell_cap > 0 && !ca->cost) { ctx->err = "cost == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (ca->C_cap > 0 && ca->custom_count && !ca->custom) { ctx->err = "custom == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if ((reinterpret_cast<uintptr_t>(ca->obstacles) | reinterpret_cast<uintptr_t>(ca->custom)) & 15) { ctx->err = "obstacles / custom not 16-byte aligned"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

/* argument checks of TebFrameArgs (NULL: no frames) */
static int32_t check_frame_args(tebgpu_ctx* ctx, const TebFrameArgs* fr) {
  if (!fr) return TEBGPU_OK;
  if (!fr->costmap_to_plan != !fr->plan_to_costmap) { ctx->err = "only one of costmap_to_plan / plan_to_costmap given"; return TEBGPU_ERR_INVALID_ARG; }
  if (fr->PV_cap < 0) { ctx->err = "PV_cap < 0"; return TEBGPU_ERR_INVALID_ARG; }
  if (fr->custom_vertices && !fr->custom_to_costmap) { ctx->err = "custom_vertices without custom_to_costmap"; return TEBGPU_ERR_INVALID_ARG; }
  if (fr->custom_vertices && (!fr->obst_vertices || fr->PV_cap < 1)) { ctx->err = "custom_vertices without obst_vertices or PV_cap"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

/* k_costmap_obstacles on arguments already checked; fr NULL or without custom_to_costmap: the custom rows verbatim */
static int32_t issue_costmap(tebgpu_ctx* ctx, const TebCostmapArgs* ca, const TebFrameArgs* fr, cudaStream_t st) {
  TebCostmapArgs a = *ca;
  if (!a.custom_count) a.custom = nullptr;
  TebFrameArgs f{};
  if (fr) f = *fr;
  if (f.custom_to_costmap && a.custom) k_costmap_obstacles<true><<<ca->S, COSTMAP_THREADS, 0, st>>>(a, f);
  else k_costmap_obstacles<false><<<ca->S, COSTMAP_THREADS, 0, st>>>(a, f);
  ctx->last_costmap_grid = ca->S;
  ctx->launches = 1;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

int32_t tebgpu_costmap_obstacles_tf_device(tebgpu_ctx* ctx, const TebCostmapArgs* ca, const TebFrameArgs* fr,
                                           void* cuda_stream) {
  int32_t rc = check_costmap_args(ctx, ca);
  if (rc || (rc = check_frame_args(ctx, fr))) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_costmap(ctx, ca, fr, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

int32_t tebgpu_costmap_obstacles_device(tebgpu_ctx* ctx, const TebCostmapArgs* ca, void* cuda_stream) {
  return tebgpu_costmap_obstacles_tf_device(ctx, ca, nullptr, cuda_stream);
}

int32_t tebgpu_costmap_obstacles(tebgpu_ctx* ctx, const TebCostmapArgs* ca) {
  return tebgpu_costmap_obstacles_tf(ctx, ca, nullptr);
}

int32_t tebgpu_costmap_obstacles_tf(tebgpu_ctx* ctx, const TebCostmapArgs* ca, const TebFrameArgs* fr) {
  int32_t rc = check_costmap_args(ctx, ca);
  if (rc || (rc = check_frame_args(ctx, fr))) return rc;
  const bool move = fr && fr->custom_to_costmap && ca->custom_count && ca->C_cap > 0;
  /* the scenes the device entry point would answer with -1 are refused here, before anything runs */
  for (int s = 0; s < ca->S; ++s) {
    const int32_t sx = ca->grid[2 * s], sy = ca->grid[2 * s + 1];
    if (sx < 0 || sy < 0) { ctx->err = "negative costmap size"; return TEBGPU_ERR_INVALID_ARG; }
    if ((long long)sx * sy > ca->cell_cap) { ctx->err = "sx * sy > cell_cap"; return TEBGPU_ERR_INVALID_ARG; }
    if (ca->custom_count && (ca->custom_count[s] < 0 || ca->custom_count[s] > ca->C_cap)) { ctx->err = "custom_count[s] outside 0 .. C_cap"; return TEBGPU_ERR_INVALID_ARG; }
    for (int k = 0; move && k < ca->custom_count[s]; ++k) {
      const TebObstacle& o = ca->custom[(size_t)s * ca->C_cap + k];
      if (o.type != TEB_OBST_LINE && o.type != TEB_OBST_PILL && o.type != TEB_OBST_POLYGON) continue;
      if (!fr->custom_vertices) { ctx->err = "custom Line / Pill / Polygon rows without custom_vertices"; return TEBGPU_ERR_INVALID_ARG; }
      if (o.vertex_begin < 0 || o.vertex_count < 1 || o.vertex_begin > fr->PV_cap - o.vertex_count ||
          (o.type != TEB_OBST_POLYGON && o.vertex_count != 2)) {
        ctx->err = "custom row vertices outside 0 .. PV_cap"; return TEBGPU_ERR_INVALID_ARG;
      }
    }
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t S = ca->S, M = ca->M_cap, cells = S * ca->cell_cap;
  const bool cu = ca->custom_count && ca->C_cap > 0;
  /* cudaMalloc'd mirrors are 256-byte aligned, so a cell_cap that is a multiple of 16 keeps the 16-byte raster loads */
  if (cells && (rc = grow_mirror(ctx, (void**)&ctx->d_ccost, &ctx->ccost_bytes, cells, st))) return rc;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_cgrid, &ctx->cgrid_bytes, S * 2 * sizeof(int32_t), st))) return rc;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_corigin, &ctx->corigin_bytes, S * 3 * sizeof(double), st))) return rc;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_crobot, &ctx->crobot_bytes, S * 3 * sizeof(double), st))) return rc;
  if (cu && (rc = grow_mirror(ctx, (void**)&ctx->d_ccustom, &ctx->ccustom_bytes, S * ca->C_cap * sizeof(TebObstacle), st))) return rc;
  if (ca->custom_count && (rc = grow_mirror(ctx, (void**)&ctx->d_ccount, &ctx->ccount_bytes, S * sizeof(int32_t), st))) return rc;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_cobst, &ctx->cobst_bytes, S * M * sizeof(TebObstacle), st))) return rc;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_cocount, &ctx->cocount_bytes, S * sizeof(int32_t), st))) return rc;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_cneeded, &ctx->cneeded_bytes, S * sizeof(int32_t), st))) return rc;
  if (cells) CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_ccost, ca->cost, cells, cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_cgrid, ca->grid, S * 2 * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_corigin, ca->origin, S * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_crobot, ca->robot, S * 3 * sizeof(double), cudaMemcpyHostToDevice, st));
  if (cu) CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_ccustom, ca->custom, S * ca->C_cap * sizeof(TebObstacle), cudaMemcpyHostToDevice, st));
  if (ca->custom_count) CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_ccount, ca->custom_count, S * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  TebCostmapArgs da = *ca;
  da.cost = cells ? ctx->d_ccost : nullptr;
  da.grid = ctx->d_cgrid; da.origin = ctx->d_corigin; da.robot = ctx->d_crobot;
  da.custom = cu ? ctx->d_ccustom : nullptr;
  da.custom_count = ca->custom_count ? ctx->d_ccount : nullptr;
  da.obstacles = ctx->d_cobst; da.obst_count = ctx->d_cocount; da.needed = ctx->d_cneeded;
  /* frames: the transforms and both vertex pools; obst_vertices goes up too, so the vertices no row moves come back as
   * the caller left them */
  TebFrameArgs df{};
  const size_t tf_bytes = S * 7 * sizeof(double), pv_bytes = fr && fr->custom_vertices ? S * fr->PV_cap * 2 * sizeof(double) : 0;
  if (move) {
    if ((rc = grow_mirror(ctx, (void**)&ctx->d_cframe, &ctx->cframe_bytes, tf_bytes + 2 * pv_bytes, st))) return rc;
    df.PV_cap = fr->PV_cap;
    df.custom_to_costmap = (const double*)ctx->d_cframe;
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_cframe, fr->custom_to_costmap, tf_bytes, cudaMemcpyHostToDevice, st));
    if (pv_bytes) {
      df.custom_vertices = (const double*)(ctx->d_cframe + tf_bytes);
      df.obst_vertices = (double*)(ctx->d_cframe + tf_bytes + pv_bytes);
      CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_cframe + tf_bytes, fr->custom_vertices, pv_bytes, cudaMemcpyHostToDevice, st));
      CUDA_TRY(ctx, cudaMemcpyAsync(df.obst_vertices, fr->obst_vertices, pv_bytes, cudaMemcpyHostToDevice, st));
    }
  }
  rc = issue_costmap(ctx, &da, move ? &df : nullptr, st);
  if (rc) return rc;
  if (pv_bytes && move) CUDA_TRY(ctx, cudaMemcpyAsync(fr->obst_vertices, df.obst_vertices, pv_bytes, cudaMemcpyDeviceToHost, st));
  std::vector<int32_t> need(S);
  CUDA_TRY(ctx, cudaMemcpyAsync(ca->obst_count, ctx->d_cocount, S * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(need.data(), ctx->d_cneeded, S * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  if (ca->needed) std::memcpy(ca->needed, need.data(), S * sizeof(int32_t));
  /* only the rows the kernel wrote reach the caller: min(needed, M_cap) per scene */
  for (size_t s = 0; s < S; ++s) {
    const size_t rows = std::min<size_t>((size_t)std::max(need[s], 0), M);
    if (rows)
      CUDA_TRY(ctx, cudaMemcpyAsync(ca->obstacles + s * M, ctx->d_cobst + s * M, rows * sizeof(TebObstacle), cudaMemcpyDeviceToHost, st));
  }
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

/* argument checks of both local-plan entry points: nothing is launched when one fails */
static int32_t check_local_plan_args(tebgpu_ctx* ctx, const TebBatch* bt, const TebLocalPlanArgs* la) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  if (!bt || !la) { ctx->err = "batch or local plan args == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->B < 1 || bt->S < 1) { ctx->err = "bad batch dimensions"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->B > ctx->lim.max_bands || bt->S > ctx->lim.max_scenes) { ctx->err = "batch exceeds the context limits"; return TEBGPU_ERR_CAPACITY; }
  if (la->G_cap < 1 || la->P_cap < 2 || la->V_cap < 0) { ctx->err = "bad local plan strides"; return TEBGPU_ERR_INVALID_ARG; }
  if (!bt->scene_id || !la->global_plan || !la->plan_begin || !la->plan_end || !la->robot || !la->robot_vel || !la->grid ||
      !la->origin || !la->plan || !la->plan_count || !la->result || (la->via && !la->via_count)) {
    ctx->err = "missing required local plan array"; return TEBGPU_ERR_INVALID_ARG;
  }
  if (!ctx->have_params) { ctx->err = "tebgpu_set_params has not been called"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

/* k_local_plan on arguments already checked; fr NULL or without plan transforms: the identity transform */
static int32_t issue_local_plan(tebgpu_ctx* ctx, const TebBatch* bt, const TebLocalPlanArgs* la, const TebFrameArgs* fr,
                                cudaStream_t st) {
  const long long grid = ((long long)bt->B * 32 + LPLAN_THREADS - 1) / LPLAN_THREADS;
  TebFrameArgs f{};
  if (fr) f = *fr;
  if (f.costmap_to_plan)
    k_local_plan<true><<<(unsigned)grid, LPLAN_THREADS, 0, st>>>(*la, f, bt->scene_id, bt->B, bt->S,
                                                                 ctx->params.global_plan_overwrite_orientation);
  else
    k_local_plan<false><<<(unsigned)grid, LPLAN_THREADS, 0, st>>>(*la, f, bt->scene_id, bt->B, bt->S,
                                                                  ctx->params.global_plan_overwrite_orientation);
  ctx->last_lplan_grid = grid;
  ctx->launches = 1;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

int32_t tebgpu_local_plan_tf_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebLocalPlanArgs* la,
                                    const TebFrameArgs* fr, void* cuda_stream) {
  int32_t rc = check_local_plan_args(ctx, bt, la);
  if (rc || (rc = check_frame_args(ctx, fr))) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_local_plan(ctx, bt, la, fr, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

int32_t tebgpu_local_plan_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebLocalPlanArgs* la, void* cuda_stream) {
  return tebgpu_local_plan_tf_device(ctx, bt, la, nullptr, cuda_stream);
}

int32_t tebgpu_local_plan(tebgpu_ctx* ctx, const TebBatch* bt, const TebLocalPlanArgs* la) {
  return tebgpu_local_plan_tf(ctx, bt, la, nullptr);
}

int32_t tebgpu_local_plan_tf(tebgpu_ctx* ctx, const TebBatch* bt, const TebLocalPlanArgs* la, const TebFrameArgs* fr) {
  int32_t rc = check_local_plan_args(ctx, bt, la);
  if (rc || (rc = check_frame_args(ctx, fr))) return rc;
  const bool tf = fr && fr->costmap_to_plan;
  /* the bands the device entry point would answer with TEB_LOCAL_PLAN_BAD_INPUT are refused here, before anything runs */
  for (int b = 0; b < bt->B; ++b) {
    if (la->plan_begin[b] < 0 || la->plan_begin[b] > la->plan_end[b] || la->plan_end[b] > la->G_cap) {
      ctx->err = "plan_begin / plan_end outside 0 .. G_cap"; return TEBGPU_ERR_INVALID_ARG;
    }
    if (bt->scene_id[b] < 0 || bt->scene_id[b] >= bt->S) { ctx->err = "scene_id[b] outside 0 .. S-1"; return TEBGPU_ERR_INVALID_ARG; }
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t B = bt->B, S = bt->S, G = la->G_cap, P = la->P_cap, V = la->V_cap;
  /* one staging buffer: every array at a 256-byte aligned offset */
  size_t off = 0;
  auto slot = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  const size_t o_gp = slot(B * G * 3 * sizeof(double)), o_begin = slot(B * 4), o_end = slot(B * 4),
               o_robot = slot(B * 3 * sizeof(double)), o_vel = slot(B * 3 * sizeof(double)), o_grid = slot(S * 2 * 4),
               o_origin = slot(S * 3 * sizeof(double)), o_sid = slot(B * 4), o_inf = slot(la->infeasible_count ? B * 4 : 0),
               o_since = slot(la->since_infeasible ? B * sizeof(double) : 0), o_plan = slot(B * P * 3 * sizeof(double)),
               o_pcount = slot(B * 4), o_goal = slot(B * 4), o_via = slot(la->via ? B * V * 2 * sizeof(double) : 0),
               o_vcount = slot(B * 4), o_result = slot(B * 4), o_needed = slot(B * 2 * 4),
               o_c2p = slot(tf ? B * 7 * sizeof(double) : 0), o_p2c = slot(tf ? B * 7 * sizeof(double) : 0);
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_lplan, &ctx->lplan_bytes, off, st))) return rc;
  char* d = ctx->d_lplan;
  auto up = [&](size_t o, const void* src, size_t bytes) -> int32_t {
    if (src && bytes) CUDA_TRY(ctx, cudaMemcpyAsync(d + o, src, bytes, cudaMemcpyHostToDevice, st));
    return TEBGPU_OK;
  };
  /* the outputs a band may leave unwritten go up too, so that they come back as the caller left them */
  if ((rc = up(o_gp, la->global_plan, B * G * 3 * sizeof(double))) || (rc = up(o_begin, la->plan_begin, B * 4)) ||
      (rc = up(o_end, la->plan_end, B * 4)) || (rc = up(o_robot, la->robot, B * 3 * sizeof(double))) ||
      (rc = up(o_vel, la->robot_vel, B * 3 * sizeof(double))) || (rc = up(o_grid, la->grid, S * 2 * 4)) ||
      (rc = up(o_origin, la->origin, S * 3 * sizeof(double))) || (rc = up(o_sid, bt->scene_id, B * 4)) ||
      (rc = up(o_inf, la->infeasible_count, B * 4)) || (rc = up(o_since, la->since_infeasible, B * sizeof(double))) ||
      (rc = up(o_goal, la->goal_idx, B * 4)) || (rc = up(o_vcount, la->via_count, B * 4)) ||
      (rc = up(o_needed, la->needed, B * 2 * 4)))
    return rc;
  TebFrameArgs df{};
  if (tf) {
    if ((rc = up(o_c2p, fr->costmap_to_plan, B * 7 * sizeof(double))) || (rc = up(o_p2c, fr->plan_to_costmap, B * 7 * sizeof(double))))
      return rc;
    df.costmap_to_plan = (const double*)(d + o_c2p);
    df.plan_to_costmap = (const double*)(d + o_p2c);
  }
  TebBatch db = *bt;
  db.scene_id = (const int32_t*)(d + o_sid);
  TebLocalPlanArgs da = *la;
  da.global_plan = (const double*)(d + o_gp);
  da.plan_begin = (int32_t*)(d + o_begin); da.plan_end = (const int32_t*)(d + o_end);
  da.robot = (const double*)(d + o_robot); da.robot_vel = (const double*)(d + o_vel);
  da.grid = (const int32_t*)(d + o_grid); da.origin = (const double*)(d + o_origin);
  da.infeasible_count = la->infeasible_count ? (const int32_t*)(d + o_inf) : nullptr;
  da.since_infeasible = la->since_infeasible ? (const double*)(d + o_since) : nullptr;
  da.plan = (double*)(d + o_plan); da.plan_count = (int32_t*)(d + o_pcount);
  da.goal_idx = la->goal_idx ? (int32_t*)(d + o_goal) : nullptr;
  da.via = la->via ? (double*)(d + o_via) : nullptr;
  da.via_count = la->via_count ? (int32_t*)(d + o_vcount) : nullptr;
  da.result = (int32_t*)(d + o_result);
  da.needed = la->needed ? (int32_t*)(d + o_needed) : nullptr;
  if ((rc = issue_local_plan(ctx, &db, &da, tf ? &df : nullptr, st))) return rc;
  auto down = [&](void* dst, size_t o, size_t bytes) -> int32_t {
    if (dst && bytes) CUDA_TRY(ctx, cudaMemcpyAsync(dst, d + o, bytes, cudaMemcpyDeviceToHost, st));
    return TEBGPU_OK;
  };
  if ((rc = down(la->plan_begin, o_begin, B * 4)) || (rc = down(la->plan_count, o_pcount, B * 4)) ||
      (rc = down(la->goal_idx, o_goal, B * 4)) || (rc = down(la->via ? la->via_count : nullptr, o_vcount, B * 4)) ||
      (rc = down(la->result, o_result, B * 4)) || (rc = down(la->needed, o_needed, B * 2 * 4)))
    return rc;
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  /* only the rows the kernel wrote reach the caller: plan_count plan rows, and via_count via-points of a band whose
   * via-points were written */
  std::vector<double> h(B * P * 3);
  CUDA_TRY(ctx, cudaMemcpy(h.data(), d + o_plan, h.size() * sizeof(double), cudaMemcpyDeviceToHost));
  for (size_t b = 0; b < B; ++b)
    std::memcpy(la->plan + b * P * 3, h.data() + b * P * 3, (size_t)std::max(la->plan_count[b], 0) * 3 * sizeof(double));
  if (la->via && V) {
    h.resize(B * V * 2);
    CUDA_TRY(ctx, cudaMemcpy(h.data(), d + o_via, h.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t b = 0; b < B; ++b)
      if (la->result[b] == TEB_LOCAL_PLAN_PLANNED || la->result[b] == TEB_LOCAL_PLAN_GOAL_REACHED)
        std::memcpy(la->via + b * V * 2, h.data() + b * V * 2, (size_t)std::max(la->via_count[b], 0) * 2 * sizeof(double));
  }
  return TEBGPU_OK;
}

/* the context parameters the controller steps read */
static TebCycleLimits cycle_limits(const TebParams& p) {
  TebCycleLimits L;
  L.max_vel_x = p.max_vel_x; L.max_vel_x_backwards = p.max_vel_x_backwards; L.max_vel_y = p.max_vel_y;
  L.max_vel_trans = p.max_vel_trans; L.max_vel_theta = p.max_vel_theta; L.min_turning_radius = p.min_turning_radius;
  L.divergence_max_chi2 = p.divergence_detection_max_chi_squared;
  L.divergence_enable = p.divergence_detection_enable;
  return L;
}

/* argument checks of the four controller-step entry points: nothing is launched when one fails */
static int32_t check_cycle_args(tebgpu_ctx* ctx, const TebBatch* bt, const TebCycleArgs* ca, bool finish) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  if (!bt || !ca) { ctx->err = "batch or cycle args == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->B < 1 || bt->B > ctx->lim.max_bands) { ctx->err = "B outside 1 .. max_bands"; return TEBGPU_ERR_INVALID_ARG; }
  if (ca->L_cap < 0 || ca->buffer_length < 0 || ca->buffer_length > ca->L_cap) {
    ctx->err = "buffer_length outside 0 .. L_cap"; return TEBGPU_ERR_INVALID_ARG;
  }
  if (!std::isfinite(ca->now)) { ctx->err = "now is not finite"; return TEBGPU_ERR_INVALID_ARG; }
  const bool missing = finish ? (!bt->n || !bt->status || !bt->chi2 || !ca->cmd || !ca->infeasible_count ||
                                 !ca->last_infeasible || !ca->last_cmd || !ca->cmd_vel || !ca->outcome)
                              : (!ca->robot_vel || !ca->last_cmd || !ca->prefer_rotdir || !ca->last_oscillation ||
                                 !ca->osc_fill || (ca->buffer_length > 0 && !ca->osc_ring));
  if (missing) { ctx->err = "missing required cycle array"; return TEBGPU_ERR_INVALID_ARG; }
  if (!ctx->have_params) { ctx->err = "tebgpu_set_params has not been called"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

static int32_t issue_cycle(tebgpu_ctx* ctx, TebBatch* bt, const TebCycleArgs* ca, bool finish, cudaStream_t st) {
  const long long grid = ((long long)bt->B + CYCLE_THREADS - 1) / CYCLE_THREADS;
  const TebCycleLimits L = cycle_limits(ctx->params);
  if (finish)
    k_finish_cycle<<<(unsigned)grid, CYCLE_THREADS, 0, st>>>(*ca, L, bt->n, bt->status, bt->chi2, bt->B);
  else
    k_backup_modes<<<(unsigned)grid, CYCLE_THREADS, 0, st>>>(*ca, L, bt->B);
  ctx->last_cycle_grid = grid;
  ctx->launches = 1;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

int32_t tebgpu_backup_modes_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebCycleArgs* ca, void* cuda_stream) {
  const int32_t rc = check_cycle_args(ctx, bt, ca, false);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  TebBatch b = *bt;
  return issue_cycle(ctx, &b, ca, false, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

int32_t tebgpu_finish_cycle_device(tebgpu_ctx* ctx, TebBatch* bt, const TebCycleArgs* ca, void* cuda_stream) {
  const int32_t rc = check_cycle_args(ctx, bt, ca, true);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_cycle(ctx, bt, ca, true, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

/* one array of a host-buffer controller step: staged in ctx->d_cycle at a 256-byte aligned offset, copied up before the
 * launch (so what a band leaves unwritten comes back as the caller left it) and back after it when the step writes it */
struct CycleSlot {
  void* host;
  size_t bytes;
  bool out;
  size_t off;
  char* dev(char* d) const { return host ? d + off : nullptr; }
};

/* both host-buffer controller steps: refuse the bands the device would answer with NO_PLAN / -1, stage, launch, copy back */
static int32_t run_cycle_host(tebgpu_ctx* ctx, TebBatch* bt, const TebCycleArgs* ca, bool finish) {
  int32_t rc = check_cycle_args(ctx, bt, ca, finish);
  if (rc) return rc;
  const size_t B = bt->B;
  for (size_t b = 0; b < B; ++b)
    if (finish ? !teb_cycle_finish_valid(*ca, (int)b) : !teb_cycle_backup_valid(*ca, (int)b)) {
      ctx->err = finish ? "local_plan_result or feasible out of range"
                        : "local_plan_result, prefer_rotdir or osc_fill out of range";
      return TEBGPU_ERR_INVALID_ARG;
    }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t I = sizeof(int32_t), D = sizeof(double);
  enum { LPR, VEL, CMD, FEAS, NCOUNT, STATUS, CHI2, INF, LINF, LOSC, LCMD, ROT, RING, FILL, CVEL, OUTC, OSC, SLOTS };
  CycleSlot s[SLOTS] = {
      {(void*)ca->local_plan_result, B * I, false, 0}, {(void*)ca->robot_vel, B * 3 * D, false, 0},
      {(void*)ca->cmd, B * 4 * D, false, 0},           {(void*)ca->feasible, B * I, false, 0},
      {bt->n, B * I, true, 0},                         {bt->status, B * I, false, 0},
      {bt->chi2, B * D, false, 0},                     {ca->infeasible_count, B * I, true, 0},
      {ca->last_infeasible, B * D, true, 0},           {ca->last_oscillation, B * D, true, 0},
      {ca->last_cmd, B * 3 * D, true, 0},              {ca->prefer_rotdir, B * I, true, 0},
      {ca->osc_ring, (size_t)ca->L_cap * B * 2 * D, true, 0}, {ca->osc_fill, B * 2 * I, true, 0},
      {ca->cmd_vel, B * 3 * D, true, 0},               {ca->outcome, B * I, true, 0},
      {ca->oscillating, B * I, true, 0}};
  /* what the step does not read stays on the host */
  const int used_finish[] = {LPR, CMD, FEAS, NCOUNT, STATUS, CHI2, INF, LINF, LCMD, CVEL, OUTC};
  const int used_backup[] = {LPR, VEL, LCMD, ROT, RING, FILL, LOSC, OSC};
  bool used[SLOTS] = {};
  if (finish) for (int k : used_finish) used[k] = true;
  else for (int k : used_backup) used[k] = true;
  if (!finish) s[LCMD].out = false;
  size_t off = 0;
  for (int k = 0; k < SLOTS; ++k) {
    if (!used[k]) s[k].host = nullptr;
    s[k].off = off;
    if (s[k].host) off += (s[k].bytes + 255) & ~(size_t)255;
  }
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_cycle, &ctx->cycle_bytes, off, st))) return rc;
  char* d = ctx->d_cycle;
  for (const CycleSlot& c : s)
    if (c.host && c.bytes) CUDA_TRY(ctx, cudaMemcpyAsync(d + c.off, c.host, c.bytes, cudaMemcpyHostToDevice, st));
  TebBatch db = *bt;
  db.n = (int32_t*)s[NCOUNT].dev(d); db.status = (int32_t*)s[STATUS].dev(d); db.chi2 = (double*)s[CHI2].dev(d);
  TebCycleArgs da = *ca;
  da.local_plan_result = (const int32_t*)s[LPR].dev(d); da.robot_vel = (const double*)s[VEL].dev(d);
  da.cmd = (const double*)s[CMD].dev(d); da.feasible = (const int32_t*)s[FEAS].dev(d);
  da.infeasible_count = (int32_t*)s[INF].dev(d); da.last_infeasible = (double*)s[LINF].dev(d);
  da.last_oscillation = (double*)s[LOSC].dev(d); da.last_cmd = (double*)s[LCMD].dev(d);
  da.prefer_rotdir = (int32_t*)s[ROT].dev(d); da.osc_ring = (double*)s[RING].dev(d); da.osc_fill = (int32_t*)s[FILL].dev(d);
  da.cmd_vel = (double*)s[CVEL].dev(d); da.outcome = (int32_t*)s[OUTC].dev(d); da.oscillating = (int32_t*)s[OSC].dev(d);
  if ((rc = issue_cycle(ctx, &db, &da, finish, st))) return rc;
  for (const CycleSlot& c : s)
    if (c.host && c.out && c.bytes) CUDA_TRY(ctx, cudaMemcpyAsync(c.host, d + c.off, c.bytes, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

int32_t tebgpu_backup_modes(tebgpu_ctx* ctx, const TebBatch* bt, const TebCycleArgs* ca) {
  if (!bt) return check_cycle_args(ctx, bt, ca, false);
  TebBatch b = *bt;
  return run_cycle_host(ctx, &b, ca, false);
}

int32_t tebgpu_finish_cycle(tebgpu_ctx* ctx, TebBatch* bt, const TebCycleArgs* ca) {
  return run_cycle_host(ctx, bt, ca, true);
}

/* argument checks of both fleet-obstacle entry points: nothing is launched when one fails. arrays: pose, last_cmd and
 * radius are required (not for the table step, which reads none of them) */
static int32_t check_fleet_args(tebgpu_ctx* ctx, const TebFleetArgs* fa, bool arrays = true) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  if (!fa) { ctx->err = "fleet args == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (fa->R < 1 || fa->S < 1 || fa->C_cap < 0) { ctx->err = "bad fleet dimensions"; return TEBGPU_ERR_INVALID_ARG; }
  if (fa->R > ctx->lim.max_bands || fa->S > ctx->lim.max_scenes) { ctx->err = "fleet exceeds the context limits"; return TEBGPU_ERR_CAPACITY; }
  if (fa->max_rows < 0 || fa->max_rows > TEB_FLEET_MAX_ROWS) { ctx->err = "max_rows outside 0 .. TEB_FLEET_MAX_ROWS"; return TEBGPU_ERR_INVALID_ARG; }
  if (!(fa->range >= 0.0)) { ctx->err = "range is NaN or negative"; return TEBGPU_ERR_INVALID_ARG; }
  if ((arrays && (!fa->pose || !fa->last_cmd || !fa->radius)) || !fa->custom_count || (fa->C_cap > 0 && !fa->custom)) {
    ctx->err = "missing required fleet array"; return TEBGPU_ERR_INVALID_ARG;
  }
  if (!fa->scene && fa->R > fa->S) { ctx->err = "scene == NULL with R > S"; return TEBGPU_ERR_INVALID_ARG; }
  if (fa->own_count && (const void*)fa->own_count == (const void*)fa->custom_count) {
    ctx->err = "own_count is custom_count"; return TEBGPU_ERR_INVALID_ARG;
  }
  if (reinterpret_cast<uintptr_t>(fa->custom) & 15) { ctx->err = "custom not 16-byte aligned"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

/* The automatic search takes the grid from FLEET_GRID_N0 candidates (R for the array step, T for the table step) on.
 * tools/fleet_grid.py on one H100 80GB HBM3 at 700 W (DESIGN §8), the uniform square fleet at range 3 m: all pairs
 * 30 us against the grid's 38 us at 2048 robots, 56 us against 35 us at 4096. */
constexpr int64_t FLEET_GRID_N0 = 4096;
constexpr int64_t FLEET_GRID_MAX_N = (int64_t)1 << 28;   /* the grid's buckets are counted in int32 */

/* the search a fleet step over N candidates runs (TEBGPU_FLEET_SEARCH_ALL_PAIRS, _GRID or _ONE_BUCKET) */
static int fleet_search(const tebgpu_ctx* ctx, const TebFleetArgs* fa, int64_t N) {
  if (ctx->fleet_search != TEBGPU_FLEET_SEARCH_AUTO) return ctx->fleet_search;
  const bool pays = N >= FLEET_GRID_N0 && N <= FLEET_GRID_MAX_N && fa->range > FLEET_H_FLOOR &&
                    std::isfinite(fa->range * fa->range);
  return pays ? TEBGPU_FLEET_SEARCH_GRID : TEBGPU_FLEET_SEARCH_ALL_PAIRS;
}

/* the grid of a step over N candidates: scratch grown to fit, counts cleared, then k_fleet_bin, the scan of the counts
 * and k_fleet_scatter; the search kernel follows on the same stream */
static int32_t issue_fleet_grid(tebgpu_ctx* ctx, const TebFleetArgs* fa, cudaStream_t st, const TebFleetTable* table,
                                int64_t N, bool one_bucket, FleetGrid* g) {
  int32_t rc;
  if (N > FLEET_GRID_MAX_N) { ctx->err = "the fleet grid holds at most 2^28 candidates"; return TEBGPU_ERR_CAPACITY; }
  size_t H = 1;
  while (H < 2 * (size_t)N) H <<= 1;
  size_t scan_bytes = 0;
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (int32_t*)nullptr, (int32_t*)nullptr, (int)(H + 1), st));
  const size_t I = sizeof(int32_t);
  const size_t parts[] = {(H + 2) * I, (H + 1) * I, N * I, N * I, N * I, N * I, scan_bytes};
  size_t off[8] = {0}, total = 0;
  for (int k = 0; k < 7; ++k) {
    off[k] = total;
    total += (parts[k] + 255) & ~(size_t)255;
  }
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_fgrid, &ctx->fgrid_bytes, total, st))) return rc;
  char* d = ctx->d_fgrid;
  g->count = (int32_t*)(d + off[0]);
  g->nfar = g->count + H + 1;
  g->start = (int32_t*)(d + off[1]);
  g->key = (int32_t*)(d + off[2]);
  g->rank = (int32_t*)(d + off[3]);
  g->idx = (int32_t*)(d + off[4]);
  g->far = (int32_t*)(d + off[5]);
  g->mask = one_bucket ? 0u : (unsigned)(H - 1);
  g->h = fleet_cell_side(fa->range);
  g->fin2 = fa->range * fa->range < INFINITY;
  const unsigned blocks = (unsigned)((N + CLAIM_THREADS - 1) / CLAIM_THREADS);
  CUDA_TRY(ctx, cudaMemsetAsync(g->count, 0, (H + 2) * I, st));
  if (table) k_fleet_bin<true><<<blocks, CLAIM_THREADS, 0, st>>>(*fa, *table, *g);
  else k_fleet_bin<false><<<blocks, CLAIM_THREADS, 0, st>>>(*fa, TebFleetTable{}, *g);
  CUDA_TRY(ctx, cub::DeviceScan::ExclusiveSum(d + off[6], scan_bytes, g->count, g->start, (int)(H + 1), st));
  k_fleet_scatter<<<blocks, CLAIM_THREADS, 0, st>>>((int)N, *g);
  return TEBGPU_OK;
}

/* k_fleet_claim (when scenes are given), then k_fleet_obstacles or the grid and k_fleet_obstacles_grid, on arguments
 * already checked; table: the candidates of tebgpu_fleet_obstacles_table, NULL for the caller's arrays */
static int32_t issue_fleet(tebgpu_ctx* ctx, const TebFleetArgs* fa, cudaStream_t st, const TebFleetTable* table = nullptr) {
  int32_t rc;
  const int64_t N = table ? table->T : fa->R;
  const int search = fleet_search(ctx, fa, N);
  FleetGrid g{};
  if (search != TEBGPU_FLEET_SEARCH_ALL_PAIRS &&
      (rc = issue_fleet_grid(ctx, fa, st, table, N, search == TEBGPU_FLEET_SEARCH_ONE_BUCKET, &g))) return rc;
  const int32_t* claims = nullptr;
  if (fa->scene) {
    if ((rc = grow_mirror(ctx, (void**)&ctx->d_fclaim, &ctx->fclaim_bytes, (size_t)fa->S * sizeof(int32_t), st))) return rc;
    CUDA_TRY(ctx, cudaMemsetAsync(ctx->d_fclaim, 0, (size_t)fa->S * sizeof(int32_t), st));
    k_fleet_claim<<<(unsigned)((fa->R + CLAIM_THREADS - 1) / CLAIM_THREADS), CLAIM_THREADS, 0, st>>>(*fa, ctx->d_fclaim);
    claims = ctx->d_fclaim;
  }
  const long long grid = ((long long)fa->R + FLEET_WARPS - 1) / FLEET_WARPS;
  if (search == TEBGPU_FLEET_SEARCH_ALL_PAIRS) {
    if (table) k_fleet_obstacles<true><<<(unsigned)grid, FLEET_THREADS, 0, st>>>(*fa, claims, *table);
    else k_fleet_obstacles<false><<<(unsigned)grid, FLEET_THREADS, 0, st>>>(*fa, claims, TebFleetTable{});
  } else {
    if (table) k_fleet_obstacles_grid<true><<<(unsigned)grid, FLEET_THREADS, 0, st>>>(*fa, claims, *table, g);
    else k_fleet_obstacles_grid<false><<<(unsigned)grid, FLEET_THREADS, 0, st>>>(*fa, claims, TebFleetTable{}, g);
  }
  ctx->last_fleet_grid = grid;
  ctx->last_fleet_search = search;
  /* the grid: k_fleet_bin, DeviceScan's init and scan kernels, k_fleet_scatter */
  ctx->launches = (fa->scene ? 2 : 1) + (search == TEBGPU_FLEET_SEARCH_ALL_PAIRS ? 0 : 4);
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

int32_t tebgpu_fleet_obstacles_device(tebgpu_ctx* ctx, const TebFleetArgs* fa, void* cuda_stream) {
  const int32_t rc = check_fleet_args(ctx, fa);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_fleet(ctx, fa, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

static int32_t run_fleet_host(tebgpu_ctx* ctx, const TebFleetArgs* fa, const TebFleetTable* table);

int32_t tebgpu_fleet_obstacles(tebgpu_ctx* ctx, const TebFleetArgs* fa) {
  int32_t rc = check_fleet_args(ctx, fa);
  if (rc) return rc;
  const size_t R = fa->R, S = fa->S, C = fa->C_cap;
  /* the robots the device entry point would answer with BAD_INPUT / SHARED_SCENE, and every non-finite input, are
   * refused here, before anything runs */
  std::vector<char> taken(S, 0);
  for (size_t r = 0; r < R; ++r) {
    const double* p = fa->pose + 3 * r;
    const double* c = fa->last_cmd + 3 * r;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) { ctx->err = "pose[r] not finite"; return TEBGPU_ERR_INVALID_ARG; }
    if (!std::isfinite(c[0]) || !std::isfinite(c[1])) { ctx->err = "last_cmd[r] not finite"; return TEBGPU_ERR_INVALID_ARG; }
    if (!std::isfinite(fa->radius[r]) || fa->radius[r] < 0.0) { ctx->err = "radius[r] negative or not finite"; return TEBGPU_ERR_INVALID_ARG; }
    const int32_t s = fa->scene ? fa->scene[r] : (int32_t)r;
    if (s < 0 || (size_t)s >= S) { ctx->err = "scene[r] outside 0 .. S-1"; return TEBGPU_ERR_INVALID_ARG; }
    if (taken[s]) { ctx->err = "two robots in one scene"; return TEBGPU_ERR_INVALID_ARG; }
    taken[s] = 1;
    const int32_t own = fa->own_count ? fa->own_count[s] : 0;
    if (own < 0 || (size_t)own > C) { ctx->err = "own_count[s] outside 0 .. C_cap"; return TEBGPU_ERR_INVALID_ARG; }
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return run_fleet_host(ctx, fa, nullptr);
}

/* the host-buffer fleet steps on arguments already checked: stage the arrays given (NULL ones stay NULL), launch on the
 * context's stream, copy the outputs back and synchronise. table: the device copy of the candidates' table, or NULL */
static int32_t run_fleet_host(tebgpu_ctx* ctx, const TebFleetArgs* fa, const TebFleetTable* table) {
  int32_t rc;
  const size_t R = fa->R, S = fa->S, C = fa->C_cap;
  cudaStream_t st = ctx->stream;
  const size_t I = sizeof(int32_t), D = sizeof(double);
  enum { POSE, CMD, RAD, WORLD, SCENE, OWN, CUSTOM, CCOUNT, NEED, STATUS, SLOTS };
  CycleSlot sl[SLOTS] = {
      {(void*)fa->pose, R * 3 * D, false, 0},      {(void*)fa->last_cmd, R * 3 * D, false, 0},
      {(void*)fa->radius, R * D, false, 0},        {(void*)fa->world, R * I, false, 0},
      {(void*)fa->scene, R * I, false, 0},         {(void*)fa->own_count, S * I, false, 0},
      {fa->custom, S * C * sizeof(TebObstacle), true, 0}, {fa->custom_count, S * I, true, 0},
      {fa->needed, R * I, true, 0},                {fa->status, R * I, true, 0}};
  size_t off = 0;
  for (CycleSlot& c : sl) {
    c.off = off;
    if (c.host) off += (c.bytes + 255) & ~(size_t)255;
  }
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_fleet, &ctx->fleet_bytes, off, st))) return rc;
  char* d = ctx->d_fleet;
  /* the outputs go up too, so what the step leaves unwritten comes back as the caller left it */
  for (const CycleSlot& c : sl)
    if (c.host && c.bytes) CUDA_TRY(ctx, cudaMemcpyAsync(d + c.off, c.host, c.bytes, cudaMemcpyHostToDevice, st));
  TebFleetArgs da = *fa;
  da.pose = (const double*)sl[POSE].dev(d); da.last_cmd = (const double*)sl[CMD].dev(d);
  da.radius = (const double*)sl[RAD].dev(d); da.world = (const int32_t*)sl[WORLD].dev(d);
  da.scene = (const int32_t*)sl[SCENE].dev(d); da.own_count = (const int32_t*)sl[OWN].dev(d);
  da.custom = (TebObstacle*)sl[CUSTOM].dev(d); da.custom_count = (int32_t*)sl[CCOUNT].dev(d);
  da.needed = (int32_t*)sl[NEED].dev(d); da.status = (int32_t*)sl[STATUS].dev(d);
  if ((rc = issue_fleet(ctx, &da, st, table))) return rc;
  for (const CycleSlot& c : sl)
    if (c.host && c.out && c.bytes) CUDA_TRY(ctx, cudaMemcpyAsync(c.host, d + c.off, c.bytes, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

/* the table checks of the fleet-table entry points: rows first .. first + R - 1 lie in the table */
static int32_t check_fleet_table(tebgpu_ctx* ctx, const TebFleetArgs* fa, const TebFleetTable* t) {
  if (!t || !t->rows) { ctx->err = "fleet table or its rows == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (t->T < 1 || t->first < 0 || (int64_t)t->first + fa->R > t->T) {
    ctx->err = "fleet table rows first .. first + R - 1 outside 0 .. T - 1"; return TEBGPU_ERR_INVALID_ARG;
  }
  if (reinterpret_cast<uintptr_t>(t->rows) & 15) { ctx->err = "fleet table rows not 16-byte aligned"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

static int32_t check_fleet_publish_args(tebgpu_ctx* ctx, const TebFleetArgs* fa, const TebFleetTable* t) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  if (!fa) { ctx->err = "fleet args == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (fa->R < 1) { ctx->err = "bad fleet dimensions"; return TEBGPU_ERR_INVALID_ARG; }
  if (fa->R > ctx->lim.max_bands) { ctx->err = "fleet exceeds the context limits"; return TEBGPU_ERR_CAPACITY; }
  if (!fa->pose || !fa->last_cmd || !fa->radius) { ctx->err = "missing required fleet array"; return TEBGPU_ERR_INVALID_ARG; }
  return check_fleet_table(ctx, fa, t);
}

static int32_t issue_fleet_publish(tebgpu_ctx* ctx, const TebFleetArgs* fa, const TebFleetTable* t, cudaStream_t st) {
  k_fleet_publish<<<(unsigned)((fa->R + CLAIM_THREADS - 1) / CLAIM_THREADS), CLAIM_THREADS, 0, st>>>(*fa, *t);
  ctx->launches = 1;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

int32_t tebgpu_fleet_publish_device(tebgpu_ctx* ctx, const TebFleetArgs* fa, const TebFleetTable* t, void* cuda_stream) {
  const int32_t rc = check_fleet_publish_args(ctx, fa, t);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_fleet_publish(ctx, fa, t, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

int32_t tebgpu_fleet_publish(tebgpu_ctx* ctx, const TebFleetArgs* fa, const TebFleetTable* t) {
  int32_t rc = check_fleet_publish_args(ctx, fa, t);
  if (rc) return rc;
  const size_t R = fa->R, I = sizeof(int32_t), D = sizeof(double);
  for (size_t r = 0; r < R; ++r) {
    const double* p = fa->pose + 3 * r;
    const double* c = fa->last_cmd + 3 * r;
    if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) { ctx->err = "pose[r] not finite"; return TEBGPU_ERR_INVALID_ARG; }
    if (!std::isfinite(c[0]) || !std::isfinite(c[1])) { ctx->err = "last_cmd[r] not finite"; return TEBGPU_ERR_INVALID_ARG; }
    if (!std::isfinite(fa->radius[r]) || fa->radius[r] < 0.0) { ctx->err = "radius[r] negative or not finite"; return TEBGPU_ERR_INVALID_ARG; }
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  /* the robots' rows only: the device table is rows first .. first + R - 1 of the caller's */
  const size_t rows_bytes = R * sizeof(TebFleetRow);
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_ftable, &ctx->ftable_bytes, rows_bytes, st))) return rc;
  enum { POSE, CMD, RAD, WORLD, SLOTS };
  CycleSlot sl[SLOTS] = {{(void*)fa->pose, R * 3 * D, false, 0}, {(void*)fa->last_cmd, R * 3 * D, false, 0},
                         {(void*)fa->radius, R * D, false, 0},   {(void*)fa->world, R * I, false, 0}};
  size_t off = 0;
  for (CycleSlot& c : sl) {
    c.off = off;
    if (c.host) off += (c.bytes + 255) & ~(size_t)255;
  }
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_fleet, &ctx->fleet_bytes, off, st))) return rc;
  char* d = ctx->d_fleet;
  for (const CycleSlot& c : sl)
    if (c.host && c.bytes) CUDA_TRY(ctx, cudaMemcpyAsync(d + c.off, c.host, c.bytes, cudaMemcpyHostToDevice, st));
  TebFleetArgs da = *fa;
  da.pose = (const double*)sl[POSE].dev(d); da.last_cmd = (const double*)sl[CMD].dev(d);
  da.radius = (const double*)sl[RAD].dev(d); da.world = (const int32_t*)sl[WORLD].dev(d);
  const TebFleetTable dt = {(int32_t)R, 0, ctx->d_ftable};
  if ((rc = issue_fleet_publish(ctx, &da, &dt, st))) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(t->rows + t->first, ctx->d_ftable, rows_bytes, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

int32_t tebgpu_fleet_obstacles_table_device(tebgpu_ctx* ctx, const TebFleetArgs* fa, const TebFleetTable* t,
                                            void* cuda_stream) {
  int32_t rc = check_fleet_args(ctx, fa, false);
  if (rc || (rc = check_fleet_table(ctx, fa, t))) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_fleet(ctx, fa, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream, t);
}

int32_t tebgpu_fleet_obstacles_table(tebgpu_ctx* ctx, const TebFleetArgs* fa, const TebFleetTable* t) {
  int32_t rc = check_fleet_args(ctx, fa, false);
  if (rc || (rc = check_fleet_table(ctx, fa, t))) return rc;
  const size_t R = fa->R, S = fa->S, C = fa->C_cap, T = t->T;
  /* what the device entry point would answer with BAD_INPUT / SHARED_SCENE, and every non-finite live row, are refused
   * here, before anything runs */
  for (size_t q = 0; q < T; ++q) {
    const TebFleetRow& w = t->rows[q];
    if (!w.live) continue;
    if (!std::isfinite(w.x) || !std::isfinite(w.y) || !std::isfinite(w.vx) || !std::isfinite(w.vy)) {
      ctx->err = "live fleet row not finite"; return TEBGPU_ERR_INVALID_ARG;
    }
    if (!std::isfinite(w.radius) || w.radius < 0.0) { ctx->err = "live fleet row radius negative or not finite"; return TEBGPU_ERR_INVALID_ARG; }
  }
  std::vector<char> taken(S, 0);
  for (size_t r = 0; r < R; ++r) {
    if (!t->rows[t->first + r].live) { ctx->err = "the robot's own fleet row is not live"; return TEBGPU_ERR_INVALID_ARG; }
    const int32_t s = fa->scene ? fa->scene[r] : (int32_t)r;
    if (s < 0 || (size_t)s >= S) { ctx->err = "scene[r] outside 0 .. S-1"; return TEBGPU_ERR_INVALID_ARG; }
    if (taken[s]) { ctx->err = "two robots in one scene"; return TEBGPU_ERR_INVALID_ARG; }
    taken[s] = 1;
    const int32_t own = fa->own_count ? fa->own_count[s] : 0;
    if (own < 0 || (size_t)own > C) { ctx->err = "own_count[s] outside 0 .. C_cap"; return TEBGPU_ERR_INVALID_ARG; }
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t bytes = T * sizeof(TebFleetRow);
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_ftable, &ctx->ftable_bytes, bytes, st))) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_ftable, t->rows, bytes, cudaMemcpyHostToDevice, st));
  const TebFleetTable dt = {t->T, t->first, ctx->d_ftable};
  TebFleetArgs ha = *fa;
  ha.pose = ha.last_cmd = ha.radius = nullptr;
  ha.world = nullptr;
  return run_fleet_host(ctx, &ha, &dt);
}

int32_t tebgpu_compute_cost(tebgpu_ctx* ctx, const TebBatch* bt, const TebOptimizeArgs* args) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  if (!args) return TEBGPU_ERR_INVALID_ARG;
  rc = check_path(ctx, bt, false);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rc = upload_batch(ctx, bt);
  if (rc) return rc;
  TebBatch d = mirror_batch(ctx, bt);
  cudaStream_t st = ctx->stream;
  DevBatch db = make_devbatch(ctx, &d);
  KParams kp = make_kparams(ctx, bt, 1.0); /* buildGraph() default weight_multiplier (optimal_planner.h:536) */
  const int B = bt->B, tb = 128, gb = ((B > bt->S ? B : bt->S) + tb - 1) / tb;
  k_begin<<<gb, tb, 0, st>>>(db, kp);
  launch_build_graph(db, kp, B, (size_t)(bt->M_cap > 0 ? bt->M_cap : 1) * sizeof(TebObstacle), st);
  launch_linearize(ctx, db, kp, B, bt->M_cap, st);
  if (kp.has_vor) launch_vor(db, kp, B, (size_t)(bt->M_cap > 0 ? bt->M_cap : 1) * sizeof(TebObstacle), st);
  k_cost_only<<<gb, tb, 0, st>>>(db, kp, *args);
  ctx->launches = 4;
  CUDA_TRY(ctx, cudaGetLastError());
  if (bt->cost) CUDA_TRY(ctx, cudaMemcpyAsync(bt->cost, ctx->d_cost, (size_t)B * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (bt->chi2) CUDA_TRY(ctx, cudaMemcpyAsync(bt->chi2, ctx->d_chi2, (size_t)B * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (bt->status) CUDA_TRY(ctx, cudaMemcpyAsync(bt->status, ctx->d_status, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

int32_t tebgpu_h_signature(tebgpu_ctx* ctx, const TebBatch* bt, int32_t use_timediffs, double* h_out, int32_t device_ptrs) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  if (!h_out) return TEBGPU_ERR_INVALID_ARG;
  /* The 2-D signature's product over the M - 1 obstacle differences (long double in the reference) is carried as an
   * fp64 mantissa and a binary exponent, so its range is not what limits M. What does is the O(M^2) product per band,
   * one CTA per band, and the staged table in shared memory: larger scenes need a design of their own (DESIGN §9). */
  if (global_table(bt->M_cap)) { ctx->err = "the H-signature supports at most 1024 obstacles per scene"; return TEBGPU_ERR_UNSUPPORTED; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  TebBatch d = *bt;
  if (!device_ptrs) {
    rc = upload_batch(ctx, bt);
    if (rc) return rc;
    d = mirror_batch(ctx, bt);
  }
  cudaStream_t st = ctx->stream;
  DevBatch db = make_devbatch(ctx, &d);
  KParams kp = make_kparams(ctx, bt, 1.0);
  const int B = bt->B;
  const bool three_d = ctx->params.include_dynamic_obstacles != 0; /* homotopy_class_planner.hpp:50 */
  const size_t stride = three_d ? (size_t)(bt->M_cap > 0 ? bt->M_cap : 1) : 2;
  const size_t smem = hsig_smem_bytes(bt->n_cap, bt->M_cap);
  if (smem > 232448) { ctx->err = "h-signature staging exceeds shared memory"; return TEBGPU_ERR_CAPACITY; }
  double* d_out = device_ptrs ? h_out : ctx->d_hsig; /* [B][stride] <= [max_bands][max(max_obstacles, 2)] */
  if (three_d) {
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_hsig3d, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_hsig3d<<<B, HSIG_THREADS, smem, st>>>(db, kp, use_timediffs, d_out);
  } else {
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_hsig2d, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_hsig2d<<<B, HSIG_THREADS, smem, st>>>(db, kp, d_out);
  }
  ctx->launches = 1;
  CUDA_TRY(ctx, cudaGetLastError());
  if (!device_ptrs) {
    CUDA_TRY(ctx, cudaMemcpyAsync(h_out, d_out, (size_t)B * stride * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaStreamSynchronize(st));
  }
  return TEBGPU_OK;
}

/* argument checks of both factor-table entry points: only S, M_cap, obstacles and obst_count of the batch are read */
static int32_t check_hsig_factors_args(tebgpu_ctx* ctx, const TebBatch* bt, const TebHsigFactors* f) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  if (!bt || !f) { ctx->err = "batch or factors == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->S < 1 || bt->M_cap < 0) { ctx->err = "bad batch dimensions"; return TEBGPU_ERR_INVALID_ARG; }
  if (bt->S > ctx->lim.max_scenes || bt->M_cap > ctx->lim.max_obstacles) { ctx->err = "batch exceeds the context limits"; return TEBGPU_ERR_CAPACITY; }
  if (!bt->obst_count || (bt->M_cap > 0 && !bt->obstacles)) { ctx->err = "missing required batch array"; return TEBGPU_ERR_INVALID_ARG; }
  if (!f->factor || !f->factor_exp || !f->factor_count) { ctx->err = "missing factor table array"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

/* k_hsig_factors + k_hsig_factors_combine on device arrays, arguments already checked */
static int32_t issue_hsig_factors(tebgpu_ctx* ctx, const TebBatch* d, const TebHsigFactors* f, cudaStream_t st) {
  const int S = d->S, M_cap = d->M_cap, P_cap = hsig_parts(M_cap), lb = (M_cap + HSF_THREADS - 1) / HSF_THREADS;
  const size_t cells = (size_t)S * P_cap * M_cap;
  int32_t rc;
  ctx->launches = 0;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_hsf_part, &ctx->hsf_part_bytes, cells * (sizeof(double2) + sizeof(int)) + 16, st))) return rc;
  double2* pm = reinterpret_cast<double2*>(ctx->d_hsf_part);
  int* pe = reinterpret_cast<int*>(pm + cells);
  if (M_cap > 0) {
    k_hsig_factors<<<dim3(S, lb * P_cap), HSF_THREADS, 0, st>>>(d->obstacles, d->obst_count, M_cap, pm, pe);
    ++ctx->launches;
  }
  k_hsig_factors_combine<<<dim3(S, lb > 0 ? lb : 1), HSF_THREADS, 0, st>>>(d->obst_count, M_cap, pm, pe, f->factor,
                                                                             f->factor_exp, f->factor_count);
  ++ctx->launches;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

/* the in-call factor table of S x M_cap rows in ctx->d_hsf_tab */
static int32_t hsig_table_scratch(tebgpu_ctx* ctx, int S, int M_cap, TebHsigFactors* t, cudaStream_t st) {
  const size_t rows = (size_t)S * M_cap;
  int32_t rc = grow_mirror(ctx, (void**)&ctx->d_hsf_tab, &ctx->hsf_tab_bytes,
                           rows * 2 * sizeof(double) + rows * sizeof(int32_t) + (size_t)S * sizeof(int32_t) + 16, st);
  if (rc) return rc;
  t->factor = reinterpret_cast<double*>(ctx->d_hsf_tab);
  t->factor_exp = reinterpret_cast<int32_t*>(t->factor + 2 * rows);
  t->factor_count = t->factor_exp + rows;
  return TEBGPU_OK;
}

int32_t tebgpu_hsig_factors_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebHsigFactors* factors, void* cuda_stream) {
  const int32_t rc = check_hsig_factors_args(ctx, bt, factors);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_hsig_factors(ctx, bt, factors, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

int32_t tebgpu_hsig_factors(tebgpu_ctx* ctx, const TebBatch* bt, const TebHsigFactors* factors) {
  int32_t rc = check_hsig_factors_args(ctx, bt, factors);
  if (rc) return rc;
  for (int sc = 0; sc < bt->S; ++sc)
    if (bt->obst_count[sc] < 0 || bt->obst_count[sc] > bt->M_cap) { ctx->err = "obst_count[s] outside 0 .. M_cap"; return TEBGPU_ERR_INVALID_ARG; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t S = bt->S, rows = S * bt->M_cap;
  if (rows) CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_obst, bt->obstacles, rows * sizeof(TebObstacle), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_ocount, bt->obst_count, S * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  TebBatch d = *bt;
  d.obstacles = ctx->d_obst; d.obst_count = ctx->d_ocount;
  TebHsigFactors t{};
  if ((rc = hsig_table_scratch(ctx, bt->S, bt->M_cap, &t, st))) return rc;
  if ((rc = issue_hsig_factors(ctx, &d, &t, st))) return rc;
  if (rows) {
    CUDA_TRY(ctx, cudaMemcpyAsync(factors->factor, t.factor, rows * 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(factors->factor_exp, t.factor_exp, rows * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(factors->factor_count, t.factor_count, S * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

/* the signatures of every band of d (device arrays, batch checked); f: a device factor table, or NULL: built here */
static int32_t issue_hsig_scenes(tebgpu_ctx* ctx, const TebBatch* d, const TebHsigFactors* f, int32_t use_timediffs,
                                 double* out, cudaStream_t st) {
  DevBatch db = make_devbatch(ctx, d);
  KParams kp = make_kparams(ctx, d, 1.0);
  const int B = d->B, Mc = d->M_cap > 0 ? d->M_cap : 1;
  int32_t rc;
  if (ctx->params.include_dynamic_obstacles) { /* homotopy_class_planner.hpp:50 */
    const size_t smem = (size_t)3 * d->n_cap * sizeof(double);
    k_hsig3d_scene<<<dim3(B, (Mc + HS3_ROWS - 1) / HS3_ROWS), 256, smem, st>>>(db, kp, use_timediffs, out);
    ctx->launches = 1;
    CUDA_TRY(ctx, cudaGetLastError());
    return TEBGPU_OK;
  }
  TebHsigFactors t{};
  int64_t launches = 0;
  if (!f) {
    if ((rc = hsig_table_scratch(ctx, d->S, d->M_cap, &t, st))) return rc;
    if ((rc = issue_hsig_factors(ctx, d, &t, st))) return rc;
    launches = ctx->launches;
    f = &t;
  }
  const int C_cap = (Mc + HS2_ROWS - 1) / HS2_ROWS;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_hs_part, &ctx->hs_part_bytes, (size_t)B * C_cap * 3 * sizeof(double), st))) return rc;
  const size_t smem = (size_t)2 * d->n_cap * sizeof(double);
  k_hsig2d_scene<<<dim3(B, C_cap), HS2_ROWS, smem, st>>>(db, kp, f->factor, f->factor_exp, f->factor_count, ctx->d_hs_part);
  k_hsig2d_scene_sum<<<(B + 127) / 128, 128, 0, st>>>(db, f->factor_count, ctx->d_hs_part, out);
  ctx->launches = launches + 2;
  CUDA_TRY(ctx, cudaGetLastError());
  return TEBGPU_OK;
}

int32_t tebgpu_h_signature_scenes_device(tebgpu_ctx* ctx, const TebBatch* bt, const TebHsigFactors* factors,
                                         int32_t use_timediffs, double* h_out, void* cuda_stream) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  if (!h_out) { ctx->err = "h_out == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (factors && (!factors->factor || !factors->factor_exp || !factors->factor_count)) { ctx->err = "missing factor table array"; return TEBGPU_ERR_INVALID_ARG; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  return issue_hsig_scenes(ctx, bt, factors, use_timediffs, h_out, cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream);
}

int32_t tebgpu_h_signature_scenes(tebgpu_ctx* ctx, const TebBatch* bt, const TebHsigFactors* factors,
                                  int32_t use_timediffs, double* h_out) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  if (!h_out) { ctx->err = "h_out == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  const bool three_d = ctx->params.include_dynamic_obstacles != 0;
  if (factors && !three_d && (!factors->factor || !factors->factor_exp || !factors->factor_count)) { ctx->err = "missing factor table array"; return TEBGPU_ERR_INVALID_ARG; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = upload_batch(ctx, bt))) return rc;
  const TebBatch d = mirror_batch(ctx, bt);
  cudaStream_t st = ctx->stream;
  TebHsigFactors t{};
  const TebHsigFactors* f = nullptr;
  if (factors && !three_d) { /* the caller's table goes up into the in-call table's place */
    const size_t S = bt->S, rows = S * bt->M_cap;
    if ((rc = hsig_table_scratch(ctx, bt->S, bt->M_cap, &t, st))) return rc;
    if (rows) {
      CUDA_TRY(ctx, cudaMemcpyAsync(t.factor, factors->factor, rows * 2 * sizeof(double), cudaMemcpyHostToDevice, st));
      CUDA_TRY(ctx, cudaMemcpyAsync(t.factor_exp, factors->factor_exp, rows * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    }
    CUDA_TRY(ctx, cudaMemcpyAsync(t.factor_count, factors->factor_count, S * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    f = &t;
  }
  const size_t stride = three_d ? (size_t)(bt->M_cap > 0 ? bt->M_cap : 1) : 2, bytes = (size_t)bt->B * stride * sizeof(double);
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_hs_out, &ctx->hs_out_bytes, bytes, st))) return rc;
  if ((rc = issue_hsig_scenes(ctx, &d, f, use_timediffs, ctx->d_hs_out, st))) return rc;
  CUDA_TRY(ctx, cudaMemcpyAsync(h_out, ctx->d_hs_out, bytes, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

int32_t tebgpu_build_system(tebgpu_ctx* ctx, const TebBatch* bt, int32_t outer_index, double* Hb_out, double* chi2_out,
                            int32_t device_ptrs) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  rc = check_path(ctx, bt, false);
  if (rc) return rc;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  TebBatch d = *bt;
  if (!device_ptrs) {
    rc = upload_batch(ctx, bt);
    if (rc) return rc;
    d = mirror_batch(ctx, bt);
  }
  cudaStream_t st = ctx->stream;
  DevBatch db = make_devbatch(ctx, &d);
  double mult = 1.0;
  for (int o = 0; o < outer_index; ++o) mult *= ctx->params.weight_adapt_factor;
  KParams kp = make_kparams(ctx, bt, mult);
  const int B = bt->B, tb = 128, gb = ((B > bt->S ? B : bt->S) + tb - 1) / tb;
  k_begin<<<gb, tb, 0, st>>>(db, kp);
  launch_build_graph(db, kp, B, (size_t)(bt->M_cap > 0 ? bt->M_cap : 1) * sizeof(TebObstacle), st);
  prof_begin(ctx, st, 3); launch_linearize(ctx, db, kp, B, bt->M_cap, st); prof_end(ctx, st);
  if (kp.has_vor) launch_vor(db, kp, B, (size_t)(bt->M_cap > 0 ? bt->M_cap : 1) * sizeof(TebObstacle), st);
  ctx->launches = 3;
  CUDA_TRY(ctx, cudaGetLastError());
  const size_t per_band = (size_t)4 * bt->n_cap * HROW;
  if (Hb_out)
    CUDA_TRY(ctx, cudaMemcpyAsync(Hb_out, ctx->Hb, (size_t)B * per_band * sizeof(double),
                                  device_ptrs ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
  if (chi2_out) {
    /* sum the tile partials on the host side of the call */
    std::string hold;
    const size_t cnt = (size_t)B * db.chunks * 4;
    double* tmp = new (std::nothrow) double[cnt];
    int32_t* hn = new (std::nothrow) int32_t[B];
    if (!tmp || !hn) { delete[] tmp; delete[] hn; return TEBGPU_ERR_CUDA; }
    cudaError_t e1 = cudaMemcpyAsync(tmp, ctx->chi_parts, cnt * sizeof(double), cudaMemcpyDeviceToHost, st);
    cudaError_t e2 = cudaMemcpyAsync(hn, d.n, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st);
    cudaError_t e3 = cudaStreamSynchronize(st);
    if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) { delete[] tmp; delete[] hn; ctx->err = "chi2 readback failed"; return TEBGPU_ERR_CUDA; }
    double* host_chi = device_ptrs ? new (std::nothrow) double[B] : chi2_out;
    for (int b = 0; b < B; ++b) {
      double s = 0;
      const int used = (hn[b] + db.tile - 1) / db.tile;
      for (int c = 0; c < used; ++c)
        for (int k = 0; k < 4; ++k) s += tmp[((size_t)b * db.chunks + c) * 4 + k];
      host_chi[b] = s;
    }
    if (device_ptrs) {
      cudaMemcpy(chi2_out, host_chi, (size_t)B * sizeof(double), cudaMemcpyHostToDevice);
      delete[] host_chi;
    }
    delete[] tmp;
    delete[] hn;
  }
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

/* kernel A's chi2 by family of band b (obstacles, via, time-optimal, other): spec_decide's sum, the used tiles in
 * order, family by family, over the host copy of the tile partials */
static void fold_chi_parts(const double* parts, const DevBatch& db, int b, int n, double* out4) {
  double cur[4] = {0, 0, 0, 0};
  const int used = (n + db.tile - 1) / db.tile;
  for (int ch = 0; ch < used; ++ch)
    for (int c = 0; c < 4; ++c) cur[c] += parts[((size_t)b * db.chunks + ch) * 4 + c];
  for (int c = 0; c < 4; ++c) out4[c] = cur[c];
}

int32_t tebgpu_read_linearize_outputs(tebgpu_ctx* ctx, int32_t B, int32_t n_cap, double* rhs_out, double* chi_parts_out,
                                      double* dmax_parts_out) {
  if (!ctx || B < 1 || B > ctx->lim.max_bands || n_cap < 3 || n_cap > ctx->lim.max_poses) return TEBGPU_ERR_INVALID_ARG;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int tile = ctx->linearize_variant == 1 ? TP : KA2_TP; /* make_devbatch's tile: the layout of the partials */
  const size_t tiles = (size_t)B * ((n_cap + tile - 1) / tile);
  if (rhs_out) CUDA_TRY(ctx, cudaMemcpyAsync(rhs_out, ctx->rhs, (size_t)B * 4 * n_cap * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (chi_parts_out) CUDA_TRY(ctx, cudaMemcpyAsync(chi_parts_out, ctx->chi_parts, tiles * 4 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (dmax_parts_out) CUDA_TRY(ctx, cudaMemcpyAsync(dmax_parts_out, ctx->dmax_parts, tiles * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

/* one band's state in the TEBGPU_EVAL_STATE layout */
static void pack_band_state(const BandState& x, double* s) {
  s[0] = x.lambda; s[1] = x.ni; s[2] = x.current_chi;
  for (int c = 0; c < 4; ++c) { s[3 + c] = x.parts_cur[c]; s[7 + c] = x.parts_last[c]; }
  s[11] = x.status; s[12] = x.active; s[13] = x.lm_iters;
}

int32_t tebgpu_read_band_state(tebgpu_ctx* ctx, int32_t B, double* out) {
  if (!ctx || !out || B < 1 || B > ctx->lim.max_bands) return TEBGPU_ERR_INVALID_ARG;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  std::vector<BandState> bs((size_t)B);
  CUDA_TRY(ctx, cudaMemcpyAsync(bs.data(), ctx->state, (size_t)B * sizeof(BandState), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  for (int b = 0; b < B; ++b) pack_band_state(bs[b], out + (size_t)b * TEBGPU_EVAL_STATE);
  return TEBGPU_OK;
}

int32_t tebgpu_build_system_graph(tebgpu_ctx* ctx, const TebBatch* bt, int32_t outer_index, const int32_t* list,
                                  int32_t list_len, double* Hb_out, double* chi_fam_out, uint64_t* assoc_out,
                                  uint64_t* assoc3_out, uint64_t* occ_out, int32_t* via_idx_out, double* dyn_t_out) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  if (outer_index < 0) return TEBGPU_ERR_INVALID_ARG;
  rc = check_path(ctx, bt, false);
  if (rc) return rc;
  const int B = bt->B, n_cap = bt->n_cap;
  if (list) {
    if (list_len < 0 || list_len > B) { ctx->err = "bad band list"; return TEBGPU_ERR_INVALID_ARG; }
    std::vector<char> seen((size_t)B, 0);
    for (int s = 0; s < list_len; ++s) {
      const int b = list[s];
      if (b < 0 || b >= B || seen[b]) { ctx->err = "bad band list"; return TEBGPU_ERR_INVALID_ARG; }
      seen[b] = 1;
    }
  }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rc = upload_batch(ctx, bt);
  if (rc) return rc;
  TebBatch d = mirror_batch(ctx, bt);
  cudaStream_t st = ctx->stream;
  DevBatch db = make_devbatch(ctx, &d);
  double mult = 1.0;
  for (int o = 0; o < outer_index; ++o) mult *= ctx->params.weight_adapt_factor;
  KParams kp = make_kparams(ctx, bt, mult);
  /* k_vor takes blockIdx.x as the band and has no list form; optimize never forks the side stream when it runs */
  if (list && kp.has_vor) { ctx->err = "a band list cannot be combined with the velocity-obstacle ratio"; return TEBGPU_ERR_INVALID_ARG; }
  /* everything the graph build and kernel A write starts as all-ones bytes (a NaN), so what no kernel wrote shows */
  const size_t hb_len = (size_t)B * 4 * n_cap * HROW, aw = (size_t)B * n_cap * db.MW, ow = (size_t)B * n_cap * db.OW;
  const size_t vl = (size_t)B * (bt->V_cap > 0 ? bt->V_cap : 0), parts_len = (size_t)B * db.chunks * 4;
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->Hb, 0xff, hb_len * sizeof(double), st));
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->rhs, 0xff, (size_t)B * 4 * n_cap * sizeof(double), st));
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->assoc, 0xff, aw * sizeof(uint64_t), st));
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->assoc3, 0xff, aw * sizeof(uint64_t), st));
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->occ, 0xff, ow * sizeof(uint64_t), st));
  if (vl) CUDA_TRY(ctx, cudaMemsetAsync(ctx->via_idx, 0xff, vl * sizeof(int32_t), st));
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->dyn_t, 0xff, (size_t)B * n_cap * sizeof(double), st));
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->chi_parts, 0xff, parts_len * sizeof(double), st));
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->dmax_parts, 0xff, (size_t)B * db.chunks * sizeof(double), st));
  const int tb = 128, gb = ((B > bt->S ? B : bt->S) + tb - 1) / tb;
  const size_t smem_g = (size_t)(bt->M_cap > 0 ? bt->M_cap : 1) * sizeof(TebObstacle);
  k_begin<<<gb, tb, 0, st>>>(db, kp);
  DevBatch dl = db;
  if (list) { /* the side stream's form: the list and its length in device memory, grids over the whole batch */
    if (list_len > 0)
      CUDA_TRY(ctx, cudaMemcpyAsync(ctx->spec.list, list, (size_t)list_len * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(ctx->spec.cnt, &list_len, sizeof(int32_t), cudaMemcpyHostToDevice, st));
    dl.a_list = ctx->spec.list;
    dl.a_cnt = ctx->spec.cnt;
  }
  launch_build_graph(dl, kp, B, smem_g, st);
  launch_linearize(ctx, dl, kp, B, bt->M_cap, st);
  if (kp.has_vor) launch_vor(db, kp, B, smem_g, st);
  ctx->launches = 3 + (kp.has_vor ? 1 : 0);
  CUDA_TRY(ctx, cudaGetLastError());
  std::vector<double> parts(parts_len);
  CUDA_TRY(ctx, cudaMemcpyAsync(parts.data(), ctx->chi_parts, parts_len * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (Hb_out) CUDA_TRY(ctx, cudaMemcpyAsync(Hb_out, ctx->Hb, hb_len * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (assoc_out) CUDA_TRY(ctx, cudaMemcpyAsync(assoc_out, ctx->assoc, aw * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  if (assoc3_out) CUDA_TRY(ctx, cudaMemcpyAsync(assoc3_out, ctx->assoc3, aw * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  if (occ_out) CUDA_TRY(ctx, cudaMemcpyAsync(occ_out, ctx->occ, ow * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  if (via_idx_out && vl) CUDA_TRY(ctx, cudaMemcpyAsync(via_idx_out, ctx->via_idx, vl * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (dyn_t_out) CUDA_TRY(ctx, cudaMemcpyAsync(dyn_t_out, ctx->dyn_t, (size_t)B * n_cap * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  if (chi_fam_out) {
    /* a band no kernel linearised (not listed, or not active) keeps the all-ones pattern */
    std::vector<char> ran((size_t)B, list ? 0 : 1);
    if (list)
      for (int s = 0; s < list_len; ++s) ran[list[s]] = 1;
    for (int b = 0; b < B; ++b) {
      if (ran[b]) fold_chi_parts(parts.data(), db, b, bt->n[b], chi_fam_out + (size_t)b * 4);
      else std::memset(chi_fam_out + (size_t)b * 4, 0xff, 4 * sizeof(double));
    }
  }
  return TEBGPU_OK;
}

int32_t tebgpu_solve_system(tebgpu_ctx* ctx, int32_t B, int32_t n_cap, const double* Hb, const int32_t* n,
                            const double* lambda, const double* nu, const int32_t* active, int32_t K, const int32_t* qmax,
                            const int32_t* list, int32_t list_len, int32_t lat_cap, double* dx_out, double* ok_out,
                            double* lambda_out) {
  if (!ctx || !n || !dx_out || !ok_out || !lambda_out) return TEBGPU_ERR_INVALID_ARG;
  if (B < 1 || n_cap < 3 || !(K == 2 || K == 4 || K == 6 || K == 8)) { ctx->err = "bad solve dimensions"; return TEBGPU_ERR_INVALID_ARG; }
  if (B > ctx->lim.max_bands || n_cap > ctx->lim.max_poses) { ctx->err = "solve exceeds the context limits"; return TEBGPU_ERR_CAPACITY; }
  const bool retry = qmax != nullptr;
  if (retry && (!list || list_len < 0 || list_len > B || !lambda)) { ctx->err = "a retry round needs its list and lambda"; return TEBGPU_ERR_INVALID_ARG; }
  if ((lambda == nullptr) != (nu == nullptr)) { ctx->err = "lambda and nu go together"; return TEBGPU_ERR_INVALID_ARG; }
  if (lat_cap < 0 || (lat_cap > 0 && (!retry || ctx->solver != 2 || ctx->warp_solver != 4))) {
    ctx->err = "lat_cap applies to retry rounds of solve mapping 4";
    return TEBGPU_ERR_INVALID_ARG;
  }
  for (int b = 0; b < B; ++b)
    if (n[b] < 3 || n[b] > n_cap) { ctx->err = "n[b] outside 3 .. n_cap"; return TEBGPU_ERR_INVALID_ARG; }
  if (retry)
    for (int s = 0; s < list_len; ++s)
      if (list[s] < 0 || list[s] >= B || qmax[list[s]] < 0 || qmax[list[s]] > 10) { ctx->err = "bad retry list"; return TEBGPU_ERR_INVALID_ARG; }
  const bool use_bcr = ctx->solver == 1 && n_cap <= BCR_MAX_POSES && kb_bcr_smem_bytes(n_cap, 0) <= 232448 &&
                       ctx->lim.max_poses <= BCR_MAX_POSES;
  if (ctx->solver == 1 && !use_bcr) { ctx->err = "block cyclic reduction needs max_poses <= 256"; return TEBGPU_ERR_UNSUPPORTED; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t per_band = (size_t)4 * n_cap * HROW;
  if (Hb) CUDA_TRY(ctx, cudaMemcpyAsync(ctx->Hb, Hb, (size_t)B * per_band * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_n, n, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  std::vector<BandState> bs((size_t)B);
  for (int b = 0; b < B; ++b) {
    std::memset(&bs[b], 0, sizeof(BandState));
    bs[b].lambda = lambda ? lambda[b] : 0.0;
    bs[b].ni = nu ? nu[b] : 2.0;
    bs[b].active = active ? (active[b] != 0) : 1;
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->state, bs.data(), (size_t)B * sizeof(BandState), cudaMemcpyHostToDevice, st));
  DevBatch db;
  std::memset(&db, 0, sizeof(db));
  db.B = B; db.n_cap = n_cap; db.S = 1;
  db.n = ctx->d_n; db.Hb = ctx->Hb; db.state = ctx->state; db.dmax_parts = ctx->dmax_parts; db.defer = ctx->defer;
  db.tile = ctx->linearize_variant == 1 ? TP : KA2_TP; /* the tiles of kernel A's partials (tebgpu_build_system) */
  db.chunks = (n_cap + db.tile - 1) / db.tile;
  SpecBufs spec = ctx->spec;
  spec.K = K; spec.sel_list = nullptr; spec.sel_cnt = nullptr; spec.defer = nullptr; spec.skip_tag = 0; spec.lat_cap = 0;
  /* retry rounds read list g % SPEC_LISTS and its length cnt[g]: round 1 = running round index 1 */
  const int round = retry ? 1 : 0, g = retry ? 1 : 0;
  const int it = lambda ? 1 : 0; /* iteration 0 of round 0 takes lambda from kernel A's partials */
  if (retry) {
    CUDA_TRY(ctx, cudaMemcpyAsync(spec.qmax, qmax, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (list_len > 0)
      CUDA_TRY(ctx, cudaMemcpyAsync(spec.list + (size_t)(g % SPEC_LISTS) * B, list, (size_t)list_len * sizeof(int32_t),
                                    cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(spec.cnt + g, &list_len, sizeof(int32_t), cudaMemcpyHostToDevice, st));
  }
  const int bk = B * K;
  const size_t sys = (size_t)((bk + 31) / 32) * 32;    /* whole warps of systems */
  const size_t dx_len = sys * 4 * n_cap;
  CUDA_TRY(ctx, cudaMemsetAsync(spec.dx, 0xff, dx_len * sizeof(double), st));
  CUDA_TRY(ctx, cudaMemsetAsync(spec.res, 0xff, (size_t)B * SPEC_K_MAX * RES_STRIDE * sizeof(double), st));
  if (ctx->solver == 2) {
    ctx->launches = launch_spec_solve(ctx, db, spec, K, it, round, g, st, lat_cap);
  } else if (use_bcr) {
    const size_t smem = kb_bcr_smem_bytes(n_cap, 0);
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_solve_seq<1, KB_BCR_THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_solve_seq<1, KB_BCR_THREADS><<<bk, KB_BCR_THREADS, smem, st>>>(db, spec, it, round, g);
    ctx->launches = 1;
  } else {
    const size_t smem = per_band * sizeof(double) + 16;
    if (smem > 232448) { ctx->err = "band staging exceeds shared memory"; return TEBGPU_ERR_CAPACITY; }
    CUDA_TRY(ctx, cudaFuncSetAttribute(k_solve_seq<0, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_solve_seq<0, 32><<<bk, 32, smem, st>>>(db, spec, it, round, g);
    ctx->launches = 1;
  }
  CUDA_TRY(ctx, cudaGetLastError());
  std::vector<double> dx(dx_len), res((size_t)B * SPEC_K_MAX * RES_STRIDE);
  CUDA_TRY(ctx, cudaMemcpyAsync(dx.data(), spec.dx, dx_len * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(res.data(), spec.res, res.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  /* system t = K slot + k sits in lane t & 31 of warp t >> 5, row r at r * 32; slot = band (round 0) or list position */
  std::memset(dx_out, 0xff, (size_t)B * K * 4 * n_cap * sizeof(double));
  const int slots = retry ? list_len : B;
  for (int s = 0; s < slots; ++s) {
    const int b = retry ? list[s] : s;
    for (int k = 0; k < K; ++k) {
      const size_t t = (size_t)K * s + k;
      const double* src = dx.data() + (t >> 5) * 32 * 4 * n_cap + (t & 31);
      double* dst = dx_out + ((size_t)b * K + k) * 4 * n_cap;
      for (int r = 0; r < 4 * n_cap; ++r) dst[r] = src[(size_t)r * 32];
    }
  }
  for (int b = 0; b < B; ++b)
    for (int k = 0; k < K; ++k) {
      ok_out[(size_t)b * K + k] = res[((size_t)b * SPEC_K_MAX + k) * RES_STRIDE + 5];
      lambda_out[(size_t)b * K + k] = res[((size_t)b * SPEC_K_MAX + k) * RES_STRIDE + 6];
    }
  return TEBGPU_OK;
}

int32_t tebgpu_eval_trials(tebgpu_ctx* ctx, TebBatch* bt, int32_t outer_index, int32_t iteration, int32_t K, const double* dx,
                           const double* ok, const double* lambda_k, const double* state, const int32_t* qmax,
                           const int32_t* list, int32_t list_len, double* res_out, double* chi_lin, double* state_out,
                           int32_t* qmax_out, int32_t* need_out, int32_t* next_list, int32_t* next_len) {
  int32_t rc = check_batch(ctx, bt);
  if (rc) return rc;
  if (!dx || !ok || !lambda_k || !state || outer_index < 0 || iteration < 0) return TEBGPU_ERR_INVALID_ARG;
  if (!(K == 2 || K == 4 || K == 6 || K == 8)) { ctx->err = "bad speculation width"; return TEBGPU_ERR_INVALID_ARG; }
  rc = check_path(ctx, bt, true);
  if (rc) return rc;
  const int B = bt->B, n_cap = bt->n_cap;
  const bool retry = qmax != nullptr;
  for (int b = 0; b < B; ++b)
    if (bt->n[b] < 3 || bt->n[b] > n_cap) { ctx->err = "n[b] outside 3 .. n_cap"; return TEBGPU_ERR_INVALID_ARG; }
  if (retry) {
    if (!list || list_len < 0 || list_len > B) { ctx->err = "a retry round needs its list"; return TEBGPU_ERR_INVALID_ARG; }
    std::vector<char> seen((size_t)B, 0);
    for (int s = 0; s < list_len; ++s) {
      const int b = list[s];
      if (b < 0 || b >= B || seen[b] || qmax[b] < 0 || qmax[b] > 10) { ctx->err = "bad retry list"; return TEBGPU_ERR_INVALID_ARG; }
      seen[b] = 1;
    }
  }
  const size_t smem = eval_bytes(ctx, n_cap, bt->M_cap, K);
  if (smem > 232448) { ctx->err = "trial-evaluation staging exceeds shared memory"; return TEBGPU_ERR_CAPACITY; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  rc = upload_batch(ctx, bt);
  if (rc) return rc;
  TebBatch d = mirror_batch(ctx, bt);
  cudaStream_t st = ctx->stream;
  DevBatch db = make_devbatch(ctx, &d);
  double mult = 1.0;
  for (int o = 0; o < outer_index; ++o) mult *= ctx->params.weight_adapt_factor;
  KParams kp = make_kparams(ctx, bt, mult);
  const int tb = 128, gb = ((B > bt->S ? B : bt->S) + tb - 1) / tb;
  const size_t smem_g = (size_t)(bt->M_cap > 0 ? bt->M_cap : 1) * sizeof(TebObstacle);
  k_begin<<<gb, tb, 0, st>>>(db, kp);
  launch_build_graph(db, kp, B, smem_g, st);
  launch_linearize(ctx, db, kp, B, bt->M_cap, st);
  if (kp.has_vor) launch_vor(db, kp, B, smem_g, st);
  /* the band state before the round replaces what buildGraph set (kernel A above ran for every band) */
  std::vector<BandState> bs((size_t)B);
  for (int b = 0; b < B; ++b) {
    const double* s = state + (size_t)b * TEBGPU_EVAL_STATE;
    BandState& x = bs[b];
    std::memset(&x, 0, sizeof(x));
    x.lambda = s[0]; x.ni = s[1]; x.current_chi = s[2]; x.chi2_final = s[2];
    for (int c = 0; c < 4; ++c) { x.parts_cur[c] = s[3 + c]; x.parts_last[c] = s[7 + c]; }
    x.status = (int32_t)s[11]; x.active = s[12] != 0; x.lm_iters = (int32_t)s[13];
  }
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->state, bs.data(), (size_t)B * sizeof(BandState), cudaMemcpyHostToDevice, st));
  /* the trials, in the solver's interleaved scratch: system K slot + k in lane & 31 of warp >> 5, row r at r * 32, slot =
   * band (round 0) or list position; res rows 0 .. 4 all-ones (a NaN), res[5] / res[6] what the solve wrote */
  SpecBufs spec = ctx->spec;
  spec.K = K; spec.sel_list = nullptr; spec.sel_cnt = nullptr; spec.defer = nullptr; spec.skip_tag = 0; spec.lat_cap = 0;
  const int round = retry ? 1 : 0, g = retry ? 1 : 0; /* retry rounds read list g % SPEC_LISTS and its length cnt[g] */
  const int slots = retry ? list_len : B;
  const size_t rows = (size_t)4 * n_cap;
  const size_t sys = (((size_t)B * K + 31) / 32) * 32;
  std::vector<double> hdx(sys * rows), hres((size_t)B * SPEC_K_MAX * RES_STRIDE);
  std::memset(hdx.data(), 0xff, hdx.size() * sizeof(double));
  std::memset(hres.data(), 0xff, hres.size() * sizeof(double));
  for (int s = 0; s < slots; ++s) {
    const int b = retry ? list[s] : s;
    for (int k = 0; k < K; ++k) {
      const size_t t = (size_t)K * s + k;
      const double* src = dx + ((size_t)b * K + k) * rows;
      double* dst = hdx.data() + (t >> 5) * 32 * rows + (t & 31);
      for (size_t r = 0; r < rows; ++r) dst[r * 32] = src[r];
    }
  }
  for (int b = 0; b < B; ++b)
    for (int k = 0; k < K; ++k) {
      hres[((size_t)b * SPEC_K_MAX + k) * RES_STRIDE + 5] = ok[(size_t)b * K + k];
      hres[((size_t)b * SPEC_K_MAX + k) * RES_STRIDE + 6] = lambda_k[(size_t)b * K + k];
    }
  CUDA_TRY(ctx, cudaMemcpyAsync(spec.dx, hdx.data(), hdx.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(spec.res, hres.data(), hres.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  CUDA_TRY(ctx, cudaMemsetAsync(spec.need, 0xff, (size_t)B * sizeof(int32_t), st));
  CUDA_TRY(ctx, cudaMemsetAsync(spec.cnt, 0, 3 * sizeof(int32_t), st)); /* list lengths of rounds 0 .. 2 */
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->defer, 0, (size_t)B * sizeof(int32_t), st));
  CUDA_TRY(ctx, cudaMemsetAsync(ctx->arrive, 0, (size_t)B * sizeof(int32_t), st));
  if (retry) {
    CUDA_TRY(ctx, cudaMemcpyAsync(spec.qmax, qmax, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    if (list_len > 0)
      CUDA_TRY(ctx, cudaMemcpyAsync(spec.list + (size_t)(g % SPEC_LISTS) * B, list, (size_t)list_len * sizeof(int32_t),
                                    cudaMemcpyHostToDevice, st));
    CUDA_TRY(ctx, cudaMemcpyAsync(spec.cnt + g, &list_len, sizeof(int32_t), cudaMemcpyHostToDevice, st));
  } else {
    CUDA_TRY(ctx, cudaMemsetAsync(spec.qmax, 0xff, (size_t)B * sizeof(int32_t), st));
  }
  launch_trial_eval(ctx, spec, db, kp, B, K, smem, iteration, round, g, 1, st);
  ctx->launches = 4 + (kp.has_vor ? 1 : 0);
  CUDA_TRY(ctx, cudaGetLastError());
  std::vector<double> parts((size_t)B * db.chunks * 4);
  std::vector<int32_t> hq((size_t)B), hneed((size_t)B), hlist((size_t)B);
  int32_t hcnt = 0;
  CUDA_TRY(ctx, cudaMemcpyAsync(hres.data(), spec.res, hres.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(parts.data(), ctx->chi_parts, parts.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(bs.data(), ctx->state, (size_t)B * sizeof(BandState), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(hq.data(), spec.qmax, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(hneed.data(), spec.need, (size_t)B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(hlist.data(), spec.list + (size_t)((g + 1) % SPEC_LISTS) * B, (size_t)B * sizeof(int32_t),
                                cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(&hcnt, spec.cnt + g + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(bt->poses, ctx->d_poses, (size_t)B * n_cap * 4 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  for (int b = 0; b < B; ++b) {
    if (res_out)
      for (int k = 0; k < K; ++k)
        for (int c = 0; c < 5; ++c) res_out[((size_t)b * K + k) * 5 + c] = hres[((size_t)b * SPEC_K_MAX + k) * RES_STRIDE + c];
    if (chi_lin) fold_chi_parts(parts.data(), db, b, bt->n[b], chi_lin + (size_t)b * 4);
    if (state_out) pack_band_state(bs[b], state_out + (size_t)b * TEBGPU_EVAL_STATE);
    if (qmax_out) qmax_out[b] = hq[b];
    if (need_out) need_out[b] = hneed[b];
  }
  if (next_len) *next_len = hcnt;
  if (next_list)
    for (int s = 0; s < hcnt && s < B; ++s) next_list[s] = hlist[s];
  return TEBGPU_OK;
}

/* ------------------------------------------------------------------ the one collective: all-gather of the costs */
#define NCCL_TRY(ctx, expr)                                                                              \
  do {                                                                                                   \
    ncclResult_t _r = (expr);                                                                            \
    if (_r != ncclSuccess) {                                                                             \
      (ctx)->err = std::string(#expr) + ": " + (nccl_api().GetErrorString ? nccl_api().GetErrorString(_r) : "NCCL error"); \
      return TEBGPU_ERR_CUDA;                                                                            \
    }                                                                                                    \
  } while (0)

int32_t tebgpu_comm_get_unique_id(void* id_out) {
  static_assert(sizeof(ncclUniqueId) == TEBGPU_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
  if (!id_out) return TEBGPU_ERR_INVALID_ARG;
  NcclApi& api = nccl_api();
  if (!api.ok()) { std::fprintf(stderr, "tebgpu_comm_get_unique_id: %s\n", api.error.c_str()); return TEBGPU_ERR_UNSUPPORTED; }
  ncclUniqueId id;
  if (api.GetUniqueId(&id) != ncclSuccess) return TEBGPU_ERR_CUDA;
  std::memcpy(id_out, &id, sizeof(id));
  return TEBGPU_OK;
}

int32_t tebgpu_comm_init(tebgpu_ctx* ctx, const void* id, int32_t world_size, int32_t rank) {
  if (!ctx || !id || world_size < 1 || rank < 0 || rank >= world_size) return TEBGPU_ERR_INVALID_ARG;
  NcclApi& api = nccl_api();
  if (!api.ok()) { ctx->err = api.error.empty() ? "NCCL unavailable" : api.error; return TEBGPU_ERR_UNSUPPORTED; }
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  if (ctx->comm) { api.CommDestroy(ctx->comm); ctx->comm = nullptr; }
  ncclUniqueId uid;
  std::memcpy(&uid, id, sizeof(uid));
  NCCL_TRY(ctx, api.CommInitRank(&ctx->comm, world_size, uid, rank));
  ctx->world = world_size;
  ctx->rank = rank;
  if (ctx->d_gather) { cudaFree(ctx->d_gather); ctx->d_gather = nullptr; }
  CUDA_TRY(ctx, cudaMalloc(&ctx->d_gather, (size_t)world_size * ctx->lim.max_bands * sizeof(double)));
  return TEBGPU_OK;
}

int32_t tebgpu_comm_destroy(tebgpu_ctx* ctx) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->comm) { nccl_api().CommDestroy(ctx->comm); ctx->comm = nullptr; }
  ctx->world = 1; ctx->rank = 0;
  return TEBGPU_OK;
}

int32_t tebgpu_gather_costs(tebgpu_ctx* ctx, const double* cost_local, int32_t count_local, double* cost_all, int32_t device_ptrs,
                            void* cuda_stream) {
  if (!ctx || !cost_local || !cost_all || count_local < 1) return TEBGPU_ERR_INVALID_ARG;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = (device_ptrs && cuda_stream) ? (cudaStream_t)cuda_stream : ctx->stream;
  const size_t bytes = (size_t)count_local * sizeof(double);
  if (!ctx->comm) { /* one rank: the gathered vector is the local one */
    if (device_ptrs) { if (cost_all != cost_local) CUDA_TRY(ctx, cudaMemcpyAsync(cost_all, cost_local, bytes, cudaMemcpyDeviceToDevice, st)); }
    else std::memmove(cost_all, cost_local, bytes);
    return TEBGPU_OK;
  }
  if (device_ptrs) {
    NCCL_TRY(ctx, nccl_api().AllGather(cost_local, cost_all, (size_t)count_local, ncclDouble, ctx->comm, st));
    return TEBGPU_OK;
  }
  if (count_local > ctx->lim.max_bands) { ctx->err = "gather of more than max_bands costs"; return TEBGPU_ERR_CAPACITY; }
  CUDA_TRY(ctx, cudaMemcpyAsync(ctx->d_cost, cost_local, bytes, cudaMemcpyHostToDevice, st));
  NCCL_TRY(ctx, nccl_api().AllGather(ctx->d_cost, ctx->d_gather, (size_t)count_local, ncclDouble, ctx->comm, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(cost_all, ctx->d_gather, bytes * ctx->world, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

int32_t tebgpu_optimize_batch_gather(tebgpu_ctx* ctx, const TebBatch* bt, const TebOptimizeArgs* args, double* cost_all) {
  if (!ctx || !bt || !cost_all || !bt->cost) return TEBGPU_ERR_INVALID_ARG;
  /* the device-side costs of the host entry point live in d_cost: gather them before they travel to the host */
  int32_t rc = tebgpu_optimize_batch(ctx, bt, args);
  if (rc) return rc;
  if (!ctx->comm) { std::memcpy(cost_all, bt->cost, (size_t)bt->B * sizeof(double)); return TEBGPU_OK; }
  cudaStream_t st = ctx->stream;
  NCCL_TRY(ctx, nccl_api().AllGather(ctx->d_cost, ctx->d_gather, (size_t)bt->B, ncclDouble, ctx->comm, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(cost_all, ctx->d_gather, (size_t)bt->B * ctx->world * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

/* the second collective: the fleet table, rank g's rows [g cap, (g + 1) cap) to every rank, in place */
static int32_t check_fleet_gather(tebgpu_ctx* ctx, const TebFleetTable* t, int32_t cap) {
  if (!ctx) return TEBGPU_ERR_INVALID_ARG;
  if (!t || !t->rows) { ctx->err = "fleet table or its rows == NULL"; return TEBGPU_ERR_INVALID_ARG; }
  if (cap < 1 || (int64_t)t->T != (int64_t)ctx->world * cap) { ctx->err = "fleet gather needs cap >= 1 and T == world * cap"; return TEBGPU_ERR_INVALID_ARG; }
  if (reinterpret_cast<uintptr_t>(t->rows) & 15) { ctx->err = "fleet table rows not 16-byte aligned"; return TEBGPU_ERR_INVALID_ARG; }
  return TEBGPU_OK;
}

int32_t tebgpu_fleet_gather_device(tebgpu_ctx* ctx, const TebFleetTable* t, int32_t cap, void* cuda_stream) {
  const int32_t rc = check_fleet_gather(ctx, t, cap);
  if (rc) return rc;
  if (!ctx->comm) return TEBGPU_OK;          /* one rank: the table is whole */
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream;
  const size_t bytes = (size_t)cap * sizeof(TebFleetRow);
  NCCL_TRY(ctx, nccl_api().AllGather((const char*)t->rows + (size_t)ctx->rank * bytes, t->rows, bytes, ncclChar, ctx->comm, st));
  return TEBGPU_OK;
}

int32_t tebgpu_fleet_gather(tebgpu_ctx* ctx, const TebFleetTable* t, int32_t cap) {
  int32_t rc = check_fleet_gather(ctx, t, cap);
  if (rc) return rc;
  if (!ctx->comm) return TEBGPU_OK;
  CUDA_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t bytes = (size_t)cap * sizeof(TebFleetRow), all = bytes * ctx->world;
  if ((rc = grow_mirror(ctx, (void**)&ctx->d_ftable, &ctx->ftable_bytes, all, st))) return rc;
  char* d = (char*)ctx->d_ftable;
  const size_t mine = (size_t)ctx->rank * bytes;
  CUDA_TRY(ctx, cudaMemcpyAsync(d + mine, (const char*)t->rows + mine, bytes, cudaMemcpyHostToDevice, st));
  NCCL_TRY(ctx, nccl_api().AllGather(d + mine, d, bytes, ncclChar, ctx->comm, st));
  CUDA_TRY(ctx, cudaMemcpyAsync(t->rows, d, all, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(ctx, cudaStreamSynchronize(st));
  return TEBGPU_OK;
}

int32_t tebgpu_select_best(const double* cost, int32_t count, int32_t last_best, int32_t initial_plan,
                           double selection_cost_hysteresis, double selection_prefer_initial_plan) {
  /* HomotopyClassPlanner::selectBestTeb homotopy_class_planner.cpp:564-616 */
  if (!cost || count <= 0) return -1;
  double min_cost = 1.7976931348623157e308;
  int best = -1;
  for (int i = 0; i < count; ++i) {
    double teb_cost;
    if (i == last_best) teb_cost = cost[i] * selection_cost_hysteresis;
    else if (i == initial_plan) teb_cost = cost[i] * selection_prefer_initial_plan;
    else teb_cost = cost[i];
    if (teb_cost < min_cost) { best = i; min_cost = teb_cost; }
  }
  return best;
}

int32_t tebgpu_auto_resize_host(double* rec, int32_t n, int32_t n_cap, double dt_ref, double dt_hysteresis,
                                int32_t min_samples, int32_t max_samples, int32_t fast_mode) {
  if (!rec || n < 1 || n > n_cap) return TEBGPU_ERR_INVALID_ARG;
  int nn = teb_auto_resize_records(rec, n, n_cap, dt_ref, dt_hysteresis, min_samples, max_samples, fast_mode);
  return nn < 0 ? TEBGPU_ERR_CAPACITY : nn;
}

}  /* extern "C" */
