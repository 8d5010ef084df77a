/*
 * teb_oracle.h — CPU oracle for the TEB optimisation hot path (TEST INFRASTRUCTURE ONLY).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library. The product (teb_local_planner_b200/) never links or calls it.
 *
 * PARITY PINNED against the reference's own code: oracle/_ref/libteb_ref.so (make ref) is src/optimal_planner.cpp +
 * src/timed_elastic_band.cpp + src/obstacles.cpp and their headers, compiled where they lie under /root/reference against
 * stand-ins for the absent third-party code (oracle/ref_shims/: Eigen, boost, ROS messages, the g2o optimizer).
 * tests/test_reference_pin.py compares this restatement with it BIT FOR BIT: every edge (errors, information,
 * Jacobians), H / b / chi2, whole optimizeTEB calls (poses, n, cost, LM trials) on 24 feature scenarios, autoResize,
 * initTrajectoryToGoal, penalties, distances, TebConfig defaults; tests/golden/golden_ref_v1.npz holds vectors generated
 * from it. What stays restated from published behaviour is only the g2o optimizer itself (libg2o + CSparse: third-party,
 * NOT under /root/reference; SURVEY.md Appendix A, upstream g2o 2018.3.25 / 2020.5.3), anchored on the reference's call
 * sites (src/optimal_planner.cpp:161-179, 385-387, 1057-1072).
 */
#ifndef TEB_ORACLE_H
#define TEB_ORACLE_H

#include "../include/teb_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define ORACLE_JAC_G2O       0  /* numeric central differences, delta=1e-9, except EdgeKinematicsDiffDrive and
                                   EdgeTimeOptimal (the analytic overrides compiled into the reference) */
#define ORACLE_JAC_ANALYTIC  1  /* closed-form Jacobians for every edge (second opinion for the kernels)  */
#define ORACLE_SOLVER_BANDED 0
#define ORACLE_SOLVER_DENSE  1

typedef struct OracleOptions {
  int32_t jac_mode;
  int32_t solver;
  int32_t verbose;
  int32_t pin_threads;  /* batch driver: pin worker t to the t-th CPU of the affinity mask (timing runs) */
} OracleOptions;

typedef struct OracleStats {
  double  chi2_final;      /* chi2 of the state after the last LM iteration (currentChi)              */
  double  lambda_final;
  int32_t lm_iters;        /* inner iterations executed over all outer iterations                     */
  int32_t lm_trials;       /* factorisations attempted                                                */
  int32_t rejected;        /* rejected trials                                                         */
  int32_t n_edges_last;    /* active edges in the last graph                                          */
  int32_t status;          /* TEB_STATUS_* bits                                                       */
  int32_t n_final;
  double  nu_final;        /* LM nu after the last LM iteration (2^11 after ten rejected trials)       */
} OracleStats;

/* One band, one optimizeTEB call (optimal_planner.cpp:182-231). rec [n_cap][4] in/out, n in/out. */
int32_t teb_oracle_optimize(const TebParams* cfg, double* rec, int32_t* n, int32_t n_cap,
                            const TebObstacle* obst, int32_t M, const double* via, int32_t V,
                            const double* vel_start4, const double* vel_goal4, int32_t prefer_rotdir,
                            const TebOptimizeArgs* args, const OracleOptions* opt,
                            double* cost_out, OracleStats* stats, const double* obst_vertices /* [PV][2] or NULL */);

/* Whole batch with the TebBatch layout; `threads` host threads, one band at a time per thread
 * (the reference's optimizeAllTEBs model, homotopy_class_planner.cpp:466-493). */
int32_t teb_oracle_optimize_batch(const TebParams* cfg, const TebBatch* batch, const TebOptimizeArgs* args,
                                  const OracleOptions* opt, int32_t threads);

/* buildGraph + computeActiveErrors + buildSystem at the current state (no LM step).
 * H_dense: [N][N] full symmetric, b: [N], N = 4n-7 in g2o order (dt_0, pose_1, dt_1, ..., dt_{n-2}).
 * Returns N, or <0. weight_multiplier as in buildGraph (optimal_planner.cpp:323). */
int32_t teb_oracle_build_system(const TebParams* cfg, const double* rec, int32_t n,
                                const TebObstacle* obst, int32_t M, const double* via, int32_t V,
                                const double* vel_start4, const double* vel_goal4, int32_t prefer_rotdir,
                                double weight_multiplier, int32_t jac_mode,
                                double* H_dense, double* b, double* chi2, const double* obst_vertices /* or NULL */);

/* Per-edge dump (errors, information, Jacobians, vertex ids) of the graph at the given state; 64 doubles per active edge,
 * layout in teb_oracle.c. Lets tests compare the restatement with oracle/_ref edge by edge. */
int32_t teb_oracle_dump_edges(const TebParams* cfg, const double* rec, int32_t n, const TebObstacle* obst, int32_t M,
                              const double* via, int32_t V, const double* vel_start4, const double* vel_goal4,
                              int32_t prefer_rotdir, double weight_multiplier, int32_t jac_mode, double* rows,
                              int32_t max_rows, const double* obst_vertices);

/* chi2 of LM trial states by the device's four families (obstacle / inflated / dynamic-obstacle edges, via-points,
 * time-optimal, every other edge including the velocity-obstacle ratio), accumulated in long double. The graph is built
 * once at rec_graph with the weight multiplier, which freezes the obstacle association, the dynamic-obstacle times and
 * the via-point assignment; every edge's error is then evaluated at each of the T states rec_trials [T][n][4].
 * chi_out [T][4]. Returns 0, or <0. */
int32_t teb_oracle_trial_chi2(const TebParams* cfg, const double* rec_graph, int32_t n, const TebObstacle* obst, int32_t M,
                              const double* via, int32_t V, const double* vel_start4, const double* vel_goal4,
                              int32_t prefer_rotdir, double weight_multiplier, const double* rec_trials, int32_t T,
                              double* chi_out, const double* obst_vertices);

/* The structure buildGraph() gives the band at rec with the weight multiplier, read off the active edges:
 * assoc_out [n][MW] bit m of pose i for an obstacle / inflated-obstacle edge on pose i whose obstacle is obst[m] (and,
 * with the velocity-obstacle ratio, for the ratio edges anchored at pose i, which carry pose 0's association);
 * assoc3_out [n][MW] bit m where pose i carries three such edges (the legacy centre pose); via_idx_out [V] the pose of
 * each via-point's edge, -1 where it has none; dyn_t_out [n] the frozen time t of pose i's dynamic-obstacle edges, NaN
 * where it has none. MW >= ceil(M / 64). Returns 0, or <0. */
int32_t teb_oracle_graph(const TebParams* cfg, const double* rec, int32_t n, const TebObstacle* obst, int32_t M,
                         const double* via, int32_t V, const double* vel_start4, const double* vel_goal4,
                         int32_t prefer_rotdir, double weight_multiplier, int32_t MW, uint64_t* assoc_out,
                         uint64_t* assoc3_out, int32_t* via_idx_out, double* dyn_t_out, const double* obst_vertices);

/* g2o's accept / reject chain of one LM iteration, the function teb_oracle_optimize's LM loop runs for every trial.
 * From currentChi, lambda, nu and q0 trials already consumed in the iteration, it takes the trials k = 0 .. count-1
 * (trial chi2 temp_chi[k], computeScale() sum scale_sum[k] without the 1e-3, ok[k] == 0: failed factorisation) while
 * the iteration goes on. out_i: [0] accepted trial (last accepted k, or -1), [1] trials consumed, [2] Terminate,
 * [3] TEB_STATUS_* bits added, [4] 1 when the iteration needs more trials than given, [5] trials of the iteration
 * after these (q). out_d: lambda, nu, currentChi after them. Returns 0, or <0. */
int32_t teb_oracle_lm_decide(double current_chi, double lambda, double nu, int32_t q0, int32_t count, const double* temp_chi,
                             const double* scale_sum, const int32_t* ok, int32_t* out_i, double* out_d);

/* TimedElasticBand::autoResize (timed_elastic_band.cpp:227-286). Returns new n. */
int32_t teb_oracle_auto_resize(double* rec, int32_t n, int32_t n_cap, double dt_ref, double dt_hysteresis,
                               int32_t min_samples, int32_t max_samples, int32_t fast_mode);

/* TimedElasticBand::initTrajectoryToGoal(start, goal, diststep, max_vel_x, min_samples, backwards)
 * (timed_elastic_band.cpp:325-387). Returns n. */
int32_t teb_oracle_init_trajectory(const double* start3, const double* goal3, double diststep, double max_vel_x,
                                   int32_t min_samples, int32_t guess_backwards_motion, double* rec, int32_t n_cap);

/* BaseRobotFootprintModel::calculateDistance (t = 0) / estimateSpatioTemporalDistance of the configured footprint to
 * one obstacle, every footprint x obstacle combination; grad3 (optional) = d dist / d(x, y, theta) in closed form. */
double teb_oracle_distance(const TebParams* cfg, const double* pose3, const TebObstacle* obst, const double* obst_vertices,
                           double t, double* grad3);

/* HomotopyClassPlanner::calculateEquivalenceClass (homotopy_class_planner.hpp:46-63) on the positions of one band:
 * include_dynamic_obstacles == 0 -> HSignature::calculateHSignature (h_signature.h:97-186, long double accumulation),
 * out[0..1] = (Re, Im); else HSignature3d::calculateHSignature (:282-353), out[0..M). use_timediffs as in the C-ABI. */
int32_t teb_oracle_h_signature(const TebParams* cfg, const double* rec, int32_t n, const TebObstacle* obst, int32_t M,
                               int32_t use_timediffs, double* out);

/* helpers exposed for unit tests */
double teb_oracle_normalize_theta(double t);
double teb_oracle_average_angle(double a, double b);
double teb_oracle_penalty_interval(double v, double a, double eps);
double teb_oracle_penalty_interval2(double v, double a, double b, double eps);
double teb_oracle_penalty_below(double v, double a, double eps);

#ifdef __cplusplus
}
#endif
#endif
