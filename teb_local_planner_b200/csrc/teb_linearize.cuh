/*
 * teb_linearize.cuh — "kernel A", second generation (k_linearize2p below is its persistent form, the default): residuals + closed-form Jacobians of every edge
 * family + banded J^T Omega J / b assembly, ONE THREAD PER POSE, ONE WARP PER TILE, no block-wide barrier on the path.
 *
 * Mapping. A warp owns KA2_TP = 29 consecutive poses of one band; lane l <-> pose / anchor i = q0 - 2 + l (two halo
 * anchors on the left, one halo segment on the right, recomputed by the neighbouring tile: 9 % redundancy instead of
 * any cross-warp synchronisation). A CTA is KA2_W = 4 such warps over adjacent tiles; it shares one TMA-staged pose
 * range and the scene's obstacle table (two 1-D bulk copies on one mbarrier, issued before anything else is known).
 *   P1  sin/cos of the own pose, derivative bundle of the own segment (registers; the right neighbour's bundle arrives
 *       by warp shuffles), unary terms (obstacles / dynamic obstacles / via-points) of the own pose in registers
 *   P2  sqrt(weight)-scaled Jacobian rows of the chain edges anchored at the own pose, written as a COMPACT record
 *       (structural zeros are not stored) into the warp's shared-memory region, element-major ([element][lane]: every
 *       access of the warp is one contiguous 256-byte run, no bank conflicts); __syncwarp
 *   P3  the four band rows of the own pose (4 x 11 entries + 4 rhs) are accumulated IN REGISTERS from the records of
 *       the three anchors that touch them; structural zeros are compiled out, rows whose residual is exactly zero
 *       (inactive penalties: most velocity / acceleration rows of a converged band) are skipped at run time
 *   P4  the 384 bytes of a pose go through a padded shared-memory slot and leave with one TMA bulk store per lane
 *       (cp.async.bulk.global.shared::cta; the default), or as 128-bit global stores straight from the registers
 *       (OUT_DIRECT, TEBGPU_KA_STAGED=0: slower - every store instruction fills half a 32-byte
 *       sector); b also goes to the compact rhs array
 *
 * Arithmetic = the computeError bodies cited in teb_device.cuh / below, Jacobians in closed form; identical formulas to
 * the first-generation kernel (k_linearize in teb_kernels.cuh, kept as variant 1), different summation order.
 * Replaces g2o BlockSolver::buildSystem for every edge of optimal_planner.cpp:444-1021 (SURVEY.md par. 3.3 step 2).
 */
#pragma once

#include "teb_kernels.cuh"

namespace tebgpu {

constexpr int KA2_W = 4;             /* warps (tiles) per CTA */
constexpr int KA2_THREADS = 32 * KA2_W;
constexpr int KA2_TP = 29;           /* poses (band row groups) produced per warp: lanes 2 .. 30 */
constexpr int KA2_SLOTS = KA2_W * KA2_TP + 4; /* poses staged per CTA: slot j <-> pose P0 - 2 + j */
constexpr int KA2_NT = 32;           /* record stride: element-major within the warp's region */
constexpr int OUT_STRIDE = 50;       /* doubles per staging slot: 48 + 2 pad -> 400 B lane stride, conflict-free STS.128 */

/* Compact Jacobian record of one anchor (columns: x_a y_a th_a dt_a x_b y_b th_b [dt_b x_c y_c th_c]).
 * Only the columns that can be non-zero are stored; MASK bit c = column c is stored. */
template <bool HOLO>
struct JL {
  static constexpr int V = 0;                       /* EdgeVelocity v row (holonomic: vx)      7 */
  static constexpr int W = V + 7;                   /* omega row                                3 */
  static constexpr int K0 = W + 3;                  /* EdgeKinematics* row 0                    6 */
  static constexpr int K1 = K0 + 6;                 /* row 1 (forward drive / turning radius)   6 */
  static constexpr int SP = K1 + 6;                 /* EdgeShortestPath                         4 */
  static constexpr int ROT = SP + 4;                /* EdgePreferRotDir                         2 */
  static constexpr int VY = ROT + 2;                /* holonomic vy row                         6 */
  static constexpr int A0 = VY + (HOLO ? 6 : 0);    /* EdgeAcceleration row x                  11 */
  static constexpr int A1 = A0 + 11;                /* row theta                                5 */
  static constexpr int A2 = A1 + 5;                 /* holonomic row y                         11 */
  static constexpr int E = A2 + (HOLO ? 11 : 0);    /* residuals: v, w, k0, k1, sp, rot, a0, a1 [, vy, a2] */
  static constexpr int COUNT = E + (HOLO ? 10 : 8);
};
constexpr unsigned M_V = 0x7Fu, M_W = (1u << 2) | (1u << 3) | (1u << 6), M_K = 0x77u, M_SP = 0x33u,
                   M_ROT = (1u << 2) | (1u << 6), M_VY = 0x3Fu, M_A0 = 0x7FFu,
                   M_A1 = (1u << 2) | (1u << 3) | (1u << 6) | (1u << 7) | (1u << 10);
enum { E_V = 0, E_W = 1, E_K0 = 2, E_K1 = 3, E_SP = 4, E_ROT = 5, E_A0 = 6, E_A1 = 7, E_VY = 8, E_A2 = 9 };

__host__ __device__ constexpr int cidx(unsigned mask, int col) {
  int k = 0;
  for (int c = 0; c < col; ++c) k += (mask >> c) & 1u;
  return k;
}

/* write access to the own record: element-major shared memory, rec points at [0][slot] */
struct JRec {
  double* rec;
  template <int BASE, unsigned MASK, int COL>
  __device__ __forceinline__ void set(double v) const {
    if constexpr ((MASK >> COL) & 1u) rec[(BASE + cidx(MASK, COL)) * KA2_NT] = v;
  }
  __device__ __forceinline__ void res(int base_e, int k, double v) const { rec[(base_e + k) * KA2_NT] = v; }
};

struct KA2Smem {
  static constexpr int POSES = KA2_SLOTS * 4;
  static constexpr int START = 24;
  template <bool HOLO>
  __host__ __device__ static constexpr int rec_doubles() { /* records of the 32 lanes; later the 32 output slots */
    return JL<HOLO>::COUNT * 32 > OUT_STRIDE * 32 ? JL<HOLO>::COUNT * 32 : OUT_STRIDE * 32;
  }
  template <bool HOLO>
  __host__ __device__ static constexpr int warp_doubles() { return rec_doubles<HOLO>() + START; }
};
template <bool HOLO>
__host__ __device__ inline size_t ka2_smem_bytes(int M_cap) {
  const size_t d = KA2Smem::POSES + (size_t)KA2_W * KA2Smem::warp_doubles<HOLO>() + 2;
  return d * sizeof(double) + (size_t)(M_cap > 0 ? M_cap : 1) * sizeof(TebObstacle) + 64;
}

/* ------------------------------------------------------------------ P2: Jacobian rows of the chain edges anchored at
 * pose a (sqrt(weight)-scaled). sd = derivative bundle of segment a, sd2 = bundle of segment a+1 (from the right
 * neighbour lane). Returns the anchor's chi2 ("other" family). */
template <bool HOLO>
__device__ __forceinline__ double anchor_rows2(const KParams& kp, const DevBatch& db, int b, int a, int n,
                                               const double* pa /* sP + 4 slot */, double ca, double sa, double cb,
                                               double sb, const SegDer& sd, const SegDer& sd2, const JRec J,
                                               double* sStart) {
  using L = JL<HOLO>;
  const double* pb = pa + 4;
  const double v1 = sd.v, w1 = sd.w, idt1 = sd.idt;
  const double dx = pb[0] - pa[0], dy = pb[1] - pa[1];
  const bool fa = (a == 0), fb = (a + 1 == n - 1);
  /* columns of fixed poses carry no unknowns (g2o skips fixed vertices, SURVEY App. A.3): multiply by 0 / 1 masks */
  const double ma = fa ? 0.0 : 1.0, mb = fb ? 0.0 : 1.0;
  double csum = 0;
  if (HOLO && kp.has_vel && kp.holo_vel) { /* EdgeVelocityHolonomic edge_velocity.h:236-273 */
    const HoloDer h = holo_derivs(pa[0], pa[1], pa[2], ca, sa, pb[0], pb[1], pb[2], pa[3]);
    double e[3], sl[3], c0, c1;
    holo_velocity_terms(kp, h.vx, h.vy, h.w, e, sl, c0, c1);
    const double kx = kp.sw_vel_x, ky = kp.sw_vel_y, kw = kp.sw_vel_th * sl[2];
    J.set<L::V, M_V, 0>(ma * kx * (sl[0] * h.dvx[0] - c0 * h.dvy[0]));
    J.set<L::V, M_V, 1>(ma * kx * (sl[0] * h.dvx[1] - c0 * h.dvy[1]));
    J.set<L::V, M_V, 2>(ma * kx * (sl[0] * h.dvx[2] - c0 * h.dvy[2]));
    J.set<L::V, M_V, 3>(kx * (-sl[0] * h.vx + c0 * h.vy) * h.idt);
    J.set<L::V, M_V, 4>(mb * kx * (sl[0] * h.dvx[3] - c0 * h.dvy[3]));
    J.set<L::V, M_V, 5>(mb * kx * (sl[0] * h.dvx[4] - c0 * h.dvy[4]));
    J.set<L::VY, M_VY, 0>(ma * ky * (sl[1] * h.dvy[0] - c1 * h.dvx[0]));
    J.set<L::VY, M_VY, 1>(ma * ky * (sl[1] * h.dvy[1] - c1 * h.dvx[1]));
    J.set<L::VY, M_VY, 2>(ma * ky * (sl[1] * h.dvy[2] - c1 * h.dvx[2]));
    J.set<L::VY, M_VY, 3>(ky * (-sl[1] * h.vy + c1 * h.vx) * h.idt);
    J.set<L::VY, M_VY, 4>(mb * ky * (sl[1] * h.dvy[3] - c1 * h.dvx[3]));
    J.set<L::VY, M_VY, 5>(mb * ky * (sl[1] * h.dvy[4] - c1 * h.dvx[4]));
    J.set<L::W, M_W, 2>(-ma * kw * h.idt);
    J.set<L::W, M_W, 3>(-kw * h.w * h.idt);
    J.set<L::W, M_W, 6>(mb * kw * h.idt);
    const double e0 = kx * e[0], e1 = ky * e[1], e2 = kp.sw_vel_th * e[2];
    J.res(L::E, E_V, e0); J.res(L::E, E_VY, e1); J.res(L::E, E_W, e2);
    csum += e0 * e0 + e1 * e1 + e2 * e2;
  } else if (kp.has_vel) { /* EdgeVelocity edge_velocity.h:113-114 */
    double s0, s1;
    const double e0 = pen_interval2(v1, -kp.p.max_vel_x_backwards, kp.p.max_vel_x, kp.p.penalty_epsilon, s0);
    const double e1 = pen_interval(w1, kp.p.max_vel_theta, kp.p.penalty_epsilon, s1);
    const double k0 = kp.sw_vel_x * s0, k1 = kp.sw_vel_th * s1;
    J.set<L::V, M_V, 0>(ma * k0 * sd.dv[0]); J.set<L::V, M_V, 1>(ma * k0 * sd.dv[1]); J.set<L::V, M_V, 2>(ma * k0 * sd.dv[2]);
    J.set<L::V, M_V, 3>(-k0 * v1 * idt1);
    J.set<L::V, M_V, 4>(mb * k0 * sd.dv[3]); J.set<L::V, M_V, 5>(mb * k0 * sd.dv[4]); J.set<L::V, M_V, 6>(mb * k0 * sd.dv[5]);
    J.set<L::W, M_W, 2>(-ma * k1 * idt1); J.set<L::W, M_W, 3>(-k1 * w1 * idt1); J.set<L::W, M_W, 6>(mb * k1 * idt1);
    const double r0 = kp.sw_vel_x * e0, r1 = kp.sw_vel_th * e1;
    J.res(L::E, E_V, r0); J.res(L::E, E_W, r1);
    csum += r0 * r0 + r1 * r1;
  }
  if (kp.has_kin) { /* EdgeKinematicsDiffDrive / Carlike edge_kinematics.h:94-101, :118-148, :203-215 */
    const double A = (ca + cb) * dy - (sa + sb) * dx;
    const double sA = sgn(A) * kp.sw_kin_nh;
    J.set<L::K0, M_K, 0>(ma * (sa + sb) * sA); J.set<L::K0, M_K, 1>(-ma * (ca + cb) * sA);
    J.set<L::K0, M_K, 2>(ma * (-sa * dy - ca * dx) * sA);
    J.set<L::K0, M_K, 4>(-mb * (sa + sb) * sA); J.set<L::K0, M_K, 5>(mb * (ca + cb) * sA);
    J.set<L::K0, M_K, 6>(mb * (-sb * dy - cb * dx) * sA);
    const double r0 = kp.sw_kin_nh * fabs(A);
    J.res(L::E, E_K0, r0);
    double r1 = 0;
    if (!kp.carlike) {
      double dd;
      const double e1 = pen_below(dx * ca + dy * sa, 0, 0, dd);
      dd *= kp.sw_kin_2;
      J.set<L::K1, M_K, 0>(-ma * ca * dd); J.set<L::K1, M_K, 1>(-ma * sa * dd); J.set<L::K1, M_K, 2>(ma * (-sa * dx + ca * dy) * dd);
      J.set<L::K1, M_K, 4>(mb * ca * dd); J.set<L::K1, M_K, 5>(mb * sa * dd);
      r1 = kp.sw_kin_2 * e1;
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
          const double iad = 1.0 / fabs(ad);
          r = nrm * iad;
          dr_dn = iad;
          dr_dad = -nrm * sgn(ad) * (iad * iad);
        }
        double s1;
        const double e1 = pen_below(r, kp.p.min_turning_radius, 0.0, s1);
        s1 *= kp.sw_kin_2;
        J.set<L::K1, M_K, 0>(-ma * s1 * dr_dn * ux); J.set<L::K1, M_K, 1>(-ma * s1 * dr_dn * uy); J.set<L::K1, M_K, 2>(-ma * s1 * dr_dad);
        J.set<L::K1, M_K, 4>(mb * s1 * dr_dn * ux); J.set<L::K1, M_K, 5>(mb * s1 * dr_dn * uy); J.set<L::K1, M_K, 6>(mb * s1 * dr_dad);
        r1 = kp.sw_kin_2 * e1;
      }
    }
    J.res(L::E, E_K1, r1);
    csum += r0 * r0 + r1 * r1;
  }
  if (kp.has_sp) { /* EdgeShortestPath edge_shortest_path.h:78 */
    const double nrm = sqrt(dx * dx + dy * dy);
    const double inr = nrm > 0 ? 1.0 / nrm : 0.0;
    J.set<L::SP, M_SP, 0>(-ma * kp.sw_sp * dx * inr); J.set<L::SP, M_SP, 1>(-ma * kp.sw_sp * dy * inr);
    J.set<L::SP, M_SP, 4>(mb * kp.sw_sp * dx * inr); J.set<L::SP, M_SP, 5>(mb * kp.sw_sp * dy * inr);
    const double r = kp.sw_sp * nrm;
    J.res(L::E, E_SP, r);
    csum += r * r;
  }
  if (kp.has_rot && a < 3) { /* EdgePreferRotDir edge_prefer_rotdir.h:85, first three pairs optimal_planner.cpp:983 */
    const int rd = db.prefer_rotdir ? db.prefer_rotdir[b] : 0;
    if (rd == TEB_ROTDIR_LEFT || rd == TEB_ROTDIR_RIGHT) {
      const double meas = (rd == TEB_ROTDIR_LEFT) ? 1.0 : -1.0;
      double s0;
      const double e0 = pen_below(meas * normalize_theta(pb[2] - pa[2]), 0, 0, s0);
      J.set<L::ROT, M_ROT, 2>(-ma * kp.sw_rot * s0 * meas);
      J.set<L::ROT, M_ROT, 6>(mb * kp.sw_rot * s0 * meas);
      const double r = kp.sw_rot * e0;
      J.res(L::E, E_ROT, r);
      csum += r * r;
    }
  }
  if (HOLO && kp.has_acc && kp.holo_acc) {
    /* EdgeAccelerationHolonomic / Start / Goal edge_acceleration.h:487-540, :580-620, :672-712; rows x, theta, y */
    const HoloDer h1 = holo_derivs(pa[0], pa[1], pa[2], ca, sa, pb[0], pb[1], pb[2], pa[3]);
    const double sw[3] = {kp.sw_acc_x, kp.sw_acc_th, kp.sw_acc_y};
    const double lim[3] = {kp.p.acc_lim_x, kp.p.acc_lim_theta, kp.p.acc_lim_y};
    const double v1r[3] = {h1.vx, h1.w, h1.vy};
    double d1[3][6];
#pragma unroll
    for (int k = 0; k < 6; ++k) { d1[0][k] = h1.dvx[k]; d1[2][k] = h1.dvy[k]; d1[1][k] = 0; }
    d1[1][2] = -h1.idt; d1[1][5] = h1.idt;
    const double mc = (a + 2 == n - 1) ? 0.0 : 1.0;
    double R[3][11];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int k = 0; k < 11; ++k) R[r][k] = 0;
    double er[3] = {0, 0, 0};
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
        R[r][0] = -2 * kk * d1[r][0] * ma; R[r][1] = -2 * kk * d1[r][1] * ma; R[r][2] = -2 * kk * d1[r][2] * ma;
        R[r][3] = kk * (2 * v1r[r] * h1.idt - acc);
        R[r][4] = 2 * kk * (d2[r][0] - d1[r][3]) * mb; R[r][5] = 2 * kk * (d2[r][1] - d1[r][4]) * mb;
        R[r][6] = 2 * kk * (d2[r][2] - d1[r][5]) * mb;
        R[r][7] = kk * (-2 * v2r[r] * h2.idt - acc);
        R[r][8] = 2 * kk * d2[r][3] * mc; R[r][9] = 2 * kk * d2[r][4] * mc; R[r][10] = 2 * kk * d2[r][5] * mc;
        er[r] = sw[r] * e;
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
          R[r][0] = -kk * d1[r][0] * ma; R[r][1] = -kk * d1[r][1] * ma; R[r][2] = -kk * d1[r][2] * ma;
          R[r][3] = kk * (v1r[r] * h1.idt - acc);
          R[r][4] = -kk * d1[r][3] * mb; R[r][5] = -kk * d1[r][4] * mb; R[r][6] = -kk * d1[r][5] * mb;
          er[r] = sw[r] * e;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 11; ++k) {
      J.rec[(L::A0 + k) * KA2_NT] = R[0][k];
      if ((M_A1 >> k) & 1u) J.rec[(L::A1 + cidx(M_A1, k)) * KA2_NT] = R[1][k];
      J.rec[(L::A2 + k) * KA2_NT] = R[2][k];
    }
    J.res(L::E, E_A0, er[0]); J.res(L::E, E_A1, er[1]); J.res(L::E, E_A2, er[2]);
    csum += er[0] * er[0] + er[1] * er[1] + er[2] * er[2];
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
          S[4] = kk * d1[r][3] * mb; S[5] = kk * d1[r][4] * mb; S[6] = kk * d1[r][5] * mb;
          sStart[START_E + r] = sw[r] * e;
          csum += sStart[START_E + r] * sStart[START_E + r];
        }
      }
    }
  } else if (kp.has_acc) {
    double r0 = 0, r1 = 0;
    if (a <= n - 3) { /* EdgeAcceleration edge_acceleration.h:134-145 */
      const double v2 = sd2.v, w2 = sd2.w, idt2 = sd2.idt;
      const double dt1 = pa[3], dt2 = pb[3];
      const double iT = 1.0 / (dt1 + dt2);
      const double acc = (v2 - v1) * 2 * iT;
      const double accr = (w2 - w1) * 2 * iT;
      double s0, s1;
      const double e0 = pen_interval(acc, kp.p.acc_lim_x, kp.p.penalty_epsilon, s0);
      const double e1 = pen_interval(accr, kp.p.acc_lim_theta, kp.p.penalty_epsilon, s1);
      const double k0 = kp.sw_acc_x * s0 * iT, k1 = kp.sw_acc_th * s1 * iT;
      const double mc = (a + 2 == n - 1) ? 0.0 : 1.0;
      J.set<L::A0, M_A0, 0>(-2 * k0 * sd.dv[0] * ma); J.set<L::A0, M_A0, 1>(-2 * k0 * sd.dv[1] * ma); J.set<L::A0, M_A0, 2>(-2 * k0 * sd.dv[2] * ma);
      J.set<L::A0, M_A0, 3>(k0 * (2 * v1 * idt1 - acc));
      J.set<L::A0, M_A0, 4>(2 * k0 * (sd2.dv[0] - sd.dv[3]) * mb); J.set<L::A0, M_A0, 5>(2 * k0 * (sd2.dv[1] - sd.dv[4]) * mb);
      J.set<L::A0, M_A0, 6>(2 * k0 * (sd2.dv[2] - sd.dv[5]) * mb);
      J.set<L::A0, M_A0, 7>(k0 * (-2 * v2 * idt2 - acc));
      J.set<L::A0, M_A0, 8>(2 * k0 * sd2.dv[3] * mc); J.set<L::A0, M_A0, 9>(2 * k0 * sd2.dv[4] * mc); J.set<L::A0, M_A0, 10>(2 * k0 * sd2.dv[5] * mc);
      J.set<L::A1, M_A1, 2>(2 * k1 * idt1 * ma);
      J.set<L::A1, M_A1, 3>(k1 * (2 * w1 * idt1 - accr));
      J.set<L::A1, M_A1, 6>(2 * k1 * (-idt2 - idt1) * mb);
      J.set<L::A1, M_A1, 7>(k1 * (-2 * w2 * idt2 - accr));
      J.set<L::A1, M_A1, 10>(2 * k1 * idt2 * mc);
      r0 = kp.sw_acc_x * e0; r1 = kp.sw_acc_th * e1;
    } else { /* a == n-2: EdgeAccelerationGoal edge_acceleration.h:420-433 */
      const double* vg = db.vel_goal + 4 * (size_t)b;
      if (vg[3] != 0) {
        const double acc = (vg[0] - v1) * idt1;
        const double accr = (vg[2] - w1) * idt1;
        double s0, s1;
        const double e0 = pen_interval(acc, kp.p.acc_lim_x, kp.p.penalty_epsilon, s0);
        const double e1 = pen_interval(accr, kp.p.acc_lim_theta, kp.p.penalty_epsilon, s1);
        const double k0 = kp.sw_acc_x * s0 * idt1, k1 = kp.sw_acc_th * s1 * idt1;
        J.set<L::A0, M_A0, 0>(-k0 * sd.dv[0] * ma); J.set<L::A0, M_A0, 1>(-k0 * sd.dv[1] * ma); J.set<L::A0, M_A0, 2>(-k0 * sd.dv[2] * ma);
        J.set<L::A0, M_A0, 3>(k0 * (v1 * idt1 - acc));
        J.set<L::A0, M_A0, 4>(-k0 * sd.dv[3] * mb); J.set<L::A0, M_A0, 5>(-k0 * sd.dv[4] * mb); J.set<L::A0, M_A0, 6>(-k0 * sd.dv[5] * mb);
        J.set<L::A1, M_A1, 2>(k1 * idt1 * ma); J.set<L::A1, M_A1, 3>(k1 * (w1 * idt1 - accr)); J.set<L::A1, M_A1, 6>(-k1 * idt1 * mb);
        r0 = kp.sw_acc_x * e0; r1 = kp.sw_acc_th * e1;
      }
    }
    J.res(L::E, E_A0, r0); J.res(L::E, E_A1, r1);
    csum += r0 * r0 + r1 * r1;
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
        S0[4] = k0 * sd.dv[3] * mb; S0[5] = k0 * sd.dv[4] * mb; S0[6] = k0 * sd.dv[5] * mb;
        S1[0] = S1[1] = S1[2] = S1[4] = S1[5] = 0;
        S1[3] = k1 * (-w1 * idt1 - accr);
        S1[6] = k1 * idt1 * mb;
        sStart[START_E] = kp.sw_acc_x * e0; sStart[START_E + 1] = kp.sw_acc_th * e1;
        csum += sStart[START_E] * sStart[START_E] + sStart[START_E + 1] * sStart[START_E + 1];
      }
    }
  }
  return csum;
}

/* ------------------------------------------------------------------ P3: one Jacobian row of the anchor D poses back.
 * The pose owns the local columns l = 4 D + c (c = 0..3) of that anchor; acc[c][o] += J[l] J[l - o], brow[c] -= J[l] e.
 * Everything is resolved at compile time (column masks, local indices), so the body is straight-line FMA code. */
template <int D, int BASE, unsigned MASK, int NC>
__device__ __forceinline__ void gram_row(const double* __restrict__ jr_base, double e, double (&acc)[4][11], double (&brow)[4]) {
  constexpr int LMAX = (4 * D + 3 < NC - 1) ? 4 * D + 3 : NC - 1; /* highest local column this pose touches */
  if constexpr (4 * D < NC) {
    double jr[NC];
#pragma unroll
    for (int col = 0; col < NC; ++col) jr[col] = (((MASK >> col) & 1u) && col <= LMAX) ? jr_base[(BASE + cidx(MASK, col)) * KA2_NT] : 0.0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int l = 4 * D + c;
      if (l < NC && ((MASK >> l) & 1u)) {
        const double jl = jr[l];
        brow[c] -= jl * e;
#pragma unroll
        for (int o = 0; o <= 10; ++o) {
          const int col = l - o;
          if (col >= 0 && ((MASK >> col) & 1u)) acc[c][o] += jl * jr[col];
        }
      }
    }
  }
}

/* all rows of the anchor D poses back (record at jr_base = sJ + slot - D) */
template <bool HOLO, int D>
__device__ __forceinline__ void gram_anchor(const KParams& kp, const double* __restrict__ jr_base, double (&acc)[4][11],
                                            double (&brow)[4]) {
  using L = JL<HOLO>;
  const double* E = jr_base + L::E * KA2_NT;
  if (D < 2) { /* 7-column rows reach local columns 0..6 only */
    if (kp.has_vel) {
      const double ev = E[E_V * KA2_NT], ew = E[E_W * KA2_NT];
      if (ev != 0) gram_row<D, L::V, M_V, 7>(jr_base, ev, acc, brow);
      if (ew != 0) gram_row<D, L::W, M_W, 7>(jr_base, ew, acc, brow);
      if (HOLO) {
        const double ey = E[E_VY * KA2_NT];
        if (ey != 0) gram_row<D, L::VY, M_VY, 6>(jr_base, ey, acc, brow);
      }
    }
    if (kp.has_kin) {
      const double e0 = E[E_K0 * KA2_NT], e1 = E[E_K1 * KA2_NT];
      if (e0 != 0) gram_row<D, L::K0, M_K, 7>(jr_base, e0, acc, brow);
      if (e1 != 0) gram_row<D, L::K1, M_K, 7>(jr_base, e1, acc, brow);
    }
    if (kp.has_sp) {
      const double e = E[E_SP * KA2_NT];
      if (e != 0) gram_row<D, L::SP, M_SP, 6>(jr_base, e, acc, brow);
    }
    if (kp.has_rot) {
      const double e = E[E_ROT * KA2_NT];
      if (e != 0) gram_row<D, L::ROT, M_ROT, 7>(jr_base, e, acc, brow);
    }
  }
  if (kp.has_acc) {
    const double e0 = E[E_A0 * KA2_NT], e1 = E[E_A1 * KA2_NT];
    if (e0 != 0) gram_row<D, L::A0, M_A0, 11>(jr_base, e0, acc, brow);
    if (e1 != 0) gram_row<D, L::A1, M_A1, 11>(jr_base, e1, acc, brow);
    if (HOLO) {
      const double e2 = E[E_A2 * KA2_NT];
      if (e2 != 0) gram_row<D, L::A2, M_A0, 11>(jr_base, e2, acc, brow);
    }
  }
}

/* EdgeAccelerationStart rows (anchor 0 only; CTA-shared dense 3 x 7 block): local column l = 4 D + c */
template <bool HOLO, int D>
__device__ __forceinline__ void gram_start(const double* sStart, double (&acc)[4][11], double (&brow)[4]) {
#pragma unroll
  for (int k = 0; k < (HOLO ? 3 : 2); ++k) {
    const double e = sStart[START_E + k];
    if (e == 0) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int l = 4 * D + c;
      if (l <= 6) {
        const double jl = sStart[7 * k + l];
        brow[c] -= jl * e;
#pragma unroll
        for (int o = 0; o <= 6; ++o)
          if (o <= l) acc[c][o] += jl * sStart[7 * k + l - o];
      }
    }
  }
}

/* unary terms of pose i with the first association word already in a register (prefetched before the TMA wait) */
/* GT (global-table path): so is the scene's table in global memory, mask0 the pose's first OCCUPANCY word, and only
 * the association words it marks are read */
template <bool GEOM, bool GT = false>
__device__ __forceinline__ void unary_terms2(const KParams& kp, const DevBatch& db, int b, int sc, int i, int n, double px,
                                             double py, double cs, double sn, const TebObstacle* so, unsigned long long mask0,
                                             double U[6], double ub[3], double& chi_obst, double& chi_via) {
  if (i < 1 || i > n - 2) return;
  const double* pool = db.obst_vertices + (size_t)sc * db.PV_cap * 2; /* only dereferenced for vertex-list obstacles */
  if (kp.has_obst) {
    const unsigned long long* assoc = db.assoc + ((size_t)b * db.n_cap + i) * db.MW;
    const unsigned long long* oc = db.occ + ((size_t)b * db.n_cap + i) * db.OW;
    unsigned long long ow = mask0;
    int o = 1;
    for (int w = 0; GT ? true : w < db.MW; ++w) {
      if constexpr (GT) { /* next non-zero association word, in increasing order */
        while (ow == 0ull && o < db.OW) ow = oc[o++];
        if (ow == 0ull) break;
        w = ((o - 1) << 6) + __ffsll((long long)ow) - 1;
        ow &= ow - 1;
      }
      unsigned long long mask = GT ? assoc[w] : (w == 0) ? mask0 : assoc[w];
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
        if (kappa != 0 || beta != 0) {
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
      if (kappa != 0 || beta != 0) {
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
      if (e > 0) {
        const double gx = dx / e, gy = dy / e;
        U[0] += wv * gx * gx; U[1] += wv * gx * gy; U[2] += wv * gy * gy;
        ub[0] -= wv * e * gx; ub[1] -= wv * e * gy;
      }
    }
  }
}

__device__ __forceinline__ double shfl_down1(double v) { return __shfl_down_sync(0xffffffffu, v, 1); }

/* ------------------------------------------------------------------ P1 - P4 and the tile partials of one warp tile
 * (shared by k_linearize2 and k_linearize2p). Lane `lane` owns pose / anchor i, whose staged record starts at pa (the
 * next poses follow at pa + 4, pa + 8); so is the scene's obstacle table (shared or global memory), mask0 the first
 * association (GT: occupancy) word of pose i, sW / sStart the warp's record region and start block, tile the index of
 * the tile partials. mid() runs between P1 and P2, after the neighbour shuffles: it must leave the warp's records and
 * start block zeroed and the warp converged. */
template <bool HOLO, bool GEOM, bool OUT_DIRECT, bool GT, class Mid>
__device__ __forceinline__ void ka2_tile(const DevBatch& db, const KParams& kp, int b, int s, int n, int i, int lane,
                                         const double* pa, const TebObstacle* so, unsigned long long mask0, double* sW,
                                         double* sStart, int tile, Mid mid) {
  const bool out = (lane >= 2 && lane <= 30 && i < n);
  double chi[4] = {0, 0, 0, 0}; /* obstacles, via, time-optimal, other */
  const bool have_pose = (i >= 0 && i < n);
  double cs = 1, sn = 0;
  SegDer sd;
  sd.v = 0; sd.w = 0; sd.idt = 0;
#pragma unroll
  for (int k = 0; k < 6; ++k) sd.dv[k] = 0;
  double U[6] = {0, 0, 0, 0, 0, 0}, ub[3] = {0, 0, 0};
  /* ---- P1 */
  if (have_pose) {
    sincos(pa[2], &sn, &cs);
    if (i <= n - 2) sd = seg_derivs(kp, pa[0], pa[1], pa[2], cs, sn, pa[4], pa[5], pa[6], pa[3]);
    if (out) unary_terms2<GEOM, GT>(kp, db, b, s, i, n, pa[0], pa[1], cs, sn, so, mask0, U, ub, chi[0], chi[1]);
  }
  /* the right neighbour's sin / cos and segment bundle (lane 31 receives nothing useful and anchors nothing) */
  SegDer sd2;
  const double cb = shfl_down1(cs), sb = shfl_down1(sn);
  sd2.v = shfl_down1(sd.v); sd2.w = shfl_down1(sd.w); sd2.idt = shfl_down1(sd.idt);
#pragma unroll
  for (int k = 0; k < 6; ++k) sd2.dv[k] = shfl_down1(sd.dv[k]);
  mid();
  /* ---- P2: chain edges anchored at i */
  if (have_pose && i <= n - 2 && lane < 31) {
    JRec J;
    J.rec = sW + lane;
    const double c3 = anchor_rows2<HOLO>(kp, db, b, i, n, pa, cs, sn, cb, sb, sd, sd2, J, sStart);
    if (lane >= 2) chi[3] += c3; /* halo anchors belong to the previous tile */
  }
  __syncwarp();
  /* ---- P3: band rows of pose i */
  double acc[4][11];
  double brow[4] = {0, 0, 0, 0};
#pragma unroll
  for (int c = 0; c < 4; ++c)
#pragma unroll
    for (int k = 0; k < 11; ++k) acc[c][k] = 0;
  double dm = 0;
  if (out) {
    const double* rec = sW + lane;
    if (i <= n - 2) gram_anchor<HOLO, 0>(kp, rec, acc, brow);
    if (i >= 1) gram_anchor<HOLO, 1>(kp, rec - 1, acc, brow);
    if (i >= 2) gram_anchor<HOLO, 2>(kp, rec - 2, acc, brow); /* anchor i-2 <= n-3 always exists here */
    if (kp.has_acc) {
      if (i == 0) gram_start<HOLO, 0>(sStart, acc, brow);
      if (i == 1) gram_start<HOLO, 1>(sStart, acc, brow);
    }
    /* unary block (obstacles, dynamic obstacles, via-points) and the time-optimal term */
    acc[0][0] += U[0]; brow[0] += ub[0];
    acc[1][0] += U[2]; acc[1][1] += U[1]; brow[1] += ub[1];
    acc[2][0] += U[5]; acc[2][1] += U[4]; acc[2][2] += U[3]; brow[2] += ub[2];
    if (kp.has_time && i <= n - 2) { /* EdgeTimeOptimal edge_time_optimal.h:93 */
      chi[2] += kp.p.weight_optimaltime * pa[3] * pa[3];
      acc[3][0] += kp.p.weight_optimaltime; brow[3] -= kp.p.weight_optimaltime * pa[3];
    }
    if (i == 0 || i >= n - 1) { /* fixed start / goal pose, non-existent dt_{n-1}: identity rows (first / last lane only) */
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (c == 3 && i <= n - 2) continue; /* dt_0 is a real unknown */
#pragma unroll
        for (int k = 0; k < 11; ++k) acc[c][k] = 0;
        acc[c][0] = 1.0;
        brow[c] = 0;
      }
      dm = (i <= n - 2) ? fabs(acc[3][0]) : 0.0;
    } else {
      dm = fmax(fmax(fabs(acc[0][0]), fabs(acc[1][0])), fmax(fabs(acc[2][0]), fabs(acc[3][0])));
    }
  }
  /* ---- P4 */
  if (OUT_DIRECT) {
    if (out) {
      double2* g2 = reinterpret_cast<double2*>(db.Hb + ((size_t)b * 4 * db.n_cap + 4 * (size_t)i) * HROW);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
#pragma unroll
        for (int k = 0; k < 5; ++k) g2[6 * c + k] = make_double2(acc[c][2 * k], acc[c][2 * k + 1]);
        g2[6 * c + 5] = make_double2(acc[c][10], brow[c]);
      }
      double2* r2 = reinterpret_cast<double2*>(db.rhs + (size_t)b * 4 * db.n_cap + 4 * (size_t)i);
      r2[0] = make_double2(brow[0], brow[1]);
      r2[1] = make_double2(brow[2], brow[3]);
    }
  } else {
    __syncwarp(); /* every lane is done reading the records (and the poses): the region becomes the output slots */
    if (out) {
      double2* o2 = reinterpret_cast<double2*>(sW + (size_t)lane * OUT_STRIDE);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
#pragma unroll
        for (int k = 0; k < 5; ++k) o2[6 * c + k] = make_double2(acc[c][2 * k], acc[c][2 * k + 1]);
        o2[6 * c + 5] = make_double2(acc[c][10], brow[c]);
      }
      double2* r2 = reinterpret_cast<double2*>(db.rhs + (size_t)b * 4 * db.n_cap + 4 * (size_t)i);
      r2[0] = make_double2(brow[0], brow[1]);
      r2[1] = make_double2(brow[2], brow[3]);
      fence_proxy_async();
      tma_store_1d(db.Hb + ((size_t)b * 4 * db.n_cap + 4 * (size_t)i) * HROW, o2, 4 * HROW * 8u);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  /* tile partials: chi2 by family and the max diagonal of the real rows (computeLambdaInit), fixed order */
#pragma unroll
  for (int k = 0; k < 4; ++k) chi[k] = warp_sum(chi[k]);
  dm = warp_max(dm);
  if (lane == 0) {
    double* cp = db.chi_parts + ((size_t)b * db.chunks + tile) * 4;
    cp[0] = chi[0]; cp[1] = chi[1]; cp[2] = chi[2]; cp[3] = chi[3];
    db.dmax_parts[(size_t)b * db.chunks + tile] = dm;
  }
}

/* ------------------------------------------------------------------ k_linearize2 */
/* GT = global-table path (M_cap > STAGED_MAX_OBST): no TMA copy of the scene's obstacle table, rows read from global
 * memory, associations walked via the occupancy words */
template <bool HOLO, bool GEOM, bool OUT_DIRECT, bool GT = false>
__global__ void __launch_bounds__(KA2_THREADS, 3) k_linearize2(const __grid_constant__ DevBatch db, const __grid_constant__ KParams kp) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  using L = JL<HOLO>;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* sP = reinterpret_cast<double*>(smem_raw);                      /* poses, slot j <-> pose P0 + j */
  double* sW = sP + KA2Smem::POSES + (size_t)warp * KA2Smem::warp_doubles<HOLO>(); /* this warp's records / output slots */
  double* sStart = sW + KA2Smem::rec_doubles<HOLO>();                    /* EdgeAccelerationStart rows (tile of anchor 0) */
  uint64_t* bar = reinterpret_cast<uint64_t*>(sP + KA2Smem::POSES + (size_t)KA2_W * KA2Smem::warp_doubles<HOLO>());
  TebObstacle* so_s = reinterpret_cast<TebObstacle*>((reinterpret_cast<uintptr_t>(bar) + 16 + 15) & ~static_cast<uintptr_t>(15));

  /* everything the prologue needs is loaded at once: no chain of dependent global loads */
  const int y = blockIdx.y;
  int b = y, skip = 0;
  if (db.a_list) { if (y < *db.a_cnt) b = db.a_list[y]; else skip = 1; }
  else if (db.skip_tag != 0 && deferred_since(db.defer[y], db.skip_tag)) skip = 1;
  if (skip) return; /* uniform for the CTA */
  const int active = db.state[b].active;
  const int n = db.n[b];
  const int s = db.scene_id[b];
  const int P0 = blockIdx.x * (KA2_W * KA2_TP) - 2;                       /* pose of slot 0 */
  const int lo = max(P0, 0), hi = min(P0 + KA2_SLOTS, db.n_cap);          /* staged range: independent of n */
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
  }
  if (!active || P0 + 2 >= n) return;                                     /* uniform for the CTA, nothing in flight yet */
  if (tid == 0) {
    const uint32_t bytesP = (uint32_t)(hi - lo) * 32u;
    const uint32_t bytesO = GT ? 0u : (uint32_t)db.M_cap * (uint32_t)sizeof(TebObstacle);
    mbar_expect_tx(bar, bytesP + bytesO);
    tma_load_1d(sP + (size_t)(lo - P0) * 4, db.poses + ((size_t)b * db.n_cap + lo) * 4, bytesP, bar);
    if (bytesO) tma_load_1d(so_s, db.obstacles + (size_t)s * db.M_cap, bytesO, bar);
  }
  const int slot = warp * KA2_TP + lane;
  const int i = P0 + slot;                                                /* pose / anchor of this lane */
  const int q0 = P0 + 2 + warp * KA2_TP;                                  /* first pose this warp produces */
  const bool out = (lane >= 2 && lane <= 30 && i < n);
  /* while the copies are in flight: association word of the own pose, zeroed record and start block */
  unsigned long long mask0 = 0ull;
  if (out && kp.has_obst && i >= 1 && i <= n - 2)
    mask0 = GT ? db.occ[((size_t)b * db.n_cap + i) * db.OW] : db.assoc[((size_t)b * db.n_cap + i) * db.MW];
  {
    double* rec = sW + lane;
#pragma unroll
    for (int e = 0; e < L::COUNT; ++e) rec[e * 32] = 0.0;
    if (lane < KA2Smem::START) sStart[lane] = 0.0;
  }
  __syncthreads(); /* the mbarrier initialisation is visible to every waiting thread (the only block-wide barrier) */
  mbar_wait(bar, 0);
  if (q0 >= n) return; /* whole warp: tile beyond the band */
  ka2_tile<HOLO, GEOM, OUT_DIRECT, GT>(db, kp, b, s, n, i, lane, sP + 4 * slot, GT ? db.obstacles + (size_t)s * db.M_cap : so_s,
                                       mask0, sW, sStart, blockIdx.x * KA2_W + warp,
                                       [] { __syncwarp(); /* start block zeroed by other lanes */ });
  if (!OUT_DIRECT && out) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); /* the slot must outlive the copy's read */
}

/* ------------------------------------------------------------------ k_linearize2p
 * Kernel A in a PERSISTENT grid of one-warp CTAs, as many as are resident. A unit is one (band slot, tile) pair: slot y
 * of the launch (band y, or a_list[y] for the first *a_cnt slots of a listed launch) and its tile t = 0 .. chunks - 1,
 * unit y chunks + t. Warp w of G takes the units w, w + G, w + 2G, ... and skips, before it touches shared memory, a
 * unit whose band is deferred (skip_tag) or inactive or whose first pose q0 = 29 t is >= n. Per unit it runs
 * k_linearize2's P1 - P4 (ka2_tile: same lanes, same formulas, same fold order, the padded output slot and one bulk
 * store per lane, the tile partials at (b, t)), so every output is the same bits. What differs:
 *   - the tile's 33-pose window (poses q0 - 2 .. q0 + 30) is double-buffered on two per-warp mbarriers: the NEXT unit's
 *     window is TMA-issued as soon as the current unit's P1 has run, so it arrives while P2 - P4 run;
 *   - the previous unit's bulk stores drain while the current unit runs P1: the region they read becomes this unit's
 *     records only after cp.async.bulk.wait_group.read 0;
 *   - obstacle rows are read from global memory (L2: 64 B per row, one table per 32 bands on C3) with the staged
 *     association walk; the GT build walks the occupancy words as k_linearize2<., ., ., true> does. A shared copy of
 *     the table would cost a resident warp per SM (20.3 KB per warp with C3's 4 KB table: 11 warps instead of 12).
 * No prologue per tile (mbarrier set-up, block barrier, cold window and table loads) and no idle warp in a band's last
 * CTA. Non-holonomic builds: 15.6 KB of shared memory per warp, 12 warps per SM (the 168-register cap); holonomic
 * builds: 20.5 KB, 10 warps per SM. */
constexpr int KA2P_SLOTS = KA2_TP + 4; /* poses staged per unit: slot j <-> pose q0 - 2 + j */
template <bool HOLO>
__host__ __device__ constexpr size_t ka2p_smem_bytes() {
  return (2 * KA2P_SLOTS * 4 + KA2Smem::warp_doubles<HOLO>()) * sizeof(double) + 2 * sizeof(uint64_t);
}

template <bool HOLO, bool GEOM, bool GT = false>
__global__ void __launch_bounds__(32, 12) k_linearize2p(const __grid_constant__ DevBatch db, const __grid_constant__ KParams kp,
                                                        int B) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  using L = JL<HOLO>;
  const int lane = threadIdx.x;
  double* sPw = reinterpret_cast<double*>(smem_raw);                        /* two windows of KA2P_SLOTS poses */
  double* sW = sPw + 2 * KA2P_SLOTS * 4;                                     /* records / output slots */
  double* sStart = sW + KA2Smem::rec_doubles<HOLO>();                        /* EdgeAccelerationStart rows */
  uint64_t* bar = reinterpret_cast<uint64_t*>(sW + KA2Smem::warp_doubles<HOLO>());

  const int units = (db.a_list ? *db.a_cnt : B) * db.chunks;
  const int step = (int)gridDim.x;
  /* the first unit at or after u of this warp that has work: its band, n and first pose (every lane computes the same) */
  auto next_unit = [&](int u, int& b, int& n, int& q0) {
    for (; u < units; u += step) {
      const int y = u / db.chunks;
      const int t = u - y * db.chunks;
      int bb = y;
      if (db.a_list) bb = db.a_list[y];
      else if (db.skip_tag != 0 && deferred_since(db.defer[y], db.skip_tag)) continue;
      const int nn = db.n[bb];
      if (!db.state[bb].active || t * KA2_TP >= nn) continue;
      b = bb; n = nn; q0 = t * KA2_TP;
      return u;
    }
    return units;
  };
  /* lane 0: the window of the unit (b, q0) into buffer k; the range staged does not depend on n, as in k_linearize2 */
  auto issue = [&](int k, int b, int q0) {
    const int P0 = q0 - 2;
    const int lo = max(P0, 0), hi = min(P0 + KA2P_SLOTS, db.n_cap);
    const uint32_t bytes = (uint32_t)(hi - lo) * 32u;
    mbar_expect_tx(&bar[k], bytes);
    tma_load_1d(sPw + (size_t)k * KA2P_SLOTS * 4 + (size_t)(lo - P0) * 4, db.poses + ((size_t)b * db.n_cap + lo) * 4, bytes, &bar[k]);
  };

  int b = 0, n = 0, q0 = 0;
  int u = next_unit((int)blockIdx.x, b, n, q0);
  if (u >= units) return;
  if (lane == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    mbar_fence_init();
  }
  __syncwarp();
  if (lane == 0) issue(0, b, q0);
  int k = 0;           /* buffer of the current unit */
  uint32_t parity = 0; /* bit j: parity of bar[j]'s next phase */
  while (u < units) {
    const int s = db.scene_id[b];
    const int i = q0 - 2 + lane;                                            /* pose / anchor of this lane */
    unsigned long long mask0 = 0ull;
    if (lane >= 2 && lane <= 30 && i < n && kp.has_obst && i >= 1 && i <= n - 2)
      mask0 = GT ? db.occ[((size_t)b * db.n_cap + i) * db.OW] : db.assoc[((size_t)b * db.n_cap + i) * db.MW];
    mbar_wait(&bar[k], (parity >> k) & 1u);
    parity ^= 1u << k;
    int b_nx = 0, n_nx = 0, q0_nx = 0, u_nx = units;
    ka2_tile<HOLO, GEOM, false, GT>(db, kp, b, s, n, i, lane, sPw + (size_t)k * KA2P_SLOTS * 4 + 4 * lane,
                                    db.obstacles + (size_t)s * db.M_cap, mask0, sW, sStart, q0 / KA2_TP, [&] {
      /* the next unit's window goes into the other buffer, which the previous unit finished reading before its P4 */
      u_nx = next_unit(u + step, b_nx, n_nx, q0_nx);
      if (lane == 0 && u_nx < units) issue(k ^ 1, b_nx, q0_nx);
      /* the previous unit's bulk stores have read their output slots: the region becomes this unit's records */
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      __syncwarp();
      double* rec = sW + lane;
#pragma unroll
      for (int e = 0; e < L::COUNT; ++e) rec[e * 32] = 0.0;
      if (lane < KA2Smem::START) sStart[lane] = 0.0;
      __syncwarp(); /* records and start block zeroed by every lane */
    });
    u = u_nx; b = b_nx; n = n_nx; q0 = q0_nx;
    k ^= 1;
  }
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); /* the slots must outlive the copies' reads */
}

}  // namespace tebgpu
