/*
 * teb_hsig.cuh — batched H-signatures: HomotopyClassPlanner::calculateEquivalenceClass (homotopy_class_planner.hpp:46-63)
 * for every band of a batch, the step that decides which candidates exist before they are optimised
 * (renewAndAnalyzeOldTebs homotopy_class_planner.cpp:214-256, graph search graph_search.cpp).
 *
 *   k_hsig2d  HSignature::calculateHSignature   h_signature.h:97-186   one complex value per band
 *   k_hsig3d  HSignature3d::calculateHSignature h_signature.h:282-353  one value per (band, obstacle)
 *
 * One CTA per band. The reference accumulates the 2-D signature in long double on one thread; here every (segment,
 * obstacle) term is evaluated by its own thread in fp64 and summed by a fixed-order block reduction. Two places where
 * fp64 alone would part from long double are handled explicitly:
 *   - the skip rule |o_l - o_j| < 0.05 is decided on the exact difference (hsig_closer_than_skip), not on the rounded one;
 *   - A_l = f0 / prod_j (o_l - o_j) is carried as an fp64 mantissa and a binary exponent, and the sum over (k, l) is
 *     taken at the largest exponent and scaled once, so that a partial product may leave the fp64 range (far obstacles
 *     listed before near ones) and the result overflows / underflows only where (double) of the long double one does.
 */
#pragma once

#include <climits>

#include "teb_kernels.cuh"

namespace tebgpu {

constexpr int HSIG_THREADS = 256;

__host__ __device__ inline size_t hsig_smem_bytes(int n_cap, int M_cap) {
  const size_t Mc = M_cap > 0 ? M_cap : 1;
  return ((size_t)4 * Mc + (size_t)3 * n_cap + 2 * (HSIG_THREADS / 32) + (Mc + 1) / 2 + 8) * sizeof(double);
}

/* |(ax, ay) - (bx, by)| < 0.05 on the exact difference: each coordinate difference as a two-sum (hi + lo exactly), the
 * squared modulus as a double-double, compared with 0.05 * 0.05 as a double-double. Differs from the exact decision only
 * within about 1e-30 relative of the threshold (long double's own decision: about 1e-19). */
__device__ __forceinline__ bool hsig_closer_than_skip(double ax, double ay, double bx, double by) {
  const double dx = ax - bx, vx = dx - ax, ex = (ax - (dx - vx)) + (-bx - vx);
  const double dy = ay - by, vy = dy - ay, ey = (ay - (dy - vy)) + (-by - vy);
  const double px = dx * dx, pxe = fma(dx, dx, -px);
  const double py = dy * dy, pye = fma(dy, dy, -py);
  const double s = px + py, vs = s - px, se = (px - (s - vs)) + (py - vs);
  const double lo = se + pxe + pye + 2.0 * (dx * ex + dy * ey) + (ex * ex + ey * ey);
  const double c = 0.05, c2 = c * c, c2e = fma(c, c, -c2);
  return (s - c2) + (lo - c2e) < 0.0; /* s - c2 is exact here (Sterbenz): this path runs only when s is within 1e-12 of c2 */
}

/* the band's n and scene_id index the staging and the scene's tables; obst_count is range-checked by the caller */
__device__ __forceinline__ bool hsig_band_ok(const DevBatch& db, int n, int sc) {
  return n >= 0 && n <= db.n_cap && sc >= 0 && sc < db.S;
}

__global__ void __launch_bounds__(HSIG_THREADS) k_hsig2d(DevBatch db, KParams kp, double* out) {
  extern __shared__ __align__(16) unsigned char hs_raw[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = db.n[b];
  const int sc = db.scene_id[b];
  const int M = hsig_band_ok(db, n, sc) ? db.obst_count[sc] : -1;
  const int Mc = db.M_cap > 0 ? db.M_cap : 1;
  if (M < 0 || M > db.M_cap) { /* a scene the batch cannot describe (device pointers only): no signature */
    if (tid == 0) { out[2 * b] = NAN; out[2 * b + 1] = NAN; }
    return;
  }
  double* sox = reinterpret_cast<double*>(hs_raw);
  double* soy = sox + Mc;
  double* sAr = soy + Mc;
  double* sAi = sAr + Mc;
  double* spx = sAi + Mc;
  double* spy = spx + db.n_cap;
  double* sred = spy + 2 * db.n_cap; /* [2][warps] */
  int* sE = reinterpret_cast<int*>(sred + 2 * (HSIG_THREADS / 32)); /* [Mc] binary exponent of A_l */
  __shared__ int sEmax;
  if (M == 0 || n < 1) { /* obstacles->empty(): hsignature_ = 0 (:100-104) */
    if (tid == 0) { out[2 * b] = 0; out[2 * b + 1] = 0; }
    return;
  }
  if (tid == 0) sEmax = INT_MIN;
  const TebObstacle* go = db.obstacles + (size_t)sc * db.M_cap;
  for (int l = tid; l < M; l += HSIG_THREADS) { sox[l] = go[l].x; soy[l] = go[l].y; } /* getCentroidCplx() */
  const double* P = db.poses + (size_t)b * db.n_cap * 4;
  for (int k = tid; k < n; k += HSIG_THREADS) { spx[k] = P[4 * k]; spy[k] = P[4 * k + 1]; }
  __syncthreads();
  /* f0 parameters a, b (:108-111) and the coarse map rectangle spanned by start / goal (:121-135) */
  const int m = max(M - 1, 5);
  const int a = (int)ceil((double)m / 2.0);
  const int bq = m - a;
  const double sx = spx[0], sy = spy[0];
  const double dx = spx[n - 1] - sx, dy = spy[n - 1] - sy;
  double blx, bly, trx, try_;
  if (hypot(dx, dy) < 3.0) { blx = sx; bly = sy - 3; trx = sx + 3; try_ = sy + 3; }
  else { blx = sx + dy; bly = sy - dx; trx = sx + dx - dy; try_ = sy + dy + dx; } /* normal = (-dy, dx) */
  /* A_l = f0(o_l) / prod_{j != l, |o_l - o_j| >= 0.05} (o_l - o_j)  (:149-163), as (ar + i ai) * 2^E: the long double
   * product of the reference may pass far outside the fp64 range on its way to an O(1) value */
  for (int l = tid; l < M; l += HSIG_THREADS) {
    const double ox = sox[l], oy = soy[l];
    const double pa = kp.p.h_signature_prescaler * (double)a;
    double ar = pa * (ox - blx), ai = pa * (oy - bly);
    ar *= (double)bq; ai *= (double)bq;
    { const double cr = ox - trx, ci = oy - try_; const double tr = ar * cr - ai * ci; ai = ar * ci + ai * cr; ar = tr; }
    int E = 0;
    for (int j = 0; j < M; ++j) {
      if (j == l) continue;
      const double cr = ox - sox[j], ci = oy - soy[j];
      const double den = cr * cr + ci * ci;
      /* skip really close obstacles; near the threshold the decision is taken on the exact difference */
      if (den < 0.0025 * (1 - 1e-12)) continue;
      if (den <= 0.0025 * (1 + 1e-12) && hsig_closer_than_skip(ox, oy, sox[j], soy[j])) continue;
      const double tr = (ar * cr + ai * ci) / den;
      ai = (ai * cr - ar * ci) / den;
      ar = tr;
      const double mx = fmax(fabs(ar), fabs(ai));
      if ((mx > 0x1p+400 || mx < 0x1p-400) && mx > 0 && mx < INFINITY) { /* renormalise: exact scaling by 2^-e */
        int e;
        frexp(mx, &e);
        ar = ldexp(ar, -e); ai = ldexp(ai, -e);
        E += e;
      }
    }
    sAr[l] = ar; sAi[l] = ai;
    sE[l] = (ar == 0 && ai == 0) ? INT_MIN : E;
    if (ar != 0 || ai != 0) atomicMax(&sEmax, E);
  }
  __syncthreads();
  /* every A_l at the largest exponent (exact unless a term falls below 2^-1022 of the largest one) */
  const int Emax = sEmax;
  for (int l = tid; l < M; l += HSIG_THREADS) {
    if (sE[l] != INT_MIN) { sAr[l] = ldexp(sAr[l], sE[l] - Emax); sAi[l] = ldexp(sAi[l], sE[l] - Emax); }
  }
  __syncthreads();
  /* sum over segments k and obstacles l of A_l * (ln|z2-o|/|z1-o| + i * smallest-magnitude angle difference) (:165-182) */
  double hr = 0, hi = 0;
  const int pairs = (n - 1) * M;
  for (int idx = tid; idx < pairs; idx += HSIG_THREADS) {
    const int k = idx / M, l = idx - k * M;
    const double ox = sox[l], oy = soy[l];
    const double x1 = spx[k] - ox, y1 = spy[k] - oy, x2 = spx[k + 1] - ox, y2 = spy[k + 1] - oy;
    const double d2 = hypot(x2, y2), d1 = hypot(x1, y1);
    if (d2 == 0 || d1 == 0) continue;
    const double lr = log(d2) - log(d1);
    const double ad = atan2(y2, x2) - atan2(y1, x1);
    double li = ad;
    const double two_pi = 2 * 3.14159265358979323846;
    if (fabs(ad + two_pi) < fabs(li)) li = ad + two_pi;
    if (fabs(ad - two_pi) < fabs(li)) li = ad - two_pi;
    if (fabs(ad + 2 * two_pi) < fabs(li)) li = ad + 2 * two_pi;
    if (fabs(ad - 2 * two_pi) < fabs(li)) li = ad - 2 * two_pi;
    hr += sAr[l] * lr - sAi[l] * li;
    hi += sAr[l] * li + sAi[l] * lr;
  }
  hr = warp_sum(hr); hi = warp_sum(hi);
  const int lane = tid & 31, w = tid >> 5;
  if (lane == 0) { sred[w] = hr; sred[HSIG_THREADS / 32 + w] = hi; }
  __syncthreads();
  if (tid == 0) {
    double r = 0, i = 0;
    for (int q = 0; q < HSIG_THREADS / 32; ++q) { r += sred[q]; i += sred[HSIG_THREADS / 32 + q]; }
    /* one scaling to the true exponent: inf / 0 exactly where the long double value lies outside the fp64 range */
    if (Emax != INT_MIN) { r = ldexp(r, Emax); i = ldexp(i, Emax); }
    out[2 * b] = r; out[2 * b + 1] = i;
  }
}

__global__ void __launch_bounds__(HSIG_THREADS) k_hsig3d(DevBatch db, KParams kp, int use_timediffs, double* out) {
  extern __shared__ __align__(16) unsigned char hs_raw[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = db.n[b];
  const int sc = db.scene_id[b];
  const int M = hsig_band_ok(db, n, sc) ? db.obst_count[sc] : -1;
  const int Mc = db.M_cap > 0 ? db.M_cap : 1;
  if (M < 0 || M > db.M_cap) { /* a scene the batch cannot describe (device pointers only): no signature */
    for (int l = tid; l < Mc; l += HSIG_THREADS) out[(size_t)b * Mc + l] = NAN;
    return;
  }
  double* spx = reinterpret_cast<double*>(hs_raw) + 4 * Mc;
  double* spy = spx + db.n_cap;
  double* sT = spy + db.n_cap; /* transition time at pose k */
  const double* P = db.poses + (size_t)b * db.n_cap * 4;
  for (int k = tid; k < n; k += HSIG_THREADS) { spx[k] = P[4 * k]; spy[k] = P[4 * k + 1]; }
  __syncthreads();
  if (tid == 0) { /* transition times, sequential like the reference (:305-315) */
    double t = 0;
    for (int k = 0; k < n; ++k) {
      sT[k] = t;
      if (k + 1 < n) t += use_timediffs ? P[4 * k + 3] : hypot(spx[k + 1] - spx[k], spy[k + 1] - spy[k]) / kp.p.max_vel_x;
    }
  }
  __syncthreads();
  const TebObstacle* go = db.obstacles + (size_t)sc * db.M_cap;
  const int lane = tid & 31, w = tid >> 5;
  for (int l = w; l < Mc; l += HSIG_THREADS / 32) { /* rows past M (and the one row of M_cap = 0) are written as 0 */
    double H = 0;
    if (l < M) {
      /* obstacle world line s1 -> s2 over 120 s (predictCentroidConstantVelocity), the "conductor" (:291-298) */
      const double tt = 120;
      const double s1x = go[l].x, s1y = go[l].y, s1z = 0;
      const double s2x = go[l].x + tt * go[l].vx, s2y = go[l].y + tt * go[l].vy, s2z = tt;
      const double dsx = s2x - s1x, dsy = s2y - s1y, dsz = s2z - s1z;
      const double ds2 = dsx * dsx + dsy * dsy + dsz * dsz;
      for (int k = lane; k + 1 < n; k += 32) {
        const double dirx = spx[k + 1] - spx[k], diry = spy[k + 1] - spy[k], dirz = sT[k + 1] - sT[k];
        if (sqrt(dirx * dirx + diry * diry + dirz * dirz) < 1e-15) continue; /* coincident poses */
        double rx = spx[k], ry = spy[k], rz = sT[k];
        const double dlx = 0.1 * dirx, dly = 0.1 * diry, dlz = 0.1 * dirz;
        for (int i = 0; i < 10; ++i) {
          const double p1x = s1x - rx, p1y = s1y - ry, p1z = s1z - rz;
          const double p2x = s2x - rx, p2y = s2y - ry, p2z = s2z - rz;
          const double cx = p1y * p2z - p1z * p2y, cy = p1z * p2x - p1x * p2z, cz = p1x * p2y - p1y * p2x;
          const double dx = (dsy * cz - dsz * cy) / ds2, dy = (dsz * cx - dsx * cz) / ds2, dz = (dsx * cy - dsy * cx) / ds2;
          const double n1 = sqrt(p1x * p1x + p1y * p1y + p1z * p1z), n2 = sqrt(p2x * p2x + p2y * p2y + p2z * p2z);
          const double ax = dy * p2z - dz * p2y, ay = dz * p2x - dx * p2z, az = dx * p2y - dy * p2x;
          const double bx = dy * p1z - dz * p1y, by = dz * p1x - dx * p1z, bz = dx * p1y - dy * p1x;
          const double inv = 1.0 / (dx * dx + dy * dy + dz * dz);
          H += inv * (ax / n2 - bx / n1) * dlx + inv * (ay / n2 - by / n1) * dly + inv * (az / n2 - bz / n1) * dlz;
          rx += dlx; ry += dly; rz += dlz;
        }
      }
    }
    H = warp_sum(H);
    if (lane == 0) out[(size_t)b * Mc + l] = H / (4.0 * 3.14159265358979323846);
  }
}

}  // namespace tebgpu
