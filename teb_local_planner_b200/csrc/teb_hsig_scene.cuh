/*
 * teb_hsig_scene.cuh — H-signatures of scenes of up to 16384 obstacles, from a per-scene factor table.
 *
 * HSignature::calculateHSignature (h_signature.h:97-186) forms, for every band,
 *     A_l = f0(o_l) / prod_{j != l, |o_l - o_j| >= 0.05} (o_l - o_j)
 * where only f0 depends on the band (through the map rectangle spanned by its start and goal, :121-152). The product
 *     Q_l = 1 / prod_{j != l, |o_l - o_j| >= 0.05} (o_l - o_j)
 * depends only on the scene (the reference's own TODO at :120), so it is built once per scene and cycle:
 *
 *   k_hsig_factors          Q_l of every row of every scene, all-pairs ("n-body") tiles: one thread per row l, the
 *                           scene's rows j staged tile by tile through shared memory, the j range cut into parts of
 *                           HSF_JCHUNK rows, one part per CTA (a 16384-row scene: 64 row blocks x 8 parts = 512 CTAs)
 *   k_hsig_factors_combine  the parts of every row multiplied in part order: the factor table
 *   k_hsig2d_scene          per band and chunk of HS2_ROWS obstacles: A_l = f0(o_l) * Q_l and the sum over segments of
 *                           A_l * L_kl, hypot / log / atan2 of z_k - o_l once per (pose, obstacle)
 *   k_hsig2d_scene_sum      per band: the chunks' partial sums in chunk order
 *   k_hsig3d_scene          HSignature3d::calculateHSignature (h_signature.h:282-353) per (band, chunk of HS3_ROWS
 *                           obstacles), obstacles read from global memory / L2, only the band's poses in shared memory
 *
 * Every partition depends on the scene's obst_count (factors) or on the band's own n and M (signatures) only, never on
 * S, B, M_cap or a position in the batch, and every reduction runs in a fixed order without atomics: a scene's table and
 * a band's signature are the same bits in every batch. Mantissa / exponent pairs as in k_hsig2d (teb_hsig.cuh): a
 * partial product may leave the fp64 range (far obstacles listed before near ones); the value is renormalised by an
 * exact 2^-e whenever its larger part leaves [2^-400, 2^400].
 */
#pragma once

#include <climits>

#include "teb_hsig.cuh"

namespace tebgpu {

constexpr int HSF_THREADS = 256;  /* rows l per factor CTA, and rows j per staged tile */
constexpr int HSF_JCHUNK = 2048;  /* rows j per part of the product */
constexpr int HS2_ROWS = 256;     /* obstacles per CTA of k_hsig2d_scene (one per thread) */
constexpr int HS3_ROWS = 64;      /* obstacles per CTA of k_hsig3d_scene (8 per warp) */

__host__ __device__ inline int hsig_parts(int M) { return M > 0 ? (M + HSF_JCHUNK - 1) / HSF_JCHUNK : 1; }

/* (ar, ai) * 2^E kept with its larger part inside [2^-400, 2^400] (exact scaling; 0, inf and NaN are left alone) */
__device__ __forceinline__ void hsig_renorm(double& ar, double& ai, int& E) {
  const double mx = fmax(fabs(ar), fabs(ai));
  if ((mx > 0x1p+400 || mx < 0x1p-400) && mx > 0 && mx < INFINITY) {
    int e;
    frexp(mx, &e);
    ar = ldexp(ar, -e); ai = ldexp(ai, -e);
    E += e;
  }
}

/* part p of Q_l: prod over j in [p * HSF_JCHUNK, min(M, (p + 1) * HSF_JCHUNK)) of 1 / (o_l - o_j), skip rule of
 * k_hsig2d. grid (S, row blocks x parts of M_cap); pm [S][parts(M_cap)][M_cap] (re, im), pe the exponents */
__global__ void __launch_bounds__(HSF_THREADS) k_hsig_factors(const TebObstacle* __restrict__ obst,
                                                              const int32_t* __restrict__ obst_count, int M_cap,
                                                              double2* __restrict__ pm, int* __restrict__ pe) {
  __shared__ double sx[HSF_THREADS], sy[HSF_THREADS];
  const int s = blockIdx.x, tid = threadIdx.x;
  const int P_cap = hsig_parts(M_cap);
  const int lb = blockIdx.y / P_cap, p = blockIdx.y - lb * P_cap;
  const int M = obst_count[s];
  if (M < 1 || M > M_cap) return; /* no rows, or a count the table cannot describe: the combine writes the row */
  const int j0 = p * HSF_JCHUNK, j1 = min(M, j0 + HSF_JCHUNK);
  if (lb * HSF_THREADS >= M || j0 >= M) return;
  const TebObstacle* go = obst + (size_t)s * M_cap;
  const int l = lb * HSF_THREADS + tid;
  const bool own = l < M;
  const double ox = own ? go[l].x : 0, oy = own ? go[l].y : 0; /* getCentroidCplx() */
  double ar = 1, ai = 0;
  int E = 0;
  for (int t = j0; t < j1; t += HSF_THREADS) {
    __syncthreads();
    if (t + tid < j1) { sx[tid] = go[t + tid].x; sy[tid] = go[t + tid].y; }
    __syncthreads();
    const int cnt = min(HSF_THREADS, j1 - t);
    if (!own) continue;
    for (int jj = 0; jj < cnt; ++jj) {
      if (t + jj == l) continue;
      const double cr = ox - sx[jj], ci = oy - sy[jj];
      const double den = cr * cr + ci * ci;
      /* skip really close obstacles; near the threshold the decision is taken on the exact difference */
      if (den < 0.0025 * (1 - 1e-12)) continue;
      if (den <= 0.0025 * (1 + 1e-12) && hsig_closer_than_skip(ox, oy, sx[jj], sy[jj])) continue;
      const double tr = (ar * cr + ai * ci) / den;
      ai = (ai * cr - ar * ci) / den;
      ar = tr;
      hsig_renorm(ar, ai, E);
    }
  }
  if (!own) return;
  const size_t at = ((size_t)s * P_cap + p) * M_cap + l;
  pm[at] = make_double2(ar, ai);
  pe[at] = (ar == 0 && ai == 0) ? INT_MIN : E;
}

/* Q_l = the parts multiplied in part order; rows past obst_count (and every row of a scene whose count is outside
 * 0 .. M_cap) are 0 with exponent INT_MIN, factor_count[s] = obst_count[s] or -1. grid (S, row blocks of M_cap) */
__global__ void __launch_bounds__(HSF_THREADS) k_hsig_factors_combine(const int32_t* __restrict__ obst_count, int M_cap,
                                                                      const double2* __restrict__ pm,
                                                                      const int* __restrict__ pe, double* factor,
                                                                      int32_t* factor_exp, int32_t* factor_count) {
  const int s = blockIdx.x, l = blockIdx.y * HSF_THREADS + threadIdx.x;
  const int M = obst_count[s];
  const bool bad = M < 0 || M > M_cap;
  if (l == 0) factor_count[s] = bad ? -1 : M;
  if (l >= M_cap) return;
  const size_t row = (size_t)s * M_cap + l;
  double r = 0, i = 0;
  int E = INT_MIN;
  if (!bad && l < M) {
    const int P = hsig_parts(M), P_cap = hsig_parts(M_cap);
    r = 1; E = 0;
    for (int p = 0; p < P; ++p) {
      const size_t at = ((size_t)s * P_cap + p) * M_cap + l;
      const double2 m = pm[at];
      const int e = pe[at];
      if (e == INT_MIN) { r = 0; i = 0; break; }
      const double tr = r * m.x - i * m.y;
      i = r * m.y + i * m.x;
      r = tr;
      E += e;
      hsig_renorm(r, i, E);
    }
    if (r == 0 && i == 0) E = INT_MIN;
  }
  factor[2 * row] = r; factor[2 * row + 1] = i;
  factor_exp[row] = E;
}

/* the band's scene and count when the band and its scene can be described, else -1 */
__device__ __forceinline__ int hsig_scene_count(const DevBatch& db, int b, int& n, int& sc) {
  n = db.n[b];
  sc = db.scene_id[b];
  const int M = hsig_band_ok(db, n, sc) ? db.obst_count[sc] : -1;
  return (M < 0 || M > db.M_cap) ? -1 : M;
}

/* chunk c of band b: obstacles [c * HS2_ROWS, min(M, (c + 1) * HS2_ROWS)), one per thread. part[b][c] = (Re, Im, E) of
 * the chunk's sum at its largest exponent E (INT_MIN: every A_l of the chunk is 0). grid (B, chunks of M_cap) */
__global__ void __launch_bounds__(HS2_ROWS) k_hsig2d_scene(DevBatch db, KParams kp, const double* __restrict__ factor,
                                                           const int32_t* __restrict__ factor_exp,
                                                           const int32_t* __restrict__ factor_count, double* part) {
  extern __shared__ __align__(16) unsigned char hs_raw[];
  __shared__ int swE[HS2_ROWS / 32];
  __shared__ double sred[2 * (HS2_ROWS / 32)];
  const int b = blockIdx.x, c = blockIdx.y, tid = threadIdx.x;
  const int C_cap = (max(db.M_cap, 1) + HS2_ROWS - 1) / HS2_ROWS;
  int n, sc;
  const int M = hsig_scene_count(db, b, n, sc);
  if (M < 1 || n < 1 || factor_count[sc] != M || c * HS2_ROWS >= M) return; /* k_hsig2d_scene_sum writes those bands */
  double* spx = reinterpret_cast<double*>(hs_raw);
  double* spy = spx + db.n_cap;
  const double* P = db.poses + (size_t)b * db.n_cap * 4;
  for (int k = tid; k < n; k += HS2_ROWS) { spx[k] = P[4 * k]; spy[k] = P[4 * k + 1]; }
  __syncthreads();
  /* f0 parameters a, b (:108-111) and the coarse map rectangle spanned by start / goal (:121-135), as k_hsig2d */
  const int m = max(M - 1, 5);
  const int a = (int)ceil((double)m / 2.0);
  const int bq = m - a;
  const double sx = spx[0], sy = spy[0];
  const double dx = spx[n - 1] - sx, dy = spy[n - 1] - sy;
  double blx, bly, trx, try_;
  if (hypot(dx, dy) < 3.0) { blx = sx; bly = sy - 3; trx = sx + 3; try_ = sy + 3; }
  else { blx = sx + dy; bly = sy - dx; trx = sx + dx - dy; try_ = sy + dy + dx; } /* normal = (-dy, dx) */
  /* A_l = f0(o_l) * Q_l as (ar + i ai) * 2^E, the larger part in [0.5, 1) */
  const int l = c * HS2_ROWS + tid;
  const bool own = l < M;
  const TebObstacle* go = db.obstacles + (size_t)sc * db.M_cap;
  const double ox = own ? go[l].x : 0, oy = own ? go[l].y : 0;
  double ar = 0, ai = 0;
  int E = INT_MIN;
  if (own) {
    const size_t row = (size_t)sc * db.M_cap + l;
    const double pa = kp.p.h_signature_prescaler * (double)a;
    double fr = pa * (ox - blx), fi = pa * (oy - bly);
    fr *= (double)bq; fi *= (double)bq;
    { const double cr = ox - trx, ci = oy - try_; const double tr = fr * cr - fi * ci; fi = fr * ci + fi * cr; fr = tr; }
    const double qr = factor[2 * row], qi = factor[2 * row + 1];
    const int qe = factor_exp[row];
    ar = fr * qr - fi * qi;
    ai = fr * qi + fi * qr;
    const double mx = fmax(fabs(ar), fabs(ai));
    if (qe == INT_MIN || mx == 0) { ar = 0; ai = 0; }
    else {
      E = qe;
      if (mx < INFINITY) { int e; frexp(mx, &e); ar = ldexp(ar, -e); ai = ldexp(ai, -e); E += e; }
    }
  }
  /* the chunk's largest exponent, then every A_l at it (exact unless a term falls below 2^-1022 of the largest one) */
  int wE = E;
  for (int o = 16; o > 0; o >>= 1) wE = max(wE, __shfl_xor_sync(0xffffffffu, wE, o));
  const int lane = tid & 31, w = tid >> 5;
  if (lane == 0) swE[w] = wE;
  __syncthreads();
  int Ec = INT_MIN;
  for (int q = 0; q < HS2_ROWS / 32; ++q) Ec = max(Ec, swE[q]);
  if (E != INT_MIN) { ar = ldexp(ar, E - Ec); ai = ldexp(ai, E - Ec); }
  /* sum over segments k of A_l * (ln|z2-o|/|z1-o| + i * smallest-magnitude angle difference) (:165-182); each pose's
   * modulus, logarithm and angle are formed once and serve the segments on both sides of it */
  double hr = 0, hi = 0;
  if (own && E != INT_MIN) {
    const double two_pi = 2 * 3.14159265358979323846;
    double x = spx[0] - ox, y = spy[0] - oy;
    double d1 = hypot(x, y), lg1 = log(d1), an1 = atan2(y, x);
    for (int k = 1; k < n; ++k) {
      x = spx[k] - ox; y = spy[k] - oy;
      const double d2 = hypot(x, y), lg2 = log(d2), an2 = atan2(y, x);
      if (d2 != 0 && d1 != 0) {
        const double lr = lg2 - lg1;
        const double ad = an2 - an1;
        double li = ad;
        if (fabs(ad + two_pi) < fabs(li)) li = ad + two_pi;
        if (fabs(ad - two_pi) < fabs(li)) li = ad - two_pi;
        if (fabs(ad + 2 * two_pi) < fabs(li)) li = ad + 2 * two_pi;
        if (fabs(ad - 2 * two_pi) < fabs(li)) li = ad - 2 * two_pi;
        hr += ar * lr - ai * li;
        hi += ar * li + ai * lr;
      }
      d1 = d2; lg1 = lg2; an1 = an2;
    }
  }
  hr = warp_sum(hr); hi = warp_sum(hi);
  if (lane == 0) { sred[w] = hr; sred[HS2_ROWS / 32 + w] = hi; }
  __syncthreads();
  if (tid == 0) {
    double r = 0, i = 0;
    for (int q = 0; q < HS2_ROWS / 32; ++q) { r += sred[q]; i += sred[HS2_ROWS / 32 + q]; }
    double* o = part + ((size_t)b * C_cap + c) * 3;
    o[0] = r; o[1] = i; o[2] = (double)Ec;
  }
}

/* one thread per band: NaN for a band or scene the batch cannot describe and for a table built at another count, 0 for
 * M = 0 or n < 1, else the chunks' sums at the largest exponent, in chunk order, scaled once to the true exponent */
__global__ void k_hsig2d_scene_sum(DevBatch db, const int32_t* __restrict__ factor_count, const double* __restrict__ part,
                                   double* out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= db.B) return;
  const int C_cap = (max(db.M_cap, 1) + HS2_ROWS - 1) / HS2_ROWS;
  int n, sc;
  const int M = hsig_scene_count(db, b, n, sc);
  double r = NAN, i = NAN;
  if (M >= 0 && factor_count[sc] == M) {
    r = 0; i = 0;
    if (M > 0 && n >= 1) {
      const int C = (M + HS2_ROWS - 1) / HS2_ROWS;
      const double* p = part + (size_t)b * C_cap * 3;
      int Emax = INT_MIN;
      for (int c = 0; c < C; ++c) Emax = max(Emax, (int)p[3 * c + 2]);
      if (Emax != INT_MIN) {
        for (int c = 0; c < C; ++c) {
          const int e = (int)p[3 * c + 2];
          if (e == INT_MIN) continue;
          r += ldexp(p[3 * c], e - Emax);
          i += ldexp(p[3 * c + 1], e - Emax);
        }
        /* one scaling to the true exponent: inf / 0 exactly where the long double value lies outside the fp64 range */
        r = ldexp(r, Emax); i = ldexp(i, Emax);
      }
    }
  }
  out[2 * b] = r; out[2 * b + 1] = i;
}

/* HSignature3d::calculateHSignature for the obstacles [c * HS3_ROWS, (c + 1) * HS3_ROWS) of band b, one warp per
 * obstacle, the same arithmetic per obstacle as k_hsig3d. grid (B, chunks of max(M_cap, 1)) */
__global__ void __launch_bounds__(256) k_hsig3d_scene(DevBatch db, KParams kp, int use_timediffs, double* out) {
  extern __shared__ __align__(16) unsigned char hs_raw[];
  const int b = blockIdx.x, c = blockIdx.y, tid = threadIdx.x;
  const int Mc = db.M_cap > 0 ? db.M_cap : 1;
  const int l0 = c * HS3_ROWS, l1 = min(Mc, l0 + HS3_ROWS);
  int n, sc;
  const int M = hsig_scene_count(db, b, n, sc);
  if (M < 0) { /* a scene the batch cannot describe (device pointers only): no signature */
    for (int l = l0 + tid; l < l1; l += 256) out[(size_t)b * Mc + l] = NAN;
    return;
  }
  double* spx = reinterpret_cast<double*>(hs_raw);
  double* spy = spx + db.n_cap;
  double* sT = spy + db.n_cap; /* transition time at pose k */
  const double* P = db.poses + (size_t)b * db.n_cap * 4;
  for (int k = tid; k < n; k += 256) { spx[k] = P[4 * k]; spy[k] = P[4 * k + 1]; }
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
  for (int l = l0 + w; l < l1; l += 8) { /* rows past M (and the one row of M_cap = 0) are written as 0 */
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
