/*
 * teb_device.cuh — device-side arithmetic of the TEB cost terms (residuals and closed-form Jacobians).
 *
 * Every function cites the reference body it reproduces (paths relative to the reference checkout):
 *   g2o_types/penalties.h, misc.h, pose_se2.h, obstacles.h, robot_footprint_model.h, g2o_types/edge_*.h.
 * The reference linearises numerically (central differences, delta 1e-9) for all edges except
 * EdgeKinematicsDiffDrive / EdgeTimeOptimal; the closed forms here use the same branch predicates as the
 * computeError bodies and the sub-gradient policy of SURVEY.md Appendix B (0 at ||0||, sign(0) = 0).
 */
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/teb_b200.h"

#define TEB_PI 3.14159265358979323846

namespace tebgpu {

/* Parameters as seen by the kernels: the POD mirror plus values derived once per launch on the host. */
struct KParams {
  TebParams p;
  double w_obst;       /* weight_obstacle * weight_multiplier (optimal_planner.cpp:453)            */
  double sw_vel_x, sw_vel_th, sw_acc_x, sw_acc_th, sw_kin_nh, sw_kin_2, sw_sp, sw_rot; /* sqrt of chain weights */
  int32_t inflated;    /* inflation_dist > min_obstacle_dist (optimal_planner.cpp:450)              */
  int32_t carlike;     /* !(min_turning_radius == 0 || weight_kinematics_turning_radius == 0) (:355) */
  int32_t has_vel, has_acc, has_kin, has_sp, has_rot, has_time, has_obst, has_dyn, has_via;
  int32_t pow_exponent; /* obstacle_cost_exponent != 1 && min_obstacle_dist > 0                     */
  int32_t has_vor;      /* weight_velocity_obstacle_ratio > 0 (optimal_planner.cpp:362)              */
  int32_t holo_vel;     /* max_vel_y != 0: EdgeVelocityHolonomic (optimal_planner.cpp:722, :745)        */
  int32_t holo_acc;     /* max_vel_y != 0 && acc_lim_y != 0: EdgeAccelerationHolonomic* (:778, :824)     */
  double sw_vel_y, sw_acc_y;
  int32_t generic;      /* Line / Polygon footprint or Line / Pill / Polygon obstacles present: vertex-list distance path */
  int32_t _padg;
  const double* fp_geom; /* device copy of the footprint definition for that path, see FP_* below */
};

/* ------------------------------------------------------------------ g2o/stuff/misc.h (SURVEY App. A.7) */
__device__ __forceinline__ double normalize_theta(double theta) {
  if (theta >= -TEB_PI && theta < TEB_PI) return theta;
  double multiplier = floor(theta / (2 * TEB_PI));
  theta = theta - multiplier * 2 * TEB_PI;
  if (theta >= TEB_PI) theta -= 2 * TEB_PI;
  if (theta < -TEB_PI) theta += 2 * TEB_PI;
  return theta;
}
__device__ __forceinline__ double sgn(double x) { return x > 0 ? 1.0 : (x < 0 ? -1.0 : 0.0); }

/* ------------------------------------------------------------------ penalties.h:57-117 and slopes :127-189 */
__device__ __forceinline__ double pen_interval(double var, double a, double eps, double& slope) {
  if (var < -a + eps) { slope = -1; return (-var - (a - eps)); }
  if (var <= a - eps) { slope = 0; return 0.; }
  slope = 1;
  return (var - (a - eps));
}
__device__ __forceinline__ double pen_interval2(double var, double a, double b, double eps, double& slope) {
  if (var < a + eps) { slope = -1; return (-var + (a + eps)); }
  if (var <= b - eps) { slope = 0; return 0.; }
  slope = 1;
  return (var - (b - eps));
}
__device__ __forceinline__ double pen_below(double var, double a, double eps, double& slope) {
  if (var >= a + eps) { slope = 0; return 0.; }
  slope = -1;
  return (-var + (a + eps));
}

/* ------------------------------------------------------------------ segment quantities shared by EdgeVelocity /
 * EdgeAcceleration{,Start,Goal} (edge_velocity.h:97-111, edge_acceleration.h:103-145, :316-341, :408-433). */
struct SegVal { double v, w, vx, vy; }; /* vx, vy: velocity in the frame of the first pose (holonomic edges) */

__device__ __forceinline__ SegVal seg_value(const KParams& kp, double xa, double ya, double tha, double ca, double sa,
                                            double xb, double yb, double thb, double dt) {
  const double dx = xb - xa, dy = yb - ya;
  double dist = sqrt(dx * dx + dy * dy);
  const double ad = normalize_theta(thb - tha);
  if (kp.p.exact_arc_length && ad != 0) {
    const double radius = dist / (2 * sin(ad / 2));
    dist = fabs(ad * radius);
  }
  const double u = 100 * (dx * ca + dy * sa);
  SegVal s;
  s.v = dist / dt * (u / (1 + fabs(u)));  /* fast_sigmoid misc.h:95 */
  s.w = ad / dt;
  const double idt = 1.0 / dt;
  s.vx = (ca * dx + sa * dy) * idt;       /* edge_velocity.h:250-254 */
  s.vy = (-sa * dx + ca * dy) * idt;
  return s;
}

/* value + derivatives: dv[0..5] = d v / d(xa, ya, tha, xb, yb, thb); d v/d dt = -v/dt;
 * d w / d(tha, thb, dt) = (-1/dt, 1/dt, -w/dt). */
struct SegDer { double v, w, idt, dv[6]; };

__device__ __forceinline__ SegDer seg_derivs(const KParams& kp, double xa, double ya, double tha, double ca, double sa,
                                             double xb, double yb, double thb, double dt) {
  const double dx = xb - xa, dy = yb - ya;
  const double d2 = dx * dx + dy * dy;
  const double dist = sqrt(d2);
  const double ad = normalize_theta(thb - tha);
  const double idist = dist > 0 ? 1.0 / dist : 0.0;
  const double ux = dx * idist, uy = dy * idist;
  double L = dist, gfac = 1.0, dLth = 0.0;
  if (kp.p.exact_arc_length && ad != 0) {
    const double h = ad / 2, sh = sin(h);
    const double q = ad / (2 * sh);
    gfac = fabs(q);
    dLth = dist * sgn(q) * (2 * sh - ad * cos(h)) / (4 * sh * sh);
    L = fabs(ad * (dist / (2 * sh)));
  }
  const double proj = dx * ca + dy * sa;
  const double u = 100 * proj;
  const double den = 1 + fabs(u);
  const double sig = u / den;
  const double dsig100 = 100.0 / (den * den);
  const double idt = 1.0 / dt;
  SegDer s;
  s.idt = idt;
  s.v = L / dt * sig;
  s.w = ad / dt;
  const double a = gfac * sig * idt;      /* coefficient of d dist */
  const double bq = L * dsig100 * idt;    /* coefficient of d proj */
  s.dv[0] = -a * ux - bq * ca;
  s.dv[1] = -a * uy - bq * sa;
  s.dv[2] = -dLth * sig * idt + bq * (-dx * sa + dy * ca);
  s.dv[3] = a * ux + bq * ca;
  s.dv[4] = a * uy + bq * sa;
  s.dv[5] = dLth * sig * idt;
  return s;
}

/* holonomic segment velocities and their derivatives: d[0..5] wrt (xa, ya, tha, xb, yb, thb); d/d dt = -value/dt
 * (edge_velocity.h:247-256, edge_acceleration.h:502-517) */
struct HoloDer { double vx, vy, w, idt, dvx[6], dvy[6]; };
__device__ __forceinline__ HoloDer holo_derivs(double xa, double ya, double tha, double ca, double sa, double xb, double yb,
                                               double thb, double dt) {
  const double dx = xb - xa, dy = yb - ya;
  const double rdx = ca * dx + sa * dy, rdy = -sa * dx + ca * dy;
  HoloDer h;
  h.idt = 1.0 / dt;
  h.vx = rdx * h.idt; h.vy = rdy * h.idt; h.w = normalize_theta(thb - tha) * h.idt;
  h.dvx[0] = -ca * h.idt; h.dvx[1] = -sa * h.idt; h.dvx[2] = rdy * h.idt; h.dvx[3] = ca * h.idt; h.dvx[4] = sa * h.idt; h.dvx[5] = 0;
  h.dvy[0] = sa * h.idt; h.dvy[1] = -ca * h.idt; h.dvy[2] = -rdx * h.idt; h.dvy[3] = -sa * h.idt; h.dvy[4] = ca * h.idt; h.dvy[5] = 0;
  return h;
}
/* EdgeVelocityHolonomic bounds coupled through max_vel_trans (edge_velocity.h:258-269): returns the three residuals,
 * their slopes and the bound-coupling factors k0 = d bound_x / d vy, k1 = d bound_y / d vx (0 when inactive). */
__device__ __forceinline__ void holo_velocity_terms(const KParams& kp, double vx, double vy, double w, double (&e)[3],
                                                    double (&sl)[3], double& k0, double& k1) {
  const double vt2 = kp.p.max_vel_trans * kp.p.max_vel_trans;
  const double rem_y = sqrt(fmax(0.0, vt2 - vx * vx)), rem_x = sqrt(fmax(0.0, vt2 - vy * vy));
  const double mvy = fmin(rem_y, kp.p.max_vel_y), mvx = fmin(rem_x, kp.p.max_vel_x), mvxb = fmin(rem_x, kp.p.max_vel_x_backwards);
  e[0] = pen_interval2(vx, -mvxb, mvx, 0.0, sl[0]);
  e[1] = pen_interval(vy, mvy, 0.0, sl[1]);
  e[2] = pen_interval(w, kp.p.max_vel_theta, kp.p.penalty_epsilon, sl[2]);
  const double lim0 = sl[0] < 0 ? kp.p.max_vel_x_backwards : kp.p.max_vel_x;
  k0 = (sl[0] != 0 && !(lim0 < rem_x) && rem_x > 0) ? (-vy / rem_x) : 0.0;
  k1 = (sl[1] != 0 && !(kp.p.max_vel_y < rem_y) && rem_y > 0) ? (-vx / rem_y) : 0.0;
}

/* ------------------------------------------------------------------ footprint / obstacle distance
 * Obstacle::getMinimumDistance (obstacles.h:358, :502), getMinimumSpatioTemporalDistance (:382, :526),
 * BaseRobotFootprintModel::calculateDistance / estimateSpatioTemporalDistance
 * (robot_footprint_model.h:160-176 Point, :263-278 Circular, :351-372 TwoCircles). (ox, oy) is the obstacle
 * centroid already advanced to time t for dynamic edges. Returns d, fills grad = d d / d(x, y, theta). */
__device__ __forceinline__ double footprint_distance(const KParams& kp, double px, double py, double c, double s,
                                                     double ox, double oy, double orad, double grad[3]) {
  if (kp.p.footprint_type == TEB_FOOTPRINT_TWO_CIRCLES) {
    const double fo = kp.p.footprint_front_offset, ro = kp.p.footprint_rear_offset;
    const double fx = px + fo * c - ox, fy = py + fo * s - oy;
    const double rx = px - ro * c - ox, ry = py - ro * s - oy;
    const double nf = sqrt(fx * fx + fy * fy), nr = sqrt(rx * rx + ry * ry);
    const double df = nf - orad - kp.p.footprint_front_radius;
    const double dr = nr - orad - kp.p.footprint_rear_radius;
    if (df < dr) { /* std::min(dist_front, dist_rear) */
      const double inv = nf > 0 ? 1.0 / nf : 0.0;
      grad[0] = fx * inv; grad[1] = fy * inv;
      grad[2] = fo * (-s * grad[0] + c * grad[1]);
      return df;
    }
    const double inv = nr > 0 ? 1.0 / nr : 0.0;
    grad[0] = rx * inv; grad[1] = ry * inv;
    grad[2] = -ro * (-s * grad[0] + c * grad[1]);
    return dr;
  }
  const double dx = px - ox, dy = py - oy;
  const double nrm = sqrt(dx * dx + dy * dy);
  const double inv = nrm > 0 ? 1.0 / nrm : 0.0;
  grad[0] = dx * inv; grad[1] = dy * inv; grad[2] = 0;
  double d = nrm - orad;
  if (kp.p.footprint_type == TEB_FOOTPRINT_CIRCULAR) d -= kp.p.footprint_radius;
  return d;
}
/* distance only (association, trial chi2) */
__device__ __forceinline__ double footprint_distance_only(const KParams& kp, double px, double py, double c, double s,
                                                          double ox, double oy, double orad) {
  if (kp.p.footprint_type == TEB_FOOTPRINT_TWO_CIRCLES) {
    const double fo = kp.p.footprint_front_offset, ro = kp.p.footprint_rear_offset;
    const double fx = px + fo * c - ox, fy = py + fo * s - oy;
    const double rx = px - ro * c - ox, ry = py - ro * s - oy;
    const double df = sqrt(fx * fx + fy * fy) - orad - kp.p.footprint_front_radius;
    const double dr = sqrt(rx * rx + ry * ry) - orad - kp.p.footprint_rear_radius;
    return df < dr ? df : dr;
  }
  const double dx = px - ox, dy = py - oy;
  double d = sqrt(dx * dx + dy * dy) - orad;
  if (kp.p.footprint_type == TEB_FOOTPRINT_CIRCULAR) d -= kp.p.footprint_radius;
  return d;
}


/* ------------------------------------------------------------------ vertex-list shapes (distance_calculations.h)
 * Line / Polygon footprints (robot_footprint_model.h:439-560, :635-760) and Line / Pill / Polygon obstacles
 * (obstacles.h:597-1045). A shape is a vertex list: 1 vertex = point, 2 = one segment, k > 2 = closed polygon, i.e. the
 * edge enumeration of distance_point_to_polygon_2d / distance_segment_to_polygon_2d / distance_polygon_to_polygon_2d
 * (:172-262). The function returns the distance and its gradient: with the closest points c_r (robot) and c_o
 * (obstacle), n = (c_r - c_o)/|.|, d d/d(x, y) = n and d d/d theta = n . J (c_r - p); 0 when the shapes intersect.
 * Kept out of line and only referenced by the GEOM = true kernel instantiations (chosen at launch when kp.generic), so
 * that the Point / Circular fast path keeps its registers; the footprint definition is read from a small device array instead of the kernel parameters
 * (taking their address would spill them to local memory). */
enum { FP_RADIUS = 0, FP_FRONT_OFF = 1, FP_FRONT_RAD = 2, FP_REAR_OFF = 3, FP_REAR_RAD = 4, FP_LINE = 5, FP_COUNT = 9,
       FP_VERTS = 10, FP_DOUBLES = 10 + 2 * TEB_MAX_FOOTPRINT_VERTICES };
struct Dist4 { double d, gx, gy, gt; };

/* closest_point_on_line_segment_2d distance_calculations.h:60-75 */
__device__ __forceinline__ void closest_on_segment(double px, double py, double ax, double ay, double bx, double by,
                                                   double& qx, double& qy) {
  const double dx = bx - ax, dy = by - ay;
  const double sq = dx * dx + dy * dy;
  if (sq == 0) { qx = ax; qy = ay; return; }
  const double u = ((px - ax) * dx + (py - ay) * dy) / sq;
  if (u <= 0) { qx = ax; qy = ay; }
  else if (u >= 1) { qx = bx; qy = by; }
  else { qx = ax + u * dx; qy = ay + u * dy; }
}
/* check_line_segments_intersection_2d distance_calculations.h:97-127 */
__device__ __forceinline__ bool segments_intersect(double l1sx, double l1sy, double l1ex, double l1ey, double l2sx,
                                                   double l2sy, double l2ex, double l2ey) {
  const double l1x = l1ex - l1sx, l1y = l1ey - l1sy, l2x = l2ex - l2sx, l2y = l2ey - l2sy;
  const double denom = l1x * l2y - l2x * l1y;
  if (denom == 0) return false;
  const bool dp = denom > 0;
  const double ax = l1sx - l2sx, ay = l1sy - l2sy;
  const double s_numer = l1x * ay - l1y * ax;
  if ((s_numer < 0) == dp) return false;
  const double t_numer = l2x * ay - l2y * ax;
  if ((t_numer < 0) == dp) return false;
  if (((s_numer > denom) == dp) || ((t_numer > denom) == dp)) return false;
  return true;
}
/* distance_segment_to_segment_2d distance_calculations.h:139-156; (c1x, c1y) on line 1, (c2x, c2y) on line 2 */
__device__ __forceinline__ double seg_seg_dist(double l1sx, double l1sy, double l1ex, double l1ey, double l2sx, double l2sy,
                                               double l2ex, double l2ey, double& c1x, double& c1y, double& c2x, double& c2y) {
  if (segments_intersect(l1sx, l1sy, l1ex, l1ey, l2sx, l2sy, l2ex, l2ey)) { c1x = c2x = l1sx; c1y = c2y = l1sy; return 0.0; }
  double qx, qy, best, d;
  closest_on_segment(l1sx, l1sy, l2sx, l2sy, l2ex, l2ey, qx, qy);
  best = sqrt((l1sx - qx) * (l1sx - qx) + (l1sy - qy) * (l1sy - qy));
  c1x = l1sx; c1y = l1sy; c2x = qx; c2y = qy;
  closest_on_segment(l1ex, l1ey, l2sx, l2sy, l2ex, l2ey, qx, qy);
  d = sqrt((l1ex - qx) * (l1ex - qx) + (l1ey - qy) * (l1ey - qy));
  if (d < best) { best = d; c1x = l1ex; c1y = l1ey; c2x = qx; c2y = qy; }
  closest_on_segment(l2sx, l2sy, l1sx, l1sy, l1ex, l1ey, qx, qy);
  d = sqrt((l2sx - qx) * (l2sx - qx) + (l2sy - qy) * (l2sy - qy));
  if (d < best) { best = d; c2x = l2sx; c2y = l2sy; c1x = qx; c1y = qy; }
  closest_on_segment(l2ex, l2ey, l1sx, l1sy, l1ex, l1ey, qx, qy);
  d = sqrt((l2ex - qx) * (l2ex - qx) + (l2ey - qy) * (l2ey - qy));
  if (d < best) { best = d; c2x = l2ex; c2y = l2ey; c1x = qx; c1y = qy; }
  return best;
}

__device__ __noinline__ Dist4 generic_distance(int fp_type, const double* __restrict__ fp, const double* __restrict__ pool,
                                               double px, double py, double c, double s, double ox, double oy,
                                               double orad_in, int otype, int vbegin, int vcount, double offx, double offy) {
  /* obstacle shape: vertex list in the pool (+ the constant-velocity offset) or the single point (ox, oy) */
  const bool olist = otype >= TEB_OBST_LINE && vcount >= 1 && pool != nullptr;
  const int ok = olist ? vcount : 1;
  const double* ov = olist ? pool + 2 * (size_t)vbegin : nullptr;
  const bool obst_first = (otype == TEB_OBST_LINE || otype == TEB_OBST_PILL);
  const double orad = (otype == TEB_OBST_CIRCULAR || otype == TEB_OBST_PILL) ? orad_in : 0.0;
  const int oe = ok <= 2 ? 1 : ok;
  double best = 1.7976931348623157e308, bcrx = px, bcry = py, bcox = px, bcoy = py;
  const int nsub = (fp_type == TEB_FOOTPRINT_TWO_CIRCLES) ? 2 : 1;
  for (int sub = 0; sub < nsub; ++sub) {
    int rk = 1;
    double rrad = 0;
    if (fp_type == TEB_FOOTPRINT_CIRCULAR) rrad = fp[FP_RADIUS];
    else if (fp_type == TEB_FOOTPRINT_TWO_CIRCLES) rrad = sub == 0 ? fp[FP_FRONT_RAD] : fp[FP_REAR_RAD];
    else if (fp_type == TEB_FOOTPRINT_LINE) rk = 2;
    else if (fp_type == TEB_FOOTPRINT_POLYGON) rk = (int)fp[FP_COUNT];
    const int re = rk <= 2 ? 1 : rk;
    double sbest = 1.7976931348623157e308, scrx = px, scry = py, scox = px, scoy = py;
    for (int i = 0; i < re; ++i) {
      /* robot edge i in the world frame (transformToWorld robot_footprint_model.h:604-612, :757-766) */
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
          o0x = ov[2 * j] + offx; o0y = ov[2 * j + 1] + offy;
          o1x = ov[2 * j1] + offx; o1y = ov[2 * j1 + 1] + offy;
        } else { o0x = o1x = ox + offx; o0y = o1y = oy + offy; }
        double ax, ay, bx, by, d;
        if (rk == 1 && ok == 1) {
          ax = r0x; ay = r0y; bx = o0x; by = o0y;
          d = sqrt((r0x - o0x) * (r0x - o0x) + (r0y - o0y) * (r0y - o0y));
        } else if (rk == 1) {
          closest_on_segment(r0x, r0y, o0x, o0y, o1x, o1y, bx, by);
          ax = r0x; ay = r0y;
          d = sqrt((r0x - bx) * (r0x - bx) + (r0y - by) * (r0y - by));
        } else if (ok == 1) {
          closest_on_segment(o0x, o0y, r0x, r0y, r1x, r1y, ax, ay);
          bx = o0x; by = o0y;
          d = sqrt((o0x - ax) * (o0x - ax) + (o0y - ay) * (o0y - ay));
        } else if (obst_first) {
          d = seg_seg_dist(o0x, o0y, o1x, o1y, r0x, r0y, r1x, r1y, bx, by, ax, ay);
        } else {
          d = seg_seg_dist(r0x, r0y, r1x, r1y, o0x, o0y, o1x, o1y, ax, ay, bx, by);
        }
        if (d < sbest) { sbest = d; scrx = ax; scry = ay; scox = bx; scoy = by; }
      }
    }
    const double dsub = sbest - orad - rrad;
    /* <=: the rear circle (sub 1) wins an exact front / rear tie, as in footprint_distance (same distance, one gradient) */
    if (dsub <= best) { best = dsub; bcrx = scrx; bcry = scry; bcox = scox; bcoy = scoy; }
  }
  Dist4 r;
  r.d = best;
  double nx = bcrx - bcox, ny = bcry - bcoy;
  const double nn = sqrt(nx * nx + ny * ny);
  if (nn > 0) { nx /= nn; ny /= nn; } else { nx = 0; ny = 0; }
  r.gx = nx; r.gy = ny;
  r.gt = -nx * (bcry - py) + ny * (bcrx - px);
  return r;
}

/* calculateDistance / estimateSpatioTemporalDistance of the configured footprint to one obstacle row. (ox, oy) is the
 * position already advanced to time t (fast path), (offx, offy) = t * velocity the same shift for vertex lists. */
template <bool GEOM>
__device__ __forceinline__ double robot_obstacle_distance(const KParams& kp, const double* pool, double px, double py,
                                                          double c, double s, const TebObstacle& ob, double ox, double oy,
                                                          double offx, double offy, double grad[3]) {
  if (GEOM) { /* instantiations without vertex-list shapes carry no call at all: the fast path keeps its registers */
    const Dist4 r = generic_distance(kp.p.footprint_type, kp.fp_geom, pool, px, py, c, s, ob.x, ob.y, ob.radius, ob.type,
                                     ob.vertex_begin, ob.vertex_count, offx, offy);
    grad[0] = r.gx; grad[1] = r.gy; grad[2] = r.gt;
    return r.d;
  }
  return footprint_distance(kp, px, py, c, s, ox, oy, ob.radius, grad);
}
template <bool GEOM>
__device__ __forceinline__ double robot_obstacle_distance_only(const KParams& kp, const double* pool, double px, double py,
                                                               double c, double s, const TebObstacle& ob, double ox,
                                                               double oy, double offx, double offy) {
  if (GEOM)
    return generic_distance(kp.p.footprint_type, kp.fp_geom, pool, px, py, c, s, ob.x, ob.y, ob.radius, ob.type,
                            ob.vertex_begin, ob.vertex_count, offx, offy).d;
  return footprint_distance_only(kp, px, py, c, s, ox, oy, ob.radius);
}

/* EdgeObstacle / EdgeInflatedObstacle residual pair (edge_obstacle.h:85-106, :207-233): returns weighted
 * chi2, kappa = sum_k w_k slope_k^2, beta = sum_k w_k e_k slope_k so that H += kappa g g^T, b -= beta g. */
__device__ __forceinline__ double obstacle_terms(const KParams& kp, double d, double& kappa, double& beta) {
  double s0;
  double e0 = pen_below(d, kp.p.min_obstacle_dist, kp.p.penalty_epsilon, s0);
  if (kp.pow_exponent) {
    const double base = e0 / kp.p.min_obstacle_dist;
    const double ex = kp.p.obstacle_cost_exponent;
    s0 *= (e0 > 0) ? ex * pow(base, ex - 1.0) : 0.0;
    e0 = kp.p.min_obstacle_dist * pow(base, ex);
  }
  double chi = kp.w_obst * e0 * e0;
  kappa = kp.w_obst * s0 * s0;
  beta = kp.w_obst * e0 * s0;
  if (kp.inflated) {
    double s1;
    const double e1 = pen_below(d, kp.p.inflation_dist, 0.0, s1);
    chi += kp.p.weight_inflation * e1 * e1;
    kappa += kp.p.weight_inflation * s1 * s1;
    beta += kp.p.weight_inflation * e1 * s1;
  }
  return chi;
}
/* EdgeDynamicObstacle (edge_dynamic_obstacle.h:93-104); information diag(weight_dynamic_obstacle * 1,
 * weight_dynamic_obstacle_inflation) (optimal_planner.cpp:652-653, called without multiplier :343). */
__device__ __forceinline__ double dynamic_terms(const KParams& kp, double d, double& kappa, double& beta) {
  double s0, s1;
  const double e0 = pen_below(d, kp.p.min_obstacle_dist, kp.p.penalty_epsilon, s0);
  const double e1 = pen_below(d, kp.p.dynamic_obstacle_inflation_dist, 0.0, s1);
  kappa = kp.p.weight_dynamic_obstacle * s0 * s0 + kp.p.weight_dynamic_obstacle_inflation * s1 * s1;
  beta = kp.p.weight_dynamic_obstacle * e0 * s0 + kp.p.weight_dynamic_obstacle_inflation * e1 * s1;
  return kp.p.weight_dynamic_obstacle * e0 * e0 + kp.p.weight_dynamic_obstacle_inflation * e1 * e1;
}

/* EdgeVelocityObstacleRatio (edge_velocity_obstacle_ratio.h:82-122): velocity bounds scaled by the proximity ratio of
 * the first pose to an associated obstacle. Returns the ratio and d ratio / d distance. */
__device__ __forceinline__ double proximity_ratio(const KParams& kp, double d, double& dratio) {
  double ratio;
  dratio = 0;
  if (d < kp.p.obstacle_proximity_lower_bound) ratio = 0;
  else if (d > kp.p.obstacle_proximity_upper_bound) ratio = 1;
  else {
    ratio = (d - kp.p.obstacle_proximity_lower_bound) / (kp.p.obstacle_proximity_upper_bound - kp.p.obstacle_proximity_lower_bound);
    dratio = 1.0 / (kp.p.obstacle_proximity_upper_bound - kp.p.obstacle_proximity_lower_bound);
  }
  dratio *= kp.p.obstacle_proximity_ratio_max_vel;
  return ratio * kp.p.obstacle_proximity_ratio_max_vel;
}

/* ------------------------------------------------------------------ TMA (1-D bulk copy) + mbarrier wrappers */
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
/* global -> shared bulk copy; bytes multiple of 16, both addresses 16-byte aligned */
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
/* shared -> global bulk copy */
__device__ __forceinline__ void tma_store_1d(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)),
               "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_store_commit_wait() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

}  // namespace tebgpu
