/*
 * teb_frame.h — the arithmetic the node does with a transform it has already looked up: tf2's doTransform of a plan pose
 * (transformGlobalPlan, pruneGlobalPlan, the goal-reached test, estimateLocalGoalOrientation) and the Eigen isometry of
 * the custom obstacles (updateObstacleContainerWithCustomObstacles, with PolygonObstacle::finalizePolygon). One routine
 * compiled for the host and for the device (k_local_plan in teb_local_plan.cuh, k_costmap_obstacles in teb_costmap.cuh),
 * like teb_plan.h.
 *
 * tf2, tf2_geometry_msgs, tf2_eigen and Eigen are not part of the reference checkout; these routines restate ROS Noetic's
 * code (tf2 LinearMath Matrix3x3 / Quaternion / Transform, tf2/impl/utils.h, tf2_eigen's transformToEigen) and Eigen
 * 3.3's QuaternionBase::toRotationMatrix and fixed-size matrix-vector product as an x86-64 SSE2 build evaluates them.
 *
 * A transform is 7 doubles in geometry_msgs/Transform order: tx, ty, tz, qx, qy, qz, qw; the quaternion is taken as
 * given, not normalised. A 3x3 basis is stored row-major, m[3 * i + j]. Every product and sum is a round-to-nearest
 * helper of teb_plan.h, so FMA contraction cannot move a bit.
 */
#ifndef TEB_FRAME_H
#define TEB_FRAME_H

#include "teb_plan.h"

TEB_HD inline double teb_sub(double a, double b) { return teb_add(a, -b); }

/* tf2::Matrix3x3::setRotation(q): s = 2 / |q|^2, so a non-unit quaternion still gives a rotation */
TEB_HD inline void teb_tf2_basis(const double* q, double* m) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double d = teb_add(teb_add(teb_add(teb_mul(x, x), teb_mul(y, y)), teb_mul(z, z)), teb_mul(w, w));
  const double s = 2.0 / d;
  const double xs = teb_mul(x, s), ys = teb_mul(y, s), zs = teb_mul(z, s);
  const double wx = teb_mul(w, xs), wy = teb_mul(w, ys), wz = teb_mul(w, zs);
  const double xx = teb_mul(x, xs), xy = teb_mul(x, ys), xz = teb_mul(x, zs);
  const double yy = teb_mul(y, ys), yz = teb_mul(y, zs), zz = teb_mul(z, zs);
  m[0] = 1.0 - teb_add(yy, zz); m[1] = teb_sub(xy, wz);       m[2] = teb_add(xz, wy);
  m[3] = teb_add(xy, wz);       m[4] = 1.0 - teb_add(xx, zz); m[5] = teb_sub(yz, wx);
  m[6] = teb_sub(xz, wy);       m[7] = teb_add(yz, wx);       m[8] = 1.0 - teb_add(xx, yy);
}

/* Eigen::QuaternionBase::toRotationMatrix() of Quaterniond(w, x, y, z): no division by |q|^2, unlike setRotation */
TEB_HD inline void teb_eigen_basis(const double* q, double* m) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double tx = teb_mul(2.0, x), ty = teb_mul(2.0, y), tz = teb_mul(2.0, z);
  const double twx = teb_mul(tx, w), twy = teb_mul(ty, w), twz = teb_mul(tz, w);
  const double txx = teb_mul(tx, x), txy = teb_mul(ty, x), txz = teb_mul(tz, x);
  const double tyy = teb_mul(ty, y), tyz = teb_mul(tz, y), tzz = teb_mul(tz, z);
  m[0] = 1.0 - teb_add(tyy, tzz); m[1] = teb_sub(txy, twz);       m[2] = teb_add(txz, twy);
  m[3] = teb_add(txy, twz);       m[4] = 1.0 - teb_add(txx, tzz); m[5] = teb_sub(tyz, twx);
  m[6] = teb_sub(txz, twy);       m[7] = teb_add(tyz, twx);       m[8] = 1.0 - teb_add(txx, tyy);
}

/* x and y of basis * (vx, vy, vz) + origin: tf2's Transform::operator()(v) (v.dot3 of the basis rows, then + origin) and
 * Eigen's Affine3d * Vector3d (translation + the product, whose rows 0 and 1 the SSE2 packet path sums as
 * (m0 v0 + m1 v1) + m2 v2) both round as ((m[3i] vx + m[3i+1] vy) + m[3i+2] vz) + o[i] */
TEB_HD inline void teb_frame_point(const double* m, const double* o, double vx, double vy, double vz, double* out) {
  for (int i = 0; i < 2; ++i) {
    const double* r = m + 3 * i;
    out[i] = teb_add(teb_add(teb_add(teb_mul(r[0], vx), teb_mul(r[1], vy)), teb_mul(r[2], vz)), o[i]);
  }
}

/* tf2 Matrix3x3 operator*(a, b): c[i][j] = (b[0][j] a[i][0] + b[1][j] a[i][1]) + b[2][j] a[i][2] */
TEB_HD inline void teb_tf2_basis_product(const double* a, const double* b, double* c) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      c[3 * i + j] = teb_add(teb_add(teb_mul(b[j], a[3 * i]), teb_mul(b[3 + j], a[3 * i + 1])), teb_mul(b[6 + j], a[3 * i + 2]));
}

/* tf2::Matrix3x3::getRotation: the trace branch, or the branch of the largest diagonal element i (ties as tf2 decides
 * them); q = (x, y, z, w) */
TEB_HD inline void teb_tf2_get_rotation(const double* m, double* q) {
  const double trace = teb_add(teb_add(m[0], m[4]), m[8]);
  if (trace > 0.0) {
    double s = sqrt(teb_add(trace, 1.0));
    q[3] = teb_mul(s, 0.5);
    s = 0.5 / s;
    q[0] = teb_mul(teb_sub(m[7], m[5]), s);
    q[1] = teb_mul(teb_sub(m[2], m[6]), s);
    q[2] = teb_mul(teb_sub(m[3], m[1]), s);
  } else {
    const int i = m[0] < m[4] ? (m[4] < m[8] ? 2 : 1) : (m[0] < m[8] ? 2 : 0);
    const int j = (i + 1) % 3, k = (i + 2) % 3;
    double s = sqrt(teb_add(teb_sub(teb_sub(m[4 * i], m[4 * j]), m[4 * k]), 1.0));
    q[i] = teb_mul(s, 0.5);
    s = 0.5 / s;
    q[3] = teb_mul(teb_sub(m[3 * k + j], m[3 * j + k]), s);
    q[j] = teb_mul(teb_add(m[3 * j + i], m[3 * i + j]), s);
    q[k] = teb_mul(teb_add(m[3 * k + i], m[3 * i + k]), s);
  }
}

/* tf2::getYaw (tf2/impl/utils.h): the two gimbal branches at |sarg| >= 0.99999, else atan2 of the rotated x axis */
TEB_HD inline double teb_tf2_get_yaw(const double* q) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double sqx = teb_mul(x, x), sqy = teb_mul(y, y), sqz = teb_mul(z, z), sqw = teb_mul(w, w);
  const double sarg = teb_mul(-2.0, teb_sub(teb_mul(x, z), teb_mul(w, y))) / teb_add(teb_add(teb_add(sqx, sqy), sqz), sqw);
  if (sarg <= -0.99999) return teb_mul(-2.0, atan2(y, x));
  if (sarg >= 0.99999) return teb_mul(2.0, atan2(y, x));
  return atan2(teb_mul(2.0, teb_add(teb_mul(x, y), teb_mul(w, z))), teb_sub(teb_sub(teb_add(sqw, sqx), sqy), sqz));
}

/* tf2 Quaternion operator*(a, b), the raw product (no normalisation) */
TEB_HD inline void teb_tf2_quat_mul(const double* a, const double* b, double* c) {
  const double ax = a[0], ay = a[1], az = a[2], aw = a[3], bx = b[0], by = b[1], bz = b[2], bw = b[3];
  c[0] = teb_sub(teb_add(teb_add(teb_mul(aw, bx), teb_mul(ax, bw)), teb_mul(ay, bz)), teb_mul(az, by));
  c[1] = teb_sub(teb_add(teb_add(teb_mul(aw, by), teb_mul(ay, bw)), teb_mul(az, bx)), teb_mul(ax, bz));
  c[2] = teb_sub(teb_add(teb_add(teb_mul(aw, bz), teb_mul(az, bw)), teb_mul(ax, by)), teb_mul(ay, bx));
  c[3] = teb_sub(teb_sub(teb_sub(teb_mul(aw, bw), teb_mul(ax, bx)), teb_mul(ay, by)), teb_mul(az, bz));
}

/* the quaternion of a plan row's yaw, as teb_plan_yaw models it: (0, 0, sin(yaw / 2), cos(yaw / 2)) */
TEB_HD inline void teb_yaw_quat(double yaw, double* q) {
  q[0] = 0.0; q[1] = 0.0; q[2] = sin(yaw / 2); q[3] = cos(yaw / 2);
}

/* tf2::getYaw of the orientation tf2::doTransform gives a plan row of heading yaw under a transform of basis tb:
 * getRotation(tb * setRotation(row quaternion)) */
TEB_HD inline double teb_frame_row_yaw(const double* tb, double yaw) {
  double q[4], r[9], c[9];
  teb_yaw_quat(yaw, q);
  teb_tf2_basis(q, r);
  teb_tf2_basis_product(tb, r, c);
  teb_tf2_get_rotation(c, q);
  return teb_tf2_get_yaw(q);
}

/* estimateLocalGoalOrientation's near-goal heading: getYaw(rotation * global_orientation), the transform's quaternion
 * t[3..6] times the last row's */
TEB_HD inline double teb_frame_goal_yaw(const double* t, double yaw) {
  double g[4], c[4];
  teb_yaw_quat(yaw, g);
  teb_tf2_quat_mul(t + 3, g, c);
  return teb_tf2_get_yaw(c);
}

/* Eigen's v.isApprox(w) of two 2-vectors at dummy_precision 1e-12 (fixPolygonClosure) */
TEB_HD inline bool teb_eigen_is_approx(double ax, double ay, double bx, double by) {
  const double dx = teb_sub(ax, bx), dy = teb_sub(ay, by);
  const double na = teb_add(teb_mul(ax, ax), teb_mul(ay, ay)), nb = teb_add(teb_mul(bx, bx), teb_mul(by, by));
  return teb_add(teb_mul(dx, dx), teb_mul(dy, dy)) <= teb_mul(teb_mul(1e-12, 1e-12), nb < na ? nb : na);
}

/* PolygonObstacle::calcCentroid (obstacles.cpp:57-126) of the n vertices v[2 * i], v[2 * i + 1], after
 * fixPolygonClosure (:48-55): c[0], c[1] */
TEB_HD inline void teb_polygon_centroid(const double* v, int n, double* c) {
  if (n <= 0) { c[0] = c[1] = NAN; return; }
  if (n == 1) { c[0] = v[0]; c[1] = v[1]; return; }
  if (n == 2) { c[0] = teb_mul(0.5, teb_add(v[0], v[2])); c[1] = teb_mul(0.5, teb_add(v[1], v[3])); return; }
  auto cross = [&](int i, int j) { return teb_sub(teb_mul(v[2 * i], v[2 * j + 1]), teb_mul(v[2 * j], v[2 * i + 1])); };
  double A = 0.0;
  for (int i = 0; i < n - 1; ++i) A = teb_add(A, cross(i, i + 1));
  A = teb_add(A, cross(n - 1, 0));
  A = teb_mul(A, 0.5);
  if (A != 0) {
    double cx = 0.0, cy = 0.0;
    for (int i = 0; i < n; ++i) {
      const int j = i + 1 < n ? i + 1 : 0;
      const double aux = cross(i, j);
      cx = teb_add(cx, teb_mul(teb_add(v[2 * i], v[2 * j]), aux));
      cy = teb_add(cy, teb_mul(teb_add(v[2 * i + 1], v[2 * j + 1]), aux));
    }
    const double den = teb_mul(6.0, A);
    c[0] = cx / den; c[1] = cy / den;
    return;
  }
  int ic = 0, jc = 0;
  double best = 0.0;
  for (int i = 0; i < n; ++i)
    for (int j = i + 1; j < n; ++j) {
      const double dx = teb_sub(v[2 * j], v[2 * i]), dy = teb_sub(v[2 * j + 1], v[2 * i + 1]);
      const double d = sqrt(teb_add(teb_mul(dx, dx), teb_mul(dy, dy)));
      if (d > best) { best = d; ic = i; jc = j; }
    }
  c[0] = teb_mul(0.5, teb_add(v[2 * ic], v[2 * jc]));
  c[1] = teb_mul(0.5, teb_add(v[2 * ic + 1], v[2 * jc + 1]));
}

#endif
