/*
 * teb_oracle.c — CPU restatement of the reference's TEB optimisation path ("g2o mode").
 * TEST INFRASTRUCTURE ONLY — see teb_oracle.h. Parity is PINNED by oracle/_ref (the reference's own sources compiled
 * against stand-in headers): bit-identical on every compared quantity, tests/test_reference_pin.py. Only the g2o
 * optimizer internals (third-party, absent from /root/reference) remain restated from published behaviour.
 *
 * What is restated and from where (all paths relative to /root/reference):
 *   penalties                         include/teb_local_planner/g2o_types/penalties.h:57-117
 *   fast_sigmoid / cross2d            include/teb_local_planner/misc.h:95, :120
 *   PoseSE2::plus / average           include/teb_local_planner/pose_se2.h:238-243, :266-269
 *   obstacle distances                include/teb_local_planner/obstacles.h:358-361, 382-385, 502-505, 526-529
 *   footprint distances               include/teb_local_planner/robot_footprint_model.h:160-176, 263-278, 351-372
 *   edge computeError bodies          include/teb_local_planner/g2o_types/edge_*.h (cited per function)
 *   buildGraph / AddEdges*            src/optimal_planner.cpp:323-366, 444-548, 646-718, 720-997
 *   optimizeTEB / optimizeGraph       src/optimal_planner.cpp:182-231, 368-402
 *   computeCurrentCost                src/optimal_planner.cpp:1041-1094
 *   autoResize / initTrajectoryToGoal src/timed_elastic_band.cpp:227-286, 325-387
 *   g2o LM / numeric Jacobians / quadratic form / helpers: SURVEY.md Appendix A (upstream g2o,
 *   call sites src/optimal_planner.cpp:161-179, 385-387).
 *
 * Structure mirrors g2o on purpose (heap-allocated polymorphic edges rebuilt every outer iteration,
 * generic numeric linearisation through computeError callbacks, sparse(banded) Cholesky per LM trial)
 * so that timing it is a fair "reference CPU path" baseline.
 */
#ifndef _GNU_SOURCE
#define _GNU_SOURCE /* pthread_setaffinity_np, sched_getaffinity (thread pinning of the batch driver) */
#endif
#include "teb_oracle.h"

#include <float.h>
#include <math.h>
#include <pthread.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

#define HBW 10 /* half bandwidth of H in g2o vertex-id order (acceleration edge spans 11 scalars) */

/* ------------------------------------------------------------------ g2o/stuff/misc.h helpers (App. A.7) */
double teb_oracle_normalize_theta(double theta) {
  if (theta >= -M_PI && theta < M_PI) return theta;
  double multiplier = floor(theta / (2 * M_PI));
  theta = theta - multiplier * 2 * M_PI;
  if (theta >= M_PI) theta -= 2 * M_PI;
  if (theta < -M_PI) theta += 2 * M_PI;
  return theta;
}
double teb_oracle_average_angle(double a, double b) {
  double x = cos(a) + cos(b), y = sin(a) + sin(b);
  if (x == 0 && y == 0) return 0;
  return atan2(y, x);
}
static inline double nt(double t) { return teb_oracle_normalize_theta(t); }
static inline double sgn(double x) { return x > 0 ? 1.0 : (x < 0 ? -1.0 : 0.0); }

/* ------------------------------------------------------------------ penalties.h:57-117 */
double teb_oracle_penalty_interval(double var, double a, double eps) {
  if (var < -a + eps) return (-var - (a - eps));
  if (var <= a - eps) return 0.;
  return (var - (a - eps));
}
double teb_oracle_penalty_interval2(double var, double a, double b, double eps) {
  if (var < a + eps) return (-var + (a + eps));
  if (var <= b - eps) return 0.;
  return (var - (b - eps));
}
double teb_oracle_penalty_below(double var, double a, double eps) {
  if (var >= a + eps) return 0.;
  return (-var + (a + eps));
}
/* slopes (penalties.h:127-189) */
static inline double d_interval(double var, double a, double eps) {
  if (var < -a + eps) return -1;
  if (var <= a - eps) return 0;
  return 1;
}
static inline double d_interval2(double var, double a, double b, double eps) {
  if (var < a + eps) return -1;
  if (var <= b - eps) return 0;
  return 1;
}
static inline double d_below(double var, double a, double eps) { return (var >= a + eps) ? 0.0 : -1.0; }

static inline double fast_sigmoid(double x) { return x / (1 + fabs(x)); } /* misc.h:95 */

/* ------------------------------------------------------------------ band / graph data structures */
enum EdgeType {
  E_OBST = 0, E_INFL, E_DYN, E_VIA, E_VEL, E_ACC, E_ACC_START, E_ACC_GOAL, E_TIMEOPT, E_SHORTEST,
  E_KIN_DD, E_KIN_CL, E_ROTDIR, E_VEL_OBST_RATIO, E_VEL_HOLO, E_ACC_HOLO, E_ACC_HOLO_START, E_ACC_HOLO_GOAL, E_NTYPES
};

typedef struct Graph Graph;

typedef struct Edge {
  int type;
  int nv;          /* number of vertices */
  int vkind[5];    /* 0 pose, 1 timediff */
  int vidx[5];     /* pose / timediff index in the band */
  int dim;         /* error dimension (<= 3) */
  double info[3];  /* diagonal information matrix */
  double err[3];   /* cached _error */
  double t;        /* EdgeDynamicObstacle::t_ */
  double meas;     /* EdgePreferRotDir::_measurement */
  const TebObstacle* ob;
  const double* via;
  const double* twist; /* vel_start / vel_goal */
  void (*compute_error)(struct Edge*, Graph*);
  double J[5][9];  /* per vertex: row-major dim x vdim */
} Edge;

struct Graph {
  const TebParams* cfg;
  double* rec;  /* [n][4] */
  int n;
  const TebObstacle* obst;
  int M;
  const double* pverts; /* vertex pool of the scene's Line / Pill / Polygon obstacles: [PV][2] */
  const double* via;
  int V;
  double vel_start[4], vel_goal[4];
  int rotdir;
  Edge** edges;
  int n_edges, cap_edges;
  int N;          /* number of scalar unknowns */
  double* Hb;     /* banded lower [N][HBW+1]: Hb[r][k] = H[r][r-k] */
  double* b;      /* [N] */
  double* x;      /* [N] solution */
  double* work;   /* factor storage [N][HBW+1] */
  double* backup; /* [n][4] state backup (push/pop) */
  double* Hd;     /* dense workspace (optional) */
  int* opv;       /* obstacles_per_vertex_: [n][M] indices (optimal_planner.h:690) */
  int* opv_cnt;   /* [n] */
};

static inline int pose_fixed(const Graph* g, int i) { return i == 0 || i == g->n - 1; }
/* hessian index of first scalar of a vertex in g2o id order (pose_i id=2i, dt_i id=2i+1; fixed excluded):
 * dt_0, pose_1, dt_1, pose_2, ..., pose_{n-2}, dt_{n-2}  (optimal_planner.cpp:426-437, App. A.1) */
static inline int hidx(const Graph* g, int kind, int i) {
  if (kind == 1) return 4 * i;
  if (pose_fixed(g, i)) return -1;
  return 4 * i - 3;
}
static inline int vdim(int kind) { return kind == 0 ? 3 : 1; }

static inline double* P(Graph* g, int i) { return g->rec + 4 * i; }
static inline double DT(Graph* g, int i) { return g->rec[4 * i + 3]; }

/* ------------------------------------------------------------------ distances */
/* Obstacle::getMinimumDistance (Point obstacles.h:358, Circular :502) */
static inline double obst_dist(const TebObstacle* o, double px, double py) {
  double dx = px - o->x, dy = py - o->y;
  return sqrt(dx * dx + dy * dy) - o->radius;
}
/* getMinimumSpatioTemporalDistance (Point obstacles.h:382, Circular :526) */
static inline double obst_dist_t(const TebObstacle* o, double px, double py, double t) {
  double dx = o->x + t * o->vx - px, dy = o->y + t * o->vy - py;
  return sqrt(dx * dx + dy * dy) - o->radius;
}

/* ------------------------------------------------------------------ generic shapes (distance_calculations.h)
 * Line / Polygon footprints (robot_footprint_model.h:439-560, :635-760) and Line / Pill / Polygon obstacles
 * (obstacles.h:597-1045). A shape is a vertex list: 1 vertex = point, 2 = one segment, k > 2 = closed polygon
 * (k edges), exactly the edge enumeration of distance_point_to_polygon_2d / distance_segment_to_polygon_2d /
 * distance_polygon_to_polygon_2d (:172-262). Besides the distance the functions return the pair of closest points,
 * from which the closed-form gradient follows: d d / d(x, y) = n, d d / d theta = n . J (c_robot - p), n the unit
 * vector from the obstacle's to the robot's closest point (0 when the shapes intersect). */
#define ORACLE_SMALL_SHAPE 64   /* obstacle vertex lists up to this length are copied to the stack, longer ones to the heap */

/* closest_point_on_line_segment_2d distance_calculations.h:60-75 */
static void closest_on_segment(const double* pt, const double* a, const double* b, double* out) {
  double dx = b[0] - a[0], dy = b[1] - a[1];
  double sq = dx * dx + dy * dy;
  if (sq == 0) { out[0] = a[0]; out[1] = a[1]; return; }
  double u = ((pt[0] - a[0]) * dx + (pt[1] - a[1]) * dy) / sq;
  if (u <= 0) { out[0] = a[0]; out[1] = a[1]; }
  else if (u >= 1) { out[0] = b[0]; out[1] = b[1]; }
  else { out[0] = a[0] + u * dx; out[1] = a[1] + u * dy; }
}
static double pt_dist(const double* a, const double* b) {
  double dx = a[0] - b[0], dy = a[1] - b[1];
  return sqrt(dx * dx + dy * dy);
}
/* check_line_segments_intersection_2d distance_calculations.h:97-127 */
static int segments_intersect(const double* l1s, const double* l1e, const double* l2s, const double* l2e) {
  double l1x = l1e[0] - l1s[0], l1y = l1e[1] - l1s[1];
  double l2x = l2e[0] - l2s[0], l2y = l2e[1] - l2s[1];
  double denom = l1x * l2y - l2x * l1y;
  if (denom == 0) return 0;
  int denom_pos = denom > 0;
  double ax = l1s[0] - l2s[0], ay = l1s[1] - l2s[1];
  double s_numer = l1x * ay - l1y * ax;
  if ((s_numer < 0) == denom_pos) return 0;
  double t_numer = l2x * ay - l2y * ax;
  if ((t_numer < 0) == denom_pos) return 0;
  if (((s_numer > denom) == denom_pos) || ((t_numer > denom) == denom_pos)) return 0;
  return 1;
}
/* distance_segment_to_segment_2d distance_calculations.h:139-156; c1 on line1, c2 on line2 */
static double seg_seg_dist(const double* l1s, const double* l1e, const double* l2s, const double* l2e, double* c1, double* c2) {
  if (segments_intersect(l1s, l1e, l2s, l2e)) { c1[0] = c2[0] = l1s[0]; c1[1] = c2[1] = l1s[1]; return 0; }
  double q[2], best, d;
  closest_on_segment(l1s, l2s, l2e, q); best = pt_dist(l1s, q);
  c1[0] = l1s[0]; c1[1] = l1s[1]; c2[0] = q[0]; c2[1] = q[1];
  closest_on_segment(l1e, l2s, l2e, q); d = pt_dist(l1e, q);
  if (d < best) { best = d; c1[0] = l1e[0]; c1[1] = l1e[1]; c2[0] = q[0]; c2[1] = q[1]; }
  closest_on_segment(l2s, l1s, l1e, q); d = pt_dist(l2s, q);
  if (d < best) { best = d; c2[0] = l2s[0]; c2[1] = l2s[1]; c1[0] = q[0]; c1[1] = q[1]; }
  closest_on_segment(l2e, l1s, l1e, q); d = pt_dist(l2e, q);
  if (d < best) { best = d; c2[0] = l2e[0]; c2[1] = l2e[1]; c1[0] = q[0]; c1[1] = q[1]; }
  return best;
}
static int shape_edges(int k) { return k <= 1 ? 1 : (k == 2 ? 1 : k); }
/* minimum distance between the robot shape rv[rk] and the obstacle shape ov[ok]; obst_first: the obstacle segment is
 * line1 of distance_segment_to_segment_2d (LineObstacle / PillObstacle, obstacles.h:659, :806), else the robot's */
static double shape_distance(const double* rv, int rk, const double* ov, int ok, int obst_first, double* cr, double* co) {
  double best = HUGE_VAL;
  cr[0] = rv[0]; cr[1] = rv[1]; co[0] = ov[0]; co[1] = ov[1];
  int re = shape_edges(rk), oe = shape_edges(ok);
  for (int i = 0; i < re; ++i) {
    const double* r0 = rv + 2 * i;
    const double* r1 = rv + 2 * ((i + 1) % rk);
    for (int j = 0; j < oe; ++j) {
      const double* o0 = ov + 2 * j;
      const double* o1 = ov + 2 * ((j + 1) % ok);
      double a[2], b[2], d;
      if (rk == 1 && ok == 1) { a[0] = r0[0]; a[1] = r0[1]; b[0] = o0[0]; b[1] = o0[1]; d = pt_dist(r0, o0); }
      else if (rk == 1) { closest_on_segment(r0, o0, o1, b); a[0] = r0[0]; a[1] = r0[1]; d = pt_dist(r0, b); }
      else if (ok == 1) { closest_on_segment(o0, r0, r1, a); b[0] = o0[0]; b[1] = o0[1]; d = pt_dist(o0, a); }
      else if (obst_first) d = seg_seg_dist(o0, o1, r0, r1, b, a);
      else d = seg_seg_dist(r0, r1, o0, o1, a, b);
      if (d < best) { best = d; cr[0] = a[0]; cr[1] = a[1]; co[0] = b[0]; co[1] = b[1]; }
    }
  }
  return best;
}
static int generic_pair(const TebParams* c, const TebObstacle* o) {
  return c->footprint_type >= TEB_FOOTPRINT_LINE || o->type >= TEB_OBST_LINE;
}
/* calculateDistance / estimateSpatioTemporalDistance for every footprint x obstacle combination; grad may be NULL */
static double generic_distance(const TebParams* c, const double* pose, const TebObstacle* o, const double* pool, double t,
                               double* grad) {
  double ov_small[2 * ORACLE_SMALL_SHAPE], *ov = ov_small;
  int ok;
  double offx = t * o->vx, offy = t * o->vy;
  if (o->type >= TEB_OBST_LINE && o->vertex_count >= 1 && pool) {
    ok = o->vertex_count;
    if (ok > ORACLE_SMALL_SHAPE) ov = (double*)malloc(sizeof(double) * 2 * (size_t)ok);
    for (int k = 0; k < ok; ++k) {
      ov[2 * k] = pool[2 * (o->vertex_begin + k)] + offx;
      ov[2 * k + 1] = pool[2 * (o->vertex_begin + k) + 1] + offy;
    }
  } else { ok = 1; ov[0] = o->x + offx; ov[1] = o->y + offy; }
  const int obst_first = (o->type == TEB_OBST_LINE || o->type == TEB_OBST_PILL);
  const double orad = (o->type == TEB_OBST_CIRCULAR || o->type == TEB_OBST_PILL) ? o->radius : 0.0;
  double cs = cos(pose[2]), sn = sin(pose[2]);
  double rv[2 * TEB_MAX_FOOTPRINT_VERTICES];
  double best = HUGE_VAL, bcr[2] = {pose[0], pose[1]}, bco[2] = {pose[0], pose[1]};
  int nsub = (c->footprint_type == TEB_FOOTPRINT_TWO_CIRCLES) ? 2 : 1;
  for (int sub = 0; sub < nsub; ++sub) {
    int rk = 1;
    double rrad = 0;
    switch (c->footprint_type) {
      case TEB_FOOTPRINT_CIRCULAR: rv[0] = pose[0]; rv[1] = pose[1]; rrad = c->footprint_radius; break;
      case TEB_FOOTPRINT_TWO_CIRCLES: {
        double off = sub == 0 ? c->footprint_front_offset : -c->footprint_rear_offset;
        rv[0] = pose[0] + off * cs; rv[1] = pose[1] + off * sn;
        rrad = sub == 0 ? c->footprint_front_radius : c->footprint_rear_radius;
        break;
      }
      case TEB_FOOTPRINT_LINE: /* LineRobotFootprint::transformToWorld robot_footprint_model.h:604-612 */
        rk = 2;
        for (int k = 0; k < 2; ++k) {
          double lx = c->footprint_line[2 * k], ly = c->footprint_line[2 * k + 1];
          rv[2 * k] = pose[0] + cs * lx - sn * ly;
          rv[2 * k + 1] = pose[1] + sn * lx + cs * ly;
        }
        break;
      case TEB_FOOTPRINT_POLYGON: /* PolygonRobotFootprint::transformToWorld :757-766 */
        rk = c->footprint_vertex_count;
        for (int k = 0; k < rk; ++k) {
          double lx = c->footprint_vertices[2 * k], ly = c->footprint_vertices[2 * k + 1];
          rv[2 * k] = pose[0] + cs * lx - sn * ly;
          rv[2 * k + 1] = pose[1] + sn * lx + cs * ly;
        }
        break;
      default: rv[0] = pose[0]; rv[1] = pose[1]; break;
    }
    double cr[2], co[2];
    double d = shape_distance(rv, rk, ov, ok, obst_first, cr, co) - orad - rrad;
    /* <=: the rear circle (sub 1) wins an exact front / rear tie, as in footprint_grad (same distance, one gradient) */
    if (d <= best) { best = d; bcr[0] = cr[0]; bcr[1] = cr[1]; bco[0] = co[0]; bco[1] = co[1]; }
  }
  if (ov != ov_small) free(ov);
  if (grad) {
    double nx = bcr[0] - bco[0], ny = bcr[1] - bco[1];
    double nn = sqrt(nx * nx + ny * ny);
    if (nn > 0) { nx /= nn; ny /= nn; } else { nx = ny = 0; }
    grad[0] = nx; grad[1] = ny;
    grad[2] = -nx * (bcr[1] - pose[1]) + ny * (bcr[0] - pose[0]);
  }
  return best;
}
/* BaseRobotFootprintModel::calculateDistance (robot_footprint_model.h:160, :263, :351, :496, :690) */
static double footprint_dist(const TebParams* c, const double* pose, const TebObstacle* o, const double* pool) {
  if (generic_pair(c, o)) return generic_distance(c, pose, o, pool, 0.0, NULL);
  switch (c->footprint_type) {
    case TEB_FOOTPRINT_CIRCULAR: return obst_dist(o, pose[0], pose[1]) - c->footprint_radius;
    case TEB_FOOTPRINT_TWO_CIRCLES: {
      double cx = cos(pose[2]), sy = sin(pose[2]);
      double df = obst_dist(o, pose[0] + c->footprint_front_offset * cx, pose[1] + c->footprint_front_offset * sy) -
                  c->footprint_front_radius;
      double dr = obst_dist(o, pose[0] - c->footprint_rear_offset * cx, pose[1] - c->footprint_rear_offset * sy) -
                  c->footprint_rear_radius;
      return df < dr ? df : dr; /* std::min(front, rear) */
    }
    default: return obst_dist(o, pose[0], pose[1]);
  }
}
/* estimateSpatioTemporalDistance (robot_footprint_model.h:172, :275, :366) */
static double footprint_dist_t(const TebParams* c, const double* pose, const TebObstacle* o, const double* pool, double t) {
  if (generic_pair(c, o)) return generic_distance(c, pose, o, pool, t, NULL);
  switch (c->footprint_type) {
    case TEB_FOOTPRINT_CIRCULAR: return obst_dist_t(o, pose[0], pose[1], t) - c->footprint_radius;
    case TEB_FOOTPRINT_TWO_CIRCLES: {
      double cx = cos(pose[2]), sy = sin(pose[2]);
      double df = obst_dist_t(o, pose[0] + c->footprint_front_offset * cx, pose[1] + c->footprint_front_offset * sy, t) -
                  c->footprint_front_radius;
      double dr = obst_dist_t(o, pose[0] - c->footprint_rear_offset * cx, pose[1] - c->footprint_rear_offset * sy, t) -
                  c->footprint_rear_radius;
      return df < dr ? df : dr;
    }
    default: return obst_dist_t(o, pose[0], pose[1], t);
  }
}

/* ------------------------------------------------------------------ edge cost functions (computeError) */
/* EdgeObstacle::computeError g2o_types/edge_obstacle.h:85-106 */
static void ce_obstacle(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double dist = footprint_dist(c, P(g, e->vidx[0]), e->ob, g->pverts);
  e->err[0] = teb_oracle_penalty_below(dist, c->min_obstacle_dist, c->penalty_epsilon);
  if (c->obstacle_cost_exponent != 1.0 && c->min_obstacle_dist > 0.0)
    e->err[0] = c->min_obstacle_dist * pow(e->err[0] / c->min_obstacle_dist, c->obstacle_cost_exponent);
}
/* EdgeInflatedObstacle::computeError edge_obstacle.h:207-233 */
static void ce_inflated(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double dist = footprint_dist(c, P(g, e->vidx[0]), e->ob, g->pverts);
  e->err[0] = teb_oracle_penalty_below(dist, c->min_obstacle_dist, c->penalty_epsilon);
  if (c->obstacle_cost_exponent != 1.0 && c->min_obstacle_dist > 0.0)
    e->err[0] = c->min_obstacle_dist * pow(e->err[0] / c->min_obstacle_dist, c->obstacle_cost_exponent);
  e->err[1] = teb_oracle_penalty_below(dist, c->inflation_dist, 0.0);
}
/* EdgeDynamicObstacle::computeError edge_dynamic_obstacle.h:93-104 */
static void ce_dynamic(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double dist = footprint_dist_t(c, P(g, e->vidx[0]), e->ob, g->pverts, e->t);
  e->err[0] = teb_oracle_penalty_below(dist, c->min_obstacle_dist, c->penalty_epsilon);
  e->err[1] = teb_oracle_penalty_below(dist, c->dynamic_obstacle_inflation_dist, 0.0);
}
/* EdgeViaPoint::computeError edge_via_point.h:81-89 */
static void ce_via(Edge* e, Graph* g) {
  const double* p = P(g, e->vidx[0]);
  double dx = p[0] - e->via[0], dy = p[1] - e->via[1];
  e->err[0] = sqrt(dx * dx + dy * dy);
}
/* shared by velocity / acceleration edges: dist (optionally arc length), direction sigmoid */
static inline void seg_vel(const TebParams* c, const double* p1, const double* p2, double dt, double* vel, double* omega) {
  double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
  double dist = sqrt(dx * dx + dy * dy);
  double angle_diff = nt(p2[2] - p1[2]);
  if (c->exact_arc_length && angle_diff != 0) {
    double radius = dist / (2 * sin(angle_diff / 2));
    dist = fabs(angle_diff * radius);
  }
  double v = dist / dt;
  v *= fast_sigmoid(100 * (dx * cos(p1[2]) + dy * sin(p1[2])));
  *vel = v;
  *omega = angle_diff / dt;
}
/* EdgeVelocity::computeError edge_velocity.h:92-117 */
static void ce_velocity(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double vel, omega;
  seg_vel(c, P(g, e->vidx[0]), P(g, e->vidx[1]), DT(g, e->vidx[2]), &vel, &omega);
  e->err[0] = teb_oracle_penalty_interval2(vel, -c->max_vel_x_backwards, c->max_vel_x, c->penalty_epsilon);
  e->err[1] = teb_oracle_penalty_interval(omega, c->max_vel_theta, c->penalty_epsilon);
}
/* EdgeAcceleration::computeError edge_acceleration.h:93-150 */
static void ce_acceleration(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double dt1 = DT(g, e->vidx[3]), dt2 = DT(g, e->vidx[4]);
  double vel1, vel2, omega1, omega2;
  seg_vel(c, P(g, e->vidx[0]), P(g, e->vidx[1]), dt1, &vel1, &omega1);
  seg_vel(c, P(g, e->vidx[1]), P(g, e->vidx[2]), dt2, &vel2, &omega2);
  double acc_lin = (vel2 - vel1) * 2 / (dt1 + dt2);
  e->err[0] = teb_oracle_penalty_interval(acc_lin, c->acc_lim_x, c->penalty_epsilon);
  double acc_rot = (omega2 - omega1) * 2 / (dt1 + dt2);
  e->err[1] = teb_oracle_penalty_interval(acc_rot, c->acc_lim_theta, c->penalty_epsilon);
}
/* EdgeAccelerationStart::computeError edge_acceleration.h:311-345 */
static void ce_acc_start(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double dt = DT(g, e->vidx[2]);
  double vel2, omega2;
  seg_vel(c, P(g, e->vidx[0]), P(g, e->vidx[1]), dt, &vel2, &omega2);
  double vel1 = e->twist[0];
  double acc_lin = (vel2 - vel1) / dt;
  e->err[0] = teb_oracle_penalty_interval(acc_lin, c->acc_lim_x, c->penalty_epsilon);
  double omega1 = e->twist[2];
  double acc_rot = (omega2 - omega1) / dt;
  e->err[1] = teb_oracle_penalty_interval(acc_rot, c->acc_lim_theta, c->penalty_epsilon);
}
/* EdgeAccelerationGoal::computeError edge_acceleration.h:402-437 */
static void ce_acc_goal(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double dt = DT(g, e->vidx[2]);
  double vel1, omega1;
  seg_vel(c, P(g, e->vidx[0]), P(g, e->vidx[1]), dt, &vel1, &omega1);
  double vel2 = e->twist[0];
  double acc_lin = (vel2 - vel1) / dt;
  e->err[0] = teb_oracle_penalty_interval(acc_lin, c->acc_lim_x, c->penalty_epsilon);
  double omega2 = e->twist[2];
  double acc_rot = (omega2 - omega1) / dt;
  e->err[1] = teb_oracle_penalty_interval(acc_rot, c->acc_lim_theta, c->penalty_epsilon);
}
/* EdgeVelocityObstacleRatio::computeError edge_velocity_obstacle_ratio.h:82-122 */
static void ce_vel_obst_ratio(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double vel, omega;
  seg_vel(c, P(g, e->vidx[0]), P(g, e->vidx[1]), DT(g, e->vidx[2]), &vel, &omega);
  double dist_to_obstacle = footprint_dist(c, P(g, e->vidx[0]), e->ob, g->pverts);
  double ratio;
  if (dist_to_obstacle < c->obstacle_proximity_lower_bound) ratio = 0;
  else if (dist_to_obstacle > c->obstacle_proximity_upper_bound) ratio = 1;
  else ratio = (dist_to_obstacle - c->obstacle_proximity_lower_bound) /
               (c->obstacle_proximity_upper_bound - c->obstacle_proximity_lower_bound);
  ratio *= c->obstacle_proximity_ratio_max_vel;
  const double max_vel_fwd = ratio * c->max_vel_x;
  const double max_omega = ratio * c->max_vel_theta;
  e->err[0] = teb_oracle_penalty_interval(vel, max_vel_fwd, 0);
  e->err[1] = teb_oracle_penalty_interval(omega, max_omega, 0);
}
/* holonomic segment velocities in the frame of the first pose (edge_velocity.h:247-254, edge_acceleration.h:502-517) */
static inline void seg_vel_holo(const double* p1, const double* p2, double dt, double* vx, double* vy, double* omega) {
  double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
  double c1 = cos(p1[2]), s1 = sin(p1[2]);
  double r_dx = c1 * dx + s1 * dy;
  double r_dy = -s1 * dx + c1 * dy;
  *vx = r_dx / dt;
  *vy = r_dy / dt;
  *omega = nt(p2[2] - p1[2]) / dt;
}
/* EdgeVelocityHolonomic::computeError edge_velocity.h:236-273 */
static void ce_velocity_holo(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double vx, vy, omega;
  seg_vel_holo(P(g, e->vidx[0]), P(g, e->vidx[1]), DT(g, e->vidx[2]), &vx, &vy, &omega);
  double rem_y = sqrt(fmax(0.0, c->max_vel_trans * c->max_vel_trans - vx * vx));
  double rem_x = sqrt(fmax(0.0, c->max_vel_trans * c->max_vel_trans - vy * vy));
  double max_vel_y = fmin(rem_y, c->max_vel_y);
  double max_vel_x = fmin(rem_x, c->max_vel_x);
  double max_vel_x_backwards = fmin(rem_x, c->max_vel_x_backwards);
  e->err[0] = teb_oracle_penalty_interval2(vx, -max_vel_x_backwards, max_vel_x, 0.0);
  e->err[1] = teb_oracle_penalty_interval(vy, max_vel_y, 0.0);
  e->err[2] = teb_oracle_penalty_interval(omega, c->max_vel_theta, c->penalty_epsilon);
}
/* EdgeAccelerationHolonomic::computeError edge_acceleration.h:487-540 */
static void ce_acc_holo(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double dt1 = DT(g, e->vidx[3]), dt2 = DT(g, e->vidx[4]);
  double v1x, v1y, w1, v2x, v2y, w2;
  seg_vel_holo(P(g, e->vidx[0]), P(g, e->vidx[1]), dt1, &v1x, &v1y, &w1);
  seg_vel_holo(P(g, e->vidx[1]), P(g, e->vidx[2]), dt2, &v2x, &v2y, &w2);
  double dt12 = dt1 + dt2;
  e->err[0] = teb_oracle_penalty_interval((v2x - v1x) * 2 / dt12, c->acc_lim_x, c->penalty_epsilon);
  e->err[1] = teb_oracle_penalty_interval((v2y - v1y) * 2 / dt12, c->acc_lim_y, c->penalty_epsilon);
  e->err[2] = teb_oracle_penalty_interval((w2 - w1) * 2 / dt12, c->acc_lim_theta, c->penalty_epsilon);
}
/* EdgeAccelerationHolonomicStart::computeError edge_acceleration.h:580-620 */
static void ce_acc_holo_start(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double dt = DT(g, e->vidx[2]);
  double v2x, v2y, w2;
  seg_vel_holo(P(g, e->vidx[0]), P(g, e->vidx[1]), dt, &v2x, &v2y, &w2);
  e->err[0] = teb_oracle_penalty_interval((v2x - e->twist[0]) / dt, c->acc_lim_x, c->penalty_epsilon);
  e->err[1] = teb_oracle_penalty_interval((v2y - e->twist[1]) / dt, c->acc_lim_y, c->penalty_epsilon);
  e->err[2] = teb_oracle_penalty_interval((w2 - e->twist[2]) / dt, c->acc_lim_theta, c->penalty_epsilon);
}
/* EdgeAccelerationHolonomicGoal::computeError edge_acceleration.h:672-712 */
static void ce_acc_holo_goal(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  double dt = DT(g, e->vidx[2]);
  double v1x, v1y, w1;
  seg_vel_holo(P(g, e->vidx[0]), P(g, e->vidx[1]), dt, &v1x, &v1y, &w1);
  e->err[0] = teb_oracle_penalty_interval((e->twist[0] - v1x) / dt, c->acc_lim_x, c->penalty_epsilon);
  e->err[1] = teb_oracle_penalty_interval((e->twist[1] - v1y) / dt, c->acc_lim_y, c->penalty_epsilon);
  e->err[2] = teb_oracle_penalty_interval((e->twist[2] - w1) / dt, c->acc_lim_theta, c->penalty_epsilon);
}
/* EdgeTimeOptimal::computeError edge_time_optimal.h:88-96 */
static void ce_timeopt(Edge* e, Graph* g) { e->err[0] = DT(g, e->vidx[0]); }
/* EdgeShortestPath::computeError edge_shortest_path.h:73-81 */
static void ce_shortest(Edge* e, Graph* g) {
  const double *p1 = P(g, e->vidx[0]), *p2 = P(g, e->vidx[1]);
  double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
  e->err[0] = sqrt(dx * dx + dy * dy);
}
/* EdgeKinematicsDiffDrive::computeError edge_kinematics.h:89-105 */
static void ce_kin_dd(Edge* e, Graph* g) {
  const double *p1 = P(g, e->vidx[0]), *p2 = P(g, e->vidx[1]);
  double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
  e->err[0] = fabs((cos(p1[2]) + cos(p2[2])) * dy - (sin(p1[2]) + sin(p2[2])) * dx);
  double dot = dx * cos(p1[2]) + dy * sin(p1[2]);
  e->err[1] = teb_oracle_penalty_below(dot, 0, 0);
}
/* EdgeKinematicsCarlike::computeError edge_kinematics.h:198-218 */
static void ce_kin_cl(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  const double *p1 = P(g, e->vidx[0]), *p2 = P(g, e->vidx[1]);
  double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
  e->err[0] = fabs((cos(p1[2]) + cos(p2[2])) * dy - (sin(p1[2]) + sin(p2[2])) * dx);
  double angle_diff = nt(p2[2] - p1[2]);
  double norm = sqrt(dx * dx + dy * dy);
  if (angle_diff == 0)
    e->err[1] = 0;
  else if (c->exact_arc_length)
    e->err[1] = teb_oracle_penalty_below(fabs(norm / (2 * sin(angle_diff / 2))), c->min_turning_radius, 0.0);
  else
    e->err[1] = teb_oracle_penalty_below(norm / fabs(angle_diff), c->min_turning_radius, 0.0);
}
/* EdgePreferRotDir::computeError edge_prefer_rotdir.h:80-88 */
static void ce_rotdir(Edge* e, Graph* g) {
  const double *p1 = P(g, e->vidx[0]), *p2 = P(g, e->vidx[1]);
  e->err[0] = teb_oracle_penalty_below(e->meas * nt(p2[2] - p1[2]), 0, 0);
}

/* ------------------------------------------------------------------ Jacobians */
static inline int edge_vertex_fixed(const Graph* g, const Edge* e, int k) {
  return e->vkind[k] == 0 && pose_fixed(g, e->vidx[k]);
}

/* VertexPose::oplusImpl -> PoseSE2::plus (vertex_pose.h:195, pose_se2.h:238); VertexTimeDiff::oplusImpl (vertex_timediff.h:113) */
static inline void vertex_oplus(Graph* g, int kind, int idx, const double* d) {
  double* r = g->rec + 4 * idx;
  if (kind == 0) {
    r[0] += d[0];
    r[1] += d[1];
    r[2] = nt(r[2] + d[2]);
  } else {
    r[3] += d[0];
  }
}

/* g2o BaseMultiEdge/BaseBinaryEdge/BaseUnaryEdge::linearizeOplus numeric default (App. A.3) */
static void linearize_numeric(Edge* e, Graph* g) {
  const double delta = 1e-9;
  const double scalar = 1.0 / (2 * delta);
  double err_before[3] = {e->err[0], e->err[1], e->err[2]};
  for (int k = 0; k < e->nv; ++k) {
    if (edge_vertex_fixed(g, e, k)) continue;
    int vd = vdim(e->vkind[k]);
    double* r = g->rec + 4 * e->vidx[k];
    for (int d = 0; d < vd; ++d) {
      double add[3] = {0, 0, 0};
      double save[4] = {r[0], r[1], r[2], r[3]}; /* push() */
      add[d] = delta;
      vertex_oplus(g, e->vkind[k], e->vidx[k], add);
      e->compute_error(e, g);
      double eb0 = e->err[0], eb1 = e->err[1], eb2 = e->err[2];
      r[0] = save[0]; r[1] = save[1]; r[2] = save[2]; r[3] = save[3]; /* pop() */
      add[d] = -delta;
      vertex_oplus(g, e->vkind[k], e->vidx[k], add);
      e->compute_error(e, g);
      eb0 -= e->err[0];
      eb1 -= e->err[1];
      eb2 -= e->err[2];
      r[0] = save[0]; r[1] = save[1]; r[2] = save[2]; r[3] = save[3];
      e->J[k][0 * vd + d] = scalar * eb0;
      if (e->dim > 1) e->J[k][1 * vd + d] = scalar * eb1;
      if (e->dim > 2) e->J[k][2 * vd + d] = scalar * eb2;
    }
  }
  e->err[0] = err_before[0];
  e->err[1] = err_before[1];
  e->err[2] = err_before[2];
}

/* EdgeKinematicsDiffDrive::linearizeOplus — the analytic override compiled into the reference
 * (edge_kinematics.h:107-151, `#if 1`). */
static void linearize_kin_dd_reference(Edge* e, Graph* g) {
  const double *p1 = P(g, e->vidx[0]), *p2 = P(g, e->vidx[1]);
  double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
  double cos1 = cos(p1[2]), cos2 = cos(p2[2]), sin1 = sin(p1[2]), sin2 = sin(p2[2]);
  double aux1 = sin1 + sin2, aux2 = cos1 + cos2;
  double dd_error_1 = dx * cos1, dd_error_2 = dy * sin1;
  double dd_dev = d_below(dd_error_1 + dd_error_2, 0, 0);
  double dev_nh_abs = sgn((cos1 + cos2) * dy - (sin1 + sin2) * dx);
  double* Ji = e->J[0];
  double* Jj = e->J[1];
  Ji[0] = aux1 * dev_nh_abs;
  Ji[1] = -aux2 * dev_nh_abs;
  Ji[3] = -cos1 * dd_dev;
  Ji[4] = -sin1 * dd_dev;
  Ji[2] = (-dd_error_2 - dd_error_1) * dev_nh_abs;
  Ji[5] = (-sin1 * dx + cos1 * dy) * dd_dev;
  Jj[0] = -aux1 * dev_nh_abs;
  Jj[1] = aux2 * dev_nh_abs;
  Jj[3] = cos1 * dd_dev;
  Jj[4] = sin1 * dd_dev;
  Jj[2] = (-sin2 * dy - cos2 * dx) * dev_nh_abs;
  Jj[5] = 0;
}

/* ---- closed-form Jacobians for every edge (ORACLE_JAC_ANALYTIC); derivations in DESIGN.md §4 ---- */
typedef struct SegD {
  double v, w;
  double dv[7]; /* d v / d (x1,y1,th1,x2,y2,th2,dt) */
  double dw[7];
} SegD;

static void seg_derivs(const TebParams* c, const double* p1, const double* p2, double dt, SegD* s) {
  double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
  double dist = sqrt(dx * dx + dy * dy);
  double ad = nt(p2[2] - p1[2]);
  double c1 = cos(p1[2]), s1 = sin(p1[2]);
  double ux = dist > 0 ? dx / dist : 0.0, uy = dist > 0 ? dy / dist : 0.0;
  double L = dist, gfac = 1.0, dg = 0.0;
  if (c->exact_arc_length && ad != 0) {
    double h = ad / 2, sh = sin(h);
    gfac = fabs(ad / (2 * sh));
    double q = ad / (2 * sh);
    double dq = (2 * sh - ad * cos(h)) / (4 * sh * sh);
    dg = sgn(q) * dq;
    L = fabs(ad * (dist / (2 * sh)));
  }
  double dL[7] = {-gfac * ux, -gfac * uy, -dist * dg, gfac * ux, gfac * uy, dist * dg, 0};
  double proj = dx * c1 + dy * s1;
  double u = 100 * proj;
  double sig = u / (1 + fabs(u));
  double dsig = 1.0 / ((1 + fabs(u)) * (1 + fabs(u)));
  double dproj[7] = {-c1, -s1, -dx * s1 + dy * c1, c1, s1, 0, 0};
  s->v = L / dt * sig;
  s->w = ad / dt;
  for (int k = 0; k < 6; ++k) s->dv[k] = (dL[k] * sig + L * 100 * dsig * dproj[k]) / dt;
  s->dv[6] = -s->v / dt;
  s->dw[0] = s->dw[1] = s->dw[3] = s->dw[4] = 0;
  s->dw[2] = -1 / dt;
  s->dw[5] = 1 / dt;
  s->dw[6] = -s->w / dt;
}

/* distance gradient of the footprint model wrt (x,y,theta); pos of obstacle given (ox,oy) */
static void footprint_grad(const TebParams* c, const double* pose, double ox, double oy, double orad, double* dist,
                           double grad[3]) {
  double px = pose[0], py = pose[1];
  if (c->footprint_type == TEB_FOOTPRINT_TWO_CIRCLES) {
    double cx = cos(pose[2]), sy = sin(pose[2]);
    double fx = px + c->footprint_front_offset * cx - ox, fy = py + c->footprint_front_offset * sy - oy;
    double rx = px - c->footprint_rear_offset * cx - ox, ry = py - c->footprint_rear_offset * sy - oy;
    double nf = sqrt(fx * fx + fy * fy), nr = sqrt(rx * rx + ry * ry);
    double df = nf - orad - c->footprint_front_radius, dr = nr - orad - c->footprint_rear_radius;
    if (df < dr) {
      *dist = df;
      double ux = nf > 0 ? fx / nf : 0, uy = nf > 0 ? fy / nf : 0;
      grad[0] = ux; grad[1] = uy;
      grad[2] = c->footprint_front_offset * (-sy * ux + cx * uy);
    } else {
      *dist = dr;
      double ux = nr > 0 ? rx / nr : 0, uy = nr > 0 ? ry / nr : 0;
      grad[0] = ux; grad[1] = uy;
      grad[2] = -c->footprint_rear_offset * (-sy * ux + cx * uy);
    }
    return;
  }
  double dx = px - ox, dy = py - oy;
  double nrm = sqrt(dx * dx + dy * dy);
  *dist = nrm - orad - (c->footprint_type == TEB_FOOTPRINT_CIRCULAR ? c->footprint_radius : 0.0);
  grad[0] = nrm > 0 ? dx / nrm : 0;
  grad[1] = nrm > 0 ? dy / nrm : 0;
  grad[2] = 0;
}

typedef struct HoloD {
  double vx, vy, w;
  double dvx[7], dvy[7], dw[7]; /* d / d (x1,y1,th1,x2,y2,th2,dt) */
} HoloD;
static void holo_derivs(const double* p1, const double* p2, double dt, HoloD* h) {
  double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
  double c1 = cos(p1[2]), s1 = sin(p1[2]);
  double rdx = c1 * dx + s1 * dy, rdy = -s1 * dx + c1 * dy;
  double idt = 1.0 / dt;
  h->vx = rdx * idt; h->vy = rdy * idt; h->w = nt(p2[2] - p1[2]) * idt;
  double a[7] = {-c1, -s1, rdy, c1, s1, 0, 0}, b[7] = {s1, -c1, -rdx, -s1, c1, 0, 0};
  for (int k = 0; k < 6; ++k) { h->dvx[k] = a[k] * idt; h->dvy[k] = b[k] * idt; h->dw[k] = 0; }
  h->dvx[6] = -h->vx * idt; h->dvy[6] = -h->vy * idt;
  h->dw[2] = -idt; h->dw[5] = idt; h->dw[6] = -h->w * idt;
}

static void linearize_analytic(Edge* e, Graph* g) {
  const TebParams* c = g->cfg;
  memset(e->J, 0, sizeof(e->J));
  switch (e->type) {
    case E_OBST:
    case E_INFL:
    case E_DYN: {
      double dist, gr[3];
      double ox = e->ob->x, oy = e->ob->y;
      if (e->type == E_DYN) { ox += e->t * e->ob->vx; oy += e->t * e->ob->vy; }
      if (generic_pair(c, e->ob)) dist = generic_distance(c, P(g, e->vidx[0]), e->ob, g->pverts, e->type == E_DYN ? e->t : 0.0, gr);
      else footprint_grad(c, P(g, e->vidx[0]), ox, oy, e->ob->radius, &dist, gr);
      double s0 = d_below(dist, c->min_obstacle_dist, c->penalty_epsilon);
      if (e->type != E_DYN && c->obstacle_cost_exponent != 1.0 && c->min_obstacle_dist > 0.0) {
        double e0 = teb_oracle_penalty_below(dist, c->min_obstacle_dist, c->penalty_epsilon);
        s0 *= (e0 > 0) ? c->obstacle_cost_exponent * pow(e0 / c->min_obstacle_dist, c->obstacle_cost_exponent - 1.0) : 0.0;
      }
      for (int d = 0; d < 3; ++d) e->J[0][d] = s0 * gr[d];
      if (e->type == E_INFL) {
        double s1 = d_below(dist, c->inflation_dist, 0.0);
        for (int d = 0; d < 3; ++d) e->J[0][3 + d] = s1 * gr[d];
      } else if (e->type == E_DYN) {
        double s1 = d_below(dist, c->dynamic_obstacle_inflation_dist, 0.0);
        for (int d = 0; d < 3; ++d) e->J[0][3 + d] = s1 * gr[d];
      }
      break;
    }
    case E_VIA: {
      const double* p = P(g, e->vidx[0]);
      double dx = p[0] - e->via[0], dy = p[1] - e->via[1];
      double nrm = sqrt(dx * dx + dy * dy);
      e->J[0][0] = nrm > 0 ? dx / nrm : 0;
      e->J[0][1] = nrm > 0 ? dy / nrm : 0;
      break;
    }
    case E_VEL: {
      SegD s;
      seg_derivs(c, P(g, e->vidx[0]), P(g, e->vidx[1]), DT(g, e->vidx[2]), &s);
      double s0 = d_interval2(s.v, -c->max_vel_x_backwards, c->max_vel_x, c->penalty_epsilon);
      double s1 = d_interval(s.w, c->max_vel_theta, c->penalty_epsilon);
      for (int d = 0; d < 3; ++d) {
        e->J[0][d] = s0 * s.dv[d];       e->J[0][3 + d] = s1 * s.dw[d];
        e->J[1][d] = s0 * s.dv[3 + d];   e->J[1][3 + d] = s1 * s.dw[3 + d];
      }
      e->J[2][0] = s0 * s.dv[6];
      e->J[2][1] = s1 * s.dw[6];
      break;
    }
    case E_ACC: {
      SegD a, bq;
      double dt1 = DT(g, e->vidx[3]), dt2 = DT(g, e->vidx[4]);
      seg_derivs(c, P(g, e->vidx[0]), P(g, e->vidx[1]), dt1, &a);
      seg_derivs(c, P(g, e->vidx[1]), P(g, e->vidx[2]), dt2, &bq);
      double T = dt1 + dt2;
      double acc = (bq.v - a.v) * 2 / T, accr = (bq.w - a.w) * 2 / T;
      double s0 = d_interval(acc, c->acc_lim_x, c->penalty_epsilon);
      double s1 = d_interval(accr, c->acc_lim_theta, c->penalty_epsilon);
      for (int d = 0; d < 3; ++d) {
        /* pose1: only segment a (as first pose) */
        e->J[0][d] = s0 * (-2 * a.dv[d] / T);             e->J[0][3 + d] = s1 * (-2 * a.dw[d] / T);
        /* pose2: second pose of a, first pose of b */
        e->J[1][d] = s0 * (2 * (bq.dv[d] - a.dv[3 + d]) / T); e->J[1][3 + d] = s1 * (2 * (bq.dw[d] - a.dw[3 + d]) / T);
        /* pose3: second pose of b */
        e->J[2][d] = s0 * (2 * bq.dv[3 + d] / T);         e->J[2][3 + d] = s1 * (2 * bq.dw[3 + d] / T);
      }
      e->J[3][0] = s0 * (-2 * a.dv[6] / T - acc / T);
      e->J[3][1] = s1 * (-2 * a.dw[6] / T - accr / T);
      e->J[4][0] = s0 * (2 * bq.dv[6] / T - acc / T);
      e->J[4][1] = s1 * (2 * bq.dw[6] / T - accr / T);
      break;
    }
    case E_ACC_START: {
      SegD s;
      double dt = DT(g, e->vidx[2]);
      seg_derivs(c, P(g, e->vidx[0]), P(g, e->vidx[1]), dt, &s);
      double acc = (s.v - e->twist[0]) / dt, accr = (s.w - e->twist[2]) / dt;
      double s0 = d_interval(acc, c->acc_lim_x, c->penalty_epsilon);
      double s1 = d_interval(accr, c->acc_lim_theta, c->penalty_epsilon);
      for (int d = 0; d < 3; ++d) {
        e->J[0][d] = s0 * s.dv[d] / dt;       e->J[0][3 + d] = s1 * s.dw[d] / dt;
        e->J[1][d] = s0 * s.dv[3 + d] / dt;   e->J[1][3 + d] = s1 * s.dw[3 + d] / dt;
      }
      e->J[2][0] = s0 * (s.dv[6] / dt - acc / dt);
      e->J[2][1] = s1 * (s.dw[6] / dt - accr / dt);
      break;
    }
    case E_ACC_GOAL: {
      SegD s;
      double dt = DT(g, e->vidx[2]);
      seg_derivs(c, P(g, e->vidx[0]), P(g, e->vidx[1]), dt, &s);
      double acc = (e->twist[0] - s.v) / dt, accr = (e->twist[2] - s.w) / dt;
      double s0 = d_interval(acc, c->acc_lim_x, c->penalty_epsilon);
      double s1 = d_interval(accr, c->acc_lim_theta, c->penalty_epsilon);
      for (int d = 0; d < 3; ++d) {
        e->J[0][d] = -s0 * s.dv[d] / dt;       e->J[0][3 + d] = -s1 * s.dw[d] / dt;
        e->J[1][d] = -s0 * s.dv[3 + d] / dt;   e->J[1][3 + d] = -s1 * s.dw[3 + d] / dt;
      }
      e->J[2][0] = s0 * (-s.dv[6] / dt - acc / dt);
      e->J[2][1] = s1 * (-s.dw[6] / dt - accr / dt);
      break;
    }
    case E_VEL_OBST_RATIO: {
      SegD s;
      seg_derivs(c, P(g, e->vidx[0]), P(g, e->vidx[1]), DT(g, e->vidx[2]), &s);
      double dist, gr[3];
      if (generic_pair(c, e->ob)) dist = generic_distance(c, P(g, e->vidx[0]), e->ob, g->pverts, 0.0, gr);
      else footprint_grad(c, P(g, e->vidx[0]), e->ob->x, e->ob->y, e->ob->radius, &dist, gr);
      double ratio, dratio = 0;
      if (dist < c->obstacle_proximity_lower_bound) ratio = 0;
      else if (dist > c->obstacle_proximity_upper_bound) ratio = 1;
      else {
        ratio = (dist - c->obstacle_proximity_lower_bound) / (c->obstacle_proximity_upper_bound - c->obstacle_proximity_lower_bound);
        dratio = 1.0 / (c->obstacle_proximity_upper_bound - c->obstacle_proximity_lower_bound);
      }
      ratio *= c->obstacle_proximity_ratio_max_vel;
      dratio *= c->obstacle_proximity_ratio_max_vel;
      double s0 = d_interval(s.v, ratio * c->max_vel_x, 0), s1 = d_interval(s.w, ratio * c->max_vel_theta, 0);
      /* e = |var| - a outside the interval: d e / d a = -1 whenever the penalty is active */
      double a0 = (s0 != 0) ? -c->max_vel_x * dratio : 0.0, a1 = (s1 != 0) ? -c->max_vel_theta * dratio : 0.0;
      for (int d = 0; d < 3; ++d) {
        e->J[0][d] = s0 * s.dv[d] + a0 * gr[d];       e->J[0][3 + d] = s1 * s.dw[d] + a1 * gr[d];
        e->J[1][d] = s0 * s.dv[3 + d];                e->J[1][3 + d] = s1 * s.dw[3 + d];
      }
      e->J[2][0] = s0 * s.dv[6];
      e->J[2][1] = s1 * s.dw[6];
      break;
    }
    case E_VEL_HOLO: {
      const double *p1 = P(g, e->vidx[0]), *p2 = P(g, e->vidx[1]);
      double dt = DT(g, e->vidx[2]);
      HoloD h;
      holo_derivs(p1, p2, dt, &h);
      double vt2 = c->max_vel_trans * c->max_vel_trans;
      double rem_y = sqrt(fmax(0.0, vt2 - h.vx * h.vx)), rem_x = sqrt(fmax(0.0, vt2 - h.vy * h.vy));
      double mvy = fmin(rem_y, c->max_vel_y), mvx = fmin(rem_x, c->max_vel_x), mvxb = fmin(rem_x, c->max_vel_x_backwards);
      double s0 = d_interval2(h.vx, -mvxb, mvx, 0.0), s1 = d_interval(h.vy, mvy, 0.0);
      double s2 = d_interval(h.w, c->max_vel_theta, c->penalty_epsilon);
      /* bound derivative: d rem_x / d vy = -vy / rem_x when rem_x is the active (smaller) bound and positive */
      double lim0 = s0 < 0 ? c->max_vel_x_backwards : c->max_vel_x;
      double k0 = (s0 != 0 && !(lim0 < rem_x) && rem_x > 0) ? (-h.vy / rem_x) : 0.0; /* d bound / d vy */
      double k1 = (s1 != 0 && !(c->max_vel_y < rem_y) && rem_y > 0) ? (-h.vx / rem_y) : 0.0; /* d bound / d vx */
      for (int d = 0; d < 3; ++d) {
        e->J[0][0 * 3 + d] = s0 * h.dvx[d] - k0 * h.dvy[d];         e->J[1][0 * 3 + d] = s0 * h.dvx[3 + d] - k0 * h.dvy[3 + d];
        e->J[0][1 * 3 + d] = s1 * h.dvy[d] - k1 * h.dvx[d];         e->J[1][1 * 3 + d] = s1 * h.dvy[3 + d] - k1 * h.dvx[3 + d];
        e->J[0][2 * 3 + d] = s2 * h.dw[d];                          e->J[1][2 * 3 + d] = s2 * h.dw[3 + d];
      }
      e->J[2][0] = s0 * h.dvx[6] - k0 * h.dvy[6];
      e->J[2][1] = s1 * h.dvy[6] - k1 * h.dvx[6];
      e->J[2][2] = s2 * h.dw[6];
      break;
    }
    case E_ACC_HOLO: {
      double dt1 = DT(g, e->vidx[3]), dt2 = DT(g, e->vidx[4]);
      HoloD a, bq;
      holo_derivs(P(g, e->vidx[0]), P(g, e->vidx[1]), dt1, &a);
      holo_derivs(P(g, e->vidx[1]), P(g, e->vidx[2]), dt2, &bq);
      double T = dt1 + dt2;
      double acc[3] = {(bq.vx - a.vx) * 2 / T, (bq.vy - a.vy) * 2 / T, (bq.w - a.w) * 2 / T};
      double sl[3] = {d_interval(acc[0], c->acc_lim_x, c->penalty_epsilon), d_interval(acc[1], c->acc_lim_y, c->penalty_epsilon),
                      d_interval(acc[2], c->acc_lim_theta, c->penalty_epsilon)};
      const double* da[3] = {a.dvx, a.dvy, a.dw};
      const double* db[3] = {bq.dvx, bq.dvy, bq.dw};
      for (int r = 0; r < 3; ++r) {
        for (int d = 0; d < 3; ++d) {
          e->J[0][r * 3 + d] = sl[r] * (-2 * da[r][d] / T);
          e->J[1][r * 3 + d] = sl[r] * (2 * (db[r][d] - da[r][3 + d]) / T);
          e->J[2][r * 3 + d] = sl[r] * (2 * db[r][3 + d] / T);
        }
        e->J[3][r] = sl[r] * (-2 * da[r][6] / T - acc[r] / T);
        e->J[4][r] = sl[r] * (2 * db[r][6] / T - acc[r] / T);
      }
      break;
    }
    case E_ACC_HOLO_START:
    case E_ACC_HOLO_GOAL: {
      double dt = DT(g, e->vidx[2]);
      HoloD h;
      holo_derivs(P(g, e->vidx[0]), P(g, e->vidx[1]), dt, &h);
      double sg = (e->type == E_ACC_HOLO_START) ? 1.0 : -1.0; /* start: (v_seg - v0)/dt, goal: (v_goal - v_seg)/dt */
      double val[3] = {h.vx, h.vy, h.w};
      double acc[3], sl[3];
      double lim[3] = {c->acc_lim_x, c->acc_lim_y, c->acc_lim_theta};
      const double* dd[3] = {h.dvx, h.dvy, h.dw};
      for (int r = 0; r < 3; ++r) {
        acc[r] = sg * (val[r] - e->twist[r]) / dt;
        sl[r] = d_interval(acc[r], lim[r], c->penalty_epsilon);
        for (int d = 0; d < 3; ++d) {
          e->J[0][r * 3 + d] = sl[r] * sg * dd[r][d] / dt;
          e->J[1][r * 3 + d] = sl[r] * sg * dd[r][3 + d] / dt;
        }
        e->J[2][r] = sl[r] * (sg * dd[r][6] / dt - acc[r] / dt);
      }
      break;
    }
    case E_TIMEOPT: e->J[0][0] = 1; break;
    case E_SHORTEST: {
      const double *p1 = P(g, e->vidx[0]), *p2 = P(g, e->vidx[1]);
      double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
      double nrm = sqrt(dx * dx + dy * dy);
      double ux = nrm > 0 ? dx / nrm : 0, uy = nrm > 0 ? dy / nrm : 0;
      e->J[0][0] = -ux; e->J[0][1] = -uy;
      e->J[1][0] = ux;  e->J[1][1] = uy;
      break;
    }
    case E_KIN_DD: linearize_kin_dd_reference(e, g); break;
    case E_KIN_CL: {
      const double *p1 = P(g, e->vidx[0]), *p2 = P(g, e->vidx[1]);
      double dx = p2[0] - p1[0], dy = p2[1] - p1[1];
      double cos1 = cos(p1[2]), cos2 = cos(p2[2]), sin1 = sin(p1[2]), sin2 = sin(p2[2]);
      double A = (cos1 + cos2) * dy - (sin1 + sin2) * dx;
      double sa = sgn(A);
      e->J[0][0] = (sin1 + sin2) * sa;
      e->J[0][1] = -(cos1 + cos2) * sa;
      e->J[0][2] = (-sin1 * dy - cos1 * dx) * sa;
      e->J[1][0] = -(sin1 + sin2) * sa;
      e->J[1][1] = (cos1 + cos2) * sa;
      e->J[1][2] = (-sin2 * dy - cos2 * dx) * sa;
      double ad = nt(p2[2] - p1[2]);
      double nrm = sqrt(dx * dx + dy * dy);
      if (ad != 0) {
        double ux = nrm > 0 ? dx / nrm : 0, uy = nrm > 0 ? dy / nrm : 0;
        double r, dr_dn, dr_dad;
        if (c->exact_arc_length) {
          double h = ad / 2, sh = sin(h);
          double q = nrm / (2 * sh);
          r = fabs(q);
          dr_dn = sgn(q) / (2 * sh);
          dr_dad = sgn(q) * (-nrm * cos(h) / (4 * sh * sh));
        } else {
          r = nrm / fabs(ad);
          dr_dn = 1 / fabs(ad);
          dr_dad = -nrm * sgn(ad) / (ad * ad);
        }
        double s1 = d_below(r, c->min_turning_radius, 0.0);
        e->J[0][3] = s1 * dr_dn * (-ux);
        e->J[0][4] = s1 * dr_dn * (-uy);
        e->J[0][5] = s1 * (-dr_dad);
        e->J[1][3] = s1 * dr_dn * ux;
        e->J[1][4] = s1 * dr_dn * uy;
        e->J[1][5] = s1 * dr_dad;
      }
      break;
    }
    case E_ROTDIR: {
      const double *p1 = P(g, e->vidx[0]), *p2 = P(g, e->vidx[1]);
      double s0 = d_below(e->meas * nt(p2[2] - p1[2]), 0, 0);
      e->J[0][2] = -s0 * e->meas;
      e->J[1][2] = s0 * e->meas;
      break;
    }
    default: break;
  }
}

static void linearize(Edge* e, Graph* g, int jac_mode) {
  if (jac_mode == ORACLE_JAC_ANALYTIC) {
    linearize_analytic(e, g);
    return;
  }
  /* g2o mode: USE_ANALYTIC_JACOBI is defined (teb_config.h:52) but only two overrides are compiled in */
  if (e->type == E_KIN_DD) {
    linearize_kin_dd_reference(e, g);
  } else if (e->type == E_TIMEOPT) {
    e->J[0][0] = 1; /* edge_time_optimal.h:98-107 */
  } else {
    linearize_numeric(e, g);
  }
}

/* ------------------------------------------------------------------ graph construction (buildGraph) */
static Edge* new_edge(Graph* g, int type, int dim, void (*ce)(Edge*, Graph*)) {
  Edge* e = (Edge*)calloc(1, sizeof(Edge)); /* `new EdgeXxx` per edge per outer iteration, as the reference does */
  e->type = type;
  e->dim = dim;
  e->compute_error = ce;
  if (g->n_edges == g->cap_edges) {
    g->cap_edges = g->cap_edges ? 2 * g->cap_edges : 1024;
    g->edges = (Edge**)realloc(g->edges, sizeof(Edge*) * g->cap_edges);
  }
  g->edges[g->n_edges++] = e;
  return e;
}
static inline void set_vertex(Edge* e, int k, int kind, int idx) {
  e->vkind[k] = kind;
  e->vidx[k] = idx;
  if (k + 1 > e->nv) e->nv = k + 1;
}

/* AddEdgesObstacles optimal_planner.cpp:444-548 */
static void add_edges_obstacles(Graph* g, double weight_multiplier) {
  const TebParams* c = g->cfg;
  if (c->weight_obstacle == 0 || weight_multiplier == 0 || g->obst == NULL) return;
  int inflated = c->inflation_dist > c->min_obstacle_dist;
  const int first_vertex = c->weight_velocity_obstacle_ratio == 0 ? 1 : 0;
  int* list = (int*)malloc(sizeof(int) * (g->M + 2));
  for (int i = first_vertex; i < g->n - 1; ++i) {
    int cnt = 0;
    double left_min = DBL_MAX, right_min = DBL_MAX;
    int left = -1, right = -1;
    const double* p = P(g, i);
    double ox = cos(p[2]), oy = sin(p[2]); /* orientationUnitVec */
    for (int m = 0; m < g->M; ++m) {
      const TebObstacle* ob = &g->obst[m];
      if (c->include_dynamic_obstacles && ob->dynamic) continue;
      double dist = footprint_dist(c, p, ob, g->pverts);
      if (dist < c->min_obstacle_dist * c->obstacle_association_force_inclusion_factor) {
        list[cnt++] = m;
        continue;
      }
      if (dist > c->min_obstacle_dist * c->obstacle_association_cutoff_factor) continue;
      /* cross2d(pose_orient, centroid - position) > 0 -> left (misc.h:120) */
      double cx = ob->x - p[0], cy = ob->y - p[1];
      if (ox * cy - cx * oy > 0) {
        if (dist < left_min) { left_min = dist; left = m; }
      } else {
        if (dist < right_min) { right_min = dist; right = m; }
      }
    }
    if (left >= 0) list[cnt++] = left;
    if (right >= 0) list[cnt++] = right;
    for (int k = 0; k < cnt; ++k) g->opv[(size_t)i * (g->M + 2) + k] = list[k];
    g->opv_cnt[i] = cnt;
    if (i == 0) continue;
    for (int k = 0; k < cnt; ++k) {
      Edge* e;
      if (inflated) {
        e = new_edge(g, E_INFL, 2, ce_inflated);
        e->info[0] = c->weight_obstacle * weight_multiplier;
        e->info[1] = c->weight_inflation;
      } else {
        e = new_edge(g, E_OBST, 1, ce_obstacle);
        e->info[0] = c->weight_obstacle * weight_multiplier;
      }
      set_vertex(e, 0, 0, i);
      e->ob = &g->obst[list[k]];
    }
  }
  free(list);
}

/* AddEdgesObstaclesLegacy optimal_planner.cpp:551-643 (note: the centre pose receives three identical edges:
 * the explicit one plus neighbourIdx = 0 on both sides) */
static void add_obstacle_edge(Graph* g, int i, int m, int inflated, double weight_multiplier) {
  const TebParams* c = g->cfg;
  Edge* e;
  if (inflated) {
    e = new_edge(g, E_INFL, 2, ce_inflated);
    e->info[0] = c->weight_obstacle * weight_multiplier;
    e->info[1] = c->weight_inflation;
  } else {
    e = new_edge(g, E_OBST, 1, ce_obstacle);
    e->info[0] = c->weight_obstacle * weight_multiplier;
  }
  set_vertex(e, 0, 0, i);
  e->ob = &g->obst[m];
}
static int find_closest_pose(Graph* g, const double* pt, int begin_idx);
/* TimedElasticBand::findClosestTrajectoryPose(const Obstacle&) timed_elastic_band.cpp:532-547: Point -> position,
 * Line -> segment (:480-500), Polygon -> vertex list (:502-530), everything else (Circular, Pill) -> centroid */
static int find_closest_pose_obstacle(Graph* g, const TebObstacle* ob) {
  const double* v = g->pverts ? g->pverts + 2 * (size_t)ob->vertex_begin : NULL;
  int k = ob->vertex_count;
  if (ob->type == TEB_OBST_POLYGON && k == 0) return 0;
  if (ob->type == TEB_OBST_POLYGON && k == 1) return find_closest_pose(g, v, 0);
  if (ob->type == TEB_OBST_LINE || (ob->type == TEB_OBST_POLYGON && k >= 2)) {
    double min_dist = DBL_MAX;
    int min_idx = -1;
    for (int i = 0; i < g->n; i++) {
      const double* pt = P(g, i);
      double q[2], d;
      if (ob->type == TEB_OBST_LINE || k == 2) {
        closest_on_segment(pt, v, v + 2 * (k - 1), q);
        d = pt_dist(pt, q);
      } else {
        d = DBL_MAX;
        for (int j = 0; j < k; ++j) {
          closest_on_segment(pt, v + 2 * j, v + 2 * ((j + 1) % k), q);
          double dj = pt_dist(pt, q);
          if (dj < d) d = dj;
        }
      }
      if (d < min_dist) { min_dist = d; min_idx = i; }
    }
    return min_idx;
  }
  double pt[2] = {ob->x, ob->y};
  return find_closest_pose(g, pt, 0);
}
static void add_edges_obstacles_legacy(Graph* g, double weight_multiplier) {
  const TebParams* c = g->cfg;
  if (c->weight_obstacle == 0 || weight_multiplier == 0 || g->obst == NULL) return;
  int inflated = c->inflation_dist > c->min_obstacle_dist;
  for (int m = 0; m < g->M; ++m) {
    const TebObstacle* ob = &g->obst[m];
    if (c->include_dynamic_obstacles && ob->dynamic) continue;
    int index;
    if (c->obstacle_poses_affected >= g->n) index = g->n / 2;
    else index = find_closest_pose_obstacle(g, ob);
    if ((index <= 1) || (index > g->n - 2)) continue;
    add_obstacle_edge(g, index, m, inflated, weight_multiplier);
    for (int nb = 0; nb < (int)floor(c->obstacle_poses_affected / 2); nb++) {
      if (index + nb < g->n) add_obstacle_edge(g, index + nb, m, inflated, weight_multiplier);
      if (index - nb >= 0) add_obstacle_edge(g, index - nb, m, inflated, weight_multiplier);
    }
  }
}

/* AddEdgesVelocityObstacleRatio optimal_planner.cpp:999-1021 */
static void add_edges_velocity_obstacle_ratio(Graph* g) {
  const TebParams* c = g->cfg;
  for (int index = 0; index < g->n - 1; ++index) {
    for (int k = 0; k < g->opv_cnt[index]; ++k) {
      Edge* e = new_edge(g, E_VEL_OBST_RATIO, 2, ce_vel_obst_ratio);
      set_vertex(e, 0, 0, index);
      set_vertex(e, 1, 0, index + 1);
      set_vertex(e, 2, 1, index);
      e->info[0] = c->weight_velocity_obstacle_ratio;
      e->info[1] = c->weight_velocity_obstacle_ratio;
      e->ob = &g->obst[g->opv[(size_t)index * (g->M + 2) + k]];
    }
  }
}

/* AddEdgesDynamicObstacles optimal_planner.cpp:646-673 (called with weight_multiplier = 1, :343) */
static void add_edges_dynamic_obstacles(Graph* g, double weight_multiplier) {
  const TebParams* c = g->cfg;
  if (c->weight_obstacle == 0 || weight_multiplier == 0 || g->obst == NULL) return;
  for (int m = 0; m < g->M; ++m) {
    if (!g->obst[m].dynamic) continue;
    double time = DT(g, 0);
    for (int i = 1; i < g->n - 1; ++i) {
      Edge* e = new_edge(g, E_DYN, 2, ce_dynamic);
      e->t = time;
      set_vertex(e, 0, 0, i);
      e->info[0] = c->weight_dynamic_obstacle * weight_multiplier;
      e->info[1] = c->weight_dynamic_obstacle_inflation;
      e->ob = &g->obst[m];
      time += DT(g, i);
    }
  }
}

/* TimedElasticBand::findClosestTrajectoryPose(point) timed_elastic_band.cpp:455-478 */
static int find_closest_pose(Graph* g, const double* pt, int begin_idx) {
  int n = g->n;
  if (begin_idx < 0 || begin_idx >= n) return -1;
  double min_dist_sq = DBL_MAX;
  int min_idx = -1;
  for (int i = begin_idx; i < n; i++) {
    double dx = pt[0] - P(g, i)[0], dy = pt[1] - P(g, i)[1];
    double dist_sq = dx * dx + dy * dy;
    if (dist_sq < min_dist_sq) { min_dist_sq = dist_sq; min_idx = i; }
  }
  return min_idx;
}

/* AddEdgesViaPoints optimal_planner.cpp:675-718 */
static void add_edges_via_points(Graph* g) {
  const TebParams* c = g->cfg;
  if (c->weight_viapoint == 0 || g->via == NULL || g->V == 0) return;
  int start_pose_idx = 0;
  int n = g->n;
  if (n < 3) return;
  for (int k = 0; k < g->V; ++k) {
    const double* vp = g->via + 2 * k;
    int index = find_closest_pose(g, vp, start_pose_idx);
    if (c->via_points_ordered) start_pose_idx = index + 2;
    if (index > n - 2) index = n - 2;
    if (index < 1) {
      if (c->via_points_ordered) index = 1;
      else continue;
    }
    Edge* e = new_edge(g, E_VIA, 1, ce_via);
    set_vertex(e, 0, 0, index);
    e->info[0] = c->weight_viapoint;
    e->via = vp;
  }
}

/* AddEdgesVelocity optimal_planner.cpp:720-769 (non-holonomic branch) */
static void add_edges_velocity(Graph* g) {
  const TebParams* c = g->cfg;
  if (c->max_vel_y != 0) { /* holonomic robot (optimal_planner.cpp:745-767) */
    if (c->weight_max_vel_x == 0 && c->weight_max_vel_y == 0 && c->weight_max_vel_theta == 0) return;
    for (int i = 0; i < g->n - 1; ++i) {
      Edge* e = new_edge(g, E_VEL_HOLO, 3, ce_velocity_holo);
      set_vertex(e, 0, 0, i);
      set_vertex(e, 1, 0, i + 1);
      set_vertex(e, 2, 1, i);
      e->info[0] = c->weight_max_vel_x;
      e->info[1] = c->weight_max_vel_y;
      e->info[2] = c->weight_max_vel_theta;
    }
    return;
  }
  if (c->weight_max_vel_x == 0 && c->weight_max_vel_theta == 0) return;
  for (int i = 0; i < g->n - 1; ++i) {
    Edge* e = new_edge(g, E_VEL, 2, ce_velocity);
    set_vertex(e, 0, 0, i);
    set_vertex(e, 1, 0, i + 1);
    set_vertex(e, 2, 1, i);
    e->info[0] = c->weight_max_vel_x;
    e->info[1] = c->weight_max_vel_theta;
  }
}

/* AddEdgesAcceleration optimal_planner.cpp:771-873 (non-holonomic branch) */
static void add_edges_acceleration(Graph* g) {
  const TebParams* c = g->cfg;
  if (c->weight_acc_lim_x == 0 && c->weight_acc_lim_theta == 0) return;
  int n = g->n;
  if (!(c->max_vel_y == 0 || c->acc_lim_y == 0)) { /* holonomic robot (optimal_planner.cpp:824-871) */
    if (g->vel_start[3] != 0) {
      Edge* e = new_edge(g, E_ACC_HOLO_START, 3, ce_acc_holo_start);
      set_vertex(e, 0, 0, 0); set_vertex(e, 1, 0, 1); set_vertex(e, 2, 1, 0);
      e->twist = g->vel_start;
      e->info[0] = c->weight_acc_lim_x; e->info[1] = c->weight_acc_lim_y; e->info[2] = c->weight_acc_lim_theta;
    }
    for (int i = 0; i < n - 2; ++i) {
      Edge* e = new_edge(g, E_ACC_HOLO, 3, ce_acc_holo);
      set_vertex(e, 0, 0, i); set_vertex(e, 1, 0, i + 1); set_vertex(e, 2, 0, i + 2);
      set_vertex(e, 3, 1, i); set_vertex(e, 4, 1, i + 1);
      e->info[0] = c->weight_acc_lim_x; e->info[1] = c->weight_acc_lim_y; e->info[2] = c->weight_acc_lim_theta;
    }
    if (g->vel_goal[3] != 0) {
      Edge* e = new_edge(g, E_ACC_HOLO_GOAL, 3, ce_acc_holo_goal);
      set_vertex(e, 0, 0, n - 2); set_vertex(e, 1, 0, n - 1); set_vertex(e, 2, 1, n - 2);
      e->twist = g->vel_goal;
      e->info[0] = c->weight_acc_lim_x; e->info[1] = c->weight_acc_lim_y; e->info[2] = c->weight_acc_lim_theta;
    }
    return;
  }
  if (g->vel_start[3] != 0) {
    Edge* e = new_edge(g, E_ACC_START, 2, ce_acc_start);
    set_vertex(e, 0, 0, 0);
    set_vertex(e, 1, 0, 1);
    set_vertex(e, 2, 1, 0);
    e->twist = g->vel_start;
    e->info[0] = c->weight_acc_lim_x;
    e->info[1] = c->weight_acc_lim_theta;
  }
  for (int i = 0; i < n - 2; ++i) {
    Edge* e = new_edge(g, E_ACC, 2, ce_acceleration);
    set_vertex(e, 0, 0, i);
    set_vertex(e, 1, 0, i + 1);
    set_vertex(e, 2, 0, i + 2);
    set_vertex(e, 3, 1, i);
    set_vertex(e, 4, 1, i + 1);
    e->info[0] = c->weight_acc_lim_x;
    e->info[1] = c->weight_acc_lim_theta;
  }
  if (g->vel_goal[3] != 0) {
    Edge* e = new_edge(g, E_ACC_GOAL, 2, ce_acc_goal);
    set_vertex(e, 0, 0, n - 2);
    set_vertex(e, 1, 0, n - 1);
    set_vertex(e, 2, 1, n - 2); /* TimeDiffVertex(sizeTimeDiffs()-1) */
    e->twist = g->vel_goal;
    e->info[0] = c->weight_acc_lim_x;
    e->info[1] = c->weight_acc_lim_theta;
  }
}

/* AddEdgesTimeOptimal :877-893, AddEdgesShortestPath :895-913 */
static void add_edges_time_optimal(Graph* g) {
  const TebParams* c = g->cfg;
  if (c->weight_optimaltime == 0) return;
  for (int i = 0; i < g->n - 1; ++i) {
    Edge* e = new_edge(g, E_TIMEOPT, 1, ce_timeopt);
    set_vertex(e, 0, 1, i);
    e->info[0] = c->weight_optimaltime;
  }
}
static void add_edges_shortest_path(Graph* g) {
  const TebParams* c = g->cfg;
  if (c->weight_shortest_path == 0) return;
  for (int i = 0; i < g->n - 1; ++i) {
    Edge* e = new_edge(g, E_SHORTEST, 1, ce_shortest);
    set_vertex(e, 0, 0, i);
    set_vertex(e, 1, 0, i + 1);
    e->info[0] = c->weight_shortest_path;
  }
}
/* AddEdgesKinematicsDiffDrive :916-936, AddEdgesKinematicsCarlike :938-958 */
static void add_edges_kinematics(Graph* g) {
  const TebParams* c = g->cfg;
  int carlike = !(c->min_turning_radius == 0 || c->weight_kinematics_turning_radius == 0); /* :355 */
  if (!carlike) {
    if (c->weight_kinematics_nh == 0 && c->weight_kinematics_forward_drive == 0) return;
  } else {
    if (c->weight_kinematics_nh == 0 && c->weight_kinematics_turning_radius == 0) return;
  }
  for (int i = 0; i < g->n - 1; i++) {
    Edge* e = carlike ? new_edge(g, E_KIN_CL, 2, ce_kin_cl) : new_edge(g, E_KIN_DD, 2, ce_kin_dd);
    set_vertex(e, 0, 0, i);
    set_vertex(e, 1, 0, i + 1);
    e->info[0] = c->weight_kinematics_nh;
    e->info[1] = carlike ? c->weight_kinematics_turning_radius : c->weight_kinematics_forward_drive;
  }
}
/* AddEdgesPreferRotDir :961-997 */
static void add_edges_prefer_rotdir(Graph* g) {
  const TebParams* c = g->cfg;
  if (g->rotdir == TEB_ROTDIR_NONE || c->weight_prefer_rotdir == 0) return;
  if (g->rotdir != TEB_ROTDIR_RIGHT && g->rotdir != TEB_ROTDIR_LEFT) return;
  for (int i = 0; i < g->n - 1 && i < 3; ++i) {
    Edge* e = new_edge(g, E_ROTDIR, 1, ce_rotdir);
    set_vertex(e, 0, 0, i);
    set_vertex(e, 1, 0, i + 1);
    e->info[0] = c->weight_prefer_rotdir;
    e->meas = (g->rotdir == TEB_ROTDIR_LEFT) ? 1 : -1;
  }
}

static void clear_graph(Graph* g) {
  for (int k = 0; k < g->n_edges; ++k) free(g->edges[k]);
  g->n_edges = 0;
}

/* buildGraph optimal_planner.cpp:323-366 */
static int build_graph(Graph* g, double weight_multiplier) {
  const TebParams* c = g->cfg;
  /* AddTEBVertices resizes and clears obstacles_per_vertex_ (optimal_planner.cpp:427-439) */
  free(g->opv); free(g->opv_cnt);
  g->opv = (int*)malloc(sizeof(int) * (size_t)g->n * (g->M + 2));
  g->opv_cnt = (int*)calloc((size_t)g->n, sizeof(int));
  if (c->legacy_obstacle_association) add_edges_obstacles_legacy(g, weight_multiplier);
  else add_edges_obstacles(g, weight_multiplier);
  if (c->include_dynamic_obstacles) add_edges_dynamic_obstacles(g, 1.0);
  add_edges_via_points(g);
  add_edges_velocity(g);
  add_edges_acceleration(g);
  add_edges_time_optimal(g);
  add_edges_shortest_path(g);
  add_edges_kinematics(g);
  add_edges_prefer_rotdir(g);
  if (c->weight_velocity_obstacle_ratio > 0) add_edges_velocity_obstacle_ratio(g);
  /* initializeOptimization(): edges whose vertices are all fixed are not active (App. A.1) */
  int w = 0;
  for (int k = 0; k < g->n_edges; ++k) {
    Edge* e = g->edges[k];
    int all_fixed = 1;
    for (int v = 0; v < e->nv; ++v)
      if (!edge_vertex_fixed(g, e, v)) all_fixed = 0;
    if (all_fixed) free(e);
    else g->edges[w++] = e;
  }
  g->n_edges = w;
  g->N = 4 * g->n - 7;
  return 0;
}

/* ------------------------------------------------------------------ errors / quadratic form */
static double compute_active_errors(Graph* g) {
  double chi2 = 0;
  for (int k = 0; k < g->n_edges; ++k) {
    Edge* e = g->edges[k];
    e->compute_error(e, g);
    for (int d = 0; d < e->dim; ++d) chi2 += e->err[d] * e->info[d] * e->err[d];
  }
  return chi2;
}
static inline void H_add(Graph* g, int r, int q, double v) {
  if (r < q) { int t = r; r = q; q = t; }
  g->Hb[(size_t)r * (HBW + 1) + (r - q)] += v;
}

/* BlockSolver::buildSystem: linearizeOplus + constructQuadraticForm per edge (App. A.3) */
static void build_system(Graph* g, int jac_mode) {
  memset(g->Hb, 0, sizeof(double) * (size_t)g->N * (HBW + 1));
  memset(g->b, 0, sizeof(double) * (size_t)g->N);
  for (int k = 0; k < g->n_edges; ++k) {
    Edge* e = g->edges[k];
    linearize(e, g, jac_mode);
    double omega_r[3];
    for (int d = 0; d < e->dim; ++d) omega_r[d] = -e->info[d] * e->err[d];
    for (int i = 0; i < e->nv; ++i) {
      if (edge_vertex_fixed(g, e, i)) continue;
      int di = vdim(e->vkind[i]);
      int hi = hidx(g, e->vkind[i], e->vidx[i]);
      const double* A = e->J[i];
      for (int a = 0; a < di; ++a) {
        double s = 0;
        for (int d = 0; d < e->dim; ++d) s += A[d * di + a] * omega_r[d];
        g->b[hi + a] += s;
      }
      /* H_ii += A^T Omega A (lower triangle only) */
      for (int a = 0; a < di; ++a)
        for (int bq = 0; bq <= a; ++bq) {
          double s = 0;
          for (int d = 0; d < e->dim; ++d) s += A[d * di + a] * e->info[d] * A[d * di + bq];
          H_add(g, hi + a, hi + bq, s);
        }
      for (int j = i + 1; j < e->nv; ++j) {
        if (edge_vertex_fixed(g, e, j)) continue;
        int dj = vdim(e->vkind[j]);
        int hj = hidx(g, e->vkind[j], e->vidx[j]);
        const double* Bm = e->J[j];
        for (int a = 0; a < di; ++a)
          for (int bq = 0; bq < dj; ++bq) {
            double s = 0;
            for (int d = 0; d < e->dim; ++d) s += A[d * di + a] * e->info[d] * Bm[d * dj + bq];
            H_add(g, hi + a, hj + bq, s);
          }
      }
    }
  }
}

/* ------------------------------------------------------------------ linear solvers */
/* banded Cholesky (LL^T), lower storage; stand-in for LinearSolverCSparse (App. A.6). Returns 0 on
 * non-positive pivot. */
static int solve_banded(Graph* g, double lambda) {
  const int N = g->N, W = HBW + 1;
  double* L = g->work;
  memcpy(L, g->Hb, sizeof(double) * (size_t)N * W);
  for (int r = 0; r < N; ++r) L[(size_t)r * W] += lambda;
  for (int j = 0; j < N; ++j) {
    /* row j of L: entries L[j][j-k], k = HBW..0 */
    int kmax = j < HBW ? j : HBW;
    for (int k = kmax; k >= 0; --k) {
      int col = j - k;
      double s = L[(size_t)j * W + k];
      /* subtract sum_{m < col} L[j][m] L[col][m], m >= j-HBW */
      int m0 = j - HBW; if (m0 < 0) m0 = 0;
      for (int m = m0; m < col; ++m) s -= L[(size_t)j * W + (j - m)] * L[(size_t)col * W + (col - m)];
      if (k == 0) {
        if (!(s > 0) || !isfinite(s)) return 0;
        L[(size_t)j * W] = sqrt(s);
      } else {
        L[(size_t)j * W + k] = s / L[(size_t)col * W];
      }
    }
  }
  double* x = g->x;
  for (int j = 0; j < N; ++j) {
    double s = g->b[j];
    int m0 = j - HBW; if (m0 < 0) m0 = 0;
    for (int m = m0; m < j; ++m) s -= L[(size_t)j * W + (j - m)] * x[m];
    x[j] = s / L[(size_t)j * W];
  }
  for (int j = N - 1; j >= 0; --j) {
    double s = x[j];
    int m1 = j + HBW; if (m1 > N - 1) m1 = N - 1;
    for (int m = j + 1; m <= m1; ++m) s -= L[(size_t)m * W + (m - j)] * x[m];
    x[j] = s / L[(size_t)j * W];
  }
  return 1;
}
static int solve_dense(Graph* g, double lambda) {
  const int N = g->N, W = HBW + 1;
  if (!g->Hd) g->Hd = (double*)malloc(sizeof(double) * (size_t)N * N);
  double* A = g->Hd;
  memset(A, 0, sizeof(double) * (size_t)N * N);
  for (int r = 0; r < N; ++r)
    for (int k = 0; k <= HBW && k <= r; ++k) A[(size_t)r * N + (r - k)] = g->Hb[(size_t)r * W + k];
  for (int r = 0; r < N; ++r) A[(size_t)r * N + r] += lambda;
  for (int j = 0; j < N; ++j) {
    for (int i = j; i < N; ++i) {
      double s = A[(size_t)i * N + j];
      for (int m = 0; m < j; ++m) s -= A[(size_t)i * N + m] * A[(size_t)j * N + m];
      if (i == j) {
        if (!(s > 0) || !isfinite(s)) return 0;
        A[(size_t)j * N + j] = sqrt(s);
      } else {
        A[(size_t)i * N + j] = s / A[(size_t)j * N + j];
      }
    }
  }
  double* x = g->x;
  for (int j = 0; j < N; ++j) {
    double s = g->b[j];
    for (int m = 0; m < j; ++m) s -= A[(size_t)j * N + m] * x[m];
    x[j] = s / A[(size_t)j * N + j];
  }
  for (int j = N - 1; j >= 0; --j) {
    double s = x[j];
    for (int m = j + 1; m < N; ++m) s -= A[(size_t)m * N + j] * x[m];
    x[j] = s / A[(size_t)j * N + j];
  }
  return 1;
}

/* SparseOptimizer::update: every non-fixed vertex oplus its slice of x */
static void apply_update(Graph* g) {
  for (int i = 0; i < g->n - 1; ++i) {
    if (!pose_fixed(g, i)) vertex_oplus(g, 0, i, g->x + hidx(g, 0, i));
    vertex_oplus(g, 1, i, g->x + hidx(g, 1, i));
  }
}

/* ------------------------------------------------------------------ Levenberg-Marquardt (App. A.4/A.5) */
typedef struct LMState { double lambda, ni; } LMState;

/* The decision on one trial, the body of g2o's do-while after update(x) and computeActiveErrors: rho from the trial's
 * chi2 and computeScale() sum (scale_sum, without the 1e-3), the lambda / nu update, the status bits. A failed
 * factorisation counts as tempChi = DBL_MAX. *q counts the trials of the iteration; *stop is set when the loop ends
 * after this trial. Returns 1 when the trial is accepted. */
static int lm_decide_trial(double* currentChi, LMState* lm, double tempChi, double scale_sum, int ok, int* q, double* rho,
                           int32_t* status, int* stop) {
  if (!ok) { *status |= TEB_STATUS_CHOL_FAILED; tempChi = DBL_MAX; }
  *rho = (*currentChi - tempChi);
  *rho /= scale_sum + 1e-3;
  int accepted = 0;
  *stop = 0;
  if (*rho > 0 && isfinite(tempChi)) {
    double alpha = 1. - pow((2 * *rho - 1), 3);
    alpha = alpha < (2. / 3.) ? alpha : (2. / 3.);
    double scaleFactor = (1. / 3.) > alpha ? (1. / 3.) : alpha;
    lm->lambda *= scaleFactor;
    lm->ni = 2;
    *currentChi = tempChi;
    accepted = 1;
  } else {
    lm->lambda *= lm->ni;
    lm->ni *= 2;
    if (!isfinite(lm->lambda)) { *status |= TEB_STATUS_NONFINITE; *stop = 1; return 0; }
  }
  (*q)++;
  *stop = !(*rho < 0 && *q < 10);
  return accepted;
}
/* the iteration's Terminate verdict once its trial loop has ended (optimization_algorithm_levenberg.cpp) */
static int lm_terminates(int q, double rho, const LMState* lm) { return q == 10 || rho == 0 || !isfinite(lm->lambda); }

int32_t teb_oracle_lm_decide(double current_chi, double lambda, double nu, int32_t q0, int32_t count, const double* temp_chi,
                             const double* scale_sum, const int32_t* ok, int32_t* out_i, double* out_d) {
  if (!out_i || !out_d || count < 0 || q0 < 0 || (count > 0 && (!temp_chi || !scale_sum || !ok))) return -1;
  LMState lm = {lambda, nu};
  int q = q0, stop = 0, accepted = -1, used = 0;
  int32_t status = 0;
  double rho = 0;
  for (int k = 0; k < count && q < 10 && !stop; ++k, ++used)
    if (lm_decide_trial(&current_chi, &lm, temp_chi[k], scale_sum[k], ok[k] != 0, &q, &rho, &status, &stop)) accepted = k;
  out_i[0] = accepted;
  out_i[1] = used;
  out_i[2] = stop && lm_terminates(q, rho, &lm);
  out_i[3] = status;
  out_i[4] = !stop; /* the iteration needs more trials than the sequence holds */
  out_i[5] = q;
  out_d[0] = lm.lambda;
  out_d[1] = lm.ni;
  out_d[2] = current_chi;
  return 0;
}

/* returns 1 = OK, 0 = Terminate */
static int lm_solve(Graph* g, int iteration, LMState* lm, const OracleOptions* opt, OracleStats* st) {
  double currentChi = compute_active_errors(g);
  double tempChi = currentChi;
  build_system(g, opt->jac_mode);
  if (iteration == 0) {
    double maxDiagonal = 0;
    for (int r = 0; r < g->N; ++r) {
      double d = fabs(g->Hb[(size_t)r * (HBW + 1)]);
      if (d > maxDiagonal) maxDiagonal = d;
    }
    lm->lambda = 1e-5 * maxDiagonal;
    lm->ni = 2;
  }
  double rho = 0;
  int qmax = 0, stop = 0;
  do {
    memcpy(g->backup, g->rec, sizeof(double) * 4 * (size_t)g->n); /* _optimizer->push() */
    int ok2 = (opt->solver == ORACLE_SOLVER_DENSE) ? solve_dense(g, lm->lambda) : solve_banded(g, lm->lambda);
    if (!ok2) {
      /* g2o still calls update(x) with whatever the solver left in x; CSparse leaves x = b on failure.
       * The state is restored below (tempChi = DBL_MAX -> reject), so only the cached errors differ. */
      memcpy(g->x, g->b, sizeof(double) * (size_t)g->N);
    }
    st->lm_trials++;
    apply_update(g);
    tempChi = compute_active_errors(g);
    double scale = 0;
    for (int j = 0; j < g->N; ++j) scale += g->x[j] * (lm->lambda * g->x[j] + g->b[j]);
    if (!lm_decide_trial(&currentChi, lm, tempChi, scale, ok2, &qmax, &rho, &st->status, &stop)) {
      memcpy(g->rec, g->backup, sizeof(double) * 4 * (size_t)g->n); /* pop() */
      st->rejected++;
    }
  } while (!stop);
  st->chi2_final = currentChi;
  st->lambda_final = lm->lambda;
  st->nu_final = lm->ni;
  if (opt->verbose) fprintf(stderr, "LMTRIALS %d %d %.6g %.6g\n", iteration, qmax, currentChi, lm->lambda);
  return !lm_terminates(qmax, rho, lm);
}

/* SparseOptimizer::optimize(iterations) */
static int optimize_graph_lm(Graph* g, int iterations, const OracleOptions* opt, OracleStats* st) {
  LMState lm = {0, 2};
  int ok = 1, cj = 0;
  for (int i = 0; i < iterations && ok; ++i) {
    ok = lm_solve(g, i, &lm, opt, st);
    if (g->cfg->divergence_detection_enable) st->chi2_final = compute_active_errors(g); /* batch statistics */
    ++cj;
  }
  if (!ok) st->status |= TEB_STATUS_TERMINATED; else st->status &= ~TEB_STATUS_TERMINATED;
  return cj;
}

/* computeCurrentCost optimal_planner.cpp:1041-1094 (graph exists; uses the cached _error of every edge) */
static double compute_current_cost(Graph* g, double obst_scale, double via_scale, int alt_time) {
  double cost = 0;
  if (alt_time)
    for (int i = 0; i < g->n - 1; ++i) cost += DT(g, i);
  for (int k = 0; k < g->n_edges; ++k) {
    const Edge* e = g->edges[k];
    double cur = 0;
    for (int d = 0; d < e->dim; ++d) cur += e->err[d] * e->info[d] * e->err[d];
    if (e->type == E_OBST || e->type == E_INFL || e->type == E_DYN) cur *= obst_scale;
    else if (e->type == E_VIA) cur *= via_scale;
    else if (e->type == E_TIMEOPT && alt_time) continue;
    cost += cur;
  }
  return cost;
}

/* ------------------------------------------------------------------ autoResize timed_elastic_band.cpp:227-286 */
static void rec_insert(double* rec, int* n, int at, const double* r4) {
  memmove(rec + 4 * (at + 1), rec + 4 * at, sizeof(double) * 4 * (size_t)(*n - at));
  memcpy(rec + 4 * at, r4, sizeof(double) * 4);
  (*n)++;
}
int32_t teb_oracle_auto_resize(double* rec, int32_t n, int32_t n_cap, double dt_ref, double dt_hysteresis,
                               int32_t min_samples, int32_t max_samples, int32_t fast_mode) {
  /* rec[i] = (x,y,theta,dt_i); sizeTimeDiffs() = n-1. Pose i+1 travels with dt_i when inserting/deleting. */
  int modified = 1;
  for (int rep = 0; rep < 100 && modified; ++rep) {
    modified = 0;
    for (int i = 0; i < n - 1; ++i) {
      double dti = rec[4 * i + 3];
      if (dti > dt_ref + dt_hysteresis && (n - 1) < max_samples) {
        if (dti > 2 * dt_ref) {
          if (n + 1 > n_cap) return TEBGPU_ERR_CAPACITY;
          double newtime = 0.5 * dti;
          rec[4 * i + 3] = newtime;
          /* insertPose(i+1, average(Pose(i),Pose(i+1))); insertTimeDiff(i+1,newtime) */
          double nr[4];
          nr[0] = (rec[4 * i] + rec[4 * (i + 1)]) / 2;
          nr[1] = (rec[4 * i + 1] + rec[4 * (i + 1) + 1]) / 2;
          nr[2] = teb_oracle_average_angle(rec[4 * i + 2], rec[4 * (i + 1) + 2]);
          nr[3] = newtime;
          rec_insert(rec, &n, i + 1, nr);
          i--;
          modified = 1;
        } else {
          if (i < n - 2) rec[4 * (i + 1) + 3] += rec[4 * i + 3] - dt_ref;
          rec[4 * i + 3] = dt_ref;
        }
      } else if (dti < dt_ref - dt_hysteresis && (n - 1) > min_samples) {
        if (i < n - 2) {
          /* TimeDiff(i+1) += TimeDiff(i); deleteTimeDiff(i); deletePose(i+1) */
          double merged = rec[4 * (i + 1) + 3] + rec[4 * i + 3];
          memmove(rec + 4 * (i + 1), rec + 4 * (i + 2), sizeof(double) * 4 * (size_t)(n - i - 2));
          n--;
          rec[4 * i + 3] = merged;
          i--;
        } else {
          /* last interval: TimeDiff(i-1) += TimeDiff(i); deleteTimeDiff(i); deletePose(i) */
          rec[4 * (i - 1) + 3] += rec[4 * i + 3];
          memmove(rec + 4 * i, rec + 4 * (i + 1), sizeof(double) * 4 * (size_t)(n - i - 1));
          n--;
        }
        modified = 1;
      }
    }
    if (fast_mode) break;
  }
  rec[4 * (n - 1) + 3] = 0.0;
  return n;
}

/* initTrajectoryToGoal(start, goal, diststep, max_vel_x, min_samples, guess_backwards) timed_elastic_band.cpp:325-387 */
int32_t teb_oracle_init_trajectory(const double* start, const double* goal, double diststep, double max_vel_x,
                                   int32_t min_samples, int32_t guess_backwards_motion, double* rec, int32_t n_cap) {
  int n = 0;
#define ADD_POSE(X, Y, T) do { if (n >= n_cap) return TEBGPU_ERR_CAPACITY; rec[4*n]=(X); rec[4*n+1]=(Y); rec[4*n+2]=(T); rec[4*n+3]=0; n++; } while (0)
#define ADD_POSE_DT(X, Y, T, D) do { rec[4*(n-1)+3]=(D); ADD_POSE(X, Y, T); } while (0)
  ADD_POSE(start[0], start[1], start[2]);
  double timestep = 0.1;
  if (diststep != 0) {
    double ptgx = goal[0] - start[0], ptgy = goal[1] - start[1];
    double dir_to_goal = atan2(ptgy, ptgx);
    double dx = diststep * cos(dir_to_goal), dy = diststep * sin(dir_to_goal);
    double orient_init = dir_to_goal;
    if (guess_backwards_motion && (ptgx * cos(start[2]) + ptgy * sin(start[2])) < 0) orient_init = nt(orient_init + M_PI);
    double dist_to_goal = sqrt(ptgx * ptgx + ptgy * ptgy);
    double no_steps_d = dist_to_goal / fabs(diststep);
    unsigned int no_steps = (unsigned int)floor(no_steps_d);
    if (max_vel_x > 0) timestep = diststep / max_vel_x;
    for (unsigned int i = 1; i <= no_steps; i++) {
      if (i == no_steps && no_steps_d == (float)no_steps) break;
      ADD_POSE_DT(start[0] + i * dx, start[1] + i * dy, orient_init, timestep);
    }
  }
  if (n < min_samples - 1) {
    while (n < min_samples - 1) {
      const double* back = rec + 4 * (n - 1);
      double ix = (back[0] + goal[0]) / 2, iy = (back[1] + goal[1]) / 2;
      double it = teb_oracle_average_angle(back[2], goal[2]);
      if (max_vel_x > 0) timestep = sqrt((ix - back[0]) * (ix - back[0]) + (iy - back[1]) * (iy - back[1])) / max_vel_x;
      ADD_POSE_DT(ix, iy, it, timestep);
    }
  }
  {
    const double* back = rec + 4 * (n - 1);
    if (max_vel_x > 0) timestep = sqrt((goal[0] - back[0]) * (goal[0] - back[0]) + (goal[1] - back[1]) * (goal[1] - back[1])) / max_vel_x;
    ADD_POSE_DT(goal[0], goal[1], goal[2], timestep);
  }
#undef ADD_POSE
#undef ADD_POSE_DT
  return n;
}

/* ------------------------------------------------------------------ optimizeTEB optimal_planner.cpp:182-231 */
static void graph_alloc(Graph* g, int n_cap) {
  int Ncap = 4 * n_cap;
  g->Hb = (double*)malloc(sizeof(double) * (size_t)Ncap * (HBW + 1));
  g->work = (double*)malloc(sizeof(double) * (size_t)Ncap * (HBW + 1));
  g->b = (double*)malloc(sizeof(double) * (size_t)Ncap);
  g->x = (double*)malloc(sizeof(double) * (size_t)Ncap);
  g->backup = (double*)malloc(sizeof(double) * 4 * (size_t)n_cap);
}
static void graph_free(Graph* g) {
  clear_graph(g);
  free(g->opv); free(g->opv_cnt);
  free(g->edges); free(g->Hb); free(g->work); free(g->b); free(g->x); free(g->backup); free(g->Hd);
}

int32_t teb_oracle_optimize(const TebParams* cfg, double* rec, int32_t* n_io, int32_t n_cap,
                            const TebObstacle* obst, int32_t M, const double* via, int32_t V,
                            const double* vel_start4, const double* vel_goal4, int32_t prefer_rotdir,
                            const TebOptimizeArgs* args, const OracleOptions* opt,
                            double* cost_out, OracleStats* stats, const double* obst_vertices) {
  OracleStats st;
  memset(&st, 0, sizeof(st));
  OracleOptions o = {ORACLE_JAC_G2O, ORACLE_SOLVER_BANDED, 0, 0};
  if (opt) o = *opt;
  int rc = 0;
  if (!cfg->optimization_activate) { st.status |= TEB_STATUS_DISABLED; goto done; }
  {
    Graph g;
    memset(&g, 0, sizeof(g));
    g.cfg = cfg; g.rec = rec; g.n = *n_io; g.obst = obst; g.M = M; g.via = via; g.V = V; g.pverts = obst_vertices;
    memcpy(g.vel_start, vel_start4, sizeof(double) * 4);
    memcpy(g.vel_goal, vel_goal4, sizeof(double) * 4);
    g.rotdir = prefer_rotdir;
    graph_alloc(&g, n_cap);
    double weight_multiplier = 1.0;
    int fast_mode = !cfg->include_dynamic_obstacles;
    int success = 1;
    for (int i = 0; i < args->iterations_outerloop; ++i) {
      if (cfg->teb_autosize) {
        int nn = teb_oracle_auto_resize(rec, g.n, n_cap, cfg->dt_ref, cfg->dt_hysteresis, cfg->min_samples,
                                        cfg->max_samples, fast_mode);
        if (nn < 0) { rc = nn; success = 0; break; }
        g.n = nn;
      }
      rc = build_graph(&g, weight_multiplier);
      if (rc) { success = 0; break; }
      /* optimizeGraph guards optimal_planner.cpp:370-382 */
      if (cfg->max_vel_x < 0.01) { st.status |= TEB_STATUS_DISABLED; success = 0; clear_graph(&g); break; }
      if (g.n < cfg->min_samples || g.n < 3) { st.status |= TEB_STATUS_TOO_FEW_POSES; success = 0; clear_graph(&g); break; }
      const int iters = optimize_graph_lm(&g, args->iterations_innerloop, &o, &st);
      st.lm_iters += iters;
      st.n_edges_last = g.n_edges;
      if (!iters) { success = 0; clear_graph(&g); break; } /* optimizeGraph: if (!iter) return false (:393) */
      if (args->compute_cost_afterwards && i == args->iterations_outerloop - 1 && cost_out)
        *cost_out = compute_current_cost(&g, args->obst_cost_scale, args->viapoint_cost_scale, args->alternative_time_cost);
      clear_graph(&g);
      weight_multiplier *= cfg->weight_adapt_factor;
    }
    if (success) st.status |= TEB_STATUS_OPTIMIZED; /* optimizeTEB returned true: also with no outer iteration */
    *n_io = g.n;
    graph_free(&g);
  }
done:
  st.n_final = *n_io;
  if (stats) *stats = st;
  return rc;
}


/* ------------------------------------------------------------------ H-signatures (h_signature.h) */
#include <complex.h>
typedef long double complex lcplx;

/* HSignature::calculateHSignature h_signature.h:97-186: 2-D homology signature, obstacle centroids as poles */
static void h_signature_2d(const TebParams* c, const double* rec, int n, const TebObstacle* obst, int M, double* out) {
  out[0] = out[1] = 0;
  if (M == 0 || n < 1) return;
  int m = M - 1 > 5 ? M - 1 : 5;
  int a = (int)ceil((double)m / 2.0);
  int b = m - a;
  lcplx start = (long double)rec[0] + I * (long double)rec[1];
  lcplx end = (long double)rec[4 * (n - 1)] + I * (long double)rec[4 * (n - 1) + 1];
  lcplx delta = end - start;
  lcplx normal = -cimagl(delta) + I * creall(delta);
  lcplx bl, tr;
  if (cabsl(delta) < 3.0) { bl = start + (0 - 3.0L * I); tr = start + (3.0L + 3.0L * I); }
  else { bl = start - normal; tr = start + delta + normal; }
  lcplx H = 0;
  for (int k = 0; k + 1 < n; ++k) {
    lcplx z1 = (long double)rec[4 * k] + I * (long double)rec[4 * k + 1];
    lcplx z2 = (long double)rec[4 * (k + 1)] + I * (long double)rec[4 * (k + 1) + 1];
    for (int l = 0; l < M; ++l) {
      lcplx ol = (long double)obst[l].x + I * (long double)obst[l].y;
      lcplx f0 = (long double)c->h_signature_prescaler * (long double)a * (ol - bl) * (long double)b * (ol - tr);
      lcplx Al = f0;
      for (int j = 0; j < M; ++j) {
        if (j == l) continue;
        lcplx oj = (long double)obst[j].x + I * (long double)obst[j].y;
        lcplx diff = ol - oj;
        if (cabsl(diff) < 0.05) continue;
        Al /= diff;
      }
      double diff2 = (double)cabsl(z2 - ol), diff1 = (double)cabsl(z1 - ol);
      if (diff2 == 0 || diff1 == 0) continue;
      double log_real = log(diff2) - log(diff1);
      double arg_diff = (double)(cargl(z2 - ol) - cargl(z1 - ol));
      double prop[5] = {arg_diff, arg_diff + 2 * M_PI, arg_diff - 2 * M_PI, arg_diff + 4 * M_PI, arg_diff - 4 * M_PI};
      double log_imag = prop[0];
      for (int q = 1; q < 5; ++q)
        if (fabs(prop[q]) < fabs(log_imag)) log_imag = prop[q]; /* std::min_element(..., smaller_than_abs) */
      lcplx lv = (long double)log_real + I * (long double)log_imag;
      H += Al * lv;
    }
  }
  out[0] = (double)creall(H);
  out[1] = (double)cimagl(H);
}

/* HSignature3d::calculateHSignature h_signature.h:282-353: x-y-t signature, one value per obstacle ("current" along the
 * obstacle's constant-velocity world line, Biot-Savart integral along the trajectory, 10 steps per segment) */
static void h_signature_3d(const TebParams* c, const double* rec, int n, const TebObstacle* obst, int M, int use_dt, double* out) {
  for (int l = 0; l < M; ++l) {
    double H = 0, transition_time = 0, next_transition_time = 0;
    const double t = 120;
    double s1[3] = {obst[l].x, obst[l].y, 0};
    double s2[3] = {obst[l].x + t * obst[l].vx, obst[l].y + t * obst[l].vy, t};
    double ds[3] = {s2[0] - s1[0], s2[1] - s1[1], s2[2] - s1[2]};
    double ds2 = ds[0] * ds[0] + ds[1] * ds[1] + ds[2] * ds[2];
    for (int k = 0; k + 1 < n; ++k) {
      const double* z1 = rec + 4 * k;
      const double* z2 = rec + 4 * (k + 1);
      transition_time = next_transition_time;
      if (!use_dt) next_transition_time += cabsl(((long double)z2[0] - z1[0]) + I * ((long double)z2[1] - z1[1])) / c->max_vel_x;
      else next_transition_time += z1[3];
      double dir[3] = {z2[0] - z1[0], z2[1] - z1[1], next_transition_time - transition_time};
      if (sqrt(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]) < 1e-15) continue;
      double r[3] = {z1[0], z1[1], transition_time};
      double dl[3] = {0.1 * dir[0], 0.1 * dir[1], 0.1 * dir[2]}; /* 1.0 / num_int_steps_per_segment * direction_vec */
      for (int i = 0; i < 10; ++i) {
        double p1[3] = {s1[0] - r[0], s1[1] - r[1], s1[2] - r[2]};
        double p2[3] = {s2[0] - r[0], s2[1] - r[1], s2[2] - r[2]};
        double cr[3] = {p1[1] * p2[2] - p1[2] * p2[1], p1[2] * p2[0] - p1[0] * p2[2], p1[0] * p2[1] - p1[1] * p2[0]};
        double d[3] = {(ds[1] * cr[2] - ds[2] * cr[1]) / ds2, (ds[2] * cr[0] - ds[0] * cr[2]) / ds2, (ds[0] * cr[1] - ds[1] * cr[0]) / ds2};
        double n1 = sqrt(p1[0] * p1[0] + p1[1] * p1[1] + p1[2] * p1[2]), n2 = sqrt(p2[0] * p2[0] + p2[1] * p2[1] + p2[2] * p2[2]);
        double dxp2[3] = {d[1] * p2[2] - d[2] * p2[1], d[2] * p2[0] - d[0] * p2[2], d[0] * p2[1] - d[1] * p2[0]};
        double dxp1[3] = {d[1] * p1[2] - d[2] * p1[1], d[2] * p1[0] - d[0] * p1[2], d[0] * p1[1] - d[1] * p1[0]};
        double inv = 1.0 / (d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        double phi[3];
        for (int q = 0; q < 3; ++q) phi[q] = inv * (dxp2[q] / n2 - dxp1[q] / n1);
        H += phi[0] * dl[0] + phi[1] * dl[1] + phi[2] * dl[2];
        for (int q = 0; q < 3; ++q) r[q] += dl[q];
      }
    }
    out[l] = H / (4.0 * M_PI);
  }
}

int32_t teb_oracle_h_signature(const TebParams* cfg, const double* rec, int32_t n, const TebObstacle* obst, int32_t M,
                               int32_t use_timediffs, double* out) {
  if (!cfg || !rec || !out || n < 1) return -1;
  if (cfg->include_dynamic_obstacles) h_signature_3d(cfg, rec, n, obst, M, use_timediffs, out);
  else h_signature_2d(cfg, rec, n, obst, M, out);
  return 0;
}

double teb_oracle_distance(const TebParams* cfg, const double* pose3, const TebObstacle* obst, const double* obst_vertices,
                           double t, double* grad3) {
  if (!generic_pair(cfg, obst)) {
    double d;
    if (grad3) footprint_grad(cfg, pose3, obst->x + t * obst->vx, obst->y + t * obst->vy, obst->radius, &d, grad3);
    return t == 0 ? footprint_dist(cfg, pose3, obst, obst_vertices) : footprint_dist_t(cfg, pose3, obst, obst_vertices, t);
  }
  return generic_distance(cfg, pose3, obst, obst_vertices, t, grad3);
}

int32_t teb_oracle_build_system(const TebParams* cfg, const double* rec_in, int32_t n,
                                const TebObstacle* obst, int32_t M, const double* via, int32_t V,
                                const double* vel_start4, const double* vel_goal4, int32_t prefer_rotdir,
                                double weight_multiplier, int32_t jac_mode,
                                double* H_dense, double* b, double* chi2, const double* obst_vertices) {
  Graph g;
  memset(&g, 0, sizeof(g));
  double* rec = (double*)malloc(sizeof(double) * 4 * (size_t)n);
  memcpy(rec, rec_in, sizeof(double) * 4 * (size_t)n);
  g.cfg = cfg; g.rec = rec; g.n = n; g.obst = obst; g.M = M; g.via = via; g.V = V; g.pverts = obst_vertices;
  memcpy(g.vel_start, vel_start4, sizeof(double) * 4);
  memcpy(g.vel_goal, vel_goal4, sizeof(double) * 4);
  g.rotdir = prefer_rotdir;
  graph_alloc(&g, n);
  int rc = build_graph(&g, weight_multiplier);
  if (rc) { graph_free(&g); free(rec); return rc; }
  double c2 = compute_active_errors(&g);
  build_system(&g, jac_mode);
  int N = g.N;
  if (H_dense) {
    memset(H_dense, 0, sizeof(double) * (size_t)N * N);
    for (int r = 0; r < N; ++r)
      for (int k = 0; k <= HBW && k <= r; ++k) {
        double v = g.Hb[(size_t)r * (HBW + 1) + k];
        H_dense[(size_t)r * N + (r - k)] = v;
        H_dense[(size_t)(r - k) * N + r] = v;
      }
  }
  if (b) memcpy(b, g.b, sizeof(double) * (size_t)N);
  if (chi2) *chi2 = c2;
  graph_free(&g);
  free(rec);
  return N;
}

int32_t teb_oracle_trial_chi2(const TebParams* cfg, const double* rec_graph, int32_t n, const TebObstacle* obst, int32_t M,
                              const double* via, int32_t V, const double* vel_start4, const double* vel_goal4,
                              int32_t prefer_rotdir, double weight_multiplier, const double* rec_trials, int32_t T,
                              double* chi_out, const double* obst_vertices) {
  if (!cfg || !rec_graph || !chi_out || n < 3 || T < 0 || (T > 0 && !rec_trials)) return -1;
  Graph g;
  memset(&g, 0, sizeof(g));
  double* rec = (double*)malloc(sizeof(double) * 4 * (size_t)n);
  memcpy(rec, rec_graph, sizeof(double) * 4 * (size_t)n);
  g.cfg = cfg; g.rec = rec; g.n = n; g.obst = obst; g.M = M; g.via = via; g.V = V; g.pverts = obst_vertices;
  memcpy(g.vel_start, vel_start4, sizeof(double) * 4);
  memcpy(g.vel_goal, vel_goal4, sizeof(double) * 4);
  g.rotdir = prefer_rotdir;
  graph_alloc(&g, n);
  int rc = build_graph(&g, weight_multiplier);
  if (rc) { graph_free(&g); free(rec); return rc; }
  for (int t = 0; t < T; ++t) {
    memcpy(rec, rec_trials + (size_t)t * 4 * n, sizeof(double) * 4 * (size_t)n);
    long double fam[4] = {0, 0, 0, 0};
    for (int k = 0; k < g.n_edges; ++k) {
      Edge* e = g.edges[k];
      e->compute_error(e, &g);
      /* compute_current_cost's classification; the velocity-obstacle-ratio edge is one of the others */
      const int f = (e->type == E_OBST || e->type == E_INFL || e->type == E_DYN) ? 0
                    : e->type == E_VIA                                         ? 1
                    : e->type == E_TIMEOPT                                     ? 2
                                                                               : 3;
      for (int d = 0; d < e->dim; ++d) fam[f] += (long double)e->err[d] * e->info[d] * e->err[d];
    }
    for (int f = 0; f < 4; ++f) chi_out[4 * (size_t)t + f] = (double)fam[f];
  }
  graph_free(&g);
  free(rec);
  return 0;
}

int32_t teb_oracle_graph(const TebParams* cfg, const double* rec_in, int32_t n, const TebObstacle* obst, int32_t M,
                         const double* via, int32_t V, const double* vel_start4, const double* vel_goal4,
                         int32_t prefer_rotdir, double weight_multiplier, int32_t MW, uint64_t* assoc_out,
                         uint64_t* assoc3_out, int32_t* via_idx_out, double* dyn_t_out, const double* obst_vertices) {
  if (!cfg || !rec_in || n < 3 || M < 0 || MW < (M + 63) / 64 || MW < 1) return -1;
  Graph g;
  memset(&g, 0, sizeof(g));
  double* rec = (double*)malloc(sizeof(double) * 4 * (size_t)n);
  memcpy(rec, rec_in, sizeof(double) * 4 * (size_t)n);
  g.cfg = cfg; g.rec = rec; g.n = n; g.obst = obst; g.M = M; g.via = via; g.V = V; g.pverts = obst_vertices;
  memcpy(g.vel_start, vel_start4, sizeof(double) * 4);
  memcpy(g.vel_goal, vel_goal4, sizeof(double) * 4);
  g.rotdir = prefer_rotdir;
  graph_alloc(&g, n);
  int rc = build_graph(&g, weight_multiplier);
  if (rc) { graph_free(&g); free(rec); return rc; }
  /* obstacle / inflated edges per (pose, obstacle): 1, or 3 on the legacy centre pose */
  int* cnt = (int*)calloc((size_t)n * (M > 0 ? M : 1), sizeof(int));
  if (assoc_out) memset(assoc_out, 0, sizeof(uint64_t) * (size_t)n * MW);
  if (assoc3_out) memset(assoc3_out, 0, sizeof(uint64_t) * (size_t)n * MW);
  if (via_idx_out)
    for (int v = 0; v < V; ++v) via_idx_out[v] = -1;
  if (dyn_t_out)
    for (int i = 0; i < n; ++i) dyn_t_out[i] = NAN;
  for (int k = 0; k < g.n_edges; ++k) {
    const Edge* e = g.edges[k];
    const int i = e->vidx[0];
    if (e->type == E_OBST || e->type == E_INFL || e->type == E_VEL_OBST_RATIO) {
      const int m = (int)(e->ob - obst);
      if (assoc_out) assoc_out[(size_t)i * MW + (m >> 6)] |= 1ull << (m & 63);
      if (e->type != E_VEL_OBST_RATIO) ++cnt[(size_t)i * M + m];
    } else if (e->type == E_VIA) {
      if (via_idx_out) via_idx_out[(e->via - via) / 2] = i;
    } else if (e->type == E_DYN) {
      if (dyn_t_out) dyn_t_out[i] = e->t;
    }
  }
  if (assoc3_out)
    for (int i = 0; i < n; ++i)
      for (int m = 0; m < M; ++m)
        if (cnt[(size_t)i * M + m] == 3) assoc3_out[(size_t)i * MW + (m >> 6)] |= 1ull << (m & 63);
  free(cnt);
  graph_free(&g);
  free(rec);
  return 0;
}

/* Per-edge dump of the graph buildGraph() produces at the given state, in insertion order, after computeActiveErrors
 * and linearisation: rows of 64 doubles, same layout as oracle/ref_driver.cpp's teb_ref_build_system(edges_out):
 * [0] error dimension, [1] vertex count, [2..4] error, [5..7] information diagonal, [8 + 9 k ...] Jacobian of vertex k
 * (row major dim x vdim, zero for fixed vertices), [53 + k] vertex dimension, [58 + k] g2o vertex id (pose i: 2 i,
 * dt_i: 2 i + 1, optimal_planner.cpp:426-437). Returns the number of active edges (or <0). */
int32_t teb_oracle_dump_edges(const TebParams* cfg, const double* rec_in, int32_t n, const TebObstacle* obst, int32_t M,
                              const double* via, int32_t V, const double* vel_start4, const double* vel_goal4,
                              int32_t prefer_rotdir, double weight_multiplier, int32_t jac_mode, double* rows,
                              int32_t max_rows, const double* obst_vertices) {
  Graph g;
  memset(&g, 0, sizeof(g));
  double* rec = (double*)malloc(sizeof(double) * 4 * (size_t)n);
  memcpy(rec, rec_in, sizeof(double) * 4 * (size_t)n);
  g.cfg = cfg; g.rec = rec; g.n = n; g.obst = obst; g.M = M; g.via = via; g.V = V; g.pverts = obst_vertices;
  memcpy(g.vel_start, vel_start4, sizeof(double) * 4);
  memcpy(g.vel_goal, vel_goal4, sizeof(double) * 4);
  g.rotdir = prefer_rotdir;
  graph_alloc(&g, n);
  int rc = build_graph(&g, weight_multiplier);
  if (rc) { graph_free(&g); free(rec); return rc; }
  compute_active_errors(&g);
  for (int k = 0; k < g.n_edges; ++k) {
    Edge* e = g.edges[k];
    memset(e->J, 0, sizeof(e->J));
    linearize(e, &g, jac_mode);
    if (k >= max_rows) continue;
    double* row = rows + 64 * (size_t)k;
    memset(row, 0, 64 * sizeof(double));
    row[0] = e->dim; row[1] = e->nv;
    for (int d = 0; d < e->dim; ++d) { row[2 + d] = e->err[d]; row[5 + d] = e->info[d]; }
    for (int v = 0; v < e->nv && v < 5; ++v) {
      const int vd = vdim(e->vkind[v]);
      row[53 + v] = vd;
      row[58 + v] = 2 * e->vidx[v] + (e->vkind[v] == 1 ? 1 : 0);
      if (edge_vertex_fixed(&g, e, v)) continue;
      for (int d = 0; d < e->dim; ++d)
        for (int a = 0; a < vd; ++a) row[8 + 9 * v + d * vd + a] = e->J[v][d * vd + a];
    }
  }
  const int ne = g.n_edges;
  graph_free(&g);
  free(rec);
  return ne;
}

/* ------------------------------------------------------------------ batch driver (thread per band) */
typedef struct BatchJob {
  const TebParams* cfg; const TebBatch* batch; const TebOptimizeArgs* args; const OracleOptions* opt;
  int next; pthread_mutex_t mu; int rc;
} BatchJob;
typedef struct BatchThread { BatchJob* job; int index; } BatchThread;

/* pin the calling worker to the index-th CPU of the process affinity mask (round robin) */
static void pin_worker(int index) {
  cpu_set_t allowed;
  CPU_ZERO(&allowed);
  if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return;
  const int cnt = CPU_COUNT(&allowed);
  if (cnt <= 0) return;
  int want = index % cnt, seen = 0;
  for (int c = 0; c < CPU_SETSIZE; ++c) {
    if (!CPU_ISSET(c, &allowed)) continue;
    if (seen++ == want) {
      cpu_set_t one;
      CPU_ZERO(&one);
      CPU_SET(c, &one);
      pthread_setaffinity_np(pthread_self(), sizeof(one), &one);
      return;
    }
  }
}

static void* batch_worker(void* p) {
  BatchThread* me = (BatchThread*)p;
  BatchJob* job = me->job;
  if (job->opt && job->opt->pin_threads && me->index >= 0) pin_worker(me->index);
  const TebBatch* bt = job->batch;
  for (;;) {
    pthread_mutex_lock(&job->mu);
    int bidx = job->next++;
    pthread_mutex_unlock(&job->mu);
    if (bidx >= bt->B) break;
    int s = bt->scene_id ? bt->scene_id[bidx] : 0;
    const double zero4[4] = {0, 0, 0, 1};
    double cost = HUGE_VAL;
    OracleStats st;
    int nb = bt->n[bidx];
    int rc = teb_oracle_optimize(job->cfg, bt->poses + (size_t)bidx * bt->n_cap * 4, &nb, bt->n_cap,
                                 bt->obstacles + (size_t)s * bt->M_cap, bt->obst_count ? bt->obst_count[s] : 0,
                                 bt->via ? bt->via + (size_t)bidx * bt->V_cap * 2 : NULL,
                                 bt->via_count ? bt->via_count[bidx] : 0,
                                 bt->vel_start ? bt->vel_start + 4 * bidx : zero4,
                                 bt->vel_goal ? bt->vel_goal + 4 * bidx : zero4,
                                 bt->prefer_rotdir ? bt->prefer_rotdir[bidx] : 0, job->args, job->opt, &cost, &st,
                                 (bt->obst_vertices && bt->PV_cap > 0) ? bt->obst_vertices + (size_t)s * bt->PV_cap * 2 : NULL);
    bt->n[bidx] = nb;
    if (bt->cost) bt->cost[bidx] = cost;
    if (bt->chi2) bt->chi2[bidx] = st.chi2_final;
    if (bt->status) bt->status[bidx] = st.status;
    if (bt->lm_iters) bt->lm_iters[bidx] = st.lm_iters;
    if (rc) job->rc = rc;
  }
  return NULL;
}

int32_t teb_oracle_optimize_batch(const TebParams* cfg, const TebBatch* batch, const TebOptimizeArgs* args,
                                  const OracleOptions* opt, int32_t threads) {
  BatchJob job;
  job.cfg = cfg; job.batch = batch; job.args = args; job.opt = opt; job.next = 0; job.rc = 0;
  pthread_mutex_init(&job.mu, NULL);
  if (threads < 1) threads = 1;
  if (threads > batch->B) threads = batch->B;
  if (threads == 1) {
    BatchThread me = {&job, -1}; /* the caller's thread: never re-pinned */
    batch_worker(&me);
  } else {
    pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * threads);
    BatchThread* arg = (BatchThread*)malloc(sizeof(BatchThread) * threads);
    for (int t = 0; t < threads; ++t) { arg[t].job = &job; arg[t].index = t; pthread_create(&th[t], NULL, batch_worker, &arg[t]); }
    for (int t = 0; t < threads; ++t) pthread_join(th[t], NULL);
    free(arg);
    free(th);
  }
  pthread_mutex_destroy(&job.mu);
  return job.rc;
}
