"""Footprint-to-obstacle distance cases at the edges of BaseRobotFootprintModel::calculateDistance /
estimateSpatioTemporalDistance (robot_footprint_model.h) over the vertex-list routines of distance_calculations.h, shared
by tests/test_reference_pin_distance.py (the oracle against the reference's own code) and tests/test_gpu_distance.py
(graph build, kernel A, k_vor and the trial evaluation against the oracle). Plain numpy; every builder asserts on the
host, in exact rational arithmetic, the property its case claims.

Construction. Headings are 0, so cos / sin are exactly 1 / 0 on every side. Coordinates, offsets, radii, velocities and
times are small multiples of 2^-6, and every segment whose closest point is searched at the case pose has a squared
length that makes u = (p - a).d / |d|^2 an exact binary fraction (asserted for the case pose): every closest point,
difference and squared distance is then exact in fp64, so a distance is the correctly rounded square root of an exact
number on every side and FMA contraction on the device cannot decide a comparison differently from the uncontracted
oracle. The large polygons (65 and 70 vertices on a circle, rounded to the grid) are the exception: they claim only
which edge is nearest, by a margin far above rounding.

Each case is one obstacle (its own scene and vertex pool) and one pose. The GPU and graph tests put the pose at index
K_CASE of a straight heading-0 band of N_BAND poses DX apart with time differences DT, so that the case pose sits at the
time T_CASE a moving obstacle is built for.
"""
import math
from fractions import Fraction as F

import numpy as np

from teb_local_planner_b200 import abi, scenes

N_BAND, K_CASE, DX, DT = 9, 4, 0.25, 0.25
T_CASE = K_CASE * DT                        # 1.0: time of the case pose in its band
MIN_D, EPS, INFL, DYN_INFL = 0.5, 0.125, 0.75, 0.875
FORCE_D, CUT_D = 1.0, 2.0                   # MIN_D * 2, MIN_D * 4 (association)

# footprint name -> (type, definition)
FOOTPRINTS = {
    "point": (abi.TEB_FOOTPRINT_POINT, None),
    "circular": (abi.TEB_FOOTPRINT_CIRCULAR, 0.25),
    "two_circles": (abi.TEB_FOOTPRINT_TWO_CIRCLES, (0.5, 0.25, 0.5, 0.25)),        # front off, rad, rear off, rad
    "two_circles_uneq": (abi.TEB_FOOTPRINT_TWO_CIRCLES, (0.5, 0.25, 0.25, 0.125)),
    "line": (abi.TEB_FOOTPRINT_LINE, ((-0.25, 0.0), (0.75, 0.0))),
    "line_zero": (abi.TEB_FOOTPRINT_LINE, ((0.25, 0.0), (0.25, 0.0))),
    "polygon1": (abi.TEB_FOOTPRINT_POLYGON, ((0.25, 0.0),)),
    "polygon2": (abi.TEB_FOOTPRINT_POLYGON, ((-0.25, 0.0), (0.75, 0.0))),
    "polygon3": (abi.TEB_FOOTPRINT_POLYGON, ((-0.25, -0.25), (0.25, -0.25), (0.25, 0.25))),
    "polygon4": (abi.TEB_FOOTPRINT_POLYGON, ((-0.25, -0.25), (0.75, -0.25), (0.75, 0.25), (-0.25, 0.25))),
    # the unit square around the pose, 4 vertices per side (collinear neighbours, 16 edges of length 0.25)
    "polygon16": (abi.TEB_FOOTPRINT_POLYGON, tuple([(-0.5 + 0.25 * k, -0.5) for k in range(4)] +
                                                   [(0.5, -0.5 + 0.25 * k) for k in range(4)] +
                                                   [(0.5 - 0.25 * k, 0.5) for k in range(4)] +
                                                   [(-0.5, 0.5 - 0.25 * k) for k in range(4)])),
}
RIGHT_EXTENT = {"point": 0.0, "circular": 0.25, "two_circles": 0.75, "two_circles_uneq": 0.75, "line": 0.75,
                "line_zero": 0.25, "polygon1": 0.25, "polygon2": 0.75, "polygon3": 0.25, "polygon4": 0.75,
                "polygon16": 0.5}   # largest x of the footprint at pose (0, 0, 0), reached on y = 0


def params(fp, **kw):
    """the thresholds of every case: min_obstacle_dist 0.5, penalty_epsilon 0.125, inflation 0.75, dynamic inflation
    0.875, association force / cutoff distances 1 / 2"""
    p = abi.default_params()
    p.min_obstacle_dist, p.penalty_epsilon, p.inflation_dist, p.dynamic_obstacle_inflation_dist = MIN_D, EPS, INFL, DYN_INFL
    p.obstacle_association_force_inclusion_factor, p.obstacle_association_cutoff_factor = 2.0, 4.0
    p.include_dynamic_obstacles = 0
    kind, dfn = FOOTPRINTS[fp]
    p.footprint_type = kind
    if kind == abi.TEB_FOOTPRINT_CIRCULAR:
        p.footprint_radius = dfn
    elif kind == abi.TEB_FOOTPRINT_TWO_CIRCLES:
        p.footprint_front_offset, p.footprint_front_radius, p.footprint_rear_offset, p.footprint_rear_radius = dfn
    elif kind == abi.TEB_FOOTPRINT_LINE:
        scenes.set_line_footprint(p, dfn[0], dfn[1])
    elif kind == abi.TEB_FOOTPRINT_POLYGON:
        scenes.set_polygon_footprint(p, dfn)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


class Case:
    """fp: footprint name; obst: one OBST_DTYPE row (vertex_begin 0 in its own pool); verts: [k][2] pool or None;
    pose: (x, y), heading 0; t: None (static) or the time of estimateSpatioTemporalDistance (T_CASE);
    d: the exact distance where the case claims one (Fraction), else None; smooth: the distance is differentiable at
    the pose (the closed-form gradient is compared with a central difference there)"""

    def __init__(self, name, fp, obst, verts, pose, t=None, d=None, smooth=True):
        self.name, self.fp, self.obst, self.verts = name, fp, obst, verts
        self.pose, self.t, self.d, self.smooth = (float(pose[0]), float(pose[1])), t, d, smooth

    def params(self, **kw):
        return params(self.fp, **kw)

    def pose3(self):
        return np.array([self.pose[0], self.pose[1], 0.0])

    def band(self):
        """N_BAND heading-0 poses DX apart along x, the case pose at index K_CASE, dt DT"""
        rec = np.zeros((N_BAND, 4))
        rec[:, 0] = self.pose[0] + DX * (np.arange(N_BAND) - K_CASE)
        rec[:, 1] = self.pose[1]
        rec[:-1, 3] = DT
        return rec

    def __repr__(self):
        return f"Case({self.name})"


# ------------------------------------------------------------------------------------------------ obstacle rows
def _row(kind, x, y, radius=0.0, v=(0.0, 0.0), count=0):
    ob = np.zeros(1, abi.OBST_DTYPE)
    ob["type"], ob["x"], ob["y"], ob["radius"] = kind, x, y, radius
    ob["vx"], ob["vy"] = v
    ob["dynamic"] = int(v[0] != 0 or v[1] != 0)
    ob["vertex_begin"], ob["vertex_count"] = 0, count
    return ob


def point(x, y, v=(0.0, 0.0)):
    return _row(abi.TEB_OBST_POINT, x, y, v=v), None


def circle(x, y, r, v=(0.0, 0.0)):
    return _row(abi.TEB_OBST_CIRCULAR, x, y, r, v=v), None


def line(a, b, v=(0.0, 0.0)):
    return _row(abi.TEB_OBST_LINE, 0.5 * (a[0] + b[0]), 0.5 * (a[1] + b[1]), v=v, count=2), np.array([a, b], float)


def pill(a, b, r, v=(0.0, 0.0)):
    return _row(abi.TEB_OBST_PILL, 0.5 * (a[0] + b[0]), 0.5 * (a[1] + b[1]), r, v=v, count=2), np.array([a, b], float)


def polygon(vs, v=(0.0, 0.0)):
    vs = np.array(vs, float).reshape(-1, 2)
    c = scenes.polygon_centroid(vs)                     # getCentroid(): only the association's left / right test reads it
    return _row(abi.TEB_OBST_POLYGON, c[0], c[1], v=v, count=len(vs)), vs


# ------------------------------------------------------------------------------------------------ exact geometry
class Trace:
    """what the vertex-list enumeration met at one pose, in rationals: every u of closest_point_on_line_segment_2d,
    every intersection test (denom, accepted), the squared distance of every robot-edge x obstacle-edge pair of each
    footprint part, the part's radius sum"""

    def __init__(self):
        self.us, self.tests, self.parts = [], [], []


def _closest(tr, p, a, b):
    dx, dy = b[0] - a[0], b[1] - a[1]
    sq = dx * dx + dy * dy
    if sq == 0:
        return a
    u = ((p[0] - a[0]) * dx + (p[1] - a[1]) * dy) / sq
    tr.us.append(u)
    if u <= 0:
        return a
    if u >= 1:
        return b
    return (a[0] + u * dx, a[1] + u * dy)


def _d2(p, q):
    return (p[0] - q[0]) ** 2 + (p[1] - q[1]) ** 2


def _intersect(tr, l1s, l1e, l2s, l2e):
    """check_line_segments_intersection_2d, decision for decision"""
    l1 = (l1e[0] - l1s[0], l1e[1] - l1s[1])
    l2 = (l2e[0] - l2s[0], l2e[1] - l2s[1])
    denom = l1[0] * l2[1] - l2[0] * l1[1]
    hit = False
    if denom != 0:
        pos = denom > 0
        ax, ay = l1s[0] - l2s[0], l1s[1] - l2s[1]
        s = l1[0] * ay - l1[1] * ax
        t = l2[0] * ay - l2[1] * ax
        hit = not ((s < 0) == pos or (t < 0) == pos or (s > denom) == pos or (t > denom) == pos)
    tr.tests.append((denom, hit))
    return hit


def _seg_seg(tr, l1s, l1e, l2s, l2e):
    if _intersect(tr, l1s, l1e, l2s, l2e):
        return F(0)
    return min(_d2(l1s, _closest(tr, l1s, l2s, l2e)), _d2(l1e, _closest(tr, l1e, l2s, l2e)),
               _d2(l2s, _closest(tr, l2s, l1s, l1e)), _d2(l2e, _closest(tr, l2e, l1s, l1e)))


def _edges(vs):
    k = len(vs)
    return [(vs[i], vs[(i + 1) % k]) for i in range(1 if k <= 2 else k)]


def _pairs(tr, rv, ov, obst_first):
    out = []
    for r0, r1 in _edges(rv):
        for o0, o1 in _edges(ov):
            if len(rv) == 1 and len(ov) == 1:
                out.append(_d2(r0, o0))
            elif len(rv) == 1:
                out.append(_d2(r0, _closest(tr, r0, o0, o1)))
            elif len(ov) == 1:
                out.append(_d2(o0, _closest(tr, o0, r0, r1)))
            elif obst_first:
                out.append(_seg_seg(tr, o0, o1, r0, r1))
            else:
                out.append(_seg_seg(tr, r0, r1, o0, o1))
    return out


def robot_parts(fp, pose):
    """[(vertex list, radius)] of the footprint at (x, y, 0): one part, two for TwoCircles (front, rear)"""
    kind, dfn = FOOTPRINTS[fp]
    x, y = F(pose[0]), F(pose[1])
    if kind == abi.TEB_FOOTPRINT_POINT:
        return [([(x, y)], F(0))]
    if kind == abi.TEB_FOOTPRINT_CIRCULAR:
        return [([(x, y)], F(dfn))]
    if kind == abi.TEB_FOOTPRINT_TWO_CIRCLES:
        fo, fr, ro, rr = (F(v) for v in dfn)
        return [([(x + fo, y)], fr), ([(x - ro, y)], rr)]
    return [([(x + F(a), y + F(b)) for a, b in dfn], F(0))]


def obstacle_shape(row, verts, t):
    """(vertex list at time t, radius, obstacle segment first)"""
    kind = int(row["type"][0])
    off = (F(0), F(0)) if t is None else (F(t) * F(float(row["vx"][0])), F(t) * F(float(row["vy"][0])))
    if kind >= abi.TEB_OBST_LINE:
        vs = [(F(float(a)) + off[0], F(float(b)) + off[1]) for a, b in verts]
    else:
        vs = [(F(float(row["x"][0])) + off[0], F(float(row["y"][0])) + off[1])]
    rad = F(float(row["radius"][0])) if kind in (abi.TEB_OBST_CIRCULAR, abi.TEB_OBST_PILL) else F(0)
    return vs, rad, kind in (abi.TEB_OBST_LINE, abi.TEB_OBST_PILL)


def trace(fp, row, verts, pose, t=None, limit=None):
    """the enumeration at pose; limit: read only the first `limit` obstacle vertices"""
    tr = Trace()
    ov, orad, first = obstacle_shape(row, verts, t)
    if limit is not None:
        ov = ov[:limit]
    for rv, rrad in robot_parts(fp, pose):
        tr.parts.append((_pairs(tr, rv, ov, first), orad + rrad))
    return tr


def _sqrt(q):
    """the exact square root of a non-negative rational, or None"""
    a, b = math.isqrt(q.numerator), math.isqrt(q.denominator)
    return F(a, b) if a * a == q.numerator and b * b == q.denominator else None


def part_min(tr, k):
    pairs, rad = tr.parts[k]
    return min(pairs), rad


def exact_distance(tr):
    """min over the parts of sqrt(min pair d2) - radii, where every part's square root is rational; else None"""
    ds = []
    for k in range(len(tr.parts)):
        q, rad = part_min(tr, k)
        r = _sqrt(q)
        if r is None:
            return None
        ds.append(r - rad)
    return min(ds)


def _dyadic(q):
    return q.denominator & (q.denominator - 1) == 0 and q.denominator <= 2 ** 30


def check_exact_inputs(case):
    """the construction rule at the case pose: grid inputs and exact binary u everywhere"""
    for v in (case.pose[0], case.pose[1]) + ((case.t,) if case.t is not None else ()):
        assert _dyadic(F(v)), (case.name, v)
    tr = trace(case.fp, case.obst, case.verts, case.pose, case.t)
    if case.verts is None or len(case.verts) <= 16:
        assert all(_dyadic(u) for u in tr.us), (case.name, [u for u in tr.us if not _dyadic(u)])
    return tr


# ------------------------------------------------------------------------------------------------ the cases
def _case(name, fp, ob, pose, t=None, d=None, smooth=True, claim=None):
    row, verts = ob
    c = Case(name, fp, row, verts, pose, t, d, smooth)
    tr = check_exact_inputs(c)
    if d is not None:
        assert exact_distance(tr) == d, (name, exact_distance(tr), d)
    if claim is not None:
        assert claim(tr), name
    return c


def _ties(tr, k=0):
    """number of robot x obstacle pairs of part k at the part's minimum"""
    pairs, _ = tr.parts[k]
    return sum(1 for q in pairs if q == min(pairs))


def _obstacle_at(kind, X, v=(0.0, 0.0)):
    """obstacle of `kind` whose leftmost points lie at x = X on y = 0 (and, for segments, above and below it)"""
    r = 0.25
    if kind == "point":
        return point(X, 0.0, v)
    if kind == "circular":
        return circle(X + r, 0.0, r, v)
    if kind == "line":
        return line((X, -0.5), (X, 0.5), v)
    if kind == "pill":
        return pill((X + r, -0.5), (X + r, 0.5), r, v)
    if kind == "polygon1":
        return polygon([(X, 0.0)], v)
    if kind == "polygon2":
        return polygon([(X, 0.0), (X + 1.0, 0.0)], v)
    if kind == "polygon3":
        return polygon([(X, 0.0), (X + 0.5, -0.5), (X + 0.5, 0.5)], v)
    if kind == "polygon4":
        return polygon([(X, -0.5), (X + 1.0, -0.5), (X + 1.0, 0.5), (X, 0.5)], v)
    raise KeyError(kind)


GRID_OBSTACLES = ["point", "circular", "line", "pill", "polygon1", "polygon2", "polygon3", "polygon4"]
FLAT_RIGHT = ("polygon3", "polygon4", "polygon16")     # footprints whose right side is a vertical edge
FLAT_LEFT = ("line", "pill", "polygon4")               # obstacles whose left side is a vertical edge (parallel: a kink)


def grid_cases():
    """every footprint x every obstacle kind, right of the robot: touching (distance 0: vertex on edge, collinear
    edges, endpoint on edge) and at exactly min_obstacle_dist + penalty_epsilon; the moving shapes reach both only at
    T_CASE"""
    out = []
    for fp in FOOTPRINTS:
        for kind in GRID_OBSTACLES:
            for what, gap in (("contact", 0.0), ("at_min_eps", MIN_D + EPS)):
                X = RIGHT_EXTENT[fp] + gap
                out.append(_case(f"grid_{fp}_{kind}_{what}", fp, _obstacle_at(kind, X), (0.0, 0.0), d=F(gap),
                                 smooth=gap > 0 and (fp not in FLAT_RIGHT or kind not in FLAT_LEFT)))
            if kind in ("line", "pill", "polygon3", "polygon4") and fp in ("point", "two_circles", "line", "polygon4"):
                X = RIGHT_EXTENT[fp]
                out.append(_case(f"grid_{fp}_{kind}_moving_contact", fp, _obstacle_at(kind, X + 0.5, v=(-0.5, 0.0)),
                                 (0.0, 0.0), t=T_CASE, d=F(0), smooth=False))
    return out


def contact_cases():
    out = []
    # crossing edges: line footprint x line obstacle, rectangle x triangle
    out.append(_case("cross_line_line", "line", line((0.25, -0.5), (0.25, 0.5)), (0.0, 0.0), d=F(0), smooth=False,
                     claim=lambda tr: any(h for _, h in tr.tests)))
    out.append(_case("cross_polygon4_polygon3", "polygon4", polygon([(0.5, 0.0), (1.0, -0.5), (1.0, 0.5)]), (0.0, 0.0),
                     d=F(0), smooth=False, claim=lambda tr: any(h for _, h in tr.tests)))
    # an endpoint of the obstacle segment on the robot's edge: the intersection test accepts it for denom > 0 only
    for nm, a, b, sign in (("pos", (0.25, 0.5), (0.25, 0.0), 1), ("neg", (0.25, 0.0), (0.25, 0.5), -1)):
        def claim(tr, sign=sign):
            den, hit = tr.tests[0]
            return den * sign > 0 and hit == (sign > 0)
        out.append(_case(f"touch_endpoint_denom_{nm}", "line", line(a, b), (0.0, 0.0), d=F(0), smooth=False, claim=claim))
        out.append(_case(f"touch_endpoint_denom_{nm}_pill", "polygon2", pill(a, b, 0.125), (0.0, 0.0), d=F(-1, 8),
                         smooth=False, claim=claim))
    # a vertex of a diamond on the rectangle's top edge; a vertex of the robot on the obstacle's edge
    out.append(_case("vertex_on_edge_obstacle", "polygon4", polygon([(0.25, 0.25), (0.5, 0.5), (0.25, 0.75), (0.0, 0.5)]),
                     (0.0, 0.0), d=F(0), smooth=False))
    out.append(_case("vertex_on_edge_robot", "polygon3", line((0.25, 0.25), (1.25, 0.25)), (0.0, 0.0), d=F(0), smooth=False))
    # collinear overlap (denom = 0)
    out.append(_case("collinear_overlap_line", "line", line((0.25, 0.0), (1.25, 0.0)), (0.0, 0.0), d=F(0), smooth=False,
                     claim=lambda tr: all(den == 0 for den, _ in tr.tests)))
    out.append(_case("collinear_overlap_pill", "polygon4", pill((0.25, 0.25), (1.25, 0.25), 0.25), (0.0, 0.0), d=F(-1, 4),
                     smooth=False))
    out.append(_case("collinear_overlap_polygon", "polygon4", polygon([(0.5, 0.25), (1.0, 0.25), (1.0, 0.75), (0.5, 0.75)]),
                     (0.0, 0.0), d=F(0), smooth=False))
    # the pose exactly on a point obstacle
    # (a polygon footprint has no interior: the point inside the rectangle is 0.25 from its top and bottom edges)
    for fp, d in (("point", F(0)), ("circular", F(-1, 4)), ("line", F(0)), ("polygon2", F(0)), ("polygon4", F(1, 4))):
        out.append(_case(f"pose_on_point_{fp}", fp, point(0.5, 0.25), (0.5, 0.25), d=d, smooth=False))
    out.append(_case("pose_on_point_polygon_obstacle", "point", polygon([(0.5, 0.25)]), (0.5, 0.25), d=F(0), smooth=False))
    return out


def parallel_and_clamp_cases():
    out = []
    # parallel, disjoint, overlapping projections: two of the four endpoint combinations tie at 0.5
    # (obstacle start -> robot and robot end -> obstacle, both 0.5; the other two combinations sqrt(0.5))
    out.append(_case("parallel_tie", "line", line((0.25, 0.5), (1.25, 0.5)), (0.0, 0.0), d=F(1, 2), smooth=False,
                     claim=lambda tr: tr.tests[0] == (0, False)))
    out.append(_case("parallel_tie_polygons", "polygon4", polygon([(0.25, 0.75), (1.25, 0.75), (1.25, 1.25), (0.25, 1.25)]),
                     (0.0, 0.0), d=F(1, 2), smooth=False))
    # collinear, disjoint: the two combinations that meet at the same pair of endpoints tie
    out.append(_case("collinear_gap", "line", line((1.25, 0.0), (2.25, 0.0)), (0.0, 0.0), d=F(1, 2),
                     claim=lambda tr: tr.tests[0][0] == 0))
    # the foot of the perpendicular exactly at u = 0 / u = 1
    for fp in ("point", "line", "two_circles"):
        ext = F(RIGHT_EXTENT[fp])
        out.append(_case(f"clamp_u0_{fp}", fp, line((float(ext) + 0.5, 0.0), (float(ext) + 0.5, 1.0)), (0.0, 0.0),
                         d=F(1, 2), claim=lambda tr: F(0) in tr.us))
        out.append(_case(f"clamp_u1_{fp}", fp, line((float(ext) + 0.5, -1.0), (float(ext) + 0.5, 0.0)), (0.0, 0.0),
                         d=F(1, 2), claim=lambda tr: F(1) in tr.us))
    out.append(_case("clamp_u0_perpendicular", "point", polygon([(0.0, 0.5), (1.0, 0.5), (1.0, 1.5)]), (0.0, 0.0), d=F(1, 2),
                     claim=lambda tr: F(0) in tr.us))
    out.append(_case("clamp_u1_perpendicular", "point", pill((-1.0, 0.75), (0.0, 0.75), 0.25), (0.0, 0.0), d=F(1, 2),
                     claim=lambda tr: F(1) in tr.us))
    # zero-length segments: obstacle line, pill, and the footprint line
    out.append(_case("zero_line_obstacle_point", "point", line((0.5, 0.5), (0.5, 0.5)), (0.125, 0.0), d=F(5, 8)))
    out.append(_case("zero_line_obstacle_line", "line", line((0.25, 0.75), (0.25, 0.75)), (0.0, 0.0), d=F(3, 4),
                     claim=lambda tr: tr.tests[0][0] == 0))
    out.append(_case("zero_pill_polygon4", "polygon4", pill((1.25, 0.0), (1.25, 0.0), 0.25), (0.0, 0.0), d=F(1, 4)))
    out.append(_case("zero_footprint_line_point", "line_zero", point(0.25, 0.625), (0.0, 0.0), d=F(5, 8)))
    out.append(_case("zero_footprint_line_line", "line_zero", line((-0.75, 0.5), (1.25, 0.5)), (0.0, 0.0), d=F(1, 2)))
    out.append(_case("zero_footprint_line_polygon", "line_zero", polygon([(0.75, -0.5), (1.25, -0.5), (1.25, 0.5), (0.75, 0.5)]),
                     (0.0, 0.0), d=F(1, 2)))
    return out


def tie_cases():
    out = []
    # exterior corner bisector: both edges clamp to the shared vertex (the same pair twice)
    out.append(_case("corner_bisector_outside", "point", polygon([(0.5, 0.5), (1.0, 0.5), (1.0, 1.0), (0.5, 1.0)]),
                     (0.25, 0.25), claim=lambda tr: _ties(tr) == 2))
    # interior corner bisector: two edges at the same distance
    out.append(_case("corner_bisector_inside", "point", polygon([(-1.0, -1.0), (1.0, -1.0), (1.0, 1.0), (-1.0, 1.0)]),
                     (0.5, 0.5), d=F(1, 2), smooth=False, claim=lambda tr: _ties(tr) == 2))
    # two robot edges at the same distance: outside the rectangle's corner (one vertex) and inside it (top / bottom)
    out.append(_case("robot_edges_tie_corner", "polygon4", point(1.0, 0.5), (0.0, 0.0), claim=lambda tr: _ties(tr) == 2))
    out.append(_case("robot_edges_tie_inside", "polygon4", point(0.25, 0.0), (0.0, 0.0), d=F(1, 4), smooth=False,
                     claim=lambda tr: _ties(tr) == 2))
    # TwoCircles front / rear ties (df == dr) against a Point, a Circular and a Line obstacle, equal and unequal offsets
    def tc_tie(tr):
        (qf, rf), (qr, rr) = part_min(tr, 0), part_min(tr, 1)
        sf, sr = _sqrt(qf), _sqrt(qr)
        return (qf == qr and rf == rr) if sf is None or sr is None else sf - rf == sr - rr
    out.append(_case("tc_tie_point_issue", "two_circles", point(0.0, 1.0), (0.0, 0.0), smooth=False, claim=tc_tie))
    out.append(_case("tc_tie_point", "two_circles", point(0.0, 0.375), (0.0, 0.0), d=F(3, 8), smooth=False, claim=tc_tie))
    out.append(_case("tc_tie_circular", "two_circles", circle(0.0, -0.375, 0.125), (0.0, 0.0), d=F(1, 4), smooth=False,
                     claim=tc_tie))
    out.append(_case("tc_tie_line", "two_circles", line((-1.0, 0.375), (1.0, 0.375)), (0.0, 0.0), d=F(1, 8), smooth=False,
                     claim=tc_tie))
    out.append(_case("tc_uneq_tie_point", "two_circles_uneq", point(0.0625, 0.0), (0.0, 0.0), d=F(3, 16), smooth=False,
                     claim=tc_tie))
    out.append(_case("tc_uneq_tie_circular", "two_circles_uneq", circle(0.0625, 0.0, 0.0625), (0.0, 0.0), d=F(1, 8),
                     smooth=False, claim=tc_tie))
    out.append(_case("tc_uneq_tie_line", "two_circles_uneq", line((0.0625, -1.0), (0.0625, 1.0)), (0.0, 0.0), d=F(3, 16),
                     smooth=False, claim=tc_tie))
    out.append(_case("tc_tie_point_moving", "two_circles", point(0.0, 0.875, v=(0.0, -0.5)), (0.0, 0.0), t=T_CASE,
                     d=F(3, 8), smooth=False, claim=tc_tie))
    return out


def containment_cases():
    """the reference has no interior test: the distance is to the nearest edge (parallel edges and the two circles'
    tie in the square are kinks)"""
    big = [(-2.0, -2.0), (2.0, -2.0), (2.0, 2.0), (-2.0, 2.0)]
    out = []
    out.append(_case("robot_inside_polygon_point", "point", polygon(big), (1.5, 0.0), d=F(1, 2)))
    out.append(_case("robot_inside_polygon_rect", "polygon4", polygon(big), (0.0, 0.0), d=F(5, 4), smooth=False))
    out.append(_case("robot_inside_polygon_tc", "two_circles", polygon(big), (0.0, 0.0), d=F(5, 4), smooth=False))
    out.append(_case("obstacle_inside_robot_point", "polygon16", point(0.125, 0.0), (0.0, 0.0), d=F(3, 8)))
    out.append(_case("obstacle_inside_robot_polygon", "polygon16", polygon([(-0.125, -0.125), (0.125, -0.125), (0.125, 0.125)]),
                     (0.0, 0.0), d=F(3, 8), smooth=False))
    out.append(_case("obstacle_inside_robot_line", "polygon4", line((0.0, -0.125), (0.5, -0.125)), (0.0, 0.0), d=F(1, 8),
                     smooth=False))
    return out


def threshold_cases():
    """exactly at the penalty and association thresholds, reached through vertex-list distances (parallel edges are a
    kink in theta)"""
    out = []
    out.append(_case("thr_min_eps_line_point", "line", point(0.25, 0.625), (0.0, 0.0), d=F(MIN_D + EPS)))
    out.append(_case("thr_inflation_polygon", "point", polygon([(-0.5, 0.75), (0.5, 0.75), (0.5, 1.25), (-0.5, 1.25)]),
                     (0.0, 0.0), d=F(INFL)))
    out.append(_case("thr_inflation_rect_line", "polygon4", line((-1.0, -1.0), (1.0, -1.0)), (0.0, 0.0), d=F(INFL), smooth=False))
    out.append(_case("thr_dyn_inflation_moving_line", "line", line((-0.5, 1.875), (0.5, 1.875), v=(0.0, -1.0)), (0.0, 0.0),
                     t=T_CASE, d=F(DYN_INFL), smooth=False))
    out.append(_case("thr_dyn_inflation_moving_polygon", "polygon4",
                     polygon([(-0.5, -1.625), (0.5, -1.625), (0.5, -2.625), (-0.5, -2.625)], v=(0.0, 0.5)), (0.0, 0.0),
                     t=T_CASE, d=F(DYN_INFL), smooth=False))
    out.append(_case("thr_force_d_pill", "point", pill((-0.5, 1.25), (0.5, 1.25), 0.25), (0.0, 0.0), d=F(FORCE_D)))
    out.append(_case("thr_force_d_rect_polygon", "polygon4", polygon([(-0.5, 1.25), (0.5, 1.25), (0.5, 1.75), (-0.5, 1.75)]),
                     (0.0, 0.0), d=F(FORCE_D), smooth=False))
    out.append(_case("thr_cut_d_polygon", "point", polygon([(-0.5, -2.0), (0.5, -2.0), (0.5, -2.5), (-0.5, -2.5)]),
                     (0.0, 0.0), d=F(CUT_D)))
    out.append(_case("thr_cut_d_line_line", "line", line((-0.5, 2.0), (0.5, 2.0)), (0.0, 0.0), d=F(CUT_D), smooth=False))
    # centroid dead ahead (cross product 0: the obstacle counts as right), between force_d and cut_d
    out.append(_case("centroid_dead_ahead_line", "point", line((1.5, -0.5), (1.5, 0.5)), (0.0, 0.0), d=F(3, 2)))
    out.append(_case("centroid_dead_ahead_polygon", "polygon4", polygon([(2.0, -0.5), (2.5, -0.5), (2.5, 0.5), (2.0, 0.5)]),
                     (0.0, 0.0), d=F(5, 4), smooth=False))
    return out


def _round_polygon(k, radius=4.0):
    a = 2 * np.pi * np.arange(k) / k
    return np.round(np.stack([radius * np.cos(a), radius * np.sin(a)], 1) * 64) / 64


def large_polygon_cases():
    """regular 65 / 70-gons of radius 4 on the 2^-6 grid, the pose outside a vertex past index 64: the nearest
    point lies on an edge past the first 64 and the polygon of the first 64 vertices is farther by far more than
    rounding (0.019 in squared distance for 65 vertices)"""
    out = []
    for k, j in ((65, 64), (70, 68)):
        vs = _round_polygon(k)
        ang = 2 * np.pi * j / k
        for fp, v, t in (("point", (0.0, 0.0), None), ("polygon4", (0.0, 0.0), None), ("point", (0.25, -0.25), T_CASE)):
            reach = 4.5 if fp == "point" else 5.0      # the rectangle reaches 0.25 behind the pose
            pose = tuple(np.round(reach * np.array([np.cos(ang), np.sin(ang)]) * 64) / 64)
            row, verts = polygon(vs - np.array(v) * (t or 0.0), v=v)

            def claim(tr, fp=fp, row=row, verts=verts, pose=pose, t=t):
                pairs = tr.parts[0][0]
                first64 = trace(fp, row, verts, pose, t, limit=64).parts[0][0]
                return (max(i % k for i, q in enumerate(pairs) if q == min(pairs)) >= 64 and
                        min(first64) > min(pairs) + F(1, 100))
            out.append(_case(f"polygon{k}_nearest_past_64_{fp}{'_moving' if t else ''}", fp, (row, verts), pose, t=t,
                             claim=claim))
    return out


def all_cases():
    cs = (grid_cases() + contact_cases() + parallel_and_clamp_cases() + tie_cases() + containment_cases() +
          threshold_cases() + large_polygon_cases())
    names = [c.name for c in cs]
    assert len(set(names)) == len(names)
    return cs


def path_cases():
    """the cases whose obstacle is a Point or Circular and whose footprint is Point / Circular / TwoCircles: the
    kernels take the fast path for them unless the batch holds a vertex pool"""
    return [c for c in all_cases() if c.verts is None and c.fp in ("point", "circular", "two_circles", "two_circles_uneq")]


def far_line():
    """a Line obstacle far from every case: its vertex pool switches the kernels to the vertex-list path"""
    return line((1000.0, 1000.0), (1001.0, 1000.0))
