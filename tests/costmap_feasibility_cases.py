"""isTrajectoryFeasible against the local costmap (base_local_planner::CostmapModel::footprintCost), restated in plain
Python, and the hand-computed cases that pin the restatement.

base_local_planner and costmap_2d are not part of the reference checkout, so nothing here is compiled from reference
sources: `world_to_map`, `line_cells`, `line_cost`, `point_cost` and `footprint_cost` restate navigation's ROS Noetic
code (Costmap2D::worldToMap, base_local_planner's LineIterator, CostmapModel::lineCost / pointCost / footprintCost and
WorldModel::footprintCost's vertex transform) step by step, as include/teb_b200.h defines it at TebCostmapWorld.
`verdict` runs the reference's loop (optimal_planner.cpp:1250-1310) over feasibility_cases.ref_queries. Plain Python
floats: every product and sum is rounded on its own, as in the reference's x86 build; math.cos / math.sin are glibc's.
"""
import math

import numpy as np

from tests import feasibility_cases as fc

LETHAL, INSCRIBED, NO_INFORMATION = 254, 253, 255


class Raster:
    """one scene's costmap: cost[my * sx + mx], size (sx, sy) in cells, origin (ox, oy) and resolution r"""

    def __init__(self, cost, sx, sy, ox, oy, r):
        self.cost = np.asarray(cost, np.uint8).reshape(-1)
        self.sx, self.sy, self.ox, self.oy, self.r = int(sx), int(sy), float(ox), float(oy), float(r)

    @classmethod
    def filled(cls, sx, sy, ox=0.0, oy=0.0, r=0.25, value=0, cells=()):
        """a map of `value` with the listed cells ((mx, my, cost), ...) set"""
        c = np.full(sx * sy, value, np.uint8)
        for mx, my, v in cells:
            c[my * sx + mx] = v
        return cls(c, sx, sy, ox, oy, r)

    def get(self, mx, my):
        return int(self.cost[my * self.sx + mx])


def world_to_map(m, wx, wy):
    """Costmap2D::worldToMap: (mx, my), or None off the map. A quotient past the int range is off the map (x86's
    truncation gives INT_MIN there, which the unsigned compare refuses)."""
    if wx < m.ox or wy < m.oy:
        return None
    qx, qy = (wx - m.ox) / m.r, (wy - m.oy) / m.r
    if not (qx < 2147483648.0 and qy < 2147483648.0):
        return None
    mx, my = int(qx), int(qy)
    if mx < m.sx and my < m.sy:
        return mx, my
    return None


def line_cells(x0, y0, x1, y1):
    """the cells of base_local_planner's LineIterator from (x0, y0) to (x1, y1), inclusive, by its advance()"""
    dx, dy = abs(x1 - x0), abs(y1 - y0)
    xinc1 = xinc2 = 1 if x1 >= x0 else -1
    yinc1 = yinc2 = 1 if y1 >= y0 else -1
    if dx >= dy:
        xinc1, yinc2 = 0, 0
        den, num, numadd, numpixels = dx, dx // 2, dy, dx
    else:
        xinc2, yinc1 = 0, 0
        den, num, numadd, numpixels = dy, dy // 2, dx, dy
    x, y, out = x0, y0, []
    for _ in range(numpixels + 1):
        out.append((x, y))
        num += numadd
        if num >= den:
            num -= den
            x += xinc1
            y += yinc1
        x += xinc2
        y += yinc2
    return out


def line_cell(x0, y0, x1, y1, k):
    """the k-th cell of the same walk in closed form: the minor axis has stepped (den // 2 + k * numadd) // den times"""
    dx, dy = abs(x1 - x0), abs(y1 - y0)
    sx, sy = (1 if x1 >= x0 else -1), (1 if y1 >= y0 else -1)
    if dx >= dy:
        m = (dx // 2 + k * dy) // dx if dx else 0
        return x0 + sx * k, y0 + sy * m
    m = (dy // 2 + k * dx) // dy
    return x0 + sx * m, y0 + sy * k


def point_cost(m, mx, my):
    """CostmapModel::pointCost: 255 -> -2, 254 -> -1, otherwise the cost (253 is not negative here)"""
    c = m.get(mx, my)
    if c == NO_INFORMATION:
        return -2
    if c == LETHAL:
        return -1
    return c


def line_cost(m, x0, x1, y0, y1):
    """CostmapModel::lineCost: the first negative point cost in walk order, otherwise the largest cost"""
    best = 0
    for mx, my in line_cells(x0, y0, x1, y1):
        p = point_cost(m, mx, my)
        if p < 0:
            return p
        if best < p:
            best = p
    return best


def transform(x, y, th, footprint, cs=None):
    """WorldModel::footprintCost's vertices: (x + (fx c - fy s), y + (fx s + fy c)), c and s computed once"""
    c, s = (math.cos(th), math.sin(th)) if cs is None else cs
    return [(x + (fx * c - fy * s), y + (fx * s + fy * c)) for fx, fy in footprint]


def footprint_cost(m, x, y, th, footprint, cs=None):
    """CostmapModel::footprintCost at the pose: -3 off the map, -2 / -1 as pointCost (plus 253 -> -1 for a footprint of
    fewer than 3 points, which reads the centre cell only), otherwise the largest cost on the outline"""
    centre = world_to_map(m, x, y)
    if centre is None:
        return -3
    if len(footprint) < 3:
        c = m.get(*centre)
        if c == NO_INFORMATION:
            return -2
        if c in (LETHAL, INSCRIBED):
            return -1
        return c
    v = transform(x, y, th, footprint, cs)
    best = 0
    F = len(v)
    for i in range(F):
        a, b = world_to_map(m, *v[i]), world_to_map(m, *v[(i + 1) % F])
        if a is None or b is None:
            return -3
        lc = line_cost(m, a[0], b[0], a[1], b[1])
        best = max(lc, best)
        if lc < 0:
            return lc
    return best


def verdict(m, queries, footprint, max_queries=None, cs=None):
    """(feasible, query_count, query_cost) of the reference loop over the queries: the first query whose cost is -1
    makes the band infeasible (0); -2 and -3 are free. More queries than max_queries, all tested ones free: -1 with
    the full count, as tebgpu_check_feasible. query_cost holds the tested queries' costs."""
    qc = []
    limit = len(queries) if max_queries is None else min(len(queries), max_queries)
    for k in range(limit):
        x, y, th = (float(v) for v in queries[k])
        c = footprint_cost(m, x, y, th, footprint, None if cs is None else cs[k])
        qc.append(c)
        if c == -1:
            return 0, k + 1, qc
    if limit < len(queries):
        return -1, len(queries), qc
    return 1, len(queries), qc


def band_verdict(m, rec, n, footprint, inscribed, look_ahead_idx=-1, lookahead_distance=-1.0, ang_res=math.pi,
                 max_queries=None):
    """verdict over feasibility_cases.ref_queries of the band; a non-finite checked pose gives -1 with no query"""
    L = fc.look_ahead(rec, n, look_ahead_idx, lookahead_distance)
    if any(not np.isfinite(rec[i, :3]).all() for i in range(L + 1)):
        return -1, 0, []
    q = fc.ref_queries(rec, n, inscribed, look_ahead_idx, lookahead_distance, ang_res)
    return verdict(m, q, footprint, max_queries)


def near_cell_edge(m, x, y, th, footprint, tol=1e-9):
    """True when the centre or a transformed vertex lies within `tol` cells of a cell edge (where the device's cos /
    sin, which may differ from glibc's in the last bit, can move a vertex into the next cell)"""
    pts = [(x, y)] + (transform(x, y, th, footprint) if len(footprint) >= 3 else [])
    for wx, wy in pts:
        for q in ((wx - m.ox) / m.r, (wy - m.oy) / m.r):
            if abs(q - round(q)) < tol:
                return True
    return False


# ---- hand cases: (name, raster, pose, footprint, expected footprintCost)

SQUARE = [(-0.3, -0.3), (0.3, -0.3), (0.3, 0.3), (-0.3, 0.3)]


def hand_cases():
    """the footprint-cost cases of tests/test_costmap_feasibility_cases.py, for the device test to replay: every entry
    (name, raster, (x, y, theta), footprint, expected cost)"""
    out = []
    r = Raster.filled
    # F = 0, 1, 2 read the centre cell only: 253 / 254 -> -1, 255 -> -2, a cost -> the cost
    for F in (0, 1, 2):
        fp = [(0.5, 0.0), (0.0, 0.5)][:F]
        for v, want in ((253, -1), (254, -1), (255, -2), (100, 100), (0, 0)):
            out.append((f"centre_F{F}_{v}", r(8, 8, value=0, cells=[(2, 2, v)]), (0.6, 0.6, 0.0), fp, want))
    # off-map centre: below the origin, at ox + sx r, inside
    m = r(8, 8, ox=1.0, oy=2.0, r=0.125)
    out.append(("centre_at_origin", m, (1.0, 2.0, 0.0), [], 0))
    out.append(("centre_below_origin", m, (math.nextafter(1.0, 0.0), 2.5, 0.0), [], -3))
    out.append(("centre_at_far_edge", m, (1.0 + 8 * 0.125, 2.5, 0.0), [], -3))
    out.append(("centre_off_square", m, (5.0, 2.5, 0.0), SQUARE, -3))
    # F >= 3: lethal inside the polygon but off the outline is free; 253 on the outline is free (its cost counts)
    sq = [(-0.5, -0.5), (0.5, -0.5), (0.5, 0.5), (-0.5, 0.5)]              # 4 x 4 cells at r = 0.25
    out.append(("lethal_inside", r(12, 12, cells=[(5, 5, 254), (6, 6, 254)]), (1.5, 1.5, 0.0), sq, 0))
    out.append(("inscribed_on_outline", r(12, 12, cells=[(4, 4, 253)]), (1.5, 1.5, 0.0), sq, 253))
    out.append(("max_cost", r(12, 12, cells=[(4, 5, 17), (8, 6, 200), (6, 8, 99)]), (1.5, 1.5, 0.0), sq, 200))
    # the first negative in walk order: edge 0 runs (4, 4) -> (8, 4), then (8, 4) -> (8, 8), (8, 8) -> (4, 8), (4, 8) -> (4, 4)
    out.append(("unknown_before_lethal", r(12, 12, cells=[(5, 4, 255), (7, 4, 254)]), (1.5, 1.5, 0.0), sq, -2))
    out.append(("lethal_before_unknown", r(12, 12, cells=[(5, 4, 254), (7, 4, 255)]), (1.5, 1.5, 0.0), sq, -1))
    out.append(("unknown_edge0_lethal_edge1", r(12, 12, cells=[(6, 4, 255), (8, 6, 254)]), (1.5, 1.5, 0.0), sq, -2))
    out.append(("closing_edge_alone", r(12, 12, cells=[(4, 6, 254)]), (1.5, 1.5, 0.0), sq, -1))
    # a vertex leaving the map: -3, unless an earlier edge already met a negative cost
    out.append(("vertex_off_map", r(12, 12), (0.375, 1.5, 0.0), sq, -3))
    out.append(("lethal_before_off_map", r(12, 12, cells=[(1, 6, 254)]), (0.375, 1.5, 0.0),
                [(-0.125, 0.5), (-0.125, -0.5), (-0.5, 0.0)], -1))
    # vertices exactly on cell edges at dyadic resolutions, theta = 0 so the trig is exact
    for res in (0.125, 0.25):
        m = r(16, 16, r=res, cells=[(6, 6, 254)])
        out.append((f"edge_vertex_{res}", m, (6 * res, 6 * res, 0.0), [(0.0, 0.0), (res, 0.0), (0.0, res)], -1))
        out.append((f"edge_vertex_below_{res}", m, (6 * res, 6 * res, 0.0),
                    [(-res, -res), (math.nextafter(0.0, -1.0), -res), (-res, math.nextafter(0.0, -1.0))], 0))
    # a single-cell polygon (every edge zero length) and a 16-vertex circle turned by a non-trivial angle
    out.append(("single_cell", r(8, 8, cells=[(3, 3, 60)]), (0.875, 0.875, 0.3), [(0.01, 0.0), (0.0, 0.01), (-0.01, 0.0)], 60))
    circ = [(0.4 * math.cos(2 * math.pi * k / 16), 0.4 * math.sin(2 * math.pi * k / 16)) for k in range(16)]
    out.append(("circle16", r(16, 16, value=3, cells=[(10, 8, 254)]), (2.0, 2.0, 0.7), circ, None))
    return out


def random_fleet(S, sx, sy, res, seed, F, bands_per_scene=4):
    """bands like random_cases' laid over scenes.costmap_raster maps: (raster dict, rec [B][n_cap][4], n [B], scene_id [B],
    footprint [F][2]). Poses are centred in the maps, so queries reach lethal, inscribed, unknown cells and the edges."""
    from teb_local_planner_b200 import scenes
    rng = np.random.default_rng(seed)
    ras = scenes.costmap_raster(S, sx, sy, res, 0.05, seed=seed)
    B = S * bands_per_scene
    rec = np.zeros((B, fc.N_CAP, 4))
    n = rng.integers(2, 40, B).astype(np.int32)
    sid = np.repeat(np.arange(S, dtype=np.int32), bands_per_scene)
    for b in range(B):
        ox, oy, r = ras["origin"][sid[b]]
        w, h = sx * r, sy * r
        x0, y0 = ox + rng.uniform(0.05, 0.95) * w, oy + rng.uniform(0.05, 0.95) * h
        a = rng.uniform(-math.pi, math.pi)
        step = rng.uniform(0.02, 0.15, n[b])
        turn = np.cumsum(rng.normal(0, 0.2, n[b])) + a
        x = x0 + np.cumsum(step * np.cos(turn))
        y = y0 + np.cumsum(step * np.sin(turn))
        th = rng.uniform(-math.pi, math.pi, n[b]) if rng.random() < 0.3 else turn
        rec[b, :n[b]] = np.stack([x, y, th, np.full(n[b], 0.3)], 1)
    if F == 0:
        fp = np.zeros((0, 2))
    elif F < 3:
        fp = rng.uniform(-0.3, 0.3, (F, 2))
    elif F == 4:
        fp = np.array([(-0.25, -0.2), (0.35, -0.2), (0.35, 0.2), (-0.25, 0.2)]) + rng.uniform(-0.02, 0.02, (4, 2))
    else:
        ang = np.sort(rng.uniform(0, 2 * math.pi, F))
        rad = rng.uniform(0.15, 0.45, F)
        fp = np.stack([rad * np.cos(ang), rad * np.sin(ang)], 1)
    return ras, rec, n, sid, fp


def raster_of(ras, s):
    sx, sy = (int(v) for v in ras["grid"][s])
    ox, oy, r = ras["origin"][s]
    return Raster(ras["cost"][s, :sx * sy], sx, sy, ox, oy, r)
