"""Bands for isTrajectoryFeasible (optimal_planner.cpp:1250-1310) at the edges of its look-ahead cut and of its
interpolation between poses, shared by tests/test_feasibility_cases.py (the claims against the drop-in layer's and the
reference's op 12) and tests/test_gpu_feasibility.py (the device check against both). Plain numpy; every builder
asserts on the host the property its case claims, with `ref_queries`, a direct transcription of the reference loop.

A case is one band and the check's arguments. `discs` (x, y, r) are op 12's recording costmap: a query collides when
hypot(x - cx, y - cy) <= r. On the device the same world is a Point footprint, circular obstacles of the discs' radii
and collision_distance 0. `disc_cases` keeps every disc at least 1e-9 from every query, except exact dyadic contacts.
"""
import math

import numpy as np

N_CAP = 64
TWO_PI = 2 * math.pi


def normalize_theta(t):
    """g2o::normalize_theta, evaluated as the reference evaluates it"""
    if -math.pi <= t < math.pi:
        return t
    m = math.floor(t / TWO_PI)
    t = t - m * 2.0 * math.pi
    if t >= math.pi:
        t -= TWO_PI
    if t < -math.pi:
        t += TWO_PI
    return t


def look_ahead(rec, n, look_ahead_idx, lookahead_distance):
    L = look_ahead_idx
    if L < 0 or L >= n:
        L = n - 1
    if lookahead_distance > 0:
        for i in range(1, n):
            if math.hypot(rec[i, 0] - rec[0, 0], rec[i, 1] - rec[0, 1]) > lookahead_distance:
                L = i - 1
                break
    return L


def segment_samples(p, q, inscribed, ang_res):
    """(extra samples, angular test, distance test) of the segment p -> q"""
    dr = normalize_theta(normalize_theta(q[2]) - normalize_theta(p[2]))
    dx, dy = q[0] - p[0], q[1] - p[1]
    norm = math.sqrt(dx * dx + dy * dy)
    ang, dist = abs(dr) > ang_res, norm > inscribed
    if not (ang or dist):
        return 0, ang, dist
    return int(max(math.ceil(abs(dr) / ang_res), math.ceil(norm / inscribed))) - 1, ang, dist


def ref_queries(rec, n, inscribed, look_ahead_idx=-1, lookahead_distance=-1.0, ang_res=math.pi):
    """every footprint query of the reference loop, in order, as [k][3]"""
    L = look_ahead(rec, n, look_ahead_idx, lookahead_distance)
    out = []
    for i in range(L + 1):
        p = rec[i]
        out.append((p[0], p[1], p[2]))
        if i < L:
            q = rec[i + 1]
            k, _, _ = segment_samples(p, q, inscribed, ang_res)
            dr = normalize_theta(normalize_theta(q[2]) - normalize_theta(p[2]))
            sx, sy, sr = (q[0] - p[0]) / (k + 1.0), (q[1] - p[1]) / (k + 1.0), dr / (k + 1.0)
            x, y, t = p[0], p[1], p[2]
            for _ in range(k):
                x, y = x + sx, y + sy
                t = normalize_theta(t + sr)
                out.append((x, y, t))
    return np.array(out, float).reshape(-1, 3)


def ref_verdict(queries, discs):
    """(feasible 1 / 0, query_count) of op 12 with the discs"""
    for k, (x, y, _) in enumerate(queries):
        for cx, cy, r in discs:
            if math.hypot(x - cx, y - cy) <= r:
                return 0, k + 1
    return 1, len(queries)


class Case:
    def __init__(self, name, rec, n, inscribed, look_ahead_idx=-1, lookahead_distance=-1.0, ang_res=math.pi,
                 discs=(), claim=None):
        full = np.zeros((max(N_CAP, n), 4))
        full[:n] = np.asarray(rec, float)[:n]
        self.name, self.rec, self.n = name, full, n
        self.inscribed, self.look_ahead_idx, self.lookahead_distance, self.ang_res = inscribed, look_ahead_idx, lookahead_distance, ang_res
        self.discs = [tuple(float(v) for v in d) for d in discs]
        self.queries = ref_queries(self.rec, n, inscribed, look_ahead_idx, lookahead_distance, ang_res)
        self.feasible, self.count = ref_verdict(self.queries, self.discs)
        if claim is not None:
            assert claim(self), name

    def op12_args(self, with_discs=True):
        d = self.discs if with_discs else []
        return [self.inscribed, self.inscribed + 0.2, self.look_ahead_idx, self.lookahead_distance, self.ang_res, len(d)] + \
            [v for disc in d for v in disc]

    def op12_cap(self):
        """output doubles op 12 needs for this case"""
        return 2 + 3 * (len(self.queries) + 8)

    def __repr__(self):
        return f"Case({self.name})"


def _line(n, dx=0.25, dy=0.0, th=0.0, x0=0.0, y0=0.0):
    rec = np.zeros((n, 4))
    rec[:, 0] = x0 + dx * np.arange(n)
    rec[:, 1] = y0 + dy * np.arange(n)
    rec[:, 2] = th
    rec[:-1, 3] = 0.3
    return rec


def _samples(c, i):
    return segment_samples(c.rec[i], c.rec[i + 1], c.inscribed, c.ang_res)


def band_cases():
    cs = []
    # band lengths: n = 0 (no query, feasible), 1, 2, n_cap
    cs.append(Case("n0", np.zeros((0, 4)), 0, 0.5, claim=lambda c: len(c.queries) == 0))
    cs.append(Case("n1", _line(1), 1, 0.5, claim=lambda c: len(c.queries) == 1))
    cs.append(Case("n2", _line(2, dx=1.0), 2, 0.3, claim=lambda c: len(c.queries) == 2 + 3))
    cs.append(Case("n_cap", _line(N_CAP, dx=0.3, dy=0.05), N_CAP, 0.1, claim=lambda c: c.n == N_CAP and
                   all(_samples(c, i)[0] == 3 for i in range(N_CAP - 1))))
    # headings across +-pi: the wrapped difference is small, the raw one is not
    rec = _line(6, dx=0.05)
    rec[:, 2] = [3.0, 3.1, -3.1, -3.0, -3.1, 3.12]
    cs.append(Case("wrap_pi", rec, 6, 0.5, ang_res=0.15, claim=lambda c: all(not _samples(c, i)[1] for i in range(5))
                   and abs(c.rec[2, 2] - c.rec[1, 2]) > 6))
    cs.append(Case("wrap_pi_fine", rec, 6, 0.5, ang_res=0.02, claim=lambda c: all(_samples(c, i)[1] for i in range(5))
                   and any(abs(q[2]) > 3.1 for q in c.queries)))
    # coincident poses and zero-length segments, with and without a turn
    rec = _line(5, dx=0.0)
    rec[3:, 2] = 1.0
    cs.append(Case("coincident", rec, 5, 0.2, ang_res=0.3, claim=lambda c: _samples(c, 0) == (0, False, False)
                   and _samples(c, 2) == (3, True, False)))
    # look-ahead index: -1, 0, n - 1, n, > n
    rec = _line(8, dx=0.4, dy=0.1)
    for lai in (-1, 0, 7, 8, 20, 3):
        L = 7 if lai in (-1, 7, 8, 20) else lai
        cs.append(Case(f"look_ahead_{lai}", rec, 8, 0.15, look_ahead_idx=lai,
                       claim=lambda c, L=L: look_ahead(c.rec, c.n, c.look_ahead_idx, c.lookahead_distance) == L))
    # look-ahead distance: off (0 and -1), cutting mid-band, and an exact tie on a 3-4-5 triangle
    for ld, L in ((0.0, 7), (-1.0, 7), (1.3, 3), (1.2, 2)):
        cs.append(Case(f"distance_{ld}", rec, 8, 0.15, lookahead_distance=ld,
                       claim=lambda c, L=L: look_ahead(c.rec, c.n, -1, c.lookahead_distance) == L))
    tri = _line(4, dx=0.0)
    tri[:, 0] = [0.0, 0.75, 1.5, 2.25]
    tri[:, 1] = [0.0, 1.0, 2.0, 3.0]            # 1.25, 2.5, 3.75 from pose 0: dyadic 3-4-5 triangles, hypot is exact
    for ld, L in ((2.5, 2), (2.4375, 1), (3.75, 3)):
        cs.append(Case(f"tie_{ld}", tri, 4, 1.0, lookahead_distance=ld,
                       claim=lambda c, L=L: look_ahead(c.rec, c.n, -1, c.lookahead_distance) == L and
                       math.hypot(c.rec[2, 0], c.rec[2, 1]) == 2.5 and math.hypot(c.rec[3, 0], c.rec[3, 1]) == 3.75))
    # look-ahead distance that extends past a smaller look-ahead index (the reference overwrites it)
    cs.append(Case("distance_after_index", rec, 8, 0.15, look_ahead_idx=1, lookahead_distance=1.3,
                   claim=lambda c: look_ahead(c.rec, c.n, 1, 1.3) == 3))
    # which test triggers: only the angular one, only the distance one, both, neither
    rec = _line(3, dx=0.1)
    rec[1:, 2] = [0.9, 1.8]
    cs.append(Case("angular_only", rec, 3, 0.5, ang_res=0.2, claim=lambda c: _samples(c, 0) == (4, True, False)))
    cs.append(Case("distance_only", _line(3, dx=0.9), 3, 0.2, ang_res=0.2, claim=lambda c: _samples(c, 0) == (4, False, True)))
    rec = _line(3, dx=0.9)
    rec[1:, 2] = [0.9, 1.8]
    cs.append(Case("both", rec, 3, 0.2, ang_res=0.1, claim=lambda c: _samples(c, 0) == (8, True, True)))
    cs.append(Case("neither", _line(3, dx=0.1), 3, 0.2, ang_res=0.2, claim=lambda c: _samples(c, 0) == (0, False, False)))
    # norm == inscribed_radius and |delta_rot| == angular_resolution exactly: strict >, no samples
    rec = _line(3, dx=0.0)
    rec[:, 0] = [0.0, 0.375, 0.75]
    rec[:, 1] = [0.0, 0.5, 1.0]
    cs.append(Case("norm_equal", rec, 3, 0.625, claim=lambda c: _samples(c, 0) == (0, False, False)
                   and math.sqrt(0.375 * 0.375 + 0.5 * 0.5) == 0.625))
    rec = _line(3, dx=0.0625)
    rec[:, 2] = [0.0, 0.5, -0.0]
    cs.append(Case("rot_equal", rec, 3, 0.5, ang_res=0.5, claim=lambda c: _samples(c, 0) == (0, False, False)
                   and _samples(c, 1) == (0, False, False)))
    # small inscribed radii: many samples per segment
    cs.append(Case("many_samples", _line(5, dx=0.8, dy=0.3), 5, 0.004, claim=lambda c: len(c.queries) > 800))
    cs.append(Case("many_samples_turn", np.c_[_line(4, dx=0.5)[:, :2], [0.0, 2.0, -2.0, 1.0], [0.3, 0.3, 0.3, 0.0]], 4,
                   0.01, ang_res=0.001, claim=lambda c: len(c.queries) > 5000))
    return cs


def random_cases(count=60, seed=11):
    """bands like the drop-in pin's: wiggly, random headings on a third of them, every argument random"""
    rng = np.random.default_rng(seed)
    cs = []
    for k in range(count):
        n = int(rng.integers(2, 40))
        x = np.cumsum(rng.uniform(0.05, 0.3, n))
        y = np.cumsum(rng.normal(0, 0.15, n))
        th = rng.uniform(-math.pi, math.pi, n) if rng.random() < 0.3 else np.arctan2(np.gradient(y), np.gradient(x))
        rec = np.stack([x, y, th, np.full(n, 0.3)], 1)
        cs.append(Case(f"random_{k}", rec, n, rng.uniform(0.05, 0.4), int(rng.integers(-1, n + 2)),
                       [0.0, 1.0, 3.0][int(rng.integers(3))], rng.uniform(0.1, 0.6)))
    return cs


def _gap(queries, k, center):
    """distance from `center` to the nearest query other than k whose position differs from query k"""
    d = [math.hypot(q[0] - center[0], q[1] - center[1]) for j, q in enumerate(queries)
         if j != k and (q[0], q[1]) != (queries[k][0], queries[k][1])]
    return min(d) if d else 1.0


def _with_discs(c, name, discs, claim):
    return Case(name, c.rec[:c.n], c.n, c.inscribed, c.look_ahead_idx, c.lookahead_distance, c.ang_res, discs, claim)


def _clear(c, discs):
    """every query is at least 1e-9 from every disc boundary"""
    return all(abs(math.hypot(q[0] - d[0], q[1] - d[1]) - d[2]) >= 1e-9 for q in c.queries for d in discs)


def disc_cases():
    """the band cases with discs: far away (feasible), centred on one query (the first query it holds decides), one of
    them an interpolated query, and exact dyadic contacts"""
    out = []
    rng = np.random.default_rng(12)
    for c in band_cases() + random_cases(30, seed=13):
        q = c.queries
        if len(q) == 0 or len(q) > 2000:
            continue
        far = [(q[:, 0].max() + 5.0, q[:, 1].max() + 5.0, 1.0)]
        out.append(_with_discs(c, c.name + "_far", far, lambda d: d.feasible == 1 and _clear(d, d.discs)))
        L = look_ahead(c.rec, c.n, c.look_ahead_idx, c.lookahead_distance)
        pose_idx, k = set(), 0
        for i in range(L + 1):
            pose_idx.add(k)
            k += 1 + (segment_samples(c.rec[i], c.rec[i + 1], c.inscribed, c.ang_res)[0] if i < L else 0)
        inter = [j for j in range(len(q)) if j not in pose_idx]
        picks = [int(rng.integers(len(q)))] + ([inter[int(rng.integers(len(inter)))]] if inter else [])
        for j in picks:
            centre = (q[j, 0] + 1e-4, q[j, 1] - 1e-4)
            r = min(0.05, 0.5 * _gap(q, j, centre))
            if r < 1e-3:
                continue
            tag = "inter" if j in inter else "pose"
            out.append(_with_discs(c, f"{c.name}_{tag}_{j}", [centre + (r,)],
                                   lambda d, j=j: d.feasible == 0 and d.count <= j + 1 and _clear(d, d.discs)))
    # exact contacts: a disc through a pose at a 3-4-5 offset (dyadic, hypot exact on every side)
    rec = _line(6, dx=0.5)
    for k, (ox, oy, r) in enumerate(((0.375, 0.5, 0.625), (-0.1875, 0.25, 0.3125))):
        centre = (rec[3, 0] + ox, rec[3, 1] + oy, r)
        out.append(Case(f"contact_{k}", rec, 6, 1.0, discs=[centre],
                        claim=lambda d: d.feasible == 0 and d.count == 4 and math.hypot(d.queries[3][0] - d.discs[0][0],
                                                                                        d.queries[3][1] - d.discs[0][1]) == d.discs[0][2]))
    return out
