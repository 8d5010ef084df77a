"""Seeded synthetic planning scenes (SURVEY.md §8d / BASELINE.md §3).

A *request* is one planning problem (start, goal, obstacle table); a *candidate* is one initial band
of that request in its own homotopy-like class (lateral sinusoid of amplitude A_k). The batch axis of
the optimizer is candidates x requests.
"""
import math

import numpy as np

from . import abi


def demo_scene_obstacles():
    """The three obstacles of test_optim_node (reference src/test_optim_node.cpp:106-117)."""
    o = np.zeros(3, abi.OBST_DTYPE)
    o["x"], o["y"] = [-3.0, 6.0, 0.0], [1.0, 2.0, 0.1]
    o["vx"], o["vy"] = [0.1, -0.3, 0.0], [-0.3, -0.2, 0.0]
    o["dynamic"] = [1, 1, 0]
    return o


def make_band(n, amplitude, max_vel_x=0.4, dt_ref=0.3, length=None):
    """Straight line start(-L/2,0,0) -> goal(L/2,0,0) plus lateral offset A*sin(pi s)."""
    L = max_vel_x * dt_ref * (n - 1) if length is None else length
    s = np.linspace(0.0, 1.0, n)
    x = -L / 2 + L * s
    y = amplitude * np.sin(np.pi * s)
    th = np.zeros(n)
    th[1:-1] = np.arctan2(y[2:] - y[1:-1], x[2:] - x[1:-1])
    seg = np.hypot(np.diff(x), np.diff(y))
    rec = np.zeros((n, 4))
    rec[:, 0], rec[:, 1], rec[:, 2] = x, y, th
    rec[:-1, 3] = seg / max_vel_x
    return rec


def make_obstacles(rng, M, L, inflated=False, moving=False, M_cap=None):
    M_cap = M if M_cap is None else M_cap
    o = np.zeros(M_cap, abi.OBST_DTYPE)
    k = 0
    lo, hi = -L / 2 + 1.0, L / 2 - 1.0
    if hi <= lo:
        lo, hi = -L / 2, L / 2
    while k < M:
        x, y = rng.uniform(lo, hi), rng.uniform(-3.0, 3.0)
        if min(np.hypot(x + L / 2, y), np.hypot(x - L / 2, y)) < 0.3:
            continue
        o[k]["x"], o[k]["y"] = x, y
        if inflated:
            o[k]["radius"] = rng.uniform(0.0, 0.3)
            o[k]["type"] = abi.TEB_OBST_CIRCULAR
        if moving:
            o[k]["vx"], o[k]["vy"] = rng.uniform(-0.3, 0.3, 2)
            o[k]["dynamic"] = 1
        k += 1
    return o


def make_batch(n, M, candidates, requests=1, seed=0, inflated=False, moving=False, via_points=0,
               n_cap=None, amp=2.0, max_vel_x=0.4, dt_ref=0.3):
    """Build a HostBatch of `candidates * requests` bands; scene s = request s."""
    n_cap = n if n_cap is None else n_cap
    B = candidates * requests
    L = max_vel_x * dt_ref * (n - 1)
    poses = np.zeros((B, n_cap, 4))
    obst = np.zeros((requests, max(M, 1)), abi.OBST_DTYPE)
    via = np.zeros((B, via_points, 2)) if via_points else None
    via_count = np.full(B, via_points, np.int32) if via_points else None
    scene_id = np.zeros(B, np.int32)
    for r in range(requests):
        rng = np.random.default_rng(seed * 100003 + r)
        obst[r, :M] = make_obstacles(rng, M, L, inflated, moving)[:M]
        for k in range(candidates):
            b = r * candidates + k
            brng = np.random.default_rng((seed * 100003 + r) * 1000003 + k)
            A = brng.uniform(-amp, amp)
            poses[b, :n] = make_band(n, A, max_vel_x, dt_ref)
            scene_id[b] = r
            if via_points:
                sv = np.linspace(0.2, 0.8, via_points)
                via[b, :, 0] = -L / 2 + L * sv
                via[b, :, 1] = A * np.sin(np.pi * sv)
    hb = abi.HostBatch(poses, np.full(B, n, np.int32), obst, np.full(requests, M, np.int32), scene_id,
                       via, via_count)
    return hb


def config_params(name):
    """TebParams for the BASELINE.md §3 configs (ctor defaults + per-config overrides)."""
    p = abi.default_params()
    if name == "C1":
        p.no_inner_iterations, p.no_outer_iterations = 4, 3
    elif name == "C2":
        p.min_turning_radius = 0.0
    elif name == "C3":
        p.min_turning_radius = 0.5
    elif name == "C4":
        p.include_dynamic_obstacles = 1
        p.weight_viapoint = 1.0
    else:
        raise ValueError(name)
    return p


CONFIG_SHAPES = {
    # name: (n poses, M obstacles, candidates, inflated, moving, via-points)
    "C1": (50, 5, 1, False, False, 0),
    "C2": (100, 20, 32, False, False, 0),
    "C3": (200, 64, 128, True, False, 0),
    "C4": (150, 32, 512, False, True, 4),
}


def make_config_batch(name, requests=1, seed=0, candidates=None, autosize=False):
    n, M, cand, inflated, moving, via_pts = CONFIG_SHAPES[name]
    cand = cand if candidates is None else candidates
    p = config_params(name)
    p.teb_autosize = int(autosize)
    n_cap = n if not autosize else min(2 * n, 512)
    hb = make_batch(n, M, cand, requests, seed, inflated, moving, via_pts, n_cap=n_cap)
    return p, hb


def polygon_centroid(v):
    """PolygonObstacle::calcCentroid (reference src/obstacles.cpp:56-119) for non-degenerate polygons."""
    v = np.asarray(v, float)
    if len(v) == 1:
        return v[0].copy()
    if len(v) == 2:
        return 0.5 * (v[0] + v[1])
    w = np.roll(v, -1, axis=0)
    aux = v[:, 0] * w[:, 1] - w[:, 0] * v[:, 1]
    A = 0.5 * aux.sum()
    return ((v + w) * aux[:, None]).sum(0) / (6 * A)


def add_shape_obstacles(hb, seed=0, kinds=(abi.TEB_OBST_LINE, abi.TEB_OBST_PILL, abi.TEB_OBST_POLYGON), every=2):
    """Turn every `every`-th obstacle of each scene into a Line / Pill / Polygon obstacle around its old position
    (vertices go to the scene's vertex pool, (x, y) becomes getCentroid()). Returns a new HostBatch."""
    obst = hb.obstacles.copy()
    pools = []
    for s in range(hb.S):
        rng = np.random.default_rng(seed * 7919 + s)
        pool = []
        for m in range(0, int(hb.obst_count[s]), every):
            kind = kinds[(m // every) % len(kinds)]
            c = np.array([obst[s, m]["x"], obst[s, m]["y"]])
            if kind == abi.TEB_OBST_POLYGON:
                nv = int(rng.integers(3, 6))
                ang = np.sort(rng.uniform(0, 2 * np.pi, nv))
                v = c + np.stack([np.cos(ang), np.sin(ang)], 1) * rng.uniform(0.15, 0.5, (nv, 1))
            else:
                a = rng.uniform(0, np.pi)
                h = rng.uniform(0.2, 0.6)
                v = np.array([c - h * np.array([np.cos(a), np.sin(a)]), c + h * np.array([np.cos(a), np.sin(a)])])
            ctr = polygon_centroid(v)
            obst[s, m]["x"], obst[s, m]["y"] = ctr
            obst[s, m]["type"] = kind
            obst[s, m]["radius"] = rng.uniform(0.05, 0.25) if kind == abi.TEB_OBST_PILL else 0.0
            obst[s, m]["vertex_begin"], obst[s, m]["vertex_count"] = len(pool), len(v)
            pool.extend(v.tolist())
        pools.append(pool)
    pv = max(1, max(len(p) for p in pools))
    verts = np.zeros((hb.S, pv, 2))
    for s, pool in enumerate(pools):
        if pool:
            verts[s, :len(pool)] = pool
    return abi.HostBatch(hb.poses.copy(), hb.n.copy(), obst, hb.obst_count.copy(), hb.scene_id.copy(),
                         hb.via.copy() if hb.V_cap > 0 else None, hb.via_count.copy() if hb.V_cap > 0 else None,
                         hb.vel_start.copy(), hb.vel_goal.copy(), hb.prefer_rotdir.copy(), verts)


def set_line_footprint(p, start=(-0.3, 0.0), end=(0.4, 0.0)):
    p.footprint_type = abi.TEB_FOOTPRINT_LINE
    p.footprint_line[0], p.footprint_line[1], p.footprint_line[2], p.footprint_line[3] = start[0], start[1], end[0], end[1]
    return p


def set_polygon_footprint(p, vertices=((-0.25, -0.2), (0.35, -0.2), (0.35, 0.2), (-0.25, 0.2))):
    p.footprint_type = abi.TEB_FOOTPRINT_POLYGON
    p.footprint_vertex_count = len(vertices)
    for k, (x, y) in enumerate(vertices):
        p.footprint_vertices[2 * k], p.footprint_vertices[2 * k + 1] = x, y
    return p


def costmap_scene(M, n=100, candidates=3, seed=0, amp=0.6, shapes=True):
    """A scene the way a local costmap produces it: one point obstacle per occupied 5 cm cell (two walls along the
    corridor and blobs of cells near the band), plus a few circular, line and moving obstacles. Exactly M rows.
    -> (TebParams, HostBatch) with C3's parameters, moving obstacles switched on and autoResize off."""
    p = config_params("C3")
    p.include_dynamic_obstacles = 1
    p.teb_autosize = 0
    rng = np.random.default_rng(seed)
    L = 0.4 * 0.3 * (n - 1)
    cells = set()
    res = 0.05
    for y in (-1.6, 1.6):                              # walls of the corridor
        for x in np.arange(-L / 2, L / 2, res):
            cells.add((round(x / res), round(y / res)))
    while len(cells) < M:                              # blobs of occupied cells beside the band
        cx, cy = rng.uniform(-L / 2 + 1, L / 2 - 1), rng.choice([-1, 1]) * rng.uniform(0.8, 3.0)
        r = rng.uniform(0.05, 0.4)
        for gx in range(round((cx - r) / res), round((cx + r) / res) + 1):
            for gy in range(round((cy - r) / res), round((cy + r) / res) + 1):
                if (gx * res - cx) ** 2 + (gy * res - cy) ** 2 <= r * r:
                    cells.add((gx, gy))
    cells = sorted(cells, key=lambda c: rng.random())[:M]
    o = np.zeros(M, abi.OBST_DTYPE)
    o["x"] = [c[0] * res for c in cells]
    o["y"] = [c[1] * res for c in cells]
    pool = np.zeros((0, 2))
    if shapes:
        k = rng.choice(M, 12, replace=False)
        o["type"][k[:4]], o["radius"][k[:4]] = abi.TEB_OBST_CIRCULAR, 0.1
        o["dynamic"][k[4:8]] = 1                       # moving points
        o["vx"][k[4:8]], o["vy"][k[4:8]] = rng.uniform(-0.3, 0.3, 4), rng.uniform(-0.3, 0.3, 4)
        pool = np.zeros((8, 2))
        for j, m in enumerate(k[8:]):                  # short line segments centred on their cell
            pool[2 * j] = (o["x"][m] - 0.1, o["y"][m] - 0.05)
            pool[2 * j + 1] = (o["x"][m] + 0.1, o["y"][m] + 0.05)
            o["type"][m], o["vertex_begin"][m], o["vertex_count"][m] = abi.TEB_OBST_LINE, 2 * j, 2
    poses = np.zeros((candidates, n, 4))
    brng = np.random.default_rng(seed + 1)
    for b in range(candidates):
        poses[b] = make_band(n, brng.uniform(-amp, amp), 0.4, 0.3)
    hb = abi.HostBatch(poses, np.full(candidates, n, np.int32), o, np.array([M], np.int32),
                       obst_vertices=pool[None] if shapes else None)
    return p, hb


def costmap_raster(S, sx=120, sy=120, res=0.05, lethal=0.05, seed=0, cell_cap=None):
    """A fleet of S local costmaps the way costmap_2d fills them, for tebgpu_costmap_obstacles: two walls and blobs of
    LETHAL_OBSTACLE (254) cells until `lethal` of the cells are lethal, an inflation ring around them (253 next to a
    lethal cell, lower costs further out) and a 4 x 4 patch of NO_INFORMATION (255), so the raster holds values next to
    254 that must not count. Each map is centred near its robot (a rolling window), whose yaw is drawn over (-pi, pi].
    -> dict(cost [S][cell_cap] uint8 (row my holds cells my * sx .. my * sx + sx - 1; cell_cap defaults to sx * sy
    rounded up to 16 bytes), grid [S][2] int32, origin [S][3] (ox, oy, res), robot [S][3] (x, y, yaw))."""
    rng = np.random.default_rng(seed)
    cap = ((sx * sy + 15) // 16) * 16 if cell_cap is None else int(cell_cap)
    cost = np.zeros((S, cap), np.uint8)
    grid = np.tile(np.array([sx, sy], np.int32), (S, 1))
    origin = np.zeros((S, 3))
    robot = np.zeros((S, 3))
    yy, xx = np.mgrid[0:sy, 0:sx]
    ring = [(dx, dy, math.hypot(dx, dy)) for dx in range(-4, 5) for dy in range(-4, 5) if 0 < math.hypot(dx, dy) <= 4]
    for s in range(S):
        rx, ry = rng.uniform(-20, 20, 2)
        origin[s] = (rx - 0.5 * sx * res + rng.uniform(-0.3, 0.3), ry - 0.5 * sy * res + rng.uniform(-0.3, 0.3), res)
        robot[s] = (rx, ry, rng.uniform(-math.pi, math.pi))
        m = np.zeros((sy, sx), bool)
        if sx > 0 and sy > 0:
            for wy in (int(0.15 * sy), int(0.85 * sy)):                   # two walls
                m[wy, int(0.1 * sx):int(0.9 * sx)] = True
            target = lethal * sx * sy
            while m.sum() < target:                                       # blobs
                cx, cy, r = rng.uniform(0, sx), rng.uniform(0, sy), rng.uniform(1.0, 6.0)
                m |= (xx - cx) ** 2 + (yy - cy) ** 2 <= r * r
        d = np.full((sy, sx), np.inf)                                     # distance to the nearest lethal cell, in cells
        pad = np.pad(m, 4)
        for dx, dy, h in ring:
            d = np.where(pad[4 + dy:4 + dy + sy, 4 + dx:4 + dx + sx], np.minimum(d, h), d)
        c = np.zeros((sy, sx), np.uint8)
        c[d <= 1.0] = 253                                                 # INSCRIBED_INFLATED_OBSTACLE
        far = (d > 1.0) & np.isfinite(d)
        c[far] = (252 * np.exp(-1.5 * (d[far] - 1.0))).astype(np.uint8)
        c[m] = 254
        if sx >= 4 and sy >= 4:                                           # NO_INFORMATION
            px, py = rng.integers(0, sx - 3), rng.integers(0, sy - 3)
            c[py:py + 4, px:px + 4] = 255
        cost[s, :sx * sy] = c.reshape(-1)
    return dict(cost=cost, grid=grid, origin=origin, robot=robot)


def global_plans(B, G_cap=2048, S=4, spacing=0.05, seed=0):
    """A fleet of B robots following global plans, for tebgpu_local_plan: plans at costmap-like spacing (`spacing` m
    between rows, yaw along the path) of four kinds by b % 4: smooth curves, loops that pass back by the robot (the
    closest-row search meets two minima), zig-zags, and short plans that end inside the costmap window. Some rows are
    repeated (coincident rows), the live rows start at a random plan_begin at or before the robot's row, and the robot
    stands near that row, slightly off the path, some robots stopped. Scene s has a square costmap of 80 .. 160 cells at
    0.05 m. -> dict(global_plan [B][G_cap][3] (NaN past plan_end), plan_begin [B], plan_end [B] int32, robot [B][3],
    robot_vel [B][3], scene_id [B] int32, grid [S][2] int32, origin [S][3])."""
    rng = np.random.default_rng(seed)
    gp = np.full((B, G_cap, 3), np.nan)
    begin, end = np.zeros(B, np.int32), np.zeros(B, np.int32)
    robot, vel = np.zeros((B, 3)), np.zeros((B, 3))
    sid = (np.arange(B) % S).astype(np.int32)
    side = rng.integers(80, 161, S)
    grid = np.stack([side, side], 1).astype(np.int32)
    origin = np.zeros((S, 3))
    origin[:, 2] = 0.05
    for b in range(B):
        kind = b % 4
        n = int(rng.integers(5, 60)) if kind == 3 else int(rng.integers(G_cap // 2, G_cap + 1))
        head = rng.uniform(-math.pi, math.pi)
        turn = rng.uniform(-0.02, 0.02, n)
        if kind == 1:                               # a loop of radius ~1 m two fifths of the way along
            k0 = int(0.4 * n)
            turn[k0:k0 + int(2 * math.pi / (spacing / 1.0))] = spacing / 1.0
        elif kind == 2:                             # zig-zag: turn by +-1 rad every 10 rows
            turn[::10] = np.where(np.arange(len(turn[::10])) % 2 == 0, 1.0, -1.0)
        th = head + np.cumsum(turn)
        step = np.full(n, spacing) * rng.uniform(0.8, 1.2, n)
        step[rng.random(n) < 0.03] = 0.0            # coincident rows
        xy = np.cumsum(np.stack([step * np.cos(th), step * np.sin(th)], 1), 0) + rng.uniform(-20, 20, 2)
        yaw = np.arctan2(np.diff(xy[:, 1], append=xy[-1, 1]), np.diff(xy[:, 0], append=xy[-1, 0]))
        gp[b, :n, :2], gp[b, :n, 2] = xy, yaw
        r0 = int(rng.integers(0, max(1, n // 3))) if kind != 3 else int(rng.integers(0, n))
        if kind == 1:
            r0 = int(0.4 * n) - 1                   # the loop comes back by the robot
        begin[b], end[b] = int(rng.integers(0, r0 + 1)), n
        off = rng.choice([0.0, 0.01, 0.1, 0.5]) * rng.uniform(-1, 1, 2)
        robot[b] = (xy[r0, 0] + off[0], xy[r0, 1] + off[1], yaw[r0] + rng.uniform(-0.3, 0.3))
        vel[b] = (0.0, 0.0, 0.0) if rng.random() < 0.3 else (rng.uniform(-0.2, 0.5), rng.uniform(-0.1, 0.1), rng.uniform(-0.5, 0.5))
    return dict(global_plan=gp, plan_begin=begin, plan_end=end, robot=robot, robot_vel=vel, scene_id=sid, grid=grid,
                origin=origin)
