"""The persistent trial evaluation k_trial_eval2p (batches of more than 2 x SMs bands), band by band.

k_trial_eval2p runs k_trial_eval2's per-band code in G = resident CTAs per SM x SMs CTAs; CTA c takes the slots c, c + G,
c + 2G, ... (every band in round 0, the retry list in retry rounds, its length read on the device). What only it does -
skip inactive bands, stage band j + 1 by cp.async into the buffer band j just left, copy the obstacle table again only
when the scene changes - runs only when a CTA takes a second slot. So every case here reads G from the device
(TebGpu.last_trial_eval) and asserts that the launch was k_trial_eval2p and that there were more than 3 G slots (a
ragged last pass included), or, for the short retry lists, fewer than G.

  a. one round through TebGpu.eval_trials: rows, state, qmax, need, the next list (as a set) and the poses bit-equal to
     k_trial_eval3 (TEBGPU_EVAL3=1, any batch size, contracted to the same bits) for every band; the decisions of every
     band against teb_oracle_lm_decide, the chi2 of a sample (every band in slot >= 2 G, at most ~60) against
     teb_oracle_trial_chi2 at 1e-12 per family. Cases: scene patterns along a CTA's slots (same scene, A -> B -> A, many
     rows -> few, empty -> full), long and short bands in one CTA with NaN / +-1e300 trial rows where the next band ends,
     inactive bands, retry lists longer and shorter than G and empty, K = 2 .. 8, the staged, GEOM and global-table
     builds, and a permuted batch (each band keeps its bits wherever it sits);
  b. optimize in the throughput regime (B > 3 G at every speculation width the schedule uses): n, poses, cost, chi2,
     status and lm_iters bit-equal to TEBGPU_EVAL3=1, on C1 with autosize, C3, C4, shapes_polygon, vor, a scene padded
     past 1024 rows and the split round-0 schedule; bands in the last slot of their CTA against the oracle at 1e-6."""
import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import banded_reference as R
from tests import oracle_binding as O
from tests import scenarios
from tests.test_gpu_parity import _report as _write_report
from tests.test_gpu_trial_eval import Round, _bits, _ctx, _same_bits, _sms, _state, check_chi2, check_decisions

pytestmark = pytest.mark.gpu

CHI2_SAMPLE = 60      # bands per round checked against teb_oracle_trial_chi2 (CPU time)
GT_ROWS = 1100        # a table of more than 1024 rows: the global-table builds
# lambda after an accepted trial, against teb_oracle_lm_decide: the device cubes 2 rho - 1 by products, the oracle with
# pow, and 1 - (2 rho - 1)^3 cancels when rho is near 1, so the ulps of the cube grow in the factor. Up to 3 ulp were seen
# in a round of ~1400 bands here; the device's lambda is pinned bit for bit against k_trial_eval3.
LAMBDA_ULPS = 4
_slots = {}


def _report(key, value):
    _slots[key] = value
    _write_report("trial_eval_persistent", dict(sorted(_slots.items())))


# ------------------------------------------------------------------ batches
def _params(cfg):
    p = scenes.config_params("C4" if cfg == "shapes_polygon" else "C3")
    p.teb_autosize = 0
    if cfg == "shapes_polygon":
        scenes.set_polygon_footprint(p)
    return p


def _tables(cfg, counts, L, gt, seed):
    """obstacle tables of len(counts) scenes, scene s with counts[s] rows (M_cap = max(counts)); gt: every non-empty
    table padded to GT_ROWS rows with far points"""
    M_cap = max(counts)
    shapes = cfg == "shapes_polygon"
    ob = np.zeros((len(counts), M_cap), abi.OBST_DTYPE)
    for s, M in enumerate(counts):
        ob[s, :M] = scenes.make_obstacles(np.random.default_rng(seed + s), M, L, inflated=not shapes, moving=shapes)[:M]
    cnt = np.array(counts, np.int32)
    verts = None
    if shapes:
        h = scenes.add_shape_obstacles(abi.HostBatch(np.zeros((1, 3, 4)), [3], ob, cnt), seed=seed)
        ob, verts = h.obstacles, h.obst_vertices
        ob["dynamic"][:, ::3] = 0
    if gt:
        big = np.zeros((len(counts), GT_ROWS), abi.OBST_DTYPE)
        big["x"], big["y"] = 1000.0, 1000.0
        big[:, :M_cap] = ob
        for s, M in enumerate(counts):
            big[s, M:]["x"], big[s, M:]["y"] = 1000.0, 1000.0
        cnt = np.where(cnt > 0, GT_ROWS, 0).astype(np.int32)
        ob = big
    return ob, cnt, verts


def _batch(cfg, scene_of, n_of, n_cap, counts, gt=False, seed=0):
    """band b of len(scene_of) bands: scene scene_of[b], n_of[b] poses, a lateral amplitude of its own"""
    B = len(scene_of)
    L = 0.4 * 0.3 * (max(n_of) - 1)
    ob, cnt, verts = _tables(cfg, counts, max(L, 1.0), gt, seed)
    poses = np.zeros((B, n_cap, 4))
    rng = np.random.default_rng(seed)
    for b in range(B):
        n = int(n_of[b])
        poses[b, :n] = scenes.make_band(n, rng.uniform(-1.5, 1.5), 0.4, 0.3, length=max(0.4 * 0.3 * (n - 1), 0.5))
    return abi.HostBatch(poses, np.asarray(n_of, np.int32), ob, cnt, np.asarray(scene_of, np.int32), obst_vertices=verts)


def _subset(hb, src):
    sel = lambda a: a[src].copy()
    return abi.HostBatch(sel(hb.poses), sel(hb.n), hb.obstacles, hb.obst_count, sel(hb.scene_id), None, None,
                         sel(hb.vel_start), sel(hb.vel_goal), sel(hb.prefer_rotdir), hb.obst_vertices if hb.PV_cap else None)


def _grids(p, hb, Ks):
    """{K: G} - the grid k_trial_eval2p launches for hb's n_cap, table and footprint, read from the device on a batch of
    2 x SMs + 1 copies of hb's bands, all inactive"""
    B0 = 2 * _sms() + 1
    probe = _subset(hb, np.arange(B0) % hb.B)
    g = _ctx(probe, p)
    out = {}
    try:
        for K in Ks:
            g.eval_trials(probe.copy(), K, 0.0, 1.0, 1.0, _state(B0, active=0))
            build, G = g.last_trial_eval()
            assert build == "eval2p", build
            out[K] = G
    finally:
        g.close()
    return out


def _real_steps(g, hb, K, outer=1, bad_every=3):
    """real LM steps at 1e-5 max diag, every bad_every-th band's scaled by 50 (rejected trials)"""
    Hb, _ = g.build_system(hb, outer)
    base = 1e-5 * R.max_real_diag(Hb, hb.n)
    dx, ok, lam = g.solve_system(hb.n.copy(), K, Hb=Hb, lam=base, nu=np.full(hb.B, 2.0))
    dx = dx.copy()
    dx[::bad_every] *= 50.0
    for b in range(hb.B):
        dx[b, :, 4 * int(hb.n[b]):] = 0.0
    return base, dx, ok, lam


# ------------------------------------------------------------------ one round, against k_trial_eval3 and the oracle
def _round(p, hb, K, dx, ok, lam, st, iteration=1, qmax=None, order=None, build="eval2"):
    g = _ctx(hb, p, build)
    try:
        rd = Round(g, p, hb, K, dx, ok, lam, st, 1, iteration=iteration, qmax=qmax, order=order)
        rd.launch = g.last_trial_eval()
    finally:
        g.close()
    return rd


def _same_outputs(a, b, perm=None):
    """a's outputs of band perm[i] are b's of band i (perm None: the identity)"""
    perm = np.arange(a.hb.B) if perm is None else perm
    for key in ("res", "state", "qmax", "need"):
        x, y = a.out[key][perm], b.out[key]
        assert (_same_bits(x, y) if x.dtype == np.float64 else np.array_equal(x, y)), key
    assert _same_bits(a.after.poses[perm], b.after.poses), "poses"
    assert set(a.out["next_list"].tolist()) == set(perm[b.out["next_list"]].tolist()), "next list"


def _check(name, p, hb, K, dx, ok, lam, st, G, min_slots=3, iteration=1, qmax=None, order=None, no_chi2=()):
    """eval2p against eval3 bit for bit, the decisions of every band and a chi2 sample against the oracle (bands in
    slot >= 2 G, except no_chi2). min_slots: more than that many slots per CTA and a ragged last pass; 0: fewer slots
    than CTAs"""
    rd = _round(p, hb, K, dx, ok, lam, st, iteration, qmax, order)
    build, grid = rd.launch
    slots = hb.B if order is None else len(order)
    assert build == "eval2p" and grid == G, (build, grid, G)
    if min_slots:
        assert slots > min_slots * G and slots % G != 0, f"{slots} slots on {G} CTAs"
    else:
        assert slots < G
    _report(f"eval2p_slots/{name}", f"G {G}, {slots} slots, {slots / G:.2f} per CTA")
    ref = _round(p, hb, K, dx, ok, lam, st, iteration, qmax, order, build="eval3")
    assert ref.launch[0] == "eval3"
    _same_outputs(rd, ref)
    check_decisions(rd, "eval2p", lam_ulps=LAMBDA_ULPS)
    slot = {b: b for b in range(hb.B)} if order is None else {int(b): s for s, b in enumerate(order)}
    late = [b for b in rd.bands() if slot[b] >= 2 * G and b not in no_chi2]
    rng = np.random.default_rng(slots)
    sample = late if len(late) <= CHI2_SAMPLE else sorted(rng.choice(late, CHI2_SAMPLE, replace=False).tolist())
    list(check_chi2(rd, "eval2p", bands=sample))
    return rd


# ------------------------------------------------------------------ a. scenes along a CTA's slots
# scene rows: A = M_cap, B few, C empty, D some; per CTA c (c % 4) the scenes of its slots c, c + G, c + 2G, c + 3G
SCENE_ROWS = [40, 9, 0, 25]
SCENE_PATTERNS = [(0, 0, 0, 0),   # same -> same: no restage
                  (0, 1, 0, 1),   # A -> B -> A, many rows -> few
                  (2, 0, 2, 3),   # empty -> full -> empty
                  (3, 1, 3, 0)]


def _scene_case(cfg, G, gt, n=120, n_cap=150, seed=3):
    B = 3 * G + G // 2 + 1
    scene_of = [SCENE_PATTERNS[(s % G) % 4][s // G] for s in range(B)]
    n_of = [n - (s % 7) for s in range(B)]
    return _batch(cfg, scene_of, n_of, n_cap, SCENE_ROWS, gt, seed)


@pytest.mark.parametrize("cfg,K,gt", [("C3", 2, False), ("shapes_polygon", 6, False), ("C3", 4, True),
                                      ("shapes_polygon", 2, True)])
def test_scene_changes_along_a_ctas_slots(cfg, K, gt):
    p = _params(cfg)
    G = _grids(p, _scene_case(cfg, 4, gt), [K])[K]
    hb = _scene_case(cfg, G, gt)
    g = _ctx(hb, p)
    try:
        base, dx, ok, lam = _real_steps(g, hb, K)
    finally:
        g.close()
    name = f"scenes/{cfg}/K{K}/{'gt' if gt else 'staged'}"
    rd = _check(name, p, hb, K, dx, ok, lam, _state(hb.B, lam=base), G)
    # the batch permuted: other bands share each CTA, every band keeps its bits
    perm = np.random.default_rng(K).permutation(hb.B)
    hp = _subset(hb, perm)
    rp = _round(p, hp, K, dx[perm], ok[perm], lam[perm], _state(hb.B, lam=base[perm]))
    assert rp.launch == rd.launch
    _same_outputs(rd, rp, perm)


# ------------------------------------------------------------------ a. long and short bands in one CTA
SHORT_N = (3, 29, 30, 31)


def test_long_and_short_bands_in_one_cta():
    """n_cap = 512, K = 8 (one CTA per SM): CTA c alternates 512 / 481-pose bands with 3 / 29 / 30 / 31-pose ones,
    long first on even c, short first on odd c; the long bands' last two trials carry NaN / +-1e300 in the rows where
    the next short band ends, so that a short band staged short or reading past its N shows it"""
    K, n_cap = 8, 512
    p = _params("C3")
    probe = _batch("C3", [0, 0], [512, 3], n_cap, [24], seed=5)
    G = _grids(p, probe, [K])[K]
    assert G == _sms(), f"{G} CTAs: the staging of a 512-pose band at K = 8 leaves room for one CTA per SM"
    B = 3 * G + G // 2 + 1
    long_ = lambda s: (s % G) % 2 == (s // G) % 2
    shorts = iter(SHORT_N * B)
    n_of = [(512 if (s // (2 * G)) % 2 == 0 else 481) if long_(s) else next(shorts) for s in range(B)]
    hb = _batch("C3", [0] * B, n_of, n_cap, [24], seed=5)
    g = _ctx(hb, p)
    try:
        base, dx, ok, lam = _real_steps(g, hb, K)
    finally:
        g.close()
    poison = []
    for s in range(B - G):
        if long_(s) and not long_(s + G):
            ns = n_of[s + G]
            lo, hi = 4 * max(ns - 2, 0), 4 * ns + 4
            dx[s, K - 1, lo:hi] = np.nan
            dx[s, K - 2, lo:hi:2], dx[s, K - 2, lo + 1:hi:2] = 1e300, -1e300
            ok[s, K - 2:] = 1.0
            poison.append(s)
    assert len(poison) >= G
    # the poisoned trials' chi2 overflows differently in long double: the oracle's chi2 is checked on the other bands
    rd = _check("ragged_n/C3/K8", p, hb, K, dx, ok, lam, _state(hb.B, lam=base), G, no_chi2=set(poison))
    assert all(np.isnan(rd.out["res"][s, K - 1, :4]).any() for s in poison)


# ------------------------------------------------------------------ a. inactive bands
@pytest.mark.parametrize("cfg,K", [("shapes_polygon", 4), ("C3", 8)])
def test_inactive_bands(cfg, K):
    """every other band inactive; then: CTA 0's first slot, every slot of CTA 1, the last slots and a fifth of the
    rest inactive"""
    p = _params(cfg)
    G = _grids(p, _scene_case(cfg, 4, False), [K])[K]
    hb = _scene_case(cfg, G, False, seed=11)
    g = _ctx(hb, p)
    try:
        base, dx, ok, lam = _real_steps(g, hb, K)
    finally:
        g.close()
    B = hb.B
    act = np.ones(B)
    act[::2] = 0
    _check(f"inactive_every_other/{cfg}/K{K}", p, hb, K, dx, ok, lam, _state(B, lam=base, active=act), G)
    act = (np.random.default_rng(K).random(B) > 0.2).astype(float)
    act[0] = 0
    act[1::G] = 0
    act[B - G // 3:] = 0
    _check(f"inactive_mixed/{cfg}/K{K}", p, hb, K, dx, ok, lam, _state(B, lam=base, active=act), G)


# ------------------------------------------------------------------ a. retry rounds
@pytest.mark.parametrize("cfg,K,gt", [("C3", 6, False), ("C3", 4, True), ("shapes_polygon", 8, False)])
def test_retry_rounds(cfg, K, gt):
    """retry lists in random order over bands with q0 of 4 / 6 / 8 / 9: longer than G (with inactive bands on it),
    shorter than G, empty; bands not on the list keep their all-ones rows"""
    p = _params(cfg)
    G = _grids(p, _scene_case(cfg, 4, gt), [K])[K]
    hb = _scene_case(cfg, G, gt, seed=7)
    B = hb.B
    g = _ctx(hb, p)
    try:
        base, dx, ok, lam = _real_steps(g, hb, K, outer=0)
        lin = g.eval_trials(hb.copy(), 2, dx[:, :2], ok[:, :2], lam[:, :2], _state(B), outer_index=0, iteration=0)["chi_lin"]
    finally:
        g.close()
    rng = np.random.default_rng(K)
    q0 = rng.choice([4, 6, 8, 9], B).astype(np.int32)
    cur = np.array([((c[0] + c[1]) + c[2]) + c[3] for c in lin])
    lam0 = np.array([R.spec_lambda(base[b], 2.0, int(q0[b])) for b in range(B)])
    act = np.ones(B)
    act[rng.choice(B, B // 10, replace=False)] = 0
    st = _state(B, lam=lam0, nu=2.0 ** (q0 + 1), chi=cur, parts_cur=lin, active=act)
    tag = f"{cfg}/K{K}/{'gt' if gt else 'staged'}"
    long_list = rng.permutation(B)[:3 * G + G // 3 + 1].astype(np.int32)
    assert (act[long_list] == 0).any()
    for nm, order, ms in (("long", long_list, 3), ("short", rng.permutation(B)[:G // 2].astype(np.int32), 0),
                          ("empty", np.zeros(0, np.int32), 0)):
        rd = _check(f"retry_{nm}/{tag}", p, hb, K, dx, ok, lam, st, G, min_slots=ms, qmax=q0, order=order)
        listed = set(order.tolist())
        for b in range(B):
            if b not in listed:
                assert (_bits(rd.out["res"][b]) == np.uint64(0xFFFFFFFFFFFFFFFF)).all()


# ------------------------------------------------------------------ b. optimize in the throughput regime
E2E = ["C1_autosize", "C3", "C4", "shapes_polygon", "vor", "padded", "split"]


def _e2e_batch(name, requests):
    if name == "C1_autosize":
        return scenes.make_config_batch("C1", requests=requests, candidates=32, seed=51, autosize=True)
    if name in ("C3", "vor", "padded"):
        p, hb = scenes.make_config_batch("C3", requests=requests, candidates=32, seed=52)
        if name == "vor":
            p.obstacle_poses_affected = 10
            p.weight_velocity_obstacle_ratio = 2.0
            p.obstacle_proximity_lower_bound, p.obstacle_proximity_upper_bound = 0.2, 1.0
        if name == "padded":
            ob = np.zeros((hb.S, GT_ROWS), abi.OBST_DTYPE)
            ob["x"], ob["y"] = 1000.0, 1000.0
            ob[:, :hb.M_cap] = hb.obstacles
            hb = abi.HostBatch(hb.poses, hb.n, ob, np.full(hb.S, GT_ROWS, np.int32), hb.scene_id)
        return p, hb
    if name == "C4":
        return scenes.make_config_batch("C4", requests=requests, candidates=32, seed=53)
    if name == "shapes_polygon":
        p, hb = scenes.make_config_batch("C4", requests=requests, candidates=32, seed=54)
        hb = scenes.add_shape_obstacles(hb, seed=2)
        hb.obstacles["dynamic"][:, ::3] = 0
        scenes.set_polygon_footprint(p)
        return p, hb
    if name == "split":
        return scenes.make_config_batch("C2", requests=requests, candidates=32, seed=55)
    raise KeyError(name)


def _optimize(p, hb0, args, env, monkeypatch):
    """env values None: the variable unset (the default)"""
    for k, v in env.items():
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)
    g = T.TebGpu(hb0.B, hb0.n_cap, hb0.S, max(hb0.M_cap, 1), hb0.V_cap, max_obst_vertices=hb0.PV_cap)
    try:
        g.set_params(p)
        h = hb0.copy()
        g.optimize(h, args)
        return h, g.last_trial_eval()
    finally:
        g.close()


@pytest.mark.parametrize("name", E2E)
def test_optimize_in_the_throughput_regime_matches_eval3(name, monkeypatch):
    p, small = _e2e_batch(name, 1)
    grids = _grids(p, small, (2, 4, 6))
    requests = max(3 * max(grids.values()) // 32 + 2, _sms() * 4 // 8 + 4)
    p, hb0 = _e2e_batch(name, requests)
    assert hb0.B > 3 * max(grids.values()) and hb0.B * 8 > _sms() * 4 * 32   # the {6, 4} / {2, 4, 4} schedule
    _report(f"eval2p_slots/optimize/{name}", f"G {grids}, B {hb0.B}")
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale,
                         p.selection_viapoint_cost_scale, False)
    env = {"TEBGPU_OVERLAP": "1", "TEBGPU_SPLIT": "1"} if name == "split" else {}
    h, launch = _optimize(p, hb0, args, dict(env, TEBGPU_EVAL3=None), monkeypatch)
    assert launch[0] == "eval2p" and launch[1] in grids.values(), launch
    h3, launch3 = _optimize(p, hb0, args, dict(env, TEBGPU_EVAL3="1"), monkeypatch)
    assert launch3[0] == "eval3"
    assert np.array_equal(h.n, h3.n) and np.array_equal(h.status, h3.status) and np.array_equal(h.lm_iters, h3.lm_iters)
    for key in ("poses", "cost", "chi2"):
        assert _same_bits(getattr(h, key), getattr(h3, key)), key
    assert np.all(h.status & abi.TEB_STATUS_OPTIMIZED) and np.all(np.isfinite(h.cost))
    # bands in the last slot of their CTA (at every width), from four scenes, against the oracle
    last = hb0.B - min(grids.values())
    for b in range(hb0.B - 1, last, -41)[:4]:
        ref, cost, _ = O.optimize_band(p, hb0.poses[b], hb0.n[b], args=args, jac_mode=O.JAC_ANALYTIC, n_cap=hb0.n_cap,
                                       **scenarios.band_kwargs(hb0, b))
        assert len(ref) == h.n[b], f"band {b}: n {h.n[b]} vs oracle {len(ref)}"
        assert np.abs(ref - h.poses[b, :h.n[b]]).max() < 1e-6, f"band {b}"
        assert abs(cost - h.cost[b]) <= 1e-6 * max(abs(cost), 1.0), f"band {b}: cost {h.cost[b]} vs {cost}"
