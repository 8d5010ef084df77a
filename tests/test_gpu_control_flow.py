"""The control flow around the kernels: how issue_optimize chains rounds, LM iterations and outer iterations (per-band
BandState, the rotating retry lists, the deferral tags, the side stream's retry rounds and its carried autoResize /
buildGraph / kernel A of the next outer iteration, the split round 0, CUDA-graph capture and replay).

Bands built to take one exit (tests/control_flow_bands.py): Z ends every first LM iteration with ten failed
factorisations (nu = 2^11, Terminate; in the latency regime's {8, 2} schedule the tenth falls in round 1 on the side
stream, so with one inner iteration Z is carried into the next outer iteration), N takes one trial per LM iteration and
never terminates, D is resized once and disabled, P ends each outer iteration on rho == 0 after one trial, and S takes
Z's exit in the first outer iteration while the carried autoResize still changes it. Warm-started converged bands (the output of a 1 x 30 run fed back,
as a planner does every cycle) are compared on their poses only: their decisions are near-ties.

Checked against the oracle at the argument edges of optimizeTEB (no outer / no inner iteration), and every switch that
is meant to change only the schedule against every other, bit for bit, in one latency-regime batch (32 bands) and one
throughput batch (> 2112 bands on the 132 SMs of an H100)."""
import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi
from tests import control_flow_bands as cf

pytestmark = pytest.mark.gpu
NU_TEN_REJECTIONS = 2.0 ** 11
LAT_KINDS = ["Z", "N", "O", "S", "W", "W", "N", "O"] * 4            # 32 bands; N directly before healthy bands
THROUGHPUT_REPS = 67                                                  # 67 x 32 = 2144 bands


def _gpu(hb, p, max_obstacles=None, **switches):
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, max_obstacles or max(hb.M_cap, 1), hb.V_cap, max_obst_vertices=hb.PV_cap)
    g.set_params(p)
    for name, v in switches.items():
        getattr(g, "set_" + name)(v)
    return g


def _run(hb, p, a, env=None, monkeypatch=None, max_obstacles=None, **switches):
    """one optimize on a fresh context -> (batch after the call, band-state read-back)"""
    if env:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
    g = _gpu(hb, p, max_obstacles, **switches)
    h = hb.copy()
    g.optimize(h, a)
    st = g.band_state(h.B)
    g.close()
    if env:
        for k in env:
            monkeypatch.delenv(k)
    return h, st


def _bit_equal(x, y, bands=None):
    """n, poses, cost, chi2, status, lm_iters and the band state of two runs are identical (NaN where NaN)"""
    (ha, sa), (hb, sb) = x, y
    sel = slice(None) if bands is None else bands
    pairs = [(ha.n, hb.n), (ha.status, hb.status), (ha.lm_iters, hb.lm_iters), (ha.poses, hb.poses), (ha.cost, hb.cost),
             (ha.chi2, hb.chi2), (sa, sb)]
    return all(np.array_equal(u[sel], v[sel], equal_nan=True) for u, v in pairs)


def _warm_bands(p, count, seed=9):
    """ordinary bands after a 1 x 30 optimize on the device: what a planner feeds back every cycle"""
    hb = cf.ordinary_batch(candidates=count, seed=seed)
    g = _gpu(hb, p)
    g.optimize(hb, cf.args(30, 1))
    g.close()
    return hb


def _batch(p, oracle, kinds, reps=1):
    """the kinds of LAT_KINDS ('W' a warm-started band), replicated `reps` times"""
    hb = cf.mixed_batch([k if k != "W" else "O" for k in kinds] * reps, s_band=cf.shifting_band(p, oracle))
    w = _warm_bands(p, sum(k == "W" for k in kinds), seed=9)
    j = 0
    for b, k in enumerate(kinds * reps):
        if k == "W":
            cf.set_band(hb, b, w.poses[j % w.B], int(w.n[j % w.B]))
            j += 1
    return hb


def _check_oracle(oracle, p, hb, a, h, st, bands, kinds, pose_tol=1e-6):
    """the device result of `bands` against the oracle with the device's Jacobians"""
    for b in bands:
        ro, co, so = oracle.optimize_band(p, hb.poses[b], int(hb.n[b]), args=a, jac_mode=oracle.JAC_ANALYTIC,
                                          n_cap=hb.n_cap, **cf.band_kwargs(hb, b))
        kind = kinds[b % len(kinds)]
        where = (b, kind)
        assert h.n[b] == len(ro), where
        d = np.abs(h.poses[b, :h.n[b]] - ro)
        assert np.array_equal(np.isnan(h.poses[b, :h.n[b]]), np.isnan(ro)) and np.nanmax(d, initial=0) <= pose_tol, where
        if kind in "WS":
            continue   # warm-started bands and S once resized converge to chi2 ~ 1e-25: their decisions are ties
        assert h.status[b] == so.status and h.lm_iters[b] == so.lm_iters, (where, h.status[b], so.status)
        if so.lm_iters:
            assert st[b, 1] == so.nu_final, where
            if kind in "ZND":
                assert st[b, 0] == so.lambda_final, where
            else:   # lambda multiplies the accept factors of every LM iteration: it carries their round-off
                assert abs(st[b, 0] - so.lambda_final) <= 1e-6 * abs(so.lambda_final), where
        for mine, theirs in ((h.cost[b], co), (h.chi2[b], so.chi2_final)):
            assert (np.isnan(mine) and np.isnan(theirs)) or mine == theirs or abs(mine - theirs) <= 1e-6 * abs(theirs) + 1e-12, where


# ------------------------------------------------------------------------------------------------ argument edges
@pytest.mark.parametrize("autosize", [True, False])
@pytest.mark.parametrize("outer,inner", cf.EDGES)
def test_argument_edges_match_oracle(oracle, outer, inner, autosize):
    """Z, N, ordinary bands and a band a second autoResize pass would change, at no outer / no inner iteration and
    around: n, status, lm_iters, nu exact, lambda exact on Z / N and 1e-6 elsewhere, poses 1e-6, cost and chi2 1e-6
    (1e-12 absolute near 0) or the same inf / NaN - with graph replay and without"""
    p = cf.params(autosize)
    kinds = ["Z", "N", "O", "O", "O", "R"]
    hb = cf.mixed_batch(kinds[:5] + ["O"])
    rec, n = cf.resize_twice_band(p, oracle.auto_resize)
    cf.set_band(hb, 5, rec, n)
    a = cf.args(inner, outer)
    runs = [_run(hb, p, a, graph=m) for m in (0, 1)]
    assert _bit_equal(*runs)
    h, st = runs[0]
    _check_oracle(oracle, p, hb, a, h, st, range(hb.B), kinds)
    if outer > 0 and inner == 0:
        assert not (h.status & abi.TEB_STATUS_OPTIMIZED).any() and np.isinf(h.cost).all() and not h.lm_iters.any()
        if autosize:    # autoResize ran once: a second pass would have moved R
            once = oracle.auto_resize(rec, n, p.dt_ref, p.dt_hysteresis, p.min_samples, p.max_samples, 1)
            assert np.array_equal(h.poses[5, :h.n[5]], once)
    if outer == 0:
        assert (h.status == abi.TEB_STATUS_OPTIMIZED).all() and np.isinf(h.cost).all()
        assert np.array_equal(h.poses, hb.poses, equal_nan=True)
    if outer > 0 and inner > 0:
        assert h.lm_iters[0] == outer and st[0, 1] == NU_TEN_REJECTIONS and h.cost[0] == 0.0
        assert h.lm_iters[1] == outer * inner and h.status[1] == abi.TEB_STATUS_OPTIMIZED | abi.TEB_STATUS_CHOL_FAILED
    # P: rho == 0 on the first trial of every outer iteration (needs the shortest-path edges: a batch of its own)
    pp = cf.params(autosize, shortest_path=True)
    hp = cf.mixed_batch(["P", "O", "O"])
    runs = [_run(hp, pp, a, graph=m) for m in (0, 1)]
    assert _bit_equal(*runs)
    h, st = runs[0]
    _check_oracle(oracle, pp, hp, a, h, st, range(hp.B), ["P", "O", "O"])
    if outer > 0 and inner > 0:
        assert h.lm_iters[0] == outer and st[0, 1] == 4.0 and st[0, 0] > 0
        assert h.status[0] == abi.TEB_STATUS_OPTIMIZED | abi.TEB_STATUS_TERMINATED


def test_constructed_bands_are_what_they_claim(oracle):
    """Z's system is exactly zero on the device as in the oracle; N's chi2 is NaN"""
    p = cf.params()
    hb = cf.mixed_batch(["Z", "N"])
    g = _gpu(hb, p)
    Hb, chi2 = g.build_system(hb)
    lin = g.linearize_outputs(hb.B, hb.n_cap)
    g.close()
    assert chi2[0] == 0.0 and not lin["rhs"][0].any() and lin["dmax_parts"][0].max() == 0.0
    assert np.isnan(chi2[1])


@pytest.mark.parametrize("outer,inner", cf.EDGES)
def test_disabled_band_resized_once(oracle, outer, inner):
    p = cf.params()
    p.max_vel_x = 0.005
    hb = cf.mixed_batch(["O", "O"])
    for b in range(2):
        cf.set_band(hb, b, cf.d_band(20 + b, hb.n_cap), 20 + b)
    a = cf.args(inner, outer)
    h, st = _run(hb, p, a)
    _check_oracle(oracle, p, hb, a, h, st, range(2), ["D"])
    assert np.isinf(h.cost).all() and not h.lm_iters.any()
    if outer:
        assert (h.status == abi.TEB_STATUS_DISABLED).all() and (h.n > hb.n).all()


# ------------------------------------------------------------------------------------------------ coverage
@pytest.mark.parametrize("regime", ["latency", "throughput"])
@pytest.mark.parametrize("inner", [1, 2])
def test_carried_boundaries(oracle, regime, inner):
    """optimize is prefix-consistent in the outer loop, so the band state after an outer-prefix run is the state at the
    end of that outer iteration of the full run. Z and S end the first outer iteration with ten rejections; in the
    latency regime the tenth falls in round 1 on the side stream, so at inner = 1 they are carried: the side stream runs
    the next outer iteration's autoResize / buildGraph / kernel A for them. For S that autoResize changes the band, and
    S's result after two and four outer iterations must be the oracle's. Warm-started bands are counted, not asserted:
    in these batches they end no LM iteration with ten rejections."""
    p = cf.params()
    reps = 1 if regime == "latency" else THROUGHPUT_REPS
    hb = _batch(p, oracle, LAT_KINDS, reps)
    kinds = LAT_KINDS * reps
    z, s_ = (np.array([k == c for k in kinds]) for c in "ZS")
    warm = np.array([k in "WO" for k in kinds])
    h1, st1 = _run(hb, p, cf.args(inner, 1))
    carried = st1[:, 1] == NU_TEN_REJECTIONS
    assert carried[z | s_].all() and int(carried[z | s_].sum()) == 8 * reps
    counts = [int((carried & warm).sum())]
    for o in (2, 3):
        h, st = _run(hb, p, cf.args(inner, o))
        assert (st[z, 1] == NU_TEN_REJECTIONS).all()
        counts.append(int(((st[:, 1] == NU_TEN_REJECTIONS) & warm).sum()))
        if o == 2:
            one_s = np.flatnonzero(s_)[:4]
            _check_oracle(oracle, p, hb, cf.args(inner, 2), h, st, one_s, LAT_KINDS)
            twice = hb.poses[one_s[0], :hb.n[one_s[0]]]
            for _ in range(2):
                twice = oracle.auto_resize(twice, len(twice), p.dt_ref, p.dt_hysteresis, p.min_samples, p.max_samples, 1)
            assert h.n[one_s[0]] == len(twice)
    print(f"{regime} inner={inner}: carried out of outer 1: Z + S {int(carried[z | s_].sum())}; "
          f"warm / ordinary bands with ten rejections at outer 1..3: {counts}")
    h, st = _run(hb, p, cf.args(inner, 4))
    sample = range(hb.B) if regime == "latency" else list(range(32)) + list(range(hb.B - 32, hb.B))
    _check_oracle(oracle, p, hb, cf.args(inner, 4), h, st, sample, LAT_KINDS)


# ------------------------------------------------------------------------------------------------ schedule matrix
SCHEDULES = {
    "graph_off": dict(graph=0), "graph_on": dict(graph=1),
    "overlap_off": dict(env={"TEBGPU_OVERLAP": "0"}), "overlap_on": dict(env={"TEBGPU_OVERLAP": "1"}),
    "split": dict(env={"TEBGPU_OVERLAP": "1", "TEBGPU_SPLIT": "1"}),
    "k2": dict(speculation=2), "k4": dict(speculation=4), "k8": dict(speculation=8),
    "eval3": dict(env={"TEBGPU_EVAL3": "1"}), "ka_oneshot": dict(env={"TEBGPU_KA_PERSIST": "0"}),
}
TPB_FORMS = {f"form{f}": dict(warp_solver=0, solve_form=f) for f in (1, 11, 22, 33)}
TPB_FORMS["warp1"] = dict(warp_solver=1)


def _pad_scene(hb, rows=1100):
    """the same scene with rows far outside every threshold appended past 1024 (the global-table path)"""
    obst = np.zeros((hb.S, rows), abi.OBST_DTYPE)
    obst[:, :hb.M_cap] = hb.obstacles
    obst[:, hb.M_cap:]["x"] = np.linspace(-500, 500, rows - hb.M_cap)
    obst[:, hb.M_cap:]["y"] = -1000.0
    return abi.HostBatch(hb.poses.copy(), hb.n.copy(), obst, np.full(hb.S, rows, np.int32), hb.scene_id.copy(),
                         None, None, hb.vel_start.copy(), hb.vel_goal.copy(), hb.prefer_rotdir.copy())


@pytest.mark.parametrize("regime", ["latency", "throughput"])
def test_every_schedule_gives_the_same_bits(oracle, regime, monkeypatch):
    p = cf.params()
    reps = 1 if regime == "latency" else THROUGHPUT_REPS
    hb = _batch(p, oracle, LAT_KINDS, reps)
    kinds = LAT_KINDS * reps
    a = cf.args(1, 4)
    # the throughput regime's retry rounds launch k_solve_lat and k_solve_tpb and let the list length pick one, so
    # which elimination order a band gets depends on the schedule there: its schedules are compared on k_solve_tpb
    fixed = {} if regime == "latency" else dict(warp_solver=0)
    base = _run(hb, p, a, **fixed)
    for name, sw in SCHEDULES.items():
        assert _bit_equal(base, _run(hb, p, a, monkeypatch=monkeypatch, **dict(fixed, **sw))), name
    # the thread-per-system solve in every form and the warp solve eliminate in the same order
    tpb = _run(hb, p, a, warp_solver=0)
    for name, sw in TPB_FORMS.items():
        assert _bit_equal(tpb, _run(hb, p, a, **sw)), name
    auto = _run(hb, p, a)
    # k_solve_lat (the default's solve while a round fits three waves of CTAs) eliminates in another order: the same
    # control flow on the constructed bands, poses within 1e-8
    zn = np.array([k in "ZN" for k in kinds])
    (h0, s0), (h1, s1) = auto, tpb
    assert np.array_equal(h0.lm_iters[zn], h1.lm_iters[zn]) and np.array_equal(h0.status[zn], h1.status[zn])
    assert np.array_equal(s0[zn][:, 1], s1[zn][:, 1])
    assert np.nanmax(np.abs(h0.poses[zn] - h1.poses[zn]), initial=0) <= 1e-8
    padded = _run(_pad_scene(hb), p, a, max_obstacles=1100, **fixed)
    assert _bit_equal(base, padded), "scene padded past 1024 rows"
    h, st = base
    sample = range(hb.B) if regime == "latency" else list(range(32)) + list(range(hb.B - 32, hb.B))
    _check_oracle(oracle, p, hb, a, h, st, sample, LAT_KINDS)


@pytest.mark.parametrize("regime", ["latency", "throughput"])
def test_healthy_bands_do_not_see_nan_neighbours(oracle, regime):
    """every healthy band is bit-equal to the same batch with the N bands replaced by copies of healthy ones"""
    p = cf.params()
    reps = 1 if regime == "latency" else THROUGHPUT_REPS
    hb = _batch(p, oracle, LAT_KINDS, reps)
    kinds = LAT_KINDS * reps
    clean = hb.copy()
    for b, k in enumerate(kinds):
        if k == "N":
            cf.set_band(clean, b, cf.z_band(40, hb.n_cap), 40, cf.Z_VEL4)
    healthy = np.array([k != "N" for k in kinds])
    for inner, outer in ((1, 4), (5, 2)):
        assert _bit_equal(_run(hb, p, cf.args(inner, outer)), _run(clean, p, cf.args(inner, outer)), healthy), (inner, outer)


# ------------------------------------------------------------------------------------------------ graph replay
def _requests(p):
    """three requests of the same dimensions: poses, n, obstacle rows / counts, scene ids and via counts change"""
    out = []
    for r in range(3):
        base = cf.mixed_batch(["O"] * 10 + ["Z", "N"], seed=20 + r)
        obst = np.zeros((2, 16), abi.OBST_DTYPE)
        obst[0] = base.obstacles[0]
        obst[1] = cf.ordinary_batch(seed=40 + r).obstacles[0]
        counts = np.array([16 - 3 * r, 9 + r], np.int32)
        via = np.zeros((12, 3, 2))
        via[:, :, 0] = np.linspace(-1.0, 1.5, 3)
        hb = abi.HostBatch(base.poses.copy(), base.n.copy() - np.array([r] * 10 + [0, 0], np.int32), obst, counts,
                           np.array([(b + r) % 2 for b in range(12)], np.int32), via, np.full(12, r, np.int32),
                           base.vel_start.copy(), base.vel_goal.copy())
        hb.poses[:10, :, 1] *= 1.0 + 0.1 * r
        hb.poses[np.arange(12), hb.n - 1, 3] = 0.0
        out.append(hb)
    return out


def test_graph_replay_across_requests(monkeypatch):
    """one captured graph replayed on three requests of the same dimensions equals a graph-off run each time, through
    the host entry point and through the device entry point with the same device buffers refilled"""
    import torch
    p = cf.params()
    p.weight_viapoint = 1.0
    a = cf.args(2, 3)
    reqs = _requests(p)
    g = _gpu(reqs[0], p, graph=1)
    for hb in reqs:
        h = hb.copy()
        g.optimize(h, a)
        assert _bit_equal((h, g.band_state(h.B)), _run(hb, p, a, graph=0))
    assert g.info(6) == 1
    dev = torch.device("cuda:0")
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).reshape(-1).copy()).to(dev)
    h0 = reqs[0]
    bufs = dict(poses=t(h0.poses), n=t(h0.n), scene_id=t(h0.scene_id), obstacles=t(h0.obstacles), obst_count=t(h0.obst_count),
                via=t(h0.via), via_count=t(h0.via_count), vel_start=t(h0.vel_start), vel_goal=t(h0.vel_goal),
                prefer_rotdir=t(h0.prefer_rotdir), cost=t(np.zeros(h0.B)), chi2=t(np.zeros(h0.B)),
                status=t(np.zeros(h0.B, np.int32)), lm_iters=t(np.zeros(h0.B, np.int32)))
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = h0.B, h0.n_cap, h0.S, h0.M_cap, h0.V_cap, 0
    for k, v in bufs.items():
        setattr(bs, k, v.data_ptr())
    for hb in reqs:
        for k in ("poses", "n", "scene_id", "obstacles", "obst_count", "via", "via_count", "vel_start", "vel_goal"):
            bufs[k].copy_(t(getattr(hb, k)))
        g.optimize_device(bs, a)
        g.synchronize()
        back = lambda k, like: bufs[k].cpu().numpy().view(like.dtype).reshape(like.shape)
        h = hb.copy()
        h.poses[:], h.n[:], h.cost[:], h.chi2[:] = back("poses", hb.poses), back("n", hb.n), back("cost", hb.cost), back("chi2", hb.chi2)
        h.status[:], h.lm_iters[:] = back("status", hb.status), back("lm_iters", hb.lm_iters)
        assert _bit_equal((h, g.band_state(h.B)), _run(hb, p, a, graph=0))
    assert g.info(6) == 2
    g.close()
