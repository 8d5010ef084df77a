"""The persistent kernel A (k_linearize2p, the default) against the one-shot k_linearize2 (TEBGPU_KA_PERSIST=0), bit for
bit, through tebgpu_build_system_graph (run on an H100: pytest -m gpu).

k_linearize2p runs k_linearize2's per-pose arithmetic unchanged; only the schedule differs (one-warp CTAs take
(band slot, 29-pose tile) units round robin, double-buffer the next unit's pose window, drain the previous unit's bulk
stores while the current one runs P1). So every output must be the same bits: H|b, rhs, the chi2 and max-diagonal tile
partials, the graph words, and the all-ones pattern of whatever neither build wrote. Cases: every scenario, kernel A's
tile edges, holonomic and vertex-list builds, scenes padded past 1024 rows (the global-table build), listed launches
(the retry side stream's form) in any order, empty and full, inactive bands, and batches where the test reads G from
the context and every warp takes at least three units, the last pass ragged, with scene changes along a warp's units.
Optimize runs where the split schedule defers bands (skip_tag) must give the same bits as well.
"""
import os

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import scenarios
from tests.test_gpu_linearize import NS, _ones, _padded, _same, _shape_batch, _shape_params

pytestmark = pytest.mark.gpu


def _ctx(hb, p, persist, max_bands=None):
    old = os.environ.get("TEBGPU_KA_PERSIST")
    os.environ["TEBGPU_KA_PERSIST"] = "1" if persist else "0"
    try:
        g = T.TebGpu(max_bands or hb.B, hb.n_cap, hb.S, max(hb.M_cap, 1), hb.V_cap, max_obst_vertices=hb.PV_cap)
    finally:
        if old is None:
            del os.environ["TEBGPU_KA_PERSIST"]
        else:
            os.environ["TEBGPU_KA_PERSIST"] = old
    g.set_params(p)
    return g


def _run(g, hb, outer, bands=None):
    out = g.build_system(hb, outer, bands=bands, graph=True)
    out.update(g.linearize_outputs(hb.B, hb.n_cap))
    return out


def _compare(hb, p, outers=(1,), lists=(None,), max_bands=None):
    """every output of both builds, bit for bit; returns the persistent build's (build, grid) of the last launch"""
    gp, go = _ctx(hb, p, True, max_bands), _ctx(hb, p, False, max_bands)
    try:
        for outer in outers:
            for lst in lists:
                a, b = _run(gp, hb, outer, lst), _run(go, hb, outer, lst)
                assert gp.last_linearize()[0] == "persistent" and go.last_linearize()[0] == "oneshot"
                for k in a:
                    assert _same(a[k], b[k]), f"outer {outer}, list {lst}: {k} differs"
        return gp.last_linearize()
    finally:
        gp.close()
        go.close()


@pytest.mark.parametrize("name", scenarios.ALL)
def test_every_scenario_is_bit_identical(name):
    p, hb = scenarios.scenario(name)
    _compare(hb, p, outers=(0, 3))


def test_tile_edges_are_bit_identical():
    p = _shape_params()
    for delta in (0, 1, 3):
        for n in NS:
            if n + delta <= 512:
                _compare(_shape_batch([n], n + delta), p)
    _compare(_shape_batch(NS, 512, two_scenes=True), p)


@pytest.mark.parametrize("name", ["C3", "holonomic", "shapes_polygon", "legacy"])
def test_global_table_is_bit_identical(name):
    p, hb = scenarios.scenario(name, candidates=5)
    big = _padded(hb, 1100)
    assert big.M_cap > 1024
    _compare(big, p, lists=(None, [3, 1], []))


@pytest.mark.parametrize("name", ["C2", "via_ordered", "shapes_polygon", "holonomic"])
def test_listed_launches_are_bit_identical(name):
    p, hb = scenarios.scenario(name, candidates=6)
    rng = np.random.default_rng(len(name))
    lists = [[], list(range(hb.B)), list(range(hb.B))[::-1], [int(hb.B - 1), 0], [int(x) for x in rng.permutation(hb.B)[:3]]]
    _compare(hb, p, lists=lists)


def _many_units_batch(G, n_cap=512, seed=0):
    """a batch whose units fill G warps at least 3 x over with a ragged last pass: mostly full bands, some short ones
    (tiles past n skipped), some below min_samples (inactive), scenes in random order along every warp's units"""
    rng = np.random.default_rng(seed)
    ns, live = [], 0
    while live < 3 * G + G // 3 or live % G == 0:   # units with work, the 4-pose bands being inactive
        n = int(rng.choice([n_cap, n_cap, n_cap, n_cap - 1, 465, 300, 117, 4]))
        ns.append(n)
        live += (n + 28) // 29 if n > 4 else 0
    B = len(ns)
    hb = _shape_batch([int(x) for x in ns], n_cap, two_scenes=True, seed=seed)
    sid = rng.integers(0, 2, B).astype(np.int32)
    return abi.HostBatch(hb.poses, hb.n, hb.obstacles, hb.obst_count, sid, hb.via, hb.via_count)


def _grid(p):
    """G of the persistent build, read from the context after a launch with more units than resident warps"""
    hb = _shape_batch([512] * 200, 512)
    g = _ctx(hb, p, True)
    try:
        g.build_system(hb, 1, graph=True)
        build, G = g.last_linearize()
    finally:
        g.close()
    assert build == "persistent" and 0 < G < 200 * 18
    return G


def _units_per_warp(hb, G, p):
    live = 0
    for b in range(hb.B):
        n = int(hb.n[b])
        if n >= max(3, p.min_samples):
            live += (n + 28) // 29
    return live / G


def test_every_warp_takes_several_units():
    p = _shape_params()
    p.min_samples = 5                          # the 4-pose bands are inactive
    G = _grid(p)
    for seed in (0, 1):
        hb = _many_units_batch(G, seed=seed)
        assert _units_per_warp(hb, G, p) >= 3.0, "the batch must give every warp at least three units"
        assert round(_units_per_warp(hb, G, p) * G) % G != 0
        build, grid = _compare(hb, p)
        assert (build, grid) == ("persistent", G)
        # and as a listed launch over a permutation of most bands
        lst = [int(x) for x in np.random.default_rng(seed).permutation(hb.B)[: hb.B - 5]]
        _compare(hb, p, lists=(lst,))


def test_inactive_bands_keep_the_all_ones_pattern():
    p = _shape_params()
    p.min_samples = 10
    hb = _shape_batch([40, 5, 9, 120, 3, 64], 128)
    gp = _ctx(hb, p, True)
    try:
        out = _run(gp, hb, 1)
    finally:
        gp.close()
    for b in (1, 2, 4):
        assert _ones(out["Hb"][b]) and _ones(out["rhs"][b]) and _ones(out["chi_parts"][b]) and _ones(out["dmax_parts"][b])
    _compare(hb, p)


def _optimize(hb, p, persist, args, overlap, monkeypatch):
    with monkeypatch.context() as m:
        m.setenv("TEBGPU_OVERLAP", "1" if overlap else "0")
        m.setenv("TEBGPU_SPLIT", "1")
        g = _ctx(hb, p, persist)
    try:
        h = hb.copy()
        g.optimize(h, args)
        return h, g.last_linearize(), g.launch_count()
    finally:
        g.close()


def test_optimize_with_deferred_bands_is_bit_identical(monkeypatch):
    """with the retry rounds on the side stream (TEBGPU_OVERLAP=1) and the split round 0 (TEBGPU_SPLIT=1), the bands
    that needed retry rounds are deferred: the next kernel A on the main stream skips them by skip_tag and the side
    stream runs it for them from a band list. Same bits with either build, and the same bits as one stream."""
    n, M, cand, inflated, moving, via_pts = scenes.CONFIG_SHAPES["C3"]
    p = scenes.config_params("C3")
    p.teb_autosize = 0
    hb = scenes.make_batch(n, M, 32, 80, seed=1000, inflated=inflated, moving=moving, via_points=via_pts)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale,
                         p.selection_viapoint_cost_scale, False)
    a, la, ca = _optimize(hb, p, True, args, True, monkeypatch)
    b, lb, cb = _optimize(hb, p, False, args, True, monkeypatch)
    c, lc, cc = _optimize(hb, p, True, args, False, monkeypatch)
    assert la[0] == "persistent" and lb[0] == "oneshot" and lc[0] == "persistent"
    # the side stream ran: its listed kernel-A launches and its share of round 0 add to the one-stream count
    assert ca == cb and ca > cc, (ca, cb, cc)
    for k in ("poses", "n", "cost", "chi2", "status", "lm_iters"):
        assert _same(getattr(a, k), getattr(b, k)), k
        assert _same(getattr(a, k), getattr(c, k)), k
