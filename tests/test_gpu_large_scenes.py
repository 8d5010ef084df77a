"""Scenes of more than 1024 obstacles (run on an H100: pytest -m gpu). Batches of M_cap 1025 .. 16384 run the
global-table instantiations of the default kernels (obstacle rows read from global memory, associations walked via
the occupancy words); M_cap <= 1024 keeps the staged kernels.

  * same bits on both paths: every scenario padded past 1024 rows with static points 1000 m away (never associated,
    exactly zero terms under the legacy association), real rows first or moved to indices >= 2048
  * oracle parity at 2000 / 4096 / 16384 costmap-like obstacles: kernel A at 1e-12, optimizeTEB at 1e-6 per pose
    component with identical n, LM iterations and status
  * association edge cases (equal distances, obstacles exactly at force_d / cut_d) against the oracle at 1e-12
  * the contract: limits, unsupported modes, BAD_INPUT from a row past index 1024
"""
import os

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests.scenarios import ALL, scenario

pytestmark = pytest.mark.gpu
PAD_AT = 1000.0


def _gpu(hb, p, max_obstacles=None):
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, max_obstacles or max(hb.M_cap, 1), hb.V_cap, max_obst_vertices=hb.PV_cap)
    g.set_params(p)
    return g


def _args(p):
    return abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale,
                         p.selection_viapoint_cost_scale, False)


def _padded(hb, M_cap, real_at):
    """hb with every scene padded to M_cap rows: static points PAD_AT m away, real rows at real_at .. real_at + M"""
    ob = np.zeros((hb.S, M_cap), abi.OBST_DTYPE)
    ob["x"], ob["y"] = PAD_AT, PAD_AT
    cnt = np.zeros(hb.S, np.int32)
    for s in range(hb.S):
        M = int(hb.obst_count[s])
        ob[s, real_at:real_at + M] = hb.obstacles[s, :M]
        cnt[s] = M_cap
    return abi.HostBatch(hb.poses.copy(), hb.n.copy(), ob, cnt, hb.scene_id.copy(),
                         hb.via.copy() if hb.V_cap else None, hb.via_count.copy() if hb.V_cap else None,
                         hb.vel_start.copy(), hb.vel_goal.copy(), hb.prefer_rotdir.copy(),
                         hb.obst_vertices.copy() if hb.PV_cap else None)


def _same(a, b):
    for f in ("poses", "n", "cost", "chi2", "status", "lm_iters"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


@pytest.mark.parametrize("layout", ["real_first", "real_last"])
@pytest.mark.parametrize("name", ALL)
def test_padded_scene_gives_the_same_bits_on_both_paths(name, layout):
    p, hb0 = scenario(name)
    # real_first: M_cap 1100 (MW = 18, one occupancy word); real_last: real rows from index 2048 (high mask words and
    # occupancy bits), M_cap 2048 + M
    big = _padded(hb0, 1100, 0) if layout == "real_first" else _padded(hb0, 2048 + int(hb0.M_cap), 2048)
    assert big.M_cap > 1024
    args = _args(p)
    gs, gg = _gpu(hb0, p), _gpu(big, p)
    # kernel A + association
    for outer in (0, 2):
        Hs, cs = gs.build_system(hb0, outer)
        Hg, cg = gg.build_system(big, outer)
        assert np.array_equal(Hs, Hg) and np.array_equal(cs, cg)
    # the automatic latency path (graph captured, then replayed) and the thread-per-system solver
    for mode in ("auto", "tpb"):
        if mode == "tpb":
            gs.set_warp_solver(0)
            gg.set_warp_solver(0)
        for _ in range(2 if mode == "auto" else 1):
            hs, hg = hb0.copy(), big.copy()
            gs.optimize(hs, args)
            gg.optimize(hg, args)
            _same(hs, hg)
    gs.close()
    gg.close()


def _kernel_a_vs_oracle(oracle, p, hb, outer_index=1):
    g = _gpu(hb, p)
    Hb, chi2 = g.build_system(hb, outer_index)
    g.close()
    for b in range(hb.B):
        n = hb.n[b]
        kw = dict(obst_vertices=hb.obst_vertices[0] if hb.PV_cap else None, vel_start=hb.vel_start[b],
                  vel_goal=hb.vel_goal[b])
        Hd, bd, c2 = oracle.build_system(p, hb.poses[b], n, hb.obstacles[0][:hb.obst_count[0]],
                                         weight_multiplier=2.0 ** outer_index, jac_mode=oracle.JAC_ANALYTIC, **kw)
        N = 4 * n - 7
        ref = np.zeros((4 * n, 12))
        ref[:, 0] = 1.0
        for r in range(N):
            for k in range(min(r, 10) + 1):
                ref[r + 3, k] = Hd[r, r - k]
            ref[r + 3, 11] = bd[r]
        got = Hb[b, :4 * n]
        assert np.abs(got[:, :11] - ref[:, :11]).max() <= 1e-12 * np.abs(ref[:, :11]).max()
        assert np.abs(got[:, 11] - ref[:, 11]).max() <= 1e-12 * max(np.abs(ref[:, 11]).max(), 1.0)
        assert abs(chi2[b] - c2) <= 1e-12 * max(c2, 1.0)


MODES = ["nonlegacy", "legacy", "vor"]


def _mode(p, mode):
    if mode == "legacy":
        p.legacy_obstacle_association, p.obstacle_poses_affected = 1, 10
    elif mode == "vor":
        p.weight_velocity_obstacle_ratio = 2.0
        p.obstacle_proximity_lower_bound, p.obstacle_proximity_upper_bound = 0.2, 1.0
    return p


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M", [2000, 4096, 16384])
def test_large_scene_matches_oracle(oracle, M, mode):
    p, hb0 = scenes.costmap_scene(M, candidates=3, seed=M)
    p = _mode(p, mode)
    _kernel_a_vs_oracle(oracle, p, hb0)
    args = _args(p)
    g = _gpu(hb0, p)
    hg = hb0.copy()
    g.optimize(hg, args)
    g.close()
    ha = hb0.copy()
    oracle.optimize_batch(p, ha, args, jac_mode=oracle.JAC_ANALYTIC, threads=8)
    assert np.array_equal(hg.n, ha.n)
    assert np.array_equal(hg.lm_iters, ha.lm_iters) and np.array_equal(hg.status, ha.status)
    for b in range(hg.B):
        assert np.abs(hg.poses[b, :hg.n[b]] - ha.poses[b, :ha.n[b]]).max() < 1e-6
    assert np.allclose(hg.cost, ha.cost, rtol=1e-6)


def _edge_scene(real_at):
    """a straight band on exact binary coordinates; beside several poses: five copies of one point (equal distances),
    points exactly at force_d = 0.75 and at cut_d = 2.5 on either side; padded past 1024 rows"""
    p = scenes.config_params("C2")
    n = 29
    rec = np.zeros((1, n, 4))
    rec[0, :, 0] = -3.5 + 0.25 * np.arange(n)
    rec[0, :-1, 3] = 0.625
    rows = []
    for i in (3, 8, 14, 20, 25):
        x = rec[0, i, 0]
        rows += [(x, 1.0)] * 5 + [(x, -1.25)] * 5       # closest on either side for i >= 14: the lowest index wins
        if i < 14:
            rows += [(x, 0.75), (x, -0.75), (x, 2.5), (x, -2.5), (x + 0.25, 0.75)]
    M = len(rows)
    ob = np.zeros(real_at + M, abi.OBST_DTYPE)
    ob["x"], ob["y"] = PAD_AT, PAD_AT
    ob["x"][real_at:], ob["y"][real_at:] = [r[0] for r in rows], [r[1] for r in rows]
    if real_at + M <= 1024:
        ob = np.concatenate([ob, np.zeros(1100 - len(ob), abi.OBST_DTYPE)])
        ob["x"][real_at + M:], ob["y"][real_at + M:] = PAD_AT, PAD_AT
    hb = abi.HostBatch(rec, np.array([n], np.int32), ob, np.array([len(ob)], np.int32))
    return p, hb


@pytest.mark.parametrize("legacy", [False, True])
@pytest.mark.parametrize("real_at", [0, 1500])
def test_association_edge_cases_match_oracle(oracle, legacy, real_at):
    p, hb = _edge_scene(real_at)
    assert hb.M_cap > 1024
    if legacy:
        p.legacy_obstacle_association, p.obstacle_poses_affected = 1, 6
    _kernel_a_vs_oracle(oracle, p, hb, outer_index=0)


def test_limits_and_unsupported_modes():
    p, hb = scenes.costmap_scene(64, candidates=2, seed=3)
    T.TebGpu(2, 100, 1, 16384, 0).close()
    with pytest.raises(T.TebGpuError):
        T.TebGpu(2, 100, 1, 16385, 0)
    # a 16384-capable context runs a 64-obstacle batch through the unchanged staged path
    args = _args(p)
    ga, gb = _gpu(hb, p), _gpu(hb, p, max_obstacles=16384)
    ha, hb_ = hb.copy(), hb.copy()
    ga.optimize(ha, args)
    gb.optimize(hb_, args)
    _same(ha, hb_)
    ga.close()
    # M_cap > 1024: the kernels without a global-table instantiation fail loudly
    pb, big = scenes.costmap_scene(1500, candidates=2, seed=3)
    g = _gpu(big, pb)
    g.optimize(big.copy(), args)
    for setter, value, calls in ((g.set_solver, 0, ("optimize",)), (g.set_solver, 1, ("optimize",)),
                                 (g.set_linearize_variant, 1, ("optimize", "build_system", "compute_cost"))):
        setter(value)
        for call in calls:
            with pytest.raises(T.TebGpuError, match="rc=-3"):
                getattr(g, call)(big.copy(), *(() if call == "build_system" else (args,)))
        setter(2 if setter == g.set_solver else 0)
    with pytest.raises(T.TebGpuError, match="rc=-3"):
        g.h_signature(big.copy())
    g.close()
    gb.close()
    os.environ["TEBGPU_EVAL_V1"] = "1"
    try:
        g = _gpu(big, pb)
    finally:
        del os.environ["TEBGPU_EVAL_V1"]
    with pytest.raises(T.TebGpuError, match="rc=-3"):
        g.optimize(big.copy(), args)
    g.close()


def test_bad_row_past_index_1024_is_reported():
    import torch
    p, hb0 = scenes.costmap_scene(1500, candidates=2, seed=5, shapes=False)
    hb0.obstacles["type"][0, 1200] = 9                 # unknown obstacle type
    args = _args(p)
    g = _gpu(hb0, p)
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(a.view(np.uint8).reshape(-1)).to(dev)
    poses, n, sid, ob, oc = t(hb0.poses), t(hb0.n), t(hb0.scene_id), t(hb0.obstacles), t(hb0.obst_count)
    vs, vg = t(hb0.vel_start), t(hb0.vel_goal)
    cost = torch.zeros(hb0.B, dtype=torch.float64, device=dev)
    chi2 = torch.zeros_like(cost)
    status = torch.zeros(hb0.B, dtype=torch.int32, device=dev)
    iters = torch.zeros_like(status)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap = hb0.B, hb0.n_cap, hb0.S, hb0.M_cap, 0
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count = ob.data_ptr(), oc.data_ptr()
    bs.vel_start, bs.vel_goal = vs.data_ptr(), vg.data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = cost.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    g.optimize_device(bs, args)
    g.synchronize()
    st = status.cpu().numpy()
    assert np.all(st & abi.TEB_STATUS_BAD_INPUT) and not np.any(st & abi.TEB_STATUS_OPTIMIZED)
    g.close()
