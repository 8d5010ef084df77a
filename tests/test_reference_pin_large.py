"""The oracle restatement against the reference's own code (oracle/_ref/libteb_ref.so, see tests/ref_binding.py) on
scenes of more than 1024 obstacles: whole optimizeTEB calls bit-equal. Where the library cannot be built the calls are
answered from tests/golden/golden_ref_large_v1.npz (recorded by tests/golden/make_golden_ref_large.py)."""
import os

import numpy as np
import pytest

from teb_local_planner_b200 import abi, scenes
from tests import ref_binding as rb

GOLDEN_LARGE = os.path.join(os.path.dirname(__file__), "golden", "golden_ref_large_v1.npz")
pytestmark = pytest.mark.skipif(not (rb.live() or os.path.exists(GOLDEN_LARGE)),
                                reason="neither oracle/_ref/libteb_ref.so nor its recorded large-scene calls exist")


@pytest.fixture(scope="module")
def ref():
    if not rb.live():   # answer from the large-scene recording as well
        if rb._replay is None:
            rb._replay = rb._load(rb.GOLDEN_CALLS) if os.path.exists(rb.GOLDEN_CALLS) else {}
        rb._replay.update(rb._load(GOLDEN_LARGE))
    return rb


@pytest.mark.parametrize("legacy", [False, True])
def test_optimize_teb_bit_equal_beyond_1024_obstacles(oracle, ref, legacy):
    """costmap-like scene of 1500 rows (points on a 5 cm grid, circular, line and moving obstacles): poses, n, cost and
    the LM trials of the reference's code and of the restatement are identical"""
    p, hb = scenes.costmap_scene(1500, n=60, candidates=2, seed=11)
    if legacy:
        p.legacy_obstacle_association, p.obstacle_poses_affected = 1, 10
    assert hb.M_cap > 1024
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale,
                         p.selection_viapoint_cost_scale, False)
    for b in range(hb.B):
        n = int(hb.n[b])
        kw = dict(obstacles=hb.obstacles[0][:hb.obst_count[0]], vel_start=hb.vel_start[b], vel_goal=hb.vel_goal[b],
                  obst_vertices=hb.obst_vertices[0])
        ro, co, so = oracle.optimize_band(p, hb.poses[b], n, args=args, jac_mode=oracle.JAC_G2O, n_cap=hb.n_cap, **kw)
        rr, cr, sr, ok = ref.optimize_band(p, hb.poses[b], n, args=args, n_cap=hb.n_cap, **kw)
        assert ok and len(ro) == len(rr), (b, len(ro), len(rr))
        assert ref.same(ro, rr), b
        assert co == cr
        assert so.lm_trials == sr["lm_trials"] and so.rejected == sr["rejected"]
        assert np.isfinite(co) and so.status & abi.TEB_STATUS_OPTIMIZED
