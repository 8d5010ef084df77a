"""The oracle against the reference's own code (oracle/_ref/libteb_ref.so, see tests/ref_binding.py) at every parameter
switch of buildGraph: the configurations of tests/param_cases.py take each edge family make_kparams restates to both
sides and to its boundary. For every configuration and band:
  * the graph, edge by edge (dimension, vertex ids, error, information, Jacobian) and the assembled H / b / chi2, at
    obstacle weight multipliers 1 and weight_adapt_factor^3;
  * whole optimizeTEB calls: poses, n, cost, LM trials, rejections, Terminate and the failed-factorisation flag.
The bar is bit equality, as in tests/test_reference_pin.py. This is what makes the closed-form oracle the yardstick of
tests/test_gpu_params.py at these configurations. Where the library cannot be built the calls are answered from
tests/golden/golden_ref_params_v1.npz (recorded by tests/golden/make_golden_ref_params.py)."""
import os

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import param_cases as pc
from tests import ref_binding as rb
from tests import scenarios

GOLDEN_PARAMS = os.path.join(os.path.dirname(__file__), "golden", "golden_ref_params_v1.npz")
pytestmark = pytest.mark.skipif(not (rb.live() or os.path.exists(GOLDEN_PARAMS)),
                                reason="neither oracle/_ref/libteb_ref.so nor its recorded parameter-switch calls exist")


@pytest.fixture(scope="module")
def ref():
    rb.add_recording(GOLDEN_PARAMS)
    return rb


@pytest.mark.parametrize("name", pc.ALL)
def test_graph_edges_bit_equal(oracle, ref, name):
    p, hb = pc.case(name)
    for b in range(hb.B):
        n = int(hb.n[b])
        kw = scenarios.band_kwargs(hb, b)
        for wm in (1.0, pc.weight_multiplier(p, 3)):
            Ho, bo, co = oracle.build_system(p, hb.poses[b], n, weight_multiplier=wm, jac_mode=oracle.JAC_G2O, **kw)
            Hr, br, cr, er = ref.build_system(p, hb.poses[b], n, weight_multiplier=wm, want_edges=True, **kw)
            eo = oracle.dump_edges(p, hb.poses[b], n, weight_multiplier=wm, jac_mode=oracle.JAC_G2O, **kw)
            where = (name, b, wm)
            assert eo.shape == er.shape, (where, eo.shape, er.shape)
            if isinstance(er, np.ndarray):      # the library itself: name the part that differs
                assert np.array_equal(eo[:, 53:], er[:, 53:]), (where, "graph structure differs")
                assert np.array_equal(eo[:, :8], er[:, :8], equal_nan=True), (where, "errors / information differ")
            assert ref.same(eo, er), (where, "Jacobians differ")
            assert ref.same(Ho, Hr) and ref.same(bo, br), where
            assert co == cr or (np.isnan(co) and np.isnan(cr)), where


@pytest.mark.parametrize("name", pc.ALL)
def test_optimize_teb_bit_equal(oracle, ref, name):
    p, hb = pc.case(name)
    a = pc.args(p)
    for b in range(hb.B):
        n = int(hb.n[b])
        kw = scenarios.band_kwargs(hb, b)
        ro, co, so = oracle.optimize_band(p, hb.poses[b], n, args=a, jac_mode=oracle.JAC_G2O, n_cap=hb.n_cap, **kw)
        rr, cr, sr, ok = ref.optimize_band(p, hb.poses[b], n, args=a, n_cap=hb.n_cap, **kw)
        where = (name, b)
        assert len(ro) == len(rr) and ref.same(ro, rr), where
        assert bool(so.status & abi.TEB_STATUS_OPTIMIZED) == ok, where
        assert co == cr or (np.isnan(co) and np.isnan(cr)), (where, co, cr)
        assert so.lm_trials == sr["lm_trials"] and so.rejected == sr["rejected"], where
        assert bool(so.status & abi.TEB_STATUS_TERMINATED) == sr["terminated"], where
        assert bool(so.status & abi.TEB_STATUS_CHOL_FAILED) == sr["chol_failed"], where


def test_every_predicate_takes_both_sides():
    """the table reaches both truth values of each make_kparams predicate (restated here from buildGraph), and the
    boundaries of the inflated / exponent / legacy-index branches"""
    seen = {}

    def note(k, v):
        seen.setdefault(k, set()).add(bool(v))
    for name in pc.ALL:
        p, hb = pc.case(name)
        holo = p.max_vel_y != 0
        car = not (p.min_turning_radius == 0 or p.weight_kinematics_turning_radius == 0)
        note("inflated", p.inflation_dist > p.min_obstacle_dist)
        note("inflated_boundary", p.inflation_dist == p.min_obstacle_dist)
        note("dyn_inflated", p.dynamic_obstacle_inflation_dist > p.min_obstacle_dist)
        note("dyn_inflated_boundary", p.dynamic_obstacle_inflation_dist == p.min_obstacle_dist)
        note("carlike", car)
        note("holo_vel", holo)
        note("holo_acc", holo and p.acc_lim_y != 0)
        note("has_vel_holo", holo and not (p.weight_max_vel_x == 0 and p.weight_max_vel_y == 0 and p.weight_max_vel_theta == 0))
        note("has_vel", not (p.weight_max_vel_x == 0 and p.weight_max_vel_theta == 0))
        note("has_acc", not (p.weight_acc_lim_x == 0 and p.weight_acc_lim_theta == 0))
        note("has_kin_car", car and not (p.weight_kinematics_nh == 0 and p.weight_kinematics_turning_radius == 0))
        note("has_kin_diff", not car and not (p.weight_kinematics_nh == 0 and p.weight_kinematics_forward_drive == 0))
        note("has_sp", p.weight_shortest_path != 0)
        note("has_rot", p.weight_prefer_rotdir != 0)
        note("has_time", p.weight_optimaltime != 0)
        note("has_obst", p.weight_obstacle != 0)
        note("has_dyn", p.include_dynamic_obstacles and p.weight_obstacle != 0)
        note("has_via", p.weight_viapoint != 0)
        note("pow_exponent", p.obstacle_cost_exponent != 1.0 and p.min_obstacle_dist > 0.0)
        note("exponent_below_1", p.obstacle_cost_exponent < 1.0 and p.min_obstacle_dist > 0.0)
        note("has_vor", p.weight_velocity_obstacle_ratio > 0 and not p.legacy_obstacle_association)
        note("legacy_all_at_middle", p.legacy_obstacle_association and p.obstacle_poses_affected >= int(hb.n.min()))
        note("penalty_epsilon0", p.penalty_epsilon == 0)
        note("force_above_cutoff", p.obstacle_association_force_inclusion_factor > p.obstacle_association_cutoff_factor)
        note("exact_arc_length", p.exact_arc_length)
    missing = {k: v for k, v in seen.items() if v != {True, False}}
    assert not missing, missing
