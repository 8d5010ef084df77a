"""CPU checks of teb_oracle_graph, the oracle's reading of the structure buildGraph() gives a band (obstacle association
bit words, the legacy multiplicity-3 words, via-point poses, dynamic-obstacle times). tests/test_gpu_linearize.py holds
k_build_graph to it bit for bit, so it is checked here three ways:
  * on every scenario it agrees with teb_oracle_dump_edges: the unary pose edges of pose i are popcount(assoc) +
    2 popcount(assoc3) obstacle edges, one edge per via-point on the pose and one per dynamic obstacle where the pose
    has a time; poses 0 and n-1 carry none;
  * the chi2 of the obstacle and via families rebuilt from the structure alone (distance, penalties and weights per
    associated obstacle) is teb_oracle_trial_chi2's at the linearisation point;
  * one hand-worked case per branch of the association and of the via-point assignment.
"""
import math

import numpy as np
import pytest

from teb_local_planner_b200 import abi
from tests import oracle_binding as O
from tests import scenarios


def _popcount(words):
    return sum(bin(int(w)).count("1") for w in np.asarray(words).ravel())


def _bits(words):
    out = []
    for w, word in enumerate(np.asarray(words).ravel()):
        word = int(word)
        while word:
            low = word & -word
            out.append(64 * w + low.bit_length() - 1)
            word ^= low
    return out


@pytest.mark.parametrize("name", scenarios.ALL)
def test_structure_matches_dumped_edges(oracle, name):
    p, hb = scenarios.scenario(name)
    for b in range(hb.B):
        n = int(hb.n[b])
        kw = scenarios.band_kwargs(hb, b)
        for outer in (0, 3):
            gr = O.graph(p, hb.poses[b], n, weight_multiplier=2.0 ** outer, **kw)
            rows = O.dump_edges(p, hb.poses[b], n, weight_multiplier=2.0 ** outer, **kw)
            unary = np.zeros(n, int)
            for r in rows:
                if int(r[1]) == 1 and int(r[58]) % 2 == 0:
                    unary[int(r[58]) // 2] += 1
            obs = kw["obstacles"]
            D = int(np.count_nonzero(obs["dynamic"])) if p.include_dynamic_obstacles else 0
            via_on = np.bincount(gr["via_idx"][gr["via_idx"] >= 0], minlength=n)
            assert unary[0] == 0 and unary[n - 1] == 0
            for i in range(1, n - 1):
                own = _popcount(gr["assoc"][i]) + 2 * _popcount(gr["assoc3"][i])
                dyn = D if np.isfinite(gr["dyn_t"][i]) else 0
                assert unary[i] == own + via_on[i] + dyn, (name, b, i, unary[i], own, via_on[i], dyn)
            # every legacy multiplicity-3 bit is also an association bit
            assert np.array_equal(gr["assoc3"] & gr["assoc"], gr["assoc3"])
            if D:
                assert np.isfinite(gr["dyn_t"][1:n - 1]).all() and np.isnan(gr["dyn_t"][[0, n - 1]]).all()
            if not p.legacy_obstacle_association and p.weight_velocity_obstacle_ratio == 0:
                assert not gr["assoc"][0].any()


def _obstacle_chi2(p, rec, n, gr, obs, verts, mult):
    """obstacle family from the structure alone (EdgeObstacle / EdgeInflatedObstacle / EdgeDynamicObstacle errors)"""
    L = O.lib()
    inflated = p.inflation_dist > p.min_obstacle_dist
    total = 0.0
    for i in range(1, n - 1):
        pose = rec[i, :3]
        three = set(_bits(gr["assoc3"][i]))
        for m in _bits(gr["assoc"][i]):
            d = O.distance(p, pose, obs[m], verts)
            e0 = L.teb_oracle_penalty_below(d, p.min_obstacle_dist, p.penalty_epsilon)
            if p.obstacle_cost_exponent != 1.0 and p.min_obstacle_dist > 0:
                e0 = p.min_obstacle_dist * (e0 / p.min_obstacle_dist) ** p.obstacle_cost_exponent
            c = p.weight_obstacle * mult * e0 * e0
            if inflated:
                e1 = L.teb_oracle_penalty_below(d, p.inflation_dist, 0.0)
                c += p.weight_inflation * e1 * e1
            total += 3 * c if m in three else c
        if np.isfinite(gr["dyn_t"][i]):
            for m in np.flatnonzero(obs["dynamic"]):
                d = O.distance(p, pose, obs[m], verts, t=float(gr["dyn_t"][i]))
                e0 = L.teb_oracle_penalty_below(d, p.min_obstacle_dist, p.penalty_epsilon)
                e1 = L.teb_oracle_penalty_below(d, p.dynamic_obstacle_inflation_dist, 0.0)
                total += p.weight_dynamic_obstacle * e0 * e0 + p.weight_dynamic_obstacle_inflation * e1 * e1
    return total


@pytest.mark.parametrize("name", scenarios.ALL)
def test_structure_gives_trial_chi2_families(oracle, name):
    p, hb = scenarios.scenario(name)
    for b in range(hb.B):
        n = int(hb.n[b])
        kw = scenarios.band_kwargs(hb, b)
        rec = hb.poses[b][:n]
        for outer in (0, 3):
            mult = 2.0 ** outer
            gr = O.graph(p, rec, n, weight_multiplier=mult, **kw)
            fam = O.trial_chi2(p, rec, n, rec[None], weight_multiplier=mult, **kw)[0]
            obst = _obstacle_chi2(p, rec, n, gr, kw["obstacles"], kw["obst_vertices"], mult)
            assert abs(obst - fam[0]) <= 1e-12 * max(fam[0], 1e-300) + 1e-300, (name, b, obst, fam[0])
            via = 0.0
            for v, i in enumerate(gr["via_idx"]):
                if i >= 0:
                    dx, dy = rec[i, 0] - kw["via"][v, 0], rec[i, 1] - kw["via"][v, 1]
                    via += p.weight_viapoint * (dx * dx + dy * dy)
            assert abs(via - fam[1]) <= 1e-12 * max(fam[1], 1e-300) + 1e-300, (name, b, via, fam[1])


# ------------------------------------------------------------------ hand-worked branches
def _line(n, dx=0.5):
    """straight band along +x, theta 0, poses at i dx, dt 0.5 (dyadic: every distance below is exact)"""
    rec = np.zeros((n, 4))
    rec[:, 0] = dx * np.arange(n)
    rec[:, 3] = 0.5
    rec[n - 1, 3] = 0.0
    return rec


def _params(**kw):
    p = abi.default_params()
    p.min_obstacle_dist, p.inflation_dist = 0.5, 0.0
    p.obstacle_association_force_inclusion_factor, p.obstacle_association_cutoff_factor = 2.0, 4.0  # 1.0 / 2.0 m
    p.include_dynamic_obstacles = 0
    p.footprint_type = abi.TEB_FOOTPRINT_POINT
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _obst(*rows, dynamic=()):
    ob = np.zeros(len(rows), abi.OBST_DTYPE)
    for m, (x, y) in enumerate(rows):
        ob[m]["x"], ob[m]["y"] = x, y
        ob[m]["type"] = abi.TEB_OBST_POINT
    for m in dynamic:
        ob[m]["dynamic"] = 1
    return ob


def _pose_bits(gr, i):
    return _bits(gr["assoc"][i])


def test_nonlegacy_association_branches(oracle):
    n = 9
    rec = _line(n)
    p = _params()
    # pose 4 sits at x = 2. Candidates beyond force_d = 1 and within cut_d = 2:
    #   obstacles 0 / 1 at distance 1.25 on the left (equal distances: the lowest index wins),
    #   obstacle 2 exactly at force_d (1.0, not forced: strict <), on the right, and obstacle 3 further right at 1.25
    ob = _obst((2.0 - 0.75, 1.0), (2.0 + 0.75, 1.0), (2.0, -1.0), (2.0 + 0.75, -1.0))
    gr = O.graph(p, rec, n, ob)
    assert math.hypot(0.75, 1.0) == 1.25
    assert _pose_bits(gr, 4) == [0, 2]          # lowest index among the equal left candidates; 2 closest on the right
    # exactly at cut_d (2.0) is still a candidate (strict >), just beyond it is not
    gr = O.graph(p, rec, n, _obst((2.0, 2.0)))
    assert 0 in _pose_bits(gr, 4)
    gr = O.graph(p, rec, n, _obst((2.0, 2.0 + 2.0 ** -20)))
    assert 0 not in _pose_bits(gr, 4)
    # just inside force_d: forced, together with the closest left / right candidates
    gr = O.graph(p, rec, n, _obst((2.0, 1.0 - 2.0 ** -20), (2.0, 1.5), (2.0, -1.5)))
    assert _pose_bits(gr, 4) == [0, 1, 2]
    # dead ahead of pose 1 (cross product 0): the right side; obstacle 1 on the right but further loses to it
    gr = O.graph(p, rec, n, _obst((0.5 + 1.5, 0.0), (0.5, -1.75)))
    assert _pose_bits(gr, 1) == [0]
    # dynamic rows are not associated under include_dynamic_obstacles (they get dynamic edges with frozen times)
    p.include_dynamic_obstacles = 1
    gr = O.graph(p, rec, n, _obst((2.0, 0.25), (2.0, -0.25), dynamic=(0,)))
    assert all(0 not in _pose_bits(gr, i) for i in range(n)) and 1 in _pose_bits(gr, 4)
    assert np.array_equal(gr["dyn_t"][1:n - 1], 0.5 * np.arange(1, n - 1))
    assert np.isnan(gr["dyn_t"][[0, n - 1]]).all()
    # pose 0 is associated only to feed the velocity-obstacle ratio
    p = _params()
    gr = O.graph(p, rec, n, _obst((0.0, 0.25)))
    assert not gr["assoc"][0].any()
    p.weight_velocity_obstacle_ratio = 1.0
    gr = O.graph(p, rec, n, _obst((0.0, 0.25)))
    assert _pose_bits(gr, 0) == [0]


def test_legacy_association_branches(oracle):
    n = 12
    rec = _line(n)
    for opa, want in ((1, {5: 1}), (2, {5: 3}), (3, {5: 3}), (10, {5: 3, 4: 1, 6: 1, 3: 1, 7: 1, 2: 1, 8: 1, 1: 1, 9: 1})):
        p = _params(legacy_obstacle_association=1, obstacle_poses_affected=opa)
        gr = O.graph(p, rec, n, _obst((2.5, 0.3)))     # closest pose 5
        got = {i: (3 if gr["assoc3"][i].any() else 1) for i in range(1, n - 1) if gr["assoc"][i].any()}
        assert got == want, (opa, got)
    p = _params(legacy_obstacle_association=1, obstacle_poses_affected=4)
    # closest-pose ties: the first pose wins (strict <); x = 2.25 is equidistant from poses 4 and 5
    gr = O.graph(p, rec, n, _obst((2.25, 0.0)))
    assert gr["assoc3"][4].any() and not gr["assoc3"][5].any()
    # closest pose <= 1 or = n - 1: no edge at all
    for x in (0.0, 0.5, 0.5 * (n - 1), 9.0):
        gr = O.graph(p, rec, n, _obst((x, 0.0)))
        assert not gr["assoc"].any(), x
    gr = O.graph(p, rec, n, _obst((0.5 * (n - 2), 0.0)))   # n - 2 is associated
    assert gr["assoc3"][n - 2].any()
    # obstacle_poses_affected >= n: index n / 2 whatever the distance
    p = _params(legacy_obstacle_association=1, obstacle_poses_affected=n)
    gr = O.graph(p, rec, n, _obst((0.0, 0.0)))
    assert gr["assoc3"][n // 2].any()


def test_via_point_branches(oracle):
    n = 8
    rec = _line(n)
    p = _params(weight_viapoint=1.0)
    via = np.array([[-3.0, 0.0],      # before the start: closest pose 0
                    [100.0, 0.0],     # beyond the goal: closest pose n-1 -> n-2
                    [1.25, 0.5],      # tie between poses 2 and 3: the first wins
                    [1.0, 0.25],      # two on pose 2
                    [2.0, 0.0]])      # exactly on pose 4
    gr = O.graph(p, rec, n, _obst(), via=via)
    assert list(gr["via_idx"]) == [-1, n - 2, 2, 2, 4]
    p.via_points_ordered = 1
    # ordered: the search starts two poses past the previous via-point; before the start -> pose 1
    gr = O.graph(p, rec, n, _obst(), via=via)
    # [0] closest pose 0 -> pinned to 1, next search from 2; [1] pose n-1 -> n-2, next search from n+1; [2] a search
    # that starts past n finds no pose -> pinned to 1, the next restarts from -1 + 2 = 1; [3] from 1: pose 2, next from
    # 4; [4] from 4: pose 4
    assert list(gr["via_idx"]) == [1, n - 2, 1, 2, 4]
