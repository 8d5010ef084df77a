"""The footprint-to-obstacle distance on the device, case by case (tests/distance_cases.py), through the graph build,
kernel A, k_vor and the trial evaluation, against the oracle (run on an H100: pytest -m gpu).

Each case's band (Case.band: heading-0 poses, the case pose at an interior index) runs in a batch of every case of one
footprint, one scene per band. The footprint batches are compared with tests/test_gpu_linearize.check_band (H|b within
1e-12 of the oracle's closed-form system, chi2 by family within 1e-12, association and multiplicity-3 words bit equal):
  a. on the staged path and, padded past 1024 rows, on the global-table path; k_linearize2p and k_linearize2
     (TEBGPU_KA_PERSIST=0); legacy and non-legacy association; include_dynamic_obstacles 0 and 1;
     weight_velocity_obstacle_ratio 0 and 1 (k_vor);
  b. eval_trials with two trials per band, dx = 0 and a dyadic dx that carries the case pose onto the case from 2^-4
     away, against teb_oracle_trial_chi2 within 1e-12 per family, in every trial-evaluation build (eval2 wide, one CTA
     per band and persistent, eval3, the first-generation kernel);
  c. path consistency: every Point / Circular case with a Point / Circular / TwoCircles footprint runs without a vertex
     pool (the fast-path instantiations) and with a far Line obstacle added (the vertex-list instantiations); both meet
     the bars of a. and b. The TwoCircles front / rear ties are decided alike on both paths (the rear circle wins).
The worst errors per build go to the parity report (tests/test_gpu_parity._report)."""
import os

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi
from tests import distance_cases as dc
from tests import banded_reference as R
from tests import test_gpu_trial_eval as TE
from tests.test_gpu_linearize import check_band, _padded

pytestmark = pytest.mark.gpu

CASES = dc.all_cases()
FOOTPRINTS = list(dc.FOOTPRINTS)
SHIFT = 2.0 ** -4      # the trial state is the case: the linearisation point has the case pose SHIFT to the left


def _batch(cases, far=False, shift=0.0):
    """one band per case, one scene per band; far: every scene also holds dc.far_line() (a vertex pool)"""
    B = len(cases)
    extra = [dc.far_line()] if far else []
    M = 1 + len(extra)
    pools = [[] if c.verts is None else list(c.verts) for c in cases]
    rows = np.zeros((B, M), abi.OBST_DTYPE)
    for b, c in enumerate(cases):
        rows[b, 0] = c.obst[0]
        for m, (row, verts) in enumerate(extra):
            rows[b, 1 + m] = row[0]
            rows[b, 1 + m]["vertex_begin"] = len(pools[b])
            pools[b] += list(verts)
    PV = max(len(pl) for pl in pools)
    verts = None
    if PV:
        verts = np.zeros((B, PV, 2))
        for b, pl in enumerate(pools):
            if pl:
                verts[b, :len(pl)] = pl
    poses = np.stack([c.band() for c in cases])
    poses[:, dc.K_CASE, 0] -= shift
    return abi.HostBatch(poses, np.full(B, dc.N_BAND, np.int32), rows, np.full(B, M, np.int32),
                         np.arange(B, dtype=np.int32), obst_vertices=verts)


def _ctx(hb, p, env=None, build="eval2", max_bands=None):
    env = dict(env or {})
    env.update(zip(("TEBGPU_EVAL3", "TEBGPU_EVAL_V1"), {"eval2": ("0", "0"), "eval3": ("1", "0"), "v1": ("0", "1")}[build]))
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        g = T.TebGpu(max_bands or hb.B, hb.n_cap, hb.S, max(hb.M_cap, 1), hb.V_cap, max_obst_vertices=hb.PV_cap)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v
    g.set_params(p)
    return g


CONFIGS = {   # name -> (params, environment, padded past 1024 rows)
    "staged": (dict(), {}, False),
    "legacy": (dict(legacy_obstacle_association=1), {}, False),
    "dynamic": (dict(include_dynamic_obstacles=1), {}, False),
    "legacy_dynamic": (dict(legacy_obstacle_association=1, include_dynamic_obstacles=1), {}, False),
    "vor": (dict(weight_velocity_obstacle_ratio=1.0, obstacle_proximity_lower_bound=0.25,
                 obstacle_proximity_upper_bound=1.0), {}, False),
    "vor_legacy_dynamic": (dict(weight_velocity_obstacle_ratio=1.0, obstacle_proximity_lower_bound=0.25,
                                obstacle_proximity_upper_bound=1.0, legacy_obstacle_association=1,
                                include_dynamic_obstacles=1), {}, False),
    "ka_oneshot": (dict(), {"TEBGPU_KA_PERSIST": "0"}, False),
    "ka_oneshot_legacy_dynamic": (dict(legacy_obstacle_association=1, include_dynamic_obstacles=1),
                                  {"TEBGPU_KA_PERSIST": "0"}, False),
    "global_table": (dict(), {}, True),
    "global_table_legacy_dynamic": (dict(legacy_obstacle_association=1, include_dynamic_obstacles=1), {}, True),
}


def _linearize(cases, cfg, far=False, tag=""):
    kw, env, padded = CONFIGS[cfg]
    p = dc.params(cases[0].fp, **kw)
    hb = _batch(cases, far=far)
    if padded:
        hb = _padded(hb, 1100)
        assert hb.M_cap > 1024
    g = _ctx(hb, p, env)
    try:
        for outer in (0, 2):
            out = g.build_system(hb, outer, graph=True)
            for b in range(hb.B):
                check_band(p, hb, out, b, outer, f"distance/{cfg}{tag}")
    finally:
        g.close()


@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("fp", FOOTPRINTS)
def test_case_bands_against_oracle(fp, cfg):
    _linearize([c for c in CASES if c.fp == fp], cfg)


def _onto(hb, K=2):
    """trial 0: dx = 0; trial 1: + SHIFT on x of the case pose"""
    dx = np.zeros((hb.B, K, 4 * hb.n_cap))
    dx[:, 1, 4 * dc.K_CASE] = SHIFT
    return dx


def _trials(cases, far=False, tag=""):
    sms = TE._sms()
    p = dc.params(cases[0].fp, include_dynamic_obstacles=1)
    hb = _batch(cases, far=far, shift=SHIFT)
    K = 2
    dx = _onto(hb, K)
    ok = np.ones((hb.B, K))
    for build, B in (("eval2", hb.B), ("eval2", 2 * sms), ("eval2", 2 * sms + 40), ("eval3", hb.B), ("v1", hb.B)):
        big, src = TE._embed(hb, B, np.arange(hb.B)) if B > hb.B else (hb, np.arange(hb.B))
        g = _ctx(big, p, build=build, max_bands=B)
        try:
            Hb, _ = g.build_system(big, 0)
            base = 1e-5 * R.max_real_diag(Hb, big.n)
            rd = TE.Round(g, p, big, K, dx[src], ok[src], base[:, None] * np.ones((1, K)), TE._state(B, lam=base), 0,
                          iteration=1)
            name, _ = g.last_trial_eval()
            assert name == TE._build_name(build, B, sms), (build, B, name)
            for b in range(hb.B):       # the trial state of trial 1 is the case band itself
                assert np.array_equal(rd.trial_state(b, 1)[:dc.N_BAND], cases[b].band())
            list(TE.check_chi2(rd, f"distance/{name}{tag}", bands=list(range(hb.B))))
            TE.check_decisions(rd, f"distance/{name}{tag}")
        finally:
            g.close()


@pytest.mark.parametrize("fp", FOOTPRINTS)
def test_case_trials_against_oracle_in_every_build(fp):
    _trials([c for c in CASES if c.fp == fp])


PATH_FPS = sorted({c.fp for c in dc.path_cases()})


@pytest.mark.parametrize("path", ["fast", "vertex_list"])
@pytest.mark.parametrize("fp", PATH_FPS)
def test_fast_and_vertex_list_paths_meet_the_same_bars(fp, path):
    cases = [c for c in dc.path_cases() if c.fp == fp]
    far = path == "vertex_list"
    for cfg in ("staged", "legacy_dynamic", "vor", "global_table"):
        _linearize(cases, cfg, far=far, tag=f"/{path}")
    _trials(cases, far=far, tag=f"/{path}")
