"""The costmap-to-obstacle restatement of tests/costmap_cases.py pinned on hand-computed cases, and its numpy form held
bit equal to it on drawn rasters. CPU only."""
import math

import numpy as np
import pytest

from teb_local_planner_b200 import abi, scenes
from tests import costmap_cases as cm


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


@pytest.mark.parametrize("case", cm.cases(), ids=lambda c: c.name)
def test_restatement_gives_the_hand_computed_rows(case):
    want = cm.expected_rows(case)
    for f in (cm.restate, cm.restate_np):
        got = f(case.flat(), case.sx, case.sy, case.origin, case.robot, case.behind, case.include, case.custom)
        assert _bytes(got) == _bytes(want), (f.__name__, got, want)


def test_custom_rows_are_verbatim_and_every_point_byte_is_defined():
    c = [x for x in cm.cases() if x.name == "custom_after_points"][0]
    got = cm.restate(c.flat(), c.sx, c.sy, c.origin, c.robot, c.behind, True, c.custom)
    assert _bytes(got[2:]) == _bytes(c.custom)
    pts = got[:2]
    assert (pts["type"] == abi.TEB_OBST_POINT).all() and (pts["dynamic"] == 0).all()
    for k in ("vx", "vy", "radius", "vertex_begin", "vertex_count", "_pad"):
        assert (pts[k] == 0).all() and not np.signbit(pts[k]).any(), k


def test_only_lethal_cells_of_a_drawn_raster_count():
    r = scenes.costmap_raster(2, 40, 30, seed=1)
    for s in range(2):
        c = r["cost"][s, :1200].reshape(30, 40)
        assert {253, 254, 255} <= set(np.unique(c)) and (c < 253).any()
        rows = cm.restate(r["cost"][s], 40, 30, r["origin"][s], r["robot"][s], math.inf)
        assert len(rows) == int((c[:-1, :-1] == 254).sum())


@pytest.mark.parametrize("seed", range(4))
def test_numpy_form_is_bit_equal_to_the_scalar_form(seed):
    rng = np.random.default_rng(seed)
    sx, sy = (int(v) for v in rng.integers(2, 70, 2))
    r = scenes.costmap_raster(3, sx, sy, res=float(rng.choice([0.05, 0.1, 0.03])), lethal=0.2, seed=seed)
    for s in range(3):
        for behind in (0.0, 1.5, math.inf, -1.0, math.nan, 0.7):
            a = cm.restate(r["cost"][s], sx, sy, r["origin"][s], r["robot"][s], behind)
            b = cm.restate_np(r["cost"][s], sx, sy, r["origin"][s], r["robot"][s], behind)
            assert _bytes(a) == _bytes(b), (seed, s, behind)
