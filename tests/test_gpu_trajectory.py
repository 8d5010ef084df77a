"""getVelocityProfile / getFullTrajectory on the device (tebgpu_read_trajectory / _device, k_read_trajectory).

Every case of tests/trajectory_cases.py is read out in a non-holonomic and a holonomic context and compared with op 9 /
op 10 of the drop-in layer (teb_host_band_op) and of the reference (teb_ref_band_op, or its answers recorded in
tests/golden/golden_ref_traj_v1.npz):
  * x, y, time_from_start and omega bit equal to both;
  * theta bit equal to the band's record, and modulo 2 pi within 1e-15 of both ops' theta (they return it through
    getYaw(createQuaternionFromYaw(theta)));
  * the non-holonomic vx bit equal, sign included: random bands keep off the sign tie, and the tie cases sit on it where
    the trigonometry is exact (heading 0, a pure-y step, vx == 0);
  * the holonomic vx / vy within 1e-12 |step| / |dt| (device cos / sin against glibc).
n = 0 and n = 1, and the zero and negative time differences the reference cannot load, are compared with the drop-in
layer only. Then: band selection, batch position, the two entry points, rows the device entry point cannot read,
argument errors and stream order behind a plan cycle."""
import ctypes as C
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import trajectory_cases as tc

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HOLO_TOL = 1e-12


def _case_batch(cases):
    """one band per case, stride N_CAP, the case's boundary velocities (and active flags) in vel_start / vel_goal"""
    poses = np.stack([c.padded() for c in cases])
    return abi.HostBatch(poses, np.array([c.n for c in cases], np.int32), np.zeros((1, 1), abi.OBST_DTYPE),
                         np.zeros(1, np.int32), vel_start=np.stack([c.vs for c in cases]),
                         vel_goal=np.stack([c.vg for c in cases]))


def _ctx(B, n_cap, max_vel_y=0.0, params=None):
    g = T.TebGpu(B, n_cap, 1, 1, 0)
    p = abi.default_params() if params is None else params
    p.max_vel_y = max_vel_y
    g.set_params(p)
    return g


@pytest.fixture(scope="module")
def host_op():
    return tc.host_band_op()


@pytest.fixture(scope="module")
def readouts():
    """every case read out in one batch per context: {max_vel_y: (profile, trajectory, points)}"""
    cases = tc.all_cases()
    hb = _case_batch(cases)
    out = {}
    for mvy in tc.MAX_VEL_Y:
        g = _ctx(hb.B, tc.N_CAP, mvy)
        out[mvy] = g.read_trajectory(hb)
        assert g.info(14) == (hb.B + 3) // 4
        g.close()
    return cases, out


def _segment_scale(c):
    """|step| / |dt| of segments 1 .. n - 1; 0 where dt == 0 (the twist is exactly zero there)"""
    d = c.rec[1:, :2] - c.rec[:-1, :2]
    dt = np.abs(c.rec[:-1, 3])
    return np.where(dt > 0, np.hypot(d[:, 0], d[:, 1]) / np.where(dt > 0, dt, 1.0), 0.0)


def _expect(c, mvy, prof, traj, want_prof, want_traj):
    n = c.n
    wp, wt = np.asarray(want_prof).reshape(-1, 3), np.asarray(want_traj).reshape(-1, 7)
    assert len(wp) == n + 1 and len(wt) == n, c.name
    p, t = prof[:n + 1], traj[:n]
    assert np.isnan(prof[n + 1:]).all() and np.isnan(traj[n:]).all(), c.name      # rows past n are not written
    assert np.array_equal(p[:, 2], wp[:, 2]), c.name                                # omega
    assert np.array_equal(t[:, [0, 1, 5, 6]], wt[:, [0, 1, 5, 6]]), c.name          # x, y, omega, time_from_start
    assert np.array_equal(t[:, 2], c.rec[:, 2]), c.name                             # theta as stored
    assert all(abs(math.remainder(a - b, 2 * math.pi)) <= 1e-15 for a, b in zip(t[:, 2], wt[:, 2])), c.name
    if mvy == 0:
        assert np.array_equal(p[:, :2], wp[:, :2]) and np.array_equal(t[:, 3:5], wt[:, 3:5]), c.name
        assert (p[:, 1][1:n] == 0).all(), c.name
        return
    seg = _segment_scale(c)
    ps = np.zeros(n + 1)
    ps[1:n] = seg                                           # boundary rows: scale 0, bit equal
    ts = np.zeros(n)
    if n > 2:
        ts[1:n - 1] = np.maximum(seg[:-1], seg[1:])
    assert (np.abs(p[:, :2] - wp[:, :2]) <= HOLO_TOL * ps[:, None]).all(), c.name
    assert (np.abs(t[:, 3:5] - wt[:, 3:5]) <= HOLO_TOL * ts[:, None]).all(), c.name


def test_read_out_equals_the_host_layer(readouts, host_op):
    cases, out = readouts
    for mvy in tc.MAX_VEL_Y:
        prof, traj, pts = out[mvy]
        assert np.array_equal(pts, [c.n for c in cases])
        for b, c in enumerate(cases):
            _expect(c, mvy, prof[b], traj[b], host_op(9, c, mvy), host_op(10, c, mvy))


@pytest.mark.skipif(not tc.reference_available(), reason="neither oracle/_ref/libteb_ref.so nor its recorded calls exist")
def test_read_out_equals_the_reference(readouts):
    tc.use_recording()
    cases, out = readouts
    compared = 0
    for mvy in tc.MAX_VEL_Y:
        prof, traj, _ = out[mvy]
        for b, c in enumerate(cases):
            if c.on_reference:
                _expect(c, mvy, prof[b], traj[b], tc.ref_band_op(9, c, mvy), tc.ref_band_op(10, c, mvy))
                compared += 1
    assert compared == 2 * (len(cases) - 4)


def test_the_defined_rows(readouts):
    """the rows the header defines, stated directly: boundary rows as stored whatever their flag, n = 0 / 1, the sign
    tie, zero time differences, coincident poses"""
    cases, out = readouts
    by = {c.name: b for b, c in enumerate(cases)}
    for mvy in tc.MAX_VEL_Y:
        prof, traj, _ = out[mvy]
        c = cases[by["inactive_boundaries"]]
        p, t = prof[by["inactive_boundaries"]], traj[by["inactive_boundaries"]]
        assert c.vs[3] == 0 and c.vg[3] == 0
        assert np.array_equal(p[0], c.vs[:3]) and np.array_equal(p[c.n], c.vg[:3])
        assert np.array_equal(t[0, 3:6], c.vs[:3]) and np.array_equal(t[c.n - 1, 3:6], c.vg[:3])
        c = cases[by["n0"]]
        assert np.array_equal(prof[by["n0"], 0], c.vg[:3]) and np.isnan(traj[by["n0"]]).all()
        c = cases[by["n1"]]
        assert np.array_equal(prof[by["n1"], :2], [c.vs[:3], c.vg[:3]])
        assert np.array_equal(traj[by["n1"], 0], [*c.rec[0, :3], *c.vs[:3], 0.0])
        c = cases[by["tie_pure_y"]]
        ties = np.flatnonzero(tc.exact_ties(c.rec)) + 1                 # profile rows of the tie segments
        p = prof[by["tie_pure_y"]]
        assert (p[ties, 0] == 0).all()
        assert (p[ties, 1] == (0 if mvy == 0 else (c.rec[ties, 1] - c.rec[ties - 1, 1]) / c.rec[ties - 1, 3])).all()
        c = cases[by["zero_dt"]]
        k = int(np.flatnonzero(c.rec[:-1, 3] == 0)[0]) + 1
        assert (prof[by["zero_dt"], k] == 0).all()
        c = cases[by["coincident"]]
        same = np.flatnonzero(tc.segment_geometry(c.rec)[1] == 0) + 1
        assert (prof[by["coincident"], same, :2] == 0).all()


def test_band_selection_gives_the_full_read_out_rows():
    cases = tc.all_cases()
    hb = _case_batch(cases)
    g = _ctx(hb.B, tc.N_CAP, 0.3)
    full = g.read_trajectory(hb)
    rng = np.random.default_rng(3)
    for bands in ([4], [0, 0, 0], list(range(hb.B))[::-1], rng.integers(0, hb.B, 3 * hb.B).tolist()):
        sel = g.read_trajectory(hb, bands=bands)
        assert g.info(14) == (len(bands) + 3) // 4
        for x, y in zip(full, sel):
            assert np.array_equal(x[bands], y, equal_nan=True)
    prof, traj, pts = g.read_trajectory(hb, bands=[7, 2], trajectory=False)
    assert traj is None and np.array_equal(prof, full[0][[7, 2]], equal_nan=True) and np.array_equal(pts, full[2][[7, 2]])
    prof, traj, pts = g.read_trajectory(hb, bands=[2, 7], profile=False)
    assert prof is None and np.array_equal(traj, full[1][[2, 7]], equal_nan=True)
    g.close()


def test_bits_do_not_depend_on_the_batch_position():
    cases = tc.all_cases()
    hb = _case_batch(cases)
    g = _ctx(hb.B, tc.N_CAP, 0.3)
    a = g.read_trajectory(hb)
    perm = np.random.default_rng(4).permutation(hb.B)
    b = g.read_trajectory(_case_batch([cases[i] for i in perm]))
    for x, y in zip(a, b):
        assert np.array_equal(x[perm], y, equal_nan=True)
    for i in (0, 4, hb.B - 1):
        one = g.read_trajectory(_case_batch([cases[i]]))
        for x, y in zip(a, one):
            assert np.array_equal(x[i:i + 1], y, equal_nan=True)
    g.close()


DEV_FIELDS = ("poses", "n", "scene_id", "obstacles", "obst_count", "obst_vertices", "via", "via_count", "vel_start",
              "vel_goal", "prefer_rotdir", "cost", "chi2", "status", "lm_iters")


class DeviceBatch:
    """torch copies of a HostBatch's arrays and the TebBatch of their device pointers"""

    def __init__(self, hb):
        dev = torch.device("cuda:0")
        self.hb = hb
        self.t = {k: torch.from_numpy(np.ascontiguousarray(getattr(hb, k)).view(np.uint8).reshape(-1).copy()).to(dev)
                  for k in DEV_FIELDS}
        bs = abi.TebBatch()
        bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap, hb.PV_cap
        for k, v in self.t.items():
            setattr(bs, k, v.data_ptr() if v.numel() else None)
        if hb.V_cap == 0:
            bs.via = None
        self.bs = bs

    def snapshot(self):
        return {k: v.cpu().numpy().copy() for k, v in self.t.items()}

    def read(self):
        h = self.hb.copy()
        for k in ("poses", "n", "cost", "chi2", "status", "lm_iters"):
            like = getattr(h, k)
            like[...] = self.t[k].cpu().numpy().view(like.dtype).reshape(like.shape)
        return h


def _device_read(g, db, bands=None, stream=None, pad=2):
    """tebgpu_read_trajectory_device into NaN-filled tensors (points 77), `pad` spare rows behind the R read"""
    dev = torch.device("cuda:0")
    R = db.hb.B if bands is None else len(bands)
    nc = db.hb.n_cap
    prof = torch.full((R + pad, nc + 1, 3), math.nan, dtype=torch.float64, device=dev)
    traj = torch.full((R + pad, nc, 7), math.nan, dtype=torch.float64, device=dev)
    pts = torch.full((R + pad,), 77, dtype=torch.int32, device=dev)
    bl = None if bands is None else torch.tensor(bands, dtype=torch.int32, device=dev)
    g.read_trajectory_device(db.bs, trajectory=traj, profile=prof, points=pts, bands=bl,
                             stream=torch.cuda.current_stream().cuda_stream if stream is None else stream)
    torch.cuda.synchronize()
    return prof.cpu().numpy(), traj.cpu().numpy(), pts.cpu().numpy()


def _c3_batch(B, seed):
    p, hb = scenes.make_config_batch("C3", candidates=B, seed=seed)
    rng = np.random.default_rng(seed)
    hb.vel_start[:, :3] = rng.normal(0, 0.2, (hb.B, 3))
    hb.vel_goal[:, :3] = rng.normal(0, 0.2, (hb.B, 3))
    hb.vel_goal[::3, 3] = 0.0                                   # free goal velocity: still reported as stored
    return p, hb


@pytest.mark.parametrize("max_vel_y", tc.MAX_VEL_Y)
def test_host_and_device_entry_points_give_the_same_bits_and_leave_the_batch_alone(max_vel_y):
    p, hb = _c3_batch(24, 5)
    hb.n[1::4] = [150, 2, 1, 0, 77, 199]                        # rows past n stay NaN
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
    p.max_vel_y = max_vel_y
    g.set_params(p)
    db = DeviceBatch(hb)
    for bands in (None, [3, 3, 0, 23, 11]):
        before = db.snapshot()
        h = g.read_trajectory(hb, bands=bands)
        d = _device_read(g, db, bands)
        assert all(np.array_equal(before[k], v) for k, v in db.snapshot().items())          # TebBatch untouched
        R = len(h[2])
        for x, y in zip(h, d):
            assert np.array_equal(x, y[:R], equal_nan=True)
        assert np.isnan(d[0][R:]).all() and np.isnan(d[1][R:]).all() and (d[2][R:] == 77).all()   # nothing past R
        for r in range(R):
            n = h[2][r]
            assert np.isnan(d[0][r, n + 1:]).all() and np.isnan(d[1][r, n:]).all() and not np.isnan(d[1][r, :n]).any()
    g.close()


def test_device_entry_point_marks_the_rows_it_cannot_read():
    p, hb = _c3_batch(8, 6)
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
    g.set_params(p)
    want = g.read_trajectory(hb, bands=[0, 3])
    h = hb.copy()
    h.n[1] = hb.n_cap + 1
    h.n[2] = -1
    db = DeviceBatch(h)
    prof, traj, pts = _device_read(g, db, bands=[0, 1, 2, -1, hb.B, 3])
    assert g.launch_count() == 1
    assert np.array_equal(pts[:6], [hb.n[0], -1, -1, -1, -1, hb.n[3]])
    assert np.isnan(prof[1:5]).all() and np.isnan(traj[1:5]).all()        # a bad row gets points = -1 and nothing else
    for x, y in zip(want[:2], (prof, traj)):
        assert np.array_equal(x, y[[0, 5]], equal_nan=True)
    g.close()


def test_argument_errors_launch_nothing():
    p, hb = _c3_batch(4, 8)
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
    g.set_params(p)
    g.optimize(hb.copy(), abi.make_args(1, 1))
    launches = g.launch_count()
    assert launches > 1
    L = g.lib
    prof = np.full((hb.B, hb.n_cap + 1, 3), np.nan)
    pts = np.zeros(hb.B, np.int32)
    bands = np.array([0, 1], np.int32)

    def args(**kw):
        ta = abi.TebTrajectoryArgs()
        ta.profile, ta.points = abi.ptr(prof), abi.ptr(pts)
        for k, v in kw.items():
            setattr(ta, k, v)
        return ta
    db = DeviceBatch(hb)
    for kw in (dict(points=None), dict(profile=None), dict(bands=abi.ptr(bands), count=-1)):
        ta = args(**kw)
        assert L.tebgpu_read_trajectory(g.ctx, C.byref(hb.struct()), C.byref(ta)) == abi.TEBGPU_ERR_INVALID_ARG, kw
        assert L.tebgpu_read_trajectory_device(g.ctx, C.byref(db.bs), C.byref(ta), None) == abi.TEBGPU_ERR_INVALID_ARG, kw
        assert g.launch_count() == launches, kw
    assert L.tebgpu_read_trajectory(g.ctx, None, C.byref(args())) == abi.TEBGPU_ERR_INVALID_ARG
    assert L.tebgpu_read_trajectory(g.ctx, C.byref(hb.struct()), None) == abi.TEBGPU_ERR_INVALID_ARG
    for field in ("poses", "n", "vel_start", "vel_goal"):
        bs = hb.struct()
        setattr(bs, field, None)
        assert L.tebgpu_read_trajectory(g.ctx, C.byref(bs), C.byref(args())) == abi.TEBGPU_ERR_INVALID_ARG, field
        bs = abi.TebBatch.from_buffer_copy(db.bs)
        setattr(bs, field, None)
        assert L.tebgpu_read_trajectory_device(g.ctx, C.byref(bs), C.byref(args()), None) == abi.TEBGPU_ERR_INVALID_ARG, field
    # the host entry point refuses what the device entry point answers with -1
    for bad in ([0, hb.B], [-1]):
        bl = np.array(bad, np.int32)
        assert L.tebgpu_read_trajectory(g.ctx, C.byref(hb.struct()), C.byref(args(bands=abi.ptr(bl), count=len(bl)))) \
            == abi.TEBGPU_ERR_INVALID_ARG, bad
    for v in (hb.n_cap + 1, -1):
        h = hb.copy()
        h.n[1] = v
        assert L.tebgpu_read_trajectory(g.ctx, C.byref(h.struct()), C.byref(args())) == abi.TEBGPU_ERR_INVALID_ARG, v
    assert g.launch_count() == launches
    assert np.isnan(prof).all()
    # count == 0 is a valid empty read: nothing is launched
    assert L.tebgpu_read_trajectory(g.ctx, C.byref(hb.struct()), C.byref(args(bands=abi.ptr(bands), count=0))) == abi.TEBGPU_OK
    assert g.launch_count() == 0 and np.isnan(prof).all()
    g.close()


def test_plan_then_read_on_one_stream_matches_plan_and_read_on_host_buffers():
    p, hb = _c3_batch(16, 9)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
    g.set_params(p)
    start, goal = hb.poses[:, 1, :3].copy(), hb.poses[np.arange(hb.B), hb.n - 1, :3].copy()
    db = DeviceBatch(hb)
    dev = torch.device("cuda:0")
    cmd = torch.zeros((hb.B, 4), dtype=torch.float64, device=dev)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g.plan_device(db.bs, args, cmd, start=torch.from_numpy(start).to(dev), goal=torch.from_numpy(goal).to(dev),
                      stream=s.cuda_stream)
        d = _device_read(g, db, bands=[5, 0, 15, 5], stream=s.cuda_stream)
    h = hb.copy()
    g.plan(h, start, goal, args)
    want = g.read_trajectory(h, bands=[5, 0, 15, 5])
    for x, y in zip(want, d):
        assert np.array_equal(x, y[:4], equal_nan=True)
    assert not np.array_equal(h.n, hb.n) or not np.array_equal(h.poses, hb.poses)    # the cycle did change the bands
    g.close()
