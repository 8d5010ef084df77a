"""TebOptimalPlanner::plan followed by getVelocityCommand on the device (tebgpu_plan_batch / _device, teb_plan.cuh).

The band operations are compared with the drop-in layer's (teb_host_band_op: initTrajectoryToGoal, updateAndPruneTEB,
getVelocityCommand, pinned bit for bit against the reference by tests/test_host_pin.py) and with the oracle's
init_trajectory; the path decision with a plain-Python restatement of optimal_planner.cpp:259-269 / :300-309. Every case
runs through both entry points, which must give the same bits. Cold starts and plan initialisations may differ from
the host in the last ulp of the device trig (bar 1e-12, the worst value is printed); warm starts move records and
must be bit equal. Whole cycles run the optimizer on C1 / C3 batches and compare with the host-buffer loop (host
prune + tebgpu_optimize_batch)."""
import ctypes as C
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import oracle_binding as ob

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
N_CAP = 48
P_CAP = 24


@pytest.fixture(scope="module")
def host_op():
    from teb_local_planner_b200 import build as b
    b.build()
    b.build_host()
    fn = C.CDLL(b.HOST_PIN).teb_host_band_op
    fn.restype = C.c_int32
    fn.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]

    def run(op, rec, args, cap=8192):
        rec = None if rec is None else np.ascontiguousarray(rec, dtype=np.float64)
        a = np.ascontiguousarray(args, dtype=np.float64)
        out = np.full(cap, np.nan)
        k = fn(op, None if rec is None else rec.ctypes.data, 0 if rec is None else len(rec), a.ctypes.data, len(a),
               out.ctypes.data, cap)
        assert k >= 0, (op, k)
        return out[:k].copy()
    return run


def _params(min_samples=3, backwards=0, overwrite=1, optimize=False):
    p = abi.default_params()
    p.min_samples = min_samples
    p.allow_init_with_backwards_motion = backwards
    p.global_plan_overwrite_orientation = overwrite
    p.optimization_activate = int(optimize)
    return p


def _empty_batch(B, n_cap=N_CAP):
    obst = np.zeros((1, 1), abi.OBST_DTYPE)
    return abi.HostBatch(np.zeros((B, n_cap, 4)), np.zeros(B, np.int32), obst, [0])


def _gpu(hb, p, **switches):
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, max(hb.M_cap, 1), hb.V_cap, max_obst_vertices=hb.PV_cap)
    g.set_params(p)
    for name, v in switches.items():
        getattr(g, "set_" + name)(v)
    return g


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

    def load(self, hb):
        for k in DEV_FIELDS:
            self.t[k].copy_(torch.from_numpy(np.ascontiguousarray(getattr(hb, k)).view(np.uint8).reshape(-1).copy()))

    def read(self):
        h = self.hb.copy()
        for k in ("poses", "n", "cost", "chi2", "status", "lm_iters"):
            like = getattr(h, k)
            like[...] = self.t[k].cpu().numpy().view(like.dtype).reshape(like.shape)
        return h


def _both(g, hb, args, start=None, goal=None, look=1, prevent=0, plan=None, count=None, keep=None):
    """the same cycle through tebgpu_plan_batch and tebgpu_plan_batch_device: identical bits; returns the host run.
    keep: a dict that holds the device buffers across calls (the same addresses every cycle)"""
    h = hb.copy()
    cmd, path = g.plan(h, start, goal, args, look, prevent, initial_plan=plan, plan_count=count)
    dev = torch.device("cuda:0")
    f = lambda a, dt=torch.float64: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)
    inputs = [f(start), f(goal), f(plan), f(count, torch.int32)]
    if keep is not None and keep:
        keep["db"].load(hb)
        for t, v in zip(keep["inputs"], inputs):
            if t is not None:
                t.copy_(v)
    elif keep is not None:
        keep.update(db=DeviceBatch(hb), inputs=inputs, cmd=torch.zeros((hb.B, 4), dtype=torch.float64, device=dev),
                    path=torch.full((hb.B,), -2, dtype=torch.int32, device=dev))
    else:
        keep = dict(db=DeviceBatch(hb), inputs=inputs, cmd=torch.zeros((hb.B, 4), dtype=torch.float64, device=dev),
                    path=torch.full((hb.B,), -2, dtype=torch.int32, device=dev))
    db, dcmd, dpath, ins = keep["db"], keep["cmd"], keep["path"], keep["inputs"]
    g.plan_device(db.bs, args, dcmd, start=ins[0], goal=ins[1], path=dpath, initial_plan=ins[2], plan_count=ins[3],
                  look_ahead_poses=look, prevent_near_goal=prevent, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    d = db.read()
    for k in ("poses", "n", "status", "lm_iters", "cost", "chi2"):
        assert np.array_equal(getattr(h, k), getattr(d, k), equal_nan=True), k
    assert np.array_equal(cmd, dcmd.cpu().numpy(), equal_nan=True)
    assert np.array_equal(path, dpath.cpu().numpy())
    return h, cmd, path


def _normalize_theta(t):
    """g2o::normalize_theta"""
    if -math.pi <= t < math.pi:
        return t
    t = t - math.floor(t / (2 * math.pi)) * 2 * math.pi
    if t >= math.pi:
        t -= 2 * math.pi
    if t < -math.pi:
        t += 2 * math.pi
    return t


def _expected_path(rec, n, goal, dist, ang):
    if n == 0:
        return abi.TEB_PLAN_PATH_COLD
    bx, by, bt = rec[n - 1, :3]
    dx, dy = goal[0] - bx, goal[1] - by
    near = math.sqrt(dx * dx + dy * dy) < dist and abs(_normalize_theta(goal[2] - bt)) < ang
    return abi.TEB_PLAN_PATH_WARM if near else abi.TEB_PLAN_PATH_REINIT


def _velocity_command(rec, n, look, prevent, dt_ref, max_vel_y):
    """getVelocityCommand (optimal_planner.cpp:1135-1168) restated"""
    if n < 2:
        return [0.0, 0.0, 0.0, 0.0]
    target = max(1, min(look, n - 1 - prevent))
    dt = 0.0
    for k in range(target):
        dt += rec[k, 3]
        if dt >= dt_ref * target:
            target = k + 1
            break
    if dt <= 0:
        return [0.0, 0.0, 0.0, 0.0]
    p1, p2 = rec[0], rec[target]
    sx, sy = p2[0] - p1[0], p2[1] - p1[1]
    c, s = math.cos(p1[2]), math.sin(p1[2])
    along = c * sx + s * sy
    if max_vel_y == 0:
        vx, vy = float(np.sign(along)) * math.sqrt(sx * sx + sy * sy) / dt, 0.0
    else:
        vx, vy = along / dt, (-s * sx + c * sy) / dt
    return [vx, vy, _normalize_theta(p2[2] - p1[2]) / dt, 1.0]


def _band(rng, n):
    x = np.cumsum(rng.uniform(0.05, 0.3, n))
    y = np.cumsum(rng.normal(0, 0.04, n))
    th = np.arctan2(np.gradient(y), np.gradient(x)) + rng.normal(0, 0.05, n) if n > 1 else np.zeros(n)
    dt = rng.uniform(0.05, 0.6, n)
    dt[-1] = 0
    return np.stack([x, y, th, dt], 1)


def test_cold_start(host_op):
    """n == 0: initTrajectoryToGoal(start, goal, 0, max_vel_x, min_samples, backwards) - random pairs, the goal behind
    the start, start == goal; same n as the host layer and the oracle, poses within 1e-12"""
    rng = np.random.default_rng(11)
    args = abi.make_args(0, 0, False)
    worst = 0.0
    B = 16
    for min_samples in range(3, 21):
        for backwards in (0, 1):
            p = _params(min_samples, backwards)
            hb = _empty_batch(B)
            s = np.stack([rng.uniform(-3, 3, B), rng.uniform(-3, 3, B), rng.uniform(-math.pi, math.pi, B)], 1)
            g_ = np.stack([rng.uniform(-3, 3, B), rng.uniform(-3, 3, B), rng.uniform(-math.pi, math.pi, B)], 1)
            g_[0] = s[0]                                                        # start == goal
            g_[1, :2] = s[1, :2] - 2.0 * np.array([math.cos(s[1, 2]), math.sin(s[1, 2])])   # goal behind the start
            g = _gpu(hb, p)
            h, cmd, path = _both(g, hb, args, s, g_)
            g.close()
            assert (path == abi.TEB_PLAN_PATH_COLD).all()
            for b in range(B):
                ref = host_op(1, None, list(s[b]) + list(g_[b]) + [0.0, p.max_vel_x, min_samples, backwards]).reshape(-1, 4)
                orc = ob.init_trajectory(s[b], g_[b], 0.0, p.max_vel_x, min_samples, bool(backwards))
                assert h.n[b] == len(ref) == len(orc)
                worst = max(worst, np.abs(h.poses[b, :h.n[b]] - ref).max(), np.abs(h.poses[b, :h.n[b]] - orc).max())
    print(f"cold start: worst |device - host| = {worst:.3e}")
    assert worst <= 1e-12


def _line_band(n, step=0.5):
    """poses on the x axis at dyadic coordinates, so distances and ties between them are exact"""
    rec = np.zeros((n, 4))
    rec[:, 0] = step * np.arange(n)
    rec[:, 3] = 0.25
    rec[-1, 3] = 0
    return rec


def test_warm_start_prune(host_op):
    """n > 0 and the goal close: updateAndPruneTEB - every prune index 0 .. 10, lookahead clipped by n - min_samples
    (zero, negative), a distance tie, the start exactly on a pose, n == n_cap; surviving records bit equal"""
    cases = []
    for k in range(0, 11):                          # start just past pose k: poses 1 .. k are pruned (at most 10)
        cases.append((30, [0.5 * k + 0.125, 0.0625, 0.3]))
    cases += [(5, [1.3, 0.0, 0.0]), (3, [0.9, 0.0, 0.0]), (2, [0.6, 0.0, 0.0]), (1, [0.1, 0.0, 0.0]),   # lookahead 2, 0, -1, -2
              (30, [0.5 * 4 + 0.25, 0.0, 0.0]),     # tie between poses 4 and 5: stops at 4
              (30, [1.5, 0.0, 0.1]),                # exactly on pose 3
              (N_CAP, [0.5 * 7 + 0.125, 0.0, 0.0]),  # n == n_cap
              (30, [-0.3, 0.2, 0.0])]                # behind pose 0: nothing pruned
    B = len(cases)
    hb = _empty_batch(B)
    s = np.zeros((B, 3))
    goal = np.zeros((B, 3))
    for b, (n, st) in enumerate(cases):
        hb.poses[b, :n] = _line_band(n)
        hb.n[b] = n
        s[b] = st
        goal[b] = [hb.poses[b, n - 1, 0] + 0.0625, 0.03125, 0.25]
    p = _params(3)
    g = _gpu(hb, p)
    h, cmd, path = _both(g, hb, abi.make_args(0, 0, False), s, goal)
    g.close()
    assert (path == abi.TEB_PLAN_PATH_WARM).all()
    expect_pruned = list(range(11)) + [2, 0, 0, 0, 4, 3, 7, 0]
    for b, (n, _) in enumerate(cases):
        ref = host_op(4, hb.poses[b, :n], list(s[b]) + list(goal[b]) + [3]).reshape(-1, 4)
        assert h.n[b] == len(ref) == n - min(expect_pruned[b], 10), (b, h.n[b], len(ref))
        assert np.array_equal(h.poses[b, :h.n[b]], ref), b
        assert np.array_equal(h.poses[b, h.n[b] - 1, :3], goal[b])
        assert h.n[b] == 1 or np.array_equal(h.poses[b, 0, :3], s[b])   # one pose: the goal overwrites the start


def test_reinit_decision(host_op):
    """goal distance exactly at force_reinit_new_goal_dist, the angle exactly at force_reinit_new_goal_angular (both
    re-initialise: the test is strict), a goal heading across +-pi; the same path code as the host"""
    p = _params(3)
    p.force_reinit_new_goal_dist, p.force_reinit_new_goal_angular = 0.75, 0.5
    back = [(2.0, 0.0, 0.0)] * 6 + [(2.0, 0.0, 3.1), (2.0, 0.0, -3.1), (2.0, 0.0, 3.1)]
    goals = [(2.75, 0.0, 0.0), (2.5, 0.0, 0.0), (2.0, 0.0, 0.5), (2.0, 0.0, 0.25), (2.0, 0.75, -0.5), (2.45, 0.6, 0.0),
             (2.0, 0.0, -3.1), (2.0, 0.0, 3.0), (2.0, 0.0, -2.5)]
    B = len(goals)
    hb = _empty_batch(B)
    for b in range(B):
        hb.poses[b, :5] = _line_band(5)
        hb.poses[b, 4, :3] = back[b]
        hb.n[b] = 5
    s = np.tile([0.1, 0.0, 0.0], (B, 1))
    goal = np.array(goals, float)
    g = _gpu(hb, p)
    h, cmd, path = _both(g, hb, abi.make_args(0, 0, False), s, goal)
    g.close()
    want = [_expected_path(hb.poses[b], 5, goal[b], 0.75, 0.5) for b in range(B)]
    assert list(path) == want
    assert want[:5] == [2, 1, 2, 1, 2] and want[6:] == [1, 1, 2]
    for b in range(B):
        if want[b] == abi.TEB_PLAN_PATH_REINIT:
            ref = host_op(1, None, list(s[b]) + list(goal[b]) + [0.0, p.max_vel_x, 3, 0]).reshape(-1, 4)
            assert h.n[b] == len(ref) and np.abs(h.poses[b, :h.n[b]] - ref).max() <= 1e-12


@pytest.mark.parametrize("overwrite", [0, 1])
def test_initial_plan(host_op, overwrite):
    """plan(initial_plan): plan lengths 1, 2, min_samples - 1 and P_cap, orientation estimated or taken; a plan that
    needs more than n_cap poses gets TEB_STATUS_CAPACITY and leaves the band untouched"""
    rng = np.random.default_rng(12 + overwrite)
    min_samples = 6
    p = _params(min_samples, backwards=1, overwrite=overwrite)
    lens = [1, 2, min_samples - 1, P_CAP] * 3
    B = len(lens)
    plan = np.zeros((B, P_CAP, 3))
    for b in range(B):
        pts = np.cumsum(rng.normal(0.2, 0.3, (P_CAP, 2)), 0) * (-1 if b % 2 else 1)
        plan[b] = np.concatenate([pts, rng.uniform(-math.pi, math.pi, (P_CAP, 1))], 1)
    count = np.array(lens, np.int32)
    worst = 0.0
    for n_cap in (N_CAP, P_CAP - 2):                 # at P_CAP - 2 records a P_cap-point plan does not fit
        hb = _empty_batch(B, n_cap=n_cap)
        hb.poses[:] = 7.0                              # what a band left untouched still holds
        g = _gpu(hb, p)
        h, cmd, path = _both(g, hb, abi.make_args(0, 0, False), plan=plan, count=count)
        g.close()
        for b in range(B):
            P = count[b]
            if max(P - 1, 1, min_samples - 1) + 1 > hb.n_cap:
                assert h.status[b] & abi.TEB_STATUS_CAPACITY and path[b] == abi.TEB_PLAN_PATH_NONE
                assert h.n[b] == 0 and np.array_equal(h.poses[b], hb.poses[b])
                continue
            ref = host_op(2, None, [p.max_vel_x, p.max_vel_theta, overwrite, min_samples, 1, P] + plan[b, :P].reshape(-1).tolist())
            ref = ref.reshape(-1, 4)
            assert path[b] == abi.TEB_PLAN_PATH_COLD and h.n[b] == len(ref)
            worst = max(worst, np.abs(h.poses[b, :h.n[b]] - ref).max())
    print(f"initial plan: worst |device - host| = {worst:.3e}")
    assert worst <= 1e-12


def test_velocity_command(host_op):
    """getVelocityCommand after the cycle: look_ahead_poses from 1 to past n, prevent_look_ahead_poses_near_goal, the
    early exit on dt_ref, dt <= 0 and n < 2 (ok = 0, zeros), holonomic and not"""
    rng = np.random.default_rng(13)
    B = 24
    hb = _empty_batch(B)
    for b in range(B):
        n = 1 if b == 0 else int(rng.integers(2, 30))
        rec = _band(rng, n)
        if b == 1:
            rec[:, 3] = 0.0                          # dt <= 0
        if b == 2:
            rec[:, 3] = 0.05                         # no early exit
        hb.poses[b, :n], hb.n[b] = rec, n
    s = hb.poses[:, 0, :3].copy()                    # start on pose 0, goal on the last pose: nothing pruned
    goal = np.stack([hb.poses[b, hb.n[b] - 1, :3] for b in range(B)])
    for max_vel_y in (0.0, 0.3):
        for look, prevent in ((1, 0), (3, 0), (7, 0), (40, 0), (5, 2), (40, 3)):
            p = _params(3)
            p.max_vel_y = max_vel_y
            g = _gpu(hb, p)
            h, cmd, path = _both(g, hb, abi.make_args(0, 0, False), s, goal, look, prevent)
            g.close()
            for b in range(B):
                n = h.n[b]
                want = _velocity_command(h.poses[b], n, look, prevent, p.dt_ref, max_vel_y)
                assert cmd[b, 3] == want[3], (b, look, prevent)
                assert np.abs(cmd[b, :3] - want[:3]).max() <= 1e-12, (b, cmd[b], want)
                if prevent == 0:
                    ref = host_op(8, h.poses[b, :n], [look, max_vel_y])
                    assert ref[0] == cmd[b, 3] and np.abs(cmd[b, :3] - ref[1:]).max() <= 1e-12
                if cmd[b, 3] == 0:
                    assert (cmd[b, :3] == 0).all()
    assert cmd[0, 3] == 0 and cmd[1, 3] == 0


def _move(start, cmd, period=0.2):
    """the robot follows its command for one control period"""
    th = start[:, 2]
    vx, vy, om = cmd[:, 0], cmd[:, 1], cmd[:, 2]
    out = start.copy()
    out[:, 0] += (vx * np.cos(th) - vy * np.sin(th)) * period
    out[:, 1] += (vx * np.sin(th) + vy * np.cos(th)) * period
    out[:, 2] = np.arctan2(np.sin(th + om * period), np.cos(th + om * period))
    return out


@pytest.mark.parametrize("name,requests", [("C1", 1), ("C3", 20)])
def test_whole_cycles(host_op, name, requests):
    """10 planning cycles on C1 (latency regime) and C3 (throughput regime) batches: path codes, n, status, LM
    iterations identical to the host-buffer loop (host updateAndPruneTEB + tebgpu_optimize_batch) and poses within
    1e-9, each cycle started from the device's state; graph replay on and off give the same bits, and a cycle repeated on
    the same buffers captures no new graph. C3 x 20 requests = 2560 bands: the throughput regime on 132 SMs."""
    p, hb0 = scenes.make_config_batch(name, requests=requests)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True)
    B = hb0.B
    goal = np.stack([hb0.poses[b, hb0.n[b] - 1, :3] for b in range(B)]) + [0.01, 0.0, 0.0]
    start = hb0.poses[:, 0, :3].copy()
    g_on = _gpu(hb0, p, graph=1)
    g_off = _gpu(hb0, p, graph=0)
    g_host = _gpu(hb0, p)
    cur = hb0.copy()
    graphs = None
    keep_on, keep_off = {}, {}
    for cycle in range(10):
        h_on, cmd, path = _both(g_on, cur, args, start, goal, look=2, keep=keep_on)
        h_off, cmd_off, path_off = _both(g_off, cur, args, start, goal, look=2, keep=keep_off)
        for k in ("poses", "n", "status", "lm_iters", "cost", "chi2"):
            assert np.array_equal(getattr(h_on, k), getattr(h_off, k), equal_nan=True), (cycle, k)
        assert np.array_equal(cmd, cmd_off) and np.array_equal(path, path_off)
        # the host-buffer loop from the same state
        ref = cur.copy()
        want_path = []
        for b in range(B):
            n = ref.n[b]
            want_path.append(_expected_path(ref.poses[b], n, goal[b], p.force_reinit_new_goal_dist, p.force_reinit_new_goal_angular))
            assert want_path[-1] == abi.TEB_PLAN_PATH_WARM
            out = host_op(4, ref.poses[b, :n], list(start[b]) + list(goal[b]) + [p.min_samples]).reshape(-1, 4)
            ref.poses[b] = 0
            ref.poses[b, :len(out)], ref.n[b] = out, len(out)
        g_host.optimize(ref, args)
        assert list(path) == want_path
        for k in ("n", "status", "lm_iters"):
            assert np.array_equal(getattr(h_on, k), getattr(ref, k)), (cycle, k)
        for b in range(B):
            assert np.abs(h_on.poses[b, :h_on.n[b]] - ref.poses[b, :ref.n[b]]).max() <= 1e-9, (cycle, b)
        for b in range(B):
            want = _velocity_command(h_on.poses[b], h_on.n[b], 2, 0, p.dt_ref, p.max_vel_y)
            assert cmd[b, 3] == want[3] and np.abs(cmd[b, :3] - want[:3]).max() <= 1e-12
        if graphs is None:
            graphs = g_on.info(6)
        assert g_on.info(6) == graphs                 # same buffers, same key: replayed, not captured again
        cur = h_on
        start = _move(h_on.poses[:, 0, :3], cmd)
    for g in (g_on, g_off, g_host):
        g.close()


def test_plan_launch_count_leaves_optimize_alone():
    """the plan cycle adds its two launches to the optimize sequence; a plain optimize is unchanged by a plan call"""
    p, hb = scenes.make_config_batch("C1")
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True)
    g = _gpu(hb, p, graph=0)
    h = hb.copy()
    g.optimize(h, args)
    plain = g.launch_count()
    s = hb.poses[:, 0, :3].copy()
    goal = np.stack([hb.poses[b, hb.n[b] - 1, :3] for b in range(hb.B)])
    g.plan(hb.copy(), s, goal, args)
    assert g.launch_count() == plain + 2
    h2 = hb.copy()
    g.optimize(h2, args)
    assert g.launch_count() == plain
    assert np.array_equal(h.poses, h2.poses) and np.array_equal(h.lm_iters, h2.lm_iters)
    g.close()


def test_input_errors():
    """non-finite start / goal / plan rows and a plan_count outside 1 .. P_cap: TEBGPU_ERR_INVALID_ARG from the host
    entry point, TEB_STATUS_BAD_INPUT for that band (left untouched, path -1) from the device entry point; the other
    bands are planned as without the bad one"""
    B = 6
    hb = _empty_batch(B)
    rng = np.random.default_rng(14)
    s = np.stack([rng.uniform(-1, 1, B), rng.uniform(-1, 1, B), rng.uniform(-1, 1, B)], 1)
    goal = s + [2.0, 0.5, 0.3]
    p = _params(5)
    g = _gpu(hb, p)
    args = abi.make_args(0, 0, False)
    _, good_cmd, _ = _both(g, hb, args, s, goal)
    good = hb.copy()
    g.plan(good, s, goal, args)
    dev = torch.device("cuda:0")
    for what in ("start", "goal"):
        bad_s, bad_g = s.copy(), goal.copy()
        (bad_s if what == "start" else bad_g)[2, 1] = np.nan
        with pytest.raises(T.TebGpuError, match="rc=-1"):
            g.plan(hb.copy(), bad_s, bad_g, args)
        db = DeviceBatch(hb)
        cmd = torch.zeros((B, 4), dtype=torch.float64, device=dev)
        path = torch.zeros(B, dtype=torch.int32, device=dev)
        ts, tg = torch.from_numpy(bad_s).to(dev), torch.from_numpy(bad_g).to(dev)
        g.plan_device(db.bs, args, cmd, start=ts, goal=tg, path=path, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        d = db.read()
        assert d.status[2] & abi.TEB_STATUS_BAD_INPUT and path[2].item() == -1 and d.n[2] == 0
        others = [b for b in range(B) if b != 2]
        assert np.array_equal(d.poses[others], good.poses[others]) and np.array_equal(d.n[others], good.n[others])
        assert np.array_equal(cmd.cpu().numpy()[others], good_cmd[others])
        assert not (d.status[others] & abi.TEB_STATUS_BAD_INPUT).any()
    plan = np.tile(np.linspace([0, 0, 0], [2, 1, 0.5], P_CAP), (B, 1, 1))
    for bad_count, bad_row in ((0, None), (P_CAP + 1, None), (P_CAP, 3)):
        count = np.full(B, P_CAP, np.int32)
        count[4] = bad_count
        pl = plan.copy()
        if bad_row is not None:
            pl[4, bad_row, 2] = np.inf
        with pytest.raises(T.TebGpuError, match="rc=-1"):
            g.plan(hb.copy(), None, None, args, initial_plan=pl, plan_count=count)
        db = DeviceBatch(hb)
        cmd = torch.zeros((B, 4), dtype=torch.float64, device=dev)
        path = torch.zeros(B, dtype=torch.int32, device=dev)
        g.plan_device(db.bs, args, cmd, path=path, initial_plan=torch.from_numpy(pl).to(dev),
                      plan_count=torch.from_numpy(count).to(dev), stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        d = db.read()
        assert d.status[4] & abi.TEB_STATUS_BAD_INPUT and path[4].item() == -1 and d.n[4] == 0
        assert (path.cpu().numpy()[[0, 1, 2, 3, 5]] == abi.TEB_PLAN_PATH_COLD).all()
    g.close()
