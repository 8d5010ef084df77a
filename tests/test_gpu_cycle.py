"""The controller steps around plan() on the device (tebgpu_backup_modes / tebgpu_finish_cycle and their _device forms,
teb_cycle.cuh) held to the restatement of tests/cycle_cases.py: every output and state array bit equal, except vx / vy
after the trans cut (CUDA hypot, within 4 ulp) and the steering angle (CUDA atan, within 1e-15). Multi-cycle runs step the
restatement from the device's previous state, so a last-ulp difference cannot compound. Also host bits == device bits,
batch-position invariance, untouched skipped bands, the out-of-range-state codes, argument errors that launch nothing, and
a closed costmap -> local plan -> backup modes -> plan -> check -> finish loop on one stream, held to the same loop with
both new steps restated on the host."""
import ctypes as C
import math

import numpy as np
import pytest

import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes
from tests import cycle_cases as cc

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DEV = "cuda:0"
NOW = 100.0
STATE_KEYS = abi.CYCLE_STATE


def params(**kw):
    p = abi.default_params()
    p.max_vel_trans = p.max_vel_x
    p.divergence_detection_enable, p.divergence_detection_max_chi_squared = 1, 10.0
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.fixture(scope="module")
def gpu():
    g = T.TebGpu(4096, 64, 1, 64, 0)
    yield g
    g.close()


def fleet(B, L, cap, seed):
    """a random fleet at every boundary: codes, counters near INT32_MAX, stamps around `recently`, rocking and moving
    last commands with signed zeros and NaNs, rings of every fill and head"""
    rng = np.random.default_rng(seed)
    st = abi.make_cycle_state(B, L)
    st["infeasible_count"][:] = rng.choice([0, 1, 9, 10, cc.INT32_MAX - 1, cc.INT32_MAX], B)
    st["last_infeasible"][:] = rng.choice([-np.inf, 0.0, 95.0, NOW], B)
    st["last_oscillation"][:] = rng.choice([-np.inf, NOW - 10.0, NOW - 9.5, NOW - 20.0], B)
    rock = np.stack([rng.normal(0, 0.01, B), np.zeros(B), np.where(rng.random(B) < 0.5, 1, -1) * rng.uniform(0, 0.03, B)], 1)
    moving = rng.uniform(-0.6, 0.6, (B, 3))
    st["last_cmd"][:] = np.where(rng.random((B, 1)) < 0.6, rock, moving)
    st["last_cmd"][rng.random(B) < 0.05, 0] = -0.0
    st["last_cmd"][rng.random(B) < 0.03, 2] = np.nan
    st["prefer_rotdir"][:] = rng.integers(0, 3, B)
    if L:
        st["osc_ring"][:] = np.stack([rng.normal(0, 0.02, (L, B)), np.resize([0.03, -0.03], (L, B)) *
                                      rng.uniform(0, 1, (L, B))], 2)
    st["osc_fill"][:, 0] = rng.integers(0, cap + 1, B)
    st["osc_fill"][:, 1] = rng.integers(0, max(cap, 1), B)
    ins = dict(
        robot_vel=np.where(rng.random((B, 3)) < 0.2, 0.0, rng.normal(0, 0.3, (B, 3))),
        lpr=rng.choice([0, 0, 0, 0, 1, 2, 3, 4], B).astype(np.int32),
        n=rng.integers(0, 50, B).astype(np.int32),
        status=rng.choice([1, 1, 1, 1 | 16, 0, 1 | 64, 1 | 128, 2], B).astype(np.int32),
        chi2=rng.choice([1.0, 10.0, 11.0, np.nan], B),
        cmd=np.concatenate([rng.uniform(-1.0, 1.0, (B, 3)), rng.choice([1.0, 1.0, 1.0, 0.0], (B, 1))], 1),
        feasible=rng.choice([1, 1, 1, 0, -1], B).astype(np.int32))
    ins["robot_vel"][rng.random(B) < 0.05, 2] = np.nan
    ins["cmd"][rng.random(B) < 0.05, 0] = np.nan
    ins["cmd"][rng.random(B) < 0.05, 2] = -0.0
    return st, ins


def ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    same = (a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))
    return np.where(same, 0.0, np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b))))


def assert_same(got, want, steering=False, label=""):
    for k, w in want.items():
        g = got[k]
        if k in ("cmd_vel", "last_cmd"):
            assert (ulps(g[:, :2], w[:, :2]) <= 4).all(), (label, k)
            if steering:
                d = np.abs(g[:, 2] - w[:, 2])
                assert ((d <= 1e-15) | (np.isnan(g[:, 2]) & np.isnan(w[:, 2]))).all(), (label, k)
            else:
                assert (ulps(g[:, 2], w[:, 2]) == 0).all(), (label, k)
        else:
            assert np.asarray(g).tobytes() == np.asarray(w).tobytes(), (label, k)


def _t(x, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV) if x is not None else None


def _p(t):
    return None if t is None else t.data_ptr()


def run_device(g, step, st, ins, now=NOW, feasible=True, lpr=True, **scalars):
    """one step through the _device entry point on torch tensors; returns the state and outputs as numpy"""
    B = len(st["prefer_rotdir"])
    L = st["osc_ring"].shape[0]
    scalars.setdefault("buffer_length", L)
    d = {k: _t(v.copy()) for k, v in st.items()}
    x = dict(robot_vel=_t(ins["robot_vel"]), lpr=_t(ins["lpr"]) if lpr else None, cmd=_t(ins["cmd"]),
             feasible=_t(ins["feasible"]) if feasible else None, n=_t(ins["n"].copy()), status=_t(ins["status"]),
             chi2=_t(ins["chi2"]), cmd_vel=torch.zeros((B, 3), dtype=torch.float64, device=DEV),
             outcome=torch.full((B,), -2, dtype=torch.int32, device=DEV),
             oscillating=torch.full((B,), -2, dtype=torch.int32, device=DEV))
    ca = abi.make_cycle_args(now, L_cap=L, **scalars, local_plan_result=_p(x["lpr"]), robot_vel=_p(x["robot_vel"]),
                             cmd=_p(x["cmd"]), feasible=_p(x["feasible"]), cmd_vel=_p(x["cmd_vel"]),
                             outcome=_p(x["outcome"]), oscillating=_p(x["oscillating"]),
                             **{k: (_p(d[k]) if d[k].numel() else None) for k in STATE_KEYS})
    bs = abi.TebBatch()
    bs.B, bs.n, bs.status, bs.chi2 = B, _p(x["n"]), _p(x["status"]), _p(x["chi2"])
    (g.backup_modes_device if step == "backup" else g.finish_cycle_device)(bs, ca)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in d.items()}
    if step == "backup":
        out["oscillating"] = x["oscillating"].cpu().numpy()
    else:
        out.update(n=x["n"].cpu().numpy(), cmd_vel=x["cmd_vel"].cpu().numpy(), outcome=x["outcome"].cpu().numpy())
    return out


def run_host(g, step, st, ins, now=NOW, feasible=True, lpr=True, **scalars):
    if step == "backup":
        return g.backup_modes(st, ins["robot_vel"], now, ins["lpr"] if lpr else None, **scalars)
    return g.finish_cycle(st, ins["n"], ins["status"], ins["chi2"], ins["cmd"], now,
                          ins["feasible"] if feasible else None, ins["lpr"] if lpr else None, **scalars)


def restate(p, step, st, ins, now=NOW, feasible=True, lpr=True, **scalars):
    if step == "backup":
        return cc.backup_modes(st, ins["robot_vel"], now, p, ins["lpr"] if lpr else None, **scalars)
    return cc.finish_cycle(st, ins["n"], ins["status"], ins["chi2"], ins["cmd"], now, p,
                           ins["feasible"] if feasible else None, ins["lpr"] if lpr else None, **scalars)


SCALAR_SETS = [dict(), dict(use_proportional_saturation=True), dict(cmd_angle_instead_rotvel=True, wheelbase=-0.7),
               dict(cmd_angle_instead_rotvel=True, use_proportional_saturation=True, wheelbase=1.3),
               dict(oscillation_recovery=False), dict(oscillation_v_eps=0.3, oscillation_omega_eps=0.5,
                                                      oscillation_recovery_min_duration=0.0)]
PARAM_SETS = [dict(), dict(max_vel_y=0.3, max_vel_trans=0.45), dict(min_turning_radius=0.5, max_vel_x_backwards=0.0),
              dict(max_vel_trans=0.0, min_turning_radius=-0.4), dict(divergence_detection_enable=0)]


@pytest.mark.parametrize("cap", [0, 1, 2, 7, 10, 50])
@pytest.mark.parametrize("j", range(len(SCALAR_SETS)))
def test_both_steps_match_the_restatement(gpu, cap, j):
    for i, pk in enumerate(PARAM_SETS):
        p = params(**pk)
        gpu.set_params(p)
        L = cap + (i % 2) * 3              # L_cap above buffer_length too
        st, ins = fleet(700, L, cap, seed=100 * cap + 10 * j + i)
        sc = dict(SCALAR_SETS[j], buffer_length=cap)
        for step in ("backup", "finish"):
            got = run_device(gpu, step, st, ins, **sc)
            want = restate(p, step, st, ins, **sc)
            assert_same(got, want, sc.get("cmd_angle_instead_rotvel", False), (step, i))
            assert got.keys() == want.keys()
            host = run_host(gpu, step, st, ins, **sc)
            for k in got:
                assert np.asarray(host[k]).tobytes() == np.asarray(got[k]).tobytes(), (step, k)


@pytest.mark.parametrize("feasible,lpr", [(False, True), (True, False), (False, False)])
def test_null_feasible_and_local_plan_result(gpu, feasible, lpr):
    p = params()
    gpu.set_params(p)
    st, ins = fleet(300, 10, 10, seed=7)
    for step in ("backup", "finish"):
        got = run_device(gpu, step, st, ins, feasible=feasible, lpr=lpr, buffer_length=10)
        assert_same(got, restate(p, step, st, ins, feasible=feasible, lpr=lpr, buffer_length=10))


@pytest.mark.parametrize("cap", [1, 4, 9])
def test_multi_cycle_runs_step_from_the_devices_state(gpu, cap):
    """3 x buffer_length cycles: the detector rings fill, wrap and recover; each cycle the restatement starts from the
    device's state"""
    p = params(min_turning_radius=0.3)
    gpu.set_params(p)
    st, ins = fleet(512, cap, cap, seed=cap)
    st["osc_fill"][:] = 0
    rng = np.random.default_rng(cap)
    now = 50.0
    for k in range(3 * cap):
        ins["robot_vel"] = rng.normal(0, 0.2, (512, 3))
        ins["lpr"] = rng.choice([0, 0, 0, 0, 3, 1], 512).astype(np.int32)
        ins["status"] = rng.choice([1, 1, 1, 0], 512).astype(np.int32)
        rock = np.where(np.arange(512) % 3 == 0, (-1) ** k * 0.02, rng.uniform(-0.5, 0.5, 512))
        ins["cmd"] = np.stack([rng.normal(0, 0.01, 512), np.zeros(512), rock, np.ones(512)], 1)
        got = run_device(gpu, "backup", st, ins, now=now, buffer_length=cap, oscillation_recovery_min_duration=1.0)
        assert_same(got, restate(p, "backup", st, ins, now=now, buffer_length=cap,
                                 oscillation_recovery_min_duration=1.0), label=k)
        st = {kk: got[kk] for kk in STATE_KEYS}
        got = run_device(gpu, "finish", st, ins, now=now, buffer_length=cap)
        assert_same(got, restate(p, "finish", st, ins, now=now, buffer_length=cap), label=k)
        st = {kk: got[kk] for kk in STATE_KEYS}
        now += 0.2
    assert (st["prefer_rotdir"] != cc.ROT_NONE).any()


def test_results_do_not_depend_on_the_band_position(gpu):
    p = params()
    gpu.set_params(p)
    st, ins = fleet(1000, 12, 12, seed=3)
    perm = np.random.default_rng(4).permutation(1000)
    inv = np.argsort(perm)
    pst = {k: (v[:, perm] if k == "osc_ring" else v[perm]) for k, v in st.items()}
    pins = {k: v[perm] for k, v in ins.items()}
    for step in ("backup", "finish"):
        a = run_device(gpu, step, st, ins, buffer_length=12)
        b = run_device(gpu, step, pst, pins, buffer_length=12)
        for k in a:
            bk = b[k][:, inv] if k == "osc_ring" else b[k][inv]
            assert a[k].tobytes() == bk.tobytes(), (step, k)


def test_skipped_bands_are_untouched(gpu):
    p = params()
    gpu.set_params(p)
    st, ins = fleet(256, 8, 8, seed=5)
    got = run_device(gpu, "backup", st, ins, buffer_length=8)
    skip = (ins["lpr"] == cc.GOAL_REACHED) | (ins["lpr"] == cc.EMPTY) | (ins["lpr"] == cc.BAD_INPUT)
    assert skip.any() and (got["oscillating"][skip] == -2).all()
    for k in STATE_KEYS:
        g, w = (got[k][:, skip], st[k][:, skip]) if k == "osc_ring" else (got[k][skip], st[k][skip])
        assert g.tobytes() == w.tobytes(), k
    assert ((got["oscillating"][~skip] == 0) | (got["oscillating"][~skip] == 1)).all()


def test_out_of_range_state_codes(gpu):
    p = params()
    gpu.set_params(p)
    st, ins = fleet(64, 6, 6, seed=6)
    ins["lpr"][:] = 0
    ins["lpr"][1], ins["lpr"][2] = 5, -1
    st["osc_fill"][3] = (7, 0)
    st["osc_fill"][4] = (2, 6)
    st["osc_fill"][5] = (-1, 0)
    st["prefer_rotdir"][6] = 3
    ins["feasible"][7] = 2
    bad_b, bad_f = [1, 2, 3, 4, 5, 6], [1, 2, 7]
    got = run_device(gpu, "backup", st, ins, buffer_length=6)
    assert (got["oscillating"][bad_b] == -1).all()
    for k in STATE_KEYS:
        g, w = (got[k][:, bad_b], st[k][:, bad_b]) if k == "osc_ring" else (got[k][bad_b], st[k][bad_b])
        assert g.tobytes() == w.tobytes(), k
    got = run_device(gpu, "finish", st, ins, buffer_length=6)
    assert (got["outcome"][bad_f] == cc.NO_PLAN).all() and (got["cmd_vel"][bad_f] == 0).all()
    assert (got["n"][bad_f] == ins["n"][bad_f]).all() and (got["infeasible_count"][bad_f] == st["infeasible_count"][bad_f]).all()
    assert_same(got, restate(p, "finish", st, ins, buffer_length=6))
    for bad in ([1], [3], [4], [5], [6]):
        s2, i2 = fleet(64, 6, 6, seed=6)
        i2["lpr"][:] = 0
        for b in bad:
            i2["lpr"][b], s2["osc_fill"][b], s2["prefer_rotdir"][b] = ins["lpr"][b], st["osc_fill"][b], st["prefer_rotdir"][b]
        with pytest.raises(T.TebGpuError, match="rc=-1"):
            run_host(gpu, "backup", s2, i2, buffer_length=6)
    i2 = dict(ins, lpr=np.zeros(64, np.int32))
    with pytest.raises(T.TebGpuError, match="rc=-1"):
        run_host(gpu, "finish", st, i2, buffer_length=6)


def test_argument_errors_launch_nothing(gpu):
    p = params()
    gpu.set_params(p)
    B = 16
    st, ins = fleet(B, 4, 4, seed=8)
    run_device(gpu, "finish", st, ins, buffer_length=4)
    grid = gpu.last_cycle_grid()
    assert grid == 1
    L = gpu.lib
    for step in ("backup", "finish"):
        fn, fnd = ((L.tebgpu_backup_modes, L.tebgpu_backup_modes_device) if step == "backup"
                   else (L.tebgpu_finish_cycle, L.tebgpu_finish_cycle_device))
        req = (["robot_vel", "last_cmd", "prefer_rotdir", "last_oscillation", "osc_fill", "osc_ring"] if step == "backup"
               else ["cmd", "infeasible_count", "last_infeasible", "last_cmd", "cmd_vel", "outcome"])
        breq = [] if step == "backup" else ["n", "status", "chi2"]

        def call(mod=None, bmod=None, host=True, **sc):
            s = {k: v.copy() for k, v in st.items()}
            outc = np.full(B, 77, np.int32)
            osc = np.full(B, 77, np.int32)
            cv = np.full((B, 3), 77.0)
            n, status, chi2 = ins["n"].copy(), ins["status"].copy(), ins["chi2"].copy()
            ca = abi.make_cycle_args(sc.pop("now", NOW), **dict(dict(buffer_length=4, L_cap=4), **sc),
                                     local_plan_result=abi.ptr(ins["lpr"]), robot_vel=abi.ptr(ins["robot_vel"]),
                                     cmd=abi.ptr(ins["cmd"]), feasible=abi.ptr(ins["feasible"]), cmd_vel=abi.ptr(cv),
                                     outcome=abi.ptr(outc), oscillating=abi.ptr(osc),
                                     **{k: abi.ptr(s[k]) for k in STATE_KEYS})
            bs = abi.TebBatch()
            bs.B, bs.n, bs.status, bs.chi2 = B, abi.ptr(n), abi.ptr(status), abi.ptr(chi2)
            if mod:
                setattr(ca, mod, None)
            if bmod:
                setattr(bs, *bmod)
            rc = fn(gpu.ctx, C.byref(bs), C.byref(ca)) if host else fnd(gpu.ctx, C.byref(bs), C.byref(ca), None)
            assert (outc == 77).all() and (osc == 77).all() and (cv == 77.0).all() and (n == ins["n"]).all()
            for k in STATE_KEYS:
                assert s[k].tobytes() == st[k].tobytes()
            return rc

        for host in (True, False):
            for k in req:
                assert call(mod=k, host=host) == abi.TEBGPU_ERR_INVALID_ARG, (step, k)
            for k in breq:
                assert call(bmod=(k, None), host=host) == abi.TEBGPU_ERR_INVALID_ARG, (step, k)
            assert call(bmod=("B", 0), host=host) == abi.TEBGPU_ERR_INVALID_ARG
            assert call(bmod=("B", 4097), host=host) == abi.TEBGPU_ERR_INVALID_ARG
            assert call(host=host, L_cap=-1, buffer_length=0) == abi.TEBGPU_ERR_INVALID_ARG
            assert call(host=host, L_cap=4, buffer_length=5) == abi.TEBGPU_ERR_INVALID_ARG
            assert call(host=host, buffer_length=-1) == abi.TEBGPU_ERR_INVALID_ARG
            for now in (math.nan, math.inf, -math.inf):
                assert call(host=host, now=now) == abi.TEBGPU_ERR_INVALID_ARG
        assert fn(gpu.ctx, None, None) == abi.TEBGPU_ERR_INVALID_ARG
    assert gpu.last_cycle_grid() == grid


def test_a_direction_set_by_the_step_plans_as_one_set_directly():
    p, hb0 = scenes.make_config_batch("C2", candidates=8, seed=3)
    p.weight_prefer_rotdir = 50.0
    p.max_vel_trans = p.max_vel_x
    g = T.TebGpu(hb0.B, hb0.n_cap, hb0.S, hb0.M_cap, hb0.V_cap)
    g.set_params(p)
    B = hb0.B
    st = abi.make_cycle_state(B, 4)
    st["osc_ring"][:3, :, 1] = np.array([0.01, -0.01, 0.01])[:, None]
    st["osc_fill"][:] = (3, 0)
    st["last_cmd"][:, 2] = -0.003
    vel = np.zeros((B, 3))
    vel[::2, 2] = 0.1
    out = g.backup_modes(st, vel, NOW, buffer_length=4)
    direct = np.where(np.arange(B) % 2 == 0, abi.TEB_ROTDIR_LEFT, abi.TEB_ROTDIR_RIGHT).astype(np.int32)
    assert (out["oscillating"] == 1).all() and (out["prefer_rotdir"] == direct).all()
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    runs = []
    for rot in (out["prefer_rotdir"], direct.copy(), np.zeros(B, np.int32)):
        hb = hb0.copy()
        hb.prefer_rotdir = np.ascontiguousarray(rot, np.int32)
        g.optimize(hb, args)
        runs.append(hb)
    g.close()
    assert runs[0].poses.tobytes() == runs[1].poses.tobytes() and runs[0].cost.tobytes() == runs[1].cost.tobytes()
    assert runs[0].poses.tobytes() != runs[2].poses.tobytes()


# ---- the closed loop: costmap -> local plan -> backup modes -> plan -> check -> finish on one stream

def _closed_loop(restated, cycles=20, B=24, P_cap=160, M_cap=2048, n_cap=96, Lb=10):
    d = scenes.global_plans(B, 1024, S=B, seed=21)
    r = scenes.costmap_raster(B, 60, 60, 0.05, 0.03, seed=22)
    r["origin"][:, 0] = d["robot"][:, 0] - 1.5
    r["origin"][:, 1] = d["robot"][:, 1] - 1.5
    sx = 60
    for s in range(4, 8):          # a lethal blob under robots 4 .. 7: their plans collide at pose 0
        for my in range(27, 33):
            r["cost"][s, my * sx + 27: my * sx + 33] = 254
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 0
    p.max_vel_trans = p.max_vel_x
    g = T.TebGpu(B, n_cap, B, M_cap, 0)
    g.set_params(p)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=DEV)
    f64, i32 = torch.float64, torch.int32
    cost, grid, origin = t(r["cost"]), t(r["grid"]), t(r["origin"])
    robot = t(d["robot"].copy())
    obst, ocount = z(B * M_cap * 64, torch.uint8), z(B, i32)
    gp, begin, end = t(d["global_plan"]), t(d["plan_begin"].copy()), t(d["plan_end"])
    plan, pcount, result = z((B, P_cap, 3), f64), z(B, i32), z(B, i32)
    st0 = abi.make_cycle_state(B, Lb)
    for b in range(4):             # rings seeded to oscillate on the first cycle
        st0["osc_ring"][: Lb - 1, b, 1] = np.resize([0.01, -0.01], Lb - 1)
        st0["osc_fill"][b] = (Lb - 1, 0)
        st0["last_cmd"][b, 2] = 0.003 * (-1) ** b
    state = {k: t(v) for k, v in st0.items()}
    vel, since = z((B, 3), f64), z(B, f64)
    poses, n, sid = z((B, n_cap, 4), f64), z(B, i32), t(np.arange(B, dtype=np.int32))
    vs = np.zeros((B, 4))
    vs[:, 3] = 1.0
    vstart, vgoal = t(vs), t(vs)
    costo, chi2, status, iters = z(B, f64), z(B, f64), z(B, i32), z(B, i32)
    cmd, path, feas, qc = z((B, 4), f64), z(B, i32), z(B, i32), z(B, i32)
    cmd_vel, outcome, osc = z((B, 3), f64), z(B, i32), z(B, i32)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, B, M_cap, 0, 0
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
    bs.vel_start, bs.vel_goal, bs.prefer_rotdir = vstart.data_ptr(), vgoal.data_ptr(), state["prefer_rotdir"].data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = costo.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.include_costmap_obstacles, ca.behind_robot_dist = B, r["cost"].shape[1], M_cap, 1, 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = cost.data_ptr(), grid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    la = abi.make_local_plan_args(1024, P_cap, 0, max_lookahead_dist=2.0, global_plan=gp.data_ptr(),
                                  plan_begin=begin.data_ptr(), plan_end=end.data_ptr(), robot=robot.data_ptr(),
                                  robot_vel=vel.data_ptr(), grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  infeasible_count=state["infeasible_count"].data_ptr(), since_infeasible=since.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), result=result.data_ptr())
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    fa = abi.make_feasibility_args(0.1, max_queries=512, collision_distance=0.05, feasible=feas.data_ptr(),
                                   query_count=qc.data_ptr())
    sc = dict(buffer_length=Lb, oscillation_recovery_min_duration=2.0)
    dt, now = 0.2, 1000.0
    s = torch.cuda.Stream()
    trace = []
    for k in range(cycles):
        cy = abi.make_cycle_args(now, L_cap=Lb, **sc, local_plan_result=result.data_ptr(), robot_vel=vel.data_ptr(),
                                 cmd=cmd.data_ptr(), feasible=feas.data_ptr(), cmd_vel=cmd_vel.data_ptr(),
                                 outcome=outcome.data_ptr(), oscillating=osc.data_ptr(),
                                 **{kk: state[kk].data_ptr() for kk in STATE_KEYS})
        with torch.cuda.stream(s):
            since.copy_(now - state["last_infeasible"])
            g.costmap_obstacles_device(ca, stream=s.cuda_stream)
            g.local_plan_device(bs, la, stream=s.cuda_stream)
            if restated:
                s.synchronize()
                h = {kk: v.cpu().numpy() for kk, v in state.items()}
                o = cc.backup_modes(h, vel.cpu().numpy(), now, p, result.cpu().numpy(), **sc)
                for kk in STATE_KEYS:
                    state[kk].copy_(t(o[kk]))
                written = o["oscillating"] != -2      # a band the step skips keeps its previous answer
                osc.copy_(t(np.where(written, o["oscillating"], osc.cpu().numpy())))
            else:
                g.backup_modes_device(bs, cy, stream=s.cuda_stream)
            g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, path=path,
                          stream=s.cuda_stream)
            g.check_feasible_device(bs, fa, stream=s.cuda_stream)
            if restated:
                s.synchronize()
                h = {kk: v.cpu().numpy() for kk, v in state.items()}
                o = cc.finish_cycle(h, n.cpu().numpy(), status.cpu().numpy(), chi2.cpu().numpy(), cmd.cpu().numpy(),
                                    now, p, feas.cpu().numpy(), result.cpu().numpy(), **sc)
                for kk in STATE_KEYS:
                    state[kk].copy_(t(o[kk]))
                n.copy_(t(o["n"]))
                cmd_vel.copy_(t(o["cmd_vel"]))
                outcome.copy_(t(o["outcome"]))
            else:
                g.finish_cycle_device(bs, cy, stream=s.cuda_stream)
            # the robots follow their commands
            th = robot[:, 2]
            robot[:, 0] += (cmd_vel[:, 0] * torch.cos(th) - cmd_vel[:, 1] * torch.sin(th)) * dt
            robot[:, 1] += (cmd_vel[:, 0] * torch.sin(th) + cmd_vel[:, 1] * torch.cos(th)) * dt
            robot[:, 2] += cmd_vel[:, 2] * dt
            vel.copy_(cmd_vel)
        s.synchronize()
        rec = dict(n=n, status=status, path=path, cmd_vel=cmd_vel, outcome=outcome, oscillating=osc, result=result,
                   feasible=feas, **state)
        trace.append({kk: v.cpu().numpy().copy() for kk, v in rec.items()})
        now += dt
    g.close()
    return trace


def test_closed_loop_on_one_stream_matches_the_restated_steps():
    dev = _closed_loop(False)
    ref = _closed_loop(True)
    for k, (a, b) in enumerate(zip(dev, ref)):
        for key in a:
            assert a[key].tobytes() == b[key].tobytes(), (k, key)
    # the loop went through the branches: commands, failures at the blobs, an oscillation and its direction
    outs = np.concatenate([c["outcome"] for c in dev])
    assert (outs == cc.COMMAND).any() and (outs >= cc.PLAN_FAILED).any()
    assert (dev[0]["oscillating"][:4] == 1).all() and (dev[0]["prefer_rotdir"][:4] != cc.ROT_NONE).all()
    assert all((c["outcome"][4:8] != cc.COMMAND).all() for c in dev)
    assert (dev[-1]["infeasible_count"][4:8] > 0).all()
