"""The controller steps around plan() (tebgpu_backup_modes_device / tebgpu_finish_cycle_device) for N robots: each
kernel alone, and a closed loop with the tail of the cycle on the device against the same loop with the tail on the host.

  alone   k_backup_modes and k_finish_cycle over N robots with full detector rings (buffer_length 50), CUDA events
          around each launch, the median of --reps launches after 3 warm-up launches, at every --robots count;
  loop    every cycle, on one stream: tebgpu_local_plan_device, tebgpu_backup_modes_device, tebgpu_plan_batch_device,
          tebgpu_check_feasible_device, tebgpu_finish_cycle_device and a torch op that moves every robot by cmd_vel and
          feeds it back as its odometry; one synchronisation per K cycles. The host-tail loop runs the same device steps
          up to the check, then copies status, chi2, cmd, feasible, the local-plan result and n to the host, applies the
          outcome table and saturateVelocity there with numpy (vectorised, without the oscillation detector, so the
          comparison favours the host) and copies cmd_vel and n back before the move: one synchronisation per cycle.

    python tools/control_cycle.py --robots 1024 8192 --loop-robots 1024 --cycles 20 [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query)."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi, scenes  # noqa: E402
from tools.local_plan import card, move  # noqa: E402


def kernel_times(B, reps, torch):
    """median ms of each step alone over B robots whose rings are full"""
    dev = torch.device("cuda:0")
    L = 50
    g = T.TebGpu(B, 8, 1, 1, 0)
    p = abi.default_params()
    abi.make_cycle_args(0.0, params=p)
    g.set_params(p)
    rng = np.random.default_rng(1)
    st = abi.make_cycle_state(B, L)
    st["osc_ring"][:] = rng.normal(0, 0.05, st["osc_ring"].shape)
    st["osc_fill"][:] = (L, 0)
    st["last_cmd"][:] = rng.normal(0, 0.05, (B, 3))
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    d = {k: t(v) for k, v in st.items()}
    vel, cmd = t(rng.normal(0, 0.2, (B, 3))), t(np.concatenate([rng.normal(0, 0.3, (B, 3)), np.ones((B, 1))], 1))
    n, status, chi2 = t(np.full(B, 20, np.int32)), t(np.ones(B, np.int32)), t(np.ones(B))
    cmd_vel, outcome = torch.zeros((B, 3), dtype=torch.float64, device=dev), torch.zeros(B, dtype=torch.int32, device=dev)
    ca = abi.make_cycle_args(100.0, buffer_length=L, robot_vel=vel.data_ptr(), cmd=cmd.data_ptr(),
                             cmd_vel=cmd_vel.data_ptr(), outcome=outcome.data_ptr(),
                             **{k: d[k].data_ptr() for k in abi.CYCLE_STATE})
    bs = abi.TebBatch()
    bs.B, bs.n, bs.status, bs.chi2 = B, n.data_ptr(), status.data_ptr(), chi2.data_ptr()
    stream = torch.cuda.current_stream().cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    res = {}
    for name, fn in (("backup_modes", g.backup_modes_device), ("finish_cycle", g.finish_cycle_device)):
        ms = []
        for r in range(reps + 3):
            n.fill_(20)
            ev[0].record()
            fn(bs, ca, stream=stream)
            ev[1].record()
            torch.cuda.synchronize()
            if r >= 3:
                ms.append(ev[0].elapsed_time(ev[1]))
        res[name + "_ms"] = float(np.median(ms))
    res["grid_ctas"] = g.last_cycle_grid()
    g.close()
    return res


def host_tail(p, status, chi2, cmd, feas, result, n):
    """the finish step's outcome table and saturateVelocity in numpy (no detector, no steering angle)"""
    ok = ((status & abi.TEB_STATUS_OPTIMIZED) != 0) & ((status & (abi.TEB_STATUS_CAPACITY | abi.TEB_STATUS_BAD_INPUT)) == 0)
    ok &= (feas == 1) & (cmd[:, 3] != 0) & (result == abi.TEB_LOCAL_PLAN_PLANNED)
    vx, vy, om = cmd[:, 0].copy(), cmd[:, 1].copy(), cmd[:, 2].copy()
    with np.errstate(divide="ignore", invalid="ignore"):
        rx = np.where(vx > p.max_vel_x, p.max_vel_x / vx, 1.0)
        if p.max_vel_x_backwards > 0:
            rx = np.where(vx < -p.max_vel_x_backwards, -p.max_vel_x_backwards / vx, rx)
        ry = np.where(np.abs(vy) > p.max_vel_y, np.abs(p.max_vel_y / vy), 1.0)
        ro = np.where(np.abs(om) > p.max_vel_theta, np.abs(p.max_vel_theta / om), 1.0)
        vx, vy, om = vx * rx, vy * ry, om * ro
        lin = np.hypot(vx, vy)
        r = np.where(lin > p.max_vel_trans, p.max_vel_trans / lin, 1.0)
    cv = np.stack([vx * r, vy * r, om], 1)
    cv[~ok] = 0.0
    n = np.where(ok | (result != abi.TEB_LOCAL_PLAN_PLANNED), n, 0).astype(np.int32)
    n[result == abi.TEB_LOCAL_PLAN_GOAL_REACHED] = 0
    return cv, n


def loop_times(B, cycles, period, torch):
    dev = torch.device("cuda:0")
    G, P_cap, n_cap, L = 2000, 128, 128, 50
    d = scenes.global_plans(B, G, S=4, seed=7)
    S = d["grid"].shape[0]
    p = scenes.config_params("C2")
    abi.make_cycle_args(0.0, params=p)
    g = T.TebGpu(B, n_cap, S, 1, 0)
    g.set_params(p)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
    f64, i32 = torch.float64, torch.int32
    gp, begin, end = t(d["global_plan"]), t(d["plan_begin"]), t(d["plan_end"])
    robot0, vel = t(d["robot"]), t(d["robot_vel"])
    robot = robot0.clone()
    grid, origin, sid = t(d["grid"]), t(d["origin"]), t(d["scene_id"])
    plan, pcount, result = z((B, P_cap, 3), f64), z(B, i32), z(B, i32)
    state = {k: t(v) for k, v in abi.make_cycle_state(B, L).items()}
    since = z(B, f64)
    la = abi.make_local_plan_args(G, P_cap, 0, global_plan=gp.data_ptr(), plan_begin=begin.data_ptr(),
                                  plan_end=end.data_ptr(), robot=robot.data_ptr(), robot_vel=vel.data_ptr(),
                                  grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  infeasible_count=state["infeasible_count"].data_ptr(), since_infeasible=since.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), result=result.data_ptr())
    poses, n = z((B, n_cap, 4), f64), z(B, i32)
    obst, ocount = z((S, 64), torch.uint8), z(S, i32)
    vs = np.zeros((B, 4))
    vs[:, 3] = 1.0
    vstart, vgoal = t(vs), t(vs.copy())
    cost, chi2, status, iters = z(B, f64), z(B, f64), z(B, i32), z(B, i32)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, S, 1, 0, 0
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
    bs.vel_start, bs.vel_goal, bs.prefer_rotdir = vstart.data_ptr(), vgoal.data_ptr(), state["prefer_rotdir"].data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = cost.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True)
    cmd, feas, qc = z((B, 4), f64), z(B, i32), z(B, i32)
    cmd_vel, outcome = z((B, 3), f64), z(B, i32)
    fa = abi.make_feasibility_args(0.1, max_queries=512, feasible=feas.data_ptr(), query_count=qc.data_ptr())
    stream = torch.cuda.current_stream().cuda_stream
    clock = [100.0]

    def cycle(device_tail):
        now = clock[0]
        clock[0] += period
        since.copy_(now - state["last_infeasible"])
        ca = abi.make_cycle_args(now, buffer_length=L, local_plan_result=result.data_ptr(), robot_vel=vel.data_ptr(),
                                 cmd=cmd.data_ptr(), feasible=feas.data_ptr(), cmd_vel=cmd_vel.data_ptr(),
                                 outcome=outcome.data_ptr(), **{k: state[k].data_ptr() for k in abi.CYCLE_STATE})
        g.local_plan_device(bs, la, stream=stream)
        if device_tail:
            g.backup_modes_device(bs, ca, stream=stream)
        g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, stream=stream)
        g.check_feasible_device(bs, fa, stream=stream)
        if device_tail:
            g.finish_cycle_device(bs, ca, stream=stream)
        else:
            h = [x.cpu().numpy() for x in (status, chi2, cmd, feas, result, n)]
            cv, nn = host_tail(p, *h)
            cmd_vel.copy_(t(cv))
            n.copy_(t(nn))
        robot.copy_(move(robot, cmd_vel, period, torch))
        vel.copy_(cmd_vel)

    def block(K, device_tail):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(K):
            cycle(device_tail)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / K

    res = {}
    for name, dt in (("device_tail", True), ("host_tail", False)):
        robot.copy_(robot0)
        n.zero_()
        block(2, dt)
        res[name + "_ms_per_cycle"] = float(np.median([1e3 * block(cycles, dt) for _ in range(3)]))
    res["outcomes_last_cycle"] = np.bincount(outcome.cpu().numpy(), minlength=9).tolist()
    g.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--robots", type=int, nargs="+", default=[1024, 8192])
    ap.add_argument("--loop-robots", type=int, default=1024)
    ap.add_argument("--cycles", type=int, default=20)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--period", type=float, default=0.2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    res = dict(card=card(), alone={str(B): kernel_times(B, a.reps, torch) for B in a.robots},
               loop=dict(robots=a.loop_robots, cycles=a.cycles, **loop_times(a.loop_robots, a.cycles, a.period, torch)))
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
