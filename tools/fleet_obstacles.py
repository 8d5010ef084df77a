"""The other robots of a fleet as custom obstacle rows (tebgpu_fleet_obstacles_device) for R robots: the step alone,
the host route it replaces, and its share of a full cycle.

  step    k_fleet_obstacles (and k_fleet_claim with scenes given) over R robots spread over a square at a density of
          one robot per 4 m^2, range 3 m, CUDA events around each call, the median of --reps calls after 3 warm-up
          calls, at every --robots count and every --max-rows;
  host    the route a fleet has without the step: copy every pose and last_cmd to the host, find each robot's nearest
          max_rows neighbours with numpy (all pairs in blocks of 256 robots, argpartition, then the (d2, index) sort),
          build the rows and copy custom and custom_count back; host clock around the whole route, which ends in a
          synchronise. Only at --host-robots counts (all pairs in numpy take seconds past ~10^4 robots);
  loop    every cycle, on one stream: the fleet step, tebgpu_costmap_obstacles_device (the custom rows only),
          tebgpu_local_plan_device, tebgpu_backup_modes_device, tebgpu_plan_batch_device, tebgpu_check_feasible_device,
          tebgpu_finish_cycle_device and a torch op that moves every robot by cmd_vel; CUDA events around the fleet step
          and around the whole cycle, summed over --cycles cycles.

    python tools/fleet_obstacles.py --robots 1024 8192 32768 --max-rows 8 32 --host-robots 1024 8192 \\
        --loop-robots 1024 8192 [--json out.json]

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

RANGE = 3.0


def fleet(R, seed=1):
    """R robots on a square of 4 R m^2, headings and commands drawn at random"""
    rng = np.random.default_rng(seed)
    side = 2.0 * np.sqrt(R)
    pose = np.column_stack([rng.uniform(0, side, (R, 2)), rng.uniform(-np.pi, np.pi, R)])
    cmd = np.column_stack([rng.uniform(-0.2, 0.4, R), np.zeros(R), rng.uniform(-0.3, 0.3, R)])
    return pose, cmd, np.full(R, 0.3)


def host_rows(pose, cmd, radius, max_rows, C_cap):
    """the neighbour search and the rows on the host, vectorised: (custom [R][C_cap] OBST_DTYPE, custom_count [R])"""
    R = len(pose)
    out = np.zeros((R, C_cap), abi.OBST_DTYPE)
    cnt = np.zeros(R, np.int32)
    c, s = np.cos(pose[:, 2]), np.sin(pose[:, 2])
    vx, vy = c * cmd[:, 0] - s * cmd[:, 1], s * cmd[:, 0] + c * cmd[:, 1]
    moving = ~(np.sqrt(cmd[:, 0] * cmd[:, 0] + cmd[:, 1] * cmd[:, 1]) < 0.001)
    vx, vy = np.where(moving, vx, 0.0), np.where(moving, vy, 0.0)
    K = min(max_rows, C_cap, R - 1)
    for b0 in range(0, R, 256):
        rows = np.arange(b0, min(R, b0 + 256))
        dx = pose[None, :, 0] - pose[rows, None, 0]
        dy = pose[None, :, 1] - pose[rows, None, 1]
        d2 = dx * dx + dy * dy
        d2[np.arange(len(rows)), rows] = np.inf
        d2[~(d2 <= RANGE * RANGE)] = np.inf
        part = np.argpartition(d2, K - 1, axis=1)[:, :K] if K < R else np.argsort(d2, axis=1)
        key = d2[np.arange(len(rows))[:, None], part]
        order = np.lexsort((part, key), axis=1)
        q = np.take_along_axis(part, order, 1)
        ok = np.isfinite(np.take_along_axis(key, order, 1))
        cnt[rows] = ok.sum(1)
        o = out[rows, :K]
        o["x"], o["y"], o["vx"], o["vy"] = pose[q, 0], pose[q, 1], vx[q], vy[q]
        o["radius"], o["dynamic"], o["type"] = radius[q], moving[q], 1
        out[rows, :K] = np.where(ok, o, np.zeros((), abi.OBST_DTYPE))
    return out, cnt


def step_times(R, max_rows, reps, torch):
    dev = torch.device("cuda:0")
    g = T.TebGpu(R, 8, R, 64)
    pose, cmd, rad = fleet(R)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    tp, tc, tr = t(pose), t(cmd), t(rad)
    custom = torch.zeros(R * max_rows * 64, dtype=torch.uint8, device=dev)
    cc, need, st = (torch.zeros(R, dtype=torch.int32, device=dev) for _ in range(3))
    fa = abi.make_fleet_args(R, R, max_rows, max_rows, RANGE, pose=tp, last_cmd=tc, radius=tr, custom=custom,
                             custom_count=cc, needed=need, status=st)
    s = torch.cuda.Stream()                         # not the legacy default stream: its handle 0 means the context's
    stream = s.cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ms = []
    for r in range(reps + 3):
        ev[0].record(s)
        g.fleet_obstacles_device(fa, stream=stream)
        ev[1].record(s)
        torch.cuda.synchronize()
        if r >= 3:
            ms.append(ev[0].elapsed_time(ev[1]))
    res = dict(step_ms=float(np.median(ms)), grid=g.last_fleet_grid(), mean_needed=float(need.float().mean()),
               truncated=int((st == abi.TEB_FLEET_TRUNCATED).sum()))
    g.close()
    return res


def host_route(R, max_rows, reps, torch):
    """D2H of pose and last_cmd, the numpy search, H2D of the rows and counts"""
    dev = torch.device("cuda:0")
    pose, cmd, rad = fleet(R)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    tp, tc = t(pose), t(cmd)
    custom = torch.zeros(R * max_rows * 64, dtype=torch.uint8, device=dev)
    cc = torch.zeros(R, dtype=torch.int32, device=dev)
    ms = []
    for r in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        hp, hc = tp.cpu().numpy(), tc.cpu().numpy()
        rows, cnt = host_rows(hp, hc, rad, max_rows, max_rows)
        custom.copy_(torch.from_numpy(rows.view(np.uint8).reshape(-1)).to(dev, non_blocking=False))
        cc.copy_(torch.from_numpy(cnt).to(dev))
        torch.cuda.synchronize()
        if r >= 1:
            ms.append(1e3 * (time.perf_counter() - t0))
    return dict(host_route_ms=float(np.median(ms)))


def loop_share(B, cycles, max_rows, torch, period=0.2):
    """the fleet step's share of a full cycle on one stream (CUDA events)"""
    dev = torch.device("cuda:0")
    G, P_cap, n_cap, L = 2000, 128, 128, 50
    d = scenes.global_plans(B, G, S=4, seed=7)
    p = scenes.config_params("C2")
    p.include_dynamic_obstacles = 1
    abi.make_cycle_args(0.0, params=p)
    C_cap = max_rows
    g = T.TebGpu(B, n_cap, B, C_cap, 0)
    g.set_params(p)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
    f64, i32 = torch.float64, torch.int32
    gp, begin, end = t(d["global_plan"]), t(d["plan_begin"]), t(d["plan_end"])
    robot, vel = t(d["robot"]), t(d["robot_vel"])
    grid, origin = t(d["grid"][d["scene_id"]]), t(d["origin"][d["scene_id"]])
    sid = t(np.arange(B, dtype=np.int32))
    plan, pcount, result = z((B, P_cap, 3), f64), z(B, i32), z(B, i32)
    state = {k: t(v) for k, v in abi.make_cycle_state(B, L).items()}
    since = z(B, f64)
    la = abi.make_local_plan_args(G, P_cap, 0, global_plan=gp.data_ptr(), plan_begin=begin.data_ptr(),
                                  plan_end=end.data_ptr(), robot=robot.data_ptr(), robot_vel=vel.data_ptr(),
                                  grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  infeasible_count=state["infeasible_count"].data_ptr(), since_infeasible=since.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), result=result.data_ptr())
    poses, n = z((B, n_cap, 4), f64), z(B, i32)
    obst, ocount = z(B * C_cap * 64, torch.uint8), z(B, i32)
    custom, ccount = z(B * C_cap * 64, torch.uint8), z(B, i32)
    fneed, fstat = z(B, i32), z(B, i32)
    vs = np.zeros((B, 4))
    vs[:, 3] = 1.0
    vstart, vgoal = t(vs), t(vs.copy())
    cost, chi2, status, iters = z(B, f64), z(B, f64), z(B, i32), z(B, i32)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, B, C_cap, 0, 0
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
    bs.vel_start, bs.vel_goal, bs.prefer_rotdir = vstart.data_ptr(), vgoal.data_ptr(), state["prefer_rotdir"].data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = cost.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = B, 0, C_cap, C_cap, 0
    nogrid = z((B, 2), i32)                         # 0 x 0 rasters: the custom rows only
    ca.grid, ca.origin, ca.robot = nogrid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.custom, ca.custom_count = custom.data_ptr(), ccount.data_ptr()
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    fl = abi.make_fleet_args(B, B, C_cap, max_rows, RANGE, pose=robot, last_cmd=state["last_cmd"],
                             radius=t(np.full(B, 0.3)), custom=custom, custom_count=ccount, needed=fneed, status=fstat)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True)
    cmd, feas, qc = z((B, 4), f64), z(B, i32), z(B, i32)
    cmd_vel, outcome = z((B, 3), f64), z(B, i32)
    fa = abi.make_feasibility_args(0.1, max_queries=512, feasible=feas.data_ptr(), query_count=qc.data_ptr())
    s = torch.cuda.Stream()
    stream = s.cuda_stream
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(cycles + 2)]
    now = 100.0
    since.copy_(now - state["last_infeasible"])
    torch.cuda.synchronize()
    for k in range(cycles + 2):
        cy = abi.make_cycle_args(now, buffer_length=L, local_plan_result=result.data_ptr(), robot_vel=vel.data_ptr(),
                                 cmd=cmd.data_ptr(), feasible=feas.data_ptr(), cmd_vel=cmd_vel.data_ptr(),
                                 outcome=outcome.data_ptr(), **{kk: state[kk].data_ptr() for kk in abi.CYCLE_STATE})
        e = evs[k]
        e[0].record(s)
        g.fleet_obstacles_device(fl, stream=stream)
        e[1].record(s)
        g.costmap_obstacles_device(ca, stream=stream)
        g.local_plan_device(bs, la, stream=stream)
        g.backup_modes_device(bs, cy, stream=stream)
        g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, stream=stream)
        g.check_feasible_device(bs, fa, stream=stream)
        g.finish_cycle_device(bs, cy, stream=stream)
        with torch.cuda.stream(s):
            robot.copy_(move(robot, cmd_vel, period, torch))
            vel.copy_(cmd_vel)
            since.copy_(now + period - state["last_infeasible"])
        e[2].record(s)
        now += period
    torch.cuda.synchronize()
    step = sum(evs[k][0].elapsed_time(evs[k][1]) for k in range(2, cycles + 2))
    total = sum(evs[k][0].elapsed_time(evs[k][2]) for k in range(2, cycles + 2))
    res = dict(robots=B, cycles=cycles, step_ms_per_cycle=step / cycles, cycle_ms=total / cycles,
               step_share=step / total, mean_needed_last=float(fneed.float().mean()),
               dynamic_rows_last=int((custom.view(-1, 64)[:, 40:44].contiguous().view(torch.int32) == 1).sum()))
    g.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--robots", type=int, nargs="+", default=[1024, 8192, 32768])
    ap.add_argument("--max-rows", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--host-robots", type=int, nargs="+", default=[1024, 8192])
    ap.add_argument("--loop-robots", type=int, nargs="+", default=[1024, 8192])
    ap.add_argument("--cycles", type=int, default=10)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    res = dict(card=card(), range_m=RANGE, step={}, host={}, loop={})
    for R in a.robots:
        for m in a.max_rows:
            res["step"][f"{R}/{m}"] = step_times(R, m, a.reps, torch)
    for R in a.host_robots:
        for m in a.max_rows:
            res["host"][f"{R}/{m}"] = host_route(R, m, 3, torch)
    for R in a.loop_robots:
        res["loop"][str(R)] = loop_share(R, a.cycles, 8, torch)
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
