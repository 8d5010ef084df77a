"""The fleet table (tebgpu_fleet_publish_device + tebgpu_fleet_obstacles_table_device): what one rank of a sharded fleet
pays per cycle, and the table step's share of a cycle of a fleet of two robot kinds in two contexts.

  rank    R_local robots of a fleet of T robots spread over a square at one robot per 4 m^2 (range 3 m, max_rows 8):
          the table holds all T rows (published beforehand in chunks of R_local rows); timed is the rank's publish of its
          R_local rows plus its table step over all T rows, CUDA events around each pair of calls, the median of --reps
          after 3 warm-up calls, at every --pairs (R_local, T). Beside it tebgpu_fleet_obstacles_device over R_local
          robots (T = R_local), the single-context step;
  mixed   two contexts (C2 circular robots and C3 car-like TwoCircles robots, half the fleet each) on one stream: both
          publish, both run the table step, then each runs tebgpu_costmap_obstacles_device (custom rows only),
          tebgpu_local_plan_device, tebgpu_backup_modes_device, tebgpu_plan_batch_device, tebgpu_check_feasible_device
          and tebgpu_finish_cycle_device, and a torch op moves every robot by cmd_vel; CUDA events around the fleet
          steps and around the whole cycle, summed over --cycles cycles.

The cross-GPU gather (one ncclAllGather of 64 T bytes) needs two GPUs and is not timed here.

    python tools/fleet_table.py --pairs 8192:8192 8192:32768 8192:65536 32768:262144 --mixed 1024 8192 [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query)."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi, scenes  # noqa: E402
from tools.fleet_obstacles import RANGE, fleet  # noqa: E402
from tools.local_plan import card, move  # noqa: E402

MAX_ROWS = 8


def rank_times(R, Tn, reps, torch):
    dev = torch.device("cuda:0")
    g = T.TebGpu(R, 8, R, 64)
    pose, cmd, rad = fleet(Tn)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    tp, tc, tr = t(pose), t(cmd), t(rad)
    rows = torch.zeros(Tn * abi.FLEET_ROW_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    custom = torch.zeros(R * MAX_ROWS * 64, dtype=torch.uint8, device=dev)
    cc, need, st = (torch.zeros(R, dtype=torch.int32, device=dev) for _ in range(3))
    s = torch.cuda.Stream()
    stream = s.cuda_stream
    for lo in range(0, Tn, R):                      # the other ranks' rows, as the gather would leave them
        hi = min(Tn, lo + R)
        fp = abi.make_fleet_args(hi - lo, 1, 0, 0, 0.0, pose=tp[lo:hi], last_cmd=tc[lo:hi], radius=tr[lo:hi])
        g.fleet_publish_device(fp, abi.make_fleet_table(Tn, lo, rows), stream=stream)
    mine = slice(Tn - R, Tn)                        # this rank's robots: the last R rows
    fa = abi.make_fleet_args(R, R, MAX_ROWS, MAX_ROWS, RANGE, pose=tp[mine], last_cmd=tc[mine], radius=tr[mine],
                             custom=custom, custom_count=cc, needed=need, status=st)
    tb = abi.make_fleet_table(Tn, Tn - R, rows)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ms, arr = [], []
    for r in range(reps + 3):
        ev[0].record(s)
        g.fleet_publish_device(fa, tb, stream=stream)
        g.fleet_obstacles_table_device(fa, tb, stream=stream)
        ev[1].record(s)
        g.fleet_obstacles_device(fa, stream=stream)
        ev[2].record(s)
        torch.cuda.synchronize()
        if r >= 3:
            ms.append(ev[0].elapsed_time(ev[1]))
            arr.append(ev[1].elapsed_time(ev[2]))
    g.fleet_publish_device(fa, tb, stream=stream)
    g.fleet_obstacles_table_device(fa, tb, stream=stream)
    torch.cuda.synchronize()
    res = dict(publish_plus_table_ms=float(np.median(ms)), array_step_at_T_eq_R_ms=float(np.median(arr)),
               grid=g.last_fleet_grid(), mean_needed=float(need.float().mean()),
               truncated=int((st == abi.TEB_FLEET_TRUNCATED).sum()))
    g.close()
    return res


def _kind(k, B, dev, torch, G, P_cap, n_cap, L, C_cap, d, lo, hi, robot, vel, radius_all, custom, ccount, rows, Tn,
          first):
    """one robot kind's context and the arrays of its cycle (robots lo .. hi - 1 of the fleet arrays)"""
    p = scenes.config_params("C2" if k == 0 else "C3")
    if k == 1:
        p.footprint_type = abi.TEB_FOOTPRINT_TWO_CIRCLES
        p.footprint_front_offset, p.footprint_front_radius = 0.2, 0.2
        p.footprint_rear_offset, p.footprint_rear_radius = 0.2, 0.2
    p.include_dynamic_obstacles = 1
    n = hi - lo
    g = T.TebGpu(n, n_cap, n, C_cap, 0)
    g.set_params(p)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
    f64, i32 = torch.float64, torch.int32
    sl = slice(lo, hi)
    gp, begin, end = t(d["global_plan"][sl]), t(d["plan_begin"][sl]), t(d["plan_end"][sl])
    grid, origin = t(d["grid"][d["scene_id"]][sl]), t(d["origin"][d["scene_id"]][sl])
    K = dict(g=g, p=p, sl=sl, state={kk: t(v) for kk, v in abi.make_cycle_state(n, L).items()}, since=z(n, f64),
             plan=z((n, P_cap, 3), f64), pcount=z(n, i32), result=z(n, i32), poses=z((n, n_cap, 4), f64), n=z(n, i32),
             sid=t(np.arange(n, dtype=np.int32)), obst=z(n * C_cap * 64, torch.uint8), ocount=z(n, i32),
             cost=z(n, f64), chi2=z(n, f64), status=z(n, i32), iters=z(n, i32), cmd=z((n, 4), f64), feas=z(n, i32),
             qc=z(n, i32), outcome=z(n, i32), fneed=z(n, i32), fstat=z(n, i32), nogrid=z((n, 2), i32), gp=gp,
             begin=begin, end=end, grid=grid, origin=origin)
    vs = np.zeros((n, 4))
    vs[:, 3] = 1.0
    K["vstart"], K["vgoal"] = t(vs), t(vs.copy())
    st = K["state"]
    K["la"] = abi.make_local_plan_args(G, P_cap, 0, global_plan=gp.data_ptr(), plan_begin=begin.data_ptr(),
                                       plan_end=end.data_ptr(), robot=robot[sl].data_ptr(), robot_vel=vel[sl].data_ptr(),
                                       grid=grid.data_ptr(), origin=origin.data_ptr(),
                                       infeasible_count=st["infeasible_count"].data_ptr(),
                                       since_infeasible=K["since"].data_ptr(), plan=K["plan"].data_ptr(),
                                       plan_count=K["pcount"].data_ptr(), result=K["result"].data_ptr())
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = n, n_cap, n, C_cap, 0, 0
    bs.poses, bs.n, bs.scene_id = K["poses"].data_ptr(), K["n"].data_ptr(), K["sid"].data_ptr()
    bs.obstacles, bs.obst_count = K["obst"].data_ptr(), K["ocount"].data_ptr()
    bs.vel_start, bs.vel_goal, bs.prefer_rotdir = K["vstart"].data_ptr(), K["vgoal"].data_ptr(), st["prefer_rotdir"].data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = (K["cost"].data_ptr(), K["chi2"].data_ptr(), K["status"].data_ptr(),
                                                 K["iters"].data_ptr())
    K["bs"] = bs
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = n, 0, C_cap, C_cap, 0
    ca.grid, ca.origin, ca.robot = K["nogrid"].data_ptr(), origin.data_ptr(), robot[sl].data_ptr()
    ca.custom, ca.custom_count = custom[sl].data_ptr(), ccount[sl].data_ptr()
    ca.obstacles, ca.obst_count = K["obst"].data_ptr(), K["ocount"].data_ptr()
    K["ca"] = ca
    K["fl"] = abi.make_fleet_args(n, n, C_cap, MAX_ROWS, RANGE, pose=robot[sl], last_cmd=st["last_cmd"],
                                  radius=radius_all[sl], custom=custom[sl], custom_count=ccount[sl], needed=K["fneed"],
                                  status=K["fstat"])
    K["tb"] = abi.make_fleet_table(Tn, first, rows)
    K["args"] = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True)
    K["fa"] = abi.make_feasibility_args(0.1, max_queries=512, feasible=K["feas"].data_ptr(), query_count=K["qc"].data_ptr())
    return K


def mixed_share(B, cycles, torch, period=0.2):
    """the table steps' share of a cycle of a two-kind fleet on one stream (CUDA events)"""
    dev = torch.device("cuda:0")
    G, P_cap, n_cap, L = 2000, 128, 128, 50
    C_cap = MAX_ROWS
    d = scenes.global_plans(B, G, S=4, seed=7)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
    f64, i32 = torch.float64, torch.int32
    robot, vel = t(d["robot"]), t(d["robot_vel"])
    radius = t(np.where(np.arange(B) < B // 2, 0.25, 0.4))
    custom, ccount = z((B, C_cap * 64), torch.uint8), z(B, i32)
    cmd_vel = z((B, 3), f64)
    rows = z(B * abi.FLEET_ROW_DTYPE.itemsize, torch.uint8)
    kinds = [_kind(k, B, dev, torch, G, P_cap, n_cap, L, C_cap, d, lo, hi, robot, vel, radius, custom, ccount, rows, B, lo)
             for k, (lo, hi) in enumerate(((0, B // 2), (B // 2, B)))]
    s = torch.cuda.Stream()
    stream = s.cuda_stream
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(cycles + 2)]
    now = 100.0
    for K in kinds:
        K["since"].copy_(now - K["state"]["last_infeasible"])
    torch.cuda.synchronize()
    for c in range(cycles + 2):
        e = evs[c]
        e[0].record(s)
        for K in kinds:
            K["g"].fleet_publish_device(K["fl"], K["tb"], stream=stream)
        for K in kinds:
            K["g"].fleet_obstacles_table_device(K["fl"], K["tb"], stream=stream)
        e[1].record(s)
        for K in kinds:
            g, st, sl = K["g"], K["state"], K["sl"]
            cy = abi.make_cycle_args(now, buffer_length=L, local_plan_result=K["result"].data_ptr(),
                                     robot_vel=vel[sl].data_ptr(), cmd=K["cmd"].data_ptr(), feasible=K["feas"].data_ptr(),
                                     cmd_vel=cmd_vel[sl].data_ptr(), outcome=K["outcome"].data_ptr(),
                                     **{kk: st[kk].data_ptr() for kk in abi.CYCLE_STATE})
            g.costmap_obstacles_device(K["ca"], stream=stream)
            g.local_plan_device(K["bs"], K["la"], stream=stream)
            g.backup_modes_device(K["bs"], cy, stream=stream)
            g.plan_device(K["bs"], K["args"], K["cmd"], initial_plan=K["plan"], plan_count=K["pcount"], P_cap=P_cap,
                          stream=stream)
            g.check_feasible_device(K["bs"], K["fa"], stream=stream)
            g.finish_cycle_device(K["bs"], cy, stream=stream)
        with torch.cuda.stream(s):
            robot.copy_(move(robot, cmd_vel, period, torch))
            vel.copy_(cmd_vel)
            for K in kinds:
                K["since"].copy_(now + period - K["state"]["last_infeasible"])
        e[2].record(s)
        now += period
    torch.cuda.synchronize()
    step = sum(evs[k][0].elapsed_time(evs[k][1]) for k in range(2, cycles + 2))
    total = sum(evs[k][0].elapsed_time(evs[k][2]) for k in range(2, cycles + 2))
    rowsv = custom.view(-1, 64)
    other = 0
    for k, K in enumerate(kinds):             # neighbour rows of the other kind (its radius) in this kind's scenes
        r = rowsv.view(B, C_cap, 64)[K["sl"]].reshape(-1, 64)[:, 32:40].contiguous().view(torch.float64).view(-1)
        other += int((r == (0.4 if k == 0 else 0.25)).sum())
    res = dict(robots=B, cycles=cycles, table_steps_ms_per_cycle=step / cycles, cycle_ms=total / cycles,
               table_share=step / total, other_kind_rows_last=other)
    for K in kinds:
        K["g"].close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", nargs="+", default=["8192:8192", "8192:32768", "8192:65536", "32768:262144"])
    ap.add_argument("--mixed", type=int, nargs="+", default=[1024, 8192])
    ap.add_argument("--cycles", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    res = dict(card=card(), range_m=RANGE, max_rows=MAX_ROWS, rank={}, mixed={}, gather="not measured (one GPU)")
    for pr in a.pairs:
        R, Tn = (int(v) for v in pr.split(":"))
        res["rank"][pr] = rank_times(R, Tn, a.reps, torch)
    for B in a.mixed:
        res["mixed"][str(B)] = mixed_share(B, a.cycles, torch)
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
