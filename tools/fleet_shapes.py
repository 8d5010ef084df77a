"""Footprint rows against circle rows (tebgpu_fleet_obstacles_shaped_device against tebgpu_fleet_obstacles_device), on
the same fleets.

  step    R robots on a square at one robot per 4 m^2 (tools/fleet_obstacles.fleet, range 3 m, max_rows 8), half of them
          C3 car-like robots published as their TwoCircles footprint, half as a 0.5 x 0.3 m rectangle; the circle step
          publishes every robot as one circle. Both searches (all pairs, grid) at every --step R; the two steps
          alternate, CUDA events around each call, the median of --reps after 3 warm-up calls.
  cycle   R C3 robots in one context on one stream: the fleet step, tebgpu_costmap_obstacles_tf_device (custom rows only,
          identity frames), tebgpu_local_plan_device, tebgpu_backup_modes_device, tebgpu_plan_batch_device,
          tebgpu_check_feasible_device, tebgpu_finish_cycle_device, a torch op moving every robot. Three fleets: circle
          rows; TwoCircles rows (circles only); rectangle rows (Polygon rows with their vertices, so the plan runs its
          vertex-list instantiations). CUDA events around each whole cycle, summed over --cycles after 2 warm-up cycles.

    python tools/fleet_shapes.py --step 1024 8192 32768 --cycle 1024 8192 [--json out.json]

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
RECT = [(abi.TEB_OBST_POLYGON, [[0.25, 0.15], [-0.25, 0.15], [-0.25, -0.15], [0.25, -0.15]])]


def c3_params():
    p = scenes.config_params("C3")
    p.footprint_type = abi.TEB_FOOTPRINT_TWO_CIRCLES
    p.footprint_front_offset, p.footprint_front_radius = 0.2, 0.2
    p.footprint_rear_offset, p.footprint_rear_radius = 0.2, 0.2
    p.include_dynamic_obstacles = 1
    return p


def step_times(R, reps, torch):
    dev = torch.device("cuda:0")
    g = T.TebGpu(R, 8, R, 64)
    pose, cmd, rad = fleet(R)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    kinds = [abi.fleet_shape_from_params(c3_params()), RECT]
    kind = t((np.arange(R) % 2).astype(np.int32))
    C_cap, PV = 2 * MAX_ROWS, 4 * MAX_ROWS
    custom = torch.zeros(R * C_cap * 64, dtype=torch.uint8, device=dev)
    cv = torch.zeros((R, PV, 2), dtype=torch.float64, device=dev)
    cc, need, st = (torch.zeros(R, dtype=torch.int32, device=dev) for _ in range(3))
    tp, tc, tr = t(pose), t(cmd), t(rad)          # held: the args keep only their addresses
    fa = abi.make_fleet_args(R, R, C_cap, MAX_ROWS, RANGE, pose=tp, last_cmd=tc, radius=tr, custom=custom,
                             custom_count=cc, needed=need, status=st)
    sh = abi.make_fleet_shapes(kinds, PV, kind=kind, custom_vertices=cv)
    s = torch.cuda.Stream()
    res = {}
    for mode, name in ((abi.TEBGPU_FLEET_SEARCH_ALL_PAIRS, "all_pairs"), (abi.TEBGPU_FLEET_SEARCH_GRID, "grid")):
        g.set_fleet_search(mode)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        circ, shp = [], []
        for r in range(reps + 3):
            ev[0].record(s)
            g.fleet_obstacles_device(fa, stream=s.cuda_stream)
            ev[1].record(s)
            g.fleet_obstacles_shaped_device(fa, sh, stream=s.cuda_stream)
            ev[2].record(s)
            torch.cuda.synchronize()
            if r >= 3:
                circ.append(ev[0].elapsed_time(ev[1]))
                shp.append(ev[1].elapsed_time(ev[2]))
        res[name] = dict(circle_ms=float(np.median(circ)), shaped_ms=float(np.median(shp)),
                         rows_per_robot=float(cc.float().mean()), truncated=int((st == abi.TEB_FLEET_TRUNCATED).sum()))
    g.close()
    return res


def cycle_time(B, cycles, rows, torch, period=0.2):
    """rows: "circle", "two_circles" or "rectangle"; ms per cycle and the rows per scene of the last cycle"""
    dev = torch.device("cuda:0")
    G, P_cap, n_cap, L = 2000, 128, 128, 50
    C_cap = MAX_ROWS if rows == "circle" else 2 * MAX_ROWS
    PV = 4 * MAX_ROWS if rows == "rectangle" else 0
    M_cap = C_cap
    d = scenes.global_plans(B, G, S=4, seed=7)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
    f64, i32 = torch.float64, torch.int32
    p = c3_params()
    g = T.TebGpu(B, n_cap, B, M_cap, 0, max_obst_vertices=PV)
    g.set_params(p)
    robot, vel = t(d["robot"]), t(d["robot_vel"])
    gp, begin, end = t(d["global_plan"]), t(d["plan_begin"]), t(d["plan_end"])
    grid, origin = t(d["grid"][d["scene_id"]]), t(d["origin"][d["scene_id"]])
    state = {k: t(v) for k, v in abi.make_cycle_state(B, L).items()}
    since, plan, pcount, result = z(B, f64), z((B, P_cap, 3), f64), z(B, i32), z(B, i32)
    poses, nn, sid = z((B, n_cap, 4), f64), z(B, i32), t(np.arange(B, dtype=np.int32))
    obst, ocount, ov = z(B * M_cap * 64, torch.uint8), z(B, i32), z((B, max(PV, 1), 2), f64)
    cost, chi2, status, iters, cmd = z(B, f64), z(B, f64), z(B, i32), z(B, i32), z((B, 4), f64)
    feas, qc, outcome, nogrid, cmd_vel = z(B, i32), z(B, i32), z(B, i32), z((B, 2), i32), z((B, 3), f64)
    custom, ccount, fneed, fstat, cv = z(B * C_cap * 64, torch.uint8), z(B, i32), z(B, i32), z(B, i32), z((B, max(PV, 1), 2), f64)
    vs = np.zeros((B, 4))
    vs[:, 3] = 1.0
    vstart, vgoal = t(vs), t(vs.copy())
    la = abi.make_local_plan_args(G, P_cap, 0, global_plan=gp.data_ptr(), plan_begin=begin.data_ptr(),
                                  plan_end=end.data_ptr(), robot=robot.data_ptr(), robot_vel=vel.data_ptr(),
                                  grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  infeasible_count=state["infeasible_count"].data_ptr(), since_infeasible=since.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), result=result.data_ptr())
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, B, M_cap, 0, PV
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), nn.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count, bs.obst_vertices = obst.data_ptr(), ocount.data_ptr(), ov.data_ptr() if PV else None
    bs.vel_start, bs.vel_goal, bs.prefer_rotdir = vstart.data_ptr(), vgoal.data_ptr(), state["prefer_rotdir"].data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = cost.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = B, 0, M_cap, C_cap, 0
    ca.grid, ca.origin, ca.robot = nogrid.data_ptr(), origin.data_ptr(), robot.data_ptr()
    ca.custom, ca.custom_count = custom.data_ptr(), ccount.data_ptr()
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    ident = t(np.tile([0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0], (B, 1)))
    frames = abi.make_frame_args(custom_to_costmap=ident.data_ptr(), custom_vertices=cv.data_ptr() if PV else None,
                                 obst_vertices=ov.data_ptr() if PV else None, PV_cap=PV)
    radius, kind = t(np.full(B, 0.4)), z(B, i32)   # held: the args keep only their addresses
    fl = abi.make_fleet_args(B, B, C_cap, MAX_ROWS, RANGE, pose=robot, last_cmd=state["last_cmd"], radius=radius,
                             custom=custom, custom_count=ccount, needed=fneed, status=fstat)
    kinds = [abi.fleet_shape_from_params(p) if rows == "two_circles" else RECT]
    sh = abi.make_fleet_shapes(kinds, PV, kind=kind, custom_vertices=cv if PV else None)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True)
    fa = abi.make_feasibility_args(0.1, max_queries=512, feasible=feas.data_ptr(), query_count=qc.data_ptr())
    s = torch.cuda.Stream()
    stream = s.cuda_stream
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(2)] for _ in range(cycles + 2)]
    now = 100.0
    since.copy_(now - state["last_infeasible"])
    torch.cuda.synchronize()
    for c in range(cycles + 2):
        evs[c][0].record(s)
        if rows == "circle":
            g.fleet_obstacles_device(fl, stream=stream)
        else:
            g.fleet_obstacles_shaped_device(fl, sh, stream=stream)
        cy = abi.make_cycle_args(now, buffer_length=L, local_plan_result=result.data_ptr(), robot_vel=vel.data_ptr(),
                                 cmd=cmd.data_ptr(), feasible=feas.data_ptr(), cmd_vel=cmd_vel.data_ptr(),
                                 outcome=outcome.data_ptr(), **{k: state[k].data_ptr() for k in abi.CYCLE_STATE})
        g.costmap_obstacles_device(ca, stream=stream, frames=frames)
        g.local_plan_device(bs, la, stream=stream)
        g.backup_modes_device(bs, cy, stream=stream)
        g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, stream=stream)
        g.check_feasible_device(bs, fa, stream=stream)
        g.finish_cycle_device(bs, cy, stream=stream)
        with torch.cuda.stream(s):
            robot.copy_(move(robot, cmd_vel, period, torch))
            vel.copy_(cmd_vel)
            since.copy_(now + period - state["last_infeasible"])
        evs[c][1].record(s)
        now += period
    torch.cuda.synchronize()
    total = sum(evs[k][0].elapsed_time(evs[k][1]) for k in range(2, cycles + 2))
    res = dict(cycle_ms=total / cycles, rows_per_scene=float(ocount.float().mean()),
               commands=int((outcome == abi.TEB_CYCLE_COMMAND).sum()))
    g.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--step", type=int, nargs="+", default=[1024, 8192, 32768])
    ap.add_argument("--cycle", type=int, nargs="+", default=[1024, 8192])
    ap.add_argument("--cycles", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    res = dict(card=card(), range_m=RANGE, max_rows=MAX_ROWS, step={}, cycle={})
    for R in a.step:
        res["step"][str(R)] = step_times(R, a.reps, torch)
    for B in a.cycle:
        # the three fleets alternate over two rounds, so drift of the card shows as a spread between rounds
        out = {k: [] for k in ("circle", "two_circles", "rectangle")}
        for _ in range(2):
            for k in out:
                out[k].append(cycle_time(B, a.cycles, k, torch))
        res["cycle"][str(B)] = out
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
