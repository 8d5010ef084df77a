"""The local-plan step (tebgpu_local_plan_device) for N robots following global plans, alone and inside a closed loop.

  alone   k_local_plan over N robots with G-row global plans (scenes.global_plans), CUDA events around each launch;
  loop    every cycle, on one stream: tebgpu_local_plan_device cuts each robot's plan at its current pose,
          tebgpu_plan_batch_device plans from those rows (warm start after the first cycle) and gives the command, and a
          torch op moves every robot by its command for one control period and feeds the command back as its odometry.
          One synchronisation per K cycles; nothing goes through the host. The step's share of a cycle is the alone time
          over the loop's time per cycle.

    python tools/local_plan.py --robots 1024 --rows 2000 --cycles 20 [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi, scenes  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=20).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:
        return "unknown"


def move(pose, cmd, period, torch):
    th = pose[:, 2]
    vx, vy, om = cmd[:, 0], cmd[:, 1], cmd[:, 2]
    nxt = pose.clone()
    nxt[:, 0] += (vx * torch.cos(th) - vy * torch.sin(th)) * period
    nxt[:, 1] += (vx * torch.sin(th) + vy * torch.cos(th)) * period
    nxt[:, 2] = torch.atan2(torch.sin(th + om * period), torch.cos(th + om * period))
    return nxt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--robots", type=int, default=1024)
    ap.add_argument("--rows", type=int, default=2000)
    ap.add_argument("--cycles", type=int, default=20)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--config", default="C2")
    ap.add_argument("--period", type=float, default=0.2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda:0")
    B, G, P_cap, V_cap, n_cap = a.robots, a.rows, 128, 32, 128
    d = scenes.global_plans(B, G, S=4, seed=7)
    S = d["grid"].shape[0]
    p = scenes.config_params(a.config)
    g = T.TebGpu(B, n_cap, S, 1, V_cap)
    g.set_params(p)
    t = lambda x, dt=None: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    gp, begin, end = t(d["global_plan"]), t(d["plan_begin"]), t(d["plan_end"])
    robot, vel = t(d["robot"]), t(d["robot_vel"])
    grid, origin, sid = t(d["grid"]), t(d["origin"]), t(d["scene_id"])
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
    plan, pcount, result = z((B, P_cap, 3), torch.float64), z((B,), torch.int32), z((B,), torch.int32)
    via, vcount = z((B, V_cap, 2), torch.float64), z((B,), torch.int32)
    la = abi.make_local_plan_args(G, P_cap, V_cap, viapoint_sep=0.5, global_plan=gp.data_ptr(),
                                  plan_begin=begin.data_ptr(), plan_end=end.data_ptr(), robot=robot.data_ptr(),
                                  robot_vel=vel.data_ptr(), grid=grid.data_ptr(), origin=origin.data_ptr(),
                                  plan=plan.data_ptr(), plan_count=pcount.data_ptr(), via=via.data_ptr(),
                                  via_count=vcount.data_ptr(), result=result.data_ptr())
    # the plan batch: no obstacles, the local plan's via-points
    poses, n = z((B, n_cap, 4), torch.float64), z((B,), torch.int32)
    obst, ocount = z((S, 64), torch.uint8), z((S,), torch.int32)
    vs = np.zeros((B, 4))
    vs[:, 3] = 1.0
    vstart, vgoal = t(vs), t(vs.copy())
    cost, chi2, status, iters = z((B,), torch.float64), z((B,), torch.float64), z((B,), torch.int32), z((B,), torch.int32)
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, n_cap, S, 1, V_cap, 0
    bs.poses, bs.n, bs.scene_id = poses.data_ptr(), n.data_ptr(), sid.data_ptr()
    bs.obstacles, bs.obst_count, bs.via, bs.via_count = obst.data_ptr(), ocount.data_ptr(), via.data_ptr(), vcount.data_ptr()
    bs.vel_start, bs.vel_goal = vstart.data_ptr(), vgoal.data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = cost.data_ptr(), chi2.data_ptr(), status.data_ptr(), iters.data_ptr()
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True)
    cmd = z((B, 4), torch.float64)
    stream = torch.cuda.current_stream().cuda_stream

    # alone: the same robots every launch (plan_begin restored, so every launch prunes the same rows)
    begin0 = begin.clone()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    alone = []
    for r in range(a.reps + 3):
        begin.copy_(begin0)
        ev[0].record()
        g.local_plan_device(bs, la, stream=stream)
        ev[1].record()
        torch.cuda.synchronize()
        if r >= 3:
            alone.append(ev[0].elapsed_time(ev[1]))
    codes = np.bincount(result.cpu().numpy(), minlength=5).tolist()
    live = (end - begin).cpu().numpy()

    def block(K):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(K):
            g.local_plan_device(bs, la, stream=stream)
            g.plan_device(bs, args, cmd, initial_plan=plan, plan_count=pcount, P_cap=P_cap, stream=stream)
            robot.copy_(move(robot, cmd, a.period, torch))
            vel.copy_(cmd[:, :3])
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / K

    block(2)
    loop_ms = [1e3 * block(a.cycles) for _ in range(3)]
    moved = np.median((begin - begin0).cpu().numpy())
    res = dict(card=card(), config=a.config, robots=B, rows=G, live_rows_mean=float(live.mean()),
               local_plan_ms=float(np.median(alone)), local_plan_results=codes, cycles=a.cycles,
               loop_ms_per_cycle=float(np.median(loop_ms)),
               local_plan_share=float(np.median(alone) / np.median(loop_ms)), grid_ctas=g.last_local_plan_grid(),
               median_rows_pruned=float(moved))
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
