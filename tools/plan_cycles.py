"""Closed-loop planning cycles of N robots, one band each: the device-resident loop against the host-buffer loop.

Every cycle each robot plans from its current pose to its goal (TebOptimalPlanner::plan) and reads its velocity command
(getVelocityCommand); a torch op then moves every robot by its command for one control period. Two loops run in the
same process, alternated cycle block by cycle block:
  device  tebgpu_plan_batch_device on torch buffers: warm start, optimize and command stay on the GPU, one
          synchronisation at the end of the K cycles;
  host    the bands copied to the host every cycle, updateAndPruneTEB / initTrajectoryToGoal per band on the CPU (the
          drop-in layer's TimedElasticBand through teb_host_band_op), tebgpu_optimize_batch, getVelocityCommand.
It also reports k_plan_begin's and k_velocity_command's share of a device cycle (tebgpu_get_plan_kernel_times).

    python tools/plan_cycles.py --robots 1024 --cycles 20 [--config C2] [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query)."""
import argparse
import ctypes as C
import json
import math
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


def host_band_op():
    from teb_local_planner_b200 import build as b
    b.build_host()
    fn = C.CDLL(b.HOST_PIN).teb_host_band_op
    fn.restype = C.c_int32
    fn.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]
    out = np.empty(4 * 520)

    def run(op, rec, args):
        a = np.ascontiguousarray(args, dtype=np.float64)
        r = None if rec is None else np.ascontiguousarray(rec)
        k = fn(op, None if r is None else r.ctypes.data, 0 if r is None else len(r), a.ctypes.data, len(a), out.ctypes.data, out.size)
        return out[:k].reshape(-1, 4).copy()
    return run


def move(pose, cmd, period, torch):
    """one control period along the command (robot frame velocities)"""
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
    ap.add_argument("--cycles", type=int, default=20)
    ap.add_argument("--blocks", type=int, default=3, help="alternated blocks of --cycles cycles per loop")
    ap.add_argument("--config", default="C2")
    ap.add_argument("--period", type=float, default=0.2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda:0")
    p, hb0 = scenes.make_config_batch(a.config, requests=a.robots, candidates=1, autosize=True)
    B = hb0.B
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True)
    goal_np = np.stack([hb0.poses[b, hb0.n[b] - 1, :3] for b in range(B)])
    start_np = hb0.poses[:, 0, :3].copy()
    g = T.TebGpu(B, hb0.n_cap, hb0.S, max(hb0.M_cap, 1), hb0.V_cap, max_obst_vertices=hb0.PV_cap)
    g.set_params(p)
    # device-resident state
    fields = ("poses", "n", "scene_id", "obstacles", "obst_count", "obst_vertices", "via", "via_count", "vel_start",
              "vel_goal", "prefer_rotdir", "cost", "chi2", "status", "lm_iters")
    t = {k: torch.from_numpy(np.ascontiguousarray(getattr(hb0, k)).view(np.uint8).reshape(-1).copy()).to(dev) for k in fields}
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = B, hb0.n_cap, hb0.S, hb0.M_cap, hb0.V_cap, hb0.PV_cap
    for k, v in t.items():
        setattr(bs, k, v.data_ptr() if v.numel() else None)
    if hb0.V_cap == 0:
        bs.via = None
    start = torch.from_numpy(start_np).to(dev)
    goal = torch.from_numpy(goal_np).to(dev)
    cmd = torch.zeros((B, 4), dtype=torch.float64, device=dev)
    op = host_band_op()
    stream = torch.cuda.current_stream().cuda_stream

    def device_block(K):
        nonlocal start
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(K):
            g.plan_device(bs, args, cmd, start=start, goal=goal, look_ahead_poses=1, stream=stream)
            start.copy_(move(start, cmd, a.period, torch))   # ordered after the cycle: the same stream
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / K

    hb = hb0.copy()
    hstart = start_np.copy()

    def host_block(K):
        nonlocal hstart
        t0 = time.perf_counter()
        for _ in range(K):
            for b in range(B):
                n = hb.n[b]
                out = op(4, hb.poses[b, :n], list(hstart[b]) + list(goal_np[b]) + [p.min_samples])
                hb.poses[b, :len(out)], hb.n[b] = out, len(out)
            g.optimize(hb, args)
            c = np.zeros((B, 4))
            for b in range(B):
                r = op(8, hb.poses[b, :hb.n[b]], [1, p.max_vel_y]).reshape(-1)
                c[b] = [r[1], r[2], r[3], r[0]]
            hstart = move(torch.from_numpy(hstart), torch.from_numpy(c), a.period, torch).numpy()
        return (time.perf_counter() - t0) / K

    device_block(2)   # warm-up: capture / first launches
    host_block(1)
    dev_ms, host_ms = [], []
    for _ in range(a.blocks):
        dev_ms.append(1e3 * device_block(a.cycles))
        host_ms.append(1e3 * host_block(a.cycles))
    g.set_profiling(1)
    g.plan_device(bs, args, cmd, start=start, goal=goal, look_ahead_poses=1, stream=stream)
    torch.cuda.synchronize()
    plan_k = g.plan_kernel_times()
    opt_k = g.kernel_times()
    g.set_profiling(0)
    total = sum(v[0] for v in opt_k.values()) + sum(v[0] for v in plan_k.values())
    res = dict(card=card(), config=a.config, robots=B, cycles=a.cycles, blocks=a.blocks,
               device_ms_per_cycle=float(np.median(dev_ms)), host_ms_per_cycle=float(np.median(host_ms)),
               speedup=float(np.median(host_ms) / np.median(dev_ms)),
               k_plan_begin_ms=plan_k["k_plan_begin"][0], k_velocity_command_ms=plan_k["k_velocity_command"][0],
               kernels_ms_one_cycle=total,
               new_kernels_share=(plan_k["k_plan_begin"][0] + plan_k["k_velocity_command"][0]) / total if total else math.nan)
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    g.close()


if __name__ == "__main__":
    main()
