"""Time of the trajectory read-out (tebgpu_read_trajectory_device: getVelocityProfile + getFullTrajectory) after a
plan cycle, CUDA events around the calls, against the device-to-host copy of the batch's records it replaces.

  C3 at --bands bands (default 8192: 128 requests of 64 candidates), one tebgpu_plan_batch_device cycle first;
  the read-out of every band, and of one winner per request (tebgpu_select_best over each request's costs);
  the winners' read-out followed by the copy of its rows to pinned host memory;
  the copy of the batch's poses, n, vel_start and vel_goal to pinned host memory (what a host-side read-out needs).

    python tools/trajectory_readout.py [--bands 8192] [--reps 50] [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query), then one JSON line."""
import argparse
import json
import os
import subprocess
import sys

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


DEV_FIELDS = ("poses", "n", "scene_id", "obstacles", "obst_count", "obst_vertices", "via", "via_count", "vel_start",
              "vel_goal", "prefer_rotdir", "cost", "chi2", "status", "lm_iters")


def device_batch(hb, torch):
    dev = torch.device("cuda:0")
    t = {k: torch.from_numpy(np.ascontiguousarray(getattr(hb, k)).view(np.uint8).reshape(-1).copy()).to(dev) for k in DEV_FIELDS}
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap, bs.PV_cap = hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap, hb.PV_cap
    for k, v in t.items():
        setattr(bs, k, v.data_ptr() if v.numel() else None)
    if hb.V_cap == 0:
        bs.via = None
    return t, bs


def time_ms(fn, reps, torch):
    for _ in range(3):                                  # warm-up: module load, first launches
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bands", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement runs on the GPU only")
    # a stream of its own: the calls and the timing events share it (handle 0 would mean the context's own stream)
    with torch.cuda.stream(torch.cuda.Stream()):
        run(a, torch)


def run(a, torch):
    res = dict(card=card())
    print("card, power limit:", res["card"])
    requests = 128 if a.bands % 128 == 0 else 1
    cand = a.bands // requests
    p, hb = scenes.make_config_batch("C3", requests=requests, candidates=cand, seed=1)
    B, nc = hb.B, hb.n_cap
    g = T.TebGpu(B, nc, hb.S, hb.M_cap, hb.V_cap)
    g.set_params(p)
    t, bs = device_batch(hb, torch)
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    start = torch.from_numpy(np.ascontiguousarray(hb.poses[:, 0, :3])).to(dev)
    goal = torch.from_numpy(np.ascontiguousarray(hb.poses[np.arange(B), hb.n - 1, :3])).to(dev)
    cmd = torch.zeros((B, 4), dtype=torch.float64, device=dev)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    g.plan_device(bs, args, cmd, start=start, goal=goal, stream=stream)
    torch.cuda.synchronize()
    n = t["n"].view(torch.int32).cpu().numpy()
    cost = t["cost"].view(torch.float64).cpu().numpy()
    winners = np.array([r * cand + g.lib.tebgpu_select_best(np.ascontiguousarray(cost[r * cand:(r + 1) * cand]).ctypes.data,
                                                            cand, -1, -1, 1.0, 1.0) for r in range(requests)], np.int32)
    res["c3"] = dict(bands=B, requests=requests, n_cap=nc, mean_n=round(float(n.mean()), 1))

    def outputs(R):
        return (torch.empty((R, nc + 1, 3), dtype=torch.float64, device=dev), torch.empty((R, nc, 7), dtype=torch.float64, device=dev),
                torch.empty(R, dtype=torch.int32, device=dev))
    prof, traj, pts = outputs(B)
    ms_all = time_ms(lambda: g.read_trajectory_device(bs, trajectory=traj, profile=prof, points=pts, stream=stream), a.reps, torch)
    grid_all = g.info(14)
    wb = torch.from_numpy(winners).to(dev)
    wprof, wtraj, wpts = outputs(requests)
    ms_win = time_ms(lambda: g.read_trajectory_device(bs, trajectory=wtraj, profile=wprof, points=wpts, bands=wb, stream=stream),
                     a.reps, torch)
    grid_win = g.info(14)
    assert (pts.cpu().numpy() == n).all() and (wpts.cpu().numpy() == n[winners]).all()
    hprof, htraj, hpts = (torch.empty(x.shape, dtype=x.dtype, pin_memory=True) for x in (wprof, wtraj, wpts))

    def winners_to_host():
        g.read_trajectory_device(bs, trajectory=wtraj, profile=wprof, points=wpts, bands=wb, stream=stream)
        for h, d in ((hprof, wprof), (htraj, wtraj), (hpts, wpts)):
            h.copy_(d, non_blocking=True)
    ms_win_host = time_ms(winners_to_host, a.reps, torch)
    records = {k: torch.empty(t[k].shape, dtype=t[k].dtype, pin_memory=True) for k in ("poses", "n", "vel_start", "vel_goal")}

    def records_to_host():
        for k, h in records.items():
            h.copy_(t[k], non_blocking=True)
    ms_d2h = time_ms(records_to_host, a.reps, torch)
    rec_bytes = sum(t[k].numel() for k in records)
    out_bytes = lambda R: R * ((nc + 1) * 3 + nc * 7) * 8 + R * 4
    res["c3"].update(readout_all_ms=round(ms_all, 4), readout_all_grid=grid_all, readout_all_out_bytes=out_bytes(B),
                     readout_winners_ms=round(ms_win, 4), readout_winners_grid=grid_win,
                     readout_winners_to_host_ms=round(ms_win_host, 4), winners_out_bytes=out_bytes(requests),
                     records_d2h_ms=round(ms_d2h, 4), records_bytes=rec_bytes)
    g.close()
    print(f"C3 {B} bands ({requests} requests x {cand}), n_cap {nc}: read-out of every band {ms_all:.4f} ms (grid {grid_all}), "
          f"of the {requests} winners {ms_win:.4f} ms (grid {grid_win}), winners read out and copied to the host "
          f"{ms_win_host:.4f} ms; copy of the batch's records to the host {ms_d2h:.4f} ms ({rec_bytes / 1e6:.1f} MB)")
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
