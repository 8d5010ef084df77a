"""Time of one isTrajectoryFeasible check over a whole batch (tebgpu_check_feasible_device), CUDA events around the call.

  C3 at --bands bands (default 8192), look-ahead index 5 and the whole band;
  scenes.costmap_scene at M = 64 / 1024 / 1025 / 4096 / 16384 obstacles with --costmap-bands bands (default 2048),
  the whole band;
  one tebgpu_plan_batch_device cycle on the C3 batch, for scale.

    python tools/feasibility.py [--bands 8192] [--costmap-bands 2048] [--reps 20] [--json out.json]

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


def check_case(p, hb, torch, reps, inscribed, look_ahead_idx, max_queries, collision_distance=0.0):
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, max(hb.M_cap, 1), hb.V_cap, max_obst_vertices=hb.PV_cap)
    g.set_params(p)
    t, bs = device_batch(hb, torch)
    dev = torch.device("cuda:0")
    f = torch.zeros(hb.B, dtype=torch.int32, device=dev)
    k = torch.zeros(hb.B, dtype=torch.int32, device=dev)
    fa = abi.make_feasibility_args(inscribed, look_ahead_idx, max_queries=max_queries, collision_distance=collision_distance,
                                   feasible=f.data_ptr(), query_count=k.data_ptr())
    stream = torch.cuda.current_stream().cuda_stream
    ms = time_ms(lambda: g.check_feasible_device(bs, fa, stream=stream), reps, torch)
    build, grid = g.last_feasibility_check()
    fv, kv = f.cpu().numpy(), k.cpu().numpy()
    g.close()
    return dict(ms=round(ms, 4), build=build, grid=grid, feasible=int((fv == 1).sum()), infeasible=int((fv == 0).sum()),
                undecided=int((fv == -1).sum()), mean_queries=round(float(kv.mean()), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bands", type=int, default=8192)
    ap.add_argument("--costmap-bands", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=20)
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
    inscribed = 0.2                                      # a footprint of that inscribed radius samples every 20 cm
    requests = 128 if a.bands % 128 == 0 else 1             # C3 requests of bands / 128 candidates each
    p, hb = scenes.make_config_batch("C3", requests=requests, candidates=a.bands // requests, seed=1)
    res["c3"] = dict(bands=hb.B, n=int(hb.n.max()), M=hb.M_cap)
    for name, lai in (("look_ahead_5", 5), ("whole_band", -1)):
        r = check_case(p, hb, torch, a.reps, inscribed, lai, 4096, collision_distance=0.0)
        res["c3"][name] = r
        print(f"C3 {hb.B} bands, {name}: {r}")
    # one plan cycle on the same batch, for scale
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap)
    g.set_params(p)
    t, bs = device_batch(hb, torch)
    dev = torch.device("cuda:0")
    start = torch.from_numpy(np.ascontiguousarray(hb.poses[:, 0, :3])).to(dev)
    goal = torch.from_numpy(np.ascontiguousarray(hb.poses[np.arange(hb.B), hb.n - 1, :3])).to(dev)
    cmd = torch.zeros((hb.B, 4), dtype=torch.float64, device=dev)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    stream = torch.cuda.current_stream().cuda_stream
    poses0 = t["poses"].clone()
    n0 = t["n"].clone()

    def cycle():
        t["poses"].copy_(poses0)
        t["n"].copy_(n0)
        g.plan_device(bs, args, cmd, start=start, goal=goal, stream=stream)
    res["c3"]["plan_cycle_ms"] = round(time_ms(cycle, max(3, a.reps // 4), torch), 3)
    print(f"C3 {hb.B} bands, one plan_batch_device cycle: {res['c3']['plan_cycle_ms']} ms")
    g.close()
    res["costmap"] = {}
    for M in (64, 1024, 1025, 4096, 16384):
        pc, hc = scenes.costmap_scene(M, n=100, candidates=a.costmap_bands, seed=2)
        pc.footprint_type, pc.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.15
        r = check_case(pc, hc, torch, a.reps, inscribed, -1, 4096)
        res["costmap"][str(M)] = r
        print(f"costmap M={M}, {hc.B} bands, whole band: {r}")
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
