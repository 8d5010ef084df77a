"""Time of the costmap-to-obstacle conversion (tebgpu_costmap_obstacles_device), CUDA events around the calls, against
the uploads it replaces and one plan cycle for scale.

  1, 256 and 2048 scenes of 120 x 120 cells at 5 cm (scenes.costmap_raster), at two lethal fractions;
  the conversion of every scene into its [M_cap] table (M_cap: the largest scene's row count, rounded up to 64);
  the host-to-device copy of the rasters from pinned memory (what the conversion needs uploaded);
  the host-to-device copy of the equivalent [S][M_cap] tables from pinned memory (what a host-built table needs);
  one tebgpu_plan_batch_device cycle of a C2-like fleet on the converted tables: one band per scene, 100 poses, warm.

    python tools/costmap_obstacles.py [--scenes 1,256,2048] [--reps 50] [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query), then one JSON line."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi, scenes  # noqa: E402
from tools.trajectory_readout import card, time_ms  # noqa: E402

SIDE, RES = 120, 0.05


def fleet(S, lethal, seed=0):
    """S rasters: 64 distinct ones drawn, repeated with their own robot poses"""
    base = scenes.costmap_raster(min(S, 64), SIDE, SIDE, RES, lethal, seed=seed)
    k = np.arange(S) % len(base["cost"])
    return {key: np.ascontiguousarray(v[k]) for key, v in base.items()}


def run(a, torch):
    res = dict(card=card(), side=SIDE, resolution=RES, rows=[])
    print("card, power limit:", res["card"])
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 0
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    for S in [int(x) for x in a.scenes.split(",")]:
        for lethal in (0.05, 0.2):
            f = fleet(S, lethal)
            cell_cap = f["cost"].shape[1]
            g = T.TebGpu(S, 100, S, 16384, 0)
            g.set_params(p)
            _, _, need = g.costmap_obstacles(f["cost"], f["grid"], f["origin"], f["robot"], 64)   # needed: the row counts
            M_cap = int(-(-max(int(need.max()), 1) // 64) * 64)
            d = {k: torch.from_numpy(v).to(dev) for k, v in f.items()}
            obst = torch.empty((S, M_cap * 64), dtype=torch.uint8, device=dev)
            ocount = torch.empty(S, dtype=torch.int32, device=dev)
            ca = abi.TebCostmapArgs()
            ca.S, ca.cell_cap, ca.M_cap, ca.include_costmap_obstacles, ca.behind_robot_dist = S, cell_cap, M_cap, 1, 1.5
            ca.cost, ca.grid, ca.origin, ca.robot = (d[k].data_ptr() for k in ("cost", "grid", "origin", "robot"))
            ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
            ms_conv = time_ms(lambda: g.costmap_obstacles_device(ca, stream=stream), a.reps, torch)
            assert (ocount.cpu().numpy() == need).all()
            h_raster = torch.from_numpy(f["cost"]).pin_memory()
            d_raster = torch.empty_like(h_raster, device=dev)
            ms_raster = time_ms(lambda: d_raster.copy_(h_raster, non_blocking=True), a.reps, torch)
            h_table = torch.empty((S, M_cap * 64), dtype=torch.uint8, pin_memory=True)
            h_table.copy_(obst.cpu())
            d_table = torch.empty_like(h_table, device=dev)
            ms_table = time_ms(lambda: d_table.copy_(h_table, non_blocking=True), a.reps, torch)
            # one band per scene, from its robot towards a goal 2.5 m ahead: a cold cycle, then the timed warm cycles
            B, nc = S, 100
            start = f["robot"].copy()
            goal = start.copy()
            goal[:, 0] += 2.5 * np.cos(start[:, 2])
            goal[:, 1] += 2.5 * np.sin(start[:, 2])
            t = dict(poses=torch.zeros((B, nc, 4), dtype=torch.float64, device=dev), n=torch.zeros(B, dtype=torch.int32, device=dev),
                     sid=torch.arange(B, dtype=torch.int32, device=dev), cost=torch.zeros(B, dtype=torch.float64, device=dev),
                     chi2=torch.zeros(B, dtype=torch.float64, device=dev), status=torch.zeros(B, dtype=torch.int32, device=dev),
                     iters=torch.zeros(B, dtype=torch.int32, device=dev))
            vel = torch.zeros((B, 4), dtype=torch.float64, device=dev)
            vel[:, 3] = 1.0
            bs = abi.TebBatch()
            bs.B, bs.n_cap, bs.S, bs.M_cap = B, nc, S, M_cap
            bs.poses, bs.n, bs.scene_id = t["poses"].data_ptr(), t["n"].data_ptr(), t["sid"].data_ptr()
            bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
            bs.vel_start = bs.vel_goal = vel.data_ptr()
            bs.cost, bs.chi2, bs.status, bs.lm_iters = (t[k].data_ptr() for k in ("cost", "chi2", "status", "iters"))
            st, gl = torch.from_numpy(start).to(dev), torch.from_numpy(goal).to(dev)
            cmd = torch.zeros((B, 4), dtype=torch.float64, device=dev)
            ms_plan = time_ms(lambda: g.plan_device(bs, args, cmd, start=st, goal=gl, stream=stream), max(3, a.reps // 10), torch)
            bad = int((t["status"].cpu().numpy() & abi.TEB_STATUS_BAD_INPUT).astype(bool).sum())
            g.close()
            row = dict(scenes=S, lethal=lethal, max_rows=int(need.max()), mean_rows=round(float(need.mean()), 1), M_cap=M_cap,
                       convert_ms=round(ms_conv, 4), raster_h2d_ms=round(ms_raster, 4), raster_bytes=int(h_raster.numel()),
                       table_h2d_ms=round(ms_table, 4), table_bytes=int(h_table.numel()), plan_cycle_ms=round(ms_plan, 3),
                       plan_bad_input_bands=bad)
            res["rows"].append(row)
            print(f"{S:5d} scenes, lethal {lethal:.2f}: rows mean {row['mean_rows']} max {row['max_rows']} (M_cap {M_cap}); "
                  f"convert {ms_conv:.4f} ms, raster H2D {ms_raster:.4f} ms ({row['raster_bytes'] / 1e6:.2f} MB), "
                  f"table H2D {ms_table:.4f} ms ({row['table_bytes'] / 1e6:.2f} MB), plan cycle {ms_plan:.3f} ms")
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="1,256,2048")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement runs on the GPU only")
    with torch.cuda.stream(torch.cuda.Stream()):
        run(a, torch)


if __name__ == "__main__":
    main()
