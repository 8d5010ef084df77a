"""Time of isTrajectoryFeasible for a fleet against its costmaps (tebgpu_check_feasible_costmap_device) beside the
obstacle-table check on the same fleet (tebgpu_check_feasible_device), CUDA events around the calls.

  scenes: scenes.costmap_raster maps of 120 x 120 and 400 x 400 cells at 5 cm (64 distinct maps, repeated), one per robot;
  tables: each scene's obstacle table from its raster (tebgpu_costmap_obstacles_device, every lethal cell a row, M_cap:
          the largest row count rounded up to 64), the table check's world;
  bands:  C3 candidate bands (scenes.make_config_batch("C3")) moved so that pose 0 is the map's robot;
  1024 and 8192 robots; the costmap check with a 4- and a 16-vertex footprint, the table check with C3's footprint
  model and collision_distance 0. Both checks: the whole band, interpolation step 0.1, max_queries 2048.

    python tools/costmap_feasibility.py [--robots 1024,8192] [--sides 120,400] [--reps 20] [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query), then one JSON line."""
import argparse
import json
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi, scenes  # noqa: E402
from tools.trajectory_readout import card, time_ms  # noqa: E402

RES, INSCRIBED, MAX_Q = 0.05, 0.1, 2048
BEHIND = 1e9            # every lethal cell becomes a row: the table holds the same obstacles as the raster


def footprint(F):
    if F == 4:
        return np.array([(-0.25, -0.2), (0.35, -0.2), (0.35, 0.2), (-0.25, 0.2)])
    a = 2 * math.pi * np.arange(F) / F
    return np.stack([0.3 * np.cos(a), 0.3 * np.sin(a)], 1)


def fleet(B, side, seed=0):
    """B robots, each on its own copy of one of 64 rasters, with C3 bands moved onto them"""
    base = scenes.costmap_raster(64, side, side, RES, 0.05, seed=seed)
    k = np.arange(B) % 64
    ras = {key: np.ascontiguousarray(v[k]) for key, v in base.items()}
    p, hb = scenes.make_config_batch("C3", candidates=64, seed=seed)
    j = np.arange(B) % hb.B
    poses = hb.poses[j].copy()
    n = hb.n[j].copy()
    poses[:, :, 0] += (ras["robot"][:, 0] - poses[:, 0, 0])[:, None]
    poses[:, :, 1] += (ras["robot"][:, 1] - poses[:, 0, 1])[:, None]
    return p, ras, poses, n


def run(a, torch):
    res = dict(card=card(), resolution=RES, inscribed_radius=INSCRIBED, max_queries=MAX_Q, rows=[])
    print("card, power limit:", res["card"])
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    for side in [int(x) for x in a.sides.split(",")]:
        for B in [int(x) for x in a.robots.split(",")]:
            p, ras, poses, n = fleet(B, side)
            S, nc = B, poses.shape[1]
            g = T.TebGpu(B, nc, S, 16384, 0)
            g.set_params(p)
            d = {k: torch.from_numpy(v).to(dev) for k, v in ras.items()}
            # the tables, converted on the device from the same rasters
            _, _, need = g.costmap_obstacles(ras["cost"][:64], ras["grid"][:64], ras["origin"][:64], ras["robot"][:64], 64,
                                             behind_robot_dist=BEHIND)
            M_cap = int(-(-max(int(need.max()), 1) // 64) * 64)
            obst = torch.zeros((S, M_cap * 64), dtype=torch.uint8, device=dev)
            ocount = torch.zeros(S, dtype=torch.int32, device=dev)
            ca = abi.TebCostmapArgs()
            ca.S, ca.cell_cap, ca.M_cap, ca.include_costmap_obstacles, ca.behind_robot_dist = S, ras["cost"].shape[1], M_cap, 1, BEHIND
            ca.cost, ca.grid, ca.origin, ca.robot = (d[k].data_ptr() for k in ("cost", "grid", "origin", "robot"))
            ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
            g.costmap_obstacles_device(ca, stream=stream)
            assert (ocount.cpu().numpy() >= 0).all(), "a table overflowed M_cap"
            t = dict(poses=torch.from_numpy(poses).to(dev), n=torch.from_numpy(n).to(dev),
                     sid=torch.arange(B, dtype=torch.int32, device=dev))
            bs = abi.TebBatch()
            bs.B, bs.n_cap, bs.S, bs.M_cap = B, nc, S, M_cap
            bs.poses, bs.n, bs.scene_id = t["poses"].data_ptr(), t["n"].data_ptr(), t["sid"].data_ptr()
            bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
            f = torch.zeros(B, dtype=torch.int32, device=dev)
            k = torch.zeros(B, dtype=torch.int32, device=dev)
            fa = abi.make_feasibility_args(INSCRIBED, max_queries=MAX_Q, feasible=f.data_ptr(), query_count=k.data_ptr())
            reps = a.reps
            ms_table = time_ms(lambda: g.check_feasible_device(bs, fa, stream=stream), reps, torch)
            table = dict(feasible=int((f == 1).sum()), infeasible=int((f == 0).sum()), queries=int(k.sum()))
            row = dict(side=side, robots=B, M_cap=M_cap, mean_rows=round(float(ocount.float().mean()), 1),
                       table_ms=round(ms_table, 4), table_verdicts=table)
            for F in (4, 16):
                w = abi.make_costmap_world(ras["cost"].shape[1], d["cost"].data_ptr(), d["grid"].data_ptr(),
                                           d["origin"].data_ptr(), footprint(F))
                ms = time_ms(lambda: g.check_feasible_costmap_device(bs, fa, w, stream=stream), reps, torch)
                row[f"costmap_F{F}_ms"] = round(ms, 4)
                row[f"costmap_F{F}_verdicts"] = dict(feasible=int((f == 1).sum()), infeasible=int((f == 0).sum()),
                                                     queries=int(k.sum()))
            g.close()
            res["rows"].append(row)
            print(f"{side}x{side} cells, {B} robots, {row['mean_rows']} table rows (M_cap {M_cap}): table "
                  f"{ms_table:.3f} ms {table}; costmap F=4 {row['costmap_F4_ms']:.3f} ms {row['costmap_F4_verdicts']}, "
                  f"F=16 {row['costmap_F16_ms']:.3f} ms {row['costmap_F16_verdicts']}")
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--robots", default="1024,8192")
    ap.add_argument("--sides", default="120,400")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement runs on the GPU only")
    with torch.cuda.stream(torch.cuda.Stream()):
        run(a, torch)


if __name__ == "__main__":
    main()
