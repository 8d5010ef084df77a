"""Time of the voxel-layer step (tebgpu_costmap_voxel_layer_device), CUDA events around the calls, against uploading
host-built rasters of the same size and against the obstacle layer's step on the same points.

  1024 and 8192 robots; 120 x 120 windows and the largest square that fits one CTA (tebgpu_get_info key 22), at 5 cm;
  a laser ring of 360 points at 0.2 m (a third of the beams hitting at 0.5 .. 2.4 m, the rest at 3.5 m) plus a depth
  cloud of 1000 or 4000 points at 0.3 m (a 70 x 24 degree view ahead, ranges 0.5 .. 3.5 m); K = 1 (the laser and the
  cloud as one source) and K = 2 (one source each); z_voxels 10 at 0.1 m, combine mode, a rectangular footprint;
  the host-to-device copy of the same [S][cell_cap] master rasters from pinned memory;
  the obstacle layer's step over the same points as one source (tebgpu_costmap_obstacle_layer_device).
Every time is the median of --repeats runs of --reps calls each (min and max beside it).

    python tools/costmap_voxel_layer.py [--reps 20] [--repeats 5] [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query), then one JSON line."""
import argparse
import json
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi  # noqa: E402
from tests import costmap_window_cases as cw  # noqa: E402
from tests import obstacle_layer_cases as ol  # noqa: E402
from tests import voxel_layer_cases as vl  # noqa: E402
from tools.costmap_obstacle_layer import spread, FOOTPRINT, RES  # noqa: E402
from tools.trajectory_readout import card  # noqa: E402

LASER = 360
VOXEL = dict(vl.PARAMS, mode=vl.COMBINE, z_voxels=10, z_resolution=0.1, max_obstacle_height=1.0)
SOURCE = dict(vl.SOURCE, obstacle_range=2.5, raytrace_range=3.0, min_obstacle_height=0.05)


def setup(S, side, C, seed=0):
    rng = np.random.default_rng(seed)
    robot = np.column_stack([rng.uniform(-50, 50, (S, 2)), rng.uniform(-np.pi, np.pi, S)])
    lo = robot[:, :2] - side * RES / 2 + rng.uniform(-0.5, 0.5, (S, 2))
    org = np.column_stack([[cw.snap(lo[s, 0], robot[s, 0], side, RES) for s in range(S)],
                           [cw.snap(lo[s, 1], robot[s, 1], side, RES) for s in range(S)], np.full(S, RES)])
    ang = robot[:, 2:3] + np.linspace(-np.pi, np.pi, LASER, endpoint=False)[None, :]
    dist = np.where(rng.uniform(0, 1, (S, LASER)) < 1 / 3, rng.uniform(0.5, 2.4, (S, LASER)), 3.5)
    laser = np.stack([robot[:, None, 0] + dist * np.cos(ang), robot[:, None, 1] + dist * np.sin(ang),
                      np.full((S, LASER), 0.2)], -1)
    az = robot[:, 2:3] + rng.uniform(-math.radians(35), math.radians(35), (S, C))
    el = rng.uniform(-math.radians(12), math.radians(12), (S, C))
    rr = rng.uniform(0.5, 3.5, (S, C))
    cloud = np.stack([robot[:, None, 0] + rr * np.cos(el) * np.cos(az), robot[:, None, 1] + rr * np.cos(el) * np.sin(az),
                      0.3 + rr * np.sin(el)], -1)
    sensors = np.stack([np.column_stack([robot[:, :2], np.full(S, 0.2)]),
                        np.column_stack([robot[:, :2], np.full(S, 0.3)])], 1)
    master = np.tile(rng.choice(np.array([0, 254, 255], np.uint8), side * side, p=[0.8, 0.1, 0.1]), (S, 1))
    return laser.astype(np.float32), cloud.astype(np.float32), sensors, robot, lo, org, master


def run(a, torch):
    res = dict(card=card(), resolution=RES, rows=[])
    print("card, power limit:", res["card"])
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    g = T.TebGpu(64, 64, 8192, 64, 0)
    g.set_params(abi.default_params())
    big = int(math.isqrt(g.voxel_layer_max_cell_cap()))
    tt = lambda v: torch.from_numpy(np.ascontiguousarray(v)).to(dev)
    for S in (1024, 8192):
        for side in (120, big):
            for C in (1000, 4000):
                laser, cloud, sensors, robot, lo, org, master = setup(S, side, C)
                cap, P = side * side, max(LASER, C)
                common = dict(robot=tt(robot), grid=tt(np.full((S, 2), side, np.int32)), origin=tt(org), cost=tt(master),
                              status=torch.zeros(S, dtype=torch.int32, device=dev))
                for K in (1, 2):
                    if K == 1:
                        pts = np.concatenate([laser, cloud], 1)[:, None]
                        cnt, sen = np.full((S, 1), LASER + C, np.int32), sensors[:, 1:2]
                    else:
                        pts = np.zeros((S, 2, P, 3), np.float32)
                        pts[:, 0, :LASER], pts[:, 1, :C] = laser, cloud
                        cnt, sen = np.tile(np.array([LASER, C], np.int32), (S, 1)), sensors
                    vox, lay = vl.reset_rows(S, cap)
                    d = dict(common, points=tt(pts), point_count=tt(cnt), sensor_origin=tt(sen),
                             voxels=tt(vox.view(np.int32)), layer=tt(lay), layer_origin=tt(lo))
                    args = abi.make_voxel_layer_args(S, cap, pts.shape[2], [abi.make_observation_source(**SOURCE)] * K,
                                                     np.array(FOOTPRINT), **VOXEL, **{k: v.data_ptr() for k, v in d.items()})
                    ms = spread(lambda: g.costmap_voxel_layer_device(args, stream=stream), a, torch)
                    assert (d["status"].cpu().numpy() == vl.OK).all()
                    row = dict(robots=S, window=f"{side}x{side}", laser=LASER, cloud=C, K=K, step_ms=ms)
                    if K == 1:
                        ob = dict(common, points=tt(pts[:, 0]), point_count=tt(cnt[:, 0]), sensor_origin=tt(sen[:, 0]),
                                  layer=tt(lay), layer_origin=tt(lo))
                        oargs = abi.make_obstacle_layer_args(S, cap, pts.shape[2], np.array(FOOTPRINT),
                                                             **dict(ol.PARAMS, mode=ol.COMBINE, obstacle_range=2.5,
                                                                    raytrace_range=3.0, min_obstacle_height=0.05,
                                                                    layer_max_obstacle_height=1.0),
                                                             **{k: v.data_ptr() for k, v in ob.items()})
                        row["obstacle_layer_ms"] = spread(lambda: g.costmap_obstacle_layer_device(oargs, stream=stream),
                                                          a, torch)
                        pinned = torch.empty((S, cap), dtype=torch.uint8, pin_memory=True)
                        pinned.copy_(d["cost"].cpu())
                        row["upload_pinned_ms"] = spread(lambda: d["cost"].copy_(pinned, non_blocking=True), a, torch)
                        del ob, pinned
                    res["rows"].append(row)
                    extra = "" if K == 2 else (f", obstacle layer {row['obstacle_layer_ms']['median']:.4f} ms, "
                                               f"pinned upload {row['upload_pinned_ms']['median']:.4f} ms")
                    print(f"{S:5d} robots, {side}^2, laser {LASER} + cloud {C:4d}, K={K}: voxel layer "
                          f"{ms['median']:.4f} ms [{ms['min']:.4f}, {ms['max']:.4f}]{extra}")
                    del d
                    torch.cuda.empty_cache()
                del common
    g.close()
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measurement runs on the GPU only")
    with torch.cuda.stream(torch.cuda.Stream()):
        run(a, torch)


if __name__ == "__main__":
    main()
