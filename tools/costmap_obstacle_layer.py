"""Time of the obstacle-layer step (tebgpu_costmap_obstacle_layer_device), CUDA events around the calls, against
uploading host-built rasters of the same size and against building them on the host.

  1024 and 8192 robots; 120 x 120 and 400 x 400 windows at 5 cm; 360 and 1440 points per robot, a laser ring around
  each robot (a third of the beams hitting at 0.5 .. 2.4 m and marking, the rest at 3.5 m, clearing only), a
  rectangular footprint; both modes (combine: on top of a static window in the master row; standalone);
  the host-to-device copy of the same [S][cell_cap] master rasters from pinned memory;
  the host build: tests/obstacle_layer_cases.py's numpy restatement, timed on up to 64 robots and scaled to S (an
  extrapolation, marked so in the output).
Every time is the median of --repeats runs of --reps calls each (min and max beside it). "cells/s" is the number of
cells the rays visit (counted by the restatement on 8 robots and scaled to S, an estimate) over the step's time; "row
bytes" is the layer row read and written plus the master row written (and read, in combine mode), against the data
sheet's 3.35 TB/s.

    python tools/costmap_obstacle_layer.py [--reps 20] [--repeats 5] [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query), then one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi  # noqa: E402
from tests import costmap_window_cases as cw  # noqa: E402
from tests import obstacle_layer_cases as ol  # noqa: E402
from tools.trajectory_readout import card, time_ms  # noqa: E402

RES, HBM_TBS = 0.05, 3.35
FOOTPRINT = [(-0.3, -0.25), (0.3, -0.25), (0.3, 0.25), (-0.3, 0.25)]


def spread(fn, a, torch):
    v = sorted(time_ms(fn, a.reps, torch) for _ in range(a.repeats))
    return dict(median=round(v[len(v) // 2], 4), min=round(v[0], 4), max=round(v[-1], 4))


def setup(S, side, P, mode, seed=0):
    rng = np.random.default_rng(seed)
    robot = np.column_stack([rng.uniform(-50, 50, (S, 2)), rng.uniform(-np.pi, np.pi, S)])
    lo = robot[:, :2] - side * RES / 2 + rng.uniform(-0.5, 0.5, (S, 2))
    grid = np.full((S, 2), side, np.int32)
    org = np.column_stack([[cw.snap(lo[s, 0], robot[s, 0], side, RES) for s in range(S)],
                           [cw.snap(lo[s, 1], robot[s, 1], side, RES) for s in range(S)], np.full(S, RES)])
    sensor = np.column_stack([robot[:, :2], np.full(S, 0.2)])
    ang = robot[:, 2:3] + np.linspace(-np.pi, np.pi, P, endpoint=False)[None, :]
    dist = np.where(rng.uniform(0, 1, (S, P)) < 1 / 3, rng.uniform(0.5, 2.4, (S, P)), 3.5)
    pts = np.stack([sensor[:, None, 0] + dist * np.cos(ang), sensor[:, None, 1] + dist * np.sin(ang),
                    np.full((S, P), 0.2)], -1).astype(np.float32)
    layer = np.full((S, side * side), 255, np.uint8)
    master = np.tile(rng.choice(np.array([0, 254, 255], np.uint8), side * side, p=[0.8, 0.1, 0.1]), (S, 1))
    return dict(points=pts, point_count=np.full(S, P, np.int32), sensor_origin=sensor, robot=robot, grid=grid,
                layer=layer, layer_origin=lo, origin=org, cost=master)


def ray_cells(h, k, p):
    """cells the rays of the first k robots visit, by the restatement"""
    n = 0
    for s in range(k):
        ox, oy = h["layer_origin"][s]
        nox = ox + ol.shift_cells(ox, h["robot"][s, 0], h["grid"][s, 0], RES) * RES
        noy = oy + ol.shift_cells(oy, h["robot"][s, 1], h["grid"][s, 1], RES) * RES
        side = int(h["grid"][s, 0])
        c0 = ol.world_to_map(h["sensor_origin"][s, 0], h["sensor_origin"][s, 1], nox, noy, RES, side, side)
        ml = ol.cell_distance(p["raytrace_range"], RES)
        for x, y, _ in h["points"][s].astype(np.float64):
            wx, wy = ol.clamp_to_map(x, y, h["sensor_origin"][s, 0], h["sensor_origin"][s, 1], nox, noy,
                                     nox + side * RES, noy + side * RES)
            c1 = ol.world_to_map(wx, wy, nox, noy, RES, side, side)
            if c0 and c1:
                n += len(ol.raytrace_line(c0[0], c0[1], c1[0], c1[1], side, ml))
    return n


def run(a, torch):
    res = dict(card=card(), resolution=RES, rows=[])
    print("card, power limit:", res["card"])
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    g = T.TebGpu(64, 64, 8192, 64, 0)
    g.set_params(abi.default_params())
    for S in (1024, 8192):
        for side in (120, 400):
            for P in (360, 1440):
                for mode in (ol.COMBINE, ol.STANDALONE):
                    h = setup(S, side, P, mode)
                    d = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in h.items()}
                    d["status"] = torch.zeros(S, dtype=torch.int32, device=dev)
                    p = dict(ol.PARAMS, mode=mode)
                    args = abi.make_obstacle_layer_args(S, side * side, P, np.array(FOOTPRINT), **p,
                                                        **{k: v.data_ptr() for k, v in d.items()})
                    ms = spread(lambda: g.costmap_obstacle_layer_device(args, stream=stream), a, torch)
                    assert (d["status"].cpu().numpy() == ol.OK).all()
                    pinned = torch.empty((S, side * side), dtype=torch.uint8, pin_memory=True)
                    pinned.copy_(d["cost"].cpu())
                    up = spread(lambda: d["cost"].copy_(pinned, non_blocking=True), a, torch)
                    k = min(S, 64)
                    sub = {kk: v[:k] for kk, v in h.items()}
                    t0 = time.perf_counter()
                    ol.obstacle_layer_np(p, sub["points"], sub["point_count"], sub["sensor_origin"], sub["robot"],
                                         sub["grid"], side * side, sub["layer"], sub["layer_origin"], sub["cost"],
                                         sub["origin"], FOOTPRINT)
                    host_ms = (time.perf_counter() - t0) * 1e3 * S / k
                    cells = ray_cells(h, 8, p) * S / 8
                    nbytes = S * side * side * (4 if mode == ol.COMBINE else 3)
                    row = dict(robots=S, window=f"{side}x{side}", points=P, mode="combine" if mode == ol.COMBINE else "standalone",
                               step_ms=ms, upload_pinned_ms=up, host_build_ms_extrapolated=round(host_ms, 1),
                               ray_cells_per_s_estimated=round(cells / (ms["median"] * 1e-3), -6),
                               row_TBs=round(nbytes / (ms["median"] * 1e-3) / 1e12, 3),
                               row_share=round(nbytes / (ms["median"] * 1e-3) / 1e12 / HBM_TBS, 3))
                    res["rows"].append(row)
                    print(f"{S:5d} robots, {side}^2, {P:4d} points, {row['mode']:10s}: step {ms['median']:.4f} ms "
                          f"[{ms['min']:.4f}, {ms['max']:.4f}], pinned upload {up['median']:.4f} ms, host ~{host_ms:.0f} ms "
                          f"(extrapolated), rays ~{row['ray_cells_per_s_estimated'] / 1e9:.1f} G cells/s, rows "
                          f"{row['row_TBs']} TB/s ({100 * row['row_share']:.1f}% of {HBM_TBS})")
                    del d, pinned
                    torch.cuda.empty_cache()
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
