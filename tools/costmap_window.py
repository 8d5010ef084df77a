"""Time of the rolling-window step (tebgpu_costmap_window_device), CUDA events around the calls, against uploading
host-built rasters of the same size and against building them on the host.

  1024 and 8192 robots; 120 x 120 and 400 x 400 windows at 5 cm; a 4000 x 4000 map (16 MB) and an 8000 x 8000 map
  (64 MB, more than the H100's 50 MB L2), both at 5 cm, robots spread over the map;
  the window step without a transform and with a planar costmap -> map transform (both launches);
  the host-to-device copy of the same [S][cell_cap] rasters from pinned memory;
  the host build: tests/costmap_window_cases.py's numpy restatement, timed per robot on up to 64 robots and scaled to
  S (an extrapolation, marked so in the output);
  a 20-cycle fleet loop (raster, costmap conversion, plan cycle of a C2-like fleet) fed by the window step against the
  same loop fed by the pinned upload, at 1024 robots with 120 x 120 windows on the 4000 x 4000 map.
Every time is the median of --repeats runs of --reps calls each (min and max beside it). The bandwidth share is the
raster bytes stored over the time, against the data sheet's 3.35 TB/s; the map gathers come on top of it.

    python tools/costmap_window.py [--reps 20] [--repeats 5] [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query), then one JSON line."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi, scenes  # noqa: E402
from tests import costmap_window_cases as cw  # noqa: E402
from tools.trajectory_readout import card, time_ms  # noqa: E402

RES, HBM_TBS = 0.05, 3.35


def spread(fn, a, torch):
    v = sorted(time_ms(fn, a.reps, torch) for _ in range(a.repeats))
    return dict(median=round(v[len(v) // 2], 4), min=round(v[0], 4), max=round(v[-1], 4))


def setup(S, side, m, torch, seed=0):
    rng = np.random.default_rng(seed)
    msy, msx = m["data"].shape
    xy = rng.uniform([m["mox"], m["moy"]], [m["mox"] + msx * RES, m["moy"] + msy * RES], (S, 2))
    robot = np.column_stack([xy, rng.uniform(-np.pi, np.pi, S)])
    origin = np.column_stack([xy - 3.0, np.full(S, RES)])
    grid = np.full((S, 2), side, np.int32)
    tf = np.tile([0.4, -0.3, 0.0, 0.0, 0.0, np.sin(0.01), np.cos(0.01)], (S, 1))
    return robot, origin, grid, tf


def device_args(S, side, robot, origin, grid, tf, torch):
    dev = torch.device("cuda:0")
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    d = dict(robot=t(robot), origin=t(origin), grid=t(grid), tf=t(tf), map_id=torch.zeros(S, dtype=torch.int32, device=dev),
             cost=torch.empty((S, side * side), dtype=torch.uint8, device=dev),
             status=torch.empty(S, dtype=torch.int32, device=dev))
    wa = abi.TebCostmapWindowArgs()
    wa.S, wa.cell_cap = S, side * side
    wa.robot, wa.map_id, wa.origin = d["robot"].data_ptr(), d["map_id"].data_ptr(), d["origin"].data_ptr()
    wa.grid, wa.cost, wa.status = d["grid"].data_ptr(), d["cost"].data_ptr(), d["status"].data_ptr()
    return wa, d


def run(a, torch):
    res = dict(card=card(), resolution=RES, rows=[], loop=None)
    print("card, power limit:", res["card"])
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(1)
    g = T.TebGpu(1024, 100, 8192, 4096, 0)
    g.set_params(abi.default_params())
    for side_m in (4000, 8000):
        m = cw.random_map(rng, side_m, side_m, -side_m * RES / 2, -side_m * RES / 2, RES)
        sm, arrays = abi.make_static_maps([m["data"]], [(m["mox"], m["moy"], m["mr"])])
        keep = {k: torch.from_numpy(v).to(dev) for k, v in arrays.items()}
        sm.data, sm.offset, sm.size, sm.origin = (keep[k].data_ptr() for k in ("data", "offset", "size", "origin"))
        for S in (1024, 8192):
            for side in (120, 400):
                robot, origin, grid, tf = setup(S, side, m, torch)
                wa, d = device_args(S, side, robot, origin, grid, tf, torch)
                ms_id = spread(lambda: g.costmap_window_device(sm, wa, stream=stream), a, torch)
                assert (d["status"].cpu().numpy() == 0).all()
                wa.costmap_to_map = d["tf"].data_ptr()
                ms_tf = spread(lambda: g.costmap_window_device(sm, wa, stream=stream), a, torch)
                h = torch.empty((S, side * side), dtype=torch.uint8, pin_memory=True)
                h.copy_(d["cost"].cpu())
                ms_h2d = spread(lambda: d["cost"].copy_(h, non_blocking=True), a, torch)
                k = min(S, 64)
                t0 = time.perf_counter()
                cw.window_np([m], robot[:k], np.zeros(k, np.int32), origin[:k], grid[:k], side * side)
                host_ms = (time.perf_counter() - t0) * 1e3 * S / k
                nbytes = S * side * side
                row = dict(map=f"{side_m}x{side_m}", map_bytes=side_m * side_m, robots=S, window=f"{side}x{side}",
                           raster_bytes=nbytes, window_ms=ms_id, window_tf_ms=ms_tf, upload_pinned_ms=ms_h2d,
                           host_build_ms_extrapolated=round(host_ms, 1),
                           window_store_TBs=round(nbytes / (ms_id["median"] * 1e-3) / 1e12, 3),
                           window_store_share=round(nbytes / (ms_id["median"] * 1e-3) / 1e12 / HBM_TBS, 3),
                           grid_ctas=int(g.last_window_grid()))
                res["rows"].append(row)
                print(f"map {side_m}^2, {S:5d} robots, {side}^2 windows ({nbytes / 1e6:.1f} MB): window {ms_id['median']:.4f} "
                      f"ms (tf {ms_tf['median']:.4f}), pinned upload {ms_h2d['median']:.4f} ms, host build ~{host_ms:.0f} ms, "
                      f"stores {row['window_store_TBs']} TB/s ({100 * row['window_store_share']:.1f}% of {HBM_TBS})")
                del d, h
                torch.cuda.empty_cache()
        if side_m == 4000:
            res["loop"] = fleet_loop(g, sm, m, a, torch, stream)
        del keep
    g.close()
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


def fleet_loop(g, sm, m, a, torch, stream, S=1024, side=120, cycles=20):
    """20 cycles of (raster, conversion, plan) with the raster from the window step or from a pinned upload"""
    dev = torch.device("cuda:0")
    robot, origin, grid, tf = setup(S, side, m, torch, seed=2)
    wa, d = device_args(S, side, robot, origin, grid, tf, torch)
    g.costmap_window_device(sm, wa, stream=stream)
    h = torch.empty((S, side * side), dtype=torch.uint8, pin_memory=True)
    h.copy_(d["cost"].cpu())
    p = scenes.config_params("C2")
    p.footprint_type, p.footprint_radius = abi.TEB_FOOTPRINT_CIRCULAR, 0.2
    p.include_dynamic_obstacles = 0
    g.set_params(p)
    args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale, 1.0, False)
    M_cap = 4096
    obst = torch.empty((S, M_cap * 64), dtype=torch.uint8, device=dev)
    ocount = torch.empty(S, dtype=torch.int32, device=dev)
    ca = abi.TebCostmapArgs()
    ca.S, ca.cell_cap, ca.M_cap, ca.include_costmap_obstacles, ca.behind_robot_dist = S, side * side, M_cap, 1, 1.5
    ca.cost, ca.grid, ca.origin, ca.robot = (d[k].data_ptr() for k in ("cost", "grid", "origin", "robot"))
    ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
    nc = 100
    z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
    tt = dict(poses=z((S, nc, 4), torch.float64), n=z(S, torch.int32), sid=torch.arange(S, dtype=torch.int32, device=dev),
              cost=z(S, torch.float64), chi2=z(S, torch.float64), status=z(S, torch.int32), iters=z(S, torch.int32))
    vel = z((S, 4), torch.float64)
    vel[:, 3] = 1.0
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap = S, nc, S, M_cap
    bs.poses, bs.n, bs.scene_id = tt["poses"].data_ptr(), tt["n"].data_ptr(), tt["sid"].data_ptr()
    bs.obstacles, bs.obst_count = obst.data_ptr(), ocount.data_ptr()
    bs.vel_start = bs.vel_goal = vel.data_ptr()
    bs.cost, bs.chi2, bs.status, bs.lm_iters = (tt[k].data_ptr() for k in ("cost", "chi2", "status", "iters"))
    goal = robot.copy()
    goal[:, 0] += 2.5 * np.cos(robot[:, 2])
    goal[:, 1] += 2.5 * np.sin(robot[:, 2])
    st, gl = torch.from_numpy(robot).to(dev), torch.from_numpy(goal).to(dev)
    cmd = z((S, 4), torch.float64)

    def loop(window):
        tt["n"].zero_()
        for _ in range(cycles):
            if window:
                g.costmap_window_device(sm, wa, stream=stream)
            else:
                d["cost"].copy_(h, non_blocking=True)
            g.costmap_obstacles_device(ca, stream=stream)
            g.plan_device(bs, args, cmd, start=st, goal=gl, stream=stream)

    out = {}
    for name, w in (("window", True), ("upload", False), ("window_again", True), ("upload_again", False)):
        v = sorted(time_ms(lambda: loop(w), 1, torch) for _ in range(a.repeats))
        out[name + "_ms"] = dict(median=round(v[len(v) // 2], 3), min=round(v[0], 3), max=round(v[-1], 3))
    out.update(robots=S, window=f"{side}x{side}", cycles=cycles)
    print(f"20-cycle loop, {S} robots, {side}^2 windows: with the window step {out['window_ms']['median']:.3f} ms "
          f"({out['window_again_ms']['median']:.3f}), with the pinned upload {out['upload_ms']['median']:.3f} ms "
          f"({out['upload_again_ms']['median']:.3f})")
    return out


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
