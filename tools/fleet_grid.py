"""The fleet steps' two neighbour searches, all pairs (tebgpu_set_fleet_search 1) and the grid (2), on the same seeded
inputs: each workload runs both searches alternately on one stream, CUDA events around every call, the median of --reps
calls after 3 warm-up calls of each; the outputs of the two (custom rows, custom_count, needed, status) are compared byte
for byte in the same run.

  array     tebgpu_fleet_obstacles_device over R robots of tools/fleet_obstacles.py's uniform square (one robot per
            4 m^2, range 3 m: about 7 neighbours), max_rows 8;
  table     tebgpu_fleet_obstacles_table_device: the last R_local of T published rows of the same square;
  worlds    W worlds of 8 robots, every world spread over the same 6 m x 6 m square (the array step over all W * 8
            robots, or the table step for the last 32768 of W * 8 rows);
  one_cell  the worst case: every robot inside one 1 m x 1 m square, range 3 m (every robot is every robot's neighbour).

    python tools/fleet_grid.py [--reps 20] [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query)."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi  # noqa: E402
from tools.fleet_obstacles import RANGE, fleet  # noqa: E402
from tools.local_plan import card  # noqa: E402

MAX_ROWS = 8
SEARCHES = {"all_pairs": abi.TEBGPU_FLEET_SEARCH_ALL_PAIRS, "grid": abi.TEBGPU_FLEET_SEARCH_GRID}


def worlds_fleet(W, per=8, seed=2):
    rng = np.random.default_rng(seed)
    R = W * per
    pose = np.column_stack([rng.uniform(0, 6.0, (R, 2)), rng.uniform(-np.pi, np.pi, R)])
    cmd = np.column_stack([rng.uniform(-0.2, 0.4, R), np.zeros(R), rng.uniform(-0.3, 0.3, R)])
    return pose, cmd, np.full(R, 0.3), np.repeat(np.arange(W, dtype=np.int32), per)


def one_cell_fleet(R, seed=3):
    pose, cmd, rad = fleet(R, seed)
    pose[:, :2] = np.random.default_rng(seed).uniform(0.0, 1.0, (R, 2))
    return pose, cmd, rad


def compare(pose, cmd, rad, world, R, reps, torch, table=False):
    """both searches on the robots' last R of len(pose) (table: every robot published, the last R stepped); returns
    the medians, the byte comparison and the mean neighbour count"""
    dev = torch.device("cuda:0")
    N = len(pose)
    g = T.TebGpu(R, 8, R, 64)
    t = lambda x: None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    tp, tc, tr, tw = t(pose), t(cmd), t(rad), t(world)
    s = torch.cuda.Stream()
    stream = s.cuda_stream
    mine = slice(N - R, N)
    rows = tb = None
    if table:
        rows = torch.zeros(N * abi.FLEET_ROW_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        for lo in range(0, N, R):
            hi = min(N, lo + R)
            fp = abi.make_fleet_args(hi - lo, 1, 0, 0, 0.0, pose=tp[lo:hi], last_cmd=tc[lo:hi], radius=tr[lo:hi],
                                     world=None if tw is None else tw[lo:hi])
            g.fleet_publish_device(fp, abi.make_fleet_table(N, lo, rows), stream=stream)
        tb = abi.make_fleet_table(N, N - R, rows)
    outs, args = {}, {}
    for name in SEARCHES:
        o = dict(custom=torch.zeros(R * MAX_ROWS * 64, dtype=torch.uint8, device=dev),
                 cc=torch.zeros(R, dtype=torch.int32, device=dev), need=torch.zeros(R, dtype=torch.int32, device=dev),
                 st=torch.zeros(R, dtype=torch.int32, device=dev))
        outs[name] = o
        args[name] = abi.make_fleet_args(R, R, MAX_ROWS, MAX_ROWS, RANGE, pose=tp[mine], last_cmd=tc[mine],
                                         radius=tr[mine], world=None if tw is None else tw[mine], custom=o["custom"],
                                         custom_count=o["cc"], needed=o["need"], status=o["st"])
    ms = {name: [] for name in SEARCHES}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    for r in range(reps + 3):
        for k, (name, mode) in enumerate(SEARCHES.items()):
            g.set_fleet_search(mode)
            ev[2 * k].record(s)
            if table:
                g.fleet_obstacles_table_device(args[name], tb, stream=stream)
            else:
                g.fleet_obstacles_device(args[name], stream=stream)
            ev[2 * k + 1].record(s)
            assert g.last_fleet_search() == name
        torch.cuda.synchronize()
        if r >= 3:
            for k, name in enumerate(SEARCHES):
                ms[name].append(ev[2 * k].elapsed_time(ev[2 * k + 1]))
    a, b = outs["all_pairs"], outs["grid"]
    same = all(torch.equal(a[k], b[k]) for k in a)
    res = dict(robots=R, candidates=N, all_pairs_ms=float(np.median(ms["all_pairs"])),
               grid_ms=float(np.median(ms["grid"])), bytes_equal=bool(same),
               mean_needed=float(a["need"].float().mean()), truncated=int((a["st"] == abi.TEB_FLEET_TRUNCATED).sum()))
    res["speedup"] = res["all_pairs_ms"] / res["grid_ms"]
    g.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--array", type=int, nargs="+", default=[1024, 2048, 4096, 6144, 8192, 12288, 16384, 32768])
    ap.add_argument("--table", nargs="+", default=["8192:65536", "32768:262144", "32768:1048576"])
    ap.add_argument("--one-cell", type=int, nargs="+", default=[8192, 32768])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    res = dict(card=card(), range_m=RANGE, max_rows=MAX_ROWS, reps=a.reps, array={}, table={}, worlds={}, one_cell={})
    print("card, power limit:", res["card"], flush=True)
    for R in a.array:
        pose, cmd, rad = fleet(R)
        res["array"][str(R)] = compare(pose, cmd, rad, None, R, a.reps, torch)
        print("array", R, res["array"][str(R)], flush=True)
    for pr in a.table:
        R, Tn = (int(v) for v in pr.split(":"))
        pose, cmd, rad = fleet(Tn)
        res["table"][pr] = compare(pose, cmd, rad, None, R, a.reps, torch, table=True)
        print("table", pr, res["table"][pr], flush=True)
    pose, cmd, rad, world = worlds_fleet(4096)
    res["worlds"]["array 4096 x 8"] = compare(pose, cmd, rad, world, len(pose), a.reps, torch)
    print("worlds array", res["worlds"]["array 4096 x 8"], flush=True)
    pose, cmd, rad, world = worlds_fleet(32768)
    res["worlds"]["table 32768 x 8"] = compare(pose, cmd, rad, world, 32768, a.reps, torch, table=True)
    print("worlds table", res["worlds"]["table 32768 x 8"], flush=True)
    for R in a.one_cell:
        pose, cmd, rad = one_cell_fleet(R)
        res["one_cell"][str(R)] = compare(pose, cmd, rad, None, R, a.reps, torch)
        print("one cell", R, res["one_cell"][str(R)], flush=True)
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    if not all(v["bytes_equal"] for grp in ("array", "table", "worlds", "one_cell") for v in res[grp].values()):
        sys.exit("the two searches wrote different bytes")


if __name__ == "__main__":
    main()
