"""Neighbours by footprints against neighbours by centres (TebFleetShapes.select), on the same fleets.

R robots on a square at one robot per 4 m^2 (tools/fleet_obstacles.fleet, range 3 m, max_rows 8) in one context whose
footprint is C3's TwoCircles model; half of them are published as a 0.5 x 0.3 m rectangle, half as a 4 x 1 m polygon.
tebgpu_fleet_obstacles_shaped_device under TEB_FLEET_SELECT_CENTRES and TEB_FLEET_SELECT_FOOTPRINTS, each under all
pairs and under the grid, the two rules alternating on one stream; CUDA events around each call, the median of --reps
after 3 warm-up calls. Also the rows each rule writes, and how many (scene, row) slots differ between the two rules.

    python tools/fleet_reach.py --step 1024 8192 32768 [--json out.json]

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
from tools.fleet_shapes import MAX_ROWS, RECT, c3_params  # noqa: E402
from tools.local_plan import card  # noqa: E402

LONG = [(abi.TEB_OBST_POLYGON, [[2.0, 0.5], [-2.0, 0.5], [-2.0, -0.5], [2.0, -0.5]])]


def step_times(R, reps, torch):
    dev = torch.device("cuda:0")
    g = T.TebGpu(R, 8, R, 64)
    g.set_params(c3_params())
    pose, cmd, _ = fleet(R)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    kinds = [RECT, LONG]
    kind = t((np.arange(R) % 2).astype(np.int32))
    C_cap, PV = MAX_ROWS, 4 * MAX_ROWS
    tp, tc = t(pose), t(cmd)                      # held: the args keep only their addresses
    outs = {}
    for sel in (abi.TEB_FLEET_SELECT_CENTRES, abi.TEB_FLEET_SELECT_FOOTPRINTS):
        custom = torch.zeros(R * C_cap * 64, dtype=torch.uint8, device=dev)
        cv = torch.zeros((R, PV, 2), dtype=torch.float64, device=dev)
        cc, need, st = (torch.zeros(R, dtype=torch.int32, device=dev) for _ in range(3))
        fa = abi.make_fleet_args(R, R, C_cap, MAX_ROWS, RANGE, pose=tp, last_cmd=tc, custom=custom, custom_count=cc,
                                 needed=need, status=st)
        outs[sel] = dict(fa=fa, sh=abi.make_fleet_shapes(kinds, PV, sel, kind=kind, custom_vertices=cv), custom=custom,
                         cc=cc, need=need, st=st)
    s = torch.cuda.Stream()
    res = {}
    for mode, name in ((abi.TEBGPU_FLEET_SEARCH_ALL_PAIRS, "all_pairs"), (abi.TEBGPU_FLEET_SEARCH_GRID, "grid")):
        g.set_fleet_search(mode)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ms = {abi.TEB_FLEET_SELECT_CENTRES: [], abi.TEB_FLEET_SELECT_FOOTPRINTS: []}
        for r in range(reps + 3):
            ev[0].record(s)
            o = outs[abi.TEB_FLEET_SELECT_CENTRES]
            g.fleet_obstacles_shaped_device(o["fa"], o["sh"], stream=s.cuda_stream)
            ev[1].record(s)
            o = outs[abi.TEB_FLEET_SELECT_FOOTPRINTS]
            g.fleet_obstacles_shaped_device(o["fa"], o["sh"], stream=s.cuda_stream)
            ev[2].record(s)
            torch.cuda.synchronize()
            if r >= 3:
                ms[abi.TEB_FLEET_SELECT_CENTRES].append(ev[0].elapsed_time(ev[1]))
                ms[abi.TEB_FLEET_SELECT_FOOTPRINTS].append(ev[1].elapsed_time(ev[2]))
        c, f = outs[abi.TEB_FLEET_SELECT_CENTRES], outs[abi.TEB_FLEET_SELECT_FOOTPRINTS]
        rows_c = c["custom"].view(R, C_cap, 64)
        rows_f = f["custom"].view(R, C_cap, 64)
        slot = torch.arange(C_cap, device=dev)[None, :]
        used = (slot < torch.maximum(c["cc"], f["cc"])[:, None])
        differ = used & ((rows_c != rows_f).any(-1) | (slot >= c["cc"][:, None]) | (slot >= f["cc"][:, None]))
        res[name] = dict(centres_ms=float(np.median(ms[abi.TEB_FLEET_SELECT_CENTRES])),
                         footprints_ms=float(np.median(ms[abi.TEB_FLEET_SELECT_FOOTPRINTS])),
                         centres_rows=int(c["cc"].sum()), footprints_rows=int(f["cc"].sum()),
                         centres_needed=int(c["need"].sum()), footprints_needed=int(f["need"].sum()),
                         rows_differ=int(differ.sum()), robots_differ=int(differ.any(1).sum()))
    g.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--step", type=int, nargs="+", default=[1024, 8192, 32768])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    res = dict(card=card(), range_m=RANGE, max_rows=MAX_ROWS, step={})
    for R in a.step:
        res["step"][str(R)] = step_times(R, a.reps, torch)
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
