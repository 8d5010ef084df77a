"""k_solve_tpb per launch in each form (factor streamed through HBM, or recomputed in segments of C rows), alternated in
one process: python tools/solve_forms.py [--widths 2 4 6] [--forms 1 11 22 33] [--reps 3] [--calls 10]

C3 at 8192 bands (32 candidates x 256 requests), one LM iteration per optimize call, so that every round-0 launch
solves all bands at the fixed width K. CUDA events around every launch (the library's profiling pass). For each width
the forms run in turn, `reps` times, `calls` calls each; prints one JSON line with the median and spread (max - min) of
the per-launch time per (K, form), the card, its power limit and SM clock, and checks that every form left the same
costs."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", type=int, nargs="+", default=[2, 4, 6])
    ap.add_argument("--forms", type=int, nargs="+", default=[1, 11, 22, 33])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--requests", type=int, default=256)
    a = ap.parse_args()
    n, M, cand, inflated, moving, via_pts = scenes.CONFIG_SHAPES["C3"]
    p = scenes.config_params("C3")
    p.teb_autosize = 0
    hb = scenes.make_batch(n, M, 32, a.requests, seed=1000, inflated=inflated, moving=moving, via_points=via_pts)
    args = abi.make_args(1, 1, True, p.selection_obst_cost_scale, p.selection_viapoint_cost_scale, False)
    g = T.TebGpu(hb.B, hb.n_cap, hb.S, max(hb.M_cap, 1), hb.V_cap)
    g.set_params(p)
    info_before = gpu_info()
    result = {"workload": "C3", "bands": hb.B, "gpu": info_before, "ms_per_launch": {}}
    for K in a.widths:
        g.set_speculation(K)
        times = {f: [] for f in a.forms}
        costs = {}
        for f in a.forms:   # warm-up of every form at this width
            g.set_solve_form(f)
            h = hb.copy(); g.optimize(h, args)
        for _ in range(a.reps):
            for f in a.forms:
                g.set_solve_form(f)
                g.set_profiling(True)
                for _ in range(a.calls):
                    h = hb.copy(); g.optimize(h, args)
                ms, cnt = g.kernel_times()["k_solve_tpb"]
                g.set_profiling(False)
                times[f].append(ms / cnt)
                costs[f] = h.cost.copy()
        for f in a.forms:
            assert np.array_equal(costs[f], costs[a.forms[0]], equal_nan=True), f"K {K}: form {f} changed the costs"
        result["ms_per_launch"][str(K)] = {str(f): {"median": float(np.median(v)), "spread": float(np.ptp(v)), "runs": v}
                                           for f, v in times.items()}
    result["gpu_after"] = gpu_info()
    print(json.dumps(result))
    g.close()


if __name__ == "__main__":
    main()
