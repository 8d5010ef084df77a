"""Times costmap-like scenes (scenes.costmap_scene: walls and blobs of 5 cm cells as point obstacles, plus a few
circular, line and moving obstacles) on both obstacle-table paths: M = 64 and 1024 (staged: the table in shared
memory) and 1025, 4096, 16384 (global table, read from L2).
Two regimes: one 32-candidate request (latency regime, CUDA-graph replay) and a throughput batch of BANDS bands.
python tools/large_scenes.py [BANDS=2048] [REPS=3] -> one JSON line per (M, regime), then the card."""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import teb_local_planner_b200 as T
from teb_local_planner_b200 import abi, scenes

bands = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
for M in (64, 1024, 1025, 4096, 16384):
    for regime, B in (("latency_32", 32), ("throughput", bands)):
        p, hb = scenes.costmap_scene(M, n=100, candidates=B, seed=7)
        args = abi.make_args(p.no_inner_iterations, p.no_outer_iterations, True, p.selection_obst_cost_scale,
                             p.selection_viapoint_cost_scale, False)
        g = T.TebGpu(hb.B, hb.n_cap, hb.S, hb.M_cap, hb.V_cap, max_obst_vertices=hb.PV_cap)
        g.set_params(p)
        h = hb.copy(); g.optimize(h, args)     # warm-up (and graph capture in the latency regime)
        t0 = time.perf_counter()
        for _ in range(reps):
            h = hb.copy(); g.optimize(h, args)
        ms = (time.perf_counter() - t0) / reps * 1e3
        g.set_profiling(True)                  # separate, profiled pass: per-kernel CUDA-event times
        h = hb.copy(); g.optimize(h, args)
        kt = {k: round(v[0], 3) for k, v in g.kernel_times().items() if v[1]}
        g.close()
        print(json.dumps({"M": M, "path": "global" if M > 1024 else "staged", "regime": regime, "bands": B,
                          "ms_per_call": round(ms, 3), "kernel_ms_per_call": kt,
                          "optimized": int(np.sum(h.status & abi.TEB_STATUS_OPTIMIZED != 0)), "card": card}), flush=True)
