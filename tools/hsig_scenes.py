"""Times the scene H-signature entry points on one H100: the factor-table step (k_hsig_factors + k_hsig_factors_combine)
per scene and the 2-D signature step (k_hsig2d_scene + k_hsig2d_scene_sum) per band, at M = 1024, 4096 and 16384 rows
with B = 1, 32 and 1024 bands on one costmap scene (scenes.costmap_scene, 100 poses per band).

  * step times: CUDA events on the call's stream around 20 back-to-back calls, median of 7 such windows after a
    warm-up; each step is two launches, so a step time includes the second kernel and the gap between them;
  * share of the fp64 bound: the step's operations (DESIGN §6: per pair of the product 17 fp64 operations; per
    (pose, obstacle) hypot, log and atan2, counted as 60; per term 16) at the H100 SXM data sheet's non-tensor FP64
    rate of 34 TFLOP/s (the kernels use no tensor cores), over the step time;
  * at M = 1024: tebgpu_h_signature against the new entry with its factor table built in the same window, end to end
    (a host clock around 20 calls on the context's stream ending in a synchronise: tebgpu_h_signature takes no stream),
    on the costmap batch, and both outputs compared on a ring scene (tests/hsig_scene_cases.py) whose 32 candidates have
    finite, non-zero signatures in several classes.

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query)."""
import argparse
import json
import os
import statistics
import sys
import time

import ctypes as C

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi, scenes  # noqa: E402
from tools.local_plan import card  # noqa: E402
from tests import hsig_cases as hc  # noqa: E402
from tests import hsig_scene_cases as sc  # noqa: E402

FP64_PEAK = 34e12


def batch(M, B, n=100, seed=0):
    p, hb = scenes.costmap_scene(M, n=n, candidates=B, seed=seed, shapes=False)
    p.include_dynamic_obstacles = 0
    return p, hb


def device_batch(torch, hb):
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).to(dev)
    keep = [t(hb.poses), t(hb.n), t(hb.scene_id), t(hb.obstacles), t(hb.obst_count), t(hb.vel_start), t(hb.vel_goal)]
    bs = abi.TebBatch()
    bs.B, bs.n_cap, bs.S, bs.M_cap, bs.V_cap = hb.B, hb.n_cap, hb.S, hb.M_cap, 0
    bs.poses, bs.n, bs.scene_id, bs.obstacles, bs.obst_count, bs.vel_start, bs.vel_goal = (k.data_ptr() for k in keep)
    return bs, keep


def host_timed(g, fn, reps, calls=20):
    """ms per call: a host clock around `calls` back-to-back calls on the context's stream ending in a synchronise,
    median of `reps` such windows, after a warm-up window"""
    fn()
    g.synchronize()
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for _ in range(calls):
            fn()
        g.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0) / calls)
    return statistics.median(ms)


def event_timed(torch, s, fn, reps, calls=20):
    """ms per call: CUDA events on stream s around `calls` back-to-back calls issued to s, median of `reps` windows"""
    fn()
    s.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        for _ in range(calls):
            fn()
        b.record(s)
        b.synchronize()
        ms.append(a.elapsed_time(b) / calls)
    return statistics.median(ms)


def compare_entries(torch, reps):
    """tebgpu_h_signature and tebgpu_h_signature_scenes on one batch of 32 candidates around a 1024-row ring scene"""
    case = sc._ring(1024, seed=3)
    case.bands = hc.bundle((-3.0, -1.0), (3.0, 1.2), 40, list(np.linspace(-1.9, 1.9, 32)))
    hb, _ = hc.batch([case])
    p = case.params()
    g = T.TebGpu(hb.B, hb.n_cap, 1, hb.M_cap, 0)
    g.set_params(p)
    old, new = g.h_signature(hb), g.h_signature_scenes(hb)
    g.close()
    thr = p.h_signature_threshold
    return {"compare_scene": case.name, "compare_bands": hb.B, "max_abs_H": float(np.abs(old).max()),
            "max_abs_diff_old_new": float(np.abs(old - new).max()),
            "same_classes": hc.partition(list(old), 2, thr) == hc.partition(list(new), 2, thr),
            "classes": len({tuple(r) for r in hc.partition(list(new), 2, thr)})}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda:0")
    res = {"card": card(), "rows": []}
    for M in (1024, 4096, 16384):
        for B in (1, 32, 1024):
            p, hb = batch(M, B)
            g = T.TebGpu(B, hb.n_cap, 1, M, 0)
            g.set_params(p)
            bs, keep = device_batch(torch, hb)
            f = (torch.zeros(M * 2, dtype=torch.float64, device=dev), torch.zeros(M, dtype=torch.int32, device=dev),
                 torch.zeros(1, dtype=torch.int32, device=dev))
            fs = abi.make_hsig_factors(*(x.data_ptr() for x in f))
            out = torch.zeros((B, 2), dtype=torch.float64, device=dev)
            s = torch.cuda.Stream()
            st = s.cuda_stream
            t_f = event_timed(torch, s, lambda: g.hsig_factors_device(bs, fs, stream=st), a.reps)
            t_s = event_timed(torch, s, lambda: g.h_signature_scenes_device(bs, out, factors=fs, stream=st), a.reps)
            n = int(hb.n[0])
            pairs = M * (M - 1)
            fl_f, fl_s = 17.0 * pairs, B * (60.0 * n * M + 16.0 * (n - 1) * M + 30.0 * M)
            row = {"M": M, "B": B, "n": n, "factor_step_ms_per_scene": t_f, "signature_step_ms": t_s,
                   "signature_step_us_per_band": 1e3 * t_s / B,
                   "factor_step_share_fp64": fl_f / (t_f * 1e-3) / FP64_PEAK,
                   "signature_step_share_fp64": fl_s / (t_s * 1e-3) / FP64_PEAK}
            if M <= 1024:
                old = torch.zeros((B, 2), dtype=torch.float64, device=dev)
                t_o = host_timed(g, lambda: g._check(g.lib.tebgpu_h_signature(g.ctx, C.byref(bs), 1, old.data_ptr(), 1),
                                                     "tebgpu_h_signature"), a.reps)
                t_new = host_timed(g, lambda: (g.hsig_factors_device(bs, fs), g.h_signature_scenes_device(bs, out, factors=fs)),
                                   a.reps)
                row.update({"old_entry_end_to_end_ms": t_o, "new_entry_with_factors_end_to_end_ms": t_new})
            g.close()
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    res["compare"] = compare_entries(torch, a.reps)
    print(json.dumps(res["compare"]))
    print(json.dumps({"card": res["card"]}))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
