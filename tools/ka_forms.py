"""Kernel A alone, form against form: python tools/ka_forms.py [runs] [label=path/to/libteb_b200.so[:ENV=VAL,...]] ...

C3 at 8192 bands (32 candidates x 256 requests, autoResize off), outer iteration 1: every form runs
tebgpu_build_system (graph build + kernel A, no read-back) with the library's CUDA-event profiling on and reports
kernel A's mean time per launch over 5 calls. The input is the same for every call and every form, so a throw-away form
whose outputs mean nothing still linearises the same bands. The forms are alternated in one process, each run creating
its context afresh (one warm-up call first); the median and spread over the runs go out as one JSON line, with the
card, its power limit and SM clock read in the same process.

Built-in forms: "persistent" (the library as built) and "oneshot" (the same library with TEBGPU_KA_PERSIST=0).
Further forms name another build of the library; the environment settings after ':' apply while its context is
created."""
import ctypes as C, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import teb_local_planner_b200 as T
from teb_local_planner_b200 import scenes

runs = int(sys.argv[1]) if len(sys.argv) > 1 else 3
forms = [("persistent", T.LIB_PATH, {}), ("oneshot", T.LIB_PATH, {"TEBGPU_KA_PERSIST": "0"})]
for a in sys.argv[2:]:
    label, spec = a.split("=", 1)
    path, _, envs = spec.partition(":")
    forms.append((label, os.path.abspath(path), dict(e.split("=", 1) for e in envs.split(",") if e)))

n, M, cand, inflated, moving, via_pts = scenes.CONFIG_SHAPES["C3"]
p = scenes.config_params("C3")
p.teb_autosize = 0
hb = scenes.make_batch(n, M, 32, 256, seed=1000, inflated=inflated, moving=moving, via_points=via_pts)
libs = {}


def context(path, env):
    if path not in libs:
        T._lib, T.LIB_PATH = None, path
        libs[path] = T.load_library()
    T._lib = libs[path]
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        g = T.TebGpu(hb.B, hb.n_cap, hb.S, max(hb.M_cap, 1), hb.V_cap)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v
    g.set_params(p)
    return g


times = {f[0]: [] for f in forms}
info = {}
for r in range(runs):
    for label, path, env in forms:
        g = context(path, env)
        bs = hb.struct()
        g._check(g.lib.tebgpu_build_system(g.ctx, C.byref(bs), 1, None, None, 0), "warm-up")
        g.set_profiling(True)
        for _ in range(5):
            g._check(g.lib.tebgpu_build_system(g.ctx, C.byref(bs), 1, None, None, 0), "tebgpu_build_system")
        ms, cnt = g.kernel_times()["k_linearize"]
        times[label].append(ms / cnt)
        info[label] = dict(zip(("build", "grid"), g.last_linearize()))
        g.close()
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
print(json.dumps({"workload": "C3", "bands": hb.B, "runs": runs, "gpu": smi,
                  "ms_per_launch": {k: {"median": float(np.median(v)), "spread": float(np.max(v) - np.min(v)), "all": v,
                                        **info[k]} for k, v in times.items()}}))
