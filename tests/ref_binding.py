"""ctypes binding of oracle/_ref/libteb_ref.so — the REFERENCE'S OWN sources (src/optimal_planner.cpp,
src/timed_elastic_band.cpp, src/obstacles.cpp and the headers they include) compiled against the shims in
oracle/ref_shims/ (Eigen / boost / ROS message stand-ins and a restated g2o optimizer). TEST INFRASTRUCTURE: it pins the
oracle restatement; nothing in the product may load it.

The library can only be built where the reference sources are (`make -C oracle ref`, also done by
__graft_entry__.build()). Everywhere else each call is answered from tests/golden/golden_ref_calls_v1.npz: what the
library returned for exactly the same inputs (keyed by a hash of them), recorded by tests/golden/make_golden_ref_calls.py.
Arrays the tests compare bit for bit are stored as SHA-256 digests (`Digest`, compared with `same`); values compared
with a tolerance are stored in full, the planner's final bands in fixed point (see storage_error)."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

from teb_local_planner_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libteb_ref.so")
REFERENCE_TREE = "/root/reference"
GOLDEN_CALLS = os.path.join(ROOT, "tests", "golden", "golden_ref_calls_v1.npz")
QUANTUM = 2.0 ** -20    # fixed-point step of the recorded arrays that are compared with a tolerance of 1e-5

_lib = None
_live = None
_replay = None
_recording = None


def build_ref():
    if os.path.isdir(REFERENCE_TREE):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "ref"])
    return REF_SO


def live():
    """True where the reference library itself answers (built here, or built elsewhere and copied along)"""
    global _live
    if _live is None:
        try:
            build_ref()
        except Exception:
            pass
        _live = os.path.exists(REF_SO)
    return _live


def available():
    return live() or os.path.exists(GOLDEN_CALLS)


# ----------------------------------------------------------------------------------------------- recorded calls
class Digest:
    """An array the reference returned, known by its shape and the SHA-256 of its values"""

    def __init__(self, shape, sha):
        self.shape, self.sha = tuple(int(d) for d in shape), bytes(sha)

    def __len__(self):
        return self.shape[0]


def _sha(a):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float64) + 0.0)   # + 0.0: -0.0 hashes as 0.0, as np.array_equal treats it
    return hashlib.sha256(a.tobytes()).digest()[:8]


def same(mine, ref):
    """np.array_equal of an array with a reference array or with its Digest"""
    if isinstance(ref, Digest):
        mine = np.asarray(mine)
        return mine.shape == ref.shape and _sha(mine) == ref.sha
    return np.array_equal(mine, ref)


def storage_error():
    """bound on |recorded - returned| of the fixed-point arrays (0 where the library itself answers)"""
    return 0.0 if live() else QUANTUM / 2


def _key(name, inputs):
    h = hashlib.sha256(name.encode())
    for x in inputs:
        if isinstance(x, np.ndarray):
            x = np.ascontiguousarray(x)
            h.update(f"{x.dtype.str}{x.shape}".encode())
            h.update(x.tobytes())
        elif isinstance(x, (C.Structure, C.Array)):
            h.update(C.string_at(C.addressof(x), C.sizeof(x)))
        elif isinstance(x, (bool, np.bool_)):
            h.update(repr(bool(x)).encode())
        elif isinstance(x, (int, np.integer)):
            h.update(repr(int(x)).encode())
        elif isinstance(x, (float, np.floating)):
            h.update(repr(float(x)).encode())
        else:
            h.update(repr(x).encode())
        h.update(b"|")
    return h.digest()[:8]


def _call(name, inputs, compute, digest=(), fixed=()):
    """compute() -> tuple of the library's outputs; without the library the recorded outputs for the same inputs come
    back instead: Digest at the positions in `digest`, fixed-point arrays at `fixed`, float64 arrays elsewhere"""
    key = _key(name, inputs)
    if live():
        out = tuple(compute())
        if _recording is not None:
            _recording[key] = [(np.shape(x), _sha(x)) if i in digest else (np.shape(x), _to_fixed(x)) if i in fixed else
                               np.asarray(x, np.float64) for i, x in enumerate(out)]
        return out
    global _replay
    if _replay is None:
        _replay = _load(GOLDEN_CALLS)
    if key not in _replay:
        raise KeyError(f"{name}: no recorded reference call with these inputs in {os.path.basename(GOLDEN_CALLS)} "
                       "(inputs changed? re-record with tests/golden/make_golden_ref_calls.py)")
    return _replay[key]


def recorded(name, inputs, compute):
    """a whole computation over the reference library, every output kept as a Digest"""
    if not live():
        return _call(name, inputs, None)
    out = tuple(compute())
    return _call(name, inputs, lambda: out, digest=range(len(out)))


def _to_fixed(a):
    """int32 multiples of QUANTUM, each element stored as its difference to the element 4 places earlier (the same column
    of the previous pose), which keeps the numbers small"""
    q = np.round(np.asarray(a, np.float64).reshape(-1) / QUANTUM).astype(np.int64)
    d = q.copy()
    d[4:] -= q[:-4]
    assert np.abs(d).max(initial=0) < 2 ** 31
    return d.astype(np.int32)


def _from_fixed(d, shape):
    q = np.zeros(len(d), np.int64)
    for r in range(4):
        q[r::4] = np.cumsum(d[r::4].astype(np.int64))
    return (q * QUANTUM).reshape(shape)


def start_recording():
    global _recording
    _recording = {}


def save_recording(path):
    """keys [C][8], items per call first[C+1]; per item kind (0 float64, 1 fixed point, 2 digest), shape, offset into the pool"""
    keys, first, kind, ndim, shape, pos = [], [0], [], [], [], []
    pools = {0: [], 1: [], 2: []}
    sizes = {0: 0, 1: 0, 2: 0}
    for key, items in _recording.items():
        keys.append(np.frombuffer(key, np.uint8))
        for it in items:
            if isinstance(it, np.ndarray):
                k, shp, val = 0, it.shape, it.reshape(-1)
            elif isinstance(it[1], bytes):
                k, shp, val = 2, it[0], np.frombuffer(it[1], np.uint8)[None]
            else:
                k, shp, val = 1, it[0], it[1]
            kind.append(k)
            ndim.append(len(shp))
            shape.append(list(shp) + [0] * (3 - len(shp)))
            pos.append(sizes[k])
            pools[k].append(val)
            sizes[k] += len(val)
        first.append(len(kind))
    np.savez_compressed(path, keys=np.array(keys, np.uint8), first=np.array(first, np.int64), kind=np.array(kind, np.int8),
                        ndim=np.array(ndim, np.int8), shape=np.array(shape, np.int64), pos=np.array(pos, np.int64),
                        f64=np.concatenate(pools[0] or [np.zeros(0)]),
                        fixed=np.concatenate(pools[1] or [np.zeros(0, np.int32)]).astype(np.int32),
                        dig=np.concatenate(pools[2] or [np.zeros((0, 8), np.uint8)]).reshape(-1, 8))


def _load(path):
    z = np.load(path, allow_pickle=False)
    f64, fixed = z["f64"], z["fixed"]
    kinds, ndims, shapes, poss, first, dig = z["kind"], z["ndim"], z["shape"], z["pos"], z["first"], z["dig"]
    out = {}
    for c, key in enumerate(z["keys"]):
        items = []
        for i in range(first[c], first[c + 1]):
            k, shp, p = int(kinds[i]), tuple(int(d) for d in shapes[i][:ndims[i]]), int(poss[i])
            size = int(np.prod(shp, dtype=np.int64))
            if k == 2:
                items.append(Digest(shp, dig[p].tobytes()))
            elif k == 1:
                items.append(_from_fixed(fixed[p:p + size], shp))
            else:
                items.append(f64[p:p + size].reshape(shp))
        out[key.tobytes()] = tuple(items)
    return out


def add_recording(path):
    """answer calls from the recording at `path` as well, where the library itself does not answer"""
    global _replay
    if live():
        return
    if _replay is None:
        _replay = _load(GOLDEN_CALLS) if os.path.exists(GOLDEN_CALLS) else {}
    _replay.update(_load(path))


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError("oracle/_ref/libteb_ref.so is missing (it can only be built where /root/reference exists)")
        L = C.CDLL(REF_SO)
        vp, d, i = C.c_void_p, C.c_double, C.c_int32
        L.teb_ref_abi.restype = i
        L.teb_ref_default_params.restype = None
        L.teb_ref_default_params.argtypes = [C.POINTER(abi.TebParams)]
        L.teb_ref_penalty.restype = d
        L.teb_ref_penalty.argtypes = [i, d, d, d, d]
        L.teb_ref_fast_sigmoid.restype = d
        L.teb_ref_fast_sigmoid.argtypes = [d]
        L.teb_ref_distance.restype = d
        L.teb_ref_distance.argtypes = [vp, vp, vp, vp, d]
        L.teb_ref_auto_resize.restype = i
        L.teb_ref_auto_resize.argtypes = [vp, i, i, d, d, i, i, i]
        L.teb_ref_init_trajectory.restype = i
        L.teb_ref_init_trajectory.argtypes = [vp, vp, d, d, i, i, vp, i]
        L.teb_ref_update_and_prune.restype = i
        L.teb_ref_update_and_prune.argtypes = [vp, i, i, vp, vp, i]
        L.teb_ref_optimize.restype = i
        L.teb_ref_optimize.argtypes = [vp, vp, C.POINTER(i), i, vp, i, vp, vp, i, vp, vp, i, vp, C.POINTER(d), vp]
        L.teb_ref_compute_cost.restype = d
        L.teb_ref_compute_cost.argtypes = [vp, vp, i, vp, i, vp, vp, i, vp, vp, i, vp]
        L.teb_ref_build_system.restype = i
        L.teb_ref_build_system.argtypes = [vp, vp, i, vp, i, vp, vp, i, vp, vp, i, d, vp, vp, C.POINTER(d), vp, i, C.POINTER(i)]
        L.teb_ref_optimize_batch.restype = i
        L.teb_ref_optimize_batch.argtypes = [vp, vp, vp, i, i]
        L.teb_ref_h_signature.restype = i
        L.teb_ref_h_signature.argtypes = [vp, vp, i, vp, i, vp, i, vp, vp]
        L.teb_ref_hcp_explore.restype = i
        L.teb_ref_hcp_explore.argtypes = [vp, vp, vp, vp, vp, i, vp, i, vp, i, vp, i]
        L.teb_ref_hcp_plan.restype = i
        L.teb_ref_hcp_plan.argtypes = [vp, vp, vp, vp, vp, i, vp, i, vp, i, vp, i]
        L.teb_ref_band_op.restype = i
        L.teb_ref_band_op.argtypes = [i, vp, i, vp, i, vp, i]
        assert L.teb_ref_abi() == 6
        _lib = L
    return _lib


def _common(obstacles, via, vel_start, vel_goal, obst_vertices):
    ob = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    v = np.zeros((0, 2)) if via is None else np.ascontiguousarray(via, dtype=np.float64).reshape(-1, 2)
    vs = np.array([0, 0, 0, 1.0]) if vel_start is None else np.ascontiguousarray(vel_start, dtype=np.float64)
    vg = np.array([0, 0, 0, 1.0]) if vel_goal is None else np.ascontiguousarray(vel_goal, dtype=np.float64)
    pv = None if obst_vertices is None or len(obst_vertices) == 0 else np.ascontiguousarray(obst_vertices, dtype=np.float64).reshape(-1, 2)
    return ob, v, vs, vg, pv


def default_params():
    def compute():
        p = abi.TebParams()
        lib().teb_ref_default_params(C.byref(p))
        return (np.frombuffer(C.string_at(C.addressof(p), C.sizeof(p)), np.uint8),)
    raw, = _call("default_params", (), compute)
    return abi.TebParams.from_buffer_copy(np.asarray(raw, np.uint8).tobytes())


def penalties(calls):
    """penalty functions of penalties.h: calls = [(which, var, a, b, eps)] (which: 0 interval, 1 interval2, 2 below)"""
    calls = np.ascontiguousarray(calls, dtype=np.float64).reshape(-1, 5)
    return _call("penalties", (calls,), lambda: (np.array([lib().teb_ref_penalty(int(w), v, a, b, e) for w, v, a, b, e in calls]),),
                 digest=(0,))[0]


def distances(params, poses, obstacles, obst_vertices=None, ts=None):
    """calculateDistance (t < 0) / estimateSpatioTemporalDistance (t >= 0) of the configured footprint: pose q to
    obstacle q for every row q"""
    poses = np.ascontiguousarray(poses, dtype=np.float64).reshape(-1, 3)
    ob = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE).reshape(-1)
    pv = None if obst_vertices is None else np.ascontiguousarray(obst_vertices, dtype=np.float64).reshape(-1, 2)
    ts = np.ascontiguousarray(ts, dtype=np.float64)

    def compute():
        return (np.array([lib().teb_ref_distance(C.addressof(params), poses[q].ctypes.data, ob[q:q + 1].ctypes.data,
                                                 pv.ctypes.data if pv is not None else None, float(ts[q])) for q in range(len(ts))]),)
    return _call("distances", (params, poses, ob, pv, ts), compute)[0]


def auto_resize(rec, n, dt_ref, dt_hyst, min_samples, max_samples, fast_mode, n_cap=None):
    n_cap = max(rec.shape[0], 4 * n) if n_cap is None else n_cap
    buf = np.zeros((n_cap, 4))
    buf[:n] = rec[:n]
    inputs = (buf, n, n_cap, dt_ref, dt_hyst, min_samples, max_samples, int(fast_mode))

    def compute():
        nn = lib().teb_ref_auto_resize(buf.ctypes.data, n, n_cap, dt_ref, dt_hyst, min_samples, max_samples, int(fast_mode))
        if nn < 0:
            raise RuntimeError("teb_ref_auto_resize: capacity")
        return (buf[:nn].copy(),)
    return _call("auto_resize", inputs, compute, digest=(0,))[0]


def init_trajectory(start, goal, diststep, max_vel_x, min_samples, backwards=False, n_cap=256):
    buf = np.zeros((n_cap, 4))
    s, g = np.ascontiguousarray(start, dtype=np.float64), np.ascontiguousarray(goal, dtype=np.float64)

    def compute():
        n = lib().teb_ref_init_trajectory(s.ctypes.data, g.ctypes.data, diststep, max_vel_x, min_samples, int(backwards), buf.ctypes.data, n_cap)
        if n < 0:
            raise RuntimeError("teb_ref_init_trajectory: capacity")
        return (buf[:n].copy(),)
    return _call("init_trajectory", (s, g, diststep, max_vel_x, min_samples, int(backwards), n_cap), compute, digest=(0,))[0]


def update_and_prune(rec, n, new_start, new_goal, min_samples=3):
    buf = np.ascontiguousarray(rec[:n], dtype=np.float64).copy()
    s, g = np.ascontiguousarray(new_start, dtype=np.float64), np.ascontiguousarray(new_goal, dtype=np.float64)
    nn = lib().teb_ref_update_and_prune(buf.ctypes.data, n, n, s.ctypes.data, g.ctypes.data, min_samples)
    return buf[:nn].copy()


def optimize_band(params, rec, n, obstacles, via=None, vel_start=None, vel_goal=None, rotdir=0, args=None, n_cap=None,
                  obst_vertices=None):
    """TebOptimalPlanner::optimizeTEB of the reference on one band. Returns (rec[n_new], cost, stats dict, ok)."""
    n_cap = rec.shape[0] if n_cap is None else n_cap
    buf = np.zeros((n_cap, 4))
    buf[:n] = rec[:n]
    ob, v, vs, vg, pv = _common(obstacles, via, vel_start, vel_goal, obst_vertices)
    args = abi.make_args(params.no_inner_iterations, params.no_outer_iterations) if args is None else args

    def compute():
        nn = C.c_int32(n)
        cost = C.c_double(np.inf)
        st = np.zeros(6)
        rc = lib().teb_ref_optimize(C.addressof(params), buf.ctypes.data, C.byref(nn), n_cap, ob.ctypes.data if len(ob) else None, len(ob),
                                    pv.ctypes.data if pv is not None else None, v.ctypes.data if len(v) else None, len(v),
                                    vs.ctypes.data, vg.ctypes.data, int(rotdir), C.addressof(args), C.byref(cost), st.ctypes.data)
        if rc < 0:
            raise RuntimeError("teb_ref_optimize: capacity")
        return buf[:nn.value].copy(), cost.value, st, rc
    band, cost, st, rc = _call("optimize_band", (params, buf, n, n_cap, ob, pv, v, vs, vg, int(rotdir), args), compute, digest=(0,))
    stats = {"lm_trials": int(st[0]), "rejected": int(st[1]), "terminated": bool(st[2]), "chol_failed": bool(st[3]),
             "diverged": bool(st[4]), "optimized": bool(st[5])}
    return band, float(cost), stats, bool(rc)


def optimize_batch(params, hb, args, threads=1, pin=False):
    """In-place on the HostBatch arrays: one band at a time per host thread (the reference's optimizeAllTEBs model)."""
    bs = hb.struct()
    rc = lib().teb_ref_optimize_batch(C.addressof(params), C.addressof(bs), C.addressof(args), int(threads), int(bool(pin)))
    if rc != 0:
        raise RuntimeError(f"teb_ref_optimize_batch rc={rc}")
    return hb


def compute_cost(params, rec, n, obstacles, via=None, vel_start=None, vel_goal=None, rotdir=0, args=None, obst_vertices=None):
    rec = np.ascontiguousarray(rec[:n], dtype=np.float64)
    ob, v, vs, vg, pv = _common(obstacles, via, vel_start, vel_goal, obst_vertices)
    args = abi.make_args() if args is None else args

    def compute():
        return (lib().teb_ref_compute_cost(C.addressof(params), rec.ctypes.data, n, ob.ctypes.data if len(ob) else None, len(ob),
                                           pv.ctypes.data if pv is not None else None, v.ctypes.data if len(v) else None, len(v),
                                           vs.ctypes.data, vg.ctypes.data, int(rotdir), C.addressof(args)),)
    return float(_call("compute_cost", (params, rec, n, ob, pv, v, vs, vg, int(rotdir), args), compute)[0])


def build_system(params, rec, n, obstacles, via=None, vel_start=None, vel_goal=None, rotdir=0, weight_multiplier=1.0,
                 obst_vertices=None, want_edges=False):
    """buildGraph + buildSystem of the reference: dense (H, b, chi2) in g2o order (N = 4n - 7) [+ per-edge rows]."""
    N0 = 4 * n - 7
    rec = np.ascontiguousarray(rec[:n], dtype=np.float64)
    ob, v, vs, vg, pv = _common(obstacles, via, vel_start, vel_goal, obst_vertices)
    max_edges = 64 * n + 4 * n * max(len(ob), 1) if want_edges else 0

    def compute():
        H = np.zeros((N0, N0))
        b = np.zeros(N0)
        chi2 = C.c_double(0)
        edges = np.zeros((max_edges, 64)) if want_edges else None
        ne = C.c_int32(0)
        N = lib().teb_ref_build_system(C.addressof(params), rec.ctypes.data, n, ob.ctypes.data if len(ob) else None, len(ob),
                                       pv.ctypes.data if pv is not None else None, v.ctypes.data if len(v) else None, len(v),
                                       vs.ctypes.data, vg.ctypes.data, int(rotdir), float(weight_multiplier), H.ctypes.data,
                                       b.ctypes.data, C.byref(chi2), edges.ctypes.data if want_edges else None, max_edges, C.byref(ne))
        if N != N0:
            raise RuntimeError(f"teb_ref_build_system: N = {N}, expected {N0}")
        return (H, b, chi2.value) + ((edges[:ne.value],) if want_edges else ())
    out = _call("build_system", (params, rec, n, ob, pv, v, vs, vg, int(rotdir), float(weight_multiplier), bool(want_edges)),
                compute, digest=(0, 1, 3))
    return (out[0], out[1], float(out[2])) + ((out[3],) if want_edges else ())


def h_signature(params, rec, n, obstacles, use_timediffs=True, obst_vertices=None):
    """calculateEquivalenceClass by the reference's own h_signature.h: complex H (2-D) or M values (x-y-t), plus
    (isValid, isReasonable)"""
    rec = np.ascontiguousarray(rec[:n], dtype=np.float64)
    ob = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    pv = None if obst_vertices is None or len(obst_vertices) == 0 else np.ascontiguousarray(obst_vertices, dtype=np.float64).reshape(-1, 2)

    def compute():
        out = np.zeros(max(2, len(ob)))
        flags = np.zeros(2, np.int32)
        rc = lib().teb_ref_h_signature(C.addressof(params), rec.ctypes.data, n, ob.ctypes.data if len(ob) else None, len(ob),
                                       pv.ctypes.data if pv is not None else None, int(use_timediffs), out.ctypes.data, flags.ctypes.data)
        if rc != 0:
            raise RuntimeError(f"teb_ref_h_signature rc={rc}")
        return out, flags
    out, flags = _call("h_signature", (params, rec, n, ob, pv, int(use_timediffs)), compute)
    val = out[:len(ob)].copy() if params.include_dynamic_obstacles else complex(out[0], out[1])
    return val, bool(flags[0]), bool(flags[1])


def hcp_explore(params, hcp, start, goal, obstacles, obst_vertices=None, cycles=1, prm=False):
    """exploreEquivalenceClassesAndInitTebs of the reference's HomotopyClassPlanner on a fresh planner (clearPlanner()
    between cycles). hcp: dict with max_number_classes, obstacle_heading_threshold and, for the roadmap, area width /
    length scale / number of samples. Returns a list (per cycle) of lists of candidate bands [n][4]."""
    ob = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    pv = None if obst_vertices is None or len(obst_vertices) == 0 else np.ascontiguousarray(obst_vertices, dtype=np.float64).reshape(-1, 2)
    h = np.array([hcp["max_number_classes"], hcp["obstacle_heading_threshold"], hcp.get("roadmap_graph_area_width", 6.0),
                  hcp.get("roadmap_graph_area_length_scale", 1.0), hcp.get("roadmap_graph_no_samples", 15), 1.0 if prm else 0.0])
    s, g = np.ascontiguousarray(start, dtype=np.float64), np.ascontiguousarray(goal, dtype=np.float64)

    def compute():
        cap, ccap = 1 << 18, 4096
        out = np.zeros(cap)
        counts = np.zeros(ccap, np.int32)
        w = lib().teb_ref_hcp_explore(C.addressof(params), h.ctypes.data, s.ctypes.data, g.ctypes.data, ob.ctypes.data if len(ob) else None,
                                      len(ob), pv.ctypes.data if pv is not None else None, cycles, out.ctypes.data, cap, counts.ctypes.data, ccap)
        if w < 0:
            raise RuntimeError("teb_ref_hcp_explore: capacity")
        nb = int(counts[:cycles].sum())
        return out[:4 * int(counts[cycles:cycles + nb].sum())], counts[:cycles + nb]
    out, counts = _call("hcp_explore", (params, h, s, g, ob, pv, cycles), compute)
    res, ci, pos = [], cycles, 0
    for c in range(cycles):
        bands = []
        for _ in range(int(counts[c])):
            n = int(counts[ci]); ci += 1
            bands.append(out[pos:pos + 4 * n].reshape(n, 4).copy())
            pos += 4 * n
        res.append(bands)
    return res


def hcp_plan(params, hcp, starts, goal, obstacles, obst_vertices=None, prm=False):
    """consecutive HomotopyClassPlanner::plan(start_c, goal) calls on one reference planner. Returns per cycle
    (ok, best_index, [(cost, band[n][4]), ...]). Replayed bands are fixed point (see storage_error)."""
    ob = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    pv = None if obst_vertices is None or len(obst_vertices) == 0 else np.ascontiguousarray(obst_vertices, dtype=np.float64).reshape(-1, 2)
    h = np.array([hcp["max_number_classes"], hcp["obstacle_heading_threshold"], hcp.get("roadmap_graph_area_width", 6.0),
                  hcp.get("roadmap_graph_area_length_scale", 1.0), hcp.get("roadmap_graph_no_samples", 15), 1.0 if prm else 0.0])
    st = np.ascontiguousarray(starts, dtype=np.float64).reshape(-1, 3)
    g = np.ascontiguousarray(goal, dtype=np.float64)
    cycles = len(st)

    def compute():
        """-> costs, bands (flat), counts: the library writes (cost, band) per candidate into one buffer"""
        cap, ccap = 1 << 20, 1 << 14
        out = np.zeros(cap)
        counts = np.zeros(ccap, np.int32)
        w = lib().teb_ref_hcp_plan(C.addressof(params), h.ctypes.data, st.ctypes.data, g.ctypes.data, ob.ctypes.data if len(ob) else None,
                                   len(ob), pv.ctypes.data if pv is not None else None, cycles, out.ctypes.data, cap, counts.ctypes.data, ccap)
        if w < 0:
            raise RuntimeError("teb_ref_hcp_plan: capacity")
        nb = int(counts[0:3 * cycles:3].sum())
        costs, bands, pos = [], [], 0
        for n in counts[3 * cycles:3 * cycles + nb]:
            costs.append(out[pos])
            bands.append(out[pos + 1:pos + 1 + 4 * int(n)])
            pos += 1 + 4 * int(n)
        return np.array(costs), np.concatenate(bands) if bands else np.zeros(0), counts[:3 * cycles + nb]
    costs, bands, counts = _call("hcp_plan", (params, h, st, g, ob, pv), compute, fixed=(1,))
    res, ci, k, pos = [], 3 * cycles, 0, 0
    for c in range(cycles):
        cands = []
        for _ in range(int(counts[3 * c])):
            n = int(counts[ci]); ci += 1
            cands.append((float(costs[k]), bands[pos:pos + 4 * n].reshape(n, 4).copy()))
            k += 1
            pos += 4 * n
        res.append((bool(counts[3 * c + 2]), int(counts[3 * c + 1]), cands))
    return res


def band_op(op, rec, args, cap=8192):
    """teb_ref_band_op: one TimedElasticBand / TebOptimalPlanner operation of the reference (tests/test_host_pin.py)"""
    rec = None if rec is None else np.ascontiguousarray(rec, dtype=np.float64)
    a = np.ascontiguousarray(args, dtype=np.float64)

    def compute():
        out = np.full(cap, np.nan)
        k = lib().teb_ref_band_op(op, rec.ctypes.data if rec is not None else None, 0 if rec is None else len(rec), a.ctypes.data,
                                  len(a), out.ctypes.data, cap)
        assert k >= 0, (op, k)
        return (out[:k].copy(),)
    return _call("band_op", (op, rec, a, cap), compute, digest=(0,))[0]
