"""ctypes binding of oracle/libteb_oracle.so — TEST INFRASTRUCTURE (the checker, never the product)."""
import ctypes as C
import os
import subprocess

import numpy as np

from teb_local_planner_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_SO = os.path.join(ORACLE_DIR, "libteb_oracle.so")

JAC_G2O, JAC_ANALYTIC = 0, 1
SOLVER_BANDED, SOLVER_DENSE = 0, 1


class OracleOptions(C.Structure):
    _fields_ = [("jac_mode", C.c_int32), ("solver", C.c_int32), ("verbose", C.c_int32), ("pin_threads", C.c_int32)]


class OracleStats(C.Structure):
    _fields_ = [("chi2_final", C.c_double), ("lambda_final", C.c_double), ("lm_iters", C.c_int32),
                ("lm_trials", C.c_int32), ("rejected", C.c_int32), ("n_edges_last", C.c_int32),
                ("status", C.c_int32), ("n_final", C.c_int32), ("nu_final", C.c_double)]


def build_oracle():
    src = os.path.join(ORACLE_DIR, "teb_oracle.c")
    if (not os.path.exists(ORACLE_SO)) or os.path.getmtime(ORACLE_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-s"])
    return ORACLE_SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        # on the GPU box only the prebuilt .so travels; build when sources are newer (CPU container)
        try:
            build_oracle()
        except Exception:
            if not os.path.exists(ORACLE_SO):
                raise
        L = C.CDLL(ORACLE_SO)
        dp, ip, vp = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.c_void_p
        L.teb_oracle_optimize.restype = C.c_int32
        L.teb_oracle_optimize.argtypes = [C.POINTER(abi.TebParams), vp, ip, C.c_int32, vp, C.c_int32, vp, C.c_int32,
                                          vp, vp, C.c_int32, C.POINTER(abi.TebOptimizeArgs), C.POINTER(OracleOptions),
                                          dp, C.POINTER(OracleStats), vp]
        L.teb_oracle_optimize_batch.restype = C.c_int32
        L.teb_oracle_optimize_batch.argtypes = [C.POINTER(abi.TebParams), C.POINTER(abi.TebBatch),
                                                C.POINTER(abi.TebOptimizeArgs), C.POINTER(OracleOptions), C.c_int32]
        L.teb_oracle_build_system.restype = C.c_int32
        L.teb_oracle_build_system.argtypes = [C.POINTER(abi.TebParams), vp, C.c_int32, vp, C.c_int32, vp, C.c_int32,
                                              vp, vp, C.c_int32, C.c_double, C.c_int32, vp, vp, dp, vp]
        L.teb_oracle_auto_resize.restype = C.c_int32
        L.teb_oracle_auto_resize.argtypes = [vp, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_int32]
        L.teb_oracle_init_trajectory.restype = C.c_int32
        L.teb_oracle_init_trajectory.argtypes = [vp, vp, C.c_double, C.c_double, C.c_int32, C.c_int32, vp, C.c_int32]
        for f in ("teb_oracle_normalize_theta",):
            getattr(L, f).restype = C.c_double
            getattr(L, f).argtypes = [C.c_double]
        L.teb_oracle_average_angle.restype = C.c_double
        L.teb_oracle_average_angle.argtypes = [C.c_double, C.c_double]
        L.teb_oracle_penalty_interval.restype = C.c_double
        L.teb_oracle_penalty_interval.argtypes = [C.c_double] * 3
        L.teb_oracle_penalty_interval2.restype = C.c_double
        L.teb_oracle_penalty_interval2.argtypes = [C.c_double] * 4
        L.teb_oracle_penalty_below.restype = C.c_double
        L.teb_oracle_penalty_below.argtypes = [C.c_double] * 3
        _lib = L
    return _lib


def _verts(obst_vertices):
    if obst_vertices is None or len(obst_vertices) == 0:
        return None, None
    v = np.ascontiguousarray(obst_vertices, dtype=np.float64).reshape(-1, 2)
    return v, v.ctypes.data


def distance(params, pose, obstacle, obst_vertices=None, t=0.0, want_grad=False):
    """calculateDistance / estimateSpatioTemporalDistance of the configured footprint to one obstacle row"""
    L = lib()
    L.teb_oracle_distance.restype = C.c_double
    L.teb_oracle_distance.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p]
    pose = np.ascontiguousarray(pose, dtype=np.float64)
    ob = np.ascontiguousarray(obstacle, dtype=abi.OBST_DTYPE).reshape(1)
    v, vptr = _verts(obst_vertices)
    g = np.zeros(3)
    d = L.teb_oracle_distance(C.addressof(params), pose.ctypes.data, ob.ctypes.data, vptr, float(t),
                              g.ctypes.data if want_grad else None)
    return (d, g) if want_grad else d


def h_signature(params, rec, n, obstacles, use_timediffs=True):
    """calculateEquivalenceClass on one band: complex H (2-D) or an array of M values (x-y-t)"""
    L = lib()
    L.teb_oracle_h_signature.restype = C.c_int32
    L.teb_oracle_h_signature.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    rec = np.ascontiguousarray(rec[:n], dtype=np.float64)
    ob = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    out = np.zeros(max(2, len(ob)))
    rc = L.teb_oracle_h_signature(C.addressof(params), rec.ctypes.data, n, ob.ctypes.data if len(ob) else None, len(ob),
                                  int(use_timediffs), out.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"teb_oracle_h_signature rc={rc}")
    return out[:len(ob)].copy() if params.include_dynamic_obstacles else complex(out[0], out[1])


def optimize_band(params, rec, n, obstacles, via=None, vel_start=None, vel_goal=None, rotdir=0,
                  args=None, jac_mode=JAC_G2O, solver=SOLVER_BANDED, n_cap=None, obst_vertices=None):
    """One optimizeTEB on one band. Returns (rec[n_new], cost, stats)."""
    L = lib()
    n_cap = rec.shape[0] if n_cap is None else n_cap
    buf = np.zeros((n_cap, 4))
    buf[:n] = rec[:n]
    obstacles = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    via = np.zeros((0, 2)) if via is None else np.ascontiguousarray(via, dtype=np.float64)
    vs = np.array([0, 0, 0, 1.0]) if vel_start is None else np.ascontiguousarray(vel_start, dtype=np.float64)
    vg = np.array([0, 0, 0, 1.0]) if vel_goal is None else np.ascontiguousarray(vel_goal, dtype=np.float64)
    args = abi.make_args(params.no_inner_iterations, params.no_outer_iterations) if args is None else args
    opt = OracleOptions(jac_mode, solver, 0, 0)
    nn = C.c_int32(n)
    cost = C.c_double(np.inf)
    st = OracleStats()
    rc = L.teb_oracle_optimize(C.byref(params), buf.ctypes.data, C.byref(nn), n_cap,
                               obstacles.ctypes.data if len(obstacles) else None, len(obstacles),
                               via.ctypes.data if len(via) else None, len(via), vs.ctypes.data, vg.ctypes.data,
                               rotdir, C.byref(args), C.byref(opt), C.byref(cost), C.byref(st), _verts(obst_vertices)[1])
    if rc != 0:
        raise RuntimeError(f"teb_oracle_optimize rc={rc}")
    return buf[:nn.value].copy(), cost.value, st


def optimize_batch(params, hb, args, jac_mode=JAC_G2O, solver=SOLVER_BANDED, threads=1, pin=False):
    """In-place on the HostBatch arrays. pin: worker t runs on the t-th CPU of the affinity mask (timing runs)."""
    L = lib()
    opt = OracleOptions(jac_mode, solver, 0, int(bool(pin)))
    bs = hb.struct()
    rc = L.teb_oracle_optimize_batch(C.byref(params), C.byref(bs), C.byref(args), C.byref(opt), threads)
    if rc != 0:
        raise RuntimeError(f"teb_oracle_optimize_batch rc={rc}")
    return hb


def build_system(params, rec, n, obstacles, via=None, vel_start=None, vel_goal=None, rotdir=0,
                 weight_multiplier=1.0, jac_mode=JAC_G2O, obst_vertices=None):
    """Dense (H, b, chi2) of one band in g2o order (N = 4n-7)."""
    L = lib()
    N = 4 * n - 7
    H = np.zeros((N, N))
    b = np.zeros(N)
    chi2 = C.c_double(0)
    rec = np.ascontiguousarray(rec[:n], dtype=np.float64)
    obstacles = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    via = np.zeros((0, 2)) if via is None else np.ascontiguousarray(via, dtype=np.float64)
    vs = np.array([0, 0, 0, 1.0]) if vel_start is None else np.ascontiguousarray(vel_start, dtype=np.float64)
    vg = np.array([0, 0, 0, 1.0]) if vel_goal is None else np.ascontiguousarray(vel_goal, dtype=np.float64)
    rc = L.teb_oracle_build_system(C.byref(params), rec.ctypes.data, n,
                                   obstacles.ctypes.data if len(obstacles) else None, len(obstacles),
                                   via.ctypes.data if len(via) else None, len(via), vs.ctypes.data, vg.ctypes.data,
                                   rotdir, weight_multiplier, jac_mode, H.ctypes.data, b.ctypes.data, C.byref(chi2),
                                   _verts(obst_vertices)[1])
    if rc < 0:
        raise RuntimeError(f"teb_oracle_build_system rc={rc}")
    return H, b, chi2.value


def dump_edges(params, rec, n, obstacles, via=None, vel_start=None, vel_goal=None, rotdir=0, weight_multiplier=1.0,
               jac_mode=JAC_G2O, obst_vertices=None):
    """rows [n_edges][64] of the graph at this state (layout: oracle/teb_oracle.c teb_oracle_dump_edges)"""
    L = lib()
    L.teb_oracle_dump_edges.restype = C.c_int32
    L.teb_oracle_dump_edges.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.c_int32,
                                        C.c_void_p]
    rec = np.ascontiguousarray(rec[:n], dtype=np.float64)
    obstacles = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    via = np.zeros((0, 2)) if via is None else np.ascontiguousarray(via, dtype=np.float64)
    vs = np.array([0, 0, 0, 1.0]) if vel_start is None else np.ascontiguousarray(vel_start, dtype=np.float64)
    vg = np.array([0, 0, 0, 1.0]) if vel_goal is None else np.ascontiguousarray(vel_goal, dtype=np.float64)
    cap = 64 * n + 4 * n * max(len(obstacles), 1)
    rows = np.zeros((cap, 64))
    ne = L.teb_oracle_dump_edges(C.addressof(params), rec.ctypes.data, n, obstacles.ctypes.data if len(obstacles) else None,
                                 len(obstacles), via.ctypes.data if len(via) else None, len(via), vs.ctypes.data, vg.ctypes.data,
                                 int(rotdir), float(weight_multiplier), int(jac_mode), rows.ctypes.data, cap, _verts(obst_vertices)[1])
    if ne < 0:
        raise RuntimeError(f"teb_oracle_dump_edges rc={ne}")
    return rows[:ne]


def trial_chi2(params, rec_graph, n, trials, obstacles, via=None, vel_start=None, vel_goal=None, rotdir=0,
               weight_multiplier=1.0, obst_vertices=None):
    """chi2 by family (obstacles, via, time-optimal, other) [T][4] of the trial states trials [T][>= n][4], with the graph
    built at rec_graph (association, dynamic-obstacle times and via-points frozen there)"""
    L = lib()
    L.teb_oracle_trial_chi2.restype = C.c_int32
    L.teb_oracle_trial_chi2.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                        C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_void_p, C.c_int32, C.c_void_p,
                                        C.c_void_p]
    rec = np.ascontiguousarray(rec_graph[:n], dtype=np.float64)
    tr = np.ascontiguousarray(np.asarray(trials, dtype=np.float64)[:, :n])
    obstacles = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    via = np.zeros((0, 2)) if via is None else np.ascontiguousarray(via, dtype=np.float64)
    vs = np.array([0, 0, 0, 1.0]) if vel_start is None else np.ascontiguousarray(vel_start, dtype=np.float64)
    vg = np.array([0, 0, 0, 1.0]) if vel_goal is None else np.ascontiguousarray(vel_goal, dtype=np.float64)
    out = np.zeros((tr.shape[0], 4))
    rc = L.teb_oracle_trial_chi2(C.addressof(params), rec.ctypes.data, n, obstacles.ctypes.data if len(obstacles) else None,
                                 len(obstacles), via.ctypes.data if len(via) else None, len(via), vs.ctypes.data,
                                 vg.ctypes.data, int(rotdir), float(weight_multiplier), tr.ctypes.data, tr.shape[0],
                                 out.ctypes.data, _verts(obst_vertices)[1])
    if rc != 0:
        raise RuntimeError(f"teb_oracle_trial_chi2 rc={rc}")
    return out


def graph(params, rec, n, obstacles, via=None, vel_start=None, vel_goal=None, rotdir=0, weight_multiplier=1.0,
          obst_vertices=None, MW=None):
    """the structure buildGraph() gives the band (teb_oracle_graph) -> dict(assoc [n][MW] uint64, assoc3 [n][MW] uint64,
    via_idx [V] (-1: no edge), dyn_t [n] (NaN: no dynamic-obstacle edge on the pose))"""
    L = lib()
    L.teb_oracle_graph.restype = C.c_int32
    L.teb_oracle_graph.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                   C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_void_p]
    rec = np.ascontiguousarray(rec[:n], dtype=np.float64)
    obstacles = np.ascontiguousarray(obstacles, dtype=abi.OBST_DTYPE)
    via = np.zeros((0, 2)) if via is None else np.ascontiguousarray(via, dtype=np.float64)
    vs = np.array([0, 0, 0, 1.0]) if vel_start is None else np.ascontiguousarray(vel_start, dtype=np.float64)
    vg = np.array([0, 0, 0, 1.0]) if vel_goal is None else np.ascontiguousarray(vel_goal, dtype=np.float64)
    MW = max(1, (len(obstacles) + 63) // 64) if MW is None else MW
    out = dict(assoc=np.zeros((n, MW), np.uint64), assoc3=np.zeros((n, MW), np.uint64),
               via_idx=np.zeros(len(via), np.int32), dyn_t=np.zeros(n))
    rc = L.teb_oracle_graph(C.addressof(params), rec.ctypes.data, n, obstacles.ctypes.data if len(obstacles) else None,
                            len(obstacles), via.ctypes.data if len(via) else None, len(via), vs.ctypes.data, vg.ctypes.data,
                            int(rotdir), float(weight_multiplier), int(MW), out["assoc"].ctypes.data,
                            out["assoc3"].ctypes.data, out["via_idx"].ctypes.data, out["dyn_t"].ctypes.data,
                            _verts(obst_vertices)[1])
    if rc != 0:
        raise RuntimeError(f"teb_oracle_graph rc={rc}")
    return out


def lm_decide(current_chi, lam, nu, q0, temp_chi, scale_sum, ok):
    """g2o's accept / reject chain over a sequence of trials -> dict(accepted, used, terminate, status, need, q, lambda,
    nu, current_chi)"""
    L = lib()
    L.teb_oracle_lm_decide.restype = C.c_int32
    L.teb_oracle_lm_decide.argtypes = [C.c_double, C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p]
    tc = np.ascontiguousarray(temp_chi, dtype=np.float64)
    sc = np.ascontiguousarray(scale_sum, dtype=np.float64)
    okk = np.ascontiguousarray(ok, dtype=np.int32)
    oi = np.zeros(6, np.int32)
    od = np.zeros(3)
    rc = L.teb_oracle_lm_decide(float(current_chi), float(lam), float(nu), int(q0), tc.size, tc.ctypes.data, sc.ctypes.data,
                                okk.ctypes.data, oi.ctypes.data, od.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"teb_oracle_lm_decide rc={rc}")
    return dict(accepted=int(oi[0]), used=int(oi[1]), terminate=bool(oi[2]), status=int(oi[3]), need=bool(oi[4]),
                q=int(oi[5]), lam=float(od[0]), nu=float(od[1]), current_chi=float(od[2]))


def auto_resize(rec, n, dt_ref, dt_hyst, min_samples, max_samples, fast_mode, n_cap=None):
    L = lib()
    n_cap = max(rec.shape[0], 4 * n) if n_cap is None else n_cap
    buf = np.zeros((n_cap, 4))
    buf[:n] = rec[:n]
    nn = L.teb_oracle_auto_resize(buf.ctypes.data, n, n_cap, dt_ref, dt_hyst, min_samples, max_samples, int(fast_mode))
    if nn < 0:
        raise RuntimeError(f"auto_resize rc={nn}")
    return buf[:nn].copy()


def init_trajectory(start, goal, diststep, max_vel_x, min_samples, backwards=False, n_cap=64):
    L = lib()
    buf = np.zeros((n_cap, 4))
    s = np.ascontiguousarray(start, dtype=np.float64)
    g = np.ascontiguousarray(goal, dtype=np.float64)
    n = L.teb_oracle_init_trajectory(s.ctypes.data, g.ctypes.data, diststep, max_vel_x, min_samples, int(backwards),
                                     buf.ctypes.data, n_cap)
    if n < 0:
        raise RuntimeError(f"init_trajectory rc={n}")
    return buf[:n].copy()
