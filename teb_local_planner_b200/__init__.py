"""teb_local_planner_b200 — H100-native (sm_90a) batched Timed-Elastic-Band optimizer.

Python side: ctypes loader for the in-tree CUDA library (C-ABI in include/teb_b200.h) and a thin
`TebGpu` convenience wrapper used by tests and bench.py. There is no CPU fallback: if the CUDA
library is missing or no GPU is present, loading / creating a context raises.
"""
import ctypes as C
import os

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libteb_b200.so")
_lib = None


def load_library(build_if_missing=False):
    """Load libteb_b200.so (raises if it has not been built: run `python __graft_entry__.py` / build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if build_if_missing:
            from . import build as _b
            _b.build()
        else:
            raise RuntimeError(f"{LIB_PATH} is missing: build the CUDA extension first "
                               "(python -c 'import __graft_entry__ as g; g.build()'). There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.tebgpu_default_params.restype = None
    L.tebgpu_default_params.argtypes = [C.POINTER(abi.TebParams)]
    L.tebgpu_sizeof.restype = C.c_int32
    L.tebgpu_sizeof.argtypes = [C.c_int32]
    L.tebgpu_create.restype = C.c_int32
    L.tebgpu_create.argtypes = [C.POINTER(abi.TebGpuLimits), C.c_int32, C.POINTER(vp)]
    L.tebgpu_destroy.restype = C.c_int32
    L.tebgpu_destroy.argtypes = [vp]
    L.tebgpu_last_error_string.restype = C.c_char_p
    L.tebgpu_last_error_string.argtypes = [vp]
    L.tebgpu_set_params.restype = C.c_int32
    L.tebgpu_set_params.argtypes = [vp, C.POINTER(abi.TebParams)]
    L.tebgpu_optimize_batch.restype = C.c_int32
    L.tebgpu_optimize_batch.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebOptimizeArgs)]
    L.tebgpu_optimize_batch_device.restype = C.c_int32
    L.tebgpu_optimize_batch_device.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebOptimizeArgs), vp]
    L.tebgpu_set_linearize_variant.restype = C.c_int32
    L.tebgpu_set_linearize_variant.argtypes = [vp, C.c_int32]
    L.tebgpu_set_speculation.restype = C.c_int32
    L.tebgpu_set_speculation.argtypes = [vp, C.c_int32]
    L.tebgpu_set_solver.restype = C.c_int32
    L.tebgpu_set_solver.argtypes = [vp, C.c_int32]
    L.tebgpu_synchronize.restype = C.c_int32
    L.tebgpu_synchronize.argtypes = [vp]
    L.tebgpu_last_launch_count.restype = C.c_int64
    L.tebgpu_last_launch_count.argtypes = [vp]
    L.tebgpu_comm_get_unique_id.restype = C.c_int32
    L.tebgpu_comm_get_unique_id.argtypes = [vp]
    L.tebgpu_comm_init.restype = C.c_int32
    L.tebgpu_comm_init.argtypes = [vp, vp, C.c_int32, C.c_int32]
    L.tebgpu_comm_destroy.restype = C.c_int32
    L.tebgpu_comm_destroy.argtypes = [vp]
    L.tebgpu_gather_costs.restype = C.c_int32
    L.tebgpu_gather_costs.argtypes = [vp, vp, C.c_int32, vp, C.c_int32, vp]
    L.tebgpu_optimize_batch_gather.restype = C.c_int32
    L.tebgpu_optimize_batch_gather.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebOptimizeArgs), vp]
    L.tebgpu_set_warp_solver.restype = C.c_int32
    L.tebgpu_set_warp_solver.argtypes = [vp, C.c_int32]
    L.tebgpu_set_graph.restype = C.c_int32
    L.tebgpu_set_graph.argtypes = [vp, C.c_int32]
    L.tebgpu_set_solve_form.restype = C.c_int32
    L.tebgpu_set_solve_form.argtypes = [vp, C.c_int32]
    L.tebgpu_get_info.restype = C.c_int64
    L.tebgpu_get_info.argtypes = [vp, C.c_int32]
    L.tebgpu_set_profiling.restype = C.c_int32
    L.tebgpu_set_profiling.argtypes = [vp, C.c_int32]
    L.tebgpu_get_kernel_times.restype = C.c_int32
    L.tebgpu_get_kernel_times.argtypes = [vp, C.POINTER(C.c_double * 9), C.POINTER(C.c_int64 * 9)]
    L.tebgpu_compute_cost.restype = C.c_int32
    L.tebgpu_compute_cost.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebOptimizeArgs)]
    L.tebgpu_h_signature.restype = C.c_int32
    L.tebgpu_h_signature.argtypes = [vp, C.POINTER(abi.TebBatch), C.c_int32, vp, C.c_int32]
    L.tebgpu_build_system.restype = C.c_int32
    L.tebgpu_build_system.argtypes = [vp, C.POINTER(abi.TebBatch), C.c_int32, vp, vp, C.c_int32]
    L.tebgpu_build_system_graph.restype = C.c_int32
    L.tebgpu_build_system_graph.argtypes = [vp, C.POINTER(abi.TebBatch), C.c_int32, vp, C.c_int32, vp, vp, vp, vp, vp, vp, vp]
    L.tebgpu_read_linearize_outputs.restype = C.c_int32
    L.tebgpu_read_linearize_outputs.argtypes = [vp, C.c_int32, C.c_int32, vp, vp, vp]
    L.tebgpu_solve_system.restype = C.c_int32
    L.tebgpu_solve_system.argtypes = [vp, C.c_int32, C.c_int32, vp, vp, vp, vp, vp, C.c_int32, vp, vp, C.c_int32, C.c_int32,
                                      vp, vp, vp]
    L.tebgpu_eval_trials.restype = C.c_int32
    L.tebgpu_eval_trials.argtypes = [vp, C.POINTER(abi.TebBatch), C.c_int32, C.c_int32, C.c_int32, vp, vp, vp, vp, vp, vp,
                                     C.c_int32, vp, vp, vp, vp, vp, vp, vp]
    L.tebgpu_read_band_state.restype = C.c_int32
    L.tebgpu_read_band_state.argtypes = [vp, C.c_int32, vp]
    L.tebgpu_select_best.restype = C.c_int32
    L.tebgpu_select_best.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double]
    L.tebgpu_auto_resize_host.restype = C.c_int32
    L.tebgpu_auto_resize_host.argtypes = [vp, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_int32, C.c_int32, C.c_int32]
    for which, st in enumerate((abi.TebParams, abi.TebObstacle, abi.TebBatch, abi.TebOptimizeArgs, abi.TebGpuLimits)):
        if L.tebgpu_sizeof(which) != C.sizeof(st):
            raise RuntimeError(f"ABI mismatch for {st.__name__}: C {L.tebgpu_sizeof(which)} vs ctypes {C.sizeof(st)}")
    _lib = L
    return L


class TebGpuError(RuntimeError):
    pass


class TebGpu:
    """One tebgpu context (one device, one stream, its workspaces)."""

    def __init__(self, max_bands, max_poses, max_scenes=1, max_obstacles=64, max_viapoints=0, device=0, max_obst_vertices=0):
        self.lib = load_library()
        lim = abi.TebGpuLimits(max_bands, max_poses, max_scenes, max_obstacles, max_viapoints, max_obst_vertices)
        self.ctx = C.c_void_p()
        rc = self.lib.tebgpu_create(C.byref(lim), device, C.byref(self.ctx))
        if rc != 0:
            msg = self.lib.tebgpu_last_error_string(self.ctx).decode() if self.ctx else ""
            if self.ctx:
                self.lib.tebgpu_destroy(self.ctx)
                self.ctx = None
            raise TebGpuError(f"tebgpu_create failed rc={rc} {msg}")

    def _check(self, rc, what):
        if rc != 0:
            raise TebGpuError(f"{what} rc={rc}: {self.lib.tebgpu_last_error_string(self.ctx).decode()}")

    def set_params(self, params):
        self._check(self.lib.tebgpu_set_params(self.ctx, C.byref(params)), "tebgpu_set_params")
        self.params = params

    def optimize(self, hb, args):
        """Host-buffer call: hb is an abi.HostBatch, updated in place."""
        bs = hb.struct()
        self._check(self.lib.tebgpu_optimize_batch(self.ctx, C.byref(bs), C.byref(args)), "tebgpu_optimize_batch")
        return hb

    def compute_cost(self, hb, args):
        bs = hb.struct()
        self._check(self.lib.tebgpu_compute_cost(self.ctx, C.byref(bs), C.byref(args)), "tebgpu_compute_cost")
        return hb

    def optimize_device(self, batch_struct, args, stream=None):
        self._check(self.lib.tebgpu_optimize_batch_device(self.ctx, C.byref(batch_struct), C.byref(args), stream),
                    "tebgpu_optimize_batch_device")

    def set_linearize_variant(self, v):
        self._check(self.lib.tebgpu_set_linearize_variant(self.ctx, int(v)), "tebgpu_set_linearize_variant")

    def set_speculation(self, k):
        self._check(self.lib.tebgpu_set_speculation(self.ctx, int(k)), "tebgpu_set_speculation")

    def set_warp_solver(self, mode):
        """solve kernel mapping: 0 thread per system, 1 warp per system, 2 by regime"""
        self._check(self.lib.tebgpu_set_warp_solver(self.ctx, int(mode)), "tebgpu_set_warp_solver")

    def set_solve_form(self, form):
        """k_solve_tpb's factor: 0 automatic, 1 streamed through device memory, 11 / 22 / 33 recomputed in segments of
        that many rows"""
        self._check(self.lib.tebgpu_set_solve_form(self.ctx, int(form)), "tebgpu_set_solve_form")

    def set_graph(self, mode):
        """CUDA-graph replay of the launch sequence: 0 never, 1 always, 2 automatic (latency regime)"""
        self._check(self.lib.tebgpu_set_graph(self.ctx, int(mode)), "tebgpu_set_graph")

    def set_solver(self, solver):
        self._check(self.lib.tebgpu_set_solver(self.ctx, int(solver)), "tebgpu_set_solver")

    def synchronize(self):
        self._check(self.lib.tebgpu_synchronize(self.ctx), "tebgpu_synchronize")

    def set_profiling(self, enable):
        self._check(self.lib.tebgpu_set_profiling(self.ctx, int(enable)), "tebgpu_set_profiling")

    def kernel_times(self):
        """{kernel name: (total ms, launches)} since profiling was enabled / last read."""
        ms, cnt = (C.c_double * 9)(), (C.c_int64 * 9)()
        self._check(self.lib.tebgpu_get_kernel_times(self.ctx, C.byref(ms), C.byref(cnt)), "tebgpu_get_kernel_times")
        names = ("k_begin", "k_auto_resize", "k_build_graph", "k_linearize", "k_lm_step_or_retry_rounds", "k_finalize",
                 "k_solve_tpb", "k_trial_eval", "unused")
        return {nme: (ms[i], cnt[i]) for i, nme in enumerate(names)}

    def h_signature(self, hb, use_timediffs=True):
        """calculateEquivalenceClass for every band: complex array [B] (2-D) or float array [B][M_cap] (x-y-t)"""
        import numpy as np
        three_d = bool(self.params.include_dynamic_obstacles) if hasattr(self, "params") else False
        out = np.zeros((hb.B, max(hb.M_cap, 1) if three_d else 2))
        bs = hb.struct()
        self._check(self.lib.tebgpu_h_signature(self.ctx, C.byref(bs), int(use_timediffs), out.ctypes.data, 0),
                    "tebgpu_h_signature")
        return out if three_d else out[:, 0] + 1j * out[:, 1]

    # ---- the one collective (NCCL all-gather of the per-candidate costs), behind the C-ABI
    def comm_get_unique_id(self, out128):
        """rank 0: fill the 128-byte numpy uint8 array with a fresh NCCL unique id"""
        rc = self.lib.tebgpu_comm_get_unique_id(out128.ctypes.data)
        if rc != 0:
            raise TebGpuError(f"tebgpu_comm_get_unique_id rc={rc} (NCCL not loadable?)")

    def comm_init(self, ident128, world, rank):
        self._check(self.lib.tebgpu_comm_init(self.ctx, ident128.ctypes.data, int(world), int(rank)), "tebgpu_comm_init")

    def comm_destroy(self):
        self._check(self.lib.tebgpu_comm_destroy(self.ctx), "tebgpu_comm_destroy")

    def gather_costs_device(self, d_local_ptr, count_local, d_all_ptr, stream=None):
        """device pointers, stream ordered on `stream` (cudaStream_t handle; None = the context's stream)"""
        self._check(self.lib.tebgpu_gather_costs(self.ctx, d_local_ptr, int(count_local), d_all_ptr, 1, stream),
                    "tebgpu_gather_costs")

    def gather_costs(self, local_cost):
        """host numpy vector [count] -> [world * count]"""
        import numpy as np
        local_cost = np.ascontiguousarray(local_cost, dtype=np.float64)
        out = np.zeros(self.info(3) * local_cost.size)
        self._check(self.lib.tebgpu_gather_costs(self.ctx, local_cost.ctypes.data, local_cost.size, out.ctypes.data, 0, None),
                    "tebgpu_gather_costs")
        return out

    def optimize_gather(self, hb, args):
        """tebgpu_optimize_batch + all-gather of the costs: returns the gathered [world * B] vector"""
        import numpy as np
        bs = hb.struct()
        out = np.zeros(self.info(3) * hb.B)
        self._check(self.lib.tebgpu_optimize_batch_gather(self.ctx, C.byref(bs), C.byref(args), out.ctypes.data),
                    "tebgpu_optimize_batch_gather")
        return out

    def info(self, which):
        return int(self.lib.tebgpu_get_info(self.ctx, int(which)))

    def speculation_width(self):
        """speculation width (trials solved concurrently per round) chosen by the last optimize call"""
        return self.info(0)

    EVAL_BUILDS = {0: "v1", 1: "eval2_wide", 2: "eval2", 3: "eval2p", 4: "eval3"}   # TEBGPU_EVAL_BUILD_*

    def last_trial_eval(self):
        """(build, grid in CTAs) of the last trial-evaluation launch this context issued: build is one of EVAL_BUILDS'
        names, or None before the first launch"""
        return self.EVAL_BUILDS.get(self.info(9)), self.info(8)

    KA_BUILDS = {0: "v1", 1: "oneshot", 2: "direct", 3: "persistent"}   # TEBGPU_KA_BUILD_*

    def last_linearize(self):
        """(build, grid in CTAs) of the last kernel-A launch this context issued: build is one of KA_BUILDS' names, or
        None before the first launch"""
        return self.KA_BUILDS.get(self.info(11)), self.info(10)

    def linearize_outputs(self, B, n_cap):
        """kernel A's rhs [B][4 n_cap], chi2 tile partials [B][tiles][4] and max-diagonal tile partials [B][tiles]
        (tiles = ceil(n_cap / 29), ceil(n_cap / 32) under linearize variant 1) of the last build_system call on B bands
        of n_cap poses"""
        import numpy as np
        tile = 32 if self.info(1) == 1 else 29
        tiles = (n_cap + tile - 1) // tile
        out = dict(rhs=np.empty((B, 4 * n_cap)), chi_parts=np.empty((B, tiles, 4)), dmax_parts=np.empty((B, tiles)))
        self._check(self.lib.tebgpu_read_linearize_outputs(self.ctx, int(B), int(n_cap), *(out[k].ctypes.data for k in
                                                           ("rhs", "chi_parts", "dmax_parts"))), "tebgpu_read_linearize_outputs")
        return out

    def launch_count(self):
        return int(self.lib.tebgpu_last_launch_count(self.ctx))

    def build_system(self, hb, outer_index=0, bands=None, graph=False):
        """Returns (Hb [B][4*n_cap][12], chi2 [B]) as numpy arrays (host-buffer path).

        With bands (a list of band indices: k_build_graph and kernel A run over that list as the retry side stream runs
        them) or graph=True, runs tebgpu_build_system_graph instead and returns dict(Hb, chi_fam [B][4] (obstacles, via,
        time-optimal, other), assoc, assoc3 [B][n_cap][MW] uint64, occ [B][n_cap][OW] uint64, via_idx [B][V_cap],
        dyn_t [B][n_cap]); everything starts as all-ones bytes, so what no kernel wrote keeps that pattern."""
        import numpy as np
        if bands is not None or graph:
            B, n_cap = hb.B, hb.n_cap
            MW = max(1, (hb.M_cap + 63) // 64)
            OW = (MW + 63) // 64
            order = None if bands is None else np.ascontiguousarray(bands, dtype=np.int32)
            out = dict(Hb=np.empty((B, 4 * n_cap, 12)), chi_fam=np.empty((B, 4)),
                       assoc=np.empty((B, n_cap, MW), np.uint64), assoc3=np.empty((B, n_cap, MW), np.uint64),
                       occ=np.empty((B, n_cap, OW), np.uint64), via_idx=np.empty((B, hb.V_cap), np.int32),
                       dyn_t=np.empty((B, n_cap)))
            bs = hb.struct()
            self._check(self.lib.tebgpu_build_system_graph(
                self.ctx, C.byref(bs), int(outer_index), abi.ptr(order), 0 if order is None else order.size,
                *(out[k].ctypes.data for k in ("Hb", "chi_fam", "assoc", "assoc3", "occ", "via_idx", "dyn_t"))),
                "tebgpu_build_system_graph")
            return out
        Hb = np.zeros((hb.B, 4 * hb.n_cap, 12))
        chi2 = np.zeros(hb.B)
        bs = hb.struct()
        self._check(self.lib.tebgpu_build_system(self.ctx, C.byref(bs), outer_index, Hb.ctypes.data, chi2.ctypes.data, 0),
                    "tebgpu_build_system")
        return Hb, chi2

    def solve_system(self, n, K, Hb=None, n_cap=None, lam=None, nu=None, active=None, qmax=None, order=None, lat_cap=0):
        """Solve (H + lambda_k I_real) x = b for every band and trial k < K with the context's solver / solve mapping
        (tebgpu_solve_system). Hb [B][4 n_cap][12] or None (the system of the last build_system: pass n_cap); lam / nu
        [B] or None (LM iteration 0: lambda from kernel A); active [B] or None; qmax [B] + order (list of bands): a
        retry round over `order`. Returns (dx [B][K][4 n_cap], ok [B][K], lambda [B][K]); what no kernel wrote keeps
        the all-ones NaN pattern."""
        import numpy as np
        n = np.ascontiguousarray(n, dtype=np.int32)
        B = n.size
        if Hb is not None:
            Hb = np.ascontiguousarray(Hb, dtype=np.float64)
            n_cap = Hb.shape[1] // 4
        f64 = lambda a: None if a is None else np.ascontiguousarray(np.broadcast_to(a, (B,)), dtype=np.float64)
        lam, nu = f64(lam), f64(nu)
        active = None if active is None else np.ascontiguousarray(active, dtype=np.int32)
        qmax = None if qmax is None else np.ascontiguousarray(qmax, dtype=np.int32)
        order = None if order is None else np.ascontiguousarray(order, dtype=np.int32)
        dx = np.empty((B, K, 4 * n_cap))
        ok = np.empty((B, K))
        lam_used = np.empty((B, K))
        self._check(self.lib.tebgpu_solve_system(self.ctx, B, int(n_cap), abi.ptr(Hb), n.ctypes.data, abi.ptr(lam), abi.ptr(nu),
                                                 abi.ptr(active), int(K), abi.ptr(qmax), abi.ptr(order),
                                                 0 if order is None else order.size, int(lat_cap), dx.ctypes.data,
                                                 ok.ctypes.data, lam_used.ctypes.data), "tebgpu_solve_system")
        return dx, ok, lam_used

    EVAL_STATE = 14   # band state columns: lambda, nu, currentChi, chi2 by family (current 4, last trial 4), status,
                      # active, LM iterations

    def eval_trials(self, hb, K, dx, ok, lam, state, outer_index=0, iteration=1, qmax=None, order=None):
        """One round of trial evaluation and g2o's accept / reject chain (tebgpu_eval_trials) on the graph and system
        that build_system(hb, outer_index) makes. dx [B][K][4 n_cap], ok [B][K], lam [B][K]: the trials; state
        [B][EVAL_STATE]: the band state before the round; qmax [B] + order (list of bands): a retry round over `order`.
        hb.poses receives the state after the round. Returns dict(res [B][K][5], chi_lin [B][4], state [B][EVAL_STATE],
        qmax [B], need [B], next_list)."""
        import numpy as np
        B, n_cap = hb.B, hb.n_cap
        f64 = lambda a, shape: np.ascontiguousarray(np.broadcast_to(a, shape), dtype=np.float64)
        dx, ok, lam = f64(dx, (B, K, 4 * n_cap)), f64(ok, (B, K)), f64(lam, (B, K))
        state = f64(state, (B, self.EVAL_STATE))
        qmax = None if qmax is None else np.ascontiguousarray(qmax, dtype=np.int32)
        order = None if order is None else np.ascontiguousarray(order, dtype=np.int32)
        res = np.empty((B, K, 5))
        chi_lin = np.empty((B, 4))
        st_out = np.empty((B, self.EVAL_STATE))
        q_out = np.empty(B, np.int32)
        need = np.empty(B, np.int32)
        nxt = np.empty(B, np.int32)
        nlen = C.c_int32(0)
        bs = hb.struct()
        self._check(self.lib.tebgpu_eval_trials(self.ctx, C.byref(bs), int(outer_index), int(iteration), int(K), dx.ctypes.data,
                                                ok.ctypes.data, lam.ctypes.data, state.ctypes.data, abi.ptr(qmax),
                                                abi.ptr(order), 0 if order is None else order.size, res.ctypes.data,
                                                chi_lin.ctypes.data, st_out.ctypes.data, q_out.ctypes.data, need.ctypes.data,
                                                nxt.ctypes.data, C.byref(nlen)), "tebgpu_eval_trials")
        return dict(res=res, chi_lin=chi_lin, state=st_out, qmax=q_out, need=need, next_list=nxt[:nlen.value].copy())

    def band_state(self, B):
        """[B][EVAL_STATE] state of every band after the last optimize / optimize_device call (tebgpu_read_band_state):
        lambda, nu, currentChi, chi2 by family at the current state (4) and at the last evaluated trial (4), status bits
        (without OPTIMIZED), active, LM iterations"""
        import numpy as np
        out = np.empty((int(B), self.EVAL_STATE))
        self._check(self.lib.tebgpu_read_band_state(self.ctx, int(B), out.ctypes.data), "tebgpu_read_band_state")
        return out

    def close(self):
        if self.ctx:
            self.lib.tebgpu_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
