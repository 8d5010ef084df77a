"""teb_local_planner_b200 — H100-native (sm_90a) batched Timed-Elastic-Band optimizer.

Python side: ctypes loader for the in-tree CUDA library (C-ABI in include/teb_b200.h) and a thin
`TebGpu` convenience wrapper used by tests and bench.py. There is no CPU fallback: if the CUDA
library is missing or no GPU is present, loading / creating a context raises.
"""
import ctypes as C
import math
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
    L.tebgpu_plan_batch.restype = C.c_int32
    L.tebgpu_plan_batch.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebPlanInput), C.POINTER(abi.TebOptimizeArgs)]
    L.tebgpu_plan_batch_device.restype = C.c_int32
    L.tebgpu_plan_batch_device.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebPlanInput),
                                           C.POINTER(abi.TebOptimizeArgs), vp]
    L.tebgpu_check_feasible.restype = C.c_int32
    L.tebgpu_check_feasible.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebFeasibilityArgs)]
    L.tebgpu_check_feasible_device.restype = C.c_int32
    L.tebgpu_check_feasible_device.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebFeasibilityArgs), vp]
    L.tebgpu_check_feasible_costmap.restype = C.c_int32
    L.tebgpu_check_feasible_costmap.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebFeasibilityArgs),
                                                C.POINTER(abi.TebCostmapWorld)]
    L.tebgpu_check_feasible_costmap_device.restype = C.c_int32
    L.tebgpu_check_feasible_costmap_device.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebFeasibilityArgs),
                                                       C.POINTER(abi.TebCostmapWorld), vp]
    L.tebgpu_read_trajectory.restype = C.c_int32
    L.tebgpu_read_trajectory.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebTrajectoryArgs)]
    L.tebgpu_read_trajectory_device.restype = C.c_int32
    L.tebgpu_read_trajectory_device.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebTrajectoryArgs), vp]
    L.tebgpu_costmap_obstacles.restype = C.c_int32
    L.tebgpu_costmap_obstacles.argtypes = [vp, C.POINTER(abi.TebCostmapArgs)]
    L.tebgpu_costmap_obstacles_device.restype = C.c_int32
    L.tebgpu_costmap_obstacles_device.argtypes = [vp, C.POINTER(abi.TebCostmapArgs), vp]
    L.tebgpu_local_plan.restype = C.c_int32
    L.tebgpu_local_plan.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebLocalPlanArgs)]
    L.tebgpu_local_plan_device.restype = C.c_int32
    L.tebgpu_local_plan_device.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebLocalPlanArgs), vp]
    L.tebgpu_costmap_obstacles_tf.restype = C.c_int32
    L.tebgpu_costmap_obstacles_tf.argtypes = [vp, C.POINTER(abi.TebCostmapArgs), C.POINTER(abi.TebFrameArgs)]
    L.tebgpu_costmap_obstacles_tf_device.restype = C.c_int32
    L.tebgpu_costmap_obstacles_tf_device.argtypes = [vp, C.POINTER(abi.TebCostmapArgs), C.POINTER(abi.TebFrameArgs), vp]
    L.tebgpu_costmap_window.restype = C.c_int32
    L.tebgpu_costmap_window.argtypes = [vp, C.POINTER(abi.TebStaticMaps), C.POINTER(abi.TebCostmapWindowArgs)]
    L.tebgpu_costmap_window_device.restype = C.c_int32
    L.tebgpu_costmap_window_device.argtypes = [vp, C.POINTER(abi.TebStaticMaps), C.POINTER(abi.TebCostmapWindowArgs), vp]
    L.tebgpu_costmap_obstacle_layer.restype = C.c_int32
    L.tebgpu_costmap_obstacle_layer.argtypes = [vp, C.POINTER(abi.TebObstacleLayerArgs)]
    L.tebgpu_costmap_obstacle_layer_device.restype = C.c_int32
    L.tebgpu_costmap_obstacle_layer_device.argtypes = [vp, C.POINTER(abi.TebObstacleLayerArgs), vp]
    L.tebgpu_costmap_voxel_layer.restype = C.c_int32
    L.tebgpu_costmap_voxel_layer.argtypes = [vp, C.POINTER(abi.TebVoxelLayerArgs)]
    L.tebgpu_costmap_voxel_layer_device.restype = C.c_int32
    L.tebgpu_costmap_voxel_layer_device.argtypes = [vp, C.POINTER(abi.TebVoxelLayerArgs), vp]
    L.tebgpu_local_plan_tf.restype = C.c_int32
    L.tebgpu_local_plan_tf.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebLocalPlanArgs),
                                       C.POINTER(abi.TebFrameArgs)]
    L.tebgpu_local_plan_tf_device.restype = C.c_int32
    L.tebgpu_local_plan_tf_device.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebLocalPlanArgs),
                                              C.POINTER(abi.TebFrameArgs), vp]
    for name in ("tebgpu_backup_modes", "tebgpu_finish_cycle"):
        getattr(L, name).restype = C.c_int32
        getattr(L, name).argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebCycleArgs)]
        getattr(L, name + "_device").restype = C.c_int32
        getattr(L, name + "_device").argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebCycleArgs), vp]
    L.tebgpu_fleet_obstacles.restype = C.c_int32
    L.tebgpu_fleet_obstacles.argtypes = [vp, C.POINTER(abi.TebFleetArgs)]
    L.tebgpu_fleet_obstacles_device.restype = C.c_int32
    L.tebgpu_fleet_obstacles_device.argtypes = [vp, C.POINTER(abi.TebFleetArgs), vp]
    for name in ("tebgpu_fleet_publish", "tebgpu_fleet_obstacles_table"):
        getattr(L, name).restype = C.c_int32
        getattr(L, name).argtypes = [vp, C.POINTER(abi.TebFleetArgs), C.POINTER(abi.TebFleetTable)]
        getattr(L, name + "_device").restype = C.c_int32
        getattr(L, name + "_device").argtypes = [vp, C.POINTER(abi.TebFleetArgs), C.POINTER(abi.TebFleetTable), vp]
    FA, FS, FT = C.POINTER(abi.TebFleetArgs), C.POINTER(abi.TebFleetShapes), C.POINTER(abi.TebFleetTable)
    for name, args in (("tebgpu_fleet_obstacles_shaped", [vp, FA, FS]), ("tebgpu_fleet_publish_shaped", [vp, FA, FS, FT]),
                       ("tebgpu_fleet_gather_shaped", [vp, FS, FT, C.c_int32]),
                       ("tebgpu_fleet_obstacles_table_shaped", [vp, FA, FS, FT])):
        getattr(L, name).restype = C.c_int32
        getattr(L, name).argtypes = args
        getattr(L, name + "_device").restype = C.c_int32
        getattr(L, name + "_device").argtypes = args + [vp]
    L.tebgpu_fleet_gather.restype = C.c_int32
    L.tebgpu_fleet_gather.argtypes = [vp, C.POINTER(abi.TebFleetTable), C.c_int32]
    L.tebgpu_fleet_gather_device.restype = C.c_int32
    L.tebgpu_fleet_gather_device.argtypes = [vp, C.POINTER(abi.TebFleetTable), C.c_int32, vp]
    L.tebgpu_get_plan_kernel_times.restype = C.c_int32
    L.tebgpu_get_plan_kernel_times.argtypes = [vp, C.POINTER(C.c_double * 2), C.POINTER(C.c_int64 * 2)]
    L.tebgpu_set_linearize_variant.restype = C.c_int32
    L.tebgpu_set_linearize_variant.argtypes = [vp, C.c_int32]
    L.tebgpu_set_fleet_search.restype = C.c_int32
    L.tebgpu_set_fleet_search.argtypes = [vp, C.c_int32]
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
    L.tebgpu_hsig_factors.restype = C.c_int32
    L.tebgpu_hsig_factors.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebHsigFactors)]
    L.tebgpu_hsig_factors_device.restype = C.c_int32
    L.tebgpu_hsig_factors_device.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebHsigFactors), vp]
    L.tebgpu_h_signature_scenes.restype = C.c_int32
    L.tebgpu_h_signature_scenes.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebHsigFactors), C.c_int32, vp]
    L.tebgpu_h_signature_scenes_device.restype = C.c_int32
    L.tebgpu_h_signature_scenes_device.argtypes = [vp, C.POINTER(abi.TebBatch), C.POINTER(abi.TebHsigFactors), C.c_int32,
                                                   vp, vp]
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
    for which, st in tuple(enumerate((abi.TebParams, abi.TebObstacle, abi.TebBatch, abi.TebOptimizeArgs, abi.TebGpuLimits,
                                abi.TebPlanInput, abi.TebFeasibilityArgs, abi.TebTrajectoryArgs, abi.TebCostmapArgs,
                                abi.TebLocalPlanArgs, abi.TebCycleArgs, abi.TebCostmapWorld, abi.TebFrameArgs,
                                abi.TebHsigFactors, abi.TebFleetArgs))) + ((15, None), (16, abi.TebFleetTable),
                                                                (17, abi.TebFleetShapes), (18, abi.TebStaticMaps),
                                                                (19, abi.TebCostmapWindowArgs),
                                                                (20, abi.TebObstacleLayerArgs),
                                                                (21, abi.TebVoxelLayerArgs),
                                                                (22, abi.TebObservationSource)):
        if st is None:
            if L.tebgpu_sizeof(which) != abi.FLEET_ROW_DTYPE.itemsize:
                raise RuntimeError(f"ABI mismatch for TebFleetRow: C {L.tebgpu_sizeof(which)} vs FLEET_ROW_DTYPE "
                                   f"{abi.FLEET_ROW_DTYPE.itemsize}")
            continue
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

    def plan(self, hb, start, goal, args, look_ahead_poses=1, prevent_near_goal=0, initial_plan=None, plan_count=None,
             path=True):
        """TebOptimalPlanner::plan followed by getVelocityCommand for every band (tebgpu_plan_batch), host buffers.

        hb (abi.HostBatch) is updated in place: a band with n == 0 is initialised from start to goal, a band with n > 0
        is warm started (updateAndPruneTEB) or re-initialised when the goal jumped, then optimised with `args`.
        start, goal: [B][3] (x, y, theta); or initial_plan [B][P_cap][3] (x, y, yaw) with plan_count [B] (None: P_cap
        points each), start / goal are then ignored. Returns (cmd [B][4] = vx, vy, omega, ok, path [B] TEB_PLAN_PATH_*)."""
        import numpy as np
        B = hb.B
        f64 = lambda a, shape: None if a is None else np.ascontiguousarray(np.broadcast_to(a, shape), dtype=np.float64)
        cmd = np.zeros((B, 4))
        pth = np.full(B, -2, np.int32) if path else None
        pi = abi.TebPlanInput()
        if initial_plan is not None:
            ip = np.ascontiguousarray(initial_plan, dtype=np.float64)
            pc = None if plan_count is None else np.ascontiguousarray(plan_count, dtype=np.int32)
            pi.initial_plan, pi.plan_count, pi.P_cap = abi.ptr(ip), abi.ptr(pc), ip.shape[1]
        else:
            s, g = f64(start, (B, 3)), f64(goal, (B, 3))
            pi.start, pi.goal = abi.ptr(s), abi.ptr(g)
        pi.look_ahead_poses, pi.prevent_look_ahead_poses_near_goal = int(look_ahead_poses), int(prevent_near_goal)
        pi.cmd, pi.path = abi.ptr(cmd), abi.ptr(pth)
        bs = hb.struct()
        self._check(self.lib.tebgpu_plan_batch(self.ctx, C.byref(bs), C.byref(pi), C.byref(args)), "tebgpu_plan_batch")
        return cmd, pth

    def plan_device(self, batch_struct, args, cmd, start=None, goal=None, path=None, initial_plan=None, plan_count=None,
                    P_cap=0, look_ahead_poses=1, prevent_near_goal=0, stream=None):
        """tebgpu_plan_batch_device: the same cycle over DEVICE memory (batch_struct: an abi.TebBatch of device
        pointers). cmd [B][4] float64, start / goal [B][3] float64, path [B] int32 (or None), initial_plan
        [B][P_cap][3] float64 with plan_count [B] int32 (or None): device pointers as ints, or torch tensors. Stream
        ordered on `stream` (a cudaStream_t handle; None: the context's stream); does not synchronise."""
        addr = lambda t: None if t is None else (t.data_ptr() if hasattr(t, "data_ptr") else int(t))
        pi = abi.TebPlanInput()
        pi.start, pi.goal, pi.initial_plan, pi.plan_count = addr(start), addr(goal), addr(initial_plan), addr(plan_count)
        if initial_plan is not None and not P_cap and hasattr(initial_plan, "shape"):
            P_cap = initial_plan.shape[1]
        pi.P_cap = int(P_cap)
        pi.look_ahead_poses, pi.prevent_look_ahead_poses_near_goal = int(look_ahead_poses), int(prevent_near_goal)
        pi.cmd, pi.path = addr(cmd), addr(path)
        self._check(self.lib.tebgpu_plan_batch_device(self.ctx, C.byref(batch_struct), C.byref(pi), C.byref(args), stream),
                    "tebgpu_plan_batch_device")

    def check_feasible(self, hb, inscribed_radius, look_ahead_idx=-1, lookahead_distance=-1.0, angular_resolution=math.pi,
                       collision_distance=0.0, max_queries=1024, queries=False):
        """TebOptimalPlanner::isTrajectoryFeasible for every band of hb (an abi.HostBatch) against its scene's obstacles
        (tebgpu_check_feasible), host buffers. Returns (feasible [B] int32: 1 feasible, 0 colliding, -1 undecidable,
        query_count [B] int32), and with queries=True also the query poses [B][max_queries][3] (NaN past each band's
        min(query_count, max_queries) rows)."""
        import numpy as np
        feas = np.zeros(hb.B, np.int32)
        cnt = np.zeros(hb.B, np.int32)
        q = np.full((hb.B, int(max_queries), 3), np.nan) if queries else None
        fa = abi.make_feasibility_args(inscribed_radius, look_ahead_idx, lookahead_distance, angular_resolution,
                                       collision_distance, max_queries, abi.ptr(feas), abi.ptr(cnt), abi.ptr(q))
        bs = hb.struct()
        self._check(self.lib.tebgpu_check_feasible(self.ctx, C.byref(bs), C.byref(fa)), "tebgpu_check_feasible")
        return (feas, cnt, q) if queries else (feas, cnt)

    def check_feasible_device(self, batch_struct, fargs, stream=None):
        """tebgpu_check_feasible_device: the same check over DEVICE memory (batch_struct: an abi.TebBatch of device
        pointers; fargs: an abi.TebFeasibilityArgs whose outputs are device addresses, see abi.make_feasibility_args).
        Stream ordered on `stream` (a cudaStream_t handle; None: the context's stream); does not synchronise."""
        self._check(self.lib.tebgpu_check_feasible_device(self.ctx, C.byref(batch_struct), C.byref(fargs), stream),
                    "tebgpu_check_feasible_device")

    def check_feasible_costmap(self, hb, cost, grid, origin, footprint, inscribed_radius, look_ahead_idx=-1,
                               lookahead_distance=-1.0, angular_resolution=math.pi, max_queries=1024, queries=False,
                               query_cost=False):
        """isTrajectoryFeasible for every band of hb (an abi.HostBatch; its poses, n and scene_id are read) against its
        scene's costmap, CostmapModel::footprintCost as include/teb_b200.h defines it at TebCostmapWorld
        (tebgpu_check_feasible_costmap), host buffers: cost [S][cell_cap] uint8, grid [S][2] (sx, sy), origin [S][3]
        (ox, oy, resolution), footprint [F][2] in the robot frame (F < 3: the centre cell only). Returns (feasible [B]
        int32: 1 feasible, 0 colliding, -1 undecidable, query_count [B] int32), then with queries=True the query poses
        [B][max_queries][3] and with query_cost=True each tested query's footprintCost [B][max_queries] (NaN past each
        band's min(query_count, max_queries) rows)."""
        import numpy as np
        cost = np.ascontiguousarray(cost, dtype=np.uint8)
        S = cost.shape[0]
        cost = cost.reshape(S, -1)
        grid = np.ascontiguousarray(grid, dtype=np.int32).reshape(S, 2)
        origin = np.ascontiguousarray(origin, dtype=np.float64).reshape(S, 3)
        feas = np.zeros(hb.B, np.int32)
        cnt = np.zeros(hb.B, np.int32)
        q = np.full((hb.B, int(max_queries), 3), np.nan) if queries else None
        qc = np.full((hb.B, int(max_queries)), np.nan) if query_cost else None
        fa = abi.make_feasibility_args(inscribed_radius, look_ahead_idx, lookahead_distance, angular_resolution, 0.0,
                                       max_queries, abi.ptr(feas), abi.ptr(cnt), abi.ptr(q))
        w = abi.make_costmap_world(cost.shape[1], abi.ptr(cost), abi.ptr(grid), abi.ptr(origin), footprint, abi.ptr(qc))
        bs = hb.struct()
        self._check(self.lib.tebgpu_check_feasible_costmap(self.ctx, C.byref(bs), C.byref(fa), C.byref(w)),
                    "tebgpu_check_feasible_costmap")
        return (feas, cnt) + ((q,) if queries else ()) + ((qc,) if query_cost else ())

    def check_feasible_costmap_device(self, batch_struct, fargs, world, stream=None):
        """tebgpu_check_feasible_costmap_device: the same check over DEVICE memory (batch_struct: an abi.TebBatch of
        device pointers, of which poses, n and scene_id are read; fargs: an abi.TebFeasibilityArgs whose outputs are
        device addresses; world: an abi.TebCostmapWorld of device arrays and a host footprint, see
        abi.make_costmap_world). Stream ordered on `stream` (a cudaStream_t handle; None: the context's stream); does
        not synchronise."""
        self._check(self.lib.tebgpu_check_feasible_costmap_device(self.ctx, C.byref(batch_struct), C.byref(fargs),
                                                                  C.byref(world), stream),
                    "tebgpu_check_feasible_costmap_device")

    def read_trajectory(self, hb, bands=None, profile=True, trajectory=True):
        """getVelocityProfile / getFullTrajectory of the bands of hb (an abi.HostBatch) listed in `bands` (None: all B, in
        order) on the device (tebgpu_read_trajectory), host buffers, with the context's max_vel_y. Returns (profile
        [R][n_cap + 1][3] vx, vy, omega, trajectory [R][n_cap][7] x, y, theta, vx, vy, omega, time_from_start, points
        [R] int32: each row's n); rows past n + 1 / n are NaN. profile=False / trajectory=False: None in its place."""
        import numpy as np
        bl = None if bands is None else np.ascontiguousarray(bands, dtype=np.int32).reshape(-1)
        R = hb.B if bl is None else len(bl)
        prof = np.full((R, hb.n_cap + 1, 3), np.nan) if profile else None
        traj = np.full((R, hb.n_cap, 7), np.nan) if trajectory else None
        pts = np.zeros(R, np.int32)
        ta = abi.TebTrajectoryArgs()
        ta.bands, ta.count = abi.ptr(bl), R
        ta.profile, ta.trajectory, ta.points = abi.ptr(prof), abi.ptr(traj), abi.ptr(pts)
        bs = hb.struct()
        self._check(self.lib.tebgpu_read_trajectory(self.ctx, C.byref(bs), C.byref(ta)), "tebgpu_read_trajectory")
        return prof, traj, pts

    def read_trajectory_device(self, batch_struct, trajectory=None, profile=None, points=None, bands=None, count=None,
                               stream=None):
        """tebgpu_read_trajectory_device: the same read-out over DEVICE memory (batch_struct: an abi.TebBatch of device
        pointers). trajectory [R][n_cap][7] / profile [R][n_cap + 1][3] float64 (either may be None, not both), points
        [R] int32, bands [count] int32 or None (all B bands): device pointers as ints, or torch tensors; count defaults
        to the length of a `bands` tensor. Stream ordered on `stream` (a cudaStream_t handle; None: the context's
        stream); does not synchronise."""
        addr = lambda t: None if t is None else (t.data_ptr() if hasattr(t, "data_ptr") else int(t))
        if count is None:
            count = bands.numel() if hasattr(bands, "numel") else 0
        ta = abi.TebTrajectoryArgs()
        ta.bands, ta.count = addr(bands), int(count)
        ta.profile, ta.trajectory, ta.points = addr(profile), addr(trajectory), addr(points)
        self._check(self.lib.tebgpu_read_trajectory_device(self.ctx, C.byref(batch_struct), C.byref(ta), stream),
                    "tebgpu_read_trajectory_device")

    def costmap_obstacles(self, cost, grid, origin, robot, M_cap, behind_robot_dist=1.5, include=True, custom=None,
                          custom_count=None, custom_to_costmap=None, custom_vertices=None):
        """Each scene's obstacle table from its local costmap (tebgpu_costmap_obstacles), host buffers: cost [S][cell_cap]
        uint8 (scene s's char map in its first sx * sy bytes, row my = mx + my * sx), grid [S][2] (sx, sy), origin [S][3]
        (ox, oy, resolution), robot [S][3] (x, y, yaw), custom [S][C_cap] abi.OBST_DTYPE rows appended after the points,
        custom_count [S]. Returns (obstacles [S][M_cap] abi.OBST_DTYPE, zero past each scene's written rows, obst_count
        [S]: the rows, or -1 when they do not fit M_cap, needed [S]: the rows the scene has).
        custom_to_costmap [S][7] (see abi.TebFrameArgs): the custom rows are in their own frame and are moved into the
        costmap's (tebgpu_costmap_obstacles_tf); custom_vertices [S][PV_cap][2] their Line / Pill / Polygon vertices in
        that frame, whose moved copy [S][PV_cap][2] (zero where no row moved a vertex) is then returned fourth."""
        import numpy as np
        cost = np.ascontiguousarray(cost, dtype=np.uint8)
        S = cost.shape[0]
        cost = cost.reshape(S, -1)
        grid = np.ascontiguousarray(grid, dtype=np.int32).reshape(S, 2)
        origin = np.ascontiguousarray(origin, dtype=np.float64).reshape(S, 3)
        robot = np.ascontiguousarray(robot, dtype=np.float64).reshape(S, 3)
        obst = np.zeros((S, int(M_cap)), abi.OBST_DTYPE)
        cnt = np.zeros(S, np.int32)
        need = np.zeros(S, np.int32)
        ca = abi.TebCostmapArgs()
        ca.S, ca.cell_cap, ca.M_cap = S, cost.shape[1], int(M_cap)
        ca.include_costmap_obstacles, ca.behind_robot_dist = int(bool(include)), float(behind_robot_dist)
        ca.cost, ca.grid, ca.origin, ca.robot = abi.ptr(cost), abi.ptr(grid), abi.ptr(origin), abi.ptr(robot)
        if custom is not None:
            custom = np.ascontiguousarray(custom, dtype=abi.OBST_DTYPE).reshape(S, -1)
            cc = (np.full(S, custom.shape[1], np.int32) if custom_count is None
                  else np.ascontiguousarray(custom_count, dtype=np.int32).reshape(S))
            ca.C_cap, ca.custom, ca.custom_count = custom.shape[1], abi.ptr(custom), abi.ptr(cc)
        ca.obstacles, ca.obst_count, ca.needed = abi.ptr(obst), abi.ptr(cnt), abi.ptr(need)
        if custom_to_costmap is None and custom_vertices is None:
            self._check(self.lib.tebgpu_costmap_obstacles(self.ctx, C.byref(ca)), "tebgpu_costmap_obstacles")
            return obst, cnt, need
        tf = None if custom_to_costmap is None else np.ascontiguousarray(custom_to_costmap, dtype=np.float64).reshape(S, 7)
        cv = None if custom_vertices is None else np.ascontiguousarray(custom_vertices, dtype=np.float64).reshape(S, -1, 2)
        ov = None if cv is None else np.zeros_like(cv)
        fr = abi.make_frame_args(custom_to_costmap=abi.ptr(tf), custom_vertices=abi.ptr(cv), obst_vertices=abi.ptr(ov),
                                 PV_cap=0 if cv is None else cv.shape[1])
        self._check(self.lib.tebgpu_costmap_obstacles_tf(self.ctx, C.byref(ca), C.byref(fr)), "tebgpu_costmap_obstacles_tf")
        return (obst, cnt, need) if ov is None else (obst, cnt, need, ov)

    def costmap_obstacles_device(self, args, stream=None, frames=None):
        """tebgpu_costmap_obstacles_device: the same conversion over DEVICE memory (args: an abi.TebCostmapArgs of device
        pointers, e.g. the obstacles / obst_count of the batch it feeds). Stream ordered on `stream` (a cudaStream_t
        handle; None: the context's stream); does not synchronise. frames: an abi.TebFrameArgs of device pointers
        (custom_to_costmap, custom_vertices, obst_vertices: the batch's vertex pool), or None: the custom rows verbatim."""
        if frames is None:
            self._check(self.lib.tebgpu_costmap_obstacles_device(self.ctx, C.byref(args), stream),
                        "tebgpu_costmap_obstacles_device")
        else:
            self._check(self.lib.tebgpu_costmap_obstacles_tf_device(self.ctx, C.byref(args), C.byref(frames), stream),
                        "tebgpu_costmap_obstacles_tf_device")

    def last_costmap_grid(self):
        """grid in CTAs (one per scene) of the last costmap conversion, 0 before the first"""
        return self.info(15)

    def costmap_window(self, maps, robot, map_id, origin, grid, cell_cap=None, costmap_to_map=None):
        """Every robot's local costmap cut out of the static maps (tebgpu_costmap_window), host buffers, as
        include/teb_b200.h defines it at TebStaticMaps: maps an abi.TebStaticMaps of host arrays (abi.make_static_maps),
        robot [S][3], map_id [S], origin [S][3] (ox, oy, resolution: the previous cycle's origin), grid [S][2] (sx, sy),
        cell_cap (None: the largest sx * sy rounded up to 16 bytes), costmap_to_map [S][7] or None (the identity).
        Returns (cost [S][cell_cap] uint8, origin [S][3] the snapped origins, status [S] int32 TEB_COSTMAP_WINDOW_*);
        the arguments are not modified."""
        import numpy as np
        robot = np.ascontiguousarray(robot, dtype=np.float64).reshape(-1, 3)
        S = robot.shape[0]
        mid = np.ascontiguousarray(map_id, dtype=np.int32).reshape(S)
        org = np.array(origin, dtype=np.float64).reshape(S, 3)
        grid = np.ascontiguousarray(grid, dtype=np.int32).reshape(S, 2)
        if cell_cap is None:
            cell_cap = max(16, (int((grid[:, 0].astype(np.int64) * grid[:, 1]).max()) + 15) // 16 * 16)
        tf = None if costmap_to_map is None else np.ascontiguousarray(costmap_to_map, dtype=np.float64).reshape(S, 7)
        cost = np.zeros((S, int(cell_cap)), np.uint8)
        status = np.zeros(S, np.int32)
        wa = abi.TebCostmapWindowArgs()
        wa.S, wa.cell_cap = S, int(cell_cap)
        wa.robot, wa.map_id, wa.costmap_to_map = abi.ptr(robot), abi.ptr(mid), abi.ptr(tf)
        wa.origin, wa.grid, wa.cost, wa.status = abi.ptr(org), abi.ptr(grid), abi.ptr(cost), abi.ptr(status)
        self._check(self.lib.tebgpu_costmap_window(self.ctx, C.byref(maps), C.byref(wa)), "tebgpu_costmap_window")
        return cost, org, status

    def costmap_window_device(self, maps, args, stream=None):
        """tebgpu_costmap_window_device: the same step over DEVICE memory (maps: an abi.TebStaticMaps of device arrays;
        args: an abi.TebCostmapWindowArgs of device pointers, whose cost / grid / origin are the TebCostmapArgs arrays
        the costmap conversion and the costmap check read next). Stream ordered on `stream` (a cudaStream_t handle;
        None: the context's stream); does not synchronise."""
        self._check(self.lib.tebgpu_costmap_window_device(self.ctx, C.byref(maps), C.byref(args), stream),
                    "tebgpu_costmap_window_device")

    def last_window_grid(self):
        """grid in CTAs of the last costmap window's raster launch, 0 before the first"""
        return self.info(20)

    def costmap_obstacle_layer(self, points, point_count, sensor_origin, robot, grid, layer, layer_origin, origin, cost,
                               footprint=None, flags=True, **params):
        """Every robot's obstacle layer marked and cleared from its sensor points (tebgpu_costmap_obstacle_layer), host
        buffers, as include/teb_b200.h defines it at TebObstacleLayerArgs: points [S][P_cap][3] float32, point_count [S],
        sensor_origin [S][3], robot [S][3] (x, y, yaw), grid [S][2], layer [S][cell_cap] uint8 and layer_origin [S][2]
        (the previous cycle's), origin [S][3] and cost [S][cell_cap] (the master raster), footprint [F][2] or None;
        params: the keywords of abi.make_obstacle_layer_args. Returns (layer, layer_origin, cost, origin, status, flags)
        as new arrays (flags None when flags is False); the arguments are not modified."""
        import numpy as np
        pts = np.ascontiguousarray(points, dtype=np.float32)
        S = pts.shape[0]
        pts = pts.reshape(S, -1, 3)
        cnt = np.ascontiguousarray(point_count, dtype=np.int32).reshape(S)
        sen = np.ascontiguousarray(sensor_origin, dtype=np.float64).reshape(S, 3)
        rob = np.ascontiguousarray(robot, dtype=np.float64).reshape(S, 3)
        grd = np.ascontiguousarray(grid, dtype=np.int32).reshape(S, 2)
        lay = np.array(layer, dtype=np.uint8).reshape(S, -1)
        lorg = np.array(layer_origin, dtype=np.float64).reshape(S, 2)
        org = np.array(origin, dtype=np.float64).reshape(S, 3)
        cst = np.array(cost, dtype=np.uint8).reshape(S, -1)
        status = np.zeros(S, np.int32)
        fl = np.zeros(S, np.int32) if flags else None
        a = abi.make_obstacle_layer_args(S, lay.shape[1], pts.shape[1], footprint, **params)
        a.points, a.point_count, a.sensor_origin, a.robot = abi.ptr(pts), abi.ptr(cnt), abi.ptr(sen), abi.ptr(rob)
        a.grid, a.layer, a.layer_origin, a.origin = abi.ptr(grd), abi.ptr(lay), abi.ptr(lorg), abi.ptr(org)
        a.cost, a.status, a.flags = abi.ptr(cst), abi.ptr(status), abi.ptr(fl)
        self._check(self.lib.tebgpu_costmap_obstacle_layer(self.ctx, C.byref(a)), "tebgpu_costmap_obstacle_layer")
        return lay, lorg, cst, org, status, fl

    def costmap_obstacle_layer_device(self, args, stream=None):
        """tebgpu_costmap_obstacle_layer_device: the same step over DEVICE memory (args: an abi.TebObstacleLayerArgs of
        device pointers, the footprint on the host; cost / grid / origin are the TebCostmapArgs arrays the costmap
        conversion and the costmap check read next). Stream ordered on `stream` (a cudaStream_t handle; None: the
        context's stream); does not synchronise."""
        self._check(self.lib.tebgpu_costmap_obstacle_layer_device(self.ctx, C.byref(args), stream),
                    "tebgpu_costmap_obstacle_layer_device")

    def obstacle_layer_max_cell_cap(self):
        """the largest cell_cap the obstacle layer takes: a robot's row in the opt-in shared memory of one CTA"""
        return self.info(21)

    def costmap_voxel_layer(self, points, point_count, sensor_origin, robot, grid, voxels, layer, layer_origin, origin,
                            cost, sources, footprint=None, flags=True, **params):
        """Every robot's voxel layer marked and cleared in 3-D from its sources' points (tebgpu_costmap_voxel_layer),
        host buffers, as include/teb_b200.h defines it at TebVoxelLayerArgs: points [S][K][P_cap][3] float32,
        point_count [S][K], sensor_origin [S][K][3], robot [S][3] (x, y, yaw), grid [S][2], voxels [S][cell_cap]
        uint32, layer [S][cell_cap] uint8 and layer_origin [S][2] (the previous cycle's), origin [S][3] and cost
        [S][cell_cap] (the master raster), sources: K TebObservationSource or dicts, footprint [F][2] or None; params:
        the other keywords of abi.make_voxel_layer_args. Returns (voxels, layer, layer_origin, cost, origin, status,
        flags) as new arrays (flags None when flags is False); the arguments are not modified."""
        import numpy as np
        K = len(sources)
        pts = np.ascontiguousarray(points, dtype=np.float32)
        S = pts.shape[0]
        pts = pts.reshape(S, K, -1, 3)
        cnt = np.ascontiguousarray(point_count, dtype=np.int32).reshape(S, K)
        sen = np.ascontiguousarray(sensor_origin, dtype=np.float64).reshape(S, K, 3)
        rob = np.ascontiguousarray(robot, dtype=np.float64).reshape(S, 3)
        grd = np.ascontiguousarray(grid, dtype=np.int32).reshape(S, 2)
        vox = np.array(voxels, dtype=np.uint32).reshape(S, -1)
        lay = np.array(layer, dtype=np.uint8).reshape(S, -1)
        lorg = np.array(layer_origin, dtype=np.float64).reshape(S, 2)
        org = np.array(origin, dtype=np.float64).reshape(S, 3)
        cst = np.array(cost, dtype=np.uint8).reshape(S, -1)
        status = np.zeros(S, np.int32)
        fl = np.zeros(S, np.int32) if flags else None
        a = abi.make_voxel_layer_args(S, lay.shape[1], pts.shape[2], sources, footprint, **params)
        a.points, a.point_count, a.sensor_origin, a.robot = abi.ptr(pts), abi.ptr(cnt), abi.ptr(sen), abi.ptr(rob)
        a.grid, a.voxels, a.layer, a.layer_origin = abi.ptr(grd), abi.ptr(vox), abi.ptr(lay), abi.ptr(lorg)
        a.origin, a.cost, a.status, a.flags = abi.ptr(org), abi.ptr(cst), abi.ptr(status), abi.ptr(fl)
        self._check(self.lib.tebgpu_costmap_voxel_layer(self.ctx, C.byref(a)), "tebgpu_costmap_voxel_layer")
        return vox, lay, lorg, cst, org, status, fl

    def costmap_voxel_layer_device(self, args, stream=None):
        """tebgpu_costmap_voxel_layer_device: the same step over DEVICE memory (args: an abi.TebVoxelLayerArgs of device
        pointers, the sources and the footprint on the host; cost / grid / origin are the TebCostmapArgs arrays the
        costmap conversion and the costmap check read next). Stream ordered on `stream` (a cudaStream_t handle; None:
        the context's stream); does not synchronise."""
        self._check(self.lib.tebgpu_costmap_voxel_layer_device(self.ctx, C.byref(args), stream),
                    "tebgpu_costmap_voxel_layer_device")

    def voxel_layer_max_cell_cap(self):
        """the largest cell_cap the voxel layer takes: a robot's voxel row, layer row and visited bits in the opt-in
        shared memory of one CTA"""
        return self.info(22)

    def local_plan(self, global_plan, plan_begin, plan_end, robot, robot_vel, grid, origin, P_cap, V_cap=None,
                   scene_id=None, via_count=None, infeasible_count=None, since_infeasible=None, costmap_to_plan=None,
                   plan_to_costmap=None, **scalars):
        """Each robot's local plan, goal and via-points from its global plan (tebgpu_local_plan), host buffers:
        global_plan [B][G_cap][3] (x, y, yaw), plan_begin / plan_end [B] (its live rows), robot [B][3], robot_vel [B][3]
        (vx, vy, omega), grid [S][2] and origin [S][3] of the costmaps, scene_id [B] (None: all 0). V_cap None: the
        via-points are the caller's own and via_count [B] (or None: 0) holds their counts; otherwise they are extracted
        into [B][V_cap][2]. infeasible_count / since_infeasible [B] or None. scalars: abi.make_local_plan_args' keywords.
        costmap_to_plan / plan_to_costmap [B][7] (both or neither, see abi.TebFrameArgs and abi.transform_from_se2): the
        global plans are in their own frame and robot in the costmap's (tebgpu_local_plan_tf).
        Returns a dict: plan_begin (moved by pruning), plan [B][P_cap][3] and via [B][V_cap][2] (NaN past the rows
        written), plan_count, goal_idx (-1 where not written), via_count, result (TEB_LOCAL_PLAN_*), needed [B][2]."""
        import numpy as np
        gp = np.ascontiguousarray(global_plan, dtype=np.float64)
        B, G_cap = gp.shape[0], gp.shape[1]
        i32 = lambda x, shape: np.ascontiguousarray(np.broadcast_to(x, shape), dtype=np.int32)
        f64 = lambda x, shape: np.ascontiguousarray(np.broadcast_to(x, shape), dtype=np.float64)
        out = dict(plan_begin=i32(plan_begin, (B,)).copy(), plan=np.full((B, int(P_cap), 3), np.nan),
                   plan_count=np.zeros(B, np.int32), goal_idx=np.full(B, -1, np.int32), result=np.full(B, -1, np.int32),
                   needed=np.zeros((B, 2), np.int32))
        own = V_cap is None
        out["via"] = None if own else np.full((B, int(V_cap), 2), np.nan)
        out["via_count"] = (np.zeros(B, np.int32) if via_count is None else i32(via_count, (B,)).copy()) if own else np.zeros(B, np.int32)
        grid = np.ascontiguousarray(grid, dtype=np.int32).reshape(-1, 2)
        S = grid.shape[0]
        keep = dict(pe=i32(plan_end, (B,)), rb=f64(robot, (B, 3)), rv=f64(robot_vel, (B, 3)),
                    org=f64(np.asarray(origin, np.float64).reshape(S, 3), (S, 3)),
                    sid=np.zeros(B, np.int32) if scene_id is None else i32(scene_id, (B,)),
                    inf=None if infeasible_count is None else i32(infeasible_count, (B,)),
                    since=None if since_infeasible is None else f64(since_infeasible, (B,)))
        c2p = None if costmap_to_plan is None else f64(costmap_to_plan, (B, 7))
        p2c = None if plan_to_costmap is None else f64(plan_to_costmap, (B, 7))
        la = abi.make_local_plan_args(G_cap, P_cap, 0 if own else V_cap, costmap_to_plan=abi.ptr(c2p),
                                      plan_to_costmap=abi.ptr(p2c), **scalars)
        la.global_plan, la.plan_begin, la.plan_end = abi.ptr(gp), abi.ptr(out["plan_begin"]), abi.ptr(keep["pe"])
        la.robot, la.robot_vel, la.grid, la.origin = abi.ptr(keep["rb"]), abi.ptr(keep["rv"]), abi.ptr(grid), abi.ptr(keep["org"])
        la.infeasible_count, la.since_infeasible = abi.ptr(keep["inf"]), abi.ptr(keep["since"])
        la.plan, la.plan_count, la.goal_idx = abi.ptr(out["plan"]), abi.ptr(out["plan_count"]), abi.ptr(out["goal_idx"])
        la.via, la.via_count = abi.ptr(out["via"]), (None if own and via_count is None else abi.ptr(out["via_count"]))
        la.result, la.needed = abi.ptr(out["result"]), abi.ptr(out["needed"])
        bs = abi.TebBatch()
        bs.B, bs.S, bs.scene_id = B, S, abi.ptr(keep["sid"])
        if la.frames is None:
            self._check(self.lib.tebgpu_local_plan(self.ctx, C.byref(bs), C.byref(la)), "tebgpu_local_plan")
        else:
            self._check(self.lib.tebgpu_local_plan_tf(self.ctx, C.byref(bs), C.byref(la), C.byref(la.frames)),
                        "tebgpu_local_plan_tf")
        return out

    def local_plan_device(self, batch_struct, args, stream=None, frames=None):
        """tebgpu_local_plan_device: the same step over DEVICE memory (batch_struct: an abi.TebBatch whose B, S and
        scene_id are read; args: an abi.TebLocalPlanArgs of device pointers, see abi.make_local_plan_args). Stream
        ordered on `stream` (a cudaStream_t handle; None: the context's stream); does not synchronise. frames: an
        abi.TebFrameArgs of device pointers, or None: the one make_local_plan_args kept on args (costmap_to_plan /
        plan_to_costmap), if any (tebgpu_local_plan_tf_device)."""
        if frames is None:
            frames = getattr(args, "frames", None)
        if frames is None:
            self._check(self.lib.tebgpu_local_plan_device(self.ctx, C.byref(batch_struct), C.byref(args), stream),
                        "tebgpu_local_plan_device")
        else:
            self._check(self.lib.tebgpu_local_plan_tf_device(self.ctx, C.byref(batch_struct), C.byref(args),
                                                             C.byref(frames), stream), "tebgpu_local_plan_tf_device")

    def last_local_plan_grid(self):
        """grid in CTAs (4 bands each) of the last local-plan launch, 0 before the first"""
        return self.info(16)

    def _cycle_host(self, fn, state, B, now, local_plan_result, scalars, bs, **arrays):
        """shared body of backup_modes / finish_cycle: copies the state, fills TebCycleArgs, calls `fn`"""
        import numpy as np
        i32 = lambda x, shape: None if x is None else np.ascontiguousarray(np.broadcast_to(x, shape), dtype=np.int32)
        out = {k: np.array(v, dtype=np.int32 if k in abi.CYCLE_STATE_INT else np.float64, order="C")
               for k, v in state.items()}
        L_cap = out["osc_ring"].shape[0]
        scalars.setdefault("buffer_length", L_cap)
        ca = abi.make_cycle_args(now, L_cap=L_cap, **scalars)
        keep = dict(lpr=i32(local_plan_result, (B,)))
        ca.local_plan_result = abi.ptr(keep["lpr"])
        for k in abi.CYCLE_STATE:
            setattr(ca, k, abi.ptr(out[k]) if out[k].size else None)
        for k, v in arrays.items():
            keep[k] = v
            setattr(ca, k, abi.ptr(v))
        self._check(fn(self.ctx, C.byref(bs), C.byref(ca)), fn.__name__)
        return out

    def backup_modes(self, state, robot_vel, now, local_plan_result=None, **scalars):
        """The oscillation half of configureBackupModes for every robot (tebgpu_backup_modes), host buffers. state: a
        dict as abi.make_cycle_state makes it (its osc_ring's first axis is L_cap); robot_vel [B][3] (vx, vy, omega);
        local_plan_result [B] TEB_LOCAL_PLAN_* or None (all PLANNED); scalars: abi.make_cycle_args' keywords
        (buffer_length defaults to L_cap). Returns a new state dict plus oscillating [B] (1 / 0, -2 where not written)."""
        import numpy as np
        B = len(state["prefer_rotdir"])
        osc = np.full(B, -2, np.int32)
        rv = np.ascontiguousarray(np.broadcast_to(robot_vel, (B, 3)), dtype=np.float64)
        bs = abi.TebBatch()
        bs.B = B
        out = self._cycle_host(self.lib.tebgpu_backup_modes, state, B, now, local_plan_result, scalars, bs,
                               robot_vel=rv, oscillating=osc)
        out["oscillating"] = osc
        return out

    def finish_cycle(self, state, n, status, chi2, cmd, now, feasible=None, local_plan_result=None, **scalars):
        """computeVelocityCommands from plan() on for every robot (tebgpu_finish_cycle), host buffers: n, status, chi2
        [B] of the planned batch, cmd [B][4] (TebPlanInput.cmd), feasible [B] or None (not checked), local_plan_result
        [B] or None (all PLANNED); state and scalars as for backup_modes. Returns a new state dict plus n [B] (0 where
        the planner was cleared), cmd_vel [B][3] and outcome [B] (TEB_CYCLE_*)."""
        import numpy as np
        B = len(state["prefer_rotdir"])
        i32 = lambda x: np.ascontiguousarray(np.broadcast_to(x, (B,)), dtype=np.int32).copy()
        res = dict(n=i32(n), cmd_vel=np.zeros((B, 3)), outcome=np.full(B, -1, np.int32))
        st, c2 = i32(status), np.ascontiguousarray(np.broadcast_to(chi2, (B,)), dtype=np.float64)
        cm = np.ascontiguousarray(np.broadcast_to(cmd, (B, 4)), dtype=np.float64)
        fz = None if feasible is None else i32(feasible)
        bs = abi.TebBatch()
        bs.B, bs.n, bs.status, bs.chi2 = B, abi.ptr(res["n"]), abi.ptr(st), abi.ptr(c2)
        out = self._cycle_host(self.lib.tebgpu_finish_cycle, state, B, now, local_plan_result, scalars, bs, cmd=cm,
                               feasible=fz, cmd_vel=res["cmd_vel"], outcome=res["outcome"])
        out.update(res)
        return out

    def backup_modes_device(self, batch_struct, args, stream=None):
        """tebgpu_backup_modes_device: the same step over DEVICE memory (batch_struct: an abi.TebBatch whose B is read;
        args: an abi.TebCycleArgs of device pointers, see abi.make_cycle_args). Stream ordered on `stream` (a
        cudaStream_t handle; None: the context's stream); does not synchronise."""
        self._check(self.lib.tebgpu_backup_modes_device(self.ctx, C.byref(batch_struct), C.byref(args), stream),
                    "tebgpu_backup_modes_device")

    def finish_cycle_device(self, batch_struct, args, stream=None):
        """tebgpu_finish_cycle_device: the same step over DEVICE memory (batch_struct: an abi.TebBatch whose B, n, status
        and chi2 are read; n is written). Stream ordered as backup_modes_device; does not synchronise."""
        self._check(self.lib.tebgpu_finish_cycle_device(self.ctx, C.byref(batch_struct), C.byref(args), stream),
                    "tebgpu_finish_cycle_device")

    def fleet_obstacles(self, pose, last_cmd, radius, custom, range, max_rows=8, own_count=None, custom_count=None,
                        world=None, scene=None):
        """The other robots of the fleet as custom obstacle rows of every robot's scene (tebgpu_fleet_obstacles), host
        buffers: pose [R][3] (x, y, theta in the custom obstacles' frame), last_cmd [R][3] (body vx, vy, omega: the
        controller state's last_cmd), radius [R], custom [S][C_cap] abi.OBST_DTYPE (the caller's own rows first),
        own_count [S] (None: 0), custom_count [S] (None: own_count; scenes no robot writes keep it), world / scene [R]
        (None: one world / scene r). Returns (custom [S][C_cap], a new array with the neighbour rows after each scene's
        own ones, custom_count [S], needed [R], status [R] TEB_FLEET_*)."""
        import numpy as np
        pose = np.ascontiguousarray(pose, dtype=np.float64).reshape(-1, 3)
        R = pose.shape[0]
        f64 = lambda x, shape: np.ascontiguousarray(np.broadcast_to(x, shape), dtype=np.float64)
        i32 = lambda x, shape: None if x is None else np.ascontiguousarray(np.broadcast_to(x, shape), dtype=np.int32)
        out = np.array(custom, dtype=abi.OBST_DTYPE, order="C")
        S = out.shape[0]
        out = out.reshape(S, -1)
        own = i32(own_count, (S,))
        cc = (np.zeros(S, np.int32) if own is None else own.copy()) if custom_count is None else i32(custom_count, (S,)).copy()
        keep = dict(cmd=f64(last_cmd, (R, 3)), rad=f64(radius, (R,)), world=i32(world, (R,)), scene=i32(scene, (R,)))
        needed, status = np.full(R, -2, np.int32), np.full(R, -1, np.int32)
        fa = abi.make_fleet_args(R, S, out.shape[1], max_rows, range, pose=pose, last_cmd=keep["cmd"], radius=keep["rad"],
                                 world=keep["world"], scene=keep["scene"], own_count=own,
                                 custom=out if out.size else None, custom_count=cc, needed=needed, status=status)
        self._check(self.lib.tebgpu_fleet_obstacles(self.ctx, C.byref(fa)), "tebgpu_fleet_obstacles")
        return out, cc, needed, status

    def fleet_obstacles_device(self, args, stream=None):
        """tebgpu_fleet_obstacles_device: the same step over DEVICE memory (args: an abi.TebFleetArgs of device
        pointers, see abi.make_fleet_args, which takes the fleet loop's tensors: the robot poses, the cycle state's
        last_cmd, and the costmap conversion's custom / custom_count). Stream ordered on `stream` (a cudaStream_t handle;
        None: the context's stream); does not synchronise."""
        self._check(self.lib.tebgpu_fleet_obstacles_device(self.ctx, C.byref(args), stream),
                    "tebgpu_fleet_obstacles_device")

    def fleet_publish(self, pose, last_cmd, radius, rows, first=0, world=None):
        """Robots r < R as rows first + r of a fleet table (tebgpu_fleet_publish), host buffers: pose [R][3], last_cmd
        [R][3], radius [R], world [R] (None: 0), rows [T] abi.FLEET_ROW_DTYPE. Returns a new array: rows with the
        robots' rows written."""
        import numpy as np
        pose = np.ascontiguousarray(pose, dtype=np.float64).reshape(-1, 3)
        R = pose.shape[0]
        out = np.array(rows, dtype=abi.FLEET_ROW_DTYPE, order="C").reshape(-1)
        keep = dict(cmd=np.ascontiguousarray(np.broadcast_to(last_cmd, (R, 3)), dtype=np.float64),
                    rad=np.ascontiguousarray(np.broadcast_to(radius, (R,)), dtype=np.float64),
                    world=None if world is None else np.ascontiguousarray(np.broadcast_to(world, (R,)), dtype=np.int32))
        fa = abi.make_fleet_args(R, 1, 0, 0, 0.0, pose=pose, last_cmd=keep["cmd"], radius=keep["rad"], world=keep["world"])
        tb = abi.make_fleet_table(len(out), first, out if out.size else None)
        self._check(self.lib.tebgpu_fleet_publish(self.ctx, C.byref(fa), C.byref(tb)), "tebgpu_fleet_publish")
        return out

    def fleet_publish_device(self, args, table, stream=None):
        """tebgpu_fleet_publish_device: args (abi.TebFleetArgs: R, pose, last_cmd, radius, world) and table
        (abi.TebFleetTable) of device pointers. Stream ordered on `stream` (None: the context's); does not synchronise."""
        self._check(self.lib.tebgpu_fleet_publish_device(self.ctx, C.byref(args), C.byref(table), stream),
                    "tebgpu_fleet_publish_device")

    def fleet_gather(self, rows, cap):
        """tebgpu_fleet_gather on a host table of world * cap rows: rank g's rows [g cap, (g + 1) cap) to every rank.
        Returns a new array (a copy of rows with one rank)."""
        import numpy as np
        out = np.array(rows, dtype=abi.FLEET_ROW_DTYPE, order="C").reshape(-1)
        tb = abi.make_fleet_table(len(out), 0, out if out.size else None)
        self._check(self.lib.tebgpu_fleet_gather(self.ctx, C.byref(tb), int(cap)), "tebgpu_fleet_gather")
        return out

    def fleet_gather_device(self, table, cap, stream=None):
        """tebgpu_fleet_gather_device: the in-place all-gather of a device table (abi.TebFleetTable) on the context's
        communicator, stream ordered on `stream` (None: the context's); nothing without a communicator"""
        self._check(self.lib.tebgpu_fleet_gather_device(self.ctx, C.byref(table), int(cap), stream),
                    "tebgpu_fleet_gather_device")

    def fleet_obstacles_table(self, rows, first, R, custom, range, max_rows=8, own_count=None, custom_count=None,
                              scene=None):
        """The neighbour rows of robots first .. first + R - 1 of a fleet table (tebgpu_fleet_obstacles_table), host
        buffers: rows [T] abi.FLEET_ROW_DTYPE, the rest as fleet_obstacles. Returns (custom, custom_count, needed,
        status)."""
        import numpy as np
        rows = np.ascontiguousarray(rows, dtype=abi.FLEET_ROW_DTYPE).reshape(-1)
        i32 = lambda x, shape: None if x is None else np.ascontiguousarray(np.broadcast_to(x, shape), dtype=np.int32)
        out = np.array(custom, dtype=abi.OBST_DTYPE, order="C")
        S = out.shape[0]
        out = out.reshape(S, -1)
        own = i32(own_count, (S,))
        cc = (np.zeros(S, np.int32) if own is None else own.copy()) if custom_count is None else i32(custom_count, (S,)).copy()
        sc = i32(scene, (int(R),))
        needed, status = np.full(int(R), -2, np.int32), np.full(int(R), -1, np.int32)
        fa = abi.make_fleet_args(R, S, out.shape[1], max_rows, range, scene=sc, own_count=own,
                                 custom=out if out.size else None, custom_count=cc, needed=needed, status=status)
        tb = abi.make_fleet_table(len(rows), first, rows if rows.size else None)
        self._check(self.lib.tebgpu_fleet_obstacles_table(self.ctx, C.byref(fa), C.byref(tb)),
                    "tebgpu_fleet_obstacles_table")
        return out, cc, needed, status

    def fleet_obstacles_table_device(self, args, table, stream=None):
        """tebgpu_fleet_obstacles_table_device: args (abi.TebFleetArgs; pose, last_cmd, radius and world are not read)
        and table (abi.TebFleetTable) of device pointers. Stream ordered on `stream` (None: the context's); does not
        synchronise."""
        self._check(self.lib.tebgpu_fleet_obstacles_table_device(self.ctx, C.byref(args), C.byref(table), stream),
                    "tebgpu_fleet_obstacles_table_device")

    def fleet_obstacles_shaped(self, kinds, kind, pose, last_cmd, custom, range, max_rows=8, own_count=None,
                               custom_count=None, world=None, scene=None, custom_vertices=None, own_vertex_count=None,
                               select=abi.TEB_FLEET_SELECT_CENTRES):
        """fleet_obstacles with every neighbour written as its kind's footprint (tebgpu_fleet_obstacles_shaped), host
        buffers: kinds the shape library (abi.make_fleet_shapes' list), kind [R] each robot's kind, custom_vertices
        [S][PV_cap][2] the scenes' vertex pools (None: PV_cap 0), own_vertex_count [S] (None: 0), select the neighbour
        rule (abi.TEB_FLEET_SELECT_*; footprints need set_params); the rest as fleet_obstacles. Returns (custom,
        custom_count, needed, status, custom_vertices), new arrays."""
        import numpy as np
        pose = np.ascontiguousarray(pose, dtype=np.float64).reshape(-1, 3)
        R = pose.shape[0]
        i32 = lambda x, shape: None if x is None else np.ascontiguousarray(np.broadcast_to(x, shape), dtype=np.int32)
        out = np.array(custom, dtype=abi.OBST_DTYPE, order="C")
        S = out.shape[0]
        out = out.reshape(S, -1)
        cv = np.zeros((S, 0, 2)) if custom_vertices is None else np.array(custom_vertices, np.float64, order="C").reshape(S, -1, 2)
        own = i32(own_count, (S,))
        cc = (np.zeros(S, np.int32) if own is None else own.copy()) if custom_count is None else i32(custom_count, (S,)).copy()
        keep = dict(cmd=np.ascontiguousarray(np.broadcast_to(last_cmd, (R, 3)), dtype=np.float64), world=i32(world, (R,)),
                    scene=i32(scene, (R,)), kind=i32(kind, (R,)), ownv=i32(own_vertex_count, (S,)))
        needed, status = np.full(R, -2, np.int32), np.full(R, -1, np.int32)
        fa = abi.make_fleet_args(R, S, out.shape[1], max_rows, range, pose=pose, last_cmd=keep["cmd"], world=keep["world"],
                                 scene=keep["scene"], own_count=own, custom=out if out.size else None, custom_count=cc,
                                 needed=needed, status=status)
        sh = abi.make_fleet_shapes(kinds, cv.shape[1], select, kind=keep["kind"], own_vertex_count=keep["ownv"],
                                   custom_vertices=cv if cv.size else None)
        self._check(self.lib.tebgpu_fleet_obstacles_shaped(self.ctx, C.byref(fa), C.byref(sh)),
                    "tebgpu_fleet_obstacles_shaped")
        return out, cc, needed, status, cv

    def fleet_obstacles_shaped_device(self, args, shapes, stream=None):
        """tebgpu_fleet_obstacles_shaped_device: args (abi.TebFleetArgs, radius not read) and the per-robot arrays of
        shapes (abi.make_fleet_shapes: kind, own_vertex_count, custom_vertices) of device pointers. Stream ordered on
        `stream` (None: the context's); does not synchronise."""
        self._check(self.lib.tebgpu_fleet_obstacles_shaped_device(self.ctx, C.byref(args), C.byref(shapes), stream),
                    "tebgpu_fleet_obstacles_shaped_device")

    def fleet_publish_shaped(self, kinds, kind, pose, last_cmd, radius, rows, heading, row_kind, first=0, world=None):
        """fleet_publish with the table's companions (tebgpu_fleet_publish_shaped), host buffers: heading [T] float64
        and row_kind [T] int32 get the robots' headings and kinds at first .. first + R - 1. Returns new (rows, heading,
        row_kind)."""
        import numpy as np
        pose = np.ascontiguousarray(pose, dtype=np.float64).reshape(-1, 3)
        R = pose.shape[0]
        out = np.array(rows, dtype=abi.FLEET_ROW_DTYPE, order="C").reshape(-1)
        hd = np.array(heading, np.float64, order="C").reshape(-1)
        rk = np.array(row_kind, np.int32, order="C").reshape(-1)
        keep = dict(cmd=np.ascontiguousarray(np.broadcast_to(last_cmd, (R, 3)), dtype=np.float64),
                    rad=np.ascontiguousarray(np.broadcast_to(radius, (R,)), dtype=np.float64),
                    world=None if world is None else np.ascontiguousarray(np.broadcast_to(world, (R,)), dtype=np.int32),
                    kind=np.ascontiguousarray(np.broadcast_to(kind, (R,)), dtype=np.int32))
        fa = abi.make_fleet_args(R, 1, 0, 0, 0.0, pose=pose, last_cmd=keep["cmd"], radius=keep["rad"], world=keep["world"])
        sh = abi.make_fleet_shapes(kinds, 0, kind=keep["kind"], heading=hd if hd.size else None,
                                   row_kind=rk if rk.size else None)
        tb = abi.make_fleet_table(len(out), first, out if out.size else None)
        self._check(self.lib.tebgpu_fleet_publish_shaped(self.ctx, C.byref(fa), C.byref(sh), C.byref(tb)),
                    "tebgpu_fleet_publish_shaped")
        return out, hd, rk

    def fleet_publish_shaped_device(self, args, shapes, table, stream=None):
        """tebgpu_fleet_publish_shaped_device: args, shapes (kind, heading, row_kind) and table of device pointers.
        Stream ordered on `stream` (None: the context's); does not synchronise."""
        self._check(self.lib.tebgpu_fleet_publish_shaped_device(self.ctx, C.byref(args), C.byref(shapes), C.byref(table),
                                                                stream), "tebgpu_fleet_publish_shaped_device")

    def fleet_gather_shaped(self, kinds, rows, heading, row_kind, cap):
        """tebgpu_fleet_gather_shaped on a host table and its companions. Returns new (rows, heading, row_kind)."""
        import numpy as np
        out = np.array(rows, dtype=abi.FLEET_ROW_DTYPE, order="C").reshape(-1)
        hd = np.array(heading, np.float64, order="C").reshape(-1)
        rk = np.array(row_kind, np.int32, order="C").reshape(-1)
        sh = abi.make_fleet_shapes(kinds, 0, heading=hd if hd.size else None, row_kind=rk if rk.size else None)
        tb = abi.make_fleet_table(len(out), 0, out if out.size else None)
        self._check(self.lib.tebgpu_fleet_gather_shaped(self.ctx, C.byref(sh), C.byref(tb), int(cap)),
                    "tebgpu_fleet_gather_shaped")
        return out, hd, rk

    def fleet_gather_shaped_device(self, shapes, table, cap, stream=None):
        """tebgpu_fleet_gather_shaped_device: the in-place all-gather of a device table and its companions (shapes'
        heading and row_kind) as one NCCL group; nothing without a communicator"""
        self._check(self.lib.tebgpu_fleet_gather_shaped_device(self.ctx, C.byref(shapes), C.byref(table), int(cap), stream),
                    "tebgpu_fleet_gather_shaped_device")

    def fleet_obstacles_table_shaped(self, kinds, rows, heading, row_kind, first, R, custom, range, max_rows=8,
                                     own_count=None, custom_count=None, scene=None, custom_vertices=None,
                                     own_vertex_count=None, select=abi.TEB_FLEET_SELECT_CENTRES):
        """fleet_obstacles_table with every neighbour written as its kind's footprint
        (tebgpu_fleet_obstacles_table_shaped), host buffers: heading [T], row_kind [T] the table's companions, the rest
        as fleet_obstacles_shaped / fleet_obstacles_table. Returns (custom, custom_count, needed, status,
        custom_vertices)."""
        import numpy as np
        rows = np.ascontiguousarray(rows, dtype=abi.FLEET_ROW_DTYPE).reshape(-1)
        hd = np.ascontiguousarray(heading, np.float64).reshape(-1)
        rk = np.ascontiguousarray(row_kind, np.int32).reshape(-1)
        i32 = lambda x, shape: None if x is None else np.ascontiguousarray(np.broadcast_to(x, shape), dtype=np.int32)
        out = np.array(custom, dtype=abi.OBST_DTYPE, order="C")
        S = out.shape[0]
        out = out.reshape(S, -1)
        cv = np.zeros((S, 0, 2)) if custom_vertices is None else np.array(custom_vertices, np.float64, order="C").reshape(S, -1, 2)
        own = i32(own_count, (S,))
        cc = (np.zeros(S, np.int32) if own is None else own.copy()) if custom_count is None else i32(custom_count, (S,)).copy()
        sc, ownv = i32(scene, (int(R),)), i32(own_vertex_count, (S,))
        needed, status = np.full(int(R), -2, np.int32), np.full(int(R), -1, np.int32)
        fa = abi.make_fleet_args(R, S, out.shape[1], max_rows, range, scene=sc, own_count=own,
                                 custom=out if out.size else None, custom_count=cc, needed=needed, status=status)
        sh = abi.make_fleet_shapes(kinds, cv.shape[1], select, own_vertex_count=ownv, custom_vertices=cv if cv.size else None,
                                   heading=hd if hd.size else None, row_kind=rk if rk.size else None)
        tb = abi.make_fleet_table(len(rows), first, rows if rows.size else None)
        self._check(self.lib.tebgpu_fleet_obstacles_table_shaped(self.ctx, C.byref(fa), C.byref(sh), C.byref(tb)),
                    "tebgpu_fleet_obstacles_table_shaped")
        return out, cc, needed, status, cv

    def fleet_obstacles_table_shaped_device(self, args, shapes, table, stream=None):
        """tebgpu_fleet_obstacles_table_shaped_device: args, shapes (own_vertex_count, custom_vertices, heading,
        row_kind) and table of device pointers. Stream ordered on `stream` (None: the context's); does not
        synchronise."""
        self._check(self.lib.tebgpu_fleet_obstacles_table_shaped_device(self.ctx, C.byref(args), C.byref(shapes),
                                                                        C.byref(table), stream),
                    "tebgpu_fleet_obstacles_table_shaped_device")

    def last_fleet_grid(self):
        """grid in CTAs (16 robots each) of the last fleet-obstacle launch, 0 before the first"""
        return self.info(18)

    FLEET_SEARCHES = {abi.TEBGPU_FLEET_SEARCH_ALL_PAIRS: "all_pairs", abi.TEBGPU_FLEET_SEARCH_GRID: "grid",
                      abi.TEBGPU_FLEET_SEARCH_ONE_BUCKET: "one_bucket"}

    def set_fleet_search(self, mode):
        """neighbour search of the fleet steps (abi.TEBGPU_FLEET_SEARCH_*): 0 automatic (default), 1 all pairs, 2 the
        grid, 3 the grid with every cell in one bucket. Every mode writes the same bytes."""
        self._check(self.lib.tebgpu_set_fleet_search(self.ctx, int(mode)), "tebgpu_set_fleet_search")

    def last_fleet_search(self):
        """the search the last fleet step ran: one of FLEET_SEARCHES' names, or None before the first"""
        return self.FLEET_SEARCHES.get(self.info(abi.TEBGPU_INFO_FLEET_SEARCH))

    def last_cycle_grid(self):
        """grid in CTAs (128 bands each) of the last backup-modes or finish-cycle launch, 0 before the first"""
        return self.info(17)

    FEAS_BUILDS = {0: "staged", 1: "global", 2: "costmap"}   # TEBGPU_FEAS_BUILD_*

    def last_feasibility_check(self):
        """(build, grid in CTAs) of the last feasibility-check launch: build is one of FEAS_BUILDS' names, or None
        before the first launch"""
        return self.FEAS_BUILDS.get(self.info(13)), self.info(12)

    def plan_kernel_times(self):
        """{kernel name: (total ms, launches)} of k_plan_begin and k_velocity_command since profiling was enabled"""
        ms, cnt = (C.c_double * 2)(), (C.c_int64 * 2)()
        self._check(self.lib.tebgpu_get_plan_kernel_times(self.ctx, C.byref(ms), C.byref(cnt)), "tebgpu_get_plan_kernel_times")
        return {"k_plan_begin": (ms[0], cnt[0]), "k_velocity_command": (ms[1], cnt[1])}

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
        # the 2-D rows are (Re, Im) pairs: viewed, not composed as Re + 1j * Im, which turns an infinite Im into a NaN Re
        return out if three_d else out.view(np.complex128)[:, 0].copy()

    def hsig_factors(self, hb):
        """every scene's factor table of the 2-D signature (tebgpu_hsig_factors) from hb's obstacle tables:
        (factor [S][M_cap][2] float64, factor_exp [S][M_cap] int32, factor_count [S] int32)"""
        import numpy as np
        f = (np.zeros((hb.S, hb.M_cap, 2)), np.zeros((hb.S, hb.M_cap), np.int32), np.zeros(hb.S, np.int32))
        bs = hb.struct()
        fs = abi.make_hsig_factors(*(x.ctypes.data for x in f))
        self._check(self.lib.tebgpu_hsig_factors(self.ctx, C.byref(bs), C.byref(fs)), "tebgpu_hsig_factors")
        return f

    def h_signature_scenes(self, hb, factors=None, use_timediffs=True):
        """h_signature for scenes of up to 16384 obstacles (tebgpu_h_signature_scenes), same return shapes. factors: the
        tuple hsig_factors returned for hb's scenes, or None: the table is built in the call"""
        import numpy as np
        three_d = bool(self.params.include_dynamic_obstacles) if hasattr(self, "params") else False
        out = np.zeros((hb.B, max(hb.M_cap, 1) if three_d else 2))
        bs = hb.struct()
        fs = None
        if factors is not None:
            f = [np.ascontiguousarray(x, dtype=dt) for x, dt in zip(factors, (np.float64, np.int32, np.int32))]
            fs = C.byref(abi.make_hsig_factors(*(x.ctypes.data for x in f)))
        self._check(self.lib.tebgpu_h_signature_scenes(self.ctx, C.byref(bs), fs, int(use_timediffs), out.ctypes.data),
                    "tebgpu_h_signature_scenes")
        return out if three_d else out.view(np.complex128)[:, 0].copy()

    def hsig_factors_device(self, batch_struct, factors, stream=None):
        """tebgpu_hsig_factors_device: the factor tables over DEVICE memory (batch_struct: an abi.TebBatch of device
        pointers, of which S, M_cap, obstacles and obst_count are read; factors: an abi.TebHsigFactors of device
        pointers). Stream ordered on `stream` (a cudaStream_t handle; None: the context's stream); does not synchronise."""
        self._check(self.lib.tebgpu_hsig_factors_device(self.ctx, C.byref(batch_struct), C.byref(factors), stream),
                    "tebgpu_hsig_factors_device")

    def h_signature_scenes_device(self, batch_struct, h_out, factors=None, use_timediffs=True, stream=None):
        """tebgpu_h_signature_scenes_device: the signatures over DEVICE memory into h_out (a device address or a tensor
        of B x 2 or B x max(M_cap, 1) float64). factors: an abi.TebHsigFactors of device pointers, or None: built in
        the call. Stream ordered as hsig_factors_device; does not synchronise."""
        out = h_out.data_ptr() if hasattr(h_out, "data_ptr") else h_out
        fs = None if factors is None else C.byref(factors)
        self._check(self.lib.tebgpu_h_signature_scenes_device(self.ctx, C.byref(batch_struct), fs, int(use_timediffs),
                                                              out, stream), "tebgpu_h_signature_scenes_device")

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
