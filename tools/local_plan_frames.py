"""The local-plan step and the costmap conversion with and without frames: tebgpu_local_plan_device against
tebgpu_local_plan_tf_device (each robot's global plan in its own frame), tebgpu_costmap_obstacles_device against
tebgpu_costmap_obstacles_tf_device (each scene's custom obstacles in their own frame), over N robots / scenes. With frames each robot's plan is given in its own map frame (a planar map -> odom per robot)
and the variant must cut the same rows as the plan given in odom (same_cut_fraction). CUDA events
around --reps launches after --warmup launches, all on one explicit stream (the launches, the events and the plan_begin
reset between launches); the variants alternate trial by trial and each reports the median of its --trials trials.

    python tools/local_plan_frames.py --robots 1024 8192 [--json out.json]

Prints the card name and its power limit beside the numbers (nvidia-smi, read-only query)."""
import argparse
import json
import os
import statistics
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import teb_local_planner_b200 as T  # noqa: E402
from teb_local_planner_b200 import abi, scenes  # noqa: E402
from tools.local_plan import card  # noqa: E402


def timed(torch, stream, variants, warmup, reps, trials):
    """variants: {name: fn} launching on `stream`; -> {name: median µs per launch}, the variants alternating per trial"""
    torch.cuda.synchronize()   # the inputs were written on the default stream
    with torch.cuda.stream(stream):
        for fn in variants.values():
            for _ in range(warmup):
                fn()
        stream.synchronize()
        out = {k: [] for k in variants}
        for _ in range(trials):
            for name, fn in variants.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(reps):
                    fn()
                e1.record(stream)
                e1.synchronize()
                out[name].append(e0.elapsed_time(e1) * 1e3 / reps)
    return {k: statistics.median(v) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--robots", type=int, nargs="+", default=[1024, 8192])
    ap.add_argument("--rows", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=1000)
    ap.add_argument("--trials", type=int, default=7)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda:0")
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    res = dict(card=card(), rows=a.rows, runs=[])
    for B in a.robots:
        S, P_cap, V_cap, C_cap, PV, M_cap = B, 128, 32, 8, 32, 2048
        d = scenes.global_plans(B, a.rows, S=4, seed=7)
        g = T.TebGpu(B, 64, S, M_cap, V_cap, max_obst_vertices=PV)
        g.set_params(abi.default_params())
        # each robot's map -> odom, and its plan moved into map (the planar form of doTransform), so that both variants
        # cut the same rows
        mo = np.stack([0.01 * np.arange(B), -0.02 * np.arange(B), 0.001 * np.arange(B)], 1)
        pair = [abi.transform_from_se2(*m) for m in mo]
        gpl = d["global_plan"].copy()
        cth, sth = np.cos(mo[:, 2])[:, None], np.sin(mo[:, 2])[:, None]
        x, y = d["global_plan"][..., 0], d["global_plan"][..., 1]
        gpl[..., 0] = cth * x - sth * y + mo[:, :1]
        gpl[..., 1] = sth * x + cth * y + mo[:, 1:2]
        gpl[..., 2] = d["global_plan"][..., 2] + mo[:, 2:3]
        gp_odom, gp_map = t(d["global_plan"]), t(gpl)
        gp, begin, end = gp_odom, t(d["plan_begin"]), t(d["plan_end"])
        robot, vel, grid, origin = t(d["robot"]), t(d["robot_vel"]), t(d["grid"]), t(d["origin"])
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
        plan, pcount, via, vcount = z((B, P_cap, 3), torch.float64), z(B, torch.int32), z((B, V_cap, 2), torch.float64), \
            z(B, torch.int32)
        result, gidx = z(B, torch.int32), z(B, torch.int32)
        c2p, p2c = t(np.array([p[0] for p in pair])), t(np.array([p[1] for p in pair]))
        la = abi.make_local_plan_args(a.rows, P_cap, V_cap, viapoint_sep=0.3, global_plan=gp_odom.data_ptr(),
                                      plan_begin=begin.data_ptr(), plan_end=end.data_ptr(), robot=robot.data_ptr(),
                                      robot_vel=vel.data_ptr(), grid=grid.data_ptr(), origin=origin.data_ptr(),
                                      plan=plan.data_ptr(), plan_count=pcount.data_ptr(), goal_idx=gidx.data_ptr(),
                                      via=via.data_ptr(), via_count=vcount.data_ptr(), result=result.data_ptr())
        bs = abi.TebBatch()
        sid = t(np.arange(B, dtype=np.int32) % 4)
        bs.B, bs.S, bs.scene_id = B, 4, sid.data_ptr()
        fr = abi.make_frame_args(costmap_to_plan=c2p.data_ptr(), plan_to_costmap=p2c.data_ptr())
        stream = torch.cuda.Stream()
        st = stream.cuda_stream
        saved = begin.clone()

        la_map = abi.make_local_plan_args(a.rows, P_cap, V_cap, viapoint_sep=0.3)
        for f_, _ in la._fields_:
            setattr(la_map, f_, getattr(la, f_))
        la_map.global_plan = gp_map.data_ptr()

        def lp(frames):
            begin.copy_(saved)   # the same cut every launch (pruning moves plan_begin), on the launch's stream
            g.local_plan_device(bs, la if frames is None else la_map, stream=st, frames=frames)

        def outcome(frames):
            with torch.cuda.stream(stream):
                lp(frames)
            stream.synchronize()
            return result.cpu().numpy().copy(), pcount.cpu().numpy().copy(), begin.cpu().numpy().copy()

        torch.cuda.synchronize()
        o_null, o_tf = outcome(None), outcome(fr)
        same = float(np.mean((o_null[0] == o_tf[0]) & (o_null[1] == o_tf[1]) & (o_null[2] == o_tf[2])))

        tl = timed(torch, stream, dict(null=lambda: lp(None), tf=lambda: lp(fr), copy=lambda: begin.copy_(saved)),
                   a.warmup, a.reps, a.trials)
        lp_null, lp_tf, copy_only = tl["null"], tl["tf"], tl["copy"]
        # costmap conversion: 60 x 60 rasters, C_cap custom rows per scene (a point, a circle, lines, polygons)
        r = scenes.costmap_raster(S, 60, 60, 0.05, 0.03, seed=3)
        rows = np.zeros((S, C_cap), abi.OBST_DTYPE)
        verts = np.random.default_rng(1).uniform(-3, 3, (S, PV, 2))
        rows["type"][:] = [0, 1, 2, 2, 4, 4, 0, 1]
        rows["vertex_begin"][:] = [0, 0, 0, 2, 4, 10, 0, 0]
        rows["vertex_count"][:] = [0, 0, 2, 2, 6, 8, 0, 0]
        ctf = t(np.array([p[1] for p in pair]))
        cost, cgrid, corigin, crobot = t(r["cost"]), t(r["grid"]), t(r["origin"]), t(r["robot"])
        cu, cc, cv = t(rows.view(np.uint8)), t(np.full(S, C_cap, np.int32)), t(verts)
        obst, ocount, ov = z(S * M_cap * 64, torch.uint8), z(S, torch.int32), z((S, PV, 2), torch.float64)
        ca = abi.TebCostmapArgs()
        ca.S, ca.cell_cap, ca.M_cap, ca.C_cap, ca.include_costmap_obstacles = S, r["cost"].shape[1], M_cap, C_cap, 1
        ca.behind_robot_dist = 1.5
        ca.cost, ca.grid, ca.origin, ca.robot = cost.data_ptr(), cgrid.data_ptr(), corigin.data_ptr(), crobot.data_ptr()
        ca.custom, ca.custom_count = cu.data_ptr(), cc.data_ptr()
        ca.obstacles, ca.obst_count = obst.data_ptr(), ocount.data_ptr()
        cf = abi.make_frame_args(custom_to_costmap=ctf.data_ptr(), custom_vertices=cv.data_ptr(),
                                 obst_vertices=ov.data_ptr(), PV_cap=PV)
        tc = timed(torch, stream, dict(null=lambda: g.costmap_obstacles_device(ca, stream=st),
                                       tf=lambda: g.costmap_obstacles_device(ca, stream=st, frames=cf)),
                   a.warmup, a.reps, a.trials)
        cm_null, cm_tf = tc["null"], tc["tf"]
        taken = int(o_null[1].sum())
        run = dict(robots=B, same_cut_fraction=same, local_plan_us=lp_null - copy_only, local_plan_tf_us=lp_tf - copy_only, reset_us=copy_only,
                   rows_written=taken, costmap_us=cm_null, costmap_tf_us=cm_tf, custom_rows=S * C_cap,
                   window_ms=dict(local_plan=lp_null * a.reps / 1e3, costmap=cm_null * a.reps / 1e3))
        res["runs"].append(run)
        print(json.dumps(run))
        g.close()
    print(json.dumps(dict(card=res["card"])))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
