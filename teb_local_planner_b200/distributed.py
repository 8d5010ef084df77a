"""Multi-GPU plumbing: one process per GPU, the batch axis (candidates x requests) sharded contiguously, ONE
all-gather of the per-candidate costs per plan, then HomotopyClassPlanner::selectBestTeb on the gathered costs
(reference src/homotopy_class_planner.cpp:466-493 fan-out, :564-616 selection). Bands never exchange data during
optimisation (SURVEY.md par. 8e), so there is no data-path collective.

The collective itself lives BEHIND the C-ABI (tebgpu_comm_init / tebgpu_gather_costs: ncclAllGather on the context's
stream, include/teb_b200.h). This module only
  * splits the batch axis (`shard_range`),
  * bootstraps the communicator: rank 0 creates the 128-byte NCCL id, `torch.distributed` (any backend) carries it to
    the other ranks (`init_comm`) - the same job MPI or a file would do for a C++ host,
  * restates selectBestTeb for whole request batches (`select_best_per_request`),
  * offers the same gather over a torch process group for CPU tests (`gather_costs_torch`, gloo),
  * lays out the fleet table of a sharded fleet (`fleet_layout`) and gathers it over a torch process group
    (`gather_fleet_table_torch`, with the shaped steps' heading / row_kind companions), as tebgpu_fleet_gather(_shaped)
    does over NCCL.
"""
import ctypes as C

import numpy as np


def shard_range(B, rank, world):
    """Contiguous split of the batch axis: rank g owns bands [lo, hi). Sizes differ by at most one."""
    base, rem = divmod(B, world)
    lo = rank * base + min(rank, rem)
    hi = lo + base + (1 if rank < rem else 0)
    return lo, hi


def shard_requests(requests, rank, world):
    """Requests are never split across ranks when their count allows it (selection of one request then needs no
    remote candidate, the gather is still done so that every rank knows every winner)."""
    return shard_range(requests, rank, world)


def init_comm(gpu, rank, world, device=None):
    """Collective: creates the NCCL communicator of `gpu` (a TebGpu context) across the ranks of the default torch process
    group. rank 0 draws the unique id through the C-ABI; torch.distributed only transports those 128 bytes."""
    import torch
    import torch.distributed as dist
    ident = np.zeros(128, np.uint8)
    if rank == 0:
        gpu.comm_get_unique_id(ident)
    t = torch.from_numpy(ident)
    if device is not None:
        t = t.to(device)
    dist.broadcast(t, src=0)
    ident = t.cpu().numpy().copy()
    gpu.comm_init(ident, world, rank)
    return gpu


def gather_costs_torch(local_cost, world=None, group=None):
    """The same all-gather over a torch process group (gloo on CPU): used by the CPU tests of the N > 1 host logic.
    Shards must have equal length. Returns the [world * len] tensor."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group) if world is None else world
    out = torch.empty(world * local_cost.numel(), dtype=local_cost.dtype, device=local_cost.device)
    dist.all_gather_into_tensor(out, local_cost.contiguous(), group=group)
    return out


def select_best(cost, last_best=-1, initial_plan=-1, hysteresis=1.0, prefer_initial=0.95):
    """selectBestTeb on one request's candidate costs (strict '<', first minimum wins)."""
    best, min_cost = -1, np.finfo(np.float64).max
    for i, c in enumerate(cost):
        if i == last_best:
            c = c * hysteresis
        elif i == initial_plan:
            c = c * prefer_initial
        if c < min_cost:
            best, min_cost = i, c
    return best


def select_best_per_request(all_cost, candidates, params=None, last_best=None, initial_plan=None):
    """all_cost: [requests * candidates] gathered costs. Returns the winning candidate index per request."""
    all_cost = np.asarray(all_cost, dtype=np.float64).reshape(-1, candidates)
    hyst = 1.0 if params is None else params.selection_cost_hysteresis
    pref = 0.95 if params is None else params.selection_prefer_initial_plan
    out = np.empty(all_cost.shape[0], np.int32)
    for r in range(all_cost.shape[0]):
        lb = -1 if last_best is None else int(last_best[r])
        ip = -1 if initial_plan is None else int(initial_plan[r])
        out[r] = select_best(all_cost[r], lb, ip, hyst, pref)
    return out


def fleet_layout(counts, world):
    """The fleet table of a fleet whose rank g holds counts[g] robots: every rank's shard padded to cap rows (NCCL has no
    all-gather-v), so the table has T = world * cap rows and rank g's robots are rows first[g] .. first[g] + counts[g] - 1.
    Returns (cap, first per rank)."""
    counts = [int(c) for c in counts]
    if len(counts) != world or min(counts) < 0:
        raise ValueError("one non-negative robot count per rank")
    cap = max(1, max(counts))
    return cap, [g * cap for g in range(world)]


def gather_fleet_table_torch(rows, cap, rank, world=None, group=None, heading=None, row_kind=None):
    """tebgpu_fleet_gather over a torch process group (gloo on CPU): rows is the rank's [world * cap] fleet table
    (abi.FLEET_ROW_DTYPE numpy array) with its shard at rows [rank cap, (rank + 1) cap); returns the gathered table.
    heading / row_kind (the shaped steps' companions, [world * cap] float64 / int32): gathered too, as
    tebgpu_fleet_gather_shaped does, and the return is (rows, heading, row_kind)."""
    import torch
    import torch.distributed as dist
    from . import abi
    world = dist.get_world_size(group) if world is None else world

    def gather(a, dtype):
        a = np.ascontiguousarray(a, dtype=dtype).reshape(-1)
        if len(a) != world * cap:
            raise ValueError("the fleet table must have world * cap rows")
        mine = torch.from_numpy(a[rank * cap:(rank + 1) * cap].copy().view(np.uint8))
        out = torch.empty(world * mine.numel(), dtype=torch.uint8)
        dist.all_gather_into_tensor(out, mine, group=group)
        return out.numpy().view(dtype).copy()

    table = gather(rows, abi.FLEET_ROW_DTYPE)
    if heading is None and row_kind is None:
        return table
    return table, gather(heading, np.float64), gather(row_kind, np.int32)
