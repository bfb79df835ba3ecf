"""Multi-GPU driver (one process per GPU).  The path shards by read (SURVEY §8e); the only exchange is the final merge
that replaces Stats::merge / FilterResult::merge (src/stats.cpp:1013-1082, src/filterresult.cpp:28-61, called from
src/seprocessor.cpp:108-121).

GPU path: the merge is the C ABI's own (include/fplgpu.h: fpl_comm_init + fpl_allreduce_stats — ncclAllReduce on the
context's stream); torch.distributed is only the out-of-band channel that carries rank 0's 128-byte rendezvous id and
gathers the per-read records.  The same shard / gather logic runs on gloo with host blocks in the CPU tests.

gather_engine is the other merge: every rank's whole state (fpl_state_export: both Stats blocks, the counters and the per-read
lists) travels to one rank over the torch.distributed group, which merges the images (fpl_state_merge) and so can write the
job's HTML report as well as its JSON one."""
import numpy as np
import torch
import torch.distributed as dist

from .pack import shard_reads_by_bases


def shard(batch, rank, world_size):
    """This rank's contiguous share of the batch, balanced by bases (SURVEY §8e)."""
    bounds = shard_reads_by_bases(batch.lens, world_size)
    return batch.slice(bounds[rank], bounds[rank + 1]), bounds


def agree_on_cycles(local_cycles, device=None, group=None):
    """All ranks pad their Stats blocks to the same number of cycles before the all-reduce (host blocks / gloo)."""
    t = torch.tensor([int(local_cycles)], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return int(t.item())


def allreduce_in_place(blocks, group=None):
    """Sum-all-reduce every accumulator block (int64 tensors) in place (host blocks / gloo)."""
    for b in blocks:
        dist.all_reduce(b, op=dist.ReduceOp.SUM, group=group)


def init_engine_comm(engine, rank=None, world_size=None, group=None):
    """Join `engine` (binding.Engine) to the job's NCCL communicator: rank 0 makes the id, everybody receives it
    over the existing torch.distributed group (any backend), every rank calls fpl_comm_init."""
    from .binding import Engine
    rank = dist.get_rank(group) if rank is None else rank
    world_size = dist.get_world_size(group) if world_size is None else world_size
    box = [Engine.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(box, src=0, group=group)
    engine.comm_init(box[0], rank, world_size)


def merge_engine(engine, cycles=0):
    """Stats::merge / FilterResult::merge over the ranks, in place on the device, on the engine's stream.
    cycles = 0 agrees on the longest read first (one small synchronous all-reduce)."""
    engine.allreduce_stats(cycles)


def gather_records(records, bounds, rank, world_size, group=None):
    """Concatenate per-rank record arrays in rank order == input order (contiguous shards)."""
    out = [None] * world_size
    dist.all_gather_object(out, np.asarray(records), group=group)
    return np.concatenate(out)


def gather_engine(engine, root=0, group=None):
    """Stats::merge / FilterResult::merge of every rank's engine into `root`'s, in rank order, read lists included: each rank
    exports its state, the images travel to `root` over the torch.distributed group (CUDA uint8 tensors on NCCL, host tensors
    on any other backend), and `root` merges them (fpl_state_merge).  With contiguous shards (shard()) `root` then holds the
    whole job: its report_json / report_html are those of one engine over the unsharded input.  The other ranks' engines are
    not changed.  A refusal (other options or adapters on some rank) raises FplError with `root`'s own state in its engine."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    root_global = root if group is None else dist.get_global_rank(group, root)
    dev = torch.device("cuda", engine.options.device) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    mine = engine.export_state()
    sizes = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(sizes, torch.tensor([len(mine)], dtype=torch.int64, device=dev), group=group)
    sizes = [int(n.item()) for n in sizes]
    buf = torch.zeros(max(sizes), dtype=torch.uint8, device=dev)      # gather takes equal shapes: the image, then zeros
    buf[:len(mine)] = torch.frombuffer(bytearray(mine), dtype=torch.uint8).to(dev)
    bufs = [torch.empty_like(buf) for _ in range(world)] if rank == root else None
    dist.gather(buf, bufs, dst=root_global, group=group)
    if rank != root:
        return
    images = [b[:n].cpu().numpy() for b, n in zip(bufs, sizes)]
    if root == 0:
        engine.merge_state(*images[1:])
        return
    # root's own state goes in its rank's place: start from nothing, and put it back if an image is refused
    engine.reset()
    try:
        engine.merge_state(*images)
    except Exception:
        engine.merge_state(images[root])
        raise
