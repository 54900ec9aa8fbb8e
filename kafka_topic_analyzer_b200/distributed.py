"""Multi-GPU merge: one process per GPU, partitions sharded gpu = partition mod G (SURVEY.md §8 e),
no data-path collective during the scan, ONE NCCL all-reduce (SUM over u64) at the end for every
counter / histogram / extremum / HLL register, plus — only with -c — an all-gather of the compacted
alive-key stamps (NCCL has no OR / no 64-bit max over a 32 GiB table; last-writer-wins by global seq is
associative and commutative, so re-applying every rank's (hash, stamp) list on every rank is exact).

torch.distributed is plumbing here; the pack/unpack kernels are in csrc/kta_kernels.cuh."""
from __future__ import annotations

from .metrics import KtaEngine


def allreduce_merge(engine: KtaEngine, group=None, counters_only: bool = False) -> None:
    """After this, every rank's engine holds the merged state (call finalize() to read it).
    counters_only skips the exact alive-key exchange (used to time the all-reduce part alone)."""
    import torch
    import torch.distributed as dist

    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if world == 1:
        return
    dev = torch.device("cuda", torch.cuda.current_device())
    words = engine.merge_words(world)
    buf = torch.empty(words, dtype=torch.int64, device=dev)   # u64 payload; SUM is bit-identical on i64
    # When the engine runs on torch's current stream (engine.set_stream) the three steps are ordered by that
    # stream alone — export kernel, NCCL all-reduce, import kernel — with no host synchronisation in between.
    engine.merge_export(rank, world, buf)
    dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    if not engine.shares_caller_stream:
        torch.cuda.current_stream().synchronize()
    engine.merge_import(world, buf)
    if engine.hot_keys_top_k and not counters_only:
        allgather_hot_keys(engine, group)
    if engine.count_alive_keys and not counters_only:
        n_local = engine.alive_export_count()
        counts = torch.zeros(world, dtype=torch.int64, device=dev)
        counts[rank] = n_local
        dist.all_reduce(counts, op=dist.ReduceOp.SUM, group=group)
        cap = int(counts.max().item())
        if cap == 0:
            return
        h_loc = torch.zeros(cap, dtype=torch.int32, device=dev)
        s_loc = torch.zeros(cap, dtype=torch.int64, device=dev)
        engine.alive_export(h_loc, s_loc, cap)
        h_all = torch.empty(world * cap, dtype=torch.int32, device=dev)
        s_all = torch.empty(world * cap, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(h_all, h_loc, group=group)
        dist.all_gather_into_tensor(s_all, s_loc, group=group)
        torch.cuda.current_stream().synchronize()
        cl = counts.tolist()
        for r in range(world):
            if r != rank and cl[r]:
                engine.alive_import(h_all[r * cap:], s_all[r * cap:], int(cl[r]))


def allgather_hot_keys(engine: KtaEngine, group=None) -> None:
    """Makes every rank's hot-key table topic-wide: each rank exports its entries (88 bytes each, include/kta.h
    kta_hot_key), the counts and then the entries are all-gathered, and each rank imports the other ranks' entries.  The
    table cannot travel in the SUM buffer: its entries are keyed by id, in no fixed order."""
    import torch
    import torch.distributed as dist
    from ._native import HOT_KEY_DTYPE

    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if world == 1:
        return
    dev = torch.device("cuda", torch.cuda.current_device())
    counts = torch.zeros(world, dtype=torch.int64, device=dev)
    counts[rank] = engine.hot_keys_export_count()
    dist.all_reduce(counts, op=dist.ReduceOp.SUM, group=group)
    cl = counts.tolist()
    cap = max(cl)
    if cap == 0:
        return
    size = HOT_KEY_DTYPE.itemsize
    loc = torch.zeros(cap * size, dtype=torch.uint8, device=dev)
    engine.hot_keys_export(loc, cap)
    every = torch.empty(world * cap * size, dtype=torch.uint8, device=dev)
    dist.all_gather_into_tensor(every, loc, group=group)
    torch.cuda.current_stream().synchronize()
    for r in range(world):
        if r != rank and cl[r]:
            engine.hot_keys_import(every[r * cap * size:], int(cl[r]))


# ---------------------------------------------------------------------------------------------------
# Host-side statement of the merge-buffer layout (what merge_export_kernel / merge_import_kernel do on the
# device, csrc/kta_kernels.cuh).  Used by the gloo CPU tests of the N>1 logic and usable for host-side merges.
#   [ sums (nsums u64) | world × 4 extrema slots | world × (nhll/8) words, eight one-byte registers per word
#     | timeline (3 × P × (B + 2) u64, only when the timeline is on)
#     | partitioner check ((2C + 1) × P u64, only when the check is on) ]
# Every rank fills only its own slots, so ONE SUM all-reduce hands every rank's values to every rank.  The timeline and
# partitioner segments are summed as they are (a sharded rank's foreign rows are zero); every rank must use the same
# timeline and check the same partition counts.
# ---------------------------------------------------------------------------------------------------
def merge_words(nsums: int, nhll: int, world: int, timeline_words: int = 0, partitioner_words: int = 0) -> int:
    return nsums + world * 4 + world * (nhll // 8) + timeline_words + partitioner_words


def pack_merge_buffer(sums, minmax, hll, rank: int, world: int, timeline=None, partitioner=None):
    """sums u64[nsums]; minmax = (min_ts i64, max_ts i64, min_size u64, max_size u64); hll u32[nhll];
    timeline: None, or the u64 [3][P][B + 2] arrays (any shape; taken flat); partitioner: None, or the u64 [2C + 1][P]
    partitioner-check counters (any shape; taken flat)."""
    import numpy as np
    nsums, nhll = len(sums), len(hll)
    tl = None if timeline is None else np.asarray(timeline, dtype=np.uint64).ravel()
    pt = None if partitioner is None else np.asarray(partitioner, dtype=np.uint64).ravel()
    tw = 0 if tl is None else tl.size
    buf = np.zeros(merge_words(nsums, nhll, world, tw, 0 if pt is None else pt.size), dtype=np.uint64)
    buf[:nsums] = np.asarray(sums, dtype=np.uint64)
    mm = np.array([minmax[0], minmax[1]], dtype=np.int64).view(np.uint64)
    buf[nsums + 4 * rank: nsums + 4 * rank + 2] = mm
    buf[nsums + 4 * rank + 2] = np.uint64(minmax[2])
    buf[nsums + 4 * rank + 3] = np.uint64(minmax[3])
    if nhll:
        hw = nhll // 8
        regs = np.asarray(hll, dtype=np.uint8)
        o = nsums + 4 * world + rank * hw
        buf[o:o + hw] = regs.view(np.uint64) if regs.flags["C_CONTIGUOUS"] else np.ascontiguousarray(regs).view(np.uint64)
    if tl is not None:
        buf[merge_words(nsums, nhll, world):merge_words(nsums, nhll, world, tw)] = tl
    if pt is not None:
        buf[merge_words(nsums, nhll, world, tw):] = pt
    return buf


def fold_merge_buffer(buf, nsums: int, nhll: int, world: int, timeline_words: int = 0, partitioner_words: int = 0):
    """inverse of pack after the SUM all-reduce: returns (sums, (min_ts, max_ts, min_size, max_size), hll), and the
    flat timeline segment as a fourth element when timeline_words > 0.  With partitioner_words > 0 the result has five
    elements: the timeline segment (empty without a timeline), then the flat partitioner-check segment."""
    import numpy as np
    sums = buf[:nsums].copy()
    mm = buf[nsums:nsums + 4 * world].reshape(world, 4)
    tmin = int(mm[:, 0].copy().view(np.int64).min())
    tmax = int(mm[:, 1].copy().view(np.int64).max())
    smin, smax = int(mm[:, 2].min()), int(mm[:, 3].max())
    hll = np.zeros(nhll, dtype=np.uint32)
    if nhll:
        hw = nhll // 8
        w = np.ascontiguousarray(buf[nsums + 4 * world:nsums + 4 * world + world * hw]).view(np.uint8).reshape(world, nhll)
        hll[:] = w.max(axis=0)
    base = merge_words(nsums, nhll, world)
    tl = np.asarray(buf[base:base + timeline_words], dtype=np.uint64).copy()
    if partitioner_words:
        pt = np.asarray(buf[base + timeline_words:base + timeline_words + partitioner_words], dtype=np.uint64).copy()
        return sums, (tmin, tmax, smin, smax), hll, tl, pt
    if timeline_words:
        return sums, (tmin, tmax, smin, smax), hll, tl
    return sums, (tmin, tmax, smin, smax), hll
