"""Multi-GPU frame sharding: one process per GPU, CPI frames are independent units.

The reference parallelises over CPI frames implicitly (one dask chunk = one frame on a
thread pool, ``main.py:169-194``); nothing couples frames on the hot path.  So the N-GPU
layout is: frame ``f`` of the stream belongs to rank ``f % world`` (or a contiguous range),
each rank runs its own ``FramePipeline``, and the only data that ever moves between ranks is
*input staging* when a single ingest rank holds the IQ stream:

* ``scatter_frames``      ingest rank sends each rank its own (ref, srv) frames (1/G of the data
                          per link) -- ``torch.distributed.scatter``, NCCL over NVLink on GPUs
* ``broadcast_reference`` all ranks need the same reference-channel block (one illuminator,
                          several surveillance channels / overlapped windows) -- one NCCL broadcast
* ``gather_maps``         optional: range-Doppler maps (0.6 MB/frame) back to the ingest rank

There is no reduction, no all-to-all and no collective inside the timed compute path; when
every rank reads or synthesises its own frames there is no communication at all.  The same
code runs on CPU tensors with the ``gloo`` backend (tests/test_distributed_cpu.py).
"""
from __future__ import annotations

import numpy as np


def shard_indices(nframes: int, rank: int, world: int, mode: str = "interleaved") -> np.ndarray:
    """Frame indices owned by ``rank``.  ``interleaved``: f % world == rank (keeps ranks in
    lock-step on a live stream); ``contiguous``: equal consecutive ranges (overlapped CPIs
    re-read only a half-CPI halo)."""
    if not (0 <= rank < world):
        raise ValueError("rank out of range")
    if mode == "interleaved":
        return np.arange(rank, nframes, world)
    if mode == "contiguous":
        base, extra = divmod(nframes, world)
        start = rank * base + min(rank, extra)
        return np.arange(start, start + base + (1 if rank < extra else 0))
    raise ValueError(f"unknown sharding mode {mode!r}")


def _as_real(t):
    import torch
    return torch.view_as_real(t) if t.is_complex() else t


def scatter_frames(ref_frames, srv_frames, nframes, n, src=0, device=None, mode="interleaved", group=None):
    """Ingest rank ``src`` holds ``(nframes, n)`` complex64 tensors; every rank returns its shard
    ``(ref_local, srv_local, indices)``.  Other ranks pass ``None`` for the frames."""
    import torch
    import torch.distributed as dist
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    idx = shard_indices(nframes, rank, world, mode)
    counts = [len(shard_indices(nframes, r, world, mode)) for r in range(world)]
    width = max(counts) if counts else 0
    dev = device if device is not None else (ref_frames.device if ref_frames is not None else torch.device("cpu"))
    out = []
    for frames in (ref_frames, srv_frames):
        recv = torch.zeros((width, n), dtype=torch.complex64, device=dev)
        chunks = None
        if rank == src:
            chunks = []
            for r in range(world):
                ids = torch.as_tensor(shard_indices(nframes, r, world, mode), device=frames.device)
                c = torch.zeros((width, n), dtype=torch.complex64, device=dev)
                if len(ids):
                    c[: len(ids)] = frames.index_select(0, ids).to(dev)
                chunks.append(_as_real(c).contiguous())
        dist.scatter(_as_real(recv), chunks, src=src, group=group)
        out.append(recv[: len(idx)])
    return out[0], out[1], idx


def broadcast_reference(ref_block, src=0, group=None):
    """In-place broadcast of the reference-channel block (complex64 tensor) from ``src``."""
    import torch.distributed as dist
    dist.broadcast(_as_real(ref_block), src=src, group=group)
    return ref_block


def gather_maps(maps_local, nframes, src=0, mode="interleaved", group=None):
    """Collect per-rank maps ``(nlocal, F, R+1)`` on ``src`` in stream order; others get ``None``."""
    import torch
    import torch.distributed as dist
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    counts = [len(shard_indices(nframes, r, world, mode)) for r in range(world)]
    width = max(counts) if counts else 0
    shape = (width,) + tuple(maps_local.shape[1:])
    send = torch.zeros(shape, dtype=maps_local.dtype, device=maps_local.device)
    send[: maps_local.shape[0]] = maps_local
    bufs = None
    if rank == src:
        bufs = [torch.zeros_like(_as_real(send)) for _ in range(world)]
    dist.gather(_as_real(send).contiguous(), bufs, dst=src, group=group)
    if rank != src:
        return None
    full = torch.zeros((nframes,) + tuple(maps_local.shape[1:]), dtype=maps_local.dtype, device=maps_local.device)
    for r in range(world):
        ids = shard_indices(nframes, r, world, mode)
        if len(ids):
            got = torch.view_as_complex(bufs[r]) if maps_local.is_complex() else bufs[r]
            full[torch.as_tensor(ids, device=full.device)] = got[: len(ids)]
    return full


def process_stream(process_local, ref_frames, srv_frames, nframes, n, src=0, device=None,
                   mode="interleaved", gather=True, group=None):
    """scatter -> ``process_local(ref_local, srv_local) -> maps_local`` -> (optional) gather.

    ``process_local`` is ``lambda r, s: pipe.run_device(r, s, out)`` on a GPU rank; the CPU
    tests pass a stand-in so the plumbing is exercised with gloo."""
    ref_l, srv_l, idx = scatter_frames(ref_frames, srv_frames, nframes, n, src, device, mode, group)
    maps_l = process_local(ref_l, srv_l)
    if not gather:
        return maps_l, idx
    return gather_maps(maps_l, nframes, src, mode, group), idx


def stream_frames(source, process, nframes_total, chunk, n, rank, world, device, src=0):
    """Config-3 staging: a stream of ``nframes_total`` CPI frames is held by the ingest rank ``src``; frame ``f`` belongs
    to rank ``f % world``.  The ingest rank sends every other rank its (ref, srv) frames in chunks of ``chunk`` frames
    with point-to-point operations (NCCL over NVLink / NVSwitch on GPUs, gloo in the CPU tests); on CUDA devices the
    transfers run on a side stream into two alternating buffers while the main stream computes the previous chunk.

    ``source(ids) -> (ref, srv)``   ingest rank only: tensors ``(len(ids), n)`` complex64 on ``device`` for global frame ids
    ``process(ref, srv, first)``    every rank: consume a chunk whose first LOCAL frame index is ``first`` (enqueue only)

    This is the traffic the dask graph's chunk staging (main.py:169-194, overlap at :178-181) turns into when the
    chunks live on different GPUs.  Returns the number of local frames processed."""
    import torch
    import torch.distributed as dist
    cuda = torch.device(device).type == "cuda"
    per_rank = len(shard_indices(nframes_total, rank, world))
    counts = [len(shard_indices(nframes_total, r, world)) for r in range(world)]
    nchunks = -(-max(counts) // chunk) if counts else 0
    side = torch.cuda.Stream(device=device) if cuda else None
    main = torch.cuda.current_stream(device) if cuda else None
    bufs = None
    if rank != src:
        bufs = [(torch.empty((chunk, n), dtype=torch.complex64, device=device), torch.empty((chunk, n), dtype=torch.complex64, device=device))
                for _ in range(2)]
    ready = [torch.cuda.Event() for _ in range(2)] if cuda else None      # staging of buffer k complete
    freed = [torch.cuda.Event() for _ in range(2)] if cuda else None      # compute on buffer k complete

    def ids_of(r, c):
        lo, hi = c * chunk, min((c + 1) * chunk, counts[r])
        return [k * world + r for k in range(lo, hi)]

    def stage(c):
        if rank == src:
            ops, keep = [], []
            for r in range(world):
                ids = ids_of(r, c)
                if r == src or not ids:
                    continue
                rr, ss = source(ids)
                keep.append((rr, ss))
                ops.append(dist.P2POp(dist.isend, _as_real(rr), r))
                ops.append(dist.P2POp(dist.isend, _as_real(ss), r))
            if ops:
                for w in dist.batch_isend_irecv(ops):
                    w.wait()
        else:
            m = len(ids_of(rank, c))
            if m:
                k = c & 1
                if cuda and c >= 2:
                    side.wait_event(freed[k])
                rb, sb = bufs[k]
                for w in dist.batch_isend_irecv([dist.P2POp(dist.irecv, _as_real(rb[:m]), src),
                                                 dist.P2POp(dist.irecv, _as_real(sb[:m]), src)]):
                    w.wait()
                if cuda:
                    ready[k].record(side)

    def compute(c):
        ids = ids_of(rank, c)
        if not ids:
            return
        if rank == src:
            rr, ss = source(ids)
            process(rr, ss, c * chunk)
        else:
            k = c & 1
            if cuda:
                main.wait_event(ready[k])
            rb, sb = bufs[k]
            process(rb[:len(ids)], sb[:len(ids)], c * chunk)
            if cuda:
                freed[k].record(main)

    for c in range(nchunks + 1):
        if c < nchunks:
            if cuda:
                with torch.cuda.stream(side):
                    stage(c)
            else:
                stage(c)
        if c >= 1:
            compute(c - 1)
    if cuda:
        main.wait_stream(side)
    return per_rank


def stream_benchmark(pipe, ref_d, srv_d, maps_d, nframes_total, chunk, rank, world, device, src=0):
    """Time :func:`stream_frames` with the rank's FramePipeline: the ingest rank's resident frames stand in for the
    stream (frame f reads resident frame f mod resident).  Returns (rank 0) whole-job frames/s INCLUDING the staging, the
    bytes the ingest rank sent and its egress bandwidth; time = max over ranks of the device time of one pass."""
    import torch
    import torch.distributed as dist
    n = ref_d.shape[1]
    res = ref_d.shape[0]
    nmaps = maps_d.shape[0]

    def source(ids):
        o = ids[0] % max(1, res - len(ids) + 1)          # a contiguous run of distinct resident frames (no gather copy)
        return ref_d[o:o + len(ids)], srv_d[o:o + len(ids)]

    def process(rr, ss, first):
        o = first % max(1, nmaps - rr.shape[0] + 1)
        pipe.run_device(rr, ss, maps_d[o:o + rr.shape[0]])

    main = torch.cuda.current_stream(device)
    stream_frames(source, process, nframes_total, chunk, n, rank, world, device, src)       # warm-up (NCCL channels)
    torch.cuda.synchronize(device)
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(main)
    local = stream_frames(source, process, nframes_total, chunk, n, rank, world, device, src)
    e1.record(main)
    torch.cuda.synchronize(device)
    t = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t.item())
    if rank != 0:
        return None
    sent = (nframes_total - local) * 2 * n * 8
    return {"frames": nframes_total, "value": nframes_total / (ms * 1e-3), "unit": "frames/s", "ms": round(ms, 3),
            "chunk_frames": chunk, "ingest_rank_sent_bytes": sent, "ingest_egress_GBps": round(sent / (ms * 1e-3) / 1e9, 1),
            "staging": "NCCL point-to-point (batch_isend_irecv) from rank 0 on a side stream, two alternating buffers per rank",
            "note": "frame f -> rank f % world; rank 0 holds the stream in HBM and also computes its own share; the limiter is "
                    "rank 0's NVLink egress when ingest_egress_GBps approaches its peer-copy bandwidth"}
