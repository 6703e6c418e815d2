"""Batch sharding across the GPUs of one box (SURVEY.md §8e): the utterance
batch is split contiguously over ranks, every rank runs the identical single-GPU
pipeline, and ONE exchange — a gather of the wav shards to the destination rank
over NCCL/NVLink (grouped send/recv) — assembles the result in global utterance
order.  Only the destination receives data; the other ranks send their shard and
return ``None``.  The exchange is issued per batch chunk on a side stream while
the last layer of the next chunk is still computing (``tail_events`` of the
generator), so all but the last chunk's transfer hides under compute.  The
reference has no equivalent (each accelerate rank writes its own files and
mis-indexes the uids, models/vocoders/vocoder_inference.py:360, SURVEY Q13)."""
from __future__ import annotations

import inspect

import torch
import torch.distributed as dist


def shard_bounds(n_items: int, world_size: int, rank: int):
    """Contiguous split; the first ``n_items % world_size`` ranks get one extra item."""
    base, extra = divmod(n_items, world_size)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def _chunk_bounds(n: int, chunks: int, i: int):
    """Chunk i of n items, the split `ab_generator_set_tail_events` uses: [n*i/chunks, n*(i+1)/chunks)."""
    return n * i // chunks, n * (i + 1) // chunks


def _supports(fn, name):
    try:
        return name in inspect.signature(fn).parameters
    except (TypeError, ValueError):
        return False


def gather_shards(local, n_items, world_size, rank, group=None, dst=0, out=None, chunk=None):
    """Gather ragged shards (sizes differ by at most one, possibly empty) to ``dst`` in global order.

    ``local``: this rank's shard [n_local, ...] (``None`` or empty when it has no items).  On ``dst`` the result
    [n_items, ...] is returned (``out`` if given — the destination's own shard may already sit in it); other ranks
    return ``None``.  ``chunk=(i, n)`` restricts the exchange to chunk i of n of every rank's shard.
    Every rank decides from (n_items, world_size) alone, so ranks with no items never block the others."""
    lo, hi = shard_bounds(n_items, world_size, rank)
    ops = []
    if rank == dst:
        if out is None:
            if local is None:
                raise ValueError("gather_shards: the destination needs `out` when it holds no items")
            out = torch.empty((n_items,) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
        for r in range(world_size):
            rlo, rhi = shard_bounds(n_items, world_size, r)
            if chunk is not None:
                a, b = _chunk_bounds(rhi - rlo, chunk[1], chunk[0])
                rlo, rhi = rlo + a, rlo + b
            if rhi <= rlo:
                continue
            if r == dst:
                if local is not None and out[rlo:rhi].data_ptr() != local[rlo - lo: rhi - lo].data_ptr():
                    out[rlo:rhi].copy_(local[rlo - lo: rhi - lo])
            else:
                ops.append(dist.P2POp(dist.irecv, out[rlo:rhi], _global_rank(group, r), group=group))
    elif hi > lo:
        a, b = (0, hi - lo) if chunk is None else _chunk_bounds(hi - lo, chunk[1], chunk[0])
        if b > a:
            ops.append(dist.P2POp(dist.isend, local[a:b].contiguous(), _global_rank(group, dst), group=group))
    works = dist.batch_isend_irecv(ops) if ops else []
    return (out if rank == dst else None), works


def _global_rank(group, group_rank):
    return group_rank if group is None else dist.get_global_rank(group, group_rank)


def sharded_vocoder_forward(model, mels, group=None, dst=0, chunks=4):
    """mels: the GLOBAL batch [B, n_mel, T] (every rank holds it or at least its own slice filled in).
    Returns wav [B, 1, T*hop] on rank ``dst`` and ``None`` elsewhere (ranks without items just skip).

    The generator writes the destination's own shard straight into the gathered tensor; on CUDA the transfer of
    chunk i overlaps the last layer of chunk i+1 (side stream + the generator's ``tail_events``)."""
    ws = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    if ws == 1:
        return model(mels)
    lo, hi = shard_bounds(mels.shape[0], ws, rank)
    return _sharded_forward(model, mels[lo:hi], mels.shape[0], rank, ws, group, dst, chunks)


def sharded_vocoder_inference(cfg, model, mels_local, n_global, group=None, dst=0, device=None, chunks=4):
    """The multi-GPU form of ``vocoder_inference`` (models/vocoders/gan/gan_vocoder_inference.py:11-38): every
    rank passes ITS shard of the batch (``shard_bounds(n_global, world, rank)``, host or device, any strides), runs
    the generator on it and the wav shards are gathered to ``dst``, which returns the reference's result type —
    a detached CPU tensor [n_global, T*hop] in global utterance order; the other ranks return ``None``."""
    ws = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    model.eval()
    with torch.no_grad():
        if device is None:
            device = next(model.parameters()).device
        mels_local = mels_local.to(device, non_blocking=True)
        wav = model(mels_local) if ws == 1 else _sharded_forward(model, mels_local, n_global, rank, ws, group, dst, chunks)
        if ws > 1 and rank != dst:
            return None
        wav = wav.squeeze(1).detach()
        if not wav.is_cuda:
            return wav
        # a pinned buffer is still a CPU tensor and lets the D2H copy run at full PCIe rate
        host = torch.empty(wav.shape, dtype=wav.dtype, pin_memory=True)
        host.copy_(wav, non_blocking=True)
        torch.cuda.current_stream(wav.device).synchronize()
        return host


def _sharded_forward(model, mel_local, B, rank, ws, group, dst, chunks):
    lo, hi = shard_bounds(B, ws, rank)
    if mel_local.shape[0] != hi - lo:
        raise ValueError(f"rank {rank} holds {mel_local.shape[0]} utterances, its shard of {B} has {hi - lo}")
    fwd = model.forward if hasattr(model, "forward") else model
    use_events = mel_local.is_cuda and _supports(fwd, "tail_events") and chunks > 1
    use_out = _supports(fwd, "out")
    out = local = None
    events = [torch.cuda.Event() for _ in range(chunks)] if use_events else None
    kw = {"tail_events": events} if use_events else {}
    if rank == dst:
        hop = _hop_of(model)
        if hop is not None:
            out = torch.empty((B, 1, mel_local.shape[-1] * hop), device=mel_local.device, dtype=torch.float32)
        if hi > lo:
            if out is not None and use_out:
                local = model(mel_local, out=out[lo:hi], **kw)
            else:
                local = model(mel_local, **kw)
        elif out is None:
            raise ValueError("sharded forward: a destination rank without items needs a model with cfg.preprocess.hop_size")
    elif hi > lo:
        local = model(mel_local, **kw)
    if not use_events:
        res, works = gather_shards(local, B, ws, rank, group, dst, out=out)
        for w in works:
            w.wait()
        return res
    # chunked exchange on a side stream: chunk i is sent / received as soon as its event fired
    main = torch.cuda.current_stream(mel_local.device)
    side = _side_stream(mel_local.device)
    res, all_works = out, []
    with torch.cuda.stream(side):
        if hi <= lo:
            side.wait_stream(main)
        for i in range(chunks):
            if hi > lo:
                side.wait_event(events[i])
            res, works = gather_shards(local, B, ws, rank, group, dst, out=res if rank == dst else None, chunk=(i, chunks))
            all_works += works
        for w in all_works:
            w.wait()
    main.wait_stream(side)
    for t in (local, out):
        if t is not None:
            t.record_stream(side)
    return res if rank == dst else None


_side_streams = {}


def _side_stream(device):
    key = str(device)
    if key not in _side_streams:
        _side_streams[key] = torch.cuda.Stream(device=device)
    return _side_streams[key]


def _hop_of(model):
    """Samples per mel frame: cfg.preprocess.hop_size, else the model's ``hop_length`` (Vocos, built from
    cfg.model.vocos), else None."""
    try:
        return int(model.cfg.preprocess.hop_size)
    except AttributeError:
        hop = getattr(model, "hop_length", None)
        return None if hop is None else int(hop)
