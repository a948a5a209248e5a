"""Utterance sharding over GPUs (one process per GPU, `torch.distributed`).

The generation path is embarrassingly parallel over utterances (SURVEY.md section 8e): rank r owns a contiguous
slice of the global batch, the Philox noise is keyed by the GLOBAL utterance index (so the result is independent of
the number of ranks), and the only collective is the final gather of the outputs.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_bounds(n_items: int, world: int, rank: int) -> tuple[int, int]:
    """Contiguous, balanced: the first `n_items % world` ranks get one extra row."""
    if not 0 <= rank < world:
        raise ValueError('rank out of range')
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def all_gather_rows(local: torch.Tensor, n_items: int, group=None) -> torch.Tensor:
    """Gathers ragged row-shards `[rows_r, ...]` into `[n_items, ...]` on every rank (pads to the largest shard)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return local
    rank = dist.get_rank(group)
    sizes = [shard_bounds(n_items, world, r) for r in range(world)]
    biggest = max(hi - lo for lo, hi in sizes)
    pad = torch.zeros((biggest,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    # ship raw bytes: gloo has no int16 all_gather, and NCCL does not care
    raw = pad.contiguous().view(torch.uint8).reshape(biggest, -1)
    bufs = [torch.empty_like(raw) for _ in range(world)]
    dist.all_gather(bufs, raw, group=group)
    parts = [b.view(local.dtype).reshape((biggest,) + tuple(local.shape[1:]))[: hi - lo] for b, (lo, hi) in zip(bufs, sizes)]
    return torch.cat(parts, dim=0)


def generate_sharded(generate_fn, mels, seed: int, group=None, **kw):
    """Runs `generate_fn(mels[lo:hi], seed=seed, utterance_offset=lo, **kw)` on this rank's slice of the GLOBAL batch
    `mels [B, feat, T]` and all-gathers the int16 labels.  `generate_fn` is `WaveRNNEngine.generate` of a RAW engine."""
    if getattr(getattr(generate_fn, '__self__', None), 'mode', 'RAW') == 'MOL':
        raise ValueError('sharded generation gathers int16 labels and is RAW only; run a MOL engine per GPU without sharding')
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    n = mels.shape[0]
    lo, hi = shard_bounds(n, world, rank)
    nccl = dist.is_initialized() and dist.get_backend(group) == 'nccl'
    dev = torch.device('cuda', torch.cuda.current_device()) if nccl else torch.device('cpu')
    labels = generate_fn(mels[lo:hi], seed=seed, utterance_offset=lo, **kw)['labels'] if hi > lo else None
    if world > n:
        # fewer utterances than ranks: some ranks have nothing to generate (the engine requires B >= 1) but every rank must
        # still take part in the collectives -- agree on the row width, then contribute a zero-row shard
        width = torch.tensor([labels.shape[1] if labels is not None else 0], dtype=torch.int64, device=dev)
        dist.all_reduce(width, op=dist.ReduceOp.MAX, group=group)
        if labels is None:
            labels = torch.zeros((0, int(width.item())), dtype=torch.int16, device=dev)
    return all_gather_rows(labels, n, group), (lo, hi)
