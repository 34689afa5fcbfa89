"""Rank-level sharding of the path (one process per GPU, torch.distributed).

Signatures are independent, so a batch shards into contiguous ranges with no data-path collective;
quorum counting is independent per instance, so votes shard BY INSTANCE (all votes of an instance on
one rank).  The only exchange is the final gather of the bit-packed verdict mask (n/8 bytes) and, for
the quorum stream, of the per-instance reached bits — `ncclAllGather` over NVLink on a GPU box, gloo
in the CPU tests.  Mirrors the device-level sharding inside libsbv.so (csrc/shards.h: shard_range,
quorum_shards, unpack_shards; engine.cu: shard_out, gather_unpack)."""
from __future__ import annotations

import numpy as np


def shard_range(n: int, rank: int, world: int):
    """Contiguous range [lo, hi) of rank `rank` — same rule as shards.h shard_range()."""
    return n * rank // world, n * (rank + 1) // world


def shard_instances(instance_ids: np.ndarray, n_instances: int, rank: int, world: int):
    """Boolean mask of the votes owned by `rank`: instances are range-partitioned, so every vote of
    an instance lands on the same rank and the distinct-signer count stays local."""
    lo, hi = shard_range(n_instances, rank, world)
    return (instance_ids >= lo) & (instance_ids < hi), lo, hi


def shard_votes(instance_ids: np.ndarray, n_instances: int, rank: int, world: int):
    """Vote range [vlo, vhi), instance range [ilo, ihi) and the SHARD-LOCAL instance ids of rank `rank` for a vote stream
    grouped by non-decreasing instance id (the input contract of sbv_verify_quorum, whose instance ids count from 0 on
    every engine).  The last rank also takes trailing votes whose instance id is out of range (padding)."""
    ilo, ihi = shard_range(n_instances, rank, world)
    vlo = int(np.searchsorted(instance_ids, ilo, "left"))
    vhi = instance_ids.size if rank == world - 1 else int(np.searchsorted(instance_ids, ihi, "left"))
    return vlo, vhi, ilo, ihi, (instance_ids[vlo:vhi] - np.uint32(ilo)).astype(np.uint32)


def words_per_shard(n: int, world: int) -> int:
    return (((n + world - 1) // world) + 31) // 32


def pack_bits(ok: np.ndarray, n_words: int) -> np.ndarray:
    """Verdict bytes -> uint32 words, bit i of word i/32 (k_pack_bits layout), zero padded."""
    bits = np.zeros(n_words * 32, np.uint8)
    bits[: ok.size] = ok != 0
    return np.packbits(bits.reshape(-1, 32)[:, ::-1], axis=1).view(">u4").astype(np.uint32).reshape(-1)


def unpack_bits(words: np.ndarray, n: int) -> np.ndarray:
    w = np.asarray(words, dtype=np.uint32)
    bits = ((w[:, None] >> np.arange(32, dtype=np.uint32)[None, :]) & 1).astype(np.uint8).reshape(-1)
    return bits[:n]


def gather_verdicts(local_ok: np.ndarray, n_total: int, rank: int, world: int, device=None):
    """All-gather of the packed verdict mask; returns the full verdict byte array on every rank."""
    import torch
    import torch.distributed as dist

    wp = words_per_shard(n_total, world)
    mine = torch.from_numpy(pack_bits(local_ok, wp).astype(np.int32))
    if device is not None:
        mine = mine.to(device)
    out = torch.empty(wp * world, dtype=torch.int32, device=mine.device)
    dist.all_gather_into_tensor(out, mine)
    words = out.cpu().numpy().astype(np.uint32)
    full = np.zeros(n_total, np.uint8)
    for g in range(world):
        lo, hi = shard_range(n_total, g, world)
        full[lo:hi] = unpack_bits(words[wp * g : wp * (g + 1)], hi - lo)
    return full
