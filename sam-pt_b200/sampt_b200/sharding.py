"""Frame sharding of clips across ranks (SURVEY §8e).

Ownership is ROTATED per clip: frame f of clip c belongs to rank (f + c) mod G.  Round-robin over frames keeps every 8-frame
tracker window spread over all ranks; the per-clip rotation makes the load even when T is not a multiple of G -- with G clips
of T frames every rank owns exactly T frames (round 1 gave rank r frames r, r+G, ... of EVERY clip: 56 vs 48 frames at T=50,
G=8, a 0.89 ceiling on the 8-GPU efficiency).

The one exchange step of the path is an all-gather of per-frame tracker feature maps; this module holds the index arithmetic +
the collective wrappers so they can be tested with gloo on CPU (world_size 2 / 4) and run with NCCL on the H100s.
"""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.distributed as dist


def owner(f: int, clip: int, world: int) -> int:
    return (f + clip) % world


def owned_frames(T: int, rank: int, world: int, clip: int = 0) -> List[int]:
    """frames of clip `clip` owned by `rank`, ascending."""
    first = (rank - clip) % world
    return list(range(first, T, world))


def padded_count(T: int, world: int) -> int:
    """rows every rank contributes per clip to the all-gather (the short ranks pad with zeros)."""
    return (T + world - 1) // world


def _gather_index(T: int, world: int, clip: int, n: int) -> List[int]:
    """row of frame f inside the gathered (world, n) block of a clip: owner rank r = (f + clip) % G, position (f - first_r) / G."""
    idx = []
    for f in range(T):
        r = owner(f, clip, world)
        first = (r - clip) % world
        idx.append(r * n + (f - first) // world)
    return idx


def allgather_frames(local: torch.Tensor, T: int, group=None, clip: int = 0) -> torch.Tensor:
    """local: (n_owned, ...) features of this rank's frames of one clip (increasing frame order) -> (T, ...) in frame order on
    every rank.  One collective (NCCL all_gather_into_tensor over NVLink on GPUs, gloo in the CPU tests)."""
    return allgather_clips([local], [T], group=group, clips=[clip])[0]


def allgather_clips(locals_: Sequence[torch.Tensor], Ts: Sequence[int], group=None, clips: Sequence[int] | None = None) -> List[torch.Tensor]:
    """ONE collective for several clips: locals_[i] = (n_owned_i, ...) rows this rank owns of clip clips[i] (T_i frames).
    Returns, per clip, the (T_i, ...) tensor in frame order, on every rank."""
    world = dist.get_world_size(group)
    slab = pack_clips(locals_, Ts, dist.get_rank(group), world, clips)
    out = torch.empty((world,) + tuple(slab.shape), dtype=slab.dtype, device=slab.device)
    dist.all_gather_into_tensor(out.view((world * slab.shape[0],) + tuple(slab.shape[1:])), slab, group=group)
    return unpack_clips(out, Ts, world, clips)


def pack_clips(locals_: Sequence[torch.Tensor], Ts: Sequence[int], rank: int, world: int,
               clips: Sequence[int] | None = None) -> torch.Tensor:
    """The slab `rank` contributes to the all-gather: per clip `padded_count` rows (its owned frames in increasing frame
    order, then zeros), the clips one after the other -> (sum of the padded counts, ...).  No collective."""
    clips = list(range(len(locals_))) if clips is None else list(clips)
    ns = [padded_count(T, world) for T in Ts]
    slab = torch.zeros((sum(ns),) + tuple(locals_[0].shape[1:]), dtype=locals_[0].dtype, device=locals_[0].device)
    off = 0
    for loc, T, c, n in zip(locals_, Ts, clips, ns):
        assert loc.shape[0] == len(owned_frames(T, rank, world, c)), (loc.shape, T, rank, world, c)
        slab[off:off + loc.shape[0]] = loc
        off += n
    return slab


def unpack_clips(stacked: torch.Tensor, Ts: Sequence[int], world: int, clips: Sequence[int] | None = None) -> List[torch.Tensor]:
    """stacked (world, sum of the padded counts, ...): the slabs of `pack_clips` of every rank, in rank order (what the
    all-gather delivers) -> per clip the (T_i, ...) tensor in frame order.  No collective."""
    clips = list(range(len(Ts))) if clips is None else list(clips)
    assert stacked.shape[0] == world and stacked.shape[1] == sum(padded_count(T, world) for T in Ts), (stacked.shape, Ts, world)
    tail = tuple(stacked.shape[2:])
    res = []
    off = 0
    for T, c in zip(Ts, clips):
        n = padded_count(T, world)
        block = stacked[:, off:off + n].reshape((world * n,) + tail)       # row r*n + i = i-th owned frame of rank r
        idx = torch.tensor(_gather_index(T, world, c, n), device=stacked.device)
        res.append(block.index_select(0, idx))
        off += n
    return res


def scatter_rows_by_frame(full: torch.Tensor, rank: int, world: int, clip: int = 0) -> torch.Tensor:
    """inverse view: the rows of a (T, ...) tensor this rank owns."""
    return full[owned_frames(full.shape[0], rank, world, clip)]
