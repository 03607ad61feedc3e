"""CPU, world_size 2 over gloo: the frame-sharding index arithmetic and the all-gather wrapper used on the multi-GPU path."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, T, ret):
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "sam-pt_b200"))
    from sampt_b200 import sharding
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    full = torch.arange(T * 3 * 2, dtype=torch.float32).reshape(T, 3, 2)  # "feature maps": frame f -> distinct values
    mine = full[sharding.owned_frames(T, rank, world)]
    got = sharding.allgather_frames(mine, T)
    ok = torch.equal(got, full) and torch.equal(sharding.scatter_rows_by_frame(got, rank, world), mine)
    # several clips of different lengths in ONE collective, ownership rotated per clip: owner(f, c) = (f + c) mod G
    Ts = [T, T + 3, max(T - 1, 1)]
    fulls = [torch.arange(t * 4, dtype=torch.float32).reshape(t, 4) + 1000 * c for c, t in enumerate(Ts)]
    locs = [fulls[c][sharding.owned_frames(t, rank, world, c)] for c, t in enumerate(Ts)]
    gots = sharding.allgather_clips(locs, Ts)
    ok = ok and all(torch.equal(g, f) for g, f in zip(gots, fulls))
    # the collective delivers exactly the stack of every rank's pack_clips slab: unpack_clips of that stack, with no
    # collective, is what allgather_clips returned (the one-GPU virtual-rank test of the sharded path rests on this)
    stacked = torch.stack([sharding.pack_clips([fulls[c][sharding.owned_frames(t, r, world, c)] for c, t in enumerate(Ts)], Ts, r, world)
                           for r in range(world)])
    ok = ok and all(torch.equal(g, u) for g, u in zip(gots, sharding.unpack_clips(stacked, Ts, world)))
    # the same with an explicit clip rotation (allgather_frames(..., clip=c) of gather_logits)
    rot = sharding.allgather_clips([fulls[0][sharding.owned_frames(Ts[0], rank, world, 3)]], Ts[:1], clips=[3])
    ok = ok and torch.equal(rot[0], fulls[0])
    t = torch.tensor([1.0 if ok else 0.0])
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    # max-over-ranks timing reduction used by bench.py
    ms = torch.tensor([10.0 + rank], dtype=torch.float64)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    if rank == 0:
        ret.put((float(t.item()), float(ms.item())))
    dist.destroy_process_group()


def test_allgather_frames_world2():
    for T in (50, 7):  # divisible and ragged
        ctx = mp.get_context("spawn")
        ret = ctx.Queue()
        port = _free_port()
        procs = [ctx.Process(target=_worker, args=(r, 2, port, T, ret)) for r in range(2)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
        ok, ms = ret.get(timeout=10)
        assert ok == 1.0 and ms == 11.0


def test_allgather_frames_world4_ragged():
    """the 4- and 8-GPU scaling runs: 50 frames over 4 ranks (13,13,12,12 owned frames -> padded all-gather)."""
    world, T = 4, 50
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, T, ret)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=180)
        assert p.exitcode == 0
    ok, ms = ret.get(timeout=10)
    assert ok == 1.0 and ms == 10.0 + world - 1


def test_pack_unpack_clips_reproduce_the_frames():
    """pack_clips / unpack_clips are the two halves of allgather_clips around its collective: stacking every rank's slab and
    unpacking gives back every clip in frame order, for world 1...9 and T 1...20 (T < world: ranks that own nothing), with the
    default clip numbering and with an explicit rotation; the padding rows are zero."""
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "sam-pt_b200"))
    from sampt_b200 import sharding
    for world in range(1, 10):
        for T in range(1, 21):
            Ts = [T, 21 - T, 7]
            fulls = [torch.arange(t * 6, dtype=torch.float32).reshape(t, 2, 3) + 1000 * (i + 1) for i, t in enumerate(Ts)]
            for clips in (None, [5, 0, 2 * world + 1]):
                ids = list(range(len(Ts))) if clips is None else clips
                slabs = []
                for r in range(world):
                    own = [sharding.owned_frames(t, r, world, c) for t, c in zip(Ts, ids)]
                    slab = sharding.pack_clips([f[o] for f, o in zip(fulls, own)], Ts, r, world, clips)
                    assert slab.shape == (sum(sharding.padded_count(t, world) for t in Ts), 2, 3)
                    assert int((slab != 0).any(dim=2).any(dim=1).sum()) == sum(len(o) for o in own)   # the rest is padding
                    slabs.append(slab)
                got = sharding.unpack_clips(torch.stack(slabs), Ts, world, clips)
                assert all(torch.equal(g, f) for g, f in zip(got, fulls)), (world, T, clips)


def test_owned_frames_partition_every_world_size():
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "sam-pt_b200"))
    from sampt_b200 import sharding
    for world in (1, 2, 4, 8):
        for T in (2, 50, 100):
            for clip in range(world):
                owned = [sharding.owned_frames(T, r, world, clip) for r in range(world)]
                assert sorted(f for o in owned for f in o) == list(range(T))
                assert all(sharding.owner(f, clip, world) == r for r, o in enumerate(owned) for f in o)
                n = sharding.padded_count(T, world)
                assert all(len(o) <= n for o in owned) and max(len(o) for o in owned) == n
                # the gather's reorder index is a permutation onto the un-padded rows
                idx = sharding._gather_index(T, world, clip, n)
                assert len(set(idx)) == T and all(i < world * n for i in idx)
            # G clips of T frames: the rotation gives every rank exactly T frames (round 1: 56 vs 48 at T=50, G=8)
            per_rank = [sum(len(sharding.owned_frames(T, r, world, c)) for c in range(world)) for r in range(world)]
            assert per_rank == [T] * world, (world, T, per_rank)
