"""GPU, 2 ranks over NCCL (skipped with < 2 devices): the frame-sharded path (one all-gather of PIPS feature maps) gives
the same trajectories and masks as the single-GPU path."""
import os
import socket
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, tmp, ret, tracker="pips"):
    for p in (ROOT, os.path.join(ROOT, "sam-pt_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch.distributed as dist
    from oracle import pips_ref, sam_ref
    from sampt_b200 import factory, synth
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    cfg = sam_ref.VIT_TEST
    sam_sd = synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(cfg), 5))
    pips_sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 7201))
    ckpt = synth.write_pips_checkpoint_dir(pips_sd, os.path.join(tmp, f"pips{rank}"))
    cot_sd = None
    if tracker == "cotracker":
        from oracle import cotracker_ref
        cot_sd = synth.condition_cotracker(synth.make_state_dict(cotracker_ref.cotracker_state_dict_shapes(), 31), vis_bias=0.6)
    model = factory.build_sam_pt("vit_test", sam_sd, ckpt, positive_points_per_mask=4, sam_iou_threshold=-1e9,
                                 device=torch.device("cuda", rank), cotracker_state_dict=cot_sd, cotracker_interp_shape=(64, 96))
    # ragged: 9 and 11 frames over 2 ranks, 3 clips (more clips than ranks), ownership rotated per clip
    videos = [synth.make_video_dict(9 + 2 * (c % 2), 96, 128, 4, seed=80 + c) for c in range(world + 1)]
    # 6 masks > point_tracker_mask_batch_size = 5, queried on different frames: the chain tracks 5 + 1 masks as forward does
    clip = synth.make_clip(10, 96, 128, seed=89)
    videos.append({"image": [f for f in clip["frames"]], "target_hw": (96, 128),
                   "query_points": torch.cat([synth.make_query_points(clip, 4, 89 + m, t=t) for m, t in enumerate((0, 3, 9, 0, 5, 2))])})
    res = model.forward_clips_sharded(videos, gather_logits=True)
    ok = True
    for c, v in enumerate(videos):
        # bitwise: the encoders are batch invariant and the chain runs the calls forward runs (test_gpu_sharded_one_gpu.py
        # establishes both on one device); empty masks are -inf on both sides, which torch.equal compares equal
        single = model(v)
        ok &= bool(torch.equal(res[c]["trajectories"].cpu(), single["trajectories"].cpu()))
        ok &= bool(torch.equal(res[c]["visibilities"].cpu(), single["visibilities"].cpu()))
        ok &= bool(torch.equal(res[c]["logits"].cpu(), torch.stack(single["logits"]).cpu()))
    t = torch.tensor([1.0 if ok else 0.0], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(float(t.item()))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("tracker", ["pips", "cotracker"])
def test_frame_sharded_matches_single_gpu(tmp_path, tracker):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, str(tmp_path), ret, tracker)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    assert ret.get(timeout=10) == 1.0
