"""GPU, ONE device: the frame-sharded multi-GPU path (`SamPt.forward_clips_sharded`) run rank by rank in this process.

`forward_clips_sharded` is three local stages with a collective between them.  `run_virtual` drives `world` virtual ranks
through stage A one after the other, stacks their slabs (`torch.stack` over the ranks is exactly what
`all_gather_into_tensor` delivers), runs stage C for each, stacks again and runs stage E for each.  What it returns per rank
is what that rank of a real `world`-GPU job returns, so it is compared clip by clip with `SamPt.forward` on the same clip.

The criterion is `torch.equal` everywhere.  That is sound because the encoders are bitwise batch invariant (section a): a rank
encodes frames {r, r + G, ...} of several clips in one batch, `forward` encodes a clip in one batch, and every output element
must come out with the same bits.  Only the collectives themselves are not executed here (gloo: test_sharding_gloo.py; NCCL:
test_gpu_multi.py on two devices).  Nothing reads the reference tree; weights are synthetic and inputs come from seeds."""
import pytest
import torch

pytestmark = pytest.mark.gpu

H, W = 96, 128
P = 4


# --------------------------------------------------------------------------------------------------------------- fixtures
def _sam_sd(seed, hq=False):
    from oracle import sam_ref
    from sampt_b200 import synth
    return synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(sam_ref.VIT_TEST, hq=hq), seed))


@pytest.fixture(scope="module")
def pips_ckpt(tmp_path_factory):
    from oracle import pips_ref
    from sampt_b200 import synth
    sd = synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), 7201))
    return synth.write_pips_checkpoint_dir(sd, str(tmp_path_factory.mktemp("pips")))


@pytest.fixture(scope="module")
def models(pips_ckpt):
    """SamPt with the ViT test twin: one with PIPS, one with CoTracker (vis_bias 0.6 keeps the points visible)."""
    from oracle import cotracker_ref
    from sampt_b200 import factory, synth
    cot_sd = synth.condition_cotracker(synth.make_state_dict(cotracker_ref.cotracker_state_dict_shapes(), 31), vis_bias=0.6)
    out = {}
    for name, cot in (("pips", None), ("cotracker", cot_sd)):
        out[name] = factory.build_sam_pt("vit_test", _sam_sd(5), pips_ckpt, positive_points_per_mask=P, sam_iou_threshold=-1e9,
                                         cotracker_state_dict=cot, cotracker_interp_shape=(64, 96))
        assert out[name].point_tracker_mask_batch_size == 5
    return out


def _video(T, seed, query_frames=(0,), h=H, w=W):
    """One clip with len(query_frames) masks of P points; mask m is queried on frame query_frames[m]."""
    from sampt_b200 import synth
    clip = synth.make_clip(T, h, w, seed)
    q = torch.cat([synth.make_query_points(clip, P, seed + 17 * m, t=t) for m, t in enumerate(query_frames)], dim=0)
    return {"image": [f for f in clip["frames"]], "target_hw": (h, w), "query_points": q}


def _invisible_video(T, seed):
    """Every query point lies in the first column (x / W < 0.01): on its query frame, at least, the out-of-frame relabel makes
    the whole mask invisible, so that frame's logits and score are -inf."""
    v = _video(T, seed)
    v["query_points"][:, :, 1] = torch.tensor([0.2, 0.4, 0.6, 0.8])
    return v


SCENARIOS = {
    # ragged T, 3 clips: more clips than ranks at world 2, fewer at world 4 and 8
    "ragged": lambda: [_video(9, 80), _video(11, 81), _video(10, 82)],
    # one clip on 4 ranks: ranks 1-3 run no chain and contribute an all-zero slab
    "one_clip": lambda: [_video(9, 83)],
    # one 5-frame clip on 8 ranks: ranks 5-7 own no frame at all (and T < S, CoTracker's short-clip padding)
    "short": lambda: [_video(5, 84)],
    # on 8 ranks some rank owns none of clip 0's frames but owns frames of clip 1
    "short_plus": lambda: [_video(5, 85), _video(9, 86)],
    # masks queried on different frames, clips with different numbers of masks (N_max padding of the trajectory slab)
    "masks2": lambda: [_video(10, 87, (0, 6)), _video(9, 88)],
    # more masks than point_tracker_mask_batch_size = 5: the chain must track 5 + 1 masks as forward does
    "masks6": lambda: [_video(9, 89, (0, 3, 8, 0, 5, 2)), _video(10, 90, (4,))],
    "invisible": lambda: [_invisible_video(9, 91), _video(9, 92)],
}
_cache = {}


def _scenario(models, tracker, name):
    """(videos, what SamPt.forward returns for each of them), computed once per tracker and scenario."""
    if (tracker, name) not in _cache:
        videos = SCENARIOS[name]()
        singles = []
        for v in videos:
            o = models[tracker](v)
            singles.append({"trajectories": o["trajectories"], "visibilities": o["visibilities"], "logits": torch.stack(o["logits"]),
                            "scores_per_frame": torch.tensor(o["scores_per_frame"], dtype=torch.float32)})
        _cache[(tracker, name)] = (videos, singles)
    return _cache[(tracker, name)]


# ------------------------------------------------------------------------------------------------------- virtual ranks
def gather_logits_virtual(per_rank, Ts, world):
    """What `gather_logits=True` does with its one collective per clip, on the stacked per-rank logits."""
    from sampt_b200 import sharding
    fulls = []
    for c, T in enumerate(Ts):
        slabs = [sharding.pack_clips([per_rank[r][c]["logits"].transpose(0, 1).contiguous()], [T], r, world, clips=[c])
                 for r in range(world)]
        fulls.append(sharding.unpack_clips(torch.stack(slabs), [T], world, clips=[c])[0].transpose(0, 1))
    return fulls


def run_virtual(model, videos, world, gather_logits=False):
    """`forward_clips_sharded` of every rank of a `world`-rank job, one rank after the other on this device."""
    from sampt_b200 import sharding
    states = [model._sharded_encode(videos, r, world) for r in range(world)]
    Ts = states[0]["Ts"]
    stacked = torch.stack([sharding.pack_clips(s["locs"], Ts, r, world) for r, s in enumerate(states)])
    fulls = sharding.unpack_clips(stacked, Ts, world)
    gathered = torch.stack([model._sharded_track(s, fulls, r, world) for r, s in enumerate(states)])
    per_rank = [model._sharded_decode(s, gathered, r, world) for r, s in enumerate(states)]
    if gather_logits:
        fulls = gather_logits_virtual(per_rank, Ts, world)
        for res in per_rank:
            for c, T in enumerate(Ts):
                res[c]["logits"], res[c]["frame_ids"] = fulls[c], list(range(T))
    return per_rank


def _same(a, b, what):
    a, b = a.cpu(), b.cpu()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not torch.equal(a, b):
        d = (a.double().nan_to_num(posinf=1e30, neginf=-1e30) - b.double().nan_to_num(posinf=1e30, neginf=-1e30)).abs()
        raise AssertionError(f"{what}: {int((d > 0).sum())} of {d.numel()} elements differ, max |d| = {d.max().item():.3e}")


# ---------------------------------------------------------------------------------- a. encoder batch invariance, bitwise
def _tuple(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x,)


def _check_batch_invariance(enc, clip_a, clip_b, what):
    """enc: (n,3,H,W) uint8 -> tensor or tuple of tensors with n rows.  The rows of a clip encoded in one call must equal,
    bit for bit, the rows encoded (i) frame by frame, (ii) as the owned subsets of 2 / 3 / 8 ranks put back in frame order,
    (iii) as part of a batch that mixes owned frames of two clips."""
    from sampt_b200 import sharding
    T = clip_a.shape[0]
    full_a, full_b = _tuple(enc(clip_a)), _tuple(enc(clip_b))
    for k, fa in enumerate(full_a):
        _same(torch.cat([_tuple(enc(clip_a[t:t + 1]))[k] for t in range(T)]), fa, f"{what}[{k}] frame by frame")
    for world in (2, 3, 8):
        for clip in (0, 1):   # with and without the ownership rotation
            owned = [sharding.owned_frames(T, r, world, clip) for r in range(world)]
            parts = [_tuple(enc(clip_a[o])) if o else None for o in owned]
            for k, fa in enumerate(full_a):
                locs = [p[k] if p is not None else fa[:0] for p in parts]
                stacked = torch.stack([sharding.pack_clips([l], [T], r, world, clips=[clip]) for r, l in enumerate(locs)])
                _same(sharding.unpack_clips(stacked, [T], world, clips=[clip])[0], fa, f"{what}[{k}] world {world} clip {clip}")
    for rank in (0, 1):
        oa, ob = sharding.owned_frames(T, rank, 2, 0), sharding.owned_frames(clip_b.shape[0], rank, 2, 1)
        mixed = _tuple(enc(torch.cat([clip_a[oa], clip_b[ob]])))
        for k in range(len(full_a)):
            _same(mixed[k][:len(oa)], full_a[k][oa], f"{what}[{k}] mixed batch, clip a")
            _same(mixed[k][len(oa):], full_b[k][ob], f"{what}[{k}] mixed batch, clip b")


# 480x854 is the C2 frame size: H/4 = 120, W/4 = 213 (odd), where the im2col tails live
@pytest.mark.parametrize("hw", [(96, 128), (480, 854)])
@pytest.mark.parametrize("encoder", ["pips", "cotracker", "vit", "vit_hq"])
def test_encoder_is_bitwise_batch_invariant(models, monkeypatch, encoder, hw):
    from sampt_b200 import factory, synth
    clip_a = synth.make_clip(9, hw[0], hw[1], seed=60)["frames"].cuda()
    clip_b = synth.make_clip(7, hw[0], hw[1], seed=61)["frames"].cuda()
    if encoder == "pips":
        enc = models["pips"].point_tracker.model.fnet_frames
    elif encoder == "cotracker":
        trk = models["cotracker"].point_tracker
        if hw != (96, 128):
            monkeypatch.setattr(trk, "interp_shape", (384, 512))   # the configured CoTracker resolution
        enc = lambda f: trk.model.fnet_frames(trk.resize_clip(f))  # noqa: E731
    elif encoder == "vit":
        enc = lambda f: models["pips"].sam_predictor.encode_frames(f, want_interm=False)  # noqa: E731
    else:
        from segment_anything_hq.predictor import SamPredictor
        pred = SamPredictor(sam_model=factory.build_sam("vit_test", _sam_sd(47, hq=True), hq=True).cuda().eval())
        assert pred._uses_interm()
        enc = lambda f: pred.encode_frames(f, want_interm=True)  # noqa: E731
    with torch.no_grad():
        _check_batch_invariance(enc, clip_a, clip_b, f"{encoder} {hw}")


# ---------------------------------------------------------------------- b. chain on pre-computed features == forward
@pytest.mark.parametrize("case", ["pips_t0", "pips_mixed_t", "cotracker_T14", "cotracker_T5"])
def test_track_on_features_equals_tracker_forward(models, case):
    from sampt_b200 import synth
    tracker, T, ts = {"pips_t0": ("pips", 12, (0, 0, 0, 0, 0)),
                      "pips_mixed_t": ("pips", 12, (0, 5, 11, 3, 11)),       # T - 1 included: the time-flipped pass runs
                      "cotracker_T14": ("cotracker", 14, (0, 6, 13, 2, 0)),
                      "cotracker_T5": ("cotracker", 5, (0, 2, 4, 1, 0))}[case]  # T < S: the short-clip padding branch
    trk = models[tracker].point_tracker
    clip = synth.make_clip(T, H, W, seed=70)
    q = torch.cat([synth.make_query_points(clip, 1, 70 + i, t=t) for i, t in enumerate(ts)], dim=1).cuda()   # (1, 5, 3)
    frames = clip["frames"].cuda()
    with torch.no_grad():
        traj, vis = trk(frames[None], q)
        traj_s, vis_s = trk.track_on_features(trk.shard_features(frames), q, (H, W))
    assert traj.shape == (1, T, len(ts), 2) and vis.dtype == torch.bool
    _same(traj_s, traj, f"{case} trajectories")
    _same(vis_s, vis, f"{case} visibilities")


# ------------------------------------------------------------------------------ c. virtual ranks vs SamPt.forward
CASES = [("ragged", 1, True), ("ragged", 2, True), ("ragged", 3, True), ("ragged", 4, True), ("ragged", 8, True),
         ("ragged", 3, False), ("one_clip", 4, True), ("short", 8, True), ("short", 8, False), ("short_plus", 8, True),
         ("masks2", 2, True), ("masks2", 3, False), ("masks6", 2, True), ("masks6", 4, True), ("invisible", 2, True),
         ("invisible", 3, True)]


@pytest.mark.parametrize("scenario,world,overlap", CASES)
@pytest.mark.parametrize("tracker", ["pips", "cotracker"])
def test_virtual_ranks_equal_forward(models, monkeypatch, tracker, scenario, world, overlap):
    """overlap = `SamPt.overlap_streams` (SAMPT_OVERLAP).  With True, stage A of every virtual rank enqueues its ViT launches
    on the one encoder stream and ViT slab of this device before any of them is consumed: that is legal only because the
    launches are ordered on that stream and every consumer waits for its own chunk's event."""
    from sampt_b200 import sharding
    model = models[tracker]
    videos, singles = _scenario(models, tracker, scenario)
    monkeypatch.setattr(model, "overlap_streams", overlap)
    per_rank = run_virtual(model, videos, world)
    if scenario == "invisible":   # the case is only a case if forward really produced an empty mask
        assert torch.isinf(singles[0]["logits"][0, 0]).all() and singles[0]["scores_per_frame"][0, 0] == -float("inf")
    if scenario == "short":
        assert sum(1 for r in range(world) if not sharding.owned_frames(len(videos[0]["image"]), r, world, 0)) == 3
    for c, (v, single) in enumerate(zip(videos, singles)):
        T, M = len(v["image"]), v["query_points"].shape[0]
        seen = []
        for r in range(world):
            res = per_rank[r][c]
            # the sharded results stay on the device (forward's outputs_on_cpu does not apply): a change must be noticed here
            assert all(res[k].is_cuda for k in ("trajectories", "visibilities", "logits", "scores_per_frame"))
            _same(res["trajectories"], single["trajectories"], f"clip {c} rank {r} trajectories")
            _same(res["visibilities"], single["visibilities"], f"clip {c} rank {r} visibilities")
            ids = res["frame_ids"]
            assert ids == sharding.owned_frames(T, r, world, c)
            assert res["logits"].shape == (M, len(ids), H, W) and res["scores_per_frame"].shape == (len(ids), M)
            _same(res["logits"], single["logits"][:, ids], f"clip {c} rank {r} logits of frames {ids}")
            _same(res["scores_per_frame"], single["scores_per_frame"][ids], f"clip {c} rank {r} scores of frames {ids}")
            seen += ids
        assert sorted(seen) == list(range(T))   # every frame decoded by exactly one rank
    fulls = gather_logits_virtual(per_rank, [len(v["image"]) for v in videos], world)
    for c, single in enumerate(singles):
        _same(fulls[c], single["logits"], f"clip {c} gathered logits")


def test_run_virtual_gather_logits_returns_full_clips(models):
    videos, singles = _scenario(models, "pips", "masks2")
    for res in run_virtual(models["pips"], videos, 3, gather_logits=True):
        for c, single in enumerate(singles):
            assert res[c]["frame_ids"] == list(range(len(videos[c]["image"])))
            _same(res[c]["logits"], single["logits"], f"clip {c}")


# -------------------------------------------------------------------------------------------- d. the boundary raises
@pytest.mark.parametrize("option", ["use_point_reinit", "use_patch_matching_filtering", "query_masks", "target_hw",
                                    "frame size", "PipsPlusPlusPointTracker"])
def test_unsupported_combination_raises_before_any_launch(models, monkeypatch, option):
    from sampt_b200 import native
    model = models["pips"]
    videos = [_video(6, 95), _video(6, 96)]
    exc = NotImplementedError
    if option in ("use_point_reinit", "use_patch_matching_filtering"):
        monkeypatch.setattr(model, option, True)
    elif option == "query_masks":
        del videos[1]["query_points"]
        videos[1]["query_masks"] = torch.ones((1, H, W))
        videos[1]["query_point_timestep"] = torch.zeros(1)
    elif option == "target_hw":
        videos[1]["target_hw"], exc = (H // 2, W // 2), ValueError
    elif option == "frame size":
        videos[1], exc = _video(6, 96, h=64, w=96), ValueError
    else:
        from sam_pt.point_tracker.pips_plus_plus import PipsPlusPlusPointTracker
        monkeypatch.setattr(model, "point_tracker", PipsPlusPlusPointTracker(checkpoint_path=None, stride=8, max_sequence_length=128,
                                                                             iters=16, image_size=None))
    ctx = native.get_context(model.device)
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    with pytest.raises(exc, match=option):
        model._sharded_encode(videos, 0, 2)
    assert ctx.launch_count() == n0
