"""Generate golden vectors for PIPS++ by running the UNMODIFIED reference on CPU (build container only).

    python tests/golden/make_golden_pips_plus_plus.py

Imports /root/reference's PipsPlusPlus / PipsPlusPlusPointTracker with the stub-package trick of _refimport.py (the reference's
sam_pt/point_tracker/__init__.py eagerly imports trackers whose dependencies are absent), makes `Tensor.cuda()` the identity so
that the reference's `.cuda()` calls run on CPU, runs it on seeded inputs (sampt_b200.synth) and writes
pips_plus_plus_golden.pt next to this file.  Inputs are NOT stored: they are re-generated from the seeds.
"""
import importlib
import os
import sys
import tempfile
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "sam-pt_b200"))
sys.path.insert(0, ROOT)

from sampt_b200 import synth  # noqa: E402

REF = "/root/reference"
H, W = 128, 160


def import_reference():
    saved = {k: v for k, v in sys.modules.items() if k == "sam_pt" or k.startswith("sam_pt.")}
    for k in saved:
        del sys.modules[k]
    for name, path in {"sam_pt": f"{REF}/sam_pt", "sam_pt.point_tracker": f"{REF}/sam_pt/point_tracker"}.items():
        m = types.ModuleType(name)
        m.__path__ = [path]
        sys.modules[name] = m
    sys.modules["sam_pt"].point_tracker = sys.modules["sam_pt.point_tracker"]
    for leaf in ("utils.basic", "utils.samp", "utils.misc", "utils.saverloader"):
        importlib.import_module("sam_pt.point_tracker." + leaf)
    sys.modules["sam_pt.point_tracker"].PointTracker = importlib.import_module("sam_pt.point_tracker.tracker").PointTracker
    ppp = importlib.import_module("sam_pt.point_tracker.pips_plus_plus.pips_plus_plus")
    sys.modules["sam_pt.point_tracker.pips_plus_plus"].PipsPlusPlus = ppp.PipsPlusPlus
    trk = importlib.import_module("sam_pt.point_tracker.pips_plus_plus.tracker")
    out = {"PipsPlusPlus": ppp.PipsPlusPlus, "Tracker": trk.PipsPlusPlusPointTracker}
    for k in [k for k in sys.modules if k == "sam_pt" or k.startswith("sam_pt.")]:
        del sys.modules[k]
    sys.modules.update(saved)
    return out


def window_inputs(S, N, seed, h=H, w=W):
    clip = synth.make_clip(S, h, w, seed=seed)
    q = synth.make_query_points(clip, N, seed=seed)[0, :, 1:]
    return clip["frames"][None].float(), q[None, None].repeat(1, S, 1, 1)


def tracker_run(R, sd, frames, q, iters, max_len=128, image_size=None):
    with tempfile.TemporaryDirectory() as d:
        synth.write_pips_checkpoint_dir(sd, d)
        trk = R["Tracker"](checkpoint_path=d, stride=8, max_sequence_length=max_len, iters=iters, image_size=image_size).eval()
        with torch.no_grad():
            try:
                traj, vis = trk(frames, q.clone())
            except IndexError as e:
                return {"error": f"IndexError: {e}"}
    return {"trajectories": traj.clone(), "visibilities": vis.clone()}


def main():
    torch.set_num_threads(8)
    torch.Tensor.cuda = lambda self, *a, **k: self
    R = import_reference()
    sd = synth.make_pips_plus_plus_state_dict()
    model = R["PipsPlusPlus"](stride=8).eval()
    model.load_state_dict(sd, strict=True)
    out = {"structure": {"tensors": len(model.state_dict()), "params": sum(v.numel() for v in model.state_dict().values())}}

    for S, N, iters, seed in ((8, 5, 16, 72), (128, 3, 3, 73)):
        rgbs, tr = window_inputs(S, N, seed)
        with torch.no_grad():
            p1, p2, feats, _ = model(tr, rgbs, iters=iters)
        case = {"cfg": {"S": S, "N": N, "iters": iters, "seed": seed}, "preds1": torch.stack(p1)[:, 0].clone(),
                "preds2": torch.stack(p2)[:, 0].clone(), "feats": torch.stack(feats)[:, 0].clone()}
        if S == 8:
            with torch.no_grad():
                q1, _, f2, _ = model(tr + 1.5, rgbs, iters=4, feat_init=feats)
            case["feat_init_preds1"] = torch.stack(q1)[:, 0].clone()
            case["feat_init_feats"] = torch.stack(f2)[:, 0].clone()
        out[f"window_S{S}"] = case

    # NaN below 128 px: one iteration at 96x128
    rgbs, tr = window_inputs(8, 3, 74, 96, 128)
    with torch.no_grad():
        p1, _, _, _ = model(tr, rgbs, iters=1)
    out["nan_96x128"] = bool(torch.isnan(p1[-1][:, 1:]).all())

    def clip_q(T, N, seed, t, h=H, w=W):
        clip = synth.make_clip(T, h, w, seed=seed)
        return clip["frames"][None].float(), synth.make_query_points(clip, N, seed=seed, t=t)

    trk = {}
    for name, (T, N, seed, t, iters, image_size) in {
            "t0": (12, 4, 75, 0, 4, None), "t5": (12, 4, 76, 5, 4, None), "last": (12, 3, 77, 11, 4, None),
            "image_size": (6, 3, 78, 0, 3, (160, 192)), "long140": (140, 3, 79, 0, 2, None)}.items():
        frames, q = clip_q(T, N, seed, t)
        trk[name] = {"cfg": {"T": T, "N": N, "seed": seed, "t": t, "iters": iters, "image_size": image_size},
                     "query_points": q.clone(), **tracker_run(R, sd, frames, q, iters, image_size=image_size)}
    frames, q = clip_q(12, 4, 80, 0)
    q[0, 2:, 0] = 6.0
    trk["mixed"] = {"cfg": {"T": 12, "N": 4, "seed": 80, "iters": 2}, "query_points": q.clone(), **tracker_run(R, sd, frames, q, 2)}
    out["tracker"] = trk

    path = os.path.join(HERE, "pips_plus_plus_golden.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
