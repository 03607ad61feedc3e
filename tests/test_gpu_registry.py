"""Weight names in libsampt_b200 are shared per device.  Several models of the same kind may live in one process (the test
suite itself, or a harness comparing SAM with HQ-SAM): whoever runs must see ITS weights, and a plain SAM decoder registered
after an HQ-SAM decoder must not inherit the HQ-only tensors."""
import pytest
import torch

from oracle import pips_ref, sam_ref
from sampt_b200 import synth

pytestmark = pytest.mark.gpu


def test_two_pips_models_alternate():
    from sam_pt.point_tracker.pips import Pips
    models = []
    for seed in (7201, 99):
        m = Pips(S=8, stride=4)
        m.load_state_dict(synth.condition_pips(synth.make_state_dict(pips_ref.pips_state_dict_shapes(), seed)))
        models.append(m.cuda().eval())
    frames = synth.make_clip(8, 96, 128, seed=5)["frames"].cuda()
    q = torch.tensor([[0.0, 40.0, 30.0], [0.0, 90.0, 60.0]], device="cuda")

    def run(m):
        traj, _ = m.track(m.encode_frames(frames), q, 0.9, iters=6)
        return traj.cpu()

    a0, b0 = run(models[0]), run(models[1])
    a1, b1 = run(models[0]), run(models[1])
    assert (a0 - b0).abs().max() > 1e-3          # different weights really give different tracks
    assert torch.equal(a0, a1) and torch.equal(b0, b1)


def test_plain_sam_after_hq_sam_in_one_process():
    from sampt_b200 import factory
    from segment_anything.predictor import SamPredictor
    from segment_anything_hq.predictor import SamPredictor as HQPredictor
    cfg = sam_ref.VIT_TEST
    sd_plain = synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(cfg), 31))
    sd_hq = synth.condition_sam(synth.make_state_dict(sam_ref.sam_state_dict_shapes(cfg, hq=True), 47))
    plain = SamPredictor(factory.build_sam("vit_test", sd_plain).cuda())
    hq = HQPredictor(factory.build_sam("vit_test", sd_hq, hq=True).cuda())
    img = synth.make_clip(1, 96, 128, seed=3)["frames"][0].permute(1, 2, 0).numpy()
    pts = torch.tensor([[[300.0, 200.0], [600.0, 400.0]]], device="cuda")
    lab = torch.ones((1, 2), dtype=torch.int, device="cuda")

    def run(p):
        p.set_image(img)
        m, i, _ = p.predict_torch(pts, lab, None, None, False, True)
        return m.cpu(), i.cpu()

    m0, i0 = run(plain)
    mh, _ = run(hq)
    m1, i1 = run(plain)   # used to fail: "HQ decoder expects 6 output tokens, got 5" (stale hf_* tensors in the registry)
    mh2, _ = run(hq)
    assert torch.equal(m0, m1) and torch.equal(i0, i1)
    assert torch.equal(mh, mh2)


def _gemm_through(ctx, A, B, M, N, K):
    from ctypes import c_int
    from sampt_b200 import native
    out = torch.zeros((M, N), device=A.device, dtype=torch.float32)
    with torch.cuda.device(A.device):
        native.check(native.lib().sampt_gemm_f16(
            ctx.handle, native.ptr(A), c_int(K), native.ptr(B), c_int(K), c_int(M), c_int(N), c_int(K), c_int(1), c_int(0),
            native.ptr(None), c_int(0), native.ptr(None), native.ptr(out), native.ptr(None), c_int(N), c_int(0), native.stream_ptr()), "gemm_f16")
        torch.cuda.synchronize(A.device)
    return out


def test_two_contexts_on_one_device_are_independent():
    """include/sampt_b200.h: "distinct ctxs are independent".  Kernel attributes, graph caches and scratch buffers are per context
    (round 1 kept some of them in process-global statics): a second context on the same device, used from another stream,
    gives the same results as the first one, before and after the first one is used again."""
    from sampt_b200 import native
    g = torch.Generator().manual_seed(5)
    M, N, K = 512, 512, 256          # tensor-core GEMM (dynamic shared memory attribute set per context)
    A = torch.randn((M, K), generator=g).half().cuda()
    B = (torch.randn((N, K), generator=g) / K ** 0.5).half().cuda()
    ctx_a = native.get_context("cuda")
    ctx_b = native.Context(torch.device("cuda", torch.cuda.current_device()), workspace_bytes=256 << 20)
    ref = A.float() @ B.float().T
    r_a = _gemm_through(ctx_a, A, B, M, N, K)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        r_b = _gemm_through(ctx_b, A, B, M, N, K)
    r_a2 = _gemm_through(ctx_a, A, B, M, N, K)
    assert torch.equal(r_a, r_b) and torch.equal(r_a, r_a2)
    assert (r_a - ref).abs().max() < 2e-3
    # the fp32 skinny GEMM (cluster launch, attribute set at context creation) through the second context
    from ctypes import c_int
    x = torch.randn((64, 512), generator=g).cuda()
    w = (torch.randn((256, 512), generator=g) / 512 ** 0.5).cuda()
    y = torch.empty((64, 256), device="cuda")
    native.check(native.lib().sampt_linear_f32(ctx_b.handle, native.ptr(x), c_int(512), native.ptr(w), c_int(512), native.ptr(None),
                                               native.ptr(None), c_int(0), native.ptr(y), c_int(256), c_int(64), c_int(256), c_int(512),
                                               c_int(0), native.stream_ptr()))
    torch.cuda.synchronize()
    assert (y - x @ w.T).abs().max() < 1e-4


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs in one process")
def test_two_devices_in_one_process():
    """Contexts on two devices in one process: every kernel attribute (dynamic shared memory limits) is set per device."""
    from sampt_b200 import native
    g = torch.Generator().manual_seed(6)
    M, N, K = 512, 512, 256
    A = torch.randn((M, K), generator=g).half()
    B = (torch.randn((N, K), generator=g) / K ** 0.5).half()
    outs = []
    for d in (0, 1):
        dev = torch.device("cuda", d)
        with torch.cuda.device(dev):
            outs.append(_gemm_through(native.get_context(dev), A.to(dev), B.to(dev), M, N, K).cpu())
    assert torch.equal(outs[0], outs[1])
    assert (outs[0] - A.float() @ B.float().T).abs().max() < 2e-3
