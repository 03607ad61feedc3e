// Host-side orchestration of the PIPS path (C++; one stream, no Python in the loop).
//   sampt_pips_fnet      : BasicEncoder over frames, computed ONCE per frame (InstanceNorm has no running stats so
//                          per-frame features are window-independent, SURVEY §0.7-i)         pips.py:254-287
//   sampt_pips_pyramid   : avg-pool pyramid                                                    pips.py:355-361
//   sampt_pips_track     : sliding-window chain with trajectory linking                        pips/tracker.py:42-153
#include "common.cuh"
#include "kernels.cuh"
#include "tc_api.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {

struct Act {  // channels-last activation
  float* p; int n, h, w, c;
  size_t numel() const { return (size_t)n * h * w * c; }
};

static int alloc_act(Ctx* c, Act* a, int n, int h, int w, int ch, const char* what) {
  a->n = n; a->h = h; a->w = w; a->c = ch;
  return ws_get(c, &a->p, a->numel(), what);
}

struct FnetScratch { float* stats_a; float* stats_b; double* part; };

static bool fnet_uses_tc(const Ctx* c, const std::string& prefix) {
  const TensorRef* f = c->find(prefix + "fnet.tc_flag");
  return f != nullptr && f->dims[0] == 1 && c->find(prefix + "fnet.conv2.w16") != nullptr;
}

// c->fnet_im2col: scratch for the tensor-core convolution path (im2col operand); null -> strict fp32 CUDA-core convolutions
// c->fnet_prefix: weight-name prefix of the encoder being run ("pips." or "cot."; the CoTracker BasicEncoder has the same
// architecture).  Both live in the ctx (not process-wide) so that encoders of different ctxs / devices never see each other's.

int conv_by_name(Ctx* c, cudaStream_t st, const std::string& name, const Act& in, Act* out, int R, int stride, int pad) {
  if (c->fnet_im2col != nullptr) {
    // implicit-GEMM on tensor cores: A = im2col(in) as fp16 hi|lo, B = weights hi|lo, 3 split passes (~fp32), fp32 NHWC output
    const __half* w16; const float* b;
    SAMPT_TRY(get_f16(c, c->fnet_prefix + name + ".w16", &w16));
    SAMPT_TRY(get_f32(c, c->fnet_prefix + name + ".bias", &b));
    const int K = R * R * in.c, Kp = ((K + 63) / 64) * 64;
    SAMPT_TRY(im2col_nhwc_split(c, st, in.p, c->fnet_im2col, in.n, in.h, in.w, in.c, R, R, stride, pad, Kp));
    const int Ho = (in.h + 2 * pad - R) / stride + 1, Wo = (in.w + 2 * pad - R) / stride + 1;
    GemmSeg seg{3, {0, Kp, 0}, {0, 0, Kp}};
    GemmEpi ep{};
    ep.out32 = out->p; ep.bias = b; ep.ldc = out->c;
    return gemm_tc(c, st, c->fnet_im2col, 2 * Kp, w16, 2 * Kp, in.n * Ho * Wo, out->c, Kp, seg, ep);
  }
  const float *w, *b;
  SAMPT_TRY(get_f32(c, c->fnet_prefix + name + ".weight_rsck", &w));
  SAMPT_TRY(get_f32(c, c->fnet_prefix + name + ".bias", &b));
  return conv_nhwc_f32(c, st, in.p, w, b, out->p, in.n, in.h, in.w, in.c, out->c, R, R, stride, pad);
}

// conv1 (7x7 stride 2 pad 3, 3 -> 64) on planar frames (uint8, or float holding 0..255), normalisation 2*(x/255)-1 fused:
// im2col + 3-pass tensor-core GEMM when c->fnet_im2col is set, else the fp32 CUDA-core kernel.  out: (n, H2, W2, 64) channels-last.
int conv1_frames(Ctx* c, cudaStream_t st, const void* frames, int is_f32, int n, int H, int W, float* out) {
  const int H2 = (H + 6 - 7) / 2 + 1, W2 = (W + 6 - 7) / 2 + 1;
  if (c->fnet_im2col != nullptr) {
    const __half* w16; const float* b1;
    SAMPT_TRY(get_f16(c, c->fnet_prefix + "fnet.conv1.w16", &w16));
    SAMPT_TRY(get_f32(c, c->fnet_prefix + "fnet.conv1.bias", &b1));
    SAMPT_TRY(im2col_conv1_split(c, st, frames, is_f32, c->fnet_im2col, n, H, W, 192));
    GemmSeg seg{3, {0, 192, 0}, {0, 0, 192}};
    GemmEpi ep{};
    ep.out32 = out; ep.bias = b1; ep.ldc = 64;
    return gemm_tc(c, st, c->fnet_im2col, 384, w16, 384, n * H2 * W2, 64, 192, seg, ep);
  }
  const float *w1, *b1;
  SAMPT_TRY(get_f32(c, c->fnet_prefix + "fnet.conv1.weight_rsck", &w1));
  SAMPT_TRY(get_f32(c, c->fnet_prefix + "fnet.conv1.bias", &b1));
  return conv7x7s2(c, st, frames, is_f32, w1, b1, out, n, H, W);
}

// ResidualBlock (pips.py:139-188): y = relu(IN(conv1 x)); y = relu(IN(conv2 y)); x' = IN(conv1x1 x) if stride>1; relu(x'+y)
// s1/s2/s3 are scratch buffers at least as large as the block's output.
static int res_block(Ctx* c, cudaStream_t st, const std::string& p, const Act& x, Act* out, int planes, int stride,
                     float* s1, float* s2, float* s3, FnetScratch& s) {
  const int ho = (x.h + 2 - 3) / stride + 1, wo = (x.w + 2 - 3) / stride + 1;
  Act y1{s1, x.n, ho, wo, planes}, y2{s2, x.n, ho, wo, planes}, ds{s3, x.n, ho, wo, planes};
  SAMPT_TRY(conv_by_name(c, st, p + "conv1", x, &y1, 3, stride, 1));
  SAMPT_TRY(inorm_stats(c, st, y1.p, s.stats_a, s.part, x.n, ho * wo, planes));
  SAMPT_TRY(inorm_apply(c, st, y1.p, s.stats_a, nullptr, nullptr, y1.p, x.n, ho * wo, planes, 1, 0));
  SAMPT_TRY(conv_by_name(c, st, p + "conv2", y1, &y2, 3, 1, 1));
  SAMPT_TRY(inorm_stats(c, st, y2.p, s.stats_a, s.part, x.n, ho * wo, planes));
  out->n = x.n; out->h = ho; out->w = wo; out->c = planes;
  if (stride == 1) {
    SAMPT_TRY(inorm_apply(c, st, y2.p, s.stats_a, x.p, nullptr, out->p, x.n, ho * wo, planes, 1, 1));
  } else {
    SAMPT_TRY(conv_by_name(c, st, p + "downsample.0", x, &ds, 1, stride, 0));
    SAMPT_TRY(inorm_stats(c, st, ds.p, s.stats_b, s.part, x.n, ho * wo, planes));
    SAMPT_TRY(inorm_apply(c, st, y2.p, s.stats_a, ds.p, s.stats_b, out->p, x.n, ho * wo, planes, 1, 1));
  }
  return 0;
}

static int fnet_chunk(Ctx* c, cudaStream_t st, const void* frames, int is_f32, int n, int H, int W, int stride, float* fmaps_out) {
  const int H2 = (H + 6 - 7) / 2 + 1, W2 = (W + 6 - 7) / 2 + 1;
  const int Ho = H / stride, Wo = W / stride;
  size_t big = (size_t)n * H2 * W2 * 64;  // largest activation (also >= later stages: 96ch at /4 res etc.)
  size_t cat_elems = (size_t)n * Ho * Wo * 416;
  float *bufA, *bufB, *bufC, *bufD, *bufE;
  SAMPT_TRY(ws_get(c, &bufA, big, "fnet bufA"));
  SAMPT_TRY(ws_get(c, &bufB, big, "fnet bufB"));
  SAMPT_TRY(ws_get(c, &bufC, big, "fnet bufC"));
  SAMPT_TRY(ws_get(c, &bufD, big, "fnet bufD"));
  SAMPT_TRY(ws_get(c, &bufE, big, "fnet bufE"));
  float* cat;
  SAMPT_TRY(ws_get(c, &cat, cat_elems, "fnet concat"));
  FnetScratch s;
  SAMPT_TRY(ws_get(c, &s.stats_a, (size_t)n * 256 * 2, "stats_a"));
  SAMPT_TRY(ws_get(c, &s.stats_b, (size_t)n * 256 * 2, "stats_b"));
  int nchunks = cdiv((long long)H2 * W2, 512);
  SAMPT_TRY(ws_get(c, &s.part, (size_t)n * nchunks * 256 * 2, "inorm partials"));

  Act x{bufA, n, H2, W2, 64};
  c->fnet_im2col = nullptr;
  if (fnet_uses_tc(c, c->fnet_prefix)) {
    // largest im2col operand: max(layer1: H2*W2 x 2*576, conv2: Ho*Wo x 2*3776) halves per frame
    size_t a_elems = std::max((size_t)H2 * W2 * 2 * 576, (size_t)Ho * Wo * 2 * 3776) * n;
    SAMPT_TRY(ws_get(c, &c->fnet_im2col, a_elems, "fnet im2col operand"));
  }
  SAMPT_TRY(conv1_frames(c, st, frames, is_f32, n, H, W, x.p));
  SAMPT_TRY(inorm_stats(c, st, x.p, s.stats_a, s.part, n, H2 * W2, 64));
  SAMPT_TRY(inorm_apply(c, st, x.p, s.stats_a, nullptr, nullptr, x.p, n, H2 * W2, 64, 1, 0));

  float *t1 = bufC, *t2 = bufD, *t3 = bufE;
  // layer1 (64, stride 1)
  Act a0{bufB, 0, 0, 0, 0}, a{bufA, 0, 0, 0, 0};
  SAMPT_TRY(res_block(c, st, "fnet.layer1.0.", x, &a0, 64, 1, t1, t2, t3, s));
  SAMPT_TRY(res_block(c, st, "fnet.layer1.1.", a0, &a, 64, 1, t1, t2, t3, s));  // a lives in bufA
  SAMPT_TRY(resize_ac_concat(c, st, a.p, cat, n, a.h, a.w, 64, Ho, Wo, 416, 0));
  // layer2 (96, stride 2)
  Act b0{bufB, 0, 0, 0, 0}, b{bufA, 0, 0, 0, 0};
  SAMPT_TRY(res_block(c, st, "fnet.layer2.0.", a, &b0, 96, 2, t1, t2, t3, s));
  SAMPT_TRY(res_block(c, st, "fnet.layer2.1.", b0, &b, 96, 1, t1, t2, t3, s));
  SAMPT_TRY(resize_ac_concat(c, st, b.p, cat, n, b.h, b.w, 96, Ho, Wo, 416, 64));
  // layer3 (128, stride 2)
  Act c0{bufB, 0, 0, 0, 0}, cc{bufA, 0, 0, 0, 0};
  SAMPT_TRY(res_block(c, st, "fnet.layer3.0.", b, &c0, 128, 2, t1, t2, t3, s));
  SAMPT_TRY(res_block(c, st, "fnet.layer3.1.", c0, &cc, 128, 1, t1, t2, t3, s));
  SAMPT_TRY(resize_ac_concat(c, st, cc.p, cat, n, cc.h, cc.w, 128, Ho, Wo, 416, 160));
  // layer4 (128, stride 2)
  Act d0{bufB, 0, 0, 0, 0}, d{bufA, 0, 0, 0, 0};
  SAMPT_TRY(res_block(c, st, "fnet.layer4.0.", cc, &d0, 128, 2, t1, t2, t3, s));
  SAMPT_TRY(res_block(c, st, "fnet.layer4.1.", d0, &d, 128, 1, t1, t2, t3, s));
  SAMPT_TRY(resize_ac_concat(c, st, d.p, cat, n, d.h, d.w, 128, Ho, Wo, 416, 288));
  // conv2 3x3 416->256, IN, ReLU, conv3 1x1 256->128 (pips.py:279-282)
  Act catA{cat, n, Ho, Wo, 416};
  Act y{bufB, n, Ho, Wo, 256};
  SAMPT_TRY(conv_by_name(c, st, "fnet.conv2", catA, &y, 3, 1, 1));
  SAMPT_TRY(inorm_stats(c, st, y.p, s.stats_a, s.part, n, Ho * Wo, 256));
  SAMPT_TRY(inorm_apply(c, st, y.p, s.stats_a, nullptr, nullptr, y.p, n, Ho * Wo, 256, 1, 0));
  Act out{fmaps_out, n, Ho, Wo, 128};
  SAMPT_TRY(conv_by_name(c, st, "fnet.conv3", y, &out, 1, 1, 0));
  return 0;
}

}  // namespace sampt

using namespace sampt;

static int fnet_frames(Ctx* c, cudaStream_t st, const char* prefix, const void* frames, int is_f32, int T, int H, int W, int stride,
                       float* fmaps) {
  // stride 4: PIPS (configs/model/point_tracker/pips.yaml:3) and CoTracker (cotracker_stride_4_wind_8); stride 8: PIPS++ only
  // (PipsPlusPlus(stride=8), weights "ppp.fnet.*")
  SAMPT_CHECK(stride == 4 || (stride == 8 && std::string(prefix) == "ppp."),
              "fnet: stride %d is not built for the '%s' encoder (4 for PIPS and CoTracker, 8 for PIPS++)", stride, prefix);
  c->fnet_prefix = prefix;
  const int Ho = H / stride, Wo = W / stride;
  // chunk frames so the fp32 half-res activations fit the workspace (6 buffers of n*H2*W2*64 floats + concat)
  const int H2 = (H + 6 - 7) / 2 + 1, W2 = (W + 6 - 7) / 2 + 1;
  size_t per_frame = ((size_t)H2 * W2 * 64 * 5 + (size_t)Ho * Wo * 416) * sizeof(float) + (1 << 20);
  if (fnet_uses_tc(c, c->fnet_prefix))
    per_frame += std::max((size_t)H2 * W2 * 2 * 576, (size_t)Ho * Wo * 2 * 3776) * sizeof(__half);
  int chunk = (int)std::min<size_t>((size_t)T, std::max<size_t>(1, (c->ws_bytes - (8u << 20)) / per_frame));
  SAMPT_CHECK(c->ws_bytes > per_frame + (8u << 20), "workspace too small for one frame of fnet (%zu needed)", per_frame + (8u << 20));
  if (chunk > 16) chunk = 16;
  const size_t esz = is_f32 ? sizeof(float) : sizeof(uint8_t);
  int rc = 0;
  for (int t0 = 0; t0 < T && rc == 0; t0 += chunk) {
    int n = std::min(chunk, T - t0);
    c->ws_reset();
    rc = fnet_chunk(c, st, reinterpret_cast<const char*>(frames) + (size_t)t0 * 3 * H * W * esz, is_f32, n, H, W, stride,
                    fmaps + (size_t)t0 * Ho * Wo * 128);
  }
  c->fnet_prefix = "pips.";
  return rc;
}

extern "C" int sampt_pips_fnet(sampt_ctx* ctx, const uint8_t* frames_u8, int T, int H, int W, int stride, float* fmaps,
                               void* stream) {
  return fnet_frames(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), "pips.", frames_u8, 0, T, H, W, stride, fmaps);
}

// CoTracker's BasicEncoder (same architecture as PIPS', own weights under "cot.fnet.*") over the float clip the
// reference wrapper produces by F.interpolate (sam_pt/point_tracker/cotracker/tracker.py:75-81): values 0..255, normalised
// 2*(x/255)-1 inside conv1 like upstream CoTracker.forward.
extern "C" int sampt_cotracker_fnet(sampt_ctx* ctx, const float* frames_f32, int T, int H, int W, float* fmaps, void* stream) {
  return fnet_frames(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), "cot.", frames_f32, 1, T, H, W, 4, fmaps);
}

// PIPS++'s BasicEncoder (same architecture, own weights under "ppp.fnet.*") at stride 8 over planar frames: uint8, or float32
// holding 0..255 (the tracker's image_size resize); replaces PipsPlusPlus.forward's `self.fnet(2*(rgbs/255)-1)`, once per frame.
extern "C" int sampt_pips_plus_plus_fnet(sampt_ctx* ctx, const void* frames, int is_f32, int T, int H, int W, float* fmaps,
                                         void* stream) {
  return fnet_frames(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), "ppp.", frames, is_f32, T, H, W, 8, fmaps);
}

extern "C" int sampt_pips_pyramid(sampt_ctx* ctx, const float* fmaps, int T, int H4, int W4, float* l1, float* l2,
                                  float* l3, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_TRY(avgpool2_nhwc(c, st, fmaps, l1, T, H4, W4, 128));
  SAMPT_TRY(avgpool2_nhwc(c, st, l1, l2, T, H4 / 2, W4 / 2, 128));
  SAMPT_TRY(avgpool2_nhwc(c, st, l2, l3, T, H4 / 4, W4 / 4, 128));
  return 0;
}

namespace sampt {

__global__ void set_active_kernel(const int* __restrict__ v, const int* __restrict__ wp, uint8_t* __restrict__ active, int N) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n < N) active[n] = (v[n] == wp[0]) ? 1 : 0;
}
__global__ void track_state_init_kernel(const float* __restrict__ q, float* traj, float* vis, int* start, int* cur, int T, int N,
                                        int flip) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  int t = (int)q[n * 3 + 0];  // .long() truncation (pips/tracker.py:57)
  if (flip) t = T - 1 - t;     // query_points_flipped (pips/tracker.py:162-164)
  start[n] = t; cur[n] = t;
  vis[(size_t)t * N + n] = 1.0f;
  traj[((size_t)t * N + n) * 2 + 0] = q[n * 3 + 1];
  traj[((size_t)t * N + n) * 2 + 1] = q[n * 3 + 2];
}

struct MixerW {
  const float *w0, *b0;
  const float *ln0_w[12], *ln0_b[12], *tw1[12], *tb1[12], *tw2[12], *tb2[12];
  const float *ln1_w[12], *ln1_b[12], *cw1[12], *cb1[12], *cw2[12], *cb2[12];
  const float *lnf_w, *lnf_b, *w15, *b15;
  const float *gn_w, *gn_b, *up_w, *up_b, *vis_w, *vis_b;
};

static int load_mixer(Ctx* c, MixerW* m) {
  const std::string p = "pips.delta_block.to_delta.";
  SAMPT_TRY(get_f32(c, p + "0.weight_kpad", &m->w0));
  SAMPT_TRY(get_f32(c, p + "0.bias", &m->b0));
  for (int l = 0; l < 12; ++l) {
    std::string q = p + std::to_string(l + 1);
    SAMPT_TRY(get_f32(c, q + ".0.norm.weight", &m->ln0_w[l]));
    SAMPT_TRY(get_f32(c, q + ".0.norm.bias", &m->ln0_b[l]));
    SAMPT_TRY(get_f32(c, q + ".0.fn.0.weight", &m->tw1[l]));
    SAMPT_TRY(get_f32(c, q + ".0.fn.0.bias", &m->tb1[l]));
    SAMPT_TRY(get_f32(c, q + ".0.fn.3.weight", &m->tw2[l]));
    SAMPT_TRY(get_f32(c, q + ".0.fn.3.bias", &m->tb2[l]));
    SAMPT_TRY(get_f32(c, q + ".1.norm.weight", &m->ln1_w[l]));
    SAMPT_TRY(get_f32(c, q + ".1.norm.bias", &m->ln1_b[l]));
    SAMPT_TRY(get_f32(c, q + ".1.fn.0.weight", &m->cw1[l]));
    SAMPT_TRY(get_f32(c, q + ".1.fn.0.bias", &m->cb1[l]));
    SAMPT_TRY(get_f32(c, q + ".1.fn.3.weight", &m->cw2[l]));
    SAMPT_TRY(get_f32(c, q + ".1.fn.3.bias", &m->cb2[l]));
  }
  SAMPT_TRY(get_f32(c, p + "13.weight", &m->lnf_w));
  SAMPT_TRY(get_f32(c, p + "13.bias", &m->lnf_b));
  SAMPT_TRY(get_f32(c, p + "15.weight", &m->w15));
  SAMPT_TRY(get_f32(c, p + "15.bias", &m->b15));
  SAMPT_TRY(get_f32(c, "pips.norm.weight", &m->gn_w));
  SAMPT_TRY(get_f32(c, "pips.norm.bias", &m->gn_b));
  SAMPT_TRY(get_f32(c, "pips.ffeat_updater.0.weight", &m->up_w));
  SAMPT_TRY(get_f32(c, "pips.ffeat_updater.0.bias", &m->up_b));
  SAMPT_TRY(get_f32(c, "pips.vis_predictor.0.weight", &m->vis_w));
  SAMPT_TRY(get_f32(c, "pips.vis_predictor.0.bias", &m->vis_b));
  return 0;
}

struct IterBufs { float *xin, *x, *xln, *h, *xm, *delta; };

// one refinement iteration of Pips.forward (pips.py:507-546)
static int pips_iteration(Ctx* c, cudaStream_t st, const PipsWin& w, const MixerW& m, const IterBufs& b) {
  const int M = w.N * w.S;
  SAMPT_TRY(pips_corr(c, st, w, b.xin, 520));
  SAMPT_TRY(sgemm_nt(c, st, b.xin, 520, m.w0, 520, m.b0, nullptr, 0, b.x, 512, M, 512, 520, 0));
  for (int l = 0; l < 12; ++l) {
    SAMPT_TRY(mixer_token(c, st, b.x, b.xln, w.active, w.N, m.ln0_w[l], m.ln0_b[l], m.tw1[l], m.tb1[l], m.tw2[l], m.tb2[l],
                          m.ln1_w[l], m.ln1_b[l], 1));
    SAMPT_TRY(sgemm_nt(c, st, b.xln, 512, m.cw1[l], 512, m.cb1[l], nullptr, 0, b.h, 2048, M, 2048, 512, 1));
    SAMPT_TRY(sgemm_nt(c, st, b.h, 2048, m.cw2[l], 2048, m.cb2[l], b.x, 512, b.x, 512, M, 512, 2048, 0));
  }
  SAMPT_TRY(mixer_token(c, st, b.x, b.xln, w.active, w.N, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, m.lnf_w,
                        m.lnf_b, 0));
  SAMPT_TRY(mixer_mean(c, st, b.xln, b.xm, w.N, w.S, 512));
  SAMPT_TRY(sgemm_nt(c, st, b.xm, 512, m.w15, 512, m.b15, nullptr, 0, b.delta, w.S * 130, w.N, w.S * 130, 512, 0));
  SAMPT_TRY(pips_update(c, st, w, b.delta, m.gn_w, m.gn_b, m.up_w, m.up_b));
  return 0;
}

}  // namespace sampt

// One direction of PipsPointTracker._forward (pips/tracker.py:42-153).  `flip` != 0 runs the time-reversed pass on the
// same (unflipped) feature maps by index arithmetic; traj/vis are then in flipped time order (caller flips back).
extern "C" int sampt_pips_track(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int T,
                                int H4, int W4, const float* query_points, int N, int S, int stride, float thr0, int iters,
                                int flip, int max_windows, float* traj, float* vis, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(S == 8, "sampt_pips_track: S must be 8 (pips.yaml s: 8), got %d", S);
  SAMPT_CHECK(N > 0 && T > 0, "sampt_pips_track: empty input");
  c->ws_reset();
  MixerW m;
  SAMPT_TRY(load_mixer(c, &m));
  PipsWin w{};
  w.N = N; w.S = S; w.stride = stride; w.T = T;
  w.pyr[0] = fmaps; w.pyr[1] = l1; w.pyr[2] = l2; w.pyr[3] = l3;
  w.H[0] = H4; w.W[0] = W4;
  for (int l = 1; l < 4; ++l) { w.H[l] = w.H[l - 1] / 2; w.W[l] = w.W[l - 1] / 2; }
  int *start_d, *cur_d; uint8_t* active_d;
  SAMPT_TRY(ws_get(c, &w.coords, (size_t)N * S * 2, "coords"));
  SAMPT_TRY(ws_get(c, &w.ffeats, (size_t)N * S * 128, "ffeats"));
  SAMPT_TRY(ws_get(c, &w.feat_init, (size_t)N * 128, "feat_init"));
  SAMPT_TRY(ws_get(c, &start_d, (size_t)N, "start"));
  SAMPT_TRY(ws_get(c, &cur_d, (size_t)N, "cur"));
  SAMPT_TRY(ws_get(c, &active_d, (size_t)N, "active"));
  IterBufs b;
  const int M = N * S;
  SAMPT_TRY(ws_get(c, &b.xin, (size_t)M * 520, "xin"));
  SAMPT_TRY(ws_get(c, &b.x, (size_t)M * 512, "x"));
  SAMPT_TRY(ws_get(c, &b.xln, (size_t)M * 512, "xln"));
  SAMPT_TRY(ws_get(c, &b.h, (size_t)M * 2048, "h"));
  SAMPT_TRY(ws_get(c, &b.xm, (size_t)N * 512, "xm"));
  SAMPT_TRY(ws_get(c, &b.delta, (size_t)N * S * 130, "delta"));
  w.traj = traj; w.vis = vis; w.cur = cur_d; w.active = active_d;
  SAMPT_CUDA(cudaMemsetAsync(traj, 0, (size_t)T * N * 2 * sizeof(float), st));
  SAMPT_CUDA(cudaMemsetAsync(vis, 0, (size_t)T * N * sizeof(float), st));
  SAMPT_CUDA(cudaMemsetAsync(w.feat_init, 0, (size_t)N * 128 * sizeof(float), st));
  SAMPT_CUDA(cudaMemsetAsync(b.xin, 0, (size_t)M * 520 * sizeof(float), st));
  track_state_init_kernel<<<cdiv(N, 64), 64, 0, st>>>(query_points, traj, vis, start_d, cur_d, T, N, flip);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  SAMPT_CHECK(c->pinned_bytes >= (size_t)N * 2 * sizeof(int), "pinned scratch too small");
  int* start_h = reinterpret_cast<int*>(c->pinned);
  int* cur_h = start_h + N;
  SAMPT_CUDA(cudaMemcpyAsync(start_h, start_d, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost, st));
  SAMPT_CUDA(cudaStreamSynchronize(st));
  for (int n = 0; n < N; ++n) {
    SAMPT_CHECK(start_h[n] >= 0 && start_h[n] < T, "query point %d has timestep %d outside [0,%d)", n, start_h[n], T);
    cur_h[n] = start_h[n];
  }
  int windows_done = 0;
  // per-window parameters live in device memory (w.wp) so that ONE captured CUDA graph of a window (~280 kernels:
  // activity mask, state init, 6 x {corr lookup, 12-layer mixer, update}, vis head + linking) is replayed for every window
  int* wp_d;
  SAMPT_TRY(ws_get(c, &wp_d, 16, "window params"));
  w.wp = wp_d;
  int* wp_h = reinterpret_cast<int*>(reinterpret_cast<char*>(c->pinned) + (64 << 10));
  static const bool use_graphs = []() { const char* e = getenv("SAMPT_PIPS_GRAPHS"); return !(e && e[0] == '0'); }();
  cudaGraphExec_t exec = nullptr;
  long long graph_launches = 0;
  int rc_all = 0;
  for (int f = 0; f < T - 1 && rc_all == 0; ++f) {
    if (max_windows > 0 && windows_done >= max_windows) break;
    bool any = false, born = false;
    for (int n = 0; n < N; ++n) { any |= (cur_h[n] == f); born |= (start_h[n] == f); }
    if (!any) continue;  // pips/tracker.py:69-70
    ++windows_done;
    const int n_missing = std::max(0, f + S - T);
    wp_h[0] = f; wp_h[1] = n_missing;
    for (int s = 0; s < S; ++s) {
      int t = std::min(f + s, T - 1);  // tail padding repeats the last frame (pips/tracker.py:73-78)
      wp_h[2 + s] = flip ? (T - 1 - t) : t;
    }
    SAMPT_CUDA(cudaMemcpyAsync(wp_d, wp_h, 10 * sizeof(int), cudaMemcpyHostToDevice, st));
    if (born) {  // feature-init pass: only ffeat is consumed (pips/tracker.py:81-90; the 6 mixer iterations are dead, SURVEY §0.7-iii)
      set_active_kernel<<<cdiv(N, 64), 64, 0, st>>>(start_d, wp_d, active_d, N);
      c->launches++;
      w.sample_feat = 1;
      SAMPT_TRY(pips_window_init(c, st, w));
    }
    w.sample_feat = 0;
    auto enqueue_window = [&](cudaStream_t s2) -> int {
      set_active_kernel<<<cdiv(N, 64), 64, 0, s2>>>(cur_d, wp_d, active_d, N);
      c->launches++;
      SAMPT_TRY(pips_window_init(c, s2, w));
      for (int it = 0; it < iters; ++it) SAMPT_TRY(pips_iteration(c, s2, w, m, b));
      SAMPT_TRY(pips_link(c, s2, w, m.vis_w, m.vis_b, thr0, T));
      return 0;
    };
    if (!use_graphs) {
      SAMPT_TRY(enqueue_window(st));
    } else {
      if (!exec) {
        if (!c->cap_stream) SAMPT_CUDA(cudaStreamCreateWithFlags(&c->cap_stream, cudaStreamNonBlocking));
        SAMPT_CUDA(cudaStreamSynchronize(st));
        const long long l0 = c->launches;
        SAMPT_CUDA(cudaStreamBeginCapture(c->cap_stream, cudaStreamCaptureModeRelaxed));
        int rc = enqueue_window(c->cap_stream);
        cudaGraph_t graph = nullptr;
        cudaError_t e = cudaStreamEndCapture(c->cap_stream, &graph);
        graph_launches = c->launches - l0;
        c->launches = l0;
        if (rc != 0) return rc;
        SAMPT_CHECK(e == cudaSuccess && graph != nullptr, "stream capture of the PIPS window failed: %s", cudaGetErrorString(e));
        SAMPT_CUDA(cudaGraphInstantiate(&exec, graph, 0));
        cudaGraphDestroy(graph);
      }
      cudaError_t e = cudaGraphLaunch(exec, st);
      if (e != cudaSuccess) { set_error("cudaGraphLaunch(PIPS window): %s", cudaGetErrorString(e)); rc_all = -1; break; }
      c->launches += graph_launches;
    }
    if (cudaMemcpyAsync(cur_h, cur_d, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) {
      set_error("PIPS window read-back failed: %s", cudaGetErrorString(cudaGetLastError()));
      rc_all = -1;
    }
  }
  if (exec) cudaGraphExecDestroy(exec);
  return rc_all;
}

namespace sampt {
// helpers of sampt_pips_window (the reference-compatible Pips.forward on ONE S-frame window)
__global__ void win_seed_kernel(const float* __restrict__ xys, float* __restrict__ traj, uint8_t* __restrict__ active, int N) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  traj[(size_t)n * 2 + 0] = xys[(size_t)n * 2 + 0];     // frame 0 of the (S, N, 2) state = the query position
  traj[(size_t)n * 2 + 1] = xys[(size_t)n * 2 + 1];
  active[n] = 1;
}
// coords_init (S,N,2) px -> window state (N,S,2) feature-map px (pips.py:466: coords = coords_init.clone() / stride)
__global__ void win_coords_in_kernel(const float* __restrict__ ci, float* __restrict__ coords, int N, int S, float inv_stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * S) return;
  const int n = i / S, s = i % S;
  coords[(size_t)i * 2 + 0] = ci[((size_t)s * N + n) * 2 + 0] * inv_stride;
  coords[(size_t)i * 2 + 1] = ci[((size_t)s * N + n) * 2 + 1] * inv_stride;
}
__global__ void win_feat_in_kernel(const float* __restrict__ fi, float* __restrict__ feat_init, float* __restrict__ ffeats, int N, int S) {
  const int n = blockIdx.x, c = threadIdx.x;
  const float f = fi[(size_t)n * 128 + c];
  feat_init[(size_t)n * 128 + c] = f;
  for (int s = 0; s < S; ++s) ffeats[((size_t)n * S + s) * 128 + c] = f;
}
// window state (N,S,2) feature-map px -> one slot of coord_predictions: (S,N,2) px (pips.py:546: coords * stride)
__global__ void win_coords_out_kernel(const float* __restrict__ coords, float* __restrict__ out, int N, int S, float stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * S) return;
  const int n = i / S, s = i % S;
  out[((size_t)s * N + n) * 2 + 0] = coords[(size_t)i * 2 + 0] * stride;
  out[((size_t)s * N + n) * 2 + 1] = coords[(size_t)i * 2 + 1] * stride;
}
// vis_e = Linear(128 -> 1)(ffeats)  (pips.py:568), raw logits (S,N); one warp per (n, s)
__global__ void win_vis_kernel(const float* __restrict__ ffeats, const float* __restrict__ vw, const float* __restrict__ vb,
                               float* __restrict__ vis_e, int N, int S) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= N * S) return;
  const int n = wid / S, s = wid % S;
  const float* ff = ffeats + (size_t)wid * 128;
  float a = 0.f;
  for (int k = lane; k < 128; k += 32) a = fmaf(vw[k], ff[k], a);
  a = warp_sum(a);
  if (lane == 0) vis_e[(size_t)s * N + n] = a + vb[0];
}
}  // namespace sampt

// Reference-compatible Pips.forward on one S-frame window (sam_pt/point_tracker/pips/pips.py:439-620, inference):
//   xys [N,2] px; coords_init [S,N,2] px or NULL (zero-velocity init from xys); feat_init [N,128] or NULL (bilinear sample of
//   frame 0's feature map at xys / stride); `iters` refinement iterations ->
//   coords_out [iters,S,N,2] px (coord_predictions, one entry per iteration), vis_e [S,N] raw visibility logits,
//   ffeat_out [N,128] = the INITIAL feature (what `return_feat=True` returns, pips.py:617-618).
// The pyramid (fmaps,l1,l2,l3) holds exactly S frames.
extern "C" int sampt_pips_window(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int H4, int W4,
                                 const float* xys, const float* coords_init, const float* feat_init, int N, int S, int stride, int iters,
                                 float* coords_out, float* vis_e, float* ffeat_out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(S == 8, "sampt_pips_window: S must be 8, got %d", S);
  SAMPT_CHECK(N > 0 && iters >= 0, "sampt_pips_window: empty input");
  c->ws_reset();
  MixerW m;
  SAMPT_TRY(load_mixer(c, &m));
  PipsWin w{};
  w.N = N; w.S = S; w.stride = stride; w.T = S;
  w.pyr[0] = fmaps; w.pyr[1] = l1; w.pyr[2] = l2; w.pyr[3] = l3;
  w.H[0] = H4; w.W[0] = W4;
  for (int l = 1; l < 4; ++l) { w.H[l] = w.H[l - 1] / 2; w.W[l] = w.W[l - 1] / 2; }
  uint8_t* active_d; int* cur_d; int* wp_d; float *traj_d, *vis_d;
  SAMPT_TRY(ws_get(c, &w.coords, (size_t)N * S * 2, "coords"));
  SAMPT_TRY(ws_get(c, &w.ffeats, (size_t)N * S * 128, "ffeats"));
  SAMPT_TRY(ws_get(c, &w.feat_init, (size_t)N * 128, "feat_init"));
  SAMPT_TRY(ws_get(c, &active_d, (size_t)N, "active"));
  SAMPT_TRY(ws_get(c, &cur_d, (size_t)N, "cur"));
  SAMPT_TRY(ws_get(c, &wp_d, 16, "window params"));
  SAMPT_TRY(ws_get(c, &traj_d, (size_t)S * N * 2, "traj"));
  SAMPT_TRY(ws_get(c, &vis_d, (size_t)S * N, "vis"));
  IterBufs b;
  const int M = N * S;
  SAMPT_TRY(ws_get(c, &b.xin, (size_t)M * 520, "xin"));
  SAMPT_TRY(ws_get(c, &b.x, (size_t)M * 512, "x"));
  SAMPT_TRY(ws_get(c, &b.xln, (size_t)M * 512, "xln"));
  SAMPT_TRY(ws_get(c, &b.h, (size_t)M * 2048, "h"));
  SAMPT_TRY(ws_get(c, &b.xm, (size_t)N * 512, "xm"));
  SAMPT_TRY(ws_get(c, &b.delta, (size_t)N * S * 130, "delta"));
  w.traj = traj_d; w.vis = vis_d; w.cur = cur_d; w.active = active_d; w.wp = wp_d;
  SAMPT_CUDA(cudaMemsetAsync(b.xin, 0, (size_t)M * 520 * sizeof(float), st));
  int* wp_h = reinterpret_cast<int*>(reinterpret_cast<char*>(c->pinned) + (64 << 10));
  wp_h[0] = 0; wp_h[1] = 0;
  for (int s = 0; s < S; ++s) wp_h[2 + s] = s;
  SAMPT_CUDA(cudaMemcpyAsync(wp_d, wp_h, 10 * sizeof(int), cudaMemcpyHostToDevice, st));
  win_seed_kernel<<<cdiv(N, 128), 128, 0, st>>>(xys, traj_d, active_d, N);
  c->launches++;
  w.sample_feat = feat_init ? 0 : 1;
  if (feat_init) { win_feat_in_kernel<<<N, 128, 0, st>>>(feat_init, w.feat_init, w.ffeats, N, S); c->launches++; }
  SAMPT_TRY(pips_window_init(c, st, w));   // zero-velocity coords from frame 0; ffeat sampled (or the given feat_init re-broadcast)
  if (coords_init) { win_coords_in_kernel<<<cdiv(M, 256), 256, 0, st>>>(coords_init, w.coords, N, S, 1.0f / (float)stride); c->launches++; }
  if (ffeat_out) SAMPT_CUDA(cudaMemcpyAsync(ffeat_out, w.feat_init, (size_t)N * 128 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  for (int it = 0; it < iters; ++it) {
    SAMPT_TRY(pips_iteration(c, st, w, m, b));
    win_coords_out_kernel<<<cdiv(M, 256), 256, 0, st>>>(w.coords, coords_out + (size_t)it * S * N * 2, N, S, (float)stride);
    c->launches++;
  }
  win_vis_kernel<<<cdiv((long long)M * 32, 256), 256, 0, st>>>(w.ffeats, m.vis_w, m.vis_b, vis_e, N, S);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// Unit-test entry: fused correlation lookup alone (the "first kernel", SURVEY §7.3).
extern "C" int sampt_pips_corr_lookup(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3,
                                      int S, int H4, int W4, const float* ffeats, const float* coords, int N, float* fcorr,
                                      void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(S >= 1 && S <= 8, "S must be in [1,8]");
  PipsWin w{};
  w.N = N; w.S = S; w.stride = 4; w.T = S;
  c->ws_reset();
  int* wp_d;
  SAMPT_TRY(ws_get(c, &wp_d, 16, "window params"));
  int* wp_h = reinterpret_cast<int*>(reinterpret_cast<char*>(c->pinned) + (64 << 10));
  wp_h[0] = 0; wp_h[1] = 0;
  for (int s = 0; s < 8; ++s) wp_h[2 + s] = s;
  SAMPT_CUDA(cudaMemcpyAsync(wp_d, wp_h, 10 * sizeof(int), cudaMemcpyHostToDevice, st));
  w.wp = wp_d;
  w.pyr[0] = fmaps; w.pyr[1] = l1; w.pyr[2] = l2; w.pyr[3] = l3;
  w.H[0] = H4; w.W[0] = W4;
  for (int l = 1; l < 4; ++l) { w.H[l] = w.H[l - 1] / 2; w.W[l] = w.W[l - 1] / 2; }
  w.coords = const_cast<float*>(coords);
  w.ffeats = const_cast<float*>(ffeats);
  // the PRODUCT kernel (pips_corr_kernel: gather + mixer-row assembly), then the 196 correlation columns of its [N*S, 520] rows are
  // copied out -- the unit test and bench.py's roofline entry exercise exactly the kernel the tracker runs
  uint8_t* active_d; float *traj_d, *xin;
  SAMPT_TRY(ws_get(c, &active_d, (size_t)N, "active"));
  SAMPT_TRY(ws_get(c, &traj_d, (size_t)N * 2, "traj"));
  SAMPT_TRY(ws_get(c, &xin, (size_t)N * S * 520, "xin"));
  SAMPT_CUDA(cudaMemsetAsync(active_d, 1, (size_t)N, st));
  SAMPT_CUDA(cudaMemsetAsync(traj_d, 0, (size_t)N * 2 * sizeof(float), st));
  w.active = active_d; w.traj = traj_d;
  SAMPT_TRY(pips_corr(c, st, w, xin, 520));
  SAMPT_CUDA(cudaMemcpy2DAsync(fcorr, 196 * sizeof(float), xin + 128, 520 * sizeof(float), 196 * sizeof(float), (size_t)N * S,
                               cudaMemcpyDeviceToDevice, st));
  return 0;
}

// ---- unit-test entries: one tracker stage on caller buffers, through the same launchers as the encoder and the window chain --------
static const int* test_window_params(Ctx* c, cudaStream_t st, int f, int n_missing, const int* slots_host, int S) {
  int* wp_d;
  if (ws_get(c, &wp_d, 16, "window params") != 0) return nullptr;
  int* wp_h = reinterpret_cast<int*>(reinterpret_cast<char*>(c->pinned) + (64 << 10));
  wp_h[0] = f; wp_h[1] = n_missing;
  for (int s = 0; s < 8; ++s) wp_h[2 + s] = (slots_host && s < S) ? slots_host[s] : s;
  if (cudaMemcpyAsync(wp_d, wp_h, 10 * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess) {   // the pinned staging slot is reused by the next call
    set_error("test window params: copy failed");
    return nullptr;
  }
  return wp_d;
}

static int test_active(Ctx* c, cudaStream_t st, const uint8_t* active_host, int N, uint8_t** out) {
  SAMPT_TRY(ws_get(c, out, (size_t)N, "active"));
  if (active_host) SAMPT_CUDA(cudaMemcpyAsync(*out, active_host, (size_t)N, cudaMemcpyHostToDevice, st));
  else SAMPT_CUDA(cudaMemsetAsync(*out, 1, (size_t)N, st));
  SAMPT_CUDA(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int sampt_test_pips_conv(sampt_ctx* ctx, const char* name, int tc, const void* in, int is_f32, int Nimg, int H, int W,
                                    int Cin, int Cout, int R, int stride, int pad, float* out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const std::string nm(name);
  c->ws_reset();
  c->fnet_prefix = "pips.";
  c->fnet_im2col = nullptr;
  const int Ho = (H + 2 * pad - R) / stride + 1, Wo = (W + 2 * pad - R) / stride + 1;
  if (tc) {
    const int Kp = nm == "fnet.conv1" ? 192 : ((R * R * Cin + 63) / 64) * 64;
    SAMPT_TRY(ws_get(c, &c->fnet_im2col, (size_t)Nimg * Ho * Wo * 2 * Kp, "fnet im2col operand"));
  }
  int rc;
  if (nm == "fnet.conv1") {
    SAMPT_CHECK(Cin == 3 && Cout == 64 && R == 7 && stride == 2 && pad == 3, "sampt_test_pips_conv: conv1 is 7x7 s2 p3, 3 -> 64");
    rc = conv1_frames(c, st, in, is_f32, Nimg, H, W, out);
  } else {
    SAMPT_CHECK(is_f32, "sampt_test_pips_conv: %s takes fp32 NHWC input", name);
    Act a{const_cast<float*>(static_cast<const float*>(in)), Nimg, H, W, Cin};
    Act o{out, Nimg, Ho, Wo, Cout};
    rc = conv_by_name(c, st, nm, a, &o, R, stride, pad);
  }
  c->fnet_im2col = nullptr;
  return rc;
}

extern "C" int sampt_test_pips_inorm(sampt_ctx* ctx, const float* x, const float* res, int mode, int Nimg, int HW, int C, float* y,
                                     float* stats, float* res_stats, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(mode >= 0 && mode <= 2, "sampt_test_pips_inorm: unknown mode %d", mode);
  SAMPT_CHECK(mode == 0 || res != nullptr, "sampt_test_pips_inorm: mode %d needs a residual", mode);
  c->ws_reset();
  double* part;
  SAMPT_TRY(ws_get(c, &part, (size_t)Nimg * cdiv(HW, 512) * C * 2, "inorm partials"));
  SAMPT_TRY(inorm_stats(c, st, x, stats, part, Nimg, HW, C));
  if (mode == 0) return inorm_apply(c, st, x, stats, nullptr, nullptr, y, Nimg, HW, C, 1, 0);
  if (mode == 1) return inorm_apply(c, st, x, stats, res, nullptr, y, Nimg, HW, C, 1, 1);
  SAMPT_TRY(inorm_stats(c, st, res, res_stats, part, Nimg, HW, C));
  return inorm_apply(c, st, x, stats, res, res_stats, y, Nimg, HW, C, 1, 1);
}

extern "C" int sampt_test_pips_resize(sampt_ctx* ctx, const float* in, int Nimg, int Hi, int Wi, int C, float* out, int Ho, int Wo,
                                      int Ctot, int coff, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_CHECK(C % 4 == 0 && Ctot % 4 == 0 && coff % 4 == 0 && coff + C <= Ctot, "sampt_test_pips_resize: bad channel slice");
  return resize_ac_concat(c, reinterpret_cast<cudaStream_t>(stream), in, out, Nimg, Hi, Wi, C, Ho, Wo, Ctot, coff);
}

extern "C" int sampt_test_pips_corr(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int H4, int W4,
                                    const float* ffeats, const float* coords, int N, int S, const uint8_t* active_host, int f,
                                    int n_missing, const int* slots_host, float* xin, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(S >= 1 && S <= 8 && N >= 1, "sampt_test_pips_corr: S must be in [1,8], N positive");
  c->ws_reset();
  PipsWin w{};
  w.N = N; w.S = S; w.stride = 4; w.T = S;
  w.pyr[0] = fmaps; w.pyr[1] = l1; w.pyr[2] = l2; w.pyr[3] = l3;
  w.H[0] = H4; w.W[0] = W4;
  for (int l = 1; l < 4; ++l) { w.H[l] = w.H[l - 1] / 2; w.W[l] = w.W[l - 1] / 2; }
  w.coords = const_cast<float*>(coords);
  w.ffeats = const_cast<float*>(ffeats);
  w.wp = test_window_params(c, st, f, n_missing, slots_host, S);
  if (w.wp == nullptr) return -1;
  uint8_t* active_d;
  SAMPT_TRY(test_active(c, st, active_host, N, &active_d));
  w.active = active_d;
  return pips_corr(c, st, w, xin, 520);
}

extern "C" int sampt_test_pips_window_op(sampt_ctx* ctx, int op, int N, int S, int T, int stride, int f, int n_missing,
                                         const int* slots_host, const uint8_t* active_host, const float* fmaps, int H4, int W4,
                                         float* coords, float* ffeats, float* feat_init, float* traj, float* vis, int* cur, float* x,
                                         float* xln, int layer, const float* delta, float thr0, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(N >= 1 && S == 8, "sampt_test_pips_window_op: N positive and S == 8 required");
  c->ws_reset();
  MixerW m;
  SAMPT_TRY(load_mixer(c, &m));
  PipsWin w{};
  w.N = N; w.S = S; w.stride = stride; w.T = T;
  w.pyr[0] = fmaps; w.H[0] = H4; w.W[0] = W4;
  w.coords = coords; w.ffeats = ffeats; w.feat_init = feat_init; w.traj = traj; w.vis = vis; w.cur = cur;
  w.wp = test_window_params(c, st, f, n_missing, slots_host, S);
  if (w.wp == nullptr) return -1;
  uint8_t* active_d;
  SAMPT_TRY(test_active(c, st, active_host, N, &active_d));
  w.active = active_d;
  switch (op) {
    case 0:
    case 1:
      w.sample_feat = op;
      return pips_window_init(c, st, w);
    case 2: {
      SAMPT_CHECK(layer >= 0 && layer < 12, "sampt_test_pips_window_op: layer %d out of [0, 12)", layer);
      const int l = layer;
      return mixer_token(c, st, x, xln, w.active, N, m.ln0_w[l], m.ln0_b[l], m.tw1[l], m.tb1[l], m.tw2[l], m.tb2[l], m.ln1_w[l],
                         m.ln1_b[l], 1);
    }
    case 3:
      return mixer_token(c, st, x, xln, w.active, N, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, m.lnf_w, m.lnf_b, 0);
    case 4:
      return mixer_mean(c, st, xln, x, N, S, 512);
    case 5:
      return pips_update(c, st, w, delta, m.gn_w, m.gn_b, m.up_w, m.up_b);
    case 6:
      return pips_link(c, st, w, m.vis_w, m.vis_b, thr0, T);
    default:
      set_error("sampt_test_pips_window_op: unknown op %d", op);
      return -2;
  }
}
