// Host-side orchestration of SAM's ImageEncoderViT (C++; one stream).
// Upstream: segment_anything/modeling/image_encoder.py (un-vendored; SURVEY Appendix B.1); reference call site
// sam_pt/modeling/sam_pt.py:849 (SamPredictor.set_image).  Frames are batched (B) so every GEMM has M = B*4096 (or
// B*4900 window-partitioned rows) and fills every SM.
#include <cstdlib>

#include "common.cuh"
#include "kernels.cuh"
#include "tc_api.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {

__global__ void window_map_kernel(int* __restrict__ map, int B, int G, int ws, int nW, long long total) {
  long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= total) return;
  const int L = ws * ws;
  int t = (int)(r % L);
  long long wb = r / L;
  int w = (int)(wb % (nW * nW)), b = (int)(wb / (nW * nW));
  int y = (w / nW) * ws + t / ws, x = (w % nW) * ws + t % ws;
  map[r] = (y < G && x < G) ? (b * G * G + y * G + x) : -1;
}

// ---- padding-window skip (ON by default, SAMPT_VIT_SKIP_PAD=0 disables; bit-identical, validated on hardware in round 2) -------
// A non-square frame is zero-padded to 1024 x 1024 AFTER normalisation (upstream Sam.preprocess), so every token whose 14x14
// window lies entirely in the padding is image-independent until the first GLOBAL attention block mixes all tokens: its
// value after blocks 0..fg-1 is a constant of the model (weights + pos_embed).  For 480x854 input (576x1024 resized) that
// is 10 of the 25 windows and 1408 of the 4096 tokens in 7 of ViT-H's 32 blocks.  The first encode of a (shape, weights)
// pair runs in full and saves those rows; later encodes run blocks 0..fg-1 on the live windows / tokens only (compacted
// index lists through the existing gather / row-map plumbing) and restore the saved rows before block fg.  Results are
// bit-identical: a GEMM row, a LayerNorm row and a window's attention do not depend on the other rows of the batch.
// live window w = (wy, wx) with wy < lwy, wx < lwx, row-major over the live sub-grid
__global__ void live_window_map_kernel(int* __restrict__ map, int B, int G, int ws, int lwy, int lwx, long long total) {
  long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= total) return;
  const int L = ws * ws;
  int t = (int)(r % L);
  long long wb = r / L;
  int w = (int)(wb % (lwy * lwx)), b = (int)(wb / (lwy * lwx));
  int y = (w / lwx) * ws + t / ws, x = (w % lwx) * ws + t % ws;
  map[r] = (y < G && x < G) ? (b * G * G + y * G + x) : -1;
}
// live tokens: y < rows_live && x < cols_live, row-major
__global__ void live_token_map_kernel(int* __restrict__ map, int B, int G, int rows_live, int cols_live, long long total) {
  long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= total) return;
  const int per = rows_live * cols_live;
  int i = (int)(r % per), b = (int)(r / per);
  map[r] = b * G * G + (i / cols_live) * G + (i % cols_live);
}
// constant tokens of ONE frame (everything that is not live), any fixed order
__global__ void const_token_map_kernel(int* __restrict__ map, int G, int rows_live, int cols_live) {
  int tok = blockIdx.x * blockDim.x + threadIdx.x;
  if (tok >= G * G) return;
  const int y = tok / G, x = tok % G;
  if (y < rows_live && x < cols_live) return;
  const int per_live_row = G - cols_live;
  const int idx = y < rows_live ? y * per_live_row + (x - cols_live) : rows_live * per_live_row + (y - rows_live) * G + x;
  map[idx] = tok;
}
// dst[i, :] = src[map[i], :]  (save)  /  dst[b*GG + map[i], :] = src[i, :] for every frame b  (restore)
__global__ void rows_gather_kernel(const float* __restrict__ src, const int* __restrict__ map, float* __restrict__ dst, int n, int D4) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * D4) return;
  const int r = (int)(i / D4), c = (int)(i % D4);
  reinterpret_cast<float4*>(dst)[(size_t)r * D4 + c] = reinterpret_cast<const float4*>(src)[(size_t)map[r] * D4 + c];
}
__global__ void rows_scatter_bcast_kernel(const float* __restrict__ src, const int* __restrict__ map, float* __restrict__ dst, int n, int D4,
                                          int B, int GG) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)B * n * D4) return;
  const int c = (int)(i % D4);
  const int r = (int)((i / D4) % n), b = (int)(i / ((long long)D4 * n));
  reinterpret_cast<float4*>(dst)[((size_t)b * GG + map[r]) * D4 + c] = reinterpret_cast<const float4*>(src)[(size_t)r * D4 + c];
}
static bool skip_pad_enabled() {
  static const int on = [] { const char* e = std::getenv("SAMPT_VIT_SKIP_PAD"); return (e != nullptr && e[0] == '0') ? 0 : 1; }();   // validated on hardware in round 2: on unless =0
  return on != 0;
}

static GemmSeg make_seg(int precision, int K) {
  GemmSeg s{};
  s.nseg = precision;
  if (precision == 2) {               // weights split only: A.(W_hi + W_lo)
    s.a_off[0] = 0; s.b_off[0] = 0;
    s.a_off[1] = 0; s.b_off[1] = K;
  } else {
    s.a_off[0] = 0; s.b_off[0] = 0;   // hi.hi
    s.a_off[1] = K; s.b_off[1] = 0;   // lo.hi
    s.a_off[2] = 0; s.b_off[2] = K;   // hi.lo
  }
  return s;
}

struct VitDims { int depth, D, nheads, window, G, P, C; };

// img: uint8 frames resized so that the longest side == img_size (normalisation + zero padding fused into the patch im2col), OR
// img_f32: the already preprocessed float image (B,3,img_size,img_size) of upstream ImageEncoderViT.forward (then Hr = Wr =
// img_size: nothing is known about its padding, so the padding-window skip is off)
static int vit_forward(Ctx* c, cudaStream_t st, const uint8_t* img, const float* img_f32, int B, int Hr, int Wr, const VitDims& d,
                       const int* global_idx, int n_global, int precision, const float* mean, const float* stdv, float* features,
                       float* interm) {
  const int D = d.D, G = d.G, GG = G * G, HD = D / d.nheads, ws = d.window;
  const int nW = (G + ws - 1) / ws, Lw = ws * ws;
  const int Mtok = B * GG, Mwin = B * nW * nW * Lw;
  // precision 3 ("mixed", default): MLP / patch-embed / neck GEMMs run all three split passes; the qkv and proj GEMMs run
  // two (weights split).  Their activations are bounded by the fp16 attention path anyway: qkv's OUTPUT is rounded to
  // fp16 for the attention operands and proj's INPUT is the fp16-P x fp16-V attention output, so the A_lo.W_hi pass would add
  // precision that the neighbouring fp16 rounding discards.  precision 4 = all GEMMs three passes.
  // precision 5: like 3, but the attention OUTPUT is carried as fp16 hi|lo and the proj GEMM runs all three passes -- the
  // attention kernel accumulates O in fp32, so this removes the 2^-11 rounding of proj's input; qkv stays at two passes (its
  // output is rounded to fp16 for the attention operands whatever the GEMM does).
  // precision 6: like 4 (every product to ~2^-22), but the two CORRECTION passes of the qkv / proj / lin1 / lin2 GEMMs run in
  // e4m3 wgmma at twice the fp16 rate: A_lo.B_hi and A_hi.B_lo are 2^-12 of the result, so the 2^-5 relative
  // rounding of their fp8 operands leaves a 2^-17 residual (tc_api.cuh: make_seg_f8).  2 fp16-pass equivalents instead of 3.
  const bool f8c = precision == 6;
  const int p_qkv = (precision == 3 || precision == 5) ? 2 : (precision >= 4 ? 3 : precision);
  const int p_proj = precision == 3 ? 2 : (precision >= 4 ? 3 : precision);
  if (precision >= 4) precision = 3;
  const int asp = precision >= 3 ? 2 : 1;  // A operands (activations) carried as hi|lo
  const int bsp = precision >= 2 ? 2 : 1;  // B operands (weights) carried as hi|lo
  const int Kpe = 3 * d.P * d.P;
  const std::string p = "sam.image_encoder.";
  // the encoder allocates from its own slab when one is registered (stream-level overlap with PIPS / decode)
  VitSlabGuard slab_guard(c);

  float* x;           SAMPT_TRY(ws_get(c, &x, (size_t)Mtok * D, "vit x"));
  __half* A;          SAMPT_TRY(ws_get(c, &A, (size_t)std::max(Mwin, Mtok) * std::max(D, Kpe) * asp, "vit A"));
  __half* qkv;        SAMPT_TRY(ws_get(c, &qkv, (size_t)Mwin * 3 * D, "vit qkv"));
  const int DKw = ((HD + 2 * ws + 63) / 64) * 64, DKg = ((HD + 2 * G + 63) / 64) * 64;
  const int Lkpw = ((Lw + 63) / 64) * 64;
  const size_t bh_w = (size_t)B * nW * nW * d.nheads, bh_g = (size_t)B * d.nheads;
  const size_t q_elems = std::max(bh_w * Lw * DKw, bh_g * GG * DKg);
  const size_t v_elems = std::max(bh_w * HD * Lkpw, bh_g * HD * GG);
  __half *Qx, *Kx, *Vt;
  SAMPT_TRY(ws_get(c, &Qx, q_elems, "vit Qx"));
  SAMPT_TRY(ws_get(c, &Kx, q_elems, "vit Kx"));
  SAMPT_TRY(ws_get(c, &Vt, v_elems, "vit Vt"));
  __half* att;        SAMPT_TRY(ws_get(c, &att, (size_t)Mwin * D * asp, "vit attn out"));
  __half* hbuf;       SAMPT_TRY(ws_get(c, &hbuf, (size_t)Mtok * std::max(4 * D, 9 * d.C) * asp, "vit mlp hidden"));
  float* y1;          SAMPT_TRY(ws_get(c, &y1, (size_t)Mtok * d.C * 2, "vit neck y"));
  int* wmap;          SAMPT_TRY(ws_get(c, &wmap, (size_t)Mwin, "vit window map"));
  window_map_kernel<<<cdiv(Mwin, 256), 256, 0, st>>>(wmap, B, G, ws, nW, (long long)Mwin);
  c->launches++;
  SAMPT_LAUNCH_CHECK();

  // ---- optional: skip the image-independent padding windows / tokens in the blocks before the first global block
  int fg = d.depth;
  for (int i = 0; i < n_global; ++i) fg = std::min(fg, global_idx[i]);
  const int lwy = std::min(nW, (int)cdiv(cdiv(Hr, d.P), ws)), lwx = std::min(nW, (int)cdiv(cdiv(Wr, d.P), ws));
  const int rows_live = std::min(G, lwy * ws), cols_live = std::min(G, lwx * ws);
  const int nLW = lwy * lwx, nLT = rows_live * cols_live, n_const = GG - nLT;
  const bool pad_candidate = skip_pad_enabled() && img_f32 == nullptr && fg > 0 && fg < d.depth && n_const > 0;
  int *wmap_c = nullptr, *tmap_c = nullptr, *cmap = nullptr;
  float* x_const = nullptr;   // [n_const, D] saved rows (library-owned, survives the call)
  bool compact = false;       // this call runs blocks < fg on the live rows only
  bool save_const = false;    // this call runs in full and saves the constant rows before block fg
  if (pad_candidate) {
    char key[160];
    snprintf(key, sizeof(key), "vitconst:%dx%d:g%d:w%d:d%d:D%d:fg%d:p%d", Hr, Wr, G, ws, d.depth, D, fg, precision * 100 + p_qkv * 10 + p_proj + (f8c ? 1000 : 0));
    auto it = c->owned.find(key);
    if (it == c->owned.end()) {
      void* buf = nullptr;
      SAMPT_CUDA(cudaMalloc(&buf, (size_t)n_const * D * sizeof(float)));
      c->owned[key] = {buf, 0};   // second = 1 once the rows have been saved
      it = c->owned.find(key);
    }
    x_const = reinterpret_cast<float*>(it->second.first);
    compact = it->second.second == 1;
    save_const = !compact;
    SAMPT_TRY(ws_get(c, &cmap, (size_t)n_const, "vit const-token map"));
    const_token_map_kernel<<<cdiv(GG, 256), 256, 0, st>>>(cmap, G, rows_live, cols_live);
    c->launches++;
    if (compact) {
      SAMPT_TRY(ws_get(c, &wmap_c, (size_t)B * nLW * Lw, "vit live window map"));
      SAMPT_TRY(ws_get(c, &tmap_c, (size_t)B * nLT, "vit live token map"));
      live_window_map_kernel<<<cdiv((long long)B * nLW * Lw, 256), 256, 0, st>>>(wmap_c, B, G, ws, lwy, lwx, (long long)B * nLW * Lw);
      live_token_map_kernel<<<cdiv((long long)B * nLT, 256), 256, 0, st>>>(tmap_c, B, G, rows_live, cols_live, (long long)B * nLT);
      c->launches += 2;
    }
    SAMPT_LAUNCH_CHECK();
    if (save_const) it->second.second = 2;  // "being saved by this call" (set to 1 below, after the copy is enqueued)
  }

  // ---- patch embedding (Conv2d k=16 s=16 as a GEMM) + pos_embed
  {
    if (img_f32) SAMPT_TRY(im2col_f32(c, st, img_f32, A, B, G, d.P, Kpe * asp, asp == 2 ? Kpe : 0));
    else SAMPT_TRY(preprocess_im2col(c, st, img, A, B, Hr, Wr, G, d.P, Kpe * asp, asp == 2 ? Kpe : 0, mean, stdv));
    const __half* w; const float *bias, *pos;
    SAMPT_TRY(get_f16(c, p + "patch_embed.w16", &w));
    SAMPT_TRY(get_f32(c, p + "patch_embed.proj.bias", &bias));
    SAMPT_TRY(get_f32(c, p + "pos_embed", &pos));
    GemmEpi ep{};
    ep.out32 = x; ep.resid = pos; ep.resid_mod = GG; ep.bias = bias; ep.ldc = D;
    SAMPT_TRY(gemm_tc(c, st, A, Kpe * asp, w, Kpe * bsp, Mtok, D, Kpe, make_seg(precision, Kpe), ep));
  }

  int gi = 0;
  for (int blk = 0; blk < d.depth; ++blk) {
    bool is_global = false;
    for (int i = 0; i < n_global; ++i) is_global |= (global_idx[i] == blk);
    const std::string bp = p + "blocks." + std::to_string(blk) + ".";
    const float *n1w, *n1b, *n2w, *n2b, *qkvb, *projb, *l1b, *l2b, *rph, *rpw;
    const __half *wqkv, *wproj, *wl1, *wl2;
    SAMPT_TRY(get_f32(c, bp + "norm1.weight", &n1w)); SAMPT_TRY(get_f32(c, bp + "norm1.bias", &n1b));
    SAMPT_TRY(get_f32(c, bp + "norm2.weight", &n2w)); SAMPT_TRY(get_f32(c, bp + "norm2.bias", &n2b));
    SAMPT_TRY(get_f32(c, bp + "attn.qkv.bias", &qkvb)); SAMPT_TRY(get_f32(c, bp + "attn.proj.bias", &projb));
    SAMPT_TRY(get_f32(c, bp + "mlp.lin1.bias", &l1b)); SAMPT_TRY(get_f32(c, bp + "mlp.lin2.bias", &l2b));
    SAMPT_TRY(get_f32(c, bp + "attn.rel_pos_h", &rph)); SAMPT_TRY(get_f32(c, bp + "attn.rel_pos_w", &rpw));
    SAMPT_TRY(get_f16(c, bp + "attn.qkv.w16", &wqkv)); SAMPT_TRY(get_f16(c, bp + "attn.proj.w16", &wproj));
    SAMPT_TRY(get_f16(c, bp + "mlp.lin1.w16", &wl1)); SAMPT_TRY(get_f16(c, bp + "mlp.lin2.w16", &wl2));
    // fp8-corrected operands of the three large GEMMs (registered by the host next to the hi|lo copies when precision == 6)
    const __half *w8qkv = nullptr, *w8proj = nullptr, *w8l1 = nullptr, *w8l2 = nullptr;
    const float *s8qkv = nullptr, *s8proj = nullptr, *s8l1 = nullptr, *s8l2 = nullptr;
    if (f8c) {
      SAMPT_TRY(get_f16(c, bp + "attn.proj.w8", &w8proj)); SAMPT_TRY(get_f32(c, bp + "attn.proj.w8s", &s8proj));
      SAMPT_TRY(get_f16(c, bp + "attn.qkv.w8", &w8qkv)); SAMPT_TRY(get_f32(c, bp + "attn.qkv.w8s", &s8qkv));
      SAMPT_TRY(get_f16(c, bp + "mlp.lin1.w8", &w8l1)); SAMPT_TRY(get_f32(c, bp + "mlp.lin1.w8s", &s8l1));
      SAMPT_TRY(get_f16(c, bp + "mlp.lin2.w8", &w8l2)); SAMPT_TRY(get_f32(c, bp + "mlp.lin2.w8s", &s8l2));
    }

    if (blk == fg && pad_candidate) {
      const int D4 = D / 4;
      if (save_const) {        // full run: remember the image-independent rows (taken from frame 0)
        rows_gather_kernel<<<cdiv((long long)n_const * D4, 256), 256, 0, st>>>(x, cmap, x_const, n_const, D4);
        c->launches++;
        SAMPT_LAUNCH_CHECK();
        for (auto& kv : c->owned) if (kv.second.first == x_const) kv.second.second = 1;
      } else if (compact) {    // compacted run: put them back before the first global block reads every token
        rows_scatter_bcast_kernel<<<cdiv((long long)B * n_const * D4, 256), 256, 0, st>>>(x_const, cmap, x, n_const, D4, B, GG);
        c->launches++;
        SAMPT_LAUNCH_CHECK();
      }
    }
    const bool live_only = compact && blk < fg;          // windowed block restricted to the live windows / tokens
    const int Mrows = is_global ? Mtok : (live_only ? B * nLW * Lw : Mwin);
    const int Mmlp = live_only ? B * nLT : Mtok;
    const int* blk_wmap = live_only ? wmap_c : wmap;
    const int S = is_global ? G : ws;
    const int L = S * S;
    const int nwb = is_global ? B : (live_only ? B * nLW : B * nW * nW);
    const int DK = is_global ? DKg : DKw;
    const int Lkp = is_global ? GG : Lkpw;
    // which GEMMs of this block take the fp8-corrected form (gemm_f8c_applicable; else three fp16 passes)
    const bool f8_qkv = f8c && gemm_f8c_applicable(Mrows, 3 * D, D);
    const bool f8_proj = f8c && gemm_f8c_applicable(Mrows, D, D);
    const bool f8_l1 = f8c && gemm_f8c_applicable(Mmlp, 4 * D, D);
    const bool f8_l2 = f8c && gemm_f8c_applicable(Mmlp, D, 4 * D);
    // LN1 (+ window partition with zero padding)
    SAMPT_TRY(ln_rows(c, st, x, D, is_global ? nullptr : blk_wmap, n1w, n1b, 1e-6f, A, D * asp, (asp == 2 && p_qkv == 3) ? D : 0, Mrows, D, 1,
                      f8_qkv));
    // qkv = Linear(D, 3D)
    {
      GemmEpi ep{};
      ep.out16 = qkv; ep.bias = qkvb; ep.ldc = 3 * D;
      if (f8_qkv) {
        ep.acc_scale = s8qkv;
        SAMPT_TRY(gemm_tc(c, st, A, D * 2, w8qkv, D * 2, Mrows, 3 * D, D, make_seg_f8(D), ep));
      } else {
        SAMPT_TRY(gemm_tc(c, st, A, D * asp, wqkv, D * bsp, Mrows, 3 * D, D, make_seg(p_qkv, D), ep));
      }
    }
    // attention
    SAMPT_TRY(attn_prep(c, st, qkv, 3 * D, rph, rpw, Qx, Kx, Vt, nwb, d.nheads, S, Lkp, DK, D, HD, 1.0f / sqrtf((float)HD)));
    SAMPT_TRY(attn_tc(c, st, Qx, Kx, Vt, nwb * d.nheads, L, L, Lkp, DK, HD, d.nheads, att, D * asp, (asp == 2 && p_proj == 3) ? D : 0,
                      f8_proj));
    // x = x + proj(attn)   (window un-partition via the row map; padding rows are dropped)
    {
      GemmEpi ep{};
      ep.out32 = x; ep.resid = x; ep.bias = projb; ep.ldc = D; ep.rowmap = is_global ? nullptr : blk_wmap;
      if (f8_proj) {
        ep.acc_scale = s8proj;
        SAMPT_TRY(gemm_tc(c, st, att, D * 2, w8proj, D * 2, Mrows, D, D, make_seg_f8(D), ep));
      } else {
        SAMPT_TRY(gemm_tc(c, st, att, D * asp, wproj, D * bsp, Mrows, D, D, make_seg(p_proj, D), ep));
      }
    }
    // x = x + lin2(gelu(lin1(LN2(x))))
    SAMPT_TRY(ln_rows(c, st, x, D, live_only ? tmap_c : nullptr, n2w, n2b, 1e-6f, A, D * asp, asp == 2 ? D : 0, Mmlp, D, 1, f8_l1));
    {
      GemmEpi ep{};
      ep.out16 = hbuf; ep.bias = l1b; ep.ldc = 4 * D * asp; ep.act = 1; ep.split_off = asp == 2 ? 4 * D : 0;
      ep.out_f8 = f8_l2;   // lin2's A operand in the layout lin2 will read
      if (f8_l1) {
        ep.acc_scale = s8l1;
        SAMPT_TRY(gemm_tc(c, st, A, D * 2, w8l1, D * 2, Mmlp, 4 * D, D, make_seg_f8(D), ep));
      } else {
        SAMPT_TRY(gemm_tc(c, st, A, D * asp, wl1, D * bsp, Mmlp, 4 * D, D, make_seg(precision, D), ep));
      }
    }
    {
      GemmEpi ep{};
      ep.out32 = x; ep.resid = x; ep.bias = l2b; ep.ldc = D; ep.rowmap = live_only ? tmap_c : nullptr;
      if (f8_l2) {
        ep.acc_scale = s8l2;
        SAMPT_TRY(gemm_tc(c, st, hbuf, 4 * D * 2, w8l2, 4 * D * 2, Mmlp, D, 4 * D, make_seg_f8(4 * D), ep));
      } else {
        SAMPT_TRY(gemm_tc(c, st, hbuf, 4 * D * asp, wl2, 4 * D * bsp, Mmlp, D, 4 * D, make_seg(precision, 4 * D), ep));
      }
    }
    if (is_global) {
      if (interm && gi == 0)
        SAMPT_CUDA(cudaMemcpyAsync(interm, x, (size_t)Mtok * D * sizeof(float), cudaMemcpyDeviceToDevice, st));
      ++gi;
    }
  }

  // ---- neck: conv1x1 (no bias) -> LayerNorm2d -> conv3x3 (no bias) -> LayerNorm2d
  {
    const int C = d.C;
    const __half *w0, *w2;
    const float *g1, *b1, *g3, *b3;
    SAMPT_TRY(get_f16(c, p + "neck.0.w16", &w0)); SAMPT_TRY(get_f16(c, p + "neck.2.w16", &w2));
    SAMPT_TRY(get_f32(c, p + "neck.1.weight", &g1)); SAMPT_TRY(get_f32(c, p + "neck.1.bias", &b1));
    SAMPT_TRY(get_f32(c, p + "neck.3.weight", &g3)); SAMPT_TRY(get_f32(c, p + "neck.3.bias", &b3));
    SAMPT_TRY(ln_rows(c, st, x, D, nullptr, nullptr, nullptr, 0.f, A, D * asp, asp == 2 ? D : 0, Mtok, D, 0));  // cast only
    float* y2 = y1 + (size_t)Mtok * C;
    {
      GemmEpi ep{};
      ep.out32 = y1; ep.ldc = C;
      SAMPT_TRY(gemm_tc(c, st, A, D * asp, w0, D * bsp, Mtok, C, D, make_seg(precision, D), ep));
    }
    __half* A2 = hbuf;  // Mtok * 9C * asp halves
    SAMPT_TRY(neck_ln_im2col(c, st, y1, g1, b1, A2, B, G, C, 9 * C * asp, asp == 2 ? 9 * C : 0));
    {
      GemmEpi ep{};
      ep.out32 = y2; ep.ldc = C;
      SAMPT_TRY(gemm_tc(c, st, A2, 9 * C * asp, w2, 9 * C * bsp, Mtok, C, 9 * C, make_seg(precision, 9 * C), ep));
    }
    SAMPT_TRY(neck_ln_nchw(c, st, y2, g3, b3, features, B, GG, C));
  }
  return 0;
}

}  // namespace sampt

using namespace sampt;

extern "C" int sampt_vit_encode(sampt_ctx* ctx, const uint8_t* resized_u8, int B, int Hr, int Wr, int depth, int embed_dim,
                                int num_heads, int window_size, const int* global_idx_host, int n_global, int img_size,
                                int patch_size, int out_chans, int precision, const float* pixel_mean_host,
                                const float* pixel_std_host, float* features, float* interm, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_CHECK(precision >= 1 && precision <= 6, "sampt_vit_encode: precision must be 1..6");
  SAMPT_CHECK(img_size % patch_size == 0, "img_size must be a multiple of patch_size");
  SAMPT_CHECK(Hr <= img_size && Wr <= img_size, "resized image (%dx%d) exceeds img_size %d", Hr, Wr, img_size);
  SAMPT_CHECK(embed_dim % 128 == 0 && embed_dim % num_heads == 0, "embed_dim must be a multiple of 128 and of num_heads");
  VitDims d{depth, embed_dim, num_heads, window_size, img_size / patch_size, patch_size, out_chans};
  return vit_forward(c, reinterpret_cast<cudaStream_t>(stream), resized_u8, nullptr, B, Hr, Wr, d, global_idx_host, n_global, precision,
                     pixel_mean_host, pixel_std_host, features, interm);
}

// upstream ImageEncoderViT.forward(x): x = preprocessed float image (B,3,img_size,img_size), i.e. Sam.preprocess output
extern "C" int sampt_vit_encode_f32(sampt_ctx* ctx, const float* x, int B, int depth, int embed_dim, int num_heads, int window_size,
                                    const int* global_idx_host, int n_global, int img_size, int patch_size, int out_chans,
                                    int precision, float* features, float* interm, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_CHECK(precision >= 1 && precision <= 6, "sampt_vit_encode_f32: precision must be 1..6");
  SAMPT_CHECK(img_size % patch_size == 0, "img_size must be a multiple of patch_size");
  SAMPT_CHECK(embed_dim % 128 == 0 && embed_dim % num_heads == 0, "embed_dim must be a multiple of 128 and of num_heads");
  VitDims d{depth, embed_dim, num_heads, window_size, img_size / patch_size, patch_size, out_chans};
  const float zero[3] = {0.f, 0.f, 0.f}, one[3] = {1.f, 1.f, 1.f};
  return vit_forward(c, reinterpret_cast<cudaStream_t>(stream), nullptr, x, B, img_size, img_size, d, global_idx_host, n_global,
                     precision, zero, one, features, interm);
}

// drop the saved image-independent ViT rows (must be called whenever the image-encoder weights are re-registered)
extern "C" int sampt_vit_cache_clear(sampt_ctx* ctx) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  for (auto it = c->owned.begin(); it != c->owned.end();) {
    if (it->first.compare(0, 9, "vitconst:") == 0) {
      SAMPT_CUDA(cudaDeviceSynchronize());
      cudaFree(it->second.first);
      it = c->owned.erase(it);
    } else {
      ++it;
    }
  }
  return 0;
}

extern "C" int sampt_ctx_set_vit_workspace(sampt_ctx* ctx, void* dev_ptr, size_t bytes) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  c->vit_base = reinterpret_cast<char*>(dev_ptr);
  c->vit_bytes = bytes;
  return 0;
}

extern "C" int sampt_pil_resize_u8(sampt_ctx* ctx, const uint8_t* in, int B, int H, int W, int Ho, int Wo, const int* hbounds,
                                   const int* hcoef, int hksize, const int* vbounds, const int* vcoef, int vksize, uint8_t* tmp,
                                   uint8_t* out, void* stream) {
  return pil_resize(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), in, tmp, out, B, H, W, Ho, Wo, hbounds,
                    hcoef, hksize, vbounds, vcoef, vksize);
}
