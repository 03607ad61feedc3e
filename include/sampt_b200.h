/* libsampt_b200.so — C ABI of the H100-native SAM-PT hot path.
 *
 * The reference (SysCV/sam-pt) has NO FFI: its seam is Python classes named in Hydra YAML (SURVEY.md §8b).  This
 * library sits BEHIND drop-in replacements of those classes (sam-pt_b200/sam_pt, sam-pt_b200/segment_anything[_hq])
 * and is bound with ctypes (sam-pt_b200/sampt_b200/native.py).  Each entry point below cites the reference code it
 * replaces.  Conventions:
 *   - extern "C", plain pointers and sizes, no torch types; every function returns int (0 = ok, <0 = error) and
 *     sampt_last_error() returns a thread-local message; Python surfaces non-zero codes as RuntimeError.
 *   - all tensor arguments are caller-owned DEVICE pointers unless the name ends in _host; layouts are stated per call.
 *   - every call takes a cudaStream_t (as void*) and is stream-ordered; only sampt_pips_track synchronises
 *     the stream (once per processed window, to read back N ints of linking state).
 *   - a ctx belongs to one device and is not thread-safe; distinct ctxs are independent.
 *   - there is no CPU fallback anywhere in this library.
 */
#ifndef SAMPT_B200_H
#define SAMPT_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sampt_ctx sampt_ctx;

/* dtype codes for sampt_set_tensor */
#define SAMPT_F32 0
#define SAMPT_F16 1
#define SAMPT_U8 2
#define SAMPT_I32 3
#define SAMPT_BF16 4

/* ---- context / registry -------------------------------------------------------------------------------------- */
const char* sampt_last_error(void);
int sampt_version(void);
int sampt_ctx_create(int device, sampt_ctx** out);
int sampt_ctx_destroy(sampt_ctx* ctx);
/* caller-owned scratch slab that pipelines bump-allocate from (no cudaMalloc inside the library) */
int sampt_ctx_set_workspace(sampt_ctx* ctx, void* dev_ptr, size_t bytes);
/* optional dedicated slab for sampt_vit_encode, so the encoder can run on its own stream concurrently with the PIPS and
 * decode pipelines (which use the general workspace / decoder slab) */
int sampt_ctx_set_vit_workspace(sampt_ctx* ctx, void* dev_ptr, size_t bytes);
/* optional second slab with STABLE addresses for the SAM decode chain: when set, sampt_sam_predict_refine captures one CUDA
 * graph per chain shape and replays it (one launch per frame instead of ~500).  Re-setting it drops the cached graphs
 * (must be called after decoder weights are re-registered). */
int sampt_ctx_set_decoder_workspace(sampt_ctx* ctx, void* dev_ptr, size_t bytes);
/* register a caller-owned device tensor under a name (weights in kernel-native layout; replaces the
 * load_state_dict contract of sam_pt/modeling/sam.py:18-31 and sam_pt/point_tracker/utils/saverloader.py:30-73) */
int sampt_set_tensor(sampt_ctx* ctx, const char* name, void* dev_ptr, int dtype, int ndim, const int64_t* dims);
/* forget every registered tensor whose name starts with `prefix` (a model that re-registers its weights first drops the
 * names of whatever model used the prefix before, e.g. an HQ-SAM decoder followed by a plain SAM decoder) */
int sampt_unset_tensors(sampt_ctx* ctx, const char* prefix);
/* number of kernels launched through this ctx since creation (bench.py reports the delta as gpu_launches) */
long long sampt_launch_count(sampt_ctx* ctx);

/* ---- PIPS point tracker -------------------------------------------------------------------------------------- */
/* BasicEncoder over uint8 frames (T,3,H,W) -> fmaps (T,H/4,W/4,128) fp32 channels-last.
 * Replaces Pips.forward's `rgbs = 2*(rgbs/255)-1; fmaps = self.fnet(rgbs_)` (sam_pt/point_tracker/pips/pips.py:446-455,
 * BasicEncoder.forward :254-287), computed once per frame instead of once per window. */
int sampt_pips_fnet(sampt_ctx* ctx, const uint8_t* frames_u8, int T, int H, int W, int stride, float* fmaps, void* stream);
/* CorrBlock.__init__ (pips.py:345-362): avg_pool2d pyramid levels 1..3, channels-last. */
int sampt_pips_pyramid(sampt_ctx* ctx, const float* fmaps, int T, int H4, int W4, float* l1, float* l2, float* l3,
                       void* stream);
/* PipsPointTracker._forward (sam_pt/point_tracker/pips/tracker.py:42-153) incl. Pips.forward's iteration loop
 * (pips.py:507-568).  query_points (N,3)=(t,x,y) device fp32; traj (T,N,2), vis (T,N) sigmoid visibilities (NOT yet
 * thresholded at 0.5).  flip != 0 runs the time-reversed pass (tracker.py:161-166); outputs are then in flipped time.
 * max_windows > 0 stops after that many processed windows (1 == a single Pips.forward call; 0 = whole clip). */
int sampt_pips_track(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int T, int H4,
                     int W4, const float* query_points, int N, int S, int stride, float thr0, int iters, int flip,
                     int max_windows, float* traj, float* vis, void* stream);
/* Reference-compatible Pips.forward on ONE S-frame window (sam_pt/point_tracker/pips/pips.py:439-620, inference): the pyramid
 * holds exactly S = 8 frames; xys [N,2] px; coords_init [S,N,2] px or NULL (zero-velocity init, :460-465); feat_init [N,128]
 * or NULL (bilinear_sample2d of frame 0's features, :469-475) -> coords_out [iters,S,N,2] px (one entry per refinement
 * iteration, :546), vis_e [S,N] raw visibility logits (:568), ffeat_out [N,128] the initial feature (`return_feat`, :617-618). */
int sampt_pips_window(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int H4, int W4,
                      const float* xys, const float* coords_init, const float* feat_init, int N, int S, int stride, int iters,
                      float* coords_out, float* vis_e, float* ffeat_out, void* stream);
/* CorrBlock.corr + CorrBlock.sample (pips.py:364-407) fused, for S window slots: ffeats (N,S,128), coords (N,S,2) in
 * level-0 feature pixels, pyramid levels (S,H_l,W_l,128) -> fcorr (N,S,196). */
int sampt_pips_corr_lookup(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int S,
                           int H4, int W4, const float* ffeats, const float* coords, int N, float* fcorr, void* stream);

/* ---- generic fp32 linear (unit tests; torch.nn.functional.linear semantics) ----------------------------------- */
/* Y[M,N] = act(X[M,K] W[N,K]^T + bias) (+ residual); act 0 none / 1 GELU(erf) / 2 ReLU; K,ldx,ldw multiples of 4 */
int sampt_linear_f32(sampt_ctx* ctx, const float* X, int ldx, const float* W, int ldw, const float* bias,
                     const float* residual, int ldr, float* Y, int ldy, int M, int N, int K, int act, void* stream);

/* ---- tensor-core GEMM (tensor-core / registers / TMA), the building block of ImageEncoderViT's Linear layers ------------- */
/* C = act(A[M,K] B[N,K]^T + bias) with fp16 (bf16 if is_bf16) operands and fp32 accumulation.  Exactly one of
 * out16 (fp16/bf16 [M,ldc]) / out32 (fp32 [M,ldc], optional fp32 residual added) is non-null.
 * precision 1: single pass.  2: the weights B are carried as fp16 hi|lo halves, B = [N,2K] with lo at column K (A plain):
 * A.B_hi + A.B_lo.  3: A too (A = [M,2K]); products hi.hi + lo.hi + hi.lo accumulate in the same registers tile (~fp32).
 * split_off > 0 (out16 only): additionally writes lo = fp16(v - fp16(v)) at column offset split_off.
 * Replaces torch.nn.Linear inside segment_anything.modeling.image_encoder (un-vendored; call site
 * sam_pt/modeling/sam_pt.py:849 -> SamPredictor.set_image -> ImageEncoderViT.forward). */
int sampt_gemm_f16(sampt_ctx* ctx, const void* A, int lda, const void* B, int ldb, int M, int N, int K, int precision,
                   int is_bf16, const float* bias, int act, void* out16, float* out32, const float* resid, int ldc,
                   int split_off, void* stream);

/* The same product with the two CORRECTION passes in e4m3 (e4m3 wgmma, twice the fp16 rate): the terms
 * A_lo.B_hi and A_hi.B_lo are 2^-12 of the result, so e4m3's 2^-5 rounding leaves a 2^-17 residual -- fp32-like products
 * for 2 fp16-pass equivalents instead of 3.  Rows of 2K fp16 units:
 *   A: [fp16(x) : K halves | e4m3((x - fp16(x)) * 2^12) : K bytes | e4m3(x * 2^-3) : K bytes]        (sampt_split_f8c)
 *   B: [fp16(w * 2^s) : K halves | e4m3(w * 2^(s-12)) : K bytes | e4m3((w * 2^s - fp16(w * 2^s)) * 2^3) : K bytes]
 * with s the largest exponent keeping |w| * 2^s <= 2^15; acc_scale_dev points to 2^-s.  out_f8 != 0 with split_off = N: the
 * output is written in the A layout of the next such GEMM.  Needs M >= 256, N % 256 == 0, K % 128 == 0 (the shapes of the ViT's linear layers).
 * Same role as sampt_gemm_f16 (torch.nn.Linear of the un-vendored image_encoder; call site sam_pt/modeling/sam_pt.py:849). */
int sampt_gemm_f8c(sampt_ctx* ctx, const void* A, const void* B, int M, int N, int K, const float* acc_scale_dev, const float* bias,
                   int act, void* out16, float* out32, const float* resid, int ldc, int split_off, int out_f8, void* stream);
int sampt_split_f8c(sampt_ctx* ctx, const float* x, int M, int K, void* out, void* stream);

/* softmax(Qx Kx^T) V on tensor cores with pre-extended operands (rel-pos folded into the contraction, see csrc/attn_tc.cu):
 * Qx [BH,Lq,DK], Kx [BH,Lk,DK], Vt [BH,HD,Lkp] fp16; out fp16 [(BH/nheads)*Lq, ld_out] with head h at columns h*HD.
 * Vt's keys in [Lk, Lkp) are row padding and are never read (they need not be zero or even finite).
 * NT (a key-tile size) is accepted and ignored: the kernel walks the keys in tiles of 64.
 * Replaces Attention.forward + add_decomposed_rel_pos of upstream image_encoder.py. */
int sampt_attention_f16(sampt_ctx* ctx, const void* Qx, const void* Kx, const void* Vt, int BH, int Lq, int Lk, int Lkp, int DK,
                        int HD, int NT, int nheads, void* out, int ld_out, int split_off, void* stream);

/* ---- unit-test entries, not used by the Python package -------------------------------------------------------------- */
/* Eleven entries: the ViT's tensor-core GEMM and attention block (below), four stages of the SAM prompt encoder / mask
 * decoder (attention cores, prompt encoder, upscaling tail, postprocess + refinement control), then five of the PIPS tracker. */
/* The ViT's tensor-core GEMM (csrc/gemm_tc.cu, csrc/tc_api.cuh) with every option the pipelines use:
 * C = epilogue(sum over segments i < nseg of A[:, a_off[i] : +K] . B[:, b_off[i] : +K]^T)   (offsets in fp16 units; f8[i] != 0:
 * the segment holds K e4m3 bytes).  a_off_host / b_off_host / f8_host are HOST int[nseg].  Epilogue, in this order: times
 * *acc_scale (device float, or NULL), + bias, act (0 none, 1 GELU erf, 3 GELU tanh; anything else is an error), then either
 * out32 [rows, ldc] (+ resid, read at row % resid_mod when resid_mod > 0; resid may alias out32) or out16 [M, ldc] (bf16 when
 * is_bf16; split_off > 0: lo = fp16(v - hi) at column split_off, or with out_f8 the e4m3 bytes of (v - hi) 2^12 at byte
 * 2 split_off + n and of v 2^-3 at byte 3 split_off + n).  rowmap (device int[M] or NULL): destination row of each output
 * row, -1 = dropped.  skip (device int or NULL): non-zero -> nothing is written. */
int sampt_test_gemm_tc(sampt_ctx* ctx, const void* A, int lda, const void* B, int ldb, int M, int N, int K, int nseg,
                       const int* a_off_host, const int* b_off_host, const int* f8_host, const float* bias, int act, int is_bf16,
                       void* out16, float* out32, const float* resid, int resid_mod, const int* rowmap, const int* skip,
                       const float* acc_scale, int ldc, int split_off, int out_f8, void* stream);
/* One ViT attention block between its qkv GEMM and proj (csrc/vit_pipeline.cu): operand preparation (rel-pos folding) then
 * the attention kernel, scale 1/sqrt(HD), HD = D / nheads.  qkv fp16 [nwb*S*S, 3D] (row = wb*S*S + t, columns q | k | v with
 * head h at h*HD), rel_pos_h / rel_pos_w fp32 [2S-1, HD].  Caller-owned operands: Qx, Kx fp16 [nwb*nheads, S*S, DK],
 * Vt fp16 [nwb*nheads, HD, Lkp].  out, ld_out, split_off, out_f8 as in the attention kernel (the A operand of proj). */
int sampt_test_vit_attention(sampt_ctx* ctx, const void* qkv, const float* rel_pos_h, const float* rel_pos_w, int nwb, int nheads,
                             int S, int D, int DK, int Lkp, void* Qx, void* Kx, void* Vt, void* out, int ld_out, int split_off,
                             int out_f8, void* stream);
/* One SAM decoder attention core (csrc/decoder.cu), 8 heads, on caller-owned fp32 buffers, scale 1/sqrt(head dim):
 *   kind 0: token self-attention, block per (token, head) (the decode chain's kernel for T <= 16), head dim 32: q, k, v,
 *           out [T, 256], Nk == T;
 *   kind 1: token self-attention, warp per query (the chain's kernel for T > 16), same layout; T up to the shared-memory limit;
 *   kind 2: tokens -> image, head dim 16: q, out [T, 128], k, v [Nk, 128]; keys split in slices of 256, then combined
 *           (partials in the ctx workspace);
 *   kind 3: image -> tokens, head dim 16: q, out [Nk, 128] (Nk image tokens), k, v [T, 128] (T prompt tokens). */
int sampt_test_sam_attention(sampt_ctx* ctx, int kind, const float* q, const float* k, const float* v, float* out, int T, int Nk,
                             void* stream);
/* The prompt encoder as the decode chain runs it, with the registered decoder weights: coords (K,2) in the 1024 frame, labels (K)
 * int32, box (4) or NULL, mask_in (256*256) or NULL -> tokens_out [T,256] = output tokens ++ point tokens ++ (pad point | two box
 * corners), src_out [G*G,256] = feat_tok + dense embedding (mask_downscaling(mask_in), or no_mask_embed). */
int sampt_test_sam_prompt(sampt_ctx* ctx, const float* feat_tok, int G, const float* coords, const int* labels, int K, const float* box,
                          const float* mask_in, float* tokens_out, float* src_out, void* stream);
/* The mask decoder's upscaling tail after its first ConvT: u1 [G*G, 4*64] (row = token, column = (dy*2+dx)*64 + c) -> LayerNorm2d,
 * GELU, ConvT(64->32, k2 s2), GELU, dot with hyper [n_masks, 32] (1 <= n_masks <= 4) -> low_res [n_masks, 4G, 4G]; u_out
 * [(4G)^2, 32] receives the upscaled embedding when not NULL. */
int sampt_test_sam_upscale(sampt_ctx* ctx, const float* u1, const float* hyper, int n_masks, int G, float* low_res, float* u_out,
                           void* stream);
/* Sam.postprocess_masks and one step of the refinement control: low_res [n_masks, 4G, 4G] -> out [n_masks, H, W] (bilinear to
 * 16G, crop to in_h x in_w, bilinear to H x W); bbox5 (device int[5]) = xmin, ymin, xmax, ymax, count of out[0] > 0 as
 * accumulated; then the chain's break test: skip (device int) = 1 when count < 2, else box4 (device float[4]) = the box and
 * n_done (device int) = 1. */
int sampt_test_sam_postprocess(sampt_ctx* ctx, const float* low_res, int n_masks, int G, int in_h, int in_w, int H, int W, float* out,
                               int* bbox5, float* box4, int* skip, int* n_done, void* stream);
/* Five stages of the PIPS tracker (csrc/pips_kernels.cu) through the launchers of sampt_pips_fnet / sampt_pips_track, with the
 * registered "pips.*" weights.  slots_host (HOST int[S] or NULL = 0..S-1) is the frame feeding each window slot, active_host (HOST
 * uint8[N] or NULL = all) the points taking part; f and n_missing as in the linking of sam_pt/point_tracker/pips/tracker.py:72-148. */
/* One encoder convolution by weight name ("fnet.conv1", "fnet.layer2.0.conv1", "fnet.conv2", ...): tc != 0 runs im2col + 3-pass
 * tensor-core GEMM (needs the ".w16" weights), else the fp32 CUDA-core kernel.  "fnet.conv1": in = planar frames (Nimg,3,H,W),
 * uint8 (is_f32 == 0) or float 0..255, normalised 2*(x/255)-1 on the fly; any other name: in = fp32 NHWC (Nimg,H,W,Cin).
 * out (Nimg,Ho,Wo,Cout) fp32 NHWC, Ho = (H + 2 pad - R) / stride + 1. */
int sampt_test_pips_conv(sampt_ctx* ctx, const char* name, int tc, const void* in, int is_f32, int Nimg, int H, int W, int Cin,
                         int Cout, int R, int stride, int pad, float* out, void* stream);
/* InstanceNorm2d (eps 1e-5) as ResidualBlock uses it, on x (Nimg,HW,C) NHWC -> y:  mode 0: relu(IN(x));  mode 1: relu(relu(IN(x)) +
 * res);  mode 2: relu(relu(IN(x)) + IN(res)).  stats / res_stats (Nimg,C,2) receive the (mean, rstd) pairs the kernel applies
 * (res_stats only in mode 2).  y may alias x. */
int sampt_test_pips_inorm(sampt_ctx* ctx, const float* x, const float* res, int mode, int Nimg, int HW, int C, float* y, float* stats,
                          float* res_stats, void* stream);
/* F.interpolate(bilinear, align_corners=True) of in (Nimg,Hi,Wi,C) into channels [coff, coff + C) of out (Nimg,Ho,Wo,Ctot). */
int sampt_test_pips_resize(sampt_ctx* ctx, const float* in, int Nimg, int Hi, int Wi, int C, float* out, int Ho, int Wo, int Ctot,
                           int coff, void* stream);
/* The fused correlation lookup with the whole mixer row: pyramid levels (frames,H_l,W_l,128), ffeats (N,S,128), coords (N,S,2)
 * level-0 feature px -> xin (N*S, 520) = [ffeat 128 | corr 196 | sincos(dx,dy,t) 192 | dx,dy,t | 0]; rows of inactive points are
 * not written. */
int sampt_test_pips_corr(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int H4, int W4,
                         const float* ffeats, const float* coords, int N, int S, const uint8_t* active_host, int f, int n_missing,
                         const int* slots_host, float* xin, void* stream);
/* One per-window operation on caller-owned state (S = 8): coords (N,S,2), ffeats (N,S,128), feat_init (N,128), traj (T,N,2),
 * vis (T,N), cur (N) int32.  op 0 / 1: window init (coords = traj[f] / stride, ffeats = feat_init, or with op 1 bilinear_sample2d
 * of fmaps (frames,H4,W4,128) at slot 0's frame, stored into feat_init too); 2: token mixing of mixer layer `layer` (0..11) on x
 * (N,S,512) in place, then the channel-mixing LayerNorm into xln; 3: the final LayerNorm of x into xln; 4: x (N,512) = mean over
 * S of xln; 5: feature / coordinate update from delta (N, S*130); 6: visibility head, trajectory write-back and linking with
 * threshold thr0. */
int sampt_test_pips_window_op(sampt_ctx* ctx, int op, int N, int S, int T, int stride, int f, int n_missing, const int* slots_host,
                              const uint8_t* active_host, const float* fmaps, int H4, int W4, float* coords, float* ffeats,
                              float* feat_init, float* traj, float* vis, int* cur, float* x, float* xln, int layer,
                              const float* delta, float thr0, void* stream);

/* ---- SAM image encoder ------------------------------------------------------------------------------------------ */
/* ResizeLongestSide.apply_image (PIL bilinear, bit-exact): planar uint8 (B,3,H,W) -> (B,3,Ho,Wo); coefficient tables
 * (device int32) come from sampt_b200/pil_resize.py; tmp is a (B,3,H,Wo) uint8 scratch. */
int sampt_pil_resize_u8(sampt_ctx* ctx, const uint8_t* in, int B, int H, int W, int Ho, int Wo, const int* hbounds,
                        const int* hcoef, int hksize, const int* vbounds, const int* vcoef, int vksize, uint8_t* tmp,
                        uint8_t* out, void* stream);
/* Sam.preprocess + ImageEncoderViT.forward for a batch of resized uint8 frames (B,3,Hr,Wr) -> features (B,C,g,g) fp32
 * [+ interm (B,g,g,D): output of the first global-attention block, HQ-SAM].  global_idx / pixel_mean / pixel_std are
 * HOST arrays.  precision: 1/2 as in sampt_gemm_f16 for every GEMM; 3 = 3 split passes for the MLP / patch-embed / neck GEMMs
 * and 2 (weights split) for qkv / proj, whose activations are fp16-limited by the attention path; 4 = 3 passes everywhere;
 * 5 = 3 passes except qkv (2); 6 = like 4 with the correction passes of qkv / lin1 / lin2 in e4m3 (sampt_gemm_f8c; needs the
 * "<layer>.w8" / ".w8s" tensors registered).  Replaces SamPredictor.set_image's encoder call (sam_pt.py:849). */
int sampt_vit_encode(sampt_ctx* ctx, const uint8_t* resized_u8, int B, int Hr, int Wr, int depth, int embed_dim, int num_heads,
                     int window_size, const int* global_idx_host, int n_global, int img_size, int patch_size, int out_chans,
                     int precision, const float* pixel_mean_host, const float* pixel_std_host, float* features, float* interm,
                     void* stream);

/* ---- SAM prompt encoder + mask decoder + postprocess ------------------------------------------------------------- */
/* (C, g*g) NCHW feature map -> token-major (g*g, C) */
int sampt_sam_features_to_tokens(sampt_ctx* ctx, const float* feat_nchw, float* feat_tok, int C, int GG, void* stream);
/* SamPredictor.predict_torch for one prompt set: coords (K,2) in the 1024 frame, labels (K) int32, box (4) or NULL,
 * mask_input (256*256) or NULL; multimask 0 -> 1 mask (token 0), 1 -> 3 masks (tokens 1..3).
 * logits (n,H,W), iou (n), low_res (n,256,256).  Reference call sites sam_pt/modeling/sam_pt.py:783-828. */
int sampt_sam_predict(sampt_ctx* ctx, const float* feat_tok, int G, const float* coords, const int* labels, int K,
                      const float* box, const float* mask_input, int multimask, int in_h, int in_w, int H, int W, float* logits,
                      float* iou, float* low_res, void* stream);
/* SamPt.predict_mask (sam_pt.py:760-837) fused: [positive-only call +] full call + n_refine box/mask refinements with the
 * `mask area < 2` break evaluated on the device (no host synchronisation).  n_refine_done: device int32 [1].
 * n_pos_first > 0: two-call form, the first call on the n_pos_first points of pos_coords / pos_labels (sam_pt.py:792-807); 0: single
 * initial call (:783-790); < 0: two-call form with an EMPTY positive set (first call on the padding point alone).
 * graph_slot selects an independent buffer set / CUDA-graph instance (decoder slab), so chains of different frames may be
 * replayed concurrently on different streams. */
int sampt_sam_predict_refine(sampt_ctx* ctx, const float* feat_tok, int G, const float* coords, const int* labels, int K,
                             const float* pos_coords, const int* pos_labels, int n_pos_first, int n_refine, int in_h, int in_w,
                             int H, int W, float* logits, float* iou, float* low_res, int* n_refine_done, int graph_slot,
                             void* stream);

/* upstream ImageEncoderViT.forward(x): x = the already preprocessed float image (B,3,img_size,img_size) (Sam.preprocess output:
 * normalised, zero-padded) -> features (B,out_chans,G,G) [+ first global block output].  Same pipeline as sampt_vit_encode with a
 * plain float patch im2col; the padding-window skip is off (nothing is known about the padding of a float image). */
int sampt_vit_encode_f32(sampt_ctx* ctx, const float* x, int B, int depth, int embed_dim, int num_heads, int window_size,
                         const int* global_idx_host, int n_global, int img_size, int patch_size, int out_chans, int precision,
                         float* features, float* interm, void* stream);
/* Forget the image-independent ViT rows saved by the experimental SAMPT_VIT_SKIP_PAD=1 path (csrc/vit_pipeline.cu); to be
 * called whenever the image-encoder weights are re-registered.  A no-op when that path is off. */
int sampt_vit_cache_clear(sampt_ctx* ctx);

/* ---- TinyViT image encoder of MobileSAM / Light HQ-SAM (csrc/tinyvit.cu) ------------------------------------------------
 * Upstream mobile_sam/modeling/tiny_vit_sam.py (TinyViT.forward) and sam-hq's copy of it, configuration of
 * configs/model/sam/sam_mobile_vit_tiny.yaml / samhq_light_vit_tiny.yaml (embed_dims 64/128/160/320, depths 2/2/6/2,
 * heads 2/4/5/10, windows 7/7/14/7).  Weights are registered under "sam.tinyvit." (BatchNorm folded, layouts in
 * sam-pt_b200/mobile_sam/modeling/tiny_vit_sam.py).  Work buffers come from the ViT slab (sampt_ctx_set_vit_workspace), whose size
 * for B frames sampt_tinyvit_workspace_bytes returns.
 * sampt_tinyvit_encode replaces SamPredictor.set_image's encoder call (sam_pt.py:849) for these models:
 *   is_f32 = 0: image = resized uint8 frames (B,3,Hr,Wr); Sam.preprocess (normalise with the HOST mean3 / std3, zero-pad
 *               to 1024^2) is fused into the stem's im2col;
 *   is_f32 = 1: image = upstream forward's preprocessed (B,3,1024,1024) float image (Hr, Wr, mean3, std3 unused).
 * feats (B,256,64,64) fp32; interm (B,64,64,160) or NULL: layers.1's output, sam-hq's interm_embeddings[0]. */
int sampt_tinyvit_workspace_bytes(int B, size_t* out);
int sampt_tinyvit_encode(sampt_ctx* ctx, const void* image, int is_f32, int B, int Hr, int Wr, const float* mean3,
                         const float* std3, float* feats, float* interm, void* stream);
/* Unit-test entries; each calls the launchers of sampt_tinyvit_encode.
 * stem: patch_embed.seq (TinyViT.patch_embed) -> out (B,256,256,64) token-major.
 * dwconv: one depthwise Conv2d_BN 3x3 (pad 1, stride 1|2, optional GELU) over x (B,H,W,C), w [9][C] tap-major, bias [C]
 *   -> out32 (B*Ho*Wo, C) and / or out16 (B*Ho*Wo, 2*Kp) fp16 hi|lo with zero columns [C, Kp).
 * block_attn: TinyViTBlock.forward's first half, x + attn(window_partition(pad(x))), of layers.<stage>.blocks.<blk> on x
 *   (B,H,H,C); qkv_out (B*H*H [+1], 3C) receives the qkv GEMM output (the LN(0) row last when the map is padded), attn_out
 *   (B*H*H, 2*pad64(C)) halves the proj GEMM's operand; both optional.
 * stage: layers.<stage> including its PatchMerging, x (B, R*R, C) -> out at the next stage's resolution and width.
 * neck: x (B, 4096, 320) -> feats (B,256,64,64). */
int sampt_test_tinyvit_stem(sampt_ctx* ctx, const void* image, int is_f32, int B, int Hr, int Wr, const float* mean3,
                            const float* std3, float* out, void* stream);
int sampt_test_tinyvit_dwconv(sampt_ctx* ctx, const float* x, const float* w, const float* bias, int B, int H, int W, int C,
                              int stride, int act, float* out32, void* out16, int Kp, void* stream);
int sampt_test_tinyvit_block_attn(sampt_ctx* ctx, int stage, int blk, const float* x, int B, int H, float* out, float* qkv_out,
                                  void* attn_out, void* stream);
int sampt_test_tinyvit_stage(sampt_ctx* ctx, int stage, const float* x, int B, float* out, void* stream);
int sampt_test_tinyvit_neck(sampt_ctx* ctx, const float* x, int B, float* feats, void* stream);

/* HQ-SAM (segment_anything_hq.modeling.mask_decoder_hq.MaskDecoderHQ, un-vendored m43/sam-hq @ 75c73fa; config
 * configs/model/sam/samhq_vit_huge.yaml:19-27).  sampt_sam_hq_features computes the per-frame
 * `embedding_encoder(image_embeddings) + compress_vit_feat(interm_embeddings[0])` map ([16*G*G][32], channels-last);
 * sampt_sam_set_hq_features selects it (NULL = plain SAM) for the following predict calls, whose single-mask output then
 * is mask_sam + mask_hq (hq_token_only=False).  `scratch`: caller-owned G*G*1280 floats (stream-ordered; the call never touches
 * the shared ctx workspace, so frames may be processed concurrently on different streams). */
int sampt_sam_hq_features(sampt_ctx* ctx, const float* feat_tok, const float* interm_tok, int G, float* scratch, float* out,
                          void* stream);
int sampt_sam_set_hq_features(sampt_ctx* ctx, const float* hq_features);

/* ---- CoTracker point tracker (configs/model/point_tracker/cotracker.yaml; sam_pt/point_tracker/cotracker/tracker.py) ---
 * The model itself is the un-vendored facebookresearch/co-tracker @ 4f297a9 (requirements.txt:31), checkpoint
 * cotracker_stride_4_wind_8: PARITY UNPINNED (no golden vectors in the reference; see oracle/cotracker_ref.py). */
/* F.interpolate(rgbs.float(), interp_shape, mode="bilinear") of CoTrackerPointTracker.forward (tracker.py:79-81):
 * uint8 planar (planes,H,W) -> float32 planar (planes,Ho,Wo), align_corners=False. */
int sampt_resize_bilinear_u8_f32(sampt_ctx* ctx, const uint8_t* in, int planes, int H, int W, int Ho, int Wo, float* out,
                                 void* stream);
/* CoTracker's BasicEncoder (weights "cot.fnet.*") over float32 frames (T,3,H,W) holding 0..255 -> (T,H/4,W/4,128)
 * channels-last; replaces `self.fnet(2*(rgbs/255)-1)` of upstream CoTracker.forward, once per frame instead of per window. */
int sampt_cotracker_fnet(sampt_ctx* ctx, const float* frames_f32, int T, int H, int W, float* fmaps, void* stream);
/* feat_init of the points that enter a window (upstream CoTracker.forward: bilinear_sample2d of the point's first-frame
 * feature map at its query coordinate): frame_dev (N) int32 frame index, xy_dev (N,2) feature-map px -> out (N,S,128),
 * the sample repeated over the S slots. */
int sampt_cotracker_sample_features(sampt_ctx* ctx, const float* fmaps, int H4, int W4, const int* frame_dev, const float* xy_dev,
                                    int N, int S, float* out, void* stream);
/* One sliding window of upstream CoTracker.forward_iteration (called through tracker.py:104,159 `self.model(rgbs, queries,
 * iters=6)`): `iters` x { correlation gather, flow/position/time embeddings, UpdateFormer (time/space attention blocks),
 * feature + coordinate update }, then the visibility head.  S = 8 slots.  fidx_dev: device int32[10] = {0, 0, frame index
 * feeding slot 0..7}; coords (N,8,2) feature-map px IN/OUT; ffeats (N,8,128) IN/OUT; track_mask, vis_init (N,8) fp32;
 * time_emb (8,456) fp32 sincos table; vis_out (N,8) raw visibility logits. */
int sampt_cotracker_window(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int H4, int W4,
                           const int* fidx_dev, float* coords, float* ffeats, const float* track_mask, const float* vis_init,
                           const float* time_emb, int N, int iters, int time_depth, int space_depth, float* vis_out,
                           void* stream);

/* ---- SURVEY §8(f) rows: the callers / data formats either side of the hot path ------------------------------------------- */
/* Query points from masks (sam_pt/utils/query_points.py:64-104 -> sklearn_extra.cluster.KMedoids(n_clusters=k).fit(px)
 * .cluster_centers_, un-vendored scikit-learn-extra; defaults metric="euclidean", method="alternate", init="heuristic").
 * Phase 1: pts [n,2] float32 (y,x), n <= 2048 -> D [n,n] float32 (sklearn pairwise_distances arithmetic) and rowsum [n]
 * (numpy float32 pairwise-summation order).  The caller picks the k initial medoids from `rowsum` with numpy's own
 * argpartition (the package's "heuristic" init; its tie order is implementation-defined), then
 * Phase 2: the whole alternate loop on the device (one CTA, no host round trips): medoids [k] int32 IN (initial) / OUT
 * (converged), scratch_i [2n] int32, scratch_f [n] float32, n_iter [1] int32 = iterations executed. */
int sampt_kmedoids_distances(sampt_ctx* ctx, const float* pts, int n, float* D, float* rowsum, void* stream);
int sampt_kmedoids_iterate(sampt_ctx* ctx, const float* D, int n, int k, int max_iter, int* medoids, int* scratch_i,
                           float* scratch_f, int* n_iter, void* stream);
/* Tail of the VOS harness (sam_pt/vos_eval/eval.py:304-355) fused into one kernel: background channel of zero logits, -1e8
 * before each object's query frame gt_ti[i], ground-truth overwrite (nearest resize of gt_masks [M,Hg,Wg]) on it, softmax over
 * the 1+M channels, bilinear up-sampling of the probabilities to (Ho,Wo) when need_resize (align_corners=False), optional
 * horizontal flip, argmax -> uint8 index masks out [T,Ho,Wo].  logits [M,T,H,W] float32 (SamPt.forward's output). */
int sampt_vos_index_masks(sampt_ctx* ctx, const float* logits, int M, int T, int H, int W, const float* gt_masks, int Hg,
                          int Wg, const int* gt_ti, int Ho, int Wo, int need_resize, int flip, uint8_t* out, void* stream);
/* Patch-similarity filtering of tracked points (sam_pt/modeling/sam_pt.py:597-682; use_patch_matching_filtering):
 * frames [T,3,H,W] u8, query [N,3] = (t,x,y), traj [T,N,2]; Lab (skimage rgb2lab arithmetic, channels fed B,G,R as the
 * reference does) patches of patch_size^2 pixels, sim [T,N] = exp(-||patch - query patch|| / (2 ps^2)); vis [T,N] float codes
 * IN/OUT: visible & sim <= threshold -> -3 (PATCH_NON_SIMILAR), then -4 after/before the first such frame. */
int sampt_patch_filter(sampt_ctx* ctx, const uint8_t* frames, int T, int H, int W, const float* query, const float* traj,
                       int N, int patch_size, float threshold, float* vis, float* sim, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SAMPT_B200_H */
