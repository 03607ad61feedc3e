// TinyViT-5M image encoder of MobileSAM and Light HQ-SAM (upstream mobile_sam/modeling/tiny_vit_sam.py and sam-hq's copy of
// it; configuration from configs/model/sam/sam_mobile_vit_tiny.yaml: embed_dims 64/128/160/320, depths 2/2/6/2, heads
// 2/4/5/10, windows 7/7/14/7).  Activations are one channels-last fp32 token-major stream (B*H*W, C), as in the ViT.
//
//   stem        Conv2d_BN 3->32 3x3 s2, GELU, Conv2d_BN 32->64 3x3 s2           im2col + gemm_tc
//   layers.0    2 x MBConv (1x1, dw 3x3, 1x1, + shortcut, GELU) + PatchMerging   gemm_tc, tv_dw3x3, tv_rows (GELU after the residual)
//   layers.1-3  TinyViTBlocks (window attention with a bias table, dw 3x3 local conv, MLP) + PatchMerging
//   neck        1x1 320->256, LayerNorm2d, 3x3, LayerNorm2d                        the ViT's neck launchers (vit_kernels.cu)
//
// Every 1x1 conv, linear and im2col'd 3x3 conv runs on gemm_tc with both operands carried as fp16 hi|lo and three passes
// (~fp32 products, DESIGN §5).  K is padded to a multiple of 64 with zero columns in both operands (27 -> 64, 160 -> 192,
// 288 -> 320), which is exact.  BatchNorm is folded into the conv weight and bias on the host (float64).  The depthwise
// convs, the LayerNorms and the window attention are fp32 CUDA-core kernels.
#include <algorithm>
#include <cmath>
#include <string>

#include "common.cuh"
#include "kernels.cuh"
#include "tc_api.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {

namespace {

constexpr int TV_IMG = 1024;
constexpr int TV_NSTAGE = 4;
constexpr int TV_DIMS[TV_NSTAGE] = {64, 128, 160, 320};
constexpr int TV_DEPTHS[TV_NSTAGE] = {2, 2, 6, 2};
constexpr int TV_HEADS[TV_NSTAGE] = {2, 4, 5, 10};
constexpr int TV_WIN[TV_NSTAGE] = {7, 7, 14, 7};
constexpr int TV_RES[TV_NSTAGE] = {256, 128, 64, 64};   // token grid side of each stage (before its downsample)
constexpr int TV_HD = 32;                               // head dim = key dim at every stage (attn_ratio 1)
constexpr int TV_OUT = 256;                             // neck channels

inline int pad64(int k) { return (k + 63) / 64 * 64; }
// PatchMerging keeps the resolution when out_dim is 320 / 448 / 576 (upstream PatchMerging.__init__)
inline int pm_stride(int out_dim) { return (out_dim == 320 || out_dim == 448 || out_dim == 576) ? 1 : 2; }

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// Stem conv1 im2col: Conv2d(3, 32, 3, stride 2, pad 1) over the preprocessed 1024^2 image, as the A operand of gemm_tc.
// Row m = (b*512 + oy)*512 + ox, column k = (ky*3 + kx)*3 + ci (27 of them, zero to Kp = 64), hi at k, lo at Kp + k.
// uint8 input: Sam.preprocess fused, v = (x - mean) / std inside the resized Hr x Wr frame and 0 in the padding (one fp32
// subtraction and one IEEE division, as torch computes it).  float input: upstream forward's (B,3,1024,1024) image as is.
// ---------------------------------------------------------------------------------------------------------------------
template <bool F32>
__global__ void tv_stem_im2col_kernel(const void* __restrict__ img, __half* __restrict__ A, int Hr, int Wr, int Ho, int Wo,
                                      float m0, float m1, float m2, float s0, float s1, float s2, long long total) {
  constexpr int KP = 64;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k0 = (int)(i % (KP / 8)) * 8;
  const long long m = i / (KP / 8);
  const int ox = (int)(m % Wo), oy = (int)((m / Wo) % Ho);
  const long long b = m / ((long long)Wo * Ho);
  const int S = F32 ? TV_IMG : 0;
  __half hi[8], lo[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = k0 + j;
    float v = 0.f;
    if (k < 27) {
      const int tap = k / 3, ci = k % 3;
      const int iy = 2 * oy + tap / 3 - 1, ix = 2 * ox + tap % 3 - 1;
      if (F32) {
        if (iy >= 0 && iy < S && ix >= 0 && ix < S)
          v = reinterpret_cast<const float*>(img)[((b * 3 + ci) * S + iy) * (long long)S + ix];
      } else if (iy >= 0 && iy < Hr && ix >= 0 && ix < Wr) {
        const float mean = ci == 0 ? m0 : (ci == 1 ? m1 : m2);
        const float sd = ci == 0 ? s0 : (ci == 1 ? s1 : s2);
        v = ((float)reinterpret_cast<const uint8_t*>(img)[((b * 3 + ci) * Hr + iy) * (long long)Wr + ix] - mean) / sd;
      }
    }
    hi[j] = __float2half_rn(v);
    lo[j] = __float2half_rn(v - __half2float(hi[j]));
  }
  __half* row = A + (size_t)m * (2 * KP);
  *reinterpret_cast<uint4*>(row + k0) = *reinterpret_cast<uint4*>(hi);
  *reinterpret_cast<uint4*>(row + KP + k0) = *reinterpret_cast<uint4*>(lo);
}

// ---------------------------------------------------------------------------------------------------------------------
// Depthwise 3x3 conv (pad 1, stride 1 or 2) with folded BatchNorm, optional GELU, over a token-major (B, H, W, C) fp32 map.
// One thread per (output pixel, channel): consecutive threads take consecutive channels, so every load and store is coalesced.
//   out32 != null: fp32 (B*Ho*Wo, C)
//   out16 != null: the next GEMM's A operand, hi at column c and lo at Kp + c of a 2*Kp row, zero columns [C, Kp)
// w is [9][C] (tap-major), bias [C].  Taps are accumulated in order ky, kx, then the bias is added.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void tv_dw3x3_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                                float* __restrict__ out32, __half* __restrict__ out16, int Kp, int H, int W, int C, int Ho, int Wo,
                                int stride, int act, int cols, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % cols);
  const long long m = i / cols;
  float v = 0.f;
  if (c < C) {
    const int ox = (int)(m % Wo), oy = (int)((m / Wo) % Ho);
    const long long b = m / ((long long)Wo * Ho);
    float acc = 0.f;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = oy * stride + ky - 1;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = ox * stride + kx - 1;
        if (ix < 0 || ix >= W) continue;
        acc = fmaf(in[((b * H + iy) * W + ix) * C + c], __ldg(w + (ky * 3 + kx) * C + c), acc);
      }
    }
    v = acc + __ldg(bias + c);
    if (act) v = gelu_erf(v);
    if (out32) out32[m * C + c] = v;
  }
  if (out16) {
    const __half h = __float2half_rn(v);
    out16[m * 2 * Kp + c] = h;
    out16[m * 2 * Kp + Kp + c] = __float2half_rn(v - __half2float(h));
  }
}

int tv_dw3x3(Ctx* c, cudaStream_t st, const float* in, const float* w, const float* bias, float* out32, __half* out16, int Kp, int B,
             int H, int W, int C, int stride, int act) {
  SAMPT_CHECK(stride == 1 || stride == 2, "tv_dw3x3: stride %d must be 1 or 2", stride);
  SAMPT_CHECK(out32 != nullptr || out16 != nullptr, "tv_dw3x3: no output");
  SAMPT_CHECK(out16 == nullptr || Kp >= C, "tv_dw3x3: Kp %d < C %d", Kp, C);
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const int cols = out16 ? Kp : C;
  const long long total = (long long)B * Ho * Wo * cols;
  tv_dw3x3_kernel<<<cdiv(total, 256), 256, 0, st>>>(in, w, bias, out32, out16, Kp, H, W, C, Ho, Wo, stride, act, cols, total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Row kernel, one warp per row of a (M, C) fp32 matrix, C % 32 == 0, C <= 320:
//   mode 0: y = x            mode 1: y = LayerNorm(x) (two-pass mean / variance, eps)            mode 2: y = GELU(x)
// y goes to the A operand (hi | lo, 2*Kp halves per row, zero columns [C, Kp)) and, when out32 != null, to out32 (may alias
// x).  beta_row != 0 appends row M = LN(0) = beta: the value every zero-padded window token has after the attention's
// LayerNorm (the qkv GEMM turns it into the one key / value row of the padding).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
tv_rows_kernel(const float* x, int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int mode, float* out32,
               __half* __restrict__ A, int Kp, int M, int beta_row) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M + (beta_row ? 1 : 0)) return;
  const int nper = C / 32;
  float v[10];
  if (row == M) {
#pragma unroll
    for (int i = 0; i < 10; ++i) if (i < nper) v[i] = beta[lane + 32 * i];
  } else {
    const float* xp = x + row * C;
#pragma unroll
    for (int i = 0; i < 10; ++i) if (i < nper) v[i] = xp[lane + 32 * i];
    if (mode == 1) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 10; ++i) if (i < nper) s += v[i];
      const float mean = warp_sum(s) / (float)C;
      float sq = 0.f;
#pragma unroll
      for (int i = 0; i < 10; ++i) if (i < nper) { const float d = v[i] - mean; sq += d * d; }
      const float rstd = 1.0f / sqrtf(warp_sum(sq) / (float)C + eps);
#pragma unroll
      for (int i = 0; i < 10; ++i) if (i < nper) v[i] = (v[i] - mean) * rstd * gamma[lane + 32 * i] + beta[lane + 32 * i];
    } else if (mode == 2) {
#pragma unroll
      for (int i = 0; i < 10; ++i) if (i < nper) v[i] = gelu_erf(v[i]);
    }
    if (out32) {
      float* op = out32 + row * C;
#pragma unroll
      for (int i = 0; i < 10; ++i) if (i < nper) op[lane + 32 * i] = v[i];
    }
  }
  __half* o = A + row * 2 * Kp;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    if (i < nper) {
      const __half h = __float2half_rn(v[i]);
      o[lane + 32 * i] = h;
      o[Kp + lane + 32 * i] = __float2half_rn(v[i] - __half2float(h));
    }
  }
  for (int cc = C + lane; cc < Kp; cc += 32) { o[cc] = __float2half_rn(0.f); o[Kp + cc] = __float2half_rn(0.f); }
}

int tv_rows(Ctx* c, cudaStream_t st, const float* x, int C, const float* gamma, const float* beta, float eps, int mode, float* out32,
            __half* A, int Kp, int M, int beta_row) {
  SAMPT_CHECK(C % 32 == 0 && C <= 320 && Kp >= C, "tv_rows: C=%d must be a multiple of 32, <= 320 and <= Kp=%d", C, Kp);
  SAMPT_CHECK(mode >= 0 && mode <= 2, "tv_rows: mode %d", mode);
  SAMPT_CHECK(!beta_row || beta != nullptr, "tv_rows: the beta row needs beta");
  const long long rows = (long long)M + (beta_row ? 1 : 0);
  tv_rows_kernel<<<cdiv(rows, 8), 256, 0, st>>>(x, C, gamma, beta, eps, mode, out32, A, Kp, M, beta_row);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Window attention with TinyViT's bias table, fp32.  One CTA per (window, head, frame), 8 warps.
//   qkv   (B*H*W + 1, 3C) fp32, token-major rows; row B*H*W = qkv(LN(0)), the key / value of every zero-padded token.
//         Head h owns columns [96h, 96h+96) laid out q | k | v (upstream qkv.view(B, N, heads, -1).split([32, 32, 32])).
//   ab    (heads, ws*ws): bias of tokens i, j = ab[h, |r_i - r_j|*ws + |c_i - c_j|] (token n = r*ws + c in the window).
//   out   the proj GEMM's A operand, rows in token order (valid tokens only), hi at column 32h + d, lo at Kp + 32h + d.
// A window's keys / values are read straight from qkv through the window and padding index arithmetic into shared memory
// (row pitch 33: conflict-free for both the key-per-lane score loop and the dim-per-lane PV loop).  Each warp takes one
// query at a time: lane j owns keys j, j+32, ...; the softmax runs over the whole row in registers; then lane d sums p.V.
// ---------------------------------------------------------------------------------------------------------------------
template <int WS>
__global__ void __launch_bounds__(256)
tv_window_attn_kernel(const float* __restrict__ qkv, const float* __restrict__ ab, __half* __restrict__ out, int Kp, int H, int W, int C,
                      int nheads, int nWx, float scale) {
  constexpr int L = WS * WS, KPL = (L + 31) / 32, PITCH = TV_HD + 1;
  extern __shared__ float sm[];
  float* sk = sm;                  // [L][33]
  float* sv = sk + L * PITCH;      // [L][33]
  float* sb = sv + L * PITCH;      // [L] bias table of this head
  float* sp = sb + L;              // [8][L] probabilities per warp
  const int wy = blockIdx.x / nWx, wx = blockIdx.x % nWx, h = blockIdx.y, b = blockIdx.z;
  const int ld = 3 * C;
  const long long pad_row = (long long)gridDim.z * H * W;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < L * TV_HD; i += 256) {
    const int t = i / TV_HD, d = i % TV_HD;
    const int ty = wy * WS + t / WS, tx = wx * WS + t % WS;
    const long long row = (ty < H && tx < W) ? ((long long)b * H + ty) * W + tx : pad_row;
    const float* rp = qkv + row * ld + h * 3 * TV_HD;
    sk[t * PITCH + d] = rp[TV_HD + d];
    sv[t * PITCH + d] = rp[2 * TV_HD + d];
  }
  for (int i = threadIdx.x; i < L; i += 256) sb[i] = ab[h * L + i];
  __syncthreads();
  float* p = sp + warp * L;
  for (int t = warp; t < L; t += 8) {
    const int ry = t / WS, rx = t % WS;
    const int ty = wy * WS + ry, tx = wx * WS + rx;
    if (ty >= H || tx >= W) continue;                   // warp-uniform: padded queries are discarded upstream
    const long long orow = ((long long)b * H + ty) * W + tx;
    const float q = qkv[orow * ld + h * 3 * TV_HD + lane];
    float s[KPL];
#pragma unroll
    for (int i = 0; i < KPL; ++i) s[i] = 0.f;
#pragma unroll 8
    for (int d = 0; d < TV_HD; ++d) {
      const float qd = __shfl_sync(0xffffffffu, q, d);
#pragma unroll
      for (int i = 0; i < KPL; ++i) {
        const int j = lane + 32 * i;
        if (j < L) s[i] = fmaf(qd, sk[j * PITCH + d], s[i]);
      }
    }
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < KPL; ++i) {
      const int j = lane + 32 * i;
      if (j < L) {
        const int dy = abs(ry - j / WS), dx = abs(rx - j % WS);
        s[i] = s[i] * scale + sb[dy * WS + dx];
        mx = fmaxf(mx, s[i]);
      }
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < KPL; ++i) {
      const int j = lane + 32 * i;
      if (j < L) { s[i] = expf(s[i] - mx); sum += s[i]; }
    }
    const float inv = 1.0f / warp_sum(sum);
#pragma unroll
    for (int i = 0; i < KPL; ++i) {
      const int j = lane + 32 * i;
      if (j < L) p[j] = s[i] * inv;
    }
    __syncwarp();
    float o = 0.f;
    for (int j = 0; j < L; ++j) o = fmaf(p[j], sv[j * PITCH + lane], o);
    __syncwarp();
    __half* op = out + orow * 2 * Kp;
    const __half hv = __float2half_rn(o);
    op[h * TV_HD + lane] = hv;
    op[Kp + h * TV_HD + lane] = __float2half_rn(o - __half2float(hv));
    if (h == 0)
      for (int cc = C + lane; cc < Kp; cc += 32) { op[cc] = __float2half_rn(0.f); op[Kp + cc] = __float2half_rn(0.f); }
  }
}

int tv_window_attn(Ctx* c, cudaStream_t st, const float* qkv, const float* ab, __half* out, int Kp, int B, int H, int W, int C,
                   int nheads, int ws) {
  SAMPT_CHECK(C == nheads * TV_HD && Kp >= C, "tv_window_attn: C=%d must be %d heads x %d (Kp=%d)", C, nheads, TV_HD, Kp);
  const int nWy = (H + ws - 1) / ws, nWx = (W + ws - 1) / ws;
  dim3 grid(nWy * nWx, nheads, B);
  const float scale = (float)(1.0 / std::sqrt((double)TV_HD));
  const size_t smem = (size_t)(ws * ws * (2 * (TV_HD + 1) + 1 + 8)) * sizeof(float);
  if (ws == 7) {
    SAMPT_TRY(ensure_func_smem(c, "tv_window_attn_kernel<7>", tv_window_attn_kernel<7>, smem));
    tv_window_attn_kernel<7><<<grid, 256, smem, st>>>(qkv, ab, out, Kp, H, W, C, nheads, nWx, scale);
  } else if (ws == 14) {
    SAMPT_TRY(ensure_func_smem(c, "tv_window_attn_kernel<14>", tv_window_attn_kernel<14>, smem));
    tv_window_attn_kernel<14><<<grid, 256, smem, st>>>(qkv, ab, out, Kp, H, W, C, nheads, nWx, scale);
  } else {
    SAMPT_CHECK(false, "tv_window_attn: window %d not built (7 and 14)", ws);
  }
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------------------
const std::string TV_PREFIX = "sam.tinyvit.";

// three fp16 passes A_hi.B_hi + A_lo.B_hi + A_hi.B_lo over operands of 2*Kp halves per row
GemmSeg seg3(int Kp) {
  GemmSeg s{};
  s.nseg = 3;
  s.a_off[0] = 0;  s.b_off[0] = 0;
  s.a_off[1] = Kp; s.b_off[1] = 0;
  s.a_off[2] = 0;  s.b_off[2] = Kp;
  return s;
}

// Y[M, N] = act(A W^T + bias) (+ resid): A [M, 2Kp] and W [N, 2Kp] hi|lo, W registered as w 2^s with "<name>s" = 2^-s
// (the accumulator scale).  Epilogue order: scale -> bias -> act -> residual.
int tv_gemm(Ctx* c, cudaStream_t st, const __half* A, const std::string& wname, int M, int N, int Kp, const float* bias, int act,
            float* out32, const float* resid) {
  const __half* w;
  const float* ws;
  SAMPT_TRY(get_f16(c, wname, &w));
  SAMPT_TRY(get_f32(c, wname + "s", &ws));
  GemmEpi ep{};
  ep.out32 = out32; ep.resid = resid; ep.bias = bias; ep.act = act; ep.ldc = N; ep.acc_scale = ws;
  return gemm_tc(c, st, A, 2 * Kp, w, 2 * Kp, M, N, Kp, seg3(Kp), ep);
}

namespace {

struct TvBufs {
  float *X, *X2, *F, *QKV;
  __half* A;
};

// per-frame buffer sizes (elements): the largest use of each buffer over the whole encoder
constexpr size_t TV_X_PER = 65536ull * 64;          // stage-0 tokens x 64 (also >= every later stage's tokens x C)
constexpr size_t TV_F_PER = 65536ull * 256;         // MBConv hidden (also the stem conv1 output, PatchMerging hidden, MLP hidden
                                                    // as fp16 hi|lo, the neck's two fp32 maps)
constexpr size_t TV_QKV_PER = 16384ull * 384;       // stage-1 qkv
constexpr size_t TV_A_PER = 65536ull * 2 * 320;     // stem conv2's im2col operand, the largest A

size_t tv_workspace_bytes(int B) {
  const size_t f = sizeof(float), h = sizeof(__half);
  return (2 * TV_X_PER * f + TV_F_PER * f + TV_QKV_PER * f + TV_A_PER * h) * (size_t)B + 1024 * f + 8 * 256;
}


int tv_alloc(Ctx* c, int B, TvBufs* t) {
  SAMPT_TRY(ws_get(c, &t->X, TV_X_PER * B, "tinyvit x"));
  SAMPT_TRY(ws_get(c, &t->X2, TV_X_PER * B, "tinyvit x2"));
  SAMPT_TRY(ws_get(c, &t->F, TV_F_PER * B, "tinyvit hidden"));
  SAMPT_TRY(ws_get(c, &t->QKV, TV_QKV_PER * B + 1024, "tinyvit qkv"));
  SAMPT_TRY(ws_get(c, &t->A, TV_A_PER * B, "tinyvit A"));
  return 0;
}

// patch_embed.seq -> X (B*256*256, 64)
int tv_stem(Ctx* c, cudaStream_t st, const void* img, int is_f32, int B, int Hr, int Wr, const float* mean, const float* stdv,
            TvBufs& t) {
  const std::string p = TV_PREFIX + "patch_embed.seq.";
  const float *b0, *b2;
  SAMPT_TRY(get_f32(c, p + "0.b", &b0));
  SAMPT_TRY(get_f32(c, p + "2.b", &b2));
  const int H1 = TV_IMG / 2, H2 = TV_IMG / 4;
  const long long M1 = (long long)B * H1 * H1, M2 = (long long)B * H2 * H2;
  const long long total = M1 * 8;
  if (is_f32)
    tv_stem_im2col_kernel<true><<<cdiv(total, 256), 256, 0, st>>>(img, t.A, TV_IMG, TV_IMG, H1, H1, 0.f, 0.f, 0.f, 1.f, 1.f, 1.f, total);
  else
    tv_stem_im2col_kernel<false><<<cdiv(total, 256), 256, 0, st>>>(img, t.A, Hr, Wr, H1, H1, mean[0], mean[1], mean[2], stdv[0],
                                                                   stdv[1], stdv[2], total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  SAMPT_TRY(tv_gemm(c, st, t.A, p + "0.w16", (int)M1, 32, 64, b0, 1, t.F, nullptr));       // conv1 + BN, GELU
  SAMPT_TRY(im2col_nhwc_split(c, st, t.F, t.A, B, H1, H1, 32, 3, 3, 2, 1, 320));           // k = (ky*3 + kx)*32 + ci
  SAMPT_TRY(tv_gemm(c, st, t.A, p + "2.w16", (int)M2, 64, 320, b2, 0, t.X, nullptr));      // conv2 + BN
  return 0;
}

// PatchMerging: the split of X (Kp_in = pad64(Cin)) is in A.  X <- conv3(GELU(dw(GELU(conv1(x)))))
int tv_patch_merging(Ctx* c, cudaStream_t st, const std::string& p, int B, int H, int Cin, int Cout, TvBufs& t) {
  const float *b1, *dw, *b2, *b3;
  SAMPT_TRY(get_f32(c, p + "conv1.b", &b1));
  SAMPT_TRY(get_f32(c, p + "conv2.w", &dw)); SAMPT_TRY(get_f32(c, p + "conv2.b", &b2));
  SAMPT_TRY(get_f32(c, p + "conv3.b", &b3));
  const int s = pm_stride(Cout), Ho = (H - 1) / s + 1;
  SAMPT_TRY(tv_gemm(c, st, t.A, p + "conv1.w16", B * H * H, Cout, pad64(Cin), b1, 1, t.F, nullptr));
  SAMPT_TRY(tv_dw3x3(c, st, t.F, dw, b2, nullptr, t.A, pad64(Cout), B, H, H, Cout, s, 1));
  SAMPT_TRY(tv_gemm(c, st, t.A, p + "conv3.w16", B * Ho * Ho, Cout, pad64(Cout), b3, 0, t.X, nullptr));
  return 0;
}

// MBConv: the split of X (Kp = 64) is in A on entry and on exit.  X <- GELU(X + conv3(GELU(dw(GELU(conv1(X))))))
int tv_mbconv(Ctx* c, cudaStream_t st, const std::string& p, int B, int H, int C, TvBufs& t) {
  const float *b1, *dw, *b2, *b3;
  SAMPT_TRY(get_f32(c, p + "conv1.b", &b1));
  SAMPT_TRY(get_f32(c, p + "conv2.w", &dw)); SAMPT_TRY(get_f32(c, p + "conv2.b", &b2));
  SAMPT_TRY(get_f32(c, p + "conv3.b", &b3));
  const int M = B * H * H, Ch = 4 * C;
  SAMPT_TRY(tv_gemm(c, st, t.A, p + "conv1.w16", M, Ch, pad64(C), b1, 1, t.F, nullptr));
  SAMPT_TRY(tv_dw3x3(c, st, t.F, dw, b2, nullptr, t.A, pad64(Ch), B, H, H, Ch, 1, 1));
  SAMPT_TRY(tv_gemm(c, st, t.A, p + "conv3.w16", M, C, pad64(Ch), b3, 0, t.X, t.X));     // + shortcut
  // GELU after the residual, written as fp32 (the next shortcut) and as the next GEMM's hi|lo operand
  return tv_rows(c, st, t.X, C, nullptr, nullptr, 0.f, 2, t.X, t.A, pad64(C), M, 0);
}

// x = x + proj(attn(window_partition(pad(x)))) over X (B, H, H, C)
int tv_block_attn(Ctx* c, cudaStream_t st, const std::string& p, int B, int H, int C, int heads, int ws, TvBufs& t) {
  const float *nw, *nb, *qb, *pb, *ab;
  SAMPT_TRY(get_f32(c, p + "attn.norm.weight", &nw)); SAMPT_TRY(get_f32(c, p + "attn.norm.bias", &nb));
  SAMPT_TRY(get_f32(c, p + "attn.qkv.bias", &qb)); SAMPT_TRY(get_f32(c, p + "attn.proj.bias", &pb));
  SAMPT_TRY(get_f32(c, p + "attn.attention_biases", &ab));
  const int M = B * H * H, Kp = pad64(C);
  // LN rows of the valid tokens + one LN(0) = beta row for the zero padding (skipped when the map tiles exactly)
  const int pad_row = (H % ws) != 0;
  SAMPT_TRY(tv_rows(c, st, t.X, C, nw, nb, 1e-5f, 1, nullptr, t.A, Kp, M, pad_row));
  SAMPT_TRY(tv_gemm(c, st, t.A, p + "attn.qkv.w16", M + pad_row, 3 * C, Kp, qb, 0, t.QKV, nullptr));
  SAMPT_TRY(tv_window_attn(c, st, t.QKV, ab, t.A, Kp, B, H, H, C, heads, ws));
  return tv_gemm(c, st, t.A, p + "attn.proj.w16", M, C, Kp, pb, 0, t.X, t.X);
}

// one TinyViTBlock over X: attention half, local_conv (depthwise 3x3 + BN, no residual), x = x + mlp(x)
int tv_block(Ctx* c, cudaStream_t st, const std::string& p, int B, int H, int C, int heads, int ws, TvBufs& t) {
  SAMPT_TRY(tv_block_attn(c, st, p, B, H, C, heads, ws, t));
  const float *lw, *lb, *nw, *nb, *f1b, *f2b;
  SAMPT_TRY(get_f32(c, p + "local_conv.w", &lw)); SAMPT_TRY(get_f32(c, p + "local_conv.b", &lb));
  SAMPT_TRY(get_f32(c, p + "mlp.norm.weight", &nw)); SAMPT_TRY(get_f32(c, p + "mlp.norm.bias", &nb));
  SAMPT_TRY(get_f32(c, p + "mlp.fc1.bias", &f1b)); SAMPT_TRY(get_f32(c, p + "mlp.fc2.bias", &f2b));
  const int M = B * H * H, Kp = pad64(C), Ch = 4 * C;
  SAMPT_TRY(tv_dw3x3(c, st, t.X, lw, lb, t.X2, nullptr, 0, B, H, H, C, 1, 0));
  std::swap(t.X, t.X2);
  SAMPT_TRY(tv_rows(c, st, t.X, C, nw, nb, 1e-5f, 1, nullptr, t.A, Kp, M, 0));
  // fc1 + GELU straight into fc2's hi|lo operand (held in the hidden buffer, free during the blocks)
  {
    const __half* w;
    const float* ws;
    SAMPT_TRY(get_f16(c, p + "mlp.fc1.w16", &w));
    SAMPT_TRY(get_f32(c, p + "mlp.fc1.w16s", &ws));
    __half* hb = reinterpret_cast<__half*>(t.F);
    GemmEpi ep{};
    ep.out16 = hb; ep.bias = f1b; ep.act = 1; ep.ldc = 2 * Ch; ep.split_off = Ch; ep.acc_scale = ws;
    SAMPT_TRY(gemm_tc(c, st, t.A, 2 * Kp, w, 2 * Kp, M, Ch, Kp, seg3(Kp), ep));
    SAMPT_TRY(tv_gemm(c, st, hb, p + "mlp.fc2.w16", M, C, Ch, f2b, 0, t.X, t.X));
  }
  return 0;
}

// layers.i with its downsample.  Input X at stage i's resolution and width; output X at the next one's.
int tv_stage(Ctx* c, cudaStream_t st, int i, int B, TvBufs& t) {
  const int H = TV_RES[i], C = TV_DIMS[i];
  const std::string p = TV_PREFIX + "layers." + std::to_string(i) + ".";
  if (i == 0) {
    SAMPT_TRY(tv_rows(c, st, t.X, C, nullptr, nullptr, 0.f, 0, nullptr, t.A, pad64(C), B * H * H, 0));
    for (int j = 0; j < TV_DEPTHS[0]; ++j) SAMPT_TRY(tv_mbconv(c, st, p + "blocks." + std::to_string(j) + ".", B, H, C, t));
  } else {
    for (int j = 0; j < TV_DEPTHS[i]; ++j)
      SAMPT_TRY(tv_block(c, st, p + "blocks." + std::to_string(j) + ".", B, H, C, TV_HEADS[i], TV_WIN[i], t));
    if (i + 1 < TV_NSTAGE) SAMPT_TRY(tv_rows(c, st, t.X, C, nullptr, nullptr, 0.f, 0, nullptr, t.A, pad64(C), B * H * H, 0));
  }
  if (i + 1 < TV_NSTAGE) SAMPT_TRY(tv_patch_merging(c, st, p + "downsample.", B, H, C, TV_DIMS[i + 1], t));
  return 0;
}

// neck over X (B*64*64, 320) -> feats (B, 256, 64, 64)
int tv_neck(Ctx* c, cudaStream_t st, int B, TvBufs& t, float* feats) {
  const int G = 64, M = B * G * G, Cin = TV_DIMS[TV_NSTAGE - 1];
  const float *g1, *b1, *g3, *b3;
  SAMPT_TRY(get_f32(c, TV_PREFIX + "neck.1.weight", &g1)); SAMPT_TRY(get_f32(c, TV_PREFIX + "neck.1.bias", &b1));
  SAMPT_TRY(get_f32(c, TV_PREFIX + "neck.3.weight", &g3)); SAMPT_TRY(get_f32(c, TV_PREFIX + "neck.3.bias", &b3));
  float* y1 = t.F;
  float* y2 = t.F + (size_t)M * TV_OUT;
  SAMPT_TRY(tv_rows(c, st, t.X, Cin, nullptr, nullptr, 0.f, 0, nullptr, t.A, pad64(Cin), M, 0));
  SAMPT_TRY(tv_gemm(c, st, t.A, TV_PREFIX + "neck.0.w16", M, TV_OUT, pad64(Cin), nullptr, 0, y1, nullptr));
  SAMPT_TRY(neck_ln_im2col(c, st, y1, g1, b1, t.A, B, G, TV_OUT, 2 * 9 * TV_OUT, 9 * TV_OUT));
  SAMPT_TRY(tv_gemm(c, st, t.A, TV_PREFIX + "neck.2.w16", M, TV_OUT, 9 * TV_OUT, nullptr, 0, y2, nullptr));
  return neck_ln_nchw(c, st, y2, g3, b3, feats, B, G * G, TV_OUT);
}

// stage i's input / output shapes (tokens per frame, channels)
void stage_io(int i, long long* in_tok, int* in_c, long long* out_tok, int* out_c) {
  *in_tok = (long long)TV_RES[i] * TV_RES[i];
  *in_c = TV_DIMS[i];
  if (i + 1 < TV_NSTAGE) {
    const int Ho = (TV_RES[i] - 1) / pm_stride(TV_DIMS[i + 1]) + 1;
    *out_tok = (long long)Ho * Ho;
    *out_c = TV_DIMS[i + 1];
  } else {
    *out_tok = *in_tok;
    *out_c = *in_c;
  }
}

}  // namespace
}  // namespace sampt

using namespace sampt;

extern "C" int sampt_tinyvit_workspace_bytes(int B, size_t* out) {
  SAMPT_CHECK(B >= 1, "sampt_tinyvit_workspace_bytes: B=%d", B);
  *out = tv_workspace_bytes(B);
  return 0;
}

extern "C" int sampt_tinyvit_encode(sampt_ctx* ctx, const void* image, int is_f32, int B, int Hr, int Wr, const float* mean3,
                                    const float* std3, float* feats, float* interm, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(B >= 1, "sampt_tinyvit_encode: B=%d", B);
  SAMPT_CHECK(is_f32 || (Hr >= 1 && Wr >= 1 && Hr <= TV_IMG && Wr <= TV_IMG), "sampt_tinyvit_encode: resized frame %dx%d exceeds %d",
              Hr, Wr, TV_IMG);
  SAMPT_CHECK(is_f32 || (mean3 != nullptr && std3 != nullptr), "sampt_tinyvit_encode: uint8 input needs mean and std");
  VitSlabGuard slab(c);
  TvBufs t;
  SAMPT_TRY(tv_alloc(c, B, &t));
  SAMPT_TRY(tv_stem(c, st, image, is_f32, B, Hr, Wr, mean3, std3, t));
  for (int i = 0; i < TV_NSTAGE; ++i) {
    SAMPT_TRY(tv_stage(c, st, i, B, t));
    if (i == 1 && interm)   // sam-hq: interm_embeddings[0] = layers.1's output (after its PatchMerging), (B, 64, 64, 160)
      SAMPT_CUDA(cudaMemcpyAsync(interm, t.X, (size_t)B * 64 * 64 * TV_DIMS[2] * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return tv_neck(c, st, B, t, feats);
}

// ---- unit-test entries: each runs the same launchers as sampt_tinyvit_encode out of the same workspace
extern "C" int sampt_test_tinyvit_stem(sampt_ctx* ctx, const void* image, int is_f32, int B, int Hr, int Wr, const float* mean3,
                                       const float* std3, float* out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  VitSlabGuard slab(c);
  TvBufs t;
  SAMPT_TRY(tv_alloc(c, B, &t));
  SAMPT_TRY(tv_stem(c, st, image, is_f32, B, Hr, Wr, mean3, std3, t));
  SAMPT_CUDA(cudaMemcpyAsync(out, t.X, (size_t)B * 256 * 256 * 64 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// depthwise conv with weights w [9][C] and bias [C]: out32 (B*Ho*Wo, C) and / or out16 (B*Ho*Wo, 2*Kp) hi|lo
extern "C" int sampt_test_tinyvit_dwconv(sampt_ctx* ctx, const float* x, const float* w, const float* bias, int B, int H, int W, int C,
                                         int stride, int act, float* out32, void* out16, int Kp, void* stream) {
  return tv_dw3x3(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), x, w, bias, out32,
                  reinterpret_cast<__half*>(out16), Kp, B, H, W, C, stride, act);
}

// the attention half of block `blk` of stage `stage` (1..3) on x (B, H, H, C) -> out = x + attn(...).  qkv_out (optional):
// the qkv GEMM's output, (B*H*H + 1, 3C) with the LN(0) row last when H is not a multiple of the window (else B*H*H rows);
// attn_out (optional): the proj GEMM's A operand (B*H*H, 2*pad64(C)) fp16 hi|lo
extern "C" int sampt_test_tinyvit_block_attn(sampt_ctx* ctx, int stage, int blk, const float* x, int B, int H, float* out,
                                             float* qkv_out, void* attn_out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(stage >= 1 && stage < TV_NSTAGE && blk >= 0 && blk < TV_DEPTHS[stage], "sampt_test_tinyvit_block_attn: stage %d block %d",
              stage, blk);
  const int C = TV_DIMS[stage];
  SAMPT_CHECK(H >= 1 && (long long)H * H * C <= (long long)TV_RES[stage] * TV_RES[stage] * C, "sampt_test_tinyvit_block_attn: H=%d", H);
  VitSlabGuard slab(c);
  TvBufs t;
  SAMPT_TRY(tv_alloc(c, B, &t));
  const size_t n = (size_t)B * H * H * C;
  SAMPT_CUDA(cudaMemcpyAsync(t.X, x, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  const std::string p = TV_PREFIX + "layers." + std::to_string(stage) + ".blocks." + std::to_string(blk) + ".";
  SAMPT_TRY(tv_block_attn(c, st, p, B, H, C, TV_HEADS[stage], TV_WIN[stage], t));
  SAMPT_CUDA(cudaMemcpyAsync(out, t.X, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  const size_t rows = (size_t)B * H * H + ((H % TV_WIN[stage]) != 0);
  if (qkv_out) SAMPT_CUDA(cudaMemcpyAsync(qkv_out, t.QKV, rows * 3 * C * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (attn_out)
    SAMPT_CUDA(cudaMemcpyAsync(attn_out, t.A, (size_t)B * H * H * 2 * pad64(C) * sizeof(__half), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// layers.<stage> with its downsample: x (B, R_i*R_i, C_i) -> out (B, R_o*R_o, C_o)
extern "C" int sampt_test_tinyvit_stage(sampt_ctx* ctx, int stage, const float* x, int B, float* out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(stage >= 0 && stage < TV_NSTAGE, "sampt_test_tinyvit_stage: stage %d", stage);
  long long in_tok, out_tok;
  int in_c, out_c;
  stage_io(stage, &in_tok, &in_c, &out_tok, &out_c);
  VitSlabGuard slab(c);
  TvBufs t;
  SAMPT_TRY(tv_alloc(c, B, &t));
  SAMPT_CUDA(cudaMemcpyAsync(t.X, x, (size_t)B * in_tok * in_c * sizeof(float), cudaMemcpyDeviceToDevice, st));
  SAMPT_TRY(tv_stage(c, st, stage, B, t));
  SAMPT_CUDA(cudaMemcpyAsync(out, t.X, (size_t)B * out_tok * out_c * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// neck: x (B, 64*64, 320) -> feats (B, 256, 64, 64)
extern "C" int sampt_test_tinyvit_neck(sampt_ctx* ctx, const float* x, int B, float* feats, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  VitSlabGuard slab(c);
  TvBufs t;
  SAMPT_TRY(tv_alloc(c, B, &t));
  SAMPT_CUDA(cudaMemcpyAsync(t.X, x, (size_t)B * 4096 * 320 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return tv_neck(c, st, B, t, feats);
}
