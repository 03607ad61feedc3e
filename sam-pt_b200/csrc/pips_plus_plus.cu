// PIPS++ (reference sam_pt/point_tracker/pips_plus_plus/pips_plus_plus.py, PipsPlusPlus(stride=8)) on one window and
// PipsPlusPlusPointTracker._forward (pips_plus_plus/tracker.py:25-65) over the windows of one direction.
//
//   fnet          the PIPS BasicEncoder (pips_pipeline.cu: fnet_frames), weights under "ppp.fnet.*", stride 8, once per frame
//   pyramid       sampt_pips_pyramid (avg_pool2d 2x2, 4 levels)
//   row           ppp_row_kernel: correlation targets feats1/2/4, 3 x 4 levels x 49 bilinear correlation samples straight from
//                 the channels-last pyramid (no dense volume), posemb_sincos_2d_xy(flow) and flow -> the 718-column DeltaBlock
//                 input, written as the temporal-im2col A operand (hi | lo) of first_block_conv
//   DeltaBlock    17 Conv1d(k=3, pad 1) + dense on gemm_tc with three fp16 passes (weights registered times 2^s, tinyvit.cu's
//                 tv_gemm); InstanceNorm1d over the S frames of a (point, channel) with a two-pass variance; ReLU, bias and
//                 the residual (zero-padded in the middle of the channels when they grow) in the im2col / epilogue
//   update        coords += delta on every frame, frame 0 re-locked
//
// Layouts: GEMM rows m = n*S + s (point-major, the reference's B*N, S); coords (S, N, 2) in feature-map pixels; the three
// correlation targets (3, S, N, 128) with a block stride, so that the next window's feat_init is a prefix of them.
// Window slot s reads frame fbase + fdir*s of the pyramid (fdir = -1: the time-reversed pass without a flipped copy).
#include <algorithm>
#include <string>

#include "common.cuh"
#include "kernels.cuh"
#include "tc_api.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {

namespace {

constexpr int PPP_C = 128;                 // latent_dim
constexpr int PPP_ROW = 3 * 196 + 130;     // 718: [corr 588 | posemb 128 | flow 2]
constexpr int PPP_KP0 = 2176;              // 3 * 718 = 2154 padded to a multiple of 64
constexpr int PPP_NBLK = 8;
constexpr int PPP_CIN[PPP_NBLK] = {128, 128, 128, 256, 256, 512, 512, 1024};
constexpr int PPP_COUT[PPP_NBLK] = {128, 128, 256, 256, 512, 512, 1024, 1024};
constexpr int PPP_DENSE_N = 32;            // dense 1024 -> 2, registered with 30 zero rows (gemm_tc needs N % 32 == 0)

struct PppWin {
  const float* pyr[4];
  int H[4], W[4];
  int N, S;
  int fbase, fdir;     // window slot s reads pyramid frame fbase + fdir * s
  float* coords;       // (S, N, 2) feature-map pixels
  float* feats;        // (3, S, N, 128): feats1, feats2, feats4
  size_t fstride;      // elements between the three blocks of `feats`
};

__device__ __forceinline__ float bilinear_c(const float* fm, int H, int W, float x, float y, int c) {
  // utils/samp.py bilinear_sample2d: indices clamped, weights from the unclamped coordinates
  const float x0f = floorf(x), y0f = floorf(y);
  const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
  const int x0c = min(max(x0, 0), W - 1), x1c = min(max(x1, 0), W - 1);
  const int y0c = min(max(y0, 0), H - 1), y1c = min(max(y1, 0), H - 1);
  const float x1f = (float)x1, y1f = (float)y1;
  const float w00 = (x1f - x) * (y1f - y), w01 = (x - x0f) * (y1f - y), w10 = (x1f - x) * (y - y0f), w11 = (x - x0f) * (y - y0f);
  return w00 * fm[((size_t)y0c * W + x0c) * PPP_C + c] + w01 * fm[((size_t)y0c * W + x1c) * PPP_C + c] +
         w10 * fm[((size_t)y1c * W + x0c) * PPP_C + c] + w11 * fm[((size_t)y1c * W + x1c) * PPP_C + c];
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// One CTA per (point n, slot s), 256 threads.
//   mode 0: the three targets are read from w.feats (feat_init, iteration 0)
//   mode 1: all three are bilinear_sample2d(frame of slot 0, coords[0, n]) (iteration 0 without feat_init, :468-472)
//   mode 2: feats1 is read; feats2 / feats4 are resampled from slot max(s-2, 0) / max(s-4, 0) at that slot's coords (:488-504)
// Sampled targets are written back to w.feats.  Then out[b*196 + l*49 + a*7 + c] = bilinear(corr_b,l)(x = cx + a-3,
// y = cy + c-3) with zero padding outside the map (CorrBlock.sample, :378-405: the window is TRANSPOSED, x takes the row
// offset), corr = target . fmap / sqrt(128); then posemb_sincos_2d_xy(flow, 128) (utils/misc.py:10-27) and flow, where
// flow[s] = coords[s+1] - coords[s] and the last frame repeats the one before (:520-521).
// The row goes to A rows (n, s+1-k), columns k*718 + col, k = 0..2 (temporal im2col, pad 1); this CTA also writes the zero
// tap of its own row at the window's ends and the zero columns [2154, 2176).  out32 (optional): the fp32 row, (M, 718).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ppp_row_kernel(PppWin w, int mode, const float* __restrict__ omega, __half* __restrict__ A, float* __restrict__ out32) {
  const int n = blockIdx.x / w.S, s = blockIdx.x % w.S;
  const int N = w.N, S = w.S;
  __shared__ __align__(16) float tg[3][PPP_C];
  __shared__ float D[3][4][64];
  __shared__ float row[PPP_ROW];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const size_t fm0 = (size_t)w.H[0] * w.W[0] * PPP_C;
  for (int i = t; i < 3 * PPP_C; i += 256) {
    const int b = i / PPP_C, c = i % PPP_C;
    float* dst = w.feats + b * w.fstride + ((size_t)s * N + n) * PPP_C + c;
    int src = -1;
    if (mode == 1) src = 0;
    else if (mode == 2 && b > 0) src = max(s - 2 * b, 0);
    float v;
    if (src < 0) {
      v = *dst;
    } else {
      const float* fm = w.pyr[0] + (size_t)(w.fbase + w.fdir * src) * fm0;
      v = bilinear_c(fm, w.H[0], w.W[0], w.coords[((size_t)src * N + n) * 2 + 0], w.coords[((size_t)src * N + n) * 2 + 1], c);
      *dst = v;
    }
    tg[b][c] = v;
  }
  __syncthreads();
  const float cx0 = w.coords[((size_t)s * N + n) * 2 + 0];
  const float cy0 = w.coords[((size_t)s * N + n) * 2 + 1];
  const int fi = w.fbase + w.fdir * s;
  // 3 targets x 4 levels x 64 pixels: warp `warp` takes pixels 8*warp .. 8*warp+7 of each (target, level) patch
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    const int H = w.H[l], W = w.W[l];
    const float sc = 1.0f / (float)(1 << l);
    const int bx = (int)floorf(cx0 * sc) - 3, by = (int)floorf(cy0 * sc) - 3;
    const float* fm = w.pyr[l] + (size_t)fi * H * W * PPP_C;
    float4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int pidx = warp * 8 + j, py = by + (pidx >> 3), px = bx + (pidx & 7);
      v[j] = (py >= 0 && py < H && px >= 0 && px < W)
                 ? __ldg(reinterpret_cast<const float4*>(fm + ((size_t)py * W + px) * PPP_C + lane * 4))
                 : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const float4 q = *reinterpret_cast<const float4*>(&tg[b][lane * 4]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = warp_sum(q.x * v[j].x + q.y * v[j].y + q.z * v[j].z + q.w * v[j].w);
        if (lane == 0) D[b][l][warp * 8 + j] = d / 11.3137083f;   // / sqrt(128) in fp32 (torch.sqrt(tensor(128.)))
      }
    }
  }
  __syncthreads();
  for (int i = t; i < 588; i += 256) {
    const int b = i / 196, r196 = i % 196, l = r196 / 49, r = r196 % 49, a = r / 7, c = r % 7;
    const float sc = 1.0f / (float)(1 << l);
    const float cx = cx0 * sc, cy = cy0 * sc;
    const int H = w.H[l], W = w.W[l];
    // grid_sample(align_corners=True) round trip x -> 2x/(W-1)-1 -> ((g+1)/2)(W-1), as bilinear_sampler computes it
    const float sx = cx + (float)(a - 3), sy = cy + (float)(c - 3);
    const float gx = 2.0f * sx / (float)(W - 1) - 1.0f, gy = 2.0f * sy / (float)(H - 1) - 1.0f;
    const float ux = ((gx + 1.0f) * 0.5f) * (float)(W - 1), uy = ((gy + 1.0f) * 0.5f) * (float)(H - 1);
    const float x0f = floorf(ux), y0f = floorf(uy);
    const float fx = ux - x0f, fy = uy - y0f;
    const int bx = (int)floorf(cx) - 3, by = (int)floorf(cy) - 3;
    const int ix = (int)x0f - bx, iy = (int)y0f - by;
    const float* Dl = D[b][l];
    auto at = [&](int yy, int xx) -> float { return (yy >= 0 && yy < 8 && xx >= 0 && xx < 8) ? Dl[yy * 8 + xx] : 0.f; };
    row[i] = (1.f - fx) * (1.f - fy) * at(iy, ix) + fx * (1.f - fy) * at(iy, ix + 1) + (1.f - fx) * fy * at(iy + 1, ix) +
             fx * fy * at(iy + 1, ix + 1);
  }
  {
    const int s0 = min(s, S - 2);
    const float fx = w.coords[((size_t)(s0 + 1) * N + n) * 2 + 0] - w.coords[((size_t)s0 * N + n) * 2 + 0];
    const float fy = w.coords[((size_t)(s0 + 1) * N + n) * 2 + 1] - w.coords[((size_t)s0 * N + n) * 2 + 1];
    if (t < 128) {
      const int k = t & 31, part = t >> 5;
      const float arg = __fmul_rn(part < 2 ? fx : fy, omega[k]);
      row[588 + t] = (part & 1) ? cosf(arg) : sinf(arg);
    }
    if (t == 128) row[716] = fx;
    if (t == 129) row[717] = fy;
  }
  __syncthreads();
  const size_t m = (size_t)n * S + s;
  if (out32) for (int i = t; i < PPP_ROW; i += 256) out32[m * PPP_ROW + i] = row[i];
  for (int i = t; i < 3 * PPP_ROW; i += 256) {
    const int k = i / PPP_ROW, col = i % PPP_ROW;
    const int sd = s + 1 - k;              // A row fed by this frame through tap k
    if (sd >= 0 && sd < S) {
      const float v = row[col];
      const __half h = __float2half_rn(v);
      __half* o = A + ((size_t)n * S + sd) * (2 * PPP_KP0);
      o[k * PPP_ROW + col] = h;
      o[PPP_KP0 + k * PPP_ROW + col] = __float2half_rn(v - __half2float(h));
    }
  }
  __half* o = A + m * (2 * PPP_KP0);
  const __half z = __float2half_rn(0.f);
  if (s == 0) for (int i = t; i < PPP_ROW; i += 256) { o[i] = z; o[PPP_KP0 + i] = z; }
  if (s == S - 1) for (int i = t; i < PPP_ROW; i += 256) { o[2 * PPP_ROW + i] = z; o[PPP_KP0 + 2 * PPP_ROW + i] = z; }
  for (int i = 3 * PPP_ROW + t; i < PPP_KP0; i += 256) { o[i] = z; o[PPP_KP0 + i] = z; }
}

// ---------------------------------------------------------------------------------------------------------------------
// Temporal im2col of a (M = N*S, C) fp32 activation into the A operand of gemm_tc (2*Kp halves per row, hi | lo):
// column k*C + c of row (n, s) = f(x[n, s+k-1, c]) for taps = 3 (zero outside the point's own S frames, Conv1dPad's "same"
// padding), or f(x[n, s, c]) for taps = 1; columns [taps*C, Kp) are zero.  f = ReLU((x - mean) * rstd) with stats (N, C, 2),
// or ReLU(x), or x.  writeback (ReLU without stats only): x <- f(x) in place, which is race-free because ReLU is idempotent.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void ppp_im2col_kernel(float* x, const float* __restrict__ stats, int relu, int writeback, __half* __restrict__ A, int N, int S,
                                  int C, int taps, int Kp, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k = (int)(i % Kp);
  const long long m = i / Kp;
  const int n = (int)(m / S), s = (int)(m % S);
  float v = 0.f;
  if (k < taps * C) {
    const int tap = k / C, c = k % C;
    const int ss = taps == 3 ? s + tap - 1 : s;
    if (ss >= 0 && ss < S) {
      const size_t src = ((size_t)n * S + ss) * C + c;
      v = x[src];
      if (stats) v = (v - stats[((size_t)n * C + c) * 2]) * stats[((size_t)n * C + c) * 2 + 1];
      if (relu) v = fmaxf(v, 0.f);
      if (writeback && ss == s) x[src] = v;
    }
  }
  const __half h = __float2half_rn(v);
  A[m * 2 * Kp + k] = h;
  A[m * 2 * Kp + Kp + k] = __float2half_rn(v - __half2float(h));
}

// InstanceNorm1d statistics (eps 1e-5, biased, no affine) over the S frames of each (point, channel): two passes (mean, then
// the sum of squared deviations from it).  One thread per (n, c); consecutive threads take consecutive channels.
__global__ void ppp_inorm_stats_kernel(const float* __restrict__ x, float* __restrict__ stats, int N, int S, int C) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  const int n = i / C, c = i % C;
  const float* p = x + (size_t)n * S * C + c;
  float sum = 0.f;
  for (int s = 0; s < S; ++s) sum += p[(size_t)s * C];
  const float mean = sum / (float)S;
  float sq = 0.f;
  for (int s = 0; s < S; ++s) { const float d = p[(size_t)s * C] - mean; sq = fmaf(d, d, sq); }
  stats[(size_t)i * 2] = mean;
  stats[(size_t)i * 2 + 1] = 1.0f / sqrtf(sq / (float)S + 1e-5f);
}

// identity of a ResidualBlock1d whose channels grow: y[m, ch1 + c] = x[m, c], zero elsewhere, ch1 = (Cout - Cin) / 2 (:97-102)
__global__ void ppp_pad_identity_kernel(const float* __restrict__ x, float* __restrict__ y, int Cin, int Cout, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % Cout);
  const long long m = i / Cout;
  const int ch1 = (Cout - Cin) / 2;
  y[i] = (c >= ch1 && c < ch1 + Cin) ? x[m * Cin + c - ch1] : 0.f;
}

// coords += delta (:529), then frame 0 re-locked to `lock` (:533).  pre (optional): the pre-lock coords * stride, (S, N, 2)
// (coord_predictions1 entry of this iteration, :531).  delta rows m = n*S + s with leading dimension ldd.
__global__ void ppp_update_kernel(float* __restrict__ coords, const float* __restrict__ lock, const float* __restrict__ delta, int ldd,
                                  float* __restrict__ pre, int N, int S, float stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * S) return;
  const int s = i / N, n = i % N;
  const float* d = delta + ((size_t)n * S + s) * ldd;
  float x = coords[(size_t)i * 2 + 0] + d[0], y = coords[(size_t)i * 2 + 1] + d[1];
  if (pre) { pre[(size_t)i * 2 + 0] = x * stride; pre[(size_t)i * 2 + 1] = y * stride; }
  if (s == 0) { x = lock[n * 2 + 0]; y = lock[n * 2 + 1]; }
  coords[(size_t)i * 2 + 0] = x;
  coords[(size_t)i * 2 + 1] = y;
}

// px (S, N, 2) -> coords = px / stride (:458) and lock = coords[0]
__global__ void ppp_coords_in_kernel(const float* __restrict__ px, float* __restrict__ coords, float* __restrict__ lock, int N, int S,
                                     float stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * S) return;
  const float x = px[(size_t)i * 2 + 0] / stride, y = px[(size_t)i * 2 + 1] / stride;
  coords[(size_t)i * 2 + 0] = x;
  coords[(size_t)i * 2 + 1] = y;
  if (i < N) { lock[i * 2 + 0] = x; lock[i * 2 + 1] = y; }
}

__global__ void ppp_scale_kernel(const float* __restrict__ in, float* __restrict__ out, float f, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = in[i] * f;
}

// trajs (T, N, 2): every frame <- q (N, 2) (zero-velocity init, tracker.py:34); or, with from >= 0, frames [from, T) <- frame
// from - 1 (the future filled with the last prediction, :57)
__global__ void ppp_fill_kernel(float* __restrict__ traj, const float* __restrict__ q, int from, int N, int T) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * T * 2) return;
  const int t = i / (2 * N), r = i % (2 * N);
  if (from < 0) traj[i] = q[r];
  else if (t >= from) traj[i] = traj[(size_t)(from - 1) * 2 * N + r];
}

// PipsPlusPlusPointTracker.forward's image_size resize (tracker.py:72-77): F.interpolate(rgbs / 255, size, mode="bilinear") * 255,
// ATen upsample_bilinear2d with align_corners=False, over uint8 or float32 planar frames -> float32 planar frames
template <typename TIn>
__global__ void ppp_resize_kernel(const TIn* __restrict__ in, float* __restrict__ out, int H, int W, int Ho, int Wo, float sy, float sx,
                                  long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho);
  const long long plane = i / ((long long)Wo * Ho);
  const float fy = fmaxf(sy * ((float)oy + 0.5f) - 0.5f, 0.f), fx = fmaxf(sx * ((float)ox + 0.5f) - 0.5f, 0.f);
  const int y0 = min((int)fy, H - 1), x0 = min((int)fx, W - 1);
  const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  const float ly1 = fy - (float)y0, lx1 = fx - (float)x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
  const TIn* p = in + plane * H * W;
  auto v = [&](int y, int x) { return (float)p[(size_t)y * W + x] / 255.0f; };
  out[i] = (ly0 * (lx0 * v(y0, x0) + lx1 * v(y0, x1)) + ly1 * (lx0 * v(y1, x0) + lx1 * v(y1, x1))) * 255.0f;
}

namespace {

struct PppBufs {
  float *coords, *lock, *X, *Y, *Z, *stats, *D;
  __half* A;
};

int pad64i(int k) { return (k + 63) / 64 * 64; }

int launch_im2col(Ctx* c, cudaStream_t st, float* x, const float* stats, int relu, int writeback, __half* A, int N, int S, int C,
                  int taps, int Kp) {
  const long long total = (long long)N * S * Kp;
  ppp_im2col_kernel<<<cdiv(total, 256), 256, 0, st>>>(x, stats, relu, writeback, A, N, S, C, taps, Kp, total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

int launch_inorm_stats(Ctx* c, cudaStream_t st, const float* x, float* stats, int N, int S, int C) {
  ppp_inorm_stats_kernel<<<cdiv((long long)N * C, 128), 128, 0, st>>>(x, stats, N, S, C);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

std::string blk(int i, const char* conv) { return "ppp.delta_block.basicblock_list." + std::to_string(i) + "." + conv + ".conv"; }

// ResidualBlock1d i (:77-105) on x (M, Cin) -> out (M, Cout); y is scratch (M, Cout).  Block 0 skips the first IN + ReLU; its
// im2col applies DeltaBlock's first_block_relu instead and writes the ReLU'd input back to x, which is the block's identity.
int ppp_res_block(Ctx* c, cudaStream_t st, int i, float* x, float* y, float* out, PppBufs& b, int N, int S) {
  const int Cin = PPP_CIN[i], Cout = PPP_COUT[i], M = N * S;
  const float *b1, *b2;
  SAMPT_TRY(get_f32(c, blk(i, "conv1") + ".bias", &b1));
  SAMPT_TRY(get_f32(c, blk(i, "conv2") + ".bias", &b2));
  if (i == 0) {
    SAMPT_TRY(launch_im2col(c, st, x, nullptr, 1, 1, b.A, N, S, Cin, 3, 3 * Cin));
  } else {
    SAMPT_TRY(launch_inorm_stats(c, st, x, b.stats, N, S, Cin));
    SAMPT_TRY(launch_im2col(c, st, x, b.stats, 1, 0, b.A, N, S, Cin, 3, 3 * Cin));
  }
  SAMPT_TRY(tv_gemm(c, st, b.A, blk(i, "conv1") + ".w16", M, Cout, 3 * Cin, b1, 0, y, nullptr));
  SAMPT_TRY(launch_inorm_stats(c, st, y, b.stats, N, S, Cout));
  SAMPT_TRY(launch_im2col(c, st, y, b.stats, 1, 0, b.A, N, S, Cout, 3, 3 * Cout));
  const float* resid = x;
  if (Cout != Cin) {
    const long long total = (long long)M * Cout;
    ppp_pad_identity_kernel<<<cdiv(total, 256), 256, 0, st>>>(x, out, Cin, Cout, total);
    c->launches++;
    SAMPT_LAUNCH_CHECK();
    resid = out;   // the epilogue reads the residual before it writes the same element
  }
  return tv_gemm(c, st, b.A, blk(i, "conv2") + ".w16", M, Cout, 3 * Cout, b2, 0, out, resid);
}

// DeltaBlock after the input row (:327-336): b.A holds first_block_conv's operand -> b.D (M, 32), delta in columns 0, 1
int ppp_delta_block(Ctx* c, cudaStream_t st, PppBufs& b, int N, int S) {
  const int M = N * S;
  const float *b0, *bd;
  SAMPT_TRY(get_f32(c, "ppp.delta_block.first_block_conv.conv.bias", &b0));
  SAMPT_TRY(get_f32(c, "ppp.delta_block.dense.bias", &bd));
  // first_block_norm is never applied (:328-329); first_block_relu happens in block 0's im2col
  SAMPT_TRY(tv_gemm(c, st, b.A, "ppp.delta_block.first_block_conv.conv.w16", M, 128, PPP_KP0, b0, 0, b.X, nullptr));
  float *x = b.X, *o = b.Z;
  for (int i = 0; i < PPP_NBLK; ++i) {
    SAMPT_TRY(ppp_res_block(c, st, i, x, b.Y, o, b, N, S));
    std::swap(x, o);
  }
  // final_relu (final_norm is never applied, :333), dense 1024 -> 2 (registered as 32 rows)
  SAMPT_TRY(launch_im2col(c, st, x, nullptr, 1, 0, b.A, N, S, 1024, 1, 1024));
  return tv_gemm(c, st, b.A, "ppp.delta_block.dense.w16", M, PPP_DENSE_N, 1024, bd, 0, b.D, nullptr);
}

int ppp_alloc(Ctx* c, PppBufs* b, int N, int S) {
  const size_t M = (size_t)N * S;
  SAMPT_TRY(ws_get(c, &b->coords, (size_t)S * N * 2, "ppp coords"));
  SAMPT_TRY(ws_get(c, &b->lock, (size_t)N * 2, "ppp lock"));
  SAMPT_TRY(ws_get(c, &b->X, M * 1024, "ppp X"));
  SAMPT_TRY(ws_get(c, &b->Y, M * 1024, "ppp Y"));
  SAMPT_TRY(ws_get(c, &b->Z, M * 1024, "ppp Z"));
  SAMPT_TRY(ws_get(c, &b->stats, (size_t)N * 1024 * 2, "ppp stats"));
  SAMPT_TRY(ws_get(c, &b->D, M * PPP_DENSE_N, "ppp delta"));
  SAMPT_TRY(ws_get(c, &b->A, M * 2 * 3072, "ppp A operand"));
  return 0;
}

int launch_row(Ctx* c, cudaStream_t st, const PppWin& w, int mode, __half* A, float* out32) {
  const float* omega;
  SAMPT_TRY(get_f32(c, "ppp.omega", &omega));
  ppp_row_kernel<<<w.N * w.S, 256, 0, st>>>(w, mode, omega, A, out32);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// PipsPlusPlus.forward on one window (:436-546).  trajs_e0 (S, N, 2) px; w.feats holds feat_init when have_init.
// coords_out (optional): (iters + 1, S, N, 2) = coord_predictions1 (pre-lock per iteration, then the final locked coords);
// final_px (optional): the final locked coords * stride, (S, N, 2) (may alias trajs_e0).
int ppp_window(Ctx* c, cudaStream_t st, PppWin& w, PppBufs& b, const float* trajs_e0, int have_init, int iters, float stride,
               float* coords_out, float* final_px) {
  const int N = w.N, S = w.S, M = N * S;
  w.coords = b.coords;
  ppp_coords_in_kernel<<<cdiv(M, 256), 256, 0, st>>>(trajs_e0, b.coords, b.lock, N, S, stride);
  c->launches++;
  for (int it = 0; it < iters; ++it) {
    SAMPT_TRY(launch_row(c, st, w, it == 0 ? (have_init ? 0 : 1) : 2, b.A, nullptr));
    SAMPT_TRY(ppp_delta_block(c, st, b, N, S));
    ppp_update_kernel<<<cdiv(M, 256), 256, 0, st>>>(b.coords, b.lock, b.D, PPP_DENSE_N,
                                                    coords_out ? coords_out + (size_t)it * M * 2 : nullptr, N, S, stride);
    c->launches++;
  }
  if (iters == 0) {
    // the targets are still returned (:545): computed as at iteration 0
    SAMPT_TRY(launch_row(c, st, w, have_init ? 0 : 1, b.A, nullptr));
  }
  if (coords_out) {
    ppp_scale_kernel<<<cdiv(M * 2, 256), 256, 0, st>>>(b.coords, coords_out + (size_t)iters * M * 2, stride, M * 2);
    c->launches++;
  }
  if (final_px) {
    ppp_scale_kernel<<<cdiv(M * 2, 256), 256, 0, st>>>(b.coords, final_px, stride, M * 2);
    c->launches++;
  }
  SAMPT_LAUNCH_CHECK();
  return 0;
}

void set_pyr(PppWin* w, const float* l0, const float* l1, const float* l2, const float* l3, int H8, int W8) {
  w->pyr[0] = l0; w->pyr[1] = l1; w->pyr[2] = l2; w->pyr[3] = l3;
  w->H[0] = H8; w->W[0] = W8;
  for (int l = 1; l < 4; ++l) { w->H[l] = w->H[l - 1] / 2; w->W[l] = w->W[l - 1] / 2; }
}

int check_geometry(int H8, int W8, int S, const char* who) {
  SAMPT_CHECK((H8 >> 3) >= 2 && (W8 >> 3) >= 2,
              "%s: the coarsest correlation level of a %dx%d feature map has fewer than 2 rows or columns (frames below 128 px "
              "give NaN trajectories in the reference)", who, H8, W8);
  SAMPT_CHECK(S >= 2, "%s: a window needs at least 2 frames, got %d", who, S);
  return 0;
}

}  // namespace
}  // namespace sampt

using namespace sampt;

extern "C" int sampt_pips_plus_plus_window(sampt_ctx* ctx, const float* l0, const float* l1, const float* l2, const float* l3, int H8,
                                           int W8, const float* trajs_e0, const float* feat_init, int N, int S, int stride, int iters,
                                           float* coords_out, float* feats_out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_TRY(check_geometry(H8, W8, S, "sampt_pips_plus_plus_window"));
  SAMPT_CHECK(N >= 1 && iters >= 0 && stride > 0, "sampt_pips_plus_plus_window: N >= 1, iters >= 0 and stride > 0 required");
  c->ws_reset();
  PppBufs b;
  SAMPT_TRY(ppp_alloc(c, &b, N, S));
  PppWin w{};
  set_pyr(&w, l0, l1, l2, l3, H8, W8);
  w.N = N; w.S = S; w.fbase = 0; w.fdir = 1;
  w.feats = feats_out; w.fstride = (size_t)S * N * PPP_C;
  if (feat_init) SAMPT_CUDA(cudaMemcpyAsync(feats_out, feat_init, 3 * w.fstride * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return ppp_window(c, st, w, b, trajs_e0, feat_init != nullptr, iters, (float)stride, coords_out, nullptr);
}

extern "C" int sampt_pips_plus_plus_track(sampt_ctx* ctx, const float* l0, const float* l1, const float* l2, const float* l3, int H8,
                                          int W8, int t0, int dir, int Tdir, const float* query, int N, int max_len, int stride,
                                          int iters, float* traj, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(dir == 1 || dir == -1, "sampt_pips_plus_plus_track: dir must be 1 or -1, got %d", dir);
  SAMPT_CHECK(max_len >= 2 && N >= 1 && iters >= 0 && stride > 0, "sampt_pips_plus_plus_track: bad arguments");
  SAMPT_CHECK(t0 >= 0 && t0 + dir * (Tdir - 1) >= 0, "sampt_pips_plus_plus_track: frames out of range");
  SAMPT_TRY(check_geometry(H8, W8, std::min(Tdir, max_len), "sampt_pips_plus_plus_track"));
  c->ws_reset();
  const int Smax = std::min(Tdir, max_len);
  PppBufs b;
  SAMPT_TRY(ppp_alloc(c, &b, N, Smax));
  float* feats;
  const size_t fstride = (size_t)Smax * N * PPP_C;
  SAMPT_TRY(ws_get(c, &feats, 3 * fstride, "ppp feats"));
  ppp_fill_kernel<<<cdiv((long long)N * Tdir * 2, 256), 256, 0, st>>>(traj, query, -1, N, Tdir);
  c->launches++;
  int cur = 0;
  bool have_init = false;
  for (;;) {
    int end = cur + max_len;
    if (end > Tdir) {
      const int diff = end - Tdir;
      end -= diff;
      cur = std::max(cur - diff, 0);
    }
    PppWin w{};
    set_pyr(&w, l0, l1, l2, l3, H8, W8);
    w.N = N; w.S = end - cur; w.fbase = t0 + dir * cur; w.fdir = dir;
    w.feats = feats; w.fstride = fstride;   // feat_init of the next window = the first S_local slots (:52)
    float* seq = traj + (size_t)cur * N * 2;
    SAMPT_TRY(ppp_window(c, st, w, b, seq, have_init, iters, (float)stride, nullptr, seq));
    have_init = true;
    if (end < Tdir) {
      ppp_fill_kernel<<<cdiv((long long)N * Tdir * 2, 256), 256, 0, st>>>(traj, nullptr, end, N, Tdir);
      c->launches++;
    }
    if (end >= Tdir) break;
    cur = cur + max_len - 1;
  }
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// image_size resize of PipsPlusPlusPointTracker.forward: planes of (H, W), uint8 (is_f32 = 0) or float32 -> float32 (Ho, Wo)
extern "C" int sampt_pips_plus_plus_resize(sampt_ctx* ctx, const void* in, int is_f32, int planes, int H, int W, int Ho, int Wo, float* out,
                                           void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(planes > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, "sampt_pips_plus_plus_resize: empty input");
  const long long total = (long long)planes * Ho * Wo;
  const float sy = (float)H / (float)Ho, sx = (float)W / (float)Wo;
  if (is_f32) ppp_resize_kernel<float><<<cdiv(total, 256), 256, 0, st>>>(static_cast<const float*>(in), out, H, W, Ho, Wo, sy, sx, total);
  else ppp_resize_kernel<uint8_t><<<cdiv(total, 256), 256, 0, st>>>(static_cast<const uint8_t*>(in), out, H, W, Ho, Wo, sy, sx, total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// ---- unit-test entries: one stage on caller buffers, through the launchers the window runs ---------------------------------
extern "C" int sampt_test_pips_plus_plus_row(sampt_ctx* ctx, const float* l0, const float* l1, const float* l2, const float* l3, int H8,
                                             int W8, const float* coords, float* feats, int N, int S, int mode, float* row,
                                             void* A, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_TRY(check_geometry(H8, W8, S, "sampt_test_pips_plus_plus_row"));
  SAMPT_CHECK(mode >= 0 && mode <= 2 && N >= 1, "sampt_test_pips_plus_plus_row: mode must be 0, 1 or 2");
  PppWin w{};
  set_pyr(&w, l0, l1, l2, l3, H8, W8);
  w.N = N; w.S = S; w.fbase = 0; w.fdir = 1;
  w.coords = const_cast<float*>(coords);
  w.feats = feats; w.fstride = (size_t)S * N * PPP_C;
  return launch_row(c, reinterpret_cast<cudaStream_t>(stream), w, mode, reinterpret_cast<__half*>(A), row);
}

// Conv1dPad(k=3) of DeltaBlock by weight name ("first_block_conv" or "basicblock_list.<i>.conv<1|2>") on x (N*S, Cin) fp32, with
// f = identity (pre 0), ReLU (pre 1) or ReLU(InstanceNorm1d) (pre 2) applied to the input first -> out (N*S, Cout) fp32
extern "C" int sampt_test_pips_plus_plus_tconv(sampt_ctx* ctx, const char* name, const float* x, int N, int S, int Cin, int Cout,
                                               int pre, float* out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(pre >= 0 && pre <= 2 && N >= 1 && S >= 1, "sampt_test_pips_plus_plus_tconv: bad arguments");
  c->ws_reset();
  PppBufs b;
  SAMPT_TRY(ppp_alloc(c, &b, N, S));
  const std::string p = std::string("ppp.delta_block.") + name + ".conv";
  const TensorRef* wt = c->find(p + ".w16");
  SAMPT_CHECK(wt != nullptr && wt->ndim == 2 && wt->dims[0] == Cout && wt->dims[1] == 2 * pad64i(3 * Cin),
              "sampt_test_pips_plus_plus_tconv: %s is not a registered %d -> %d conv", p.c_str(), Cin, Cout);
  const float* bias;
  SAMPT_TRY(get_f32(c, p + ".bias", &bias));
  SAMPT_CUDA(cudaMemcpyAsync(b.X, x, (size_t)N * S * Cin * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (pre == 2) SAMPT_TRY(launch_inorm_stats(c, st, b.X, b.stats, N, S, Cin));
  const int Kp = pad64i(3 * Cin);
  SAMPT_TRY(launch_im2col(c, st, b.X, pre == 2 ? b.stats : nullptr, pre != 0, 0, b.A, N, S, Cin, 3, Kp));
  return tv_gemm(c, st, b.A, p + ".w16", N * S, Cout, Kp, bias, 0, out, nullptr);
}

// InstanceNorm1d statistics over time: x (N*S, C) -> stats (N, C, 2) = (mean, rstd)
extern "C" int sampt_test_pips_plus_plus_inorm(sampt_ctx* ctx, const float* x, int N, int S, int C, float* stats, void* stream) {
  SAMPT_CHECK(N >= 1 && S >= 1 && C >= 1, "sampt_test_pips_plus_plus_inorm: empty input");
  return launch_inorm_stats(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), x, stats, N, S, C);
}

// block >= 0: ResidualBlock1d `block` on x (N*S, Cin) -> out (N*S, Cout).  block == -1: the whole DeltaBlock from the fp32 input
// rows x (N*S, 718) -> out (N*S, 2) delta.  Block 0's input is expected already ReLU'd, as DeltaBlock feeds it.
extern "C" int sampt_test_pips_plus_plus_residual(sampt_ctx* ctx, int block, const float* x, int N, int S, float* out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(block >= -1 && block < PPP_NBLK && N >= 1 && S >= 1, "sampt_test_pips_plus_plus_residual: bad arguments");
  c->ws_reset();
  PppBufs b;
  SAMPT_TRY(ppp_alloc(c, &b, N, S));
  const int M = N * S;
  if (block >= 0) {
    SAMPT_CUDA(cudaMemcpyAsync(b.X, x, (size_t)M * PPP_CIN[block] * sizeof(float), cudaMemcpyDeviceToDevice, st));
    SAMPT_TRY(ppp_res_block(c, st, block, b.X, b.Y, b.Z, b, N, S));
    SAMPT_CUDA(cudaMemcpyAsync(out, b.Z, (size_t)M * PPP_COUT[block] * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  SAMPT_CUDA(cudaMemcpyAsync(b.Y, x, (size_t)M * PPP_ROW * sizeof(float), cudaMemcpyDeviceToDevice, st));
  SAMPT_TRY(launch_im2col(c, st, b.Y, nullptr, 0, 0, b.A, N, S, PPP_ROW, 3, PPP_KP0));
  SAMPT_TRY(ppp_delta_block(c, st, b, N, S));
  SAMPT_CUDA(cudaMemcpy2DAsync(out, 2 * sizeof(float), b.D, PPP_DENSE_N * sizeof(float), 2 * sizeof(float), M, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// coords (S, N, 2) feature-map px, updated in place with delta (N*S, 2) and frame 0 set to lock (N, 2); pre (S, N, 2) optional
extern "C" int sampt_test_pips_plus_plus_update(sampt_ctx* ctx, float* coords, const float* lock, const float* delta, int N, int S,
                                                int stride, float* pre, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_CHECK(N >= 1 && S >= 1, "sampt_test_pips_plus_plus_update: empty input");
  ppp_update_kernel<<<cdiv(N * S, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(coords, lock, delta, 2, pre, N, S,
                                                                                          (float)stride);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}
