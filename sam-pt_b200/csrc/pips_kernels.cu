// PIPS hot-path kernels (strict fp32).  Reference: /root/reference/sam_pt/point_tracker/pips/pips.py.
//
// HBM layout chosen for the correlation gather: feature maps are channels-last (T, H/4, W/4, 128) fp32 so that one
// pixel's 128 channels are one 512 B contiguous line -> a warp reads a pixel with one coalesced float4 load per lane.
// The encoder keeps channels-last throughout so no transposes are needed.
#include "common.cuh"
#include "kernels.cuh"

namespace sampt {

// =====================================================================================================
// fnet: BasicEncoder (pips.py:191-287)
// =====================================================================================================

// conv1: 7x7 stride 2 pad 3, 3 -> 64, input = uint8 planar frames normalised on the fly 2*(x/255)-1 (pips.py:446).
// weights [kh][kw][ci][co] (co contiguous).  One thread = one output pixel x 16 output channels.
template <typename TIn>
__global__ void __launch_bounds__(256)
conv7x7s2_kernel(const TIn* __restrict__ frames, const float* __restrict__ w, const float* __restrict__ bias,
                    float* __restrict__ out, int H, int W, int Ho, int Wo) {
  __shared__ float ws[7 * 7 * 3 * 64];
  for (int i = threadIdx.x; i < 7 * 7 * 3 * 64; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const int img = blockIdx.y;
  const int cg = threadIdx.x & 3;  // 4 channel groups of 16
  const long long pix = (long long)blockIdx.x * 64 + (threadIdx.x >> 2);
  if (pix >= (long long)Ho * Wo) return;
  const int oy = (int)(pix / Wo), ox = (int)(pix % Wo);
  const TIn* f = frames + (size_t)img * 3 * H * W;
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = bias[cg * 16 + j];
  for (int r = 0; r < 7; ++r) {
    int iy = oy * 2 + r - 3;
    if (iy < 0 || iy >= H) continue;
    for (int s = 0; s < 7; ++s) {
      int ix = ox * 2 + s - 3;
      if (ix < 0 || ix >= W) continue;
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        float v = 2.0f * ((float)f[(size_t)ci * H * W + (size_t)iy * W + ix] / 255.0f) - 1.0f;
        const float* wp = ws + ((r * 7 + s) * 3 + ci) * 64 + cg * 16;
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[j] = fmaf(v, wp[j], acc[j]);
      }
    }
  }
  float* o = out + ((size_t)img * Ho * Wo + pix) * 64 + cg * 16;
#pragma unroll
  for (int j = 0; j < 16; j += 4) *reinterpret_cast<float4*>(o + j) = make_float4(acc[j], acc[j + 1], acc[j + 2], acc[j + 3]);
}

int conv7x7s2(Ctx* c, cudaStream_t st, const void* frames, int is_f32, const float* w, const float* bias, float* out, int Nimg,
              int H, int W) {
  const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
  dim3 g(cdiv((long long)Ho * Wo, 64), Nimg);
  if (is_f32) conv7x7s2_kernel<float><<<g, 256, 0, st>>>((const float*)frames, w, bias, out, H, W, Ho, Wo);
  else conv7x7s2_kernel<uint8_t><<<g, 256, 0, st>>>((const uint8_t*)frames, w, bias, out, H, W, Ho, Wo);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// Generic implicit-GEMM convolution, channels-last, fp32:  out[n,oy,ox,co] = bias[co] + sum_{r,s,ci} in[n,iy,ix,ci] * w[r,s,ci,co]
// GEMM view: M = N*Ho*Wo pixels, Ncol = Cout, K = R*S*Cin.  BK=16 channels of one (r,s) tap per k-tile (Cin % 16 == 0).
template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (BN / TN))
conv_nhwc_f32_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                     float* __restrict__ out, int Nimg, int H, int W, int Cin, int Ho, int Wo, int Cout, int R, int S,
                     int stride, int pad, const int* skip) {
  if (skip != nullptr && *skip != 0) return;
  constexpr int BK = 16;
  constexpr int NT = (BM / TM) * (BN / TN);
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];
  const int tid = threadIdx.x;
  const long long Mtot = (long long)Nimg * Ho * Wo;
  const long long m0 = (long long)blockIdx.y * BM;
  const int n0 = blockIdx.x * BN;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  constexpr int A_F4 = BM * BK / 4, B_F4 = BN * BK / 4;
  constexpr int A_PER = (A_F4 + NT - 1) / NT, B_PER = (B_F4 + NT - 1) / NT;
  float4 ra[A_PER], rb[B_PER];
  // per-thread pixel decomposition of its A rows (fixed over the k loop)
  int a_img[A_PER], a_oy[A_PER], a_ox[A_PER];
  bool a_ok[A_PER];
#pragma unroll
  for (int i = 0; i < A_PER; ++i) {
    int idx = tid + i * NT;
    int r = idx / (BK / 4);
    long long gm = m0 + r;
    a_ok[i] = (idx < A_F4) && (gm < Mtot);
    long long g = a_ok[i] ? gm : 0;
    a_img[i] = (int)(g / ((long long)Ho * Wo));
    int rem = (int)(g % ((long long)Ho * Wo));
    a_oy[i] = rem / Wo;
    a_ox[i] = rem % Wo;
  }
  const int cin_tiles = Cin / BK;
  const int nk = R * S * cin_tiles;

  auto gload = [&](int kt) {
    int tap = kt / cin_tiles, c0 = (kt % cin_tiles) * BK;
    int r = tap / S, s = tap % S;
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int idx = tid + i * NT;
      int c = (idx % (BK / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (a_ok[i]) {
        int iy = a_oy[i] * stride + r - pad, ix = a_ox[i] * stride + s - pad;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W)
          v = *reinterpret_cast<const float4*>(in + (((size_t)a_img[i] * H + iy) * W + ix) * Cin + c0 + c);
      }
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int idx = tid + i * NT;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < B_F4) {
        int kk = idx / (BN / 4), cn = (idx % (BN / 4)) * 4;
        int gn = n0 + cn;
        if (gn < Cout) v = *reinterpret_cast<const float4*>(w + ((size_t)tap * Cin + c0 + kk) * Cout + gn);
      }
      rb[i] = v;
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int idx = tid + i * NT;
      if (idx < A_F4) {
        int r = idx / (BK / 4), c = (idx % (BK / 4)) * 4;
        As[buf][c + 0][r] = ra[i].x; As[buf][c + 1][r] = ra[i].y; As[buf][c + 2][r] = ra[i].z; As[buf][c + 3][r] = ra[i].w;
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int idx = tid + i * NT;
      if (idx < B_F4) {
        int kk = idx / (BN / 4), cn = (idx % (BN / 4)) * 4;
        *reinterpret_cast<float4*>(&Bs[buf][kk][cn]) = rb[i];
      }
    }
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload(kt + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        float4 v = *reinterpret_cast<const float4*>(&As[buf][k][ty * TM + i]);
        a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        float4 v = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * TN + j]);
        b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    long long gm = m0 + ty * TM + i;
    if (gm >= Mtot) continue;
#pragma unroll
    for (int j = 0; j < TN; j += 4) {
      int gn = n0 + tx * TN + j;
      if (gn >= Cout) continue;
      float4 v = make_float4(acc[i][j], acc[i][j + 1], acc[i][j + 2], acc[i][j + 3]);
      if (bias) { v.x += bias[gn]; v.y += bias[gn + 1]; v.z += bias[gn + 2]; v.w += bias[gn + 3]; }
      *reinterpret_cast<float4*>(out + (size_t)gm * Cout + gn) = v;
    }
  }
}

int conv_nhwc_f32(Ctx* c, cudaStream_t st, const float* in, const float* w, const float* bias, float* out, int Nimg,
                  int H, int W, int Cin, int Cout, int R, int S, int stride, int pad, const int* skip) {
  SAMPT_CHECK(Cin % 16 == 0 && Cout % 4 == 0, "conv_nhwc_f32: Cin %% 16 and Cout %% 4 required (Cin=%d Cout=%d)", Cin, Cout);
  int Ho = (H + 2 * pad - R) / stride + 1, Wo = (W + 2 * pad - S) / stride + 1;
  long long M = (long long)Nimg * Ho * Wo;
  if (Cout % 64 == 0 || Cout >= 96) {
    dim3 grid(cdiv(Cout, 64), cdiv(M, 128));
    conv_nhwc_f32_kernel<128, 64, 8, 4><<<grid, 256, 0, st>>>(in, w, bias, out, Nimg, H, W, Cin, Ho, Wo, Cout, R, S, stride, pad, skip);
  } else {
    dim3 grid(cdiv(Cout, 32), cdiv(M, 128));
    conv_nhwc_f32_kernel<128, 32, 8, 4><<<grid, 128, 0, st>>>(in, w, bias, out, Nimg, H, W, Cin, Ho, Wo, Cout, R, S, stride, pad, skip);
  }
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Tensor-core path of the encoder's convolutions: explicit im2col into the fp16 hi|lo operand layout of gemm_tc (3-pass
// split precision ~ fp32), the GEMM then writes fp32 NHWC + bias.  Row m = output pixel, column k = (r*S + s)*Cin + ci,
// K padded to a multiple of 64 with zeros; `lo` half at column offset Kp.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void im2col_nhwc_split_kernel(const float* __restrict__ in, __half* __restrict__ A, int Nimg, int H, int W, int Cin,
                                         int Ho, int Wo, int R, int S, int stride, int pad, int Kp, long long total) {
  // one thread = 8 consecutive k (16 B of hi + 16 B of lo)
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int kg = (int)(i % (Kp / 8));
  const long long m = i / (Kp / 8);
  const int k0 = kg * 8;
  const int ox = (int)(m % Wo), oy = (int)((m / Wo) % Ho), img = (int)(m / ((long long)Wo * Ho));
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = 0.f;
  const int K = R * S * Cin;
  if (k0 < K) {
    const int tap = k0 / Cin, c0 = k0 % Cin;  // Cin % 8 == 0 -> the 8 k's share one tap
    const int iy = oy * stride + tap / S - pad, ix = ox * stride + tap % S - pad;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
      const float* src = in + (((size_t)img * H + iy) * W + ix) * Cin + c0;
      const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
  }
  __half hi[8], lo[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    hi[j] = __float2half_rn(v[j]);
    lo[j] = __float2half_rn(v[j] - __half2float(hi[j]));
  }
  __half* row = A + (size_t)m * (2 * Kp);
  *reinterpret_cast<uint4*>(row + k0) = *reinterpret_cast<uint4*>(hi);
  *reinterpret_cast<uint4*>(row + Kp + k0) = *reinterpret_cast<uint4*>(lo);
}
int im2col_nhwc_split(Ctx* c, cudaStream_t st, const float* in, __half* A, int Nimg, int H, int W, int Cin, int R, int S, int stride,
                      int pad, int Kp) {
  SAMPT_CHECK(Cin % 8 == 0 && Kp % 64 == 0 && Kp >= R * S * Cin, "im2col_nhwc_split: Cin %% 8, Kp %% 64 required");
  const int Ho = (H + 2 * pad - R) / stride + 1, Wo = (W + 2 * pad - S) / stride + 1;
  const long long total = (long long)Nimg * Ho * Wo * (Kp / 8);
  im2col_nhwc_split_kernel<<<cdiv(total, 256), 256, 0, st>>>(in, A, Nimg, H, W, Cin, Ho, Wo, R, S, stride, pad, Kp, total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}
// first layer: 7x7 stride 2 pad 3 on uint8 planar frames, normalisation 2*(x/255)-1 fused; k = (r*7 + s)*3 + ci, Kp = 192
template <typename TIn>
__global__ void im2col_conv1_split_kernel(const TIn* __restrict__ frames, __half* __restrict__ A, int H, int W, int Ho,
                                             int Wo, int Kp, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int kg = (int)(i % (Kp / 8));
  const long long m = i / (Kp / 8);
  const int ox = (int)(m % Wo), oy = (int)((m / Wo) % Ho), img = (int)(m / ((long long)Wo * Ho));
  const TIn* f = frames + (size_t)img * 3 * H * W;
  __half hi[8], lo[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = kg * 8 + j;
    float v = 0.f;
    if (k < 147) {
      const int tap = k / 3, ci = k % 3;
      const int iy = oy * 2 + tap / 7 - 3, ix = ox * 2 + tap % 7 - 3;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = 2.0f * ((float)f[(size_t)ci * H * W + (size_t)iy * W + ix] / 255.0f) - 1.0f;
    }
    hi[j] = __float2half_rn(v);
    lo[j] = __float2half_rn(v - __half2float(hi[j]));
  }
  __half* row = A + (size_t)m * (2 * Kp);
  *reinterpret_cast<uint4*>(row + kg * 8) = *reinterpret_cast<uint4*>(hi);
  *reinterpret_cast<uint4*>(row + Kp + kg * 8) = *reinterpret_cast<uint4*>(lo);
}
// frames: uint8 (is_f32 == 0) or float32 holding 0..255 values (is_f32 == 1, the CoTracker wrapper's resized clip)
int im2col_conv1_split(Ctx* c, cudaStream_t st, const void* frames, int is_f32, __half* A, int Nimg, int H, int W, int Kp) {
  const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
  const long long total = (long long)Nimg * Ho * Wo * (Kp / 8);
  if (is_f32)
    im2col_conv1_split_kernel<float><<<cdiv(total, 256), 256, 0, st>>>((const float*)frames, A, H, W, Ho, Wo, Kp, total);
  else
    im2col_conv1_split_kernel<uint8_t><<<cdiv(total, 256), 256, 0, st>>>((const uint8_t*)frames, A, H, W, Ho, Wo, Kp, total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// InstanceNorm2d (no affine, eps 1e-5, biased variance; pips.py:207-209), channels-last.
// pass 1 sums d = x - xc and d^2 per (image, row-chunk) and channel, xc = the channel's pixel at the centre of the image (index
// HW/2).  The shift keeps E[d^2] - E[d]^2 well conditioned when the mean is large against the spread (a nearly constant channel with
// an O(1) conv bias, as black or letterboxed frames produce): from sums of x and x^2 the fp32 rounding would cost a relative
// variance error ~ u (mean/std)^2.  Where xc is far from the mean on the scale of the spread (mean - xc)^2 > 8 (var + eps),
// pass 2 sums d = x - mean instead and replaces that channel's statistics.
// shift = null: pass 1; else pass 2, shift[(img*C + c)*2] = the mean of pass 1.
// 256 threads = (C/4 float4 channel lanes) x (256/(C/4) pixel rows): 16-byte coalesced loads, `rows` pixels in flight per lane
// group, fp32 partial sums over <= 64 pixels promoted to fp64 before the cross-row / cross-chunk reduction.
__global__ void __launch_bounds__(256)
inorm_partial_kernel(const float* __restrict__ x, const float* __restrict__ shift, double* __restrict__ part, int HW, int C, int chunk) {
  const int img = blockIdx.z, ch = blockIdx.y;
  const int c4n = C >> 2, rows = 256 / c4n;
  const int lane4 = threadIdx.x % c4n, row = threadIdx.x / c4n;
  const int p0 = ch * chunk, p1 = min(HW, p0 + chunk);
  __shared__ double red[256][8];
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f), ss = make_float4(0.f, 0.f, 0.f, 0.f);
  double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (row < rows) {
    const float* base = x + (size_t)img * HW * C + lane4 * 4;
    float4 x0;
    if (shift) {
      const float* sp = shift + ((size_t)img * C + lane4 * 4) * 2;
      x0 = make_float4(sp[0], sp[2], sp[4], sp[6]);
    } else {
      x0 = *reinterpret_cast<const float4*>(base + (size_t)(HW / 2) * C);
    }
    int cnt = 0;
#pragma unroll 4
    for (int p = p0 + row; p < p1; p += rows) {
      float4 v = *reinterpret_cast<const float4*>(base + (size_t)p * C);
      v.x -= x0.x; v.y -= x0.y; v.z -= x0.z; v.w -= x0.w;
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      ss.x = fmaf(v.x, v.x, ss.x); ss.y = fmaf(v.y, v.y, ss.y); ss.z = fmaf(v.z, v.z, ss.z); ss.w = fmaf(v.w, v.w, ss.w);
      if (++cnt == 64) {
        acc[0] += s.x; acc[1] += ss.x; acc[2] += s.y; acc[3] += ss.y; acc[4] += s.z; acc[5] += ss.z; acc[6] += s.w; acc[7] += ss.w;
        s = make_float4(0.f, 0.f, 0.f, 0.f); ss = make_float4(0.f, 0.f, 0.f, 0.f); cnt = 0;
      }
    }
    acc[0] += s.x; acc[1] += ss.x; acc[2] += s.y; acc[3] += ss.y; acc[4] += s.z; acc[5] += ss.z; acc[6] += s.w; acc[7] += ss.w;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[threadIdx.x][k] = acc[k];
  __syncthreads();
  if (row == 0) {
    for (int r = 1; r < rows; ++r)
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += red[r * c4n + lane4][k];
    double* o = part + (((size_t)img * gridDim.y + ch) * C + lane4 * 4) * 2;
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = acc[k];  // [c][sum, sumsq] for the 4 channels of this lane
  }
}
// stats[(img*C + c)*2 + {0,1}] = (mean, rstd); shift as in inorm_partial_kernel (it may alias stats: each thread reads its own
// channel's shift before writing it)
__global__ void inorm_final_kernel(const float* __restrict__ x, const float* shift, const double* __restrict__ part, float* stats,
                                   int nchunks, int C, int HW, float eps) {
  const int img = blockIdx.y;
  const int cidx = blockIdx.x * blockDim.x + threadIdx.x;
  if (cidx >= C) return;
  double s = 0.0, ss = 0.0;
  for (int ch = 0; ch < nchunks; ++ch) {
    size_t o = (((size_t)img * nchunks + ch) * C + cidx) * 2;
    s += part[o];
    ss += part[o + 1];
  }
  const double dmean = s / HW;   // mean of d
  double var = ss / HW - dmean * dmean;
  if (var < 0) var = 0;
  const double xc = (double)x[((size_t)img * HW + HW / 2) * C + cidx];
  const double x0 = shift ? (double)shift[((size_t)img * C + cidx) * 2] : xc;
  // pass 2 keeps pass 1's statistics where they are as accurate (relative variance error gamma_64 (1 + (mean - xc)^2 / var))
  if (shift && (x0 - xc) * (x0 - xc) <= 8.0 * (var + (double)eps)) return;
  stats[((size_t)img * C + cidx) * 2] = (float)(x0 + dmean);
  stats[((size_t)img * C + cidx) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
}
// pass 2: y = relu?( (x-mean)*rstd [+ res] ).  res_stats != null -> residual is itself instance-normed first
// (the `downsample` branch of ResidualBlock, pips.py:176-178,185-188); post_relu applies relu AFTER the residual add.
__global__ void inorm_apply_kernel(const float* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ res,
                                   const float* __restrict__ res_stats, float* __restrict__ y, long long total4, int HW,
                                   int C, int relu_before_add, int relu_after) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  long long e = i * 4;
  int cidx = (int)(e % C);
  int img = (int)(e / ((long long)HW * C));
  float4 v = *reinterpret_cast<const float4*>(x + e);
  const float* sp = stats + ((size_t)img * C + cidx) * 2;
  float o[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    o[j] = (o[j] - sp[2 * j]) * sp[2 * j + 1];
    if (relu_before_add) o[j] = fmaxf(o[j], 0.f);
  }
  if (res) {
    float4 r = *reinterpret_cast<const float4*>(res + e);
    float rr[4] = {r.x, r.y, r.z, r.w};
    if (res_stats) {
      const float* rp = res_stats + ((size_t)img * C + cidx) * 2;
#pragma unroll
      for (int j = 0; j < 4; ++j) rr[j] = (rr[j] - rp[2 * j]) * rp[2 * j + 1];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] += rr[j];
  }
  if (relu_after) {
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = fmaxf(o[j], 0.f);
  }
  *reinterpret_cast<float4*>(y + e) = make_float4(o[0], o[1], o[2], o[3]);
}

int inorm_stats(Ctx* c, cudaStream_t st, const float* x, float* stats, double* part, int Nimg, int HW, int C) {
  const int chunk = 512;
  int nchunks = cdiv(HW, chunk);
  SAMPT_CHECK(C % 4 == 0 && C <= 1024, "inorm_stats: unsupported channel count %d", C);
  dim3 g1(1, nchunks, Nimg);
  dim3 g2(cdiv(C, 64), Nimg);
  inorm_partial_kernel<<<g1, 256, 0, st>>>(x, nullptr, part, HW, C, chunk);   // shifted by the centre pixel
  SAMPT_LAUNCH_CHECK();
  inorm_final_kernel<<<g2, 64, 0, st>>>(x, nullptr, part, stats, nchunks, C, HW, 1e-5f);
  SAMPT_LAUNCH_CHECK();
  inorm_partial_kernel<<<g1, 256, 0, st>>>(x, stats, part, HW, C, chunk);     // centred on pass 1's mean
  SAMPT_LAUNCH_CHECK();
  inorm_final_kernel<<<g2, 64, 0, st>>>(x, stats, part, stats, nchunks, C, HW, 1e-5f);
  SAMPT_LAUNCH_CHECK();
  c->launches += 4;
  return 0;
}
int inorm_apply(Ctx* c, cudaStream_t st, const float* x, const float* stats, const float* res, const float* res_stats,
                float* y, int Nimg, int HW, int C, int relu_before_add, int relu_after) {
  long long total4 = (long long)Nimg * HW * C / 4;
  inorm_apply_kernel<<<cdiv(total4, 256), 256, 0, st>>>(x, stats, res, res_stats, y, total4, HW, C, relu_before_add, relu_after);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// F.interpolate(mode=bilinear, align_corners=True) into a channel slice of the concat buffer (pips.py:275-279).
__global__ void resize_ac_concat_kernel(const float* __restrict__ in, float* __restrict__ out, int Hi, int Wi, int C,
                                        int Ho, int Wo, int Ctot, int coff, long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int c4 = (int)(i % (C / 4));
  long long p = i / (C / 4);
  int ox = (int)(p % Wo);
  int oy = (int)((p / Wo) % Ho);
  int img = (int)(p / ((long long)Wo * Ho));
  // ATen area_pixel_compute_source_index(align_corners=True): scale = (in-1)/(out-1), src = scale*dst
  float sy = (Ho > 1) ? (float)(Hi - 1) / (float)(Ho - 1) : 0.f;
  float sx = (Wo > 1) ? (float)(Wi - 1) / (float)(Wo - 1) : 0.f;
  float fy = sy * oy, fx = sx * ox;
  int y0 = (int)fy, x0 = (int)fx;
  int y1 = y0 + ((y0 < Hi - 1) ? 1 : 0), x1 = x0 + ((x0 < Wi - 1) ? 1 : 0);
  float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
  const float* b = in + (size_t)img * Hi * Wi * C + c4 * 4;
  float4 v00 = *reinterpret_cast<const float4*>(b + ((size_t)y0 * Wi + x0) * C);
  float4 v01 = *reinterpret_cast<const float4*>(b + ((size_t)y0 * Wi + x1) * C);
  float4 v10 = *reinterpret_cast<const float4*>(b + ((size_t)y1 * Wi + x0) * C);
  float4 v11 = *reinterpret_cast<const float4*>(b + ((size_t)y1 * Wi + x1) * C);
  float4 r;
  r.x = hy * (hx * v00.x + lx * v01.x) + ly * (hx * v10.x + lx * v11.x);
  r.y = hy * (hx * v00.y + lx * v01.y) + ly * (hx * v10.y + lx * v11.y);
  r.z = hy * (hx * v00.z + lx * v01.z) + ly * (hx * v10.z + lx * v11.z);
  r.w = hy * (hx * v00.w + lx * v01.w) + ly * (hx * v10.w + lx * v11.w);
  *reinterpret_cast<float4*>(out + (((size_t)img * Ho + oy) * Wo + ox) * Ctot + coff + c4 * 4) = r;
}
int resize_ac_concat(Ctx* c, cudaStream_t st, const float* in, float* out, int Nimg, int Hi, int Wi, int C, int Ho, int Wo,
                     int Ctot, int coff) {
  long long total = (long long)Nimg * Ho * Wo * (C / 4);
  resize_ac_concat_kernel<<<cdiv(total, 256), 256, 0, st>>>(in, out, Hi, Wi, C, Ho, Wo, Ctot, coff, total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// correlation pyramid (pips.py:355-361): avg_pool2d(2, stride 2) (floor), channels-last
// =====================================================================================================
__global__ void avgpool2_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int Hi, int Wi, int Ho, int Wo,
                                     int C, long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int c4 = (int)(i % (C / 4));
  long long p = i / (C / 4);
  int ox = (int)(p % Wo);
  int oy = (int)((p / Wo) % Ho);
  int img = (int)(p / ((long long)Wo * Ho));
  const float* b = in + (((size_t)img * Hi + 2 * oy) * Wi + 2 * ox) * C + c4 * 4;
  float4 a = *reinterpret_cast<const float4*>(b);
  float4 bb = *reinterpret_cast<const float4*>(b + C);
  float4 cc = *reinterpret_cast<const float4*>(b + (size_t)Wi * C);
  float4 d = *reinterpret_cast<const float4*>(b + (size_t)Wi * C + C);
  float4 r;
  r.x = (a.x + bb.x + cc.x + d.x) * 0.25f;
  r.y = (a.y + bb.y + cc.y + d.y) * 0.25f;
  r.z = (a.z + bb.z + cc.z + d.z) * 0.25f;
  r.w = (a.w + bb.w + cc.w + d.w) * 0.25f;
  *reinterpret_cast<float4*>(out + (((size_t)img * Ho + oy) * Wo + ox) * C + c4 * 4) = r;
}
int avgpool2_nhwc(Ctx* c, cudaStream_t st, const float* in, float* out, int Nimg, int Hi, int Wi, int C) {
  int Ho = Hi / 2, Wo = Wi / 2;
  long long total = (long long)Nimg * Ho * Wo * (C / 4);
  avgpool2_nhwc_kernel<<<cdiv(total, 256), 256, 0, st>>>(in, out, Hi, Wi, Ho, Wo, C, total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// per-window state init: coords = xys/stride for all S (pips.py:460-463), ffeats = feat_init or
// bilinear_sample2d(fmaps[:,0]) (utils/samp.py:6-66: clamp indices, UNCLAMPED weights)
// =====================================================================================================
__global__ void pips_window_init_kernel(PipsWin w) {
  const int n = blockIdx.x, c = threadIdx.x;  // 128 threads
  if (!w.active[n]) return;
  const int frame = w.wp[0];
  const float x = w.traj[((size_t)frame * w.N + n) * 2 + 0] / (float)w.stride;
  const float y = w.traj[((size_t)frame * w.N + n) * 2 + 1] / (float)w.stride;
  if (c < w.S) {
    w.coords[((size_t)n * w.S + c) * 2 + 0] = x;
    w.coords[((size_t)n * w.S + c) * 2 + 1] = y;
  }
  float f;
  if (w.sample_feat) {
    const int H = w.H[0], W = w.W[0];
    const float* fm = w.pyr[0] + (size_t)w.wp[2] * H * W * 128;
    float x0f = floorf(x), y0f = floorf(y);
    int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
    int x0c = min(max(x0, 0), W - 1), x1c = min(max(x1, 0), W - 1);
    int y0c = min(max(y0, 0), H - 1), y1c = min(max(y1, 0), H - 1);
    float x1f = (float)x1, y1f = (float)y1;
    float w00 = (x1f - x) * (y1f - y), w01 = (x - x0f) * (y1f - y), w10 = (x1f - x) * (y - y0f), w11 = (x - x0f) * (y - y0f);
    f = w00 * fm[((size_t)y0c * W + x0c) * 128 + c] + w01 * fm[((size_t)y0c * W + x1c) * 128 + c] +
        w10 * fm[((size_t)y1c * W + x0c) * 128 + c] + w11 * fm[((size_t)y1c * W + x1c) * 128 + c];
    w.feat_init[(size_t)n * 128 + c] = f;
  } else {
    f = w.feat_init[(size_t)n * 128 + c];
  }
  for (int s = 0; s < w.S; ++s) w.ffeats[((size_t)n * w.S + s) * 128 + c] = f;
}

// =====================================================================================================
// fused correlation lookup + mixer-input assembly (pips.py:364-407 + :521-531 + utils/misc.py:30-55)
//
// One CTA per (point n, window slot s).  The dense (B,S,N,H,W) correlation volume of the reference is never
// built: bilinear-sampling a correlation map == correlating with the 4 neighbouring feature vectors and
// blending (SURVEY §0.7-v).  Per level an 8x8 pixel patch x 128 ch is gathered (one warp = one pixel = one
// coalesced 512 B line, float4 per lane), dotted with ffeats[n,s] held in registers, warp-shuffle reduced into
// shared memory, then the 7x7 window is produced in the reference's TRANSPOSED order (pips.py:378-384):
//     out[l*49 + a*7 + b] = bilinear(corr_l)(x = cx + a-3, y = cy + b-3), zero outside the map.
// Algorithmic bytes: S*L*64*128*4 B = 1 MiB per point per iteration (SURVEY §8d).
// The same CTA then writes the mixer row  [ffeat 128 | corr 196 | sincos(dx,dy,t) 192 | (dx,dy,t) 3 | pad 1].
// =====================================================================================================
__global__ void __launch_bounds__(256)
pips_corr_kernel(PipsWin w, float* __restrict__ xin, int ldx) {
  const int n = blockIdx.x / w.S, s = blockIdx.x % w.S;
  if (!w.active[n]) return;
  __shared__ float D[4][64];
  __shared__ float sflow[3];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* ff = w.ffeats + ((size_t)n * w.S + s) * 128;
  const float4 q = *reinterpret_cast<const float4*>(ff + lane * 4);
  const float cx0 = w.coords[((size_t)n * w.S + s) * 2 + 0];
  const float cy0 = w.coords[((size_t)n * w.S + s) * 2 + 1];
  const int fi = w.wp[2 + s];
  // 4 levels x 64 pixels = 256 dots, 8 warps -> 32 dots per warp; all loads issued before the reductions (ILP)
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    const int H = w.H[l], W = w.W[l];
    const float sc = 1.0f / (float)(1 << l);
    const float cx = cx0 * sc, cy = cy0 * sc;
    const int bx = (int)floorf(cx) - 3, by = (int)floorf(cy) - 3;
    const float* fm = w.pyr[l] + (size_t)fi * H * W * 128;
    float part[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int pidx = warp * 8 + j;  // 0..63 -> (row = y index, col = x index)
      int py = by + (pidx >> 3), px = bx + (pidx & 7);
      float d = 0.f;
      if (py >= 0 && py < H && px >= 0 && px < W) {
        float4 v = __ldg(reinterpret_cast<const float4*>(fm + ((size_t)py * W + px) * 128 + lane * 4));
        d = q.x * v.x + q.y * v.y + q.z * v.z + q.w * v.w;
      }
      part[j] = d;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float d = warp_sum(part[j]);
      if (lane == 0) D[l][warp * 8 + j] = d * 0.08838834764831845f;  // 1/sqrt(128)  (pips.py:406)
    }
  }
  if (threadIdx.x == 0) {
    sflow[0] = cx0 - w.coords[((size_t)n * w.S + 0) * 2 + 0];
    sflow[1] = cy0 - w.coords[((size_t)n * w.S + 0) * 2 + 1];
    // times_ = linspace(0, S, S)  (pips.py:527) with torch's two-sided rule: step = S/(S-1); slots below S/2 are s * step, the
    // others S - step * (S-1-s), each product and difference rounded on its own (no fma contraction)
    if (w.S <= 1) sflow[2] = 0.f;
    else {
      const float step = (float)w.S / (float)(w.S - 1);
      sflow[2] = (s < w.S / 2) ? __fmul_rn((float)s, step) : __fsub_rn((float)w.S, __fmul_rn(step, (float)(w.S - 1 - s)));
    }
  }
  __syncthreads();
  float* row = xin + ((size_t)n * w.S + s) * ldx;
  const int t = threadIdx.x;
  if (t < 128) row[t] = ff[t];
  if (t < 196) {
    int l = t / 49, r = t % 49, a = r / 7, b = r % 7;
    const float sc = 1.0f / (float)(1 << l);
    const float cx = cx0 * sc, cy = cy0 * sc;
    // grid_sample(align_corners=True) round trip: x -> 2x/(W-1)-1 -> ((g+1)/2)*(W-1); reproduce it so the bilinear
    // weights see the same float rounding as the reference (pips.py:325-329)
    const int H = w.H[l], W = w.W[l];
    float sx = cx + (float)(a - 3), sy = cy + (float)(b - 3);
    float gx = 2.0f * sx / (float)(W - 1) - 1.0f, gy = 2.0f * sy / (float)(H - 1) - 1.0f;
    float ux = ((gx + 1.0f) * 0.5f) * (float)(W - 1), uy = ((gy + 1.0f) * 0.5f) * (float)(H - 1);
    float x0f = floorf(ux), y0f = floorf(uy);
    float fx = ux - x0f, fy = uy - y0f;
    const int bx = (int)floorf(cx) - 3, by = (int)floorf(cy) - 3;
    int ix = (int)x0f - bx, iy = (int)y0f - by;  // index into the 8x8 patch
    auto at = [&](int yy, int xx) -> float { return (yy >= 0 && yy < 8 && xx >= 0 && xx < 8) ? D[l][yy * 8 + xx] : 0.f; };
    float v = (1.f - fx) * (1.f - fy) * at(iy, ix) + fx * (1.f - fy) * at(iy, ix + 1) + (1.f - fx) * fy * at(iy + 1, ix) +
              fx * fy * at(iy + 1, ix + 1);
    row[128 + t] = v;
  }
  if (t < 96) {
    // get_3d_embedding(C=64): div_term = arange(0,64,2)*(1000/64); pe[0::2]=sin, pe[1::2]=cos; blocks x,y,z
    int d = t / 32, k = t % 32;
    float div = (float)(2 * k) * (1000.0f / 64.0f);
    float arg = sflow[d] * div;
    row[324 + d * 64 + 2 * k] = sinf(arg);
    row[324 + d * 64 + 2 * k + 1] = cosf(arg);
  }
  if (t < 3) row[516 + t] = sflow[t];
  if (t == 3) row[519] = 0.f;
}


int pips_window_init(Ctx* c, cudaStream_t st, const PipsWin& w) {
  pips_window_init_kernel<<<w.N, 128, 0, st>>>(w);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}
int pips_corr(Ctx* c, cudaStream_t st, const PipsWin& w, float* xin, int ldx) {
  pips_corr_kernel<<<w.N * w.S, 256, 0, st>>>(w, xin, ldx);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// MLP-Mixer pieces (pips.py:96-128)
// =====================================================================================================
// token mixing + the following pre-norm, one CTA per point (S rows x 512):
//   x += Conv1d(4S->S)(GELU(Conv1d(S->4S)(LN(x))))   over the S axis;   xln = LN_next(x)
// S = 8 fixed (pips.yaml s: 8).  256 threads, 2 channels each.
__global__ void __launch_bounds__(256)
mixer_token_kernel(float* __restrict__ x, float* __restrict__ xln, const uint8_t* __restrict__ active,
                   const float* __restrict__ ln_w, const float* __restrict__ ln_b, const float* __restrict__ w1,
                   const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                   const float* __restrict__ ln2_w, const float* __restrict__ ln2_b, int do_token_mix) {
  constexpr int S = 8, D = 512, HID = 32;
  const int n = blockIdx.x;
  if (active && !active[n]) return;
  __shared__ float sw1[HID * S], sb1[HID], sw2[S * HID], sb2[S];
  __shared__ float red[32];
  __shared__ float mean[S], rstd[S];
  const int t = threadIdx.x;
  if (do_token_mix) {
    for (int i = t; i < HID * S; i += 256) { sw1[i] = w1[i]; sw2[i] = w2[i]; }
    if (t < HID) sb1[t] = b1[t];
    if (t < S) sb2[t] = b2[t];
  }
  float* xp = x + (size_t)n * S * D;
  float v[S][2];
#pragma unroll
  for (int s = 0; s < S; ++s) { v[s][0] = xp[s * D + t]; v[s][1] = xp[s * D + 256 + t]; }

  auto row_stats = [&]() {
#pragma unroll
    for (int s = 0; s < S; ++s) {
      float m = block_sum(v[s][0] + v[s][1], red) * (1.0f / D);
      float d0 = v[s][0] - m, d1 = v[s][1] - m;
      float var = block_sum(d0 * d0 + d1 * d1, red) * (1.0f / D);
      if (t == 0) { mean[s] = m; rstd[s] = (1.0f / sqrtf(var + 1e-5f)); }
    }
    __syncthreads();
  };

  if (do_token_mix) {
    row_stats();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ch = t + h * 256;
      float xn[S];
      const float g = ln_w[ch], bta = ln_b[ch];
#pragma unroll
      for (int s = 0; s < S; ++s) xn[s] = (v[s][h] - mean[s]) * rstd[s] * g + bta;
      float out[S];
#pragma unroll
      for (int s = 0; s < S; ++s) out[s] = sb2[s];
#pragma unroll 4
      for (int j = 0; j < HID; ++j) {
        float hsum = sb1[j];
#pragma unroll
        for (int s = 0; s < S; ++s) hsum = fmaf(sw1[j * S + s], xn[s], hsum);
        hsum = gelu_erf(hsum);
#pragma unroll
        for (int s = 0; s < S; ++s) out[s] = fmaf(sw2[s * HID + j], hsum, out[s]);
      }
#pragma unroll
      for (int s = 0; s < S; ++s) v[s][h] += out[s];
    }
#pragma unroll
    for (int s = 0; s < S; ++s) { xp[s * D + t] = v[s][0]; xp[s * D + 256 + t] = v[s][1]; }
    __syncthreads();
  }
  // following pre-norm (channel-mix LN, or the final LN when do_token_mix == 0)
  row_stats();
  float* op = xln + (size_t)n * S * D;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int ch = t + h * 256;
    const float g = ln2_w[ch], bta = ln2_b[ch];
#pragma unroll
    for (int s = 0; s < S; ++s) op[s * D + ch] = (v[s][h] - mean[s]) * rstd[s] * g + bta;
  }
}
int mixer_token(Ctx* c, cudaStream_t st, float* x, float* xln, const uint8_t* active, int N, const float* ln_w,
                const float* ln_b, const float* w1, const float* b1, const float* w2, const float* b2, const float* ln2_w,
                const float* ln2_b, int do_token_mix) {
  mixer_token_kernel<<<N, 256, 0, st>>>(x, xln, active, ln_w, ln_b, w1, b1, w2, b2, ln2_w, ln2_b, do_token_mix);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// mean over S of the final-LN output (Reduce 'b n c -> b c', pips.py:126): xm[n, c] = mean_s xln[n, s, c]
__global__ void mixer_mean_kernel(const float* __restrict__ xln, float* __restrict__ xm, int S, int D) {
  const int n = blockIdx.x;
  for (int ch = threadIdx.x; ch < D; ch += blockDim.x) {
    float a = 0.f;
    for (int s = 0; s < S; ++s) a += xln[((size_t)n * S + s) * D + ch];
    xm[(size_t)n * D + ch] = a / (float)S;
  }
}
int mixer_mean(Ctx* c, cudaStream_t st, const float* xln, float* xm, int N, int S, int D) {
  mixer_mean_kernel<<<N, 256, 0, st>>>(xln, xm, S, D);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// feature / coordinate update (pips.py:533-546): one CTA per (n, s), 128 threads
//   ffeats += GELU(Linear128(GroupNorm(1,128)(dfeat)));  coords += dxy;  coords[s=0] locked
// =====================================================================================================
__global__ void __launch_bounds__(128)
pips_update_kernel(PipsWin w, const float* __restrict__ delta, const float* __restrict__ gn_w,
                   const float* __restrict__ gn_b, const float* __restrict__ up_w, const float* __restrict__ up_b) {
  const int n = blockIdx.x / w.S, s = blockIdx.x % w.S;
  if (!w.active[n]) return;
  __shared__ float g[128];
  __shared__ float red[32];
  const int t = threadIdx.x;
  const float* d = delta + ((size_t)n * w.S + s) * 130;
  float v = d[2 + t];
  float m = block_sum(v, red) * (1.0f / 128.0f);
  float dv = v - m;
  float var = block_sum(dv * dv, red) * (1.0f / 128.0f);
  g[t] = dv * (1.0f / sqrtf(var + 1e-5f)) * gn_w[t] + gn_b[t];
  __syncthreads();
  float acc = up_b[t];
  const float* wr = up_w + (size_t)t * 128;
#pragma unroll 8
  for (int k = 0; k < 128; k += 4) {
    float4 ww = *reinterpret_cast<const float4*>(wr + k);
    acc = fmaf(ww.x, g[k], acc);
    acc = fmaf(ww.y, g[k + 1], acc);
    acc = fmaf(ww.z, g[k + 2], acc);
    acc = fmaf(ww.w, g[k + 3], acc);
  }
  w.ffeats[((size_t)n * w.S + s) * 128 + t] += gelu_erf(acc);
  if (t < 2 && s > 0) w.coords[((size_t)n * w.S + s) * 2 + t] += d[t];
}
int pips_update(Ctx* c, cudaStream_t st, const PipsWin& w, const float* delta, const float* gn_w, const float* gn_b,
                const float* up_w, const float* up_b) {
  pips_update_kernel<<<w.N * w.S, 128, 0, st>>>(w, delta, gn_w, gn_b, up_w, up_b);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// =====================================================================================================
// window tail: vis head (pips.py:568) + state write-back + trajectory linking (pips/tracker.py:104-148)
// one thread per point (N is small); fully on device so the chain needs no per-point host logic.
// =====================================================================================================
__global__ void pips_link_kernel(PipsWin w, const float* __restrict__ vis_w, const float* __restrict__ vis_b, float thr0,
                                 int T) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= w.N) return;
  if (!w.active[n]) return;
  const int f = w.wp[0], n_missing = w.wp[1], S = w.S;
  // vis logits for each window slot, sigmoid, write frames f+1 .. f+S-1-n_missing
  for (int s = 1; s < S - n_missing; ++s) {
    const float* ff = w.ffeats + ((size_t)n * S + s) * 128;
    float a = vis_b[0];
    for (int k = 0; k < 128; ++k) a = fmaf(vis_w[k], ff[k], a);
    float v = 1.0f / (1.0f + expf(-a));
    w.vis[(size_t)(f + s) * w.N + n] = v;
    w.traj[((size_t)(f + s) * w.N + n) * 2 + 0] = w.coords[((size_t)n * S + s) * 2 + 0] * (float)w.stride;
    w.traj[((size_t)(f + s) * w.N + n) * 2 + 1] = w.coords[((size_t)n * S + s) * 2 + 1] * (float)w.stride;
  }
  // linking: latest frame in (f, f+S-1-n_missing] whose visibility > thr; thr relaxes by 0.02 per wrap
  float thr = thr0;
  const int earliest = f + 1, last = f + S - n_missing - 1;
  int nxt = last;
  for (int guard = 0; guard < 100000; ++guard) {
    if (!(w.vis[(size_t)nxt * w.N + n] <= thr)) break;
    nxt -= 1;
    if (nxt < earliest) { thr -= 0.02f; nxt = last; }
  }
  w.cur[n] = nxt;
}
int pips_link(Ctx* c, cudaStream_t st, const PipsWin& w, const float* vis_w, const float* vis_b, float thr0, int T) {
  pips_link_kernel<<<cdiv(w.N, 64), 64, 0, st>>>(w, vis_w, vis_b, thr0, T);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

}  // namespace sampt
