// CoTracker v1 (cotracker_stride_4_wind_8) window update on the H100, strict fp32.
// Upstream: co-tracker @ 4f297a9, cotracker/models/core/cotracker/{cotracker.py,blocks.py}, models/core/embeddings.py
// (un-vendored, requirements.txt:31; SURVEY Appendix B.3, PARITY UNPINNED).  Reference call sites:
// sam_pt/point_tracker/cotracker/tracker.py:104,159 (model(rgbs, queries, iters=6)).
//
// The encoder, the correlation pyramid and the fused correlation gather are shared with PIPS (pips_kernels.cu); this file
// adds the transformer input assembly, the UpdateFormer (time / space attention blocks) and the state update.
#include <cstdlib>

#include "common.cuh"
#include "kernels.cuh"
#include "tc_api.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {

constexpr int CT_IN = 456, CT_HID = 384, CT_HEADS = 8, CT_HD = 48;

// ---------------------------------------------------------------------------------------------------------------------
// transformer input: x[n, s, :] = [xy-flow emb (2 + 64 + 64) | corr 196 | ffeat 128 | track_mask, vis_init] + pos[n] + time[s]
// one CTA per (point n, slot s); the correlation gather is the same as pips_corr_kernel.
// pos[n] = bilinear sample of the MAE-style 2-D sincos table (computed in fp64 like the numpy reference, rounded to fp32)
// at the window's first-frame coordinate of the point.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float pos_table(int x, int y, int ch) {
  // table[y, x, :] = [sin(x w_k) (114) | cos(x w_k) (114) | sin(y w_k) (114) | cos(y w_k) (114)], w_k = 10000^(-k/114)
  const int half = CT_IN / 2, q = half / 2;  // 228, 114
  const int axis = ch / half, r = ch % half;
  const int k = r % q;
  const double omega = 1.0 / pow(10000.0, (double)k / (double)q);
  const double a = (double)(axis == 0 ? x : y) * omega;
  return (float)(r < q ? sin(a) : cos(a));
}

// pos[n] = bilinear sample (utils/samp.py semantics: clamped indices, unclamped weights) of the integer-grid sincos table at
// the point's first-slot coordinate AT WINDOW START (upstream forward_iteration computes it once, before the iterations).
__global__ void __launch_bounds__(256)
cot_pos_kernel(PipsWin w, float* __restrict__ pos /*[N,456]*/) {
  const int n = blockIdx.x;
  const float x = w.coords[((size_t)n * w.S + 0) * 2 + 0], y = w.coords[((size_t)n * w.S + 0) * 2 + 1];
  const int H0 = w.H[0], W0 = w.W[0];
  const float x0f = floorf(x), y0f = floorf(y);
  const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
  const int x0c = min(max(x0, 0), W0 - 1), x1c = min(max(x1, 0), W0 - 1), y0c = min(max(y0, 0), H0 - 1), y1c = min(max(y1, 0), H0 - 1);
  const float w00 = ((float)x1 - x) * ((float)y1 - y), w01 = (x - x0f) * ((float)y1 - y), w10 = ((float)x1 - x) * (y - y0f),
              w11 = (x - x0f) * (y - y0f);
  for (int ch = threadIdx.x; ch < CT_IN; ch += 256)
    pos[(size_t)n * CT_IN + ch] = w00 * pos_table(x0c, y0c, ch) + w01 * pos_table(x1c, y0c, ch) + w10 * pos_table(x0c, y1c, ch) +
                                  w11 * pos_table(x1c, y1c, ch);
}

__global__ void __launch_bounds__(256)
cot_input_kernel(PipsWin w, const float* __restrict__ track_mask /*[N,S]*/, const float* __restrict__ vis_init /*[N,S]*/,
                 const float* __restrict__ time_emb /*[S,456]*/, const float* __restrict__ pos /*[N,456]*/,
                 float* __restrict__ xin /*[N*S,456]*/) {
  const int n = blockIdx.x / w.S, s = blockIdx.x % w.S;
  __shared__ float D[4][64];
  __shared__ float sflow[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* ff = w.ffeats + ((size_t)n * w.S + s) * 128;
  const float4 q = *reinterpret_cast<const float4*>(ff + lane * 4);
  const float cx0 = w.coords[((size_t)n * w.S + s) * 2 + 0];
  const float cy0 = w.coords[((size_t)n * w.S + s) * 2 + 1];
  const int fi = w.wp[2 + s];
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
      int pidx = warp * 8 + j;
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
      if (lane == 0) D[l][warp * 8 + j] = d * 0.08838834764831845f;
    }
  }
  if (threadIdx.x == 0) {
    sflow[0] = cx0 - w.coords[((size_t)n * w.S + 0) * 2 + 0];
    sflow[1] = cy0 - w.coords[((size_t)n * w.S + 0) * 2 + 1];
  }
  __syncthreads();
  float* row = xin + ((size_t)n * w.S + s) * CT_IN;
  for (int ch = threadIdx.x; ch < CT_IN; ch += 256) {
    float v;
    if (ch < 2) {
      v = sflow[ch];
    } else if (ch < 130) {
      // get_2d_embedding(flow, 64, cat_coords): [xy | pe_x (sin even / cos odd) | pe_y]
      const int e = ch - 2, d = e / 64, k = (e % 64) / 2;
      const float arg = sflow[d] * ((float)(2 * k) * (1000.0f / 64.0f));
      v = (e & 1) ? cosf(arg) : sinf(arg);
    } else if (ch < 326) {
      const int t = ch - 130;
      const int l = t / 49, r = t % 49, a = r / 7, b = r % 7;
      const float sc = 1.0f / (float)(1 << l);
      const float cx = cx0 * sc, cy = cy0 * sc;
      const int H = w.H[l], W = w.W[l];
      float sx = cx + (float)(a - 3), sy = cy + (float)(b - 3);
      float gx = 2.0f * sx / (float)(W - 1) - 1.0f, gy = 2.0f * sy / (float)(H - 1) - 1.0f;
      float ux = ((gx + 1.0f) * 0.5f) * (float)(W - 1), uy = ((gy + 1.0f) * 0.5f) * (float)(H - 1);
      float xf = floorf(ux), yf = floorf(uy);
      float fx = ux - xf, fy = uy - yf;
      const int bx = (int)floorf(cx) - 3, by = (int)floorf(cy) - 3;
      int ix = (int)xf - bx, iy = (int)yf - by;
      auto at = [&](int yy, int xx) -> float { return (yy >= 0 && yy < 8 && xx >= 0 && xx < 8) ? D[l][yy * 8 + xx] : 0.f; };
      v = (1.f - fx) * (1.f - fy) * at(iy, ix) + fx * (1.f - fy) * at(iy, ix + 1) + (1.f - fx) * fy * at(iy + 1, ix) +
          fx * fy * at(iy + 1, ix + 1);
    } else if (ch < 454) {
      v = ff[ch - 326];
    } else if (ch == 454) {
      v = track_mask[(size_t)n * w.S + s];
    } else {
      v = vis_init[(size_t)n * w.S + s];
    }
    row[ch] = v + pos[(size_t)n * CT_IN + ch] + time_emb[(size_t)s * CT_IN + ch];
  }
}

// LayerNorm without affine (eps 1e-6) over 384 channels, fp32 -> fp32, one warp per row
__global__ void __launch_bounds__(256)
ln384_kernel(const float* __restrict__ x, float* __restrict__ y, int M) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* p = x + (size_t)row * CT_HID;
  float4 v[3];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) { v[i] = *reinterpret_cast<const float4*>(p + (i * 32 + lane) * 4); s += v[i].x + v[i].y + v[i].z + v[i].w; }
  const float mean = warp_sum(s) * (1.0f / CT_HID);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    sq += a * a + b * b + c * c + d * d;
  }
  const float rstd = 1.0f / sqrtf(warp_sum(sq) * (1.0f / CT_HID) + 1e-6f);
#pragma unroll
  for (int i = 0; i < 3; ++i)
    *reinterpret_cast<float4*>(y + (size_t)row * CT_HID + (i * 32 + lane) * 4) =
        make_float4((v[i].x - mean) * rstd, (v[i].y - mean) * rstd, (v[i].z - mean) * rstd, (v[i].w - mean) * rstd);
}

// The same LayerNorm writing the GEMM operand of the tensor-core path: fp16 hi | lo, row pitch 2 * 384 (see gemm_tc.cu: three passes)
__global__ void __launch_bounds__(256)
ln384_split_kernel(const float* __restrict__ x, __half* __restrict__ y, int M) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* p = x + (size_t)row * CT_HID;
  float4 v[3];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) { v[i] = *reinterpret_cast<const float4*>(p + (i * 32 + lane) * 4); s += v[i].x + v[i].y + v[i].z + v[i].w; }
  const float mean = warp_sum(s) * (1.0f / CT_HID);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    sq += a * a + b * b + c * c + d * d;
  }
  const float rstd = 1.0f / sqrtf(warp_sum(sq) * (1.0f / CT_HID) + 1e-6f);
  __half* o = y + (size_t)row * 2 * CT_HID;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int col = (i * 32 + lane) * 4;
    const float r0 = (v[i].x - mean) * rstd, r1 = (v[i].y - mean) * rstd, r2 = (v[i].z - mean) * rstd, r3 = (v[i].w - mean) * rstd;
    const __half2 h0 = __floats2half2_rn(r0, r1), h1 = __floats2half2_rn(r2, r3);
    const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
    const __half2 l0 = __floats2half2_rn(r0 - f0.x, r1 - f0.y), l1 = __floats2half2_rn(r2 - f1.x, r3 - f1.y);
    *reinterpret_cast<uint2*>(o + col) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
    *reinterpret_cast<uint2*>(o + CT_HID + col) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
  }
}
// x [rows, K] fp32 -> fp16 hi | lo [rows, 2K]
__global__ void __launch_bounds__(256)
cot_split_kernel(const float* __restrict__ x, __half* __restrict__ out, long long n4, int K) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n4) return;
  const long long e = i * 4, r = e / K;
  const int cidx = (int)(e % K);
  const float4 v = *reinterpret_cast<const float4*>(x + e);
  const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
  const __half2 l0 = __floats2half2_rn(v.x - f0.x, v.y - f0.y), l1 = __floats2half2_rn(v.z - f1.x, v.w - f1.y);
  __half* o = out + r * 2 * K + cidx;
  *reinterpret_cast<uint2*>(o) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
  *reinterpret_cast<uint2*>(o + K) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
}

// Multi-head attention inside token groups (timm Attention core).  qkv [M, 3*384] with columns [q | k | v], head h at h*48.
// token row of (group g, position l) = g*gstride + l*lstride.  One CTA per (group, head): K/V staged in shared memory,
// one warp per query row (lanes over keys for the scores, over channels for the output).
__global__ void __launch_bounds__(256)
cot_attn_kernel(const float* __restrict__ qkv, float* __restrict__ out, int L, int gstride, int lstride) {
  extern __shared__ float sm[];
  float* sk = sm;                         // [L][49]
  float* sv = sm + (size_t)L * 49;        // [L][49]
  float* sp = sv + (size_t)L * 49;        // [8 warps][L] probabilities
  const int g = blockIdx.x, h = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < L * CT_HD; i += 256) {
    const int l = i / CT_HD, d = i % CT_HD;
    const float* r = qkv + (size_t)(g * gstride + l * lstride) * (3 * CT_HID) + h * CT_HD + d;
    sk[l * 49 + d] = r[CT_HID];
    sv[l * 49 + d] = r[2 * CT_HID];
  }
  __syncthreads();
  const float scale = 1.0f / sqrtf((float)CT_HD);
  float* pw = sp + (size_t)warp * L;
  // blockIdx.z splits the queries of a group (space attention at 256 points has only 8 groups x 8 heads = 64 (group, head) pairs)
  const int qchunk = (L + gridDim.z - 1) / gridDim.z, q_begin = blockIdx.z * qchunk, q_end = min(L, q_begin + qchunk);
  for (int lq = q_begin + warp; lq < q_end; lq += 8) {
    const float* qr = qkv + (size_t)(g * gstride + lq * lstride) * (3 * CT_HID) + h * CT_HD;
    float qv[CT_HD];
#pragma unroll
    for (int d = 0; d < CT_HD; ++d) qv[d] = qr[d];
    float mx = -INFINITY;
    for (int j = lane; j < L; j += 32) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < CT_HD; ++d) s = fmaf(qv[d], sk[j * 49 + d], s);
      s *= scale;
      pw[j] = s;
      mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j < L; j += 32) { float p = expf(pw[j] - mx); pw[j] = p; sum += p; }
    sum = warp_sum(sum);
    __syncwarp();
    const float inv = 1.0f / sum;
    for (int d = lane; d < CT_HD; d += 32) {
      float a = 0.f;
      for (int j = 0; j < L; ++j) a = fmaf(pw[j], sv[j * 49 + d], a);
      out[(size_t)(g * gstride + lq * lstride) * CT_HID + h * CT_HD + d] = a * inv;
    }
    __syncwarp();
  }
}

// state update after the UpdateFormer (upstream forward_iteration tail): ffeat += GELU(Linear(GroupNorm(1,128)(dfeat)));
// coords += dxy (all slots: CoTracker does NOT lock the first frame).  one CTA per (n, s), 128 threads.
__global__ void __launch_bounds__(128)
cot_update_kernel(PipsWin w, const float* __restrict__ delta /*[N*S,130]*/, const float* __restrict__ gn_w, const float* __restrict__ gn_b,
                  const float* __restrict__ up_w, const float* __restrict__ up_b) {
  const int n = blockIdx.x / w.S, s = blockIdx.x % w.S;
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
    acc = fmaf(ww.x, g[k], acc); acc = fmaf(ww.y, g[k + 1], acc); acc = fmaf(ww.z, g[k + 2], acc); acc = fmaf(ww.w, g[k + 3], acc);
  }
  w.ffeats[((size_t)n * w.S + s) * 128 + t] += gelu_erf(acc);
  if (t < 2) w.coords[((size_t)n * w.S + s) * 2 + t] += d[t];
}
__global__ void cot_vis_kernel(PipsWin w, const float* __restrict__ vis_w, const float* __restrict__ vis_b, float* __restrict__ vis_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (n, s)
  if (i >= w.N * w.S) return;
  const float* ff = w.ffeats + (size_t)i * 128;
  float a = vis_b[0];
  for (int k = 0; k < 128; ++k) a = fmaf(vis_w[k], ff[k], a);
  vis_out[i] = a;
}

// F.interpolate(rgbs.float(), interp_shape, mode="bilinear") of the reference wrapper (cotracker/tracker.py:79-81): ATen
// upsample_bilinear2d, align_corners=False, no antialiasing.  uint8 planar (n,3,H,W) -> float32 planar (n,3,Ho,Wo).
__global__ void resize_bilinear_u8_f32_kernel(const uint8_t* __restrict__ in, float* __restrict__ out, int H, int W, int Ho, int Wo,
                                              float sy, float sx, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho);
  const long long plane = i / ((long long)Wo * Ho);
  const float fy = fmaxf(sy * ((float)oy + 0.5f) - 0.5f, 0.f), fx = fmaxf(sx * ((float)ox + 0.5f) - 0.5f, 0.f);
  const int y0 = min((int)fy, H - 1), x0 = min((int)fx, W - 1);
  const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
  const float ly1 = fy - (float)y0, lx1 = fx - (float)x0, ly0 = 1.f - ly1, lx0 = 1.f - lx1;
  const uint8_t* p = in + plane * H * W;
  out[i] = ly0 * (lx0 * (float)p[(size_t)y0 * W + x0] + lx1 * (float)p[(size_t)y0 * W + x1]) +
           ly1 * (lx0 * (float)p[(size_t)y1 * W + x0] + lx1 * (float)p[(size_t)y1 * W + x1]);
}

// feat_init of newly born points (upstream CoTracker.forward: bilinear_sample2d(fmaps[first frame of the point], coords)):
// out[n, s, :] = sample for every slot s.  clamp indices, UNCLAMPED weights (utils/samp.py semantics).  one CTA per point.
__global__ void cot_sample_kernel(const float* __restrict__ fmaps, int H, int W, const int* __restrict__ frame, const float* __restrict__ xy,
                                  float* __restrict__ out, int S) {
  const int n = blockIdx.x, c = threadIdx.x;
  const float x = xy[n * 2 + 0], y = xy[n * 2 + 1];
  const float* fm = fmaps + (size_t)frame[n] * H * W * 128;
  const float x0f = floorf(x), y0f = floorf(y);
  const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
  const int x0c = min(max(x0, 0), W - 1), x1c = min(max(x1, 0), W - 1), y0c = min(max(y0, 0), H - 1), y1c = min(max(y1, 0), H - 1);
  const float x1f = (float)x1, y1f = (float)y1;
  const float w00 = (x1f - x) * (y1f - y), w01 = (x - x0f) * (y1f - y), w10 = (x1f - x) * (y - y0f), w11 = (x - x0f) * (y - y0f);
  const float f = w00 * fm[((size_t)y0c * W + x0c) * 128 + c] + w01 * fm[((size_t)y0c * W + x1c) * 128 + c] +
                  w10 * fm[((size_t)y1c * W + x0c) * 128 + c] + w11 * fm[((size_t)y1c * W + x1c) * 128 + c];
  for (int s = 0; s < S; ++s) out[((size_t)n * S + s) * 128 + c] = f;
}

struct CotBlockW {
  const float *qkv_w, *qkv_b, *proj_w, *proj_b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
  const __half *qkv_w16, *proj_w16, *fc1_w16, *fc2_w16;   // fp16 hi | lo copies [N, 2K] (registered by the host), or null
};

static int load_block(Ctx* c, const std::string& p, CotBlockW* b) {
  SAMPT_TRY(get_f32(c, p + "attn.qkv.weight", &b->qkv_w)); SAMPT_TRY(get_f32(c, p + "attn.qkv.bias", &b->qkv_b));
  SAMPT_TRY(get_f32(c, p + "attn.proj.weight", &b->proj_w)); SAMPT_TRY(get_f32(c, p + "attn.proj.bias", &b->proj_b));
  SAMPT_TRY(get_f32(c, p + "mlp.fc1.weight", &b->fc1_w)); SAMPT_TRY(get_f32(c, p + "mlp.fc1.bias", &b->fc1_b));
  SAMPT_TRY(get_f32(c, p + "mlp.fc2.weight", &b->fc2_w)); SAMPT_TRY(get_f32(c, p + "mlp.fc2.bias", &b->fc2_b));
  b->qkv_w16 = b->proj_w16 = b->fc1_w16 = b->fc2_w16 = nullptr;
  if (c->find(p + "attn.qkv.w16") != nullptr) {
    SAMPT_TRY(get_f16(c, p + "attn.qkv.w16", &b->qkv_w16)); SAMPT_TRY(get_f16(c, p + "attn.proj.w16", &b->proj_w16));
    SAMPT_TRY(get_f16(c, p + "mlp.fc1.w16", &b->fc1_w16)); SAMPT_TRY(get_f16(c, p + "mlp.fc2.w16", &b->fc2_w16));
  }
  return 0;
}

struct CotBufs {
  float *x, *h, *qkv, *att, *mlp;
  __half *h16, *att16, *mlp16;   // hi | lo operands of the tensor-core path (null: fp32 CUDA-core GEMMs)
};

// Y[M, N] (fp32, + bias, + residual) or the next operand (fp16 hi | lo, GELU-tanh) = X16 . W16^T in three tensor-core passes
// (A_hi.B_hi + A_lo.B_hi + A_hi.B_lo into one fp32 register accumulator: products exact to ~2^-22, i.e. fp32-level like the CUDA-core
// path it replaces).  The UpdateFormer is 21.5 M parameters x (8 N) token rows x 6 iterations x ~24 windows x 2 directions: at
// N = 256 points (C5) that is 25 TFLOP per clip -- 1.2 s on the fp32 pipes, the longest serial stage of a frame-sharded C5 clip.
static int cot_tcg(Ctx* c, cudaStream_t st, const __half* X16, const __half* W16, const float* bias, const float* resid, float* Y32,
                   __half* Y16, int act, int M, int N, int K) {
  GemmSeg seg{};
  seg.nseg = 3;
  seg.a_off[0] = 0; seg.b_off[0] = 0;
  seg.a_off[1] = K; seg.b_off[1] = 0;
  seg.a_off[2] = 0; seg.b_off[2] = K;
  GemmEpi ep{};
  ep.bias = bias; ep.act = act;
  if (Y16) { ep.out16 = Y16; ep.ldc = 2 * N; ep.split_off = N; }
  else { ep.out32 = Y32; ep.ldc = N; ep.resid = resid; }
  return gemm_tc(c, st, X16, 2 * K, W16, 2 * K, M, N, K, seg, ep);
}

// LayerNorm of M rows: fp32 into y32, or the fp16 hi | lo operand of the tensor-core path into y16 (exactly one is non-null)
static int cot_ln(Ctx* c, cudaStream_t st, const float* x, float* y32, __half* y16, int M) {
  if (y16) ln384_split_kernel<<<cdiv(M, 8), 256, 0, st>>>(x, y16, M);
  else ln384_kernel<<<cdiv(M, 8), 256, 0, st>>>(x, y32, M);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// x [M, K] fp32 -> fp16 hi | lo [M, 2K]
static int cot_split(Ctx* c, cudaStream_t st, const float* x, __half* out, int M, int K) {
  const long long n4 = (long long)M * K / 4;
  cot_split_kernel<<<cdiv(n4, 256), 256, 0, st>>>(x, out, n4, K);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// attention core over G groups of L tokens.  qsplit CTAs share a group's queries; qsplit <= 0 picks the count the window uses
// (double it while the grid is under two waves and every chunk keeps >= 8 queries).
static int cot_attn(Ctx* c, cudaStream_t st, const float* qkv, float* out, int G, int L, int gstride, int lstride, int qsplit) {
  size_t smem = ((size_t)L * 49 * 2 + (size_t)8 * L) * sizeof(float);
  SAMPT_CHECK(smem <= 200 * 1024, "cot_attn: %d tokens per group do not fit shared memory", L);
  SAMPT_TRY(ensure_func_smem(c, "cot_attn_kernel", cot_attn_kernel, 200 * 1024));
  if (qsplit <= 0) {
    qsplit = 1;
    while (qsplit < 8 && G * CT_HEADS * qsplit < 2 * c->num_sms && L / (2 * qsplit) >= 8) qsplit *= 2;
  }
  cot_attn_kernel<<<dim3(G, CT_HEADS, qsplit), 256, smem, st>>>(qkv, out, L, gstride, lstride);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// AttnBlock: x += proj(attn(LN(x))) ; x += fc2(gelu_tanh(fc1(LN(x))))    (groups: G x L tokens)
// tc: the four GEMMs on tensor cores (three fp16 hi | lo passes; needs the ".w16" weights and b.h16 / att16 / mlp16), else fp32 sgemm
static int attn_block(Ctx* c, cudaStream_t st, const CotBlockW& w, CotBufs& b, bool tc, int M, int G, int L, int gstride, int lstride) {
  if (tc) {
    SAMPT_CHECK(w.qkv_w16 != nullptr && b.h16 != nullptr, "cot attn_block: the tensor-core path needs the .w16 weights");
    SAMPT_TRY(cot_ln(c, st, b.x, nullptr, b.h16, M));
    SAMPT_TRY(cot_tcg(c, st, b.h16, w.qkv_w16, w.qkv_b, nullptr, b.qkv, nullptr, 0, M, 3 * CT_HID, CT_HID));
  } else {
    SAMPT_TRY(cot_ln(c, st, b.x, b.h, nullptr, M));
    SAMPT_TRY(sgemm_nt(c, st, b.h, CT_HID, w.qkv_w, CT_HID, w.qkv_b, nullptr, 0, b.qkv, 3 * CT_HID, M, 3 * CT_HID, CT_HID, 0));
  }
  SAMPT_TRY(cot_attn(c, st, b.qkv, b.att, G, L, gstride, lstride, 0));
  if (tc) {
    SAMPT_TRY(cot_split(c, st, b.att, b.att16, M, CT_HID));
    SAMPT_TRY(cot_tcg(c, st, b.att16, w.proj_w16, w.proj_b, b.x, b.x, nullptr, 0, M, CT_HID, CT_HID));
    SAMPT_TRY(cot_ln(c, st, b.x, nullptr, b.h16, M));
    SAMPT_TRY(cot_tcg(c, st, b.h16, w.fc1_w16, w.fc1_b, nullptr, nullptr, b.mlp16, 3, M, 4 * CT_HID, CT_HID));   // GELU(tanh), hi | lo out
    SAMPT_TRY(cot_tcg(c, st, b.mlp16, w.fc2_w16, w.fc2_b, b.x, b.x, nullptr, 0, M, CT_HID, 4 * CT_HID));
    return 0;
  }
  SAMPT_TRY(sgemm_nt(c, st, b.att, CT_HID, w.proj_w, CT_HID, w.proj_b, b.x, CT_HID, b.x, CT_HID, M, CT_HID, CT_HID, 0));
  SAMPT_TRY(cot_ln(c, st, b.x, b.h, nullptr, M));
  SAMPT_TRY(sgemm_nt(c, st, b.h, CT_HID, w.fc1_w, CT_HID, w.fc1_b, nullptr, 0, b.mlp, 4 * CT_HID, M, 4 * CT_HID, CT_HID, 3));
  SAMPT_TRY(sgemm_nt(c, st, b.mlp, 4 * CT_HID, w.fc2_w, 4 * CT_HID, w.fc2_b, b.x, CT_HID, b.x, CT_HID, M, CT_HID, 4 * CT_HID, 0));
  return 0;
}

// GroupNorm / ffeat updater / visibility head weights
struct CotHeadW {
  const float *gn_w, *gn_b, *up_w, *up_b, *vis_w, *vis_b;
};

static int load_head(Ctx* c, CotHeadW* h) {
  SAMPT_TRY(get_f32(c, "cot.norm.weight", &h->gn_w)); SAMPT_TRY(get_f32(c, "cot.norm.bias", &h->gn_b));
  SAMPT_TRY(get_f32(c, "cot.ffeat_updater.0.weight", &h->up_w)); SAMPT_TRY(get_f32(c, "cot.ffeat_updater.0.bias", &h->up_b));
  SAMPT_TRY(get_f32(c, "cot.vis_predictor.0.weight", &h->vis_w)); SAMPT_TRY(get_f32(c, "cot.vis_predictor.0.bias", &h->vis_b));
  return 0;
}

static int cot_pos(Ctx* c, cudaStream_t st, const PipsWin& w, float* pos) {
  cot_pos_kernel<<<w.N, 256, 0, st>>>(w, pos);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

static int cot_input(Ctx* c, cudaStream_t st, const PipsWin& w, const float* track_mask, const float* vis_init, const float* time_emb,
                     const float* pos, float* xin) {
  cot_input_kernel<<<w.N * w.S, 256, 0, st>>>(w, track_mask, vis_init, time_emb, pos, xin);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

static int cot_update(Ctx* c, cudaStream_t st, const PipsWin& w, const float* delta, const CotHeadW& h) {
  cot_update_kernel<<<w.N * w.S, 128, 0, st>>>(w, delta, h.gn_w, h.gn_b, h.up_w, h.up_b);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

static int cot_vis(Ctx* c, cudaStream_t st, const PipsWin& w, const CotHeadW& h, float* vis_out) {
  cot_vis_kernel<<<cdiv(w.N * w.S, 128), 128, 0, st>>>(w, h.vis_w, h.vis_b, vis_out);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

static PipsWin cot_win(const float* fmaps, const float* l1, const float* l2, const float* l3, int H4, int W4, const int* fidx_dev,
                       float* coords, float* ffeats, int N) {
  PipsWin w{};
  w.N = N; w.S = 8; w.stride = 4; w.T = 8;
  w.pyr[0] = fmaps; w.pyr[1] = l1; w.pyr[2] = l2; w.pyr[3] = l3;
  w.H[0] = H4; w.W[0] = W4;
  for (int l = 1; l < 4; ++l) { w.H[l] = w.H[l - 1] / 2; w.W[l] = w.W[l - 1] / 2; }
  w.coords = coords; w.ffeats = ffeats;
  w.wp = fidx_dev;
  return w;
}

}  // namespace sampt

using namespace sampt;

// One CoTracker window (upstream CoTracker.forward_iteration): `iters` refinement iterations over S = 8 frames for N points.
//   pyramid levels (T,H_l,W_l,128) channels-last (as for PIPS); fidx_dev: device int32[10] = [0, 0, frame index feeding slot 0..7];
//   coords (N,S,2) feature-map px IN/OUT; ffeats (N,S,128) IN/OUT; track_mask (N,S), vis_init (N,S) fp32;
//   time_emb (S,456) fp32 table; vis_out (N,S) raw visibility logits.
extern "C" int sampt_cotracker_window(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int H4,
                                      int W4, const int* fidx_dev, float* coords, float* ffeats, const float* track_mask,
                                      const float* vis_init, const float* time_emb, int N, int iters, int time_depth, int space_depth,
                                      float* vis_out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int S = 8, M = N * S;
  SAMPT_CHECK(N > 0, "sampt_cotracker_window: no points");
  SAMPT_CHECK(time_depth >= space_depth && space_depth > 0 && time_depth % space_depth == 0, "unsupported block layout");
  c->ws_reset();
  const std::string p = "cot.updateformer.";
  std::vector<CotBlockW> tb(time_depth), sb(space_depth);
  for (int i = 0; i < time_depth; ++i) SAMPT_TRY(load_block(c, p + "time_blocks." + std::to_string(i) + ".", &tb[i]));
  for (int i = 0; i < space_depth; ++i) SAMPT_TRY(load_block(c, p + "space_blocks." + std::to_string(i) + ".", &sb[i]));
  const float *in_w, *in_b, *fh_w, *fh_b;
  SAMPT_TRY(get_f32(c, p + "input_transform.weight", &in_w)); SAMPT_TRY(get_f32(c, p + "input_transform.bias", &in_b));
  SAMPT_TRY(get_f32(c, p + "flow_head.weight", &fh_w)); SAMPT_TRY(get_f32(c, p + "flow_head.bias", &fh_b));
  CotHeadW hw;
  SAMPT_TRY(load_head(c, &hw));
  const PipsWin w = cot_win(fmaps, l1, l2, l3, H4, W4, fidx_dev, coords, ffeats, N);
  CotBufs b;
  float *xin, *delta, *pos;
  SAMPT_TRY(ws_get(c, &xin, (size_t)M * CT_IN, "cot xin"));
  SAMPT_TRY(ws_get(c, &pos, (size_t)N * CT_IN, "cot pos"));
  SAMPT_TRY(ws_get(c, &b.x, (size_t)M * CT_HID, "cot x"));
  SAMPT_TRY(ws_get(c, &b.h, (size_t)M * CT_HID, "cot h"));
  SAMPT_TRY(ws_get(c, &b.qkv, (size_t)M * 3 * CT_HID, "cot qkv"));
  SAMPT_TRY(ws_get(c, &b.att, (size_t)M * CT_HID, "cot att"));
  SAMPT_TRY(ws_get(c, &b.mlp, (size_t)M * 4 * CT_HID, "cot mlp"));
  SAMPT_TRY(ws_get(c, &delta, (size_t)M * 130, "cot delta"));
  // UpdateFormer GEMMs on tensor cores (three fp16 hi | lo passes) once the token count fills 128-row tiles; SAMPT_COT_TC=0 keeps fp32
  static const int cot_tc_on = [] { const char* e = std::getenv("SAMPT_COT_TC"); return (e != nullptr && e[0] == '0') ? 0 : 1; }();
  b.h16 = b.att16 = b.mlp16 = nullptr;
  // (each block then runs on tensor cores when its own ".w16" weights are registered)
  const bool tc = cot_tc_on && M >= 128 && tb[0].qkv_w16 != nullptr;
  if (tc) {
    SAMPT_TRY(ws_get(c, &b.h16, (size_t)M * 2 * CT_HID, "cot h16"));
    SAMPT_TRY(ws_get(c, &b.att16, (size_t)M * 2 * CT_HID, "cot att16"));
    SAMPT_TRY(ws_get(c, &b.mlp16, (size_t)M * 8 * CT_HID, "cot mlp16"));
  }
  SAMPT_TRY(cot_pos(c, st, w, pos));
  for (int it = 0; it < iters; ++it) {
    SAMPT_TRY(cot_input(c, st, w, track_mask, vis_init, time_emb, pos, xin));
    SAMPT_TRY(sgemm_nt(c, st, xin, CT_IN, in_w, CT_IN, in_b, nullptr, 0, b.x, CT_HID, M, CT_HID, CT_IN, 0));
    int j = 0;
    for (int i = 0; i < time_depth; ++i) {
      // time attention: N groups of S consecutive tokens (token row = n*S + s)
      SAMPT_TRY(attn_block(c, st, tb[i], b, tc && tb[i].qkv_w16 != nullptr, M, N, S, S, 1));
      if (i % (time_depth / space_depth) == 0) {
        // space attention: S groups of N tokens (row = s + n*S)
        SAMPT_TRY(attn_block(c, st, sb[j], b, tc && sb[j].qkv_w16 != nullptr, M, S, N, 1, S));
        ++j;
      }
    }
    // flow_head: 384 -> 130
    SAMPT_TRY(sgemm_nt(c, st, b.x, CT_HID, fh_w, CT_HID, fh_b, nullptr, 0, delta, 130, M, 130, CT_HID, 0));
    SAMPT_TRY(cot_update(c, st, w, delta, hw));
  }
  return cot_vis(c, st, w, hw, vis_out);
}

extern "C" int sampt_resize_bilinear_u8_f32(sampt_ctx* ctx, const uint8_t* in, int planes, int H, int W, int Ho, int Wo, float* out,
                                            void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)planes * Ho * Wo;
  if (total == 0) return 0;
  resize_bilinear_u8_f32_kernel<<<cdiv(total, 256), 256, 0, st>>>(in, out, H, W, Ho, Wo, (float)H / (float)Ho, (float)W / (float)Wo, total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

extern "C" int sampt_cotracker_sample_features(sampt_ctx* ctx, const float* fmaps, int H4, int W4, const int* frame_dev,
                                               const float* xy_dev, int N, int S, float* out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  if (N <= 0) return 0;
  cot_sample_kernel<<<N, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(fmaps, H4, W4, frame_dev, xy_dev, out, S);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// unit-test entries (include/sampt_b200.h): each runs the launchers of sampt_cotracker_window on caller-owned buffers
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int sampt_test_cotracker_input(sampt_ctx* ctx, const float* fmaps, const float* l1, const float* l2, const float* l3, int H4,
                                          int W4, const int* slots_host, const float* coords, const float* ffeats, const float* track_mask,
                                          const float* vis_init, const float* time_emb, int N, float* pos, float* xin, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(N >= 1 && slots_host != nullptr, "sampt_test_cotracker_input: N positive and 8 slot frames required");
  c->ws_reset();
  int fidx_h[10] = {0, 0};
  for (int s = 0; s < 8; ++s) fidx_h[2 + s] = slots_host[s];
  int* fidx_d;
  SAMPT_TRY(ws_get(c, &fidx_d, 16, "cot test slots"));
  SAMPT_CUDA(cudaMemcpyAsync(fidx_d, fidx_h, sizeof(fidx_h), cudaMemcpyHostToDevice, st));
  SAMPT_CUDA(cudaStreamSynchronize(st));
  const PipsWin w = cot_win(fmaps, l1, l2, l3, H4, W4, fidx_d, const_cast<float*>(coords), const_cast<float*>(ffeats), N);
  SAMPT_TRY(cot_pos(c, st, w, pos));
  return cot_input(c, st, w, track_mask, vis_init, time_emb, pos, xin);
}

extern "C" int sampt_test_cotracker_ln(sampt_ctx* ctx, int op, const float* x, int M, int K, float* y32, void* y16, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(M >= 1, "sampt_test_cotracker_ln: no rows");
  switch (op) {
    case 0:
    case 1:
      SAMPT_CHECK(K == CT_HID, "sampt_test_cotracker_ln: LayerNorm rows have %d channels", CT_HID);
      return cot_ln(c, st, x, op == 0 ? y32 : nullptr, op == 1 ? static_cast<__half*>(y16) : nullptr, M);
    case 2:
      SAMPT_CHECK(K >= 4 && K % 4 == 0, "sampt_test_cotracker_ln: split needs K a positive multiple of 4");
      return cot_split(c, st, x, static_cast<__half*>(y16), M, K);
    default:
      set_error("sampt_test_cotracker_ln: unknown op %d", op);
      return -2;
  }
}

extern "C" int sampt_test_cotracker_attn(sampt_ctx* ctx, const float* qkv, float* out, int G, int L, int gstride, int lstride, int qsplit,
                                         void* stream) {
  SAMPT_CHECK(G >= 1 && L >= 1 && qsplit <= 8, "sampt_test_cotracker_attn: G, L positive and qsplit <= 8 required");
  return cot_attn(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), qkv, out, G, L, gstride, lstride, qsplit);
}

extern "C" int sampt_test_cotracker_block(sampt_ctx* ctx, int kind, int blk, int tc, float* x, int N, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK((kind == 0 || kind == 1) && N >= 1, "sampt_test_cotracker_block: kind 0 (time) or 1 (space), N positive");
  c->ws_reset();
  const int S = 8, M = N * S;
  CotBlockW w;
  SAMPT_TRY(load_block(c, std::string("cot.updateformer.") + (kind ? "space_blocks." : "time_blocks.") + std::to_string(blk) + ".", &w));
  SAMPT_CHECK(!tc || w.qkv_w16 != nullptr, "sampt_test_cotracker_block: tc = 1 needs the .w16 weights");
  CotBufs b;
  b.x = x;
  SAMPT_TRY(ws_get(c, &b.h, (size_t)M * CT_HID, "cot h"));
  SAMPT_TRY(ws_get(c, &b.qkv, (size_t)M * 3 * CT_HID, "cot qkv"));
  SAMPT_TRY(ws_get(c, &b.att, (size_t)M * CT_HID, "cot att"));
  SAMPT_TRY(ws_get(c, &b.mlp, (size_t)M * 4 * CT_HID, "cot mlp"));
  b.h16 = b.att16 = b.mlp16 = nullptr;
  if (tc) {
    SAMPT_TRY(ws_get(c, &b.h16, (size_t)M * 2 * CT_HID, "cot h16"));
    SAMPT_TRY(ws_get(c, &b.att16, (size_t)M * 2 * CT_HID, "cot att16"));
    SAMPT_TRY(ws_get(c, &b.mlp16, (size_t)M * 8 * CT_HID, "cot mlp16"));
  }
  if (kind == 0) return attn_block(c, st, w, b, tc != 0, M, N, S, S, 1);
  return attn_block(c, st, w, b, tc != 0, M, S, N, 1, S);
}

extern "C" int sampt_test_cotracker_update(sampt_ctx* ctx, const float* delta, float* coords, float* ffeats, int N, float* vis_out,
                                           void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(N >= 1, "sampt_test_cotracker_update: no points");
  CotHeadW hw;
  SAMPT_TRY(load_head(c, &hw));
  const PipsWin w = cot_win(nullptr, nullptr, nullptr, nullptr, 0, 0, nullptr, coords, ffeats, N);
  SAMPT_TRY(cot_update(c, st, w, delta, hw));
  return cot_vis(c, st, w, hw, vis_out);
}
