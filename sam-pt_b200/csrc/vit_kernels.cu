// Memory-bound helper kernels of the SAM ViT encoder path (everything that is not a tensor-core contraction):
// PIL-exact uint8 resize, preprocess + patch im2col, LayerNorm (+ window partition gather, fp16 hi|lo output),
// attention operand preparation (rel-pos folding), neck im2col, final LayerNorm2d -> NCHW.
// Upstream arithmetic: segment_anything/modeling/image_encoder.py (un-vendored; SURVEY Appendix B.1).
#include "common.cuh"
#include "kernels.cuh"
#include "tc_common.cuh"
#include "tc_api.cuh"

namespace sampt {

// ---------------------------------------------------------------------------------------------------------------------
// Pillow-exact bilinear resize of uint8 images (ImagingResample: horizontal pass then vertical pass, 22-bit fixed point
// coefficients, round-half-up accumulate, clip8).  Coefficient tables are computed on the host exactly as Pillow's
// precompute_coeffs / normalize_coeffs_8bpc do (sampt_b200/pil_resize.py) -- ResizeLongestSide.apply_image parity.
// ---------------------------------------------------------------------------------------------------------------------
// horizontal: in planar (B,3,H,W) u8 -> tmp planar (B,3,H,Wo) u8
__global__ void pil_resize_h_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, const int* __restrict__ bounds,
                                    const int* __restrict__ kk, int ksize, int H, int W, int Wo, long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int xo = (int)(i % Wo);
  long long row = i / Wo;  // (b*3 + c)*H + y
  const uint8_t* src = in + row * W;
  int xmin = bounds[2 * xo], xcnt = bounds[2 * xo + 1];
  const int* k = kk + (size_t)xo * ksize;
  int ss = 1 << 21;
  for (int x = 0; x < xcnt; ++x) ss += (int)src[xmin + x] * k[x];
  ss >>= 22;
  out[i] = (uint8_t)min(max(ss, 0), 255);
}
// vertical: tmp planar (B,3,H,Wo) u8 -> out planar (B,3,Ho,Wo) u8
__global__ void pil_resize_v_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, const int* __restrict__ bounds,
                                    const int* __restrict__ kk, int ksize, int H, int Ho, int Wo, long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int xo = (int)(i % Wo);
  int yo = (int)((i / Wo) % Ho);
  long long plane = i / ((long long)Wo * Ho);
  const uint8_t* src = in + plane * H * Wo + xo;
  int ymin = bounds[2 * yo], ycnt = bounds[2 * yo + 1];
  const int* k = kk + (size_t)yo * ksize;
  int ss = 1 << 21;
  for (int y = 0; y < ycnt; ++y) ss += (int)src[(size_t)(ymin + y) * Wo] * k[y];
  ss >>= 22;
  out[i] = (uint8_t)min(max(ss, 0), 255);
}
int pil_resize(Ctx* c, cudaStream_t st, const uint8_t* in, uint8_t* tmp, uint8_t* out, int B, int H, int W, int Ho, int Wo,
               const int* hb, const int* hk, int hks, const int* vb, const int* vk, int vks) {
  long long t1 = (long long)B * 3 * H * Wo, t2 = (long long)B * 3 * Ho * Wo;
  pil_resize_h_kernel<<<cdiv(t1, 256), 256, 0, st>>>(in, tmp, hb, hk, hks, H, W, Wo, t1);
  SAMPT_LAUNCH_CHECK();
  pil_resize_v_kernel<<<cdiv(t2, 256), 256, 0, st>>>(tmp, out, vb, vk, vks, H, Ho, Wo, t2);
  SAMPT_LAUNCH_CHECK();
  c->launches += 2;
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Sam.preprocess ((x-mean)/std, zero pad to 1024^2) fused with the patch-embed im2col:
//   A[(b*G + py)*G + px][c*P*P + iy*P + ix] = norm(img[b, c, py*P+iy, px*P+ix])   (0 beyond the resized image)
// output fp16 hi (| lo at column split_off)
// ---------------------------------------------------------------------------------------------------------------------
// float variant: the image is ALREADY normalised and zero-padded (upstream ImageEncoderViT.forward(x) takes Sam.preprocess output)
__global__ void im2col_f32_kernel(const float* __restrict__ img, __half* __restrict__ A, int G, int P, int ld, int split_off,
                                  long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int K = 3 * P * P, S = G * P;
  int k = (int)(i % K);
  long long tok = i / K;
  int px = (int)(tok % G), py = (int)((tok / G) % G), b = (int)(tok / ((long long)G * G));
  int ch = k / (P * P), iy = (k / P) % P, ix = k % P;
  const float v = img[(((size_t)b * 3 + ch) * S + py * P + iy) * S + px * P + ix];
  __half h = __float2half_rn(v);
  A[(size_t)tok * ld + k] = h;
  if (split_off > 0) A[(size_t)tok * ld + split_off + k] = __float2half_rn(v - __half2float(h));
}
int im2col_f32(Ctx* c, cudaStream_t st, const float* img, __half* A, int B, int G, int P, int ld, int split_off) {
  long long total = (long long)B * G * G * 3 * P * P;
  im2col_f32_kernel<<<cdiv(total, 256), 256, 0, st>>>(img, A, G, P, ld, split_off, total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

__global__ void preprocess_im2col_kernel(const uint8_t* __restrict__ img, __half* __restrict__ A, int B, int Hr, int Wr, int G,
                                         int P, int ld, int split_off, float m0, float m1, float m2, float s0, float s1,
                                         float s2, long long total) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int K = 3 * P * P;
  int k = (int)(i % K);
  long long tok = i / K;
  int px = (int)(tok % G), py = (int)((tok / G) % G), b = (int)(tok / ((long long)G * G));
  int ch = k / (P * P), iy = (k / P) % P, ix = k % P;
  int y = py * P + iy, x = px * P + ix;
  float v = 0.f;
  if (y < Hr && x < Wr) {
    float mean = ch == 0 ? m0 : (ch == 1 ? m1 : m2);
    float sd = ch == 0 ? s0 : (ch == 1 ? s1 : s2);
    v = ((float)img[(((size_t)b * 3 + ch) * Hr + y) * Wr + x] - mean) / sd;
  }
  __half h = __float2half_rn(v);
  A[(size_t)tok * ld + k] = h;
  if (split_off > 0) A[(size_t)tok * ld + split_off + k] = __float2half_rn(v - __half2float(h));
}
int preprocess_im2col(Ctx* c, cudaStream_t st, const uint8_t* img, __half* A, int B, int Hr, int Wr, int G, int P, int ld,
                      int split_off, const float* mean, const float* stdv) {
  long long total = (long long)B * G * G * 3 * P * P;
  preprocess_im2col_kernel<<<cdiv(total, 256), 256, 0, st>>>(img, A, B, Hr, Wr, G, P, ld, split_off, mean[0], mean[1], mean[2],
                                                             stdv[0], stdv[1], stdv[2], total);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Row LayerNorm / cast with optional gather (window partition + zero padding), fp16 hi (| lo) output.
//   out[r, :] = gamma * (x[src[r], :] - mean) * rstd + beta   (src[r] < 0 -> zeros: padding is applied AFTER the norm,
//   upstream Block.forward: norm1 -> window_partition(pad))
// one warp per output row; D % 128 == 0, D <= 1536
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ln_rows_kernel(const float* __restrict__ x, int ldx, const int* __restrict__ src, const float* __restrict__ gamma,
               const float* __restrict__ beta, float eps, __half* __restrict__ out, int ldo, int split_off, int Mout, int D,
               int normalize, int f8) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= Mout) return;
  const int nv = D / 128;  // float4 per lane
  __half* o = out + (size_t)row * ldo;
  int s = src ? src[row] : row;
  if (s < 0) {
    for (int i = 0; i < nv; ++i) {
      int col = (i * 32 + lane) * 4;
      *reinterpret_cast<uint2*>(o + col) = make_uint2(0u, 0u);
      if (split_off > 0) *reinterpret_cast<uint2*>(o + split_off + col) = make_uint2(0u, 0u);   // (f8: the same 2*D bytes, zero = 0.0 in e4m3)
    }
    return;
  }
  const float* xp = x + (size_t)s * ldx;
  float4 v[12];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    if (i < nv) {
      v[i] = *reinterpret_cast<const float4*>(xp + (i * 32 + lane) * 4);
      sum += v[i].x + v[i].y + v[i].z + v[i].w;
    }
  }
  float mean = 0.f, rstd = 1.f;
  if (normalize) {
    mean = warp_sum(sum) / (float)D;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < 12; ++i) {
      if (i < nv) {
        float a = v[i].x - mean, b = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
        sq += a * a + b * b + cc * cc + d * d;
      }
    }
    rstd = 1.0f / sqrtf(warp_sum(sq) / (float)D + eps);
  }
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    if (i < nv) {
      int col = (i * 32 + lane) * 4;
      float r[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
      if (normalize) {
        float4 g = *reinterpret_cast<const float4*>(gamma + col);
        float4 bb = *reinterpret_cast<const float4*>(beta + col);
        r[0] = (r[0] - mean) * rstd * g.x + bb.x;
        r[1] = (r[1] - mean) * rstd * g.y + bb.y;
        r[2] = (r[2] - mean) * rstd * g.z + bb.z;
        r[3] = (r[3] - mean) * rstd * g.w + bb.w;
      }
      __half2 h0 = __floats2half2_rn(r[0], r[1]), h1 = __floats2half2_rn(r[2], r[3]);
      *reinterpret_cast<uint2*>(o + col) = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
      if (split_off > 0 && f8) {
        // fp8 correction operands (tc_api.cuh): e4m3(remainder * 2^12) | e4m3(value * 2^-3), D bytes each behind the hi block
        float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        uint8_t* ob = reinterpret_cast<uint8_t*>(o + split_off) + col;
        *reinterpret_cast<uint32_t*>(ob) = tc::cvt_e4m3x4((r[0] - f0.x) * F8_LO_SCALE, (r[1] - f0.y) * F8_LO_SCALE,
                                                          (r[2] - f1.x) * F8_LO_SCALE, (r[3] - f1.y) * F8_LO_SCALE);
        *reinterpret_cast<uint32_t*>(ob + split_off) =
            tc::cvt_e4m3x4(r[0] * F8_HI_SCALE, r[1] * F8_HI_SCALE, r[2] * F8_HI_SCALE, r[3] * F8_HI_SCALE);
      } else if (split_off > 0) {
        float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        __half2 l0 = __floats2half2_rn(r[0] - f0.x, r[1] - f0.y), l1 = __floats2half2_rn(r[2] - f1.x, r[3] - f1.y);
        *reinterpret_cast<uint2*>(o + split_off + col) =
            make_uint2(*reinterpret_cast<uint32_t*>(&l0), *reinterpret_cast<uint32_t*>(&l1));
      }
    }
  }
}
int ln_rows(Ctx* c, cudaStream_t st, const float* x, int ldx, const int* src, const float* gamma, const float* beta, float eps,
            __half* out, int ldo, int split_off, int Mout, int D, int normalize, int f8) {
  SAMPT_CHECK(D % 128 == 0 && D <= 1536, "ln_rows: D=%d must be a multiple of 128 and <= 1536", D);
  SAMPT_CHECK(!f8 || split_off == D, "ln_rows: the fp8 layout puts the byte blocks right behind the D hi halves");
  ln_rows_kernel<<<cdiv(Mout, 8), 256, 0, st>>>(x, ldx, src, gamma, beta, eps, out, ldo, split_off, Mout, D, normalize, f8);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Attention operand preparation (see attn_tc.cu): from qkv [Mrows, 3*D] fp16 (row = wb*L + t) build
//   Qx [BH, L, DK], Kx [BH, L, DK], Vt [BH, HD, Lkp]     BH = nwb * nheads, L = S*S tokens, token t = ty*S + tx
// (V^T keys in [L, Lkp) are row padding that attn_tc never reads)
// One CTA per (chunk of TC tokens sharing rows of the grid, head, wb).  Register tiled 4x4 (t, j) dot products.
// ---------------------------------------------------------------------------------------------------------------------
template <int HD>
__global__ void __launch_bounds__(256)
attn_prep_kernel(const __half* __restrict__ qkv, int ldq, const float* __restrict__ relh, const float* __restrict__ relw,
                 __half* __restrict__ Qx, __half* __restrict__ Kx, __half* __restrict__ Vt, int S, int L, int Lkp, int DK,
                 int D, int nheads, float scale, int TC) {
  // shared memory: q (half, padded rows), v (half, padded rows), one rel-pos table (fp32), extended Q columns (half)
  constexpr int QP = HD + 8;  // row pitch in halves (16 B aligned, breaks the 160 B bank pattern)
  extern __shared__ __align__(16) unsigned char smraw[];
  const int EXT = DK - HD;
  __half* sq = reinterpret_cast<__half*>(smraw);              // [TC][QP]
  __half* sv = sq + (size_t)TC * QP;                          // [TC][QP]
  __half* qext = sv + (size_t)TC * QP;                        // [TC][EXT]
  float* sr = reinterpret_cast<float*>(qext + (size_t)TC * EXT);  // [2S-1][HD+2]
  const int chunk = blockIdx.x, h = blockIdx.y, wb = blockIdx.z;
  const int t0 = chunk * TC;
  const int nt = min(TC, L - t0);
  const int tid = threadIdx.x;
  const size_t bh = (size_t)wb * nheads + h;
  constexpr int SEG = HD / 8;  // 16-byte segments per head row
  // ---- phase 1: coalesced 16 B loads of q / k / v head rows; K' (dot part) and scaled Q' are written straight back
  for (int i = tid; i < TC * SEG; i += 256) {
    const int t = i / SEG, sgm = i % SEG;
    uint4 qv = make_uint4(0u, 0u, 0u, 0u), vv = make_uint4(0u, 0u, 0u, 0u);
    if (t < nt) {
      const __half* rowp = qkv + (size_t)(wb * L + t0 + t) * ldq + h * HD + sgm * 8;
      qv = *reinterpret_cast<const uint4*>(rowp);
      const uint4 kv = *reinterpret_cast<const uint4*>(rowp + D);
      vv = *reinterpret_cast<const uint4*>(rowp + 2 * D);
      *reinterpret_cast<uint4*>(Kx + (bh * L + t0 + t) * DK + sgm * 8) = kv;
      __half2* q2 = reinterpret_cast<__half2*>(&qv);
      uint4 qs;
      __half2* o2 = reinterpret_cast<__half2*>(&qs);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = __half22float2(q2[j]);
        o2[j] = __floats2half2_rn(f.x * scale, f.y * scale);
      }
      *reinterpret_cast<uint4*>(Qx + (bh * L + t0 + t) * DK + sgm * 8) = qs;
    }
    *reinterpret_cast<uint4*>(sq + (size_t)t * QP + sgm * 8) = qv;
    *reinterpret_cast<uint4*>(sv + (size_t)t * QP + sgm * 8) = vv;
  }
  // K' extended columns: one-hots of (ky, kx) + zero padding, 16 B at a time
  for (int i = tid; i < TC * (EXT / 8); i += 256) {
    const int t = i / (EXT / 8), e0 = (i % (EXT / 8)) * 8;
    if (t < nt) {
      const int tt = t0 + t, ty = tt / S, tx = tt % S;
      __half hv[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int e = e0 + j;
        hv[j] = __float2half_rn((e == ty || e == S + tx) ? 1.f : 0.f);
      }
      *reinterpret_cast<uint4*>(Kx + (bh * L + tt) * DK + HD + e0) = *reinterpret_cast<uint4*>(hv);
    }
  }
  // zero the unused tail of the extended Q columns
  for (int i = tid; i < TC * (EXT - 2 * S); i += 256) {
    const int t = i / (EXT - 2 * S), e = 2 * S + i % (EXT - 2 * S);
    qext[(size_t)t * EXT + e] = __float2half_rn(0.f);
  }
  __syncthreads();
  // V^T: thread = (d, group of 8 consecutive tokens) -> one 16 B store
  {
    const int ngrp = (TC + 7) / 8;
    for (int i = tid; i < HD * ngrp; i += 256) {
      const int g = i / HD, d = i % HD;  // consecutive threads -> consecutive d: conflict-free shared-memory reads
      __half hv[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int t = g * 8 + j;
        hv[j] = (t < nt) ? sv[(size_t)t * QP + d] : __float2half_rn(0.f);
      }
      if (t0 + g * 8 < Lkp) *reinterpret_cast<uint4*>(Vt + (bh * HD + d) * Lkp + t0 + g * 8) = *reinterpret_cast<uint4*>(hv);
    }
  }
  // ---- phase 2: rel_h(q, j) = q . Rh[ty - j + S-1] ; rel_w(q, j) = q . Rw[tx - j + S-1]
  // work item = 2 horizontally adjacent tokens x JT offsets j.  Both tokens share the grid row, so for rel_h they need the
  // SAME JT table rows, and for rel_w rows shifted by one (JT+1 distinct rows): ~10 shared-memory loads per 56 FMAs.
  const int JT = (S % 8 == 0) ? 8 : 7;
  const int njt = (S + JT - 1) / JT;
  const int npair = TC / 2;
  constexpr int RP = HD + 2;  // table row pitch (even: float2 loads)
  for (int pass = 0; pass < 2; ++pass) {
    const float* R = pass == 0 ? relh : relw;
    __syncthreads();
    for (int i = tid; i < (2 * S - 1) * HD; i += 256) sr[(i / HD) * RP + (i % HD)] = R[i];
    __syncthreads();
    for (int item = tid; item < npair * njt; item += 256) {
      const int pr = item / njt, jb = (item % njt) * JT;
      const int tl = 2 * pr;                       // local token index of the pair's first token
      if (tl >= nt) continue;
      const int tt = t0 + tl;
      const int ty = tt / S, tx0 = tt % S;         // S is even -> tl+1 lies in the same grid row
      float acc0[8], acc1[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) { acc0[e] = 0.f; acc1[e] = 0.f; }
      // table row of slot e:  pass 0: ty - (jb+e) + S-1 ;  pass 1: (tx0+1) - (jb+e) + S-1   (slot e serves token1 @ j=jb+e
      // and token0 @ j=jb+e-1)
      int rrow[9];
#pragma unroll
      for (int e = 0; e < 9; ++e) {
        int idx = (pass == 0 ? ty : tx0 + 1) - (jb + e) + S - 1;
        rrow[e] = min(max(idx, 0), 2 * S - 2) * RP;
      }
      const __half* q0 = sq + (size_t)tl * QP;
      const __half* q1 = q0 + QP;
      for (int d = 0; d < HD; d += 2) {
        const float2 a0 = __half22float2(*reinterpret_cast<const __half2*>(q0 + d));
        const float2 a1 = __half22float2(*reinterpret_cast<const __half2*>(q1 + d));
        float2 rr[9];
#pragma unroll
        for (int e = 0; e < 9; ++e) rr[e] = *reinterpret_cast<const float2*>(sr + rrow[e] + d);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float2 r0 = (pass == 0) ? rr[e] : rr[e + 1];  // token0 at j = jb+e
          acc0[e] = fmaf(a0.x, r0.x, acc0[e]);
          acc0[e] = fmaf(a0.y, r0.y, acc0[e]);
          acc1[e] = fmaf(a1.x, rr[e].x, acc1[e]);
          acc1[e] = fmaf(a1.y, rr[e].y, acc1[e]);
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int j = jb + e;
        if (e < JT && j < S) {
          qext[(size_t)tl * EXT + pass * S + j] = __float2half_rn(acc0[e]);
          qext[(size_t)(tl + 1) * EXT + pass * S + j] = __float2half_rn(acc1[e]);
        }
      }
    }
  }
  __syncthreads();
  // extended Q columns -> global, 16 B at a time
  for (int i = tid; i < TC * (EXT / 8); i += 256) {
    const int t = i / (EXT / 8), e0 = (i % (EXT / 8)) * 8;
    if (t < nt) *reinterpret_cast<uint4*>(Qx + (bh * L + t0 + t) * DK + HD + e0) = *reinterpret_cast<const uint4*>(qext + (size_t)t * EXT + e0);
  }
}
int attn_prep(Ctx* c, cudaStream_t st, const __half* qkv, int ldq, const float* relh, const float* relw, __half* Qx, __half* Kx,
              __half* Vt, int nwb, int nheads, int S, int Lkp, int DK, int D, int HD, float scale) {
  {   // round-2 kernel (attn_prep2.cu: rel-pos products on the tensor cores); falls through for shapes it does not cover
    const int rc = attn_prep2(c, st, qkv, ldq, relh, relw, Qx, Kx, Vt, nwb, nheads, S, Lkp, DK, D, HD, scale);
    if (rc <= 0) return rc;
  }
  const int L = S * S;
  const int TC = (S == 14) ? 200 : 64;  // one whole 14x14 window (padded to a multiple of 8) or one row of the 64x64 grid
  SAMPT_CHECK(HD == 80 || HD == 64, "attn_prep: head_dim %d not built (80 = ViT-H, 64 = ViT-B/L/test)", HD);
  SAMPT_CHECK(DK >= HD + 2 * S && (DK - HD) % 8 == 0 && Lkp % 8 == 0 && Lkp >= L, "attn_prep: unsupported sizes (S=%d DK=%d Lkp=%d)", S, DK, Lkp);
  SAMPT_CHECK(D % 8 == 0 && ldq % 8 == 0, "attn_prep: D and ldq must be multiples of 8");
  dim3 grid(cdiv(L, TC), nheads, nwb);
  const int EXT = DK - HD;
  size_t smem = (size_t)TC * (HD + 8) * 2 * 2 + (size_t)TC * EXT * 2 + (size_t)(2 * S - 1) * (HD + 2) * sizeof(float);
  if (HD == 80) {
    SAMPT_TRY(ensure_func_smem(c, "attn_prep_kernel<80>", attn_prep_kernel<80>, 160 * 1024));
    attn_prep_kernel<80><<<grid, 256, smem, st>>>(qkv, ldq, relh, relw, Qx, Kx, Vt, S, L, Lkp, DK, D, nheads, scale, TC);
  } else {
    SAMPT_TRY(ensure_func_smem(c, "attn_prep_kernel<64>", attn_prep_kernel<64>, 160 * 1024));
    attn_prep_kernel<64><<<grid, 256, smem, st>>>(qkv, ldq, relh, relw, Qx, Kx, Vt, S, L, Lkp, DK, D, nheads, scale, TC);
  }
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// neck: im2col for the 3x3 conv (pad 1) over the 64x64 token grid, from fp32 LayerNorm2d'ed tokens.
//   A[b*G*G + y*G + x][(ky*3+kx)*C + c] = LN(y1[b, y+ky-1, x+kx-1, :])[c]    (0 outside)
// fused: LayerNorm2d (over channels, eps 1e-6) is applied on the fly per source token (one warp per (token, tap)).
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
neck_ln_im2col_kernel(const float* __restrict__ y1, const float* __restrict__ gamma, const float* __restrict__ beta,
                      __half* __restrict__ A, int B, int G, int C, int ld, int split_off, float eps) {
  const long long wid = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const long long total = (long long)B * G * G * 9;
  if (wid >= total) return;
  const int tap = (int)(wid % 9);
  const long long tok = wid / 9;
  const int x = (int)(tok % G), y = (int)((tok / G) % G), b = (int)(tok / ((long long)G * G));
  const int sy = y + tap / 3 - 1, sx = x + tap % 3 - 1;
  __half* o = A + (size_t)tok * ld + tap * C;
  const int per = C / 32;  // 8 for C = 256
  if (sy < 0 || sy >= G || sx < 0 || sx >= G) {
    for (int i = 0; i < per; ++i) {
      o[lane * per + i] = __float2half_rn(0.f);
      if (split_off > 0) o[split_off + lane * per + i] = __float2half_rn(0.f);
    }
    return;
  }
  const float* src = y1 + (((size_t)b * G + sy) * G + sx) * C + lane * per;
  float v[8];
  float s = 0.f;
  for (int i = 0; i < per; ++i) { v[i] = src[i]; s += v[i]; }
  float mean = warp_sum(s) / (float)C;
  float sq = 0.f;
  for (int i = 0; i < per; ++i) { float d = v[i] - mean; sq += d * d; }
  float rstd = 1.0f / sqrtf(warp_sum(sq) / (float)C + eps);
  for (int i = 0; i < per; ++i) {
    float r = (v[i] - mean) * rstd * gamma[lane * per + i] + beta[lane * per + i];
    __half hh = __float2half_rn(r);
    o[lane * per + i] = hh;
    if (split_off > 0) o[split_off + lane * per + i] = __float2half_rn(r - __half2float(hh));
  }
}
int neck_ln_im2col(Ctx* c, cudaStream_t st, const float* y1, const float* gamma, const float* beta, __half* A, int B, int G, int C,
                   int ld, int split_off) {
  SAMPT_CHECK(C == 256, "neck_ln_im2col: out_chans must be 256");
  long long total = (long long)B * G * G * 9;
  neck_ln_im2col_kernel<<<cdiv(total, 8), 256, 0, st>>>(y1, gamma, beta, A, B, G, C, ld, split_off, 1e-6f);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// final LayerNorm2d of the neck + transpose to NCHW: in [B*G*G, C] fp32 -> out [B, C, G, G] fp32 (SamPredictor.features)
__global__ void __launch_bounds__(256)
neck_ln_nchw_kernel(const float* __restrict__ y2, const float* __restrict__ gamma, const float* __restrict__ beta,
                    float* __restrict__ out, int B, int GG, int C, float eps) {
  // block = 32 tokens x all channels, transposed through shared memory for coalesced NCHW stores
  __shared__ float tile[32][257];
  const int tok0 = blockIdx.x * 32;
  const int b = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int tt = warp; tt < 32; tt += 8) {
    int tok = tok0 + tt;
    const float* src = y2 + ((size_t)b * GG + tok) * C;
    float v[8];
    float s = 0.f;
    for (int i = 0; i < 8; ++i) { v[i] = src[lane + 32 * i]; s += v[i]; }
    float mean = warp_sum(s) / (float)C;
    float sq = 0.f;
    for (int i = 0; i < 8; ++i) { float d = v[i] - mean; sq += d * d; }
    float rstd = 1.0f / sqrtf(warp_sum(sq) / (float)C + eps);
    for (int i = 0; i < 8; ++i) {
      int ch = lane + 32 * i;
      tile[tt][ch] = (v[i] - mean) * rstd * gamma[ch] + beta[ch];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 32 * C; i += 256) {
    int ch = i / 32, tt = i % 32;
    out[((size_t)b * C + ch) * GG + tok0 + tt] = tile[tt][ch];
  }
}
int neck_ln_nchw(Ctx* c, cudaStream_t st, const float* y2, const float* gamma, const float* beta, float* out, int B, int GG, int C) {
  SAMPT_CHECK(C == 256 && GG % 32 == 0, "neck_ln_nchw: C must be 256 and G*G a multiple of 32");
  dim3 grid(GG / 32, B);
  neck_ln_nchw_kernel<<<grid, 256, 0, st>>>(y2, gamma, beta, out, B, GG, C, 1e-6f);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

}  // namespace sampt
