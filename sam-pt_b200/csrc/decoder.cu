// SAM prompt encoder + mask decoder (two-way transformer) + postprocess + on-device refinement control, strict fp32.
// Upstream: segment_anything/modeling/{prompt_encoder,mask_decoder,transformer,sam}.py (un-vendored; SURVEY Appendix B.2);
// reference call sites sam_pt/modeling/sam_pt.py:783-828 (predict_torch x (1|2 + <=12 refinements) per frame and mask).
//
// Every kernel takes a `skip` flag pointer: once the refinement loop's break condition (mask area < 2 px, sam_pt.py:812)
// has fired on the device, the remaining iterations' kernels return immediately, so the whole 13-call chain of a frame is
// enqueued without a single host synchronisation (the reference does ~6 syncs per iteration, SURVEY §0.6).
#include <cstdlib>

#include "common.cuh"
#include "kernels.cuh"
#include "tc_api.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {

#define SKIP_RETURN(skip) \
  if ((skip) != nullptr && *(skip) != 0) return;

// ------------------------------------------------------------------------------------------------------------------
// prompt encoder, sparse part: tokens = [iou_token, mask_tokens(4) [, hq_token], points..., pad | box corners]
// one block (256 threads = embedding channels) per prompt token
// ------------------------------------------------------------------------------------------------------------------
struct PromptArgs {
  const float* coords;    // [K,2] in the 1024 input frame
  const int* labels;      // [K]
  int K;
  const float* box;       // [4] or null (device)
  int use_box;            // 1: box corners appended (and no pad point), 0: pad point appended
  const float* gauss;     // [2,128]
  const float* pt_emb[4]; // point_embeddings.{0..3}.weight [256]
  const float* not_a_point;
  const float* out_tokens; // [n_out_tok,256] iou_token ++ mask_tokens (++ hq token)
  int n_out_tok;
  float img_size;
};

__global__ void __launch_bounds__(256)
prompt_tokens_kernel(PromptArgs a, float* __restrict__ tokens, const int* skip) {
  SKIP_RETURN(skip);
  const int t = blockIdx.x, ch = threadIdx.x;
  float* out = tokens + (size_t)t * 256;
  if (t < a.n_out_tok) { out[ch] = a.out_tokens[(size_t)t * 256 + ch]; return; }
  const int i = t - a.n_out_tok;
  float x, y;
  int label;                       // -1: not a point (user label -1 or the pad point)
  const float* emb = nullptr;      // learned embedding added to the PE: point_embeddings[0|1] for user labels 0 / 1, [2|3] for
                                   // the box corners; any other user label gets the PE alone (upstream PromptEncoder._embed_points)
  if (i < a.K) {
    x = a.coords[2 * i]; y = a.coords[2 * i + 1]; label = a.labels[i];
    if (label == 0 || label == 1) emb = a.pt_emb[label];
  } else if (!a.use_box) { x = 0.f; y = 0.f; label = -1; }
  else { int cidx = i - a.K; x = a.box[2 * cidx]; y = a.box[2 * cidx + 1]; label = 2 + cidx; emb = a.pt_emb[2 + cidx]; }
  // +0.5 (pixel centre), normalise to [0,1], 2c-1, @ G, * 2pi, [sin | cos]
  x = (x + 0.5f) / a.img_size; y = (y + 0.5f) / a.img_size;
  float cx = 2.f * x - 1.f, cy = 2.f * y - 1.f;
  const int k = ch & 127;
  float v = cx * a.gauss[k] + cy * a.gauss[128 + k];
  v = 2.0f * 3.14159265358979323846f * v;
  float pe = (ch < 128) ? sinf(v) : cosf(v);
  if (label == -1) pe = a.not_a_point[ch];
  else if (emb != nullptr) pe += emb[ch];
  out[ch] = pe;
}

// ------------------------------------------------------------------------------------------------------------------
// prompt encoder, dense part fused with `src = image_embedding + dense`:
//   mask_input == null : src[tok] = feat[tok] + no_mask_embed
//   else               : src[tok] = feat[tok] + conv1x1(GELU(LN(conv2x2s2(GELU(LN(conv2x2s2(mask)))))))
// feat is token-major [4096,256]; one warp per token
// ------------------------------------------------------------------------------------------------------------------
struct DenseW {
  const float *w0, *b0, *ln1w, *ln1b, *w3, *b3, *ln4w, *ln4b, *w6, *b6, *no_mask;
};
__global__ void __launch_bounds__(256)
dense_src_kernel(const float* __restrict__ feat, const float* __restrict__ mask_in, DenseW w, float* __restrict__ src, int G,
                 const int* skip) {
  SKIP_RETURN(skip);
  const int tok = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (tok >= G * G) return;
  const float* f = feat + (size_t)tok * 256;
  float* o = src + (size_t)tok * 256;
  if (mask_in == nullptr) {
    for (int c = lane; c < 256; c += 32) o[c] = f[c] + w.no_mask[c];
    return;
  }
  const int ty = tok / G, tx = tok % G;
  const int MW = 4 * G;  // 256
  // stage 1: 2x2 positions, 4 channels each (every lane computes everything: 64 MACs)
  float h1[4][4];
#pragma unroll
  for (int py = 0; py < 2; ++py)
#pragma unroll
    for (int px = 0; px < 2; ++px) {
      float v[4];
#pragma unroll
      for (int co = 0; co < 4; ++co) v[co] = w.b0[co];
#pragma unroll
      for (int ky = 0; ky < 2; ++ky)
#pragma unroll
        for (int kx = 0; kx < 2; ++kx) {
          float m = mask_in[(size_t)(ty * 4 + py * 2 + ky) * MW + tx * 4 + px * 2 + kx];
#pragma unroll
          for (int co = 0; co < 4; ++co) v[co] = fmaf(m, w.w0[co * 4 + ky * 2 + kx], v[co]);
        }
      float mean = 0.25f * (v[0] + v[1] + v[2] + v[3]);
      float var = 0.f;
#pragma unroll
      for (int co = 0; co < 4; ++co) { float d = v[co] - mean; var += d * d; }
      var *= 0.25f;
      float rstd = 1.0f / sqrtf(var + 1e-6f);
#pragma unroll
      for (int co = 0; co < 4; ++co) h1[py * 2 + px][co] = gelu_erf(w.ln1w[co] * ((v[co] - mean) * rstd) + w.ln1b[co]);
    }
  // stage 2: conv 2x2 s2 (4 -> 16) over the 2x2 positions, LN over 16, GELU
  float h2[16];
  float mean = 0.f;
#pragma unroll
  for (int co = 0; co < 16; ++co) {
    float v = w.b3[co];
#pragma unroll
    for (int ci = 0; ci < 4; ++ci)
#pragma unroll
      for (int p = 0; p < 4; ++p) v = fmaf(h1[p][ci], w.w3[(co * 4 + ci) * 4 + p], v);
    h2[co] = v;
    mean += v;
  }
  mean *= (1.0f / 16.0f);
  float var = 0.f;
#pragma unroll
  for (int co = 0; co < 16; ++co) { float d = h2[co] - mean; var += d * d; }
  var *= (1.0f / 16.0f);
  float rstd = 1.0f / sqrtf(var + 1e-6f);
#pragma unroll
  for (int co = 0; co < 16; ++co) h2[co] = gelu_erf(w.ln4w[co] * ((h2[co] - mean) * rstd) + w.ln4b[co]);
  // stage 3: 1x1 conv 16 -> 256, + image embedding
  for (int c = lane; c < 256; c += 32) {
    float v = w.b6[c];
#pragma unroll
    for (int ci = 0; ci < 16; ++ci) v = fmaf(h2[ci], w.w6[c * 16 + ci], v);
    o[c] = f[c] + v;
  }
}

// NCHW (256, G*G) -> token-major (G*G, 256)
__global__ void nchw_to_tok_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int GG) {
  __shared__ float tile[32][33];
  int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32x8
  for (int j = ty; j < 32; j += 8) tile[j][tx] = in[(size_t)(c0 + j) * GG + t0 + tx];
  __syncthreads();
  for (int j = ty; j < 32; j += 8) out[(size_t)(t0 + j) * C + c0 + tx] = tile[tx][j];
}

// ------------------------------------------------------------------------------------------------------------------
// row-wise helpers on small token matrices
// ------------------------------------------------------------------------------------------------------------------
// y = a + b (elementwise), n4 float4
__global__ void add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ y, long long n4,
                           const int* skip) {
  SKIP_RETURN(skip);
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 u = reinterpret_cast<const float4*>(a)[i], v = reinterpret_cast<const float4*>(b)[i];
  reinterpret_cast<float4*>(y)[i] = make_float4(u.x + v.x, u.y + v.y, u.z + v.z, u.w + v.w);
}
// LayerNorm over 256 channels, one warp per row: y = LN(x (+ add)) ; eps 1e-5 (nn.LayerNorm default in the transformer)
__global__ void __launch_bounds__(256)
ln256_kernel(const float* __restrict__ x, const float* __restrict__ add, const float* __restrict__ g, const float* __restrict__ b,
             float* __restrict__ y, int M, float eps, const int* skip) {
  SKIP_RETURN(skip);
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  float v[8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i] = x[(size_t)row * 256 + lane + 32 * i];
    if (add) v[i] += add[(size_t)row * 256 + lane + 32 * i];
    s += v[i];
  }
  float mean = warp_sum(s) * (1.0f / 256.0f);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { float d = v[i] - mean; sq += d * d; }
  float rstd = 1.0f / sqrtf(warp_sum(sq) * (1.0f / 256.0f) + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = lane + 32 * i;
    y[(size_t)row * 256 + c] = (v[i] - mean) * rstd * g[c] + b[c];
  }
}

// ------------------------------------------------------------------------------------------------------------------
// attention cores (projections are done with sgemm_nt)
// ------------------------------------------------------------------------------------------------------------------
// tokens attend: q [T, H*dh], k/v [Nk, H*dh]; out [T, H*dh].  One block per (token, head); Nk up to 4096 (+ small T case).
template <int DH>
__global__ void __launch_bounds__(256)
attn_q_small_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, float* __restrict__ out,
                    int Nk, int H, const int* skip) {
  SKIP_RETURN(skip);
  const int t = blockIdx.x, h = blockIdx.y;
  const int ld = H * DH;
  __shared__ float sq[DH];
  __shared__ float red[32];
  __shared__ float sacc[8][DH];
  if (threadIdx.x < DH) sq[threadIdx.x] = q[(size_t)t * ld + h * DH + threadIdx.x];
  __syncthreads();
  const float scale = 1.0f / sqrtf((float)DH);
  // pass 1: max
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < Nk; j += 256) {
    const float* kp = k + (size_t)j * ld + h * DH;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < DH; ++d) s = fmaf(sq[d], kp[d], s);
    mx = fmaxf(mx, s * scale);
  }
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x < 32) {
    float m = threadIdx.x < 8 ? red[threadIdx.x] : -INFINITY;
    m = warp_max(m);
    if (threadIdx.x == 0) red[0] = m;
  }
  __syncthreads();
  mx = red[0];
  __syncthreads();
  // pass 2: exp, sum, weighted V
  float acc[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = 0.f;
  float lsum = 0.f;
  for (int j = threadIdx.x; j < Nk; j += 256) {
    const float* kp = k + (size_t)j * ld + h * DH;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < DH; ++d) s = fmaf(sq[d], kp[d], s);
    float p = expf(s * scale - mx);
    lsum += p;
    const float* vp = v + (size_t)j * ld + h * DH;
#pragma unroll
    for (int d = 0; d < DH; ++d) acc[d] = fmaf(p, vp[d], acc[d]);
  }
  lsum = block_sum(lsum, red);
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = warp_sum(acc[d]);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int d = 0; d < DH; ++d) sacc[threadIdx.x >> 5][d] = acc[d];
  }
  __syncthreads();
  if (threadIdx.x < DH) {
    float a = 0.f;
    for (int w = 0; w < 8; ++w) a += sacc[w][threadIdx.x];
    out[(size_t)t * ld + h * DH + threadIdx.x] = a / lsum;
  }
}

// Self-attention among the prompt / output tokens, any T (8 ... 263 tokens: BASELINE configs[4] carries 256 query points).
// grid (ceil(T / 32) query tiles, H heads); the head's K and V (T x DH, padded rows) sit in shared memory; ONE WARP PER QUERY:
// lanes stride over the keys for the scores (q from registers via shuffle-free broadcast reads), warp max / sum, probabilities to
// shared memory, then lane d accumulates output channel d.  Replaces the block-per-(token, head) kernel above for T > 16, whose
// 256-thread reductions of 32 accumulators cost 170 us per call at T = 263.
template <int DH>
__global__ void __launch_bounds__(256)
attn_tok_self_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, float* __restrict__ out,
                     int T, int H, const int* skip) {
  SKIP_RETURN(skip);
  static_assert(DH == 32, "one lane per output channel");
  extern __shared__ float sm_ts[];
  const int KP = DH + 1;
  float* sk = sm_ts;                        // [T][DH + 1]
  float* sv = sk + (size_t)T * KP;          // [T][DH + 1]
  float* sp = sv + (size_t)T * KP;          // [8 warps][T] probabilities
  float* sq = sp + (size_t)8 * T;           // [8 warps][DH]
  const int h = blockIdx.y, ld = H * DH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < T * DH; i += 256) {
    const int t = i / DH, d = i % DH;
    sk[t * KP + d] = k[(size_t)t * ld + h * DH + d];
    sv[t * KP + d] = v[(size_t)t * ld + h * DH + d];
  }
  __syncthreads();
  const float scale = 1.0f / sqrtf((float)DH);
  float* pw = sp + (size_t)warp * T;
  float* qw = sq + warp * DH;
  for (int t = blockIdx.x * 32 + warp; t < min(T, blockIdx.x * 32 + 32); t += 8) {
    qw[lane] = q[(size_t)t * ld + h * DH + lane] * scale;
    __syncwarp();
    float mx = -INFINITY;
    for (int j = lane; j < T; j += 32) {
      const float* kp = sk + j * KP;
      float sdot = 0.f;
#pragma unroll
      for (int d = 0; d < DH; ++d) sdot = fmaf(qw[d], kp[d], sdot);
      pw[j] = sdot;
      mx = fmaxf(mx, sdot);
    }
    mx = warp_max(mx);
    float lsum = 0.f;
    for (int j = lane; j < T; j += 32) {
      const float pj = expf(pw[j] - mx);
      pw[j] = pj;
      lsum += pj;
    }
    lsum = warp_sum(lsum);
    __syncwarp();
    float acc = 0.f;
    for (int j = 0; j < T; ++j) acc = fmaf(pw[j], sv[j * KP + lane], acc);
    out[(size_t)t * ld + h * DH + lane] = acc / lsum;
    __syncwarp();   // pw / qw are rewritten by the next query of this warp
  }
}

// tokens -> image attention, split over the keys (flash-decoding style): grid (S splits, H heads).  Each block stages its
// slice of K/V (keys_per_split x DH, read exactly once, coalesced) in shared memory; warp w serves tokens w, w+8, ...;
// lanes stride over the slice's keys.  Partial (max, sum, acc[DH]) per (token, head, split) -> combine kernel.
template <int DH, int KPS>
__global__ void __launch_bounds__(256)
attn_t2i_partial_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                        float* __restrict__ part, int T, int Nk, int H, const int* skip) {
  SKIP_RETURN(skip);
  __shared__ float sk[KPS][DH + 1];
  __shared__ float sv[KPS][DH + 1];
  const int split = blockIdx.x, h = blockIdx.y, nsplit = gridDim.x;
  const int ld = H * DH;
  const int j0 = split * KPS;
  for (int i = threadIdx.x; i < KPS * DH; i += 256) {
    int j = i / DH, d = i % DH;
    float kv = 0.f, vv = 0.f;
    if (j0 + j < Nk) { kv = k[(size_t)(j0 + j) * ld + h * DH + d]; vv = v[(size_t)(j0 + j) * ld + h * DH + d]; }
    sk[j][d] = kv; sv[j][d] = vv;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float scale = 1.0f / sqrtf((float)DH);
  const int nvalid = min(KPS, Nk - j0);
  for (int t = warp; t < T; t += 8) {
    float qv[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) qv[d] = q[(size_t)t * ld + h * DH + d];
    float sc[KPS / 32];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < KPS / 32; ++i) {
      int j = lane + 32 * i;
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < DH; ++d) s = fmaf(qv[d], sk[j][d], s);
      s *= scale;
      sc[i] = (j < nvalid) ? s : -INFINITY;
      mx = fmaxf(mx, sc[i]);
    }
    mx = warp_max(mx);
    float acc[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) acc[d] = 0.f;
    float lsum = 0.f;
#pragma unroll
    for (int i = 0; i < KPS / 32; ++i) {
      int j = lane + 32 * i;
      float p = (j < nvalid) ? expf(sc[i] - mx) : 0.f;
      lsum += p;
#pragma unroll
      for (int d = 0; d < DH; ++d) acc[d] = fmaf(p, sv[j][d], acc[d]);
    }
    lsum = warp_sum(lsum);
#pragma unroll
    for (int d = 0; d < DH; ++d) acc[d] = warp_sum(acc[d]);
    if (lane == 0) {
      float* o = part + (((size_t)t * H + h) * nsplit + split) * (DH + 2);
      o[0] = mx; o[1] = lsum;
#pragma unroll
      for (int d = 0; d < DH; ++d) o[2 + d] = acc[d];
    }
  }
}
template <int DH>
__global__ void attn_t2i_combine_kernel(const float* __restrict__ part, float* __restrict__ out, int T, int H, int nsplit,
                                        const int* skip) {
  SKIP_RETURN(skip);
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // (t, h, d)
  if (idx >= T * H * DH) return;
  const int d = idx % DH, h = (idx / DH) % H, t = idx / (DH * H);
  const float* p = part + ((size_t)t * H + h) * nsplit * (DH + 2);
  float mx = -INFINITY;
  for (int s = 0; s < nsplit; ++s) mx = fmaxf(mx, p[s * (DH + 2)]);
  float l = 0.f, a = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    float w = expf(p[s * (DH + 2)] - mx);
    l += w * p[s * (DH + 2) + 1];
    a += w * p[s * (DH + 2) + 2 + d];
  }
  out[(size_t)t * H * DH + h * DH + d] = a / l;
}

// image tokens attend to the prompt tokens: q [N, H*DH], k/v [T, H*DH].  One thread per (image token, head); a WARP holds 32 image
// tokens of ONE head, so every k / v row it needs is the same for all lanes: the rows are read from shared memory as warp-uniform
// 16-byte broadcasts (8 loads per token instead of 32 scalar ones -- the kernel was bound by shared-memory instruction issue).
// k/v pass through shared memory in chunks of 32 tokens (32 KB: several CTAs per SM whatever T is -- BASELINE configs[4] has 256
// query points = 263 tokens); ONE pass with an online softmax (running max / sum / weighted sum rescaled when the max moves).
template <int DH>
__global__ void __launch_bounds__(256)
attn_kv_small_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, float* __restrict__ out,
                     int N, int T, int H, const int* skip) {
  SKIP_RETURN(skip);
  static_assert(DH % 4 == 0, "rows are read as float4");
  constexpr int TCH = 32, MAXH = 8;
  __shared__ __align__(16) float sk[TCH * MAXH * DH], sv[TCH * MAXH * DH];
  const int ld = H * DH;
  const int gw = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int h = gw % H, n = (gw / H) * 32 + lane;
  const bool live = n < N;
  const float scale = 1.0f / sqrtf((float)DH);
  float qv[DH];
#pragma unroll
  for (int d = 0; d < DH; d += 4) {
    const float4 t = live ? *reinterpret_cast<const float4*>(q + (size_t)n * ld + h * DH + d) : make_float4(0.f, 0.f, 0.f, 0.f);
    qv[d] = t.x; qv[d + 1] = t.y; qv[d + 2] = t.z; qv[d + 3] = t.w;
  }
  float acc[DH];
#pragma unroll
  for (int d = 0; d < DH; ++d) acc[d] = 0.f;
  float mx = -INFINITY, lsum = 0.f;
  for (int t0 = 0; t0 < T; t0 += TCH) {
    const int nt = min(TCH, T - t0);
    __syncthreads();
    for (int i = threadIdx.x; i < nt * ld / 4; i += 256) {
      reinterpret_cast<float4*>(sk)[i] = reinterpret_cast<const float4*>(k + (size_t)t0 * ld)[i];
      reinterpret_cast<float4*>(sv)[i] = reinterpret_cast<const float4*>(v + (size_t)t0 * ld)[i];
    }
    __syncthreads();
    for (int t = 0; t < nt; ++t) {
      const float4* kp = reinterpret_cast<const float4*>(sk + t * ld + h * DH);
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < DH / 4; ++d) {
        const float4 kk = kp[d];
        s = fmaf(qv[4 * d], kk.x, s); s = fmaf(qv[4 * d + 1], kk.y, s); s = fmaf(qv[4 * d + 2], kk.z, s); s = fmaf(qv[4 * d + 3], kk.w, s);
      }
      s *= scale;
      const float mn = fmaxf(mx, s);
      const float corr = expf(mx - mn), p = expf(s - mn);   // first token: exp(-inf) = 0 rescales the (zero) state
      mx = mn;
      lsum = fmaf(lsum, corr, p);
      const float4* vp = reinterpret_cast<const float4*>(sv + t * ld + h * DH);
#pragma unroll
      for (int d = 0; d < DH / 4; ++d) {
        const float4 vv = vp[d];
        acc[4 * d] = fmaf(acc[4 * d], corr, p * vv.x); acc[4 * d + 1] = fmaf(acc[4 * d + 1], corr, p * vv.y);
        acc[4 * d + 2] = fmaf(acc[4 * d + 2], corr, p * vv.z); acc[4 * d + 3] = fmaf(acc[4 * d + 3], corr, p * vv.w);
      }
    }
  }
  if (!live) return;
  const float inv = 1.0f / lsum;
#pragma unroll
  for (int d = 0; d < DH; d += 4)
    *reinterpret_cast<float4*>(out + (size_t)n * ld + h * DH + d) = make_float4(acc[d] * inv, acc[d + 1] * inv, acc[d + 2] * inv, acc[d + 3] * inv);
}

// ------------------------------------------------------------------------------------------------------------------
// heads: 3-layer MLPs (ReLU) on single token rows: block b -> job b
// ------------------------------------------------------------------------------------------------------------------
struct Mlp3Job { const float* x; const float *w0, *b0, *w1, *b1, *w2, *b2; int n_out; float* y; };
struct Mlp3Jobs { Mlp3Job j[8]; };
__global__ void __launch_bounds__(256)
mlp3_kernel(Mlp3Jobs jobs, const int* skip) {
  SKIP_RETURN(skip);
  const Mlp3Job& J = jobs.j[blockIdx.x];
  __shared__ float a[256], b[256];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  a[t] = J.x[t];
  __syncthreads();
  // each warp produces outputs warp, warp+8, ...: the 256-long weight row is read coalesced (8 floats per lane)
  auto layer = [&](const float* __restrict__ w, const float* __restrict__ bias, const float* in, float* out, int nout, bool relu) {
    for (int o = warp; o < nout; o += 8) {
      const float* wr = w + (size_t)o * 256;
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s = fmaf(wr[lane + 32 * i], in[lane + 32 * i], s);
      s = warp_sum(s);
      if (lane == 0) { s += bias[o]; out[o] = relu ? fmaxf(s, 0.f) : s; }
    }
  };
  layer(J.w0, J.b0, a, b, 256, true);
  __syncthreads();
  layer(J.w1, J.b1, b, a, 256, true);
  __syncthreads();
  layer(J.w2, J.b2, a, J.y, J.n_out, false);
}

// ------------------------------------------------------------------------------------------------------------------
// output upscaling tail fused with the hyper-network dot product:
//   up1 = ConvT(256->64,k2,s2)(src) was produced by a GEMM as u1[tok][(dy*2+dx)*64 + c]  (128x128 pixels x 64 ch)
//   low_res[m][Y][X] = sum_c hyper[m][c] * GELU( ConvT(64->32,k2,s2)( GELU(LN2d(up1)) ) )[c][Y][X]
// one thread per low-res output pixel (256x256)
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
upscale_mask_kernel(const float* __restrict__ u1, const float* __restrict__ lnw, const float* __restrict__ lnb,
                    const float* __restrict__ w2 /*[64][32][2][2]*/, const float* __restrict__ b2, const float* __restrict__ hyper,
                    int n_masks, float* __restrict__ low_res, int G, float* __restrict__ u_out /*[R*R][32] or null*/, const int* skip) {
  SKIP_RETURN(skip);
  __shared__ float sw[64 * 32 * 4];
  __shared__ float sh[4 * 32];
  for (int i = threadIdx.x; i < 64 * 32 * 4; i += 256) sw[i] = w2[i];
  if (threadIdx.x < n_masks * 32) sh[threadIdx.x] = hyper[threadIdx.x];
  __syncthreads();
  const int R = 4 * G;  // 256
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= R * R) return;
  const int Y = pix / R, X = pix % R;
  const int y2 = Y >> 1, x2 = X >> 1, dy2 = Y & 1, dx2 = X & 1;        // position in the 128x128 map + sub-pixel
  const int ty = y2 >> 1, tx = x2 >> 1, dy1 = y2 & 1, dx1 = x2 & 1;    // token + sub-pixel of the first ConvT
  const float* p = u1 + ((size_t)(ty * G + tx)) * 256 + (dy1 * 2 + dx1) * 64;
  float v[64];
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < 64; c += 4) {
    float4 t = *reinterpret_cast<const float4*>(p + c);
    v[c] = t.x; v[c + 1] = t.y; v[c + 2] = t.z; v[c + 3] = t.w;
    s += t.x + t.y + t.z + t.w;
  }
  float mean = s * (1.0f / 64.0f);
  float sq = 0.f;
#pragma unroll
  for (int c = 0; c < 64; ++c) { float d = v[c] - mean; sq += d * d; }
  float rstd = 1.0f / sqrtf(sq * (1.0f / 64.0f) + 1e-6f);
#pragma unroll
  for (int c = 0; c < 64; ++c) v[c] = gelu_erf(lnw[c] * ((v[c] - mean) * rstd) + lnb[c]);
  float outm[4] = {0.f, 0.f, 0.f, 0.f};
  const int sub = dy2 * 2 + dx2;
  for (int co = 0; co < 32; ++co) {
    float a = b2[co];
#pragma unroll
    for (int ci = 0; ci < 64; ++ci) a = fmaf(v[ci], sw[(ci * 32 + co) * 4 + sub], a);
    a = gelu_erf(a);
    if (u_out) u_out[(size_t)pix * 32 + co] = a;
    for (int m = 0; m < n_masks; ++m) outm[m] = fmaf(sh[m * 32 + co], a, outm[m]);
  }
  for (int m = 0; m < n_masks; ++m) low_res[(size_t)m * R * R + pix] = outm[m];
}

// ------------------------------------------------------------------------------------------------------------------
// HQ-SAM (MaskDecoderHQ of m43/sam-hq, un-vendored; SURVEY Appendix B.2 last paragraph)
// ------------------------------------------------------------------------------------------------------------------
// hq_features = embedding_encoder(image_embeddings) + compress_vit_feat(interm[0]); both are ConvT(k2,s2) -> LN2d -> GELU ->
// ConvT(k2,s2) stacks: the first ConvT of each was produced by a GEMM as e1[tok][(dy*2+dx)*64 + c] / c1[tok][(dy*2+dx)*256 + c].
// one thread per low-res (256x256) pixel, 32 output channels.
__global__ void __launch_bounds__(256)
hq_features_kernel(const float* __restrict__ e1, const float* __restrict__ c1, const float* __restrict__ e_lnw,
                   const float* __restrict__ e_lnb, const float* __restrict__ e_w2 /*[64][32][2][2]*/, const float* __restrict__ e_b2,
                   const float* __restrict__ c_lnw, const float* __restrict__ c_lnb, const float* __restrict__ c_w2 /*[256][32][2][2]*/,
                   const float* __restrict__ c_b2, float* __restrict__ out /*[R*R][32]*/, int G) {
  const int R = 4 * G;
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= R * R) return;
  const int Y = pix / R, X = pix % R;
  const int y2 = Y >> 1, x2 = X >> 1, sub = (Y & 1) * 2 + (X & 1);
  const int ty = y2 >> 1, tx = x2 >> 1, sub1 = (y2 & 1) * 2 + (x2 & 1);
  float acc[32];
#pragma unroll
  for (int co = 0; co < 32; ++co) acc[co] = e_b2[co] + c_b2[co];
  {  // embedding_encoder branch (64 channels)
    const float* p = e1 + (size_t)(ty * G + tx) * 256 + sub1 * 64;
    float s = 0.f;
    for (int c = 0; c < 64; ++c) s += p[c];
    float mean = s * (1.0f / 64.0f), sq = 0.f;
    for (int c = 0; c < 64; ++c) { float d = p[c] - mean; sq += d * d; }
    float rstd = 1.0f / sqrtf(sq * (1.0f / 64.0f) + 1e-6f);
    for (int ci = 0; ci < 64; ++ci) {
      float v = gelu_erf(e_lnw[ci] * ((p[ci] - mean) * rstd) + e_lnb[ci]);
#pragma unroll
      for (int co = 0; co < 32; ++co) acc[co] = fmaf(v, __ldg(e_w2 + (ci * 32 + co) * 4 + sub), acc[co]);
    }
  }
  {  // compress_vit_feat branch (256 channels)
    const float* p = c1 + (size_t)(ty * G + tx) * 1024 + sub1 * 256;
    float s = 0.f;
    for (int c = 0; c < 256; ++c) s += p[c];
    float mean = s * (1.0f / 256.0f), sq = 0.f;
    for (int c = 0; c < 256; ++c) { float d = p[c] - mean; sq += d * d; }
    float rstd = 1.0f / sqrtf(sq * (1.0f / 256.0f) + 1e-6f);
    for (int ci = 0; ci < 256; ++ci) {
      float v = gelu_erf(c_lnw[ci] * ((p[ci] - mean) * rstd) + c_lnb[ci]);
#pragma unroll
      for (int co = 0; co < 32; ++co) acc[co] = fmaf(v, __ldg(c_w2 + (ci * 32 + co) * 4 + sub), acc[co]);
    }
  }
#pragma unroll
  for (int co = 0; co < 32; co += 4)
    *reinterpret_cast<float4*>(out + (size_t)pix * 32 + co) = make_float4(acc[co], acc[co + 1], acc[co + 2], acc[co + 3]);
}
// LayerNorm2d(64) + GELU in place on a channels-last [pixels][64] map, one warp per pixel
__global__ void __launch_bounds__(256)
ln64_gelu_kernel(float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ b, int npix, const int* skip) {
  SKIP_RETURN(skip);
  const int pix = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (pix >= npix) return;
  float* p = x + (size_t)pix * 64;
  float a = p[lane], c = p[lane + 32];
  float mean = warp_sum(a + c) * (1.0f / 64.0f);
  float da = a - mean, dc = c - mean;
  float rstd = 1.0f / sqrtf(warp_sum(da * da + dc * dc) * (1.0f / 64.0f) + 1e-6f);
  p[lane] = gelu_erf(g[lane] * (da * rstd) + b[lane]);
  p[lane + 32] = gelu_erf(g[lane + 32] * (dc * rstd) + b[lane + 32]);
}
// low_res[pix] += hyper_hq . (maskfeature[pix] + hq_features[pix])      (mask = mask_sam + mask_hq, hq_token_only=False)
__global__ void hq_mask_add_kernel(const float* __restrict__ mf, const float* __restrict__ hqf, const float* __restrict__ hyper_hq,
                                   float* __restrict__ low_res, int npix, const int* skip) {
  SKIP_RETURN(skip);
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= npix) return;
  float a = 0.f;
#pragma unroll
  for (int c = 0; c < 32; c += 4) {
    float4 u = *reinterpret_cast<const float4*>(mf + (size_t)pix * 32 + c);
    float4 v = *reinterpret_cast<const float4*>(hqf + (size_t)pix * 32 + c);
    a = fmaf(hyper_hq[c], u.x + v.x, a);
    a = fmaf(hyper_hq[c + 1], u.y + v.y, a);
    a = fmaf(hyper_hq[c + 2], u.z + v.z, a);
    a = fmaf(hyper_hq[c + 3], u.w + v.w, a);
  }
  low_res[pix] += a;
}

// ------------------------------------------------------------------------------------------------------------------
// Sam.postprocess_masks fused: bilinear (align_corners=False) 256^2 -> 1024^2, crop [:in_h,:in_w], bilinear -> (H,W);
// + bounding box / area of (logit > 0) for the refinement loop (sam_pt.py:811-820)
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void src_index(float scale, int dst, int in_size, int& i0, int& i1, float& l1) {
  float s = scale * ((float)dst + 0.5f) - 0.5f;
  if (s < 0.f) s = 0.f;
  i0 = (int)s;
  if (i0 > in_size - 1) i0 = in_size - 1;
  i1 = i0 + ((i0 < in_size - 1) ? 1 : 0);
  l1 = s - (float)i0;
}
__device__ __forceinline__ float up4_sample(const float* __restrict__ lr, int R, int S, int y, int x) {
  // value of the (virtual) S x S up-sampled map at integer (y, x)
  const float sc = (float)R / (float)S;
  int y0, y1, x0, x1; float ly, lx;
  src_index(sc, y, R, y0, y1, ly);
  src_index(sc, x, R, x0, x1, lx);
  float hy = 1.f - ly, hx = 1.f - lx;
  return hy * (hx * lr[y0 * R + x0] + lx * lr[y0 * R + x1]) + ly * (hx * lr[y1 * R + x0] + lx * lr[y1 * R + x1]);
}
__global__ void __launch_bounds__(256)
postprocess_kernel(const float* __restrict__ low_res, int n_masks, int R, int S, int in_h, int in_w, int H, int W,
                   float* __restrict__ out, int* __restrict__ bbox /*[5]: xmin ymin xmax ymax count (mask 0)*/, const int* skip) {
  SKIP_RETURN(skip);
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  const long long HW = (long long)H * W;
  int xmin = 0x7fffffff, ymin = 0x7fffffff, xmax = -1, ymax = -1, cnt = 0;
  if (i < HW * n_masks) {
    const int m = (int)(i / HW);
    const int y = (int)((i % HW) / W), x = (int)(i % W);
    const float* lr = low_res + (size_t)m * R * R;
    const float sy = (float)in_h / (float)H, sx = (float)in_w / (float)W;
    int y0, y1, x0, x1; float ly, lx;
    src_index(sy, y, in_h, y0, y1, ly);
    src_index(sx, x, in_w, x0, x1, lx);
    float hy = 1.f - ly, hx = 1.f - lx;
    float v = hy * (hx * up4_sample(lr, R, S, y0, x0) + lx * up4_sample(lr, R, S, y0, x1)) +
              ly * (hx * up4_sample(lr, R, S, y1, x0) + lx * up4_sample(lr, R, S, y1, x1));
    out[i] = v;
    if (m == 0 && v > 0.f) { xmin = xmax = x; ymin = ymax = y; cnt = 1; }
  }
  if (bbox) {
    // block reduce then 5 atomics per block
    __shared__ int sred[5][8];
    for (int o = 16; o > 0; o >>= 1) {
      xmin = min(xmin, __shfl_xor_sync(0xffffffffu, xmin, o));
      ymin = min(ymin, __shfl_xor_sync(0xffffffffu, ymin, o));
      xmax = max(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
      ymax = max(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { sred[0][w] = xmin; sred[1][w] = ymin; sred[2][w] = xmax; sred[3][w] = ymax; sred[4][w] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int k = 1; k < 8; ++k) {
        sred[0][0] = min(sred[0][0], sred[0][k]); sred[1][0] = min(sred[1][0], sred[1][k]);
        sred[2][0] = max(sred[2][0], sred[2][k]); sred[3][0] = max(sred[3][0], sred[3][k]);
        sred[4][0] += sred[4][k];
      }
      if (sred[4][0] > 0) {
        atomicMin(&bbox[0], sred[0][0]); atomicMin(&bbox[1], sred[1][0]);
        atomicMax(&bbox[2], sred[2][0]); atomicMax(&bbox[3], sred[3][0]);
        atomicAdd(&bbox[4], sred[4][0]);
      }
    }
  }
}
// refinement control (sam_pt.py:810-820): count<2 -> stop; else box = (xmin,ymin,xmax,ymax) in ORIGINAL pixels (the
// reference passes it to predict_torch without apply_boxes, SURVEY §0.8); resets the accumulators for the next call.
__global__ void refine_ctl_kernel(int* bbox, float* box_out, int* skip, int* n_done) {
  if (*skip == 0) {
    if (bbox[4] < 2) *skip = 1;
    else {
      box_out[0] = (float)bbox[0]; box_out[1] = (float)bbox[1]; box_out[2] = (float)bbox[2]; box_out[3] = (float)bbox[3];
      if (n_done) *n_done += 1;
    }
  }
  bbox[0] = 0x7fffffff; bbox[1] = 0x7fffffff; bbox[2] = -1; bbox[3] = -1; bbox[4] = 0;
}
__global__ void init_ctl_kernel(int* bbox, int* skip, int* n_done) {
  bbox[0] = 0x7fffffff; bbox[1] = 0x7fffffff; bbox[2] = -1; bbox[3] = -1; bbox[4] = 0;
  *skip = 0;
  if (n_done) *n_done = 0;
}

// ====================================================================================================================
// host orchestration
// ====================================================================================================================
struct AttnW {
  const float *qw, *qb, *kw, *kb, *vw, *vb, *ow, *ob; int internal;
  // image-side projections on tensor cores: weights as fp16 hi|lo [N, 2K] (null: that projection is token-side only)
  const __half *qw16 = nullptr, *kw16 = nullptr, *vw16 = nullptr, *ow16 = nullptr;
};
struct LayerW {
  AttnW self_attn, t2i, i2t;
  const float *n1w, *n1b, *n2w, *n2b, *n3w, *n3b, *n4w, *n4b;
  const float *l1w, *l1b, *l2w, *l2b;
  const float *pek_t2i, *peq_i2t;  // key_pe @ Wk^T (t2i) and key_pe @ Wq^T (i2t): constant, precomputed at load time
};
struct DecW {
  LayerW layer[2];
  AttnW final_attn; const float *nfw, *nfb, *pek_final;
  const float *up0_w /*[256 tok-in][4*64]^T as [4*64][256]*/, *up0_b4 /*[256] bias tiled over the 4 sub-pixels*/;
  const __half* up0_w16 = nullptr;  // the same matrix as fp16 hi|lo [256, 512] for the tensor-core path
  bool tc = false;                  // image-side GEMMs (4096-row operands) on the tensor-core split-precision GEMM
  const float *up_lnw, *up_lnb, *up3_w, *up3_b;
  Mlp3Job hyper[4], iou;
  DenseW dense;
  PromptArgs prompt;
  int n_out_tok;
  // HQ-SAM
  int hq = 0;
  Mlp3Job hq_mlp;
  const float *mf0_w, *mf0_b, *mf_lnw, *mf_lnb, *mf3_w, *mf3_b;
  const float *enc0_w, *enc0_b4, *enc_lnw, *enc_lnb, *enc3_w, *enc3_b;
  const float *cv0_w, *cv0_b4, *cv_lnw, *cv_lnb, *cv3_w, *cv3_b;
  int vit_dim = 0;
};

static int load_attn(Ctx* c, const std::string& p, AttnW* a, int internal) {
  a->internal = internal;
  SAMPT_TRY(get_f32(c, p + "q_proj.weight", &a->qw)); SAMPT_TRY(get_f32(c, p + "q_proj.bias", &a->qb));
  SAMPT_TRY(get_f32(c, p + "k_proj.weight", &a->kw)); SAMPT_TRY(get_f32(c, p + "k_proj.bias", &a->kb));
  SAMPT_TRY(get_f32(c, p + "v_proj.weight", &a->vw)); SAMPT_TRY(get_f32(c, p + "v_proj.bias", &a->vb));
  SAMPT_TRY(get_f32(c, p + "out_proj.weight", &a->ow)); SAMPT_TRY(get_f32(c, p + "out_proj.bias", &a->ob));
  return 0;
}
static bool decoder_tc_enabled() {
  static const int on = [] { const char* e = std::getenv("SAMPT_DECODER_TC"); return (e != nullptr && e[0] == '0') ? 0 : 1; }();
  return on != 0;
}
static int load_w16(Ctx* c, const std::string& name, const __half** out) { return get_f16(c, name, out); }
static int load_mlp3(Ctx* c, const std::string& p, Mlp3Job* j, int n_out) {
  SAMPT_TRY(get_f32(c, p + "layers.0.weight", &j->w0)); SAMPT_TRY(get_f32(c, p + "layers.0.bias", &j->b0));
  SAMPT_TRY(get_f32(c, p + "layers.1.weight", &j->w1)); SAMPT_TRY(get_f32(c, p + "layers.1.bias", &j->b1));
  SAMPT_TRY(get_f32(c, p + "layers.2.weight", &j->w2)); SAMPT_TRY(get_f32(c, p + "layers.2.bias", &j->b2));
  j->n_out = n_out;
  return 0;
}
static int load_dec(Ctx* c, DecW* w) {
  const std::string md = "sam.mask_decoder.", tr = md + "transformer.", pe = "sam.prompt_encoder.";
  for (int i = 0; i < 2; ++i) {
    const std::string lp = tr + "layers." + std::to_string(i) + ".";
    LayerW& L = w->layer[i];
    SAMPT_TRY(load_attn(c, lp + "self_attn.", &L.self_attn, 256));
    SAMPT_TRY(load_attn(c, lp + "cross_attn_token_to_image.", &L.t2i, 128));
    SAMPT_TRY(load_attn(c, lp + "cross_attn_image_to_token.", &L.i2t, 128));
    SAMPT_TRY(get_f32(c, lp + "norm1.weight", &L.n1w)); SAMPT_TRY(get_f32(c, lp + "norm1.bias", &L.n1b));
    SAMPT_TRY(get_f32(c, lp + "norm2.weight", &L.n2w)); SAMPT_TRY(get_f32(c, lp + "norm2.bias", &L.n2b));
    SAMPT_TRY(get_f32(c, lp + "norm3.weight", &L.n3w)); SAMPT_TRY(get_f32(c, lp + "norm3.bias", &L.n3b));
    SAMPT_TRY(get_f32(c, lp + "norm4.weight", &L.n4w)); SAMPT_TRY(get_f32(c, lp + "norm4.bias", &L.n4b));
    SAMPT_TRY(get_f32(c, lp + "mlp.lin1.weight", &L.l1w)); SAMPT_TRY(get_f32(c, lp + "mlp.lin1.bias", &L.l1b));
    SAMPT_TRY(get_f32(c, lp + "mlp.lin2.weight", &L.l2w)); SAMPT_TRY(get_f32(c, lp + "mlp.lin2.bias", &L.l2b));
    SAMPT_TRY(get_f32(c, lp + "pek_t2i", &L.pek_t2i)); SAMPT_TRY(get_f32(c, lp + "peq_i2t", &L.peq_i2t));
  }
  SAMPT_TRY(load_attn(c, tr + "final_attn_token_to_image.", &w->final_attn, 128));
  w->tc = decoder_tc_enabled() && c->find(md + "output_upscaling.0.w16") != nullptr;
  if (w->tc) {
    for (int i = 0; i < 2; ++i) {
      const std::string lp = tr + "layers." + std::to_string(i) + ".";
      SAMPT_TRY(load_w16(c, lp + "cross_attn_token_to_image.k_proj.w16", &w->layer[i].t2i.kw16));
      SAMPT_TRY(load_w16(c, lp + "cross_attn_token_to_image.v_proj.w16", &w->layer[i].t2i.vw16));
      SAMPT_TRY(load_w16(c, lp + "cross_attn_image_to_token.q_proj.w16", &w->layer[i].i2t.qw16));
      SAMPT_TRY(load_w16(c, lp + "cross_attn_image_to_token.out_proj.w16", &w->layer[i].i2t.ow16));
    }
    SAMPT_TRY(load_w16(c, tr + "final_attn_token_to_image.k_proj.w16", &w->final_attn.kw16));
    SAMPT_TRY(load_w16(c, tr + "final_attn_token_to_image.v_proj.w16", &w->final_attn.vw16));
    SAMPT_TRY(load_w16(c, md + "output_upscaling.0.w16", &w->up0_w16));
  }
  SAMPT_TRY(get_f32(c, tr + "norm_final_attn.weight", &w->nfw)); SAMPT_TRY(get_f32(c, tr + "norm_final_attn.bias", &w->nfb));
  SAMPT_TRY(get_f32(c, tr + "pek_final", &w->pek_final));
  SAMPT_TRY(get_f32(c, md + "output_upscaling.0.weight_gemm", &w->up0_w));
  SAMPT_TRY(get_f32(c, md + "output_upscaling.0.bias4", &w->up0_b4));
  SAMPT_TRY(get_f32(c, md + "output_upscaling.1.weight", &w->up_lnw)); SAMPT_TRY(get_f32(c, md + "output_upscaling.1.bias", &w->up_lnb));
  SAMPT_TRY(get_f32(c, md + "output_upscaling.3.weight", &w->up3_w)); SAMPT_TRY(get_f32(c, md + "output_upscaling.3.bias", &w->up3_b));
  for (int i = 0; i < 4; ++i) SAMPT_TRY(load_mlp3(c, md + "output_hypernetworks_mlps." + std::to_string(i) + ".", &w->hyper[i], 32));
  SAMPT_TRY(load_mlp3(c, md + "iou_prediction_head.", &w->iou, 4));
  DenseW& d = w->dense;
  SAMPT_TRY(get_f32(c, pe + "mask_downscaling.0.weight", &d.w0)); SAMPT_TRY(get_f32(c, pe + "mask_downscaling.0.bias", &d.b0));
  SAMPT_TRY(get_f32(c, pe + "mask_downscaling.1.weight", &d.ln1w)); SAMPT_TRY(get_f32(c, pe + "mask_downscaling.1.bias", &d.ln1b));
  SAMPT_TRY(get_f32(c, pe + "mask_downscaling.3.weight", &d.w3)); SAMPT_TRY(get_f32(c, pe + "mask_downscaling.3.bias", &d.b3));
  SAMPT_TRY(get_f32(c, pe + "mask_downscaling.4.weight", &d.ln4w)); SAMPT_TRY(get_f32(c, pe + "mask_downscaling.4.bias", &d.ln4b));
  SAMPT_TRY(get_f32(c, pe + "mask_downscaling.6.weight", &d.w6)); SAMPT_TRY(get_f32(c, pe + "mask_downscaling.6.bias", &d.b6));
  SAMPT_TRY(get_f32(c, pe + "no_mask_embed.weight", &d.no_mask));
  PromptArgs& pa = w->prompt;
  SAMPT_TRY(get_f32(c, pe + "pe_layer.positional_encoding_gaussian_matrix", &pa.gauss));
  for (int i = 0; i < 4; ++i) SAMPT_TRY(get_f32(c, pe + "point_embeddings." + std::to_string(i) + ".weight", &pa.pt_emb[i]));
  SAMPT_TRY(get_f32(c, pe + "not_a_point_embed.weight", &pa.not_a_point));
  SAMPT_TRY(get_f32(c, md + "output_tokens", &pa.out_tokens));
  const TensorRef* ot = c->find(md + "output_tokens");
  pa.n_out_tok = (int)ot->dims[0];
  w->n_out_tok = pa.n_out_tok;
  w->hq = c->find(md + "hf_mlp.layers.0.weight") != nullptr;
  if (w->hq) {
    SAMPT_CHECK(pa.n_out_tok == 6, "HQ decoder expects 6 output tokens (iou, 4 mask, hq), got %d", pa.n_out_tok);
    SAMPT_TRY(load_mlp3(c, md + "hf_mlp.", &w->hq_mlp, 32));
    SAMPT_TRY(get_f32(c, md + "embedding_maskfeature.0.weight_rsck", &w->mf0_w)); SAMPT_TRY(get_f32(c, md + "embedding_maskfeature.0.bias", &w->mf0_b));
    SAMPT_TRY(get_f32(c, md + "embedding_maskfeature.1.weight", &w->mf_lnw)); SAMPT_TRY(get_f32(c, md + "embedding_maskfeature.1.bias", &w->mf_lnb));
    SAMPT_TRY(get_f32(c, md + "embedding_maskfeature.3.weight_rsck", &w->mf3_w)); SAMPT_TRY(get_f32(c, md + "embedding_maskfeature.3.bias", &w->mf3_b));
    SAMPT_TRY(get_f32(c, md + "embedding_encoder.0.weight_gemm", &w->enc0_w)); SAMPT_TRY(get_f32(c, md + "embedding_encoder.0.bias4", &w->enc0_b4));
    SAMPT_TRY(get_f32(c, md + "embedding_encoder.1.weight", &w->enc_lnw)); SAMPT_TRY(get_f32(c, md + "embedding_encoder.1.bias", &w->enc_lnb));
    SAMPT_TRY(get_f32(c, md + "embedding_encoder.3.weight", &w->enc3_w)); SAMPT_TRY(get_f32(c, md + "embedding_encoder.3.bias", &w->enc3_b));
    SAMPT_TRY(get_f32(c, md + "compress_vit_feat.0.weight_gemm", &w->cv0_w)); SAMPT_TRY(get_f32(c, md + "compress_vit_feat.0.bias4", &w->cv0_b4));
    SAMPT_TRY(get_f32(c, md + "compress_vit_feat.1.weight", &w->cv_lnw)); SAMPT_TRY(get_f32(c, md + "compress_vit_feat.1.bias", &w->cv_lnb));
    SAMPT_TRY(get_f32(c, md + "compress_vit_feat.3.weight", &w->cv3_w)); SAMPT_TRY(get_f32(c, md + "compress_vit_feat.3.bias", &w->cv3_b));
    w->vit_dim = (int)c->find(md + "compress_vit_feat.0.weight_gemm")->dims[1];
  }
  return 0;
}

struct DecBufs {
  float *tokens, *queries, *qpe, *tq, *tk, *tv, *ta, *tmp, *mlp_h;   // token side  (T rows)
  float *src, *keys, *ik, *iv, *iq, *ia;                            // image side  (4096 rows)
  __half *keys16 = nullptr, *ia16 = nullptr;                         // fp16 hi|lo copies of keys [GG,512] / ia [GG,256] (tensor-core path)
  float *u1, *hyper, *iou4, *part;
  float *u_sam, *mf1, *mf2;  // HQ only
  int T;
};

#define LAUNCH_OK() do { c->launches++; SAMPT_LAUNCH_CHECK(); } while (0)

static int sg(Ctx* c, cudaStream_t st, const float* X, int ldx, const float* W, const float* b, const float* resid, int ldr,
              float* Y, int ldy, int M, int N, int K, int act, const int* skip) {
  return sgemm_nt_skip(c, st, X, ldx, W, K, b, resid, ldr, Y, ldy, M, N, K, act, skip);
}

// x [rows, K] fp32 -> out [rows, 2K] fp16: hi = fp16(x) | lo = fp16(x - hi)   (A operand of the split-precision tensor-core GEMM)
__global__ void __launch_bounds__(256)
split_f32_kernel(const float* __restrict__ x, __half* __restrict__ out, long long n4 /* rows*K/4 */, int K, const int* skip) {
  SKIP_RETURN(skip);
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n4) return;
  const long long e = i * 4;
  const long long r = e / K;
  const int cidx = (int)(e % K);
  const float4 v = *reinterpret_cast<const float4*>(x + e);
  const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
  const __half2 l0 = __floats2half2_rn(v.x - f0.x, v.y - f0.y), l1 = __floats2half2_rn(v.z - f1.x, v.w - f1.y);
  __half* o = out + r * 2 * K + cidx;
  *reinterpret_cast<uint2*>(o) = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
  *reinterpret_cast<uint2*>(o + K) = make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
}
static int split_rows(Ctx* c, cudaStream_t st, const float* x, __half* out, int rows, int K, const int* skip) {
  const long long n4 = (long long)rows * K / 4;
  split_f32_kernel<<<cdiv(n4, 256), 256, 0, st>>>(x, out, n4, K, skip);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}
// Y = X W^T + b (+ resid), X given as fp16 hi|lo [M, 2K], W as fp16 hi|lo [N, 2K]: three tensor-core passes A_hi.B_hi + A_lo.B_hi +
// A_hi.B_lo into one fp32 register accumulator (products exact to ~2^-22: the decoder stays at fp32-level accuracy).  The residual is
// indexed like Y (same leading dimension).
static int tcg(Ctx* c, cudaStream_t st, const __half* X16, const __half* W16, const float* b, const float* resid, float* Y, int ldy,
               int M, int N, int K, const int* skip) {
  GemmSeg seg{};
  seg.nseg = 3;
  seg.a_off[0] = 0; seg.b_off[0] = 0;
  seg.a_off[1] = K; seg.b_off[1] = 0;
  seg.a_off[2] = 0; seg.b_off[2] = K;
  GemmEpi ep{};
  ep.out32 = Y; ep.ldc = ldy; ep.bias = b; ep.resid = resid; ep.skip = skip;
  return gemm_tc(c, st, X16, 2 * K, W16, 2 * K, M, N, K, seg, ep);
}

// The attention cores of the decoder, 8 heads.  Each launcher is shared by the decode chain and the unit-test entries.
// Token self-attention, head dim 32 (q/k/v/out [T, 256]): kind 0 = attn_q_small_kernel (block per token and head), the chain's
// choice for T <= 16; kind 1 = attn_tok_self_kernel (warp per query, the head's K/V in dynamic shared memory).
static int launch_tok_self(Ctx* c, cudaStream_t st, int kind, const float* q, const float* k, const float* v, float* out, int T,
                           const int* skip) {
  if (kind == 1) {
    const size_t smem = ((size_t)2 * T * 33 + (size_t)8 * T + 8 * 32) * sizeof(float);
    SAMPT_CHECK(smem <= 200 * 1024, "too many prompt tokens (%d) for the token self-attention", T);
    SAMPT_TRY(ensure_func_smem(c, "attn_tok_self_kernel<32>", attn_tok_self_kernel<32>, 200 * 1024));
    attn_tok_self_kernel<32><<<dim3(cdiv(T, 32), 8), 256, smem, st>>>(q, k, v, out, T, 8, skip);
  } else {
    attn_q_small_kernel<32><<<dim3(T, 8), 256, 0, st>>>(q, k, v, out, T, 8, skip);
  }
  LAUNCH_OK();
  return 0;
}
// Tokens -> image, head dim 16: q [T, 128] over k/v [Nk, 128], split over the keys in slices of 256 (part: T*8*nsplit*18 floats).
static int launch_t2i(Ctx* c, cudaStream_t st, const float* q, const float* k, const float* v, float* part, float* out, int T, int Nk,
                      const int* skip) {
  constexpr int KPS = 256;
  const int nsplit = (Nk + KPS - 1) / KPS;
  attn_t2i_partial_kernel<16, KPS><<<dim3(nsplit, 8), 256, 0, st>>>(q, k, v, part, T, Nk, 8, skip);
  LAUNCH_OK();
  attn_t2i_combine_kernel<16><<<cdiv(T * 128, 128), 128, 0, st>>>(part, out, T, 8, nsplit, skip);
  LAUNCH_OK();
  return 0;
}
// Image -> tokens, head dim 16: q [N, 128] over k/v [T, 128].
static int launch_i2t(Ctx* c, cudaStream_t st, const float* q, const float* k, const float* v, float* out, int N, int T, const int* skip) {
  attn_kv_small_kernel<16><<<cdiv((long long)cdiv(N, 32) * 8, 8), 256, 0, st>>>(q, k, v, out, N, T, 8, skip);
  LAUNCH_OK();
  return 0;
}

// tokens -> image attention: queries attend over the 4096 image tokens.  q_in already includes the query PE.
static int attn_tok_to_img(Ctx* c, cudaStream_t st, const AttnW& a, const float* q_in, const float* keys, const float* pek,
                           DecBufs& b, float* out /*[T,256]*/, const float* resid, int GG, const int* skip) {
  const int T = b.T;
  SAMPT_TRY(sg(c, st, q_in, 256, a.qw, a.qb, nullptr, 0, b.tq, 128, T, 128, 256, 0, skip));
  if (a.kw16 != nullptr) {   // tensor cores: b.keys16 holds the hi|lo split of `keys` (kept in sync by the caller)
    SAMPT_TRY(tcg(c, st, b.keys16, a.kw16, a.kb, pek, b.ik, 128, GG, 128, 256, skip));           // (keys + key_pe) Wk^T
    SAMPT_TRY(tcg(c, st, b.keys16, a.vw16, a.vb, nullptr, b.iv, 128, GG, 128, 256, skip));
  } else {
    SAMPT_TRY(sg(c, st, keys, 256, a.kw, a.kb, pek, 128, b.ik, 128, GG, 128, 256, 0, skip));   // (keys + key_pe) Wk^T
    SAMPT_TRY(sg(c, st, keys, 256, a.vw, a.vb, nullptr, 0, b.iv, 128, GG, 128, 256, 0, skip));
  }
  SAMPT_TRY(launch_t2i(c, st, b.tq, b.ik, b.iv, b.part, b.ta, T, GG, skip));
  SAMPT_TRY(sg(c, st, b.ta, 128, a.ow, a.ob, resid, 256, out, 256, T, 256, 128, 0, skip));
  return 0;
}

static int two_way_layer(Ctx* c, cudaStream_t st, const LayerW& L, int idx, DecBufs& b, int GG, const int* skip) {
  const int T = b.T;
  // (1) self attention on the prompt tokens
  if (idx == 0) {
    SAMPT_TRY(sg(c, st, b.queries, 256, L.self_attn.qw, L.self_attn.qb, nullptr, 0, b.tq, 256, T, 256, 256, 0, skip));
    SAMPT_TRY(sg(c, st, b.queries, 256, L.self_attn.kw, L.self_attn.kb, nullptr, 0, b.tk, 256, T, 256, 256, 0, skip));
  } else {
    add_kernel<<<cdiv(T * 64, 256), 256, 0, st>>>(b.queries, b.tokens, b.qpe, (long long)T * 64, skip);
    LAUNCH_OK();
    SAMPT_TRY(sg(c, st, b.qpe, 256, L.self_attn.qw, L.self_attn.qb, nullptr, 0, b.tq, 256, T, 256, 256, 0, skip));
    SAMPT_TRY(sg(c, st, b.qpe, 256, L.self_attn.kw, L.self_attn.kb, nullptr, 0, b.tk, 256, T, 256, 256, 0, skip));
  }
  SAMPT_TRY(sg(c, st, b.queries, 256, L.self_attn.vw, L.self_attn.vb, nullptr, 0, b.tv, 256, T, 256, 256, 0, skip));
  SAMPT_TRY(launch_tok_self(c, st, T > 16 ? 1 : 0, b.tq, b.tk, b.tv, b.ta, T, skip));
  // layer 0 replaces the queries, later layers add (upstream skip_first_layer_pe)
  SAMPT_TRY(sg(c, st, b.ta, 256, L.self_attn.ow, L.self_attn.ob, idx == 0 ? nullptr : b.queries, 256, b.tmp, 256, T, 256, 256, 0, skip));
  ln256_kernel<<<cdiv(T, 8), 256, 0, st>>>(b.tmp, nullptr, L.n1w, L.n1b, b.queries, T, 1e-5f, skip);
  LAUNCH_OK();
  // (2) cross attention tokens -> image
  add_kernel<<<cdiv(T * 64, 256), 256, 0, st>>>(b.queries, b.tokens, b.qpe, (long long)T * 64, skip);
  LAUNCH_OK();
  SAMPT_TRY(attn_tok_to_img(c, st, L.t2i, b.qpe, b.keys, L.pek_t2i, b, b.tmp, b.queries, GG, skip));
  ln256_kernel<<<cdiv(T, 8), 256, 0, st>>>(b.tmp, nullptr, L.n2w, L.n2b, b.queries, T, 1e-5f, skip);
  LAUNCH_OK();
  // (3) MLP
  SAMPT_TRY(sg(c, st, b.queries, 256, L.l1w, L.l1b, nullptr, 0, b.mlp_h, 2048, T, 2048, 256, 2, skip));
  SAMPT_TRY(sg(c, st, b.mlp_h, 2048, L.l2w, L.l2b, b.queries, 256, b.tmp, 256, T, 256, 2048, 0, skip));
  ln256_kernel<<<cdiv(T, 8), 256, 0, st>>>(b.tmp, nullptr, L.n3w, L.n3b, b.queries, T, 1e-5f, skip);
  LAUNCH_OK();
  // (4) cross attention image -> tokens
  add_kernel<<<cdiv(T * 64, 256), 256, 0, st>>>(b.queries, b.tokens, b.qpe, (long long)T * 64, skip);
  LAUNCH_OK();
  if (L.i2t.qw16 != nullptr) SAMPT_TRY(tcg(c, st, b.keys16, L.i2t.qw16, L.i2t.qb, L.peq_i2t, b.iq, 128, GG, 128, 256, skip));
  else SAMPT_TRY(sg(c, st, b.keys, 256, L.i2t.qw, L.i2t.qb, L.peq_i2t, 128, b.iq, 128, GG, 128, 256, 0, skip));  // (keys+pe) Wq^T
  SAMPT_TRY(sg(c, st, b.qpe, 256, L.i2t.kw, L.i2t.kb, nullptr, 0, b.tk, 128, T, 128, 256, 0, skip));
  SAMPT_TRY(sg(c, st, b.queries, 256, L.i2t.vw, L.i2t.vb, nullptr, 0, b.tv, 128, T, 128, 256, 0, skip));
  SAMPT_TRY(launch_i2t(c, st, b.iq, b.tk, b.tv, b.ia, GG, T, skip));
  if (L.i2t.ow16 != nullptr) {
    SAMPT_TRY(split_rows(c, st, b.ia, b.ia16, GG, 128, skip));
    SAMPT_TRY(tcg(c, st, b.ia16, L.i2t.ow16, L.i2t.ob, b.keys, b.src, 256, GG, 256, 128, skip));          // keys + attn_out
  } else {
    SAMPT_TRY(sg(c, st, b.ia, 128, L.i2t.ow, L.i2t.ob, b.keys, 256, b.src, 256, GG, 256, 128, 0, skip));   // keys + attn_out
  }
  ln256_kernel<<<cdiv(GG, 8), 256, 0, st>>>(b.src, nullptr, L.n4w, L.n4b, b.keys, GG, 1e-5f, skip);
  LAUNCH_OK();
  if (L.i2t.ow16 != nullptr) SAMPT_TRY(split_rows(c, st, b.keys, b.keys16, GG, 256, skip));   // keys changed: refresh the hi|lo copy
  return 0;
}

struct DecodeCall {
  const float* feat_tok;     // [GG,256] token-major image embedding
  const float* coords; const int* labels; int K;
  const float* box; int use_box;
  const float* mask_in;      // [256*256] or null
  int n_masks, tok0;         // output masks = mask tokens [tok0, tok0+n_masks)
  int in_h, in_w, H, W;
  float* logits;             // [n_masks, H, W]
  float* iou;                // [n_masks]
  float* low_res;            // [n_masks, 256, 256]
  int* bbox;                 // [5] or null
  const int* skip;
  const float* hq_feat;      // [256*256][32] HQ features of this frame, or null (plain SAM)
};

// prompt encoder: sparse tokens [T, 256] (output tokens first) and src = image embedding + dense embedding [G*G, 256]
static int encode_prompt(Ctx* c, cudaStream_t st, const DecW& w, const DecodeCall& d, int G, float* tokens, float* src) {
  const int T = w.n_out_tok + d.K + (d.use_box ? 2 : 1);
  PromptArgs pa = w.prompt;
  pa.coords = d.coords; pa.labels = d.labels; pa.K = d.K; pa.box = d.box; pa.use_box = d.use_box; pa.img_size = (float)(G * 16);
  prompt_tokens_kernel<<<T, 256, 0, st>>>(pa, tokens, d.skip);
  LAUNCH_OK();
  dense_src_kernel<<<cdiv(G * G, 8), 256, 0, st>>>(d.feat_tok, d.mask_in, w.dense, src, G, d.skip);
  LAUNCH_OK();
  return 0;
}
// LN2d + GELU + ConvT(64->32) + GELU + hyper-network dot on the first ConvT's output u1 [G*G, 4*64] -> low_res [n_masks, 4G, 4G]
static int launch_upscale(Ctx* c, cudaStream_t st, const DecW& w, const float* u1, const float* hyper, int n_masks, float* low_res,
                          int G, float* u_out, const int* skip) {
  upscale_mask_kernel<<<cdiv(16 * G * G, 256), 256, 0, st>>>(u1, w.up_lnw, w.up_lnb, w.up3_w, w.up3_b, hyper, n_masks, low_res, G,
                                                             u_out, skip);
  LAUNCH_OK();
  return 0;
}
static int launch_postprocess(Ctx* c, cudaStream_t st, const float* low_res, int n_masks, int G, int in_h, int in_w, int H, int W,
                              float* out, int* bbox, const int* skip) {
  postprocess_kernel<<<cdiv((long long)n_masks * H * W, 256), 256, 0, st>>>(low_res, n_masks, 4 * G, 16 * G, in_h, in_w, H, W, out,
                                                                           bbox, skip);
  LAUNCH_OK();
  return 0;
}

static int decode_once(Ctx* c, cudaStream_t st, DecW& w, DecBufs& b, const DecodeCall& d, int G) {
  const int GG = G * G;
  const int T = w.n_out_tok + d.K + (d.use_box ? 2 : 1);
  b.T = T;
  SAMPT_TRY(encode_prompt(c, st, w, d, G, b.tokens, b.keys));
  SAMPT_CUDA(cudaMemcpyAsync(b.queries, b.tokens, (size_t)T * 256 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (w.tc) SAMPT_TRY(split_rows(c, st, b.keys, b.keys16, GG, 256, d.skip));
  for (int i = 0; i < 2; ++i) SAMPT_TRY(two_way_layer(c, st, w.layer[i], i, b, GG, d.skip));
  // final token -> image attention
  add_kernel<<<cdiv(T * 64, 256), 256, 0, st>>>(b.queries, b.tokens, b.qpe, (long long)T * 64, d.skip);
  LAUNCH_OK();
  SAMPT_TRY(attn_tok_to_img(c, st, w.final_attn, b.qpe, b.keys, w.pek_final, b, b.tmp, b.queries, GG, d.skip));
  ln256_kernel<<<cdiv(T, 8), 256, 0, st>>>(b.tmp, nullptr, w.nfw, w.nfb, b.queries, T, 1e-5f, d.skip);
  LAUNCH_OK();
  // heads
  Mlp3Jobs jobs{};
  for (int m = 0; m < d.n_masks; ++m) {
    jobs.j[m] = w.hyper[d.tok0 + m];
    jobs.j[m].x = b.queries + (size_t)(1 + d.tok0 + m) * 256;
    jobs.j[m].y = b.hyper + m * 32;
  }
  jobs.j[d.n_masks] = w.iou;
  jobs.j[d.n_masks].x = b.queries;
  jobs.j[d.n_masks].y = b.iou4;
  int njobs = d.n_masks + 1;
  const bool hq = w.hq && d.hq_feat != nullptr;
  if (hq) {
    SAMPT_CHECK(d.n_masks == 1, "HQ decoder: only single-mask output (multimask_output=False) is built");
    jobs.j[njobs] = w.hq_mlp;
    jobs.j[njobs].x = b.queries + (size_t)5 * 256;  // hq token row
    jobs.j[njobs].y = b.hyper + 4 * 32;
    ++njobs;
  }
  mlp3_kernel<<<njobs, 256, 0, st>>>(jobs, d.skip);
  LAUNCH_OK();
  // upscaling: ConvT(256->64) as GEMM [GG,256] x [256(4 sub-pixels x 64), 256]^T, then fused LN+GELU+ConvT+GELU+hyper dot
  if (w.tc) SAMPT_TRY(tcg(c, st, b.keys16, w.up0_w16, w.up0_b4, nullptr, b.u1, 256, GG, 256, 256, d.skip));
  else SAMPT_TRY(sg(c, st, b.keys, 256, w.up0_w, w.up0_b4, nullptr, 0, b.u1, 256, GG, 256, 256, 0, d.skip));
  SAMPT_TRY(launch_upscale(c, st, w, b.u1, b.hyper, d.n_masks, d.low_res, G, hq ? b.u_sam : nullptr, d.skip));
  if (hq) {
    // upscaled_embedding_hq = embedding_maskfeature(upscaled_embedding_sam) + hq_features ; mask += hyper_hq . that
    const int R = 4 * G;
    SAMPT_TRY(conv_nhwc_f32(c, st, b.u_sam, w.mf0_w, w.mf0_b, b.mf1, 1, R, R, 32, 64, 3, 3, 1, 1, d.skip));
    ln64_gelu_kernel<<<cdiv(R * R, 8), 256, 0, st>>>(b.mf1, w.mf_lnw, w.mf_lnb, R * R, d.skip);
    LAUNCH_OK();
    SAMPT_TRY(conv_nhwc_f32(c, st, b.mf1, w.mf3_w, w.mf3_b, b.mf2, 1, R, R, 64, 32, 3, 3, 1, 1, d.skip));
    hq_mask_add_kernel<<<cdiv(R * R, 256), 256, 0, st>>>(b.mf2, d.hq_feat, b.hyper + 4 * 32, d.low_res, R * R, d.skip);
    LAUNCH_OK();
  }
  SAMPT_TRY(launch_postprocess(c, st, d.low_res, d.n_masks, G, d.in_h, d.in_w, d.H, d.W, d.logits, d.bbox, d.skip));
  // iou predictions of the selected tokens
  SAMPT_CUDA(cudaMemcpyAsync(d.iou, b.iou4 + d.tok0, d.n_masks * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

static int alloc_dec_bufs(Ctx* c, DecBufs* b, int Tmax, int GG) {
  SAMPT_TRY(ws_get(c, &b->tokens, (size_t)Tmax * 256, "dec tokens"));
  SAMPT_TRY(ws_get(c, &b->queries, (size_t)Tmax * 256, "dec queries"));
  SAMPT_TRY(ws_get(c, &b->qpe, (size_t)Tmax * 256, "dec qpe"));
  SAMPT_TRY(ws_get(c, &b->tq, (size_t)Tmax * 256, "dec tq"));
  SAMPT_TRY(ws_get(c, &b->tk, (size_t)Tmax * 256, "dec tk"));
  SAMPT_TRY(ws_get(c, &b->tv, (size_t)Tmax * 256, "dec tv"));
  SAMPT_TRY(ws_get(c, &b->ta, (size_t)Tmax * 256, "dec ta"));
  SAMPT_TRY(ws_get(c, &b->tmp, (size_t)Tmax * 256, "dec tmp"));
  SAMPT_TRY(ws_get(c, &b->mlp_h, (size_t)Tmax * 2048, "dec mlp"));
  SAMPT_TRY(ws_get(c, &b->src, (size_t)GG * 256, "dec src"));
  SAMPT_TRY(ws_get(c, &b->keys, (size_t)GG * 256, "dec keys"));
  SAMPT_TRY(ws_get(c, &b->ik, (size_t)GG * 128, "dec ik"));
  SAMPT_TRY(ws_get(c, &b->iv, (size_t)GG * 128, "dec iv"));
  SAMPT_TRY(ws_get(c, &b->iq, (size_t)GG * 128, "dec iq"));
  SAMPT_TRY(ws_get(c, &b->ia, (size_t)GG * 128, "dec ia"));
  SAMPT_TRY(ws_get(c, &b->keys16, (size_t)GG * 512, "dec keys16"));
  SAMPT_TRY(ws_get(c, &b->ia16, (size_t)GG * 256, "dec ia16"));
  SAMPT_TRY(ws_get(c, &b->u1, (size_t)GG * 256, "dec u1"));
  SAMPT_TRY(ws_get(c, &b->hyper, (size_t)8 * 32, "dec hyper"));
  SAMPT_TRY(ws_get(c, &b->u_sam, (size_t)16 * GG * 32, "dec u_sam"));
  SAMPT_TRY(ws_get(c, &b->mf1, (size_t)16 * GG * 64, "dec mf1"));
  SAMPT_TRY(ws_get(c, &b->mf2, (size_t)16 * GG * 32, "dec mf2"));
  SAMPT_TRY(ws_get(c, &b->iou4, (size_t)8, "dec iou"));
  SAMPT_TRY(ws_get(c, &b->part, (size_t)Tmax * 8 * ((GG + 255) / 256) * 18, "dec attn partials"));
  return 0;
}

}  // namespace sampt

using namespace sampt;

extern "C" int sampt_sam_features_to_tokens(sampt_ctx* ctx, const float* feat_nchw, float* feat_tok, int C, int GG, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_CHECK(C % 32 == 0 && GG % 32 == 0, "features_to_tokens: C and G*G must be multiples of 32");
  nchw_to_tok_kernel<<<dim3(GG / 32, C / 32), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(feat_nchw, feat_tok, C, GG);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// SamPredictor.predict_torch (one call): prompt encoder + mask decoder + postprocess_masks.
extern "C" int sampt_sam_predict(sampt_ctx* ctx, const float* feat_tok, int G, const float* coords, const int* labels, int K,
                                 const float* box, const float* mask_input, int multimask, int in_h, int in_w, int H, int W,
                                 float* logits, float* iou, float* low_res, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  c->ws_reset();
  DecW w;
  SAMPT_TRY(load_dec(c, &w));
  DecBufs b;
  SAMPT_TRY(alloc_dec_bufs(c, &b, w.n_out_tok + K + 2, G * G));
  DecodeCall d{};
  d.feat_tok = feat_tok; d.coords = coords; d.labels = labels; d.K = K; d.box = box; d.use_box = box ? 1 : 0;
  d.mask_in = mask_input; d.n_masks = multimask ? 3 : 1; d.tok0 = multimask ? 1 : 0;
  d.in_h = in_h; d.in_w = in_w; d.H = H; d.W = W; d.logits = logits; d.iou = iou; d.low_res = low_res; d.bbox = nullptr; d.skip = nullptr;
  d.hq_feat = w.hq ? c->hq_feat : nullptr;
  return decode_once(c, st, w, b, d, G);
}

// SamPt.predict_mask (sam_pt.py:760-837) for negative_points_per_mask == 0 or > 0, with the iterative box refinement
// loop run entirely on the device.  coords/labels: visible points already mapped by apply_coords (1024 frame).
// n_pos_first: if > 0, a first call uses only the n_pos_first positive points and feeds its low-res mask to the second call
// (sam_pt.py:792-807); 0 = single initial call (:783-790); < 0 = the two-call form with an EMPTY positive set (negatives are visible
// but every positive point is occluded: the reference still runs the first predict_torch, on the padding point alone).
// outputs: logits [H,W], iou [1], low_res [256,256], n_refine_done [1] (int, device).
namespace sampt {

struct RefineShape { int G, K, npos, nref, in_h, in_w, H, W; int two_pass; };
struct RefinePtrs {
  const float* feat_tok; const float* coords; const int* labels; const float* pos_coords; const int* pos_labels;
  float* logits; float* iou; float* low_res; int* n_done; int* bbox; int* skip; float* box;
  const float* hq_feat = nullptr;
};

// enqueue the whole predict_mask chain (sam_pt.py:781-828) on `st`
static int enqueue_refine_chain(Ctx* c, cudaStream_t st, DecW& w, DecBufs& b, const RefineShape& s, const RefinePtrs& p) {
  init_ctl_kernel<<<1, 1, 0, st>>>(p.bbox, p.skip, p.n_done);
  c->launches++;
  DecodeCall d{};
  d.feat_tok = p.feat_tok; d.n_masks = 1; d.tok0 = 0; d.in_h = s.in_h; d.in_w = s.in_w; d.H = s.H; d.W = s.W;
  d.logits = p.logits; d.iou = p.iou; d.low_res = p.low_res; d.skip = nullptr; d.hq_feat = p.hq_feat;
  if (s.two_pass) {
    d.coords = p.pos_coords; d.labels = p.pos_labels; d.K = s.npos; d.box = nullptr; d.use_box = 0; d.mask_in = nullptr; d.bbox = nullptr;
    SAMPT_TRY(decode_once(c, st, w, b, d, s.G));
    d.mask_in = p.low_res;
  }
  d.coords = p.coords; d.labels = p.labels; d.K = s.K; d.box = nullptr; d.use_box = 0; d.bbox = p.bbox;
  if (!s.two_pass) d.mask_in = nullptr;
  SAMPT_TRY(decode_once(c, st, w, b, d, s.G));
  for (int it = 0; it < s.nref; ++it) {
    refine_ctl_kernel<<<1, 1, 0, st>>>(p.bbox, p.box, p.skip, p.n_done);
    c->launches++;
    d.box = p.box; d.use_box = 1; d.mask_in = p.low_res; d.skip = p.skip;
    SAMPT_TRY(decode_once(c, st, w, b, d, s.G));
  }
  SAMPT_LAUNCH_CHECK();
  return 0;
}

// One captured CUDA graph per chain shape: the ~500 kernels of a frame's 13 predict_torch calls replay as ONE launch.
// Buffers are carved from the decoder slab (stable addresses) ONCE PER SLOT, sized for `Kcap` prompt points, and shared by
// every graph of that slot: a slot's chains are stream-ordered (one stream per slot), so graphs that differ only in the number
// of visible prompt points K reuse the same memory and a new K costs a capture (~ms), not another ~60 MB buffer set.
// (Round 1 allocated a full buffer set per (K, npos, slot): a clip whose visible-point count varied filled the slab.)
struct SlotBufs {
  DecBufs bufs;
  float *feat, *coords, *pos_coords, *logits, *iou, *low, *box, *hqfeat = nullptr;
  int *labels, *pos_labels, *n_done, *bbox, *skip;
  int Kcap = 0, GG = 0, HW = 0, n_out_tok = 0;
  bool hq = false;
};
struct RefineGraph {
  RefineShape shape;
  cudaGraphExec_t exec = nullptr;
  long long launches = 0;
};
constexpr int DEC_KCAP_MIN = 320;      // 256 query points + other objects' positives (BASELINE configs[4]) without a re-carve
constexpr size_t DEC_MAX_GRAPHS = 512;

static void* dec_alloc(Ctx* c, size_t bytes) {
  size_t a = (c->dec_off + 255) & ~size_t(255);
  if (a + bytes > c->dec_bytes) return nullptr;
  c->dec_off = a + bytes;
  return c->dec_base + a;
}
template <typename T>
static int dec_get(Ctx* c, T** out, size_t count, const char* what) {
  *out = reinterpret_cast<T*>(dec_alloc(c, count * sizeof(T)));
  if (!*out) { set_error("decoder workspace exhausted allocating %s", what); return -3; }
  return 0;
}

// drop every captured graph and every slot's buffers (nothing may be in flight: synchronises the device)
static int dec_evict_all(Ctx* c) {
  SAMPT_CUDA(cudaDeviceSynchronize());
  for (auto& kv : c->graph_cache) {
    RefineGraph* g = reinterpret_cast<RefineGraph*>(kv.second);
    if (g->exec) cudaGraphExecDestroy(g->exec);
    delete g;
  }
  c->graph_cache.clear();
  for (auto& kv : c->dec_slots) delete reinterpret_cast<SlotBufs*>(kv.second);
  c->dec_slots.clear();
  c->dec_off = 0;
  return 0;
}

static int carve_slot(Ctx* c, DecW& w, const RefineShape& s, bool hq, int Kcap, SlotBufs** out) {
  SlotBufs* sb = new SlotBufs();
  sb->Kcap = Kcap; sb->GG = s.G * s.G; sb->HW = s.H * s.W; sb->hq = hq; sb->n_out_tok = w.n_out_tok;
  const int GG = sb->GG, Tmax = w.n_out_tok + Kcap + 2;
  DecBufs& b = sb->bufs;
  int rc = 0;
#define DG(ptr, count, what) if (rc == 0) rc = dec_get(c, &(ptr), (size_t)(count), what)
  DG(b.tokens, Tmax * 256, "tokens"); DG(b.queries, Tmax * 256, "queries"); DG(b.qpe, Tmax * 256, "qpe"); DG(b.tq, Tmax * 256, "tq");
  DG(b.tk, Tmax * 256, "tk"); DG(b.tv, Tmax * 256, "tv"); DG(b.ta, Tmax * 256, "ta"); DG(b.tmp, Tmax * 256, "tmp");
  DG(b.mlp_h, (size_t)Tmax * 2048, "mlp_h");
  DG(b.src, (size_t)GG * 256, "src"); DG(b.keys, (size_t)GG * 256, "keys"); DG(b.ik, (size_t)GG * 128, "ik"); DG(b.iv, (size_t)GG * 128, "iv");
  DG(b.iq, (size_t)GG * 128, "iq"); DG(b.ia, (size_t)GG * 128, "ia"); DG(b.u1, (size_t)GG * 256, "u1"); DG(b.hyper, 256, "hyper");
  DG(b.keys16, (size_t)GG * 512, "keys16"); DG(b.ia16, (size_t)GG * 256, "ia16");
  if (hq) { DG(b.u_sam, (size_t)16 * GG * 32, "u_sam"); DG(b.mf1, (size_t)16 * GG * 64, "mf1"); DG(b.mf2, (size_t)16 * GG * 32, "mf2"); }
  else { b.u_sam = b.mf1 = b.mf2 = nullptr; }
  DG(b.iou4, 8, "iou4"); DG(b.part, (size_t)Tmax * 8 * ((GG + 255) / 256) * 18, "attn partials");
  DG(sb->feat, (size_t)GG * 256, "feat stage"); DG(sb->coords, (size_t)Kcap * 2, "coords"); DG(sb->labels, Kcap, "labels");
  DG(sb->pos_coords, (size_t)Kcap * 2, "pos coords"); DG(sb->pos_labels, Kcap, "pos labels");
  DG(sb->logits, (size_t)s.H * s.W, "logits stage"); DG(sb->iou, 8, "iou"); DG(sb->low, (size_t)16 * GG, "low_res");
  DG(sb->n_done, 8, "n_done"); DG(sb->bbox, 8, "bbox"); DG(sb->skip, 8, "skip"); DG(sb->box, 8, "box");
  if (hq) DG(sb->hqfeat, (size_t)16 * GG * 32, "hq features stage");
#undef DG
  if (rc != 0) { delete sb; return rc; }
  if (hq) SAMPT_CUDA(cudaMemset(sb->hqfeat, 0, (size_t)16 * GG * 32 * sizeof(float)));
  *out = sb;
  return 0;
}

static int build_refine_graph(Ctx* c, DecW& w, const RefineShape& s, SlotBufs* sb, RefineGraph** out) {
  RefineGraph* g = new RefineGraph();
  g->shape = s;
  DecBufs b = sb->bufs;   // copy: decode_once writes b.T
  const int GG = sb->GG;
  RefinePtrs p{sb->feat, sb->coords, sb->labels, sb->pos_coords, sb->pos_labels, sb->logits, sb->iou, sb->low, sb->n_done, sb->bbox,
               sb->skip, sb->box};
  if (sb->hq) p.hq_feat = sb->hqfeat;
  if (!c->cap_stream) SAMPT_CUDA(cudaStreamCreateWithFlags(&c->cap_stream, cudaStreamNonBlocking));
  // eager warm-up on the capture stream (sets function attributes, touches every code path), then capture.  The slot's buffers
  // may still be in use by an earlier graph of this slot on the caller's stream, and cap_stream does not synchronise with the
  // legacy default stream (pending weight uploads): wait for the device.
  SAMPT_CUDA(cudaDeviceSynchronize());
  SAMPT_CUDA(cudaMemsetAsync(sb->feat, 0, (size_t)GG * 256 * sizeof(float), c->cap_stream));
  SAMPT_CUDA(cudaMemsetAsync(sb->coords, 0, (size_t)sb->Kcap * 2 * sizeof(float), c->cap_stream));
  SAMPT_CUDA(cudaMemsetAsync(sb->labels, 0, (size_t)sb->Kcap * sizeof(int), c->cap_stream));
  SAMPT_CUDA(cudaMemsetAsync(sb->pos_coords, 0, (size_t)sb->Kcap * 2 * sizeof(float), c->cap_stream));
  SAMPT_CUDA(cudaMemsetAsync(sb->pos_labels, 0, (size_t)sb->Kcap * sizeof(int), c->cap_stream));
  const long long l0 = c->launches;
  int rc = enqueue_refine_chain(c, c->cap_stream, w, b, s, p);
  if (rc != 0) { delete g; return rc; }
  SAMPT_CUDA(cudaStreamSynchronize(c->cap_stream));
  g->launches = c->launches - l0;
  SAMPT_CUDA(cudaStreamBeginCapture(c->cap_stream, cudaStreamCaptureModeRelaxed));
  rc = enqueue_refine_chain(c, c->cap_stream, w, b, s, p);
  cudaGraph_t graph = nullptr;
  cudaError_t e = cudaStreamEndCapture(c->cap_stream, &graph);
  c->launches -= g->launches;  // the capture pass did not execute anything
  if (rc != 0) { delete g; return rc; }
  SAMPT_CHECK(e == cudaSuccess && graph != nullptr, "stream capture of the decode chain failed: %s", cudaGetErrorString(e));
  SAMPT_CUDA(cudaGraphInstantiate(&g->exec, graph, 0));
  cudaGraphDestroy(graph);
  *out = g;
  return 0;
}

}  // namespace sampt

extern "C" int sampt_ctx_set_decoder_workspace(sampt_ctx* ctx, void* dev_ptr, size_t bytes) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_TRY(dec_evict_all(c));
  c->dec_base = reinterpret_cast<char*>(dev_ptr);
  c->dec_bytes = bytes;
  c->dec_off = 0;
  return 0;
}

extern "C" int sampt_sam_predict_refine(sampt_ctx* ctx, const float* feat_tok, int G, const float* coords, const int* labels, int K,
                                        const float* pos_coords, const int* pos_labels, int n_pos_first, int n_refine, int in_h,
                                        int in_w, int H, int W, float* logits, float* iou, float* low_res, int* n_refine_done,
                                        int graph_slot, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DecW w;
  SAMPT_TRY(load_dec(c, &w));
  RefineShape s{G, K, n_pos_first > 0 ? n_pos_first : 0, n_refine, in_h, in_w, H, W, n_pos_first != 0 ? 1 : 0};
  if (c->dec_base == nullptr) {
    // eager path (no decoder slab registered): buffers from the shared workspace, kernels launched one by one.  NOT safe for
    // concurrent use from several streams (one shared workspace): the Python side forces a single decode stream here.
    c->ws_reset();
    DecBufs b;
    SAMPT_TRY(alloc_dec_bufs(c, &b, w.n_out_tok + K + 2, G * G));
    int *bbox, *skip; float* box;
    SAMPT_TRY(ws_get(c, &bbox, 8, "bbox"));
    SAMPT_TRY(ws_get(c, &skip, 1, "skip"));
    SAMPT_TRY(ws_get(c, &box, 4, "box"));
    RefinePtrs p{feat_tok, coords, labels, pos_coords, pos_labels, logits, iou, low_res, n_refine_done, bbox, skip, box};
    p.hq_feat = w.hq ? c->hq_feat : nullptr;
    return enqueue_refine_chain(c, st, w, b, s, p);
  }
  const bool hq = w.hq && c->hq_feat != nullptr;
  const int GG = G * G;
  // graph_slot: independent buffer sets / graph instances so that several frames' chains can replay CONCURRENTLY on
  // different streams (each chain is a long sequence of tiny kernels: latency-, not throughput-bound).  Contract: all calls
  // with the same slot are issued on the same stream.
  SlotBufs* sb = nullptr;
  for (int attempt = 0; attempt < 2 && sb == nullptr; ++attempt) {
    auto sit = c->dec_slots.find(graph_slot);
    if (sit != c->dec_slots.end()) {
      sb = reinterpret_cast<SlotBufs*>(sit->second);
      if (sb->Kcap < K || sb->GG != GG || sb->HW < H * W || sb->hq != hq || sb->n_out_tok != w.n_out_tok) {
        SAMPT_TRY(dec_evict_all(c));   // the slot's buffers do not fit this call: re-carve everything
        sb = nullptr;
        continue;
      }
    } else {
      const int Kcap = std::max(DEC_KCAP_MIN, ((K + 63) / 64) * 64);
      int rc = carve_slot(c, w, s, hq, Kcap, &sb);
      if (rc == -3 && attempt == 0 && !c->dec_slots.empty()) { SAMPT_TRY(dec_evict_all(c)); sb = nullptr; continue; }
      if (rc != 0) return rc;
      c->dec_slots[graph_slot] = sb;
    }
  }
  SAMPT_CHECK(sb != nullptr, "decoder slab (%zu bytes) too small for slot %d (K=%d, %dx%d)", c->dec_bytes, graph_slot, K, H, W);
  std::vector<int> key{G, K, s.npos, s.two_pass, n_refine, in_h, in_w, H, W, w.n_out_tok, hq ? 1 : 0, graph_slot};
  RefineGraph* g = nullptr;
  auto it = c->graph_cache.find(key);
  if (it == c->graph_cache.end()) {
    if (c->graph_cache.size() >= DEC_MAX_GRAPHS) {   // bound the number of instantiated graphs: start over
      SAMPT_TRY(dec_evict_all(c));
      return sampt_sam_predict_refine(ctx, feat_tok, G, coords, labels, K, pos_coords, pos_labels, n_pos_first, n_refine, in_h, in_w, H,
                                      W, logits, iou, low_res, n_refine_done, graph_slot, stream);
    }
    // weights may not change between capture and replay: the cache is dropped by sampt_ctx_set_decoder_workspace,
    // which the Python side calls whenever SAM's decoder weights are (re)registered
    SAMPT_TRY(build_refine_graph(c, w, s, sb, &g));
    c->graph_cache[key] = g;
  } else {
    g = reinterpret_cast<RefineGraph*>(it->second);
  }
  SAMPT_CUDA(cudaMemcpyAsync(sb->feat, feat_tok, (size_t)GG * 256 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  SAMPT_CUDA(cudaMemcpyAsync(sb->coords, coords, (size_t)K * 2 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  SAMPT_CUDA(cudaMemcpyAsync(sb->labels, labels, (size_t)K * sizeof(int), cudaMemcpyDeviceToDevice, st));
  if (s.npos > 0) {
    SAMPT_CUDA(cudaMemcpyAsync(sb->pos_coords, pos_coords, (size_t)s.npos * 2 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    SAMPT_CUDA(cudaMemcpyAsync(sb->pos_labels, pos_labels, (size_t)s.npos * sizeof(int), cudaMemcpyDeviceToDevice, st));
  }
  if (hq) SAMPT_CUDA(cudaMemcpyAsync(sb->hqfeat, c->hq_feat, (size_t)16 * GG * 32 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  SAMPT_CUDA(cudaGraphLaunch(g->exec, st));
  c->launches += g->launches;
  SAMPT_CUDA(cudaMemcpyAsync(logits, sb->logits, (size_t)H * W * sizeof(float), cudaMemcpyDeviceToDevice, st));
  SAMPT_CUDA(cudaMemcpyAsync(iou, sb->iou, sizeof(float), cudaMemcpyDeviceToDevice, st));
  SAMPT_CUDA(cudaMemcpyAsync(low_res, sb->low, (size_t)16 * GG * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (n_refine_done) SAMPT_CUDA(cudaMemcpyAsync(n_refine_done, sb->n_done, sizeof(int), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// HQ-SAM: per-frame `hq_features` = embedding_encoder(image_embeddings) + compress_vit_feat(interm_embeddings[0])
// (MaskDecoderHQ.predict_masks prologue).  feat_tok [G*G,256], interm_tok [G*G,vit_dim] (output of the first global
// attention block, token-major) -> out [16*G*G][32] channels-last low-res map.
extern "C" int sampt_sam_hq_features(sampt_ctx* ctx, const float* feat_tok, const float* interm_tok, int G, float* scratch,
                                     float* out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DecW w;
  SAMPT_TRY(load_dec(c, &w));
  SAMPT_CHECK(w.hq, "sampt_sam_hq_features: the registered mask decoder is not an HQ decoder");
  SAMPT_CHECK(scratch != nullptr, "sampt_sam_hq_features: caller-owned scratch of G*G*1280 floats is required");
  const int GG = G * G;
  // caller-owned scratch (NOT the shared ctx workspace): frames are decoded concurrently on several streams
  float* e1 = scratch;
  float* c1 = scratch + (size_t)GG * 256;
  SAMPT_TRY(sgemm_nt(c, st, feat_tok, 256, w.enc0_w, 256, w.enc0_b4, nullptr, 0, e1, 256, GG, 256, 256, 0));
  SAMPT_TRY(sgemm_nt(c, st, interm_tok, w.vit_dim, w.cv0_w, w.vit_dim, w.cv0_b4, nullptr, 0, c1, 1024, GG, 1024, w.vit_dim, 0));
  hq_features_kernel<<<cdiv(16 * GG, 256), 256, 0, st>>>(e1, c1, w.enc_lnw, w.enc_lnb, w.enc3_w, w.enc3_b, w.cv_lnw, w.cv_lnb, w.cv3_w,
                                                        w.cv3_b, out, G);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}
// Select the HQ features used by subsequent sampt_sam_predict / sampt_sam_predict_refine calls (NULL = plain SAM masks).
extern "C" int sampt_sam_set_hq_features(sampt_ctx* ctx, const float* hq_features) {
  reinterpret_cast<Ctx*>(ctx)->hq_feat = hq_features;
  return 0;
}

// ---- unit-test entries: one decoder stage on caller buffers, through the same launchers as the decode chain -------------------
extern "C" int sampt_test_sam_attention(sampt_ctx* ctx, int kind, const float* q, const float* k, const float* v, float* out, int T,
                                        int Nk, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(T >= 1 && Nk >= 1, "sampt_test_sam_attention: T (%d) and Nk (%d) must be positive", T, Nk);
  switch (kind) {
    case 0:
    case 1:
      SAMPT_CHECK(Nk == T, "sampt_test_sam_attention: token self-attention needs Nk == T (got %d, %d)", Nk, T);
      return launch_tok_self(c, st, kind, q, k, v, out, T, nullptr);
    case 2: {
      c->ws_reset();
      float* part;
      SAMPT_TRY(ws_get(c, &part, (size_t)T * 8 * ((Nk + 255) / 256) * 18, "attention partials"));
      return launch_t2i(c, st, q, k, v, part, out, T, Nk, nullptr);
    }
    case 3:
      return launch_i2t(c, st, q, k, v, out, Nk, T, nullptr);
    default:
      set_error("sampt_test_sam_attention: unknown kind %d", kind);
      return -2;
  }
}

extern "C" int sampt_test_sam_prompt(sampt_ctx* ctx, const float* feat_tok, int G, const float* coords, const int* labels, int K,
                                     const float* box, const float* mask_in, float* tokens_out, float* src_out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  DecW w;
  SAMPT_TRY(load_dec(c, &w));
  DecodeCall d{};
  d.feat_tok = feat_tok; d.coords = coords; d.labels = labels; d.K = K; d.box = box; d.use_box = box ? 1 : 0; d.mask_in = mask_in;
  return encode_prompt(c, reinterpret_cast<cudaStream_t>(stream), w, d, G, tokens_out, src_out);
}

extern "C" int sampt_test_sam_upscale(sampt_ctx* ctx, const float* u1, const float* hyper, int n_masks, int G, float* low_res,
                                      float* u_out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_CHECK(n_masks >= 1 && n_masks <= 4, "sampt_test_sam_upscale: n_masks %d out of [1, 4]", n_masks);
  DecW w;
  SAMPT_TRY(load_dec(c, &w));
  return launch_upscale(c, reinterpret_cast<cudaStream_t>(stream), w, u1, hyper, n_masks, low_res, G, u_out, nullptr);
}

extern "C" int sampt_test_sam_postprocess(sampt_ctx* ctx, const float* low_res, int n_masks, int G, int in_h, int in_w, int H, int W,
                                          float* out, int* bbox5, float* box4, int* skip, int* n_done, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  c->ws_reset();
  int* acc;   // the chain's accumulator; refine_ctl_kernel resets it, so the caller gets a copy taken before that
  SAMPT_TRY(ws_get(c, &acc, 8, "bbox"));
  init_ctl_kernel<<<1, 1, 0, st>>>(acc, skip, n_done);
  LAUNCH_OK();
  SAMPT_TRY(launch_postprocess(c, st, low_res, n_masks, G, in_h, in_w, H, W, out, acc, nullptr));
  SAMPT_CUDA(cudaMemcpyAsync(bbox5, acc, 5 * sizeof(int), cudaMemcpyDeviceToDevice, st));
  refine_ctl_kernel<<<1, 1, 0, st>>>(acc, box4, skip, n_done);
  LAUNCH_OK();
  return 0;
}
