// Interactive point correction (sam_pt/modeling/sam_pt_interactive.py): the per-frame work of the simulator that is not the
// SAM decoder itself.
//
//   J&F counts  davis2017-evaluation's db_eval_iou / db_eval_boundary reduced to eight exact integer counts per frame, for T
//               frames in one call.  P = logits > 0, G = gt != 0.
//                 jf_bmap_kernel     _seg2bmap of P and G (b = S^E | S^S | S^SE, last row S^E, last column S^S, corner 0) into
//                                    one byte per pixel (bit 0 = dP, bit 1 = dG); |P&G|, |P|G|, |P|, |G|, |dP|, |dG|
//                 jf_rowdist_kernel  per pixel, horizontal distance to the nearest dP / dG pixel of its row, capped at r + 1
//                 jf_match_kernel    cv2.dilate(., disk(r)) evaluated only where the other mask has boundary pixels: a dP pixel
//                                    at (y, x) is matched iff some row y+dy has a dG pixel within the disk's half-width at dy
//               The float64 J and F are formed from the counts on the host, exactly as numpy does.
//   categories  TP/TN/FP/FN of P against G sampled at the rounded (rint: half to even, as torch.round) point coordinates, and
//               the "correct" flag of the point given its label.
//   DBSCAN      sklearn.cluster.DBSCAN(eps, min_samples).fit(points).labels_ for integer-valued points:
//                 dbscan_count_kernel   neighbour counts (squared integer distance <= eps*eps in float64, self included)
//                 dbscan_union_kernel   union-find over core-core edges; a root is always linked under the SMALLER root, so the
//                                       final root of a component is its smallest core index whatever the scheduling
//                 dbscan_root_kernel    flatten
//                 dbscan_rank_kernel    cluster label of each root = number of smaller roots (clusters numbered in the order
//                                       sklearn's _dbscan_inner creates them)
//                 dbscan_label_kernel   core: its component's label; border: the smallest label among its core neighbours (the
//                                       first cluster to reach it in sklearn's expansion order); noise: -1
#include <algorithm>
#include <climits>

#include "common.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {

constexpr int JF_MAX_R = 64;           // r = ceil(0.008 * |(H, W)|) reaches 64 at ~8000 px of diagonal
constexpr int JF_MAX_W = 16384;        // one image row in shared memory (jf_rowdist_kernel)
constexpr int DB_MAX_N = 1 << 20;
constexpr int DB_TILE = 256;

// block-wide sum of NV per-thread ints, added to dst[0..NV) (unsigned long long) with one atomic each per block
template <int NV>
__device__ __forceinline__ void block_add(unsigned long long* dst, const unsigned (&v)[NV]) {
  __shared__ unsigned s[NV];
  if (threadIdx.x < NV) s[threadIdx.x] = 0;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const unsigned w = __reduce_add_sync(0xffffffffu, v[k]);
    if ((threadIdx.x & 31) == 0 && w) atomicAdd(&s[k], w);
  }
  __syncthreads();
  if (threadIdx.x < NV && s[threadIdx.x]) atomicAdd(dst + threadIdx.x, (unsigned long long)s[threadIdx.x]);
}

__global__ void __launch_bounds__(256)
jf_bmap_kernel(const float* __restrict__ logits, const uint8_t* __restrict__ gt, int H, int W, uint8_t* __restrict__ bm,
               unsigned long long* __restrict__ counts) {
  const int t = blockIdx.y;
  const long long HW = (long long)H * W;
  const float* lg = logits + t * HW;
  const uint8_t* g = gt + t * HW;
  uint8_t* b = bm + t * HW;
  unsigned v[6] = {0, 0, 0, 0, 0, 0};
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < HW; idx += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(idx / W), x = (int)(idx - (long long)y * W);
    const bool has_e = x + 1 < W, has_s = y + 1 < H;
    const unsigned p = lg[idx] > 0.f, q = g[idx] != 0;
    const unsigned pe = has_e ? lg[idx + 1] > 0.f : 0u, qe = has_e ? g[idx + 1] != 0 : 0u;
    const unsigned ps = has_s ? lg[idx + W] > 0.f : 0u, qs = has_s ? g[idx + W] != 0 : 0u;
    const unsigned pse = has_e && has_s ? lg[idx + W + 1] > 0.f : 0u, qse = has_e && has_s ? g[idx + W + 1] != 0 : 0u;
    unsigned bp, bq;
    if (!has_e && !has_s) {
      bp = bq = 0;
    } else if (!has_s) {           // last row
      bp = p ^ pe;
      bq = q ^ qe;
    } else if (!has_e) {           // last column
      bp = p ^ ps;
      bq = q ^ qs;
    } else {
      bp = (p ^ pe) | (p ^ ps) | (p ^ pse);
      bq = (q ^ qe) | (q ^ qs) | (q ^ qse);
    }
    b[idx] = (uint8_t)(bp | (bq << 1));
    v[0] += p & q;
    v[1] += p | q;
    v[2] += p;
    v[3] += q;
    v[4] += bp;
    v[5] += bq;
  }
  block_add<6>(counts + t * 8, v);
}

// one CTA per (row, frame); out[x] = dP | dG << 8, each the distance to the nearest boundary pixel of the row, capped at r + 1
__global__ void __launch_bounds__(256)
jf_rowdist_kernel(const uint8_t* __restrict__ bm, int H, int W, int r, uint16_t* __restrict__ hd) {
  extern __shared__ uint8_t row[];
  const int y = blockIdx.x, t = blockIdx.y;
  const long long off = ((long long)t * H + y) * W;
  for (int x = threadIdx.x; x < W; x += blockDim.x) row[x] = bm[off + x];
  __syncthreads();
  for (int x = threadIdx.x; x < W; x += blockDim.x) {
    int dp = r + 1, dq = r + 1;
    for (int d = 0; d <= r && (dp > r || dq > r); ++d) {
      const uint8_t a = x - d >= 0 ? row[x - d] : 0, c = x + d < W ? row[x + d] : 0;
      const uint8_t m = a | c;
      if ((m & 1) && dp > r) dp = d;
      if ((m & 2) && dq > r) dq = d;
    }
    hd[off + x] = (uint16_t)(dp | (dq << 8));
  }
}

__global__ void __launch_bounds__(256)
jf_match_kernel(const uint8_t* __restrict__ bm, const uint16_t* __restrict__ hd, int H, int W, int r,
                unsigned long long* __restrict__ counts) {
  __shared__ int half[2 * JF_MAX_R + 1];     // half[dy + r] = largest k with k^2 + dy^2 <= r^2 (skimage.morphology.disk)
  for (int i = threadIdx.x; i <= 2 * r; i += blockDim.x) {
    const int dy = i - r;
    int k = 0;
    while ((k + 1) * (k + 1) + dy * dy <= r * r) ++k;
    half[i] = k;
  }
  __syncthreads();
  const int t = blockIdx.y;
  const long long HW = (long long)H * W;
  const uint8_t* b = bm + t * HW;
  const uint16_t* h = hd + t * HW;
  unsigned v[2] = {0, 0};       // fg_match = |dP & dil(dG)|, gt_match = |dG & dil(dP)|
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < HW; idx += (long long)gridDim.x * blockDim.x) {
    const uint8_t m = b[idx];
    if (!m) continue;
    const int y = (int)(idx / W), x = (int)(idx - (long long)y * W);
    bool fp = !(m & 1), gp = !(m & 2);          // "already decided" for the bits this pixel does not carry
    const int y0 = max(0, y - r), y1 = min(H - 1, y + r);
    for (int yy = y0; yy <= y1 && !(fp && gp); ++yy) {
      const uint16_t d = h[(long long)yy * W + x];
      const int hw = half[yy - y + r];
      if (!fp && (d >> 8) <= hw) fp = true, ++v[0];
      if (!gp && (d & 0xff) <= hw) gp = true, ++v[1];
    }
  }
  block_add<2>(counts + t * 8 + 6, v);
}

__global__ void __launch_bounds__(128)
point_categories_kernel(const float* __restrict__ logits, const uint8_t* __restrict__ gt, int H, int W, const float* __restrict__ xy,
                        const int* __restrict__ labels, int n, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int x = __float2int_rn(xy[2 * i]), y = __float2int_rn(xy[2 * i + 1]);
  if (x < 0) x += W;          // Python indexing: a negative index counts from the end
  if (y < 0) y += H;
  if (x < 0 || x >= W || y < 0 || y >= H) {
    out[i] = -1;
    return;
  }
  const long long idx = (long long)y * W + x;
  const bool p = logits[idx] > 0.f, g = gt[idx] != 0;
  const bool tp = p && g, tn = !p && !g, fp = p && !g, fn = !p && g;
  const bool positive = labels[i] == 1;
  const bool correct = positive ? (tp || fn) : (tn || fp);
  out[i] = (int)tp | ((int)tn << 1) | ((int)fp << 2) | ((int)fn << 3) | ((int)correct << 4);
}

// ------------------------------------------------------------------------------------------------------------- DBSCAN
__device__ __forceinline__ int2 db_point(const float* pts, int j) {
  return make_int2(__float2int_rn(pts[2 * j]), __float2int_rn(pts[2 * j + 1]));
}
__device__ __forceinline__ bool db_near(int2 a, int2 b, double eps2) {
  const long long dy = a.x - b.x, dx = a.y - b.y;
  return (double)(dy * dy + dx * dx) <= eps2;
}

__global__ void __launch_bounds__(DB_TILE)
dbscan_count_kernel(const float* __restrict__ pts, int n, double eps2, int min_samples, int* __restrict__ core,
                    int* __restrict__ parent) {
  __shared__ int2 tile[DB_TILE];
  const int i = blockIdx.x * DB_TILE + threadIdx.x;
  const int2 a = i < n ? db_point(pts, i) : make_int2(0, 0);
  int cnt = 0;
  for (int j0 = 0; j0 < n; j0 += DB_TILE) {
    __syncthreads();
    if (j0 + threadIdx.x < n) tile[threadIdx.x] = db_point(pts, j0 + threadIdx.x);
    __syncthreads();
    const int m = min(DB_TILE, n - j0);
    for (int k = 0; k < m; ++k) cnt += db_near(a, tile[k], eps2);
  }
  if (i < n) {
    core[i] = cnt >= min_samples;
    parent[i] = i;
  }
}

__device__ __forceinline__ int uf_find(volatile int* p, int x) {
  int nx;
  while ((nx = p[x]) != x) {   // path halving; a parent only ever moves to a smaller ancestor, so the race is benign
    const int nnx = p[nx];
    if (nnx != nx) p[x] = nnx;
    x = nx;
  }
  return x;
}

__device__ void uf_unite(int* p, int a, int b) {
  volatile int* vp = p;
  int ra = uf_find(vp, a), rb = uf_find(vp, b);
  while (ra != rb) {
    if (ra > rb) { const int s = ra; ra = rb; rb = s; }
    const int old = atomicCAS(&p[rb], rb, ra);     // link the larger root under the smaller one
    if (old == rb) break;
    rb = uf_find(vp, old);
    ra = uf_find(vp, ra);
  }
}

__global__ void __launch_bounds__(DB_TILE)
dbscan_union_kernel(const float* __restrict__ pts, int n, double eps2, const int* __restrict__ core, int* parent) {
  __shared__ int2 tile[DB_TILE];
  __shared__ int tcore[DB_TILE];
  const int i = blockIdx.x * DB_TILE + threadIdx.x;
  const bool ci = i < n && core[i];
  const int2 a = i < n ? db_point(pts, i) : make_int2(0, 0);
  for (int j0 = blockIdx.x * DB_TILE; j0 < n; j0 += DB_TILE) {    // pairs j > i only: earlier tiles hold no such j
    __syncthreads();
    if (j0 + threadIdx.x < n) {
      tile[threadIdx.x] = db_point(pts, j0 + threadIdx.x);
      tcore[threadIdx.x] = core[j0 + threadIdx.x];
    }
    __syncthreads();
    if (!ci) continue;
    const int m = min(DB_TILE, n - j0);
    for (int k = max(0, i + 1 - j0); k < m; ++k)
      if (tcore[k] && db_near(a, tile[k], eps2)) uf_unite(parent, i, j0 + k);
  }
}

__global__ void dbscan_root_kernel(int n, const int* __restrict__ core, int* parent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && core[i]) parent[i] = uf_find(parent, i);
}

// rank[i] = number of component roots (core i with parent[i] == i) before i; one CTA of 1024 threads
__global__ void __launch_bounds__(1024)
dbscan_rank_kernel(int n, const int* __restrict__ core, const int* __restrict__ parent, int* __restrict__ rank) {
  __shared__ int s[1024];
  const int per = (n + 1023) / 1024;
  const int lo = threadIdx.x * per, hi = min(n, lo + per);
  int c = 0;
  for (int i = lo; i < hi; ++i) c += core[i] && parent[i] == i;
  s[threadIdx.x] = c;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {        // inclusive Hillis-Steele scan
    const int add = threadIdx.x >= o ? s[threadIdx.x - o] : 0;
    __syncthreads();
    s[threadIdx.x] += add;
    __syncthreads();
  }
  int base = s[threadIdx.x] - c;
  for (int i = lo; i < hi; ++i) {
    rank[i] = base;
    base += core[i] && parent[i] == i;
  }
}

__global__ void __launch_bounds__(DB_TILE)
dbscan_label_kernel(const float* __restrict__ pts, int n, double eps2, const int* __restrict__ core,
                    const int* __restrict__ parent, const int* __restrict__ rank, int* __restrict__ labels) {
  __shared__ int2 tile[DB_TILE];
  __shared__ int troot[DB_TILE];              // root of a core point, INT_MAX for a non-core point
  const int i = blockIdx.x * DB_TILE + threadIdx.x;
  const bool ci = i < n && core[i];
  const int2 a = i < n ? db_point(pts, i) : make_int2(0, 0);
  int root = ci ? parent[i] : INT_MAX;
  for (int j0 = 0; j0 < n; j0 += DB_TILE) {
    __syncthreads();
    if (j0 + threadIdx.x < n) {
      tile[threadIdx.x] = db_point(pts, j0 + threadIdx.x);
      troot[threadIdx.x] = core[j0 + threadIdx.x] ? parent[j0 + threadIdx.x] : INT_MAX;
    }
    __syncthreads();
    if (ci || i >= n) continue;
    const int m = min(DB_TILE, n - j0);
    for (int k = 0; k < m; ++k)
      if (troot[k] < root && db_near(a, tile[k], eps2)) root = troot[k];
  }
  if (i < n) labels[i] = root == INT_MAX ? -1 : rank[root];
}

}  // namespace sampt

using namespace sampt;

extern "C" int sampt_jf_counts(sampt_ctx* ctx, const float* logits, const uint8_t* gt, int T, int H, int W, int radius,
                               uint8_t* scratch, long long* counts, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(T >= 1 && H >= 1 && W >= 1 && W <= JF_MAX_W && T <= 65535 && H <= 65535,
              "sampt_jf_counts: T=%d H=%d W=%d outside [1,65535] x [1,65535] x [1,%d]", T, H, W, JF_MAX_W);
  SAMPT_CHECK(radius >= 0 && radius <= JF_MAX_R, "sampt_jf_counts: radius %d outside [0, %d]", radius, JF_MAX_R);
  const long long HW = (long long)H * W;
  uint8_t* bm = scratch;
  uint16_t* hd = reinterpret_cast<uint16_t*>(scratch + ((T * HW + 1) & ~1LL));
  unsigned long long* cnt = reinterpret_cast<unsigned long long*>(counts);
  SAMPT_CUDA(cudaMemsetAsync(cnt, 0, sizeof(long long) * 8 * T, st));
  const unsigned nb = (unsigned)std::min<long long>(cdiv(HW, 256), 2 * c->num_sms);
  jf_bmap_kernel<<<dim3(nb, T), 256, 0, st>>>(logits, gt, H, W, bm, cnt);
  jf_rowdist_kernel<<<dim3(H, T), 256, W, st>>>(bm, H, W, radius, hd);
  jf_match_kernel<<<dim3(nb, T), 256, 0, st>>>(bm, hd, H, W, radius, cnt);
  c->launches += 3;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

extern "C" int sampt_point_categories(sampt_ctx* ctx, const float* logits, const uint8_t* gt, int H, int W, const float* xy,
                                      const int* labels, int n, int* out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(H >= 1 && W >= 1 && n >= 0, "sampt_point_categories: H=%d W=%d n=%d", H, W, n);
  if (n == 0) return 0;
  point_categories_kernel<<<cdiv(n, 128), 128, 0, st>>>(logits, gt, H, W, xy, labels, n, out);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

extern "C" int sampt_dbscan(sampt_ctx* ctx, const float* pts, int n, double eps, int min_samples, int* labels, int* scratch,
                            void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(n >= 1 && n <= DB_MAX_N, "sampt_dbscan: n = %d outside [1, %d]", n, DB_MAX_N);
  SAMPT_CHECK(eps > 0.0, "sampt_dbscan: eps must be > 0 (got %g)", eps);
  const double eps2 = eps * eps;
  int* core = scratch;
  int* parent = scratch + n;
  int* rank = scratch + 2 * n;
  const unsigned nb = cdiv(n, DB_TILE);
  dbscan_count_kernel<<<nb, DB_TILE, 0, st>>>(pts, n, eps2, min_samples, core, parent);
  dbscan_union_kernel<<<nb, DB_TILE, 0, st>>>(pts, n, eps2, core, parent);
  dbscan_root_kernel<<<cdiv(n, 256), 256, 0, st>>>(n, core, parent);
  dbscan_rank_kernel<<<1, 1024, 0, st>>>(n, core, parent, rank);
  dbscan_label_kernel<<<nb, DB_TILE, 0, st>>>(pts, n, eps2, core, parent, rank, labels);
  c->launches += 5;
  SAMPT_LAUNCH_CHECK();
  return 0;
}
