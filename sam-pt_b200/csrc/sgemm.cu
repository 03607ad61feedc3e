// FP32 CUDA-core GEMM  Y[M,N] = act(X[M,K] . W[N,K]^T + bias) (+ residual)   -- the strict-fp32 path.
//
// Used where the reference's numerics must be kept at float32 (PIPS MLP-Mixer: the 1e-3 px tolerance with a
// 6-iteration feedback loop, SURVEY §7 "parity under chaos"; SAM prompt/mask decoder: 12 mask->box->mask
// refinement iterations).  Tensor-core GEMMs (wgmma) live in gemm_tc.cu and serve the ViT encoder.
#include <cooperative_groups.h>
#include <cstdlib>

#include "common.cuh"
#include "kernels.cuh"

namespace sampt {

// Small-M variant (M <= MAXM rows, e.g. the prompt tokens of the mask decoder or the N*S rows of the PIPS mixer):
// weight-bandwidth bound, so the grid is spread over the N (output column) axis and every weight row is read exactly once,
// coalesced.  One warp = one output column x all M rows; lanes split K (float4 per lane per step); X is staged through
// shared memory in K chunks of 128; a warp-shuffle reduction per row finishes the dot products.
template <int MAXM>
__global__ void __launch_bounds__(256)
sgemm_smallm_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ W, int ldw, const float* __restrict__ bias,
                    const float* residual, int ldr, float* Y, int ldy, int M, int N, int K, int act, const int* skip) {
  if (skip != nullptr && *skip != 0) return;
  constexpr int KC = 128;
  __shared__ __align__(16) float xs[MAXM][KC];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + warp;
  float acc[MAXM];
#pragma unroll
  for (int m = 0; m < MAXM; ++m) acc[m] = 0.f;
  for (int k0 = 0; k0 < K; k0 += KC) {
    // the weight row does not depend on the staged X tile: issue its load first so both latencies overlap
    const int kk = k0 + lane * 4;
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n < N && kk < K) w = __ldg(reinterpret_cast<const float4*>(W + (size_t)n * ldw + kk));
    __syncthreads();
    for (int i = threadIdx.x; i < MAXM * (KC / 4); i += 256) {
      int m = i / (KC / 4), c = (i % (KC / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < M && k0 + c < K) v = *reinterpret_cast<const float4*>(X + (size_t)m * ldx + k0 + c);
      *reinterpret_cast<float4*>(&xs[m][c]) = v;
    }
    __syncthreads();
    if (n < N) {
#pragma unroll
      for (int m = 0; m < MAXM; ++m) {
        float4 x = *reinterpret_cast<const float4*>(&xs[m][lane * 4]);
        acc[m] = fmaf(w.x, x.x, acc[m]);
        acc[m] = fmaf(w.y, x.y, acc[m]);
        acc[m] = fmaf(w.z, x.z, acc[m]);
        acc[m] = fmaf(w.w, x.w, acc[m]);
      }
    }
  }
  if (n >= N) return;
#pragma unroll
  for (int m = 0; m < MAXM; ++m) {
    float v = warp_sum(acc[m]);
    if (lane == (m & 31) && m < M) {
      if (bias) v += bias[n];
      if (act == 1) v = gelu_erf(v);
      else if (act == 2) v = fmaxf(v, 0.f);
      else if (act == 3) v = gelu_tanh(v);
      if (residual) v += residual[(size_t)m * ldr + n];
      Y[(size_t)m * ldy + n] = v;
    }
  }
}

// cp.async multi-stage FP32 GEMM.  The shapes on this path (PIPS mixer: 64 rows; mask decoder: 4096 x {128,256} outputs
// with K = 128..2048) launch only ~30-250 CTAs, i.e. at most one or two per SM, so a kernel that loads a k-tile, waits,
// computes, waits again is bound by global-memory LATENCY (measured: 15-60 us for 0.1-0.3 GFLOP).  Here every thread keeps
// STAGES-1 k-tiles (BK = 32) in flight with cp.async (16 B, zero-fill on the K / M / N tails), and the shared-memory tiles
// are k-contiguous with a 36-float pitch + strided row ownership (row = ty + 16*i) so that the float4 operand reads are
// bank-conflict free.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N_>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N_) : "memory"); }

template <int BM, int BN, int TM, int TN, int STAGES>
__global__ void __launch_bounds__(256)
sgemm_pipe_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ W, int ldw, const float* __restrict__ bias,
                  const float* residual, int ldr, float* Y, int ldy, int M, int N, int K, int act, const int* skip) {
  if (skip != nullptr && *skip != 0) return;
  constexpr int BK = 32, PITCH = BK + 4;
  static_assert(BM / TM == 16 && BN / TN == 16, "16x16 thread layout");
  extern __shared__ __align__(16) float smem_f[];
  float* As = smem_f;                               // [STAGES][BM][PITCH]
  float* Bs = smem_f + (size_t)STAGES * BM * PITCH;  // [STAGES][BN][PITCH]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int nk = (K + BK - 1) / BK;

  auto issue = [&](int kt) {
    if (kt < nk) {
      const int st = kt % STAGES, k0 = kt * BK;
      float* as = As + (size_t)st * BM * PITCH;
      float* bs = Bs + (size_t)st * BN * PITCH;
      for (int i = tid; i < BM * (BK / 4); i += 256) {
        const int r = i / (BK / 4), c = (i % (BK / 4)) * 4;
        const bool ok = (m0 + r < M) && (k0 + c < K);
        cp_async16(as + r * PITCH + c, ok ? (X + (size_t)(m0 + r) * ldx + k0 + c) : X, ok);
      }
      for (int i = tid; i < BN * (BK / 4); i += 256) {
        const int r = i / (BK / 4), c = (i % (BK / 4)) * 4;
        const bool ok = (n0 + r < N) && (k0 + c < K);
        cp_async16(bs + r * PITCH + c, ok ? (W + (size_t)(n0 + r) * ldw + k0 + c) : W, ok);
      }
    }
    cp_async_commit();
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) issue(s);
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    issue(kt + STAGES - 1);  // refills the stage consumed in the previous iteration
    const float* as = As + (size_t)(kt % STAGES) * BM * PITCH;
    const float* bs = Bs + (size_t)(kt % STAGES) * BN * PITCH;
#pragma unroll
    for (int k = 0; k < BK; k += 4) {
      float4 a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = *reinterpret_cast<const float4*>(as + (ty + 16 * i) * PITCH + k);
#pragma unroll
      for (int j = 0; j < TN; ++j) b[j] = *reinterpret_cast<const float4*>(bs + (tx + 16 * j) * PITCH + k);
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) {
          acc[i][j] = fmaf(a[i].x, b[j].x, acc[i][j]);
          acc[i][j] = fmaf(a[i].y, b[j].y, acc[i][j]);
          acc[i][j] = fmaf(a[i].z, b[j].z, acc[i][j]);
          acc[i][j] = fmaf(a[i].w, b[j].w, acc[i][j]);
        }
    }
  }
  cp_async_wait<0>();
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int gm = m0 + ty + 16 * i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int gn = n0 + tx + 16 * j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[gn];
      if (act == 1) v = gelu_erf(v);
      else if (act == 2) v = fmaxf(v, 0.f);
      else if (act == 3) v = gelu_tanh(v);
      if (residual) v += residual[(size_t)gm * ldr + gn];
      Y[(size_t)gm * ldy + gn] = v;
    }
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// Skinny GEMM for M <= 64 rows (the N*S = 64 rows of the PIPS MLP-Mixer at 8 points: 1296 GEMMs per C2 clip on the tracker's
// serial chain).  The pipelined kernel above gives such a shape 32-128 CTAs that each walk the whole K in 32-wide tiles with a
// barrier per tile: 25-85 us for 0.13 GFLOP, bound by the length of that loop.  Here every CTA owns a BM x 32 output tile and
// ONE K chunk of <= 256: the whole chunk of X and W (<= 96 KB) is requested with cp.async at once (four commit groups, consumed
// as they land), so a CTA pays one memory round trip; K is split over a thread-block CLUSTER of KS = 1/2/4/8 CTAs whose partial
// tiles are summed through distributed shared memory in fixed rank order (deterministic: no atomics), rank r finishing rows
// [r*BM/KS, (r+1)*BM/KS) with bias / activation / residual.  128 CTAs for both mixer shapes (2048 x 512: 64 tiles x 2;
// 512 x 2048: 16 tiles x 8); FMA-issue bound at ~2.4 us per CTA.
// Shared-memory layout: k-contiguous rows with a (KC + 4)-float pitch; thread (rg, cg) owns rows rg + 16 i and columns cg + 16 j,
// which makes the float4 operand reads of a warp conflict free.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int SK_BN = 32, SK_KC = 256, SK_SUB = 64, SK_PITCH = SK_KC + 4;

template <int BM>
__global__ void __launch_bounds__(256)
sgemm_skinny_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ W, int ldw, const float* __restrict__ bias,
                    const float* residual, int ldr, float* Y, int ldy, int M, int N, int K, int kc, int act, const int* skip) {
  if (skip != nullptr && *skip != 0) return;   // uniform over the grid: no CTA reaches a cluster barrier
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  constexpr int TM = BM / 16;
  extern __shared__ __align__(16) float smem_f[];
  float* As = smem_f;                          // [BM][SK_PITCH]
  float* Bs = smem_f + (size_t)BM * SK_PITCH;  // [SK_BN][SK_PITCH]
  const int tid = threadIdx.x, cgp = tid & 15, rg = tid >> 4;
  const int n0 = blockIdx.x * SK_BN;
  const int KS = gridDim.y, rank = blockIdx.y;   // cluster dims (1, KS, 1): blockIdx.y is the rank inside the cluster
  // taller problems (up to a few hundred rows: the mask decoder's token side with 256 query points) run as blockIdx.z row blocks
  const int mz = blockIdx.z * BM;
  X += (size_t)mz * ldx;
  M = min(BM, M - mz);
  const int k_begin = rank * kc;
  const int nsub = (min(kc, max(K - k_begin, 0)) + SK_SUB - 1) / SK_SUB;

  for (int sub = 0; sub < SK_KC / SK_SUB; ++sub) {
    if (sub < nsub) {
      const int kb = sub * SK_SUB;
      for (int i = tid; i < BM * (SK_SUB / 4); i += 256) {
        const int r = i / (SK_SUB / 4), c = kb + (i % (SK_SUB / 4)) * 4;
        const bool ok = r < M && k_begin + c < K && c < kc;
        cp_async16(As + r * SK_PITCH + c, ok ? (X + (size_t)r * ldx + k_begin + c) : X, ok);
      }
      for (int i = tid; i < SK_BN * (SK_SUB / 4); i += 256) {
        const int r = i / (SK_SUB / 4), c = kb + (i % (SK_SUB / 4)) * 4;
        const bool ok = n0 + r < N && k_begin + c < K && c < kc;
        cp_async16(Bs + r * SK_PITCH + c, ok ? (W + (size_t)(n0 + r) * ldw + k_begin + c) : W, ok);
      }
    }
    cp_async_commit();
  }

  float acc[TM][2];
#pragma unroll
  for (int i = 0; i < TM; ++i) acc[i][0] = acc[i][1] = 0.f;

#pragma unroll
  for (int sub = 0; sub < SK_KC / SK_SUB; ++sub) {
    if (sub == 0) cp_async_wait<3>();
    else if (sub == 1) cp_async_wait<2>();
    else if (sub == 2) cp_async_wait<1>();
    else cp_async_wait<0>();
    __syncthreads();
    if (sub < nsub) {
      const float* as = As + sub * SK_SUB;
      const float* bs = Bs + sub * SK_SUB;
#pragma unroll 4
      for (int k = 0; k < SK_SUB; k += 4) {
        float4 a[TM], b[2];
#pragma unroll
        for (int i = 0; i < TM; ++i) a[i] = *reinterpret_cast<const float4*>(as + (rg + 16 * i) * SK_PITCH + k);
#pragma unroll
        for (int j = 0; j < 2; ++j) b[j] = *reinterpret_cast<const float4*>(bs + (cgp + 16 * j) * SK_PITCH + k);
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            acc[i][j] = fmaf(a[i].x, b[j].x, acc[i][j]);
            acc[i][j] = fmaf(a[i].y, b[j].y, acc[i][j]);
            acc[i][j] = fmaf(a[i].z, b[j].z, acc[i][j]);
            acc[i][j] = fmaf(a[i].w, b[j].w, acc[i][j]);
          }
      }
    }
  }
  // partial tile -> this CTA's shared memory (over the dead A chunk), then the cluster sums the KS partials in rank order
  __syncthreads();
  float* P = smem_f;   // [BM][SK_BN + 1]
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) P[(rg + 16 * i) * (SK_BN + 1) + cgp + 16 * j] = acc[i][j];
  cluster.sync();
  const int rows_per = BM / KS;   // KS divides 16 <= BM
  for (int e = tid; e < rows_per * SK_BN; e += 256) {
    const int m = rank * rows_per + e / SK_BN, col = e % SK_BN, n = n0 + col;
    float v = 0.f;
    for (int s = 0; s < KS; ++s) v += cluster.map_shared_rank(P, s)[m * (SK_BN + 1) + col];
    if (m < M && n < N) {
      if (bias) v += bias[n];
      if (act == 1) v = gelu_erf(v);
      else if (act == 2) v = fmaxf(v, 0.f);
      else if (act == 3) v = gelu_tanh(v);
      if (residual) v += residual[(size_t)(mz + m) * ldr + n];
      Y[(size_t)(mz + m) * ldy + n] = v;
    }
  }
  cluster.sync();   // nobody leaves while a peer may still read its partial tile
}

template <int BM>
static int launch_skinny(cudaStream_t st, const float* X, int ldx, const float* W, int ldw, const float* bias, const float* residual,
                         int ldr, float* Y, int ldy, int M, int N, int K, int act, const int* skip, int num_sms) {
  // K split: chunks of <= 256 (multiples of 64), cluster size 1/2/4/8; prefer enough CTAs to cover the SMs
  const int n_tiles = cdiv(N, SK_BN), m_blocks = cdiv(M, BM);
  int ks = 1;
  while (ks < 8 && (cdiv(K, ks) > SK_KC || n_tiles * m_blocks * ks < num_sms / 2) && cdiv(K, 2 * ks) >= SK_SUB) ks *= 2;
  const int kc = cdiv(cdiv(K, ks), SK_SUB) * SK_SUB;
  if (kc > SK_KC) return 1;   // K > 2048: not a shape of this path
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(n_tiles, ks, m_blocks);
  cfg.blockDim = dim3(256, 1, 1);
  cfg.dynamicSmemBytes = (size_t)(BM + SK_BN) * SK_PITCH * sizeof(float);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = ks; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, sgemm_skinny_kernel<BM>, X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, kc, act, skip);
  return e == cudaSuccess ? 0 : 2;
}
static bool skinny_enabled() {
  static const int on = [] { const char* e = std::getenv("SAMPT_SGEMM_SKINNY"); return (e != nullptr && e[0] == '0') ? 0 : 1; }();
  return on != 0;
}

template <int BM, int BN, int TM, int TN, int STAGES>
static int launch_pipe(cudaStream_t st, const float* X, int ldx, const float* W, int ldw, const float* bias, const float* residual,
                       int ldr, float* Y, int ldy, int M, int N, int K, int act, const int* skip) {
  constexpr size_t smem = (size_t)STAGES * (BM + BN) * 36 * sizeof(float);
  // the dynamic shared-memory limit of every instantiation is raised per device by sgemm_init() (called from sampt_ctx_create)
  dim3 grid(cdiv(N, BN), cdiv(M, BM));
  sgemm_pipe_kernel<BM, BN, TM, TN, STAGES><<<grid, 256, smem, st>>>(X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, act, skip);
  return 0;
}

// set the dynamic shared-memory attributes once, outside of any stream capture (called from sampt_ctx_create)
int sgemm_init() {
  SAMPT_CUDA(cudaFuncSetAttribute(sgemm_pipe_kernel<64, 16, 4, 1, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * (64 + 16) * 36 * 4));
  SAMPT_CUDA(cudaFuncSetAttribute(sgemm_pipe_kernel<64, 64, 4, 4, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * (64 + 64) * 36 * 4));
  SAMPT_CUDA(cudaFuncSetAttribute(sgemm_pipe_kernel<128, 64, 8, 4, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 3 * (128 + 64) * 36 * 4));
  SAMPT_CUDA(cudaFuncSetAttribute(sgemm_skinny_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (64 + SK_BN) * SK_PITCH * 4));
  SAMPT_CUDA(cudaFuncSetAttribute(sgemm_skinny_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (32 + SK_BN) * SK_PITCH * 4));
  return 0;
}

int sgemm_nt(Ctx* c, cudaStream_t st, const float* X, int ldx, const float* W, int ldw, const float* bias,
             const float* residual, int ldr, float* Y, int ldy, int M, int N, int K, int act) {
  return sgemm_nt_skip(c, st, X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, act, nullptr);
}

int sgemm_nt_skip(Ctx* c, cudaStream_t st, const float* X, int ldx, const float* W, int ldw, const float* bias,
                  const float* residual, int ldr, float* Y, int ldy, int M, int N, int K, int act, const int* skip) {
  SAMPT_CHECK((K % 4) == 0 && (ldx % 4) == 0 && (ldw % 4) == 0, "sgemm_nt: K/ldx/ldw must be multiples of 4 (K=%d ldx=%d ldw=%d)", K, ldx, ldw);
  if (M <= 0 || N <= 0) return 0;
  if (M <= 16) {
    sgemm_smallm_kernel<16><<<cdiv(N, 8), 256, 0, st>>>(X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, act, skip);
  } else if (M <= 32) {
    sgemm_smallm_kernel<32><<<cdiv(N, 8), 256, 0, st>>>(X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, act, skip);
  } else if (M <= 64 || (M <= 512 && skinny_enabled() && K <= 8 * SK_KC)) {
    int rc = 1;
    if (skinny_enabled() && K <= 8 * SK_KC) rc = launch_skinny<64>(st, X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, act, skip, c->num_sms);
    SAMPT_CHECK(rc != 2, "sgemm_nt: cluster launch of the skinny kernel failed (%s)", cudaGetErrorString(cudaGetLastError()));
    if (rc == 1) SAMPT_TRY((launch_pipe<64, 16, 4, 1, 4>(st, X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, act, skip)));
  } else {
    // tile choice: the largest tile that still yields enough CTAs for 132 SMs
    const long long t128 = (long long)cdiv(M, 128) * cdiv(N, 64), t64 = (long long)cdiv(M, 64) * cdiv(N, 64);
    if (t128 >= 2 * c->num_sms) {
      SAMPT_TRY((launch_pipe<128, 64, 8, 4, 3>(st, X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, act, skip)));
    } else if (t64 >= c->num_sms / 2) {
      SAMPT_TRY((launch_pipe<64, 64, 4, 4, 4>(st, X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, act, skip)));
    } else {
      SAMPT_TRY((launch_pipe<64, 16, 4, 1, 4>(st, X, ldx, W, ldw, bias, residual, ldr, Y, ldy, M, N, K, act, skip)));
    }
  }
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

}  // namespace sampt
