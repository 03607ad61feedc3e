// Tensor-core GEMM for the SAM ViT encoder:  C[M,N] = epilogue( A[M,K] . B[N,K]^T ),  fp16/bf16 operands, fp32 accumulate.
//
// sm_90a design (one CTA per 128x128 output tile, 288 threads, TWO CTAs per SM):
//   warp 8          TMA producer : cp.async.bulk.tensor 2-D boxes (64 halves x rows, 128B swizzle) into a 3-stage smem ring,
//                                  completion on per-stage mbarriers
//   warpgroups 0,1  consumers    : wgmma.mma_async m64n128 (k16 fp16/bf16, k32 e4m3) on 64 rows each, fp32 accumulators in
//                                  registers, one k-block in flight; then bias / GELU / residual / fp16|fp32|split store
// Two resident CTAs (97 KB of shared memory and <= 112 registers per thread each) let one CTA's epilogue -- for the ViT's lin1
// the GELU and the fp16 + two e4m3 stores take as long as its MMAs -- run while the other CTA keeps the tensor pipe busy.
//
// "Split" precision (accuracy dial, DESIGN.md §precision): an operand x is carried as fp16 hi + fp16 lo
// (lo = fp16(x - hi)); the K loop then runs over up to three segments  A_hi.B_hi + A_lo.B_hi + A_hi.B_lo  accumulating
// into the same registers.  Segments are described by column offsets into the A / B matrices, so the kernel is the same.
// e4m3 segments (precision 6, tc_api.cuh) run FIRST, into the zeroed accumulator, and the fp16 segments after them: wgmma's
// fp8 accumulation does not keep full fp32 precision, which is harmless while the accumulator holds only the 2^-12-sized
// correction terms but would round away the low bits of the fp16 main product if that were already in it.  The fp16 wgmmas
// then add at fp32 on top.  gemm_tc() reorders the caller's segments so (the sum does not depend on the order); one register
// tile instead of two is what fits two CTAs on an SM.
#include "common.cuh"
#include "tc_common.cuh"
#include "kernels.cuh"
#include "tc_api.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {

using namespace tc;

constexpr int G_BM = 128, G_BN = 128, G_BK = 64, G_STAGES = 3;
constexpr int G_A_BYTES = G_BM * G_BK * 2;  // 16 KB
constexpr int G_B_BYTES = G_BN * G_BK * 2;  // 16 KB
constexpr int G_STAGE_BYTES = G_A_BYTES + G_B_BYTES;
constexpr int G_SMEM_BYTES = G_STAGES * G_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
constexpr int G_THREADS = 288;

__global__ void __launch_bounds__(G_THREADS, 2)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, int M, int N, int K,
               GemmSeg seg, GemmEpi ep) {
  if (ep.skip != nullptr && *ep.skip != 0) return;   // uniform over the grid
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + G_STAGES * G_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + G_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (N + G_BN - 1) / G_BN;
  const int m_blk = blockIdx.x / n_tiles, n_blk = blockIdx.x % n_tiles;
  // k-blocks of 128 bytes per operand row: 64 fp16 or 128 e4m3 elements
  int seg_kb[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) seg_kb[i] = i < seg.nseg ? (seg.f8[i] ? K / (2 * G_BK) : K / G_BK) : 0;

  if (threadIdx.x == 0) {
    for (int i = 0; i < G_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 256); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      uint32_t it = 0;
      for (int sg = 0; sg < seg.nseg; ++sg) {
        for (int kb = 0; kb < seg_kb[sg]; ++kb, ++it) {
          const int s = it % G_STAGES;
          const uint32_t ph = (it / G_STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          const int kk = kb * G_BK;   // in fp16 units of the tensor map (an e4m3 block is the same 128 bytes)
          uint8_t* sa = smem + s * G_STAGE_BYTES;
          mbar_expect_tx(&full_bar[s], G_STAGE_BYTES);
          tma_load_2d(sa, &tmA, &full_bar[s], seg.a_off[sg] + kk, m_blk * G_BM);
          tma_load_2d(sa + G_A_BYTES, &tmB, &full_bar[s], seg.b_off[sg] + kk, n_blk * G_BN);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumers: warpgroup g owns rows [64 g, 64 g + 64)
  const int g = warp >> 2, w = warp & 3;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  uint32_t it = 0;
  int prev_s = -1;
  for (int sg = 0; sg < seg.nseg; ++sg) {
    const bool f8 = seg.f8[sg] != 0;
    for (int kb = 0; kb < seg_kb[sg]; ++kb, ++it) {
      const int s = it % G_STAGES;
      mbar_wait(&full_bar[s], (it / G_STAGES) & 1);
      const uint32_t sa = smem_u32(smem + s * G_STAGE_BYTES);
      const uint64_t adesc = make_smem_desc_sw128(sa + g * 64 * 128);
      const uint64_t bdesc = make_smem_desc_sw128(sa + G_A_BYTES);
      wgmma_fence();
      if (f8) {
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n128k32_e4m3(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k));
      } else if (ep.is_bf16) {
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n128k16_bf16(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k));
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n128k16_f16(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k));
      }
      wgmma_commit();
      wgmma_wait<1>();   // the previous k-block's wgmmas have finished reading their stage
      if (prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
      prev_s = s;
    }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);

  // -------------------------------------------------------------- epilogue straight from the accumulator registers
  const float acc_scale = ep.acc_scale ? __ldg(ep.acc_scale) : 1.0f;
  const int c2 = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m_blk * G_BM + g * 64 + w * 16 + (lane >> 2) + 8 * h;
    if (m >= M) continue;
    long long drow = m;
    if (ep.rowmap) drow = ep.rowmap[m];
    if (drow < 0) continue;   // a padding row dropped by rowmap
#pragma unroll
    for (int i = 0; i < G_BN / 8; ++i) {
      const int n = n_blk * G_BN + 8 * i + c2;
      if (n >= N) continue;   // N % 8 == 0: the pair is in or out together
      float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
      v0 *= acc_scale; v1 *= acc_scale;
      if (ep.bias) { v0 += __ldg(ep.bias + n); v1 += __ldg(ep.bias + n + 1); }
      if (ep.act == 1) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
      else if (ep.act == 3) { v0 = gelu_tanh(v0); v1 = gelu_tanh(v1); }
      if (ep.out32) {
        float* o = ep.out32 + (size_t)drow * ep.ldc + n;
        if (ep.resid) {
          const long long rrow = ep.resid_mod > 0 ? (drow % ep.resid_mod) : drow;
          const float2 t = *reinterpret_cast<const float2*>(ep.resid + (size_t)rrow * ep.ldc + n);
          v0 += t.x; v1 += t.y;
        }
        *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
      } else if (ep.is_bf16) {
        *reinterpret_cast<__nv_bfloat162*>(ep.out16 + (size_t)drow * ep.ldc + n) = __floats2bfloat162_rn(v0, v1);
      } else {
        __half* o = ep.out16 + (size_t)drow * ep.ldc + n;
        const __half2 hv = __floats2half2_rn(v0, v1);
        *reinterpret_cast<__half2*>(o) = hv;
        const float2 hf = __half22float2(hv);
        if (ep.split_off > 0 && ep.out_f8) {
          // fp8 correction operands of the next GEMM (tc_api.cuh): remainder * 2^12 and value * 2^-3 as e4m3 bytes
          uint8_t* ob = reinterpret_cast<uint8_t*>(ep.out16 + (size_t)drow * ep.ldc + ep.split_off) + n;
          uint16_t l8, h8;
          asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(l8) : "f"((v1 - hf.y) * F8_LO_SCALE), "f"((v0 - hf.x) * F8_LO_SCALE));
          asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(h8) : "f"(v1 * F8_HI_SCALE), "f"(v0 * F8_HI_SCALE));
          *reinterpret_cast<uint16_t*>(ob) = l8;
          *reinterpret_cast<uint16_t*>(ob + ep.split_off) = h8;
        } else if (ep.split_off > 0) {
          *reinterpret_cast<__half2*>(o + ep.split_off) = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
        }
      }
    }
  }
}

// the shapes on which precision 6 runs its correction passes in e4m3 (the ViT's linear layers; other GEMMs keep three fp16
// passes): whole 128-element e4m3 k-blocks
bool gemm_f8c_applicable(int M, int N, int K) { return M >= 256 && N % 256 == 0 && K % (2 * G_BK) == 0; }

int gemm_tc(Ctx* c, cudaStream_t st, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const GemmSeg& seg,
            const GemmEpi& ep) {
  SAMPT_CHECK(K % G_BK == 0 && K > 0, "gemm_tc: K (%d) must be a positive multiple of %d", K, G_BK);
  SAMPT_CHECK(N % 32 == 0, "gemm_tc: N (%d) must be a multiple of 32", N);
  SAMPT_CHECK(seg.nseg >= 1 && seg.nseg <= 3, "gemm_tc: nseg out of range");
  SAMPT_CHECK((ep.out16 != nullptr) != (ep.out32 != nullptr), "gemm_tc: exactly one of out16/out32 must be set");
  SAMPT_CHECK(ep.ldc % 8 == 0, "gemm_tc: ldc must be a multiple of 8");
  SAMPT_CHECK(ep.act == 0 || ep.act == 1 || ep.act == 3, "gemm_tc: act %d is not 0 (none), 1 (GELU erf) or 3 (GELU tanh)", ep.act);
  const bool f8 = (seg.f8[0] | seg.f8[1] | seg.f8[2]) != 0;
  SAMPT_CHECK(!f8 || K % (2 * G_BK) == 0, "gemm_tc: e4m3 segments need K %% 128 == 0 (K = %d)", K);
  SAMPT_CHECK(!f8 || !ep.is_bf16, "gemm_tc: e4m3 segments go with fp16 operands");
  CUtensorMap tmA, tmB;
  // the A/B matrices may carry several K segments side by side (hi | lo): inner extent = lda / ldb
  SAMPT_TRY(make_tmap_2d_f16(&tmA, A, (uint64_t)lda, (uint64_t)M, (uint64_t)lda * 2, G_BK, G_BM));
  SAMPT_TRY(make_tmap_2d_f16(&tmB, B, (uint64_t)ldb, (uint64_t)N, (uint64_t)ldb * 2, G_BK, G_BN));
  const int m_tiles = (M + G_BM - 1) / G_BM, n_tiles = (N + G_BN - 1) / G_BN;
  const int grid = m_tiles * n_tiles;
  // e4m3 segments first (see the header), each group in the caller's order
  GemmSeg ord{};
  ord.nseg = seg.nseg;
  int j = 0;
  for (int pass = 1; pass >= 0; --pass)
    for (int i = 0; i < seg.nseg; ++i)
      if ((seg.f8[i] != 0) == (pass == 1)) { ord.a_off[j] = seg.a_off[i]; ord.b_off[j] = seg.b_off[i]; ord.f8[j] = seg.f8[i]; ++j; }
  SAMPT_TRY(ensure_func_smem(c, "gemm_tc_kernel", gemm_tc_kernel, G_SMEM_BYTES));
  gemm_tc_kernel<<<grid, G_THREADS, G_SMEM_BYTES, st>>>(tmA, tmB, M, N, K, ord, ep);
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

}  // namespace sampt

using namespace sampt;

// Unit-test / building-block entry: C = act(A B^T + bias), fp16 operands (bf16 if is_bf16), fp32 accumulation.
// precision: 1 = single pass; 2 = B (weights) carried as hi|lo (B is [N, 2K], lo at column K), A plain; 3 = both carried as hi|lo.
extern "C" int sampt_gemm_f16(sampt_ctx* ctx, const void* A, int lda, const void* B, int ldb, int M, int N, int K, int precision,
                              int is_bf16, const float* bias, int act, void* out16, float* out32, const float* resid, int ldc,
                              int split_off, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  GemmSeg seg{};
  seg.nseg = precision;
  SAMPT_CHECK(precision >= 1 && precision <= 3, "precision must be 1, 2 or 3");
  // precision 1: A.B ; 2: A.(B_hi + B_lo)  (weights carried as hi|lo) ; 3: A_hi.B_hi + A_lo.B_hi + A_hi.B_lo
  if (precision == 2) {
    seg.a_off[0] = 0; seg.b_off[0] = 0;
    seg.a_off[1] = 0; seg.b_off[1] = K;
  } else {
    seg.a_off[0] = 0; seg.b_off[0] = 0;
    seg.a_off[1] = K; seg.b_off[1] = 0;
    seg.a_off[2] = 0; seg.b_off[2] = K;
  }
  GemmEpi ep{};
  ep.out16 = reinterpret_cast<__half*>(out16);
  ep.out32 = out32;
  ep.resid = resid;
  ep.bias = bias;
  ep.rowmap = nullptr;
  ep.ldc = ldc;
  ep.act = act;
  ep.split_off = split_off;
  ep.is_bf16 = is_bf16;
  return gemm_tc(c, reinterpret_cast<cudaStream_t>(stream), A, lda, B, ldb, M, N, K, seg, ep);
}

// fp8-corrected split GEMM (tc_api.cuh, "precision 6"): C = act((A_hi.B_hi + A_lo8.B_hi8 + A_hi8.B_lo8) * acc_scale + bias).
// A [M, 2K] and B [N, 2K] fp16 units in the layouts of tc_api.cuh (sampt_split_f8c builds A; the host builds B once per weight).
extern "C" int sampt_gemm_f8c(sampt_ctx* ctx, const void* A, const void* B, int M, int N, int K, const float* acc_scale_dev,
                              const float* bias, int act, void* out16, float* out32, const float* resid, int ldc, int split_off,
                              int out_f8, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_CHECK(gemm_f8c_applicable(M, N, K), "sampt_gemm_f8c: needs M >= 256, N %% 256 == 0, K %% 128 == 0 (got %d x %d x %d)", M, N, K);
  GemmEpi ep{};
  ep.out16 = reinterpret_cast<__half*>(out16);
  ep.out32 = out32;
  ep.resid = resid;
  ep.bias = bias;
  ep.ldc = ldc;
  ep.act = act;
  ep.split_off = split_off;
  ep.out_f8 = out_f8;
  ep.acc_scale = acc_scale_dev;
  return gemm_tc(c, reinterpret_cast<cudaStream_t>(stream), A, 2 * K, B, 2 * K, M, N, K, make_seg_f8(K), ep);
}

// Unit-test entry: gemm_tc with every GemmSeg / GemmEpi field supplied by the caller (include/sampt_b200.h).
extern "C" int sampt_test_gemm_tc(sampt_ctx* ctx, const void* A, int lda, const void* B, int ldb, int M, int N, int K, int nseg,
                                  const int* a_off_host, const int* b_off_host, const int* f8_host, const float* bias, int act,
                                  int is_bf16, void* out16, float* out32, const float* resid, int resid_mod, const int* rowmap,
                                  const int* skip, const float* acc_scale, int ldc, int split_off, int out_f8, void* stream) {
  SAMPT_CHECK(nseg >= 1 && nseg <= 3, "sampt_test_gemm_tc: nseg %d out of range", nseg);
  GemmSeg seg{};
  seg.nseg = nseg;
  for (int i = 0; i < nseg; ++i) { seg.a_off[i] = a_off_host[i]; seg.b_off[i] = b_off_host[i]; seg.f8[i] = f8_host[i]; }
  GemmEpi ep{};
  ep.out16 = reinterpret_cast<__half*>(out16);
  ep.out32 = out32;
  ep.resid = resid;
  ep.bias = bias;
  ep.rowmap = rowmap;
  ep.ldc = ldc;
  ep.act = act;
  ep.split_off = split_off;
  ep.is_bf16 = is_bf16;
  ep.resid_mod = resid_mod;
  ep.skip = skip;
  ep.acc_scale = acc_scale;
  ep.out_f8 = out_f8;
  return gemm_tc(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), A, lda, B, ldb, M, N, K, seg, ep);
}

// x [M, K] fp32 -> the A operand of sampt_gemm_f8c: [fp16(x) | e4m3((x - fp16(x)) * 2^12) | e4m3(x * 2^-3)], 2K fp16 units per row
extern "C" int sampt_split_f8c(sampt_ctx* ctx, const float* x, int M, int K, void* out, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  return ln_rows(c, reinterpret_cast<cudaStream_t>(stream), x, K, nullptr, nullptr, nullptr, 0.f, reinterpret_cast<__half*>(out), 2 * K, K,
                 M, K, 0, 1);
}
