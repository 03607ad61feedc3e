// Fused attention for SAM's ViT (windowed 14x14 and global 64x64) on sm_90a tensor cores (wgmma).
//
// Decomposed relative position bias (upstream segment_anything image_encoder.add_decomposed_rel_pos; SURVEY App. B.1)
// is folded INTO the QK^T contraction by extending the head dimension:
//     Q' = [ q*scale | rel_h(q, 0..S-1) | rel_w(q, 0..S-1) | 0 ]      rel_h(q,j) = q . Rh[qy - j + S-1]
//     K' = [ k       | onehot(ky)       | onehot(kx)       | 0 ]
//     Q'.K'^T = scale*q.k + rel_h(q, ky) + rel_w(q, kx)
// so the kernel is plain flash attention with K-dim DK = pad64(hd + 2S) for QK^T and hd for PV.  Q'/K'/V^T are
// produced by vit_attn_prep (vit_kernels.cu).  Zero-padded window tokens are ordinary keys (no masking), exactly as in
// the reference; only the tile padding (keys >= Lk) is masked.
//
// One CTA = one (batch*window*head, 128-query tile), 288 threads.  Warp 8: TMA producer (Q' once, then K' / V^T tiles of
// 64 keys through a ring of 2-4 stages).  Warpgroups 0 and 1 own 64 query rows each: S = Q'K'^T by wgmma from shared
// memory into registers, online softmax on the accumulator fragment (a row lives in one quad of lanes), P rounded to fp16
// IN REGISTERS and fed straight back as the A operand of the P.V wgmma; the running output O stays in registers.
#include "common.cuh"
#include "tc_common.cuh"
#include "kernels.cuh"
#include "tc_api.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {
using namespace tc;

struct AttnParams {
  int Lq, Lk;        // valid queries / keys per batch-head
  int DKB;           // DK / 64
  int HD;            // head dim (multiple of 16, <= 128)
  int nheads;
  int stages;        // K'/V^T ring depth
  __half* out;       // [BH/nheads * Lq, ld_out]: row = (bh / nheads) * Lq + q, col = (bh % nheads) * HD + d
  int ld_out;
  int split_off;     // >0: also write the fp16 residual lo (or, with out_f8, the e4m3 operands) at this column offset
  int out_f8;        // with split_off > 0: fp8 correction operands of the proj GEMM (tc_api.cuh) instead of the fp16 remainder
};

constexpr int A_THREADS = 288;
constexpr int A_KT = 64;             // keys per tile
constexpr int A_Q_BLK = 128 * 128;   // one 64-column block of the 128-row Q' tile
constexpr int A_K_BLK = A_KT * 128;  // one 64-column block of a K' tile
constexpr float A_LOG2E = 1.4426950408889634f;

template <int HDT> __device__ __forceinline__ void wgmma_pv(float (&d)[HDT / 2], const uint32_t (&a)[4], uint64_t db);
template <> __device__ __forceinline__ void wgmma_pv<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t db) { wgmma_m64n64k16_f16_rs(d, a, db); }
template <> __device__ __forceinline__ void wgmma_pv<80>(float (&d)[40], const uint32_t (&a)[4], uint64_t db) { wgmma_m64n80k16_f16_rs(d, a, db); }
template <> __device__ __forceinline__ void wgmma_pv<96>(float (&d)[48], const uint32_t (&a)[4], uint64_t db) { wgmma_m64n96k16_f16_rs(d, a, db); }
template <> __device__ __forceinline__ void wgmma_pv<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t db) { wgmma_m64n128k16_f16_rs(d, a, db); }

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

template <int HDT>   // head-dim bound (64 | 80 | 96 | 128): the N of the P.V wgmma and the running-output registers
__global__ void __launch_bounds__(A_THREADS, 1)
attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int stage_bytes = p.DKB * A_K_BLK + HDT * 128;   // K' tile + V^T tile (HDT rows of 64 keys), 1024-byte multiple
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + p.DKB * A_Q_BLK;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(sKV + p.stages * stage_bytes);
  uint64_t* full = q_full + 1;
  uint64_t* empty = full + p.stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, bh = blockIdx.y;
  const int ntiles = (p.Lk + A_KT - 1) / A_KT;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < p.stages; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 256); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmK);
      tma_prefetch_desc(&tmV);
      mbar_expect_tx(q_full, p.DKB * A_Q_BLK);
      for (int kb = 0; kb < p.DKB; ++kb) tma_load_3d(sQ + kb * A_Q_BLK, &tmQ, q_full, kb * 64, qt * 128, bh);
      for (int j = 0; j < ntiles; ++j) {
        const int s = j % p.stages;
        mbar_wait(empty + s, ((j / p.stages) & 1) ^ 1);
        uint8_t* sK = sKV + s * stage_bytes;
        mbar_expect_tx(full + s, p.DKB * A_K_BLK + p.HD * 128);
        for (int kb = 0; kb < p.DKB; ++kb) tma_load_3d(sK + kb * A_K_BLK, &tmK, full + s, kb * 64, j * A_KT, bh);
        tma_load_3d(sK + p.DKB * A_K_BLK, &tmV, full + s, j * A_KT, 0, bh);
      }
    }
    return;
  }

  // -------------------------------------------------------------- softmax warpgroups: g owns query rows [64 g, 64 g + 64)
  const int g = warp >> 2, w = warp & 3;
  const int c2 = 2 * (lane & 3);
  const uint64_t qdesc = make_smem_desc_sw128(smem_u32(sQ) + g * 64 * 128);
  float o[HDT / 2];
#pragma unroll
  for (int i = 0; i < HDT / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // rows 16 w + lane / 4 (+ 8)
  mbar_wait(q_full, 0);
  for (int j = 0; j < ntiles; ++j) {
    const int s = j % p.stages;
    mbar_wait(full + s, (j / p.stages) & 1);
    const uint32_t sK = smem_u32(sKV + s * stage_bytes);
    const uint64_t vdesc = make_smem_desc_sw128(sK + p.DKB * A_K_BLK);
    // ---- S = Q' K'^T  (64 x 64 per warpgroup)
    float sc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) sc[i] = 0.f;
    wgmma_fence();
    for (int kb = 0; kb < p.DKB; ++kb) {
      const uint64_t ad = qdesc + (uint64_t)((kb * A_Q_BLK) >> 4);
      const uint64_t bd = make_smem_desc_sw128(sK + kb * A_K_BLK);
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64k16_f16(sc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k));
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    // ---- online softmax on the fragment: sc[4 i + 2 h + e] = S[row h][key 8 i + c2 + e]
    const int valid = p.Lk - j * A_KT;
    float alpha[2];
    uint32_t pa[4][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * i + c2 + e < valid) mx = fmaxf(mx, sc[4 * i + 2 * h + e]);
      const float m_new = fmaxf(m_run[h], quad_max(mx));   // finite: key 0 of every tile is valid
      alpha[h] = ex2_approx((m_run[h] - m_new) * A_LOG2E);  // 0 on the first tile (m_run = -inf)
      m_run[h] = m_new;
      const float mb = -m_new * A_LOG2E;
      float ls = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = (8 * i + c2 + e < valid) ? ex2_approx(fmaf(sc[4 * i + 2 * h + e], A_LOG2E, mb)) : 0.f;
          sc[4 * i + 2 * h + e] = x;
          ls += x;
        }
      l_run[h] = l_run[h] * alpha[h] + ls;   // per-thread partial row sum (the quad is summed once, at the end)
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        __half2 hv = __floats2half2_rn(sc[8 * kk + 2 * jj], sc[8 * kk + 2 * jj + 1]);
        pa[kk][jj] = *reinterpret_cast<uint32_t*>(&hv);
      }
#pragma unroll
    for (int i = 0; i < HDT / 8; ++i) {
      o[4 * i + 0] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }
    // ---- O += P V  (A = P from registers, B = V^T tile, 16 keys = 32 bytes per step)
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_pv<HDT>(o, pa[kk], vdesc + (uint64_t)(2 * kk));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    mbar_arrive(empty + s);
  }

  // -------------------------------------------------------------- output: fp16 hi (+ lo | e4m3 operands)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float inv = 1.0f / quad_sum(l_run[h]);
    const int qrow = qt * 128 + g * 64 + w * 16 + (lane >> 2) + 8 * h;
    if (qrow >= p.Lq) continue;
    const size_t orow = (size_t)(bh / p.nheads) * p.Lq + qrow;
    __half* op = p.out + orow * p.ld_out + (size_t)(bh % p.nheads) * p.HD;
#pragma unroll
    for (int i = 0; i < HDT / 8; ++i) {
      const int d = 8 * i + c2;
      if (d >= p.HD) continue;
      const float a = o[4 * i + 2 * h] * inv, b = o[4 * i + 2 * h + 1] * inv;
      const __half2 hv = __floats2half2_rn(a, b);
      *reinterpret_cast<__half2*>(op + d) = hv;
      const float2 hf = __half22float2(hv);
      if (p.split_off > 0 && p.out_f8) {
        // e4m3(remainder * 2^12) | e4m3(value * 2^-3): split_off BYTES each, right behind the split_off hi halves of the row
        uint8_t* ob = reinterpret_cast<uint8_t*>(p.out + orow * p.ld_out + p.split_off) + (size_t)(bh % p.nheads) * p.HD + d;
        uint16_t l8, h8;
        asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(l8) : "f"((b - hf.y) * F8_LO_SCALE), "f"((a - hf.x) * F8_LO_SCALE));
        asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(h8) : "f"(b * F8_HI_SCALE), "f"(a * F8_HI_SCALE));
        *reinterpret_cast<uint16_t*>(ob) = l8;
        *reinterpret_cast<uint16_t*>(ob + p.split_off) = h8;
      } else if (p.split_off > 0) {
        *reinterpret_cast<__half2*>(op + p.split_off + d) = __floats2half2_rn(a - hf.x, b - hf.y);
      }
    }
  }
}

template <int HDT>
static int launch_attn(Ctx* c, cudaStream_t st, const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, AttnParams p,
                       dim3 grid, const char* name) {
  const size_t fixed = (size_t)p.DKB * A_Q_BLK + 1024 /*align*/ + 256 /*barriers*/;
  const size_t stage = (size_t)p.DKB * A_K_BLK + (size_t)HDT * 128;
  p.stages = 4;
  while (p.stages > 2 && fixed + p.stages * stage > 227 * 1024) --p.stages;
  const size_t smem = fixed + p.stages * stage;
  SAMPT_CHECK(smem <= 227 * 1024, "attn_tc: tile configuration needs %zu B of shared memory (> 227 KB)", smem);
  SAMPT_TRY(ensure_func_smem(c, name, attn_tc_kernel<HDT>, 227 * 1024));
  attn_tc_kernel<HDT><<<grid, A_THREADS, smem, st>>>(tmQ, tmK, tmV, p);
  return 0;
}

int attn_tc(Ctx* c, cudaStream_t st, const __half* Qx, const __half* Kx, const __half* Vt, int BH, int Lq, int Lk, int Lkp,
            int DK, int HD, int nheads, __half* out, int ld_out, int split_off, int out_f8) {
  SAMPT_CHECK(DK % 64 == 0 && DK > 0 && DK <= 256, "attn_tc: DK=%d must be a multiple of 64 and <= 256", DK);
  SAMPT_CHECK(HD % 16 == 0 && HD > 0 && HD <= 128, "attn_tc: HD=%d must be a multiple of 16 and <= 128", HD);
  SAMPT_CHECK(Lkp % 8 == 0 && Lkp >= Lk && Lk > 0, "attn_tc: Lkp=%d must be a multiple of 8 and >= Lk", Lkp);
  CUtensorMap tmQ, tmK, tmV;
  SAMPT_TRY(make_tmap_3d_f16(&tmQ, Qx, DK, Lq, BH, (uint64_t)DK * 2, (uint64_t)Lq * DK * 2, 64, 128, 1));
  SAMPT_TRY(make_tmap_3d_f16(&tmK, Kx, DK, Lk, BH, (uint64_t)DK * 2, (uint64_t)Lk * DK * 2, 64, A_KT, 1));
  // V^T rows have the pitch Lkp but only Lk valid keys: TMA zero-fills the tail of the last tile, so whatever the padding
  // [Lk, Lkp) holds never meets a P = 0 (0 * NaN would poison the row)
  SAMPT_TRY(make_tmap_3d_f16(&tmV, Vt, Lk, HD, BH, (uint64_t)Lkp * 2, (uint64_t)HD * Lkp * 2, 64, HD, 1));
  AttnParams p;
  p.Lq = Lq; p.Lk = Lk; p.DKB = DK / 64; p.HD = HD; p.nheads = nheads; p.stages = 2;
  p.out = out; p.ld_out = ld_out; p.split_off = split_off; p.out_f8 = out_f8;
  const dim3 grid((Lq + 127) / 128, BH);
  if (HD <= 64) SAMPT_TRY(launch_attn<64>(c, st, tmQ, tmK, tmV, p, grid, "attn_tc_kernel<64>"));
  else if (HD <= 80) SAMPT_TRY(launch_attn<80>(c, st, tmQ, tmK, tmV, p, grid, "attn_tc_kernel<80>"));
  else if (HD <= 96) SAMPT_TRY(launch_attn<96>(c, st, tmQ, tmK, tmV, p, grid, "attn_tc_kernel<96>"));
  else SAMPT_TRY(launch_attn<128>(c, st, tmQ, tmK, tmV, p, grid, "attn_tc_kernel<128>"));
  c->launches++;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

}  // namespace sampt

using namespace sampt;

// Unit-test entry: softmax(Qx Kx^T) V with pre-extended operands (see header comment).  NT (a key-tile size) is accepted
// for ABI stability and not used: the kernel always walks the keys in tiles of 64.
extern "C" int sampt_attention_f16(sampt_ctx* ctx, const void* Qx, const void* Kx, const void* Vt, int BH, int Lq, int Lk, int Lkp,
                                   int DK, int HD, int NT, int nheads, void* out, int ld_out, int split_off, void* stream) {
  (void)NT;
  return attn_tc(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const __half*>(Qx),
                 reinterpret_cast<const __half*>(Kx), reinterpret_cast<const __half*>(Vt), BH, Lq, Lk, Lkp, DK, HD, nheads,
                 reinterpret_cast<__half*>(out), ld_out, split_off);
}

// Unit-test entry: what one ViT block runs between its qkv GEMM and proj (vit_pipeline.cu): attn_prep + attn_tc, scale 1/sqrt(HD).
extern "C" int sampt_test_vit_attention(sampt_ctx* ctx, const void* qkv, const float* rel_pos_h, const float* rel_pos_w, int nwb,
                                        int nheads, int S, int D, int DK, int Lkp, void* Qx, void* Kx, void* Vt, void* out, int ld_out,
                                        int split_off, int out_f8, void* stream) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  SAMPT_CHECK(nheads > 0 && D % nheads == 0, "sampt_test_vit_attention: D (%d) must be a multiple of nheads (%d)", D, nheads);
  const int HD = D / nheads, L = S * S;
  __half *q = reinterpret_cast<__half*>(Qx), *k = reinterpret_cast<__half*>(Kx), *v = reinterpret_cast<__half*>(Vt);
  SAMPT_TRY(attn_prep(c, st, reinterpret_cast<const __half*>(qkv), 3 * D, rel_pos_h, rel_pos_w, q, k, v, nwb, nheads, S, Lkp, DK, D, HD,
                      1.0f / sqrtf((float)HD)));
  return attn_tc(c, st, q, k, v, nwb * nheads, L, L, Lkp, DK, HD, nheads, reinterpret_cast<__half*>(out), ld_out, split_off, out_f8);
}
