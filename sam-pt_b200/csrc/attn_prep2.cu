// Attention operand preparation for the ViT, round-2 kernel (supersedes attn_prep_kernel of vit_kernels.cu).
//
// Same outputs (see attn_tc.cu / attn_ws.cu):  Q' = [q*scale | rel_h(q, 0..S-1) | rel_w(q, 0..S-1) | 0]   [BH, L, DK]
//                                               K' = [k       | onehot(ky)       | onehot(kx)       | 0]   [BH, L, DK]
//                                               V^T                                                        [BH, HD, Lkp]
// (keys of V^T in [L, Lkp) are row padding that attn_tc never reads; they are left as they are)
// with rel_h(q, j) = q . Rh[qy - j + S-1], rel_w(q, j) = q . Rw[qx - j + S-1] (upstream add_decomposed_rel_pos, unscaled q).
//
// Round 1 computed the 2S dot products per query on the CUDA cores (440 k FMA per 14x14 window-head, fed from shared memory at
// ~1 load per 5 FMA): 0.66 ms per 10-frame launch for 0.9 GB of traffic, 1.3 TB/s.  Here they are ONE small tensor-core product
// per CTA:  T = q [TC x HD] . Rcat^T [HD x 2(2S-1)],  Rcat = [Rh ; Rw], as legacy mma.sync m16n8k16 tiles (the operands are tiny
// and live in shared memory; a wgmma pipeline would be set-up cost only), with Rcat carried as fp16 hi + lo so that the table is
// exact to ~2^-22 -- the fp32 table of the reference -- and q as the fp16 it already is.  The shifted pick
// Q'ext[t][j] = T[t][qy - j + S-1] is then a shared-memory gather while the rows are assembled.  Everything else is coalesced
// 16-byte traffic, so the kernel is bound by its algorithmic bytes (read qkv once, write Q', K', V^T once).
#include <cstdlib>
#include <mma.h>

#include "common.cuh"
#include "kernels.cuh"

namespace sampt {

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldmatrix_x2(uint32_t (&r)[2], const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(a));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit_wait_all() {
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// Rcat = [Rh ; Rw] (2(2S-1) rows, zero padded to NRP) as fp16 hi | lo tables with the shared-memory row pitch QP, built once per
// launch so that every CTA fetches it with plain 16-byte asynchronous copies
template <int HD>
__global__ void relpos_table_kernel(const float* __restrict__ relh, const float* __restrict__ relw, __half* __restrict__ tab, int S,
                                    int NRP) {
  constexpr int QP = HD + 8;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NRP * QP) return;
  const int r = i / QP, d = i % QP;
  float v = 0.f;
  if (d < HD) {
    if (r < 2 * S - 1) v = relh[(size_t)r * HD + d];
    else if (r < 2 * (2 * S - 1)) v = relw[(size_t)(r - (2 * S - 1)) * HD + d];
  }
  const __half hi = __float2half_rn(v);
  tab[i] = hi;
  tab[(size_t)NRP * QP + i] = __float2half_rn(v - __half2float(hi));
}

// grid (chunks of TC tokens, heads, windows*frames); 256 threads.  TC % 16 == 0.
// All global loads of a CTA (q and v tiles, the table) are issued up front as cp.async 16-byte copies and overlap with the K' rows,
// which are copied global -> global through registers in batches of four independent loads; V^T leaves in 128-byte runs.
template <int HD>
__global__ void __launch_bounds__(256, 2)
attn_prep2_kernel(const __half* __restrict__ qkv, int ldq, const __half* __restrict__ tab, __half* __restrict__ Qx,
                  __half* __restrict__ Kx, __half* __restrict__ Vt, int S, int L, int Lkp, int DK, int D, int nheads, float scale, int TC,
                  int NRP /* padded table rows: multiple of 8 >= 2(2S-1) */) {
  constexpr int QP = HD + 8;            // row pitch in halves: 16 B aligned, conflict-free for ldmatrix
  constexpr int KS = HD / 16;           // k-steps of the MMA
  extern __shared__ __align__(16) unsigned char smraw[];
  __half* sq = reinterpret_cast<__half*>(smraw);                 // [TC][QP]   q (unscaled)
  __half* sv = sq + (size_t)TC * QP;                             // [TC][QP]   v, later re-used for T
  const int TP = NRP + 8;                                        // T row pitch (halves)
  const size_t svt = (size_t)TC * (size_t)max(QP, TP);          // the v tile and (later) T share this region
  __half* sRh = sv + svt;                                        // [NRP][QP]  Rcat hi
  __half* sRl = sRh + (size_t)NRP * QP;                          // [NRP][QP]  Rcat lo
  __half* sT = sv;                                               // [TC][TP]   T = q . Rcat^T as fp16 (aliases sv once V^T is out)
  const int chunk = blockIdx.x, h = blockIdx.y, wb = blockIdx.z;
  const int t0 = chunk * TC;
  const int nt = min(TC, L - t0);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const size_t bh = (size_t)wb * nheads + h;
  constexpr int SEG = HD / 8;           // 16-byte segments per head row
  const __half* gq = qkv + ((size_t)wb * L + t0) * ldq + h * HD;

  // ---- phase 1: asynchronous copies of q, v and the table into shared memory; rows beyond nt are zeroed
  for (int i = tid; i < TC * SEG; i += 256) {
    const int t = i / SEG, sgm = i % SEG;
    if (t < nt) {
      cp_async16(sq + (size_t)t * QP + sgm * 8, gq + (size_t)t * ldq + sgm * 8);
      cp_async16(sv + (size_t)t * QP + sgm * 8, gq + (size_t)t * ldq + 2 * D + sgm * 8);
    } else {
      *reinterpret_cast<uint4*>(sq + (size_t)t * QP + sgm * 8) = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(sv + (size_t)t * QP + sgm * 8) = make_uint4(0u, 0u, 0u, 0u);
    }
  }
  for (int i = tid; i < 2 * NRP * QP / 8; i += 256) cp_async16(sRh + (size_t)i * 8, tab + (size_t)i * 8);
  asm volatile("cp.async.commit_group;" ::: "memory");
  // ---- phase 2 (overlaps the copies): K' rows = [k | onehot(ky) | onehot(kx) | 0], global -> global
  {
    const int n_items = nt * SEG;
    for (int i0 = tid; i0 < n_items; i0 += 4 * 256) {
      uint4 kv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * 256;
        if (i < n_items) kv[u] = *reinterpret_cast<const uint4*>(gq + (size_t)(i / SEG) * ldq + D + (i % SEG) * 8);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * 256;
        if (i < n_items) *reinterpret_cast<uint4*>(Kx + (bh * L + t0 + i / SEG) * DK + (i % SEG) * 8) = kv[u];
      }
    }
    const int EXT = DK - HD;
    for (int i = tid; i < nt * (EXT / 8); i += 256) {
      const int t = i / (EXT / 8), e0 = (i % (EXT / 8)) * 8;
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
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  // ---- phase 3: V^T.  A warp writes 4 rows d x 8 groups of 8 keys: 4 runs of 128 contiguous bytes per store instruction; the
  //      8 values of a group are read in a lane-rotated order so that the 8 lanes of a run hit 8 different banks
  {
    const int ngrp = (TC + 7) / 8;
    const int ngrp8 = (ngrp + 7) / 8;                 // groups are handed out 8 at a time
    for (int w = warp; w < (HD / 4) * ngrp8; w += 8) {
      const int d = (w / ngrp8) * 4 + (lane >> 3);
      const int g = (w % ngrp8) * 8 + (lane & 7);
      if (g < ngrp) {
        __half hv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int jj = (j + (lane & 7)) & 7;
          const int t = g * 8 + jj;
          hv[jj] = (t < nt) ? sv[(size_t)t * QP + d] : __float2half_rn(0.f);
        }
        if (t0 + g * 8 < Lkp) *reinterpret_cast<uint4*>(Vt + (bh * HD + d) * Lkp + t0 + g * 8) = *reinterpret_cast<uint4*>(hv);
      }
    }
  }
  __syncthreads();   // sv is dead from here: T goes over it
  // ---- phase 4: T[TC x NRP] = q . Rcat^T on the tensor cores (mma.sync m16n8k16, fp32 accumulate, Rcat = hi + lo)
  {
    const int mt = TC / 16, ntile = NRP / 8;
    for (int m = warp; m < mt; m += 8) {
      uint32_t af[KS][4];
#pragma unroll
      for (int ks = 0; ks < KS; ++ks)
        ldmatrix_x4(af[ks], sq + (size_t)(m * 16 + (lane & 15)) * QP + ks * 16 + (lane >> 4) * 8);
      for (int n = 0; n < ntile; ++n) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          uint32_t bh_[2], bl_[2];
          const size_t off = (size_t)(n * 8 + (lane & 7)) * QP + ks * 16 + ((lane >> 3) & 1) * 8;
          ldmatrix_x2(bh_, sRh + off);
          ldmatrix_x2(bl_, sRl + off);
          mma_16816(acc, af[ks], bh_);
          mma_16816(acc, af[ks], bl_);
        }
        const int r0 = m * 16 + (lane >> 2), c0 = n * 8 + 2 * (lane & 3);
        *reinterpret_cast<__half2*>(sT + (size_t)r0 * TP + c0) = __floats2half2_rn(acc[0], acc[1]);
        *reinterpret_cast<__half2*>(sT + (size_t)(r0 + 8) * TP + c0) = __floats2half2_rn(acc[2], acc[3]);
      }
    }
  }
  __syncthreads();
  // ---- phase 5: Q' rows, 16 B per thread-step: [q*scale (HD) | T[t][ty - j + S-1] (S) | T[t][(2S-1) + tx - j + S-1] (S) | 0]
  {
    const int cpr = DK / 8;  // 16-byte chunks per row
    for (int i = tid; i < nt * cpr; i += 256) {
      const int t = i / cpr, c8 = (i % cpr) * 8;
      const int tt = t0 + t, ty = tt / S, tx = tt % S;
      __half hv[8];
      if (c8 + 8 <= HD) {
        const uint4 qv = *reinterpret_cast<const uint4*>(sq + (size_t)t * QP + c8);
        const __half2* q2 = reinterpret_cast<const __half2*>(&qv);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(q2[j]);
          reinterpret_cast<__half2*>(hv)[j] = __floats2half2_rn(f.x * scale, f.y * scale);
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int col = c8 + j;
          __half v;
          if (col < HD) v = __float2half_rn(__half2float(sq[(size_t)t * QP + col]) * scale);
          else if (col < HD + S) v = sT[(size_t)t * TP + (ty - (col - HD) + S - 1)];
          else if (col < HD + 2 * S) v = sT[(size_t)t * TP + (2 * S - 1) + (tx - (col - HD - S) + S - 1)];
          else v = __float2half_rn(0.f);
          hv[j] = v;
        }
      }
      *reinterpret_cast<uint4*>(Qx + (bh * L + tt) * DK + c8) = *reinterpret_cast<uint4*>(hv);
    }
  }
}


// ---- global-attention blocks (S = 64: 4096 tokens, 2(2S-1) = 254 table rows) ---------------------------------------------------
// The 90 KB hi | lo table would be re-fetched by every CTA of a (chunk, head, frame) grid (10240 CTAs x 90 KB per 10-frame launch,
// as much as the operands themselves), so this variant is PERSISTENT: one CTA per SM loads the table once and walks items
// (frame, head, chunk of TC = 64 tokens), prefetching the q / v tiles of the next item with cp.async while the current one is
// transposed, multiplied and written.  Same arithmetic and output as attn_prep2_kernel.
template <int HD>
__global__ void __launch_bounds__(256, 1)
attn_prep2_persistent_kernel(const __half* __restrict__ qkv, int ldq, const __half* __restrict__ tab, __half* __restrict__ Qx,
                             __half* __restrict__ Kx, __half* __restrict__ Vt, int S, int L, int Lkp, int DK, int D, int nheads, int nwb,
                             float scale, int NRP) {
  constexpr int QP = HD + 8, KS = HD / 16, SEG = HD / 8, TC = 64;
  extern __shared__ __align__(16) unsigned char smraw[];
  const int TP = NRP + 8;
  __half* sRh = reinterpret_cast<__half*>(smraw);                // [NRP][QP] Rcat hi
  __half* sRl = sRh + (size_t)NRP * QP;                          // [NRP][QP] Rcat lo
  __half* sqb = sRl + (size_t)NRP * QP;                          // [2][TC][QP] q (unscaled), double buffered
  __half* svb = sqb + (size_t)2 * TC * QP;                       // [2][TC][QP] v
  __half* sT = svb + (size_t)2 * TC * QP;                        // [TC][TP]    T = q . Rcat^T
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nchunk = (L + TC - 1) / TC;
  const long long n_items = (long long)nwb * nheads * nchunk;

  auto prefetch = [&](long long item, int buf) {
    if (item < n_items) {
      const int chunk = (int)(item % nchunk), h = (int)((item / nchunk) % nheads), wb = (int)(item / ((long long)nchunk * nheads));
      const int t0 = chunk * TC, nt = min(TC, L - t0);
      const __half* gq = qkv + ((size_t)wb * L + t0) * ldq + h * HD;
      __half* sq = sqb + (size_t)buf * TC * QP;
      __half* sv = svb + (size_t)buf * TC * QP;
      for (int i = tid; i < TC * SEG; i += 256) {
        const int t = i / SEG, sgm = i % SEG;
        if (t < nt) {
          cp_async16(sq + (size_t)t * QP + sgm * 8, gq + (size_t)t * ldq + sgm * 8);
          cp_async16(sv + (size_t)t * QP + sgm * 8, gq + (size_t)t * ldq + 2 * D + sgm * 8);
        } else {
          *reinterpret_cast<uint4*>(sq + (size_t)t * QP + sgm * 8) = make_uint4(0u, 0u, 0u, 0u);
          *reinterpret_cast<uint4*>(sv + (size_t)t * QP + sgm * 8) = make_uint4(0u, 0u, 0u, 0u);
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  for (int i = tid; i < 2 * NRP * QP / 8; i += 256) cp_async16(sRh + (size_t)i * 8, tab + (size_t)i * 8);
  prefetch(blockIdx.x, 0);   // (the table rides in the first group)
  int buf = 0;
  for (long long item = blockIdx.x; item < n_items; item += gridDim.x, buf ^= 1) {
    prefetch(item + gridDim.x, buf ^ 1);
    const int chunk = (int)(item % nchunk), h = (int)((item / nchunk) % nheads), wb = (int)(item / ((long long)nchunk * nheads));
    const int t0 = chunk * TC, nt = min(TC, L - t0);
    const size_t bh = (size_t)wb * nheads + h;
    const __half* gq = qkv + ((size_t)wb * L + t0) * ldq + h * HD;
    const __half* sq = sqb + (size_t)buf * TC * QP;
    const __half* sv = svb + (size_t)buf * TC * QP;
    // ---- K' rows = [k | onehot(ky) | onehot(kx) | 0], global -> global (independent of the tiles in flight)
    {
      const int n_it = nt * SEG;
      for (int i0 = tid; i0 < n_it; i0 += 4 * 256) {
        uint4 kv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = i0 + u * 256;
          if (i < n_it) kv[u] = *reinterpret_cast<const uint4*>(gq + (size_t)(i / SEG) * ldq + D + (i % SEG) * 8);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = i0 + u * 256;
          if (i < n_it) *reinterpret_cast<uint4*>(Kx + (bh * L + t0 + i / SEG) * DK + (i % SEG) * 8) = kv[u];
        }
      }
      const int EXT = DK - HD;
      for (int i = tid; i < nt * (EXT / 8); i += 256) {
        const int t = i / (EXT / 8), e0 = (i % (EXT / 8)) * 8;
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
    asm volatile("cp.async.wait_group 1;" ::: "memory");   // everything but the prefetch of the next item has landed
    __syncthreads();
    // ---- V^T: a warp writes 4 rows d x 8 groups of 8 keys = 4 runs of 128 contiguous bytes; lane-rotated reads (bank spread)
    {
      constexpr int ngrp = TC / 8;
      for (int w = warp; w < (HD / 4); w += 8) {
        const int d = w * 4 + (lane >> 3);
        const int g = lane & 7;
        __half hv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int jj = (j + (lane & 7)) & 7;
          const int t = g * 8 + jj;
          hv[jj] = (t < nt) ? sv[(size_t)t * QP + d] : __float2half_rn(0.f);
        }
        if (g < ngrp && t0 + g * 8 < Lkp) *reinterpret_cast<uint4*>(Vt + (bh * HD + d) * Lkp + t0 + g * 8) = *reinterpret_cast<uint4*>(hv);
      }
    }
    // ---- T[TC x NRP] = q . Rcat^T (mma.sync m16n8k16, fp32 accumulate, Rcat = hi + lo); 4 m-tiles x 2 column halves over 8 warps
    {
      const int m = warp & 3, nhalf = warp >> 2, ntile = NRP / 8;
      uint32_t af[KS][4];
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) ldmatrix_x4(af[ks], sq + (size_t)(m * 16 + (lane & 15)) * QP + ks * 16 + (lane >> 4) * 8);
      for (int n = nhalf; n < ntile; n += 2) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          uint32_t bh_[2], bl_[2];
          const size_t off = (size_t)(n * 8 + (lane & 7)) * QP + ks * 16 + ((lane >> 3) & 1) * 8;
          ldmatrix_x2(bh_, sRh + off);
          ldmatrix_x2(bl_, sRl + off);
          mma_16816(acc, af[ks], bh_);
          mma_16816(acc, af[ks], bl_);
        }
        const int r0 = m * 16 + (lane >> 2), c0 = n * 8 + 2 * (lane & 3);
        *reinterpret_cast<__half2*>(sT + (size_t)r0 * TP + c0) = __floats2half2_rn(acc[0], acc[1]);
        *reinterpret_cast<__half2*>(sT + (size_t)(r0 + 8) * TP + c0) = __floats2half2_rn(acc[2], acc[3]);
      }
    }
    __syncthreads();
    // ---- Q' rows: [q*scale (HD) | T[t][ty - j + S-1] (S) | T[t][(2S-1) + tx - j + S-1] (S) | 0]
    {
      const int cpr = DK / 8;
      for (int i = tid; i < nt * cpr; i += 256) {
        const int t = i / cpr, c8 = (i % cpr) * 8;
        const int tt = t0 + t, ty = tt / S, tx = tt % S;
        __half hv[8];
        if (c8 + 8 <= HD) {
          const uint4 qv = *reinterpret_cast<const uint4*>(sq + (size_t)t * QP + c8);
          const __half2* q2 = reinterpret_cast<const __half2*>(&qv);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(q2[j]);
            reinterpret_cast<__half2*>(hv)[j] = __floats2half2_rn(f.x * scale, f.y * scale);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int col = c8 + j;
            __half v;
            if (col < HD) v = __float2half_rn(__half2float(sq[(size_t)t * QP + col]) * scale);
            else if (col < HD + S) v = sT[(size_t)t * TP + (ty - (col - HD) + S - 1)];
            else if (col < HD + 2 * S) v = sT[(size_t)t * TP + (2 * S - 1) + (tx - (col - HD - S) + S - 1)];
            else v = __float2half_rn(0.f);
            hv[j] = v;
          }
        }
        *reinterpret_cast<uint4*>(Qx + (bh * L + tt) * DK + c8) = *reinterpret_cast<uint4*>(hv);
      }
    }
    __syncthreads();   // sq / sv[buf] and sT are free for the prefetch / product of the iteration after next
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

static bool attn_prep2_enabled() {
  // ON unless SAMPT_ATTN_PREP2=0.  Parity-tested on hardware (encoder, C1, full C2); 436 us per windowed launch in the step against
  // 634 us for attn_prep_kernel (gpurun_out/kernel_table_prep2b.md); the first version (plain loads, uncoalesced V^T) took 748 us.
  static const int on = [] { const char* e = std::getenv("SAMPT_ATTN_PREP2"); return (e != nullptr && e[0] == '0') ? 0 : 1; }();
  return on != 0;
}

// returns 1 when the shape is not covered (caller falls back to attn_prep_kernel), 0 on success, < 0 on error
int attn_prep2(Ctx* c, cudaStream_t st, const __half* qkv, int ldq, const float* relh, const float* relw, __half* Qx, __half* Kx,
               __half* Vt, int nwb, int nheads, int S, int Lkp, int DK, int D, int HD, float scale) {
  if (!attn_prep2_enabled()) return 1;
  if (!(HD == 80 || HD == 64) || DK % 8 != 0 || DK < HD + 2 * S || (DK - HD) % 8 != 0 || Lkp % 8 != 0 || D % 8 != 0 || ldq % 8 != 0) return 1;
  const int L = S * S;
  const int NRP = ((2 * (2 * S - 1) + 7) / 8) * 8;
  const int QP = HD + 8, TP = NRP + 8;
  const bool persistent = L > 256;                               // global blocks: table too large to re-fetch per (chunk, head, frame)
  static const int global_on = [] { const char* e = std::getenv("SAMPT_ATTN_PREP2_GLOBAL"); return (e != nullptr && e[0] == '0') ? 0 : 1; }();
  if (persistent && !global_on) return 1;
  const int TC = persistent ? 64 : ((L + 15) / 16) * 16;         // windowed: a whole 14x14 window (208 rows)
  const size_t sv_or_t = (size_t)TC * (size_t)std::max(QP, TP);
  const size_t smem = persistent ? (2 * (size_t)NRP * QP + 4 * (size_t)TC * QP + (size_t)TC * TP) * sizeof(__half)
                                 : ((size_t)TC * QP + sv_or_t + 2 * (size_t)NRP * QP) * sizeof(__half);
  if (smem > (persistent ? 220 : 110) * 1024) return 1;          // windowed: two CTAs per SM
  // the fp16 hi | lo table, library-owned (grows on demand)
  const size_t tab_bytes = 2 * (size_t)NRP * QP * sizeof(__half);
  auto it = c->owned.find("attn_prep2:table");
  if (it == c->owned.end() || it->second.second < tab_bytes) {
    if (it != c->owned.end()) { SAMPT_CUDA(cudaDeviceSynchronize()); cudaFree(it->second.first); }
    void* buf = nullptr;
    SAMPT_CUDA(cudaMalloc(&buf, tab_bytes));
    c->owned["attn_prep2:table"] = {buf, tab_bytes};
    it = c->owned.find("attn_prep2:table");
  }
  __half* tab = reinterpret_cast<__half*>(it->second.first);
  dim3 grid(cdiv(L, TC), nheads, nwb);
  const long long n_items = (long long)cdiv(L, TC) * nheads * nwb;
  const int pgrid = (int)std::min<long long>(n_items, c->num_sms);
  if (HD == 80) {
    relpos_table_kernel<80><<<cdiv(NRP * QP, 256), 256, 0, st>>>(relh, relw, tab, S, NRP);
    if (persistent) {
      SAMPT_TRY(ensure_func_smem(c, "attn_prep2_persistent_kernel<80>", attn_prep2_persistent_kernel<80>, 220 * 1024));
      attn_prep2_persistent_kernel<80><<<pgrid, 256, smem, st>>>(qkv, ldq, tab, Qx, Kx, Vt, S, L, Lkp, DK, D, nheads, nwb, scale, NRP);
    } else {
      SAMPT_TRY(ensure_func_smem(c, "attn_prep2_kernel<80>", attn_prep2_kernel<80>, 110 * 1024));
      attn_prep2_kernel<80><<<grid, 256, smem, st>>>(qkv, ldq, tab, Qx, Kx, Vt, S, L, Lkp, DK, D, nheads, scale, TC, NRP);
    }
  } else {
    relpos_table_kernel<64><<<cdiv(NRP * QP, 256), 256, 0, st>>>(relh, relw, tab, S, NRP);
    if (persistent) {
      SAMPT_TRY(ensure_func_smem(c, "attn_prep2_persistent_kernel<64>", attn_prep2_persistent_kernel<64>, 220 * 1024));
      attn_prep2_persistent_kernel<64><<<pgrid, 256, smem, st>>>(qkv, ldq, tab, Qx, Kx, Vt, S, L, Lkp, DK, D, nheads, nwb, scale, NRP);
    } else {
      SAMPT_TRY(ensure_func_smem(c, "attn_prep2_kernel<64>", attn_prep2_kernel<64>, 110 * 1024));
      attn_prep2_kernel<64><<<grid, 256, smem, st>>>(qkv, ldq, tab, Qx, Kx, Vt, S, L, Lkp, DK, D, nheads, scale, TC, NRP);
    }
  }
  c->launches += 2;
  SAMPT_LAUNCH_CHECK();
  return 0;
}

}  // namespace sampt
