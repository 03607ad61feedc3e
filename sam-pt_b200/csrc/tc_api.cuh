// Launcher-level API of the tensor-core kernels (gemm_tc.cu, attn_tc.cu), used by the ViT pipeline.
#pragma once
#include "common.cuh"

namespace sampt {

struct GemmEpi {
  // outputs (exactly one of out16 / out32 is used)
  __half* out16 = nullptr;       // fp16 output [M, ldc]  (bf16 when is_bf16)
  float* out32 = nullptr;        // fp32 output [rows, ldc]
  const float* resid = nullptr;  // fp32 residual added to out32 (indexed like out32, or row % resid_mod), may alias out32
  const float* bias = nullptr;   // [N] or null
  const int* rowmap = nullptr;   // [M] destination row for out32/resid (-1 = drop the row), or null = identity
  int ldc = 0;
  int act = 0;                   // 0 none, 1 GELU(erf), 3 GELU(tanh)
  int split_off = 0;             // >0: also write lo = fp16(v - hi) at column offset split_off (out16 only)
  int is_bf16 = 0;
  int resid_mod = 0;             // >0: residual row = dest row % resid_mod (broadcast of pos_embed over the frame batch)
  const int* skip = nullptr;     // device flag: != 0 -> the whole kernel returns at once (the mask decoder's on-device break)
  const float* acc_scale = nullptr;  // device scalar multiplied into the accumulator first (fp8-corrected GEMM: 2^-sB of the weight)
  int out_f8 = 0;                // with split_off > 0: instead of lo = fp16(v - hi) write the fp8 correction operands behind the hi
                                 // block: e4m3((v - hi) * 2^12) at BYTE offset 2*split_off + n, e4m3(v * 2^-3) at 3*split_off + n
};

// K-loop segments for split precision: segment i multiplies A[:, a_off[i] : a_off[i]+K] with B[:, b_off[i] : b_off[i]+K]
// (offsets in fp16 units).  f8[i] != 0: the segment's operands are e4m3 BYTES (K of them = K/2 fp16 units starting at the
// offset), multiplied with wgmma e4m3 at twice the fp16 rate.  gemm_tc issues every e4m3 segment before the fp16 ones into the
// one fp32 accumulator (gemm_tc.cu), whatever order the caller lists them in.
struct GemmSeg { int nseg; int a_off[3]; int b_off[3]; int f8[3]; };

// fp8-corrected split GEMM ("precision 6"), operand rows of 2K fp16 units:
//   A row: [ fp16(x) : K halves | e4m3((x - fp16(x)) * 2^12) : K bytes | e4m3(x * 2^-3) : K bytes ]
//   B row: [ fp16(w * 2^sB) : K halves | e4m3(w * 2^(sB-12)) : K bytes | e4m3((w * 2^sB - fp16(w * 2^sB)) * 2^3) : K bytes ]
// so that hi.hi (fp16) + lo8.hi8 + hi8.lo8 all accumulate at scale 2^sB; the epilogue multiplies by acc_scale = 2^-sB.
constexpr float F8_LO_SCALE = 4096.0f;   // 2^12 on the activation remainder
constexpr float F8_HI_SCALE = 0.125f;    // 2^-3 on the activation itself
inline GemmSeg make_seg_f8(int K) {
  GemmSeg s{};
  s.nseg = 3;
  s.a_off[0] = 0;             s.b_off[0] = 0;             s.f8[0] = 0;   // hi16 . hi16
  s.a_off[1] = K;             s.b_off[1] = K;             s.f8[1] = 1;   // lo8  . hi8
  s.a_off[2] = K + K / 2;     s.b_off[2] = K + K / 2;     s.f8[2] = 1;   // hi8  . lo8
  return s;
}

int gemm_tc(Ctx* c, cudaStream_t st, const void* A, int lda, const void* B, int ldb, int M, int N, int K, const GemmSeg& seg,
            const GemmEpi& ep);
bool gemm_f8c_applicable(int M, int N, int K);   // shapes the fp8-corrected segments (GemmSeg::f8) run on

// out_f8: the output row carries the fp8 correction operands of the proj GEMM instead of the fp16 remainder
int attn_tc(Ctx* c, cudaStream_t st, const __half* Qx, const __half* Kx, const __half* Vt, int BH, int Lq, int Lk, int Lkp,
            int DK, int HD, int nheads, __half* out, int ld_out, int split_off, int out_f8 = 0);

}  // namespace sampt
