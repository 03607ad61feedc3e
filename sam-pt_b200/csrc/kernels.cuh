// Internal launcher declarations shared by the pipelines (not part of the C ABI; see include/sampt_b200.h).
#pragma once
#include "common.cuh"

namespace sampt {

// ---- fp32 GEMM (sgemm.cu):  Y = act(X W^T + bias) (+ residual);  act: 0 none, 1 GELU(erf), 2 ReLU, 3 GELU(tanh)
int sgemm_nt(Ctx* c, cudaStream_t st, const float* X, int ldx, const float* W, int ldw, const float* bias,
             const float* residual, int ldr, float* Y, int ldy, int M, int N, int K, int act);

int sgemm_init();
int sgemm_nt_skip(Ctx* c, cudaStream_t st, const float* X, int ldx, const float* W, int ldw, const float* bias,
                  const float* residual, int ldr, float* Y, int ldy, int M, int N, int K, int act, const int* skip);

// ---- PIPS (pips_kernels.cu)
struct PipsWin {
  int N, S, stride, T;
  const int* wp;           // device "window params": [0] = current frame f, [1] = n_missing, [2+s] = real frame index feeding
                           // window slot s (tail padding / flipped pass).  In device memory so a captured CUDA graph of
                           // one window can be replayed for every window of the clip.
  const float* pyr[4];     // pyramid level base pointers, each (T, H_l, W_l, 128) channels-last
  int H[4], W[4];
  float* coords;           // (N, S, 2) feature-map pixels
  float* ffeats;           // (N, S, 128)
  float* feat_init;        // (N, 128)
  float* traj;             // (T, N, 2) image pixels (pass-local time order)
  float* vis;              // (T, N)
  int* cur;                // (N) current_point_frames
  const uint8_t* active;   // (N) 1 = point takes part in this window
  int sample_feat;         // 1: feat_init <- bilinear_sample2d(fmaps[slot 0]) (init pass), 0: use stored feat_init
};

int conv_nhwc_f32(Ctx* c, cudaStream_t st, const float* in, const float* w, const float* bias, float* out, int Nimg,
                  int H, int W, int Cin, int Cout, int R, int S, int stride, int pad, const int* skip = nullptr);
int im2col_nhwc_split(Ctx* c, cudaStream_t st, const float* in, __half* A, int Nimg, int H, int W, int Cin, int R, int S, int stride,
                      int pad, int Kp);
int im2col_conv1_split(Ctx* c, cudaStream_t st, const void* frames, int is_f32, __half* A, int Nimg, int H, int W, int Kp);
int conv7x7s2(Ctx* c, cudaStream_t st, const void* frames, int is_f32, const float* w, const float* bias, float* out, int Nimg,
              int H, int W);
int inorm_stats(Ctx* c, cudaStream_t st, const float* x, float* stats, double* part, int Nimg, int HW, int C);
int inorm_apply(Ctx* c, cudaStream_t st, const float* x, const float* stats, const float* res, const float* res_stats,
                float* y, int Nimg, int HW, int C, int relu_before_add, int relu_after);
int resize_ac_concat(Ctx* c, cudaStream_t st, const float* in, float* out, int Nimg, int Hi, int Wi, int C, int Ho, int Wo,
                     int Ctot, int coff);
int avgpool2_nhwc(Ctx* c, cudaStream_t st, const float* in, float* out, int Nimg, int Hi, int Wi, int C);
int pips_window_init(Ctx* c, cudaStream_t st, const PipsWin& w);
int pips_corr(Ctx* c, cudaStream_t st, const PipsWin& w, float* xin, int ldx);
int mixer_token(Ctx* c, cudaStream_t st, float* x, float* xln, const uint8_t* active, int N, const float* ln_w,
                const float* ln_b, const float* w1, const float* b1, const float* w2, const float* b2, const float* ln2_w,
                const float* ln2_b, int do_token_mix);
int mixer_mean(Ctx* c, cudaStream_t st, const float* xln, float* xm, int N, int S, int D);
int pips_update(Ctx* c, cudaStream_t st, const PipsWin& w, const float* delta, const float* gn_w, const float* gn_b,
                const float* up_w, const float* up_b);
int pips_link(Ctx* c, cudaStream_t st, const PipsWin& w, const float* vis_w, const float* vis_b, float thr0, int T);

// ---- split-precision GEMM with a power-of-two weight scale (tinyvit.cu): Y[M, N] = act(A W^T 2^-s + bias) (+ resid), A and W
// hi|lo with 2*Kp halves per row, W registered under `wname` and its accumulator scale 2^-s under `wname + "s"`
int tv_gemm(Ctx* c, cudaStream_t st, const __half* A, const std::string& wname, int M, int N, int Kp, const float* bias, int act,
            float* out32, const float* resid);

}  // namespace sampt

namespace sampt {
// ---- SAM ViT helper kernels (vit_kernels.cu)
int pil_resize(Ctx* c, cudaStream_t st, const uint8_t* in, uint8_t* tmp, uint8_t* out, int B, int H, int W, int Ho, int Wo,
               const int* hb, const int* hk, int hks, const int* vb, const int* vk, int vks);
int preprocess_im2col(Ctx* c, cudaStream_t st, const uint8_t* img, __half* A, int B, int Hr, int Wr, int G, int P, int ld,
                      int split_off, const float* mean, const float* stdv);
int im2col_f32(Ctx* c, cudaStream_t st, const float* img, __half* A, int B, int G, int P, int ld, int split_off);
int ln_rows(Ctx* c, cudaStream_t st, const float* x, int ldx, const int* src, const float* gamma, const float* beta, float eps,
            __half* out, int ldo, int split_off, int Mout, int D, int normalize, int f8 = 0);
int attn_prep(Ctx* c, cudaStream_t st, const __half* qkv, int ldq, const float* relh, const float* relw, __half* Qx, __half* Kx,
              __half* Vt, int nwb, int nheads, int S, int Lkp, int DK, int D, int HD, float scale);
int attn_prep2(Ctx* c, cudaStream_t st, const __half* qkv, int ldq, const float* relh, const float* relw, __half* Qx, __half* Kx,
               __half* Vt, int nwb, int nheads, int S, int Lkp, int DK, int D, int HD, float scale);
int neck_ln_im2col(Ctx* c, cudaStream_t st, const float* y1, const float* gamma, const float* beta, __half* A, int B, int G, int C,
                   int ld, int split_off);
int neck_ln_nchw(Ctx* c, cudaStream_t st, const float* y2, const float* gamma, const float* beta, float* out, int B, int GG, int C);
}  // namespace sampt
