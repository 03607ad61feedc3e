// Shared infrastructure of libsampt_b200.so: error reporting, the per-device context (weight registry +
// bump-allocated workspace), small device helpers.  sm_90a only.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <string>
#include <unordered_map>
#include <vector>
#include <map>

namespace sampt {

// ---------------------------------------------------------------- error handling (thread-local message)
void set_error(const char* fmt, ...);
const char* last_error();

#define SAMPT_CUDA(expr)                                                                         \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      sampt::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return -1;                                                                                 \
    }                                                                                            \
  } while (0)

#define SAMPT_CHECK(cond, ...)                 \
  do {                                         \
    if (!(cond)) {                             \
      sampt::set_error(__VA_ARGS__);           \
      return -2;                               \
    }                                          \
  } while (0)

#define SAMPT_TRY(expr)        \
  do {                         \
    int _r = (expr);           \
    if (_r != 0) return _r;    \
  } while (0)

#define SAMPT_LAUNCH_CHECK() SAMPT_CUDA(cudaGetLastError())

// ---------------------------------------------------------------- context
struct TensorRef {
  void* ptr = nullptr;
  int dtype = 0;  // 0 = f32, 1 = f16, 2 = u8, 3 = i32, 4 = bf16
  int ndim = 0;
  int64_t dims[6] = {0, 0, 0, 0, 0, 0};
  int64_t numel() const {
    int64_t n = 1;
    for (int i = 0; i < ndim; ++i) n *= dims[i];
    return n;
  }
};

struct Ctx {
  int device = 0;
  int num_sms = 132;
  std::unordered_map<std::string, TensorRef> tensors;  // caller-owned device memory, registered by name
  // workspace: caller-owned slab, bump allocated per pipeline call
  char* ws_base = nullptr;
  size_t ws_bytes = 0;
  size_t ws_off = 0;
  // pinned host scratch for tiny read-backs
  void* pinned = nullptr;
  size_t pinned_bytes = 0;
  long long launches = 0;  // kernels launched through this ctx (bench.py reports it as gpu_launches)
  // decoder slab + captured CUDA graphs of the SAM refinement chain (decoder.cu)
  char* dec_base = nullptr;
  size_t dec_bytes = 0, dec_off = 0;
  cudaStream_t cap_stream = nullptr;
  std::map<std::vector<int>, void*> graph_cache;
  std::map<int, void*> dec_slots;   // per decode slot: one buffer set carved from the slab, shared by the slot's graphs
  const float* hq_feat = nullptr;  // HQ-SAM features of the current frame (decoder.cu), caller-owned
  // library-owned device buffers that outlive a call (e.g. the ViT's image-independent padding tokens, vit_pipeline.cu);
  // freed by sampt_vit_cache_clear / sampt_ctx_destroy
  std::map<std::string, std::pair<void*, size_t>> owned;
  // per-DEVICE lazily applied kernel attributes (cudaFuncSetAttribute is per device: a process-wide `static bool` would skip the
  // second device of a multi-GPU process) and per-ctx scratch of the encoder pipelines
  std::map<std::string, size_t> func_smem;
  __half* fnet_im2col = nullptr;        // im2col operand of the tensor-core BasicEncoder path (null -> fp32 CUDA-core convs)
  std::string fnet_prefix = "pips.";    // weight-name prefix of the encoder being run ("pips." | "cot.")

  const TensorRef* find(const std::string& name) const {
    auto it = tensors.find(name);
    return it == tensors.end() ? nullptr : &it->second;
  }
  // optional dedicated slab for the ViT encoder so that it can run on its own stream concurrently with the PIPS / decode
  // pipelines (which bump-allocate from the general workspace)
  char* vit_base = nullptr;
  size_t vit_bytes = 0;
  void ws_reset() { ws_off = 0; }
  void* ws_alloc(size_t bytes) {
    size_t a = (ws_off + 255) & ~size_t(255);
    if (a + bytes > ws_bytes) return nullptr;
    ws_off = a + bytes;
    return ws_base + a;
  }
};

template <typename T>
inline int ws_get(Ctx* c, T** out, size_t count, const char* what) {
  *out = reinterpret_cast<T*>(c->ws_alloc(count * sizeof(T)));
  if (!*out) {
    set_error("workspace exhausted allocating %s (%zu bytes, %zu of %zu used)", what, count * sizeof(T), c->ws_off,
              c->ws_bytes);
    return -3;
  }
  return 0;
}

inline int get_f32(const Ctx* c, const std::string& name, const float** out) {
  const TensorRef* t = c->find(name);
  if (!t) { set_error("tensor '%s' is not registered", name.c_str()); return -4; }
  if (t->dtype != 0) { set_error("tensor '%s' is not float32", name.c_str()); return -4; }
  *out = reinterpret_cast<const float*>(t->ptr);
  return 0;
}
inline int get_f16(const Ctx* c, const std::string& name, const __half** out) {
  const TensorRef* t = c->find(name);
  if (!t) { set_error("tensor '%s' is not registered", name.c_str()); return -4; }
  if (t->dtype != 1) { set_error("tensor '%s' is not float16", name.c_str()); return -4; }
  *out = reinterpret_cast<const __half*>(t->ptr);
  return 0;
}

// raise a kernel's dynamic shared-memory limit once per ctx (= per device)
template <typename F>
inline int ensure_func_smem(Ctx* c, const char* key, F func, size_t bytes) {
  auto it = c->func_smem.find(key);
  if (it == c->func_smem.end() || it->second < bytes) {
    SAMPT_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    c->func_smem[key] = bytes;
  }
  return 0;
}

inline unsigned cdiv(long long a, long long b) { return (unsigned)((a + b - 1) / b); }

// ---------------------------------------------------------------- device helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// exact (erf) GELU, as torch.nn.GELU() default
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// tanh-approximated GELU, torch.nn.GELU(approximate="tanh")
__device__ __forceinline__ float gelu_tanh(float x) {
  return 0.5f * x * (1.0f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
}

// block-wide sum for blockDim.x <= 1024; `red` must hold 32 floats
__device__ __forceinline__ float block_sum(float v, float* red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  int nw = (blockDim.x + 31) >> 5;
  float r = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (w == 0) r = warp_sum(r);
  if (threadIdx.x == 0) red[0] = r;
  __syncthreads();
  r = red[0];
  return r;
}

}  // namespace sampt
