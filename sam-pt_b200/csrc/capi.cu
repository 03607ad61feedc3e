// Context management + small generic entry points of the C ABI (include/sampt_b200.h).
#include "common.cuh"
#include "kernels.cuh"
#include "../../include/sampt_b200.h"

namespace sampt {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }
}  // namespace sampt

using namespace sampt;

extern "C" const char* sampt_last_error(void) { return last_error(); }
extern "C" int sampt_version(void) { return 1; }

extern "C" int sampt_ctx_create(int device, sampt_ctx** out) {
  SAMPT_CHECK(out != nullptr, "sampt_ctx_create: out is null");
  SAMPT_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  SAMPT_CUDA(cudaGetDeviceProperties(&prop, device));
  SAMPT_CHECK(prop.major == 9 && prop.minor == 0, "libsampt_b200 is built for sm_90a only; device %d is sm_%d%d", device, prop.major,
              prop.minor);
  Ctx* c = new Ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  c->pinned_bytes = 1 << 20;
  SAMPT_CUDA(cudaMallocHost(&c->pinned, c->pinned_bytes));
  SAMPT_TRY(sgemm_init());
  *out = reinterpret_cast<sampt_ctx*>(c);
  return 0;
}
extern "C" int sampt_ctx_destroy(sampt_ctx* ctx) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  if (!c) return 0;
  if (c->pinned) cudaFreeHost(c->pinned);
  for (auto& kv : c->owned) cudaFree(kv.second.first);
  delete c;
  return 0;
}
extern "C" int sampt_ctx_set_workspace(sampt_ctx* ctx, void* dev_ptr, size_t bytes) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  c->ws_base = reinterpret_cast<char*>(dev_ptr);
  c->ws_bytes = bytes;
  c->ws_off = 0;
  return 0;
}
extern "C" int sampt_set_tensor(sampt_ctx* ctx, const char* name, void* dev_ptr, int dtype, int ndim, const int64_t* dims) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  SAMPT_CHECK(ndim >= 0 && ndim <= 6, "sampt_set_tensor(%s): ndim %d out of range", name, ndim);
  TensorRef t;
  t.ptr = dev_ptr; t.dtype = dtype; t.ndim = ndim;
  for (int i = 0; i < ndim; ++i) t.dims[i] = dims[i];
  c->tensors[std::string(name)] = t;
  return 0;
}
extern "C" int sampt_unset_tensors(sampt_ctx* ctx, const char* prefix) {
  Ctx* c = reinterpret_cast<Ctx*>(ctx);
  const std::string p(prefix);
  for (auto it = c->tensors.begin(); it != c->tensors.end();) {
    if (it->first.compare(0, p.size(), p) == 0) it = c->tensors.erase(it);
    else ++it;
  }
  return 0;
}
extern "C" long long sampt_launch_count(sampt_ctx* ctx) { return reinterpret_cast<Ctx*>(ctx)->launches; }

extern "C" int sampt_linear_f32(sampt_ctx* ctx, const float* X, int ldx, const float* W, int ldw, const float* bias,
                                const float* residual, int ldr, float* Y, int ldy, int M, int N, int K, int act, void* stream) {
  return sgemm_nt(reinterpret_cast<Ctx*>(ctx), reinterpret_cast<cudaStream_t>(stream), X, ldx, W, ldw, bias, residual, ldr,
                  Y, ldy, M, N, K, act);
}
