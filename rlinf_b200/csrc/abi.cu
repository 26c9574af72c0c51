// ABI bookkeeping: version, error strings, device info, per-device scratch.
#include "common.cuh"

namespace rb {
static unsigned long long g_launches = 0;
void count_launch(int n) { g_launches += (unsigned long long)n; }
unsigned long long launches() { return g_launches; }
double* device_scratch(int n_doubles_min) {
  static double* ptr[64] = {nullptr};
  static int cap[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  if (cap[dev] < n_doubles_min) {
    // grow-only; the old block is intentionally leaked if a larger one is ever needed while
    // earlier launches may still reference it (sizes used by this library are fixed and tiny).
    int n = n_doubles_min < 4096 ? 4096 : n_doubles_min;
    double* p = nullptr;
    if (cudaMalloc(&p, sizeof(double) * (size_t)n) != cudaSuccess) return nullptr;
    cudaMemset(p, 0, sizeof(double) * (size_t)n);
    ptr[dev] = p;
    cap[dev] = n;
  }
  return ptr[dev];
}
float* partials_scratch(int64_t n_floats_min) {
  static float* ptr[64] = {nullptr};
  static int64_t cap[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  if (cap[dev] < n_floats_min) {  // grow-only, the old block is leaked (captured graphs may still reference it)
    float* p = nullptr;
    if (cudaMalloc(&p, sizeof(float) * (size_t)n_floats_min) != cudaSuccess) return nullptr;
    ptr[dev] = p;
    cap[dev] = n_floats_min;
  }
  return ptr[dev];
}
}  // namespace rb

namespace rb { unsigned long long launches(); }
extern "C" uint64_t rb200_launch_count(void) { return rb::launches(); }

extern "C" int rb200_abi_version(void) { return RB200_ABI_VERSION; }

extern "C" const char* rb200_strerror(int code) {
  switch (code) {
    case RB200_OK: return "ok";
    case RB200_E_NULL: return "required pointer is NULL";
    case RB200_E_SHAPE: return "non-positive or inconsistent dimension";
    case RB200_E_ARG: return "invalid scalar argument";
    case RB200_E_ALIGN: return "pointer not sufficiently aligned";
    case RB200_E_UNSUPPORTED: return "unsupported configuration";
    default:
      if (code > 0) return cudaGetErrorString((cudaError_t)code);
      return "unknown rlinf_b200 error";
  }
}

extern "C" int rb200_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  RB_CHECK_CUDA(cudaGetDevice(&dev));
  int v = 0;
  if (sm_count) { RB_CHECK_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev)); *sm_count = v; }
  if (cc_major) { RB_CHECK_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev)); *cc_major = v; }
  if (cc_minor) { RB_CHECK_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev)); *cc_minor = v; }
  return RB200_OK;
}
