// Order-preserving integer keys of fp32 and bf16 values, shared by the radix selects of topk.cu and action_sample.cu:
// a < b as floats (no NaN) <=> key(a) < key(b) as unsigned.  A positive NaN keys above +inf, a negative NaN below -inf.
// For a bf16 value v, Key<bf16>'s 16-bit key is the top half of Key<float>::of((float)v).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace {

template <typename T>
struct Key;
template <>
struct Key<float> {
  static constexpr int kBits = 32;
  __device__ static __forceinline__ uint32_t of(float x) {
    const uint32_t u = __float_as_uint(x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  }
  __device__ static __forceinline__ float value(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
  }
  __device__ static __forceinline__ uint32_t raw(const float* p) { return of(*p); }
};
template <>
struct Key<__nv_bfloat16> {
  static constexpr int kBits = 16;
  __device__ static __forceinline__ uint32_t of16(uint32_t u) { return (u & 0x8000u) ? (~u & 0xffffu) : (u | 0x8000u); }
  __device__ static __forceinline__ float value(uint32_t k) {
    const uint32_t u = (k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu);
    return __uint_as_float(u << 16);
  }
  __device__ static __forceinline__ uint32_t raw(const __nv_bfloat16* p) {
    return of16(*reinterpret_cast<const unsigned short*>(p));
  }
};

}  // namespace
