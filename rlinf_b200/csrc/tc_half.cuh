// Device helpers shared by the fp16-split wgmma kernels of the PPO update (tc_gemm_h.cu, tc_forward_h.cu,
// tc_backward_h.cu): operand scaling, the fp32 -> fp16 (hi, lo) split, bulk copies and ring-slot release.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

#include "tma.cuh"

namespace rb {
namespace tch {

constexpr int kWeightScaleLog2 = 10;  // weights are stored as fp16 (hi, lo) of w * 2^10 (|w| <~ 1: both halves normal)

// 1-D bulk copy global -> shared, completion counted on an mbarrier
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   tma::smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(tma::smem_u32(bar))
               : "memory");
}
// one warp's share of freeing a ring slot (the barrier counts one arrival per reading warp)
__device__ __forceinline__ void warp_arrive(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) tma::mbar_arrive(bar);
}

// Operand layouts: K-major SWIZZLE_64B (forward pack: 64-B rows, SBO 512), MN-major SWIZZLE_128B (dgrad pack: SBO 1024 B
// between 8 K-rows, LBO 4096 B between 64-wide N groups), MN-major SWIZZLE_64B (wgrad H: SBO 512, LBO 2048).
constexpr uint32_t kSw128 = 1, kSw64 = 2;

// 2^s as a float (s in [-126, 127])
__device__ __forceinline__ float pow2i(int s) { return __int_as_float((s + 127) << 23); }
// power-of-two scale that brings max|x| = amax to [2^13, 2^14): fp16 keeps 11 bits for every |x| >= amax * 2^-27
__device__ __forceinline__ int scale_log2_for(float amax) {
  const int e = (int)((__float_as_uint(amax) >> 23) & 0xffu) - 127;
  if (!(amax > 0.0f) || e < -120) return 0;
  int s = 13 - e;
  return s > 100 ? 100 : (s < -100 ? -100 : s);
}

// Scale of an input operand (the observations of layer 0).  Unscaled, the (hi, lo) split of x is exact to 2^-22
// relative down to |x| = 2^-3 and to 2^-25 absolute below (lo in fp16's subnormals), and hi stays finite below 65520; so
// for max|x| in [2^-1, 2^15) every element is split to within 2^-24 * max|x|, fp32-level against the |W|.|x| of the
// product, and the operand stays unscaled: its results are those of the unscaled split bit for bit.  Outside that range
// (tiny inputs lose bits to subnormals, huge ones overflow to inf) it is scaled like a gradient operand.
__device__ __forceinline__ int input_scale_log2_for(float amax) {
  const int e = (int)((__float_as_uint(amax) >> 23) & 0xffu) - 127;
  return (e >= -1 && e <= 14) ? 0 : scale_log2_for(amax);
}

// (x0, x1) -> packed fp16 pairs hi = rn(x), lo = rn(x - hi)
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 hh = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(hh);
  const __half2 ll = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&hh);
  lo = *reinterpret_cast<const uint32_t*>(&ll);
}

// wgmma A fragment (m64k16, this thread's rows r0 / r0 + 8, k columns c0 + 2t + {0, 1, 8, 9}) of a row-major fp32
// [rows x 32] SWIZZLE_128B landing tile, scaled and split into fp16 hi / lo
__device__ __forceinline__ void a_frag_rows(const uint8_t* tile, int r0, int c0, float scale, uint32_t (&hi)[4],
                                            uint32_t (&lo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + (i & 1) * 8, c = c0 + (i >> 1) * 8;
    const float2 x = *reinterpret_cast<const float2*>(tile + r * 128 + ((((c >> 2) ^ (r & 7))) << 4) + (c & 3) * 4);
    split2(x.x * scale, x.y * scale, hi[i], lo[i]);
  }
}

// the forward epilogue's tanh (MUFU exp, 3e-7 absolute)
__device__ __forceinline__ float tanh_fast(float x) {
  const float t = __expf(-2.0f * fabsf(x));
  return copysignf(__fdividef(1.0f - t, 1.0f + t), x);
}

// One split item = (row r, 8 floats cp of its 32): the two 16-byte chunks of fp32 row r (SWIZZLE_128B, 128-B rows) ->
// one 16-byte chunk each of fp16 hi and lo row r (SWIZZLE_64B, 64-B rows), as packed half2 words of x * scale
__device__ __forceinline__ void split_item(const uint8_t* src, int r, int cp, float scale, uint4& hi, uint4& lo) {
  const uint8_t* srow = src + r * 128;
  const float4 x0 = *reinterpret_cast<const float4*>(srow + (((2 * cp) ^ (r & 7)) << 4));
  const float4 x1 = *reinterpret_cast<const float4*>(srow + (((2 * cp + 1) ^ (r & 7)) << 4));
  split2(x0.x * scale, x0.y * scale, hi.x, lo.x);
  split2(x0.z * scale, x0.w * scale, hi.y, lo.y);
  split2(x1.x * scale, x1.y * scale, hi.z, lo.z);
  split2(x1.z * scale, x1.w * scale, hi.w, lo.w);
}
// split_item with a scale per column: sc[0..7] for the 8 floats of the item
__device__ __forceinline__ void split_item_cols(const uint8_t* src, int r, int cp, const float* sc, uint4& hi, uint4& lo) {
  const uint8_t* srow = src + r * 128;
  const float4 x0 = *reinterpret_cast<const float4*>(srow + (((2 * cp) ^ (r & 7)) << 4));
  const float4 x1 = *reinterpret_cast<const float4*>(srow + (((2 * cp + 1) ^ (r & 7)) << 4));
  const float4 s0 = *reinterpret_cast<const float4*>(sc), s1 = *reinterpret_cast<const float4*>(sc + 4);
  split2(x0.x * s0.x, x0.y * s0.y, hi.x, lo.x);
  split2(x0.z * s0.z, x0.w * s0.w, hi.y, lo.y);
  split2(x1.x * s1.x, x1.y * s1.y, hi.z, lo.z);
  split2(x1.z * s1.z, x1.w * s1.w, hi.w, lo.w);
}
__device__ __forceinline__ int split_item_dst(int r, int cp) { return r * 64 + ((cp ^ ((r >> 1) & 3)) << 4); }

// fp32 [R rows x 32 floats] SWIZZLE_128B tile -> fp16 hi / lo [R rows x 32 halfs] SWIZZLE_64B tiles
template <int NT>
__device__ __forceinline__ void split_tile(const uint8_t* __restrict__ src, uint8_t* __restrict__ hi, uint8_t* __restrict__ lo,
                                           int rows, int t, float scale) {
  const int items = rows * 4;
#pragma unroll 2
  for (int i = t; i < items; i += NT) {
    const int r = i >> 2, cp = i & 3;
    uint4 h, l;
    split_item(src, r, cp, scale, h, l);
    *reinterpret_cast<uint4*>(hi + split_item_dst(r, cp)) = h;
    *reinterpret_cast<uint4*>(lo + split_item_dst(r, cp)) = l;
  }
}

// One warp: a landed fp32 [32 rows x 32 floats] SWIZZLE_128B box (4 KB) split over itself - fp16 hi [32 x 32 halfs]
// SWIZZLE_64B in its first 2 KB, lo in the second.  A (hi, lo) pair takes the 4 bytes of its float, so it fits; every
// lane holds its 4 items in registers until the whole warp has read the box.
__device__ __forceinline__ void split_box_in_place(uint8_t* box, int lane, float scale) {
  uint4 h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) split_item(box, (lane >> 2) + 8 * j, lane & 3, scale, h[j], l[j]);
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int d = split_item_dst((lane >> 2) + 8 * j, lane & 3);
    *reinterpret_cast<uint4*>(box + d) = h[j];
    *reinterpret_cast<uint4*>(box + 2048 + d) = l[j];
  }
}

}  // namespace tch
}  // namespace rb
