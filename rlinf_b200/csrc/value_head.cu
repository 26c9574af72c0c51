// Value head of the reasoning PPO critic on a plan's rows, read in place: the reference's LinearForLastLayer(H, 1)
// (rlinf/hybrid_engines/megatron/megatron_model_manager.py:136-162) - a bf16 nn.Linear without bias whose output is
// cast with .float() - evaluated only on the rows a critic loss reads, and its backward.
//
//   forward   v[i]  = float(bf16(sum_h x[rows[i], h] w[h]))                    one warp per row
//   backward  dx[t] = bf16(bf16(g[inv_map[t]]) w), zeros where inv_map[t] < 0   every row of the shard written once
//             dw    = bf16(sum_i bf16(g[i]) x[rows[i]])                         fp32 partials over fixed row chunks,
//                                                                               then a fixed-order finish
// g is rounded to bf16 first: the backward of .float() casts the gradient back to the Linear's dtype.  Sums are
// fp32 in an order fixed by n and H alone: no floating-point atomics, nothing that depends on the SM count.
//
// Bytes (HBM): forward n H 2 read; backward n H 2 read (dW) + T H 2 written (dX), plus the dW partials
// ceil(n / kChunk) H 4, written and read once, which stay in L2 at the sizes of a micro-batch.
#include <cuda_bf16.h>

#include "common.cuh"

namespace {

constexpr int kVec = 8;                   // bf16 per 16-byte access
constexpr int kFwdThreads = 256;          // 8 rows per CTA
constexpr int kChunk = 64;                // rows per dW partial
constexpr int kWgThreads = 128;           // 128 x 8 = 1024 columns per dW partial CTA
constexpr int kFinThreads = 256;          // 8 warps x 32 columns per finish CTA

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[kVec]) {
  const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 t = __bfloat1622float2(p[k]);
    f[2 * k] = t.x;
    f[2 * k + 1] = t.y;
  }
}

__device__ __forceinline__ uint4 pack8(const float (&f)[kVec]) {
  uint4 u;
  __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int k = 0; k < 4; ++k) p[k] = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
  return u;
}

__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// lane l accumulates 16-byte vectors l, l + 32, ... of its row in order, then a fixed butterfly over the warp
__global__ void __launch_bounds__(kFwdThreads) value_head_fwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                                     int64_t row_stride,
                                                                     const int64_t* __restrict__ rows, int64_t n,
                                                                     int nvec, const uint4* __restrict__ w,
                                                                     float* __restrict__ v) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * (kFwdThreads / 32) + (threadIdx.x >> 5);
  if (i >= n) return;
  const int64_t r = rows[i];
  if (r < 0) {
    if (lane == 0) v[i] = 0.0f;
    return;
  }
  const uint4* xr = reinterpret_cast<const uint4*>(x + r * row_stride);
  float acc = 0.0f;
  constexpr int kU = 4;
  for (int c0 = lane; c0 < nvec; c0 += 32 * kU) {
    uint4 xs[kU], ws[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int c = c0 + 32 * u;
      if (c < nvec) {
        xs[u] = __ldcs(xr + c);
        ws[u] = __ldg(w + c);
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      if (c0 + 32 * u < nvec) {
        float a[kVec], b[kVec];
        unpack8(xs[u], a);
        unpack8(ws[u], b);
#pragma unroll
        for (int k = 0; k < kVec; ++k) acc = fmaf(a[k], b[k], acc);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) v[i] = round_bf16(acc);
}

// dx[t] = bf16(bf16(g[inv_map[t]]) * w): one 16-byte vector per thread and iteration
__global__ void __launch_bounds__(256) value_head_dx_kernel(const int64_t* __restrict__ inv_map, int64_t T, int nvec,
                                                            const float* __restrict__ g, const uint4* __restrict__ w,
                                                            uint4* __restrict__ dx) {
  const int64_t total = T * nvec;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
    const int64_t t = e / nvec;
    const int c = (int)(e - t * nvec);
    const int64_t m = inv_map[t];
    float o[kVec];
    if (m < 0) {
#pragma unroll
      for (int k = 0; k < kVec; ++k) o[k] = 0.0f;
    } else {
      const float gb = round_bf16(g[m]);
      float b[kVec];
      unpack8(__ldg(w + c), b);
#pragma unroll
      for (int k = 0; k < kVec; ++k) o[k] = gb * b[k];
    }
    __stcs(dx + e, pack8(o));
  }
}

// partial[chunk, h] = sum over the chunk's rows, in order, of bf16(g[i]) x[rows[i], h] (pad rows skipped).  The
// chunk's row indices and gradients are staged in shared memory first, so the row loads do not wait on index loads.
__global__ void __launch_bounds__(kWgThreads) value_head_dw_partial_kernel(const __nv_bfloat16* __restrict__ x,
                                                                           int64_t row_stride,
                                                                           const int64_t* __restrict__ rows,
                                                                           int64_t n, int nvec,
                                                                           const float* __restrict__ g,
                                                                           float* __restrict__ partial) {
  __shared__ int64_t srow[kChunk];
  __shared__ float sg[kChunk];
  const int64_t i0 = (int64_t)blockIdx.x * kChunk;
  for (int u = threadIdx.x; u < kChunk; u += kWgThreads) {
    const int64_t i = i0 + u;
    const int64_t r = i < n ? rows[i] : -1;
    srow[u] = r;
    sg[u] = r < 0 ? 0.0f : round_bf16(g[i]);
  }
  __syncthreads();
  const int c = blockIdx.y * kWgThreads + threadIdx.x;
  if (c >= nvec) return;
  float acc[kVec];
#pragma unroll
  for (int k = 0; k < kVec; ++k) acc[k] = 0.0f;
  constexpr int kU = 8;
#pragma unroll 1
  for (int ub = 0; ub < kChunk; ub += kU) {
    uint4 xs[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int64_t r = srow[ub + u];
      xs[u] = r < 0 ? make_uint4(0u, 0u, 0u, 0u) : __ldcs(reinterpret_cast<const uint4*>(x + r * row_stride) + c);
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      float a[kVec];
      unpack8(xs[u], a);
      const float gu = sg[ub + u];
#pragma unroll
      for (int k = 0; k < kVec; ++k) acc[k] = fmaf(gu, a[k], acc[k]);
    }
  }
  float4* p = reinterpret_cast<float4*>(partial + (int64_t)blockIdx.x * nvec * kVec + (int64_t)c * kVec);
  p[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  p[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// dw[h] = bf16(sum over chunks of partial[chunk, h]): warp w sums chunks w, w + 8, ... in order, then warp 0 adds the
// eight warp sums in order
__global__ void __launch_bounds__(kFinThreads) value_head_dw_finish_kernel(const float* __restrict__ partial,
                                                                           int64_t nchunk, int H,
                                                                           __nv_bfloat16* __restrict__ dw) {
  __shared__ float red[kFinThreads / 32][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int h = blockIdx.x * 32 + lane;
  float acc = 0.0f;
  for (int64_t ch = warp; ch < nchunk; ch += kFinThreads / 32) acc += partial[ch * H + h];
  red[warp][lane] = acc;
  __syncthreads();
  if (warp == 0) {
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < kFinThreads / 32; ++k) s += red[k][lane];
    dw[h] = __float2bfloat16_rn(s);
  }
}

int64_t num_chunks(int64_t n) { return (n + kChunk - 1) / kChunk; }

bool bad_h(int64_t H) { return H % 64 != 0 || H < 64 || H > 8192; }

int grid_for(int64_t total) {
  const int64_t cap = (int64_t)rb::sm_count() * 16;  // a grid-stride loop: the bits do not depend on the grid
  int64_t b = (total + 255) / 256;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

}  // namespace

extern "C" int64_t rb200_value_head_workspace_bytes(int64_t n, int64_t H) {
  if (n <= 0 || bad_h(H)) return -1;
  return num_chunks(n) * H * 4;
}

extern "C" int rb200_value_head_fwd(const void* x, int64_t row_stride, const int64_t* rows, int64_t n, int64_t H,
                                    const void* w, float* v, rb200_stream_t stream) {
  if (!x || !rows || !w || !v) return RB200_E_NULL;
  if (n <= 0 || bad_h(H) || row_stride < H) return RB200_E_SHAPE;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w)) & 15 || row_stride % kVec != 0)
    return RB200_E_ALIGN;
  const int64_t blocks = (n + kFwdThreads / 32 - 1) / (kFwdThreads / 32);
  if (blocks > 0x7fffffff) return RB200_E_SHAPE;
  value_head_fwd_kernel<<<(unsigned)blocks, kFwdThreads, 0, rb::as_stream(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), row_stride, rows, n, (int)(H / kVec), static_cast<const uint4*>(w), v);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_value_head_bwd(const void* x, int64_t row_stride, const int64_t* rows, int64_t n, int64_t H,
                                    const float* g, const void* w, const int64_t* inv_map, int64_t T, void* dx,
                                    void* dw, void* workspace, int64_t workspace_bytes, rb200_stream_t stream) {
  if (!g || (!dx && !dw)) return RB200_E_NULL;
  if (bad_h(H)) return RB200_E_SHAPE;
  const int nvec = (int)(H / kVec);
  cudaStream_t st = rb::as_stream(stream);
  if (dx) {
    if (!inv_map || !w) return RB200_E_NULL;
    if (T <= 0) return RB200_E_SHAPE;
    if ((reinterpret_cast<uintptr_t>(dx) | reinterpret_cast<uintptr_t>(w)) & 15) return RB200_E_ALIGN;
  }
  if (dw) {
    if (!x || !rows || !workspace) return RB200_E_NULL;
    if (n <= 0 || row_stride < H) return RB200_E_SHAPE;
    if (workspace_bytes < rb200_value_head_workspace_bytes(n, H)) return RB200_E_ARG;
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(workspace)) & 15 || row_stride % kVec != 0)
      return RB200_E_ALIGN;
    if (num_chunks(n) > 0x7fffffff) return RB200_E_SHAPE;
  }
  if (dx) {
    value_head_dx_kernel<<<grid_for(T * nvec), 256, 0, st>>>(inv_map, T, nvec, g, static_cast<const uint4*>(w),
                                                              static_cast<uint4*>(dx));
    rb::count_launch();
  }
  if (dw) {
    const int64_t nchunk = num_chunks(n);
    float* partial = static_cast<float*>(workspace);
    const dim3 grid((unsigned)nchunk, (unsigned)((nvec + kWgThreads - 1) / kWgThreads));
    value_head_dw_partial_kernel<<<grid, kWgThreads, 0, st>>>(static_cast<const __nv_bfloat16*>(x), row_stride, rows,
                                                              n, nvec, g, partial);
    rb::count_launch();
    value_head_dw_finish_kernel<<<(unsigned)(H / 32), kFinThreads, 0, st>>>(partial, nchunk, (int)H,
                                                                             static_cast<__nv_bfloat16*>(dw));
    rb::count_launch();
  }
  RB_RETURN_LAUNCH();
}
