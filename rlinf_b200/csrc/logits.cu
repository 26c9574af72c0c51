// SURVEY 8(f)3: token log-probabilities and entropies straight from the logits, forward and backward, one pass each.
//
// Reference op chains replaced (rlinf/utils/utils.py):
//   compute_logprobs_from_logits  (:454-492)  logprobs = -F.cross_entropy(logits, target, reduction="none")
//   compute_entropy_from_logits   (:495-512)  logp = log_softmax(logits); p = exp(logp); H = -sum(where(p > 0, p*logp, 0))
// and what their callers do around them: `logits.div_(temperature)` (workers/actor/fsdp_actor_worker.py:478) and the
// OpenVLA action-bin window `logits[..., :vocab-n_bins] = -inf; logits[..., vocab:] = -inf`
// (models/embodiment/openvla_oft/rlinf/openvla_oft_action_model.py:546-551), folded in as `inv_temperature` and
// `[v_lo, v_hi)`.  The reference materialises log_softmax (N x V), exp of it (N x V), the product (N x V) and autograd
// keeps them for the backward; here the forward reads every logit ONCE and writes 12 bytes per row (logprob, entropy,
// logsumexp), and the backward reads the logits once more and writes the gradient once:
//   z_i = x_i * inv_T;  lse = log sum exp z;  logprob = z_target - lse;  H = lse - sum_i p_i z_i,  p_i = exp(z_i - lse)
//   (accumulated relative to the running maximum: H = log s - sum e^(z-m) (z-m) / s, no cancellation)
//   dL/dx_i = inv_T * ( g_lp * (1[i = target] - p_i)  -  g_H * p_i * (z_i - lse + H) )
// HBM-bound: algorithmic bytes = N*V*sizeof(logit) forward, 2x that backward.  One CTA per row for vocabulary-sized rows
// (online softmax per thread over 16-byte loads, one block combine), one warp per row for short windows.
#include <cuda_bf16.h>

#include "common.cuh"
#include "softmax_acc.cuh"

namespace {

constexpr int kThreads = 256;

using rb::smx::Acc;
using rb::smx::acc_add4;
using rb::smx::acc_init;
using rb::smx::warp_merge;

template <typename T>
__device__ __forceinline__ float load1(const T* p);
template <>
__device__ __forceinline__ float load1<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float load1<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// 16-byte streaming load -> VPT floats
template <typename T>
struct Vec;
template <>
struct Vec<float> {
  static constexpr int N = 4;
  __device__ static __forceinline__ void load(const float* p, float (&v)[4]) {
    const float4 x = __ldcs(reinterpret_cast<const float4*>(p));
    v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
  }
  __device__ static __forceinline__ void store(float* p, const float (&v)[4]) {
    __stcs(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
  }
};
template <>
struct Vec<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ static __forceinline__ void load(const __nv_bfloat16* p, float (&v)[8]) {
    const uint4 x = __ldcs(reinterpret_cast<const uint4*>(p));
    const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      v[2 * i] = __uint_as_float(w[i] << 16);
      v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ static __forceinline__ void store(__nv_bfloat16* p, const float (&v)[8]) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
    __stcs(reinterpret_cast<uint4*>(p), make_uint4(w[0], w[1], w[2], w[3]));
  }
};

struct LArgs {
  const void* logits;
  const int64_t* target;
  int64_t N;          // rows
  int64_t L;          // rows per batch item (row r -> batch r / L, position r % L)
  int64_t batch_stride, row_stride;  // in elements
  int64_t d_batch_stride, d_row_stride;  // strides of dlogits (backward)
  int V, v_lo, v_hi;
  float inv_t;
  float* logprob;
  float* entropy;     // nullable (forward)
  float* lse;         // nullable (forward); required (backward)
  const float* g_lp;  // backward, nullable
  const float* g_h;   // backward, nullable
  const float* h_in;  // backward: entropies of the forward (needed iff g_h)
  void* dlogits;      // backward, same dtype as logits
};

template <typename T>
__device__ __forceinline__ const T* row_ptr(const LArgs& a, int64_t r) {
  return static_cast<const T*>(a.logits) + (r / a.L) * a.batch_stride + (r % a.L) * a.row_stride;
}
template <typename T>
__device__ __forceinline__ T* drow_ptr(const LArgs& a, int64_t r) {
  return static_cast<T*>(a.dlogits) + (r / a.L) * a.d_batch_stride + (r % a.L) * a.d_row_stride;
}

// reduction of one row segment [lo, hi) by NT cooperating threads (thread rank t): vector loads on the aligned middle
template <typename T, int NT>
__device__ __forceinline__ Acc row_reduce(const T* x, int lo, int hi, float inv_t, int t) {
  constexpr int VPT = Vec<T>::N;
  Acc a;
  acc_init(a);
  // scalar head up to the first 16-byte aligned element
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x + lo);
  int head = (int)(((16 - (addr & 15)) & 15) / sizeof(T));
  if (head > hi - lo) head = hi - lo;
  const int mid0 = lo + head;
  const int nvec = (hi - mid0) / VPT;
  const int tail0 = mid0 + nvec * VPT;
  for (int i = lo + t; i < mid0; i += NT) acc_add4(a, load1(x + i) * inv_t, -INFINITY, -INFINITY, -INFINITY);
  for (int i = tail0 + t; i < hi; i += NT) acc_add4(a, load1(x + i) * inv_t, -INFINITY, -INFINITY, -INFINITY);
  const T* xm = x + mid0;
#pragma unroll 4
  for (int i = t; i < nvec; i += NT) {
    float v[VPT];
    Vec<T>::load(xm + (size_t)i * VPT, v);
#pragma unroll
    for (int j = 0; j < VPT; j += 4) acc_add4(a, v[j] * inv_t, v[j + 1] * inv_t, v[j + 2] * inv_t, v[j + 3] * inv_t);
  }
  return a;
}

__device__ __forceinline__ void finish_row(const LArgs& a, int64_t r, const Acc& acc, float z_t, bool t_in) {
  rb::smx::finish_row(acc, z_t, t_in, r, a.logprob, a.entropy, a.lse);
}

// ---- forward: one CTA per row ----
template <typename T>
__global__ void __launch_bounds__(kThreads) fwd_block_kernel(LArgs a) {
  __shared__ Acc part[kThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int64_t r = blockIdx.x; r < a.N; r += gridDim.x) {
    const T* x = row_ptr<T>(a, r);
    Acc acc = warp_merge(row_reduce<T, kThreads>(x, a.v_lo, a.v_hi, a.inv_t, t));
    if (lane == 0) part[warp] = acc;
    __syncthreads();
    if (warp == 0) {
      Acc b;
      if (lane < kThreads / 32) b = part[lane];
      else acc_init(b);
      b = warp_merge(b);
      if (lane == 0) {
        const int64_t tg = a.target[r];
        const bool t_in = tg >= a.v_lo && tg < a.v_hi;
        finish_row(a, r, b, t_in ? load1(x + tg) * a.inv_t : 0.f, t_in);
      }
    }
    __syncthreads();
  }
}

// ---- forward: one warp per row (short windows) ----
template <typename T>
__global__ void __launch_bounds__(kThreads) fwd_warp_kernel(LArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t w0 = (int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  for (int64_t r = w0; r < a.N; r += (int64_t)gridDim.x * (kThreads / 32)) {
    const T* x = row_ptr<T>(a, r);
    const Acc acc = warp_merge(row_reduce<T, 32>(x, a.v_lo, a.v_hi, a.inv_t, lane));
    if (lane == 0) {
      const int64_t tg = a.target[r];
      const bool t_in = tg >= a.v_lo && tg < a.v_hi;
      finish_row(a, r, acc, t_in ? load1(x + tg) * a.inv_t : 0.f, t_in);
    }
  }
}

// ---- backward: elementwise over the row given lse (and H), NT threads per row ----
template <typename T, int NT>
__device__ __forceinline__ void row_backward(const LArgs& a, int64_t r, int t) {
  constexpr int VPT = Vec<T>::N;
  const T* x = row_ptr<T>(a, r);
  T* dx = drow_ptr<T>(a, r);
  const float lse = a.lse[r];
  const float glp = a.g_lp ? a.g_lp[r] : 0.f;
  const float gh = a.g_h ? a.g_h[r] : 0.f;
  const float H = a.g_h ? a.h_in[r] : 0.f;
  const int64_t tg = a.target[r];
  const float it = a.inv_t;
  auto grad = [&](float xv, int i) -> float {
    const float z = xv * it;
    const float lp = z - lse;
    const float p = __expf(lp);
    float g = -glp * p;
    if (gh != 0.f && p > 0.f) g -= gh * p * (lp + H);
    if (i == tg) g += glp;
    return g * it;
  };
  auto store1 = [&](int i, float g) {
    if constexpr (sizeof(T) == 4) reinterpret_cast<float*>(dx)[i] = g;
    else reinterpret_cast<__nv_bfloat16*>(dx)[i] = __float2bfloat16_rn(g);
  };
  // outside the window the (masked) logits get no gradient
  for (int i = t; i < a.v_lo; i += NT) store1(i, 0.f);
  for (int i = a.v_hi + t; i < a.V; i += NT) store1(i, 0.f);
  const int lo = a.v_lo, hi = a.v_hi;
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x + lo);
  const uintptr_t daddr = reinterpret_cast<uintptr_t>(dx + lo);
  int head = (int)(((16 - (addr & 15)) & 15) / sizeof(T));
  if (head > hi - lo) head = hi - lo;
  const bool vec_ok = ((addr ^ daddr) & 15) == 0;
  const int mid0 = lo + head;
  const int nvec = vec_ok ? (hi - mid0) / VPT : 0;
  const int tail0 = mid0 + nvec * VPT;
  for (int i = lo + t; i < mid0; i += NT) store1(i, grad(load1(x + i), i));
  for (int i = tail0 + t; i < hi; i += NT) store1(i, grad(load1(x + i), i));
#pragma unroll 2
  for (int i = t; i < nvec; i += NT) {
    float v[VPT], g[VPT];
    Vec<T>::load(x + mid0 + (size_t)i * VPT, v);
#pragma unroll
    for (int j = 0; j < VPT; ++j) g[j] = grad(v[j], mid0 + i * VPT + j);
    Vec<T>::store(dx + mid0 + (size_t)i * VPT, g);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) bwd_block_kernel(LArgs a) {
  for (int64_t r = blockIdx.x; r < a.N; r += gridDim.x) row_backward<T, kThreads>(a, r, threadIdx.x);
}
template <typename T>
__global__ void __launch_bounds__(kThreads) bwd_warp_kernel(LArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t w0 = (int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  for (int64_t r = w0; r < a.N; r += (int64_t)gridDim.x * (kThreads / 32)) row_backward<T, 32>(a, r, lane);
}

int check(const LArgs& a, int dtype) {
  if (!a.logits || !a.target) return RB200_E_NULL;
  if (dtype != 0 && dtype != 1) return RB200_E_UNSUPPORTED;
  if (a.N <= 0 || a.V <= 0 || a.L <= 0 || a.v_lo < 0 || a.v_hi > a.V || a.v_lo >= a.v_hi) return RB200_E_SHAPE;
  if (!(a.inv_t > 0.f)) return RB200_E_SHAPE;
  return RB200_OK;
}

int grid_for(int64_t rows_per_block_unit, int64_t N) {
  const int64_t cap = (int64_t)rb::sm_count() * 8;
  const int64_t blocks = (N + rows_per_block_unit - 1) / rows_per_block_unit;
  return (int)(blocks < cap ? blocks : cap);
}

}  // namespace

extern "C" int rb200_logits_logprob_entropy_fwd(const void* logits, int dtype, const int64_t* target, int64_t N, int64_t L,
                                                int64_t batch_stride, int64_t row_stride, int V, int v_lo, int v_hi,
                                                double inv_temperature, float* logprob, float* entropy, float* lse,
                                                rb200_stream_t stream) {
  LArgs a{};
  a.logits = logits; a.target = target; a.N = N; a.L = L; a.batch_stride = batch_stride; a.row_stride = row_stride;
  a.V = V; a.v_lo = v_lo; a.v_hi = v_hi; a.inv_t = (float)inv_temperature; a.logprob = logprob; a.entropy = entropy;
  a.lse = lse;
  int e = check(a, dtype);
  if (e) return e;
  if (!logprob) return RB200_E_NULL;
  cudaStream_t st = rb::as_stream(stream);
  const bool wide = (v_hi - v_lo) > 2048;
  if (wide) {
    if (dtype == 0) fwd_block_kernel<float><<<grid_for(1, N), kThreads, 0, st>>>(a);
    else fwd_block_kernel<__nv_bfloat16><<<grid_for(1, N), kThreads, 0, st>>>(a);
  } else {
    if (dtype == 0) fwd_warp_kernel<float><<<grid_for(kThreads / 32, N), kThreads, 0, st>>>(a);
    else fwd_warp_kernel<__nv_bfloat16><<<grid_for(kThreads / 32, N), kThreads, 0, st>>>(a);
  }
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_logits_logprob_entropy_bwd(const void* logits, int dtype, const int64_t* target, int64_t N, int64_t L,
                                                int64_t batch_stride, int64_t row_stride, int V, int v_lo, int v_hi,
                                                double inv_temperature, const float* lse, const float* entropy,
                                                const float* grad_logprob, const float* grad_entropy, void* dlogits,
                                                int64_t d_batch_stride, int64_t d_row_stride, rb200_stream_t stream) {
  LArgs a{};
  a.logits = logits; a.target = target; a.N = N; a.L = L; a.batch_stride = batch_stride; a.row_stride = row_stride;
  a.V = V; a.v_lo = v_lo; a.v_hi = v_hi; a.inv_t = (float)inv_temperature; a.lse = const_cast<float*>(lse);
  a.h_in = entropy; a.g_lp = grad_logprob; a.g_h = grad_entropy; a.dlogits = dlogits;
  a.d_batch_stride = d_batch_stride; a.d_row_stride = d_row_stride;
  int e = check(a, dtype);
  if (e) return e;
  if (!lse || !dlogits || (grad_entropy && !entropy)) return RB200_E_NULL;
  cudaStream_t st = rb::as_stream(stream);
  const bool wide = V > 2048;
  if (wide) {
    if (dtype == 0) bwd_block_kernel<float><<<grid_for(1, N), kThreads, 0, st>>>(a);
    else bwd_block_kernel<__nv_bfloat16><<<grid_for(1, N), kThreads, 0, st>>>(a);
  } else {
    if (dtype == 0) bwd_warp_kernel<float><<<grid_for(kThreads / 32, N), kThreads, 0, st>>>(a);
    else bwd_warp_kernel<__nv_bfloat16><<<grid_for(kThreads / 32, N), kThreads, 0, st>>>(a);
  }
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
