// Top-k filtered token log-probabilities and entropies from the logits, forward and backward (the OpenVLA action head
// with `rollout.sampling_params.top_k > 0`).
//
// Reference order (models/embodiment/openvla_oft/rlinf/openvla_oft_action_model.py:532-559, the same in
// models/embodiment/openvla/openvla_action_model.py:564-591): logits / T, TopKLogitsWarper(top_k) over the whole padded
// vocabulary, the action-bin window, then compute_logprobs_from_logits / compute_entropy_from_logits.  Per row x [0, V):
//   thr = the k-th largest x (with multiplicity); column i is kept iff v_lo <= i < v_hi and x_i >= thr (ties at the k-th
//   value are all kept); lse / logprob / entropy are the logits kernels' formulas over the kept columns only; a target
//   that is not kept has logprob -inf; a row with no kept column has logprob NaN, entropy -0.0 and lse -inf, as the
//   reference gives; the gradient is 0 at every column that is not kept and dz_of (softmax_acc.cuh) at the others.
// The selection runs on the unscaled x (exact; the reference selects on x / T rounded to the logits' dtype, which can
// only add a tie at the k-th value).
//
// Forward: one CTA per row.  The row is staged in shared memory when it fits (HBM is read once), then a radix select
// on order-preserving integer keys (16-bit for bf16, 32-bit for fp32), 11 bits per pass, finds thr: the first digit's
// histogram is counted while the row is staged, later passes count only the keys that share the digits chosen so far,
// and a block scan from the top picks the digit that holds the k-th key.  The histograms are integer counts in shared
// memory, so their values do not depend on the order of the adds.  The masked softmax pass then reads only
// [v_lo, v_hi).
// Backward: one CTA per row, elementwise from the saved thr and lse, one read of the row and one write of dlogits.
// No floating-point or global atomics; rows are independent, so nothing depends on the grid size or the SM count.
#include <cuda_bf16.h>

#include "common.cuh"
#include "radix_key.cuh"
#include "softmax_acc.cuh"

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxSmem = 232448;       // sm_90 opt-in shared memory per block

using rb::smx::Acc;
using rb::smx::acc_add4;
using rb::smx::acc_init;
using rb::smx::warp_merge;

template <typename T>
__device__ __forceinline__ float ld1(const T* p) {
  if constexpr (sizeof(T) == 4) return *reinterpret_cast<const float*>(p);
  else return __bfloat162float(*p);
}

// 16 bytes = VPT values, from a generic pointer (shared memory or global) or streaming from global
template <typename T>
struct V16 {
  static constexpr int N = 16 / sizeof(T);
  __device__ static __forceinline__ void unpack(const uint4& x, float (&v)[N]) {
    if constexpr (sizeof(T) == 4) {
      v[0] = __uint_as_float(x.x); v[1] = __uint_as_float(x.y); v[2] = __uint_as_float(x.z); v[3] = __uint_as_float(x.w);
    } else {
      const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        v[2 * i] = __uint_as_float(w[i] << 16);
        v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
      }
    }
  }
  __device__ static __forceinline__ void load(const T* p, float (&v)[N]) {
    unpack(*reinterpret_cast<const uint4*>(p), v);
  }
  __device__ static __forceinline__ void store_cs(T* p, const float (&v)[N]) {
    uint4 o;
    if constexpr (sizeof(T) == 4) {
      o = make_uint4(__float_as_uint(v[0]), __float_as_uint(v[1]), __float_as_uint(v[2]), __float_as_uint(v[3]));
    } else {
      uint32_t w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
        w[i] = *reinterpret_cast<const uint32_t*>(&h);
      }
      o = make_uint4(w[0], w[1], w[2], w[3]);
    }
    __stcs(reinterpret_cast<uint4*>(p), o);
  }
};

struct TArgs {
  const void* logits;
  const int64_t* target;
  int64_t N, L;
  int64_t batch_stride, row_stride;
  int64_t d_batch_stride, d_row_stride;
  int V, v_lo, v_hi, k;
  float inv_t;
  int stage;          // forward: stage the row in shared memory
  float* logprob;
  float* entropy;     // nullable
  float* lse;         // nullable (forward); required (backward)
  float* thr;         // forward output / backward input
  const float* g_lp;  // backward, nullable
  const float* g_h;   // backward, nullable
  const float* h_in;  // backward: the forward's entropies (needed iff g_h)
  void* dlogits;
  // forward on the fused LM head's accumulator block (lmhead_topk.cu): row j of the block is position
  // (j % 128) of row tile rt0 + j / 128, batch item (rt / tpb), position ((rt % tpb) * 128 + j % 128) < L_rows
  int tiled, tpb;
  int64_t rt0, L_rows;
};

template <typename T>
__device__ __forceinline__ const T* row_ptr(const TArgs& a, int64_t r) {
  return static_cast<const T*>(a.logits) + (r / a.L) * a.batch_stride + (r % a.L) * a.row_stride;
}

// [lo, hi) of a row split into a scalar head up to the first 16-byte boundary, whole 16-byte vectors and a scalar tail
struct Split {
  int mid0, nvec, tail0;
};
template <typename T>
__device__ __forceinline__ Split split(const T* x, int lo, int hi) {
  const uintptr_t addr = reinterpret_cast<uintptr_t>(x + lo);
  int head = (int)(((16 - (addr & 15)) & 15) / sizeof(T));
  if (head > hi - lo) head = hi - lo;
  Split s;
  s.mid0 = lo + head;
  s.nvec = (hi - s.mid0) / V16<T>::N;
  s.tail0 = s.mid0 + s.nvec * V16<T>::N;
  return s;
}

constexpr int kDigit = 11;                       // radix digit width: 2048 bins
constexpr int kBins = 1 << kDigit;

struct __align__(16) Shared {
  uint32_t hist[kBins];
  uint32_t wsum[kWarps];
  uint32_t sel_digit, sel_below;  // the chosen digit and the count of keys in the bins above it
  Acc part[kWarps];
};

// count one key into the histogram of the digit (key >> shift) & (2^bits - 1) if its higher bits equal prefix.
// Integer shared-memory counts: the histogram is the same whatever order the adds land in.
__device__ __forceinline__ void count_key(uint32_t key, int shift, int bits, uint32_t prefix, bool first,
                                          uint32_t* hist) {
  if (first || (key >> (shift + bits)) == prefix) atomicAdd(&hist[(key >> shift) & ((1u << bits) - 1u)], 1u);
}
template <typename T>
__device__ __forceinline__ void count_vec(const uint4& v, int shift, int bits, uint32_t prefix, bool first,
                                          uint32_t* hist) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if constexpr (sizeof(T) == 4) {
      count_key(Key<float>::of(__uint_as_float(w[i])), shift, bits, prefix, first, hist);
    } else {
      count_key(Key<T>::of16(w[i] & 0xffffu), shift, bits, prefix, first, hist);
      count_key(Key<T>::of16(w[i] >> 16), shift, bits, prefix, first, hist);
    }
  }
}

// histogram of the digit over src[0, V) (generic pointer: the staged row or the row in global memory)
template <typename T>
__device__ __forceinline__ void hist_sweep(const T* src, int V, int shift, int bits, uint32_t prefix, bool first,
                                           uint32_t* hist) {
  const int t = threadIdx.x;
  const Split sp = split(src, 0, V);
  for (int i = t; i < sp.mid0; i += kThreads) count_key(Key<T>::raw(src + i), shift, bits, prefix, first, hist);
  for (int i = sp.tail0 + t; i < V; i += kThreads) count_key(Key<T>::raw(src + i), shift, bits, prefix, first, hist);
  const T* xm = src + sp.mid0;
#pragma unroll 4
  for (int i = t; i < sp.nvec; i += kThreads)
    count_vec<T>(*reinterpret_cast<const uint4*>(xm + (size_t)i * V16<T>::N), shift, bits, prefix, first, hist);
}

// From the histogram of a digit of `bits` bits: the digit that holds the kk-th largest key, and the count of keys in the
// bins above it.  Thread t owns bins [t per, t per + per); a suffix scan over the threads gives each thread the count
// of keys in its bins and above, and the one thread whose bins hold the kk-th key walks them from the top.
__device__ __forceinline__ void pick_digit(Shared& sh, int bits, uint32_t kk) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int nb = 1 << bits;
  const int per = (nb + kThreads - 1) / kThreads;
  const int b0 = min(t * per, nb), b1 = min(b0 + per, nb);
  uint32_t c = 0;
  for (int b = b0; b < b1; ++b) c += sh.hist[b];
  uint32_t s = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_down_sync(0xffffffffu, s, o);
    if (lane + o < 32) s += u;
  }
  if (lane == 0) sh.wsum[warp] = s;
  __syncthreads();
  uint32_t above = 0;
  for (int w = warp + 1; w < kWarps; ++w) above += sh.wsum[w];
  const uint32_t S = s + above;  // keys in bins >= b0
  if (c > 0 && S >= kk && S - c < kk) {
    uint32_t cum = S - c;
    for (int b = b1 - 1; b >= b0; --b) {
      const uint32_t h = sh.hist[b];
      if (cum + h >= kk) {
        sh.sel_digit = (uint32_t)b;
        sh.sel_below = cum;
        break;
      }
      cum += h;
    }
  }
}

// k-th largest key of the row by radix select, kDigit bits per pass (bf16: 11 + 5, fp32: 11 + 11 + 10).  The first
// pass's histogram is counted by the caller (staged) or here (first_done = false).  Every thread returns the key.
template <typename T>
__device__ uint32_t radix_select(const T* src, int V, int k, Shared& sh, bool first_done) {
  constexpr int KB = Key<T>::kBits;
  uint32_t prefix = 0;  // the key bits above the current digit
  uint32_t kk = (uint32_t)k;
  int done = 0;
#pragma unroll 1
  while (done < KB) {
    const int bits = min(kDigit, KB - done);
    const int shift = KB - done - bits;
    if (!(done == 0 && first_done)) {
      for (int b = threadIdx.x; b < kBins; b += kThreads) sh.hist[b] = 0;
      __syncthreads();
      hist_sweep<T>(src, V, shift, bits, prefix, done == 0, sh.hist);
    }
    __syncthreads();
    pick_digit(sh, bits, kk);
    __syncthreads();
    kk -= sh.sel_below;
    prefix = (prefix << bits) | sh.sel_digit;
    done += bits;
    __syncthreads();
  }
  return prefix;
}

// masked softmax statistics of src[lo, hi): z = x * inv_t where x >= thr, -inf elsewhere
template <typename T>
__device__ __forceinline__ Acc masked_reduce(const T* src, int lo, int hi, float thr, float inv_t, int t) {
  constexpr int VPT = V16<T>::N;
  Acc a;
  acc_init(a);
  const Split sp = split(src, lo, hi);
  auto zf = [&](float x) { return x >= thr ? x * inv_t : -INFINITY; };
  for (int i = lo + t; i < sp.mid0; i += kThreads) acc_add4(a, zf(ld1(src + i)), -INFINITY, -INFINITY, -INFINITY);
  for (int i = sp.tail0 + t; i < hi; i += kThreads) acc_add4(a, zf(ld1(src + i)), -INFINITY, -INFINITY, -INFINITY);
  const T* xm = src + sp.mid0;
#pragma unroll 4
  for (int i = t; i < sp.nvec; i += kThreads) {
    float v[VPT];
    V16<T>::load(xm + (size_t)i * VPT, v);
#pragma unroll
    for (int j = 0; j < VPT; j += 4) acc_add4(a, zf(v[j]), zf(v[j + 1]), zf(v[j + 2]), zf(v[j + 3]));
  }
  return a;
}

// ---- forward: one CTA per row ----
template <typename T>
__global__ void __launch_bounds__(kThreads, 3) topk_fwd_kernel(TArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  Shared& sh = *reinterpret_cast<Shared*>(smem_raw);
  uint8_t* stage_base = smem_raw + sizeof(Shared);
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int64_t j = blockIdx.x; j < a.N; j += gridDim.x) {
    int64_t r = j;
    const T* x;
    if (a.tiled) {
      const int64_t rt = a.rt0 + j / 128, p = (rt % a.tpb) * 128 + j % 128;
      if (p >= a.L_rows) continue;  // the whole CTA skips a padding row of the tile
      r = (rt / a.tpb) * a.L_rows + p;
      x = static_cast<const T*>(a.logits) + j * a.row_stride;
    } else {
      x = row_ptr<T>(a, r);
    }
    const T* src = x;
    if (a.stage) {
      // staged with the row's 16-byte phase, so the vector split of any range is the same in shared memory; the
      // first digit's histogram is counted on the way
      constexpr int KB = Key<T>::kBits;
      for (int b = t; b < kBins; b += kThreads) sh.hist[b] = 0;
      __syncthreads();
      T* s = reinterpret_cast<T*>(stage_base + (reinterpret_cast<uintptr_t>(x) & 15));
      const Split sp = split(x, 0, a.V);
      for (int i = t; i < sp.mid0; i += kThreads) {
        s[i] = x[i];
        count_key(Key<T>::raw(x + i), KB - kDigit, kDigit, 0, true, sh.hist);
      }
      for (int i = sp.tail0 + t; i < a.V; i += kThreads) {
        s[i] = x[i];
        count_key(Key<T>::raw(x + i), KB - kDigit, kDigit, 0, true, sh.hist);
      }
#pragma unroll 4
      for (int i = t; i < sp.nvec; i += kThreads) {
        const size_t o = sp.mid0 + (size_t)i * V16<T>::N;
        const uint4 v = __ldcs(reinterpret_cast<const uint4*>(x + o));
        *reinterpret_cast<uint4*>(s + o) = v;
        count_vec<T>(v, KB - kDigit, kDigit, 0, true, sh.hist);
      }
      src = s;
    }
    const float thr = Key<T>::value(radix_select<T>(src, a.V, a.k, sh, a.stage != 0));
    Acc acc = warp_merge(masked_reduce<T>(src, a.v_lo, a.v_hi, thr, a.inv_t, t));
    if (lane == 0) sh.part[warp] = acc;
    __syncthreads();
    if (warp == 0) {
      Acc b;
      if (lane < kWarps) b = sh.part[lane];
      else acc_init(b);
      b = warp_merge(b);
      if (lane == 0) {
        a.thr[r] = thr;
        if (b.m == -INFINITY) {  // no kept column: the reference's NaN log-prob and -0.0 entropy
          a.logprob[r] = __int_as_float(0x7fc00000);
          if (a.entropy) a.entropy[r] = -0.f;
          if (a.lse) a.lse[r] = -INFINITY;
        } else {
          const int64_t tg = a.target[r];
          const float xt = (tg >= a.v_lo && tg < a.v_hi) ? ld1(src + tg) : -INFINITY;
          const bool t_in = xt >= thr;
          rb::smx::finish_row(b, t_in ? xt * a.inv_t : 0.f, t_in, r, a.logprob, a.entropy, a.lse);
        }
      }
    }
    __syncthreads();
  }
}

// ---- backward: one CTA per row, elementwise given thr, lse (and H) ----
template <typename T>
__global__ void __launch_bounds__(kThreads) topk_bwd_kernel(TArgs a) {
  constexpr int VPT = V16<T>::N;
  const int t = threadIdx.x;
  for (int64_t r = blockIdx.x; r < a.N; r += gridDim.x) {
    const T* x = row_ptr<T>(a, r);
    T* dx = static_cast<T*>(a.dlogits) + (r / a.L) * a.d_batch_stride + (r % a.L) * a.d_row_stride;
    const float thr = a.thr[r];
    const float lse = a.lse[r];
    const float glp = a.g_lp ? a.g_lp[r] : 0.f;
    const float gh = a.g_h ? a.g_h[r] : 0.f;
    const float H = a.g_h ? a.h_in[r] : 0.f;
    const int64_t tg = a.target[r];
    const int lo = a.v_lo, hi = a.v_hi;
    // a column that is not kept (outside the window or below thr) gets no gradient; a row with no kept column none
    auto grad = [&](float xv, int i) -> float {
      return xv >= thr ? rb::smx::dz_of(xv, a.inv_t, lse, glp, gh, H, i == tg) : 0.f;
    };
    auto store1 = [&](int i, float g) {
      if constexpr (sizeof(T) == 4) reinterpret_cast<float*>(dx)[i] = g;
      else reinterpret_cast<__nv_bfloat16*>(dx)[i] = __float2bfloat16_rn(g);
    };
    for (int i = t; i < lo; i += kThreads) store1(i, 0.f);
    for (int i = hi + t; i < a.V; i += kThreads) store1(i, 0.f);
    const Split sp = split(x, lo, hi);
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(x + lo) ^ reinterpret_cast<uintptr_t>(dx + lo)) & 15) == 0;
    const int nvec = vec_ok ? sp.nvec : 0;
    const int tail0 = sp.mid0 + nvec * VPT;
    for (int i = lo + t; i < sp.mid0; i += kThreads) store1(i, grad(ld1(x + i), i));
    for (int i = tail0 + t; i < hi; i += kThreads) store1(i, grad(ld1(x + i), i));
#pragma unroll 2
    for (int i = t; i < nvec; i += kThreads) {
      float v[VPT], g[VPT];
      V16<T>::unpack(__ldcs(reinterpret_cast<const uint4*>(x + sp.mid0 + (size_t)i * VPT)), v);
#pragma unroll
      for (int j = 0; j < VPT; ++j) g[j] = grad(v[j], sp.mid0 + i * VPT + j);
      V16<T>::store_cs(dx + sp.mid0 + (size_t)i * VPT, g);
    }
  }
}

int check(const TArgs& a, int dtype) {
  if (!a.logits || !a.target || !a.thr) return RB200_E_NULL;
  if (dtype != 0 && dtype != 1) return RB200_E_UNSUPPORTED;
  if (a.N <= 0 || a.V <= 0 || a.L <= 0 || a.v_lo < 0 || a.v_hi > a.V || a.v_lo >= a.v_hi) return RB200_E_SHAPE;
  if (!(a.inv_t > 0.f)) return RB200_E_SHAPE;
  return RB200_OK;
}

int grid_rows(int64_t N) {
  const int64_t cap = (int64_t)rb::sm_count() * 8;
  return (int)(N < cap ? N : cap);
}

template <typename T>
int launch_fwd(TArgs a, cudaStream_t st) {
  const int64_t stage_bytes = (int64_t)a.V * (int64_t)sizeof(T) + 16;
  a.stage = (int64_t)sizeof(Shared) + stage_bytes <= kMaxSmem;
  const int smem = (int)sizeof(Shared) + (a.stage ? (int)stage_bytes : 0);
  static bool attr_done = false;
  if (!attr_done) {
    RB_CHECK_CUDA(cudaFuncSetAttribute(topk_fwd_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
    attr_done = true;
  }
  topk_fwd_kernel<T><<<grid_rows(a.N), kThreads, smem, st>>>(a);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

}  // namespace

namespace rb {
namespace topk {
// the forward over a block of nt row tiles of raw fp32 logits [nt * 128, ld] (lmhead_topk.cu's ACC pass), writing
// row r's outputs at r
int fwd_tiles(const float* block, int64_t ld, int V, int v_lo, int v_hi, double inv_temperature, int top_k,
              const int64_t* target, int64_t rt0, int64_t nt, int tpb, int64_t L_rows, float* logprob, float* entropy,
              float* lse, float* threshold, cudaStream_t st) {
  TArgs a{};
  a.logits = block; a.target = target; a.N = nt * 128; a.L = 1; a.row_stride = ld; a.V = V; a.v_lo = v_lo;
  a.v_hi = v_hi; a.k = top_k; a.inv_t = (float)inv_temperature; a.logprob = logprob; a.entropy = entropy; a.lse = lse;
  a.thr = threshold; a.tiled = 1; a.tpb = tpb; a.rt0 = rt0; a.L_rows = L_rows;
  return launch_fwd<float>(a, st);
}
}  // namespace topk
}  // namespace rb

extern "C" int rb200_logits_topk_logprob_entropy_fwd(const void* logits, int dtype, const int64_t* target, int64_t N,
                                                     int64_t L, int64_t batch_stride, int64_t row_stride, int V,
                                                     int v_lo, int v_hi, double inv_temperature, int top_k,
                                                     float* logprob, float* entropy, float* lse, float* threshold,
                                                     rb200_stream_t stream) {
  TArgs a{};
  a.logits = logits; a.target = target; a.N = N; a.L = L; a.batch_stride = batch_stride; a.row_stride = row_stride;
  a.V = V; a.v_lo = v_lo; a.v_hi = v_hi; a.k = top_k; a.inv_t = (float)inv_temperature;
  a.logprob = logprob; a.entropy = entropy; a.lse = lse; a.thr = threshold;
  int e = check(a, dtype);
  if (e) return e;
  if (!logprob) return RB200_E_NULL;
  if (top_k < 1 || top_k >= V) return RB200_E_ARG;
  cudaStream_t st = rb::as_stream(stream);
  return dtype == 0 ? launch_fwd<float>(a, st) : launch_fwd<__nv_bfloat16>(a, st);
}

extern "C" int rb200_logits_topk_logprob_entropy_bwd(const void* logits, int dtype, const int64_t* target, int64_t N,
                                                     int64_t L, int64_t batch_stride, int64_t row_stride, int V,
                                                     int v_lo, int v_hi, double inv_temperature,
                                                     const float* threshold, const float* lse, const float* entropy,
                                                     const float* grad_logprob, const float* grad_entropy,
                                                     void* dlogits, int64_t d_batch_stride, int64_t d_row_stride,
                                                     rb200_stream_t stream) {
  TArgs a{};
  a.logits = logits; a.target = target; a.N = N; a.L = L; a.batch_stride = batch_stride; a.row_stride = row_stride;
  a.V = V; a.v_lo = v_lo; a.v_hi = v_hi; a.inv_t = (float)inv_temperature; a.thr = const_cast<float*>(threshold);
  a.lse = const_cast<float*>(lse); a.h_in = entropy; a.g_lp = grad_logprob; a.g_h = grad_entropy; a.dlogits = dlogits;
  a.d_batch_stride = d_batch_stride; a.d_row_stride = d_row_stride;
  int e = check(a, dtype);
  if (e) return e;
  if (!lse || !dlogits || (grad_entropy && !entropy)) return RB200_E_NULL;
  cudaStream_t st = rb::as_stream(stream);
  if (dtype == 0) topk_bwd_kernel<float><<<grid_rows(N), kThreads, 0, st>>>(a);
  else topk_bwd_kernel<__nv_bfloat16><<<grid_rows(N), kThreads, 0, st>>>(a);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
