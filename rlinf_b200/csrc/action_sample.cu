// Action-token sampling of the OpenVLA-OFT rollout: the bin window, temperature, top-k, the draw, its log-prob and the
// de-tokenised action, from the logits (rb200_logits_sample_step) or from the fused LM head's window block
// (lmhead_sample.cu, through rb::asmp::sample_tiles).
//
// Reference (OpenVLAOFTForRLActionPrediction.predict_action_batch, openvla_oft_action_model.py:350-410): -inf outside
// [vocab_size - n_action_bins, vocab_size), then with do_sample logits / T, TopKLogitsWarper(top_k), log_softmax, exp,
// torch.multinomial, else argmax; the tokens are de-tokenised to bin centres and unnormalised on the host (:390-404,
// _unnormalize_actions :167-203), and compute_logprobs_from_logits runs on the masked processed logits (:406-410).
// Because the window is applied before top-k, only the window's W = v_hi - v_lo columns matter; nothing else is read.
//
// One warp per row, lane l holding columns l + 32 q of the window (q < NJ):
//   top-k: thr = the k-th largest window value, found by a 1-bit-per-pass radix select on topk.cu's integer keys (each
//          pass counts the keys >= a candidate with an integer warp reduction); kept iff x >= thr, ties all kept;
//   sample: z = x * inv_T; m = max over kept; e = exp(z - m); an inclusive scan of e in column order (per q a fixed
//          shuffle scan, plus the carry of the columns before); the token is the first column of positive weight
//          (e > 0) whose prefix sum reaches u * total, u in (0, 1] from Philox4_32_10(seed, r, offset), and total is
//          the scan's last element.  Each lane sums over its own shuffle tree, so the prefix sums are not monotone in
//          the last bit: a kept column of weight 0 (a -inf logit, or exp(z - m) underflowing) can carry a larger prefix
//          sum than the positive column before it, and is never a candidate.  A target past every positive column's
//          prefix sum (the tree can round those below the total) takes the last column of positive weight;
//          logprob = (z_t - m) - log(total);
//   greedy: the argmax of x (lowest index on ties, NaN wins, as torch.argmax); logprob over the whole window at T = 1.
// A NaN in the window makes total NaN: the scan then finds no column and the token falls back to the last kept column,
// inside the window, with a NaN log-prob.  No floating-point or global atomics; rows are independent, so nothing
// depends on the grid or the SM count.
//
// With a step struct (one generate step of the plain OpenVLA decode loop, OpenVLAForRLActionPrediction.
// predict_action_batch, openvla_action_model.py:610-756, or the OFT call under a graph): the Philox offset is read from a
// device counter that the entry then advances by 1 on the same stream (rollout.cu's rb200_counter_add), so a captured
// graph draws fresh numbers on every replay; and row r = b * L + p writes its outputs at b * out_row_stride + col0 + p
// and de-tokenises with dimension (col0 + p) % action_dim, so step j of a [bsz, A] buffer is column col0 = j.
#include <cuda_bf16.h>
#include <curand_kernel.h>

#include "common.cuh"
#include "radix_key.cuh"

namespace {

constexpr int kWarps = 8;            // rows per CTA
constexpr int kMaxWindow = 1024;
constexpr int kMaxGrid = 1 << 16;    // CTAs; more rows are walked in a grid-stride loop

struct SArgs {
  const void* x;         // the logits, or the fused head's fp32 window block
  int64_t N, L, batch_stride, row_stride;
  int v_lo, W, do_sample, k;
  float inv_t;
  uint64_t seed, offset;
  rb200_action_bins bins;
  int has_bins;
  int64_t* token;
  float* logprob;
  double* action;
  // the fused head's block: row j is position (j % 128) of row tile rt0 + j / 128, batch item rt / tpb, position
  // (rt % tpb) * 128 + j % 128 < L (padding rows are skipped); its columns are the window's
  int tiled, tpb;
  int64_t rt0;
  // a step struct: Philox offset from *offset_dev when set; row r (in rows of out_L positions) writes at
  // (r / out_L) * out_stride + col0 + r % out_L.  Without a step struct out_L = out_stride = L and col0 = 0.
  const int64_t* offset_dev;
  int64_t out_L, out_stride;
  int col0;
};

template <typename T>
__device__ __forceinline__ float ld1(const T* p) {
  if constexpr (sizeof(T) == 4) return *p;
  else return __bfloat162float(*p);
}

// the key of a window value: topk.cu's Key<T>, taken from the exact fp32 value (a bf16 key is the fp32 key's top half)
template <typename T>
__device__ __forceinline__ uint32_t key_of(float x) {
  return Key<float>::of(x) >> (32 - Key<T>::kBits);
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// numpy's 0.5 * (n + 1) * (high - low + 1e-8) + low, one rounding per operation, no FMA contraction
__device__ __forceinline__ double unnormalize(double n, double lo, double hi) {
  return __dadd_rn(__dmul_rn(__dmul_rn(0.5, __dadd_rn(n, 1.0)), __dadd_rn(__dsub_rn(hi, lo), 1e-8)), lo);
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kWarps * 32) sample_kernel(const SArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * kWarps;
  for (int64_t j = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); j < a.N; j += stride) {
    int64_t r, p;
    const T* xw;  // column 0 of the window
    if (a.tiled) {
      const int64_t rt = a.rt0 + j / 128;
      p = (rt % a.tpb) * 128 + j % 128;
      if (p >= a.L) continue;  // a padding row of the tile: the whole warp skips it
      r = (rt / a.tpb) * a.L + p;
      xw = static_cast<const T*>(a.x) + j * a.row_stride;
    } else {
      r = j;
      p = j % a.L;
      xw = static_cast<const T*>(a.x) + (j / a.L) * a.batch_stride + p * a.row_stride + a.v_lo;
    }
    float x[NJ];
#pragma unroll
    for (int q = 0; q < NJ; ++q) {
      const int c = lane + 32 * q;
      x[q] = c < a.W ? ld1(xw + c) : -INFINITY;
    }

    // kept columns: c < W and not x < thr (a NaN is kept, so that it reaches the sum)
    float thr = -INFINITY;
    const bool filter = a.do_sample && a.k > 0 && a.k < a.W;
    if (filter) {
      constexpr int KB = Key<T>::kBits;
      uint32_t pre = 0;  // the largest key with at least k window keys >= it: the k-th largest key
#pragma unroll 1
      for (int b = KB - 1; b >= 0; --b) {
        const uint32_t cand = pre | (1u << b);
        uint32_t cnt = 0;
#pragma unroll
        for (int q = 0; q < NJ; ++q) cnt += (lane + 32 * q < a.W && key_of<T>(x[q]) >= cand) ? 1u : 0u;
        if (__reduce_add_sync(0xffffffffu, cnt) >= (uint32_t)a.k) pre = cand;
      }
      thr = Key<T>::value(pre);
    }
    const float inv_t = a.do_sample ? a.inv_t : 1.f;
    auto kept = [&](int q) { return lane + 32 * q < a.W && !(x[q] < thr); };

    float m = -INFINITY;
#pragma unroll
    for (int q = 0; q < NJ; ++q)
      if (kept(q)) m = fmaxf(m, x[q] * inv_t);
    m = warp_max(m);
    // inclusive prefix sums of exp(z - m) in column order, and which columns have a positive weight
    float cum[NJ];
    bool pos[NJ];
    float carry = 0.f;
#pragma unroll
    for (int q = 0; q < NJ; ++q) {
      float s = kept(q) ? expf(x[q] * inv_t - m) : 0.f;
      pos[q] = s > 0.f;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float u = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += u;
      }
      cum[q] = carry + s;
      carry += __shfl_sync(0xffffffffu, s, 31);
    }
    const float total = carry;

    uint32_t tok;  // window column
    if (a.do_sample) {
      curandStatePhilox4_32_10_t st;
      const uint64_t off = a.offset_dev ? (uint64_t)*a.offset_dev : a.offset;
      curand_init(a.seed, (unsigned long long)r, off, &st);
      const float target = curand_uniform(&st) * total;  // (0, total]
      // only a column of positive weight can be drawn: a zero-weight column's prefix sum, on its own shuffle tree, can
      // exceed the one of the positive column before it
      uint32_t first = 0xffffffffu, last_pos = 0, last_kept = 0;
#pragma unroll
      for (int q = 0; q < NJ; ++q) {
        const uint32_t c = lane + 32 * q;
        if (pos[q]) {
          if (first == 0xffffffffu && cum[q] >= target) first = c;
          last_pos = c + 1;
        }
        if (kept(q)) last_kept = c + 1;
      }
      first = __reduce_min_sync(0xffffffffu, first);
      last_pos = __reduce_max_sync(0xffffffffu, last_pos);
      last_kept = __reduce_max_sync(0xffffffffu, last_kept);
      // total is >= 1 (the maximum's weight) or NaN, which no prefix sum reaches
      tok = first != 0xffffffffu ? first : (total == total ? last_pos : last_kept) - 1;
    } else {
      // argmax, lowest index on ties, NaN above everything (torch.argmax); within a lane q ascends with the column
      float bv = x[0];
      uint32_t bi = lane;
#pragma unroll
      for (int q = 1; q < NJ; ++q) {
        if (lane + 32 * q < a.W && (x[q] > bv || (x[q] != x[q] && bv == bv))) {
          bv = x[q];
          bi = lane + 32 * q;
        }
      }
      if (bi >= (uint32_t)a.W) bv = -INFINITY;  // lane >= W (W < 32) holds no column
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
        const bool onan = ov != ov, bnan = bv != bv;
        const bool better = (onan && !bnan) || ov > bv || ((ov == bv || (onan && bnan)) && oi < bi);
        if (better) {
          bv = ov;
          bi = oi;
        }
      }
      tok = bi;
    }
    float zt = 0.f;
#pragma unroll
    for (int q = 0; q < NJ; ++q)
      if (lane + 32 * q == tok) zt = x[q] * inv_t;
    zt = __shfl_sync(0xffffffffu, zt, tok & 31);
    if (lane == 0) {
      const int64_t id = (int64_t)a.v_lo + tok;
      const int64_t op = a.col0 + r % a.out_L;  // output column (= p without a step struct)
      const int64_t o = (r / a.out_L) * a.out_stride + op;
      a.token[o] = id;
      a.logprob[o] = (zt - m) - logf(total);
      if (a.has_bins) {
        const rb200_action_bins& B = a.bins;
        int64_t d = B.vocab_size - id - 1;
        d = d < 0 ? 0 : (d > B.n_bins - 1 ? B.n_bins - 1 : d);
        const double n = B.bin_centers[d];
        const int ad = (int)(op % B.action_dim);
        a.action[o] = B.mask[ad] ? unnormalize(n, B.low[ad], B.high[ad]) : n;
      }
    }
  }
}

template <typename T>
int launch(const SArgs& a, cudaStream_t st) {
  const int64_t blocks = (a.N + kWarps - 1) / kWarps;
  const int grid = (int)(blocks < kMaxGrid ? blocks : kMaxGrid);
  if (a.W <= 256) sample_kernel<T, 8><<<grid, kWarps * 32, 0, st>>>(a);
  else sample_kernel<T, 32><<<grid, kWarps * 32, 0, st>>>(a);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

void apply_step(SArgs& a, const rb200_sample_step* s, int64_t L) {
  a.out_L = L;
  if (s) {
    a.offset_dev = s->offset_dev;
    a.out_stride = s->out_row_stride;
    a.col0 = s->col0;
  } else {
    a.out_stride = L;
  }
}

// the counter advance after the sampler's launch: every row has read the offset before it runs
int advance(const rb200_sample_step* s, cudaStream_t st) {
  if (!s || !s->offset_dev) return RB200_OK;
  return rb200_counter_add(reinterpret_cast<uint64_t*>(const_cast<int64_t*>(s->offset_dev)), 1, st);
}

SArgs make_args(int v_lo, int v_hi, int do_sample, double inv_temperature, int top_k, uint64_t seed, uint64_t offset,
                const rb200_action_bins* bins, int64_t* token, float* logprob, double* action) {
  SArgs a{};
  a.v_lo = v_lo; a.W = v_hi - v_lo; a.do_sample = do_sample != 0; a.k = top_k; a.inv_t = (float)inv_temperature;
  a.seed = seed; a.offset = offset; a.token = token; a.logprob = logprob; a.action = action;
  if (bins) {
    a.bins = *bins;
    a.has_bins = 1;
  }
  return a;
}

}  // namespace

namespace rb {
namespace asmp {
// everything but the row addressing; the caller checks the window against its V
int check_common(int W, int do_sample, double inv_temperature, const rb200_action_bins* bins, const int64_t* token,
                 const float* logprob, const double* action) {
  if (!token || !logprob) return RB200_E_NULL;
  if (W < 1 || W > kMaxWindow) return RB200_E_SHAPE;
  if (do_sample && !(inv_temperature > 0.0 && (float)inv_temperature < INFINITY)) return RB200_E_ARG;
  if (bins) {
    if (!action || !bins->bin_centers || !bins->low || !bins->high || !bins->mask) return RB200_E_NULL;
    if (bins->n_bins < 1 || bins->action_dim < 1) return RB200_E_SHAPE;
  }
  return RB200_OK;
}

// the step struct against the call's L: a layout that every row's outputs fit in, columns not overlapping the next row's;
// NULL is the dense layout
int check_step(const rb200_sample_step* s, int64_t L) {
  if (!s) return RB200_OK;
  if (s->col0 < 0 || s->out_row_stride < (int64_t)s->col0 + L) return RB200_E_SHAPE;
  return RB200_OK;
}

// the sampler over a block of nt row tiles of the window's raw fp32 logits [nt * 128, ld] (lmhead_sample.cu's ACC
// pass), writing row r's outputs at r; with a step struct (nullable) at its layout in rows of out_L positions, out_L
// being the caller's L (the tiles may group the rows differently), then the counter advance
int sample_tiles(const float* block, int64_t ld, int v_lo, int v_hi, int do_sample, double inv_temperature, int top_k,
                 uint64_t seed, uint64_t offset, const rb200_action_bins* bins, int64_t rt0, int64_t nt, int tpb,
                 int64_t L_rows, int64_t* token, float* logprob, double* action, const rb200_sample_step* step,
                 int64_t out_L, cudaStream_t st) {
  SArgs a = make_args(v_lo, v_hi, do_sample, inv_temperature, top_k, seed, offset, bins, token, logprob, action);
  a.x = block; a.N = nt * 128; a.L = L_rows; a.row_stride = ld; a.tiled = 1; a.tpb = tpb; a.rt0 = rt0;
  apply_step(a, step, step ? out_L : L_rows);
  int e = launch<float>(a, st);
  return e ? e : advance(step, st);
}
}  // namespace asmp
}  // namespace rb

extern "C" int rb200_logits_sample_step(const void* logits, int dtype, int64_t N, int64_t L, int64_t batch_stride,
                                        int64_t row_stride, int V, int v_lo, int v_hi, int do_sample,
                                        double inv_temperature, int top_k, uint64_t seed, uint64_t offset,
                                        const rb200_action_bins* bins, int64_t* token, float* logprob, double* action,
                                        const rb200_sample_step* step, rb200_stream_t stream) {
  if (!logits) return RB200_E_NULL;
  if (dtype != 0 && dtype != 1) return RB200_E_UNSUPPORTED;
  if (N <= 0 || L <= 0 || N % L != 0 || V <= 0 || v_lo < 0 || v_hi > V || v_lo >= v_hi) return RB200_E_SHAPE;
  int e = rb::asmp::check_common(v_hi - v_lo, do_sample, inv_temperature, bins, token, logprob, action);
  if (e || (e = rb::asmp::check_step(step, L))) return e;
  SArgs a = make_args(v_lo, v_hi, do_sample, inv_temperature, top_k, seed, offset, bins, token, logprob, action);
  a.x = logits; a.N = N; a.L = L; a.batch_stride = batch_stride; a.row_stride = row_stride;
  apply_step(a, step, L);
  cudaStream_t st = rb::as_stream(stream);
  e = dtype == 0 ? launch<float>(a, st) : launch<__nv_bfloat16>(a, st);
  return e ? e : advance(step, st);
}
