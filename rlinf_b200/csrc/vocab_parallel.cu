// Vocabulary-parallel (tensor-parallel) log-probabilities and entropies: the small kernels around the per-rank row
// passes of lmhead.cu and logits.cu.
// Rank k of P owns the vocabulary shard [k * Vs, (k + 1) * Vs) (equal shards: the vocabulary is padded so that P
// divides it).  Each rank reduces its shard to one 16-byte record per row, {m, s, t, z_t}: the running softmax
// statistics of softmax_acc.cuh over the shard's part of the window, and the scaled logit of the target column when
// the rank owns it (else 0).  The caller gathers the records of all ranks into [P, N, 4]; vp_combine_kernel merges
// them in rank order and finishes each row exactly as the single-GPU kernels do, so every rank gets the same bits.
#include "common.cuh"
#include "softmax_acc.cuh"

namespace {

using rb::smx::Acc;

__global__ void __launch_bounds__(256) shift_target_kernel(const int64_t* __restrict__ target, int64_t N,
                                                           int64_t vocab_start, int64_t* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < N) out[r] = target[r] - vocab_start;
}

// the per-range partials [n_ranges, N, 3] of the fused forward merged in range order (combine_kernel's order), plus
// the target's z: one record per row.  n_ranges = 0 gives the empty record {-inf, 0, 0, 0}.
__global__ void __launch_bounds__(256) range_record_kernel(const float* __restrict__ part, const float* __restrict__ zt,
                                                           const int64_t* __restrict__ local_target, int64_t N,
                                                           int n_ranges, int lo, int hi, float4* __restrict__ rec) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= N) return;
  Acc a;
  rb::smx::acc_init(a);
  for (int k = 0; k < n_ranges; ++k) {
    const float* p = part + ((size_t)k * N + r) * 3;
    Acc b;
    b.m = p[0];
    b.s = p[1];
    b.t = p[2];
    rb::smx::acc_merge(a, b);
  }
  const int64_t tl = n_ranges > 0 ? local_target[r] : -1;
  rec[r] = make_float4(a.m, a.s, a.t, (tl >= lo && tl < hi) ? zt[r] : 0.f);
}

__global__ void __launch_bounds__(256) vp_combine_kernel(const float4* __restrict__ rec, int n_ranks, int64_t N,
                                                         const int64_t* __restrict__ target, int vocab_shard, int v_lo,
                                                         int v_hi, float* logprob, float* entropy, float* lse) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= N) return;
  Acc a;
  rb::smx::acc_init(a);
  for (int k = 0; k < n_ranks; ++k) {
    const float4 v = rec[(size_t)k * N + r];
    Acc b;
    b.m = v.x;
    b.s = v.y;
    b.t = v.z;
    rb::smx::acc_merge(a, b);
  }
  const int64_t tg = target[r];
  const bool t_in = tg >= v_lo && tg < v_hi;
  rb::smx::finish_row(a, t_in ? rec[(size_t)(tg / vocab_shard) * N + r].w : 0.f, t_in, r, logprob, entropy, lse);
}

unsigned blocks(int64_t N) { return (unsigned)((N + 255) / 256); }

}  // namespace

namespace rb {
namespace vp {

int shift_target(const int64_t* target, int64_t N, int64_t vocab_start, int64_t* out, cudaStream_t st) {
  shift_target_kernel<<<blocks(N), 256, 0, st>>>(target, N, vocab_start, out);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

int range_record(const float* part, const float* zt, const int64_t* local_target, int64_t N, int n_ranges, int lo,
                 int hi, float* rec, cudaStream_t st) {
  range_record_kernel<<<blocks(N), 256, 0, st>>>(part, zt, local_target, N, n_ranges, lo, hi,
                                                 reinterpret_cast<float4*>(rec));
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

}  // namespace vp
}  // namespace rb

extern "C" int rb200_vp_combine(const float* records, int n_ranks, int64_t N, const int64_t* target, int vocab_shard,
                                int v_lo, int v_hi, float* logprob, float* entropy, float* lse, rb200_stream_t stream) {
  if (!records || !target || !logprob) return RB200_E_NULL;
  if ((reinterpret_cast<uintptr_t>(records) & 15) != 0) return RB200_E_ALIGN;
  if (n_ranks <= 0 || N <= 0 || vocab_shard <= 0 || v_lo < 0 || v_lo >= v_hi ||
      (int64_t)v_hi > (int64_t)n_ranks * vocab_shard)
    return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  vp_combine_kernel<<<blocks(N), 256, 0, st>>>(reinterpret_cast<const float4*>(records), n_ranks, N, target,
                                               vocab_shard, v_lo, v_hi, logprob, entropy, lse);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
