// Response-rows plan under Megatron sequence and context parallelism: which rows of one rank's hidden-state shard the
// reasoning loss reads, and how the rank's response rows, their log-probs and their dX travel between the ranks.
//
// Ownership is preprocess_packed_seqs': sequence b occupies N_b = cu[b + 1] - cu[b] padded positions.  With cp = 1 it
// sits at CP-local rows cu[b] + p.  With cp > 1, half = N_b / (2 cp) and start = cu[b] / cp, CP rank c holds positions
// [half c, half (c + 1)) at local rows start + ..., and [N_b - half (c + 1), N_b - half c) at start + half + ...  Under
// sequence parallelism TP rank k holds local rows [k Ts, (k + 1) Ts), Ts = T_c / tp.  Response token j of sequence b is
// predicted at position n_b - r_b - 1 + j; its target is responses[b, j].
//
// A CP rank's compact rows are its prediction rows in ascending local row (so the rows of TP shard k are one range
// [off_k, off_k + cnt_k) of them).  Every CTA computes the counts of all (cp, tp) ranks (pass 1, one block scan per CP
// rank), then rebuilds each CP rank's per-sequence offsets (pass 2) and writes its share of the maps; each output
// entry is written by one thread.  Sentinel -1 = a pad row or the zero row the caller appends.
#include <cuda_bf16.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int64_t kMaxBsz = 8192;
constexpr int kMaxRanks = 64;  // tp * cp

// status[0] bits (mirror of RB200_RR_*)
enum Err { E_RESP = 1, E_PROMPT = 2, E_BOUNDS = 4, E_ORDER = 8, E_CAPACITY = 32, E_SHARD = 64, E_ALIGN = 128 };

struct Args {
  const int64_t *cu, *n, *resp, *responses;
  int64_t bsz, L, Tc, Ts, cap_c, cap_k;
  int tp, cp, sp, k, c;
  int64_t *rows, *send, *unpad, *slot_map, *targets, *cell_map, *cells, *hidden_map, *status;
};

// the prediction rows of sequence b on CP rank c: two runs of positions [pA, pA + cA) at local rows tA.., and
// [pB, pB + cB) at tB..  (run B is empty with cp = 1)
struct Runs {
  int64_t pA, cA, tA, pB, cB, tB, p0, start, half;
};

__device__ __forceinline__ Runs runs_of(const Args& A, int64_t b, int c) {
  Runs s{};
  const int64_t N = A.cu[b + 1] - A.cu[b], rb = A.resp[b];
  s.p0 = A.n[b] - rb - 1;
  const int64_t p1 = s.p0 + (rb > 0 ? rb : 0);
  int64_t a0, a1, b0 = 0, b1 = 0;
  if (A.cp == 1) {
    s.start = A.cu[b];
    s.half = N;
    a0 = 0;
    a1 = N;
  } else {
    s.start = A.cu[b] / A.cp;
    s.half = N / (2 * A.cp);
    a0 = s.half * c;
    a1 = a0 + s.half;
    b0 = N - s.half * (c + 1);
    b1 = b0 + s.half;
  }
  s.pA = max(s.p0, a0);
  s.cA = max(min(p1, a1) - s.pA, (int64_t)0);
  s.tA = s.start + s.pA - a0;
  s.pB = max(s.p0, b0);
  s.cB = max(min(p1, b1) - s.pB, (int64_t)0);
  s.tB = s.start + s.half + s.pB - b0;
  return s;
}

__device__ __forceinline__ int64_t overlap(int64_t t0, int64_t cnt, int64_t lo, int64_t hi) {
  return max(min(t0 + cnt, hi) - max(t0, lo), (int64_t)0);
}

// exclusive block scan of one int64 per thread, returns the prefix and the block total in *total
__device__ int64_t block_exclusive_scan(int64_t v, int64_t* warp_tot, int64_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[warp] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t run = 0;
    for (int w = 0; w < kThreads / 32; ++w) {
      const int64_t t = warp_tot[w];
      warp_tot[w] = run;
      run += t;
    }
    *total = run;
  }
  __syncthreads();
  const int64_t r = warp_tot[warp] + x - v;
  __syncthreads();
  return r;
}

// last b in [0, n) with key[b] <= x (key ascending), or -1
__device__ __forceinline__ int64_t upper_index(const int64_t* key, int64_t n, int64_t x) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (key[mid] <= x) lo = mid + 1;
    else hi = mid;
  }
  return lo - 1;
}

__global__ void __launch_bounds__(kThreads) mp_plan_kernel(Args A) {
  extern __shared__ int64_t o[];  // [bsz + 1] compact offset of each sequence on the CP rank of the current pass
  __shared__ int64_t warp_tot[kThreads / 32], tot;
  __shared__ int64_t cnt[kMaxRanks];  // [cp][tp]: rows of rank (c, k) in its shard (SP), or R_c in every k
  __shared__ int err;
  const int64_t bsz = A.bsz, L = A.L;
  const int tp = A.tp, cp = A.cp;
  if (threadIdx.x == 0) err = 0;
  __syncthreads();

  const int64_t per = (bsz + kThreads - 1) / kThreads;
  const int64_t bb0 = min((int64_t)threadIdx.x * per, bsz), bb1 = min(bb0 + per, bsz);
  int bad = 0;
  for (int64_t b = bb0; b < bb1; ++b) {
    const int64_t rb = A.resp[b], s = A.cu[b], nb = A.n[b], N = A.cu[b + 1] - s;
    if (rb < 0 || rb > L) bad |= E_RESP;
    if (nb - rb < 1) bad |= E_PROMPT;
    if (s < 0) bad |= E_BOUNDS;
    if (s + nb > A.cu[b + 1]) bad |= E_ORDER;
    if (cp > 1 && (N % (2 * cp) != 0 || (b == 0 && s % (2 * cp) != 0))) bad |= E_ALIGN;
  }
  if (threadIdx.x == 0 && (A.cu[bsz] / cp > A.Tc || (A.sp && A.Tc % tp != 0))) bad |= E_SHARD;
  if (bad) atomicOr(&err, bad);
  __syncthreads();
  const bool ok = err == 0;  // with bad lengths the runs are meaningless: count nothing, write sentinels

  // pass 1: counts of every rank
  for (int c = 0; c < cp; ++c) {
    for (int k = 0; k < (A.sp ? tp : 1); ++k) {
      const int64_t lo = A.sp ? k * A.Ts : 0, hi = A.sp ? lo + A.Ts : A.Tc;
      int64_t v = 0;
      for (int64_t b = bb0; ok && b < bb1; ++b) {
        const Runs s = runs_of(A, b, c);
        v += overlap(s.tA, s.cA, lo, hi) + overlap(s.tB, s.cB, lo, hi);
      }
      block_exclusive_scan(v, warp_tot, &tot);
      if (threadIdx.x == 0) {
        if (A.sp) cnt[c * tp + k] = tot;
        else
          for (int kk = 0; kk < tp; ++kk) cnt[c * tp + kk] = tot;
      }
    }
  }
  __syncthreads();
  int64_t Rmax_c = 1, Rmax_k = 1, Rc = 0;
  for (int c = 0; c < cp; ++c) {
    int64_t r = 0;
    for (int k = 0; k < (A.sp ? tp : 1); ++k) r += cnt[c * tp + k];
    Rmax_c = max(Rmax_c, r);
    if (c == A.c) Rc = r;
  }
  if (A.sp)
    for (int k = 0; k < tp; ++k) Rmax_k = max(Rmax_k, cnt[A.c * tp + k]);
  else
    Rmax_k = Rc;
  int64_t off_k = 0;  // first compact row of this rank's shard
  for (int k = 0; A.sp && k < A.k; ++k) off_k += cnt[A.c * tp + k];
  const int64_t mine = A.sp ? cnt[A.c * tp + A.k] : Rc;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    A.status[0] = err | ((Rc > A.cap_c || (A.sp && Rmax_k > A.cap_k)) ? E_CAPACITY : 0);
    for (int i = 0; i < cp * tp; ++i) A.status[1 + i] = cnt[i];
  }
  const int64_t nc = min(Rc, A.cap_c), nk = A.sp ? min(Rmax_k, A.cap_k) : 0;
  const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, gstride = (int64_t)gridDim.x * blockDim.x;

  // pass 2: each CP rank's offsets; its compact rows' cells, and this rank's own maps
  for (int c = 0; c < cp; ++c) {
    int64_t v = 0;
    for (int64_t b = bb0; ok && b < bb1; ++b) {
      const Runs s = runs_of(A, b, c);
      v += s.cA + s.cB;
    }
    int64_t run = block_exclusive_scan(v, warp_tot, &tot);
    for (int64_t b = bb0; b < bb1; ++b) {
      o[b] = run;
      if (ok) {
        const Runs s = runs_of(A, b, c);
        run += s.cA + s.cB;
      }
    }
    if (threadIdx.x == 0) o[bsz] = tot;
    __syncthreads();
    const int64_t R = ok ? o[bsz] : 0;
    for (int64_t i = gtid; i < R; i += gstride) {  // compact row i of CP rank c
      const int64_t b = upper_index(o, bsz, i), q = i - o[b];
      const Runs s = runs_of(A, b, c);
      const int64_t p = q < s.cA ? s.pA + q : s.pB + (q - s.cA);
      const int64_t t = q < s.cA ? s.tA + q : s.tB + (q - s.cA);
      const int64_t j = p - s.p0;
      A.cell_map[b * L + j] = c * Rmax_c + i;
      if (c != A.c || i >= nc) continue;
      A.rows[i] = t;
      A.targets[i] = A.responses[b * L + j];
      A.cells[i] = b * L + j;
      if (A.sp) {
        const int64_t kk = t / A.Ts;
        int64_t off = 0;
        for (int x = 0; x < kk; ++x) off += cnt[c * tp + x];
        A.unpad[i] = kk * Rmax_k + (i - off);
        if (kk == A.k && i - off < nk) A.send[i - off] = t - kk * A.Ts;
      } else {
        A.unpad[i] = i;
      }
    }
    if (c == A.c) {  // the rows of this rank's hidden shard: compact row (no SP) or reduce-scatter slot (SP)
      const int64_t nrows = A.sp ? A.Ts : A.Tc, base = A.sp ? A.k * A.Ts : 0;
      for (int64_t x = gtid; x < nrows; x += gstride) {
        const int64_t t = base + x;
        int64_t m = -1;
        int64_t lo = 0, hi = bsz;  // last b with start_b <= t
        while (ok && lo < hi) {
          const int64_t mid = (lo + hi) >> 1;
          if ((cp == 1 ? A.cu[mid] : A.cu[mid] / cp) <= t) lo = mid + 1;
          else hi = mid;
        }
        const int64_t b = lo - 1;
        if (ok && b >= 0) {
          const Runs s = runs_of(A, b, c);
          int64_t i = -1;
          if (t >= s.tA && t < s.tA + s.cA) i = o[b] + (t - s.tA);
          else if (t >= s.tB && t < s.tB + s.cB) i = o[b] + s.cA + (t - s.tB);
          if (i >= 0) m = A.sp ? i - off_k : i;
          if (m >= (A.sp ? nk : nc)) m = -1;
        }
        A.hidden_map[x] = m;
      }
    }
    __syncthreads();  // o is rebuilt for the next CP rank
  }
  // response cells past r_b (and every cell of an invalid plan), the send list's pads, the slot map
  const int64_t ncell = bsz * L, nslot = A.sp ? (int64_t)tp * nk : 0;
  for (int64_t i = gtid; i < ncell + nk + nslot; i += gstride) {
    if (i < ncell) {
      const int64_t b = i / L, j = i - b * L;
      if (!ok || j >= A.resp[b]) A.cell_map[i] = -1;
    } else if (i < ncell + nk) {
      const int64_t m = i - ncell;
      if (!ok || m >= mine) A.send[m] = -1;
    } else {  // slot (k', m) of the [tp, Rmax_k] reduce-scatter layout: the compact row it carries, or -1
      const int64_t q = i - ncell - nk, kk = q / nk, m = q - kk * nk;
      int64_t off = 0;
      for (int x = 0; x < kk; ++x) off += cnt[A.c * tp + x];
      A.slot_map[q] = (ok && m < cnt[A.c * tp + kk]) ? off + m : -1;
    }
  }
}

// dst[i, :] = bf16(src[idx[i], :]) (round to nearest even, once), zeros where idx[i] < 0; 8 columns per thread
__global__ void __launch_bounds__(256) pack_grad_kernel(const float* __restrict__ src, const int64_t* __restrict__ idx,
                                                        __nv_bfloat16* __restrict__ dst, int64_t n_out, int64_t H) {
  const int64_t vpr = H / 8, total = n_out * vpr;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / vpr, v = i - row * vpr, s = idx[row];
    uint4 out = make_uint4(0u, 0u, 0u, 0u);
    if (s >= 0) {
      const float4* p = reinterpret_cast<const float4*>(src + s * H + v * 8);
      const float4 a = p[0], b = p[1];
      __nv_bfloat162 h[4] = {__floats2bfloat162_rn(a.x, a.y), __floats2bfloat162_rn(a.z, a.w),
                             __floats2bfloat162_rn(b.x, b.y), __floats2bfloat162_rn(b.z, b.w)};
      out = *reinterpret_cast<uint4*>(h);
    }
    reinterpret_cast<uint4*>(dst)[i] = out;
  }
}

}  // namespace

extern "C" int rb200_response_rows_mp_plan(const int64_t* cu_seqlens_padded, const int64_t* seq_lengths,
                                           const int64_t* response_lengths, const int64_t* responses, int64_t bsz,
                                           int64_t L, int64_t T_c, int tp_size, int cp_size, int sequence_parallel,
                                           int tp_rank, int cp_rank, int64_t capacity_c, int64_t capacity_k,
                                           int64_t* rows, int64_t* send, int64_t* unpad, int64_t* slot_map,
                                           int64_t* targets, int64_t* cell_map, int64_t* cells, int64_t* hidden_map,
                                           int64_t* status, rb200_stream_t stream) {
  if (!cu_seqlens_padded || !seq_lengths || !response_lengths || !responses || !cell_map || !hidden_map || !status)
    return RB200_E_NULL;
  if (capacity_c > 0 && (!rows || !unpad || !targets || !cells)) return RB200_E_NULL;
  if (sequence_parallel && capacity_k > 0 && (!send || !slot_map)) return RB200_E_NULL;
  if (bsz <= 0 || bsz > kMaxBsz || L <= 0 || T_c <= 0 || capacity_c < 0 || capacity_k < 0) return RB200_E_SHAPE;
  if (tp_size < 1 || cp_size < 1 || tp_size * cp_size > kMaxRanks) return RB200_E_ARG;
  if (tp_rank < 0 || tp_rank >= tp_size || cp_rank < 0 || cp_rank >= cp_size) return RB200_E_ARG;
  const int sp = sequence_parallel ? 1 : 0;
  Args A{cu_seqlens_padded, seq_lengths, response_lengths, responses, bsz, L, T_c, sp ? T_c / tp_size : T_c,
         capacity_c, capacity_k, tp_size, cp_size, sp, tp_rank, cp_rank,
         rows, send, unpad, slot_map, targets, cell_map, cells, hidden_map, status};
  const size_t smem = (size_t)(bsz + 1) * sizeof(int64_t);
  cudaError_t e = cudaFuncSetAttribute(mp_plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  const int64_t total = capacity_c + bsz * L + T_c + (int64_t)tp_size * capacity_k;
  int64_t blocks = (total + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)rb::sm_count() * 4;
  if (blocks > cap) blocks = cap;
  mp_plan_kernel<<<(unsigned)blocks, kThreads, smem, rb::as_stream(stream)>>>(A);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_response_rows_mp_pack_grad(const float* dx, const int64_t* idx, void* out, int64_t n_out,
                                                int64_t H, rb200_stream_t stream) {
  if (!dx || !idx || !out) return RB200_E_NULL;
  if (n_out <= 0 || H <= 0 || H % 8 != 0) return RB200_E_SHAPE;
  if ((reinterpret_cast<uintptr_t>(dx) | reinterpret_cast<uintptr_t>(out)) & 15) return RB200_E_ARG;
  int64_t blocks = (n_out * (H / 8) + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * 16;
  if (blocks > cap) blocks = cap;
  pack_grad_kernel<<<(unsigned)(blocks < 1 ? 1 : blocks), 256, 0, rb::as_stream(stream)>>>(
      dx, idx, static_cast<__nv_bfloat16*>(out), n_out, H);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
