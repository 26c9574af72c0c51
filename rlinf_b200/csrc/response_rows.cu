// Response-rows plan of the LM-head log-probabilities: which rows of the flattened [T, H] hidden states the loss reads,
// for the three batch layouts of the reasoning workers (padded, FSDP-packed, Megatron THD).  One launch turns the
// per-sequence lengths into the index maps that rb200_gather_rows moves data with: hidden -> compact rows, compact
// log-probs / entropies -> [bsz, L], [bsz, L] gradients -> compact, compact dX -> [T, H].
//
// Sequence b: a_b = the row of its first response token, r_b = its response length, s_b = its first row.  It owns
// n_b = r_b + shift compact rows (0 when r_b = 0), at offset o_b = sum_{i<b} n_i, holding the hidden rows
// a_b - 1 + k, k < n_b.  Compact row o_b + j predicts response token j (target = token at a_b + j); with shift 1
// (the FSDP-packed entropy alignment) row o_b + j + 1 holds that column's entropy.
// Every CTA rebuilds the per-sequence table (a_b, r_b, o_b) in shared memory with a block scan, so the plan needs no
// second launch; each output entry is then written by one thread.  Sentinel -1 = the zero row the caller appends.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int64_t kMaxBsz = 8192;

enum Layout { kPadded = 0, kFsdpPacked = 1, kMegatronThd = 2 };
// status[1] bits (mirror of RB200_RR_*)
enum Err { E_RESP = 1, E_PROMPT = 2, E_BOUNDS = 4, E_ORDER = 8, E_MAXPROMPT = 16, E_CAPACITY = 32 };

struct Args {
  int layout, shift;
  const int64_t *len0, *len1, *resp, *tokens;
  int64_t bsz, S, L, T, capacity;
  int64_t *rows, *targets, *cell_map, *hidden_map, *cells, *status;
};

// exclusive block scan of one int64 per thread (kThreads threads), returns the prefix and the block total in *total
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
  int64_t lo = 0, hi = n;  // answer + 1 in [lo, hi]
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (key[mid] <= x) lo = mid + 1;
    else hi = mid;
  }
  return lo - 1;
}

__global__ void __launch_bounds__(kThreads) plan_kernel(Args A) {
  extern __shared__ int64_t sm[];
  int64_t* a = sm;              // [bsz]   a_b
  int64_t* o = sm + A.bsz;      // [bsz+1] o_b, o[bsz] = R
  int64_t* r = sm + 2 * A.bsz + 1;  // [bsz] r_b
  __shared__ int64_t warp_tot[kThreads / 32], tot_span, tot_n;
  __shared__ int err;
  const int64_t bsz = A.bsz, L = A.L;
  if (threadIdx.x == 0) err = 0;

  // each thread owns a contiguous chunk of sequences
  const int64_t per = (bsz + kThreads - 1) / kThreads;
  const int64_t b0 = min((int64_t)threadIdx.x * per, bsz), b1 = min(b0 + per, bsz);
  int64_t span = 0, cnt = 0;  // FSDP packed stream length of the chunk, compact rows of the chunk
  int bad = 0;
  for (int64_t b = b0; b < b1; ++b) {
    const int64_t rb = A.resp[b];
    if (rb < 0 || rb > L) bad |= E_RESP;
    cnt += rb > 0 ? rb + A.shift : 0;
    if (A.layout == kFsdpPacked) span += A.len0[b] + rb;
  }
  const int64_t span0 = block_exclusive_scan(span, warp_tot, &tot_span);
  const int64_t cnt0 = block_exclusive_scan(cnt, warp_tot, &tot_n);
  span = span0;
  cnt = cnt0;
  for (int64_t b = b0; b < b1; ++b) {
    const int64_t rb = A.resp[b];
    int64_t s, ab;
    if (A.layout == kPadded) {
      s = b * A.S;
      ab = s + A.S - L;
    } else if (A.layout == kFsdpPacked) {
      const int64_t p = A.len0[b];
      s = span;
      ab = s + p;
      span += p + rb;
      if (p > A.S) bad |= E_MAXPROMPT;
    } else {
      s = A.len0[b];
      const int64_t n = A.len1[b];
      ab = s + n - rb;
      if (s + n > A.len0[b + 1]) bad |= E_ORDER;  // the sequence overruns its padded segment
    }
    if (ab - s < 1) bad |= E_PROMPT;
    if (s < 0 || ab + rb > A.T) bad |= E_BOUNDS;
    a[b] = ab;
    r[b] = rb;
    o[b] = cnt;
    cnt += rb > 0 ? rb + A.shift : 0;
  }
  if (threadIdx.x == 0) o[bsz] = tot_n;
  if (bad) atomicOr(&err, bad);
  __syncthreads();
  // ascending and non-overlapping: sequence b starts at or after the end of sequence b - 1
  for (int64_t b = (int64_t)threadIdx.x + 1; b < bsz; b += kThreads) {
    int64_t s;
    if (A.layout == kPadded) s = b * A.S;
    else if (A.layout == kFsdpPacked) s = a[b] - A.len0[b];
    else s = A.len0[b];
    if (s < a[b - 1] + r[b - 1]) atomicOr(&err, (int)E_ORDER);
  }
  if (A.layout == kMegatronThd && threadIdx.x == 0 && A.len0[0] < 0) atomicOr(&err, (int)E_BOUNDS);
  __syncthreads();
  const int64_t R = o[bsz];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    A.status[0] = R;
    A.status[1] = err | (R > A.capacity ? E_CAPACITY : 0);
    A.cells[0] = -1;
  }

  const int64_t nc = min(R, A.capacity), ncell = bsz * L;
  const int64_t total = nc + ncell + A.T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < nc) {  // compact row c: its hidden row, target and response cell
      const int64_t c = i, b = upper_index(o, bsz, c), k = c - o[b];
      const int64_t row = a[b] - 1 + k, nxt = row + 1;
      const bool lp = k < r[b];
      A.rows[c] = row;
      A.targets[c] = (lp && nxt >= 0 && nxt < A.T) ? A.tokens[nxt] : -1;
      A.cells[1 + c] = lp ? b * L + k : -1;
    } else if (i < nc + ncell) {  // response cell (b, j): the compact row of its log-prob
      const int64_t q = i - nc, b = q / L, j = q - b * L;
      A.cell_map[q] = j < r[b] ? o[b] + j : -1;
    } else {  // hidden row t: its compact row
      const int64_t t = i - nc - ncell;
      // a[b] - 1 is ascending for valid plans; sequences without rows own nothing
      int64_t lo = 0, hi = bsz;
      while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] - 1 <= t) lo = mid + 1;
        else hi = mid;
      }
      const int64_t b = lo - 1;
      int64_t m = -1;
      if (b >= 0) {
        const int64_t k = t - (a[b] - 1), n = o[b + 1] - o[b];
        if (k < n && o[b] + k < nc) m = o[b] + k;
      }
      A.hidden_map[t] = m;
    }
  }
}

}  // namespace

extern "C" int rb200_response_rows_plan(int layout, const int64_t* len0, const int64_t* len1,
                                        const int64_t* response_lengths, int64_t bsz, int64_t S, int64_t L, int64_t T,
                                        int entropy_shift, const int64_t* tokens, int64_t capacity, int64_t* rows,
                                        int64_t* targets, int64_t* cell_map, int64_t* hidden_map, int64_t* cells,
                                        int64_t* status, rb200_stream_t stream) {
  if (!response_lengths || !tokens || !cell_map || !hidden_map || !cells || !status) return RB200_E_NULL;
  if (capacity > 0 && (!rows || !targets)) return RB200_E_NULL;
  if (layout < kPadded || layout > kMegatronThd) return RB200_E_ARG;
  if ((layout != kPadded && !len0) || (layout == kMegatronThd && !len1)) return RB200_E_NULL;
  if (entropy_shift != 0 && entropy_shift != 1) return RB200_E_ARG;
  if (bsz <= 0 || bsz > kMaxBsz || L <= 0 || T <= 0 || capacity < 0) return RB200_E_SHAPE;
  if (layout == kPadded && (S < L + 1 || bsz * S != T)) return RB200_E_SHAPE;
  Args A{layout, entropy_shift, len0, len1, response_lengths, tokens, bsz, S, L, T, capacity,
         rows, targets, cell_map, hidden_map, cells, status};
  const size_t smem = (size_t)(3 * bsz + 1) * sizeof(int64_t);
  cudaError_t e = cudaFuncSetAttribute(plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  const int64_t total = capacity + bsz * L + T;
  int64_t blocks = (total + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)rb::sm_count() * 4;
  if (blocks > cap) blocks = cap;
  plan_kernel<<<(unsigned)blocks, kThreads, smem, rb::as_stream(stream)>>>(A);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
