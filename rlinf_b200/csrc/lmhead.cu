// SURVEY 8(f)3 fused into the LM-head GEMM: token log-probabilities and entropies from the last hidden states X [N, H]
// and the LM-head weight W [V, H] (bf16), forward and backward, without ever storing the logits X.W^T.
//   z = (X . W^T) * inv_T  (fp32 accumulation of bf16 products), columns outside [v_lo, v_hi) = -inf
//   logprob = z_t - lse,  H = lse - sum p_i z_i,  lse           (the statistics and row finish of softmax_acc.cuh)
//   dz_i = inv_T * (g_lp * (1[i = t] - p_i) - g_H * p_i * (z_i - lse + H)),  dX = dZ . W,  dW = dZ^T . X
// One bf16 wgmma mainloop (m64n128k16, both operands from shared memory, K-major or MN-major per operand) with four
// epilogues:
//   FWD  softmax statistics: a work item is (128-row tile, contiguous range of 256-wide vocabulary tiles); it keeps its
//        rows' (m, s, t) in registers across the range and writes one partial per (range, row); combine_kernel merges
//        the partials in range order.  z_target is written by the one thread whose tile holds the target column.
//   DZ   (backward, per vocabulary chunk [c0, c0 + width)): recompute z, form dZ from the saved lse / H, round to bf16
//        and store it into the workspace [N, ld].
//   DW   dW[c0:c0+width] = dZ^T . X over all N rows (A and B MN-major), written once in bf16.
//   DX   dX_acc (+)= dZ . W[c0:c0+width] (A K-major, B MN-major) into an fp32 workspace; the last chunk writes bf16 dX.
// Everything runs in a fixed order: no atomics, and no output depends on the SM count or on scheduling.
// Rows are addressed through the row geometry of the logits kernels (row r = (b, p), b = r / L, p = r % L, element
// (b, p, h) at b * batch_stride + p * row_stride + h), as a 3-D TMA map [bsz, L, H]: row tiles never straddle two batch
// items, positions >= L are zero-filled by TMA and masked in the epilogues.
#include "lmhead_core.cuh"

namespace {

// merge the per-range partials of each row in range order, then the row finish of the logits kernels
__global__ void __launch_bounds__(256) combine_kernel(const float* __restrict__ part, const float* __restrict__ zt,
                                                      const int64_t* __restrict__ target, int64_t N, int n_ranges,
                                                      int v_lo, int v_hi, float* logprob, float* entropy, float* lse) {
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
  const int64_t tgr = target[r];
  const bool t_in = tgr >= v_lo && tgr < v_hi;
  rb::smx::finish_row(a, t_in ? zt[r] : 0.f, t_in, r, logprob, entropy, lse);
}

// the FWD pass over [g.v_lo, g.v_hi): per-range partials at P.part, the target's z at P.zt (workspace)
int fwd_partials(Params& P, const Geo& g, const void* hidden, const void* weight, const int64_t* target,
                 double inv_temperature, void* workspace, cudaStream_t st) {
  P = Params{};
  base_params(P, g, inv_temperature);
  if (x_map(&P.a, hidden, g, BM) || w_map(&P.b, weight, g, BN)) return RB200_E_UNSUPPORTED;
  P.n_kb = g.H / BK;
  P.n_ranges = g.n_ranges; P.tiles_per_range = g.tiles_per_range; P.n_vtiles = g.n_vtiles;
  P.target = target;
  P.part = static_cast<float*>(workspace);
  P.zt = P.part + (size_t)g.n_ranges * g.N * 3;
  return launch<FWD>(P, (int)(g.row_tiles * g.n_ranges), st);
}


// The backward over [g.v_lo, g.v_hi) in chunks of vc columns.  dX is summed in fp32 in dx_acc over the chunks; with dx
// the last chunk writes it there in bf16 instead, without dx it stays in dx_acc.
int bwd_chunks(const Geo& g, const void* hidden, const void* weight, const int64_t* target, double inv_temperature,
               const float* lse, const float* entropy, const float* grad_logprob, const float* grad_entropy, int64_t vc,
               __nv_bfloat16* dz, float* dx_acc, __nv_bfloat16* dx, __nv_bfloat16* dw, cudaStream_t st,
               rb::lmh::DzLaunch dz_launch = nullptr, const float* thr = nullptr) {
  const int H = g.H, V = g.V, v_lo = g.v_lo, v_hi = g.v_hi;
  if (dw) {  // rows outside the window get no gradient
    if (v_lo > 0) RB_CHECK_CUDA(cudaMemsetAsync(dw, 0, (size_t)v_lo * H * 2, st));
    if (v_hi < V) RB_CHECK_CUDA(cudaMemsetAsync(dw + (size_t)v_hi * H, 0, (size_t)(V - v_hi) * H * 2, st));
  }
  const int n_ntiles = (int)cdiv(H, BN);
  int e;
  for (int64_t c0 = v_lo; c0 < v_hi; c0 += vc) {
    const int width = (int)((v_hi - c0) < vc ? (v_hi - c0) : vc);
    Params P{};
    base_params(P, g, inv_temperature);
    P.c0 = (int)c0; P.width = width; P.ld = (int)vc;
    P.target = target; P.lse = lse; P.h_in = entropy; P.g_lp = grad_logprob; P.g_h = grad_entropy;
    P.dz = dz; P.dx_acc = dx_acc; P.dx = dx; P.dw = dw;
    P.n_ntiles = n_ntiles;
    P.first = c0 == v_lo;
    P.last = dx && c0 + width >= v_hi;
    // (a) dZ of the chunk
    Params A = P;
    if (x_map(&A.a, hidden, g, BM) || w_map(&A.b, weight, g, BN)) return RB200_E_UNSUPPORTED;
    A.n_kb = H / BK;
    split_ranges(g.row_tiles, width, A.n_vtiles, A.n_ranges, A.tiles_per_range);
    A.thr = thr;
    if ((e = dz_launch ? dz_launch(&A, (int)(g.row_tiles * A.n_ranges), st)
                       : launch<DZ>(A, (int)(g.row_tiles * A.n_ranges), st)))
      return e;
    // (b) dW[c0 : c0 + width] = dZ^T . X over all rows
    if (dw) {
      Params B = P;
      if (dz_map(&B.a, dz, g, width, vc, 64, 64) || x_map(&B.b, hidden, g, 64)) return RB200_E_UNSUPPORTED;
      B.kpb = (int)cdiv(g.L, BK);
      B.n_kb = (int)(g.bsz * B.kpb);
      if ((e = launch<DW>(B, (int)(cdiv(width, BM) * n_ntiles), st))) return e;
    }
    // (c) dX (+)= dZ . W[c0 : c0 + width]
    if (dx_acc || dx) {
      Params C = P;
      if (dz_map(&C.a, dz, g, width, vc, 64, BM) || w_map(&C.b, weight, g, 64)) return RB200_E_UNSUPPORTED;
      C.n_kb = (int)cdiv(width, BK);
      if ((e = launch<DX>(C, (int)(g.row_tiles * n_ntiles), st))) return e;
    }
  }
  return RB200_OK;
}

// ---- vocabulary-parallel shard (rank k owns global columns [vocab_start, vocab_start + Vs)) ----
// the shard's part of the global window [v_lo, v_hi), in shard columns; lo >= hi when the shard misses the window
void shard_window(int64_t vocab_start, int Vs, int v_lo, int v_hi, int& lo, int& hi) {
  const int64_t l = v_lo - vocab_start, h = v_hi - vocab_start;
  lo = (int)(l < 0 ? 0 : (l > Vs ? Vs : l));
  hi = (int)(h < 0 ? 0 : (h > Vs ? Vs : h));
}
// the shard-local targets (target - vocab_start) head the workspace; the kernels' own workspace follows
int64_t vp_target_bytes(int64_t N) { return cdiv(N * 8, 256) * 256; }

int vp_check(int Vs, int64_t vocab_start, int v_lo, int v_hi, double inv_temperature) {
  if (Vs <= 0 || vocab_start < 0 || vocab_start % Vs != 0 || v_lo < 0 || v_lo >= v_hi) return RB200_E_SHAPE;
  if (!(inv_temperature > 0.0)) return RB200_E_ARG;
  return RB200_OK;
}

}  // namespace

namespace rb {
namespace vp {
int shift_target(const int64_t* target, int64_t N, int64_t vocab_start, int64_t* out, cudaStream_t st);
int range_record(const float* part, const float* zt, const int64_t* local_target, int64_t N, int n_ranges, int lo,
                 int hi, float* rec, cudaStream_t st);
}  // namespace vp
}  // namespace rb

namespace rb {
namespace lmh {
// The backward of rb200_lmhead_logprob_entropy_bwd with the dZ kernel launched by dz_launch (given the chunk's Params
// with thr set): the top-k backward of lmhead_topk.cu runs this object's DW / DX kernels through it.
int bwd_masked(const void* hidden, const void* weight, const int64_t* target, int64_t N, int64_t L, int64_t batch_stride,
               int64_t row_stride, int H, int V, int v_lo, int v_hi, double inv_temperature, const float* thr,
               const float* lse, const float* entropy, const float* grad_logprob, const float* grad_entropy,
               void* d_hidden, void* d_weight, void* workspace, int64_t workspace_bytes, DzLaunch dz_launch,
               cudaStream_t st) {
  Geo g;
  int e = make_geo(g, N, L, batch_stride, row_stride, H, V, v_lo, v_hi);
  if (e) return e;
  if (!d_hidden && !d_weight) return RB200_OK;
  const int64_t vc = bwd_chunk(g, workspace_bytes, (int64_t)N * H * 4);
  if (vc == 0) return RB200_E_ARG;
  __nv_bfloat16* dz = static_cast<__nv_bfloat16*>(workspace);
  float* dx_acc = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + dz_ws_bytes(g, vc));
  return bwd_chunks(g, hidden, weight, target, inv_temperature, lse, entropy, grad_logprob, grad_entropy, vc, dz,
                    d_hidden ? dx_acc : nullptr, static_cast<__nv_bfloat16*>(d_hidden),
                    static_cast<__nv_bfloat16*>(d_weight), st, dz_launch, thr);
}
}  // namespace lmh
}  // namespace rb

extern "C" int64_t rb200_lmhead_workspace_bytes(int64_t N, int64_t L, int H, int V, int v_lo, int v_hi,
                                                int64_t vocab_chunk) {
  Geo g;
  if (make_geo(g, N, L, L * H, H, H, V, v_lo, v_hi) != RB200_OK) return -1;
  const int64_t whole = cdiv(v_hi - v_lo, BN) * BN;
  int64_t vc = vocab_chunk <= 0 ? whole : cdiv(vocab_chunk, BN) * BN;
  if (vc > whole) vc = whole;
  const int64_t f = fwd_ws_bytes(g), b = bwd_ws_bytes(g, vc);
  return f > b ? f : b;
}

extern "C" int rb200_lmhead_logprob_entropy_fwd(const void* hidden, const void* weight, const int64_t* target, int64_t N,
                                                int64_t L, int64_t batch_stride, int64_t row_stride, int H, int V,
                                                int v_lo, int v_hi, double inv_temperature, float* logprob,
                                                float* entropy, float* lse, void* workspace, int64_t workspace_bytes,
                                                rb200_stream_t stream) {
  int e = check_ptrs(hidden, weight, target, workspace);
  if (e) return e;
  if (!logprob || !workspace) return RB200_E_NULL;
  if (!(inv_temperature > 0.0)) return RB200_E_ARG;
  Geo g;
  if ((e = make_geo(g, N, L, batch_stride, row_stride, H, V, v_lo, v_hi))) return e;
  if (workspace_bytes < fwd_ws_bytes(g)) return RB200_E_ARG;
  cudaStream_t st = rb::as_stream(stream);
  Params P;
  if ((e = fwd_partials(P, g, hidden, weight, target, inv_temperature, workspace, st))) return e;
  combine_kernel<<<(unsigned)cdiv(N, 256), 256, 0, st>>>(P.part, P.zt, target, N, g.n_ranges, v_lo, v_hi, logprob,
                                                          entropy, lse);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_lmhead_logprob_entropy_bwd(const void* hidden, const void* weight, const int64_t* target, int64_t N,
                                                int64_t L, int64_t batch_stride, int64_t row_stride, int H, int V,
                                                int v_lo, int v_hi, double inv_temperature, const float* lse,
                                                const float* entropy, const float* grad_logprob,
                                                const float* grad_entropy, void* d_hidden, void* d_weight,
                                                void* workspace, int64_t workspace_bytes, rb200_stream_t stream) {
  int e = check_ptrs(hidden, weight, target, workspace);
  if (e) return e;
  if (!lse || !workspace || (grad_entropy && !entropy)) return RB200_E_NULL;
  if (((reinterpret_cast<uintptr_t>(d_hidden) | reinterpret_cast<uintptr_t>(d_weight)) & 3) != 0) return RB200_E_ALIGN;
  if (!(inv_temperature > 0.0)) return RB200_E_ARG;
  Geo g;
  if ((e = make_geo(g, N, L, batch_stride, row_stride, H, V, v_lo, v_hi))) return e;
  if (!d_hidden && !d_weight) return RB200_OK;
  const int64_t vc = bwd_chunk(g, workspace_bytes, (int64_t)N * H * 4);
  if (vc == 0) return RB200_E_ARG;
  __nv_bfloat16* dz = static_cast<__nv_bfloat16*>(workspace);
  float* dx_acc = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + dz_ws_bytes(g, vc));
  return bwd_chunks(g, hidden, weight, target, inv_temperature, lse, entropy, grad_logprob, grad_entropy, vc, dz,
                    d_hidden ? dx_acc : nullptr, static_cast<__nv_bfloat16*>(d_hidden),
                    static_cast<__nv_bfloat16*>(d_weight), rb::as_stream(stream));
}

extern "C" int64_t rb200_lmhead_vp_workspace_bytes(int64_t N, int64_t L, int H, int Vs, int64_t vocab_start, int v_lo,
                                                   int v_hi, int64_t vocab_chunk) {
  if (vp_check(Vs, vocab_start, v_lo, v_hi, 1.0)) return -1;
  int lo, hi;
  shard_window(vocab_start, Vs, v_lo, v_hi, lo, hi);
  if (lo >= hi) {  // no mainloop: only the shape checks of a full shard
    Geo g;
    return make_geo(g, N, L, L * H, H, H, Vs, 0, Vs) != RB200_OK ? -1 : vp_target_bytes(N);
  }
  Geo g;
  if (make_geo(g, N, L, L * H, H, H, Vs, lo, hi) != RB200_OK) return -1;
  const int64_t f = fwd_ws_bytes(g);
  if (vocab_chunk < 0) return vp_target_bytes(N) + f;
  const int64_t whole = cdiv(hi - lo, BN) * BN;
  int64_t vc = vocab_chunk == 0 ? whole : cdiv(vocab_chunk, BN) * BN;
  if (vc > whole) vc = whole;
  const int64_t b = dz_ws_bytes(g, vc);  // the backward's dX sum is the caller's fp32 output
  return vp_target_bytes(N) + (f > b ? f : b);
}

extern "C" int rb200_lmhead_vp_partials_fwd(const void* hidden, const void* weight_shard, const int64_t* target,
                                            int64_t N, int64_t L, int64_t batch_stride, int64_t row_stride, int H,
                                            int Vs, int64_t vocab_start, int v_lo, int v_hi, double inv_temperature,
                                            float* record, void* workspace, int64_t workspace_bytes,
                                            rb200_stream_t stream) {
  int e = check_ptrs(hidden, weight_shard, target, workspace);
  if (e) return e;
  if (!record || !workspace) return RB200_E_NULL;
  if ((reinterpret_cast<uintptr_t>(record) & 15) != 0) return RB200_E_ALIGN;
  if ((e = vp_check(Vs, vocab_start, v_lo, v_hi, inv_temperature))) return e;
  int lo, hi;
  shard_window(vocab_start, Vs, v_lo, v_hi, lo, hi);
  Geo g;
  if ((e = make_geo(g, N, L, batch_stride, row_stride, H, Vs, lo < hi ? lo : 0, lo < hi ? hi : Vs))) return e;
  cudaStream_t st = rb::as_stream(stream);
  if (lo >= hi) return rb::vp::range_record(nullptr, nullptr, nullptr, N, 0, 0, 0, record, st);
  if (workspace_bytes < vp_target_bytes(N) + fwd_ws_bytes(g)) return RB200_E_ARG;
  int64_t* local_target = static_cast<int64_t*>(workspace);
  if ((e = rb::vp::shift_target(target, N, vocab_start, local_target, st))) return e;
  Params P;
  if ((e = fwd_partials(P, g, hidden, weight_shard, local_target, inv_temperature,
                        static_cast<uint8_t*>(workspace) + vp_target_bytes(N), st)))
    return e;
  return rb::vp::range_record(P.part, P.zt, local_target, N, g.n_ranges, lo, hi, record, st);
}

extern "C" int rb200_lmhead_vp_logprob_entropy_bwd(const void* hidden, const void* weight_shard, const int64_t* target,
                                                   int64_t N, int64_t L, int64_t batch_stride, int64_t row_stride,
                                                   int H, int Vs, int64_t vocab_start, int v_lo, int v_hi,
                                                   double inv_temperature, const float* lse, const float* entropy,
                                                   const float* grad_logprob, const float* grad_entropy,
                                                   float* d_hidden_partial, void* d_weight_shard, void* workspace,
                                                   int64_t workspace_bytes, rb200_stream_t stream) {
  int e = check_ptrs(hidden, weight_shard, target, workspace);
  if (e) return e;
  if (!lse || !workspace || (grad_entropy && !entropy)) return RB200_E_NULL;
  if (((reinterpret_cast<uintptr_t>(d_hidden_partial) | reinterpret_cast<uintptr_t>(d_weight_shard)) & 7) != 0)
    return RB200_E_ALIGN;
  if ((e = vp_check(Vs, vocab_start, v_lo, v_hi, inv_temperature))) return e;
  int lo, hi;
  shard_window(vocab_start, Vs, v_lo, v_hi, lo, hi);
  Geo g;
  if ((e = make_geo(g, N, L, batch_stride, row_stride, H, Vs, lo < hi ? lo : 0, lo < hi ? hi : Vs))) return e;
  if (!d_hidden_partial && !d_weight_shard) return RB200_OK;
  cudaStream_t st = rb::as_stream(stream);
  if (lo >= hi) {  // the shard misses the window: no gradient
    if (d_hidden_partial) RB_CHECK_CUDA(cudaMemsetAsync(d_hidden_partial, 0, (size_t)N * H * 4, st));
    if (d_weight_shard) RB_CHECK_CUDA(cudaMemsetAsync(d_weight_shard, 0, (size_t)Vs * H * 2, st));
    return RB200_OK;
  }
  const int64_t vc = bwd_chunk(g, workspace_bytes - vp_target_bytes(N), 0);
  if (vc == 0) return RB200_E_ARG;
  int64_t* local_target = static_cast<int64_t*>(workspace);
  if ((e = rb::vp::shift_target(target, N, vocab_start, local_target, st))) return e;
  return bwd_chunks(g, hidden, weight_shard, local_target, inv_temperature, lse, entropy, grad_logprob, grad_entropy,
                    vc, reinterpret_cast<__nv_bfloat16*>(static_cast<uint8_t*>(workspace) + vp_target_bytes(N)),
                    d_hidden_partial, nullptr, static_cast<__nv_bfloat16*>(d_weight_shard), st);
}
