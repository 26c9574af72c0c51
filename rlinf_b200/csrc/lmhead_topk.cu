// Top-k filtered log-probabilities and entropies fused into the LM head (the OpenVLA action head with top_k > 0):
// hidden states X [N, H] and W [V, H] (bf16) in, the top_k-th largest logit of each row over the whole vocabulary, then
// lse / logprob / entropy over the window's columns that reach it (csrc/topk.cu's semantics).
// The threshold needs every column, not only the window's, so the forward runs per block of whole 128-row tiles:
//   ACC  the lmhead mainloop over [0, V) stores the raw fp32 accumulator [block rows, ld] in the workspace;
//   then topk.cu's forward on that block (fp32, inv_T) writes logprob, entropy, lse and the threshold of its rows.
// The block is as many row tiles as the workspace holds.  The backward is lmhead.cu's, chunk by chunk over the window,
// with the DZT epilogue: dZ masked by acc >= thr[row] on the same mainloop's raw accumulator (same operands, majorness
// and k-block order as ACC, so the same bits), then lmhead.cu's DW / DX kernels.  No atomics; nothing depends on the
// SM count or on the row block.
#include "lmhead_core.cuh"

namespace rb {
namespace lmh {
int bwd_masked(const void* hidden, const void* weight, const int64_t* target, int64_t N, int64_t L, int64_t batch_stride,
               int64_t row_stride, int H, int V, int v_lo, int v_hi, double inv_temperature, const float* thr,
               const float* lse, const float* entropy, const float* grad_logprob, const float* grad_entropy,
               void* d_hidden, void* d_weight, void* workspace, int64_t workspace_bytes, DzLaunch dz_launch,
               cudaStream_t st);
}  // namespace lmh
namespace topk {
int fwd_tiles(const float* block, int64_t ld, int V, int v_lo, int v_hi, double inv_temperature, int top_k,
              const int64_t* target, int64_t rt0, int64_t nt, int tpb, int64_t L_rows, float* logprob, float* entropy,
              float* lse, float* threshold, cudaStream_t st);
}  // namespace topk
}  // namespace rb

namespace {

constexpr int64_t kRowBlockBudget = 512ll << 20;  // bytes of the fp32 accumulator block when row_block <= 0

int64_t acc_ld(int V) { return cdiv(V, 4) * 4; }  // accumulator row length: 16-byte rows
int64_t tile_bytes(int V) { return (int64_t)BM * acc_ld(V) * 4; }

// row tiles per block: row_block rows (rounded up to whole tiles) or what kRowBlockBudget allows, at least one
int64_t block_tiles(const Geo& g, int64_t row_block) {
  int64_t nt = row_block > 0 ? cdiv(row_block, BM) : kRowBlockBudget / tile_bytes(g.V);
  if (nt < 1) nt = 1;
  return nt < g.row_tiles ? nt : g.row_tiles;
}

int dzt_launch(const void* params, int items, cudaStream_t st) {
  return launch<DZT>(*static_cast<const Params*>(params), items, st);
}

}  // namespace

extern "C" int64_t rb200_lmhead_topk_workspace_bytes(int64_t N, int64_t L, int H, int V, int v_lo, int v_hi,
                                                     int64_t row_block, int64_t vocab_chunk) {
  Geo g;
  if (make_geo(g, N, L, L * H, H, H, V, v_lo, v_hi) != RB200_OK) return -1;
  const int64_t whole = cdiv(v_hi - v_lo, BN) * BN;
  int64_t vc = vocab_chunk <= 0 ? whole : cdiv(vocab_chunk, BN) * BN;
  if (vc > whole) vc = whole;
  const int64_t f = block_tiles(g, row_block) * tile_bytes(V), b = bwd_ws_bytes(g, vc);
  return f > b ? f : b;
}

extern "C" int rb200_lmhead_topk_logprob_entropy_fwd(const void* hidden, const void* weight, const int64_t* target,
                                                     int64_t N, int64_t L, int64_t batch_stride, int64_t row_stride,
                                                     int H, int V, int v_lo, int v_hi, double inv_temperature,
                                                     int top_k, float* logprob, float* entropy, float* lse,
                                                     float* threshold, void* workspace, int64_t workspace_bytes,
                                                     rb200_stream_t stream) {
  int e = check_ptrs(hidden, weight, target, workspace);
  if (e) return e;
  if (!logprob || !threshold || !workspace) return RB200_E_NULL;
  if (!(inv_temperature > 0.0)) return RB200_E_ARG;
  Geo g;
  if ((e = make_geo(g, N, L, batch_stride, row_stride, H, V, v_lo, v_hi))) return e;
  if (top_k < 1 || top_k >= V) return RB200_E_ARG;
  const int64_t nt_max = workspace_bytes / tile_bytes(V) < g.row_tiles ? workspace_bytes / tile_bytes(V) : g.row_tiles;
  if (nt_max < 1) return RB200_E_ARG;
  cudaStream_t st = rb::as_stream(stream);
  for (int64_t rt0 = 0; rt0 < g.row_tiles; rt0 += nt_max) {
    const int64_t nt = g.row_tiles - rt0 < nt_max ? g.row_tiles - rt0 : nt_max;
    Params P{};
    base_params(P, g, inv_temperature);
    if (x_map(&P.a, hidden, g, BM) || w_map(&P.b, weight, g, BN)) return RB200_E_UNSUPPORTED;
    P.row_tiles = (int)nt;
    P.rt0 = (int)rt0;
    P.n_kb = H / BK;
    P.c0 = 0;
    P.width = V;
    P.ld = (int)acc_ld(V);
    P.acc_out = static_cast<float*>(workspace);
    split_ranges(nt, V, P.n_vtiles, P.n_ranges, P.tiles_per_range);
    if ((e = launch<ACC>(P, (int)(nt * P.n_ranges), st))) return e;
    if ((e = rb::topk::fwd_tiles(P.acc_out, P.ld, V, v_lo, v_hi, inv_temperature, top_k, target, rt0, nt, (int)g.tpb,
                                 g.L, logprob, entropy, lse, threshold, st)))
      return e;
  }
  return RB200_OK;
}

extern "C" int rb200_lmhead_topk_logprob_entropy_bwd(const void* hidden, const void* weight, const int64_t* target,
                                                     int64_t N, int64_t L, int64_t batch_stride, int64_t row_stride,
                                                     int H, int V, int v_lo, int v_hi, double inv_temperature,
                                                     const float* threshold, const float* lse, const float* entropy,
                                                     const float* grad_logprob, const float* grad_entropy,
                                                     void* d_hidden, void* d_weight, void* workspace,
                                                     int64_t workspace_bytes, rb200_stream_t stream) {
  int e = check_ptrs(hidden, weight, target, workspace);
  if (e) return e;
  if (!threshold || !lse || !workspace || (grad_entropy && !entropy)) return RB200_E_NULL;
  if (((reinterpret_cast<uintptr_t>(d_hidden) | reinterpret_cast<uintptr_t>(d_weight)) & 3) != 0) return RB200_E_ALIGN;
  if (!(inv_temperature > 0.0)) return RB200_E_ARG;
  return rb::lmh::bwd_masked(hidden, weight, target, N, L, batch_stride, row_stride, H, V, v_lo, v_hi, inv_temperature,
                             threshold, lse, entropy, grad_logprob, grad_entropy, d_hidden, d_weight, workspace,
                             workspace_bytes, dzt_launch, rb::as_stream(stream));
}
