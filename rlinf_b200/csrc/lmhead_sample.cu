// Action-token sampling fused into the LM head (the OpenVLA-OFT rollout): hidden states X [N, H] and W [V, H] (bf16)
// in, action_sample.cu's tokens, log-probs and actions out, without the full-vocabulary logits.
// The rollout applies the bin window before top-k, so only the window's W rows of the weight are needed:
//   ACC  the lmhead mainloop over [v_lo, v_hi) stores the raw fp32 accumulator [row tiles * 128, ld] in the workspace
//        (about 1 KiB per row at the 256-column OpenVLA window);
//   then action_sample.cu's sampler runs on that block.
// No atomics; nothing depends on the SM count.
#include "lmhead_core.cuh"

namespace rb {
namespace asmp {
int sample_tiles(const float* block, int64_t ld, int v_lo, int v_hi, int do_sample, double inv_temperature, int top_k,
                 uint64_t seed, uint64_t offset, const rb200_action_bins* bins, int64_t rt0, int64_t nt, int tpb,
                 int64_t L_rows, int64_t* token, float* logprob, double* action, const rb200_sample_step* step,
                 int64_t out_L, cudaStream_t st);
int check_common(int W, int do_sample, double inv_temperature, const rb200_action_bins* bins, const int64_t* token,
                 const float* logprob, const double* action);
int check_step(const rb200_sample_step* step, int64_t L);
}  // namespace asmp
}  // namespace rb

namespace {

int64_t window_ld(int W) { return cdiv(W, 4) * 4; }  // block row length: 16-byte rows

}  // namespace

extern "C" int64_t rb200_lmhead_sample_workspace_bytes(int64_t N, int64_t L, int H, int V, int v_lo, int v_hi) {
  Geo g;
  if (make_geo(g, N, L, L * H, H, H, V, v_lo, v_hi) != RB200_OK) return -1;
  return g.row_tiles * BM * window_ld(v_hi - v_lo) * 4;
}

// step may be NULL (dense outputs, the host offset, no counter advance).  A call with a step struct and L == 1 (one
// position per sample, a generate step on [bsz, H] rows) runs the GEMM over the bsz rows as one item of bsz positions, so that its row tiles
// hold 128 samples instead of one each; the sampler still writes one output row per sample.
extern "C" int rb200_lmhead_sample_step(const void* hidden, const void* weight, int64_t N, int64_t L,
                                        int64_t batch_stride, int64_t row_stride, int H, int V, int v_lo, int v_hi,
                                        int do_sample, double inv_temperature, int top_k, uint64_t seed,
                                        uint64_t offset, const rb200_action_bins* bins, int64_t* token, float* logprob,
                                        double* action, void* workspace, int64_t workspace_bytes,
                                        const rb200_sample_step* step, rb200_stream_t stream) {
  if (!hidden || !weight || !workspace) return RB200_E_NULL;
  if (((reinterpret_cast<uintptr_t>(hidden) | reinterpret_cast<uintptr_t>(weight) |
        reinterpret_cast<uintptr_t>(workspace)) & 15) != 0)
    return RB200_E_ALIGN;
  const int64_t out_L = L;
  if (step && L == 1 && N > 1) {
    L = N;
    row_stride = batch_stride;
    batch_stride = N * row_stride;
  }
  Geo g;
  int e = make_geo(g, N, L, batch_stride, row_stride, H, V, v_lo, v_hi);
  if (e) return e;
  const int W = v_hi - v_lo;
  if ((e = rb::asmp::check_common(W, do_sample, inv_temperature, bins, token, logprob, action))) return e;
  if ((e = rb::asmp::check_step(step, out_L))) return e;
  const int64_t ld = window_ld(W);
  if (workspace_bytes < g.row_tiles * BM * ld * 4) return RB200_E_ARG;
  Params P{};
  base_params(P, g, 1.0);
  if (x_map(&P.a, hidden, g, BM) || w_map(&P.b, weight, g, BN)) return RB200_E_UNSUPPORTED;
  P.rt0 = 0;
  P.n_kb = H / BK;
  P.c0 = v_lo;
  P.width = W;
  P.ld = (int)ld;
  P.acc_out = static_cast<float*>(workspace);
  split_ranges(g.row_tiles, W, P.n_vtiles, P.n_ranges, P.tiles_per_range);
  cudaStream_t st = rb::as_stream(stream);
  if ((e = launch<ACC>(P, (int)(g.row_tiles * P.n_ranges), st))) return e;
  return rb::asmp::sample_tiles(P.acc_out, ld, v_lo, v_hi, do_sample, inv_temperature, top_k, seed, offset, bins, 0,
                                g.row_tiles, (int)g.tpb, g.L, token, logprob, action, step, out_L, st);
}
