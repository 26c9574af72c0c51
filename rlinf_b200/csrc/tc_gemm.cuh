// Host-side interface of the fp16-split tensor-core GEMMs (tc_gemm_h.cu), grouped over up to two towers per launch.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rb {
namespace tc {

constexpr int BM = 128, BN = 256, BK = 32;  // BK fp32 = 128 bytes = one swizzle span

enum Epi { EPI_STORE = 0, EPI_BIAS_TANH = 1, EPI_TANHGRAD = 2 };

// debug/experiment switches (rb200_debug_set_flags): bit 1 (2) = round-1 fused-rollout layers (one-k-step weight prefetch);
// bit 2 (4) = hidden-layer backward as separate wgrad + dgrad launches instead of the fused dgrad_wgrad kernel
extern int g_debug_flags;

}  // namespace tc

namespace tch {

struct GemmLaunch {        // one group (tower) of a forward / dgrad launch
  const float* a;          // [M,K] fp32 streamed operand (activations or activation gradients)
  const float* b_hi;       // PACKED fp16 weight tiles of w * 2^10 for this launch's mode (pack_weights): per k-block of 32
                           // one contiguous 32 KB block = hi tile | lo tile, pre-swizzled as the MMA reads them; b_mn = 0
                           // takes the forward pack, b_mn = 1 the dgrad pack
  float* c;                // [M,256] fp32 result
  const float* bias;       // EPI_BIAS_TANH
  const float* h;          // EPI_TANHGRAD: previous activation [M,256]
  float* colsum;           // EPI_TANHGRAD: [256] += column sums of the output, or NULL
  const float* amax_in;    // device max|a| (gradient operands: scaled into fp16 range), or NULL
  float* amax_out;         // EPI_TANHGRAD: atomicMax of |output| (feeds the next gradient GEMM), or NULL
  const float* amax_x;     // device max|a| of an INPUT operand (observations; input_scale_log2_for), or NULL
};
struct WgradLaunch {
  const float* z;          // [n,256] activation gradients
  const float* h;          // [n,IN]  layer inputs
  float* dW;               // [256,IN] +=
  const float* amax_z;     // device max|z| or NULL
  const float* amax_h;     // device [IN] per-column max|h| of an INPUT operand (observations; input_scale_log2_for per
                           // column), or NULL (unscaled, as for the tanh outputs in [-1, 1] of the hidden layers)
};
struct SplitSpec {
  const float* src;        // weight matrix [256 out, K in] fp32
  float* hi;               // forward pack: 256*K floats of storage (typed float*: the cache lives in the fp32 wsplit buffer)
  float* lo;               // dgrad pack (K == 256 only) or NULL
  int64_t n;               // 256 * K
};

// epi: rb::tc::Epi.  b_mn = 0: C = epi(A . W^T) (forward, W [256,K]);  b_mn = 1: C = epi(A . W) (dgrad, W [256,256]).
int launch(const GemmLaunch* groups, int ngroups, int64_t M, int K, int epi, int b_mn, cudaStream_t st);
// The forward C = epi(A . W^T) for K <= 256 (tc_forward_h.cu): epi EPI_STORE or EPI_BIAS_TANH, the forward packs'
// weights resident in shared memory; bit-identical to launch(..., b_mn = 0), which stays the path for K > 256.
int forward(const GemmLaunch* groups, int ngroups, int64_t M, int K, int epi, cudaStream_t st);
int wgrad(const WgradLaunch* groups, int ngroups, int64_t n, int IN, cudaStream_t st);
struct BackwardLaunch {    // one group of the backward through a square hidden layer (tc_backward_h.cu)
  const float* z;          // [n,256] dZ_L
  const float* wpack;      // dgrad pack of W_L (split_weights)
  const float* h;          // [n,256] H_{L-1}
  float* dzprev;           // [n,256] dZ_{L-1} = (dZ_L . W_L) * (1 - H_{L-1}^2)
  float* dW;               // [256,256] += dZ_L^T . H_{L-1}
  float* colsum;           // [256] += column sums of dZ_{L-1}, or NULL
  const float* amax_in;    // device max|dZ_L| or NULL
  float* amax_out;         // atomicMax of |dZ_{L-1}|, or NULL
  float* scratch;          // with colsum: [ceil(n/16), 256] floats of 16-row column sums (may be a dead [n,256] tensor)
};
// Both GEMMs of the layer in one pass over dZ_L and H_{L-1} (bit 2 of g_debug_flags: the wgrad + launch pair).
int dgrad_wgrad(const BackwardLaunch* groups, int ngroups, int64_t n, cudaStream_t st);
// Weight packs (one launch for all matrices).  Forward pack: k-block kb (32 input features) = the [256 out x 32 k] tile
// in the K-major SWIZZLE_64B layout, hi (16 KB) then lo (16 KB).  Dgrad pack: k-block kb (32 OUTPUT features = the
// reduction index of dZ . W) = four [32 out x 64 in] SWIZZLE_128B groups, hi (16 KB) then lo (16 KB).  Both are what
// TMA tensor loads of the plain [256, K] fp16 copies produced in the first version - as 512 / 256 row requests of 64 /
// 128 bytes per k-block, which is what bounded the kernel (tools/gemm_role_probe.py: 884 clk per k-block waiting for the
// weight tile); packed, a k-block is one 32 KB bulk copy.
int split_weights(const SplitSpec* specs, int count, cudaStream_t st);
// Deterministic reductions: out[q][i] += sum_{s < nslab} part[q][s * stride + i] in slot order, for up to 8 segments q.
struct SlotSums {
  const float* part[8];
  float* out[8];
  int len[8];
  int count, nslab;
  int64_t stride;
};
int sum_slots(const SlotSums& s, cudaStream_t st);

}  // namespace tch
}  // namespace rb
