// The mask-count stage of the token-level losses (count_kernel and totals_kernel of token_loss.cu), shared with the
// critic loss (token_critic_loss.cu): both cut rows into kTokenSeg-token segments and use the front of a
// rb200_token_loss_workspace_bytes(bsz, L) workspace for the counts and its fixed partial slots.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rb {

constexpr int kTokenThreads = 256;
constexpr int kTokenPerThread = 4;
constexpr int kTokenSeg = kTokenThreads * kTokenPerThread;  // tokens per (segment, row) CTA
constexpr int kTokenSlots = 11;                             // fp64 partial slots per (segment, row)

struct TokenCounts {
  int64_t nseg;               // segments per row
  const long long* row_cnt;   // [bsz] mask count of each row
  const long long* total;     // mask count of the micro-batch
  double* partials;           // [bsz, nseg, kTokenSlots]
};

// Launches the two count kernels (2 launches) on `st` and returns where their results and the partials lie.
TokenCounts token_mask_counts(const uint8_t* mask, int64_t mask_stride, int64_t bsz, int64_t L, void* workspace,
                              cudaStream_t st);

}  // namespace rb
