// Forward GEMM of the MLP towers, C = tanh(A . W^T * scale + b) (or the plain product), for K % 32 == 0, K <= 256,
// up to two groups (towers) per launch, with the fp16-split arithmetic of tc_h_gemm_kernel<0> (tc_gemm_h.cu): the same
// operand scaling, the same split in registers (a_frag_rows), weights * 2^10 from the same forward pack, the same MMA
// order per accumulator (k ascending; lo.hi, hi.lo, hi.hi) and the same epilogue (acc * out_scale, + bias, tanh_fast).
//
// Why a second kernel: tc_h_gemm_kernel<0> streams the 32 KB weight tile of every k-block through its ring next to the
// 16 KB activation tile, so a 128 x 256 output tile pulls 256 KB of weights from L2 for 128 KB of activations, and both
// consumer warpgroups leave the tensor cores together for the epilogue.  Here
//   - a CTA owns one column half (128 output units) of one group, and its half of the weight pack (128 KB at K = 256)
//     stays resident in shared memory for the whole launch: the ring carries activations only;
//   - each of three consumer warpgroups owns whole 64-row tiles (m64n128k16, a 64-float accumulator) and they take
//     the CTA's tiles in turn, so one warpgroup's epilogue runs while the others' wgmmas keep the tensor cores busy;
//   - each consumer warpgroup has a ring of its own, fed by its own producer lane, and frees a slot as soon as the
//     wgmmas that read its A fragments are issued (the issue waits for the fragment registers, so the shared-memory
//     loads are done), not when they retire.
// One ring per warpgroup rather than one shared ring: a slot of a shared ring would alternate between the
// warpgroups' boxes, and a warpgroup that runs ahead could wait on a slot whose previous box (another warpgroup's)
// has not landed yet - the same parity as the phase it wants, so the wait would pass on stale data.
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_gemm.cuh"
#include "tc_half.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace rb {
namespace tch {

using rb::tc::BK;
using rb::tc::BN;

// Grid = CTA slot x group x column half, the half fastest: the two CTAs of a 64-row tile (four for layer 0, whose
// groups read the same X) are adjacent, run side by side, and the second read of the activation tile hits L2.
constexpr int kFwdRows = 64;                        // rows of a tile: one warpgroup's m64
constexpr int kFwdCols = BN / 2;                    // output units of a CTA
constexpr int kFwdBox = kFwdRows * BK * 4;          // 8 KB: fp32 [64 rows x 32 k] SWIZZLE_128B activation box
constexpr int kFwdW16 = kFwdCols * BK * 2;          // 8 KB: the CTA's half of a pack tile (hi or lo)
constexpr int kFwdWkb = 2 * kFwdW16;                // 16 KB per k-block: hi | lo
constexpr int kFwdWAll = (BN / BK) * kFwdWkb;       // 128 KB at K = 256
// Three consumer warpgroups (0-2; warpgroup 3 = producer): with two, the update's forward took 79.7 ms, with three
// 74.2 ms (DESIGN.md section 6).  Four do not fit: at 96 registers per thread ptxas serialises the wgmmas and spills.
constexpr int kFwdConsumers = 3;
constexpr int kFwdStages = 4;                       // per consumer warpgroup: 32 KB, half a tile at K = 256
constexpr int kFwdRingBytes = kFwdConsumers * kFwdStages * kFwdBox;  // 96 KB
constexpr int kFwdThreads = 128 * (kFwdConsumers + 1);
// Launched at 65536 / 512 = 128 registers per thread (__launch_bounds__(512, 1)); setmaxnreg.inc only gets what the
// producer warpgroup's setmaxnreg.dec gave back.  A consumer needs about 130.
constexpr int kFwdLaunchRegs = 65536 / kFwdThreads / 8 * 8;
constexpr int kFwdProducerRegs = 40, kFwdConsumerRegs = 152;
static_assert(128 * (kFwdLaunchRegs - kFwdProducerRegs) >= 128 * kFwdConsumers * (kFwdConsumerRegs - kFwdLaunchRegs),
              "register pool");

struct FwdBarriers {
  uint64_t full[kFwdConsumers][kFwdStages];   // activation box landed (tx bytes)
  uint64_t empty[kFwdConsumers][kFwdStages];  // the wgmmas reading its A fragments are issued (one arrival per warp)
  uint64_t w_full;             // resident weights (bulk-copy tx bytes)
  alignas(16) float bias[kFwdCols];
};

struct FwdGroup {
  const float* bias;     // [256], or NULL: C = the scaled product
  const float* amax_in;  // [1] max|A| of a gradient operand (scale_log2_for), or NULL
  const float* amax_x;   // [1] max|A| of an input operand (input_scale_log2_for), or NULL
  float* c;              // [M,256]
};

struct FwdParams {
  CUtensorMap a[2];          // [M,K] fp32, boxes [64 rows x 32 k] SWIZZLE_128B
  const uint8_t* wpack[2];   // forward packs (split_weights)
  FwdGroup g[2];
  int64_t M;
  int K, ngroups;
};

__global__ void __launch_bounds__(kFwdThreads, 1) tc_h_fwd_kernel(const __grid_constant__ FwdParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tma::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* wst = smem + kFwdRingBytes;
  FwdBarriers* bars = reinterpret_cast<FwdBarriers*>(wst + kFwdWAll);
  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = blockIdx.x & 1, grp = (blockIdx.x >> 1) % P.ngroups;
  const int cta = blockIdx.x / (2 * P.ngroups), n_cta = gridDim.x / (2 * P.ngroups);
  const FwdGroup& G = P.g[grp];
  const int64_t n_tiles = (P.M + kFwdRows - 1) / kFwdRows;
  const int n_kb = P.K / BK;

  if (threadIdx.x == 0) {
    for (int w = 0; w < kFwdConsumers; ++w)
      for (int s = 0; s < kFwdStages; ++s) {
        tma::mbar_init(&bars->full[w][s], 1);
        tma::mbar_init(&bars->empty[w][s], 4);
      }
    tma::mbar_init(&bars->w_full, 1);
    tma::fence_barrier_init();
  }
  for (int i = threadIdx.x; i < kFwdCols; i += kFwdThreads) bars->bias[i] = G.bias ? G.bias[half * kFwdCols + i] : 0.f;
  __syncthreads();

  // The CTA's j-th tile is cta + j n_cta, taken by consumer warpgroup j % kFwdConsumers; its k-block kb is box
  // (j / kFwdConsumers) n_kb + kb of that warpgroup's ring.
  if (wg == kFwdConsumers) {
    // ================= producer: lane 0 of warp 12 + w feeds the ring of consumer warpgroup w =================
    wg::setmaxnreg_dec<kFwdProducerRegs>();
    const int w = warp - 4 * kFwdConsumers;
    if (lane == 0 && w < kFwdConsumers) {
      tma::prefetch_desc(&P.a[grp]);
      if (w == 0) {
        // the CTA's half of every k-block of the pack: rows 128 half + [0, 128) of the hi tile and of the lo tile
        const uint8_t* wsrc = P.wpack[grp] + half * kFwdW16;
        tma::mbar_arrive_expect_tx(&bars->w_full, n_kb * kFwdWkb);
        for (int kb = 0; kb < n_kb; ++kb) {
          bulk_load(wst + kb * kFwdWkb, wsrc + (size_t)kb * 4 * kFwdW16, kFwdW16, &bars->w_full);
          bulk_load(wst + kb * kFwdWkb + kFwdW16, wsrc + (size_t)kb * 4 * kFwdW16 + 2 * kFwdW16, kFwdW16, &bars->w_full);
        }
      }
      uint8_t* ring = smem + w * kFwdStages * kFwdBox;
      uint32_t s = 0, ph = 0;
      for (int64_t tile = cta + (int64_t)w * n_cta; tile < n_tiles; tile += (int64_t)kFwdConsumers * n_cta) {
        for (int kb = 0; kb < n_kb; ++kb) {
          tma::mbar_wait(&bars->empty[w][s], ph ^ 1u);
          tma::mbar_arrive_expect_tx(&bars->full[w][s], kFwdBox);
          tma::load_2d(ring + s * kFwdBox, &P.a[grp], kb * BK, (int)(tile * kFwdRows), &bars->full[w][s]);  // rows >= M: 0
          if (++s == kFwdStages) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    // ================= consumers: whole 64-row tiles, in turn =================
    wg::setmaxnreg_inc<kFwdConsumerRegs>();
    const int g = lane >> 2, t = lane & 3;
    const int r_lo = (warp & 3) * 16 + g;  // this thread's tile rows r_lo and r_lo + 8
    const int sa = G.amax_in ? scale_log2_for(__ldg(G.amax_in)) : (G.amax_x ? input_scale_log2_for(__ldg(G.amax_x)) : 0);
    const float a_scale = pow2i(sa);
    const float out_scale = pow2i(-(sa + kWeightScaleLog2));
    const bool tanh_out = G.bias != nullptr;
    float* cbase = G.c + half * kFwdCols;
    const uint32_t w0 = tma::smem_u32(wst);
    const uint8_t* ring = smem + wg * kFwdStages * kFwdBox;
    uint64_t* full = bars->full[wg];
    uint64_t* empty = bars->empty[wg];
    // box q of the warpgroup's ring sits in stage q % kFwdStages, filled in phase q / kFwdStages
    auto load_a = [&](uint32_t q, uint32_t(&ah)[BK / 16][4], uint32_t(&al)[BK / 16][4]) {
      tma::mbar_wait_brk(&full[q % kFwdStages], (q / kFwdStages) & 1u);
      const uint8_t* st = ring + (q % kFwdStages) * kFwdBox;
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) a_frag_rows(st, r_lo, k * 16 + 2 * t, a_scale, ah[k], al[k]);
    };
    tma::mbar_wait_brk(&bars->w_full, 0u);
    for (int64_t j = wg;; j += kFwdConsumers) {
      const int64_t tile = cta + j * n_cta;
      if (tile >= n_tiles) break;
      const uint32_t q0 = (uint32_t)(j / kFwdConsumers) * n_kb;
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      // k-block kb's wgmmas are one group; once they are issued, its box is released (the issue waited for the
      // fragment registers, so every shared-memory load of the box has completed; an arrive placed right behind the
      // loads could overtake them).  While the group runs, the group of kb - 1 is retired (wait<1>) and the A rows of
      // kb + 1 are split into the fragment registers kb - 1 read.
      auto step = [&](int kb, const uint32_t(&ah)[BK / 16][4], const uint32_t(&al)[BK / 16][4],
                      uint32_t(&nh)[BK / 16][4], uint32_t(&nl)[BK / 16][4]) {
        const uint32_t wb = w0 + kb * kFwdWkb;
        wg::fence();  // the A fragments were written by ordinary instructions
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // K-major SW64 as in the pack, 128 rows of 64 B: the next 16 k are 32 B further along the rows
          const uint64_t b_hi = wg::desc(wb + k * 32, 16, 512, kSw64);
          const uint64_t b_lo = wg::desc(wb + kFwdW16 + k * 32, 16, 512, kSw64);
          wg::Mma<128, 0>::run(acc, al[k], b_hi, 1u);  // small terms first
          wg::Mma<128, 0>::run(acc, ah[k], b_lo, 1u);
          wg::Mma<128, 0>::run(acc, ah[k], b_hi, 1u);
        }
        wg::commit();
        warp_arrive(&empty[(q0 + kb) % kFwdStages]);
        wg::wait<1>();
        if (kb + 1 < n_kb) load_a(q0 + kb + 1, nh, nl);
      };
      uint32_t ah0[BK / 16][4], al0[BK / 16][4], ah1[BK / 16][4], al1[BK / 16][4];
      load_a(q0, ah0, al0);
      for (int kb = 0; kb < n_kb; kb += 2) {
        step(kb, ah0, al0, ah1, al1);
        if (kb + 1 < n_kb) step(kb + 1, ah1, al1, ah0, al0);
      }
      wg::wait<0>();
      wg::fence_operand(acc);
      // ---- epilogue straight from the accumulator registers: 8-byte stores, each quad of lanes writes 32 B of a row ----
      const int64_t row0 = tile * kFwdRows + r_lo, row1 = row0 + 8;
      const bool ok0 = row0 < P.M, ok1 = row1 < P.M;
#pragma unroll
      for (int jj = 0; jj < kFwdCols / 8; ++jj) {
        const int col = 8 * jj + 2 * t;
        float v0 = acc[4 * jj] * out_scale, v1 = acc[4 * jj + 1] * out_scale;
        float v2 = acc[4 * jj + 2] * out_scale, v3 = acc[4 * jj + 3] * out_scale;
        if (tanh_out) {
          const float2 b = *reinterpret_cast<const float2*>(&bars->bias[col]);
          v0 = tanh_fast(v0 + b.x); v1 = tanh_fast(v1 + b.y);
          v2 = tanh_fast(v2 + b.x); v3 = tanh_fast(v3 + b.y);
        }
        if (ok0) *reinterpret_cast<float2*>(cbase + row0 * BN + col) = make_float2(v0, v1);
        if (ok1) *reinterpret_cast<float2*>(cbase + row1 * BN + col) = make_float2(v2, v3);
      }
    }
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
int encode_f32_sw128(CUtensorMap* out, const float* base, uint64_t rows, uint64_t cols, uint32_t box_rows);

int forward(const GemmLaunch* L, int ngroups, int64_t M, int K, int epi, cudaStream_t st) {
  if (ngroups < 1 || ngroups > 2 || K % BK != 0 || K <= 0 || K > BN || M <= 0) return RB200_E_SHAPE;
  if (epi != rb::tc::EPI_STORE && epi != rb::tc::EPI_BIAS_TANH) return RB200_E_UNSUPPORTED;
  FwdParams P{};
  P.M = M; P.K = K; P.ngroups = ngroups;
  for (int g = 0; g < ngroups; ++g) {
    const GemmLaunch& l = L[g];
    const uintptr_t al = reinterpret_cast<uintptr_t>(l.a) | reinterpret_cast<uintptr_t>(l.b_hi) |
                         reinterpret_cast<uintptr_t>(l.c);
    if (al & 15) return RB200_E_ALIGN;
    if (epi == rb::tc::EPI_BIAS_TANH && !l.bias) return RB200_E_NULL;
    if (encode_f32_sw128(&P.a[g], l.a, (uint64_t)M, (uint64_t)K, kFwdRows)) return RB200_E_UNSUPPORTED;
    P.wpack[g] = reinterpret_cast<const uint8_t*>(l.b_hi);
    P.g[g] = FwdGroup{epi == rb::tc::EPI_BIAS_TANH ? l.bias : nullptr, l.amax_in, l.amax_x, l.c};
  }
  static bool attr_done = false;
  constexpr int kSmem = kFwdRingBytes + kFwdWAll + 1024 + (int)sizeof(FwdBarriers);
  static_assert(kSmem <= 232448, "tc_h_fwd_kernel shared memory");
  if (!attr_done) {
    const cudaError_t ce = cudaFuncSetAttribute(tc_h_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (ce != cudaSuccess) return (int)ce;
    attr_done = true;
  }
  // one CTA per SM: sm_count / (2 ngroups) CTA slots per (group, half), each taking every n_cta-th 64-row tile
  const int64_t n_tiles = (M + kFwdRows - 1) / kFwdRows;
  int n_cta = rb::sm_count() / (2 * ngroups);
  if (n_cta > n_tiles) n_cta = (int)n_tiles;
  if (n_cta < 1) n_cta = 1;
  tc_h_fwd_kernel<<<n_cta * ngroups * 2, kFwdThreads, kSmem, st>>>(P);
  rb::count_launch();
  const cudaError_t ce = cudaPeekAtLastError();
  return ce == cudaSuccess ? 0 : (int)ce;
}

}  // namespace tch
}  // namespace rb
