// Backward through a square hidden layer of the MLP towers in one pass over its inputs (fp16-split wgmma, fp32 in/out):
//     dW_L      += dZ_L^T . H_{L-1}                         (wgrad)
//     dZ_{L-1}   = (dZ_L . W_L) * (1 - H_{L-1}^2)           (dgrad, + column sums for the bias gradient, + max|dZ_{L-1}|)
// Both GEMMs read dZ_L and H_{L-1}; run as tc_h_wgrad_kernel + tc_h_gemm_kernel<1> they read both twice from HBM.
// Here every 32-sample k-block of dZ_L and H_{L-1} lands once per CTA, is split into fp16 (hi, lo) once, and feeds both.
// The arithmetic is that of the two kernels (same operand scaling, same split, same MMA order per accumulator: samples /
// features ascending, then lo.hi, hi.lo, hi.hi; same sample chunks), so dZ_{L-1}, max|dZ_{L-1}| and dW are bit-identical
// to theirs; only the column sums are added in another order.
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

// Grid = groups x 2 halves x sample chunks (the chunks of tc_h_wgrad_kernel).  The two CTAs of a chunk (adjacent in the
// grid, so they run side by side and the second read of dZ hits L2) split the work by columns of H: CTA `half` owns
//   dW[:, 128 half + 128)  - needs all of dZ and its 128 columns of H;
//   dZ_{L-1}[:, 128 half + 128) - needs all of dZ (the contraction index), the matching 128 columns of W_L, and the
//   same 128 columns of H for the 1 - h^2 factor.
// So a CTA reads dZ whole and only its half of H.  The dgrad is computed transposed, dZ_{L-1}^T[c, m] =
// sum_k W[k, c] dZ[m, k], so that its wgmma N is the 32 samples of a k-block and one k-block of split dZ serves as the
// dgrad's B (K-major) and the wgrad's A (MN-major) without a second copy.  The CTA's half of the dgrad pack (128 KB)
// stays resident in shared memory: streamed per k-block it is 128 KB of L2 reads per 48 KB of activations, and a
// ring small enough to fit next to the operand tiles leaves the wgmmas waiting on L2 latency.
// Warpgroups 0 / 1: consumers.  Consumer w owns dW rows [128 w, +128) (two m64n128 accumulators, 128 registers) and
// dZ_{L-1} columns 128 half + [64 w, +64) (one m64n32 accumulator per k-block, 16 registers; its epilogue runs behind
// the same k-block's wgrad wgmmas).  Warpgroup 2: warp 8 lane 0 issues the weight load and the TMA loads of the two
// stages; warps 9-11 split each landed fp32 box into fp16 (hi, lo) in place.  A stage is busy from its TMA until its
// wgmmas retire (the dgrad epilogue reads its H rows from global memory / L2, as tc_h_gemm_kernel<1> does), so with
// two stages the TMA and split of k-block i + 1 overlap the wgmmas of k-block i.
constexpr int kBwThreads = 384;
constexpr int kBwZ32 = BK * BN * 4;                       // 32 KB: dZ of a k-block, 8 boxes [32 samples x 32 features]
constexpr int kBwH32 = BK * 128 * 4;                      // 16 KB: the CTA's 128 columns of H, 4 boxes
constexpr int kBwStageBytes = kBwZ32 + kBwH32;            // 48 KB: 12 boxes of 4 KB, each fp32 as landed, then hi | lo
constexpr int kBwBox = 4096, kBwLo = 2048;                // box stride; lo half of a split box
constexpr int kBwW16 = BK * 128 * 2;                      // 8 KB: two 64-column groups of a dgrad-pack k-block, one half
constexpr int kBwWBytes = 2 * kBwW16;                     // 16 KB per k-block: hi | lo
constexpr int kBwWAll = (BN / BK) * kBwWBytes;            // 128 KB: the CTA's half of the whole pack
constexpr int kBwRingBytes = 2 * kBwStageBytes + kBwWAll;  // 2 x 48 + 128 KB
constexpr int kBwSplitThreads = 96;                       // warps 9-11
// Launched at 168 registers per thread (__launch_bounds__(384, 1)), the CTA can only raise the consumers by what the
// producers give back; setmaxnreg.inc waits until it can.  A split warp holds a whole box (32 words): 64 producer
// registers, so 216 for the consumers.
constexpr int kBwLaunchRegs = 65536 / kBwThreads / 8 * 8;
constexpr int kBwProducerRegs = 64, kBwConsumerRegs = 216;
static_assert(128 * (kBwLaunchRegs - kBwProducerRegs) >= 256 * (kBwConsumerRegs - kBwLaunchRegs), "register pool");
constexpr int64_t kBwSlot = 256 * 256;                    // per (chunk, group) partial of dW

struct BwBarriers {
  uint64_t full[2];      // stage landed: TMA tx bytes
  uint64_t op_full[2];   // stage split (one arrival per split thread, after its proxy fence)
  uint64_t op_empty[2];  // wgmmas reading the stage retired (one arrival per consumer warp)
  uint64_t w_full;       // resident weights: bulk-copy tx bytes
};

struct BwParams {
  CUtensorMap z[2], h[2];     // [n,256] fp32, boxes [32 samples x 32 columns] SWIZZLE_128B
  const float* hg[2];         // the same H (epilogue reads)
  const uint8_t* wpack[2];    // dgrad packs
  float* dzprev[2];
  float* p16[2];              // [ceil(n/16), 256] column sums of dZ_{L-1} over 16-row groups, or NULL
  const float* amax_in[2];
  float* amax_out[2];
  float* part;                // [chunk][group] slots of kBwSlot floats (summed in chunk order by sum_slots)
  int64_t n;
  int kb_per_chunk, ngroups;
};

__global__ void __launch_bounds__(kBwThreads, 1) tc_h_dgrad_wgrad_kernel(const __grid_constant__ BwParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tma::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* wst = smem + 2 * kBwStageBytes;
  BwBarriers* bars = reinterpret_cast<BwBarriers*>(smem + kBwRingBytes);
  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = blockIdx.x % P.ngroups;
  const int rest = blockIdx.x / P.ngroups;
  const int half = rest & 1, chunk = rest >> 1;
  const int n_kb_total = (int)((P.n + BK - 1) / BK);
  const int kb0 = chunk * P.kb_per_chunk;
  const int kb1 = (kb0 + P.kb_per_chunk < n_kb_total) ? kb0 + P.kb_per_chunk : n_kb_total;
  const int n_kb = kb1 - kb0;
  // dZ is scaled by 2^s before the split (s from its published max), the weights are stored * 2^kWeightScaleLog2
  const int s_z = P.amax_in[grp] ? scale_log2_for(__ldg(P.amax_in[grp])) : 0;

  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) {
      tma::mbar_init(&bars->full[s], 1);
      tma::mbar_init(&bars->op_full[s], kBwSplitThreads);
      tma::mbar_init(&bars->op_empty[s], 8);
    }
    tma::mbar_init(&bars->w_full, 1);
    tma::fence_barrier_init();
  }
  __syncthreads();
  if (n_kb <= 0) return;

  // k-block it uses stage it & 1, for the (it >> 1)-th time: its barriers complete phase it >> 1
  if (wg == 2) {
    wg::setmaxnreg_dec<kBwProducerRegs>();
    if (warp > 8) {  // split: warp 9 + w owns boxes w, w + 3, w + 6, w + 9 of a stage (dZ 0-7, H 8-11)
      const float z_scale = pow2i(s_z);
      for (int it = 0; it < n_kb; ++it) {
        uint8_t* st = smem + (it & 1) * kBwStageBytes;
        tma::mbar_wait(&bars->full[it & 1], (it >> 1) & 1u);
#pragma unroll 1
        for (int b = warp - 9; b < 12; b += 3) split_box_in_place(st + b * kBwBox, lane, b < BN / 32 ? z_scale : 1.0f);
        tma::fence_proxy_async();  // generic-proxy stores -> the wgmmas' async-proxy reads
        tma::mbar_arrive(&bars->op_full[it & 1]);
      }
    } else if (lane == 0) {  // warp 8: loads
      tma::prefetch_desc(&P.z[grp]);
      tma::prefetch_desc(&P.h[grp]);
      // the CTA's dgrad-pack groups 2 half, 2 half + 1 (output columns 128 half + [0, 128)) of every k-block, hi | lo
      const uint8_t* wsrc = P.wpack[grp] + half * 2 * 4096;
      tma::mbar_arrive_expect_tx(&bars->w_full, kBwWAll);
      for (int kb = 0; kb < BN / BK; ++kb) {
        bulk_load(wst + kb * kBwWBytes, wsrc + (size_t)kb * 32768, kBwW16, &bars->w_full);
        bulk_load(wst + kb * kBwWBytes + kBwW16, wsrc + (size_t)kb * 32768 + 16384, kBwW16, &bars->w_full);
      }
      for (int it = 0; it < n_kb; ++it) {
        uint8_t* st = smem + (it & 1) * kBwStageBytes;
        uint64_t* full = &bars->full[it & 1];
        tma::mbar_wait(&bars->op_empty[it & 1], ((it >> 1) & 1u) ^ 1u);  // wgmmas of k-block it - 2 retired
        tma::mbar_arrive_expect_tx(full, kBwStageBytes);
        const int m0 = (kb0 + it) * BK;  // samples >= n are zero-filled
        for (int b = 0; b < BN / 32; ++b) tma::load_2d(st + b * kBwBox, &P.z[grp], b * 32, m0, full);
        for (int b = 0; b < 4; ++b) tma::load_2d(st + kBwZ32 + b * kBwBox, &P.h[grp], half * 128 + b * 32, m0, full);
      }
    }
  } else {
    wg::setmaxnreg_inc<kBwConsumerRegs>();
    const int g = lane >> 2, t = lane & 3;
    const float wgrad_scale = pow2i(-s_z), dgrad_scale = pow2i(-(s_z + kWeightScaleLog2));
    const int c_lo = 64 * wg + 16 * (warp & 3) + g;  // this thread's dZ_{L-1} columns 128 half + c_lo (+ 8)
    const float* hg = P.hg[grp] + 128 * half;
    float* out = P.dzprev[grp] + 128 * half;
    float* p16 = P.p16[grp];
    const int64_t n16 = (P.n + 15) / 16;
    float accw[2][64];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int i = 0; i < 64; ++i) accw[mt][i] = 0.f;
    float vmax = 0.f;
    const uint32_t st0 = tma::smem_u32(smem), wb0 = tma::smem_u32(wst) + wg * 4096;
    // Per k-block, two commit groups: the dgrad wgmmas, then the wgrad wgmmas.  wait<1> retires the dgrad group, and
    // the dgrad epilogue runs while the wgrad group keeps the tensor cores busy; wait<0> then frees the stage.  Both
    // groups are drained before the next k-block: with an accumulator of an in-flight group live across the loop's
    // back-edge, ptxas (CUDA 12.9) serialises every wgmma of the kernel (C7514).
    tma::mbar_wait_brk(&bars->w_full, 0u);
    for (int it = 0; it < n_kb; ++it) {
      const int64_t m_base = (int64_t)(kb0 + it) * BK;
      float hv[16];  // the epilogue's H values from L2, loaded before the wgmmas to hide the latency
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int64_t row = m_base + 8 * (i >> 2) + 2 * t + (i & 1);
        hv[i] = row < P.n ? __ldg(hg + row * BN + c_lo + 8 * ((i >> 1) & 1)) : 0.f;
      }
      const uint32_t zb = st0 + (it & 1) * kBwStageBytes, hb = zb + kBwZ32;
      tma::mbar_wait_brk(&bars->op_full[it & 1], (it >> 1) & 1u);
      float accd[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) accd[i] = 0.f;
      wg::fence();
      // dgrad (transposed): A = W^T (this warpgroup's 64 output columns of weight k-block kb, MN-major SW128),
      // B = dZ (K-major: box kb holds features 32 kb + [0, 32) of the 32 samples, hi | lo)
#pragma unroll 1
      for (int kb = 0; kb < BN / BK; ++kb) {
        const uint32_t wb = wb0 + kb * kBwWBytes;
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t a_hi = wg::desc(wb + k * 2048, 4096, 1024, kSw128);
          const uint64_t a_lo = wg::desc(wb + kBwW16 + k * 2048, 4096, 1024, kSw128);
          const uint64_t b_hi = wg::desc(zb + kb * kBwBox + k * 32, 16, 512, kSw64);
          const uint64_t b_lo = wg::desc(zb + kb * kBwBox + kBwLo + k * 32, 16, 512, kSw64);
          wg::MmaSS<32, 1, 0>::run(accd, a_hi, b_lo, 1u);  // dZ lo . W hi first, as in the dgrad kernel
          wg::MmaSS<32, 1, 0>::run(accd, a_lo, b_hi, 1u);
          wg::MmaSS<32, 1, 0>::run(accd, a_hi, b_hi, 1u);
        }
      }
      wg::commit();
      // wgrad: A = dZ^T (features of this warpgroup, MN-major: 32-feature boxes 4 KB apart, 16 samples = 1 KB),
      // B = H (the CTA's 128 columns, MN-major)
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t b_hi = wg::desc(hb + k * 1024, kBwBox, 512, kSw64);
        const uint64_t b_lo = wg::desc(hb + kBwLo + k * 1024, kBwBox, 512, kSw64);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const uint32_t za = zb + (4 * wg + 2 * mt) * kBwBox + k * 1024;
          const uint64_t a_hi = wg::desc(za, kBwBox, 512, kSw64), a_lo = wg::desc(za + kBwLo, kBwBox, 512, kSw64);
          wg::MmaSS<128, 1, 1>::run(accw[mt], a_lo, b_hi, 1u);  // small terms first
          wg::MmaSS<128, 1, 1>::run(accw[mt], a_hi, b_lo, 1u);
          wg::MmaSS<128, 1, 1>::run(accw[mt], a_hi, b_hi, 1u);
        }
      }
      wg::commit();
      wg::wait<1>();
      wg::fence_operand(accd);
      // ---- dgrad epilogue: accd[4j + 2hh + e] = (column c_lo + 8 hh, sample 8j + 2t + e) ----
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int c = c_lo + 8 * hh;
        float v[4][2];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int64_t row = m_base + 8 * j + 2 * t + e;
            const bool ok = row < P.n;
            const float h = hv[4 * j + 2 * hh + e];
            float x = accd[4 * j + 2 * hh + e] * dgrad_scale;
            x = ok ? x * (1.0f - h * h) : 0.f;
            vmax = fmaxf(vmax, fabsf(x));
            if (ok) out[row * BN + c] = x;
            v[j][e] = x;
          }
        // column sums of the two 16-row groups in the reduction tree of tc_h_gemm_kernel<1>'s epilogue: row r + row
        // r + 8, then pairs of adjacent rows, then pairs of those (t ^ 1), then pairs of those (t ^ 2)
        if (p16 != nullptr) {
#pragma unroll
          for (int gi = 0; gi < 2; ++gi) {
            float p = (v[2 * gi][0] + v[2 * gi + 1][0]) + (v[2 * gi][1] + v[2 * gi + 1][1]);
            p += __shfl_xor_sync(0xffffffffu, p, 1);
            p += __shfl_xor_sync(0xffffffffu, p, 2);
            const int64_t grp16 = m_base / 16 + gi;
            if (t == 0 && grp16 < n16) p16[grp16 * BN + 128 * half + c] = p;
          }
        }
      }
      wg::wait<0>();
      warp_arrive(&bars->op_empty[it & 1]);
    }
    wg::fence_operand(accw[0]);
    wg::fence_operand(accw[1]);
    // ---- dW partial of the chunk (this CTA's columns) ----
    float* slot = P.part + (size_t)(chunk * P.ngroups + grp) * kBwSlot;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int f = 128 * wg + 64 * mt + 16 * (warp & 3) + g;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = 128 * half + 8 * j + 2 * t;
        *reinterpret_cast<float2*>(slot + (size_t)f * BN + col) =
            make_float2(accw[mt][4 * j] * wgrad_scale, accw[mt][4 * j + 1] * wgrad_scale);
        *reinterpret_cast<float2*>(slot + (size_t)(f + 8) * BN + col) =
            make_float2(accw[mt][4 * j + 2] * wgrad_scale, accw[mt][4 * j + 3] * wgrad_scale);
      }
    }
    if (P.amax_out[grp] != nullptr) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
      if (lane == 0 && vmax > 0.f) atomicMax(reinterpret_cast<unsigned int*>(P.amax_out[grp]), __float_as_uint(vmax));
    }
  }
}

// Column sums of dZ_{L-1} in the order of tc_h_gemm_kernel<1> + sum_slots, from the 16-row group sums: that kernel's
// CTA `cta` (of per_group) takes 128-row tiles cta, cta + per_group, ...; its consumer warp q adds the sum of rows
// [16 q, 16 q + 16) of each tile to its running sum in tile order; the CTA's slot is the sum of its 8 warps' running
// sums in warp order; sum_slots adds the slots in CTA order.  Block = (group, cta, column half), thread = (q, column).
struct ColsumOrderArgs {
  const float* p16[2];
  float* part;  // [per_group][ngroups][256]
  int64_t n16, n_tiles;
  int per_group, ngroups;
};
__global__ void __launch_bounds__(1024) colsum_order_kernel(const ColsumOrderArgs a) {
  __shared__ float red[8][128];
  const int h = blockIdx.x & 1, slot = blockIdx.x >> 1;  // slot = cta * ngroups + grp
  const int grp = slot % a.ngroups, cta = slot / a.ngroups;
  const int q = threadIdx.x >> 7, cl = threadIdx.x & 127, col = 128 * h + cl;
  const float* p = (grp ? a.p16[1] : a.p16[0]) + col;
  float acc = 0.f;
  for (int64_t tile = cta; tile < a.n_tiles; tile += a.per_group) {
    const int64_t g16 = tile * 8 + q;
    if (g16 < a.n16) acc += __ldg(p + g16 * BN);  // groups past the last row add 0 there
  }
  red[q][cl] = acc;
  __syncthreads();
  if (q == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w][cl];
    a.part[(size_t)slot * BN + col] = s;
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
int encode_f32_sw128(CUtensorMap* out, const float* base, uint64_t rows, uint64_t cols, uint32_t box_rows);

static int dgrad_wgrad_fused(const BackwardLaunch* L, int ngroups, int64_t n, cudaStream_t st) {
  BwParams P{};
  P.n = n; P.ngroups = ngroups;
  for (int g = 0; g < ngroups; ++g) {
    const uintptr_t al = reinterpret_cast<uintptr_t>(L[g].z) | reinterpret_cast<uintptr_t>(L[g].h) |
                         reinterpret_cast<uintptr_t>(L[g].wpack) | reinterpret_cast<uintptr_t>(L[g].dzprev) |
                         reinterpret_cast<uintptr_t>(L[g].dW);
    if (al & 15) return RB200_E_ALIGN;
    if (L[g].colsum && !L[g].scratch) return RB200_E_NULL;
    int e = encode_f32_sw128(&P.z[g], L[g].z, (uint64_t)n, BN, 32);
    if (!e) e = encode_f32_sw128(&P.h[g], L[g].h, (uint64_t)n, BN, 32);
    if (e) return RB200_E_UNSUPPORTED;
    P.hg[g] = L[g].h;
    P.wpack[g] = reinterpret_cast<const uint8_t*>(L[g].wpack);
    P.dzprev[g] = L[g].dzprev;
    P.p16[g] = L[g].colsum ? L[g].scratch : nullptr;
    P.amax_in[g] = L[g].amax_in;
    P.amax_out[g] = L[g].amax_out;
  }
  static bool attr_done = false;
  constexpr int kSmem = kBwRingBytes + 1024 + (int)sizeof(BwBarriers);
  static_assert(kSmem <= 232448, "tc_h_dgrad_wgrad_kernel shared memory");
  if (!attr_done) {
    const cudaError_t ce = cudaFuncSetAttribute(tc_h_dgrad_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (ce != cudaSuccess) return (int)ce;
    attr_done = true;
  }
  // the sample chunks of wgrad(): dW is summed over the same chunks in the same order
  const int n_kb = (int)((n + BK - 1) / BK);
  int chunks = rb::sm_count() / (2 * ngroups);
  if (chunks < 1) chunks = 1;
  if (chunks > n_kb) chunks = n_kb;
  P.kb_per_chunk = (n_kb + chunks - 1) / chunks;
  chunks = (n_kb + P.kb_per_chunk - 1) / P.kb_per_chunk;  // every chunk non-empty: each writes its slot
  // the CTA count of launch() for this shape: the column sums are added in its order
  const int64_t n_tiles = (n + rb::tc::BM - 1) / rb::tc::BM;
  int per_group = rb::sm_count() / ngroups;
  if (per_group > n_tiles) per_group = (int)n_tiles;
  if (per_group < 1) per_group = 1;
  const int64_t dw_floats = (int64_t)chunks * ngroups * kBwSlot;
  if (!(P.part = rb::partials_scratch(dw_floats + (int64_t)per_group * ngroups * BN))) return RB200_E_UNSUPPORTED;
  tc_h_dgrad_wgrad_kernel<<<ngroups * 2 * chunks, kBwThreads, kSmem, st>>>(P);
  rb::count_launch();
  cudaError_t ce = cudaPeekAtLastError();
  if (ce != cudaSuccess) return (int)ce;
  rb::tch::SlotSums ss{};
  ss.count = ngroups;
  ss.nslab = chunks;
  ss.stride = ngroups * kBwSlot;
  for (int g = 0; g < ngroups; ++g) {
    ss.part[g] = P.part + g * kBwSlot;
    ss.out[g] = L[g].dW;
    ss.len[g] = (int)kBwSlot;
  }
  int e = rb::tch::sum_slots(ss, st);
  if (e) return e;
  ColsumOrderArgs ca{};
  rb::tch::SlotSums cs{};
  ca.part = P.part + dw_floats;
  ca.n16 = (n + 15) / 16;
  ca.n_tiles = n_tiles;
  ca.per_group = per_group;
  ca.ngroups = ngroups;
  cs.nslab = per_group;
  cs.stride = (int64_t)ngroups * BN;
  for (int g = 0; g < ngroups; ++g) {
    ca.p16[g] = P.p16[g] ? P.p16[g] : P.p16[0];
    if (L[g].colsum) {
      cs.part[cs.count] = ca.part + g * BN;
      cs.out[cs.count] = L[g].colsum;
      cs.len[cs.count++] = BN;
    }
  }
  if (!cs.count) return 0;
  // a group without column sums has its slots computed from another group's data and never read
  colsum_order_kernel<<<per_group * ngroups * 2, 1024, 0, st>>>(ca);
  rb::count_launch();
  ce = cudaPeekAtLastError();
  if (ce != cudaSuccess) return (int)ce;
  return rb::tch::sum_slots(cs, st);
}

int dgrad_wgrad(const BackwardLaunch* L, int ngroups, int64_t n, cudaStream_t st) {
  if (ngroups < 1 || ngroups > 2 || n <= 0) return RB200_E_SHAPE;
  for (int g = 0; g < ngroups; ++g)
    if (!L[g].z || !L[g].wpack || !L[g].h || !L[g].dzprev || !L[g].dW) return RB200_E_NULL;
  if (!(rb::tc::g_debug_flags & 4)) return dgrad_wgrad_fused(L, ngroups, n, st);
  WgradLaunch w[2];
  GemmLaunch d[2];
  for (int g = 0; g < ngroups; ++g) {
    w[g] = WgradLaunch{L[g].z, L[g].h, L[g].dW, L[g].amax_in};
    d[g] = GemmLaunch{L[g].z, L[g].wpack, L[g].dzprev, nullptr, L[g].h, L[g].colsum, L[g].amax_in, L[g].amax_out};
  }
  int e = wgrad(w, ngroups, n, BN, st);
  return e ? e : launch(d, ngroups, n, BN, rb::tc::EPI_TANHGRAD, 1, st);
}

}  // namespace tch
}  // namespace rb

// ---- unit-test entry (tests/test_gpu_tc_backward_fused.py) ------------------------------------------------------------
// ngroups (1 or 2) towers stacked along the first dimension: Z, H, dZprev [ngroups, n, 256], W, dW [ngroups, 256, 256],
// colsum [ngroups, 256] (nullable), amax_in / amax_out [ngroups] (nullable).
// work: >= ngroups * (131072 + 256 * ceil(n / 16)) floats.
extern "C" int rb200_tc_dgrad_wgrad_h(const float* Z, const float* W, const float* H, float* dZprev, float* dW,
                                      float* colsum, const float* amax_in, float* amax_out, int64_t n, int ngroups,
                                      float* work, rb200_stream_t stream) {
  if (!Z || !W || !H || !dZprev || !dW || !work) return RB200_E_NULL;
  if (n <= 0 || ngroups < 1 || ngroups > 2) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  constexpr int64_t kW = 256 * 256;
  const int64_t n16 = (n + 15) / 16 * 256;
  rb::tch::SplitSpec sp[2];
  rb::tch::BackwardLaunch l[2];
  for (int g = 0; g < ngroups; ++g) {
    // forward pack (always written by split_weights), then the dgrad pack
    sp[g] = rb::tch::SplitSpec{W + g * kW, work + 2 * g * kW, work + (2 * g + 1) * kW, kW};
    l[g] = rb::tch::BackwardLaunch{Z + g * n * 256, sp[g].lo, H + g * n * 256, dZprev + g * n * 256, dW + g * kW,
                                   colsum ? colsum + g * 256 : nullptr, amax_in ? amax_in + g : nullptr,
                                   amax_out ? amax_out + g : nullptr, work + 2 * ngroups * kW + g * n16};
  }
  int e = rb::tch::split_weights(sp, ngroups, st);
  return e ? e : rb::tch::dgrad_wgrad(l, ngroups, n, st);
}
