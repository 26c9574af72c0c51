// fp32-accurate GEMMs of the MLP towers on Hopper wgmma (fp16 inputs, fp32 accumulators) through a 2-way fp16 split.
//     a = a_hi + a_lo, b = b_hi + b_lo (fp16 numbers, 11 significant bits each; operands pre-scaled by a power of two so
//     that both halves stay in fp16's normal range);  a.b ~= a_lo.b_hi + a_hi.b_lo + a_hi.b_hi   (dropped a_lo.b_lo ~ 2^-22)
// Weights come as pre-swizzled fp16 (hi | lo) packs per k-block; activations stay plain fp32 in HBM and are split in
// registers; one launch serves both towers.
// Gradients are tiny (1e-6 .. 1e-10): their producer publishes max|x| and the consumer scales by 2^s (exact) so that the
// maximum sits at 2^13; the fp32 accumulator is scaled back in the epilogue (exact).
// Reference op chains replaced: nn.Linear + tanh of MLPPolicy.backbone / ValueHead.mlp
// (rlinf/models/embodiment/mlp_policy/mlp_policy.py:91-98, modules/value_head.py:37-45) and autograd's dgrad / wgrad.
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_gemm.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace rb {
namespace tch {

using rb::tc::BK;
using rb::tc::BM;
using rb::tc::BN;

// Forward / dgrad kernel (persistent, one CTA per SM): a producer warp fills a ring of stages (fp32 landing tile of the
// streamed operand, [128 rows x 32 k] TMA SWIZZLE_128B, + the packed weight tile of the k-block, one 32 KB bulk copy);
// warpgroups 0 / 1 own rows 0-63 / 64-127 of the 128 x 256 output tile, split their fp32 rows into fp16 hi / lo wgmma A
// fragments in registers and keep the fp32 accumulator in registers through the epilogue.
constexpr int kStages = 4;
constexpr int kA32 = BM * BK * 4;              // 16 KB fp32 landing tile of the streamed operand
constexpr int kB16 = BN * BK * 2;              // 16 KB per fp16 half of the weight tile
constexpr int kWBytes = 2 * kB16;              // 32 KB: W hi | W lo
constexpr int kStageBytes = kA32 + kWBytes;    // 48 KB
constexpr int kRingBytes = kStages * kStageBytes;  // 192 KB
constexpr int kThreads = 288;  // the block is resourced as three whole warpgroups: 168 registers per thread (a larger
                               // register count fails to launch), so ptxas serialises the six wgmmas of a k-block
constexpr int kWeightScaleLog2 = 10;  // weights are stored as fp16 (hi, lo) of w * 2^10 (|w| <~ 1: both halves normal)

// 1-D bulk copy global -> shared, completion counted on an mbarrier
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   tma::smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(tma::smem_u32(bar))
               : "memory");
}
// barrier over the 256 consumer threads only (the producer warp runs ahead)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Operand layouts: K-major SWIZZLE_64B (forward pack: 64-B rows, SBO 512), MN-major SWIZZLE_128B (dgrad pack: SBO 1024 B
// between 8 K-rows, LBO 4096 B between 64-wide N groups), MN-major SWIZZLE_64B (wgrad H: SBO 512, LBO 2048).
constexpr uint32_t kSw128 = 1, kSw64 = 2;

__device__ __forceinline__ float tanh_fast(float x) {
  const float t = __expf(-2.0f * fabsf(x));
  return copysignf(__fdividef(1.0f - t, 1.0f + t), x);
}

// 2^s as a float (s in [-126, 127])
__device__ __forceinline__ float pow2i(int s) { return __int_as_float((s + 127) << 23); }
// power-of-two scale that brings max|x| = amax to [2^13, 2^14): fp16 keeps 11 bits for every |x| >= amax * 2^-27
__device__ __forceinline__ int scale_log2_for(float amax) {
  const int e = (int)((__float_as_uint(amax) >> 23) & 0xffu) - 127;
  if (!(amax > 0.0f) || e < -120) return 0;
  int s = 13 - e;
  return s > 100 ? 100 : (s < -100 ? -100 : s);
}

// (x0, x1) -> packed fp16 pairs hi = rn(x), lo = rn(x - hi)
__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 hh = __floats2half2_rn(x0, x1);
  const float2 hf = __half22float2(hh);
  const __half2 ll = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&hh);
  lo = *reinterpret_cast<const uint32_t*>(&ll);
}

// fp32 [R rows x 32 floats] SWIZZLE_128B tile -> fp16 hi / lo [R rows x 32 halfs] SWIZZLE_64B tiles; item = (row, 8 floats)
template <int NT>
__device__ __forceinline__ void split_tile(const uint8_t* __restrict__ src, uint8_t* __restrict__ hi, uint8_t* __restrict__ lo,
                                           int rows, int t, float scale) {
  const int items = rows * 4;
#pragma unroll 2
  for (int i = t; i < items; i += NT) {
    const int r = i >> 2, cp = i & 3;
    const uint8_t* srow = src + r * 128;
    const float4 x0 = *reinterpret_cast<const float4*>(srow + (((2 * cp) ^ (r & 7)) << 4));
    const float4 x1 = *reinterpret_cast<const float4*>(srow + (((2 * cp + 1) ^ (r & 7)) << 4));
    const float v[8] = {x0.x * scale, x0.y * scale, x0.z * scale, x0.w * scale,
                        x1.x * scale, x1.y * scale, x1.z * scale, x1.w * scale};
    uint32_t h[4], l[4];  // packed half2 words (no 16-byte reinterpretation of a 4-byte-aligned local array)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 hh = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
      const float2 hf = __half22float2(hh);
      const __half2 ll = __floats2half2_rn(v[2 * j] - hf.x, v[2 * j + 1] - hf.y);
      h[j] = *reinterpret_cast<const uint32_t*>(&hh);
      l[j] = *reinterpret_cast<const uint32_t*>(&ll);
    }
    const int doff = r * 64 + ((cp ^ ((r >> 1) & 3)) << 4);
    *reinterpret_cast<uint4*>(hi + doff) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(lo + doff) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

// wgmma A fragment (m64k16, this thread's rows r0 / r0 + 8, k columns c0 + 2t + {0, 1, 8, 9}) of a row-major fp32
// [rows x 32] SWIZZLE_128B landing tile, scaled and split into fp16 hi / lo
__device__ __forceinline__ void a_frag_rows(const uint8_t* tile, int r0, int c0, float scale, uint32_t (&hi)[4],
                                            uint32_t (&lo)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + (i & 1) * 8, c = c0 + (i >> 1) * 8;
    const float2 x = *reinterpret_cast<const float2*>(tile + r * 128 + ((((c >> 2) ^ (r & 7))) << 4) + (c & 3) * 4);
    split2(x.x * scale, x.y * scale, hi[i], lo[i]);
  }
}

struct __align__(16) Barriers {
  uint64_t full[kStages];   // landing tile + weight tile arrived (tx bytes)
  uint64_t empty[kStages];  // both consumer warpgroups' wgmmas reading the stage have completed (one arrival per warp)
  alignas(16) float bias[BN];  // forward: the layer bias
  float csum[8][BN];           // dgrad: column sums of the output per consumer warp (one writer per slot: deterministic)
};

struct Group {
  const float* bias;    // [256]                         (EPI_BIAS_TANH)
  const float* h;       // [M,256] previous activation   (EPI_TANHGRAD)
  float* colsum;        // [256] += column sums of the output, or NULL
  const float* amax_in; // [1] max|A| published by A's producer (gradient GEMMs), or NULL = no scaling
  float* amax_out;      // [1] atomicMax of |output| for the next gradient GEMM, or NULL
  float* c;             // [M,256] output
};

struct GemmParams {
  CUtensorMap a[2];
  const uint8_t* wpack[2];  // packed weight tiles of each group (32 KB per k-block: hi | lo)
  Group g[2];
  float* part;  // [gridDim.x][256] per-CTA column sums (summed in CTA order by sum_slots)
  int64_t M;
  int K;
  int epi;
  int ngroups;
};

template <int B_MN>
__global__ void __launch_bounds__(kThreads, 1) tc_h_gemm_kernel(const __grid_constant__ GemmParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tma::smem_u32(smem_raw) & 1023u)) & 1023u);
  Barriers* bars = reinterpret_cast<Barriers*>(smem + kRingBytes);

  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = blockIdx.x % P.ngroups;
  const int cta = blockIdx.x / P.ngroups, n_cta = gridDim.x / P.ngroups;
  const Group& G = P.g[grp];
  const int64_t n_tiles = (P.M + BM - 1) / BM;
  const int n_kb = P.K / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      tma::mbar_init(&bars->full[s], 1);
      tma::mbar_init(&bars->empty[s], 8);
    }
    tma::fence_barrier_init();
  }
  for (int i = threadIdx.x; i < BN; i += kThreads) bars->bias[i] = (P.epi == rb::tc::EPI_BIAS_TANH) ? G.bias[i] : 0.f;
  for (int i = threadIdx.x; i < 8 * BN; i += kThreads) bars->csum[i / BN][i % BN] = 0.f;
  __syncthreads();

  if (wg == 2) {
    // ================= producer =================
    if (threadIdx.x == 256) {
      tma::prefetch_desc(&P.a[grp]);
      uint32_t s = 0, ph = 0;
      for (int64_t tile = cta; tile < n_tiles; tile += n_cta) {
        for (int kb = 0; kb < n_kb; ++kb) {
          tma::mbar_wait(&bars->empty[s], ph ^ 1u);
          uint8_t* st = smem + s * kStageBytes;
          tma::mbar_arrive_expect_tx(&bars->full[s], kStageBytes);
          tma::load_2d(st, &P.a[grp], kb * BK, (int)(tile * BM), &bars->full[s]);  // rows >= M are zero-filled
          bulk_load(st + kA32, P.wpack[grp] + (size_t)kb * kWBytes, kWBytes, &bars->full[s]);  // hi | lo
          if (++s == kStages) { s = 0; ph ^= 1u; }
        }
      }
    }
  } else {
    // ================= consumers: 64 rows each =================
    const int cw = wg;
    const int g = lane >> 2, t = lane & 3;
    const int r_lo = cw * 64 + (warp & 3) * 16 + g;  // this thread's tile rows r_lo and r_lo + 8
    // operand scaling: A by 2^sa (from the published amax), weights are stored * 2^kWeightScaleLog2
    const int sa = G.amax_in ? scale_log2_for(__ldg(G.amax_in)) : 0;
    const float a_scale = pow2i(sa);
    const float out_scale = pow2i(-(sa + kWeightScaleLog2));
    float vmax = 0.f;
    uint32_t s = 0, ph = 0;
    for (int64_t tile = cta; tile < n_tiles; tile += n_cta) {
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      for (int kb = 0; kb < n_kb; ++kb) {
        tma::mbar_wait(&bars->full[s], ph);
        const uint8_t* st = smem + s * kStageBytes;
        const uint32_t wbase = tma::smem_u32(st + kA32);
        uint32_t ah[BK / 16][4], al[BK / 16][4];
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) a_frag_rows(st, r_lo, k * 16 + 2 * t, a_scale, ah[k], al[k]);
        wg::fence();  // the A fragments were written by ordinary instructions
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // forward: K-major SW64, the next 16 k are 32 B further along the 64-B rows; dgrad: MN-major SW128, 16 K-rows of 128 B
          const uint64_t b_hi = B_MN ? wg::desc(wbase + k * 2048, 4096, 1024, kSw128) : wg::desc(wbase + k * 32, 16, 512, kSw64);
          const uint64_t b_lo = B_MN ? wg::desc(wbase + kB16 + k * 2048, 4096, 1024, kSw128)
                                     : wg::desc(wbase + kB16 + k * 32, 16, 512, kSw64);
          wg::Mma<256, B_MN>::run(acc, al[k], b_hi, 1u);  // small terms first
          wg::Mma<256, B_MN>::run(acc, ah[k], b_lo, 1u);
          wg::Mma<256, B_MN>::run(acc, ah[k], b_hi, 1u);
        }
        wg::commit();
        wg::wait<0>();
        __syncwarp();
        if (lane == 0) tma::mbar_arrive(&bars->empty[s]);
        if (++s == kStages) { s = 0; ph ^= 1u; }
      }
      // ---- epilogue straight from the accumulator registers: 8-byte stores, each quad of lanes writes 32 B of a row ----
      const int64_t row0 = tile * BM + r_lo, row1 = row0 + 8;
      const bool ok0 = row0 < P.M, ok1 = row1 < P.M;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = 8 * j + 2 * t;
        float v0 = acc[4 * j] * out_scale, v1 = acc[4 * j + 1] * out_scale;
        float v2 = acc[4 * j + 2] * out_scale, v3 = acc[4 * j + 3] * out_scale;
        if (P.epi == rb::tc::EPI_BIAS_TANH) {
          const float2 b = *reinterpret_cast<const float2*>(&bars->bias[col]);
          v0 = tanh_fast(v0 + b.x); v1 = tanh_fast(v1 + b.y);
          v2 = tanh_fast(v2 + b.x); v3 = tanh_fast(v3 + b.y);
        } else if (P.epi == rb::tc::EPI_TANHGRAD) {
          const float2 h0 = ok0 ? __ldg(reinterpret_cast<const float2*>(G.h + row0 * BN + col)) : make_float2(0.f, 0.f);
          const float2 h1 = ok1 ? __ldg(reinterpret_cast<const float2*>(G.h + row1 * BN + col)) : make_float2(0.f, 0.f);
          v0 = ok0 ? v0 * (1.0f - h0.x * h0.x) : 0.f; v1 = ok0 ? v1 * (1.0f - h0.y * h0.y) : 0.f;
          v2 = ok1 ? v2 * (1.0f - h1.x * h1.x) : 0.f; v3 = ok1 ? v3 * (1.0f - h1.y * h1.y) : 0.f;
          vmax = fmaxf(vmax, fmaxf(fmaxf(fabsf(v0), fabsf(v1)), fmaxf(fabsf(v2), fabsf(v3))));
          if (G.colsum != nullptr) {
            float c0 = v0 + v2, c1 = v1 + v3;
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
              c0 += __shfl_xor_sync(0xffffffffu, c0, o);
              c1 += __shfl_xor_sync(0xffffffffu, c1, o);
            }
            if (g == 0) {
              bars->csum[warp][col] += c0;
              bars->csum[warp][col + 1] += c1;
            }
          }
        }
        if (ok0) *reinterpret_cast<float2*>(G.c + row0 * BN + col) = make_float2(v0, v1);
        if (ok1) *reinterpret_cast<float2*>(G.c + row1 * BN + col) = make_float2(v2, v3);
      }
    }
    if (G.amax_out != nullptr && P.epi == rb::tc::EPI_TANHGRAD) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
      if (lane == 0 && vmax > 0.f) atomicMax(reinterpret_cast<unsigned int*>(G.amax_out), __float_as_uint(vmax));
    }
  }
  __syncthreads();
  if (P.part != nullptr)
    for (int i = threadIdx.x; i < BN; i += kThreads) {
      float s = 0.f;
      for (int w = 0; w < 8; ++w) s += bars->csum[w][i];
      P.part[(size_t)blockIdx.x * BN + i] = s;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Weight-gradient GEMM:  dW[256, IN] += sum_m dZ[m, :]^T . H[m, :]     (IN % 32 == 0, <= 256); the reduction index m
// (sample) is the strided one for both operands.  Grid = ngroups x 2 output tiles (128 rows of dW) x sample chunks;
// each CTA writes its chunk's partial to a slot, the slots are summed in chunk order.  dZ^T fragments go straight into
// registers, H is split into fp16 MN-major tiles (two operand slots).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kWgLand = 3;
constexpr int kWgA32 = 128 * BK * 4;                          // 16 KB of dZ
constexpr int kWgB32 = 256 * BK * 4, kWgB16 = 256 * BK * 2;   // 32 KB / 16 KB of H (sized for IN = 256)
constexpr int kWgLandBytes = kWgA32 + kWgB32;                 // 48 KB
constexpr int kWgOpBytes = 2 * kWgB16;                        // 32 KB: H hi | H lo
constexpr int kWgRingBytes = kWgLand * kWgLandBytes + 2 * kWgOpBytes;  // 144 + 64 KB

struct WgBarriers {
  uint64_t full[kWgLand], empty[kWgLand];  // landing ring: TMA tx bytes / consumers done reading (one arrival per warp)
};

struct WgradParams {
  CUtensorMap z[2], h[2];
  float* dW[2];
  float* part;             // [chunk][group][256 x IN] per-CTA partials of dW (summed in chunk order by sum_slots)
  const float* amax_z[2];  // max|dZ| per group (or NULL)
  int64_t n;
  int IN, kb_per_chunk, ngroups;
};

template <int NW>  // wgmma N: 128 or 256 (columns >= IN are computed on padding and dropped)
__global__ void __launch_bounds__(kThreads, 1) tc_h_wgrad_kernel(const __grid_constant__ WgradParams P) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tma::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* op = smem + kWgLand * kWgLandBytes;  // 2 x (H hi | H lo)
  WgBarriers* bars = reinterpret_cast<WgBarriers*>(smem + kWgRingBytes);
  const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = blockIdx.x % P.ngroups;
  const int rest = blockIdx.x / P.ngroups;
  const int out_tile = rest & 1, chunk = rest >> 1;
  const int IN = P.IN;
  const int n_kb_total = (int)((P.n + BK - 1) / BK);
  const int kb0 = chunk * P.kb_per_chunk;
  const int kb1 = (kb0 + P.kb_per_chunk < n_kb_total) ? kb0 + P.kb_per_chunk : n_kb_total;
  const int n_kb = kb1 - kb0;
  const uint32_t b32_bytes = (uint32_t)IN * BK * 4;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kWgLand; ++s) {
      tma::mbar_init(&bars->full[s], 1);
      tma::mbar_init(&bars->empty[s], 8);
    }
    tma::fence_barrier_init();
  }
  __syncthreads();
  if (n_kb <= 0) return;

  if (wg == 2) {
    {  // producer warp
      const int n_box = 4 + IN / 32;
      for (int it = 0; it < n_kb; ++it) {
        const int s = it % kWgLand;
        const uint32_t ph = (it / kWgLand) & 1u;
        if (lane == 0) {
          tma::mbar_wait(&bars->empty[s], ph ^ 1u);
          tma::mbar_arrive_expect_tx(&bars->full[s], kWgA32 + b32_bytes);
        }
        __syncwarp();
        if (lane < n_box) {
          uint8_t* st = smem + s * kWgLandBytes;
          const int m0 = (kb0 + it) * BK;  // samples >= n are zero-filled
          if (lane < 4) tma::load_2d(st + lane * 4096, &P.z[grp], out_tile * 128 + lane * 32, m0, &bars->full[s]);
          else tma::load_2d(st + kWgA32 + (lane - 4) * 4096, &P.h[grp], (lane - 4) * 32, m0, &bars->full[s]);
        }
      }
    }
  } else {
    const int cw = wg;
    const int g = lane >> 2, t = lane & 3;
    const int f_lo = cw * 64 + (warp & 3) * 16 + g;  // this thread's rows of the dW tile: f_lo and f_lo + 8
    const int sz = P.amax_z[grp] ? scale_log2_for(__ldg(P.amax_z[grp])) : 0;
    const float z_scale = pow2i(sz), out_scale = pow2i(-sz);
    float acc[NW / 2];
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[i] = 0.f;
    for (int it = 0; it < n_kb; ++it) {
      const int s = it % kWgLand;
      const uint32_t ph = (it / kWgLand) & 1u;
      tma::mbar_wait(&bars->full[s], ph);
      const uint8_t* st = smem + s * kWgLandBytes;
      uint8_t* hop = op + (it & 1) * kWgOpBytes;
      // H groups of [32 samples x 32 floats] (4 KB) -> [32 samples x 32 halfs] (2 KB), contiguous on both sides.  The slot
      // was last read by the wgmmas of k-block it - 2, which every consumer thread waited for before the barrier of it - 1.
      split_tile<256>(st + kWgA32, hop, hop + kWgB16, (IN / 32) * 32, threadIdx.x, 1.0f);
      tma::fence_proxy_async();
      consumer_sync();
      const uint32_t hb = tma::smem_u32(hop);
      // dZ^T fragments: A(m = feature f, k = sample) = dZ box f / 32 at (sample, f % 32)
      uint32_t ah[BK / 16][4], al[BK / 16][4];
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int f = f_lo + (i & 1) * 8, m = k * 16 + 2 * t + (i >> 1) * 8;
          const uint8_t* box = st + (f >> 5) * 4096;
          const int fc = f & 31;
          const float x0 = *reinterpret_cast<const float*>(box + m * 128 + (((fc >> 2) ^ (m & 7)) << 4) + (fc & 3) * 4);
          const float x1 =
              *reinterpret_cast<const float*>(box + (m + 1) * 128 + (((fc >> 2) ^ ((m + 1) & 7)) << 4) + (fc & 3) * 4);
          split2(x0 * z_scale, x1 * z_scale, ah[k][i], al[k][i]);
        }
      }
      wg::fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint64_t b_hi = wg::desc(hb + k * 1024, 2048, 512, kSw64);  // next 16 samples = two 8-sample atoms
        const uint64_t b_lo = wg::desc(hb + kWgB16 + k * 1024, 2048, 512, kSw64);
        wg::Mma<NW, 1>::run(acc, al[k], b_hi, 1u);
        wg::Mma<NW, 1>::run(acc, ah[k], b_lo, 1u);
        wg::Mma<NW, 1>::run(acc, ah[k], b_hi, 1u);
      }
      wg::commit();
      wg::wait<0>();
      __syncwarp();
      if (lane == 0) tma::mbar_arrive(&bars->empty[s]);
    }
    float* slot = P.part + (size_t)(chunk * P.ngroups + grp) * 256 * IN;
    const int row0 = out_tile * 128 + f_lo;
#pragma unroll
    for (int j = 0; j < NW / 8; ++j) {
      const int col = 8 * j + 2 * t;
      if (col < IN) {
        *reinterpret_cast<float2*>(slot + (size_t)row0 * IN + col) =
            make_float2(acc[4 * j] * out_scale, acc[4 * j + 1] * out_scale);
        *reinterpret_cast<float2*>(slot + (size_t)(row0 + 8) * IN + col) =
            make_float2(acc[4 * j + 2] * out_scale, acc[4 * j + 3] * out_scale);
      }
    }
  }
}

// ---- weights -> packed fp16 (hi, lo) tiles of w * 2^kWeightScaleLog2, all hidden matrices of the policy in ONE launch ----
struct SplitJob {
  const float* src;   // [256 out, K in]
  uint8_t* fwd;       // forward pack
  uint8_t* dgrad;     // dgrad pack or NULL
  int K;
};
struct SplitJobs {
  SplitJob j[8];
  int count;
};
// item = (out row o, 8 consecutive inputs): 16 bytes of hi and of lo in each pack
__global__ void __launch_bounds__(256) split_half_kernel(SplitJobs jobs) {
  const float scale = (float)(1 << kWeightScaleLog2);
  for (int q = 0; q < jobs.count; ++q) {
    const SplitJob& J = jobs.j[q];
    const int cpr = J.K / 8;  // 16-byte chunks per row
    const int64_t items = (int64_t)BN * cpr;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += stride) {
      const int o = (int)(i / cpr), c8 = (int)(i - (int64_t)o * cpr);  // inputs [8*c8, 8*c8+8)
      const float4 x0 = *reinterpret_cast<const float4*>(J.src + (size_t)o * J.K + 8 * c8);
      const float4 x1 = *reinterpret_cast<const float4*>(J.src + (size_t)o * J.K + 8 * c8 + 4);
      const float v[8] = {x0.x * scale, x0.y * scale, x0.z * scale, x0.w * scale,
                          x1.x * scale, x1.y * scale, x1.z * scale, x1.w * scale};
      uint32_t h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const __half2 hh = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
        const float2 hf = __half22float2(hh);
        const __half2 ll = __floats2half2_rn(v[2 * j] - hf.x, v[2 * j + 1] - hf.y);
        h[j] = *reinterpret_cast<const uint32_t*>(&hh);
        l[j] = *reinterpret_cast<const uint32_t*>(&ll);
      }
      {  // forward pack: k-block = 8*c8 / 32, tile row o (64 B), chunk (c8 & 3) swizzled by ((o >> 1) & 3)
        const int kb = c8 >> 2, ch = c8 & 3;
        uint8_t* d = J.fwd + (size_t)kb * (2 * kB16) + o * 64 + ((ch ^ ((o >> 1) & 3)) << 4);
        *reinterpret_cast<uint4*>(d) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(d + kB16) = make_uint4(l[0], l[1], l[2], l[3]);
      }
      if (J.dgrad != nullptr) {  // dgrad pack: k-block = o / 32, group = input / 64, row o % 32 (128 B), chunk swizzled by (row & 7)
        const int kb = o >> 5, r = o & 31, grp = c8 >> 3, ch = c8 & 7;
        uint8_t* d = J.dgrad + (size_t)kb * (2 * kB16) + grp * 4096 + r * 128 + ((ch ^ (r & 7)) << 4);
        *reinterpret_cast<uint4*>(d) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(d + kB16) = make_uint4(l[0], l[1], l[2], l[3]);
      }
    }
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
int encode_f32_sw128(CUtensorMap* out, const float* base, uint64_t rows, uint64_t cols, uint32_t box_rows);

int launch(const GemmLaunch* L, int ngroups, int64_t M, int K, int epi, int b_mn, cudaStream_t st) {
  if (ngroups < 1 || ngroups > 2 || K % BK != 0 || K <= 0 || M <= 0) return RB200_E_SHAPE;
  GemmParams P{};
  P.M = M; P.K = K; P.epi = epi; P.ngroups = ngroups;
  for (int g = 0; g < ngroups; ++g) {
    const GemmLaunch& l = L[g];
    const uintptr_t al = reinterpret_cast<uintptr_t>(l.a) | reinterpret_cast<uintptr_t>(l.b_hi) |
                         reinterpret_cast<uintptr_t>(l.c) | reinterpret_cast<uintptr_t>(l.h);
    if (al & 15) return RB200_E_ALIGN;
    if (encode_f32_sw128(&P.a[g], l.a, (uint64_t)M, (uint64_t)K, BM)) return RB200_E_UNSUPPORTED;
    P.wpack[g] = reinterpret_cast<const uint8_t*>(l.b_hi);
    P.g[g] = Group{l.bias, l.h, l.colsum, l.amax_in, l.amax_out, l.c};
  }
  static bool attr_done = false;
  constexpr int kSmem = kRingBytes + 1024 + (int)sizeof(Barriers);
  static_assert(kSmem <= 232448, "tc_h_gemm_kernel shared memory");
  if (!attr_done) {
    cudaError_t ce = cudaFuncSetAttribute(tc_h_gemm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (ce == cudaSuccess) ce = cudaFuncSetAttribute(tc_h_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (ce != cudaSuccess) return (int)ce;
    attr_done = true;
  }
  // one launch serves both towers (grouped tile scheduling): it fills the tail wave of small per-rank batches
  const int64_t n_tiles = (M + BM - 1) / BM;
  int per_group = rb::sm_count() / ngroups;
  if (per_group > n_tiles) per_group = (int)n_tiles;
  if (per_group < 1) per_group = 1;
  rb::tch::SlotSums ss{};
  ss.nslab = per_group;
  ss.stride = (int64_t)ngroups * BN;
  if (epi == rb::tc::EPI_TANHGRAD)
    for (int g = 0; g < ngroups; ++g)
      if (L[g].colsum) {
        if (!P.part && !(P.part = rb::partials_scratch((int64_t)per_group * ngroups * BN))) return RB200_E_UNSUPPORTED;
        ss.part[ss.count] = P.part + g * BN;
        ss.out[ss.count] = L[g].colsum;
        ss.len[ss.count++] = BN;
      }
  if (b_mn) tc_h_gemm_kernel<1><<<per_group * ngroups, kThreads, kSmem, st>>>(P);
  else tc_h_gemm_kernel<0><<<per_group * ngroups, kThreads, kSmem, st>>>(P);
  rb::count_launch();
  cudaError_t ce = cudaPeekAtLastError();
  if (ce != cudaSuccess) return (int)ce;
  return ss.count ? rb::tch::sum_slots(ss, st) : 0;
}

int wgrad(const WgradLaunch* L, int ngroups, int64_t n, int IN, cudaStream_t st) {
  if (ngroups < 1 || ngroups > 2 || n <= 0 || IN <= 0 || IN > 256 || IN % 32 != 0) return RB200_E_SHAPE;
  WgradParams P{};
  P.n = n; P.IN = IN; P.ngroups = ngroups;
  for (int g = 0; g < ngroups; ++g) {
    const uintptr_t al = reinterpret_cast<uintptr_t>(L[g].z) | reinterpret_cast<uintptr_t>(L[g].h) |
                         reinterpret_cast<uintptr_t>(L[g].dW);
    if (al & 15) return RB200_E_ALIGN;
    int e = encode_f32_sw128(&P.z[g], L[g].z, (uint64_t)n, 256, 32);
    if (!e) e = encode_f32_sw128(&P.h[g], L[g].h, (uint64_t)n, (uint64_t)IN, 32);
    if (e) return RB200_E_UNSUPPORTED;
    P.dW[g] = L[g].dW;
    P.amax_z[g] = L[g].amax_z;
  }
  static bool attr_done = false;
  constexpr int kSmem = kWgRingBytes + 1024 + (int)sizeof(WgBarriers);
  static_assert(kSmem <= 232448, "tc_h_wgrad_kernel shared memory");
  if (!attr_done) {
    cudaError_t ce = cudaFuncSetAttribute(tc_h_wgrad_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (ce == cudaSuccess) ce = cudaFuncSetAttribute(tc_h_wgrad_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (ce != cudaSuccess) return (int)ce;
    attr_done = true;
  }
  const int n_kb = (int)((n + BK - 1) / BK);
  int chunks = rb::sm_count() / (2 * ngroups);
  if (chunks < 1) chunks = 1;
  if (chunks > n_kb) chunks = n_kb;
  P.kb_per_chunk = (n_kb + chunks - 1) / chunks;
  chunks = (n_kb + P.kb_per_chunk - 1) / P.kb_per_chunk;  // every chunk non-empty: each writes its slot
  const int64_t slab = 256 * (int64_t)IN;
  if (!(P.part = rb::partials_scratch(chunks * ngroups * slab))) return RB200_E_UNSUPPORTED;
  const dim3 grid(ngroups * 2 * chunks);
  if (IN <= 128) tc_h_wgrad_kernel<128><<<grid, kThreads, kSmem, st>>>(P);
  else tc_h_wgrad_kernel<256><<<grid, kThreads, kSmem, st>>>(P);
  rb::count_launch();
  cudaError_t ce = cudaPeekAtLastError();
  if (ce != cudaSuccess) return (int)ce;
  rb::tch::SlotSums ss{};
  ss.count = ngroups;
  ss.nslab = chunks;
  ss.stride = ngroups * slab;
  for (int g = 0; g < ngroups; ++g) {
    ss.part[g] = P.part + g * slab;
    ss.out[g] = L[g].dW;
    ss.len[g] = (int)slab;
  }
  return rb::tch::sum_slots(ss, st);
}

__global__ void __launch_bounds__(256) sum_slots_kernel(const SlotSums s) {
  const int q = blockIdx.y;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < s.len[q]; i += gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < s.nslab; ++k) acc += s.part[q][k * s.stride + i];
    s.out[q][i] += acc;
  }
}

int sum_slots(const SlotSums& s, cudaStream_t st) {
  if (s.count < 1 || s.count > 8 || s.nslab < 1) return RB200_E_SHAPE;
  int len = 0;
  for (int q = 0; q < s.count; ++q) len = s.len[q] > len ? s.len[q] : len;
  int blocks = (len + 255) / 256;
  if (blocks > 4 * rb::sm_count()) blocks = 4 * rb::sm_count();
  sum_slots_kernel<<<dim3(blocks, s.count), 256, 0, st>>>(s);
  rb::count_launch();
  cudaError_t ce = cudaPeekAtLastError();
  return ce == cudaSuccess ? 0 : (int)ce;
}

int split_weights(const SplitSpec* specs, int count, cudaStream_t st) {
  if (count < 1 || count > 8) return RB200_E_SHAPE;
  SplitJobs jobs{};
  jobs.count = count;
  int64_t total = 0;
  for (int i = 0; i < count; ++i) {
    const int64_t K = specs[i].n / BN;
    if (K * BN != specs[i].n || K % BK != 0 || (specs[i].lo != nullptr && K != BN)) return RB200_E_SHAPE;
    jobs.j[i] = SplitJob{specs[i].src, reinterpret_cast<uint8_t*>(specs[i].hi), reinterpret_cast<uint8_t*>(specs[i].lo), (int)K};
    total = specs[i].n / 8 > total ? specs[i].n / 8 : total;
  }
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * 4;
  if (blocks > cap) blocks = cap;
  split_half_kernel<<<(int)blocks, 256, 0, st>>>(jobs);
  rb::count_launch();
  cudaError_t ce = cudaPeekAtLastError();
  return ce == cudaSuccess ? 0 : (int)ce;
}

}  // namespace tch

namespace tc {
int g_debug_flags = 0;

}  // namespace tc
}  // namespace rb

// Experiment switches of the kernels (see tc_gemm.cuh); not part of the product surface.
extern "C" int rb200_debug_set_flags(int flags) {
  rb::tc::g_debug_flags = flags;
  return RB200_OK;
}

// ---- unit-test entries (tests/test_gpu_tc_gemm.py) --------------------------------------------------------------------
// C[M,256] = A[M,K] . B[256,K]^T (mode 0, forward) or A[M,256] . B[256,256] (mode 1, dgrad form: B is [out=K, in=N]);
// work: >= 256*K floats (fp16 hi/lo copies of B).  amax (device float, nullable) exercises the gradient scaling.
extern "C" int rb200_tc_gemm_h(const float* A, const float* B, float* C, int64_t M, int K, int mode, const float* amax,
                               float* work, rb200_stream_t stream) {
  if (!A || !B || !C || !work) return RB200_E_NULL;
  if (M <= 0 || K <= 0 || K % rb::tc::BK != 0) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  const int64_t nb = (int64_t)rb::tc::BN * K;
  if (mode && K != rb::tc::BN) return RB200_E_SHAPE;
  // forward pack always; the dgrad pack (square matrices only) behind it
  rb::tch::SplitSpec sp{B, work, mode ? work + nb : nullptr, nb};
  int e = rb::tch::split_weights(&sp, 1, st);
  if (e) return e;
  rb::tch::GemmLaunch l{};
  l.a = A; l.b_hi = mode ? sp.lo : sp.hi; l.b_lo = nullptr; l.c = C; l.amax_in = amax;
  return rb::tch::launch(&l, 1, M, K, rb::tc::EPI_STORE, mode ? 1 : 0, st);
}

extern "C" int rb200_tc_wgrad_h(const float* Z, const float* H, float* dW, int64_t n, int IN, const float* amax,
                                rb200_stream_t stream) {
  if (!Z || !H || !dW) return RB200_E_NULL;
  rb::tch::WgradLaunch l{Z, H, dW, amax};
  return rb::tch::wgrad(&l, 1, n, IN, rb::as_stream(stream));
}
