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
#include <cuda_bf16.h>

#include "common.cuh"
#include "softmax_acc.cuh"
#include "tc_half.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace rb {
namespace lmh {
int encode_bf16_sw128(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t s1_bytes,
                      uint64_t s2_bytes, uint32_t box0, uint32_t box1);
}
}  // namespace rb

namespace {

using rb::smx::Acc;
using rb::tch::kSw128;
using rb::tch::warp_arrive;
namespace tma = rb::tma;
namespace wg = rb::wg;

// Every operand is a rank-3 tensor map (a matrix is [1, rows, cols]), so every load is the 3-D form.
// CTA tile: BM (GEMM M) x BN (GEMM N), K-blocks of 64 bf16 = one 128-byte swizzle span.  Consumer warpgroup w owns
// columns [128 w, 128 w + 128) of the tile over all 128 rows (two m64n128 accumulators), so both read the same A stage.
constexpr int BM = 128, BN = 256, BK = 64;
constexpr int kABytes = BM * BK * 2;          // 16 KB
constexpr int kBBytes = BN * BK * 2;          // 32 KB
constexpr int kBox64 = 64 * BK * 2;           // 8 KB: one [64 x 64] box (MN-major operands come in these)
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kStages = 4;
constexpr int kRingBytes = kStages * kStageBytes;  // 192 KB
constexpr int kThreads = 384;                      // consumer warpgroups 0 / 1, producer warpgroup 2
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
static_assert(128 * kProducerRegs + 256 * kConsumerRegs <= 65536, "register file");
// Work decomposition of FWD / DZ: about kTargetItems work items, so that the vocabulary ranges depend on N, V and the
// window only.  Items are rasterised in groups of kGroupRows row tiles: the CTAs resident at one time share their X
// tiles and their W ranges through L2.
constexpr int kTargetItems = 512;
constexpr int kGroupRows = 16;

enum Mode { FWD = 0, DZ = 1, DW = 2, DX = 3 };

struct __align__(16) Bars {
  uint64_t full[kStages];
  uint64_t empty[kStages];  // one arrival per consumer warp
  Acc xwg[BM];              // FWD: warpgroup 1's row statistics, merged into warpgroup 0's
};
constexpr int kSmem = kRingBytes + 1024 + (int)sizeof(Bars);
static_assert(kSmem <= 232448, "lmhead shared memory");

struct Params {
  CUtensorMap a, b;
  int64_t N, L;
  int bsz, tpb;         // batch items, 128-row tiles per batch item
  int row_tiles;        // bsz * tpb
  int H, v_lo, v_hi;
  float inv_t;
  int n_kb;             // k-blocks per tile
  int kpb;              // DW: 64-row k-blocks per batch item
  int n_ranges, tiles_per_range, n_vtiles;  // FWD / DZ: 256-wide vocabulary tiles of the window / chunk
  int n_ntiles;         // DW / DX: 256-wide column tiles of H
  int c0, width, ld;    // backward chunk [c0, c0 + width) and the workspace row length (elements)
  int first, last;      // DX: first / last chunk
  const int64_t* target;
  float* part;          // FWD: [n_ranges, N, 3] (m, s, t)
  float* zt;            // FWD: [N] z of the target column
  const float* lse;
  const float* h_in;
  const float* g_lp;
  const float* g_h;
  __nv_bfloat16* dz;    // [N, ld]
  float* dx_acc;        // [N, H]
  __nv_bfloat16* dx;    // [N, H]
  __nv_bfloat16* dw;    // [V, H]
};

// FWD / DZ item -> (row tile, range): groups of kGroupRows row tiles, row tile fastest inside a group
__device__ __forceinline__ void item_rows_ranges(const Params& P, int item, int& rt, int& ri) {
  const int per_group = kGroupRows * P.n_ranges;
  const int grp = item / per_group, loc = item - grp * per_group;
  const int g0 = grp * kGroupRows;
  const int gn = min(kGroupRows, P.row_tiles - g0);
  rt = g0 + loc % gn;
  ri = loc / gn;
}

__device__ __forceinline__ void named_sync_consumers() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <int MODE>
__global__ void __launch_bounds__(kThreads, 1) lmhead_kernel(const __grid_constant__ Params P) {
  constexpr int TA = MODE == DW ? 1 : 0;                 // A MN-major: dZ^T
  constexpr int TB = (MODE == DW || MODE == DX) ? 1 : 0;  // B MN-major: X (DW) / W (DX)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (tma::smem_u32(smem_raw) & 1023u)) & 1023u);
  Bars* bars = reinterpret_cast<Bars*>(smem + kRingBytes);
  const int wgi = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  // ---- the CTA's work item ----
  int rt = 0, ri = 0, nt = 0, mt = 0, tile0 = 0, tile1 = 1;
  if (MODE == FWD || MODE == DZ) {
    item_rows_ranges(P, blockIdx.x, rt, ri);
    tile0 = ri * P.tiles_per_range;
    tile1 = min(tile0 + P.tiles_per_range, P.n_vtiles);
  } else if (MODE == DX) {
    rt = blockIdx.x / P.n_ntiles;
    nt = blockIdx.x % P.n_ntiles;
  } else {
    mt = blockIdx.x / P.n_ntiles;
    nt = blockIdx.x % P.n_ntiles;
  }
  const int bi = rt / P.tpb, p0 = (rt % P.tpb) * BM;  // batch item and first position of the row tile
  const int vbase = MODE == FWD ? P.v_lo : P.c0;      // FWD / DZ: first vocabulary column of tile 0

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      tma::mbar_init(&bars->full[s], 1);
      tma::mbar_init(&bars->empty[s], 8);
    }
    tma::fence_barrier_init();
  }
  __syncthreads();

  if (wgi == 2) {
    // ================= producer: one lane =================
    wg::setmaxnreg_dec<kProducerRegs>();
    if (threadIdx.x == 256) {
      tma::prefetch_desc(&P.a);
      tma::prefetch_desc(&P.b);
      uint32_t s = 0, ph = 0;
      for (int tile = tile0; tile < tile1; ++tile) {
        for (int kb = 0; kb < P.n_kb; ++kb) {
          tma::mbar_wait(&bars->empty[s], ph ^ 1u);
          uint8_t* sa = smem + s * kStageBytes;
          uint8_t* sb = sa + kABytes;
          uint64_t* full = &bars->full[s];
          tma::mbar_arrive_expect_tx(full, kStageBytes);  // out-of-bounds parts of a box count too (zero-filled)
          if (MODE == FWD || MODE == DZ) {
            tma::load_3d(sa, &P.a, kb * BK, p0, bi, full);                 // X [128 rows x 64 h]
            tma::load_3d(sb, &P.b, kb * BK, vbase + tile * BN, 0, full);   // W [256 v x 64 h]
          } else if (MODE == DX) {
            tma::load_3d(sa, &P.a, kb * BK, p0, bi, full);                 // dZ [128 rows x 64 v]
#pragma unroll
            for (int i = 0; i < 4; ++i) tma::load_3d(sb + i * kBox64, &P.b, nt * BN + 64 * i, P.c0 + kb * BK, 0, full);
          } else {
            const int b = kb / P.kpb, pp = (kb % P.kpb) * BK;                // k-block = 64 positions of one batch item
#pragma unroll
            for (int i = 0; i < 2; ++i) tma::load_3d(sa + i * kBox64, &P.a, mt * BM + 64 * i, pp, b, full);  // dZ
#pragma unroll
            for (int i = 0; i < 4; ++i) tma::load_3d(sb + i * kBox64, &P.b, nt * BN + 64 * i, pp, b, full);  // X
          }
          if (++s == kStages) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // ================= consumers =================
  wg::setmaxnreg_inc<kConsumerRegs>();
  const int w = wgi;
  const int g = lane >> 2, t = lane & 3;
  const int rr = (warp & 3) * 16 + g;  // rows rr, rr + 8 of each m64 half: local row of index i is 64 (i >> 1) + rr + 8 (i & 1)
  // per-row state of the FWD / DZ epilogues (the 4 rows this thread holds in every tile)
  int64_t row[4];
  bool rok[4];
  int64_t tg[4];
  float r_lse[4], r_h[4], r_glp[4], r_gh[4];
  Acc st[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    rb::smx::acc_init(st[i]);
    const int p = p0 + 64 * (i >> 1) + rr + 8 * (i & 1);
    rok[i] = (MODE != DW) && p < P.L;
    row[i] = (int64_t)bi * P.L + p;
    tg[i] = -1;
    r_lse[i] = r_h[i] = r_glp[i] = r_gh[i] = 0.f;
    if ((MODE == FWD || MODE == DZ) && rok[i]) tg[i] = __ldg(P.target + row[i]);
    if (MODE == DZ && rok[i]) {
      r_lse[i] = __ldg(P.lse + row[i]);
      r_glp[i] = P.g_lp ? __ldg(P.g_lp + row[i]) : 0.f;
      r_gh[i] = P.g_h ? __ldg(P.g_h + row[i]) : 0.f;
      r_h[i] = P.g_h ? __ldg(P.h_in + row[i]) : 0.f;
    }
  }

  uint32_t q = 0;  // the CTA's k-block q sits in stage q % kStages, filled in phase q / kStages
  for (int tile = tile0; tile < tile1; ++tile) {
    float acc[2][64];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[h][i] = 0.f;
    for (int kb = 0; kb < P.n_kb; ++kb, ++q) {
      const uint32_t s = q % kStages;
      tma::mbar_wait_brk(&bars->full[s], (q / kStages) & 1u);
      const uint32_t sa = tma::smem_u32(smem + s * kStageBytes), sb = sa + kABytes + w * 2 * kBox64;
      wg::fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        // K-major: 128-byte rows, the next 16 k are 32 B further along; MN-major: 16 k = 16 rows of 128 B, the next
        // 64 columns are the next [64 x 64] box
        const uint64_t bd = TB ? wg::desc(sb + k * 2048, kBox64, 1024, kSw128) : wg::desc(sb + k * 32, 16, 1024, kSw128);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t ad = TA ? wg::desc(sa + h * kBox64 + k * 2048, kBox64, 1024, kSw128)
                                 : wg::desc(sa + h * kBox64 + k * 32, 16, 1024, kSw128);
          wg::MmaSS<128, TA, TB, wg::bf16>::run(acc[h], ad, bd, 1u);
        }
      }
      wg::commit();
      wg::wait<1>();
      if (kb > 0) warp_arrive(&bars->empty[(q - 1) % kStages]);
    }
    wg::wait<0>();
    wg::fence_operand(acc[0]);
    wg::fence_operand(acc[1]);
    warp_arrive(&bars->empty[(q - 1) % kStages]);

    // ---- epilogues, straight from the accumulator registers: element (i, j, e) of acc[i >> 1][4 j + 2 (i & 1) + e]
    // is local row 64 (i >> 1) + rr + 8 (i & 1), local column 128 w + 8 j + 2 t + e ----
    if (MODE == FWD || MODE == DZ) {
      const int vt = vbase + tile * BN + 128 * w;  // global column of the warpgroup's local column 0
      const int lim = (MODE == FWD ? P.v_hi : P.c0 + P.width) - vt;  // local columns >= lim are outside
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t rel64 = tg[i] - vt;
        const int rel = (rel64 >= 0 && rel64 < lim) ? (int)rel64 : -1;  // local column of the target, or none
        const float* a = acc[i >> 1] + 2 * (i & 1);
        if (MODE == FWD) {
#pragma unroll
          for (int j = 0; j < 16; j += 2) {
            float z[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const int c = 8 * (j + (u >> 1)) + 2 * t + (u & 1);
              const float v = a[4 * (j + (u >> 1)) + (u & 1)] * P.inv_t;
              if (c == rel && rok[i]) P.zt[row[i]] = v;
              z[u] = c < lim ? v : -INFINITY;
            }
            rb::smx::acc_add4(st[i], z[0], z[1], z[2], z[3]);
          }
        } else {
          if (!rok[i]) continue;
          __nv_bfloat16* drow = P.dz + row[i] * P.ld + (vt - P.c0);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            float gv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * j + 2 * t + e;
              gv[e] = c < lim ? rb::smx::dz_of(a[4 * j + e], P.inv_t, r_lse[i], r_glp[i], r_gh[i], r_h[i], c == rel)
                              : 0.f;
            }
            const int c = 8 * j + 2 * t;
            if (c + 1 < lim) *reinterpret_cast<uint32_t*>(drow + c) = pack_bf16(gv[0], gv[1]);
            else if (c < lim) drow[c] = __float2bfloat16_rn(gv[0]);
          }
        }
      }
    } else if (MODE == DX) {
      const int h0 = nt * BN + 128 * w;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (!rok[i]) continue;
        const float* a = acc[i >> 1] + 2 * (i & 1);
        float* arow = P.dx_acc + row[i] * P.H;
        __nv_bfloat16* xrow = P.dx + row[i] * P.H;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int h = h0 + 8 * j + 2 * t;
          if (h >= P.H) continue;  // H % 64 == 0: both columns of the pair are in or out together
          float2 v = make_float2(a[4 * j], a[4 * j + 1]);
          if (!P.first) {
            const float2 o = *reinterpret_cast<const float2*>(arow + h);
            v.x += o.x;
            v.y += o.y;
          }
          if (P.last) *reinterpret_cast<uint32_t*>(xrow + h) = pack_bf16(v.x, v.y);
          else *reinterpret_cast<float2*>(arow + h) = v;
        }
      }
    } else {  // DW: rows are vocabulary columns of the chunk, columns are hidden units
      const int h0 = nt * BN + 128 * w;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = mt * BM + 64 * (i >> 1) + rr + 8 * (i & 1);
        if (m >= P.width) continue;
        const float* a = acc[i >> 1] + 2 * (i & 1);
        __nv_bfloat16* wrow = P.dw + (int64_t)(P.c0 + m) * P.H;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int h = h0 + 8 * j + 2 * t;
          if (h < P.H) *reinterpret_cast<uint32_t*>(wrow + h) = pack_bf16(a[4 * j], a[4 * j + 1]);
        }
      }
    }
  }

  if (MODE == FWD) {
    // the 4 lanes of a quad hold the same rows: merge them, then warpgroup 1's statistics into warpgroup 0's
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        Acc b;
        b.m = __shfl_xor_sync(0xffffffffu, st[i].m, o);
        b.s = __shfl_xor_sync(0xffffffffu, st[i].s, o);
        b.t = __shfl_xor_sync(0xffffffffu, st[i].t, o);
        rb::smx::acc_merge(st[i], b);
      }
    }
    if (w == 1 && t == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) bars->xwg[64 * (i >> 1) + rr + 8 * (i & 1)] = st[i];
    }
    named_sync_consumers();
    if (w == 0 && t == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (!rok[i]) continue;
        rb::smx::acc_merge(st[i], bars->xwg[64 * (i >> 1) + rr + 8 * (i & 1)]);
        float* pp = P.part + ((size_t)ri * P.N + row[i]) * 3;
        pp[0] = st[i].m;
        pp[1] = st[i].s;
        pp[2] = st[i].t;
      }
    }
  }
}

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

// ---- host ----------------------------------------------------------------------------------------------------------
struct Geo {
  int64_t N, L, bsz, batch_stride, row_stride;
  int H, V, v_lo, v_hi;
  int64_t tpb, row_tiles;
  int n_vtiles, n_ranges, tiles_per_range;
};

int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// vocabulary ranges of a row-tile count and a vocabulary width: a function of the shapes only
void split_ranges(int64_t row_tiles, int width, int& n_vtiles, int& n_ranges, int& tiles_per_range) {
  n_vtiles = (int)cdiv(width, BN);
  int64_t want = cdiv(kTargetItems, row_tiles);
  if (want > n_vtiles) want = n_vtiles;
  if (want < 1) want = 1;
  tiles_per_range = (int)cdiv(n_vtiles, want);
  n_ranges = (int)cdiv(n_vtiles, tiles_per_range);
}

int make_geo(Geo& g, int64_t N, int64_t L, int64_t batch_stride, int64_t row_stride, int H, int V, int v_lo, int v_hi) {
  if (N <= 0 || L <= 0 || N % L != 0 || V <= 0 || v_lo < 0 || v_hi > V || v_lo >= v_hi) return RB200_E_SHAPE;
  if (H < 64 || H > 8192 || H % 64 != 0) return RB200_E_SHAPE;
  g.N = N; g.L = L; g.bsz = N / L; g.H = H; g.V = V; g.v_lo = v_lo; g.v_hi = v_hi;
  g.row_stride = row_stride;
  g.batch_stride = g.bsz > 1 ? batch_stride : L * row_stride;
  if (row_stride < H || row_stride % 8 != 0 || g.batch_stride % 8 != 0 || g.batch_stride <= 0) return RB200_E_SHAPE;
  if (L > INT32_MAX || g.bsz > INT32_MAX) return RB200_E_SHAPE;
  g.tpb = cdiv(L, BM);
  g.row_tiles = g.bsz * g.tpb;
  if (g.row_tiles * kTargetItems > INT32_MAX) return RB200_E_SHAPE;
  split_ranges(g.row_tiles, v_hi - v_lo, g.n_vtiles, g.n_ranges, g.tiles_per_range);
  return RB200_OK;
}

int64_t fwd_ws_bytes(const Geo& g) { return cdiv(((int64_t)g.n_ranges * 3 + 1) * g.N * 4, 256) * 256; }
int64_t dz_ws_bytes(const Geo& g, int64_t vc) { return g.N * vc * 2; }
int64_t bwd_ws_bytes(const Geo& g, int64_t vc) {
  const int64_t whole = cdiv(g.v_hi - g.v_lo, BN) * BN;
  return dz_ws_bytes(g, vc) + (vc < whole ? g.N * g.H * 4 : 0);
}

void base_params(Params& P, const Geo& g, double inv_t) {
  P.N = g.N; P.L = g.L; P.bsz = (int)g.bsz; P.tpb = (int)g.tpb; P.row_tiles = (int)g.row_tiles;
  P.H = g.H; P.v_lo = g.v_lo; P.v_hi = g.v_hi; P.inv_t = (float)inv_t;
}

int x_map(CUtensorMap* m, const void* x, const Geo& g, uint32_t box_rows) {
  return rb::lmh::encode_bf16_sw128(m, x, g.H, g.L, g.bsz, g.row_stride * 2, g.batch_stride * 2, 64, box_rows);
}
int w_map(CUtensorMap* m, const void* w, const Geo& g, uint32_t box_rows) {
  return rb::lmh::encode_bf16_sw128(m, w, g.H, g.V, 1, (uint64_t)g.H * 2, (uint64_t)g.H * g.V * 2, 64, box_rows);
}
int dz_map(CUtensorMap* m, const void* dz, const Geo& g, int width, int64_t ld, uint32_t box0, uint32_t box_rows) {
  return rb::lmh::encode_bf16_sw128(m, dz, width, g.L, g.bsz, ld * 2, g.L * ld * 2, box0, box_rows);
}

template <int MODE>
int launch(const Params& P, int items, cudaStream_t st) {
  static bool attr_done = false;
  if (!attr_done) {
    const cudaError_t ce = cudaFuncSetAttribute(lmhead_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (ce != cudaSuccess) return (int)ce;
    attr_done = true;
  }
  lmhead_kernel<MODE><<<items, kThreads, kSmem, st>>>(P);
  rb::count_launch();
  const cudaError_t ce = cudaPeekAtLastError();
  return ce == cudaSuccess ? RB200_OK : (int)ce;
}

int check_ptrs(const void* hidden, const void* weight, const void* target, const void* ws) {
  if (!hidden || !weight || !target) return RB200_E_NULL;
  if (((reinterpret_cast<uintptr_t>(hidden) | reinterpret_cast<uintptr_t>(weight) | reinterpret_cast<uintptr_t>(ws)) &
       15) != 0)
    return RB200_E_ALIGN;
  return RB200_OK;
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

// vocabulary chunk of the backward from the workspace: the whole window if its dZ fits, else what is left after an
// fp32 [N, H] dX accumulator (dx_acc_bytes), in whole 256-column tiles; 0 when not even one tile fits
int64_t bwd_chunk(const Geo& g, int64_t workspace_bytes, int64_t dx_acc_bytes) {
  const int64_t whole = cdiv(g.v_hi - g.v_lo, BN) * BN;
  if (workspace_bytes >= dz_ws_bytes(g, whole)) return whole;
  const int64_t vc = (workspace_bytes - dx_acc_bytes) / (2 * g.N) / BN * BN;
  return vc < BN ? 0 : vc;
}

// The backward over [g.v_lo, g.v_hi) in chunks of vc columns.  dX is summed in fp32 in dx_acc over the chunks; with dx
// the last chunk writes it there in bf16 instead, without dx it stays in dx_acc.
int bwd_chunks(const Geo& g, const void* hidden, const void* weight, const int64_t* target, double inv_temperature,
               const float* lse, const float* entropy, const float* grad_logprob, const float* grad_entropy, int64_t vc,
               __nv_bfloat16* dz, float* dx_acc, __nv_bfloat16* dx, __nv_bfloat16* dw, cudaStream_t st) {
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
    if ((e = launch<DZ>(A, (int)(g.row_tiles * A.n_ranges), st))) return e;
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
