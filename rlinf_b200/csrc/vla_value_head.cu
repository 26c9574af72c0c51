// Value head of the OpenVLA / OpenVLA-OFT policies: the reference's ValueHead(H, (512, 128), O, "gelu",
// bias_last=False) (models/embodiment/modules/value_head.py) applied in bf16 to one hidden row per sample, and
// autograd's backward through it.  The widths, GELU and the missing last bias are compile-time constants.
//
//   forward   z0 = bf16(x W0^T + b0)   a0 = bf16(gelu(z0))         [n, 512]
//             z1 = bf16(a0 W1^T + b1)  a1 = bf16(gelu(z1))         [n, 128]
//             v  = bf16(a1 W2^T)                                   [n, O]
//   backward  da1 = bf16(gv W2)   dz1 = bf16(da1 gelu'(z1))   da0 = bf16(dz1 W1)   dz0 = bf16(da0 gelu'(z0))
//             dX = bf16(dz0 W0)   dW0 = bf16(dz0^T X)   db0 = bf16(sum dz0)   dW1 = bf16(dz1^T a0)   db1 = bf16(sum dz1)
//             dW2 = bf16(gv^T a1)
// Every sum is fp32; gelu and gelu' are evaluated in fp32 on the bf16 input, in ATen's form.
//
// Kernels (mma.sync m16n8k16 bf16 with fp32 accumulation, one instruction shape for every n):
//   l0_fwd_kernel     layer 0.  64 x 128 output tiles; the K = H dimension is split into 8 slices of whole 32-column
//                     k-blocks fixed by H alone, one CTA each, in an 8-CTA cluster.  The slices' fp32 tiles are added
//                     in slice order through distributed shared memory, then + b0 and rounded: z0.
//   tail_fwd_kernel   16 rows per CTA: gelu(z0) in shared memory, layer 1 on the tensor cores (W1 from L2), gelu, and
//                     the O <= 32 dot products of layer 2 in column order.
//   tail_bwd_kernel   16 rows per CTA: da1 and dz1 (SIMT, o in order), da0 on the tensor cores, dz0; writes dz0, dz1
//                     and, when dW1 is wanted, a0 to the workspace.
//   gemm_kernel       dX = dz0 W0 (K = 512), and one grouped launch of dW0 = dz0^T X and dW1 = dz1^T a0 (K = n, every
//                     k-block in order in one CTA: no split over n).
//   small_grads_kernel  db0, db1, dW2: 8 warps stride the rows in a fixed interleave, then warp 0 adds them in order.
// A row's values depend only on the row and the parameters (tiles never mix rows, and the K slicing depends on H
// alone), so they are the same bits for any n, position or row stride.  No floating-point atomics; every reduction
// order is fixed by (n, H); nothing depends on the grid size beyond that or on the SM count.
#include <cooperative_groups.h>
#include <cuda_bf16.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace {

typedef __nv_bfloat16 bf16;

constexpr int kD0 = 512, kD1 = 128, kMaxO = 32;
constexpr int kBM = 64, kBN = 128, kBK = 32, kStages = 3, kThreads = 128;
constexpr int kSplit = 8;      // K slices of layer 0 = the cluster size
constexpr int kRows = 16;      // rows per tail CTA
constexpr int kSmallWarps = 8;
// shared-memory tiles: A as [64][32 + 8] ([m][k]) or [32][64 + 8] ([k][m]); B as [128][32 + 8] or [32][128 + 8]
constexpr int kAElems = kBM * (kBK + 8) > kBK * (kBM + 8) ? kBM * (kBK + 8) : kBK * (kBM + 8);
constexpr int kBElems = kBN * (kBK + 8) > kBK * (kBN + 8) ? kBN * (kBK + 8) : kBK * (kBN + 8);
constexpr int kStageElems = kAElems + kBElems;
constexpr int kSmemBytes = kStages * kStageElems * 2;
constexpr int kRedLd = kBN + 4;
static_assert(kBM * kRedLd * 4 <= kSmemBytes, "the slice tile reuses the pipeline's shared memory");

__device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float round_bf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// ATen's GeluCUDAKernelImpl / GeluBackwardCUDAKernelImpl (approximate='none') in fp32
__device__ __forceinline__ float gelu(float x) { return x * 0.5f * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float gelu_grad(float dy, float x) {
  const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
  const float pdf = expf(-0.5f * x * x) * 0.39894228040143267794f;
  return dy * (cdf + x * pdf);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp16(void* dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_u32(dst)), "l"(src), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm4_t(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}

__device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t pack2(bf16 lo, bf16 hi) {
  return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

// C[m][n] = sum_k A[m][k] B[k][n] over a 64 x 128 tile.  AT: A[m][k] at a[k lda + m], else a[m lda + k].
// BT: B[k][n] at b[k ldb + n], else b[n ldb + k].  Rows m >= M, columns n >= N and k >= K read as zeros.
struct Gemm {
  const bf16* a;
  int64_t lda;
  const bf16* b;
  int64_t ldb;
  bf16* c;
  int64_t ldc;
  int M, N, K, tiles_n, tiles;
};

template <bool AT, bool BT>
__device__ __forceinline__ void load_stage(bf16* sA, bf16* sB, const Gemm& g, int m0, int n0, int k0) {
  const int t = threadIdx.x;
#pragma unroll
  for (int i = 0; i < kBM * kBK / 8 / kThreads; ++i) {
    const int c = t + i * kThreads;
    if (!AT) {
      const int r = c >> 2, kc = (c & 3) * 8, m = m0 + r, k = k0 + kc;
      const bool v = m < g.M && k < g.K;
      cp16(sA + r * (kBK + 8) + kc, v ? g.a + (int64_t)m * g.lda + k : g.a, v);
    } else {
      const int r = c >> 3, mc = (c & 7) * 8, k = k0 + r, m = m0 + mc;
      const bool v = k < g.K && m < g.M;
      cp16(sA + r * (kBM + 8) + mc, v ? g.a + (int64_t)k * g.lda + m : g.a, v);
    }
  }
#pragma unroll
  for (int i = 0; i < kBN * kBK / 8 / kThreads; ++i) {
    const int c = t + i * kThreads;
    if (!BT) {
      const int r = c >> 2, kc = (c & 3) * 8, n = n0 + r, k = k0 + kc;
      const bool v = n < g.N && k < g.K;
      cp16(sB + r * (kBK + 8) + kc, v ? g.b + (int64_t)n * g.ldb + k : g.b, v);
    } else {
      const int r = c >> 4, nc = (c & 15) * 8, k = k0 + r, n = n0 + nc;
      const bool v = k < g.K && n < g.N;
      cp16(sB + r * (kBN + 8) + nc, v ? g.b + (int64_t)k * g.ldb + n : g.b, v);
    }
  }
}

// four warps as 2 x 2, each a 32 x 64 warp tile: acc[mi][ni] is the m16n8 tile (wm 32 + 16 mi, wn 64 + 8 ni); k-blocks
// [kb0, kb1) in order through a three-stage cp.async ring
template <bool AT, bool BT>
__device__ __forceinline__ void mainloop(float (&acc)[2][8][4], bf16* smem, const Gemm& g, int m0, int n0, int kb0,
                                         int kb1) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wm = (warp & 1) * 32, wn = (warp >> 1) * 64;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0f;
  const int nk = kb1 - kb0;
#pragma unroll
  for (int s = 0; s < kStages - 1; ++s) {
    if (s < nk) load_stage<AT, BT>(smem + s * kStageElems, smem + s * kStageElems + kAElems, g, m0, n0, (kb0 + s) * kBK);
    cp_commit();
  }
#pragma unroll 1
  for (int i = 0; i < nk; ++i) {
    cp_wait<kStages - 2>();
    __syncthreads();
    const int nx = i + kStages - 1;
    if (nx < nk) {
      bf16* st = smem + (nx % kStages) * kStageElems;
      load_stage<AT, BT>(st, st + kAElems, g, m0, n0, (kb0 + nx) * kBK);
    }
    cp_commit();
    const bf16* sA = smem + (i % kStages) * kStageElems;
    const bf16* sB = sA + kAElems;
#pragma unroll
    for (int kk = 0; kk < kBK; kk += 16) {
      uint32_t a[2][4], b[4][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int mr = wm + mi * 16;
        if (!AT) {
          ldsm4(a[mi], sA + (mr + (lane & 15)) * (kBK + 8) + kk + (lane >> 4) * 8);
        } else {
          const int q = lane >> 3;
          ldsm4_t(a[mi], sA + (kk + (lane & 7) + (q >> 1) * 8) * (kBM + 8) + mr + (q & 1) * 8);
        }
      }
#pragma unroll
      for (int nj = 0; nj < 4; ++nj) {
        const int nc = wn + nj * 16;
        if (!BT) {
          ldsm4(b[nj], sB + (nc + (lane & 7) + (lane >> 4) * 8) * (kBK + 8) + kk + ((lane >> 3) & 1) * 8);
        } else {
          const int q = lane >> 3;
          ldsm4_t(b[nj], sB + (kk + (lane & 7) + (q & 1) * 8) * (kBN + 8) + nc + (q >> 1) * 8);
        }
      }
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 8; ++ni) mma(acc[mi][ni], a[mi], b[ni >> 1][(ni & 1) * 2], b[ni >> 1][(ni & 1) * 2 + 1]);
    }
  }
  cp_wait<0>();
  __syncthreads();
}

// z0 = bf16(x W0^T + b0): blockIdx = (row block, 128-column block, K slice); the cluster is the 8 slices of one tile
__global__ void __cluster_dims__(1, 1, kSplit) __launch_bounds__(kThreads)
    l0_fwd_kernel(const bf16* __restrict__ x, int64_t row_stride, int n, int H, const bf16* __restrict__ w0,
                  const bf16* __restrict__ b0, bf16* __restrict__ z0) {
  __shared__ __align__(16) unsigned char smem[kSmemBytes];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * kBN;
  const int nkb = H / kBK;
  const Gemm g{x, row_stride, w0, H, nullptr, 0, n, kD0, H, 0, 0};
  float acc[2][8][4];
  mainloop<false, false>(acc, reinterpret_cast<bf16*>(smem), g, m0, n0, rank * nkb / kSplit,
                         (rank + 1) * nkb / kSplit);
  float* red = reinterpret_cast<float*>(smem);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wm = (warp & 1) * 32, wn = (warp >> 1) * 64;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 8; ++ni) {
      const int r = wm + mi * 16 + (lane >> 2), c = wn + ni * 8 + (lane & 3) * 2;
      red[r * kRedLd + c] = acc[mi][ni][0];
      red[r * kRedLd + c + 1] = acc[mi][ni][1];
      red[(r + 8) * kRedLd + c] = acc[mi][ni][2];
      red[(r + 8) * kRedLd + c + 1] = acc[mi][ni][3];
    }
  cluster.sync();
  // slice CTA `rank` finishes rows [8 rank, 8 rank + 8) of the tile, adding the slices in slice order
  for (int e = threadIdx.x; e < 8 * kBN; e += kThreads) {
    const int r = rank * 8 + e / kBN, c = e % kBN;
    float s = cluster.map_shared_rank(red, 0)[r * kRedLd + c];
#pragma unroll
    for (int q = 1; q < kSplit; ++q) s += cluster.map_shared_rank(red, q)[r * kRedLd + c];
    const int row = m0 + r;
    if (row < n) z0[(int64_t)row * kD0 + n0 + c] = __float2bfloat16_rn(s + to_f(b0[n0 + c]));
  }
  cluster.sync();  // no CTA leaves while another reads its slice
}

// layers 1 and 2 on kRows rows: a0 = gelu(z0) in shared memory, z1 = bf16(a0 W1^T + b1) (warp w: columns 32 w ..),
// a1 = bf16(gelu(z1)), v = bf16(a1 W2^T) with each dot product in column order
__global__ void __launch_bounds__(kThreads) tail_fwd_kernel(const bf16* __restrict__ z0, int n,
                                                            const bf16* __restrict__ w1, const bf16* __restrict__ b1,
                                                            const bf16* __restrict__ w2, int O, bf16* __restrict__ z1,
                                                            bf16* __restrict__ v) {
  __shared__ __align__(16) bf16 sA[kRows][kD0 + 8];
  __shared__ __align__(16) bf16 sH[kRows][kD1 + 8];
  __shared__ float sW2[kMaxO][kD1 + 1];
  const int r0 = blockIdx.x * kRows;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, gr = lane >> 2, tq = lane & 3;
  for (int e = threadIdx.x; e < O * kD1; e += kThreads) sW2[e / kD1][e % kD1] = to_f(w2[e]);
  for (int c = threadIdx.x; c < kRows * kD0 / 8; c += kThreads) {
    const int r = c / (kD0 / 8), col = (c % (kD0 / 8)) * 8;
    uint4 u = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + r < n) u = __ldg(reinterpret_cast<const uint4*>(z0 + (int64_t)(r0 + r) * kD0 + col));
    bf16* p = reinterpret_cast<bf16*>(&u);
#pragma unroll
    for (int k = 0; k < 8; ++k) p[k] = __float2bfloat16_rn(gelu(to_f(p[k])));
    *reinterpret_cast<uint4*>(&sA[r][col]) = u;
  }
  __syncthreads();
  float acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.0f;
#pragma unroll 4
  for (int k0 = 0; k0 < kD0; k0 += 16) {
    uint32_t a[4];
    a[0] = *reinterpret_cast<const uint32_t*>(&sA[gr][k0 + 2 * tq]);
    a[1] = *reinterpret_cast<const uint32_t*>(&sA[gr + 8][k0 + 2 * tq]);
    a[2] = *reinterpret_cast<const uint32_t*>(&sA[gr][k0 + 8 + 2 * tq]);
    a[3] = *reinterpret_cast<const uint32_t*>(&sA[gr + 8][k0 + 8 + 2 * tq]);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bf16* wr = w1 + (int64_t)(warp * 32 + j * 8 + gr) * kD0 + k0 + 2 * tq;
      mma(acc[j], a, __ldg(reinterpret_cast<const unsigned int*>(wr)),
          __ldg(reinterpret_cast<const unsigned int*>(wr + 8)));
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = warp * 32 + j * 8 + 2 * tq;
    const float bb0 = to_f(b1[c]), bb1 = to_f(b1[c + 1]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = gr + 8 * h;
      const bf16 za = __float2bfloat16_rn(acc[j][2 * h] + bb0), zb = __float2bfloat16_rn(acc[j][2 * h + 1] + bb1);
      if (z1 && r0 + r < n) *reinterpret_cast<uint32_t*>(z1 + (int64_t)(r0 + r) * kD1 + c) = pack2(za, zb);
      sH[r][c] = __float2bfloat16_rn(gelu(to_f(za)));
      sH[r][c + 1] = __float2bfloat16_rn(gelu(to_f(zb)));
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < kRows * O; e += kThreads) {
    const int r = e / O, o = e % O;
    if (r0 + r >= n) continue;
    float s = 0.0f;
#pragma unroll 16
    for (int k = 0; k < kD1; ++k) s = fmaf(to_f(sH[r][k]), sW2[o][k], s);
    v[(int64_t)(r0 + r) * O + o] = __float2bfloat16_rn(s);
  }
}

// the tail of the backward on kRows rows: da1 = bf16(gv W2) and dz1 = bf16(da1 gelu'(z1)) with thread k owning
// column k; da0 = bf16(dz1 W1) on the tensor cores (warp w: columns 128 w ..); dz0 = bf16(da0 gelu'(z0))
__global__ void __launch_bounds__(kThreads) tail_bwd_kernel(const bf16* __restrict__ gv, int O,
                                                            const bf16* __restrict__ z0, const bf16* __restrict__ z1,
                                                            int n, const bf16* __restrict__ w1,
                                                            const bf16* __restrict__ w2, bf16* __restrict__ dz0,
                                                            bf16* __restrict__ dz1, bf16* __restrict__ a0) {
  __shared__ float sG[kRows][kMaxO];
  __shared__ __align__(16) bf16 sD[kRows][kD1 + 8];
  const int r0 = blockIdx.x * kRows;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, gr = lane >> 2, tq = lane & 3;
  for (int e = threadIdx.x; e < kRows * kMaxO; e += kThreads) {
    const int r = e / kMaxO, o = e % kMaxO;
    sG[r][o] = (r0 + r < n && o < O) ? to_f(gv[(int64_t)(r0 + r) * O + o]) : 0.0f;
  }
  const int k = threadIdx.x;  // kThreads == kD1
  float w2c[kMaxO];
#pragma unroll
  for (int o = 0; o < kMaxO; ++o) w2c[o] = o < O ? to_f(w2[o * kD1 + k]) : 0.0f;
  __syncthreads();
#pragma unroll 4
  for (int r = 0; r < kRows; ++r) {
    float s = 0.0f;
#pragma unroll
    for (int o = 0; o < kMaxO; ++o)
      if (o < O) s = fmaf(sG[r][o], w2c[o], s);
    const bool live = r0 + r < n;
    const float z = live ? to_f(z1[(int64_t)(r0 + r) * kD1 + k]) : 0.0f;
    const bf16 d = __float2bfloat16_rn(gelu_grad(round_bf(s), z));
    sD[r][k] = d;
    if (live) dz1[(int64_t)(r0 + r) * kD1 + k] = d;
  }
  __syncthreads();
  float acc[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0.0f;
#pragma unroll 2
  for (int k0 = 0; k0 < kD1; k0 += 16) {
    uint32_t a[4];
    a[0] = *reinterpret_cast<const uint32_t*>(&sD[gr][k0 + 2 * tq]);
    a[1] = *reinterpret_cast<const uint32_t*>(&sD[gr + 8][k0 + 2 * tq]);
    a[2] = *reinterpret_cast<const uint32_t*>(&sD[gr][k0 + 8 + 2 * tq]);
    a[3] = *reinterpret_cast<const uint32_t*>(&sD[gr + 8][k0 + 8 + 2 * tq]);
    const bf16* wk = w1 + (int64_t)(k0 + 2 * tq) * kD0 + warp * 128 + gr;  // B[k][c] = W1[k][c]
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const bf16* p = wk + j * 8;
      mma(acc[j], a, pack2(p[0], p[kD0]), pack2(p[8 * kD0], p[9 * kD0]));
    }
  }
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int c = warp * 128 + j * 8 + 2 * tq;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + gr + 8 * h;
      if (row >= n) continue;
      const int64_t off = (int64_t)row * kD0 + c;
      const __nv_bfloat162 z = *reinterpret_cast<const __nv_bfloat162*>(z0 + off);
      const float za = __low2float(z), zb = __high2float(z);
      *reinterpret_cast<uint32_t*>(dz0 + off) =
          pack2(__float2bfloat16_rn(gelu_grad(round_bf(acc[j][2 * h]), za)),
                __float2bfloat16_rn(gelu_grad(round_bf(acc[j][2 * h + 1]), zb)));
      if (a0) *reinterpret_cast<uint32_t*>(a0 + off) = pack2(__float2bfloat16_rn(gelu(za)), __float2bfloat16_rn(gelu(zb)));
    }
  }
}

// C = bf16(A B) for up to two problems in one launch (blockIdx.x walks g0's tiles, then g1's); every k-block of a
// tile in order in one CTA
template <bool AT, bool BT>
__global__ void __launch_bounds__(kThreads) gemm_kernel(Gemm g0, Gemm g1) {
  __shared__ __align__(16) unsigned char smem[kSmemBytes];
  int t = blockIdx.x;
  const bool second = t >= g0.tiles;
  const Gemm g = second ? g1 : g0;
  if (second) t -= g0.tiles;
  const int m0 = (t / g.tiles_n) * kBM, n0 = (t % g.tiles_n) * kBN;
  float acc[2][8][4];
  mainloop<AT, BT>(acc, reinterpret_cast<bf16*>(smem), g, m0, n0, 0, (g.K + kBK - 1) / kBK);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wm = (warp & 1) * 32, wn = (warp >> 1) * 64;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 8; ++ni) {
      const int c = n0 + wn + ni * 8 + (lane & 3) * 2;
      if (c >= g.N) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = m0 + wm + mi * 16 + (lane >> 2) + 8 * h;
        if (r < g.M)
          *reinterpret_cast<uint32_t*>(g.c + (int64_t)r * g.ldc + c) =
              pack2(__float2bfloat16_rn(acc[mi][ni][2 * h]), __float2bfloat16_rn(acc[mi][ni][2 * h + 1]));
      }
    }
}

// 32 output columns per CTA: [0, 512) db0, [512, 640) db1, then dW2 flattened as o 128 + k.  Warp w adds rows
// w, w + 8, ... in order; warp 0 adds the eight warp sums in order.
__global__ void __launch_bounds__(kSmallWarps * 32) small_grads_kernel(const bf16* __restrict__ dz0,
                                                                       const bf16* __restrict__ dz1,
                                                                       const bf16* __restrict__ gv, int O,
                                                                       const bf16* __restrict__ z1, int n,
                                                                       bf16* __restrict__ db0, bf16* __restrict__ db1,
                                                                       bf16* __restrict__ dw2) {
  __shared__ float red[kSmallWarps][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + lane;
  const int kind = blockIdx.x < kD0 / 32 ? 0 : blockIdx.x < (kD0 + kD1) / 32 ? 1 : 2;
  bf16* out = kind == 0 ? db0 : kind == 1 ? db1 : dw2;
  if (!out) return;
  float acc = 0.0f;
  if (kind == 0) {
#pragma unroll 4
    for (int i = warp; i < n; i += kSmallWarps) acc += to_f(dz0[(int64_t)i * kD0 + col]);
  } else if (kind == 1) {
    const int c = col - kD0;
#pragma unroll 4
    for (int i = warp; i < n; i += kSmallWarps) acc += to_f(dz1[(int64_t)i * kD1 + c]);
  } else {
    const int o = (col - kD0 - kD1) / kD1, c = (col - kD0 - kD1) % kD1;
#pragma unroll 4
    for (int i = warp; i < n; i += kSmallWarps)
      acc = fmaf(to_f(gv[(int64_t)i * O + o]), round_bf(gelu(to_f(z1[(int64_t)i * kD1 + c]))), acc);
  }
  red[warp][lane] = acc;
  __syncthreads();
  if (warp == 0) {
    float s = red[0][lane];
#pragma unroll
    for (int w = 1; w < kSmallWarps; ++w) s += red[w][lane];
    out[col - (kind == 0 ? 0 : kind == 1 ? kD0 : kD0 + kD1)] = __float2bfloat16_rn(s);
  }
}

bool bad_h(int64_t H) { return H % 64 != 0 || H < 64 || H > 8192; }
bool misaligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }
constexpr int64_t kMaxRows = 0x7fffffff - kBM;

Gemm gemm(const bf16* a, int64_t lda, const bf16* b, int64_t ldb, bf16* c, int64_t ldc, int M, int N, int K) {
  const int tn = (N + kBN - 1) / kBN;
  return Gemm{a, lda, b, ldb, c, ldc, M, N, K, tn, tn * ((M + kBM - 1) / kBM)};
}

}  // namespace

extern "C" int64_t rb200_vla_value_head_workspace_bytes(int64_t n, int64_t H) {
  if (n < 0 || n > kMaxRows || bad_h(H)) return -1;
  return n * (kD0 + kD1 + kD0) * 2;
}

extern "C" int rb200_vla_value_head_fwd(const void* x, int64_t row_stride, int64_t n, int64_t H, const void* w0,
                                        const void* b0, const void* w1, const void* b1, const void* w2, int O, void* z0,
                                        void* z1, void* v, rb200_stream_t stream) {
  if (!x || !w0 || !b0 || !w1 || !b1 || !w2 || !z0 || !v) return RB200_E_NULL;
  if (n < 0 || n > kMaxRows || bad_h(H) || row_stride < H || O < 1 || O > kMaxO) return RB200_E_SHAPE;
  if (misaligned(x) || misaligned(w0) || misaligned(w1) || misaligned(z0) || (z1 && misaligned(z1)) ||
      row_stride % 8 != 0)
    return RB200_E_ALIGN;
  if (n == 0) return RB200_OK;
  cudaStream_t st = rb::as_stream(stream);
  const dim3 grid((unsigned)((n + kBM - 1) / kBM), kD0 / kBN, kSplit);
  l0_fwd_kernel<<<grid, kThreads, 0, st>>>(static_cast<const bf16*>(x), row_stride, (int)n, (int)H,
                                           static_cast<const bf16*>(w0), static_cast<const bf16*>(b0),
                                           static_cast<bf16*>(z0));
  rb::count_launch();
  tail_fwd_kernel<<<(unsigned)((n + kRows - 1) / kRows), kThreads, 0, st>>>(
      static_cast<const bf16*>(z0), (int)n, static_cast<const bf16*>(w1), static_cast<const bf16*>(b1),
      static_cast<const bf16*>(w2), O, static_cast<bf16*>(z1), static_cast<bf16*>(v));
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_vla_value_head_bwd(const void* x, int64_t row_stride, int64_t n, int64_t H, const void* w0,
                                        const void* w1, const void* w2, int O, const void* z0, const void* z1,
                                        const void* gv, void* dx, void* dw0, void* db0, void* dw1, void* db1,
                                        void* dw2, void* workspace, int64_t workspace_bytes, rb200_stream_t stream) {
  if (!dx && !dw0 && !db0 && !dw1 && !db1 && !dw2) return RB200_E_NULL;
  if (!w1 || !w2 || !z0 || !z1 || !gv || !workspace || (dx && !w0) || (dw0 && !x)) return RB200_E_NULL;
  if (n < 0 || n > kMaxRows || bad_h(H) || O < 1 || O > kMaxO || (dw0 && row_stride < H)) return RB200_E_SHAPE;
  if (workspace_bytes < rb200_vla_value_head_workspace_bytes(n, H)) return RB200_E_ARG;
  if (misaligned(z0) || misaligned(z1) || misaligned(workspace) || (dx && (misaligned(dx) || misaligned(w0))) ||
      (dw0 && (misaligned(dw0) || misaligned(x) || row_stride % 8 != 0)) || (dw1 && misaligned(dw1)))
    return RB200_E_ALIGN;
  cudaStream_t st = rb::as_stream(stream);
  const int N = (int)n;
  bf16* wdz0 = static_cast<bf16*>(workspace);
  bf16* wdz1 = wdz0 + n * kD0;
  bf16* wa0 = wdz1 + n * kD1;
  const bf16* gvb = static_cast<const bf16*>(gv);
  if (N > 0) {
    tail_bwd_kernel<<<(unsigned)((n + kRows - 1) / kRows), kThreads, 0, st>>>(
        gvb, O, static_cast<const bf16*>(z0), static_cast<const bf16*>(z1), N, static_cast<const bf16*>(w1),
        static_cast<const bf16*>(w2), wdz0, wdz1, dw1 ? wa0 : nullptr);
    rb::count_launch();
  }
  if (dx && N > 0) {
    const Gemm g = gemm(wdz0, kD0, static_cast<const bf16*>(w0), H, static_cast<bf16*>(dx), H, N, (int)H, kD0);
    const Gemm none{};
    gemm_kernel<false, true><<<(unsigned)g.tiles, kThreads, 0, st>>>(g, none);
    rb::count_launch();
  }
  if (dw0 || dw1) {  // K = n; n = 0 writes the empty sums' zeros
    const Gemm gw0 = dw0 ? gemm(wdz0, kD0, static_cast<const bf16*>(x), row_stride, static_cast<bf16*>(dw0), H, kD0,
                                (int)H, N)
                         : Gemm{};
    const Gemm gw1 = dw1 ? gemm(wdz1, kD1, wa0, kD0, static_cast<bf16*>(dw1), kD0, kD1, kD0, N) : Gemm{};
    const Gemm first = dw0 ? gw0 : gw1, second = dw0 ? gw1 : Gemm{};
    gemm_kernel<true, true><<<(unsigned)(first.tiles + second.tiles), kThreads, 0, st>>>(first, second);
    rb::count_launch();
  }
  if (db0 || db1 || dw2) {
    small_grads_kernel<<<(unsigned)((kD0 + kD1 + O * kD1) / 32), kSmallWarps * 32, 0, st>>>(
        wdz0, wdz1, gvb, O, static_cast<const bf16*>(z1), N, static_cast<bf16*>(db0), static_cast<bf16*>(db1),
        static_cast<bf16*>(dw2));
    rb::count_launch();
  }
  RB_RETURN_LAUNCH();
}
