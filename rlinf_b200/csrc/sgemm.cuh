// fp32 SIMT GEMM (exact fp32 FMA accumulation) for the MLP towers' layer 0 where the tensor-core kernels do not take
// the shape (row gather, obs % 32 != 0, obs > 256 in the weight gradient) and for the synthetic env.
// C[M,N] = epilogue( sum_k A(m,k) * B(k,n) ), 128x128x8 tiles, 256 threads, 8x8 micro-tile per thread,
// register-prefetched double-buffered shared memory.  Operand layouts are template parameters so the same
// kernel serves the forward (X.W^T) and the weight gradient (dZ^T.X, split over the sample axis: one stored partial per
// split that the caller sums in split order).
#pragma once
#include "common.cuh"

namespace rb {
namespace gemm {

constexpr int BM = 128, BN = 128, BK = 8, NT = 256;

enum AMode { A_KCONTIG = 0, A_MCONTIG = 1 };  // A(m,k) stored [M,K] (k fastest) or [K,M] (m fastest)
enum BMode { B_KCONTIG = 0, B_NCONTIG = 1 };  // B(k,n) stored [N,K] (k fastest) or [K,N] (n fastest)
enum Epi { EPI_BIAS_TANH = 0, EPI_STORE = 1 };

struct GemmArgs {
  const float* A;
  const float* B;
  float* C;
  const int64_t* a_rows;  // optional row gather for A (A_KCONTIG) or for B rows r (wgrad layer 0: B_NCONTIG rows)
  const int64_t* b_rows;
  const float* bias;  // [N]          (EPI_BIAS_TANH)
  int64_t M;          // rows of C; for the wgrad form this is N_out and K is the (huge) reduction over samples
  int N, lda, ldb, ldc;
  int64_t K;
  int64_t k_per_split;  // reduction range per blockIdx.z
  int64_t c_split_stride;  // EPI_STORE: split z writes its partial to C + z * c_split_stride (0: all splits share C)
};

__device__ __forceinline__ float4 ld4(const float* p, bool vec, int valid) {
  // loads p[0..3]; `valid` = number of in-range elements (0..4); vec => 16-byte aligned & all valid
  if (vec) return *reinterpret_cast<const float4*>(p);
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  if (valid > 0) r.x = p[0];
  if (valid > 1) r.y = p[1];
  if (valid > 2) r.z = p[2];
  if (valid > 3) r.w = p[3];
  return r;
}

template <int AM, int BMODE, int EPI>
__global__ void __launch_bounds__(NT) sgemm_kernel(GemmArgs p) {
  __shared__ __align__(16) float As[2][BK][BM];
  __shared__ __align__(16) float Bs[2][BK][BN];
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int64_t kbeg = (int64_t)blockIdx.z * p.k_per_split;
  const int64_t kend = (kbeg + p.k_per_split < p.K) ? kbeg + p.k_per_split : p.K;
  const int tx = tid & 15, ty = tid >> 4;

  // ---- tile load plans (one float4 per thread per tile) ----
  // KCONTIG: 128 rows x 8 k -> thread: row = tid/2, kq = (tid&1)*4 ; stored transposed
  // M/N CONTIG: 8 k x 128 cols -> thread: kk = tid/32, cq = (tid&31)*4 ; stored directly
  const int a_row = (AM == A_KCONTIG) ? (tid >> 1) : ((tid & 31) * 4);
  const int a_k = (AM == A_KCONTIG) ? ((tid & 1) * 4) : (tid >> 5);
  const int b_col = (BMODE == B_KCONTIG) ? (tid >> 1) : ((tid & 31) * 4);
  const int b_k = (BMODE == B_KCONTIG) ? ((tid & 1) * 4) : (tid >> 5);

  const bool a_vec_ok = ((p.lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.A) & 15) == 0);
  const bool b_vec_ok = ((p.ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.B) & 15) == 0);

  const float* a_ptr = nullptr;  // A_KCONTIG: row base pointer (fixed over k)
  bool a_row_ok = false;
  if (AM == A_KCONTIG) {
    const int64_t m = m0 + a_row;
    a_row_ok = m < p.M;
    if (a_row_ok) a_ptr = p.A + (p.a_rows ? p.a_rows[m] : m) * p.lda;
  }
  const float* b_ptr = nullptr;
  bool b_col_ok = false;
  if (BMODE == B_KCONTIG) {
    const int n = n0 + b_col;
    b_col_ok = n < p.N;
    if (b_col_ok) b_ptr = p.B + (int64_t)n * p.ldb;
  }

  auto load_a = [&](int64_t k0) -> float4 {
    if (AM == A_KCONTIG) {
      const int64_t k = k0 + a_k;
      if (!a_row_ok || k >= kend) return make_float4(0.f, 0.f, 0.f, 0.f);
      const int valid = (int)((kend - k) < 4 ? (kend - k) : 4);
      return ld4(a_ptr + k, a_vec_ok && valid == 4, valid);
    } else {  // A(m,k) = A[k*lda + m], m fastest. k is the reduction index (sample row for wgrad)
      const int64_t k = k0 + a_k;
      const int64_t m = m0 + a_row;
      if (k >= kend || m >= p.M) return make_float4(0.f, 0.f, 0.f, 0.f);
      const int64_t src = p.a_rows ? p.a_rows[k] : k;
      const int valid = (int)((p.M - m) < 4 ? (p.M - m) : 4);
      return ld4(p.A + src * p.lda + m, a_vec_ok && valid == 4, valid);
    }
  };
  auto load_b = [&](int64_t k0) -> float4 {
    if (BMODE == B_KCONTIG) {
      const int64_t k = k0 + b_k;
      if (!b_col_ok || k >= kend) return make_float4(0.f, 0.f, 0.f, 0.f);
      const int valid = (int)((kend - k) < 4 ? (kend - k) : 4);
      return ld4(b_ptr + k, b_vec_ok && valid == 4, valid);
    } else {  // B(k,n) = B[k*ldb + n]
      const int64_t k = k0 + b_k;
      const int n = n0 + b_col;
      if (k >= kend || n >= p.N) return make_float4(0.f, 0.f, 0.f, 0.f);
      const int64_t src = p.b_rows ? p.b_rows[k] : k;
      const int valid = (p.N - n) < 4 ? (p.N - n) : 4;
      return ld4(p.B + src * p.ldb + n, b_vec_ok && valid == 4, valid);
    }
  };
  auto store_a = [&](int buf, float4 v) {
    if (AM == A_KCONTIG) {
      As[buf][a_k + 0][a_row] = v.x;
      As[buf][a_k + 1][a_row] = v.y;
      As[buf][a_k + 2][a_row] = v.z;
      As[buf][a_k + 3][a_row] = v.w;
    } else {
      *reinterpret_cast<float4*>(&As[buf][a_k][a_row]) = v;
    }
  };
  auto store_b = [&](int buf, float4 v) {
    if (BMODE == B_KCONTIG) {
      Bs[buf][b_k + 0][b_col] = v.x;
      Bs[buf][b_k + 1][b_col] = v.y;
      Bs[buf][b_k + 2][b_col] = v.z;
      Bs[buf][b_k + 3][b_col] = v.w;
    } else {
      *reinterpret_cast<float4*>(&Bs[buf][b_k][b_col]) = v;
    }
  };

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra = load_a(kbeg), rb_ = load_b(kbeg);
  store_a(0, ra);
  store_b(0, rb_);
  __syncthreads();
  int buf = 0;
  for (int64_t k0 = kbeg; k0 < kend; k0 += BK) {
    const bool has_next = (k0 + BK) < kend;
    if (has_next) {
      ra = load_a(k0 + BK);
      rb_ = load_b(k0 + BK);
    }
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (has_next) {
      store_a(buf ^ 1, ra);
      store_b(buf ^ 1, rb_);
      __syncthreads();
      buf ^= 1;
    }
  }

  // ---- epilogue ----
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= p.M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + (jh == 0 ? tx * 4 : 64 + tx * 4);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (n + j >= p.N) continue;
        const float v = acc[i][jh * 4 + j];
        p.C[blockIdx.z * p.c_split_stride + m * p.ldc + n + j] = EPI == EPI_BIAS_TANH ? tanhf(v + p.bias[n + j]) : v;
      }
    }
  }
}

template <int AM, int BMODE, int EPI>
int launch_gemm(const GemmArgs& p, int splits, cudaStream_t st) {
  dim3 grid((unsigned)((p.M + BM - 1) / BM), (unsigned)((p.N + BN - 1) / BN), (unsigned)splits);
  sgemm_kernel<AM, BMODE, EPI><<<grid, NT, 0, st>>>(p); rb::count_launch();
  cudaError_t e = cudaPeekAtLastError();
  return e == cudaSuccess ? 0 : (int)e;
}


}  // namespace gemm
}  // namespace rb
