// Stand-alone probe: how fast can one strip-per-CTA kernel pull a [T,B] step-major tensor through TMA / LDG?
// (Used to find what bounds the GAE kernel; build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o
//  tools/tma_probe tools/tma_probe.cu ; run on the GPU box.)
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x)                                                                        \
  do {                                                                               \
    cudaError_t e_ = (x);                                                            \
    if (e_ != cudaSuccess) {                                                         \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      fflush(stdout);                                                                \
      exit(1);                                                                       \
    }                                                                                \
  } while (0)

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint64_t* b, uint32_t c) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(c) : "memory");
}
__device__ __forceinline__ void mb_expect(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory");
}
__device__ __forceinline__ void mb_wait(uint64_t* b, uint32_t ph) {
  uint32_t ok = 0, spins = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(s32(b)), "r"(ph)
        : "memory");
    if (++spins > (1u << 26)) __trap();
  }
}
__device__ __forceinline__ void tma_ld(void* dst, const CUtensorMap* m, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          s32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(s32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// Each CTA: strip = blockIdx.x % n_strips (box_w columns), segment = blockIdx.x / n_strips (seg_rows rows, walked
// BACKWARDS in tiles of box_h rows like the GAE scan).  narr arrays are read per tile (row bases arr*arr_rows).
__global__ void __launch_bounds__(64) tma_pull(const __grid_constant__ CUtensorMap tm, int n_strips, int seg_rows,
                                               int box_w, int box_h, int esize, int stages, int narr, int arr_rows,
                                               int row_base, float* sink) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (s32(smem_raw) & 1023u)) & 1023u);
  __shared__ uint64_t full[16], empty[16];
  const int strip = blockIdx.x % n_strips, seg = blockIdx.x / n_strips;
  const int tile_bytes = box_w * box_h * esize;
  const int stage_bytes = ((tile_bytes * narr + 1023) / 1024) * 1024;
  const int n_iter = seg_rows / box_h;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mb_init(&full[s], 1);
      mb_init(&empty[s], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int it = 0; it < n_iter; ++it) {
      const int s = it % stages;
      if (it >= stages) mb_wait(&empty[s], ((it / stages) - 1) & 1);
      mb_expect(&full[s], tile_bytes * narr);
      const int t0 = row_base + seg * seg_rows + seg_rows - (it + 1) * box_h;
      for (int a = 0; a < narr; ++a)
        tma_ld(smem + s * stage_bytes + a * tile_bytes, &tm, strip * box_w, a * arr_rows + t0, &full[s]);
    }
  } else if (threadIdx.x == 32) {
    float acc = 0.f;
    for (int it = 0; it < n_iter; ++it) {
      const int s = it % stages;
      mb_wait(&full[s], (it / stages) & 1);
      acc += *reinterpret_cast<volatile float*>(smem + s * stage_bytes);
      mb_arrive(&empty[s]);
    }
    if (acc == 123.456f) sink[0] = acc;
  }
}

// LDG version: 4 warps, lane -> column (float) or 16-B vector; each warp walks rows with stride 4, unroll 8.
template <int VEC>
__global__ void __launch_bounds__(128) ldg_pull(const float* __restrict__ base, int B, int n_strips, int seg_rows,
                                                int narr, int arr_rows, int row_base, float* sink) {
  const int strip = blockIdx.x % n_strips, seg = blockIdx.x / n_strips;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc = 0.f;
  const int col = strip * 32 * VEC + lane * VEC;
  for (int a = 0; a < narr; ++a) {
    const float* p = base + (size_t)(a * arr_rows + row_base + seg * seg_rows) * B + col;
#pragma unroll 8
    for (int r = seg_rows - 1 - warp; r >= 0; r -= 4) {
      if (VEC == 1) acc += __ldg(p + (size_t)r * B);
      else {
        float4 v = __ldg(reinterpret_cast<const float4*>(p + (size_t)r * B));
        acc += v.x + v.y + v.z + v.w;
      }
    }
  }
  if (acc == 123.456f) sink[0] = acc;
}

static PFN_cuTensorMapEncodeTiled_v12000 get_enc() {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
  return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
}

int main() {
  const int T = 512, B = 4096, NBUF = 20;  // 20 x 8 MB x narr(<=3) > L2
  const size_t rows_total = (size_t)NBUF * T * 3;
  float* buf;
  CK(cudaMalloc(&buf, rows_total * B * 4));
  CK(cudaMemset(buf, 0, rows_total * B * 4));
  float* sink;
  CK(cudaMalloc(&sink, 4));
  auto enc = get_enc();
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  CK(cudaFuncSetAttribute(tma_pull, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));

  struct V {
    const char* name;
    int esize, box_w, box_h, stages, narr, segs, promo;
  };
  // promo: 0 none, 1 = 64B, 2 = 128B, 3 = 256B
  V vs[] = {
      {"f32 32x64 st4 narr3 (GAE v3 shape)", 4, 32, 64, 4, 3, 1, 2},
      {"f32 32x64 st4 narr1", 4, 32, 64, 4, 1, 1, 2},
      {"f32 32x64 st8 narr1", 4, 32, 64, 8, 1, 1, 2},
      {"f32 32x64 st4 narr3 promo256", 4, 32, 64, 4, 3, 1, 3},
      {"f32 32x64 st4 narr3 promo none", 4, 32, 64, 4, 3, 1, 0},
      {"f32 32x16 st8 narr3", 4, 32, 16, 8, 3, 1, 2},
      {"f32 64x32 st4 narr3 (64 strips)", 4, 64, 32, 4, 3, 1, 2},
      {"f32 64x32 st4 narr3 x2 segs", 4, 64, 32, 4, 3, 2, 2},
      {"f32 128x16 st4 narr3 x4 segs", 4, 128, 16, 4, 3, 4, 2},
      {"f32 32x64 st4 narr3 x2 segs (256 CTAs)", 4, 32, 64, 2, 3, 2, 2},
      {"f32 32x32 st3 narr3 x4 segs (512 CTAs)", 4, 32, 32, 2, 3, 4, 2},
      {"u8 32x64 st4 narr1", 1, 32, 64, 4, 1, 1, 2},
      {"u8 128x64 st4 narr1", 1, 128, 64, 4, 1, 1, 2},
  };
  for (const V& v : vs) {
    // the tensor is viewed as [rows_total, B] of esize-byte elements over the same allocation
    CUtensorMap tm;
    cuuint64_t gdim[2] = {(cuuint64_t)B, (cuuint64_t)rows_total};
    cuuint64_t gstr[1] = {(cuuint64_t)B * v.esize};
    cuuint32_t box[2] = {(cuuint32_t)v.box_w, (cuuint32_t)v.box_h};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&tm, v.esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, buf, gdim,
                     gstr, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                     (CUtensorMapL2promotion)v.promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      printf("%s: encode failed %d\n", v.name, (int)r);
      continue;
    }
    const int n_strips = B / v.box_w;
    const int grid = n_strips * v.segs;
    const int seg_rows = T / v.segs;
    const int tile_bytes = v.box_w * v.box_h * v.esize;
    const int smem = ((tile_bytes * v.narr + 1023) / 1024) * 1024 * v.stages + 1024;
    float ms_best = 1e9f;
    for (int rep = 0; rep < 3; ++rep) {
      CK(cudaEventRecord(e0));
      for (int i = 0; i < NBUF; ++i)
        tma_pull<<<grid, 64, smem>>>(tm, n_strips, seg_rows, v.box_w, v.box_h, v.esize, v.stages, v.narr, NBUF * T,
                                     i * T, sink);
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      CK(cudaGetLastError());
      float ms;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      if (ms < ms_best) ms_best = ms;
    }
    const double bytes = (double)T * B * v.esize * v.narr;
    printf("TMA %-44s grid %4d smem %6d: %7.2f us/launch  %7.1f GB/s\n", v.name, grid, smem, ms_best * 1e3 / NBUF,
           bytes / (ms_best * 1e-3 / NBUF) / 1e9);
    fflush(stdout);
  }
  // LDG variants
  for (int vec = 1; vec <= 4; vec += 3)
    for (int segs = 1; segs <= 4; segs *= 2)
      for (int narr = 1; narr <= 3; narr += 2) {
        const int n_strips = B / (32 * vec);
        const int grid = n_strips * segs;
        float ms_best = 1e9f;
        for (int rep = 0; rep < 3; ++rep) {
          CK(cudaEventRecord(e0));
          for (int i = 0; i < NBUF; ++i) {
            if (vec == 1) ldg_pull<1><<<grid, 128>>>(buf, B, n_strips, T / segs, narr, NBUF * T, i * T, sink);
            else ldg_pull<4><<<grid, 128>>>(buf, B, n_strips, T / segs, narr, NBUF * T, i * T, sink);
          }
          CK(cudaEventRecord(e1));
          CK(cudaEventSynchronize(e1));
          CK(cudaGetLastError());
          float ms;
          CK(cudaEventElapsedTime(&ms, e0, e1));
          if (ms < ms_best) ms_best = ms;
        }
        const double bytes = (double)T * B * 4 * narr;
        printf("LDG vec%d narr%d segs%d grid %4d: %7.2f us/launch  %7.1f GB/s\n", vec, narr, segs, grid,
               ms_best * 1e3 / NBUF, bytes / (ms_best * 1e-3 / NBUF) / 1e9);
        fflush(stdout);
      }
  return 0;
}
