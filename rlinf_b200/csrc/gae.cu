// K1: GAE reverse scan over [T,B] trajectories + normalisation statistics; normalise kernel.
// Reference: compute_gae_advantages_and_returns, rlinf/algorithms/advantages.py:24-86 (a Python
// loop of T iterations x ~8 eager CPU ops) and safe_normalize, rlinf/algorithms/utils.py:397-404.
//
// Parity contract: adv/ret are BIT-IDENTICAL to the reference's fp32 arithmetic.  The recurrence
//     nd = !done[t+1];  delta = (r[t] + (gamma*V[t+1])*nd) - V[t]
//     g  = delta + ((gamma*lambda)*nd) * g;   ret[t] = g + V[t];   adv[t] = ret[t] - V[t]
// rounds after every op (no FMA contraction: __fmul_rn/__fadd_rn) and is evaluated in the
// reference's sequential order.  fp32 addition is not associative, so a re-associated parallel scan
// over T cannot be bit-exact; instead each trajectory's chain runs sequentially (2 dependent fp32 ops
// per step ~ 9 cycles -> ~2.5 us for T=512, below the HBM time of the tile) and the memory-level
// parallelism comes from TMA: one elected thread streams [R x 32] tiles of rewards / values / dones
// (/ mask) through an S-stage mbarrier ring in shared memory, newest timestep first.
//
// HBM traffic (algorithmic): r 4 + V 4 + done 1 (+ mask 1) read, adv 4 + ret 4 written = 17 B/step.
#include <type_traits>

#include "common.cuh"
#include "tma.cuh"

namespace {

constexpr int kW = 32;  // trajectories (columns) per CTA = one warp

// Statistics accumulator: fp32 partial sums over one tile of <= 16 values, folded into fp64 totals once per
// tile (keeps the fp64 pipe and the F2F conversions out of the per-row instruction stream).
struct Acc {
  double s = 0, ss = 0;
  float ts = 0.f, tss = 0.f;
  int n = 0;
  __device__ __forceinline__ void add(float x) {
    n += 1;
    ts += x;
    tss = fmaf(x, x, tss);
  }
  __device__ __forceinline__ void fold() {
    s += (double)ts;
    ss += (double)tss;
    ts = 0.f;
    tss = 0.f;
  }
};

// One step of the recurrence for one trajectory. Kept in one place so both kernels round identically.
template <bool HAS_V>
__device__ __forceinline__ void gae_step(float r, float vt, float v_next, uint8_t done_next, float gamma,
                                         float coef, float& g, float& ret, float& adv) {
  const float nd = done_next ? 0.0f : 1.0f;
  float delta;
  if (HAS_V) {
    const float boot = __fmul_rn(__fmul_rn(gamma, v_next), nd);
    delta = __fsub_rn(__fadd_rn(r, boot), vt);
  } else {
    delta = r;
  }
  g = __fadd_rn(delta, __fmul_rn(__fmul_rn(coef, nd), g));
  if (HAS_V) {
    ret = __fadd_rn(g, vt);
    adv = __fsub_rn(ret, vt);
  } else {
    ret = g;
    adv = g;
  }
}

__device__ __forceinline__ void flush_stats(const Acc& a, const Acc& r, double* stats) {
  double v[6] = {(double)a.n, a.s, a.ss, (double)r.n, r.s, r.ss};
#pragma unroll
  for (int k = 0; k < 6; ++k) v[k] = rb::warp_sum(v[k]);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 6; ++k)
      if (v[k] != 0.0) atomicAdd(&stats[k], v[k]);
  }
}

// ---------------------------------------------------------------------------------------------
// TMA-pipelined, warp-specialised kernel. One CTA per 32 trajectories, 10 warps:
//   warp 0      producer : one thread streams [64 steps x 32 traj] tiles (rewards, values(+1 row), dones, mask) with TMA
//   warps 1-4   delta    : delta_t and the recurrence coefficient c_t = (gamma*lambda)*!done  (no dependence on g)
//   warp 5      chain    : g_t = delta_t + c_t * g_{t+1}, strictly sequential, 2 dependent fp32 ops per step
//   warps 6-9   epilogue : ret = g + V, adv = ret - V staged in smem, statistics, TMA tile stores
// A single warp doing all of this is issue-bound (~107 cycles / step); splitting the work
// that does not depend on the carry across warps leaves ~9 cycles / step on the sequential warp.
// Stage hand-off: full (TMA) -> dready (delta warps) -> gready (chain) -> empty (epilogue), all mbarriers.
// Requires B % 16 == 0 (16-byte global strides for the byte tensors) and 16-byte aligned bases.
// ---------------------------------------------------------------------------------------------
// Box size: small [16 x 32] boxes pay a per-box overhead (tools/tma_probe.cu), hence 64 steps per stage.  The loads are
// NOT what bounds this kernel; the epilogue warps were - see the comment there.
constexpr int kRW = 64;       // timesteps per TMA stage
constexpr int kStagesWS = 4;  // 4 x 44.4 KB
struct __align__(128) StageWS {
  float r[kRW][kW];
  float v[kRW + 1][kW];    // rows t0 .. t0+64 (the extra row is V[t+1] of the tile's last step)
  uint8_t d[kRW][kW];      // done AFTER step t (rows t0+1 .. t0+64 of dones)
  uint8_t m[kRW][kW];
  float2 dc[kRW][kW];      // {delta_t, c_t}
  float g[kRW][kW];
};
constexpr int kDW = 4;                  // delta warps
constexpr int kEW = 4;                  // epilogue warps
constexpr uint32_t kWsThreads = 32 * (1 + kDW + 1 + kEW);  // producer + delta + chain + epilogue = 320

template <bool HAS_V, bool HAS_MASK, bool HAS_STATS>
__global__ void __launch_bounds__(kWsThreads) gae_tma_kernel(const __grid_constant__ CUtensorMap tm_r,
                                                             const __grid_constant__ CUtensorMap tm_v,
                                                             const __grid_constant__ CUtensorMap tm_d,
                                                             const __grid_constant__ CUtensorMap tm_m,
                                                             const __grid_constant__ CUtensorMap tm_adv,
                                                             const __grid_constant__ CUtensorMap tm_ret,
                                                             float* __restrict__ adv, float* __restrict__ ret,
                                                             double* __restrict__ stats, int T, int B, float gamma,
                                                             float coef) {
  extern __shared__ uint8_t smem_raw[];
  // pointer arithmetic without an integer round trip keeps the shared address space (LDS/STS, not generic LD/ST)
  StageWS* stages = reinterpret_cast<StageWS*>(smem_raw + ((128u - (rb::tma::smem_u32(smem_raw) & 127u)) & 127u));
  __shared__ __align__(8) uint64_t full_bar[kStagesWS], dready_bar[kStagesWS], gready_bar[kStagesWS],
      empty_bar[kStagesWS];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col0 = blockIdx.x * kW;
  const int n_iter = (T + kRW - 1) / kRW;

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStagesWS; ++s) {
      rb::tma::mbar_init(&full_bar[s], 1);
      rb::tma::mbar_init(&dready_bar[s], kDW);
      rb::tma::mbar_init(&gready_bar[s], 1);
      rb::tma::mbar_init(&empty_bar[s], 1);  // the epilogue warp that issued the tile's TMA stores
    }
    rb::tma::fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      rb::tma::prefetch_desc(&tm_r);
      rb::tma::prefetch_desc(&tm_d);
      if (HAS_V) rb::tma::prefetch_desc(&tm_v);
      if (HAS_MASK) rb::tma::prefetch_desc(&tm_m);
      constexpr uint32_t kBytes = sizeof(float) * kRW * kW + (HAS_V ? sizeof(float) * (kRW + 1) * kW : 0) + kRW * kW +
                                  (HAS_MASK ? kRW * kW : 0);
      for (int it = 0; it < n_iter; ++it) {
        const int s = it % kStagesWS;
        const uint32_t ph = (uint32_t)(it / kStagesWS) & 1u;
        rb::tma::mbar_wait(&empty_bar[s], ph ^ 1u);
        const int t0 = T - (it + 1) * kRW;  // may be negative on the last tile: OOB rows are zero-filled
        rb::tma::mbar_arrive_expect_tx(&full_bar[s], kBytes);
        rb::tma::load_2d(&stages[s].r[0][0], &tm_r, col0, t0, &full_bar[s]);
        if (HAS_V) rb::tma::load_2d(&stages[s].v[0][0], &tm_v, col0, t0, &full_bar[s]);
        rb::tma::load_2d(&stages[s].d[0][0], &tm_d, col0, t0 + 1, &full_bar[s]);
        if (HAS_MASK) rb::tma::load_2d(&stages[s].m[0][0], &tm_m, col0, t0, &full_bar[s]);
      }
    }
  } else if (warp <= kDW) {
    // ---- delta warps: rows rr = w, w+kDW, ... of every tile ----
    const int w = warp - 1;
    for (int it = 0; it < n_iter; ++it) {
      const int s = it % kStagesWS;
      const uint32_t ph = (uint32_t)(it / kStagesWS) & 1u;
      rb::tma::mbar_wait(&full_bar[s], ph);
      StageWS& st = stages[s];
#pragma unroll 8
      for (int k = 0; k < kRW / kDW; ++k) {
        const int rr = kDW * k + w;
        const float nd = st.d[rr][lane] ? 0.0f : 1.0f;
        float delta;
        if (HAS_V) {
          const float boot = __fmul_rn(__fmul_rn(gamma, st.v[rr + 1][lane]), nd);
          delta = __fsub_rn(__fadd_rn(st.r[rr][lane], boot), st.v[rr][lane]);
        } else {
          delta = st.r[rr][lane];
        }
        st.dc[rr][lane] = make_float2(delta, __fmul_rn(coef, nd));
      }
      __syncwarp();
      if (lane == 0) rb::tma::mbar_arrive(&dready_bar[s]);
    }
  } else if (warp == kDW + 1) {
    // ---- chain warp: the only sequential part ----
    float g = 0.0f;
    for (int it = 0; it < n_iter; ++it) {
      const int s = it % kStagesWS;
      const uint32_t ph = (uint32_t)(it / kStagesWS) & 1u;
      rb::tma::mbar_wait(&dready_bar[s], ph);
      StageWS& st = stages[s];
#pragma unroll 1
      for (int base = kRW - 16; base >= 0; base -= 16) {  // 16 steps at a time: loads hoisted above the chain
        float2 dc[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) dc[k] = st.dc[base + k][lane];
#pragma unroll
        for (int k = 15; k >= 0; --k) {
          g = __fadd_rn(dc[k].x, __fmul_rn(dc[k].y, g));
          st.g[base + k][lane] = g;
        }
      }
      __syncwarp();
      if (lane == 0) rb::tma::mbar_arrive(&gready_bar[s]);
    }
  } else {
    // ---- epilogue warps: warp e owns rows [16e, 16e+16) of every tile ----
    // Round-1 measurements behind this shape: (1) per-row global stores cost ~45-90 issue cycles per warp
    // instruction (time of v1-v3 == #STG per warp x ~60 cycles), so results are staged in shared memory (ret in
    // place of g, adv in the dead delta/coef buffer) and leave as two TMA tile stores per 64-step tile; (2) with the
    // stores gone the epilogue was issue-bound (~37 instructions per step on ONE warp per tile), hence 4 warps per
    // tile and a branch-free statistics path.
    const int e = warp - (kDW + 2);
    const int col = col0 + lane;
    const bool in_range = col < B;
    Acc acc_a, acc_r;
    int rows_done = 0;
    if (e == 0 && lane == 0) {
      rb::tma::prefetch_desc(&tm_adv);
      rb::tma::prefetch_desc(&tm_ret);
    }
    constexpr int kRE = kRW / kEW;
    for (int it = 0; it < n_iter; ++it) {
      const int s = it % kStagesWS;
      const uint32_t ph = (uint32_t)(it / kStagesWS) & 1u;
      const int t0 = T - (it + 1) * kRW;
      rb::tma::mbar_wait(&gready_bar[s], ph);
      StageWS& st = stages[s];
      float (*adv_s)[kW] = reinterpret_cast<float (*)[kW]>(&st.dc[0][0]);  // [kRW][32] floats, 8 KB of the 16 KB
      if (t0 >= 0) {
#pragma unroll
        for (int k = 0; k < kRE; ++k) {
          const int rr = e * kRE + k;
          const float g = st.g[rr][lane];
          float rt, ad;
          if (HAS_V) {
            const float vt = st.v[rr][lane];
            rt = __fadd_rn(g, vt);
            ad = __fsub_rn(rt, vt);
            st.g[rr][lane] = rt;
          } else {
            rt = g;
            ad = g;
          }
          adv_s[rr][lane] = ad;
          if (HAS_STATS) {
            if (HAS_MASK) {
              const bool valid = st.m[rr][lane] != 0;
              acc_a.n += valid ? 1 : 0;
              const float am = valid ? ad : 0.0f, rm = valid ? rt : 0.0f;
              acc_a.ts += am;
              acc_a.tss = fmaf(am, am, acc_a.tss);
              acc_r.ts += rm;
              acc_r.tss = fmaf(rm, rm, acc_r.tss);
            } else {  // OOB columns were zero-filled by TMA: they add exact zeros, the count is fixed up below
              acc_a.ts += ad;
              acc_a.tss = fmaf(ad, ad, acc_a.tss);
              acc_r.ts += rt;
              acc_r.tss = fmaf(rt, rt, acc_r.tss);
            }
          }
        }
        rows_done += kRE;
      } else {
        // ragged first tile (T % 64 != 0): plain stores for the rows that exist, no negative TMA store coordinates
        for (int k = 0; k < kRE; ++k) {
          const int rr = e * kRE + k;
          const int t = t0 + rr;
          if (t < 0) continue;
          const float g = st.g[rr][lane];
          float rt = g, ad = g;
          if (HAS_V) {
            const float vt = st.v[rr][lane];
            rt = __fadd_rn(g, vt);
            ad = __fsub_rn(rt, vt);
          }
          if (in_range) {
            const size_t o = (size_t)t * B + col;
            adv[o] = ad;
            ret[o] = rt;
          }
          if (HAS_STATS) {
            const bool valid = HAS_MASK ? (st.m[rr][lane] != 0) : true;
            if (HAS_MASK) acc_a.n += valid ? 1 : 0;
            else rows_done += 1;
            const float am = valid ? ad : 0.0f, rm = valid ? rt : 0.0f;
            acc_a.ts += am;
            acc_a.tss = fmaf(am, am, acc_a.tss);
            acc_r.ts += rm;
            acc_r.tss = fmaf(rm, rm, acc_r.tss);
          }
        }
      }
      if (HAS_STATS) {
        acc_a.fold();
        acc_r.fold();
      }
      rb::tma::fence_proxy_async();  // generic-proxy smem writes -> visible to the async (TMA) proxy
      asm volatile("bar.sync 1, %0;" ::"n"(32 * kEW) : "memory");  // all four row groups of the tile are staged
      if (e == (it % kEW) && lane == 0) {  // rotate the issuing warp so the smem-read wait is spread
        if (t0 >= 0) {
          rb::tma::store_2d(&tm_adv, &adv_s[0][0], col0, t0);  // cols >= B are clipped by TMA
          rb::tma::store_2d(&tm_ret, &st.g[0][0], col0, t0);
          rb::tma::store_commit();
          rb::tma::store_wait_read();  // smem may be reused once the stores have read it
        }
        rb::tma::mbar_arrive(&empty_bar[s]);
      }
    }
    if (lane == 0) rb::tma::store_wait_all();
    if (HAS_STATS) {
      if (!HAS_MASK) acc_a.n = in_range ? rows_done : 0;
      else if (!in_range) acc_a.n = 0;  // mask bytes of OOB columns are zero-filled anyway
      acc_r.n = acc_a.n;
    }
    if (HAS_STATS) flush_stats(acc_a, acc_r, stats);
  }
}

// ---------------------------------------------------------------------------------------------
// Generic kernel (any B, any alignment): one thread per trajectory, register prefetch of U rows.
// ---------------------------------------------------------------------------------------------
template <bool HAS_V, bool HAS_MASK, bool HAS_STATS>
__global__ void __launch_bounds__(32) gae_generic_kernel(const float* __restrict__ rewards,
                                                         const float* __restrict__ values,
                                                         const uint8_t* __restrict__ dones,
                                                         const uint8_t* __restrict__ mask, float* __restrict__ adv,
                                                         float* __restrict__ ret, double* __restrict__ stats, int T,
                                                         int B, float gamma, float coef) {
  constexpr int U = 8;
  const int col = blockIdx.x * 32 + threadIdx.x;
  const bool in_range = col < B;
  Acc acc_a, acc_r;
  if (in_range) {
    float v_next = HAS_V ? values[(size_t)T * B + col] : 0.0f;
    float g = 0.0f;
    for (int t_hi = T - 1; t_hi >= 0; t_hi -= U) {
      float r[U], v[U];
      uint8_t d[U], m[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int t = t_hi - u;
        const bool ok = t >= 0;
        const size_t o = (size_t)(ok ? t : 0) * B + col;
        r[u] = ok ? rewards[o] : 0.0f;
        v[u] = (HAS_V && ok) ? values[o] : 0.0f;
        d[u] = ok ? dones[o + B] : (uint8_t)0;
        m[u] = (HAS_MASK && ok) ? mask[o] : (uint8_t)1;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int t = t_hi - u;
        if (t >= 0) {
          float rt, ad;
          gae_step<HAS_V>(r[u], v[u], v_next, d[u], gamma, coef, g, rt, ad);
          v_next = v[u];
          const size_t o = (size_t)t * B + col;
          adv[o] = ad;
          ret[o] = rt;
          if (HAS_STATS && m[u]) {
            acc_a.add(ad);
            acc_r.add(rt);
          }
        }
      }
      if (HAS_STATS) {
        acc_a.fold();
        acc_r.fold();
      }
    }
  }
  if (HAS_STATS) flush_stats(acc_a, acc_r, stats);
}

// x <- (x - mean) / (std + eps); stats = {n, sum, sumsq}; unbiased variance; skip when n == 0.
__global__ void __launch_bounds__(256) normalize_kernel(float* __restrict__ x, const double* __restrict__ stats,
                                                        int64_t n, float eps) {
  const double cnt = stats[0];
  if (cnt <= 0.0) return;
  const double mean_d = stats[1] / cnt;
  const double var_d = (stats[2] - stats[1] * mean_d) / (cnt - 1.0);  // n==1 -> 0/0 = NaN like torch.std
  const float mean = (float)mean_d;
  const float stdv = (float)sqrt(var_d > 0.0 || !(var_d == var_d) ? var_d : 0.0);
  const float den = __fadd_rn(stdv, eps);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n4 = ((reinterpret_cast<uintptr_t>(x) & 15) == 0) ? n / 4 : 0;
  float4* x4 = reinterpret_cast<float4*>(x);
  for (int64_t k = i; k < n4; k += stride) {
    float4 v = x4[k];
    v.x = __fdiv_rn(__fsub_rn(v.x, mean), den);
    v.y = __fdiv_rn(__fsub_rn(v.y, mean), den);
    v.z = __fdiv_rn(__fsub_rn(v.z, mean), den);
    v.w = __fdiv_rn(__fsub_rn(v.w, mean), den);
    x4[k] = v;
  }
  for (int64_t k = n4 * 4 + i; k < n; k += stride) x[k] = __fdiv_rn(__fsub_rn(x[k], mean), den);
}

template <bool HAS_V, bool HAS_MASK, bool HAS_STATS>
int launch_gae(const float* rewards, const float* values, const uint8_t* dones, const uint8_t* mask, float* adv,
               float* ret, double* stats, int T, int B, float gamma, float coef, cudaStream_t st) {
  const bool aligned = (B % 16 == 0) && ((reinterpret_cast<uintptr_t>(rewards) & 15) == 0) &&
                       (!HAS_V || (reinterpret_cast<uintptr_t>(values) & 15) == 0) &&
                       ((reinterpret_cast<uintptr_t>(dones) & 15) == 0) &&
                       (!HAS_MASK || (reinterpret_cast<uintptr_t>(mask) & 15) == 0) &&
                       (((reinterpret_cast<uintptr_t>(adv) | reinterpret_cast<uintptr_t>(ret)) & 15) == 0);
  const int grid = (B + kW - 1) / kW;
  if (aligned) {
    CUtensorMap tm_r, tm_v, tm_d, tm_m;
    int e = rb::encode_tmap_2d(&tm_r, rewards, 4, (uint64_t)T, (uint64_t)B, kRW, kW);
    if (!e && HAS_V) e = rb::encode_tmap_2d(&tm_v, values, 4, (uint64_t)T + 1, (uint64_t)B, kRW + 1, kW);
    if (!e) e = rb::encode_tmap_2d(&tm_d, dones, 1, (uint64_t)T + 1, (uint64_t)B, kRW, kW);
    if (!e && HAS_MASK) e = rb::encode_tmap_2d(&tm_m, mask, 1, (uint64_t)T, (uint64_t)B, kRW, kW);
    CUtensorMap tm_adv, tm_ret;
    if (!e) e = rb::encode_tmap_2d(&tm_adv, adv, 4, (uint64_t)T, (uint64_t)B, kRW, kW);
    if (!e) e = rb::encode_tmap_2d(&tm_ret, ret, 4, (uint64_t)T, (uint64_t)B, kRW, kW);
    if (!HAS_V) tm_v = tm_r;
    if (!HAS_MASK) tm_m = tm_d;
    if (!e) {
      constexpr int kSmem = kStagesWS * (int)sizeof(StageWS) + 128;
      static bool attr_done = false;
      if (!attr_done) {
        cudaError_t ce = cudaFuncSetAttribute(gae_tma_kernel<HAS_V, HAS_MASK, HAS_STATS>,
                                              cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
        if (ce != cudaSuccess) return (int)ce;
        attr_done = true;
      }
      gae_tma_kernel<HAS_V, HAS_MASK, HAS_STATS>
          <<<grid, kWsThreads, kSmem, st>>>(tm_r, tm_v, tm_d, tm_m, tm_adv, tm_ret, adv, ret, stats, T, B, gamma, coef);
      rb::count_launch();
      RB_RETURN_LAUNCH();
    }
    // descriptor encode failed (e.g. driver entry point unavailable): use the generic kernel
  }
  gae_generic_kernel<HAS_V, HAS_MASK, HAS_STATS>
      <<<grid, 32, 0, st>>>(rewards, values, dones, mask, adv, ret, stats, T, B, gamma, coef); rb::count_launch();
  RB_RETURN_LAUNCH();
}

}  // namespace

extern "C" int rb200_gae(const float* rewards, const float* values, const uint8_t* dones, const uint8_t* loss_mask,
                         float* adv, float* ret, double* stats, int T, int B, double gamma, double gae_lambda,
                         rb200_stream_t stream) {
  if (!rewards || !dones || !adv || !ret) return RB200_E_NULL;
  if (T <= 0 || B <= 0) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  if (!values) {  // critic-free: the reference forces gamma = lambda = 1 (advantages.py:61-64)
    gamma = 1.0;
    gae_lambda = 1.0;
  }
  const float gamma_f = (float)gamma;
  const float coef_f = (float)(gamma * gae_lambda);  // product in double, then one rounding
  if (stats) RB_CHECK_CUDA(cudaMemsetAsync(stats, 0, 6 * sizeof(double), st));
#define RB_GAE(V, M, S) \
  return launch_gae<V, M, S>(rewards, values, dones, loss_mask, adv, ret, stats, T, B, gamma_f, coef_f, st)
  if (values) {
    if (stats) {
      if (loss_mask) RB_GAE(true, true, true);
      RB_GAE(true, false, true);
    }
    RB_GAE(true, false, false);
  } else {
    if (stats) {
      if (loss_mask) RB_GAE(false, true, true);
      RB_GAE(false, false, true);
    }
    RB_GAE(false, false, false);
  }
#undef RB_GAE
}

extern "C" int rb200_normalize(float* x, const double* stats, int64_t n_elems, float eps, rb200_stream_t stream) {
  if (!x || !stats) return RB200_E_NULL;
  if (n_elems <= 0) return RB200_E_SHAPE;
  int64_t blocks = (n_elems / 4 + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  normalize_kernel<<<(int)blocks, 256, 0, rb::as_stream(stream)>>>(x, stats, n_elems, eps); rb::count_launch();
  RB_RETURN_LAUNCH();
}
