// Persistent tensor-core rollout: the whole T-step actor/critic inference + synthetic-env loop of one rank in ONE kernel,
// every hidden layer (and the env's s.W_s product) on Hopper wgmma.  Replaces EnvWorker.interact /
// MultiStepRolloutWorker.generate (rlinf/workers/env/env_worker.py:1059-1349, huggingface_worker.py:678-781) for the MLP
// policy with the device-resident synthetic env; same buffers, row alignment, random streams and draw order as
// rollout_fused.cu / the per-kernel CUDA-graph path.  CTA c owns environments [32c, 32c+32) and computes every layer
// TRANSPOSED, D[hidden unit, env] = W . X^T, with the 2-way fp16 split of tc_gemm_h.cu (three MMAs per product).
// Roles (416 threads): warpgroup 0 = env (Philox noise, x.W_s, dynamics finish, next observation operand), 1 = actor
// tower (+ mean head, sampling), 2 = value tower (+ value head, truncation bootstrap), warp 12 = weight-stream producer
// (one ring per warpgroup).  Each warpgroup issues its own layers and finishes them from its accumulator registers.
// The truncation bootstrap rides in 32 extra columns (N = 64) of the next step's value tower.
#include <cuda_fp16.h>
#include <curand_kernel.h>

#include "common.cuh"
#include "episode_stats.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace {

using rb::tma::mbar_arrive;
using rb::tma::mbar_init;
using rb::tma::mbar_wait;
using rb::tma::smem_u32;

constexpr int kH = 256;
constexpr int kNE = 32;        // environments per CTA (MMA N)
constexpr int kMaxActTc = 8;   // action dims held in shared memory
constexpr int kMaxObsTc = 128; // one M tile of the env product
constexpr int kStageBytes = 16384, kHalfTile = 8192;  // [128 rows x 32 k] fp16 hi | lo
// One weight ring per consuming warpgroup: with a shared ring a warpgroup a lap ahead would take a slot's old phase.
constexpr int kStages = 5;
constexpr int kEnvSlot0 = 0, kEnvSlots = 1, kActSlot0 = 1, kActSlots = 2, kValSlot0 = 3, kValSlots = 2;
static_assert(kValSlot0 + kValSlots == kStages, "ring slots");
constexpr int kThreads = 13 * 32;
constexpr int kWScaleLog2 = 10;  // weights are stored as fp16 (hi, lo) of w * 2^10
constexpr float kHalfLog2Pi = 0.91893853320467274178f;

// Cycle probe, off by default (-DRB200_ROLLOUT_TC_PROBE, built and read by tools/rollout_tc_probe.py): clock64() sums
// per CTA over the rollout, one 8-byte slot each.  Waits are summed by the waiting thread (the producer lane, thread 0
// of each consumer warpgroup); kT* slots are sums over steps t < T of (stamp - the step's obs-ready stamp).
#ifdef RB200_ROLLOUT_TC_PROBE
#define TC_PROBE(...) __VA_ARGS__
enum ProbeSlot {
  kPrEmptyWait, kPrEmptyPolls, kPrStages,  // producer: cycles in unsuccessful empty waits, their number, stages issued
  kPwEnvFull, kPwActFull, kPwValFull,      // consumer waits on full (env, actor, value warpgroup: tid >> 7)
  kTActTower, kTSample,                    // actor: tower done, actions sampled (thread 128)
  kTEnvProduct, kTEnvVhead, kTObsReady,    // env: x.W_s done, value head seen, next observation ready (thread 0)
  kTValTower, kTValHead,                   // value: tower done, head done (thread 256)
  kTSteps, kProbeSlots
};
__device__ unsigned long long* g_tc_probe;  // [grid][kProbeSlots]
#else
#define TC_PROBE(...)
#endif

// shared-memory map (bytes from the 1024-aligned base)
constexpr int kOffRing = 0;
constexpr int kOffObuf = kOffRing + kStages * kStageBytes;  // [hi|lo][kb<=4][64 rows][64 B]: rows 0-31 obs, 32-63 final obs
constexpr int kObufHalf = 4 * 64 * 64;                      // 16 KB
constexpr int kOffAbuf = kOffObuf + 2 * kObufHalf;          // [hi|lo][kb 8][32 rows][64 B] | fp32 h3 [32][256] | fp32 zs
constexpr int kAbufHalf = 8 * 32 * 64;                      // 16 KB
constexpr int kOffVbuf = kOffAbuf + 2 * kAbufHalf;          // [hi|lo][kb 8][64 rows][64 B] | fp32 g3 [64][256]
constexpr int kVbufHalf = 8 * 64 * 64;                      // 32 KB
constexpr int kOffMisc = kOffVbuf + 2 * kVbufHalf;

struct Misc {
  float mw[kMaxActTc * kH];
  float vw[kH];
  float mean[kNE * kMaxActTc];
  float act[kNE * kMaxActTc];
  float rew[kNE];
  float er[kNE], uu[kNE];  // reward noise / termination uniform of this step (env warps -> finishing warps)
  int flag[kNE];
  int el[kNE];
  int nflag;
  uint64_t full[kStages], empty[kStages];
  uint64_t vhead, obs_ready;
  TC_PROBE(unsigned long long probe[kProbeSlots]; long long t_obs;)
};
constexpr int kArgsBytes = 512;  // shared-memory copy of the kernel arguments for the out-of-line helpers
constexpr int kOffArgs = kOffMisc + (((int)sizeof(Misc) + 15) & ~15);
constexpr int kSmemBytes = kOffMisc + (int)sizeof(Misc) + kArgsBytes + 1024;
static_assert(kSmemBytes <= 232448, "rollout_tc shared memory");

// Chunked variant (num_action_chunks = C > 1, act = C*A): the C*A actions of a chunk step are kept behind the argument
// copy (the C = 1 map above is unchanged); the mean head [C*A, 256] is read through L2 and the value head [C, 256]
// takes the place of Misc::mw.
constexpr int kMaxChunks = 8;
constexpr int kMaxActChunk = 32;  // C*A
struct ChunkSmem {
  float act[kNE * kMaxActChunk];  // [env][C*A] actions of this chunk step
  int orf[kNE];                   // term | trunc << 1 of the sub-steps so far (OR over the chunk)
};
constexpr int kOffChunk = kOffArgs + kArgsBytes;
constexpr int kSmemBytesChunk = kOffChunk + (int)sizeof(ChunkSmem) + 1024;
static_assert(kSmemBytesChunk <= 232448, "rollout_tc chunked shared memory");
static_assert(kMaxChunks * kH <= kMaxActTc * kH, "chunked value head in Misc::mw");
__device__ __forceinline__ ChunkSmem* chunk_smem(Misc* ms) {
  return reinterpret_cast<ChunkSmem*>(reinterpret_cast<uint8_t*>(ms) + (kOffChunk - kOffMisc));
}

// Episode statistics of the training rollout (kStats): the running fp32 return of the CTA's environments (loaded from
// and stored back to the caller's ret [B], so episodes span rollouts) and the caller's fp64 sums acc [B,4].  They sit
// behind the C = 1 / chunked maps above, so the kernels without statistics keep their shared-memory layout.
struct StatsSmem {
  float ret[kNE];
  double* acc;
};
struct EpStats {
  float* ret;   // [B]
  double* acc;  // [B,4]: count, sum return, sum length, sum reward
};
template <bool kChunk>
constexpr int kOffStats = kOffChunk + (kChunk ? (int)sizeof(ChunkSmem) : 0);
template <bool kChunk, bool kStats>
constexpr int kSmemTotal =
    kStats ? kOffStats<kChunk> + (int)sizeof(StatsSmem) + 1024 : (kChunk ? kSmemBytesChunk : kSmemBytes);
static_assert(kOffStats<true> % 8 == 0 && kOffStats<false> % 8 == 0, "StatsSmem alignment");
static_assert(kSmemTotal<true, true> <= 232448 && kSmemTotal<false, true> <= 232448, "rollout_tc statistics shared memory");
template <bool kChunk>
__device__ __forceinline__ StatsSmem* stats_smem(Misc* ms) {
  return reinterpret_cast<StatsSmem*>(reinterpret_cast<uint8_t*>(ms) + (kOffStats<kChunk> - kOffMisc));
}

struct TcArgs {
  rb200_mlp_layout L;
  const float* params;
  const uint8_t* pack;   // pre-split, pre-swizzled weight stream (rb200_rollout_tc_prepare)
  const float* w_a;      // [act, obs]
  float* states;         // [T+1, B, obs]
  float* actions;        // [T, B, act]
  float* logp;           // [T, B, act]
  float* values;         // [T+1, B, C]
  float* rewards;        // [T, B, C]
  uint8_t* term;         // [T+1, B, C]
  uint8_t* trunc;
  uint8_t* done;
  float* final_obs;      // [B, obs]
  float* final_values;   // [B, C]
  int32_t* elapsed;      // [B]
  const float* policy_noise;
  const float* env_noise;
  const uint64_t* counter_p;
  const uint64_t* counter_e;
  uint64_t seed_p, seed_e, offset_p;
  int T, B, obs, act;    // T = chunk steps, act = C*A
  int max_episode_steps, auto_reset, bootstrap_on_done;
  float gamma, p_term, noise_std, reward_noise_std;
  int C;                 // num_action_chunks (1 in the unchunked kernel)
};
static_assert(sizeof(TcArgs) <= kArgsBytes, "TcArgs shared-memory copy");

// 1-D bulk copy global -> shared, completion counted on an mbarrier
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void named_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// byte offset of element (row, k in [0,32)) inside a [rows x 32 fp16] SWIZZLE_64B tile
__device__ __forceinline__ uint32_t sw64_off(int row, int kk) {
  return (uint32_t)(row * 64 + ((((kk >> 3) ^ ((row >> 1) & 3))) << 4) + (kk & 7) * 2);
}
__device__ __forceinline__ void store_split(uint8_t* hi_base, uint32_t half_bytes, uint32_t off, float v) {
  const __half h = __float2half_rn(v);
  const __half l = __float2half_rn(v - __half2float(h));
  *reinterpret_cast<__half*>(hi_base + off) = h;
  *reinterpret_cast<__half*>(hi_base + half_bytes + off) = l;
}
__device__ __forceinline__ float tanh_fast(float x) {  // same formula as the tensor-core GEMM epilogues
  const float t = __expf(-2.0f * fabsf(x));
  return copysignf(__fdividef(1.0f - t, 1.0f + t), x);
}
__device__ __forceinline__ float dot256(const float* row, const float* w, int lane) {
  const float4 g0 = *reinterpret_cast<const float4*>(row + lane * 4);
  const float4 g1 = *reinterpret_cast<const float4*>(row + 128 + lane * 4);
  const float4 w0 = *reinterpret_cast<const float4*>(w + lane * 4);
  const float4 w1 = *reinterpret_cast<const float4*>(w + 128 + lane * 4);
  float s = g0.x * w0.x + g0.y * w0.y + g0.z * w0.z + g0.w * w0.w + g1.x * w1.x + g1.y * w1.y + g1.z * w1.z +
            g1.w * w1.w;
  return rb::warp_sum(s);
}

// weight-stream segments in stage units (one stage = one 128-row tile x one 32-wide k-block, hi | lo; inside a layer
// the stages are ordered k-block outer, M tile inner)
struct Segs {
  int env, a0, v0, a1, v1, a2, v2, total, nkb0;
};
__host__ __device__ inline Segs make_segs(int obs) {
  Segs s;
  s.nkb0 = obs / 32;
  s.env = 0;
  s.a0 = s.nkb0;
  s.v0 = 3 * s.nkb0;
  s.a1 = 5 * s.nkb0;
  s.v1 = s.a1 + 16;
  s.a2 = s.a1 + 32;
  s.v2 = s.a1 + 48;
  s.total = s.a1 + 64;
  return s;
}

// ---- Philox draws as out-of-line functions: inlined at every use (8 + 8 + 1 sites, ~700 instructions each) the kernel
//      was 230 KB of SASS executed by 16 warps at different program counters - far beyond the instruction caches ----
struct EnvDraws {
  float e[4];  // state noise of observation columns lane, lane+32, lane+64, lane+96
  float er, u; // reward noise and termination uniform (lane 0's stream only)
};
// the draws of env_finish_kernel (rollout.cu) for one (environment row, lane) stream of one step, in its order
__device__ __noinline__ EnvDraws env_draws(unsigned long long seed, unsigned long long subseq, unsigned long long offset,
                                           int nk, int lane0) {
  curandStatePhilox4_32_10_t st;
  curand_init(seed, subseq, offset, &st);
  EnvDraws d;
#pragma unroll
  for (int k = 0; k < 4; ++k) d.e[k] = (k < nk) ? curand_normal(&st) : 0.f;
  d.er = 0.f;
  d.u = 1.f;
  if (lane0) {
    d.er = curand_normal(&st);
    d.u = curand_uniform(&st);
  }
  return d;
}
// the N(0,1) reset state that FOLLOWS those draws in the same stream
__device__ __noinline__ EnvDraws env_reset_draws(unsigned long long seed, unsigned long long subseq,
                                                 unsigned long long offset, int nk, int lane0) {
  curandStatePhilox4_32_10_t st;
  curand_init(seed, subseq, offset, &st);
  for (int k = 0; k < nk; ++k) (void)curand_normal(&st);
  if (lane0) {
    (void)curand_normal(&st);
    (void)curand_uniform(&st);
  }
  EnvDraws d;
#pragma unroll
  for (int k = 0; k < 4; ++k) d.e[k] = (k < nk) ? curand_normal(&st) : 0.f;
  d.er = 0.f;
  d.u = 1.f;
  return d;
}
__device__ __noinline__ float policy_draw(unsigned long long seed, unsigned long long subseq, unsigned long long offset) {
  curandStatePhilox4_32_10_t st;
  curand_init(seed, subseq, offset, &st);
  return curand_normal(&st);
}

// Dynamics finish of 4 environments [w8*4, w8*4+4) by one warp (8 warps share a step: the actor group is idle once the
// actions are sampled, so it takes half of the environments).  Array stages over the 4 environments - all loads, then
// the math, then all stores - keep 4-16 independent chains in flight per lane.  zs = x.W_s (env product), eps_s = this
// step's N(0,1) draws, both fp32 [32][obs] in the (now free) actor buffer.  Same arithmetic order as env_finish_kernel
// (rollout.cu) except tanh (MUFU-based tanh_fast, 3e-7 abs).
// kChunk: t counts env sub-steps, chunk step n = t / C, sub-step c = t % C, with the semantics of
// env_substep_kernel + chunk_finish_kernel: sub-step c uses action columns [cA, (c+1)A), no reset inside the chunk,
// flags OR-ed over the chunk and written to column C-1 only, one auto-reset after the last sub-step.
// kStats: the raw reward goes into the running return; an episode is recorded (ManiskillEnv._record_metrics) at the
// chunk's last sub-step where the chunk is done with auto-reset, and for every environment at the rollout's last chunk
// step without it (should_record in EnvWorker._run_interact_once); a recorded episode restarts the return on auto-reset.
template <bool kChunk, bool kStats>
__device__ __noinline__ void env_finish4(const TcArgs& p, Misc* ms, uint8_t* obuf, uint32_t ob_half, const float* zs,
                                            const float* eps_s, int w8, int lane, int t, int e0, int nE, int nk,
                                            uint64_t c_e, bool boot) {
  const int obs = p.obs, B = p.B, T = p.T;
  const int Cn = kChunk ? p.C : 1;
  const int n = kChunk ? t / Cn : t, sub = t - n * Cn;
  const bool last = !kChunk || sub == Cn - 1;
  const int A = kChunk ? p.act / Cn : p.act;
  const int nzw = Cn * (obs + 2) + obs;  // env_noise row: per sub-step eps[obs] | eps_r | u, then reset[obs]
  ChunkSmem* cs = chunk_smem(ms);
  float v[4][4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i][k] = 0.f;
    if (k < nk) {
      const int c = lane + 32 * k;
      float wa[kMaxActTc];
#pragma unroll
      for (int a = 0; a < kMaxActTc; ++a) wa[a] = a < A ? __ldg(p.w_a + a * obs + c) : 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int e = w8 * 4 + i;
        float z = zs[e * obs + c];
        if constexpr (kChunk) {
          const float* ac = cs->act + e * kMaxActChunk + sub * A;
#pragma unroll
          for (int a = 0; a < kMaxActTc; ++a) z = fmaf(a < A ? ac[a] : 0.f, wa[a], z);
        } else {
          const float4 a0 = *reinterpret_cast<const float4*>(ms->act + e * kMaxActTc);
          const float4 a1 = *reinterpret_cast<const float4*>(ms->act + e * kMaxActTc + 4);
          z = fmaf(a0.x, wa[0], z); z = fmaf(a0.y, wa[1], z); z = fmaf(a0.z, wa[2], z); z = fmaf(a0.w, wa[3], z);
          z = fmaf(a1.x, wa[4], z); z = fmaf(a1.y, wa[5], z); z = fmaf(a1.z, wa[6], z); z = fmaf(a1.w, wa[7], z);
        }
        float ep = eps_s[e * obs + c];
        if (p.env_noise && e < nE) ep = p.env_noise[((size_t)n * B + e0 + e) * nzw + sub * (obs + 2) + c];
        v[i][k] = tanh_fast(z + p.noise_std * ep);
      }
    }
  }
  float sq[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) sq[i] = (v[i][0] * v[i][0] + v[i][1] * v[i][1]) + (v[i][2] * v[i][2] + v[i][3] * v[i][3]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int i = 0; i < 4; ++i) sq[i] += __shfl_xor_sync(0xffffffffu, sq[i], o);
  }
  bool reset[4];
  float rw[4];
  int bits[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = w8 * 4 + i;
    float er = ms->er[e], u = ms->uu[e];
    if (p.env_noise && e < nE) {
      const float* nz = p.env_noise + ((size_t)n * B + e0 + e) * nzw + sub * (obs + 2);
      er = nz[obs];
      u = nz[obs + 1];
    }
    const int el = ms->el[e] + 1;
    bool term = u < p.p_term;
    bool trunc = p.max_episode_steps > 0 && el >= p.max_episode_steps;
    if (kChunk && sub > 0) {
      term |= (cs->orf[e] & 1) != 0;
      trunc |= (cs->orf[e] & 2) != 0;
    }
    const bool done = term || trunc;
    reset[i] = last && done && p.auto_reset;
    const bool flagged = last && boot && (p.bootstrap_on_done ? done : trunc);
    rw[i] = -sq[i] / (float)obs + p.reward_noise_std * er;
    bits[i] = (term ? 1 : 0) | (trunc ? 2 : 0) | (done ? 4 : 0) | (flagged ? 8 : 0) | ((reset[i] ? 0 : el) << 4);
  }
  __syncwarp();  // every lane has read ms->el before lane 0 rewrites the per-environment slots
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = w8 * 4 + i;
      if (e < nE) {
        const int64_t row = e0 + e;
        const size_t o = ((size_t)(n + 1) * B + row) * Cn + sub;
        const int fl = last ? bits[i] : 0;  // flags of a chunk go to its last column
        p.term[o] = fl & 1;
        p.trunc[o] = (fl >> 1) & 1;
        p.done[o] = (fl >> 2) & 1;
        if (kChunk) cs->orf[e] = bits[i] & 3;
        if constexpr (kStats) {
          StatsSmem* ss = stats_smem<kChunk>(ms);
          const float r = __fadd_rn(ss->ret[e], rw[i]);
          const bool rec = last && (p.auto_reset ? (bits[i] & 4) != 0 : n == T - 1);
          if (rec) rb::episode_finish(ss->acc + (size_t)row * 4, r, ms->el[e] + 1);  // el before the reset
          ss->ret[e] = (rec && p.auto_reset) ? 0.f : r;
        }
        ms->el[e] = bits[i] >> 4;
        ms->flag[e] = (bits[i] >> 3) & 1;
        ms->rew[e] = rw[i];
        // flagged: written by the value warps with the bootstrap
        if (!(bits[i] & 8)) p.rewards[((size_t)n * B + row) * Cn + sub] = rw[i];
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int e = w8 * 4 + i;
    if (e >= nE) continue;
    const int64_t row = e0 + e;
    float nw[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) nw[k] = v[i][k];
    if (reset[i]) {  // warp-uniform, rare (one env-step in ~80): fresh state from the same stream, same draw order
      if (p.env_noise) {
        const float* nz = p.env_noise + ((size_t)n * B + row) * nzw + Cn * (obs + 2);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (k < nk) nw[k] = nz[lane + 32 * k];
      } else {
        // chunked: chunk_finish_kernel's fresh window, 32 outputs behind the last sub-step's
        const EnvDraws d = kChunk ? env_draws(p.seed_e, (unsigned long long)row * 32ull + lane,
                                              (c_e * (uint64_t)Cn + (uint64_t)t) * 64ull + 32ull, nk, 0)
                                  : env_reset_draws(p.seed_e, (unsigned long long)row * 32ull + lane,
                                                    (c_e + (uint64_t)t) * 64ull, nk, lane == 0);
#pragma unroll
        for (int k = 0; k < 4; ++k) nw[k] = d.e[k];
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k < nk) {
        const int c = lane + 32 * k;
        // inside a chunk only the next sub-step's operand (rows 0..31) is written
        if (last && n == T - 1) p.final_obs[(size_t)row * obs + c] = v[i][k];
        if (last) store_split(obuf, ob_half, (uint32_t)k * 4096u + sw64_off(kNE + e, lane), v[i][k]);  // pre-reset observation
        store_split(obuf, ob_half, (uint32_t)k * 4096u + sw64_off(e, lane), nw[k]);
        if (last) p.states[((size_t)(n + 1) * B + row) * obs + c] = nw[k];
      }
    }
  }
}

// D[hidden unit, env] = W . X^T for one layer, by one warpgroup: weight stages from its ring (k-block outer, 128-row tile
// inner), X = fp16 hi | lo K-major tiles of N rows.  Accumulators stay in registers: the output overwrites X in place.
template <int N, int NT>
struct LayerAcc {
  float d[NT][2][N / 2];
};

template <int N, int NT>
__device__ __forceinline__ void layer_mma(LayerAcc<N, NT>& acc, Misc* ms, uint32_t ring_a, int slot0, int nslots,
                                          uint32_t stage0, int nkb, uint32_t b_addr, uint32_t b_half, uint32_t b_kb_stride,
                                          int lane) {
#pragma unroll
  for (int m = 0; m < NT; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < N / 2; ++i) acc.d[m][h][i] = 0.f;
#pragma unroll 1
  for (int kb = 0; kb < nkb; ++kb) {
    const uint32_t sb = b_addr + (uint32_t)kb * b_kb_stride;
#pragma unroll
    for (int m = 0; m < NT; ++m) {
      const uint32_t idx = stage0 + (uint32_t)(kb * NT + m);
      const uint32_t slot = (uint32_t)slot0 + idx % (uint32_t)nslots, ph = (idx / (uint32_t)nslots) & 1u;
      TC_PROBE(const long long pt0 = clock64();)
      mbar_wait(&ms->full[slot], ph);
      TC_PROBE(if ((threadIdx.x & 127) == 0) ms->probe[kPwEnvFull + (threadIdx.x >> 7)] += clock64() - pt0;)
      const uint32_t a = ring_a + slot * kStageBytes;
      rb::wg::fence();
#pragma unroll
      for (int k = 0; k < 2; ++k) {  // two k-steps of 16 = 32 B along the 64-B rows
        const uint64_t b_hi = rb::wg::desc(sb + k * 32, 16, 512, 2), b_lo = rb::wg::desc(sb + b_half + k * 32, 16, 512, 2);
#pragma unroll
        for (int h = 0; h < 2; ++h) {  // rows 64h .. 64h + 63 of the 128-row weight tile
          const uint64_t a_hi = rb::wg::desc(a + h * 4096 + k * 32, 16, 512, 2);
          const uint64_t a_lo = rb::wg::desc(a + kHalfTile + h * 4096 + k * 32, 16, 512, 2);
          rb::wg::MmaSS<N>::run(acc.d[m][h], a_lo, b_hi, 1u);  // small terms first
          rb::wg::MmaSS<N>::run(acc.d[m][h], a_hi, b_lo, 1u);
          rb::wg::MmaSS<N>::run(acc.d[m][h], a_hi, b_hi, 1u);
        }
      }
      rb::wg::commit();
      rb::wg::wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&ms->empty[slot]);
    }
  }
}

// out = tanh(acc * 2^-10 + bias) as the next layer's fp16 operand or (last layer) fp32 [env][256]; units
// j = 128 m + 64 h + 16 w + g (+ 8), environments e = 8 c + 2 t (+ 1).
template <int N>
__device__ __forceinline__ void layer_epilogue(const LayerAcc<N, 2>& acc, const float* bias, uint8_t* buf, uint32_t half_bytes,
                                               uint32_t kb_bytes, int last, int w, int lane) {
  const float out_scale = 1.0f / (float)(1 << kWScaleLog2);
  const int g = lane >> 2, t = lane & 3;
  float* f32 = reinterpret_cast<float*>(buf);
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int j = m * 128 + h * 64 + w * 16 + g + 8 * r;
        const float b = __ldg(bias + j);
#pragma unroll
        for (int c = 0; c < N / 8; ++c)
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const int e = 8 * c + 2 * t + u;
            const float v = tanh_fast(acc.d[m][h][4 * c + 2 * r + u] * out_scale + b);
            if (last) f32[e * kH + j] = v;
            else store_split(buf, half_bytes, (uint32_t)(j >> 5) * kb_bytes + sw64_off(e, j & 31), v);
          }
      }
}

// MMAs, barrier (the operand is read), epilogue, barrier (the next operand is complete).
template <int N>
__device__ __noinline__ void tower_layer(Misc* ms, uint32_t ring_a, int slot0, uint32_t stage0, int nkb, uint32_t b_addr,
                                         uint32_t b_half, uint32_t b_kb_stride, const float* bias, uint8_t* buf,
                                         uint32_t half_bytes, uint32_t kb_bytes, int last, int bar_id, int w, int lane) {
  LayerAcc<N, 2> acc;
  layer_mma<N, 2>(acc, ms, ring_a, slot0, 2, stage0, nkb, b_addr, b_half, b_kb_stride, lane);
  named_sync(bar_id, 128);
  layer_epilogue<N>(acc, bias, buf, half_bytes, kb_bytes, last, w, lane);
  rb::tma::fence_proxy_async();
  named_sync(bar_id, 128);
}

// kChunk: num_action_chunks = p.C > 1.  Per chunk step the towers run once; the env warpgroup runs C x.W_s products and
// the env and actor warpgroups C dynamics finishes, the first one after the value tower has read the observation tile.
// kStats: episode statistics of the rollout into es (env_finish4).
template <bool kChunk, bool kStats>
__global__ void __launch_bounds__(kThreads, 1) rollout_tc_kernel(const TcArgs p, const EpStats es) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ring = smem + kOffRing;
  uint8_t* obuf = smem + kOffObuf;
  uint8_t* abuf = smem + kOffAbuf;
  uint8_t* vbuf = smem + kOffVbuf;
  Misc* ms = reinterpret_cast<Misc*>(smem + kOffMisc);
  // out-of-line helpers read the arguments from shared memory (a reference to the kernel parameter would be copied to
  // the local-memory stack of every thread)
  TcArgs* pa = reinterpret_cast<TcArgs*>(smem + kOffMisc + ((sizeof(Misc) + 15) & ~size_t(15)));

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int obs = p.obs, act = p.act, T = p.T, B = p.B;
  const int e0 = blockIdx.x * kNE;
  int nE = B - e0;
  if (nE > kNE) nE = kNE;
  const Segs sg = make_segs(obs);
  const float* P = p.params;
  const uint64_t c_p = p.counter_p ? p.counter_p[0] : 0ull;
  const uint64_t c_e = p.counter_e ? p.counter_e[0] : 0ull;
  const float out_scale = 1.0f / (float)(1 << kWScaleLog2);
  const bool boot = p.auto_reset != 0;  // the value head exists (rb200_rollout_tc_supported)
  const uint32_t ring_a = smem_u32(ring), obuf_a = smem_u32(obuf), abuf_a = smem_u32(abuf), vbuf_a = smem_u32(vbuf);
  const uint32_t ob_half = (uint32_t)sg.nkb0 * 4096u;

  // ---- setup ----
  for (int i = tid; i < (int)(sizeof(TcArgs) / 4); i += kThreads)
    reinterpret_cast<uint32_t*>(pa)[i] = reinterpret_cast<const uint32_t*>(&p)[i];
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&ms->full[s], 1);
      mbar_init(&ms->empty[s], 4);  // one arrival per warp of the consuming warpgroup
    }
    mbar_init(&ms->vhead, 4);
    mbar_init(&ms->obs_ready, 1);
    ms->nflag = 0;
    TC_PROBE(for (int s = 0; s < kProbeSlots; ++s) ms->probe[s] = 0ull; ms->t_obs = clock64();)
    rb::tma::fence_barrier_init();
  }
  const int Cn = kChunk ? p.C : 1;
  if constexpr (kChunk) {
    for (int i = tid; i < Cn * kH; i += kThreads) ms->mw[i] = P[p.L.vw3 + i];  // value head [C, 256]
    if (tid < kNE) chunk_smem(ms)->orf[tid] = 0;
  } else {
    for (int i = tid; i < act * kH; i += kThreads) ms->mw[i] = P[p.L.mw + i];
    for (int i = tid; i < kH; i += kThreads) ms->vw[i] = P[p.L.vw3 + i];
  }
  for (int i = tid; i < 2 * kNE * obs; i += kThreads) {  // rows 0..31 = current observation, rows 32..63 = zeros
    const int r = i / obs, c = i - r * obs;
    const float v = (r < nE) ? p.states[(size_t)(e0 + r) * obs + c] : 0.f;
    store_split(obuf, ob_half, (uint32_t)(c >> 5) * 4096u + sw64_off(r, c & 31), v);
  }
  for (int i = tid; i < kNE * kMaxActTc; i += kThreads) ms->act[i] = 0.f;
  if (tid < kNE) {
    ms->el[tid] = tid < nE ? p.elapsed[e0 + tid] : 0;
    ms->flag[tid] = 0;
    ms->rew[tid] = 0.f;
  }
  if constexpr (kStats) {
    StatsSmem* ss = stats_smem<kChunk>(ms);
    if (tid < kNE) ss->ret[tid] = tid < nE ? es.ret[e0 + tid] : 0.f;
    if (tid == 0) ss->acc = es.acc;
  }
  rb::tma::fence_proxy_async();
  __syncthreads();

  // per-step stream lengths (in stages) of the three consumers: env product, actor tower, value tower
  const uint32_t n_env = (uint32_t)sg.nkb0, n_tower = 2u * (uint32_t)sg.nkb0 + 32u;
  if (warp == 12) {
    // ======== weight-stream producer: three rings, polled with test_wait (no ring waits for another) ========
    if (lane == 0) {
      const uint32_t total[3] = {(uint32_t)(T * Cn) * n_env, (uint32_t)T * n_tower, (uint32_t)(T + 1) * n_tower};
      const int slot0[3] = {kEnvSlot0, kActSlot0, kValSlot0}, nslots[3] = {kEnvSlots, kActSlots, kValSlots};
      uint32_t j[3] = {0u, 0u, 0u};
      while (j[0] < total[0] || j[1] < total[1] || j[2] < total[2]) {
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          if (j[q] >= total[q]) continue;
          const uint32_t slot = (uint32_t)slot0[q] + j[q] % (uint32_t)nslots[q], ph = (j[q] / (uint32_t)nslots[q]) & 1u;
          TC_PROBE(const long long pt0 = clock64();)
          if (!rb::tma::mbar_test_wait(&ms->empty[slot], ph ^ 1u)) {
            TC_PROBE(ms->probe[kPrEmptyWait] += clock64() - pt0; ++ms->probe[kPrEmptyPolls];)
            continue;
          }
          TC_PROBE(++ms->probe[kPrStages];)
          // pack stage of position j in this stream (pack order: env, a0, v0, a1, v1, a2, v2)
          int stage;
          if (q == 0) {
            stage = sg.env + (int)(j[q] % n_env);
          } else {
            const int i = (int)(j[q] % n_tower), l0 = 2 * sg.nkb0;
            const bool v = q == 2;
            stage = i < l0 ? (v ? sg.v0 : sg.a0) + i : (i < l0 + 16 ? (v ? sg.v1 : sg.a1) + i - l0 : (v ? sg.v2 : sg.a2) + i - l0 - 16);
          }
          rb::tma::mbar_arrive_expect_tx(&ms->full[slot], kStageBytes);
          bulk_load(ring + slot * kStageBytes, p.pack + (size_t)stage * kStageBytes, kStageBytes, &ms->full[slot]);
          ++j[q];
        }
      }
    }
  } else if (warp >= 4 && warp < 8) {
    // ================= actor tower: layers, mean head, sampling =================
    const int w = warp & 3, gt = tid - 128;
    const float* bias[3] = {P + p.L.bb0, P + p.L.bb1, P + p.L.bb2};
    float* h3 = reinterpret_cast<float*>(abuf);
    uint32_t p_obs = 0;
    for (int t = 0; t < T; ++t) {
      if (t > 0) {
        mbar_wait(&ms->obs_ready, p_obs);
        p_obs ^= 1u;
      }
      TC_PROBE(const long long t_obs = *reinterpret_cast<volatile long long*>(&ms->t_obs);)
      const uint32_t base = (uint32_t)t * n_tower, l0 = 2u * (uint32_t)sg.nkb0;
      tower_layer<kNE>(ms, ring_a, kActSlot0, base, sg.nkb0, obuf_a, ob_half, 4096u, bias[0], abuf, kAbufHalf, 2048u, 0, 1, w,
                       lane);
      tower_layer<kNE>(ms, ring_a, kActSlot0, base + l0, 8, abuf_a, kAbufHalf, 2048u, bias[1], abuf, kAbufHalf, 2048u, 0, 1,
                       w, lane);
      tower_layer<kNE>(ms, ring_a, kActSlot0, base + l0 + 16, 8, abuf_a, kAbufHalf, 2048u, bias[2], abuf, kAbufHalf, 2048u, 1,
                       1, w, lane);
      TC_PROBE(if (gt == 0) ms->probe[kTActTower] += clock64() - t_obs;)
      if constexpr (kChunk) {
        // ---- chunked mean head [C*A, 256] from L2: warp w takes actions w, w+4, ..., its weight row in registers,
        //      one warp-reduced dot product per environment; lane e then samples (e, a) ----
        float* cact = chunk_smem(ms)->act;
        for (int a = w; a < act; a += 4) {
          const float4* wr = reinterpret_cast<const float4*>(P + p.L.mw + (size_t)a * kH);
          const float4 w0 = __ldg(wr + lane), w1 = __ldg(wr + 32 + lane);
          float mine = 0.f;
#pragma unroll 4
          for (int e = 0; e < kNE; ++e) {
            const float4 g0 = *reinterpret_cast<const float4*>(h3 + e * kH + lane * 4);
            const float4 g1 = *reinterpret_cast<const float4*>(h3 + e * kH + 128 + lane * 4);
            float s = g0.x * w0.x + g0.y * w0.y + g0.z * w0.z + g0.w * w0.w + g1.x * w1.x + g1.y * w1.y +
                      g1.z * w1.z + g1.w * w1.w;
            s = rb::warp_sum(s);
            if (lane == e) mine = s;
          }
          if (lane < nE) {
            const int64_t row = e0 + lane;
            const float mean = mine + P[p.L.mb + a];
            const float sd = expf(P[p.L.logstd + a]);
            const float z = p.policy_noise ? p.policy_noise[((size_t)t * B + row) * act + a]
                                           : policy_draw(p.seed_p, (unsigned long long)(row * act + a),
                                                         p.offset_p + 4ull * (c_p + (uint64_t)t));
            const float xa = mean + sd * z;
            const float d = xa - mean;
            const size_t o = ((size_t)t * B + row) * act + a;
            p.actions[o] = xa;
            p.logp[o] = -(d * d) / (2.0f * (sd * sd)) - logf(sd) - kHalfLog2Pi;
            cact[lane * kMaxActChunk + a] = xa;
          }
        }
      } else {
      // ---- mean head + Normal sample + log-prob: one (env, action) pair per thread.  Each thread does its own
      //      256-long dot product (float4 reads rotated by the lane so that a warp touches every bank once): no
      //      warp reductions, no shared-memory hand-off between head and sampling ----
      for (int i = gt; i < kNE * act; i += 128) {
        const int e = i / act, a = i - e * act;
        const float4* hr = reinterpret_cast<const float4*>(h3 + e * kH);
        const float4* wr = reinterpret_cast<const float4*>(ms->mw + a * kH);
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll 8
        for (int j = 0; j < 64; ++j) {
          const int kk = (j + lane) & 63;
          const float4 hv = hr[kk], wv = wr[kk];
          s0 = fmaf(hv.x, wv.x, s0);
          s1 = fmaf(hv.y, wv.y, s1);
          s2 = fmaf(hv.z, wv.z, s2);
          s3 = fmaf(hv.w, wv.w, s3);
        }
        const float mean = ((s0 + s1) + (s2 + s3)) + P[p.L.mb + a];
        if (e < nE) {
          const int64_t row = e0 + e;
          const float ls = P[p.L.logstd + a];
          const float sd = expf(ls);
          float z;
          if (p.policy_noise) {
            z = p.policy_noise[((size_t)t * B + row) * act + a];
          } else {
            z = policy_draw(p.seed_p, (unsigned long long)(row * act + a), p.offset_p + 4ull * (c_p + (uint64_t)t));
          }
          const float xa = mean + sd * z;
          const float d = xa - mean;
          const float var = sd * sd;
          const size_t o = ((size_t)t * B + row) * act + a;
          p.actions[o] = xa;
          p.logp[o] = -(d * d) / (2.0f * var) - logf(sd) - kHalfLog2Pi;
          ms->act[e * kMaxActTc + a] = xa;
        }
      }
      }
      TC_PROBE(if (gt == 0) ms->probe[kTSample] += clock64() - t_obs;)
      // ---- env finish, shared with the env warps (barrier 4 = actor + env groups): #1 actions sampled / h3 dead,
      //      #2 zs + eps in the actor buffer, #3 next observation operand complete (#2 and #3 once per sub-step) ----
      named_sync(4, 256);
      for (int c = 0; c < Cn; ++c) {
        named_sync(4, 256);
        env_finish4<kChunk, kStats>(*pa, ms, obuf, ob_half, reinterpret_cast<const float*>(abuf),
                            reinterpret_cast<const float*>(abuf + kAbufHalf), w, lane, t * Cn + c, e0, nE, sg.nkb0, c_e,
                            boot);
        rb::tma::fence_proxy_async();
        named_sync(4, 256);
      }
    }
  } else if (warp >= 8) {
    // ================= value tower: layers, value head, truncation bootstrap =================
    const int w = warp & 3;
    const float* bias[3] = {P + p.L.vb0, P + p.L.vb1, P + p.L.vb2};
    float* g3 = reinterpret_cast<float*>(vbuf);
    uint32_t p_obs = 0;
    for (int t = 0; t <= T; ++t) {
      if (t > 0) {
        mbar_wait(&ms->obs_ready, p_obs);
        p_obs ^= 1u;
      }
      // the value tower runs with N = 64 columns when any environment was flagged for the truncation bootstrap
      // (columns 32..63 = its pre-reset observation)
      const int nv = (*reinterpret_cast<volatile int*>(&ms->nflag) > 0) ? 2 * kNE : kNE;
      TC_PROBE(const long long t_obs = *reinterpret_cast<volatile long long*>(&ms->t_obs);
               const bool pr = (tid & 127) == 0 && t < T;)
      const uint32_t s0 = (uint32_t)t * n_tower, s1 = s0 + 2u * (uint32_t)sg.nkb0, s2 = s1 + 16u;
      if (nv == kNE) {
        tower_layer<kNE>(ms, ring_a, kValSlot0, s0, sg.nkb0, obuf_a, ob_half, 4096u, bias[0], vbuf, kVbufHalf, 4096u, 0, 2, w, lane);
        tower_layer<kNE>(ms, ring_a, kValSlot0, s1, 8, vbuf_a, kVbufHalf, 4096u, bias[1], vbuf, kVbufHalf, 4096u, 0, 2, w, lane);
        tower_layer<kNE>(ms, ring_a, kValSlot0, s2, 8, vbuf_a, kVbufHalf, 4096u, bias[2], vbuf, kVbufHalf, 4096u, 1, 2, w, lane);
      } else {
        tower_layer<2 * kNE>(ms, ring_a, kValSlot0, s0, sg.nkb0, obuf_a, ob_half, 4096u, bias[0], vbuf, kVbufHalf, 4096u, 0, 2, w, lane);
        tower_layer<2 * kNE>(ms, ring_a, kValSlot0, s1, 8, vbuf_a, kVbufHalf, 4096u, bias[1], vbuf, kVbufHalf, 4096u, 0, 2, w, lane);
        tower_layer<2 * kNE>(ms, ring_a, kValSlot0, s2, 8, vbuf_a, kVbufHalf, 4096u, bias[2], vbuf, kVbufHalf, 4096u, 1, 2, w, lane);
      }
      TC_PROBE(if (pr) ms->probe[kTValTower] += clock64() - t_obs;)
      // ---- value head (columns 0..31: V(obs_t)) and bootstrap (columns 32..63: V(final_obs_{t-1}) where flagged) ----
      //      chunked: C outputs per environment, the bootstrap uses output 0 and goes to the chunk's last column
      if constexpr (kChunk) {
        for (int e = w; e < nv; e += 4) {
          const int eb = e < kNE ? e : e - kNE;
          if (eb >= nE || (e >= kNE && !ms->flag[eb])) continue;  // warp-uniform
          for (int c = 0; c < Cn; ++c) {
            const float v = dot256(g3 + e * kH, ms->mw + c * kH, lane);
            if (lane != 0) continue;
            if (e < kNE) {
              p.values[((size_t)t * B + e0 + e) * Cn + c] = v;
            } else {
              if (c == 0)
                p.rewards[((size_t)(t - 1) * B + e0 + eb) * Cn + Cn - 1] = __fadd_rn(ms->rew[eb], __fmul_rn(p.gamma, v));
              p.final_values[(size_t)(e0 + eb) * Cn + c] = v;
            }
          }
        }
      } else {
      for (int e = w; e < nv; e += 4) {
        if (e < kNE) {
          const float v = dot256(g3 + e * kH, ms->vw, lane);
          if (lane == 0 && e < nE) p.values[(size_t)t * B + e0 + e] = v;
        } else {
          const int eb = e - kNE;
          if (ms->flag[eb] && eb < nE) {  // warp-uniform
            const float v = dot256(g3 + e * kH, ms->vw, lane);
            if (lane == 0) {
              p.rewards[(size_t)(t - 1) * B + e0 + eb] = __fadd_rn(ms->rew[eb], __fmul_rn(p.gamma, v));
              p.final_values[e0 + eb] = v;
            }
          }
        }
      }
      }
      __syncwarp();
      TC_PROBE(if (pr) ms->probe[kTValHead] += clock64() - t_obs;)
      if (lane == 0) mbar_arrive(&ms->vhead);
    }
  } else {
    // ================= env warps: noise, x.W_s, dynamics finish, auto-reset, next observation operand =================
    const int ew = warp, gt = tid;
    const int g = lane >> 2, tq = lane & 3;
    float* zs = reinterpret_cast<float*>(abuf);  // [32][obs] fp32, aliases the actor buffer (free between barrier #1 and the next L0)
    float* eps_s = reinterpret_cast<float*>(abuf + kAbufHalf);  // [32][obs] fp32 draws of this step
    const int nk = sg.nkb0;                       // observation columns per lane
    uint32_t p_vh = 0;
    for (int t = 0; t < T * Cn; ++t) {  // env (sub-)steps
      const int sub = kChunk ? t % Cn : 0;
      // ---- 1. Philox draws of this step for my 8 environments (same streams / order as env_finish_kernel; chunked:
      //         env_substep_kernel, window ((c_e + n) C + c) * 64) ----
      float eps[8][4], eps_r[8], uu[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        eps_r[i] = 0.f;
        uu[i] = 1.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) eps[i][k] = 0.f;
      }
      if (!p.env_noise) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int e = ew * 8 + i;
          if (e < nE) {
            const EnvDraws d = env_draws(p.seed_e, (unsigned long long)(e0 + e) * 32ull + lane,
                                         (c_e * (uint64_t)Cn + (uint64_t)t) * 64ull, nk, lane == 0);
#pragma unroll
            for (int k = 0; k < 4; ++k) eps[i][k] = d.e[k];
            eps_r[i] = d.er;
            uu[i] = d.u;
          }
        }
      }
      // ---- 2. x.W_s of this step (the observation operand is complete: barrier #3 of the previous step) ----
      LayerAcc<kNE, 1> zacc;
      layer_mma<kNE, 1>(zacc, ms, ring_a, kEnvSlot0, kEnvSlots, (uint32_t)t * n_env, sg.nkb0, obuf_a, ob_half, 4096u, lane);
      TC_PROBE(if (gt == 0 && sub == 0) ms->probe[kTEnvProduct] += clock64() - ms->t_obs;)
      // ---- 3. wait for the value head, meet the actor group (#1: h3 dead, actions sampled), then park x.W_s
      //         (fp32 [32][obs]) and this step's draws in the free actor buffer ----
      //         (chunked: at the first sub-step; the later ones overwrite only the actor buffer and the observation
      //         rows 0..31, which no tower reads before the next chunk step)
      if (sub == 0) {
        mbar_wait(&ms->vhead, p_vh);  // the value head of this step has consumed flag / rew of the previous step
        p_vh ^= 1u;
        TC_PROBE(if (gt == 0) ms->probe[kTEnvVhead] += clock64() - ms->t_obs;)
        named_sync(4, 256);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int e = ew * 8 + i;
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (k < nk) eps_s[e * obs + lane + 32 * k] = eps[i][k];
        if (lane == 0) {
          ms->er[e] = eps_r[i];
          ms->uu[e] = uu[i];
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int c = h * 64 + ew * 16 + g + 8 * r;  // observation column (row of the env product)
          if (c < obs) {
#pragma unroll
            for (int cc = 0; cc < kNE / 8; ++cc)
#pragma unroll
              for (int u = 0; u < 2; ++u) zs[(8 * cc + 2 * tq + u) * obs + c] = zacc.d[0][h][4 * cc + 2 * r + u] * out_scale;
          }
        }
      named_sync(4, 256);
      // ---- 4. finish 4 environments per warp (the actor group takes environments 0..15) ----
      env_finish4<kChunk, kStats>(*pa, ms, obuf, ob_half, zs, eps_s, 4 + ew, lane, t, e0, nE, nk, c_e, boot);
      rb::tma::fence_proxy_async();
      named_sync(4, 256);
      if (sub == Cn - 1 && gt == 0) {
        int n = 0;
        for (int e = 0; e < kNE; ++e) n += ms->flag[e];
        ms->nflag = n;
        TC_PROBE(const long long now = clock64(); ms->probe[kTObsReady] += now - ms->t_obs; ++ms->probe[kTSteps];
                 ms->t_obs = now;)
        __threadfence_block();
        mbar_arrive(&ms->obs_ready);
      }
    }
    if (gt < nE) p.elapsed[e0 + gt] = ms->el[gt];  // written by this group, ordered by the last named barrier
    if constexpr (kStats)
      if (gt < nE) es.ret[e0 + gt] = stats_smem<kChunk>(ms)->ret[gt];
  }
  TC_PROBE(__syncthreads(); if (tid < kProbeSlots) g_tc_probe[blockIdx.x * kProbeSlots + tid] = ms->probe[tid];)
}

// ---- weight packing: fp32 parameters -> the streamed [stage][hi|lo][128 rows x 32 k] SWIZZLE_64B fp16 tiles --------------
struct PackArgs {
  const float* params;
  const float* w_s;  // [obs_in, obs_out]
  uint8_t* pack;
  int64_t w_off[6];  // a0 v0 a1 v1 a2 v2 weight offsets in params ([256 out, in] row-major)
  int obs;
};

__global__ void __launch_bounds__(256) pack_kernel(PackArgs a) {
  const Segs sg = make_segs(a.obs);
  const int64_t items = (int64_t)sg.total * 128 * 4;  // (stage, row, 16-byte chunk)
  const float scale = (float)(1 << kWScaleLog2);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += (int64_t)gridDim.x * blockDim.x) {
    const int cp = (int)(i & 3), r = (int)((i >> 2) & 127), stage = (int)(i >> 9);
    // which segment / tile / k-block
    int seg, rel;
    if (stage < sg.a0) { seg = -1; rel = stage; }
    else if (stage < sg.v0) { seg = 0; rel = stage - sg.a0; }
    else if (stage < sg.a1) { seg = 1; rel = stage - sg.v0; }
    else if (stage < sg.v1) { seg = 2; rel = stage - sg.a1; }
    else if (stage < sg.a2) { seg = 3; rel = stage - sg.v1; }
    else if (stage < sg.v2) { seg = 4; rel = stage - sg.a2; }
    else { seg = 5; rel = stage - sg.v2; }
    const int ntile = seg < 0 ? 1 : 2;  // stream order inside a layer: k-block outer, M tile inner (the MMA issue order)
    const int kb = rel / ntile, m = rel - kb * ntile;
    const int in_dim = (seg < 2) ? a.obs : kH;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = kb * 32 + cp * 8 + j;
      const int out = m * 128 + r;
      float w;
      if (seg < 0) w = (out < a.obs) ? a.w_s[(size_t)k * a.obs + out] : 0.f;  // A[c_out][k_in] = W_s[k_in][c_out]
      else w = a.params[a.w_off[seg] + (size_t)out * in_dim + k];
      v[j] = w * scale;
    }
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __half2 hh = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
      const float2 hf = __half22float2(hh);
      const __half2 ll = __floats2half2_rn(v[2 * j] - hf.x, v[2 * j + 1] - hf.y);
      h[j] = *reinterpret_cast<const uint32_t*>(&hh);
      l[j] = *reinterpret_cast<const uint32_t*>(&ll);
    }
    uint8_t* dst = a.pack + (size_t)stage * kStageBytes + r * 64 + ((cp ^ ((r >> 1) & 3)) << 4);
    *reinterpret_cast<uint4*>(dst) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(dst + kHalfTile) = make_uint4(l[0], l[1], l[2], l[3]);
  }
}

}  // namespace

extern "C" int rb200_rollout_tc_supported(const rb200_mlp_layout* L, int num_action_chunks, int B) {
  if (!L) return RB200_E_NULL;
  const int Cn = num_action_chunks;
  if (L->hidden != kH) return RB200_E_UNSUPPORTED;
  if (Cn == 1) {
    if (L->act_dim <= 0 || L->act_dim > kMaxActTc || L->value_dim != 1) return RB200_E_UNSUPPORTED;
  } else {
    if (Cn < 2 || Cn > kMaxChunks || L->value_dim != Cn) return RB200_E_UNSUPPORTED;
    if (L->act_dim <= 0 || L->act_dim > kMaxActChunk || L->act_dim % Cn != 0 || L->act_dim / Cn > kMaxActTc)
      return RB200_E_UNSUPPORTED;
  }
  if (L->obs_dim < 32 || L->obs_dim > kMaxObsTc || (L->obs_dim % 32) != 0) return RB200_E_UNSUPPORTED;
  if (B <= 0) return RB200_E_UNSUPPORTED;
  return RB200_OK;
}

namespace {
// the pack holds the hidden layers and W_s only: any layout one of the kernels runs (value_dim == C in both)
int pack_supported(const rb200_mlp_layout* L) { return rb200_rollout_tc_supported(L, L->value_dim, 1); }
}  // namespace

extern "C" int64_t rb200_rollout_tc_pack_bytes(const rb200_mlp_layout* L) {
  if (!L || pack_supported(L)) return 0;
  return (int64_t)make_segs(L->obs_dim).total * kStageBytes;
}

extern "C" int rb200_rollout_tc_prepare(const rb200_mlp_layout* L, const float* params, const float* w_s, void* pack,
                                        rb200_stream_t stream) {
  if (!L || !params || !w_s || !pack) return RB200_E_NULL;
  int e = pack_supported(L);
  if (e) return e;
  if (reinterpret_cast<uintptr_t>(pack) & 15) return RB200_E_ALIGN;
  PackArgs a{};
  a.params = params; a.w_s = w_s; a.pack = static_cast<uint8_t*>(pack); a.obs = L->obs_dim;
  a.w_off[0] = L->bw0; a.w_off[1] = L->vw0; a.w_off[2] = L->bw1; a.w_off[3] = L->vw1; a.w_off[4] = L->bw2; a.w_off[5] = L->vw2;
  const int64_t items = (int64_t)make_segs(L->obs_dim).total * 512;
  pack_kernel<<<(int)((items + 255) / 256), 256, 0, rb::as_stream(stream)>>>(a);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

namespace {
template <bool kChunk, bool kStats>
int launch_rollout_tc(const rb200_mlp_layout* L, const float* params, const void* pack, const rb200_rollout_args& r,
                      rb200_stream_t stream) {
  if (!params || !pack || !r.w_a || !r.states || !r.actions || !r.logprobs || !r.values || !r.rewards ||
      !r.terminations || !r.truncations || !r.dones || !r.final_obs || !r.final_values || !r.elapsed)
    return RB200_E_NULL;
  if (r.T <= 0) return RB200_E_SHAPE;
  if (reinterpret_cast<uintptr_t>(pack) & 15) return RB200_E_ALIGN;
  TcArgs a{};
  a.L = *L; a.params = params; a.pack = static_cast<const uint8_t*>(pack); a.w_a = r.w_a; a.states = r.states;
  a.actions = r.actions; a.logp = r.logprobs; a.values = r.values; a.rewards = r.rewards; a.term = r.terminations;
  a.trunc = r.truncations; a.done = r.dones; a.final_obs = r.final_obs; a.final_values = r.final_values;
  a.elapsed = r.elapsed; a.policy_noise = r.policy_noise; a.env_noise = r.env_noise; a.counter_p = r.counter_policy;
  a.counter_e = r.counter_env; a.seed_p = r.seed_policy; a.seed_e = r.seed_env; a.offset_p = r.offset_policy;
  a.T = r.T; a.B = r.B; a.obs = L->obs_dim; a.act = L->act_dim; a.max_episode_steps = r.max_episode_steps;
  a.auto_reset = r.auto_reset; a.bootstrap_on_done = r.bootstrap_on_done; a.gamma = (float)r.gamma;
  a.p_term = (float)r.p_term; a.noise_std = (float)r.noise_std; a.reward_noise_std = (float)r.reward_noise_std;
  a.C = r.num_action_chunks;
  const int smem = kSmemTotal<kChunk, kStats>;
  static bool attr_done = false;
  if (!attr_done) {
    RB_CHECK_CUDA(cudaFuncSetAttribute(rollout_tc_kernel<kChunk, kStats>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       smem));
    attr_done = true;
  }
  const int grid = (r.B + kNE - 1) / kNE;
  rollout_tc_kernel<kChunk, kStats><<<grid, kThreads, smem, rb::as_stream(stream)>>>(
      a, EpStats{r.episode_return, r.episode_acc});
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
}  // namespace

#ifdef RB200_ROLLOUT_TC_PROBE
// probe builds only: where the next rollout_tc_kernel launches write their slots ([grid][slots] uint64, device memory)
extern "C" int rb200_rollout_tc_probe_buffer(unsigned long long* buf) {
  RB_CHECK_CUDA(cudaMemcpyToSymbol(g_tc_probe, &buf, sizeof(buf)));
  return RB200_OK;
}
extern "C" int rb200_rollout_tc_probe_slots() { return kProbeSlots; }
#endif

extern "C" int rb200_rollout_tc(const rb200_mlp_layout* L, const float* params, const void* pack,
                                const rb200_rollout_args* a, rb200_stream_t stream) {
  if (!a) return RB200_E_NULL;
  int e = rb200_rollout_tc_supported(L, a->num_action_chunks, a->B);
  if (e) return e;
  if (!a->episode_return != !a->episode_acc) return RB200_E_NULL;
  const bool chunk = a->num_action_chunks > 1, stats = a->episode_return != nullptr;
  if (!chunk && !stats) return launch_rollout_tc<false, false>(L, params, pack, *a, stream);
  if (chunk && !stats) return launch_rollout_tc<true, false>(L, params, pack, *a, stream);
  if (!chunk) return launch_rollout_tc<false, true>(L, params, pack, *a, stream);
  return launch_rollout_tc<true, true>(L, params, pack, *a, stream);
}
