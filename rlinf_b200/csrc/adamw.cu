// K4: global grad-norm clip + AdamW on one flat fp32 buffer (params | grads | exp_avg | exp_avg_sq).
// Reference: FSDPModelManager.optimizer_step, rlinf/hybrid_engines/fsdp/fsdp_model_manager.py:429-463;
// the no_shard clip path strategy/fsdp.py:363-369 == torch.nn.utils.clip_grad_norm_(params, max_norm):
//     total_norm = ||g||_2 ; coef = min(1, max_norm / (total_norm + 1e-6)) ; g *= coef
// non-finite norm => the optimiser step is skipped (:442-447); torch.optim.AdamW (decoupled decay):
//     p *= 1 - lr*wd ; m += (g-m)(1-b1) ; v = b2 v + (1-b2) g^2
//     p -= (lr / (1-b1^t)) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
// with two lr groups (actor / value_head, build_optimizer :501-590).
// 28 B/param algorithmic (read p,g,m,v; write p,m,v) + 4 B/param for the norm pass.
// The decision (skip / clip coefficient / step count) is taken on the device: no host sync.
#include "common.cuh"

namespace {

constexpr int kMaxGroups = 8;
struct Groups {
  int64_t end[kMaxGroups];
  int n;
};

__global__ void __launch_bounds__(256) sqnorm_kernel(const float* __restrict__ g, int64_t n, double* __restrict__ out) {
  __shared__ double red[32];
  double v[1] = {0.0};
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool al = (reinterpret_cast<uintptr_t>(g) & 15) == 0;
  const int64_t n4 = al ? n / 4 : 0;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (int64_t k = i0; k < n4; k += stride) {
    const float4 x = g4[k];
    v[0] += (double)x.x * x.x + (double)x.y * x.y + (double)x.z * x.z + (double)x.w * x.w;
  }
  for (int64_t k = n4 * 4 + i0; k < n; k += stride) v[0] += (double)g[k] * g[k];
  rb::block_sum<1>(v, red);
  if (threadIdx.x == 0) atomicAdd(out, v[0]);
}

// state: {step_count, last_grad_norm, last_clip_coef, skipped}
__global__ void adamw_prepare_kernel(const double* __restrict__ grad_sq, double* __restrict__ state, float max_norm,
                                     float grad_scale) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  // grads in the buffer are (grad_scale x) the true gradient sum; the norm is of the scaled gradient
  const double norm = sqrt(grad_sq[0]) * (double)grad_scale;
  const float norm_f = (float)norm;
  const bool finite = isfinite(norm_f);
  state[1] = norm;
  if (!finite) {
    state[2] = 0.0;
    state[3] = 1.0;
    return;
  }
  float coef = 1.0f;
  if (max_norm > 0.0f) {
    coef = __fdiv_rn(max_norm, __fadd_rn(norm_f, 1e-6f));
    coef = fminf(coef, 1.0f);
  }
  state[2] = (double)coef;
  state[3] = 0.0;
  state[0] += 1.0;
}

__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                    float* __restrict__ m, float* __restrict__ v, int64_t n,
                                                    Groups grp, const double* __restrict__ lr_dev, double beta1,
                                                    double beta2, double eps, double wd, float grad_scale,
                                                    const double* __restrict__ state) {
  if (state[3] != 0.0) return;  // non-finite grad norm: skip the whole step
  const double step = state[0];
  const float gmul = (float)state[2] * grad_scale;  // clip coefficient x (1/world_size etc.)
  // scalar factors are formed in double (as Python floats in torch.optim) and rounded once
  const double bc1 = 1.0 - pow(beta1, step);
  const float bc2_sqrt = (float)sqrt(1.0 - pow(beta2, step));
  const float one_m_b1 = (float)(1.0 - beta1), b2 = (float)beta2, one_m_b2 = (float)(1.0 - beta2);
  const float eps_f = (float)eps;
  // lr < 0 marks a FROZEN group: parameters, moments untouched (torch.optim.AdamW skips parameters that are not in a
  // param group / have grad None: the actor during critic warm-up, fsdp_model_manager.py:523-531; a value head that
  // received no gradient).  Encoded as step_size = NaN.
  float decay[kMaxGroups], step_size[kMaxGroups];
#pragma unroll
  for (int k = 0; k < kMaxGroups; ++k) {
    const double lr = k < grp.n ? lr_dev[k] : 0.0;  // read at execution time: LR schedules under CUDA-graph replay
    decay[k] = (float)(1.0 - lr * wd);
    step_size[k] = lr < 0.0 ? __int_as_float(0x7fc00000) : (float)(lr / bc1);
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float dk = decay[0], sk = step_size[0];
#pragma unroll
    for (int k = 1; k < kMaxGroups; ++k)
      if (k < grp.n && i >= grp.end[k - 1]) {
        dk = decay[k];
        sk = step_size[k];
      }
    if (sk != sk) continue;  // frozen group
    const float gi = __fmul_rn(g[i], gmul);
    float pi = p[i];
    pi = __fmul_rn(pi, dk);
    float mi = m[i];
    mi = __fadd_rn(mi, __fmul_rn(__fsub_rn(gi, mi), one_m_b1));  // lerp_(g, 1-b1)
    float vi = v[i];
    vi = __fadd_rn(__fmul_rn(vi, b2), __fmul_rn(__fmul_rn(gi, gi), one_m_b2));  // mul_(b2).addcmul_(g,g,1-b2)
    const float denom = __fadd_rn(__fdiv_rn(sqrtf(vi), bc2_sqrt), eps_f);
    pi = __fsub_rn(pi, __fmul_rn(sk, __fdiv_rn(mi, denom)));  // addcdiv_(m, denom, -step_size)
    p[i] = pi;
    m[i] = mi;
    v[i] = vi;
  }
}

}  // namespace

extern "C" int rb200_grad_sqnorm(const float* grads, int64_t n, double* out_sq, rb200_stream_t stream) {
  if (!grads || !out_sq) return RB200_E_NULL;
  if (n <= 0) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  RB_CHECK_CUDA(cudaMemsetAsync(out_sq, 0, sizeof(double), st));
  int64_t blocks = (n / 4 + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * 4;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  sqnorm_kernel<<<(int)blocks, 256, 0, st>>>(grads, n, out_sq); rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_adamw_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                                    const int64_t* group_end_host, const double* group_lr_dev, int n_groups,
                                    double beta1, double beta2, double eps, double weight_decay, float max_grad_norm,
                                    float grad_scale, const double* grad_sq, double* state, rb200_stream_t stream) {
  if (!params || !grads || !exp_avg || !exp_avg_sq || !group_end_host || !group_lr_dev || !grad_sq || !state)
    return RB200_E_NULL;
  if (n <= 0 || n_groups <= 0 || n_groups > kMaxGroups) return RB200_E_SHAPE;
  Groups grp;
  grp.n = n_groups;
  int64_t prev = 0;
  for (int k = 0; k < kMaxGroups; ++k) {
    grp.end[k] = k < n_groups ? group_end_host[k] : n;
    if (grp.end[k] < prev || grp.end[k] > n) return RB200_E_SHAPE;
    prev = grp.end[k];
  }
  if (grp.end[n_groups - 1] != n) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  adamw_prepare_kernel<<<1, 32, 0, st>>>(grad_sq, state, max_grad_norm, grad_scale); rb::count_launch();
  int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * 4;
  if (blocks > cap) blocks = cap;
  adamw_kernel<<<(int)blocks, 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, n, grp, group_lr_dev, beta1, beta2, eps,
                                            weight_decay, grad_scale, state); rb::count_launch();
  RB_RETURN_LAUNCH();
}
