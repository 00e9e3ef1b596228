// Flat Adam: one launch over the scorer's flat parameter / gradient buffers (torch.optim.Adam semantics:
// exp_avg.lerp_(g, 1-b1); exp_avg_sq = b2*v + (1-b2) g^2; p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps)).
// The reference trains with torch.optim from its config (allrank/main.py:82); this kernel is the equivalent
// single-launch optimiser for the flat storage (128-bit vectorised, HBM-bound: 28 bytes per parameter).
#include <cmath>
#include <cstdint>
#include <cuda_runtime.h>

#include "common.h"

namespace arb {

__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                   float* __restrict__ m, float* __restrict__ v, long long n,
                                                   float lr_over_bc1, float beta1, float beta2, float eps,
                                                   float inv_sqrt_bc2, float weight_decay, float grad_scale,
                                                   const float* __restrict__ dev_state) {
  const long long i4 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) return;
  if (dev_state) { lr_over_bc1 = dev_state[1]; inv_sqrt_bc2 = dev_state[2]; }   // step count kept on the device (graphs)
  if (i4 + 4 <= n) {
    float4 pp = *reinterpret_cast<float4*>(p + i4);
    const float4 gg = *reinterpret_cast<const float4*>(g + i4);
    float4 mm = *reinterpret_cast<float4*>(m + i4);
    float4 vv = *reinterpret_cast<float4*>(v + i4);
    float* pa = &pp.x; const float* ga = &gg.x; float* ma = &mm.x; float* va = &vv.x;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float gr = ga[e] * grad_scale + weight_decay * pa[e];
      ma[e] = ma[e] + (gr - ma[e]) * (1.0f - beta1);
      va[e] = beta2 * va[e] + (1.0f - beta2) * gr * gr;
      pa[e] -= lr_over_bc1 * ma[e] / (sqrtf(va[e]) * inv_sqrt_bc2 + eps);
    }
    *reinterpret_cast<float4*>(p + i4) = pp;
    *reinterpret_cast<float4*>(m + i4) = mm;
    *reinterpret_cast<float4*>(v + i4) = vv;
  } else {
    for (long long i = i4; i < n; ++i) {
      const float gr = g[i] * grad_scale + weight_decay * p[i];
      m[i] = m[i] + (gr - m[i]) * (1.0f - beta1);
      v[i] = beta2 * v[i] + (1.0f - beta2) * gr * gr;
      p[i] -= lr_over_bc1 * m[i] / (sqrtf(v[i]) * inv_sqrt_bc2 + eps);
    }
  }
}

// Step counter on the device (CUDA-graph replay: the host cannot pass a new step number): state[0] += 1, then the
// bias-corrected factors of that step for adam_kernel.
__global__ void adam_prep_kernel(float* __restrict__ state, float lr, float beta1, float beta2) {
  const double t = double(state[0]) + 1.0;
  state[0] = float(t);
  state[1] = float(double(lr) / (1.0 - pow(double(beta1), t)));
  state[2] = float(1.0 / sqrt(1.0 - pow(double(beta2), t)));
}

}  // namespace arb

static int adam_check(const float* params, const float* grads, const float* exp_avg, const float* exp_avg_sq, int64_t n) {
  if (!params || !grads || !exp_avg || !exp_avg_sq || n <= 0) {
    arb_set_error("arb_adam_step: null pointer or bad argument");
    return ARB_E_INVALID_ARG;
  }
  if ((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) | reinterpret_cast<uintptr_t>(exp_avg) |
       reinterpret_cast<uintptr_t>(exp_avg_sq)) & 15) {
    arb_set_error("arb_adam_step: buffers must be 16-byte aligned");
    return ARB_E_INVALID_ARG;
  }
  return ARB_OK;
}

extern "C" int32_t arb_adam_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                                     float lr, float beta1, float beta2, float eps, float weight_decay, float* state,
                                     float grad_scale, void* stream) {
  if (int rc = adam_check(params, grads, exp_avg, exp_avg_sq, n)) return rc;
  if (!state) { arb_set_error("arb_adam_step_dev: null state"); return ARB_E_INVALID_ARG; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long threads = (n + 3) / 4;
  ProfScope ps(ARB_PROF_OPTIM, 28.0 * double(n), st);
  if (int rc = launch(arb::adam_prep_kernel, dim3(1), dim3(1), 0, st, /*pdl=*/false, state, lr, beta1, beta2)) return rc;
  return launch(arb::adam_kernel, dim3(unsigned((threads + 255) / 256)), dim3(256), 0, st, /*pdl=*/false, params, grads,
                exp_avg, exp_avg_sq, n, 0.f, beta1, beta2, eps, 0.f, weight_decay, grad_scale, state);
}

extern "C" int32_t arb_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                                 float lr, float beta1, float beta2, float eps, float weight_decay, int32_t step,
                                 float grad_scale, void* stream) {
  if (!params || !grads || !exp_avg || !exp_avg_sq || n <= 0 || step <= 0) {
    arb_set_error("arb_adam_step: null pointer or bad argument");
    return ARB_E_INVALID_ARG;
  }
  if ((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) | reinterpret_cast<uintptr_t>(exp_avg) |
       reinterpret_cast<uintptr_t>(exp_avg_sq)) & 15) {
    arb_set_error("arb_adam_step: buffers must be 16-byte aligned");
    return ARB_E_INVALID_ARG;
  }
  const double bc1 = 1.0 - std::pow(double(beta1), double(step));
  const double bc2 = 1.0 - std::pow(double(beta2), double(step));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long threads = (n + 3) / 4;
  ProfScope ps(ARB_PROF_OPTIM, 28.0 * double(n), st);
  return launch(arb::adam_kernel, dim3(unsigned((threads + 255) / 256)), dim3(256), 0, st, /*pdl=*/false, params, grads,
                exp_avg, exp_avg_sq, n, float(lr / bc1), beta1, beta2, eps, float(1.0 / std::sqrt(bc2)), weight_decay,
                grad_scale, nullptr);
}
