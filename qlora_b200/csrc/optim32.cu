// 32-bit Lion, RMSprop and AdEMAMix: one elementwise kernel template over the update rule, fp32 state, fp32 math.
//
// Replaces (upstream bitsandbytes, un-vendored; reached from HF's optimizer factory for optim='lion_32bit',
// 'paged_lion_32bit', 'rmsprop_bnb', 'rmsprop_bnb_32bit', 'ademamix', 'paged_ademamix_32bit'):
//   clion32bit_grad_*, crmsprop32bit_grad_*   (kernel kOptimizer32bit1State<T, LION | RMSPROP>)
//   cademamix32bit_grad_*                      (kernel kOptimizer32bit2State<T, ADEMAMIX>)
// Rules (g = gnorm_scale * grad; every operation a correctly rounded fp32 one, so no FMA contraction):
//   Lion:     c = b1*m + (1-b1)*g ; if (wd > 0) p = p*(1 - lr*wd) ; p = p - lr*sign(c) ; m = b2*m + (1-b2)*g
//   RMSprop:  if (wd > 0) g = g + wd*p ; v = alpha*v + (1-alpha)*g*g ; p = p - lr*(g / (sqrt(v) + eps))
//   AdEMAMix: m1 = b1*m1 + (1-b1)*g ; m2 = b3_t*m2 + (1-b3_t)*g ; nu = b2*nu + (1-b2)*g*g
//             p = p - lr*((m1/c1 + alpha_t*m2) / (sqrt(nu)/c2 + eps)) ; if (wd > 0) p = p*(1 - lr*wd)
// AdEMAMix's per-step scalars (c1, c2, alpha_t, b3_t) are computed from the DEVICE step count in double and rounded to fp32
// once per launch, so a launch depends on no host state and one captured launch serves every step.  HBM-bound: Lion and
// RMSprop move 2 x (p, state) + g, AdEMAMix 2 x (p, m1, m2, nu) + g per element.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include "nf4_common.cuh"
#include "qb200_internal.h"

namespace qb200 {

enum class Rule { kLion, kRMSprop, kAdEMAMix };

struct Optim32Hyper {
  float lr, beta1, beta2, beta3, alpha, eps, weight_decay, decay;   // decay = 1 - lr*wd (wd > 0), else 1
  float t_alpha, t_beta3;                                            // AdEMAMix schedules; 0 = none
};

struct StepScalars {
  float c1, c2, alpha_t, beta3_t;
};

template <Rule R>
__device__ __forceinline__ StepScalars step_scalars(const Optim32Hyper& h, const float* step_dev) {
  StepScalars s{1.0f, 1.0f, h.alpha, h.beta3};
  if constexpr (R == Rule::kAdEMAMix) {
    const double t = double(__ldg(step_dev));
    s.c1 = float(1.0 - pow(double(h.beta1), t));
    s.c2 = float(sqrt(1.0 - pow(double(h.beta2), t)));
    if (h.t_alpha > 0.0f) s.alpha_t = float(fmin(t * double(h.alpha) / double(h.t_alpha), double(h.alpha)));
    if (h.t_beta3 > 0.0f) {
      const double lb1 = log(double(h.beta1)), lb3 = log(double(h.beta3)), f = t / double(h.t_beta3);
      s.beta3_t = float(fmin(exp(lb1 * lb3 / ((1.0 - f) * lb3 + f * lb1)), double(h.beta3)));
    }
  }
  return s;
}

// One element: p and g widened to fp32; s0 (and s1, s2 for AdEMAMix) the fp32 state, updated in place.
template <Rule R>
__device__ __forceinline__ float update(float p, float g, float& s0, float& s1, float& s2, const Optim32Hyper& h, const StepScalars& c) {
  if constexpr (R == Rule::kLion) {
    const float u = __fadd_rn(__fmul_rn(h.beta1, s0), __fmul_rn(1.0f - h.beta1, g));
    if (h.decay != 1.0f) p = __fmul_rn(p, h.decay);
    const float sgn = u > 0.0f ? 1.0f : (u < 0.0f ? -1.0f : 0.0f);
    p = __fsub_rn(p, __fmul_rn(h.lr, sgn));
    s0 = __fadd_rn(__fmul_rn(h.beta2, s0), __fmul_rn(1.0f - h.beta2, g));
  } else if constexpr (R == Rule::kRMSprop) {
    if (h.weight_decay > 0.0f) g = __fadd_rn(g, __fmul_rn(h.weight_decay, p));
    s0 = __fadd_rn(__fmul_rn(h.alpha, s0), __fmul_rn(1.0f - h.alpha, __fmul_rn(g, g)));
    p = __fsub_rn(p, __fmul_rn(h.lr, __fdiv_rn(g, __fadd_rn(__fsqrt_rn(s0), h.eps))));
  } else {
    s0 = __fadd_rn(__fmul_rn(h.beta1, s0), __fmul_rn(1.0f - h.beta1, g));
    s1 = __fadd_rn(__fmul_rn(c.beta3_t, s1), __fmul_rn(1.0f - c.beta3_t, g));
    s2 = __fadd_rn(__fmul_rn(h.beta2, s2), __fmul_rn(1.0f - h.beta2, __fmul_rn(g, g)));
    const float num = __fadd_rn(__fdiv_rn(s0, c.c1), __fmul_rn(c.alpha_t, s1));
    const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(s2), c.c2), h.eps);
    p = __fsub_rn(p, __fmul_rn(h.lr, __fdiv_rn(num, den)));
    if (h.decay != 1.0f) p = __fmul_rn(p, h.decay);
  }
  return p;
}

constexpr int kOptimThreads = 256;

// Grid-stride over 16-byte vectors of p and g (VEC elements; the fp32 state moves as VEC/4 float4s per array) when
// every pointer is 16-byte aligned, then a scalar tail; the whole range element by element otherwise.
template <Rule R, typename T>
__global__ void __launch_bounds__(kOptimThreads) optim32bit_kernel(T* __restrict__ p, const T* __restrict__ g, float* __restrict__ s0,
                                                                  float* __restrict__ s1, float* __restrict__ s2, int64_t n, bool vec_ok,
                                                                  Optim32Hyper h, const float* __restrict__ step_dev,
                                                                  const float* __restrict__ gnorm_scale_dev) {
  constexpr int VEC = 16 / sizeof(T);
  constexpr bool kThree = R == Rule::kAdEMAMix;
  const StepScalars c = step_scalars<R>(h, step_dev);
  const float gs = gnorm_scale_dev != nullptr ? __ldg(gnorm_scale_dev) : 1.0f;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t tid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nvec = vec_ok ? n / VEC : 0;
  for (int64_t v = tid; v < nvec; v += stride) {
    const int64_t i0 = v * VEC;
    alignas(16) T pv[VEC];
    alignas(16) T gv[VEC];
    alignas(16) float a[VEC], b[VEC], d[VEC];
    *reinterpret_cast<uint4*>(pv) = *reinterpret_cast<const uint4*>(p + i0);
    *reinterpret_cast<uint4*>(gv) = __ldg(reinterpret_cast<const uint4*>(g + i0));
#pragma unroll
    for (int k = 0; k < VEC / 4; ++k) {
      reinterpret_cast<float4*>(a)[k] = reinterpret_cast<const float4*>(s0 + i0)[k];
      if constexpr (kThree) {
        reinterpret_cast<float4*>(b)[k] = reinterpret_cast<const float4*>(s1 + i0)[k];
        reinterpret_cast<float4*>(d)[k] = reinterpret_cast<const float4*>(s2 + i0)[k];
      }
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j)
      pv[j] = from_f32<T>(update<R>(to_f32<T>(pv[j]), __fmul_rn(gs, to_f32<T>(gv[j])), a[j], b[j], d[j], h, c));
    *reinterpret_cast<uint4*>(p + i0) = *reinterpret_cast<const uint4*>(pv);
#pragma unroll
    for (int k = 0; k < VEC / 4; ++k) {
      reinterpret_cast<float4*>(s0 + i0)[k] = reinterpret_cast<const float4*>(a)[k];
      if constexpr (kThree) {
        reinterpret_cast<float4*>(s1 + i0)[k] = reinterpret_cast<const float4*>(b)[k];
        reinterpret_cast<float4*>(s2 + i0)[k] = reinterpret_cast<const float4*>(d)[k];
      }
    }
  }
  for (int64_t i = nvec * VEC + tid; i < n; i += stride) {
    float a = s0[i], b = 0.0f, d = 0.0f;
    if constexpr (kThree) {
      b = s1[i];
      d = s2[i];
    }
    p[i] = from_f32<T>(update<R>(to_f32<T>(p[i]), __fmul_rn(gs, to_f32<T>(g[i])), a, b, d, h, c));
    s0[i] = a;
    if constexpr (kThree) {
      s1[i] = b;
      s2[i] = d;
    }
  }
}

static bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15u) == 0; }

template <Rule R, typename T>
static int launch_optim32(void* p, const void* g, float* s0, float* s1, float* s2, int64_t n, const Optim32Hyper& h, const float* step_dev,
                          const float* gnorm_scale_dev, cudaStream_t stream, const char* what) {
  constexpr int VEC = 16 / sizeof(T);
  const bool vec_ok = aligned16(p) && aligned16(g) && aligned16(s0) && (R != Rule::kAdEMAMix || (aligned16(s1) && aligned16(s2)));
  const int64_t items = vec_ok ? n / VEC + n % VEC : n;
  int64_t blocks = (items + kOptimThreads - 1) / kOptimThreads;
  if (blocks > int64_t(device_sm_count()) * 8) blocks = int64_t(device_sm_count()) * 8;
  optim32bit_kernel<R, T><<<unsigned(blocks), kOptimThreads, 0, stream>>>(static_cast<T*>(p), static_cast<const T*>(g), s0, s1, s2, n,
                                                                          vec_ok, h, step_dev, gnorm_scale_dev);
  return check_launch(what);
}

template <Rule R>
static int dispatch_optim32(void* p, int dtype, const void* g, float* s0, float* s1, float* s2, int64_t n, const Optim32Hyper& h,
                            const float* step_dev, const float* gnorm_scale_dev, void* stream, const char* what) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (dtype) {
    case kF32: return launch_optim32<R, float>(p, g, s0, s1, s2, n, h, step_dev, gnorm_scale_dev, s, what);
    case kF16: return launch_optim32<R, __half>(p, g, s0, s1, s2, n, h, step_dev, gnorm_scale_dev, s, what);
    case kBF16: return launch_optim32<R, __nv_bfloat16>(p, g, s0, s1, s2, n, h, step_dev, gnorm_scale_dev, s, what);
  }
  return 0;   // unreachable: the entry points reject other dtypes first
}

static bool bad_dtype(int dtype) { return dtype != kF32 && dtype != kF16 && dtype != kBF16; }

static Optim32Hyper hyper(float lr, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float t_alpha,
                          float t_beta3) {
  return Optim32Hyper{lr, beta1, beta2, beta3, alpha, eps, weight_decay, weight_decay > 0.0f ? 1.0f - lr * weight_decay : 1.0f,
                      t_alpha, t_beta3};
}

}  // namespace qb200

using namespace qb200;

extern "C" int qb200_lion32bit_step_dev(void* p, int dtype, const void* g, float* m, int64_t n, float lr, float beta1, float beta2,
                                        float weight_decay, const float* step_dev, const float* gnorm_scale_dev, void* stream) {
  (void)step_dev;
  if (n < 0 || (n > 0 && (!p || !g || !m))) return set_error(QB200_EINVAL, "lion32bit_step_dev: null pointer or n < 0");
  if (bad_dtype(dtype)) return set_error(QB200_EINVAL, "lion32bit_step_dev: dtype must be 0 (fp32), 1 (fp16) or 2 (bf16)");
  if (n == 0) return 0;
  return dispatch_optim32<Rule::kLion>(p, dtype, g, m, nullptr, nullptr, n, hyper(lr, beta1, beta2, 0.0f, 0.0f, 0.0f, weight_decay, 0.0f, 0.0f),
                                       nullptr, gnorm_scale_dev, stream, "lion32bit_step_dev");
}

extern "C" int qb200_rmsprop32bit_step_dev(void* p, int dtype, const void* g, float* v, int64_t n, float lr, float alpha, float eps,
                                           float weight_decay, const float* step_dev, const float* gnorm_scale_dev, void* stream) {
  (void)step_dev;
  if (n < 0 || (n > 0 && (!p || !g || !v))) return set_error(QB200_EINVAL, "rmsprop32bit_step_dev: null pointer or n < 0");
  if (bad_dtype(dtype)) return set_error(QB200_EINVAL, "rmsprop32bit_step_dev: dtype must be 0 (fp32), 1 (fp16) or 2 (bf16)");
  if (n == 0) return 0;
  return dispatch_optim32<Rule::kRMSprop>(p, dtype, g, v, nullptr, nullptr, n,
                                          hyper(lr, 0.0f, 0.0f, 0.0f, alpha, eps, weight_decay, 0.0f, 0.0f), nullptr, gnorm_scale_dev,
                                          stream, "rmsprop32bit_step_dev");
}

extern "C" int qb200_ademamix32bit_step_dev(void* p, int dtype, const void* g, float* m1, float* m2, float* nu, int64_t n, float lr,
                                            float beta1, float beta2, float beta3, float alpha, float t_alpha, float t_beta3, float eps,
                                            float weight_decay, const float* step_dev, const float* gnorm_scale_dev, void* stream) {
  if (n < 0 || (n > 0 && (!p || !g || !m1 || !m2 || !nu || !step_dev)))
    return set_error(QB200_EINVAL, "ademamix32bit_step_dev: null pointer or n < 0");
  if (bad_dtype(dtype)) return set_error(QB200_EINVAL, "ademamix32bit_step_dev: dtype must be 0 (fp32), 1 (fp16) or 2 (bf16)");
  if (!(t_alpha >= 0.0f) || !(t_beta3 >= 0.0f))
    return set_error(QB200_EINVAL, "ademamix32bit_step_dev: t_alpha and t_beta3 must be positive (0 = no schedule)");
  if (n == 0) return 0;
  return dispatch_optim32<Rule::kAdEMAMix>(p, dtype, g, m1, m2, nu, n,
                                           hyper(lr, beta1, beta2, beta3, alpha, eps, weight_decay, t_alpha, t_beta3), step_dev,
                                           gnorm_scale_dev, stream, "ademamix32bit_step_dev");
}
