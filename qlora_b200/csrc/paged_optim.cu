// 32-bit AdamW with (optionally) unified-memory "paged" state — SURVEY.md 8f-3.
//
// Replaces (upstream bitsandbytes, un-vendored; reached from qlora.py:198 `optim='paged_adamw_32bit'` through HF's
// optimizer factory -> bitsandbytes.optim.AdamW(is_paged=True, optim_bits=32)):
//   cget_managed_ptr / cprefetch           (csrc/pythonInterface.c: cudaMallocManaged + cudaMemPrefetchAsync)
//   cadam32bit_grad_{fp32,fp16,bf16}       (kernel kOptimizer32bit2State<T, ADAM>)
// Update rule (restated from upstream's kernel; one fused elementwise pass, fp32 state, fp32 math):
//   g  = gnorm_scale * grad
//   m  = beta1*m + (1-beta1)*g ;  v = beta2*v + (1-beta2)*g*g
//   c1 = 1 - beta1^t ; c2 = sqrt(1 - beta2^t) ; step_size = -lr*c2/c1
//   p  = p + step_size * m / (sqrt(v) + eps*c2) ;  if (wd > 0) p = p * (1 - lr*wd)
// HBM-bound: per element 2 x (p, m, v) + 1 x g bytes.  Unlike every other entry point the managed allocator DOES
// allocate (as upstream's cget_managed_ptr does); ownership stays with the caller (qb200_managed_free).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include "nf4_common.cuh"
#include "qb200_internal.h"

namespace qb200 {

template <typename T>
__global__ void __launch_bounds__(256) adamw32bit_kernel(T* __restrict__ p, const T* __restrict__ g, float* __restrict__ m,
                                                         float* __restrict__ v, int64_t n, float beta1, float beta2, float eps_c2,
                                                         float step_size, float decay, float gnorm_scale) {
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float gi = __fmul_rn(gnorm_scale, to_f32<T>(g[i]));
    const float mi = __fadd_rn(__fmul_rn(m[i], beta1), __fmul_rn(1.0f - beta1, gi));
    const float vi = __fadd_rn(__fmul_rn(v[i], beta2), __fmul_rn(1.0f - beta2, __fmul_rn(gi, gi)));
    m[i] = mi;
    v[i] = vi;
    float pi = to_f32<T>(p[i]);
    pi = __fadd_rn(pi, __fmul_rn(step_size, __fdiv_rn(mi, __fadd_rn(__fsqrt_rn(vi), eps_c2))));
    if (decay != 1.0f) pi = __fmul_rn(pi, decay);
    p[i] = from_f32<T>(pi);
  }
}

// Same update with the step count (and optionally the gradient scale, e.g. a clip coefficient) read from DEVICE memory:
// nothing about the launch depends on host state, so it can be captured once in a CUDA graph and replayed every step
// (the host-scalar form bakes beta^t into the launch arguments).
template <typename T>
__global__ void __launch_bounds__(256) adamw32bit_dev_kernel(T* __restrict__ p, const T* __restrict__ g, float* __restrict__ m,
                                                             float* __restrict__ v, int64_t n, float lr, float beta1, float beta2,
                                                             float eps, float decay, const float* __restrict__ step_dev,
                                                             const float* __restrict__ gnorm_scale_dev) {
  const float t = __ldg(step_dev);
  const float c1 = 1.0f - powf(beta1, t);
  const float c2 = sqrtf(1.0f - powf(beta2, t));
  const float step_size = -lr * c2 / c1;
  const float eps_c2 = eps * c2;
  const float gnorm_scale = gnorm_scale_dev != nullptr ? __ldg(gnorm_scale_dev) : 1.0f;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float gi = __fmul_rn(gnorm_scale, to_f32<T>(g[i]));
    const float mi = __fadd_rn(__fmul_rn(m[i], beta1), __fmul_rn(1.0f - beta1, gi));
    const float vi = __fadd_rn(__fmul_rn(v[i], beta2), __fmul_rn(1.0f - beta2, __fmul_rn(gi, gi)));
    m[i] = mi;
    v[i] = vi;
    float pi = to_f32<T>(p[i]);
    pi = __fadd_rn(pi, __fmul_rn(step_size, __fdiv_rn(mi, __fadd_rn(__fsqrt_rn(vi), eps_c2))));
    if (decay != 1.0f) pi = __fmul_rn(pi, decay);
    p[i] = from_f32<T>(pi);
  }
}

template <typename T>
static int launch_adamw_dev(void* p, const void* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                            float weight_decay, const float* step_dev, const float* gnorm_scale_dev, cudaStream_t stream) {
  const float decay = weight_decay > 0.0f ? 1.0f - lr * weight_decay : 1.0f;
  int64_t blocks = (n + 255) / 256;
  if (blocks > int64_t(device_sm_count()) * 16) blocks = int64_t(device_sm_count()) * 16;
  adamw32bit_dev_kernel<T><<<unsigned(blocks), 256, 0, stream>>>(static_cast<T*>(p), static_cast<const T*>(g), m, v, n, lr, beta1, beta2,
                                                                eps, decay, step_dev, gnorm_scale_dev);
  return check_launch("adamw32bit_step_dev");
}

template <typename T>
static int launch_adamw(void* p, const void* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                        float weight_decay, int step, float gnorm_scale, cudaStream_t stream) {
  const float c1 = 1.0f - powf(beta1, float(step));
  const float c2 = sqrtf(1.0f - powf(beta2, float(step)));
  const float step_size = -lr * c2 / c1;
  const float decay = weight_decay > 0.0f ? 1.0f - lr * weight_decay : 1.0f;
  int64_t blocks = (n + 255) / 256;
  if (blocks > int64_t(device_sm_count()) * 16) blocks = int64_t(device_sm_count()) * 16;
  adamw32bit_kernel<T><<<unsigned(blocks), 256, 0, stream>>>(static_cast<T*>(p), static_cast<const T*>(g), m, v, n, beta1, beta2,
                                                            eps * c2, step_size, decay, gnorm_scale);
  return check_launch("adamw32bit_step");
}

}  // namespace qb200

using namespace qb200;

extern "C" int qb200_adamw32bit_step(void* p, int dtype, const void* g, float* m, float* v, int64_t n, float lr, float beta1,
                                     float beta2, float eps, float weight_decay, int step, float gnorm_scale, void* stream) {
  if (n < 0 || (n > 0 && (!p || !g || !m || !v))) return set_error(QB200_EINVAL, "adamw32bit_step: null pointer");
  if (step < 1) return set_error(QB200_EINVAL, "adamw32bit_step: step counts from 1");
  if (n == 0) return 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (dtype) {
    case kF32: return launch_adamw<float>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, step, gnorm_scale, s);
    case kF16: return launch_adamw<__half>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, step, gnorm_scale, s);
    case kBF16: return launch_adamw<__nv_bfloat16>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, step, gnorm_scale, s);
  }
  return set_error(QB200_EINVAL, "adamw32bit_step: dtype must be 0 (fp32), 1 (fp16) or 2 (bf16)");
}

extern "C" int qb200_adamw32bit_step_dev(void* p, int dtype, const void* g, float* m, float* v, int64_t n, float lr, float beta1,
                                         float beta2, float eps, float weight_decay, const float* step_dev,
                                         const float* gnorm_scale_dev, void* stream) {
  if (n < 0 || (n > 0 && (!p || !g || !m || !v || !step_dev))) return set_error(QB200_EINVAL, "adamw32bit_step_dev: null pointer");
  if (n == 0) return 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (dtype) {
    case kF32: return launch_adamw_dev<float>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, step_dev, gnorm_scale_dev, s);
    case kF16: return launch_adamw_dev<__half>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, step_dev, gnorm_scale_dev, s);
    case kBF16: return launch_adamw_dev<__nv_bfloat16>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, step_dev, gnorm_scale_dev, s);
  }
  return set_error(QB200_EINVAL, "adamw32bit_step_dev: dtype must be 0 (fp32), 1 (fp16) or 2 (bf16)");
}

extern "C" int qb200_managed_alloc(int64_t bytes, void** out) {
  if (!out || bytes <= 0) return set_error(QB200_EINVAL, "managed_alloc: bad arguments");
  const cudaError_t e = cudaMallocManaged(out, size_t(bytes), cudaMemAttachGlobal);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return set_error(int(e), "managed_alloc: cudaMallocManaged failed");
  }
  return 0;
}

extern "C" int qb200_managed_free(void* ptr) {
  if (!ptr) return 0;
  const cudaError_t e = cudaFree(ptr);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return set_error(int(e), "managed_free: cudaFree failed");
  }
  return 0;
}

extern "C" int qb200_prefetch(const void* ptr, int64_t bytes, int device, void* stream) {
  if (!ptr || bytes <= 0) return set_error(QB200_EINVAL, "prefetch: bad arguments");
  const cudaError_t e = cudaMemPrefetchAsync(ptr, size_t(bytes), device < 0 ? cudaCpuDeviceId : device, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return set_error(int(e), "prefetch: cudaMemPrefetchAsync failed");
  }
  return 0;
}
