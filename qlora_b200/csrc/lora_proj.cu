// U[M, R] = scale * X[M, K] . A[R, K]^T for at most 16 tokens — the `lora_A` projection of an attached adapter during
// generation (peft: lora_A(dropout(x)); qlora.py:817-834 with an unmerged PeftModel).  cuBLAS serves this 1 x 4096 x 64
// product with a split-K GEMM + reduce (~10 us per projection in a decode chain, more than the NF4 GEMV it accompanies);
// here it is one 256-thread CTA per adapter row: the eight warps split the contraction in 256-element chunks (one 16-byte
// load per lane, two chunks in flight), every token's partial dot products stay in registers, warps meet in shared memory,
// one rounding to the operand type (bf16 or fp16).
// Programmatic dependent launch on both sides: the skinny kernel that consumes U prefetches its weights while this runs.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "nf4_table.cuh"
#include "qb200_internal.h"
#include "sm90_ptx.cuh"

namespace qb200 {

constexpr int kProjWarps = 8;

template <typename T16>
__device__ __forceinline__ float dot8(const uint4& a, const uint4& b) {
  using T2 = typename Vec2<T16>::type;
  const T2* a2 = reinterpret_cast<const T2*>(&a);
  const T2* b2 = reinterpret_cast<const T2*>(&b);
  float acc = 0.0f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 fa = widen2(a2[i]), fb = widen2(b2[i]);
    acc = fmaf(fa.x, fb.x, acc);
    acc = fmaf(fa.y, fb.y, acc);
  }
  return acc;
}

template <typename T16, int MT>   // operand type (bf16, fp16); token slots kept in registers (1, 4, 8, 16); M <= MT
__global__ void __launch_bounds__(32 * kProjWarps) lora_project_kernel(const T16* __restrict__ x, int64_t ld_x, const T16* __restrict__ a,
                                                                       float scale, T16* __restrict__ u, int64_t ld_u, int M, int K) {
  __shared__ float s_part[kProjWarps][MT];
  const int j = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();                       // x is the previous kernel's output; the adapter may have just been updated
  const T16* arow = a + int64_t(j) * K;
  float acc[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc[m] = 0.0f;
  constexpr int kStride = kProjWarps * 256;
  for (int k0 = (warp * 32 + lane) * 8; k0 < K; k0 += 2 * kStride) {
    const int k1 = k0 + kStride;
    const bool two = k1 < K;                   // both chunks' loads are issued before either is consumed
    const uint4 a0 = __ldg(reinterpret_cast<const uint4*>(arow + k0));
    const uint4 a1 = two ? __ldg(reinterpret_cast<const uint4*>(arow + k1)) : make_uint4(0, 0, 0, 0);
    uint4 x0[MT], x1[MT];
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      x0[m] = m < M ? *reinterpret_cast<const uint4*>(x + int64_t(m) * ld_x + k0) : make_uint4(0, 0, 0, 0);
      x1[m] = (m < M && two) ? *reinterpret_cast<const uint4*>(x + int64_t(m) * ld_x + k1) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int m = 0; m < MT; ++m) acc[m] += dot8<T16>(a0, x0[m]) + dot8<T16>(a1, x1[m]);
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], o);
    if (lane == 0) s_part[warp][m] = acc[m];
  }
  __syncthreads();
  if (threadIdx.x < M) {
    float v = 0.0f;
#pragma unroll
    for (int w = 0; w < kProjWarps; ++w) v += s_part[w][threadIdx.x];
    u[int64_t(threadIdx.x) * ld_u + j] = round16<T16>(v * scale);
  }
}

template <typename T16, int MT>
static int launch_project(const void* x, int64_t ld_x, const void* a, float scale, void* u, int64_t ld_u, int M, int K, int R,
                          cudaStream_t stream) {
  return launch_pdl(lora_project_kernel<T16, MT>, unsigned(R), 32 * kProjWarps, 0, stream, "lora_project", static_cast<const T16*>(x),
                    ld_x, static_cast<const T16*>(a), scale, static_cast<T16*>(u), ld_u, M, K);
}

template <typename T16>
static int launch_project_m(const void* x, int64_t ld_x, const void* a, float scale, void* u, int64_t ld_u, int M, int K, int R,
                            cudaStream_t s) {
  if (M == 1) return launch_project<T16, 1>(x, ld_x, a, scale, u, ld_u, M, K, R, s);
  if (M <= 4) return launch_project<T16, 4>(x, ld_x, a, scale, u, ld_u, M, K, R, s);
  if (M <= 8) return launch_project<T16, 8>(x, ld_x, a, scale, u, ld_u, M, K, R, s);
  return launch_project<T16, 16>(x, ld_x, a, scale, u, ld_u, M, K, R, s);
}

// lora_project_kernel with one adapter per token (MixedLora): CTA (j, y) computes column j of U for tokens [MT y, MT y + MT),
// each token against row j of its own A.  Per token the loads, the chunking and the fp32 sum order are lora_project_kernel's.
template <typename T16, int MT>   // token slots per CTA (1, 4, 8)
__global__ void __launch_bounds__(32 * kProjWarps) lora_project_mixed_kernel(const T16* __restrict__ x, int64_t ld_x, MixedLora mix,
                                                                             T16* __restrict__ u, int64_t ld_u, int M, int K) {
  __shared__ float s_part[kProjWarps][MT];
  const int j = blockIdx.x, m0 = blockIdx.y * MT, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cols = int(gridDim.x);
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();
  const T16* arow[MT];                          // row j of the token's A, or null: no adapter, or j beyond its rank
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    const qb200_lora_adapter* ad = m0 + m < M ? mix.adapter(m0 + m) : nullptr;
    arow[m] = ad != nullptr && j < MixedLora::rank(*ad, cols) ? static_cast<const T16*>(ad->A) + int64_t(j) * K : nullptr;
  }
  const T16* xm = x + int64_t(m0) * ld_x;
  float acc[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc[m] = 0.0f;
  constexpr int kStride = kProjWarps * 256;
  for (int k0 = (warp * 32 + lane) * 8; k0 < K; k0 += 2 * kStride) {
    const int k1 = k0 + kStride;
    const bool two = k1 < K;
    uint4 a0[MT], a1[MT], x0[MT], x1[MT];
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      const bool live = arow[m] != nullptr;
      a0[m] = live ? __ldg(reinterpret_cast<const uint4*>(arow[m] + k0)) : make_uint4(0, 0, 0, 0);
      a1[m] = (live && two) ? __ldg(reinterpret_cast<const uint4*>(arow[m] + k1)) : make_uint4(0, 0, 0, 0);
      x0[m] = live ? *reinterpret_cast<const uint4*>(xm + int64_t(m) * ld_x + k0) : make_uint4(0, 0, 0, 0);
      x1[m] = (live && two) ? *reinterpret_cast<const uint4*>(xm + int64_t(m) * ld_x + k1) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int m = 0; m < MT; ++m) acc[m] += dot8<T16>(a0[m], x0[m]) + dot8<T16>(a1[m], x1[m]);
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], o);
    if (lane == 0) s_part[warp][m] = acc[m];
  }
  __syncthreads();
  if (threadIdx.x < MT && m0 + int(threadIdx.x) < M) {
    const int m = m0 + threadIdx.x;
    const qb200_lora_adapter* ad = mix.adapter(m);
    T16 out = round16<T16>(0.0f);
    if (ad != nullptr && j < MixedLora::rank(*ad, cols)) {
      float v = 0.0f;
#pragma unroll
      for (int w = 0; w < kProjWarps; ++w) v += s_part[w][threadIdx.x];
      out = round16<T16>(v * ad->scale);
    }
    u[int64_t(m) * ld_u + j] = out;
  }
}

template <typename T16, int MT>
static int launch_project_mixed(const void* x, int64_t ld_x, const MixedLora& mix, void* u, int64_t ld_u, int M, int K, int R,
                                cudaStream_t stream) {
  const dim3 grid(unsigned(R), unsigned((M + MT - 1) / MT));
  return launch_pdl(lora_project_mixed_kernel<T16, MT>, grid, 32 * kProjWarps, 0, stream, "lora_project_mixed",
                    static_cast<const T16*>(x), ld_x, mix, static_cast<T16*>(u), ld_u, M, K);
}

template <typename T16>
static int launch_project_mixed_m(const void* x, int64_t ld_x, const MixedLora& mix, void* u, int64_t ld_u, int M, int K, int R,
                                  cudaStream_t s) {
  if (M == 1) return launch_project_mixed<T16, 1>(x, ld_x, mix, u, ld_u, M, K, R, s);
  if (M <= 4) return launch_project_mixed<T16, 4>(x, ld_x, mix, u, ld_u, M, K, R, s);
  return launch_project_mixed<T16, 8>(x, ld_x, mix, u, ld_u, M, K, R, s);
}

}  // namespace qb200

using namespace qb200;

extern "C" int qb200_lora_project_mixed(int dtype, const void* x, int64_t ld_x, const qb200_lora_adapter* table, int n_adapters,
                                        const int32_t* row_adapter, void* u, int64_t ld_u, int64_t M, int64_t K, int64_t R,
                                        void* stream) {
  if (dtype != QB200_DTYPE_BF16 && dtype != QB200_DTYPE_F16)
    return set_error(QB200_EINVAL, "lora_project_mixed: dtype must be 2 (bf16) or 1 (fp16)");
  if (!x || !table || !row_adapter || !u) return set_error(QB200_EINVAL, "lora_project_mixed: null pointer");
  if (n_adapters < 1) return set_error(QB200_EINVAL, "lora_project_mixed: n_adapters must be positive");
  if (M < 1 || M > int64_t(65535) * 8 || K < 8 || K % 8 != 0 || K > INT32_MAX)
    return set_error(QB200_EINVAL, "lora_project_mixed: bad shape");
  if (R < 8 || R > kMaxLoraRank || R % 8 != 0)
    return set_error(QB200_EUNSUPPORTED, "lora_project_mixed: R must be a multiple of 8 in [8, 256]");
  if (ld_x == 0) ld_x = K;
  if (ld_u == 0) ld_u = R;
  if (ld_x < K || ld_x % 8 != 0 || ld_u < R) return set_error(QB200_EINVAL, "lora_project_mixed: bad row pitch");
  if (reinterpret_cast<uintptr_t>(x) % 16 || reinterpret_cast<uintptr_t>(table) % 8 || reinterpret_cast<uintptr_t>(row_adapter) % 4)
    return set_error(QB200_EINVAL, "lora_project_mixed: x must be 16-byte, the table 8-byte and row_adapter 4-byte aligned");
  const MixedLora mix{row_adapter, table, n_adapters};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == QB200_DTYPE_F16) return launch_project_mixed_m<__half>(x, ld_x, mix, u, ld_u, int(M), int(K), int(R), s);
  return launch_project_mixed_m<__nv_bfloat16>(x, ld_x, mix, u, ld_u, int(M), int(K), int(R), s);
}

extern "C" int qb200_lora_project_typed(int dtype, const void* x, int64_t ld_x, const void* a, float scale, void* u, int64_t ld_u,
                                        int64_t M, int64_t K, int64_t R, void* stream) {
  if (dtype != QB200_DTYPE_BF16 && dtype != QB200_DTYPE_F16)
    return set_error(QB200_EINVAL, "lora_project_typed: dtype must be 2 (bf16) or 1 (fp16)");
  if (!x || !a || !u) return set_error(QB200_EINVAL, "lora_project: null pointer");
  if (M < 1 || M > 16) return set_error(QB200_EUNSUPPORTED, "lora_project: 1..16 tokens (larger batches are a library GEMM)");
  if (K < 8 || K % 8 != 0 || K > INT32_MAX || R < 1 || R > 65535) return set_error(QB200_EINVAL, "lora_project: bad shape");
  if (ld_x == 0) ld_x = K;
  if (ld_u == 0) ld_u = R;
  if (ld_x < K || ld_x % 8 != 0 || ld_u < R) return set_error(QB200_EINVAL, "lora_project: bad row pitch");
  if (reinterpret_cast<uintptr_t>(x) % 16 || reinterpret_cast<uintptr_t>(a) % 16)
    return set_error(QB200_EINVAL, "lora_project: x and A must be 16-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == QB200_DTYPE_F16) return launch_project_m<__half>(x, ld_x, a, scale, u, ld_u, int(M), int(K), int(R), s);
  return launch_project_m<__nv_bfloat16>(x, ld_x, a, scale, u, ld_u, int(M), int(K), int(R), s);
}

extern "C" int qb200_lora_project(const void* x, int64_t ld_x, const void* a, float scale, void* u, int64_t ld_u, int64_t M,
                                  int64_t K, int64_t R, void* stream) {
  return qb200_lora_project_typed(QB200_DTYPE_BF16, x, ld_x, a, scale, u, ld_u, M, K, R, stream);
}
