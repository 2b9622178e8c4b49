// Shared device helpers for the NF4 + double-quant kernels (sm_90a).
//
// Numeric contract (SURVEY.md Appendix A; bitsandbytes csrc/kernels.cu
// dQuantizeNF4 / dDequantizeNF4 / dQuantize<0> [upstream, un-vendored]):
// every fp32 operation is a single round-to-nearest IEEE op, spelled with
// __fmul_rn / __fadd_rn / __fdiv_rn so that neither -fmad nor fast-math flags
// can contract or approximate them.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace qb200 {

enum DType : int { kF32 = 0, kF16 = 1, kBF16 = 2 };

// A.1 — NF4 codebook, index = nibble (fp32-exact literals).
#define QB200_NF4_LUT_INIT                                                                             \
  {                                                                                                    \
    -1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f, -0.28444138169288635f,  \
        -0.18477343022823334f, -0.09105003625154495f, 0.0f, 0.07958029955625534f, 0.16093020141124725f, \
        0.24611230194568634f, 0.33791524171829224f, 0.44070982933044434f, 0.5626170039176941f,         \
        0.7229568362236023f, 1.0f                                                                      \
  }

// A.2 — dQuantizeNF4 as a 4-level bisection over the 15 ascending thresholds
// (strict '>', ties go to the lower code, NaN -> 0): the same function as the
// upstream nested-if tree.
__device__ __forceinline__ uint32_t nf4_code(float x) {
  // level 1
  const bool b3 = x > 0.03979014977812767f;
  // level 2
  const float t2 = b3 ? 0.3893125355243683f : -0.33967943489551544f;
  const bool b2 = x > t2;
  // level 3
  const float t1 = b3 ? (b2 ? 0.6427869200706482f : 0.2035212516784668f)
                      : (b2 ? -0.13791173323988914f : -0.6106329262256622f);
  const bool b1 = x > t1;
  // level 4
  const float t0 = b3 ? (b2 ? (b1 ? 0.8614784181118011f : 0.5016634166240692f)
                            : (b1 ? 0.2920137718319893f : 0.1202552504837513f))
                      : (b2 ? (b1 ? -0.045525018125772476f : -0.23460740596055984f)
                            : (b1 ? -0.4599952697753906f : -0.8480964004993439f));
  const bool b0 = x > t0;
  return (uint32_t(b3) << 3) | (uint32_t(b2) << 2) | (uint32_t(b1) << 1) | uint32_t(b0);
}

// Same function by table: the 15 thresholds are >= 0.080 apart, so each cell of width 1/16 of [-1, 1] holds at most one.
// cell(x) = low bits of fma(x, 16, 2^23 + 16) (round-to-nearest-even of 16 x + 16, monotone in x); the table gives, per
// cell, the number of thresholds in lower cells and the one threshold inside it (+inf if none):
//   code = base[cell] + (x > thr[cell]).
// ~7 instructions per value, most of them off the ALU pipe, against ~28 for the select tree (which bound K1: ncu ALU 84 %,
// 18-21 % of HBM peak).  Generated and checked against the tree on 2.1e7 values incl. +-5000 ulps around every threshold
// and cell edge (numpy float32: the add rounds exactly like the fma since 16 x is exact); the GPU tests compare the
// packed bytes bit-for-bit with the CPU restatement of the tree.
struct __align__(8) Nf4Cell {   // one 64-bit shared-memory load per look-up
  uint32_t thr_bits, base;
};
#define QB200_NF4_CELLS_INIT                                                                                              \
  {                                                                                                                       \
    {0x7f800000u, 0u}, {0x7f800000u, 0u}, {0xbf591cd9u, 0u}, {0x7f800000u, 1u}, {0x7f800000u, 1u}, {0x7f800000u, 1u},      \
        {0xbf1c5270u, 1u}, {0x7f800000u, 2u}, {0x7f800000u, 2u}, {0xbeeb8480u, 2u}, {0x7f800000u, 3u}, {0xbeadea76u, 3u},  \
        {0xbe703cecu, 4u}, {0x7f800000u, 5u}, {0xbe0d38bcu, 5u}, {0xbd3a7871u, 6u}, {0x7f800000u, 7u}, {0x3d22faffu, 7u},  \
        {0x3df64863u, 8u}, {0x3e5067e0u, 9u}, {0x7f800000u, 10u}, {0x3e9582d4u, 10u}, {0x3ec753f9u, 11u},                  \
        {0x7f800000u, 12u}, {0x3f006d03u, 12u}, {0x7f800000u, 13u}, {0x3f248dafu, 13u}, {0x7f800000u, 14u},                \
        {0x7f800000u, 14u}, {0x7f800000u, 14u}, {0x3f5c89d9u, 14u}, {0x7f800000u, 15u}, {0x7f800000u, 15u}                \
  }
constexpr int kNf4Cells = 33;

// `cells` is a shared-memory copy of the table.  NaN (0 * inf of an all-zero block) -> fmaxf gives -1 -> cell 0 -> code 0,
// like the tree; |x| <= 1 + 1 ulp by construction (x = v / absmax), the clamp keeps any other input inside the table.
__device__ __forceinline__ uint32_t nf4_code_cells(float x, const Nf4Cell* __restrict__ cells) {
  const float xc = fminf(fmaxf(x, -1.0f), 1.0f);
  const uint32_t cell = __float_as_uint(__fmaf_rn(xc, 16.0f, 8388624.0f)) - 0x4B000000u;   // 2^23 + 16; bits(2^23)
  const Nf4Cell c = cells[cell];
  return c.base + (xc > __uint_as_float(c.thr_bits) ? 1u : 0u);
}

// A.4 — dQuantize<0>(code, x): 7-step pivot search then neighbour rounding.
// `code` may live in shared or global memory.
__device__ __forceinline__ uint32_t code256_search(const float* __restrict__ code, float x) {
  int pivot = 127, upper_pivot = 255, lower_pivot = 0;
  float lower = -1.0f, upper = 1.0f, val = code[pivot];
#pragma unroll
  for (int step = 64; step > 0; step >>= 1) {
    if (x > val) {
      lower_pivot = pivot;
      lower = val;
      pivot += step;
    } else {
      upper_pivot = pivot;
      upper = val;
      pivot -= step;
    }
    val = code[pivot];
  }
  if (upper_pivot == 255) upper = code[upper_pivot];
  if (lower_pivot == 0) lower = code[lower_pivot];
  if (x > val) {
    const float mid = __fmul_rn(__fadd_rn(upper, val), 0.5f);
    return x > mid ? upper_pivot : pivot;
  } else {
    const float mid = __fmul_rn(__fadd_rn(lower, val), 0.5f);
    return x < mid ? lower_pivot : pivot;
  }
}

// A.5 line 1 — nested absmax: two separately rounded fp32 ops, never an FMA.
__device__ __forceinline__ float nested_absmax(float code_val, float absmax2, float offset) {
  return __fadd_rn(__fmul_rn(code_val, absmax2), offset);
}

// Packed-word element order.  A 32-bit little-endian word holds bytes b0..b3;
// byte j = (element 2j << 4) | element 2j+1  (even element in the HIGH nibble).
__device__ __forceinline__ uint32_t nf4_nibble(uint32_t word, int e /*0..7*/) {
  return (word >> (8 * (e >> 1) + ((e & 1) ? 0 : 4))) & 0xFu;
}

template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <>
__device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

}  // namespace qb200
