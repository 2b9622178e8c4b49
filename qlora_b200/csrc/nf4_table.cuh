// Register-resident product table of one NF4 block: the 16 values  T16_rne(LUT[j] * absmax)  a block can take (with an fp16
// state under bf16 compute: bf16_rne(fp16_rne(LUT[j] * absmax))), kept as
// low-byte / high-byte planes so that PRMT byte permutes resolve 4 nibbles at a time (2 PRMT per weight, nothing else per
// weight: no shared-memory look-up, no multiply, no convert).  Shared by the fused GEMM (nf4_gemm_wgmma.cuh), the skinny
// forward (nf4_gemv.cu) and the standalone dequantize kernel (nf4_quant.cu): all three emit bit-identical weights.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "nf4_common.cuh"
#include "sm90_ptx.cuh"

namespace qb200 {

// The 16-bit operand type T16 of the fused kernels (__nv_bfloat16 or __half): its two-element vector, round-to-nearest-even
// from fp32 (one value, or two packed low | high) and the exact widening back to fp32.
template <typename T16>
struct Vec2 {
  using type = __nv_bfloat162;
};
template <>
struct Vec2<__half> {
  using type = __half2;
};
template <typename T16>
__device__ __forceinline__ T16 round16(float v) {
  if constexpr (std::is_same<T16, __half>::value) return __float2half_rn(v);
  else return __float2bfloat16_rn(v);
}
template <typename T16>
__device__ __forceinline__ uint32_t round16x2(float lo, float hi) {
  if constexpr (std::is_same<T16, __half>::value) return ptx::cvt_f16x2(lo, hi);
  else return ptx::cvt_bf16x2(lo, hi);
}
__device__ __forceinline__ float widen(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float widen(__half v) { return __half2float(v); }
__device__ __forceinline__ float2 widen2(__nv_bfloat162 v) { return __bfloat1622float2(v); }
__device__ __forceinline__ float2 widen2(__half2 v) { return __half22float2(v); }
// fp16 output of a bf16-compute launch (fp16 activations under bf16 compute): the bf16-rounded result rounded to fp16, which
// is what `.to(torch.float16)` does to it.
__device__ __forceinline__ __half bf16_to_f16(__nv_bfloat16 v) { return __float2half_rn(__bfloat162float(v)); }

struct Nf4Table {
  uint32_t tl[4], th[4];  // low / high byte planes of the 16 products
};

// kStateF16 (bf16 compute over an fp16 quant state): every product is first rounded to fp16 (subnormals kept, as
// cvt.rn.f16x2.f32 does) and widened, then rounded to T16 — the two roundings of `dequantize_4bit(W, fp16 state).to(bf16)`.
template <typename T16 = __nv_bfloat16, bool kStateF16 = false>
__device__ __forceinline__ void build_table(float am, Nf4Table& t) {
  constexpr float lut[16] = QB200_NF4_LUT_INIT;
  uint32_t p[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float lo = __fmul_rn(lut[2 * i], am), hi = __fmul_rn(lut[2 * i + 1], am);
    if constexpr (kStateF16) {
      const uint32_t h = ptx::cvt_f16x2(lo, hi);
      const float2 w = __half22float2(*reinterpret_cast<const __half2*>(&h));
      lo = w.x;
      hi = w.y;
    }
    p[i] = round16x2<T16>(lo, hi);
  }
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    t.tl[g] = ptx::prmt(p[2 * g], p[2 * g + 1], 0x6420);
    t.th[g] = ptx::prmt(p[2 * g], p[2 * g + 1], 0x7531);
  }
}

// 4 nibbles in sel[15:0] (positions 0..3) -> two 16-bit-pair words holding elements
// (pos1, pos0) and (pos3, pos2): the even element of a byte is its HIGH nibble.
__device__ __forceinline__ void lookup4(uint32_t sel, uint32_t sel_shr1, const Nf4Table& t, uint32_t& w01, uint32_t& w23) {
  const uint32_t sel_a = sel & 0x7777u;                          // index within an 8-entry half table
  const uint32_t sel_b = (sel_shr1 & 0x4444u) | 0x3210u;         // bit3 of each nibble -> pick half
  const uint32_t lo = ptx::prmt(ptx::prmt(t.tl[0], t.tl[1], sel_a), ptx::prmt(t.tl[2], t.tl[3], sel_a), sel_b);
  const uint32_t hi = ptx::prmt(ptx::prmt(t.th[0], t.th[1], sel_a), ptx::prmt(t.th[2], t.th[3], sel_a), sel_b);
  w01 = ptx::prmt(lo, hi, 0x4051);
  w23 = ptx::prmt(lo, hi, 0x6273);
}

// one packed word (8 nibbles) -> 8 values in element (memory) order
__device__ __forceinline__ uint4 dequant_word(uint32_t w, const Nf4Table& t) {
  uint4 o;
  lookup4(w, w >> 1, t, o.x, o.y);
  lookup4(w >> 16, w >> 17, t, o.z, o.w);
  return o;
}

}  // namespace qb200
