// NF4 / 8-bit blockwise quantize + dequantize kernels for sm_90a (K1-K4 of SURVEY.md 2.4).
//
// These are HBM-bound streaming kernels: 128-bit coalesced loads/stores, one 32-bit
// packed word (8 NF4 codes) per thread, no shared-memory staging needed (no reuse).
// Roofline: bytes moved / measured HBM copy bandwidth (MEASURED_PEAKS.json).
//   quantize  bf16: 2 B in + 0.5 B + 4/64 B out per element
//   dequantize bf16: 0.5 B + 1/64 B (+4/16384 B) in, 2 B out per element
//
// Reference being replaced (un-vendored upstream bitsandbytes, SURVEY.md 2.4):
//   K1 kQuantizeBlockwise<T,64,2,0,NF4>      32-thread CTAs, 2 elems/thread
//   K2 kQuantizeBlockwise<float,256,2,0,General8bit>
//   K3 kDequantizeBlockwise<float,512,64,8,General8bit>
//   K4 kDequantizeBlockwise<T,512,64,8,NF4>  64-thread CTAs, 8 B/thread
#include <stdlib.h>

#include <type_traits>

#include "nf4_common.cuh"
#include "nf4_table.cuh"
#include "qb200_internal.h"

namespace qb200 {

__device__ __constant__ float c_nf4_lut[16] = QB200_NF4_LUT_INIT;

// ------------------------------------------------------------------ K1 ----------------
// One thread = 8 consecutive elements = one packed 32-bit word.  G = BS/8 threads share
// a quant block; absmax by xor-shuffles (G <= 32) or a shared-memory pass (G > 32, one
// CTA per quant block).
template <typename T>
__device__ __forceinline__ void load8(const T* __restrict__ A, int64_t i0, int64_t n, bool vec_ok, float (&v)[8]);

template <>
__device__ __forceinline__ void load8<float>(const float* __restrict__ A, int64_t i0, int64_t n, bool vec_ok,
                                             float (&v)[8]) {
  if (vec_ok && i0 + 8 <= n) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(A + i0));
    const float4 b = __ldg(reinterpret_cast<const float4*>(A + i0 + 4));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (i0 + j < n) ? A[i0 + j] : 0.0f;
  }
}

template <typename T16>
__device__ __forceinline__ void load8_16(const T16* __restrict__ A, int64_t i0, int64_t n, bool vec_ok, float (&v)[8]) {
  if (vec_ok && i0 + 8 <= n) {
    const uint4 raw = __ldg(reinterpret_cast<const uint4*>(A + i0));
    const T16* h = reinterpret_cast<const T16*>(&raw);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = to_f32<T16>(h[j]);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (i0 + j < n) ? to_f32<T16>(A[i0 + j]) : 0.0f;
  }
}
template <>
__device__ __forceinline__ void load8<__half>(const __half* __restrict__ A, int64_t i0, int64_t n, bool vec_ok,
                                              float (&v)[8]) {
  load8_16<__half>(A, i0, n, vec_ok, v);
}
template <>
__device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* __restrict__ A, int64_t i0, int64_t n,
                                                     bool vec_ok, float (&v)[8]) {
  load8_16<__nv_bfloat16>(A, i0, n, vec_ok, v);
}

__device__ const Nf4Cell g_nf4_cells[kNf4Cells] = QB200_NF4_CELLS_INIT;

// Reciprocal-and-scale of the quantizers (K1, K2) in the two arithmetic modes of SURVEY.md A.5(i):
//   ieee   (default): inv = 1.0f / absmax correctly rounded, x = v * inv correctly rounded — what the CPU oracle computes;
//   approx          : inv = rcp.approx.ftz.f32(absmax), x = mul.ftz.f32(v, inv) — what `1.0f / absmax` and `v * inv` compile
//                     to under nvcc --use_fast_math, the flag upstream bitsandbytes builds its kernels with.  rcp.approx is
//                     within 1 ulp of the IEEE reciprocal, so the two modes can differ only for values within ~1 ulp of one
//                     of the 15 decision thresholds (measured: a few nibbles per 10^7 on N(0, 0.02) weights).
// Only the mode a real bitsandbytes binary was built with reproduces its packed bytes bit for bit; with no such binary
// available here, `ieee` is the default because it is the mode the oracle can restate exactly.
template <bool kApprox>
__device__ __forceinline__ float quant_recip(float absmax) {
  if (kApprox) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(absmax));
    return r;
  }
  return __fdiv_rn(1.0f, absmax);
}
template <bool kApprox>
__device__ __forceinline__ float quant_scale(float v, float inv) {
  if (kApprox) {
    float r;
    asm("mul.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(v), "f"(inv));
    return r;
  }
  return __fmul_rn(v, inv);
}

// every thread of the CTA calls this before quantize_store8 (blockDim.x >= 64)
__device__ __forceinline__ void stage_cells(Nf4Cell* s_cells) {
  if (threadIdx.x < kNf4Cells) s_cells[threadIdx.x] = g_nf4_cells[threadIdx.x];
  __syncthreads();
}

// Shared-memory address of the cell table, pre-biased so that the raw bits of fma(x, 16, 2^23 + 16) index it directly:
//   &cells[bits - 0x4B000000] = base + 8 * bits - 8 * 0x4B000000   (mod 2^32).
// The bias arrives as a kernel parameter (kCellBias) so that ptxas keeps base - bias in ONE register and the address is one
// LEA per value; with a literal it re-splits the sum into LEA + VIADD.
constexpr uint32_t kCellBias = 0x58000000u;   // 8 * 0x4B000000 mod 2^32
__device__ __forceinline__ uint32_t cells_biased_addr(const Nf4Cell* s_cells, uint32_t cell_bias) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(s_cells)) - cell_bias;
}

template <bool kApprox>
__device__ __forceinline__ void quantize_store8(const float (&v)[8], float absmax, int64_t i0, int64_t n,
                                                uint8_t* __restrict__ packed, uint32_t cells_biased) {
  // reciprocal then multiply (A.3): absmax==0 -> inv=+inf -> 0*inf=NaN -> code 0 (both modes).
  const float inv = quant_recip<kApprox>(absmax);
  // nf4_code_cells() per value with the table address folded into one shift-add, and the packed word
  //   sum_j ((code[2j] << 4) | code[2j+1]) << 8j
  // accumulated Horner-style from the top nibble down: one integer multiply-add + one predicated increment per value
  // instead of select / shift / or (K1 is issue-bound: every instruction per value counts)
  constexpr int order[8] = {6, 7, 4, 5, 2, 3, 0, 1};
  uint32_t word = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float xc = fminf(fmaxf(quant_scale<kApprox>(v[order[j]], inv), -1.0f), 1.0f);
    const uint32_t bits = __float_as_uint(__fmaf_rn(xc, 16.0f, 8388624.0f));
    uint32_t thr, base;
    asm("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(thr), "=r"(base) : "r"(cells_biased + (bits << 3)));
    asm("{\n\t.reg .pred p;\n\tsetp.gt.f32 p, %1, %2;\n\tmad.lo.u32 %0, %0, 16, %3;\n\t@p add.u32 %0, %0, 1;\n\t}"
        : "+r"(word)
        : "f"(xc), "f"(__uint_as_float(thr)), "r"(base));   // word = word * 16 + base + (xc > thr)
  }
  if (i0 + 8 <= n) {
    *reinterpret_cast<uint32_t*>(packed + (i0 >> 1)) = word;
  } else if (i0 < n) {
    const int nbytes = int((n - i0 + 1) >> 1);
    for (int j = 0; j < nbytes; ++j) packed[(i0 >> 1) + j] = uint8_t(word >> (8 * j));
  }
}

template <typename T, int G, bool kApprox>  // G = threads per quant block, 8/16/32
__global__ void __launch_bounds__(256) quantize_nf4_shfl_kernel(const T* __restrict__ A, int64_t n, bool vec_ok,
                                                                uint8_t* __restrict__ packed,
                                                                float* __restrict__ absmax, uint32_t cell_bias) {
  __shared__ Nf4Cell s_cells[kNf4Cells];
  const int64_t tid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t i0 = tid * 8;
  float v[8];
  load8<T>(A, i0, n, vec_ok, v);
  stage_cells(s_cells);
  float m = 0.0f;
#pragma unroll
  for (int j = 0; j < 8; ++j) m = fmaxf(m, fabsf(v[j]));
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x % G) == 0 && i0 < n) absmax[tid / G] = m;
  quantize_store8<kApprox>(v, m, i0, n, packed, cells_biased_addr(s_cells, cell_bias));
}

template <typename T, bool kApprox>  // one CTA (= BS/8 threads, 64..512) per quant block
__global__ void quantize_nf4_cta_kernel(const T* __restrict__ A, int64_t n, bool vec_ok, uint8_t* __restrict__ packed,
                                        float* __restrict__ absmax, uint32_t cell_bias) {
  __shared__ float s_max[16];
  __shared__ float s_all;
  __shared__ Nf4Cell s_cells[kNf4Cells];
  const int64_t i0 = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  float v[8];
  load8<T>(A, i0, n, vec_ok, v);
  stage_cells(s_cells);
  float m = 0.0f;
#pragma unroll
  for (int j = 0; j < 8; ++j) m = fmaxf(m, fabsf(v[j]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float mm = 0.0f;
    for (int w = 0; w < int(blockDim.x >> 5); ++w) mm = fmaxf(mm, s_max[w]);
    s_all = mm;
    absmax[blockIdx.x] = mm;
  }
  __syncthreads();
  quantize_store8<kApprox>(v, s_all, i0, n, packed, cells_biased_addr(s_cells, cell_bias));
}

// process-wide arithmetic mode of K1/K2 (0 = ieee, 1 = approx); QB200_QUANT_MATH=approx or qb200_set_quant_math(1)
static int g_quant_math = -1;
static int quant_math() {
  if (g_quant_math < 0) {
    const char* e = getenv("QB200_QUANT_MATH");
    g_quant_math = (e && (e[0] == 'a' || e[0] == 'A' || e[0] == '1')) ? 1 : 0;
  }
  return g_quant_math;
}

template <typename T, bool kApprox>
static int launch_quantize_nf4_mode(const T* A, int64_t n, int blocksize, uint8_t* packed, float* absmax, cudaStream_t stream);

template <typename T>
static int launch_quantize_nf4(const T* A, int64_t n, int blocksize, uint8_t* packed, float* absmax, cudaStream_t stream) {
  return quant_math() ? launch_quantize_nf4_mode<T, true>(A, n, blocksize, packed, absmax, stream)
                      : launch_quantize_nf4_mode<T, false>(A, n, blocksize, packed, absmax, stream);
}

template <typename T, bool kApprox>
static int launch_quantize_nf4_mode(const T* A, int64_t n, int blocksize, uint8_t* packed, float* absmax,
                                    cudaStream_t stream) {
  if (n == 0) return 0;
  const bool vec_ok = (reinterpret_cast<uintptr_t>(A) % 16 == 0) && (reinterpret_cast<uintptr_t>(packed) % 4 == 0);
  if (reinterpret_cast<uintptr_t>(packed) % 4 != 0) return set_error(QB200_EINVAL, "packed output must be 4-byte aligned");
  const int64_t nthreads = (n + 7) / 8;
  if (blocksize <= 256) {
    const int threads = 256;
    const int64_t blocks = (nthreads + threads - 1) / threads;
    switch (blocksize) {
      case 64: quantize_nf4_shfl_kernel<T, 8, kApprox><<<(unsigned)blocks, threads, 0, stream>>>(A, n, vec_ok, packed, absmax, kCellBias); break;
      case 128: quantize_nf4_shfl_kernel<T, 16, kApprox><<<(unsigned)blocks, threads, 0, stream>>>(A, n, vec_ok, packed, absmax, kCellBias); break;
      case 256: quantize_nf4_shfl_kernel<T, 32, kApprox><<<(unsigned)blocks, threads, 0, stream>>>(A, n, vec_ok, packed, absmax, kCellBias); break;
      default: return set_error(QB200_EINVAL, "blocksize must be a power of two in [64, 4096]");
    }
  } else {
    const int64_t nblocks = (n + blocksize - 1) / blocksize;
    quantize_nf4_cta_kernel<T, kApprox><<<(unsigned)nblocks, blocksize / 8, 0, stream>>>(A, n, vec_ok, packed, absmax, kCellBias);
  }
  return check_launch("quantize_nf4");
}

// ------------------------------------------------------------------ K2 ----------------
// One warp per quant block (any blocksize, ragged tail ok): coalesced fp32 loads, absmax
// by warp shuffle, then the 7-step search in a shared copy of the 256-entry codebook.
template <bool kApprox>
__global__ void __launch_bounds__(256) quantize_8bit_kernel(const float* __restrict__ code, const float* __restrict__ A,
                                                            int64_t n, int blocksize, uint8_t* __restrict__ out,
                                                            float* __restrict__ absmax) {
  __shared__ float s_code[256];
  s_code[threadIdx.x] = code[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t nblocks = (n + blocksize - 1) / blocksize;
  const int64_t warps_total = int64_t(gridDim.x) * (blockDim.x >> 5);
  for (int64_t b = int64_t(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); b < nblocks; b += warps_total) {
    const int64_t lo = b * blocksize;
    const int64_t hi = (lo + blocksize < n) ? lo + blocksize : n;
    float m = 0.0f;
    for (int64_t i = lo + lane; i < hi; i += 32) m = fmaxf(m, fabsf(A[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) absmax[b] = m;
    const float inv = quant_recip<kApprox>(m);
    for (int64_t i = lo + lane; i < hi; i += 32) out[i] = uint8_t(code256_search(s_code, quant_scale<kApprox>(A[i], inv)));
  }
}

// ------------------------------------------------------------------ K3 ----------------
__global__ void __launch_bounds__(256) dequantize_8bit_kernel(const float* __restrict__ code,
                                                              const uint8_t* __restrict__ A,
                                                              const float* __restrict__ absmax, int64_t n, int blocksize,
                                                              float* __restrict__ out) {
  __shared__ float s_code[256];
  s_code[threadIdx.x] = code[threadIdx.x];
  __syncthreads();
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const bool pow2 = (blocksize & (blocksize - 1)) == 0;
  const int shift = 31 - __clz(blocksize);
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = __fmul_rn(s_code[A[i]], __ldg(absmax + (pow2 ? (i >> shift) : (i / blocksize))));
}

// ------------------------------------------------------------------ K4 ----------------
// One thread = one 32-bit packed word = 8 outputs (one 16 B store for 16-bit outputs).
// NESTED: absmax recomputed in registers from (u8 code, codebook, absmax2, offset).
template <typename T>
__device__ __forceinline__ void store8(T* __restrict__ out, int64_t i0, int64_t n, bool vec_ok, const float (&w)[8]);

template <>
__device__ __forceinline__ void store8<float>(float* __restrict__ out, int64_t i0, int64_t n, bool vec_ok,
                                              const float (&w)[8]) {
  if (vec_ok && i0 + 8 <= n) {
    *reinterpret_cast<float4*>(out + i0) = make_float4(w[0], w[1], w[2], w[3]);
    *reinterpret_cast<float4*>(out + i0 + 4) = make_float4(w[4], w[5], w[6], w[7]);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (i0 + j < n) out[i0 + j] = w[j];
  }
}
template <typename T16>
__device__ __forceinline__ void store8_16(T16* __restrict__ out, int64_t i0, int64_t n, bool vec_ok,
                                          const float (&w)[8]) {
  if (vec_ok && i0 + 8 <= n) {
    uint4 raw;
    T16* h = reinterpret_cast<T16*>(&raw);
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = from_f32<T16>(w[j]);
    *reinterpret_cast<uint4*>(out + i0) = raw;
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (i0 + j < n) out[i0 + j] = from_f32<T16>(w[j]);
  }
}
template <>
__device__ __forceinline__ void store8<__half>(__half* __restrict__ out, int64_t i0, int64_t n, bool vec_ok,
                                               const float (&w)[8]) {
  store8_16<__half>(out, i0, n, vec_ok, w);
}
template <>
__device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* __restrict__ out, int64_t i0, int64_t n,
                                                      bool vec_ok, const float (&w)[8]) {
  store8_16<__nv_bfloat16>(out, i0, n, vec_ok, w);
}

// kUnroll independent packed words per thread per iteration (all loads issued before any use) so that
// enough bytes are in flight per SM to cover HBM latency; consecutive lanes own consecutive words, so every
// load is a coalesced 128 B and every store a coalesced 512 B (bf16) per warp instruction.
constexpr int kDeqUnroll = 4;

template <typename T, bool NESTED>
__global__ void __launch_bounds__(256) dequantize_nf4_kernel(const uint8_t* __restrict__ packed,
                                                             const float* __restrict__ absmax,      // !NESTED
                                                             const uint8_t* __restrict__ absmax_u8,  // NESTED
                                                             const float* __restrict__ code256,
                                                             const float* __restrict__ absmax2,
                                                             const float* __restrict__ offset_ptr, int64_t n,
                                                             int blocksize, int blocksize2, bool vec_ok,
                                                             T* __restrict__ out) {
  __shared__ float s_lut[16];
  __shared__ float s_code[256];
  if (threadIdx.x < 16) s_lut[threadIdx.x] = c_nf4_lut[threadIdx.x];
  float offset = 0.0f;
  if (NESTED) {
    s_code[threadIdx.x] = code256[threadIdx.x];
    offset = __ldg(offset_ptr);
  }
  __syncthreads();
  const int64_t nwords = (n + 7) / 8;
  const int64_t nbytes = (n + 1) / 2;
  const int bs_shift = 31 - __clz(blocksize);      // blocksize is a power of two
  const bool bs2_pow2 = (blocksize2 & (blocksize2 - 1)) == 0;
  const int bs2_shift = 31 - __clz(blocksize2);    // 64-bit integer division is ~100 instructions: shift when possible
  const int64_t tile = int64_t(blockDim.x) * kDeqUnroll;
  for (int64_t base = int64_t(blockIdx.x) * tile + threadIdx.x; base < nwords; base += int64_t(gridDim.x) * tile) {
    uint32_t word[kDeqUnroll];
    uint32_t code[kDeqUnroll];
    float scale[kDeqUnroll];
#pragma unroll
    for (int u = 0; u < kDeqUnroll; ++u) {
      const int64_t w = base + int64_t(u) * blockDim.x;
      word[u] = 0;
      code[u] = 0;
      scale[u] = 0.0f;
      if (w < nwords) {
        if (vec_ok && (w + 1) * 4 <= nbytes) {
          word[u] = __ldg(reinterpret_cast<const uint32_t*>(packed) + w);
        } else {
          for (int j = 0; j < 4; ++j)
            if (w * 4 + j < nbytes) word[u] |= uint32_t(packed[w * 4 + j]) << (8 * j);
        }
        const int64_t b = (w * 8) >> bs_shift;
        if (NESTED) {
          code[u] = __ldg(absmax_u8 + b);
          scale[u] = __ldg(absmax2 + (bs2_pow2 ? (b >> bs2_shift) : (b / blocksize2)));
        } else {
          scale[u] = __ldg(absmax + b);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kDeqUnroll; ++u) {
      const int64_t w = base + int64_t(u) * blockDim.x;
      if (w >= nwords) continue;
      const float am = NESTED ? nested_absmax(s_code[code[u]], scale[u], offset) : scale[u];
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = __fmul_rn(s_lut[nf4_nibble(word[u], e)], am);
      store8<T>(out, w * 8, n, vec_ok, v);
    }
  }
}

// Fast path for the shapes that matter (16-bit output, n % 8 == 0, n < 2^31, aligned pointers, power-of-two block
// sizes): 32-bit indices, no per-element guards, the nibble is turned into a byte offset into the shared LUT with one
// shift + one mask (LUT index pre-scaled by 4), two products per cvt.rn.bf16x2 / cvt.rn.f16x2.
template <typename T16, bool NESTED>
__global__ void __launch_bounds__(256) dequantize_nf4_fast_kernel(const uint32_t* __restrict__ packed,
                                                                  const float* __restrict__ absmax,
                                                                  const uint8_t* __restrict__ absmax_u8,
                                                                  const float* __restrict__ code256,
                                                                  const float* __restrict__ absmax2,
                                                                  const float* __restrict__ offset_ptr, uint32_t nwords,
                                                                  int bs_shift /* log2(blocksize/8) */, int bs2_shift,
                                                                  uint4* __restrict__ out) {
  __shared__ float s_lut[16];
  __shared__ float s_code[256];
  if (threadIdx.x < 16) s_lut[threadIdx.x] = c_nf4_lut[threadIdx.x];
  float offset = 0.0f;
  if (NESTED) {
    s_code[threadIdx.x] = code256[threadIdx.x];
    offset = __ldg(offset_ptr);
  }
  __syncthreads();
  const uint32_t lut_base = static_cast<uint32_t>(__cvta_generic_to_shared(s_lut));
  const uint32_t tile = blockDim.x * kDeqUnroll;
  for (uint32_t base = blockIdx.x * tile + threadIdx.x; base < nwords; base += gridDim.x * tile) {
    uint32_t word[kDeqUnroll];
    uint32_t code[kDeqUnroll];
    float scale[kDeqUnroll];
#pragma unroll
    for (int u = 0; u < kDeqUnroll; ++u) {
      const uint32_t w = base + u * blockDim.x;
      word[u] = 0;
      code[u] = 0;
      scale[u] = 0.0f;
      if (w < nwords) {
        word[u] = __ldg(packed + w);
        const uint32_t b = w >> bs_shift;
        if (NESTED) {
          code[u] = __ldg(absmax_u8 + b);
          scale[u] = __ldg(absmax2 + (b >> bs2_shift));
        } else {
          scale[u] = __ldg(absmax + b);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kDeqUnroll; ++u) {
      const uint32_t w = base + u * blockDim.x;
      if (w >= nwords) continue;
      const float am = NESTED ? nested_absmax(s_code[code[u]], scale[u], offset) : scale[u];
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {   // byte j = (elem 2j << 4) | elem 2j+1
        const uint32_t hi_off = (word[u] >> (8 * j + 2)) & 0x3Cu;                       // (byte >> 4) * 4
        const uint32_t lo_off = (j == 0 ? (word[u] << 2) : (word[u] >> (8 * j - 2))) & 0x3Cu;   // (byte & 15) * 4
        float lo_v, hi_v;
        asm("ld.shared.f32 %0, [%1];" : "=f"(hi_v) : "r"(lut_base + hi_off));
        asm("ld.shared.f32 %0, [%1];" : "=f"(lo_v) : "r"(lut_base + lo_off));
        const float e0 = __fmul_rn(hi_v, am), e1 = __fmul_rn(lo_v, am);
        if constexpr (sizeof(T16) == 2 && std::is_same<T16, __nv_bfloat16>::value) {
          asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o[j]) : "f"(e1), "f"(e0));
        } else {
          asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(o[j]) : "f"(e1), "f"(e0));
        }
      }
      out[w] = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// Main path (16-bit output, n % 32 == 0, 32-byte aligned output, power-of-two block sizes): a 16-byte vector of packed
// nibbles = 32 values of ONE quant block = 64 B of output; a warp expands kTabVecs runs of 32 consecutive vectors per
// iteration, one vector per lane per run.
//   * the block's 16 possible outputs  T16_rne(LUT[j] * absmax)  are built once per vector as a register product table
//     (nf4_table.cuh: 32 instructions per 32 values) and every nibble is resolved with PRMT byte permutes — 2 per value,
//     no shared-memory look-up, multiply or convert per value (the LUT-in-shared-memory kernel above issues 9.4
//     instructions per value and stalls on the shared-memory queue: ncu issue-active 61-68 %, mio_throttle 3.3);
//   * loads are 512 contiguous bytes per warp instruction.  A run's 2 KB of output goes through a per-warp shared-memory
//     stage, so each of its four 16-byte warp stores writes 512 contiguous bytes (4 whole lines).  Storing each lane's
//     64 B straight from registers writes 16 B at a 64 B stride per instruction (16 lines, every sector half-written) and
//     ran at 1.25-1.39 TB/s against 2.16-2.50 TB/s for the same loads with a contiguous store mapping
//     (tools/stream_perf.py, H100 80GB HBM3 at 700 W; this kernel: 2.44-2.66 TB/s).  The stage slot of a lane's k-th 16 B is rotated by lane / 2, which keeps both the
//     writes (64 B per lane) and the reads (16 B per lane) free of bank conflicts;
//   * kTabVecs runs in flight per thread, the next iteration's vectors + absmax statistics prefetched before the current
//     ones are expanded; the grid is capped at kTabCtasPerSm CTAs per SM (about two waves at the registers this kernel
//     takes) and a grid-stride loop takes the rest.  Two runs per thread and the two-wave grid measured 5-10 % above one
//     run and a persistent one-wave grid; a second vector in flight without the stage did not help (1.1-1.2 TB/s).
// kPdl: the bf16 weight copy of the scratch GEMM path (launch_dequant_scratch), launched with programmatic stream
// serialization: it lets the GEMM queued behind it start its prologue at once and issues its first loads (the frozen
// quant state) before it waits for the previous kernel, whose reads of a recycled scratch buffer must end before any store.
constexpr int kTabWarps = 8;        // warps per CTA: 256 threads, one s_code entry each
constexpr int kTabVecs = 2;         // runs of 32 vectors per warp and iteration
constexpr int kTabCtasPerSm = 8;
template <typename T16, bool NESTED, bool kPdl = false>
__global__ void __launch_bounds__(32 * kTabWarps) dequantize_nf4_tab_kernel(const uint4* __restrict__ packed,
                                                                            const float* __restrict__ absmax,
                                                                            const uint8_t* __restrict__ absmax_u8,
                                                                            const float* __restrict__ code256,
                                                                            const float* __restrict__ absmax2,
                                                                            const float* __restrict__ offset_ptr, uint32_t nvec,
                                                                            int bs_shift /* log2(blocksize / 32) */, int bs2_shift,
                                                                            uint8_t* __restrict__ out) {
  __shared__ float s_code[256];
  __shared__ uint4 s_stage[kTabWarps][128];   // one run's output per warp: 32 vectors x 4 16-byte chunks
  float offset = 0.0f;
  if (NESTED) {
    s_code[threadIdx.x] = code256[threadIdx.x];
    offset = __ldg(offset_ptr);
    __syncthreads();
  }
  if constexpr (kPdl) ptx::grid_dep_launch();
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr uint32_t kSpan = 32 * kTabVecs;   // vectors per warp and iteration
  const uint32_t stride = gridDim.x * kTabWarps * kSpan;
  uint32_t base = (blockIdx.x * kTabWarps + warp) * kSpan;
  uint4 w_next[kTabVecs];
  uint32_t code_next[kTabVecs];
  float scale_next[kTabVecs];
  auto fetch = [&](uint32_t b0) {
#pragma unroll
    for (int u = 0; u < kTabVecs; ++u) {
      uint32_t v = b0 + u * 32 + lane;
      v = v < nvec ? v : nvec - 1;                       // clamped: the prefetch past the end re-reads the last vector
      w_next[u] = __ldg(packed + v);
      const uint32_t b = v >> bs_shift;
      code_next[u] = 0;
      if (NESTED) {
        code_next[u] = __ldg(absmax_u8 + b);
        scale_next[u] = __ldg(absmax2 + (b >> bs2_shift));
      } else {
        scale_next[u] = __ldg(absmax + b);
      }
    }
  };
  fetch(base);
  if constexpr (kPdl) ptx::grid_dep_wait();           // no global store before this point
  uint4* out16 = reinterpret_cast<uint4*>(out);
  for (; base < nvec; base += stride) {               // warp-uniform: the __syncwarp()s below see the whole warp
    uint4 w[kTabVecs];
    float am[kTabVecs];
#pragma unroll
    for (int u = 0; u < kTabVecs; ++u) {
      w[u] = w_next[u];
      am[u] = NESTED ? nested_absmax(s_code[code_next[u]], scale_next[u], offset) : scale_next[u];
    }
    fetch(base + stride);
#pragma unroll
    for (int u = 0; u < kTabVecs; ++u) {
      const uint32_t v0 = base + u * 32;              // first vector of the run
      Nf4Table tab;
      build_table<T16>(am[u], tab);
      const uint4 o[4] = {dequant_word(w[u].x, tab), dequant_word(w[u].y, tab), dequant_word(w[u].z, tab),
                          dequant_word(w[u].w, tab)};
#pragma unroll
      for (int k = 0; k < 4; ++k) s_stage[warp][4 * lane + ((k + (lane >> 1)) & 3)] = o[k];
      __syncwarp();
#pragma unroll
      for (int j = 0; j < 4; ++j) {                   // chunk c of the run = 16-byte piece c % 4 of vector v0 + c / 4
        const uint32_t c = 32 * j + lane, src = c >> 2;
        const uint4 val = s_stage[warp][4 * src + (((c & 3) + (src >> 1)) & 3)];
        if (v0 + src < nvec) out16[uint64_t(v0) * 4 + c] = val;
      }
      __syncwarp();                                   // the stage is rewritten by the next run
    }
  }
}

// CTAs of dequantize_nf4_tab_kernel for nvec vectors: kTabVecs runs of 32 vectors per warp, at most kTabCtasPerSm CTAs
// per SM (the grid-stride loop takes the rest)
static unsigned tab_grid(uint32_t nvec) {
  const int64_t per_cta = int64_t(kTabWarps) * 32 * kTabVecs;
  const int64_t tb = (int64_t(nvec) + per_cta - 1) / per_cta, tb_max = int64_t(device_sm_count()) * kTabCtasPerSm;
  return unsigned(tb < tb_max ? tb : tb_max);
}

// QB200_DEQUANT_LUT=1 keeps the shared-memory-LUT kernels for every shape (A/B measurements, tests of that path)
static bool dequant_lut_path() {
  static const bool v = env_int("QB200_DEQUANT_LUT", 0) == 1;
  return v;
}

template <typename T>
static int launch_dequantize_nf4(const uint8_t* packed, const float* absmax, const uint8_t* absmax_u8,
                                 const float* code256, const float* absmax2, const float* offset, int64_t n,
                                 int blocksize, int blocksize2, T* out, cudaStream_t stream) {
  if (n == 0) return 0;
  // every kernel takes both forms' state pointers (those of the other form are null; blocksize2 = 1 for a plain state)
  const bool nested = absmax_u8 != nullptr;
  const bool vec_ok = (reinterpret_cast<uintptr_t>(out) % 16 == 0) && (reinterpret_cast<uintptr_t>(packed) % 4 == 0);
  const int64_t nwords = (n + 7) / 8;
  const int threads = 256;
  int64_t blocks = (nwords + threads * kDeqUnroll - 1) / (threads * kDeqUnroll);
  if constexpr (sizeof(T) == 2) {
    const bool bs2_pow2 = (blocksize2 & (blocksize2 - 1)) == 0;
    if (vec_ok && n % 8 == 0 && n < (int64_t(1) << 31) && bs2_pow2) {
      int bs_shift = 0, bs2_shift = 0;
      while ((8 << bs_shift) < blocksize) ++bs_shift;
      while ((1 << bs2_shift) < blocksize2) ++bs2_shift;
      if (n % 32 == 0 && reinterpret_cast<uintptr_t>(out) % 32 == 0 && reinterpret_cast<uintptr_t>(packed) % 16 == 0 &&
          !dequant_lut_path()) {
        const uint32_t nvec = uint32_t(n / 32);
        const auto kern = nested ? dequantize_nf4_tab_kernel<T, true> : dequantize_nf4_tab_kernel<T, false>;
        kern<<<tab_grid(nvec), threads, 0, stream>>>(reinterpret_cast<const uint4*>(packed), absmax, absmax_u8, code256, absmax2,
                                                     offset, nvec, bs_shift - 2, bs2_shift, reinterpret_cast<uint8_t*>(out));
        return check_launch("dequantize_nf4");
      }
      const int64_t fb_max = int64_t(device_sm_count()) * 16;
      const int64_t fb = blocks > fb_max ? fb_max : blocks;
      const auto kern = nested ? dequantize_nf4_fast_kernel<T, true> : dequantize_nf4_fast_kernel<T, false>;
      kern<<<(unsigned)fb, threads, 0, stream>>>(reinterpret_cast<const uint32_t*>(packed), absmax, absmax_u8, code256, absmax2, offset,
                                                 uint32_t(nwords), bs_shift, bs2_shift, reinterpret_cast<uint4*>(out));
      return check_launch("dequantize_nf4");
    }
  }
  const int64_t max_blocks = int64_t(device_sm_count()) * 8 * 8;  // grid-stride beyond a few waves of 8 resident CTAs/SM
  if (blocks > max_blocks) blocks = max_blocks;
  const auto kern = nested ? dequantize_nf4_kernel<T, true> : dequantize_nf4_kernel<T, false>;
  kern<<<(unsigned)blocks, threads, 0, stream>>>(packed, absmax, absmax_u8, code256, absmax2, offset, n, blocksize, blocksize2, vec_ok,
                                                 out);
  return check_launch("dequantize_nf4");
}

static bool valid_blocksize(int bs) { return bs >= 64 && bs <= 4096 && (bs & (bs - 1)) == 0; }

int launch_dequant_scratch(const qb200_nf4_problem& q, int64_t N, int64_t K, void* out, cudaStream_t stream) {
  const uint32_t nvec = uint32_t(N * K / 32);   // 32 values (16 packed bytes) per vector; blocks of 64, nested blocks of 256
  using BF = __nv_bfloat16;
  const auto kern = q.absmax_u8 != nullptr ? dequantize_nf4_tab_kernel<BF, true, true> : dequantize_nf4_tab_kernel<BF, false, true>;
  return launch_pdl(kern, tab_grid(nvec), 256, 0, stream, "dequantize_nf4_scratch", reinterpret_cast<const uint4*>(q.packed),
                    q.absmax_f32, q.absmax_u8, q.code256, q.absmax2, q.offset, nvec, 1, 8, static_cast<uint8_t*>(out));
}

}  // namespace qb200

using namespace qb200;

extern "C" int qb200_set_quant_math(int mode) {
  if (mode != 0 && mode != 1) return set_error(QB200_EINVAL, "set_quant_math: 0 = ieee, 1 = approx (rcp.approx.ftz + mul.ftz)");
  g_quant_math = mode;
  return 0;
}
extern "C" int qb200_get_quant_math(void) { return quant_math(); }

extern "C" int qb200_quantize_nf4(const void* A, int a_dtype, int64_t n, int blocksize, uint8_t* packed, float* absmax,
                                  void* stream) {
  if (n < 0 || (n > 0 && (!A || !packed || !absmax))) return set_error(QB200_EINVAL, "quantize_nf4: null pointer");
  if (!valid_blocksize(blocksize)) return set_error(QB200_EINVAL, "blocksize must be a power of two in [64, 4096]");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (a_dtype) {
    case kF32: return launch_quantize_nf4(static_cast<const float*>(A), n, blocksize, packed, absmax, s);
    case kF16: return launch_quantize_nf4(static_cast<const __half*>(A), n, blocksize, packed, absmax, s);
    case kBF16: return launch_quantize_nf4(static_cast<const __nv_bfloat16*>(A), n, blocksize, packed, absmax, s);
  }
  return set_error(QB200_EINVAL, "quantize_nf4: dtype must be 0 (fp32), 1 (fp16) or 2 (bf16)");
}

extern "C" int qb200_quantize_blockwise_8bit(const float* code256, const float* A, int64_t n, int blocksize,
                                             uint8_t* out, float* absmax, void* stream) {
  if (n < 0 || (n > 0 && (!code256 || !A || !out || !absmax))) return set_error(QB200_EINVAL, "quantize_8bit: null pointer");
  if (blocksize <= 0) return set_error(QB200_EINVAL, "quantize_8bit: blocksize must be positive");
  if (n == 0) return 0;
  const int64_t nblocks = (n + blocksize - 1) / blocksize;
  int64_t blocks = (nblocks + 7) / 8;
  if (blocks > int64_t(device_sm_count()) * 8) blocks = int64_t(device_sm_count()) * 8;
  if (quant_math())
    quantize_8bit_kernel<true><<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(code256, A, n, blocksize, out, absmax);
  else
    quantize_8bit_kernel<false><<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(code256, A, n, blocksize, out, absmax);
  return check_launch("quantize_blockwise_8bit");
}

extern "C" int qb200_dequantize_blockwise_8bit(const float* code256, const uint8_t* A, const float* absmax, int64_t n,
                                               int blocksize, float* out, void* stream) {
  if (n < 0 || (n > 0 && (!code256 || !A || !out || !absmax))) return set_error(QB200_EINVAL, "dequantize_8bit: null pointer");
  if (blocksize <= 0) return set_error(QB200_EINVAL, "dequantize_8bit: blocksize must be positive");
  if (n == 0) return 0;
  int64_t blocks = (n + 255) / 256;
  if (blocks > int64_t(device_sm_count()) * 8) blocks = int64_t(device_sm_count()) * 8;
  dequantize_8bit_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(code256, A, absmax, n, blocksize, out);
  return check_launch("dequantize_blockwise_8bit");
}

static int dequant_dispatch(const uint8_t* packed, const float* absmax, const uint8_t* absmax_u8, const float* code256,
                            const float* absmax2, const float* offset, int64_t n, int blocksize, int blocksize2,
                            void* out, int out_dtype, void* stream) {
  if (!valid_blocksize(blocksize)) return set_error(QB200_EINVAL, "blocksize must be a power of two in [64, 4096]");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (out_dtype) {
    case kF32: return launch_dequantize_nf4(packed, absmax, absmax_u8, code256, absmax2, offset, n, blocksize, blocksize2, static_cast<float*>(out), s);
    case kF16: return launch_dequantize_nf4(packed, absmax, absmax_u8, code256, absmax2, offset, n, blocksize, blocksize2, static_cast<__half*>(out), s);
    case kBF16: return launch_dequantize_nf4(packed, absmax, absmax_u8, code256, absmax2, offset, n, blocksize, blocksize2, static_cast<__nv_bfloat16*>(out), s);
  }
  return set_error(QB200_EINVAL, "dequantize_nf4: dtype must be 0 (fp32), 1 (fp16) or 2 (bf16)");
}

extern "C" int qb200_dequantize_nf4(const uint8_t* packed, const float* absmax, int64_t n, int blocksize, void* out,
                                    int out_dtype, void* stream) {
  if (n < 0 || (n > 0 && (!packed || !absmax || !out))) return set_error(QB200_EINVAL, "dequantize_nf4: null pointer");
  return dequant_dispatch(packed, absmax, nullptr, nullptr, nullptr, nullptr, n, blocksize, 1, out, out_dtype, stream);
}

extern "C" int qb200_dequantize_nf4_nested(const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                                           const float* absmax2, const float* offset, int64_t n, int blocksize,
                                           int blocksize2, void* out, int out_dtype, void* stream) {
  if (n < 0 || (n > 0 && (!packed || !absmax_u8 || !code256 || !absmax2 || !offset || !out)))
    return set_error(QB200_EINVAL, "dequantize_nf4_nested: null pointer");
  if (blocksize2 <= 0) return set_error(QB200_EINVAL, "dequantize_nf4_nested: blocksize2 must be positive");
  return dequant_dispatch(packed, nullptr, absmax_u8, code256, absmax2, offset, n, blocksize, blocksize2, out, out_dtype, stream);
}

// ---- upstream-named aliases (void return; errors recorded, never exit()) -------------
extern "C" void cquantize_blockwise_fp32_nf4(float*, float* A, float* absmax, unsigned char* out, int blocksize, const int n) {
  (void)qb200_quantize_nf4(A, kF32, n, blocksize, out, absmax, nullptr);
}
extern "C" void cquantize_blockwise_fp16_nf4(float*, void* A, float* absmax, unsigned char* out, int blocksize, const int n) {
  (void)qb200_quantize_nf4(A, kF16, n, blocksize, out, absmax, nullptr);
}
extern "C" void cquantize_blockwise_bf16_nf4(float*, void* A, float* absmax, unsigned char* out, int blocksize, const int n) {
  (void)qb200_quantize_nf4(A, kBF16, n, blocksize, out, absmax, nullptr);
}
extern "C" void cdequantize_blockwise_fp32_nf4(float*, unsigned char* A, float* absmax, float* out, int blocksize, const int n, void* stream) {
  (void)qb200_dequantize_nf4(A, absmax, n, blocksize, out, kF32, stream);
}
extern "C" void cdequantize_blockwise_fp16_nf4(float*, unsigned char* A, float* absmax, void* out, int blocksize, const int n, void* stream) {
  (void)qb200_dequantize_nf4(A, absmax, n, blocksize, out, kF16, stream);
}
extern "C" void cdequantize_blockwise_bf16_nf4(float*, unsigned char* A, float* absmax, void* out, int blocksize, const int n, void* stream) {
  (void)qb200_dequantize_nf4(A, absmax, n, blocksize, out, kBF16, stream);
}
extern "C" void cquantize_blockwise_fp32(float* code, float* A, float* absmax, unsigned char* out, int blocksize, const int n) {
  (void)qb200_quantize_blockwise_8bit(code, A, n, blocksize, out, absmax, nullptr);
}
extern "C" void cdequantize_blockwise_fp32(float* code, unsigned char* A, float* absmax, float* out, int blocksize, const int n, void* stream) {
  (void)qb200_dequantize_blockwise_8bit(code, A, absmax, n, blocksize, out, stream);
}
