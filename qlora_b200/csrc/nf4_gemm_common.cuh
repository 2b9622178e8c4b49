// Shared pieces of the fused NF4 dequant + wgmma GEMM kernel (sm_90a): launch parameters, the register-resident
// product-table dequant (16 x T16_rne(LUT[j]*absmax) per NF4 block, T16 = bf16 or fp16; nibbles resolved with PRMT byte permutes), the
// nested-absmax prefetch helper and the wgmma shared-memory descriptors.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdlib.h>

#include "nf4_common.cuh"
#include "nf4_table.cuh"
#include "qb200_internal.h"
#include "sm90_ptx.cuh"

namespace qb200 {
namespace gemm {

constexpr int kBlockF = 128;   // features per work unit (two wgmma M=64 halves)
constexpr int kBlockC = 64;    // contraction per step (one NF4 block; 128 B of 16-bit values = one swizzle row)
constexpr int kMmaK = 16;
constexpr int kATileBytes = kBlockF * kBlockC * 2;    // 16 KB: one dequantized wgmma A-operand tile
constexpr int kWTileBytes = kBlockF * kBlockC / 2;    // 4 KB: the packed nibbles of that tile
constexpr int kAuxBytes = 1024 + 3 * 1024;            // barriers (1 KB), one code256 copy per problem of a group

constexpr int kMaxProb = 3;    // problems per grouped launch (q/k/v, gate/up)

// One Linear4bit of a (possibly grouped) launch: the quantization state of W[N,K] plus its output / bias.
struct Prob {
  const uint8_t* packed;     // packed nibbles, row-major [N, K/2]
  const uint8_t* absmax_u8;  // nested state (or null)
  const float* code256;
  const float* absmax2;
  const float* offset;
  const float* absmax_f32;   // non-nested state (or null)
  const void* bias;          // [F] of the operand type (bf16 / fp16), or null (forward only)
  const float* row_scale;    // [N] or null: the absmax of every NF4 block of row n of W is multiplied by row_scale[n]
                             // (forward: Out = In . (diag(s) W)^T; dX: Out = In . diag(s) W).  Written by earlier kernels.
  void* out;                 // [T, F] of the operand type (or fp32 when Params::out_f32), row pitch ld_out elements
  int64_t ld_out;
};

struct Params {
  Prob pr[kMaxProb];
  int nprob;                 // 1..kMaxProb
  int group_sum;             // 0: every problem has its own output (forward q/k/v, gate/up: same input, outputs side by side)
                             // 1: ONE output, the problems are segments of one long contraction (dX of q/k/v: sum_p dY_p . W_p)
  int T, F, C;
  int K;                     // row pitch of W[N,K] in elements
  int N;                     // rows of W
  int lora_r;                // > 0: ceil(r / 64) extra 16-bit contraction steps per problem  Out += U_p[T,r] . V_p^T
  int out_f32;               // 1: the drain writes fp32 (Linear4bit called with fp32 activations: no separate cast pass)
  float* ws;                 // split-K: fp32 partial sums [ksplit, T, F] (null otherwise)
  int debug;                 // ablation flags for performance triage (QB200_DEBUG_FLAGS; 0 in production):
                             //   1 = skip dequant math+stores, 2 = skip MMA issue, 4 = skip epilogue stores
};

using qb200::build_table;
using qb200::dequant_word;
using qb200::lookup4;
using qb200::Nf4Table;

template <bool kNested>
struct AbsmaxFetch {
  uint32_t code;
  float a2;
  float am;
  __device__ __forceinline__ void issue(const Prob& p, int64_t blk, bool valid) {
    if (kNested) {
      code = valid ? uint32_t(__ldg(p.absmax_u8 + blk)) : 0u;
      a2 = valid ? __ldg(p.absmax2 + (blk >> 8)) : 0.0f;
    } else {
      am = valid ? __ldg(p.absmax_f32 + blk) : 0.0f;
    }
  }
  __device__ __forceinline__ float resolve(const float* s_code, float offset, bool valid) const {
    if (kNested) return valid ? nested_absmax(s_code[code], a2, offset) : 0.0f;
    return am;
  }
};

// wgmma shared-memory matrix descriptors (sm_90): start >> 4 at [0,14), LBO >> 4 at [16,30), SBO >> 4 at [32,46),
// base offset 0 (tiles are 1024-byte aligned), layout type at [62,64): 1 = SWIZZLE_128B.
__device__ __forceinline__ uint64_t make_desc_kmajor_sw128(uint32_t smem_addr) {
  // K-major, SWIZZLE_128B: rows of 128 B, 8-row groups 1024 B apart (SBO); LBO unused (=1).
  return uint64_t((smem_addr >> 4) & 0x3FFFu) | (uint64_t(1) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}
__device__ __forceinline__ uint64_t make_desc_mnmajor_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  // MN-major, SWIZZLE_128B: atoms of 64 (MN) x 8 (K) elements = 1024 B; LBO = stride between
  // 64-element groups along MN, SBO = stride between 8-row groups along K.
  return uint64_t((smem_addr >> 4) & 0x3FFFu) | (uint64_t((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         (uint64_t((sbo_bytes >> 4) & 0x3FFFu) << 32) | (uint64_t(1) << 62);
}

}  // namespace gemm
}  // namespace qb200
