// NF4(+double-quant) skinny forward GEMM for 1..16 tokens: y[m, n] = sum_k x[m, k] * W[n, k] (+ bias) (+ sum_j U[m, j] * V[n, j],
// the LoRA term of an unmerged adapter).
//
// Replaces the reference's bs-1 generation path (SURVEY.md 2.4 K6 `kgemm_4bit_inference_naive`, reached from
// examples/guanaco_generate.py:63-78 and qlora.py:817-834 through bnb.matmul_4bit when A.numel() == A.shape[-1];
// README.md:135 calls 4-bit inference slow) and the few-token forward calls below the wgmma tile sizes.
// The packed weight (N*K/2 B) + u8 absmax (N*K/64 B) are streamed exactly once; W is never materialised.
//
// Warp-level tensor-core path (mma.sync m16n8k16 bf16 or f16, fp32 accumulate) — the one place this library uses mma.sync:
// the kernel is bound by the NF4 look-up on the ALU pipe (~3 PRMT/LOP/SHF per weight), not by tensor throughput, and
// mma.sync takes its operands from registers: the look-up output (16-bit pair words holding the same bit-exact weights
// T16_rne(LUT[j] * absmax) as every other path; T16 = bf16 or fp16, the operand type of the launch) IS the B fragment, so nothing is unpacked, multiplied or staged per
// weight, and 8 tokens cost the same as one.  (Round-1 history: a scalar-FMA GEMV paid look-up + unpack + FMA per weight
// and token — ncu ALU pipe 61 %, DRAM 10 %, 12.1 us at 4096^2 for one token and 29.7 us for four.)
//
// Mapping (PTX m16n8k16 fragments; g = lane >> 2, t = lane & 3): a warp owns 8 weight rows (B column n = g); within one
// step its 4 thread columns t own 4 DIFFERENT 64-value NF4 blocks of the row — the contraction index is only a label,
// so the "k slots" of an MMA are mapped to real positions of thread t's block, for A and B alike.  Each thread therefore
// builds one product table per 32 B of packed nibbles it streams (one block): the table cost is amortised over 64
// weights and every global weight load is a full 32-byte sector.  A CTA = one 8-row tile with the contraction split over
// its warps; partial sums meet in shared memory.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "nf4_common.cuh"
#include "nf4_table.cuh"
#include "qb200_internal.h"
#include "sm90_ptx.cuh"

namespace qb200 {
namespace skinny {

constexpr int kRows = 8;      // weight rows per CTA (MMA n)
constexpr int kMaxNT = 2;     // up to 2 groups of 8 tokens per launch

using Table = Nf4Table;   // nf4_table.cuh: 16 16-bit products of one NF4 block as low-byte / high-byte planes

// (a & b) | c in one LOP3 with all three operands in registers (with immediates the compiler needs two)
__device__ __forceinline__ uint32_t and_or(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

// One packed word (8 nibbles, byte j = (element 2j << 4) | element 2j+1) -> 4 16-bit pair words in element order.
// Per half (4 nibbles): PRMT picks entry (n & 7) from the first and the second 8 table entries, a third PRMT chooses
// between them on bit 3 of the nibble; same for the high-byte plane; two more PRMTs interleave the planes.
// prmt reads only bits [15:0] of its selector, so the selector words are prepared once for both halves.
__device__ __forceinline__ void lookup8(uint32_t word, const Table& t, uint32_t k4444, uint32_t k3210, uint32_t (&w)[4]) {
  const uint32_t sa = word & 0x77777777u;
  const uint32_t sb = and_or(word >> 1, k4444, k3210);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint32_t sel_a = h ? (sa >> 16) : sa, sel_b = h ? (sb >> 16) : sb;
    const uint32_t lo = ptx::prmt(ptx::prmt(t.tl[0], t.tl[1], sel_a), ptx::prmt(t.tl[2], t.tl[3], sel_a), sel_b);
    const uint32_t hi = ptx::prmt(ptx::prmt(t.th[0], t.th[1], sel_a), ptx::prmt(t.th[2], t.th[3], sel_a), sel_b);
    w[2 * h] = ptx::prmt(lo, hi, 0x4051);
    w[2 * h + 1] = ptx::prmt(lo, hi, 0x6273);
  }
}

#define QB200_MMA_16816(ty)                                                                                               \
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." ty "." ty ".f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};" \
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])                                                      \
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1))
template <typename T16>
__device__ __forceinline__ void mma_16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  if constexpr (std::is_same<T16, __half>::value) QB200_MMA_16816("f16");
  else QB200_MMA_16816("bf16");
}
#undef QB200_MMA_16816

// LoRA term of one output value: sum_j U[m, j] * V[row, j] over the rank (T16 operands, fp32 sum) — the extra contraction
// steps the wgmma kernel runs on the tensor core, here 8..256 multiply-adds in the epilogue.  U = scaling * x . A^T [M, r]
// comes from the caller (one small GEMM), V = lora_B.weight [N, r]; rows are 16-byte aligned (r % 8 == 0).
template <typename T16>
__device__ __forceinline__ float lora_dot(const T16* __restrict__ u, const T16* __restrict__ v, int r) {
  using T2 = typename Vec2<T16>::type;
  float acc = 0.0f;
  // chunks of 64 ranks, summed in rank order into one accumulator: r <= 64 is one chunk, the sum it always was
  for (int c0 = 0; c0 < r; c0 += 64) {
    // all (at most 8 + 8) 16-byte loads of the chunk are issued before its first multiply: one memory round trip per
    // chunk, not r / 8 of them
    uint4 a[8], b[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (c0 + 8 * i < r) {
        a[i] = *reinterpret_cast<const uint4*>(u + c0 + 8 * i);     // produced by the previous kernel: plain load
        b[i] = __ldg(reinterpret_cast<const uint4*>(v + c0 + 8 * i));
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (c0 + 8 * i < r) {
        const T2* a2 = reinterpret_cast<const T2*>(&a[i]);
        const T2* b2 = reinterpret_cast<const T2*>(&b[i]);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 fa = widen2(a2[e]), fb = widen2(b2[e]);
          acc = fmaf(fa.x, fb.x, acc);
          acc = fmaf(fa.y, fb.y, acc);
        }
      }
    }
  }
  return acc;
}

struct BlockRegs {
  uint4 lo, hi;      // 32 B of packed nibbles = one 64-value block
  uint32_t code;     // nested: u8 absmax code
  float scale;       // nested: absmax2 of the block's group; plain: fp32 absmax
};

__device__ __forceinline__ void cp_async_16(uint32_t dst_smem, const void* src, bool valid) {
  // src-size 0 zero-fills the 16 destination bytes (src is still a valid address)
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

constexpr int kSlabRowBytes = 512;       // x slab of one step: 4 blocks x 64 values x 2 B per token

// Output type of a skinny launch: T16, or fp16 for a bf16-compute launch with fp16 output (kOutF16), which stores the
// bf16-rounded result rounded to fp16.
template <typename T16, bool kOutF16>
using SkinnyOut = typename std::conditional<kOutF16, __half, T16>::type;
template <typename T16, bool kOutF16>
__device__ __forceinline__ SkinnyOut<T16, kOutF16> round_out(float v) {
  if constexpr (kOutF16) return bf16_to_f16(round16<T16>(v));
  else return round16<T16>(v);
}

// NT: groups of 8 tokens; kWarps: contraction split inside the CTA; kRing: blocks in flight per thread.
// (4 warps x 4 blocks in flight measured faster than 8 warps x 2: 11.2 vs 11.5-13.2 us at 4096^2, one token, ncu.)
//
// A operand.  One step of a warp covers 4 consecutive NF4 blocks (256 positions) of its 8 weight rows; the matching x
// slab [tokens][256] is copied global -> shared once per step with coalesced 16-byte cp.async (one instruction per token
// row) and read back as MMA A quads with conflict-free 128-bit shared loads (16-byte chunk index XOR-swizzled by block and
// token parity).  Loading the quads straight from global costs one L1 tag look-up per (token, block) line and instruction —
// 32 per load at 8 tokens — and made the first version L1-bound above 8 tokens (ncu: LSU wavefronts 73 %).
//
// The A quad is 8 consecutive positions of ONE token used as it lands in registers: fragment rows g and g + 8 then both
// belong to token g, row g seeing positions (0,1,4,5) and row g + 8 positions (2,3,6,7) of the 8.  MMA 1 pairs it with
// B = weights (0,1 | 4,5) — its rows g are the wanted partial sums — and MMA 2 with B = weights (2,3 | 6,7) — its rows g + 8
// are; the other half of each result is discarded.  Half of the MMA is wasted, but no register is moved between the
// look-up and the tensor core.
//
// B operand.  Each thread keeps kRing blocks (32 B of nibbles + absmax statistics each) in flight in registers
// (the first version waited on one block at a time: ncu long-scoreboard 5.6 stalls / issue).
// kStateF16: bf16 compute over an fp16 quant state (build_table); kOutF16: see SkinnyOut.
// kMixed: every token m reads its own adapter (MixedLora below): lora_v is unused and lora_r is the column count of U.
template <typename T16, int NT, int kWarps, int kRing, bool kNested, bool kStateF16, bool kOutF16, bool kMixed>
__device__ __forceinline__ void
skinny_body(const T16* __restrict__ x, const uint8_t* __restrict__ packed, const uint8_t* __restrict__ absmax_u8,
            const float* __restrict__ code256, const float* __restrict__ absmax2, const float* __restrict__ offset_ptr,
            const float* __restrict__ absmax_f32, const T16* __restrict__ bias, SkinnyOut<T16, kOutF16>* __restrict__ y, int M,
            int N, int K, const T16* __restrict__ lora_u, int ld_u, const T16* __restrict__ lora_v,
            int lora_r, int64_t ld_x, int64_t ld_y, const float* __restrict__ row_scale, MixedLora mix) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  // [kWarps][NT * 8 tokens][512 B] x slabs, then 256 floats codebook; the slabs are re-used for the partial sums at the end
  uint8_t* slab_base = smem_raw;
  float* s_code = reinterpret_cast<float*>(smem_raw + kWarps * NT * 8 * kSlabRowBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n = blockIdx.x * kRows + g;                      // N % 8 == 0: always a valid row
  const int nblk = K >> 6;
  const int ntok = min(M, NT * 8);
  const uint8_t* __restrict__ wrow = packed + int64_t(n) * (K >> 1);
  const int64_t blk_base = int64_t(n) * nblk;
  const uint32_t slab = static_cast<uint32_t>(__cvta_generic_to_shared(slab_base + warp * NT * 8 * kSlabRowBytes));

  auto fetch = [&](int b, BlockRegs& r) {
    r.lo = r.hi = make_uint4(0, 0, 0, 0);
    r.code = 0;
    r.scale = 0.0f;
    if (b < nblk) {
      const uint4* src = reinterpret_cast<const uint4*>(wrow + (int64_t(b) << 5));
      r.lo = __ldg(src);
      r.hi = __ldg(src + 1);
      if (kNested) {
        r.code = __ldg(absmax_u8 + blk_base + b);
        r.scale = __ldg(absmax2 + ((blk_base + b) >> 8));
      } else {
        r.scale = __ldg(absmax_f32 + blk_base + b);
      }
    }
  };
  // x slab of the block group starting at block `bg` -> this warp's shared buffer.  Lane L copies 16 B = positions
  // [8 L, 8 L + 8) of the 256; block L >> 3, chunk L & 7.  Blocks beyond the row are zero-filled.
  auto stage = [&](int bg) {
    const int blk = lane >> 3, j = lane & 7;
    const bool valid = bg + blk < nblk;
    const T16* src = x + (valid ? (int64_t(bg) << 6) + (lane << 3) : 0);
    for (int tok = 0; tok < ntok; ++tok) {
      const uint32_t dst = slab + tok * kSlabRowBytes + blk * 128 + ((j ^ (blk | ((tok & 1) << 2))) << 4);
      cp_async_16(dst, src + int64_t(tok) * ld_x, valid);
    }
  };

  // this thread's blocks: 4 * (warp + kWarps s) + t, s = 0, 1, ...; group base (warp-uniform) bg = 4 * (warp + kWarps s)
  // Programmatic dependent launch: the next kernel of the stream may start its own weight prefetch while this one runs;
  // the packed weights / absmax statistics are constants of the model, so they are fetched BEFORE waiting for the
  // previous kernel — only x (and later bias / y) can be its output.
  ptx::grid_dep_launch();
  const int b0 = 4 * warp + t;
  BlockRegs ring[kRing];
#pragma unroll
  for (int u = 0; u < kRing; ++u) fetch(b0 + 4 * kWarps * u, ring[u]);
  ptx::grid_dep_wait();
  stage(4 * warp);
  // optional per-row weight scale (an earlier kernel's output: read after the wait); every block of this thread is in row n
  const float rs = row_scale != nullptr ? __ldg(row_scale + n) : 1.0f;
  float offset = 0.0f;
  if (kNested) {
    for (int i = threadIdx.x; i < 256; i += 32 * kWarps) s_code[i] = __ldg(code256 + i);
    offset = __ldg(offset_ptr);
  }
  __syncthreads();

  float acc[NT][2][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[nt][0][i] = acc[nt][1][i] = 0.0f;

  // fragment read address of (token group nt, word j): slab + (nt*8 + g) * 512 + t * 128 + ((j ^ swz) << 4)
  const uint32_t frag = slab + g * kSlabRowBytes + t * 128;
  const uint32_t swz = t | ((g & 1) << 2);
  uint32_t k4444 = 0x44444444u, k3210 = 0x32103210u;          // kept in registers for the 3-register LOP3 of lookup8
  asm volatile("" : "+r"(k4444), "+r"(k3210));

  // mma.sync is warp-collective: trip counts depend on the warp's block group only; a thread whose own block lies beyond
  // the row (K/64 not a multiple of 4) runs the step with an all-zero table against the zero-filled slab
  for (int bg = 4 * warp; bg < nblk; bg += 4 * kWarps * kRing) {
#pragma unroll
    for (int u = 0; u < kRing; ++u) {
      const int bgu = bg + 4 * kWarps * u;
      if (bgu >= nblk) break;
      const int b = bgu + t;
      cp_async_wait_all();
      __syncwarp();
      const BlockRegs cur = ring[u];
      fetch(b + 4 * kWarps * kRing, ring[u]);
      float am = kNested ? nested_absmax(s_code[cur.code], cur.scale, offset) : cur.scale;
      if (row_scale != nullptr) am = __fmul_rn(am, rs);
      if (b >= nblk) am = 0.0f;
      Table tab;
      build_table<T16, kStateF16>(am, tab);
      const uint32_t words[8] = {cur.lo.x, cur.lo.y, cur.lo.z, cur.lo.w, cur.hi.x, cur.hi.y, cur.hi.z, cur.hi.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t w[4];                                        // weights 8j..8j+7 of the block, 16-bit pairs in element order
        lookup8(words[j], tab, k4444, k3210, w);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const uint4 v = lds128(frag + nt * 8 * kSlabRowBytes + ((j ^ swz) << 4));   // x[token, 64 b + 8 j .. + 8)
          mma_16816<T16>(acc[nt][0], v.x, v.y, v.z, v.w, w[0], w[2]);
          mma_16816<T16>(acc[nt][1], v.x, v.y, v.z, v.w, w[1], w[3]);
        }
      }
      __syncwarp();                                           // every lane has read the slab: overwrite it
      if (bgu + 4 * kWarps < nblk) stage(bgu + 4 * kWarps);
    }
  }

  // wanted halves: acc[.][0] rows g (c0, c1) and acc[.][1] rows g + 8 (c2, c3), both = (token g, weight rows 2t, 2t+1)
  __syncthreads();                                            // all slabs are dead: re-use the space for the partial sums
  float* s_red = reinterpret_cast<float*>(smem_raw);          // [kWarps][NT][8 tokens * 8 rows]
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    float* r = s_red + (warp * NT + nt) * 8 * kRows;
    r[g * kRows + 2 * t] = acc[nt][0][0] + acc[nt][1][2];
    r[g * kRows + 2 * t + 1] = acc[nt][0][1] + acc[nt][1][3];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < NT * 8 * kRows; e += 32 * kWarps) {
    const int nt = e / (8 * kRows), i = e % (8 * kRows);
    const int m = nt * 8 + i / kRows, row = blockIdx.x * kRows + i % kRows;
    if (m >= M) continue;
    float v = 0.0f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) v += s_red[(w * NT + nt) * 8 * kRows + i];
    if constexpr (kMixed) {
      const qb200_lora_adapter* ad = mix.adapter(m);
      const int r = ad != nullptr ? mix.rank(*ad, lora_r) : 0;
      if (r > 0) v += lora_dot(lora_u + int64_t(m) * ld_u, static_cast<const T16*>(ad->B) + int64_t(row) * r, r);
    } else {
      if (lora_r > 0) v += lora_dot(lora_u + int64_t(m) * ld_u, lora_v + int64_t(row) * lora_r, lora_r);
    }
    if (bias != nullptr) v += widen(bias[row]);
    y[int64_t(m) * ld_y + row] = round_out<T16, kOutF16>(v);
  }
}

template <typename T16, int NT, int kWarps, int kRing, bool kNested, bool kStateF16, bool kOutF16>
__global__ void __launch_bounds__(32 * kWarps, 4)
nf4_skinny_kernel(const T16* __restrict__ x, const uint8_t* __restrict__ packed, const uint8_t* __restrict__ absmax_u8,
                  const float* __restrict__ code256, const float* __restrict__ absmax2, const float* __restrict__ offset_ptr,
                  const float* __restrict__ absmax_f32, const T16* __restrict__ bias, SkinnyOut<T16, kOutF16>* __restrict__ y, int M,
                  int N, int K, const T16* __restrict__ lora_u, int ld_u, const T16* __restrict__ lora_v,
                  int lora_r, int64_t ld_x, int64_t ld_y, const float* __restrict__ row_scale) {
  skinny_body<T16, NT, kWarps, kRing, kNested, kStateF16, kOutF16, false>(x, packed, absmax_u8, code256, absmax2, offset_ptr,
                                                                        absmax_f32, bias, y, M, N, K, lora_u, ld_u, lora_v, lora_r,
                                                                        ld_x, ld_y, row_scale, MixedLora{});
}

template <typename T16, int NT, int kWarps, int kRing, bool kNested, bool kStateF16, bool kOutF16>
__global__ void __launch_bounds__(32 * kWarps, 4)
nf4_skinny_kernel_mixed(const T16* __restrict__ x, const uint8_t* __restrict__ packed, const uint8_t* __restrict__ absmax_u8,
                        const float* __restrict__ code256, const float* __restrict__ absmax2, const float* __restrict__ offset_ptr,
                        const float* __restrict__ absmax_f32, const T16* __restrict__ bias, SkinnyOut<T16, kOutF16>* __restrict__ y,
                        int M, int N, int K, const T16* __restrict__ lora_u, int ld_u, int lora_r, int64_t ld_x, int64_t ld_y,
                        MixedLora mix) {
  skinny_body<T16, NT, kWarps, kRing, kNested, kStateF16, kOutF16, true>(x, packed, absmax_u8, code256, absmax2, offset_ptr,
                                                                       absmax_f32, bias, y, M, N, K, lora_u, ld_u, nullptr, lora_r,
                                                                       ld_x, ld_y, nullptr, mix);
}

// q's row pitches are resolved (non-zero).  Both instantiations take the full set of state pointers: the nested one reads
// only absmax_u8 / code256 / absmax2 / offset, the plain one only absmax_f32.
template <typename T16, bool kStateF16, bool kOutF16, int NT, int kWarps, int kRing>
static int launch_cfg(const qb200_nf4_problem& q, const float* row_scale, int M, int N, int K, int R, cudaStream_t stream) {
  constexpr int smem = kWarps * NT * 8 * kSlabRowBytes + 256 * int(sizeof(float));
  static_assert(smem <= 48 * 1024, "static opt-in not needed below 48 KB");
  const auto kern = q.absmax_u8 != nullptr ? nf4_skinny_kernel<T16, NT, kWarps, kRing, true, kStateF16, kOutF16>
                                           : nf4_skinny_kernel<T16, NT, kWarps, kRing, false, kStateF16, kOutF16>;
  return launch_pdl(kern, unsigned(N / kRows), 32 * kWarps, smem, stream, "nf4_skinny", static_cast<const T16*>(q.in), q.packed,
                    q.absmax_u8, q.code256, q.absmax2, q.offset, q.absmax_f32, static_cast<const T16*>(q.bias),
                    static_cast<SkinnyOut<T16, kOutF16>*>(q.out), M, N, K, static_cast<const T16*>(q.U), int(q.ld_u),
                    static_cast<const T16*>(q.V), R, q.ld_in, q.ld_out, row_scale);
}

template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }

// ONE token — the case the reference has a dedicated kernel for (kgemm_4bit_inference_naive runs when A.numel() ==
// A.shape[-1], i.e. model.generate() with batch 1).  Same MMA mapping as nf4_skinny_kernel above, specialised:
//   * the x slab of a step is one 512-byte row: a single cp.async per lane stages it, kBuf steps ahead (double-buffered),
//     and every fragment row reads it back as a broadcast — result rows 1..7 repeat row 0 and are never stored;
//   * a block's registers are consumed in place and refilled right after its last look-up (the general kernel copies the
//     block out first: 273 register moves per 256 weights, 7.4 issue slots per weight against 4.7 here);
//   * loads beyond the row are clamped to its last block and cancelled by an all-zero product table: no load is predicated.
// Measured (CUDA graph of back-to-back launches over weight copies larger than L2, µs per launch, general kernel -> this):
// 4096^2 8.85 -> 8.45, 11008x4096 16.97 -> 15.97, 4096x11008 19.11 -> 16.69.  What bounds it is the ALU pipe: the exact
// look-up costs 2.1 PRMT + 1.3 other ALU instructions per weight at 64 lanes/clk/SM (ncu, 4096x11008: ALU pipe 64 % of its
// peak while SMs are active, issue slots 44 %, SMs active 71 % of the kernel) — a ceiling of ~2.7 TB/s of packed weights,
// 0.42 of the HBM roofline, before launch and tail; DESIGN.md 4.3.
// kMixed: as in skinny_body.
template <typename T16, int kWarps, int kRing, int kBuf, bool kNested, bool kStateF16, bool kOutF16, bool kMixed>
__device__ __forceinline__ void
skinny_1tok_body(const T16* __restrict__ x, const uint8_t* __restrict__ packed, const uint8_t* __restrict__ absmax_u8,
                 const float* __restrict__ code256, const float* __restrict__ absmax2, const float* __restrict__ offset_ptr,
                 const float* __restrict__ absmax_f32, const T16* __restrict__ bias, SkinnyOut<T16, kOutF16>* __restrict__ y,
                 int N, int K, const T16* __restrict__ lora_u, const T16* __restrict__ lora_v, int lora_r,
                 const float* __restrict__ row_scale, MixedLora mix) {
  using T2 = typename Vec2<T16>::type;
  constexpr int kWarpSlab = kBuf * kSlabRowBytes;
  static_assert(kRing % kBuf == 0, "the slab of ring slot u is buffer u % kBuf");
  static_assert(32 * kWarps >= 16 * kRows, "the LoRA epilogue uses 16 lanes per weight row");
  extern __shared__ __align__(128) uint8_t smem_raw[];
  // [kWarps][kBuf][512 B] x slabs, then 256 floats codebook; the slabs are re-used for the partial sums at the end
  float* s_code = reinterpret_cast<float*>(smem_raw + kWarps * kWarpSlab);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n = blockIdx.x * kRows + g;                      // N % 8 == 0: always a valid row
  const int nblk = K >> 6;
  const int ngrp = (nblk + 3) >> 2;                          // block groups of the row; this warp takes warp, warp + kWarps, ...
  const int nsteps = ngrp > warp ? (ngrp - warp + kWarps - 1) / kWarps : 0;
  const uint8_t* __restrict__ wrow = packed + int64_t(n) * (K >> 1);
  const int64_t blk_base = int64_t(n) * nblk;
  const uint32_t slab = static_cast<uint32_t>(__cvta_generic_to_shared(smem_raw + warp * kWarpSlab));

  // block of (step s, thread column t), clamped into the row
  auto fetch = [&](int s, BlockRegs& r) {
    const int b = min(4 * (warp + kWarps * s) + t, nblk - 1);
    const uint4* src = reinterpret_cast<const uint4*>(wrow + (b << 5));
    r.lo = __ldg(src);
    r.hi = __ldg(src + 1);
    if (kNested) {
      r.code = __ldg(absmax_u8 + blk_base + b);
      r.scale = __ldg(absmax2 + ((blk_base + b) >> 8));
    } else {
      r.scale = __ldg(absmax_f32 + blk_base + b);
    }
  };
  // x slab of step s -> buffer `buf` of this warp: lane L copies 16 B = positions [8 L, 8 L + 8) of the 256 (block L >> 3,
  // chunk L & 7, chunk index XOR-swizzled by the block); blocks beyond the row are zero-filled
  auto stage = [&](int s, int buf) {
    const int bg = 4 * (warp + kWarps * s);
    const int blk = lane >> 3, j = lane & 7;
    const bool valid = bg + blk < nblk;
    cp_async_16(slab + buf * kSlabRowBytes + blk * 128 + ((j ^ blk) << 4), x + (valid ? (bg << 6) + (lane << 3) : 0), valid);
  };

  // programmatic dependent launch, as in nf4_skinny_kernel: weights and codebook first, then wait for the producer of x
  ptx::grid_dep_launch();
  BlockRegs ring[kRing];
#pragma unroll
  for (int u = 0; u < kRing; ++u) fetch(u, ring[u]);
  float offset = 0.0f;
  if (kNested) {
    for (int i = threadIdx.x; i < 256; i += 32 * kWarps) s_code[i] = __ldg(code256 + i);
    offset = __ldg(offset_ptr);
  }
  ptx::grid_dep_wait();
#pragma unroll
  for (int u = 0; u < kBuf; ++u) {
    if (u < nsteps) stage(u, u);
    cp_async_commit();
  }
  const float rs = row_scale != nullptr ? __ldg(row_scale + n) : 1.0f;   // as in nf4_skinny_kernel
  __syncthreads();

  float acc[2][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) acc[0][i] = acc[1][i] = 0.0f;

  // fragment read address of word j of this thread's block: slab + buffer + t * 128 + ((j ^ t) << 4), the same for every
  // fragment row g (a broadcast); the 8 swizzled offsets are loop invariants kept in registers
  uint32_t fword[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) fword[j] = slab + t * 128 + ((j ^ t) << 4);
  uint32_t k4444 = 0x44444444u, k3210 = 0x32103210u;          // kept in registers for the 3-register LOP3 of lookup8
  asm volatile("" : "+r"(k4444), "+r"(k3210));

  // mma.sync is warp-collective: trip counts depend on the warp's block groups only; a thread whose own block lies beyond
  // the row (K/64 not a multiple of 4) runs the step with an all-zero table against the zero-filled slab
  for (int s0 = 0; s0 < nsteps; s0 += kRing) {
#pragma unroll
    for (int u = 0; u < kRing; ++u) {
      const int s = s0 + u;
      if (s >= nsteps) break;
      cp_async_wait_group<kBuf - 1>();                        // the slab of step s has landed (later ones may be in flight)
      __syncwarp();
      BlockRegs& cur = ring[u];
      float am = kNested ? nested_absmax(s_code[cur.code], cur.scale, offset) : cur.scale;
      if (row_scale != nullptr) am = __fmul_rn(am, rs);
      if (4 * (warp + kWarps * s) + t >= nblk) am = 0.0f;
      Table tab;
      build_table<T16, kStateF16>(am, tab);
      const int buf_off = (u % kBuf) * kSlabRowBytes;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t word = j == 0 ? cur.lo.x : j == 1 ? cur.lo.y : j == 2 ? cur.lo.z : j == 3 ? cur.lo.w
                            : j == 4 ? cur.hi.x : j == 5 ? cur.hi.y : j == 6 ? cur.hi.z : cur.hi.w;
        uint32_t w[4];                                        // weights 8j..8j+7 of the block, 16-bit pairs in element order
        lookup8(word, tab, k4444, k3210, w);
        const uint4 v = lds128(fword[j] + buf_off);           // x[64 b + 8 j .. + 8)
        mma_16816<T16>(acc[0], v.x, v.y, v.z, v.w, w[0], w[2]);
        mma_16816<T16>(acc[1], v.x, v.y, v.z, v.w, w[1], w[3]);
      }
      fetch(s + kRing, cur);                                  // clamped: a step beyond the row re-reads its last block
      __syncwarp();                                           // every lane has read the slab: overwrite it
      if (s + kBuf < nsteps) stage(s + kBuf, u % kBuf);
      cp_async_commit();
    }
  }
  cp_async_wait_group<0>();

  // wanted halves: acc[0] rows g (c0, c1) and acc[1] rows g + 8 (c2, c3), both = weight rows 2t, 2t+1; every g holds the
  // same token, lanes g == 0 publish
  __syncthreads();                                            // all slabs are dead: re-use the space for the partial sums
  float* s_red = reinterpret_cast<float*>(smem_raw);          // [kWarps + 1][8 rows]; the last row holds the LoRA terms
  if (g == 0) {
    s_red[warp * kRows + 2 * t] = acc[0][0] + acc[1][2];
    s_red[warp * kRows + 2 * t + 1] = acc[0][1] + acc[1][3];
  }
  if constexpr (kMixed) {                                     // the token's own adapter, or none
    const qb200_lora_adapter* ad = mix.adapter(0);
    lora_r = ad != nullptr ? mix.rank(*ad, lora_r) : 0;
    if (ad != nullptr) lora_v = static_cast<const T16*>(ad->B);
  }
  if (lora_r > 0) {
    // 16 lanes per weight row, 4 rank entries of each 64-rank chunk each (r <= 256: up to 4 chunks), every chunk summed by
    // xor-shuffles and the chunk sums added in rank order (r <= 64: one chunk, the sum it always was).  All loads are issued
    // before the first multiply; they overlap the barrier.
    constexpr int kChunks = kMaxLoraRank / 64;
    const int row = threadIdx.x >> 4, c = (threadIdx.x & 15) << 2;
    const T16* vrow = lora_v + int64_t(blockIdx.x * kRows + row) * lora_r;
    uint2 a[kChunks], b[kChunks];
#pragma unroll
    for (int k = 0; k < kChunks; ++k) {
      if (row < kRows && 64 * k + c < lora_r) {
        a[k] = *reinterpret_cast<const uint2*>(lora_u + 64 * k + c);
        b[k] = __ldg(reinterpret_cast<const uint2*>(vrow + 64 * k + c));
      }
    }
    float sum = 0.0f;
#pragma unroll
    for (int k = 0; k < kChunks; ++k) {
      if (64 * k >= lora_r) break;
      float part = 0.0f;
      if (row < kRows && 64 * k + c < lora_r) {
        const float2 a0 = widen2(*reinterpret_cast<const T2*>(&a[k].x));
        const float2 a1 = widen2(*reinterpret_cast<const T2*>(&a[k].y));
        const float2 b0 = widen2(*reinterpret_cast<const T2*>(&b[k].x));
        const float2 b1 = widen2(*reinterpret_cast<const T2*>(&b[k].y));
        part = fmaf(a0.x, b0.x, fmaf(a0.y, b0.y, fmaf(a1.x, b1.x, a1.y * b1.y)));
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
      sum = k == 0 ? part : sum + part;
    }
    if (row < kRows && (threadIdx.x & 15) == 0) s_red[kWarps * kRows + row] = sum;
  }
  __syncthreads();
  if (threadIdx.x < kRows) {
    const int row = blockIdx.x * kRows + threadIdx.x;
    float v = 0.0f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) v += s_red[w * kRows + threadIdx.x];
    if (lora_r > 0) v += s_red[kWarps * kRows + threadIdx.x];
    if (bias != nullptr) v += widen(bias[row]);
    y[row] = round_out<T16, kOutF16>(v);
  }
}

template <typename T16, int kWarps, int kRing, int kBuf, bool kNested, bool kStateF16, bool kOutF16>
__global__ void __launch_bounds__(32 * kWarps, 4)
nf4_skinny_kernel_1tok(const T16* __restrict__ x, const uint8_t* __restrict__ packed, const uint8_t* __restrict__ absmax_u8,
                       const float* __restrict__ code256, const float* __restrict__ absmax2, const float* __restrict__ offset_ptr,
                       const float* __restrict__ absmax_f32, const T16* __restrict__ bias, SkinnyOut<T16, kOutF16>* __restrict__ y,
                       int N, int K, const T16* __restrict__ lora_u, const T16* __restrict__ lora_v, int lora_r,
                       const float* __restrict__ row_scale) {
  skinny_1tok_body<T16, kWarps, kRing, kBuf, kNested, kStateF16, kOutF16, false>(x, packed, absmax_u8, code256, absmax2, offset_ptr,
                                                                               absmax_f32, bias, y, N, K, lora_u, lora_v, lora_r,
                                                                               row_scale, MixedLora{});
}

template <typename T16, int kWarps, int kRing, int kBuf, bool kNested, bool kStateF16, bool kOutF16>
__global__ void __launch_bounds__(32 * kWarps, 4)
nf4_skinny_kernel_1tok_mixed(const T16* __restrict__ x, const uint8_t* __restrict__ packed, const uint8_t* __restrict__ absmax_u8,
                             const float* __restrict__ code256, const float* __restrict__ absmax2, const float* __restrict__ offset_ptr,
                             const float* __restrict__ absmax_f32, const T16* __restrict__ bias,
                             SkinnyOut<T16, kOutF16>* __restrict__ y, int N, int K, const T16* __restrict__ lora_u, int lora_r,
                             MixedLora mix) {
  skinny_1tok_body<T16, kWarps, kRing, kBuf, kNested, kStateF16, kOutF16, true>(x, packed, absmax_u8, code256, absmax2, offset_ptr,
                                                                              absmax_f32, bias, y, N, K, lora_u, nullptr, lora_r,
                                                                              nullptr, mix);
}

// launch_cfg with one adapter per token (nf4_skinny_kernel_mixed); q.V is unused.
template <typename T16, bool kStateF16, bool kOutF16, int NT, int kWarps, int kRing>
static int launch_cfg_mixed(const qb200_nf4_problem& q, const MixedLora& mix, int M, int N, int K, int R, cudaStream_t stream) {
  constexpr int smem = kWarps * NT * 8 * kSlabRowBytes + 256 * int(sizeof(float));
  const auto kern = q.absmax_u8 != nullptr ? nf4_skinny_kernel_mixed<T16, NT, kWarps, kRing, true, kStateF16, kOutF16>
                                           : nf4_skinny_kernel_mixed<T16, NT, kWarps, kRing, false, kStateF16, kOutF16>;
  return launch_pdl(kern, unsigned(N / kRows), 32 * kWarps, smem, stream, "nf4_skinny_mixed", static_cast<const T16*>(q.in),
                    q.packed, q.absmax_u8, q.code256, q.absmax2, q.offset, q.absmax_f32, static_cast<const T16*>(q.bias),
                    static_cast<SkinnyOut<T16, kOutF16>*>(q.out), M, N, K, static_cast<const T16*>(q.U), int(q.ld_u), R, q.ld_in,
                    q.ld_out, mix);
}

// One token: row pitches do not matter.  State pointers as in launch_cfg.
template <typename T16, bool kStateF16, bool kOutF16, int kWarps, int kRing, int kBuf>
static int launch_1tok(const qb200_nf4_problem& q, const float* row_scale, int N, int K, int R, cudaStream_t stream) {
  constexpr int kSlabs = kWarps * kBuf * kSlabRowBytes;
  constexpr int kRed = (kWarps + 1) * kRows * int(sizeof(float));
  constexpr int smem = (kSlabs > kRed ? kSlabs : kRed) + 256 * int(sizeof(float));
  const auto kern = q.absmax_u8 != nullptr ? nf4_skinny_kernel_1tok<T16, kWarps, kRing, kBuf, true, kStateF16, kOutF16>
                                           : nf4_skinny_kernel_1tok<T16, kWarps, kRing, kBuf, false, kStateF16, kOutF16>;
  return launch_pdl(kern, unsigned(N / kRows), 32 * kWarps, smem, stream, "nf4_skinny_1tok", static_cast<const T16*>(q.in), q.packed,
                    q.absmax_u8, q.code256, q.absmax2, q.offset, q.absmax_f32, static_cast<const T16*>(q.bias),
                    static_cast<SkinnyOut<T16, kOutF16>*>(q.out), N, K, static_cast<const T16*>(q.U), static_cast<const T16*>(q.V), R,
                    row_scale);
}

// launch_1tok with the token's own adapter (nf4_skinny_kernel_1tok_mixed); q.V is unused.
template <typename T16, bool kStateF16, bool kOutF16, int kWarps, int kRing, int kBuf>
static int launch_1tok_mixed(const qb200_nf4_problem& q, const MixedLora& mix, int N, int K, int R, cudaStream_t stream) {
  constexpr int kSlabs = kWarps * kBuf * kSlabRowBytes;
  constexpr int kRed = (kWarps + 1) * kRows * int(sizeof(float));
  constexpr int smem = (kSlabs > kRed ? kSlabs : kRed) + 256 * int(sizeof(float));
  const auto kern = q.absmax_u8 != nullptr ? nf4_skinny_kernel_1tok_mixed<T16, kWarps, kRing, kBuf, true, kStateF16, kOutF16>
                                           : nf4_skinny_kernel_1tok_mixed<T16, kWarps, kRing, kBuf, false, kStateF16, kOutF16>;
  return launch_pdl(kern, unsigned(N / kRows), 32 * kWarps, smem, stream, "nf4_skinny_1tok_mixed", static_cast<const T16*>(q.in),
                    q.packed, q.absmax_u8, q.code256, q.absmax2, q.offset, q.absmax_f32, static_cast<const T16*>(q.bias),
                    static_cast<SkinnyOut<T16, kOutF16>*>(q.out), N, K, static_cast<const T16*>(q.U), R, mix);
}

// 16 tokens per launch (more tokens = more passes over the packed weights, which stay in L2); q's row pitches are resolved.
// mix.table != nullptr: one adapter per token (the mixed kernels, no row scale).
template <typename T16, bool kStateF16, bool kOutF16>
static int launch_chunks(qb200_nf4_problem q, const float* row_scale, MixedLora mix, int M, int N, int K, int R, cudaStream_t stream) {
  constexpr int kChunk = 8 * kMaxNT;
  for (int m0 = 0; m0 < M; m0 += kChunk) {
    const int mc = M - m0 < kChunk ? M - m0 : kChunk;
    int rc;
    if (mix.table != nullptr) {
      if (mc == 1)
        rc = launch_1tok_mixed<T16, kStateF16, kOutF16, 4, 4, 2>(q, mix, N, K, R, stream);
      else if (mc <= 8)
        rc = launch_cfg_mixed<T16, kStateF16, kOutF16, 1, 4, 4>(q, mix, mc, N, K, R, stream);
      else
        rc = launch_cfg_mixed<T16, kStateF16, kOutF16, 2, 4, 4>(q, mix, mc, N, K, R, stream);
      mix.rows += kChunk;
    } else if (mc == 1)
      rc = launch_1tok<T16, kStateF16, kOutF16, 4, 4, 2>(q, row_scale, N, K, R, stream);
    else if (mc <= 8)
      rc = launch_cfg<T16, kStateF16, kOutF16, 1, 4, 4>(q, row_scale, mc, N, K, R, stream);
    else
      rc = launch_cfg<T16, kStateF16, kOutF16, 2, 4, 4>(q, row_scale, mc, N, K, R, stream);
    if (rc) return rc;
    q.in = static_cast<const T16*>(q.in) + int64_t(kChunk) * q.ld_in;
    if (q.U) q.U = static_cast<const T16*>(q.U) + int64_t(kChunk) * q.ld_u;
    q.out = static_cast<SkinnyOut<T16, kOutF16>*>(q.out) + int64_t(kChunk) * q.ld_out;
  }
  return 0;
}

}  // namespace skinny

// Internal: forward skinny GEMM, 16 tokens per launch, with the skinny kernels of `kernels`; optional LoRA term
// y += U[M,R] . V[N,R]^T  (R = 0: none); optional row_scale[N] (null: none) multiplies row n of W; in / out / U may be column
// slices of wider row-major buffers (row pitches ld_in / ld_out / ld_u in elements, 0 = dense); caller has validated
// pointers/shapes (K % 64 == 0, N % 8 == 0, R % 8 == 0, R <= kMaxLoraRank = 256, 16-byte aligned in / U rows and V).
int launch_nf4_skinny(const qb200_nf4_problem& prob, const float* row_scale, int M, int N, int K, int R, Nf4Kernels kernels,
                      cudaStream_t stream) {
  if (M < 1) return set_error(QB200_EINVAL, "nf4_skinny: M must be positive");
  qb200_nf4_problem q = prob;   // advanced by one chunk of tokens per launch
  if (R == 0) q.U = q.V = nullptr;
  if (q.ld_u == 0) q.ld_u = R;
  if (q.ld_in == 0) q.ld_in = K;
  if (q.ld_out == 0) q.ld_out = N;
  return with_nf4_types(kernels, [&](auto t) {
    using Ty = decltype(t);
    return skinny::launch_chunks<typename Ty::T16, Ty::kStateF16, Ty::kOutF16>(q, row_scale, MixedLora{}, M, N, K, R, stream);
  });
}

int launch_nf4_skinny_mixed(const qb200_nf4_problem& prob, const int32_t* row_adapter, int n_adapters, int M, int N, int K, int R,
                            Nf4Kernels kernels, cudaStream_t stream) {
  if (M < 1) return set_error(QB200_EINVAL, "nf4_skinny: M must be positive");
  const MixedLora mix{row_adapter, static_cast<const qb200_lora_adapter*>(prob.V), n_adapters};
  qb200_nf4_problem q = prob;
  q.V = nullptr;
  if (q.ld_u == 0) q.ld_u = R;
  if (q.ld_in == 0) q.ld_in = K;
  if (q.ld_out == 0) q.ld_out = N;
  return with_nf4_types(kernels, [&](auto t) {
    using Ty = decltype(t);
    return skinny::launch_chunks<typename Ty::T16, Ty::kStateF16, Ty::kOutF16>(q, nullptr, mix, M, N, K, R, stream);
  });
}

}  // namespace qb200
