// Segmented LoRA for mixed-adapter batches of any token count (SGMV in Punica and S-LoRA): the rows of a batch are grouped by
// adapter on the device, and tensor-core kernels run one (segment tile x column tile) per CTA, each tile with its own
// adapter's weights read through the adapter table.  Nothing here reads device memory on the host, so a batch can be
// captured in a CUDA graph or traced by torch.compile and switched between requests by a copy into the row-index buffer.
//
//   lora_segment_table_kernel   one CTA: a stable counting sort of the M row indices into n + 1 buckets (one per adapter, the
//                               last for "no adapter"), giving the row permutation, the bucket offsets and a list of tiles
//                               (adapter, first sorted row, rows) of at most 64 rows, padded with empty tiles up to the
//                               host-known bound ceil(M / 64) + n.
//   lora_segmented_kernel       <kShrink = false> the expand: y_t = rn(y_t + U_t . B_a^T) in place on the base launch's 16-bit
//                               output, fp32 sum; rows without an adapter are not written.
//                               <kShrink = true> the shrink: U_t = rn(s_a . x_t . A_a^T), fp32 sum; columns at and beyond
//                               the adapter's rank are zero; rows without an adapter are not written.
//   lora_segmented_grad_kernel  the backward's G = rn(s_a . dY_p . B_a) and input-gradient term G_p . A_{p,a} (DESIGN.md §6d).
//   lora_weight_grad_kernel     dA_a = rn(G^T . x_lora) and dB_a = rn(dY^T . U) over each adapter's sorted rows.
// All are one warpgroup of wgmma m64n128k16 (bf16 or fp16 in, fp32 accumulate) per 64-row x 128-column tile, with the next
// 64-wide contraction chunk loaded into registers while the current one is multiplied.  grid.z is the problem of a
// grouped launch (q/k/v, gate/up): each problem has its own adapter table and U, and all share the segment table.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "nf4_gemm_common.cuh"
#include "nf4_table.cuh"
#include "qb200_internal.h"
#include "sm90_ptx.cuh"

namespace qb200 {
namespace seg {

constexpr int kTileM = 64;            // sorted rows per tile
constexpr int kTileN = 128;           // output columns per CTA
constexpr int kChunk = 64;            // contraction elements per shared-memory chunk
constexpr int kThreads = 128;         // one warpgroup
constexpr int kTableThreads = 1024;
// Buckets whose counts and tile offsets (8 bytes each) fit the 48 KB a launch may use without opting in, less 1 KB for the
// table kernel's static shared memory (272 bytes: the scan's warp sums and carries).
constexpr int kSmemBuckets = (48 * 1024 - 1024) / 8;
constexpr int kMaxProb = 3;

// The workspace of one segment table, every part 16-byte aligned: perm [M] int32, offsets [n + 2] int32 (bucket b holds sorted
// rows [off[b], off[b + 1]), off[n + 1] = M), tiles [ceil(M / kTileM) + n] int4 (adapter, first sorted row, rows, 0), and the
// global counts / tile offsets [2 (n + 1)] int32 used when n + 1 > kSmemBuckets.
struct Layout {
  int64_t perm, off, tiles, hist, bytes;
  int64_t n_tiles;
};
__host__ __device__ inline int64_t align16(int64_t b) { return (b + 15) & ~int64_t(15); }
__host__ __device__ inline Layout layout(int64_t M, int64_t n) {
  Layout L;
  L.n_tiles = (M + kTileM - 1) / kTileM + n;
  L.perm = 0;
  L.off = align16(4 * M);
  L.tiles = L.off + align16(4 * (n + 2));
  L.hist = L.tiles + 16 * L.n_tiles;
  L.bytes = L.hist + align16(8 * (n + 1));
  return L;
}

__device__ __forceinline__ int bucket(const int32_t* rows, int t, int n) {
  const int a = rows[t];
  return (a >= 0 && a < n) ? a : n;
}

template <bool kSmem>
__global__ void __launch_bounds__(kTableThreads) lora_segment_table_kernel(const int32_t* __restrict__ rows, int M, int n,
                                                                          uint8_t* __restrict__ ws) {
  extern __shared__ int s_dyn[];
  __shared__ int s_wsum[2][32];
  __shared__ int s_carry[2];
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();                              // the row indices may be the previous kernel's output
  const Layout L = layout(M, n);
  int* perm = reinterpret_cast<int*>(ws + L.perm);
  int* off = reinterpret_cast<int*>(ws + L.off);
  int4* tiles = reinterpret_cast<int4*>(ws + L.tiles);
  const int nb = n + 1;
  int* cnt = kSmem ? s_dyn : reinterpret_cast<int*>(ws + L.hist);   // counts, then bucket offsets, then scatter cursors
  int* toff = cnt + nb;                                              // tile offsets
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < nb; i += kTableThreads) cnt[i] = 0;
  if (tid < 2) s_carry[tid] = 0;
  __syncthreads();
  for (int t = tid; t < M; t += kTableThreads) atomicAdd(&cnt[bucket(rows, t, n)], 1);
  __syncthreads();
  // exclusive scan of (rows, tiles) over the buckets, 1024 at a time; the "no adapter" bucket has no tiles
  for (int c0 = 0; c0 < nb; c0 += kTableThreads) {
    const int i = c0 + tid;
    const int v = i < nb ? cnt[i] : 0;
    const int w = i < n ? (v + kTileM - 1) / kTileM : 0;
    int iv = v, iw = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, iv, o), b = __shfl_up_sync(0xffffffffu, iw, o);
      if (lane >= o) iv += a, iw += b;
    }
    if (lane == 31) s_wsum[0][warp] = iv, s_wsum[1][warp] = iw;
    __syncthreads();
    if (warp == 0) {
      int sv = s_wsum[0][lane], sw = s_wsum[1][lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, sv, o), b = __shfl_up_sync(0xffffffffu, sw, o);
        if (lane >= o) sv += a, sw += b;
      }
      s_wsum[0][lane] = sv - s_wsum[0][lane];
      s_wsum[1][lane] = sw - s_wsum[1][lane];
    }
    __syncthreads();
    const int ev = s_carry[0] + s_wsum[0][warp] + iv - v, ew = s_carry[1] + s_wsum[1][warp] + iw - w;
    if (i < nb) cnt[i] = ev, toff[i] = ew, off[i] = ev;
    __syncthreads();
    if (tid == kTableThreads - 1) s_carry[0] = ev + v, s_carry[1] = ew + w;
    __syncthreads();
  }
  if (tid == 0) off[nb] = M;
  const int used = s_carry[1];
  for (int a = tid; a < n; a += kTableThreads) {
    const int first = cnt[a], rows_a = (a + 1 < nb ? cnt[a + 1] : M) - first;
    for (int j = 0; j * kTileM < rows_a; ++j)
      tiles[toff[a] + j] = make_int4(a, first + j * kTileM, min(kTileM, rows_a - j * kTileM), 0);
  }
  for (int64_t j = used + tid; j < L.n_tiles; j += kTableThreads) tiles[j] = make_int4(0, 0, 0, 0);
  __syncthreads();
  // stable scatter by one warp, 32 rows at a time in row order; each group of equal buckets takes its slots from the cursor
  if (warp == 0) {
    int b_next = lane < M ? bucket(rows, lane, n) : -1;
    for (int base = 0; base < M; base += 32) {
      const int t = base + lane, b = b_next;
      b_next = t + 32 < M ? bucket(rows, t + 32, n) : -1;
      const unsigned peers = __match_any_sync(0xffffffffu, b);
      const int leader = __ffs(peers) - 1;
      int pos = 0;
      if (lane == leader && b >= 0) {
        pos = cnt[b];
        cnt[b] = pos + __popc(peers);
      }
      pos = __shfl_sync(0xffffffffu, pos, leader);
      if (b >= 0) perm[pos + __popc(peers & ((1u << lane) - 1u))] = t;
      __syncwarp();
    }
  }
}

// The operands of one launch, per problem: the adapter table, the gathered operand X (expand: U [M, R]; shrink: the shared x
// [M, K]) and the output (expand: y [M, N], updated in place; shrink: U [M, R]).
struct Problems {
  const qb200_lora_adapter* table[kMaxProb];
  const void* X[kMaxProb];
  void* out[kMaxProb];
};

// element z of a kernel-parameter array, without copying the array to local memory as a dynamic index would
template <typename T>
__device__ __forceinline__ T pick(const T (&v)[kMaxProb], int z) {
  return z == 0 ? v[0] : (z == 1 ? v[1] : v[2]);
}

// C[tile rows, column tile] = X[perm rows, :len] . Op[columns, :len]^T with, per tile of adapter a (rank r_a, clamped to the
// R columns of U and down to a multiple of 8 as in MixedLora::rank):
//   expand: len = r_a, Op = B_a [N, r_a] (row pitch: the entry's rank), out y += C, columns [0, N);
//   shrink: len = K, Op = A_a [r_a, K], out U = s_a . C for columns < r_a and 0 for [r_a, R).
// One warpgroup: per 64-wide chunk of the contraction, the gathered X rows [64 x 64] and the Op rows [128 x 64] are stored
// K-major with the 128-byte swizzle and contracted by four m64n128k16 wgmma; elements at and beyond len are loaded as zero,
// so every chunk runs all four and no data-dependent branch sits between them.
// Every row index comes from the segment table and is checked against [0, M); an adapter index outside [0, n), an entry whose
// rank is not a positive multiple of 8, or (expand) a clamped rank of 0 makes the tile write nothing.
template <typename T16, bool kShrink>
__global__ void __launch_bounds__(kThreads) lora_segmented_kernel(Problems p, const uint8_t* __restrict__ ws, int64_t ld_x,
                                                                  int64_t ld_out, int M, int n, int N, int K, int R) {
  __shared__ __align__(1024) uint4 sX[kTileM * kChunk / 8];
  __shared__ __align__(1024) uint4 sO[kTileN * kChunk / 8];
  __shared__ int s_row[kTileM];
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();                              // the segment table, U and y are earlier kernels' outputs
  const Layout L = layout(M, n);
  const int z = blockIdx.z;
  const int4 tile = reinterpret_cast<const int4*>(ws + L.tiles)[blockIdx.x];
  const int a = tile.x, rows_t = min(tile.z, kTileM);
  if (rows_t <= 0 || a < 0 || a >= n) return;
  const qb200_lora_adapter ad = pick(p.table, z)[a];
  if (ad.rank <= 0 || (ad.rank & 7)) return;
  const int rank = MixedLora::rank(ad, R);
  const int n0 = blockIdx.y * kTileN;
  const int len = kShrink ? K : rank;
  const int cols = kShrink ? rank : N;               // rows of Op that exist; the others are loaded as zero
  if (rank == 0 || n0 >= (kShrink ? R : N)) return;
  const T16* X = static_cast<const T16*>(pick(p.X, z));
  const T16* op = static_cast<const T16*>(kShrink ? ad.A : ad.B);
  const int64_t ld_op = kShrink ? K : ad.rank;
  const int tid = threadIdx.x;
  if (tid < kTileM) {
    const int* perm = reinterpret_cast<const int*>(ws + L.perm);
    const int first = tile.y;
    int t = -1;
    if (tid < rows_t && first >= 0 && first + tid < M) t = perm[first + tid];
    s_row[tid] = (t >= 0 && t < M) ? t : -1;
  }
  __syncthreads();
  T16* out = static_cast<T16*>(pick(p.out, z));
  if (kShrink && n0 >= rank) {                       // U columns [n0, n0 + 128) of this tile lie beyond the rank: zeros
    for (int v = tid; v < kTileM * kTileN / 2; v += kThreads) {
      const int r = v / (kTileN / 2), c = n0 + 2 * (v % (kTileN / 2)), t = s_row[r];
      if (t >= 0 && c < R) *reinterpret_cast<uint32_t*>(out + int64_t(t) * ld_out + c) = 0u;
    }
    return;
  }

  // 16-byte vector v of a chunk: row v / 8, K offset 8 (v % 8); stored at row 128 B apart, 16-byte unit (v % 8) ^ (row % 8)
  constexpr int kXv = kTileM * kChunk / 8 / kThreads, kOv = kTileN * kChunk / 8 / kThreads;
  uint4 rx[kXv], ro[kOv];
  auto load = [&](int k0) {
#pragma unroll
    for (int i = 0; i < kXv; ++i) {
      const int v = tid + i * kThreads, r = v >> 3, k = k0 + (v & 7) * 8, t = s_row[r];
      rx[i] = (t >= 0 && k < len) ? *reinterpret_cast<const uint4*>(X + int64_t(t) * ld_x + k) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int i = 0; i < kOv; ++i) {
      const int v = tid + i * kThreads, c = n0 + (v >> 3), k = k0 + (v & 7) * 8;
      ro[i] = (c < cols && k < len) ? __ldg(reinterpret_cast<const uint4*>(op + int64_t(c) * ld_op + k)) : make_uint4(0, 0, 0, 0);
    }
  };
  auto swz = [](int v) { return (v & ~7) | ((v ^ (v >> 3)) & 7); };

  float acc[ptx::kWgmmaMaxAcc];
#pragma unroll
  for (int i = 0; i < ptx::kWgmmaMaxAcc; ++i) acc[i] = 0.0f;
  const uint64_t x_desc = gemm::make_desc_kmajor_sw128(ptx::smem_u32(sX));
  const uint64_t o_desc = gemm::make_desc_kmajor_sw128(ptx::smem_u32(sO));
  load(0);
  for (int k0 = 0; k0 < len; k0 += kChunk) {
#pragma unroll
    for (int i = 0; i < kXv; ++i) sX[swz(tid + i * kThreads)] = rx[i];
#pragma unroll
    for (int i = 0; i < kOv; ++i) sO[swz(tid + i * kThreads)] = ro[i];
    ptx::fence_proxy_async_smem();                   // the stores above are read by wgmma through the async proxy
    __syncthreads();
    if (k0 + kChunk < len) load(k0 + kChunk);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < kChunk / 16; ++k) {
      const uint64_t adv = uint64_t((k * 16 * 2) >> 4);
      ptx::wgmma<T16, kTileN, 0>(acc, x_desc + adv, o_desc + adv, 1u);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>(acc);
    __syncthreads();
  }

  // accumulator 4 j + 2 h + {0, 1}: row 16 warp + lane / 4 + 8 h, columns n0 + 8 j + 2 (lane % 4) + {0, 1}
  using T2 = typename Vec2<T16>::type;
  const int warp = tid >> 5, lane = tid & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = s_row[16 * warp + (lane >> 2) + 8 * h];
    if (t < 0) continue;
#pragma unroll
    for (int j = 0; j < kTileN / 8; ++j) {
      const int c = n0 + 8 * j + 2 * (lane & 3);
      if (c >= (kShrink ? R : N)) continue;
      uint32_t* dst = reinterpret_cast<uint32_t*>(out + int64_t(t) * ld_out + c);
      const float s0 = acc[4 * j + 2 * h], s1 = acc[4 * j + 2 * h + 1];
      if constexpr (kShrink) {
        *dst = c < rank ? round16x2<T16>(s0 * ad.scale, s1 * ad.scale) : 0u;
      } else {
        uint32_t y = *dst;
        const float2 f = widen2(*reinterpret_cast<const T2*>(&y));
        *dst = round16x2<T16>(f.x + s0, f.y + s1);
      }
    }
  }
}

// ---- backward -----------------------------------------------------------------------------------------------------------
// The operands the backward contracts are stored MN-major in memory (B_a [N, r_a] contracted over N, A_a [r_a, K] over r_a,
// and every operand of a weight gradient over the token rows).  They are gathered here into the same K-major 128-byte
// swizzled shared-memory layout the forward kernels use: each thread assembles one 16-byte vector from 8 elements along the
// contraction, with consecutive threads on consecutive MN indices so each of the 8 loads is coalesced across the warp.
template <int kRows>
__device__ __forceinline__ int swz_t(int v) {     // vector v = (MN index v % kRows, contraction group v / kRows)
  const int r = v % kRows, g = v / kRows;
  return r * 8 + (g ^ (r & 7));
}

__device__ __forceinline__ uint4 pack8(const uint16_t (&h)[8]) {
  return make_uint4(h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16), h[4] | (uint32_t(h[5]) << 16),
                    h[6] | (uint32_t(h[7]) << 16));
}

// Per tile of adapter a (rank r_a clamped as in lora_segmented_kernel), C[tile rows, column tile] = X[perm rows, :len] .
// Op[columns, :len]^T where Op is read MN-major:
//   kInput = false, the G shrink: len = N, X = dY_p [M, N], Op[c, k] = B_a[k, c] (c < r_a), out G_p = s_a . C for columns
//     < r_a and 0 for [r_a, R); grid.z is the problem.
//   kInput = true, the input-gradient term: len = r_a of problem p, X = G_p [M, R], Op[c, k] = A_{p,a}[k, c] (c < K);
//     kSum: out_0 = rn(out_0 + sum_p C_p) in place, every problem summed in the accumulators before the one rounding (q/k/v
//     share one dX, so a problem per CTA would race); !kSum: out_p = rn(C_p), grid.z the problem (the dropped inputs).
// Rows without an adapter, and tiles whose entries are not usable (index outside [0, n), a rank that is not a positive
// multiple of 8), are not written.
template <typename T16, bool kInput, bool kSum>
__global__ void __launch_bounds__(kThreads) lora_segmented_grad_kernel(Problems p, int nprob, const uint8_t* __restrict__ ws,
                                                                       int64_t ld_x, int64_t ld_out, int M, int n, int C, int R) {
  __shared__ __align__(1024) uint4 sX[kTileM * kChunk / 8];
  __shared__ __align__(1024) uint4 sO[kTileN * kChunk / 8];
  __shared__ int s_row[kTileM];
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();                              // the segment table, dY / G and the output are earlier kernels' outputs
  const Layout L = layout(M, n);
  const int4 tile = reinterpret_cast<const int4*>(ws + L.tiles)[blockIdx.x];
  const int a = tile.x, rows_t = min(tile.z, kTileM);
  if (rows_t <= 0 || a < 0 || a >= n) return;
  const int n0 = blockIdx.y * kTileN;
  const int out_cols = kInput ? C : R;
  if (n0 >= out_cols) return;
  const int tid = threadIdx.x;
  if (tid < kTileM) {
    const int* perm = reinterpret_cast<const int*>(ws + L.perm);
    const int first = tile.y;
    int t = -1;
    if (tid < rows_t && first >= 0 && first + tid < M) t = perm[first + tid];
    s_row[tid] = (t >= 0 && t < M) ? t : -1;
  }
  __syncthreads();

  constexpr int kXv = kTileM * kChunk / 8 / kThreads, kOv = kTileN * kChunk / 8 / kThreads;
  uint4 rx[kXv], ro[kOv];
  auto swz = [](int v) { return (v & ~7) | ((v ^ (v >> 3)) & 7); };
  float acc[ptx::kWgmmaMaxAcc];
#pragma unroll
  for (int i = 0; i < ptx::kWgmmaMaxAcc; ++i) acc[i] = 0.0f;
  const uint64_t x_desc = gemm::make_desc_kmajor_sw128(ptx::smem_u32(sX));
  const uint64_t o_desc = gemm::make_desc_kmajor_sw128(ptx::smem_u32(sO));
  const int z0 = kSum ? 0 : int(blockIdx.z), z1 = kSum ? nprob : int(blockIdx.z) + 1;
  float scale = 0.0f;
  int rank_g = -1;                                   // G: the rank of this tile's adapter, -1 while unusable
  bool any = false;
  for (int z = z0; z < z1; ++z) {
    const qb200_lora_adapter ad = pick(p.table, z)[a];
    if (ad.rank <= 0 || (ad.rank & 7)) continue;
    const int rank = MixedLora::rank(ad, R);
    if (!kInput) rank_g = rank, scale = ad.scale;
    if (rank == 0 || (!kInput && n0 >= rank)) continue;
    any = true;
    const int len = kInput ? rank : C, cols = kInput ? C : rank;
    const T16* X = static_cast<const T16*>(pick(p.X, z));
    const uint16_t* op = static_cast<const uint16_t*>(kInput ? ad.A : ad.B);
    const int64_t ld_op = kInput ? int64_t(C) : int64_t(ad.rank);
    auto load = [&](int k0) {
#pragma unroll
      for (int i = 0; i < kXv; ++i) {
        const int v = tid + i * kThreads, r = v >> 3, k = k0 + (v & 7) * 8, t = s_row[r];
        rx[i] = (t >= 0 && k < len) ? *reinterpret_cast<const uint4*>(X + int64_t(t) * ld_x + k) : make_uint4(0, 0, 0, 0);
      }
      // opaque per chunk: otherwise the 64 element addresses are hoisted out of the chunk loop and the kernel spills
      const uint16_t* opk = op + int64_t(k0) * ld_op;
      int64_t ld = ld_op;
      asm volatile("" : "+l"(opk), "+l"(ld));
#pragma unroll
      for (int i = 0; i < kOv; ++i) {
        const int v = tid + i * kThreads, c = n0 + v % kTileN, g = (v / kTileN) * 8;
        uint16_t h[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) h[e] = (c < cols && k0 + g + e < len) ? __ldg(opk + (g + e) * ld + c) : uint16_t(0);
        ro[i] = pack8(h);
      }
    };
    load(0);
    for (int k0 = 0; k0 < len; k0 += kChunk) {
#pragma unroll
      for (int i = 0; i < kXv; ++i) sX[swz(tid + i * kThreads)] = rx[i];
#pragma unroll
      for (int i = 0; i < kOv; ++i) sO[swz_t<kTileN>(tid + i * kThreads)] = ro[i];
      ptx::fence_proxy_async_smem();
      __syncthreads();
      if (k0 + kChunk < len) load(k0 + kChunk);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < kChunk / 16; ++k) {
        const uint64_t adv = uint64_t((k * 16 * 2) >> 4);
        ptx::wgmma<T16, kTileN, 0>(acc, x_desc + adv, o_desc + adv, 1u);
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>(acc);
      __syncthreads();
    }
  }
  if (kInput ? !any : rank_g <= 0) return;

  using T2 = typename Vec2<T16>::type;
  const int warp = tid >> 5, lane = tid & 31;
  T16* out = static_cast<T16*>(pick(p.out, kSum ? 0 : int(blockIdx.z)));
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = s_row[16 * warp + (lane >> 2) + 8 * h];
    if (t < 0) continue;
#pragma unroll
    for (int j = 0; j < kTileN / 8; ++j) {
      const int c = n0 + 8 * j + 2 * (lane & 3);
      if (c >= out_cols) continue;
      uint32_t* dst = reinterpret_cast<uint32_t*>(out + int64_t(t) * ld_out + c);
      const float s0 = acc[4 * j + 2 * h], s1 = acc[4 * j + 2 * h + 1];
      if constexpr (!kInput) {
        *dst = c < rank_g ? round16x2<T16>(s0 * scale, s1 * scale) : 0u;
      } else if constexpr (kSum) {
        uint32_t y = *dst;
        const float2 f = widen2(*reinterpret_cast<const T2*>(&y));
        *dst = round16x2<T16>(f.x + s0, f.y + s1);
      } else {
        *dst = round16x2<T16>(s0, s1);
      }
    }
  }
}

// The operands of a weight-gradient launch, per problem: the adapter table, P [M, R] (G or U), Q [M, D] (the adapters'
// input or dY) and the flat output.
struct WgradProblems {
  const qb200_lora_adapter* table[kMaxProb];
  const void* P[kMaxProb];
  const void* Q[kMaxProb];
  void* out[kMaxProb];
};

// Segmented weight gradient: for adapter a with rank r_a and rank offset o_a = rank_off[a], over the sorted rows t of its
// bucket, D_a[i, j] = rn(sum_t P[t, i] . Q[t, j]) for i < r_a, j < D, written to the flat output at o_a . D:
//   !kTransOut: [r_a, D] row-major (dA_a = G^T . x_lora: P = G, Q = x_lora, D = K);
//   kTransOut:  [D, r_a] row-major (dB_a = dY^T . U: P = U, Q = dY, D = N).
// One CTA per (adapter, 64 ranks, 128 columns, problem) contracts 64 rows per step in a fixed order; an adapter without rows
// writes zeros.  A rank offset with o_a < 0 or o_a + r_a > total writes nothing, so no device value leads outside the
// output's total . D elements; row indices are checked against [0, M) and the bucket offsets clamped to it.
template <typename T16, bool kTransOut>
__global__ void __launch_bounds__(kThreads) lora_weight_grad_kernel(WgradProblems p, const int64_t* __restrict__ rank_off,
                                                                    int64_t total, const uint8_t* __restrict__ ws, int64_t ld_p,
                                                                    int64_t ld_q, int M, int n, int D, int R) {
  __shared__ __align__(1024) uint4 sP[kTileM * kChunk / 8];
  __shared__ __align__(1024) uint4 sQ[kTileN * kChunk / 8];
  __shared__ int s_row[2][kChunk];
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();                              // the segment table and the operands are earlier kernels' outputs
  const int rt = (R + kTileM - 1) / kTileM;
  const int a = int(blockIdx.x / unsigned(rt)), i0 = int(blockIdx.x % unsigned(rt)) * kTileM;
  const int j0 = blockIdx.y * kTileN, z = blockIdx.z;
  if (a >= n || j0 >= D) return;
  const qb200_lora_adapter ad = pick(p.table, z)[a];
  if (ad.rank <= 0 || (ad.rank & 7)) return;
  const int rank = MixedLora::rank(ad, R);
  if (i0 >= rank) return;
  const int64_t off = rank_off[a];
  if (off < 0 || off > total - rank) return;
  const Layout L = layout(M, n);
  const int* perm = reinterpret_cast<const int*>(ws + L.perm);
  const int* boff = reinterpret_cast<const int*>(ws + L.off);
  const int b0 = max(0, min(boff[a], M)), b1 = max(b0, min(boff[a + 1], M));
  const uint16_t* P = static_cast<const uint16_t*>(pick(p.P, z));
  const uint16_t* Q = static_cast<const uint16_t*>(pick(p.Q, z));
  const int tid = threadIdx.x;
  auto rows = [&](int buf, int c0) {
    if (tid < kChunk) {
      int t = -1;
      if (c0 + tid < b1) t = perm[c0 + tid];
      s_row[buf][tid] = (t >= 0 && t < M) ? t : -1;
    }
  };
  constexpr int kPv = kTileM * kChunk / 8 / kThreads, kQv = kTileN * kChunk / 8 / kThreads;
  uint4 rp[kPv], rq[kQv];
  auto load = [&](int buf) {
#pragma unroll
    for (int i = 0; i < kPv; ++i) {
      const int v = tid + i * kThreads, c = i0 + v % kTileM, g = (v / kTileM) * 8;
      uint16_t h[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int t = s_row[buf][g + e];
        h[e] = (t >= 0 && c < rank) ? P[int64_t(t) * ld_p + c] : uint16_t(0);
      }
      rp[i] = pack8(h);
    }
#pragma unroll
    for (int i = 0; i < kQv; ++i) {
      const int v = tid + i * kThreads, c = j0 + v % kTileN, g = (v / kTileN) * 8;
      uint16_t h[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int t = s_row[buf][g + e];
        h[e] = (t >= 0 && c < D) ? Q[int64_t(t) * ld_q + c] : uint16_t(0);
      }
      rq[i] = pack8(h);
    }
  };

  float acc[ptx::kWgmmaMaxAcc];
#pragma unroll
  for (int i = 0; i < ptx::kWgmmaMaxAcc; ++i) acc[i] = 0.0f;
  const uint64_t p_desc = gemm::make_desc_kmajor_sw128(ptx::smem_u32(sP));
  const uint64_t q_desc = gemm::make_desc_kmajor_sw128(ptx::smem_u32(sQ));
  rows(0, b0);
  __syncthreads();
  if (b0 < b1) load(0);
  for (int c0 = b0, it = 0; c0 < b1; c0 += kChunk, ++it) {
#pragma unroll
    for (int i = 0; i < kPv; ++i) sP[swz_t<kTileM>(tid + i * kThreads)] = rp[i];
#pragma unroll
    for (int i = 0; i < kQv; ++i) sQ[swz_t<kTileN>(tid + i * kThreads)] = rq[i];
    ptx::fence_proxy_async_smem();
    if (c0 + kChunk < b1) rows((it + 1) & 1, c0 + kChunk);
    __syncthreads();
    if (c0 + kChunk < b1) load((it + 1) & 1);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < kChunk / 16; ++k) {
      const uint64_t adv = uint64_t((k * 16 * 2) >> 4);
      ptx::wgmma<T16, kTileN, 0>(acc, p_desc + adv, q_desc + adv, 1u);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>(acc);
    __syncthreads();
  }

  // accumulator 4 j + 2 h + {0, 1}: rank i0 + 16 warp + lane / 4 + 8 h, columns j0 + 8 j + 2 (lane % 4) + {0, 1}
  T16* out = static_cast<T16*>(pick(p.out, z)) + off * int64_t(D);
  const int warp = tid >> 5, lane = tid & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int i = i0 + 16 * warp + (lane >> 2) + 8 * h;
    if (i >= rank) continue;
#pragma unroll
    for (int j = 0; j < kTileN / 8; ++j) {
      const int c = j0 + 8 * j + 2 * (lane & 3);
      if (c >= D) continue;
      const uint32_t v = round16x2<T16>(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      if constexpr (kTransOut) {
        uint16_t* o = reinterpret_cast<uint16_t*>(out);
        o[int64_t(c) * rank + i] = uint16_t(v & 0xFFFFu);
        o[int64_t(c + 1) * rank + i] = uint16_t(v >> 16);
      } else {
        *reinterpret_cast<uint32_t*>(out + int64_t(i) * D + c) = v;
      }
    }
  }
}

}  // namespace seg
}  // namespace qb200

using namespace qb200;

extern "C" int64_t qb200_lora_segment_workspace_size(int64_t M, int n_adapters) {
  if (M < 1 || M > INT32_MAX || n_adapters < 1) return 0;
  const seg::Layout L = seg::layout(M, n_adapters);
  return L.n_tiles > INT32_MAX ? 0 : L.bytes;
}

extern "C" int qb200_lora_segment_table(const int32_t* row_adapter, int64_t M, int n_adapters, void* workspace,
                                        int64_t workspace_bytes, void* stream) {
  if (!row_adapter || !workspace) return set_error(QB200_EINVAL, "lora_segment_table: null pointer");
  if (n_adapters < 1) return set_error(QB200_EINVAL, "lora_segment_table: n_adapters must be positive");
  if (M < 1 || M > INT32_MAX) return set_error(QB200_EINVAL, "lora_segment_table: bad shape");
  const int64_t need = qb200_lora_segment_workspace_size(M, n_adapters);
  if (need == 0) return set_error(QB200_EUNSUPPORTED, "lora_segment_table: more tiles than a grid can hold");
  if (workspace_bytes < need) return set_error(QB200_EINVAL, "lora_segment_table: workspace smaller than qb200_lora_segment_workspace_size");
  if (reinterpret_cast<uintptr_t>(workspace) % 16 || reinterpret_cast<uintptr_t>(row_adapter) % 4)
    return set_error(QB200_EINVAL, "lora_segment_table: the workspace must be 16-byte and row_adapter 4-byte aligned");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool smem = n_adapters + 1 <= seg::kSmemBuckets;
  const size_t bytes = smem ? size_t(2) * (n_adapters + 1) * sizeof(int) : 0;
  const auto kern = smem ? seg::lora_segment_table_kernel<true> : seg::lora_segment_table_kernel<false>;
  return launch_pdl(kern, 1, seg::kTableThreads, bytes, s, "lora_segment_table", row_adapter, int(M), n_adapters,
                    static_cast<uint8_t*>(workspace));
}

// The checks shared by the shrink and the expand; fills `p` from the host arrays.
static int segmented_args(const char* what, int dtype, int nprob, const qb200_lora_adapter* const* tables, const void* const* X,
                          void* const* out, int n_adapters, const void* workspace, int64_t workspace_bytes, int64_t M,
                          int64_t R, seg::Problems& p) {
  char msg[160];
  if (dtype != QB200_DTYPE_BF16 && dtype != QB200_DTYPE_F16) {
    snprintf(msg, sizeof(msg), "%s: dtype must be 2 (bf16) or 1 (fp16)", what);
    return set_error(QB200_EINVAL, msg);
  }
  if (nprob < 1 || nprob > seg::kMaxProb || !tables || !X || !out || !workspace) {
    snprintf(msg, sizeof(msg), "%s: 1..3 problems and no null pointer", what);
    return set_error(QB200_EINVAL, msg);
  }
  if (n_adapters < 1) {
    snprintf(msg, sizeof(msg), "%s: n_adapters must be positive", what);
    return set_error(QB200_EINVAL, msg);
  }
  if (R < 8 || R > kMaxLoraRank || R % 8 != 0) {
    snprintf(msg, sizeof(msg), "%s: R must be a multiple of 8 in [8, 256]", what);
    return set_error(QB200_EUNSUPPORTED, msg);
  }
  const int64_t need = qb200_lora_segment_workspace_size(M, n_adapters);
  if (M < 1 || M > INT32_MAX || need == 0) {
    snprintf(msg, sizeof(msg), "%s: bad shape", what);
    return set_error(QB200_EINVAL, msg);
  }
  if (workspace_bytes < need || reinterpret_cast<uintptr_t>(workspace) % 16) {
    snprintf(msg, sizeof(msg), "%s: the workspace must be 16-byte aligned and hold qb200_lora_segment_workspace_size bytes", what);
    return set_error(QB200_EINVAL, msg);
  }
  for (int i = 0; i < nprob; ++i) {
    if (!tables[i] || !X[i] || !out[i]) {
      snprintf(msg, sizeof(msg), "%s: null pointer", what);
      return set_error(QB200_EINVAL, msg);
    }
    if (reinterpret_cast<uintptr_t>(tables[i]) % 8 || reinterpret_cast<uintptr_t>(X[i]) % 16 || reinterpret_cast<uintptr_t>(out[i]) % 4) {
      snprintf(msg, sizeof(msg), "%s: tables must be 8-byte, inputs 16-byte and outputs 4-byte aligned", what);
      return set_error(QB200_EINVAL, msg);
    }
    p.table[i] = tables[i];
    p.X[i] = X[i];
    p.out[i] = out[i];
  }
  return 0;
}

template <bool kShrink>
static int launch_segmented(int dtype, int nprob, const seg::Problems& p, const void* workspace, int64_t ld_x, int64_t ld_out,
                            int M, int n, int N, int K, int R, cudaStream_t s) {
  const dim3 grid(unsigned(seg::layout(M, n).n_tiles), unsigned(((kShrink ? R : N) + seg::kTileN - 1) / seg::kTileN), unsigned(nprob));
  const char* what = kShrink ? "lora_shrink_segmented" : "lora_expand_segmented";
  const auto* ws = static_cast<const uint8_t*>(workspace);
  if (dtype == QB200_DTYPE_F16)
    return launch_pdl(seg::lora_segmented_kernel<__half, kShrink>, grid, seg::kThreads, 0, s, what, p, ws, ld_x, ld_out, M, n, N, K, R);
  return launch_pdl(seg::lora_segmented_kernel<__nv_bfloat16, kShrink>, grid, seg::kThreads, 0, s, what, p, ws, ld_x, ld_out, M, n,
                    N, K, R);
}

extern "C" int qb200_lora_shrink_segmented(int dtype, int nprob, const void* x, int64_t ld_x, const qb200_lora_adapter* const* tables,
                                           void* const* U, int64_t ld_u, int n_adapters, const void* workspace,
                                           int64_t workspace_bytes, int64_t M, int64_t K, int64_t R, void* stream) {
  const void* xs[seg::kMaxProb] = {x, x, x};
  seg::Problems p{};
  int rc = segmented_args("lora_shrink_segmented", dtype, nprob, tables, xs, U, n_adapters, workspace, workspace_bytes, M, R, p);
  if (rc) return rc;
  if (K < 8 || K % 8 != 0 || K > INT32_MAX) return set_error(QB200_EINVAL, "lora_shrink_segmented: bad shape");
  if (ld_x == 0) ld_x = K;
  if (ld_u == 0) ld_u = R;
  if (ld_x < K || ld_x % 8 != 0 || ld_u < R || ld_u % 2 != 0) return set_error(QB200_EINVAL, "lora_shrink_segmented: bad row pitch");
  return launch_segmented<true>(dtype, nprob, p, workspace, ld_x, ld_u, int(M), n_adapters, 0, int(K), int(R),
                                static_cast<cudaStream_t>(stream));
}

extern "C" int qb200_lora_expand_segmented(int dtype, int nprob, const qb200_lora_adapter* const* tables, const void* const* U,
                                           int64_t ld_u, void* const* out, int64_t ld_out, int n_adapters, const void* workspace,
                                           int64_t workspace_bytes, int64_t M, int64_t N, int64_t R, void* stream) {
  seg::Problems p{};
  int rc = segmented_args("lora_expand_segmented", dtype, nprob, tables, U, out, n_adapters, workspace, workspace_bytes, M, R, p);
  if (rc) return rc;
  if (N < 8 || N % 8 != 0 || N > INT32_MAX || int64_t(N + seg::kTileN - 1) / seg::kTileN > 65535)
    return set_error(QB200_EINVAL, "lora_expand_segmented: bad shape");
  if (ld_u == 0) ld_u = R;
  if (ld_out == 0) ld_out = N;
  if (ld_u < R || ld_u % 8 != 0 || ld_out < N || ld_out % 2 != 0)
    return set_error(QB200_EINVAL, "lora_expand_segmented: bad row pitch");
  return launch_segmented<false>(dtype, nprob, p, workspace, ld_u, ld_out, int(M), n_adapters, int(N), 0, int(R),
                                 static_cast<cudaStream_t>(stream));
}

extern "C" int qb200_lora_grad_shrink_segmented(int dtype, int nprob, const void* const* dY, int64_t ld_dy,
                                                const qb200_lora_adapter* const* tables, void* const* G, int64_t ld_g,
                                                int n_adapters, const void* workspace, int64_t workspace_bytes, int64_t M,
                                                int64_t N, int64_t R, void* stream) {
  seg::Problems p{};
  int rc = segmented_args("lora_grad_shrink_segmented", dtype, nprob, tables, dY, G, n_adapters, workspace, workspace_bytes, M, R,
                          p);
  if (rc) return rc;
  if (N < 8 || N % 8 != 0 || N > INT32_MAX) return set_error(QB200_EINVAL, "lora_grad_shrink_segmented: bad shape");
  if (ld_dy == 0) ld_dy = N;
  if (ld_g == 0) ld_g = R;
  if (ld_dy < N || ld_dy % 8 != 0 || ld_g < R || ld_g % 2 != 0)
    return set_error(QB200_EINVAL, "lora_grad_shrink_segmented: bad row pitch");
  const int n = n_adapters;
  const dim3 grid(unsigned(seg::layout(M, n).n_tiles), unsigned((R + seg::kTileN - 1) / seg::kTileN), unsigned(nprob));
  const auto* ws = static_cast<const uint8_t*>(workspace);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const char* what = "lora_grad_shrink_segmented";
  if (dtype == QB200_DTYPE_F16)
    return launch_pdl(seg::lora_segmented_grad_kernel<__half, false, false>, grid, seg::kThreads, 0, s, what, p, nprob, ws, ld_dy,
                      ld_g, int(M), n, int(N), int(R));
  return launch_pdl(seg::lora_segmented_grad_kernel<__nv_bfloat16, false, false>, grid, seg::kThreads, 0, s, what, p, nprob, ws,
                    ld_dy, ld_g, int(M), n, int(N), int(R));
}

extern "C" int qb200_lora_grad_input_segmented(int dtype, int nprob, int accumulate, const qb200_lora_adapter* const* tables,
                                               const void* const* G, int64_t ld_g, void* const* dx, int64_t ld_dx, int n_adapters,
                                               const void* workspace, int64_t workspace_bytes, int64_t M, int64_t K, int64_t R,
                                               void* stream) {
  if (accumulate != 0 && accumulate != 1) return set_error(QB200_EINVAL, "lora_grad_input_segmented: accumulate must be 0 or 1");
  void* one[seg::kMaxProb] = {dx ? dx[0] : nullptr, dx ? dx[0] : nullptr, dx ? dx[0] : nullptr};
  seg::Problems p{};
  int rc = segmented_args("lora_grad_input_segmented", dtype, nprob, tables, G, accumulate ? one : dx, n_adapters, workspace,
                          workspace_bytes, M, R, p);
  if (rc) return rc;
  if (K < 8 || K % 8 != 0 || K > INT32_MAX || (K + seg::kTileN - 1) / seg::kTileN > 65535)
    return set_error(QB200_EINVAL, "lora_grad_input_segmented: bad shape");
  if (ld_g == 0) ld_g = R;
  if (ld_dx == 0) ld_dx = K;
  if (ld_g < R || ld_g % 8 != 0 || ld_dx < K || ld_dx % 2 != 0)
    return set_error(QB200_EINVAL, "lora_grad_input_segmented: bad row pitch");
  const int n = n_adapters;
  const dim3 grid(unsigned(seg::layout(M, n).n_tiles), unsigned((K + seg::kTileN - 1) / seg::kTileN), unsigned(accumulate ? 1 : nprob));
  const auto* ws = static_cast<const uint8_t*>(workspace);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const char* what = "lora_grad_input_segmented";
  const bool f16 = dtype == QB200_DTYPE_F16;
  if (accumulate)
    return f16 ? launch_pdl(seg::lora_segmented_grad_kernel<__half, true, true>, grid, seg::kThreads, 0, s, what, p, nprob, ws, ld_g,
                            ld_dx, int(M), n, int(K), int(R))
               : launch_pdl(seg::lora_segmented_grad_kernel<__nv_bfloat16, true, true>, grid, seg::kThreads, 0, s, what, p, nprob, ws,
                            ld_g, ld_dx, int(M), n, int(K), int(R));
  return f16 ? launch_pdl(seg::lora_segmented_grad_kernel<__half, true, false>, grid, seg::kThreads, 0, s, what, p, nprob, ws, ld_g,
                          ld_dx, int(M), n, int(K), int(R))
             : launch_pdl(seg::lora_segmented_grad_kernel<__nv_bfloat16, true, false>, grid, seg::kThreads, 0, s, what, p, nprob, ws,
                          ld_g, ld_dx, int(M), n, int(K), int(R));
}

extern "C" int qb200_lora_weight_grad_segmented(int dtype, int nprob, int transpose_out, const qb200_lora_adapter* const* tables,
                                                const int64_t* rank_offsets, int64_t rank_total, const void* const* P, int64_t ld_p,
                                                const void* const* Q, int64_t ld_q, void* const* out, int n_adapters,
                                                const void* workspace, int64_t workspace_bytes, int64_t M, int64_t D, int64_t R,
                                                void* stream) {
  const char* what = "lora_weight_grad_segmented";
  seg::Problems p{};
  int rc = segmented_args(what, dtype, nprob, tables, P, out, n_adapters, workspace, workspace_bytes, M, R, p);
  if (rc) return rc;
  if (transpose_out != 0 && transpose_out != 1) return set_error(QB200_EINVAL, "lora_weight_grad_segmented: transpose_out must be 0 or 1");
  if (!Q || !rank_offsets) return set_error(QB200_EINVAL, "lora_weight_grad_segmented: null pointer");
  if (reinterpret_cast<uintptr_t>(rank_offsets) % 8)
    return set_error(QB200_EINVAL, "lora_weight_grad_segmented: rank_offsets must be 8-byte aligned");
  seg::WgradProblems w{};
  for (int i = 0; i < nprob; ++i) {
    if (!Q[i]) return set_error(QB200_EINVAL, "lora_weight_grad_segmented: null pointer");
    if (reinterpret_cast<uintptr_t>(Q[i]) % 16)
      return set_error(QB200_EINVAL, "lora_weight_grad_segmented: inputs must be 16-byte aligned");
    w.table[i] = p.table[i];
    w.P[i] = p.X[i];
    w.Q[i] = Q[i];
    w.out[i] = p.out[i];
  }
  const int64_t rt = (R + seg::kTileM - 1) / seg::kTileM;
  if (D < 8 || D % 8 != 0 || D > INT32_MAX || (D + seg::kTileN - 1) / seg::kTileN > 65535 || int64_t(n_adapters) * rt > INT32_MAX)
    return set_error(QB200_EINVAL, "lora_weight_grad_segmented: bad shape");
  if (rank_total < 8 || rank_total > INT64_MAX / D)
    return set_error(QB200_EINVAL, "lora_weight_grad_segmented: rank_total must be at least 8");
  if (ld_p == 0) ld_p = R;
  if (ld_q == 0) ld_q = D;
  if (ld_p < R || ld_q < D) return set_error(QB200_EINVAL, "lora_weight_grad_segmented: bad row pitch");
  const dim3 grid(unsigned(n_adapters * rt), unsigned((D + seg::kTileN - 1) / seg::kTileN), unsigned(nprob));
  const auto* ws = static_cast<const uint8_t*>(workspace);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool f16 = dtype == QB200_DTYPE_F16;
  const int m = int(M), d = int(D), r = int(R);
  if (transpose_out)
    return f16 ? launch_pdl(seg::lora_weight_grad_kernel<__half, true>, grid, seg::kThreads, 0, s, what, w, rank_offsets, rank_total, ws,
                            ld_p, ld_q, m, n_adapters, d, r)
               : launch_pdl(seg::lora_weight_grad_kernel<__nv_bfloat16, true>, grid, seg::kThreads, 0, s, what, w, rank_offsets,
                            rank_total, ws, ld_p, ld_q, m, n_adapters, d, r);
  return f16 ? launch_pdl(seg::lora_weight_grad_kernel<__half, false>, grid, seg::kThreads, 0, s, what, w, rank_offsets, rank_total, ws,
                          ld_p, ld_q, m, n_adapters, d, r)
             : launch_pdl(seg::lora_weight_grad_kernel<__nv_bfloat16, false>, grid, seg::kThreads, 0, s, what, w, rank_offsets,
                          rank_total, ws, ld_p, ld_q, m, n_adapters, d, r);
}
