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
// DoRA over the same tables (DESIGN.md §6e):
//   dora_gather_a_kernel        every adapter's A stacked into [sum r, K] rows, the input of one fused forward P = A . W^T.
//   dora_gram_kernel            G_a = A_a . A_a^T per adapter, fp32.
//   dora_norm_kernel            n_a = sqrt(||W_f||^2 + 2 s B_a P_a + s^2 B_a G_a B_a^T) and c_a = m_a / n_a per row f, fp32.
//   lora_segmented_kernel<kDora> the expand with DoRA's magnitude scale in the epilogue.
//   dora_grad_scale_kernel      dQ = rn(dY . c_a), dD = rn(dY . (c_a - 1)) and dm_a = rn(sum_t dY . Q / n_a) per bucket.
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

// The expand's DoRA operands, per problem: c [n, N] fp32 and (dropout) Q [M, N], read as rn(xd . W^T) and overwritten with
// the pre-scale term rn(Qb + U . B_a^T); its row pitch is the output's.
struct DoraProblems : Problems {
  const float* c[kMaxProb];
  void* q[kMaxProb];
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
// kDora (expand only; DoRA's magnitude scale c = c_a[column] of the tile's adapter, C = U . B_a^T in fp32):
//   1: y = rn(c . (y + C));   2 (dropout): y = rn(y + (c - 1) . Qb + c . C) and Q = rn(Qb + C) in place of Qb.
template <typename T16, bool kShrink, int kDora = 0>
__global__ void __launch_bounds__(kThreads) lora_segmented_kernel(std::conditional_t<(kDora != 0), DoraProblems, Problems> p,
                                                                  const uint8_t* __restrict__ ws, int64_t ld_x,
                                                                  int64_t ld_out, int M, int n, int N, int K, int R) {
  static_assert(kDora == 0 || !kShrink, "DoRA scales the expand only");
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
      } else if constexpr (kDora != 0) {
        const float2 cc = *reinterpret_cast<const float2*>(pick(p.c, z) + int64_t(a) * N + c);
        uint32_t y = *dst;
        const float2 f = widen2(*reinterpret_cast<const T2*>(&y));
        if constexpr (kDora == 1) {
          *dst = round16x2<T16>(cc.x * (f.x + s0), cc.y * (f.y + s1));
        } else {
          uint32_t* qdst = reinterpret_cast<uint32_t*>(static_cast<T16*>(pick(p.q, z)) + int64_t(t) * ld_out + c);
          uint32_t qv = *qdst;
          const float2 qb = widen2(*reinterpret_cast<const T2*>(&qv));
          *dst = round16x2<T16>(f.x + (cc.x - 1.0f) * qb.x + cc.x * s0, f.y + (cc.y - 1.0f) * qb.y + cc.y * s1);
          *qdst = round16x2<T16>(qb.x + s0, qb.y + s1);
        }
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

// ---- DoRA ---------------------------------------------------------------------------------------------------------------
// An adapter's entry is usable when its rank is a positive multiple of 8 whose clamped rank is not 0 and its rank offset keeps
// [off, off + rank) inside [0, total); the kernels below treat the rows and outputs of any other adapter as the base's.
__device__ __forceinline__ int dora_rank(const qb200_lora_adapter& ad, const int64_t* rank_off, int a, int64_t total, int R,
                                         int64_t& off) {
  if (ad.rank <= 0 || (ad.rank & 7)) return 0;
  const int rank = MixedLora::rank(ad, R);
  off = rank_off[a];
  return (off < 0 || off > total - rank) ? 0 : rank;
}

// out_p[j, :] = A_{p,a}[j - off_a, :] for every stacked row j of adapter a = stack_rows[j]; zeros for a row that lies
// outside its adapter's clamped rank.  One CTA per (stacked row, problem), 16 bytes per thread per step.
struct GatherProblems {
  const qb200_lora_adapter* table[kMaxProb];
  void* out[kMaxProb];
};
__global__ void __launch_bounds__(kThreads) dora_gather_a_kernel(GatherProblems p, const int32_t* __restrict__ stack_rows,
                                                                 const int64_t* __restrict__ rank_off, int64_t total, int n, int K,
                                                                 int R) {
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();
  const int64_t j = blockIdx.x;
  const int z = blockIdx.z;
  const int a = stack_rows[j];
  const uint4* src = nullptr;
  if (a >= 0 && a < n) {
    const qb200_lora_adapter ad = pick(p.table, z)[a];
    int64_t off = 0;
    const int rank = dora_rank(ad, rank_off, a, total, R, off);
    if (j >= off && j - off < rank) src = reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(ad.A) + (j - off) * K);
  }
  uint4* dst = reinterpret_cast<uint4*>(static_cast<uint16_t*>(pick(p.out, z)) + j * K);
  for (int v = threadIdx.x; v < K / 8; v += kThreads) dst[v] = src ? __ldg(src + v) : make_uint4(0, 0, 0, 0);
}

// G_a = A_a . A_a^T [r_a, r_a] row-major at gram_off[a] of problem z's fp32 buffer (an offset that would write past gram_total
// writes nothing).  One CTA of 256 threads per (adapter, 64 x 64 tile, problem), 4 x 4 outputs per thread, K in chunks of 32
// summed in order.
constexpr int kGramTile = 64, kGramChunk = 32, kGramThreads = 256;
struct NormProblems {
  const qb200_lora_adapter* table[kMaxProb];
  const void* const* mag[kMaxProb];    // DEVICE: n pointers to each adapter's magnitude [N]
  const float* P[kMaxProb];            // [total, N]: row off_a + j is A_a[j] . W^T
  const float* norm2[kMaxProb];        // ||W_f||^2 [N]
  float* gram[kMaxProb];               // sum_a r_a^2
  float* c[kMaxProb];                  // [n, N]
  float* nrm[kMaxProb];                // [n, N]
};
template <typename T16>
__device__ __forceinline__ float h2f(uint16_t h) {
  if constexpr (std::is_same_v<T16, __half>) return __half2float(__ushort_as_half(h));
  else return __uint_as_float(uint32_t(h) << 16);
}
template <typename T16>
__device__ __forceinline__ uint16_t f2h(float f) {
  if constexpr (std::is_same_v<T16, __half>) return __half_as_ushort(__float2half_rn(f));
  else return __bfloat16_as_ushort(__float2bfloat16_rn(f));
}

template <typename T16>
__global__ void __launch_bounds__(kGramThreads) dora_gram_kernel(NormProblems p, const int64_t* __restrict__ rank_off,
                                                                 const int64_t* __restrict__ gram_off, int64_t total,
                                                                 int64_t gram_total, int n, int K, int R) {
  __shared__ float sI[kGramChunk][kGramTile + 1];
  __shared__ float sJ[kGramChunk][kGramTile + 1];
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();
  const int rt = (R + kGramTile - 1) / kGramTile;
  const int a = int(blockIdx.x / unsigned(rt * rt)), tile = int(blockIdx.x % unsigned(rt * rt));
  const int i0 = (tile / rt) * kGramTile, j0 = (tile % rt) * kGramTile, z = blockIdx.z;
  if (a >= n) return;
  const qb200_lora_adapter ad = pick(p.table, z)[a];
  int64_t off = 0;
  const int rank = dora_rank(ad, rank_off, a, total, R, off);
  if (i0 >= rank || j0 >= rank) return;
  const int64_t g0 = gram_off[a];
  if (g0 < 0 || g0 > gram_total - int64_t(rank) * rank) return;
  const uint16_t* A = static_cast<const uint16_t*>(ad.A);
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += kGramChunk) {
#pragma unroll
    for (int e = 0; e < kGramTile * kGramChunk / kGramThreads; ++e) {
      const int v = tid + e * kGramThreads, r = v / kGramChunk, k = v % kGramChunk;
      const int ri = i0 + r, rj = j0 + r;
      sI[k][r] = ri < rank && k0 + k < K ? h2f<T16>(A[int64_t(ri) * K + k0 + k]) : 0.0f;
      sJ[k][r] = rj < rank && k0 + k < K ? h2f<T16>(A[int64_t(rj) * K + k0 + k]) : 0.0f;
    }
    __syncthreads();
#pragma unroll 8
    for (int k = 0; k < kGramChunk; ++k) {
      float vi[4], vj[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) vi[u] = sI[k][ty * 4 + u], vj[u] = sJ[k][tx * 4 + u];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int w = 0; w < 4; ++w) acc[u][w] = fmaf(vi[u], vj[w], acc[u][w]);
    }
    __syncthreads();
  }
  float* g = pick(p.gram, z) + g0;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int i = i0 + ty * 4 + u, j = j0 + tx * 4 + w;
      if (i < rank && j < rank) g[int64_t(i) * rank + j] = acc[u][w];
    }
}

// n_a[f]^2 = ||W_f||^2 + 2 s_a sum_j B_a[f, j] P[off_a + j, f] + s_a^2 sum_{j,k} B_a[f, j] G_a[j, k] B_a[f, k], clamped at 0;
// c_a[f] = m_a[f] / n_a[f].  One CTA of 256 threads per (adapter, 64 rows f, problem): four threads per row, thread q taking
// the j (cross term) and k (quadratic term) congruent to q mod 4, reduced in a fixed order.  An unusable adapter gets c = n = 0.
constexpr int kNormRows = 64, kNormGRows = 8;
template <typename T16>
__global__ void __launch_bounds__(kGramThreads) dora_norm_kernel(NormProblems p, const int64_t* __restrict__ rank_off,
                                                                 const int64_t* __restrict__ gram_off, int64_t total,
                                                                 int64_t gram_total, int n, int N, int R) {
  __shared__ uint16_t sB[kNormRows][kMaxLoraRank + 8];
  __shared__ float sG[kNormGRows][kMaxLoraRank];
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();
  const int a = blockIdx.x, f0 = blockIdx.y * kNormRows, z = blockIdx.z;
  const int tid = threadIdx.x, q = tid & 3, fl = tid >> 2, f = f0 + fl;
  const qb200_lora_adapter ad = pick(p.table, z)[a];
  int64_t off = 0;
  int rank = dora_rank(ad, rank_off, a, total, R, off);
  const int64_t g0 = gram_off[a];
  if (rank && (g0 < 0 || g0 > gram_total - int64_t(rank) * rank)) rank = 0;
  float* c_out = pick(p.c, z) + int64_t(a) * N;
  float* n_out = pick(p.nrm, z) + int64_t(a) * N;
  if (rank == 0) {
    if (q == 0 && f < N) c_out[f] = 0.0f, n_out[f] = 0.0f;
    return;
  }
  const uint16_t* B = static_cast<const uint16_t*>(ad.B);
  for (int v = tid; v < kNormRows * rank; v += kGramThreads) {
    const int r = v / rank, k = v % rank;
    sB[r][k] = f0 + r < N ? B[int64_t(f0 + r) * ad.rank + k] : uint16_t(0);
  }
  __syncthreads();
  const bool live = f < N;
  const float* P = pick(p.P, z) + off * N;
  float cross = 0.0f;
  if (live)
    for (int j = q; j < rank; j += 4) cross = fmaf(h2f<T16>(sB[fl][j]), P[int64_t(j) * N + f], cross);
  const float* G = pick(p.gram, z) + g0;
  float quad = 0.0f;
  for (int j0 = 0; j0 < rank; j0 += kNormGRows) {
    for (int v = tid; v < kNormGRows * rank; v += kGramThreads) {
      const int r = v / rank, k = v % rank;
      sG[r][k] = j0 + r < rank ? G[int64_t(j0 + r) * rank + k] : 0.0f;
    }
    __syncthreads();
    if (live) {
#pragma unroll
      for (int jj = 0; jj < kNormGRows; ++jj) {
        float h = 0.0f;
        for (int k = q; k < rank; k += 4) h = fmaf(sG[jj][k], h2f<T16>(sB[fl][k]), h);
        if (j0 + jj < rank) quad = fmaf(h2f<T16>(sB[fl][j0 + jj]), h, quad);
      }
    }
    __syncthreads();
  }
  cross += __shfl_xor_sync(0xffffffffu, cross, 1);
  cross += __shfl_xor_sync(0xffffffffu, cross, 2);
  quad += __shfl_xor_sync(0xffffffffu, quad, 1);
  quad += __shfl_xor_sync(0xffffffffu, quad, 2);
  if (!live || q != 0) return;
  const float s = ad.scale;
  const float n2 = fmaxf(pick(p.norm2, z)[f] + (2.0f * s) * cross + (s * s) * quad, 0.0f);
  const float nrm = sqrtf(n2);
  const uint16_t* mag = static_cast<const uint16_t*>(pick(p.mag, z)[a]);
  c_out[f] = (mag ? h2f<T16>(mag[f]) : 0.0f) / nrm;
  n_out[f] = nrm;
}

// Per bucket b (an adapter, or b = n: the rows without one) and problem, over the bucket's sorted rows t, columns f:
//   dQ[t] = rn(dY[t] . c_a),  kDropout: dD[t] = rn(dY[t] . (c_a - 1)),  dm_a = rn(sum_t dY[t] . Q[t] / n_a)
// where Q is the expand's pre-scale output (kDropout) or y / c_a (no dropout; an element with c = 0 adds nothing).  Rows
// without a usable adapter copy dY into dQ and write dD = 0; an adapter without rows gets dm = 0.  One CTA of 256 threads
// per (bucket, 64 columns, problem): eight row groups of 32 threads x 2 columns, row i of the bucket to group i % 8, the
// groups' fp32 sums added in group order.
struct ScaleProblems {
  const qb200_lora_adapter* table[kMaxProb];
  const void* dy[kMaxProb];
  const void* q[kMaxProb];             // Q (dropout) or y, row pitch ld
  const float* c[kMaxProb];            // [n, N]
  const float* nrm[kMaxProb];          // [n, N]
  void* dq[kMaxProb];
  void* dd[kMaxProb];
  void* dm[kMaxProb];                  // [n, N] of the compute dtype
};
constexpr int kScaleCols = 64, kScaleGroups = 8;
template <typename T16, bool kDropout>
__global__ void __launch_bounds__(kGramThreads) dora_grad_scale_kernel(ScaleProblems p, const int64_t* __restrict__ rank_off,
                                                                       int64_t total, const uint8_t* __restrict__ ws, int64_t ld,
                                                                       int M, int n, int N, int R) {
  __shared__ float2 s_part[kScaleGroups][kScaleCols / 2];
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();
  const int b = blockIdx.x, z = blockIdx.z;
  const int tid = threadIdx.x, g = tid >> 5, col = blockIdx.y * kScaleCols + 2 * (tid & 31);
  const Layout L = layout(M, n);
  const int* perm = reinterpret_cast<const int*>(ws + L.perm);
  const int* boff = reinterpret_cast<const int*>(ws + L.off);
  const int b0 = max(0, min(boff[b], M)), b1 = max(b0, min(boff[b + 1], M));
  int rank = 0;
  if (b < n) {
    int64_t off = 0;
    rank = dora_rank(pick(p.table, z)[b], rank_off, b, total, R, off);
  }
  using T2 = typename Vec2<T16>::type;
  const bool live = col < N;
  float2 cc = make_float2(1.0f, 1.0f), acc = make_float2(0.0f, 0.0f);
  if (rank && live) cc = *reinterpret_cast<const float2*>(pick(p.c, z) + int64_t(b) * N + col);
  const T16* dy = static_cast<const T16*>(pick(p.dy, z));
  const T16* qy = static_cast<const T16*>(pick(p.q, z));
  T16* dq = static_cast<T16*>(pick(p.dq, z));
  T16* dd = static_cast<T16*>(pick(p.dd, z));
  if (live) {
    for (int i = b0 + g; i < b1; i += kScaleGroups) {
      const int t = perm[i];
      if (t < 0 || t >= M) continue;
      const int64_t e = int64_t(t) * ld + col;
      const uint32_t dv = *reinterpret_cast<const uint32_t*>(dy + e);
      if (!rank) {
        *reinterpret_cast<uint32_t*>(dq + e) = dv;
        if (kDropout) *reinterpret_cast<uint32_t*>(dd + e) = 0u;
        continue;
      }
      const float2 d = widen2(*reinterpret_cast<const T2*>(&dv));
      const uint32_t qv = *reinterpret_cast<const uint32_t*>(qy + e);
      float2 qf = widen2(*reinterpret_cast<const T2*>(&qv));
      if (!kDropout) qf = make_float2(cc.x != 0.0f ? qf.x / cc.x : 0.0f, cc.y != 0.0f ? qf.y / cc.y : 0.0f);
      *reinterpret_cast<uint32_t*>(dq + e) = round16x2<T16>(d.x * cc.x, d.y * cc.y);
      if (kDropout) *reinterpret_cast<uint32_t*>(dd + e) = round16x2<T16>(d.x * (cc.x - 1.0f), d.y * (cc.y - 1.0f));
      acc.x = fmaf(d.x, qf.x, acc.x);
      acc.y = fmaf(d.y, qf.y, acc.y);
    }
  }
  if (b >= n) return;
  s_part[g][tid & 31] = acc;
  __syncthreads();
  if (g != 0 || !live) return;
  float2 sum = s_part[0][tid];
#pragma unroll
  for (int k = 1; k < kScaleGroups; ++k) sum.x += s_part[k][tid].x, sum.y += s_part[k][tid].y;
  uint32_t out = 0u;
  if (rank && b1 > b0) {
    const float2 nv = *reinterpret_cast<const float2*>(pick(p.nrm, z) + int64_t(b) * N + col);
    out = round16x2<T16>(sum.x / nv.x, sum.y / nv.y);
  }
  *reinterpret_cast<uint32_t*>(static_cast<T16*>(pick(p.dm, z)) + int64_t(b) * N + col) = out;
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

// ---- DoRA entry points --------------------------------------------------------------------------------------------------
// The checks the DoRA entry points share: dtype, problem count, adapter count, R and the per-problem tables.
static int dora_args(const char* what, int dtype, int nprob, const qb200_lora_adapter* const* tables, int n_adapters, int64_t R) {
  char msg[160];
  if (dtype != QB200_DTYPE_BF16 && dtype != QB200_DTYPE_F16) {
    snprintf(msg, sizeof(msg), "%s: dtype must be 2 (bf16) or 1 (fp16)", what);
    return set_error(QB200_EINVAL, msg);
  }
  if (nprob < 1 || nprob > seg::kMaxProb || !tables) {
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
  for (int i = 0; i < nprob; ++i) {
    if (!tables[i]) {
      snprintf(msg, sizeof(msg), "%s: null pointer", what);
      return set_error(QB200_EINVAL, msg);
    }
    if (reinterpret_cast<uintptr_t>(tables[i]) % 8) {
      snprintf(msg, sizeof(msg), "%s: tables must be 8-byte aligned", what);
      return set_error(QB200_EINVAL, msg);
    }
  }
  return 0;
}

// every pointer of a per-problem array present and `align`-byte aligned
template <typename T>
static bool all_set(const T* const* v, int nprob, int align) {
  if (!v) return false;
  for (int i = 0; i < nprob; ++i)
    if (!v[i] || reinterpret_cast<uintptr_t>(v[i]) % align) return false;
  return true;
}

extern "C" int qb200_dora_stack_a(int dtype, int nprob, const qb200_lora_adapter* const* tables, const int32_t* stack_rows,
                                  const int64_t* rank_offsets, int64_t rank_total, void* const* out, int n_adapters, int64_t K,
                                  int64_t R, void* stream) {
  const char* what = "dora_stack_a";
  int rc = dora_args(what, dtype, nprob, tables, n_adapters, R);
  if (rc) return rc;
  if (!stack_rows || !rank_offsets || !all_set(out, nprob, 16))
    return set_error(QB200_EINVAL, "dora_stack_a: null pointer, or an output that is not 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(rank_offsets) % 8 || reinterpret_cast<uintptr_t>(stack_rows) % 4)
    return set_error(QB200_EINVAL, "dora_stack_a: rank_offsets must be 8-byte and stack_rows 4-byte aligned");
  if (K < 8 || K % 8 != 0 || K > INT32_MAX || rank_total < 8 || rank_total > INT32_MAX)
    return set_error(QB200_EINVAL, "dora_stack_a: bad shape");
  seg::GatherProblems p{};
  for (int i = 0; i < nprob; ++i) p.table[i] = tables[i], p.out[i] = out[i];
  const dim3 grid(unsigned(rank_total), 1, unsigned(nprob));
  return launch_pdl(seg::dora_gather_a_kernel, grid, seg::kThreads, 0, static_cast<cudaStream_t>(stream), what, p, stack_rows,
                    rank_offsets, rank_total, n_adapters, int(K), int(R));
}

extern "C" int qb200_dora_norm_segmented(int dtype, int nprob, const qb200_lora_adapter* const* tables, const void* const* mag_tables,
                                         const int64_t* rank_offsets, const int64_t* gram_offsets, int64_t rank_total,
                                         int64_t gram_total, const float* const* P, const float* const* row_norm2,
                                         float* const* gram, float* const* c, float* const* norm, int n_adapters, int64_t N,
                                         int64_t K, int64_t R, void* stream) {
  const char* what = "dora_norm_segmented";
  int rc = dora_args(what, dtype, nprob, tables, n_adapters, R);
  if (rc) return rc;
  if (!rank_offsets || !gram_offsets || !all_set(mag_tables, nprob, 8) || !all_set(P, nprob, 4) || !all_set(row_norm2, nprob, 4) ||
      !all_set(gram, nprob, 4) || !all_set(c, nprob, 8) || !all_set(norm, nprob, 8))
    return set_error(QB200_EINVAL, "dora_norm_segmented: null pointer, or c / norm not 8-byte and the other arrays not 4-byte aligned");
  if (reinterpret_cast<uintptr_t>(rank_offsets) % 8 || reinterpret_cast<uintptr_t>(gram_offsets) % 8)
    return set_error(QB200_EINVAL, "dora_norm_segmented: rank_offsets and gram_offsets must be 8-byte aligned");
  const int64_t rt = (R + seg::kGramTile - 1) / seg::kGramTile;
  if (N < 8 || N % 8 != 0 || N > INT32_MAX || (N + seg::kNormRows - 1) / seg::kNormRows > 65535 || K < 8 || K > INT32_MAX ||
      int64_t(n_adapters) * rt * rt > INT32_MAX || rank_total < 8 || gram_total < 64)
    return set_error(QB200_EINVAL, "dora_norm_segmented: bad shape");
  seg::NormProblems p{};
  for (int i = 0; i < nprob; ++i) {
    p.table[i] = tables[i];
    p.mag[i] = static_cast<const void* const*>(mag_tables[i]);
    p.P[i] = P[i], p.norm2[i] = row_norm2[i], p.gram[i] = gram[i], p.c[i] = c[i], p.nrm[i] = norm[i];
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool f16 = dtype == QB200_DTYPE_F16;
  const dim3 g_grid(unsigned(n_adapters * rt * rt), 1, unsigned(nprob));
  rc = f16 ? launch_pdl(seg::dora_gram_kernel<__half>, g_grid, seg::kGramThreads, 0, s, what, p, rank_offsets, gram_offsets,
                        rank_total, gram_total, n_adapters, int(K), int(R))
           : launch_pdl(seg::dora_gram_kernel<__nv_bfloat16>, g_grid, seg::kGramThreads, 0, s, what, p, rank_offsets, gram_offsets,
                        rank_total, gram_total, n_adapters, int(K), int(R));
  if (rc) return rc;
  const dim3 n_grid(unsigned(n_adapters), unsigned((N + seg::kNormRows - 1) / seg::kNormRows), unsigned(nprob));
  return f16 ? launch_pdl(seg::dora_norm_kernel<__half>, n_grid, seg::kGramThreads, 0, s, what, p, rank_offsets, gram_offsets,
                          rank_total, gram_total, n_adapters, int(N), int(R))
             : launch_pdl(seg::dora_norm_kernel<__nv_bfloat16>, n_grid, seg::kGramThreads, 0, s, what, p, rank_offsets, gram_offsets,
                          rank_total, gram_total, n_adapters, int(N), int(R));
}

extern "C" int qb200_dora_expand_segmented(int dtype, int nprob, int dropout, const qb200_lora_adapter* const* tables,
                                           const void* const* U, int64_t ld_u, const float* const* c, void* const* Q,
                                           void* const* out, int64_t ld_out, int n_adapters, const void* workspace,
                                           int64_t workspace_bytes, int64_t M, int64_t N, int64_t R, void* stream) {
  const char* what = "dora_expand_segmented";
  if (dropout != 0 && dropout != 1) return set_error(QB200_EINVAL, "dora_expand_segmented: dropout must be 0 or 1");
  seg::DoraProblems p{};
  int rc = segmented_args(what, dtype, nprob, tables, U, out, n_adapters, workspace, workspace_bytes, M, R, p);
  if (rc) return rc;
  if (!all_set(c, nprob, 8) || (dropout && !all_set(Q, nprob, 4)))
    return set_error(QB200_EINVAL, "dora_expand_segmented: null pointer, or c not 8-byte or Q not 4-byte aligned");
  if (N < 8 || N % 8 != 0 || N > INT32_MAX || int64_t(N + seg::kTileN - 1) / seg::kTileN > 65535)
    return set_error(QB200_EINVAL, "dora_expand_segmented: bad shape");
  if (ld_u == 0) ld_u = R;
  if (ld_out == 0) ld_out = N;
  if (ld_u < R || ld_u % 8 != 0 || ld_out < N || ld_out % 2 != 0)
    return set_error(QB200_EINVAL, "dora_expand_segmented: bad row pitch");
  for (int i = 0; i < nprob; ++i) p.c[i] = c[i], p.q[i] = dropout ? Q[i] : nullptr;
  const dim3 grid(unsigned(seg::layout(M, n_adapters).n_tiles), unsigned((N + seg::kTileN - 1) / seg::kTileN), unsigned(nprob));
  const auto* ws = static_cast<const uint8_t*>(workspace);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int m = int(M), n = n_adapters, nn = int(N), r = int(R);
  if (dtype == QB200_DTYPE_F16)
    return dropout ? launch_pdl(seg::lora_segmented_kernel<__half, false, 2>, grid, seg::kThreads, 0, s, what, p, ws, ld_u, ld_out, m, n,
                                nn, 0, r)
                   : launch_pdl(seg::lora_segmented_kernel<__half, false, 1>, grid, seg::kThreads, 0, s, what, p, ws, ld_u, ld_out, m, n,
                                nn, 0, r);
  return dropout ? launch_pdl(seg::lora_segmented_kernel<__nv_bfloat16, false, 2>, grid, seg::kThreads, 0, s, what, p, ws, ld_u, ld_out,
                              m, n, nn, 0, r)
                 : launch_pdl(seg::lora_segmented_kernel<__nv_bfloat16, false, 1>, grid, seg::kThreads, 0, s, what, p, ws, ld_u, ld_out,
                              m, n, nn, 0, r);
}

extern "C" int qb200_dora_grad_scale_segmented(int dtype, int nprob, int dropout, const qb200_lora_adapter* const* tables,
                                               const int64_t* rank_offsets, int64_t rank_total, const void* const* dY,
                                               const void* const* Q, const float* const* c, const float* const* norm, int64_t ld,
                                               void* const* dQ, void* const* dD, void* const* dm, int n_adapters,
                                               const void* workspace, int64_t workspace_bytes, int64_t M, int64_t N, int64_t R,
                                               void* stream) {
  const char* what = "dora_grad_scale_segmented";
  if (dropout != 0 && dropout != 1) return set_error(QB200_EINVAL, "dora_grad_scale_segmented: dropout must be 0 or 1");
  seg::Problems base{};
  int rc = segmented_args(what, dtype, nprob, tables, dY, dQ, n_adapters, workspace, workspace_bytes, M, R, base);
  if (rc) return rc;
  if (!rank_offsets || !all_set(Q, nprob, 4) || !all_set(c, nprob, 8) || !all_set(norm, nprob, 8) || !all_set(dm, nprob, 4) ||
      (dropout && !all_set(dD, nprob, 4)) || reinterpret_cast<uintptr_t>(rank_offsets) % 8)
    return set_error(QB200_EINVAL, "dora_grad_scale_segmented: null pointer or misaligned array");
  if (N < 8 || N % 8 != 0 || N > INT32_MAX || (N + seg::kScaleCols - 1) / seg::kScaleCols > 65535 || rank_total < 8)
    return set_error(QB200_EINVAL, "dora_grad_scale_segmented: bad shape");
  if (ld == 0) ld = N;
  if (ld < N || ld % 2 != 0) return set_error(QB200_EINVAL, "dora_grad_scale_segmented: bad row pitch");
  seg::ScaleProblems p{};
  for (int i = 0; i < nprob; ++i) {
    p.table[i] = tables[i], p.dy[i] = dY[i], p.q[i] = Q[i], p.c[i] = c[i], p.nrm[i] = norm[i];
    p.dq[i] = dQ[i], p.dd[i] = dropout ? dD[i] : nullptr, p.dm[i] = dm[i];
  }
  const dim3 grid(unsigned(n_adapters + 1), unsigned((N + seg::kScaleCols - 1) / seg::kScaleCols), unsigned(nprob));
  const auto* ws = static_cast<const uint8_t*>(workspace);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int m = int(M), n = n_adapters, nn = int(N), r = int(R);
  if (dtype == QB200_DTYPE_F16)
    return dropout ? launch_pdl(seg::dora_grad_scale_kernel<__half, true>, grid, seg::kGramThreads, 0, s, what, p, rank_offsets,
                                rank_total, ws, ld, m, n, nn, r)
                   : launch_pdl(seg::dora_grad_scale_kernel<__half, false>, grid, seg::kGramThreads, 0, s, what, p, rank_offsets,
                                rank_total, ws, ld, m, n, nn, r);
  return dropout ? launch_pdl(seg::dora_grad_scale_kernel<__nv_bfloat16, true>, grid, seg::kGramThreads, 0, s, what, p, rank_offsets,
                              rank_total, ws, ld, m, n, nn, r)
                 : launch_pdl(seg::dora_grad_scale_kernel<__nv_bfloat16, false>, grid, seg::kGramThreads, 0, s, what, p, rank_offsets,
                              rank_total, ws, ld, m, n, nn, r);
}
