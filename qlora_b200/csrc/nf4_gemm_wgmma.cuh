// Persistent fused NF4 dequant + wgmma GEMM (the production kernel; DESIGN.md 4.1).
//
// One CTA per SM.  Work unit = 128 features (two wgmma M=64 halves, one per consumer warpgroup) x up to 128 tokens (wgmma
// N = 16..128), 64-wide contraction steps.  Per step the CTA dequantizes its 128 feature rows once into a T16 A tile in
// shared memory and TMA-loads the 128-row activation block; both warpgroups' MMAs read them straight from shared memory.
// T16, the operand type of a launch, is bf16 or fp16: the tile layouts, swizzle and descriptors are the same for both.
// Under bf16 compute the quant state may be fp16 (kStateF16: double-rounded product table) and the output fp16 (kOutF16).
//
// Schedule (host: nf4_gemm_sm90.cu).  The output of a launch is a strip of `n_fb x T` token-rows (n_fb = 128-feature blocks
// of all problems of the launch, T = tokens); CTA c owns the CONTIGUOUS range [start[c], start[c+1]) of that strip and
// cuts it into units at feature-block boundaries and every 128 tokens, so a unit may hold any multiple of 16 tokens.  The
// host places the range boundaries with a cost model, which removes the wave quantization of whole-tile schedules.  Token
// counts so small that even this leaves most SMs idle take the split-K schedule instead (fp32 partials + reduce kernel).
//
// Grouped launches (Params::nprob > 1): problems that share their shape run as ONE launch — either side by side
// (forward q/k/v or gate/up of one input: the strip simply spans all problems) or as segments of one long contraction
// accumulated in the same registers (dX of q/k/v: dX = sum_p dY_p . W_p, no separate adds).
//
// Roles (640 threads): warps 0-7 two consumer warpgroups (wgmma issue, accumulators in registers, output stores) |
// warps 8-19 dequantizers: THREE groups of four warps take the contraction steps round-robin; a thread owns one 64-value
// NF4 block per step: 16-entry product table, PRMT lookups, eight st.shared.v4 into the A slot, fence.proxy.async, arrive —
// and only THEN the global loads (nibbles + statistics) of the group's next step: fence.proxy.async orders all of the
// thread's earlier memory operations and would otherwise wait for loads issued before it.  The group's first thread also
// issues the step's activation TMA load once the slot is free.  There is no separate producer warp: 20 warps are five per
// SM sub-partition, which leaves 96 registers a thread; a 21st warp would leave 80, less than the 64 accumulators of an
// m64n128 tile and their addressing need.
//
// Barrier protocol (shared memory of the CTA):
//   full_in[s]  arrive.expect_tx + TMA complete_tx (issued by the dequant group of the step) -> consumers
//   full_a[s]   4 dequant-warp arrivals (or the group's LoRA V tile, lora_bar)           -> consumers
//   empty[s]    8 consumer-warp arrivals once the step's wgmma group has completed      -> dequantizers
//   lora_bar[g] TMA of a LoRA V tile into an A slot, one barrier per dequant group      -> that group
// The consumers keep one wgmma group in flight: step g's slot is released after wgmma.wait_group 1 in step g + 1.
//
// Programmatic dependent launch: the kernel is launched with programmatic stream serialization, signals
// griddepcontrol.launch_dependents once its prologue is done and executes griddepcontrol.wait before the first read of
// anything an earlier kernel may have written (activations, U, V) and before the first output store.  The packed weights
// and their statistics are frozen since load time, so the dequant groups fill the A ring while the previous kernel drains.
#pragma once
#include "nf4_gemm_common.cuh"

namespace qb200 {
namespace gemm {
namespace wg {

constexpr int kUnitF = kBlockF;        // features per unit (two M=64 warpgroup halves)
constexpr int kUnitT = 128;            // max tokens per unit (wgmma N)
constexpr int kInSlotBytes = kUnitT * kBlockC * 2;  // 16 KB: one activation block
constexpr int kStages = 6;             // activation slots = A slots (6 x 32 KB)
constexpr int kMaxCtas = 160;          // >= SMs of the device (H100 SXM: 132)
constexpr int kSmemTiles = kStages * (kInSlotBytes + kATileBytes);   // 192 KB
constexpr int kSmemBytes = kSmemTiles + kAuxBytes + 1024;

struct Maps {
  CUtensorMap in[kMaxProb];   // activations In_p[T, C]   (forward groups: the same tensor for every problem)
  CUtensorMap u[kMaxProb];    // LoRA U_p[T, r]
  CUtensorMap v[kMaxProb];    // LoRA V_p: [F, r] forward, [r, F] dX
};

struct Sched {
  int ksplit;                    // > 1: split-K schedule — every 128 x 128 tile's contraction is divided over `ksplit` work units
  int n_tt;                      // split-K: 128-token tiles per feature block
  int n_work;                    // split-K: number of work units; CTA c runs units c, c + num_ctas, ...
  int t_pad;                     // range schedule: T rounded up to a multiple of 16
  int start[kMaxCtas + 1];       // range schedule: CTA c owns token-rows [start[c], start[c+1]) of the n_fb x t_pad strip
};

struct Work {
  int next;    // cursor of the CTA's following unit
  int prob;    // problem that owns the unit (side-by-side groups); 0 for contraction-sum groups
  int f0;      // first feature row
  int t0;      // first token
  int nt;      // tokens (multiple of 16, <= kUnitT)
  int kb0;     // first NF4 contraction step
  int nkb;     // NF4 contraction steps per segment
  int nseg;    // contraction segments (contraction-sum groups: one per problem)
  int lora;    // 1: a 16-bit LoRA step follows the NF4 steps of every segment
  int split;   // split-K index (0 when the unit covers the whole contraction)
};

// Decode the unit at cursor `a` of a CTA whose range ends at `end`.
__device__ __forceinline__ Work decode_work(int a, int end, int num_ctas, const Sched& sched, const Params& p, int num_kb,
                                            int has_lora) {
  Work w;
  int fb;
  if (sched.ksplit > 1) {
    const int tile = a / sched.ksplit;
    w.split = a - tile * sched.ksplit;
    const int per = (num_kb + sched.ksplit - 1) / sched.ksplit;
    w.kb0 = w.split * per;
    w.nkb = (num_kb - w.kb0) < per ? (num_kb - w.kb0) : per;
    w.lora = (has_lora && w.split == 0) ? 1 : 0;
    fb = tile / sched.n_tt;
    w.t0 = (tile - fb * sched.n_tt) * kUnitT;
    const int rem = p.T - w.t0;                          // few-token calls issue narrow MMAs and store only what exists
    w.nt = rem >= kUnitT ? kUnitT : ((rem + 15) & ~15);
    w.prob = 0;
    w.nseg = 1;
    w.next = a + num_ctas;
  } else {
    const int fbg = a / sched.t_pad;
    w.t0 = a - fbg * sched.t_pad;
    int ntok = sched.t_pad - w.t0;
    if (end - a < ntok) ntok = end - a;
    if (ntok > kUnitT) ntok = kUnitT;
    w.next = a + ntok;
    w.nt = ntok;
    if (p.group_sum || p.nprob == 1) {
      w.prob = 0;
      fb = fbg;
      w.nseg = p.group_sum ? p.nprob : 1;
    } else {
      const int n_fb = (p.F + kUnitF - 1) / kUnitF;
      w.prob = fbg / n_fb;
      fb = fbg - w.prob * n_fb;
      w.nseg = 1;
    }
    w.split = 0;
    w.kb0 = 0;
    w.nkb = num_kb;
    w.lora = has_lora;
  }
  w.f0 = fb * kUnitF;
  return w;
}

#ifndef QB200_NUM_GROUPS
#define QB200_NUM_GROUPS 3
#endif
constexpr int kNumGroups = QB200_NUM_GROUPS;                    // dequant groups
constexpr int kGroupWarps = 4;                                  // 128 threads: one NF4 block (A-tile row) each
constexpr int kConsumerWarps = 8;                               // two warpgroups
constexpr int kFirstDequantWarp = kConsumerWarps;
constexpr int kNumThreads = 32 * (kFirstDequantWarp + kNumGroups * kGroupWarps);   // 640

// Output of warpgroup `wg`'s 64 x kN part of a unit straight from the accumulator registers (kOutF16: see consume_unit).
template <typename T16, int kN, bool kOutF16, int kAcc, typename SchedT>
__device__ __forceinline__ void store_unit(const Work& w, const Params& p, const SchedT& sched, int wg, int warp, int lane,
                                           float (&acc)[kAcc]) {
  // Thread (warp w of the warpgroup, lane l) holds features
  // f0 + 64 wg + 16 w + l / 4 (+ 8) for tokens t0 + 8 j + 2 (l % 4) + {0, 1}.
  ptx::grid_dep_wait();   // the output buffer (and bias) may still be in use by an earlier kernel; no-op after the first call
  if (p.debug & 4) return;
  const Prob& pr = p.pr[w.prob];
  const int fa = w.f0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int tl = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int f = fa + 8 * h;
    if (f >= p.F) continue;
    if (sched.ksplit > 1) {   // fp32 partial sums into the workspace [ksplit, T, F]; bias is added by the reduce
      float* ws = p.ws + (int64_t(w.split) * p.T) * p.F + f;
#pragma unroll
      for (int j = 0; j < kN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int t = w.t0 + 8 * j + tl + e;
          if (t < p.T) ws[int64_t(t) * p.F] = acc[4 * j + 2 * h + e];
        }
      continue;
    }
    const T16* bias = static_cast<const T16*>(pr.bias);
    const float bias_v = bias != nullptr ? widen(bias[f]) : 0.0f;
#pragma unroll
    for (int j = 0; j < kN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int t = w.t0 + 8 * j + tl + e;
        if (t >= p.T || 8 * j + tl + e >= w.nt) continue;
        const T16 o = round16<T16>(acc[4 * j + 2 * h + e] + bias_v);
        if constexpr (kOutF16)
          static_cast<__half*>(pr.out)[int64_t(t) * pr.ld_out + f] = bf16_to_f16(o);
        else if (!p.out_f32)
          static_cast<T16*>(pr.out)[int64_t(t) * pr.ld_out + f] = o;
        else   // the 16-bit rounding of the reference's GEMM output first, then widened: one store pass, no cast kernel
          static_cast<float*>(pr.out)[int64_t(t) * pr.ld_out + f] = widen(o);
      }
  }
}

// Consumer warpgroup `wg`: all steps of one unit with wgmma N = kN (>= the unit's tokens), then the output stores.
// kOutF16 (bf16 compute only): the output is fp16, the bf16-rounded result rounded again (p.out_f32 is not read).
template <typename T16, int kN, bool kTrans, bool kOutF16>
__device__ __forceinline__ void consume_unit(const Work& w, const Params& p, const Sched& sched, int wg, int warp, int lane,
                                             uint32_t smem_base, uint32_t aux, uint32_t& g, float (&acc)[ptx::kWgmmaMaxAcc]) {
  auto in_tile = [&](int s) { return smem_base + uint32_t(s) * kInSlotBytes; };
  auto a_tile = [&](int s) { return smem_base + uint32_t(kStages) * kInSlotBytes + uint32_t(s) * kATileBytes; };
  auto full_in = [&](int s) { return aux + 8u * uint32_t(s); };
  auto full_a = [&](int s) { return aux + 8u * uint32_t(kStages + s); };
  auto empty = [&](int s) { return aux + 8u * uint32_t(2 * kStages + s); };
  const int nsteps = w.nseg * (w.nkb + w.lora);
  for (int kb = 0; kb < nsteps; ++kb, ++g) {
    const int s = int(g % kStages);
    const uint32_t ph = (g / kStages) & 1;
    ptx::mbar_wait(full_in(s), ph);
    ptx::mbar_wait(full_a(s), ph);
    // this warpgroup's 64 features: rows 64 wg.. of the K-major tile, or the wg-th 64-feature atom of the MN-major tile
    const uint32_t a_addr = a_tile(s) + uint32_t(wg) * 8192u;
    const uint64_t a_desc = kTrans ? make_desc_mnmajor_sw128(a_addr, 8192, 1024) : make_desc_kmajor_sw128(a_addr);
    const uint64_t b_desc = make_desc_kmajor_sw128(in_tile(s));
    if (!(p.debug & 2)) {
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockC / kMmaK; ++k) {
        const uint64_t a_adv = kTrans ? uint64_t((k * 2 * 1024) >> 4) : uint64_t((k * kMmaK * 2) >> 4);
        const uint64_t b_adv = uint64_t((k * kMmaK * 2) >> 4);
        ptx::wgmma<T16, kN, kTrans ? 1 : 0>(acc, a_desc + a_adv, b_desc + b_adv, (kb | k) != 0 ? 1u : 0u);
      }
      ptx::wgmma_commit();
    }
    if (kb > 0) {                 // the previous step's group is complete: release its slots
      ptx::wgmma_wait<1>(acc);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(empty(int((g - 1) % kStages)));
    }
  }
  ptx::wgmma_wait<0>(acc);
  __syncwarp();
  if (lane == 0) ptx::mbar_arrive(empty(int((g - 1) % kStages)));
  store_unit<T16, kN, kOutF16>(w, p, sched, wg, warp, lane, acc);
}

// kStateF16: bf16 compute over an fp16 quant state (the double-rounded product table of build_table); kOutF16: see
// consume_unit.  Both are false for every fp16-compute instantiation.
template <typename T16, bool kTrans, bool kNested, bool kStateF16, bool kOutF16>
__global__ void __launch_bounds__(kNumThreads, 1)
nf4_gemm_wgmma_kernel(const __grid_constant__ Maps maps, const __grid_constant__ Params p, const __grid_constant__ Sched sched) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - ptx::smem_u32(smem_raw));

  auto in_tile = [&](int s) { return smem_base + uint32_t(s) * kInSlotBytes; };
  auto a_tile = [&](int s) { return smem_base + uint32_t(kStages) * kInSlotBytes + uint32_t(s) * kATileBytes; };
  constexpr uint32_t kAuxOff = uint32_t(kSmemTiles);
  const uint32_t aux = smem_base + kAuxOff;
  auto full_in = [&](int s) { return aux + 8u * uint32_t(s); };
  auto full_a = [&](int s) { return aux + 8u * uint32_t(kStages + s); };
  auto empty = [&](int s) { return aux + 8u * uint32_t(2 * kStages + s); };
  auto lora_bar = [&](int g) { return aux + 8u * uint32_t(3 * kStages + g); };
  static_assert(8 * (3 * kStages + kNumGroups) <= 1024, "barrier table overflows its 1 KB");
  float* s_code = reinterpret_cast<float*>(smem_gen + kAuxOff + 1024);   // [kMaxProb][256]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_ctas = gridDim.x;
  const int num_kb = (p.C + kBlockC - 1) / kBlockC;
  const int has_lora = p.lora_r > 0 ? 1 : 0;
  // this CTA's cursor range: unit indices (split-K) or token-rows of the output strip (range schedule)
  const int cur0 = sched.ksplit > 1 ? int(blockIdx.x) : sched.start[blockIdx.x];
  const int cur_end = sched.ksplit > 1 ? sched.n_work : sched.start[blockIdx.x + 1];

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nprob; ++i) {
      ptx::tma_prefetch_desc(&maps.in[i]);
      if (has_lora) {
        ptx::tma_prefetch_desc(&maps.u[i]);
        ptx::tma_prefetch_desc(&maps.v[i]);
      }
    }
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(full_in(s), 1);
      ptx::mbar_init(full_a(s), kGroupWarps);
      ptx::mbar_init(empty(s), kConsumerWarps);
    }
    for (int g = 0; g < kNumGroups; ++g) ptx::mbar_init(lora_bar(g), 1);
    ptx::fence_barrier_init();
  }
  if (kNested && threadIdx.x < 256) {
    // the codebooks are part of the frozen quantization state: never written by a preceding kernel, safe before the PDL wait
    for (int i = 0; i < p.nprob; ++i) s_code[i * 256 + threadIdx.x] = __ldg(p.pr[i].code256 + threadIdx.x);
  }
  __syncthreads();
  ptx::grid_dep_launch();

  if (warp >= kFirstDequantWarp) {
    // ===================== dequantizers (kNumGroups groups) =====================
    const int dw = warp - kFirstDequantWarp;
    const int group = dw >> 2;                           // takes steps g = group, group + kNumGroups, ...
    const int t = (dw & 3) * 32 + lane;                  // 0..127 within the group
    float offs0 = 0.0f, offs1 = 0.0f, offs2 = 0.0f;
    if (kNested) {
      offs0 = __ldg(p.pr[0].offset);
      if (p.nprob > 1) offs1 = __ldg(p.pr[1].offset);
      if (p.nprob > 2) offs2 = __ldg(p.pr[2].offset);
    }
    // a row scale is the output of an earlier kernel, unlike the frozen NF4 state: scaled launches give up the prologue overlap
    if (p.pr[0].row_scale != nullptr || (p.nprob > 1 && p.pr[1].row_scale != nullptr) ||
        (p.nprob > 2 && p.pr[2].row_scale != nullptr))
      ptx::grid_dep_wait();
    const int kblocks_per_row = p.K >> 6;
    int r;
    uint32_t st_base;
    if (!kTrans) {
      r = t;                                             // feature row of this thread's NF4 block
      st_base = uint32_t(r * 128);
    } else {
      r = t & 63;                                        // contraction row (n index) within the step
      const uint32_t hb = uint32_t(t >> 6);              // which 64-feature half (= MN atom of the A tile)
      st_base = hb * 8192u + uint32_t((r >> 3) * 1024 + (r & 7) * 128);
    }
    const int64_t row_bytes = int64_t(p.K >> 1);
    // 32 B of packed nibbles (one NF4 block) of step kb for this thread, straight from global/L2 (16 B aligned: K % 64 == 0)
    auto w_ptr = [&](const uint8_t* packed, int f0, int kb) -> const uint4* {
      if (!kTrans) return reinterpret_cast<const uint4*>(packed + int64_t(f0 + r) * row_bytes + int64_t(kb) * 32);
      const int n = kb * kBlockC + r;
      const int kcol = f0 + (t >> 6) * 64;
      return reinterpret_cast<const uint4*>(packed + int64_t(n) * row_bytes + (kcol >> 1));
    };
    const uint32_t st_xor = uint32_t(r & 7);
    auto blk_of = [&](int f0, int kb) -> int64_t {
      if (!kTrans) return int64_t(f0 + r) * kblocks_per_row + kb;
      const int n = kb * kBlockC + r;
      const int kcol = f0 + (t >> 6) * 64;
      return int64_t(n) * kblocks_per_row + (kcol >> 6);
    };
    // Iterator over this group's steps (global step g = group, group + kNumGroups, ...) across the CTA's units: (seg, i) = segment
    // and step-in-segment inside the current unit `u` (i < u.nkb: NF4 step kb = u.kb0 + i, i == u.nkb: the segment's LoRA
    // step).  Units are decoded only when the cursor moves to the next one.
    int cur = cur0, seg = 0, i = 0;
    uint32_t lora_cnt = 0;                   // LoRA steps this group has handled (phase of its lora_bar)
    Work u{};
    int per = 1;
    bool fresh = true;                       // (unit, segment) changed since the last prefetch: recompute the load addresses
    auto advance = [&](int n) {
      i += n;
      while (true) {
        while (i >= per && seg < u.nseg) {
          i -= per;
          ++seg;
          fresh = true;
        }
        if (seg < u.nseg) return;
        cur = u.next;                        // past the end of the unit: i steps into the next one
        if (cur >= cur_end) return;
        u = decode_work(cur, cur_end, num_ctas, sched, p, num_kb, has_lora);
        per = u.nkb + u.lora;
        seg = 0;
        fresh = true;
      }
    };
    if (cur < cur_end) {
      u = decode_work(cur, cur_end, num_ctas, sched, p, num_kb, has_lora);
      per = u.nkb + u.lora;
      advance(group);
    }
    AbsmaxFetch<kNested> fetch;
    bool valid_cur = false;
    int pi_cur = 0;
    const float* rs_ptr = nullptr;           // row scale of the current problem (null: unscaled)
    float rs_cur = 1.0f;
    uint4 raw0 = make_uint4(0, 0, 0, 0), raw1 = make_uint4(0, 0, 0, 0);   // nibbles of the step this group handles next
    // Global loads of the group's next step (iterator already advanced).  Issued right AFTER the step's fence.proxy.async +
    // arrive.  Addresses advance incrementally (kNumGroups contraction steps per turn) and are recomputed only when the unit
    // or segment changes.
    const uint4* wp_next = nullptr;
    int64_t blk_next = 0;
    int kb_prev = 0;
    const int64_t wp_stride = kTrans ? int64_t(kBlockC) * row_bytes : int64_t(32);          // bytes per contraction step
    const int64_t blk_stride = kTrans ? int64_t(kBlockC) * kblocks_per_row : int64_t(1);    // NF4 blocks per contraction step
    auto prefetch_step = [&]() {
      if (cur >= cur_end || i >= u.nkb) return;             // nothing left / LoRA step: no NF4 data
      const int kb = u.kb0 + i;
      if (fresh) {
        pi_cur = p.group_sum ? seg : u.prob;
        rs_ptr = p.pr[pi_cur].row_scale;
        wp_next = w_ptr(p.pr[pi_cur].packed, u.f0, kb);
        blk_next = blk_of(u.f0, kb);
        fresh = false;
      } else {
        const int dk = kb - kb_prev;
        wp_next = reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(wp_next) + dk * wp_stride);
        blk_next += dk * blk_stride;
      }
      kb_prev = kb;
      if (!kTrans)
        valid_cur = (u.f0 + r) < p.N;
      else
        valid_cur = (kb * kBlockC + r) < p.N && (u.f0 + (t >> 6) * 64) < p.K;
      fetch.issue(p.pr[pi_cur], blk_next, valid_cur);
      if (rs_ptr != nullptr) rs_cur = valid_cur ? __ldg(rs_ptr + (kTrans ? kb * kBlockC + r : u.f0 + r)) : 0.0f;
      raw0 =valid_cur ? __ldg(wp_next) : make_uint4(0, 0, 0, 0);
      raw1 = valid_cur ? __ldg(wp_next + 1) : make_uint4(0, 0, 0, 0);
    };
    prefetch_step();
    for (uint32_t g = uint32_t(group); cur < cur_end; g += kNumGroups) {
      const int sa = int(g % kStages);
      const uint32_t empty_ph = ((g / kStages) & 1) ^ 1;
      if (i < u.nkb) {
        const float offset = pi_cur == 0 ? offs0 : (pi_cur == 1 ? offs1 : offs2);
        float am = fetch.resolve(s_code + pi_cur * 256, offset, valid_cur);
        if (rs_ptr != nullptr) am = __fmul_rn(am, rs_cur);
        Nf4Table tab;
        build_table<T16, kStateF16>(am, tab);
        const uint32_t words[8] = {raw0.x, raw0.y, raw0.z, raw0.w, raw1.x, raw1.y, raw1.z, raw1.w};
        ptx::mbar_wait(empty(sa), empty_ph);
        const uint32_t dst = a_tile(sa) + st_base;
        if (!(p.debug & 1))
#pragma unroll
          for (int w8 = 0; w8 < 8; ++w8) {
            const uint4 o = dequant_word(words[w8], tab);
            asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(dst + ((uint32_t(w8) ^ st_xor) << 4)), "r"(o.x),
                         "r"(o.y), "r"(o.z), "r"(o.w)
                         : "memory");
          }
        ptx::fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(full_a(sa));
      } else {
        // LoRA step: the A-operand tile is plain T16 (V rows of this unit's 128 features x r), TMA'd straight into the A
        // slot in the same canonical layout the dequantizers produce (K-major fwd / MN-major dX).
        const int lora_pi = p.group_sum ? seg : u.prob;
        ptx::mbar_wait(empty(sa), empty_ph);
        if (t == 0) {
          ptx::grid_dep_wait();   // the adapters are written by the optimizer step
          ptx::mbar_arrive_expect_tx(lora_bar(group), kATileBytes);
          if (!kTrans) {
            ptx::tma_load_2d(a_tile(sa), &maps.v[lora_pi], lora_bar(group), 0, u.f0);                   // V[F, r]: box {64, 128}
          } else {
            ptx::tma_load_2d(a_tile(sa), &maps.v[lora_pi], lora_bar(group), u.f0, 0);                   // Vt[r, F]: 2 x box {64, 64}
            ptx::tma_load_2d(a_tile(sa) + 8192u, &maps.v[lora_pi], lora_bar(group), u.f0 + 64, 0);
          }
        }
        ptx::mbar_wait(lora_bar(group), lora_cnt & 1u);
        ++lora_cnt;
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(full_a(sa));
      }
      if (t == 0) {
        // this step's activation block (LoRA step: U[T, r], columns >= r zero-filled); the box is always 128 rows: rows past
        // T are zero-filled, rows past the unit are loaded but not multiplied.  Issued after the A tile so that the first
        // steps' dequantization overlaps the previous kernel; the slot is free (empty[sa] was waited for above).
        ptx::grid_dep_wait();   // activations / U come from earlier kernels
        const int pi = p.group_sum ? seg : u.prob;
        const bool lora_step = i >= u.nkb;
        ptx::mbar_arrive_expect_tx(full_in(sa), kInSlotBytes);
        ptx::tma_load_2d(in_tile(sa), lora_step ? &maps.u[pi] : &maps.in[pi], full_in(sa), lora_step ? 0 : (u.kb0 + i) * kBlockC,
                         u.t0);
      }
      advance(kNumGroups);
      prefetch_step();      // loads of this group's next step fly while the other groups run
    }
  } else {
    // ===================== consumers: two warpgroups, wgmma + output =====================
    const int wg = warp >> 2;
    uint32_t g = 0;
    float acc[ptx::kWgmmaMaxAcc];
#pragma unroll
    for (int i = 0; i < ptx::kWgmmaMaxAcc; ++i) acc[i] = 0.0f;
    for (int a = cur0; a < cur_end;) {
      const Work w = decode_work(a, cur_end, num_ctas, sched, p, num_kb, has_lora);
      a = w.next;
      switch (w.nt >> 4) {
        case 1: consume_unit<T16, 16, kTrans, kOutF16>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
        case 2: consume_unit<T16, 32, kTrans, kOutF16>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
        case 3: consume_unit<T16, 48, kTrans, kOutF16>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
        case 4: consume_unit<T16, 64, kTrans, kOutF16>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
        case 5: consume_unit<T16, 80, kTrans, kOutF16>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
        case 6: consume_unit<T16, 96, kTrans, kOutF16>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
        case 7: consume_unit<T16, 112, kTrans, kOutF16>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
        default: consume_unit<T16, 128, kTrans, kOutF16>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
      }
    }
  }
}

// =====================================================================================================================
// TMA-fed GEMM over a bf16 copy of the weights (DESIGN.md 4.1): the scratch path of training token counts.
//
// At T >= the scratch threshold the host first writes W_p as bf16 [N, K] into a caller-lent scratch with the bit-exact
// table kernel (nf4_quant.cu, once per problem and call) and then launches this kernel, so each weight is dequantized once
// per call instead of once per 128-token unit.  Both operands arrive by TMA and the tensor core sets the pace.
//
// Units are 128 features x up to 256 tokens (wgmma m64nNk16, N <= 256, one M=64 half per consumer warpgroup), with the same
// LoRA step, grouped forms and epilogue as the fused kernel above; the A tile of a step is the same 16 KB K-major (forward)
// or MN-major (dX) tile the dequantizers build, loaded from the scratch instead.  Each output element sums the same products
// in the same order (NF4 steps in order, then the LoRA step) as the fused kernel.
//
// Schedule (sc::Sched, host: launch_scratch_gemm).  The units are the 256-token tiles of the n_fb x T strip, numbered
// feature-block-major with the token tile fastest.  CTA c runs units c, c + P, c + 2P, ... (P = gridDim.x) for the full
// rounds, so the P units in flight cover about P / n_tt consecutive feature blocks: each 128 x C weight tile is read by
// n_tt CTAs at about the same time and can stay in L2 between them, instead of coming from HBM once per token tile (a
// contiguous range per CTA puts the P concurrent units on P different weight tiles, more than L2 holds at C = 4096).  The
// rest of the strip is cut into token ranges, one per CTA, by the host's range planner, which balances them against each
// CTA's round cost (plan_scratch).
//
// Roles (384 threads): warps 0-7 two consumer warpgroups (setmaxnreg 232: 128 accumulators of m64n256) | warps 8-11 the
// producer warpgroup (setmaxnreg 40), whose first thread issues every TMA.
// Barriers: full[s] arrive.expect_tx by the producer + TMA complete_tx of the A and activation tiles -> consumers;
//           empty[s] 8 consumer-warp arrivals once the step's wgmma group has completed -> producer.
// Programmatic dependent launch: the producer waits (griddepcontrol.wait) before its first load (the scratch is the output
// of the dequant kernel launched just before), the consumers before their first output store.
namespace sc {
constexpr int kUnitT = 256;                                 // max tokens per unit (wgmma N)
constexpr int kInSlotBytes = kUnitT * kBlockC * 2;          // 32 KB: one activation block
constexpr int kStages = 4;                                  // 4 x (16 KB A + 32 KB activations)
constexpr int kSmemTiles = kStages * (kInSlotBytes + kATileBytes);   // 192 KB
constexpr int kSmemBytes = kSmemTiles + 1024 + 1024;        // + barriers, + 1 KB alignment of the swizzled tiles
constexpr int kConsumerWarps = 8;
constexpr int kNumThreads = 32 * (kConsumerWarps + 4);      // 384
constexpr int kConsumerRegs = 232;
constexpr int kProducerRegs = 40;
static_assert(2 * 128 * kConsumerRegs + 128 * kProducerRegs <= 65536, "register split exceeds the register file");

struct Maps {
  CUtensorMap in[kMaxProb];   // activations In_p[T, C], box {64, 256}
  CUtensorMap u[kMaxProb];    // LoRA U_p[T, r], box {64, 256}
  CUtensorMap v[kMaxProb];    // LoRA V_p: [F, r] forward, [r, F] dX (as in wg::Maps)
  CUtensorMap w[kMaxProb];    // bf16 W_p[N, K] in the scratch: box {64, 128} forward (K-major A), {64, 64} dX (MN-major A)
};

// A CTA's cursor is a token-row of the strip: below tail0 it is the first row of one of its round units, from tail0 on it
// walks the CTA's tail range.  Both rise monotonically, since the tail holds the strip's last units.
struct Sched {
  int t_pad;                     // T rounded up to a multiple of 16
  int n_tt;                      // 256-token tiles per feature block
  int n_rr;                      // units of the full rounds (a multiple of the CTA count)
  int tail0;                     // first token-row of unit n_rr, where the tail begins
  int start[kMaxCtas + 1];       // tail: CTA c owns token-rows [start[c], start[c+1]) of the strip
  static constexpr int ksplit = 1;   // no split-K (store_unit)
};

// First token-row of unit u.
__device__ __forceinline__ int unit_row(int u, const Sched& sched) {
  return (u / sched.n_tt) * sched.t_pad + (u % sched.n_tt) * kUnitT;
}

// Decode the unit at cursor `a` of a CTA whose tail range ends at `end`.
__device__ __forceinline__ Work decode_work(int a, int end, const Sched& sched, const Params& p, int num_kb, int has_lora) {
  Work w;
  const int fbg = a / sched.t_pad;
  w.t0 = a - fbg * sched.t_pad;
  int ntok = sched.t_pad - w.t0;
  if (ntok > kUnitT) ntok = kUnitT;
  if (a < sched.tail0) {         // a round unit: the CTA's next one is gridDim.x units further on, or its tail
    const int u = fbg * sched.n_tt + w.t0 / kUnitT + int(gridDim.x);
    w.next = u < sched.n_rr ? unit_row(u, sched) : sched.start[blockIdx.x];
  } else {
    if (end - a < ntok) ntok = end - a;
    w.next = a + ntok;
  }
  w.nt = ntok;
  int fb = fbg;
  w.prob = 0;
  w.nseg = p.group_sum ? p.nprob : 1;
  if (!p.group_sum && p.nprob > 1) {
    const int n_fb = (p.F + kUnitF - 1) / kUnitF;
    w.prob = fbg / n_fb;
    fb = fbg - w.prob * n_fb;
  }
  w.f0 = fb * kUnitF;
  w.split = 0;
  w.kb0 = 0;
  w.nkb = num_kb;
  w.lora = has_lora;
  return w;
}

// Consumer warpgroup `wg`: all steps of one unit with wgmma N = kN (>= the unit's tokens), then the output stores.
template <int kN, bool kTrans>
__device__ __forceinline__ void consume_unit(const Work& w, const Params& p, const Sched& sched, int wg, int warp, int lane,
                                             uint32_t smem_base, uint32_t aux, uint32_t& g, float (&acc)[ptx::kWgmmaWideAcc]) {
  auto in_tile = [&](int s) { return smem_base + uint32_t(s) * kInSlotBytes; };
  auto a_tile = [&](int s) { return smem_base + uint32_t(kStages) * kInSlotBytes + uint32_t(s) * kATileBytes; };
  auto full = [&](int s) { return aux + 8u * uint32_t(s); };
  auto empty = [&](int s) { return aux + 8u * uint32_t(kStages + s); };
  const int nsteps = w.nseg * (w.nkb + w.lora);
  for (int kb = 0; kb < nsteps; ++kb, ++g) {
    const int s = int(g % kStages);
    ptx::mbar_wait(full(s), (g / kStages) & 1);
    const uint32_t a_addr = a_tile(s) + uint32_t(wg) * 8192u;
    const uint64_t a_desc = kTrans ? make_desc_mnmajor_sw128(a_addr, 8192, 1024) : make_desc_kmajor_sw128(a_addr);
    const uint64_t b_desc = make_desc_kmajor_sw128(in_tile(s));
    if (!(p.debug & 2)) {
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockC / kMmaK; ++k) {
        const uint64_t a_adv = kTrans ? uint64_t((k * 2 * 1024) >> 4) : uint64_t((k * kMmaK * 2) >> 4);
        const uint64_t b_adv = uint64_t((k * kMmaK * 2) >> 4);
        ptx::wgmma<__nv_bfloat16, kN, kTrans ? 1 : 0>(acc, a_desc + a_adv, b_desc + b_adv, (kb | k) != 0 ? 1u : 0u);
      }
      ptx::wgmma_commit();
    }
    if (kb > 0) {                 // the previous step's group is complete: release its slot
      ptx::wgmma_wait<1>(acc);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(empty(int((g - 1) % kStages)));
    }
  }
  ptx::wgmma_wait<0>(acc);
  __syncwarp();
  if (lane == 0) ptx::mbar_arrive(empty(int((g - 1) % kStages)));
  store_unit<__nv_bfloat16, kN, false>(w, p, sched, wg, warp, lane, acc);
}

template <bool kTrans>
__global__ void __launch_bounds__(kNumThreads, 1)
nf4_scratch_gemm_kernel(const __grid_constant__ Maps maps, const __grid_constant__ Params p, const __grid_constant__ Sched sched) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  auto in_tile = [&](int s) { return smem_base + uint32_t(s) * kInSlotBytes; };
  auto a_tile = [&](int s) { return smem_base + uint32_t(kStages) * kInSlotBytes + uint32_t(s) * kATileBytes; };
  const uint32_t aux = smem_base + uint32_t(kSmemTiles);
  auto full = [&](int s) { return aux + 8u * uint32_t(s); };
  auto empty = [&](int s) { return aux + 8u * uint32_t(kStages + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_kb = (p.C + kBlockC - 1) / kBlockC;
  const int has_lora = p.lora_r > 0 ? 1 : 0;
  const int cur0 = sched.n_rr > 0 ? unit_row(int(blockIdx.x), sched) : sched.start[blockIdx.x];
  const int cur_end = sched.start[blockIdx.x + 1];

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nprob; ++i) {
      ptx::tma_prefetch_desc(&maps.in[i]);
      ptx::tma_prefetch_desc(&maps.w[i]);
      if (has_lora) {
        ptx::tma_prefetch_desc(&maps.u[i]);
        ptx::tma_prefetch_desc(&maps.v[i]);
      }
    }
    for (int s = 0; s < kStages; ++s) {
      ptx::mbar_init(full(s), 1);
      ptx::mbar_init(empty(s), kConsumerWarps);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::grid_dep_launch();

  if (warp >= kConsumerWarps) {
    // ===================== producer =====================
    ptx::setmaxnreg_dec<kProducerRegs>();
    if (warp == kConsumerWarps && ptx::elect_one()) {
      ptx::grid_dep_wait();   // the scratch, the activations and the adapters are outputs of earlier kernels
      uint32_t g = 0;
      for (int a = cur0; a < cur_end;) {
        const Work w = decode_work(a, cur_end, sched, p, num_kb, has_lora);
        a = w.next;
        for (int seg = 0; seg < w.nseg; ++seg) {
          const int pi = p.group_sum ? seg : w.prob;
          for (int i = 0; i < w.nkb + w.lora; ++i, ++g) {
            const int s = int(g % kStages);
            ptx::mbar_wait(empty(s), ((g / kStages) & 1) ^ 1);
            ptx::mbar_arrive_expect_tx(full(s), kATileBytes + kInSlotBytes);
            // A: the step's 128 features x 64 contraction of W (or the unit's LoRA V tile), in the consumers' layout
            const bool lora = i >= w.nkb;
            const CUtensorMap* am = lora ? &maps.v[pi] : &maps.w[pi];
            const int c = lora ? 0 : (w.kb0 + i) * kBlockC;
            if (!kTrans) {
              ptx::tma_load_2d(a_tile(s), am, full(s), c, w.f0);
            } else {
              ptx::tma_load_2d(a_tile(s), am, full(s), w.f0, c);
              ptx::tma_load_2d(a_tile(s) + 8192u, am, full(s), w.f0 + 64, c);
            }
            // activations (LoRA step: U); the box is always 256 rows, rows past T zero-filled, rows past the unit unused
            ptx::tma_load_2d(in_tile(s), lora ? &maps.u[pi] : &maps.in[pi], full(s), c, w.t0);
          }
        }
      }
    }
  } else {
    // ===================== consumers: two warpgroups, wgmma + output =====================
    ptx::setmaxnreg_inc<kConsumerRegs>();
    const int wg = warp >> 2;
    uint32_t g = 0;
    float acc[ptx::kWgmmaWideAcc];
#pragma unroll
    for (int i = 0; i < ptx::kWgmmaWideAcc; ++i) acc[i] = 0.0f;
    for (int a = cur0; a < cur_end;) {
      const Work w = decode_work(a, cur_end, sched, p, num_kb, has_lora);
      a = w.next;
      // N: the unit's tokens rounded up to 16 up to 128, to 32 above
      if (w.nt <= 128) {
        switch (w.nt >> 4) {
          case 1: consume_unit<16, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          case 2: consume_unit<32, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          case 3: consume_unit<48, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          case 4: consume_unit<64, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          case 5: consume_unit<80, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          case 6: consume_unit<96, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          case 7: consume_unit<112, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          default: consume_unit<128, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
        }
      } else {
        switch ((w.nt + 31) >> 5) {
          case 5: consume_unit<160, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          case 6: consume_unit<192, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          case 7: consume_unit<224, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
          default: consume_unit<256, kTrans>(w, p, sched, wg, warp, lane, smem_base, aux, g, acc); break;
        }
      }
    }
  }
}

}  // namespace sc
}  // namespace wg
}  // namespace gemm
}  // namespace qb200
