// Host side of the fused NF4 dequant + wgmma GEMM: TMA tensor maps, range / split-K schedule, launches and the C-ABI
// entry points declared in include/qlora_b200.h.  Kernel: nf4_gemm_wgmma.cuh (one persistent CTA per SM).
//
// Replaces, per Linear4bit call of the reference (SURVEY.md 8a rows a8-a11; qlora.py:249 -> bitsandbytes MatMul4Bit
// [upstream, un-vendored]):  dequantize_blockwise (K3) -> absmax += offset -> dequantize_4bit (K4: bf16 W to HBM) -> cuBLAS
// with ONE kernel in which W never exists in HBM:
//     Out[t, f] = sum_c In[t, c] * Wop[f, c]            t in [0,T)  f in [0,F)  c in [0,C)
//       forward  (kTrans=0):  In = X [M,K],  F = N, C = K, Wop[f,c] = W[f, c]   -> Y  = X . W^T (+bias)
//       backward (kTrans=1):  In = dY[M,N],  F = K, C = N, Wop[f,c] = W[c, f]   -> dX = dY . W
// Roofline: tensor pipe. FLOPs = 2*T*F*C; algorithmic bytes = F*C/2 + F*C/64 + 4*ceil(F*C/16384) + 1028 + 2*T*C + 2*T*F.
#include "nf4_gemm_wgmma.cuh"
#include <math.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <set>

namespace qb200 {
namespace gemm {

using namespace wg;

// ---------------------------------------------------------------- host side -----------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(sym);
  }
  return fn;
}

// cuTensorMapEncodeTiled is a driver-API call and needs a context current on the CALLING thread.  A thread that has made
// no runtime call yet (e.g. torch's autograd worker for device 0 when this library's backward is the first node it runs) has
// none: bind the runtime's primary context of the thread's current device and let the caller retry.
static bool bind_primary_context() { return cudaFree(nullptr) == cudaSuccess; }

static int make_map_2d(CUtensorMap* m, CUtensorMapDataType dt, const void* base, uint64_t inner, uint64_t outer,
                       uint64_t row_pitch_bytes, uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle sw) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return set_error(QB200_EDRIVER, "cuTensorMapEncodeTiled not available from the driver");
  const cuuint64_t dims[2] = {inner, outer};
  const cuuint64_t strides[1] = {row_pitch_bytes};
  const cuuint32_t box[2] = {box_inner, box_outer};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_ERROR_INVALID_CONTEXT && bind_primary_context())
    r = enc(m, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (CUresult %d) inner=%llu outer=%llu pitch=%llu", int(r),
             (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)row_pitch_bytes);
    return set_error(QB200_EDRIVER, buf);
  }
  return 0;
}

// Largest token count served by the warp-level skinny kernel (nf4_gemv.cu) instead of the tensor-core wgmma kernel.
static int skinny_max_m() {
  static int v = env_int("QB200_SKINNY_MAX_M", 16);
  return v;
}

static int debug_flags() {
  static int v = env_int("QB200_DEBUG_FLAGS", 0);
  return v;
}

// SMs of the CURRENT device (the library may serve several GPUs from one process: device_map='auto' in qlora.py); one
// persistent CTA per SM
static int num_ctas() {
  static int ctas[kMaxDevices] = {0};
  const int dev = current_device();
  if (ctas[dev] == 0) {
    ctas[dev] = device_sm_count();
    // QB200_RESERVED_SMS: plan for fewer CTAs than the device has SMs, leaving SMs to kernels that run concurrently
    // (an overlapped NCCL allreduce): the schedule is static, so a launch that does not get all the SMs it planned for needs
    // a whole second round
    static int reserved = env_int("QB200_RESERVED_SMS", 0);
    if (reserved > 0 && ctas[dev] - reserved >= 16) ctas[dev] -= reserved;
    if (ctas[dev] > kMaxCtas) ctas[dev] = kMaxCtas;
  }
  return ctas[dev];
}

// Split-K reduce: out[t, f] = T16( sum_s ws[s, t, f] + bias[f] ), 4 features per thread (float4 loads, 8 B stores).
// kOutF16 (bf16 compute only): out is fp16, the bf16-rounded sum rounded again; out_f32 is not read.
template <typename T16, bool kOutF16>
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ ws, const T16* __restrict__ bias,
                                                            void* __restrict__ out, int64_t ld_out, int out_f32, int64_t TF, int F,
                                                            int ksplit) {
  // programmatic dependent launch: this grid is queued while the GEMM kernel that writes `ws` still runs (its launch
  // latency disappears), waits for that kernel to complete, and lets the next kernel of the stream start its prologue
  ptx::grid_dep_launch();
  ptx::grid_dep_wait();
  const int64_t i4 = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i4 >= TF) return;
  float4 acc = __ldg(reinterpret_cast<const float4*>(ws + i4));
  for (int s2 = 1; s2 < ksplit; ++s2) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(ws + int64_t(s2) * TF + i4));
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  const int64_t t = i4 / F;
  const int f = int(i4 - t * F);
  if (bias != nullptr) {
    acc.x += widen(bias[f]); acc.y += widen(bias[f + 1]);
    acc.z += widen(bias[f + 2]); acc.w += widen(bias[f + 3]);
  }
  uint2 o;
  o.x = round16x2<T16>(acc.x, acc.y);
  o.y = round16x2<T16>(acc.z, acc.w);
  if constexpr (kOutF16) {   // the bf16 pairs widened exactly, then rounded to fp16
    uint2 h;
    h.x = ptx::cvt_f16x2(__uint_as_float(o.x << 16), __uint_as_float(o.x & 0xFFFF0000u));
    h.y = ptx::cvt_f16x2(__uint_as_float(o.y << 16), __uint_as_float(o.y & 0xFFFF0000u));
    *reinterpret_cast<uint2*>(static_cast<__half*>(out) + t * ld_out + f) = h;
  } else if (!out_f32) {
    *reinterpret_cast<uint2*>(static_cast<T16*>(out) + t * ld_out + f) = o;
  } else {   // the T16-rounded sum, widened (Linear4bit called with fp32 activations)
    float4 w;
    if constexpr (std::is_same<T16, __half>::value) {
      const float2 lo = widen2(*reinterpret_cast<const __half2*>(&o.x)), hi = widen2(*reinterpret_cast<const __half2*>(&o.y));
      w = make_float4(lo.x, lo.y, hi.x, hi.y);
    } else {
      w.x = __uint_as_float(o.x << 16); w.y = __uint_as_float(o.x & 0xFFFF0000u);
      w.z = __uint_as_float(o.y << 16); w.w = __uint_as_float(o.y & 0xFFFF0000u);
    }
    *reinterpret_cast<float4*>(static_cast<float*>(out) + t * ld_out + f) = w;
  }
}

// Split-K plan for small token counts: the range schedule gives every CTA a full pass over the contraction, so with T
// tokens per feature block spread over ctas/n_fb CTAs each CTA's MMAs shrink to a few tokens while its dequant work (and
// the fixed cost of a contraction step) stays whole.  Up to QB200_SPLITK_MAX_T tokens, when the 128x128 tiles fill at most
// half of the SMs, every tile's contraction is divided over `ksplit` CTAs instead (>= 4 contraction steps each, at most
// 8 splits).
static int plan_ksplit(int T, int F, int C) {
  static int max_t = env_int("QB200_SPLITK_MAX_T", 768);
  if (T > max_t) return 1;
  const int n_tiles = ((F + kUnitF - 1) / kUnitF) * ((T + kUnitT - 1) / kUnitT);
  const int ctas = num_ctas();
  const int num_kb = (C + kBlockC - 1) / kBlockC;
  if (n_tiles * 2 > ctas) return 1;
  int ks = ctas / n_tiles;
  if (ks > 8) ks = 8;
  if (ks > num_kb / 4) ks = num_kb / 4;
  if (ks < 2) return 1;
  const int per = (num_kb + ks - 1) / ks;
  return (num_kb + per - 1) / per;   // drop empty splits
}

// ---- range schedule -------------------------------------------------------------------------------------------------
// Cost of one unit in SM cycles: every contraction step costs the larger of the dequant period (the dequant groups
// produce one 128 x 64 A tile per `dq` cycles whatever the token count; 1 500 is the period measured inside the 7B training
// step on an H100) and the MMA time (proportional to the tokens: a step is 128 x 64 multiply-adds per token, 4 cycles per
// token at the dense bf16 rate of an H100 SM), plus the output stores and the pipeline refill between units.  The per-unit
// terms are estimates, not fitted; QB200_COST_* override every constant for sweeps.
// The scratch kernel (sc::, 256-token units) has no dequant period: a step costs at least the TMA load of its 16 KB weight
// tile (QB200_COST_SCRATCH_STEP, about 400 cycles of an SM's share of L2 bandwidth; an estimate), else the MMA time.
struct CostModel {
  double dq, per_tok, unit, drain_tok;
};
static const CostModel& cost_model(int unit_t) {
  static CostModel cm = {double(env_int("QB200_COST_DQ", 1500)), env_int("QB200_COST_TOK_X100", 400) / 100.0,
                         double(env_int("QB200_COST_UNIT", 3000)), env_int("QB200_COST_DRAIN_X100", 1200) / 100.0};
  static CostModel cm_scratch = {double(env_int("QB200_COST_SCRATCH_STEP", 400)), cm.per_tok, cm.unit, cm.drain_tok};
  return unit_t == sc::kUnitT ? cm_scratch : cm;
}
static inline double unit_cost(const CostModel& cm, int ntok, int nsteps) {
  const double mma = cm.per_tok * ntok + 24.0;
  return nsteps * (mma > cm.dq ? mma : cm.dq) + cm.unit + cm.drain_tok * ntok;
}

// Greedy walk over the strip from token-row pos0 on with a per-CTA cycle budget, CTA c starting from the load base[c] (null:
// none); returns the CTAs used (start[] filled).
static int walk_ranges(const CostModel& cm, int unit_t, int n_fbg, int t_pad, int nsteps, int pos0, const double* base,
                       double budget, int max_ctas, int* start) {
  const int64_t total = int64_t(n_fbg) * t_pad;
  int64_t pos = pos0;
  int c = 0;
  start[0] = pos0;
  while (pos < total) {
    if (c == max_ctas) return max_ctas + 1;   // does not fit
    double acc = base ? base[c] : 0.0;
    while (pos < total) {
      const int t0 = int(pos % t_pad);
      int maxlen = t_pad - t0;
      if (maxlen > unit_t) maxlen = unit_t;
      if (acc + unit_cost(cm, maxlen, nsteps) <= budget) {
        pos += maxlen;
        acc += unit_cost(cm, maxlen, nsteps);
        continue;
      }
      int len = 0;                                      // largest multiple of 16 that still fits the budget
      for (int l = maxlen - 16; l >= 16; l -= 16)
        if (acc + unit_cost(cm, l, nsteps) <= budget) {
          len = l;
          break;
        }
      if (len == 0 && acc == 0.0) len = 16;             // always make progress
      pos += len;
      break;
    }
    start[++c] = int(pos);
  }
  return c;
}

struct RangeKey {
  int unit_t, n_fbg, t_pad, nsteps, ctas;
  bool operator<(const RangeKey& o) const {
    if (unit_t != o.unit_t) return unit_t < o.unit_t;
    if (n_fbg != o.n_fbg) return n_fbg < o.n_fbg;
    if (t_pad != o.t_pad) return t_pad < o.t_pad;
    if (nsteps != o.nsteps) return nsteps < o.nsteps;
    return ctas < o.ctas;
  }
};
struct RangePlan {
  int n_ctas;
  int start[kMaxCtas + 1];
};

// Balanced contiguous partition of the strip's token-rows from pos0 on over the SMs: the smallest per-CTA budget (bisection)
// for which the greedy walk needs at most `ctas` CTAs, for units of at most `unit_t` tokens (wg::kUnitT or sc::kUnitT), each
// CTA starting from the load base[c] (null: none).  Returns the CTAs used; start[c] for the unused ones is the strip's end.
static int balance_ranges(int unit_t, int n_fbg, int t_pad, int nsteps, int ctas, int pos0, const double* base, int* start) {
  const CostModel& cm = cost_model(unit_t);
  int tmp[kMaxCtas + 2];
  const int64_t total = int64_t(n_fbg) * t_pad;
  double lo = 0.0, hi = 0.0;
  for (int64_t pos = pos0; pos < total;) {
    const int t0 = int(pos % t_pad);
    const int len = (t_pad - t0) < unit_t ? (t_pad - t0) : unit_t;
    hi += unit_cost(cm, len, nsteps);
    pos += len;
  }
  if (base) hi += *std::max_element(base, base + ctas);
  lo = hi / ctas * 0.5;
  for (int iter = 0; iter < 48; ++iter) {
    const double mid = 0.5 * (lo + hi);
    if (walk_ranges(cm, unit_t, n_fbg, t_pad, nsteps, pos0, base, mid, ctas, tmp) <= ctas)
      hi = mid;
    else
      lo = mid;
  }
  const int n_ctas = walk_ranges(cm, unit_t, n_fbg, t_pad, nsteps, pos0, base, hi, ctas, start);
  for (int c = n_ctas + 1; c <= kMaxCtas; ++c) start[c] = start[n_ctas];
  return n_ctas;
}

// The range schedule of the fused kernel, cached per shape (host work at capture time only).
static const RangePlan& plan_ranges(int unit_t, int n_fbg, int t_pad, int nsteps, int ctas) {
  static std::map<RangeKey, RangePlan> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  const RangeKey key{unit_t, n_fbg, t_pad, nsteps, ctas};
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  RangePlan plan{};
  plan.n_ctas = balance_ranges(unit_t, n_fbg, t_pad, nsteps, ctas, 0, nullptr, plan.start);
  return cache.emplace(key, plan).first->second;
}

// Largest planned cost of a CTA whose load base[c] (null: none) is followed by the range [start[c], start[c+1]).
static double plan_peak(const CostModel& cm, int unit_t, int t_pad, int nsteps, int ctas, const double* base, const int* start) {
  double peak = 0.0;
  for (int c = 0; c < ctas; ++c) {
    double acc = base ? base[c] : 0.0;
    for (int pos = start[c]; pos < start[c + 1];) {
      const int t0 = pos % t_pad;
      const int len = std::min({t_pad - t0, unit_t, start[c + 1] - pos});
      acc += unit_cost(cm, len, nsteps);
      pos += len;
    }
    peak = std::max(peak, acc);
  }
  return peak;
}

// The scratch kernel's schedule (sc::Sched, nf4_gemm_wgmma.cuh), cached per shape: full rounds of whole 256-token units,
// round-robin over the CTAs, then the rest of the strip cut into token ranges with each CTA's round cost as its starting
// load.  The range schedule of the whole strip (no rounds) is the yardstick and the fall-back: the most rounds are taken
// for which no CTA's planned cost exceeds that schedule's largest by more than one 16-token step, the resolution of the
// range schedule itself.  Token counts that are a multiple of 256 keep every full round; ragged ones, whose short last
// token tiles load the rounds unevenly, may keep fewer.
struct ScratchPlan {
  int n_ctas;
  sc::Sched sched;
};
static const ScratchPlan& plan_scratch(int n_fbg, int t_pad, int nsteps, int ctas) {
  static std::map<RangeKey, ScratchPlan> cache;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  const RangeKey key{sc::kUnitT, n_fbg, t_pad, nsteps, ctas};
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  const CostModel& cm = cost_model(sc::kUnitT);
  ScratchPlan plan{};
  sc::Sched& s = plan.sched;
  s.t_pad = t_pad;
  s.n_tt = (t_pad + sc::kUnitT - 1) / sc::kUnitT;
  int range_start[kMaxCtas + 1];
  const int range_ctas = balance_ranges(sc::kUnitT, n_fbg, t_pad, nsteps, ctas, 0, nullptr, range_start);
  const double limit = plan_peak(cm, sc::kUnitT, t_pad, nsteps, ctas, nullptr, range_start) + 16 * (cm.per_tok * nsteps + cm.drain_tok);
  for (int rounds = n_fbg * s.n_tt / ctas; rounds > 0; --rounds) {
    s.n_rr = rounds * ctas;
    s.tail0 = (s.n_rr / s.n_tt) * t_pad + (s.n_rr % s.n_tt) * sc::kUnitT;
    double base[kMaxCtas] = {};
    for (int u = 0; u < s.n_rr; ++u) {
      const int t0 = (u % s.n_tt) * sc::kUnitT;
      base[u % ctas] += unit_cost(cm, std::min(t_pad - t0, sc::kUnitT), nsteps);
    }
    balance_ranges(sc::kUnitT, n_fbg, t_pad, nsteps, ctas, s.tail0, base, s.start);
    if (plan_peak(cm, sc::kUnitT, t_pad, nsteps, ctas, base, s.start) <= limit) {
      plan.n_ctas = ctas;   // every CTA runs its rounds, whether or not it gets a piece of the tail
      return cache.emplace(key, plan).first->second;
    }
  }
  s.n_rr = 0;
  s.tail0 = 0;
  memcpy(s.start, range_start, sizeof(s.start));
  plan.n_ctas = range_ctas;
  return cache.emplace(key, plan).first->second;
}

struct GroupArgs {
  int nprob;
  const qb200_nf4_problem* pr;
  int R;
  int M, N, K;
  Nf4Variant v;
  void* workspace;
  int64_t workspace_bytes;
  const float* const* row_scales;   // [nprob] or null; an entry may be null (that problem is unscaled)
};

// The dynamic-shared-memory opt-in of `kern`, made once per (device, kernel): the attribute belongs to the device's context.
static int allow_dynamic_smem(const void* kern, int bytes) {
  static std::mutex mu;
  static std::set<std::pair<int, const void*>> done;
  const std::pair<int, const void*> key{current_device(), kern};
  std::lock_guard<std::mutex> lock(mu);
  if (done.count(key)) return 0;
  const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return set_error(int(e), "cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed");
  done.insert(key);
  return 0;
}

// The strip that the range and scratch schedules cut into units: n_fbg feature blocks (those of every problem, unless the
// problems sum into one output) x t_pad token rows, every unit `nsteps` contraction steps long.
struct Strip {
  int t_pad, n_fbg, nsteps;
};
static int plan_strip(const Params& p, Strip& s) {
  s.t_pad = (p.T + 15) & ~15;
  const int n_fb = (p.F + kUnitF - 1) / kUnitF;
  s.n_fbg = p.group_sum ? n_fb : n_fb * p.nprob;
  if (int64_t(s.n_fbg) * s.t_pad > INT32_MAX) return set_error(QB200_EUNSUPPORTED, "nf4_linear: M x N too large for one launch");
  s.nsteps = (p.group_sum ? p.nprob : 1) * ((p.C + kBlockC - 1) / kBlockC + (p.lora_r + kBlockC - 1) / kBlockC);
  return 0;
}

// Launch parameters and the activation / LoRA tensor maps of a group, shared by both GEMM kernels; activation and U boxes
// are `unit_t` rows (the kernel's largest unit).
template <typename MapsT>
static int fill_launch(const GroupArgs& g, bool trans, int unit_t, MapsT& maps, Params& p) {
  const int T = g.M, F = trans ? g.K : g.N, C = trans ? g.N : g.K;
  const CUtensorMapDataType dt = g.v.kernels == Nf4Kernels::kF16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  p = Params{};
  p.nprob = g.nprob;
  p.group_sum = (trans && g.nprob > 1) ? 1 : 0;
  p.T = T; p.F = F; p.C = C; p.K = g.K; p.N = g.N;
  p.lora_r = g.R;
  p.out_f32 = g.v.out_f32 ? 1 : 0;
  p.debug = debug_flags();
  for (int i = 0; i < g.nprob; ++i) {
    const qb200_nf4_problem& q = g.pr[i];
    const int64_t ld_in = q.ld_in > 0 ? q.ld_in : C;
    int rc = make_map_2d(&maps.in[i], dt, q.in, uint64_t(C), uint64_t(T), uint64_t(ld_in) * 2,
                         kBlockC, unit_t, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    if (g.R > 0) {
      // U[T, r] is a K-major B operand like the activation; V is [F, r] (forward, K-major A operand) or [r, F] (dX, MN-major)
      const int64_t ld_u = q.ld_u > 0 ? q.ld_u : g.R;
      rc = make_map_2d(&maps.u[i], dt, q.U, uint64_t(g.R), uint64_t(T), uint64_t(ld_u) * 2, kBlockC,
                       unit_t, CU_TENSOR_MAP_SWIZZLE_128B);
      if (rc) return rc;
      if (!trans)
        rc = make_map_2d(&maps.v[i], dt, q.V, uint64_t(g.R), uint64_t(F), uint64_t(g.R) * 2, kBlockC,
                         kBlockF, CU_TENSOR_MAP_SWIZZLE_128B);
      else
        rc = make_map_2d(&maps.v[i], dt, q.V, uint64_t(F), uint64_t(g.R), uint64_t(F) * 2, kBlockC,
                         kBlockC, CU_TENSOR_MAP_SWIZZLE_128B);
      if (rc) return rc;
    } else {
      maps.u[i] = maps.in[i];
      maps.v[i] = maps.in[i];
    }
    Prob& d = p.pr[i];
    d.packed = q.packed;
    d.absmax_u8 = q.absmax_u8;
    d.code256 = q.code256;
    d.absmax2 = q.absmax2;
    d.offset = q.offset;
    d.absmax_f32 = q.absmax_u8 ? nullptr : q.absmax_f32;
    d.bias = q.bias;
    d.row_scale = g.row_scales ? g.row_scales[i] : nullptr;
    d.out = p.group_sum ? g.pr[0].out : q.out;
    d.ld_out = (p.group_sum ? g.pr[0].ld_out : q.ld_out) > 0 ? (p.group_sum ? g.pr[0].ld_out : q.ld_out) : F;
  }
  for (int i = g.nprob; i < kMaxProb; ++i) {
    maps.in[i] = maps.in[0];
    maps.u[i] = maps.u[0];
    maps.v[i] = maps.v[0];
    p.pr[i] = p.pr[0];
  }
  return 0;
}

template <bool kTrans>
static int launch_gemm(const GroupArgs& g, cudaStream_t stream) {
  const int T = g.M, F = kTrans ? g.K : g.N, C = kTrans ? g.N : g.K;
  const bool nested = g.pr[0].absmax_u8 != nullptr;
  Maps maps;
  Params p;
  int rc = fill_launch(g, kTrans, kUnitT, maps, p);
  if (rc) return rc;
  const int ctas = num_ctas();
  Sched sched{};
  int n_ctas;
  // split-K only for single problems whose caller lent a large enough fp32 workspace [ksplit, T, F], and whose output the
  // reduce's 4-feature vector stores can reach: F and the row pitch multiples of 4, the base 8-byte (16-bit output) or
  // 16-byte (fp32 output) aligned
  int ksplit = g.nprob == 1 ? plan_ksplit(T, F, C) : 1;
  const uintptr_t out_align = p.out_f32 ? 16 : 8;
  if (ksplit > 1 && (g.workspace == nullptr || g.workspace_bytes < int64_t(ksplit) * T * F * 4 ||
                     reinterpret_cast<uintptr_t>(g.workspace) % 16 != 0 || F % 4 != 0 || p.pr[0].ld_out % 4 != 0 ||
                     reinterpret_cast<uintptr_t>(p.pr[0].out) % out_align != 0))
    ksplit = 1;
  if (ksplit > 1) {
    sched.ksplit = ksplit;
    sched.n_tt = (T + kUnitT - 1) / kUnitT;
    sched.n_work = ((F + kUnitF - 1) / kUnitF) * sched.n_tt * ksplit;
    sched.t_pad = 16;
    n_ctas = sched.n_work < ctas ? sched.n_work : ctas;
    p.ws = static_cast<float*>(g.workspace);
  } else {
    Strip s;
    rc = plan_strip(p, s);
    if (rc) return rc;
    sched.ksplit = 1;
    sched.t_pad = s.t_pad;
    const RangePlan& plan = plan_ranges(kUnitT, s.n_fbg, s.t_pad, s.nsteps, ctas);
    n_ctas = plan.n_ctas;
    memcpy(sched.start, plan.start, sizeof(sched.start));
  }
  return with_nf4_types(g.v.kernels, [&](auto t) {
    using Ty = decltype(t);
    using T16 = typename Ty::T16;
    const auto kern = nested ? nf4_gemm_wgmma_kernel<T16, kTrans, true, Ty::kStateF16, Ty::kOutF16>
                             : nf4_gemm_wgmma_kernel<T16, kTrans, false, Ty::kStateF16, Ty::kOutF16>;
    rc = allow_dynamic_smem(reinterpret_cast<const void*>(kern), kSmemBytes);
    if (rc) return rc;
    rc = launch_pdl(kern, unsigned(n_ctas), kNumThreads, kSmemBytes, stream, kTrans ? "nf4_linear_bwd_dx" : "nf4_linear_fwd", maps,
                    p, sched);
    if (rc || ksplit == 1) return rc;
    const int64_t TF = int64_t(T) * F;
    return launch_pdl(splitk_reduce_kernel<T16, Ty::kOutF16>, unsigned((TF / 4 + 255) / 256), 256, 0, stream, "splitk_reduce",
                      static_cast<const float*>(g.workspace), static_cast<const T16*>(p.pr[0].bias), p.pr[0].out, p.pr[0].ld_out,
                      p.out_f32, TF, F, ksplit);
  });
}

// Smallest token count served by the scratch path (dequantize W once into a bf16 scratch, then the TMA-fed GEMM); smaller
// counts keep the fused kernel.  QB200_SCRATCH_MIN_M overrides it (tests force either path).
static int scratch_min_m() {
  static int v = env_int("QB200_SCRATCH_MIN_M", 1536);
  return v;
}

// Bytes of bf16 weight scratch a call of this shape needs: nprob copies of W [N, K], or 0 below the threshold.
static int64_t scratch_bytes(int64_t nprob, int64_t M, int64_t N, int64_t K) {
  return M >= scratch_min_m() ? nprob * N * K * 2 : 0;
}

// The scratch kernel stores a bf16 output by TMA, which needs a 16-byte aligned base and row pitch: true when every output
// of the call has them (a dX group writes one output), or when the output is fp32 (stored from registers).
static bool out_tma_aligned(int is_bwd, int nprob, const qb200_nf4_problem* probs, int64_t F, bool out_f32) {
  if (out_f32) return true;
  for (int i = 0; i < (is_bwd ? 1 : nprob); ++i) {
    const int64_t ld = probs[i].ld_out > 0 ? probs[i].ld_out : F;
    if (reinterpret_cast<uintptr_t>(probs[i].out) % 16 != 0 || ld % 8 != 0) return false;
  }
  return true;
}

template <bool kTrans>
static int launch_scratch_gemm(const GroupArgs& g, bool w_in_workspace, cudaStream_t stream) {
  sc::Maps maps;
  Params p;
  int rc = fill_launch(g, kTrans, sc::kUnitT, maps, p);
  if (rc) return rc;
  const int64_t w_bytes = int64_t(g.N) * g.K * 2;
  for (int i = 0; i < kMaxProb; ++i) {
    if (i >= g.nprob) {
      maps.w[i] = maps.w[0];
      maps.out[i] = maps.out[0];
      continue;
    }
    // W_p as bf16 [N, K]: box {64, 128} = the K-major forward A tile, {64, 64} = one 64-feature atom of the MN-major dX tile
    const void* w = static_cast<const uint8_t*>(g.workspace) + i * w_bytes;
    rc = make_map_2d(&maps.w[i], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, w, uint64_t(g.K), uint64_t(g.N), uint64_t(g.K) * 2, kBlockC,
                     kTrans ? kBlockC : kBlockF, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    // Out_p as bf16 [T, F]: box {64 features, 16 tokens} = one 16-token slice of a warpgroup's staging tile (the caller
    // guarantees a 16-byte aligned base and pitch: out_tma_aligned); fp32 outputs are stored from registers
    if (p.out_f32) {
      maps.out[i] = maps.in[i];
    } else {
      rc = make_map_2d(&maps.out[i], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, p.pr[i].out, uint64_t(p.F), uint64_t(p.T),
                       uint64_t(p.pr[i].ld_out) * 2, 64, sc::kOutBoxT, CU_TENSOR_MAP_SWIZZLE_128B);
      if (rc) return rc;
    }
  }
  Strip s;
  rc = plan_strip(p, s);
  if (rc) return rc;
  const ScratchPlan& plan = plan_scratch(s.n_fbg, s.t_pad, s.nsteps, num_ctas());
  // w_in_workspace: an earlier call on the same weights left every W_p there (the checkpoint recompute's copy, read again
  // by the dX launch).  QB200_DEBUG_FLAGS bit 16 skips the copies too (wrong results by design: their share of the step).
  if (!w_in_workspace && !(debug_flags() & 16)) {
    for (int i = 0; i < g.nprob; ++i) {
      rc = launch_dequant_scratch(g.pr[i], g.N, g.K, static_cast<uint8_t*>(g.workspace) + i * w_bytes, stream);
      if (rc) return rc;
    }
  }
  const auto kern = sc::nf4_scratch_gemm_kernel<kTrans>;
  rc = allow_dynamic_smem(reinterpret_cast<const void*>(kern), sc::kSmemBytes);
  if (rc) return rc;
  return launch_pdl(kern, unsigned(plan.n_ctas), sc::kNumThreads, sc::kSmemBytes, stream,
                    kTrans ? "nf4_linear_bwd_dx_scratch" : "nf4_linear_fwd_scratch", maps, p, plan.sched);
}

static int validate_shape(int64_t M, int64_t N, int64_t K) {
  if (M <= 0 || N <= 0 || K <= 0 || M > INT32_MAX || N > INT32_MAX || K > INT32_MAX)
    return set_error(QB200_EINVAL, "nf4_linear: bad shape");
  if (K % 64 != 0) return set_error(QB200_EUNSUPPORTED, "nf4_linear: K must be a multiple of 64 (NF4 blocks must not straddle rows)");
  if (N % 8 != 0) return set_error(QB200_EUNSUPPORTED, "nf4_linear: N must be a multiple of 8 (16-byte TMA row pitch)");
  return 0;
}

static int validate_problem(const qb200_nf4_problem& q, int is_bwd, int64_t R, int64_t N, int64_t K, bool need_out) {
  if (!q.in || !q.packed || (need_out && !q.out)) return set_error(QB200_EINVAL, "nf4_linear: null pointer");
  const bool nested = q.absmax_u8 != nullptr;
  if (nested && (!q.code256 || !q.absmax2 || !q.offset)) return set_error(QB200_EINVAL, "nf4_linear: incomplete nested state");
  if (!nested && !q.absmax_f32) return set_error(QB200_EINVAL, "nf4_linear: neither nested nor fp32 absmax given");
  if (reinterpret_cast<uintptr_t>(q.in) % 16 || reinterpret_cast<uintptr_t>(q.packed) % 16)
    return set_error(QB200_EINVAL, "nf4_linear: input and packed weight must be 16-byte aligned");
  const int64_t C = is_bwd ? N : K, F = is_bwd ? K : N;
  if (q.ld_in != 0 && (q.ld_in < C || q.ld_in % 8 != 0)) return set_error(QB200_EINVAL, "nf4_linear: ld_in must be >= the row length and a multiple of 8");
  if (q.ld_out != 0 && q.ld_out < F) return set_error(QB200_EINVAL, "nf4_linear: ld_out must be >= the row length");
  if (is_bwd && q.bias != nullptr) return set_error(QB200_EINVAL, "nf4_linear: bias applies to the forward only");
  if (R != 0) {
    if (!q.U || !q.V) return set_error(QB200_EINVAL, "nf4_linear_lora: null LoRA operand");
    if (reinterpret_cast<uintptr_t>(q.U) % 16 || reinterpret_cast<uintptr_t>(q.V) % 16)
      return set_error(QB200_EINVAL, "nf4_linear_lora: LoRA operands must be 16-byte aligned");
    if (q.ld_u != 0 && (q.ld_u < R || q.ld_u % 8 != 0)) return set_error(QB200_EINVAL, "nf4_linear_lora: ld_u must be >= R and a multiple of 8");
  }
  return 0;
}

}  // namespace gemm
}  // namespace qb200

using namespace qb200;

extern "C" int qb200_has_fused_gemm(void) { return 1; }

// The kernels for compute `dtype` over a quant state of `state_dtype` writing `out_dtype`: the one list of supported
// combinations.  bf16 compute takes a bf16, fp16 or fp32 state and writes bf16, fp32 or fp16; it reads the double-rounded table
// only for an fp16 state (a bf16 or fp32 state gives the table bf16_rn(LUT[j] * absmax)).  fp16 compute takes an fp16 or fp32
// state, whose table is the same, and writes fp16 or fp32.  False for every other combination.
static bool nf4_variant(int dtype, int state_dtype, int out_dtype, Nf4Variant& v) {
  const bool state_f16 = state_dtype == QB200_DTYPE_F16, out_f16 = out_dtype == QB200_DTYPE_F16;
  v.out_f32 = out_dtype == QB200_DTYPE_F32;
  if (dtype == QB200_DTYPE_F16) {
    v.kernels = Nf4Kernels::kF16;
    return (state_f16 || state_dtype == QB200_DTYPE_F32) && (out_f16 || v.out_f32);
  }
  v.kernels = state_f16 ? (out_f16 ? Nf4Kernels::kBf16StateF16OutF16 : Nf4Kernels::kBf16StateF16)
                        : (out_f16 ? Nf4Kernels::kBf16OutF16 : Nf4Kernels::kBf16);
  return dtype == QB200_DTYPE_BF16 && (state_f16 || state_dtype == QB200_DTYPE_F32 || state_dtype == QB200_DTYPE_BF16) &&
         (out_f16 || v.out_f32 || out_dtype == QB200_DTYPE_BF16);
}

// ---- general entry point: 1..3 problems of one shape in ONE launch, each with an optional row scale; 16-bit operands of
// type `dtype` (QB200_DTYPE_BF16 or QB200_DTYPE_F16) over a quant state of `state_dtype`, output of `out_dtype` -----------
// Training token counts (M >= scratch_min_m()) under bf16 compute over a bf16 or fp32 state, with a bf16 or fp32 output and
// no row-scale array, take the scratch path: `workspace` must then hold scratch_bytes() of 32-byte aligned device memory.  A
// bf16 output whose base or row pitch is not 16-byte aligned (TMA stores) runs the fused kernel instead.  fp16
// compute, fp16 states, fp16 outputs and row-scaled launches keep the fused kernel at every token count, as do the four
// entry points without a workspace (fused_only).  w_in_workspace (null: none) is qb200_nf4_linear_group_reuse's flag: in,
// the scratch already holds every W_p; out, this call left every W_p there.
static int linear_group(int is_bwd, int dtype, int state_dtype, int out_dtype, int nprob, const qb200_nf4_problem* probs,
                        const float* const* row_scales, int64_t R, int64_t M, int64_t N, int64_t K, void* workspace,
                        int64_t workspace_bytes, void* stream, bool fused_only = false, int* w_in_workspace = nullptr) {
  const bool reuse = w_in_workspace != nullptr && *w_in_workspace != 0;
  if (w_in_workspace) *w_in_workspace = 0;
  Nf4Variant v;
  if (!nf4_variant(dtype, state_dtype, out_dtype, v))
    return set_error(QB200_EINVAL, "nf4_linear_group_ex: unsupported (dtype, state_dtype, out_dtype): bf16 compute takes a bf16, fp16 "
                                   "or fp32 state and writes bf16, fp32 or fp16; fp16 compute takes an fp16 or fp32 state and "
                                   "writes fp16 or fp32");
  if (!probs || nprob < 1 || nprob > gemm::kMaxProb) return set_error(QB200_EINVAL, "nf4_linear_group: 1..3 problems per launch");
  int rc = gemm::validate_shape(M, N, K);
  if (rc) return rc;
  if (R != 0 && (R < 0 || R > kMaxLoraRank || R % 8 != 0))
    return set_error(QB200_EUNSUPPORTED, "nf4_linear_lora: rank must be a multiple of 8 in [8, 256]");
  const bool nested = probs[0].absmax_u8 != nullptr;
  for (int i = 0; i < nprob; ++i) {
    rc = gemm::validate_problem(probs[i], is_bwd, R, N, K, !(is_bwd && i > 0));
    if (rc) return rc;
    if ((probs[i].absmax_u8 != nullptr) != nested)
      return set_error(QB200_EUNSUPPORTED, "nf4_linear_group: all problems must be nested or all plain");
    if (row_scales && reinterpret_cast<uintptr_t>(row_scales[i]) % 4 != 0)
      return set_error(QB200_EINVAL, "nf4_linear_group_scaled: row scales must be 4-byte aligned fp32");
  }
  const gemm::GroupArgs g{nprob, probs, int(R), int(M), int(N), int(K), v, workspace, workspace_bytes, row_scales};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // forward with at most 16 tokens and a 16-bit output: warp-level skinny kernels (nf4_gemv.cu), SURVEY.md 8f-2 — with LoRA
  // operands too (the reference generates with the adapters attached: base GEMV + peft's two small matmuls; here the U . V^T
  // term is the kernel's epilogue)
  // A grouped forward (q/k/v, gate/up) is nprob launches of them, chained by programmatic dependent launch.
  if (!is_bwd && !v.out_f32 && M <= gemm::skinny_max_m() && !(gemm::debug_flags() & 8)) {
    for (int i = 0; i < nprob; ++i) {
      rc = launch_nf4_skinny(probs[i], row_scales ? row_scales[i] : nullptr, int(M), int(N), int(K), int(R), v.kernels, s);
      if (rc) return rc;
    }
    return 0;
  }
  if (!fused_only && v.kernels == Nf4Kernels::kBf16 && !row_scales && M >= gemm::scratch_min_m() &&
      gemm::out_tma_aligned(is_bwd, nprob, probs, is_bwd ? K : N, v.out_f32)) {
    const int64_t need = gemm::scratch_bytes(nprob, M, N, K);
    if (workspace == nullptr || workspace_bytes < need || reinterpret_cast<uintptr_t>(workspace) % 32 != 0)
      return set_error(QB200_EINVAL, "nf4_linear: this token count needs a 32-byte aligned bf16 weight scratch of "
                                     "qb200_nf4_linear_scratch_size() bytes in `workspace`");
    rc = is_bwd ? gemm::launch_scratch_gemm<true>(g, reuse, s) : gemm::launch_scratch_gemm<false>(g, reuse, s);
    if (rc == 0 && w_in_workspace) *w_in_workspace = (reuse || !(gemm::debug_flags() & 16)) ? 1 : 0;
    return rc;
  }
  return is_bwd ? gemm::launch_gemm<true>(g, s) : gemm::launch_gemm<false>(g, s);
}

extern "C" int qb200_nf4_linear_group_typed(int is_bwd, int dtype, int nprob, const qb200_nf4_problem* probs,
                                            const float* const* row_scales, int64_t R, int64_t M, int64_t N, int64_t K, int out_dtype,
                                            void* workspace, int64_t workspace_bytes, void* stream) {
  Nf4Variant v;
  if (!nf4_variant(dtype, dtype, dtype, v))
    return set_error(QB200_EINVAL, "nf4_linear_group_typed: dtype must be 2 (bf16) or 1 (fp16)");
  if (out_dtype != dtype && out_dtype != QB200_DTYPE_F32)
    return set_error(QB200_EINVAL, dtype == QB200_DTYPE_BF16 ? "nf4_linear_group: out_dtype must be 2 (bf16) or 0 (fp32)"
                                                             : "nf4_linear_group_typed: out_dtype must be 1 (fp16) or 0 (fp32)");
  return linear_group(is_bwd, dtype, dtype, out_dtype, nprob, probs, row_scales, R, M, N, K, workspace, workspace_bytes, stream);
}

extern "C" int qb200_nf4_linear_group(int is_bwd, int nprob, const qb200_nf4_problem* probs, int64_t R, int64_t M, int64_t N,
                                      int64_t K, int out_dtype, void* workspace, int64_t workspace_bytes, void* stream) {
  return qb200_nf4_linear_group_typed(is_bwd, QB200_DTYPE_BF16, nprob, probs, nullptr, R, M, N, K, out_dtype, workspace,
                                      workspace_bytes, stream);
}

extern "C" int qb200_nf4_linear_group_scaled(int is_bwd, int nprob, const qb200_nf4_problem* probs, const float* const* row_scales,
                                             int64_t R, int64_t M, int64_t N, int64_t K, int out_dtype, void* workspace,
                                             int64_t workspace_bytes, void* stream) {
  if (!row_scales) return set_error(QB200_EINVAL, "nf4_linear_group_scaled: null row-scale array (NULL entries mean unscaled)");
  return qb200_nf4_linear_group_typed(is_bwd, QB200_DTYPE_BF16, nprob, probs, row_scales, R, M, N, K, out_dtype, workspace,
                                      workspace_bytes, stream);
}

extern "C" int qb200_nf4_linear_group_ex(int is_bwd, int dtype, int state_dtype, int nprob, const qb200_nf4_problem* probs, int64_t R,
                                         int64_t M, int64_t N, int64_t K, int out_dtype, void* workspace, int64_t workspace_bytes,
                                         void* stream) {
  return linear_group(is_bwd, dtype, state_dtype, out_dtype, nprob, probs, nullptr, R, M, N, K, workspace, workspace_bytes, stream);
}

extern "C" int qb200_nf4_linear_group_reuse(int is_bwd, int dtype, int state_dtype, int nprob, const qb200_nf4_problem* probs,
                                            int64_t R, int64_t M, int64_t N, int64_t K, int out_dtype, void* workspace,
                                            int64_t workspace_bytes, int* w_in_workspace, void* stream) {
  return linear_group(is_bwd, dtype, state_dtype, out_dtype, nprob, probs, nullptr, R, M, N, K, workspace, workspace_bytes, stream,
                      false, w_in_workspace);
}

extern "C" int qb200_nf4_linear_group_mixed(int dtype, int state_dtype, int nprob, const qb200_nf4_problem* probs, int n_adapters,
                                            const int32_t* row_adapter, int64_t R, int64_t M, int64_t N, int64_t K, int out_dtype,
                                            void* stream) {
  Nf4Variant v;
  if (!nf4_variant(dtype, state_dtype, out_dtype, v))
    return set_error(QB200_EINVAL, "nf4_linear_group_mixed: unsupported (dtype, state_dtype, out_dtype), as for nf4_linear_group_ex");
  if (v.out_f32) return set_error(QB200_EUNSUPPORTED, "nf4_linear_group_mixed: 16-bit outputs only");
  if (!probs || nprob < 1 || nprob > gemm::kMaxProb) return set_error(QB200_EINVAL, "nf4_linear_group: 1..3 problems per launch");
  if (!row_adapter || n_adapters < 1) return set_error(QB200_EINVAL, "nf4_linear_group_mixed: null row_adapter or no adapters");
  if (reinterpret_cast<uintptr_t>(row_adapter) % 4) return set_error(QB200_EINVAL, "nf4_linear_group_mixed: row_adapter must be 4-byte aligned");
  int rc = gemm::validate_shape(M, N, K);
  if (rc) return rc;
  if (M > gemm::skinny_max_m()) return set_error(QB200_EUNSUPPORTED, "nf4_linear_group_mixed: skinny token counts only (QB200_SKINNY_MAX_M)");
  if (R < 8 || R > kMaxLoraRank || R % 8 != 0)
    return set_error(QB200_EUNSUPPORTED, "nf4_linear_group_mixed: R must be a multiple of 8 in [8, 256]");
  const bool nested = probs[0].absmax_u8 != nullptr;
  for (int i = 0; i < nprob; ++i) {
    rc = gemm::validate_problem(probs[i], 0, R, N, K, true);
    if (rc) return rc;
    if ((probs[i].absmax_u8 != nullptr) != nested)
      return set_error(QB200_EUNSUPPORTED, "nf4_linear_group: all problems must be nested or all plain");
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  for (int i = 0; i < nprob; ++i) {
    rc = launch_nf4_skinny_mixed(probs[i], row_adapter, n_adapters, int(M), int(N), int(K), int(R), v.kernels, s);
    if (rc) return rc;
  }
  return 0;
}

extern "C" int64_t qb200_nf4_linear_scratch_size(int nprob, int64_t M, int64_t N, int64_t K, int is_bwd) {
  (void)is_bwd;   // the copy is W [N, K] in both directions
  if (nprob < 1 || nprob > gemm::kMaxProb || M <= 0 || N <= 0 || K <= 0 || M > INT32_MAX || N > INT32_MAX || K > INT32_MAX) return 0;
  return gemm::scratch_bytes(nprob, M, N, K);
}

extern "C" int64_t qb200_nf4_linear_workspace_size(int64_t M, int64_t N, int64_t K, int is_bwd) {
  if (M <= 0 || N <= 0 || K <= 0 || M > INT32_MAX || N > INT32_MAX || K > INT32_MAX) return 0;
  const int T = int(M), F = int(is_bwd ? K : N), C = int(is_bwd ? N : K);
  if (F % 4 != 0) return 0;
  if (!is_bwd && M <= gemm::skinny_max_m()) return 0;   // skinny kernels (with or without LoRA operands): no workspace
  const int ks = gemm::plan_ksplit(T, F, C);
  return ks > 1 ? int64_t(ks) * T * F * 4 : 0;
}

// One bf16 problem: the single-problem entry points.  The four that take no workspace pass fused_only: un-split schedule,
// fused kernel at every token count.
static int linear_one(int is_bwd, const void* in, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                      const float* absmax2, const float* offset, const float* absmax_f32, const void* bias, const void* U,
                      const void* V, int64_t R, void* out, int64_t M, int64_t N, int64_t K, void* workspace, int64_t workspace_bytes,
                      void* stream, bool fused_only) {
  qb200_nf4_problem q{};
  q.in = in; q.packed = packed; q.absmax_u8 = absmax_u8; q.code256 = code256; q.absmax2 = absmax2; q.offset = offset;
  q.absmax_f32 = absmax_f32; q.bias = bias; q.U = U; q.V = V; q.out = out;
  return linear_group(is_bwd, QB200_DTYPE_BF16, QB200_DTYPE_BF16, QB200_DTYPE_BF16, 1, &q, nullptr, R, M, N, K, workspace,
                      workspace_bytes, stream, fused_only);
}

extern "C" int qb200_nf4_linear_ex(int is_bwd, const void* in, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                                   const float* absmax2, const float* offset, const float* absmax_f32, const void* bias,
                                   const void* U, const void* V, int64_t R, void* out, int64_t M, int64_t N, int64_t K,
                                   void* workspace, int64_t workspace_bytes, void* stream) {
  return linear_one(is_bwd, in, packed, absmax_u8, code256, absmax2, offset, absmax_f32, bias, U, V, R, out, M, N, K, workspace,
                    workspace_bytes, stream, false);
}

extern "C" int qb200_nf4_linear_fwd(const void* X, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                                    const float* absmax2, const float* offset, const float* absmax_f32, const void* bias,
                                    void* Y, int64_t M, int64_t N, int64_t K, void* stream) {
  return linear_one(0, X, packed, absmax_u8, code256, absmax2, offset, absmax_f32, bias, nullptr, nullptr, 0, Y, M, N, K, nullptr, 0,
                    stream, true);
}

extern "C" int qb200_nf4_linear_bwd_dx(const void* dY, const uint8_t* packed, const uint8_t* absmax_u8,
                                       const float* code256, const float* absmax2, const float* offset,
                                       const float* absmax_f32, void* dX, int64_t M, int64_t N, int64_t K, void* stream) {
  return linear_one(1, dY, packed, absmax_u8, code256, absmax2, offset, absmax_f32, nullptr, nullptr, nullptr, 0, dX, M, N, K, nullptr,
                    0, stream, true);
}

// ---- fused LoRA variants (SURVEY.md 8f-1: the caller's low-rank update folded into the same launch) ------------
extern "C" int qb200_nf4_linear_fwd_lora(const void* X, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                                         const float* absmax2, const float* offset, const float* absmax_f32, const void* bias,
                                         const void* U, const void* V, int64_t R, void* Y, int64_t M, int64_t N, int64_t K,
                                         void* stream) {
  if (R == 0) return set_error(QB200_EINVAL, "nf4_linear_fwd_lora: R must be > 0");
  return linear_one(0, X, packed, absmax_u8, code256, absmax2, offset, absmax_f32, bias, U, V, R, Y, M, N, K, nullptr, 0, stream, true);
}

extern "C" int qb200_nf4_linear_bwd_dx_lora(const void* dY, const uint8_t* packed, const uint8_t* absmax_u8,
                                            const float* code256, const float* absmax2, const float* offset,
                                            const float* absmax_f32, const void* U, const void* Vt, int64_t R, void* dX,
                                            int64_t M, int64_t N, int64_t K, void* stream) {
  if (R == 0) return set_error(QB200_EINVAL, "nf4_linear_bwd_dx_lora: R must be > 0");
  return linear_one(1, dY, packed, absmax_u8, code256, absmax2, offset, absmax_f32, nullptr, U, Vt, R, dX, M, N, K, nullptr, 0, stream,
                    true);
}
