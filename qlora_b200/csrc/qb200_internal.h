// Internal helpers shared by the translation units of libqlora_b200.so.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/qlora_b200.h"

namespace qb200 {
// Records a thread-local message and returns `code` (so callers can `return set_error(...)`).
int set_error(int code, const char* msg);
// cudaPeekAtLastError() after a launch -> 0 or the cudaError_t (message recorded).
int check_launch(const char* what);
// Integer value of environment variable `name` (atoi), or `dflt` when it is unset.
int env_int(const char* name, int dflt);
// Per-device caches are indexed by current_device(): the calling thread's current device, 0 if it is unknown or >= kMaxDevices.
constexpr int kMaxDevices = 16;
int current_device();
// Streaming multiprocessors of the current device (cached per device); grid sizes are multiples of it.
int device_sm_count();
// Programmatic dependent launch for every launch_pdl (QB200_PDL=0 disables it: A/B timing).
bool use_pdl();

// Launches kern<<<grid, block, smem, stream>>>(args...) with programmatic stream serialization when use_pdl(): the kernel
// may start its prologue while the previous kernel of the stream still runs.  Returns 0 or the error (message recorded).
template <typename... KArgs, typename... Args>
int launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, const char* what,
               const Args&... args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = use_pdl() ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, args...);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    char msg[160];
    snprintf(msg, sizeof(msg), "%s: cudaLaunchKernelEx failed", what);
    return set_error(int(e), msg);
  }
  return check_launch(what);
}

// The kernels of an NF4 linear launch, one value per set compiled: the 16-bit operand type T16 and, under bf16 compute, the
// weights of an fp16 quant state (kStateF16: bf16_rn(fp16_rn(LUT[j] * absmax))) and an fp16 output (kOutF16: the bf16-rounded
// result rounded to fp16).  fp16 compute reads the same table for an fp16 or fp32 state and has no fp16-output form.
enum class Nf4Kernels { kBf16, kBf16StateF16, kBf16OutF16, kBf16StateF16OutF16, kF16 };

// A launch's kernels plus out_f32: a 16-bit output widened to fp32 (never with kOutF16).
struct Nf4Variant {
  Nf4Kernels kernels;
  bool out_f32;
};

// The compile-time parameters of one Nf4Kernels value.
template <typename T16_, bool kStateF16_, bool kOutF16_>
struct Nf4Types {
  using T16 = T16_;
  static constexpr bool kStateF16 = kStateF16_;
  static constexpr bool kOutF16 = kOutF16_;
};

// fn(Nf4Types<...>{}) for the parameters of `k`: the one place the kernel templates are instantiated from a runtime value.
template <typename Fn>
auto with_nf4_types(Nf4Kernels k, Fn&& fn) {
  using BF = __nv_bfloat16;
  switch (k) {
    case Nf4Kernels::kBf16StateF16: return fn(Nf4Types<BF, true, false>{});
    case Nf4Kernels::kBf16OutF16: return fn(Nf4Types<BF, false, true>{});
    case Nf4Kernels::kBf16StateF16OutF16: return fn(Nf4Types<BF, true, true>{});
    case Nf4Kernels::kF16: return fn(Nf4Types<__half, false, false>{});
    case Nf4Kernels::kBf16: break;
  }
  return fn(Nf4Types<BF, false, false>{});
}

// LoRA ranks of the NF4 linear entry points: multiples of 8 up to this.  The wgmma kernels contract them in one 64-wide step
// per 64 ranks, the skinny kernels in 64-rank chunks of their epilogue.
constexpr int kMaxLoraRank = 256;

// The adapters of a mixed-adapter launch (qb200_lora_project_mixed, qb200_nf4_linear_group_mixed): token m uses table[rows[m]]
// when that index is in [0, n), no adapter otherwise, so no device index can make a kernel read outside the table.
struct MixedLora {
  const int32_t* rows;                 // DEVICE: one adapter index per token
  const qb200_lora_adapter* table;     // DEVICE: n entries
  int n;
  __device__ __forceinline__ const qb200_lora_adapter* adapter(int m) const {
    const int a = rows[m];
    return (a >= 0 && a < n) ? table + a : nullptr;
  }
  // the rank a kernel uses: the entry's, clamped to the `cols` columns of U and down to a multiple of 8 (16-byte rows)
  __device__ __forceinline__ static int rank(const qb200_lora_adapter& ad, int cols) { return max(0, min(ad.rank, cols)) & ~7; }
};

// Forward skinny GEMM (nf4_gemv.cu) used by qb200_nf4_linear_group for M <= 16 and a 16-bit output: problem q with its
// optional LoRA term U[M,R] . V[N,R]^T (R = 0: none) and an optional per-row weight scale row_scale[N] (null: none), run by
// the skinny kernels of `kernels`.
int launch_nf4_skinny(const qb200_nf4_problem& q, const float* row_scale, int M, int N, int K, int R, Nf4Kernels kernels,
                      cudaStream_t stream);

// launch_nf4_skinny with one adapter per token: q.V is the DEVICE adapter table (n_adapters entries), q.U the [M, R] projection
// of qb200_lora_project_mixed, row_adapter the DEVICE index of every token; no row scale.
int launch_nf4_skinny_mixed(const qb200_nf4_problem& q, const int32_t* row_adapter, int n_adapters, int M, int N, int K, int R,
                            Nf4Kernels kernels, cudaStream_t stream);

// dequantize_4bit(W, state) of problem q as bf16 [N, K] into `out` (32-byte aligned) with the table kernel of nf4_quant.cu —
// the weights the fused GEMM builds in shared memory, bit for bit (blocks of 64, nested blocks of 256).  Launched with
// programmatic dependent launch; the scratch GEMM path reads the copy in the next kernel.
int launch_dequant_scratch(const qb200_nf4_problem& q, int64_t N, int64_t K, void* out, cudaStream_t stream);
}  // namespace qb200
