// Internal helpers shared by the translation units of libqlora_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/qlora_b200.h"

namespace qb200 {
// Records a thread-local message and returns `code` (so callers can `return set_error(...)`).
int set_error(int code, const char* msg);
// cudaPeekAtLastError() after a launch -> 0 or the cudaError_t (message recorded).
int check_launch(const char* what);
// Streaming multiprocessors of the calling thread's current device (cached per device); grid sizes are multiples of it.
int device_sm_count();
// Forward skinny GEMM (nf4_gemv.cu) used by qb200_nf4_linear_group for M <= 16, with an optional LoRA term U[M,R] . V[N,R]^T
// and an optional per-row weight scale row_scale[N] (null: none); ld_* are row pitches in elements (0 = dense).
int launch_nf4_skinny(const void* x, int64_t ld_x, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                      const float* absmax2, const float* offset, const float* absmax_f32, const void* bias, void* y, int64_t ld_y,
                      int M, int N, int K, const void* U, int64_t ld_u, const void* V, int R, const float* row_scale,
                      cudaStream_t stream);
}  // namespace qb200
