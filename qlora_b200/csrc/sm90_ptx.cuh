// Thin inline-PTX wrappers for the sm_90a features the fused kernel uses:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory descriptors), proxy fences,
// programmatic dependent launch.  Spellings follow the PTX ISA.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace qb200 {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ---------------------------------------------------------------- mbarrier ------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}

// Watchdog'd wait: a protocol bug traps (host sees a launch failure) instead of hanging the GPU.  No printf here: a
// function call anywhere in the kernel makes ptxas serialize the wgmma pipeline.
#ifndef QB200_WATCHDOG_CYCLES
#define QB200_WATCHDOG_CYCLES (4000000000LL)  // ~2 s at 1.98 GHz
#endif
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > QB200_WATCHDOG_CYCLES) __trap();
}

// ---------------------------------------------------------------- proxy fences --------
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------- TMA -----------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap* m, uint32_t bar, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst_smem),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

// Shared -> global tensor store of one box at coordinates {c0, c1}; the box is clipped at the tensor's bounds.  Completion
// is tracked per thread by bulk async-groups: commit after the stores, then wait_group_read before the shared source is
// written again, wait_group before the results must be visible.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src_smem, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(src_smem), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(kPending) : "memory");
}
template <int kPending>
__device__ __forceinline__ void bulk_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(kPending) : "memory");
}

// ---------------------------------------------------------------- shared-memory matrix store, named barrier ----
// Four 8x8 b16 matrices, transposed: lane l supplies the row address of matrix l / 8, row l % 8; register r_k holds the
// lane's pair (row l / 4, columns 2 (l % 4) + {0, 1}) of matrix k, which lands in memory row 2 (l % 4) + {0, 1}, column l / 4.
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2),
               "r"(r3)
               : "memory");
}
// bar.sync over the 128 threads of one warpgroup (id 1.. : barrier 0 is __syncthreads)
__device__ __forceinline__ void bar_sync_warpgroup(uint32_t id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// One lane of a CONVERGED warp (elect.sync): the loop around it stays warp-uniform.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- programmatic dependent launch ----
// griddepcontrol.wait: block until every prerequisite grid of this (programmatically launched) grid has completed and its
// memory is visible; a no-op for a normally launched grid.  launch_dependents: this CTA no longer holds back the launch of
// a dependent grid (which may begin its own prologue while this grid is still running).
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- wgmma ---------------
// D[regs] (+)= A[smem desc] . B[smem desc], bf16 or f16 in, fp32 accumulate, one warpgroup (128 threads) per instruction.
// Accumulator fragment of m64nNk16 (thread t of the warpgroup, warp w = t / 32, lane l): d[4 j + 0, 1] = D[16 w + l / 4,
// 8 j + 2 (l % 4) + {0, 1}], d[4 j + 2, 3] = the same columns of row 16 w + l / 4 + 8.
constexpr int kWgmmaMaxAcc = 64;   // fp32 accumulators per thread of m64n128
constexpr int kWgmmaWideAcc = 128; // fp32 accumulators per thread of m64n256
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending, int kAcc>
__device__ __forceinline__ void wgmma_wait(float (&d)[kAcc]) {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory");
  // the accumulators are written asynchronously: tie them to the wait so no read is scheduled before it
#pragma unroll
  for (int i = 0; i < kAcc; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// setmaxnreg: move registers between the warpgroups of a CTA (every warp of the warpgroup executes it)
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// generated: one wrapper per N = 16, 32, ..., 128 and 160, 192, 224, 256 (the immediate shape); kTnspA = 1 for an MN-major A operand.  The A and B
// type is bf16 or f16 (T16 = __nv_bfloat16 / __half); both read the same shared-memory layouts and accumulate in fp32.
#define QB200_WGMMA_M64N16(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n16k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n16(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N16("f16");
  else QB200_WGMMA_M64N16("bf16");
}
#undef QB200_WGMMA_M64N16
#define QB200_WGMMA_M64N32(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n32k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n32(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N32("f16");
  else QB200_WGMMA_M64N32("bf16");
}
#undef QB200_WGMMA_M64N32
#define QB200_WGMMA_M64N48(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n48k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, %27, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n48(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N48("f16");
  else QB200_WGMMA_M64N48("bf16");
}
#undef QB200_WGMMA_M64N48
#define QB200_WGMMA_M64N64(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n64(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N64("f16");
  else QB200_WGMMA_M64N64("bf16");
}
#undef QB200_WGMMA_M64N64
#define QB200_WGMMA_M64N80(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n80k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, %43, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n80(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N80("f16");
  else QB200_WGMMA_M64N80("bf16");
}
#undef QB200_WGMMA_M64N80
#define QB200_WGMMA_M64N96(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n96k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, %51, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n96(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N96("f16");
  else QB200_WGMMA_M64N96("bf16");
}
#undef QB200_WGMMA_M64N96
#define QB200_WGMMA_M64N112(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n112k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p, 1, 1, %59, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n112(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N112("f16");
  else QB200_WGMMA_M64N112("bf16");
}
#undef QB200_WGMMA_M64N112
#define QB200_WGMMA_M64N128(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n128(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N128("f16");
  else QB200_WGMMA_M64N128("bf16");
}
#undef QB200_WGMMA_M64N128
#define QB200_WGMMA_M64N160(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n160k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, %80, %81, p, 1, 1, %83, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n160(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N160("f16");
  else QB200_WGMMA_M64N160("bf16");
}
#undef QB200_WGMMA_M64N160
#define QB200_WGMMA_M64N192(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n192k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, %99, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n192(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N192("f16");
  else QB200_WGMMA_M64N192("bf16");
}
#undef QB200_WGMMA_M64N192
#define QB200_WGMMA_M64N224(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %114, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n224k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111}, %112, %113, p, 1, 1, %115, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n224(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N224("f16");
  else QB200_WGMMA_M64N224("bf16");
}
#undef QB200_WGMMA_M64N224
#define QB200_WGMMA_M64N256(ty)                                                                                                      \
  asm volatile(                                                                                                              \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"                                                                 \
      "wgmma.mma_async.sync.aligned.m64n256k16.f32." ty "." ty " {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, 0;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127]) \
      : "l"(da), "l"(db), "r"(scale_d), "n"(kTnspA))
template <typename T16, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma_m64n256(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (std::is_same<T16, __half>::value) QB200_WGMMA_M64N256("f16");
  else QB200_WGMMA_M64N256("bf16");
}
#undef QB200_WGMMA_M64N256
template <typename T16, int N, int kTnspA, int kAcc>
__device__ __forceinline__ void wgmma(float (&d)[kAcc], uint64_t da, uint64_t db, uint32_t scale_d) {
  // N = 16..128 for the 64-accumulator fused kernel; the 128-accumulator scratch kernel adds N = 160..256 in steps of 32
  static_assert(N % 16 == 0 && N >= 16 && 2 * kAcc >= N && (N <= 128 || (kAcc == kWgmmaWideAcc && N % 32 == 0)),
                "m64nNk16 with N = 16..128, or N = 160..256 in steps of 32 for the wide accumulator");
  if constexpr (N == 16) wgmma_m64n16<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 32) wgmma_m64n32<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 48) wgmma_m64n48<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 64) wgmma_m64n64<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 80) wgmma_m64n80<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 96) wgmma_m64n96<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 112) wgmma_m64n112<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 128) wgmma_m64n128<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 160) wgmma_m64n160<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 192) wgmma_m64n192<T16, kTnspA>(d, da, db, scale_d);
  else if constexpr (N == 224) wgmma_m64n224<T16, kTnspA>(d, da, db, scale_d);
  else wgmma_m64n256<T16, kTnspA>(d, da, db, scale_d);
}

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}
// d = {hi: bf16(hi_f), lo: bf16(lo_f)}, round-to-nearest-even
__device__ __forceinline__ uint32_t cvt_bf16x2(float lo_f, float hi_f) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi_f), "f"(lo_f));
  return d;
}

__device__ __forceinline__ uint32_t cvt_f16x2(float lo_f, float hi_f) {
  uint32_t d;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi_f), "f"(lo_f));
  return d;
}
}  // namespace ptx
}  // namespace qb200
