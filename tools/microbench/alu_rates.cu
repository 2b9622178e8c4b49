// Issue rates of the integer instructions the NF4 look-up is made of, per SM and clock, on the GPU this runs on.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench/alu_rates tools/microbench/alu_rates.cu
// Each kernel runs kIters x 32 independent instructions of one kind per thread (8 accumulators x 4), with enough warps
// (1..8 per SM sub-partition) to saturate the pipe; rate = warp instructions x 32 lanes / (SM cycles).
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

constexpr int kIters = 2048;

template <int OP>
__global__ void rate_kernel(uint32_t* out, uint32_t seed, long long* cycles) {
  uint32_t a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = seed * (threadIdx.x + 1) + i * 0x9E3779B9u;
  uint32_t s0 = seed ^ 0x3210u, s1 = seed | 0x7654u;
  float f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = 1.0f + float(a[i] & 1023) * 1e-6f;
  const long long t0 = clock64();
  for (int it = 0; it < kIters; ++it) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (OP == 0) asm volatile("prmt.b32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(s0), "r"(s1));            // PRMT, register selector
        if (OP == 1) asm volatile("prmt.b32 %0, %0, %1, 0x4051;" : "+r"(a[i]) : "r"(s0));                  // PRMT, immediate selector
        if (OP == 2) asm volatile("lop3.b32 %0, %0, %1, %2, 0xEA;" : "+r"(a[i]) : "r"(s0), "r"(s1));       // LOP3
        if (OP == 3) asm volatile("shf.r.wrap.b32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(s0), "r"(s1));        // SHF
        if (OP == 4) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(s0), "r"(s1));            // IMAD
        if (OP == 5) asm volatile("mul.rn.f32 %0, %0, %1;" : "+f"(f[i]) : "f"(1.0000001f));                  // FMUL
        if (OP == 6) asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(s1));                          // IMAD.HI
        if (OP == 7) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(s1));                             // IADD3
        if (OP == 8) asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(a[i]) : "f"(f[i]), "f"(__uint_as_float(a[i])));   // F2FP pack
      }
    }
  }
  const long long t1 = clock64();
  uint32_t acc = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) acc += a[i] + __float_as_uint(f[i]);
  if (acc == 0x12345678u) out[0] = acc;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int OP>
static void run(const char* name, int sms) {
  uint32_t* out;
  long long* cyc;
  cudaMalloc(&out, 4);
  cudaMalloc(&cyc, sizeof(long long) * sms);
  for (int warps_per_smsp : {1, 2, 4, 8}) {
    const int threads = 32 * 4 * (warps_per_smsp > 8 ? 8 : warps_per_smsp);
    const int ctas_per_sm = warps_per_smsp > 8 ? 2 : 1;
    rate_kernel<OP><<<sms * ctas_per_sm, threads>>>(out, 12345u, cyc);   // warm-up
    cudaDeviceSynchronize();
    long long* h = new long long[sms * ctas_per_sm];
    cudaFree(cyc);
    cudaMalloc(&cyc, sizeof(long long) * sms * ctas_per_sm);
    rate_kernel<OP><<<sms * ctas_per_sm, threads>>>(out, 12345u, cyc);
    cudaDeviceSynchronize();
    cudaMemcpy(h, cyc, sizeof(long long) * sms * ctas_per_sm, cudaMemcpyDeviceToHost);
    double avg = 0;
    for (int i = 0; i < sms * ctas_per_sm; ++i) avg += double(h[i]);
    avg /= sms * ctas_per_sm;
    const double lane_inst_per_sm = double(kIters) * 32.0 * threads * ctas_per_sm;
    printf("{\"op\": \"%s\", \"warps_per_smsp\": %d, \"lanes_per_clk_per_sm\": %.1f}\n", name, warps_per_smsp, lane_inst_per_sm / avg);
    delete[] h;
  }
  cudaFree(out);
  cudaFree(cyc);
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  const int sms = p.multiProcessorCount;
  run<0>("prmt_reg", sms);
  run<1>("prmt_imm", sms);
  run<2>("lop3", sms);
  run<3>("shf", sms);
  run<4>("imad", sms);
  run<5>("fmul", sms);
  run<6>("imad_hi", sms);
  run<7>("iadd", sms);
  run<8>("f2fp_bf16x2", sms);
  return 0;
}
