// Which exact NF4 look-up feeds mma.sync fastest?  Weights per clock per SM for one 64-value block per thread and iteration,
// registers only (no global traffic), the look-up output consumed by 16 HMMAs as in nf4_gemv.cu:
//   method 0: per-block product table (16 x bf16(LUT[j] * absmax) as byte planes), nibbles resolved with PRMT   (production)
//   method 1: constant fp32 LUT in shared memory: nibble -> byte offset -> LDS -> FMUL by absmax -> cvt.rn.bf16x2
//   method 2: half of the words by method 0, half by method 1
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I qlora_b200/csrc -o tools/microbench/lookup_rates tools/microbench/lookup_rates.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#include "nf4_table.cuh"

using namespace qb200;

__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// method 1: 8 nibbles of a word -> 4 bf16x2 words in element order (even element = high nibble of its byte)
__device__ __forceinline__ void lookup8_lds(uint32_t word, uint32_t lut, float am, uint32_t (&w)[4]) {
  const uint32_t lo4 = (word << 2) & 0x3C3C3C3Cu;   // odd elements, x4
  const uint32_t hi4 = (word >> 2) & 0x3C3C3C3Cu;   // even elements, x4
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t oe = ptx::prmt(hi4, 0u, 0x4440u + j), oo = ptx::prmt(lo4, 0u, 0x4440u + j);
    float ve, vo;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(ve) : "r"(lut + oe));
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(vo) : "r"(lut + oo));
    w[j] = ptx::cvt_bf16x2(__fmul_rn(ve, am), __fmul_rn(vo, am));
  }
}

template <int METHOD>
__global__ void __launch_bounds__(128, 4) lookup_kernel(float* out, uint32_t seed, int iters, long long* cycles) {
  __shared__ float s_lut[16];
  constexpr float lutc[16] = QB200_NF4_LUT_INIT;
  if (threadIdx.x < 16) s_lut[threadIdx.x] = lutc[threadIdx.x];
  __syncthreads();
  const uint32_t lut = static_cast<uint32_t>(__cvta_generic_to_shared(s_lut));
  uint32_t words[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) words[i] = (seed + threadIdx.x * 2654435761u) * (i + 3);
  float acc[2][4] = {};
  const uint32_t a0 = 0x3f803f80u, a1 = 0x3f803f80u, a2 = 0x3f803f80u, a3 = 0x3f803f80u;
  float am = 0.01f + float(threadIdx.x) * 1e-5f;
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
    am += 1e-7f;
    Nf4Table tab;
    if (METHOD != 1) build_table(am, tab);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t word = words[j] ^ uint32_t(it * 0x01010101);
      uint32_t w[4];
      if (METHOD == 0 || (METHOD == 2 && (j & 1))) {
        const uint4 o = dequant_word(word, tab);
        w[0] = o.x; w[1] = o.y; w[2] = o.z; w[3] = o.w;
      } else {
        lookup8_lds(word, lut, am, w);
      }
      mma16816(acc[0], a0, a1, a2, a3, w[0], w[2]);
      mma16816(acc[1], a0, a1, a2, a3, w[1], w[3]);
    }
  }
  const long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc[0][0] + acc[0][1] + acc[1][2] + acc[1][3];
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int METHOD>
static void run(const char* name, int sms) {
  const int ctas = sms * 4, iters = 512;
  float* out;
  long long* cyc;
  cudaMalloc(&out, sizeof(float) * ctas * 128);
  cudaMalloc(&cyc, sizeof(long long) * ctas);
  for (int rep = 0; rep < 2; ++rep) lookup_kernel<METHOD><<<ctas, 128>>>(out, 12345u, iters, cyc);
  cudaDeviceSynchronize();
  long long* h = new long long[ctas];
  cudaMemcpy(h, cyc, sizeof(long long) * ctas, cudaMemcpyDeviceToHost);
  double avg = 0;
  for (int i = 0; i < ctas; ++i) avg += double(h[i]);
  avg /= ctas;
  // 4 resident CTAs x 128 threads x 64 weights per iteration per SM
  printf("{\"method\": \"%s\", \"weights_per_clk_per_sm\": %.2f, \"err\": \"%s\"}\n", name, 4.0 * 128 * 64 * iters / avg,
         cudaGetErrorString(cudaGetLastError()));
  delete[] h;
  cudaFree(out);
  cudaFree(cyc);
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  run<0>("prmt_product_table", p.multiProcessorCount);
  run<1>("lds_lut_fmul_cvt", p.multiProcessorCount);
  run<2>("half_and_half", p.multiProcessorCount);
  return 0;
}
