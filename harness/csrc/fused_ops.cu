// Caller-side elementwise fusions for the benchmark harness (NOT part of the qlora_b200 product / C-ABI):
// the decoder layer around the NF4 linears spends ~25 % of a training step in tiny torch elementwise kernels.
//   hops_rope_qk   : RoPE (HF rotate_half form) on q and k in one launch; backward = same kernel with sign = -1
//   hops_swiglu_fwd: silu(gate) * up
//   hops_swiglu_bwd: d_gate, d_up from (gate, up, d_out)
// bf16 in / bf16 out, fp32 math, 16 B vector accesses.  sm_90a.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

__device__ __forceinline__ float lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pack(float a, float b) {
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(b), "f"(a));
  return d;
}

// x: [rows = b*s*h, d] (two tensors q and k, n_q and n_k rows), cos/sin: [s, d]; row -> position s = (row / h) % S.
// y[i] = x[i]*cos[i] + x[i ^ half]*sign*sin_signed[i]    (sin_signed = cat(-sin, sin))
__global__ void __launch_bounds__(256) rope_qk_kernel(const uint4* __restrict__ q, const uint4* __restrict__ k, uint4* __restrict__ qo,
                                                      uint4* __restrict__ ko, const uint4* __restrict__ cosv,
                                                      const uint4* __restrict__ sinv, int64_t rows_q, int64_t rows_k, int heads_q,
                                                      int heads_k, int S, int d, float sign) {
  // one thread owns the vector pair (v, v + d/2) of a head: x is read once, and so are cos / sin (cos[v + d/2] = cos[v],
  // sin_signed[v + d/2] = -sin_signed[v] by construction of the tables)
  const int vec_per_row = d / 8;             // uint4 = 8 bf16
  const int half_vec = vec_per_row / 2;
  const int64_t total = (rows_q + rows_k) * half_vec;
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += int64_t(gridDim.x) * blockDim.x) {
    int64_t row = idx / half_vec;
    const int v = int(idx - row * half_vec);
    const bool is_k = row >= rows_q;
    const uint4* src = is_k ? k : q;
    uint4* dst = is_k ? ko : qo;
    int heads = heads_q;
    if (is_k) {
      row -= rows_q;
      heads = heads_k;
    }
    const int pos = int((row / heads) % S);
    const uint4 x0 = __ldg(src + row * vec_per_row + v);
    const uint4 x1 = __ldg(src + row * vec_per_row + v + half_vec);
    const uint4 c = __ldg(cosv + int64_t(pos) * vec_per_row + v);
    const uint4 s = __ldg(sinv + int64_t(pos) * vec_per_row + v);
    const uint32_t a0[4] = {x0.x, x0.y, x0.z, x0.w}, a1[4] = {x1.x, x1.y, x1.z, x1.w};
    const uint32_t ca[4] = {c.x, c.y, c.z, c.w}, sa[4] = {s.x, s.y, s.z, s.w};
    uint32_t o0[4], o1[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float sl = sign * lo(sa[j]), sh = sign * hi(sa[j]);
      o0[j] = pack(fmaf(lo(a1[j]), sl, lo(a0[j]) * lo(ca[j])), fmaf(hi(a1[j]), sh, hi(a0[j]) * hi(ca[j])));
      o1[j] = pack(fmaf(lo(a0[j]), -sl, lo(a1[j]) * lo(ca[j])), fmaf(hi(a0[j]), -sh, hi(a1[j]) * hi(ca[j])));
    }
    dst[row * vec_per_row + v] = make_uint4(o0[0], o0[1], o0[2], o0[3]);
    dst[row * vec_per_row + v + half_vec] = make_uint4(o1[0], o1[1], o1[2], o1[3]);
  }
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }

__global__ void __launch_bounds__(256) swiglu_fwd_kernel(const uint4* __restrict__ g, const uint4* __restrict__ u, uint4* __restrict__ out,
                                                         int64_t nvec) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += int64_t(gridDim.x) * blockDim.x) {
    const uint4 gv = __ldg(g + i), uv = __ldg(u + i);
    const uint32_t ga[4] = {gv.x, gv.y, gv.z, gv.w}, ua[4] = {uv.x, uv.y, uv.z, uv.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float g0 = lo(ga[j]), g1 = hi(ga[j]);
      // match torch: silu(g) rounded to bf16, then * u rounded to bf16
      const float s0 = lo(pack(g0 * sigmoidf_(g0), 0.f)), s1 = lo(pack(g1 * sigmoidf_(g1), 0.f));
      o[j] = pack(s0 * lo(ua[j]), s1 * hi(ua[j]));
    }
    out[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const uint4* __restrict__ g, const uint4* __restrict__ u,
                                                         const uint4* __restrict__ dy, uint4* __restrict__ dg, uint4* __restrict__ du,
                                                         int64_t nvec) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += int64_t(gridDim.x) * blockDim.x) {
    const uint4 gv = __ldg(g + i), uv = __ldg(u + i), yv = __ldg(dy + i);
    const uint32_t ga[4] = {gv.x, gv.y, gv.z, gv.w}, ua[4] = {uv.x, uv.y, uv.z, uv.w}, ya[4] = {yv.x, yv.y, yv.z, yv.w};
    uint32_t og[4], ou[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float r_g[2], r_u[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float gg = h ? hi(ga[j]) : lo(ga[j]);
        const float uu = h ? hi(ua[j]) : lo(ua[j]);
        const float yy = h ? hi(ya[j]) : lo(ya[j]);
        const float sg = sigmoidf_(gg);
        const float silu = gg * sg;
        r_u[h] = yy * silu;                                   // d_up
        r_g[h] = yy * uu * (sg * (1.0f + gg * (1.0f - sg)));  // d_gate
      }
      og[j] = pack(r_g[0], r_g[1]);
      ou[j] = pack(r_u[0], r_u[1]);
    }
    dg[i] = make_uint4(og[0], og[1], og[2], og[3]);
    du[i] = make_uint4(ou[0], ou[1], ou[2], ou[3]);
  }
}


// RMSNorm over the last dimension (frozen fp32 weight, as qlora.py:400-401 keeps the norms in fp32): one warp per row,
// bf16 in/out, fp32 statistics.  y = x * rstd * w;  backward (no dW: the weight is frozen):
//   dx = rstd * (g*w - xhat * mean(g*w*xhat)),  xhat = x * rstd.
template <bool kBwd>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const uint4* __restrict__ x, const float* __restrict__ w, const uint4* __restrict__ dy,
                                                      uint4* __restrict__ out, float* __restrict__ rstd_io, int64_t rows, int d, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = int64_t(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = d / 8;
  const uint4* xr = x + row * nvec;
  float rstd;
  if (!kBwd) {
    float ss = 0.f;
    for (int v = lane; v < nvec; v += 32) {
      const uint4 a = __ldg(xr + v);
      const uint32_t aa[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) ss += lo(aa[j]) * lo(aa[j]) + hi(aa[j]) * hi(aa[j]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    rstd = rsqrtf(ss / float(d) + eps);
    if (lane == 0) rstd_io[row] = rstd;
    for (int v = lane; v < nvec; v += 32) {
      const uint4 a = __ldg(xr + v);
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
      const uint32_t aa[4] = {a.x, a.y, a.z, a.w};
      const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
      uint32_t o4[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) o4[j] = pack(lo(aa[j]) * rstd * ww[2 * j], hi(aa[j]) * rstd * ww[2 * j + 1]);
      out[row * nvec + v] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
    }
  } else {
    rstd = rstd_io[row];
    const uint4* gr = dy + row * nvec;
    float dot = 0.f;
    for (int v = lane; v < nvec; v += 32) {
      const uint4 a = __ldg(xr + v), g = __ldg(gr + v);
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
      const uint32_t aa[4] = {a.x, a.y, a.z, a.w}, gg[4] = {g.x, g.y, g.z, g.w};
      const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) dot += lo(gg[j]) * ww[2 * j] * lo(aa[j]) + hi(gg[j]) * ww[2 * j + 1] * hi(aa[j]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    const float c = dot * rstd * rstd / float(d);    // mean(g*w*xhat) * rstd  (xhat = x*rstd)
    for (int v = lane; v < nvec; v += 32) {
      const uint4 a = __ldg(xr + v), g = __ldg(gr + v);
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
      const uint32_t aa[4] = {a.x, a.y, a.z, a.w}, gg[4] = {g.x, g.y, g.z, g.w};
      const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
      uint32_t o4[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        o4[j] = pack(rstd * (lo(gg[j]) * ww[2 * j] - lo(aa[j]) * c), rstd * (hi(gg[j]) * ww[2 * j + 1] - hi(aa[j]) * c));
      out[row * nvec + v] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
    }
  }
}

// Single-pass variant for d <= 8192: one CTA of 128 threads per row, the row lives in registers (up to 8 uint4 per thread), so
// x (and dy) are read exactly once; the two-pass warp-per-row kernel above re-reads them and exposes one warp's load latency
// per row (12.9 / 17.7 us forward / backward at [2048, 4096] against ~6 / ~9 us of HBM time).
// Optional fusion of the residual connection around the norm (x_new = x + delta; y = norm(x_new)):
//   forward : `add` = delta, the sum is also written to `sum_out` (the new residual stream);
//   backward: `add` = the gradient arriving at x_new along the residual path, out = add + d(norm)/dx.
template <bool kBwd, int kVec>
__global__ void __launch_bounds__(128) rmsnorm_row_kernel(const uint4* __restrict__ x, const float* __restrict__ w, const uint4* __restrict__ dy,
                                                          uint4* __restrict__ out, float* __restrict__ rstd_io, int d, float eps,
                                                          const uint4* __restrict__ add, uint4* __restrict__ sum_out) {
  __shared__ float red[4];
  const int64_t row = blockIdx.x;
  const int nvec = d / 8;
  const uint4* xr = x + row * nvec;
  const uint4* gr = kBwd ? dy + row * nvec : nullptr;
  uint4 xa[kVec], ga[kVec];
#pragma unroll
  for (int j = 0; j < kVec; ++j) {
    const int v = threadIdx.x + j * 128;
    xa[j] = v < nvec ? __ldg(xr + v) : make_uint4(0, 0, 0, 0);
    if (kBwd) ga[j] = v < nvec ? __ldg(gr + v) : make_uint4(0, 0, 0, 0);
    if (!kBwd && add != nullptr && v < nvec) {     // residual add in bf16 (as torch's x + delta), kept for the caller
      const uint4 dv = __ldg(add + row * nvec + v);
      xa[j] = make_uint4(pack(lo(xa[j].x) + lo(dv.x), hi(xa[j].x) + hi(dv.x)), pack(lo(xa[j].y) + lo(dv.y), hi(xa[j].y) + hi(dv.y)),
                         pack(lo(xa[j].z) + lo(dv.z), hi(xa[j].z) + hi(dv.z)), pack(lo(xa[j].w) + lo(dv.w), hi(xa[j].w) + hi(dv.w)));
      sum_out[row * nvec + v] = xa[j];
    }
  }
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < kVec; ++j) {
    const int v = threadIdx.x + j * 128;
    if (v >= nvec) continue;
    const uint32_t aa[4] = {xa[j].x, xa[j].y, xa[j].z, xa[j].w};
    if (!kBwd) {
#pragma unroll
      for (int q = 0; q < 4; ++q) acc += lo(aa[q]) * lo(aa[q]) + hi(aa[q]) * hi(aa[q]);
    } else {
      const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
      const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
      const uint32_t gg[4] = {ga[j].x, ga[j].y, ga[j].z, ga[j].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) acc += lo(gg[q]) * ww[2 * q] * lo(aa[q]) + hi(gg[q]) * ww[2 * q + 1] * hi(aa[q]);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  acc = red[0] + red[1] + red[2] + red[3];
  float rstd, c = 0.f;
  if (!kBwd) {
    rstd = rsqrtf(acc / float(d) + eps);
    if (threadIdx.x == 0) rstd_io[row] = rstd;
  } else {
    rstd = rstd_io[row];
    c = acc * rstd * rstd / float(d);
  }
#pragma unroll
  for (int j = 0; j < kVec; ++j) {
    const int v = threadIdx.x + j * 128;
    if (v >= nvec) continue;
    const float4 w0 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v), w1 = __ldg(reinterpret_cast<const float4*>(w) + 2 * v + 1);
    const float ww[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    const uint32_t aa[4] = {xa[j].x, xa[j].y, xa[j].z, xa[j].w};
    uint32_t o4[4];
    if (!kBwd) {
#pragma unroll
      for (int q = 0; q < 4; ++q) o4[q] = pack(lo(aa[q]) * rstd * ww[2 * q], hi(aa[q]) * rstd * ww[2 * q + 1]);
    } else {
      const uint32_t gg[4] = {ga[j].x, ga[j].y, ga[j].z, ga[j].w};
      uint32_t ad[4] = {0u, 0u, 0u, 0u};
      if (add != nullptr) {
        const uint4 av = __ldg(add + row * nvec + v);
        ad[0] = av.x; ad[1] = av.y; ad[2] = av.z; ad[3] = av.w;
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
        o4[q] = pack(lo(ad[q]) + rstd * (lo(gg[q]) * ww[2 * q] - lo(aa[q]) * c), hi(ad[q]) + rstd * (hi(gg[q]) * ww[2 * q + 1] - hi(aa[q]) * c));
    }
    out[row * nvec + v] = make_uint4(o4[0], o4[1], o4[2], o4[3]);
  }
}

template <bool kBwd>
bool launch_rmsnorm_row(const void* x, const float* w, const void* dy, void* out, float* rstd, int64_t rows, int d, float eps, cudaStream_t s,
                        const void* add = nullptr, void* sum_out = nullptr) {
  const int nvec = d / 8;
  if (d % 8 != 0 || nvec > 8 * 128 || rows > 0x7fffffff) return false;
  const uint4 *xp = static_cast<const uint4*>(x), *gp = static_cast<const uint4*>(dy), *ap = static_cast<const uint4*>(add);
  uint4 *op = static_cast<uint4*>(out), *sp = static_cast<uint4*>(sum_out);
  if (nvec <= 2 * 128)
    rmsnorm_row_kernel<kBwd, 2><<<unsigned(rows), 128, 0, s>>>(xp, w, gp, op, rstd, d, eps, ap, sp);
  else if (nvec <= 4 * 128)
    rmsnorm_row_kernel<kBwd, 4><<<unsigned(rows), 128, 0, s>>>(xp, w, gp, op, rstd, d, eps, ap, sp);
  else
    rmsnorm_row_kernel<kBwd, 8><<<unsigned(rows), 128, 0, s>>>(xp, w, gp, op, rstd, d, eps, ap, sp);
  return true;
}

// Counter-based dropout (LoRA branch, --lora_dropout 0.1 of the reference recipe): element i of call site `salt` at step
// `*seed` is kept iff a 16-bit hash lane >= p * 65536; kept values are scaled by 1 / (1 - p).  The mask is a pure function
// of (seed, salt, i): the checkpoint recompute and the backward regenerate it instead of storing it, and the seed lives
// in device memory so a CUDA-graph replay sees the step's value.  Backward of dropout = the same kernel on the gradient.
__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__global__ void __launch_bounds__(256) dropout_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int64_t nvec, uint32_t thr16,
                                                      float scale, const int64_t* __restrict__ seed, uint64_t salt) {
  const uint64_t key = splitmix64(uint64_t(*seed) * 0xD1342543DE82EF95ull + salt);
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec; i += int64_t(gridDim.x) * blockDim.x) {
    const uint4 v = __ldg(x + i);
    const uint64_t r0 = splitmix64(key ^ uint64_t(2 * i)), r1 = splitmix64(key ^ uint64_t(2 * i + 1));
    const uint32_t xa[4] = {v.x, v.y, v.z, v.w};
    const uint32_t rr[4] = {uint32_t(r0), uint32_t(r0 >> 32), uint32_t(r1), uint32_t(r1 >> 32)};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = (rr[j] & 0xFFFFu) >= thr16 ? lo(xa[j]) * scale : 0.0f;
      const float b = (rr[j] >> 16) >= thr16 ? hi(xa[j]) * scale : 0.0f;
      o[j] = pack(a, b);
    }
    out[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

int sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1)
    n = 132;
  return n;
}

unsigned grid_for(int64_t n) {
  int64_t b = (n + 255) / 256;
  static const int64_t cap = int64_t(sm_count()) * 16;   // grid-stride beyond 16 CTAs per SM
  return unsigned(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace

extern "C" int hops_rope_qk(const void* q, const void* k, void* qo, void* ko, const void* cosv, const void* sinv, int64_t rows_q,
                            int64_t rows_k, int heads_q, int heads_k, int S, int d, float sign, void* stream) {
  if (d % 16 != 0) return -1;
  const int64_t total = (rows_q + rows_k) * (d / 16);
  rope_qk_kernel<<<grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(q), static_cast<const uint4*>(k), static_cast<uint4*>(qo), static_cast<uint4*>(ko),
      static_cast<const uint4*>(cosv), static_cast<const uint4*>(sinv), rows_q, rows_k, heads_q, heads_k, S, d, sign);
  return int(cudaPeekAtLastError());
}

extern "C" int hops_swiglu_fwd(const void* g, const void* u, void* out, int64_t n, void* stream) {
  if (n % 8 != 0) return -1;
  swiglu_fwd_kernel<<<grid_for(n / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const uint4*>(g), static_cast<const uint4*>(u),
                                                                                     static_cast<uint4*>(out), n / 8);
  return int(cudaPeekAtLastError());
}

extern "C" int hops_swiglu_bwd(const void* g, const void* u, const void* dy, void* dg, void* du, int64_t n, void* stream) {
  if (n % 8 != 0) return -1;
  swiglu_bwd_kernel<<<grid_for(n / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const uint4*>(g), static_cast<const uint4*>(u),
                                                                                     static_cast<const uint4*>(dy), static_cast<uint4*>(dg),
                                                                                     static_cast<uint4*>(du), n / 8);
  return int(cudaPeekAtLastError());
}

extern "C" int hops_rmsnorm_fwd(const void* x, const float* w, void* y, float* rstd, int64_t rows, int d, float eps, void* stream) {
  if (d % 8 != 0) return -1;
  if (launch_rmsnorm_row<false>(x, w, nullptr, y, rstd, rows, d, eps, static_cast<cudaStream_t>(stream))) return int(cudaPeekAtLastError());
  rmsnorm_kernel<false><<<unsigned((rows + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(x), w, nullptr, static_cast<uint4*>(y), rstd, rows, d, eps);
  return int(cudaPeekAtLastError());
}

extern "C" int hops_rmsnorm_bwd(const void* x, const float* w, const void* dy, void* dx, float* rstd, int64_t rows, int d, void* stream) {
  if (d % 8 != 0) return -1;
  if (launch_rmsnorm_row<true>(x, w, dy, dx, rstd, rows, d, 0.f, static_cast<cudaStream_t>(stream))) return int(cudaPeekAtLastError());
  rmsnorm_kernel<true><<<unsigned((rows + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(x), w, static_cast<const uint4*>(dy), static_cast<uint4*>(dx), rstd, rows, d, 0.f);
  return int(cudaPeekAtLastError());
}

extern "C" int hops_dropout(const void* x, void* out, int64_t n, float p, const int64_t* seed, uint64_t salt, void* stream) {
  if (n % 8 != 0 || p < 0.f || p >= 1.f) return -1;
  const uint32_t thr16 = uint32_t(p * 65536.0f + 0.5f);
  dropout_kernel<<<grid_for(n / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const uint4*>(x), static_cast<uint4*>(out), n / 8,
                                                                                 thr16, 1.0f / (1.0f - p), seed, salt);
  return int(cudaPeekAtLastError());
}

// residual add fused with the norm: x_new = x + delta (written to sum_out), y = rmsnorm(x_new); d <= 8192 only (-2 otherwise)
extern "C" int hops_add_rmsnorm_fwd(const void* x, const void* delta, const float* w, void* sum_out, void* y, float* rstd, int64_t rows, int d,
                                    float eps, void* stream) {
  if (!launch_rmsnorm_row<false>(x, w, nullptr, y, rstd, rows, d, eps, static_cast<cudaStream_t>(stream), delta, sum_out)) return -2;
  return int(cudaPeekAtLastError());
}
// dx = g_residual + d(rmsnorm)/dx (x = the SUM saved by the forward); d <= 8192 only
extern "C" int hops_add_rmsnorm_bwd(const void* x_sum, const float* w, const void* dy, const void* g_residual, void* dx, float* rstd,
                                    int64_t rows, int d, void* stream) {
  if (!launch_rmsnorm_row<true>(x_sum, w, dy, dx, rstd, rows, d, 0.f, static_cast<cudaStream_t>(stream), g_residual, nullptr)) return -2;
  return int(cudaPeekAtLastError());
}
