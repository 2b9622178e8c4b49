/*
 * qlora_b200 — C-ABI of the H100-native NF4 + double-quant Linear4bit hot path.
 *
 * This is the drop-in boundary: the entry points a bitsandbytes-style Python
 * host binds with ctypes for the path /root/reference/qlora.py reaches through
 *   qlora.py:15      import bitsandbytes as bnb
 *   qlora.py:249     bnb.nn.Linear4bit            (module whose fwd/bwd this is)
 *   qlora.py:318-326 BitsAndBytesConfig(load_in_4bit, nf4, double_quant, bf16)
 * The reference's own FFI for this path is bitsandbytes' ctypes binding of
 * libbitsandbytes_cudaXXX.so (csrc/pythonInterface.c [upstream, un-vendored; pin
 * bitsandbytes==0.40.0, requirements.txt:1]); each function below names the
 * upstream symbol(s) it replaces.
 *
 * Conventions (all functions):
 *   - plain pointers + sizes; every buffer is a caller-allocated DEVICE buffer
 *     (the library never allocates, frees or synchronises);
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *     launches are asynchronous and CUDA-graph capturable;
 *   - return 0 on success, >0 = cudaError_t of a failed launch/API call,
 *     <0 = argument error (QB200_E*); never exit()s the process (upstream's
 *     CUDA_CHECK_RETURN does);  qb200_last_error() gives a thread-local message;
 *   - dtype codes: 0 = fp32, 1 = fp16, 2 = bf16.
 */
#ifndef QLORA_B200_H_
#define QLORA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QB200_DTYPE_F32 0
#define QB200_DTYPE_F16 1
#define QB200_DTYPE_BF16 2

#define QB200_EINVAL (-1)      /* bad argument (null pointer, bad dtype/blocksize) */
#define QB200_EUNSUPPORTED (-2) /* shape not supported by the fused kernel          */
#define QB200_EDRIVER (-3)     /* cuTensorMapEncodeTiled unavailable / failed       */

/* Library/ABI version (major*10000 + minor*100 + patch). */
int qb200_version(void);
/* Thread-local description of the last non-zero return code ("" if none). */
const char* qb200_last_error(void);
/* 1 if the library was compiled with the sm_90a fused wgmma path. */
int qb200_has_fused_gemm(void);

/* ---- arithmetic mode of the quantizers (K1, K2) -----------------------------------
 * 0 = ieee (default): inv = 1.0f/absmax and x = v*inv correctly rounded — bit-exact with oracle/nf4_oracle.{py,c}.
 * 1 = approx: rcp.approx.ftz.f32 + mul.ftz.f32, i.e. what those two expressions compile to under nvcc --use_fast_math,
 *     the flag upstream bitsandbytes builds csrc/kernels.cu with (SURVEY.md A.5(i)).  The two modes differ only for values
 *     within ~1 ulp of a decision threshold.  Also selectable with QB200_QUANT_MATH=approx.  Dequantize is unaffected. */
int qb200_set_quant_math(int mode);
int qb200_get_quant_math(void);

/* ---- K1: first-level NF4 quantize --------------------------------------------------
 * Replaces cquantize_blockwise_{fp16,bf16,fp32}_nf4(code, A, absmax, out, blocksize, n)
 * [upstream csrc/pythonInterface.c; kernel kQuantizeBlockwise<T,BS,2,0,NF4>].
 * A: n values of `a_dtype`; packed: (n+1)/2 bytes; absmax: ceil(n/blocksize) fp32.
 * blocksize in {64,128,256,512,1024,2048,4096}. Bit-exact with oracle/nf4_oracle.{py,c}. */
int qb200_quantize_nf4(const void* A, int a_dtype, int64_t n, int blocksize, uint8_t* packed, float* absmax,
                       void* stream);

/* ---- K2: 8-bit blockwise quantize against a 256-entry codebook (second level) ------
 * Replaces cquantize_blockwise_fp32(code, A, absmax, out, blocksize, n)
 * [kernel kQuantizeBlockwise<float,BS,2,0,General8bit>]. */
int qb200_quantize_blockwise_8bit(const float* code256, const float* A, int64_t n, int blocksize, uint8_t* out,
                                  float* absmax, void* stream);

/* ---- K3: 8-bit blockwise dequantize -------------------------------------------------
 * Replaces cdequantize_blockwise_fp32(code, A, absmax, out, blocksize, n[, stream]). */
int qb200_dequantize_blockwise_8bit(const float* code256, const uint8_t* A, const float* absmax, int64_t n,
                                    int blocksize, float* out, void* stream);

/* ---- K4: NF4 dequantize with fp32 absmax --------------------------------------------
 * Replaces cdequantize_blockwise_{fp16,bf16,fp32}_nf4(NULL, A, absmax, out, blocksize, n[, stream]).
 * out: n values of `out_dtype`. */
int qb200_dequantize_nf4(const uint8_t* packed, const float* absmax, int64_t n, int blocksize, void* out,
                         int out_dtype, void* stream);

/* ---- K3+add+K4 in one launch: NF4 dequantize from the nested (double-quant) state ---
 * Replaces the reference's three-step dequantize_4bit for nested states:
 *   cdequantize_blockwise_fp32 (K3)  ->  torch `absmax += offset`  ->  cdequantize_blockwise_*_nf4 (K4).
 * absmax = fadd_rn(fmul_rn(code256[absmax_u8[b]], absmax2[b / blocksize2]), *offset). */
int qb200_dequantize_nf4_nested(const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                                const float* absmax2, const float* offset, int64_t n, int blocksize, int blocksize2,
                                void* out, int out_dtype, void* stream);

/* ---- K5 (forward): fused dequant + wgmma GEMM -------------------------------------
 * Replaces, for MatMul4Bit.forward [upstream autograd/_functions.py]:
 *   dequantize_4bit (K3, add, K4: bf16 W written to HBM)  +  torch.nn.functional.linear (cuBLAS).
 * Y[M,N] = X[M,K] . W[N,K]^T (+ bias[N]);  X,Y,bias bf16 row-major; W given by the nested
 * NF4 state (blocksize 64 / 256).  W is dequantized tile-by-tile in shared memory and
 * never materialised in HBM.  Requires K % 64 == 0 and N % 8 == 0 (QB200_EUNSUPPORTED otherwise).
 * absmax_f32 may be given INSTEAD of (absmax_u8, code256, absmax2, offset) for a non-nested state. */
int qb200_nf4_linear_fwd(const void* X, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                         const float* absmax2, const float* offset, const float* absmax_f32, const void* bias,
                         void* Y, int64_t M, int64_t N, int64_t K, void* stream);

/* ---- K5 (backward dX): same kernel, W consumed MN-major -----------------------------
 * Replaces, for MatMul4Bit.backward: dequantize_4bit + torch.matmul(grad_out, W_deq).
 * dX[M,K] = dY[M,N] . W[N,K].  Same shape requirements as the forward (K % 64 == 0, N % 8 == 0). */
int qb200_nf4_linear_bwd_dx(const void* dY, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                            const float* absmax2, const float* offset, const float* absmax_f32, void* dX,
                            int64_t M, int64_t N, int64_t K, void* stream);

/* ---- K5 + LoRA (SURVEY.md 8f-1): the caller's low-rank update folded into the same launch ----------------
 * Replaces peft lora.Linear4bit.forward's  `result = base(x); result += lora_B(lora_A(x)) * scaling`  (two extra GEMMs and
 * two elementwise passes over [M,N]) by ceil(R/64) extra bf16 contraction steps accumulated in the same register accumulators
 * (ranks [64j, 64j+64) in step j, after the NF4 steps):
 *   forward : Y  = X . W^T (+bias) + U . V^T      U[M,R] = scaling * (X . A^T) (bf16),  V[N,R] = lora_B.weight
 *   backward: dX = dY . W          + U . Vt       U[M,R] = scaling * (dY . B)  (bf16),  Vt[R,K] = lora_A.weight
 * R: LoRA rank, a multiple of 8 in [8, 256] (columns/rows beyond R are zero-filled by TMA); every entry point that takes R
 * (these two, _ex, _group, _group_scaled, _group_typed, _group_ex, _group_reuse) returns QB200_EUNSUPPORTED before any
 * launch for any other nonzero R. */
int qb200_nf4_linear_fwd_lora(const void* X, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                              const float* absmax2, const float* offset, const float* absmax_f32, const void* bias,
                              const void* U, const void* V, int64_t R, void* Y, int64_t M, int64_t N, int64_t K,
                              void* stream);
int qb200_nf4_linear_bwd_dx_lora(const void* dY, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                                 const float* absmax2, const float* offset, const float* absmax_f32, const void* U,
                                 const void* Vt, int64_t R, void* dX, int64_t M, int64_t N, int64_t K, void* stream);

/* ---- general form: optional LoRA operands (R = 0: none) and optional split-K workspace -----------------------
 * For very small token counts the contraction is split over several clusters; the fp32 partial sums need a caller-lent
 * DEVICE workspace of qb200_nf4_linear_workspace_size() bytes (0 = not needed).  Without a workspace the un-split
 * schedule is used, as it is for an output whose base is not 8-byte (16-bit output) or 16-byte (fp32 output) aligned or
 * whose row pitch is not a multiple of 4 elements.  is_bwd: 0 forward (in = X, out = Y, V = lora_B.weight [N,R]),
 * 1 backward-dX (in = dY, out = dX, V = lora_A.weight [R,K]; bias must be NULL). */
int64_t qb200_nf4_linear_workspace_size(int64_t M, int64_t N, int64_t K, int is_bwd);
/* Training token counts: at M >= a threshold (default 1536, env QB200_SCRATCH_MIN_M) a call in bf16 compute over a bf16 or fp32
 * state, with a bf16 or fp32 output and no row scale, writes each of its nprob weights once as bf16 [N,K] into the caller-lent
 * `workspace` and runs a TMA-fed GEMM over that copy (same weights and summation order as the fused kernel).  This returns
 * the bytes that needs (nprob*N*K*2), 0 below the threshold; the workspace must be 32-byte aligned.  A call that needs the
 * scratch and gets a NULL, short or misaligned workspace returns QB200_EINVAL before any launch.  The four entry points above
 * take no workspace and keep the fused kernel at every M. */
int64_t qb200_nf4_linear_scratch_size(int nprob, int64_t M, int64_t N, int64_t K, int is_bwd);
int qb200_nf4_linear_ex(int is_bwd, const void* in, const uint8_t* packed, const uint8_t* absmax_u8, const float* code256,
                        const float* absmax2, const float* offset, const float* absmax_f32, const void* bias, const void* U,
                        const void* V, int64_t R, void* out, int64_t M, int64_t N, int64_t K, void* workspace,
                        int64_t workspace_bytes, void* stream);

/* ---- grouped form: 1..3 Linear4bit of ONE shape [N,K] in one launch --------------------------------------------
 * Replaces, per decoder layer of the reference's model (qlora.py:249 collects q/k/v/o/gate/up/down as LoRA targets),
 * the three (two) separate MatMul4Bit calls on the SAME activation (q/k/v, gate/up) and, in backward, their three (two)
 * dX GEMMs plus autograd's accumulation of the input gradient:
 *   is_bwd = 0: out_p[M,N] = in_p . W_p^T (+bias_p) + U_p . V_p^T      for every problem p (in_p may be one tensor)
 *   is_bwd = 1: out_0[M,K] = sum_p ( in_p . W_p + U_p . V_p )           ONE output, accumulated in registers (out_p, p>0 ignored)
 * Row pitches (elements; 0 = contiguous) let the outputs be column slices of one [M, nprob*N] buffer and U_p column
 * slices of one [M, nprob*R] projection.  out_dtype: QB200_DTYPE_BF16, or QB200_DTYPE_F32 = the bf16-rounded result
 * widened in the epilogue (Linear4bit.forward called with fp32 activations, qlora.py:396-405: no separate cast kernel).
 * workspace: split-K workspace, single problems only (see qb200_nf4_linear_workspace_size); may be NULL. */
typedef struct qb200_nf4_problem {
  const void* in;            /* bf16 activations: X_p [M,K] (forward) or dY_p [M,N] (backward) */
  int64_t ld_in;             /* row pitch of `in` */
  const uint8_t* packed;     /* NF4 state of W_p[N,K] (same meaning as in qb200_nf4_linear_fwd) */
  const uint8_t* absmax_u8;
  const float* code256;
  const float* absmax2;
  const float* offset;
  const float* absmax_f32;
  const void* bias;          /* bf16 [N] or NULL (forward only) */
  const void* U;             /* bf16 [M,R] or NULL when R == 0 */
  int64_t ld_u;
  const void* V;             /* bf16: lora_B.weight [N,R] (forward) / lora_A.weight [R,K] (backward) */
  void* out;
  int64_t ld_out;
} qb200_nf4_problem;
int qb200_nf4_linear_group(int is_bwd, int nprob, const qb200_nf4_problem* probs, int64_t R, int64_t M, int64_t N, int64_t K,
                           int out_dtype, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- grouped form with a per-row weight scale (DoRA's magnitude over the NF4 base) ------------------------------------
 * Same as qb200_nf4_linear_group, with W_p replaced by diag(s_p) . W_p:  row_scales[p] is a DEVICE fp32 array of N values
 * (4-byte aligned) or NULL (problem p unscaled).  The scale multiplies the absmax of every NF4 block of row n, so
 *   is_bwd = 0: out_p = in_p . (diag(s_p) W_p)^T (+bias_p) + U_p . V_p^T      (s_p scales output feature n)
 *   is_bwd = 1: out_0 = sum_p ( in_p . diag(s_p) W_p + U_p . V_p )             (s_p scales contraction index n)
 * The LoRA term and the bias are not scaled.  row_scales itself is a HOST array of nprob pointers and must not be NULL.
 * The scales may be written by the preceding kernel on the stream; a scaled launch reads them only after that kernel is done. */
int qb200_nf4_linear_group_scaled(int is_bwd, int nprob, const qb200_nf4_problem* probs, const float* const* row_scales, int64_t R,
                                  int64_t M, int64_t N, int64_t K, int out_dtype, void* workspace, int64_t workspace_bytes,
                                  void* stream);

/* ---- grouped form for either 16-bit compute type (fp16 compute: bnb_4bit_compute_dtype=torch.float16) ---------------
 * qb200_nf4_linear_group_scaled with every 16-bit operand (in, bias, U, V and a 16-bit out) of type `dtype`:
 *   QB200_DTYPE_BF16: the same launches as qb200_nf4_linear_group[_scaled];
 *   QB200_DTYPE_F16 : the weights are fp16_rn(LUT[j]*absmax) -- dequantize_4bit's value for an fp16 or fp32 state, cast to
 *                     fp16 -- and the result is rounded to fp16 once.
 * out_dtype: `dtype`, or QB200_DTYPE_F32 = the dtype-rounded result widened.  row_scales may be NULL (no problem scaled).
 * Forward calls with at most 16 tokens and a 16-bit output run the skinny kernels; the split-K workspace works as above.
 * An unknown dtype, or an out_dtype that is neither `dtype` nor fp32, returns QB200_EINVAL. */
int qb200_nf4_linear_group_typed(int is_bwd, int dtype, int nprob, const qb200_nf4_problem* probs, const float* const* row_scales,
                                 int64_t R, int64_t M, int64_t N, int64_t K, int out_dtype, void* workspace, int64_t workspace_bytes,
                                 void* stream);

/* ---- grouped form with the quant state's dtype and an fp16 output under bf16 compute ---------------------------------
 * qb200_nf4_linear_group_typed without row scales, for a quant state of `state_dtype` (the dtype `dequantize_4bit` returns
 * for it).  The weights are exactly `dequantize_4bit(W, state).to(dtype)`:
 *   dtype QB200_DTYPE_BF16: state bf16 or fp32 -> bf16_rn(LUT[j]*absmax);  state fp16 -> bf16_rn(fp16_rn(LUT[j]*absmax))
 *                           (fp16 subnormals kept).  out_dtype bf16, fp32 (the bf16-rounded result widened) or fp16 (the
 *                           bf16-rounded result rounded to fp16: `Linear4bit.forward`'s output cast for fp16 activations).
 *   dtype QB200_DTYPE_F16 : state fp16 or fp32 -> fp16_rn(LUT[j]*absmax); out_dtype fp16 or fp32.
 * Every other (dtype, state_dtype, out_dtype), including fp16 compute over a bf16 state, returns QB200_EINVAL before any
 * launch.  Forward calls with at most 16 tokens and a 16-bit output run the skinny kernels; the split-K workspace works as
 * above. */
int qb200_nf4_linear_group_ex(int is_bwd, int dtype, int state_dtype, int nprob, const qb200_nf4_problem* probs, int64_t R, int64_t M,
                              int64_t N, int64_t K, int out_dtype, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- grouped form that reuses the bf16 weight copy of an earlier call ------------------------------------------------
 * qb200_nf4_linear_group_ex with an in / out flag about the workspace (NULL: exactly qb200_nf4_linear_group_ex).  A call
 * that takes the scratch path (bf16 compute over a bf16 or fp32 state, M >= the scratch threshold, a bf16 or fp32 output)
 * first writes the bf16 W_p [N, K] of every problem into the workspace, in problem order, then runs the GEMM over them.
 *   in : nonzero = the workspace already holds those W_p, left there by an earlier call on the same packed weights and quant
 *        states that reported 1 (e.g. a gradient-checkpoint recompute's forward, reused by the dX launch of the same
 *        layer).  A call that takes the scratch path then launches only the GEMM; any other call ignores the flag.
 *   out: 1 when this call left every W_p in the workspace (it took the scratch path), else 0; 0 on error.
 * A workspace too short or misaligned for the scratch path returns QB200_EINVAL before any launch, whatever the flag says. */
int qb200_nf4_linear_group_reuse(int is_bwd, int dtype, int state_dtype, int nprob, const qb200_nf4_problem* probs, int64_t R,
                                 int64_t M, int64_t N, int64_t K, int out_dtype, void* workspace, int64_t workspace_bytes,
                                 int* w_in_workspace, void* stream);

/* U[M,R] = scale * X[M,K] . A[R,K]^T for 1..16 tokens (bf16 in / out, fp32 sum, one rounding): the lora_A projection that
 * feeds qb200_nf4_linear_group's U operand during generation with an unmerged adapter — peft `lora.Linear.forward`'s
 * `lora_A(dropout(x))` (qlora.py:817-834 through PeftModel); replaces a split-K cuBLAS GEMM + reduce per projection.
 * ld_x / ld_u: row pitches in elements (0 = dense); x, A 16-byte aligned, K % 8 == 0.  Larger M: QB200_EUNSUPPORTED. */
int qb200_lora_project(const void* x, int64_t ld_x, const void* A, float scale, void* U, int64_t ld_u, int64_t M, int64_t K,
                       int64_t R, void* stream);
/* qb200_lora_project with x, A and U of type `dtype` (QB200_DTYPE_BF16: the same launch; QB200_DTYPE_F16: fp16 operands,
 * fp32 sum, one fp16 rounding).  An unknown dtype returns QB200_EINVAL. */
int qb200_lora_project_typed(int dtype, const void* x, int64_t ld_x, const void* A, float scale, void* U, int64_t ld_u, int64_t M,
                             int64_t K, int64_t R, void* stream);

/* ---- mixed-adapter batches: every token row uses its own LoRA adapter (peft `adapter_names`, "__base__" = none) ----------
 * An adapter table is a DEVICE array of n_adapters entries; row_adapter a DEVICE int32 array of one adapter index per token.
 * Token t with a(t) = row_adapter[t] in [0, n_adapters) computes, with U_t = scale_a . x_t . A_a^T rounded once to the operand
 * type,  y_t = x_t . W^T (+bias) + U_t . B_a^T  (one rounding);  any other index means "no adapter": y_t = x_t . W^T (+bias),
 * so no device index can make a kernel read outside the table.  A and B are dense, 16-byte aligned; rank a multiple of 8 in
 * [8, 256] and at most the R columns of U (a kernel clamps it to those columns).  Switching a CUDA graph between batches is
 * a copy into row_adapter: no host argument depends on which adapters the batch uses. */
typedef struct qb200_lora_adapter {
  const void* A;   /* lora_A.weight [rank, K] */
  const void* B;   /* lora_B.weight [N, rank] */
  float scale;     /* LoRA scaling */
  int32_t rank;
} qb200_lora_adapter;

/* U[M, R] (row pitch ld_u, 0 = R) for any M >= 1: U[t, j] = scale_a . x_t . A_a[j]^T for j < rank_a, 0 for the other columns
 * and for rows without an adapter.  Per token the arithmetic of qb200_lora_project_typed (same chunking, fp32 sum order and
 * rounding), so a batch with one adapter gives its bits.  dtype: QB200_DTYPE_BF16 or QB200_DTYPE_F16 (x, A and U).
 * ld_x: 0 = K.  x 16-byte and the table 8-byte aligned, K % 8 == 0; R a multiple of 8 in [8, 256] (QB200_EUNSUPPORTED
 * otherwise). */
int qb200_lora_project_mixed(int dtype, const void* x, int64_t ld_x, const qb200_lora_adapter* table, int n_adapters,
                             const int32_t* row_adapter, void* U, int64_t ld_u, int64_t M, int64_t K, int64_t R, void* stream);

/* qb200_nf4_linear_group_ex's forward with one adapter per token: for every problem p, probs[p].V is that linear's DEVICE
 * adapter table (n_adapters entries, the same indices for every problem) and probs[p].U its [M, R] qb200_lora_project_mixed
 * output; row_adapter is shared.  One skinny launch per problem (16 tokens per launch).  Token counts above
 * QB200_SKINNY_MAX_M and an fp32 output return QB200_EUNSUPPORTED; no workspace is needed. */
int qb200_nf4_linear_group_mixed(int dtype, int state_dtype, int nprob, const qb200_nf4_problem* probs, int n_adapters,
                                 const int32_t* row_adapter, int64_t R, int64_t M, int64_t N, int64_t K, int out_dtype, void* stream);

/* Segmented LoRA: a mixed-adapter batch of any token count with no read-back to the host.  The rows are grouped by adapter on
 * the device (qb200_lora_segment_table), then tensor-core kernels run one tile of up to 64 rows of one adapter per CTA.
 * For a batch of M rows over an adapter table of n_adapters entries:
 *   1. y = the base launch (qb200_nf4_linear_group_ex without LoRA operands), 16-bit;
 *   2. U [M, R] = qb200_lora_project_mixed, or qb200_lora_shrink_segmented (rows with an adapter only);
 *   3. qb200_lora_segment_table;
 *   4. qb200_lora_expand_segmented: y_t = rn(y_t + U_t . B_a^T), fp32 sum, in place; rows without an adapter keep y's bits.
 * The result is rounded twice (the base output, then the sum), where qb200_nf4_linear_group_mixed rounds once.  Indices and
 * ranks are clamped as in qb200_lora_project_mixed.  Argument errors return QB200_EINVAL (QB200_EUNSUPPORTED for an R outside
 * the multiples of 8 in [8, 256]) before any launch. */

/* Bytes of the segment table's workspace for M rows and n_adapters adapters; it depends on nothing else.  0 for M < 1,
 * n_adapters < 1 or a table too large for one grid. */
int64_t qb200_lora_segment_workspace_size(int64_t M, int n_adapters);
/* The segment table of the DEVICE row indices row_adapter [M] into the lent DEVICE workspace (16-byte aligned, at least
 * qb200_lora_segment_workspace_size bytes): a stable counting sort of the rows into one bucket per adapter plus one for
 * "no adapter", the bucket offsets and the list of 64-row tiles the two kernels below run over.  One CTA. */
int qb200_lora_segment_table(const int32_t* row_adapter, int64_t M, int n_adapters, void* workspace, int64_t workspace_bytes,
                             void* stream);
/* U_p[t, j] = rn(scale_a . x_t . A_a[j]^T) for the rows t with an adapter a and j < rank_a, 0 for j in [rank_a, R); rows
 * without an adapter are not written.  x [M, K] (ld_x: 0 = K) is shared by the nprob (1..3) problems, tables[p] and U[p] are
 * problem p's DEVICE adapter table and [M, R] output (ld_u: 0 = R).  dtype: QB200_DTYPE_BF16 or QB200_DTYPE_F16. */
int qb200_lora_shrink_segmented(int dtype, int nprob, const void* x, int64_t ld_x, const qb200_lora_adapter* const* tables,
                                void* const* U, int64_t ld_u, int n_adapters, const void* workspace, int64_t workspace_bytes,
                                int64_t M, int64_t K, int64_t R, void* stream);
/* out_p[t] = rn(out_p[t] + U_p[t] . B_a^T) over N columns (a multiple of 8; ld_out: 0 = N, even) for every row t with an
 * adapter a, in place; U[p] [M, R] (ld_u: 0 = R, a multiple of 8, 16-byte aligned) and tables[p] as for the shrink. */
int qb200_lora_expand_segmented(int dtype, int nprob, const qb200_lora_adapter* const* tables, const void* const* U, int64_t ld_u,
                                void* const* out, int64_t ld_out, int n_adapters, const void* workspace, int64_t workspace_bytes,
                                int64_t M, int64_t N, int64_t R, void* stream);

/* Segmented LoRA backward: training several adapters over one base in one batch.  For the forward above (U_p saved), dY_p
 * the output gradients and the same segment table:
 *   G_p [M, R]   = qb200_lora_grad_shrink_segmented     G_p[t] = rn(s_a . dY_p[t] . B_a), zero beyond rank_a;
 *   dX           = the base dX launch (16-bit), then qb200_lora_grad_input_segmented with accumulate = 1:
 *                  dX[t] = rn(dX[t] + sum_p G_p[t] . A_{p,a}), the problems summed in fp32 before the one rounding;
 *                  or, when each problem's adapter reads its own (dropped) input, accumulate = 0: dxl_p[t] = rn(G_p[t] . A_{p,a});
 *   dA_p, dB_p   = qb200_lora_weight_grad_segmented     dA_a = rn(sum_{rows of a} G^T . x_lora), dB_a = rn(sum dY^T . U).
 * Every sum is fp32 in a fixed order (no atomics), so equal inputs give equal bits.  Rows without an adapter are not written
 * by the first two; indices and ranks are clamped as in qb200_lora_project_mixed.  Argument errors return QB200_EINVAL
 * (QB200_EUNSUPPORTED for an R outside the multiples of 8 in [8, 256]) before any launch. */

/* G[p][t, j] = rn(scale_a . dY[p][t] . B_a[:, j]) for j < rank_a, 0 for j in [rank_a, R), over the N columns of dY[p]
 * (N a multiple of 8; ld_dy: 0 = N, a multiple of 8, 16-byte aligned rows); G[p] [M, R] (ld_g: 0 = R, even).  tables[p] as for
 * qb200_lora_shrink_segmented. */
int qb200_lora_grad_shrink_segmented(int dtype, int nprob, const void* const* dY, int64_t ld_dy, const qb200_lora_adapter* const* tables,
                                     void* const* G, int64_t ld_g, int n_adapters, const void* workspace, int64_t workspace_bytes,
                                     int64_t M, int64_t N, int64_t R, void* stream);
/* accumulate = 1: dx[0][t] = rn(dx[0][t] + sum_p G[p][t] . A_{p,a}) in place (dx[0] only is read);  accumulate = 0:
 * dx[p][t] = rn(G[p][t] . A_{p,a}).  K columns (a multiple of 8; ld_dx: 0 = K, even), G[p] [M, R] (ld_g: 0 = R, a multiple
 * of 8, 16-byte aligned). */
int qb200_lora_grad_input_segmented(int dtype, int nprob, int accumulate, const qb200_lora_adapter* const* tables,
                                    const void* const* G, int64_t ld_g, void* const* dx, int64_t ld_dx, int n_adapters,
                                    const void* workspace, int64_t workspace_bytes, int64_t M, int64_t K, int64_t R, void* stream);
/* For each adapter a and problem p, over the rows t of a (the segment table's bucket, in sorted order):
 *   D_a[i, j] = rn(sum_t P[p][t, i] . Q[p][t, j]),  i < rank_a, j < D,
 * written to out[p] at element rank_offsets[a] . D: transpose_out = 0 as [rank_a, D] (dA_a: P = G, Q = the adapters' input,
 * D = K), 1 as [D, rank_a] (dB_a: P = U, Q = dY, D = N).  rank_offsets is a DEVICE int64 [n_adapters] array (8-byte aligned)
 * of the ranks' exclusive prefix sums, shared by the problems; each out[p] holds rank_total . D elements, and an adapter
 * whose offset would write past them writes nothing.  An adapter without rows gets zeros.  P[p] [M, R] (ld_p: 0 = R) and
 * Q[p] [M, D] (ld_q: 0 = D), 16-byte aligned; D a multiple of 8. */
int qb200_lora_weight_grad_segmented(int dtype, int nprob, int transpose_out, const qb200_lora_adapter* const* tables,
                                     const int64_t* rank_offsets, int64_t rank_total, const void* const* P, int64_t ld_p,
                                     const void* const* Q, int64_t ld_q, void* const* out, int n_adapters, const void* workspace,
                                     int64_t workspace_bytes, int64_t M, int64_t D, int64_t R, void* stream);

/* Segmented DoRA (QDoRA): several DoRA adapters over one NF4 base in one batch (DESIGN.md §6e).  Adapter a of problem p has
 * the table entry {A, B, s, r} of the LoRA kernels above and a magnitude m_a [N] of the compute dtype; with the detached norm
 * n_a[f] = ||W_f + s . (B_a A_a)_f|| and c_a = m_a / n_a (fp32 [n_adapters, N] per problem):
 *   norms    qb200_dora_stack_a, the fused forward P = A_stack . W^T with an fp32 output, qb200_dora_norm_segmented;
 *   forward  the base launch (and, with dropout, Qb = rn(xd . W^T)), U as for the LoRA forward, qb200_dora_expand_segmented;
 *   backward qb200_dora_grad_scale_segmented, then the LoRA backward's launches with dQ in place of dY.
 * The ranks are shared by the problems: rank_offsets [n_adapters] (DEVICE int64, the ranks' exclusive prefix sums, 8-byte
 * aligned) place adapter a's rows in [off_a, off_a + r_a) of rank_total.  An entry whose rank is not a positive multiple of 8
 * or whose offset would reach past rank_total is unusable: its rows take the base only, as rows without an adapter do.  Every
 * sum is fp32 in a fixed order (no atomics).  Argument errors return QB200_EINVAL (QB200_EUNSUPPORTED for an R outside the
 * multiples of 8 in [8, 256]) before any launch.  dtype: QB200_DTYPE_BF16 or QB200_DTYPE_F16. */

/* out[p] [rank_total, K] (16-byte aligned): row j = A_{p,a}[j - off_a] of the adapter a = stack_rows[j] (DEVICE int32
 * [rank_total]), zeros for a row outside its adapter's clamped rank.  K a multiple of 8. */
int qb200_dora_stack_a(int dtype, int nprob, const qb200_lora_adapter* const* tables, const int32_t* stack_rows,
                       const int64_t* rank_offsets, int64_t rank_total, void* const* out, int n_adapters, int64_t K, int64_t R,
                       void* stream);
/* Two launches: gram[p] (fp32, gram_total elements) holds G_a = A_a . A_a^T [r_a, r_a] at gram_offsets[a] (DEVICE int64,
 * exclusive prefix sums of r_a^2); then c[p] and norm[p] (fp32 [n_adapters, N], 8-byte aligned) get, for every row f,
 *   n_a[f] = sqrt(max(0, row_norm2[p][f] + 2 s_a sum_j B_a[f, j] P[p][off_a + j, f] + s_a^2 (B_a G_a B_a^T)[f, f])),
 *   c_a[f] = m_a[f] / n_a[f],
 * with P[p] [rank_total, N] fp32 from the fused forward over qb200_dora_stack_a's rows, row_norm2[p] = ||W_f||^2 fp32 [N], and
 * mag_tables[p] a DEVICE array of n_adapters pointers to the magnitudes.  An unusable entry gets c = n = 0. */
int qb200_dora_norm_segmented(int dtype, int nprob, const qb200_lora_adapter* const* tables, const void* const* mag_tables,
                              const int64_t* rank_offsets, const int64_t* gram_offsets, int64_t rank_total, int64_t gram_total,
                              const float* const* P, const float* const* row_norm2, float* const* gram, float* const* c,
                              float* const* norm, int n_adapters, int64_t N, int64_t K, int64_t R, void* stream);
/* qb200_lora_expand_segmented with the magnitude scale c[p] (fp32 [n_adapters, N], 8-byte aligned) of each row's adapter,
 * over the segment table of the forward:  dropout = 0: out_p[t] = rn(c_a . (out_p[t] + U_p[t] . B_a^T));  dropout = 1:
 * out_p[t] = rn(out_p[t] + (c_a - 1) . Q_p[t] + c_a . U_p[t] . B_a^T) and Q_p[t] = rn(Q_p[t] + U_p[t] . B_a^T) in place, Q_p
 * read as rn(xd_p . W_p^T) (row pitch ld_out).  Rows without an adapter are not written. */
int qb200_dora_expand_segmented(int dtype, int nprob, int dropout, const qb200_lora_adapter* const* tables, const void* const* U,
                                int64_t ld_u, const float* const* c, void* const* Q, void* const* out, int64_t ld_out, int n_adapters,
                                const void* workspace, int64_t workspace_bytes, int64_t M, int64_t N, int64_t R, void* stream);
/* Per problem p and row t of adapter a (the forward's segment table):  dQ[p][t] = rn(dY[p][t] . c_a);  dropout = 1 also
 * dD[p][t] = rn(dY[p][t] . (c_a - 1));  dm[p][a . N + f] = rn(sum_{t of a} dY[p][t, f] . Q[p][t, f] / n_a[f]), the sum fp32
 * in sorted-row order.  Q[p] is the expand's pre-scale output with dropout, else the forward's output y, read as y / c_a (an
 * element with c_a = 0 adds nothing).  Rows without a usable adapter copy dY into dQ and get dD = 0; an adapter without rows
 * gets dm = 0.  dY, Q, dQ and dD share the row pitch ld (0 = N, even); dm[p] holds n_adapters . N elements. */
int qb200_dora_grad_scale_segmented(int dtype, int nprob, int dropout, const qb200_lora_adapter* const* tables,
                                    const int64_t* rank_offsets, int64_t rank_total, const void* const* dY, const void* const* Q,
                                    const float* const* c, const float* const* norm, int64_t ld, void* const* dQ, void* const* dD,
                                    void* const* dm, int n_adapters, const void* workspace, int64_t workspace_bytes, int64_t M,
                                    int64_t N, int64_t R, void* stream);

/* ---- paged 32-bit AdamW (SURVEY.md 8f-3; qlora.py:198 optim='paged_adamw_32bit') ---------------------------
 * Replaces cadam32bit_grad_{fp32,fp16,bf16} (kernel kOptimizer32bit2State<T,ADAM>) and cget_managed_ptr / cprefetch.
 * One fused elementwise pass: p, g of `dtype`; m, v fp32; `step` counts from 1; gnorm_scale multiplies the gradient.
 * qb200_managed_alloc is the ONE allocating entry point (cudaMallocManaged, like upstream's cget_managed_ptr); the
 * caller owns the memory and releases it with qb200_managed_free.  qb200_prefetch: device < 0 = host. */
int qb200_adamw32bit_step(void* p, int dtype, const void* g, float* m, float* v, int64_t n, float lr, float beta1,
                          float beta2, float eps, float weight_decay, int step, float gnorm_scale, void* stream);
/* Graph-capturable form: `step_dev` is a DEVICE float holding the step count (from 1), `gnorm_scale_dev` an optional DEVICE
 * float multiplying the gradient (e.g. the clip coefficient of --max_grad_norm 0.3); nothing host-side changes per step. */
int qb200_adamw32bit_step_dev(void* p, int dtype, const void* g, float* m, float* v, int64_t n, float lr, float beta1,
                              float beta2, float eps, float weight_decay, const float* step_dev, const float* gnorm_scale_dev,
                              void* stream);
/* ---- 32-bit Lion, RMSprop and AdEMAMix (optim='lion_32bit', 'rmsprop_bnb', 'ademamix' and their paged forms) -----------
 * Replace clion32bit_grad_*, crmsprop32bit_grad_* (kOptimizer32bit1State<T, LION | RMSPROP>) and cademamix32bit_grad_*
 * (kOptimizer32bit2State<T, ADEMAMIX>).  One fused elementwise pass each: p, g of `dtype`; state fp32; every operation a
 * correctly rounded fp32 one.  `gnorm_scale_dev` is an optional DEVICE float multiplying the gradient.  They allocate nothing
 * and read no host state per step, so one captured launch can be replayed every step.
 *   Lion:     c = b1*m + (1-b1)*g; if (wd > 0) p *= 1 - lr*wd; p -= lr*sign(c); m = b2*m + (1-b2)*g.  `step_dev` is unused.
 *   RMSprop:  if (wd > 0) g += wd*p; v = alpha*v + (1-alpha)*g*g; p -= lr*(g / (sqrt(v) + eps)).  `step_dev` is unused.
 *   AdEMAMix: `step_dev` is a DEVICE float holding the step count t (from 1); m1, m2 the fast and slow EMAs, nu the second
 *             moment.  t_alpha, t_beta3 > 0 set the warm-up schedules of alpha and beta3, 0 means none; a negative or NaN
 *             value returns QB200_EINVAL.
 * Null pointers, n < 0 and an unknown dtype return QB200_EINVAL before any launch. */
int qb200_lion32bit_step_dev(void* p, int dtype, const void* g, float* m, int64_t n, float lr, float beta1, float beta2,
                             float weight_decay, const float* step_dev, const float* gnorm_scale_dev, void* stream);
int qb200_rmsprop32bit_step_dev(void* p, int dtype, const void* g, float* v, int64_t n, float lr, float alpha, float eps,
                                float weight_decay, const float* step_dev, const float* gnorm_scale_dev, void* stream);
int qb200_ademamix32bit_step_dev(void* p, int dtype, const void* g, float* m1, float* m2, float* nu, int64_t n, float lr, float beta1,
                                 float beta2, float beta3, float alpha, float t_alpha, float t_beta3, float eps, float weight_decay,
                                 const float* step_dev, const float* gnorm_scale_dev, void* stream);
int qb200_managed_alloc(int64_t bytes, void** out);
int qb200_managed_free(void* ptr);
int qb200_prefetch(const void* ptr, int64_t bytes, int device, void* stream);

/* ---- upstream-named compatibility aliases -------------------------------------------
 * Same symbols and argument order bitsandbytes' ctypes layer binds (>=0.45 spelling,
 * with the trailing stream on dequantize); void return like upstream, errors are
 * recorded in qb200_last_error() instead of exit(1). `code` is ignored for NF4. */
void cquantize_blockwise_fp32_nf4(float* code, float* A, float* absmax, unsigned char* out, int blocksize, const int n);
void cquantize_blockwise_fp16_nf4(float* code, void* A, float* absmax, unsigned char* out, int blocksize, const int n);
void cquantize_blockwise_bf16_nf4(float* code, void* A, float* absmax, unsigned char* out, int blocksize, const int n);
void cdequantize_blockwise_fp32_nf4(float* code, unsigned char* A, float* absmax, float* out, int blocksize, const int n, void* stream);
void cdequantize_blockwise_fp16_nf4(float* code, unsigned char* A, float* absmax, void* out, int blocksize, const int n, void* stream);
void cdequantize_blockwise_bf16_nf4(float* code, unsigned char* A, float* absmax, void* out, int blocksize, const int n, void* stream);
void cquantize_blockwise_fp32(float* code, float* A, float* absmax, unsigned char* out, int blocksize, const int n);
void cdequantize_blockwise_fp32(float* code, unsigned char* A, float* absmax, float* out, int blocksize, const int n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* QLORA_B200_H_ */
