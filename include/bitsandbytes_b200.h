/*
 * bitsandbytes_b200.h -- the C ABI of libbitsandbytes_b200.so (sm_90a only).
 *
 * This is the drop-in boundary: every symbol in section 1 has the SAME name,
 * argument order and argument meaning as the symbol the reference's Python layer
 * binds through ctypes (reference bitsandbytes/cextension.py loads the library,
 * bitsandbytes/backends/cuda/ops.py:16-66 declares the argtypes).  The reference
 * definitions are in csrc/pythonInterface.cpp and csrc/gemm_4bit.cu; each
 * declaration below cites the line it replaces.
 *
 * Conventions (identical to the reference, SURVEY.md section 8b):
 *   - plain C ABI, no name mangling, no torch types;
 *   - pointers are raw DEVICE pointers (tensor.data_ptr()); NULL where noted;
 *   - element counts are 32-bit `int`;
 *   - `stream` is a cudaStream_t passed as void*;
 *   - the caller allocates every buffer, outputs included; the library keeps no
 *     pointer after return and allocates no device memory on this path, except a
 *     stream-ordered split-K scratch (cudaMallocAsync/cudaFreeAsync on `stream`)
 *     inside cgemm_4bit_* for mid-sized M;
 *   - kernels are asynchronous on `stream`; the caller selects the device.
 *
 * Error behaviour: the reference prints and calls exit(1) when a launch fails
 * (csrc/compat.cuh:78-85).  This library instead records the failure; the host
 * layer polls cbnb_b200_last_error() after every call and raises.  `void` entry
 * points stay `void`.
 *
 * Section 2 holds native additions (stream-taking quantize, fused int8 linear,
 * sharded-linear helpers).  Section 3 lists symbols the reference loader insists on
 * (cextension.py:112-115) that are outside the hot path; they exist and fail loudly.
 */
#ifndef BITSANDBYTES_B200_H
#define BITSANDBYTES_B200_H

#include <stddef.h>
#include <stdbool.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* bnb_stream_t;  /* cudaStream_t */
typedef uint16_t bnb_half;   /* IEEE fp16 bits  */
typedef uint16_t bnb_bf16;   /* bfloat16 bits   */

/* =====================================================================
 * 1. Reference-compatible hot-path symbols
 * ===================================================================== */

/* ---- blockwise dequantize: out[i] = T(value(A[i]) * absmax[i / blocksize]) ----
 * n = number of OUTPUT elements.  8-bit variants take the 256-entry `code`;
 * _nf4/_fp4 variants ignore `code` (NULL allowed), A holds two codes per byte,
 * element 2b in the high nibble.
 * Replaces reference csrc/pythonInterface.cpp:346-362 (fp16), :392-408 (fp32),
 * :428-444 (bf16); kernel csrc/kernels.cu:465-529. */
void cdequantize_blockwise_fp32(float* code, unsigned char* A, float* absmax, float* out, int blocksize, int n, bnb_stream_t stream);
void cdequantize_blockwise_fp32_fp4(float* code, unsigned char* A, float* absmax, float* out, int blocksize, int n, bnb_stream_t stream);
void cdequantize_blockwise_fp32_nf4(float* code, unsigned char* A, float* absmax, float* out, int blocksize, int n, bnb_stream_t stream);
void cdequantize_blockwise_fp16(float* code, unsigned char* A, float* absmax, bnb_half* out, int blocksize, int n, bnb_stream_t stream);
void cdequantize_blockwise_fp16_fp4(float* code, unsigned char* A, float* absmax, bnb_half* out, int blocksize, int n, bnb_stream_t stream);
void cdequantize_blockwise_fp16_nf4(float* code, unsigned char* A, float* absmax, bnb_half* out, int blocksize, int n, bnb_stream_t stream);
void cdequantize_blockwise_bf16(float* code, unsigned char* A, float* absmax, bnb_bf16* out, int blocksize, int n, bnb_stream_t stream);
void cdequantize_blockwise_bf16_fp4(float* code, unsigned char* A, float* absmax, bnb_bf16* out, int blocksize, int n, bnb_stream_t stream);
void cdequantize_blockwise_bf16_nf4(float* code, unsigned char* A, float* absmax, bnb_bf16* out, int blocksize, int n, bnb_stream_t stream);

/* ---- blockwise quantize: absmax[b] = max|A| over block b; out = codes ----
 * NO stream argument in the reference ABI: launches on the legacy default stream
 * (reference csrc/ops.cu:44-63).  n = number of INPUT elements.
 * Replaces reference csrc/pythonInterface.cpp:364-390 (fp16, fp32), :410-426 (bf16);
 * kernels csrc/kernels.cu:269-463. */
void cquantize_blockwise_fp32(float* code, float* A, float* absmax, unsigned char* out, int blocksize, int n);
void cquantize_blockwise_fp32_fp4(float* code, float* A, float* absmax, unsigned char* out, int blocksize, int n);
void cquantize_blockwise_fp32_nf4(float* code, float* A, float* absmax, unsigned char* out, int blocksize, int n);
void cquantize_blockwise_fp16(float* code, bnb_half* A, float* absmax, unsigned char* out, int blocksize, int n);
void cquantize_blockwise_fp16_fp4(float* code, bnb_half* A, float* absmax, unsigned char* out, int blocksize, int n);
void cquantize_blockwise_fp16_nf4(float* code, bnb_half* A, float* absmax, unsigned char* out, int blocksize, int n);
void cquantize_blockwise_bf16(float* code, bnb_bf16* A, float* absmax, unsigned char* out, int blocksize, int n);
void cquantize_blockwise_bf16_fp4(float* code, bnb_bf16* A, float* absmax, unsigned char* out, int blocksize, int n);
void cquantize_blockwise_bf16_nf4(float* code, bnb_bf16* A, float* absmax, unsigned char* out, int blocksize, int n);

/* ---- 4-bit dequant-fused GEMM: out[M,N] = A[M,K] . dequant(B)[N,K]^T + bias ----
 * B: packed codes of the row-major [N,K] weight; absmax: fp32 per block, or -- when
 * absmax_8bit != NULL (double quant) -- the level-2 absmax with
 *   scale[i] = absmax_code[absmax_8bit[i]] * absmax[i >> 8] + *absmax_offset.
 * quant_type: 1 = FP4, 2 = NF4.  bias may be NULL.  K % blocksize == 0 required.
 * Replaces reference csrc/gemm_4bit.cu:136-168 (dispatch :45-134; kernels
 * gemm_4bit_simt.cu:109-480, gemm_4bit_sm80.cu:127-457). */
void cgemm_4bit_bf16(const bnb_bf16* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, bnb_bf16* out, const bnb_bf16* bias, int M, int N, int K, int blocksize, int quant_type, bnb_stream_t stream);
void cgemm_4bit_fp16(const bnb_half* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, bnb_half* out, const bnb_half* bias, int M, int N, int K, int blocksize, int quant_type, bnb_stream_t stream);
void cgemm_4bit_fp32(const float* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, float* out, const float* bias, int M, int N, int K, int blocksize, int quant_type, bnb_stream_t stream);

/* ---- legacy GEMV behind F.gemv_4bit: out[m] = sum_k A[k] * datatype[B[m,k]] * absmax ----
 * m = N (output features), n = 1, k = K; `datatype` = 16 fp32 code values.
 * Replaces reference csrc/pythonInterface.cpp:594-613; kernel csrc/kernels.cu:1452-1567. */
void cgemm_4bit_inference_naive_fp16(int m, int n, int k, bnb_half* A, unsigned char* B, float* absmax, float* datatype, bnb_half* out, int lda, int ldb, int ldc, int blocksize, bnb_stream_t stream);
void cgemm_4bit_inference_naive_bf16(int m, int n, int k, bnb_bf16* A, unsigned char* B, float* absmax, float* datatype, bnb_bf16* out, int lda, int ldb, int ldc, int blocksize, bnb_stream_t stream);
void cgemm_4bit_inference_naive_fp32(int m, int n, int k, float* A, unsigned char* B, float* absmax, float* datatype, float* out, int lda, int ldb, int ldc, int blocksize, bnb_stream_t stream);

/* ---- LLM.int8() ----
 * get_context: reference csrc/pythonInterface.cpp:522 returns a heap Context*
 * (cuBLAS handle).  Here the GEMM is our own kernel; the returned pointer is an
 * opaque non-NULL token kept only for ABI compatibility. */
void* get_context(void);

/* C_i32[M,N] = acts_i8[M,K] . weights_i8[N,K]^T, exact.  Argument naming follows the
 * reference's column-major view: m = N (weight rows), n = M (tokens), k = K;
 * A = weights [N,K], B = activations [M,K], lda = ldb = K, ldc = N; row_scale unused.
 * Returns 0 on success, 100 (ERR_NOT_IMPLEMENTED) if k % 16 != 0 (caller falls back).
 * Replaces reference csrc/pythonInterface.cpp:524-529; csrc/ops.cu:282-404 (cublasLtMatmul). */
int cigemmlt_32(void* context, int m, int n, int k, const int8_t* A, const int8_t* B, void* C, float* row_scale, int lda, int ldb, int ldc, bnb_stream_t stream);

/* out_fp16 = fp16( fma( float(A_i32) * rowStats[r] * colStats[c], 6.200012e-05f, bias[c] ) )
 * Replaces reference csrc/pythonInterface.cpp:545-549; kernel csrc/kernels.cu:1396-1448. */
void cdequant_mm_int32_fp16(int* A, float* rowStats, float* colStats, bnb_half* out, bnb_half* bias, int numRows, int numCols, bnb_stream_t stream);

/* Row-wise absmax int8 quantisation of fp16 A[rows, cols]; |a| >= threshold excluded
 * from the row statistic and written as 0 when threshold > 0.
 * Replaces reference csrc/pythonInterface.cpp:551-555; kernel csrc/kernels.cu:1331-1385. */
void cint8_vector_quant(bnb_half* A, int8_t* out, float* rowStats, float threshold, int rows, int cols, bnb_stream_t stream);

/* Element-wise helpers of the reference's paged-memory utilities: A[i] = value, A[i] = i, A[i] *= B[i]
 * (legacy default stream, as in the reference).  Outside the hot path; present so that the reference's loader and
 * its functional.fill / arange / _mul helpers find them.
 * Replaces reference csrc/pythonInterface.cpp:586-592; kernel csrc/kernels.cu:1569-1583. */
void cfill_fp32(float* A, float* B, float value, long n);
void cfill_uint8(unsigned char* A, unsigned char* B, unsigned char value, long n);
void carange_fp32(float* A, float* B, float value, long n);
void c_mul_fp32(float* A, float* B, float value, long n);

/* =====================================================================
 * 2. Native additions (no reference counterpart)
 * ===================================================================== */

/* 0 = no error since the last call; otherwise a code, with a message retrievable below.
 * Polling clears the flag. */
int cbnb_b200_last_error(void);
const char* cbnb_b200_last_error_message(void);
/* "sm_90a; wgmma ..." build description */
const char* cbnb_b200_build_info(void);

/* Stream-taking quantize (the reference ABI above has none).  quant_type 0/1/2,
 * dtype 0 = fp32, 1 = fp16, 2 = bf16. */
void cbnb_b200_quantize_blockwise(const float* code, const void* A, float* absmax, unsigned char* out, int blocksize, int n, int quant_type, int dtype, bnb_stream_t stream);

/* Fused all-gather for a column-sharded layer (no reference counterpart: the reference is single-device).
 * The wgmma kernel's epilogue stores every output element to outs[0..n_outs): outs[0] is the local
 * [M, ldc] buffer, the others the same location in the peer GPUs' buffers mapped into this process
 * (CUDA IPC / symmetric memory), so the exchange rides on the GEMM's own stores over NVLink.
 * `outs` is a HOST array.  Returns 0, or 100 if the shape does not take the wgmma path. */
int cbnb_b200_gemm_4bit_multi_out(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, void* const* outs, int n_outs, const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, bnb_stream_t stream);

/* Which kernel a (M, N, K, blocksize, dtype) 4-bit GEMM takes: 0 = CUDA-core GEMV,
 * 1 = wgmma GEMM, 2 = generic CUDA-core kernel, 3 = mma.sync decode kernel (M <= 8).
 * For tests / bench bookkeeping. */
int cbnb_b200_gemm_4bit_path(int M, int N, int K, int blocksize, int dtype);
/* Force a path for the next calls on this thread (-1 = automatic). */
void cbnb_b200_gemm_4bit_force_path(int path);

/* Developer / test entry for the wgmma 4-bit GEMM (csrc/gemm4_tc.cu): explicit token tile mt (16 | 32 | 64 | 128;
 * 0 = by M) and forced K split per tile (0 = production rule; s = up to s ways, at least one 128-deep stage per
 * split).  `trace` must be NULL (the name and argument list are kept for ABI stability).  Returns 0, or 100 when
 * the shape or the options are not served (a forced split must fit one co-resident wave of CTAs). */
int cbnb_b200_gemm_4bit_pair(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, void* out, const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, int mt, int force_splits, long long* trace, bnb_stream_t stream);

/* Strided-output variant used by the column-sharded linear: out has row stride ldc
 * (elements), so a shard writes its [M, N_shard] block into the gathered [M, N]. */
void cbnb_b200_gemm_4bit_strided(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, void* out, const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, bnb_stream_t stream);

/* Fused LLM.int8() linear: out[M,N] = T( (CA . CB^T) * SCA[m] * SCB[n] / 127^2 + bias[n] ),
 * int8 wgmma GEMM with the dequant epilogue in-kernel (no int32 round trip through HBM).
 * dtype 1 = fp16, 2 = bf16.  Returns 0 / 100 like cigemmlt_32. */
int cbnb_b200_int8_scaled_mm(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB, const void* bias, void* out, int M, int N, int K, int dtype, bnb_stream_t stream);

/* LLM.int8() mixed decomposition (reference backends/default/ops.py:64-100) in ONE GEMM launch: the int8 part as
 * cbnb_b200_int8_scaled_mm plus, in the same epilogue, the outlier term subA[M, jpad] . subBT[N, jpad]^T
 * (operands of the output type, fp32 accumulation), added to the rounded int8 result and rounded once more, as
 * the reference's `output.addmm(subA, subB)` does.  jpad: multiple of 8, <= 64.  Returns 0 / 100. */
int cbnb_b200_int8_mixed_mm(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB, const void* bias, const void* subA, const void* subBT, int jpad, void* out, int M, int N, int K, int dtype, bnb_stream_t stream);

/* Builds the two operands of the outlier term in one launch: subA[m, j] = A[m, cols[j]] and
 * subBT[n, j] = T((float(CB[n, cols[j]]) * SCB[n]) * (1/127))  (reference _ops.py:118-121), zero-padded from J to
 * jpad columns.  cols: J int64 column indices on the device (torch.nonzero of the outlier flags). */
void cbnb_b200_int8_outlier_prep(const void* A, const int8_t* CB, const float* SCB, const long long* cols, int J, int jpad, int M, int N, int K, int dtype, void* subA, void* subBT, bnb_stream_t stream);

/* Column-wise half of int8_double_quant (reference backends/cuda/ops.py:262-296: five PyTorch kernels there):
 * col_stats[c] = max_r |A[r,c]| over the entries below `threshold` (all entries when threshold == 0),
 * out[r,c] = int8(rint(float(T(A[r,c] * 127)) / col_stats[c])), outliers -> 0.  dtype 1 = fp16, 2 = bf16.  Returns 0 / 100. */
int cbnb_b200_int8_col_quant(const void* A, int8_t* out, float* col_stats, float threshold, int rows, int cols, int dtype, bnb_stream_t stream);

/* CA[:, cols[j]] = 0 for the J outlier columns (reference backends/cuda/ops.py:233-236). */
void cbnb_b200_int8_zero_columns(int8_t* CA, const long long* cols, int J, int rows, int K, bnb_stream_t stream);

/* Fused row quantisation + outlier-column detection without a host sync:
 * col_flags[c] = 1 if any |A[r,c]| >= threshold.  dtype 1 = fp16, 2 = bf16 (A is read as
 * that type; the reference kernel is fp16-only). */
void cbnb_b200_int8_vector_quant_flags(const void* A, int8_t* out, float* rowStats, int* col_flags, float threshold, int rows, int cols, int dtype, bnb_stream_t stream);

/* =====================================================================
 * 3. Present for loader compatibility, outside the hot path
 * ===================================================================== */
/* cextension.py:114-115 sets .restype on these at load time; they must resolve. */
void* cget_managed_ptr(size_t bytes);
void cprefetch(void* ptr, size_t bytes, int device);
/* exported by the reference, unused by its Python layer (SURVEY.md section 2.2). */
int cigemmlt_8(void* context, int m, int n, int k, const int8_t* A, const int8_t* B, void* C, float* row_scale, int lda, int ldb, int ldc, bnb_stream_t stream);
int cigemmlt_8_rowscale(void* context, int m, int n, int k, const int8_t* A, const int8_t* B, void* C, float* row_scale, int lda, int ldb, int ldc, bnb_stream_t stream);

/* =====================================================================
 * 4. Optimizers (SURVEY.md section 8 row f-4)
 * ===================================================================== */
/* Replaces reference csrc/pythonInterface.cpp:446-473 (MAKE_CFUNC32; bound in bitsandbytes/backends/cuda/ops.py:985-1031):
 * one in-place update of p (dtype of g) with fp32 state; max_unorm > 0 first accumulates the squared update norm in
 * unorm[0] (LAMB / LARS trust ratio).  Legacy default stream, like the reference.
 * Full list: c{adam,lion,ademamix}32bit_grad_{fp32,fp16,bf16}, c{momentum,rmsprop,adagrad}32bit_grad_{32,16}. */
void cadam32bit_grad_fp32(float* g, float* p, float* state1, float* state2, float* unorm, float max_unorm, float param_norm, const float beta1, const float beta2, const float beta3, const float alpha, const float eps, const float weight_decay, const int step, const float lr, const float gnorm_scale, bool skip_zeros, const int n);
/* Replaces reference csrc/pythonInterface.cpp:475-520 (MAKE_CBLOCKWISE8; bound in backends/cuda/ops.py:1033-1066):
 * blockwise (256) 8-bit state: state bytes + per-block absmax + 256-entry code books (quantiles).
 * Full list: c{adam,momentum,rmsprop,adagrad,lion,ademamix}_8bit_blockwise_grad_{fp32,fp16,bf16}. */
void cadam_8bit_blockwise_grad_fp32(float* p, float* g, unsigned char* state1, unsigned char* state2, float beta1, float beta2, float beta3, float alpha, float eps, int step, float lr, float* quantiles1, float* quantiles2, float* absmax1, float* absmax2, float weight_decay, const float gnorm_scale, bool skip_zeros, int n);
/* The same two updates with an explicit stream, 64-bit element count, optimizer id (0 adam/lamb, 1 momentum/lars,
 * 2 rmsprop, 3 adagrad, 4 lion, 5 ademamix) and dtype id (0 fp32, 1 fp16, 2 bf16).  Return 0, or 100 for an unknown id. */
int cbnb_b200_optimizer_update_32bit(int optimizer, int dtype, const void* g, void* p, float* state1, float* state2, float* unorm, float max_unorm, float param_norm, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, int step, float lr, float gnorm_scale, bool skip_zeros, long long n, bnb_stream_t stream);
int cbnb_b200_optimizer_update_8bit_blockwise(int optimizer, int dtype, void* p, const void* g, unsigned char* state1, unsigned char* state2, float beta1, float beta2, float beta3, float alpha, float eps, int step, float lr, const float* quantiles1, const float* quantiles2, float* absmax1, float* absmax2, float weight_decay, float gnorm_scale, bool skip_zeros, long long n, bnb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* BITSANDBYTES_B200_H */
