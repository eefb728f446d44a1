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

/* Partial GEMM of a row-sharded layer (input features split across ranks; no reference counterpart).
 * outs[0..n_outs)[m, n] (fp32, row stride ldc) = sum_k A[m, k] * W[n, k], accumulated in fp32 with no bias and no
 * rounding, by the kernel and K split the plain 4-bit GEMM takes for the same shape and dtype (0 = fp32, 1 = fp16,
 * 2 = bf16, 3 = fp32 with TF32 allowed; see cbnb_b200_gemm_4bit_path).  `outs` is a HOST array of at most 8 device
 * addresses: the local buffer and, for the fused exchange, the same slot in the peers' buffers.  Returns 0, 1 for a bad
 * destination list, or 100 for a dtype it does not serve. */
int cbnb_b200_gemm_4bit_partial(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, float* const* outs, int n_outs, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, bnb_stream_t stream);

/* The partial GEMM of a sequence-parallel row-sharded layer: cbnb_b200_gemm_4bit_partial (same kernel, K split and
 * fp32 sums) with the rows scattered instead of copied.  Row m is stored to outs[m / rows_per_out] at row
 * m % rows_per_out (row stride ldc), so `outs` is in RANK order: outs[s] receives the tokens of rank s.  Returns 0, 1
 * unless 1 <= n_outs <= 8, rows_per_out >= 1 and n_outs * rows_per_out == M (error message set), or 100 for a dtype it
 * does not serve. */
int cbnb_b200_gemm_4bit_partial_scatter(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, float* const* outs, int n_outs, int rows_per_out, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, bnb_stream_t stream);

/* out[m, n] (row stride ldc) = T( (((P_0 + P_1) + ...) + P_{world-1})[m, n] + bias[n] ), P_r = parts + r * part_stride,
 * each [M, N] fp32 with row stride N: the partials summed in rank order in fp32, the bias (T[N] or NULL) added in fp32,
 * one rounding to T.  dtype 0 or 3 = fp32, 1 = fp16, 2 = bf16.  Returns 0, or 100 for a dtype or argument it does not
 * serve. */
int cbnb_b200_reduce_partials(const float* parts, int world, long long part_stride, void* out, const void* bias, int M, int N, int ldc, int dtype, bnb_stream_t stream);

/* cbnb_b200_reduce_partials over n_parts (1..8) separate [M, N] fp32 partials, parts[r] in rank order (a rank's own
 * buffer or a peer's symmetric-memory mapping), restricted to the rows [row0, row0 + rows): out[m, n] (row stride ldc,
 * m < rows) = T( (((P_0 + P_1) + ...) + P_{n_parts-1})[row0 + m, n] + bias[n] ), the same bits as
 * cbnb_b200_reduce_partials.  Returns 0, 1 with the error message set for bad arguments (n_parts outside 1..8, a null
 * or misaligned pointer, a window past M, ldc < N), or 100 for a dtype it does not serve. */
int cbnb_b200_reduce_partials_ptrs(const float* const* parts, int n_parts, int row0, int rows, void* out, const void* bias, int M, int N, int ldc, int dtype, bnb_stream_t stream);

/* Which kernel a (M, N, K, blocksize, dtype) 4-bit GEMM takes: 0 = CUDA-core GEMV,
 * 1 = wgmma GEMM, 2 = generic CUDA-core kernel, 3 = mma.sync decode kernel (M <= 8).
 * dtype for the 4-bit GEMM entries below: 0 = fp32, 1 = fp16, 2 = bf16, 3 = fp32 with TF32 allowed -- the
 * caller's fp32 matmul precision is "tf32": from 4 tokens on (K % 64 == 0, power-of-two blocksize >= 32) the
 * wgmma GEMM runs on TF32 tensor cores with weights rna_tf32(fp32 dequantised weight); otherwise as dtype 0.
 * For tests / bench bookkeeping. */
int cbnb_b200_gemm_4bit_path(int M, int N, int K, int blocksize, int dtype);
/* 1 when an unforced path-1 call takes the staged route (fp16 / bf16, large M: each weight panel decoded once into a
 * per-stream workspace, then the wgmma GEMM on shared-memory operands; the same bits as the fused kernel), else 0.
 * A forced path 1 always runs the fused kernel. */
int cbnb_b200_gemm_4bit_staged_route(int M, int N, int K, int blocksize, int dtype);
/* Force a path for the next calls on this thread (-1 = automatic). */
void cbnb_b200_gemm_4bit_force_path(int path);

/* Developer / test entry for the wgmma 4-bit GEMM (csrc/gemm4_tc.cu): explicit token tile mt (16 | 32 | 64 | 128 |
 * 256, at most 128 for dtype 3; 0 = by M) and forced K split per tile (0 = production rule; s = up to s ways, at
 * least one stage per split: 128 deep, 64 deep at mt = 256 and for dtype 3).  dtype 1, 2 or 3 (TF32).  `trace` must be NULL (the name and argument list are kept for ABI stability).  Returns 0, or 100 when
 * the shape or the options are not served (a forced split must fit one co-resident wave of CTAs). */
int cbnb_b200_gemm_4bit_pair(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, void* out, const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, int mt, int force_splits, long long* trace, bnb_stream_t stream);

/* Grouped 4-bit GEMM of a mixture-of-experts layer (no reference counterpart; the 4-bit form of grouped_mm with a 3-D
 * weight): out[m, :] (row stride ldc) = T( A[m, :] . W_e^T (fp32 accumulation) + bias[e * N .. (e + 1) * N) ) for the
 * rows of expert e, end_{e-1} <= m < end_e, and 0 for end_{E-1} <= m < M.  A is [M, K] fp16 / bf16 (dtype 1 / 2) with
 * rows sorted by expert; B, absmax (and the nested statistics) are E experts' [N, K] weights quantised as ONE [E * N, K]
 * tensor, expert e being rows [e * N, (e + 1) * N); bias is T[E * N] or NULL; offs is int32[E] on the device, offs[e]
 * the end row of expert e, clamped on the device as end_e = min(max(offs[e], end_{e-1}), M) (end_{-1} = 0), so that no
 * routing makes the kernel read or write outside its operands.  Each expert's rows are bit for bit those of
 * cbnb_b200_gemm_4bit_pair on that expert alone at the same token tile with force_splits = 1.  Nothing is read back to
 * the host: the call can be captured in a CUDA graph.  Returns 0, 1 with the error message set for bad arguments (NULL
 * operand, M < 0, N, K or E < 1, ldc < N, bad quant_type, absmax_8bit without absmax_code), or 100 with nothing
 * written for what it does not serve: fp32 A (dtype 0 / 3), K not a multiple of 64, E > 1024, a blocksize that is not a
 * power of two >= 32, A or B not 16-byte aligned.  A failure past those checks (a tensor map the driver does not encode,
 * a failed shared-memory opt-in or launch) also returns 100, with the error message set: 100 with no message means
 * "not served", 100 with a message an error (the Python layer polls the message first and raises it).  The _mt form is the test entry with token tile mt (16 | 32 | 64 |
 * 128; 0 = the production rule, the smallest of those that holds 2 ceil(M / E) tokens). */
int cbnb_b200_gemm_4bit_grouped(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, const int* offs, int E, void* out, const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, bnb_stream_t stream);
int cbnb_b200_gemm_4bit_grouped_mt(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, const int* offs, int E, void* out, const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, int mt, bnb_stream_t stream);

/* Row-sharded (input-feature-sharded) expert layers.  cbnb_b200_gemm_4bit_grouped_partial: out[m, n] (fp32, row stride
 * ldc) = A[m, :] . W_e[n, :] summed in fp32, no bias and no rounding, for the rows of expert e, and 0 for the rows past
 * end_{E-1}; A, B, offs as in cbnb_b200_gemm_4bit_grouped, absmax plain fp32 (a shard never carries nested statistics).
 * mt: token tile 16 | 32 | 64 | 128, 0 = the grouped GEMM's rule for (M, E).  With the same tile, T(P + bias_e) is
 * cbnb_b200_gemm_4bit_grouped_mt's output bit for bit.  Returns 0; 1 with the error message set for bad arguments
 * (NULL operand, M < 0, N, K or E < 1, ldc < N, bad quant_type or mt); 100 with nothing written for what it does not
 * serve (fp32 A, K not a multiple of 64, E > 1024, a bad blocksize, misaligned A or B), or 100 with the message set
 * when a launch fails.
 * cbnb_b200_reduce_partials_grouped: out[m, n] (row stride ldc) = T(((parts[0] + parts[1]) + ... + parts[world-1])[m, n]
 * + bias[e * N + n]) for the rows of expert e (end rows clamped on the device from offs, as the grouped GEMM does), 0
 * for the rows past end_{E-1}; the partials [M, N] at row stride N, one every part_stride elements; bias T[E * N] or
 * NULL.  The element arithmetic of cbnb_b200_reduce_partials.  dtype 1 = fp16, 2 = bf16.  Returns 0, or 100 for a dtype,
 * world or E (1..1024) it does not serve.  Neither call reads offs on the host. */
int cbnb_b200_gemm_4bit_grouped_partial(const void* A, const uint8_t* B, const float* absmax, const int* offs, int E, float* out, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, int mt, bnb_stream_t stream);
int cbnb_b200_reduce_partials_grouped(const float* parts, int world, long long part_stride, const int* offs, int E, void* out, const void* bias, int M, int N, int ldc, int dtype, bnb_stream_t stream);

/* Developer / test entries for the staged route.  _staged: the whole route with token tile mt (128 | 256,
 * 0 = by the shape) and panel_rows output features per panel (a multiple of 128 whose decoded rows fit the 32 MB
 * per-stream workspace, 0 = the largest such), stores to outs[0..n_outs) as _multi_out; returns 0, or 100 when not
 * served.  _dequantize_4bit_panel: rows [n0, n0 + rows) of a [N, K] 4-bit weight decoded into out[rows, K]
 * (n0 % 128 == 0), bit-identical to the same rows of F.dequantize_4bit.  _gemm_decoded: the staged GEMM alone,
 * out[M, N] = A[M, K] . W[N, K]^T (+ bias) on an already decoded W.  dtype 1 = fp16, 2 = bf16. */
int cbnb_b200_gemm_4bit_staged(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, void* const* outs, int n_outs, const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype, int mt, int panel_rows, bnb_stream_t stream);
int cbnb_b200_dequantize_4bit_panel(const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset, void* out, int blocksize, int quant_type, int dtype, int n0, int rows, int K, bnb_stream_t stream);
int cbnb_b200_gemm_decoded(const void* A, const void* W, void* out, const void* bias, int M, int N, int K, int ldc, int dtype, int mt, bnb_stream_t stream);

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

/* The weight of LLM.int8()'s input gradient in one pass: out[n, k] (row stride ldo >= cols) =
 * T(float(CB[n, k]) * s[n]), s[n] = SCB[n] * fp32(1/127), the bits of `CB.to(T).mul_(SCB.unsqueeze(1).mul(1.0 / 127.0))`.
 * CB [rows, cols] int8 contiguous, SCB [rows] fp32.  dtype 1 = fp16, 2 = bf16.  Returns 0; 1 with the error message set
 * for bad arguments; 100, with nothing written, for any other dtype. */
int cbnb_b200_int8_dequant_rows(const int8_t* CB, const float* SCB, void* out, int ldo, int rows, int cols, int dtype, bnb_stream_t stream);

/* CA[:, cols[j]] = 0 for the J outlier columns (reference backends/cuda/ops.py:233-236). */
void cbnb_b200_int8_zero_columns(int8_t* CA, const long long* cols, int J, int rows, int K, bnb_stream_t stream);

/* The same decomposition with the outlier columns and their count kept on the device: no launch depends on them, so
 * the three calls below can be captured once in a CUDA graph and replayed for any outlier set.
 *
 * cols[0 .. *count) = the flagged columns of col_flags[K] in ascending order (what torch.nonzero gives), and *count.
 * cols holds K ints.  One CTA. */
void cbnb_b200_int8_outlier_compact(const int* col_flags, int K, int* cols, int* count, bnb_stream_t stream);

/* CA[:, cols[j]] = 0 for every j < *count, and the outlier operands at a fixed capacity of 64 columns:
 * subA[M, 64] and subBT[N, 64] as cbnb_b200_int8_outlier_prep builds them for j < min(*count, 64), zeros after. */
void cbnb_b200_int8_outlier_prep_dev(const void* A, int8_t* CA, const int8_t* CB, const float* SCB, const int* cols, const int* count, int M, int N, int K, int dtype, void* subA, void* subBT, bnb_stream_t stream);

/* cbnb_b200_int8_mixed_mm with J = *count read on the device.  The first min(J, 64) outlier columns come from
 * subA / subBT [*, 64]; columns 64 .. J-1 are gathered from A (T[M, K]) and CB through cols, 64 at a time, and continue
 * the same fp32 sum in column order.  For J <= 64 the result is bit-identical to cbnb_b200_int8_mixed_mm (J = 0: to
 * cbnb_b200_int8_scaled_mm).  Returns 0 / 100. */
int cbnb_b200_int8_mixed_mm_dev(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB, const void* bias, const void* A, const void* subA, const void* subBT, const int* cols, const int* count, void* out, int M, int N, int K, int dtype, bnb_stream_t stream);

/* Grouped LLM.int8() GEMM of a mixture-of-experts layer (no reference counterpart).  CB [E * N, K] int8 and SCB [E * N]
 * are E experts' [N, K] weights quantised row-wise as one tensor; offs[E] (int32, on the device) the expert end rows,
 * clamped on the device as end_e = min(max(offs[e], end_{e-1}), M).
 * cbnb_b200_int8_grouped_outliers (threshold > 0): the per-expert outliers, from A (T[M, K]) and A16 (A as fp16, whose
 * row codes and statistics are CA / SCA): ends[E], flags[E, K], each expert's ascending outlier columns cols[E, K] and
 * count[E], subA [M, 64] from each row's own expert's list, subBT [E * N, 64] for the experts with rows, and CA zeroed
 * in each row's expert's outlier columns when the expert has more than one row.  Returns 0 / 1 (bad arguments, message
 * set).
 * cbnb_b200_int8_grouped_mm: out[m, :] (row stride N) = cbnb_b200_int8_scaled_mm (count NULL) or
 * cbnb_b200_int8_mixed_mm_dev (count, cols, subA, subBT and A from cbnb_b200_int8_grouped_outliers) on the rows of expert
 * e alone, with CB / SCB / bias (T[E * N] or NULL) at e * N; rows past end_{E-1} are +0.  Returns 0; 1 for bad arguments
 * (message set); 100 with no message for what is not served (K % 16 != 0, E > 1024); 100 with the message set when the
 * launch fails.  dtype 1 = fp16, 2 = bf16. */
int cbnb_b200_int8_grouped_outliers(const void* A, const void* A16, int8_t* CA, const int8_t* CB, const float* SCB, const int* offs, int E, float threshold, int* ends, int* flags, int* cols, int* count, void* subA, void* subBT, int M, int N, int K, int dtype, bnb_stream_t stream);
int cbnb_b200_int8_grouped_mm(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB, const void* bias, const int* offs, int E, const void* A, const void* subA, const void* subBT, const int* cols, const int* count, void* out, int M, int N, int K, int dtype, bnb_stream_t stream);

/* Fused row quantisation + outlier-column detection without a host sync:
 * col_flags[c] = 1 if any |A[r,c]| >= threshold.  dtype 1 = fp16, 2 = bf16 (A is read as
 * that type; the reference kernel is fp16-only). */
void cbnb_b200_int8_vector_quant_flags(const void* A, int8_t* out, float* rowStats, int* col_flags, float threshold, int rows, int cols, int dtype, bnb_stream_t stream);

/* Tensor-parallel LLM.int8() (bitsandbytes_b200/parallel.py).  All return 0, or 100 with the error message set.
 * The two halves of cbnb_b200_int8_vector_quant_flags, same kernel and rounding: the row statistics and the outlier
 * flags (int32, zeroed by the caller, NULL at threshold 0) without codes; the codes from given row statistics. */
int cbnb_b200_int8_row_stats(const void* A, float* rowStats, int* col_flags, float threshold, int rows, int cols, int dtype, bnb_stream_t stream);
int cbnb_b200_int8_quant_with_stats(const void* A, int8_t* out, const float* rowStats, float threshold, int rows, int cols, int dtype, bnb_stream_t stream);
/* The int8 GEMM (epi 0 int32, 1 fp16, 2 bf16; jpad > 0: the outlier term of cbnb_b200_int8_mixed_mm) storing every
 * output element to each of outs[0..n_outs), n_outs <= 8, row stride ldc.  A shape the kernel does not take (K % 16,
 * alignment, jpad > 64) returns 100 without an error message. */
int cbnb_b200_int8_gemm_multi_out(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB, const void* bias, const void* subA, const void* subBT, int jpad, void* const* outs, int n_outs, int M, int N, int K, int ldc, int epi, bnb_stream_t stream);
/* The int32 partial GEMM of a sequence-parallel K-sharded layer: cbnb_b200_int8_gemm_multi_out at epi 0 with the rows
 * scattered instead of copied.  Row m is stored to outs[m / rows_per_out] at row m % rows_per_out (row stride ldc), so
 * `outs` is in RANK order: outs[s] receives the tokens of rank s.  Returns 0; 1 with the error message set unless
 * 1 <= n_outs <= 8, rows_per_out >= 1, n_outs * rows_per_out == M and ldc >= N; 100 for a shape the kernel does not
 * take (K % 16, alignment). */
int cbnb_b200_int8_gemm_partial_scatter(const int8_t* CA, const int8_t* CB, int32_t* const* outs, int n_outs, int rows_per_out, int M, int N, int K, int ldc, bnb_stream_t stream);
/* out = the int8 GEMM epilogue (dtype 1 fp16, 2 bf16) of sum_r parts[r], the exact int32 partials of a K-sharded
 * layer, with SCA, SCB, bias and, for jpad > 0, the outlier term subA[M, jpad] . subBT[N, jpad]^T. */
int cbnb_b200_int8_reduce_partials(const int* parts, int world, long long part_stride, const float* SCA, const float* SCB, const void* bias, const void* subA, const void* subBT, int jpad, void* out, int M, int N, int ldc, int dtype, bnb_stream_t stream);

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
/* Multi-tensor steps: one kernel launch updates `count` tensors that share the optimizer, the dtype, every scalar and
 * (8-bit) the code books; each tensor brings its pointers, element count and its own step.  The results are those of
 * one single-tensor call per tensor, bit for bit.  state1 / state2 are float (32-bit) or unsigned char (8-bit) arrays;
 * state2 and absmax2 are NULL for one-state optimizers; absmax1 / absmax2 are unused by the 32-bit call.  count may
 * be 0 and at most cbnb_b200_optimizer_multi_capacity(); the 32-bit call has no trust ratio (max_unorm = 0).  Return 0,
 * or 100 with cbnb_b200_last_error_message() set. */
typedef struct bnb_b200_optim_tensor {
    void* p;
    const void* g;
    void* state1;
    void* state2;
    float* absmax1;
    float* absmax2;
    long long n;
    union {
        struct {
            int step;
            int reserved; /* 0 */
        };
        int* step_ptr; /* the _dev entries only (_multi_dev, _peers_dev): the tensor's step counter in device memory */
    };
} bnb_b200_optim_tensor_t;
int cbnb_b200_optimizer_multi_capacity(void);
int cbnb_b200_optimizer_update_32bit_multi(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, float gnorm_scale, bool skip_zeros, bnb_stream_t stream);
int cbnb_b200_optimizer_update_8bit_blockwise_multi(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, const float* quantiles1, const float* quantiles2, float gnorm_scale, bool skip_zeros, bnb_stream_t stream);
/* Capturable multi-tensor steps, for CUDA graphs: as the _multi entries, but each descriptor's step_ptr points to the
 * tensor's int32 step counter in device memory, and lr_dev, if not NULL, points to an fp32 learning rate in device
 * memory that is used instead of lr.  Per call, one kernel does ++*step_ptr for every descriptor, then the update
 * kernel reads the counters and lr_dev, on the same stream: a captured call reads the current values at every replay.
 * Each descriptor needs its own counter.  The results are those of the _multi entries given the advanced steps and the
 * learning rate, bit for bit.  Return 0, or 100 with the message set (also for a NULL step_ptr). */
int cbnb_b200_optimizer_update_32bit_multi_dev(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, const float* lr_dev, float gnorm_scale, bool skip_zeros, bnb_stream_t stream);
int cbnb_b200_optimizer_update_8bit_blockwise_multi_dev(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, const float* lr_dev, const float* quantiles1, const float* quantiles2, float gnorm_scale, bool skip_zeros, bnb_stream_t stream);
/* Data-parallel multi-tensor steps (sharded optimizer state, ZeRO stage 1): each descriptor is a piece of a rank's
 * local flat gradient and parameter buffers of `numel` elements, g = grad_local + o_g and p = param_local + o_p (byte
 * offsets).  The gradient of element i is T(fp32(((G_0[i] + G_1[i]) + ...) + G_{world-1}[i]) * grad_scale), G_r the
 * dtype array at grad_srcs[r] + o_g: an fp32 sum in rank order, rounded once; the parameter is read from p, and the new
 * value is written to param_dsts[d] + o_p for each of the ndst destinations (not to p unless param_local is one of
 * them).  Everything else is the _multi entries' arithmetic with gnorm_scale = 1, bit for bit.  1 <= world, ndst <= 8;
 * AdEMAMix (id 5) is refused.  count <= cbnb_b200_optimizer_peers_capacity().  Return 0; 100 for a bad count or id;
 * 1 for a bad source, destination, base, code book or a piece outside the local buffers -- with
 * cbnb_b200_last_error_message() set and nothing launched. */
int cbnb_b200_optimizer_peers_capacity(void);
int cbnb_b200_optimizer_update_32bit_multi_peers(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, const void* const* grad_srcs, int world, void* const* param_dsts, int ndst, const void* grad_local, const void* param_local, long long numel, float grad_scale, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, bool skip_zeros, bnb_stream_t stream);
int cbnb_b200_optimizer_update_8bit_blockwise_multi_peers(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, const void* const* grad_srcs, int world, void* const* param_dsts, int ndst, const void* grad_local, const void* param_local, long long numel, float grad_scale, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, const float* quantiles1, const float* quantiles2, bool skip_zeros, bnb_stream_t stream);
/* Clipped data-parallel steps: the _peers entries plus gnorm_scale_dev, an fp32 factor in device memory (the clip
 * coefficient of cbnb_b200_optimizer_clip_coef) that every CTA reads once and applies where the _multi entries apply
 * gnorm_scale: the results are those of the _multi entries on the reduced gradient with gnorm_scale = *gnorm_scale_dev,
 * bit for bit (fp32 32-bit Lion: as the _peers entries).  NULL means 1: the _peers entries' bits.  Return codes and
 * checks as the _peers entries. */
int cbnb_b200_optimizer_update_32bit_multi_peers_scaled(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, const void* const* grad_srcs, int world, void* const* param_dsts, int ndst, const void* grad_local, const void* param_local, long long numel, float grad_scale, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, bool skip_zeros, const float* gnorm_scale_dev, bnb_stream_t stream);
int cbnb_b200_optimizer_update_8bit_blockwise_multi_peers_scaled(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, const void* const* grad_srcs, int world, void* const* param_dsts, int ndst, const void* grad_local, const void* param_local, long long numel, float grad_scale, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, const float* quantiles1, const float* quantiles2, bool skip_zeros, const float* gnorm_scale_dev, bnb_stream_t stream);
/* Capturable data-parallel steps, for CUDA graphs: the _peers_scaled entries (gnorm_scale_dev NULL: 1) with each
 * descriptor's step_ptr pointing to the tensor's int32 step counter in device memory, as in the _multi_dev entries, and
 * lr_dev, an fp32 value in device memory read in place of lr when not NULL.  These entries read the counters and do NOT
 * advance them, unlike the _multi_dev entries: a parameter's step must advance on every rank, also on ranks that hold
 * no piece of it and for zero-size tensors, so the caller advances its counters (once per step, before the call).  With
 * counters holding k and *lr_dev == lr, the bits of the _peers_scaled entries with step k and that lr.  Return codes
 * and checks as the _peers_scaled entries, plus 100 with the message set for a NULL step_ptr. */
int cbnb_b200_optimizer_update_32bit_multi_peers_dev(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, const void* const* grad_srcs, int world, void* const* param_dsts, int ndst, const void* grad_local, const void* param_local, long long numel, float grad_scale, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, bool skip_zeros, const float* gnorm_scale_dev, const float* lr_dev, bnb_stream_t stream);
int cbnb_b200_optimizer_update_8bit_blockwise_multi_peers_dev(int optimizer, int dtype, const bnb_b200_optim_tensor_t* tensors, int count, const void* const* grad_srcs, int world, void* const* param_dsts, int ndst, const void* grad_local, const void* param_local, long long numel, float grad_scale, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr, const float* quantiles1, const float* quantiles2, bool skip_zeros, const float* gnorm_scale_dev, const float* lr_dev, bnb_stream_t stream);
/* The norm of the reduced gradient over one rank's pieces, for global gradient clipping: each element's gradient is
 * T(fp32 rank-order sum of the world sources * grad_scale), formed as the _peers entries form it, and the call adds
 * the sum of its squares (inf_norm: takes the max of |g|, NaN kept) in fp64 into *acc, in stream order after earlier
 * work: a rank's flats and capacity chunks fold into one value.  Deterministic (fixed per-CTA partials, summed in
 * index order; no floating-point atomics), no host synchronisation.  Only each descriptor's g and n are read; the
 * pieces must lie inside [grad_local, + numel).  Return 0; 100 for a bad count or dtype id, or when the partials'
 * scratch cannot be allocated; 1 for a bad source, base, accumulator or piece -- with the message set and nothing
 * launched. */
int cbnb_b200_optimizer_grad_norm_peers(int dtype, const bnb_b200_optim_tensor_t* tensors, int count, const void* const* grad_srcs, int world, const void* grad_local, long long numel, float grad_scale, bool inf_norm, double* acc, bnb_stream_t stream);
/* The global norm and clip coefficient from the world ranks' accumulated values (device memory, rank order): out[0] =
 * the fp32 total norm (L2: fp64 rank-order sum, fp64 sqrt, rounded once; inf_norm: the max); out[1] = the
 * coefficient, the bits of torch's (max_norm / (out[0] + 1e-6)).clamp(max=1.0) on an fp32 tensor (NaN kept).  One
 * tiny kernel, no host synchronisation.  Return 0, or 1 with the message set for world < 1 or a null / misaligned
 * buffer. */
int cbnb_b200_optimizer_clip_coef(const double* rank_values, int world, bool inf_norm, float max_norm, float* out, bnb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* BITSANDBYTES_B200_H */
