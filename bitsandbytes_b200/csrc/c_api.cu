// c_api.cu -- the extern "C" boundary of libbitsandbytes_b200.so.
//
// Mirrors the shape of the reference's csrc/pythonInterface.cpp (un-mangled wrappers over
// templated launchers); see include/bitsandbytes_b200.h for the per-symbol citations.
#include "common.cuh"
#include "hopper_ptx.cuh"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <type_traits>

#define BNB200_STR2(x) #x
#define BNB200_STR(x) BNB200_STR2(x)

namespace bnb200 {

// ---------------------------------------------------------------- launcher declarations
template <typename T, int QT>
void launch_quantize_blockwise(const float* code, const T* A, float* absmax, uint8_t* out, int blocksize, long long n,
                               cudaStream_t stream);
template <typename T, int QT>
void launch_dequantize_blockwise(const float* code, const uint8_t* A, const float* absmax, T* out, int blocksize,
                                 long long n, cudaStream_t stream);
// optim.cu
bool launch_optimizer32bit(int opt, int dtype, const void* g, void* p, float* s1, float* s2, float* unorm,
                           float max_unorm, float param_norm, float beta1, float beta2, float beta3, float alpha,
                           float eps, float wd, int step, float lr, float gnorm_scale, bool skip_zeros, long n,
                           cudaStream_t st);
bool launch_optimizer8bit_blockwise(int opt, int dtype, void* p, const void* g, unsigned char* s1, unsigned char* s2,
                                    float beta1, float beta2, float beta3, float alpha, float eps, int step, float lr,
                                    const float* q1, const float* q2, float* a1, float* a2, float wd,
                                    float gnorm_scale, bool skip_zeros, long n, cudaStream_t st);

template <typename T>
void launch_gemv4_simt(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                       const float* absmax_code, const float* absmax_offset, const float* lut16, int quant_type,
                       T* out, const T* bias, int M, int N, int K, int ldc, int blocksize, cudaStream_t stream);
template <typename T>
bool launch_gemv4_mma(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                      const float* absmax_code, const float* absmax_offset, T* out, const T* bias, int M, int N, int K,
                      int ldc, int blocksize, int quant_type, cudaStream_t stream);
template <typename T>
bool launch_gemm4_tc(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                     const float* absmax_code, const float* absmax_offset, T* out, const T* bias, int M, int N, int K,
                     int ldc, int blocksize, int quant_type, cudaStream_t stream, void* const* peers = nullptr,
                     int n_peers = 0, int mt_override = 0, int force_splits = 0);
void launch_int8_vector_quant(const void* A, int8_t* out, float* rowStats, int* col_flags, float threshold, int rows,
                              int cols, int dtype, cudaStream_t stream);
void launch_dequant_mm_int32_fp16(const int* A, const float* rowStats, const float* colStats, __half* out,
                                  const __half* bias, int numRows, int numCols, cudaStream_t stream);
int launch_int8_gemm(const int8_t* acts, const int8_t* weights, void* out, const float* SCA, const float* SCB,
                     const void* bias, int M, int N, int K, int ldc, int epi, cudaStream_t stream,
                     const void* subA = nullptr, const void* subBT = nullptr, int jpad = 0);
void launch_int8_outlier_prep(const void* A, const int8_t* CB, const float* SCB, const long long* cols, int J, int jpad,
                              int M, int N, int K, int dtype, void* subA, void* subBT, cudaStream_t stream);
void launch_int8_zero_columns(int8_t* CA, const long long* cols, int J, int rows, int K, cudaStream_t stream);
bool launch_int8_col_quant(const void* A, int8_t* out, float* col_stats, float threshold, int rows, int cols, int dtype,
                           cudaStream_t stream);

template <typename T, int FUNC> void launch_elementwise(T* A, const T* B, T value, long n);

// ---------------------------------------------------------------- error plumbing
namespace {
std::mutex g_err_mu;
int g_err_code = 0;
char g_err_msg[512] = {0};
thread_local int t_forced_path = -1;
} // namespace

void set_last_error(const char* where, cudaError_t err) {
    std::lock_guard<std::mutex> lk(g_err_mu);
    g_err_code = (int)err == 0 ? -1 : (int)err;
    snprintf(g_err_msg, sizeof(g_err_msg), "bitsandbytes_b200: %s failed: %s (%s)", where, cudaGetErrorName(err),
             cudaGetErrorString(err));
    fprintf(stderr, "%s\n", g_err_msg);
}

void set_last_error_msg(const char* msg) {
    std::lock_guard<std::mutex> lk(g_err_mu);
    g_err_code = -1;
    snprintf(g_err_msg, sizeof(g_err_msg), "bitsandbytes_b200: %s", msg);
    fprintf(stderr, "%s\n", g_err_msg);
}

int device_sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return kNumSMsH100;
    if (cached[dev] == 0) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = kNumSMsH100;
        cached[dev] = v;
    }
    return cached[dev];
}

// ---------------------------------------------------------------- TMA descriptor encoding
bool encode_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, int swizzle_bytes, uint64_t rows, uint64_t cols,
                    uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols) {
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                 const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                 CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess) {
            fn = reinterpret_cast<EncodeFn>(p);
        } else {
            (void)cudaGetLastError();
        }
    }
    if (fn == nullptr) {
        set_last_error_msg("cuTensorMapEncodeTiled is not available from the driver");
        return false;
    }
    if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (row_stride_bytes & 15) != 0) return false;
    const CUtensorMapDataType dt = elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT16;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {row_stride_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(out, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swizzle_bytes == 0 ? CU_TENSOR_MAP_SWIZZLE_NONE
                                       : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B),
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char msg[128];
        snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
        set_last_error_msg(msg);
        return false;
    }
    return true;
}

// ---------------------------------------------------------------- 4-bit GEMM dispatch
// path: 0 = CUDA-core GEMV, 1 = wgmma GEMM, 2 = CUDA-core generic, 3 = mma.sync decode kernel (M <= 8)
static int simt_max_m() {
    static int v = -2;
    if (v == -2) {
        const char* e = getenv("BNB_B200_SIMT_MAX_M");
        v = e ? atoi(e) : 1;  // the CUDA-core GEMV serves a single token
    }
    return v;
}

// path 3: the mma.sync decode kernel (gemv4_mma.cu), M <= 8
static int mma_max_m() {
    static int v = -2;
    if (v == -2) {
        const char* e = getenv("BNB_B200_MMA_MAX_M");
        v = e ? atoi(e) : 8;
        if (v > 16) v = 16;  // the mma.sync decode kernel serves up to two groups of 8 tokens
    }
    return v;
}

static bool tc_shape_ok(int M, int N, int K, int blocksize, int dtype) {
    (void)M;
    (void)N;
    if (dtype == 0) return false;  // fp32 activations: CUDA cores (exact fp32 products)
    if (K < 64 || (K % 64) != 0) return false;
    if (blocksize < 32 || (blocksize & (blocksize - 1)) != 0) return false;
    return true;
}

static int choose_path(int M, int N, int K, int blocksize, int dtype) {
    if (t_forced_path >= 0) {
        if ((t_forced_path == 1 || t_forced_path == 3) && !tc_shape_ok(M, N, K, blocksize, dtype)) return 2;
        return t_forced_path;
    }
    if (!tc_shape_ok(M, N, K, blocksize, dtype)) return 2;
    if (M <= simt_max_m()) return 0;
    // 5..8 tokens against a large weight: the tensor-core GEMM (decode cost independent of M) takes over from the
    // mma.sync decode kernel
    if (M <= mma_max_m() && (M <= 4 || (long long)N * K <= 2LL * 4096 * 4096)) return 3;
    return 1;
}

template <typename T>
static void gemm_4bit_dispatch(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                               const float* absmax_code, const float* absmax_offset, T* out, const T* bias, int M,
                               int N, int K, int ldc, int blocksize, int quant_type, int dtype, cudaStream_t stream) {
    if (M <= 0 || N <= 0) return;
    if (quant_type != kFP4 && quant_type != kNF4) {
        set_last_error_msg("gemm_4bit: quant_type must be 1 (FP4) or 2 (NF4)");
        return;
    }
    const int path = choose_path(M, N, K, blocksize, dtype);
    if (path == 3) {
        if constexpr (!std::is_same<T, float>::value) {
            if (launch_gemv4_mma<T>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, ldc,
                                    blocksize, quant_type, stream))
                return;
            if (launch_gemm4_tc<T>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, ldc,
                                   blocksize, quant_type, stream))
                return;
        }
    }
    if (path == 1) {
        if constexpr (!std::is_same<T, float>::value) {
            if (launch_gemm4_tc<T>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, ldc,
                                   blocksize, quant_type, stream))
                return;
        }
    }
    launch_gemv4_simt<T>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, nullptr, quant_type, out, bias, M, N,
                         K, ldc, blocksize, stream);
}

} // namespace bnb200

using namespace bnb200;

#pragma GCC visibility push(default)
extern "C" {

// =====================================================================================
// dequantize
// =====================================================================================
#define BNB200_DEQ(NAME, T, QT)                                                                                        \
    void NAME(float* code, unsigned char* A, float* absmax, T* out, int blocksize, const int n, cudaStream_t stream) { \
        launch_dequantize_blockwise<T, QT>(code, A, absmax, out, blocksize, (long long)n, stream);                     \
    }
BNB200_DEQ(cdequantize_blockwise_fp32, float, kGeneral8bit)
BNB200_DEQ(cdequantize_blockwise_fp32_fp4, float, kFP4)
BNB200_DEQ(cdequantize_blockwise_fp32_nf4, float, kNF4)
BNB200_DEQ(cdequantize_blockwise_fp16, __half, kGeneral8bit)
BNB200_DEQ(cdequantize_blockwise_fp16_fp4, __half, kFP4)
BNB200_DEQ(cdequantize_blockwise_fp16_nf4, __half, kNF4)
BNB200_DEQ(cdequantize_blockwise_bf16, __nv_bfloat16, kGeneral8bit)
BNB200_DEQ(cdequantize_blockwise_bf16_fp4, __nv_bfloat16, kFP4)
BNB200_DEQ(cdequantize_blockwise_bf16_nf4, __nv_bfloat16, kNF4)
#undef BNB200_DEQ

// =====================================================================================
// quantize (reference ABI: no stream -> legacy default stream, reference ops.cu:44-63)
// =====================================================================================
#define BNB200_Q(NAME, T, QT)                                                                                          \
    void NAME(float* code, T* A, float* absmax, unsigned char* out, int blocksize, const int n) {                      \
        launch_quantize_blockwise<T, QT>(code, A, absmax, out, blocksize, (long long)n, (cudaStream_t)0);              \
    }
BNB200_Q(cquantize_blockwise_fp32, float, kGeneral8bit)
BNB200_Q(cquantize_blockwise_fp32_fp4, float, kFP4)
BNB200_Q(cquantize_blockwise_fp32_nf4, float, kNF4)
BNB200_Q(cquantize_blockwise_fp16, __half, kGeneral8bit)
BNB200_Q(cquantize_blockwise_fp16_fp4, __half, kFP4)
BNB200_Q(cquantize_blockwise_fp16_nf4, __half, kNF4)
BNB200_Q(cquantize_blockwise_bf16, __nv_bfloat16, kGeneral8bit)
BNB200_Q(cquantize_blockwise_bf16_fp4, __nv_bfloat16, kFP4)
BNB200_Q(cquantize_blockwise_bf16_nf4, __nv_bfloat16, kNF4)
#undef BNB200_Q

void cbnb_b200_quantize_blockwise(const float* code, const void* A, float* absmax, unsigned char* out, int blocksize,
                                  int n, int quant_type, int dtype, cudaStream_t stream) {
#define BNB200_QS(T)                                                                                                   \
    switch (quant_type) {                                                                                              \
    case kGeneral8bit:                                                                                                 \
        launch_quantize_blockwise<T, kGeneral8bit>(code, (const T*)A, absmax, out, blocksize, n, stream);              \
        break;                                                                                                         \
    case kFP4: launch_quantize_blockwise<T, kFP4>(code, (const T*)A, absmax, out, blocksize, n, stream); break;        \
    case kNF4: launch_quantize_blockwise<T, kNF4>(code, (const T*)A, absmax, out, blocksize, n, stream); break;        \
    default: set_last_error_msg("quantize_blockwise: bad quant_type"); break;                                          \
    }
    if (dtype == 0) {
        BNB200_QS(float)
    } else if (dtype == 1) {
        BNB200_QS(__half)
    } else if (dtype == 2) {
        BNB200_QS(__nv_bfloat16)
    } else {
        set_last_error_msg("quantize_blockwise: bad dtype");
    }
#undef BNB200_QS
}

// =====================================================================================
// 4-bit GEMM
// =====================================================================================
void cgemm_4bit_bf16(const __nv_bfloat16* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                     const float* absmax_code, const float* absmax_offset, __nv_bfloat16* out,
                     const __nv_bfloat16* bias, int M, int N, int K, int blocksize, int quant_type,
                     cudaStream_t stream) {
    gemm_4bit_dispatch<__nv_bfloat16>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, N,
                                      blocksize, quant_type, 2, stream);
}

void cgemm_4bit_fp16(const __half* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                     const float* absmax_code, const float* absmax_offset, __half* out, const __half* bias, int M,
                     int N, int K, int blocksize, int quant_type, cudaStream_t stream) {
    gemm_4bit_dispatch<__half>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, N, blocksize,
                               quant_type, 1, stream);
}

void cgemm_4bit_fp32(const float* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                     const float* absmax_code, const float* absmax_offset, float* out, const float* bias, int M, int N,
                     int K, int blocksize, int quant_type, cudaStream_t stream) {
    gemm_4bit_dispatch<float>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, N, blocksize,
                              quant_type, 0, stream);
}

void cbnb_b200_gemm_4bit_strided(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                                 const float* absmax_code, const float* absmax_offset, void* out, const void* bias,
                                 int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype,
                                 cudaStream_t stream) {
    if (dtype == 0)
        gemm_4bit_dispatch<float>((const float*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset, (float*)out,
                                  (const float*)bias, M, N, K, ldc, blocksize, quant_type, 0, stream);
    else if (dtype == 1)
        gemm_4bit_dispatch<__half>((const __half*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset, (__half*)out,
                                   (const __half*)bias, M, N, K, ldc, blocksize, quant_type, 1, stream);
    else if (dtype == 2)
        gemm_4bit_dispatch<__nv_bfloat16>((const __nv_bfloat16*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset,
                                          (__nv_bfloat16*)out, (const __nv_bfloat16*)bias, M, N, K, ldc, blocksize,
                                          quant_type, 2, stream);
    else
        set_last_error_msg("gemm_4bit_strided: bad dtype");
}

// Fused all-gather: the tensor-core kernel's epilogue stores every output element to outs[0..n_outs)
// (outs[0] = the local buffer, the rest = the same location in the peer GPUs' buffers, mapped into
// this process -- CUDA IPC / symmetric memory).  Returns 0, or 100 when the shape does not take
// the tensor-core path (the caller then falls back to local output + a collective).
int cbnb_b200_gemm_4bit_multi_out(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                                  const float* absmax_code, const float* absmax_offset, void* const* outs, int n_outs,
                                  const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type,
                                  int dtype, cudaStream_t stream) {
    if (n_outs < 1 || n_outs > 8 || outs == nullptr) {
        set_last_error_msg("gemm_4bit_multi_out: 1 <= n_outs <= 8");
        return 1;
    }
    if (M <= 0 || N <= 0) return 0;
    if (!tc_shape_ok(M, N, K, blocksize, dtype)) return 100;
    bool ok = false;
    if (dtype == 1)
        ok = launch_gemm4_tc<__half>((const __half*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset,
                                     (__half*)outs[0], (const __half*)bias, M, N, K, ldc, blocksize, quant_type, stream,
                                     outs + 1, n_outs - 1);
    else if (dtype == 2)
        ok = launch_gemm4_tc<__nv_bfloat16>((const __nv_bfloat16*)A, B, absmax, absmax_8bit, absmax_code,
                                            absmax_offset, (__nv_bfloat16*)outs[0], (const __nv_bfloat16*)bias, M, N, K,
                                            ldc, blocksize, quant_type, stream, outs + 1, n_outs - 1);
    return ok ? 0 : 100;
}

// Developer / test entry: the tensor-core kernel of gemm4_tc.cu with an explicit token tile (mt = 16 | 32 | 64 |
// 128, 0 = automatic) and a forced K split per tile (0 = the production rule).  `trace` must be NULL.  Returns 0, or
// 100 when the shape or the options are not served by that kernel.
int cbnb_b200_gemm_4bit_pair(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                             const float* absmax_code, const float* absmax_offset, void* out, const void* bias, int M,
                             int N, int K, int ldc, int blocksize, int quant_type, int dtype, int mt, int force_splits,
                             long long* trace, cudaStream_t stream) {
    if (M <= 0 || N <= 0) return 0;
    if (trace != nullptr || force_splits < 0) return 100;
    bool ok = false;
    if (dtype == 1)
        ok = launch_gemm4_tc<__half>((const __half*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset,
                                     (__half*)out, (const __half*)bias, M, N, K, ldc, blocksize, quant_type, stream,
                                     nullptr, 0, mt, force_splits);
    else if (dtype == 2)
        ok = launch_gemm4_tc<__nv_bfloat16>((const __nv_bfloat16*)A, B, absmax, absmax_8bit, absmax_code,
                                            absmax_offset, (__nv_bfloat16*)out, (const __nv_bfloat16*)bias, M, N, K,
                                            ldc, blocksize, quant_type, stream, nullptr, 0, mt, force_splits);
    return ok ? 0 : 100;
}

int cbnb_b200_gemm_4bit_path(int M, int N, int K, int blocksize, int dtype) {
    return choose_path(M, N, K, blocksize, dtype);
}

void cbnb_b200_gemm_4bit_force_path(int path) { t_forced_path = path; }

// legacy GEMV (F.gemv_4bit): m = output features, k = inner dim, `datatype` = 16 code values
#define BNB200_NAIVE(NAME, T)                                                                                          \
    void NAME(int m, int n, int k, T* A, unsigned char* B, float* absmax, float* datatype, T* out, int lda, int ldb,   \
              int ldc, int blocksize, cudaStream_t stream) {                                                           \
        (void)n;                                                                                                       \
        (void)lda;                                                                                                     \
        (void)ldb;                                                                                                     \
        (void)ldc;                                                                                                     \
        launch_gemv4_simt<T>(A, B, absmax, nullptr, nullptr, nullptr, datatype, kNF4, out, nullptr, 1, m, k, m,        \
                             blocksize, stream);                                                                       \
    }
BNB200_NAIVE(cgemm_4bit_inference_naive_fp16, __half)
BNB200_NAIVE(cgemm_4bit_inference_naive_bf16, __nv_bfloat16)
BNB200_NAIVE(cgemm_4bit_inference_naive_fp32, float)
#undef BNB200_NAIVE

// =====================================================================================
// LLM.int8()
// =====================================================================================
void* get_context(void) {
    static int token = 0x200;
    return &token;
}

int cigemmlt_32(void* context, int m, int n, int k, const int8_t* A, const int8_t* B, void* C, float* row_scale,
                int lda, int ldb, int ldc, cudaStream_t stream) {
    (void)context;
    (void)row_scale;
    // reference column-major view: m = weight rows (N), n = tokens (M), k = K; A = weights, B = activations
    if (lda != k || ldb != k) return 100;
    return launch_int8_gemm(/*acts=*/B, /*weights=*/A, C, nullptr, nullptr, nullptr, /*M=*/n, /*N=*/m, /*K=*/k, ldc,
                            /*epi=*/0, stream);
}

int cigemmlt_8(void*, int, int, int, const int8_t*, const int8_t*, void*, float*, int, int, int, cudaStream_t) {
    return 100;  // int8 accumulation is unused by the reference's Python layer (SURVEY.md section 2.2)
}

int cigemmlt_8_rowscale(void*, int, int, int, const int8_t*, const int8_t*, void*, float*, int, int, int,
                        cudaStream_t) {
    return 100;
}

int cbnb_b200_int8_scaled_mm(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB, const void* bias,
                             void* out, int M, int N, int K, int dtype, cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) return 100;
    return launch_int8_gemm(CA, CB, out, SCA, SCB, bias, M, N, K, N, dtype, stream);
}

// LLM.int8() mixed decomposition in one GEMM launch: the int8 part as above plus, in the same epilogue, the
// outlier term subA[M, jpad] . subBT[N, jpad]^T (both of the output type, built by cbnb_b200_int8_outlier_prep).
int cbnb_b200_int8_mixed_mm(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB, const void* bias,
                            const void* subA, const void* subBT, int jpad, void* out, int M, int N, int K, int dtype,
                            cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) return 100;
    return launch_int8_gemm(CA, CB, out, SCA, SCB, bias, M, N, K, N, dtype, stream, subA, subBT, jpad);
}

void cbnb_b200_int8_outlier_prep(const void* A, const int8_t* CB, const float* SCB, const long long* cols, int J,
                                 int jpad, int M, int N, int K, int dtype, void* subA, void* subBT,
                                 cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) {
        set_last_error_msg("int8_outlier_prep: dtype must be 1 (fp16) or 2 (bf16)");
        return;
    }
    if (J < 0 || jpad < J || (jpad % 8) != 0) {
        set_last_error_msg("int8_outlier_prep: need 0 <= J <= jpad, jpad a multiple of 8");
        return;
    }
    launch_int8_outlier_prep(A, CB, SCB, cols, J, jpad, M, N, K, dtype, subA, subBT, stream);
}

void cbnb_b200_int8_zero_columns(int8_t* CA, const long long* cols, int J, int rows, int K, cudaStream_t stream) {
    launch_int8_zero_columns(CA, cols, J, rows, K, stream);
}

// Column-wise absmax + int8 codes of A[rows, cols] (the column half of the reference's int8_double_quant,
// backends/cuda/ops.py:262-296, used by MatMul8bitLt.backward).  dtype 1 = fp16, 2 = bf16.  Returns 0 / 100.
int cbnb_b200_int8_col_quant(const void* A, int8_t* out, float* col_stats, float threshold, int rows, int cols, int dtype,
                             cudaStream_t stream) {
    return launch_int8_col_quant(A, out, col_stats, threshold, rows, cols, dtype, stream) ? 0 : 100;
}

void cdequant_mm_int32_fp16(int* A, float* rowStats, float* colStats, __half* out, __half* bias, int numRows,
                            int numCols, cudaStream_t stream) {
    launch_dequant_mm_int32_fp16(A, rowStats, colStats, out, bias, numRows, numCols, stream);
}

void cint8_vector_quant(__half* A, int8_t* out, float* rowStats, float threshold, int rows, int cols,
                        cudaStream_t stream) {
    launch_int8_vector_quant(A, out, rowStats, nullptr, threshold, rows, cols, 1, stream);
}

void cbnb_b200_int8_vector_quant_flags(const void* A, int8_t* out, float* rowStats, int* col_flags, float threshold,
                                       int rows, int cols, int dtype, cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) {
        set_last_error_msg("int8_vector_quant_flags: dtype must be 1 (fp16) or 2 (bf16)");
        return;
    }
    launch_int8_vector_quant(A, out, rowStats, col_flags, threshold, rows, cols, dtype, stream);
}

// =====================================================================================
// diagnostics / loader compatibility
// =====================================================================================
int cbnb_b200_last_error(void) {
    std::lock_guard<std::mutex> lk(g_err_mu);
    int c = g_err_code;
    g_err_code = 0;
    return c;
}

const char* cbnb_b200_last_error_message(void) { return g_err_msg; }

const char* cbnb_b200_build_info(void) {
    return "bitsandbytes_b200: sm_90a; wgmma f16/bf16 (A from registers) + s8; TMA 128B-swizzle; CUDA " BNB200_STR(
        __CUDACC_VER_MAJOR__) "." BNB200_STR(__CUDACC_VER_MINOR__);
}

void* cget_managed_ptr(size_t bytes) {
    void* ptr = nullptr;
    cudaError_t e = cudaMallocManaged(&ptr, bytes, cudaMemAttachHost);
    if (e != cudaSuccess) {
        set_last_error("cget_managed_ptr", e);
        return nullptr;
    }
    return ptr;
}

// reference csrc/pythonInterface.cpp:586-592 (A[i] = value / A[i] = i / A[i] *= B[i]; legacy default stream)
void cfill_fp32(float* A, float* B, float value, long n) { launch_elementwise<float, 0>(A, B, value, n); }
void cfill_uint8(unsigned char* A, unsigned char* B, unsigned char value, long n) {
    launch_elementwise<unsigned char, 0>(A, B, value, n);
}
void carange_fp32(float* A, float* B, float value, long n) { launch_elementwise<float, 1>(A, B, value, n); }
void c_mul_fp32(float* A, float* B, float value, long n) { launch_elementwise<float, 2>(A, B, value, n); }

void cprefetch(void* ptr, size_t bytes, int device) {
    int ok = 0;
    if (cudaDeviceGetAttribute(&ok, cudaDevAttrConcurrentManagedAccess, device) != cudaSuccess || !ok) return;
    cudaError_t e = cudaMemPrefetchAsync(ptr, bytes, device, 0);
    if (e != cudaSuccess) set_last_error("cprefetch", e);
}

// ---------------------------------------------------------------------------------------------------------------
// Optimizers (SURVEY.md section 8 row f-4).  The reference-named entry points (reference
// csrc/pythonInterface.cpp:446-520: no stream argument -> legacy default stream) and the stream-taking native pair.
// optimizer ids: 0 adam (also lamb), 1 momentum (also lars), 2 rmsprop, 3 adagrad, 4 lion, 5 ademamix.
// ---------------------------------------------------------------------------------------------------------------
int cbnb_b200_optimizer_update_32bit(int optimizer, int dtype, const void* g, void* p, float* state1, float* state2,
                                     float* unorm, float max_unorm, float param_norm, float beta1, float beta2,
                                     float beta3, float alpha, float eps, float weight_decay, int step, float lr,
                                     float gnorm_scale, bool skip_zeros, long long n, cudaStream_t stream) {
    return launch_optimizer32bit(optimizer, dtype, g, p, state1, state2, unorm, max_unorm, param_norm, beta1, beta2, beta3,
                                 alpha, eps, weight_decay, step, lr, gnorm_scale, skip_zeros, (long)n, stream)
               ? 0
               : 100;
}

int cbnb_b200_optimizer_update_8bit_blockwise(int optimizer, int dtype, void* p, const void* g, unsigned char* state1,
                                              unsigned char* state2, float beta1, float beta2, float beta3, float alpha,
                                              float eps, int step, float lr, const float* quantiles1,
                                              const float* quantiles2, float* absmax1, float* absmax2,
                                              float weight_decay, float gnorm_scale, bool skip_zeros, long long n,
                                              cudaStream_t stream) {
    return launch_optimizer8bit_blockwise(optimizer, dtype, p, g, state1, state2, beta1, beta2, beta3, alpha, eps, step, lr,
                                          quantiles1, quantiles2, absmax1, absmax2, weight_decay, gnorm_scale,
                                          skip_zeros, (long)n, stream)
               ? 0
               : 100;
}

#define BNB200_C32(name, id, ctype, suffix, dt)                                                                        \
    void c##name##32bit_grad_##suffix(ctype* g, ctype* p, float* state1, float* state2, float* unorm, float max_unorm,  \
                                      float param_norm, const float beta1, const float beta2, const float beta3,        \
                                      const float alpha, const float eps, const float weight_decay, const int step,     \
                                      const float lr, const float gnorm_scale, bool skip_zeros, const int n) {          \
        launch_optimizer32bit(id, dt, g, p, state1, state2, unorm, max_unorm, param_norm, beta1, beta2, beta3, alpha,  \
                              eps, weight_decay, step, lr, gnorm_scale, skip_zeros, n, 0);                              \
    }
BNB200_C32(adam, 0, float, fp32, 0)
BNB200_C32(adam, 0, __half, fp16, 1)
BNB200_C32(adam, 0, __nv_bfloat16, bf16, 2)
BNB200_C32(momentum, 1, float, 32, 0)
BNB200_C32(momentum, 1, __half, 16, 1)
BNB200_C32(rmsprop, 2, float, 32, 0)
BNB200_C32(rmsprop, 2, __half, 16, 1)
BNB200_C32(adagrad, 3, float, 32, 0)
BNB200_C32(adagrad, 3, __half, 16, 1)
BNB200_C32(lion, 4, float, fp32, 0)
BNB200_C32(lion, 4, __half, fp16, 1)
BNB200_C32(lion, 4, __nv_bfloat16, bf16, 2)
BNB200_C32(ademamix, 5, float, fp32, 0)
BNB200_C32(ademamix, 5, __half, fp16, 1)
BNB200_C32(ademamix, 5, __nv_bfloat16, bf16, 2)
#undef BNB200_C32

#define BNB200_C8(name, id, ctype, suffix, dt)                                                                         \
    void c##name##_8bit_blockwise_grad_##suffix(ctype* p, ctype* g, unsigned char* state1, unsigned char* state2,       \
                                                float beta1, float beta2, float beta3, float alpha, float eps,          \
                                                int step, float lr, float* quantiles1, float* quantiles2,               \
                                                float* absmax1, float* absmax2, float weight_decay,                     \
                                                const float gnorm_scale, bool skip_zeros, int n) {                      \
        launch_optimizer8bit_blockwise(id, dt, p, g, state1, state2, beta1, beta2, beta3, alpha, eps, step, lr,         \
                                       quantiles1, quantiles2, absmax1, absmax2, weight_decay, gnorm_scale, skip_zeros, \
                                       n, 0);                                                                           \
    }
#define BNB200_C8_ALL(name, id)                                                                                        \
    BNB200_C8(name, id, float, fp32, 0)                                                                                \
    BNB200_C8(name, id, __half, fp16, 1)                                                                               \
    BNB200_C8(name, id, __nv_bfloat16, bf16, 2)
BNB200_C8_ALL(adam, 0)
BNB200_C8_ALL(momentum, 1)
BNB200_C8_ALL(rmsprop, 2)
BNB200_C8_ALL(adagrad, 3)
BNB200_C8_ALL(lion, 4)
BNB200_C8_ALL(ademamix, 5)
#undef BNB200_C8_ALL
#undef BNB200_C8

} // extern "C"
#pragma GCC visibility pop
