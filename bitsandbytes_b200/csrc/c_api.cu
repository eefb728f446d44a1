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
int optimizer_list_capacity();
bool launch_optimizer32bit_list(int opt, int dtype, const OptimTensor* ts, int count, float beta1, float beta2,
                                float beta3, float alpha, float eps, float wd, float lr, float gnorm_scale,
                                bool skip_zeros, cudaStream_t st);
bool launch_optimizer8bit_blockwise_list(int opt, int dtype, const OptimTensor* ts, int count, float beta1, float beta2,
                                         float beta3, float alpha, float eps, float wd, float lr, const float* q1,
                                         const float* q2, float gnorm_scale, bool skip_zeros, cudaStream_t st);
bool launch_optimizer32bit_list_dev(int opt, int dtype, const OptimTensor* ts, int count, float beta1, float beta2,
                                    float beta3, float alpha, float eps, float wd, float lr, const float* lr_dev,
                                    float gnorm_scale, bool skip_zeros, cudaStream_t st);
bool launch_optimizer8bit_blockwise_list_dev(int opt, int dtype, const OptimTensor* ts, int count, float beta1,
                                             float beta2, float beta3, float alpha, float eps, float wd, float lr,
                                             const float* lr_dev, const float* q1, const float* q2, float gnorm_scale,
                                             bool skip_zeros, cudaStream_t st);
int optimizer_peers_capacity();
int optimizer_max_peers();
bool launch_optimizer32bit_list_peers(int opt, int dtype, const OptimTensor* ts, int count,
                                      const void* const* grad_srcs, int world, void* const* param_dsts, int ndst,
                                      const void* grad_local, const void* param_local, float grad_scale, float beta1,
                                      float beta2, float beta3, float alpha, float eps, float wd, float lr,
                                      bool skip_zeros, const float* gnorm_scale_dev, bool dev, const float* lr_dev,
                                      cudaStream_t st);
bool launch_optimizer8bit_blockwise_list_peers(int opt, int dtype, const OptimTensor* ts, int count,
                                               const void* const* grad_srcs, int world, void* const* param_dsts,
                                               int ndst, const void* grad_local, const void* param_local,
                                               float grad_scale, float beta1, float beta2, float beta3, float alpha,
                                               float eps, float wd, float lr, const float* q1, const float* q2,
                                               bool skip_zeros, const float* gnorm_scale_dev, bool dev,
                                               const float* lr_dev, cudaStream_t st);
bool launch_optimizer_grad_norm_peers(int dtype, const OptimTensor* ts, int count, const void* const* grad_srcs,
                                      int world, const void* grad_local, float grad_scale, bool inf, double* acc,
                                      cudaStream_t st);
void launch_optimizer_clip_coef(const double* values, int world, bool inf, float max_norm, float* out,
                                cudaStream_t st);

// PART = true: the partial instances (fp32 accumulators to every destination of an OutList<float>, no bias, no
// rounding)
template <typename T, bool PART = false>
void launch_gemv4_simt(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                       const float* absmax_code, const float* absmax_offset, const float* lut16, int quant_type,
                       typename OutArg<T, PART>::type out, const T* bias, int M, int N, int K, int ldc, int blocksize,
                       cudaStream_t stream);
template <typename T, bool PART = false>
bool launch_gemv4_mma(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                      const float* absmax_code, const float* absmax_offset, typename OutArg<T, PART>::type out,
                      const T* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, cudaStream_t stream);
template <typename T, bool PART = false>
bool launch_gemm4_tc(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                     const float* absmax_code, const float* absmax_offset, const OutList<OutElem<T, PART>>& outs,
                     const T* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, cudaStream_t stream,
                     int mt_override = 0, int force_splits = 0);
template <typename T, bool PART = false>
bool launch_gemm4_staged(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                         const float* absmax_code, const float* absmax_offset, const OutList<OutElem<T, PART>>& outs,
                         const T* bias, int M, int N, int K, int ldc, int blocksize, int quant_type,
                         cudaStream_t stream, int mt_override = 0, int panel_rows = 0);
template <typename T>
bool launch_gemm4_grouped(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                          const float* absmax_code, const float* absmax_offset, const int* offs, int E, T* out,
                          const T* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int mt,
                          cudaStream_t stream);
template <typename T>
bool launch_gemm4_grouped_partial(const T* A, const uint8_t* B, const float* absmax, const int* offs, int E, float* out,
                                  int M, int N, int K, int ldc, int blocksize, int quant_type, int mt,
                                  cudaStream_t stream);
// partials.cu
bool launch_reduce_partials(const float* parts, int world, long long part_stride, void* out, const void* bias, int M,
                            int N, int ldc, int dtype, cudaStream_t stream);
bool launch_reduce_partials_grouped(const float* parts, int world, long long part_stride, const int* offs, int E,
                                    void* out, const void* bias, int M, int N, int ldc, int dtype, cudaStream_t stream);
int max_reduce_parts();
bool launch_reduce_partials_ptrs(const float* const* parts, int n_parts, int row0, int rows, void* out,
                                 const void* bias, int N, int ldc, int dtype, cudaStream_t stream);
template <typename T>
bool launch_gemm_decoded(const T* A, const T* W, T* out, const T* bias, int M, int N, int K, int ldc, int mt,
                         cudaStream_t stream);
template <typename T>
void launch_dequantize4_panel(const uint8_t* codes, const float* absmax, const uint8_t* absmax_8bit,
                              const float* absmax_code, const float* absmax_offset, T* out, int blocksize,
                              int quant_type, int n0, int rows, int K, cudaStream_t stream);
int staged_plan(int M, int N, int K, int sms, int* panel_rows);
void launch_int8_vector_quant(const void* A, int8_t* out, float* rowStats, int* col_flags, float threshold, int rows,
                              int cols, int dtype, cudaStream_t stream);
void launch_dequant_mm_int32_fp16(const int* A, const float* rowStats, const float* colStats, __half* out,
                                  const __half* bias, int numRows, int numCols, cudaStream_t stream);
int launch_int8_gemm(const int8_t* acts, const int8_t* weights, void* out, const float* SCA, const float* SCB,
                     const void* bias, int M, int N, int K, int ldc, int epi, cudaStream_t stream,
                     const void* subA = nullptr, const void* subBT = nullptr, int jpad = 0,
                     const int* jcount = nullptr, const int* cols = nullptr, const void* A = nullptr,
                     void* const* outs = nullptr, int n_outs = 0, int rows_per_out = 0);
void launch_int8_row_stats(const void* A, float* rowStats, int* col_flags, float threshold, int rows, int cols,
                           int dtype, cudaStream_t stream);
void launch_int8_quant_with_stats(const void* A, int8_t* out, const float* rowStats, float threshold, int rows,
                                  int cols, int dtype, cudaStream_t stream);
bool launch_reduce_int8_partials(const int* parts, int world, long long part_stride, const float* SCA, const float* SCB,
                                 const void* bias, const void* subA, const void* subBT, int jpad, void* out, int M,
                                 int N, int ldc, int dtype, cudaStream_t stream);
void launch_int8_outlier_prep(const void* A, const int8_t* CB, const float* SCB, const long long* cols, int J, int jpad,
                              int M, int N, int K, int dtype, void* subA, void* subBT, cudaStream_t stream);
void launch_int8_outlier_prep_dev(const void* A, int8_t* CA, const int8_t* CB, const float* SCB, const int* cols,
                                  const int* count, int cap, int M, int N, int K, int dtype, void* subA, void* subBT,
                                  cudaStream_t stream);
void launch_int8_outlier_compact(const int* col_flags, int K, int* cols, int* count, cudaStream_t stream);
void launch_int8_grouped_outliers(const void* A, const void* A16, int8_t* CA, const int8_t* CB, const float* SCB,
                                  const int* offs, int E, float threshold, int* ends, int* flags, int* cols, int* count,
                                  void* subA, void* subBT, int M, int N, int K, int dtype, cudaStream_t stream);
int launch_int8_gemm_grouped(const int8_t* CA, const int8_t* CB, void* out, const float* SCA, const float* SCB,
                             const void* bias, const int* offs, int E, int M, int N, int K, int epi, const void* A,
                             const void* subA, const void* subBT, const int* cols, const int* count,
                             cudaStream_t stream);
void launch_int8_zero_columns(int8_t* CA, const long long* cols, int J, int rows, int K, cudaStream_t stream);
bool launch_int8_col_quant(const void* A, int8_t* out, float* col_stats, float threshold, int rows, int cols, int dtype,
                           cudaStream_t stream);
bool launch_int8_dequant_rows(const int8_t* CB, const float* SCB, void* out, int ldo, int rows, int cols, int dtype,
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
    const CUtensorMapDataType dt = elem_bytes == 1   ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                   : elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                                     : CU_TENSOR_MAP_DATA_TYPE_UINT16;
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {row_stride_bytes};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapSwizzle swz = swizzle_bytes == 0    ? CU_TENSOR_MAP_SWIZZLE_NONE
                                   : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                   : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                         : CU_TENSOR_MAP_SWIZZLE_128B;
    CUresult r = fn(out, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
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
// Path 1 has two forms: the fused kernel, and at large M the staged route (staged_route() below).
// dtype: 0 = fp32, 1 = fp16, 2 = bf16, 3 = fp32 with TF32 allowed (the caller's fp32 matmul precision is "tf32")
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

// dtype 3: fp32 activations take the TF32 instance of the wgmma GEMM from this many tokens on: the measured crossover
// against the CUDA-core kernel on an H100 (DESIGN.md section 7)
constexpr int kTf32MinM = 4;

// the staged route from this many tokens on (fp16 / bf16): the fused kernel decodes every weight once per 256-token tile, the
// staged route once per call.  The measured crossover on an H100 (tools/time_gemm4_staged.py, DESIGN.md section 7):
// at 1024 tokens the route still loses on the 11008 x 4096 weight, from 2048 on it wins where its panels take no
// more waves of 256-token tiles than the fused kernel's grid.
constexpr int kStagedMinM = 2048;

static bool tc_shape_ok(int M, int N, int K, int blocksize, int dtype) {
    (void)M;
    (void)N;
    if (dtype == 0) return false;  // fp32 activations: CUDA cores (exact fp32 products)
    if (K < 64 || (K % 64) != 0) return false;
    if (blocksize < 32 || (blocksize & (blocksize - 1)) != 0) return false;
    return true;
}

static int choose_path(int M, int N, int K, int blocksize, int dtype) {
    if (dtype == 3) {
        // TF32 where the wgmma GEMM serves the shape and, unforced, from kTf32MinM tokens; otherwise the fp32 route
        const bool tc = tc_shape_ok(M, N, K, blocksize, dtype) && (t_forced_path >= 0 ? t_forced_path == 1 : M >= kTf32MinM);
        return tc ? 1 : choose_path(M, N, K, blocksize, 0);
    }
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

// Whether an unforced path-1 call with 16-bit activations takes the staged route (decode every weight panel once,
// then the wgmma GEMM on shared-memory operands) instead of the fused kernel: from kStagedMinM tokens, where the
// 256-token tiles fill every SM (the route never splits K) and its panels (each a launch of its own) take no more
// waves than the fused kernel's persistent grid.  A forced path 1 keeps the fused kernel.
static bool staged_route(int M, int N, int K, int blocksize, int dtype) {
    if (t_forced_path >= 0 || (dtype != 1 && dtype != 2) || M < kStagedMinM) return false;
    if (choose_path(M, N, K, blocksize, dtype) != 1) return false;
    const int sms = device_sm_count();
    const long long tiles = (long long)((M + 255) / 256) * ((N + 127) / 128);
    int panel = 0;
    const int staged_waves = staged_plan(M, N, K, sms, &panel);
    return staged_waves > 0 && tiles >= sms && staged_waves <= (tiles + sms - 1) / sms;
}

template <typename TO> static OutList<TO> as_list(TO* out) { return OutList<TO>{{out}, 1}; }
template <typename TO> static const OutList<TO>& as_list(const OutList<TO>& outs) { return outs; }

// outs[0..n) of a C entry, which has checked 1 <= n <= kMaxOuts
template <typename TO, typename P> static OutList<TO> out_list(P const* outs, int n) {
    OutList<TO> l{};
    for (int i = 0; i < n; ++i) l.p[i] = (TO*)outs[i];
    l.n = n;
    return l;
}

// The 4-bit GEMM of the plain, multi-destination and partial entries.  out: T* (one destination of T), OutList<T> (a
// list of destinations of T) or, for the partial instances (PART), OutList<float>.  Returns false, with nothing
// computed, for a bad quant_type (the error message set) or for a list of T that no kernel serves.
template <typename T, bool PART = false, typename Out = typename OutArg<T, PART>::type>
static bool gemm_4bit_dispatch(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                               const float* absmax_code, const float* absmax_offset, Out out, const T* bias, int M,
                               int N, int K, int ldc, int blocksize, int quant_type, int dtype, cudaStream_t stream) {
    if (M <= 0 || N <= 0) return true;
    if (quant_type != kFP4 && quant_type != kNF4) {
        set_last_error_msg("gemm_4bit: quant_type must be 1 (FP4) or 2 (NF4)");
        return false;
    }
    // The GEMV, the mma.sync decode kernel and the CUDA-core kernel store to one destination of T.  A list of T, even
    // of one destination, therefore takes path 1 (staged or fused, by staged_route) wherever the wgmma GEMM serves the
    // shape, and is refused elsewhere.  At M <= 8 the plain call takes path 0 or 3 instead, so there a list's
    // destinations do not hold the plain call's bits.
    constexpr bool kList = !PART && std::is_same<Out, OutList<T>>::value;
    int path = 1;
    if constexpr (kList) {
        if (!tc_shape_ok(M, N, K, blocksize, dtype)) return false;
    } else {
        path = choose_path(M, N, K, blocksize, dtype);
    }
    const OutList<OutElem<T, PART>>& outs = as_list(out);
    if (path == 1 && staged_route(M, N, K, blocksize, dtype)) {
        if constexpr (!std::is_same<T, float>::value) {
            if (launch_gemm4_staged<T, PART>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, outs, bias, M, N,
                                             K, ldc, blocksize, quant_type, stream))
                return true;
        }
    }
    if constexpr (!kList && !std::is_same<T, float>::value) {
        if (path == 3) {
            if (launch_gemv4_mma<T, PART>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K,
                                          ldc, blocksize, quant_type, stream))
                return true;
            if (launch_gemm4_tc<T, PART>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, outs, bias, M, N, K,
                                         ldc, blocksize, quant_type, stream))
                return true;
        }
    }
    // (fp32 takes path 1 only as dtype 3: the TF32 instance)
    if (path == 1 && launch_gemm4_tc<T, PART>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, outs, bias, M, N,
                                              K, ldc, blocksize, quant_type, stream))
        return true;
    if constexpr (kList) {
        return false;
    } else {
        launch_gemv4_simt<T, PART>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, nullptr, quant_type, out,
                                   bias, M, N, K, ldc, blocksize, stream);
        return true;
    }
}

// The element type of the ABI's dtype id (0 and 3 fp32, 1 fp16, 2 bf16): calls f(T()) and returns true for an id in
// the entry's kIds (bits 1 << id), false for any other.
constexpr unsigned kIdF16 = 1u << 1, kIdBF16 = 1u << 2, kIdTF32 = 1u << 3, kIdAny = 0xfu;
template <unsigned kIds, typename F> static bool with_dtype(int dtype, F&& f) {
    if (dtype < 0 || dtype > 3 || (kIds & (1u << dtype)) == 0) return false;
    if (dtype == 1) {
        f(__half());
    } else if (dtype == 2) {
        f(__nv_bfloat16());
    } else if constexpr ((kIds & (1u | kIdTF32)) != 0) {
        f(float());
    }
    return true;
}

// The grouped GEMM's token tile: the smallest of 16, 32, 64 and 128 tokens that holds twice the mean rows per expert,
// 2 ceil(M / E), since under top-k routing many experts get more rows than the mean.  Measured on an H100
// (tools/time_grouped_gemm4.py, DESIGN.md section 7): at a mean of 16 rows the 32-token tile is the fastest (Qwen3-30B-A3B,
// 256 tokens: 242 us against 334 us at 16 for gate_up), at a mean of 64 the 128-token tile (Mixtral-8x7B, 256 tokens:
// 664 us against 766 us at 64 for gate_up), and at a mean of 4 the 16-token tile.  The exception measured: at one token
// the down projections run 7-11 % faster at 64 tokens than at the rule's 16.
static int grouped_tile(int M, int E) {
    const long long want = 2LL * ((M + E - 1) / E);
    return want <= 16 ? 16 : want <= 32 ? 32 : want <= 64 ? 64 : 128;
}

// The grouped GEMM of the entries below: 0; 1 with the error message set for bad arguments; 100 when not served,
// with nothing written and no message; or 100 with the error message set when a launch past those checks fails.
static int gemm_4bit_grouped(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                             const float* absmax_code, const float* absmax_offset, const int* offs, int E, void* out,
                             const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype,
                             int mt, cudaStream_t stream) {
    if (A == nullptr || B == nullptr || absmax == nullptr || offs == nullptr || out == nullptr || M < 0 || N <= 0 ||
        K <= 0 || E < 1 || ldc < N || (quant_type != kFP4 && quant_type != kNF4) ||
        (absmax_8bit != nullptr && absmax_code == nullptr)) {
        set_last_error_msg("gemm_4bit_grouped: needs A, B, absmax, offs and out, M >= 0, N, K >= 1, E >= 1, ldc >= N, "
                           "quant_type 1 (FP4) or 2 (NF4), and absmax_code with absmax_8bit");
        return 1;
    }
    if (M == 0) return 0;
    if (mt == 0) mt = grouped_tile(M, E);
    bool ok = false;
    const bool known = with_dtype<kIdF16 | kIdBF16>(dtype, [&](auto t) {
        using T = decltype(t);
        if constexpr (!std::is_same<T, float>::value) {
            ok = launch_gemm4_grouped<T>((const T*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset, offs, E,
                                         (T*)out, (const T*)bias, M, N, K, ldc, blocksize, quant_type, mt, stream);
        }
    });
    return known && ok ? 0 : 100;
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
    const bool known = with_dtype<kIdAny>(dtype, [&](auto t) {
        using T = decltype(t);
        gemm_4bit_dispatch<T>((const T*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset, (T*)out, (const T*)bias,
                              M, N, K, ldc, blocksize, quant_type, dtype, stream);
    });
    if (!known) set_last_error_msg("gemm_4bit_strided: bad dtype");
}

// Fused all-gather: the tensor-core kernel's epilogue stores every output element to outs[0..n_outs)
// (outs[0] = the local buffer, the rest = the same location in the peer GPUs' buffers, mapped into
// this process -- CUDA IPC / symmetric memory).  Returns 0, or 100 when the shape does not take
// the tensor-core path (the caller then falls back to local output + a collective).
int cbnb_b200_gemm_4bit_multi_out(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                                  const float* absmax_code, const float* absmax_offset, void* const* outs, int n_outs,
                                  const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type,
                                  int dtype, cudaStream_t stream) {
    if (n_outs < 1 || n_outs > kMaxOuts || outs == nullptr) {
        set_last_error_msg("gemm_4bit_multi_out: 1 <= n_outs <= 8");
        return 1;
    }
    if (M <= 0 || N <= 0) return 0;
    bool ok = false;
    with_dtype<kIdF16 | kIdBF16>(dtype, [&](auto t) {
        using T = decltype(t);
        ok = gemm_4bit_dispatch<T, false, OutList<T>>((const T*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset,
                                                      out_list<T>(outs, n_outs), (const T*)bias, M, N, K, ldc,
                                                      blocksize, quant_type, dtype, stream);
    });
    return ok ? 0 : 100;
}

// Partial GEMM of a row-sharded layer: outs[0..n_outs)[m, n] (row stride ldc, fp32) = the fp32 sum over k of
// A[m, k] * W[n, k], with no bias and no rounding, computed by the kernel (and the K split) that the plain call of the
// same shape takes.  outs is a host array of device addresses (local buffers, or peers' mapped buffers).  Returns 0,
// 1 for a bad destination list, or 100 for a dtype the entry does not serve.
int cbnb_b200_gemm_4bit_partial(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                                const float* absmax_code, const float* absmax_offset, float* const* outs, int n_outs,
                                int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype,
                                cudaStream_t stream) {
    if (n_outs < 1 || n_outs > kMaxOuts || outs == nullptr) {
        set_last_error_msg("gemm_4bit_partial: 1 <= n_outs <= 8");
        return 1;
    }
    const bool known = with_dtype<kIdAny>(dtype, [&](auto t) {
        using T = decltype(t);
        gemm_4bit_dispatch<T, true>((const T*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset,
                                    out_list<float>(outs, n_outs), nullptr, M, N, K, ldc, blocksize, quant_type, dtype,
                                    stream);
    });
    return known ? 0 : 100;
}

// The partial GEMM of a sequence-parallel row-sharded layer: cbnb_b200_gemm_4bit_partial with the rows scattered
// instead of copied.  Row m is stored to outs[m / rows_per_out] at row m % rows_per_out (row stride ldc, fp32), so
// outs is in rank order: outs[s] receives the tokens of rank s.  Same kernel and K split as the partial entry.
// Returns 0, 1 unless 1 <= n_outs <= 8, rows_per_out >= 1 and n_outs * rows_per_out == M, or 100 for a bad dtype.
int cbnb_b200_gemm_4bit_partial_scatter(const void* A, const uint8_t* B, const float* absmax,
                                        const uint8_t* absmax_8bit, const float* absmax_code,
                                        const float* absmax_offset, float* const* outs, int n_outs, int rows_per_out,
                                        int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype,
                                        cudaStream_t stream) {
    if (n_outs < 1 || n_outs > kMaxOuts || outs == nullptr || rows_per_out < 1 ||
        (long long)n_outs * rows_per_out != M) {
        set_last_error_msg("gemm_4bit_partial_scatter: needs 1 <= n_outs <= 8, rows_per_out >= 1 and "
                           "n_outs * rows_per_out == M");
        return 1;
    }
    OutList<float> list = out_list<float>(outs, n_outs);
    list.rows_per_out = rows_per_out;
    const bool known = with_dtype<kIdAny>(dtype, [&](auto t) {
        using T = decltype(t);
        gemm_4bit_dispatch<T, true>((const T*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset, list, nullptr, M,
                                    N, K, ldc, blocksize, quant_type, dtype, stream);
    });
    return known ? 0 : 100;
}

// out[m, n] (row stride ldc) = T(((parts[0] + parts[1]) + ... + parts[world - 1])[m, n] + bias[n]): the partials
// [M, N] (row stride N, one every part_stride elements) summed in rank order in fp32, the bias added in fp32, one
// rounding.  dtype 0 or 3 = fp32, 1 = fp16, 2 = bf16.  Returns 0, or 100 for a dtype or world it does not serve.
int cbnb_b200_reduce_partials(const float* parts, int world, long long part_stride, void* out, const void* bias, int M,
                              int N, int ldc, int dtype, cudaStream_t stream) {
    return launch_reduce_partials(parts, world, part_stride, out, bias, M, N, ldc, dtype, stream) ? 0 : 100;
}

// cbnb_b200_reduce_partials over partials in separate buffers: out[m, n] (row stride ldc, m < rows) =
// T(((parts[0] + parts[1]) + ... + parts[n_parts - 1])[row0 + m, n] + bias[n]), each parts[r] an [M, N] fp32 partial at
// row stride N -- a rank's own buffer or a peer's symmetric-memory mapping -- listed in rank order.  The same
// element-wise arithmetic as cbnb_b200_reduce_partials, so the same bits.  dtype 0 or 3 = fp32, 1 = fp16, 2 = bf16.
// Returns 0; 1 with the error message set unless 1 <= n_parts <= 8, every partial is non-null and 4-byte aligned, out
// (and bias, when given) are aligned to their element, 0 <= row0, 0 <= rows, row0 + rows <= M and ldc >= N; or 100
// for a dtype it does not serve.
int cbnb_b200_reduce_partials_ptrs(const float* const* parts, int n_parts, int row0, int rows, void* out,
                                   const void* bias, int M, int N, int ldc, int dtype, cudaStream_t stream) {
    if (dtype < 0 || dtype > 3) return 100;
    const uintptr_t esz = dtype == 1 || dtype == 2 ? 2 : 4;
    bool ok = parts != nullptr && n_parts >= 1 && n_parts <= max_reduce_parts() && row0 >= 0 && rows >= 0 && M >= 0 &&
              N >= 0 && (long long)row0 + rows <= M && ldc >= N && out != nullptr &&
              (reinterpret_cast<uintptr_t>(out) & (esz - 1)) == 0 &&
              (reinterpret_cast<uintptr_t>(bias) & (esz - 1)) == 0;
    for (int r = 0; ok && r < n_parts; ++r)
        ok = parts[r] != nullptr && (reinterpret_cast<uintptr_t>(parts[r]) & 3) == 0;
    if (!ok) {
        set_last_error_msg("reduce_partials_ptrs: needs 1 <= n_parts <= 8 non-null, 4-byte aligned partials, out and "
                           "bias aligned to their element, 0 <= row0, 0 <= rows, row0 + rows <= M and ldc >= N");
        return 1;
    }
    return launch_reduce_partials_ptrs(parts, n_parts, row0, rows, out, bias, N, ldc, dtype, stream) ? 0 : 100;
}

// Developer / test entry: the tensor-core kernel of gemm4_tc.cu with an explicit token tile (mt = 16 | 32 | 64 |
// 128 | 256, 0 = automatic; 128 at most for dtype 3, the TF32 instance) and a forced K split per tile (0 = the
// production rule).  `trace` must be NULL.  Returns 0, or 100 when the shape or the options are not served by that
// kernel.
int cbnb_b200_gemm_4bit_pair(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                             const float* absmax_code, const float* absmax_offset, void* out, const void* bias, int M,
                             int N, int K, int ldc, int blocksize, int quant_type, int dtype, int mt, int force_splits,
                             long long* trace, cudaStream_t stream) {
    if (M <= 0 || N <= 0) return 0;
    if (trace != nullptr || force_splits < 0) return 100;
    bool ok = false;
    with_dtype<kIdF16 | kIdBF16 | kIdTF32>(dtype, [&](auto t) {
        using T = decltype(t);
        ok = launch_gemm4_tc<T>((const T*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset, as_list((T*)out),
                                (const T*)bias, M, N, K, ldc, blocksize, quant_type, stream, mt, force_splits);
    });
    return ok ? 0 : 100;
}

// Developer / test entry: the staged route with a chosen token tile (mt = 128 | 256, 0 = by the shape) and
// panel (panel_rows: a multiple of 128 whose decoded rows fit the 32 MB workspace, 0 = the largest that does), every
// element stored to outs[0..n_outs) as in cbnb_b200_gemm_4bit_multi_out.  dtype 1 or 2.  Returns 0, or 100 when the
// route does not serve the shape or the options.
int cbnb_b200_gemm_4bit_staged(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                               const float* absmax_code, const float* absmax_offset, void* const* outs, int n_outs,
                               const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int dtype,
                               int mt, int panel_rows, cudaStream_t stream) {
    if (n_outs < 1 || n_outs > kMaxOuts || outs == nullptr) return 100;
    if (M <= 0 || N <= 0) return 0;
    bool ok = false;
    with_dtype<kIdF16 | kIdBF16>(dtype, [&](auto t) {
        using T = decltype(t);
        ok = launch_gemm4_staged<T>((const T*)A, B, absmax, absmax_8bit, absmax_code, absmax_offset,
                                    out_list<T>(outs, n_outs), (const T*)bias, M, N, K, ldc, blocksize, quant_type,
                                    stream, mt, panel_rows);
    });
    return ok ? 0 : 100;
}

// The staged route's two phases on their own, for tests and timing: rows [n0, n0 + rows) of a [N, K] 4-bit weight
// decoded into out[rows, K] (returns 100 unless K % 64 == 0, n0 % 128 == 0, blocksize a power of two >= 32 and the
// codes 16-byte aligned), and the staged GEMM on such a decoded weight W[N, K] (mt = 128 | 256).
int cbnb_b200_dequantize_4bit_panel(const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                                    const float* absmax_code, const float* absmax_offset, void* out, int blocksize,
                                    int quant_type, int dtype, int n0, int rows, int K, cudaStream_t stream) {
    if (rows <= 0) return 0;
    if (K < 64 || (K % 64) != 0 || n0 < 0 || (n0 % 128) != 0 || blocksize < 32 || (blocksize & (blocksize - 1)) != 0 ||
        (quant_type != kNF4 && quant_type != kFP4) || (reinterpret_cast<uintptr_t>(B) & 15) != 0)
        return 100;
    const bool known = with_dtype<kIdF16 | kIdBF16>(dtype, [&](auto t) {
        using T = decltype(t);
        launch_dequantize4_panel<T>(B, absmax, absmax_8bit, absmax_code, absmax_offset, (T*)out, blocksize, quant_type,
                                    n0, rows, K, stream);
    });
    return known ? 0 : 100;
}

int cbnb_b200_gemm_decoded(const void* A, const void* W, void* out, const void* bias, int M, int N, int K, int ldc,
                           int dtype, int mt, cudaStream_t stream) {
    bool ok = false;
    with_dtype<kIdF16 | kIdBF16>(dtype, [&](auto t) {
        using T = decltype(t);
        ok = launch_gemm_decoded<T>((const T*)A, (const T*)W, (T*)out, (const T*)bias, M, N, K, ldc, mt, stream);
    });
    return ok ? 0 : 100;
}

// The grouped 4-bit GEMM of a mixture-of-experts layer (no reference counterpart): out[m, :] (row stride ldc) =
// T(A[m, :] . W_e^T + bias[e * N ..]) for the rows of expert e, end_{e-1} <= m < end_e, and 0 for the rows past
// end_{E-1}.  B is E experts' [N, K] weights quantised as one [E * N, K] tensor; offs[E] (int32, on the device) holds the
// end rows, clamped on the device as end_e = min(max(offs[e], end_{e-1}), M).  Returns 0, 1 with the error message set
// for bad arguments, or 100, with nothing written, for what the kernel does not serve.  A failure past those checks (a
// tensor map, the shared-memory opt-in or the launch) also returns 100, with the error message set.
int cbnb_b200_gemm_4bit_grouped(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                                const float* absmax_code, const float* absmax_offset, const int* offs, int E, void* out,
                                const void* bias, int M, int N, int K, int ldc, int blocksize, int quant_type,
                                int dtype, cudaStream_t stream) {
    return gemm_4bit_grouped(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, offs, E, out, bias, M, N, K, ldc,
                             blocksize, quant_type, dtype, 0, stream);
}

// Developer / test entry: cbnb_b200_gemm_4bit_grouped at token tile mt (16 | 32 | 64 | 128; 0 = the production rule).
int cbnb_b200_gemm_4bit_grouped_mt(const void* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                                   const float* absmax_code, const float* absmax_offset, const int* offs, int E,
                                   void* out, const void* bias, int M, int N, int K, int ldc, int blocksize,
                                   int quant_type, int dtype, int mt, cudaStream_t stream) {
    return gemm_4bit_grouped(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, offs, E, out, bias, M, N, K, ldc,
                             blocksize, quant_type, dtype, mt, stream);
}

// The grouped fp32 partial of a row-sharded expert layer: out[m, n] (fp32, row stride ldc) = A[m, :] . W_e[n, :] for
// the rows of expert e, with no bias and no rounding, and 0 for the rows past end_{E-1}; offs and B as in
// cbnb_b200_gemm_4bit_grouped, with plain fp32 absmax.  mt: the token tile (16 | 32 | 64 | 128), 0 = the grouped GEMM's
// rule for (M, E), so that a shard runs the unsharded layer's tile.  Returns 0; 1 with the error message set for bad
// arguments; 100, with nothing written, for what the kernel does not serve (nested statistics, K % 64 != 0, E > 1024);
// or 100 with the error message set when a launch past those checks fails.
int cbnb_b200_gemm_4bit_grouped_partial(const void* A, const uint8_t* B, const float* absmax, const int* offs, int E,
                                        float* out, int M, int N, int K, int ldc, int blocksize, int quant_type,
                                        int dtype, int mt, cudaStream_t stream) {
    if (A == nullptr || B == nullptr || absmax == nullptr || offs == nullptr || out == nullptr || M < 0 || N <= 0 ||
        K <= 0 || E < 1 || ldc < N || (quant_type != kFP4 && quant_type != kNF4) ||
        (mt != 0 && mt != 16 && mt != 32 && mt != 64 && mt != 128)) {
        set_last_error_msg("gemm_4bit_grouped_partial: needs A, B, absmax, offs and out, M >= 0, N, K >= 1, E >= 1, "
                           "ldc >= N, quant_type 1 (FP4) or 2 (NF4) and mt 0, 16, 32, 64 or 128");
        return 1;
    }
    if (M == 0) return 0;
    if (mt == 0) mt = grouped_tile(M, E);
    bool ok = false;
    const bool known = with_dtype<kIdF16 | kIdBF16>(dtype, [&](auto t) {
        using T = decltype(t);
        if constexpr (!std::is_same<T, float>::value) {
            ok = launch_gemm4_grouped_partial<T>((const T*)A, B, absmax, offs, E, out, M, N, K, ldc, blocksize,
                                                 quant_type, mt, stream);
        }
    });
    return known && ok ? 0 : 100;
}

// The reduction of a row-sharded expert layer: out[m, n] (row stride ldc) = T(((parts[0] + parts[1]) + ... +
// parts[world - 1])[m, n] + bias[e * N + n]) for the rows of expert e (end rows clamped on the device from offs[E], as
// the grouped GEMM clamps them), and 0 for the rows past end_{E-1}.  The partials are [M, N] at row stride N, one every
// part_stride elements; bias is [E, N] or NULL.  The arithmetic of cbnb_b200_reduce_partials: without a bias and
// without tail rows, the same bits.  dtype 1 = fp16, 2 = bf16.  Returns 0, or 100 for a dtype, world or E it does not
// serve.
int cbnb_b200_reduce_partials_grouped(const float* parts, int world, long long part_stride, const int* offs, int E,
                                      void* out, const void* bias, int M, int N, int ldc, int dtype,
                                      cudaStream_t stream) {
    return launch_reduce_partials_grouped(parts, world, part_stride, offs, E, out, bias, M, N, ldc, dtype, stream) ? 0
                                                                                                                   : 100;
}

int cbnb_b200_gemm_4bit_path(int M, int N, int K, int blocksize, int dtype) {
    return choose_path(M, N, K, blocksize, dtype);
}

int cbnb_b200_gemm_4bit_staged_route(int M, int N, int K, int blocksize, int dtype) {
    return staged_route(M, N, K, blocksize, dtype) ? 1 : 0;
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

// The same decomposition with the outlier columns and their count kept on the device, so that no launch depends on
// them and the three launches can be captured in a CUDA graph: compact the flags, build the operands (64 columns,
// zero-padded) and zero CA's outlier columns, then the GEMM, which reads the count and gathers any columns past 64.
void cbnb_b200_int8_outlier_compact(const int* col_flags, int K, int* cols, int* count, cudaStream_t stream) {
    launch_int8_outlier_compact(col_flags, K, cols, count, stream);
}

void cbnb_b200_int8_outlier_prep_dev(const void* A, int8_t* CA, const int8_t* CB, const float* SCB, const int* cols,
                                     const int* count, int M, int N, int K, int dtype, void* subA, void* subBT,
                                     cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) {
        set_last_error_msg("int8_outlier_prep_dev: dtype must be 1 (fp16) or 2 (bf16)");
        return;
    }
    launch_int8_outlier_prep_dev(A, CA, CB, SCB, cols, count, 64, M, N, K, dtype, subA, subBT, stream);
}

int cbnb_b200_int8_mixed_mm_dev(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB, const void* bias,
                                const void* A, const void* subA, const void* subBT, const int* cols, const int* count,
                                void* out, int M, int N, int K, int dtype, cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) return 100;
    return launch_int8_gemm(CA, CB, out, SCA, SCB, bias, M, N, K, N, dtype, stream, subA, subBT, 64, count, cols, A);
}

// ---------------------------------------------------------------- grouped LLM.int8() (mixture-of-experts layers)
// The per-expert outliers of cbnb_b200_int8_grouped_mm, on the device: ends[E] (the clamped end rows), flags[E, K] (the
// columns where a row of expert e of A16, the fp16 activations, has |a| >= threshold), cols[E, K] / count[E] (each
// expert's ascending list), subA [M, 64] (each row's own expert's first 64 outlier columns of A), subBT [E * N, 64]
// (each routed expert's dequantised weight columns), and CA zeroed in each row's expert's outlier columns when the
// expert has more than one row.  Nothing depends on the data but the values written.  Returns 0, or 1 with the error
// message set for bad arguments.
int cbnb_b200_int8_grouped_outliers(const void* A, const void* A16, int8_t* CA, const int8_t* CB, const float* SCB,
                                    const int* offs, int E, float threshold, int* ends, int* flags, int* cols,
                                    int* count, void* subA, void* subBT, int M, int N, int K, int dtype,
                                    cudaStream_t stream) {
    if (A == nullptr || A16 == nullptr || CA == nullptr || CB == nullptr || SCB == nullptr || offs == nullptr ||
        ends == nullptr || flags == nullptr || cols == nullptr || count == nullptr || subA == nullptr ||
        subBT == nullptr || E < 1 || E > kMaxExperts || M < 0 || N <= 0 || K <= 0 || !(threshold > 0.f) ||
        (dtype != 1 && dtype != 2)) {
        set_last_error_msg("int8_grouped_outliers: needs every operand, 1 <= E <= 1024, M >= 0, N, K >= 1, "
                           "threshold > 0 and dtype 1 (fp16) or 2 (bf16)");
        return 1;
    }
    launch_int8_grouped_outliers(A, A16, CA, CB, SCB, offs, E, threshold, ends, flags, cols, count, subA, subBT, M, N,
                                 K, dtype, stream);
    return 0;
}

// The grouped LLM.int8() GEMM of a mixture-of-experts layer (no reference counterpart): out[m, :] (row stride N) = the
// epilogue of cbnb_b200_int8_scaled_mm (count NULL) or cbnb_b200_int8_mixed_mm_dev (count from
// cbnb_b200_int8_grouped_outliers) with expert e's weights CB[e * N ..], SCB[e * N ..], bias[e * N ..] for the rows of
// expert e, end_{e-1} <= m < end_e, and +0 for the rows past end_{E-1}; offs[E] (int32, on the device) holds the end
// rows, clamped on the device as end_e = min(max(offs[e], end_{e-1}), M).  Each expert's rows are bit for bit what
// those entries give on that expert's rows alone.  Returns 0; 1 with the error message set for bad arguments; 100, with
// nothing written and no message, for what the kernel does not serve (K % 16 != 0, E > 1024, unaligned codes); 100
// with the error message set when the launch fails.
int cbnb_b200_int8_grouped_mm(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB, const void* bias,
                              const int* offs, int E, const void* A, const void* subA, const void* subBT,
                              const int* cols, const int* count, void* out, int M, int N, int K, int dtype,
                              cudaStream_t stream) {
    if (CA == nullptr || CB == nullptr || SCA == nullptr || SCB == nullptr || offs == nullptr || out == nullptr ||
        M < 0 || N <= 0 || K <= 0 || E < 1 || (dtype != 1 && dtype != 2)) {
        set_last_error_msg("int8_grouped_mm: needs CA, CB, SCA, SCB, offs and out, M >= 0, N, K >= 1, E >= 1 and "
                           "dtype 1 (fp16) or 2 (bf16)");
        return 1;
    }
    const int rc =
        launch_int8_gemm_grouped(CA, CB, out, SCA, SCB, bias, offs, E, M, N, K, dtype, A, subA, subBT, cols, count,
                                 stream);
    return rc == 0 ? 0 : 100;
}

// Column-wise absmax + int8 codes of A[rows, cols] (the column half of the reference's int8_double_quant,
// backends/cuda/ops.py:262-296, used by MatMul8bitLt.backward).  dtype 1 = fp16, 2 = bf16.  Returns 0 / 100.
int cbnb_b200_int8_col_quant(const void* A, int8_t* out, float* col_stats, float threshold, int rows, int cols, int dtype,
                             cudaStream_t stream) {
    return launch_int8_col_quant(A, out, col_stats, threshold, rows, cols, dtype, stream) ? 0 : 100;
}

// The weight of LLM.int8()'s input gradient in one pass: out[n, k] (row stride ldo) = T(float(CB[n, k]) * s[n]), s[n] =
// SCB[n] * fp32(1/127), the bits of `CB.to(T, copy=True).mul_(SCB.unsqueeze(1).mul(1.0 / 127.0))`.  CB [rows, cols]
// contiguous.  dtype 1 = fp16, 2 = bf16.  Returns 0; 1 with the error message set for bad arguments; 100, with nothing
// written, for any other dtype.
int cbnb_b200_int8_dequant_rows(const int8_t* CB, const float* SCB, void* out, int ldo, int rows, int cols, int dtype,
                                cudaStream_t stream) {
    const bool empty = rows == 0 || cols == 0;
    if (rows < 0 || cols < 0 || ldo < cols || (!empty && (CB == nullptr || SCB == nullptr || out == nullptr))) {
        set_last_error_msg("int8_dequant_rows: needs CB, SCB and out, rows >= 0, cols >= 0 and ldo >= cols");
        return 1;
    }
    return launch_int8_dequant_rows(CB, SCB, out, ldo, rows, cols, dtype, stream) ? 0 : 100;
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

// ---------------------------------------------------------------- tensor-parallel LLM.int8() (parallel.py)
// The two halves of cbnb_b200_int8_vector_quant_flags, for a row-parallel layer whose ranks combine their row
// statistics (a max) before quantising: rowStats[rows] and col_flags[cols] (int32, zeroed by the caller; NULL when
// threshold == 0) without codes, then the codes of A from given statistics, with the same rounding.  dtype 1 = fp16,
// 2 = bf16.  Return 0, or 100 with the error message set.
int cbnb_b200_int8_row_stats(const void* A, float* rowStats, int* col_flags, float threshold, int rows, int cols,
                             int dtype, cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) {
        set_last_error_msg("int8_row_stats: dtype must be 1 (fp16) or 2 (bf16)");
        return 100;
    }
    launch_int8_row_stats(A, rowStats, col_flags, threshold, rows, cols, dtype, stream);
    return 0;
}

int cbnb_b200_int8_quant_with_stats(const void* A, int8_t* out, const float* rowStats, float threshold, int rows,
                                    int cols, int dtype, cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) {
        set_last_error_msg("int8_quant_with_stats: dtype must be 1 (fp16) or 2 (bf16)");
        return 100;
    }
    launch_int8_quant_with_stats(A, out, rowStats, threshold, rows, cols, dtype, stream);
    return 0;
}

// The int8 GEMM of cbnb_b200_int8_scaled_mm (epi 1 / 2, with the outlier term of cbnb_b200_int8_mixed_mm when
// jpad > 0) or of cigemmlt_32 (epi 0: int32 accumulators, jpad 0), storing every output element to each of
// outs[0 .. n_outs) (1 <= n_outs <= 8, device addresses: local buffers or peers' mapped buffers) at row stride ldc.
// Every destination holds the bits of the single-destination call.  Returns 0; 100 with the error message set for bad
// arguments; 100 without a message when the shape is not served (K % 16, alignment: the caller takes another route).
int cbnb_b200_int8_gemm_multi_out(const int8_t* CA, const int8_t* CB, const float* SCA, const float* SCB,
                                  const void* bias, const void* subA, const void* subBT, int jpad, void* const* outs,
                                  int n_outs, int M, int N, int K, int ldc, int epi, cudaStream_t stream) {
    if (outs == nullptr || n_outs < 1 || n_outs > 8 || epi < 0 || epi > 2 || ldc < N || (epi == 0 && jpad != 0)) {
        set_last_error_msg("int8_gemm_multi_out: needs 1 <= n_outs <= 8, epi 0 / 1 / 2, ldc >= N, no outliers at epi 0");
        return 100;
    }
    return launch_int8_gemm(CA, CB, nullptr, SCA, SCB, bias, M, N, K, ldc, epi, stream, subA, subBT, jpad, nullptr,
                            nullptr, nullptr, outs, n_outs);
}

// The int32 partial GEMM of a sequence-parallel K-sharded int8 layer: cbnb_b200_int8_gemm_multi_out at epi 0 with the
// rows scattered instead of copied.  Row m is stored to outs[m / rows_per_out] at row m % rows_per_out (row stride
// ldc), so outs is in rank order: outs[s] receives the tokens of rank s.  Returns 0; 1 with the error message set
// unless 1 <= n_outs <= 8, rows_per_out >= 1, n_outs * rows_per_out == M and ldc >= N; 100 when the shape is not
// served (K % 16, alignment: the caller takes another route).
int cbnb_b200_int8_gemm_partial_scatter(const int8_t* CA, const int8_t* CB, int32_t* const* outs, int n_outs,
                                        int rows_per_out, int M, int N, int K, int ldc, cudaStream_t stream) {
    if (outs == nullptr || n_outs < 1 || n_outs > 8 || rows_per_out < 1 || (long long)n_outs * rows_per_out != M ||
        ldc < N) {
        set_last_error_msg("int8_gemm_partial_scatter: needs 1 <= n_outs <= 8, rows_per_out >= 1, "
                           "n_outs * rows_per_out == M and ldc >= N");
        return 1;
    }
    return launch_int8_gemm(CA, CB, nullptr, nullptr, nullptr, nullptr, M, N, K, ldc, 0, stream, nullptr, nullptr, 0,
                            nullptr, nullptr, nullptr, reinterpret_cast<void* const*>(outs), n_outs, rows_per_out);
}

// out[m, n] (row stride ldc) = the int8 GEMM epilogue of cbnb_b200_int8_scaled_mm / cbnb_b200_int8_mixed_mm applied
// to sum_r parts[r][m, n]: the int32 partials of a K-sharded layer ([M, N] each, row stride N, one every part_stride
// elements), summed exactly, then dequantised with SCA[M] / SCB[N], the bias, and for jpad > 0 the outlier term of
// subA[M, jpad] . subBT[N, jpad]^T.  dtype 1 = fp16, 2 = bf16.  Returns 0, or 100 with the error message set.
int cbnb_b200_int8_reduce_partials(const int* parts, int world, long long part_stride, const float* SCA,
                                   const float* SCB, const void* bias, const void* subA, const void* subBT, int jpad,
                                   void* out, int M, int N, int ldc, int dtype, cudaStream_t stream) {
    if (!launch_reduce_int8_partials(parts, world, part_stride, SCA, SCB, bias, subA, subBT, jpad, out, M, N, ldc, dtype,
                                     stream)) {
        set_last_error_msg("int8_reduce_partials: needs world >= 1, ldc >= N, dtype 1 / 2, jpad a multiple of 8 "
                           "<= 64 with 16-byte aligned outlier operands");
        return 100;
    }
    return 0;
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
    return "bitsandbytes_b200: sm_90a; wgmma f16/bf16 (A from registers or shared memory) + s8; TMA 128B-swizzle; CUDA " BNB200_STR(
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

// Multi-tensor steps: one launch updates `count` tensors that share every per-launch scalar (and, 8-bit, the code
// books); each tensor brings its own pointers, size and step.  count <= cbnb_b200_optimizer_multi_capacity().
int cbnb_b200_optimizer_multi_capacity(void) { return optimizer_list_capacity(); }

static bool optimizer_list_ok(const char* what, int optimizer, int dtype, const OptimTensor* tensors, int count) {
    char msg[160];
    if (count < 0 || count > optimizer_list_capacity() || (count > 0 && tensors == nullptr))
        snprintf(msg, sizeof(msg), "%s: %d tensors (at most %d per call)", what, count, optimizer_list_capacity());
    else if (optimizer < 0 || optimizer > 5 || dtype < 0 || dtype > 2)
        snprintf(msg, sizeof(msg), "%s: unknown optimizer id %d or dtype id %d", what, optimizer, dtype);
    else
        return true;
    set_last_error_msg(msg);
    return false;
}

int cbnb_b200_optimizer_update_32bit_multi(int optimizer, int dtype, const OptimTensor* tensors, int count, float beta1,
                                           float beta2, float beta3, float alpha, float eps, float weight_decay,
                                           float lr, float gnorm_scale, bool skip_zeros, cudaStream_t stream) {
    if (!optimizer_list_ok("optimizer_update_32bit_multi", optimizer, dtype, tensors, count)) return 100;
    launch_optimizer32bit_list(optimizer, dtype, tensors, count, beta1, beta2, beta3, alpha, eps, weight_decay, lr,
                               gnorm_scale, skip_zeros, stream);
    return 0;
}

int cbnb_b200_optimizer_update_8bit_blockwise_multi(int optimizer, int dtype, const OptimTensor* tensors, int count,
                                                    float beta1, float beta2, float beta3, float alpha, float eps,
                                                    float weight_decay, float lr, const float* quantiles1,
                                                    const float* quantiles2, float gnorm_scale, bool skip_zeros,
                                                    cudaStream_t stream) {
    if (!optimizer_list_ok("optimizer_update_8bit_blockwise_multi", optimizer, dtype, tensors, count)) return 100;
    launch_optimizer8bit_blockwise_list(optimizer, dtype, tensors, count, beta1, beta2, beta3, alpha, eps,
                                        weight_decay, lr, quantiles1, quantiles2, gnorm_scale, skip_zeros, stream);
    return 0;
}

// Capturable multi-tensor steps: each descriptor's step_ptr is the tensor's int32 step counter in device memory, which
// the call advances before the update reads it; lr_dev, if not NULL, is read in place of lr.  A CUDA graph that
// captured the call therefore uses the current steps and learning rate at every replay.
static bool optimizer_steps_ok(const char* what, const OptimTensor* tensors, int count) {
    for (int i = 0; i < count; ++i) {
        if (tensors[i].step_ptr == nullptr) {
            char msg[160];
            snprintf(msg, sizeof(msg), "%s: tensor %d has no step counter (step_ptr is NULL)", what, i);
            set_last_error_msg(msg);
            return false;
        }
    }
    return true;
}

int cbnb_b200_optimizer_update_32bit_multi_dev(int optimizer, int dtype, const OptimTensor* tensors, int count,
                                               float beta1, float beta2, float beta3, float alpha, float eps,
                                               float weight_decay, float lr, const float* lr_dev, float gnorm_scale,
                                               bool skip_zeros, cudaStream_t stream) {
    const char* what = "optimizer_update_32bit_multi_dev";
    if (!optimizer_list_ok(what, optimizer, dtype, tensors, count) || !optimizer_steps_ok(what, tensors, count))
        return 100;
    launch_optimizer32bit_list_dev(optimizer, dtype, tensors, count, beta1, beta2, beta3, alpha, eps, weight_decay, lr,
                                   lr_dev, gnorm_scale, skip_zeros, stream);
    return 0;
}

int cbnb_b200_optimizer_update_8bit_blockwise_multi_dev(int optimizer, int dtype, const OptimTensor* tensors, int count,
                                                        float beta1, float beta2, float beta3, float alpha, float eps,
                                                        float weight_decay, float lr, const float* lr_dev,
                                                        const float* quantiles1, const float* quantiles2,
                                                        float gnorm_scale, bool skip_zeros, cudaStream_t stream) {
    const char* what = "optimizer_update_8bit_blockwise_multi_dev";
    if (!optimizer_list_ok(what, optimizer, dtype, tensors, count) || !optimizer_steps_ok(what, tensors, count))
        return 100;
    launch_optimizer8bit_blockwise_list_dev(optimizer, dtype, tensors, count, beta1, beta2, beta3, alpha, eps,
                                            weight_decay, lr, lr_dev, quantiles1, quantiles2, gnorm_scale, skip_zeros,
                                            stream);
    return 0;
}

// Data-parallel steps of one rank's pieces of flat buffers (optim/sharded.py): the _multi entries with the gradient
// summed over `world` source buffers in rank order and the new parameters written to `ndst` destination buffers.  Every
// descriptor's g and p must lie inside the local flat buffers [grad_local, + numel) and [param_local, + numel).
int cbnb_b200_optimizer_peers_capacity(void) { return optimizer_peers_capacity(); }

static bool optimizer_peers_ok(const char* what, int optimizer, const OptimTensor* tensors, int count, int dtype,
                               const void* const* grad_srcs, int world, void* const* param_dsts, int ndst,
                               const void* grad_local, const void* param_local, long long numel) {
    char msg[200];
    msg[0] = 0;
    const uintptr_t es = dtype == 0 ? 4 : 2;
    auto misaligned = [es](const void* v) { return v == nullptr || (reinterpret_cast<uintptr_t>(v) % es) != 0; };
    if (optimizer == 5)
        snprintf(msg, sizeof(msg), "%s: AdEMAMix has no data-parallel step", what);
    else if (world < 1 || world > optimizer_max_peers() || ndst < 1 || ndst > optimizer_max_peers() ||
             grad_srcs == nullptr || param_dsts == nullptr)
        snprintf(msg, sizeof(msg), "%s: %d gradient sources and %d parameter destinations (1..%d each)", what, world,
                 ndst, optimizer_max_peers());
    else if (misaligned(grad_local) || misaligned(param_local) || numel < 0)
        snprintf(msg, sizeof(msg), "%s: the local flat buffers must be non-null and aligned to their element", what);
    for (int r = 0; !msg[0] && r < world; ++r)
        if (misaligned(grad_srcs[r]))
            snprintf(msg, sizeof(msg), "%s: gradient source %d is null or not aligned to its element", what, r);
    for (int r = 0; !msg[0] && r < ndst; ++r)
        if (misaligned(param_dsts[r]))
            snprintf(msg, sizeof(msg), "%s: parameter destination %d is null or not aligned to its element", what, r);
    for (int i = 0; !msg[0] && i < count; ++i) {
        const long long go = static_cast<const char*>(tensors[i].g) - static_cast<const char*>(grad_local);
        const long long po = static_cast<const char*>(tensors[i].p) - static_cast<const char*>(param_local);
        const long long bytes = tensors[i].n * (long long)es, end = numel * (long long)es;
        if (tensors[i].n < 0 || go < 0 || po < 0 || go % (long long)es || po % (long long)es || go + bytes > end ||
            po + bytes > end)
            snprintf(msg, sizeof(msg), "%s: tensor %d lies outside the local flat buffers of %lld elements", what, i,
                     numel);
    }
    if (!msg[0]) return true;
    set_last_error_msg(msg);
    return false;
}

// count and ids: 100; everything else optimizer_peers_ok checks: 1 (the message set either way)
static bool optimizer_peers_ids_ok(const char* what, int optimizer, int dtype, const OptimTensor* tensors, int count) {
    if (count < 0 || count > optimizer_peers_capacity() || (count > 0 && tensors == nullptr) || optimizer < 0 ||
        optimizer > 5 || dtype < 0 || dtype > 2) {
        char msg[160];
        snprintf(msg, sizeof(msg), "%s: %d tensors (at most %d per call), optimizer id %d, dtype id %d", what, count,
                 optimizer_peers_capacity(), optimizer, dtype);
        set_last_error_msg(msg);
        return false;
    }
    return true;
}

// dev (the _peers_dev entries): the descriptors carry step pointers (NULL: 100) and lr_dev, if not NULL, replaces lr
static int optimizer_32bit_peers(const char* what, int optimizer, int dtype, const OptimTensor* tensors, int count,
                                 const void* const* grad_srcs, int world, void* const* param_dsts, int ndst,
                                 const void* grad_local, const void* param_local, long long numel, float grad_scale,
                                 float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay,
                                 float lr, bool skip_zeros, const float* gnorm_scale_dev, bool dev,
                                 const float* lr_dev, cudaStream_t stream) {
    if (!optimizer_peers_ids_ok(what, optimizer, dtype, tensors, count)) return 100;
    if (dev && !optimizer_steps_ok(what, tensors, count)) return 100;
    if (!optimizer_peers_ok(what, optimizer, tensors, count, dtype, grad_srcs, world, param_dsts, ndst, grad_local,
                            param_local, numel))
        return 1;
    launch_optimizer32bit_list_peers(optimizer, dtype, tensors, count, grad_srcs, world, param_dsts, ndst, grad_local,
                                     param_local, grad_scale, beta1, beta2, beta3, alpha, eps, weight_decay, lr,
                                     skip_zeros, gnorm_scale_dev, dev, lr_dev, stream);
    return 0;
}

static int optimizer_8bit_peers(const char* what, int optimizer, int dtype, const OptimTensor* tensors, int count,
                                const void* const* grad_srcs, int world, void* const* param_dsts, int ndst,
                                const void* grad_local, const void* param_local, long long numel, float grad_scale,
                                float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay,
                                float lr, const float* quantiles1, const float* quantiles2, bool skip_zeros,
                                const float* gnorm_scale_dev, bool dev, const float* lr_dev, cudaStream_t stream) {
    if (!optimizer_peers_ids_ok(what, optimizer, dtype, tensors, count)) return 100;
    if (dev && !optimizer_steps_ok(what, tensors, count)) return 100;
    if (!optimizer_peers_ok(what, optimizer, tensors, count, dtype, grad_srcs, world, param_dsts, ndst, grad_local,
                            param_local, numel))
        return 1;
    if (quantiles1 == nullptr || (optimizer == 0 && quantiles2 == nullptr)) {
        char msg[160];
        snprintf(msg, sizeof(msg), "%s: missing code book", what);
        set_last_error_msg(msg);
        return 1;
    }
    launch_optimizer8bit_blockwise_list_peers(optimizer, dtype, tensors, count, grad_srcs, world, param_dsts, ndst,
                                              grad_local, param_local, grad_scale, beta1, beta2, beta3, alpha, eps,
                                              weight_decay, lr, quantiles1, quantiles2, skip_zeros, gnorm_scale_dev,
                                              dev, lr_dev, stream);
    return 0;
}

int cbnb_b200_optimizer_update_32bit_multi_peers(int optimizer, int dtype, const OptimTensor* tensors, int count,
                                                 const void* const* grad_srcs, int world, void* const* param_dsts,
                                                 int ndst, const void* grad_local, const void* param_local,
                                                 long long numel, float grad_scale, float beta1, float beta2,
                                                 float beta3, float alpha, float eps, float weight_decay, float lr,
                                                 bool skip_zeros, cudaStream_t stream) {
    return optimizer_32bit_peers("optimizer_update_32bit_multi_peers", optimizer, dtype, tensors, count, grad_srcs,
                                 world, param_dsts, ndst, grad_local, param_local, numel, grad_scale, beta1, beta2,
                                 beta3, alpha, eps, weight_decay, lr, skip_zeros, nullptr, false, nullptr, stream);
}

int cbnb_b200_optimizer_update_8bit_blockwise_multi_peers(int optimizer, int dtype, const OptimTensor* tensors,
                                                          int count, const void* const* grad_srcs, int world,
                                                          void* const* param_dsts, int ndst, const void* grad_local,
                                                          const void* param_local, long long numel, float grad_scale,
                                                          float beta1, float beta2, float beta3, float alpha, float eps,
                                                          float weight_decay, float lr, const float* quantiles1,
                                                          const float* quantiles2, bool skip_zeros,
                                                          cudaStream_t stream) {
    return optimizer_8bit_peers("optimizer_update_8bit_blockwise_multi_peers", optimizer, dtype, tensors, count,
                                grad_srcs, world, param_dsts, ndst, grad_local, param_local, numel, grad_scale, beta1,
                                beta2, beta3, alpha, eps, weight_decay, lr, quantiles1, quantiles2, skip_zeros,
                                nullptr, false, nullptr, stream);
}

// The clipped data-parallel steps: as the _peers entries, with the gradient factor (gnorm_scale of the _multi
// entries) read by each CTA from gnorm_scale_dev in device memory; NULL means 1, the _peers entries' bits.
int cbnb_b200_optimizer_update_32bit_multi_peers_scaled(int optimizer, int dtype, const OptimTensor* tensors, int count,
                                                        const void* const* grad_srcs, int world,
                                                        void* const* param_dsts, int ndst, const void* grad_local,
                                                        const void* param_local, long long numel, float grad_scale,
                                                        float beta1, float beta2, float beta3, float alpha, float eps,
                                                        float weight_decay, float lr, bool skip_zeros,
                                                        const float* gnorm_scale_dev, cudaStream_t stream) {
    return optimizer_32bit_peers("optimizer_update_32bit_multi_peers_scaled", optimizer, dtype, tensors, count,
                                 grad_srcs, world, param_dsts, ndst, grad_local, param_local, numel, grad_scale, beta1,
                                 beta2, beta3, alpha, eps, weight_decay, lr, skip_zeros, gnorm_scale_dev, false, nullptr,
                                 stream);
}

int cbnb_b200_optimizer_update_8bit_blockwise_multi_peers_scaled(
    int optimizer, int dtype, const OptimTensor* tensors, int count, const void* const* grad_srcs, int world,
    void* const* param_dsts, int ndst, const void* grad_local, const void* param_local, long long numel,
    float grad_scale, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr,
    const float* quantiles1, const float* quantiles2, bool skip_zeros, const float* gnorm_scale_dev,
    cudaStream_t stream) {
    return optimizer_8bit_peers("optimizer_update_8bit_blockwise_multi_peers_scaled", optimizer, dtype, tensors, count,
                                grad_srcs, world, param_dsts, ndst, grad_local, param_local, numel, grad_scale, beta1,
                                beta2, beta3, alpha, eps, weight_decay, lr, quantiles1, quantiles2, skip_zeros,
                                gnorm_scale_dev, false, nullptr, stream);
}

// Capturable data-parallel steps: the _peers_scaled entries with each descriptor's step_ptr pointing to the tensor's
// int32 step counter in device memory, and lr_dev, if not NULL, read in place of lr.  Unlike the _multi_dev entries
// they read the counters and do not advance them: a parameter's step advances on every rank, also on ranks that hold
// no piece of it, so the caller advances its counters once per step before the call.
int cbnb_b200_optimizer_update_32bit_multi_peers_dev(int optimizer, int dtype, const OptimTensor* tensors, int count,
                                                     const void* const* grad_srcs, int world, void* const* param_dsts,
                                                     int ndst, const void* grad_local, const void* param_local,
                                                     long long numel, float grad_scale, float beta1, float beta2,
                                                     float beta3, float alpha, float eps, float weight_decay, float lr,
                                                     bool skip_zeros, const float* gnorm_scale_dev,
                                                     const float* lr_dev, cudaStream_t stream) {
    return optimizer_32bit_peers("optimizer_update_32bit_multi_peers_dev", optimizer, dtype, tensors, count,
                                 grad_srcs, world, param_dsts, ndst, grad_local, param_local, numel, grad_scale, beta1,
                                 beta2, beta3, alpha, eps, weight_decay, lr, skip_zeros, gnorm_scale_dev, true, lr_dev,
                                 stream);
}

int cbnb_b200_optimizer_update_8bit_blockwise_multi_peers_dev(
    int optimizer, int dtype, const OptimTensor* tensors, int count, const void* const* grad_srcs, int world,
    void* const* param_dsts, int ndst, const void* grad_local, const void* param_local, long long numel,
    float grad_scale, float beta1, float beta2, float beta3, float alpha, float eps, float weight_decay, float lr,
    const float* quantiles1, const float* quantiles2, bool skip_zeros, const float* gnorm_scale_dev,
    const float* lr_dev, cudaStream_t stream) {
    return optimizer_8bit_peers("optimizer_update_8bit_blockwise_multi_peers_dev", optimizer, dtype, tensors, count,
                                grad_srcs, world, param_dsts, ndst, grad_local, param_local, numel, grad_scale, beta1,
                                beta2, beta3, alpha, eps, weight_decay, lr, quantiles1, quantiles2, skip_zeros,
                                gnorm_scale_dev, true, lr_dev, stream);
}

// The norm of the reduced gradient over one rank's pieces (gradient clipping, optim/sharded.py): each element's
// gradient is formed as the _peers entries form it; the launch's sum of squares (or max |g|, inf_norm) is added
// (max-ed) into *acc in fp64, in stream order.  Only each descriptor's g and n are read.
int cbnb_b200_optimizer_grad_norm_peers(int dtype, const OptimTensor* tensors, int count, const void* const* grad_srcs,
                                        int world, const void* grad_local, long long numel, float grad_scale,
                                        bool inf_norm, double* acc, cudaStream_t stream) {
    const char* what = "optimizer_grad_norm_peers";
    char msg[200];
    msg[0] = 0;
    if (count < 0 || count > optimizer_peers_capacity() || (count > 0 && tensors == nullptr) || dtype < 0 ||
        dtype > 2) {
        snprintf(msg, sizeof(msg), "%s: %d tensors (at most %d per call), dtype id %d", what, count,
                 optimizer_peers_capacity(), dtype);
        set_last_error_msg(msg);
        return 100;
    }
    const uintptr_t es = dtype == 0 ? 4 : 2;
    auto misaligned = [](const void* v, uintptr_t a) { return v == nullptr || (reinterpret_cast<uintptr_t>(v) % a); };
    if (world < 1 || world > optimizer_max_peers() || grad_srcs == nullptr)
        snprintf(msg, sizeof(msg), "%s: %d gradient sources (1..%d)", what, world, optimizer_max_peers());
    else if (misaligned(grad_local, es) || numel < 0)
        snprintf(msg, sizeof(msg), "%s: the local flat gradient must be non-null and aligned to its element", what);
    else if (misaligned(acc, sizeof(double)))
        snprintf(msg, sizeof(msg), "%s: the accumulator must be a non-null, aligned double", what);
    for (int r = 0; !msg[0] && r < world; ++r)
        if (misaligned(grad_srcs[r], es))
            snprintf(msg, sizeof(msg), "%s: gradient source %d is null or not aligned to its element", what, r);
    for (int i = 0; !msg[0] && i < count; ++i) {
        const long long go = static_cast<const char*>(tensors[i].g) - static_cast<const char*>(grad_local);
        if (tensors[i].n < 0 || go < 0 || go % (long long)es || go + tensors[i].n * (long long)es > numel * (long long)es)
            snprintf(msg, sizeof(msg), "%s: tensor %d lies outside the local flat gradient of %lld elements", what, i,
                     numel);
    }
    if (msg[0]) {
        set_last_error_msg(msg);
        return 1;
    }
    return launch_optimizer_grad_norm_peers(dtype, tensors, count, grad_srcs, world, grad_local, grad_scale, inf_norm,
                                            acc, stream)
               ? 0
               : 100;
}

// The global norm and the clip coefficient from the ranks' values of cbnb_b200_optimizer_grad_norm_peers
int cbnb_b200_optimizer_clip_coef(const double* rank_values, int world, bool inf_norm, float max_norm, float* out,
                                  cudaStream_t stream) {
    if (world < 1 || rank_values == nullptr || reinterpret_cast<uintptr_t>(rank_values) % sizeof(double) ||
        out == nullptr || reinterpret_cast<uintptr_t>(out) % sizeof(float)) {
        char msg[160];
        snprintf(msg, sizeof(msg), "optimizer_clip_coef: %d rank values (at least 1), and non-null aligned buffers",
                 world);
        set_last_error_msg(msg);
        return 1;
    }
    launch_optimizer_clip_coef(rank_values, world, inf_norm, max_norm, out, stream);
    return 0;
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
