// int8.cu -- the LLM.int8() hot path for sm_90a.
//
//   int8_vector_quant   replaces reference kInt8VectorQuant (csrc/kernels.cu:1331-1385):
//                       one read of A instead of two (the row is held in registers between
//                       the absmax pass and the quantise pass) and, optionally, outlier-column
//                       flags in the same pass (the reference finds them with 3-4 torch kernels
//                       and a host sync, backends/cuda/ops.py:230-236).
//   int8 GEMM           lives in int8_gemm.cu.
//   dequant_mm_int32    replaces reference kdequant_mm_int32_fp16 (csrc/kernels.cu:1396-1448).
#include "common.cuh"
#include "hopper_ptx.cuh"

namespace bnb200 {

namespace {

// ======================================================================================
// row-wise int8 quantisation
// ======================================================================================
constexpr int kVqThreads = 256;
constexpr int kVqVecs = 4;  // 16-byte vectors cached per thread -> rows up to 256*4*8 = 8192 columns

template <typename T> __device__ __forceinline__ void unpack8(const uint4& r, float (&v)[8]);
template <> __device__ __forceinline__ void unpack8<__half>(const uint4& r, float (&v)[8]) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        v[2 * i] = f.x;
        v[2 * i + 1] = f.y;
    }
}
template <> __device__ __forceinline__ void unpack8<__nv_bfloat16>(const uint4& r, float (&v)[8]) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        v[2 * i] = __uint_as_float(w[i] << 16);
        v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
}

__device__ __forceinline__ float block_max(float m, float* sred) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = m;
    __syncthreads();
    float r = sred[0];
#pragma unroll
    for (int w = 1; w < kVqThreads / 32; ++w) r = fmaxf(r, sred[w]);
    return r;
}

__device__ __forceinline__ int8_t quant_one(float v, float scale) {
    // __float2int_rn(val * scale) truncated to int8, reference kernels.cu:1376-1381
    return (int8_t)__float2int_rn(mul_ftz(v, scale));
}

// One CTA per row.  thr_stat = threshold as the reference's first pass sees it (rounded to T),
// thr = raw fp32 threshold used by the second pass (reference kernels.cu:1358 vs :1378).
template <typename T, bool kVec>
__global__ void __launch_bounds__(kVqThreads)
    int8_vector_quant_kernel(const T* __restrict__ A, int8_t* __restrict__ out, float* __restrict__ rowStats,
                             int* __restrict__ col_flags, float thr, float thr_stat, int rows, int cols) {
    __shared__ float sred[kVqThreads / 32];
    const int row = blockIdx.x;
    const T* a = A + (long long)row * cols;
    int8_t* o = out + (long long)row * cols;
    const bool sparse = thr > 0.0f;

    // T(-FLT_MIN) is -0.0 for 16-bit T (reference kernels.cu:1353); max with -0.0 keeps it for an
    // all-outlier row.
    float m = -0.0f;

    if constexpr (kVec) {
        uint4 cache[kVqVecs];
        const int nvec = cols >> 3;
#pragma unroll
        for (int j = 0; j < kVqVecs; ++j) {
            const int vi = threadIdx.x + j * kVqThreads;
            cache[j] = make_uint4(0, 0, 0, 0);
            if (vi < nvec) cache[j] = ldg_stream_v4(a + 8 * vi);
        }
#pragma unroll
        for (int j = 0; j < kVqVecs; ++j) {
            const int vi = threadIdx.x + j * kVqThreads;
            if (vi < nvec) {
                float v[8];
                unpack8<T>(cache[j], v);
#pragma unroll
                for (int t = 0; t < 8; ++t) {
                    const float av = fabsf(v[t]);
                    if (!sparse || av < thr_stat) m = fmaxf(m, av);
                    if (sparse && col_flags != nullptr && av >= thr) col_flags[8 * vi + t] = 1;
                }
            }
        }
        const float row_absmax = block_max(m, sred);
        if (threadIdx.x == 0) rowStats[row] = row_absmax;
        const float scale = div_approx_ftz(127.0f, row_absmax);  // __fdividef
#pragma unroll
        for (int j = 0; j < kVqVecs; ++j) {
            const int vi = threadIdx.x + j * kVqThreads;
            if (vi < nvec) {
                float v[8];
                unpack8<T>(cache[j], v);
                uint32_t w[2] = {0u, 0u};
#pragma unroll
                for (int t = 0; t < 8; ++t) {
                    int8_t q = (!sparse || fabsf(v[t]) < thr) ? quant_one(v[t], scale) : (int8_t)0;
                    w[t >> 2] |= (uint32_t)(uint8_t)q << (8 * (t & 3));
                }
                stg_stream_v2(o + 8 * vi, make_uint2(w[0], w[1]));
            }
        }
    } else {
        for (int c = threadIdx.x; c < cols; c += kVqThreads) {
            const float av = fabsf(DT<T>::to_f32(a[c]));
            if (!sparse || av < thr_stat) m = fmaxf(m, av);
            if (sparse && col_flags != nullptr && av >= thr) col_flags[c] = 1;
        }
        const float row_absmax = block_max(m, sred);
        if (threadIdx.x == 0) rowStats[row] = row_absmax;
        const float scale = div_approx_ftz(127.0f, row_absmax);
        for (int c = threadIdx.x; c < cols; c += kVqThreads) {
            const float v = DT<T>::to_f32(a[c]);
            o[c] = (!sparse || fabsf(v) < thr) ? quant_one(v, scale) : (int8_t)0;
        }
    }
}

// ======================================================================================
// int32 -> fp16 dequantisation epilogue as a stand-alone kernel (cdequant_mm_int32_fp16 ABI)
// ======================================================================================
__global__ void __launch_bounds__(256)
    dequant_mm_int32_fp16_kernel(const int* __restrict__ A, const float* __restrict__ rowStats,
                                 const float* __restrict__ colStats, __half* __restrict__ out,
                                 const __half* __restrict__ bias, int numRows, int numCols, int vec_ok) {
    const int row = blockIdx.y;
    const float rs = __ldg(rowStats + row);
    const int* a = A + (long long)row * numCols;
    __half* o = out + (long long)row * numCols;
    if (vec_ok) {
        const int nvec = numCols >> 2;
        for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += gridDim.x * blockDim.x) {
            const uint4 x = ldg_stream_v4(a + 4 * v);
            const float4 cs = __ldg(reinterpret_cast<const float4*>(colStats) + v);
            float b[4] = {0.f, 0.f, 0.f, 0.f};
            if (bias != nullptr) {
                const uint2 bb = __ldg(reinterpret_cast<const uint2*>(bias) + v);
                const float2 b01 = __half22float2(*reinterpret_cast<const __half2*>(&bb.x));
                const float2 b23 = __half22float2(*reinterpret_cast<const __half2*>(&bb.y));
                b[0] = b01.x; b[1] = b01.y; b[2] = b23.x; b[3] = b23.y;
            }
            const uint32_t lo = pack2<__half>(dequant_value((int)x.x, rs, cs.x, b[0]),
                                              dequant_value((int)x.y, rs, cs.y, b[1]));
            const uint32_t hi = pack2<__half>(dequant_value((int)x.z, rs, cs.z, b[2]),
                                              dequant_value((int)x.w, rs, cs.w, b[3]));
            stg_stream_v2(o + 4 * v, make_uint2(lo, hi));
        }
    } else {
        for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < numCols; c += gridDim.x * blockDim.x) {
            const float b = bias != nullptr ? __half2float(bias[c]) : 0.f;
            o[c] = __float2half_rn(dequant_value(a[c], rs, __ldg(colStats + c), b));
        }
    }
}

// ======================================================================================
// outlier decomposition glue (reference backends/default/ops.py:79-90 does this with torch indexing,
// int8_vectorwise_dequant and .t()): one launch gathers the outlier columns of the activations,
//     subA[m, j]  = A[m, cols[j]]                                  (zero-padded to jpad columns)
// and dequantises the matching weight columns, already in the [N, jpad] layout the GEMM epilogue reads,
//     subBT[n, j] = T( (float(CB[n, cols[j]]) * SCB[n]) * (1/127) )  (reference _ops.py:118-121: fp32, then A.dtype)
// ======================================================================================
template <typename T>
__global__ void __launch_bounds__(256)
    int8_outlier_prep_kernel(const T* __restrict__ A, const int8_t* __restrict__ CB, const float* __restrict__ SCB,
                             const long long* __restrict__ cols, int J, int jpad, int M, int N, int K,
                             T* __restrict__ subA, T* __restrict__ subBT) {
    const long long total = (long long)(M + N) * jpad;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long r = idx / jpad;
        const int j = (int)(idx - r * jpad);
        const long long col = j < J ? cols[j] : 0;
        if (r < M) {
            subA[idx] = j < J ? A[r * K + col] : DT<T>::from_f32(0.f);
        } else {
            const long long n = r - M;
            float v = 0.f;
            if (j < J) v = __fmul_rn(__fmul_rn((float)CB[n * K + col], __ldg(SCB + n)), 7.874015718698502e-3f);
            subBT[n * jpad + j] = DT<T>::from_f32(v);
        }
    }
}

// CA[:, cols[j]] = 0 for every outlier column (reference backends/cuda/ops.py:233-236, a torch index_put there)
__global__ void __launch_bounds__(256)
    int8_zero_columns_kernel(int8_t* __restrict__ CA, const long long* __restrict__ cols, int J, int rows, int K) {
    const long long total = (long long)rows * J;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long r = idx / J;
        CA[r * K + cols[idx - r * J]] = 0;
    }
}


// ---------------------------------------------------------------------------------------------------------------
// Column-wise int8 quantisation for MatMul8bitLt.backward (SURVEY.md section 8 row f-1): the reference computes it
// with five PyTorch kernels (backends/cuda/ops.py:262-296: abs, mask, amax over rows, masked_fill, mul / div / round /
// cast).  Here: one pass for the column absmax (entries >= threshold excluded), one for the codes:
//     q[r, c] = int8( rint( float( T(A[r, c] * 127) ) / col_stats[c] ) ),   outliers -> 0
// (the product is rounded to T, as `A.mul(127.0)` on a T tensor is; the division is fp32 round-to-nearest, as the
// T / fp32 type promotion makes it; a column without a non-outlier entry divides 0 by 0 and casts the NaN to 0).
// A warp walks rows; a lane owns 8 consecutive columns (16-byte loads, 8-byte stores of the codes).
template <typename T>
__global__ void __launch_bounds__(256) int8_col_absmax_kernel(const T* __restrict__ A, float* __restrict__ col_stats,
                                                              float threshold, int rows, int cols, int rows_per_cta) {
    const int c0 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 8;  // this lane's first column
    const int r_begin = blockIdx.y * rows_per_cta + (threadIdx.x >> 5);
    const int r_end = min(rows, (blockIdx.y + 1) * rows_per_cta);
    if (c0 >= cols) return;
    float m[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const bool full = c0 + 8 <= cols && (cols & 7) == 0;
    for (int r = r_begin; r < r_end; r += 8) {
        float v[8];
        if (full) {
            unpack8<T>(__ldg(reinterpret_cast<const uint4*>(A + (long long)r * cols + c0)), v);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = c0 + j < cols ? DT<T>::to_f32(A[(long long)r * cols + c0 + j]) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float a = fabsf(v[j]);
            if (!(threshold > 0.0f && a >= threshold)) m[j] = fmaxf(m[j], a);
        }
    }
    // non-negative floats order like their bit patterns: an integer atomicMax combines the CTAs' partial maxima
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (c0 + j < cols && m[j] > 0.f) atomicMax(reinterpret_cast<int*>(col_stats) + c0 + j, __float_as_int(m[j]));
}

template <typename T>
__global__ void __launch_bounds__(256) int8_col_quant_kernel(const T* __restrict__ A, const float* __restrict__ col_stats,
                                                             int8_t* __restrict__ out, float threshold, int rows, int cols,
                                                             int rows_per_cta) {
    const int c0 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 8;
    const int r_begin = blockIdx.y * rows_per_cta + (threadIdx.x >> 5);
    const int r_end = min(rows, (blockIdx.y + 1) * rows_per_cta);
    if (c0 >= cols) return;
    const bool full = c0 + 8 <= cols && (cols & 7) == 0;
    float cs[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) cs[j] = c0 + j < cols ? col_stats[c0 + j] : 1.f;
    for (int r = r_begin; r < r_end; r += 8) {
        float v[8];
        if (full) {
            unpack8<T>(__ldg(reinterpret_cast<const uint4*>(A + (long long)r * cols + c0)), v);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = c0 + j < cols ? DT<T>::to_f32(A[(long long)r * cols + c0 + j]) : 0.f;
        }
        alignas(8) int8_t q[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float x = v[j];
            if (threshold > 0.0f && fabsf(x) >= threshold) x = 0.f;
            x = DT<T>::to_f32(DT<T>::from_f32(__fmul_rn(x, 127.0f)));
            const float d = __fdiv_rn(x, cs[j]);
            q[j] = (d == d) ? (int8_t)__float2int_rn(d) : (int8_t)0;
        }
        if (full) {
            *reinterpret_cast<uint2*>(out + (long long)r * cols + c0) = *reinterpret_cast<const uint2*>(q);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (c0 + j < cols) out[(long long)r * cols + c0 + j] = q[j];
        }
    }
}

} // namespace

// ---------------------------------------------------------------- launch wrappers
void launch_int8_outlier_prep(const void* A, const int8_t* CB, const float* SCB, const long long* cols, int J, int jpad,
                              int M, int N, int K, int dtype, void* subA, void* subBT, cudaStream_t stream) {
    if (jpad <= 0 || M + N <= 0) return;
    const long long total = (long long)(M + N) * jpad;
    long long want = (total + 255) / 256;
    const int grid = (int)(want < 132 * 16 ? want : 132 * 16);
    if (dtype == 1)
        int8_outlier_prep_kernel<__half><<<grid, 256, 0, stream>>>((const __half*)A, CB, SCB, cols, J, jpad, M, N, K,
                                                                   (__half*)subA, (__half*)subBT);
    else
        int8_outlier_prep_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)A, CB, SCB, cols, J, jpad,
                                                                          M, N, K, (__nv_bfloat16*)subA,
                                                                          (__nv_bfloat16*)subBT);
    BNB200_CHECK_LAUNCH("int8_outlier_prep");
}

// q_col[rows, cols] + col_stats[cols] of A[rows, cols]; dtype: 1 fp16, 2 bf16 (false: dtype not served)
bool launch_int8_col_quant(const void* A, int8_t* out, float* col_stats, float threshold, int rows, int cols, int dtype,
                           cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) return false;
    if (rows <= 0 || cols <= 0) return true;
    cudaMemsetAsync(col_stats, 0, sizeof(float) * (size_t)cols, stream);
    const int col_ctas = (cols + 255) / 256;
    // enough row slices to fill the machine, at least 8 rows (one per warp) each
    int slices = (4 * device_sm_count() + col_ctas - 1) / col_ctas;
    if (slices > (rows + 7) / 8) slices = (rows + 7) / 8;
    if (slices < 1) slices = 1;
    const int rows_per_cta = (((rows + slices - 1) / slices) + 7) / 8 * 8;
    const dim3 grid(col_ctas, (rows + rows_per_cta - 1) / rows_per_cta);
#define BNB200_COLQ(T)                                                                                                 \
    int8_col_absmax_kernel<T><<<grid, 256, 0, stream>>>((const T*)A, col_stats, threshold, rows, cols, rows_per_cta);  \
    int8_col_quant_kernel<T><<<grid, 256, 0, stream>>>((const T*)A, col_stats, out, threshold, rows, cols, rows_per_cta)
    if (dtype == 1) {
        BNB200_COLQ(__half);
    } else {
        BNB200_COLQ(__nv_bfloat16);
    }
#undef BNB200_COLQ
    BNB200_CHECK_LAUNCH("int8_col_quant");
    return true;
}

void launch_int8_zero_columns(int8_t* CA, const long long* cols, int J, int rows, int K, cudaStream_t stream) {
    if (J <= 0 || rows <= 0) return;
    const long long total = (long long)rows * J;
    long long want = (total + 255) / 256;
    const int grid = (int)(want < 132 * 16 ? want : 132 * 16);
    int8_zero_columns_kernel<<<grid, 256, 0, stream>>>(CA, cols, J, rows, K);
    BNB200_CHECK_LAUNCH("int8_zero_columns");
}

void launch_int8_vector_quant(const void* A, int8_t* out, float* rowStats, int* col_flags, float threshold, int rows,
                              int cols, int dtype /*1 fp16, 2 bf16*/, cudaStream_t stream) {
    if (rows <= 0 || cols <= 0) return;
    const bool vec = (cols % 8 == 0) && (cols <= kVqThreads * kVqVecs * 8) &&
                     ((reinterpret_cast<uintptr_t>(A) & 15) == 0) && ((reinterpret_cast<uintptr_t>(out) & 7) == 0);
    // threshold as the statistic pass of the reference compares it: rounded to the input type
    float thr_stat = threshold;
    if (dtype == 1) thr_stat = __half2float(__float2half_rn(threshold));
    if (dtype == 2) thr_stat = __bfloat162float(__float2bfloat16_rn(threshold));
    if (dtype == 1) {
        const __half* a = reinterpret_cast<const __half*>(A);
        if (vec)
            int8_vector_quant_kernel<__half, true>
                <<<rows, kVqThreads, 0, stream>>>(a, out, rowStats, col_flags, threshold, thr_stat, rows, cols);
        else
            int8_vector_quant_kernel<__half, false>
                <<<rows, kVqThreads, 0, stream>>>(a, out, rowStats, col_flags, threshold, thr_stat, rows, cols);
    } else {
        const __nv_bfloat16* a = reinterpret_cast<const __nv_bfloat16*>(A);
        if (vec)
            int8_vector_quant_kernel<__nv_bfloat16, true>
                <<<rows, kVqThreads, 0, stream>>>(a, out, rowStats, col_flags, threshold, thr_stat, rows, cols);
        else
            int8_vector_quant_kernel<__nv_bfloat16, false>
                <<<rows, kVqThreads, 0, stream>>>(a, out, rowStats, col_flags, threshold, thr_stat, rows, cols);
    }
    BNB200_CHECK_LAUNCH("int8_vector_quant");
}

void launch_dequant_mm_int32_fp16(const int* A, const float* rowStats, const float* colStats, __half* out,
                                  const __half* bias, int numRows, int numCols, cudaStream_t stream) {
    if (numRows <= 0 || numCols <= 0) return;
    const bool vec = (numCols % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(out) & 7) == 0) &&
                     ((reinterpret_cast<uintptr_t>(colStats) & 15) == 0) &&
                     (bias == nullptr || (reinterpret_cast<uintptr_t>(bias) & 7) == 0);
    int per_row = vec ? (numCols / 4 + 255) / 256 : (numCols + 255) / 256;
    if (per_row > 64) per_row = 64;
    // blockIdx.y carries the row; 65535 rows per launch
    for (int r0 = 0; r0 < numRows; r0 += 65535) {
        const int nr = (numRows - r0 < 65535) ? numRows - r0 : 65535;
        dim3 grid(per_row, nr);
        dequant_mm_int32_fp16_kernel<<<grid, 256, 0, stream>>>(A + (long long)r0 * numCols, rowStats + r0, colStats,
                                                               out + (long long)r0 * numCols, bias, nr, numCols,
                                                               vec ? 1 : 0);
    }
    BNB200_CHECK_LAUNCH("dequant_mm_int32_fp16");
}

} // namespace bnb200
