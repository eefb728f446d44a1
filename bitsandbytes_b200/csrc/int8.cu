// int8.cu -- the LLM.int8() hot path for sm_90a.
//
//   int8_vector_quant   replaces reference kInt8VectorQuant (csrc/kernels.cu:1331-1385):
//                       one read of A instead of two (the row is held in registers between
//                       the absmax pass and the quantise pass) and, optionally, outlier-column
//                       flags in the same pass (the reference finds them with 3-4 torch kernels
//                       and a host sync, backends/cuda/ops.py:230-236).
//   outlier compaction  the outlier flags -> the ascending column list and its count, on the device, for the
//                       route that a CUDA graph can capture (no torch.nonzero, no host sync).
//   int8 GEMM           lives in int8_gemm.cu.
//   dequant_mm_int32    replaces reference kdequant_mm_int32_fp16 (csrc/kernels.cu:1396-1448).
//   int8_dequant_rows   the weight of the input gradient, W = T(CB * SCB / 127), in one pass (the reference's
//                       MatMul8bitLt.backward builds it with two torch kernels and a temporary).
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
// MODE 0: statistics, flags and codes.  MODE 1: the row statistics and the outlier flags only (no codes).  MODE 2: the
// codes only, from the statistics given in rowStats -- the two halves of MODE 0, for a row-parallel layer whose ranks
// combine their statistics (a max over the ranks) before quantising.
template <typename T, bool kVec, int MODE = 0>
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
        float row_absmax;
        if constexpr (MODE != 2) {
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
            row_absmax = block_max(m, sred);
            if (threadIdx.x == 0) rowStats[row] = row_absmax;
            if constexpr (MODE == 1) return;
        } else {
            row_absmax = rowStats[row];
        }
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
        float row_absmax;
        if constexpr (MODE != 2) {
            for (int c = threadIdx.x; c < cols; c += kVqThreads) {
                const float av = fabsf(DT<T>::to_f32(a[c]));
                if (!sparse || av < thr_stat) m = fmaxf(m, av);
                if (sparse && col_flags != nullptr && av >= thr) col_flags[c] = 1;
            }
            row_absmax = block_max(m, sred);
            if (threadIdx.x == 0) rowStats[row] = row_absmax;
            if constexpr (MODE == 1) return;
        } else {
            row_absmax = rowStats[row];
        }
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
// With `count` set (the capturable route), the outlier count is read from device memory: the operands hold the first
// min(count, jpad) columns, and the launch also zeroes CA[:, cols[j]] for all `count` of them (the job of
// int8_zero_columns on the eager route).  The grid does not depend on the count.
template <typename T, typename Idx>
__global__ void __launch_bounds__(256)
    int8_outlier_prep_kernel(const T* __restrict__ A, const int8_t* __restrict__ CB, const float* __restrict__ SCB,
                             const Idx* __restrict__ cols, const int* __restrict__ count, int J, int jpad, int M, int N,
                             int K, T* __restrict__ subA, T* __restrict__ subBT, int8_t* __restrict__ CA) {
    if (count != nullptr) {
        const int all = *count;
        J = min(all, jpad);
        const long long zeros = (long long)M * all;
        for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < zeros;
             idx += (long long)gridDim.x * blockDim.x) {
            const long long r = idx / all;
            CA[r * K + cols[idx - r * all]] = 0;
        }
    }
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

// The outlier columns in ascending order (the order torch.nonzero gives) and their count, without a host round trip.
// One CTA walks the flags in tiles of 1024 columns: a ballot per warp counts and ranks the flagged columns of the warp,
// and the counts of the warps before it place them.
constexpr int kCompactThreads = 1024;
__device__ __forceinline__ void outlier_compact(const int* __restrict__ flags, int K, int* __restrict__ cols,
                                                int* __restrict__ count) {
    __shared__ int s_warp[kCompactThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int base = 0;
    for (int c0 = 0; c0 < K; c0 += kCompactThreads) {
        const int c = c0 + threadIdx.x;
        const bool f = c < K && flags[c] != 0;
        const unsigned ballot = __ballot_sync(0xffffffffu, f);
        if (lane == 0) s_warp[warp] = __popc(ballot);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kCompactThreads / 32; ++w) {
            const int n = s_warp[w];
            before += w < warp ? n : 0;
            total += n;
        }
        if (f) cols[base + before + __popc(ballot & ((1u << lane) - 1u))] = c;
        base += total;
        __syncthreads();  // s_warp is rewritten by the next tile
    }
    if (threadIdx.x == 0) *count = base;
}

__global__ void __launch_bounds__(kCompactThreads)
    int8_outlier_compact_kernel(const int* __restrict__ flags, int K, int* __restrict__ cols, int* __restrict__ count) {
    outlier_compact(flags, K, cols, count);
}

// ---------------------------------------------------------------------------------------------------------------
// The grouped (mixture-of-experts) route: each expert's outlier columns are those where one of ITS rows has
// |a| >= threshold, as a Linear8bitLt call on that expert's rows alone finds them.  The row codes and statistics do not
// depend on the expert (int8_vector_quant_kernel gives them); the flags, the column lists and the operands do.
// end_e = min(max(offs[e], end_{e-1}), M), end_{-1} = 0: the grouped GEMMs' clamp of the expert ends, one thread per expert.
constexpr int kEndsThreads = 1024;
static_assert(kMaxExperts <= kEndsThreads, "one thread per expert");
__global__ void __launch_bounds__(kEndsThreads)
    int8_group_ends_kernel(const int* __restrict__ offs, int E, int M, int* __restrict__ ends) {
    __shared__ int s_warp[kEndsThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int v = threadIdx.x < E ? max(offs[threadIdx.x], 0) : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v = max(v, o);
    }
    if (lane == 31) s_warp[warp] = v;
    __syncthreads();
    for (int w = 0; w < warp; ++w) v = max(v, s_warp[w]);
    if (threadIdx.x < E) ends[threadIdx.x] = min(v, M);
}

// the expert of row m < ends[E - 1]: the first e with ends[e] > m
__device__ __forceinline__ int expert_of_row(const int* __restrict__ ends, int E, int m) {
    int lo = 0, hi = E - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(ends + mid) > m) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

// flags[e, c] = 1 where a row of expert e has |A16[m, c]| >= thr (A16: the activations as fp16, as LLM.int8() quantises
// them; the comparison of int8_vector_quant_kernel's flags).  One CTA per row; rows past end_{E-1} flag nothing.
__global__ void __launch_bounds__(256)
    int8_grouped_flags_kernel(const __half* __restrict__ A16, const int* __restrict__ ends, int E, int K, float thr,
                              int* __restrict__ flags) {
    const int m = blockIdx.x;
    if (m >= __ldg(ends + E - 1)) return;
    const __half* a = A16 + (long long)m * K;
    int* f = flags + (long long)expert_of_row(ends, E, m) * K;
    for (int c = threadIdx.x; c < K; c += 256)
        if (fabsf(__half2float(a[c])) >= thr) f[c] = 1;
}

// each expert's flags -> its ascending column list cols[e, :count[e]], one CTA per expert
__global__ void __launch_bounds__(kCompactThreads)
    int8_outlier_compact_grouped_kernel(const int* __restrict__ flags, int K, int* __restrict__ cols,
                                        int* __restrict__ count) {
    const long long off = (long long)blockIdx.x * K;
    outlier_compact(flags + off, K, cols + off, count + blockIdx.x);
}

// The operands of the grouped GEMM's outlier term, one warp per row of [subA rows M | subBT rows E * N]:
//   subA[m, j]  = A[m, cols_e[j]] for the first min(count_e, 64) columns of row m's expert e, zero-padded to 64 (rows
//                 past end_{E-1}: zeros), and CA[m, cols_e[j]] = 0 for all count_e of them when the expert has more than
//                 one row (int8_vectorwise_quant's rows > 1 rule: a single row's outliers are zero codes already);
//   subBT[e * N + n, j] = T((float(CB[e * N + n, cols_e[j]]) * SCB[e * N + n]) * (1/127)) for the first
//                 min(count_e, 64) columns, zero-padded to a multiple of 8 -- the columns the GEMM reads -- and written
//                 only for experts with rows and outliers.
// The grid depends on the shapes only.
constexpr int kOutlierCap = 64;
template <typename T>
__global__ void __launch_bounds__(256)
    int8_grouped_outlier_prep_kernel(const T* __restrict__ A, int8_t* __restrict__ CA, const int8_t* __restrict__ CB,
                                     const float* __restrict__ SCB, const int* __restrict__ ends,
                                     const int* __restrict__ cols, const int* __restrict__ count, int E, int M, int N,
                                     int K, T* __restrict__ subA, T* __restrict__ subBT) {
    const int lane = threadIdx.x & 31;
    const long long rows = (long long)M + (long long)E * N;
    const int m_tail = __ldg(ends + E - 1);
    for (long long r = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; r < rows; r += ((long long)gridDim.x * 256) >> 5) {
        if (r < M) {
            T* sa = subA + r * kOutlierCap;
            if (r >= m_tail) {
                sa[lane] = DT<T>::from_f32(0.f);
                sa[lane + 32] = DT<T>::from_f32(0.f);
                continue;
            }
            const int e = expert_of_row(ends, E, (int)r);
            const int all = __ldg(count + e);
            const int J = min(all, kOutlierCap);
            const int* ce = cols + (long long)e * K;
            const T* a = A + r * K;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = lane + 32 * h;
                sa[j] = j < J ? a[__ldg(ce + j)] : DT<T>::from_f32(0.f);
            }
            const int rows_e = __ldg(ends + e) - (e > 0 ? __ldg(ends + e - 1) : 0);
            if (rows_e > 1)
                for (int j = lane; j < all; j += 32) CA[r * K + __ldg(ce + j)] = 0;
        } else {
            const long long w = r - M;
            const int e = (int)(w / N);
            if (__ldg(ends + e) == (e > 0 ? __ldg(ends + e - 1) : 0)) continue;  // no rows: never read
            const int J = min(__ldg(count + e), kOutlierCap);
            const int jpad = (J + 7) & ~7;
            const int* ce = cols + (long long)e * K;
            const float scb = __ldg(SCB + w);
            for (int j = lane; j < jpad; j += 32) {
                float v = 0.f;
                if (j < J) v = __fmul_rn(__fmul_rn((float)CB[w * K + __ldg(ce + j)], scb), 7.874015718698502e-3f);
                subBT[w * kOutlierCap + j] = DT<T>::from_f32(v);
            }
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
                                                              float threshold, int rows, int cols, int rows_per_cta,
                                                              int vec_ok) {
    const int c0 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 8;  // this lane's first column
    const int r_begin = blockIdx.y * rows_per_cta + (threadIdx.x >> 5);
    const int r_end = min(rows, (blockIdx.y + 1) * rows_per_cta);
    if (c0 >= cols) return;
    float m[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const bool full = vec_ok && c0 + 8 <= cols;
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
                                                             int rows_per_cta, int vec_ok) {
    const int c0 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 8;
    const int r_begin = blockIdx.y * rows_per_cta + (threadIdx.x >> 5);
    const int r_end = min(rows, (blockIdx.y + 1) * rows_per_cta);
    if (c0 >= cols) return;
    const bool full = vec_ok && c0 + 8 <= cols;
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

// ---------------------------------------------------------------------------------------------------------------
// The dequantised int8 weight for the input gradient of LLM.int8(): out[n, k] (row stride ldo) = T(float(CB[n, k]) * s)
// with s = SCB[n] * fp32(1/127), the arithmetic of `CB.to(T).mul_(SCB.unsqueeze(1).mul(1.0 / 127.0))` (an fp32 scale,
// one fp32 product, one rounding to T) in one read of the codes and one write of T.
// blockIdx.y walks rows, blockIdx.x chunks of 16-code vectors within a row.  kVec: the codes and the output are
// 16-byte aligned at the same column of every row (aligned bases, (ldo - cols) % 8 == 0), so a row is a scalar head up
// to the first 16-byte aligned code, 16-code vectors (one 16-byte load, two 16-byte stores) and a scalar tail; the head
// and tail are the first CTA's.  Otherwise every element is scalar.
constexpr int kDqThreads = 256;

template <typename T>
__device__ __forceinline__ void dequant_rows_one(const int8_t* cb, T* o, int k, float s) {
    o[k] = DT<T>::from_f32(__fmul_rn((float)cb[k], s));
}

template <typename T, bool kVec>
__global__ void __launch_bounds__(kDqThreads)
    int8_dequant_rows_kernel(const int8_t* __restrict__ CB, const float* __restrict__ SCB, T* __restrict__ out,
                             long long ldo, int rows, int cols) {
    for (int n = blockIdx.y; n < rows; n += gridDim.y) {
        const int8_t* cb = CB + (long long)n * cols;
        T* o = out + (long long)n * ldo;
        const float s = __fmul_rn(__ldg(SCB + n), 7.874015718698502e-3f);
        if constexpr (kVec) {
            const int head = min((int)((16 - (((long long)n * cols) & 15)) & 15), cols);
            const int nvec = (cols - head) >> 4;
            const int tail0 = head + 16 * nvec;
            const int v = blockIdx.x * kDqThreads + threadIdx.x;
            if (v < nvec) {
                const int k0 = head + 16 * v;
                const uint4 q = ldg_stream_v4(cb + k0);
                const uint32_t w[4] = {q.x, q.y, q.z, q.w};
                uint32_t p[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const uint32_t b = w[i >> 1] >> (16 * (i & 1));
                    p[i] = pack2<T>(__fmul_rn((float)(int8_t)(b & 0xffu), s), __fmul_rn((float)(int8_t)(b >> 8), s));
                }
                *reinterpret_cast<uint4*>(o + k0) = make_uint4(p[0], p[1], p[2], p[3]);
                *reinterpret_cast<uint4*>(o + k0 + 8) = make_uint4(p[4], p[5], p[6], p[7]);
            }
            const int t = threadIdx.x;
            if (blockIdx.x == 0) {
                if (t < head) dequant_rows_one(cb, o, t, s);
                if (t >= 32 && t - 32 < cols - tail0) dequant_rows_one(cb, o, tail0 + t - 32, s);
            }
        } else {
            for (int k = blockIdx.x * kDqThreads + threadIdx.x; k < cols; k += gridDim.x * kDqThreads)
                dequant_rows_one(cb, o, k, s);
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
        int8_outlier_prep_kernel<__half, long long><<<grid, 256, 0, stream>>>(
            (const __half*)A, CB, SCB, cols, nullptr, J, jpad, M, N, K, (__half*)subA, (__half*)subBT, nullptr);
    else
        int8_outlier_prep_kernel<__nv_bfloat16, long long><<<grid, 256, 0, stream>>>(
            (const __nv_bfloat16*)A, CB, SCB, cols, nullptr, J, jpad, M, N, K, (__nv_bfloat16*)subA,
            (__nv_bfloat16*)subBT, nullptr);
    BNB200_CHECK_LAUNCH("int8_outlier_prep");
}

// The capturable route: `count` and `cols` on the device (from launch_int8_outlier_compact), subA[M, cap] and
// subBT[N, cap] of a fixed capacity `cap`, CA zeroed in the outlier columns.
void launch_int8_outlier_prep_dev(const void* A, int8_t* CA, const int8_t* CB, const float* SCB, const int* cols,
                                  const int* count, int cap, int M, int N, int K, int dtype, void* subA, void* subBT,
                                  cudaStream_t stream) {
    if (M + N <= 0) return;
    // sized by the operands; the zeroing of up to M x K codes strides over the same grid
    const long long total = (long long)(M + N) * cap;
    const long long want = (total + 255) / 256;
    const int grid = (int)(want < 132 * 16 ? want : 132 * 16);
    if (dtype == 1)
        int8_outlier_prep_kernel<__half, int><<<grid, 256, 0, stream>>>(
            (const __half*)A, CB, SCB, cols, count, 0, cap, M, N, K, (__half*)subA, (__half*)subBT, CA);
    else
        int8_outlier_prep_kernel<__nv_bfloat16, int><<<grid, 256, 0, stream>>>(
            (const __nv_bfloat16*)A, CB, SCB, cols, count, 0, cap, M, N, K, (__nv_bfloat16*)subA,
            (__nv_bfloat16*)subBT, CA);
    BNB200_CHECK_LAUNCH("int8_outlier_prep_dev");
}

void launch_int8_outlier_compact(const int* col_flags, int K, int* cols, int* count, cudaStream_t stream) {
    int8_outlier_compact_kernel<<<1, kCompactThreads, 0, stream>>>(col_flags, K, cols, count);
    BNB200_CHECK_LAUNCH("int8_outlier_compact");
}

// The per-expert outliers of the grouped int8 GEMM (launch_int8_gemm_grouped), in four launches whose grids depend on
// the shapes only: the clamped ends[E] of offs, flags[E, K] from A16 (the fp16 activations), each expert's column list
// cols[E, K] and count[E], then subA [M, 64], subBT [E * N, 64] and CA's zeroed outlier columns.  A is T[M, K] (dtype
// 1 fp16, 2 bf16).
void launch_int8_grouped_outliers(const void* A, const void* A16, int8_t* CA, const int8_t* CB, const float* SCB,
                                  const int* offs, int E, float threshold, int* ends, int* flags, int* cols, int* count,
                                  void* subA, void* subBT, int M, int N, int K, int dtype, cudaStream_t stream) {
    int8_group_ends_kernel<<<1, kEndsThreads, 0, stream>>>(offs, E, M, ends);
    cudaMemsetAsync(flags, 0, sizeof(int) * (size_t)E * K, stream);
    if (M > 0) int8_grouped_flags_kernel<<<M, 256, 0, stream>>>((const __half*)A16, ends, E, K, threshold, flags);
    int8_outlier_compact_grouped_kernel<<<E, kCompactThreads, 0, stream>>>(flags, K, cols, count);
    const long long warps = (long long)M + (long long)E * N;
    const long long want = (warps + 7) / 8;
    const int grid = (int)(want < 132 * 16 ? want : 132 * 16);
    if (dtype == 1)
        int8_grouped_outlier_prep_kernel<__half><<<grid, 256, 0, stream>>>(
            (const __half*)A, CA, CB, SCB, ends, cols, count, E, M, N, K, (__half*)subA, (__half*)subBT);
    else
        int8_grouped_outlier_prep_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(
            (const __nv_bfloat16*)A, CA, CB, SCB, ends, cols, count, E, M, N, K, (__nv_bfloat16*)subA,
            (__nv_bfloat16*)subBT);
    BNB200_CHECK_LAUNCH("int8_grouped_outliers");
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
    // 16-byte loads of A and 8-byte stores of the codes: whole rows of 8-column groups and aligned bases (a contiguous
    // view may start at any element of its storage)
    const int vec_ok = (cols % 8 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0) &&
                       ((reinterpret_cast<uintptr_t>(out) & 7) == 0);
#define BNB200_COLQ(T)                                                                                                 \
    int8_col_absmax_kernel<T><<<grid, 256, 0, stream>>>((const T*)A, col_stats, threshold, rows, cols, rows_per_cta,   \
                                                        vec_ok);                                                       \
    int8_col_quant_kernel<T><<<grid, 256, 0, stream>>>((const T*)A, col_stats, out, threshold, rows, cols, rows_per_cta, \
                                                       vec_ok)
    if (dtype == 1) {
        BNB200_COLQ(__half);
    } else {
        BNB200_COLQ(__nv_bfloat16);
    }
#undef BNB200_COLQ
    BNB200_CHECK_LAUNCH("int8_col_quant");
    return true;
}

// out[rows, cols] (row stride ldo) = T(CB[n, k] * (SCB[n] * fp32(1/127))); dtype: 1 fp16, 2 bf16 (false: dtype not
// served, nothing launched)
bool launch_int8_dequant_rows(const int8_t* CB, const float* SCB, void* out, int ldo, int rows, int cols, int dtype,
                              cudaStream_t stream) {
    if (dtype != 1 && dtype != 2) return false;
    if (rows <= 0 || cols <= 0) return true;
    const bool vec = ((reinterpret_cast<uintptr_t>(CB) & 15) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0) &&
                     ((ldo - cols) % 8 == 0);
    const int per_row = vec ? cols / 16 : cols;  // threads' work items per row
    const int chunks = (per_row + kDqThreads - 1) / kDqThreads;
    const dim3 grid(chunks > 0 ? chunks : 1, rows < 65535 ? rows : 65535);
#define BNB200_DQR(T)                                                                                                  \
    if (vec)                                                                                                           \
        int8_dequant_rows_kernel<T, true><<<grid, kDqThreads, 0, stream>>>(CB, SCB, (T*)out, ldo, rows, cols);        \
    else                                                                                                               \
        int8_dequant_rows_kernel<T, false><<<grid, kDqThreads, 0, stream>>>(CB, SCB, (T*)out, ldo, rows, cols)
    if (dtype == 1) {
        BNB200_DQR(__half);
    } else {
        BNB200_DQR(__nv_bfloat16);
    }
#undef BNB200_DQR
    BNB200_CHECK_LAUNCH("int8_dequant_rows");
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

namespace {

template <int MODE>
void vector_quant_mode(const void* A, int8_t* out, float* rowStats, int* col_flags, float threshold, int rows, int cols,
                       int dtype, cudaStream_t stream) {
    const bool vec = (cols % 8 == 0) && (cols <= kVqThreads * kVqVecs * 8) &&
                     ((reinterpret_cast<uintptr_t>(A) & 15) == 0) && ((reinterpret_cast<uintptr_t>(out) & 7) == 0);
    float thr_stat = threshold;
    if (dtype == 1) thr_stat = __half2float(__float2half_rn(threshold));
    if (dtype == 2) thr_stat = __bfloat162float(__float2bfloat16_rn(threshold));
#define BNB200_VQ(T)                                                                                                   \
    if (vec)                                                                                                           \
        int8_vector_quant_kernel<T, true, MODE><<<rows, kVqThreads, 0, stream>>>((const T*)A, out, rowStats, col_flags, \
                                                                                 threshold, thr_stat, rows, cols);     \
    else                                                                                                               \
        int8_vector_quant_kernel<T, false, MODE><<<rows, kVqThreads, 0, stream>>>((const T*)A, out, rowStats,          \
                                                                                  col_flags, threshold, thr_stat, rows, \
                                                                                  cols)
    if (dtype == 1) {
        BNB200_VQ(__half);
    } else {
        BNB200_VQ(__nv_bfloat16);
    }
#undef BNB200_VQ
}

} // namespace

// The two halves of launch_int8_vector_quant (same kernel, same rounding): the row statistics and outlier flags of
// A[rows, cols] without codes, and the codes from given statistics (outliers -> 0 when threshold > 0).
void launch_int8_row_stats(const void* A, float* rowStats, int* col_flags, float threshold, int rows, int cols,
                           int dtype, cudaStream_t stream) {
    if (rows <= 0 || cols <= 0) return;
    vector_quant_mode<1>(A, nullptr, rowStats, col_flags, threshold, rows, cols, dtype, stream);
    BNB200_CHECK_LAUNCH("int8_row_stats");
}

void launch_int8_quant_with_stats(const void* A, int8_t* out, const float* rowStats, float threshold, int rows,
                                  int cols, int dtype, cudaStream_t stream) {
    if (rows <= 0 || cols <= 0) return;
    vector_quant_mode<2>(A, out, const_cast<float*>(rowStats), nullptr, threshold, rows, cols, dtype, stream);
    BNB200_CHECK_LAUNCH("int8_quant_with_stats");
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
