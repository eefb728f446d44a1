// gemv4_simt.cu -- fused 4-bit dequant GEMV / skinny GEMM on CUDA cores (sm_90a).
//
// Replaces the reference's gemm_4bit_simt (reference csrc/gemm_4bit_simt.cu:109-480) and the
// legacy kgemm_4bit_inference_naive (reference csrc/kernels.cu:1452-1567).  Two jobs:
//   (1) fp32 activations (the tensor cores have no exact fp32 mode) and shapes the
//       tensor-core kernel does not take (K % 64 != 0, unaligned pointers);
//   (2) a simple always-correct reference for the tensor-core path in tests.
//
// One warp per output feature n; the 32 lanes split K in 8-element chunks (4 packed bytes,
// one coalesced 128-byte read per warp per step), kUnroll steps in flight.  Up to MB = 4
// tokens are accumulated per pass (blockIdx.y walks M in chunks of MB; beyond 65535 chunks, the
// gridDim.y limit, the launcher covers M in several launches).
//
// Numerics are those of the tensor-core path and of dequantize + matmul, not of the
// reference SIMT kernel (which additionally rounds every product to T,
// gemm_4bit_simt.cu:353,452-453):  W_T = rn_T(value * scale), fp32 fma accumulation, bias
// added in fp32, one rounding to T.  For T = fp32 there is no weight rounding.
#include "common.cuh"
#include "decode4.cuh"

#include <type_traits>

namespace bnb200 {

namespace {

constexpr int kWarpsPerCta = 8;
constexpr int kMB = 4;
constexpr int kUnroll = 4;

template <typename T> __device__ __forceinline__ float round_through(float v);
template <> __device__ __forceinline__ float round_through<float>(float v) { return v; }
template <> __device__ __forceinline__ float round_through<__half>(float v) {
    return __half2float(__float2half_rn(v));
}
template <> __device__ __forceinline__ float round_through<__nv_bfloat16>(float v) {
    return __bfloat162float(__float2bfloat16_rn(v));
}

// 8 consecutive activations -> fp32
template <typename T> __device__ __forceinline__ void load_a8(const T* p, float (&a)[8]);
template <> __device__ __forceinline__ void load_a8<float>(const float* p, float (&a)[8]) {
    const float4 x = __ldg(reinterpret_cast<const float4*>(p));
    const float4 y = __ldg(reinterpret_cast<const float4*>(p) + 1);
    a[0] = x.x; a[1] = x.y; a[2] = x.z; a[3] = x.w;
    a[4] = y.x; a[5] = y.y; a[6] = y.z; a[7] = y.w;
}
template <> __device__ __forceinline__ void load_a8<__half>(const __half* p, float (&a)[8]) {
    const uint4 r = __ldg(reinterpret_cast<const uint4*>(p));
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        a[2 * i] = f.x;
        a[2 * i + 1] = f.y;
    }
}
template <> __device__ __forceinline__ void load_a8<__nv_bfloat16>(const __nv_bfloat16* p, float (&a)[8]) {
    const uint4 r = __ldg(reinterpret_cast<const uint4*>(p));
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        a[2 * i] = __uint_as_float(w[i] << 16);
        a[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
}

struct Scale {
    const float* absmax;
    const uint8_t* absmax_8bit;
    const float* absmax_code;
    float offset;
    __device__ __forceinline__ float at(long long idx) const {
        if (absmax_8bit != nullptr) {
            const float c = __ldg(absmax_code + __ldg(absmax_8bit + idx));
            return __fadd_rn(mul_ftz(c, __ldg(absmax + (idx >> 8))), offset);
        }
        return __ldg(absmax + idx);
    }
};

// `lut` = 16 fp32 code values (NF4 / FP4 table, or the caller's `datatype` array for the
// legacy gemv entry point).  VEC, the vector body: K % 8 == 0, blocksize % 8 == 0, 16-byte aligned A rows and
// 4-byte aligned B rows; otherwise the scalar body.  A CTA serves up to MB tokens from m_first + blockIdx.y * MB.
// PART (here and in gemv4_fast_kernel): the partial instance, fp32 sums to the destinations of `out` (store_partial:
// every one, or each row to its own), no bias.
template <typename T, bool PART, bool VEC>
__device__ __forceinline__ void
    gemv4_simt_body(const T* __restrict__ A, const uint8_t* __restrict__ B, Scale sc,
                      const float* __restrict__ lut16_gmem, int quant_type, typename OutArg<T, PART>::type out,
                      const T* __restrict__ bias, int M, int N, int K, int ldc, int blocksize, int m_first) {
    // power-of-two block sizes (all the API allows) index by shift; anything else divides
    const int log2_bs = ((blocksize & (blocksize - 1)) == 0) ? (31 - __clz(blocksize)) : -1;
    __shared__ float2 lut2[256];
    __shared__ float lut16[16];
    if (threadIdx.x < 16) {
        float v;
        if (lut16_gmem != nullptr)
            v = lut16_gmem[threadIdx.x];
        else
            v = quant_type == kNF4 ? nf4_value(threadIdx.x) : fp4_value(threadIdx.x);
        lut16[threadIdx.x] = v;
    }
    __syncthreads();
    lut2[threadIdx.x] = make_float2(lut16[threadIdx.x >> 4], lut16[threadIdx.x & 15]);
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    const int m_base = m_first + blockIdx.y * kMB;
    if (n >= N) return;
    const int mcount = (M - m_base < kMB) ? (M - m_base) : kMB;

    float acc[kMB];
#pragma unroll
    for (int i = 0; i < kMB; ++i) acc[i] = 0.f;

    const long long e_row = (long long)n * K;  // flat element index of W[n, 0]

    if constexpr (VEC) {
        const uint8_t* brow = B + (e_row >> 1);
        const int chunks = K >> 3;  // 8-element chunks
        for (int c0 = lane; c0 < chunks; c0 += 32 * kUnroll) {
            uint32_t q[kUnroll];
            float s[kUnroll];
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                const int c = c0 + 32 * u;
                q[u] = 0x77777777u;
                s[u] = 0.f;
                if (c < chunks) {
                    q[u] = ldg_stream_u32(brow + 4 * c);
                    s[u] = sc.at(log2_bs >= 0 ? ((e_row + 8ll * c) >> log2_bs) : ((e_row + 8ll * c) / blocksize));
                }
            }
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                const int c = c0 + 32 * u;
                if (c < chunks) {
                    float w[8];
#pragma unroll
                    for (int b = 0; b < 4; ++b) {
                        const float2 v = lut2[(q[u] >> (8 * b)) & 0xffu];
                        w[2 * b] = round_through<T>(mul_ftz(v.x, s[u]));
                        w[2 * b + 1] = round_through<T>(mul_ftz(v.y, s[u]));
                    }
#pragma unroll
                    for (int i = 0; i < kMB; ++i) {
                        if (i < mcount) {
                            float a[8];
                            load_a8<T>(A + (long long)(m_base + i) * K + 8 * c, a);
#pragma unroll
                            for (int t = 0; t < 8; ++t) acc[i] = fmaf(a[t], w[t], acc[i]);
                        }
                    }
                }
            }
        }
    } else {
        // scalar path: any K, any alignment, any blocksize
        for (int k = lane; k < K; k += 32) {
            const long long e = e_row + k;
            const uint8_t byte = B[e >> 1];
            const unsigned qv = (e & 1) ? (byte & 0x0Fu) : (byte >> 4);
            const float w = round_through<T>(mul_ftz(lut16[qv], sc.at(log2_bs >= 0 ? (e >> log2_bs) : (e / blocksize))));
#pragma unroll
            for (int i = 0; i < kMB; ++i)
                if (i < mcount) acc[i] = fmaf(DT<T>::to_f32(A[(long long)(m_base + i) * K + k]), w, acc[i]);
        }
    }

#pragma unroll
    for (int i = 0; i < kMB; ++i) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
    }
    if (lane == 0) {
        if constexpr (PART) {
#pragma unroll
            for (int i = 0; i < kMB; ++i)
                if (i < mcount) store_partial(out, m_base + i, n, ldc, acc[i]);
        } else {
            const float b = bias != nullptr ? DT<T>::to_f32(bias[n]) : 0.f;
#pragma unroll
            for (int i = 0; i < kMB; ++i)
                if (i < mcount) out[(long long)(m_base + i) * ldc + n] = DT<T>::from_f32(acc[i] + b);
        }
    }
}

// ---------------------------------------------------------------------------------------
// Decode-time GEMV (M <= 8, 16-bit activations): HBM-bound streaming of the packed weight.
//
// One warp per output feature.  Each lane owns 32 consecutive k (one 16-byte load of codes,
// one scale when blocksize >= 32); a warp covers 1024 k per step and issues the loads of
// kSteps steps before touching any of them, so ~2 KB per warp (>= 50 KB per SM) is in flight.
// Codes are expanded with the same register-resident PRMT table as the tensor-core kernel
// (bit-identical weights), widened to fp32 and accumulated with FFMA; activations come
// through L1 (they are M x K x 2 bytes, re-read by every warp).
// ---------------------------------------------------------------------------------------
constexpr int kFastSteps = 4;

template <typename T> __device__ __forceinline__ void widen2(uint32_t pair, float& lo, float& hi);
template <> __device__ __forceinline__ void widen2<__nv_bfloat16>(uint32_t pair, float& lo, float& hi) {
    lo = __uint_as_float(pair << 16);
    hi = __uint_as_float(pair & 0xffff0000u);
}
template <> __device__ __forceinline__ void widen2<__half>(uint32_t pair, float& lo, float& hi) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&pair));
    lo = f.x;
    hi = f.y;
}

template <typename T, int QT, int MB, bool PART>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
    gemv4_fast_kernel(const T* __restrict__ A, const uint8_t* __restrict__ B, const float* absmax,
                      const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset,
                      typename OutArg<T, PART>::type out, const T* __restrict__ bias, int M, int N, int K, int ldc,
                      int log2_bs) {
    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    if (n >= N) return;
    ScaleSrc sc{absmax, absmax_8bit, absmax_code,
                (absmax_8bit != nullptr && absmax_offset != nullptr) ? __ldg(absmax_offset) : 0.f};
    // 32 codes per lane never straddle a quantisation block (blocksize >= 32, K % 32 == 0)
    const long long e_row = (long long)n * K;
    const uint8_t* brow = B + (e_row >> 1);

    float acc[MB];
#pragma unroll
    for (int i = 0; i < MB; ++i) acc[i] = 0.f;

    for (int k_base = 0; k_base < K; k_base += 1024 * kFastSteps) {
        uint4 q[kFastSteps];
        float s[kFastSteps];
#pragma unroll
        for (int u = 0; u < kFastSteps; ++u) {
            const int k0 = k_base + u * 1024 + lane * 32;
            q[u] = make_uint4(0, 0, 0, 0);
            s[u] = 0.f;
            if (k0 < K) {
                q[u] = ldg_stream_v4(brow + (k0 >> 1));
                s[u] = sc.load((e_row + k0) >> log2_bs);
            }
        }
#pragma unroll
        for (int u = 0; u < kFastSteps; ++u) {
            const int k0 = k_base + u * 1024 + lane * 32;
            if (k0 < K) {
                uint32_t r[16];
                DecodeTable tab;
                build_table<T, QT>(s[u], tab);
                decode_word(q[u].x, tab, r + 0);
                decode_word(q[u].y, tab, r + 4);
                decode_word(q[u].z, tab, r + 8);
                decode_word(q[u].w, tab, r + 12);
                float w[32];
#pragma unroll
                for (int j = 0; j < 16; ++j) widen2<T>(r[j], w[2 * j], w[2 * j + 1]);
#pragma unroll
                for (int i = 0; i < MB; ++i) {
                    if (i < M) {
                        const uint4* ap = reinterpret_cast<const uint4*>(A + (long long)i * K + k0);
#pragma unroll
                        for (int v = 0; v < 4; ++v) {
                            const uint4 av = __ldg(ap + v);
                            const uint32_t aw[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
                            for (int t = 0; t < 4; ++t) {
                                float a0, a1;
                                widen2<T>(aw[t], a0, a1);
                                acc[i] = fmaf(a0, w[8 * v + 2 * t], acc[i]);
                                acc[i] = fmaf(a1, w[8 * v + 2 * t + 1], acc[i]);
                            }
                        }
                    }
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < MB; ++i) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
    }
    if (lane == 0) {
        if constexpr (PART) {
#pragma unroll
            for (int i = 0; i < MB; ++i)
                if (i < M) store_partial(out, i, n, ldc, acc[i]);
        } else {
            const float b = bias != nullptr ? DT<T>::to_f32(bias[n]) : 0.f;
#pragma unroll
            for (int i = 0; i < MB; ++i)
                if (i < M) out[(long long)i * ldc + n] = DT<T>::from_f32(acc[i] + b);
        }
    }
}

template <typename T, bool PART, bool VEC>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
    gemv4_simt_kernel(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                      const float* absmax_code, const float* absmax_offset, const float* lut16, int quant_type,
                      typename OutArg<T, PART>::type out, const T* bias, int M, int N, int K, int ldc, int blocksize,
                      int m_first) {
    // the offset is fetched on the device: no host sync on the launch path
    Scale sc{absmax, absmax_8bit, absmax_code,
             (absmax_8bit != nullptr && absmax_offset != nullptr) ? __ldg(absmax_offset) : 0.f};
    gemv4_simt_body<T, PART, VEC>(A, B, sc, lut16, quant_type, out, bias, M, N, K, ldc, blocksize, m_first);
}

} // namespace

template <typename T, bool PART>
void launch_gemv4_simt(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                       const float* absmax_code, const float* absmax_offset, const float* lut16, int quant_type,
                       typename OutArg<T, PART>::type out, const T* bias, int M, int N, int K, int ldc, int blocksize,
                       cudaStream_t stream) {
    if (M <= 0 || N <= 0) return;
    if constexpr (!std::is_same<T, float>::value) {
        const bool pow2 = blocksize >= 32 && (blocksize & (blocksize - 1)) == 0;
        const bool fast_ok = lut16 == nullptr && M <= 8 && (K % 32 == 0) && pow2 &&
                             ((reinterpret_cast<uintptr_t>(A) & 15) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0) &&
                             (quant_type == kNF4 || quant_type == kFP4);
        if (fast_ok) {
            const dim3 g((N + kWarpsPerCta - 1) / kWarpsPerCta);
            const int l2 = ilog2_pow2(blocksize);
#define BNB200_FAST(QT, MBV)                                                                                           \
    gemv4_fast_kernel<T, QT, MBV, PART><<<g, kWarpsPerCta * 32, 0, stream>>>(A, B, absmax, absmax_8bit, absmax_code,   \
                                                                             absmax_offset, out, bias, M, N, K, ldc, l2)
            if (quant_type == kNF4) {
                if (M == 1) BNB200_FAST(kNF4, 1);
                else if (M == 2) BNB200_FAST(kNF4, 2);
                else if (M <= 4) BNB200_FAST(kNF4, 4);
                else BNB200_FAST(kNF4, 8);
            } else {
                if (M == 1) BNB200_FAST(kFP4, 1);
                else if (M == 2) BNB200_FAST(kFP4, 2);
                else if (M <= 4) BNB200_FAST(kFP4, 4);
                else BNB200_FAST(kFP4, 8);
            }
#undef BNB200_FAST
            BNB200_CHECK_LAUNCH("gemv4_fast");
            return;
        }
    }
    const bool vec_ok = (K % 8 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0) &&
                        ((reinterpret_cast<uintptr_t>(B) & 3) == 0) && (blocksize % 8 == 0);
    // gridDim.y is at most 65535: from 262 141 tokens on, M is covered in launches of 65535 groups of kMB tokens,
    // each told its first token.  (A loop over the groups inside the kernel instead takes the fp32 vector body from
    // 64 to 170 registers, ptxas -v.)
    constexpr int kMaxGroups = 65535;
    const int m_groups = (M - 1) / kMB + 1;
    for (int g0 = 0; g0 < m_groups; g0 += kMaxGroups) {
        const dim3 grid((N + kWarpsPerCta - 1) / kWarpsPerCta, m_groups - g0 < kMaxGroups ? m_groups - g0 : kMaxGroups);
        if (vec_ok)
            gemv4_simt_kernel<T, PART, true><<<grid, kWarpsPerCta * 32, 0, stream>>>(
                A, B, absmax, absmax_8bit, absmax_code, absmax_offset, lut16, quant_type, out, bias, M, N, K, ldc,
                blocksize, g0 * kMB);
        else
            gemv4_simt_kernel<T, PART, false><<<grid, kWarpsPerCta * 32, 0, stream>>>(
                A, B, absmax, absmax_8bit, absmax_code, absmax_offset, lut16, quant_type, out, bias, M, N, K, ldc,
                blocksize, g0 * kMB);
        BNB200_CHECK_LAUNCH("gemv4_simt");
    }
}

#define INST(T)                                                                                                        \
    template void launch_gemv4_simt<T, false>(const T*, const uint8_t*, const float*, const uint8_t*, const float*,    \
                                              const float*, const float*, int, T*, const T*, int, int, int, int, int,  \
                                              cudaStream_t);                                                           \
    template void launch_gemv4_simt<T, true>(const T*, const uint8_t*, const float*, const uint8_t*, const float*,     \
                                             const float*, const float*, int, OutList<float>, const T*, int, int, int, \
                                             int, int, cudaStream_t);
INST(float)
INST(__half)
INST(__nv_bfloat16)

} // namespace bnb200
