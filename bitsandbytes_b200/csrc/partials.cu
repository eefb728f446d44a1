// partials.cu -- the rank-order reduction of a row-sharded 4-bit layer (bitsandbytes_b200/parallel.py).
//
// Every rank r of a row-parallel layer computes P_r[M, N], the fp32 partial product of its K slice
// (cbnb_b200_gemm_4bit_partial), and every rank then holds all of them.  This kernel produces
//
//     out[m, n] = T( (((P_0 + P_1) + P_2) + ... + P_{w-1})[m, n] + bias[n] )
//
// fp32 additions in rank order, the bias added in fp32, one rounding to T: every rank computes the same bits, and
// with one rank the result is the plain GEMM's, T(acc + bias) (bias 0 when absent, as in the GEMM epilogues).
// The kernel reads 4 * w * M * N bytes and writes M * N elements: HBM-bound, so each thread moves 16-byte vectors.
//
// The LLM.int8() layer (reduce_int8_partials_kernel) has exact int32 partials P_r = CA_r . CB_r^T instead: their sum is
// the unsharded GEMM's accumulator whatever the order, and the kernel then applies the GEMM's own per-element epilogue
// (int8_epilogue_value: dequantisation, fp16 rounding, the bf16 bias rule, the outlier term of the fused route), so that
// every rank holds the unsharded layer's output bit for bit.
#include <type_traits>

#include "common.cuh"
#include "int8_epilogue.cuh"

namespace bnb200 {

namespace {

constexpr int kReduceThreads = 256;
constexpr int kMaxParts = 8;  // partial buffers the pointer-list reduction takes: one per rank of a node

template <typename T> __device__ __forceinline__ void store_vec(T* dst, const float (&v)[16 / sizeof(T)]);
template <> __device__ __forceinline__ void store_vec<float>(float* dst, const float (&v)[4]) {
    *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
}
template <> __device__ __forceinline__ void store_vec<__half>(__half* dst, const float (&v)[8]) {
    *reinterpret_cast<uint4*>(dst) = make_uint4(pack2<__half>(v[0], v[1]), pack2<__half>(v[2], v[3]),
                                                pack2<__half>(v[4], v[5]), pack2<__half>(v[6], v[7]));
}
template <> __device__ __forceinline__ void store_vec<__nv_bfloat16>(__nv_bfloat16* dst, const float (&v)[8]) {
    *reinterpret_cast<uint4*>(dst) =
        make_uint4(pack2<__nv_bfloat16>(v[0], v[1]), pack2<__nv_bfloat16>(v[2], v[3]),
                   pack2<__nv_bfloat16>(v[4], v[5]), pack2<__nv_bfloat16>(v[6], v[7]));
}

// The element-wise arithmetic both fp32 reductions share, so that they give the same bits: the first partial taken
// as it is, each further one added in fp32 (round to nearest) in rank order, then the bias added in fp32 and one
// rounding to T.
__device__ __forceinline__ void first4(float* s, const float4 v) {
    s[0] = v.x;
    s[1] = v.y;
    s[2] = v.z;
    s[3] = v.w;
}
__device__ __forceinline__ void add4(float* s, const float4 v) {
    s[0] = __fadd_rn(s[0], v.x);
    s[1] = __fadd_rn(s[1], v.y);
    s[2] = __fadd_rn(s[2], v.z);
    s[3] = __fadd_rn(s[3], v.w);
}
template <typename T, bool VEC, int V>
__device__ __forceinline__ void bias_round_store(float (&s)[V], const T* __restrict__ bias, T* __restrict__ out, int m,
                                                 int n, int ldc) {
#pragma unroll
    for (int j = 0; j < V; ++j) s[j] = __fadd_rn(s[j], bias != nullptr ? DT<T>::to_f32(bias[n + j]) : 0.f);
    T* dst = out + (long long)m * ldc + n;
    if constexpr (VEC) {
        store_vec<T>(dst, s);
    } else {
        dst[0] = DT<T>::from_f32(s[0]);
    }
}

// VEC: V = 16 / sizeof(T) consecutive outputs per thread, 16-byte loads of the partials and one 16-byte store
// (N % V == 0, ldc % V == 0, part_stride % 4 == 0, 16-byte aligned bases); otherwise one element per thread.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kReduceThreads)
    reduce_partials_kernel(const float* __restrict__ parts, int world, long long part_stride, T* __restrict__ out,
                           const T* __restrict__ bias, int M, int N, int ldc) {
    constexpr int V = VEC ? 16 / (int)sizeof(T) : 1;
    const int per_row = N / V;
    const long long total = (long long)M * per_row;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int m = (int)(i / per_row);
        const int n = (int)(i - (long long)m * per_row) * V;
        const float* src = parts + (long long)m * N + n;
        float s[V];
        if constexpr (VEC) {
#pragma unroll
            for (int h = 0; h < V / 4; ++h) first4(s + 4 * h, __ldcs(reinterpret_cast<const float4*>(src) + h));
            for (int r = 1; r < world; ++r) {
#pragma unroll
                for (int h = 0; h < V / 4; ++h)
                    add4(s + 4 * h, __ldcs(reinterpret_cast<const float4*>(src + r * part_stride) + h));
            }
        } else {
            s[0] = src[0];
            for (int r = 1; r < world; ++r) s[0] = __fadd_rn(s[0], src[r * part_stride]);
        }
        bias_round_store<T, VEC>(s, bias, out, m, n, ldc);
    }
}

// The same reduction over partials that live in separate buffers, parts.p[0 .. n_parts) in rank order (on the GPU:
// the peers' symmetric-memory slots, read over NVLink), restricted to the rows [row0, row0 + rows) of the [M, N]
// partials; out row m is partial row row0 + m.  Every load of an element group, one per rank, is issued before the
// first add, so that the remote reads overlap; the adds then run in rank order as above.
struct PartPtrs {
    const float* p[kMaxParts];
};

template <typename T, bool VEC>
__global__ void __launch_bounds__(kReduceThreads)
    reduce_partials_ptrs_kernel(const PartPtrs parts, int n_parts, int row0, T* __restrict__ out,
                                const T* __restrict__ bias, int rows, int N, int ldc) {
    constexpr int V = VEC ? 16 / (int)sizeof(T) : 1;
    const int per_row = N / V;
    const long long total = (long long)rows * per_row;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int m = (int)(i / per_row);
        const int n = (int)(i - (long long)m * per_row) * V;
        const long long off = (long long)(row0 + m) * N + n;
        float s[V];
        if constexpr (VEC) {
            float4 v[kMaxParts][V / 4];
#pragma unroll
            for (int r = 0; r < kMaxParts; ++r) {
                if (r < n_parts) {
#pragma unroll
                    for (int h = 0; h < V / 4; ++h) v[r][h] = __ldcs(reinterpret_cast<const float4*>(parts.p[r] + off) + h);
                }
            }
#pragma unroll
            for (int h = 0; h < V / 4; ++h) first4(s + 4 * h, v[0][h]);
#pragma unroll
            for (int r = 1; r < kMaxParts; ++r) {
                if (r < n_parts) {
#pragma unroll
                    for (int h = 0; h < V / 4; ++h) add4(s + 4 * h, v[r][h]);
                }
            }
        } else {
            float v[kMaxParts];
#pragma unroll
            for (int r = 0; r < kMaxParts; ++r)
                if (r < n_parts) v[r] = __ldcs(parts.p[r] + off);
            s[0] = v[0];
#pragma unroll
            for (int r = 1; r < kMaxParts; ++r)
                if (r < n_parts) s[0] = __fadd_rn(s[0], v[r]);
        }
        bias_round_store<T, VEC>(s, bias, out, m, n, ldc);
    }
}

// The reduction of a row-sharded expert layer (the grouped partials of cbnb_b200_gemm_4bit_grouped_partial): the
// arithmetic of reduce_partials_kernel, with the bias of the expert that owns row m, bias[e(m) * N + n], and zeros in
// the rows past end_{E-1}.  Each CTA first clamps offs into its own table of end rows, end_e = min(max(offs[0..e], 0),
// M) -- the prefix maximum the grouped GEMM computes -- so that nothing is read on the host; a row's expert is then
// the number of end rows <= m, found by binary search.
constexpr int kEndsPer = kMaxExperts / kReduceThreads;
static_assert(kEndsPer * kReduceThreads == kMaxExperts, "each thread clamps kEndsPer experts");

template <typename T, bool VEC>
__global__ void __launch_bounds__(kReduceThreads)
    reduce_partials_grouped_kernel(const float* __restrict__ parts, int world, long long part_stride,
                                   const int* __restrict__ offs, int E, T* __restrict__ out, const T* __restrict__ bias,
                                   int M, int N, int ldc) {
    __shared__ int gend[kMaxExperts];
    __shared__ int wmax[kReduceThreads / 32];
    {
        // thread t clamps experts [t * kEndsPer, (t + 1) * kEndsPer): a running maximum over its own, a warp scan of
        // the maxima by shuffles, then the maxima of the warps before it
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        const int e0 = threadIdx.x * kEndsPer;
        int v[kEndsPer];
        int run = 0;
#pragma unroll
        for (int i = 0; i < kEndsPer; ++i) {
            v[i] = e0 + i < E ? max(__ldg(offs + e0 + i), 0) : 0;
            run = max(run, v[i]);
        }
        int inc = run;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc = max(inc, o);
        }
        if (lane == 31) wmax[warp] = inc;
        __syncthreads();
        int r = __shfl_up_sync(0xffffffffu, inc, 1);
        if (lane == 0) r = 0;
        for (int w = 0; w < warp; ++w) r = max(r, wmax[w]);
#pragma unroll
        for (int i = 0; i < kEndsPer; ++i) {
            r = max(r, v[i]);
            if (e0 + i < E) gend[e0 + i] = min(r, M);
        }
        __syncthreads();
    }
    const int m_tail = gend[E - 1];
    constexpr int V = VEC ? 16 / (int)sizeof(T) : 1;
    const int per_row = N / V;
    const long long total = (long long)M * per_row;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int m = (int)(i / per_row);
        const int n = (int)(i - (long long)m * per_row) * V;
        float s[V];
        const T* b = nullptr;
        if (m >= m_tail) {
#pragma unroll
            for (int j = 0; j < V; ++j) s[j] = 0.f;
        } else {
            // the expert of row m: the first e with end_e > m (there is one, since m < end_{E-1})
            int lo = 0, hi = E - 1;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (gend[mid] > m) hi = mid;
                else lo = mid + 1;
            }
            if (bias != nullptr) b = bias + (long long)lo * N;
            const float* src = parts + (long long)m * N + n;
            if constexpr (VEC) {
#pragma unroll
                for (int h = 0; h < V / 4; ++h) first4(s + 4 * h, __ldcs(reinterpret_cast<const float4*>(src) + h));
                for (int r = 1; r < world; ++r) {
#pragma unroll
                    for (int h = 0; h < V / 4; ++h)
                        add4(s + 4 * h, __ldcs(reinterpret_cast<const float4*>(src + r * part_stride) + h));
                }
            } else {
                s[0] = src[0];
                for (int r = 1; r < world; ++r) s[0] = __fadd_rn(s[0], src[r * part_stride]);
            }
        }
        bias_round_store<T, VEC>(s, b, out, m, n, ldc);
    }
}

template <typename T>
void launch_grouped_typed(const float* parts, int world, long long part_stride, const int* offs, int E, T* out,
                          const T* bias, int M, int N, int ldc, cudaStream_t stream) {
    constexpr int V = 16 / (int)sizeof(T);
    const bool vec = N % V == 0 && ldc % V == 0 && part_stride % 4 == 0 &&
                     (reinterpret_cast<uintptr_t>(parts) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    const long long items = (long long)M * (vec ? N / V : N);
    const long long blocks = (items + kReduceThreads - 1) / kReduceThreads;
    const long long cap = (long long)device_sm_count() * 8;
    const int grid = (int)(blocks < cap ? blocks : cap);
    if (vec)
        reduce_partials_grouped_kernel<T, true><<<grid, kReduceThreads, 0, stream>>>(parts, world, part_stride, offs, E,
                                                                                     out, bias, M, N, ldc);
    else
        reduce_partials_grouped_kernel<T, false><<<grid, kReduceThreads, 0, stream>>>(parts, world, part_stride, offs,
                                                                                      E, out, bias, M, N, ldc);
    BNB200_CHECK_LAUNCH("reduce_partials_grouped");
}

template <typename T>
void launch_typed(const float* parts, int world, long long part_stride, T* out, const T* bias, int M, int N, int ldc,
                  cudaStream_t stream) {
    constexpr int V = 16 / (int)sizeof(T);
    const bool vec = N % V == 0 && ldc % V == 0 && part_stride % 4 == 0 &&
                     (reinterpret_cast<uintptr_t>(parts) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    const long long items = (long long)M * (vec ? N / V : N);
    // a few waves of resident CTAs, each thread looping over the rest
    const long long blocks = (items + kReduceThreads - 1) / kReduceThreads;
    const long long cap = (long long)device_sm_count() * 8;
    const int grid = (int)(blocks < cap ? blocks : cap);
    if (vec)
        reduce_partials_kernel<T, true><<<grid, kReduceThreads, 0, stream>>>(parts, world, part_stride, out, bias, M, N,
                                                                             ldc);
    else
        reduce_partials_kernel<T, false><<<grid, kReduceThreads, 0, stream>>>(parts, world, part_stride, out, bias, M,
                                                                              N, ldc);
    BNB200_CHECK_LAUNCH("reduce_partials");
}

template <typename T>
void launch_ptrs_typed(const PartPtrs& parts, int n_parts, int row0, T* out, const T* bias, int rows, int N, int ldc,
                       cudaStream_t stream) {
    constexpr int V = 16 / (int)sizeof(T);
    bool vec = N % V == 0 && ldc % V == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    for (int r = 0; r < n_parts; ++r) vec = vec && (reinterpret_cast<uintptr_t>(parts.p[r]) & 15) == 0;
    const long long items = (long long)rows * (vec ? N / V : N);
    const long long blocks = (items + kReduceThreads - 1) / kReduceThreads;
    const long long cap = (long long)device_sm_count() * 8;
    const int grid = (int)(blocks < cap ? blocks : cap);
    if (vec)
        reduce_partials_ptrs_kernel<T, true><<<grid, kReduceThreads, 0, stream>>>(parts, n_parts, row0, out, bias, rows,
                                                                                  N, ldc);
    else
        reduce_partials_ptrs_kernel<T, false><<<grid, kReduceThreads, 0, stream>>>(parts, n_parts, row0, out, bias,
                                                                                   rows, N, ldc);
    BNB200_CHECK_LAUNCH("reduce_partials_ptrs");
}

// EPI 1: fp16 out, 2: bf16 out.  VEC: 8 consecutive outputs per thread, two 16-byte loads of each rank's int32 partial
// and one 16-byte store (N % 8 == 0, ldc % 8 == 0, part_stride % 4 == 0, 16-byte aligned bases); otherwise one output
// per thread.  jpad > 0: add the outlier term sum_j subA[m, j] * subBT[n, j] over the jpad (zero-padded) columns, in
// column order, as the GEMM's JMAX instances do.
template <int EPI, bool VEC>
__global__ void __launch_bounds__(kReduceThreads)
    reduce_int8_partials_kernel(const int* __restrict__ parts, int world, long long part_stride,
                                const float* __restrict__ SCA, const float* __restrict__ SCB, const void* __restrict__ bias,
                                const uint4* __restrict__ subA, const uint4* __restrict__ subBT, int jpad,
                                void* __restrict__ out, int M, int N, int ldc) {
    using T = typename std::conditional<EPI == 1, __half, __nv_bfloat16>::type;
    constexpr int V = VEC ? 8 : 1;
    const int per_row = N / V;
    const long long total = (long long)M * per_row;
    const T* b_t = reinterpret_cast<const T*>(bias);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int m = (int)(i / per_row);
        const int n = (int)(i - (long long)m * per_row) * V;
        const int* src = parts + (long long)m * N + n;
        int acc[V];
        if constexpr (VEC) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int4 v = __ldcs(reinterpret_cast<const int4*>(src) + h);
                acc[4 * h] = v.x;
                acc[4 * h + 1] = v.y;
                acc[4 * h + 2] = v.z;
                acc[4 * h + 3] = v.w;
            }
            for (int r = 1; r < world; ++r) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int4 v = __ldcs(reinterpret_cast<const int4*>(src + r * part_stride) + h);
                    acc[4 * h] += v.x;
                    acc[4 * h + 1] += v.y;
                    acc[4 * h + 2] += v.z;
                    acc[4 * h + 3] += v.w;
                }
            }
        } else {
            acc[0] = src[0];
            for (int r = 1; r < world; ++r) acc[0] += src[r * part_stride];
        }
        float ol[V];
#pragma unroll
        for (int u = 0; u < V; ++u) ol[u] = 0.f;
        for (int q = 0; q < jpad / 8; ++q) {
            float a8[8];
            i8_unpack8<EPI>(__ldg(subA + (long long)m * (jpad / 8) + q), a8);
#pragma unroll
            for (int u = 0; u < V; ++u) {
                float b8[8];
                i8_unpack8<EPI>(__ldg(subBT + (long long)(n + u) * (jpad / 8) + q), b8);
#pragma unroll
                for (int x = 0; x < 8; ++x) ol[u] = fmaf(a8[x], b8[x], ol[u]);
            }
        }
        const float sca = __ldg(SCA + m);
        float f[V];
#pragma unroll
        for (int u = 0; u < V; ++u) {
            const float b = b_t != nullptr ? DT<T>::to_f32(b_t[n + u]) : 0.f;
            f[u] = int8_epilogue_value<EPI>(acc[u], sca, __ldg(SCB + n + u), b, b_t != nullptr, jpad > 0, ol[u]);
        }
        T* dst = reinterpret_cast<T*>(out) + (long long)m * ldc + n;
        if constexpr (VEC) {
            store_vec<T>(dst, f);
        } else {
            dst[0] = DT<T>::from_f32(f[0]);
        }
    }
}

} // namespace

bool launch_reduce_int8_partials(const int* parts, int world, long long part_stride, const float* SCA, const float* SCB,
                                 const void* bias, const void* subA, const void* subBT, int jpad, void* out, int M,
                                 int N, int ldc, int dtype, cudaStream_t stream) {
    if (world < 1 || part_stride < 0 || ldc < N || (dtype != 1 && dtype != 2)) return false;
    if (jpad < 0 || jpad > 64 || jpad % 8 != 0) return false;
    if (jpad > 0 && (subA == nullptr || subBT == nullptr || (reinterpret_cast<uintptr_t>(subA) & 15) != 0 ||
                     (reinterpret_cast<uintptr_t>(subBT) & 15) != 0))
        return false;
    if (M <= 0 || N <= 0) return true;
    const bool vec = N % 8 == 0 && ldc % 8 == 0 && part_stride % 4 == 0 &&
                     (reinterpret_cast<uintptr_t>(parts) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    const long long items = (long long)M * (vec ? N / 8 : N);
    const long long blocks = (items + kReduceThreads - 1) / kReduceThreads;
    const long long cap = (long long)device_sm_count() * 8;
    const int grid = (int)(blocks < cap ? blocks : cap);
    const uint4* a = reinterpret_cast<const uint4*>(subA);
    const uint4* bt = reinterpret_cast<const uint4*>(subBT);
#define BNB200_RI8(E, VEC)                                                                                             \
    reduce_int8_partials_kernel<E, VEC><<<grid, kReduceThreads, 0, stream>>>(parts, world, part_stride, SCA, SCB, bias, \
                                                                             a, bt, jpad, out, M, N, ldc)
    if (dtype == 1) {
        if (vec) BNB200_RI8(1, true);
        else BNB200_RI8(1, false);
    } else {
        if (vec) BNB200_RI8(2, true);
        else BNB200_RI8(2, false);
    }
#undef BNB200_RI8
    BNB200_CHECK_LAUNCH("reduce_int8_partials");
    return true;
}

bool launch_reduce_partials(const float* parts, int world, long long part_stride, void* out, const void* bias, int M,
                            int N, int ldc, int dtype, cudaStream_t stream) {
    if (world < 1 || part_stride < 0 || ldc < N) return false;
    if (M <= 0 || N <= 0) return true;
    if (dtype == 0 || dtype == 3)
        launch_typed<float>(parts, world, part_stride, (float*)out, (const float*)bias, M, N, ldc, stream);
    else if (dtype == 1)
        launch_typed<__half>(parts, world, part_stride, (__half*)out, (const __half*)bias, M, N, ldc, stream);
    else if (dtype == 2)
        launch_typed<__nv_bfloat16>(parts, world, part_stride, (__nv_bfloat16*)out, (const __nv_bfloat16*)bias, M, N,
                                    ldc, stream);
    else
        return false;
    return true;
}

bool launch_reduce_partials_grouped(const float* parts, int world, long long part_stride, const int* offs, int E,
                                    void* out, const void* bias, int M, int N, int ldc, int dtype, cudaStream_t stream) {
    if (world < 1 || part_stride < 0 || ldc < N || E < 1 || E > kMaxExperts || offs == nullptr) return false;
    if (M <= 0 || N <= 0) return true;
    if (dtype == 1)
        launch_grouped_typed<__half>(parts, world, part_stride, offs, E, (__half*)out, (const __half*)bias, M, N, ldc,
                                     stream);
    else if (dtype == 2)
        launch_grouped_typed<__nv_bfloat16>(parts, world, part_stride, offs, E, (__nv_bfloat16*)out,
                                            (const __nv_bfloat16*)bias, M, N, ldc, stream);
    else
        return false;
    return true;
}

int max_reduce_parts() { return kMaxParts; }

// The caller (c_api.cu) has checked the arguments: 1 <= n_parts <= kMaxParts, the window inside M, aligned pointers.
bool launch_reduce_partials_ptrs(const float* const* parts, int n_parts, int row0, int rows, void* out,
                                 const void* bias, int N, int ldc, int dtype, cudaStream_t stream) {
    if (dtype < 0 || dtype > 3) return false;
    if (rows <= 0 || N <= 0) return true;
    PartPtrs p{};
    for (int r = 0; r < n_parts; ++r) p.p[r] = parts[r];
    if (dtype == 0 || dtype == 3)
        launch_ptrs_typed<float>(p, n_parts, row0, (float*)out, (const float*)bias, rows, N, ldc, stream);
    else if (dtype == 1)
        launch_ptrs_typed<__half>(p, n_parts, row0, (__half*)out, (const __half*)bias, rows, N, ldc, stream);
    else
        launch_ptrs_typed<__nv_bfloat16>(p, n_parts, row0, (__nv_bfloat16*)out, (const __nv_bfloat16*)bias, rows, N,
                                         ldc, stream);
    return true;
}

} // namespace bnb200
