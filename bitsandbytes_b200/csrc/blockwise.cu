// blockwise.cu -- blockwise quantize / dequantize for sm_90a (HBM-roofline kernels).
//
// Replaces the reference's kQuantizeBlockwise / kQuantizeBlockwiseSmall /
// kDequantizeBlockwise (reference csrc/kernels.cu:269-529, launchers csrc/ops.cu:36-94).
// Same results, different machine mapping:
//   * no CUB block load/store through shared memory: every thread moves 16-byte
//     vectors straight between HBM and registers, lanes of a warp on consecutive
//     vectors (fully coalesced, 512 B per warp instruction);
//   * per-block absmax by warp-shuffle butterflies (sub-warp groups when a quant
//     block is owned by fewer than 32 lanes, one smem hop when it spans warps);
//   * streaming cache hints (ld.global.nc.L1::no_allocate / st.global.L1::no_allocate);
//   * persistent grid sized as a multiple of the SM count.
//
// Numerics (must stay bit-identical to the reference CUDA kernels):
//   absmax  = max |x| (exact);  inv = rcp.approx.ftz(absmax)   [fast-math 1.0f/x]
//   code    = decision procedure on mul.ftz(x, inv)
//   dequant = T( mul.ftz(value(code), absmax) )                 [one rounding]
#include "common.cuh"
#include "decode4.cuh"
#include "q8_search.cuh"

#include <cstdlib>
#include <type_traits>

namespace bnb200 {

// =====================================================================================
// value -> code
// =====================================================================================

// NF4: reference kernels.cu:110-153.  The tree is a binary search with strict '>' over
// the 15 midpoints, i.e. code = #{pivots p : x > p}.  We evaluate it as a 4-level
// branch-free search (SEL on constants), identical result, NaN -> 0.
__device__ __forceinline__ unsigned quantize_nf4(float x) {
    unsigned c;
    if (x > 0.03979014977812767f) {
        if (x > 0.3893125355243683f) {
            if (x > 0.6427869200706482f)
                c = (x > 0.8614784181118011f) ? 15u : 14u;
            else
                c = (x > 0.5016634166240692f) ? 13u : 12u;
        } else {
            if (x > 0.2035212516784668f)
                c = (x > 0.2920137718319893f) ? 11u : 10u;
            else
                c = (x > 0.1202552504837513f) ? 9u : 8u;
        }
    } else {
        if (x > -0.33967943489551544f) {
            if (x > -0.13791173323988914f)
                c = (x > -0.045525018125772476f) ? 7u : 6u;
            else
                c = (x > -0.23460740596055984f) ? 5u : 4u;
        } else {
            if (x > -0.6106329262256622f)
                c = (x > -0.4599952697753906f) ? 3u : 2u;
            else
                c = (x > -0.8480964004993439f) ? 1u : 0u;
        }
    }
    return c;
}

// FP4: reference kernels.cu:64-106.
__device__ __forceinline__ unsigned quantize_fp4(float x) {
    unsigned sign = (x < 0.0f) ? 8u : 0u;
    float a = fabsf(x);
    unsigned c;
    if (a > 0.29166667f) {
        if (a > 0.583333f)
            c = (a > 0.8333333f) ? 3u : 2u;
        else
            c = (a > 0.4166667f) ? 5u : 4u;
    } else {
        if (a > 0.0859375f)
            c = (a > 0.20833333f) ? 7u : 6u;
        else
            c = (a > 0.00260417f) ? 1u : 0u;
    }
    return c + sign;
}

// The same two decision procedures as ONE table look-up + ONE comparison (the fast kernel's form).
// Both procedures are "which interval between consecutive pivots holds x" (NF4: 15 pivots on [-1, 1]; FP4: 7 on
// |x|), and no two pivots are closer than 0.08, so a uniform grid of width 1/16 has at most one pivot per cell:
//     t = int((x + 1) * 16)  [NF4]   /   int(|x| * 16)  [FP4]          (NaN -> 0, where every comparison is false)
//     entry t = { the pivot inside cell t (or +inf), code below it | (code below ^ code above) << 8 }
//     code = below ^ (x > pivot ? (below ^ above) : 0)
// x is a * rcp(absmax) with |a| <= absmax, so |x| <= 1 + 2^-22 and t stays inside the 33- / 17-entry table.
// Equality with the trees above for every such fp32 value (and NaN) is proved exhaustively on the CPU
// (tools/micro/q4_lut_equiv.c); a cell edge is never within rounding distance of a pivot.
constexpr int kQ4LutNF4 = 33, kQ4LutFP4 = 17;

template <int QT> __device__ __forceinline__ void build_q4_lut(float2* lut, int t) {
    constexpr float kPivNF4[15] = {-0.8480964004993439f, -0.6106329262256622f, -0.4599952697753906f,
                                   -0.33967943489551544f, -0.23460740596055984f, -0.13791173323988914f,
                                   -0.045525018125772476f, 0.03979014977812767f, 0.1202552504837513f,
                                   0.2035212516784668f, 0.2920137718319893f, 0.3893125355243683f,
                                   0.5016634166240692f, 0.6427869200706482f, 0.8614784181118011f};
    constexpr float kPivFP4[7] = {0.00260417f, 0.0859375f, 0.20833333f, 0.29166667f, 0.4166667f, 0.583333f, 0.8333333f};
    constexpr unsigned kCodeFP4[8] = {0u, 1u, 6u, 7u, 4u, 5u, 2u, 3u};  // code of the interval below pivot i / above the last
    const float lo = QT == kNF4 ? (float)t * 0.0625f - 1.0f : (float)t * 0.0625f;
    const float hi = lo + 0.0625f;
    int r = 0;  // pivots below the cell
    if (QT == kNF4) {
#pragma unroll
        for (int i = 0; i < 15; ++i) r += kPivNF4[i] < lo ? 1 : 0;
    } else {
#pragma unroll
        for (int i = 0; i < 7; ++i) r += kPivFP4[i] < lo ? 1 : 0;
    }
    float pivot = __int_as_float(0x7f800000);
    unsigned below, above;
    if (QT == kNF4) {
        below = (unsigned)r;
        above = below;
        if (r < 15) {
            float pv = 0.f;
#pragma unroll
            for (int i = 0; i < 15; ++i) pv = i == r ? kPivNF4[i] : pv;
            if (pv < hi) {
                pivot = pv;
                above = below + 1u;
            }
        }
    } else {
        unsigned cb = 0u, ca = 0u;
        float pv = 2.0f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            cb = i == r ? kCodeFP4[i] : cb;
            ca = i == r + 1 ? kCodeFP4[i] : ca;
        }
#pragma unroll
        for (int i = 0; i < 7; ++i) pv = i == r ? kPivFP4[i] : pv;
        below = cb;
        above = cb;
        if (r < 7 && pv < hi) {
            pivot = pv;
            above = ca;
        }
    }
    lut[t] = make_float2(pivot, __uint_as_float(below | ((below ^ above) << 8)));
}

template <int QT> __device__ __forceinline__ unsigned quantize4_lut(const float2* __restrict__ lut, float x) {
    if (QT == kNF4) {
        const float2 e = lut[__float2int_rz(fmaf(x, 16.0f, 16.0f))];
        const unsigned w = __float_as_uint(e.y);
        return (w & 0xffu) ^ ((x > e.x) ? (w >> 8) : 0u);
    } else {
        const float a = fabsf(x);
        const float2 e = lut[__float2int_rz(a * 16.0f)];
        const unsigned w = __float_as_uint(e.y);
        return ((w & 0xffu) ^ ((a > e.x) ? (w >> 8) : 0u)) | ((x < 0.0f) ? 8u : 0u);
    }
}

// 8-bit dynamic map: reference kernels.cu:160-219 (dQuantize<0>).  Same 7-step search
// from pivot 127 and the same midpoint rule; the code book lives in shared memory.
__device__ __forceinline__ unsigned quantize_8bit(const float* __restrict__ scode, float x) {
    int pivot = 127, upper_pivot = 255, lower_pivot = 0;
    float lower = -1.0f, upper = 1.0f;
    float val = scode[pivot];
#pragma unroll
    for (int i = 64; i > 0; i >>= 1) {
        bool gt = x > val;
        lower_pivot = gt ? pivot : lower_pivot;
        lower = gt ? val : lower;
        upper_pivot = gt ? upper_pivot : pivot;
        upper = gt ? upper : val;
        pivot += gt ? i : -i;
        val = scode[pivot];
    }
    if (upper_pivot == 255) upper = scode[255];
    if (lower_pivot == 0) lower = scode[0];
    if (x > val) {
        // (upper + val) * 0.5f : add then mul, both ftz under fast-math; operands are
        // code-book values (|v| <= 1, never denormal sums that matter) -> plain ops.
        float midpoint = mul_ftz(upper + val, 0.5f);
        return (x > midpoint) ? (unsigned)upper_pivot : (unsigned)pivot;
    } else {
        float midpoint = mul_ftz(lower + val, 0.5f);
        return (x < midpoint) ? (unsigned)lower_pivot : (unsigned)pivot;
    }
}

// =====================================================================================
// quantize
// =====================================================================================
//
// Work decomposition: a CTA of 256 threads owns a tile of 256*EPT consecutive
// elements (EPT = 16).  A quant block of BS elements is owned by G = BS/EPT threads
// (G = 2..256, power of two), thread j of the group loading 16-byte vectors
// j, j+G, j+2G, ... of the block, so that every load instruction of a warp covers
// contiguous memory.  VE = elements per 16-byte vector (4 for fp32, 8 for 16-bit).

template <typename T> struct VecIO;

template <> struct VecIO<float> {
    static constexpr int VE = 4;
    __device__ static __forceinline__ void load(const float* p, float (&v)[4]) {
        uint4 r = ldg_stream_v4(p);
        v[0] = __uint_as_float(r.x);
        v[1] = __uint_as_float(r.y);
        v[2] = __uint_as_float(r.z);
        v[3] = __uint_as_float(r.w);
    }
};

template <> struct VecIO<__half> {
    static constexpr int VE = 8;
    __device__ static __forceinline__ void load(const __half* p, float (&v)[8]) {
        uint4 r = ldg_stream_v4(p);
        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
            float2 f = __half22float2(h);
            v[2 * i] = f.x;
            v[2 * i + 1] = f.y;
        }
    }
};

template <> struct VecIO<__nv_bfloat16> {
    static constexpr int VE = 8;
    __device__ static __forceinline__ void load(const __nv_bfloat16* p, float (&v)[8]) {
        uint4 r = ldg_stream_v4(p);
        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            v[2 * i] = __uint_as_float(w[i] << 16);
            v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
        }
    }
};

template <int QT>
__device__ __forceinline__ unsigned quantize_8bit_any(const float* scode, const float2* sfin, const uint32_t* sbr, float x) {
    return QT == kGeneral8bitFast ? quantize_8bit_fast(scode, sfin, sbr, x) : quantize_8bit(scode, x);
}

constexpr int kQThreads = 256;
constexpr int kQEPT = 16; // elements per thread

// Fast path: n is a multiple of the quant block, base pointers 16-byte aligned.
template <typename T, int QT>
__global__ void __launch_bounds__(kQThreads)
    quantize_blockwise_kernel(const float* __restrict__ code, const T* __restrict__ A, float* __restrict__ absmax,
                              uint8_t* __restrict__ out, int log2_bs, long long n_full_tiles_elems, long long n) {
    constexpr int VE = VecIO<T>::VE;
    constexpr int V = kQEPT / VE; // vectors per thread
    __shared__ float scode[256];
    __shared__ float swarp[kQThreads / 32];
    __shared__ float2 sfin[QT == kGeneral8bitFast ? 257 : 1];
    __shared__ uint32_t sbr[QT == kGeneral8bitFast ? kQ8Cells : 1];
    __shared__ float2 q4lut[QT == kNF4 ? kQ4LutNF4 : (QT == kFP4 ? kQ4LutFP4 : 1)];
    constexpr bool k8 = QT == kGeneral8bit || QT == kGeneral8bitFast;
    // the code book's own (cold, 1 KB) fetch is issued first and parked in a register; the look-up tables are built
    // AFTER the first tile's loads are in flight, so neither latency delays the data
    float creg = 0.f;
    if (k8) creg = __ldg(code + threadIdx.x);
    bool tables_ready = false;

    const int bs = 1 << log2_bs;
    const int G = bs / kQEPT;           // threads per quant block (>= 2)
    const int j = threadIdx.x & (G - 1); // index inside the group (G is a power of two)
    const int grp = threadIdx.x / G;     // quant block inside the CTA tile
    constexpr long long kTile = (long long)kQThreads * kQEPT;

    for (long long tile = (long long)blockIdx.x * kTile; tile < n_full_tiles_elems; tile += (long long)gridDim.x * kTile) {
        const long long blk_base = tile + (long long)grp * bs; // first element of this thread's quant block
        float x[V][VE];
#pragma unroll
        for (int v = 0; v < V; ++v) VecIO<T>::load(A + blk_base + (long long)(j + v * G) * VE, x[v]);
        if (!tables_ready) {
            tables_ready = true;
            if (k8) {
                scode[threadIdx.x] = creg;
                __syncthreads();
                if (QT == kGeneral8bitFast) {
                    build_q8_final(scode, sfin);
                    build_q8_bracket(scode, sbr);
                    __syncthreads();
                }
            } else {
                if (threadIdx.x < (QT == kNF4 ? kQ4LutNF4 : kQ4LutFP4)) build_q4_lut<QT>(q4lut, threadIdx.x);
                __syncthreads();
            }
        }

        float m = -3.402823466e+38f;
#pragma unroll
        for (int v = 0; v < V; ++v)
#pragma unroll
            for (int e = 0; e < VE; ++e) m = max_ftz(m, abs_ftz(x[v][e]));

        // reduce over the G threads that own the block
        if (G <= 32) {
            for (int o = G >> 1; o > 0; o >>= 1) m = max_ftz(m, __shfl_xor_sync(0xffffffffu, m, o));
        } else {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = max_ftz(m, __shfl_xor_sync(0xffffffffu, m, o));
            __syncthreads(); // protect swarp from the previous iteration's readers
            if ((threadIdx.x & 31) == 0) swarp[threadIdx.x >> 5] = m;
            __syncthreads();
            const int wpg = G >> 5; // warps per group
            const int w0 = (threadIdx.x >> 5) & ~(wpg - 1);
            float mm = swarp[w0];
            for (int w = 1; w < wpg; ++w) mm = max_ftz(mm, swarp[w0 + w]);
            m = mm;
        }
        if (j == 0) absmax[blk_base >> log2_bs] = m;
        const float inv = rcp_approx_ftz(m);

#pragma unroll
        for (int v = 0; v < V; ++v) {
            const long long e0 = blk_base + (long long)(j + v * G) * VE;
            if (k8) {
                uint32_t w[VE / 4];
#pragma unroll
                for (int q = 0; q < VE / 4; ++q) {
                    uint32_t b0 = quantize_8bit_any<QT>(scode, sfin, sbr, mul_ftz(x[v][4 * q + 0], inv));
                    uint32_t b1 = quantize_8bit_any<QT>(scode, sfin, sbr, mul_ftz(x[v][4 * q + 1], inv));
                    uint32_t b2 = quantize_8bit_any<QT>(scode, sfin, sbr, mul_ftz(x[v][4 * q + 2], inv));
                    uint32_t b3 = quantize_8bit_any<QT>(scode, sfin, sbr, mul_ftz(x[v][4 * q + 3], inv));
                    w[q] = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
                }
                if (VE == 4)
                    stg_stream_u32(out + e0, w[0]);
                else
                    stg_stream_v2(out + e0, make_uint2(w[0], w[VE / 4 - 1]));
            } else {
                uint32_t w = 0;
#pragma unroll
                for (int p = 0; p < VE / 2; ++p) {
                    float x0 = mul_ftz(x[v][2 * p], inv), x1 = mul_ftz(x[v][2 * p + 1], inv);
                    uint32_t hi = quantize4_lut<QT>(q4lut, x0);
                    uint32_t lo = quantize4_lut<QT>(q4lut, x1);
                    w |= ((hi << 4) | lo) << (8 * p);
                }
                if (VE == 4)
                    stg_stream_u16(out + (e0 >> 1), (uint16_t)w);
                else
                    stg_stream_u32(out + (e0 >> 1), w);
            }
        }
    }
}

// Generic path: one warp per quant block, scalar accesses; handles the ragged last
// block, unaligned pointers and block sizes the fast path does not take.  `first_block`
// lets the launcher use it for just the tail.
template <typename T, int QT>
__global__ void __launch_bounds__(256)
    quantize_blockwise_generic_kernel(const float* __restrict__ code, const T* __restrict__ A,
                                      float* __restrict__ absmax, uint8_t* __restrict__ out, int bs,
                                      long long first_block, long long n) {
    __shared__ float scode[256];
    constexpr bool k8 = QT == kGeneral8bit || QT == kGeneral8bitFast;  // the tail always takes the plain walk
    if (k8) {
        scode[threadIdx.x] = code[threadIdx.x];
        __syncthreads();
    }
    const int lane = threadIdx.x & 31;
    const long long nblocks = (n + bs - 1) / bs;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long b = first_block + (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < nblocks;
         b += warps_total) {
        const long long lo = b * bs;
        const long long hi = (lo + bs < n) ? lo + bs : n;
        float m = -3.402823466e+38f;
        for (long long i = lo + lane; i < hi; i += 32) m = max_ftz(m, abs_ftz(DT<T>::to_f32(A[i])));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = max_ftz(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) absmax[b] = m;
        const float inv = rcp_approx_ftz(m);
        if (k8) {
            for (long long i = lo + lane; i < hi; i += 32)
                out[i] = (uint8_t)quantize_8bit(scode, mul_ftz(DT<T>::to_f32(A[i]), inv));
        } else {
            // bytes [lo/2, (hi+1)/2): element past the end reads as 0.0f (reference pads with T(0))
            for (long long i = lo + 2 * lane; i < hi; i += 64) {
                float a0 = DT<T>::to_f32(A[i]);
                float a1 = (i + 1 < hi) ? DT<T>::to_f32(A[i + 1]) : 0.0f;
                float x0 = mul_ftz(a0, inv), x1 = mul_ftz(a1, inv);
                uint32_t q0 = QT == kNF4 ? quantize_nf4(x0) : quantize_fp4(x0);
                uint32_t q1 = QT == kNF4 ? quantize_nf4(x1) : quantize_fp4(x1);
                out[i >> 1] = (uint8_t)((q0 << 4) | q1);
            }
        }
    }
}

template <typename T, int QT>
void launch_quantize_blockwise_impl(const float* code, const T* A, float* absmax, uint8_t* out, int blocksize,
                                    long long n, cudaStream_t stream);

template <typename T, int QT>
void launch_quantize_blockwise(const float* code, const T* A, float* absmax, uint8_t* out, int blocksize, long long n,
                               cudaStream_t stream) {
    if (QT == kGeneral8bit) {
        // default: the bracket-table search (bit-identical, CPU-proven and GPU-tested); BNB_B200_Q8_WALK=1 keeps the
        // reference's 7-step walk for A/B measurements
        static const bool fast = [] {
            const char* e = getenv("BNB_B200_Q8_WALK");
            return !(e != nullptr && e[0] == '1');
        }();
        if (fast) {
            launch_quantize_blockwise_impl<T, kGeneral8bitFast>(code, A, absmax, out, blocksize, n, stream);
            return;
        }
    }
    launch_quantize_blockwise_impl<T, QT>(code, A, absmax, out, blocksize, n, stream);
}

template <typename T, int QT>
void launch_quantize_blockwise_impl(const float* code, const T* A, float* absmax, uint8_t* out, int blocksize,
                                    long long n, cudaStream_t stream) {
    if (n <= 0) return;
    const bool pow2 = blocksize > 0 && (blocksize & (blocksize - 1)) == 0;
    const bool aligned = ((reinterpret_cast<uintptr_t>(A) & 15) == 0) && ((reinterpret_cast<uintptr_t>(out) & 7) == 0);
    constexpr long long kTile = (long long)kQThreads * kQEPT; // 4096 elements
    long long fast_elems = 0;
    if (pow2 && aligned && blocksize >= 2 * kQEPT && blocksize <= kTile) fast_elems = (n / kTile) * kTile;
    const int sms = device_sm_count();
    if (fast_elems > 0) {
        long long tiles = fast_elems / kTile;
        int grid = (int)(tiles < (long long)sms * 8 ? tiles : (long long)sms * 8);
        quantize_blockwise_kernel<T, QT>
            <<<grid, kQThreads, 0, stream>>>(code, A, absmax, out, ilog2_pow2(blocksize), fast_elems, n);
        BNB200_CHECK_LAUNCH("quantize_blockwise");
    }
    if (fast_elems < n) {
        // fast_elems is a multiple of 4096 and (when > 0) blocksize divides 4096.
        long long first_block = fast_elems / blocksize;
        long long nblocks = (n + blocksize - 1) / blocksize - first_block;
        long long want = (nblocks + 7) / 8;
        int grid = (int)(want < (long long)sms * 8 ? want : (long long)sms * 8);
        quantize_blockwise_generic_kernel<T, QT>
            <<<grid, 256, 0, stream>>>(code, A, absmax, out, blocksize, first_block, n);
        BNB200_CHECK_LAUNCH("quantize_blockwise_generic");
    }
}

// =====================================================================================
// dequantize
// =====================================================================================
//
constexpr int kDqThreads = 256;
constexpr int kDqUnroll = 8;

// 8-bit codes (any output type) and 4-bit codes -> fp32.  Every thread produces 16 bytes of output per step
// (8 x 16-bit or 4 x fp32), lanes on consecutive 16-byte slots; kDqUnroll independent steps are in flight per
// thread and the loads of the NEXT round are issued before the current round is decoded (software pipeline),
// the first round before the look-up table is even built -- so the table's own fetch (a cold 1 KB read) overlaps
// the data instead of delaying it.
template <typename T, int QT>
__global__ void __launch_bounds__(kDqThreads)
    dequantize_blockwise_kernel(const float* __restrict__ code, const uint8_t* __restrict__ A,
                                const float* __restrict__ absmax, T* __restrict__ out, int log2_bs,
                                long long n_vec /* number of full 16-byte output vectors */) {
    constexpr int OE = 16 / DT<T>::kBytes; // output elements per vector: 8 or 4
    // 8-bit: the 256-entry code book.  4-bit (fp32 output only): 16 values, one private column per lane
    // (index = code * 32 + lane): conflict-free by construction.
    __shared__ float scode[QT == kGeneral8bit ? 256 : 16 * 32];
    float creg = 0.f;
    if (QT == kGeneral8bit) creg = __ldg(code + threadIdx.x);

    const long long stride = (long long)gridDim.x * kDqThreads * kDqUnroll;
    uint32_t packed[kDqUnroll][2];
    float s[kDqUnroll];
    auto load = [&](long long v0) {
#pragma unroll
        for (int u = 0; u < kDqUnroll; ++u) {
            const long long v = v0 + (long long)u * kDqThreads;
            packed[u][0] = packed[u][1] = 0;
            s[u] = 0.f;
            if (v < n_vec) {
                const long long e0 = v * OE;
                if (QT == kGeneral8bit) {
                    if (OE == 8) {
                        uint2 r = ldg_stream_v2(A + e0);
                        packed[u][0] = r.x;
                        packed[u][1] = r.y;
                    } else {
                        packed[u][0] = ldg_stream_u32(A + e0);
                    }
                } else {
                    if (OE == 8)
                        packed[u][0] = ldg_stream_u32(A + (e0 >> 1));
                    else
                        packed[u][0] = ldg_stream_u16(A + (e0 >> 1));
                }
                s[u] = __ldg(absmax + (e0 >> log2_bs));
            }
        }
    };
    long long v0 = (long long)blockIdx.x * kDqThreads * kDqUnroll + threadIdx.x;
    load(v0);
    if (QT == kGeneral8bit) {
        scode[threadIdx.x] = creg;
    } else {
        const int lane = threadIdx.x & 31;
        if (threadIdx.x < 32) {
#pragma unroll
            for (int c = 0; c < 16; ++c) scode[c * 32 + lane] = code4_value<QT>(c);
        }
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;

    for (; v0 < n_vec; v0 += stride) {
        uint32_t cur[kDqUnroll][2];
        float cs[kDqUnroll];
#pragma unroll
        for (int u = 0; u < kDqUnroll; ++u) {
            cur[u][0] = packed[u][0];
            cur[u][1] = packed[u][1];
            cs[u] = s[u];
        }
        if (v0 + stride < n_vec) load(v0 + stride);
#pragma unroll
        for (int u = 0; u < kDqUnroll; ++u) {
            const long long v = v0 + (long long)u * kDqThreads;
            if (v < n_vec) {
                float f[OE];
                if (QT == kGeneral8bit) {
#pragma unroll
                    for (int e = 0; e < OE; ++e) {
                        uint32_t q = (cur[u][e >> 2] >> (8 * (e & 3))) & 0xffu;
                        f[e] = mul_ftz(scode[q], cs[u]);
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < OE; ++e) {
                        // element 2b sits in the high nibble of byte b
                        uint32_t q = (cur[u][0] >> (8 * (e >> 1) + ((e & 1) ? 0 : 4))) & 0xfu;
                        f[e] = mul_ftz(scode[q * 32 + lane], cs[u]);
                    }
                }
                uint4 o;
                if constexpr (OE == 4) {
                    o = make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                                   __float_as_uint(f[3]));
                } else {
                    o = make_uint4(pack2<T>(f[0], f[1]), pack2<T>(f[2], f[3]), pack2<T>(f[4], f[5]),
                                   pack2<T>(f[6], f[7]));
                }
                stg_stream_v4(out + v * OE, o);
            }
        }
    }
}

// 4-bit -> fp16 / bf16 (the weight path of Linear4bit): register-table decode, no shared-memory look-ups.
//   * a lane owns 64 consecutive elements (32 bytes of codes = two 16-byte loads; one quantisation block at the
//     default block size, half of one / several of them for other block sizes -- always whole tables): it
//     builds the 16-entry table rn_T(value * scale) once (decode4.cuh: 16 FMUL + 8 packed roundings, exactly the
//     reference's one-rounding result) and translates the codes with PRMT only;
//   * the 128 bytes a lane produces go through a per-warp 4 KB staging tile (16-byte chunks XOR-swizzled by the
//     row, so both the lane-major writes and the row-major reads are bank-conflict-free) and leave as fully
//     coalesced 512-byte warp stores;
//   * grid = a multiple of the SM count, several CTAs per SM: each thread has 32 B of codes + its scale in
//     flight, i.e. > 32 KB of reads per SM, which covers the HBM latency-bandwidth product.
constexpr int kD4Warps = 8;

template <typename T, int QT>
__global__ void __launch_bounds__(kD4Warps * 32, 4)
    dequantize4_prmt_kernel(const uint8_t* __restrict__ A, const float* __restrict__ absmax, T* __restrict__ out,
                            int log2_bs, long long n_units /* 64-element units */) {
    __shared__ __align__(128) uint8_t stage[kD4Warps][4096];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool two = log2_bs == 5;
    uint8_t* tile = stage[warp];
    const long long step = (long long)gridDim.x * kD4Warps * 32;
    for (long long u0 = ((long long)blockIdx.x * kD4Warps + warp) * 32; u0 < n_units; u0 += step) {
        const long long u = u0 + lane;
        uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
        float s0 = 0.f, s1 = 0.f;
        if (u < n_units) {
            // default caching: the two halves of a 32-byte sector are fetched by consecutive instructions
            q0 = __ldg(reinterpret_cast<const uint4*>(A + u * 32));
            q1 = __ldg(reinterpret_cast<const uint4*>(A + u * 32 + 16));
            s0 = __ldg(absmax + ((u * 64) >> log2_bs));
            if (two) s1 = __ldg(absmax + ((u * 64 + 32) >> log2_bs));
        }
        uint32_t r[32];
        DecodeTable tab;
        build_table<T, QT>(s0, tab);
        decode_word(q0.x, tab, r + 0);
        decode_word(q0.y, tab, r + 4);
        decode_word(q0.z, tab, r + 8);
        decode_word(q0.w, tab, r + 12);
        if (two) build_table<T, QT>(s1, tab);
        decode_word(q1.x, tab, r + 16);
        decode_word(q1.y, tab, r + 20);
        decode_word(q1.z, tab, r + 24);
        decode_word(q1.w, tab, r + 28);
        uint8_t* row = tile + lane * 128;
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<uint4*>(row + ((j ^ (lane & 7)) << 4)) = make_uint4(r[4 * j], r[4 * j + 1], r[4 * j + 2], r[4 * j + 3]);
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int rr = 4 * k + (lane >> 3), q = lane & 7;  // 16-byte chunk 32 k + lane of the warp's 4 KB
            const uint4 v = *reinterpret_cast<const uint4*>(tile + rr * 128 + ((q ^ (rr & 7)) << 4));
            if (u0 + rr < n_units) stg_stream_v4(out + (u0 + rr) * 64 + q * 8, v);
        }
        __syncwarp();
    }
}

// Generic path: one element per thread; tail / unaligned / tiny or non-power-of-two blocks.
template <typename T, int QT>
__global__ void __launch_bounds__(256)
    dequantize_blockwise_generic_kernel(const float* __restrict__ code, const uint8_t* __restrict__ A,
                                        const float* __restrict__ absmax, T* __restrict__ out, int bs,
                                        long long first, long long n) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = first + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float s = absmax[i / bs];
        float val;
        if (QT == kGeneral8bit) {
            val = code[A[i]];
        } else {
            uint8_t byte = A[i >> 1];
            val = code4_value<QT>((i & 1) ? (byte & 0x0Fu) : (byte >> 4));
        }
        out[i] = DT<T>::from_f32(mul_ftz(val, s));
    }
}

template <typename T, int QT>
void launch_dequantize_blockwise(const float* code, const uint8_t* A, const float* absmax, T* out, int blocksize,
                                 long long n, cudaStream_t stream) {
    if (n <= 0) return;
    constexpr int OE = 16 / DT<T>::kBytes;
    const bool pow2 = blocksize > 0 && (blocksize & (blocksize - 1)) == 0;
    const bool aligned = ((reinterpret_cast<uintptr_t>(out) & 15) == 0) && ((reinterpret_cast<uintptr_t>(A) & 7) == 0);
    long long n_vec = 0;
    if (pow2 && aligned && blocksize >= OE) n_vec = n / OE;
    const int sms = device_sm_count();
    if constexpr (QT != kGeneral8bit && !std::is_same<T, float>::value) {
        // 4-bit -> 16-bit: the register-table kernel on the whole 64-element units, the generic kernel on the tail
        const bool a16 = (reinterpret_cast<uintptr_t>(A) & 15) == 0;
        if (pow2 && aligned && a16 && blocksize >= 32 && n >= 64) {
            const long long n_units = n / 64;
            const long long want = (n_units + kD4Warps * 32 - 1) / (kD4Warps * 32);
            const int grid = (int)(want < (long long)sms * 4 ? want : (long long)sms * 4);  // 4 resident CTAs per SM
            dequantize4_prmt_kernel<T, QT><<<grid, kD4Warps * 32, 0, stream>>>(A, absmax, out, ilog2_pow2(blocksize), n_units);
            BNB200_CHECK_LAUNCH("dequantize4_prmt");
            n_vec = 0;
            const long long first4 = n_units * 64;
            if (first4 < n) {
                dequantize_blockwise_generic_kernel<T, QT><<<1, 256, 0, stream>>>(code, A, absmax, out, blocksize, first4, n);
                BNB200_CHECK_LAUNCH("dequantize_blockwise_generic");
            }
            return;
        }
    }
    if (n_vec > 0) {
        long long per_cta = (long long)kDqThreads * kDqUnroll;
        long long want = (n_vec + per_cta - 1) / per_cta;
        int grid = (int)(want < (long long)sms * 8 ? want : (long long)sms * 8);
        dequantize_blockwise_kernel<T, QT>
            <<<grid, kDqThreads, 0, stream>>>(code, A, absmax, out, ilog2_pow2(blocksize), n_vec);
        BNB200_CHECK_LAUNCH("dequantize_blockwise");
    }
    const long long first = n_vec * OE;
    if (first < n) {
        long long rem = n - first;
        long long want = (rem + 255) / 256;
        int grid = (int)(want < (long long)sms * 8 ? want : (long long)sms * 8);
        dequantize_blockwise_generic_kernel<T, QT><<<grid, 256, 0, stream>>>(code, A, absmax, out, blocksize, first, n);
        BNB200_CHECK_LAUNCH("dequantize_blockwise_generic");
    }
}

#define INSTANTIATE(T)                                                                                                 \
    template void launch_quantize_blockwise<T, kGeneral8bit>(const float*, const T*, float*, uint8_t*, int, long long, \
                                                             cudaStream_t);                                            \
    template void launch_quantize_blockwise<T, kFP4>(const float*, const T*, float*, uint8_t*, int, long long,         \
                                                     cudaStream_t);                                                    \
    template void launch_quantize_blockwise<T, kNF4>(const float*, const T*, float*, uint8_t*, int, long long,         \
                                                     cudaStream_t);                                                    \
    template void launch_dequantize_blockwise<T, kGeneral8bit>(const float*, const uint8_t*, const float*, T*, int,    \
                                                               long long, cudaStream_t);                               \
    template void launch_dequantize_blockwise<T, kFP4>(const float*, const uint8_t*, const float*, T*, int, long long, \
                                                       cudaStream_t);                                                  \
    template void launch_dequantize_blockwise<T, kNF4>(const float*, const uint8_t*, const float*, T*, int, long long, \
                                                       cudaStream_t);

INSTANTIATE(float)
INSTANTIATE(__half)
INSTANTIATE(__nv_bfloat16)

} // namespace bnb200
