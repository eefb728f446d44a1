// gemv4_mma.cu -- decode-time 4-bit GEMV / skinny GEMM (M <= 16 tokens) for sm_90a.
//
// The regime the reference serves with gemm_4bit_simt (reference csrc/gemm_4bit_simt.cu:109-480,
// dispatch bitsandbytes/backends/cuda/ops.py:583-623): one to a few tokens against the whole packed
// weight.  The roofline is the HBM stream of the codes (N*K/2 bytes); what actually limits a
// CUDA-core kernel is the instruction count per weight (decode + widen + FFMA).  Here the multiply-
// accumulate goes to the tensor cores through the warp-level mma.sync.m16n8k16 (the wgmma kernel's
// smallest token tile, 16, would be half padding at M = 8), so the CUDA cores only decode:
//
//   * a CTA owns 16 output features (the MMA's M); its 4 or 8 warps split K in 256-wide chunks and
//     meet in shared memory at the end;
//   * lane (g = lane / 4, t = lane % 4) owns k in [64 t, 64 t + 64) of the chunk for rows g and
//     g + 8: two 16-byte code loads per row (a warp reads 16 rows x 128 contiguous bytes), one
//     quantisation block per row, so one register table (decode4.cuh) per 64 weights;
//   * the sum over k does not care about order, so the four codes a lane feeds to one MMA are four
//     CONSECUTIVE k of its own range (k-slots 2t, 2t+1, 2t+8, 2t+9 of the instruction), and the
//     activation fragment is loaded from the same addresses: no shuffles, no shared-memory staging;
//   * tokens are the MMA's N (8 per instruction); columns beyond M are zero fragments.
//
// Numerics: W_T = rn_T(value * scale) exactly as everywhere else (decode4.cuh), products exact,
// fp32 accumulation in the tensor core, bias added in fp32, one rounding to T.
#include "common.cuh"
#include "decode4.cuh"

#include <cstdlib>

namespace bnb200 {

namespace {

constexpr int kGRows = 16;    // output features per CTA
constexpr int kGChunk = 256;  // k per warp iteration

template <typename T> struct WarpMma;
template <> struct WarpMma<__nv_bfloat16> {
    static __device__ __forceinline__ void run(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    }
};
template <> struct WarpMma<__half> {
    static __device__ __forceinline__ void run(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
    }
};

// ---------------------------------------------------------------- warp-private cp.async ring
// Decode-time shapes are latency problems: 8-30 MB must be IN FLIGHT almost at once (Little's law: ~50 KB per SM
// at HBM latency), but a register prefetch of one chunk per warp (2 KB) holds 32 KB per SM.  Each warp therefore
// owns a ring of kRing stages in shared memory, filled with cp.async (16 bytes per lane and row half, 4 bytes per
// scale): a lane only ever reads back the bytes it copied itself, so `cp.async.wait_group` is all the
// synchronisation there is -- no barrier, no __syncwarp.  ncu (profiles/r02_decode_regime.md) showed the kernel short of
// WARPS, not of bytes in flight or issue slots (20 % of the warp slots, ALU pipe 53 %, issue 31 %): so the register
// budget is 64 (32 resident warps per SM: decode and MMA go word by word instead of 32 codes at a time) and the ring
// is 2 deep (32 warps x 1 stage x 2 KB = 64 KB in flight per SM while the other stage is decoded).
constexpr int kRing = 2;
constexpr int kRingStageBytes = 4 * 512 + 4 * 128;  // 4 code parts [32 lanes x 16 B] + 4 scale parts [32 lanes x 4 B]

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ uint4 lds_v4(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ float lds_f1(uint32_t a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
    return v;
}

// W = warps per CTA (they split K in 256-wide chunks and meet in shared memory at the end).  Activations come
// through L1 (every CTA on an SM reads the same M x K slice).  Measured and dropped: staging the activations with
// cp.async (slower, it bypasses L1), 3 or 4 CTAs per SM through a register cap, a byte-indexed shared-memory decode
// table (profiles/r02_decode_regime.md).
// NT = groups of 8 tokens (1: M <= 8, 2: M <= 16): the decoded weight fragments feed NT MMAs each.
// PART: the partial instance (fp32 sums to the destinations of `out` by store_partial, no bias, no rounding).
template <typename T, int QT, int W, int NT, bool PART>
__global__ void __launch_bounds__(W * 32, 32 / W)
    gemv4_mma_kernel(const T* __restrict__ A, const uint8_t* __restrict__ B, const float* absmax,
                     const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset,
                     typename OutArg<T, PART>::type out, const T* __restrict__ bias, int M, int N, int K, int ldc,
                     int log2_bs) {
    __shared__ float red[W][kGRows * 8 * NT];
    extern __shared__ __align__(16) uint8_t ring_smem[];
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int g = lane >> 2;
    const int t = lane & 3;
    const int n0 = blockIdx.x * kGRows;
    const bool nested = absmax_8bit != nullptr;
    ScaleSrc sc{absmax, absmax_8bit, absmax_code, (nested && absmax_offset != nullptr) ? __ldg(absmax_offset) : 0.f};
    const bool two_scales = log2_bs == 5;  // blocksize 32: two quantisation blocks per 64 codes
    bool tok_ok[NT];                       // this lane's tokens (MMA column g of token group u)
    const T* arow[NT];
#pragma unroll
    for (int u = 0; u < NT; ++u) {
        tok_ok[u] = g + 8 * u < M;
        arow[u] = A + (long long)(tok_ok[u] ? g + 8 * u : 0) * K;
    }

    // this lane's two weight rows (rows past N contribute zero fragments)
    long long e_row[2];
    bool row_ok[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int n = n0 + g + 8 * h;
        row_ok[h] = n < N;
        e_row[h] = (long long)(row_ok[h] ? n : 0) * K;
    }

    float c[NT][4];
#pragma unroll
    for (int u = 0; u < NT; ++u) c[u][0] = c[u][1] = c[u][2] = c[u][3] = 0.f;
    const int nchunks = (K + kGChunk - 1) / kGChunk;
    const int my_chunks = warp < nchunks ? (nchunks - warp + W - 1) / W : 0;  // chunks warp, warp + W, ...

    // ring stage of this warp: code part p (0: row g lo 16 B, 1: row g hi, 2: row g+8 lo, 3: row g+8 hi) of lane l at
    // p * 512 + 16 l; scale part p at 2048 + p * 128 + 4 l  (conflict-free both ways)
    const uint32_t ring0 = static_cast<uint32_t>(__cvta_generic_to_shared(ring_smem)) + (uint32_t)warp * (kRing * kRingStageBytes);
    auto issue = [&](int i) {
        if (i < my_chunks) {
            const int kb = (warp + W * i) * kGChunk + 64 * t;
            const uint32_t st = ring0 + (uint32_t)(i % kRing) * kRingStageBytes;
            if (kb < K) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (row_ok[h]) {
                        const long long e = e_row[h] + kb;
                        const uint8_t* src = B + (e >> 1);
                        cp_async16(st + (2 * h) * 512 + lane * 16, src);
                        cp_async16(st + (2 * h + 1) * 512 + lane * 16, src + 16);
                        if (!nested) {
                            cp_async4(st + 2048 + (2 * h) * 128 + lane * 4, absmax + (e >> log2_bs));
                            if (two_scales) cp_async4(st + 2048 + (2 * h + 1) * 128 + lane * 4, absmax + ((e + 32) >> log2_bs));
                        }
                    }
                }
            }
        }
        cp_async_commit();  // (an empty group keeps the group count in step with the iteration count)
    };
#pragma unroll
    for (int i = 0; i < kRing - 1; ++i) issue(i);

    // double-quantised statistics are computed, not copied: one chunk ahead in registers
    float ns[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
    auto fetch_nested = [&](int i) {
        ns[0][0] = ns[0][1] = ns[1][0] = ns[1][1] = 0.f;
        if (nested && i < my_chunks) {
            const int kb = (warp + W * i) * kGChunk + 64 * t;
            if (kb < K) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (row_ok[h]) {
                        const long long e = e_row[h] + kb;
                        ns[h][0] = sc.load(e >> log2_bs);
                        ns[h][1] = two_scales ? sc.load((e + 32) >> log2_bs) : ns[h][0];
                    }
                }
            }
        }
    };
    fetch_nested(0);

    for (int i = 0; i < my_chunks; ++i) {
        const int kb = (warp + W * i) * kGChunk + 64 * t;
        const bool k_ok = kb < K;
        issue(i + kRing - 1);
        cp_async_wait<kRing - 1>();  // this lane's copies of stage i have landed
        const uint32_t st = ring0 + (uint32_t)(i % kRing) * kRingStageBytes;
        float sv[2][2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            sv[h][0] = sv[h][1] = 0.f;
            if (k_ok && row_ok[h]) {
                if (nested) {
                    sv[h][0] = ns[h][0];
                    sv[h][1] = ns[h][1];
                } else {
                    sv[h][0] = lds_f1(st + 2048 + (2 * h) * 128 + lane * 4);
                    sv[h][1] = two_scales ? lds_f1(st + 2048 + (2 * h + 1) * 128 + lane * 4) : sv[h][0];
                }
            }
        }
        fetch_nested(i + 1);

        DecodeTable tab0, tab1;
        build_table<T, QT>(sv[0][0], tab0);
        build_table<T, QT>(sv[1][0], tab1);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            if (hh == 1 && two_scales) {
                build_table<T, QT>(sv[0][1], tab0);
                build_table<T, QT>(sv[1][1], tab1);
            }
            // 32 codes of row g and of row g + 8: k [kb + 32 hh, +32)
            uint4 qa = make_uint4(0, 0, 0, 0), qb = make_uint4(0, 0, 0, 0);
            if (k_ok && row_ok[0]) qa = lds_v4(st + hh * 512 + lane * 16);
            if (k_ok && row_ok[1]) qb = lds_v4(st + (2 + hh) * 512 + lane * 16);
            const uint32_t wa[4] = {qa.x, qa.y, qa.z, qa.w};
            const uint32_t wb[4] = {qb.x, qb.y, qb.z, qb.w};
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                // one packed word = 8 consecutive k = two MMAs (k-slots 2t, 2t+1, 2t+8, 2t+9 each)
                uint32_t ra[4], rb[4];
                decode_word(wa[w], tab0, ra);
                decode_word(wb[w], tab1, rb);
#pragma unroll
                for (int u = 0; u < NT; ++u) {
                    uint4 av = make_uint4(0, 0, 0, 0);  // activations of token g + 8u at the same 8 k
                    if (tok_ok[u] && k_ok) av = __ldg(reinterpret_cast<const uint4*>(arow[u] + kb) + 4 * hh + w);
                    WarpMma<T>::run(c[u], ra[0], rb[0], ra[1], rb[1], av.x, av.y);
                    WarpMma<T>::run(c[u], ra[2], rb[2], ra[3], rb[3], av.z, av.w);
                }
            }
        }
    }
    cp_async_wait<0>();

    // accumulator fragment: c0/c1 = (row g, tokens 8u + 2t, 8u + 2t+1), c2/c3 = (row g + 8, same tokens)
#pragma unroll
    for (int u = 0; u < NT; ++u) {
        float* r = red[warp] + u * 8 * kGRows;
        r[(2 * t) * kGRows + g] = c[u][0];
        r[(2 * t + 1) * kGRows + g] = c[u][1];
        r[(2 * t) * kGRows + g + 8] = c[u][2];
        r[(2 * t + 1) * kGRows + g + 8] = c[u][3];
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < kGRows * 8 * NT; idx += W * 32) {
        const int tok = idx / kGRows;  // idx = token * 16 + row
        const int n = n0 + (idx % kGRows);
        if (tok < M && n < N) {
            float acc = 0.f;
#pragma unroll
            for (int w = 0; w < W; ++w) acc += red[w][idx];
            if constexpr (PART) {
                store_partial(out, tok, n, ldc, acc);
            } else {
                const float b = bias != nullptr ? DT<T>::to_f32(bias[n]) : 0.f;
                out[(long long)tok * ldc + n] = DT<T>::from_f32(acc + b);
            }
        }
    }
}

// the ring needs the dynamic shared-memory opt-in (per device and instantiation)
template <typename T, int QT, int W, int NT, bool PART>
bool launch_mma_variant(dim3 grid, cudaStream_t stream, const T* A, const uint8_t* B, const float* absmax,
                        const uint8_t* absmax_8bit, const float* absmax_code, const float* absmax_offset,
                        typename OutArg<T, PART>::type out, const T* bias, int M, int N, int K, int ldc, int l2) {
    auto kern = gemv4_mma_kernel<T, QT, W, NT, PART>;
    constexpr int kSmem = W * kRing * kRingStageBytes;
    static bool attr_set[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return false;
    if (!attr_set[dev]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem) != cudaSuccess) {
            set_last_error("gemv4_mma smem attr", cudaGetLastError());
            return false;
        }
        attr_set[dev] = true;
    }
    kern<<<grid, W * 32, kSmem, stream>>>(A, B, absmax, absmax_8bit, absmax_code, absmax_offset, out, bias, M, N, K, ldc,
                                          l2);
    return true;
}

} // namespace

// M <= 16, 16-bit activations, K % 64 == 0, power-of-two blocksize >= 32, 16-byte aligned A and B.
template <typename T, bool PART>
bool launch_gemv4_mma(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                      const float* absmax_code, const float* absmax_offset, typename OutArg<T, PART>::type out,
                      const T* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, cudaStream_t stream) {
    if (M <= 0 || N <= 0) return true;
    if (M > 16 || K < 64 || (K % 64) != 0) return false;
    if (blocksize < 32 || (blocksize & (blocksize - 1)) != 0) return false;
    if ((reinterpret_cast<uintptr_t>(A) & 15) != 0 || (reinterpret_cast<uintptr_t>(B) & 15) != 0) return false;
    if (quant_type != kNF4 && quant_type != kFP4) return false;
    const dim3 grid((N + kGRows - 1) / kGRows);
    const int l2 = ilog2_pow2(blocksize);
    // Few row tiles (small N): 8 warps per CTA split K so that the machine is covered; otherwise 4
    // warps, which run more k-chunks each and keep the prefetch pipeline busy.
    static const int forced_w = [] {
        const char* e = getenv("BNB_B200_GEMV_WARPS");
        return e ? atoi(e) : 0;
    }();
    // Narrow layers (N <= 2048: fewer than one CTA per SM at 8 warps): 16 warps per CTA split K into single
    // 256-wide chunks so that the whole packed weight is in flight at once (measured, 1024 x 4096, M = 1..8:
    // 5.9-6.6 us against 6.7-7.2; wider layers lose 5-15 % with 16 warps, profiles/r02_decode_regime.md).
    int warps = ((long long)grid.x * 4 >= 12LL * device_sm_count()) ? 4 : 8;
    if (K >= 16 * kGChunk && (int)grid.x <= 128) warps = 16;
    if (forced_w == 4 || forced_w == 8 || forced_w == 16) warps = forced_w;
#define BNB200_GEMV_MMA(QT, WV)                                                                                        \
    do {                                                                                                               \
        if (M <= 8)                                                                                                    \
            ok = launch_mma_variant<T, QT, WV, 1, PART>(grid, stream, A, B, absmax, absmax_8bit, absmax_code,               \
                                                  absmax_offset, out, bias, M, N, K, ldc, l2);                        \
        else                                                                                                           \
            ok = launch_mma_variant<T, QT, WV, 2, PART>(grid, stream, A, B, absmax, absmax_8bit, absmax_code,               \
                                                  absmax_offset, out, bias, M, N, K, ldc, l2);                        \
    } while (0)
    bool ok = false;
    if (quant_type == kNF4) {
        if (warps == 4) BNB200_GEMV_MMA(kNF4, 4);
        else if (warps == 8) BNB200_GEMV_MMA(kNF4, 8);
        else BNB200_GEMV_MMA(kNF4, 16);
    } else {
        if (warps == 4) BNB200_GEMV_MMA(kFP4, 4);
        else if (warps == 8) BNB200_GEMV_MMA(kFP4, 8);
        else BNB200_GEMV_MMA(kFP4, 16);
    }
#undef BNB200_GEMV_MMA
    if (!ok) return false;
    BNB200_CHECK_LAUNCH("gemv4_mma");
    return true;
}

template bool launch_gemv4_mma<__nv_bfloat16, false>(const __nv_bfloat16*, const uint8_t*, const float*,
                                                     const uint8_t*, const float*, const float*, __nv_bfloat16*,
                                                     const __nv_bfloat16*, int, int, int, int, int, int, cudaStream_t);
template bool launch_gemv4_mma<__half, false>(const __half*, const uint8_t*, const float*, const uint8_t*, const float*,
                                              const float*, __half*, const __half*, int, int, int, int, int, int,
                                              cudaStream_t);
template bool launch_gemv4_mma<__nv_bfloat16, true>(const __nv_bfloat16*, const uint8_t*, const float*, const uint8_t*,
                                                    const float*, const float*, OutList<float>, const __nv_bfloat16*, int,
                                                    int, int, int, int, int, cudaStream_t);
template bool launch_gemv4_mma<__half, true>(const __half*, const uint8_t*, const float*, const uint8_t*, const float*,
                                             const float*, OutList<float>, const __half*, int, int, int, int, int, int,
                                             cudaStream_t);

} // namespace bnb200
