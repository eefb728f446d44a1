// int8_gemm.cu -- the LLM.int8() GEMM for sm_90a:  C[M,N] = A[M,K] . B[N,K]^T, int8 x int8 -> int32.
//
// Replaces reference igemmlt<32,0> -> cublasLtMatmul (csrc/ops.cu:282-404) with a wgmma s8 kernel: both
// operands TMA-staged (128-byte swizzle), int32 accumulators in registers, exact.  The epilogue either
// stores int32 (cigemmlt_32 ABI) or applies the dequantisation of reference kdequant_mm_int32_fp16
// (csrc/kernels.cu:1396-1448),
//     fp16/bf16( fma(acc * SCA[m] * SCB[n], 1/127^2, bias[n]) ),
// in-kernel, which removes the 2 x M x N x 4-byte int32 round trip through HBM -- and, for LLM.int8()'s
// mixed decomposition (reference backends/default/ops.py:64-100: `output.addmm(subA, subB)` after the int8
// matmul), adds the OUTLIER term  sum_j subA[m, j] * subB[j, n]  (fp16/bf16 products, fp32 accumulation)
// in the same epilogue, so the second pass over out[M, N] and the cuBLAS call of the reference chain are gone.
#include "common.cuh"
#include "hopper_ptx.cuh"

namespace bnb200 {

namespace {

// ======================================================================================
// Warp-specialised kernel, one 128 x 128 output tile per CTA:
//   * CTA tile 128 tokens (two consumer warpgroups of 64 rows, the wgmma M dimension) x 128 features
//     (the wgmma N dimension), K in 128-byte k-blocks, a TMA ring (128-byte swizzle) of up to 6 stages;
//   * each consumer warpgroup issues four wgmma m64n128k32 per stage from shared-memory descriptors and
//     releases the previous stage once its wgmma group has completed (wgmma.wait_group 1);
//   * the epilogue dequantises straight from the accumulator registers.
// Warps: 0..7 = consumers, 8 = TMA producer.
// ======================================================================================
constexpr int kI8BK = 128;        // int8 elements per stage = one 128-byte swizzled row
constexpr int kI8TileM = 128;     // tokens per CTA tile
constexpr int kI8TileN = 128;     // output features per CTA tile
constexpr int kI8Consumers = 256;
constexpr int kI8Threads = kI8Consumers + 32;
constexpr int kI8StageBytes = (kI8TileM + kI8TileN) * kI8BK;

template <int JMAX> struct I8Cfg {
    // with the outlier term, 2 x 128 rows x JMAX T values of it share the 227 KB
    static constexpr int kStages = JMAX > 0 ? 5 : 6;
};

// EPI: 0 = int32 out, 1 = fp16 out, 2 = bf16 out (fused dequant)
struct I8Params {
    void* out;
    const float* SCA;   // [M]  row stats of the activations
    const float* SCB;   // [N]  row stats of the weights
    const void* bias;   // T[N] or NULL
    const void* subA;   // T[M, jpad]  outlier columns of the activations (zero-padded to jpad), or NULL
    const void* subBT;  // T[N, jpad]  dequantised weight columns CB[:, cols] * SCB / 127, or NULL
    int jpad;           // padded outlier count (multiple of 8, <= JMAX)
    int M, N, K, ldc;
    int kblocks;
    int n_tiles;
};

// 8 consecutive T -> fp32
template <int EPI> __device__ __forceinline__ void i8_unpack8(const uint4& r, float (&v)[8]) {
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (EPI == 1) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
            v[2 * i] = f.x;
            v[2 * i + 1] = f.y;
        } else {
            v[2 * i] = __uint_as_float(w[i] << 16);
            v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
        }
    }
}

// JMAX: capacity of the fused outlier term (0 = none): subA of the CTA's 128 tokens and subBT of its 128 features
// are staged in shared memory after the main loop.
template <int EPI, int JMAX>
__global__ void __launch_bounds__(kI8Threads, 1)
    int8_gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                        const I8Params p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    constexpr int kStages = I8Cfg<JMAX>::kStages;
    uint8_t* stages = smem;                                                       // [stages][A 16 KB | B 16 KB]
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * kI8StageBytes);
    uint64_t* full = bars;              // [stages] TMA -> consumers
    uint64_t* empty = bars + kStages;   // [stages] the 8 consumer warps -> TMA
    uint4* s_suba = reinterpret_cast<uint4*>(smem + kStages * kI8StageBytes + 256);  // [128][JMAX] of T
    uint4* s_subb = s_suba + kI8TileM * (JMAX / 8);                                  // [128][JMAX] of T

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n0 = (blockIdx.x % p.n_tiles) * kI8TileN;
    const int m0 = (blockIdx.x / p.n_tiles) * kI8TileM;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            ptx::mbar_init(&full[s], 1);
            ptx::mbar_init(&empty[s], kI8Consumers / 32);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp == kI8Consumers / 32) {
        // ================================================================== TMA producer
        if (ptx::elect_one()) {
            ptx::prefetch_tmap(&tmap_a);
            ptx::prefetch_tmap(&tmap_b);
            for (int i = 0; i < p.kblocks; ++i) {
                const int s = i % kStages;
                ptx::mbar_wait(&empty[s], ((i / kStages) & 1u) ^ 1u);
                uint8_t* sa = stages + s * kI8StageBytes;
                ptx::mbar_arrive_expect_tx(&full[s], kI8StageBytes);
                // (rows past M / N and k columns past K are out of bounds for the tensor maps: TMA zero-fills them)
                ptx::tma_load_2d(sa, &tmap_a, &full[s], i * kI8BK, m0);
                ptx::tma_load_2d(sa + kI8TileM * kI8BK, &tmap_b, &full[s], i * kI8BK, n0);
            }
        }
        return;
    }

    // ====================================================================== consumers
    const int wg = warp >> 2;
    const int g = lane >> 2, t = lane & 3;
    int32_t acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0;
    int prev_s = -1;
    for (int i = 0; i < p.kblocks; ++i) {
        const int s = i % kStages;
        ptx::mbar_wait(&full[s], (i / kStages) & 1u);
        const uint32_t sa = ptx::smem_u32(stages + s * kI8StageBytes) + wg * 64 * kI8BK;  // this warpgroup's 64 rows
        const uint32_t sb = ptx::smem_u32(stages + s * kI8StageBytes) + kI8TileM * kI8BK;
        const uint64_t adesc = ptx::make_sw128_kmajor_desc(sa);
        const uint64_t bdesc = ptx::make_sw128_kmajor_desc(sb);
        ptx::wgmma_fence();
#pragma unroll
        for (int j = 0; j < kI8BK / 32; ++j) ptx::wgmma_m64n128k32_s8_ss(acc, adesc + 2 * j, bdesc + 2 * j);
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();  // the previous stage's wgmma group has completed: release its slot
        if (prev_s >= 0) {
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(&empty[prev_s]);
        }
        prev_s = s;
    }
    ptx::wgmma_wait<0>();
#pragma unroll
    for (int j = 0; j < 64; ++j) ptx::fence_operand(acc[j]);

    // ====================================================================== epilogue
    // acc[4j + e]: token row rl + 8 * (e >= 2), feature column 8j + 2t + (e & 1)
    const int rl = wg * 64 + (warp & 3) * 16 + g;
    if constexpr (JMAX > 0) {
        // stage the outlier operands (zero rows past M / N), thread e owns row e & 127 of one of the two
        const int e = threadIdx.x;
        const int r = e & 127;
        const bool is_b = e >= 128;
        const int gr = (is_b ? n0 : m0) + r;
        const bool ok = gr < (is_b ? p.N : p.M);
        const uint16_t* src = reinterpret_cast<const uint16_t*>(is_b ? p.subBT : p.subA) + (long long)(ok ? gr : 0) * p.jpad;
        uint4* dst = (is_b ? s_subb : s_suba) + r * (JMAX / 8);
#pragma unroll
        for (int q = 0; q < JMAX / 8; ++q)
            dst[q] = (ok && 8 * q < p.jpad) ? __ldg(reinterpret_cast<const uint4*>(src) + q) : make_uint4(0, 0, 0, 0);
        asm volatile("bar.sync 1, 256;" ::: "memory");
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + rl + 8 * h;
        if (m >= p.M) continue;
        float sca = 0.f;
        if (EPI != 0) sca = __ldg(p.SCA + m);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int n = n0 + 8 * j + 2 * t;  // this thread's two consecutive columns n, n + 1
            const int v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if (EPI == 0) {
                int* dst = reinterpret_cast<int*>(p.out) + (long long)m * p.ldc + n;
                if (n + 1 < p.N && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) {
                    *reinterpret_cast<int2*>(dst) = make_int2(v0, v1);
                } else {
                    if (n < p.N) dst[0] = v0;
                    if (n + 1 < p.N) dst[1] = v1;
                }
            } else {
            // outlier term of this token and columns n, n + 1: sum_j subA[m, j] * subBT[n, j] in j order (fp32 fma)
            float ol[2] = {0.f, 0.f};
            if constexpr (JMAX > 0) {
                const uint4* arow = s_suba + (rl + 8 * h) * (JMAX / 8);
                const uint4* brow = s_subb + (8 * j + 2 * t) * (JMAX / 8);
#pragma unroll
                for (int q = 0; q < JMAX / 8; ++q) {
                    if (8 * q < p.jpad) {
                        float a8[8], b8[8], c8[8];
                        i8_unpack8<EPI>(arow[q], a8);
                        i8_unpack8<EPI>(brow[q], b8);
                        i8_unpack8<EPI>(brow[JMAX / 8 + q], c8);
#pragma unroll
                        for (int x = 0; x < 8; ++x) {
                            ol[0] = fmaf(a8[x], b8[x], ol[0]);
                            ol[1] = fmaf(a8[x], c8[x], ol[1]);
                        }
                    }
                }
            }
            float f[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int nn = n + u;
                const int v = u ? v1 : v0;
                const float scb = nn < p.N ? __ldg(p.SCB + nn) : 0.f;
                float b = 0.f;
                if (p.bias != nullptr && nn < p.N) {
                    if (EPI == 1) b = __half2float(reinterpret_cast<const __half*>(p.bias)[nn]);
                    else b = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.bias)[nn]);
                }
                if (EPI == 1) {
                    f[u] = dequant_value(v, sca, scb, b);
                    // reference: the int8 result is an fp16 tensor, then addmm adds the fp32-accumulated
                    // outlier product and rounds once more
                    if constexpr (JMAX > 0) f[u] = __half2float(__float2half_rn(f[u])) + ol[u];
                } else {
                    // bf16 output, bit-identical to the reference chain (backends/cuda/ops.py:186-210): the kernel
                    // result is fp16, a non-fp16 bias is added by `out.add_(bias)` on the fp16 tensor (fp32 add,
                    // one rounding to fp16), then `.to(bfloat16)`.
                    f[u] = __half2float(__float2half_rn(dequant_value(v, sca, scb, 0.f)));
                    if (p.bias != nullptr) f[u] = __half2float(__float2half_rn(f[u] + b));
                    if constexpr (JMAX > 0) f[u] = __bfloat162float(__float2bfloat16_rn(f[u])) + ol[u];
                }
            }
            const uint32_t w = EPI == 1 ? pack2<__half>(f[0], f[1]) : pack2<__nv_bfloat16>(f[0], f[1]);
            uint16_t* dst = reinterpret_cast<uint16_t*>(p.out) + (long long)m * p.ldc + n;
            if (n + 1 < p.N && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
                *reinterpret_cast<uint32_t*>(dst) = w;
            } else {
                if (n < p.N) dst[0] = (uint16_t)w;
                if (n + 1 < p.N) dst[1] = (uint16_t)(w >> 16);
            }
            }
        }
    }
}

template <int EPI, int JMAX = 0>
int launch_i8(const CUtensorMap& ta, const CUtensorMap& tb, I8Params& p, cudaStream_t stream) {
    constexpr size_t smem_bytes =
        1024 + size_t(I8Cfg<JMAX>::kStages) * kI8StageBytes + 256 + size_t(kI8TileM + kI8TileN) * JMAX * 2;
    static bool attr_set[64] = {};  // the shared-memory opt-in is per device
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 1;
    auto kern = int8_gemm_tc_kernel<EPI, JMAX>;
    p.kblocks = (p.K + kI8BK - 1) / kI8BK;
    if (!attr_set[dev]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes) != cudaSuccess) {
            set_last_error("int8_gemm_tc smem attr", cudaGetLastError());
            return 1;
        }
        attr_set[dev] = true;
    }
    p.n_tiles = (p.N + kI8TileN - 1) / kI8TileN;
    const int m_tiles = (p.M + kI8TileM - 1) / kI8TileM;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(p.n_tiles * m_tiles, 1, 1);
    cfg.blockDim = dim3(kI8Threads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, ta, tb, p);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        set_last_error("int8_gemm_tc launch", e);
        return 1;
    }
    BNB200_CHECK_LAUNCH("int8_gemm_tc");
    return 0;
}

} // namespace

// epi: 0 int32, 1 fp16, 2 bf16.  Returns 0 ok, 100 "not implemented for this shape".
// subA / subBT / jpad: the fused outlier term (epi 1 / 2 only; jpad a multiple of 8, <= 64), or NULL / 0.
int launch_int8_gemm(const int8_t* acts, const int8_t* weights, void* out, const float* SCA,
                                const float* SCB, const void* bias, int M, int N, int K, int ldc, int epi,
                                cudaStream_t stream, const void* subA, const void* subBT, int jpad) {
    if (M <= 0 || N <= 0) return 0;
    if (K <= 0 || (K % 16) != 0) return 100;
    if (jpad != 0 && (epi == 0 || jpad < 0 || jpad > 64 || (jpad % 8) != 0 || subA == nullptr || subBT == nullptr ||
                      (reinterpret_cast<uintptr_t>(subA) & 15) != 0 || (reinterpret_cast<uintptr_t>(subBT) & 15) != 0))
        return 100;
    if ((reinterpret_cast<uintptr_t>(acts) & 15) != 0 || (reinterpret_cast<uintptr_t>(weights) & 15) != 0) return 100;
    CUtensorMap ta, tb;
    if (!encode_tmap_2d(&ta, acts, 1, 128, (uint64_t)M, (uint64_t)K, (uint64_t)K, kI8TileM, kI8BK)) return 100;
    if (!encode_tmap_2d(&tb, weights, 1, 128, (uint64_t)N, (uint64_t)K, (uint64_t)K, kI8TileN, kI8BK)) return 100;
    I8Params p{};
    p.out = out;
    p.SCA = SCA;
    p.SCB = SCB;
    p.bias = bias;
    p.M = M;
    p.N = N;
    p.K = K;
    p.ldc = ldc;
    p.subA = subA;
    p.subBT = subBT;
    p.jpad = jpad;
    if (jpad > 0) {
        // fused outlier term, capacity = next of {8, 16, 32, 64}
#define BNB200_I8_J(E)                                                                                                 \
        if (jpad <= 8) return launch_i8<E, 8>(ta, tb, p, stream);                                                      \
        if (jpad <= 16) return launch_i8<E, 16>(ta, tb, p, stream);                                                    \
        if (jpad <= 32) return launch_i8<E, 32>(ta, tb, p, stream);                                                    \
        return launch_i8<E, 64>(ta, tb, p, stream);
        if (epi == 1) {
            BNB200_I8_J(1)
        }
        BNB200_I8_J(2)
#undef BNB200_I8_J
    }
    switch (epi) {
    case 0: return launch_i8<0>(ta, tb, p, stream);
    case 1: return launch_i8<1>(ta, tb, p, stream);
    default: return launch_i8<2>(ta, tb, p, stream);
    }
}

} // namespace bnb200
