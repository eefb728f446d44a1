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
#include <type_traits>

#include "common.cuh"
#include "hopper_ptx.cuh"
#include "int8_epilogue.cuh"

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

constexpr int kI8MaxOuts = 8;

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
    // kDevJ instance: the outlier count J on the device (subA / subBT then hold min(J, JMAX) columns at a row pitch of
    // JMAX), and what the columns past JMAX are gathered from
    const int* jcount;
    const int* cols;    // [J] ascending outlier columns
    const void* A;      // T[M, K] activations
    const int8_t* CB;   // [N, K] weight codes
};

// the parameters of a kMulti instance: every output element is stored to outs[0 .. n_outs) (row stride ldc) instead
// of `out` (a type of its own, so that the single-destination instances keep their parameter block)
struct I8MultiParams : I8Params {
    void* outs[kI8MaxOuts];
    int n_outs;
    // EPI 0 only: 0 = every row to every destination; > 0 = row m to outs[m / rows_per_out] only, at row
    // m % rows_per_out (scatter_row: each rank of a sequence-parallel layer receives its own tokens' partials)
    int rows_per_out;
};
// the parameters of a kGrouped instance: every expert of a mixture-of-experts layer in one launch.  CB / SCB / bias are
// the E experts' [N, K] weights stacked ([E * N, K], [E * N], [E * N]); offs[E] the expert end rows, clamped on the
// device; jcount / cols (kDevJ) the per-expert outlier counts [E] and ascending lists [E, K], subBT [E * N, JMAX]
struct I8GroupedParams : I8Params {
    const int* offs;
    int E;
};
template <bool kMulti, bool kGrouped = false>
using I8ParamsOf = typename std::conditional<
    kMulti, I8MultiParams, typename std::conditional<kGrouped, I8GroupedParams, I8Params>::type>::type;

// kGrouped: the group table past the outlier operands' shared memory: gend[e] = end_e, gtp[e] = the 128-row m-tiles of
// experts 0..e-1 (gtp[E] = all of them), then the scan's per-warp totals
constexpr int kI8Warps = kI8Threads / 32;
constexpr int kI8GroupTabBytes = (2 * kMaxExperts + 1 + 2 * kI8Warps) * 4;

// kGrouped: the group table, built by the whole CTA (every CTA builds the same one).  Thread t takes experts
// [t * kPer, t * kPer + kPer): end_e = min(M, max(0, offs[0..e])) -- the clamp of the 4-bit grouped GEMM, as a prefix
// maximum -- then the m-tile counts ceil((end_e - end_{e-1}) / 128) and their exclusive prefix sum, each scan over the
// warp by shuffles and across the warps through shared memory.  Ends with a __syncthreads.
__device__ __forceinline__ void i8_group_table(const int* __restrict__ offs, int E, int M, int* gend) {
    constexpr int kPer = (kMaxExperts + kI8Threads - 1) / kI8Threads;
    static_assert(kMaxExperts <= (kI8Threads - 1) * kPer, "the last thread must hold no expert");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int* gtp = gend + kMaxExperts;
    int* wtot = gtp + kMaxExperts + 1;  // [kI8Warps] maxima, then [kI8Warps] tile counts
    const int e0 = threadIdx.x * kPer;
    int v[kPer];
    int run = 0;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
        v[i] = e0 + i < E ? max(__ldg(offs + e0 + i), 0) : 0;
        run = max(run, v[i]);
    }
    int inc = run;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc = max(inc, o);
    }
    if (lane == 31) wtot[warp] = inc;
    __syncthreads();
    int r = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) r = 0;
    for (int w2 = 0; w2 < warp; ++w2) r = max(r, wtot[w2]);
    int prev = min(r, M);
    int cnt[kPer], tiles = 0;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
        r = max(r, v[i]);
        v[i] = min(r, M);  // end_e (experts past E: end_{E-1}, no rows)
        cnt[i] = (v[i] - prev + kI8TileM - 1) / kI8TileM;
        prev = v[i];
        tiles += cnt[i];
    }
    int incs = tiles;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incs, d);
        if (lane >= d) incs += o;
    }
    if (lane == 31) wtot[kI8Warps + warp] = incs;
    __syncthreads();
    int base = incs - tiles;
    for (int w2 = 0; w2 < warp; ++w2) base += wtot[kI8Warps + w2];
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
        if (e0 + i < E) {
            gend[e0 + i] = v[i];
            gtp[e0 + i] = base;
        }
        base += cnt[i];
    }
    if (threadIdx.x == kI8Threads - 1) gtp[E] = base;  // the last thread's experts are past E: base is the total
    __syncthreads();
}

// kGrouped: the unit's expert e (the last e with gtp[e] <= g for the CTA's m-tile g, which has m-tiles since g < gtp[E]),
// its first row m0, its end row and its first row of the stacked weights.  Looked up where each role needs it, through
// volatile reads, rather than held across the main loop: held, the values cost the device-count instances more spills.
struct I8Unit {
    int e, m0, m_end, wrow;
};
__device__ __forceinline__ I8Unit i8_unit(const int* gend_, int E, int N, int n_tiles) {
    const volatile int* gend = gend_;
    const volatile int* gtp = gend_ + kMaxExperts;
    const int g = blockIdx.x / n_tiles;
    int lo = 0;
#pragma unroll
    for (int step = kMaxExperts / 2; step >= 1; step >>= 1)
        if (lo + step < E && gtp[lo + step] <= g) lo += step;
    I8Unit u;
    u.e = lo;
    u.m0 = (lo > 0 ? gend[lo - 1] : 0) + (g - gtp[lo]) * kI8TileM;
    u.m_end = gend[lo];
    u.wrow = lo * N;
    return u;
}

// kGrouped: rows [end_{E-1}, M) belong to no expert: +0, each CTA's 256 consumer threads storing a strided share
__device__ __forceinline__ void i8_zero_tail(uint16_t* out, int m_tail, int M, int N, int ldc) {
    const long long n_tail = (long long)(M - m_tail) * N;
    for (long long i = (long long)blockIdx.x * kI8Consumers + threadIdx.x; i < n_tail;
         i += (long long)gridDim.x * kI8Consumers)
        out[(m_tail + i / N) * ldc + i % N] = 0;
}

// JMAX: capacity of the fused outlier term (0 = none): subA of the CTA's 128 tokens and subBT of its 128 features
// are staged in shared memory after the main loop.
// kDevJ (JMAX = 64): the outlier count is read from device memory, so one launch serves any J.  The first JMAX columns
// come from subA / subBT; the rest are gathered from A and CB, JMAX at a time, into the same shared-memory buffers and
// continue the same fp32 sum in column order.
// kMulti: every output element goes to each of p.outs[0 .. p.n_outs) (a local buffer and the peers' mapped buffers of a
// tensor-parallel layer) instead of p.out; the values are those of the single-destination instance.
// kGrouped: every expert of a mixture-of-experts layer in one launch (I8GroupedParams).  A unit is a 128-row m-tile of
// one expert and a 128-feature n-tile; blockIdx.x runs the units in (m-tile, n-tile) order, and the CTAs past the
// device-known unit count only zero the tail rows.  Expert e's j-th m-tile starts at row end_{e-1} + 128 j; rows of it
// past end_e are the next expert's, computed with the wrong weights and not stored.  Every stored element is the one the
// plain (kDevJ) instance gives on that expert's rows alone.
template <int EPI, int JMAX, bool kDevJ = false, bool kMulti = false, bool kGrouped = false>
__global__ void __launch_bounds__(kI8Threads, 1)
    int8_gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                        const I8ParamsOf<kMulti, kGrouped> p) {
    static_assert(!(kGrouped && kMulti), "the grouped instances have one destination");
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
    int m0 = (blockIdx.x / p.n_tiles) * kI8TileM;
    // kGrouped: the unit's expert, its end row and its first row of the stacked weights (e * N)
    int ge = 0, m_end = p.M, wrow = 0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            ptx::mbar_init(&full[s], 1);
            ptx::mbar_init(&empty[s], kI8Consumers / 32);
        }
        ptx::fence_barrier_init();
    }
    if constexpr (kGrouped) {
        int* gend = reinterpret_cast<int*>(s_subb + kI8TileN * (JMAX / 8));
        const int* gtp = gend + kMaxExperts;
        i8_group_table(p.offs, p.E, p.M, gend);
        if (blockIdx.x / p.n_tiles >= gtp[p.E]) {  // past the units
            if (threadIdx.x < kI8Consumers) i8_zero_tail(reinterpret_cast<uint16_t*>(p.out), gend[p.E - 1], p.M, p.N, p.ldc);
            return;
        }
    }
    __syncthreads();

    if (warp == kI8Consumers / 32) {
        // ================================================================== TMA producer
        if constexpr (kGrouped) {
            const I8Unit u = i8_unit(reinterpret_cast<const int*>(s_subb + kI8TileN * (JMAX / 8)), p.E, p.N, p.n_tiles);
            m0 = u.m0;
            wrow = u.wrow;
        }
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
                // (kGrouped: rows of the expert's stacked weights; a tile reaching past its N features loads the next
                // expert's rows, whose results are not stored)
                ptx::tma_load_2d(sa + kI8TileM * kI8BK, &tmap_b, &full[s], i * kI8BK, wrow + n0);
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
    if constexpr (kGrouped) {
        const I8Unit u = i8_unit(reinterpret_cast<const int*>(s_subb + kI8TileN * (JMAX / 8)), p.E, p.N, p.n_tiles);
        ge = u.e;
        m0 = u.m0;
        m_end = u.m_end;
        wrow = u.wrow;
    }

    // ====================================================================== epilogue
    // acc[4j + e]: token row rl + 8 * (e >= 2), feature column 8j + 2t + (e & 1)
    const int rl = wg * 64 + (warp & 3) * 16 + g;
    int J = 0;                   // kDevJ: the outlier count
    float olr[kDevJ ? 64 : 1];   // kDevJ: the outlier term of this thread's outputs, (h, j, u) at 32 h + 2 j + u
    if constexpr (kDevJ) {
        static_assert(JMAX == 64, "the device-count instance stages 64 columns at a time");
        J = __ldg(p.jcount + ge);  // (kGrouped: the unit's expert's count and list)
        const int* cols = p.cols + (long long)ge * p.K;
#pragma unroll
        for (int i = 0; i < 64; ++i) olr[i] = 0.f;
        // thread e stages row e & 127 of one of the two operands, as below
        const int e = threadIdx.x;
        const int r = e & 127;
        const bool is_b = e >= 128;
        const int gr = (is_b ? n0 : m0) + r;
        const bool ok = gr < (is_b ? p.N : p.M);
        const int grow = gr + (is_b ? wrow : 0);  // the row of subBT / SCB / CB (kGrouped: of the stacked weights)
        uint4* dst = (is_b ? s_subb : s_suba) + r * (JMAX / 8);
        for (int c0 = 0; c0 < J; c0 += JMAX) {
            const int jc = min(J - c0, JMAX);
            const int jpad = (jc + 7) & ~7;
            if (c0 == 0) {
                const uint16_t* src =
                    reinterpret_cast<const uint16_t*>(is_b ? p.subBT : p.subA) + (long long)(ok ? grow : 0) * JMAX;
#pragma unroll
                for (int q = 0; q < JMAX / 8; ++q)
                    dst[q] = (ok && 8 * q < jpad) ? __ldg(reinterpret_cast<const uint4*>(src) + q) : make_uint4(0, 0, 0, 0);
            } else {
                asm volatile("bar.sync 1, 256;" ::: "memory");  // every consumer is done with the previous chunk
                // subA[m, j] = A[m, cols[j]]; subBT[n, j] = T((float(CB[n, cols[j]]) * SCB[n]) * (1/127)), as the prep
                // kernel builds them
                const float scb = ok && is_b ? __ldg(p.SCB + grow) : 0.f;
                for (int q = 0; q < JMAX / 8; ++q) {
                    uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                    for (int x = 0; x < 8; ++x) {
                        const int jj = 8 * q + x;
                        if (ok && jj < jc) {
                            const long long at = (long long)grow * p.K + __ldg(cols + c0 + jj);
                            uint32_t bits;
                            if (is_b) {
                                const float v = __fmul_rn(__fmul_rn((float)p.CB[at], scb), 7.874015718698502e-3f);
                                bits = EPI == 1 ? __half_as_ushort(__float2half_rn(v))
                                                : __bfloat16_as_ushort(__float2bfloat16_rn(v));
                            } else {
                                bits = reinterpret_cast<const uint16_t*>(p.A)[at];
                            }
                            w[x >> 1] |= bits << (16 * (x & 1));
                        }
                    }
                    dst[q] = make_uint4(w[0], w[1], w[2], w[3]);
                }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            // 8 columns at a time for all 64 outputs: each output still sums its columns in order.  The loop keeps the
            // code small; unrolled over all 64 columns, as the JMAX instances are, this epilogue is ~10 k instructions
            // and took 2.7x as long at J = 5 and 4096 tokens
#pragma unroll 1
            for (int q = 0; q < jpad / 8; ++q) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float a8[8];
                    i8_unpack8<EPI>(s_suba[(rl + 8 * h) * (JMAX / 8) + q], a8);
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const uint4* brow = s_subb + (8 * j + 2 * t) * (JMAX / 8);
                        float b8[8], c8[8];
                        i8_unpack8<EPI>(brow[q], b8);
                        i8_unpack8<EPI>(brow[JMAX / 8 + q], c8);
#pragma unroll
                        for (int x = 0; x < 8; ++x) {
                            olr[32 * h + 2 * j] = fmaf(a8[x], b8[x], olr[32 * h + 2 * j]);
                            olr[32 * h + 2 * j + 1] = fmaf(a8[x], c8[x], olr[32 * h + 2 * j + 1]);
                        }
                    }
                }
            }
        }
    } else if constexpr (JMAX > 0) {
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
    // with no outlier column at all the result is the plain int8 one: -0 + (+0) would otherwise turn a -0 into +0
    const bool add_ol = JMAX > 0 && (!kDevJ || J > 0);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + rl + 8 * h;
        if (m >= m_end) continue;  // (kGrouped: rows past the expert's end are the next expert's)
        float sca = 0.f;
        if (EPI != 0) sca = __ldg(p.SCA + m);
        // scattered rows: row m's one destination, found once for the column loop (a 128-token tile may span ranks)
        int* srow = nullptr;
        if constexpr (EPI == 0 && kMulti) {
            if (p.rows_per_out > 0) {
                const ScatterRow sr = scatter_row(m, p.rows_per_out);
                srow = reinterpret_cast<int*>(p.outs[sr.out]) + (long long)sr.row * p.ldc;
            }
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int n = n0 + 8 * j + 2 * t;  // this thread's two consecutive columns n, n + 1
            const int v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if (EPI == 0) {
                // (the single-destination store is spelled out apart, so that it compiles as before)
                if constexpr (kMulti) {
                    const int n_dst = srow != nullptr ? 1 : p.n_outs;
                    for (int d = 0; d < n_dst; ++d) {
                        int* dst =
                            (srow != nullptr ? srow : reinterpret_cast<int*>(p.outs[d]) + (long long)m * p.ldc) + n;
                        if (n + 1 < p.N && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) {
                            *reinterpret_cast<int2*>(dst) = make_int2(v0, v1);
                        } else {
                            if (n < p.N) dst[0] = v0;
                            if (n + 1 < p.N) dst[1] = v1;
                        }
                    }
                } else {
                int* dst = reinterpret_cast<int*>(p.out) + (long long)m * p.ldc + n;
                if (n + 1 < p.N && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) {
                    *reinterpret_cast<int2*>(dst) = make_int2(v0, v1);
                } else {
                    if (n < p.N) dst[0] = v0;
                    if (n + 1 < p.N) dst[1] = v1;
                }
                }
            } else {
            // outlier term of this token and columns n, n + 1: sum_j subA[m, j] * subBT[n, j] in j order (fp32 fma)
            float ol[2] = {0.f, 0.f};
            if constexpr (kDevJ) {
                ol[0] = olr[32 * h + 2 * j];
                ol[1] = olr[32 * h + 2 * j + 1];
            } else if constexpr (JMAX > 0) {
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
                const float scb = nn < p.N ? __ldg(p.SCB + wrow + nn) : 0.f;
                float b = 0.f;
                if (p.bias != nullptr && nn < p.N) {
                    if (EPI == 1) b = __half2float(reinterpret_cast<const __half*>(p.bias)[wrow + nn]);
                    else b = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.bias)[wrow + nn]);
                }
                f[u] = int8_epilogue_value<EPI>(v, sca, scb, b, p.bias != nullptr, add_ol, ol[u]);
            }
            const uint32_t w = EPI == 1 ? pack2<__half>(f[0], f[1]) : pack2<__nv_bfloat16>(f[0], f[1]);
            if constexpr (kMulti) {
                for (int d = 0; d < p.n_outs; ++d) {
                    uint16_t* dst = reinterpret_cast<uint16_t*>(p.outs[d]) + (long long)m * p.ldc + n;
                    if (n + 1 < p.N && (reinterpret_cast<uintptr_t>(dst) & 3) == 0) {
                        *reinterpret_cast<uint32_t*>(dst) = w;
                    } else {
                        if (n < p.N) dst[0] = (uint16_t)w;
                        if (n + 1 < p.N) dst[1] = (uint16_t)(w >> 16);
                    }
                }
            } else {
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
    if constexpr (kGrouped) {
        const int* gend = reinterpret_cast<const int*>(s_subb + kI8TileN * (JMAX / 8));
        i8_zero_tail(reinterpret_cast<uint16_t*>(p.out), gend[p.E - 1], p.M, p.N, p.ldc);
    }
}

template <int EPI, int JMAX = 0, bool kDevJ = false, bool kMulti = false, bool kGrouped = false>
int launch_i8(const CUtensorMap& ta, const CUtensorMap& tb, I8ParamsOf<kMulti, kGrouped>& p, cudaStream_t stream) {
    constexpr size_t smem_bytes = 1024 + size_t(I8Cfg<JMAX>::kStages) * kI8StageBytes + 256 +
                                  size_t(kI8TileM + kI8TileN) * JMAX * 2 + (kGrouped ? kI8GroupTabBytes : 0);
    static_assert(smem_bytes <= 227 * 1024, "shared memory");
    static bool attr_set[64] = {};  // the shared-memory opt-in is per device
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 1;
    auto kern = int8_gemm_tc_kernel<EPI, JMAX, kDevJ, kMulti, kGrouped>;
    p.kblocks = (p.K + kI8BK - 1) / kI8BK;
    if (!attr_set[dev]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes) != cudaSuccess) {
            set_last_error("int8_gemm_tc smem attr", cudaGetLastError());
            return 1;
        }
        attr_set[dev] = true;
    }
    p.n_tiles = (p.N + kI8TileN - 1) / kI8TileN;
    // kGrouped: the m-tiles are counted on the device; each expert adds at most one partial tile, so ceil(M / 128) + E
    // bounds them and sizes the grid
    int m_tiles = (p.M + kI8TileM - 1) / kI8TileM;
    if constexpr (kGrouped) m_tiles += p.E;
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
// jcount / cols / A: the outlier count on the device, the ascending outlier columns and the T[M, K] activations they
// index (epi 1 / 2 only; jpad = 64 is then the row pitch of subA / subBT), or NULL.
// outs / n_outs: 1 <= n_outs <= 8 destinations (device addresses, row stride ldc) that each receive every output element
// in place of `out` (not with jcount), or NULL / 0.
// rows_per_out > 0 (epi 0 with outs only): row m goes to outs[m / rows_per_out] only, at row m % rows_per_out.
int launch_int8_gemm(const int8_t* acts, const int8_t* weights, void* out, const float* SCA,
                                const float* SCB, const void* bias, int M, int N, int K, int ldc, int epi,
                                cudaStream_t stream, const void* subA, const void* subBT, int jpad,
                                const int* jcount, const int* cols, const void* A, void* const* outs, int n_outs,
                                int rows_per_out) {
    if (n_outs < 0 || n_outs > kI8MaxOuts || (n_outs > 0 && (outs == nullptr || jcount != nullptr))) return 100;
    if (rows_per_out < 0 || (rows_per_out > 0 && (epi != 0 || n_outs == 0 || (long long)n_outs * rows_per_out != M)))
        return 100;
    if (M <= 0 || N <= 0) return 0;
    if (K <= 0 || (K % 16) != 0) return 100;
    if (jpad != 0 && (epi == 0 || jpad < 0 || jpad > 64 || (jpad % 8) != 0 || subA == nullptr || subBT == nullptr ||
                      (reinterpret_cast<uintptr_t>(subA) & 15) != 0 || (reinterpret_cast<uintptr_t>(subBT) & 15) != 0))
        return 100;
    if (jcount != nullptr && (jpad != 64 || cols == nullptr || A == nullptr)) return 100;
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
    p.jcount = jcount;
    p.cols = cols;
    p.A = A;
    p.CB = weights;
    if (n_outs > 0) {
        I8MultiParams pm{};
        static_cast<I8Params&>(pm) = p;
        for (int d = 0; d < n_outs; ++d) pm.outs[d] = outs[d];
        pm.n_outs = n_outs;
        pm.rows_per_out = rows_per_out;
        if (epi == 0) return launch_i8<0, 0, false, true>(ta, tb, pm, stream);
#define BNB200_I8_MULTI(E)                                                                                             \
        if (jpad == 0) return launch_i8<E, 0, false, true>(ta, tb, pm, stream);                                         \
        if (jpad <= 8) return launch_i8<E, 8, false, true>(ta, tb, pm, stream);                                         \
        if (jpad <= 16) return launch_i8<E, 16, false, true>(ta, tb, pm, stream);                                       \
        if (jpad <= 32) return launch_i8<E, 32, false, true>(ta, tb, pm, stream);                                       \
        return launch_i8<E, 64, false, true>(ta, tb, pm, stream);
        if (epi == 1) {
            BNB200_I8_MULTI(1)
        }
        BNB200_I8_MULTI(2)
#undef BNB200_I8_MULTI
    }
    if (jcount != nullptr)
        return epi == 1 ? launch_i8<1, 64, true>(ta, tb, p, stream) : launch_i8<2, 64, true>(ta, tb, p, stream);
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

// The grouped int8 GEMM of a mixture-of-experts layer (epi 1 fp16 / 2 bf16): out[m, n] (row stride N) = the fused
// epilogue of launch_int8_gemm with SCB / bias at e * N + n for the rows of expert e, end_{e-1} <= m < end_e, and +0 for
// the rows past end_{E-1}.  CB [E * N, K] and SCB [E * N] are the experts' weights stacked; offs[E] the end rows
// (int32, on the device), clamped as end_e = min(max(offs[e], end_{e-1}), M).  With count set (the outlier term): count[E]
// and cols[E, K] the per-expert outlier counts and ascending lists, subA [M, 64] each row's own expert's first 64
// outlier columns, subBT [E * N, 64] each expert's dequantised weight columns, A [M, K] the activations for the columns
// past 64.  Returns 0, or 100 with nothing launched for what the instances do not serve; a failed launch returns 1 with
// the error message set.
int launch_int8_gemm_grouped(const int8_t* CA, const int8_t* CB, void* out, const float* SCA, const float* SCB,
                             const void* bias, const int* offs, int E, int M, int N, int K, int epi, const void* A,
                             const void* subA, const void* subBT, const int* cols, const int* count,
                             cudaStream_t stream) {
    if (epi != 1 && epi != 2) return 100;
    if (E < 1 || E > kMaxExperts || N <= 0 || (long long)E * N > 0x7fffffffLL || K <= 0 || (K % 16) != 0) return 100;
    if (count != nullptr && (cols == nullptr || A == nullptr || subA == nullptr || subBT == nullptr ||
                             (reinterpret_cast<uintptr_t>(subA) & 15) != 0 ||
                             (reinterpret_cast<uintptr_t>(subBT) & 15) != 0))
        return 100;
    if ((reinterpret_cast<uintptr_t>(CA) & 15) != 0 || (reinterpret_cast<uintptr_t>(CB) & 15) != 0) return 100;
    if (M <= 0) return 0;
    CUtensorMap ta, tb;
    if (!encode_tmap_2d(&ta, CA, 1, 128, (uint64_t)M, (uint64_t)K, (uint64_t)K, kI8TileM, kI8BK)) return 100;
    if (!encode_tmap_2d(&tb, CB, 1, 128, (uint64_t)E * N, (uint64_t)K, (uint64_t)K, kI8TileN, kI8BK)) return 100;
    I8GroupedParams p{};
    p.out = out;
    p.SCA = SCA;
    p.SCB = SCB;
    p.bias = bias;
    p.M = M;
    p.N = N;
    p.K = K;
    p.ldc = N;
    p.offs = offs;
    p.E = E;
    if (count != nullptr) {
        p.subA = subA;
        p.subBT = subBT;
        p.jpad = 64;
        p.jcount = count;
        p.cols = cols;
        p.A = A;
        p.CB = CB;
        return epi == 1 ? launch_i8<1, 64, true, false, true>(ta, tb, p, stream)
                        : launch_i8<2, 64, true, false, true>(ta, tb, p, stream);
    }
    return epi == 1 ? launch_i8<1, 0, false, false, true>(ta, tb, p, stream)
                    : launch_i8<2, 0, false, false, true>(ta, tb, p, stream);
}

} // namespace bnb200
