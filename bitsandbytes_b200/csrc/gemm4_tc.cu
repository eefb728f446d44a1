// gemm4_tc.cu -- NF4/FP4 dequant-fused GEMM on Hopper warpgroup tensor cores (wgmma, sm_90a).
//
// Replaces the reference's mma.sync kernel gemm_4bit_sm80_m16n8k16 (reference
// csrc/gemm_4bit_sm80.cu:127-457) and the dequantize + cuBLAS fallback the reference takes for
// M > 4 (reference bitsandbytes/backends/cuda/ops.py:617-623, 904-916).  Contract (reference
// _ops.py:239-295, gemm_4bit_mma.cuh:99-101):
//
//     out[m, n] = T( sum_k X[m, k] * W_T[n, k]  (fp32 accumulate)  + bias[n] )
//     W_T[n, k] = rn_T( value(code[n, k]) * scale[(n*K + k) / blocksize] )      (one rounding)
//     scale[i]  = absmax[i]                                       (plain)
//               = absmax_code[absmax_8bit[i]] * absmax[i >> 8] + offset   (double quant)
//
// Design ("swap-AB, weights through registers"):
//   * The wgmma M dimension (64 rows per warpgroup, two warpgroups) carries the OUTPUT FEATURES n;
//     the tokens m are the wgmma N dimension (MT = 16..256).  A CTA owns out[m0:m0+MT, n0:n0+128].
//   * A pipeline stage is BK k-elements (128; 64 at MT = 256).  A producer thread stages with TMA, per stage,
//     the packed codes of the CTA's 128 rows (128 x BK/2 bytes, BK/2-byte swizzle) and the activation tile
//     X[m0:m0+MT, k0:k0+BK] (BK/64 128-byte-swizzled sub-tiles), the K-major B operand of wgmma.
//   * Every consumer thread reads the codes of its two rows for the whole stage (ld.shared, 16 bytes per
//     32 codes) and decodes them straight into the register fragment of wgmma's A operand, with the exact
//     reference rounding -- a per-block 16-entry table built with 16 FMUL + 8 cvt.rn, once per (row,
//     quantisation block) in the stage, and looked up with PRMT only.  The decoded weights never pass
//     through shared memory, whose bandwidth is then left to the activation operand.
//   * Two A-fragment register sets alternate between stages, so the decode of stage i+1 overlaps the
//     wgmma of stage i (wgmma.wait_group 1 before a set is overwritten).
//   * Accumulators live in registers; the epilogue adds the bias, rounds to T, stages the tile in shared
//     memory and stores it in 16-byte row pieces, or -- for split-K, which fills the 132 SMs when the tile
//     grid is small -- writes fp32 partials to an L2-resident workspace with a last-arriver reduction in
//     deterministic split order.
//
// 384 threads = a producer warpgroup (one thread issues every TMA load of the ring) and two consumer warpgroups
// (decode + wgmma + epilogue).  Launch bounds allow 168 registers per thread; the producer gives registers back
// (setmaxnreg.dec to 40) and the consumers take them (setmaxnreg.inc to 232), which the 256-token tile needs (128
// accumulators, two A-fragment sets, the decode state).  The grid is persistent: min(units, SMs) CTAs, each running
// every gridDim-th (tile, K split) unit, with the ring's slot and phase carried across units, so the producer loads
// the next tile while the consumers run the epilogue.  (Measured on an H100: the persistent loop itself is neutral;
// it is kept because the one-tile-per-CTA form of this kernel makes ptxas spill at MT = 256.)
//
// T = float is the TF32 instance (fp32 activations when the caller allows TF32): wgmma k8 steps on TF32 operands,
// weights rna_tf32(fp32 dequantised weight) decoded by decode_word_tf32, 64-deep stages of fp32 activations, MT <= 128,
// an fp32 epilogue that adds the bias and rounds nothing.
//
// QT = kDecoded is the staged instance of the large-M route (launch_gemm4_staged, below): the weights arrive already
// decoded, as a [N, K] panel that the producer loads like the activations, and both wgmma operands come from shared
// memory.
//
// PART is the partial instance (cbnb_b200_gemm_4bit_partial, a row-sharded layer's K slice): the output and its
// copies are fp32, and the epilogue stores the accumulators -- the split order's sums under split-K -- with no bias
// and no rounding, straight from the fragments.  With rows_per_out > 0 (cbnb_b200_gemm_4bit_partial_scatter, a
// sequence-parallel layer) each output row goes to one copy only, the one of the rank that owns the token.
// GROUPED && PART is the grouped partial instance (cbnb_b200_gemm_4bit_grouped_partial, a row-sharded expert layer):
// each expert's fp32 rows, masked at the expert's end row, and fp32 zeros in the tail rows.
#include "common.cuh"
#include "decode4.cuh"
#include "hopper_ptx.cuh"

#include <cstdlib>
#include <mutex>
#include <type_traits>

namespace bnb200 {

// blockwise.cu: rows [n0, n0 + rows) of a 4-bit weight decoded to T, bit-identical to F.dequantize_4bit
template <typename T>
void launch_dequantize4_panel(const uint8_t* codes, const float* absmax, const uint8_t* absmax_8bit,
                              const float* absmax_code, const float* absmax_offset, T* out, int blocksize,
                              int quant_type, int n0, int rows, int K, cudaStream_t stream);

namespace {

constexpr int kTileN = 128;        // output features per CTA (two warpgroups of 64)
constexpr int kConsumers = 256;    // threads of the two consumer warpgroups
constexpr int kThreads = 128 + kConsumers;  // producer warpgroup + consumers
// per-thread registers after the hand-off: 128 x 40 + 256 x 232 <= 64K, the SM's register file
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
static_assert(128 * kProducerRegs + kConsumers * kConsumerRegs <= 65536, "register hand-off exceeds the SM");
constexpr int kBarEpi = 1;    // named barrier of the consumers' epilogue
// QT of the staged instance: the weights arrive already decoded to T, a [N, K] panel (launch_gemm4_staged)
constexpr int kDecoded = -1;

struct Gemm4Params {
    const uint8_t* B;            // packed codes [N, K/2]
    const float* absmax;         // fp32 per block, or level-2 absmax when nested
    const uint8_t* absmax_8bit;  // NULL unless double quant
    const float* absmax_code;    // 256-entry code for absmax_8bit
    const float* absmax_offset;  // scalar
    const void* bias;            // T[N] or NULL
    void* out;                   // T[M, ldc]
    void* peer_out[7];           // further copies of the output tile (peer GPUs' gather buffers, same ldc): the
    int n_peers;                 //   epilogue stores every element to all of them (fused all-gather)
    int out_vec;                 // every output base is 16-byte aligned and ldc % 8 == 0: 16-byte stores
    float* ws_partial;           // split-K partials [tiles][splits][MT][128]
    int* ws_counter;             // two per output tile, zero on entry, reset on exit
    int M, N, K, ldc;
    int log2_bs;
    int scale_mask;              // a new quantisation block can start only at 32-code chunks q with (q & mask) == 0
    int kblocks_total;           // number of stages = ceil(K / BK)
    int n_tiles;                 // N tiles of 128 (tile = m_tile * n_tiles + n_tile)
    int tiles_total;
    int splits;                  // K splits per tile (1 = none)
    int rows_per_out;            // PART only: 0 = every row to out and the peers; > 0 = row m to copy m / rows_per_out
                                 //   (0 = out, d = peer_out[d - 1]) at row m % rows_per_out (OutList::rows_per_out)
    // GROUPED only: B is E experts' [N, K] weights stacked ([E * N, K / 2] codes, N per expert), and the activation
    // rows of expert e are [end_{e-1}, end_e), end_e = min(max(offs[e], end_{e-1}), M) read on the device
    const int* offs;
    int E;
};

// The grouped instances (GROUPED = true) serve 1 <= E <= kMaxExperts experts per launch: their group table (the
// clamped end row and the exclusive prefix of the m-tile counts of every expert, plus the scan's per-warp totals) sits
// in shared memory past the barriers.
constexpr int kGroupTabBytes = (2 * kMaxExperts + 1 + 2 * kThreads / 32) * 4;

// The partial instances' store of element (m, n) of the fp32 output (m < M, n < N), routed as p.rows_per_out says.
__device__ __forceinline__ void store_partial(const Gemm4Params& p, int m, int n, float v) {
    if (p.rows_per_out > 0) {
        const int d = m / p.rows_per_out;
        float* dst = reinterpret_cast<float*>(d == 0 ? p.out : p.peer_out[d - 1]);
        dst[(long long)(m - d * p.rows_per_out) * p.ldc + n] = v;
    } else {
        const long long o = (long long)m * p.ldc + n;
        reinterpret_cast<float*>(p.out)[o] = v;
        for (int r = 0; r < p.n_peers; ++r) reinterpret_cast<float*>(p.peer_out[r])[o] = v;
    }
}

// the staged instance: D[64 x MT] += A[64 x 16] * X[MT x 16]^T with both operands from descriptors
template <typename T, int MT>
__device__ __forceinline__ void wgmma_step_ss(float (&d)[MT / 2], uint64_t a_desc, uint64_t b_desc) {
    constexpr bool bf = std::is_same<T, __nv_bfloat16>::value;
    static_assert(MT == 128 || MT == 256, "staged token tile");
    if constexpr (MT == 128) {
        if constexpr (bf) ptx::wgmma_m64n128k16_bf16_ss(d, a_desc, b_desc); else ptx::wgmma_m64n128k16_f16_ss(d, a_desc, b_desc);
    } else {
        if constexpr (bf) ptx::wgmma_m64n256k16_bf16_ss(d, a_desc, b_desc); else ptx::wgmma_m64n256k16_f16_ss(d, a_desc, b_desc);
    }
}

// one k16 step of a 64-row warpgroup tile: D[64 x MT] += A[64 x 16] (registers) * X[MT x 16]^T (descriptor)
// (T = float: one k8 step with TF32 operands)
template <typename T, int MT>
__device__ __forceinline__ void wgmma_step(float (&d)[MT / 2], const uint32_t (&a)[4], uint64_t b_desc) {
    constexpr bool bf = std::is_same<T, __nv_bfloat16>::value;
    if constexpr (std::is_same<T, float>::value) {
        static_assert(MT <= 128, "TF32 token tile");
        if constexpr (MT == 16) ptx::wgmma_m64n16k8_tf32_rs(d, a, b_desc);
        else if constexpr (MT == 32) ptx::wgmma_m64n32k8_tf32_rs(d, a, b_desc);
        else if constexpr (MT == 64) ptx::wgmma_m64n64k8_tf32_rs(d, a, b_desc);
        else ptx::wgmma_m64n128k8_tf32_rs(d, a, b_desc);
    } else if constexpr (MT == 16) {
        if constexpr (bf) ptx::wgmma_m64n16k16_bf16_rs(d, a, b_desc); else ptx::wgmma_m64n16k16_f16_rs(d, a, b_desc);
    } else if constexpr (MT == 32) {
        if constexpr (bf) ptx::wgmma_m64n32k16_bf16_rs(d, a, b_desc); else ptx::wgmma_m64n32k16_f16_rs(d, a, b_desc);
    } else if constexpr (MT == 64) {
        if constexpr (bf) ptx::wgmma_m64n64k16_bf16_rs(d, a, b_desc); else ptx::wgmma_m64n64k16_f16_rs(d, a, b_desc);
    } else if constexpr (MT == 128) {
        if constexpr (bf) ptx::wgmma_m64n128k16_bf16_rs(d, a, b_desc); else ptx::wgmma_m64n128k16_f16_rs(d, a, b_desc);
    } else {
        static_assert(MT == 256, "token tile");
        if constexpr (bf) ptx::wgmma_m64n256k16_bf16_rs(d, a, b_desc); else ptx::wgmma_m64n256k16_f16_rs(d, a, b_desc);
    }
}

// Pipeline stage = BK k-elements: BK/kSubK activation sub-tiles of 128-byte rows (the swizzle atom: 64 16-bit or 32
// fp32 elements) and the packed codes of 128 rows.  The 256-token tile takes 64-deep stages: a 128-deep one (72 KB)
// leaves room for two stages only, and two 128-deep A-fragment sets (64 registers) next to its 128 accumulators would
// not fit the consumers' register budget.  The TF32 instance (T = float) takes 64-deep stages at every tile: eight k8
// steps, so its two A-fragment sets are the 64 registers of the 16-bit kernel's 128-deep ones.  The epilogue stages
// the output tile in a buffer of its own (the producer is already filling the ring for the CTA's next tile), and the
// ring takes as many stages as fit next to it, at most 8.
// The staged instance (SS) loads a [128 x 64] tile of the decoded weight panel per stage (128-byte rows, 128-byte
// swizzle: the K-major A operand of wgmma) and stages the epilogue in slices of 64 tokens, so that the 256-token tile
// keeps four 48 KB stages (its whole 68 KB tile next to them leaves room for three).
template <typename T, int MT, bool SS = false> struct StageCfg {
    static constexpr bool kTf32 = std::is_same<T, float>::value;
    static constexpr int kBK = (MT == 256 || kTf32 || SS) ? 64 : 128;
    static constexpr int kSteps = kBK / (kTf32 ? 8 : 16);       // wgmma k16 (k8 for TF32) steps
    static constexpr int kChunks = kBK / 32;                     // 16-byte (32-code) pieces of a code row
    static constexpr int kSubK = 128 / (int)sizeof(T);           // k-elements of one sub-tile row
    static constexpr int kXSubBytes = MT * 128;                  // one sub-tile
    static constexpr int kXStageBytes = (kBK / kSubK) * kXSubBytes;
    static constexpr int kWRowBytes = SS ? kBK * (int)sizeof(T)  // decoded weights of one row (128 bytes)
                                         : kBK / 2;              // packed codes of one row (TMA, kWRowBytes-byte swizzle)
    static constexpr int kWStageBytes = kTileN * kWRowBytes;
    static constexpr int kStageBytes = kXStageBytes + kWStageBytes;
    // epilogue staging: one output row of the tile (128 x T) plus 16 bytes, so that the fragment stores (four
    // token rows two apart per warp instruction) fall on distinct banks
    static constexpr int kOutPitch = kTileN * (int)sizeof(T) + 16;
    static constexpr int kOutSlices = SS ? MT / 64 : 1;          // the tile is staged and stored in token slices
    static constexpr int kOutBytes = MT / kOutSlices * kOutPitch;
    static constexpr int kSlack = 1024 + 256;                    // base alignment + barriers
    static constexpr int kRing = (227 * 1024 - kSlack - kOutBytes) / kStageBytes;
    static constexpr int kStages = kRing > 8 ? 8 : kRing;
    static constexpr int kSmemBytes = kSlack + kStages * kStageBytes + kOutBytes;
    static_assert(kStages >= (SS ? 4 : 2) && kSmemBytes <= 227 * 1024, "shared memory");
};

// The 16 codes of a 16-byte chunk (stage-row words w[4q .. 4q+3]) that this thread's A fragments need (byte `t` of
// each, t = lane % 4): wgmma k16 step 2q+u reads byte t of words 4q+2u (k 2t, 2t+1) and 4q+2u+1 (k 8+2t, 9+2t).
__device__ __forceinline__ uint32_t gather_bytes(uint4 v, uint32_t sel) {
    return prmt(prmt(v.x, v.y, sel), prmt(v.z, v.w, sel), 0x5410);
}

// TF32: a k8 step is one word of the chunk (8 codes, word i = step 4q + i), of which thread t needs codes t and t + 4:
// byte t/2 and byte t/2 + 2, the high nibble for even t.  `sel` gathers those two bytes of words (x, y) and of
// (z, w); the code nibbles are then moved into one word: nibble n = 2j + h holds byte j of the h-th gathered pair,
// that is k8 step 4q + 2h + j/2 and k t + 4 (j & 1).  `shr` = 4 for even t, 0 for odd; `mul` = 1 << (4 - shr).
__device__ __forceinline__ uint32_t gather_nibbles(uint4 v, uint32_t sel, uint32_t shr, uint32_t mul) {
    const uint32_t r0 = prmt(v.x, v.y, sel) >> shr;
    const uint32_t r1 = prmt(v.z, v.w, sel) * mul;
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, 0x0F0F0F0F, 0xE4;" : "=r"(r) : "r"(r0), "r"(r1));  // (r0 & m) | (r1 & ~m)
    return r;
}

// GROUPED: the group table, past the barriers' 256 bytes of the shared memory: gend[e] = end_e, then gtp[e] = the m-tiles
// of experts 0..e-1 (gtp[E] = all of them), then the scan's per-warp totals.  (Taken where it is used: a table pointer
// held across the kernel changes cicc's register moves in the other instances.)
template <typename Cfg> __device__ __forceinline__ int* group_table(uint8_t* so) {
    return reinterpret_cast<int*>(so + Cfg::kOutBytes + 256);
}

// GROUPED: the number of units, gtp[E] m-tiles times the n-tiles.  Each role reads it from the table after its register
// hand-off (a volatile read, which stays there): held from the table build on, across the hand-off, it cost the
// plain-statistics MT = 64 instances a spill.
template <typename Cfg> __device__ __forceinline__ int grouped_units(uint8_t* so, const Gemm4Params& p) {
    return *reinterpret_cast<const volatile int*>(group_table<Cfg>(so) + kMaxExperts + p.E) * p.n_tiles;
}

template <typename T, int QT, int MT, bool DQ, bool PART, bool GROUPED = false>
__global__ void __launch_bounds__(kThreads, 1)
    gemm4_tc_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                    const Gemm4Params p) {
    constexpr bool kSS = QT == kDecoded;  // the staged instance: weights from a decoded panel, no decode here
    using Cfg = StageCfg<T, MT, kSS>;
    constexpr bool kTf32 = Cfg::kTf32;
    constexpr int kBK = Cfg::kBK;
    constexpr int kSteps = Cfg::kSteps;
    constexpr int kChunks = Cfg::kChunks;
    constexpr int kStages = Cfg::kStages;
    constexpr int kXSubBytes = Cfg::kXSubBytes;
    constexpr int kXStageBytes = Cfg::kXStageBytes;
    constexpr int kWRowBytes = Cfg::kWRowBytes;
    constexpr int kWStageBytes = Cfg::kWStageBytes;

    // ------------------------------------------------------------------ shared memory
    // aligned by an offset from the __shared__ array itself, so that the compiler keeps the shared address space
    // (ld.shared for the codes, not generic loads)
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sx = smem;                              // [kStages][BK/kSubK][MT x 128 B] activations
    uint8_t* sw = smem + kStages * kXStageBytes;     // [kStages][128 x BK/2 B]        packed codes (SS: 128 x 128 B)
    uint8_t* so = smem + kStages * Cfg::kStageBytes; // [MT][kOutPitch]                epilogue staging
    uint64_t* bars = reinterpret_cast<uint64_t*>(so + Cfg::kOutBytes);
    uint64_t* full = bars;                   // [kStages] TMA (1 arrive + bytes) -> consumers
    uint64_t* empty = bars + kStages;        // [kStages] the 8 consumer warps -> producer (slot free for the next load)

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // Work units u = (tile, K split), ordered (tile, split); tile = m_tile * n_tiles + n_tile.  A CTA runs units
    // blockIdx.x, blockIdx.x + gridDim.x, ...; a split launch is one wave, one unit per CTA.
    // GROUPED: no K split; m_tile counts the m-tiles of all experts in expert order (expert e's j-th m-tile starts at
    // row end_{e-1} + j * MT), and the number of units is known once the group table is built.
    const int splits = GROUPED ? 1 : p.splits;
    int units = p.tiles_total * splits;
    const int per = (p.kblocks_total + splits - 1) / splits;
    struct Unit {
        int tile, split, n0, m0, st_begin, nst;
        int m_end, wrow;  // GROUPED: the expert's end row, and its first row of the stacked weight (e * N)
    };
    auto unit_at = [&](int u) {
        Unit w;
        w.tile = u / splits;
        w.split = u - w.tile * splits;
        w.n0 = (w.tile % p.n_tiles) * kTileN;
        w.m0 = (w.tile / p.n_tiles) * MT;
        if constexpr (GROUPED) {
            // the expert of m-tile g: the last e with gtp[e] <= g, which has m-tiles since g < gtp[E]
            const int g = w.tile / p.n_tiles;
            const int* gend = group_table<Cfg>(so);
            const int* gtp = gend + kMaxExperts;
            int lo = 0;
#pragma unroll
            for (int step = kMaxExperts / 2; step >= 1; step >>= 1)
                if (lo + step < p.E && gtp[lo + step] <= g) lo += step;
            w.m0 = (lo > 0 ? gend[lo - 1] : 0) + (g - gtp[lo]) * MT;
            w.m_end = gend[lo];
            w.wrow = lo * p.N;
        }
        w.st_begin = w.split * per;
        const int st_end = w.st_begin + per < p.kblocks_total ? w.st_begin + per : p.kblocks_total;
        w.nst = st_end - w.st_begin;  // >= 1 by construction
        return w;
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            ptx::mbar_init(&full[s], 1);
            ptx::mbar_init(&empty[s], kConsumers / 32);
        }
        ptx::fence_barrier_init();
    }
    if constexpr (GROUPED) {
        // The group table, built by the whole CTA before the role split (every CTA builds the same one): thread t
        // takes experts [t * kPer, t * kPer + kPer).  end_e = min(M, max(0, offs[0..e])) -- the clamp of the
        // contract, as a prefix maximum -- then the m-tile counts ceil((end_e - end_{e-1}) / MT) and their
        // exclusive prefix sum, each scan over the warp by shuffles and across the 12 warps through shared memory.
        constexpr int kPer = (kMaxExperts + kThreads - 1) / kThreads;
        constexpr int kWarps = kThreads / 32;
        int* gend = group_table<Cfg>(so);
        int* gtp = gend + kMaxExperts;
        static_assert(kMaxExperts <= (kThreads - 1) * kPer, "the last thread must hold no expert");
        int* wtot = gtp + kMaxExperts + 1;  // [kWarps] maxima, then [kWarps] tile counts
        const int e0 = threadIdx.x * kPer;
        int v[kPer];
        int run = 0;
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            v[i] = e0 + i < p.E ? max(__ldg(p.offs + e0 + i), 0) : 0;
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
        int prev = min(r, p.M);
        int cnt[kPer], tiles = 0;
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            r = max(r, v[i]);
            v[i] = min(r, p.M);  // end_e (experts past E: end_{E-1}, no rows)
            cnt[i] = (v[i] - prev + MT - 1) / MT;
            prev = v[i];
            tiles += cnt[i];
        }
        int incs = tiles;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, incs, d);
            if (lane >= d) incs += o;
        }
        if (lane == 31) wtot[kWarps + warp] = incs;
        __syncthreads();
        int base = incs - tiles;
        for (int w2 = 0; w2 < warp; ++w2) base += wtot[kWarps + w2];
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            if (e0 + i < p.E) {
                gend[e0 + i] = v[i];
                gtp[e0 + i] = base;
            }
            base += cnt[i];
        }
        if (threadIdx.x == kThreads - 1) gtp[p.E] = base;  // the last thread's experts are past E: base is the total
    }
    __syncthreads();

    // The ring runs continuously over the CTA's units: its slot and phase carry from one unit to the next.
    // ====================================================================== producer (warpgroup 0)
    // (the role test is made provably warp-uniform, as setmaxnreg requires of the whole warpgroup)
    if (__shfl_sync(0xffffffffu, threadIdx.x / 128, 0) == 0) {
        ptx::setmaxnreg_dec<kProducerRegs>();
        if constexpr (GROUPED) units = grouped_units<Cfg>(so, p);
        if (threadIdx.x == 0) {
            ptx::prefetch_tmap(&tmap_x);
            ptx::prefetch_tmap(&tmap_w);
            int slot = 0;
            uint32_t phase = 0;  // parity of the slot's current round
            bool wrapped = false;
            for (int u = blockIdx.x; u < units; u += gridDim.x) {
                const Unit w = unit_at(u);
                for (int j = 0; j < w.nst; ++j) {
                    // the slot's previous load has been consumed by all 8 consumer warps
                    if (wrapped) ptx::mbar_wait(&empty[slot], phase ^ 1u);
                    const int k0 = (w.st_begin + j) * kBK;
                    ptx::mbar_arrive_expect_tx(&full[slot], kWStageBytes + kXStageBytes);
                    // rows past M, rows past N and columns past K are out of bounds for the tensor maps: TMA
                    // zero-fills.  Packed codes of the tile's 128 output features: bytes [k0/2, k0/2 + BK/2).
                    // (GROUPED: rows of the expert's stacked weight; a tile reaching past its N features loads the
                    // next expert's codes, which the consumers give zero scales and the epilogue never stores)
                    ptx::tma_load_2d(sw + slot * kWStageBytes, &tmap_w, &full[slot], kSS ? k0 : k0 / 2,
                                     GROUPED ? w.wrow + w.n0 : w.n0);
#pragma unroll
                    for (int h = 0; h < kBK / Cfg::kSubK; ++h)
                        ptx::tma_load_2d(sx + slot * kXStageBytes + h * kXSubBytes, &tmap_x, &full[slot],
                                         k0 + Cfg::kSubK * h, w.m0);
                    if (++slot == kStages) {
                        slot = 0;
                        phase ^= 1u;
                        wrapped = true;
                    }
                }
            }
        }
        return;
    }

    // ====================================================================== consumers (warpgroups 1, 2)
    ptx::setmaxnreg_inc<kConsumerRegs>();
    if constexpr (GROUPED) units = grouped_units<Cfg>(so, p);
    const int ct = threadIdx.x - 128;         // consumer thread 0..255
    const int wg = ct >> 7;                   // consumer warpgroup: feature rows [64 wg, 64 wg + 64) of the tile
    const int g = lane >> 2, t = lane & 3;
    const int row0 = wg * 64 + (warp & 3) * 16 + g;  // this thread's two rows: row0, row0 + 8
    const ScaleSrc sc{p.absmax, p.absmax_8bit, p.absmax_code, (DQ && p.absmax_offset) ? __ldg(p.absmax_offset) : 0.0f};
    const uint32_t sel = (uint32_t)t | ((uint32_t)(t + 4) << 4);
    const uint32_t smask = (uint32_t)p.scale_mask;
    // the TMA swizzle of the code rows: 16-byte chunk c of row r sits at chunk c ^ ((r * kWRowBytes / 128) % kChunks)
    const uint32_t swz[2] = {(uint32_t)((row0 * kWRowBytes) >> 7) & (kChunks - 1),
                             (uint32_t)(((row0 + 8) * kWRowBytes) >> 7) & (kChunks - 1)};

    int slot = 0;
    uint32_t phase = 0;
    for (int u = blockIdx.x; u < units; u += gridDim.x) {
        const Unit w = unit_at(u);
        const int n0 = w.n0, m0 = w.m0, st_begin = w.st_begin, nst = w.nst;
        const int na = n0 + row0, nb = na + 8;
        const bool a_ok = na < p.N, b_ok = nb < p.N;
        // scale element base of the row: GROUPED counts from the start of the stacked weight, (e * N + n) * K
        const long long e_a = (long long)((GROUPED ? w.wrow : 0) + (a_ok ? na : 0)) * p.K;
        const long long e_b = (long long)((GROUPED ? w.wrow : 0) + (b_ok ? nb : 0)) * p.K;

        // Scales of one stage, one per (row, quantisation block): the 32 codes of a chunk lie inside one block (blocks
        // are >= 32 and aligned), and a block can begin only at a chunk q with (q & smask) == 0.  Fetched one stage ahead.
        float scl[2][kChunks];
        auto fetch = [&](int i) {
            const long long kk = (long long)(st_begin + i) * kBK;
#pragma unroll
            for (int q = 0; q < kChunks; ++q) {
                if ((q & smask) == 0) {
                    const bool in_k = i < nst && kk + 32 * q < p.K;
                    scl[0][q] = (in_k && a_ok) ? sc.load_as<DQ>((e_a + kk + 32 * q) >> p.log2_bs) : 0.f;
                    scl[1][q] = (in_k && b_ok) ? sc.load_as<DQ>((e_b + kk + 32 * q) >> p.log2_bs) : 0.f;
                }
            }
        };

        float acc[MT / 2];
#pragma unroll
        for (int j = 0; j < MT / 2; ++j) acc[j] = 0.f;

        uint32_t afr[2][kSteps][4];  // two A-fragment sets: [set][k16 step][reg]

        // decode stage i (smem stage s) into A set `a`: all of the stage's code loads first, then the tables and PRMTs
        auto decode = [&](int s, uint32_t (&a)[kSteps][4]) {
            const uint8_t* wt = sw + s * kWStageBytes;
            uint4 v[2][kChunks];
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int q = 0; q < kChunks; ++q)
                    v[r][q] = *reinterpret_cast<const uint4*>(wt + (row0 + 8 * r) * kWRowBytes + (((uint32_t)q ^ swz[r]) << 4));
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                if constexpr (kTf32) {
                    // gather_nibbles: bytes t/2 and t/2 + 2 of two words, the high nibble for even t
                    const uint32_t tsel = (uint32_t)(t >> 1) * 0x1111u + 0x6420u;
                    const uint32_t tshr = (t & 1) ? 0u : 4u;
                    const uint32_t tmul = (t & 1) ? 16u : 1u;
                    DecodeTableTf32 tab;
#pragma unroll
                    for (int q = 0; q < kChunks; ++q) {
                        if ((q & smask) == 0) build_table_tf32<QT>(scl[r][q], tab);
                        uint32_t o[8];
                        decode_word_tf32(gather_nibbles(v[r][q], tsel, tshr, tmul), tab, o);
                        // o[n]: k8 step 4q + 2(n & 1) + n/4, k t + 4((n >> 1) & 1) -> register r (k t) or 2 + r (t + 4)
#pragma unroll
                        for (int n = 0; n < 8; ++n) a[4 * q + 2 * (n & 1) + (n >> 2)][r + 2 * ((n >> 1) & 1)] = o[n];
                    }
                } else {
                    DecodeTable tab;
#pragma unroll
                    for (int q = 0; q < kChunks; ++q) {
                        if ((q & smask) == 0) build_table<T, QT>(scl[r][q], tab);
                        uint32_t o[4];
                        decode_word(gather_bytes(v[r][q], sel), tab, o);
                        // o[i]: byte i of the gathered word = word 4q+i of the row -> k16 step 2q + i/2, half i%2
#pragma unroll
                        for (int u = 0; u < 2; ++u) {
                            a[2 * q + u][r] = o[2 * u];          // rows g / g+8, k 2t..2t+1
                            a[2 * q + u][2 + r] = o[2 * u + 1];  // rows g / g+8, k 8+2t..9+2t
                        }
                    }
                }
            }
        };

        // a k16 step (k8 for TF32) is 32 bytes of an activation row: four per 128-byte sub-tile row
        auto mma_stage = [&](int s, const uint32_t (&a)[kSteps][4]) {
            const uint32_t xs = ptx::smem_u32(sx + s * kXStageBytes);
            ptx::wgmma_fence();
            if constexpr (kSS) {
                // this warpgroup's 64 weight rows: 8 KB into the stage's tile, a 1024-byte-aligned swizzle atom group
                const uint64_t a_desc = ptx::make_sw128_kmajor_desc(ptx::smem_u32(sw + s * kWStageBytes + wg * 64 * 128));
#pragma unroll
                for (int j = 0; j < kSteps; ++j)
                    wgmma_step_ss<T, MT>(acc, a_desc + 2 * j, ptx::make_sw128_kmajor_desc(xs) + 2 * j);
            } else {
#pragma unroll
                for (int j = 0; j < kSteps; ++j)
                    wgmma_step<T, MT>(acc, a[j], ptx::make_sw128_kmajor_desc(xs + (j >> 2) * kXSubBytes) + 2 * (j & 3));
            }
            ptx::wgmma_commit();
        };

        if constexpr (!kSS) fetch(0);
        int prev_s = -1;
        for (int i0 = 0; i0 < nst; i0 += 2) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = i0 + h;
                if (i < nst) {
                    const int s = slot;
                    ptx::mbar_wait(&full[s], phase);
                    if (++slot == kStages) {
                        slot = 0;
                        phase ^= 1u;
                    }
                    if constexpr (!kSS) {
                        decode(s, afr[h]);
                        fetch(i + 1);
                    }
                    mma_stage(s, afr[h]);
                    // the wgmma group of the previous stage has completed: its activation tile (and its A set) are free
                    ptx::wgmma_wait<1>();
                    if (prev_s >= 0) {
                        __syncwarp();
                        if (lane == 0) ptx::mbar_arrive(&empty[prev_s]);
                    }
                    prev_s = s;
                }
            }
        }
        ptx::wgmma_wait<0>();
#pragma unroll
        for (int j = 0; j < MT / 2; ++j) ptx::fence_operand(acc[j]);
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty[prev_s]);

        // ================================================================== epilogue
        // acc[4j + e]: feature row row0 + 8 * (e >= 2), token column 8j + 2t + (e & 1)
        T* outp = reinterpret_cast<T*>(p.out);
        if constexpr (PART && GROUPED) {
            // One destination, no scatter.  Rows past the expert's end belong to a later expert or to the tail and
            // were computed with this expert's weights: they are left to the unit (or the tail loop) that owns them.
            // The unit is looked up again here for the reason given at the rounded epilogue below, and the rows are
            // addressed from this thread's first one: with the absolute row of every store, ptxas spilled 8 to 12
            // bytes in the MT = 128 instances.
            const Unit we = unit_at(u);
            const int lim = we.m_end - we.m0 - 2 * t;  // tile row 8j + 2t + (e & 1) is stored when 8j + (e & 1) < lim
            float* dst = reinterpret_cast<float*>(p.out) + (long long)(we.m0 + 2 * t) * p.ldc;
#pragma unroll
            for (int j = 0; j < MT / 8; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int n = e >= 2 ? nb : na;
                    if (8 * j + (e & 1) < lim && n < p.N) dst[(long long)(8 * j + (e & 1)) * p.ldc + n] = acc[4 * j + e];
                }
            continue;
        } else if constexpr (PART) {
            // a warp instruction stores four 32-byte row pieces: whole sectors, without the staging buffer, which at
            // fp32 would not fit next to the 256-token tile's ring
            if (splits == 1) {
                // When every row of the tile goes to one destination (one destination; or, scattered, a tile inside
                // one rank's tokens) its base is found once per tile, not per element as store_partial does.
                float* dst = nullptr;
                long long dst_off = 0;
                if (p.rows_per_out == 0) {
                    if (p.n_peers == 0) dst = reinterpret_cast<float*>(p.out);
                } else {
                    const int d = m0 / p.rows_per_out;
                    if ((min(m0 + MT, p.M) - 1) / p.rows_per_out == d) {
                        dst = reinterpret_cast<float*>(d == 0 ? p.out : p.peer_out[d - 1]);
                        dst_off = (long long)d * p.rows_per_out * p.ldc;
                    }
                }
#pragma unroll
                for (int j = 0; j < MT / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int m = m0 + 8 * j + 2 * t + (e & 1);
                        const int n = e >= 2 ? nb : na;
                        if (m < p.M && n < p.N) {
                            if (dst != nullptr) dst[(long long)m * p.ldc + n - dst_off] = acc[4 * j + e];
                            else store_partial(p, m, n, acc[4 * j + e]);
                        }
                    }
                continue;
            }
        }
        if (splits == 1) {
            const T* bias = reinterpret_cast<const T*>(p.bias);
            // (GROUPED: the expert's weight row base and end row are looked up again rather than held through the
            // main loop, where they would cost the plain-statistics instances a spill at MT = 64 and 128)
            const Unit we = GROUPED ? unit_at(u) : w;
            const float bias_a = (bias != nullptr && a_ok) ? DT<T>::to_f32(bias[(GROUPED ? we.wrow : 0) + na]) : 0.f;
            const float bias_b = (bias != nullptr && b_ok) ? DT<T>::to_f32(bias[(GROUPED ? we.wrow : 0) + nb]) : 0.f;
            // Stage the rounded tile as [token][feature] rows -- once both warpgroups are done reading the previous
            // unit's tile there -- then store it in 16-byte row pieces of kVec elements: each token row of the tile is
            // 128 contiguous elements of the output.  (fp32: the bias is added in fp32 and nothing is rounded.)
            constexpr int kPitch = Cfg::kOutPitch;
            constexpr int kVec = 16 / (int)sizeof(T);
            constexpr int kSliceT = MT / Cfg::kOutSlices;  // tokens per staged slice
            if constexpr (Cfg::kOutSlices == 1) {
                ptx::bar_sync(kBarEpi, kConsumers);
#pragma unroll
                for (int j = 0; j < MT / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        *reinterpret_cast<T*>(so + (8 * j + 2 * t + (e & 1)) * kPitch + (row0 + 8 * (e >> 1)) * (int)sizeof(T)) =
                            DT<T>::from_f32(acc[4 * j + e] + (e >= 2 ? bias_b : bias_a));
                ptx::bar_sync(kBarEpi, kConsumers);
                for (int idx = ct; idx < MT * (kTileN / kVec); idx += kConsumers) {
                    const int c = idx / (kTileN / kVec), n = n0 + kVec * (idx % (kTileN / kVec));
                    const int m = m0 + c;
                    // (GROUPED: rows past the expert's end are the next expert's, computed and discarded)
                    if (m >= (GROUPED ? we.m_end : p.M) || n >= p.N) continue;
                    const uint8_t* src = so + c * kPitch + (n - n0) * (int)sizeof(T);
                    const long long o = (long long)m * p.ldc + n;
                    if (p.out_vec && n + kVec <= p.N) {
                        const uint4 val = *reinterpret_cast<const uint4*>(src);
                        *reinterpret_cast<uint4*>(outp + o) = val;
                        for (int r = 0; r < p.n_peers; ++r) *reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.peer_out[r]) + o) = val;
                    } else {
                        for (int x = 0; x < kVec && n + x < p.N; ++x) {
                            const T val = reinterpret_cast<const T*>(src)[x];
                            outp[o + x] = val;
                            for (int r = 0; r < p.n_peers; ++r) reinterpret_cast<T*>(p.peer_out[r])[o + x] = val;
                        }
                    }
                }
            } else {
                // the staged instance: slices of kSliceT tokens (every j unrolled, the slice test predicated, so
                // that the accumulators stay in registers)
                for (int sl = 0; sl < Cfg::kOutSlices; ++sl) {
                    ptx::bar_sync(kBarEpi, kConsumers);
#pragma unroll
                    for (int j = 0; j < MT / 8; ++j) {
                        if (j / (kSliceT / 8) != sl) continue;
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            *reinterpret_cast<T*>(so + (8 * j - sl * kSliceT + 2 * t + (e & 1)) * kPitch +
                                                  (row0 + 8 * (e >> 1)) * (int)sizeof(T)) =
                                DT<T>::from_f32(acc[4 * j + e] + (e >= 2 ? bias_b : bias_a));
                    }
                    ptx::bar_sync(kBarEpi, kConsumers);
                    for (int idx = ct; idx < kSliceT * (kTileN / kVec); idx += kConsumers) {
                        const int c = idx / (kTileN / kVec), n = n0 + kVec * (idx % (kTileN / kVec));
                        const int m = m0 + sl * kSliceT + c;
                        if (m >= p.M || n >= p.N) continue;
                        const uint8_t* src = so + c * kPitch + (n - n0) * (int)sizeof(T);
                        const long long o = (long long)m * p.ldc + n;
                        if (p.out_vec && n + kVec <= p.N) {
                            const uint4 val = *reinterpret_cast<const uint4*>(src);
                            *reinterpret_cast<uint4*>(outp + o) = val;
                            for (int r = 0; r < p.n_peers; ++r) *reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.peer_out[r]) + o) = val;
                        } else {
                            for (int x = 0; x < kVec && n + x < p.N; ++x) {
                                const T val = reinterpret_cast<const T*>(src)[x];
                                outp[o + x] = val;
                                for (int r = 0; r < p.n_peers; ++r) reinterpret_cast<T*>(p.peer_out[r])[o + x] = val;
                            }
                        }
                    }
                }
            }
            continue;
        }

        // ---- split-K: every split CTA publishes its fp32 partial tile (layout [column m][row n], so that the
        // later reads are 128-byte coalesced), the splits of a tile rendezvous on a counter, and EACH of them then
        // reduces a 1/splits share of the columns (in split order: deterministic).  The launch is COOPERATIVE (all
        // CTAs of the <= one-wave grid are resident together), so the short wait cannot starve; it is bounded anyway.
        const int split = w.split;
        float* ws_tile = p.ws_partial + (long long)w.tile * splits * kTileN * MT;
        float* my = ws_tile + (long long)split * kTileN * MT;
#pragma unroll
        for (int j = 0; j < MT / 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) my[(8 * j + 2 * t + (e & 1)) * kTileN + row0 + 8 * (e >> 1)] = acc[4 * j + e];
        __threadfence();
        ptx::bar_sync(kBarEpi, kConsumers);
        int* arrive = p.ws_counter + w.tile;
        int* done = p.ws_counter + p.tiles_total + w.tile;
        if (ct == 0) {
            atomicAdd(arrive, 1);
            unsigned long long t0 = 0;
            unsigned spins = 0;
            while (atomicAdd(arrive, 0) < splits) {
                __nanosleep(64);
                if ((++spins & 0xFFF) == 0) {  // bounded: trap after 10 s instead of hanging the device (no printf:
                                               // a call would serialise the wgmma pipeline)
                    unsigned long long now;
                    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
                    if (t0 == 0) t0 = now;
                    else if (now - t0 > 10000000000ull) __trap();
                }
            }
            __threadfence();
        }
        ptx::bar_sync(kBarEpi, kConsumers);
        {
            const int e = ct;                        // 0..255 over the two consumer warpgroups
            const int rn = e & (kTileN - 1);         // output feature inside the tile
            const int cg = e >> 7;                   // 0..1
            const int nn = n0 + rn;
            float bias_r = 0.f;
            if (p.bias != nullptr && nn < p.N) bias_r = DT<T>::to_f32(reinterpret_cast<const T*>(p.bias)[nn]);
            for (int c = split + splits * cg; c < MT; c += splits * 2) {
                const int m = m0 + c;
                if (m >= p.M) break;
                float a = 0.f;
                for (int sp = 0; sp < splits; ++sp) a += __ldcg(ws_tile + ((long long)sp * MT + c) * kTileN + rn);
                if (nn < p.N) {
                    if constexpr (PART) {
                        store_partial(p, m, nn, a);
                    } else {
                        const T val = DT<T>::from_f32(a + bias_r);
                        const long long idx = (long long)m * p.ldc + nn;
                        outp[idx] = val;
                        for (int r = 0; r < p.n_peers; ++r) reinterpret_cast<T*>(p.peer_out[r])[idx] = val;
                    }
                }
            }
        }
        ptx::bar_sync(kBarEpi, kConsumers);
        if (ct == 0) {
            // last split out resets the tile's counters for the next launch
            if (atomicAdd(done, 1) == splits - 1) {
                *arrive = 0;
                *done = 0;
                __threadfence();
            }
        }
    }
    if constexpr (GROUPED) {
        // rows [end_{E-1}, M) belong to no expert: zeros (fp32 for PART), each CTA's consumers storing a strided share
        const int m_tail = group_table<Cfg>(so)[p.E - 1];
        const long long n_tail = (long long)(p.M - m_tail) * p.N;
        T* outp = reinterpret_cast<T*>(p.out);
        for (long long i = (long long)blockIdx.x * kConsumers + ct; i < n_tail; i += (long long)gridDim.x * kConsumers) {
            const long long m = m_tail + i / p.N;
            if constexpr (PART) reinterpret_cast<float*>(p.out)[m * p.ldc + i % p.N] = 0.f;
            else outp[m * p.ldc + i % p.N] = DT<T>::from_f32(0.f);
        }
    }
}

// ------------------------------------------------------------------ host side
struct Workspace {
    void* ptr = nullptr;
    size_t bytes = 0;
    int* counters = nullptr;
    size_t n_counters = 0;
};

// Split-K scratch: one FIXED-SIZE block per (device, stream), so that launches on different streams never
// share partials or counters and the launch path never reallocates.  32 MB covers every split this
// library launches (<= one wave of 132 CTAs x 128 x 256 fp32 = 17.3 MB).  The only allocation happens on the first split-K call of a stream; it is
// made capture-safe (relaxed capture mode around cudaMalloc) so that a CUDA-graph capture whose first
// split-K GEMM is inside the capture still works.  The registry evicts its least recently used entry.
constexpr size_t kWsBytes = size_t(32) << 20;
constexpr size_t kWsCounters = 8192;
constexpr int kMaxWs = 64;
struct WsEntry {
    int device;
    cudaStream_t stream;
    Workspace ws;
    bool used;
    unsigned long long stamp;
};
WsEntry g_ws[kMaxWs];
unsigned long long g_ws_clock = 0;
std::mutex g_ws_mu;  // the registry is shared by every host thread that launches GEMMs

Workspace* get_workspace(cudaStream_t stream, size_t partial_bytes, size_t n_counters) {
    if (partial_bytes > kWsBytes || n_counters > kWsCounters) return nullptr;
    std::lock_guard<std::mutex> lk(g_ws_mu);
    int dev = 0;
    cudaGetDevice(&dev);
    WsEntry* e = nullptr;
    WsEntry* lru = &g_ws[0];
    for (int i = 0; i < kMaxWs; ++i) {
        if (g_ws[i].used && g_ws[i].device == dev && g_ws[i].stream == stream) {
            e = &g_ws[i];
            break;
        }
        if (!g_ws[i].used) {
            if (lru->used) lru = &g_ws[i];
        } else if (lru->used && g_ws[i].stamp < lru->stamp) {
            lru = &g_ws[i];
        }
    }
    if (e != nullptr) {
        e->stamp = ++g_ws_clock;
        return &e->ws;
    }
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    cudaThreadExchangeStreamCaptureMode(&mode);
    e = lru;
    if (e->used) {
        // evict: cudaFree waits for the device, so no kernel can still be using the block
        int prev = dev;
        cudaSetDevice(e->device);
        cudaFree(e->ws.ptr);
        cudaFree(e->ws.counters);
        cudaSetDevice(prev);
        e->used = false;
    }
    Workspace w{};
    bool ok = cudaMalloc(&w.ptr, kWsBytes) == cudaSuccess &&
              cudaMalloc(reinterpret_cast<void**>(&w.counters), kWsCounters * sizeof(int)) == cudaSuccess &&
              cudaMemset(w.counters, 0, kWsCounters * sizeof(int)) == cudaSuccess;  // synchronous: visible to every stream
    cudaThreadExchangeStreamCaptureMode(&mode);
    if (!ok) {
        (void)cudaGetLastError();
        if (w.ptr) cudaFree(w.ptr);
        if (w.counters) cudaFree(w.counters);
        return nullptr;
    }
    w.bytes = kWsBytes;
    w.n_counters = kWsCounters;
    e->ws = w;
    e->device = dev;
    e->stream = stream;
    e->used = true;
    e->stamp = ++g_ws_clock;
    return &e->ws;
}

template <typename T, int QT, int MT, bool DQ, bool PART, bool GROUPED = false>
bool launch_mt(const T* A, Gemm4Params& p, int force_splits, cudaStream_t stream) {
    constexpr bool kSS = QT == kDecoded;
    using Cfg = StageCfg<T, MT, kSS>;
    constexpr int kBK = Cfg::kBK;
    constexpr size_t smem_bytes = Cfg::kSmemBytes + (GROUPED ? kGroupTabBytes : 0);
    static_assert(smem_bytes <= 227 * 1024, "shared memory");
    static_assert(!GROUPED || (!kSS && !std::is_same<T, float>::value),
                  "the grouped instances decode 4-bit codes to fp16 / bf16");
    static_assert(!(GROUPED && PART && DQ), "the grouped partial instances take plain statistics");
    // the shared-memory opt-in is PER DEVICE (one process may drive several GPUs)
    static bool attr_set[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return false;
    auto kern = gemm4_tc_kernel<T, QT, MT, DQ, PART, GROUPED>;
    if (!attr_set[dev]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes) != cudaSuccess) {
            set_last_error("gemm4_tc smem attr", cudaGetLastError());
            return false;
        }
        attr_set[dev] = true;
    }
    CUtensorMap tmap, tmap_w;
    // activations [M, K]: MT x kSubK boxes (128-byte rows), 128-byte swizzle (fp32 for the TF32 instance)
    if (!encode_tmap_2d(&tmap, A, (int)sizeof(T), 128, (uint64_t)p.M, (uint64_t)p.K, (uint64_t)p.K * sizeof(T),
                        (uint32_t)MT, (uint32_t)Cfg::kSubK))
        return false;
    if constexpr (kSS) {
        // the decoded panel [N, K] of T, 128 x 64 boxes (128-byte rows), 128-byte swizzle
        if (!encode_tmap_2d(&tmap_w, p.B, (int)sizeof(T), 128, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)p.K * sizeof(T),
                            (uint32_t)kTileN, (uint32_t)kBK))
            return false;
    } else {
        // packed codes as a [N, K/2] byte matrix (GROUPED: [E * N, K/2]), 128 x BK/2-byte boxes, BK/2-byte swizzle
        if (!encode_tmap_2d(&tmap_w, p.B, 1, Cfg::kWRowBytes, (uint64_t)p.N * (GROUPED ? p.E : 1), (uint64_t)p.K / 2,
                            (uint64_t)p.K / 2, (uint32_t)kTileN, (uint32_t)Cfg::kWRowBytes))
            return false;
    }
    p.kblocks_total = (p.K + kBK - 1) / kBK;
    // Every row starts at n * K, a multiple of the largest power of two dividing K, and every stage at a multiple of
    // BK: a quantisation block can begin only at 32-code chunks that are multiples of min(blocksize, that, BK).
    int gran = 1 << p.log2_bs;
    if ((p.K & -p.K) < gran) gran = p.K & -p.K;
    if (kBK < gran) gran = kBK;
    p.scale_mask = gran / 32 - 1;
    const int n_tiles = (p.N + kTileN - 1) / kTileN;
    // GROUPED: the m-tiles are counted on the device; each expert adds at most one partial tile, so ceil(M / MT) + E
    // bounds them and sizes the grid
    const int m_tiles = (p.M + MT - 1) / MT + (GROUPED ? p.E : 0);
    const int sms = device_sm_count();
    const int tiles = n_tiles * m_tiles;

    // K-splitting for small problems: a uniform split so that ONE wave covers the machine.  Split CTAs exchange
    // fp32 partials through an L2-resident workspace and every split reduces its share of the columns.  (The grouped
    // instances never split K.)
    int splits = 1;
    if (!GROUPED && (force_splits > 0 || tiles * 2 <= sms)) {
        int v = force_splits > 0 ? force_splits : sms / tiles;
        // >= two stages per split by default, >= one when the split is forced
        const int max_by_k = force_splits > 0 ? p.kblocks_total : (p.kblocks_total / 2 > 0 ? p.kblocks_total / 2 : 1);
        if (v > max_by_k) v = max_by_k;
        if (v > 16) v = 16;
        if (v < 1) v = 1;
        const int per = (p.kblocks_total + v - 1) / v;
        splits = (p.kblocks_total + per - 1) / per;  // no empty split
    }
    // a forced split must still be one co-resident wave (the splits of a tile wait for each other)
    if (splits > 1 && tiles * splits > sms) return false;
    // the staged route keeps its weight panel in the split-K workspace: it must never split
    if (kSS && splits != 1) {
        set_last_error_msg("gemm4_tc: the staged GEMM was asked to split K");
        return false;
    }
    p.splits = splits;
    p.n_tiles = n_tiles;
    p.tiles_total = tiles;
    p.ws_partial = nullptr;
    p.ws_counter = nullptr;
    if (splits > 1) {
        Workspace* ws = get_workspace(stream, size_t(tiles) * splits * kTileN * MT * sizeof(float), 2 * (size_t)tiles);
        if (ws == nullptr) {
            set_last_error_msg("gemm4_tc: could not allocate the split-K workspace");
            return false;
        }
        p.ws_partial = reinterpret_cast<float*>(ws->ptr);
        p.ws_counter = ws->counters;
    }
    // persistent: at most one CTA per SM, each running every gridDim-th unit (a split launch is one unit per CTA)
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(tiles * splits < sms ? tiles * splits : sms, 1, 1);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    int na = 0;
    if (splits > 1) {
        // the splits of a tile rendezvous in the epilogue: a COOPERATIVE launch makes the runtime schedule the
        // whole (<= one wave) grid at once, so the wait cannot starve behind other streams' kernels
        attr[na].id = cudaLaunchAttributeCooperative;
        attr[na].val.cooperative = 1;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, tmap, tmap_w, p);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        set_last_error("gemm4_tc launch", e);
        return false;
    }
    BNB200_CHECK_LAUNCH("gemm4_tc");
    return true;
}

} // namespace

// Returns true if the tensor-core path handled the call.  Every output element is stored to each of outs.p[0..n)
// (same ldc).
// `mt_override`: token tile (16 | 32 | 64 | 128 | 256, 0 = by M); `force_splits`: K split per tile (0 = by the grid).
template <typename T, bool PART>
bool launch_gemm4_tc(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                     const float* absmax_code, const float* absmax_offset, const OutList<OutElem<T, PART>>& outs,
                     const T* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, cudaStream_t stream,
                     int mt_override, int force_splits) {
    if (outs.n < 1 || outs.n > kMaxOuts) return false;
    if (M <= 0 || N <= 0) return true;
    if (K < 64 || (K % 64) != 0) return false;
    if (blocksize < 32 || (blocksize & (blocksize - 1)) != 0) return false;
    if ((reinterpret_cast<uintptr_t>(A) & 15) != 0 || (reinterpret_cast<uintptr_t>(B) & 15) != 0) return false;
    if (quant_type != kNF4 && quant_type != kFP4) return false;

    // 256-token tiles decode each weight half as often as 128-token ones, but a grid of them that does not fill one
    // wave leaves SMs idle (or needs a K split): they are taken when they alone fill every SM.  The TF32 instance stops
    // at 128 tokens: one 64-deep fp32 stage of a 256-token tile (68 KB) next to its 132 KB of epilogue staging leaves
    // room for a single ring stage.
    constexpr bool tf32 = std::is_same<T, float>::value;
    int MT = 128;
    if (M <= 16) MT = 16;
    else if (M <= 32) MT = 32;
    else if (M <= 64) MT = 64;
    else if (!tf32 && (long long)((M + 255) / 256) * ((N + kTileN - 1) / kTileN) >= device_sm_count()) MT = 256;
    if (mt_override != 0) {
        if (mt_override != 16 && mt_override != 32 && mt_override != 64 && mt_override != 128 &&
            (tf32 || mt_override != 256))
            return false;
        MT = mt_override;
    }

    Gemm4Params p{};
    p.B = B;
    p.absmax = absmax;
    p.absmax_8bit = absmax_8bit;
    p.absmax_code = absmax_code;
    p.absmax_offset = absmax_offset;
    p.bias = bias;
    p.out = outs.p[0];
    p.n_peers = outs.n - 1;
    for (int r = 1; r < outs.n; ++r) p.peer_out[r - 1] = outs.p[r];
    p.rows_per_out = outs.rows_per_out;
    p.M = M;
    p.N = N;
    p.K = K;
    p.ldc = ldc;
    p.log2_bs = ilog2_pow2(blocksize);
    bool vec = (ldc % (16 / (int)sizeof(T))) == 0;
    for (int r = 0; r < outs.n; ++r) vec = vec && (reinterpret_cast<uintptr_t>(outs.p[r]) & 15) == 0;
    p.out_vec = vec ? 1 : 0;

#define BNB200_DISPATCH_MT(QT, DQ)                                                                                     \
    switch (MT) {                                                                                                      \
    case 16: return launch_mt<T, QT, 16, DQ, PART>(A, p, force_splits, stream);                                        \
    case 32: return launch_mt<T, QT, 32, DQ, PART>(A, p, force_splits, stream);                                        \
    case 64: return launch_mt<T, QT, 64, DQ, PART>(A, p, force_splits, stream);                                        \
    case 128: return launch_mt<T, QT, 128, DQ, PART>(A, p, force_splits, stream);                                      \
    default:                                                                                                           \
        if constexpr (tf32) return false;                                                                              \
        else return launch_mt<T, QT, 256, DQ, PART>(A, p, force_splits, stream);                                       \
    }
    const bool dq = absmax_8bit != nullptr;
    if (quant_type == kNF4) {
        if (dq) {
            BNB200_DISPATCH_MT(kNF4, true)
        } else {
            BNB200_DISPATCH_MT(kNF4, false)
        }
    } else {
        if (dq) {
            BNB200_DISPATCH_MT(kFP4, true)
        } else {
            BNB200_DISPATCH_MT(kFP4, false)
        }
    }
#undef BNB200_DISPATCH_MT
}

// ------------------------------------------------------------------ the staged route
// At large M the fused kernel decodes every weight once per token tile (M / 256 times).  The staged route decodes
// each weight once: it loops over panels of `panel_rows` output features (a multiple of 128), decodes the panel into
// the stream's workspace block (dequantize4_prmt_kernel, the fused kernel's table decode and scale fetch: the same
// bits) and runs the staged instance of gemm4_tc_kernel over all M tokens of that panel.  Both launches go on
// `stream`, so a panel is never overwritten while the GEMM before it still reads it.  Same A values, same k16 order,
// same instruction shape, accumulation from zero and one rounding in the same epilogue: the output is the fused
// kernel's, bit for bit.  The panel lives in the per-stream split-K block, so the staged GEMM never splits K.
int staged_max_panel_rows(int K, int elem_bytes) {
    const long long rows = (long long)kWsBytes / ((long long)K * elem_bytes);
    return rows >= kTileN ? (int)(rows / kTileN * kTileN) : 0;
}

// Each panel is a launch of its own, so the last wave of every panel's 256-token tiles runs partly empty.  The panel
// is the one (a multiple of 128 rows that fits the workspace) whose panels take the fewest waves in all, the largest
// of those (fewest launches).  Returns that wave count and sets *panel_rows; 0 when no panel fits.
int staged_plan(int M, int N, int K, int sms, int* panel_rows) {
    const int max_units = staged_max_panel_rows(K, 2) / kTileN;
    const long long m_tiles = (M + 255) / 256;
    const int n_units = (N + kTileN - 1) / kTileN;
    long long best = 0;
    for (int u = 1; u <= max_units && u <= n_units; ++u) {
        const long long full = n_units / u, rest = n_units % u;
        const long long waves = full * ((m_tiles * u + sms - 1) / sms) + (rest ? (m_tiles * rest + sms - 1) / sms : 0);
        if (best == 0 || waves <= best) {
            best = waves;
            *panel_rows = u * kTileN;
        }
    }
    return (int)best;
}

// panel_rows 0: the panel of staged_plan (DESIGN.md section 3.1).  outs: as in launch_gemm4_tc.
template <typename T, bool PART>
bool launch_gemm4_staged(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                         const float* absmax_code, const float* absmax_offset, const OutList<OutElem<T, PART>>& outs,
                         const T* bias, int M, int N, int K, int ldc, int blocksize, int quant_type,
                         cudaStream_t stream, int mt_override, int panel_rows) {
    static_assert(!std::is_same<T, float>::value, "the staged route has 16-bit instances only");
    if (outs.n < 1 || outs.n > kMaxOuts) return false;
    if (M <= 0 || N <= 0) return true;
    if (K < 64 || (K % 64) != 0) return false;
    if (blocksize < 32 || (blocksize & (blocksize - 1)) != 0) return false;
    if ((reinterpret_cast<uintptr_t>(A) & 15) != 0 || (reinterpret_cast<uintptr_t>(B) & 15) != 0) return false;
    if (quant_type != kNF4 && quant_type != kFP4) return false;
    const int max_rows = staged_max_panel_rows(K, (int)sizeof(T));
    const int sms = device_sm_count();
    if (panel_rows == 0) staged_plan(M, N, K, sms, &panel_rows);
    if (panel_rows <= 0 || panel_rows % kTileN != 0 || panel_rows > max_rows) return false;
    const int n_pad = (N + kTileN - 1) / kTileN * kTileN;
    if (panel_rows > n_pad) panel_rows = n_pad;

    // 256-token tiles where the whole weight's tiles fill the SMs (every shape the dispatcher routes here)
    int MT = (long long)((M + 255) / 256) * (n_pad / kTileN) >= sms ? 256 : 128;
    if (mt_override != 0) {
        if (mt_override != 128 && mt_override != 256) return false;
        MT = mt_override;
    }
    Workspace* ws = get_workspace(stream, (size_t)panel_rows * K * sizeof(T), 0);
    if (ws == nullptr) {
        set_last_error_msg("gemm4_tc: could not allocate the staged route's workspace");
        return false;
    }
    T* panel = reinterpret_cast<T*>(ws->ptr);
    bool vec = (ldc % (16 / (int)sizeof(T))) == 0;
    for (int r = 0; r < outs.n; ++r) vec = vec && (reinterpret_cast<uintptr_t>(outs.p[r]) & 15) == 0;
    for (int n0 = 0; n0 < N; n0 += panel_rows) {
        const int rows = N - n0 < panel_rows ? N - n0 : panel_rows;
        launch_dequantize4_panel<T>(B, absmax, absmax_8bit, absmax_code, absmax_offset, panel, blocksize, quant_type,
                                    n0, rows, K, stream);
        // the panel's columns of the output: n0 is a multiple of 128, so every base keeps its 16-byte alignment
        Gemm4Params p{};
        p.B = reinterpret_cast<const uint8_t*>(panel);
        p.bias = bias != nullptr ? bias + n0 : nullptr;
        p.out = outs.p[0] + n0;
        p.n_peers = outs.n - 1;
        for (int r = 1; r < outs.n; ++r) p.peer_out[r - 1] = outs.p[r] + n0;
        p.rows_per_out = outs.rows_per_out;
        p.M = M;
        p.N = rows;
        p.K = K;
        p.ldc = ldc;
        p.log2_bs = ilog2_pow2(blocksize);
        p.out_vec = vec ? 1 : 0;
        const bool ok = MT == 256 ? launch_mt<T, kDecoded, 256, false, PART>(A, p, 1, stream)
                                  : launch_mt<T, kDecoded, 128, false, PART>(A, p, 1, stream);
        if (!ok) return false;
    }
    return true;
}

#define BNB200_STAGED_INST(T, PART)                                                                                    \
    template bool launch_gemm4_staged<T, PART>(const T*, const uint8_t*, const float*, const uint8_t*, const float*,   \
                                               const float*, const OutList<OutElem<T, PART>>&, const T*, int, int,     \
                                               int, int, int, int, cudaStream_t, int, int);
BNB200_STAGED_INST(__nv_bfloat16, false)
BNB200_STAGED_INST(__half, false)
BNB200_STAGED_INST(__nv_bfloat16, true)
BNB200_STAGED_INST(__half, true)
#undef BNB200_STAGED_INST

// The staged GEMM alone on an already decoded weight W[N, K] (no workspace): for timing the route's phases.
template <typename T>
bool launch_gemm_decoded(const T* A, const T* W, T* out, const T* bias, int M, int N, int K, int ldc, int mt,
                         cudaStream_t stream) {
    if (M <= 0 || N <= 0) return true;
    if (K < 64 || (K % 64) != 0 || (mt != 128 && mt != 256)) return false;
    if ((reinterpret_cast<uintptr_t>(A) & 15) != 0 || (reinterpret_cast<uintptr_t>(W) & 15) != 0) return false;
    Gemm4Params p{};
    p.B = reinterpret_cast<const uint8_t*>(W);
    p.bias = bias;
    p.out = out;
    p.M = M;
    p.N = N;
    p.K = K;
    p.ldc = ldc;
    p.out_vec = ((ldc % (16 / (int)sizeof(T))) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) ? 1 : 0;
    return mt == 256 ? launch_mt<T, kDecoded, 256, false, false>(A, p, 1, stream)
                     : launch_mt<T, kDecoded, 128, false, false>(A, p, 1, stream);
}
template bool launch_gemm_decoded<__nv_bfloat16>(const __nv_bfloat16*, const __nv_bfloat16*, __nv_bfloat16*,
                                                 const __nv_bfloat16*, int, int, int, int, int, cudaStream_t);
template bool launch_gemm_decoded<__half>(const __half*, const __half*, __half*, const __half*, int, int, int, int, int,
                                          cudaStream_t);

#define BNB200_TC_INST(T, PART)                                                                                        \
    template bool launch_gemm4_tc<T, PART>(const T*, const uint8_t*, const float*, const uint8_t*, const float*,       \
                                           const float*, const OutList<OutElem<T, PART>>&, const T*, int, int, int,    \
                                           int, int, int, cudaStream_t, int, int);
BNB200_TC_INST(__nv_bfloat16, false)
BNB200_TC_INST(__half, false)
BNB200_TC_INST(float, false)  // fp32 activations and output, TF32 tensor cores
BNB200_TC_INST(__nv_bfloat16, true)
BNB200_TC_INST(__half, true)
BNB200_TC_INST(float, true)
#undef BNB200_TC_INST

// ------------------------------------------------------------------ the grouped GEMM
// Every expert of a mixture-of-experts layer in one launch of the GROUPED instances (DESIGN.md section 3.1.2):
// out[m, :] = T(A[m, :] . W_e^T + bias[e * N ..]) for end_{e-1} <= m < end_e, and 0 for end_{E-1} <= m < M, with
// W_e rows [e * N, (e + 1) * N) of the stacked 4-bit weight and end_e the device-side clamp of offs (Gemm4Params).
// Each expert's rows are bit for bit what launch_gemm4_tc gives on that expert alone at token tile mt and no K split.
// mt: 16 | 32 | 64 | 128 (the caller's tile rule).  Returns false, with nothing launched, for what the instances do
// not serve, or when the launch fails (the error message set).
template <typename T>
bool launch_gemm4_grouped(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                          const float* absmax_code, const float* absmax_offset, const int* offs, int E, T* out,
                          const T* bias, int M, int N, int K, int ldc, int blocksize, int quant_type, int mt,
                          cudaStream_t stream) {
    static_assert(!std::is_same<T, float>::value, "the grouped GEMM has 16-bit instances only");
    if (M <= 0) return true;
    if (N <= 0 || E < 1 || E > kMaxExperts || (long long)E * N > 0x7fffffffLL || K < 64 || (K % 64) != 0) return false;
    if (blocksize < 32 || (blocksize & (blocksize - 1)) != 0) return false;
    if ((reinterpret_cast<uintptr_t>(A) & 15) != 0 || (reinterpret_cast<uintptr_t>(B) & 15) != 0) return false;
    if (quant_type != kNF4 && quant_type != kFP4) return false;
    Gemm4Params p{};
    p.B = B;
    p.absmax = absmax;
    p.absmax_8bit = absmax_8bit;
    p.absmax_code = absmax_code;
    p.absmax_offset = absmax_offset;
    p.bias = bias;
    p.out = out;
    p.M = M;
    p.N = N;
    p.K = K;
    p.ldc = ldc;
    p.log2_bs = ilog2_pow2(blocksize);
    p.out_vec = ((ldc % (16 / (int)sizeof(T))) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) ? 1 : 0;
    p.offs = offs;
    p.E = E;
#define BNB200_GROUPED_MT(QT, DQ)                                                                                      \
    switch (mt) {                                                                                                      \
    case 16: return launch_mt<T, QT, 16, DQ, false, true>(A, p, 1, stream);                                            \
    case 32: return launch_mt<T, QT, 32, DQ, false, true>(A, p, 1, stream);                                            \
    case 64: return launch_mt<T, QT, 64, DQ, false, true>(A, p, 1, stream);                                            \
    case 128: return launch_mt<T, QT, 128, DQ, false, true>(A, p, 1, stream);                                          \
    default: return false;                                                                                             \
    }
    const bool dq = absmax_8bit != nullptr;
    if (quant_type == kNF4) {
        if (dq) {
            BNB200_GROUPED_MT(kNF4, true)
        } else {
            BNB200_GROUPED_MT(kNF4, false)
        }
    } else {
        if (dq) {
            BNB200_GROUPED_MT(kFP4, true)
        } else {
            BNB200_GROUPED_MT(kFP4, false)
        }
    }
#undef BNB200_GROUPED_MT
}
template bool launch_gemm4_grouped<__nv_bfloat16>(const __nv_bfloat16*, const uint8_t*, const float*, const uint8_t*,
                                                  const float*, const float*, const int*, int, __nv_bfloat16*,
                                                  const __nv_bfloat16*, int, int, int, int, int, int, int,
                                                  cudaStream_t);
template bool launch_gemm4_grouped<__half>(const __half*, const uint8_t*, const float*, const uint8_t*, const float*,
                                           const float*, const int*, int, __half*, const __half*, int, int, int, int,
                                           int, int, int, cudaStream_t);

// The grouped fp32 partial of a row-sharded expert layer: out[m, n] (row stride ldc) = A[m, :] . W_e[n, :] for
// end_{e-1} <= m < end_e, summed in fp32 with no bias and no rounding, and 0 for end_{E-1} <= m < M.  Plain fp32
// statistics only (a K shard never carries nested ones).  With the same tile, T(P + bias_e) is launch_gemm4_grouped's
// output bit for bit: same decode, same k16 order, the same accumulators, rounded once.  Returns false as
// launch_gemm4_grouped does.
template <typename T>
bool launch_gemm4_grouped_partial(const T* A, const uint8_t* B, const float* absmax, const int* offs, int E, float* out,
                                  int M, int N, int K, int ldc, int blocksize, int quant_type, int mt,
                                  cudaStream_t stream) {
    static_assert(!std::is_same<T, float>::value, "the grouped GEMM has 16-bit instances only");
    if (M <= 0) return true;
    if (N <= 0 || E < 1 || E > kMaxExperts || (long long)E * N > 0x7fffffffLL || K < 64 || (K % 64) != 0) return false;
    if (blocksize < 32 || (blocksize & (blocksize - 1)) != 0) return false;
    if ((reinterpret_cast<uintptr_t>(A) & 15) != 0 || (reinterpret_cast<uintptr_t>(B) & 15) != 0) return false;
    if (quant_type != kNF4 && quant_type != kFP4) return false;
    Gemm4Params p{};
    p.B = B;
    p.absmax = absmax;
    p.out = out;
    p.M = M;
    p.N = N;
    p.K = K;
    p.ldc = ldc;
    p.log2_bs = ilog2_pow2(blocksize);
    p.offs = offs;
    p.E = E;
#define BNB200_GROUPED_PART_MT(QT)                                                                                     \
    switch (mt) {                                                                                                      \
    case 16: return launch_mt<T, QT, 16, false, true, true>(A, p, 1, stream);                                          \
    case 32: return launch_mt<T, QT, 32, false, true, true>(A, p, 1, stream);                                          \
    case 64: return launch_mt<T, QT, 64, false, true, true>(A, p, 1, stream);                                          \
    case 128: return launch_mt<T, QT, 128, false, true, true>(A, p, 1, stream);                                        \
    default: return false;                                                                                             \
    }
    if (quant_type == kNF4) {
        BNB200_GROUPED_PART_MT(kNF4)
    } else {
        BNB200_GROUPED_PART_MT(kFP4)
    }
#undef BNB200_GROUPED_PART_MT
}
template bool launch_gemm4_grouped_partial<__nv_bfloat16>(const __nv_bfloat16*, const uint8_t*, const float*, const int*,
                                                          int, float*, int, int, int, int, int, int, int, cudaStream_t);
template bool launch_gemm4_grouped_partial<__half>(const __half*, const uint8_t*, const float*, const int*, int, float*,
                                                   int, int, int, int, int, int, int, cudaStream_t);

} // namespace bnb200
