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
//     the tokens m are the wgmma N dimension (MT = 16..128).  A CTA owns out[m0:m0+MT, n0:n0+128].
//   * A pipeline stage is 128 k-elements.  One TMA producer warp stages, per stage, the packed codes
//     of the CTA's 128 rows (128 x 64 B, 64-byte swizzle, 8 KB) and the activation tile
//     X[m0:m0+MT, k0:k0+128] (two 128-byte-swizzled sub-tiles), the K-major B operand of wgmma.
//   * Every consumer thread decodes the codes of its two rows straight into the register fragment of
//     wgmma's A operand, with the exact reference rounding -- a per-block 16-entry table built with
//     16 FMUL + 8 cvt.rn and looked up with PRMT only.  The decoded weights never pass through shared
//     memory, whose bandwidth is then left to the activation operand.
//   * Two A-fragment register sets alternate between stages, so the decode of stage i+1 overlaps the
//     wgmma of stage i (wgmma.wait_group 1 before a set is overwritten).
//   * Accumulators live in registers; the epilogue adds the bias, rounds to T and stores, or -- for
//     split-K, which fills the 132 SMs when the tile grid is small -- writes fp32 partials to an
//     L2-resident workspace with a last-arriver reduction in deterministic split order.
//
// Warp roles (288 threads): warps 0..7 = two consumer warpgroups (decode + wgmma + epilogue),
// warp 8 = TMA producer.
#include "common.cuh"
#include "decode4.cuh"
#include "hopper_ptx.cuh"

#include <cstdlib>
#include <mutex>
#include <type_traits>

namespace bnb200 {

namespace {

constexpr int kBK = 128;           // pipeline stage: 128 k-elements = two 128-byte swizzle atoms of X per row
constexpr int kTileN = 128;        // output features per CTA (two warpgroups of 64)
constexpr int kConsumers = 256;    // threads of the two consumer warpgroups
constexpr int kThreads = kConsumers + 32;

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
    float* ws_partial;           // split-K partials [tiles][splits][MT][128]
    int* ws_counter;             // two per output tile, zero on entry, reset on exit
    int M, N, K, ldc;
    int log2_bs;
    int kblocks_total;           // number of 128-wide stages = ceil(K / 128)
    int n_tiles;                 // N tiles of 128 (tile = m_tile * n_tiles + n_tile)
    int tiles_total;
    int splits;                  // K splits per tile (1 = none)
};

// one k16 step of a 64-row warpgroup tile: D[64 x MT] += A[64 x 16] (registers) * X[MT x 16]^T (descriptor)
template <typename T, int MT>
__device__ __forceinline__ void wgmma_step(float (&d)[MT / 2], const uint32_t (&a)[4], uint64_t b_desc) {
    constexpr bool bf = std::is_same<T, __nv_bfloat16>::value;
    if constexpr (MT == 16) {
        if constexpr (bf) ptx::wgmma_m64n16k16_bf16_rs(d, a, b_desc); else ptx::wgmma_m64n16k16_f16_rs(d, a, b_desc);
    } else if constexpr (MT == 32) {
        if constexpr (bf) ptx::wgmma_m64n32k16_bf16_rs(d, a, b_desc); else ptx::wgmma_m64n32k16_f16_rs(d, a, b_desc);
    } else if constexpr (MT == 64) {
        if constexpr (bf) ptx::wgmma_m64n64k16_bf16_rs(d, a, b_desc); else ptx::wgmma_m64n64k16_f16_rs(d, a, b_desc);
    } else {
        static_assert(MT == 128, "token tile");
        if constexpr (bf) ptx::wgmma_m64n128k16_bf16_rs(d, a, b_desc); else ptx::wgmma_m64n128k16_f16_rs(d, a, b_desc);
    }
}

// Pipeline stage = 128 k-elements: two 64-wide (128-byte, swizzle-atom) activation sub-tiles and the
// packed codes of 128 rows.  Ring depth: as many stages as fit next to each other in 200 KB.
template <int MT> struct StageCfg {
    static constexpr int kXSubBytes = MT * 128;                  // one 64-wide sub-tile
    static constexpr int kXStageBytes = 2 * kXSubBytes;
    static constexpr int kWStageBytes = kTileN * 64;             // packed codes: 128 rows x 64 B (TMA, 64-B swizzle)
    static constexpr int kStageBytes = kXStageBytes + kWStageBytes;
    static constexpr int kStages = (200 * 1024 / kStageBytes) > 8 ? 8 : (200 * 1024 / kStageBytes);
};

// The 16 codes of stage-row words w[4q .. 4q+3] that this thread's A fragments need (byte `t` of each,
// t = lane % 4): wgmma k16 step 2q+u reads byte t of words 4q+2u (k 2t, 2t+1) and 4q+2u+1 (k 8+2t, 9+2t).
__device__ __forceinline__ uint32_t gather_bytes(uint4 v, uint32_t sel) {
    return prmt(prmt(v.x, v.y, sel), prmt(v.z, v.w, sel), 0x5410);
}

template <typename T, int QT, int MT>
__global__ void __launch_bounds__(kThreads, 1)
    gemm4_tc_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                    const Gemm4Params p) {
    using Cfg = StageCfg<MT>;
    constexpr int kStages = Cfg::kStages;
    constexpr int kXSubBytes = Cfg::kXSubBytes;
    constexpr int kXStageBytes = Cfg::kXStageBytes;
    constexpr int kWStageBytes = Cfg::kWStageBytes;

    // ------------------------------------------------------------------ shared memory
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sx = smem;                              // [kStages][2][MT x 128 B]   activations
    uint8_t* sw = smem + kStages * kXStageBytes;     // [kStages][128 x 64 B]      packed codes
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);
    uint64_t* full = bars;                   // [kStages] TMA (1 arrive + bytes) -> consumers
    uint64_t* empty = bars + kStages;        // [kStages] the 8 consumer warps -> TMA producer

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // Linear CTA id -> (tile, K-split): ids are ordered (tile, split)
    const int splits = p.splits;
    const int tile_id = blockIdx.x / splits;
    const int split = blockIdx.x - tile_id * splits;
    const int slot0 = tile_id * splits;  // first workspace slot of this tile
    const int n0 = (tile_id % p.n_tiles) * kTileN;
    const int m0 = (tile_id / p.n_tiles) * MT;
    const int per = (p.kblocks_total + splits - 1) / splits;
    const int st_begin = split * per;
    int st_end = st_begin + per;
    if (st_end > p.kblocks_total) st_end = p.kblocks_total;
    const int nst = st_end - st_begin;  // >= 1 by construction

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            ptx::mbar_init(&full[s], 1);
            ptx::mbar_init(&empty[s], kConsumers / 32);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp == kConsumers / 32) {
        // ================================================================== TMA producer
        if (ptx::elect_one()) {
            ptx::prefetch_tmap(&tmap_x);
            ptx::prefetch_tmap(&tmap_w);
            int s = 0;
            uint32_t ph = 0;
            for (int i = 0; i < nst; ++i) {
                ptx::mbar_wait(&empty[s], ph ^ 1u);
                const int k0 = (st_begin + i) * kBK;
                ptx::mbar_arrive_expect_tx(&full[s], kWStageBytes + kXStageBytes);
                // packed codes of this CTA's 128 output features: bytes [k0/2, k0/2 + 64) of rows n0..n0+127
                ptx::tma_load_2d(sw + s * kWStageBytes, &tmap_w, &full[s], k0 / 2, n0);
                uint8_t* dst = sx + s * kXStageBytes;
                // rows past M, rows past N and columns past K are out of bounds for the tensor maps: TMA zero-fills
#pragma unroll
                for (int h = 0; h < 2; ++h) ptx::tma_load_2d(dst + h * kXSubBytes, &tmap_x, &full[s], k0 + 64 * h, m0);
                if (++s == kStages) {
                    s = 0;
                    ph ^= 1u;
                }
            }
        }
        return;
    }

    // ====================================================================== consumers
    const int wg = warp >> 2;                 // warpgroup: feature rows [64 wg, 64 wg + 64) of the tile
    const int g = lane >> 2, t = lane & 3;
    const int row0 = wg * 64 + (warp & 3) * 16 + g;  // this thread's two rows: row0, row0 + 8
    const int na = n0 + row0, nb = na + 8;
    const bool a_ok = na < p.N, b_ok = nb < p.N;
    const long long e_a = (long long)(a_ok ? na : 0) * p.K;
    const long long e_b = (long long)(b_ok ? nb : 0) * p.K;
    const ScaleSrc sc{p.absmax, p.absmax_8bit, p.absmax_code, p.absmax_offset ? __ldg(p.absmax_offset) : 0.0f};
    const uint32_t sel = (uint32_t)t | ((uint32_t)(t + 4) << 4);
    // 64-byte swizzle of the code rows: 16-byte chunk c of row r sits at chunk c ^ ((r >> 1) & 3)
    const uint32_t swz_a = (uint32_t)((row0 >> 1) & 3), swz_b = (uint32_t)(((row0 + 8) >> 1) & 3);

    // Scales of one stage: the 32 codes of a gathered word lie inside one quantisation block (blocks are
    // >= 32 and aligned), so each (row, q) needs one scale.  Fetched one stage ahead.
    float scl[2][4];
    auto fetch = [&](int i) {
        const long long kk = (long long)(st_begin + i) * kBK;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const bool in_k = i < nst && kk + 32 * q < p.K;
            scl[0][q] = (in_k && a_ok) ? sc.load((e_a + kk + 32 * q) >> p.log2_bs) : 0.f;
            scl[1][q] = (in_k && b_ok) ? sc.load((e_b + kk + 32 * q) >> p.log2_bs) : 0.f;
        }
    };

    float acc[MT / 2];
#pragma unroll
    for (int j = 0; j < MT / 2; ++j) acc[j] = 0.f;

    uint32_t afr[2][8][4];  // two A-fragment sets: [set][k16 step][reg]

    // decode stage i (smem stage s) into A set `set`
    auto decode = [&](int s, uint32_t (&a)[8][4]) {
        const uint8_t* wt = sw + s * kWStageBytes;
        float sc_cur[2][4];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int q = 0; q < 4; ++q) sc_cur[r][q] = scl[r][q];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const uint8_t* rowp = wt + (row0 + 8 * r) * 64;
            const uint32_t swz = r ? swz_b : swz_a;
            DecodeTable tab;
            float last = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const uint4 v = *reinterpret_cast<const uint4*>(rowp + (((uint32_t)q ^ swz) << 4));
                const uint32_t word = gather_bytes(v, sel);
                if (q == 0 || sc_cur[r][q] != last) {
                    build_table<T, QT>(sc_cur[r][q], tab);
                    last = sc_cur[r][q];
                }
                uint32_t o[4];
                decode_word(word, tab, o);
                // o[i]: byte i of the gathered word = word 4q+i of the row -> k16 step 2q + i/2, half i%2
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    a[2 * q + u][r] = o[2 * u];          // rows g / g+8, k 2t..2t+1
                    a[2 * q + u][2 + r] = o[2 * u + 1];  // rows g / g+8, k 8+2t..9+2t
                }
            }
        }
    };

    auto mma_stage = [&](int s, const uint32_t (&a)[8][4]) {
        const uint32_t xs = ptx::smem_u32(sx + s * kXStageBytes);
        const uint64_t d0 = ptx::make_sw128_kmajor_desc(xs);
        const uint64_t d1 = ptx::make_sw128_kmajor_desc(xs + kXSubBytes);
        ptx::wgmma_fence();
#pragma unroll
        for (int j = 0; j < 8; ++j) wgmma_step<T, MT>(acc, a[j], (j < 4 ? d0 : d1) + 2 * (j & 3));
        ptx::wgmma_commit();
    };

    fetch(0);
    int prev_s = -1;
    for (int i0 = 0; i0 < nst; i0 += 2) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int i = i0 + h;
            if (i < nst) {
                const int s = i % kStages;
                ptx::mbar_wait(&full[s], (uint32_t)(i / kStages) & 1u);
                decode(s, afr[h]);
                fetch(i + 1);
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

    // ================================================================== epilogue
    // acc[4j + e]: feature row row0 + 8 * (e >= 2), token column 8j + 2t + (e & 1)
    T* outp = reinterpret_cast<T*>(p.out);
    if (splits == 1) {
        const T* bias = reinterpret_cast<const T*>(p.bias);
        const float bias_a = (bias != nullptr && a_ok) ? DT<T>::to_f32(bias[na]) : 0.f;
        const float bias_b = (bias != nullptr && b_ok) ? DT<T>::to_f32(bias[nb]) : 0.f;
#pragma unroll
        for (int j = 0; j < MT / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int m = m0 + 8 * j + 2 * t + (e & 1);
                const bool hi = e >= 2;
                const int n = hi ? nb : na;
                if ((hi ? b_ok : a_ok) && m < p.M) {
                    const T val = DT<T>::from_f32(acc[4 * j + e] + (hi ? bias_b : bias_a));
                    const long long idx = (long long)m * p.ldc + n;
                    outp[idx] = val;
                    for (int r = 0; r < p.n_peers; ++r) reinterpret_cast<T*>(p.peer_out[r])[idx] = val;
                }
            }
        }
        return;
    }

    // ---- split-K: every split CTA publishes its fp32 partial tile (layout [column m][row n], so that the
    // later reads are 128-byte coalesced), the splits of a tile rendezvous on a counter, and EACH of them then
    // reduces a 1/splits share of the columns (in split order: deterministic).  The launch is COOPERATIVE (all
    // CTAs of the <= one-wave grid are resident together), so the short wait cannot starve; it is bounded anyway.
    float* ws_tile = p.ws_partial + (long long)slot0 * kTileN * MT;
    float* my = ws_tile + (long long)split * kTileN * MT;
#pragma unroll
    for (int j = 0; j < MT / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) my[(8 * j + 2 * t + (e & 1)) * kTileN + row0 + 8 * (e >> 1)] = acc[4 * j + e];
    __threadfence();
    asm volatile("bar.sync 1, 256;" ::: "memory");
    int* arrive = p.ws_counter + tile_id;
    int* done = p.ws_counter + p.tiles_total + tile_id;
    if (threadIdx.x == 0) {
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
    asm volatile("bar.sync 1, 256;" ::: "memory");
    {
        const int e = threadIdx.x;               // 0..255 over the two consumer warpgroups
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
                const T val = DT<T>::from_f32(a + bias_r);
                const long long idx = (long long)m * p.ldc + nn;
                outp[idx] = val;
                for (int r = 0; r < p.n_peers; ++r) reinterpret_cast<T*>(p.peer_out[r])[idx] = val;
            }
        }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (threadIdx.x == 0) {
        // last split out resets the tile's counters for the next launch
        if (atomicAdd(done, 1) == splits - 1) {
            *arrive = 0;
            *done = 0;
            __threadfence();
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
// library launches (<= one wave of 132 CTAs x 128 x 128 fp32 = 8.3 MB).  The only allocation happens on the first split-K call of a stream; it is
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

template <typename T, int QT, int MT>
bool launch_mt(const T* A, Gemm4Params& p, int force_splits, cudaStream_t stream) {
    using Cfg = StageCfg<MT>;
    constexpr size_t smem_bytes = 1024 /*align slack*/ + size_t(Cfg::kStages) * Cfg::kStageBytes + 256 /*barriers*/;
    // the shared-memory opt-in is PER DEVICE (one process may drive several GPUs)
    static bool attr_set[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return false;
    auto kern = gemm4_tc_kernel<T, QT, MT>;
    if (!attr_set[dev]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes) != cudaSuccess) {
            set_last_error("gemm4_tc smem attr", cudaGetLastError());
            return false;
        }
        attr_set[dev] = true;
    }
    CUtensorMap tmap, tmap_w;
    if (!encode_tmap_2d(&tmap, A, 2, 128, (uint64_t)p.M, (uint64_t)p.K, (uint64_t)p.K * 2, (uint32_t)MT, 64u)) return false;
    // packed codes as a [N, K/2] byte matrix, 128 x 64-byte boxes, 64-byte swizzle
    if (!encode_tmap_2d(&tmap_w, p.B, 1, 64, (uint64_t)p.N, (uint64_t)p.K / 2, (uint64_t)p.K / 2, (uint32_t)kTileN, 64u))
        return false;
    const int n_tiles = (p.N + kTileN - 1) / kTileN;
    const int m_tiles = (p.M + MT - 1) / MT;
    const int sms = device_sm_count();
    const int tiles = n_tiles * m_tiles;

    // K-splitting for small problems: a uniform split so that ONE wave covers the machine.  Split CTAs exchange
    // fp32 partials through an L2-resident workspace and every split reduces its share of the columns.
    int splits = 1;
    if (force_splits > 0 || tiles * 2 <= sms) {
        int v = force_splits > 0 ? force_splits : sms / tiles;
        // >= two 128-wide stages per split by default, >= one when the split is forced
        const int max_by_k = force_splits > 0 ? p.kblocks_total : (p.kblocks_total / 2 > 0 ? p.kblocks_total / 2 : 1);
        if (v > max_by_k) v = max_by_k;
        if (v > 16) v = 16;
        if (v < 1) v = 1;
        const int per = (p.kblocks_total + v - 1) / v;
        splits = (p.kblocks_total + per - 1) / per;  // no empty split
    }
    // a forced split must still be one co-resident wave (the splits of a tile wait for each other)
    if (splits > 1 && tiles * splits > sms) return false;
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
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(tiles * splits, 1, 1);
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

// Returns true if the tensor-core path handled the call.
// `peers` / `n_peers`: up to 7 additional output bases (same ldc) that receive a copy of every element.
// `mt_override`: token tile (16 | 32 | 64 | 128, 0 = by M); `force_splits`: K split per tile (0 = by the grid).
template <typename T>
bool launch_gemm4_tc(const T* A, const uint8_t* B, const float* absmax, const uint8_t* absmax_8bit,
                     const float* absmax_code, const float* absmax_offset, T* out, const T* bias, int M, int N, int K,
                     int ldc, int blocksize, int quant_type, cudaStream_t stream, void* const* peers, int n_peers,
                     int mt_override, int force_splits) {
    if (n_peers < 0 || n_peers > 7) return false;
    if (M <= 0 || N <= 0) return true;
    if (K < 64 || (K % 64) != 0) return false;
    if (blocksize < 32 || (blocksize & (blocksize - 1)) != 0) return false;
    if ((reinterpret_cast<uintptr_t>(A) & 15) != 0 || (reinterpret_cast<uintptr_t>(B) & 15) != 0) return false;
    if (quant_type != kNF4 && quant_type != kFP4) return false;

    int MT = 128;
    if (M <= 16) MT = 16;
    else if (M <= 32) MT = 32;
    else if (M <= 64) MT = 64;
    if (mt_override != 0) {
        if (mt_override != 16 && mt_override != 32 && mt_override != 64 && mt_override != 128) return false;
        MT = mt_override;
    }

    Gemm4Params p{};
    p.B = B;
    p.absmax = absmax;
    p.absmax_8bit = absmax_8bit;
    p.absmax_code = absmax_code;
    p.absmax_offset = absmax_offset;
    p.bias = bias;
    p.out = out;
    p.n_peers = n_peers;
    for (int r = 0; r < n_peers; ++r) p.peer_out[r] = peers[r];
    p.M = M;
    p.N = N;
    p.K = K;
    p.ldc = ldc;
    p.log2_bs = ilog2_pow2(blocksize);
    p.kblocks_total = (K + kBK - 1) / kBK;

#define BNB200_DISPATCH_MT(QT)                                                                                         \
    switch (MT) {                                                                                                      \
    case 16: return launch_mt<T, QT, 16>(A, p, force_splits, stream);                                                  \
    case 32: return launch_mt<T, QT, 32>(A, p, force_splits, stream);                                                  \
    case 64: return launch_mt<T, QT, 64>(A, p, force_splits, stream);                                                  \
    default: return launch_mt<T, QT, 128>(A, p, force_splits, stream);                                                 \
    }
    if (quant_type == kNF4) {
        BNB200_DISPATCH_MT(kNF4)
    } else {
        BNB200_DISPATCH_MT(kFP4)
    }
#undef BNB200_DISPATCH_MT
}

template bool launch_gemm4_tc<__nv_bfloat16>(const __nv_bfloat16*, const uint8_t*, const float*, const uint8_t*,
                                             const float*, const float*, __nv_bfloat16*, const __nv_bfloat16*, int,
                                             int, int, int, int, int, cudaStream_t, void* const*, int, int, int);
template bool launch_gemm4_tc<__half>(const __half*, const uint8_t*, const float*, const uint8_t*, const float*,
                                      const float*, __half*, const __half*, int, int, int, int, int, int,
                                      cudaStream_t, void* const*, int, int, int);

} // namespace bnb200
