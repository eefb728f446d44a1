// optim.cu -- optimizer updates with 32-bit and 8-bit blockwise state (SURVEY.md section 8 row f-4).
//
// What the reference does (reference csrc/kernels.cu:531-1325, launchers csrc/ops.cu:80-210, C ABI
// csrc/pythonInterface.cpp:68-125, 446-520):
//   * 32-bit state: one element-wise pass over (g, p, state1[, state2]); optionally a first pass that accumulates the
//     squared norm of the would-be update into unorm[0] for the trust-ratio clipping of LAMB / LARS (max_unorm);
//   * 8-bit state: blocks of 256 elements; a block's state bytes are dequantised through a 256-entry code book and
//     the block's absmax, updated in fp32, the new absmax of the block is reduced, the parameters are updated, and
//     the state is re-quantised with the 7-step search of the blockwise quantizer (csrc/kernels.cu:221-267; here: its
//     bracket-table form, q8_search.cuh).
// Both are HBM-bound element-wise kernels (12-20 bytes per element), so this implementation is about access shape, not
// about the tensor cores: a warp owns one 256-element block (lane l handles the 8 consecutive elements 8 l .. 8 l + 7
// through 8- and 16-byte accesses: every load and store of the warp is one contiguous segment), the block's absmax is a warp-shuffle reduction (no shared-memory
// round trip, no __syncthreads in the loop), the two code books sit in shared memory once per CTA, and the grid is
// persistent (a multiple of the SM count).  The 32-bit kernel hands a CTA a 4096-element chunk at a time.
//
// Numerics follow the reference operation by operation, including what looks accidental there, because a state
// written by one implementation must be readable by the other:
//   * the scaled gradient is rounded to the gradient's dtype before use (32-bit kernels), the parameter is rounded
//     to its dtype BEFORE the decoupled weight decay multiplies it;
//   * the 8-bit Adam step uses div.approx and sqrt.approx (the reference is compiled with --use_fast_math: this
//     file is too, see the Makefile), a NaN / Inf gradient zeroes the element's state and skips its update;
//   * elements past n in the last block take part in the absmax with the defaults g = 0, state1 = code1[128],
//     state2 = code2[0];
//   * the sign of the first state survives quantisation (code +-1 when the nearest entry has the other sign);
//   * the 1-state RMSprop / Adagrad parameter update uses the UNSCALED gradient (csrc/kernels.cu:1271-1279).
#include "common.cuh"
#include "q8_search.cuh"

#include <cfloat>
#include <type_traits>

namespace bnb200 {

namespace {

enum OptId : int { kAdam = 0, kMomentum = 1, kRmsprop = 2, kAdagrad = 3, kLion = 4, kAdemamix = 5 };

constexpr int kOptBlock = 256;  // elements per 8-bit state block (reference BLOCKSIZE_1STATE / _2STATE)

__device__ __forceinline__ float sgnf(float v) { return (float)((0.0f < v) - (v < 0.0f)); }

template <typename T> __device__ __forceinline__ T round_to(float v) { return DT<T>::from_f32(v); }
template <typename T> __device__ __forceinline__ float widen(T v) { return DT<T>::to_f32(v); }

// ---------------------------------------------------------------------------------------------------------------
// Tensor lists
// ---------------------------------------------------------------------------------------------------------------
// Every update kernel takes a list of tensors by value, as a __grid_constant__ kernel parameter (CUDA >= 12.1 allows
// 32764 bytes of parameters on sm_70+): a single-tensor call is a list of one, a multi-tensor call updates up to
// kOptimListCap tensors in one launch, with no staging buffer to upload or keep alive.  The work items of the launch
// -- 256-element blocks (8-bit state) or kOpt32Chunk-element chunks (32-bit state) -- are numbered across the list:
// start[i] items come before tensor i, start[count] is the total, and a warp (8-bit) or CTA (32-bit) finds the tensor
// of its item by binary search.  Everything but the tensor's pointers, size and step is per launch.
//
// Capturable instances (DEV = true, the _dev entries): each descriptor carries a pointer to the tensor's step counter
// in device memory instead of the step, and the learning rate may come from a device pointer (lr_dev; NULL: s.lr), so
// a CUDA graph that captured the launch reads the current values at every replay.  The counters are advanced by
// optim_step_increment_kernel, launched just before the update on the same stream: the update kernel cannot do it,
// since other warps and CTAs of the tensor read the step.  The arithmetic is that of the DEV = false instances, on the
// same values, so the results are the same bits.
constexpr int kKernelParamBytes = 32764;
constexpr int kScalarParamBytes = 128;  // the other kernel parameters (checked below)
constexpr int kOptimListCap = (kKernelParamBytes - kScalarParamBytes - 16) / (sizeof(OptimTensor) + sizeof(long long));

struct OptimList {
    long long start[kOptimListCap + 1];
    OptimTensor t[kOptimListCap];
    int count;
};
static_assert(sizeof(OptimList) + kScalarParamBytes <= kKernelParamBytes, "kernel parameters exceed 32764 bytes");

// Peer instances (PEERS = NP > 0, the _peers entries): the step of one data-parallel rank whose tensors are pieces of a
// flat buffer that every rank holds a copy of (ZeRO stage 1, optim/sharded.py).  Each descriptor keeps the rank's own
// pieces: p and g in the local flat parameter and gradient buffers, the piece's state.  The gradient of an element is
// T(fp32(((g_0 + g_1) + ...) + g_{w-1}) * grad_scale), read at the same byte offset from the local gradient base in each
// of the w source buffers, summed in rank order and rounded once; the new parameter goes to the same offset from the
// local parameter base in each of the ndst destinations (the local buffer among them).  The rest of the update is the
// PEERS = 0 arithmetic on that gradient.  The descriptor list is shorter by the peer arguments.  NP, the compiled
// bound on the number of sources (1, 2, 4 or 8; the launch takes the least that holds w), sizes the registers that hold
// the w loads in flight, so a launch over few ranks keeps the occupancy of the PEERS = 0 instances.
constexpr int kMaxPeers = 8;
struct PeerArgs {
    const void* g[kMaxPeers];  // gradient source bases, rank order (w of them)
    void* p[kMaxPeers];        // parameter destination bases (ndst of them)
    const char* g_local;       // the local flat gradient: a descriptor's g lies at g_local + offset
    const char* p_local;       // the local flat parameters
    const float* gnorm_scale_dev;  // the clip coefficient in device memory (the _scaled entries); NULL: gnorm_scale
    float grad_scale;
    int w, ndst;
};
constexpr int kPeerListCap =
    (kKernelParamBytes - kScalarParamBytes - 16 - (int)sizeof(PeerArgs)) / (sizeof(OptimTensor) + sizeof(long long));

struct PeerOptimList {
    long long start[kPeerListCap + 1];
    OptimTensor t[kPeerListCap];
    int count;
    PeerArgs peers;
};
static_assert(sizeof(PeerOptimList) + kScalarParamBytes <= kKernelParamBytes, "kernel parameters exceed 32764 bytes");

template <int PEERS> using ListOf = std::conditional_t<(PEERS > 0), PeerOptimList, OptimList>;

// the per-launch scalars
struct OptimScalars {
    float beta1, beta2, beta3, alpha, eps, weight_decay, lr, gnorm_scale;
    bool skip_zeros;
};
static_assert(sizeof(OptimScalars) + 5 * sizeof(void*) + 2 * sizeof(float) <= kScalarParamBytes, "");

// the per-launch learning rate: from device memory in the capturable instances when given
template <bool DEV> __device__ __forceinline__ float launch_lr(const OptimScalars& s, const float* lr_dev) {
    return DEV && lr_dev != nullptr ? *lr_dev : s.lr;
}
// the per-launch gradient factor: the peer instances read a clip coefficient from device memory when given, once per
// CTA, so that a clip computed on the device needs no host round trip
template <int PEERS, typename L_>
__device__ __forceinline__ float launch_gnorm_scale(const L_& L, const OptimScalars& s) {
    if constexpr (PEERS > 0) {
        if (L.peers.gnorm_scale_dev != nullptr) return *L.peers.gnorm_scale_dev;
    }
    return s.gnorm_scale;
}
// a descriptor's step: the value (DEV = false) or the device counter it points to
template <bool DEV> __device__ __forceinline__ int tensor_step(const OptimTensor& d) {
    return DEV ? *d.step_ptr : d.step;
}

// ++step of every tensor of a capturable launch, before its update kernel
__global__ void __launch_bounds__(256) optim_step_increment_kernel(const __grid_constant__ OptimList list) {
    for (int i = threadIdx.x; i < list.count; i += blockDim.x) atomicAdd(list.t[i].step_ptr, 1);
}

// the tensor of work item `item`: the last i >= lo with start[i] <= item (tensors without items are skipped)
template <typename L_>
__device__ __forceinline__ int find_tensor(const L_& L, long long item, int lo) {
    int hi = L.count - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (L.start[mid] <= item)
            lo = mid;
        else
            hi = mid - 1;
    }
    return lo;
}

// fp32 add and multiply in IEEE round-to-nearest with subnormals kept and no contraction into an fma: this file is
// compiled with --use_fast_math (flush to zero), and the peers' gradient sum must be the one a plain fp32 sum gives
__device__ __forceinline__ float add_rn(float a, float b) {
    float r;
    asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ float mul_rn(float a, float b) {
    float r;
    asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// K consecutive elements i .. i + K - 1 of src: one or two 16-byte accesses, or one 8-byte access, when `vec` (all K in
// range, src + i aligned); otherwise element by element, 0 past n
template <typename T, int K>
__device__ __forceinline__ void load_k(const T* src, long i, long n, bool vec, T (&v)[K]) {
    constexpr int B = K * (int)sizeof(T);
    if constexpr (B % 16 == 0) {
        if (vec) {
#pragma unroll
            for (int c = 0; c < B / 16; ++c) reinterpret_cast<uint4*>(v)[c] = reinterpret_cast<const uint4*>(src + i)[c];
            return;
        }
    } else if constexpr (B == 8) {
        if (vec) {
            *reinterpret_cast<uint2*>(v) = *reinterpret_cast<const uint2*>(src + i);
            return;
        }
    }
#pragma unroll
    for (int j = 0; j < K; ++j) v[j] = (i + j < n) ? src[i + j] : round_to<T>(0.0f);
}
template <typename T, int K>
__device__ __forceinline__ void store_k(T* dst, long i, long n, bool vec, const T (&v)[K]) {
    constexpr int B = K * (int)sizeof(T);
    if constexpr (B % 16 == 0) {
        if (vec) {
#pragma unroll
            for (int c = 0; c < B / 16; ++c) reinterpret_cast<uint4*>(dst + i)[c] = reinterpret_cast<const uint4*>(v)[c];
            return;
        }
    } else if constexpr (B == 8) {
        if (vec) {
            *reinterpret_cast<uint2*>(dst + i) = *reinterpret_cast<const uint2*>(v);
            return;
        }
    }
#pragma unroll
    for (int j = 0; j < K; ++j)
        if (i + j < n) dst[i + j] = v[j];
}

// Elements i .. i + K - 1 of a piece's gradient, the piece `goff` bytes from the local gradient base: the w <= NP
// sources' values are all loaded before the rank-order fp32 sum, scaled by grad_scale and rounded once to T
template <typename T, int K, int NP>
__device__ __forceinline__ void peer_grad(const PeerArgs& P, long goff, long i, long n, bool vec, T (&v)[K]) {
    alignas(K * sizeof(T) < 16 ? K * sizeof(T) : 16) T x[NP][K];
#pragma unroll
    for (int r = 0; r < NP; ++r)
        if (r < P.w) load_k<T, K>(reinterpret_cast<const T*>(static_cast<const char*>(P.g[r]) + goff), i, n, vec, x[r]);
#pragma unroll
    for (int j = 0; j < K; ++j) {
        float acc = widen<T>(x[0][j]);
#pragma unroll
        for (int r = 1; r < NP; ++r)
            if (r < P.w) acc = add_rn(acc, widen<T>(x[r][j]));
        v[j] = round_to<T>(mul_rn(acc, P.grad_scale));
    }
}

// the new parameter values of elements i .. i + K - 1 of a piece `poff` bytes from the local parameter base, to every
// destination
template <typename T, int K>
__device__ __forceinline__ void peer_store(const PeerArgs& P, long poff, long i, long n, bool vec, const T (&v)[K]) {
#pragma unroll
    for (int r = 0; r < kMaxPeers; ++r)
        if (r < P.ndst) store_k<T, K>(reinterpret_cast<T*>(static_cast<char*>(P.p[r]) + poff), i, n, vec, v);
}

// every base 16-byte aligned: then a piece's vector accesses are aligned in every buffer when they are in the local one
__device__ __forceinline__ bool peers_aligned(const PeerArgs& P) {
    uintptr_t bits = reinterpret_cast<uintptr_t>(P.g_local) | reinterpret_cast<uintptr_t>(P.p_local);
    for (int r = 0; r < P.w; ++r) bits |= reinterpret_cast<uintptr_t>(P.g[r]);
    for (int r = 0; r < P.ndst; ++r) bits |= reinterpret_cast<uintptr_t>(P.p[r]);
    return (bits & 15) == 0;
}

// ---------------------------------------------------------------------------------------------------------------
// The norm of the reduced gradient (gradient clipping over data-parallel ranks)
// ---------------------------------------------------------------------------------------------------------------
// peer_norm_kernel forms every element's gradient with peer_grad, the values the peer update will use, and
// accumulates widen(g)^2 (L2; exact in fp64 for fp32, fp16 and bf16 values) or max |g| (INF; NaN wins) in fp64.  A CTA
// takes kOpt32Chunk-element chunks of the list, each thread in a fixed order; the block's sum is a fixed shuffle tree,
// written to partials[blockIdx.x].  peer_norm_add_kernel then adds the partials in index order into *acc, in stream
// order after earlier launches: the result does not depend on timing, and one value can collect several dtype flats
// and capacity chunks.  No floating-point atomics.
constexpr int kNormThreads = 512;
constexpr int kNormChunk = 4096;  // elements per work item

// fp32 <-> fp64 without flushing subnormals (this file is compiled with --use_fast_math, i.e. -ftz)
__device__ __forceinline__ double widen64(float v) {
    double r;
    asm("cvt.f64.f32 %0, %1;" : "=d"(r) : "f"(v));
    return r;
}
__device__ __forceinline__ float narrow_rn(double v) {
    float r;
    asm("cvt.rn.f32.f64 %0, %1;" : "=f"(r) : "d"(v));
    return r;
}
// max with NaN propagation (fmax would drop a NaN)
__device__ __forceinline__ double nan_max(double a, double b) { return (a != a || a > b) ? a : b; }
template <bool INF> __device__ __forceinline__ double norm_fold(double acc, double x) {
    return INF ? nan_max(acc, fabs(x)) : fma(x, x, acc);  // (x * x is exact: the fma rounds only the sum)
}

template <typename T, int NP, bool INF>
__global__ void __launch_bounds__(kNormThreads) peer_norm_kernel(const __grid_constant__ PeerOptimList list,
                                                                 double* partials) {
    constexpr int K = 16 / (int)sizeof(T);  // elements per 16-byte access
    __shared__ double wsum[kNormThreads / 32];
    const PeerArgs& P = list.peers;
    const bool peers_vec = peers_aligned(P);
    const long long total = list.start[list.count];
    double acc = 0.0;
    int ti = 0;
    for (long long item = blockIdx.x; item < total; item += gridDim.x) {
        ti = find_tensor(list, item, ti);
        const OptimTensor& d = list.t[ti];
        const long n = d.n;
        const long goff = static_cast<const char*>(d.g) - P.g_local;
        const long c0 = (item - list.start[ti]) * kNormChunk;
        const long c1 = c0 + kNormChunk < n ? c0 + kNormChunk : n;
        if (peers_vec && (reinterpret_cast<uintptr_t>(d.g) & 15) == 0) {
            for (long i = c0 + K * threadIdx.x; i < c1; i += K * blockDim.x) {
                alignas(16) T v[K];
                peer_grad<T, K, NP>(P, goff, i, n, i + K <= n, v);  // (past n: zeros)
#pragma unroll
                for (int j = 0; j < K; ++j) acc = norm_fold<INF>(acc, widen64(widen<T>(v[j])));
            }
        } else {
            for (long i = c0 + threadIdx.x; i < c1; i += blockDim.x) {
                T v[1];
                peer_grad<T, 1, NP>(P, goff, i, n, false, v);
                acc = norm_fold<INF>(acc, widen64(widen<T>(v[0])));
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double other = __shfl_xor_sync(0xffffffffu, acc, o);
        acc = INF ? nan_max(acc, other) : acc + other;
    }
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        double v = threadIdx.x < (blockDim.x >> 5) ? wsum[threadIdx.x] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double other = __shfl_xor_sync(0xffffffffu, v, o);
            v = INF ? nan_max(v, other) : v + other;
        }
        if (threadIdx.x == 0) partials[blockIdx.x] = v;
    }
}

template <bool INF>
__global__ void __launch_bounds__(32) peer_norm_add_kernel(const double* partials, int n, double* acc) {
    if (threadIdx.x != 0) return;
    double s = *acc;
    for (int i = 0; i < n; ++i) s = INF ? nan_max(s, partials[i]) : s + partials[i];
    *acc = s;
}

// The global norm and the clip coefficient from the w ranks' values (rank order): for L2 the fp64 sum, its fp64
// square root rounded once to fp32; for INF the max.  The coefficient is, in fp32 and with torch's operations,
// min((1 / (total_norm + 1e-6)) * max_norm, 1) (`max_norm / t` on a tensor is a reciprocal and a multiply), NaN kept.
template <bool INF>
__global__ void __launch_bounds__(32) clip_coef_kernel(const double* values, int w, float max_norm, float* out) {
    if (threadIdx.x != 0) return;
    double t = values[0];
    for (int r = 1; r < w; ++r) t = INF ? nan_max(t, values[r]) : t + values[r];
    const float norm = narrow_rn(INF ? t : __dsqrt_rn(t));
    float rcp;
    asm("rcp.rn.f32 %0, %1;" : "=f"(rcp) : "f"(add_rn(norm, (float)1e-6)));
    const float coef = mul_rn(rcp, max_norm);
    out[0] = norm;
    out[1] = coef > 1.0f ? 1.0f : coef;
}

// ---------------------------------------------------------------------------------------------------------------
// 32-bit state
// ---------------------------------------------------------------------------------------------------------------
// first pass for max_unorm > 0: unorm[0] += sum of update^2 (reference csrc/kernels.cu:531-603, 729-804)
template <typename T, int OPT>
__global__ void __launch_bounds__(512) optim32_unorm_kernel(const T* g, const float* s1, const float* s2, float* unorm,
                                                            float beta1, float beta2, float eps, int step,
                                                            float gnorm_scale, long n) {
    __shared__ float wsum[16];
    const float correction1 = 1.0f / (1.0f - powf(beta1, step));
    const float correction2 = 1.0f / (1.0f - powf(beta2, step));
    float acc = 0.f;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float gv = widen<T>(round_to<T>(gnorm_scale * widen<T>(g[i])));
        float a = s1[i];
        switch (OPT) {
        case kAdam: {
            float b = s2[i];
            a = a * beta1 + ((1.0f - beta1) * gv);
            b = b * beta2 + ((1.0f - beta2) * (gv * gv));
            a *= correction1;
            b *= correction2;
            a = a / (sqrtf(b) + eps);
            a *= a;
            break;
        }
        case kMomentum:
            a = (step == 1) ? gv : a * beta1 + gv;
            a = a * a;
            break;
        case kLion:
            a = a * beta2 + ((1.0f - beta2) * gv);  // (not squared: as the reference)
            break;
        case kRmsprop:
            a = a * beta1 + ((1.0f - beta1) * gv * gv);
            a = __fdividef(gv, sqrtf(a) + eps);
            a = a * a;
            break;
        case kAdagrad:
            a = a + gv * gv;
            a = __fdividef(gv, sqrtf(a) + eps);
            a = a * a;
            break;
        default:  // AdEMAMix: no trust ratio
            a = 0.f;
            break;
        }
        acc += a;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? wsum[threadIdx.x] : 0.f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (threadIdx.x == 0) atomicAdd(unorm, v);
    }
}

// One element of the 32-bit update (reference csrc/kernels.cu:605-727 two states, 806-909 one state).  gt / pt are
// the gradient and the parameter in their storage type; a, b, c the states (c: AdEMAMix's slow EMA).
struct Opt32Args {
    float beta1, beta2, beta3, alpha, eps, weight_decay, lr, gnorm_scale;
    float correction1, correction2, step_size, update_scale;
    int step;
    bool skip_zeros;
};

template <typename T, int OPT>
__device__ __forceinline__ void opt32_element(const Opt32Args& q, T gt, T& pt, float& a, float& b, float& c) {
    gt = round_to<T>(q.gnorm_scale * widen<T>(gt));
    if (OPT == kAdemamix) {
        const float gv = widen<T>(gt);
        a = (a * q.beta1) + ((1.0f - q.beta1) * gv);
        c = (c * q.beta3) + ((1.0f - q.beta3) * gv);
        b = (b * q.beta2) + ((1.0f - q.beta2) * gv * gv);
        pt = round_to<T>(widen<T>(pt) -
                         q.lr * (((a / q.correction1) + (q.alpha * c)) / ((sqrtf(b) / q.correction2) + q.eps)));
        if (q.weight_decay > 0.0f) pt = round_to<T>(widen<T>(pt) * (1.0f - (q.lr * q.weight_decay)));
    } else if (OPT == kAdam) {
        const float gv = widen<T>(gt);
        if (!q.skip_zeros || gv != 0.0f) {
            a = a * q.beta1 + ((1.0f - q.beta1) * gv);
            b = b * q.beta2 + ((1.0f - q.beta2) * (gv * gv));
            pt = round_to<T>(widen<T>(pt) +
                             (q.update_scale * q.step_size * (a / (sqrtf(b) + (q.eps * q.correction2)))));
            if (q.weight_decay > 0.0f) pt = round_to<T>(widen<T>(pt) * (1.0f - (q.lr * q.weight_decay)));
        }
    } else {
        // coupled (L2) weight decay folds into the gradient -- not for Lion, which decays the parameter
        if (q.weight_decay > 0.0f && OPT != kLion) gt = round_to<T>(widen<T>(gt) + (widen<T>(pt) * q.weight_decay));
        const float gv = widen<T>(gt);
        if (!q.skip_zeros || gv != 0.0f) {
            switch (OPT) {
            case kMomentum:
                a = (q.step == 1) ? gv : a * q.beta1 + gv;
                pt = round_to<T>(widen<T>(pt) + q.update_scale * (-q.lr * a));
                break;
            case kLion:
                if (q.weight_decay > 0.0f) pt = round_to<T>(widen<T>(pt) * (1.0f - q.lr * q.weight_decay));
                pt = round_to<T>(widen<T>(pt) - q.update_scale * (q.lr * sgnf(a * q.beta1 + ((1.0f - q.beta1) * gv))));
                a = a * q.beta2 + ((1.0f - q.beta2) * gv);
                break;
            case kRmsprop:
                a = a * q.beta1 + ((1.0f - q.beta1) * gv * gv);
                pt = round_to<T>(widen<T>(pt) - q.update_scale * (q.lr * __fdividef(gv, sqrtf(a) + q.eps)));
                break;
            case kAdagrad:
                a = a + gv * gv;
                pt = round_to<T>(widen<T>(pt) - q.lr * __fdividef(gv, sqrtf(a) + q.eps));
                break;
            }
        }
    }
}

template <typename T> struct Vec4;  // four consecutive elements of T as one 8- or 16-byte access
template <> struct Vec4<float> { using type = float4; };
template <> struct Vec4<__half> { using type = uint2; };
template <> struct Vec4<__nv_bfloat16> { using type = uint2; };

constexpr int kOpt32Chunk = 4096;  // elements per work item of the 32-bit kernel: two passes of a 512-thread CTA

// A CTA per chunk of kOpt32Chunk elements of one tensor.  16-bit parameters whose pointers are all aligned (and, for
// AdEMAMix, whose size is a multiple of 4: s1 + n + i is 16-byte aligned only then): four consecutive elements per
// thread and iteration through 8- / 16-byte accesses -- there the rounding to T hides how the compiler contracts an
// fma, and the vector path is bit-identical to the scalar one (and to the reference); fp32 already moves 128 bytes
// per warp access.  Otherwise one element per access.  The choice is made per tensor, so a misaligned view in the list
// does not demote the others.  max_unorm > 0 (LAMB / LARS) takes a list of one: unorm and param_norm belong to it.
template <typename T, int OPT, bool DEV, int PEERS = 0>
__global__ void __launch_bounds__(512, PEERS > 0 ? 1 : 0) optim32_kernel(const __grid_constant__ ListOf<PEERS> list, const OptimScalars s,
                                                      const float* unorm, float max_unorm, float param_norm,
                                                      const float* lr_dev) {
    constexpr bool two = OPT == kAdam || OPT == kAdemamix;
    Opt32Args q;
    q.beta1 = s.beta1, q.beta2 = s.beta2, q.beta3 = s.beta3, q.alpha = s.alpha, q.eps = s.eps;
    q.weight_decay = s.weight_decay, q.lr = launch_lr<DEV>(s, lr_dev), q.gnorm_scale = launch_gnorm_scale<PEERS>(list, s);
    q.skip_zeros = s.skip_zeros;
    q.update_scale = 1.0f;
    if (max_unorm > 0.0f) {
        const float us = sqrtf(unorm[0]);
        const float cap = two ? max_unorm * param_norm : max_unorm * param_norm + s.eps;
        q.update_scale = us > cap ? cap / us : 1.0f;
    }
    const long long total = list.start[list.count];
    bool peers_vec = true;
    if constexpr (PEERS) peers_vec = peers_aligned(list.peers);
    int ti = 0;
    for (long long item = blockIdx.x; item < total; item += gridDim.x) {
        ti = find_tensor(list, item, ti);
        const OptimTensor& d = list.t[ti];
        const T* g = static_cast<const T*>(d.g);
        T* p = static_cast<T*>(d.p);
        float* s1 = static_cast<float*>(d.state1);
        float* s2 = static_cast<float*>(d.state2);
        const long n = d.n;
        q.step = tensor_step<DEV>(d);
        q.correction1 = 1.0f - powf(q.beta1, q.step);
        q.correction2 = sqrtf(1.0f - powf(q.beta2, q.step));
        q.step_size = -q.lr * q.correction2 / q.correction1;
        const long c0 = (item - list.start[ti]) * kOpt32Chunk;
        const long c1 = c0 + kOpt32Chunk < n ? c0 + kOpt32Chunk : n;
        long goff = 0, poff = 0;  // (PEERS) the piece's byte offsets in the flat buffers
        if constexpr (PEERS) {
            goff = reinterpret_cast<const char*>(g) - list.peers.g_local;
            poff = reinterpret_cast<const char*>(p) - list.peers.p_local;
        }
        auto one = [&](long i) {
            T pt = p[i];
            float a = s1[i], b = two ? s2[i] : 0.f, c = OPT == kAdemamix ? s1[n + i] : 0.f;
            if constexpr (PEERS) {
                T gt[1], pn[1];
                peer_grad<T, 1, PEERS>(list.peers, goff, i, n, false, gt);
                opt32_element<T, OPT>(q, gt[0], pt, a, b, c);
                pn[0] = pt;
                peer_store<T, 1>(list.peers, poff, i, n, false, pn);
            } else {
                opt32_element<T, OPT>(q, g[i], pt, a, b, c);
                p[i] = pt;
            }
            s1[i] = a;
            if (two) s2[i] = b;
            if (OPT == kAdemamix) s1[n + i] = c;
        };
        auto al = [](const void* v, uintptr_t m) { return (reinterpret_cast<uintptr_t>(v) & m) == 0; };
        const bool vec = sizeof(T) == 2 && al(g, sizeof(T) * 4 - 1) && al(p, sizeof(T) * 4 - 1) && al(s1, 15) &&
                         al(s2, 15) && (OPT != kAdemamix || (n & 3) == 0) && peers_vec;
        if (vec) {
            using V = typename Vec4<T>::type;
            for (long i = c0 + 4 * threadIdx.x; i < c1; i += 4 * blockDim.x) {
                if (i + 4 > n) {  // the last n % 4 elements
                    for (long j = i; j < n; ++j) one(j);
                    break;
                }
                V gv4;
                if constexpr (PEERS)
                    peer_grad<T, 4, PEERS>(list.peers, goff, i, n, true, *reinterpret_cast<T(*)[4]>(&gv4));
                else
                    gv4 = *reinterpret_cast<const V*>(g + i);
                V pv4 = *reinterpret_cast<const V*>(p + i);
                float4 a4 = *reinterpret_cast<const float4*>(s1 + i);
                float4 b4 = two ? *reinterpret_cast<const float4*>(s2 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                float4 c4 = OPT == kAdemamix ? *reinterpret_cast<const float4*>(s1 + n + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                T* gt = reinterpret_cast<T*>(&gv4);
                T* pt = reinterpret_cast<T*>(&pv4);
                float* a = reinterpret_cast<float*>(&a4);
                float* b = reinterpret_cast<float*>(&b4);
                float* c = reinterpret_cast<float*>(&c4);
#pragma unroll
                for (int k = 0; k < 4; ++k) opt32_element<T, OPT>(q, gt[k], pt[k], a[k], b[k], c[k]);
                if constexpr (PEERS)
                    peer_store<T, 4>(list.peers, poff, i, n, true, *reinterpret_cast<const T(*)[4]>(&pv4));
                else
                    *reinterpret_cast<V*>(p + i) = pv4;
                *reinterpret_cast<float4*>(s1 + i) = a4;
                if (two) *reinterpret_cast<float4*>(s2 + i) = b4;
                if (OPT == kAdemamix) *reinterpret_cast<float4*>(s1 + n + i) = c4;
            }
        } else {
            for (long i = c0 + threadIdx.x; i < c1; i += blockDim.x) one(i);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// 8-bit blockwise state
// ---------------------------------------------------------------------------------------------------------------
// Nearest entry of a sorted 256-entry code book.  The reference walks 7 steps from pivot 127 and applies a midpoint
// rule (csrc/kernels.cu:221-267: eight dependent shared-memory reads per value, two values per element); here the
// bracket-table form of q8_search.cuh returns the same code (proved for every fp32 input of magnitude <= 1 + 2^-20,
// NaN included, and any sorted code book: tools/micro/q8_lut_equiv.c) from one bracket read, a 0..3-step scan and one
// decision-table read.  The tables are built once per (persistent) CTA.
struct CodeBook {
    const float* code;     // [256]
    const float2* fin;     // [257] decision table
    const uint32_t* br;    // [kQ8Cells] bracket table
    // Domain of the proof: |x| <= 1 + 2^-20, or NaN.  x = div.approx.ftz(state, absmax) with |state| <= absmax, so
    // |x| <= 1 up to 2 ulp; a denormal absmax is flushed to zero TOGETHER with the (then also denormal) state: 0 / 0 =
    // NaN, never an infinity.
    __device__ __forceinline__ int search(float x) const { return (int)quantize_8bit_fast(code, fin, br, x); }
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// state1 code with the sign of the value kept (reference csrc/kernels.cu:1118-1125)
__device__ __forceinline__ unsigned char quant_signed(const CodeBook& cb, float s, float absmax) {
    int c = cb.search(__fdividef(s, absmax));
    if (signbit(cb.code[c]) != signbit(s)) c += (s > 0.0f) ? 1 : -1;
    return (unsigned char)c;
}

// A lane's 8 consecutive elements of a 256-element block (element j of lane l: base + 8 l + j): one 16-byte (T = 2
// bytes) or two 16-byte (fp32) accesses per tensor and an 8-byte access per state, when the block is whole and the
// pointers are aligned (`vec`); element by element with the reference's padding defaults otherwise.
template <typename T> __device__ __forceinline__ void load8(const T* src, long i0, long n, bool vec, T fill, T (&v)[8]) {
    if (vec) {
        if (sizeof(T) == 2) {
            *reinterpret_cast<uint4*>(v) = *reinterpret_cast<const uint4*>(src + i0);
        } else {
            reinterpret_cast<uint4*>(v)[0] = reinterpret_cast<const uint4*>(src + i0)[0];
            reinterpret_cast<uint4*>(v)[1] = reinterpret_cast<const uint4*>(src + i0)[1];
        }
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (i0 + j < n) ? src[i0 + j] : fill;
    }
}
template <typename T> __device__ __forceinline__ void store8(T* dst, long i0, long n, bool vec, const T (&v)[8]) {
    if (vec) {
        if (sizeof(T) == 2) {
            *reinterpret_cast<uint4*>(dst + i0) = *reinterpret_cast<const uint4*>(v);
        } else {
            reinterpret_cast<uint4*>(dst + i0)[0] = reinterpret_cast<const uint4*>(v)[0];
            reinterpret_cast<uint4*>(dst + i0)[1] = reinterpret_cast<const uint4*>(v)[1];
        }
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (i0 + j < n) dst[i0 + j] = v[j];
    }
}
__device__ __forceinline__ void load8c(const unsigned char* src, long i0, long n, bool vec, unsigned char fill,
                                       unsigned char (&v)[8]) {
    if (vec) {
        *reinterpret_cast<uint2*>(v) = *reinterpret_cast<const uint2*>(src + i0);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (i0 + j < n) ? src[i0 + j] : fill;
    }
}
__device__ __forceinline__ void store8c(unsigned char* dst, long i0, long n, bool vec, const unsigned char (&v)[8]) {
    if (vec) {
        *reinterpret_cast<uint2*>(dst + i0) = *reinterpret_cast<const uint2*>(v);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (i0 + j < n) dst[i0 + j] = v[j];
    }
}

// A warp per work item, i.e. per (tensor, 256-element block) of the list, and the fields of the item's tensor.  Kept
// in registers across items these would cost registers (and occupancy) that kernel parameters do not: a warp reads
// them from the parameter space for every item.  ONE: a list of one tensor (the single-tensor entries); the tensor
// index is then the constant 0, so the fields and the per-step values are loop invariants, as in a kernel that takes
// one tensor's pointers as its parameters.
template <typename T> struct Tensor8 {
    T* p;
    const T* g;
    unsigned char* state1;
    unsigned char* state2;  // (NULL for one-state optimizers)
    float* absmax1;
    float* absmax2;
    long n;
    long long first;  // the list's number of its block 0
    int step;
    bool aligned;     // 16-byte p / g and 8-byte state accesses allowed

    template <bool DEV, typename L_> __device__ __forceinline__ void load(const L_& L, int i) {
        const OptimTensor& d = L.t[i];
        p = static_cast<T*>(d.p);
        g = static_cast<const T*>(d.g);
        state1 = static_cast<unsigned char*>(d.state1);
        state2 = static_cast<unsigned char*>(d.state2);
        absmax1 = d.absmax1;
        absmax2 = d.absmax2;
        n = d.n;
        first = L.start[i];
        step = tensor_step<DEV>(d);
        aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g)) & 15) == 0 &&
                  ((reinterpret_cast<uintptr_t>(state1) | reinterpret_cast<uintptr_t>(state2)) & 7) == 0;
    }
};

// reference csrc/kernels.cu:914-1150
template <typename T, int OPT, bool ONE, bool DEV, int PEERS = 0>
__global__ void __launch_bounds__(256, PEERS > 0 ? 1 : 0) optim8_2state_kernel(const __grid_constant__ ListOf<PEERS> list, const OptimScalars s,
                                                            const float* qmap1, const float* qmap2,
                                                            const float* lr_dev) {
    const float beta1 = s.beta1, beta2 = s.beta2, beta3 = s.beta3, alpha = s.alpha, eps = s.eps;
    const float lr = launch_lr<DEV>(s, lr_dev);
    const float weight_decay = s.weight_decay, gnorm_scale = launch_gnorm_scale<PEERS>(list, s);
    __shared__ float code1[256];
    __shared__ float code2[256];
    __shared__ float2 fin1[257], fin2[257];
    __shared__ uint32_t br1[kQ8Cells], br2[kQ8Cells];
    code1[threadIdx.x] = qmap1[threadIdx.x];
    code2[threadIdx.x] = qmap2[threadIdx.x];
    __syncthreads();
    build_q8_bracket(code1, br1);
    build_q8_final(code1, fin1);
    build_q8_bracket(code2, br2);
    build_q8_final(code2, fin2);
    __syncthreads();
    const CodeBook cb1{code1, fin1, br1}, cb2{code2, fin2, br2};
    // (s.skip_zeros: the reference's 2-state kernel ignores it too)
    const int lane = threadIdx.x & 31;
    const long long total = list.start[list.count];
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    bool peers_vec = true;
    if constexpr (PEERS) peers_vec = peers_aligned(list.peers);
    int ti = 0;
    for (long long item = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); item < total; item += warps) {
        ti = ONE ? 0 : find_tensor(list, item, ti);
        Tensor8<T> t;
        t.template load<DEV>(list, ti);
        const float correction1 = 1.0f - __powf(beta1, t.step);
        const float correction2 = sqrtf(1.0f - __powf(beta2, t.step));
        const float step_size = __fdividef(-lr * correction2, correction1);
        T* p = t.p;
        const T* g = t.g;
        unsigned char* state1 = t.state1;
        unsigned char* state2 = t.state2;
        float* absmax1 = t.absmax1;
        float* absmax2 = t.absmax2;
        const long n = t.n, blk = (long)(item - t.first);
        const bool aligned = t.aligned;
        const long base = blk * kOptBlock;
        const float am1 = absmax1[blk], am2 = absmax2[blk];
        const float am3 = OPT == kAdemamix ? absmax1[(n + base) / kOptBlock] : 0.f;
        const long i0 = base + lane * 8;
        const bool vec = aligned && base + kOptBlock <= n && peers_vec;
        alignas(16) T gts[8];
        alignas(16) T pts[8];
        alignas(8) unsigned char c1s[8], c2s[8], c3s[8];
        if constexpr (PEERS)
            peer_grad<T, 8, PEERS>(list.peers, reinterpret_cast<const char*>(g) - list.peers.g_local, i0, n, vec, gts);
        else
            load8<T>(g, i0, n, vec, round_to<T>(0.0f), gts);
        load8c(state1, i0, n, vec, 128, c1s);
        load8c(state2, i0, n, vec, 0, c2s);
        if (OPT == kAdemamix) load8c(state1 + n, i0, n, vec && (n & 7) == 0, 128, c3s);
        float s1[8], s2[8], s3[8];
        bool finite[8];
        float m1 = -FLT_MAX, m2 = -FLT_MAX, m3 = -FLT_MAX;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float gf = widen<T>(gts[j]);
            finite[j] = !isnan(gf) && !isinf(gf);
            if (finite[j]) {
                s2[j] = code2[c2s[j]] * am2;
                const float gs = gf * gnorm_scale;
                s2[j] = (s2[j] * beta2) + (((1.0f - beta2) * gs * gs));
                s1[j] = code1[c1s[j]] * am1;
                s1[j] = (s1[j] * beta1) + (((1.0f - beta1) * gs));
                if (OPT == kAdemamix) {
                    s3[j] = code1[c3s[j]] * am3;
                    s3[j] = (s3[j] * beta3) + (((1.0f - beta3) * gs));
                }
            } else {
                s1[j] = s2[j] = s3[j] = 0.0f;
            }
            m1 = fmaxf(m1, fabsf(s1[j]));
            m2 = fmaxf(m2, fabsf(s2[j]));
            if (OPT == kAdemamix) m3 = fmaxf(m3, fabsf(s3[j]));
        }
        m1 = warp_max(m1);
        m2 = warp_max(m2);
        if (OPT == kAdemamix) m3 = warp_max(m3);
        if (lane == 0) {
            absmax1[blk] = m1;
            absmax2[blk] = m2;
            if (OPT == kAdemamix) absmax1[(n + base) / kOptBlock] = m3;
        }
        load8<T>(p, i0, n, vec, round_to<T>(0.0f), pts);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (finite[j]) {
                T pt = pts[j];
                if (OPT == kAdemamix)
                    pt = round_to<T>(widen<T>(pt) - lr * (((s1[j] / correction1) + (alpha * s3[j])) /
                                                          ((sqrtf(s2[j]) / correction2) + eps)));
                else
                    pt = round_to<T>(widen<T>(pt) +
                                     ((step_size * (__fdividef(s1[j], (sqrtf(s2[j]) + (correction2 * eps)))))));
                if (weight_decay > 0.0f) pt = round_to<T>(widen<T>(pt) * (1.0f - (lr * weight_decay)));
                pts[j] = pt;
            }
            c1s[j] = quant_signed(cb1, s1[j], m1);
            c2s[j] = (unsigned char)cb2.search(__fdividef(s2[j], m2));
            if (OPT == kAdemamix) c3s[j] = quant_signed(cb1, s3[j], m3);
        }
        if constexpr (PEERS)
            peer_store<T, 8>(list.peers, reinterpret_cast<const char*>(p) - list.peers.p_local, i0, n, vec, pts);
        else
            store8<T>(p, i0, n, vec, pts);
        store8c(state1, i0, n, vec, c1s);
        store8c(state2, i0, n, vec, c2s);
        if (OPT == kAdemamix) store8c(state1 + n, i0, n, vec && (n & 7) == 0, c3s);
    }
}

// reference csrc/kernels.cu:1152-1325
template <typename T, int OPT, bool ONE, bool DEV, int PEERS = 0>
__global__ void __launch_bounds__(256, PEERS > 0 ? 1 : 0) optim8_1state_kernel(const __grid_constant__ ListOf<PEERS> list, const OptimScalars s,
                                                            const float* qmap1, const float* lr_dev) {
    const float beta1 = s.beta1, beta2 = s.beta2, eps = s.eps, weight_decay = s.weight_decay;
    const float lr = launch_lr<DEV>(s, lr_dev);
    const float gnorm_scale = launch_gnorm_scale<PEERS>(list, s);
    const bool skip_zeros = s.skip_zeros;
    __shared__ float code1[256];
    __shared__ float2 fin1[257];
    __shared__ uint32_t br1[kQ8Cells];
    code1[threadIdx.x] = qmap1[threadIdx.x];
    __syncthreads();
    build_q8_bracket(code1, br1);
    build_q8_final(code1, fin1);
    __syncthreads();
    const CodeBook cb1{code1, fin1, br1};
    const int lane = threadIdx.x & 31;
    const long long total = list.start[list.count];
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    bool peers_vec = true;
    if constexpr (PEERS) peers_vec = peers_aligned(list.peers);
    int ti = 0;
    for (long long item = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); item < total; item += warps) {
        ti = ONE ? 0 : find_tensor(list, item, ti);
        Tensor8<T> t;
        t.template load<DEV>(list, ti);
        T* p = t.p;
        const T* g = t.g;
        unsigned char* state1 = t.state1;
        float* absmax1 = t.absmax1;
        const long n = t.n, blk = (long)(item - t.first);
        const int step = t.step;
        const bool aligned = t.aligned;
        const long base = blk * kOptBlock;
        const float am1 = absmax1[blk];
        const long i0 = base + lane * 8;
        const bool vec = aligned && base + kOptBlock <= n && peers_vec;
        alignas(16) T gts[8];
        alignas(16) T pts[8];
        alignas(8) unsigned char c1s[8];
        if constexpr (PEERS)
            peer_grad<T, 8, PEERS>(list.peers, reinterpret_cast<const char*>(g) - list.peers.g_local, i0, n, vec, gts);
        else
            load8<T>(g, i0, n, vec, round_to<T>(0.0f), gts);
        load8<T>(p, i0, n, vec, round_to<T>(0.0f), pts);
        load8c(state1, i0, n, vec, 128, c1s);
        float s1[8];
        bool act[8];
        float m1 = -FLT_MAX;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float gs = widen<T>(gts[j]) * gnorm_scale;
            act[j] = !skip_zeros || widen<T>(gts[j]) != 0.0f;
            s1[j] = code1[c1s[j]] * am1;  // (an element skipped for a zero gradient keeps its state)
            if (act[j]) {
                if (weight_decay > 0.0f) {
                    if (OPT == kLion)
                        pts[j] = round_to<T>(widen<T>(pts[j]) * (1.0f - lr * weight_decay));
                    else
                        gs += widen<T>(pts[j]) * weight_decay;
                }
                switch (OPT) {
                case kMomentum:
                    s1[j] = (step == 1) ? gs : (s1[j] * beta1) + gs;
                    break;
                case kLion:
                    // the gradient slot carries lr * sign(...) to the parameter update, in the gradient's dtype
                    gts[j] = round_to<T>(lr * sgnf(s1[j] * beta1 + ((1.0f - beta1) * gs)));
                    s1[j] = s1[j] * beta2 + ((1.0f - beta2) * gs);
                    break;
                case kRmsprop:
                    s1[j] = s1[j] * beta1 + ((1.0f - beta1) * (gs * gs));
                    break;
                case kAdagrad:
                    s1[j] = s1[j] + (gs * gs);
                    break;
                }
            }
            m1 = fmaxf(m1, fabsf(s1[j]));
        }
        m1 = warp_max(m1);
        if (lane == 0) absmax1[blk] = m1;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (act[j]) {
                T pt = pts[j];
                switch (OPT) {
                case kMomentum:
                    pt = round_to<T>(widen<T>(pt) - lr * s1[j]);
                    break;
                case kLion:
                    pt = round_to<T>(widen<T>(pt) - widen<T>(gts[j]));
                    break;
                case kRmsprop:
                case kAdagrad:
                    pt = round_to<T>(widen<T>(pt) - lr * (__fdividef(widen<T>(gts[j]), sqrtf(s1[j]) + eps)));
                    break;
                }
                pts[j] = pt;
            }
            c1s[j] = quant_signed(cb1, s1[j], m1);
        }
        if constexpr (PEERS)
            peer_store<T, 8>(list.peers, reinterpret_cast<const char*>(p) - list.peers.p_local, i0, n, vec, pts);
        else
            store8<T>(p, i0, n, vec, pts);
        store8c(state1, i0, n, vec, c1s);
    }
}

int grid_for(long work_items, int per_cta) {
    long ctas = (work_items + per_cta - 1) / per_cta;
    const long cap = 8L * device_sm_count();
    if (ctas > cap) ctas = cap;
    return ctas < 1 ? 1 : (int)ctas;
}

// the list of a launch: the tensors and the work-item prefix counts; returns the number of work items
template <typename L_> long long make_list(L_& L, const OptimTensor* ts, int count, long long per_item) {
    long long total = 0;
    for (int i = 0; i < count; ++i) {
        L.t[i] = ts[i];
        L.start[i] = total;
        total += ts[i].n > 0 ? (ts[i].n + per_item - 1) / per_item : 0;
    }
    L.start[count] = total;
    L.count = count;
    return total;
}

// The step counters of a capturable launch (dev): advanced before the update, also those of empty tensors, as the
// eager optimizer advances every step it updates.
void increment_steps(const OptimList& L, bool dev, cudaStream_t stream) {
    if (dev && L.count > 0) optim_step_increment_kernel<<<1, 256, 0, stream>>>(L);
}

// count <= kOptimListCap; unorm / max_unorm / param_norm: the LAMB / LARS trust ratio of a list of one (max_unorm = 0
// otherwise); dev: the descriptors carry step pointers and lr_dev (if not NULL) replaces s.lr
template <typename T, int OPT>
void run32(const OptimTensor* ts, int count, const OptimScalars& s, float* unorm, float max_unorm, float param_norm,
           bool dev, const float* lr_dev, cudaStream_t stream) {
    OptimList L;
    const long long chunks = make_list(L, ts, count, kOpt32Chunk);
    increment_steps(L, dev, stream);
    if (chunks == 0) {
        BNB200_CHECK_LAUNCH("optimizer32bit");
        return;
    }
    const int grid = grid_for(chunks, 1);
    const bool trust = max_unorm > 0.0f && OPT != kAdemamix;
    const T* g = static_cast<const T*>(ts[0].g);
    const float* s1 = static_cast<const float*>(ts[0].state1);
    const float* s2 = static_cast<const float*>(ts[0].state2);
    // Lion: the parameter update comes first, the norm of the NEW state feeds the next step (reference ops.cu:124-137)
    if (trust && OPT != kLion) {
        cudaMemsetAsync(unorm, 0, sizeof(float), stream);
        optim32_unorm_kernel<T, OPT><<<grid, 512, 0, stream>>>(g, s1, s2, unorm, s.beta1, s.beta2, s.eps, ts[0].step,
                                                               s.gnorm_scale, ts[0].n);
    }
    if (dev)
        optim32_kernel<T, OPT, true><<<grid, 512, 0, stream>>>(L, s, unorm, max_unorm, param_norm, lr_dev);
    else
        optim32_kernel<T, OPT, false><<<grid, 512, 0, stream>>>(L, s, unorm, max_unorm, param_norm, nullptr);
    if (trust && OPT == kLion) {
        cudaMemsetAsync(unorm, 0, sizeof(float), stream);
        optim32_unorm_kernel<T, OPT><<<grid, 512, 0, stream>>>(g, s1, s2, unorm, s.beta1, s.beta2, s.eps, ts[0].step,
                                                               s.gnorm_scale, ts[0].n);
    }
    BNB200_CHECK_LAUNCH("optimizer32bit");
}

// dev: as run32 (the capturable instances take any count: they are not specialised for a list of one)
template <typename T, int OPT>
void run8(const OptimTensor* ts, int count, const OptimScalars& s, const float* qmap1, const float* qmap2, bool dev,
          const float* lr_dev, cudaStream_t stream) {
    OptimList L;
    const long long n_blocks = make_list(L, ts, count, kOptBlock);
    increment_steps(L, dev, stream);
    if (n_blocks == 0) {
        BNB200_CHECK_LAUNCH("optimizer8bit_blockwise");
        return;
    }
    const int grid = grid_for(n_blocks, 8);
    if constexpr (OPT == kAdam || OPT == kAdemamix) {
        if (dev)
            optim8_2state_kernel<T, OPT, false, true><<<grid, 256, 0, stream>>>(L, s, qmap1, qmap2, lr_dev);
        else if (count == 1)
            optim8_2state_kernel<T, OPT, true, false><<<grid, 256, 0, stream>>>(L, s, qmap1, qmap2, nullptr);
        else
            optim8_2state_kernel<T, OPT, false, false><<<grid, 256, 0, stream>>>(L, s, qmap1, qmap2, nullptr);
    } else {
        if (dev)
            optim8_1state_kernel<T, OPT, false, true><<<grid, 256, 0, stream>>>(L, s, qmap1, lr_dev);
        else if (count == 1)
            optim8_1state_kernel<T, OPT, true, false><<<grid, 256, 0, stream>>>(L, s, qmap1, nullptr);
        else
            optim8_1state_kernel<T, OPT, false, false><<<grid, 256, 0, stream>>>(L, s, qmap1, nullptr);
    }
    BNB200_CHECK_LAUNCH("optimizer8bit_blockwise");
}

template <typename T>
bool dispatch32(int opt, const OptimTensor* ts, int count, const OptimScalars& s, float* unorm, float max_unorm,
                float param_norm, bool dev, const float* lr_dev, cudaStream_t st) {
#define BNB200_O32(ID)                                                                                                 \
    case ID:                                                                                                           \
        run32<T, ID>(ts, count, s, unorm, max_unorm, param_norm, dev, lr_dev, st);                                     \
        return true;
    switch (opt) {
        BNB200_O32(kAdam)
        BNB200_O32(kMomentum)
        BNB200_O32(kRmsprop)
        BNB200_O32(kAdagrad)
        BNB200_O32(kLion)
        BNB200_O32(kAdemamix)
    }
#undef BNB200_O32
    return false;
}

template <typename T>
bool dispatch8(int opt, const OptimTensor* ts, int count, const OptimScalars& s, const float* q1, const float* q2,
               bool dev, const float* lr_dev, cudaStream_t st) {
#define BNB200_O8(ID)                                                                                                  \
    case ID:                                                                                                           \
        run8<T, ID>(ts, count, s, q1, q2, dev, lr_dev, st);                                                            \
        return true;
    switch (opt) {
        BNB200_O8(kAdam)
        BNB200_O8(kMomentum)
        BNB200_O8(kRmsprop)
        BNB200_O8(kAdagrad)
        BNB200_O8(kLion)
        BNB200_O8(kAdemamix)
    }
#undef BNB200_O8
    return false;
}

bool list32(int opt, int dtype, const OptimTensor* ts, int count, const OptimScalars& s, float* unorm, float max_unorm,
            float param_norm, bool dev, const float* lr_dev, cudaStream_t st) {
    switch (dtype) {
    case 0: return dispatch32<float>(opt, ts, count, s, unorm, max_unorm, param_norm, dev, lr_dev, st);
    case 1: return dispatch32<__half>(opt, ts, count, s, unorm, max_unorm, param_norm, dev, lr_dev, st);
    case 2: return dispatch32<__nv_bfloat16>(opt, ts, count, s, unorm, max_unorm, param_norm, dev, lr_dev, st);
    }
    return false;
}

bool list8(int opt, int dtype, const OptimTensor* ts, int count, const OptimScalars& s, const float* q1, const float* q2,
           bool dev, const float* lr_dev, cudaStream_t st) {
    switch (dtype) {
    case 0: return dispatch8<float>(opt, ts, count, s, q1, q2, dev, lr_dev, st);
    case 1: return dispatch8<__half>(opt, ts, count, s, q1, q2, dev, lr_dev, st);
    case 2: return dispatch8<__nv_bfloat16>(opt, ts, count, s, q1, q2, dev, lr_dev, st);
    }
    return false;
}

// One peer launch (count <= kPeerListCap): 32-bit (eight = false) or 8-bit state, NP >= w sources.  AdEMAMix has no
// peer instances (its third state sits at state1 + n, relative to the whole tensor).  DEV = true (the _peers_dev
// entries): the descriptors carry step pointers and lr_dev (if not NULL) replaces s.lr, as in the _dev entries, but
// the launch does not advance the counters: a parameter's step advances on every rank, also where this rank holds no
// piece of it, so the caller advances them (optim/sharded.py, once per step for all parameters).
template <typename T, int OPT, int NP, bool DEV>
void run_peers_np(bool eight, const PeerOptimList& L, long long items, const OptimScalars& s, const float* q1,
                  const float* q2, const float* lr_dev, cudaStream_t stream) {
    if (!eight)
        optim32_kernel<T, OPT, DEV, NP><<<grid_for(items, 1), 512, 0, stream>>>(L, s, nullptr, 0.0f, 0.0f, lr_dev);
    else if constexpr (OPT == kAdam)
        optim8_2state_kernel<T, OPT, false, DEV, NP><<<grid_for(items, 8), 256, 0, stream>>>(L, s, q1, q2, lr_dev);
    else
        optim8_1state_kernel<T, OPT, false, DEV, NP><<<grid_for(items, 8), 256, 0, stream>>>(L, s, q1, lr_dev);
}

template <typename T, int OPT, bool DEV>
void run_peers_w(bool eight, const PeerOptimList& L, long long items, const OptimScalars& s, const float* q1,
                 const float* q2, const float* lr_dev, cudaStream_t stream) {
    if (L.peers.w <= 1)
        run_peers_np<T, OPT, 1, DEV>(eight, L, items, s, q1, q2, lr_dev, stream);
    else if (L.peers.w <= 2)
        run_peers_np<T, OPT, 2, DEV>(eight, L, items, s, q1, q2, lr_dev, stream);
    else if (L.peers.w <= 4)
        run_peers_np<T, OPT, 4, DEV>(eight, L, items, s, q1, q2, lr_dev, stream);
    else
        run_peers_np<T, OPT, kMaxPeers, DEV>(eight, L, items, s, q1, q2, lr_dev, stream);
}

template <typename T, int OPT>
bool run_peers(bool eight, const OptimTensor* ts, int count, const OptimScalars& s, const float* q1, const float* q2,
               const PeerArgs& P, bool dev, const float* lr_dev, cudaStream_t stream) {
    if constexpr (OPT == kAdemamix) {
        return false;
    } else {
        PeerOptimList L;
        L.peers = P;
        const long long items = make_list(L, ts, count, eight ? kOptBlock : kOpt32Chunk);
        if (items > 0) {
            if (dev)
                run_peers_w<T, OPT, true>(eight, L, items, s, q1, q2, lr_dev, stream);
            else
                run_peers_w<T, OPT, false>(eight, L, items, s, q1, q2, nullptr, stream);
        }
        BNB200_CHECK_LAUNCH(eight ? "optimizer8bit_blockwise_peers" : "optimizer32bit_peers");
        return true;
    }
}

template <typename T>
bool dispatch_peers(int opt, bool eight, const OptimTensor* ts, int count, const OptimScalars& s, const float* q1,
                    const float* q2, const PeerArgs& P, bool dev, const float* lr_dev, cudaStream_t st) {
    switch (opt) {
    case kAdam: return run_peers<T, kAdam>(eight, ts, count, s, q1, q2, P, dev, lr_dev, st);
    case kMomentum: return run_peers<T, kMomentum>(eight, ts, count, s, q1, q2, P, dev, lr_dev, st);
    case kRmsprop: return run_peers<T, kRmsprop>(eight, ts, count, s, q1, q2, P, dev, lr_dev, st);
    case kAdagrad: return run_peers<T, kAdagrad>(eight, ts, count, s, q1, q2, P, dev, lr_dev, st);
    case kLion: return run_peers<T, kLion>(eight, ts, count, s, q1, q2, P, dev, lr_dev, st);
    }
    return false;
}

bool list_peers(int opt, int dtype, bool eight, const OptimTensor* ts, int count, const OptimScalars& s,
                const float* q1, const float* q2, const PeerArgs& P, bool dev, const float* lr_dev, cudaStream_t st) {
    switch (dtype) {
    case 0: return dispatch_peers<float>(opt, eight, ts, count, s, q1, q2, P, dev, lr_dev, st);
    case 1: return dispatch_peers<__half>(opt, eight, ts, count, s, q1, q2, P, dev, lr_dev, st);
    case 2: return dispatch_peers<__nv_bfloat16>(opt, eight, ts, count, s, q1, q2, P, dev, lr_dev, st);
    }
    return false;
}

PeerArgs peer_args(const void* const* grad_srcs, int world, void* const* param_dsts, int ndst, const void* grad_local,
                   const void* param_local, float grad_scale, const float* gnorm_scale_dev) {
    PeerArgs P{};
    for (int r = 0; r < world; ++r) P.g[r] = grad_srcs[r];
    for (int r = 0; r < ndst; ++r) P.p[r] = param_dsts[r];
    P.g_local = static_cast<const char*>(grad_local);
    P.p_local = static_cast<const char*>(param_local);
    P.gnorm_scale_dev = gnorm_scale_dev;
    P.grad_scale = grad_scale;
    P.w = world;
    P.ndst = ndst;
    return P;
}

template <typename T, bool INF>
void run_norm(const PeerOptimList& L, int grid, double* partials, cudaStream_t st) {
    if (L.peers.w <= 1)
        peer_norm_kernel<T, 1, INF><<<grid, kNormThreads, 0, st>>>(L, partials);
    else if (L.peers.w <= 2)
        peer_norm_kernel<T, 2, INF><<<grid, kNormThreads, 0, st>>>(L, partials);
    else if (L.peers.w <= 4)
        peer_norm_kernel<T, 4, INF><<<grid, kNormThreads, 0, st>>>(L, partials);
    else
        peer_norm_kernel<T, kMaxPeers, INF><<<grid, kNormThreads, 0, st>>>(L, partials);
}

template <typename T>
void run_norm(bool inf, const PeerOptimList& L, int grid, double* partials, cudaStream_t st) {
    if (inf)
        run_norm<T, true>(L, grid, partials, st);
    else
        run_norm<T, false>(L, grid, partials, st);
}

OptimTensor one_tensor(void* p, const void* g, void* s1, void* s2, float* a1, float* a2, long n, int step) {
    return OptimTensor{p, g, s1, s2, a1, a2, (long long)n, step, 0};
}

} // namespace

int optimizer_list_capacity() { return kOptimListCap; }

// dtype: 0 = fp32, 1 = fp16, 2 = bf16 (the library's convention)
bool launch_optimizer32bit(int opt, int dtype, const void* g, void* p, float* s1, float* s2, float* unorm,
                           float max_unorm, float param_norm, float beta1, float beta2, float beta3, float alpha,
                           float eps, float wd, int step, float lr, float gnorm_scale, bool skip_zeros, long n,
                           cudaStream_t st) {
    const OptimTensor t = one_tensor(p, g, s1, s2, nullptr, nullptr, n, step);
    const OptimScalars s{beta1, beta2, beta3, alpha, eps, wd, lr, gnorm_scale, skip_zeros};
    return list32(opt, dtype, &t, 1, s, unorm, max_unorm, param_norm, false, nullptr, st);
}

bool launch_optimizer8bit_blockwise(int opt, int dtype, void* p, const void* g, unsigned char* s1, unsigned char* s2,
                                    float beta1, float beta2, float beta3, float alpha, float eps, int step, float lr,
                                    const float* q1, const float* q2, float* a1, float* a2, float wd,
                                    float gnorm_scale, bool skip_zeros, long n, cudaStream_t st) {
    const OptimTensor t = one_tensor(p, g, s1, s2, a1, a2, n, step);
    const OptimScalars s{beta1, beta2, beta3, alpha, eps, wd, lr, gnorm_scale, skip_zeros};
    return list8(opt, dtype, &t, 1, s, q1, q2, false, nullptr, st);
}

// count <= optimizer_list_capacity(): one launch
bool launch_optimizer32bit_list(int opt, int dtype, const OptimTensor* ts, int count, float beta1, float beta2,
                                float beta3, float alpha, float eps, float wd, float lr, float gnorm_scale,
                                bool skip_zeros, cudaStream_t st) {
    const OptimScalars s{beta1, beta2, beta3, alpha, eps, wd, lr, gnorm_scale, skip_zeros};
    return list32(opt, dtype, ts, count, s, nullptr, 0.0f, 0.0f, false, nullptr, st);
}

// the capturable list: step pointers in the descriptors, lr_dev (NULL: lr) read by the kernel
bool launch_optimizer32bit_list_dev(int opt, int dtype, const OptimTensor* ts, int count, float beta1, float beta2,
                                    float beta3, float alpha, float eps, float wd, float lr, const float* lr_dev,
                                    float gnorm_scale, bool skip_zeros, cudaStream_t st) {
    const OptimScalars s{beta1, beta2, beta3, alpha, eps, wd, lr, gnorm_scale, skip_zeros};
    return list32(opt, dtype, ts, count, s, nullptr, 0.0f, 0.0f, true, lr_dev, st);
}

bool launch_optimizer8bit_blockwise_list(int opt, int dtype, const OptimTensor* ts, int count, float beta1, float beta2,
                                         float beta3, float alpha, float eps, float wd, float lr, const float* q1,
                                         const float* q2, float gnorm_scale, bool skip_zeros, cudaStream_t st) {
    const OptimScalars s{beta1, beta2, beta3, alpha, eps, wd, lr, gnorm_scale, skip_zeros};
    return list8(opt, dtype, ts, count, s, q1, q2, false, nullptr, st);
}

bool launch_optimizer8bit_blockwise_list_dev(int opt, int dtype, const OptimTensor* ts, int count, float beta1,
                                             float beta2, float beta3, float alpha, float eps, float wd, float lr,
                                             const float* lr_dev, const float* q1, const float* q2, float gnorm_scale,
                                             bool skip_zeros, cudaStream_t st) {
    const OptimScalars s{beta1, beta2, beta3, alpha, eps, wd, lr, gnorm_scale, skip_zeros};
    return list8(opt, dtype, ts, count, s, q1, q2, true, lr_dev, st);
}

int optimizer_peers_capacity() { return kPeerListCap; }
int optimizer_max_peers() { return kMaxPeers; }

// count <= optimizer_peers_capacity(), 1 <= world, ndst <= kMaxPeers: one launch; false for an unknown id or AdEMAMix.
// dev: the descriptors carry step pointers, read and not advanced, and lr_dev (if not NULL) replaces lr.
bool launch_optimizer32bit_list_peers(int opt, int dtype, const OptimTensor* ts, int count,
                                      const void* const* grad_srcs, int world, void* const* param_dsts, int ndst,
                                      const void* grad_local, const void* param_local, float grad_scale, float beta1,
                                      float beta2, float beta3, float alpha, float eps, float wd, float lr,
                                      bool skip_zeros, const float* gnorm_scale_dev, bool dev, const float* lr_dev,
                                      cudaStream_t st) {
    const OptimScalars s{beta1, beta2, beta3, alpha, eps, wd, lr, 1.0f, skip_zeros};
    const PeerArgs P =
        peer_args(grad_srcs, world, param_dsts, ndst, grad_local, param_local, grad_scale, gnorm_scale_dev);
    return list_peers(opt, dtype, false, ts, count, s, nullptr, nullptr, P, dev, lr_dev, st);
}

bool launch_optimizer8bit_blockwise_list_peers(int opt, int dtype, const OptimTensor* ts, int count,
                                               const void* const* grad_srcs, int world, void* const* param_dsts,
                                               int ndst, const void* grad_local, const void* param_local,
                                               float grad_scale, float beta1, float beta2, float beta3, float alpha,
                                               float eps, float wd, float lr, const float* q1, const float* q2,
                                               bool skip_zeros, const float* gnorm_scale_dev, bool dev,
                                               const float* lr_dev, cudaStream_t st) {
    const OptimScalars s{beta1, beta2, beta3, alpha, eps, wd, lr, 1.0f, skip_zeros};
    const PeerArgs P =
        peer_args(grad_srcs, world, param_dsts, ndst, grad_local, param_local, grad_scale, gnorm_scale_dev);
    return list_peers(opt, dtype, true, ts, count, s, q1, q2, P, dev, lr_dev, st);
}

// count <= optimizer_peers_capacity(), 1 <= world <= kMaxPeers, dtype 0..2: adds the launch's norm value into *acc.
// false, with the error message set, when the partials' scratch cannot be allocated.
bool launch_optimizer_grad_norm_peers(int dtype, const OptimTensor* ts, int count, const void* const* grad_srcs,
                                      int world, const void* grad_local, float grad_scale, bool inf, double* acc,
                                      cudaStream_t st) {
    PeerOptimList L;
    L.peers = peer_args(grad_srcs, world, nullptr, 0, grad_local, grad_local, grad_scale, nullptr);
    const long long items = make_list(L, ts, count, kNormChunk);
    if (items == 0) return true;
    const int grid = grid_for(items, 1);
    // stream-ordered scratch: no host synchronisation, and launches on other streams never share it
    double* partials = nullptr;
    if (cudaMallocAsync(reinterpret_cast<void**>(&partials), grid * sizeof(double), st) != cudaSuccess) {
        (void)cudaGetLastError();
        set_last_error_msg("optimizer_grad_norm_peers: could not allocate the partials' scratch");
        return false;
    }
    switch (dtype) {
    case 0: run_norm<float>(inf, L, grid, partials, st); break;
    case 1: run_norm<__half>(inf, L, grid, partials, st); break;
    default: run_norm<__nv_bfloat16>(inf, L, grid, partials, st); break;
    }
    if (inf)
        peer_norm_add_kernel<true><<<1, 32, 0, st>>>(partials, grid, acc);
    else
        peer_norm_add_kernel<false><<<1, 32, 0, st>>>(partials, grid, acc);
    cudaFreeAsync(partials, st);
    BNB200_CHECK_LAUNCH("optimizer_grad_norm_peers");
    return true;
}

void launch_optimizer_clip_coef(const double* values, int world, bool inf, float max_norm, float* out,
                                cudaStream_t st) {
    if (inf)
        clip_coef_kernel<true><<<1, 32, 0, st>>>(values, world, max_norm, out);
    else
        clip_coef_kernel<false><<<1, 32, 0, st>>>(values, world, max_norm, out);
    BNB200_CHECK_LAUNCH("optimizer_clip_coef");
}

} // namespace bnb200
