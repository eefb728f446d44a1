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
// persistent (a multiple of the SM count).  The 32-bit kernels are plain grid-stride loops.
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

namespace bnb200 {

namespace {

enum OptId : int { kAdam = 0, kMomentum = 1, kRmsprop = 2, kAdagrad = 3, kLion = 4, kAdemamix = 5 };

constexpr int kOptBlock = 256;  // elements per 8-bit state block (reference BLOCKSIZE_1STATE / _2STATE)

__device__ __forceinline__ float sgnf(float v) { return (float)((0.0f < v) - (v < 0.0f)); }

template <typename T> __device__ __forceinline__ T round_to(float v) { return DT<T>::from_f32(v); }
template <typename T> __device__ __forceinline__ float widen(T v) { return DT<T>::to_f32(v); }

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

// VEC: four consecutive elements per thread and iteration through 8- / 16-byte accesses (every pointer 16-byte
// aligned; the host checks), the last n % 4 elements by the first threads of CTA 0; otherwise one element per access.
template <typename T, int OPT, bool VEC>
__global__ void __launch_bounds__(512) optim32_kernel(const T* g, T* p, float* s1, float* s2, const float* unorm,
                                                      float max_unorm, float param_norm, float beta1, float beta2,
                                                      float beta3, float alpha, float eps, float weight_decay, int step,
                                                      float lr, float gnorm_scale, bool skip_zeros, long n) {
    constexpr bool two = OPT == kAdam || OPT == kAdemamix;
    Opt32Args q;
    q.beta1 = beta1, q.beta2 = beta2, q.beta3 = beta3, q.alpha = alpha, q.eps = eps, q.weight_decay = weight_decay;
    q.lr = lr, q.gnorm_scale = gnorm_scale, q.step = step, q.skip_zeros = skip_zeros;
    q.correction1 = 1.0f - powf(beta1, step);
    q.correction2 = sqrtf(1.0f - powf(beta2, step));
    q.step_size = -lr * q.correction2 / q.correction1;
    q.update_scale = 1.0f;
    if (max_unorm > 0.0f) {
        const float us = sqrtf(unorm[0]);
        const float cap = two ? max_unorm * param_norm : max_unorm * param_norm + eps;
        q.update_scale = us > cap ? cap / us : 1.0f;
    }
    auto one = [&](long i) {
        T pt = p[i];
        float a = s1[i], b = two ? s2[i] : 0.f, c = OPT == kAdemamix ? s1[n + i] : 0.f;
        opt32_element<T, OPT>(q, g[i], pt, a, b, c);
        p[i] = pt;
        s1[i] = a;
        if (two) s2[i] = b;
        if (OPT == kAdemamix) s1[n + i] = c;
    };
    const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (long)gridDim.x * blockDim.x;
    if (!VEC) {
        for (long i = tid; i < n; i += nthreads) one(i);
        return;
    }
    using V = typename Vec4<T>::type;
    const long n4 = n >> 2;
    for (long v = tid; v < n4; v += nthreads) {
        const long i = v << 2;
        V gv4 = *reinterpret_cast<const V*>(g + i);
        V pv4 = *reinterpret_cast<const V*>(p + i);
        float4 a4 = *reinterpret_cast<const float4*>(s1 + i);
        float4 b4 = two ? *reinterpret_cast<const float4*>(s2 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        // (AdEMAMix: s1 + n + i is 16-byte aligned only when n % 4 == 0: the host sends other sizes down the scalar path)
        float4 c4 = OPT == kAdemamix ? *reinterpret_cast<const float4*>(s1 + n + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        T* gt = reinterpret_cast<T*>(&gv4);
        T* pt = reinterpret_cast<T*>(&pv4);
        float* a = reinterpret_cast<float*>(&a4);
        float* b = reinterpret_cast<float*>(&b4);
        float* c = reinterpret_cast<float*>(&c4);
#pragma unroll
        for (int k = 0; k < 4; ++k) opt32_element<T, OPT>(q, gt[k], pt[k], a[k], b[k], c[k]);
        *reinterpret_cast<V*>(p + i) = pv4;
        *reinterpret_cast<float4*>(s1 + i) = a4;
        if (two) *reinterpret_cast<float4*>(s2 + i) = b4;
        if (OPT == kAdemamix) *reinterpret_cast<float4*>(s1 + n + i) = c4;
    }
    if (tid < (n & 3)) one((n4 << 2) + tid);
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

// reference csrc/kernels.cu:914-1150
template <typename T, int OPT>
__global__ void __launch_bounds__(256) optim8_2state_kernel(T* p, const T* g, unsigned char* state1, unsigned char* state2,
                                                            float beta1, float beta2, float beta3, float alpha, float eps,
                                                            int step, float lr, const float* qmap1, const float* qmap2,
                                                            float* absmax1, float* absmax2, float weight_decay,
                                                            float gnorm_scale, bool skip_zeros, long n) {
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
    const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g)) & 15) == 0 &&
                         ((reinterpret_cast<uintptr_t>(state1) | reinterpret_cast<uintptr_t>(state2)) & 7) == 0;
    (void)skip_zeros;  // (the reference's 2-state kernel ignores it too)
    const float correction1 = 1.0f - __powf(beta1, step);
    const float correction2 = sqrtf(1.0f - __powf(beta2, step));
    const float step_size = __fdividef(-lr * correction2, correction1);
    const int lane = threadIdx.x & 31;
    const long n_blocks = (n + kOptBlock - 1) / kOptBlock;
    const long warps = (long)gridDim.x * (blockDim.x >> 5);
    for (long blk = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); blk < n_blocks; blk += warps) {
        const long base = blk * kOptBlock;
        const float am1 = absmax1[blk], am2 = absmax2[blk];
        const float am3 = OPT == kAdemamix ? absmax1[(n + base) / kOptBlock] : 0.f;
        const long i0 = base + lane * 8;
        const bool vec = aligned && base + kOptBlock <= n;
        alignas(16) T gts[8];
        alignas(16) T pts[8];
        alignas(8) unsigned char c1s[8], c2s[8], c3s[8];
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
        store8<T>(p, i0, n, vec, pts);
        store8c(state1, i0, n, vec, c1s);
        store8c(state2, i0, n, vec, c2s);
        if (OPT == kAdemamix) store8c(state1 + n, i0, n, vec && (n & 7) == 0, c3s);
    }
}

// reference csrc/kernels.cu:1152-1325
template <typename T, int OPT>
__global__ void __launch_bounds__(256) optim8_1state_kernel(T* p, const T* g, unsigned char* state1, float beta1,
                                                            float beta2, float eps, int step, float lr,
                                                            const float* qmap1, float* absmax1, float weight_decay,
                                                            float gnorm_scale, bool skip_zeros, long n) {
    __shared__ float code1[256];
    __shared__ float2 fin1[257];
    __shared__ uint32_t br1[kQ8Cells];
    code1[threadIdx.x] = qmap1[threadIdx.x];
    __syncthreads();
    build_q8_bracket(code1, br1);
    build_q8_final(code1, fin1);
    __syncthreads();
    const CodeBook cb1{code1, fin1, br1};
    const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g)) & 15) == 0 &&
                         (reinterpret_cast<uintptr_t>(state1) & 7) == 0;
    const int lane = threadIdx.x & 31;
    const long n_blocks = (n + kOptBlock - 1) / kOptBlock;
    const long warps = (long)gridDim.x * (blockDim.x >> 5);
    for (long blk = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); blk < n_blocks; blk += warps) {
        const long base = blk * kOptBlock;
        const float am1 = absmax1[blk];
        const long i0 = base + lane * 8;
        const bool vec = aligned && base + kOptBlock <= n;
        alignas(16) T gts[8];
        alignas(16) T pts[8];
        alignas(8) unsigned char c1s[8];
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

template <typename T, int OPT>
void run32(const T* g, T* p, float* s1, float* s2, float* unorm, float max_unorm, float param_norm, float beta1,
           float beta2, float beta3, float alpha, float eps, float weight_decay, int step, float lr, float gnorm_scale,
           bool skip_zeros, long n, cudaStream_t stream) {
    if (n <= 0) return;
    const int grid = grid_for(n, 512 * 4 * 2);
    const bool trust = max_unorm > 0.0f && OPT != kAdemamix;
    // Lion: the parameter update comes first, the norm of the NEW state feeds the next step (reference ops.cu:124-137)
    if (trust && OPT != kLion) {
        cudaMemsetAsync(unorm, 0, sizeof(float), stream);
        optim32_unorm_kernel<T, OPT><<<grid, 512, 0, stream>>>(g, s1, s2, unorm, beta1, beta2, eps, step, gnorm_scale, n);
    }
    auto al = [](const void* q, uintptr_t m) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & m) == 0; };
    // 16-bit parameters only: there the rounding to T hides how the compiler contracts an fma, and the vector kernel is
    // bit-identical to the scalar one (and to the reference); fp32 already moves 128 bytes per warp access
    const bool vec = sizeof(T) == 2 && al(g, sizeof(T) * 4 - 1) && al(p, sizeof(T) * 4 - 1) && al(s1, 15) && al(s2, 15) &&
                     (OPT != kAdemamix || (n & 3) == 0);
    if (vec)
        optim32_kernel<T, OPT, true><<<grid, 512, 0, stream>>>(g, p, s1, s2, unorm, max_unorm, param_norm, beta1, beta2,
                                                               beta3, alpha, eps, weight_decay, step, lr, gnorm_scale,
                                                               skip_zeros, n);
    else
        optim32_kernel<T, OPT, false><<<grid, 512, 0, stream>>>(g, p, s1, s2, unorm, max_unorm, param_norm, beta1, beta2,
                                                                beta3, alpha, eps, weight_decay, step, lr, gnorm_scale,
                                                                skip_zeros, n);
    if (trust && OPT == kLion) {
        cudaMemsetAsync(unorm, 0, sizeof(float), stream);
        optim32_unorm_kernel<T, OPT><<<grid, 512, 0, stream>>>(g, s1, s2, unorm, beta1, beta2, eps, step, gnorm_scale, n);
    }
    BNB200_CHECK_LAUNCH("optimizer32bit");
}

template <typename T, int OPT>
void run8(T* p, const T* g, unsigned char* state1, unsigned char* state2, float beta1, float beta2, float beta3,
          float alpha, float eps, int step, float lr, const float* qmap1, const float* qmap2, float* absmax1,
          float* absmax2, float weight_decay, float gnorm_scale, bool skip_zeros, long n, cudaStream_t stream) {
    if (n <= 0) return;
    const long n_blocks = (n + kOptBlock - 1) / kOptBlock;
    const int grid = grid_for(n_blocks, 8);
    if (OPT == kAdam || OPT == kAdemamix)
        optim8_2state_kernel<T, OPT><<<grid, 256, 0, stream>>>(p, g, state1, state2, beta1, beta2, beta3, alpha, eps, step,
                                                               lr, qmap1, qmap2, absmax1, absmax2, weight_decay,
                                                               gnorm_scale, skip_zeros, n);
    else
        optim8_1state_kernel<T, OPT><<<grid, 256, 0, stream>>>(p, g, state1, beta1, beta2, eps, step, lr, qmap1, absmax1,
                                                               weight_decay, gnorm_scale, skip_zeros, n);
    BNB200_CHECK_LAUNCH("optimizer8bit_blockwise");
}

template <typename T>
bool dispatch32(int opt, const T* g, T* p, float* s1, float* s2, float* unorm, float max_unorm, float param_norm,
                float beta1, float beta2, float beta3, float alpha, float eps, float wd, int step, float lr,
                float gnorm_scale, bool skip_zeros, long n, cudaStream_t st) {
#define BNB200_O32(ID)                                                                                                 \
    case ID:                                                                                                           \
        run32<T, ID>(g, p, s1, s2, unorm, max_unorm, param_norm, beta1, beta2, beta3, alpha, eps, wd, step, lr,        \
                     gnorm_scale, skip_zeros, n, st);                                                                  \
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
bool dispatch8(int opt, T* p, const T* g, unsigned char* s1, unsigned char* s2, float beta1, float beta2, float beta3,
               float alpha, float eps, int step, float lr, const float* q1, const float* q2, float* a1, float* a2,
               float wd, float gnorm_scale, bool skip_zeros, long n, cudaStream_t st) {
#define BNB200_O8(ID)                                                                                                  \
    case ID:                                                                                                           \
        run8<T, ID>(p, g, s1, s2, beta1, beta2, beta3, alpha, eps, step, lr, q1, q2, a1, a2, wd, gnorm_scale,          \
                    skip_zeros, n, st);                                                                                \
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

} // namespace

// dtype: 0 = fp32, 1 = fp16, 2 = bf16 (the library's convention)
bool launch_optimizer32bit(int opt, int dtype, const void* g, void* p, float* s1, float* s2, float* unorm,
                           float max_unorm, float param_norm, float beta1, float beta2, float beta3, float alpha,
                           float eps, float wd, int step, float lr, float gnorm_scale, bool skip_zeros, long n,
                           cudaStream_t st) {
    switch (dtype) {
    case 0:
        return dispatch32<float>(opt, (const float*)g, (float*)p, s1, s2, unorm, max_unorm, param_norm, beta1, beta2,
                                 beta3, alpha, eps, wd, step, lr, gnorm_scale, skip_zeros, n, st);
    case 1:
        return dispatch32<__half>(opt, (const __half*)g, (__half*)p, s1, s2, unorm, max_unorm, param_norm, beta1, beta2,
                                  beta3, alpha, eps, wd, step, lr, gnorm_scale, skip_zeros, n, st);
    case 2:
        return dispatch32<__nv_bfloat16>(opt, (const __nv_bfloat16*)g, (__nv_bfloat16*)p, s1, s2, unorm, max_unorm,
                                         param_norm, beta1, beta2, beta3, alpha, eps, wd, step, lr, gnorm_scale,
                                         skip_zeros, n, st);
    }
    return false;
}

bool launch_optimizer8bit_blockwise(int opt, int dtype, void* p, const void* g, unsigned char* s1, unsigned char* s2,
                                    float beta1, float beta2, float beta3, float alpha, float eps, int step, float lr,
                                    const float* q1, const float* q2, float* a1, float* a2, float wd,
                                    float gnorm_scale, bool skip_zeros, long n, cudaStream_t st) {
    switch (dtype) {
    case 0:
        return dispatch8<float>(opt, (float*)p, (const float*)g, s1, s2, beta1, beta2, beta3, alpha, eps, step, lr, q1,
                                q2, a1, a2, wd, gnorm_scale, skip_zeros, n, st);
    case 1:
        return dispatch8<__half>(opt, (__half*)p, (const __half*)g, s1, s2, beta1, beta2, beta3, alpha, eps, step, lr, q1,
                                 q2, a1, a2, wd, gnorm_scale, skip_zeros, n, st);
    case 2:
        return dispatch8<__nv_bfloat16>(opt, (__nv_bfloat16*)p, (const __nv_bfloat16*)g, s1, s2, beta1, beta2, beta3,
                                        alpha, eps, step, lr, q1, q2, a1, a2, wd, gnorm_scale, skip_zeros, n, st);
    }
    return false;
}

} // namespace bnb200
