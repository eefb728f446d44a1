// common.cuh -- shared device helpers for the sm_90a kernels.
//
// Numeric contract notes (see DESIGN.md "Numerics"):
//  * The reference CUDA library is compiled with --use_fast_math
//    (reference CMakeLists.txt:190).  That makes `1.0f / absmax` an approximate
//    MUFU reciprocal and every fp32 op flush-to-zero.  To be bit-exact with the
//    reference's quantization codes we spell those instructions out in PTX
//    instead of depending on compiler flags.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <type_traits>

namespace bnb200 {

// csrc/common.h:3-7 of the reference: DataType_t { General8bit = 0, FP4 = 1, NF4 = 2 }
enum QuantType : int { kGeneral8bit = 0, kFP4 = 1, kNF4 = 2 };
// kernel-internal variant of kGeneral8bit: the same codes through the cheaper search (blockwise.cu)
constexpr int kGeneral8bitFast = 3;

constexpr int kNumSMsH100 = 132;  // H100 SXM; the launchers ask the device

// ---------------------------------------------------------------- PTX-exact fp32 ops
__device__ __forceinline__ float mul_ftz(float a, float b) {
    float r;
    asm("mul.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// LLM.int8() dequantisation of one int32 accumulator (shared by the stand-alone kernel in int8.cu
// and the fused GEMM epilogue in int8_gemm.cu).
constexpr float kMmDequantConst = 6.200012e-05f;  // reference kernels.cu:1394 ("1/(127*127)")

__device__ __forceinline__ float dequant_value(int acc, float rs, float cs, float bias) {
    // reference kernels.cu:1436-1438: fmaf(int * rowStats * colStats, C, bias), all ftz
    float t = mul_ftz(mul_ftz((float)acc, rs), cs);
    float r;
    asm("fma.rn.ftz.f32 %0, %1, %2, %3;" : "=f"(r) : "f"(t), "f"(kMmDequantConst), "f"(bias));
    return r;
}

__device__ __forceinline__ float rcp_approx_ftz(float a) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
    return r;
}

__device__ __forceinline__ float div_approx_ftz(float a, float b) {
    float r;
    asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

__device__ __forceinline__ float abs_ftz(float a) {
    float r;
    asm("abs.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
    return r;
}

__device__ __forceinline__ float max_ftz(float a, float b) {
    float r;
    asm("max.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// ---------------------------------------------------------------- code books
// NF4: reference csrc/kernels.cu:26-43 / gemm_4bit_common.cuh:17-34.
// FP4: reference csrc/kernels.cu:15-24,59-62 (magnitude table, bit 3 = sign).
__device__ __forceinline__ float nf4_value(unsigned q) {
    // Constant-index switch keeps this usable in unrolled table builders.
    switch (q & 15u) {
    case 0: return -1.0f;
    case 1: return -0.6961928009986877f;
    case 2: return -0.5250730514526367f;
    case 3: return -0.39491748809814453f;
    case 4: return -0.28444138169288635f;
    case 5: return -0.18477343022823334f;
    case 6: return -0.09105003625154495f;
    case 7: return 0.0f;
    case 8: return 0.07958029955625534f;
    case 9: return 0.16093020141124725f;
    case 10: return 0.24611230194568634f;
    case 11: return 0.33791524171829224f;
    case 12: return 0.44070982933044434f;
    case 13: return 0.5626170039176941f;
    case 14: return 0.7229568362236023f;
    default: return 1.0f;
    }
}

__device__ __forceinline__ float fp4_value(unsigned q) {
    float m;
    switch (q & 7u) {
    case 0: m = 0.0f; break;
    case 1: m = 0.005208333333f; break;
    case 2: m = 0.66666667f; break;
    case 3: m = 1.0f; break;
    case 4: m = 0.33333333f; break;
    case 5: m = 0.5f; break;
    case 6: m = 0.16666667f; break;
    default: m = 0.25f; break;
    }
    // lut * (1 - 2*sign): code 8 is -0.0f exactly as in the reference.
    return (q & 8u) ? -m : m;
}

template <int QT> __device__ __forceinline__ float code4_value(unsigned q) {
    return QT == kNF4 ? nf4_value(q) : fp4_value(q);
}

// ---------------------------------------------------------------- dtype traits
template <typename T> struct DT;

template <> struct DT<float> {
    static constexpr int kBytes = 4;
    __device__ static __forceinline__ float to_f32(float v) { return v; }
    __device__ static __forceinline__ float from_f32(float v) { return v; }
};

template <> struct DT<__half> {
    static constexpr int kBytes = 2;
    __device__ static __forceinline__ float to_f32(__half v) { return __half2float(v); }
    __device__ static __forceinline__ __half from_f32(float v) { return __float2half_rn(v); }
};

template <> struct DT<__nv_bfloat16> {
    static constexpr int kBytes = 2;
    __device__ static __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
    __device__ static __forceinline__ __nv_bfloat16 from_f32(float v) { return __float2bfloat16_rn(v); }
};

// pack two fp32 -> one 32-bit word holding (lo, hi) as T x2 (lo at the lower address)
template <typename T> __device__ __forceinline__ uint32_t pack2(float lo, float hi);

template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

template <> __device__ __forceinline__ uint32_t pack2<__half>(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

// ---------------------------------------------------------------- memory helpers
__device__ __forceinline__ uint4 ldg_stream_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

__device__ __forceinline__ uint2 ldg_stream_v2(const void* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}

__device__ __forceinline__ uint32_t ldg_stream_u32(const void* p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}

__device__ __forceinline__ uint16_t ldg_stream_u16(const void* p) {
    uint16_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(r) : "l"(p));
    return r;
}

__device__ __forceinline__ void stg_stream_v4(void* p, uint4 v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}

__device__ __forceinline__ void stg_stream_v2(void* p, uint2 v) {
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}

__device__ __forceinline__ void stg_stream_u32(void* p, uint32_t v) {
    asm volatile("st.global.L1::no_allocate.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ void stg_stream_u16(void* p, uint16_t v) {
    asm volatile("st.global.L1::no_allocate.u16 [%0], %1;" ::"l"(p), "h"(v) : "memory");
}

__host__ __device__ __forceinline__ int ilog2_pow2(int v) {
    int r = 0;
    while ((1 << r) < v) ++r;
    return r;
}

// ---------------------------------------------------------------- host-side error plumbing
// (c_api.cu owns the storage)
void set_last_error(const char* where, cudaError_t err);
void set_last_error_msg(const char* msg);

#define BNB200_CHECK_LAUNCH(where)                                                                                     \
    do {                                                                                                               \
        cudaError_t _e = cudaPeekAtLastError();                                                                        \
        if (_e != cudaSuccess) {                                                                                       \
            (void)cudaGetLastError();                                                                                  \
            ::bnb200::set_last_error(where, _e);                                                                       \
        }                                                                                                              \
    } while (0)

int device_sm_count();

// Experts a grouped (mixture-of-experts) launch serves: the grouped GEMM's group table (gemm4_tc.cu) and the grouped
// reduction's table of end rows (partials.cu) are sized by it; _ops.MAX_EXPERTS is the same limit on the Python side.
constexpr int kMaxExperts = 1024;

// ---------------------------------------------------------------- 4-bit GEMM destinations
// The destinations of a 4-bit GEMM: every output element is stored to each of p[0..n) at the same row stride (a
// sharded layer's slot in every rank's buffer).  OutList<float> carries the partial instances' fp32 accumulators
// (cbnb_b200_gemm_4bit_partial), with no bias and no rounding.  rows_per_out > 0 (the partial instances only,
// cbnb_b200_gemm_4bit_partial_scatter) scatters the rows instead: row m goes to p[m / rows_per_out] only, at row
// m % rows_per_out, so that each rank of a sequence-parallel layer receives its own tokens.
constexpr int kMaxOuts = 8;
template <typename TO> struct OutList {
    TO* p[kMaxOuts];
    int n;
    int rows_per_out;  // 0: every row to every destination
};

// Where a scattering GEMM (rows_per_out > 0) stores output row m: destination m / rows_per_out, at its row
// m % rows_per_out.  The one statement of that rule for the 4-bit partial stores and the int8 partial scatter.
struct ScatterRow {
    int out;
    int row;
};
__device__ __forceinline__ ScatterRow scatter_row(int m, int rows_per_out) {
    const int d = m / rows_per_out;
    return {d, m - d * rows_per_out};
}

// The partial instances' store of element (m, n) of the fp32 output: to every destination of `outs`, or, with
// rows_per_out > 0, to destination m / rows_per_out at row m % rows_per_out.
__device__ __forceinline__ void store_partial(const OutList<float>& outs, int m, int n, long long ldc, float v) {
    if (outs.rows_per_out > 0) {
        const ScatterRow r = scatter_row(m, outs.rows_per_out);
        outs.p[r.out][r.row * ldc + n] = v;
    } else {
        for (int d = 0; d < outs.n; ++d) outs.p[d][m * ldc + n] = v;
    }
}
// The element a 4-bit GEMM stores: T, or fp32 for the partial instances (PART)
template <typename T, bool PART> using OutElem = typename std::conditional<PART, float, T>::type;
// The output argument of a small-M 4-bit GEMM kernel or launcher: T* (bias added, rounded once to T), or, for the
// partial instances (PART), the fp32 destinations.
template <typename T, bool PART> struct OutArg {
    using type = T* __restrict__;
};
template <typename T> struct OutArg<T, true> {
    using type = OutList<float>;
};

// ---------------------------------------------------------------- optimizer tensor lists (optim.cu, c_api.cu)
// One tensor of a multi-tensor optimizer step: the layout of bnb_b200_optim_tensor_t in include/bitsandbytes_b200.h.
struct OptimTensor {
    void* p;
    const void* g;
    void* state1;
    void* state2;     // NULL for one-state optimizers
    float* absmax1;   // 8-bit state only
    float* absmax2;
    long long n;      // elements of p
    union {
        struct {
            int step;     // this tensor's own step (1 on its first update)
            int reserved;
        };
        int* step_ptr;    // the capturable (_dev) entries: the step counter in device memory (_multi_dev advances it)
    };
};
static_assert(sizeof(OptimTensor) == 64, "bnb_b200_optim_tensor_t is 64 bytes");
static_assert(offsetof(OptimTensor, step) == 56 && offsetof(OptimTensor, step_ptr) == 56, "step union at offset 56");

} // namespace bnb200
