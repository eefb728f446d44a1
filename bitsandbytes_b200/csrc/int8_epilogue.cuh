// int8_epilogue.cuh -- the per-element LLM.int8() epilogue, shared by the int8 GEMM (int8_gemm.cu) and the reduction of
// K-sharded int32 partials (partials.cu), so that a row-parallel layer rounds exactly as the unsharded GEMM does.
#pragma once

#include "common.cuh"

namespace bnb200 {

// 8 consecutive T -> fp32 (EPI 1: fp16, otherwise bf16)
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

// One output element of the fused epilogue, before its final rounding to T (EPI 1: fp16, 2: bf16).
// acc: the exact int32 dot product; sca / scb: the row statistics of the token and of the weight row; b: the bias
// element as fp32 (0 when there is none, has_bias false); ol: the outlier term sum_j subA[m, j] * subBT[n, j] (fp32
// fma in column order), added only when add_ol.
template <int EPI>
__device__ __forceinline__ float int8_epilogue_value(int acc, float sca, float scb, float b, bool has_bias, bool add_ol,
                                                     float ol) {
    float f;
    if (EPI == 1) {
        f = dequant_value(acc, sca, scb, b);
        // reference: the int8 result is an fp16 tensor, then addmm adds the fp32-accumulated outlier product and
        // rounds once more
        if (add_ol) f = __half2float(__float2half_rn(f)) + ol;
    } else {
        // bf16 output, bit-identical to the reference chain (backends/cuda/ops.py:186-210): the kernel result is
        // fp16, a non-fp16 bias is added by `out.add_(bias)` on the fp16 tensor (fp32 add, one rounding to fp16),
        // then `.to(bfloat16)`.
        f = __half2float(__float2half_rn(dequant_value(acc, sca, scb, 0.f)));
        if (has_bias) f = __half2float(__float2half_rn(f + b));
        if (add_ol) f = __bfloat162float(__float2bfloat16_rn(f)) + ol;
    }
    return f;
}

} // namespace bnb200
