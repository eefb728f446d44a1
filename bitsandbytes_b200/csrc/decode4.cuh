// decode4.cuh -- register-resident 4-bit -> 16-bit decode shared by the wgmma GEMM and the
// CUDA-core GEMV, plus the (optionally double-quantised) scale fetch.
#pragma once

#include "common.cuh"

namespace bnb200 {

struct ScaleSrc {
    const float* absmax;
    const uint8_t* absmax_8bit;
    const float* absmax_code;
    float offset;
    // DQ: double quant, known at compile time (the kernel then carries only one of the two chains)
    template <bool DQ> __device__ __forceinline__ float load_as(long long idx) const {
        if constexpr (DQ) {
            const float c = __ldg(absmax_code + __ldg(absmax_8bit + idx));
            return __fadd_rn(mul_ftz(c, __ldg(absmax + (idx >> 8))), offset);
        } else {
            return __ldg(absmax + idx);
        }
    }
    __device__ __forceinline__ float load(long long idx) const {
        return absmax_8bit != nullptr ? load_as<true>(idx) : load_as<false>(idx);
    }
};

// NOTE on the nested (double-quant) scale: the reference has two behaviours.  Its fused
// kernels write `code[q] * absmax2 + offset`, which nvcc contracts to one fma
// (gemm_4bit_sm80.cu:292-297); its dequantize + F.linear path -- the one the reference takes for
// M > 4 (backends/cuda/ops.py:617-623, 904-916) and the one F.dequantize_4bit exposes --
// rounds the product and the sum separately.  We follow the second (mul, then add), so the
// fused GEMM sees exactly the weights F.dequantize_4bit returns.

// ---------------------------------------------------------------- register-resident decode
// W_T = rn_T(value(code) * scale) takes only 16 distinct values per quantisation block, so a
// decode thread first builds that 16-entry table (16 fp32 multiplies by immediates, 8 packed
// roundings -- bit-identical to rounding every element) and keeps it in 8 registers as two
// byte planes (low bytes / high bytes of the 16-bit entries).  Codes are then translated with
// PRMT (byte permute) only: no shared-memory look-up table, hence no bank conflicts and no
// competition with the tensor core for shared-memory bandwidth.
struct DecodeTable {
    uint32_t lo[4];  // lo[j] = low bytes of entries 4j .. 4j+3
    uint32_t hi[4];  // hi[j] = high bytes
};

template <typename T, int QT> __device__ __forceinline__ void build_table(float scale, DecodeTable& t) {
    uint32_t pr[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
        pr[j] = pack2<T>(mul_ftz(code4_value<QT>(2 * j), scale), mul_ftz(code4_value<QT>(2 * j + 1), scale));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        t.lo[j] = __byte_perm(pr[2 * j], pr[2 * j + 1], 0x6420);
        t.hi[j] = __byte_perm(pr[2 * j], pr[2 * j + 1], 0x7531);
    }
}

// One packed word = 4 bytes = 8 codes (byte b: element 2b in the high nibble) -> 4 registers of
// T pairs, element 2b in the low half.  Selector nibbles must stay < 8 (bit 3 is PRMT's
// sign-replicate flag): `c` carries code & 7, `selm` picks between the idx<8 / idx>=8 halves.
// The decode is bound by the ALU pipe (PRMT / LOP3 / SHF: one warp instruction per 2 cycles and scheduler), so the
// index preparation is kept off it where possible: the right shifts are mul.hi by a power of two (IMAD.HI, fma
// pipe), and (m & 0x4444) | 0x3210 is ONE lop3 (written as such: from `&` and `|` with two immediates ptxas makes two).
__device__ __forceinline__ uint32_t shr_fma(uint32_t x, uint32_t pow2_32_minus_s) {
    uint32_t r;
    asm("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(x), "r"(pow2_32_minus_s));
    return r;
}
__device__ __forceinline__ uint32_t sel_half(uint32_t m) {
    uint32_t r;
    asm("lop3.b32 %0, %1, 0x4444, %2, 0xEA;" : "=r"(r) : "r"(m), "r"(0x3210u));  // (m & 0x4444) | 0x3210
    return r;
}
// prmt.b32 itself (the __byte_perm intrinsic first masks the selector with 0x7777: one more ALU instruction per
// distinct selector; ours are clean by construction -- every nibble < 8)
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}
__device__ __forceinline__ void decode_word(uint32_t w, const DecodeTable& t, uint32_t* o) {
    const uint32_t c7 = w & 0x77777777u;              // PRMT reads only the low 16 bits of a selector
    const uint32_t w1 = shr_fma(w, 0x80000000u);      // w >> 1
    const uint32_t c7h = shr_fma(c7, 0x00010000u);    // c7 >> 16
    const uint32_t w17 = shr_fma(w, 0x00008000u);     // w >> 17
#pragma unroll
    for (int g = 0; g < 2; ++g) {
        const uint32_t c = g ? c7h : c7;
        const uint32_t selm = sel_half(g ? w17 : w1);
        const uint32_t lo = prmt(prmt(t.lo[0], t.lo[1], c), prmt(t.lo[2], t.lo[3], c), selm);
        const uint32_t hi = prmt(prmt(t.hi[0], t.hi[1], c), prmt(t.hi[2], t.hi[3], c), selm);
        o[2 * g] = prmt(lo, hi, 0x4051);      // (T[hi nibble of byte 0], T[lo nibble of byte 0])
        o[2 * g + 1] = prmt(lo, hi, 0x6273);  // byte 1
    }
}

} // namespace bnb200
