// decode4.cuh -- register-resident 4-bit -> 16-bit decode shared by the wgmma GEMM and the
// CUDA-core GEMV, the 4-bit -> TF32 decode of the GEMM's TF32 instance, plus the (optionally
// double-quantised) scale fetch.
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

// ---------------------------------------------------------------- TF32 decode (fp32 activations)
// W = rna_tf32(value(code) * scale): the fp32 product F.dequantize_4bit(..., torch.float32) returns (mul_ftz, the
// same scale), rounded to the nearest TF32 value, ties away from zero.  A TF32 value is the top 19 bits of its fp32
// pattern, so byte 0 of every entry is zero and the table is three byte planes: bytes 3 and 2 (the top 16 bits, as
// in DecodeTable) and byte 1.
struct DecodeTableTf32 {
    uint32_t b1[4];  // b1[j] = byte 1 of entries 4j .. 4j+3
    uint32_t b2[4];  // byte 2
    uint32_t b3[4];  // byte 3
};

__device__ __forceinline__ uint32_t rna_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

template <int QT> __device__ __forceinline__ void build_table_tf32(float scale, DecodeTableTf32& t) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        uint32_t e[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) e[i] = rna_tf32(mul_ftz(code4_value<QT>(4 * j + i), scale));
        const uint32_t ab13 = prmt(e[0], e[1], 0x7351), cd13 = prmt(e[2], e[3], 0x7351);  // (x.1, y.1, x.3, y.3)
        const uint32_t ab2 = prmt(e[0], e[1], 0x6262), cd2 = prmt(e[2], e[3], 0x6262);    // (x.2, y.2, x.2, y.2)
        t.b1[j] = prmt(ab13, cd13, 0x5410);
        t.b2[j] = prmt(ab2, cd2, 0x5410);
        t.b3[j] = prmt(ab13, cd13, 0x7632);
    }
}

// One word of 8 codes (nibble n = code n, any order the caller chooses) -> o[n] = the TF32 bit pattern of code n.
// Per four codes: three PRMT look-ups of three planes, two PRMT that interleave byte 1 with zero bytes, two that pair
// bytes 2 and 3, and one PRMT per value that joins the two halves.
__device__ __forceinline__ void decode_word_tf32(uint32_t w, const DecodeTableTf32& t, uint32_t (&o)[8]) {
    const uint32_t c7 = w & 0x77777777u;
    const uint32_t w1 = shr_fma(w, 0x80000000u);      // w >> 1
    const uint32_t c7h = shr_fma(c7, 0x00010000u);    // c7 >> 16
    const uint32_t w17 = shr_fma(w, 0x00008000u);     // w >> 17
#pragma unroll
    for (int g = 0; g < 2; ++g) {
        const uint32_t c = g ? c7h : c7;
        const uint32_t selm = sel_half(g ? w17 : w1);
        // byte i of each: the plane's byte of code 4g + i
        const uint32_t p1 = prmt(prmt(t.b1[0], t.b1[1], c), prmt(t.b1[2], t.b1[3], c), selm);
        const uint32_t p2 = prmt(prmt(t.b2[0], t.b2[1], c), prmt(t.b2[2], t.b2[3], c), selm);
        const uint32_t p3 = prmt(prmt(t.b3[0], t.b3[1], c), prmt(t.b3[2], t.b3[3], c), selm);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t lo = prmt(p1, 0u, h ? 0x3424 : 0x1404);  // (0, p1[2h], 0, p1[2h+1])
            const uint32_t hi = prmt(p2, p3, h ? 0x7362 : 0x5140);  // (p2[2h], p3[2h], p2[2h+1], p3[2h+1])
            o[4 * g + 2 * h] = prmt(lo, hi, 0x5410);
            o[4 * g + 2 * h + 1] = prmt(lo, hi, 0x7632);
        }
    }
}

} // namespace bnb200
