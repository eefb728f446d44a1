/* prmt_decode_tf32_equiv.c -- the TF32 register-table decode of the fused GEMM (bitsandbytes_b200/csrc/decode4.cuh:
 * build_table_tf32's three byte planes + decode_word_tf32's PRMT network, and gemm4_tc.cu's gather_nibbles), restated
 * with an exact emulation of the PRMT instruction.
 *   1. decode: for EVERY packed 32-bit word and 16-entry tables of TF32 bit patterns (byte 0 zero, bytes 1..3
 *      arbitrary), o[n] == table[nibble n of the word] for all eight nibbles.
 *   2. gather: for each of the four threads of a quad and 2^26 random 16-byte chunks, nibble n of the gathered word is
 *      the code of k8 step 2(n & 1) + n/4 (word of the chunk), k t + 4((n >> 1) & 1), as the fragment mapping assumes.
 * build & run:  gcc -O2 -fopenmp -o prmt_decode_tf32_equiv prmt_decode_tf32_equiv.c && ./prmt_decode_tf32_equiv */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

/* PTX prmt.b32 (default mode): selector nibble n picks byte (n & 7) of {y:x}; bit 3 replicates that byte's sign */
static uint32_t byte_perm(uint32_t x, uint32_t y, uint32_t s) {
    const uint64_t src = ((uint64_t)y << 32) | x;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) {
        const uint32_t n = (s >> (4 * i)) & 0xf;
        uint32_t b = (uint32_t)(src >> (8 * (n & 7))) & 0xff;
        if (n & 8) b = (b & 0x80) ? 0xff : 0x00;
        r |= b << (8 * i);
    }
    return r;
}

typedef struct { uint32_t b1[4], b2[4], b3[4]; } DecodeTableTf32;

static void build_planes(const uint32_t* e16, DecodeTableTf32* t) {
    for (int j = 0; j < 4; ++j) {
        const uint32_t* e = e16 + 4 * j;
        const uint32_t ab13 = byte_perm(e[0], e[1], 0x7351), cd13 = byte_perm(e[2], e[3], 0x7351);
        const uint32_t ab2 = byte_perm(e[0], e[1], 0x6262), cd2 = byte_perm(e[2], e[3], 0x6262);
        t->b1[j] = byte_perm(ab13, cd13, 0x5410);
        t->b2[j] = byte_perm(ab2, cd2, 0x5410);
        t->b3[j] = byte_perm(ab13, cd13, 0x7632);
    }
}

static uint32_t lookup(const uint32_t* p, uint32_t c, uint32_t selm) {
    return byte_perm(byte_perm(p[0], p[1], c), byte_perm(p[2], p[3], c), selm);
}

static void decode_word_tf32(uint32_t w, const DecodeTableTf32* t, uint32_t* o) {
    const uint32_t c7 = w & 0x77777777u;
    const uint32_t w1 = w >> 1;
    for (int g = 0; g < 2; ++g) {
        const uint32_t c = g ? (c7 >> 16) : c7;
        const uint32_t m = g ? (w1 >> 16) : w1;
        const uint32_t selm = (m & 0x4444u) | 0x3210u;
        const uint32_t p1 = lookup(t->b1, c, selm), p2 = lookup(t->b2, c, selm), p3 = lookup(t->b3, c, selm);
        for (int h = 0; h < 2; ++h) {
            const uint32_t lo = byte_perm(p1, 0u, h ? 0x3424 : 0x1404);
            const uint32_t hi = byte_perm(p2, p3, h ? 0x7362 : 0x5140);
            o[4 * g + 2 * h] = byte_perm(lo, hi, 0x5410);
            o[4 * g + 2 * h + 1] = byte_perm(lo, hi, 0x7632);
        }
    }
}

static uint32_t gather_nibbles(const uint32_t* v, int t) {
    const uint32_t sel = (uint32_t)(t >> 1) * 0x1111u + 0x6420u;
    const uint32_t shr = (t & 1) ? 0u : 4u, mul = (t & 1) ? 16u : 1u;
    const uint32_t r0 = byte_perm(v[0], v[1], sel) >> shr;
    const uint32_t r1 = byte_perm(v[2], v[3], sel) * mul;
    return (r0 & 0x0F0F0F0Fu) | (r1 & ~0x0F0F0F0Fu);
}

/* code k (0..7) of a packed word: element 2b in the high nibble of byte b */
static uint32_t code_of(uint32_t word, int k) { return (word >> (8 * (k >> 1) + ((k & 1) ? 0 : 4))) & 15u; }

static uint64_t rng = 0x9E3779B97F4A7C15ull;
static uint32_t next32(void) {
    rng ^= rng << 13;
    rng ^= rng >> 7;
    rng ^= rng << 17;
    return (uint32_t)(rng >> 16);
}

int main(void) {
    long long bad = 0;
    for (int trial = 0; trial < 2; ++trial) {
        uint32_t entry[16];
        for (int i = 0; i < 16; ++i) entry[i] = next32() & 0xFFFFFF00u;                      /* arbitrary bytes 1..3 */
        if (trial == 1) for (int i = 0; i < 16; ++i) entry[i] = 0xFFFFE000u ^ ((uint32_t)i << 13);  /* negative, ones */
        DecodeTableTf32 t;
        build_planes(entry, &t);
#pragma omp parallel for schedule(static) reduction(+ : bad)
        for (long long bits = 0; bits < (1LL << 32); ++bits) {
            const uint32_t w = (uint32_t)bits;
            uint32_t o[8];
            decode_word_tf32(w, &t, o);
            for (int n = 0; n < 8; ++n) bad += o[n] != entry[(w >> (4 * n)) & 15u];
        }
    }
    printf("TF32 PRMT decode: mismatches over 2 tables x all 2^32 packed words: %lld\n", bad);
    long long bad_g = 0;
    for (long long i = 0; i < (1LL << 26); ++i) {
        uint32_t v[4];
        for (int j = 0; j < 4; ++j) v[j] = next32();
        for (int t = 0; t < 4; ++t) {
            const uint32_t w = gather_nibbles(v, t);
            for (int n = 0; n < 8; ++n) {
                const int step = 2 * (n & 1) + (n >> 2), k = t + 4 * ((n >> 1) & 1);
                bad_g += ((w >> (4 * n)) & 15u) != code_of(v[step], k);
            }
        }
    }
    printf("TF32 gather: mismatches over 4 threads x 2^26 random chunks: %lld\n", bad_g);
    return (bad != 0 || bad_g != 0);
}
