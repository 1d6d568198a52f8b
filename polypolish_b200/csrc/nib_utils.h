// nib_utils.h — bit-level helpers for 4-bit packed sequences, shared by the kernels and a CPU unit test
// (tests/test_nib_utils.py compiles this header with g++): pure functions, no device state.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define PP_HD __host__ __device__ __forceinline__
#else
#define PP_HD inline
#endif

PP_HD unsigned long long pp_brev64(unsigned long long x) {
#if defined(__CUDA_ARCH__)
    return __brevll(x);
#else
    x = ((x >> 1) & 0x5555555555555555ull) | ((x & 0x5555555555555555ull) << 1);
    x = ((x >> 2) & 0x3333333333333333ull) | ((x & 0x3333333333333333ull) << 2);
    x = ((x >> 4) & 0x0F0F0F0F0F0F0F0Full) | ((x & 0x0F0F0F0F0F0F0F0Full) << 4);
    x = ((x >> 8) & 0x00FF00FF00FF00FFull) | ((x & 0x00FF00FF00FF00FFull) << 8);
    x = ((x >> 16) & 0x0000FFFF0000FFFFull) | ((x & 0x0000FFFF0000FFFFull) << 16);
    return (x >> 32) | (x << 32);
#endif
}

// bit 4j set iff nibble j of x is non-zero
PP_HD unsigned long long nibble_nonzero(unsigned long long x) {
    return (x | (x >> 1) | (x >> 2) | (x >> 3)) & 0x1111111111111111ull;
}

// 32 consecutive nibbles starting at nibble index `start` of a packed stream (16 per 64-bit word, low nibble first).
// Reads words start/16 .. start/16 + 2 (the third only when start is not word aligned).
PP_HD void load_nib32(const unsigned long long* w, uint32_t start, unsigned long long& lo, unsigned long long& hi) {
    const unsigned long long* p = w + (start >> 4);
    const uint32_t sh = (start & 15) * 4;
    const unsigned long long w0 = p[0], w1 = p[1];
    if (sh) { const unsigned long long w2 = p[2]; lo = (w0 >> sh) | (w1 << (64 - sh)); hi = (w1 >> sh) | (w2 << (64 - sh)); }
    else { lo = w0; hi = w1; }
}

// Codes of the effective read bases [ri, ri + 32) of a read of `len` bases stored at `w` (BAM nibbles); with rc the
// effective read is the reverse complement of the stored one (effective i <-> stored len-1-i, and complementing a
// BAM nibble = reversing its 4 bits, so the view is one 128-bit bit reversal).  Bases at effective indices >= len
// come out as garbage: the caller masks them.
PP_HD void load_read32(const unsigned long long* w, uint32_t len, bool rc, uint32_t ri, unsigned long long& r0, unsigned long long& r1) {
    if (!rc) { load_nib32(w, ri, r0, r1); return; }
    const int s0 = (int)len - (int)ri - 32;                  // first stored index of the window
    unsigned long long lo, hi;
    if (s0 >= 0) load_nib32(w, (uint32_t)s0, lo, hi);
    else {
        load_nib32(w, 0, lo, hi);
        const uint32_t sh = (uint32_t)(-s0) * 4;             // shift the 128-bit value left by -s0 nibbles (1..31)
        if (sh >= 64) { hi = lo << (sh - 64); lo = 0; }
        else { hi = (hi << sh) | (lo >> (64 - sh)); lo <<= sh; }
    }
    r0 = pp_brev64(hi);
    r1 = pp_brev64(lo);
}

// 2-bit A/C/G/T codes (A, C, G, T = 0, 1, 2, 3; base j at bits 2j) from 16 BAM nibbles (A, C, G, T = 1, 2, 4, 8), and in `bad`
// 01 at every field whose nibble is not one of those four.  A bad field's code is not meaningful.
PP_HD uint32_t pp_nib16_to_2bit(unsigned long long x, uint32_t& bad) {
    const unsigned long long m = 0x1111111111111111ull;
    const unsigned long long b0 = x & m, b1 = (x >> 1) & m, b2 = (x >> 2) & m, b3 = (x >> 3) & m;
    unsigned long long ok = (b0 + b1 + b2 + b3) ^ m;           // 0 in a nibble iff exactly one of its bits is set
    ok = (ok | (ok >> 1) | (ok >> 2)) & m;                      // bit 4j: nibble j is not one-hot
    unsigned long long c = (b1 | b3) | ((b2 | b3) << 1);        // nibble j = its 2-bit code (C or T: bit 0, G or T: bit 1)
    c = (c | (c >> 2)) & 0x0F0F0F0F0F0F0F0Full;
    c = (c | (c >> 4)) & 0x00FF00FF00FF00FFull;
    c = (c | (c >> 8)) & 0x0000FFFF0000FFFFull;
    ok = (ok | (ok >> 2)) & 0x0F0F0F0F0F0F0F0Full;
    ok = (ok | (ok >> 4)) & 0x00FF00FF00FF00FFull;
    ok = (ok | (ok >> 8)) & 0x0000FFFF0000FFFFull;
    bad = (uint32_t)(ok | (ok >> 16));
    return (uint32_t)(c | (c >> 16));
}

// The BAM nibbles of 16 2-bit codes (the inverse of pp_nib16_to_2bit on A/C/G/T).
PP_HD unsigned long long pp_2bit_to_nib16(uint32_t v) {
    unsigned long long x = v;
    x = (x | (x << 16)) & 0x0000FFFF0000FFFFull;
    x = (x | (x << 8)) & 0x00FF00FF00FF00FFull;
    x = (x | (x << 4)) & 0x0F0F0F0F0F0F0F0Full;
    x = (x | (x << 2)) & 0x3333333333333333ull;
    const unsigned long long m = 0x1111111111111111ull, lo = x & m, hi = (x >> 1) & m, nlo = lo ^ m, nhi = hi ^ m;
    return (nhi & nlo) | ((nhi & lo) << 1) | ((hi & nlo) << 2) | ((hi & lo) << 3);
}

// BAM nibbles of the 2-bit bases [ri, ri + 32) of a read stored at `w` (16 bases per word, base i at bits 2i of word i / 16):
// the two words load_read32 gives for the same read.  Reads words ri/16 .. ri/16 + 2.
PP_HD void read32_2bit(const uint32_t* w, uint32_t ri, unsigned long long& r0, unsigned long long& r1) {
    const uint32_t* q = w + (ri >> 4);
    const uint32_t sh = (ri & 15) * 2, x0 = q[0], x1 = q[1], x2 = q[2];
    const uint32_t a = sh ? (x0 >> sh) | (x1 << (32 - sh)) : x0, b = sh ? (x1 >> sh) | (x2 << (32 - sh)) : x1;
    r0 = pp_2bit_to_nib16(a);
    r1 = pp_2bit_to_nib16(b);
}

// Mask of nibbles (bit 4j) where r and d differ, restricted to the first vc (<= 32) nibbles of the 128-bit pair.
PP_HD void mismatch_masks(unsigned long long r0, unsigned long long r1, unsigned long long d0, unsigned long long d1, uint32_t vc,
                          unsigned long long& m0, unsigned long long& m1) {
    m0 = nibble_nonzero(r0 ^ d0);
    m1 = nibble_nonzero(r1 ^ d1);
    if (vc < 16) { m0 &= (1ull << (4 * vc)) - 1; m1 = 0; }
    else if (vc < 32) m1 &= (1ull << (4 * (vc - 16))) - 1;
}
