// crc32_core.h -- the checksum arithmetic of the PNG encoder: CRC-32 (ISO 3309 / PNG / zlib, reflected polynomial
// 0xEDB88320) of a buffer from the CRCs of its pieces, and Adler-32 from per-piece partial sums.
//
// A PNG file carries the CRC-32 of every chunk and the Adler-32 of the scanlines.  The encoder produces the IDAT
// payload as independent 32 KB DEFLATE chunks, many warps at once, so no thread ever walks the payload front to back.
// Each warp checksums what it has just written, and the pieces are joined with the rules below.
//
// CRC rule.  Write crc(M) for the standard CRC-32 of M (initial value and final inversion included, as zlib.crc32).
// For a concatenation A || B:
//     crc(A || B) = crc(A) * x^(8 * |B|)  xor  crc(B)        (polynomials over GF(2), modulo the CRC polynomial)
// (zlib's crc32_combine identity: the initial value and the inversion cancel between the two terms, and crc("") = 0.)
// Applied repeatedly, the CRC of P_0 || P_1 || ... || P_k is the xor over i of crc(P_i) * x^(8 * bytes behind P_i),
// which is what lets every piece be handled by a different thread.  A polynomial is held bit-reflected in a uint32,
// as the CRC itself is: bit 31 is the coefficient of x^0, bit 0 that of x^31.
//
// Adler rule.  With s1 = 1 + sum b_i and s2 = sum of the running s1 after every byte (both mod 65521), a buffer of N
// bytes has s2 = N + sum_i (N - i) * b_i.  A piece of n bytes starting at p with A = sum b_j and
// B = sum (n - j) * b_j (j counted inside the piece) contributes (N - p - n) * A + B to s2 and A to s1: no piece needs
// a running value from the piece before it.
//
// The same source compiles for the host (LP_CRC_FN = static inline): tests/test_crc32_core.py checks it against zlib
// on the CPU.
#pragma once
#include <cstddef>
#include <cstdint>

#ifndef LP_CRC_FN
#define LP_CRC_FN static inline
#endif

namespace crc32core {

constexpr uint32_t kPoly = 0xEDB88320u;
constexpr uint32_t kAdlerMod = 65521u;

// crc(M || p[0, n)) from c = crc(M); c = 0 starts a new message.  Bit at a time: no table to keep in memory.
LP_CRC_FN uint32_t update(uint32_t c, const uint8_t* p, size_t n) {
    c = ~c;
    for (size_t i = 0; i < n; i++) {
        c ^= p[i];
        for (int k = 0; k < 8; k++) c = (c >> 1) ^ (kPoly & (0u - (c & 1u)));
    }
    return ~c;
}

// a * b modulo the CRC polynomial
LP_CRC_FN uint32_t mulmod(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 0; i < 32; i++) {
        p ^= b & (0u - (a >> 31));                       // the coefficient of x^i in a
        a <<= 1;
        b = (b >> 1) ^ (kPoly & (0u - (b & 1u)));        // b * x
    }
    return p;
}

// x^(8 * n) modulo the CRC polynomial, by squaring
LP_CRC_FN uint32_t xpow8(uint64_t n) {
    uint32_t p = 0x80000000u, base = 0x00800000u;  // 1, x^8
    for (; n; n >>= 1) {
        if (n & 1u) p = mulmod(p, base);
        base = mulmod(base, base);
    }
    return p;
}

// crc(A || B) from crc(A), crc(B) and |B|
LP_CRC_FN uint32_t combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b) { return mulmod(crc_a, xpow8(len_b)) ^ crc_b; }

// What a piece of n bytes at offset p of an N-byte buffer adds to Adler-32's s2 (mod 65521), from its partial sums
// A = sum b_j mod 65521 and B = sum (n - j) * b_j mod 65521.
LP_CRC_FN uint32_t adler_s2_term(uint64_t N, uint64_t p, uint64_t n, uint32_t A, uint32_t B) {
    return (uint32_t)(((N - p - n) % kAdlerMod * A + B) % kAdlerMod);
}

}  // namespace crc32core
