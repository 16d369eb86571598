// Host build of lilliput_b200/csrc/crc32_core.h (the PNG encoder's checksum arithmetic) for the CPU suite
// (tests/test_crc32_core.py): the CRC-32 and Adler-32 of a buffer computed the way png_encode.cu computes them -- from
// the checksums of pieces cut at arbitrary places, each piece handled on its own and the results folded.
#include <cstdint>

#include "../../lilliput_b200/csrc/crc32_core.h"

extern "C" uint32_t crc32sim_update(uint32_t c, const uint8_t* p, long n) { return crc32core::update(c, p, (size_t)n); }

extern "C" uint32_t crc32sim_combine(uint32_t a, uint32_t b, unsigned long long len_b) { return crc32core::combine(a, b, len_b); }

// cuts[0] = 0 < ... < cuts[npieces] = n (empty pieces allowed): the pairwise rule, left to right
extern "C" uint32_t crc32sim_chain(const uint8_t* p, const long* cuts, int npieces) {
    uint32_t c = 0;
    for (int k = 0; k < npieces; k++)
        c = crc32core::combine(c, crc32core::update(0, p + cuts[k], (size_t)(cuts[k + 1] - cuts[k])), (uint64_t)(cuts[k + 1] - cuts[k]));
    return c;
}

// the same pieces, each weighted by the bytes behind it and xor-ed in any order (here: last piece first), as
// fold_checksums does across the threads of a block
extern "C" uint32_t crc32sim_fold(const uint8_t* p, const long* cuts, int npieces) {
    uint32_t x = 0;
    const long n = cuts[npieces];
    for (int k = npieces - 1; k >= 0; k--)
        x ^= crc32core::mulmod(crc32core::update(0, p + cuts[k], (size_t)(cuts[k + 1] - cuts[k])), crc32core::xpow8((uint64_t)(n - cuts[k + 1])));
    return x;
}

// Adler-32 from per-piece partial sums A = sum b_j, B = sum (len - j) b_j
extern "C" uint32_t crc32sim_adler(const uint8_t* p, const long* cuts, int npieces) {
    const uint64_t n = (uint64_t)cuts[npieces];
    uint64_t s1 = 0, s2 = 0;
    for (int k = npieces - 1; k >= 0; k--) {
        const uint64_t at = (uint64_t)cuts[k], len = (uint64_t)(cuts[k + 1] - cuts[k]);
        uint64_t A = 0, B = 0;
        for (uint64_t j = 0; j < len; j++) {
            A += p[at + j];
            B = (B + (len - j) * p[at + j]) % crc32core::kAdlerMod;
        }
        s1 += A % crc32core::kAdlerMod;
        s2 += crc32core::adler_s2_term(n, at, len, (uint32_t)(A % crc32core::kAdlerMod), (uint32_t)B);
    }
    s1 = (1 + s1) % crc32core::kAdlerMod;
    s2 = (n % crc32core::kAdlerMod + s2) % crc32core::kAdlerMod;
    return (uint32_t)((s2 << 16) | s1);
}
