// vp8_enc_core.h -- a VP8 key-frame (WebP lossy) ENCODER: per macroblock one 16x16 luma prediction or sixteen 4x4
// ones (whichever costs less distortion + lambda * estimated bits), chroma mode by prediction error, forward DCT / WHT,
// dead-zone quantisation, in-loop reconstruction; token coding with per-frame coefficient probabilities (a statistics
// walk, updates where they pay: RFC 6386 s.13.4) and per-macroblock skip flags, boolean entropy coder, frame + partition
// headers.  Valid streams that any VP8 decoder (libwebp included) reads.  NOT libwebp's encoder -- no segmentation, no
// trellis, its own mode search -- so files are not byte-comparable with the reference's (ref webp.cpp:721-729 calls
// WebPEncodeBGR / BGRA); at equal `quality` they come out at libwebp's PSNR (+-0.25 dB) and 0.92-1.10 x its size.
// What IS checked (tests): the reference's decoder and vp8_core.h decode the stream to the same pixels, those equal the
// encoder's own reconstruction, PSNR and size track libwebp's at equal quality, the device writes this file's bytes.
//
// Shares the decoder's primitives (vp8_core.h): prediction, inverse transforms, tables.
#pragma once
#include "vp8_core.h"

namespace vp8enc {

using vp8::BPS;

// ---- boolean entropy encoder (RFC 6386 s.7.3) ----------------------------------------------
struct BoolEnc {
    uint8_t* out;
    size_t pos, cap;
    uint32_t range, bottom;
    int bit_count;
    int overflow;
};
LP_VP8_INL void be_init(BoolEnc& e, uint8_t* out, size_t cap) {
    e.out = out;
    e.pos = 0;
    e.cap = cap;
    e.range = 255;
    e.bottom = 0;
    e.bit_count = 24;
    e.overflow = 0;
}
LP_VP8_INL void be_carry(BoolEnc& e) {
    size_t q = e.pos;
    while (q > 0 && e.out[q - 1] == 255) e.out[--q] = 0;
    if (q > 0) e.out[q - 1]++;
}
LP_VP8_INL void be_put(BoolEnc& e, int bit, int prob) {
    const uint32_t split = 1 + (((e.range - 1) * (uint32_t)prob) >> 8);
    if (bit) {
        e.bottom += split;
        e.range -= split;
    } else {
        e.range = split;
    }
    if (e.range < 128) {
        // renormalise: `s` doublings.  All of them at once unless one of them would emit a byte or meet the carry
        // flag on its way out of bit 31 (then the bit-by-bit form of RFC 6386 s.7.3 below, same result).
#ifdef __CUDA_ARCH__
        int s = __clz((int)e.range) - 24;
#else
        int s = __builtin_clz(e.range) - 24;
#endif
        e.range <<= s;
        if (e.bit_count > s && (e.bottom >> (32 - s)) == 0) {
            e.bottom <<= s;
            e.bit_count -= s;
            return;
        }
        while (s-- > 0) {
            if (e.bottom & 0x80000000u) be_carry(e);
            e.bottom <<= 1;
            if (!--e.bit_count) {
                if (e.pos < e.cap) e.out[e.pos++] = (uint8_t)(e.bottom >> 24);
                else e.overflow = 1;
                e.bottom &= 0xffffffu;
                e.bit_count = 8;
            }
        }
    }
}
LP_VP8_INL void be_put_bits(BoolEnc& e, uint32_t v, int n) {
    while (n-- > 0) be_put(e, (v >> n) & 1, 128);
}
LP_VP8_INL void be_put_signed(BoolEnc& e, int v, int n) {  // magnitude then sign, the decoder's bd_signed
    be_put_bits(e, (uint32_t)(v < 0 ? -v : v), n);
    be_put(e, v < 0, 128);
}
LP_VP8_FN void be_flush(BoolEnc& e) {
    int c = e.bit_count;
    uint32_t v = e.bottom;
    if (v & (1u << (32 - c))) be_carry(e);
    v <<= c & 7;
    c >>= 3;
    while (--c >= 0) v <<= 8;
    for (int i = 0; i < 4; i++) {
        if (e.pos < e.cap) e.out[e.pos++] = (uint8_t)(v >> 24);
        else e.overflow = 1;
        v <<= 8;
    }
}

// ---- forward transforms (the inverses are vp8::inverse_dct_add / inverse_wht) ----------------
LP_VP8_FN void fdct4x4(const uint8_t* src, int src_stride, const uint8_t* ref, int ref_stride, int16_t* out) {
    int tmp[16];
    for (int i = 0; i < 4; i++) {
        const int d0 = src[i * src_stride + 0] - ref[i * ref_stride + 0];
        const int d1 = src[i * src_stride + 1] - ref[i * ref_stride + 1];
        const int d2 = src[i * src_stride + 2] - ref[i * ref_stride + 2];
        const int d3 = src[i * src_stride + 3] - ref[i * ref_stride + 3];
        const int a0 = d0 + d3, a1 = d1 + d2, a2 = d1 - d2, a3 = d0 - d3;
        tmp[0 + i * 4] = (a0 + a1) * 8;
        tmp[1 + i * 4] = (a2 * 2217 + a3 * 5352 + 1812) >> 9;
        tmp[2 + i * 4] = (a0 - a1) * 8;
        tmp[3 + i * 4] = (a3 * 2217 - a2 * 5352 + 937) >> 9;
    }
    for (int i = 0; i < 4; i++) {
        const int a0 = tmp[0 + i] + tmp[12 + i], a1 = tmp[4 + i] + tmp[8 + i];
        const int a2 = tmp[4 + i] - tmp[8 + i], a3 = tmp[0 + i] - tmp[12 + i];
        out[0 + i] = (int16_t)((a0 + a1 + 7) >> 4);
        out[4 + i] = (int16_t)(((a2 * 2217 + a3 * 5352 + 12000) >> 16) + (a3 != 0));
        out[8 + i] = (int16_t)((a0 - a1 + 7) >> 4);
        out[12 + i] = (int16_t)((a3 * 2217 - a2 * 5352 + 51000) >> 16);
    }
}
// in: the 16 DC terms (element 0 of 16 coefficient blocks, stride 16); out: 16 Y2 coefficients
LP_VP8_FN void fwht(const int16_t* in, int16_t* out) {
    int tmp[16];
    for (int i = 0; i < 4; i++, in += 64) {
        const int a0 = in[0 * 16] + in[2 * 16], a1 = in[1 * 16] + in[3 * 16];
        const int a2 = in[1 * 16] - in[3 * 16], a3 = in[0 * 16] - in[2 * 16];
        tmp[0 + i * 4] = a0 + a1;
        tmp[1 + i * 4] = a3 + a2;
        tmp[2 + i * 4] = a3 - a2;
        tmp[3 + i * 4] = a0 - a1;
    }
    for (int i = 0; i < 4; i++) {
        const int a0 = tmp[0 + i] + tmp[8 + i], a1 = tmp[4 + i] + tmp[12 + i];
        const int a2 = tmp[4 + i] - tmp[12 + i], a3 = tmp[0 + i] - tmp[8 + i];
        out[0 + i] = (int16_t)((a0 + a1) >> 1);
        out[4 + i] = (int16_t)((a3 + a2) >> 1);
        out[8 + i] = (int16_t)((a3 - a2) >> 1);
        out[12 + i] = (int16_t)((a0 - a1) >> 1);
    }
}

// Dead-zone quantiser: level = (|c| + bias * step / 256) / step, clamped to the token range.
// coeffs (raster) -> levels (raster, signed); also leaves the dequantised values in coeffs.
LP_VP8_FN int quantize_block(int16_t* coeffs, int16_t* levels, const int* dq, int first, int bias_dc, int bias_ac) {
    int last = -1;
    const uint8_t zigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
    for (int n = 0; n < 16; n++) {
        const int j = zigzag[n];
        if (n < first) {
            levels[j] = 0;
            continue;  // coeffs[j] keeps the value the caller planted (DC from Y2)
        }
        const int step = dq[n > 0];
        const int c = coeffs[j], a = c < 0 ? -c : c;
        int lv = (a + ((n > 0 ? bias_ac : bias_dc) * step >> 8)) / step;
        if (lv > 2047) lv = 2047;
        levels[j] = (int16_t)(c < 0 ? -lv : lv);
        coeffs[j] = (int16_t)(levels[j] * step);
        if (lv) last = n;
    }
    return last;  // scan position of the last non-zero level, -1 if none
}

// ---- token writer: the exact mirror of vp8::get_coeffs --------------------------------------
LP_VP8_FN void put_large_value(BoolEnc& e, int v, const uint8_t* p) {
    if (v <= 4) {
        be_put(e, 0, p[3]);
        if (v == 2) be_put(e, 0, p[4]);
        else {
            be_put(e, 1, p[4]);
            be_put(e, v == 4, p[5]);
        }
    } else if (v <= 10) {
        be_put(e, 1, p[3]);
        be_put(e, 0, p[6]);
        if (v <= 6) {
            be_put(e, 0, p[7]);
            be_put(e, v == 6, 159);
        } else {
            be_put(e, 1, p[7]);
            be_put(e, v >= 9, 165);
            be_put(e, (v - 7) & 1, 145);
        }
    } else {
        be_put(e, 1, p[3]);
        be_put(e, 1, p[6]);
        const int cat = v < 19 ? 0 : v < 35 ? 1 : v < 67 ? 2 : 3;
        be_put(e, cat >> 1, p[8]);
        be_put(e, cat & 1, p[9 + (cat >> 1)]);
        const int extra = v - (3 + (8 << cat));
        const uint8_t c3[3] = {173, 148, 140}, c4[4] = {176, 155, 140, 135}, c5[5] = {180, 157, 141, 134, 130};
        const uint8_t c6[11] = {254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129};
        const int nb = cat == 3 ? 11 : cat + 3;
        const uint8_t* tab = cat == 0 ? c3 : cat == 1 ? c4 : cat == 2 ? c5 : c6;
        for (int i = 0; i < nb; i++) be_put(e, (extra >> (nb - 1 - i)) & 1, tab[i]);
    }
}
// which of the 16 levels of a block (raster order in memory) are non-zero, as a mask in ZIG-ZAG order
// (0 1 4 8 5 2 3 6 9 12 13 10 7 11 14 15): one 32-byte block load, the rest stays in registers
LP_VP8_INL uint32_t nonzero_mask(const int16_t* levels) {
    uint32_t w[8];
#ifdef __CUDA_ARCH__
    // blocks are 32-byte aligned.  The load is PTX rather than a read through a uint4 pointer: the levels are stored as
    // int16_t (by other lanes, the 4x4 trial overwriting the 16x16 levels), and the compiler may move or reuse a load
    // through another type across those stores -- a stale last position then codes trailing zeros instead of an EOB
    asm volatile("ld.v4.u32 {%0, %1, %2, %3}, [%8];\n\tld.v4.u32 {%4, %5, %6, %7}, [%8+16];"
                 : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
                 : "l"(levels)
                 : "memory");
#else
    for (int i = 0; i < 8; i++) w[i] = (uint32_t)(uint16_t)levels[2 * i] | (uint32_t)(uint16_t)levels[2 * i + 1] << 16;
#endif
#define LP_NZ(r) ((w[(r) >> 1] >> (16 * ((r) & 1)) & 0xFFFFu) ? 1u : 0u)
    return LP_NZ(0) | LP_NZ(1) << 1 | LP_NZ(4) << 2 | LP_NZ(8) << 3 | LP_NZ(5) << 4 | LP_NZ(2) << 5 | LP_NZ(3) << 6 |
           LP_NZ(6) << 7 | LP_NZ(9) << 8 | LP_NZ(12) << 9 | LP_NZ(13) << 10 | LP_NZ(10) << 11 | LP_NZ(7) << 12 |
           LP_NZ(11) << 13 | LP_NZ(14) << 14 | LP_NZ(15) << 15;
#undef LP_NZ
}
// index (zig-zag order) of the last non-zero level at or after `first`, -1 when there is none
LP_VP8_INL int last_nonzero(const int16_t* levels, int first) {
    const uint32_t mm = nonzero_mask(levels) >> first << first;
#ifdef __CUDA_ARCH__
    return 31 - __clz((int)mm);
#else
    int last = -1;
    for (int n = 0; n < 16; n++)
        if (mm >> n & 1u) last = n;
    return last;
#endif
}
// 1 when a block has a non-zero level at or after `first` (what put_coeffs returns for it)
LP_VP8_INL int block_nz(const int16_t* levels, int first) { return (nonzero_mask(levels) >> first) != 0; }
// levels in raster order; returns 1 when the block has a non-zero level at or after `first`.
LP_VP8_FN int put_coeffs(BoolEnc& e, const uint8_t* proba, int type, int ctx, int first, const int16_t* levels, int has_nz = 1) {
    const uint8_t bands[17] = {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0};
    const uint8_t zigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
    const uint8_t* tp = proba + type * (8 * 3 * 11);
    const int last = has_nz ? last_nonzero(levels, first) : -1;  // (has_nz == 0: the caller knows the block is empty)
    int n = first;
    const uint8_t* p = tp + (bands[n] * 3 + ctx) * 11;
    if (last < 0) {
        be_put(e, 0, p[0]);
        return 0;
    }
    be_put(e, 1, p[0]);
    while (n < 16) {
        const int c = levels[zigzag[n]];
        const int v = c < 0 ? -c : c;
        if (!v) {
            be_put(e, 0, p[1]);
            p = tp + (bands[++n] * 3 + 0) * 11;
            continue;
        }
        be_put(e, 1, p[1]);
        int next_ctx;
        if (v == 1) {
            be_put(e, 0, p[2]);
            next_ctx = 1;
        } else {
            be_put(e, 1, p[2]);
            put_large_value(e, v, p);
            next_ctx = 2;
        }
        be_put(e, c < 0, 128);
        if (++n == 16) break;
        p = tp + (bands[n] * 3 + next_ctx) * 11;
        if (n > last) {
            be_put(e, 0, p[0]);  // end of block
            break;
        }
        be_put(e, 1, p[0]);
    }
    return 1;
}

// ---- probability adaptation (RFC 6386 s.13.4: the frame header may replace any of the 4 x 8 x 3 x 11 coefficient
// probabilities) and the per-macroblock skip flag (s.9.11) ------------------------------------------------------------
// 256 * -log2(p / 256): the cost, in 1/256 bit, of coding the likelier-with-probability-p/256 branch
LP_VP8_TABLE uint16_t kVp8EntropyCost[256] = {
    2048, 2048, 1792, 1642, 1536, 1454, 1386, 1329, 1280, 1236, 1198, 1162, 1130, 1101, 1073, 1048,
    1024, 1002,  980,  961,  942,  924,  906,  890,  874,  859,  845,  831,  817,  804,  792,  780,
     768,  757,  746,  735,  724,  714,  705,  695,  686,  676,  668,  659,  650,  642,  634,  626,
     618,  611,  603,  596,  589,  582,  575,  568,  561,  555,  548,  542,  536,  530,  524,  518,
     512,  506,  501,  495,  490,  484,  479,  474,  468,  463,  458,  453,  449,  444,  439,  434,
     430,  425,  420,  416,  412,  407,  403,  399,  394,  390,  386,  382,  378,  374,  370,  366,
     362,  358,  355,  351,  347,  343,  340,  336,  333,  329,  326,  322,  319,  315,  312,  309,
     305,  302,  299,  296,  292,  289,  286,  283,  280,  277,  274,  271,  268,  265,  262,  259,
     256,  253,  250,  247,  245,  242,  239,  236,  234,  231,  228,  226,  223,  220,  218,  215,
     212,  210,  207,  205,  202,  200,  197,  195,  193,  190,  188,  185,  183,  181,  178,  176,
     174,  171,  169,  167,  164,  162,  160,  158,  156,  153,  151,  149,  147,  145,  143,  140,
     138,  136,  134,  132,  130,  128,  126,  124,  122,  120,  118,  116,  114,  112,  110,  108,
     106,  104,  102,  101,   99,   97,   95,   93,   91,   89,   87,   86,   84,   82,   80,   78,
      77,   75,   73,   71,   70,   68,   66,   64,   63,   61,   59,   58,   56,   54,   53,   51,
      49,   48,   46,   44,   43,   41,   40,   38,   36,   35,   33,   32,   30,   28,   27,   25,
      24,   22,   21,   19,   18,   16,   15,   13,   12,   10,    9,    7,    6,    4,    3,    1,
};

constexpr int kNumProbas = 4 * 8 * 3 * 11;
// Per-frame side memory of the bitstream pass (`aux`, kAuxBytes, 4-byte aligned, zeroed by the encoder itself):
//   uint32 stats[kNumProbas][2]  how often each adaptive branch of the token tree coded a 0 / a 1
//   uint32 counts[2]             macroblocks, macroblocks without a non-zero level
//   uint8  proba[kNumProbas]     the probabilities the frame is coded with
//   uint8  update[kNumProbas]    1 = the header replaces the default by proba[i]
//   uint8  skip_proba, use_skip
constexpr size_t kAuxStatsOff = 0, kAuxCountsOff = (size_t)kNumProbas * 8, kAuxProbaOff = kAuxCountsOff + 8,
                 kAuxUpdateOff = kAuxProbaOff + kNumProbas, kAuxSkipOff = kAuxUpdateOff + kNumProbas,
                 kAuxBytes = (kAuxSkipOff + 2 + 255) / 256 * 256;

LP_VP8_INL void stat_add(uint32_t* stats, int idx, int bit) {
#ifdef __CUDA_ARCH__
    atomicAdd(stats + 2 * idx + bit, 1u);  // the lanes of a warp walk different partitions of the same frame
#else
    stats[2 * idx + bit]++;
#endif
}

// put_coeffs with the coder replaced by counters: which adaptive branches the block takes.  (The fixed-probability
// branches -- extra bits, signs -- cannot be adapted and are not counted.)
LP_VP8_FN int record_coeffs(uint32_t* stats, int type, int ctx, int first, const int16_t* levels, int has_nz = 1) {
    const uint8_t bands[17] = {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0};
    const uint8_t zigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
    const int tb = type * (8 * 3 * 11);
    const int last = has_nz ? last_nonzero(levels, first) : -1;
    int n = first;
    int p = tb + (bands[n] * 3 + ctx) * 11;
    if (last < 0) {
        stat_add(stats, p + 0, 0);
        return 0;
    }
    stat_add(stats, p + 0, 1);
    while (n < 16) {
        const int c = levels[zigzag[n]];
        const int v = c < 0 ? -c : c;
        if (!v) {
            stat_add(stats, p + 1, 0);
            p = tb + (bands[++n] * 3 + 0) * 11;
            continue;
        }
        stat_add(stats, p + 1, 1);
        int next_ctx;
        if (v == 1) {
            stat_add(stats, p + 2, 0);
            next_ctx = 1;
        } else {
            stat_add(stats, p + 2, 1);
            next_ctx = 2;
            if (v <= 4) {  // the tree of put_large_value
                stat_add(stats, p + 3, 0);
                stat_add(stats, p + 4, v != 2);
                if (v != 2) stat_add(stats, p + 5, v == 4);
            } else if (v <= 10) {
                stat_add(stats, p + 3, 1);
                stat_add(stats, p + 6, 0);
                stat_add(stats, p + 7, v > 6);
            } else {
                stat_add(stats, p + 3, 1);
                stat_add(stats, p + 6, 1);
                const int cat = v < 19 ? 0 : v < 35 ? 1 : v < 67 ? 2 : 3;
                stat_add(stats, p + 8, cat >> 1);
                stat_add(stats, p + 9 + (cat >> 1), cat & 1);
            }
        }
        if (++n == 16) break;
        p = tb + (bands[n] * 3 + next_ctx) * 11;
        if (n > last) {
            stat_add(stats, p + 0, 0);
            break;
        }
        stat_add(stats, p + 0, 1);
    }
    return 1;
}

// all 25 blocks of a macroblock are zero: the decoder can be told to skip its tokens
LP_VP8_INL int mb_is_skippable(const int16_t* lv) {
    uint32_t any = 0;
    for (int k = 0; k < 25; k++) any |= nonzero_mask(lv + k * 16);
    return any == 0;
}

// One entry of the probability table from its counters: the frame's own frequency, adopted when the bits it saves over
// the default pay for the 8 bits (+ flag) that announce it.  `c0` / `c1` = times the branch coded 0 / 1.
LP_VP8_FN void decide_proba(uint32_t c0, uint32_t c1, int old_p, int update_p, uint8_t* proba, uint8_t* update) {
    const uint32_t total = c0 + c1;
    int new_p = total ? (int)(255u - (uint32_t)(((uint64_t)c1 * 255u) / total)) : 255;
    if (new_p < 1) new_p = 1;
    const uint64_t old_cost = (uint64_t)c0 * kVp8EntropyCost[old_p] + (uint64_t)c1 * kVp8EntropyCost[255 - old_p] + kVp8EntropyCost[update_p];
    const uint64_t new_cost = (uint64_t)c0 * kVp8EntropyCost[new_p] + (uint64_t)c1 * kVp8EntropyCost[255 - new_p] +
                              kVp8EntropyCost[255 - update_p] + 8 * 256;
    const bool use_new = new_cost < old_cost;
    *proba = (uint8_t)(use_new ? new_p : old_p);
    *update = use_new ? 1 : 0;
}

// ---- 4x4 intra modes (RFC 6386 s.8.3 / 12.3) ------------------------------------------------------------------------
// Per macroblock kModeStride bytes of mode information: [0] = the 16x16 luma mode (0..3) or kI4 when the macroblock predicts
// its sixteen 4x4 blocks one by one, [1] = the chroma mode, [2..17] = the sub-block modes in raster order.  A 16x16
// macroblock fills them with its own mode, which is what its neighbours' sub-block modes are coded against (s.8.3).
constexpr int kModeStride = 24;  // + [20..23]: which of the 25 blocks have a non-zero level (bit k = block k), see mb_nz_mask
constexpr int kI4 = 4;
constexpr int kTryI4 = 1;  // what the product encodes with (Params::try_i4 of the device launchers and of the host build)

// The macroblock's non-zero-block mask (written once by the analysis, read by the first partition and by both token
// walks instead of scanning the 25 blocks' levels again: a block's flag is what the neighbours' contexts, the skip test
// and the "no coefficients" shortcut of the token writer ask for).
LP_VP8_INL uint32_t mb_nz_mask(const uint8_t* md) { return *reinterpret_cast<const uint32_t*>(md + 20); }
LP_VP8_INL void mb_set_nz_mask(uint8_t* md, uint32_t m) { *reinterpret_cast<uint32_t*>(md + 20) = m; }

// cost, in 1/256 bit, of a bit coded with probability `p` of being 0
LP_VP8_INL int bit_cost(int bit, int p) { return kVp8EntropyCost[bit ? 255 - p : p]; }

// The ten 4x4 predictors as data (tools/gen_vp8_pred4_table.py reads them out of vp8::pred_4x4's source): entry =
// i0 | i1 << 4 | i2 << 8 | kind << 12 over the edge samples e[13] = {L, K, J, I, X, A, B, C, D, E, F, G, H} (left column
// bottom-up, corner, the row above and its four above-right samples); kind 0 = (e[i0] + 2 e[i1] + e[i2] + 2) >> 2,
// 1 = (e[i0] + e[i1] + 1) >> 1, 2 = e[i0], 3 = B_DC / B_TM (computed from the mode).  A lane can so evaluate any mode of
// any pixel without the ten-way switch of pred_4x4.
LP_VP8_TABLE uint16_t kVp8Pred4[10][16] = {
    {0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000},  // B_DC
    {0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000, 0x3000},  // B_TM
    {0x0654, 0x0765, 0x0876, 0x0987, 0x0654, 0x0765, 0x0876, 0x0987, 0x0654, 0x0765, 0x0876, 0x0987, 0x0654, 0x0765, 0x0876, 0x0987},  // B_VE
    {0x0234, 0x0234, 0x0234, 0x0234, 0x0123, 0x0123, 0x0123, 0x0123, 0x0012, 0x0012, 0x0012, 0x0012, 0x0001, 0x0001, 0x0001, 0x0001},  // B_HE
    {0x0345, 0x0456, 0x0567, 0x0678, 0x0234, 0x0345, 0x0456, 0x0567, 0x0123, 0x0234, 0x0345, 0x0456, 0x0012, 0x0123, 0x0234, 0x0345},  // B_RD
    {0x1054, 0x1065, 0x1076, 0x1087, 0x0543, 0x0654, 0x0765, 0x0876, 0x0432, 0x1054, 0x1065, 0x1076, 0x0321, 0x0543, 0x0654, 0x0765},  // B_VR
    {0x0765, 0x0876, 0x0987, 0x0a98, 0x0876, 0x0987, 0x0a98, 0x0ba9, 0x0987, 0x0a98, 0x0ba9, 0x0cba, 0x0a98, 0x0ba9, 0x0cba, 0x0ccb},  // B_LD
    {0x1065, 0x1076, 0x1087, 0x1098, 0x0765, 0x0876, 0x0987, 0x0a98, 0x1076, 0x1087, 0x1098, 0x0ba9, 0x0876, 0x0987, 0x0a98, 0x0cba},  // B_VL
    {0x1043, 0x0543, 0x0654, 0x0765, 0x1032, 0x0432, 0x1043, 0x0543, 0x1021, 0x0321, 0x1032, 0x0432, 0x1010, 0x0210, 0x1021, 0x0321},  // B_HD
    {0x1023, 0x0123, 0x1012, 0x0012, 0x1012, 0x0012, 0x1001, 0x0001, 0x1001, 0x0001, 0x2000, 0x2000, 0x2000, 0x2000, 0x2000, 0x2000},  // B_HU
};

// pixel p (= 4 * y + x) of mode `mode`; dc = (A + B + C + D + I + J + K + L + 4) >> 3
LP_VP8_INL int pred4_px(int mode, int p, const uint8_t* e, int dc) {
    // straight-line on purpose: the lanes of a warp ask for different kinds at once
    const uint32_t t = kVp8Pred4[mode][p];
    const int a = e[t & 15], b = e[(t >> 4) & 15], c = e[(t >> 8) & 15], kind = (int)(t >> 12);
    const int tm = vp8::clip8(e[5 + (p & 3)] + e[3 - (p >> 2)] - e[4]);  // B_TM: above + left - corner
    const int avg = kind == 0 ? (a + 2 * b + c + 2) >> 2 : (a + b + 1) >> 1;
    const int special = mode == vp8::B_DC ? dc : tm;
    return kind < 2 ? avg : kind == 2 ? a : special;
}

// The path of every sub-block mode through the tree of s.8.3: nodes (= index of the probability) as nibbles, the
// branch taken at each as a bit mask, length in bits 8..10.  i4_mode_cost == i4_mode<false> (checked in the tests),
// without its data-dependent branches.
LP_VP8_TABLE uint32_t kVp8BModePathNodes[10] = {0x0000000, 0x0000010, 0x0000210, 0x0043210, 0x0543210, 0x0543210, 0x0063210, 0x0763210, 0x8763210, 0x8763210};
LP_VP8_TABLE uint16_t kVp8BModePathBits[10] = {0x100, 0x201, 0x303, 0x507, 0x617, 0x637, 0x50f, 0x61f, 0x73f, 0x77f};
// The cost (1/256 bit) of every sub-block mode in every context [above][left][mode]: i4_mode_cost over
// kVp8BModesProba, tabulated (the two inputs are constants of the format; the tests compare the table with the walk).
LP_VP8_TABLE uint16_t kVp8BModeCost[10][10][10] = {
    {{38, 1154, 1728, 1874, 2103, 2019, 1628, 1777, 2225, 2135}, {193, 468, 1297, 1306, 1848, 1793, 1780, 1700, 1707, 1515}, {140, 914, 763, 1690, 1854, 1579, 1461, 1302, 1800, 1657}, {561, 641, 1388, 414, 1181, 1570, 1620, 1746, 859, 1002}, {299, 1065, 1263, 1105, 627, 1062, 1590, 1897, 860, 1135}, {277, 1113, 707, 1363, 1083, 663, 1603, 1536, 1539, 1283}, {212, 783, 1629, 1301, 1632, 2232, 720, 1563, 1716, 912}, {151, 1041, 1050, 1768, 1991, 2183, 1360, 736, 1741, 1389}, {518, 1048, 1418, 749, 747, 1296, 1501, 1626, 451, 1209}, {425, 829, 1369, 713, 1462, 1199, 1205, 1471, 1196, 530}},
    {{239, 401, 1135, 1491, 1660, 1505, 1517, 1553, 1979, 2099}, {468, 240, 961, 1230, 1713, 1616, 1832, 1568, 1675, 1385}, {501, 452, 460, 1505, 1699, 1279, 1565, 976, 2123, 2126}, {676, 648, 1389, 324, 1595, 1674, 1457, 1933, 988, 868}, {458, 787, 1043, 909, 732, 962, 1165, 1524, 851, 1025}, {506, 815, 500, 1138, 1215, 712, 1514, 1079, 1262, 1265}, {333, 629, 1463, 1244, 1889, 3936, 794, 1553, 1907, 590}, {399, 646, 746, 1343, 1860, 1348, 1513, 607, 1863, 1009}, {626, 753, 1216, 603, 1064, 1408, 1299, 1410, 537, 965}, {501, 754, 1044, 662, 1225, 1614, 1305, 1431, 1385, 514}},
    {{394, 552, 521, 1500, 1534, 975, 1606, 1136, 1661, 2182}, {659, 428, 372, 1412, 1861, 1217, 1679, 1132, 1979, 1551}, {695, 645, 241, 1962, 2082, 1191, 1533, 980, 1983, 2246}, {561, 839, 743, 863, 1124, 974, 1230, 846, 1085, 775}, {695, 880, 514, 955, 666, 890, 1056, 1187, 1525, 1121}, {746, 960, 381, 1285, 1177, 485, 1585, 1156, 1849, 1512}, {322, 777, 1059, 1783, 3319, 1274, 808, 1185, 1376, 645}, {490, 975, 482, 1774, 1519, 1782, 1115, 497, 1540, 1461}, {746, 1015, 1008, 702, 842, 1223, 1331, 781, 732, 711}, {524, 1084, 571, 1041, 1340, 880, 1045, 1142, 1198, 686}},
    {{104, 867, 1447, 1008, 1939, 1842, 1520, 1924, 1674, 1577}, {536, 303, 1203, 677, 1386, 2174, 1812, 1901, 1258, 1161}, {305, 517, 877, 1106, 1424, 3471, 1423, 1059, 1314, 1235}, {686, 732, 2180, 250, 1507, 2066, 1875, 1552, 1048, 940}, {394, 817, 1032, 657, 955, 1555, 1284, 1288, 887, 1042}, {530, 620, 1000, 936, 1197, 628, 1093, 2767, 797, 1356}, {347, 615, 1605, 1185, 3388, 1343, 1004, 1337, 1007, 655}, {218, 741, 877, 1599, 3902, 3905, 1345, 750, 1350, 1613}, {676, 752, 1584, 550, 1253, 1597, 1865, 2384, 393, 1085}, {596, 687, 1168, 424, 1089, 1501, 1482, 1487, 1088, 813}},
    {{228, 1069, 1062, 1376, 748, 978, 1513, 1519, 981, 1785}, {495, 513, 818, 940, 961, 888, 1615, 1353, 1042, 1359}, {518, 648, 591, 1039, 756, 986, 1194, 1452, 1303, 1458}, {686, 750, 1052, 668, 833, 1392, 1133, 1136, 644, 934}, {626, 1125, 1125, 996, 355, 1072, 1205, 1316, 871, 1215}, {634, 1077, 859, 1665, 644, 470, 1671, 1415, 822, 1166}, {555, 729, 1076, 1335, 3386, 1341, 818, 1334, 1073, 418}, {506, 878, 624, 1400, 883, 886, 1400, 802, 887, 1408}, {686, 1706, 1306, 977, 571, 983, 1288, 1722, 397, 1114}, {399, 870, 1451, 1068, 1069, 759, 965, 1485, 1220, 671}},
    {{333, 763, 936, 1652, 1006, 520, 1653, 1408, 1469, 2227}, {512, 494, 749, 1158, 1212, 602, 1883, 1874, 1625, 1165}, {575, 644, 489, 1975, 1206, 596, 1578, 1094, 1392, 1992}, {792, 794, 947, 578, 1013, 947, 1615, 1201, 723, 761}, {695, 1024, 675, 1079, 574, 495, 1694, 1440, 1104, 3151}, {780, 1285, 570, 1999, 1259, 235, 3146, 1387, 1795, 1458}, {453, 898, 1311, 902, 1315, 3362, 458, 1309, 1316, 804}, {394, 938, 942, 1098, 1355, 1099, 945, 586, 1359, 1103}, {561, 1017, 1016, 1013, 652, 1173, 1016, 1161, 612, 1024}, {568, 796, 631, 1003, 1006, 856, 2567, 1268, 931, 757}},
    {{265, 605, 1099, 1226, 1495, 1239, 946, 1025, 1735, 1460}, {366, 586, 905, 1056, 1406, 1244, 872, 1131, 1618, 1049}, {453, 564, 539, 1735, 1479, 1482, 1015, 882, 3193, 1148}, {555, 1097, 1576, 945, 1350, 890, 835, 1016, 1017, 486}, {705, 818, 1215, 967, 970, 633, 1219, 2463, 825, 569}, {676, 1264, 577, 868, 870, 768, 871, 1273, 1023, 944}, {296, 1147, 2048, 1798, 1649, 3696, 436, 1556, 2088, 712}, {343, 992, 1258, 1864, 1864, 1867, 618, 562, 1850, 1046}, {555, 1075, 1321, 819, 737, 1337, 1075, 1325, 1074, 485}, {289, 1170, 1308, 1175, 1642, 1645, 832, 2506, 1306, 502}},
    {{340, 720, 766, 1874, 1764, 1269, 1253, 541, 1758, 2170}, {484, 654, 693, 1509, 1455, 1406, 1219, 499, 1917, 1262}, {490, 758, 445, 3242, 1823, 1274, 1664, 536, 1867, 2130}, {524, 1106, 1092, 847, 1362, 1106, 849, 896, 955, 596}, {714, 718, 843, 723, 728, 939, 938, 856, 3096, 1051}, {518, 1342, 499, 1339, 1078, 674, 1339, 711, 1604, 1348}, {453, 1178, 1390, 1917, 1514, 3561, 306, 941, 1916, 917}, {403, 1539, 980, 2173, 1770, 3817, 1075, 268, 3633, 1588}, {561, 1373, 1108, 609, 665, 2712, 972, 787, 977, 980}, {548, 1145, 1063, 809, 1408, 948, 1143, 616, 1264, 642}},
    {{164, 985, 1244, 932, 1329, 1361, 1658, 1574, 954, 1609}, {596, 420, 927, 842, 1134, 1108, 1396, 2051, 853, 1033}, {403, 839, 729, 763, 932, 1663, 1247, 802, 1402, 1405}, {906, 880, 1078, 374, 1586, 1741, 1444, 2441, 471, 1030}, {642, 1097, 1022, 1025, 674, 1378, 1624, 2355, 407, 858}, {561, 1017, 821, 910, 703, 764, 1426, 912, 830, 1430}, {416, 1277, 1267, 868, 1281, 3328, 766, 1018, 1286, 513}, {407, 996, 599, 1006, 1265, 1268, 1262, 752, 1009, 1272}, {980, 1190, 1375, 788, 1034, 1297, 1700, 1707, 193, 1414}, {735, 887, 1297, 465, 896, 1159, 1560, 1294, 746, 749}},
    {{110, 936, 1381, 1183, 1936, 1646, 1147, 1713, 1869, 1300}, {407, 413, 1030, 1018, 1910, 1398, 1313, 1645, 1503, 786}, {343, 641, 574, 1089, 1241, 1349, 1161, 1351, 1761, 1505}, {561, 769, 1207, 351, 1689, 1433, 1331, 1912, 1215, 795}, {474, 914, 1172, 766, 712, 2759, 1433, 1438, 714, 775}, {343, 893, 785, 1146, 1148, 789, 1298, 1554, 968, 1052}, {207, 1039, 1334, 1344, 1608, 3655, 809, 1460, 1614, 704}, {228, 931, 892, 1046, 3760, 1715, 993, 825, 1718, 1314}, {768, 727, 1059, 633, 989, 1073, 1319, 1333, 609, 820}, {305, 1176, 1375, 895, 1586, 1589, 984, 1980, 1325, 489}},
};
LP_VP8_INL int i4_mode_cost_ctx(int top, int left, int mode) { return kVp8BModeCost[top][left][mode]; }
LP_VP8_INL int i4_mode_cost(int mode, const uint8_t* prob) {
    const uint32_t nodes = kVp8BModePathNodes[mode], bits = kVp8BModePathBits[mode];
    const int len = (int)(bits >> 8);
    int cost = 0;
    for (int k = 0; k < 7; k++)
        if (k < len) cost += bit_cost((int)((bits >> k) & 1u), prob[(nodes >> (4 * k)) & 15u]);
    return cost;
}

// the sub-block mode tree of s.8.3 (kVp8YModesIntra4) walked for `mode`: PUT = code it, else return its cost
template <bool PUT>
LP_VP8_FN int i4_mode(BoolEnc* e, int mode, const uint8_t* prob) {
    int cost = 0;
#define LP_BM(bit_, k_)                              \
    ((PUT ? (be_put(*e, (bit_), prob[k_]), 0) : (cost += bit_cost((bit_), prob[k_]))), (bit_))
    if (LP_BM(mode != vp8::B_DC, 0)) {
        if (LP_BM(mode != vp8::B_TM, 1)) {
            if (LP_BM(mode != vp8::B_VE, 2)) {
                if (!LP_BM(mode >= vp8::B_LD, 3)) {
                    if (LP_BM(mode != vp8::B_HE, 4)) LP_BM(mode != vp8::B_RD, 5);
                } else {
                    if (LP_BM(mode != vp8::B_LD, 6)) {
                        if (LP_BM(mode != vp8::B_VL, 7)) LP_BM(mode != vp8::B_HD, 8);
                    }
                }
            }
        }
    }
#undef LP_BM
    return cost;
}

// put_coeffs with the coder replaced by a bit count (1/256 bit) under the default probabilities: the rate estimate
// of the 16x16-versus-4x4 decision, written as a sum over scan positions so that the device can give every position a
// lane.  cost_pos = what position n adds: `v` / `vprev` = the magnitudes at scan positions n and n - 1, `last` = the
// last non-zero position (-1: none), ctx0 = the block's context.
LP_VP8_INL int cost_pos(const uint8_t* tp, int ctx0, int first, int last, int v, int vprev, int n) {
    const uint8_t bands[17] = {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0};
    if (last < 0) return n == first ? bit_cost(0, tp[(bands[n] * 3 + ctx0) * 11]) : 0;  // "no coefficients"
    if (n < first || n > last + 1 || n > 15) return 0;
    const int ctx = n == first ? ctx0 : vprev == 0 ? 0 : vprev == 1 ? 1 : 2;
    const uint8_t* p = tp + (bands[n] * 3 + ctx) * 11;
    if (n == last + 1) return bit_cost(0, p[0]);  // end of block
    int c = 0;
    if (n == first || vprev != 0) c += bit_cost(1, p[0]);  // "not the end": coded unless the previous level was zero
    if (!v) return c + bit_cost(0, p[1]);
    c += bit_cost(1, p[1]) + 256;  // + the sign
    if (v == 1) return c + bit_cost(0, p[2]);
    c += bit_cost(1, p[2]);
    if (v <= 4) return c + bit_cost(0, p[3]) + bit_cost(v != 2, p[4]) + (v != 2 ? bit_cost(v == 4, p[5]) : 0);
    if (v <= 10) return c + bit_cost(1, p[3]) + bit_cost(0, p[6]) + bit_cost(v > 6, p[7]) + (v > 6 ? 512 : 256);
    const int cat = v < 19 ? 0 : v < 35 ? 1 : v < 67 ? 2 : 3;
    return c + bit_cost(1, p[3]) + bit_cost(1, p[6]) + bit_cost(cat >> 1, p[8]) + bit_cost(cat & 1, p[9 + (cat >> 1)]) +
           256 * (cat == 3 ? 11 : cat + 3);  // extra bits: about one bit each
}
// Returns the cost of a block; *nz = what put_coeffs would return.
LP_VP8_FN int cost_coeffs(int type, int ctx, int first, const int16_t* levels, int* nz) {
    const uint8_t zigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
    const uint8_t* tp = &kVp8CoeffProba0[0][0][0][0] + type * (8 * 3 * 11);
    const int last = last_nonzero(levels, first);
    *nz = last >= 0;
    int cost = 0, vprev = 0;
    for (int n = first; n < 16; n++) {
        const int c = levels[zigzag[n]];
        const int v = c < 0 ? -c : c;
        cost += cost_pos(tp, ctx, first, last, v, vprev, n);
        vprev = v;
    }
    return cost;
}

// ---- colour conversion (BT.601 limited range, 16.16 fixed point like libwebp's importer) -----
LP_VP8_INL int rgb_to_y(int r, int g, int b) { return (16839 * r + 33059 * g + 6420 * b + (16 << 16) + (1 << 15)) >> 16; }
// r, g, b are SUMS over a 2x2 block
LP_VP8_INL int rgb_to_u(int r, int g, int b) { return vp8::clip8((-9719 * r - 19081 * g + 28800 * b + (128 << 18) + (1 << 17)) >> 18); }
LP_VP8_INL int rgb_to_v(int r, int g, int b) { return vp8::clip8((28800 * r - 24116 * g - 4684 * b + (128 << 18) + (1 << 17)) >> 18); }

// ---- quality -> quantiser index (libwebp's mapping, so `quality` means the same thing) --------
// q = 127 * (1 - cbrt(linear(quality / 100))), linear(c) = c < 0.75 ? c * 2/3 : 2c - 1.
// Integer cube root by search keeps this usable without libm on the device.
LP_VP8_HD int quality_to_q(int quality) {
    if (quality < 0) quality = 0;
    if (quality > 100) quality = 100;
    // linear_c in 1/3000 units: c < 0.75 -> c*2/3 = quality*20/3000 ; else 2c-1 = (quality*60 - 3000)/3000
    const long lin = quality < 75 ? (long)quality * 20 : (long)quality * 60 - 3000;  // / 3000
    // v = cbrt(lin/3000); find the largest k in 0..127 with ((127 - k)/127)^3 >= lin/3000  <=>  q = k
    // (q = floor(127 * (1 - v))  <=>  127 - q is the smallest integer m with m >= 127 v ... solve by scan)
    int q = 0;
    for (int k = 127; k >= 0; k--) {
        // 127*(1 - v) >= k  <=>  v <= (127 - k)/127  <=>  lin/3000 <= ((127-k)/127)^3
        const long m = 127 - k;
        if (lin * 127 * 127 * 127 <= m * m * m * 3000) {
            q = k;
            break;
        }
    }
    return q;
}

// Loop-filter level from the quantiser: stronger quantisation, stronger deblocking (0 = off).
LP_VP8_FN int filter_level_for_q(int q) {
    const int level = kVp8AcTable[q] * 3 / 10;
    return level < 2 ? 0 : level > 63 ? 63 : level;
}

// ---- the encoder ----------------------------------------------------------------------------
struct Params {
    int width, height, mb_w, mb_h;
    int q;             // quantiser index 0..127
    int filter_level;  // 0..63
    int try_i4;        // 1 = weigh sixteen 4x4 predictions against the 16x16 one per macroblock
};

// Source planes: mb_w*16 x mb_h*16 luma, half-size chroma, padded by edge replication.
// recon_*: same geometry, written here (the decoder's unfiltered reconstruction).
// levels: mb_w*mb_h*25*16 int16 (blocks 0..15 Y, 16..19 U, 20..23 V, 24 Y2), modes: kModeStride bytes per MB.
struct Buffers {
    const uint8_t *sy, *su, *sv;
    uint8_t *ry, *ru, *rv;
    int16_t* levels;
    uint8_t* modes;
};

LP_VP8_FN uint32_t sse_block(const uint8_t* a, int as, const uint8_t* b, int bs, int size) {
    uint32_t s = 0;
    for (int y = 0; y < size; y++)
        for (int x = 0; x < size; x++) {
            const int d = a[y * as + x] - b[y * bs + x];
            s += (uint32_t)(d * d);
        }
    return s;
}

// The sixteen 4x4 blocks of a macroblock predicted one by one (s.12.3): for every block the mode with the least
// prediction error + mode cost, then transform, quantisation and reconstruction, because the next block predicts from
// this one's reconstruction.  `yd` = the macroblock inside its bordered work buffer (borders and the above-right samples
// set by the caller, as the decoder sets them); top_modes / left_modes = the neighbours' sub-block modes (updated to
// this macroblock's on return).  Outputs: levels[16][16], modes[16], the reconstruction in yd.
// Returns distortion (SSE) and adds the rate estimate (1/256 bit) to *rate.
LP_VP8_FN uint32_t analyse_i4(const uint8_t* sy, int ys, uint8_t* yd, const int* y1q, int lambda4, uint8_t* top_modes,
                              uint8_t* left_modes, int16_t* levels, uint8_t* modes, uint32_t* rate) {
    uint32_t dist = 0, bits = 0;
    uint8_t tnz[4] = {0, 0, 0, 0}, lnz[4] = {0, 0, 0, 0};  // contexts of the rate estimate only
    int16_t coeffs[16];
    for (int r = 1; r < 4; r++)  // the above-right samples of the macroblock serve every row of sub-blocks
        for (int i = 16; i < 20; i++) yd[(4 * r - 1) * BPS + i] = yd[i - BPS];
    for (int n = 0; n < 16; n++) {
        const int bx = n & 3, by = n >> 2;
        uint8_t* d = yd + by * 4 * BPS + bx * 4;
        const uint8_t* src = sy + by * 4 * ys + bx * 4;
        int best_mode = 0;
        uint32_t best = 0xffffffffu;
        for (int m = 0; m < 10; m++) {
            vp8::pred_4x4(d, BPS, m);
            const uint32_t score = sse_block(src, ys, d, BPS, 4) * 256u + (uint32_t)(i4_mode_cost_ctx(top_modes[bx], left_modes[by], m) * lambda4);
            if (score < best) {
                best = score;
                best_mode = m;
            }
        }
        vp8::pred_4x4(d, BPS, best_mode);
        fdct4x4(src, ys, d, BPS, coeffs);
        quantize_block(coeffs, levels + n * 16, y1q, 0, 96, 110);
        vp8::inverse_dct_add(coeffs, d, BPS);
        dist += sse_block(src, ys, d, BPS, 4);
        int nz;
        bits += (uint32_t)i4_mode_cost_ctx(top_modes[bx], left_modes[by], best_mode) + (uint32_t)cost_coeffs(3, tnz[bx] + lnz[by], 0, levels + n * 16, &nz);
        tnz[bx] = lnz[by] = (uint8_t)nz;
        modes[n] = (uint8_t)best_mode;
        top_modes[bx] = left_modes[by] = (uint8_t)best_mode;
    }
    *rate += bits;
    return dist;
}

// Pass 1: mode decision, transform, quantisation and reconstruction of every macroblock, raster order.
LP_VP8_FN void analyse_and_reconstruct(const Params& P, const Buffers& B) {
    const int ys = P.mb_w * 16, cs = P.mb_w * 8;
    vp8::QuantMat qm;
    qm.y1[0] = kVp8DcTable[P.q];
    qm.y1[1] = kVp8AcTable[P.q];
    qm.y2[0] = kVp8DcTable[P.q] * 2;
    qm.y2[1] = (kVp8AcTable[P.q] * 101581) >> 16;
    if (qm.y2[1] < 8) qm.y2[1] = 8;
    qm.uv[0] = kVp8DcTable[P.q > 117 ? 117 : P.q];
    qm.uv[1] = kVp8AcTable[P.q];
    uint8_t yb[vp8::YB_SIZE], ub[vp8::CB_SIZE], vb[vp8::CB_SIZE];
    int16_t coeffs[25 * 16];
    for (int mb_y = 0; mb_y < P.mb_h; mb_y++)
        for (int mb_x = 0; mb_x < P.mb_w; mb_x++) {
            uint8_t* yd = yb + BPS + 8;
            uint8_t* ud = ub + BPS + 8;
            uint8_t* vd = vb + BPS + 8;
            const uint8_t* sy = B.sy + (size_t)mb_y * 16 * ys + mb_x * 16;
            const uint8_t* su = B.su + (size_t)mb_y * 8 * cs + mb_x * 8;
            const uint8_t* sv = B.sv + (size_t)mb_y * 8 * cs + mb_x * 8;
            uint8_t* py = B.ry + (size_t)mb_y * 16 * ys + mb_x * 16;
            uint8_t* pu = B.ru + (size_t)mb_y * 8 * cs + mb_x * 8;
            uint8_t* pv = B.rv + (size_t)mb_y * 8 * cs + mb_x * 8;
            // prediction borders from the reconstruction, as the decoder will see them (s.12.2)
            for (int j = 0; j < 16; j++) yd[j * BPS - 1] = mb_x > 0 ? py[j * ys - 1] : 129;
            for (int j = 0; j < 8; j++) {
                ud[j * BPS - 1] = mb_x > 0 ? pu[j * cs - 1] : 129;
                vd[j * BPS - 1] = mb_x > 0 ? pv[j * cs - 1] : 129;
            }
            for (int i = -1; i < 16; i++)
                yd[i - BPS] = mb_y > 0 ? ((i < 0 && mb_x == 0) ? 129 : py[i - ys]) : 127;
            for (int i = -1; i < 8; i++) {
                ud[i - BPS] = mb_y > 0 ? ((i < 0 && mb_x == 0) ? 129 : pu[i - cs]) : 127;
                vd[i - BPS] = mb_y > 0 ? ((i < 0 && mb_x == 0) ? 129 : pv[i - cs]) : 127;
            }
            // luma 16x16 mode: least squared prediction error
            int ymode = 0;
            uint32_t best = 0xffffffffu;
            for (int m = 0; m < 4; m++) {
                vp8::pred_block(yd, BPS, 16, m, mb_y > 0, mb_x > 0);
                const uint32_t s = sse_block(sy, ys, yd, BPS, 16);
                if (s < best) {
                    best = s;
                    ymode = m;
                }
            }
            vp8::pred_block(yd, BPS, 16, ymode, mb_y > 0, mb_x > 0);
            int uvmode = 0;
            best = 0xffffffffu;
            for (int m = 0; m < 4; m++) {
                vp8::pred_block(ud, BPS, 8, m, mb_y > 0, mb_x > 0);
                vp8::pred_block(vd, BPS, 8, m, mb_y > 0, mb_x > 0);
                const uint32_t s = sse_block(su, cs, ud, BPS, 8) + sse_block(sv, cs, vd, BPS, 8);
                if (s < best) {
                    best = s;
                    uvmode = m;
                }
            }
            vp8::pred_block(ud, BPS, 8, uvmode, mb_y > 0, mb_x > 0);
            vp8::pred_block(vd, BPS, 8, uvmode, mb_y > 0, mb_x > 0);
            // residual transforms + quantisation
            int16_t* lv = B.levels + ((size_t)mb_y * P.mb_w + mb_x) * 25 * 16;
            uint8_t* md = B.modes + ((size_t)mb_y * P.mb_w + mb_x) * kModeStride;
            for (int n = 0; n < 16; n++)
                fdct4x4(sy + (n >> 2) * 4 * ys + (n & 3) * 4, ys, yd + (n >> 2) * 4 * BPS + (n & 3) * 4, BPS, coeffs + n * 16);
            fwht(coeffs, coeffs + 24 * 16);
            quantize_block(coeffs + 24 * 16, lv + 24 * 16, qm.y2, 0, 96, 108);
            vp8::inverse_wht(coeffs + 24 * 16, coeffs);  // plants the dequantised DCs
            for (int n = 0; n < 16; n++) quantize_block(coeffs + n * 16, lv + n * 16, qm.y1, 1, 96, 110);
            // ---- 16x16 or sixteen 4x4 predictions?  Both are carried to their reconstruction; the smaller
            //      distortion + lambda * estimated bits wins (lambda = q^2 / 128 per bit, libwebp's mode lambda).
            uint8_t top_modes[4], left_modes[4];
            for (int i = 0; i < 4; i++) {
                top_modes[i] = mb_y > 0 ? (md - (size_t)P.mb_w * kModeStride)[2 + 12 + i] : (uint8_t)vp8::B_DC;
                left_modes[i] = mb_x > 0 ? (md - kModeStride)[2 + 4 * i + 3] : (uint8_t)vp8::B_DC;
            }
            bool use_i4 = false;
            // (a macroblock whose 16x16 residual quantises to DC terms only is flat: sixteen 4x4 predictions would spend
            // mode bits on nothing, so the trial is skipped -- a third of the macroblocks of a photograph)
            bool flat16 = true;
            for (int n = 0; n < 16; n++) flat16 = flat16 && !block_nz(lv + n * 16, 1);
            if (P.try_i4 && !flat16) {
                // the 16x16 candidate's reconstruction, distortion and rate
                uint8_t y16[16 * 16];
                {
                    int16_t rc[16];
                    for (int n = 0; n < 16; n++) {
                        uint8_t* d = yd + (n >> 2) * 4 * BPS + (n & 3) * 4;
                        for (int k = 0; k < 16; k++) rc[k] = coeffs[n * 16 + k];
                        uint8_t blk[4 * BPS];  // reconstruct into a scratch copy: yd keeps the prediction for the 4x4 trial's borders
                        for (int j = 0; j < 4; j++)
                            for (int i = 0; i < 4; i++) blk[j * BPS + i] = d[j * BPS + i];
                        vp8::inverse_dct_add(rc, blk, BPS);
                        for (int j = 0; j < 4; j++)
                            for (int i = 0; i < 4; i++) y16[((n >> 2) * 4 + j) * 16 + (n & 3) * 4 + i] = blk[j * BPS + i];
                    }
                }
                uint32_t d16 = sse_block(sy, ys, y16, 16, 16), r16 = 0;
                {
                    int nz;
                    r16 += (uint32_t)cost_coeffs(1, 0, 0, lv + 24 * 16, &nz);
                    uint8_t tnz[4] = {0, 0, 0, 0}, lnz[4] = {0, 0, 0, 0};
                    for (int n = 0; n < 16; n++) {
                        r16 += (uint32_t)cost_coeffs(0, tnz[n & 3] + lnz[n >> 2], 1, lv + n * 16, &nz);
                        tnz[n & 3] = lnz[n >> 2] = (uint8_t)nz;
                    }
                    r16 += (uint32_t)bit_cost(1, 145) + 512;  // "not 4x4" + about two bits of 16x16 mode
                }
                // the 4x4 candidate in a copy of the work buffer (same borders)
                uint8_t yb4[vp8::YB_SIZE];
                for (int k = 0; k < vp8::YB_SIZE; k++) yb4[k] = yb[k];
                uint8_t* yd4 = yb4 + BPS + 8;
                // above-right samples: from the row above (the decoder's rule at the right edge and on the first row)
                for (int i = 16; i < 20; i++)
                    yd4[i - BPS] = mb_y > 0 ? (mb_x < P.mb_w - 1 ? py[i - ys] : py[15 - ys]) : 127;
                int16_t lv4[16 * 16];
                uint8_t m4[16], tm4[4], lm4[4];
                for (int i = 0; i < 4; i++) {
                    tm4[i] = top_modes[i];
                    lm4[i] = left_modes[i];
                }
                const int q = qm.y1[1];
                uint32_t r4 = (uint32_t)bit_cost(0, 145);
                const uint32_t d4 = analyse_i4(sy, ys, yd4, qm.y1, (3 * q * q) >> 7, tm4, lm4, lv4, m4, &r4);
                const uint64_t lam = (uint64_t)((q * q) >> 7);
                const uint64_t s16 = (uint64_t)d16 * 256 + (uint64_t)r16 * lam, s4 = (uint64_t)d4 * 256 + (uint64_t)r4 * lam;
                if (s4 < s16) {
                    use_i4 = true;
                    for (int k = 0; k < 16 * 16; k++) lv[k] = lv4[k];
                    for (int k = 0; k < 16; k++) lv[24 * 16 + k] = 0;
                    for (int j = 0; j < 16; j++)
                        for (int i = 0; i < 16; i++) yd[j * BPS + i] = yd4[j * BPS + i];
                    md[0] = (uint8_t)kI4;
                    for (int k = 0; k < 16; k++) md[2 + k] = m4[k];
                } else {
                    for (int j = 0; j < 16; j++)
                        for (int i = 0; i < 16; i++) yd[j * BPS + i] = y16[j * 16 + i];
                }
            }
            if (!use_i4) {
                md[0] = (uint8_t)ymode;
                for (int k = 0; k < 16; k++) md[2 + k] = (uint8_t)ymode;  // what the neighbours' sub-block modes are coded against
                if (!P.try_i4 || flat16)
                    for (int n = 0; n < 16; n++) vp8::inverse_dct_add(coeffs + n * 16, yd + (n >> 2) * 4 * BPS + (n & 3) * 4, BPS);
            }
            for (int n = 0; n < 4; n++) {
                fdct4x4(su + (n >> 1) * 4 * cs + (n & 1) * 4, cs, ud + (n >> 1) * 4 * BPS + (n & 1) * 4, BPS, coeffs + (16 + n) * 16);
                fdct4x4(sv + (n >> 1) * 4 * cs + (n & 1) * 4, cs, vd + (n >> 1) * 4 * BPS + (n & 1) * 4, BPS, coeffs + (20 + n) * 16);
                quantize_block(coeffs + (16 + n) * 16, lv + (16 + n) * 16, qm.uv, 0, 110, 115);
                quantize_block(coeffs + (20 + n) * 16, lv + (20 + n) * 16, qm.uv, 0, 110, 115);
            }
            // chroma reconstruction, exactly as the decoder will do it (luma: above)
            for (int n = 0; n < 4; n++) {
                vp8::inverse_dct_add(coeffs + (16 + n) * 16, ud + (n >> 1) * 4 * BPS + (n & 1) * 4, BPS);
                vp8::inverse_dct_add(coeffs + (20 + n) * 16, vd + (n >> 1) * 4 * BPS + (n & 1) * 4, BPS);
            }
            for (int j = 0; j < 16; j++)
                for (int i = 0; i < 16; i++) py[j * ys + i] = yd[j * BPS + i];
            for (int j = 0; j < 8; j++)
                for (int i = 0; i < 8; i++) {
                    pu[j * cs + i] = ud[j * BPS + i];
                    pv[j * cs + i] = vd[j * BPS + i];
                }
            md[1] = (uint8_t)uvmode;
            {
                uint32_t mask = 0;
                for (int k = 0; k < 25; k++) mask |= (uint32_t)block_nz(lv + k * 16, 0) << k;
                mb_set_nz_mask(md, mask);
            }
        }
}

// Pass 2: the bitstream.  VP8 lets the coefficient tokens of a frame travel in up to 8 PARTITIONS, macroblock row r in
// partition r mod n (RFC 6386 s.9.5), each with its own boolean coder -- the unit of parallelism of this pass: the
// device gives every partition, and the first partition (modes), a lane of its own.  The contexts a coder needs from
// the row above (which blocks had non-zero levels) are read from that row's levels, not carried from its coder, so
// the partitions really are independent.  The serial write_bitstream below runs the same pieces one after the other
// and is what the CPU tests and the oracle use: both produce the same bytes.

// 8 partitions when the frame has 8 macroblock rows, else the largest power of two that leaves none empty
LP_VP8_HD int log2_partitions(const Params& P) {
    int l = 0;
    while (l < 3 && (2 << l) <= P.mb_h) l++;
    return l;
}
LP_VP8_HD int partition_rows(const Params& P, int part, int nparts) { return (P.mb_h - part + nparts - 1) / nparts; }
// scratch region of a partition inside the token area (nmb * 2048 + 4096 bytes): 2 KiB per macroblock + slack
LP_VP8_HD size_t partition_scratch_off(const Params& P, int part, int nparts) {
    size_t rows_before = 0;
    for (int q = 0; q < part; q++) rows_before += (size_t)partition_rows(P, q, nparts);
    return rows_before * (size_t)P.mb_w * 2048 + (size_t)part * 64;
}
LP_VP8_HD size_t partition_scratch_cap(const Params& P, int part, int nparts) {
    return (size_t)partition_rows(P, part, nparts) * (size_t)P.mb_w * 2048 + 64;
}

// ---- scratch sizing: ONE rule for the device launcher (webp_encode.cu) and the host build (oracle_webp.cpp), so that
// the CPU tests run the encoder under exactly the device's limits.
// Token partitions: the layout above, 2 KiB per macroblock (the worst partition measured uses well under half of it).
LP_VP8_HD size_t token_scratch_bytes(const Params& P) { return (size_t)P.mb_w * P.mb_h * 2048 + 4096; }
// First partition: a worst-case bound, so that it never overflows below the format's limit.  A boolean moves at most
// log2(range / new range) < 8 bits out of the coder, the coder adds 4 bytes on flush.  Summed over the costliest path
// through the fixed probabilities (oracle_webp.cpp: vp8_cpu_part0_worst_bits computes it, the tests compare) the frame
// header takes at most 16723 bits and a macroblock at most 228 -- skip flag, sixteen sub-block modes in adversarial
// contexts, chroma mode (8 bits per boolean would say 1216).  The header term holds for the fields write_part0 codes
// today -- no segmentation, no loop-filter deltas, no quantiser deltas; a header that codes more needs a new bound (the
// test comparing it with vp8_cpu_part0_worst_bits fails first).  The partition's size is a 19-bit field of the frame
// tag: a first partition that outgrows kPart0Max bytes makes no valid stream whatever the scratch.
constexpr uint32_t kPart0HeaderBits = 16768, kPart0MbBits = 232;
constexpr size_t kPart0Max = (1u << 19) - 1;
LP_VP8_HD size_t part0_scratch_bytes(const Params& P) {
    const size_t bound = ((size_t)kPart0HeaderBits + (size_t)P.mb_w * P.mb_h * kPart0MbBits + 7) / 8 + 4 + 64;
    return bound < kPart0Max ? bound : kPart0Max;
}
// write_bitstream's result when the first partition did not fit part0_scratch_bytes, i.e. would exceed the format's
// limit: large frames of fine detail coded with 4x4 prediction (4096 x 4096 noise: ~9 bytes per macroblock, 64 K
// macroblocks).  The encoder's callers then code the frame once more with 16x16 prediction only (Params::try_i4 = 0,
// < 1 byte of modes per macroblock, the idea of libwebp's partition_limit); a frame that does not fit even so (noise
// near 16383 x 16383) stays refused.
constexpr size_t kPart0TooLarge = ~(size_t)0;

// aux accessors
LP_VP8_INL uint32_t* aux_stats(uint8_t* aux) { return reinterpret_cast<uint32_t*>(aux + kAuxStatsOff); }
LP_VP8_INL uint32_t* aux_counts(uint8_t* aux) { return reinterpret_cast<uint32_t*>(aux + kAuxCountsOff); }

// first partition: frame header (with the probability updates and the skip probability decided from the statistics
// in `aux`) + per-macroblock skip flag and modes.  Returns its size, 0 when it does not fit.
LP_VP8_FN size_t write_part0(const Params& P, const Buffers& B, const uint8_t* aux, uint8_t* part0, size_t part0_cap) {
    BoolEnc h;
    be_init(h, part0, part0_cap);
    be_put_bits(h, 0, 1);  // colour space
    be_put_bits(h, 0, 1);  // clamping type: clamping required
    be_put_bits(h, 0, 1);  // no segmentation
    be_put_bits(h, 0, 1);  // normal loop filter
    be_put_bits(h, (uint32_t)P.filter_level, 6);
    be_put_bits(h, 0, 3);  // sharpness
    be_put_bits(h, 0, 1);  // no loop-filter deltas
    be_put_bits(h, (uint32_t)log2_partitions(P), 2);
    be_put_bits(h, (uint32_t)P.q, 7);
    for (int i = 0; i < 5; i++) be_put_bits(h, 0, 1);  // no quantiser deltas
    be_put_bits(h, 0, 1);                               // refresh_entropy_probs
    {
        const uint8_t* upd = &kVp8CoeffUpdateProba[0][0][0][0];
        const uint8_t* proba = aux + kAuxProbaOff;
        const uint8_t* update = aux + kAuxUpdateOff;
        for (int i = 0; i < kNumProbas; i++) {
            be_put(h, update[i], upd[i]);
            if (update[i]) be_put_bits(h, proba[i], 8);
        }
    }
    const int use_skip = aux[kAuxSkipOff + 1], skip_p = aux[kAuxSkipOff];
    be_put_bits(h, (uint32_t)use_skip, 1);  // mb_no_coeff_skip
    if (use_skip) be_put_bits(h, (uint32_t)skip_p, 8);
    for (int i = 0; i < P.mb_w * P.mb_h; i++) {
        const uint8_t* md = B.modes + (size_t)i * kModeStride;
        const int ymode = md[0], uvmode = md[1];
        const int mb_x = i % P.mb_w, mb_y = i / P.mb_w;
        if (use_skip) be_put(h, mb_nz_mask(md) == 0, skip_p);
        if (ymode == kI4) {
            be_put(h, 0, 145);  // sixteen 4x4 modes, each coded against the modes above and to the left (s.8.3)
            for (int n = 0; n < 16; n++) {
                const int bx = n & 3, by = n >> 2;
                const int top = by > 0 ? md[2 + n - 4] : mb_y > 0 ? (md - (size_t)P.mb_w * kModeStride)[2 + 12 + bx] : (int)vp8::B_DC;
                const int left = bx > 0 ? md[2 + n - 1] : mb_x > 0 ? (md - kModeStride)[2 + 4 * by + 3] : (int)vp8::B_DC;
                i4_mode<true>(&h, md[2 + n], kVp8BModesProba[top][left]);
            }
        } else {
            be_put(h, 1, 145);  // one 16x16 mode
            if (ymode == vp8::TM_PRED || ymode == vp8::H_PRED) {
                be_put(h, 1, 156);
                be_put(h, ymode == vp8::TM_PRED, 128);
            } else {
                be_put(h, 0, 156);
                be_put(h, ymode == vp8::V_PRED, 163);
            }
        }
        if (uvmode == vp8::DC_PRED) {
            be_put(h, 0, 142);
        } else {
            be_put(h, 1, 142);
            if (uvmode == vp8::V_PRED) {
                be_put(h, 0, 114);
            } else {
                be_put(h, 1, 114);
                be_put(h, uvmode == vp8::TM_PRED, 183);
            }
        }
    }
    be_flush(h);
    return h.overflow ? 0 : h.pos;
}


// The macroblocks of token partition `part` (rows part, part + nparts, ...) in the decoder's order and contexts.
// CODE = false: count the adaptive branches into aux (the statistics the probabilities are decided from) and the
// skippable macroblocks; CODE = true: write the partition with the probabilities in aux.  A macroblock without any
// non-zero level has no tokens when the frame uses skip flags, and leaves "nothing non-zero" behind as context --
// which is what its levels say anyway, so the contexts need no special case.
template <bool CODE>
LP_VP8_FN size_t walk_partition(const Params& P, const Buffers& B, int part, int nparts, uint8_t* aux, uint8_t* buf, size_t cap) {
    BoolEnc t;
    if (CODE) be_init(t, buf, cap);
    const uint8_t* proba = aux + kAuxProbaOff;
    uint32_t* stats = aux_stats(aux);
    const int use_skip = CODE ? aux[kAuxSkipOff + 1] : 0;
    uint32_t n_mb = 0, n_skip = 0;
    for (int mb_y = part; mb_y < P.mb_h; mb_y += nparts) {
        uint8_t left_nz[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        for (int mb_x = 0; mb_x < P.mb_w; mb_x++) {
            const int16_t* lv = B.levels + ((size_t)mb_y * P.mb_w + mb_x) * 25 * 16;
            const uint8_t* md = B.modes + ((size_t)mb_y * P.mb_w + mb_x) * kModeStride;
            const uint32_t nzmask = mb_nz_mask(md);
            const bool i4 = md[0] == kI4;
            const int skippable = nzmask == 0;
            n_mb++;
            n_skip += (uint32_t)skippable;
            if (skippable && (use_skip || !CODE)) {
                // statistics pass: assume the frame WILL use skip flags when it has skippable macroblocks (decided
                // in finish_statistics from the same counts), so their would-be tokens are not counted
                for (int k = 0; k < 8; k++) left_nz[k] = 0;
                if (!i4) left_nz[8] = 0;
                continue;
            }
            uint8_t tnz[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            if (mb_y > 0) {  // bottom blocks of the macroblock above, from its mask
                const uint32_t up = mb_nz_mask(md - (size_t)P.mb_w * kModeStride);
                for (int i = 0; i < 4; i++) tnz[i] = (uint8_t)((up >> (12 + i)) & 1u);
                tnz[4] = (uint8_t)((up >> 18) & 1u);
                tnz[5] = (uint8_t)((up >> 19) & 1u);
                tnz[6] = (uint8_t)((up >> 22) & 1u);
                tnz[7] = (uint8_t)((up >> 23) & 1u);
                if (!i4) {
                    // the Y2 context above is that of the nearest macroblock above that HAS a Y2 block: 4x4 macroblocks
                    // neither read nor write it (s.13.3; the decoder carries it across them)
                    int r = mb_y - 1;
                    while (r >= 0 && B.modes[((size_t)r * P.mb_w + mb_x) * kModeStride] == kI4) r--;
                    tnz[8] = r >= 0 ? (uint8_t)((mb_nz_mask(B.modes + ((size_t)r * P.mb_w + mb_x) * kModeStride) >> 24) & 1u) : 0;
                }
            }
            for (int k = i4 ? 0 : -1; k < 24; k++) {  // [Y2], 16 Y, 4 U, 4 V: the decoder's order and contexts
                int type, ti, li, first = 0;
                const int16_t* blk;
                if (k < 0) {
                    type = 1; ti = 8; li = 8; blk = lv + 24 * 16;
                } else if (k < 16) {
                    type = i4 ? 3 : 0; ti = k & 3; li = k >> 2; blk = lv + k * 16; first = i4 ? 0 : 1;
                } else {
                    const int c = k - 16;
                    type = 2; ti = 4 + (c >> 2) * 2 + (c & 1); li = 4 + (c >> 2) * 2 + ((c >> 1) & 1); blk = lv + k * 16;
                }
                const int has = (int)((nzmask >> (k < 0 ? 24 : k)) & 1u);
                const int nz = CODE ? put_coeffs(t, proba, type, tnz[ti] + left_nz[li], first, blk, has)
                                    : record_coeffs(stats, type, tnz[ti] + left_nz[li], first, blk, has);
                tnz[ti] = left_nz[li] = (uint8_t)nz;
            }
        }
    }
    if (!CODE) {
#ifdef __CUDA_ARCH__
        atomicAdd(aux_counts(aux) + 0, n_mb);
        atomicAdd(aux_counts(aux) + 1, n_skip);
#else
        aux_counts(aux)[0] += n_mb;
        aux_counts(aux)[1] += n_skip;
#endif
        return 0;
    }
    be_flush(t);
    return t.overflow ? 0 : t.pos;
}

// The statistics are a SAMPLE: every second token partition, i.e. every second macroblock row (all rows when the frame
// has a single partition).  The probabilities are estimates either way; counting half the rows halves the cost of the
// statistics walk -- it is as long as the coding walk -- for well under 1 % of file size.
LP_VP8_HD int stats_partition(int part, int nparts) { return nparts < 2 || (part & 1) == 0; }

// entries [first, first + step, ...) of the probability table from the statistics; entry 0's caller also settles the
// skip probability.  (The device spreads the 1056 entries over the 32 lanes of the frame's warp.)
LP_VP8_FN void finish_statistics(uint8_t* aux, int first, int step) {
    const uint32_t* stats = aux_stats(aux);
    const uint8_t* def = &kVp8CoeffProba0[0][0][0][0];
    const uint8_t* upd = &kVp8CoeffUpdateProba[0][0][0][0];
    for (int i = first; i < kNumProbas; i += step)
        decide_proba(stats[2 * i], stats[2 * i + 1], def[i], upd[i], aux + kAuxProbaOff + i, aux + kAuxUpdateOff + i);
    if (first == 0) {
        const uint32_t n_mb = aux_counts(aux)[0], n_skip = aux_counts(aux)[1];
        // P(not skipped) in 1/256, as the decoder reads it; a flag per macroblock only pays when some are skipped
        int sp = n_mb ? (int)(((uint64_t)(n_mb - n_skip) * 255u) / n_mb) : 255;
        if (sp < 1) sp = 1;
        if (sp > 255) sp = 255;
        aux[kAuxSkipOff] = (uint8_t)sp;
        aux[kAuxSkipOff + 1] = n_skip > 0 ? 1 : 0;
    }
}

// frame tag + start code + dimensions + (behind the first partition) the partition size table.  `sizes[nparts]`.
// Returns the payload size, 0 when it does not fit; the caller copies part0 to out + 10 and the partitions to
// out + 10 + part0_len + 3 * (nparts - 1) + (sizes in front of it).
LP_VP8_FN size_t write_frame_header(const Params& P, size_t part0_len, const size_t* sizes, int nparts, uint8_t* out,
                                    size_t out_cap) {
    size_t total = 10 + part0_len + (size_t)3 * (nparts - 1);
    bool ok = part0_len != 0 && part0_len < (1u << 19);
    for (int i = 0; i < nparts; i++) {
        ok = ok && sizes[i] != 0 && sizes[i] < (1u << 24);
        total += sizes[i];
    }
    if (!ok || total > out_cap) return 0;
    const uint32_t tag = 0u | (0u << 1) | (1u << 4) | ((uint32_t)part0_len << 5);  // key frame, profile 0, shown
    out[0] = (uint8_t)tag;
    out[1] = (uint8_t)(tag >> 8);
    out[2] = (uint8_t)(tag >> 16);
    out[3] = 0x9d;
    out[4] = 0x01;
    out[5] = 0x2a;
    out[6] = (uint8_t)P.width;
    out[7] = (uint8_t)((P.width >> 8) & 0x3f);
    out[8] = (uint8_t)P.height;
    out[9] = (uint8_t)((P.height >> 8) & 0x3f);
    uint8_t* tab = out + 10 + part0_len;
    for (int i = 0; i + 1 < nparts; i++) {  // the last partition takes what is left
        tab[3 * i + 0] = (uint8_t)sizes[i];
        tab[3 * i + 1] = (uint8_t)(sizes[i] >> 8);
        tab[3 * i + 2] = (uint8_t)(sizes[i] >> 16);
    }
    return total;
}

// part0 / tokens / aux (kAuxBytes, 4-byte aligned) are scratch areas; `out` receives the "VP8 " chunk payload.  Returns
// the payload size, kPart0TooLarge when the first partition outgrew part0_cap, 0 when anything else does not fit.
LP_VP8_FN size_t write_bitstream(const Params& P, const Buffers& B, uint8_t* part0, size_t part0_cap, uint8_t* tokens,
                                 size_t tokens_cap, uint8_t* aux, uint8_t* out, size_t out_cap) {
    const int nparts = 1 << log2_partitions(P);
    if (partition_scratch_off(P, nparts - 1, nparts) + partition_scratch_cap(P, nparts - 1, nparts) > tokens_cap) return 0;
    for (size_t i = 0; i < kAuxBytes; i++) aux[i] = 0;
    for (int q = 0; q < nparts; q++)
        if (stats_partition(q, nparts)) walk_partition<false>(P, B, q, nparts, aux, nullptr, 0);
    finish_statistics(aux, 0, 1);
    const size_t part0_len = write_part0(P, B, aux, part0, part0_cap);
    if (!part0_len) return kPart0TooLarge;
    size_t sizes[8];
    for (int q = 0; q < nparts; q++)
        sizes[q] = walk_partition<true>(P, B, q, nparts, aux, tokens + partition_scratch_off(P, q, nparts), partition_scratch_cap(P, q, nparts));
    const size_t total = write_frame_header(P, part0_len, sizes, nparts, out, out_cap);
    if (!total) return 0;
    for (size_t i = 0; i < part0_len; i++) out[10 + i] = part0[i];
    size_t at = 10 + part0_len + (size_t)3 * (nparts - 1);
    for (int q = 0; q < nparts; q++) {
        const uint8_t* src = tokens + partition_scratch_off(P, q, nparts);
        for (size_t i = 0; i < sizes[q]; i++) out[at + i] = src[i];
        at += sizes[q];
    }
    return total;
}

}  // namespace vp8enc
