// vp8_core.h -- VP8 key-frame (WebP lossy) decoding, written against the VP8 data format
// (RFC 6386) with the output conventions of libwebp's simple API, which is what
// webp_decoder_decode calls (ref webp.cpp:336-351: WebPDecodeBGRInto / WebPDecodeBGRAInto with
// default options = in-loop filter as coded, "fancy" chroma upsampling, no dithering).
//
// libwebp 1.x is a vendored BINARY in the reference (deps/linux/amd64/lib/libwebp.a); nothing
// here is taken from it except the normative constant tables in vp8_tables.h (see the generator).
// Parity is pinned on the reference's decoder itself through oracle/_ref (tests/test_webp_core.py)
// and on golden frames made by it (tests/golden).
//
// The same functions compile for the device (webp_decode.cu, LP_VP8_FN = __device__) and for the
// CPU test harness (oracle/oracle_webp.cpp).  Layout of one frame's working set:
//   y / u / v planes      mb_w*16 x mb_h*16 (and half size), reconstructed then filtered in place
//   top_modes[mb_w*4]     sub-block modes of the row above (mode context, RFC 6386 s.11.3)
//   top_nz[mb_w*9]        non-zero flags of the row above: 4 Y, 2 U, 2 V, 1 Y2 (s.13.3)
//   finfo[mb_w*mb_h]      per-macroblock loop-filter parameters (s.15.2), packed
#pragma once
#include <stdint.h>
#include <stddef.h>

#include "vp8_tables.h"

#ifndef LP_VP8_FN
#define LP_VP8_FN static inline
#endif
#ifndef LP_VP8_INL  // small primitives that must stay in registers
#define LP_VP8_INL LP_VP8_FN
#endif
#ifndef LP_VP8_HD  // the two layout helpers are also called by the host launcher
#define LP_VP8_HD LP_VP8_FN
#endif

namespace vp8 {

enum { B_DC = 0, B_TM, B_VE, B_HE, B_RD, B_VR, B_LD, B_VL, B_HD, B_HU };  // libwebp's enum order
enum { DC_PRED = B_DC, TM_PRED = B_TM, V_PRED = B_VE, H_PRED = B_HE };

// ---- boolean entropy decoder (RFC 6386 s.7) ------------------------------------------------
struct BoolDec {
    const uint8_t* p;
    const uint8_t* end;
    uint64_t value;
    uint32_t range;  // range - 1, kept in [127, 254]
    int bits;        // number of bits in `value` below the 8-bit compare window
    int eof;         // a refill found no byte left: the partition is truncated (libwebp's eof_)
};

LP_VP8_INL int clz32(uint32_t v) {
#ifdef __CUDA_ARCH__
    return __clz((int)v);
#else
    return __builtin_clz(v);
#endif
}

LP_VP8_INL void bd_init(BoolDec& b, const uint8_t* p, size_t n) {
    b.p = p;
    b.end = p + n;
    b.value = 0;
    b.range = 254;
    b.bits = -8;
    b.eof = n == 0;  // libwebp loads on init: an empty partition is already past its end
}

LP_VP8_INL void bd_fill(BoolDec& b) {
#ifdef __CUDA_ARCH__
    // device: 4 bytes per refill from two aligned word loads (the refill is on every symbol's critical path)
    if (b.p + 4 <= b.end) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(b.p);
        const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
        const uint32_t le = __funnelshift_r(q[0], q[1], 8 * (int)(a & 3));  // q[1]: inside the padded buffer
        b.p += 4;
        b.value = (b.value << 32) | __byte_perm(le, 0, 0x0123);
        b.bits += 32;
    } else {
#else
    // take up to 6 bytes per refill
    if (b.p + 6 <= b.end) {
        uint64_t w = 0;
        for (int i = 0; i < 6; i++) w = (w << 8) | b.p[i];
        b.p += 6;
        b.value = (b.value << 48) | w;
        b.bits += 48;
    } else {
#endif
        uint32_t byte = 0;  // zeros past the end, as libwebp feeds
        if (b.p < b.end) byte = *b.p++;
        else b.eof = 1;
        b.value = (b.value << 8) | byte;
        b.bits += 8;
    }
}

LP_VP8_INL int bd_bit(BoolDec& b, int prob) {
    if (b.bits < 0) bd_fill(b);
    uint32_t range = b.range;
    const uint32_t split = (range * (uint32_t)prob) >> 8;
    const uint32_t v = (uint32_t)(b.value >> b.bits);
    int bit;
    if (v > split) {
        range -= split;
        b.value -= (uint64_t)(split + 1) << b.bits;
        bit = 1;
    } else {
        range = split + 1;
        bit = 0;
    }
    const int shift = clz32(range) - 24;  // range in [1, 255]
    b.bits -= shift;
    b.range = (range << shift) - 1;
    return bit;
}

LP_VP8_FN uint32_t bd_value(BoolDec& b, int nbits) {
    uint32_t v = 0;
    while (nbits-- > 0) v |= (uint32_t)bd_bit(b, 0x80) << nbits;
    return v;
}
LP_VP8_FN int bd_signed(BoolDec& b, int nbits) {
    const int v = (int)bd_value(b, nbits);
    return bd_bit(b, 0x80) ? -v : v;
}

// ---- frame header (RFC 6386 s.9, s.19.2) ---------------------------------------------------
struct QuantMat {
    int y1[2], y2[2], uv[2];
};
struct FilterStrength {  // s.15.2: limits derived from level / sharpness
    uint8_t limit, ilevel, hev, inner;
};
struct FrameHdr {
    int width, height, mb_w, mb_h;
    int use_segment, update_map;
    uint8_t seg_proba[3];
    int filter_type;  // 0 off, 1 simple, 2 normal
    int num_parts;
    int use_skip, skip_p;
    QuantMat q[4];
    FilterStrength fs[4][2];
    uint32_t part_off[8], part_len[8];  // token partitions, offsets from the start of the VP8 payload
};

enum { VP8_OK = 0, VP8_BAD = 1 };

LP_VP8_FN int clipq(int v, int hi) { return v < 0 ? 0 : v > hi ? hi : v; }

// Parses the frame tag and the first-partition header.  `br` is left positioned on the first
// macroblock's mode bits.  `proba` receives the coefficient probabilities (s.13.4).
LP_VP8_FN int parse_frame_header(const uint8_t* data, size_t size, FrameHdr& h, BoolDec& br,
                                 uint8_t* proba /*[4*8*3*11]*/) {
    if (size < 10) return VP8_BAD;
    const uint32_t tag = data[0] | (data[1] << 8) | ((uint32_t)data[2] << 16);
    if (tag & 1) return VP8_BAD;                 // not a key frame
    if (((tag >> 1) & 7) > 3) return VP8_BAD;    // unknown profile
    if (!((tag >> 4) & 1)) return VP8_BAD;       // frame not shown
    const uint32_t part0_len = tag >> 5;
    if (data[3] != 0x9d || data[4] != 0x01 || data[5] != 0x2a) return VP8_BAD;
    h.width = ((data[7] << 8) | data[6]) & 0x3fff;
    h.height = ((data[9] << 8) | data[8]) & 0x3fff;
    if (!h.width || !h.height) return VP8_BAD;
    h.mb_w = (h.width + 15) >> 4;
    h.mb_h = (h.height + 15) >> 4;
    if ((size_t)10 + part0_len > size) return VP8_BAD;
    bd_init(br, data + 10, part0_len);

    bd_value(br, 1);  // colour space
    bd_value(br, 1);  // clamping type
    // segmentation (s.9.3)
    int seg_abs = 1, seg_q[4] = {0, 0, 0, 0}, seg_f[4] = {0, 0, 0, 0};
    h.seg_proba[0] = h.seg_proba[1] = h.seg_proba[2] = 255;
    h.use_segment = (int)bd_value(br, 1);
    h.update_map = 0;
    if (h.use_segment) {
        h.update_map = (int)bd_value(br, 1);
        if (bd_value(br, 1)) {
            seg_abs = (int)bd_value(br, 1);
            for (int s = 0; s < 4; s++) seg_q[s] = bd_value(br, 1) ? bd_signed(br, 7) : 0;
            for (int s = 0; s < 4; s++) seg_f[s] = bd_value(br, 1) ? bd_signed(br, 6) : 0;
        }
        if (h.update_map)
            for (int s = 0; s < 3; s++) h.seg_proba[s] = bd_value(br, 1) ? (uint8_t)bd_value(br, 8) : 255;
    }
    // loop filter (s.9.6)
    const int simple = (int)bd_value(br, 1);
    const int level = (int)bd_value(br, 6);
    const int sharp = (int)bd_value(br, 3);
    const int use_lf_delta = (int)bd_value(br, 1);
    int ref_delta[4] = {0, 0, 0, 0}, mode_delta[4] = {0, 0, 0, 0};
    if (use_lf_delta && bd_value(br, 1)) {
        for (int i = 0; i < 4; i++)
            if (bd_value(br, 1)) ref_delta[i] = bd_signed(br, 6);
        for (int i = 0; i < 4; i++)
            if (bd_value(br, 1)) mode_delta[i] = bd_signed(br, 6);
    }
    h.filter_type = level == 0 ? 0 : simple ? 1 : 2;
    // token partitions (s.9.5)
    h.num_parts = 1 << bd_value(br, 2);
    {
        const size_t base = (size_t)10 + part0_len;
        const size_t sz_bytes = (size_t)3 * (h.num_parts - 1);
        if (base + sz_bytes > size) return VP8_BAD;
        size_t off = base + sz_bytes, left = size - off;
        for (int p = 0; p < h.num_parts - 1; p++) {
            const uint8_t* s = data + base + 3 * p;
            size_t n = s[0] | (s[1] << 8) | ((size_t)s[2] << 16);
            if (n > left) n = left;
            h.part_off[p] = (uint32_t)off;
            h.part_len[p] = (uint32_t)n;
            off += n;
            left -= n;
        }
        h.part_off[h.num_parts - 1] = (uint32_t)off;
        h.part_len[h.num_parts - 1] = (uint32_t)left;
        if (!left) return VP8_BAD;  // the last partition must start inside the data (libwebp's ParsePartitions)
    }
    // quantizer indices (s.9.6, s.14.1)
    {
        const int base_q0 = (int)bd_value(br, 7);
        const int dqy1_dc = bd_value(br, 1) ? bd_signed(br, 4) : 0;
        const int dqy2_dc = bd_value(br, 1) ? bd_signed(br, 4) : 0;
        const int dqy2_ac = bd_value(br, 1) ? bd_signed(br, 4) : 0;
        const int dquv_dc = bd_value(br, 1) ? bd_signed(br, 4) : 0;
        const int dquv_ac = bd_value(br, 1) ? bd_signed(br, 4) : 0;
        for (int s = 0; s < 4; s++) {
            int q;
            if (h.use_segment) {
                q = seg_q[s];
                if (!seg_abs) q += base_q0;
            } else {
                q = base_q0;
            }
            QuantMat& m = h.q[s];
            m.y1[0] = kVp8DcTable[clipq(q + dqy1_dc, 127)];
            m.y1[1] = kVp8AcTable[clipq(q, 127)];
            m.y2[0] = kVp8DcTable[clipq(q + dqy2_dc, 127)] * 2;
            m.y2[1] = (kVp8AcTable[clipq(q + dqy2_ac, 127)] * 101581) >> 16;  // x155/100
            if (m.y2[1] < 8) m.y2[1] = 8;
            m.uv[0] = kVp8DcTable[clipq(q + dquv_dc, 117)];
            m.uv[1] = kVp8AcTable[clipq(q + dquv_ac, 127)];
        }
    }
    // per-segment filter strengths (s.15.2 + s.9.3 / s.9.6 deltas; intra frame => ref delta 0)
    for (int s = 0; s < 4; s++) {
        int base = level;
        if (h.use_segment) {
            base = seg_f[s];
            if (!seg_abs) base += level;
        }
        for (int i4 = 0; i4 <= 1; i4++) {
            FilterStrength& f = h.fs[s][i4];
            int lv = base;
            if (use_lf_delta) {
                lv += ref_delta[0];
                if (i4) lv += mode_delta[0];
            }
            lv = lv < 0 ? 0 : lv > 63 ? 63 : lv;
            if (lv > 0 && h.filter_type > 0) {
                int il = lv;
                if (sharp > 0) {
                    il >>= (sharp > 4) ? 2 : 1;
                    if (il > 9 - sharp) il = 9 - sharp;
                }
                if (il < 1) il = 1;
                f.ilevel = (uint8_t)il;
                f.limit = (uint8_t)(2 * lv + il);
                f.hev = (uint8_t)((lv >= 40) ? 2 : (lv >= 15) ? 1 : 0);
            } else {
                f.limit = 0;
                f.ilevel = 0;
                f.hev = 0;
            }
            f.inner = (uint8_t)i4;
        }
    }
    bd_value(br, 1);  // refresh_entropy_probs: irrelevant for a single key frame
    // coefficient probabilities (s.13.4)
    {
        const uint8_t* upd = &kVp8CoeffUpdateProba[0][0][0][0];
        const uint8_t* def = &kVp8CoeffProba0[0][0][0][0];
        for (int i = 0; i < 4 * 8 * 3 * 11; i++) proba[i] = bd_bit(br, upd[i]) ? (uint8_t)bd_value(br, 8) : def[i];
    }
    h.use_skip = (int)bd_value(br, 1);
    h.skip_p = h.use_skip ? (int)bd_value(br, 8) : 0;
    return VP8_OK;
}

// ---- residual tokens (RFC 6386 s.13) -------------------------------------------------------
LP_VP8_FN int get_large_value(BoolDec& br, const uint8_t* p) {
    int v;
    if (!bd_bit(br, p[3])) {
        if (!bd_bit(br, p[4])) v = 2;
        else v = 3 + bd_bit(br, p[5]);
    } else {
        if (!bd_bit(br, p[6])) {
            if (!bd_bit(br, p[7])) {
                v = 5 + bd_bit(br, 159);
            } else {
                v = 7 + 2 * bd_bit(br, 165);
                v += bd_bit(br, 145);
            }
        } else {
            const int bit1 = bd_bit(br, p[8]);
            const int bit0 = bd_bit(br, p[9 + bit1]);
            const int cat = 2 * bit1 + bit0;
            v = 0;
            // extra-bit probabilities of DCT categories 3..6 (s.13.2)
            if (cat == 0) {
                v = bd_bit(br, 173);
                v += v + bd_bit(br, 148);
                v += v + bd_bit(br, 140);
            } else if (cat == 1) {
                v = bd_bit(br, 176);
                v += v + bd_bit(br, 155);
                v += v + bd_bit(br, 140);
                v += v + bd_bit(br, 135);
            } else if (cat == 2) {
                v = bd_bit(br, 180);
                v += v + bd_bit(br, 157);
                v += v + bd_bit(br, 141);
                v += v + bd_bit(br, 134);
                v += v + bd_bit(br, 130);
            } else {
                const uint8_t c6[11] = {254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129};
                for (int i = 0; i < 11; i++) v += v + bd_bit(br, c6[i]);
            }
            v += 3 + (8 << cat);
        }
    }
    return v;
}

// Reads one 4x4 block's tokens; `type` selects the probability plane, `ctx` the neighbour
// context, `first` is 1 for luma blocks whose DC travels in Y2.  Dequantised coefficients go to
// out[] in raster order.  Returns the position after the last decoded token.
LP_VP8_FN int get_coeffs(BoolDec& br, const uint8_t* proba, int type, int ctx, const int* dq, int first,
                         int16_t* out) {
    const uint8_t bands[17] = {0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0};
    const uint8_t zigzag[16] = {0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15};
    const uint8_t* tp = proba + type * (8 * 3 * 11);
    int n = first;
    const uint8_t* p = tp + (bands[n] * 3 + ctx) * 11;
    for (; n < 16; ++n) {
        if (!bd_bit(br, p[0])) return n;  // end of block
        while (!bd_bit(br, p[1])) {       // run of zeros
            p = tp + (bands[++n] * 3 + 0) * 11;
            if (n == 16) return 16;
        }
        int v;
        const uint8_t* pn = tp + bands[n + 1] * 3 * 11;
        if (!bd_bit(br, p[2])) {
            v = 1;
            p = pn + 1 * 11;
        } else {
            v = get_large_value(br, p);
            p = pn + 2 * 11;
        }
        const int sv = bd_bit(br, 0x80) ? -v : v;
        out[zigzag[n]] = (int16_t)(sv * dq[n > 0]);
    }
    return 16;
}

// ---- inverse transforms (RFC 6386 s.14.3, s.14.4) ------------------------------------------
LP_VP8_FN void inverse_wht(const int16_t* in, int16_t* dst /* stride 16 */) {
    int tmp[16];
    for (int i = 0; i < 4; i++) {
        const int a0 = in[0 + i] + in[12 + i];
        const int a1 = in[4 + i] + in[8 + i];
        const int a2 = in[4 + i] - in[8 + i];
        const int a3 = in[0 + i] - in[12 + i];
        tmp[0 + i] = a0 + a1;
        tmp[8 + i] = a0 - a1;
        tmp[4 + i] = a3 + a2;
        tmp[12 + i] = a3 - a2;
    }
    for (int i = 0; i < 4; i++) {
        const int dc = tmp[0 + i * 4] + 3;
        const int a0 = dc + tmp[3 + i * 4];
        const int a1 = tmp[1 + i * 4] + tmp[2 + i * 4];
        const int a2 = tmp[1 + i * 4] - tmp[2 + i * 4];
        const int a3 = dc - tmp[3 + i * 4];
        dst[0] = (int16_t)((a0 + a1) >> 3);
        dst[16] = (int16_t)((a3 + a2) >> 3);
        dst[32] = (int16_t)((a0 - a1) >> 3);
        dst[48] = (int16_t)((a3 - a2) >> 3);
        dst += 64;
    }
}

LP_VP8_INL uint8_t clip8(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }
LP_VP8_INL int mul1(int a) { return ((a * 20091) >> 16) + a; }
LP_VP8_INL int mul2(int a) { return (a * 35468) >> 16; }

// dst += IDCT(in), clipped; dst is a stride-`bps` pixel block.  Evaluated in int: libwebp's TransformAC3 /
// TransformDC (blocks whose tokens stop before zigzag position 3) and its C transform.
LP_VP8_FN void inverse_dct_add(const int16_t* in, uint8_t* dst, int bps) {
    int tmp[16];
    for (int i = 0; i < 4; i++) {  // vertical pass
        const int a = in[i] + in[8 + i];
        const int b = in[i] - in[8 + i];
        const int c = mul2(in[4 + i]) - mul1(in[12 + i]);
        const int d = mul1(in[4 + i]) + mul2(in[12 + i]);
        tmp[4 * i + 0] = a + d;
        tmp[4 * i + 1] = b + c;
        tmp[4 * i + 2] = b - c;
        tmp[4 * i + 3] = a - d;
    }
    for (int i = 0; i < 4; i++) {  // horizontal pass
        const int dc = tmp[i] + 4;
        const int a = dc + tmp[8 + i];
        const int b = dc - tmp[8 + i];
        const int c = mul2(tmp[4 + i]) - mul1(tmp[12 + i]);
        const int d = mul1(tmp[4 + i]) + mul2(tmp[12 + i]);
        uint8_t* r = dst + i * bps;
        r[0] = clip8(r[0] + ((a + d) >> 3));
        r[1] = clip8(r[1] + ((b + c) >> 3));
        r[2] = clip8(r[2] + ((b - c) >> 3));
        r[3] = clip8(r[3] + ((a - d) >> 3));
    }
}

// The same transform as libwebp's x86 build runs it on blocks with a token past zigzag position 2
// (Transform_SSE2): 16-bit lanes throughout, wrapping adds, mulhi by 20091 and 35468 - 65536 plus the
// input, an arithmetic >> 3.  Equal to inverse_dct_add while no intermediate leaves int16, which holds for
// every coefficient within +-2048; crafted streams reach the whole int16 range.
LP_VP8_INL int wrap16(int v) { return (int16_t)v; }
LP_VP8_INL int mulhi16(int a, int k) { return (a * k) >> 16; }
LP_VP8_FN void inverse_dct_add16(const int16_t* in, uint8_t* dst, int bps) {
    const int k1 = 20091, k2 = 35468 - 65536;
    int tmp[16];
    for (int i = 0; i < 4; i++) {  // vertical pass
        const int i0 = in[i], i1 = in[4 + i], i2 = in[8 + i], i3 = in[12 + i];
        const int a = i0 + i2;
        const int b = i0 - i2;
        const int c = i1 - i3 + mulhi16(i1, k2) - mulhi16(i3, k1);
        const int d = i1 + i3 + mulhi16(i1, k1) + mulhi16(i3, k2);
        tmp[4 * i + 0] = wrap16(a + d);
        tmp[4 * i + 1] = wrap16(b + c);
        tmp[4 * i + 2] = wrap16(b - c);
        tmp[4 * i + 3] = wrap16(a - d);
    }
    for (int i = 0; i < 4; i++) {  // horizontal pass
        const int t0 = tmp[i], t1 = tmp[4 + i], t2 = tmp[8 + i], t3 = tmp[12 + i];
        const int a = t0 + 4 + t2;
        const int b = t0 + 4 - t2;
        const int c = t1 - t3 + mulhi16(t1, k2) - mulhi16(t3, k1);
        const int d = t1 + t3 + mulhi16(t1, k1) + mulhi16(t3, k2);
        uint8_t* r = dst + i * bps;
        r[0] = clip8(r[0] + (wrap16(a + d) >> 3));
        r[1] = clip8(r[1] + (wrap16(b + c) >> 3));
        r[2] = clip8(r[2] + (wrap16(b - c) >> 3));
        r[3] = clip8(r[3] + (wrap16(a - d) >> 3));
    }
}

// Per-block inverse transform classes (libwebp's NzCodeBits / DoTransform): 2 bits per block.
enum { TR_NONE = 0, TR_DC = 1, TR_AC3 = 2, TR_FULL = 3 };
LP_VP8_FN void transform_add(int cls, const int16_t* in, uint8_t* dst, int bps) {
    if (cls == TR_FULL) inverse_dct_add16(in, dst, bps);
    else if (cls != TR_NONE) inverse_dct_add(in, dst, bps);
}
// Chroma block n (0..3 U, 4..7 V) of `tr_uv`: when any block of its plane has AC (class AC3 or FULL), all four
// take the full transform (libwebp's DoUVTransform / TransformUV), else each its DC.
LP_VP8_INL int uv_transform(uint32_t tr_uv, int n) {
    const uint32_t plane = (tr_uv >> (n & 4 ? 8 : 0)) & 0xff;
    if (!((tr_uv >> 2 * n) & 3)) return TR_NONE;
    return (plane & 0xaa) ? TR_FULL : TR_DC;
}

// ---- intra prediction (RFC 6386 s.12) ------------------------------------------------------
// All predictors read the row above (dst - bps) and the column to the left (dst - 1) of a work
// buffer whose borders the caller has filled (127 above the first row, 129 left of the first
// column, s.12.2).
#define LP_AVG3(a, b, c) ((uint8_t)(((a) + 2 * (b) + (c) + 2) >> 2))
#define LP_AVG2(a, b) ((uint8_t)(((a) + (b) + 1) >> 1))

LP_VP8_FN void pred_tm(uint8_t* dst, int bps, int size) {
    const uint8_t* top = dst - bps;
    const int tl = top[-1];
    for (int y = 0; y < size; y++) {
        const int l = dst[y * bps - 1] - tl;
        for (int x = 0; x < size; x++) dst[y * bps + x] = clip8(top[x] + l);
    }
}
LP_VP8_FN void pred_fill(uint8_t* dst, int bps, int size, int v) {
    for (int y = 0; y < size; y++)
        for (int x = 0; x < size; x++) dst[y * bps + x] = (uint8_t)v;
}
// 16x16 and 8x8: mode with the edge-aware DC variants (have_top / have_left).
LP_VP8_FN void pred_block(uint8_t* dst, int bps, int size, int mode, int have_top, int have_left) {
    const int sh = size == 16 ? 4 : 3;  // log2(size)
    if (mode == DC_PRED) {
        int dc;
        if (have_top && have_left) {
            int s = 0;
            for (int i = 0; i < size; i++) s += dst[i - bps] + dst[i * bps - 1];
            dc = (s + size) >> (sh + 1);
        } else if (have_top || have_left) {
            int s = 0;
            for (int i = 0; i < size; i++) s += have_top ? dst[i - bps] : dst[i * bps - 1];
            dc = (s + (size >> 1)) >> sh;
        } else {
            dc = 0x80;
        }
        pred_fill(dst, bps, size, dc);
    } else if (mode == TM_PRED) {
        pred_tm(dst, bps, size);
    } else if (mode == V_PRED) {
        for (int y = 0; y < size; y++)
            for (int x = 0; x < size; x++) dst[y * bps + x] = dst[x - bps];
    } else {  // H_PRED
        for (int y = 0; y < size; y++) {
            const uint8_t l = dst[y * bps - 1];
            for (int x = 0; x < size; x++) dst[y * bps + x] = l;
        }
    }
}

#define LP_DST(x, y) dst[(x) + (y) * bps]
LP_VP8_FN void pred_4x4(uint8_t* dst, int bps, int mode) {
    const uint8_t* top = dst - bps;
    const int X = top[-1];
    const int A = top[0], B = top[1], C = top[2], D = top[3];
    const int E = top[4], F = top[5], G = top[6], H = top[7];
    const int I = dst[-1], J = dst[bps - 1], K = dst[2 * bps - 1], L = dst[3 * bps - 1];
    switch (mode) {
        case B_DC: {
            const int dc = (A + B + C + D + I + J + K + L + 4) >> 3;
            pred_fill(dst, bps, 4, dc);
            break;
        }
        case B_TM: pred_tm(dst, bps, 4); break;
        case B_VE: {
            const uint8_t v0 = LP_AVG3(X, A, B), v1 = LP_AVG3(A, B, C), v2 = LP_AVG3(B, C, D), v3 = LP_AVG3(C, D, E);
            for (int y = 0; y < 4; y++) {
                LP_DST(0, y) = v0;
                LP_DST(1, y) = v1;
                LP_DST(2, y) = v2;
                LP_DST(3, y) = v3;
            }
            break;
        }
        case B_HE: {
            const uint8_t h0 = LP_AVG3(X, I, J), h1 = LP_AVG3(I, J, K), h2 = LP_AVG3(J, K, L), h3 = LP_AVG3(K, L, L);
            for (int x = 0; x < 4; x++) {
                LP_DST(x, 0) = h0;
                LP_DST(x, 1) = h1;
                LP_DST(x, 2) = h2;
                LP_DST(x, 3) = h3;
            }
            break;
        }
        case B_LD:
            LP_DST(0, 0) = LP_AVG3(A, B, C);
            LP_DST(1, 0) = LP_DST(0, 1) = LP_AVG3(B, C, D);
            LP_DST(2, 0) = LP_DST(1, 1) = LP_DST(0, 2) = LP_AVG3(C, D, E);
            LP_DST(3, 0) = LP_DST(2, 1) = LP_DST(1, 2) = LP_DST(0, 3) = LP_AVG3(D, E, F);
            LP_DST(3, 1) = LP_DST(2, 2) = LP_DST(1, 3) = LP_AVG3(E, F, G);
            LP_DST(3, 2) = LP_DST(2, 3) = LP_AVG3(F, G, H);
            LP_DST(3, 3) = LP_AVG3(G, H, H);
            break;
        case B_RD:
            LP_DST(0, 3) = LP_AVG3(J, K, L);
            LP_DST(1, 3) = LP_DST(0, 2) = LP_AVG3(I, J, K);
            LP_DST(2, 3) = LP_DST(1, 2) = LP_DST(0, 1) = LP_AVG3(X, I, J);
            LP_DST(3, 3) = LP_DST(2, 2) = LP_DST(1, 1) = LP_DST(0, 0) = LP_AVG3(A, X, I);
            LP_DST(3, 2) = LP_DST(2, 1) = LP_DST(1, 0) = LP_AVG3(B, A, X);
            LP_DST(3, 1) = LP_DST(2, 0) = LP_AVG3(C, B, A);
            LP_DST(3, 0) = LP_AVG3(D, C, B);
            break;
        case B_VR:
            LP_DST(0, 0) = LP_DST(1, 2) = LP_AVG2(X, A);
            LP_DST(1, 0) = LP_DST(2, 2) = LP_AVG2(A, B);
            LP_DST(2, 0) = LP_DST(3, 2) = LP_AVG2(B, C);
            LP_DST(3, 0) = LP_AVG2(C, D);
            LP_DST(0, 3) = LP_AVG3(K, J, I);
            LP_DST(0, 2) = LP_AVG3(J, I, X);
            LP_DST(0, 1) = LP_DST(1, 3) = LP_AVG3(I, X, A);
            LP_DST(1, 1) = LP_DST(2, 3) = LP_AVG3(X, A, B);
            LP_DST(2, 1) = LP_DST(3, 3) = LP_AVG3(A, B, C);
            LP_DST(3, 1) = LP_AVG3(B, C, D);
            break;
        case B_VL:
            LP_DST(0, 0) = LP_AVG2(A, B);
            LP_DST(1, 0) = LP_DST(0, 2) = LP_AVG2(B, C);
            LP_DST(2, 0) = LP_DST(1, 2) = LP_AVG2(C, D);
            LP_DST(3, 0) = LP_DST(2, 2) = LP_AVG2(D, E);
            LP_DST(0, 1) = LP_AVG3(A, B, C);
            LP_DST(1, 1) = LP_DST(0, 3) = LP_AVG3(B, C, D);
            LP_DST(2, 1) = LP_DST(1, 3) = LP_AVG3(C, D, E);
            LP_DST(3, 1) = LP_DST(2, 3) = LP_AVG3(D, E, F);
            LP_DST(3, 2) = LP_AVG3(E, F, G);
            LP_DST(3, 3) = LP_AVG3(F, G, H);
            break;
        case B_HD:
            LP_DST(0, 0) = LP_DST(2, 1) = LP_AVG2(I, X);
            LP_DST(0, 1) = LP_DST(2, 2) = LP_AVG2(J, I);
            LP_DST(0, 2) = LP_DST(2, 3) = LP_AVG2(K, J);
            LP_DST(0, 3) = LP_AVG2(L, K);
            LP_DST(3, 0) = LP_AVG3(A, B, C);
            LP_DST(2, 0) = LP_AVG3(X, A, B);
            LP_DST(1, 0) = LP_DST(3, 1) = LP_AVG3(I, X, A);
            LP_DST(1, 1) = LP_DST(3, 2) = LP_AVG3(J, I, X);
            LP_DST(1, 2) = LP_DST(3, 3) = LP_AVG3(K, J, I);
            LP_DST(1, 3) = LP_AVG3(L, K, J);
            break;
        default:  // B_HU
            LP_DST(0, 0) = LP_AVG2(I, J);
            LP_DST(2, 0) = LP_DST(0, 1) = LP_AVG2(J, K);
            LP_DST(2, 1) = LP_DST(0, 2) = LP_AVG2(K, L);
            LP_DST(1, 0) = LP_AVG3(I, J, K);
            LP_DST(3, 0) = LP_DST(1, 1) = LP_AVG3(J, K, L);
            LP_DST(3, 1) = LP_DST(1, 2) = LP_AVG3(K, L, L);
            LP_DST(3, 2) = LP_DST(2, 2) = LP_DST(0, 3) = LP_DST(1, 3) = LP_DST(2, 3) = LP_DST(3, 3) = (uint8_t)L;
            break;
    }
}
#undef LP_DST

// ---- per-frame working set -----------------------------------------------------------------
struct Work {
    uint8_t *y, *u, *v;   // planes, strides mb_w*16 / mb_w*8
    uint8_t* top_modes;   // mb_w*4
    uint8_t* top_nz;      // mb_w*9
    uint32_t* finfo;      // mb_w*mb_h : limit | ilevel<<8 | hev<<16 | inner<<24
    uint8_t* proba;       // 1056
};
LP_VP8_HD size_t work_bytes(int mb_w, int mb_h) {
    const size_t ypl = (size_t)mb_w * 16 * mb_h * 16;
    size_t n = ypl + ypl / 2;                  // y, u, v
    n += (size_t)mb_w * 4 + (size_t)mb_w * 9;  // contexts
    n = (n + 3) & ~(size_t)3;
    n += (size_t)mb_w * mb_h * 4;              // finfo
    n += 1056;
    return (n + 255) & ~(size_t)255;
}
LP_VP8_HD void work_carve(uint8_t* base, int mb_w, int mb_h, Work& w) {
    const size_t ypl = (size_t)mb_w * 16 * mb_h * 16;
    w.y = base;
    w.u = w.y + ypl;
    w.v = w.u + ypl / 4;
    w.top_modes = w.v + ypl / 4;
    w.top_nz = w.top_modes + (size_t)mb_w * 4;
    size_t off = ypl + ypl / 2 + (size_t)mb_w * 13;
    off = (off + 3) & ~(size_t)3;
    w.finfo = (uint32_t*)(base + off);
    w.proba = base + off + (size_t)mb_w * mb_h * 4;
}

// ---- macroblock parse (RFC 6386 s.19.3, s.11, s.13) ----------------------------------------
struct MbInfo {
    uint8_t is_i4x4, ymode, uvmode, segment;
    uint8_t modes[16];   // sub-block modes when is_i4x4
    uint32_t tr_y;       // bits 2n..2n+1: TR_* class of luma block n
    uint32_t tr_uv;      // bits 2n..2n+1: TR_* class of chroma block n (0..3 U, 4..7 V), before uv_transform
    uint32_t finfo;      // loop-filter parameters, packed as in Work::finfo
};
struct RowCtx {  // state carried from the macroblock on the left
    uint8_t left_modes[4];
    uint8_t left_nz[9];
};
LP_VP8_FN void row_ctx_reset(RowCtx& rc) {
    for (int i = 0; i < 4; i++) rc.left_modes[i] = B_DC;
    for (int i = 0; i < 9; i++) rc.left_nz[i] = 0;
}

// Mode bits of one macroblock (first partition).  `tm` = the 4 sub-block modes above it.
// Returns the coded skip flag.
LP_VP8_FN int parse_mb_modes(const FrameHdr& h, BoolDec& br, uint8_t* tm, RowCtx& rc, MbInfo& mb) {
    int segment = 0;
    if (h.update_map)
        segment = !bd_bit(br, h.seg_proba[0]) ? bd_bit(br, h.seg_proba[1]) : bd_bit(br, h.seg_proba[2]) + 2;
    mb.segment = (uint8_t)segment;
    const int skip = h.use_skip ? bd_bit(br, h.skip_p) : 0;
    mb.is_i4x4 = (uint8_t)!bd_bit(br, 145);
    mb.ymode = DC_PRED;
    if (!mb.is_i4x4) {
        const int ymode = bd_bit(br, 156) ? (bd_bit(br, 128) ? TM_PRED : H_PRED) : (bd_bit(br, 163) ? V_PRED : DC_PRED);
        mb.ymode = (uint8_t)ymode;
        for (int i = 0; i < 4; i++) tm[i] = rc.left_modes[i] = (uint8_t)ymode;
    } else {
        for (int by = 0; by < 4; by++) {
            int lm = rc.left_modes[by];
            for (int bx = 0; bx < 4; bx++) {
                const uint8_t* prob = kVp8BModesProba[tm[bx]][lm];
                int i = kVp8YModesIntra4[bd_bit(br, prob[0])];
                while (i > 0) i = kVp8YModesIntra4[2 * i + bd_bit(br, prob[i])];
                lm = -i;
                tm[bx] = (uint8_t)lm;
                mb.modes[by * 4 + bx] = (uint8_t)lm;
            }
            rc.left_modes[by] = (uint8_t)lm;
        }
    }
    mb.uvmode = (uint8_t)(!bd_bit(br, 142) ? DC_PRED : !bd_bit(br, 114) ? V_PRED : bd_bit(br, 183) ? TM_PRED : H_PRED);
    return skip;
}

// Coefficient tokens of one macroblock (its row's token partition) into `coeffs` (25 blocks of
// 16, zeroed by the caller; block 24 is scratch for Y2).  `tnz` = the 9 non-zero flags above.
// Fills mb.tr_y, mb.tr_uv and mb.finfo.
LP_VP8_FN void parse_mb_residuals(const FrameHdr& h, BoolDec& tbr, const uint8_t* proba, uint8_t* tnz, RowCtx& rc,
                                  int skip, MbInfo& mb, int16_t* coeffs) {
    const QuantMat& q = h.q[mb.segment];
    uint32_t tr_y = 0, tr_uv = 0;
    if (!skip) {
        const int has_y2 = !mb.is_i4x4;
        // one loop over Y2?, 16 Y, 4 U, 4 V so the token reader is instantiated once
        for (int k = has_y2 ? -1 : 0; k < 24; k++) {
            int type, ti, li, first = 0;
            const int* dq;
            int16_t* out;
            if (k < 0) {
                type = 1; ti = 8; li = 8; dq = q.y2; out = coeffs + 24 * 16;
            } else if (k < 16) {
                type = has_y2 ? 0 : 3; ti = k & 3; li = k >> 2; dq = q.y1; out = coeffs + k * 16; first = has_y2;
            } else {
                const int c = k - 16;  // 0..3 U, 4..7 V
                type = 2; ti = 4 + (c >> 2) * 2 + (c & 1); li = 4 + (c >> 2) * 2 + ((c >> 1) & 1); dq = q.uv; out = coeffs + k * 16;
            }
            const int ctx = tnz[ti] + rc.left_nz[li];
            const int nz = get_coeffs(tbr, proba, type, ctx, dq, first, out);
            const uint8_t flag = (uint8_t)(nz > first);
            tnz[ti] = rc.left_nz[li] = flag;
            if (k < 0) {
                inverse_wht(out, coeffs);
            } else {
                // the DC may come from the Y2 transform
                const uint32_t cls = nz > 3 ? TR_FULL : nz > 1 ? TR_AC3 : out[0] != 0 ? TR_DC : TR_NONE;
                if (k < 16) tr_y |= cls << 2 * k;
                else tr_uv |= cls << 2 * (k - 16);
            }
        }
        skip = (tr_y | tr_uv) == 0;
    } else {
        for (int i = 0; i < 8; i++) tnz[i] = rc.left_nz[i] = 0;
        if (!mb.is_i4x4) tnz[8] = rc.left_nz[8] = 0;
    }
    mb.tr_y = tr_y;
    mb.tr_uv = tr_uv;
    const FilterStrength& f = h.fs[mb.segment][mb.is_i4x4];
    const uint32_t inner = f.inner | (uint32_t)(!skip);
    mb.finfo = f.limit | ((uint32_t)f.ilevel << 8) | ((uint32_t)f.hev << 16) | (inner << 24);
}

// ---- macroblock reconstruction, serial form (RFC 6386 s.12, s.14) --------------------------
// Work-buffer geometry shared with the device kernel: stride 32, luma block at column 8 of row 1,
// so the row above and the column to the left hold the prediction borders.
enum { BPS = 32, YB_SIZE = 17 * BPS, CB_SIZE = 9 * BPS };

LP_VP8_FN void reconstruct_mb(const FrameHdr& h, Work& w, int mb_x, int mb_y, const MbInfo& mb, const int16_t* coeffs,
                              uint8_t* yb, uint8_t* ub, uint8_t* vb) {
    const int mb_w = h.mb_w;
    const int ys = mb_w * 16, cs = mb_w * 8;
    uint8_t* yd = yb + BPS + 8;
    uint8_t* ud = ub + BPS + 8;
    uint8_t* vd = vb + BPS + 8;
    uint8_t* py = w.y + (size_t)mb_y * 16 * ys + mb_x * 16;
    uint8_t* pu = w.u + (size_t)mb_y * 8 * cs + mb_x * 8;
    uint8_t* pv = w.v + (size_t)mb_y * 8 * cs + mb_x * 8;
    // prediction borders (s.12.2): 127 above the first row, 129 left of the first column
    if (mb_x > 0) {
        for (int j = 0; j < 16; j++) yd[j * BPS - 1] = py[j * ys - 1];
        for (int j = 0; j < 8; j++) {
            ud[j * BPS - 1] = pu[j * cs - 1];
            vd[j * BPS - 1] = pv[j * cs - 1];
        }
    } else {
        for (int j = 0; j < 16; j++) yd[j * BPS - 1] = 129;
        for (int j = 0; j < 8; j++) ud[j * BPS - 1] = vd[j * BPS - 1] = 129;
    }
    if (mb_y > 0) {
        for (int i = 0; i < 16; i++) yd[i - BPS] = py[i - ys];
        for (int i = 0; i < 8; i++) {
            ud[i - BPS] = pu[i - cs];
            vd[i - BPS] = pv[i - cs];
        }
        if (mb_x < mb_w - 1)
            for (int i = 16; i < 20; i++) yd[i - BPS] = py[i - ys];
        else
            for (int i = 16; i < 20; i++) yd[i - BPS] = py[15 - ys];
        if (mb_x > 0) {
            yd[-1 - BPS] = py[-1 - ys];
            ud[-1 - BPS] = pu[-1 - cs];
            vd[-1 - BPS] = pv[-1 - cs];
        } else {
            yd[-1 - BPS] = ud[-1 - BPS] = vd[-1 - BPS] = 129;
        }
    } else {
        for (int i = -1; i < 20; i++) yd[i - BPS] = 127;
        for (int i = -1; i < 8; i++) ud[i - BPS] = vd[i - BPS] = 127;
    }
    if (mb.is_i4x4) {
        // the above-right samples of the macroblock serve every row of sub-blocks
        for (int r = 1; r < 4; r++)
            for (int i = 16; i < 20; i++) yd[(4 * r - 1) * BPS + i] = yd[i - BPS];
        for (int n = 0; n < 16; n++) {
            uint8_t* d = yd + (n >> 2) * 4 * BPS + (n & 3) * 4;
            pred_4x4(d, BPS, mb.modes[n]);
            transform_add((mb.tr_y >> 2 * n) & 3, coeffs + n * 16, d, BPS);
        }
    } else {
        pred_block(yd, BPS, 16, mb.ymode, mb_y > 0, mb_x > 0);
        for (int n = 0; n < 16; n++)
            transform_add((mb.tr_y >> 2 * n) & 3, coeffs + n * 16, yd + (n >> 2) * 4 * BPS + (n & 3) * 4, BPS);
    }
    pred_block(ud, BPS, 8, mb.uvmode, mb_y > 0, mb_x > 0);
    pred_block(vd, BPS, 8, mb.uvmode, mb_y > 0, mb_x > 0);
    for (int n = 0; n < 4; n++) {
        transform_add(uv_transform(mb.tr_uv, n), coeffs + (16 + n) * 16, ud + (n >> 1) * 4 * BPS + (n & 1) * 4, BPS);
        transform_add(uv_transform(mb.tr_uv, 4 + n), coeffs + (20 + n) * 16, vd + (n >> 1) * 4 * BPS + (n & 1) * 4, BPS);
    }
    for (int j = 0; j < 16; j++)
        for (int i = 0; i < 16; i++) py[j * ys + i] = yd[j * BPS + i];
    for (int j = 0; j < 8; j++)
        for (int i = 0; i < 8; i++) {
            pu[j * cs + i] = ud[j * BPS + i];
            pv[j * cs + i] = vd[j * BPS + i];
        }
}

// After the macroblock loop: whether the first partition or a token partition that some row used
// ran past its end.  libwebp refuses such a frame ("Premature end-of-file"); the flags are sticky,
// so one look at the end stands for its check after every row and macroblock.
LP_VP8_INL bool frame_truncated(const FrameHdr& h, const BoolDec& br, const BoolDec* parts) {
    bool eof = br.eof;
    for (int p = 0; p < h.num_parts && p < h.mb_h; p++) eof |= parts[p].eof != 0;
    return eof;
}

// Decodes every macroblock of the frame in raster order into the (unfiltered) planes and
// records the loop-filter parameters.  Serial by construction of the format: mode and token
// contexts chain left-to-right / top-to-bottom, and so does intra prediction.  (The device
// kernel runs the same parse functions on one lane and spreads reconstruction over the warp.)
LP_VP8_FN int decode_macroblocks(const uint8_t* data, const FrameHdr& h, BoolDec& br, Work& w) {
    const int mb_w = h.mb_w, mb_h = h.mb_h;
    for (int i = 0; i < mb_w * 4; i++) w.top_modes[i] = B_DC;
    for (int i = 0; i < mb_w * 9; i++) w.top_nz[i] = 0;
    uint8_t yb[YB_SIZE], ub[CB_SIZE], vb[CB_SIZE];
    int16_t coeffs[25 * 16];
    // one bool decoder per token partition, advanced row by row (s.9.5)
    BoolDec parts[8];
    for (int p = 0; p < h.num_parts; p++) bd_init(parts[p], data + h.part_off[p], h.part_len[p]);
    for (int mb_y = 0; mb_y < mb_h; mb_y++) {
        BoolDec& tbr = parts[mb_y & (h.num_parts - 1)];
        RowCtx rc;
        row_ctx_reset(rc);
        for (int mb_x = 0; mb_x < mb_w; mb_x++) {
            MbInfo mb;
            const int skip = parse_mb_modes(h, br, w.top_modes + mb_x * 4, rc, mb);
            for (int i = 0; i < 25 * 16; i++) coeffs[i] = 0;
            parse_mb_residuals(h, tbr, w.proba, w.top_nz + mb_x * 9, rc, skip, mb, coeffs);
            w.finfo[mb_y * mb_w + mb_x] = mb.finfo;
            reconstruct_mb(h, w, mb_x, mb_y, mb, coeffs, yb, ub, vb);
        }
    }
    return frame_truncated(h, br, parts) ? VP8_BAD : VP8_OK;
}

// ---- loop filter (RFC 6386 s.15) -----------------------------------------------------------
LP_VP8_FN int iabs(int v) { return v < 0 ? -v : v; }
LP_VP8_FN int sclip1(int v) { return v < -128 ? -128 : v > 127 ? 127 : v; }  // s.15.2 "c"
LP_VP8_FN int sclip2(int v) { return v < -16 ? -16 : v > 15 ? 15 : v; }

LP_VP8_FN void filter2(uint8_t* p, int step) {  // common_adjust with use_outer_taps
    const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
    const int a = 3 * (q0 - p0) + sclip1(p1 - q1);
    const int a1 = sclip2((a + 4) >> 3);
    const int a2 = sclip2((a + 3) >> 3);
    p[-step] = clip8(p0 + a2);
    p[0] = clip8(q0 - a1);
}
LP_VP8_FN void filter4(uint8_t* p, int step) {  // sub-block edge, no high edge variance
    const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
    const int a = 3 * (q0 - p0);
    const int a1 = sclip2((a + 4) >> 3);
    const int a2 = sclip2((a + 3) >> 3);
    const int a3 = (a1 + 1) >> 1;
    p[-2 * step] = clip8(p1 + a3);
    p[-step] = clip8(p0 + a2);
    p[0] = clip8(q0 - a1);
    p[step] = clip8(q1 - a3);
}
LP_VP8_FN void filter6(uint8_t* p, int step) {  // macroblock edge, no high edge variance
    const int p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step];
    const int q0 = p[0], q1 = p[step], q2 = p[2 * step];
    const int a = sclip1(3 * (q0 - p0) + sclip1(p1 - q1));
    const int a1 = (27 * a + 63) >> 7;
    const int a2 = (18 * a + 63) >> 7;
    const int a3 = (9 * a + 63) >> 7;
    p[-3 * step] = clip8(p2 + a3);
    p[-2 * step] = clip8(p1 + a2);
    p[-step] = clip8(p0 + a1);
    p[0] = clip8(q0 - a1);
    p[step] = clip8(q1 - a2);
    p[2 * step] = clip8(q2 - a3);
}
LP_VP8_FN int needs_filter(const uint8_t* p, int step, int t) {
    const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
    return (4 * iabs(p0 - q0) + iabs(p1 - q1)) <= t;
}
LP_VP8_FN int needs_filter2(const uint8_t* p, int step, int t, int it) {
    const int p3 = p[-4 * step], p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step];
    const int q0 = p[0], q1 = p[step], q2 = p[2 * step], q3 = p[3 * step];
    if ((4 * iabs(p0 - q0) + iabs(p1 - q1)) > t) return 0;
    return iabs(p3 - p2) <= it && iabs(p2 - p1) <= it && iabs(p1 - p0) <= it && iabs(q3 - q2) <= it &&
           iabs(q2 - q1) <= it && iabs(q1 - q0) <= it;
}
LP_VP8_FN int hev(const uint8_t* p, int step, int thresh) {
    const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
    return iabs(p1 - p0) > thresh || iabs(q1 - q0) > thresh;
}
// One sample position of an edge.  `step` crosses the edge; mb_edge selects the 6-tap variant.
LP_VP8_FN void filter_pos_simple(uint8_t* p, int step, int thresh) {
    if (needs_filter(p, step, 2 * thresh + 1)) filter2(p, step);
}
LP_VP8_FN void filter_pos_normal(uint8_t* p, int step, int thresh, int ithresh, int hev_t, int mb_edge) {
    if (!needs_filter2(p, step, 2 * thresh + 1, ithresh)) return;
    if (hev(p, step, hev_t)) filter2(p, step);
    else if (mb_edge) filter6(p, step);
    else filter4(p, step);
}
// Filters `n` positions along an edge: p walks by `along`, the filter crosses by `across`.
LP_VP8_FN void filter_edge(uint8_t* p, int along, int across, int n, int simple, int thresh, int ithresh,
                           int hev_t, int mb_edge) {
    for (int i = 0; i < n; i++, p += along) {
        if (simple) filter_pos_simple(p, across, thresh);
        else filter_pos_normal(p, across, thresh, ithresh, hev_t, mb_edge);
    }
}

// Filters one macroblock (all its edges, in the order s.15 prescribes: left MB edge, inner
// vertical edges, top MB edge, inner horizontal edges).
LP_VP8_FN void filter_macroblock(const FrameHdr& h, Work& w, int mb_x, int mb_y) {
    const uint32_t fi = w.finfo[mb_y * h.mb_w + mb_x];
    const int limit = fi & 255, ilevel = (fi >> 8) & 255, hev_t = (fi >> 16) & 255, inner = fi >> 24;
    if (limit == 0) return;
    const int ys = h.mb_w * 16, cs = h.mb_w * 8;
    uint8_t* y = w.y + (size_t)mb_y * 16 * ys + mb_x * 16;
    uint8_t* u = w.u + (size_t)mb_y * 8 * cs + mb_x * 8;
    uint8_t* v = w.v + (size_t)mb_y * 8 * cs + mb_x * 8;
    const int simple = h.filter_type == 1;
    if (mb_x > 0) {
        filter_edge(y, ys, 1, 16, simple, limit + 4, ilevel, hev_t, 1);
        if (!simple) {
            filter_edge(u, cs, 1, 8, 0, limit + 4, ilevel, hev_t, 1);
            filter_edge(v, cs, 1, 8, 0, limit + 4, ilevel, hev_t, 1);
        }
    }
    if (inner) {
        for (int k = 4; k < 16; k += 4) filter_edge(y + k, ys, 1, 16, simple, limit, ilevel, hev_t, 0);
        if (!simple) {
            filter_edge(u + 4, cs, 1, 8, 0, limit, ilevel, hev_t, 0);
            filter_edge(v + 4, cs, 1, 8, 0, limit, ilevel, hev_t, 0);
        }
    }
    if (mb_y > 0) {
        filter_edge(y, 1, ys, 16, simple, limit + 4, ilevel, hev_t, 1);
        if (!simple) {
            filter_edge(u, 1, cs, 8, 0, limit + 4, ilevel, hev_t, 1);
            filter_edge(v, 1, cs, 8, 0, limit + 4, ilevel, hev_t, 1);
        }
    }
    if (inner) {
        for (int k = 4; k < 16; k += 4) filter_edge(y + (size_t)k * ys, 1, ys, 16, simple, limit, ilevel, hev_t, 0);
        if (!simple) {
            filter_edge(u + 4 * cs, 1, cs, 8, 0, limit, ilevel, hev_t, 0);
            filter_edge(v + 4 * cs, 1, cs, 8, 0, limit, ilevel, hev_t, 0);
        }
    }
}

// ---- output: chroma upsampling + YUV -> BGR, libwebp conventions ---------------------------
// "Fancy" upsampler: 9-3-3-1 bilinear taps evaluated in libwebp's two-step rounding, then the
// 14-bit fixed-point BT.601 matrix of its VP8YUVToR/G/B.
LP_VP8_FN int yuv_clip8(int v) { return ((v & ~16383) == 0) ? (v >> 6) : (v < 0) ? 0 : 255; }
LP_VP8_FN int mult_hi(int v, int c) { return (v * c) >> 8; }
LP_VP8_FN void yuv_to_bgr(int y, int u, int v, uint8_t* bgr) {
    bgr[0] = (uint8_t)yuv_clip8(mult_hi(y, 19077) + mult_hi(u, 33050) - 17685);
    bgr[1] = (uint8_t)yuv_clip8(mult_hi(y, 19077) - mult_hi(u, 6419) - mult_hi(v, 13320) + 8708);
    bgr[2] = (uint8_t)yuv_clip8(mult_hi(y, 19077) + mult_hi(v, 26149) - 14234);
}
// Upsampled chroma sample for output pixel (x, row) of a width x height picture whose chroma
// plane `c` has stride cs.
LP_VP8_FN int upsample_at(const uint8_t* c, int cs, int width, int height, int x, int row) {
    const int ch = (height + 1) >> 1, cw = (width + 1) >> 1;
    // rows: `near` is the chroma row this output row leans on, `far` the other one
    int rn, rf;
    if (row == 0) {
        rn = rf = 0;
    } else if (row & 1) {
        rn = (row - 1) >> 1;
        rf = ((row + 1) >> 1) < ch ? (row + 1) >> 1 : rn;
    } else {
        rn = row >> 1;
        rf = rn - 1;
    }
    const uint8_t* nr = c + (size_t)rn * cs;
    const uint8_t* fr = c + (size_t)rf * cs;
    if (x == 0) return (3 * nr[0] + fr[0] + 2) >> 2;
    const int i = (x + 1) >> 1;  // pair index: pixels 2i-1 and 2i sit between chroma i-1 and i
    if (i >= cw) return (3 * nr[cw - 1] + fr[cw - 1] + 2) >> 2;  // last pixel of an even width
    const int a = nr[i - 1], b = nr[i], cc = fr[i - 1], d = fr[i];  // near-left, near-right, far-left, far-right
    const int avg = a + b + cc + d + 8;
    if (x & 1) {  // closer to near-left
        const int diag = (avg + 2 * (b + cc)) >> 3;
        return (diag + a) >> 1;
    } else {      // closer to near-right
        const int diag = (avg + 2 * (a + d)) >> 3;
        return (diag + b) >> 1;
    }
}

}  // namespace vp8
