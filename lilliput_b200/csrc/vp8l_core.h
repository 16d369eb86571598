// vp8l_core.h -- WebP lossless (VP8L) decoding, written against the "WebP Lossless Bitstream
// Specification": LSB-first bit reader, canonical prefix codes (normal + simple), meta prefix
// image, colour cache, LZ77 with the 2-D distance map, and the four inverse transforms
// (predictor, cross-colour, subtract-green, colour indexing).  Also decodes the ALPH chunk of a
// lossy frame (raw or VP8L-compressed plane + the horizontal / vertical / gradient un-filters).
//
// Stands where libwebp's VP8L decoder does behind WebPDecodeBGRInto / WebPDecodeBGRAInto
// (ref webp.cpp:336-351); libwebp is a vendored BINARY in the reference, nothing is taken from it.
// Parity is pinned on the reference's decoder itself (oracle/_ref, tests/test_webp_core.py) and on
// golden frames made by it.  The same functions compile for the device (webp_decode.cu) and for
// the CPU test harness (oracle/oracle_webp.cpp).
//
// Lossless decoding is exact by definition: every output must be bit-identical.
#pragma once
#include <stddef.h>
#include <stdint.h>

#ifndef LP_VP8_FN
#define LP_VP8_FN static inline
#endif
#ifndef LP_VP8_INL
#define LP_VP8_INL LP_VP8_FN
#endif

namespace vp8l {

enum { L_OK = 0, L_BAD = 1, L_NOMEM = 2 };

// ---- bump arena over caller memory ---------------------------------------------------------
struct Arena {
    uint8_t* base;
    size_t cap, used;
};
LP_VP8_INL void* arena_alloc(Arena& a, size_t n) {
    const size_t at = (a.used + 15) & ~(size_t)15;
    if (at + n > a.cap) return nullptr;
    a.used = at + n;
    return a.base + at;
}

// ---- bit reader (spec s.2: least-significant bit first) ------------------------------------
// Past the end the reader feeds zeros; `pos` counts every byte loaded, those zeros included.
struct Bits {
    const uint8_t* p;
    size_t n, pos;
    uint64_t val;
    int nbits;
    int eos;  // a prefix code matched no symbol
};
LP_VP8_INL void bits_init(Bits& b, const uint8_t* p, size_t n) {
    b.p = p;
    b.n = n;
    b.pos = 0;
    b.val = 0;
    b.nbits = 0;
    b.eos = 0;
}
LP_VP8_INL void bits_fill(Bits& b) {
    // 32 bits per refill (the refill is on the critical path of every symbol)
    while (b.nbits <= 32) {
        uint64_t w = 0;
        if (b.pos + 4 <= b.n) {
#ifdef __CUDA_ARCH__
            const uintptr_t a = reinterpret_cast<uintptr_t>(b.p + b.pos);
            const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
            w = __funnelshift_r(q[0], q[1], 8 * (int)(a & 3));  // q[1] may lie past the stream: inside the padded buffer
#else
            w = (uint64_t)b.p[b.pos] | ((uint64_t)b.p[b.pos + 1] << 8) | ((uint64_t)b.p[b.pos + 2] << 16) |
                ((uint64_t)b.p[b.pos + 3] << 24);
#endif
        } else {
            for (int k = 0; k < 4; k++)
                if (b.pos + k < b.n) w |= (uint64_t)b.p[b.pos + k] << (8 * k);
        }
        b.pos += 4;
        b.val |= w << b.nbits;
        b.nbits += 32;
    }
}
LP_VP8_INL uint32_t bits_read(Bits& b, int n) {  // n <= 32
    if (b.nbits < n) bits_fill(b);
    const uint32_t v = (uint32_t)(b.val & ((1ull << n) - 1));
    b.val >>= n;
    b.nbits -= n;
    return n ? v : 0;
}
// Whether the stream is unusable: a code matched nothing, or more bits have been used than the payload
// holds (libwebp's VP8LIsEndOfStream; the stream is truncated).  Sticky: the bits used only grow.
LP_VP8_INL bool bits_bad(const Bits& b) {
    return b.eos || (b.pos > b.n && (b.pos - b.n) * 8 > (size_t)b.nbits);
}

// ---- prefix codes (spec s.6.2) -------------------------------------------------------------
// Canonical code kept as per-length counts plus the symbols sorted by (length, value); codes are
// sent most-significant bit first, so decoding walks one bit at a time with a short root table
// for codes of up to 8 bits in front.
enum { kRootBits = 8 };
struct Code {
    uint16_t count[16];
    uint16_t* syms;   // arena
    uint16_t* root;   // arena, 1 << kRootBits entries: (len << 12) | symbol-index-independent symbol, 0 = walk
    int single;       // >= 0: the only symbol, decoded with zero bits
};

LP_VP8_FN int code_build(Code& c, const uint8_t* lens, int n, Arena& a) {
    for (int i = 0; i < 16; i++) c.count[i] = 0;
    int nsym = 0, last = 0;
    for (int i = 0; i < n; i++) {
        if (lens[i] > 15) return L_BAD;
        if (lens[i]) {
            c.count[lens[i]]++;
            nsym++;
            last = i;
        }
    }
    c.single = -1;
    c.syms = nullptr;
    c.root = nullptr;
    if (nsym == 0) return L_BAD;
    if (nsym == 1) {
        c.single = last;
        return L_OK;
    }
    int left = 1;
    for (int l = 1; l < 16; l++) {
        left = (left << 1) - c.count[l];
        if (left < 0) return L_BAD;
    }
    if (left != 0) return L_BAD;  // incomplete code
    c.syms = (uint16_t*)arena_alloc(a, (size_t)nsym * 2);
    c.root = (uint16_t*)arena_alloc(a, (size_t)2 << kRootBits);
    if (!c.syms || !c.root) return L_NOMEM;
    uint16_t offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; l++) offs[l + 1] = (uint16_t)(offs[l] + c.count[l]);
    for (int i = 0; i < n; i++)
        if (lens[i]) c.syms[offs[lens[i]]++] = (uint16_t)i;
    // root table: index = next kRootBits stream bits (LSB first); codes are MSB first, so the
    // canonical code of length l is bit-reversed into the low l bits of the index
    for (int i = 0; i < (1 << kRootBits); i++) c.root[i] = 0;
    int code = 0, index = 0;
    for (int l = 1; l <= kRootBits; l++) {
        for (int k = 0; k < c.count[l]; k++, code++, index++) {
            int rev = 0;
            for (int b = 0; b < l; b++) rev |= ((code >> b) & 1) << (l - 1 - b);
            // symbols above 4095 cannot be packed with the length; leave those to the walk
            if (c.syms[index] < 4096)
                for (int r = rev; r < (1 << kRootBits); r += 1 << l) c.root[r] = (uint16_t)((l << 12) | c.syms[index]);
        }
        code <<= 1;
    }
    return L_OK;
}

LP_VP8_INL int code_read(const Code& c, Bits& b) {
    if (c.single >= 0) return c.single;
    if (b.nbits < 16) bits_fill(b);
    const uint16_t e = c.root[b.val & ((1 << kRootBits) - 1)];
    if (e) {
        const int l = e >> 12;
        b.val >>= l;
        b.nbits -= l;
        return e & 4095;
    }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; l++) {
        code |= (int)(b.val & 1);
        b.val >>= 1;
        b.nbits--;
        const int cnt = c.count[l];
        if (code - first < cnt) return c.syms[index + (code - first)];
        index += cnt;
        first = (first + cnt) << 1;
        code <<= 1;
    }
    b.eos = 1;
    return 0;
}

// Reads one prefix code of `alphabet` symbols (spec s.6.2.1 simple / s.6.2.2 normal).
// `lens` is caller scratch of at least `alphabet` bytes.
LP_VP8_FN int code_read_definition(Bits& b, int alphabet, uint8_t* lens, Code& out, Arena& a) {
    for (int i = 0; i < alphabet; i++) lens[i] = 0;
    if (bits_read(b, 1)) {  // simple code: 1 or 2 symbols
        const int nsym = (int)bits_read(b, 1) + 1;
        const int first8 = (int)bits_read(b, 1);
        // a symbol past the alphabet is dropped, as libwebp drops it: the code keeps the other one, or has none
        const int s0 = (int)bits_read(b, first8 ? 8 : 1);
        if (s0 < alphabet) lens[s0] = 1;
        if (nsym == 2) {
            const int s1 = (int)bits_read(b, 8);
            if (s1 < alphabet) lens[s1] = 1;
        }
    } else {
        const uint8_t order[19] = {17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15};
        uint8_t cl[19];
        for (int i = 0; i < 19; i++) cl[i] = 0;
        const int ncodes = (int)bits_read(b, 4) + 4;
        if (ncodes > 19) return L_BAD;
        for (int i = 0; i < ncodes; i++) cl[order[i]] = (uint8_t)bits_read(b, 3);
        // the code-length code is small: decode it by canonical walk without tables
        uint16_t cnt[8], sym[19], offs[9];
        for (int i = 0; i < 8; i++) cnt[i] = 0;
        int n1 = 0, only = 0;
        for (int i = 0; i < 19; i++)
            if (cl[i]) {
                cnt[cl[i]]++;
                n1++;
                only = i;
            }
        if (n1 == 0) return L_BAD;
        if (n1 > 1) {
            int left = 1;
            for (int l = 1; l < 8; l++) {
                left = (left << 1) - cnt[l];
                if (left < 0) return L_BAD;
            }
            if (left != 0) return L_BAD;
        }
        offs[1] = 0;
        for (int l = 1; l < 8; l++) offs[l + 1] = (uint16_t)(offs[l] + cnt[l]);
        for (int i = 0; i < 19; i++)
            if (cl[i]) sym[offs[cl[i]]++] = (uint16_t)i;
        int max_symbol = alphabet;
        if (bits_read(b, 1)) {
            const int length_nbits = 2 + 2 * (int)bits_read(b, 3);
            max_symbol = 2 + (int)bits_read(b, length_nbits);
            if (max_symbol > alphabet) return L_BAD;
        }
        int symbol = 0, prev = 8;
        while (symbol < alphabet) {
            if (max_symbol-- == 0) break;
            int v;
            if (n1 == 1) {
                v = only;
            } else {
                int code = 0, first = 0, index = 0;
                v = -1;
                for (int l = 1; l < 8; l++) {
                    code |= (int)bits_read(b, 1);
                    if (code - first < cnt[l]) {
                        v = sym[index + (code - first)];
                        break;
                    }
                    index += cnt[l];
                    first = (first + cnt[l]) << 1;
                    code <<= 1;
                }
                if (v < 0) return L_BAD;
            }
            if (v < 16) {
                lens[symbol++] = (uint8_t)v;
                if (v) prev = v;
            } else {
                const int slot = v - 16;
                const int extra = slot == 0 ? 2 : slot == 1 ? 3 : 7;
                const int base = slot == 2 ? 11 : 3;
                const int rep = (int)bits_read(b, extra) + base;
                if (symbol + rep > alphabet) return L_BAD;
                const uint8_t val = (uint8_t)(slot == 0 ? prev : 0);
                for (int i = 0; i < rep; i++) lens[symbol++] = val;
            }
        }
    }
    if (bits_bad(b)) return L_BAD;
    return code_build(out, lens, alphabet, a);
}

// ---- entropy-coded image (spec s.5, s.6) ---------------------------------------------------
struct Group {
    Code c[5];  // green+length+cache, red, blue, alpha, distance
};

LP_VP8_INL int prefix_value(Bits& b, int symbol) {  // spec s.5.2.2: LZ77 prefix coding
    if (symbol < 4) return symbol + 1;
    const int extra = (symbol - 2) >> 1;
    const int offset = (2 + (symbol & 1)) << extra;
    return offset + (int)bits_read(b, extra) + 1;
}

// spec s.5.2.2: the 120 closest (dx, dy) neighbourhood positions, ordered by distance.  The list
// is "sort by dx^2+dy^2, then |dx|, then dx > 0 first" over dy in 0..7, dx in -7..8 -- built once.
struct DistMap {
    int8_t dx[120], dy[120];
};
LP_VP8_FN void dist_map_build(DistMap& m) {
    int n = 0;
    // insertion sort of the 120 candidates by (d2, |dx|, dx<0)
    for (int dy = 0; dy <= 7; dy++)
        for (int dx = -7; dx <= 8; dx++) {
            if (dy == 0 && dx <= 0) continue;
            const int key = ((dx * dx + dy * dy) << 8) | ((dx < 0 ? -dx : dx) << 1) | (dx < 0);
            int i = n++;
            while (i > 0) {
                const int px = m.dx[i - 1], py = m.dy[i - 1];
                const int pk = ((px * px + py * py) << 8) | ((px < 0 ? -px : px) << 1) | (px < 0);
                if (pk <= key) break;
                m.dx[i] = m.dx[i - 1];
                m.dy[i] = m.dy[i - 1];
                i--;
            }
            m.dx[i] = (int8_t)dx;
            m.dy[i] = (int8_t)dy;
        }
}
LP_VP8_INL int plane_code_to_distance(const DistMap& m, int xsize, int code) {
    if (code > 120) return code - 120;
    const int d = m.dy[code - 1] * xsize + m.dx[code - 1];
    return d >= 1 ? d : 1;
}

LP_VP8_INL int sub_size(int size, int bits) { return (size + (1 << bits) - 1) >> bits; }

// Decodes one entropy-coded ARGB image of xsize x ysize into `data` (arena).  META = whether a
// meta prefix image may be present (only the main image of a stream, spec s.6.2.3).
template <bool META>
LP_VP8_FN int decode_entropy_image(Bits& b, int xsize, int ysize, Arena& a, const DistMap& dm, uint32_t** out) {
    const size_t npix = (size_t)xsize * ysize;
    // colour cache
    int cache_bits = 0;
    if (bits_read(b, 1)) {
        cache_bits = (int)bits_read(b, 4);
        if (cache_bits < 1 || cache_bits > 11) return L_BAD;
    }
    // meta prefix codes
    int ngroups = 1, meta_bits = 0, meta_xs = 0;
    uint32_t* meta = nullptr;
    if (META && bits_read(b, 1)) {
        meta_bits = (int)bits_read(b, 3) + 2;
        meta_xs = sub_size(xsize, meta_bits);
        const int meta_ys = sub_size(ysize, meta_bits);
        const int rc = decode_entropy_image<false>(b, meta_xs, meta_ys, a, dm, &meta);
        if (rc) return rc;
        const size_t nm = (size_t)meta_xs * meta_ys;
        for (size_t i = 0; i < nm; i++) {
            meta[i] = (meta[i] >> 8) & 0xffff;
            if ((int)meta[i] >= ngroups) ngroups = (int)meta[i] + 1;
        }
    }
    Group* groups = (Group*)arena_alloc(a, sizeof(Group) * (size_t)ngroups);
    const int green_alphabet = 256 + 24 + (cache_bits ? (1 << cache_bits) : 0);
    uint8_t* lens = (uint8_t*)arena_alloc(a, (size_t)green_alphabet);
    if (!groups || !lens) return L_NOMEM;
    for (int g = 0; g < ngroups; g++) {
        const int alpha_sz[5] = {green_alphabet, 256, 256, 256, 40};
        for (int k = 0; k < 5; k++) {
            const int rc = code_read_definition(b, alpha_sz[k], lens, groups[g].c[k], a);
            if (rc) return rc;
        }
    }
    uint32_t* cache = nullptr;
    if (cache_bits) {
        cache = (uint32_t*)arena_alloc(a, (size_t)4 << cache_bits);
        if (!cache) return L_NOMEM;
        for (int i = 0; i < (1 << cache_bits); i++) cache[i] = 0;
    }
    uint32_t* data = (uint32_t*)arena_alloc(a, npix * 4);
    if (!data) return L_NOMEM;
    // pixels (spec s.5.2): literals, backward references, colour-cache hits
    size_t src = 0;
    int col = 0, row = 0;
    const int cache_shift = 32 - cache_bits;
    while (src < npix) {
        const Group& g = groups[meta ? meta[(size_t)(row >> meta_bits) * meta_xs + (col >> meta_bits)] : 0];
        const int code = code_read(g.c[0], b);
        if (code < 256) {
            const uint32_t red = (uint32_t)code_read(g.c[1], b);
            const uint32_t blue = (uint32_t)code_read(g.c[2], b);
            const uint32_t alpha = (uint32_t)code_read(g.c[3], b);
            const uint32_t px = (alpha << 24) | (red << 16) | ((uint32_t)code << 8) | blue;
            data[src++] = px;
            if (cache) cache[(px * 0x1e35a7bdu) >> cache_shift] = px;
            if (++col >= xsize) {
                col = 0;
                row++;
            }
        } else if (code < 256 + 24) {
            const int length = prefix_value(b, code - 256);
            const int dist_symbol = code_read(g.c[4], b);
            const int dist_code = prefix_value(b, dist_symbol);
            const int dist = plane_code_to_distance(dm, xsize, dist_code);
            if (bits_bad(b) || (size_t)dist > src || (size_t)length > npix - src) return L_BAD;
            for (int i = 0; i < length; i++) {
                const uint32_t px = data[src - dist];
                data[src++] = px;
                if (cache) cache[(px * 0x1e35a7bdu) >> cache_shift] = px;
            }
            col += length;
            while (col >= xsize) {
                col -= xsize;
                row++;
            }
        } else {
            const int key = code - (256 + 24);
            if (!cache || key >= (1 << cache_bits)) return L_BAD;
            const uint32_t px = cache[key];
            data[src++] = px;
            cache[(px * 0x1e35a7bdu) >> cache_shift] = px;
            if (++col >= xsize) {
                col = 0;
                row++;
            }
        }
        if (bits_bad(b)) return L_BAD;
    }
    *out = data;
    return L_OK;
}

// ---- transforms (spec s.4) -----------------------------------------------------------------
enum { T_PREDICTOR = 0, T_CROSS_COLOR = 1, T_SUBTRACT_GREEN = 2, T_COLOR_INDEXING = 3 };
struct Transform {
    int type, bits, xsize;  // xsize = image width this transform's inverse produces
    uint32_t* data;         // sub-image / palette
    int ncolors;
};

LP_VP8_INL uint32_t avg2(uint32_t a, uint32_t b) { return (((a ^ b) & 0xfefefefeu) >> 1) + (a & b); }
LP_VP8_INL uint32_t add_px(uint32_t a, uint32_t b) {
    const uint32_t ag = (a & 0xff00ff00u) + (b & 0xff00ff00u);
    const uint32_t rb = (a & 0x00ff00ffu) + (b & 0x00ff00ffu);
    return (ag & 0xff00ff00u) | (rb & 0x00ff00ffu);
}
LP_VP8_INL int iabs(int v) { return v < 0 ? -v : v; }
LP_VP8_INL uint32_t clip255(int v) { return v < 0 ? 0u : v > 255 ? 255u : (uint32_t)v; }
LP_VP8_INL uint32_t pred_select(uint32_t T, uint32_t L, uint32_t TL) {
    int d = 0;  // sum over channels of |L - TL| - |T - TL|
    for (int s = 0; s < 32; s += 8) {
        const int t = (T >> s) & 255, l = (L >> s) & 255, c = (TL >> s) & 255;
        d += iabs(l - c) - iabs(t - c);
    }
    return d <= 0 ? T : L;
}
LP_VP8_INL uint32_t pred_clamp_full(uint32_t L, uint32_t T, uint32_t TL) {
    uint32_t r = 0;
    for (int s = 0; s < 32; s += 8)
        r |= clip255((int)((L >> s) & 255) + (int)((T >> s) & 255) - (int)((TL >> s) & 255)) << s;
    return r;
}
LP_VP8_INL uint32_t pred_clamp_half(uint32_t A, uint32_t TL) {
    uint32_t r = 0;
    for (int s = 0; s < 32; s += 8) {
        const int a = (A >> s) & 255, c = (TL >> s) & 255;
        r |= clip255(a + (a - c) / 2) << s;  // C division: truncates toward zero
    }
    return r;
}
LP_VP8_INL uint32_t predict(int mode, uint32_t L, uint32_t T, uint32_t TR, uint32_t TL) {
    switch (mode) {
        case 1: return L;
        case 2: return T;
        case 3: return TR;
        case 4: return TL;
        case 5: return avg2(avg2(L, TR), T);
        case 6: return avg2(L, TL);
        case 7: return avg2(L, T);
        case 8: return avg2(TL, T);
        case 9: return avg2(T, TR);
        case 10: return avg2(avg2(L, TL), avg2(T, TR));
        case 11: return pred_select(T, L, TL);
        case 12: return pred_clamp_full(L, T, TL);
        case 13: return pred_clamp_half(avg2(L, T), TL);
        default: return 0xff000000u;  // 0, and the two unused codes
    }
}

// In-place inverse predictor transform of a width x height image.
LP_VP8_FN void inverse_predictor(const Transform& t, uint32_t* px, int width, int height) {
    const int tiles = sub_size(width, t.bits);
    for (int y = 0; y < height; y++) {
        uint32_t* row = px + (size_t)y * width;
        if (y == 0) {
            row[0] = add_px(row[0], 0xff000000u);
            for (int x = 1; x < width; x++) row[x] = add_px(row[x], row[x - 1]);
            continue;
        }
        const uint32_t* up = row - width;
        row[0] = add_px(row[0], up[0]);
        const uint32_t* modes = t.data + (size_t)(y >> t.bits) * tiles;
        for (int x = 1; x < width; x++) {
            const int mode = (modes[x >> t.bits] >> 8) & 15;
            // up[x + 1] at the last column is the first pixel of this row: memory order, as specified
            row[x] = add_px(row[x], predict(mode, row[x - 1], up[x], up[x + 1], up[x - 1]));
        }
    }
}

LP_VP8_INL int color_delta(int8_t t, int8_t c) { return ((int)t * (int)c) >> 5; }
LP_VP8_FN void inverse_cross_color(const Transform& t, uint32_t* px, int width, int height) {
    const int tiles = sub_size(width, t.bits);
    for (int y = 0; y < height; y++) {
        uint32_t* row = px + (size_t)y * width;
        const uint32_t* m = t.data + (size_t)(y >> t.bits) * tiles;
        for (int x = 0; x < width; x++) {
            const uint32_t code = m[x >> t.bits];
            const int8_t g2r = (int8_t)(code & 255), g2b = (int8_t)((code >> 8) & 255), r2b = (int8_t)((code >> 16) & 255);
            const uint32_t argb = row[x];
            const int8_t green = (int8_t)(argb >> 8);
            int red = (argb >> 16) & 255, blue = argb & 255;
            red = (red + color_delta(g2r, green)) & 255;
            blue = (blue + color_delta(g2b, green)) & 255;
            blue = (blue + color_delta(r2b, (int8_t)red)) & 255;
            row[x] = (argb & 0xff00ff00u) | ((uint32_t)red << 16) | (uint32_t)blue;
        }
    }
}
LP_VP8_FN void inverse_subtract_green(uint32_t* px, size_t n) {
    for (size_t i = 0; i < n; i++) {
        const uint32_t argb = px[i];
        const uint32_t g = (argb >> 8) & 255;
        uint32_t rb = argb & 0x00ff00ffu;
        rb = (rb + ((g << 16) | g)) & 0x00ff00ffu;
        px[i] = (argb & 0xff00ff00u) | rb;
    }
}
// src rows have the packed width, dst rows t.xsize pixels.
LP_VP8_FN void inverse_color_indexing(const Transform& t, const uint32_t* src, uint32_t* dst, int height) {
    const int width = t.xsize;
    const int bpp = 8 >> t.bits;
    const int src_w = sub_size(width, t.bits);
    for (int y = 0; y < height; y++) {
        const uint32_t* s = src + (size_t)y * src_w;
        uint32_t* d = dst + (size_t)y * width;
        if (t.bits == 0) {
            for (int x = 0; x < width; x++) d[x] = t.data[(s[x] >> 8) & 255];
        } else {
            uint32_t packed = 0;
            for (int x = 0; x < width; x++) {
                if ((x & ((1 << t.bits) - 1)) == 0) packed = (*s++ >> 8) & 255;
                d[x] = t.data[packed & ((1 << bpp) - 1)];
                packed >>= bpp;
            }
        }
    }
}

// ---- a whole VP8L image stream (spec s.3 - s.7) --------------------------------------------
// Decodes the stream at `b` (positioned after any header) for a width x height picture and
// returns the final ARGB pixels (arena memory).
LP_VP8_FN int decode_stream(Bits& b, int width, int height, Arena& a, uint32_t** out) {
    DistMap* dm = (DistMap*)arena_alloc(a, sizeof(DistMap));
    if (!dm) return L_NOMEM;
    dist_map_build(*dm);
    Transform tr[4];
    int ntr = 0, seen = 0;
    int xsize = width;
    while (bits_read(b, 1)) {
        if (ntr == 4) return L_BAD;
        Transform& t = tr[ntr];
        t.type = (int)bits_read(b, 2);
        if (seen & (1 << t.type)) return L_BAD;  // each transform at most once
        seen |= 1 << t.type;
        t.xsize = xsize;
        t.bits = 0;
        t.data = nullptr;
        t.ncolors = 0;
        if (t.type == T_PREDICTOR || t.type == T_CROSS_COLOR) {
            t.bits = (int)bits_read(b, 3) + 2;
            const int rc = decode_entropy_image<false>(b, sub_size(xsize, t.bits), sub_size(height, t.bits), a, *dm, &t.data);
            if (rc) return rc;
        } else if (t.type == T_COLOR_INDEXING) {
            const int n = (int)bits_read(b, 8) + 1;
            t.ncolors = n;
            t.bits = n > 16 ? 0 : n > 4 ? 1 : n > 2 ? 2 : 3;
            uint32_t* pal = nullptr;
            const int rc = decode_entropy_image<false>(b, n, 1, a, *dm, &pal);
            if (rc) return rc;
            const int table = 1 << (8 >> t.bits);
            t.data = (uint32_t*)arena_alloc(a, (size_t)table * 4);
            if (!t.data) return L_NOMEM;
            for (int i = 0; i < table; i++) t.data[i] = 0;  // out-of-range indices are transparent black
            uint32_t prev = 0;
            for (int i = 0; i < n && i < table; i++) {  // palette entries are delta coded
                prev = add_px(pal[i], prev);
                t.data[i] = prev;
            }
            xsize = sub_size(xsize, t.bits);
        }
        ntr++;
        if (bits_bad(b)) return L_BAD;
    }
    uint32_t* px = nullptr;
    int rc = decode_entropy_image<true>(b, xsize, height, a, *dm, &px);
    if (rc) return rc;
    for (int i = ntr - 1; i >= 0; i--) {
        const Transform& t = tr[i];
        if (t.type == T_PREDICTOR) inverse_predictor(t, px, t.xsize, height);
        else if (t.type == T_CROSS_COLOR) inverse_cross_color(t, px, t.xsize, height);
        else if (t.type == T_SUBTRACT_GREEN) inverse_subtract_green(px, (size_t)t.xsize * height);
        else {
            uint32_t* wide = (uint32_t*)arena_alloc(a, (size_t)t.xsize * height * 4);
            if (!wide) return L_NOMEM;
            inverse_color_indexing(t, px, wide, height);
            px = wide;
        }
    }
    *out = px;
    return L_OK;
}

// A "VP8L" chunk payload: 0x2f, 14-bit width-1, 14-bit height-1, alpha hint, 3-bit version.
LP_VP8_FN int decode_vp8l(const uint8_t* p, size_t n, int width, int height, Arena& a, uint32_t** out) {
    if (n < 5 || p[0] != 0x2f) return L_BAD;
    Bits b;
    bits_init(b, p + 1, n - 1);
    const int w = (int)bits_read(b, 14) + 1, h = (int)bits_read(b, 14) + 1;
    bits_read(b, 1);
    if (bits_read(b, 3) != 0 || w != width || h != height) return L_BAD;
    return decode_stream(b, width, height, a, out);
}

// ---- ALPH chunk of a lossy frame (container spec, "Alpha") ----------------------------------
// Header byte: bits 0-1 compression (0 raw, 1 VP8L), 2-3 filter, 4-5 pre-processing, 6-7 reserved.
// Writes width*height alpha bytes to `alpha`.
LP_VP8_FN int decode_alph(const uint8_t* p, size_t n, int width, int height, Arena& a, uint8_t* alpha) {
    if (n < 1) return L_BAD;
    const int method = p[0] & 3, filter = (p[0] >> 2) & 3, pre = (p[0] >> 4) & 3, rsrv = (p[0] >> 6) & 3;
    if (method > 1 || pre > 1 || rsrv != 0) return L_BAD;
    const size_t npix = (size_t)width * height;
    if (method == 0) {
        if (n - 1 < npix) return L_BAD;
        for (size_t i = 0; i < npix; i++) alpha[i] = p[1 + i];
    } else {
        Bits b;
        bits_init(b, p + 1, n - 1);
        uint32_t* px = nullptr;
        const int rc = decode_stream(b, width, height, a, &px);
        if (rc) return rc;
        for (size_t i = 0; i < npix; i++) alpha[i] = (uint8_t)(px[i] >> 8);  // alpha travels in green
    }
    if (filter == 0) return L_OK;
    // un-filter in place, row by row (1 horizontal, 2 vertical, 3 gradient)
    for (int y = 0; y < height; y++) {
        uint8_t* row = alpha + (size_t)y * width;
        const uint8_t* up = y ? row - width : nullptr;
        if (!up || filter == 1) {
            uint8_t pred = up ? up[0] : 0;
            for (int x = 0; x < width; x++) {
                row[x] = (uint8_t)(row[x] + pred);
                pred = row[x];
            }
        } else if (filter == 2) {
            for (int x = 0; x < width; x++) row[x] = (uint8_t)(row[x] + up[x]);
        } else {
            uint8_t left = up[0], top = up[0], tl = up[0];
            for (int x = 0; x < width; x++) {
                top = up[x];
                const int g = (int)left + (int)top - (int)tl;
                left = (uint8_t)(row[x] + (g < 0 ? 0 : g > 255 ? 255 : g));
                tl = top;
                row[x] = left;
            }
        }
    }
    return L_OK;
}

}  // namespace vp8l
