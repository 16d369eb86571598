/*
 * oracle_jpeg_dec.c -- CPU restatement of baseline JPEG decoding as the reference
 * performs it.  TEST INFRASTRUCTURE ONLY (see oracle.h).
 *
 * Reference call site: opencv_decoder_read_data (ref opencv.cpp:166-171) ->
 * cv::ImageDecoder::readData -> libjpeg-turbo 3.1.0 (ref deps/build-deps-linux.sh:171;
 * source not in tree) with its defaults: JDCT_ISLOW, do_fancy_upsampling = TRUE,
 * out_color_space = JCS_EXT_BGR (colour) or JCS_GRAYSCALE.
 *
 * Restated from ITU-T T.81 (entropy coding, marker syntax) and libjpeg-turbo's
 * published jidctint.c / jdsample.c / jdcolor.c as summarised in SURVEY.md
 * Appendix E.2.  Where libjpeg-turbo's x86 SIMD path differs from its C path on
 * out-of-range data, the SIMD behaviour is followed because that is what the
 * reference's AVX2 build executes: 16-bit wrapping dequantisation, int16
 * saturation between the two IDCT passes, true clamping of the output.
 * Pinned against oracle/_ref and tests/golden/ in tests/test_oracle_jpeg.py.
 */
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

enum { E_TRUNC = -1, E_UNSUPPORTED = -2, E_CORRUPT = -3, E_SMALL = -4 };

static const uint8_t ZIGZAG[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                   12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                   58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

typedef struct {
    uint8_t bits[17], vals[256];
    int present;
    uint16_t lut[65536]; /* (len << 8) | symbol, 0 = invalid, indexed by the next 16 bits */
} HuffTable;

typedef struct {
    int id, h, v, tq, td, ta;
    int bw, bh;     /* allocated blocks (padded to the MCU grid) */
    int dw, dh;     /* true downsampled size in samples */
    int16_t* coef;  /* bw*bh*64, natural order, quantised */
    uint8_t* plane; /* (bw*8) x (bh*8) samples after IDCT */
    int pred;
} Comp;

typedef struct {
    const uint8_t* p;
    const uint8_t* end;
    uint64_t acc;
    int nbits;
    int hit_marker;
} BitReader;

static void br_fill(BitReader* b) {
    while (b->nbits <= 56) {
        unsigned byte = 0;
        if (!b->hit_marker && b->p < b->end) {
            byte = *b->p;
            if (byte == 0xFF) {
                /* T.81 B.1.1.5: FF00 is a stuffed FF; FF FF.. is fill; anything else a marker */
                const uint8_t* q = b->p + 1;
                while (q < b->end && *q == 0xFF) q++;
                if (q < b->end && *q == 0x00) {
                    b->p = q + 1;
                } else {
                    b->hit_marker = 1; /* leave p on the FF; feed zero bits from here on */
                    byte = 0;
                }
            } else {
                b->p++;
            }
        }
        b->acc |= (uint64_t)byte << (56 - b->nbits);
        b->nbits += 8;
    }
}
static inline unsigned br_peek16(BitReader* b) {
    if (b->nbits < 32) br_fill(b);
    return (unsigned)(b->acc >> 48);
}
static inline void br_skip(BitReader* b, int n) {
    b->acc <<= n;
    b->nbits -= n;
}
static inline int br_get(BitReader* b, int n) {
    if (n == 0) return 0;
    if (b->nbits < 32) br_fill(b);
    int v = (int)(b->acc >> (64 - n));
    br_skip(b, n);
    return v;
}

static void build_lut(HuffTable* t) {
    memset(t->lut, 0, sizeof(t->lut));
    unsigned code = 0;
    int k = 0;
    for (int len = 1; len <= 16; len++) {
        for (int i = 0; i < t->bits[len]; i++, k++) {
            unsigned first = code << (16 - len), n = 1u << (16 - len);
            if (first + n > 65536) return; /* over-subscribed table: leave the rest invalid */
            for (unsigned j = 0; j < n; j++) t->lut[first + j] = (uint16_t)((len << 8) | t->vals[k]);
            code++;
        }
        code <<= 1;
    }
}

static inline int huff_decode(BitReader* b, const HuffTable* t) {
    unsigned e = t->lut[br_peek16(b)];
    if (!e) return -1;
    br_skip(b, e >> 8);
    return e & 0xFF;
}
static inline int extend(int v, int n) { return v < (1 << (n - 1)) ? v - (1 << n) + 1 : v; }

/* One 8x8 block, T.81 F.2.2: DC difference then AC run/size pairs. */
static int decode_block(BitReader* b, const HuffTable* dc, const HuffTable* ac, Comp* c, int16_t* out) {
    int s = huff_decode(b, dc);
    if (s < 0 || s > 15) return E_CORRUPT;
    int diff = s ? extend(br_get(b, s), s) : 0;
    c->pred += diff;
    out[0] = (int16_t)c->pred;
    for (int k = 1; k < 64;) {
        int rs = huff_decode(b, ac);
        if (rs < 0) return E_CORRUPT;
        int r = rs >> 4, n = rs & 15;
        if (n == 0) {
            if (r != 15) break; /* EOB */
            k += 16;            /* ZRL */
            continue;
        }
        k += r;
        if (k > 63) return E_CORRUPT;
        out[ZIGZAG[k]] = (int16_t)extend(br_get(b, n), n);
        k++;
    }
    return 0;
}

/* ---- progressive scans (T.81 Annex G; libjpeg-turbo jdphuff.c decode_mcu_{DC,AC}_{first,refine}) ---- */
typedef struct {
    int Ss, Se, Ah, Al;
    unsigned eobrun; /* blocks still covered by an end-of-band run */
} ProgState;

/* DC coefficient, first pass (G.1.2.1): difference coding as in sequential mode, value << Al. */
static int prog_dc_first(BitReader* b, const HuffTable* dc, Comp* c, const ProgState* ps, int16_t* blk) {
    int s = huff_decode(b, dc);
    if (s < 0 || s > 15) return E_CORRUPT;
    int diff = s ? extend(br_get(b, s), s) : 0;
    c->pred += diff;
    blk[0] = (int16_t)((unsigned)c->pred << ps->Al);
    return 0;
}
/* DC refinement (G.1.2.1): one more bit of precision per block. */
static int prog_dc_refine(BitReader* b, const ProgState* ps, int16_t* blk) {
    if (br_get(b, 1)) blk[0] |= (int16_t)(1 << ps->Al);
    return 0;
}
/* AC band, first pass (G.1.2.2): run/size pairs with EOBn runs spanning blocks. */
static int prog_ac_first(BitReader* b, const HuffTable* ac, ProgState* ps, int16_t* blk) {
    if (ps->eobrun > 0) {
        ps->eobrun--;
        return 0;
    }
    for (int k = ps->Ss; k <= ps->Se; k++) {
        int rs = huff_decode(b, ac);
        if (rs < 0) return E_CORRUPT;
        int r = rs >> 4, n = rs & 15;
        if (n) {
            k += r;
            if (k > 63) return E_CORRUPT;
            blk[ZIGZAG[k]] = (int16_t)((unsigned)extend(br_get(b, n), n) << ps->Al);
        } else if (r == 15) {
            k += 15; /* ZRL */
        } else {
            ps->eobrun = 1u << r;
            if (r) ps->eobrun += (unsigned)br_get(b, r);
            ps->eobrun--; /* this block is the first of the run */
            break;
        }
    }
    return 0;
}
/* AC band refinement (G.1.2.3): correction bits for already-nonzero coefficients interleaved
 * with newly-nonzero ones. */
static int prog_ac_refine(BitReader* b, const HuffTable* ac, ProgState* ps, int16_t* blk) {
    const int p1 = 1 << ps->Al, m1 = -(1 << ps->Al);
    int k = ps->Ss;
    if (ps->eobrun == 0) {
        for (; k <= ps->Se; k++) {
            int rs = huff_decode(b, ac);
            if (rs < 0) return E_CORRUPT;
            int r = rs >> 4, n = rs & 15, val = 0;
            if (n) {
                if (n != 1) return E_CORRUPT; /* size of a newly nonzero coefficient must be 1 */
                val = br_get(b, 1) ? p1 : m1;
            } else if (r != 15) {
                ps->eobrun = 1u << r;
                if (r) ps->eobrun += (unsigned)br_get(b, r);
                break; /* the rest of the block is handled by the end-of-band logic below */
            }
            /* advance over already-nonzero coefficients and r still-zero ones */
            do {
                int16_t* co = blk + ZIGZAG[k];
                if (*co != 0) {
                    if (br_get(b, 1)) {
                        if ((*co & p1) == 0) *co = (int16_t)(*co + (*co >= 0 ? p1 : m1));
                    }
                } else {
                    if (--r < 0) break; /* reached the target zero coefficient */
                }
                k++;
            } while (k <= ps->Se);
            if (val) {
                if (k > 63) return E_CORRUPT;
                blk[ZIGZAG[k]] = (int16_t)val;
            }
        }
    }
    if (ps->eobrun > 0) {
        /* in an end-of-band run: only correction bits for the nonzero coefficients that remain */
        for (; k <= ps->Se; k++) {
            int16_t* co = blk + ZIGZAG[k];
            if (*co != 0 && br_get(b, 1)) {
                if ((*co & p1) == 0) *co = (int16_t)(*co + (*co >= 0 ? p1 : m1));
            }
        }
        ps->eobrun--;
    }
    return 0;
}

/* jpeg_idct_islow with libjpeg-turbo's SIMD range behaviour. */
#define FIX_0_298631336 2446
#define FIX_0_390180644 3196
#define FIX_0_541196100 4433
#define FIX_0_765366865 6270
#define FIX_0_899976223 7373
#define FIX_1_175875602 9633
#define FIX_1_501321110 12299
#define FIX_1_847759065 15137
#define FIX_1_961570560 16069
#define FIX_2_053119869 16819
#define FIX_2_562915447 20995
#define FIX_3_072711026 25172
#define DESCALE(x, n) (((x) + (1 << ((n)-1))) >> (n))

static inline int sat16(int v) { return v < -32768 ? -32768 : v > 32767 ? 32767 : v; }

static void idct_1d(const int in[8], int out[8], int shift, int sat) {
    int z2 = in[2], z3 = in[6];
    int z1 = (z2 + z3) * FIX_0_541196100;
    int tmp2 = z1 + z3 * (-FIX_1_847759065);
    int tmp3 = z1 + z2 * FIX_0_765366865;
    int tmp0 = (in[0] + in[4]) << 13;
    int tmp1 = (in[0] - in[4]) << 13;
    int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    int t0 = in[7], t1 = in[5], t2 = in[3], t3 = in[1];
    z1 = t0 + t3;
    z2 = t1 + t2;
    z3 = t0 + t2;
    int z4 = t1 + t3;
    int z5 = (z3 + z4) * FIX_1_175875602;
    t0 *= FIX_0_298631336;
    t1 *= FIX_2_053119869;
    t2 *= FIX_3_072711026;
    t3 *= FIX_1_501321110;
    z1 *= -FIX_0_899976223;
    z2 *= -FIX_2_562915447;
    z3 *= -FIX_1_961570560;
    z4 *= -FIX_0_390180644;
    z3 += z5;
    z4 += z5;
    t0 += z1 + z3;
    t1 += z2 + z4;
    t2 += z2 + z3;
    t3 += z1 + z4;
    out[0] = DESCALE(tmp10 + t3, shift);
    out[7] = DESCALE(tmp10 - t3, shift);
    out[1] = DESCALE(tmp11 + t2, shift);
    out[6] = DESCALE(tmp11 - t2, shift);
    out[2] = DESCALE(tmp12 + t1, shift);
    out[5] = DESCALE(tmp12 - t1, shift);
    out[3] = DESCALE(tmp13 + t0, shift);
    out[4] = DESCALE(tmp13 - t0, shift);
    if (sat)
        for (int i = 0; i < 8; i++) out[i] = sat16(out[i]);
}

static void idct_block(const int16_t* coef, const uint16_t* q, uint8_t* dst, int stride) {
    int ws[64];
    for (int x = 0; x < 8; x++) {
        int in[8], out[8];
        for (int y = 0; y < 8; y++) in[y] = (int16_t)(coef[y * 8 + x] * q[y * 8 + x]); /* pmullw */
        idct_1d(in, out, 13 - 2, 1);
        for (int y = 0; y < 8; y++) ws[y * 8 + x] = out[y];
    }
    for (int y = 0; y < 8; y++) {
        int out[8];
        idct_1d(ws + y * 8, out, 13 + 2 + 3, 0);
        for (int x = 0; x < 8; x++) {
            int v = out[x];
            v = v < -128 ? -128 : v > 127 ? 127 : v; /* packsswb */
            dst[y * stride + x] = (uint8_t)(v + 128);
        }
    }
}

/* EXIF orientation (tag 0x0112 of IFD0) from an APP1 "Exif\0\0" payload. */
static int exif_orientation(const uint8_t* p, size_t n) {
    if (n < 14 || memcmp(p, "Exif\0\0", 6) != 0) return 0;
    const uint8_t* t = p + 6;
    size_t tn = n - 6;
    int le;
    if (t[0] == 'I' && t[1] == 'I') le = 1;
    else if (t[0] == 'M' && t[1] == 'M') le = 0;
    else return 0;
#define RD16(o) (le ? (t[o] | (t[(o) + 1] << 8)) : ((t[o] << 8) | t[(o) + 1]))
#define RD32(o) (le ? ((uint32_t)t[o] | ((uint32_t)t[(o) + 1] << 8) | ((uint32_t)t[(o) + 2] << 16) | ((uint32_t)t[(o) + 3] << 24)) \
                    : (((uint32_t)t[o] << 24) | ((uint32_t)t[(o) + 1] << 16) | ((uint32_t)t[(o) + 2] << 8) | t[(o) + 3]))
    if (RD16(2) != 42) return 0;
    size_t ifd = RD32(4);
    if (ifd + 2 > tn) return 0;
    int cnt = RD16(ifd);
    for (int i = 0; i < cnt; i++) {
        size_t e = ifd + 2 + (size_t)i * 12;
        if (e + 12 > tn) return 0;
        if (RD16(e) == 0x0112) {
            int v = RD16(e + 8);
            return (v >= 1 && v <= 8) ? v : 0;
        }
    }
    return 0;
}

/* jdsample.c: fancy (triangle) upsampling.  `get(r)` rows are clamped to the
 * component's true downsampled height; columns to its true downsampled width.
 * jinit_upsampler picks the h2v1 / h2v2 triangle filters only for components more
 * than two samples wide; narrower ones are replicated (h2v1_upsample / h2v2_upsample). */
static void upsample_rows(const Comp* c, int maxh, int maxv, int y, int out_w, uint8_t* out) {
    int stride = c->bw * 8;
    int hr = maxh / c->h, vr = maxv / c->v;
    int cw = c->dw;
    if (hr == 1 && vr == 1) {
        memcpy(out, c->plane + (size_t)y * stride, out_w);
        return;
    }
    if (hr == 2 && vr == 1 && cw > 2) { /* h2v1_fancy_upsample */
        const uint8_t* s = c->plane + (size_t)y * stride;
        for (int i = 0; i < cw; i++) {
            int l = s[i > 0 ? i - 1 : 0], r = s[i + 1 < cw ? i + 1 : cw - 1], v = s[i] * 3;
            int a = (i == 0) ? s[0] : (v + l + 1) >> 2;
            int b = (i == cw - 1) ? s[i] : (v + r + 2) >> 2;
            if (2 * i < out_w) out[2 * i] = (uint8_t)a;
            if (2 * i + 1 < out_w) out[2 * i + 1] = (uint8_t)b;
        }
        return;
    }
    if (hr == 1 && vr == 2) { /* h1v2_fancy_upsample */
        int cy = y >> 1, far = (y & 1) ? cy + 1 : cy - 1, bias = (y & 1) ? 2 : 1;
        if (far < 0) far = 0;
        if (far > c->dh - 1) far = c->dh - 1;
        const uint8_t* s0 = c->plane + (size_t)cy * stride;
        const uint8_t* s1 = c->plane + (size_t)far * stride;
        for (int i = 0; i < out_w; i++) out[i] = (uint8_t)((s0[i] * 3 + s1[i] + bias) >> 2);
        return;
    }
    if (hr == 2 && vr == 2 && cw > 2) { /* h2v2_fancy_upsample */
        int cy = y >> 1, far = (y & 1) ? cy + 1 : cy - 1;
        if (far < 0) far = 0;
        if (far > c->dh - 1) far = c->dh - 1;
        const uint8_t* s0 = c->plane + (size_t)cy * stride;
        const uint8_t* s1 = c->plane + (size_t)far * stride;
        for (int i = 0; i < cw; i++) {
            int cs = 3 * s0[i] + s1[i];
            int il = i > 0 ? i - 1 : 0, ir = i + 1 < cw ? i + 1 : cw - 1;
            int l = 3 * s0[il] + s1[il], r = 3 * s0[ir] + s1[ir];
            int a = (i == 0) ? (cs * 4 + 8) >> 4 : (cs * 3 + l + 8) >> 4;
            int b = (i == cw - 1) ? (cs * 4 + 7) >> 4 : (cs * 3 + r + 7) >> 4;
            if (2 * i < out_w) out[2 * i] = (uint8_t)a;
            if (2 * i + 1 < out_w) out[2 * i + 1] = (uint8_t)b;
        }
        return;
    }
    /* int_upsample / h2v1_upsample / h2v2_upsample: pixel replication */
    const uint8_t* s = c->plane + (size_t)(y / vr) * stride;
    for (int i = 0; i < out_w; i++) out[i] = s[i / hr];
}

int oracle_jpeg_decode(const uint8_t* in, size_t len, uint8_t* out, size_t out_cap, int* width,
                       int* height, int* channels, int* orientation) {
    static HuffTable* HT = NULL; /* [class][id] */
    if (!HT) HT = calloc(8, sizeof(HuffTable));
    HuffTable(*ht)[4] = (HuffTable(*)[4])HT;
    for (int i = 0; i < 8; i++) HT[i].present = 0;
    uint16_t qt[4][64];
    int qpresent[4] = {0, 0, 0, 0};
    Comp comp[4];
    memset(comp, 0, sizeof(comp));
    int ncomp = 0, W = 0, H = 0, maxh = 1, maxv = 1, restart = 0, orient = 1, have_sof = 0;
    int rc = 0, scans_done = 0, progressive = 0, prog_scans = 0;
    size_t pos = 2;
    if (len < 4 || in[0] != 0xFF || in[1] != 0xD8) return E_CORRUPT;

    while (pos + 4 <= len) {
        if (in[pos] != 0xFF) { pos++; continue; }
        uint8_t m = in[pos + 1];
        if (m == 0xFF) { pos++; continue; }
        if (m == 0xD9) break;
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) { pos += 2; continue; }
        size_t seg = ((size_t)in[pos + 2] << 8) | in[pos + 3];
        if (seg < 2 || pos + 2 + seg > len) { rc = E_TRUNC; goto done; }
        const uint8_t* p = in + pos + 4;
        size_t n = seg - 2;
        if (m == 0xDB) { /* DQT */
            while (n >= 65) {
                int pq = p[0] >> 4, tq = p[0] & 15;
                if (tq > 3) { rc = E_CORRUPT; goto done; }
                size_t need = pq ? 129 : 65;
                if (n < need) { rc = E_CORRUPT; goto done; }
                for (int i = 0; i < 64; i++)
                    qt[tq][ZIGZAG[i]] = pq ? (uint16_t)((p[1 + 2 * i] << 8) | p[2 + 2 * i]) : p[1 + i];
                qpresent[tq] = 1;
                p += need;
                n -= need;
            }
        } else if (m == 0xC4) { /* DHT */
            while (n >= 17) {
                int tc = p[0] >> 4, th = p[0] & 15;
                if (tc > 1 || th > 3) { rc = E_CORRUPT; goto done; }
                HuffTable* t = &ht[tc][th];
                int total = 0;
                t->bits[0] = 0;
                for (int i = 1; i <= 16; i++) { t->bits[i] = p[i]; total += p[i]; }
                if (total > 256 || n < (size_t)(17 + total)) { rc = E_CORRUPT; goto done; }
                memcpy(t->vals, p + 17, total);
                t->present = 1;
                build_lut(t);
                p += 17 + total;
                n -= 17 + total;
            }
        } else if (m == 0xC0 || m == 0xC1 || m == 0xC2) { /* SOF0 / SOF1 sequential, SOF2 progressive Huffman */
            progressive = (m == 0xC2);
            if (n < 6 || p[0] != 8) { rc = E_UNSUPPORTED; goto done; }
            H = (p[1] << 8) | p[2];
            W = (p[3] << 8) | p[4];
            ncomp = p[5];
            if ((ncomp != 1 && ncomp != 3) || n < (size_t)(6 + 3 * ncomp) || W < 1 || H < 1) { rc = E_UNSUPPORTED; goto done; }
            for (int i = 0; i < ncomp; i++) {
                comp[i].id = p[6 + 3 * i];
                comp[i].h = p[7 + 3 * i] >> 4;
                comp[i].v = p[7 + 3 * i] & 15;
                comp[i].tq = p[8 + 3 * i];
                if (comp[i].h < 1 || comp[i].h > 4 || comp[i].v < 1 || comp[i].v > 4 || comp[i].tq > 3) { rc = E_CORRUPT; goto done; }
                if (comp[i].h > maxh) maxh = comp[i].h;
                if (comp[i].v > maxv) maxv = comp[i].v;
            }
            if (ncomp == 1) { comp[0].h = comp[0].v = 1; maxh = maxv = 1; } /* single-component scans are never interleaved */
            for (int i = 0; i < ncomp; i++)
                if (maxh % comp[i].h || maxv % comp[i].v) { rc = E_UNSUPPORTED; goto done; }
            have_sof = 1;
            if (width) *width = W;
            if (height) *height = H;
            if (channels) *channels = ncomp == 1 ? 1 : 3;
            if (!out) { /* header-only call: still look for EXIF, which precedes SOF in practice */
                if (orientation) *orientation = orient;
                rc = 0;
                goto done;
            }
            int mx = (W + 8 * maxh - 1) / (8 * maxh), my = (H + 8 * maxv - 1) / (8 * maxv);
            for (int i = 0; i < ncomp; i++) {
                Comp* c = &comp[i];
                c->bw = mx * c->h;
                c->bh = my * c->v;
                c->dw = (W * c->h + maxh - 1) / maxh;
                c->dh = (H * c->v + maxv - 1) / maxv;
                c->coef = calloc((size_t)c->bw * c->bh * 64, sizeof(int16_t));
                c->plane = malloc((size_t)c->bw * c->bh * 64);
            }
        } else if (m >= 0xC3 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
            rc = E_UNSUPPORTED; /* lossless / differential / arithmetic */
            goto done;
        } else if (m == 0xDD) {
            if (n >= 2) restart = (p[0] << 8) | p[1];
        } else if (m == 0xE1) {
            int o = exif_orientation(p, n);
            if (o) orient = o;
        } else if (m == 0xDA) { /* SOS */
            if (!have_sof || n < 1) { rc = E_CORRUPT; goto done; }
            int ns = p[0];
            if (ns < 1 || ns > ncomp || n < (size_t)(1 + 2 * ns + 3)) { rc = E_CORRUPT; goto done; }
            Comp* sc[4];
            for (int i = 0; i < ns; i++) {
                sc[i] = NULL;
                for (int j = 0; j < ncomp; j++)
                    if (comp[j].id == p[1 + 2 * i]) sc[i] = &comp[j];
                if (!sc[i]) { rc = E_CORRUPT; goto done; }
                sc[i]->td = p[2 + 2 * i] >> 4;
                sc[i]->ta = p[2 + 2 * i] & 15;
                if (sc[i]->td > 3 || sc[i]->ta > 3) { rc = E_CORRUPT; goto done; }
                sc[i]->pred = 0;
            }
            ProgState ps = {p[1 + 2 * ns], p[2 + 2 * ns], p[3 + 2 * ns] >> 4, p[3 + 2 * ns] & 15, 0};
            if (!progressive) {
                ps.Ss = 0; ps.Se = 63; ps.Ah = ps.Al = 0;
            } else if (ps.Ss > ps.Se || ps.Se > 63 || ps.Al > 13 || (ps.Ss == 0 && ps.Se != 0) || (ps.Ss > 0 && ns != 1)) {
                rc = E_CORRUPT; /* G.1.1.1.1: DC scans carry only DC; AC scans are single-component */
                goto done;
            }
            for (int i = 0; i < ns; i++) {
                const int need_dc = !progressive || (ps.Ss == 0 && ps.Ah == 0);
                const int need_ac = !progressive || ps.Ss > 0;
                if ((need_dc && !ht[0][sc[i]->td].present) || (need_ac && !ht[1][sc[i]->ta].present)) { rc = E_CORRUPT; goto done; }
            }
            BitReader b = {in + pos + 2 + seg, in + len, 0, 0, 0};
            int mcux, mcuy;
            if (ns == 1) { /* non-interleaved: one block per MCU over the component's true block grid */
                mcux = (sc[0]->dw + 7) / 8;
                mcuy = (sc[0]->dh + 7) / 8;
            } else {
                mcux = (W + 8 * maxh - 1) / (8 * maxh);
                mcuy = (H + 8 * maxv - 1) / (8 * maxv);
            }
            int todo = restart, rstn = 0;
            for (int my = 0; my < mcuy && !rc; my++)
                for (int mxi = 0; mxi < mcux && !rc; mxi++) {
                    if (restart && todo == 0) {
                        /* byte-align, expect RSTn, reset predictors (T.81 F.2.1.3.1 / E.2.4) */
                        b.acc = 0; b.nbits = 0;
                        const uint8_t* q = b.p;
                        while (q + 1 < b.end && !(q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7)) q++;
                        if (q + 1 >= b.end) { rc = E_CORRUPT; break; }
                        b.p = q + 2;
                        b.hit_marker = 0;
                        rstn = (rstn + 1) & 7;
                        for (int i = 0; i < ns; i++) sc[i]->pred = 0;
                        ps.eobrun = 0;
                        todo = restart;
                    }
                    for (int i = 0; i < ns && !rc; i++) {
                        Comp* c = sc[i];
                        int bh_ = ns == 1 ? 1 : c->h, bv_ = ns == 1 ? 1 : c->v;
                        for (int by = 0; by < bv_ && !rc; by++)
                            for (int bx = 0; bx < bh_ && !rc; bx++) {
                                int X = mxi * bh_ + bx, Y = my * bv_ + by;
                                int16_t* blk = c->coef + ((size_t)Y * c->bw + X) * 64;
                                if (!progressive) rc = decode_block(&b, &ht[0][c->td], &ht[1][c->ta], c, blk);
                                else if (ps.Ss == 0) rc = ps.Ah == 0 ? prog_dc_first(&b, &ht[0][c->td], c, &ps, blk) : prog_dc_refine(&b, &ps, blk);
                                else rc = ps.Ah == 0 ? prog_ac_first(&b, &ht[1][c->ta], &ps, blk) : prog_ac_refine(&b, &ht[1][c->ta], &ps, blk);
                            }
                    }
                    if (restart) todo--;
                }
            if (rc) goto done;
            if (progressive) prog_scans++;
            else scans_done += ns;
            /* continue after the entropy-coded segment: find the next non-RST marker */
            const uint8_t* q = b.p;
            while (q + 1 < b.end && !(q[0] == 0xFF && q[1] != 0x00 && q[1] != 0xFF && !(q[1] >= 0xD0 && q[1] <= 0xD7))) q++;
            pos = (size_t)(q - in);
            if (!progressive && scans_done >= ncomp) break;
            continue; /* progressive: keep reading scans until EOI */
        }
        pos += 2 + seg;
    }
    if (!have_sof) { rc = E_CORRUPT; goto done; }
    if (!out) { if (orientation) *orientation = orient; goto done; }
    if (progressive ? prog_scans == 0 : scans_done < ncomp) { rc = E_TRUNC; goto done; }
    if (orientation) *orientation = orient;
    {
        int och = ncomp == 1 ? 1 : 3;
        if ((size_t)W * H * och > out_cap) { rc = E_SMALL; goto done; }
        for (int i = 0; i < ncomp; i++) {
            Comp* c = &comp[i];
            if (!qpresent[c->tq]) { rc = E_CORRUPT; goto done; }
            for (int by = 0; by < c->bh; by++)
                for (int bx = 0; bx < c->bw; bx++)
                    idct_block(c->coef + ((size_t)by * c->bw + bx) * 64, qt[c->tq],
                               c->plane + ((size_t)by * 8) * (c->bw * 8) + bx * 8, c->bw * 8);
        }
        uint8_t* rows[3];
        for (int i = 0; i < ncomp; i++) rows[i] = malloc((size_t)W + 16);
        for (int y = 0; y < H; y++) {
            for (int i = 0; i < ncomp; i++) upsample_rows(&comp[i], maxh, maxv, y, W, rows[i]);
            uint8_t* o = out + (size_t)y * W * och;
            if (ncomp == 1) {
                memcpy(o, rows[0], W);
            } else {
                for (int x = 0; x < W; x++) { /* jdcolor.c ycc_rgb_convert, JCS_EXT_BGR */
                    int Y = rows[0][x], cb = rows[1][x] - 128, cr = rows[2][x] - 128;
                    int r = Y + ((91881 * cr + 32768) >> 16);
                    int g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
                    int bl = Y + ((116130 * cb + 32768) >> 16);
                    o[3 * x + 0] = (uint8_t)(bl < 0 ? 0 : bl > 255 ? 255 : bl);
                    o[3 * x + 1] = (uint8_t)(g < 0 ? 0 : g > 255 ? 255 : g);
                    o[3 * x + 2] = (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
                }
            }
        }
        for (int i = 0; i < ncomp; i++) free(rows[i]);
    }
done:
    for (int i = 0; i < 4; i++) {
        free(comp[i].coef);
        free(comp[i].plane);
    }
    return rc;
}
