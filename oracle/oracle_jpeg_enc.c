/*
 * oracle_jpeg_enc.c -- CPU restatement of baseline JPEG encoding as the reference
 * performs it.  TEST INFRASTRUCTURE ONLY (see oracle.h).
 *
 * Reference call site: opencv_encoder_write (ref opencv.cpp:185-194) ->
 * cv::ImageEncoder::write -> libjpeg-turbo 3.1.0 defaults (jpeg_set_defaults +
 * jpeg_set_quality(q, TRUE)): JFIF APP0, 4:2:0, Annex-K quantisation tables scaled
 * by quality, Annex-K Huffman tables, JDCT_ISLOW, no restart markers, no
 * optimisation.  Restated from ITU-T T.81 and libjpeg-turbo's published
 * jccolor.c / jcsample.c / jfdctint.c / jcdctmgr.c / jccoefct.c / jchuff.c /
 * jcmarker.c as summarised in SURVEY.md Appendix E.3.
 * Pinned byte-for-byte against libjpeg-turbo (through cv2) in tests/test_oracle_jpeg_encode.py.
 */
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

static const uint8_t ZIGZAG[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                   12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                   58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

/* T.81 Annex K.1 (natural order) */
static const uint8_t STD_LUMA_Q[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                       14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                       18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                       49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
static const uint8_t STD_CHROMA_Q[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                                         24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
                                         99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                         99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
/* T.81 Annex K.3 */
static const uint8_t DC_L_BITS[17] = {0, 0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
static const uint8_t DC_C_BITS[17] = {0, 0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
static const uint8_t DC_VALS[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t AC_L_BITS[17] = {0, 0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
static const uint8_t AC_L_VALS[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71,
    0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72,
    0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37,
    0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
    0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83,
    0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3,
    0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
    0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
static const uint8_t AC_C_BITS[17] = {0, 0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
static const uint8_t AC_C_VALS[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22,
    0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1,
    0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36,
    0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
    0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a,
    0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a,
    0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba,
    0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
    0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

typedef struct { uint16_t code[256]; uint8_t size[256]; } EncTable;

static void build_enc(const uint8_t* bits, const uint8_t* vals, EncTable* t) {
    memset(t, 0, sizeof(*t));
    unsigned code = 0;
    int k = 0;
    for (int len = 1; len <= 16; len++) {
        for (int i = 0; i < bits[len]; i++, k++) {
            t->code[vals[k]] = (uint16_t)code++;
            t->size[vals[k]] = (uint8_t)len;
        }
        code <<= 1;
    }
}

typedef struct { uint8_t* p; uint8_t* end; uint64_t acc; int n; int overflow; } BitWriter;

static void bw_byte(BitWriter* w, unsigned b) {
    if (w->p < w->end) *w->p++ = (uint8_t)b; else w->overflow = 1;
}
static void bw_put(BitWriter* w, unsigned code, int size) {
    w->acc = (w->acc << size) | (code & ((1u << size) - 1));
    w->n += size;
    while (w->n >= 8) {
        unsigned b = (unsigned)(w->acc >> (w->n - 8)) & 0xFF;
        bw_byte(w, b);
        if (b == 0xFF) bw_byte(w, 0);
        w->n -= 8;
    }
}
static void bw_flush(BitWriter* w) {
    if (w->n > 0) bw_put(w, 0x7F, 8 - w->n); /* pad the last byte with 1-bits */
}

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

/* jpeg_fdct_islow: rows then columns, output scaled by 8. */
static void fdct_islow(int* d) {
    for (int pass = 0; pass < 2; pass++) {
        for (int i = 0; i < 8; i++) {
            int* p = pass == 0 ? d + i * 8 : d + i;
            int st = pass == 0 ? 1 : 8;
            int tmp0 = p[0] + p[7 * st], tmp7 = p[0] - p[7 * st];
            int tmp1 = p[st] + p[6 * st], tmp6 = p[st] - p[6 * st];
            int tmp2 = p[2 * st] + p[5 * st], tmp5 = p[2 * st] - p[5 * st];
            int tmp3 = p[3 * st] + p[4 * st], tmp4 = p[3 * st] - p[4 * st];
            int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
            int z1 = (tmp12 + tmp13) * FIX_0_541196100;
            if (pass == 0) {
                p[0] = (tmp10 + tmp11) << 2;
                p[4 * st] = (tmp10 - tmp11) << 2;
                p[2 * st] = DESCALE(z1 + tmp13 * FIX_0_765366865, 11);
                p[6 * st] = DESCALE(z1 + tmp12 * (-FIX_1_847759065), 11);
            } else {
                p[0] = DESCALE(tmp10 + tmp11, 2);
                p[4 * st] = DESCALE(tmp10 - tmp11, 2);
                p[2 * st] = DESCALE(z1 + tmp13 * FIX_0_765366865, 15);
                p[6 * st] = DESCALE(z1 + tmp12 * (-FIX_1_847759065), 15);
            }
            z1 = tmp4 + tmp7;
            int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
            int z5 = (z3 + z4) * FIX_1_175875602;
            tmp4 *= FIX_0_298631336;
            tmp5 *= FIX_2_053119869;
            tmp6 *= FIX_3_072711026;
            tmp7 *= FIX_1_501321110;
            z1 *= -FIX_0_899976223;
            z2 *= -FIX_2_562915447;
            z3 *= -FIX_1_961570560;
            z4 *= -FIX_0_390180644;
            z3 += z5;
            z4 += z5;
            int sh = pass == 0 ? 11 : 15;
            p[7 * st] = DESCALE(tmp4 + z1 + z3, sh);
            p[5 * st] = DESCALE(tmp5 + z2 + z4, sh);
            p[3 * st] = DESCALE(tmp6 + z2 + z3, sh);
            p[st] = DESCALE(tmp7 + z1 + z4, sh);
        }
    }
}

/* one block: samples (already edge-expanded plane) -> quantised coefficients, natural order */
static void block_fdct_quant(const uint8_t* s, int stride, const uint16_t* q, int16_t* out) {
    int d[64];
    for (int y = 0; y < 8; y++)
        for (int x = 0; x < 8; x++) d[y * 8 + x] = (int)s[y * stride + x] - 128;
    fdct_islow(d);
    for (int i = 0; i < 64; i++) {
        int q8 = q[i] << 3, c = d[i];
        int a = c < 0 ? -c : c;
        a = (a + (q8 >> 1)) / q8;
        out[i] = (int16_t)(c < 0 ? -a : a);
    }
}

static int nbits_of(int v) {
    int n = 0;
    while (v) { n++; v >>= 1; }
    return n;
}

static void encode_block(BitWriter* w, const int16_t* blk, int* pred, const EncTable* dc, const EncTable* ac) {
    int diff = blk[0] - *pred;
    *pred = blk[0];
    int t = diff < 0 ? -diff : diff, t2 = diff < 0 ? diff - 1 : diff;
    int n = nbits_of(t);
    bw_put(w, dc->code[n], dc->size[n]);
    if (n) bw_put(w, (unsigned)t2, n);
    int r = 0;
    for (int k = 1; k < 64; k++) {
        int v = blk[ZIGZAG[k]];
        if (v == 0) { r++; continue; }
        while (r > 15) { bw_put(w, ac->code[0xF0], ac->size[0xF0]); r -= 16; }
        t = v < 0 ? -v : v;
        t2 = v < 0 ? v - 1 : v;
        n = nbits_of(t);
        int sym = (r << 4) + n;
        bw_put(w, ac->code[sym], ac->size[sym]);
        bw_put(w, (unsigned)t2, n);
        r = 0;
    }
    if (r > 0) bw_put(w, ac->code[0], ac->size[0]);
}

static uint8_t* put_marker(uint8_t* p, int m, int len) {
    *p++ = 0xFF; *p++ = (uint8_t)m; *p++ = (uint8_t)(len >> 8); *p++ = (uint8_t)len;
    return p;
}
static uint8_t* put_dht(uint8_t* p, int tc_th, const uint8_t* bits, const uint8_t* vals) {
    int total = 0;
    for (int i = 1; i <= 16; i++) total += bits[i];
    p = put_marker(p, 0xC4, 2 + 1 + 16 + total);
    *p++ = (uint8_t)tc_th;
    memcpy(p, bits + 1, 16); p += 16;
    memcpy(p, vals, total); p += total;
    return p;
}

size_t oracle_jpeg_encode(const uint8_t* px, size_t step, int W, int H, int cn, int quality,
                          uint8_t* out, size_t out_cap) {
    if (W < 1 || H < 1 || W > 65535 || H > 65535 || (cn != 1 && cn != 3 && cn != 4)) return 0;
    if (out_cap < 1024) return 0;
    int gray = cn == 1;
    /* jpeg_quality_scaling + jpeg_add_quant_table(force_baseline) */
    if (quality <= 0) quality = 1;
    if (quality > 100) quality = 100;
    int scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
    uint16_t q[2][64];
    for (int i = 0; i < 64; i++) {
        long a = ((long)STD_LUMA_Q[i] * scale + 50) / 100, b = ((long)STD_CHROMA_Q[i] * scale + 50) / 100;
        q[0][i] = (uint16_t)(a < 1 ? 1 : a > 255 ? 255 : a);
        q[1][i] = (uint16_t)(b < 1 ? 1 : b > 255 ? 255 : b);
    }
    /* headers (jcmarker.c order) */
    uint8_t* p = out;
    *p++ = 0xFF; *p++ = 0xD8;
    p = put_marker(p, 0xE0, 16);
    memcpy(p, "JFIF\0\1\1\0\0\1\0\1\0\0", 14); p += 14;
    for (int t = 0; t < (gray ? 1 : 2); t++) {
        p = put_marker(p, 0xDB, 67);
        *p++ = (uint8_t)t;
        for (int i = 0; i < 64; i++) *p++ = (uint8_t)q[t][ZIGZAG[i]];
    }
    p = put_marker(p, 0xC0, 8 + 3 * (gray ? 1 : 3));
    *p++ = 8; *p++ = (uint8_t)(H >> 8); *p++ = (uint8_t)H; *p++ = (uint8_t)(W >> 8); *p++ = (uint8_t)W;
    *p++ = (uint8_t)(gray ? 1 : 3);
    if (gray) { *p++ = 1; *p++ = 0x11; *p++ = 0; }
    else { *p++ = 1; *p++ = 0x22; *p++ = 0; *p++ = 2; *p++ = 0x11; *p++ = 1; *p++ = 3; *p++ = 0x11; *p++ = 1; }
    p = put_dht(p, 0x00, DC_L_BITS, DC_VALS);
    p = put_dht(p, 0x10, AC_L_BITS, AC_L_VALS);
    if (!gray) {
        p = put_dht(p, 0x01, DC_C_BITS, DC_VALS);
        p = put_dht(p, 0x11, AC_C_BITS, AC_C_VALS);
    }
    p = put_marker(p, 0xDA, 6 + 2 * (gray ? 1 : 3));
    *p++ = (uint8_t)(gray ? 1 : 3);
    *p++ = 1; *p++ = 0x00;
    if (!gray) { *p++ = 2; *p++ = 0x11; *p++ = 3; *p++ = 0x11; }
    *p++ = 0; *p++ = 63; *p++ = 0;

    /* planes, edge-expanded the way jcprepct.c/jcsample.c leave them */
    int hs = gray ? 1 : 2, vs = gray ? 1 : 2;
    int mcux = (W + 8 * hs - 1) / (8 * hs), mcuy = (H + 8 * vs - 1) / (8 * vs);
    int yw = mcux * hs * 8, yh = mcuy * vs * 8;       /* luma plane, padded to the MCU grid */
    int ybw = (W + 7) / 8, ybh = (H + 7) / 8;         /* real luma blocks (width/height_in_blocks) */
    uint8_t* Yp = malloc((size_t)yw * yh);
    uint8_t *Cbp = NULL, *Crp = NULL;
    int cw = mcux * 8, chh = mcuy * 8;
    int cdw = (W + 1) / 2, cdh = (H + 1) / 2; /* true downsampled chroma size */
    if (!gray) { Cbp = malloc((size_t)cw * chh); Crp = malloc((size_t)cw * chh); }
    {
        /* full-resolution chroma rows, replicated right to 2*cw and bottom to even height */
        int fw = 2 * cw, fh = 2 * cdh;
        uint8_t *Fb = NULL, *Fr = NULL;
        if (!gray) { Fb = malloc((size_t)fw * fh); Fr = malloc((size_t)fw * fh); }
        for (int y = 0; y < H; y++) {
            const uint8_t* s = px + (size_t)y * step;
            for (int x = 0; x < W; x++) {
                if (gray) { Yp[(size_t)y * yw + x] = s[x]; continue; }
                int b = s[x * cn], g = s[x * cn + 1], r = s[x * cn + 2];
                /* jccolor.c rgb_ycc_convert */
                Yp[(size_t)y * yw + x] = (uint8_t)((19595 * r + 38470 * g + 7471 * b + 32768) >> 16);
                Fb[(size_t)y * fw + x] = (uint8_t)((-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16);
                Fr[(size_t)y * fw + x] = (uint8_t)((32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16);
            }
            for (int x = W; x < yw; x++) Yp[(size_t)y * yw + x] = Yp[(size_t)y * yw + W - 1];
            if (!gray)
                for (int x = W; x < fw; x++) {
                    Fb[(size_t)y * fw + x] = Fb[(size_t)y * fw + W - 1];
                    Fr[(size_t)y * fw + x] = Fr[(size_t)y * fw + W - 1];
                }
        }
        for (int y = H; y < yh; y++) memcpy(Yp + (size_t)y * yw, Yp + (size_t)(H - 1) * yw, yw);
        if (!gray) {
            for (int y = H; y < fh; y++) {
                memcpy(Fb + (size_t)y * fw, Fb + (size_t)(H - 1) * fw, fw);
                memcpy(Fr + (size_t)y * fw, Fr + (size_t)(H - 1) * fw, fw);
            }
            /* h2v2_downsample: bias alternates 1,2,1,2 by output column */
            for (int y = 0; y < cdh; y++)
                for (int x = 0; x < cw; x++) {
                    int bias = 1 + (x & 1);
                    const uint8_t* a = Fb + (size_t)(2 * y) * fw + 2 * x;
                    const uint8_t* c = Fr + (size_t)(2 * y) * fw + 2 * x;
                    Cbp[(size_t)y * cw + x] = (uint8_t)((a[0] + a[1] + a[fw] + a[fw + 1] + bias) >> 2);
                    Crp[(size_t)y * cw + x] = (uint8_t)((c[0] + c[1] + c[fw] + c[fw + 1] + bias) >> 2);
                }
            /* downsampled last row replicated down to the iMCU height */
            for (int y = cdh; y < chh; y++) {
                memcpy(Cbp + (size_t)y * cw, Cbp + (size_t)(cdh - 1) * cw, cw);
                memcpy(Crp + (size_t)y * cw, Crp + (size_t)(cdh - 1) * cw, cw);
            }
            free(Fb); free(Fr);
        }
        (void)cdw;
    }

    EncTable dcl, acl, dcc, acc;
    build_enc(DC_L_BITS, DC_VALS, &dcl);
    build_enc(AC_L_BITS, AC_L_VALS, &acl);
    build_enc(DC_C_BITS, DC_VALS, &dcc);
    build_enc(AC_C_BITS, AC_C_VALS, &acc);
    BitWriter w = {p, out + out_cap - 2, 0, 0, 0};
    int pred[3] = {0, 0, 0};
    for (int my = 0; my < mcuy; my++)
        for (int mx = 0; mx < mcux; mx++) {
            int16_t blk[6][64];
            int nb = 0;
            /* luma blocks; dummy blocks (jccoefct.c): AC = 0, DC = DC of the previous block in the MCU */
            for (int by = 0; by < vs; by++)
                for (int bx = 0; bx < hs; bx++, nb++) {
                    int X = mx * hs + bx, Y = my * vs + by;
                    if (X < ybw && Y < ybh) {
                        block_fdct_quant(Yp + (size_t)Y * 8 * yw + X * 8, yw, q[0], blk[nb]);
                    } else {
                        memset(blk[nb], 0, sizeof(blk[nb]));
                        blk[nb][0] = blk[nb - 1][0];
                    }
                }
            for (int i = 0; i < nb; i++) encode_block(&w, blk[i], &pred[0], &dcl, &acl);
            if (!gray) {
                block_fdct_quant(Cbp + (size_t)my * 8 * cw + mx * 8, cw, q[1], blk[0]);
                encode_block(&w, blk[0], &pred[1], &dcc, &acc);
                block_fdct_quant(Crp + (size_t)my * 8 * cw + mx * 8, cw, q[1], blk[0]);
                encode_block(&w, blk[0], &pred[2], &dcc, &acc);
            }
        }
    bw_flush(&w);
    free(Yp); free(Cbp); free(Crp);
    if (w.overflow) return 0;
    *w.p++ = 0xFF; *w.p++ = 0xD9;
    return (size_t)(w.p - out);
}
