// jpeg_scan_core.h -- Huffman entropy decoding of one JPEG image, shared by the device kernels of jpeg_decode.cu and
// the CPU suite's host build (tests/native/jpeg_scan_sim.cpp).
//
// The bit reader and symbol decoder serve every serial entropy kernel.  The rest decodes a multi-scan file --
// progressive (T.81 Annex G; libjpeg-turbo's jdphuff.c is what the reference runs) or sequential with one scan per
// component -- by walking its scans in order: every scan refines the same coefficients, and inside a scan the
// end-of-band runs chain across blocks, so one thread walks one image.  Restated in oracle/oracle_jpeg_dec.c
// (prog_*), which is pinned on the reference.  The per-image decode also walks a baseline file with restart markers
// here, as one sequential scan (jpeg_baseline_scan).
//
// Coefficients go to the scan order of the parallel decoders ([roi MCU][block in MCU], jpeg_huff_parallel.cu), which
// jpeg_idct_color_kernel reads for every kind of file.  Only blocks inside the region of interest
// keep coefficients.  An AC refinement scan reads one correction bit for every coefficient of its band that is
// already nonzero, and its zero runs skip those coefficients, so a block outside the region keeps a 64-bit mask of
// its nonzero coefficients (bit k = zigzag position k) instead: 8 bytes where the coefficients would take 128.  DC
// scans and sequential blocks outside the region need no state.  Masks are laid out like the parallel decoder's
// DC differences (JpegDecodeItem::dcdiff_off, one entry per block of the whole frame, component by component in
// raster order); a decode whose region is the whole frame needs none.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "jpeg_types.h"

#ifdef LP_JSC_HOST
#define LP_JSC_FN static inline
#else
#define LP_JSC_FN static __host__ __device__ __forceinline__
#endif

namespace lp {

// ------------------------------------------------------------------ bits and symbols

struct BitReader {
    const uint8_t* p;
    const uint8_t* end;
    uint64_t acc;
    int nbits;
    bool marker;
};

LP_JSC_FN void br_fill(BitReader& b) {
    while (b.nbits <= 56) {
        uint32_t byte = 0;
        if (!b.marker && b.p < b.end) {
            byte = *b.p;
            if (byte == 0xFF) {
                const uint8_t* q = b.p + 1;
                while (q < b.end && *q == 0xFF) q++;
                if (q < b.end && *q == 0x00) {
                    b.p = q + 1;  // stuffed FF
                } else {
                    b.marker = true;  // real marker: feed zeros from here on
                    byte = 0;
                }
            } else {
                b.p++;
            }
        }
        b.acc |= (uint64_t)byte << (56 - b.nbits);
        b.nbits += 8;
    }
}

LP_JSC_FN int huff_symbol(BitReader& b, const JpegHuffSet* hs, int t) {
    if (b.nbits < 32) br_fill(b);
    const uint32_t peek = (uint32_t)(b.acc >> 48);
    const uint32_t e = hs->look[t][peek >> 7];
    if (e) {
        const int l = e >> 8;
        b.acc <<= l;
        b.nbits -= l;
        return e & 0xFF;
    }
    int l = 10;
    int code = (int)(peek >> 6);
    while (l <= 16 && code > hs->maxcode[t][l]) {
        l++;
        code = (int)(peek >> (16 - l));
    }
    if (l > 16) return -1;
    b.acc <<= l;
    b.nbits -= l;
    return hs->vals[t][(code + hs->valoffset[t][l]) & 0xFF];
}

LP_JSC_FN int receive_extend(BitReader& b, int n) {
    if (b.nbits < 32) br_fill(b);
    const int v = (int)(b.acc >> (64 - n));
    b.acc <<= n;
    b.nbits -= n;
    return v < (1 << (n - 1)) ? v - (1 << n) + 1 : v;
}

LP_JSC_FN int br_bits(BitReader& b, int n) {
    if (n == 0) return 0;
    if (b.nbits < 32) br_fill(b);
    const int v = (int)(b.acc >> (64 - n));
    b.acc <<= n;
    b.nbits -= n;
    return v;
}

// Byte-align and continue just past the next RSTn marker; false when there is none.
LP_JSC_FN bool br_restart(BitReader& b) {
    b.acc = 0;
    b.nbits = 0;
    const uint8_t* q = b.p;
    while (q + 1 < b.end && !(q[0] == 0xFF && q[1] >= 0xD0 && q[1] <= 0xD7)) q++;
    if (q + 1 >= b.end) return false;
    b.p = q + 2;
    b.marker = false;
    return true;
}

// ------------------------------------------------------------------ block addressing

struct ScanOrder {
    int nb;               // blocks per MCU
    int kfirst[3];        // first block of component c inside a scan-order MCU
    uint32_t mask_off[3]; // first mask of component c (whole-frame block grid)
    uint32_t mask_w[3];   // blocks per row of component c's whole-frame grid
    uint32_t total;       // blocks of the whole frame
};

LP_JSC_FN ScanOrder scan_order(const JpegDecodeItem& it) {
    ScanOrder so{};
    for (int c = 0; c < it.ncomp; c++) {
        so.kfirst[c] = so.nb;
        so.nb += it.h[c] * it.v[c];
        so.mask_off[c] = so.total;
        so.mask_w[c] = (uint32_t)(it.mcus_x * it.h[c]);
        so.total += so.mask_w[c] * (uint32_t)(it.mcus_y * it.v[c]);
    }
    return so;
}

// Blocks of the region of interest (what the scan-order coefficient area holds).
LP_JSC_FN uint32_t roi_blocks(const JpegDecodeItem& it, const ScanOrder& so) {
    return (uint32_t)it.roi_mcx * (uint32_t)it.roi_mcy * (uint32_t)so.nb;
}

LP_JSC_FN bool roi_is_frame(const JpegDecodeItem& it) {
    return it.roi_mx0 == 0 && it.roi_my0 == 0 && it.roi_mcx == it.mcus_x && it.roi_mcy == it.mcus_y;
}

// What one block of a scan updates: its coefficients (inside the region), its nonzero mask (outside), never both.
struct BlockRef {
    int16_t* blk;
    uint64_t* mask;
};

// Block (X, Y) of component c in the component's whole-frame block grid, which is block `sub` (= (Y % v) * h + X % h)
// of MCU (qx, qy) = (X / h, Y / v).
LP_JSC_FN BlockRef block_ref(const JpegDecodeItem& it, const ScanOrder& so, int16_t* coef, uint64_t* masks, int c,
                             int qx, int qy, int sub, int X, int Y) {
    const int mx = qx - it.roi_mx0, my = qy - it.roi_my0;
    BlockRef r{nullptr, nullptr};
    if ((unsigned)mx < (unsigned)it.roi_mcx && (unsigned)my < (unsigned)it.roi_mcy)
        r.blk = coef + it.coef_off + (((size_t)my * it.roi_mcx + mx) * so.nb + so.kfirst[c] + sub) * 64;
    else if (masks)
        r.mask = masks + it.dcdiff_off + so.mask_off[c] + (size_t)Y * so.mask_w[c] + X;
    return r;
}

// kMasks = false: every block lies inside the region (a whole-frame decode), so r.blk is never null.
template <bool kMasks>
LP_JSC_FN bool coef_nonzero(const BlockRef& r, int k, const uint8_t* zz) {
    if (!kMasks) return r.blk[zz[k]] != 0;
    return r.blk ? r.blk[zz[k]] != 0 : (r.mask ? ((*r.mask >> k) & 1) != 0 : false);
}

template <bool kMasks>
LP_JSC_FN void coef_set(const BlockRef& r, int k, int v, const uint8_t* zz) {
    if (!kMasks || r.blk) {
        r.blk[zz[k]] = (int16_t)v;
    } else if (r.mask) {
        const uint64_t bit = 1ull << k;
        *r.mask = (int16_t)v != 0 ? (*r.mask | bit) : (*r.mask & ~bit);
    }
}

// ------------------------------------------------------------------ progressive AC blocks (jdphuff.c)

struct ProgState {
    int Ss, Se, Al;
    unsigned eobrun;
};

template <bool kMasks>
LP_JSC_FN int prog_ac_first(BitReader& b, const JpegHuffSet* hs, int ta, ProgState& ps, const BlockRef& r,
                            const uint8_t* zz) {
    if (ps.eobrun > 0) {
        ps.eobrun--;
        return 0;
    }
    for (int k = ps.Ss; k <= ps.Se; k++) {
        const int rs = huff_symbol(b, hs, ta);
        if (rs < 0) return -3;
        int rr = rs >> 4;
        const int n = rs & 15;
        if (n) {
            k += rr;
            if (k > 63) return -3;
            coef_set<kMasks>(r, k, (int)((unsigned)receive_extend(b, n) << ps.Al), zz);
        } else if (rr == 15) {
            k += 15;
        } else {
            ps.eobrun = 1u << rr;
            if (rr) ps.eobrun += (unsigned)br_bits(b, rr);
            ps.eobrun--;
            break;
        }
    }
    return 0;
}

template <bool kMasks>
LP_JSC_FN void refine_coef(const BlockRef& r, int k, int p1, int m1, const uint8_t* zz) {
    if (kMasks && !r.blk) return;  // a nonzero coefficient stays nonzero
    int16_t* co = r.blk + zz[k];
    if ((*co & p1) == 0) *co = (int16_t)(*co + (*co >= 0 ? p1 : m1));
}

template <bool kMasks>
LP_JSC_FN int prog_ac_refine(BitReader& b, const JpegHuffSet* hs, int ta, ProgState& ps, const BlockRef& r,
                             const uint8_t* zz) {
    const int p1 = 1 << ps.Al, m1 = -(1 << ps.Al);
    int k = ps.Ss;
    if (ps.eobrun == 0) {
        for (; k <= ps.Se; k++) {
            const int rs = huff_symbol(b, hs, ta);
            if (rs < 0) return -3;
            int rr = rs >> 4;
            const int n = rs & 15;
            int val = 0;
            if (n) {
                if (n != 1) return -3;
                val = br_bits(b, 1) ? p1 : m1;
            } else if (rr != 15) {
                ps.eobrun = 1u << rr;
                if (rr) ps.eobrun += (unsigned)br_bits(b, rr);
                break;
            }
            do {
                if (coef_nonzero<kMasks>(r, k, zz)) {
                    if (br_bits(b, 1)) refine_coef<kMasks>(r, k, p1, m1, zz);
                } else {
                    if (--rr < 0) break;
                }
                k++;
            } while (k <= ps.Se);
            if (val) {
                if (k > 63) return -3;
                coef_set<kMasks>(r, k, val, zz);
            }
        }
    }
    if (ps.eobrun > 0) {
        for (; k <= ps.Se; k++)
            if (coef_nonzero<kMasks>(r, k, zz) && br_bits(b, 1)) refine_coef<kMasks>(r, k, p1, m1, zz);
        ps.eobrun--;
    }
    return 0;
}

// ------------------------------------------------------------------ one multi-scan image

template <bool kMasks>
LP_JSC_FN int multiscan_decode_t(const JpegDecodeItem& it, const JpegScanDesc* scans, const JpegHuffSet* sets,
                                 const uint8_t* files, int16_t* coef, uint64_t* masks, const uint8_t* zz) {
    const ScanOrder so = scan_order(it);
    const uint8_t* file = files + it.scan_off;
    int status = 0;
    for (uint32_t s = 0; s < it.nscans && status == 0; s++) {
        const JpegScanDesc sc = scans[it.table_set + s];
        const JpegHuffSet* hs = sets + sc.table_set;
        BitReader b{file + sc.data_off, file + sc.data_off + sc.data_len, 0, 0, false};
        ProgState ps{sc.Ss, sc.Se, sc.Al, 0u};
        int pred[3] = {0, 0, 0};
        int mcux, mcuy;
        if (sc.ns == 1) {  // non-interleaved: one block per MCU over the component's true block grid
            mcux = (it.dw[sc.ci[0]] + 7) / 8;
            mcuy = (it.dh[sc.ci[0]] + 7) / 8;
        } else {
            mcux = it.mcus_x;
            mcuy = it.mcus_y;
        }
        int todo = sc.restart_interval;
        // non-interleaved scans: the MCU (qx, qy) and place in it (sx, sy) of block (mx, my), kept incrementally
        const int h1 = it.h[sc.ci[0]], v1 = it.v[sc.ci[0]];
        int qy = 0, sy = 0;
        for (int my = 0; my < mcuy && status == 0; my++, sy = sy + 1 == v1 ? (qy++, 0) : sy + 1) {
            int qx = 0, sx = 0;
            for (int mx = 0; mx < mcux && status == 0; mx++, sx = sx + 1 == h1 ? (qx++, 0) : sx + 1) {
                if (sc.restart_interval && todo == 0) {
                    if (!br_restart(b)) {
                        status = -3;
                        break;
                    }
                    pred[0] = pred[1] = pred[2] = 0;
                    ps.eobrun = 0;
                    todo = sc.restart_interval;
                }
                for (int i = 0; i < sc.ns && status == 0; i++) {
                    const int c = sc.ci[i];
                    const int bh = sc.ns == 1 ? 1 : it.h[c], bv = sc.ns == 1 ? 1 : it.v[c];
                    const int td = sc.td[i], ta = 4 + sc.ta[i];
                    for (int by = 0; by < bv && status == 0; by++) {
                        for (int bx = 0; bx < bh && status == 0; bx++) {
                            const BlockRef r = sc.ns == 1 ? block_ref(it, so, coef, masks, c, qx, qy, sy * h1 + sx, mx, my)
                                                          : block_ref(it, so, coef, masks, c, mx, my, by * bh + bx,
                                                                      mx * bh + bx, my * bv + by);
                            if (!sc.progressive) {  // sequential block: DC difference + AC run/size pairs
                                const int sz = huff_symbol(b, hs, td);
                                if (sz < 0 || sz > 15) { status = -3; break; }
                                if (sz) pred[i] += receive_extend(b, sz);
                                if (r.blk) r.blk[0] = (int16_t)pred[i];
                                for (int k = 1; k < 64;) {
                                    const int rs = huff_symbol(b, hs, ta);
                                    if (rs < 0) { status = -3; break; }
                                    const int rr = rs >> 4, n = rs & 15;
                                    if (n == 0) {
                                        if (rr != 15) break;
                                        k += 16;
                                        continue;
                                    }
                                    k += rr;
                                    if (k > 63) { status = -3; break; }
                                    const int val = receive_extend(b, n);
                                    if (r.blk) r.blk[zz[k]] = (int16_t)val;
                                    k++;
                                }
                            } else if (sc.Ss == 0) {
                                if (sc.Ah == 0) {  // DC first pass
                                    const int sz = huff_symbol(b, hs, td);
                                    if (sz < 0 || sz > 15) { status = -3; break; }
                                    if (sz) pred[i] += receive_extend(b, sz);
                                    if (r.blk) r.blk[0] = (int16_t)((unsigned)pred[i] << sc.Al);
                                } else if (br_bits(b, 1)) {  // DC refinement
                                    if (r.blk) r.blk[0] |= (int16_t)(1 << sc.Al);
                                }
                            } else {
                                status = sc.Ah == 0 ? prog_ac_first<kMasks>(b, hs, ta, ps, r, zz)
                                                    : prog_ac_refine<kMasks>(b, hs, ta, ps, r, zz);
                            }
                        }
                    }
                }
                if (sc.restart_interval) todo--;
            }
        }
    }
    return status;
}

// Decodes every scan of a multi-scan item (it.nscans scans from scans[it.table_set]) into its zeroed ROI blocks
// and zeroed masks.  `files` + it.scan_off is the item's whole file; table sets index `sets`; zz is the zigzag
// order.  Returns 0, or -3 for a damaged stream.
LP_JSC_FN int multiscan_decode(const JpegDecodeItem& it, const JpegScanDesc* scans, const JpegHuffSet* sets,
                               const uint8_t* files, int16_t* coef, uint64_t* masks, const uint8_t* zz) {
    if (roi_is_frame(it)) return multiscan_decode_t<false>(it, scans, sets, files, coef, nullptr, zz);
    if (!masks) return -3;  // refinement outside the region needs the masks
    return multiscan_decode_t<true>(it, scans, sets, files, coef, masks, zz);
}

}  // namespace lp
