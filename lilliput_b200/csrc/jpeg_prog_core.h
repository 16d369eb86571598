// jpeg_prog_core.h -- progressive JPEG entropy coding (T.81 Annex G, Huffman), written once for host and device.
//
// What libjpeg-turbo's jcphuff.c writes when OpenCV asks for IMWRITE_JPEG_PROGRESSIVE: jpeg_simple_progression's scan
// script, successive approximation, EOB runs, and (progressive mode forces optimize_coding) one optimal Huffman table
// per table a scan uses, built by jpeg_gen_optimal_table.  The input is the quantised coefficient layout of
// jpeg_encode.cu: [mcu][block-in-mcu][64] int16 in zig-zag order, dummy luma blocks all zero.
//
// A scan is coded block by block.  code_block() produces one block's share of the stream: its own symbols, then, if
// the block is the first of an EOB run, that run's EOB symbol, then the correction bits the run buffers for it.  This
// is the order jcphuff.c writes them in, so a scan is the concatenation of its blocks' shares once resolve_runs() has
// said where each run starts and how long it is.  Callers use it three times per scan: gathering symbol counts,
// sizing each block with the optimal tables, and writing.
//
// jpeg_encode.cu runs it on the device (one CTA per image, the blocks of a scan across the CTA);
// tests/native/jpeg_prog_sim.cpp builds whole files with it on the host.
#pragma once
#include <stddef.h>
#include <stdint.h>

#ifdef __CUDACC__
#define JPROG_HD __host__ __device__ __forceinline__
#else
#define JPROG_HD inline
#endif

namespace jprog {

// One scan of the script.  comp < 0: all components (the interleaved DC scans).
struct Scan {
    int comp, Ss, Se, Ah, Al;
};

constexpr int kColorScans = 10, kGrayScans = 6;
constexpr int kMaxCorrBits = 1000;  // jcphuff.c MAX_CORR_BITS

// jcparam.c jpeg_simple_progression: the YCbCr script, and the generic one for a single component.
JPROG_HD Scan scan_of(bool gray, int s) {
    const int8_t color[kColorScans][5] = {{-1, 0, 0, 0, 1}, {0, 1, 5, 0, 2},  {2, 1, 63, 0, 1}, {1, 1, 63, 0, 1},
                                          {0, 6, 63, 0, 2}, {0, 1, 63, 2, 1}, {-1, 0, 0, 1, 0}, {2, 1, 63, 1, 0},
                                          {1, 1, 63, 1, 0}, {0, 1, 63, 1, 0}};
    const int8_t mono[kGrayScans][5] = {{0, 0, 0, 0, 1}, {0, 1, 5, 0, 2}, {0, 6, 63, 0, 2},
                                        {0, 1, 63, 2, 1}, {0, 0, 0, 1, 0}, {0, 1, 63, 1, 0}};
    const int8_t* t = gray ? mono[s] : color[s];
    return Scan{t[0], t[1], t[2], t[3], t[4]};
}

// Huffman tables a scan uses: DC first scans of colour images use two (luma, chroma), DC refinement none.
JPROG_HD int scan_tables(bool gray, const Scan& s) {
    if (s.Ss == 0) return s.Ah ? 0 : (gray ? 1 : 2);
    return 1;
}

// Geometry of the coefficient layout.  Gray: one block per MCU.  Colour: 4:2:0, blocks 0..3 luma, 4 Cb, 5 Cr.
struct Geom {
    int mcus_x, mcus_y;
    int bpm;       // blocks per MCU (1 or 6)
    int ybw, ybh;  // real luma blocks: ceil(W/8) x ceil(H/8)
};

// Blocks a scan walks: interleaved scans every block of every MCU (dummy blocks too), single-component scans only
// that component's real blocks.
JPROG_HD int scan_blocks(const Geom& g, const Scan& s) {
    if (g.bpm == 1) return g.mcus_x * g.mcus_y;
    if (s.comp < 0) return g.mcus_x * g.mcus_y * 6;
    if (s.comp == 0) return g.ybw * g.ybh;
    return g.mcus_x * g.mcus_y;
}

// Block i of a scan -> (mcu, block in mcu).  A luma scan walks the luma block grid in raster order.
JPROG_HD void scan_block(const Geom& g, const Scan& s, int i, int* mcu, int* k) {
    if (g.bpm == 1) {
        *mcu = i;
        *k = 0;
    } else if (s.comp < 0) {
        *mcu = i / 6;
        *k = i % 6;
    } else if (s.comp > 0) {
        *mcu = i;
        *k = 3 + s.comp;
    } else {
        const int bx = i % g.ybw, by = i / g.ybw;
        *mcu = (by >> 1) * g.mcus_x + (bx >> 1);
        *k = ((by & 1) << 1) | (bx & 1);
    }
}

JPROG_HD bool is_dummy(const Geom& g, int mcu, int k) {
    if (g.bpm == 1 || k >= 4) return false;
    const int mx = mcu % g.mcus_x, my = mcu / g.mcus_x;
    return mx * 2 + (k & 1) >= g.ybw || my * 2 + (k >> 1) >= g.ybh;
}

// Quantised DC of a block; a dummy block carries the DC of the block before it in the MCU (jccoefct.c).
JPROG_HD int dc_of(const int16_t* coef, const Geom& g, int mcu, int k) {
    while (k > 0 && is_dummy(g, mcu, k)) k--;
    return coef[((size_t)mcu * g.bpm + k) * 64];
}

JPROG_HD int nbits(unsigned v) {
    int n = 0;
    while (v) {
        n++;
        v >>= 1;
    }
    return n;
}

// code_block's summary of a block for resolve_runs.
constexpr uint32_t kCoded = 1u << 31;  // the block codes a coefficient: a pending EOB run ends before it
constexpr uint32_t kTrail = 1u << 30;  // the block ends inside an EOB run (trailing zeros or correction bits)
constexpr uint32_t kCorrMask = 127;    // correction bits the block adds to that run

// Emitter interface: e.sym(table, symbol) for a Huffman symbol of the scan's table 0 or 1, e.bits(value, n) for n <= 16
// raw bits (the low n bits of value).
template <class E>
JPROG_HD void put_bits64(E& e, uint64_t v, int n) {
    while (n > 16) {
        n -= 16;
        e.bits((uint32_t)(v >> n), 16);
    }
    if (n) e.bits((uint32_t)v, n);
}

// EOB run of length run (1..0x7FFF): symbol (log2(run) << 4), then the bits below the leading one.
template <class E>
JPROG_HD void put_eobrun(E& e, int run) {
    const int nb = nbits((unsigned)run) - 1;
    e.sym(0, nb << 4);
    if (nb) e.bits((uint32_t)run, nb);
}

// Block i of scan s.  run: length of the EOB run that starts at this block (0 if none; from resolve_runs).
// Returns the block's summary (AC scans; 0 for DC scans).
template <class E>
JPROG_HD uint32_t code_block(const int16_t* coef, const Geom& g, const Scan& s, int i, int run, E& e) {
    int mcu, k;
    scan_block(g, s, i, &mcu, &k);
    if (s.Ss == 0) {
        const int v = dc_of(coef, g, mcu, k) >> s.Al;  // arithmetic shift (jcphuff.c IRIGHT_SHIFT)
        if (s.Ah) {
            e.bits((uint32_t)v & 1, 1);
            return 0;
        }
        // prediction: the previous block of the same component in scan order
        int pm = mcu, pk = k;
        if (g.bpm == 1 || k >= 4) pm--;
        else if (k > 0) pk--;
        else pm--, pk = 3;
        const int pred = pm >= 0 ? dc_of(coef, g, pm, pk) >> s.Al : 0;
        const int diff = v - pred;
        const int n = nbits((unsigned)(diff < 0 ? -diff : diff));
        e.sym(g.bpm == 6 && k >= 4 ? 1 : 0, n);
        if (n) e.bits((uint32_t)(diff < 0 ? diff - 1 : diff), n);
        return 0;
    }
    const int16_t* blk = coef + ((size_t)mcu * g.bpm + k) * 64;
    int r = 0;
    uint32_t f = 0;
    if (s.Ah == 0) {  // AC first: magnitudes shifted by Al
        for (int z = s.Ss; z <= s.Se; z++) {
            const int v = blk[z];
            const int a = (v < 0 ? -v : v) >> s.Al;
            if (a == 0) {
                r++;
                continue;
            }
            while (r > 15) {
                e.sym(0, 0xF0);
                r -= 16;
            }
            const int n = nbits((unsigned)a);
            e.sym(0, (r << 4) + n);
            e.bits((uint32_t)(v < 0 ? ~a : a), n);
            r = 0;
            f = kCoded;
        }
        if (run) put_eobrun(e, run);
        return f | (r > 0 ? kTrail : 0);
    }
    // AC refinement: newly nonzero coefficients (magnitude 1 after the shift) are coded with a sign bit; every
    // coefficient already nonzero contributes one correction bit, buffered until the next symbol.
    int eob = 0;
    for (int z = s.Ss; z <= s.Se; z++) {
        const int v = blk[z];
        if (((v < 0 ? -v : v) >> s.Al) == 1) eob = z;
    }
    uint64_t buf = 0;
    int br = 0;
    for (int z = s.Ss; z <= s.Se; z++) {
        const int v = blk[z];
        const int a = (v < 0 ? -v : v) >> s.Al;
        if (a == 0) {
            r++;
            continue;
        }
        while (r > 15 && z <= eob) {
            e.sym(0, 0xF0);
            r -= 16;
            put_bits64(e, buf, br);
            buf = 0;
            br = 0;
        }
        if (a > 1) {
            buf = (buf << 1) | (uint64_t)(a & 1);
            br++;
            continue;
        }
        e.sym(0, (r << 4) + 1);
        e.bits(v < 0 ? 0u : 1u, 1);
        put_bits64(e, buf, br);
        buf = 0;
        br = 0;
        r = 0;
        f = kCoded;
    }
    if (run) put_eobrun(e, run);
    put_bits64(e, buf, br);
    return f | (r > 0 || br > 0 ? kTrail : 0) | (uint32_t)br;
}

// jcphuff.c's EOB-run rules over the summaries of an AC scan's n blocks: a run ends before a block that codes a
// coefficient, when it reaches 0x7FFF blocks, when its buffered correction bits pass MAX_CORR_BITS - 63, and at the
// end of the scan.  Calls at(first_block, length) for every run.
template <class F>
JPROG_HD void resolve_runs(const uint32_t* summ, int n, F&& at) {
    int run = 0, be = 0, start = 0;
    for (int i = 0; i < n; i++) {
        const uint32_t s = summ[i];
        if (s & kCoded) {
            if (run) at(start, run);
            run = 0;
            be = 0;
            if (s & kTrail) {
                start = i;
                run = 1;
                be = (int)(s & kCorrMask);
            }
        } else {
            if (run == 0) start = i;
            run++;
            be += (int)(s & kCorrMask);
        }
        if (run == 0x7FFF || be > kMaxCorrBits - 63) {
            at(start, run);
            run = 0;
            be = 0;
        }
    }
    if (run) at(start, run);
}

// Lanes of a cooperative group for the table builder: the host runs it with one lane, the device with a warp.
struct OneLane {
    JPROG_HD int lane() const { return 0; }
    JPROG_HD int lanes() const { return 1; }
    JPROG_HD void sync() const {}
    JPROG_HD uint64_t min(uint64_t v) const { return v; }
};

JPROG_HD uint64_t merge_key(uint32_t freq, int sym) { return ((uint64_t)freq << 9) | (uint64_t)(511 - sym); }
JPROG_HD uint64_t min_u64(uint64_t a, uint64_t b) { return a < b ? a : b; }

// jchuff.c jpeg_gen_optimal_table: T.81 K.2 with a reserved symbol 256 of count 1, ties going to the larger symbol,
// K.3 length limiting to 16 bits, values listed by code length then symbol.  freq[257] is consumed; codesize[257] and
// tree[257] are work arrays shared by the group.  Writes bits[1..16] and vals; returns the number of values, or -1
// where libjpeg gives up (a code longer than 32 bits).
template <class G>
JPROG_HD int gen_optimal_table(const G& g, uint32_t* freq, int* codesize, int* tree, uint8_t* bits, uint8_t* vals) {
    for (int i = g.lane(); i < 257; i += g.lanes()) {
        codesize[i] = 0;
        tree[i] = i;
    }
    if (g.lane() == 0) freq[256] = 1;
    g.sync();
    // Each merge joins the trees rooted at c1 (the smallest count) and c2 (the next): every member's code grows by
    // one bit.  Keys order by count, then by larger symbol.
    for (;;) {
        uint64_t k1 = ~0ull;
        for (int i = g.lane(); i < 257; i += g.lanes())
            if (freq[i]) k1 = min_u64(k1, merge_key(freq[i], i));
        k1 = g.min(k1);
        const int c1 = 511 - (int)(k1 & 511);
        uint64_t k2 = ~0ull;
        for (int i = g.lane(); i < 257; i += g.lanes())
            if (freq[i] && i != c1) k2 = min_u64(k2, merge_key(freq[i], i));
        k2 = g.min(k2);
        if (k2 == ~0ull) break;
        const int c2 = 511 - (int)(k2 & 511);
        g.sync();
        for (int i = g.lane(); i < 257; i += g.lanes()) {
            const int t = tree[i];
            if (t == c1 || t == c2) {
                codesize[i]++;
                tree[i] = c1;
            }
        }
        if (g.lane() == 0) {
            freq[c1] += freq[c2];
            freq[c2] = 0;
        }
        g.sync();
    }
    int ok = 1;
    if (g.lane() == 0) {
        int cnt[33] = {0};
        for (int i = 0; i <= 256; i++) {
            if (codesize[i] > 32) ok = 0;
            else if (codesize[i]) cnt[codesize[i]]++;
        }
        int pos[33];
        pos[0] = 0;
        for (int l = 1; l <= 32; l++) pos[l] = pos[l - 1] + (l > 1 ? cnt[l - 1] : 0);
        for (int j = 0; j < 256 && ok; j++)
            if (codesize[j]) vals[pos[codesize[j]]++] = (uint8_t)j;
        int i = 32;
        for (; i > 16; i--) {
            while (cnt[i] > 0) {
                int j = i - 2;
                while (cnt[j] == 0) j--;
                cnt[i] -= 2;
                cnt[i - 1]++;
                cnt[j + 1] += 2;
                cnt[j]--;
            }
        }
        while (cnt[i] == 0) i--;
        cnt[i]--;  // the reserved symbol
        bits[0] = 0;
        for (int l = 1; l <= 16; l++) bits[l] = (uint8_t)cnt[l];
        codesize[256] = 0;
        for (int l = 1; l <= 16; l++) codesize[256] += cnt[l];  // hand the count back through the shared array
        if (!ok) codesize[256] = -1;
    }
    g.sync();
    const int n = codesize[256];
    g.sync();
    return n;
}

// Canonical codes (T.81 C.2): huff[symbol] = (length << 16) | code.
JPROG_HD void make_codes(const uint8_t* bits, const uint8_t* vals, uint32_t* huff) {
    for (int i = 0; i < 256; i++) huff[i] = 0;
    unsigned code = 0;
    int k = 0;
    for (int len = 1; len <= 16; len++) {
        for (int i = 0; i < bits[len]; i++, k++) huff[vals[k]] = ((uint32_t)len << 16) | code++;
        code <<= 1;
    }
}

// Frame header: the baseline encoder's SOI, APP0 and DQT bytes, then its SOF0 with the marker changed to SOF2.
JPROG_HD int frame_len(bool gray) { return 2 + 18 + 69 * (gray ? 1 : 2) + 10 + 3 * (gray ? 1 : 3); }
JPROG_HD int sof_type_at(bool gray) { return frame_len(gray) - (10 + 3 * (gray ? 1 : 3)) + 1; }

// Length of put_scan_header's output.
JPROG_HD int scan_header_len(bool gray, const Scan& s, const uint8_t (*bits)[17]) {
    int n = 2 + 6 + 2 * (s.comp < 0 && !gray ? 3 : 1);
    for (int t = 0; t < scan_tables(gray, s); t++) {
        n += 4 + 1 + 16;
        for (int l = 1; l <= 16; l++) n += bits[t][l];
    }
    return n;
}

// The DHT segments of a scan's tables (bits[t], vals[t], t < scan_tables) and its SOS, as jcmarker.c writes them.
// Returns the bytes written (scan_header_len).
JPROG_HD int put_scan_header(uint8_t* p, bool gray, const Scan& s, const uint8_t (*bits)[17], const uint8_t (*vals)[256]) {
    uint8_t* const p0 = p;
    const int nt = scan_tables(gray, s);
    for (int t = 0; t < nt; t++) {
        int total = 0;
        for (int l = 1; l <= 16; l++) total += bits[t][l];
        const int len = 2 + 1 + 16 + total;
        *p++ = 0xFF;
        *p++ = 0xC4;
        *p++ = (uint8_t)(len >> 8);
        *p++ = (uint8_t)len;
        // class 0 = DC, 1 = AC; id 0 = luma, 1 = chroma
        *p++ = (uint8_t)((s.Ss ? 0x10 : 0) | (s.Ss ? (s.comp > 0 ? 1 : 0) : t));
        for (int l = 1; l <= 16; l++) *p++ = bits[t][l];
        for (int v = 0; v < total; v++) *p++ = vals[t][v];
    }
    const int ns = s.comp < 0 && !gray ? 3 : 1;
    const int len = 6 + 2 * ns;
    *p++ = 0xFF;
    *p++ = 0xDA;
    *p++ = (uint8_t)(len >> 8);
    *p++ = (uint8_t)len;
    *p++ = (uint8_t)ns;
    for (int c = 0; c < ns; c++) {
        const int comp = ns == 3 ? c : (s.comp < 0 ? 0 : s.comp);
        const int tbl = comp > 0 ? 1 : 0;
        *p++ = (uint8_t)(comp + 1);
        *p++ = (uint8_t)(s.Ss == 0 ? (s.Ah == 0 ? tbl << 4 : 0) : tbl);
    }
    *p++ = (uint8_t)s.Ss;
    *p++ = (uint8_t)s.Se;
    *p++ = (uint8_t)((s.Ah << 4) | s.Al);
    return (int)(p - p0);
}

// Big-endian bit packer into 32-bit words from bit offset off.  Words other than the first and the last are this
// packer's alone; those two may be shared with a neighbouring block and go through orw (an atomicOr on the device).
template <class OrWord>
struct BitPacker {
    uint32_t* words;
    uint32_t widx;
    uint64_t acc;
    int nacc;
    bool first;
    OrWord orw;
    JPROG_HD BitPacker(uint32_t* w, uint32_t off, OrWord o) : words(w), widx(off >> 5), acc(0), nacc((int)(off & 31)), first(true), orw(o) {}
    JPROG_HD void put(uint32_t code, int size) {
        acc = (acc << size) | code;
        nacc += size;
        if (nacc >= 32) {
            const uint32_t w = (uint32_t)(acc >> (nacc - 32));
            if (first) {
                orw(&words[widx], w);
                first = false;
            } else {
                words[widx] = w;
            }
            widx++;
            nacc -= 32;
            acc &= (1ull << nacc) - 1;
        }
    }
    JPROG_HD void finish() {
        if (nacc > 0) orw(&words[widx], (uint32_t)(acc << (32 - nacc)));
    }
};

// Emitters for code_block.
struct CountBits {  // bits a block takes with the scan's tables
    const uint32_t* huff0;
    const uint32_t* huff1;
    uint32_t total;
    JPROG_HD void sym(int t, int s) { total += (t ? huff1 : huff0)[s] >> 16; }
    JPROG_HD void bits(uint32_t, int n) { total += (uint32_t)n; }
};

template <class Packer>
struct WriteBits {
    const uint32_t* huff0;
    const uint32_t* huff1;
    Packer* p;
    JPROG_HD void sym(int t, int s) {
        const uint32_t e = (t ? huff1 : huff0)[s];
        p->put(e & 0xffff, (int)(e >> 16));
    }
    JPROG_HD void bits(uint32_t v, int n) { p->put(v & ((1u << n) - 1), n); }
};

}  // namespace jprog
