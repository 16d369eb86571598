// Host build of lilliput_b200/csrc/jpeg_prog_core.h (progressive JPEG entropy coding) for the CPU suite.  Input: a
// baseline file written by the oracle's JPEG encoder (oracle/oracle_jpeg_enc.c).  Its entropy-coded data is decoded
// back to the quantised coefficients it carries -- exactly the blocks the baseline encoder coded -- and a whole
// progressive file is made from them the way jpeg_encode.cu makes it: the baseline frame header with SOF2, then every
// scan of the script (its optimal tables, SOS, the blocks' bits at offsets from the sizing pass, 1-padding, 0xFF
// stuffing), then EOI.  tests/test_jpeg_progressive_core.py compares that file with libjpeg-turbo's bytes.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../lilliput_b200/csrc/jpeg_prog_core.h"

struct StatsE {
    uint32_t (*hist)[257];
    void sym(int t, int s) { hist[t][s]++; }
    void bits(uint32_t, int) {}
};

// Huffman decoding of a baseline scan (T.81 F.2.2.3: per-length maxcode / valptr).
struct DecTable {
    int mincode[17], maxcode[18], valptr[17];
    uint8_t vals[256];
};
struct BitReader {
    std::vector<uint8_t> d;  // entropy-coded data with the stuffed zero bytes removed
    size_t pos = 0;
    int bit = 0;
    int get() {
        if (pos >= d.size()) return 1;  // past the end: the 1-padding
        const int b = (d[pos] >> (7 - bit)) & 1;
        if (++bit == 8) {
            bit = 0;
            pos++;
        }
        return b;
    }
    int receive(int n) {
        int v = 0;
        while (n--) v = (v << 1) | get();
        return v;
    }
    int decode(const DecTable& t) {
        int code = get(), l = 1;
        while (l <= 16 && code > t.maxcode[l]) {
            code = (code << 1) | get();
            l++;
        }
        return l > 16 ? -1 : t.vals[t.valptr[l] + code - t.mincode[l]];
    }
};
static int extend(int v, int n) { return n && v < (1 << (n - 1)) ? v - (1 << n) + 1 : v; }

// The coefficients of a baseline, interleaved, 4:2:0 (colour) or single-component (gray) file without restart
// markers, in the device layout: [mcu][block-in-mcu][64] zig-zag order.  Returns false on anything else.
static bool decode_baseline(const uint8_t* f, long n, int* W, int* H, int* gray, std::vector<int16_t>* coef) {
    DecTable tabs[2][2] = {};  // [class][id]
    int ncomp = 0;
    long o = 2;
    while (o + 4 <= n && f[o] == 0xFF) {
        const int m = f[o + 1], len = (f[o + 2] << 8) | f[o + 3];
        const uint8_t* p = f + o + 4;
        if (m == 0xC0) {
            *H = (p[1] << 8) | p[2];
            *W = (p[3] << 8) | p[4];
            ncomp = p[5];
        } else if (m == 0xC4) {
            for (const uint8_t* q = p; q < f + o + 2 + len;) {
                DecTable& t = tabs[q[0] >> 4][q[0] & 1];
                int code = 0, k = 0;
                for (int l = 1; l <= 16; l++) {
                    t.valptr[l] = k;
                    t.mincode[l] = code;
                    code += q[l];
                    k += q[l];
                    t.maxcode[l] = q[l] ? code - 1 : -1;
                    code <<= 1;
                }
                memcpy(t.vals, q + 17, k);
                q += 17 + k;
            }
        } else if (m == 0xDA) {
            o += 2 + len;
            break;
        }
        o += 2 + len;
    }
    if (ncomp != 1 && ncomp != 3) return false;
    BitReader br;
    for (; o + 1 < n && !(f[o] == 0xFF && f[o + 1] == 0xD9); o++) {
        br.d.push_back(f[o]);
        if (f[o] == 0xFF) o++;  // stuffed zero byte
    }
    *gray = ncomp == 1;
    const int hs = *gray ? 1 : 2, bpm = *gray ? 1 : 6;
    const int mcus = ((*W + 8 * hs - 1) / (8 * hs)) * ((*H + 8 * hs - 1) / (8 * hs));
    coef->assign((size_t)mcus * bpm * 64, 0);
    int pred[3] = {0, 0, 0};
    for (int b = 0; b < mcus * bpm; b++) {
        const int comp = *gray ? 0 : (b % 6 < 4 ? 0 : b % 6 - 3);
        const int t = comp > 0;
        int16_t* blk = coef->data() + (size_t)b * 64;
        const int s = br.decode(tabs[0][t]);
        if (s < 0) return false;
        pred[comp] += extend(br.receive(s), s);
        blk[0] = (int16_t)pred[comp];
        for (int z = 1; z < 64; z++) {
            const int rs = br.decode(tabs[1][t]);
            if (rs < 0) return false;
            if ((rs & 15) == 0) {
                if (rs != 0xF0) break;
                z += 15;
                continue;
            }
            z += rs >> 4;
            if (z > 63) return false;
            blk[z] = (int16_t)extend(br.receive(rs & 15), rs & 15);
        }
    }
    return true;
}

// baseline: a baseline file of oracle_jpeg_encode.  Returns the progressive file's length, or -1 if it does not fit in
// cap (or the input is not such a file).
extern "C" long jprog_encode(const uint8_t* baseline, long baseline_len, uint8_t* out, long cap) {
    int W = 0, H = 0, gray = 0;
    std::vector<int16_t> coef;
    if (!decode_baseline(baseline, baseline_len, &W, &H, &gray, &coef)) return -1;
    jprog::Geom g;
    const int hs = gray ? 1 : 2;
    g.mcus_x = (W + 8 * hs - 1) / (8 * hs);
    g.mcus_y = (H + 8 * hs - 1) / (8 * hs);
    g.bpm = gray ? 1 : 6;
    g.ybw = (W + 7) / 8;
    g.ybh = (H + 7) / 8;
    const size_t nblk = (size_t)g.mcus_x * g.mcus_y * g.bpm;
    // dummy blocks are all zero in the device layout (their DC is resolved from the blocks before them)
    for (size_t b = 0; b < nblk; b++)
        if (jprog::is_dummy(g, (int)(b / g.bpm), (int)(b % g.bpm))) memset(&coef[b * 64], 0, 64 * sizeof(int16_t));
    const int flen = jprog::frame_len(gray);
    if (baseline_len < flen || cap < flen + 2) return -1;
    memcpy(out, baseline, flen);
    out[jprog::sof_type_at(gray)] = 0xC2;
    long pos = flen;
    std::vector<uint32_t> summ(nblk), runs(nblk), words;
    const int nscans = gray ? jprog::kGrayScans : jprog::kColorScans;
    for (int si = 0; si < nscans; si++) {
        const jprog::Scan s = jprog::scan_of(gray, si);
        const int nb = jprog::scan_blocks(g, s);
        uint32_t hist[2][257] = {};
        StatsE st{hist};
        for (int i = 0; i < nb; i++) {
            summ[i] = jprog::code_block(coef.data(), g, s, i, 0, st);
            runs[i] = 0;
        }
        if (s.Ss)
            jprog::resolve_runs(summ.data(), nb, [&](int start, int run) {
                runs[start] = (uint32_t)run;
                hist[0][(jprog::nbits((unsigned)run) - 1) << 4]++;
            });
        uint8_t bits[2][17] = {}, vals[2][256] = {};
        uint32_t huff[2][256] = {};
        const int nt = jprog::scan_tables(gray, s);
        for (int t = 0; t < nt; t++) {
            int codesize[257], tree[257];
            if (jprog::gen_optimal_table(jprog::OneLane{}, hist[t], codesize, tree, bits[t], vals[t]) < 0) return -1;
            jprog::make_codes(bits[t], vals[t], huff[t]);
        }
        if (pos + jprog::scan_header_len(gray, s, bits) + 2 > cap) return -1;
        pos += jprog::put_scan_header(out + pos, gray, s, bits, vals);
        // sizing pass -> bit offsets, then every block writes at its own offset
        std::vector<uint32_t> off(nb + 1, 0);
        for (int i = 0; i < nb; i++) {
            jprog::CountBits c{huff[0], huff[1], 0};
            jprog::code_block(coef.data(), g, s, i, (int)runs[i], c);
            off[i + 1] = off[i] + c.total;
        }
        const uint32_t total = off[nb];
        words.assign(total / 32 + 2, 0);
        auto orw = [](uint32_t* w, uint32_t v) { *w |= v; };
        for (int i = 0; i < nb; i++) {
            jprog::BitPacker<decltype(orw)> p(words.data(), off[i], orw);
            jprog::WriteBits<decltype(p)> e{huff[0], huff[1], &p};
            jprog::code_block(coef.data(), g, s, i, (int)runs[i], e);
            p.finish();
        }
        if (total & 7) {  // pad the last byte with 1-bits
            const uint32_t padn = 8 - (total & 7), at = total & 31;
            words[total >> 5] |= ((1u << padn) - 1) << (32 - at - padn);
        }
        const uint32_t nbytes = (total + 7) >> 3;
        for (uint32_t b = 0; b < nbytes; b++) {
            const uint8_t v = (uint8_t)(words[b >> 2] >> (24 - 8 * (b & 3)));
            if (pos + 2 + 2 > cap) return -1;
            out[pos++] = v;
            if (v == 0xFF) out[pos++] = 0;
        }
    }
    if (pos + 2 > cap) return -1;
    out[pos++] = 0xFF;
    out[pos++] = 0xD9;
    return pos;
}
