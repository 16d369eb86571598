// jpeg_parse.cpp -- host-side JPEG marker parsing (ITU-T T.81 Annex B) and Huffman
// table preparation for the device decoder.  No pixel arithmetic here.
//
// Stands where cv::ImageDecoder::readHeader does for the reference
// (ref opencv.cpp:126-164): width / height / channel count / EXIF orientation.
#include <cstring>
#include <vector>

#include "kernels.cuh"
#include "jpeg_std_tables.h"
#include "lilliput_b200.h"

namespace lp {

static const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// EXIF orientation the way the reference's OpenCV 4.11 reads it (modules/imgcodecs/src/exif.cpp driven by
// grfmt_jpeg.cpp; restated from behaviour and pinned by tests/test_host_exif.py against the live reference).
// What that reader does and a tidy TIFF parser would not:
//  * only the FIRST APP1 segment of the file is looked at, whatever its identifier; its first 6 bytes are skipped
//    unread ("Exif\0\0" is never compared), so an XMP APP1 in front hides the EXIF one;
//  * a byte-order mark that is neither "II" nor "MM" reads big-endian;
//  * IFD0 entries are parsed in file order and the parse stops at the first entry whose data lies outside the
//    segment (strings, rationals); entries already read stay valid, later ones are never seen;
//  * the orientation value is the 16-bit word at entry + 8, whatever the entry's type and count say, and is
//    reported as it is (0, 9, 300 ...); of two orientation entries the first counts.
// Returns true and sets *value when an orientation entry was read.
namespace {
struct ExifBytes {
    const uint8_t* d;
    size_t n;
    bool intel;
    bool stop = false;  // OpenCV: ExifParsingError thrown
    unsigned u16(size_t o) {
        if (stop || o + 1 >= n || o + 1 < o) { stop = true; return 0; }
        return intel ? (unsigned)(d[o] | (d[o + 1] << 8)) : (unsigned)((d[o] << 8) | d[o + 1]);
    }
    uint32_t u32(size_t o) {
        if (stop || o + 3 >= n || o + 3 < o) { stop = true; return 0; }
        return intel ? ((uint32_t)d[o] | ((uint32_t)d[o + 1] << 8) | ((uint32_t)d[o + 2] << 16) | ((uint32_t)d[o + 3] << 24))
                     : (((uint32_t)d[o] << 24) | ((uint32_t)d[o + 1] << 16) | ((uint32_t)d[o + 2] << 8) | d[o + 3]);
    }
    void rationals(size_t entry, int count) {  // count (numerator, denominator) pairs at the offset the entry names
        size_t o = u32(entry + 8);
        for (int i = 0; i < count && !stop; i++, o += 8) { u32(o); u32(o + 4); }
    }
    void string(size_t entry) {
        size_t len = u32(entry + 4);
        size_t off = len > 4 ? (size_t)u32(entry + 8) : entry + 8;
        if (stop) return;
        if (off >= n || len > n - off) stop = true;
    }
};
}  // namespace

bool exif_orientation_opencv(const uint8_t* tiff, size_t n, int* value) {
    if (n == 0) return false;
    ExifBytes x{tiff, n, n >= 2 && tiff[0] == tiff[1] && tiff[0] == 'I'};
    if (x.u16(2) != 0x002A || x.stop) return false;
    size_t off = x.u32(4);
    const unsigned entries = x.u16(off);
    off += 2;
    bool found = false;
    for (unsigned i = 0; i < entries && !x.stop; i++, off += 12) {
        const unsigned tag = x.u16(off);
        if (x.stop) break;
        unsigned v = 0;
        switch (tag) {
            case 0x010E: case 0x010F: case 0x0110: case 0x0131: case 0x0132: case 0x8298:  // description, make, model, software, date, copyright
                x.string(off);
                break;
            case 0x0112:  // orientation
                v = x.u16(off + 8);
                if (!x.stop && !found) {
                    *value = (int)v;
                    found = true;
                }
                break;
            case 0x011A: case 0x011B:  // x / y resolution
                x.rationals(off, 1);
                break;
            case 0x0128: case 0x011C: case 0x0213:  // resolution unit, planar configuration, YCbCr positioning
                x.u16(off + 8);
                break;
            case 0x013E:  // white point
                x.rationals(off, 2);
                break;
            case 0x013F: case 0x0214:  // primary chromaticities, reference black / white
                x.rationals(off, 6);
                break;
            case 0x0211:  // YCbCr coefficients
                x.rationals(off, 3);
                break;
            case 0x8769:  // Exif IFD pointer
                x.u32(off + 8);
                break;
            default:
                break;
        }
    }
    return found;
}

int jpeg_parse_header(const uint8_t* in, size_t len, JpegHeader* out) {
    JpegHeader& h = *out;
    h = JpegHeader();
    if (len < 4 || in[0] != 0xFF || in[1] != 0xD8) return LP_ERR_INVALID_IMAGE;
    size_t pos = 2;
    bool have_sof = false, seen_app1 = false, undecodable = false;
    while (pos + 4 <= len) {
        if (in[pos] != 0xFF) { pos++; continue; }
        uint8_t m = in[pos + 1];
        if (m == 0xFF) { pos++; continue; }
        if (m == 0xD9) break;
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) { pos += 2; continue; }
        if (m == 0x00) { pos += 2; continue; }  // FF 00 between segments is not a marker: libjpeg skips it as garbage
        // marker codes libjpeg's read_markers has no case for ("Unsupported marker type"), and JPG
        if ((m >= 0x02 && m <= 0xBF) || (m >= 0xF0 && m <= 0xFD) || m == 0xC8) return LP_ERR_INVALID_IMAGE;
        size_t seg = ((size_t)in[pos + 2] << 8) | in[pos + 3];
        if (seg < 2 || pos + 2 + seg > len) return LP_ERR_INVALID_IMAGE;
        const uint8_t* p = in + pos + 4;
        size_t n = seg - 2;
        if (m == 0xDB) {
            while (n >= 65) {
                int pq = p[0] >> 4, tq = p[0] & 15;
                size_t need = pq ? 129 : 65;
                if (tq > 3 || n < need) return LP_ERR_INVALID_IMAGE;
                for (int i = 0; i < 64; i++)
                    h.qt[tq][kZigzag[i]] = pq ? (uint16_t)((p[1 + 2 * i] << 8) | p[2 + 2 * i]) : p[1 + i];
                h.qt_present[tq] = true;
                p += need;
                n -= need;
            }
            if (n != 0) return LP_ERR_INVALID_IMAGE;  // get_dqt: "Bogus marker length"
        } else if (m == 0xC4) {
            while (n >= 17) {
                int tc = p[0] >> 4, th = p[0] & 15;
                if (tc > 1 || th > 3) return LP_ERR_INVALID_IMAGE;
                int total = 0;
                h.huff_bits[tc][th][0] = 0;
                for (int i = 1; i <= 16; i++) { h.huff_bits[tc][th][i] = p[i]; total += p[i]; }
                if (total > 256 || n < (size_t)(17 + total)) return LP_ERR_INVALID_IMAGE;
                memset(h.huff_vals[tc][th], 0, 256);
                memcpy(h.huff_vals[tc][th], p + 17, total);
                h.huff_present[tc][th] = true;
                p += 17 + total;
                n -= 17 + total;
            }
            if (n != 0) return LP_ERR_INVALID_IMAGE;  // get_dht: "Bogus marker length"
        } else if (m == 0xC0 || m == 0xC1 || m == 0xC2) {
            if (n < 6 || have_sof) return LP_ERR_INVALID_IMAGE;  // a second frame header: "duplicate SOF"
            h.progressive = (m == 0xC2);
            int prec = p[0];
            h.height = (p[1] << 8) | p[2];
            h.width = (p[3] << 8) | p[4];
            h.ncomp = p[5];
            // get_sof / initial_setup of the reference's libjpeg-turbo: empty image, segment length that does not fit
            // the component count, more than 10 components, a dimension over 65500, a precision other than 8 or 12
            if (h.width < 1 || h.height < 1 || h.ncomp < 1) return LP_ERR_INVALID_IMAGE;
            if (n != (size_t)(6 + 3 * h.ncomp) || h.ncomp > 10) return LP_ERR_INVALID_IMAGE;
            if (h.width > 65500 || h.height > 65500 || (prec != 8 && prec != 12)) return LP_ERR_INVALID_IMAGE;
            if (prec != 8 || (h.ncomp != 1 && h.ncomp != 3) || n < (size_t)(6 + 3 * h.ncomp)) {
                have_sof = true;  // dimensions known, but not decodable here
                h.ncomp = h.ncomp == 1 ? 1 : 3;
                h.supported = false;
                pos += 2 + seg;
                continue;
            }
            for (int i = 0; i < h.ncomp; i++) {
                h.comp[i].id = p[6 + 3 * i];
                h.comp[i].h = p[7 + 3 * i] >> 4;
                h.comp[i].v = p[7 + 3 * i] & 15;
                h.comp[i].tq = p[8 + 3 * i];
                if (h.comp[i].h < 1 || h.comp[i].h > 4 || h.comp[i].v < 1 || h.comp[i].v > 4) return LP_ERR_INVALID_IMAGE;
                if (h.comp[i].tq > 3) {  // libjpeg reads such a header and fails when the decode looks for the table
                    h.comp[i].tq = 0;
                    undecodable = true;
                }
                h.maxh = h.comp[i].h > h.maxh ? h.comp[i].h : h.maxh;
                h.maxv = h.comp[i].v > h.maxv ? h.comp[i].v : h.maxv;
            }
            if (h.ncomp == 1) { h.comp[0].h = h.comp[0].v = 1; h.maxh = h.maxv = 1; }
            have_sof = true;
            h.supported = !h.progressive;
            for (int i = 0; i < h.ncomp; i++)
                if (h.maxh % h.comp[i].h || h.maxv % h.comp[i].v) h.supported = false;
            h.mcus_x = (h.width + 8 * h.maxh - 1) / (8 * h.maxh);
            h.mcus_y = (h.height + 8 * h.maxv - 1) / (8 * h.maxv);
        } else if (m >= 0xC3 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
            return LP_ERR_UNSUPPORTED;  // lossless / differential / arithmetic
        } else if (m == 0xDD) {
            if (n != 2) return LP_ERR_INVALID_IMAGE;  // get_dri: the segment is exactly 4 bytes
            h.restart_interval = (p[0] << 8) | p[1];
        } else if (m == 0xE1) {
            if (!seen_app1 && n > 6) {
                int o = 0;
                if (exif_orientation_opencv(p + 6, n - 6, &o)) h.orientation = o;
            }
            seen_app1 = true;
        } else if (m == 0xDA) {
            if (!have_sof || n < 1) return LP_ERR_INVALID_IMAGE;
            int ns = p[0];
            if (ns < 1 || ns > 3 || n != (size_t)(1 + 2 * ns + 3)) return LP_ERR_INVALID_IMAGE;  // get_sos: exact length
            if (h.comp[0].h >= 1) {  // frame components known: every selector names one of them, none twice
                for (int i = 0; i < ns; i++) {
                    bool known = false;
                    for (int j = 0; j < h.ncomp; j++) known = known || h.comp[j].id == p[1 + 2 * i];
                    if (!known) return LP_ERR_INVALID_IMAGE;  // "Invalid component ID in SOS"
                    for (int k = 0; k < i; k++)
                        if (p[1 + 2 * k] == p[1 + 2 * i]) return LP_ERR_INVALID_IMAGE;
                }
            }
            if (ns != h.ncomp) h.supported = false;  // one scan per component: serial multi-scan path
            if (h.progressive || ns != h.ncomp) {
                bool ok = true;
                for (int i = 0; i < h.ncomp; i++) {
                    // (a frame header this decoder does not take -- 12-bit, 4 components -- leaves the factors 0)
                    if (h.comp[i].h < 1 || h.comp[i].v < 1) { ok = false; break; }
                    if (h.maxh % h.comp[i].h || h.maxv % h.comp[i].v || !h.qt_present[h.comp[i].tq]) ok = false;
                }
                h.multiscan = ok;
            }
            // libjpeg-turbo fills the table slots 0 and 1 that no DHT segment defined with the Annex K tables when the
            // decode starts (jinit_huff_decoder -> std_huff_tables: Motion-JPEG frames are written without DHT), so a
            // file that lost or never had them decodes in the reference; slots 2 and 3 stay undefined
            for (int tc = 0; tc < 2; tc++)
                for (int th = 0; th < 2; th++)
                    if (!h.huff_present[tc][th]) {
                        const uint8_t* bits = tc == 0 ? (th == 0 ? kDcLBits : kDcCBits) : (th == 0 ? kAcLBits : kAcCBits);
                        const uint8_t* vals = tc == 0 ? kDcVals : (th == 0 ? kAcLVals : kAcCVals);
                        int total = 0;
                        for (int i = 0; i <= 16; i++) { h.huff_bits[tc][th][i] = bits[i]; total += i ? bits[i] : 0; }
                        memset(h.huff_vals[tc][th], 0, 256);
                        memcpy(h.huff_vals[tc][th], vals, total);
                        h.huff_present[tc][th] = true;
                    }
            for (int i = 0; i < ns && h.supported; i++) {
                int ci = -1;
                for (int j = 0; j < h.ncomp; j++)
                    if (h.comp[j].id == p[1 + 2 * i]) ci = j;
                if (ci != i) { h.supported = false; break; }
                h.comp[ci].td = p[2 + 2 * i] >> 4;
                h.comp[ci].ta = p[2 + 2 * i] & 15;
                if (h.comp[ci].td > 3 || h.comp[ci].ta > 3 || !h.huff_present[0][h.comp[ci].td] ||
                    !h.huff_present[1][h.comp[ci].ta] || !h.qt_present[h.comp[ci].tq]) {
                    // a table the scan needs was never defined (or its segment was lost to damage): the reference's
                    // header read succeeds and its decode fails ("... table 0x%02x was not defined"); same here
                    h.comp[ci].td = h.comp[ci].ta = 0;
                    undecodable = true;
                    break;
                }
            }
            // libjpeg's jpeg_make_d_derived_tbl (jdhuff.c) refuses a table whose code lengths over-subscribe the code
            // space or whose DC symbols exceed 15 (JERR_BAD_HUFF_TABLE) when the scan starts: the header reads, the
            // decode fails.  Same here, on every decode path (the parallel kernel would otherwise read a DC symbol's
            // high nibble as a run).
            for (int i = 0; i < ns && !undecodable && h.supported; i++) {
                for (int tc = 0; tc < 2 && !undecodable; tc++) {
                    const int th = tc ? h.comp[i].ta : h.comp[i].td;
                    const uint8_t* bits = h.huff_bits[tc][th];
                    unsigned code = 0;
                    int total = 0, last = 0;
                    for (int len = 1; len <= 16; len++)
                        if (bits[len]) last = len;
                    for (int len = 1; len <= last; len++) {
                        code += bits[len];
                        if (code >= (1u << len)) undecodable = true;  // "no code is allowed to be all ones" (jdhuff.c)
                        code <<= 1;
                        total += bits[len];
                    }
                    if (tc == 0)
                        for (int k = 0; k < total && k < 256; k++)
                            if (h.huff_vals[0][th][k] > 15) undecodable = true;
                }
            }
            if (undecodable) h.supported = h.multiscan = false;  // read_data refuses on the host: ErrDecodingFailed
            h.scan_offset = pos + 2 + seg;
            // upper bound of the entropy-coded segment: up to the last EOI if there is one
            size_t end = len;
            for (size_t k = len; k >= h.scan_offset + 2 && k + 64 > len; k--)
                if (in[k - 2] == 0xFF && in[k - 1] == 0xD9) { end = k - 2; break; }
            h.scan_length = end - h.scan_offset;
            return LP_OK;
        }
        pos += 2 + seg;
    }
    return have_sof ? LP_ERR_INVALID_IMAGE : LP_ERR_INVALID_IMAGE;
}

// Second walk for multi-scan files: one JpegScanDesc per SOS, with the DHT / DRI state at that point.
int jpeg_parse_scans(const uint8_t* in, size_t len, const JpegHeader& h0, JpegScanDesc* scans, int max_scans,
                     int* nscans, JpegHeader* sets, int max_sets, int* nsets) {
    JpegHeader h = h0;  // tracks DHT redefinitions between scans
    memset(h.huff_present, 0, sizeof(h.huff_present));
    h.restart_interval = 0;
    *nscans = 0;
    *nsets = 0;
    bool dirty = true;
    size_t pos = 2;
    while (pos + 4 <= len) {
        if (in[pos] != 0xFF) { pos++; continue; }
        const uint8_t m = in[pos + 1];
        if (m == 0xFF) { pos++; continue; }
        if (m == 0xD9) break;
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) { pos += 2; continue; }
        const size_t seg = ((size_t)in[pos + 2] << 8) | in[pos + 3];
        if (seg < 2 || pos + 2 + seg > len) break;  // truncated: decode the scans seen so far
        const uint8_t* p = in + pos + 4;
        size_t n = seg - 2;
        if (m == 0xC4) {
            while (n >= 17) {
                const int tc = p[0] >> 4, th = p[0] & 15;
                if (tc > 1 || th > 3) return LP_ERR_INVALID_IMAGE;
                int total = 0;
                h.huff_bits[tc][th][0] = 0;
                for (int i = 1; i <= 16; i++) { h.huff_bits[tc][th][i] = p[i]; total += p[i]; }
                if (total > 256 || n < (size_t)(17 + total)) return LP_ERR_INVALID_IMAGE;
                memset(h.huff_vals[tc][th], 0, 256);
                memcpy(h.huff_vals[tc][th], p + 17, total);
                h.huff_present[tc][th] = true;
                p += 17 + total;
                n -= 17 + total;
            }
            dirty = true;
        } else if (m == 0xDD) {
            if (n >= 2) h.restart_interval = (p[0] << 8) | p[1];
        } else if (m == 0xDA) {
            if (n < 1) return LP_ERR_INVALID_IMAGE;
            const int ns = p[0];
            if (ns < 1 || ns > h.ncomp || n < (size_t)(1 + 2 * ns + 3)) return LP_ERR_INVALID_IMAGE;
            if (*nscans >= max_scans) return LP_ERR_UNSUPPORTED;
            JpegScanDesc& sc = scans[*nscans];
            memset(&sc, 0, sizeof(sc));
            sc.ns = ns;
            sc.progressive = h.progressive;
            sc.Ss = h.progressive ? p[1 + 2 * ns] : 0;
            sc.Se = h.progressive ? p[2 + 2 * ns] : 63;
            sc.Ah = h.progressive ? p[3 + 2 * ns] >> 4 : 0;
            sc.Al = h.progressive ? p[3 + 2 * ns] & 15 : 0;
            if (sc.Ss > sc.Se || sc.Se > 63 || sc.Al > 13 || (h.progressive && sc.Ss == 0 && sc.Se != 0) ||
                (sc.Ss > 0 && ns != 1))
                return LP_ERR_INVALID_IMAGE;
            for (int i = 0; i < ns; i++) {
                int ci = -1;
                for (int j = 0; j < h.ncomp; j++)
                    if (h.comp[j].id == p[1 + 2 * i]) ci = j;
                if (ci < 0) return LP_ERR_INVALID_IMAGE;
                sc.ci[i] = ci;
                sc.td[i] = p[2 + 2 * i] >> 4;
                sc.ta[i] = p[2 + 2 * i] & 15;
                if (sc.td[i] > 3 || sc.ta[i] > 3) return LP_ERR_INVALID_IMAGE;
                const bool need_dc = !h.progressive || (sc.Ss == 0 && sc.Ah == 0);
                const bool need_ac = !h.progressive || sc.Ss > 0;
                if ((need_dc && !h.huff_present[0][sc.td[i]]) || (need_ac && !h.huff_present[1][sc.ta[i]]))
                    return LP_ERR_INVALID_IMAGE;
            }
            if (dirty) {
                if (*nsets >= max_sets) return LP_ERR_UNSUPPORTED;
                if (sets) sets[*nsets] = h;
                (*nsets)++;
                dirty = false;
            }
            sc.table_set = *nsets - 1;
            sc.restart_interval = h.restart_interval;
            // entropy-coded segment: up to the next marker that is neither a stuffed FF00 nor RSTn
            size_t q = pos + 2 + seg;
            const size_t start = q;
            while (q + 1 < len && !(in[q] == 0xFF && in[q + 1] != 0x00 && in[q + 1] != 0xFF &&
                                    !(in[q + 1] >= 0xD0 && in[q + 1] <= 0xD7)))
                q++;
            if (q + 1 >= len) q = len;
            sc.data_off = (uint32_t)start;
            sc.data_len = (uint32_t)(q - start);
            (*nscans)++;
            pos = q;
            continue;
        }
        pos += 2 + seg;
    }
    return *nscans > 0 ? LP_OK : LP_ERR_INVALID_IMAGE;
}

int jpeg_parse_scans(const uint8_t* in, size_t len, const JpegHeader& h, JpegScanDesc* scans, int max_scans,
                     int* nscans, JpegHuffSet* sets, int max_sets, int* nsets) {
    std::vector<JpegHeader> tables((size_t)(max_sets > 0 ? max_sets : 0));
    const int rc = jpeg_parse_scans(in, len, h, scans, max_scans, nscans, tables.data(), max_sets, nsets);
    if (rc == 0)
        for (int k = 0; k < *nsets; k++) jpeg_build_huff_set(tables[k], &sets[k]);
    return rc;
}

void jpeg_baseline_scan(const JpegHeader& h, JpegScanDesc* out) {
    memset(out, 0, sizeof(*out));
    out->data_off = (uint32_t)h.scan_offset;
    out->data_len = (uint32_t)h.scan_length;
    out->ns = h.ncomp;
    for (int i = 0; i < h.ncomp; i++) {
        out->ci[i] = i;
        out->td[i] = h.comp[i].td;
        out->ta[i] = h.comp[i].ta;
    }
    out->Se = 63;
    out->restart_interval = h.restart_interval;
}

size_t jpeg_multiscan_visits(const JpegHeader& h, const JpegScanDesc* scans, int nscans) {
    size_t visits = 0;
    for (int k = 0; k < nscans; k++)
        for (int c = 0; c < scans[k].ns; c++) {
            const int ci = scans[k].ci[c];
            visits += (size_t)h.mcus_x * h.mcus_y * h.comp[ci].h * h.comp[ci].v;
        }
    return visits;
}

// Canonical Huffman decode tables (T.81 Annex C / F.2.2.3) in the device layout.
void jpeg_build_huff_set(const JpegHeader& h, JpegHuffSet* out) {
    memset(out, 0, sizeof(*out));
    memset(out->long_prefix, 0xFF, sizeof(out->long_prefix));
    for (int tc = 0; tc < 2; tc++)
        for (int th = 0; th < 4; th++) {
            int t = tc * 4 + th;
            for (int l = 0; l < 18; l++) out->maxcode[t][l] = -1;
            out->maxcode[t][17] = 0x7fffffff;
            if (!h.huff_present[tc][th]) continue;
            const uint8_t* bits = h.huff_bits[tc][th];
            memcpy(out->vals[t], h.huff_vals[tc][th], 256);
            unsigned code = 0;
            int k = 0;
            for (int len = 1; len <= 16; len++) {
                out->valoffset[t][len] = k - (int)code;
                for (int i = 0; i < bits[len]; i++, k++) {
                    if (len <= 9) {
                        unsigned first = code << (9 - len), cnt = 1u << (9 - len);
                        for (unsigned j = 0; j < cnt && first + j < 512; j++)
                            out->look[t][first + j] = (uint16_t)((len << 8) | h.huff_vals[tc][th][k]);
                    }
                    // (code >> len) != 0: an over-subscribed table from a hostile DHT -- not a codeword, and its
                    // "prefix" would index outside the lookahead table on the device
                    if (tc == 1 && len > kHuffAcLookBits && (code >> len) == 0) {
                        const unsigned prefix = code >> (len - kHuffAcLookBits);
                        int j = 0;
                        while (j < kHuffLongPrefixes && out->long_prefix[th][j] != prefix &&
                               out->long_prefix[th][j] != 0xFFFF)
                            j++;
                        if (j < kHuffLongPrefixes) {
                            out->long_prefix[th][j] = (uint16_t)prefix;
                            const unsigned rest = code & ((1u << (len - kHuffAcLookBits)) - 1);
                            const unsigned first = rest << (16 - len), cnt = 1u << (16 - len);
                            for (unsigned q = 0; q < cnt; q++)
                                out->long_sub[th][j][first + q] = (uint16_t)((len << 8) | h.huff_vals[tc][th][k]);
                        }
                    }
                    code++;
                }
                out->maxcode[t][len] = bits[len] ? (int)code - 1 : -1;
                code <<= 1;
            }
        }
}

}  // namespace lp
