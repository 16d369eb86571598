// gif_decode.cu -- lilliput's GIF decoder surface (include/lp_giflib.h = ref giflib.hpp:33-52) on
// sm_90a: host container walk, device LZW decode, device full-canvas compositor.
//
// Replaces: giflib_decoder_* (ref giflib.cpp:104-347, 570-724, 1308-1431): giflib 5.2.2's
// DGifGetRecordType / DGifGetExtension / DGifGetImageHeader / DGifGetLine plus the reference's own
// compositor (ref giflib.cpp:349-568): background fill on the first frame, dispose-to-background /
// restore-previous of the previous frame's clipped rectangle, snapshot, then non-transparent,
// in-palette pixels drawn with A=255, frames that hang off the canvas clipped.  Output is the
// full-canvas BGRA frame lilliput's ops.go expects.  Lossless: bit-exact to the reference
// (tests/test_gpu_gif.py against reference-made golden frames) and to the oracle on hand-built code streams that steer
// every corner of the LZW kernel and the compositor (tests/test_gpu_gif_streams.py, both callers).
//
// One device path serves both callers: the per-image decoder (one frame per call, canvas and snapshot kept in
// the decoder between calls) and gif_decode_batch (every frame of many animations at once).  One warp per frame
// decodes its LZW code stream (a GIF code stream is serial, so the frame is the unit of parallelism; see
// gif_lzw_decode_frame), then one thread per canvas pixel composites the frames of its animation in order.  The
// batch strips the sub-block framing on the device, one warp per frame; the per-image decoder gathers the code
// stream on the host, where a single frame's serial walk over its sub-blocks is cheaper.
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"
#include "lp_giflib.h"

namespace lp {

// ------------------------------------------------------------------ container walk (host)

struct GifGcb {
    int disposal = 0, delay = 0, transparent = -1;
    bool user_input = false;
};

struct GifImage {
    int left = 0, top = 0, width = 0, height = 0;
    bool interlace = false;
    int ncolors = 0;          // local colour table entries (0 = none)
    const uint8_t* colors = nullptr;
    int min_code = 0;
};

// Sequential reader over the borrowed bytes, with giflib's record semantics.
struct GifReader {
    const uint8_t* p = nullptr;
    size_t n = 0, pos = 0;
    int sw = 0, sh = 0, bg_index = 0, gct_colors = 0;
    const uint8_t* gct = nullptr;
    uint8_t packed = 0, aspect = 0;  // logical screen descriptor bytes 10 and 12

    bool get(uint8_t* b) {
        if (pos >= n) return false;
        *b = p[pos++];
        return true;
    }
    bool open() {  // DGifOpen: signature, logical screen descriptor, global colour table
        if (n < 13 || (memcmp(p, "GIF87a", 6) && memcmp(p, "GIF89a", 6))) return false;
        sw = p[6] | (p[7] << 8);
        sh = p[8] | (p[9] << 8);
        packed = p[10];
        bg_index = p[11];
        aspect = p[12];
        pos = 13;
        if (packed & 0x80) {
            gct_colors = 1 << ((packed & 7) + 1);
            if (pos + (size_t)gct_colors * 3 > n) return false;
            gct = p + pos;
            pos += (size_t)gct_colors * 3;
        }
        return true;
    }
    // 0 = image descriptor, 1 = extension, 2 = terminator, -1 = error (incl. read past the end)
    int record() {
        uint8_t b;
        if (!get(&b)) return -1;
        return b == 0x2C ? 0 : b == 0x21 ? 1 : b == 0x3B ? 2 : -1;
    }
    // one data sub-block: *len = 0 at the terminator
    bool sub_block(const uint8_t** data, int* len) {
        uint8_t b;
        if (!get(&b)) return false;
        *len = b;
        *data = p + pos;
        if (pos + b > n) return false;
        pos += b;
        return true;
    }
    bool image_header(GifImage* im) {  // DGifGetImageHeader (+ the LZW minimum code size byte)
        if (pos + 9 > n) return false;
        im->left = p[pos] | (p[pos + 1] << 8);
        im->top = p[pos + 2] | (p[pos + 3] << 8);
        im->width = p[pos + 4] | (p[pos + 5] << 8);
        im->height = p[pos + 6] | (p[pos + 7] << 8);
        const uint8_t packed = p[pos + 8];
        pos += 9;
        im->interlace = (packed & 0x40) != 0;
        im->ncolors = 0;
        im->colors = nullptr;
        if (packed & 0x80) {
            im->ncolors = 1 << ((packed & 7) + 1);
            if (pos + (size_t)im->ncolors * 3 > n) return false;
            im->colors = p + pos;
            pos += (size_t)im->ncolors * 3;
        }
        uint8_t cs;
        if (!get(&cs)) return false;
        if (cs > 8) return false;  // giflib: D_GIF_ERR_READ_FAILED
        im->min_code = cs;
        return true;
    }
};

// DGifExtensionToGCB: only a 4-byte block is a valid graphic control block.
static bool gcb_from_block(const uint8_t* b, int len, GifGcb* g) {
    if (len != 4) return false;
    g->disposal = (b[0] >> 2) & 7;
    g->user_input = (b[0] >> 1) & 1;
    g->delay = b[1] | (b[2] << 8);
    g->transparent = (b[0] & 1) ? b[3] : -1;
    return true;
}

// ref giflib.cpp:595-636
static void background_color(const GifReader& r, const GifGcb& g, uint8_t* R, uint8_t* G, uint8_t* B, uint8_t* A) {
    const bool valid = r.gct && r.bg_index >= 0 && r.bg_index < r.gct_colors;
    if (valid) {
        *R = r.gct[r.bg_index * 3];
        *G = r.gct[r.bg_index * 3 + 1];
        *B = r.gct[r.bg_index * 3 + 2];
    } else {
        *R = *G = *B = 255;
    }
    *A = g.transparent != -1 ? 0 : 255;
}

// One entry of giflib's GifFileType::ExtensionBlocks: the first sub-block of an extension carries
// its label, the following ones CONTINUE_EXT_FUNC_CODE (0).
struct GifExt {
    int function;
    std::vector<uint8_t> bytes;
};
// EGifGCBToExtension into every graphic-control block of at least 4 bytes (ref giflib.cpp:272-291)
static void set_frame_gcb(std::vector<GifExt>& ext, const GifGcb& g) {
    for (GifExt& e : ext) {
        if (e.function != 0xF9 || e.bytes.size() < 4) continue;
        e.bytes[0] = (uint8_t)((g.transparent != -1 ? 1 : 0) | (g.user_input ? 2 : 0) | ((g.disposal & 7) << 2));
        e.bytes[1] = (uint8_t)(g.delay & 0xFF);
        e.bytes[2] = (uint8_t)((g.delay >> 8) & 0xFF);
        e.bytes[3] = (uint8_t)g.transparent;
    }
}
// giflib_get_frame_gcb (ref giflib.cpp:248-270): defaults, then every well-formed block in order
static GifGcb get_frame_gcb(const std::vector<GifExt>& ext) {
    GifGcb g;
    for (const GifExt& e : ext)
        if (e.function == 0xF9) gcb_from_block(e.bytes.data(), (int)e.bytes.size(), &g);
    return g;
}

// ref giflib.cpp:209-246: every sub-block of one extension (behind its 0x21 introducer) is appended to `ext`; every
// graphic control block to `gcbs` (a malformed one as the defaults it resets to)
static bool read_extension(GifReader& r, std::vector<GifExt>* ext, std::vector<GifGcb>* gcbs) {
    uint8_t label;
    if (!r.get(&label)) return false;
    const uint8_t* data;
    int len;
    if (!r.sub_block(&data, &len)) return false;
    bool first = true;
    while (len != 0) {
        ext->push_back(GifExt{first ? (int)label : 0, std::vector<uint8_t>(data, data + len)});
        if (first && label == 0xF9) {
            GifGcb g;
            if (gcb_from_block(data, len, &g)) gcbs->push_back(g);
            else gcbs->push_back(GifGcb());
        }
        first = false;
        if (!r.sub_block(&data, &len)) return false;
    }
    return true;
}

// ref giflib.cpp:548-565: after decoding a partial frame without a transparent index the decoder forces one (the last
// palette entry) into the frame's graphic control blocks, for the encoder's benefit
static void force_partial_transparent(std::vector<GifExt>& ext, const GifGcb& gcb, const GifImage& im, int ncolors,
                                      int cw, int chh) {
    if ((im.height < chh || im.width < cw || im.left != 0 || im.top != 0) && gcb.transparent == -1) {
        GifGcb forced = gcb;
        forced.transparent = ncolors - 1;
        set_frame_gcb(ext, forced);
    }
}

// The encoder's view of the source's logical screen (ref giflib.cpp:803-860): background index 0 unless the global
// colour table has the source's entry
static int encoder_bg_index(const GifReader& r) {
    return (r.gct && r.bg_index >= 0 && r.bg_index < r.gct_colors) ? r.bg_index : 0;
}

// giflib_encoder_setup_frame (ref giflib.cpp:862-920): the frame's GCB, with a transparent index that names the
// opaque background colour of a global-palette frame dropped (in `ext` too)
static GifGcb encoder_frame_gcb(std::vector<GifExt>& ext, const GifReader& r, bool has_local, bool bg_opaque) {
    GifGcb gcb = get_frame_gcb(ext);
    if (gcb.transparent != -1 && r.gct && !has_local && gcb.transparent == encoder_bg_index(r) && bg_opaque) {
        gcb.transparent = -1;
        set_frame_gcb(ext, gcb);
    }
    return gcb;
}

// bits per pixel of a colour map of `ncolors` entries (the image descriptor's size field + 1)
static int color_bits(int ncolors) {
    int bpp = 1;
    while ((1 << bpp) < ncolors) bpp++;
    return bpp;
}

// encode_func (ref giflib.cpp:762-771): a write that does not fit the destination fails whole and writes nothing
struct GifWriter {
    uint8_t* dst = nullptr;
    size_t dst_len = 0, dst_offset = 0;

    bool put(const void* p, size_t n) {
        if (dst_offset + n > dst_len) return false;
        memcpy(dst + dst_offset, p, n);
        dst_offset += n;
        return true;
    }
    bool put8(uint8_t b) { return put(&b, 1); }
    bool put16(int v) {
        const uint8_t b[2] = {(uint8_t)(v & 0xff), (uint8_t)((v >> 8) & 0xff)};
        return put(b, 2);
    }
};

// "GIF89a", logical screen descriptor, global colour table (ref giflib.cpp:803-860 + EGifPutScreenDesc)
static bool write_screen(GifWriter& w, const GifReader& r, int width, int height) {
    // packed byte: colour-table flag | (SColorResolution - 1) << 4 | sort flag | BitsPerPixel - 1, which for a
    // file with a global table is the source's own byte; without one giflib writes 0x07 in the low bits
    const uint8_t packed = r.gct ? r.packed : (uint8_t)((r.packed & 0x70) | 0x07);
    if (!w.put("GIF89a", 6) || !w.put16(width) || !w.put16(height) || !w.put8(packed) ||
        !w.put8((uint8_t)encoder_bg_index(r)) || !w.put8(r.aspect))
        return false;
    if (r.gct && !w.put(r.gct, (size_t)r.gct_colors * 3)) return false;
    return true;
}

// ref giflib.cpp:1100-1124 (EGifPutExtensionLeader / Block / Trailer per stored sub-block)
static bool write_extensions(GifWriter& w, const std::vector<GifExt>& ext) {
    for (size_t i = 0; i < ext.size(); i++) {
        const GifExt& b = ext[i];
        if (b.function != 0) {
            if (!w.put8(0x21) || !w.put8((uint8_t)b.function)) return false;
        }
        if (!w.put8((uint8_t)b.bytes.size()) || !w.put(b.bytes.data(), b.bytes.size())) return false;
        if (i + 1 == ext.size() || ext[i + 1].function != 0) {
            if (!w.put8(0)) return false;
        }
    }
    return true;
}

// ref giflib.cpp:1126-1183: a frame's extensions, image descriptor (at 0, 0), local colour table and LZW code size;
// the code stream follows
static bool write_frame_head(GifWriter& w, const std::vector<GifExt>& ext, int cols, int rows, bool interlace,
                             const uint8_t* local, int nlocal, int code_bits) {
    if (!write_extensions(w, ext)) return false;
    const uint8_t flags = (uint8_t)((local ? 0x80 : 0) | (interlace ? 0x40 : 0) | (local ? color_bits(nlocal) - 1 : 0));
    if (!w.put8(0x2C) || !w.put16(0) || !w.put16(0) || !w.put16(cols) || !w.put16(rows) || !w.put8(flags)) return false;
    if (local && !w.put(local, (size_t)nlocal * 3)) return false;
    return w.put8((uint8_t)code_bits);
}

// ------------------------------------------------------------------ device kernels

struct GifFrameDev {
    const uint8_t* lzw;   // concatenated sub-block payload
    uint32_t lzw_len;
    int min_code;
    uint32_t npix;
    uint8_t* indices;     // npix bytes
};

// LZW dictionary of one frame in shared memory: per entry the classic prefix link, its last pixel and the string
// length in one word, plus the FIRST pixel of the string (what the next entry needs, so that creating an entry never
// walks a chain).
struct GifLzwShared {
    uint32_t link[4096];  // prefix code | last pixel << 12 | string length << 20
    uint8_t first[4096];
};

// One frame's code stream, decoded by one warp, 32 codes per round.  giflib's DGifDecompressInput / DGifDecompressLine
// state machine (ref giflib.cpp:181-184 -> DGifGetLine): `running` counts the codes read since the last clear
// (+ clear + 2), the code width grows when it passes maxcode1 = 1 << bits, every code after the first one of a
// segment adds entry `top` = previous string + first pixel of this one.  None of that depends on the VALUES of the
// codes (clear codes aside), so a round is
//   1. widths in closed form -> prefix sum -> every lane reads its own code; the round ends in front of the first
//      clear / EOF / out-of-data code, which the next round handles alone;
//   2. validity and the entry each code creates, again in closed form; the round is cut at the first invalid code;
//   3. (length, first pixel) per code: from the table, or -- a code that names an entry created inside this round --
//      from the lane in front of the creator, by pointer jumping;
//   4. prefix sum of the lengths = where each string goes; the round is cut where the frame is full;
//   5. the new entries are written, then every lane walks its own chain backwards, storing pixels.
// The serial chain walk (one shared-memory load per pixel) is the cost that is left, and 32 of them run at once.
// (The first version kept entries as spans of the OUTPUT and copied them warp-wide from global memory: ~650 cycles
// per code, most of it the L1 miss after the store in front.)
__device__ __forceinline__ int gif_lzw_decode_frame(const GifFrameDev& f, GifLzwShared& sh) {
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int clear = 1 << f.min_code, eof = clear + 1;
    int bits = f.min_code + 1, running = clear + 2, top = clear + 2;  // maxcode1 == 1 << bits throughout
    const uint64_t total_bits = 8ull * f.lzw_len;
    uint64_t bp = 0;    // bit position of the next code
    uint32_t o = 0;     // pixels written
    int prev_code = 0, prev_len = 0, prev_first = 0;  // previous string of this segment; prev_len 0 = none
    int status = 0;
    while (o < f.npix) {
        // closed-form widths need running <= maxcode1 (true from the first clear state on for min_code >= 1; a
        // min_code of 0 starts with running 3 > 2 and gets there within two codes: those go one per round)
        const bool regular = running <= (1 << bits) || bits >= 12;
        const int r_j = min(running + lane, 4097);  // `running` when this lane's code is read
        const int w_j = regular ? min(12, max(bits, 32 - __clz(r_j - 1))) : bits;
        int incl = w_j;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(FULL, incl, d);
            if (lane >= d) incl += t;
        }
        const uint64_t at = bp + (uint64_t)(incl - w_j);
        int code = -1;
        if (at + (uint64_t)w_j <= total_bits && (regular || lane == 0)) {
            const uintptr_t a = reinterpret_cast<uintptr_t>(f.lzw + (at >> 3));
            const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);  // q[1]: inside the padded buffer
            code = (int)((__funnelshift_r(q[0], q[1], 8 * (int)(a & 3) + (int)(at & 7))) & ((1u << w_j) - 1));
        }
        const bool special = code < 0 || code == clear || code == eof || (!regular && lane > 0);
        int n = __ffs(__ballot_sync(FULL, special)) - 1;
        if (n < 0) n = 32;
        if (n == 0) {
            const int c0 = __shfl_sync(FULL, code, 0);
            if (c0 < 0 || c0 == eof) {  // data ran out / EOF code before the last pixel: an error for giflib
                status = -1;
                break;
            }
            bp += bits;  // a clear code
            bits = f.min_code + 1;
            running = clear + 2;
            top = clear + 2;
            prev_len = 0;
            continue;
        }
        // entry created by the code of lane j: none by the first code of a segment, none once the table is full
        const int made_before = prev_len ? lane : max(lane - 1, 0);
        const int top_j = min(4096, top + made_before);
        const bool creates = (lane > 0 || prev_len) && top_j < 4096 && min(running + lane + 1, 4097) - 2 == top_j;
        const bool in_table = code < clear || (code > eof && code < top);
        const bool in_round = !in_table && code > eof && (code < top_j || (code == top_j && creates));
        const bool invalid = lane < n && !in_table && !in_round;
        const int iv = __ffs(__ballot_sync(FULL, invalid)) - 1;
        const bool corrupt = iv >= 0;
        if (corrupt) n = iv;
        // (length, first pixel)
        int len = 0, first = 0;
        bool done = lane >= n;
        if (!done && in_table) {
            if (code < clear) { len = 1; first = code; }
            else { len = (int)(sh.link[code] >> 20); first = sh.first[code]; }
            done = true;
        }
        const int dep = code - top + (prev_len ? 0 : 1) - 1;  // lane whose string this code's entry extends; -1 = prev
        while (!__all_sync(FULL, done)) {
            const int src = max(dep, 0) & 31;
            const int d_len = __shfl_sync(FULL, len, src), d_first = __shfl_sync(FULL, first, src);
            const bool d_done = __shfl_sync(FULL, done, src);
            if (!done) {
                if (dep < 0) { len = prev_len + 1; first = prev_first; done = true; }
                else if (d_done) { len = d_len + 1; first = d_first; done = true; }
            }
        }
        int lsum = lane < n ? len : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(FULL, lsum, d);
            if (lane >= d) lsum += t;
        }
        const uint32_t room = f.npix - o;
        const int full_at = __ffs(__ballot_sync(FULL, lane < n && (uint32_t)lsum >= room)) - 1;
        bool complete = false;
        if (full_at >= 0) { n = full_at + 1; complete = true; }  // the codes behind are never read
        if (n == 0) { status = -1; break; }                        // (only when the first code of the round is invalid)
        // new entries: previous string + first pixel of this one
        const int p_code = __shfl_up_sync(FULL, code, 1), p_len = __shfl_up_sync(FULL, len, 1),
                  p_first = __shfl_up_sync(FULL, first, 1);
        if (lane < n && creates) {
            const int pc = lane ? p_code : prev_code, pl = lane ? p_len : prev_len, pf = lane ? p_first : prev_first;
            sh.link[top_j] = (uint32_t)pc | (uint32_t)first << 12 | (uint32_t)(pl + 1) << 20;
            sh.first[top_j] = (uint8_t)pf;
        }
        __syncwarp();
        // (Staging the strings in shared memory and storing whole words was measured: 15 % SLOWER.  The loop is bound by
        // the latency of the dependent shared-memory load with ~2.5 warps per scheduler, not by the byte stores.)
        if (lane < n) {
            uint32_t p = o + (uint32_t)(lsum - 1);  // last pixel of this string
            int c = code;
            while (c > eof) {
                const uint32_t l = sh.link[c];
                if (p < f.npix) f.indices[p] = (uint8_t)(l >> 12);
                p--;
                c = (int)(l & 0xFFFu);
            }
            if (p < f.npix) f.indices[p] = (uint8_t)c;
        }
        __syncwarp();
        // state behind the last code of the round
        const int last = n - 1;
        prev_code = __shfl_sync(FULL, code, last);
        const int n_len = __shfl_sync(FULL, len, last);
        prev_first = __shfl_sync(FULL, first, last);
        const int total = __shfl_sync(FULL, lsum, last);
        bp += (uint64_t)__shfl_sync(FULL, incl, last);
        top = min(4096, top + (prev_len ? n : max(n - 1, 0)));
        prev_len = n_len;
        if (regular) {
            running = min(running + n, 4097);
            bits = min(12, max(bits, 32 - __clz(running - 1)));
        } else if (running < 4097 && ++running > (1 << bits) && bits < 12) {
            bits++;
        }
        o += min((uint32_t)total, room);
        if (complete) break;
        if (corrupt) { status = -1; break; }
    }
    return status;
}

// Sub-block removal and LZW run one warp per FRAME (frames are independent code streams); the compositor runs one
// thread per canvas PIXEL and walks the frames of its animation in order -- disposal, snapshot and drawing only ever
// look at the same pixel of the previous state (ref giflib.cpp:349-568), so the frame sequence is a per-pixel
// recurrence over (canvas pixel, snapshot pixel).

struct GifFrameJob {
    uint64_t data_pos;   // first sub-block length byte, offset from the scratch base (batch decode only)
    uint64_t lzw_off;    // contiguous code stream (written by the deblock kernel, or gathered on the host)
    uint64_t idx_off;    // npix palette indices
    uint64_t colors_off; // colour table in force (inside the uploaded file)
    uint32_t lzw_len, npix;
    int32_t min_code;
    int32_t fl, ft, fw, fh, interlace, transparent, ncolors;
    int32_t prev_disposal, pl, pt, pw, ph;
    int32_t status;
    int32_t canvas;  // canvas index the composited frame is stored at, from `canvases`; -1: composited, not stored
};
struct GifAnimJob {
    int32_t first_frame, nframes;
    uchar4 bg;        // B, G, R, A of the background fill
    int32_t fill_bg;  // the job's first frame is the animation's first: it starts from the background fill
    uint8_t* snap;    // null: canvas and snapshot start zeroed; else resume from the canvas of the job's first
                      // frame and from this snapshot (BGRA, packed), and store the snapshot back at the end
};

constexpr int kGifDeblockWarps = 4;
__global__ void __launch_bounds__(kGifDeblockWarps * 32) gif_deblock_kernel(GifFrameJob* jobs, uint8_t* base, int n) {
    const int f = blockIdx.x * kGifDeblockWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= n) return;
    const GifFrameJob j = jobs[f];
    const uint8_t* src = base + j.data_pos;
    uint8_t* dst = base + j.lzw_off;
    uint32_t o = 0;
    while (o < j.lzw_len) {
        const uint32_t len = src[0];  // every lane reads the same byte (a broadcast load)
        if (len == 0) break;
        const uint32_t take = min(len, j.lzw_len - o);
        for (uint32_t i = lane; i < take; i += 32) dst[o + i] = src[1 + i];
        o += take;
        src += 1 + len;
    }
    for (uint32_t i = lane; i < 16; i += 32) dst[o + i] = 0;  // the word reader may look one word past the end
}

__global__ void __launch_bounds__(32) gif_lzw_kernel(GifFrameJob* jobs, uint8_t* base) {
    __shared__ GifLzwShared sh;
    GifFrameJob& j = jobs[blockIdx.x];
    GifFrameDev f{base + j.lzw_off, j.lzw_len, j.min_code, j.npix, base + j.idx_off};
    const int status = gif_lzw_decode_frame(f, sh);
    if (threadIdx.x == 0) j.status = status;
}

// (launched with 128 threads; the bound holds it at 32 registers, a full SM of warps, with no spill: the store slot's
// address would otherwise take two more)
__global__ void __launch_bounds__(128, 16)
    gif_compose_kernel(const GifAnimJob* anims, const GifFrameJob* jobs, const uint8_t* base, int cw, int chh, uint8_t* canvases,
                       size_t canvas_stride) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= cw) return;
    const GifAnimJob a = anims[blockIdx.z];
    const size_t at = ((size_t)y * cw + x) * 4;
    uchar4 px = make_uchar4(0, 0, 0, 0), snap = make_uchar4(0, 0, 0, 0);  // canvas and prev_frame_bgra start zeroed
    if (a.snap) {
        px = *reinterpret_cast<const uchar4*>(canvases + (size_t)a.first_frame * canvas_stride + at);
        snap = *reinterpret_cast<const uchar4*>(a.snap + at);
    }
    bool fill = a.fill_bg;  // the job's first frame starts from the background fill
    for (const GifFrameJob *c = jobs + a.first_frame, *end = c + a.nframes; c < end; c++) {
        if (fill) {
            px = a.bg;
            fill = false;
        } else {
            const bool in_prev = x >= c->pl && x < c->pl + c->pw && y >= c->pt && y < c->pt + c->ph;
            if (in_prev && c->prev_disposal == 2) px = a.bg;
            else if (in_prev && c->prev_disposal == 3) px = snap;
            snap = px;  // snapshot after disposal, before drawing
        }
        const int fx = x - c->fl, fy = y - c->ft;
        if (fx >= 0 && fx < c->fw && fy >= 0 && fy < c->fh) {
            int row = fy;
            if (c->interlace) {
                const int h = c->fh;
                const int n0 = (h + 7) / 8, n1 = (h + 3) / 8, n2 = (h + 1) / 4;
                if ((fy & 7) == 0) row = fy / 8;
                else if ((fy & 7) == 4) row = n0 + fy / 8;
                else if ((fy & 3) == 2) row = n0 + n1 + fy / 4;
                else row = n0 + n1 + n2 + fy / 2;
            }
            const int idx = base[c->idx_off + (size_t)row * c->fw + fx];
            if (idx != c->transparent && idx < c->ncolors) {
                const uint8_t* pal = base + c->colors_off + (size_t)idx * 3;
                px = make_uchar4(pal[2], pal[1], pal[0], 255);
            }
        }
        if (c->canvas >= 0) *reinterpret_cast<uchar4*>(canvases + (size_t)c->canvas * canvas_stride + at) = px;
    }
    // (re-read: the snapshot pointer is not held across the frame loop)
    uint8_t* const sp = anims[blockIdx.z].snap;
    if (sp) *reinterpret_cast<uchar4*>(sp + at) = snap;
}

// LZW and compositing of `nf` frame jobs, whose code streams are already contiguous, and `n` animation jobs, all in
// device memory; the jobs' offsets are relative to `base`.
static void gif_decode_launch(GifFrameJob* d_jobs, int nf, const GifAnimJob* d_anims, int n, uint8_t* base, int cw,
                              int chh, uint8_t* canvases, size_t canvas_stride, cudaStream_t st) {
    // 24 KB of dictionary per frame: let as many frames as possible share an SM (set once, thread-safe)
    static const cudaError_t carveout = cudaFuncSetAttribute(
        gif_lzw_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    (void)carveout;
    gif_lzw_kernel<<<nf, 32, 0, st>>>(d_jobs, base);
    gif_compose_kernel<<<dim3(ceil_div(cw, 128), chh, n), 128, 0, st>>>(d_anims, d_jobs, base, cw, chh, canvases,
                                                                        canvas_stride);
    g_launches += 2;
}

// ------------------------------------------------------------------ frame jobs, batch decode (xbatch.cu)

struct GifFramePlan {
    size_t data_pos = 0, colors_pos = 0;
    uint32_t lzw_len = 0;
    int left = 0, top = 0, width = 0, height = 0, interlace = 0, ncolors = 0, min_code = 0;
    int transparent = -1, disposal = 0, delay = 0;
    // what the GIF writer reads: a local colour table?, the extension blocks as the per-image decoder holds them when
    // the encoder reads them (forced transparency included, the encoder's background drop applied) and that GCB
    bool local = false;
    std::vector<GifExt> ext;
    GifGcb enc_gcb;
    size_t end_pos = 0;  // behind the frame's block terminator
};
struct GifAnimPlan {
    int sw = 0, sh = 0, loop_count = 1;
    uint32_t bgcolor = 0xFFFFFFFFu;   // gifDecoder.BackgroundColor()
    uint8_t bg[4] = {255, 255, 255, 255};  // B, G, R, A of the first frame's fill (ref giflib.cpp:595-636)
    std::vector<GifFramePlan> frames;
    std::vector<GifExt> trailing_ext;  // extension blocks behind the last frame (giflib_encoder_flush writes them)
    GifReader rd;                      // the screen descriptor and global colour table (borrows the file's bytes)
    int palette_runs = 0;              // maximal runs of consecutive frames with byte-equal colour maps
    size_t lzw_total = 0, idx_total = 0, file_len = 0;
};

// The job of frame `f`, whose sub-blocks and colour table sit at `base` + f.data_pos / f.colors_pos, drawn after a
// frame with disposal `prev_disposal` over (pl, pt, pw, ph).  That previous rectangle is clipped to the cw x chh canvas
// exactly as ref giflib.cpp:407-436 does.  lzw_off and idx_off are the caller's.
static GifFrameJob gif_frame_job(const GifFramePlan& f, size_t base, int prev_disposal, int pl, int pt, int pw, int ph,
                                 int cw, int chh) {
    GifFrameJob j{};
    j.data_pos = base + f.data_pos;
    j.colors_off = base + f.colors_pos;
    j.lzw_len = f.lzw_len;
    j.npix = (uint32_t)((size_t)f.width * f.height);
    j.min_code = f.min_code;
    j.fl = f.left; j.ft = f.top; j.fw = f.width; j.fh = f.height;
    j.interlace = f.interlace;
    j.transparent = f.transparent;
    j.ncolors = f.ncolors;
    j.prev_disposal = prev_disposal;
    if (pl < 0) { pw += pl; pl = 0; }
    if (pt < 0) { ph += pt; pt = 0; }
    if (pl + pw > cw) pw = cw - pl;
    if (pt + ph > chh) ph = chh - pt;
    j.pl = pl; j.pt = pt; j.pw = pw < 0 ? 0 : pw; j.ph = ph < 0 ? 0 : ph;
    return j;
}

// The walk gifDecoder + ImageOps.Transform would make over a WELL-FORMED file (every record readable, every
// frame with a colour table, terminator present); anything else returns nullptr and the file takes the
// per-image path, which reproduces the reference's handling of damaged files.
// first_frame_only: the walk of a Transform that stops after frame 0 (DisableAnimatedOutput).  The per-image decoder
// reads nothing behind frame 0's image data then, so neither does the plan: later records may be damaged or missing,
// max_frames is not consulted, and the blocks giflib_encoder_flush writes behind the frame are the ones the decoder
// still holds -- frame 0's own, after the forced transparency and before the encoder's background drop.  The plan's
// file span ends with frame 0's image data.
GifAnimPlan* gif_plan_parse(const uint8_t* data, size_t len, int max_frames, bool first_frame_only) {
    GifReader r;
    r.p = data;
    r.n = len;
    if (!r.open() || r.sw <= 0 || r.sh <= 0) return nullptr;
    std::unique_ptr<GifAnimPlan> p(new GifAnimPlan);
    p->sw = r.sw;
    p->sh = r.sh;
    p->file_len = len;
    p->rd = r;
    bool found_loop = false, found_gcb = false;
    GifGcb first_gcb;
    std::vector<GifExt> ext;   // as the per-image decoder's gif->ExtensionBlocks
    std::vector<GifGcb> gcbs;  // graphic control blocks since the last frame
    for (;;) {
        const int rec = r.record();
        if (rec < 0) return nullptr;
        if (rec == 2) break;
        if (rec == 1) {
            const size_t e0 = ext.size();
            if (!read_extension(r, &ext, &gcbs)) return nullptr;
            if (e0 == ext.size()) continue;
            const GifExt& e = ext[e0];
            if (e.function == 0xF9) {
                GifGcb g;
                if (!gcb_from_block(e.bytes.data(), (int)e.bytes.size(), &g)) return nullptr;  // malformed: per image
                if (!found_gcb) {
                    found_gcb = true;
                    first_gcb = g;
                }
            } else if (!found_loop && e.function == 0xFF && e.bytes.size() >= 11 && !memcmp(e.bytes.data(), "NETSCAPE2.0", 11) &&
                       e0 + 1 < ext.size() && ext[e0 + 1].function == 0) {
                const std::vector<uint8_t>& d2 = ext[e0 + 1].bytes;
                if (d2.size() >= 3 && d2[0] == 1) {
                    p->loop_count = d2[1] | (d2[2] << 8);
                    found_loop = true;
                }
            }
            continue;
        }
        GifImage im;
        if (!r.image_header(&im)) return nullptr;
        if (im.width <= 0 || im.height <= 0 || im.width > 10000 || im.height > 10000) return nullptr;
        GifFramePlan f;
        f.left = im.left; f.top = im.top; f.width = im.width; f.height = im.height;
        f.interlace = im.interlace ? 1 : 0;
        f.min_code = im.min_code;
        const uint8_t* colors = im.colors ? im.colors : r.gct;
        f.ncolors = im.colors ? im.ncolors : r.gct_colors;
        if (!colors) return nullptr;
        f.colors_pos = (size_t)(colors - data);
        f.data_pos = r.pos;
        size_t total = 0;
        for (;;) {
            const uint8_t* d;
            int n;
            if (!r.sub_block(&d, &n)) return nullptr;
            if (n == 0) break;
            total += (size_t)n;
        }
        if (total > 0xFFFFFF00u) return nullptr;
        f.lzw_len = (uint32_t)total;
        f.end_pos = r.pos;
        const GifGcb g = gcbs.empty() ? GifGcb() : gcbs.back();
        f.transparent = g.transparent;
        f.disposal = g.disposal;
        f.delay = g.delay;
        if (p->frames.empty()) {
            uint8_t R, G, B, A;
            background_color(r, g, &R, &G, &B, &A);
            p->bg[0] = B; p->bg[1] = G; p->bg[2] = R; p->bg[3] = A;
        }
        f.local = im.colors != nullptr;
        force_partial_transparent(ext, g, im, f.ncolors, r.sw, r.sh);
        if (first_frame_only) p->trailing_ext = ext;
        f.enc_gcb = encoder_frame_gcb(ext, r, f.local, p->bg[3] == 255);
        f.ext.swap(ext);
        ext.clear();  // extensions are cleared after a frame (ref giflib.cpp:289-296)
        gcbs.clear();
        const GifFramePlan* prev = p->frames.empty() ? nullptr : &p->frames.back();
        if (!prev || prev->ncolors != f.ncolors || memcmp(data + prev->colors_pos, colors, (size_t)f.ncolors * 3))
            p->palette_runs++;
        p->lzw_total += round_up(total + 32, (size_t)16);
        p->idx_total += round_up((size_t)im.width * im.height + 64, (size_t)16);
        p->frames.push_back(f);
        if (first_frame_only) {
            p->file_len = r.pos;
            break;
        }
        if ((int)p->frames.size() > max_frames) return nullptr;
    }
    if (p->frames.empty()) return nullptr;
    if (!first_frame_only) p->trailing_ext.swap(ext);
    // gifDecoder.BackgroundColor() (ref giflib.cpp:1308-1431): set when the walk meets the file's first graphic
    // control block; a file that reaches its terminator without one keeps the initial white with alpha 0
    if (found_gcb) {
        uint8_t R, G, B, A;
        background_color(r, first_gcb, &R, &G, &B, &A);
        p->bgcolor = ((uint32_t)A << 24) | ((uint32_t)R << 16) | ((uint32_t)G << 8) | B;
    } else {
        p->bgcolor = 0x00FFFFFFu;
    }
    return p.release();
}
void gif_plan_free(GifAnimPlan* p) { delete p; }
void gif_plan_info(const GifAnimPlan* p, int* width, int* height, int* nframes, uint32_t* bgcolor, int* loop_count) {
    if (width) *width = p->sw;
    if (height) *height = p->sh;
    if (nframes) *nframes = (int)p->frames.size();
    if (bgcolor) *bgcolor = p->bgcolor;
    if (loop_count) *loop_count = p->loop_count;
}
size_t gif_plan_file_bytes(const GifAnimPlan* p) { return p->file_len; }
// (a cut plan is decoded, never written: the writer's trailing extensions and palette runs stay the full walk's)
size_t gif_plan_cut(GifAnimPlan* p, int last) {
    p->frames.resize((size_t)last + 1);
    p->lzw_total = p->idx_total = 0;
    for (const GifFramePlan& f : p->frames) {
        p->lzw_total += round_up((size_t)f.lzw_len + 32, (size_t)16);
        p->idx_total += round_up((size_t)f.width * f.height + 64, (size_t)16);
    }
    p->file_len = p->frames.back().end_pos;
    return p->file_len;
}
int gif_plan_delay_ms(const GifAnimPlan* p, int frame) { return p->frames[(size_t)frame].delay * 10; }  // ref giflib.go:212
size_t gif_plan_device_bytes(const GifAnimPlan* p) {
    return round_up(p->file_len + 64, (size_t)256) + p->lzw_total + p->idx_total +
           p->frames.size() * (sizeof(GifFrameJob) + 64) + 4096;
}

int gif_decode_batch(GifAnimPlan* const* plans, const uint8_t* const* files, const size_t* file_len, int n,
                     uint8_t* d_scratch, size_t scratch_bytes, uint8_t* d_canvases, size_t canvas_stride,
                     const int* first_frame, int* h_status, cudaStream_t st, const int* canvas_of) {
    if (n <= 0) return LP_OK;
    const int nf = first_frame[n];
    std::vector<GifFrameJob> jobs((size_t)nf);
    std::vector<GifAnimJob> anims((size_t)n);
    size_t off = 0;
    std::vector<size_t> file_off((size_t)n);
    for (int a = 0; a < n; a++) {
        file_off[a] = off;
        off += round_up(file_len[a] + 64, (size_t)256);
    }
    const int cw = plans[0]->sw, chh = plans[0]->sh;
    for (int a = 0; a < n; a++) {
        const GifAnimPlan& p = *plans[a];
        if (p.sw != cw || p.sh != chh) return LP_ERR_BAD_ARGUMENT;
        anims[a].first_frame = first_frame[a];
        anims[a].nframes = (int)p.frames.size();
        anims[a].bg = make_uchar4(p.bg[0], p.bg[1], p.bg[2], p.bg[3]);
        anims[a].fill_bg = 1;
        int prev_disposal = 0, pl = 0, pt = 0, pw = 0, ph = 0;
        for (size_t k = 0; k < p.frames.size(); k++) {
            const GifFramePlan& f = p.frames[k];
            GifFrameJob& j = jobs[(size_t)first_frame[a] + k];
            j = gif_frame_job(f, file_off[a], prev_disposal, pl, pt, pw, ph, cw, chh);
            j.lzw_off = off;
            j.canvas = canvas_of ? canvas_of[first_frame[a] + k] : first_frame[a] + (int)k;
            off += round_up((size_t)f.lzw_len + 32, (size_t)16);
            prev_disposal = f.disposal;
            pl = f.left; pt = f.top; pw = f.width; ph = f.height;
        }
    }
    for (int k = 0; k < nf; k++) {
        jobs[k].idx_off = off;
        off += round_up((size_t)jobs[k].npix + 64, (size_t)16);
    }
    off = round_up(off, (size_t)256);
    const size_t jobs_off = off;
    off += round_up((size_t)nf * sizeof(GifFrameJob), (size_t)256);
    const size_t anims_off = off;
    off += round_up((size_t)n * sizeof(GifAnimJob), (size_t)256);
    if (off > scratch_bytes) return LP_ERR_BUF_TOO_SMALL;
    GifFrameJob* d_jobs = reinterpret_cast<GifFrameJob*>(d_scratch + jobs_off);
    GifAnimJob* d_anims = reinterpret_cast<GifAnimJob*>(d_scratch + anims_off);
    for (int a = 0; a < n; a++)
        LP_CUDA_OK(cudaMemcpyAsync(d_scratch + file_off[a], files[a], file_len[a], cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(d_jobs, jobs.data(), (size_t)nf * sizeof(GifFrameJob), cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(d_anims, anims.data(), (size_t)n * sizeof(GifAnimJob), cudaMemcpyHostToDevice, st));
    gif_deblock_kernel<<<ceil_div(nf, kGifDeblockWarps), kGifDeblockWarps * 32, 0, st>>>(d_jobs, d_scratch, nf);
    g_launches++;
    gif_decode_launch(d_jobs, nf, d_anims, n, d_scratch, cw, chh, d_canvases, canvas_stride, st);
    LP_CUDA_OK(cudaGetLastError());
    LP_CUDA_OK(cudaMemcpyAsync(jobs.data(), d_jobs, (size_t)nf * sizeof(GifFrameJob), cudaMemcpyDeviceToHost, st));
    LP_CUDA_OK(cudaStreamSynchronize(st));
    for (int a = 0; a < n; a++) {
        h_status[a] = 0;
        for (int k = first_frame[a]; k < first_frame[a + 1]; k++)
            if (jobs[k].status != 0) h_status[a] = LP_ERR_DECODING_FAILED;
    }
    return LP_OK;
}

// ------------------------------------------------------------------ encoder kernels
// ref giflib.cpp:934-1098 (giflib_encoder_render_frame): every BGRA pixel of a frame becomes a palette index.  The
// reference memoises "best palette entry" per 15-bit crushed colour, and the FIRST pixel that consults a bucket
// decides its entry (from the bucket's midpoint, or from the pixel itself when it is near black / white).  The memo
// lives on from frame to frame while the colour map stays byte-equal and is cleared by any other map, so a PALETTE
// RUN -- a maximal sequence of consecutive frames of one animation with byte-equal colour maps -- shares one table
// and visits its pixels in the order (frame position in the run, raster index).  The kernels take a list of frames:
//   first:  every consulting pixel offers its key (position, raster index) to its bucket's owner, atomicMin over the
//           run's table -- the owner is the pixel the serial encoder would have resolved the bucket for;
//   bucket: every claimed bucket of every run is resolved from its owner's colour and its owner frame's transparent
//           index (all 32768 buckets of a run are visited; unclaimed ones return at once);
//   map:    every pixel takes its bucket's entry; `least` is the owner's stored distance for the owner itself and the
//           pixel's own distance to the entry otherwise, exactly what the serial memo sees.
// A table may start non-empty (the per-image encoder keeps its memo between calls): a bucket present at the start is
// never claimed, and every pixel of it measures its own distance, as in the serial encoder.

struct GifEncRun {
    int16_t* lookup;             // [32768] palette index per crushed colour, -1 = absent
    unsigned long long* owner;   // [32768] (position in the run << 32 | raster index) of the bucket's first pixel
    int* owner_dist;             // [32768] distance the owner saw (measured from the compare colour)
    int first_job;               // the run's first frame
    int pad_;
};
struct GifEncJob {
    const uint8_t* frame;    // BGRA, rows `step` apart
    const uint8_t* prev;     // previous frame of the animation (same size, rows `prev_step` apart), if prev_valid
    const uint8_t* palette;  // RGB, ncolors entries
    uint8_t* pixels;         // out: width * height indices
    uint8_t* out;            // out: sub-blocked LZW code stream, out_cap bytes
    uint32_t* out_len;       // bytes written, 0xFFFFFFFF when out_cap was too small
    uint64_t step, prev_step;
    int32_t width, height, ncolors, transparent /* -1 none */, prev_valid;
    int32_t run, pos;        // palette run and the frame's position in it
    int32_t code_bits, interlace;
    uint32_t out_cap;
};

__device__ __forceinline__ int rgb_distance(int r0, int g0, int b0, int r1, int g1, int b1) {
    return abs(r0 - r1) + abs(g0 - g1) + abs(b0 - b1);
}

// grid: (blocks_x per frame * frames, max height), 128 threads; frame = blockIdx.x / blocks_x
__global__ void gif_enc_first_kernel(const GifEncJob* jobs, const GifEncRun* runs, int blocks_x) {
    const GifEncJob& j = jobs[blockIdx.x / blocks_x];
    const int x = (blockIdx.x % blocks_x) * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= j.width || y >= j.height) return;
    const uint8_t* s = j.frame + (size_t)y * j.step + (size_t)x * 4;
    if (s[3] < 128 && j.transparent != -1) return;  // becomes the transparent index, never consults the table
    const uint32_t crushed = ((uint32_t)(s[2] >> 3) << 10) | ((uint32_t)(s[1] >> 3) << 5) | (s[0] >> 3);
    const GifEncRun& r = runs[j.run];
    if (r.lookup[crushed] < 0)
        atomicMin(&r.owner[crushed], (unsigned long long)j.pos << 32 | (uint32_t)(y * j.width + x));
}

// grid: 256 blocks per run, 128 threads
__global__ void gif_enc_bucket_kernel(const GifEncJob* jobs, const GifEncRun* runs) {
    const GifEncRun& r = runs[blockIdx.x >> 8];
    const int bucket = (blockIdx.x & 255) * blockDim.x + threadIdx.x;
    const unsigned long long key = r.owner[bucket];
    if (key == ~0ull) return;
    const GifEncJob& j = jobs[r.first_job + (int)(key >> 32)];
    const uint32_t idx = (uint32_t)key;
    const uint8_t* s = j.frame + (size_t)(idx / j.width) * j.step + (size_t)(idx % j.width) * 4;
    const int B = s[0], G = s[1], R = s[2];
    const bool extreme = (R > 240 && G > 240 && B > 240) || (R < 15 && G < 15 && B < 15);
    const int Rc = extreme ? R : (R & 0xf8) | 4, Gc = extreme ? G : (G & 0xf8) | 4, Bc = extreme ? B : (B & 0xf8) | 4;
    int least = 0x7fffffff, best = 0;
    for (int i = 0; i < j.ncolors; i++) {
        if (i == j.transparent) continue;
        const int d = rgb_distance(Rc, Gc, Bc, j.palette[i * 3], j.palette[i * 3 + 1], j.palette[i * 3 + 2]);
        if (d < least) {
            least = d;
            best = i;
        }
    }
    r.lookup[bucket] = (int16_t)best;
    r.owner_dist[bucket] = least;
}

__global__ void gif_enc_map_kernel(const GifEncJob* jobs, const GifEncRun* runs, int blocks_x) {
    const GifEncJob& j = jobs[blockIdx.x / blocks_x];
    const int x = (blockIdx.x % blocks_x) * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= j.width || y >= j.height) return;
    const uint8_t* s = j.frame + (size_t)y * j.step + (size_t)x * 4;
    const int B = s[0], G = s[1], R = s[2], A = s[3];
    const uint32_t idx = (uint32_t)(y * j.width + x);
    int best;
    if (A < 128 && j.transparent != -1) {
        best = j.transparent;
    } else {
        const GifEncRun& r = runs[j.run];
        const uint32_t crushed = ((uint32_t)(R >> 3) << 10) | ((uint32_t)(G >> 3) << 5) | (B >> 3);
        best = r.lookup[crushed];
        int least;
        if (r.owner[crushed] == ((unsigned long long)j.pos << 32 | idx)) least = r.owner_dist[crushed];
        else least = rgb_distance(R, G, B, j.palette[best * 3], j.palette[best * 3 + 1], j.palette[best * 3 + 2]);
        if (j.prev_valid && j.transparent != -1) {
            const uint8_t* l = j.prev + (size_t)y * j.prev_step + (size_t)x * 4;
            if (rgb_distance(R, G, B, l[2], l[1], l[0]) < least) best = j.transparent;
        }
    }
    j.pixels[idx] = (uint8_t)best;
}

// giflib's EGifCompressLine / EGifCompressOutput / EGifBufferedOutput (egif_lib.c), one frame per CTA.
// LZW is one serial chain; lane 0 walks it with the string table as an open-addressing hash in
// shared memory.  Output = the code stream cut into 255-byte sub-blocks + the block terminator.
__global__ void __launch_bounds__(32) gif_lzw_encode_kernel(const GifEncJob* jobs) {
    __shared__ uint32_t h_key[8192];
    __shared__ uint16_t h_val[8192];
    for (int i = threadIdx.x; i < 8192; i += 32) h_key[i] = 0xFFFFFFFFu;
    __syncwarp();
    if (threadIdx.x != 0) return;
    const GifEncJob& j = jobs[blockIdx.x];
    const uint8_t* pixels = j.pixels;
    const int width = j.width, height = j.height, interlace = j.interlace, bpp = j.code_bits;
    uint8_t* out = j.out;
    const uint32_t out_cap = j.out_cap;
    const int clear = 1 << bpp, eof = clear + 1;
    const uint32_t mask = (1u << bpp) - 1;
    int running_code = eof + 1, running_bits = bpp + 1, max_code1 = 1 << running_bits;
    uint32_t shift_dword = 0;
    int shift_state = 0;
    uint32_t pos = 0, blk_start = 0;
    int blk_n = 0;
    bool overflow = false;
    auto put_byte = [&](uint32_t b) {
        if (blk_n == 0) {  // open a sub-block: reserve its count byte
            if (pos >= out_cap) { overflow = true; return; }
            blk_start = pos++;
        }
        if (pos >= out_cap) { overflow = true; return; }
        out[pos++] = (uint8_t)b;
        if (++blk_n == 255) {
            out[blk_start] = 255;
            blk_n = 0;
        }
    };
    auto put_code = [&](int code) {
        shift_dword |= (uint32_t)code << shift_state;
        shift_state += running_bits;
        while (shift_state >= 8) {
            put_byte(shift_dword & 0xff);
            shift_dword >>= 8;
            shift_state -= 8;
        }
        if (running_code >= max_code1 && code <= 4095) max_code1 = 1 << ++running_bits;
    };
    put_code(clear);
    int crnt = -1;
    const int npass = interlace ? 4 : 1;
    for (int ps = 0; ps < npass; ps++) {
        const int y0 = interlace ? (ps == 0 ? 0 : ps == 1 ? 4 : ps == 2 ? 2 : 1) : 0;
        const int dy = interlace ? (ps == 0 ? 8 : ps == 1 ? 8 : ps == 2 ? 4 : 2) : 1;
        for (int y = y0; y < height; y += dy) {
            const uint8_t* line = pixels + (size_t)y * width;
            for (int x = 0; x < width; x++) {
                const uint32_t px = line[x] & mask;
                if (crnt < 0) {
                    crnt = (int)px;
                    continue;
                }
                const uint32_t key = ((uint32_t)crnt << 8) + px;
                uint32_t h = (key * 2654435761u) >> 19;
                int found = -1;
                while (h_key[h] != 0xFFFFFFFFu) {
                    if (h_key[h] == key) {
                        found = h_val[h];
                        break;
                    }
                    h = (h + 1) & 8191;
                }
                if (found >= 0) {
                    crnt = found;
                } else {
                    put_code(crnt);
                    crnt = (int)px;
                    if (running_code >= 4095) {
                        put_code(clear);
                        running_code = eof + 1;
                        running_bits = bpp + 1;
                        max_code1 = 1 << running_bits;
                        for (int i = 0; i < 8192; i++) h_key[i] = 0xFFFFFFFFu;
                    } else {
                        h_key[h] = key;  // h stopped on the empty slot of this key's probe sequence
                        h_val[h] = (uint16_t)running_code++;
                    }
                }
            }
        }
    }
    put_code(crnt);
    put_code(eof);
    while (shift_state > 0) {  // FLUSH_OUTPUT
        put_byte(shift_dword & 0xff);
        shift_dword >>= 8;
        shift_state -= 8;
    }
    if (blk_n > 0) out[blk_start] = (uint8_t)blk_n;
    if (pos < out_cap) out[pos++] = 0;  // block terminator
    else overflow = true;
    *j.out_len = overflow ? 0xFFFFFFFFu : pos;
}

// Palette mapping and LZW of `nj` frame jobs over `nruns` palette runs (both arrays in device memory); the runs'
// owner tables must hold ~0 and their lookup tables the memo each run starts from.
static void gif_encode_launch(const GifEncJob* d_jobs, int nj, const GifEncRun* d_runs, int nruns, int max_w, int max_h,
                              cudaStream_t st) {
    const int bx = ceil_div(max_w, 128);
    const dim3 grid((unsigned)(bx * nj), (unsigned)max_h);
    gif_enc_first_kernel<<<grid, 128, 0, st>>>(d_jobs, d_runs, bx);
    gif_enc_bucket_kernel<<<256 * nruns, 128, 0, st>>>(d_jobs, d_runs);
    gif_enc_map_kernel<<<grid, 128, 0, st>>>(d_jobs, d_runs, bx);
    gif_lzw_encode_kernel<<<nj, 32, 0, st>>>(d_jobs);
    g_launches += 4;
}

// LZW slot of a frame of `npix` pixels: 12-bit codes are at most 1.5 B/pixel, plus the sub-block bytes
static size_t gif_lzw_slot(size_t npix) { return round_up(npix * 2 + npix / 100 + 4096, (size_t)256); }
constexpr size_t kGifRunTableBytes = 32768 * (sizeof(int16_t) + sizeof(unsigned long long) + sizeof(int));

// ------------------------------------------------------------------ batch GIF writer (xbatch.cu)

size_t gif_plan_encode_bytes(const GifAnimPlan* p, int ow, int oh) {
    const size_t npix = (size_t)ow * oh;
    return (size_t)p->palette_runs * (kGifRunTableBytes + sizeof(GifEncRun)) +
           p->frames.size() * (round_up(npix + 64, (size_t)256) + 2 * gif_lzw_slot(npix) + 768 + sizeof(GifEncJob) + 16) +
           8 * 4096;
}

int gif_encode_batch(GifAnimPlan* const* plans, int n, const uint8_t* d_frames, size_t frame_stride, int ow, int oh,
                     const int* first_frame, uint8_t* d_scratch, size_t scratch_bytes, uint8_t* h_stage, size_t stage_bytes,
                     uint8_t* const* out, size_t out_cap, size_t* out_len, int* status, size_t* d2h, cudaStream_t st) {
    if (n <= 0) return LP_OK;
    const int nf = first_frame[n];
    const size_t npix = (size_t)ow * oh, pix_stride = round_up(npix + 64, (size_t)256), slot = gif_lzw_slot(npix);
    if (slot > stage_bytes) return LP_ERR_BUF_TOO_SMALL;
    int nruns = 0;
    for (int a = 0; a < n; a++) nruns += plans[a]->palette_runs;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        const size_t o = off;
        off += round_up(bytes, (size_t)256);
        return o;
    };
    const size_t lookup_off = take((size_t)nruns * 32768 * sizeof(int16_t));
    const size_t owner_off = take((size_t)nruns * 32768 * sizeof(unsigned long long));
    const size_t dist_off = take((size_t)nruns * 32768 * sizeof(int));
    const size_t pal_off = take((size_t)nf * 768), pix_off = take((size_t)nf * pix_stride);
    const size_t slot_off = take((size_t)nf * slot), packed_off = take((size_t)nf * slot + 16);
    const size_t len_off = take((size_t)nf * 4), offs_off = take((size_t)(nf + 1) * 8);
    const size_t jobs_off = take((size_t)nf * sizeof(GifEncJob)), runs_off = take((size_t)nruns * sizeof(GifEncRun));
    if (off > scratch_bytes) return LP_ERR_BUF_TOO_SMALL;
    uint8_t* d = d_scratch;
    uint32_t* d_len = reinterpret_cast<uint32_t*>(d + len_off);
    unsigned long long* d_offs = reinterpret_cast<unsigned long long*>(d + offs_off);
    std::vector<GifEncJob> jobs((size_t)nf);
    std::vector<GifEncRun> runs;
    std::vector<uint8_t> pal((size_t)nf * 768, 0);
    for (int a = 0; a < n; a++) {
        const GifAnimPlan& p = *plans[a];
        int pos = 0;
        for (size_t k = 0; k < p.frames.size(); k++) {
            const GifFramePlan& f = p.frames[k];
            const int j = first_frame[a] + (int)k;
            const uint8_t* colors = p.rd.p + f.colors_pos;
            const GifFramePlan* prev = k ? &p.frames[k - 1] : nullptr;
            if (!prev || prev->ncolors != f.ncolors || memcmp(p.rd.p + prev->colors_pos, colors, (size_t)f.ncolors * 3)) {
                const size_t r = runs.size();
                runs.push_back(GifEncRun{reinterpret_cast<int16_t*>(d + lookup_off) + r * 32768,
                                         reinterpret_cast<unsigned long long*>(d + owner_off) + r * 32768,
                                         reinterpret_cast<int*>(d + dist_off) + r * 32768, j, 0});
                pos = 0;
            }
            memcpy(&pal[(size_t)j * 768], colors, (size_t)f.ncolors * 3);
            GifEncJob& e = jobs[(size_t)j];
            e.frame = d_frames + (size_t)j * frame_stride;
            e.prev = prev ? d_frames + (size_t)(j - 1) * frame_stride : nullptr;
            e.palette = d + pal_off + (size_t)j * 768;
            e.pixels = d + pix_off + (size_t)j * pix_stride;
            e.out = d + slot_off + (size_t)j * slot;
            e.out_len = d_len + j;
            e.step = e.prev_step = (size_t)ow * 4;
            e.width = ow;
            e.height = oh;
            e.ncolors = f.ncolors;
            e.transparent = f.enc_gcb.transparent;
            e.prev_valid = prev && (prev->enc_gcb.disposal == 0 || prev->enc_gcb.disposal == 1);
            e.run = (int)runs.size() - 1;
            e.pos = pos++;
            e.code_bits = std::max(2, color_bits(f.ncolors));
            e.interlace = f.interlace;
            e.out_cap = (uint32_t)slot;
        }
    }
    if ((int)runs.size() != nruns) return LP_ERR_BAD_ARGUMENT;
    // every run starts from an empty memo and no owners: lookup and owner tables (adjacent) to all ones
    LP_CUDA_OK(cudaMemsetAsync(d + lookup_off, 0xFF, dist_off - lookup_off, st));
    LP_CUDA_OK(cudaMemcpyAsync(d + pal_off, pal.data(), pal.size(), cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(d + jobs_off, jobs.data(), jobs.size() * sizeof(GifEncJob), cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(d + runs_off, runs.data(), runs.size() * sizeof(GifEncRun), cudaMemcpyHostToDevice, st));
    gif_encode_launch(reinterpret_cast<const GifEncJob*>(d + jobs_off), nf, reinterpret_cast<const GifEncRun*>(d + runs_off),
                      nruns, ow, oh, st);
    LP_CUDA_OK(cudaGetLastError());
    const int rc = compact_launch(d + slot_off, slot, d_len, (uint32_t)slot, nf, d + packed_off, d_offs, st);
    if (rc) return rc;
    std::vector<unsigned long long> offs((size_t)nf + 1);
    std::vector<uint32_t> lens((size_t)nf);
    LP_CUDA_OK(cudaMemcpyAsync(offs.data(), d_offs, offs.size() * 8, cudaMemcpyDeviceToHost, st));
    LP_CUDA_OK(cudaMemcpyAsync(lens.data(), d_len, lens.size() * 4, cudaMemcpyDeviceToHost, st));
    LP_CUDA_OK(cudaStreamSynchronize(st));
    // the packed streams come home through the staging buffer, in windows when they do not fit it at once
    const size_t total = offs[(size_t)nf];
    size_t win0 = 0, win1 = 0;
    auto stream_of = [&](int j) -> const uint8_t* {
        const size_t b = offs[(size_t)j], e = b + lens[(size_t)j];
        if (b < win0 || e > win1) {
            win0 = b;
            win1 = std::min(total, b + stage_bytes);
            if (cudaMemcpyAsync(h_stage, d + packed_off + win0, win1 - win0, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                cudaStreamSynchronize(st) != cudaSuccess)
                return nullptr;
            *d2h += win1 - win0;
        }
        return h_stage + (b - win0);
    };
    *d2h += offs.size() * 8 + lens.size() * 4;
    for (int a = 0; a < n; a++) {
        const GifAnimPlan& p = *plans[a];
        GifWriter w{out[a], out_cap, 0};
        write_screen(w, p.rd, ow, oh);  // as in Transform, a header that does not fit is not checked
        int s = LP_OK;
        for (size_t k = 0; k < p.frames.size() && s == LP_OK; k++) {
            const GifFramePlan& f = p.frames[k];
            const int j = first_frame[a] + (int)k;
            if (lens[(size_t)j] == 0xFFFFFFFFu) {
                s = LP_ERR_INVALID_IMAGE;
                break;
            }
            const uint8_t* code = lens[(size_t)j] ? stream_of(j) : h_stage;
            if (!code) return LP_ERR_CUDA;
            if (!write_frame_head(w, f.ext, ow, oh, f.interlace != 0, f.local ? p.rd.p + f.colors_pos : nullptr, f.ncolors,
                                  std::max(2, color_bits(f.ncolors))) ||
                !w.put(code, lens[(size_t)j]))
                s = LP_ERR_INVALID_IMAGE;
        }
        if (s == LP_OK && (!write_extensions(w, p.trailing_ext) || !w.put8(0x3B))) s = LP_ERR_INVALID_IMAGE;
        status[a] = s;
        out_len[a] = s == LP_OK ? w.dst_offset : 0;
    }
    return LP_OK;
}
}  // namespace lp

using namespace lp;

// The mat handle is defined in abi_opencv.cu; the adapters only need these few accessors.
namespace lp {
const uint8_t* mat_host_bytes(const void* mat, size_t* len);
int mat_bind_device_frame(void* mat, int cols, int rows, int type, uint8_t** dev, size_t* step);
void mat_mark_device_written(void* mat);
int mat_device_view(void* mat, int* cols, int* rows, int* type, const uint8_t** dev, size_t* step);
}  // namespace lp

struct giflib_decoder_struct {
    GifReader rd;
    GifImage image;                    // gif->Image
    std::vector<GifGcb> pending_gcbs;  // graphic control blocks seen since the last frame
    std::vector<GifExt> ext;           // gif->ExtensionBlocks: every sub-block since the last frame
    bool seek_clear_extensions = false;
    bool have_read_first_frame = false;
    int prev_disposal = 0, prev_delay = 0, prev_left = 0, prev_top = 0, prev_width = 0, prev_height = 0;
    uint8_t bg_r = 255, bg_g = 255, bg_b = 255, bg_a = 255;
    int image_count = 0;
    // device state owned by the decoder: the canvas persists between frames here (the reference
    // relies on the Go framebuffer keeping its bytes), plus the restore-previous snapshot and the
    // per-frame scratch (jobs, colour table, code stream, indices)
    uint8_t* d_canvas = nullptr;
    uint8_t* d_prev = nullptr;
    uint8_t* d_scratch = nullptr;
    size_t scratch_cap = 0;
};

// ref giflib.cpp:26-58.  The GifFileType fields the reference reads back from `e->gif` live here.
struct giflib_encoder_struct : GifWriter {
    bool open = false;
    int sw = 0, sh = 0;
    bool has_gct = false;
    std::vector<uint8_t> gct;  // RGB triplets
    bool have_written_first_frame = false;
    int prev_frame_disposal = 0;
    std::vector<uint8_t> prev_colors;  // colour map used by the previous frame (for the memo's reuse test)
    bool have_prev_colors = false;
    // device state: the previous frame, the memo (a one-frame palette run whose table persists between frames while
    // the colour map does), and one frame job with its run and palette
    uint8_t* d_prev = nullptr;
    uint8_t* d_table = nullptr;  // kGifRunTableBytes: lookup, owner, owner_dist
    uint8_t* d_job = nullptr;    // GifEncJob, GifEncRun, palette, out_len
    uint8_t* d_pixels = nullptr;
    uint8_t* d_out = nullptr;
    size_t pixels_cap = 0, out_cap = 0;
};

extern "C" {

giflib_decoder giflib_decoder_create(const opencv_mat buf) {
    if (!buf) return nullptr;
    size_t len = 0;
    const uint8_t* bytes = mat_host_bytes(buf, &len);
    if (!bytes) return nullptr;
    auto* d = new giflib_decoder_struct;
    d->rd.p = bytes;
    d->rd.n = len;
    if (!d->rd.open() || d->rd.sw <= 0 || d->rd.sh <= 0) {
        delete d;
        return nullptr;
    }
    return d;
}

int giflib_decoder_get_width(const giflib_decoder d) { return d->rd.sw; }
int giflib_decoder_get_height(const giflib_decoder d) { return d->rd.sh; }
int giflib_decoder_get_num_frames(const giflib_decoder d) { return d->image_count; }
int giflib_decoder_get_frame_width(const giflib_decoder d) { return d->image.width; }
int giflib_decoder_get_frame_height(const giflib_decoder d) { return d->image.height; }
int giflib_decoder_get_prev_frame_delay(const giflib_decoder d) { return d->prev_delay; }

int giflib_decoder_get_prev_frame_disposal(const giflib_decoder d) {  // ref giflib.cpp:187-199
    switch (d->prev_disposal) {
        case 2: return GIF_DISPOSE_BACKGROUND;
        case 3: return GIF_DISPOSE_PREVIOUS;
        default: return GIF_DISPOSE_NONE;
    }
}

void giflib_decoder_release(giflib_decoder d) {
    if (!d) return;
    cudaStream_t st = thread_stream();
    if (d->d_canvas) cudaFreeAsync(d->d_canvas, st);
    if (d->d_prev) cudaFreeAsync(d->d_prev, st);
    if (d->d_scratch) cudaFreeAsync(d->d_scratch, st);
    delete d;
}

// ref giflib.cpp:289-326
static giflib_decoder_frame_state seek_next_frame(giflib_decoder d) {
    if (d->seek_clear_extensions) {
        d->pending_gcbs.clear();
        d->ext.clear();
        d->seek_clear_extensions = false;
    }
    for (;;) {
        const int rec = d->rd.record();
        if (rec < 0) return giflib_decoder_error;
        if (rec == 0) return giflib_decoder_have_next_frame;
        if (rec == 1) {
            if (!read_extension(d->rd, &d->ext, &d->pending_gcbs)) return giflib_decoder_error;
        } else {
            return giflib_decoder_eof;
        }
    }
}

giflib_decoder_frame_state giflib_decoder_decode_frame_header(giflib_decoder d) {  // ref giflib.cpp:331-347
    const giflib_decoder_frame_state s = seek_next_frame(d);
    if (s != giflib_decoder_have_next_frame) return s;
    if (!d->rd.image_header(&d->image)) return giflib_decoder_error;
    return giflib_decoder_have_next_frame;
}

giflib_decoder_frame_state giflib_decoder_skip_frame(giflib_decoder d) {  // ref giflib.cpp:570-590
    const giflib_decoder_frame_state s = giflib_decoder_decode_frame_header(d);
    if (s != giflib_decoder_have_next_frame) return s;
    const uint8_t* data;
    int len;
    do {
        if (!d->rd.sub_block(&data, &len)) return giflib_decoder_error;
    } while (len != 0);
    return giflib_decoder_have_next_frame;
}

bool giflib_decoder_decode_frame(giflib_decoder d, opencv_mat mat) {  // ref giflib.cpp:640-724 + 349-568
    const GifImage& im = d->image;
    if (im.width <= 0 || im.height <= 0) return false;
    if (ensure_device()) return false;
    cudaStream_t st = thread_stream();
    // scratch: frame job, animation job, colour table and code stream (one upload), then the indices.  The host
    // gathers the code stream: one frame is too little work to hide the deblock kernel's serial walk.
    const size_t anim_pos = round_up(sizeof(GifFrameJob), (size_t)16);
    const size_t colors_pos = anim_pos + round_up(sizeof(GifAnimJob), (size_t)16), lzw_pos = colors_pos + 256 * 3;
    std::vector<uint8_t> staged(lzw_pos);
    {  // gather the LZW sub-blocks (giflib reads them through DGifGetLine)
        const uint8_t* data;
        int len;
        for (;;) {
            if (!d->rd.sub_block(&data, &len)) return false;
            if (len == 0) break;
            staged.insert(staged.end(), data, data + len);
        }
    }
    GifGcb gcb;  // ref giflib.cpp:248-270: defaults, then the last graphic control block seen
    if (!d->pending_gcbs.empty()) gcb = d->pending_gcbs.back();
    if (!d->have_read_first_frame) background_color(d->rd, gcb, &d->bg_r, &d->bg_g, &d->bg_b, &d->bg_a);
    const uint8_t* colors = im.colors ? im.colors : d->rd.gct;
    const int ncolors = im.colors ? im.ncolors : d->rd.gct_colors;
    if (!colors) {
        fprintf(stderr, "encountered error, gif frame has no color map\n");
        return false;
    }
    // the frame mat is the full canvas, BGRA
    uint8_t* frame_dev = nullptr;
    size_t frame_step = 0;
    const int cw = d->rd.sw, chh = d->rd.sh;
    if (mat_bind_device_frame(mat, cw, chh, CV_8UC4, &frame_dev, &frame_step)) return false;
    const size_t canvas_bytes = (size_t)cw * chh * 4;
    if (!d->d_canvas) {
        if (cudaMallocAsync(&d->d_canvas, canvas_bytes, st) != cudaSuccess) return false;
        if (cudaMallocAsync(&d->d_prev, canvas_bytes, st) != cudaSuccess) return false;
        cudaMemsetAsync(d->d_prev, 0, canvas_bytes, st);  // the reference's prev_frame_bgra starts zeroed
        cudaMemsetAsync(d->d_canvas, 0, canvas_bytes, st);
    }
    GifFramePlan f;
    f.colors_pos = colors_pos;
    f.lzw_len = (uint32_t)(staged.size() - lzw_pos);
    f.left = im.left; f.top = im.top; f.width = im.width; f.height = im.height;
    f.interlace = im.interlace ? 1 : 0;
    f.ncolors = ncolors;
    f.min_code = im.min_code;
    f.transparent = gcb.transparent;
    GifFrameJob job = gif_frame_job(f, 0, d->prev_disposal, d->prev_left, d->prev_top, d->prev_width, d->prev_height,
                                    cw, chh);
    job.lzw_off = lzw_pos;
    job.canvas = 0;  // (d_canvas: the one canvas the decoder keeps)
    job.idx_off = lzw_pos + round_up((size_t)f.lzw_len + 32, (size_t)16);  // the word reader may look past the end
    const size_t need = job.idx_off + round_up((size_t)job.npix + 64, (size_t)16);
    if (need > d->scratch_cap) {
        if (d->d_scratch) cudaFreeAsync(d->d_scratch, st);
        d->d_scratch = nullptr;
        d->scratch_cap = 0;
        if (cudaMallocAsync(&d->d_scratch, 2 * need, st) != cudaSuccess) return false;
        d->scratch_cap = 2 * need;
    }
    const GifAnimJob anim{0, 1, make_uchar4(d->bg_b, d->bg_g, d->bg_r, d->bg_a), d->have_read_first_frame ? 0 : 1,
                          d->d_prev};
    memcpy(staged.data(), &job, sizeof(job));
    memcpy(staged.data() + anim_pos, &anim, sizeof(anim));
    memcpy(staged.data() + colors_pos, colors, (size_t)ncolors * 3);
    cudaMemcpyAsync(d->d_scratch, staged.data(), staged.size(), cudaMemcpyHostToDevice, st);
    GifFrameJob* d_job = reinterpret_cast<GifFrameJob*>(d->d_scratch);
    gif_decode_launch(d_job, 1, reinterpret_cast<const GifAnimJob*>(d->d_scratch + anim_pos), 1, d->d_scratch, cw, chh,
                      d->d_canvas, canvas_bytes, st);
    int status = 0;
    cudaMemcpyAsync(&status, &d_job->status, sizeof(int), cudaMemcpyDeviceToHost, st);
    cudaMemcpy2DAsync(frame_dev, frame_step, d->d_canvas, (size_t)cw * 4, (size_t)cw * 4, chh,
                      cudaMemcpyDeviceToDevice, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) return false;  // `staged` stays alive until here
    if (status != 0) {
        fprintf(stderr, "encountered error, could not rasterize gif\n");
        return false;
    }
    mat_mark_device_written(mat);
    force_partial_transparent(d->ext, gcb, im, ncolors, cw, chh);
    d->prev_disposal = gcb.disposal;
    d->prev_delay = gcb.delay;
    d->prev_left = im.left;
    d->prev_top = im.top;
    d->prev_width = im.width;
    d->prev_height = im.height;
    d->have_read_first_frame = true;
    d->seek_clear_extensions = true;
    return true;
}

// ref giflib.cpp:1308-1431: a second walk over the container
static GifAnimationInfo animation_info(const uint8_t* data, size_t len) {
    GifAnimationInfo info = {1, 0, 255, 255, 255, 0, 0};
    GifReader r;
    r.p = data;
    r.n = len;
    if (!r.open()) return info;
    bool found_loop = false, found_gcb = false;
    GifGcb first_gcb;
    for (;;) {
        const int rec = r.record();
        if (rec < 0) break;  // DGifGetRecordType != GIF_OK ends the walk
        if (rec == 2) return info;  // terminator: straight to cleanup (no background fix-up)
        if (rec == 1) {
            uint8_t label;
            if (!r.get(&label)) break;
            const uint8_t* data;
            int len;
            if (!r.sub_block(&data, &len)) break;
            if (len == 0) continue;
            if (label == 0xF9) {
                GifGcb g;
                gcb_from_block(data, len, &g);
                info.duration_ms += (info.frame_count > 0 && g.delay < 2) ? 20 : g.delay * 10;
                if (!found_gcb) {
                    found_gcb = true;
                    first_gcb = g;
                    uint8_t R, G, B, A;
                    background_color(r, g, &R, &G, &B, &A);
                    info.bg_red = R; info.bg_green = G; info.bg_blue = B; info.bg_alpha = A;
                }
            } else if (!found_loop && label == 0xFF && len >= 11 && !memcmp(data, "NETSCAPE2.0", 11)) {
                if (r.sub_block(&data, &len) && len != 0) {
                    if (len >= 3 && data[0] == 1) {
                        info.loop_count = data[1] | (data[2] << 8);
                        found_loop = true;
                    }
                } else {
                    if (len == 0) continue;
                    return info;
                }
            }
            bool ok = true;
            while (len != 0) {
                if (!r.sub_block(&data, &len)) { ok = false; break; }
            }
            if (!ok) return info;
        } else {  // image descriptor
            info.frame_count++;
            GifImage im;
            if (!r.image_header(&im)) return info;
            const uint8_t* data;
            int len;
            bool ok = true;
            do {
                if (!r.sub_block(&data, &len)) { ok = false; break; }
            } while (len != 0);
            if (!ok) return info;
        }
    }
    if (!found_gcb) {
        // the reference's stand-in here is a zero-initialised GraphicsControlBlock (giflib.cpp:1331), whose
        // TransparentColor 0 is not NO_TRANSPARENT_COLOR: the colour comes out with alpha 0
        first_gcb.transparent = 0;
        uint8_t R, G, B, A;
        background_color(r, first_gcb, &R, &G, &B, &A);
        info.bg_red = R; info.bg_green = G; info.bg_blue = B; info.bg_alpha = A;
    }
    return info;
}

struct GifAnimationInfo giflib_decoder_get_animation_info(const giflib_decoder d) { return animation_info(d->rd.p, d->rd.n); }

// ------------------------------------------------------------------ encoder (ref giflib.cpp:726-1306)

giflib_encoder giflib_encoder_create(void* buf, size_t buf_len) {  // ref giflib.cpp:773-800
    auto* e = new giflib_encoder_struct;
    e->dst = static_cast<uint8_t*>(buf);
    e->dst_len = buf_len;
    e->open = true;
    return e;
}

// ref giflib.cpp:803-860 + EGifPutScreenDesc: "GIF89a", logical screen descriptor, global colour table
bool giflib_encoder_init(giflib_encoder e, const giflib_decoder d, int width, int height) {
    if (!e || !d || !e->open) return false;
    e->sw = width;
    e->sh = height;
    const GifReader& r = d->rd;
    e->has_gct = r.gct != nullptr;
    if (e->has_gct) e->gct.assign(r.gct, r.gct + (size_t)r.gct_colors * 3);
    return write_screen(*e, r, width, height);
}

bool giflib_encoder_encode_frame(giflib_encoder e, const giflib_decoder d, const opencv_mat opaque_frame) {
    if (!e || !d || !e->open || !opaque_frame) return false;
    // ---- giflib_encoder_setup_frame (ref giflib.cpp:862-920)
    const GifImage& im_in = d->image;
    const bool has_local = im_in.colors != nullptr;
    std::vector<GifExt> ext = d->ext;  // this frame's extension blocks: delay, transparent index, comments ...
    const GifGcb gcb = encoder_frame_gcb(ext, d->rd, has_local, d->bg_a == 255);
    // ---- giflib_encoder_render_frame (ref giflib.cpp:934-1098)
    int cols = 0, rows = 0, type = 0;
    const uint8_t* frame_dev = nullptr;
    size_t frame_step = 0;
    if (mat_device_view(opaque_frame, &cols, &rows, &type, &frame_dev, &frame_step)) return false;
    if (type != CV_8UC4) {
        fprintf(stderr, "[lilliput_b200] GIF encoder needs a BGRA frame\n");
        return false;
    }
    if (cols > e->sw) {
        fprintf(stderr, "encountered error, gif frame wider than gif global width\n");
        return false;
    }
    if (rows > e->sh) {
        fprintf(stderr, "encountered error, gif frame taller than gif global height\n");
        return false;
    }
    const uint8_t* colors = has_local ? im_in.colors : (e->has_gct ? e->gct.data() : nullptr);
    const int ncolors = has_local ? im_in.ncolors : (e->has_gct ? (int)e->gct.size() / 3 : 0);
    if (!colors) {
        fprintf(stderr, "encountered error, gif frame has no color map\n");
        return false;
    }
    cudaStream_t st = thread_stream();
    const size_t npix = (size_t)cols * rows;
    const size_t canvas_bytes = (size_t)e->sw * e->sh * 4;
    const size_t run_pos = round_up(sizeof(GifEncJob), (size_t)16), pal_pos = run_pos + round_up(sizeof(GifEncRun), (size_t)16);
    const size_t len_pos = pal_pos + 768, job_bytes = len_pos + sizeof(uint32_t);
    if (!e->d_prev) {
        if (cudaMallocAsync(&e->d_prev, canvas_bytes, st) != cudaSuccess) return false;
        if (cudaMallocAsync(&e->d_table, kGifRunTableBytes, st) != cudaSuccess) return false;
        if (cudaMallocAsync(&e->d_job, job_bytes, st) != cudaSuccess) return false;
        cudaMemsetAsync(e->d_prev, 0, canvas_bytes, st);
    }
    if (npix > e->pixels_cap) {
        if (e->d_pixels) cudaFreeAsync(e->d_pixels, st);
        if (e->d_out) cudaFreeAsync(e->d_out, st);
        e->pixels_cap = npix;
        e->out_cap = gif_lzw_slot(npix);
        if (cudaMallocAsync(&e->d_pixels, npix + 64, st) != cudaSuccess) return false;
        if (cudaMallocAsync(&e->d_out, e->out_cap, st) != cudaSuccess) return false;
    }
    // the memo carries over when the palette is byte-equal to the previous frame's; the owners never do
    int16_t* d_lookup = reinterpret_cast<int16_t*>(e->d_table);
    unsigned long long* d_owner = reinterpret_cast<unsigned long long*>(e->d_table + 32768 * sizeof(int16_t));
    bool clear_lookup = true;
    if (e->have_written_first_frame && e->have_prev_colors && e->prev_colors.size() == (size_t)ncolors * 3)
        clear_lookup = memcmp(e->prev_colors.data(), colors, (size_t)ncolors * 3) != 0;
    if (clear_lookup) cudaMemsetAsync(d_lookup, 0xFF, 32768 * sizeof(int16_t), st);
    cudaMemsetAsync(d_owner, 0xFF, 32768 * sizeof(unsigned long long), st);
    std::vector<uint8_t> staged(len_pos, 0);
    GifEncJob j{};
    j.frame = frame_dev;
    j.step = frame_step;
    j.prev = e->d_prev;
    j.prev_step = (size_t)e->sw * 4;
    j.palette = e->d_job + pal_pos;
    j.pixels = e->d_pixels;
    j.out = e->d_out;
    j.out_len = reinterpret_cast<uint32_t*>(e->d_job + len_pos);
    j.width = cols;
    j.height = rows;
    j.ncolors = ncolors;
    j.transparent = gcb.transparent;
    j.prev_valid = e->have_written_first_frame && (e->prev_frame_disposal == 0 || e->prev_frame_disposal == 1);
    j.run = 0;
    j.pos = 0;
    j.code_bits = std::max(2, color_bits(ncolors));
    j.interlace = im_in.interlace ? 1 : 0;
    j.out_cap = (uint32_t)e->out_cap;
    const GifEncRun run{d_lookup, d_owner, reinterpret_cast<int*>(e->d_table + 32768 * (sizeof(int16_t) + sizeof(unsigned long long))),
                        0, 0};
    memcpy(staged.data(), &j, sizeof(j));
    memcpy(staged.data() + run_pos, &run, sizeof(run));
    memcpy(staged.data() + pal_pos, colors, (size_t)std::min(ncolors, 256) * 3);
    cudaMemcpyAsync(e->d_job, staged.data(), staged.size(), cudaMemcpyHostToDevice, st);
    gif_encode_launch(reinterpret_cast<const GifEncJob*>(e->d_job), 1, reinterpret_cast<const GifEncRun*>(e->d_job + run_pos), 1,
                      cols, rows, st);
    // prev_frame_bgra = this frame (ref giflib.cpp:1091: the whole canvas)
    cudaMemcpy2DAsync(e->d_prev, (size_t)e->sw * 4, frame_dev, frame_step, (size_t)cols * 4, rows,
                      cudaMemcpyDeviceToDevice, st);
    e->prev_colors.assign(colors, colors + (size_t)ncolors * 3);
    e->have_prev_colors = true;
    e->prev_frame_disposal = gcb.disposal;
    // ---- giflib_encoder_encode_frame (ref giflib.cpp:1126-1183): extensions, image descriptor, LZW
    uint32_t out_len = 0;
    cudaMemcpyAsync(&out_len, j.out_len, sizeof(out_len), cudaMemcpyDeviceToHost, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) return false;  // `staged` stays alive until here
    if (out_len == 0xFFFFFFFFu) return false;
    if (!write_frame_head(*e, ext, cols, rows, im_in.interlace, has_local ? im_in.colors : nullptr, im_in.ncolors, j.code_bits))
        return false;
    if (e->dst_offset + out_len > e->dst_len) return false;
    if (cudaMemcpy(e->dst + e->dst_offset, e->d_out, out_len, cudaMemcpyDeviceToHost) != cudaSuccess) return false;
    e->dst_offset += out_len;
    e->have_written_first_frame = true;
    return true;
}

// ref giflib.cpp:1185-1222: trailing extension blocks, then the GIF trailer
bool giflib_encoder_flush(giflib_encoder e, const giflib_decoder d) {
    if (!e || !d || !e->open) return false;
    if (!write_extensions(*e, d->ext)) return false;
    if (!e->put8(0x3B)) return false;
    e->open = false;
    return true;
}

void giflib_encoder_release(giflib_encoder e) {
    if (!e) return;
    cudaStream_t st = thread_stream();
    if (e->d_prev) cudaFreeAsync(e->d_prev, st);
    if (e->d_table) cudaFreeAsync(e->d_table, st);
    if (e->d_job) cudaFreeAsync(e->d_job, st);
    if (e->d_pixels) cudaFreeAsync(e->d_pixels, st);
    if (e->d_out) cudaFreeAsync(e->d_out, st);
    delete e;
}

int giflib_encoder_get_output_length(giflib_encoder e) { return (int)e->dst_offset; }

}  // extern "C"

namespace lp {
int gif_header_frames(const uint8_t* data, size_t len) { return animation_info(data, len).frame_count; }
}  // namespace lp
