// xbatch.cu -- the heterogeneous batch entry point (include/lilliput_b200.h: lp_xbatch_*): N independent
// images of ANY supported format and size through ImageOps.Transform with one set of options, the
// per-image work packed into grid launches.
//
// Per-item semantics are those of lp_transform (= lilliput's NewDecoder + ImageOps.Transform,
// ref lilliput.go:129-164, ops.go:352-444).  What differs is the schedule:
//   1. headers of all items are parsed on the host by a few threads (format sniff as lilliput.go:129-164);
//   2. items are grouped by (decoder kind, source geometry) -- a group shares its Fit crop / output size
//      (ref ops.go:243-255, opencv.go:331-363), so every stage of a group is ONE launch over all its images:
//        JPEG  -> the lp_batch pipeline (batch.cu): parallel Huffman, IDCT, colour, resize, encode; multi-scan
//                 (progressive) files form groups of their own, so a chunk of baseline files never waits for the
//                 serial decode of a large progressive one.  To WebP or PNG the pipeline stops after the resize and the
//                 group's frames go to that sink's encoder
//        PNG   -> IDAT gather + warp-parallel inflate + defilter + convert (png_decode.cu; 16-bit samples keep their high
//                 byte), resize.  A PQ or HLG cICP chunk: the window's HDR frames go through one batched tone map to SDR
//                 BT.709 (tonemap.cu) between the defilter and the resize, whole, as Transform tone-maps right after the
//                 decode; no cICP is written.  An SDR cICP changes no pixel (to PNG it stays per image, below)
//        WebP  -> stills and animations: VP8 frames one per warp, VP8L / ALPH streams one per warp in arena-sized waves,
//                 a per-pixel compositor over every file's frame sequence (webp_decode.cu), resize of every canvas
//        GIF   -> every frame of every animation: LZW (one warp per frame), per-pixel compositor over the
//                 frame sequence (gif_decode.cu), resize of every composited canvas
//        DisableAnimatedOutput (GIF and animated WebP to WebP, GIF to GIF): Transform stops after frame 0, so the plan
//                 stops there too (gif_plan_parse's first-frame walk, webp_plan_first_frame); only the file up to the
//                 end of frame 0's image data is uploaded, the same kernels run over one frame per file, and the sink
//                 writes a still WebP or a one-frame GIF
//      and the sinks: JPEG (jpeg_encode.cu), lossy WebP still / animation (webp_encode.cu) carrying the ICC profile of
//      a JPEG, PNG or WebP source as WebpEncoder does, lossless WebP still / animation from PNG and GIF sources (the
//      batched VP8L encoder over every frame of a run, webp_encode.cu; a PNG's ICC profile carried the same way), GIF
//      from GIF sources (palette mapping + LZW of every frame of the task, gif_decode.cu; the container assembled on the
//      host), PNG from JPEG, PNG and WebP stills (filter, DEFLATE, checksums and container of every frame of a run in
//      three launches, png_encode.cu);
//   3. anything the grid path does not cover (gray or over-budget multi-scan JPEGs, gray PNGs, EXIF-rotated sources,
//      SDR-cICP PNGs to PNG (Transform re-attaches the chunk), lossless WebP output of JPEG and WebP sources, PNG
//      output of animations, GIF output from other formats, animations under MaxEncodeFrames or MaxEncodeDuration,
//      one-frame GIFs to WebP with no time to encode ...) and any item whose grid stage fails goes through lp_transform
//      on a worker thread -- still this library's device kernels, one image per call -- so the status and bytes of
//      EVERY item are what lp_transform would have returned.
// Two worker lanes, each with half of the device arena and its own stream, process chunks of groups
// concurrently, so one lane's PCIe copies and host-side container work overlap the other lane's kernels.
// Nothing is exchanged between images, lanes or GPUs.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"
#include "lilliput_host.hpp"
#include "lp_opencv.h"

using namespace lp;

namespace lp {
lp_batch* batch_create_in(const lp_batch_config* cfg, uint8_t* dev_arena, size_t dev_bytes, uint8_t* host_arena,
                          size_t host_bytes, bool progressive_jpeg, bool multiscan_sources, bool resize_only,
                          bool oriented_sources = false,  // (rotated and gray JPEGs are handed to lp_transform before
                          bool gray_sources = false);     // grouping, so these contexts take neither)
int batch_resized_status(lp_batch* b, int* status);
size_t batch_multiscan_pool_bytes(size_t n);
void batch_arena_used(const lp_batch* b, size_t* dev_bytes, size_t* host_bytes);
}  // namespace lp

namespace {

enum Kind { K_FALLBACK = 0, K_JPEG = 1, K_PNG = 2, K_WEBP = 3, K_GIF = 4 };
enum Sink { S_NONE = 0, S_JPEG = 1, S_WEBP = 2, S_GIF = 3, S_PNG = 4 };

struct XItem {
    Kind kind = K_FALLBACK;
    int w = 0, h = 0, ch = 0;       // decoded frame
    int ow = 0, oh = 0;             // output size
    int cx = 0, cy = 0, cw = 0, chh = 0;  // crop rectangle fed to the resize
    int jpeg_sampling = 0;          // (h0<<12)|(v0<<8)|... groups JPEGs of one component layout
    bool jpeg_multiscan = false;    // progressive, or one scan per component
    std::unique_ptr<PngHeader> png;
    bool hdr = false;                 // PNG: a cICP chunk with a PQ (16) or HLG (18) transfer, tone-mapped after the decode
    int transfer = 0, primaries = 0;  // (its code points)
    std::unique_ptr<WebpPlan> webp;  // (for WebP: the frames' spans, rectangles and blend / dispose)
    GifAnimPlan* gif = nullptr;
    int gif_frames = 0;
    size_t span = 0;           // WebP, GIF: bytes at the start of the file the device reads (first-frame items: through frame 0)
    std::vector<uint8_t> icc;  // WebP sink: the source's profile the WebP writer carries (empty: none, or not sane)
};

struct Task {
    Kind kind;
    std::vector<int> idx;  // items (for GIF: animations)
};

struct Lane {
    int id = 0;
    cudaStream_t st = nullptr;
    uint8_t* dev = nullptr;
    size_t dev_bytes = 0;
    uint8_t* host = nullptr;  // pinned
    size_t host_bytes = 0;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    double ms_decode = 0, ms_resize = 0, ms_encode = 0;
    size_t h2d = 0, d2h = 0;
    long launches = 0;
};

struct Bump {
    uint8_t* base;
    size_t cap, used = 0;
    template <class T>
    T* take(size_t bytes) {
        const size_t need = round_up(bytes, (size_t)256);
        if (used + need > cap) return nullptr;
        T* p = reinterpret_cast<T*>(base + used);
        used += need;
        return p;
    }
};

}  // namespace

struct lp_xbatch {
    lp_xbatch_config cfg;
    int device = 0;
    int threads = 4;
    Lane lanes[2];
    uint8_t* arena = nullptr;
    size_t arena_bytes = 0;
    uint8_t* host_arena = nullptr;
    size_t host_bytes = 0;
    lp_xbatch_stats stats;
    // per call
    const uint8_t* const* in = nullptr;
    const size_t* in_len = nullptr;
    uint8_t* const* out = nullptr;
    size_t out_cap = 0;
    size_t* out_len = nullptr;
    int* status = nullptr;
    lp_image_options opt;
    Sink sink = S_NONE;
    int quality = 0;
    bool lossless = false;     // S_WEBP: lossless (VP8L) frames, WebpQuality above 100
    bool progressive = false;  // S_JPEG: progressive files (JpegProgressive)
    int png_level = 1;         // S_PNG: zlib level and filter policy (png_encode_policy)
    bool png_adaptive = false;
    std::vector<XItem> items;
    std::vector<int> fallback;
    std::mutex fb_mu;
};

static void push_fallback(lp_xbatch* X, int i) {
    std::lock_guard<std::mutex> g(X->fb_mu);
    X->fallback.push_back(i);
}

// ------------------------------------------------------------------ parse

static int option_value(const lp_image_options& o, int key, int dflt) {
    int v = dflt;
    for (size_t i = 0; i + 1 < o.encode_options_len; i += 2)
        if (o.encode_options[i] == key) v = o.encode_options[i + 1];
    return v;
}

// Output size and crop of a still of w x h (ref ops.go:449-470, 243-255; opencv.go:331-363).  false: not a
// resize the grid path does (NoResize).
static bool plan_geometry(const lp_image_options& o, XItem* it) {
    if (o.resize_method == LP_OPS_FIT) {
        lilliput::calculateExpectedSize(it->w, it->h, o.width, o.height, &it->ow, &it->oh);
        if (it->ow < 1 || it->oh < 1) return false;
        lilliput::fitCropRect(it->w, it->h, it->ow, it->oh, &it->cx, &it->cy, &it->cw, &it->chh);
        return true;
    }
    if (o.resize_method == LP_OPS_RESIZE) {
        it->ow = o.width;
        it->oh = o.height;
        if (it->ow < 1 || it->oh < 1) return false;
        it->cx = it->cy = 0;
        it->cw = it->w;
        it->chh = it->h;
        return true;
    }
    return false;
}

// The profile WebpEncoder::Create hands to the WebP writer: what the decoder's ICC() read into its 32 KiB buffer
// (ICCProfileBufferSize, ref lilliput.go:15; n <= 0: none), kept only when iccHeaderIsSane
static void keep_icc(XItem* it, const uint8_t* icc, long n) {
    if (n > 0 && lilliput::iccHeaderIsSane(icc, (size_t)n)) it->icc.assign(icc, icc + n);
}

static void parse_item(lp_xbatch* X, int i) {
    XItem& it = X->items[i];
    const uint8_t* d = X->in[i];
    const size_t n = X->in_len[i];
    it.kind = K_FALLBACK;
    it.icc.clear();
    it.span = n;
    if (!d || n < 16 || X->sink == S_NONE) return;
    // To PNG every still is one frame in, the file out of the first Encode call: MaxEncodeFrames, DisableAnimatedOutput
    // and the deadline are never consulted.  A negative MaxEncodeDuration is exceeded before the frame is encoded, and
    // Transform then asks the decoder to skip to the end, which no still decoder can (ErrSkipNotSupported): per image.
    if (X->sink == S_PNG && X->opt.max_encode_duration_ns < 0) return;
    const int max_side = X->cfg.max_size > 0 ? X->cfg.max_size : 8192;
    static const uint8_t png_sig[8] = {0x89, 0x50, 0x4E, 0x47, 0x0D, 0x0A, 0x1A, 0x0A};
    thread_local std::vector<uint8_t> icc_buf(32768);
    if (d[0] == 0xFF && d[1] == 0xD8) {
        if (X->sink != S_JPEG && X->sink != S_WEBP && X->sink != S_PNG) return;
        if (X->lossless) return;  // lossless WebP output of JPEG sources: per image
        // A still to WebP: after its frame Transform checks its deadline (a zero budget fails with ErrEncodeTimeout),
        // MaxEncodeFrames == 1 asks the decoder to skip to the end (a JPEG cannot: ErrSkipNotSupported), and a negative
        // MaxEncodeDuration is exceeded at once (the same skip).  Those go per image.
        if (X->sink == S_WEBP && (X->opt.encode_timeout_ns <= 0 || X->opt.max_encode_frames == 1 || X->opt.max_encode_duration_ns < 0))
            return;
        JpegHeader h;
        if (jpeg_parse_header(d, n, &h) != LP_OK || (!h.supported && !h.multiscan)) return;
        if (h.ncomp != 3) return;
        if (h.orientation >= 2 && h.orientation <= 8) return;
        if (h.width > max_side || h.height > max_side) return;
        if (!h.supported) {  // multi-scan: damaged scans and files over the serial decoder's budget go per image
            std::vector<JpegScanDesc> scans(kMultiscanMaxScans);
            int nscans = 0, nsets = 0;
            if (jpeg_parse_scans(d, n, h, scans.data(), (int)scans.size(), &nscans, (JpegHeader*)nullptr, kMultiscanMaxSets,
                                 &nsets) != LP_OK ||
                jpeg_multiscan_visits(h, scans.data(), nscans) > kMultiscanMaxVisits)
                return;
            it.jpeg_multiscan = true;
        }
        it.w = h.width;
        it.h = h.height;
        it.ch = 3;
        it.jpeg_sampling = 0;
        for (int c = 0; c < 3; c++) it.jpeg_sampling = (it.jpeg_sampling << 8) | (h.comp[c].h << 4) | h.comp[c].v;
        if (!plan_geometry(X->opt, &it)) return;
        if (X->sink == S_WEBP)  // (its APP2 segments concatenated: the item keeps its own copy)
            keep_icc(&it, icc_buf.data(), opencv_decoder_get_jpeg_icc(const_cast<uint8_t*>(d), n, icc_buf.data(), icc_buf.size()));
        it.kind = K_JPEG;
        return;
    }
    if (!memcmp(d, png_sig, 8)) {
        if (X->sink == S_GIF) return;  // GIF output needs a GIF source: per image (ErrGifEncoderNeedsDecoder)
        std::unique_ptr<PngHeader> h(new PngHeader);
        if (png_parse(d, n, h.get()) != LP_OK) return;
        // an eXIf orientation other than 1: Transform turns the frame before the resize, which the grid does not: per image
        if (h->orientation != 1 || h->idat.empty() || h->idat_total < 2) return;
        if (h->width > max_side || h->height > max_side) return;
        uint8_t cicp[4];  // primaries, transfer, matrix, full range: the chunk Transform's decoder reports
        if (png_extract_cicp(d, n, cicp)) {
            it.hdr = cicp[1] == 16 || cicp[1] == 18;
            // an SDR tag changes no pixel, but Transform re-attaches it to a PNG output (ops.go:306-332): per image
            if (!it.hdr && X->sink == S_PNG) return;
            it.transfer = cicp[1];
            it.primaries = cicp[0];
        }
        // the IDAT payloads must form one forward run of the file (they do in every valid PNG)
        for (size_t k = 1; k < h->idat.size(); k++)
            if (h->idat[k].offset < h->idat[k - 1].offset + h->idat[k - 1].length) return;
        if (h->idat.back().offset + h->idat.back().length > n) return;
        it.w = h->width;
        it.h = h->height;
        it.ch = h->out_channels;
        if (it.ch != 3 && it.ch != 4) return;  // gray PNGs: per image
        if (!plan_geometry(X->opt, &it)) return;
        if (X->sink == S_WEBP) {
            const int icc_n = png_extract_icc(d, n, icc_buf.data(), icc_buf.size());
            // PNGs with a profile stay per image, where they went before they could carry it, under the options whose
            // result the per-image path decides after the frame: a zero encode budget (the deadline check, as for WebP
            // stills), MaxEncodeFrames == 1 and a negative MaxEncodeDuration (the skip to the end a PNG decoder
            // refuses, as a JPEG's does).  To lossless output every PNG follows that rule.
            if ((icc_n > 0 || X->lossless) &&
                (X->opt.encode_timeout_ns <= 0 || X->opt.max_encode_frames == 1 || X->opt.max_encode_duration_ns < 0))
                return;
            keep_icc(&it, icc_buf.data(), icc_n);
        }
        it.png = std::move(h);
        it.kind = K_PNG;
        return;
    }
    if (!memcmp(d, "RIFF", 4) && !memcmp(d + 8, "WEBP", 4)) {
        if (X->sink == S_GIF || X->lossless) return;  // (lossless WebP output of WebP sources: per image)
        std::unique_ptr<WebpPlan> p(new WebpPlan);
        if (!webp_plan_parse(d, n, p.get())) return;  // damaged containers: per image
        if (p->width > max_side || p->height > max_side) return;
        WebpFramePlan& f0 = p->frames[0];
        if (p->frames.size() == 1) {
            // Transform does not composite a still: it resizes the decoded frame, which must then be the canvas
            if (f0.x || f0.y || f0.width != p->width || f0.height != p->height) return;
            // a still written to WebP with no time to encode: lp_transform's deadline check follows the frame.  Only the
            // simple lossy stills the grid has always taken keep going there; the others stay with lp_transform
            const bool simple = !f0.lossless && !f0.has_alph && !p->icc_len && !p->animated && p->channels == 3;
            if (X->sink == S_WEBP && X->opt.encode_timeout_ns <= 0 && !simple) return;
            // to PNG under MaxEncodeDuration: a WebP still's frame carries a duration, which Transform holds against the
            // limit before it encodes the frame; lp_transform decides
            if (X->sink == S_PNG && X->opt.max_encode_duration_ns != 0) return;
            f0.blend = 1;  // copied onto a canvas of its own size, never disposed
            f0.dispose = 0;
        } else {
            // animations -> animated WebP, with the option gates of GIF -> WebP; Transform checks its deadline after
            // every non-final frame, so a zero budget fails there (ErrEncodeTimeout): per image.  DisableAnimatedOutput:
            // Transform encodes frame 0 and flushes before its deadline check, so whatever the budget, the file is a
            // still of the composited frame 0 and the device reads only that frame
            if (X->sink != S_WEBP || X->opt.max_encode_frames != 0 || X->opt.max_encode_duration_ns != 0) return;
            if (X->opt.disable_animated_output) it.span = webp_plan_first_frame(p.get());
            else if (X->opt.encode_timeout_ns <= 0) return;
        }
        it.w = p->width;
        it.h = p->height;
        it.ch = p->channels;
        if (!plan_geometry(X->opt, &it)) return;
        // (webp_decoder_get_icc reads no profile larger than the 32 KiB buffer)
        if (X->sink == S_WEBP && p->icc_len <= icc_buf.size()) keep_icc(&it, d + p->icc_off, (long)p->icc_len);
        it.webp = std::move(p);
        it.kind = K_WEBP;
        return;
    }
    if (!memcmp(d, "GIF8", 4)) {
        if ((X->sink != S_WEBP && X->sink != S_GIF) || X->opt.max_encode_frames != 0 || X->opt.max_encode_duration_ns != 0)
            return;
        // DisableAnimatedOutput: Transform encodes frame 0 and flushes before its deadline check, and its decoder reads
        // nothing behind that frame.  Otherwise a GIF written with no time to encode fails with ErrEncodeTimeout after
        // its first frame (Transform's deadline): per image, to GIF and to lossless WebP
        const bool first_only = X->opt.disable_animated_output != 0;
        if (!first_only && (X->sink == S_GIF || X->lossless) && X->opt.encode_timeout_ns <= 0) return;
        GifAnimPlan* p = gif_plan_parse(d, n, 4096, first_only);
        if (!p) return;
        int w = 0, h = 0, nf = 0;
        gif_plan_info(p, &w, &h, &nf, nullptr, nullptr);
        it.w = w;
        it.h = h;
        it.ch = 4;
        it.span = gif_plan_file_bytes(p);
        // a one-frame file to WebP meets the same deadline check after its frame: with no time to encode, per image
        if ((nf < 2 && X->sink == S_WEBP && !first_only && X->opt.encode_timeout_ns <= 0) || w > max_side || h > max_side ||
            !plan_geometry(X->opt, &it)) {
            gif_plan_free(p);
            return;
        }
        it.gif = p;
        it.gif_frames = nf;
        it.kind = K_GIF;
        return;
    }
}

// ------------------------------------------------------------------ sinks

// The PNG sink's file slot for a frame of ow x oh x ch: the largest file it can become, capped by the callers' buffers
// (a longer file is lp_transform's to refuse).
static size_t png_sink_slot(const lp_xbatch* X, int ow, int oh, int ch) {
    return round_up(std::min(X->out_cap, png_encode_max_file_bytes(ow, oh, ch)), (size_t)256);
}
// Device bytes the PNG sink takes from a lane's arena per frame: encoder scratch, the slot, its place in the packed copy.
static size_t png_sink_item_bytes(const lp_xbatch* X, int ow, int oh, int ch) {
    return round_up(png_encode_batch_scratch_bytes(ow, oh, ch, 1, X->png_level), (size_t)256) + 2 * png_sink_slot(X, ow, oh, ch) + 64;
}

// n encoded files in device slots (`slot` apart, d_len[k] = 0: did not fit) -> packed back to back, one D2H of lengths
// and offsets, one D2H of the packed files into the pinned staging area
static int slots_to_host(Lane& L, uint8_t* h_stage, size_t h_stage_bytes, const uint8_t* d_out, size_t slot, const uint32_t* d_len,
                         int n, uint8_t* d_packed, unsigned long long* d_off, std::vector<unsigned long long>* off,
                         std::vector<uint32_t>* len) {
    int rc = compact_launch(d_out, slot, d_len, (uint32_t)slot, n, d_packed, d_off, L.st);
    off->assign((size_t)n + 1, 0);
    len->assign((size_t)n, 0);
    if (!rc && (cudaMemcpyAsync(off->data(), d_off, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, L.st) != cudaSuccess ||
                cudaMemcpyAsync(len->data(), d_len, (size_t)n * 4, cudaMemcpyDeviceToHost, L.st) != cudaSuccess ||
                cudaStreamSynchronize(L.st) != cudaSuccess))
        rc = LP_ERR_CUDA;
    const size_t total = rc ? 0 : (size_t)(*off)[n];
    if (!rc && total > h_stage_bytes) rc = LP_ERR_CUDA;
    if (!rc && total &&
        (cudaMemcpyAsync(h_stage, d_packed, total, cudaMemcpyDeviceToHost, L.st) != cudaSuccess ||
         cudaStreamSynchronize(L.st) != cudaSuccess))
        rc = LP_ERR_CUDA;
    if (!rc) L.d2h += total + (size_t)n * 12;
    return rc;
}

// the staged files into the callers' buffers; one that did not fit its slot or the caller's buffer: let Transform decide
static void deliver_staged(lp_xbatch* X, const uint8_t* h_stage, const int* idx, int n, const std::vector<unsigned long long>& off,
                           const std::vector<uint32_t>& len, size_t slot, std::vector<int>* failed) {
    for (int k = 0; k < n; k++) {
        const int i = idx[k];
        if (len[k] == 0 || len[k] > slot || len[k] > X->out_cap) {
            failed->push_back(i);
            continue;
        }
        memcpy(X->out[i], h_stage + off[k], len[k]);
        X->out_len[i] = len[k];
        X->status[i] = LP_OK;
    }
}

// PNG sink: every frame of the run through png_encode_batch (whole files in device slots), packed and copied home.  A
// run whose slots and scratch do not fit what is left of the arena, or whose files may not fit the staging area, is
// encoded in parts.
static void png_sink(lp_xbatch* X, Lane& L, Bump& bump, uint8_t* h_stage, size_t h_stage_bytes, const std::vector<int>& idx,
                     const uint8_t* d_frames, size_t stride, int ow, int oh, int ch, std::vector<int>* failed) {
    const int n = (int)idx.size();
    const size_t slot = png_sink_slot(X, ow, oh, ch), per = png_sink_item_bytes(X, ow, oh, ch);
    const size_t mark = bump.used, room = bump.cap - bump.used;
    const size_t fixed = 4096;  // lengths, offsets and the arena's alignment
    const int part = (int)std::min<size_t>((size_t)n, std::min(room > fixed ? (room - fixed) / (per + 16) : 0, h_stage_bytes / (slot + 16)));
    if (part < 1) {
        failed->insert(failed->end(), idx.begin(), idx.end());
        return;
    }
    std::vector<unsigned long long> off;
    std::vector<uint32_t> len;
    for (int k0 = 0; k0 < n; k0 += part) {
        const int m = std::min(part, n - k0);
        bump.used = mark;  // (the part before this one has been copied home)
        uint8_t* d_out = bump.take<uint8_t>((size_t)m * slot);
        uint32_t* d_len = bump.take<uint32_t>((size_t)m * 4);
        uint8_t* d_packed = bump.take<uint8_t>((size_t)m * slot + 16);
        auto* d_off = bump.take<unsigned long long>((size_t)(m + 1) * 8);
        void* scratch = bump.take<uint8_t>(png_encode_batch_scratch_bytes(ow, oh, ch, m, X->png_level));
        int rc = d_out && d_len && d_packed && d_off && scratch ? LP_OK : LP_ERR_BUF_TOO_SMALL;
        if (!rc)
            rc = png_encode_batch(d_frames + (size_t)k0 * stride, stride, (size_t)ow * ch, ow, oh, ch, m, X->png_level, X->png_adaptive,
                                  d_out, slot, d_len, scratch, L.st);
        if (!rc) rc = slots_to_host(L, h_stage, h_stage_bytes, d_out, slot, d_len, m, d_packed, d_off, &off, &len);
        if (rc) {
            cudaGetLastError();
            failed->insert(failed->end(), idx.begin() + k0, idx.end());
            break;
        }
        deliver_staged(X, h_stage, idx.data() + k0, m, off, len, slot, failed);
    }
    bump.used = mark;
}

// The WebP sink's encoder: n resized frames of one geometry (rows packed, `stride` apart) -> lossy VP8 or, when the
// options ask for lossless output, VP8L payloads
static int webp_encode_frames(const lp_xbatch* X, const uint8_t* d_frames, size_t stride, int ow, int oh, int ch, int n,
                              std::vector<WebpEncodedFrame>* frames, cudaStream_t st) {
    if (X->lossless) return webp_encode_lossless_batch(d_frames, stride, (size_t)ow * ch, ow, oh, ch, n, frames, st);
    return webp_encode_lossy_batch(d_frames, stride, (size_t)ow * ch, ow, oh, ch, n, X->quality, frames, st);
}

// resized frames (n x ow x oh x ch, `stride` apart) -> encoded files in the callers' buffers.  h_stage: the pinned
// staging area the JPEG and PNG sinks copy their files through.
static void sink_encode(lp_xbatch* X, Lane& L, Bump& bump, uint8_t* h_stage, size_t h_stage_bytes, const std::vector<int>& idx,
                        const uint8_t* d_frames, size_t stride, int ow, int oh, int ch, std::vector<int>* failed) {
    const int n = (int)idx.size();
    if (X->sink == S_PNG) {
        png_sink(X, L, bump, h_stage, h_stage_bytes, idx, d_frames, stride, ow, oh, ch, failed);
        return;
    }
    if (X->sink == S_JPEG) {
        const size_t slot = round_up(std::min(X->out_cap, std::max((size_t)65536, (size_t)ow * oh * ch)), (size_t)256);
        uint8_t* d_out = bump.take<uint8_t>((size_t)n * slot);
        uint32_t* d_len = bump.take<uint32_t>((size_t)n * 4);
        uint8_t* d_packed = bump.take<uint8_t>((size_t)n * slot + 16);
        auto* d_off = bump.take<unsigned long long>((size_t)(n + 1) * 8);
        void* scratch = bump.take<uint8_t>(jpeg_encode_scratch_bytes(ow, oh, ch, n, slot, X->progressive));
        if (!d_out || !d_len || !d_packed || !d_off || !scratch) {
            failed->insert(failed->end(), idx.begin(), idx.end());
            return;
        }
        const bool dbg = getenv("LP_DEBUG") != nullptr;
        const auto tq0 = std::chrono::steady_clock::now();
        JpegEncodeBatch e;
        e.frames = d_frames;
        e.frame_img_stride = stride;
        e.frame_row_stride = (size_t)ow * ch;
        e.width = ow;
        e.height = oh;
        e.channels = ch;
        e.quality = X->quality;
        e.n = n;
        e.out = d_out;
        e.out_cap = slot;
        e.out_len = d_len;
        e.scratch = scratch;
        e.progressive = X->progressive;
        int rc = jpeg_encode_launch(e, L.st, nullptr);
        std::vector<unsigned long long> off;
        std::vector<uint32_t> len;
        if (!rc) rc = slots_to_host(L, h_stage, h_stage_bytes, d_out, slot, d_len, n, d_packed, d_off, &off, &len);
        if (rc) {
            cudaGetLastError();
            failed->insert(failed->end(), idx.begin(), idx.end());
            return;
        }
        const auto tq1 = std::chrono::steady_clock::now();
        if (dbg)
            fprintf(stderr, "[lilliput_b200] jpeg sink: n=%d %dx%dx%d slot=%zu total=%zu: launches + D2H %.2f ms\n", n, ow, oh, ch, slot,
                    (size_t)off[n], std::chrono::duration<double, std::milli>(tq1 - tq0).count());
        deliver_staged(X, h_stage, idx.data(), n, off, len, slot, failed);
        return;
    }
    // WebP stills, lossy or lossless, each with its source's ICC profile
    std::vector<WebpEncodedFrame> frames;
    int rc = webp_encode_frames(X, d_frames, stride, ow, oh, ch, n, &frames, L.st);
    if (rc) {
        cudaGetLastError();
        failed->insert(failed->end(), idx.begin(), idx.end());
        return;
    }
    std::vector<uint8_t> file;
    for (int k = 0; k < n; k++) {
        const int i = idx[k];
        if (frames[k].image.empty()) {
            failed->push_back(i);
            continue;
        }
        const std::vector<uint8_t>& icc = X->items[i].icc;
        webp_assemble(&frames[k], 1, icc.data(), icc.size(), 0xFFFFFFFFu, 0, &file);
        L.d2h += frames[k].image.size() + frames[k].alph.size();
        if (file.size() > X->out_cap) {  // ref webp.cpp:546-551 -> size 0 -> ErrInvalidImage (webp.go:249-251)
            X->status[i] = LP_ERR_INVALID_IMAGE;
            X->out_len[i] = 0;
            continue;
        }
        memcpy(X->out[i], file.data(), file.size());
        X->out_len[i] = file.size();
        X->status[i] = LP_OK;
    }
}

static void lane_time(Lane& L, int from, int to, double* acc) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, L.ev[from], L.ev[to]) == cudaSuccess) *acc += ms;
}

// ------------------------------------------------------------------ PNG / WebP tasks
// A task holds items of ONE decoder kind but any geometry, ordered so that equal geometries are adjacent: the
// entropy stage (inflate / boolean decoder -- the long pole, latency-bound per stream) is one launch over the whole
// task; the geometry-bound stages (resize, encode) are one launch per run of equal geometry.

struct Run {
    int k0, k1;  // positions inside the task
};
static std::vector<Run> runs_of(const lp_xbatch* X, const std::vector<int>& idx) {
    std::vector<Run> r;
    for (int k = 0; k < (int)idx.size();) {
        const XItem& a = X->items[idx[k]];
        int e = k + 1;
        while (e < (int)idx.size()) {
            const XItem& c = X->items[idx[e]];
            if (c.w != a.w || c.h != a.h || c.ch != a.ch) break;
            e++;
        }
        r.push_back(Run{k, e});
        k = e;
    }
    return r;
}

// resize of items [k0, k1) of a task (their frames at d_frames + frame_off[k]) into the task's output area
static bool resize_range(lp_xbatch* X, Lane& L, const std::vector<int>& idx, int k0, int k1, const uint8_t* d_frames,
                         const std::vector<uint64_t>& frame_off, uint8_t* d_out, const std::vector<uint64_t>& out_off) {
    for (int k = k0; k < k1;) {
        const XItem& g = X->items[idx[k]];
        int e = k + 1;
        while (e < k1) {
            const XItem& c = X->items[idx[e]];
            if (c.w != g.w || c.h != g.h || c.ch != g.ch) break;
            e++;
        }
        const size_t fs = round_up((size_t)g.w * g.h * g.ch, (size_t)256), os = round_up((size_t)g.ow * g.oh * g.ch, (size_t)256);
        ResizeArgs a{d_frames + frame_off[k], fs, (size_t)g.w * g.ch, g.ch, g.cx, g.cy, g.cw, g.chh, d_out + out_off[k], os,
                     (size_t)g.ow * g.ch, g.ow, g.oh, e - k, 3};
        if (resize_launch(a, L.st) != LP_OK) return false;
        k = e;
    }
    return true;
}

// sinks over the runs of equal geometry of a whole task (resized frames at d_out + out_off[k])
static void encode_runs(lp_xbatch* X, Lane& L, Bump& bump, const std::vector<int>& idx, const uint8_t* d_out,
                        const std::vector<uint64_t>& out_off, const std::vector<char>& ok, std::vector<int>* failed) {
    cudaEventRecord(L.ev[2], L.st);
    for (const Run& r : runs_of(X, idx)) {
        const XItem& g = X->items[idx[r.k0]];
        std::vector<int> sub;
        bool all = true;
        for (int k = r.k0; k < r.k1; k++) {
            all = all && ok[k];
            sub.push_back(idx[k]);
        }
        if (!all) {  // rare: a corrupt stream in the run -- its items take the per-image path, which reports the precise error
            failed->insert(failed->end(), sub.begin(), sub.end());
            continue;
        }
        sink_encode(X, L, bump, L.host, L.host_bytes, sub, d_out + out_off[r.k0], round_up((size_t)g.ow * g.oh * g.ch, (size_t)256),
                    g.ow, g.oh, g.ch, failed);
    }
    cudaEventRecord(L.ev[3], L.st);
    cudaEventSynchronize(L.ev[3]);
    lane_time(L, 2, 3, &L.ms_encode);
}

// PNG task.  Inflate wants every stream in flight at once and needs only the compressed stream and the scanlines
// (~1.5 x the pixel bytes); the packed frames are needed only between defilter and resize.  So: ONE inflate launch over
// the whole task, then defilter -> resize over windows of frames that reuse one buffer, then the sinks over the task.
static void run_png(lp_xbatch* X, Lane& L, const std::vector<int>& idx) {
    const int n = (int)idx.size();
    std::vector<int> failed;
    Bump bump{L.dev, L.dev_bytes};
    std::vector<PngDecodeItem> items((size_t)n);
    std::vector<SegCopy> segs;
    std::vector<uint64_t> file_off((size_t)n), frame_off((size_t)n), out_off((size_t)n);
    std::vector<int> win_first;  // first item of every frame window
    size_t in_bytes = 0, raw_bytes = 0, out_bytes = 0, win_bytes = 0, win_max = 0;
    const size_t kWindow = std::min<size_t>((size_t)12 << 30, L.dev_bytes / 5);  // frames buffer
    int max_w = 0, max_h = 0;
    for (int k = 0; k < n; k++) {
        const PngHeader& ph = *X->items[idx[k]].png;
        const size_t span = ph.idat.back().offset + ph.idat.back().length - ph.idat.front().offset;
        file_off[k] = in_bytes;
        in_bytes += round_up(span + 16, (size_t)16);
    }
    size_t zg = in_bytes;  // gathered streams follow the uploaded file spans
    for (int k = 0; k < n; k++) {
        const XItem& xi = X->items[idx[k]];
        const PngHeader& ph = *xi.png;
        PngDecodeItem& it = items[k];
        memset(&it, 0, sizeof(it));
        it.z_len = (uint32_t)ph.idat_total;
        it.width = ph.width;
        it.height = ph.height;
        it.bit_depth = ph.bit_depth;
        it.color_type = ph.color_type;
        it.src_channels = ph.src_channels;
        it.out_channels = ph.out_channels;
        it.bpp = ph.bpp;
        it.row_bytes = (uint32_t)ph.row_bytes;
        it.frame_stride = (uint32_t)((size_t)xi.w * xi.ch);
        it.interlace = ph.interlace ? 1 : 0;
        png_item_set_passes(&it);
        it.npal = ph.npal;
        it.ntrns = ph.ntrns;
        it.has_trns = ph.has_trns;
        memcpy(it.trns_rgb, ph.trns_rgb, sizeof(it.trns_rgb));
        memcpy(it.palette, ph.palette, sizeof(it.palette));
        memcpy(it.trns, ph.trns, sizeof(it.trns));
        if (ph.idat.size() == 1) {
            it.z_off = file_off[k];
        } else {
            it.z_off = zg;
            size_t o = zg;
            for (const PngSegment& sg : ph.idat) {
                segs.push_back(SegCopy{file_off[k] + (sg.offset - ph.idat.front().offset), o, (uint32_t)sg.length, 0});
                o += sg.length;
            }
            zg += round_up(ph.idat_total + 16, (size_t)16);
        }
        it.raw_off = raw_bytes;
        raw_bytes += round_up((size_t)it.raw_total + 64, (size_t)256);
        const size_t fb = round_up((size_t)xi.w * xi.h * xi.ch, (size_t)256);
        if (k == 0 || win_bytes + fb > kWindow) {  // open a new frame window
            win_first.push_back(k);
            win_bytes = 0;
        }
        frame_off[k] = win_bytes;
        it.frame_off = win_bytes;
        win_bytes += fb;
        win_max = std::max(win_max, win_bytes);
        out_off[k] = out_bytes;
        out_bytes += round_up((size_t)xi.ow * xi.oh * xi.ch, (size_t)256);
        max_w = std::max(max_w, xi.w);
        max_h = std::max(max_h, xi.h);
    }
    win_first.push_back(n);
    // HDR frames are tone-mapped between the defilter and the resize of their window, whole (before the Fit crop, as
    // Transform does); one scratch area sized for the window that needs the most
    std::vector<TmFrame> hdr;
    auto window_hdr = [&](int k0, int k1, uint8_t* frames) {
        hdr.clear();
        for (int k = k0; k < k1; k++) {
            const XItem& xi = X->items[idx[k]];
            if (xi.hdr)
                hdr.push_back(TmFrame{frames ? frames + frame_off[k] : nullptr, (size_t)xi.w * xi.ch, xi.w, xi.h, xi.ch, xi.transfer, xi.primaries});
        }
    };
    size_t tm_bytes = 0;
    for (size_t wdx = 0; wdx + 1 < win_first.size(); wdx++) {
        window_hdr(win_first[wdx], win_first[wdx + 1], nullptr);
        tm_bytes = std::max(tm_bytes, tonemap_batch_scratch_bytes(hdr.data(), (int)hdr.size()));
    }
    uint8_t* d_in = bump.take<uint8_t>(zg + 4096);
    PngDecodeItem* d_items = bump.take<PngDecodeItem>((size_t)n * sizeof(PngDecodeItem));
    SegCopy* d_segs = bump.take<SegCopy>(segs.size() * sizeof(SegCopy) + 16);
    uint8_t* d_raw = bump.take<uint8_t>(raw_bytes + 256);
    uint8_t* d_frames = bump.take<uint8_t>(win_max + 256);
    uint8_t* d_out = bump.take<uint8_t>(out_bytes + 256);
    uint8_t* d_tm = tm_bytes ? bump.take<uint8_t>(tm_bytes) : nullptr;
    if (!d_in || !d_items || !d_segs || !d_raw || !d_frames || !d_out || (tm_bytes && !d_tm)) {
        for (int i : idx) push_fallback(X, i);
        return;
    }
    bool ok = true;
    for (int k = 0; k < n && ok; k++) {
        const PngHeader& ph = *X->items[idx[k]].png;
        const size_t span = ph.idat.back().offset + ph.idat.back().length - ph.idat.front().offset;
        ok = cudaMemcpyAsync(d_in + file_off[k], X->in[idx[k]] + ph.idat.front().offset, span, cudaMemcpyHostToDevice,
                             L.st) == cudaSuccess;
        L.h2d += span;
    }
    ok = ok && cudaMemcpyAsync(d_items, items.data(), (size_t)n * sizeof(PngDecodeItem), cudaMemcpyHostToDevice, L.st) == cudaSuccess;
    if (ok && !segs.empty())
        ok = cudaMemcpyAsync(d_segs, segs.data(), segs.size() * sizeof(SegCopy), cudaMemcpyHostToDevice, L.st) == cudaSuccess;
    cudaEventRecord(L.ev[0], L.st);
    if (ok && !segs.empty()) ok = seg_copy_launch(d_segs, (int)segs.size(), d_in, L.st) == LP_OK;
    PngDecodeBatch b;
    b.items = d_items;
    b.z = d_in;
    b.raw = d_raw;
    b.frames = d_frames;
    b.n = n;
    b.max_width = max_w;
    b.max_height = max_h;
    if (ok) ok = png_inflate_launch(b, L.st) == LP_OK;
    for (size_t wdx = 0; wdx + 1 < win_first.size() && ok; wdx++) {
        const int k0 = win_first[wdx], k1 = win_first[wdx + 1];
        ok = png_unfilter_launch(b, k0, k1 - k0, L.st) == LP_OK;
        window_hdr(k0, k1, d_frames);
        if (ok && !hdr.empty()) ok = tonemap_batch_launch(hdr.data(), (int)hdr.size(), d_tm, tm_bytes, L.st) == LP_OK;
        if (ok) ok = resize_range(X, L, idx, k0, k1, d_frames, frame_off, d_out, out_off);
    }
    cudaEventRecord(L.ev[1], L.st);
    if (ok) ok = cudaMemcpyAsync(items.data(), d_items, (size_t)n * sizeof(PngDecodeItem), cudaMemcpyDeviceToHost, L.st) == cudaSuccess;
    if (ok) ok = cudaStreamSynchronize(L.st) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        for (int i : idx) push_fallback(X, i);
        return;
    }
    lane_time(L, 0, 1, &L.ms_decode);  // (the tone map and resize launches sit between the defilter launches: counted as decode)
    std::vector<char> good((size_t)n);
    for (int k = 0; k < n; k++) good[k] = items[k].status == 0;
    encode_runs(X, L, bump, idx, d_out, out_off, good, &failed);
    for (int i : failed) push_fallback(X, i);
}

// WebP task: stills and animations of any canvas size, every frame of every file.  Decode + composite is one set of
// launches over the task (webp_decode_batch: VP8 frames, VP8L / ALPH waves, the per-pixel compositor); a still is one
// frame copied onto its canvas.  Then one resize per run of equal canvas geometry (its files' canvases lie back to back)
// and the sinks: JPEG and PNG as for every still, WebP as one lossy encode of all the run's frames + the container per file with
// the source's ICC profile, background, loop count and frame durations (what WebpEncoder::Create / Encode pass on).
static void run_webp(lp_xbatch* X, Lane& L, const std::vector<int>& idx) {
    const int n = (int)idx.size();
    Bump bump{L.dev, L.dev_bytes};
    std::vector<const WebpPlan*> plans((size_t)n);
    std::vector<const uint8_t*> files((size_t)n);
    std::vector<size_t> flen((size_t)n);
    std::vector<uint64_t> canvas_off((size_t)n), out_off((size_t)n);
    std::vector<int> first((size_t)n + 1, 0);
    size_t scratch = 4096, arena = 0, canvas_bytes = 0, out_bytes = 0;
    for (int k = 0; k < n; k++) {
        const int i = idx[k];
        const XItem& it = X->items[i];
        plans[k] = it.webp.get();
        files[k] = X->in[i];
        flen[k] = it.span;
        scratch += webp_plan_device_bytes(*plans[k], flen[k]);
        arena += webp_plan_arena_bytes(*plans[k]);
        const int nf = (int)plans[k]->frames.size();
        first[k + 1] = first[k] + nf;
        canvas_off[k] = canvas_bytes;
        canvas_bytes += (size_t)nf * round_up((size_t)it.w * it.h * it.ch, (size_t)256);
        out_off[k] = out_bytes;
        out_bytes += (size_t)nf * round_up((size_t)it.ow * it.oh * it.ch, (size_t)256);
        L.h2d += flen[k];
    }
    arena = std::min(arena, L.dev_bytes / 4);  // (split_by_memory keeps a quarter of the lane for it)
    uint8_t* d_scratch = bump.take<uint8_t>(scratch);
    uint8_t* d_canvases = bump.take<uint8_t>(canvas_bytes + 256);
    uint8_t* d_out = bump.take<uint8_t>(out_bytes + 256);
    uint8_t* d_arena = arena ? bump.take<uint8_t>(arena) : nullptr;
    std::vector<int> st((size_t)n, 0);
    bool ok = d_scratch && d_canvases && d_out && (!arena || d_arena);
    if (ok)  // (the decode time starts once the files are on the device, as for the other kinds)
        ok = webp_decode_batch(plans.data(), files.data(), flen.data(), n, d_scratch, scratch, d_arena, arena, d_canvases,
                               canvas_off.data(), st.data(), L.ev[0], L.st) == LP_OK;
    cudaEventRecord(L.ev[1], L.st);
    const std::vector<Run> runs = runs_of(X, idx);
    for (size_t r = 0; r < runs.size() && ok; r++) {
        const XItem& g = X->items[idx[runs[r].k0]];
        const size_t cs = round_up((size_t)g.w * g.h * g.ch, (size_t)256), os = round_up((size_t)g.ow * g.oh * g.ch, (size_t)256);
        ResizeArgs a{d_canvases + canvas_off[runs[r].k0], cs, (size_t)g.w * g.ch, g.ch, g.cx, g.cy, g.cw, g.chh,
                     d_out + out_off[runs[r].k0], os, (size_t)g.ow * g.ch, g.ow, g.oh, first[runs[r].k1] - first[runs[r].k0], 3};
        ok = resize_launch(a, L.st) == LP_OK;
    }
    cudaEventRecord(L.ev[2], L.st);
    if (ok) ok = cudaStreamSynchronize(L.st) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        for (int i : idx) push_fallback(X, i);
        return;
    }
    lane_time(L, 0, 1, &L.ms_decode);
    lane_time(L, 1, 2, &L.ms_resize);
    std::vector<int> failed;
    cudaEventRecord(L.ev[2], L.st);
    std::vector<uint8_t> file;
    for (const Run& r : runs) {
        const XItem& g = X->items[idx[r.k0]];
        const size_t os = round_up((size_t)g.ow * g.oh * g.ch, (size_t)256);
        if (X->sink != S_WEBP) {  // JPEG, PNG: stills only; a file whose frame failed is encoded with its run, then handed over
            sink_encode(X, L, bump, L.host, L.host_bytes, std::vector<int>(idx.begin() + r.k0, idx.begin() + r.k1),
                        d_out + out_off[r.k0], os, g.ow, g.oh, g.ch, &failed);
            for (int k = r.k0; k < r.k1; k++)
                if (st[k]) failed.push_back(idx[k]);
            continue;
        }
        const int f0 = first[r.k0];
        std::vector<WebpEncodedFrame> frames;
        if (webp_encode_lossy_batch(d_out + out_off[r.k0], os, (size_t)g.ow * g.ch, g.ow, g.oh, g.ch, first[r.k1] - f0,
                                    X->quality, &frames, L.st)) {
            cudaGetLastError();
            failed.insert(failed.end(), idx.begin() + r.k0, idx.begin() + r.k1);
            continue;
        }
        for (int k = r.k0; k < r.k1; k++) {
            const int i = idx[k];
            const WebpPlan& p = *X->items[i].webp;
            bool good = st[k] == 0;
            for (int f = first[k]; f < first[k + 1] && good; f++) good = !frames[f - f0].image.empty();
            if (!good) {  // a damaged stream or an encoder refusal: the per-image path reports the precise error
                failed.push_back(i);
                continue;
            }
            for (int f = first[k]; f < first[k + 1]; f++) {
                frames[f - f0].duration = p.frames[f - first[k]].duration;
                L.d2h += frames[f - f0].image.size() + frames[f - f0].alph.size();
            }
            const std::vector<uint8_t>& icc = X->items[i].icc;
            webp_assemble(&frames[first[k] - f0], first[k + 1] - first[k], icc.data(), icc.size(), p.bgcolor, p.loop_count, &file);
            if (file.size() > X->out_cap) {  // ref webp.cpp:546-551 -> size 0 -> ErrInvalidImage (webp.go:249-251)
                X->status[i] = LP_ERR_INVALID_IMAGE;
                X->out_len[i] = 0;
                continue;
            }
            memcpy(X->out[i], file.data(), file.size());
            X->out_len[i] = file.size();
            X->status[i] = LP_OK;
        }
    }
    cudaEventRecord(L.ev[3], L.st);
    cudaEventSynchronize(L.ev[3]);
    lane_time(L, 2, 3, &L.ms_encode);
    std::sort(failed.begin(), failed.end());
    failed.erase(std::unique(failed.begin(), failed.end()), failed.end());
    for (int i : failed) push_fallback(X, i);
}

// ------------------------------------------------------------------ GIF groups (animations -> animated WebP or GIF)

// GIF sink: palette mapping + LZW of every resized frame of the task in one set of launches, the code streams packed
// and copied home at once, each file assembled on the host from the plan's container metadata
static void gif_sink(lp_xbatch* X, Lane& L, Bump& bump, const std::vector<int>& idx, const std::vector<int>& first,
                     const std::vector<GifAnimPlan*>& plans, const std::vector<int>& st, const uint8_t* d_resized,
                     size_t out_stride) {
    const int na = (int)idx.size();
    const XItem& g = X->items[idx[0]];
    size_t bytes = 0;
    for (GifAnimPlan* p : plans) bytes += gif_plan_encode_bytes(p, g.ow, g.oh);
    uint8_t* d_scratch = bump.take<uint8_t>(bytes);
    std::vector<uint8_t*> out((size_t)na);
    std::vector<size_t> olen((size_t)na, 0);
    std::vector<int> ost((size_t)na, LP_OK);
    for (int a = 0; a < na; a++) out[a] = X->out[idx[a]];
    cudaEventRecord(L.ev[2], L.st);
    int rc = d_scratch ? gif_encode_batch(plans.data(), na, d_resized, out_stride, g.ow, g.oh, first.data(), d_scratch, bytes,
                                          L.host, L.host_bytes, out.data(), X->out_cap, olen.data(), ost.data(), &L.d2h, L.st)
                       : LP_ERR_BUF_TOO_SMALL;
    cudaEventRecord(L.ev[3], L.st);
    cudaEventSynchronize(L.ev[3]);
    lane_time(L, 2, 3, &L.ms_encode);
    for (int a = 0; a < na; a++) {
        const int i = idx[a];
        if (rc || st[a] != 0) {  // a corrupt code stream: the per-image path reports the precise error
            push_fallback(X, i);
            continue;
        }
        X->status[i] = ost[a];
        X->out_len[i] = olen[a];
    }
    if (rc) cudaGetLastError();
}

static void run_gif(lp_xbatch* X, Lane& L, const std::vector<int>& idx) {
    const int na = (int)idx.size();
    const XItem& g = X->items[idx[0]];
    const int w = g.w, h = g.h, ch = 4;
    Bump bump{L.dev, L.dev_bytes};
    const size_t canvas_stride = round_up((size_t)w * h * 4, (size_t)256);
    const size_t out_stride = round_up((size_t)g.ow * g.oh * ch, (size_t)256);
    std::vector<int> first((size_t)na + 1, 0);
    size_t scratch_bytes = 0;
    std::vector<GifAnimPlan*> plans((size_t)na);
    std::vector<const uint8_t*> files((size_t)na);
    std::vector<size_t> flen((size_t)na);
    for (int a = 0; a < na; a++) {
        const XItem& it = X->items[idx[a]];
        first[a + 1] = first[a] + it.gif_frames;
        plans[a] = it.gif;
        files[a] = X->in[idx[a]];
        flen[a] = it.span;
        scratch_bytes += gif_plan_device_bytes(it.gif);
        L.h2d += flen[a];
    }
    const int nf = first[na];
    uint8_t* d_scratch = bump.take<uint8_t>(scratch_bytes + 4096);
    uint8_t* d_canvases = bump.take<uint8_t>((size_t)nf * canvas_stride + 256);
    uint8_t* d_resized = bump.take<uint8_t>((size_t)nf * out_stride + 256);
    std::vector<int> st((size_t)na, 0);
    bool ok = d_scratch && d_canvases && d_resized;
    cudaEventRecord(L.ev[0], L.st);
    if (ok)
        ok = gif_decode_batch(plans.data(), files.data(), flen.data(), na, d_scratch, scratch_bytes + 4096, d_canvases,
                              canvas_stride, first.data(), st.data(), L.st) == LP_OK;
    cudaEventRecord(L.ev[1], L.st);
    if (ok) {
        ResizeArgs r{d_canvases, canvas_stride, (size_t)w * 4, 4, g.cx, g.cy, g.cw, g.chh, d_resized, out_stride,
                     (size_t)g.ow * 4, g.ow, g.oh, nf, 3};
        ok = resize_launch(r, L.st) == LP_OK;
    }
    cudaEventRecord(L.ev[2], L.st);
    if (ok) ok = cudaStreamSynchronize(L.st) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        for (int i : idx) push_fallback(X, i);
        return;
    }
    lane_time(L, 0, 1, &L.ms_decode);
    lane_time(L, 1, 2, &L.ms_resize);
    if (X->sink == S_GIF) {
        gif_sink(X, L, bump, idx, first, plans, st, d_resized, out_stride);
        return;
    }
    cudaEventRecord(L.ev[2], L.st);
    std::vector<WebpEncodedFrame> frames;
    int rc = webp_encode_frames(X, d_resized, out_stride, g.ow, g.oh, 4, nf, &frames, L.st);
    cudaEventRecord(L.ev[3], L.st);
    cudaEventSynchronize(L.ev[3]);
    lane_time(L, 2, 3, &L.ms_encode);
    if (rc) {
        cudaGetLastError();
        for (int i : idx) push_fallback(X, i);
        return;
    }
    std::vector<uint8_t> file;
    for (int a = 0; a < na; a++) {
        const int i = idx[a];
        bool good = st[a] == 0;
        for (int f = first[a]; f < first[a + 1] && good; f++) good = !frames[f].image.empty();
        if (!good) {
            push_fallback(X, i);
            continue;
        }
        uint32_t bg = 0xFFFFFFFFu;
        int loops = 0;
        gif_plan_info(X->items[i].gif, nullptr, nullptr, nullptr, &bg, &loops);
        for (int f = first[a]; f < first[a + 1]; f++) {
            frames[f].duration = gif_plan_delay_ms(X->items[i].gif, f - first[a]);
            L.d2h += frames[f].image.size() + frames[f].alph.size();
        }
        webp_assemble(&frames[first[a]], first[a + 1] - first[a], nullptr, 0, bg, (uint32_t)loops, &file);
        if (file.size() > X->out_cap) {
            X->status[i] = LP_ERR_INVALID_IMAGE;
            X->out_len[i] = 0;
            continue;
        }
        memcpy(X->out[i], file.data(), file.size());
        X->out_len[i] = file.size();
        X->status[i] = LP_OK;
    }
}

// ------------------------------------------------------------------ JPEG groups (the lp_batch pipeline)

// Device bytes one WebP encode of a JPEG group's frames may allocate (webp_encode_lossy_batch's scratch lives outside the
// lane's arena): 1 GiB holds 717 frames of 256x256 (1.43 MiB each, webp_encode_lossy_scratch_bytes), and stays below
// what one encode of a PNG task of bench.py's config 3 takes (6.4 MiB per 512x512 RGBA frame, hundreds of frames).
static constexpr size_t kJpegWebpScratch = (size_t)1 << 30;
// Frames of a JPEG group the PNG sink is sure to have arena for (run_jpeg keeps that much out of the decode chunks' reach)
static constexpr size_t kJpegPngFrames = 512;

// WebP and PNG sinks: the group through a resize-only lp_batch context (decode + resize of every image, one chunk after
// another), then the sink's encoder over its resized frames.  WebP: in sub-batches of at most the decode chunk's image
// count and kJpegWebpScratch of encoder scratch.  PNG: out of what the context left of the lane's arena and pinned
// staging.  Items the decode refused go to the per-image path without being encoded.
static void jpeg_to_sink(lp_xbatch* X, Lane& L, lp_batch* b, const std::vector<int>& idx, const uint8_t* const* in,
                         const size_t* len) {
    const int n = (int)idx.size();
    const XItem& g = X->items[idx[0]];
    std::vector<int> st((size_t)n, LP_ERR_CUDA);
    float stage[LP_STAGE_COUNT] = {};
    if (lp_batch_stage(b, in, len, n, nullptr) != LP_OK || lp_batch_run(b, stage) != LP_OK ||
        batch_resized_status(b, st.data()) != LP_OK) {
        cudaGetLastError();
        for (int i : idx) push_fallback(X, i);
        return;
    }
    L.ms_decode += stage[LP_STAGE_HUFF_DECODE] + stage[LP_STAGE_IDCT_COLOR];
    L.ms_resize += stage[LP_STAGE_RESIZE];
    size_t stride = 0;
    const uint8_t* d_resized = lp_batch_resized_dev(b, &stride);
    int sub = n;
    if (X->sink == S_WEBP) {
        const size_t per_frame = webp_encode_lossy_scratch_bytes(g.ow, g.oh, 3, 1);
        sub = (int)std::max<size_t>(1, std::min<size_t>((size_t)lp_batch_chunk(b), kJpegWebpScratch / per_frame));
    }
    std::vector<int> failed;
    size_t dev_used = 0, host_used = 0;
    batch_arena_used(b, &dev_used, &host_used);
    Bump bump{L.dev + dev_used, L.dev_bytes - dev_used};  // (the WebP branch of sink_encode takes nothing from it)
    cudaEventRecord(L.ev[2], L.st);
    // runs of decoded items (their frames back to back), at most `sub` long; a refused item goes to the per-image path
    for (int k0 = 0; k0 < n;) {
        if (st[k0] != LP_OK) {
            failed.push_back(idx[k0++]);
            continue;
        }
        int k1 = k0 + 1;
        while (k1 < n && k1 - k0 < sub && st[k1] == LP_OK) k1++;
        sink_encode(X, L, bump, L.host + host_used, L.host_bytes - host_used, std::vector<int>(idx.begin() + k0, idx.begin() + k1),
                    d_resized + (size_t)k0 * stride, stride, g.ow, g.oh, 3, &failed);
        k0 = k1;
    }
    cudaEventRecord(L.ev[3], L.st);
    cudaEventSynchronize(L.ev[3]);
    lane_time(L, 2, 3, &L.ms_encode);
    for (int i : failed) push_fallback(X, i);
}

static void run_jpeg(lp_xbatch* X, Lane& L, const std::vector<int>& idx) {
    const int n = (int)idx.size();
    const XItem& g = X->items[idx[0]];
    const bool resize_only = X->sink != S_JPEG;  // WebP, PNG: the frames go to that sink's encoder
    size_t in_bytes = 0;
    for (int i : idx) in_bytes += X->in_len[i];
    lp_batch_config c;
    memset(&c, 0, sizeof(c));
    c.device = X->device;
    c.max_images = n;
    c.src_width = g.w;
    c.src_height = g.h;
    c.dst_width = X->opt.width;
    c.dst_height = X->opt.height;
    c.resize_method = X->opt.resize_method;
    c.jpeg_quality = X->quality;
    c.max_in_bytes = in_bytes + (1 << 20);
    // slot per output: never larger than the callers' buffers (lp_batch copies a whole result into out[i])
    c.out_cap = std::min(X->out_cap, round_up(std::max((size_t)65536, (size_t)g.ow * g.oh * 3), (size_t)256));
    if (c.out_cap >= 256) c.out_cap = c.out_cap / 256 * 256;
    // images per chunk: whole Huffman waves while the per-chunk scratch fits the lane's arena
    const size_t mcus = (size_t)ceil_div(g.w, 8) * ceil_div(g.h, 8);
    // multi-scan groups: + the nonzero masks per block, + the scan and table-set pools (batch.cu)
    const size_t per_img = (mcus * 3 + 64) * (128 + 64 + 2 + (g.jpeg_multiscan ? 8 : 0)) + (size_t)g.w * g.h * 3 + 65536;
    const size_t pools = g.jpeg_multiscan ? batch_multiscan_pool_bytes((size_t)n) : 0;
    const size_t png_room =
        X->sink == S_PNG ? std::min(L.dev_bytes / 4, std::min((size_t)n, kJpegPngFrames) * png_sink_item_bytes(X, g.ow, g.oh, 3)) : 0;
    const size_t fixed = 2 * in_bytes + (size_t)n * ((resize_only ? 0 : c.out_cap) + (size_t)g.ow * g.oh * 3 + 4096) + (64u << 20) + pools + png_room;
    const int slots = jpeg_huff_parallel_slots();
    long fit = L.dev_bytes > fixed ? (long)((L.dev_bytes - fixed) / per_img) : 0;
    if (fit < 1) {
        for (int i : idx) push_fallback(X, i);
        return;
    }
    int chunk = (int)std::min<long>(fit, 3L * std::max(slots, 1));
    if (slots > 0 && chunk > slots) chunk = chunk / slots * slots;
    c.chunk = std::max(1, std::min(chunk, n));
    lp_batch* b = batch_create_in(&c, L.dev, L.dev_bytes, L.host, L.host_bytes, X->progressive, g.jpeg_multiscan, resize_only);
    if (!b) {
        for (int i : idx) push_fallback(X, i);
        return;
    }
    std::vector<const uint8_t*> in((size_t)n);
    std::vector<size_t> len((size_t)n), olen((size_t)n, 0);
    std::vector<uint8_t*> out((size_t)n);
    std::vector<int> st((size_t)n, 0);
    for (int k = 0; k < n; k++) {
        in[k] = X->in[idx[k]];
        len[k] = X->in_len[idx[k]];
        out[k] = X->out[idx[k]];
    }
    L.h2d += in_bytes;
    if (resize_only) {
        jpeg_to_sink(X, L, b, idx, in.data(), len.data());
        lp_batch_destroy(b);
        return;
    }
    cudaEventRecord(L.ev[0], L.st);
    const int rc = lp_batch_transform(b, in.data(), len.data(), n, out.data(), olen.data(), st.data());
    for (int k = 0; k < n; k++) {
        const int i = idx[k];
        if (rc || st[k] != LP_OK) {
            push_fallback(X, i);  // whatever the batch pipeline would not take: Transform decides
            continue;
        }
        X->out_len[i] = olen[k];
        X->status[i] = LP_OK;
        L.d2h += olen[k];
    }
    lp_batch_destroy(b);
}

// ------------------------------------------------------------------ the call

extern "C" lp_xbatch* lp_xbatch_create(const lp_xbatch_config* cfg) {
    if (!cfg) return nullptr;
    if (ensure_device()) return nullptr;
    int prev = 0;
    cudaGetDevice(&prev);
    if (cudaSetDevice(cfg->device) != cudaSuccess) return nullptr;
    lp_xbatch* X = new lp_xbatch;
    X->cfg = *cfg;
    X->device = cfg->device;
    memset(&X->stats, 0, sizeof(X->stats));
    unsigned hc = std::thread::hardware_concurrency();
    X->threads = cfg->host_threads > 0 ? cfg->host_threads : (int)std::min(16u, std::max(2u, hc));
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    size_t arena = cfg->arena_bytes ? cfg->arena_bytes : (size_t)(free_b * 0.72);
    arena = arena / 2 / 4096 * 4096 * 2;
    X->host_bytes = (size_t)2 << 30;
    bool ok = cudaMalloc(&X->arena, arena) == cudaSuccess && cudaMallocHost(&X->host_arena, X->host_bytes) == cudaSuccess;
    X->arena_bytes = arena;
    for (int l = 0; l < 2 && ok; l++) {
        Lane& L = X->lanes[l];
        L.id = l;
        L.dev = X->arena + (size_t)l * (arena / 2);
        L.dev_bytes = arena / 2;
        L.host = X->host_arena + (size_t)l * (X->host_bytes / 2);
        L.host_bytes = X->host_bytes / 2;
        ok = cudaStreamCreateWithFlags(&L.st, cudaStreamNonBlocking) == cudaSuccess;
        for (int e = 0; e < 4 && ok; e++) ok = cudaEventCreate(&L.ev[e]) == cudaSuccess;
    }
    cudaSetDevice(prev);
    if (!ok) {
        fprintf(stderr, "[lilliput_b200] lp_xbatch_create: device arena (%zu B) or pinned staging allocation failed\n", arena);
        cudaGetLastError();
        lp_xbatch_destroy(X);
        return nullptr;
    }
    return X;
}

extern "C" void lp_xbatch_destroy(lp_xbatch* X) {
    if (!X) return;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(X->device);
    cudaDeviceSynchronize();
    for (Lane& L : X->lanes) {
        for (auto& e : L.ev)
            if (e) cudaEventDestroy(e);
        if (L.st) cudaStreamDestroy(L.st);
    }
    if (X->arena) cudaFree(X->arena);
    if (X->host_arena) cudaFreeHost(X->host_arena);
    cudaSetDevice(prev);
    delete X;
}

extern "C" void lp_xbatch_get_stats(const lp_xbatch* X, lp_xbatch_stats* out) {
    if (X && out) *out = X->stats;
}

template <class F>
static void parallel_for(int n, int threads, F&& fn) {
    if (n <= 0) return;
    threads = std::max(1, std::min(threads, n));
    if (threads == 1) {
        for (int i = 0; i < n; i++) fn(i);
        return;
    }
    std::atomic<int> next{0};
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; t++)
        pool.emplace_back([&]() {
            for (;;) {
                const int i = next.fetch_add(1);
                if (i >= n) break;
                fn(i);
            }
        });
    for (auto& th : pool) th.join();
}

// device bytes one item of a group needs inside a lane's arena (upper bound, sinks included)
static size_t item_device_bytes(const lp_xbatch* X, const XItem& it, int i) {
    const size_t outb = (size_t)it.ow * it.oh * 4 * 3 + (256u << 10) + (X->sink == S_PNG ? png_sink_item_bytes(X, it.ow, it.oh, it.ch) : 0);
    switch (it.kind) {
        case K_PNG: {
            // compressed span (+ its gathered copy) + inflated scanlines (the header's row bytes: twice the samples' count
            // at 16 bits) + resized output + an HDR frame's tone-map records; the packed frames live in a window buffer
            // shared by the task (a fifth of the lane's arena, reserved by split_by_memory)
            const size_t row = std::max((size_t)it.w * (it.ch == 4 ? 4 : 3), it.png ? it.png->row_bytes : 0);
            const size_t raw = (row + 2) * it.h * (it.png && it.png->interlace ? 2 : 1);
            const TmFrame tm{nullptr, 0, it.w, it.h, it.ch, it.transfer, it.primaries};
            return 2 * X->in_len[i] + raw + outb + 8192 + (it.hdr ? tonemap_batch_scratch_bytes(&tm, 1) : 0);
        }
        case K_WEBP:  // the VP8L arena (at most a quarter of the lane) is shared by the task (reserved by split_by_memory)
            return webp_plan_device_bytes(*it.webp, it.span) +
                   it.webp->frames.size() * (round_up((size_t)it.w * it.h * it.ch, (size_t)256) + outb) + 8192;
        case K_GIF:
            return gif_plan_device_bytes(it.gif) + (size_t)it.gif_frames * ((size_t)it.w * it.h * 4 + outb) + 8192 +
                   (X->sink == S_GIF ? gif_plan_encode_bytes(it.gif, it.ow, it.oh) : 0);
        default:
            return 0;
    }
}

extern "C" int lp_xbatch_transform(lp_xbatch* X, const uint8_t* const* in, const size_t* in_len, int n,
                                   const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                                   int* status) {
    if (!X || n < 0 || !opt || (n > 0 && (!in || !in_len || !out || !out_len || !status))) return LP_ERR_BAD_ARGUMENT;
    int prev = 0;
    cudaGetDevice(&prev);
    LP_CUDA_OK(cudaSetDevice(X->device));
    const auto t0 = std::chrono::steady_clock::now();
    X->in = in;
    X->in_len = in_len;
    X->out = out;
    X->out_cap = out_cap;
    X->out_len = out_len;
    X->status = status;
    X->opt = *opt;
    X->items.clear();
    X->items.resize((size_t)n);
    X->fallback.clear();
    memset(&X->stats, 0, sizeof(X->stats));
    for (Lane& L : X->lanes) {
        L.ms_decode = L.ms_resize = L.ms_encode = 0;
        L.h2d = L.d2h = 0;
        L.launches = 0;
    }
    for (int i = 0; i < n; i++) {
        status[i] = LP_ERR_UNSUPPORTED;  // every item is overwritten by its group or by the fallback
        out_len[i] = 0;
    }
    // which sink the options ask for (ref lilliput.go:176-195 NewEncoder by extension)
    std::string ext = opt->file_type ? opt->file_type : "";
    for (auto& c : ext) c = (char)tolower((unsigned char)c);
    X->sink = S_NONE;
    X->lossless = false;
    X->progressive = false;
    if (ext == ".jpeg" || ext == ".jpg") {
        X->sink = S_JPEG;
        X->quality = option_value(*opt, CV_IMWRITE_JPEG_QUALITY, 95);  // OpenCV's default
        X->progressive = option_value(*opt, CV_IMWRITE_JPEG_PROGRESSIVE, 0) != 0;
    } else if (ext == ".webp") {
        const int q = option_value(*opt, CV_IMWRITE_WEBP_QUALITY, 100);
        X->quality = q < 1 ? 1 : q;
        X->sink = S_WEBP;
        X->lossless = q > 100;
    } else if (ext == ".gif") {
        X->sink = S_GIF;
    } else if (ext == ".png") {
        X->sink = S_PNG;
        png_encode_policy(opt->encode_options, opt->encode_options_len, &X->png_level, &X->png_adaptive);
    }
    parallel_for(n, X->threads, [&](int i) { parse_item(X, i); });
    const auto t1 = std::chrono::steady_clock::now();
    // groups -> tasks that fit a lane
    std::map<std::tuple<int, int, int, int, int>, std::vector<int>> groups;
    for (int i = 0; i < n; i++) {
        const XItem& it = X->items[i];
        if (it.kind == K_FALLBACK) X->fallback.push_back(i);
        else groups[std::make_tuple((int)it.kind, it.w, it.h, it.ch, it.jpeg_sampling | (it.jpeg_multiscan ? 1 << 24 : 0))].push_back(i);
    }
    std::vector<Task> tasks;
    std::vector<double> cost;  // rough device time: the longest tasks start first
    const size_t lane_cap = X->lanes[0].dev_bytes;
    // PNG and WebP: all geometries of a kind in as few tasks as the arena allows (the map keeps equal
    // geometries adjacent); at least two, so both lanes work.  GIF: by canvas size.  JPEG: by geometry.
    std::map<int, std::vector<int>> merged;
    for (auto& kv : groups) {
        const Kind kind = (Kind)std::get<0>(kv.first);
        if (kind == K_PNG || kind == K_WEBP) merged[(int)kind].insert(merged[(int)kind].end(), kv.second.begin(), kv.second.end());
    }
    auto split_by_memory = [&](Kind kind, const std::vector<int>& g) {
        size_t total = 0;
        for (int i : g) total += item_device_bytes(X, X->items[i], i);
        const size_t half = total / 2 + 1;
        Task cur{kind, {}};
        double work = 64u << 20;  // WebP: the order key counts pixels and payload bytes, not the decoders' scratch
        // PNG: the frame window; WebP: the VP8L / ALPH arena, when some file has lossless frames or alpha planes
        size_t arena = 0;
        if (kind == K_WEBP)
            for (int i : g) arena = std::min(lane_cap / 4, arena + webp_plan_arena_bytes(*X->items[i].webp));
        const size_t reserve = (kind == K_PNG ? lane_cap / 5 : arena) + (64u << 20);
        size_t used = reserve;
        for (int i : g) {
            const size_t need = item_device_bytes(X, X->items[i], i) +
                                (kind == K_PNG ? 0 : 0);
            if (kind == K_PNG && round_up((size_t)X->items[i].w * X->items[i].h * X->items[i].ch, (size_t)256) > std::min<size_t>((size_t)12 << 30, lane_cap / 5)) {
                X->fallback.push_back(i);  // one frame larger than the window
                continue;
            }
            if (need + reserve > lane_cap) {
                X->fallback.push_back(i);
                continue;
            }
            if (!cur.idx.empty() && (used + need > lane_cap || used > half + reserve)) {
                tasks.push_back(cur);
                cost.push_back(kind == K_WEBP ? work : (double)used);
                cur.idx.clear();
                used = reserve;
                work = 64u << 20;
            }
            cur.idx.push_back(i);
            used += need;
            if (kind == K_WEBP) {
                const XItem& it = X->items[i];
                work += (double)it.span + 4096 +
                        (double)it.webp->frames.size() * ((double)it.w * it.h * it.ch + (double)it.ow * it.oh * 12 + (256u << 10));
            }
        }
        if (!cur.idx.empty()) {
            tasks.push_back(cur);
            cost.push_back(kind == K_WEBP ? work : (double)used);
        }
    };
    for (auto& kv : merged) split_by_memory((Kind)kv.first, kv.second);
    for (auto& kv : groups) {
        const Kind kind = (Kind)std::get<0>(kv.first);
        const std::vector<int>& g = kv.second;
        if (kind == K_PNG || kind == K_WEBP) continue;
        if (kind == K_JPEG) {
            // host staging bounds a JPEG task: out slots (JPEG sink only) + item mirrors come from the lane's pinned arena
            const XItem& it0 = X->items[g[0]];
            const size_t slot = (X->sink == S_JPEG ? round_up(std::min(out_cap, std::max((size_t)65536, (size_t)it0.ow * it0.oh * 3)), (size_t)256) : 0) +
                                sizeof(JpegDecodeItem) + 64;
            const size_t per = std::max<size_t>(1, X->lanes[0].host_bytes / slot);
            const size_t want = std::min(per, std::max<size_t>(1, (g.size() + 1) / 2));  // two tasks at least: both lanes work
            for (size_t a = 0; a < g.size(); a += want) {
                tasks.push_back(Task{kind, std::vector<int>(g.begin() + a, g.begin() + std::min(g.size(), a + want))});
                cost.push_back((double)tasks.back().idx.size() * it0.w * it0.h * 0.05);
            }
            continue;
        }
        split_by_memory(kind, g);
    }
    {   // longest first
        std::vector<int> order(tasks.size());
        for (size_t t = 0; t < order.size(); t++) order[t] = (int)t;
        std::sort(order.begin(), order.end(), [&](int a, int b) { return cost[a] > cost[b]; });
        std::vector<Task> sorted;
        for (int t : order) sorted.push_back(std::move(tasks[t]));
        tasks.swap(sorted);
    }
    X->stats.groups = (int)groups.size();
    // two lanes drain the task list
    std::atomic<int> next{0};
    const long launches0 = g_launches;
    std::atomic<long> lane_launches{0};
    auto lane_main = [&](int l) {
        cudaSetDevice(X->device);
        Lane& L = X->lanes[l];
        const long mine0 = g_launches;
        for (;;) {
            const int t = next.fetch_add(1);
            if (t >= (int)tasks.size()) break;
            const Task& task = tasks[t];
            switch (task.kind) {
                case K_JPEG: run_jpeg(X, L, task.idx); break;
                case K_PNG: run_png(X, L, task.idx); break;
                case K_WEBP: run_webp(X, L, task.idx); break;
                case K_GIF: run_gif(X, L, task.idx); break;
                default: for (int i : task.idx) push_fallback(X, i); break;
            }
        }
        lane_launches += g_launches - mine0;
    };
    {
        std::thread other(lane_main, 1);
        lane_main(0);
        other.join();
    }
    (void)launches0;
    const auto t2 = std::chrono::steady_clock::now();
    // everything else, one image per call, a few host threads (each has its own stream)
    const int max_size = X->cfg.max_size > 0 ? X->cfg.max_size : 8192;
    std::atomic<long> fb_launches{0};
    {
        std::vector<int> fb = X->fallback;
        parallel_for((int)fb.size(), std::min(X->threads, 8), [&](int k) {
            cudaSetDevice(X->device);
            const long l0 = g_launches;
            const int i = fb[k];
            size_t len = 0;
            status[i] = lp_transform(in[i], in_len[i], opt, out[i], out_cap, &len, max_size);
            out_len[i] = status[i] == LP_OK ? len : 0;
            fb_launches += g_launches - l0;
        });
        X->stats.fallback_items = (int)fb.size();
    }
    for (XItem& it : X->items)
        if (it.gif) {
            gif_plan_free(it.gif);
            it.gif = nullptr;
        }
    const auto t3 = std::chrono::steady_clock::now();
    auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
        return std::chrono::duration<double, std::milli>(b - a).count();
    };
    X->stats.grid_items = n - X->stats.fallback_items;
    X->stats.ms_parse = ms(t0, t1);
    X->stats.ms_grid = ms(t1, t2);
    X->stats.ms_fallback = ms(t2, t3);
    X->stats.ms_total = ms(t0, t3);
    for (Lane& L : X->lanes) {
        X->stats.ms_decode += L.ms_decode;
        X->stats.ms_resize += L.ms_resize;
        X->stats.ms_encode += L.ms_encode;
        X->stats.h2d_bytes += L.h2d;
        X->stats.d2h_bytes += L.d2h;
        X->stats.launches += (int)L.launches;
        X->stats.ms_busy_max_lane = std::max(X->stats.ms_busy_max_lane, L.ms_decode + L.ms_resize + L.ms_encode);
    }
    X->stats.launches += (int)(lane_launches.load() + fb_launches.load());
    cudaSetDevice(prev);
    return LP_OK;
}

// ------------------------------------------------------------------ library-level multi-GPU dispatch
// SURVEY 8(e): images are independent units with zero exchange -- the batch is cut into one contiguous block per
// GPU, balanced by compressed bytes, and each block runs through that GPU's own lp_xbatch (own arena, pinned
// staging, streams) on its own host thread; results land in the caller's arrays by index.  No collective, no
// peer traffic.  (bench.py's torchrun harness is the process-per-GPU form of the same sharding.)

struct lp_multi {
    std::vector<lp_xbatch*> ctx;
    std::vector<int> devices;
    std::vector<int> first;  // block boundaries of the last call (ctx.size() + 1)
};

extern "C" lp_multi* lp_multi_create(const int* devices, int n_devices, const lp_xbatch_config* tmpl) {
    if (n_devices < 1 || !devices) return nullptr;
    lp_multi* m = new lp_multi;
    for (int g = 0; g < n_devices; g++) {
        lp_xbatch_config c;
        memset(&c, 0, sizeof(c));
        if (tmpl) c = *tmpl;
        c.device = devices[g];
        lp_xbatch* x = lp_xbatch_create(&c);
        if (!x) {
            for (lp_xbatch* y : m->ctx) lp_xbatch_destroy(y);
            delete m;
            return nullptr;
        }
        m->ctx.push_back(x);
        m->devices.push_back(devices[g]);
    }
    return m;
}

extern "C" void lp_multi_destroy(lp_multi* m) {
    if (!m) return;
    for (lp_xbatch* x : m->ctx) lp_xbatch_destroy(x);
    delete m;
}

extern "C" int lp_multi_device_count(const lp_multi* m) { return m ? (int)m->ctx.size() : 0; }

// Host-only: cut n items into `parts` contiguous blocks with (nearly) equal compressed bytes (SURVEY 8(e): "contiguous
// blocks balanced by compressed bytes"); first[p] .. first[p + 1] is block p, first has parts + 1 entries.
extern "C" void lp_shard_blocks(const size_t* in_len, int n, int parts, int* first) {
    if (parts < 1 || !first) return;
    for (int p = 0; p <= parts; p++) first[p] = n < 0 ? 0 : n;
    first[0] = 0;
    if (n <= 0 || !in_len) return;
    size_t total = 0;
    for (int i = 0; i < n; i++) total += in_len[i] + 4096;  // (+ a per-image constant: tiny files still cost a launch slot)
    size_t acc = 0;
    int g = 1;
    for (int i = 0; i < n && g < parts; i++) {
        acc += in_len[i] + 4096;
        while (g < parts && acc * (size_t)parts >= total * (size_t)g) first[g++] = i + 1;
    }
}

extern "C" int lp_multi_transform(lp_multi* m, const uint8_t* const* in, const size_t* in_len, int n,
                                  const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                                  int* status) {
    if (!m || n < 0 || !opt || (n > 0 && (!in || !in_len || !out || !out_len || !status))) return LP_ERR_BAD_ARGUMENT;
    const int G = (int)m->ctx.size();
    m->first.assign((size_t)G + 1, n);
    lp_shard_blocks(in_len, n, G, m->first.data());
    std::vector<int> rc((size_t)G, LP_OK);
    std::vector<std::thread> pool;
    for (int g = 0; g < G; g++) {
        const int i0 = m->first[g], cnt = m->first[g + 1] - m->first[g];
        if (cnt <= 0) continue;
        pool.emplace_back([=, &rc]() {
            rc[g] = lp_xbatch_transform(m->ctx[g], in + i0, in_len + i0, cnt, opt, out + i0, out_cap, out_len + i0, status + i0);
        });
    }
    for (auto& t : pool) t.join();
    for (int g = 0; g < G; g++)
        if (rc[g]) return rc[g];
    return LP_OK;
}

// per-device statistics of the last call
extern "C" void lp_multi_get_stats(const lp_multi* m, int device_index, lp_xbatch_stats* out) {
    if (m && out && device_index >= 0 && device_index < (int)m->ctx.size()) lp_xbatch_get_stats(m->ctx[device_index], out);
}
