// xbatch.cu -- the heterogeneous batch entry point (include/lilliput_b200.h: lp_xbatch_*): N independent
// images of ANY supported format and size through ImageOps.Transform with one set of options, the
// per-image work packed into grid launches.
//
// Renditions (lp_xbatch_transform_renditions): k sets of options, each a Rendition record, and n * k (item, rendition)
// pairs, each with lp_transform(in[i], opts[r])'s status and bytes; lp_xbatch_transform is k = 1.  A file's container
// and header are parsed once (ItemHeaders); one gate function per source format then runs per pair, for every sink, and
// gives each item the mask of renditions it takes on the grid.  A file is uploaded and decoded once for all of them:
// PNG and WebP stills resize each decoded frame window into every rendition, JPEG groups with several renditions decode
// the bounding box of their crops through one resize-only lp_batch context that resizes each chunk into every
// rendition's geometry, and each rendition's frames then go through its own sink.  Animations (GIF, animated WebP) run
// each rendition as a task of its own.
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
//        frames -> lp_xbatch_encode_frames: no file but slice i of a caller's device tensor, w[i] x h[i] at its top-left,
//                 unpacked into u8 BGR / BGRA frames by one launch over the task (frames_pack.cu); the item passes the
//                 gates of an 8-bit RGB / RGBA PNG (parse_frame_pair), and under NoResize its frame goes to the sink
//                 unresized.  lp_xbatch_encode_clips: T slices per item, a clip of nframes >= 2 passing the gates of its
//                 animated WebP A_i (clip_gates); the frames its output reads are unpacked as an animation's canvases
//        DisableAnimatedOutput (GIF and animated WebP to WebP, GIF to GIF): Transform stops after frame 0, so the plan
//                 stops there too (gif_plan_parse's first-frame walk, webp_plan_cut); only the file up to the
//                 end of frame 0's image data is uploaded, the same kernels run over one frame per file, and the sink
//                 writes a still WebP or a one-frame GIF
//      and the sinks: JPEG (jpeg_encode.cu), lossy WebP still / animation (webp_encode.cu) carrying the ICC profile of
//      a JPEG, PNG or WebP source as WebpEncoder does, lossless WebP still / animation from PNG and GIF sources (the
//      batched VP8L encoder over every frame of a run, webp_encode.cu; a PNG's ICC profile carried the same way), GIF
//      from GIF sources (palette mapping + LZW of every frame of the task, gif_decode.cu; the container assembled on the
//      host), PNG from JPEG, PNG and WebP stills (filter, DEFLATE, checksums and container of every frame of a run in
//      three launches, png_encode.cu), and pixels instead of files (lp_xbatch_decode_frames: each run's frames packed
//      into the caller's device tensor in one launch, frames_pack.cu; lp_xbatch_decode_clips: T slots per item, an
//      animation's plan cut after its last selected frame and only the selected frames' canvases stored).  Whatever the decoder kind, a task's decoded frames go through one run walk
//      (task_runs: adjacent items that take a rendition and share a geometry), one resize launch per run, and one sink
//      entry (sink_encode) per run of resized frames;
//   3. anything the grid path does not cover (over-budget multi-scan JPEGs, gray JPEGs and EXIF-rotated sources to
//      files, gray PNGs, SDR-cICP PNGs to PNG (Transform re-attaches the chunk), lossless WebP output of JPEG and WebP
//      sources, PNG output of animations, GIF output from other formats, animations under MaxEncodeFrames or
//      MaxEncodeDuration, one-frame GIFs to WebP with no time to encode ...) and any item whose grid stage fails goes
//      through lp_transform on a worker thread -- still this library's device kernels, one image per call -- so the
//      status and bytes of EVERY item are what lp_transform would have returned.
// Two worker lanes, each with half of the device arena and its own stream, process chunks of groups
// concurrently, so one lane's PCIe copies and host-side container work overlap the other lane's kernels.
// Nothing is exchanged between images, lanes or GPUs.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <climits>
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
                          bool gray_sources = false,      // grouping, except by frame renditions)
                          const BatchGeom* geoms = nullptr, int n_geoms = 0);
int batch_resized_status(lp_batch* b, int* status);
const uint8_t* batch_resized_geom(const lp_batch* b, int g, size_t* image_stride);
size_t batch_multiscan_pool_bytes(size_t n);
void batch_arena_used(const lp_batch* b, size_t* dev_bytes, size_t* host_bytes);
int mat_device_view(void* mat, int* cols, int* rows, int* type, const uint8_t** dev, size_t* step);
int mat_bind_device_frame(void* mat, int cols, int rows, int type, uint8_t** dev, size_t* step);
}  // namespace lp

namespace {

enum Kind { K_FALLBACK = 0, K_JPEG = 1, K_PNG = 2, K_WEBP = 3, K_GIF = 4, K_FRAME = 5 };  // K_FRAME: lp_xbatch_encode_frames
enum Sink { S_NONE = 0, S_JPEG = 1, S_WEBP = 2, S_GIF = 3, S_PNG = 4, S_FRAMES = 5 };  // S_FRAMES: a frame rendition
constexpr int kMaxRenditions = LP_XBATCH_MAX_RENDITIONS;  // (a rendition mask is one 32-bit word)

// One output the call asks of every item: its options and what the sink takes from them
struct Rendition {
    lp_image_options opt;
    Sink sink = S_NONE;
    int quality = 0;
    bool lossless = false;     // S_WEBP: lossless (VP8L) frames, WebpQuality above 100
    bool progressive = false;  // S_JPEG: progressive files (JpegProgressive)
    int png_level = 1;         // S_PNG: zlib level and filter policy (png_encode_policy)
    bool png_adaptive = false;
    lp_frame_tensor dst{};     // S_FRAMES: the caller's tensor (item i's slices from i * max(1, clip_t)) and each item's
    int* frame_w = nullptr;    // frame size (its status is the pair's)
    int* frame_h = nullptr;
};

// One (item, rendition) pair.  The source fields (kind, frame, JPEG layout, PNG header, HDR tags) are the item's and
// equal in all its pairs; the output size, crop, ICC profile, and an animation's plan and span are the rendition's.
struct XItem {
    Kind kind = K_FALLBACK;
    int w = 0, h = 0, ch = 0;       // decoded frame
    int ow = 0, oh = 0;             // output size
    int cx = 0, cy = 0, cw = 0, chh = 0;  // crop rectangle fed to the resize
    int jpeg_sampling = 0;          // (h0<<12)|(v0<<8)|... groups JPEGs of one component layout
    bool jpeg_multiscan = false;    // progressive, or one scan per component
    bool jpeg_frames_only = false;  // rotated (EXIF 2..8) or gray: only frame renditions take it on the grid
    std::shared_ptr<const PngHeader> png;
    bool hdr = false;                 // PNG: a cICP chunk with a PQ (16) or HLG (18) transfer, tone-mapped after the decode
    int transfer = 0, primaries = 0;  // (its code points)
    std::unique_ptr<WebpPlan> webp;  // (for WebP: the frames' spans, rectangles and blend / dispose)
    bool webp_animation = false;     // the source has several frames (the pair's plan may be cut to frame 0)
    std::shared_ptr<GifAnimPlan> gif;
    int gif_frames = 0;
    size_t span = 0;           // WebP, GIF: bytes at the start of the file the device reads (first-frame items: through frame 0)
    int nframes = 0;                  // lp_xbatch_decode_clips: F, the frame count the decoder's header reports,
    std::vector<int> clip;            // the frames of the slots in use (the only canvases stored, the plan cut after the last)
    std::vector<int64_t> clip_ms;     // and each one's start (ms)
    int src_frames = 1;  // K_FRAME: the item's frames the output reads, slices i * T .. (nframes to an animated .webp)
    std::vector<uint8_t> icc;  // WebP sink: the source's profile the WebP writer carries (empty: none, or not sane)
};

// A task: items of ONE decoder kind, each with the renditions it runs on the grid in this task (rm, a bit per
// rendition).  Its decode runs once per item; resize and encode once per (item, rendition).  An animation's task
// holds one rendition.
struct Task {
    Kind kind;
    std::vector<int> idx;  // items (for GIF: animations)
    std::vector<uint32_t> rm;
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
    int* status = nullptr;  // (out, out_len and status: one entry per pair, item-major)
    lp_frame_tensor frames;  // lp_xbatch_encode_frames and _clips: the caller's source tensor
    int clip_t = 0;  // lp_xbatch_decode_clips: T slots per item (0: one, any other call), and the slots' outputs
    int* clip_nframes = nullptr;
    int* clip_index = nullptr;
    int64_t* clip_ms = nullptr;
    const int* src_w = nullptr;  // lp_xbatch_encode_frames: the items are slices of `frames`, of these sizes (no files)
    const int* src_h = nullptr;
    int src_t = 1;  // lp_xbatch_encode_clips: T slices per item (1 for lp_xbatch_encode_frames), the frames each item
    const int* src_nframes = nullptr;  // uses (null: one each), their durations (ms, T per item) and the loop count
    const int* src_ms = nullptr;
    int src_loops = 0;
    int k = 1;              // renditions (lp_xbatch_transform_frames: the file renditions, then the frame renditions)
    std::vector<Rendition> rend;
    std::vector<XItem> items;   // pairs: item i, rendition r at i * k + r
    std::vector<uint32_t> mask;  // per item: the renditions it takes on the grid
    std::vector<int> fallback;   // pairs
    std::mutex fb_mu;
};

static void push_fallback(lp_xbatch* X, int p) {
    std::lock_guard<std::mutex> g(X->fb_mu);
    X->fallback.push_back(p);
}

// every pair of a task: lp_transform decides
static void push_task_fallback(lp_xbatch* X, const Task& t) {
    std::lock_guard<std::mutex> g(X->fb_mu);
    for (size_t a = 0; a < t.idx.size(); a++)
        for (int r = 0; r < X->k; r++)
            if (t.rm[a] >> r & 1) X->fallback.push_back(t.idx[a] * X->k + r);
}

// the pair of item i that carries its source fields for a task: its first rendition there
static int first_pair(const lp_xbatch* X, int i, uint32_t rm) { return i * X->k + __builtin_ctz(rm); }

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

constexpr size_t kIccBufferBytes = 32768;  // ICCProfileBufferSize (ref lilliput.go:15)

// The profile WebpEncoder::Create hands to the WebP writer: what the decoder's ICC() read into its buffer (n <= 0:
// none), kept only when iccHeaderIsSane
static void keep_icc(XItem* it, const uint8_t* icc, long n) {
    if (n > 0 && lilliput::iccHeaderIsSane(icc, (size_t)n)) it->icc.assign(icc, icc + n);
}

// A multi-scan JPEG the serial decoder takes: its scans parse and stay within the work budget (otherwise per image)
static bool multiscan_in_budget(const uint8_t* d, size_t n, const JpegHeader& h) {
    std::vector<JpegScanDesc> scans(kMultiscanMaxScans);
    int nscans = 0, nsets = 0;
    return jpeg_parse_scans(d, n, h, scans.data(), (int)scans.size(), &nscans, (JpegHeader*)nullptr, kMultiscanMaxSets, &nsets) ==
               LP_OK &&
           jpeg_multiscan_visits(h, scans.data(), nscans) <= kMultiscanMaxVisits;
}

// A PNG the grid decodes: a colour (RGB / RGBA) frame of at most max_side, without an eXIf turn (Transform turns the frame
// before the resize, which the grid does not), its IDAT payloads one forward run of the file (they are in every valid PNG)
static std::shared_ptr<const PngHeader> png_grid_header(const uint8_t* d, size_t n, int max_side) {
    std::shared_ptr<PngHeader> h(new PngHeader);
    if (png_parse(d, n, h.get()) != LP_OK) return nullptr;
    if (h->orientation != 1 || h->idat.empty() || h->idat_total < 2) return nullptr;
    if (h->width > max_side || h->height > max_side) return nullptr;
    for (size_t q = 1; q < h->idat.size(); q++)
        if (h->idat[q].offset < h->idat[q - 1].offset + h->idat[q - 1].length) return nullptr;
    if (h->idat.back().offset + h->idat.back().length > n) return nullptr;
    if (h->out_channels != 3 && h->out_channels != 4) return nullptr;  // gray PNGs: per image
    return h;
}

// What an item's file is, parsed once for all its renditions when the first one needs it (-1: not parsed yet, 0: the
// grid cannot decode it, 1: it can)
struct ItemHeaders {
    int jpeg = -1;  // a baseline or multi-scan header
    JpegHeader jh;
    int jpeg_budget = -1;  // multi-scan: the scans parse and stay within the serial decoder's budget (walked lazily)
    int png = -1;
    std::shared_ptr<const PngHeader> ph;
    bool png_cicp = false;
    uint8_t cicp[4];  // primaries, transfer, matrix, full range: the chunk Transform's decoder reports
    int webp = -1;  // within max_side, and a still's frame is its canvas
    WebpPlan wp;
    int gif[2] = {-1, -1};  // the full plan, the first-frame plan
    std::shared_ptr<GifAnimPlan> gp[2];
};

// The slots of a clip of T frames over F (lp_xbatch_decode_clips' sampling rule): frame t while F <= T, otherwise frame
// floor(t * F / T); each slot's start sums the durations (ms, duration_ms(j) of frame j) of the frames before its own
template <class D>
static void select_clip(XItem* it, int F, int T, D duration_ms) {
    const int used = std::min(F, T);
    it->nframes = F;
    it->clip.resize((size_t)used);
    it->clip_ms.resize((size_t)used);
    int64_t ms = 0;
    for (int t = 0, j = 0; t < used; t++) {
        const int f = F <= T ? t : (int)((int64_t)t * F / T);
        for (; j < f; j++) ms += duration_ms(j);
        it->clip[t] = f;
        it->clip_ms[t] = ms;
    }
}

// A still written to WebP: Transform checks its deadline after the frame (a zero budget fails with ErrEncodeTimeout),
// MaxEncodeFrames == 1 asks the decoder to skip to the end and a negative MaxEncodeDuration is exceeded at once (no
// still decoder can skip: ErrSkipNotSupported).  The per-image path decides these after the frame.
static bool webp_decides_after_frame(const lp_image_options& o) {
    return o.encode_timeout_ns <= 0 || o.max_encode_frames == 1 || o.max_encode_duration_ns < 0;
}

// The gates below serve every sink.  S_FRAMES (lp_xbatch_decode_frames and _clips) is the frame Transform hands its still
// ".png" encoder, which answers at once: no deadline, frame limit or flush follows it, so only the decoders' gates apply.

// JPEG: to JPEG, lossy WebP and PNG, and into the tensor.  The file sinks take three-component upright files; the tensor
// also gray and rotated ones (the group's resize-only lp_batch context orients and decodes both).
static void jpeg_gates(XItem& it, const Rendition& R, const uint8_t* d, size_t n, int max_side, ItemHeaders* c) {
    const lp_image_options& opt = R.opt;
    const bool frames = R.sink == S_FRAMES;
    if (R.sink == S_GIF || (R.sink == S_WEBP && (R.lossless || webp_decides_after_frame(opt)))) return;
    if (c->jpeg < 0) c->jpeg = jpeg_parse_header(d, n, &c->jh) == LP_OK && (c->jh.supported || c->jh.multiscan);
    if (!c->jpeg) return;
    const JpegHeader& h = c->jh;
    const bool layout = frames ? h.ncomp == 3 || h.ncomp == 1 : h.ncomp == 3 && (h.orientation < 2 || h.orientation > 8);
    if (!layout || h.width > max_side || h.height > max_side) return;
    if (!h.supported) {  // multi-scan: damaged scans and files over the serial decoder's budget go per image
        if (c->jpeg_budget < 0) c->jpeg_budget = multiscan_in_budget(d, n, h);
        if (!c->jpeg_budget) return;
    }
    it.jpeg_multiscan = !h.supported;
    it.w = h.width;
    it.h = h.height;
    it.ch = h.ncomp;
    it.jpeg_sampling = 0;
    for (int q = 0; q < h.ncomp; q++) it.jpeg_sampling = (it.jpeg_sampling << 8) | (h.comp[q].h << 4) | h.comp[q].v;
    if (!plan_geometry(opt, &it)) return;
    // orientations 5..8: the requested size is the header's turned only under NormalizeOrientation, and Fit works on the
    // turned frame (ops.go:449-470, as lp_batch sizes its class 2)
    if (h.orientation >= 5 && h.orientation <= 8 && opt.resize_method == LP_OPS_FIT) {
        const bool turn = opt.normalize_orientation != 0;
        lilliput::calculateExpectedSize(turn ? h.height : h.width, turn ? h.width : h.height, opt.width, opt.height, &it.ow, &it.oh);
    }
    thread_local std::vector<uint8_t> icc_buf(kIccBufferBytes);
    if (R.sink == S_WEBP)  // (its APP2 segments concatenated: the item keeps its own copy)
        keep_icc(&it, icc_buf.data(), opencv_decoder_get_jpeg_icc(const_cast<uint8_t*>(d), n, icc_buf.data(), icc_buf.size()));
    it.kind = K_JPEG;
}

// PNG: a colour frame of 8 or 16 bits (png_grid_header), HDR tone-mapped.  An SDR cICP changes no pixel, but Transform
// re-attaches it to a PNG output (ops.go:306-332): per image.  GIF output needs a GIF source: per image
// (ErrGifEncoderNeedsDecoder).  To WebP, PNGs with a profile stay per image, where they went before they could carry it,
// when the WebP encoder decides after the frame; to lossless output every PNG follows that rule.
static void png_gates(XItem& it, const Rendition& R, const uint8_t* d, size_t n, int max_side, ItemHeaders* c) {
    if (c->png < 0) {
        c->ph = png_grid_header(d, n, max_side);
        c->png = c->ph != nullptr;
        if (c->png) c->png_cicp = png_extract_cicp(d, n, c->cicp);
    }
    if (!c->png) return;
    if (c->png_cicp) {
        it.hdr = c->cicp[1] == 16 || c->cicp[1] == 18;
        if (!it.hdr && R.sink == S_PNG) return;
        it.transfer = c->cicp[1];
        it.primaries = c->cicp[0];
    }
    const PngHeader& h = *c->ph;
    it.w = h.width;
    it.h = h.height;
    it.ch = h.out_channels;
    if (!plan_geometry(R.opt, &it)) return;
    thread_local std::vector<uint8_t> icc_buf(kIccBufferBytes);
    const int icc_n = R.sink == S_WEBP ? png_extract_icc(d, n, icc_buf.data(), icc_buf.size()) : 0;
    if (R.sink == S_GIF || (R.sink == S_WEBP && (icc_n > 0 || R.lossless) && webp_decides_after_frame(R.opt))) return;
    if (R.sink == S_WEBP) keep_icc(&it, icc_buf.data(), icc_n);
    it.png = c->ph;
    it.kind = K_PNG;
}

// WebP: stills to lossy WebP, PNG and the tensor, animations to lossy WebP, cut to frame 0 under DisableAnimatedOutput
// and for the tensor, or after a clip's last selected frame.  Lossless output of WebP sources: per image.
static void webp_gates(XItem& it, const Rendition& R, const uint8_t* d, size_t n, int max_side, int T, ItemHeaders* c) {
    const lp_image_options& opt = R.opt;
    if (R.sink == S_GIF || R.lossless) return;
    if (c->webp < 0) {  // damaged containers: per image
        c->webp = webp_plan_parse(d, n, &c->wp) && c->wp.width <= max_side && c->wp.height <= max_side;
        // Transform does not composite a still: it resizes the decoded frame, which must then be the canvas
        if (c->webp && c->wp.frames.size() == 1) {
            const WebpFramePlan& f0 = c->wp.frames[0];
            if (f0.x || f0.y || f0.width != c->wp.width || f0.height != c->wp.height) c->webp = 0;
        }
    }
    if (!c->webp) return;
    std::unique_ptr<WebpPlan> p(new WebpPlan(c->wp));
    WebpFramePlan& f0 = p->frames[0];
    it.webp_animation = p->frames.size() > 1;
    if (!it.webp_animation) {
        // a still written to WebP with no time to encode: lp_transform's deadline check follows the frame.  Only the
        // simple lossy stills the grid has always taken keep going there; the others stay with lp_transform
        const bool simple = !f0.lossless && !f0.has_alph && !p->icc_len && !p->animated && p->channels == 3;
        if (R.sink == S_WEBP && opt.encode_timeout_ns <= 0 && !simple) return;
        // to PNG under MaxEncodeDuration: a WebP still's frame carries a duration, which Transform holds against the
        // limit before it encodes the frame; lp_transform decides
        if (R.sink == S_PNG && opt.max_encode_duration_ns != 0) return;
        f0.blend = 1;  // copied onto a canvas of its own size, never disposed
        f0.dispose = 0;
    } else if (R.sink == S_FRAMES) {
        if (T > 0) select_clip(&it, (int)p->frames.size(), T, [&](int j) { return (int64_t)p->frames[j].duration; });
        it.span = webp_plan_cut(p.get(), T > 0 ? it.clip.back() : 0);
    } else {
        // to animated WebP, with the option gates of GIF -> WebP; Transform checks its deadline after every non-final
        // frame, so a zero budget fails there (ErrEncodeTimeout): per image.  DisableAnimatedOutput: Transform encodes
        // frame 0 and flushes before its deadline check, so whatever the budget, the file is a still of the composited
        // frame 0 and the device reads only that frame
        if (R.sink != S_WEBP || opt.max_encode_frames != 0 || opt.max_encode_duration_ns != 0) return;
        if (opt.disable_animated_output) it.span = webp_plan_cut(p.get(), 0);
        else if (opt.encode_timeout_ns <= 0) return;
    }
    it.w = p->width;
    it.h = p->height;
    it.ch = p->channels;
    if (!plan_geometry(opt, &it)) return;
    // (webp_decoder_get_icc reads no profile larger than the buffer)
    if (R.sink == S_WEBP && p->icc_len <= kIccBufferBytes) keep_icc(&it, d + p->icc_off, (long)p->icc_len);
    it.webp = std::move(p);
    it.kind = K_WEBP;
}

// GIF: to GIF and WebP, and into the tensor.  DisableAnimatedOutput and the tensor take the first-frame plan: Transform
// encodes frame 0 and flushes before its deadline check, and its decoder reads nothing behind that frame.  A clip takes
// the full plan, whose frame count must be the one GifDecoder's header walk gives (so both routes agree on F), cut after
// the last selected frame: nothing behind it is uploaded or decoded.
static void gif_gates(XItem& it, const Rendition& R, const uint8_t* d, size_t n, int max_side, int T, ItemHeaders* c) {
    const lp_image_options& opt = R.opt;
    const bool frames = R.sink == S_FRAMES;
    const bool first_only = frames ? T == 0 : opt.disable_animated_output != 0;
    if (!frames) {
        if ((R.sink != S_WEBP && R.sink != S_GIF) || opt.max_encode_frames != 0 || opt.max_encode_duration_ns != 0) return;
        // a GIF written with no time to encode fails with ErrEncodeTimeout after its first frame (Transform's deadline):
        // per image, to GIF and to lossless WebP
        if (!first_only && (R.sink == S_GIF || R.lossless) && opt.encode_timeout_ns <= 0) return;
    }
    if (c->gif[first_only] < 0) {
        c->gp[first_only].reset(gif_plan_parse(d, n, 4096, first_only), gif_plan_free);
        c->gif[first_only] = c->gp[first_only] != nullptr;
    }
    if (!c->gif[first_only]) return;
    std::shared_ptr<GifAnimPlan> p = c->gp[first_only];
    int w = 0, h = 0, nf = 0;
    gif_plan_info(p.get(), &w, &h, &nf, nullptr, nullptr);
    if (T > 0) {
        if (nf != gif_header_frames(d, n)) return;
        select_clip(&it, nf, T, [&](int j) { return (int64_t)gif_plan_delay_ms(p.get(), j); });
        nf = it.clip.back() + 1;
        gif_plan_cut(p.get(), nf - 1);
        c->gp[0].reset();  // (the cut plan is this pair's alone: another rendition would parse the file again)
        c->gif[0] = -1;
    }
    it.w = w;
    it.h = h;
    it.ch = 4;
    it.span = gif_plan_file_bytes(p.get());
    // a one-frame file to WebP meets the same deadline check after its frame: with no time to encode, per image
    if ((nf < 2 && R.sink == S_WEBP && !first_only && opt.encode_timeout_ns <= 0) || w > max_side || h > max_side ||
        !plan_geometry(opt, &it))
        return;
    it.gif = std::move(p);
    it.gif_frames = nf;
    it.kind = K_GIF;
}

// A tensor item of lp_xbatch_encode_frames: its "header" is w x h x C, with no container, so no ICC profile and no cICP,
// and it takes the gates of an 8-bit RGB / RGBA PNG (png_grid_header's size limit, png_gates) with three differences.
// Two send items per image where lp_transform fails them and the PNG gates keep an ICC-less PNG on the grid, as they
// always have:
//   - the option gates are those of a PNG with a profile: Transform checks a still's deadline and MaxEncodeFrames after
//     its frame goes to the .webp encoder (which waits for the end of the stream), and fails with ErrEncodeTimeout or
//     ErrSkipNotSupported;
//   - a negative MaxEncodeDuration, whatever the sink: Transform asks the decoder to skip to the end before the encode,
//     which it refuses (ErrSkipNotSupported).
// The third is NoResize: Transform hands a still's frame straight to the encoder, so the item takes the grid and its
// unpacked frame goes to the sink unresized.  A size outside the box stays per image, which refuses it.
//
// A clip item of lp_xbatch_encode_clips with nframes >= 2 takes the gates of what Transform does with A_i, its animated
// WebP of full-canvas, no-blend, no-dispose frames (clip_gates); one of a single frame is the tensor item above.
static bool frame_args_ok(const lp_xbatch* X, int i) {
    const int w = X->src_w[i], h = X->src_h[i];
    if (w < 1 || h < 1 || w > X->frames.width || h > X->frames.height) return false;
    if (!X->src_nframes) return true;
    const int nf = X->src_nframes[i];
    if (nf < 1 || nf > X->src_t) return false;
    for (int t = 0; nf > 1 && t < nf; t++) {  // (ANMF holds 24 bits of duration)
        const int ms = X->src_ms[(size_t)i * X->src_t + t];
        if (ms < 0 || ms > 0xFFFFFF) return false;
    }
    return true;
}

// The clip gates (nframes >= 2).  Transform decodes A_i's frames in order; each one covers the canvas without blending,
// so the composite it fits is the frame itself, and Transform fits an animation even under NoResize, to its own size
// (a copy: the resize of an unchanged size copies).  What the item's output reads, and when Transform decides after a
// frame in ways the per-image route reports:
//   - .webp: every frame goes to the encoder, which writes each with its duration, A_i's background and loop count.
//     Transform checks its deadline after every non-final frame, so a zero EncodeTimeout fails there
//     (ErrEncodeTimeout): per image.  DisableAnimatedOutput: Transform encodes frame 0 and flushes before that check,
//     so the file is a still of frame 0 and only frame 0 is read, whatever the budget.  A non-zero MaxEncodeFrames
//     makes Transform ask the decoder to skip to the end, which it cannot (ErrSkipNotSupported), unless the stream
//     ends first: per image.
//   - .jpeg and .png: the still encoder answers on frame 0, so only frame 0 is read; no deadline, frame limit or
//     DisableAnimatedOutput is consulted.
//   - any file sink: a non-zero MaxEncodeDuration is held against the frames' durations before each encode, and
//     exceeding it ends in a skip to the end: per image.
//   - .gif: per image (ErrGifEncoderNeedsDecoder).
static bool clip_gates(XItem& it, const Rendition& R, int nf) {
    const lp_image_options& opt = R.opt;
    if (R.sink == S_GIF || opt.max_encode_duration_ns != 0) return false;
    if (R.sink != S_WEBP) {
        it.src_frames = 1;
        return true;
    }
    if (opt.max_encode_frames != 0) return false;
    if (opt.disable_animated_output) {
        it.src_frames = 1;
        return true;
    }
    if (opt.encode_timeout_ns <= 0) return false;
    it.src_frames = nf;
    return true;
}

static void parse_frame_pair(const lp_xbatch* X, int i, XItem& it, const Rendition& R, int max_side) {
    const int w = X->src_w[i], h = X->src_h[i];
    if (!frame_args_ok(X, i) || w > max_side || h > max_side) return;
    const int nf = X->src_nframes ? X->src_nframes[i] : 1;
    if (nf > 1) {
        if (!clip_gates(it, R, nf)) return;
    } else if (R.opt.max_encode_duration_ns < 0 || R.sink == S_GIF || (R.sink == S_WEBP && webp_decides_after_frame(R.opt))) {
        return;
    }
    it.w = w;
    it.h = h;
    it.ch = X->frames.channels;
    if (R.opt.resize_method == LP_OPS_NO_RESIZE) {
        it.ow = it.cw = w;
        it.oh = it.chh = h;
        it.cx = it.cy = 0;
    } else if (!plan_geometry(R.opt, &it)) {
        return;
    }
    it.kind = K_FRAME;
}

// the gates of pair (i, r): it takes the grid when they pass; anything else goes to lp_transform(in[i], opts[r])
static void parse_pair(lp_xbatch* X, int i, int r, ItemHeaders* c) {
    XItem& it = X->items[(size_t)i * X->k + r];
    const Rendition& R = X->rend[r];
    const lp_image_options& opt = R.opt;
    it.kind = K_FALLBACK;
    it.icc.clear();
    const int max_side = X->cfg.max_size > 0 ? X->cfg.max_size : 8192;
    // To PNG every still is one frame in, the file out of the first Encode call: MaxEncodeFrames, DisableAnimatedOutput
    // and the deadline are never consulted.  A negative MaxEncodeDuration is exceeded before the frame is encoded, and
    // Transform then asks the decoder to skip to the end, which no still decoder can (ErrSkipNotSupported): per image.
    if (R.sink == S_NONE || (R.sink == S_PNG && opt.max_encode_duration_ns < 0)) return;
    if (X->src_w) {
        parse_frame_pair(X, i, it, R, max_side);
        return;
    }
    const uint8_t* d = X->in[i];
    const size_t n = X->in_len[i];
    const int T = X->clip_t;
    it.span = n;
    if (!d || n < 16) return;
    // into the tensor, MaxEncodeDuration is held against a frame's duration before the encode; a clip ignores it
    if (R.sink == S_FRAMES && T == 0 && opt.max_encode_duration_ns != 0) return;
    static const uint8_t png_sig[8] = {0x89, 0x50, 0x4E, 0x47, 0x0D, 0x0A, 0x1A, 0x0A};
    if (d[0] == 0xFF && d[1] == 0xD8) jpeg_gates(it, R, d, n, max_side, c);
    else if (!memcmp(d, png_sig, 8)) png_gates(it, R, d, n, max_side, c);
    else if (!memcmp(d, "RIFF", 4) && !memcmp(d + 8, "WEBP", 4)) webp_gates(it, R, d, n, max_side, T, c);
    else if (!memcmp(d, "GIF8", 4)) gif_gates(it, R, d, n, max_side, T, c);
    if (R.sink == S_FRAMES && T > 0 && it.kind != K_FALLBACK && it.clip.empty())  // a still: one slot
        select_clip(&it, 1, T, [](int) { return (int64_t)0; });
}

// every rendition of item i; the pairs that take the grid set their bits in X->mask[i]
static void parse_item(lp_xbatch* X, int i) {
    ItemHeaders c;
    uint32_t m = 0;
    for (int r = 0; r < X->k; r++) {
        parse_pair(X, i, r, &c);
        XItem& it = X->items[(size_t)i * X->k + r];
        if (it.kind != K_FALLBACK) m |= 1u << r;
        if (it.kind == K_JPEG) it.jpeg_frames_only = c.jh.ncomp == 1 || (c.jh.orientation >= 2 && c.jh.orientation <= 8);
    }
    X->mask[i] = m;
}

// ------------------------------------------------------------------ runs
// A task holds items of ONE decoder kind, ordered so that equal geometries are adjacent (a PNG or WebP task: any
// geometry; a GIF or JPEG task: one).  The entropy stage is one launch over the whole task, one decode per item whatever
// its renditions; the geometry-bound stages (resize, encode) are one launch per rendition and run of equal geometry.

struct Run {
    int k0, k1;  // task positions
};

// The runs of rendition r among task positions [k0, k1): maximal stretches of positions that take r, with one decoded
// geometry (and so one output geometry), each decoded with status LP_OK when `decoded` is given, at most `cap` long.  A
// position that does not take r ends a run, so the frames of a buffer laid out by task position (decoded frames or
// canvases, a JPEG group's resized frames) lie back to back over it.  span_holes: such a position is skipped instead,
// for a rendition's output area, which holds the frames of the positions that take it and no others.
static std::vector<Run> task_runs(const lp_xbatch* X, const Task& t, int r, int k0, int k1, bool span_holes,
                                  const int* decoded = nullptr, int cap = INT_MAX) {
    auto takes = [&](int k) { return (t.rm[k] >> r & 1) && (!decoded || decoded[k] == LP_OK); };
    std::vector<Run> out;
    for (int k = k0; k < k1;) {
        if (!takes(k)) {
            k++;
            continue;
        }
        const XItem& a = X->items[(size_t)t.idx[k] * X->k + r];
        int end = k + 1;
        for (int e = k + 1, m = 1; e < k1 && m < cap; e++) {
            if (!takes(e)) {
                if (span_holes) continue;
                break;
            }
            const XItem& c = X->items[(size_t)t.idx[e] * X->k + r];
            if (c.w != a.w || c.h != a.h || c.ch != a.ch) break;
            end = e + 1;
            m++;
        }
        out.push_back(Run{k, end});
        k = end;
    }
    return out;
}

// one resize launch over nf frames of pair g's geometry, back to back at src and at dst
static bool resize_run(Lane& L, const XItem& g, const uint8_t* src, uint8_t* dst, int nf) {
    const size_t fs = round_up((size_t)g.w * g.h * g.ch, (size_t)256), os = round_up((size_t)g.ow * g.oh * g.ch, (size_t)256);
    ResizeArgs a{src, fs, (size_t)g.w * g.ch, g.ch, g.cx, g.cy, g.cw, g.chh, dst, os, (size_t)g.ow * g.ch, g.ow, g.oh, nf, 3};
    return resize_launch(a, L.st) == LP_OK;
}

// ------------------------------------------------------------------ sinks

// The PNG sink's file slot for a frame of ow x oh x ch: the largest file it can become, capped by the callers' buffers
// (a longer file is lp_transform's to refuse).
static size_t png_sink_slot(const lp_xbatch* X, int ow, int oh, int ch) {
    return round_up(std::min(X->out_cap, png_encode_max_file_bytes(ow, oh, ch)), (size_t)256);
}
// Device bytes the PNG sink takes from a lane's arena per frame: encoder scratch, the slot, its place in the packed copy.
static size_t png_sink_item_bytes(const lp_xbatch* X, const Rendition& R, int ow, int oh, int ch) {
    return round_up(png_encode_batch_scratch_bytes(ow, oh, ch, 1, R.png_level), (size_t)256) + 2 * png_sink_slot(X, ow, oh, ch) + 64;
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

// the staged files into the callers' buffers; one that did not fit its slot or the caller's buffer, or whose decode
// failed (st), lets Transform decide
static void deliver_staged(lp_xbatch* X, const uint8_t* h_stage, const int* idx, const int* st, int n,
                           const std::vector<unsigned long long>& off, const std::vector<uint32_t>& len, size_t slot,
                           std::vector<int>* failed) {
    for (int k = 0; k < n; k++) {
        const int i = idx[k];
        if (st[k] != LP_OK || len[k] == 0 || len[k] > slot || len[k] > X->out_cap) {
            failed->push_back(i);
            continue;
        }
        memcpy(X->out[i], h_stage + off[k], len[k]);
        X->out_len[i] = len[k];
        X->status[i] = LP_OK;
    }
}

// JPEG and PNG (stills): every frame of the run encoded into a device slot of its own, the files packed and copied home
// through the pinned staging area.  A run whose slots and scratch do not fit what is left of the arena, or whose files
// may not fit the staging area, is encoded in parts.  jpeg_cap: the largest JPEG file taken from the grid (0: the
// callers' buffer size).
static void slot_sink(lp_xbatch* X, const Rendition& R, Lane& L, Bump& bump, uint8_t* h_stage, size_t h_stage_bytes,
                      const std::vector<int>& pairs, const std::vector<int>& st, const uint8_t* d_frames, size_t stride,
                      size_t jpeg_cap, std::vector<int>* failed) {
    const XItem& g = X->items[pairs[0]];
    const int n = (int)pairs.size(), ow = g.ow, oh = g.oh, ch = g.ch;
    const bool png = R.sink == S_PNG;
    const size_t slot = png ? png_sink_slot(X, ow, oh, ch)
                            : round_up(std::min(jpeg_cap ? jpeg_cap : X->out_cap, std::max((size_t)65536, (size_t)ow * oh * ch)), (size_t)256);
    auto scratch_bytes = [&](int m) {
        return png ? png_encode_batch_scratch_bytes(ow, oh, ch, m, R.png_level) : jpeg_encode_scratch_bytes(ow, oh, ch, m, slot, R.progressive);
    };
    const size_t per = round_up(scratch_bytes(1), (size_t)256) + 2 * slot + 64;  // (for PNG: png_sink_item_bytes)
    const size_t mark = bump.used, room = bump.cap - bump.used;
    const size_t fixed = 4096;  // lengths, offsets and the arena's alignment
    const int part = (int)std::min<size_t>((size_t)n, std::min(room > fixed ? (room - fixed) / (per + 16) : 0, h_stage_bytes / (slot + 16)));
    if (part < 1) {
        failed->insert(failed->end(), pairs.begin(), pairs.end());
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
        void* scratch = bump.take<uint8_t>(scratch_bytes(m));
        const uint8_t* frames = d_frames + (size_t)k0 * stride;
        int rc = d_out && d_len && d_packed && d_off && scratch ? LP_OK : LP_ERR_BUF_TOO_SMALL;
        if (!rc && png) {
            rc = png_encode_batch(frames, stride, (size_t)ow * ch, ow, oh, ch, m, R.png_level, R.png_adaptive, d_out, slot, d_len, scratch, L.st);
        } else if (!rc) {
            JpegEncodeBatch e;
            e.frames = frames;
            e.frame_img_stride = stride;
            e.frame_row_stride = (size_t)ow * ch;
            e.width = ow;
            e.height = oh;
            e.channels = ch;
            e.quality = R.quality;
            e.n = m;
            e.out = d_out;
            e.out_cap = slot;
            e.out_len = d_len;
            e.scratch = scratch;
            e.progressive = R.progressive;
            rc = jpeg_encode_launch(e, L.st, nullptr);
        }
        if (!rc) rc = slots_to_host(L, h_stage, h_stage_bytes, d_out, slot, d_len, m, d_packed, d_off, &off, &len);
        if (rc) {
            cudaGetLastError();
            failed->insert(failed->end(), pairs.begin() + k0, pairs.end());
            break;
        }
        deliver_staged(X, h_stage, pairs.data() + k0, st.data() + k0, m, off, len, slot, failed);
    }
    bump.used = mark;
}

// The WebP sink's encoder: n resized frames of one geometry (rows packed, `stride` apart) -> lossy VP8 or, when the
// options ask for lossless output, VP8L payloads
static int webp_encode_frames(const Rendition& R, const uint8_t* d_frames, size_t stride, int ow, int oh, int ch, int n,
                              std::vector<WebpEncodedFrame>* frames, cudaStream_t st) {
    if (R.lossless) return webp_encode_lossless_batch(d_frames, stride, (size_t)ow * ch, ow, oh, ch, n, frames, st);
    return webp_encode_lossy_batch(d_frames, stride, (size_t)ow * ch, ow, oh, ch, n, R.quality, frames, st);
}

// The largest JPEG file of ow x oh the lp_batch pipeline delivers from the grid: its slot, the callers' buffer size capped
// by the geometry's worst case, in whole 256-byte units; a longer file is lp_transform's
static size_t jpeg_batch_cap(const lp_xbatch* X, int ow, int oh) {
    size_t cap = std::min(X->out_cap, round_up(std::max((size_t)65536, (size_t)ow * oh * 3), (size_t)256));
    if (cap >= 256) cap = cap / 256 * 256;
    return cap;
}

// resized frames of a pair: every frame of an animation (of its plan, which DisableAnimatedOutput cuts to frame 0), one
// of a still; of a clip, its slots in use; of a tensor item, the frames its output reads
static int out_frames(const XItem& it) {
    if (!it.clip.empty()) return (int)it.clip.size();
    if (it.kind == K_GIF) return it.gif_frames;
    if (it.kind == K_FRAME) return it.src_frames;
    return it.kind == K_WEBP ? (int)it.webp->frames.size() : 1;
}

// WebP (stills and animations): one encode of every frame of the run, then each pair's file around its frames with the
// metadata WebpEncoder takes from the decoder: the ICC profile the pair kept and, from a WebP or GIF source or a tensor
// clip (A_i: background 0xFFFFFFFF, the call's loop count, the caller's durations), background, loop count and frame
// durations (webp_assemble writes none of these three into a one-frame file).  Every frame is written full-canvas with
// no blending and no disposal, as the per-image encoder writes whatever blend and dispose it receives.
static void webp_sink(lp_xbatch* X, const Rendition& R, Lane& L, const std::vector<int>& pairs, const std::vector<int>& st,
                      const uint8_t* d_frames, size_t stride, std::vector<int>* failed) {
    const XItem& g = X->items[pairs[0]];
    std::vector<int> first(pairs.size() + 1, 0);
    for (size_t q = 0; q < pairs.size(); q++) first[q + 1] = first[q] + out_frames(X->items[pairs[q]]);
    std::vector<WebpEncodedFrame> frames;
    if (webp_encode_frames(R, d_frames, stride, g.ow, g.oh, g.ch, first.back(), &frames, L.st)) {
        cudaGetLastError();
        failed->insert(failed->end(), pairs.begin(), pairs.end());
        return;
    }
    std::vector<uint8_t> file;
    for (size_t q = 0; q < pairs.size(); q++) {
        const int i = pairs[q], nf = first[q + 1] - first[q];
        const XItem& it = X->items[i];
        WebpEncodedFrame* f = &frames[first[q]];
        bool good = st[q] == LP_OK;
        for (int j = 0; j < nf && good; j++) good = !f[j].image.empty();
        if (!good) {  // a damaged stream or an encoder refusal: the per-image path reports the precise error
            failed->push_back(i);
            continue;
        }
        uint32_t bg = 0xFFFFFFFFu, loops = 0;
        if (it.kind == K_WEBP) {
            bg = it.webp->bgcolor;
            loops = it.webp->loop_count;
        } else if (it.kind == K_GIF) {
            int n = 0;
            gif_plan_info(it.gif.get(), nullptr, nullptr, nullptr, &bg, &n);
            loops = (uint32_t)n;
        } else if (it.kind == K_FRAME && nf > 1) {
            loops = (uint32_t)X->src_loops;
        }
        for (int j = 0; j < nf; j++) {
            if (it.kind == K_WEBP) f[j].duration = it.webp->frames[j].duration;
            if (it.kind == K_GIF) f[j].duration = gif_plan_delay_ms(it.gif.get(), j);
            if (it.kind == K_FRAME && nf > 1) f[j].duration = X->src_ms[(size_t)(i / X->k) * X->src_t + j];
            L.d2h += f[j].image.size() + f[j].alph.size();
        }
        webp_assemble(f, nf, it.icc.data(), it.icc.size(), bg, loops, &file);
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

// GIF (from GIF sources): palette mapping + LZW of every resized frame of the run in one set of launches, the code
// streams packed and copied home at once, each file assembled on the host from the plan's container metadata
static void gif_sink(lp_xbatch* X, Lane& L, Bump& bump, const std::vector<int>& pairs, const std::vector<int>& st,
                     const uint8_t* d_frames, size_t stride, std::vector<int>* failed) {
    const int na = (int)pairs.size();
    const XItem& g = X->items[pairs[0]];
    std::vector<GifAnimPlan*> plans((size_t)na);
    std::vector<int> first((size_t)na + 1, 0);
    std::vector<uint8_t*> out((size_t)na);
    size_t bytes = 0;
    for (int a = 0; a < na; a++) {
        const XItem& it = X->items[pairs[a]];
        plans[a] = it.gif.get();
        first[a + 1] = first[a] + it.gif_frames;
        out[a] = X->out[pairs[a]];
        bytes += gif_plan_encode_bytes(plans[a], g.ow, g.oh);
    }
    uint8_t* d_scratch = bump.take<uint8_t>(bytes);
    std::vector<size_t> olen((size_t)na, 0);
    std::vector<int> ost((size_t)na, LP_OK);
    const int rc = d_scratch ? gif_encode_batch(plans.data(), na, d_frames, stride, g.ow, g.oh, first.data(), d_scratch, bytes, L.host,
                                                L.host_bytes, out.data(), X->out_cap, olen.data(), ost.data(), &L.d2h, L.st)
                             : LP_ERR_BUF_TOO_SMALL;
    if (rc) cudaGetLastError();
    for (int a = 0; a < na; a++) {
        const int i = pairs[a];
        if (rc || st[a] != LP_OK) {  // a corrupt code stream: the per-image path reports the precise error
            failed->push_back(i);
            continue;
        }
        X->status[i] = ost[a];
        X->out_len[i] = olen[a];
    }
}

static FramePackLayout frames_layout(const lp_frame_tensor& t) {
    FramePackLayout o;
    o.data = t.data;
    o.H = t.height;
    o.W = t.width;
    o.C = t.channels;
    o.nchw = t.nchw != 0;
    o.rgb = t.rgb != 0;
    o.dtype = t.dtype;
    for (int c = 0; c < 4; c++) {
        o.scale[c] = t.scale[c];
        o.bias[c] = t.bias[c];
    }
    return o;
}

// A frame rendition (lp_xbatch_transform_frames, _decode_frames, _decode_clips): every frame of the run into its slot's
// slice of the rendition's tensor in one launch.  Item i has `slots` slices from i * slots (one, or T for a clip); slot t
// holds its t-th resized frame, and a slot past its frames is an entry of 0 x 0, which the kernel writes as zeros.  The
// table travels to the device, so items that are not neighbours in the batch land in their own slices, each with its own
// frame size (a JPEG group's turned or gray items).  A frame larger than the box is refused; a pair whose decode failed
// goes to the per-image path.  Nothing comes back to the host.
static void frames_sink(lp_xbatch* X, const Rendition& R, Lane& L, Bump& bump, const std::vector<int>& pairs, const std::vector<int>& st,
                        const uint8_t* d_frames, size_t stride, std::vector<int>* failed) {
    const lp_frame_tensor& T = R.dst;
    const int slots = std::max(1, X->clip_t);
    std::vector<FramePackItem> tab;
    std::vector<int> packed;  // pairs
    size_t at = 0;  // the pair's first frame in the run
    for (size_t q = 0; q < pairs.size(); q++) {
        const int p = pairs[q], i = p / X->k;
        const XItem& it = X->items[p];
        const int nf = out_frames(it);
        if (st[q] != LP_OK) {
            failed->push_back(p);
        } else if (it.ow > T.width || it.oh > T.height) {
            X->status[p] = LP_ERR_BUF_TOO_SMALL;
        } else {
            for (int t = 0; t < slots; t++) {
                const int64_t slice = (int64_t)i * slots + t;
                tab.push_back(t < nf ? FramePackItem{d_frames + (at + t) * stride, (uint32_t)(it.ow * it.ch), it.ow, it.oh, it.ch, slice}
                                     : FramePackItem{nullptr, 0, 0, 0, it.ch, slice});
            }
            packed.push_back(p);
        }
        at += nf;
    }
    if (tab.empty()) return;
    const size_t mark = bump.used;
    FramePackItem* d_tab = bump.take<FramePackItem>(tab.size() * sizeof(FramePackItem));
    int rc = d_tab ? LP_OK : LP_ERR_BUF_TOO_SMALL;
    if (!rc && cudaMemcpyAsync(d_tab, tab.data(), tab.size() * sizeof(FramePackItem), cudaMemcpyHostToDevice, L.st) != cudaSuccess)
        rc = LP_ERR_CUDA;
    if (!rc) rc = frames_pack_launch(d_tab, nullptr, (int)tab.size(), frames_layout(T), L.st);
    if (!rc && cudaStreamSynchronize(L.st) != cudaSuccess) rc = LP_ERR_CUDA;
    bump.used = mark;
    if (rc) {
        cudaGetLastError();
        failed->insert(failed->end(), packed.begin(), packed.end());
        return;
    }
    L.h2d += tab.size() * sizeof(FramePackItem);
    for (int p : packed) {
        const XItem& it = X->items[p];
        const int i = p / X->k;
        X->status[p] = LP_OK;
        R.frame_w[i] = it.ow;
        R.frame_h[i] = it.oh;
        if (!X->clip_t) continue;  // (a clip: the call's one rendition)
        X->clip_nframes[i] = it.nframes;
        for (size_t t = 0; t < it.clip.size(); t++) {
            X->clip_index[(size_t)i * slots + t] = it.clip[t];
            X->clip_ms[(size_t)i * slots + t] = it.clip_ms[t];
        }
    }
}

static void lane_time(Lane& L, int from, int to, double* acc) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, L.ev[from], L.ev[to]) == cudaSuccess) *acc += ms;
}

// A run of rendition r through its sink into the callers' buffers: the pairs of the task positions in [u.k0, u.k1)
// that take r, whose resized frames lie back to back `stride` apart from d_frames (one per still, every frame of an
// animation).  st (nullptr: all LP_OK): the decode status by task position; a pair whose decode failed is encoded with
// its run and then handed to lp_transform, as is a pair its sink could not write (failed).
static void sink_encode(lp_xbatch* X, Lane& L, Bump& bump, uint8_t* h_stage, size_t h_stage_bytes, const Task& t, int r,
                        Run u, const int* st, const uint8_t* d_frames, size_t stride, std::vector<int>* failed,
                        size_t jpeg_cap = 0) {
    const Rendition& R = X->rend[r];
    std::vector<int> pairs, pst;
    for (int k = u.k0; k < u.k1; k++)
        if (t.rm[k] >> r & 1) {
            pairs.push_back(t.idx[k] * X->k + r);
            pst.push_back(st ? st[k] : LP_OK);
        }
    cudaEventRecord(L.ev[2], L.st);
    if (R.sink == S_WEBP) webp_sink(X, R, L, pairs, pst, d_frames, stride, failed);
    else if (R.sink == S_GIF) gif_sink(X, L, bump, pairs, pst, d_frames, stride, failed);
    else if (R.sink == S_FRAMES) frames_sink(X, R, L, bump, pairs, pst, d_frames, stride, failed);
    else slot_sink(X, R, L, bump, h_stage, h_stage_bytes, pairs, pst, d_frames, stride, jpeg_cap, failed);
    cudaEventRecord(L.ev[3], L.st);
    cudaEventSynchronize(L.ev[3]);
    lane_time(L, 2, 3, &L.ms_encode);
}

// ------------------------------------------------------------------ PNG / WebP tasks

// PNG task.  Inflate wants every stream in flight at once and needs only the compressed stream and the scanlines
// (~1.5 x the pixel bytes); the packed frames are needed only between defilter and resize.  So: ONE inflate launch over
// the whole task, then defilter -> resize into every rendition over windows of frames that reuse one buffer, then the
// sinks over the task, one rendition after another.
static void run_png(lp_xbatch* X, Lane& L, const Task& t) {
    const std::vector<int>& idx = t.idx;
    const int n = (int)idx.size(), K = X->k;
    std::vector<int> failed;
    Bump bump{L.dev, L.dev_bytes};
    std::vector<PngDecodeItem> items((size_t)n);
    std::vector<SegCopy> segs;
    std::vector<int> rep((size_t)n);  // the pair carrying each item's source fields
    std::vector<uint64_t> file_off((size_t)n), frame_off((size_t)n), out_off((size_t)n * K);  // out_off[k * K + r]
    std::vector<int> win_first;  // first item of every frame window
    size_t in_bytes = 0, raw_bytes = 0, out_bytes = 0, win_bytes = 0, win_max = 0;
    const size_t kWindow = std::min<size_t>((size_t)12 << 30, L.dev_bytes / 5);  // frames buffer
    int max_w = 0, max_h = 0;
    for (int k = 0; k < n; k++) {
        rep[k] = first_pair(X, idx[k], t.rm[k]);
        const PngHeader& ph = *X->items[rep[k]].png;
        const size_t span = ph.idat.back().offset + ph.idat.back().length - ph.idat.front().offset;
        file_off[k] = in_bytes;
        in_bytes += round_up(span + 16, (size_t)16);
    }
    size_t zg = in_bytes;  // gathered streams follow the uploaded file spans
    for (int k = 0; k < n; k++) {
        const XItem& xi = X->items[rep[k]];
        const PngHeader& ph = *xi.png;
        PngDecodeItem& it = items[k];
        png_decode_item(ph, (uint32_t)((size_t)xi.w * xi.ch), &it);
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
        max_w = std::max(max_w, xi.w);
        max_h = std::max(max_h, xi.h);
    }
    win_first.push_back(n);
    for (int r = 0; r < K; r++)  // every rendition's resized frames, one area after another
        for (int k = 0; k < n; k++)
            if (t.rm[k] >> r & 1) {
                const XItem& o = X->items[(size_t)idx[k] * K + r];
                out_off[(size_t)k * K + r] = out_bytes;
                out_bytes += round_up((size_t)o.ow * o.oh * o.ch, (size_t)256);
            }
    // HDR frames are tone-mapped between the defilter and the resize of their window, whole (before the Fit crop, as
    // Transform does); one scratch area sized for the window that needs the most
    std::vector<TmFrame> hdr;
    auto window_hdr = [&](int k0, int k1, uint8_t* frames) {
        hdr.clear();
        for (int k = k0; k < k1; k++) {
            const XItem& xi = X->items[rep[k]];
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
        push_task_fallback(X, t);
        return;
    }
    bool ok = true;
    for (int k = 0; k < n && ok; k++) {
        const PngHeader& ph = *X->items[rep[k]].png;
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
        for (int r = 0; r < K; r++)  // the window's frames into every rendition before the next window reuses them
            for (const Run& u : task_runs(X, t, r, k0, k1, false))
                ok = ok && resize_run(L, X->items[(size_t)idx[u.k0] * K + r], d_frames + frame_off[u.k0], d_out + out_off[(size_t)u.k0 * K + r],
                                      u.k1 - u.k0);
    }
    cudaEventRecord(L.ev[1], L.st);
    if (ok) ok = cudaMemcpyAsync(items.data(), d_items, (size_t)n * sizeof(PngDecodeItem), cudaMemcpyDeviceToHost, L.st) == cudaSuccess;
    if (ok) ok = cudaStreamSynchronize(L.st) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        push_task_fallback(X, t);
        return;
    }
    lane_time(L, 0, 1, &L.ms_decode);  // (the tone map and resize launches sit between the defilter launches: counted as decode)
    for (int r = 0; r < K; r++)
        for (const Run& u : task_runs(X, t, r, 0, n, true)) {
            bool corrupt = false;
            for (int k = u.k0; k < u.k1; k++) corrupt = corrupt || ((t.rm[k] >> r & 1) && items[k].status != 0);
            if (corrupt) {  // rare: a corrupt stream in the run -- its pairs take the per-image path, which reports the precise error
                for (int k = u.k0; k < u.k1; k++)
                    if (t.rm[k] >> r & 1) failed.push_back(idx[k] * K + r);
                continue;
            }
            const XItem& g = X->items[(size_t)idx[u.k0] * K + r];
            sink_encode(X, L, bump, L.host, L.host_bytes, t, r, u, nullptr, d_out + out_off[(size_t)u.k0 * K + r],
                        round_up((size_t)g.ow * g.oh * g.ch, (size_t)256), &failed);
        }
    for (int p : failed) push_fallback(X, p);
}

// WebP task: stills and animations of any canvas size, every frame of every file.  Decode + composite is one set of
// launches over the task (webp_decode_batch: VP8 frames, VP8L / ALPH waves, the per-pixel compositor); a still is one
// frame copied onto its canvas.  Then, per rendition, one resize and one sink call per run of equal canvas geometry.
// An animation is in the task with one rendition.
static void run_webp(lp_xbatch* X, Lane& L, const Task& t) {
    const std::vector<int>& idx = t.idx;
    const int n = (int)idx.size(), K = X->k;
    Bump bump{L.dev, L.dev_bytes};
    std::vector<const WebpPlan*> plans((size_t)n);
    std::vector<const uint8_t*> files((size_t)n);
    std::vector<size_t> flen((size_t)n);
    std::vector<uint64_t> canvas_off((size_t)n), out_off((size_t)n * K);  // out_off[k * K + r]
    std::vector<int> first((size_t)n + 1, 0);  // canvases
    std::vector<int> canvas_of;  // a clip's frames: the canvas each is stored at (-1: none)
    size_t scratch = 4096, arena = 0, canvas_bytes = 0, out_bytes = 0;
    for (int k = 0; k < n; k++) {
        const XItem& it = X->items[first_pair(X, idx[k], t.rm[k])];
        plans[k] = it.webp.get();
        files[k] = X->in[idx[k]];
        flen[k] = it.span;
        scratch += webp_plan_device_bytes(*plans[k], flen[k]);
        arena += webp_plan_arena_bytes(*plans[k]);
        const int nf = out_frames(it);  // (canvases stored: every frame, or a clip's slots)
        first[k + 1] = first[k] + nf;
        canvas_off[k] = canvas_bytes;
        canvas_bytes += (size_t)nf * round_up((size_t)it.w * it.h * it.ch, (size_t)256);
        L.h2d += flen[k];
        if (!X->clip_t) continue;
        const size_t j0 = canvas_of.size();
        canvas_of.resize(j0 + plans[k]->frames.size(), -1);
        for (size_t t = 0; t < it.clip.size(); t++) canvas_of[j0 + it.clip[t]] = (int)t;
    }
    for (int r = 0; r < K; r++)  // every rendition's resized frames, one area after another
        for (int k = 0; k < n; k++)
            if (t.rm[k] >> r & 1) {
                const XItem& o = X->items[(size_t)idx[k] * K + r];
                out_off[(size_t)k * K + r] = out_bytes;
                out_bytes += (size_t)(first[k + 1] - first[k]) * round_up((size_t)o.ow * o.oh * o.ch, (size_t)256);
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
                               canvas_off.data(), st.data(), L.ev[0], L.st, canvas_of.empty() ? nullptr : canvas_of.data()) == LP_OK;
    cudaEventRecord(L.ev[1], L.st);
    for (int r = 0; r < K; r++)
        for (const Run& u : task_runs(X, t, r, 0, n, false))
            ok = ok && resize_run(L, X->items[(size_t)idx[u.k0] * K + r], d_canvases + canvas_off[u.k0], d_out + out_off[(size_t)u.k0 * K + r],
                                  first[u.k1] - first[u.k0]);
    cudaEventRecord(L.ev[2], L.st);
    if (ok) ok = cudaStreamSynchronize(L.st) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        push_task_fallback(X, t);
        return;
    }
    lane_time(L, 0, 1, &L.ms_decode);
    lane_time(L, 1, 2, &L.ms_resize);
    std::vector<int> failed;
    for (int r = 0; r < K; r++)
        for (const Run& u : task_runs(X, t, r, 0, n, true)) {
            const XItem& g = X->items[(size_t)idx[u.k0] * K + r];
            sink_encode(X, L, bump, L.host, L.host_bytes, t, r, u, st.data(), d_out + out_off[(size_t)u.k0 * K + r],
                        round_up((size_t)g.ow * g.oh * g.ch, (size_t)256), &failed);
        }
    for (int p : failed) push_fallback(X, p);
}

// Tensor task (lp_xbatch_encode_frames and _clips, one rendition): one unpack launch turns the slices every item's output
// reads (one, or a clip's frames to an animated .webp) into packed u8 frames, laid out as an animation's canvases: an
// item's frames back to back, items in task order (its "decode").  Then the path of the other kinds: per run of equal
// geometry one resize and the sink.  Under NoResize no resize runs and the sink reads the unpacked frames.  Only the item
// table crosses PCIe on the way in.
static void run_frame(lp_xbatch* X, Lane& L, const Task& t) {
    const std::vector<int>& idx = t.idx;
    const int n = (int)idx.size();
    const bool resize = X->rend[0].opt.resize_method != LP_OPS_NO_RESIZE;
    Bump bump{L.dev, L.dev_bytes};
    std::vector<uint64_t> frame_off((size_t)n), out_off((size_t)n);
    std::vector<int> first((size_t)n + 1, 0);  // frames
    size_t frame_bytes = 0, out_bytes = 0;
    uint64_t max_frame = 0;
    for (int k = 0; k < n; k++) {
        const XItem& it = X->items[idx[k]];
        const size_t fb = (size_t)it.w * it.h * it.ch;
        first[k + 1] = first[k] + it.src_frames;
        frame_off[k] = frame_bytes;
        frame_bytes += (size_t)it.src_frames * round_up(fb, (size_t)256);
        max_frame = std::max<uint64_t>(max_frame, fb);
        out_off[k] = out_bytes;
        out_bytes += (size_t)it.src_frames * round_up((size_t)it.ow * it.oh * it.ch, (size_t)256);
    }
    const int nf = first[n];
    FrameUnpackItem* d_tab = bump.take<FrameUnpackItem>((size_t)nf * sizeof(FrameUnpackItem));
    uint8_t* d_frames = bump.take<uint8_t>(frame_bytes + 256);
    uint8_t* d_out = resize ? bump.take<uint8_t>(out_bytes + 256) : d_frames;
    if (!d_tab || !d_frames || !d_out) {
        push_task_fallback(X, t);
        return;
    }
    if (!resize) out_off = frame_off;
    std::vector<FrameUnpackItem> tab((size_t)nf);
    for (int k = 0; k < n; k++) {
        const XItem& it = X->items[idx[k]];
        const size_t fs = round_up((size_t)it.w * it.h * it.ch, (size_t)256);
        for (int f = 0; f < it.src_frames; f++)
            tab[(size_t)first[k] + f] = FrameUnpackItem{d_frames + frame_off[k] + f * fs, it.w, it.h, (int64_t)idx[k] * X->src_t + f};
    }
    bool ok = cudaMemcpyAsync(d_tab, tab.data(), tab.size() * sizeof(FrameUnpackItem), cudaMemcpyHostToDevice, L.st) == cudaSuccess;
    L.h2d += tab.size() * sizeof(FrameUnpackItem);
    cudaEventRecord(L.ev[0], L.st);
    if (ok) ok = frames_unpack_launch(d_tab, nullptr, nf, max_frame, frames_layout(X->frames), L.st) == LP_OK;
    cudaEventRecord(L.ev[1], L.st);
    if (resize)
        for (const Run& u : task_runs(X, t, 0, 0, n, false))
            ok = ok && resize_run(L, X->items[idx[u.k0]], d_frames + frame_off[u.k0], d_out + out_off[u.k0], first[u.k1] - first[u.k0]);
    cudaEventRecord(L.ev[2], L.st);
    if (ok) ok = cudaStreamSynchronize(L.st) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        push_task_fallback(X, t);
        return;
    }
    lane_time(L, 0, 1, &L.ms_decode);
    lane_time(L, 1, 2, &L.ms_resize);
    std::vector<int> failed;
    for (const Run& u : task_runs(X, t, 0, 0, n, true)) {
        const XItem& g = X->items[idx[u.k0]];
        sink_encode(X, L, bump, L.host, L.host_bytes, t, 0, u, nullptr, d_out + out_off[u.k0], round_up((size_t)g.ow * g.oh * g.ch, (size_t)256),
                    &failed);
    }
    for (int p : failed) push_fallback(X, p);
}

// ------------------------------------------------------------------ GIF groups (animations -> animated WebP or GIF)

// a GIF task holds one rendition: its pairs go through the decode, resize and sink as in a call with those options
static void run_gif(lp_xbatch* X, Lane& L, const Task& t) {
    const int na = (int)t.idx.size(), r = __builtin_ctz(t.rm[0]);
    std::vector<int> idx((size_t)na);  // pairs
    for (int a = 0; a < na; a++) idx[a] = t.idx[a] * X->k + r;
    const XItem& g = X->items[idx[0]];
    Bump bump{L.dev, L.dev_bytes};
    const size_t canvas_stride = round_up((size_t)g.w * g.h * 4, (size_t)256);
    const size_t out_stride = round_up((size_t)g.ow * g.oh * 4, (size_t)256);
    std::vector<int> first((size_t)na + 1, 0), cfirst((size_t)na + 1, 0);  // frame jobs, canvases (a clip stores its slots)
    std::vector<int> canvas_of;  // a clip's frames: the canvas each is stored at (-1: none)
    size_t scratch_bytes = 0;
    std::vector<GifAnimPlan*> plans((size_t)na);
    std::vector<const uint8_t*> files((size_t)na);
    std::vector<size_t> flen((size_t)na);
    for (int a = 0; a < na; a++) {
        const XItem& it = X->items[idx[a]];
        first[a + 1] = first[a] + it.gif_frames;
        cfirst[a + 1] = cfirst[a] + out_frames(it);
        plans[a] = it.gif.get();
        files[a] = X->in[t.idx[a]];
        flen[a] = it.span;
        scratch_bytes += gif_plan_device_bytes(it.gif.get());
        L.h2d += flen[a];
        if (!X->clip_t) continue;
        canvas_of.resize((size_t)first[a + 1], -1);
        for (size_t s = 0; s < it.clip.size(); s++) canvas_of[(size_t)first[a] + it.clip[s]] = cfirst[a] + (int)s;
    }
    const int nf = cfirst[na];
    uint8_t* d_scratch = bump.take<uint8_t>(scratch_bytes + 4096);
    uint8_t* d_canvases = bump.take<uint8_t>((size_t)nf * canvas_stride + 256);
    uint8_t* d_resized = bump.take<uint8_t>((size_t)nf * out_stride + 256);
    std::vector<int> st((size_t)na, 0);
    bool ok = d_scratch && d_canvases && d_resized;
    cudaEventRecord(L.ev[0], L.st);
    if (ok)
        ok = gif_decode_batch(plans.data(), files.data(), flen.data(), na, d_scratch, scratch_bytes + 4096, d_canvases,
                              canvas_stride, first.data(), st.data(), L.st, canvas_of.empty() ? nullptr : canvas_of.data()) == LP_OK;
    cudaEventRecord(L.ev[1], L.st);
    const std::vector<Run> runs = task_runs(X, t, r, 0, na, false);
    for (const Run& u : runs)
        ok = ok && resize_run(L, X->items[idx[u.k0]], d_canvases + (size_t)cfirst[u.k0] * canvas_stride,
                              d_resized + (size_t)cfirst[u.k0] * out_stride, cfirst[u.k1] - cfirst[u.k0]);
    cudaEventRecord(L.ev[2], L.st);
    if (ok) ok = cudaStreamSynchronize(L.st) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        push_task_fallback(X, t);
        return;
    }
    lane_time(L, 0, 1, &L.ms_decode);
    lane_time(L, 1, 2, &L.ms_resize);
    std::vector<int> failed;
    for (const Run& u : runs)
        sink_encode(X, L, bump, L.host, L.host_bytes, t, r, u, st.data(), d_resized + (size_t)cfirst[u.k0] * out_stride, out_stride,
                    &failed);
    for (int p : failed) push_fallback(X, p);
}

// ------------------------------------------------------------------ JPEG groups (the lp_batch pipeline)

// Device bytes one WebP encode of a JPEG group's frames may allocate (webp_encode_lossy_batch's scratch lives outside the
// lane's arena): 1 GiB holds 717 frames of 256x256 (1.43 MiB each, webp_encode_lossy_scratch_bytes), and stays below
// what one encode of a PNG task of bench.py's config 3 takes (6.4 MiB per 512x512 RGBA frame, hundreds of frames).
static constexpr size_t kJpegWebpScratch = (size_t)1 << 30;
// Frames of a JPEG group the PNG and JPEG sinks are sure to have arena for in one part (run_jpeg keeps that much out of
// the decode chunks' reach)
static constexpr size_t kJpegPngFrames = 512;

// Arena the sink of rendition R takes from the lane for m frames of ow x oh of a JPEG group (the WebP sink: none)
static size_t jpeg_group_sink_bytes(const lp_xbatch* X, const Rendition& R, int ow, int oh, size_t m) {
    if (R.sink == S_PNG) return m * png_sink_item_bytes(X, R, ow, oh, 3);
    if (R.sink != S_JPEG) return 0;
    const size_t slot = round_up(jpeg_batch_cap(X, ow, oh), (size_t)256);
    return m * (2 * slot + 512) + jpeg_encode_scratch_bytes(ow, oh, 3, (int)m, slot, R.progressive) + 4096;
}

// A resize-only lp_batch context (decode + resize of every image into each of the group's renditions, one chunk after
// another), then each rendition's sink over its runs of decoded items: to WebP at most the decode chunk's image count
// and kJpegWebpScratch of encoder scratch long; JPEG and PNG work out of what the context left of the lane's arena and
// pinned staging.  rs: the renditions, in the order of the context's geometries.  Items the decode refused go to the
// per-image path without being encoded.
static void jpeg_to_sink(lp_xbatch* X, Lane& L, lp_batch* b, const Task& t, const std::vector<int>& rs, const uint8_t* const* in,
                         const size_t* len) {
    const std::vector<int>& idx = t.idx;
    const int n = (int)idx.size(), K = X->k;
    std::vector<int> st((size_t)n, LP_ERR_CUDA);
    float stage[LP_STAGE_COUNT] = {};
    if (lp_batch_stage(b, in, len, n, nullptr) != LP_OK || lp_batch_run(b, stage) != LP_OK ||
        batch_resized_status(b, st.data()) != LP_OK) {
        cudaGetLastError();
        push_task_fallback(X, t);
        return;
    }
    L.ms_decode += stage[LP_STAGE_HUFF_DECODE] + stage[LP_STAGE_IDCT_COLOR];
    L.ms_resize += stage[LP_STAGE_RESIZE];
    std::vector<int> failed;
    for (int k = 0; k < n; k++)
        if (st[k] != LP_OK)
            for (int r : rs)
                if (t.rm[k] >> r & 1) failed.push_back(idx[k] * K + r);
    size_t dev_used = 0, host_used = 0;
    batch_arena_used(b, &dev_used, &host_used);
    Bump bump{L.dev + dev_used, L.dev_bytes - dev_used};
    for (size_t q = 0; q < rs.size(); q++) {
        const int r = rs[q];
        const XItem& g = X->items[(size_t)idx[0] * K + r];
        size_t stride = 0;
        const uint8_t* d_resized = rs.size() > 1 ? batch_resized_geom(b, (int)q, &stride) : lp_batch_resized_dev(b, &stride);
        int cap = n;
        if (X->rend[r].sink == S_WEBP) {
            const size_t per_frame = webp_encode_lossy_scratch_bytes(g.ow, g.oh, 3, 1);
            cap = (int)std::max<size_t>(1, std::min<size_t>((size_t)lp_batch_chunk(b), kJpegWebpScratch / per_frame));
        }
        // (JPEG files are delivered from the grid up to the pipeline's slot, as a call with this rendition alone would)
        for (const Run& u : task_runs(X, t, r, 0, n, false, st.data(), cap))
            sink_encode(X, L, bump, L.host + host_used, L.host_bytes - host_used, t, r, u, nullptr, d_resized + (size_t)u.k0 * stride,
                        stride, &failed, jpeg_batch_cap(X, g.ow, g.oh));
    }
    for (int p : failed) push_fallback(X, p);
}

// A group with one rendition on the grid runs the lp_batch pipeline to that rendition's sink (to JPEG: the pipelined
// lp_batch_transform).  A group with several decodes each file once, through a resize-only context whose decoded window
// is the bounding box of the renditions' crops, and resizes it into every rendition.
static void run_jpeg(lp_xbatch* X, Lane& L, const Task& t) {
    const std::vector<int>& idx = t.idx;
    const int n = (int)idx.size(), K = X->k;
    uint32_t all = 0;
    for (uint32_t m : t.rm) all |= m;
    std::vector<int> rs;
    for (int r = 0; r < K; r++)
        if (all >> r & 1) rs.push_back(r);
    const Rendition& R = X->rend[rs[0]];
    const XItem& g = X->items[(size_t)idx[0] * K + rs[0]];  // (the source fields are the group's; the output fields rs[0]'s)
    const bool several = rs.size() > 1;
    const bool resize_only = several || R.sink != S_JPEG;  // WebP, PNG, or several renditions: the frames go to the sinks' encoders
    // a context of one frame rendition takes rotated and gray files (lp_xbatch_decode_frames' contexts, and each task of a
    // rotated or gray group); a multi-geometry context takes orientation class 0 only, and the file sinks never get them
    const bool turned = !several && R.sink == S_FRAMES;
    size_t in_bytes = 0;
    for (int i : idx) in_bytes += X->in_len[i];
    lp_batch_config c;
    memset(&c, 0, sizeof(c));
    c.device = X->device;
    c.max_images = n;
    c.src_width = g.w;
    c.src_height = g.h;
    c.dst_width = R.opt.width;
    c.dst_height = R.opt.height;
    c.resize_method = R.opt.resize_method;
    c.normalize_orientation = R.opt.normalize_orientation;  // (sizes only the turned items a frame rendition hands it)
    c.jpeg_quality = R.quality;
    c.max_in_bytes = in_bytes + (1 << 20);
    // slot per output: never larger than the callers' buffers (lp_batch copies a whole result into out[i])
    c.out_cap = jpeg_batch_cap(X, g.ow, g.oh);
    // images per chunk: whole Huffman waves while the per-chunk scratch fits the lane's arena
    const size_t mcus = (size_t)ceil_div(g.w, 8) * ceil_div(g.h, 8);
    // multi-scan groups: + the nonzero masks per block, + the scan and table-set pools (batch.cu)
    // (a context that takes rotated files: + each chunk slot's oriented crop, at most the frame)
    const size_t per_img = (mcus * 3 + 64) * (128 + 64 + 2 + (g.jpeg_multiscan ? 8 : 0)) + (size_t)g.w * g.h * 3 * (turned ? 2 : 1) + 65536;
    const size_t pools = g.jpeg_multiscan ? batch_multiscan_pool_bytes((size_t)n) : 0;
    // every rendition's resized frames stay resident for the group; the sinks run one after another, so the largest
    // sink's room is kept
    size_t resized = 0, sink_room = 0;
    std::vector<BatchGeom> geoms;
    for (int r : rs) {
        const XItem& o = X->items[(size_t)idx[0] * K + r];
        resized += (size_t)o.ow * o.oh * 3;
        geoms.push_back(BatchGeom{o.ow, o.oh, o.cx, o.cy, o.cw, o.chh});
        if (resize_only)
            sink_room = std::max(sink_room, std::min(L.dev_bytes / 4, jpeg_group_sink_bytes(X, X->rend[r], o.ow, o.oh,
                                                                                            std::min((size_t)n, kJpegPngFrames))));
    }
    const size_t fixed = 2 * in_bytes + (size_t)n * ((resize_only ? 0 : c.out_cap) + resized + 4096) + (64u << 20) + pools + sink_room;
    const int slots = jpeg_huff_parallel_slots();
    long fit = L.dev_bytes > fixed ? (long)((L.dev_bytes - fixed) / per_img) : 0;
    if (fit < 1) {
        push_task_fallback(X, t);
        return;
    }
    int chunk = (int)std::min<long>(fit, 3L * std::max(slots, 1));
    if (slots > 0 && chunk > slots) chunk = chunk / slots * slots;
    c.chunk = std::max(1, std::min(chunk, n));
    lp_batch* b = batch_create_in(&c, L.dev, L.dev_bytes, L.host, L.host_bytes, R.progressive, g.jpeg_multiscan, resize_only,
                                  turned, turned, several ? geoms.data() : nullptr, several ? (int)geoms.size() : 0);
    if (!b) {
        push_task_fallback(X, t);
        return;
    }
    std::vector<const uint8_t*> in((size_t)n);
    std::vector<size_t> len((size_t)n), olen((size_t)n, 0);
    std::vector<uint8_t*> out((size_t)n);
    std::vector<int> st((size_t)n, 0);
    for (int k = 0; k < n; k++) {
        in[k] = X->in[idx[k]];
        len[k] = X->in_len[idx[k]];
        out[k] = X->out[(size_t)idx[k] * K + rs[0]];
    }
    L.h2d += in_bytes;
    if (resize_only) {
        jpeg_to_sink(X, L, b, t, rs, in.data(), len.data());
        lp_batch_destroy(b);
        return;
    }
    cudaEventRecord(L.ev[0], L.st);
    const int rc = lp_batch_transform(b, in.data(), len.data(), n, out.data(), olen.data(), st.data());
    for (int k = 0; k < n; k++) {
        const int i = idx[k] * K + rs[0];
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

// device bytes one item of a task needs inside a lane's arena with renditions rm (upper bound, sinks included): its
// decode once, and every rendition's output
static size_t item_device_bytes(const lp_xbatch* X, int i, uint32_t rm) {
    const XItem& it = X->items[first_pair(X, i, rm)];
    size_t outb = 0, gif_enc = 0;
    for (int r = 0; r < X->k; r++) {
        if (!(rm >> r & 1)) continue;
        const XItem& o = X->items[(size_t)i * X->k + r];
        const Rendition& R = X->rend[r];
        outb += (size_t)o.ow * o.oh * 4 * 3 + (256u << 10) + (R.sink == S_PNG ? png_sink_item_bytes(X, R, o.ow, o.oh, o.ch) : 0);
        if (o.kind == K_GIF && R.sink == S_GIF) gif_enc += gif_plan_encode_bytes(o.gif.get(), o.ow, o.oh);
    }
    switch (it.kind) {
        case K_PNG: {
            // compressed span (+ its gathered copy) + inflated scanlines (the header's row bytes: twice the samples' count
            // at 16 bits) + resized outputs + an HDR frame's tone-map records; the packed frames live in a window buffer
            // shared by the task (a fifth of the lane's arena, reserved by split_by_memory)
            const size_t row = std::max((size_t)it.w * (it.ch == 4 ? 4 : 3), it.png ? it.png->row_bytes : 0);
            const size_t raw = (row + 2) * it.h * (it.png && it.png->interlace ? 2 : 1);
            const TmFrame tm{nullptr, 0, it.w, it.h, it.ch, it.transfer, it.primaries};
            return 2 * X->in_len[i] + raw + outb + 8192 + (it.hdr ? tonemap_batch_scratch_bytes(&tm, 1) : 0);
        }
        case K_WEBP:  // the VP8L arena (at most a quarter of the lane) is shared by the task (reserved by split_by_memory)
            return webp_plan_device_bytes(*it.webp, it.span) +
                   (size_t)out_frames(it) * (round_up((size_t)it.w * it.h * it.ch, (size_t)256) + outb) + 8192;
        case K_GIF:  // (canvases and resized frames: every frame, or a clip's slots)
            return gif_plan_device_bytes(it.gif.get()) + (size_t)out_frames(it) * ((size_t)it.w * it.h * 4 + outb) + 8192 + gif_enc;
        case K_FRAME:  // the unpacked frames (one, or a clip's to an animated .webp), their table entries and outputs
            return (size_t)it.src_frames * (round_up((size_t)it.w * it.h * it.ch, (size_t)256) + sizeof(FrameUnpackItem) + outb) + 8192;
        default:
            return 0;
    }
}

// which sink the options ask for (ref lilliput.go:176-195 NewEncoder by extension), and what it reads from them
static Rendition make_rendition(const lp_image_options& opt) {
    Rendition R;
    R.opt = opt;
    std::string ext = opt.file_type ? opt.file_type : "";
    for (auto& c : ext) c = (char)tolower((unsigned char)c);
    if (ext == ".jpeg" || ext == ".jpg") {
        R.sink = S_JPEG;
        R.quality = option_value(opt, CV_IMWRITE_JPEG_QUALITY, 95);  // OpenCV's default
        R.progressive = option_value(opt, CV_IMWRITE_JPEG_PROGRESSIVE, 0) != 0;
    } else if (ext == ".webp") {
        const int q = option_value(opt, CV_IMWRITE_WEBP_QUALITY, 100);
        R.quality = q < 1 ? 1 : q;
        R.sink = S_WEBP;
        R.lossless = q > 100;
    } else if (ext == ".gif") {
        R.sink = S_GIF;
    } else if (ext == ".png") {
        R.sink = S_PNG;
        png_encode_policy(opt.encode_options, opt.encode_options_len, &R.png_level, &R.png_adaptive);
    }
    return R;
}

// a frame rendition (lp_xbatch_transform_frames, _decode_frames, _decode_clips): pixels into a caller's tensor
// (none of the file sinks' fields: a ".webp" at quality 101 must not read as lossless output)
static Rendition frames_rendition(const lp_image_options& opt) {
    Rendition R;
    R.opt = opt;
    R.sink = S_FRAMES;
    return R;
}

// A framebuffer Transform hands its encoder (on the device already, or uploaded by mat_device_view) packed into slice
// `slice` of frame rendition R's tensor on this worker's stream by the grid path's kernel; item i's size is the frame's
static int pack_framebuffer(const Rendition& R, int i, lilliput::Framebuffer* f, int64_t slice) {
    const lp_frame_tensor& T = R.dst;
    int cols = 0, rows = 0, type = 0;
    const uint8_t* dev = nullptr;
    size_t step = 0;
    int rc = mat_device_view(f->mat, &cols, &rows, &type, &dev, &step);
    if (rc) return rc;
    const int ch = opencv_type_channels(type);
    if (opencv_type_depth(type) != 8 || (ch != 1 && ch != 3 && ch != 4)) return LP_ERR_UNSUPPORTED;  // (framebuffers are 8-bit)
    if (cols > T.width || rows > T.height) return LP_ERR_BUF_TOO_SMALL;
    const FramePackItem one{dev, (uint32_t)step, cols, rows, ch, slice};
    cudaStream_t st = thread_stream();
    rc = frames_pack_launch(nullptr, &one, 1, frames_layout(T), st);
    if (!rc && cudaStreamSynchronize(st) != cudaSuccess) rc = LP_ERR_CUDA;
    if (rc) return rc;
    R.frame_w[i] = cols;
    R.frame_h[i] = rows;
    return LP_OK;
}

// A frame pair's per-image route: Transform up to its encoder, whose frame goes to the item's slice of the rendition's
// tensor
static int frames_transform(lp_xbatch* X, int p, int max_size) {
    const Rendition& R = X->rend[p % X->k];
    const int i = p / X->k;
    return lilliput::TransformToFrame(X->in[i], X->in_len[i], &R.opt, max_size,
                                      [&](lilliput::Framebuffer* f) -> int { return pack_framebuffer(R, i, f, i); });
}

// lp_xbatch_decode_clips' per-image route (one rendition: the pair is the item): Transform with every selected frame
// packed into its slot's slice; the slots the stream ended before (the last ones) are zeroed
static int clips_transform(lp_xbatch* X, int i, int max_size) {
    const Rendition& R = X->rend[0];
    const int T = X->clip_t;
    int filled = 0;
    int rc = lilliput::TransformToClip(
        X->in[i], X->in_len[i], &R.opt, max_size, T,
        [&](lilliput::Framebuffer* f, int t) -> int {
            filled = t + 1;
            return pack_framebuffer(R, i, f, (int64_t)i * T + t);
        },
        &X->clip_nframes[i], X->clip_index + (size_t)i * T, X->clip_ms + (size_t)i * T);
    if (rc || filled == T) return rc;
    const lp_frame_tensor& F = R.dst;
    const size_t slice = (size_t)F.height * F.width * F.channels * frames_dtype_bytes(F.dtype);
    cudaStream_t st = thread_stream();
    if (cudaMemsetAsync((uint8_t*)F.data + ((size_t)i * T + filled) * slice, 0, (size_t)(T - filled) * slice, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess)
        return LP_ERR_CUDA;
    return LP_OK;
}

// lp_xbatch_encode_frames' and _clips' per-image route: Transform with a decoder that answers as a PNG of the frame
// would (one frame) or as WebpDecoder would for A_i (a clip), whose DecodeTo unpacks frame k's slice with the grid path's
// kernel into the framebuffer's device mirror on this worker's stream.  The per-item argument errors are refused here.
static int transform_from_frame(lp_xbatch* X, int i, const lp_image_options* opt, int max_size, uint8_t* dst, size_t* len) {
    const lp_frame_tensor& T = X->frames;
    const int w = X->src_w[i], h = X->src_h[i];
    if (!frame_args_ok(X, i)) return LP_ERR_BAD_ARGUMENT;
    const int nf = X->src_nframes ? X->src_nframes[i] : 1;
    const int* ms = X->src_ms ? X->src_ms + (size_t)i * X->src_t : nullptr;
    return lilliput::TransformFromClip(w, h, T.channels, nf, ms, X->src_loops, opt, max_size, [&](lilliput::Framebuffer* f, int k) -> int {
        uint8_t* dev = nullptr;
        size_t step = 0;
        int rc = mat_bind_device_frame(f->mat, w, h, f->Type().v, &dev, &step);
        if (rc) return rc;
        const FrameUnpackItem one{dev, w, h, (int64_t)i * X->src_t + k};
        cudaStream_t st = thread_stream();
        rc = frames_unpack_launch(nullptr, &one, 1, (uint64_t)w * h * T.channels, frames_layout(T), st);
        if (!rc && cudaStreamSynchronize(st) != cudaSuccess) rc = LP_ERR_CUDA;
        return rc;
    }, dst, X->out_cap, len);
}

// One call over n items and k renditions (rends: each one's options and sink); out, out_len and status have n * k
// item-major entries, one per pair (a frame pair's out is null); the arguments are checked
static int xbatch_call(lp_xbatch* X, const uint8_t* const* in, const size_t* in_len, int n, const Rendition* rends, int k,
                       uint8_t* const* out, size_t out_cap, size_t* out_len, int* status) {
    int prev = 0;
    cudaGetDevice(&prev);
    LP_CUDA_OK(cudaSetDevice(X->device));
    const auto t0 = std::chrono::steady_clock::now();
    const size_t np = (size_t)n * k;  // (item, rendition) pairs
    X->in = in;
    X->in_len = in_len;
    X->out = out;
    X->out_cap = out_cap;
    X->out_len = out_len;
    X->status = status;
    X->k = k;
    X->rend.clear();
    X->rend.assign(rends, rends + k);
    X->items.clear();
    X->items.resize(np);
    X->mask.assign((size_t)n, 0);
    X->fallback.clear();
    memset(&X->stats, 0, sizeof(X->stats));
    for (Lane& L : X->lanes) {
        L.ms_decode = L.ms_resize = L.ms_encode = 0;
        L.h2d = L.d2h = 0;
        L.launches = 0;
    }
    for (size_t p = 0; p < np; p++) {
        status[p] = LP_ERR_UNSUPPORTED;  // every pair is overwritten by its group or by the fallback
        out_len[p] = 0;
    }
    parallel_for(n, X->threads, [&](int i) { parse_item(X, i); });
    const auto t1 = std::chrono::steady_clock::now();
    // groups (of items with at least one rendition on the grid) -> tasks that fit a lane
    std::map<std::tuple<int, int, int, int, int>, std::vector<int>> groups;
    for (int i = 0; i < n; i++) {
        for (int r = 0; r < k; r++)
            if (!(X->mask[i] >> r & 1)) X->fallback.push_back(i * k + r);
        if (!X->mask[i]) continue;
        const XItem& it = X->items[first_pair(X, i, X->mask[i])];
        // rotated and gray JPEGs form groups of their own when the call has several renditions (below)
        const int apart = k > 1 && it.jpeg_frames_only ? 1 << 25 : 0;
        groups[std::make_tuple((int)it.kind, it.w, it.h, it.ch, it.jpeg_sampling | (it.jpeg_multiscan ? 1 << 24 : 0) | apart)].push_back(i);
    }
    std::vector<Task> tasks;
    std::vector<double> cost;  // rough device time: the longest tasks start first
    const size_t lane_cap = X->lanes[0].dev_bytes;
    // PNG, WebP and tensor items: all geometries of a kind in as few tasks as the arena allows (the map keeps equal
    // geometries adjacent); at least two, so both lanes work.  GIF: by canvas size.  JPEG: by geometry.
    std::map<int, std::vector<int>> merged;
    for (auto& kv : groups) {
        const Kind kind = (Kind)std::get<0>(kv.first);
        if (kind == K_PNG || kind == K_WEBP || kind == K_FRAME)
            merged[(int)kind].insert(merged[(int)kind].end(), kv.second.begin(), kv.second.end());
    }
    // g: items with the renditions each runs in the tasks made from it
    auto split_by_memory = [&](Kind kind, const std::vector<std::pair<int, uint32_t>>& g) {
        size_t total = 0;
        for (const auto& e : g) total += item_device_bytes(X, e.first, e.second);
        const size_t half = total / 2 + 1;
        Task cur{kind, {}, {}};
        double work = 64u << 20;  // WebP: the order key counts pixels and payload bytes, not the decoders' scratch
        // PNG: the frame window; WebP: the VP8L / ALPH arena, when some file has lossless frames or alpha planes
        size_t arena = 0;
        if (kind == K_WEBP)
            for (const auto& e : g) arena = std::min(lane_cap / 4, arena + webp_plan_arena_bytes(*X->items[first_pair(X, e.first, e.second)].webp));
        const size_t reserve = (kind == K_PNG ? lane_cap / 5 : arena) + (64u << 20);
        size_t used = reserve;
        for (const auto& e : g) {
            const int i = e.first;
            const XItem& it = X->items[first_pair(X, i, e.second)];
            const size_t need = item_device_bytes(X, i, e.second);
            // (a PNG frame larger than the window, or an item larger than the lane: lp_transform takes its pairs)
            const bool too_big = (kind == K_PNG && round_up((size_t)it.w * it.h * it.ch, (size_t)256) > std::min<size_t>((size_t)12 << 30, lane_cap / 5)) ||
                                 need + reserve > lane_cap;
            if (too_big) {
                for (int r = 0; r < k; r++)
                    if (e.second >> r & 1) X->fallback.push_back(i * k + r);
                continue;
            }
            if (!cur.idx.empty() && (used + need > lane_cap || used > half + reserve)) {
                tasks.push_back(cur);
                cost.push_back(kind == K_WEBP ? work : (double)used);
                cur.idx.clear();
                cur.rm.clear();
                used = reserve;
                work = 64u << 20;
            }
            cur.idx.push_back(i);
            cur.rm.push_back(e.second);
            used += need;
            if (kind == K_WEBP)
                work += (double)it.span + 4096 +
                        (double)it.webp->frames.size() * ((double)it.w * it.h * it.ch + (double)it.ow * it.oh * 12 + (256u << 10));
        }
        if (!cur.idx.empty()) {
            tasks.push_back(cur);
            cost.push_back(kind == K_WEBP ? work : (double)used);
        }
    };
    // an animation's renditions run as tasks of their own, one per rendition; stills take all theirs in one task
    auto per_rendition = [&](Kind kind, const std::vector<int>& g) {
        for (int r = 0; r < k; r++) {
            std::vector<std::pair<int, uint32_t>> e;
            for (int i : g) {
                const XItem& it = X->items[first_pair(X, i, X->mask[i])];
                const bool still = kind == K_WEBP && !it.webp_animation;
                if (still && r == 0) e.emplace_back(i, X->mask[i]);
                else if (!still && (X->mask[i] >> r & 1)) e.emplace_back(i, 1u << r);
            }
            if (!e.empty()) split_by_memory(kind, e);
        }
    };
    for (auto& kv : merged) {
        if ((Kind)kv.first == K_WEBP) {
            per_rendition(K_WEBP, kv.second);
            continue;
        }
        std::vector<std::pair<int, uint32_t>> e;
        for (int i : kv.second) e.emplace_back(i, X->mask[i]);
        split_by_memory((Kind)kv.first, e);
    }
    for (auto& kv : groups) {
        const Kind kind = (Kind)std::get<0>(kv.first);
        const std::vector<int>& g = kv.second;
        if (kind == K_PNG || kind == K_WEBP || kind == K_FRAME) continue;
        if (kind == K_JPEG) {
            // A rotated or gray group (only frame renditions take it, and only a context of one rendition orients and
            // decodes it) runs each rendition as tasks of its own, as animations do; any other group all its renditions
            // in one context
            uint32_t all = 0;
            for (int i : g) all |= X->mask[i];
            std::vector<uint32_t> passes;
            for (int r = 0; r < k; r++)
                if ((std::get<4>(kv.first) & 1 << 25) && (all >> r & 1)) passes.push_back(1u << r);
            if (passes.empty()) passes.push_back(all);
            for (uint32_t pass : passes) {
                std::vector<int> gp;
                for (int i : g)
                    if (X->mask[i] & pass) gp.push_back(i);
                // host staging bounds a JPEG task: out slots (the pipelined JPEG path only) + item mirrors come from the
                // lane's pinned arena
                const int r0 = __builtin_ctz(pass);
                const XItem& it0 = X->items[(size_t)gp[0] * k + r0];
                const bool pipelined = (pass & (pass - 1)) == 0 && X->rend[r0].sink == S_JPEG;
                const size_t slot = (pipelined ? round_up(std::min(out_cap, std::max((size_t)65536, (size_t)it0.ow * it0.oh * 3)), (size_t)256) : 0) +
                                    sizeof(JpegDecodeItem) + 64;
                const size_t per = std::max<size_t>(1, X->lanes[0].host_bytes / slot);
                const size_t want = std::min(per, std::max<size_t>(1, (gp.size() + 1) / 2));  // two tasks at least: both lanes work
                for (size_t a = 0; a < gp.size(); a += want) {
                    Task t{kind, std::vector<int>(gp.begin() + a, gp.begin() + std::min(gp.size(), a + want)), {}};
                    for (int i : t.idx) t.rm.push_back(X->mask[i] & pass);
                    tasks.push_back(std::move(t));
                    cost.push_back((double)tasks.back().idx.size() * it0.w * it0.h * 0.05);
                }
            }
            continue;
        }
        per_rendition(kind, g);
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
                case K_JPEG: run_jpeg(X, L, task); break;
                case K_PNG: run_png(X, L, task); break;
                case K_WEBP: run_webp(X, L, task); break;
                case K_GIF: run_gif(X, L, task); break;
                case K_FRAME: run_frame(X, L, task); break;
                default: push_task_fallback(X, task); break;
            }
        }
        lane_launches += g_launches - mine0;
    };
    {
        std::thread other(lane_main, 1);
        lane_main(0);
        other.join();
    }
    const auto t2 = std::chrono::steady_clock::now();
    // everything else, one image per call, a few host threads (each has its own stream)
    const int max_size = X->cfg.max_size > 0 ? X->cfg.max_size : 8192;
    std::atomic<long> fb_launches{0};
    {
        std::vector<int> fb = X->fallback;
        parallel_for((int)fb.size(), std::min(X->threads, 8), [&](int q) {
            cudaSetDevice(X->device);
            const long l0 = g_launches;
            const int p = fb[q], i = p / k;
            const lp_image_options* opt = &X->rend[p % k].opt;
            size_t len = 0;
            if (X->rend[p % k].sink == S_FRAMES) {
                status[p] = X->clip_t ? clips_transform(X, i, max_size) : frames_transform(X, p, max_size);
            } else if (X->src_w) {
                status[p] = transform_from_frame(X, i, opt, max_size, out[p], &len);
                out_len[p] = status[p] == LP_OK ? len : 0;
            } else {
                status[p] = lp_transform(in[i], in_len[i], opt, out[p], out_cap, &len, max_size);
                out_len[p] = status[p] == LP_OK ? len : 0;
            }
            fb_launches += g_launches - l0;
        });
        X->stats.fallback_items = (int)fb.size();
    }
    for (XItem& it : X->items) it.gif.reset();
    const auto t3 = std::chrono::steady_clock::now();
    auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
        return std::chrono::duration<double, std::milli>(b - a).count();
    };
    X->stats.grid_items = (int)np - X->stats.fallback_items;
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

extern "C" int lp_xbatch_transform_renditions(lp_xbatch* X, const uint8_t* const* in, const size_t* in_len, int n,
                                              const lp_image_options* opts, int k, uint8_t* const* out, size_t out_cap,
                                              size_t* out_len, int* status) {
    if (k < 1) return LP_ERR_BAD_ARGUMENT;
    return lp_xbatch_transform_frames(X, in, in_len, n, opts, k, out, out_cap, out_len, status, nullptr, 0);
}

extern "C" int lp_xbatch_transform(lp_xbatch* X, const uint8_t* const* in, const size_t* in_len, int n,
                                   const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                                   int* status) {
    return lp_xbatch_transform_renditions(X, in, in_len, n, opt, 1, out, out_cap, out_len, status);
}

// Weak: the host-side tests link these objects against a stand-in runtime without pointer queries (there the call's
// tensor is never on the device); the library's static runtime defines it
#pragma weak cudaPointerGetAttributes

// Whether [p, p + bytes) lies in device memory of `device` (both of its ends)
static bool on_device(const void* p, size_t bytes, int device) {
    if (!&cudaPointerGetAttributes) return false;
    for (const void* q : {p, (const void*)((const uint8_t*)p + bytes - 1)}) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, q) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        if (a.type != cudaMemoryTypeDevice || a.device != device) return false;
    }
    return true;
}

// The tensor checks of lp_xbatch_decode_frames and lp_xbatch_encode_frames: a known dtype, data aligned to it, 3 or 4
// channels, a box of at least 1 x 1, n slices within `bytes`, all of them device memory of the context's device.
// *slice: the bytes of one slice.
static int check_frame_tensor(const lp_xbatch* X, const lp_frame_tensor* t, int n, size_t* slice) {
    if (!t) return LP_ERR_BAD_ARGUMENT;
    const lp_frame_tensor& T = *t;
    const size_t es = frames_dtype_bytes(T.dtype);
    if (!es || !T.data || (uintptr_t)T.data % es || (T.channels != 3 && T.channels != 4) || T.height < 1 || T.width < 1)
        return LP_ERR_BAD_ARGUMENT;
    if (__builtin_mul_overflow((size_t)T.height * (size_t)T.width, (size_t)T.channels * es, slice) ||
        (n > 0 && *slice > T.bytes / (size_t)n))
        return LP_ERR_BAD_ARGUMENT;
    DeviceGuard g(X->device);
    if (!g.ok || !on_device(T.data, std::max<size_t>(1, *slice * (size_t)n), X->device)) return LP_ERR_BAD_ARGUMENT;
    return LP_OK;
}

// lp_xbatch_transform_frames over checked arguments (slice[j]: the bytes of one slice of frames[j].dst; X->clip_t slices
// per item, or one).  The pairs go to the callers' arrays directly when every rendition is a file's; otherwise through
// one item-major pair array of n * (k + m) entries, scattered when the call ends.  Then every frame rendition's failed
// items get all-zero slices and 0 x 0.
static int transform_frames_call(lp_xbatch* X, const uint8_t* const* in, const size_t* in_len, int n, const lp_image_options* opts,
                                 int k, uint8_t* const* out, size_t out_cap, size_t* out_len, int* status,
                                 const lp_frame_rendition* frames, int m, const size_t* slice) {
    const int K = k + m;
    std::vector<Rendition> rends;
    for (int r = 0; r < k; r++) rends.push_back(make_rendition(opts[r]));
    for (int j = 0; j < m; j++) {
        Rendition R = frames_rendition(frames[j].opt);
        R.dst = frames[j].dst;
        R.frame_w = frames[j].width;
        R.frame_h = frames[j].height;
        for (int i = 0; i < n; i++) R.frame_w[i] = R.frame_h[i] = 0;
        rends.push_back(R);
    }
    if (!m) return xbatch_call(X, in, in_len, n, rends.data(), K, out, out_cap, out_len, status);
    const size_t np = (size_t)n * K;
    std::vector<uint8_t*> pout(np, nullptr);
    std::vector<size_t> plen(np, 0);
    std::vector<int> pst(np, LP_ERR_UNSUPPORTED);
    for (size_t i = 0; i < (size_t)n; i++)
        for (int r = 0; r < k; r++) pout[i * K + r] = out[i * k + r];
    int rc = xbatch_call(X, in, in_len, n, rends.data(), K, pout.data(), out_cap, plen.data(), pst.data());
    if (rc) return rc;
    for (size_t i = 0; i < (size_t)n; i++) {
        for (int r = 0; r < k; r++) {
            status[i * k + r] = pst[i * K + r];
            out_len[i * k + r] = plen[i * K + r];
        }
        for (int j = 0; j < m; j++) frames[j].status[i] = pst[i * K + k + j];
    }
    DeviceGuard g(X->device);
    cudaStream_t st = X->lanes[0].st;
    for (int j = 0; j < m && !rc; j++) {
        const lp_frame_rendition& F = frames[j];
        const size_t per = (size_t)std::max(1, X->clip_t) * slice[j];  // an item's slices
        for (int i = 0; i < n && !rc;) {
            if (F.status[i] == LP_OK) {
                i++;
                continue;
            }
            int e = i;
            for (; e < n && F.status[e] != LP_OK; e++) F.width[e] = F.height[e] = 0;
            if (cudaMemsetAsync((uint8_t*)F.dst.data + (size_t)i * per, 0, (size_t)(e - i) * per, st) != cudaSuccess) rc = LP_ERR_CUDA;
            i = e;
        }
    }
    if (!rc && cudaStreamSynchronize(st) != cudaSuccess) rc = LP_ERR_CUDA;
    return rc;
}

extern "C" int lp_xbatch_transform_frames(lp_xbatch* X, const uint8_t* const* in, const size_t* in_len, int n,
                                          const lp_image_options* opts, int k, uint8_t* const* out, size_t out_cap,
                                          size_t* out_len, int* status, const lp_frame_rendition* frames, int m) {
    if (!X || n < 0 || k < 0 || m < 0 || k + m < 1 || k + m > kMaxRenditions || (n > 0 && (!in || !in_len)) ||
        (k > 0 && (!opts || (n > 0 && (!out || !out_len || !status)))) || (m > 0 && !frames))
        return LP_ERR_BAD_ARGUMENT;
    size_t slice[kMaxRenditions] = {};
    for (int j = 0; j < m; j++) {
        const lp_frame_rendition& F = frames[j];
        if ((n > 0 && (!F.width || !F.height || !F.status)) || check_frame_tensor(X, &F.dst, n, &slice[j])) return LP_ERR_BAD_ARGUMENT;
        const uintptr_t a0 = (uintptr_t)F.dst.data, a1 = a0 + slice[j] * (size_t)n;
        for (int q = 0; q < j; q++) {  // (no two tensors share a byte of their n slices)
            const uintptr_t b0 = (uintptr_t)frames[q].dst.data, b1 = b0 + slice[q] * (size_t)n;
            if (a0 < b1 && b0 < a1) return LP_ERR_BAD_ARGUMENT;
        }
    }
    return transform_frames_call(X, in, in_len, n, opts, k, out, out_cap, out_len, status, frames, m, slice);
}

extern "C" int lp_xbatch_decode_frames(lp_xbatch* X, const uint8_t* const* in, const size_t* in_len, int n,
                                       const lp_image_options* opt, const lp_frame_tensor* dst, int* width, int* height,
                                       int* status) {
    if (!opt || !dst) return LP_ERR_BAD_ARGUMENT;
    const lp_frame_rendition F{*opt, *dst, width, height, status};
    return lp_xbatch_transform_frames(X, in, in_len, n, nullptr, 0, nullptr, 0, nullptr, nullptr, &F, 1);
}

extern "C" int lp_xbatch_decode_clips(lp_xbatch* X, const uint8_t* const* in, const size_t* in_len, int n,
                                      const lp_image_options* opt, int frames_per_item, const lp_frame_tensor* dst, int* width,
                                      int* height, int* nframes, int* frame_index, int64_t* start_ms, int* status) {
    const int T = frames_per_item;
    if (!X || n < 0 || !opt || !dst || T < 1 || T > LP_XBATCH_MAX_CLIP_FRAMES ||
        (n > 0 && (!in || !in_len || !width || !height || !nframes || !frame_index || !start_ms || !status)))
        return LP_ERR_BAD_ARGUMENT;
    size_t slice = 0;
    if ((int64_t)n * T > INT_MAX || check_frame_tensor(X, dst, n * T, &slice)) return LP_ERR_BAD_ARGUMENT;
    const size_t slots = (size_t)n * T;
    for (int i = 0; i < n; i++) nframes[i] = 0;
    for (size_t s = 0; s < slots; s++) {
        frame_index[s] = -1;
        start_ms[s] = 0;
    }
    X->clip_t = T;
    X->clip_nframes = nframes;
    X->clip_index = frame_index;
    X->clip_ms = start_ms;
    const lp_frame_rendition F{*opt, *dst, width, height, status};
    const int rc = transform_frames_call(X, in, in_len, n, nullptr, 0, nullptr, 0, nullptr, nullptr, &F, 1, &slice);
    X->clip_t = 0;
    X->clip_nframes = X->clip_index = nullptr;
    X->clip_ms = nullptr;
    for (int i = 0; i < n && !rc; i++) {  // an item that failed: no frames, and every slot unused
        if (status[i] == LP_OK) continue;
        nframes[i] = 0;
        for (int t = 0; t < T; t++) {
            frame_index[(size_t)i * T + t] = -1;
            start_ms[(size_t)i * T + t] = 0;
        }
    }
    return rc;
}

// lp_xbatch_encode_frames (T 1, nframes null: one frame each) and lp_xbatch_encode_clips: files from the items' slices of
// a checked tensor, T per item
static int encode_tensor(lp_xbatch* X, const lp_frame_tensor& src, int n, int T, const int* nframes, const int* width,
                         const int* height, const int* duration_ms, int loop_count, const lp_image_options* opt,
                         uint8_t* const* out, size_t out_cap, size_t* out_len, int* status) {
    X->frames = src;
    X->src_w = width;
    X->src_h = height;
    X->src_t = T;
    X->src_nframes = nframes;
    X->src_ms = duration_ms;
    X->src_loops = loop_count;
    const Rendition R = opt ? make_rendition(*opt) : Rendition();  // (opt may be null when n == 0)
    const int rc = xbatch_call(X, nullptr, nullptr, n, &R, 1, out, out_cap, out_len, status);
    X->src_w = X->src_h = nullptr;
    X->src_t = 1;
    X->src_nframes = X->src_ms = nullptr;
    X->src_loops = 0;
    return rc;
}

extern "C" int lp_xbatch_encode_clips(lp_xbatch* X, const lp_frame_tensor* src, int n, int frames_per_item, const int* nframes,
                                      const int* width, const int* height, const int* duration_ms, int loop_count,
                                      const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                                      int* status) {
    const int T = frames_per_item;
    if (!X || n < 0 || T < 1 || T > LP_XBATCH_MAX_CLIP_FRAMES || loop_count < 0 || loop_count > 65535 ||
        (n > 0 && (!opt || !nframes || !width || !height || !duration_ms || !out || !out_len || !status)))
        return LP_ERR_BAD_ARGUMENT;
    size_t slice = 0;
    if ((int64_t)n * T > INT_MAX || check_frame_tensor(X, src, n * T, &slice)) return LP_ERR_BAD_ARGUMENT;
    return encode_tensor(X, *src, n, T, nframes, width, height, duration_ms, loop_count, opt, out, out_cap, out_len, status);
}

extern "C" int lp_xbatch_encode_frames(lp_xbatch* X, const lp_frame_tensor* src, int n, const int* width, const int* height,
                                       const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                                       int* status) {
    if (!X || n < 0 || (n > 0 && (!opt || !width || !height || !out || !out_len || !status))) return LP_ERR_BAD_ARGUMENT;
    size_t slice = 0;
    if (check_frame_tensor(X, src, n, &slice)) return LP_ERR_BAD_ARGUMENT;
    return encode_tensor(X, *src, n, 1, nullptr, width, height, nullptr, 0, opt, out, out_cap, out_len, status);
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

extern "C" int lp_multi_transform_renditions(lp_multi* m, const uint8_t* const* in, const size_t* in_len, int n,
                                             const lp_image_options* opts, int k, uint8_t* const* out, size_t out_cap,
                                             size_t* out_len, int* status) {
    if (!m || n < 0 || !opts || k < 1 || k > kMaxRenditions || (n > 0 && (!in || !in_len || !out || !out_len || !status)))
        return LP_ERR_BAD_ARGUMENT;
    const int G = (int)m->ctx.size();
    m->first.assign((size_t)G + 1, n);
    lp_shard_blocks(in_len, n, G, m->first.data());
    std::vector<int> rc((size_t)G, LP_OK);
    std::vector<std::thread> pool;
    for (int g = 0; g < G; g++) {
        const int i0 = m->first[g], cnt = m->first[g + 1] - m->first[g];
        if (cnt <= 0) continue;
        const size_t p0 = (size_t)i0 * k;  // (an item's renditions stay with it)
        pool.emplace_back([=, &rc]() {
            rc[g] = lp_xbatch_transform_renditions(m->ctx[g], in + i0, in_len + i0, cnt, opts, k, out + p0, out_cap, out_len + p0,
                                                   status + p0);
        });
    }
    for (auto& t : pool) t.join();
    for (int g = 0; g < G; g++)
        if (rc[g]) return rc[g];
    return LP_OK;
}

extern "C" int lp_multi_transform(lp_multi* m, const uint8_t* const* in, const size_t* in_len, int n,
                                  const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                                  int* status) {
    return lp_multi_transform_renditions(m, in, in_len, n, opt, 1, out, out_cap, out_len, status);
}

// per-device statistics of the last call
extern "C" void lp_multi_get_stats(const lp_multi* m, int device_index, lp_xbatch_stats* out) {
    if (m && out && device_index >= 0 && device_index < (int)m->ctx.size()) lp_xbatch_get_stats(m->ctx[device_index], out);
}
