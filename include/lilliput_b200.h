/*
 * lilliput_b200.h -- additive C ABI of liblilliput_b200.so: the whole-Transform
 * entry point, the batch entry point and the device-resident stage entry points.
 *
 * The per-image cgo surface lilliput binds to is in lp_opencv.h (same symbols
 * as the reference's opencv.hpp).  This header adds what the reference does not
 * have, because one synchronous image per cgo call cannot fill an H100:
 *
 *   lp_transform          one image through NewDecoder + ImageOps.Transform
 *                         (ref lilliput.go:129-164, ops.go:352-444) -- the
 *                         C++ host mirror of the Go policy layer, driving the
 *                         per-image ABI.  Exists in BOTH liblilliput_b200.so
 *                         (CUDA kernels behind the ABI) and oracle/_ref's
 *                         libref_oracle.so (the reference's own shims behind
 *                         the ABI), so parity tests call the same function on
 *                         both libraries.
 *   lp_batch_*            N independent JPEG images -> Fit/area-resize -> JPEG,
 *                         each stage one grid launch over the whole batch
 *                         (SURVEY.md 8(b) "additive batch ABI").  Per-item
 *                         semantics are those of lp_transform.
 *   lp_*_dev              single stages on DEVICE pointers, on a caller
 *                         stream, used by bench.py (roofline timing) and the
 *                         parity tests.
 *
 * All functions return 0 (LP_OK) or a negative lp_status unless stated.
 */
#ifndef LILLIPUT_B200_H
#define LILLIPUT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Mirrors lilliput's sentinel errors (ref lilliput.go:25-30) plus io.EOF. */
typedef enum lp_status {
    LP_OK = 0,
    LP_ERR_INVALID_IMAGE = -1,       /* ErrInvalidImage */
    LP_ERR_DECODING_FAILED = -2,     /* ErrDecodingFailed */
    LP_ERR_BUF_TOO_SMALL = -3,       /* ErrBufTooSmall */
    LP_ERR_FRAMEBUF_NO_PIXELS = -4,  /* ErrFrameBufNoPixels */
    LP_ERR_SKIP_NOT_SUPPORTED = -5,  /* ErrSkipNotSupported */
    LP_ERR_ENCODE_TIMEOUT = -6,      /* ErrEncodeTimeout */
    LP_ERR_EOF = -7,                 /* io.EOF */
    LP_ERR_UNSUPPORTED = -8,         /* format/feature outside SURVEY 8 scope */
    LP_ERR_CUDA = -9,                /* CUDA runtime failure (logged to stderr) */
    LP_ERR_BAD_ARGUMENT = -10,
    LP_ERR_OPENCV = -100             /* -100 - OPENCV_ERROR_* from a region op */
} lp_status;

/* ImageOpsSizeMethod (ref ops.go:17-22) */
#define LP_OPS_NO_RESIZE 0
#define LP_OPS_FIT 1
#define LP_OPS_RESIZE 2

/* ImageOptions (ref ops.go:26-65).  encode_options is the flat k,v int array
 * the Go side marshals for the C call (ref opencv.go:876-886). */
typedef struct lp_image_options {
    const char* file_type; /* ".jpeg", ".jpg", ".png", ... */
    int width;
    int height;
    int resize_method; /* LP_OPS_* */
    int normalize_orientation;
    const int* encode_options;
    size_t encode_options_len; /* number of ints (2 per option) */
    int max_encode_frames;
    int64_t max_encode_duration_ns;
    int64_t encode_timeout_ns;
    int disable_animated_output;
    int force_sdr;
} lp_image_options;

/* NewDecoder(in) + NewImageOps(max_size).Transform(d, opt, dst).
 * *out_len receives the encoded length.  ref ops.go:352, examples/main.go:82-130 */
int lp_transform(const uint8_t* in, size_t in_len, const lp_image_options* opt, uint8_t* dst,
                 size_t dst_cap, size_t* out_len, int max_size);

/* Name of the backend behind the per-image ABI: "cuda-sm90a" or "reference". */
const char* lp_backend_name(void);

/* ---- host-only container sniffers (never touch the device) ------------------
 * The Go side keeps its own copies (opencv.go:467-637); these expose the C++ mirror's so the
 * reference's unit tests for them (opencv_test.go:9-220) can be replayed against this library. */
/* detectAPNG (ref opencv.go:623-637): 1 if an acTL / fcTL / fdAT chunk is reachable, else 0. */
int lp_detect_apng(const uint8_t* in, size_t in_len);
/* detectContentLength (ref opencv.go:513-620): bytes up to and including PNG IEND / JPEG EOI,
 * in_len for anything else or when no end marker is found. */
int lp_detect_content_length(const uint8_t* in, size_t in_len);
/* makePngChunkIter + next() (ref opencv.go:468-511): -1 if `in` lacks the PNG signature, else the
 * number of chunks the iterator visits; the 4-byte types of the first min(count, cap) go to `types`. */
int lp_png_chunk_types(const uint8_t* in, size_t in_len, uint8_t* types, int cap);

/* ---- stage-level checks on HOST buffers (through the per-image ABI) -------- */
/* Decode a JPEG/PNG to packed BGR/BGRA/Gray; returns LP status, fills dims. */
int lp_decode_host(const uint8_t* in, size_t in_len, uint8_t* pixels, size_t pixels_cap,
                   int* width, int* height, int* type, int* orientation);
/* Fit (crop + INTER_AREA) exactly as Framebuffer.Fit (ref opencv.go:326-374). */
int lp_fit_host(const uint8_t* src, int src_w, int src_h, int type, uint8_t* dst, int dst_w,
                int dst_h);
/* cv::resize of a cropped view (ref opencv.cpp:196-215) with any interpolation. */
int lp_resize_host(const uint8_t* src, int src_w, int src_h, int type, int crop_x, int crop_y,
                   int crop_w, int crop_h, uint8_t* dst, int dst_w, int dst_h, int interpolation);
/* Encode packed pixels to ext; returns encoded length in *out_len. */
int lp_encode_host(const char* ext, const uint8_t* pixels, int width, int height, int type,
                   const int* opt, size_t opt_len, uint8_t* dst, size_t dst_cap, size_t* out_len);
/* EXIF orientation transform (ref opencv.cpp:217-221); dims may swap. */
int lp_orient_host(const uint8_t* src, int width, int height, int type, int orientation,
                   uint8_t* dst, int* out_w, int* out_h);

/* Framebuffer.TonemapToSDR (ref opencv.go:791-810, color_info.cpp:112-270): PQ (16) / HLG (18) pixels of a packed
 * 8-bit BGR / BGRA frame -> SDR BT.709, in place.  primaries = cICP colour primaries code point. */
int lp_tonemap_host(uint8_t* pixels, int width, int height, int type, int transfer, int primaries);

/* GIF: animation metadata as gifDecoder reports it (ref giflib.go:76-151). */
typedef struct lp_gif_info {
    int width, height, frame_count, loop_count, duration_ms;
    unsigned int background_color; /* gifDecoder.BackgroundColor(): A<<24 | R<<16 | G<<8 | B */
} lp_gif_info;
int lp_gif_get_info(const uint8_t* in, size_t in_len, lp_gif_info* info);
/* Decode up to max_frames frames through gifDecoder.DecodeTo (ref giflib.go:180-219): every frame
 * is the FULL canvas, BGRA u8, written back to back into `frames`.  delays_ms / disposals (lilliput
 * DisposeMethod values) get one entry per frame.  *n_frames = frames decoded; returns LP_OK when the
 * stream ended with EOF, else the error that stopped it (frames decoded so far are still valid). */
int lp_gif_decode_frames_host(const uint8_t* in, size_t in_len, uint8_t* frames, size_t frames_cap,
                              int max_frames, int* n_frames, int* delays_ms, int* disposals);
/* WebP: every frame exactly as webp_decoder_decode leaves it in the mat (ref webp.cpp:291-359:
 * frame-sized BGR / BGRA), packed back to back.  meta[8*i..] = width, height, channels, x_offset,
 * y_offset, delay_ms, dispose, blend.  info[0..7] = canvas width, canvas height, pixel type, frame
 * count, total duration (ms), loop count, background colour, ICC profile length.  `frames` may be
 * NULL to read `info` only. */
int lp_webp_decode_frames_host(const uint8_t* in, size_t in_len, uint8_t* frames, size_t frames_cap,
                               int max_frames, int* n_frames, int* meta, unsigned int* info);

#ifndef LP_REFERENCE_BACKEND
/* ------------------------- CUDA-only entry points -------------------------- */

/* Opaque batch context bound to one CUDA device (one per GPU / per rank). */
typedef struct lp_batch lp_batch;

/* Geometry and options shared by every image of a homogeneous batch
 * (BASELINE config 2: 4096 x 1920x1080 JPEG -> Fit 256x256 JPEG q85). */
typedef struct lp_batch_config {
    int device;          /* CUDA ordinal */
    int max_images;      /* capacity N */
    int src_width;       /* every input must decode to this size ...        */
    int src_height;      /* ... (checked per image; mismatch => per-item error) */
    int dst_width;       /* requested output size (ImageOptions.Width/Height) */
    int dst_height;
    int resize_method;   /* LP_OPS_FIT / LP_OPS_RESIZE */
    int jpeg_quality;    /* EncodeOptions[JpegQuality] */
    size_t max_in_bytes; /* capacity for the sum of compressed input sizes */
    size_t out_cap;      /* per-image output capacity in bytes */
    int chunk;           /* images per pipelined chunk (0 = default) */
    int normalize_orientation; /* ImageOptions.NormalizeOrientation (0 = false): the size requested of an
                                  image whose EXIF orientation swaps its axes (5..8) is that of the
                                  header's size turned, as Transform computes it */
} lp_batch_config;

lp_batch* lp_batch_create(const lp_batch_config* cfg);
void lp_batch_destroy(lp_batch* b);

/* Host -> host: the reference-facing call.  `in[i]` / `out[i]` are HOST buffers
 * (pinned or not); H2D of the compressed bytes and D2H of the encoded bytes are
 * inside the call.  status[i] is an lp_status per image.
 *
 * Sources taken: 8-bit Huffman-coded 3-component (YCbCr) and 1-component (gray) JPEGs of
 * the configured size, in any order in one batch, with any EXIF orientation -- baseline or extended sequential (with or without restart markers
 * and optimised tables), progressive, or sequential with one scan per component.  The
 * orientation is applied on the device, per item, as Transform applies it (whether or
 * not normalize_orientation is set); an orientation that swaps the axes may give an item
 * another output size than the top-left ones (Fit above the source size, Width != Height).
 * A gray item is decoded, oriented and resized on one channel and comes back as a
 * one-component JPEG, as Transform writes it.
 * Each item gets the status and bytes lp_transform gives it, except that multi-scan files
 * that overflow the context's scan or Huffman-table pools (sized by max_images, see
 * batch.cu) get LP_ERR_UNSUPPORTED. */
int lp_batch_transform(lp_batch* b, const uint8_t* const* in, const size_t* in_len, int n,
                       uint8_t* const* out, size_t* out_len, int* status);

/* Same pipeline split at the PCIe boundary, for device-resident timing:
 *   lp_batch_stage   parse headers (host) and copy scan data to HBM
 *   lp_batch_run     every kernel of the path on data already in HBM; fills
 *                    stage_ms[LP_STAGE_COUNT] (CUDA-event ms per stage) if non-NULL
 *   lp_batch_fetch   copy encoded bytes HBM -> host */
enum {
    LP_STAGE_HUFF_DECODE = 0,
    LP_STAGE_IDCT_COLOR = 1,
    LP_STAGE_RESIZE = 2,
    LP_STAGE_ENC_TRANSFORM = 3,
    LP_STAGE_ENC_ENTROPY = 4,
    LP_STAGE_TOTAL = 5,
    LP_STAGE_COUNT = 6
};
int lp_batch_stage(lp_batch* b, const uint8_t* const* in, const size_t* in_len, int n,
                   int* status);
int lp_batch_run(lp_batch* b, float* stage_ms);
int lp_batch_fetch(lp_batch* b, uint8_t* const* out, size_t* out_len, int* status);
/* Number of kernel launches issued by the last lp_batch_run / lp_batch_transform. */
int lp_batch_last_launches(const lp_batch* b);
/* Device-to-host bytes per image besides the encoded file (length, packed offset, item mirror). */
size_t lp_batch_d2h_overhead_per_image(void);
/* Images per pipelined chunk actually used by this context. */
int lp_batch_chunk(const lp_batch* b);
/* Channels of item i's decoded and resized frames in the staged batch: 3 (BGR), 1 (a gray source), 0 when its
 * header was refused. */
int lp_batch_item_channels(const lp_batch* b, int i);
/* Diagnostics (valid after lp_batch_fetch / lp_batch_transform): rounds the parallel Huffman
 * synchronisation needed per image. */
void lp_batch_sync_rounds(const lp_batch* b, double* mean, int* max);
/* Diagnostics: SM cycles the JPEG entropy kernel spent per phase since the last reset on the current device, summed over
 * its CTAs -- out8[0] table set-up, [1] guess pass, [2] synchronisation rounds, [3] prefix sum + write pass, [4] DC pass,
 * [5] number of CTAs (= images).  reset != 0 clears the counters after reading.  Returns an lp_status. */
int lp_huff_phase_clocks(unsigned long long* out8, int reset);
/* Device pointer to the decoded frames / resized frames of the last run (tests).  Resized frame i is at
 * i * image_stride, rows packed, in its own output size; decoded windows are slot-strided within the last chunk.
 * Slots are spaced for 3 channels; a gray item's frame is 1 channel (lp_batch_item_channels), its rows packed (resized)
 * or a 16-byte multiple apart (decoded window) from the start of its own slot. */
const uint8_t* lp_batch_decoded_dev(const lp_batch* b, size_t* image_stride);
const uint8_t* lp_batch_resized_dev(const lp_batch* b, size_t* image_stride);

/* ---- heterogeneous batch: any supported formats and sizes, one set of options ----------------
 * (BASELINE configs 3, 4, 5: PNG -> WebP, animated GIF -> animated WebP, mixed JPEG / PNG / WebP -> JPEG.)
 * Sinks with a grid path: ".jpeg", lossy ".webp", lossless ".webp" (WebpQuality above 100, from PNG and GIF sources),
 * ".gif" (from GIF sources) and ".png" (from JPEG, PNG and WebP stills; RGBA sources keep their alpha).
 * Per-item semantics, status and bytes are those of lp_transform(in[i], ..., opt, out[i], out_cap, ...).
 * Items are grouped by decoder and source geometry and every stage of a group is one grid launch
 * (csrc/xbatch.cu); whatever the grid path does not cover runs through lp_transform inside the call. */
typedef struct lp_xbatch lp_xbatch;
typedef struct lp_xbatch_config {
    int device;          /* CUDA ordinal */
    size_t arena_bytes;  /* device working memory; 0 = 72 % of what is free at creation */
    int host_threads;    /* header parsing / per-image fallback workers; 0 = auto */
    int max_size;        /* ImageOps maxSize for every item (lp_transform's max_size); 0 = 8192 */
} lp_xbatch_config;
typedef struct lp_xbatch_stats {
    int grid_items, fallback_items, groups, launches;
    double ms_parse, ms_grid, ms_fallback, ms_total; /* host wall clock of the phases */
    double ms_decode, ms_resize, ms_encode;          /* CUDA-event time of the grid stages, summed over chunks AND lanes */
    size_t h2d_bytes, d2h_bytes;
    double ms_busy_max_lane; /* the two lanes run concurrently: the larger of their per-lane stage-time sums */
} lp_xbatch_stats;
lp_xbatch* lp_xbatch_create(const lp_xbatch_config* cfg);
void lp_xbatch_destroy(lp_xbatch* x);
int lp_xbatch_transform(lp_xbatch* x, const uint8_t* const* in, const size_t* in_len, int n,
                        const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                        int* status);
void lp_xbatch_get_stats(const lp_xbatch* x, lp_xbatch_stats* out);
/* Several outputs ("renditions") of every item in one call: opts[0..k-1], k in 1..LP_XBATCH_MAX_RENDITIONS.  out,
 * out_len and status have n * k entries, item-major: pair (i, r) is at i * k + r and gets exactly the status and bytes
 * of lp_transform(in[i], in_len[i], &opts[r], ...).  Each file is uploaded and decoded once for all the renditions it
 * takes on the grid path (an animation: once per rendition); the pairs the grid path does not take run through
 * lp_transform.  grid_items and fallback_items of the stats count pairs.  lp_xbatch_transform is this call with k = 1.
 * A bad k or a null opts: LP_ERR_BAD_ARGUMENT, and nothing is written. */
#define LP_XBATCH_MAX_RENDITIONS 16
int lp_xbatch_transform_renditions(lp_xbatch* x, const uint8_t* const* in, const size_t* in_len, int n,
                                   const lp_image_options* opts, int k, uint8_t* const* out, size_t out_cap,
                                   size_t* out_len, int* status);

/* Pixels instead of files: the frame every item would be encoded from, written into the caller's device tensor.
 * Item i's frame is the one lp_transform(in[i], opt with file_type ".png") hands to its encoder: decoded, tone-mapped
 * if HDR, oriented, with Fit / Resize / NoResize applied; of a GIF or animated WebP, frame 0 composited as Transform
 * composites it.  status[i] is that call's status, width[i] x height[i] the frame's size.  opt->file_type and the
 * encode options are ignored.
 *   - slice i of dst (item i's H x W x C or C x H x W elements) holds the frame at its top-left, zero elsewhere
 *   - a gray frame is replicated to three channels; an opaque one gets 255 as channel 3 when channels == 4; a BGRA
 *     frame's alpha is dropped (not composited) when channels == 3
 *   - a frame larger than the box in either dimension: LP_ERR_BUF_TOO_SMALL
 *   - an item whose status is not LP_OK: an all-zero slice and 0 x 0
 * dst must stay allocated for the call, on the context's device; every write into it is complete when the call
 * returns.  LP_ERR_BAD_ARGUMENT, with nothing written, for: n < 0; null in / in_len / opt / width / height / status
 * with n > 0; a null dst or data; data not device memory of the context's device, or not aligned to the dtype;
 * bytes < n slices; height or width < 1; channels not 3 or 4; an unknown dtype.
 * Stats: grid_items / fallback_items count items; ms_encode is the pack; d2h_bytes carries no pixels. */
enum { LP_DTYPE_U8 = 0, LP_DTYPE_F16 = 1, LP_DTYPE_BF16 = 2, LP_DTYPE_F32 = 3 };
typedef struct lp_frame_tensor {
    void* data;              /* device memory on the context's device */
    size_t bytes;            /* capacity of data */
    int height, width;       /* box per item: item i's frame at its top-left, the rest of its slice zero */
    int channels;            /* 3 or 4 */
    int nchw;                /* 0: N x H x W x C, 1: N x C x H x W (dense, item i is slice i) */
    int rgb;                 /* 0: B, G, R[, A]   1: R, G, B[, A] */
    int dtype;               /* LP_DTYPE_* */
    float scale[4], bias[4]; /* float dtypes: out[c] = fmaf(sample, scale[c], bias[c]) in fp32, then rounded to
                                nearest into the dtype; indexed by OUTPUT channel; ignored for U8 */
} lp_frame_tensor;
int lp_xbatch_decode_frames(lp_xbatch* x, const uint8_t* const* in, const size_t* in_len, int n,
                            const lp_image_options* opt, const lp_frame_tensor* dst, int* width, int* height,
                            int* status);

/* Files and pixels of the same uploads in one call: k file renditions (opts[0..k-1], as lp_xbatch_transform_renditions)
 * and m frame renditions (frames[0..m-1], as lp_xbatch_decode_frames), 0 <= k, 0 <= m, 1 <= k + m <=
 * LP_XBATCH_MAX_RENDITIONS.
 *   - out, out_len and status have n * k item-major entries, each exactly what lp_xbatch_transform_renditions(in, in_len,
 *     n, opts, k, ...) writes there
 *   - frames[j].dst, width, height and status hold exactly what lp_xbatch_decode_frames(in, in_len, n, &frames[j].opt,
 *     &frames[j].dst, ...) writes; the slices of failed items are zero
 * Each file is uploaded and decoded once for all the renditions it takes on the grid path, file and frame alike; an
 * animation decodes once per rendition, and an EXIF-rotated or gray JPEG (which only frame renditions take there) once
 * per frame rendition.  LP_ERR_BAD_ARGUMENT, with nothing written, for: a bad k or m; n < 0; a null in / in_len with
 * n > 0; a null opts with k > 0, or null out / out_len / status with n > 0 and k > 0; a null frames with m > 0; any
 * frame rendition failing lp_xbatch_decode_frames' argument checks; two tensors whose n slices overlap.  Stats:
 * grid_items and fallback_items count all n * (k + m) pairs; d2h_bytes counts files only; h2d_bytes is the file
 * renditions' call's plus the frame renditions' pack tables.  lp_xbatch_transform_renditions is this call with m = 0,
 * lp_xbatch_decode_frames with k = 0 and m = 1. */
typedef struct lp_frame_rendition {
    lp_image_options opt; /* as lp_xbatch_decode_frames' opt (file_type and encode options ignored) */
    lp_frame_tensor dst;  /* n slices, as lp_xbatch_decode_frames' dst */
    int* width;           /* n entries each */
    int* height;
    int* status;
} lp_frame_rendition;
int lp_xbatch_transform_frames(lp_xbatch* x, const uint8_t* const* in, const size_t* in_len, int n,
                               const lp_image_options* opts, int k, uint8_t* const* out, size_t out_cap,
                               size_t* out_len, int* status, const lp_frame_rendition* frames, int m);

/* Clips instead of one frame: up to T = frames_per_item frames of every item, spread over the whole animation, written
 * into the caller's device tensor.  Slice i * T + t of dst (the same lp_frame_tensor as lp_xbatch_decode_frames, n * T
 * slices; with nchw an N x T x C x H x W tensor) holds slot t of item i.
 *   - item i's frames are the ones lp_transform(in[i], opt) hands its encoder, in order: decoded, tone-mapped if HDR,
 *     oriented, composited as Transform composites them, with Fit / Resize / NoResize applied.  opt's width, height,
 *     resize_method, normalize_orientation and force_sdr count; file_type, the encode options, max_encode_frames,
 *     max_encode_duration_ns, disable_animated_output and encode_timeout_ns are ignored.  Frame 0 is exactly what
 *     lp_xbatch_decode_frames writes for the item.
 *   - F = nframes[i], the frame count the decoder's header reports: a GIF's record walk, a WebP's container frame
 *     count, and 1 for every other source (an APNG included: Transform decodes its first frame only)
 *   - sampling: when F <= T, slot t < F holds frame t; otherwise slot t holds frame floor(t * F / T), T distinct frames
 *     with frame 0 first.  Decoding stops after the last selected frame L: nothing behind it is read, so damage behind
 *     L is never seen
 *   - frame_index[i * T + t]: the slot's frame index, -1 for an unused slot.  start_ms[i * T + t]: the sum of the
 *     durations (in ms, as the decoder reports them) of frames 0 .. index - 1; 0 for an unused slot
 *   - an unused slot is all zero, as is a slot whose frame the stream ended before delivering (its index is -1)
 *   - width[i] x height[i]: the size of every frame of the item.  status[i]: Transform's status.  A frame larger than
 *     the box in either dimension: LP_ERR_BUF_TOO_SMALL.  An item whose status is not LP_OK: T all-zero slices, 0 x 0,
 *     nframes 0, every index -1
 * Slices are packed as lp_xbatch_decode_frames packs them.  dst must stay allocated for the call, on the context's
 * device; every write into it is complete when the call returns.  LP_ERR_BAD_ARGUMENT, with nothing written, for: the
 * tensor checks of lp_xbatch_decode_frames with n * T slices in place of n; T outside 1..LP_XBATCH_MAX_CLIP_FRAMES;
 * n < 0; a null in / in_len / opt / output array with n > 0.
 * Stats: grid_items / fallback_items count items; ms_encode is the pack; d2h_bytes carries no pixels. */
#define LP_XBATCH_MAX_CLIP_FRAMES 4096
int lp_xbatch_decode_clips(lp_xbatch* x, const uint8_t* const* in, const size_t* in_len, int n,
                           const lp_image_options* opt, int frames_per_item, const lp_frame_tensor* dst, int* width,
                           int* height, int* nframes, int* frame_index, int64_t* start_ms, int* status);

/* Files from pixels: slice i of the caller's device tensor src (the same lp_frame_tensor as lp_xbatch_decode_frames)
 * holds item i's frame at its top-left, width[i] x height[i].  The frame is converted to 8-bit BGR (channels 3) or BGRA
 * (channels 4) and goes through ImageOps.Transform with opt: status and bytes of item i are exactly those of
 * lp_transform(P_i, opt, out[i], out_cap, ..., max_size), where P_i is an 8-bit PNG of that frame (colour type 2 or 6,
 * no ancillary chunks).
 *   - conversion per element of tensor channel c: U8 as is; F16 and BF16 widened to fp32 exactly, then as F32:
 *     fmaf(x, scale[c], bias[c]) in fp32, rounded half to even, clamped to [0, 255]; NaN gives 0 (+inf 255, -inf 0).
 *     rgb and nchw mean what they mean for lp_xbatch_decode_frames; channel 3, when present, is alpha.  A tensor
 *     lp_xbatch_decode_frames wrote with scale 1/255 comes back with scale 255.
 *   - width[i] or height[i] outside 1..box: that item gets LP_ERR_BAD_ARGUMENT and out_len 0; the others go on
 * The tensor's contents must be complete before the call: the library's streams do not wait on the caller's.  The call
 * only reads the tensor.  LP_ERR_BAD_ARGUMENT, with nothing written, for the tensor checks of lp_xbatch_decode_frames,
 * n < 0, and a null opt / width / height / out / out_len / status with n > 0.
 * Stats: ms_decode is the unpack; h2d_bytes carries no pixels (the item table only); d2h_bytes is the files. */
int lp_xbatch_encode_frames(lp_xbatch* x, const lp_frame_tensor* src, int n, const int* width, const int* height,
                            const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                            int* status);

/* Animations from clips: slice i * T + t of src (T = frames_per_item; the lp_frame_tensor of lp_xbatch_decode_clips,
 * n * T slices; with nchw an N x T x C x H x W tensor) holds frame t of item i at its top-left, width[i] x height[i]
 * (every frame of an item has that size).  Frames 0 .. nframes[i] - 1 are used; later slots are not read.  Frames are
 * converted as lp_xbatch_encode_frames converts them.
 *   - nframes[i] == 1: the item is the lp_xbatch_encode_frames item of slice i * T (same status and bytes); its
 *     duration is ignored
 *   - nframes[i] >= 2: status and bytes are those of lp_transform(A_i, opt, out[i], out_cap, ..., max_size), where A_i
 *     is an animated WebP of width[i] x height[i]: a VP8X chunk with the animation flag (and the alpha flag exactly
 *     when channels == 4), an ANIM chunk with background 0xFFFFFFFF and loop_count, then nframes[i] ANMF chunks, each
 *     the whole canvas at 0, 0 with no blending and no disposal, lasting duration_ms[i * T + t], whose image is a
 *     lossless VP8L frame that keeps every value (colour under alpha 0 included)
 *   - nframes[i] outside 1..T, width[i] or height[i] outside 1..box, or (nframes[i] >= 2) a duration of a used frame
 *     outside 0..0xFFFFFF: that item gets LP_ERR_BAD_ARGUMENT and out_len 0; the others go on
 * The tensor's contents must be complete before the call; the call only reads the tensor.  LP_ERR_BAD_ARGUMENT, with
 * nothing written, for: the tensor checks of lp_xbatch_decode_frames with n * T slices; T outside
 * 1..LP_XBATCH_MAX_CLIP_FRAMES; loop_count outside 0..65535; n < 0; a null opt / nframes / width / height /
 * duration_ms / out / out_len / status with n > 0.
 * Stats: grid_items / fallback_items count items; ms_decode is the unpack; h2d_bytes carries no pixels (the item table
 * only); d2h_bytes is the files.  lp_xbatch_encode_frames is this call with T = 1. */
int lp_xbatch_encode_clips(lp_xbatch* x, const lp_frame_tensor* src, int n, int frames_per_item, const int* nframes,
                           const int* width, const int* height, const int* duration_ms, int loop_count,
                           const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                           int* status);

/* ---- the same call over several GPUs of one node (SURVEY 8(e): shard by image index, no collective) ----
 * One lp_xbatch per device behind one call: the batch is cut into contiguous blocks balanced by compressed bytes,
 * every block runs on its own GPU from its own host thread, results land in the caller's arrays by index. */
typedef struct lp_multi lp_multi;
lp_multi* lp_multi_create(const int* devices, int n_devices, const lp_xbatch_config* config_template);
void lp_multi_destroy(lp_multi* m);
int lp_multi_device_count(const lp_multi* m);
int lp_multi_transform(lp_multi* m, const uint8_t* const* in, const size_t* in_len, int n,
                       const lp_image_options* opt, uint8_t* const* out, size_t out_cap, size_t* out_len,
                       int* status);
/* lp_xbatch_transform_renditions over the devices: sharded by item, so all renditions of an item run on one GPU. */
int lp_multi_transform_renditions(lp_multi* m, const uint8_t* const* in, const size_t* in_len, int n,
                                  const lp_image_options* opts, int k, uint8_t* const* out, size_t out_cap,
                                  size_t* out_len, int* status);
void lp_multi_get_stats(const lp_multi* m, int device_index, lp_xbatch_stats* out);
/* Host-only: the block boundaries lp_multi_transform uses (first[0..parts], contiguous, balanced by bytes). */
void lp_shard_blocks(const size_t* in_len, int n, int parts, int* first);

/* ---- single stages on device pointers, on `stream` (a cudaStream_t) -------- */

/* Batched crop + INTER_AREA resize of `n` packed u8 images that share one
 * geometry (ref opencv.cpp:196-215 on a opencv_mat_crop view).  src image i
 * starts at src + i*src_image_stride, rows are src_row_stride bytes apart.
 * Bit-exact to OpenCV 4.11 cv::resize(INTER_AREA) (SURVEY.md Appendix E.1/E.5). */
int lp_resize_area_dev(const uint8_t* src, size_t src_image_stride, size_t src_row_stride,
                       int channels, int crop_x, int crop_y, int crop_w, int crop_h, uint8_t* dst,
                       size_t dst_image_stride, size_t dst_row_stride, int dst_w, int dst_h, int n,
                       void* stream);

/* Batched baseline-JPEG encode of device frames into device memory (ref opencv.cpp:185-194
 * per image).  out_len[i] = 0 when image i did not fit in out_cap. */
int lp_jpeg_encode_dev(const uint8_t* frames, size_t frame_img_stride, size_t frame_row_stride,
                       int width, int height, int channels, int quality, int n, uint8_t* out,
                       size_t out_cap, uint32_t* out_len, void* stream);

/* Batched PNG encode of `n` packed device frames of one geometry (BGR / BGRA / Gray) into device memory, as lp_xbatch's
 * ".png" sink runs it: file i, complete (signature to IEND), at d_files + i*slot; d_len[i] = 0 when it did not fit.
 * level: zlib level 0..9; adaptive != 0: libpng's adaptive filter choice, else Sub on every row. */
int lp_png_encode_batch_dev(const uint8_t* d_frames, size_t img_stride, size_t row_stride, int width, int height,
                            int channels, int n, int level, int adaptive, uint8_t* d_files, size_t slot,
                            uint32_t* d_len);
/* Batched lossless WebP encode of `n` packed device BGR / BGRA frames of one geometry, as lp_xbatch's lossless ".webp"
 * sink and the per-image WebP writer run it: the "VP8L" payload of frame i is copied to payloads + offsets[i],
 * lengths[i] bytes long (payloads back to back).  part_bytes: bound on the packed output of one part of the call
 * (0 = the library's 1 GiB); a call over it is encoded in parts with the same bytes.  LP_ERR_BUF_TOO_SMALL when the
 * payloads do not fit payloads_cap. */
int lp_webp_lossless_encode_batch_dev(const uint8_t* d_frames, size_t img_stride, size_t row_step, int width, int height,
                                      int channels, int n, size_t part_bytes, uint8_t* payloads, size_t payloads_cap,
                                      size_t* offsets, size_t* lengths);
/* CRC-32 and Adler-32 of `n` bytes of device memory by the PNG encoder's device arithmetic (a warp per 32 KB piece,
 * pieces folded by the rules of csrc/crc32_core.h): for tests against zlib. */
int lp_png_checksums_dev(const uint8_t* d_data, size_t n, uint32_t* crc32, uint32_t* adler32);

/* Library-owned device/pinned memory helpers so tests and bench need no torch. */
void* lp_dev_alloc(size_t bytes);
void lp_dev_free(void* p);
void* lp_host_alloc_pinned(size_t bytes);
void lp_host_free_pinned(void* p);
int lp_memcpy_h2d(void* dst, const void* src, size_t bytes);
int lp_memcpy_d2h(void* dst, const void* src, size_t bytes);
int lp_dev_synchronize(void);
int lp_set_device(int device);
/* Time `iters` launches of fn-like stage: see bench.py (uses CUDA events). */
int lp_resize_area_time_dev(const uint8_t* src, size_t src_image_stride, size_t src_row_stride,
                            int channels, int crop_x, int crop_y, int crop_w, int crop_h,
                            uint8_t* dst, size_t dst_image_stride, size_t dst_row_stride,
                            int dst_w, int dst_h, int n, int iters, float* ms_per_iter);
#endif /* !LP_REFERENCE_BACKEND */

#ifdef __cplusplus
}
#endif
#endif
