// kernels.cuh -- internal launch interfaces between the translation units of
// liblilliput_b200.  Everything here takes DEVICE pointers and a stream.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <vector>

#include "jpeg_types.h"

namespace lp {

// ---- resize.cu ---------------------------------------------------------------------------
struct ResizeArgs {
    const uint8_t* src;
    size_t src_img_stride, src_row_stride;
    int channels;
    int crop_x, crop_y, crop_w, crop_h;
    uint8_t* dst;
    size_t dst_img_stride, dst_row_stride;
    int dst_w, dst_h;
    int n;
    int interpolation;  // 1 = INTER_LINEAR, 2 = INTER_CUBIC, 3 = INTER_AREA
    // device, n entries, or nullptr: image j of the launch reads src image index[j] and writes dst image index[j]
    // (INTER_AREA and INTER_LINEAR only)
    const int* index = nullptr;
};
int resize_launch(const ResizeArgs& a, cudaStream_t st);

// ---- jpeg_parse.cpp (host) -----------------------------------------------------------------
struct JpegComp {
    int id, h, v, tq, td, ta;
};
struct JpegHeader {
    int width = 0, height = 0, ncomp = 0;
    JpegComp comp[3];
    int maxh = 1, maxv = 1;
    uint16_t qt[4][64];  // natural order
    bool qt_present[4] = {false, false, false, false};
    uint8_t huff_bits[2][4][17];  // [class][id][len]
    uint8_t huff_vals[2][4][256];
    bool huff_present[2][4] = {{false, false, false, false}, {false, false, false, false}};
    int restart_interval = 0;
    int orientation = 1;
    size_t scan_offset = 0;  // first entropy-coded byte
    size_t scan_length = 0;  // bytes available from scan_offset (upper bound)
    bool progressive = false;
    bool supported = false;  // baseline/extended sequential Huffman, 8-bit, 1 or 3 comps, one scan
    bool multiscan = false;  // progressive, or sequential with one scan per component: serial device path
    int mcus_x = 0, mcus_y = 0;
};
// Parses markers up to and including the first SOS.  Returns 0, or a negative lp_status.
int jpeg_parse_header(const uint8_t* data, size_t len, JpegHeader* out);


// ---- jpeg_decode.cu ------------------------------------------------------------------------

// Fills the ROI / window / layout fields of `it` (whose width, height, ncomp, h, v, mcus_* are set)
// for the pixel window [x0,x1) x [y0,y1).  align16 rounds the window's x range outwards to 16 px so
// the vectorised colour step can use 16-byte stores.  Returns blocks in the ROI; *tiles (if given) = the CTAs
// jpeg_idct_color_kernel runs for the image.
uint32_t jpeg_item_set_window(JpegDecodeItem* it, int x0, int y0, int x1, int y1, bool align16,
                              uint32_t* tiles);
// Row stride of a decoded window [win_x0, win_x0 + win_w) of a `width`-pixel frame with `channels` bytes per pixel: a
// 16-byte multiple, except that whole rows are packed.
inline uint32_t jpeg_window_row_bytes(int win_x0, int win_w, int width, int channels) {
    if (win_x0 == 0 && win_w == width) return (uint32_t)win_w * channels;
    return (uint32_t)(((size_t)win_w * channels + 15) / 16 * 16);
}

void jpeg_build_huff_set(const JpegHeader& h, JpegHuffSet* out);
// Walks every SOS of a multi-scan file, snapshotting the Huffman tables / restart interval in force.
// `scans` is a caller array of max_scans entries; each new set of tables in force is copied into `sets` (a header
// whose huff_* fields hold them; nullptr: only counted) and numbered in JpegScanDesc::table_set from 0.  Returns 0
// or a negative lp_status.
int jpeg_parse_scans(const uint8_t* data, size_t len, const JpegHeader& h, JpegScanDesc* scans, int max_scans,
                     int* nscans, JpegHeader* sets, int max_sets, int* nsets);
// The same, with the sets built into device-format tables.
int jpeg_parse_scans(const uint8_t* data, size_t len, const JpegHeader& h, JpegScanDesc* scans, int max_scans,
                     int* nscans, JpegHuffSet* sets, int max_sets, int* nsets);
// The one interleaved scan of a `supported` header as a multi-scan descriptor, tables jpeg_build_huff_set(h) as set 0.
// Its bytes are the header's extent, up to the last EOI, where jpeg_parse_scans' stops at the first marker that is not
// RSTn: the per-image decode's search for the next RSTn (br_restart) may look past a first EOI.
void jpeg_baseline_scan(const JpegHeader& h, JpegScanDesc* out);
// Per-file caps of jpeg_parse_scans' arrays, and the work budget of the serial multi-scan decoder: one thread
// walks every block of every scan, so a hostile file (up to 256 scans over a large frame) is refused rather than
// queued.  Real progressive files have ~10 scans; an 8192 x 8192 4:4:4 frame with 20 scans still passes.
constexpr int kMultiscanMaxScans = 256, kMultiscanMaxSets = 64;
constexpr size_t kMultiscanMaxVisits = (size_t)1 << 26;
// Block visits of all scans of a multi-scan file.
size_t jpeg_multiscan_visits(const JpegHeader& h, const JpegScanDesc* scans, int nscans);

struct JpegDecodeBatch {
    JpegDecodeItem* items;      // device
    const JpegHuffSet* tables;  // device
    const uint8_t* scan;        // device, concatenated entropy-coded segments
    int16_t* coef;              // device
    uint8_t* frames;            // device, packed BGR / gray frames
    int n;
    int max_tiles_per_image;    // largest *tiles of jpeg_item_set_window over the batch
    // parallel Huffman scratch (all device); used when the batch holds a single-scan item
    uint8_t* clean = nullptr;
    void* states = nullptr;      // SubState[]
    uint32_t* nslots = nullptr;
    int16_t* dcdiff = nullptr;   // DC differences of ALL blocks of an image, MCU order
    // multi-scan items (JpegDecodeItem::nscans > 0): one thread walks each one's scans (jpeg_scan_core.h); `scan`
    // holds their whole files, `scans` their scan descriptors, `masks` the nonzero masks of blocks outside the
    // region of interest (nullptr when every such item decodes its whole frame)
    int n_multiscan = 0;
    const JpegScanDesc* scans = nullptr;
    uint64_t* masks = nullptr;
    // images with restart markers inside a parallel-Huffman launch: (image, interval) work list (device), one
    // thread per restart interval; their marker offsets live in `nslots` at the image's state_off, the number of
    // intervals the host expects in clean_len
    const uint2* rst_work = nullptr;
    int n_rst_work = 0;
};
// Scratch sizing for the parallel Huffman path, per image with `scan_len` entropy-coded bytes.
inline size_t huff_clean_bytes(size_t scan_len) { return ((scan_len + 48 + 15) / 16) * 16; }
inline size_t huff_nsub(size_t scan_len) { return scan_len * 8 / 1024 + 2; }
struct JpegHuffParallelArgs {
    JpegDecodeItem* items;
    const JpegHuffSet* tables;
    const uint8_t* scan;
    uint8_t* clean;
    void* states;
    uint32_t* nslots;
    int16_t* coef;
    int16_t* dcdiff;
    int n;
};
int jpeg_huff_parallel_launch(const JpegHuffParallelArgs& a, cudaStream_t st);
// Images the sync kernel can keep resident at once (SMs x CTAs per SM); chunk sizes that are a
// multiple of this avoid a mostly-empty last wave.
int jpeg_huff_parallel_slots();
// Diagnostics: clock64 cycles per phase of the sync kernels summed over CTAs (see jpeg_huff_parallel.cu)
int jpeg_huff_phase_clocks(unsigned long long out[8], int reset);
// Launches: huffman decode (each decoder clears the blocks it writes) -> fused idct + upsample + colour.
int jpeg_decode_launch(const JpegDecodeBatch& b, cudaStream_t st, cudaEvent_t ev_after_huff);

// ---- png_parse.cpp (host) / png_decode.cu ------------------------------------------------------
struct PngSegment {
    size_t offset, length;  // an IDAT payload inside the file
};
struct PngHeader {
    int width = 0, height = 0, bit_depth = 0, color_type = 0, interlace = 0;
    int src_channels = 0, out_channels = 0, bpp = 1;
    size_t row_bytes = 0;  // filtered scanline without the filter-type byte
    int npal = 0, ntrns = 0;
    bool has_trns = false;
    uint8_t palette[256 * 3] = {0};
    uint8_t trns[256] = {0};
    uint16_t trns_rgb[3] = {0, 0, 0};
    std::vector<PngSegment> idat;
    size_t idat_total = 0;
    int orientation = 1;  // from an eXIf chunk in front of the first IDAT (OpenCV reads it like a JPEG's EXIF block)
};
// EXIF orientation of a TIFF block, read the way the reference's OpenCV reads it (jpeg_parse.cpp)
bool exif_orientation_opencv(const uint8_t* tiff, size_t n, int* value);
int png_parse(const uint8_t* data, size_t len, PngHeader* out);
int png_extract_icc(const uint8_t* data, size_t len, uint8_t* dest, size_t dest_len);
// cICP code points (primaries, transfer, matrix, full range) of the chunk libpng would report; 1 if found
int png_extract_cicp(const uint8_t* data, size_t len, uint8_t* out4);

// One PNG to decode (array in HBM).  zoff: the concatenated IDAT payload (one zlib stream);
// raw: (row_bytes+1)*height bytes of filtered scanlines, defiltered in place; frame: packed output.
struct PngDecodeItem {
    uint64_t z_off, raw_off, frame_off;
    uint32_t z_len;
    int32_t width, height, bit_depth, color_type, src_channels, out_channels, bpp;
    uint32_t row_bytes, frame_stride;
    int32_t npal, ntrns, has_trns;
    uint16_t trns_rgb[3];
    uint16_t pad_;
    uint8_t palette[256 * 3];
    uint8_t trns[256];
    int32_t status;  // 0 ok, <0 corrupt stream
    uint32_t produced;
    // Adam7 (PNG spec s.8.2): the inflated stream is up to seven reduced images back to back, each
    // with its own scanline length.  A non-interlaced image is one "pass" covering everything.
    int32_t interlace, npass;
    uint32_t raw_total;               // inflated bytes expected
    uint32_t pass_off[7], pass_rb[7];  // byte offset / scanline bytes (without the filter byte)
    int32_t pass_w[7], pass_h[7];
};
// Fills npass / raw_total / pass_* from width, height, bit depth, channels, interlace.
void png_item_set_passes(PngDecodeItem* it);
struct PngDecodeBatch {
    PngDecodeItem* items;  // device
    const uint8_t* z;      // device: zlib streams
    uint8_t* raw;          // device
    uint8_t* frames;       // device
    int n;
    int max_width, max_height;
};
// inflate -> defilter -> convert to packed Gray / BGR / BGRA u8.
int png_decode_launch(const PngDecodeBatch& b, cudaStream_t st);
// the two halves, for callers that keep every stream's scanlines but only a window of frames (xbatch.cu)
int png_inflate_launch(const PngDecodeBatch& b, cudaStream_t st);
int png_unfilter_launch(const PngDecodeBatch& b, int first, int count, cudaStream_t st);

// ---- png_encode.cu ---------------------------------------------------------------------------
// zlib level and filter policy of a PNG file from OpenCV's flat encode options (key, value, ...): PngCompression given ->
// that level clamped to 0..9 with libpng's adaptive filters; absent -> level 1, Sub on every row (grfmt_png.cpp).
void png_encode_policy(const int* opt, size_t opt_len, int* level, bool* adaptive_filters);
// The largest file a frame can become (every DEFLATE chunk stored): a slot of this size always fits.
size_t png_encode_max_file_bytes(int width, int height, int channels);
// n packed device frames of one geometry (frame i at d_frames + i * img_stride) -> n complete PNG files on the device:
// file i at d_files + i * slot, d_len[i] its length, 0 when it does not fit `slot`.  Filter, DEFLATE, Adler-32, the
// chunk CRCs and the container are all written by the three kernels; `scratch` (device, png_encode_batch_scratch_bytes)
// is the caller's, so nothing is allocated here.
size_t png_encode_batch_scratch_bytes(int width, int height, int channels, int n, int level);
int png_encode_batch(const uint8_t* d_frames, size_t img_stride, size_t row_stride, int width, int height, int channels,
                     int n, int level, bool adaptive_filters, uint8_t* d_files, size_t slot, uint32_t* d_len, void* scratch,
                     cudaStream_t st);
// One packed device frame -> a complete PNG file in host memory: png_encode_batch with n = 1.
int png_encode_frame(const uint8_t* frame, size_t row_stride, int width, int height, int channels, int level,
                     bool adaptive_filters, std::vector<uint8_t>* out, cudaStream_t st);

// ---- jpeg_encode.cu ------------------------------------------------------------------------
struct JpegEncodeBatch {
    const uint8_t* frames;  // device packed frames
    size_t frame_img_stride, frame_row_stride;
    int width, height, channels;  // shared by the batch
    int quality;
    int n;
    uint8_t* out;            // device, n * out_cap
    size_t out_cap;
    uint32_t* out_len;       // device, n (0 on overflow)
    // scratch (device), sized by jpeg_encode_scratch_bytes
    void* scratch;
    // progressive output (libjpeg-turbo's jpeg_simple_progression script, optimal tables per scan)
    bool progressive = false;
    // device, n entries, or nullptr: image j of the launch reads frame index[j] and writes out slot / out_len index[j]
    const int* index = nullptr;
};
size_t jpeg_encode_scratch_bytes(int width, int height, int channels, int n, size_t out_cap, bool progressive = false);
int jpeg_encode_launch(const JpegEncodeBatch& b, cudaStream_t st, cudaEvent_t ev_after_transform);

// ---- webp_encode.cu -------------------------------------------------------------------------
struct WebpEncodedFrame {
    std::vector<uint8_t> image;  // "VP8 " or "VP8L" payload
    std::vector<uint8_t> alph;   // "ALPH" payload (lossy frames with transparency)
    bool lossless = false, has_alpha = false;
    int width = 0, height = 0, duration = 0;
};
// n packed device frames of one geometry (frame i at d_frames + i*img_stride) -> lossy VP8 payloads (+ ALPH for
// frames with transparency), ref webp.cpp:711-729 / 650-700 per frame.
int webp_encode_lossy_batch(const uint8_t* d_frames, size_t img_stride, size_t row_step, int width, int height,
                            int channels, int n, int quality, std::vector<WebpEncodedFrame>* out, cudaStream_t st);
// Device bytes webp_encode_lossy_batch allocates for n frames of one geometry (its scratch, outside any arena)
size_t webp_encode_lossy_scratch_bytes(int width, int height, int channels, int n);
void webp_assemble(const WebpEncodedFrame* frames, int n, const uint8_t* icc, size_t icc_len, uint32_t bgcolor,
                   uint32_t loop_count, std::vector<uint8_t>* file);

// ---- batch helpers of webp_decode.cu / gif_decode.cu (used by xbatch.cu) ------------------------
// A WebP file as the per-image decoder (webp_decoder_*) sees it: spans inside the file, frame properties as
// webp_decoder_get_prev_frame_* report them, background / loop count as webp_decoder_create normalises them.
struct WebpFramePlan {
    size_t img_off = 0, img_len = 0;    // "VP8 " / "VP8L" payload (with the RIFF padding byte, as decoded per image)
    size_t alph_off = 0, alph_len = 0;  // "ALPH" payload, when has_alph
    bool lossless = false, has_alph = false;
    int x = 0, y = 0, width = 0, height = 0;
    int duration = 0;
    int dispose = 0;  // 1 = dispose to background (clear the rectangle after the frame)
    int blend = 0;    // 1 = do not blend (copy the rectangle)
};
struct WebpPlan {
    int width = 0, height = 0, channels = 3;  // canvas; 4 when the container has the alpha flag
    bool animated = false;                    // the container's animation flag
    uint32_t bgcolor = 0xFFFFFFFFu, loop_count = 0;
    size_t icc_off = 0, icc_len = 0;          // ICCP payload (icc_len 0: none)
    std::vector<WebpFramePlan> frames;
};
bool webp_plan_parse(const uint8_t* data, size_t len, WebpPlan* out);
// device scratch webp_decode_batch lays out for one plan (uploaded file, VP8 work areas, lossless pixels, alpha planes,
// job records), not counting the shared VP8L arena
size_t webp_plan_device_bytes(const WebpPlan& p, size_t file_len);
// the VP8L arena all lossless / ALPH streams of a plan need to run in one wave (the per-image decoder's bound each)
size_t webp_plan_arena_bytes(const WebpPlan& p);
// decodes + composites every frame of `n` WebP files: file a's composited canvas f (plan width x height x channels,
// round_up(w * h * ch, 256) apart) lands at d_canvases + canvas_off[a] + f * that stride.  Lossless frames and ALPH
// planes decode in waves of streams whose arena slices fit d_arena.  h_status per file: 0, or the frame failed.
// ev_uploaded (optional) is recorded once the files are on the device.
int webp_decode_batch(const WebpPlan* const* plans, const uint8_t* const* files, const size_t* file_len, int n,
                      uint8_t* d_scratch, size_t scratch_bytes, uint8_t* d_arena, size_t arena_bytes, uint8_t* d_canvases,
                      const uint64_t* canvas_off, int* h_status, cudaEvent_t ev_uploaded, cudaStream_t st);
struct GifAnimPlan;
GifAnimPlan* gif_plan_parse(const uint8_t* data, size_t len, int max_frames);
void gif_plan_free(GifAnimPlan* p);
void gif_plan_info(const GifAnimPlan* p, int* width, int* height, int* nframes, uint32_t* bgcolor, int* loop_count);
int gif_plan_delay_ms(const GifAnimPlan* p, int frame);
size_t gif_plan_device_bytes(const GifAnimPlan* p);
// decodes + composites every frame of `n` animations of one canvas size: animation a, frame f lands at
// d_canvases + (first_frame[a] + f) * canvas_stride (BGRA); h_status per animation
int gif_decode_batch(GifAnimPlan* const* plans, const uint8_t* const* files, const size_t* file_len, int n,
                     uint8_t* d_scratch, size_t scratch_bytes, uint8_t* d_canvases, size_t canvas_stride,
                     const int* first_frame, int* h_status, cudaStream_t st);
// device scratch gif_encode_batch needs for one animation whose frames are resized to ow x oh
size_t gif_plan_encode_bytes(const GifAnimPlan* p, int ow, int oh);
// GIF files of `n` animations whose frames, resized to ow x oh BGRA, sit at d_frames + (first_frame[a] + f) * frame_stride:
// palette mapping + LZW of every frame (device), container assembly into out[a] (host), status and out_len per
// animation as lp_transform reports them.  h_stage: pinned staging for the code streams.
int gif_encode_batch(GifAnimPlan* const* plans, int n, const uint8_t* d_frames, size_t frame_stride, int ow, int oh,
                     const int* first_frame, uint8_t* d_scratch, size_t scratch_bytes, uint8_t* h_stage, size_t stage_bytes,
                     uint8_t* const* out, size_t out_cap, size_t* out_len, int* status, size_t* d2h, cudaStream_t st);

// ---- pixel_ops.cu --------------------------------------------------------------------------
int orient_launch(const uint8_t* src, int w, int h, int channels, int orientation, uint8_t* dst,
                  cudaStream_t st);
// EXIF orientation o of a w x h frame (golden table SURVEY.md 8a R4; values outside 2..8 are the identity): the source
// pixel that lands at (x, y) of the oriented frame.
__host__ __device__ inline void orient_source_pixel(int o, int w, int h, int x, int y, int* sx, int* sy) {
    switch (o) {
        case 2: *sx = w - 1 - x; *sy = y; break;
        case 3: *sx = w - 1 - x; *sy = h - 1 - y; break;
        case 4: *sx = x; *sy = h - 1 - y; break;
        case 5: *sx = y; *sy = x; break;
        case 6: *sx = y; *sy = h - 1 - x; break;
        case 7: *sx = w - 1 - y; *sy = h - 1 - x; break;
        case 8: *sx = w - 1 - y; *sy = x; break;
        default: *sx = x; *sy = y; break;
    }
}
// One item of orient_crop_launch: the crop [cx, cx+cw) x [cy, cy+ch) of the oriented frame, read from a decoded window
// of the w x h source (window origin win_x0, win_y0; rows src_stride bytes apart, starting at src_off) and written
// packed (rows cw * channels bytes apart) at dst_off.
struct OrientJob {
    uint64_t src_off, dst_off;
    uint32_t src_stride;
    int32_t o, cx, cy, cw, ch, win_x0, win_y0;
};
// n jobs on frames of `channels` (3: BGR, 1: gray) of one w x h source; max_cw / max_ch bound every job's crop.
// 32 x 32 tiles staged in shared memory, so the transposing orientations read and write whole rows too.
int orient_crop_launch(const OrientJob* d_jobs, int n, const uint8_t* src, uint8_t* dst, int w, int h, int channels,
                       int max_cw, int max_ch, cudaStream_t st);
int copy_region_launch(const uint8_t* src, size_t src_step, int src_ch, uint8_t* dst,
                       size_t dst_step, int dst_ch, int w, int h, cudaStream_t st);
// ---- tonemap.cu ----------------------------------------------------------------------------
int tonemap_to_sdr_launch(uint8_t* d_px, size_t step, int channels, int w, int h, int transfer, int primaries, cudaStream_t st);

int compact_launch(const uint8_t* src, size_t stride, const uint32_t* len, uint32_t cap, int n, uint8_t* dst,
                   unsigned long long* off /* n + 1 */, cudaStream_t st);
struct SegCopy {
    uint64_t src, dst;  // byte offsets from one base pointer
    uint32_t len, pad_;
};
int seg_copy_launch(const SegCopy* d_segs, int n, uint8_t* base, cudaStream_t st);
int blend_region_launch(const uint8_t* src, size_t src_step, int src_ch, uint8_t* dst,
                        size_t dst_step, int dst_ch, int w, int h, cudaStream_t st);

}  // namespace lp
