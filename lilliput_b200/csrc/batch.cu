// batch.cu -- the additive batch entry points (include/lilliput_b200.h): N independent JPEGs (baseline, restart
// interval, optimised tables, progressive or one scan per component) -> Fit / area resize -> JPEG, every stage one
// grid launch over a chunk of the batch.
//
// Multi-scan files decode side by side in one extra launch per chunk (jpeg_multiscan_kernel, one thread walking the
// scans of each file) into the same scan-order coefficient layout as the parallel decoders, so the rest of the chunk
// is unchanged.  Their scan descriptors and Huffman table sets live in batch-wide pools sized by max_images:
//   scans      kScansPerImage per image + kMultiscanMaxScans (one file's cap)
//   table sets one per image (single-scan files) + kSetsPerImage per image + kMultiscanMaxSets (one file's cap)
// libjpeg-turbo's progressive files have 10 scans and up to 9 distinct optimised table sets, so a batch made only
// of them fits.  A file that overflows a pool gets LP_ERR_UNSUPPORTED (as the restart-marker scratch does).
//
// Per-item semantics are those of ImageOps.Transform (ref ops.go:352-444) for a still JPEG with
// ImageOpsFit/ImageOpsResize and ".jpeg" output: decode (ref opencv.cpp:166), OrientationTransform (ref ops.go:392),
// Framebuffer.Fit crop + INTER_AREA (ref opencv.go:326-374), encode (ref opencv.cpp:185).
// Images are independent; nothing is exchanged between them or between GPUs.
//
// EXIF orientation (contexts made by lp_batch_create).  The items of a chunk fall into three classes:
//   0  orientation 1 (and the values Transform ignores): resized from the decoded window, as if nothing else existed
//   1  orientations 2..4 keep the axes: class 0's output size and crop, read mirrored in the source
//   2  orientations 5..8 swap them: the frame is H x W, its output size and crop are the H x W frame's
// Every item decodes only the pre-image of its oriented crop (an axis-aligned rectangle under all eight orientations);
// one launch turns the rotated items' windows into their oriented crops, packed, and each class present is resized
// (and class 2, when its size differs, encoded) through an image map, so results stay at the caller's item index.
// A chunk without rotated items launches exactly what it did before orientation was taken.
//
// Gray sources (contexts made by lp_batch_create).  A one-component file is decoded into a 1-channel window, oriented,
// resized and encoded on one channel, as Transform does, next to the colour items of its chunk.  The channel count
// is a per-item property beside the orientation class, so a chunk has up to six sub-classes, in the order of its image
// map: colour classes 0, 1, 2, then gray classes 0, 1, 2.  Each sub-class present gets one resize launch, each channel
// count with rotated items one orientation launch, each (channel count, output size) present one encode.  Slots (decoded
// window, oriented crop, resized frame) stay sized and spaced for three channels: a gray item's rows are packed at the
// start of its slot and take a third of it, and the encoder scratch is the colour geometry's (the larger), so taking
// gray files allocates nothing.  A chunk with no gray item launches exactly what it launched before gray was taken, with
// the same strides and slot layout; a chunk of unrotated gray items only launches without an image map, like a chunk of
// unrotated colour items.
#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <thread>
#include <unordered_map>
#include <utility>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"
#include "lilliput_host.hpp"

using namespace lp;

static constexpr int kScansPerImage = 16, kSetsPerImage = 10;

namespace lp {
// Device bytes of the multi-scan pools of a context for max_images = n (what batch_create_in adds for them besides
// the per-slot masks).
size_t batch_multiscan_pool_bytes(size_t n) {
    return ((kSetsPerImage * n + kMultiscanMaxSets) * sizeof(JpegHuffSet) +
            (kScansPerImage * n + kMultiscanMaxScans) * sizeof(JpegScanDesc));
}
}  // namespace lp

struct lp_batch {
    lp_batch_config cfg;
    bool progressive = false;        // JPEG output is progressive (lp_xbatch with JpegProgressive)
    bool multiscan = true;           // takes multi-scan sources (lp_xbatch groups of single-scan files do not)
    bool resize_only = false;        // lp_xbatch's WebP and PNG sinks: the chunk ends with the resized frames (no JPEG encode)
    bool orient = false;             // takes EXIF-rotated sources (lp_batch_create; lp_xbatch hands them to lp_transform)
    bool gray = false;               // takes one-component sources (lp_batch_create; lp_xbatch hands them to lp_transform)
    size_t arena_dev_used = 0, arena_host_used = 0;  // bytes carved from the caller's arenas (batch_create_in)
    cudaStream_t st = nullptr;       // kernels
    cudaStream_t st_h2d = nullptr;   // input copies (pipelined transform)
    cudaStream_t st_d2h = nullptr;   // output copies (pipelined transform)
    int chunk = 0, max_chunks = 0;
    int first_chunk = 0;  // pipelined path: size of the opening chunk (one wave of Huffman CTAs)
    int pipe_chunk = 0;   // pipelined path: size of the following chunks
    // Huffman tables of the last file seen (fast path of table_set_for)
    int last_table_idx = -1;
    bool last_present[2][4];
    uint8_t last_bits[2][4][17];
    uint8_t last_vals[2][4][256];
    // geometry (fixed by cfg)
    int W = 0, H = 0, out_w = 0, out_h = 0;
    int crop_x = 0, crop_y = 0, crop_w = 0, crop_h = 0;
    // items whose orientation swaps the axes (class 2): output size, and crop in the oriented H x W frame
    int out_w2 = 0, out_h2 = 0;
    int crop2_x = 0, crop2_y = 0, crop2_w = 0, crop2_h = 0;
    size_t oriented_bytes = 0;  // slot stride of d_oriented: the larger of the two classes' packed crops
    // resize-only contexts with several outputs: each decoded window (the union of their crops, in crop_*) is resized
    // into every geometry; geometry g's frames are at d_resized + geom_off[g], g.out_w * g.out_h * 3 bytes apart
    std::vector<BatchGeom> geoms;
    std::vector<size_t> geom_off;
    // per-image scratch layout, fixed by the first image staged into this context
    bool layout_known = false;
    uint32_t blocks = 0;
    size_t max_blocks_alloc = 0;
    size_t frame_bytes = 0, resized_bytes = 0;
    uint32_t gray_row_bytes = 0;  // row stride of an unrotated gray item's decoded window
    // device
    uint8_t* d_scan = nullptr;
    JpegDecodeItem* d_items = nullptr;
    JpegHuffSet* d_tables = nullptr;
    int16_t* d_coef = nullptr;
    uint8_t* d_frames = nullptr;
    uint8_t* d_resized = nullptr;
    uint8_t* d_enc_scratch = nullptr;
    uint8_t* d_clean = nullptr;     // parallel Huffman: unstuffed bit strings (whole batch)
    void* d_states = nullptr;       // parallel Huffman: subsequence exit states
    uint32_t* d_nslots = nullptr;
    int16_t* d_dcdiff = nullptr;    // per chunk slot: DC differences of all blocks
    uint64_t* d_masks = nullptr;    // per chunk slot: nonzero masks of all blocks (multi-scan items, jpeg_scan_core.h)
    JpegScanDesc* d_scans = nullptr;  // scan descriptors of the batch's multi-scan files
    uint32_t total_blocks = 0;      // blocks of a whole image (dcdiff slot stride)
    int win_w = 0, win_h = 0;       // decoded pixel window (crop, x range aligned out to 16)
    int win_x0 = 0;
    uint8_t* d_out = nullptr;
    uint32_t* d_out_len = nullptr;
    uint8_t* d_oriented = nullptr;  // per chunk slot: a rotated item's oriented crop
    OrientJob* d_jobs = nullptr;    // per image: the rotated items of each chunk, from the chunk's first image
    int* d_index = nullptr;         // per image: each chunk's slots ordered by sub-class (the resize / encode image maps)
    // host
    std::vector<JpegDecodeItem> items;
    std::vector<JpegHuffSet> tables;
    std::unordered_map<std::string, int> table_index;  // every distinct Huffman table set of the batch (hashed)
    size_t tables_uploaded = 0;
    std::vector<JpegScanDesc> scans;  // multi-scan files: their scans, table_set indexing `tables`
    size_t scans_uploaded = 0;
    std::vector<int> parse_status;
    std::vector<size_t> file_dev_off;
    std::vector<OrientJob> jobs;
    std::vector<int> index;
    size_t dev_off = 0, clean_off = 0, state_off = 0;
    uint8_t* h_out = nullptr;       // pinned + device-mapped: the compaction kernel writes the encoded bytes straight into it
    uint32_t* h_out_len = nullptr;  // pinned
    unsigned long long* h_off = nullptr;  // pinned + device-mapped: packed offsets, (cnt + 1) per chunk at [i0 + chunk ordinal]
    struct ChunkLayout {
        uint32_t blocks = 0, tiles = 0, total_blocks = 0;
        int ordinal = 0;
        int n_multiscan = 0;
        size_t frame_stride = 0;        // decoded-window slot stride
        // items per sub-class (top of the file): colour orientation classes 0, 1, 2, then gray 0, 1, 2
        int n_class[6] = {0, 0, 0, 0, 0, 0};
        // whether the chunk launches through the image map: not when all of it is unrotated items of one channel count
        bool mapped(int cnt) const {
            return n_class[1] + n_class[2] + n_class[3] + n_class[4] + n_class[5] > 0 && n_class[3] != cnt;
        }
        std::vector<uint2> rst_work;  // (image in chunk, restart interval) of the chunk's DRI images
        uint2* d_rst_work = nullptr;  // stream-ordered allocation, freed after the chunk's launches
    };
    size_t state_cap = 0;  // entries of d_states / d_nslots
    std::map<int, ChunkLayout> chunk_layout;  // keyed by the chunk's first image
    JpegDecodeItem* h_items_back = nullptr;
    int n = 0;
    int last_launches = 0;
    std::vector<cudaEvent_t> ev;      // 6 per chunk (stage timing)
    std::vector<cudaEvent_t> ev_h2d;  // per chunk
    std::vector<cudaEvent_t> ev_d2h;  // per chunk
    int max_tables = 0;  // table-set pool (see the top of the file)
    size_t max_scans = 0;  // scan-descriptor pool
    bool owns_mem = true;  // false: device / pinned buffers were carved from a caller's arenas (xbatch.cu)
};

static void batch_free(lp_batch* b) {
    if (!b) return;
    for (auto& kv : b->chunk_layout)
        if (kv.second.d_rst_work) cudaFree(kv.second.d_rst_work);
    if (b->owns_mem) {
    cudaFree(b->d_scan); cudaFree(b->d_items); cudaFree(b->d_tables); cudaFree(b->d_coef);
    cudaFree(b->d_frames); cudaFree(b->d_resized); cudaFree(b->d_enc_scratch);
    cudaFree(b->d_out); cudaFree(b->d_out_len);
    cudaFree(b->d_clean); cudaFree(b->d_states); cudaFree(b->d_nslots); cudaFree(b->d_dcdiff);
    cudaFree(b->d_masks); cudaFree(b->d_scans);
    cudaFree(b->d_oriented); cudaFree(b->d_jobs); cudaFree(b->d_index);
    if (b->h_out) cudaFreeHost(b->h_out);
    if (b->h_out_len) cudaFreeHost(b->h_out_len);
    if (b->h_items_back) cudaFreeHost(b->h_items_back);
    if (b->h_off) cudaFreeHost(b->h_off);
    }
    for (auto e : b->ev) cudaEventDestroy(e);
    for (auto e : b->ev_h2d) cudaEventDestroy(e);
    for (auto e : b->ev_d2h) cudaEventDestroy(e);
    if (b->st) cudaStreamDestroy(b->st);
    if (b->st_h2d) cudaStreamDestroy(b->st_h2d);
    if (b->st_d2h) cudaStreamDestroy(b->st_d2h);
    delete b;
}

namespace lp {
lp_batch* batch_create_in(const lp_batch_config* cfg, uint8_t* dev_arena, size_t dev_bytes, uint8_t* host_arena,
                          size_t host_bytes, bool progressive_jpeg = false, bool multiscan_sources = true,
                          bool resize_only = false, bool oriented_sources = false, bool gray_sources = false,
                          const BatchGeom* geoms = nullptr, int n_geoms = 0);
int batch_resized_status(lp_batch* b, int* status);
const uint8_t* batch_resized_geom(const lp_batch* b, int g, size_t* image_stride);
void batch_arena_used(const lp_batch* b, size_t* dev_bytes, size_t* host_bytes);
}
extern "C" lp_batch* lp_batch_create(const lp_batch_config* cfg) {
    return lp::batch_create_in(cfg, nullptr, 0, nullptr, 0, false, true, false, true, true);
}

// dev_arena / host_arena non-null: every device / pinned buffer is carved from them (nothing is allocated or
// freed by the context); returns nullptr when they are too small.  progressive_jpeg: write progressive JPEG files.
// multiscan_sources: take multi-scan files (and allocate their pools and masks); otherwise they get
// LP_ERR_UNSUPPORTED.  resize_only: every chunk stops after the resize, so the context has no JPEG encoder scratch and
// no output slots; it is driven by lp_batch_stage + lp_batch_run, then batch_resized_status (lp_batch_transform and
// lp_batch_fetch refuse it), and the caller encodes the frames at lp_batch_resized_dev.  oriented_sources: take
// EXIF-rotated files (and allocate the oriented-crop buffers); otherwise they get LP_ERR_UNSUPPORTED.  gray_sources: take
// one-component files (they fit the colour slots: only the image map is allocated for them); otherwise they get
// LP_ERR_UNSUPPORTED.  geoms (n_geoms > 1, resize-only contexts of unrotated colour sources only): the outputs each
// decoded window is resized into, in place of cfg's one; the window decoded is the bounding box of their crops, and
// batch_resized_geom gives each one's frames.
lp_batch* lp::batch_create_in(const lp_batch_config* cfg, uint8_t* dev_arena, size_t dev_bytes, uint8_t* host_arena,
                              size_t host_bytes, bool progressive_jpeg, bool multiscan_sources, bool resize_only,
                              bool oriented_sources, bool gray_sources, const BatchGeom* geoms, int n_geoms) {
    if (!cfg || cfg->max_images < 1 || cfg->src_width < 1 || cfg->src_height < 1) return nullptr;
    if (n_geoms > 1 && (!geoms || !resize_only || oriented_sources || gray_sources)) return nullptr;
    if (ensure_device()) return nullptr;
    DeviceGuard dev_guard(cfg->device);
    if (!dev_guard.ok) return nullptr;
    lp_batch* b = new lp_batch;
    b->cfg = *cfg;
    b->progressive = progressive_jpeg;
    b->multiscan = multiscan_sources;
    b->resize_only = resize_only;
    b->orient = oriented_sources;
    b->gray = gray_sources;
    b->owns_mem = dev_arena == nullptr;
    size_t dev_used = 0, host_used = 0;
    b->W = cfg->src_width;
    b->H = cfg->src_height;
    if (cfg->resize_method == LP_OPS_FIT) {
        // ref ops.go:170-171 + opencv.go:331-363
        lilliput::calculateExpectedSize(b->W, b->H, cfg->dst_width, cfg->dst_height, &b->out_w, &b->out_h);
        lilliput::fitCropRect(b->W, b->H, b->out_w, b->out_h, &b->crop_x, &b->crop_y, &b->crop_w, &b->crop_h);
    } else if (cfg->resize_method == LP_OPS_RESIZE) {
        b->out_w = std::max(cfg->dst_width, 1);
        b->out_h = std::max(cfg->dst_height, 1);
        b->crop_w = b->W;
        b->crop_h = b->H;
    } else {
        delete b;
        return nullptr;
    }
    // class 2 (ref ops.go:449-470): the requested size is computed from the header's size, turned only under
    // NormalizeOrientation; Fit crops the oriented H x W frame, Resize takes all of it
    if (cfg->resize_method == LP_OPS_FIT) {
        if (cfg->normalize_orientation)
            lilliput::calculateExpectedSize(b->H, b->W, cfg->dst_width, cfg->dst_height, &b->out_w2, &b->out_h2);
        else
            lilliput::calculateExpectedSize(b->W, b->H, cfg->dst_width, cfg->dst_height, &b->out_w2, &b->out_h2);
        lilliput::fitCropRect(b->H, b->W, b->out_w2, b->out_h2, &b->crop2_x, &b->crop2_y, &b->crop2_w, &b->crop2_h);
    } else {
        b->out_w2 = b->out_w;
        b->out_h2 = b->out_h;
        b->crop2_w = b->H;
        b->crop2_h = b->W;
    }
    if (n_geoms > 1) {  // the decoded window: the bounding box of every output's crop
        b->geoms.assign(geoms, geoms + n_geoms);
        int x0 = b->W, y0 = b->H, x1 = 0, y1 = 0;
        for (const BatchGeom& g : b->geoms) {
            x0 = std::min(x0, g.crop_x);
            y0 = std::min(y0, g.crop_y);
            x1 = std::max(x1, g.crop_x + g.crop_w);
            y1 = std::max(y1, g.crop_y + g.crop_h);
        }
        b->crop_x = x0;
        b->crop_y = y0;
        b->crop_w = x1 - x0;
        b->crop_h = y1 - y0;
    }
    const int slots = jpeg_huff_parallel_slots();
    // default chunk: three full waves of the per-image Huffman CTAs (no mostly-empty tail wave; larger
    // launches for the bandwidth-bound kernels); the pipelined path opens with a single wave
    b->chunk = cfg->chunk > 0 ? cfg->chunk : (slots > 0 ? 3 * slots : 512);
    b->first_chunk = slots > 0 ? std::min(slots, b->chunk) : b->chunk / 2;
    // the pipelined host-buffer path prefers finer grains (what is exposed is the first upload and the last
    // download): two waves per chunk measured best there, three for the device-resident path
    b->pipe_chunk = (cfg->chunk > 0 || slots <= 0) ? b->chunk : std::min(b->chunk, 2 * slots);
    b->chunk = std::min(b->chunk, cfg->max_images);
    b->pipe_chunk = std::max(1, std::min(b->pipe_chunk, b->chunk));
    b->max_chunks = ceil_div(cfg->max_images, b->pipe_chunk) + 3;  // + the opening chunk of the pipelined path
    // worst-case per-image layout: 4:4:4 needs the most blocks
    const size_t mcus = (size_t)ceil_div(b->W, 8) * ceil_div(b->H, 8);
    b->max_blocks_alloc = mcus * 3 + 4 * ((size_t)ceil_div(b->W, 8) + ceil_div(b->H, 8)) + 16;
    const size_t max_blocks = b->max_blocks_alloc;
    b->frame_bytes = (size_t)b->W * b->H * 3;
    b->resized_bytes = (size_t)b->out_w * b->out_h * 3;
    if (b->orient) {
        // (the two output sizes differ only under NormalizeOrientation, so without it the stride is class 0's)
        b->resized_bytes = std::max(b->resized_bytes, (size_t)b->out_w2 * b->out_h2 * 3);
        b->oriented_bytes = round_up((size_t)std::max(b->crop_w * b->crop_h, b->crop2_w * b->crop2_h) * 3, (size_t)256);
    }
    const size_t N = cfg->max_images;
    auto fail = [&]() -> lp_batch* { batch_free(b); return nullptr; };
#define BALLOC(ptr, bytes)                                                                      \
    if (dev_arena) {                                                                            \
        const size_t need_ = round_up((size_t)(bytes), (size_t)256);                            \
        if (dev_used + need_ > dev_bytes) return fail();                                        \
        (ptr) = reinterpret_cast<decltype(ptr)>(dev_arena + dev_used);                          \
        dev_used += need_;                                                                      \
    } else if (cudaMalloc(&(ptr), (bytes)) != cudaSuccess) {                                    \
        fprintf(stderr, "[lilliput_b200] lp_batch_create: cudaMalloc(%zu) failed\n", (size_t)(bytes)); \
        return fail();                                                                          \
    }
#define HALLOC(ptr, bytes)                                                                      \
    if (host_arena) {                                                                           \
        const size_t need_ = round_up((size_t)(bytes), (size_t)256);                            \
        if (host_used + need_ > host_bytes) return fail();                                      \
        (ptr) = reinterpret_cast<decltype(ptr)>(host_arena + host_used);                        \
        host_used += need_;                                                                     \
    } else if (cudaMallocHost(&(ptr), (bytes)) != cudaSuccess) {                                \
        return fail();                                                                          \
    }
    if (cudaStreamCreateWithFlags(&b->st, cudaStreamNonBlocking) != cudaSuccess) return fail();
    if (cudaStreamCreateWithFlags(&b->st_h2d, cudaStreamNonBlocking) != cudaSuccess) return fail();
    if (cudaStreamCreateWithFlags(&b->st_d2h, cudaStreamNonBlocking) != cudaSuccess) return fail();
    BALLOC(b->d_scan, cfg->max_in_bytes + 16 * N + 4096);
    BALLOC(b->d_items, N * sizeof(JpegDecodeItem));
    b->max_tables = (int)N;  // single-scan files: one set each at most
    if (b->multiscan) {
        b->max_tables += (int)(kSetsPerImage * N) + kMultiscanMaxSets;
        b->max_scans = kScansPerImage * N + kMultiscanMaxScans;
        BALLOC(b->d_scans, b->max_scans * sizeof(JpegScanDesc));
        BALLOC(b->d_masks, (size_t)b->chunk * max_blocks * sizeof(uint64_t));
    }
    BALLOC(b->d_tables, (size_t)b->max_tables * sizeof(JpegHuffSet));
    BALLOC(b->d_coef, (size_t)b->chunk * max_blocks * 64 * sizeof(int16_t));
    // (a rotated item's window is at most the frame; its slots are 256-byte aligned)
    BALLOC(b->d_frames, (size_t)b->chunk * (b->orient ? round_up(b->frame_bytes, (size_t)256) : b->frame_bytes) + 256);
    if (b->geoms.empty()) {
        BALLOC(b->d_resized, N * b->resized_bytes + 256);
    } else {
        size_t all = 0;
        for (const BatchGeom& g : b->geoms) {
            b->geom_off.push_back(all);
            all += N * ((size_t)g.out_w * g.out_h * 3);
        }
        BALLOC(b->d_resized, all + 256);
    }
    if (!b->resize_only) {
        size_t enc = jpeg_encode_scratch_bytes(b->out_w, b->out_h, 3, b->chunk, cfg->out_cap, b->progressive);
        if (b->orient)
            enc = std::max(enc, jpeg_encode_scratch_bytes(b->out_w2, b->out_h2, 3, b->chunk, cfg->out_cap, b->progressive));
        for (int c = 0; c < (b->gray ? 2 : 0); c++)  // (colour is the larger but for rounding: six blocks per 16 x 16 pixels against four)
            enc = std::max(enc, jpeg_encode_scratch_bytes(c ? b->out_w2 : b->out_w, c ? b->out_h2 : b->out_h, 1, b->chunk,
                                                          cfg->out_cap, b->progressive));
        BALLOC(b->d_enc_scratch, enc);
    }
    if (b->orient) {
        BALLOC(b->d_oriented, (size_t)b->chunk * b->oriented_bytes);
        BALLOC(b->d_jobs, N * sizeof(OrientJob));
    }
    if (b->orient || b->gray) {
        BALLOC(b->d_index, N * sizeof(int));
    }
    BALLOC(b->d_clean, cfg->max_in_bytes + 64 * N + 4096);
    b->state_cap = (cfg->max_in_bytes / 128 + 2 * N + 16) * 2;
    BALLOC(b->d_states, b->state_cap * 8);
    BALLOC(b->d_nslots, b->state_cap * 4);
    BALLOC(b->d_dcdiff, (size_t)b->chunk * max_blocks * sizeof(int16_t));
    if (!b->resize_only) {
        BALLOC(b->d_out, N * cfg->out_cap);
        BALLOC(b->d_out_len, N * sizeof(uint32_t));
    }
#undef BALLOC
    if (!b->resize_only) {
        HALLOC(b->h_out, N * cfg->out_cap);
        HALLOC(b->h_out_len, N * sizeof(uint32_t));
    }
    HALLOC(b->h_items_back, N * sizeof(JpegDecodeItem));
    if (!b->resize_only) {
        HALLOC(b->h_off, (N + (size_t)b->max_chunks + 8) * sizeof(unsigned long long));
    }
#undef HALLOC
    b->ev.resize((size_t)b->max_chunks * 6);
    b->ev_h2d.resize(b->max_chunks);
    b->ev_d2h.resize(b->max_chunks);
    for (auto& e : b->ev)
        if (cudaEventCreate(&e) != cudaSuccess) return fail();
    for (auto& e : b->ev_h2d)
        if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return fail();
    for (auto& e : b->ev_d2h)
        if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return fail();
    b->items.resize(N);
    b->parse_status.resize(N);
    b->file_dev_off.resize(N);
    if (b->orient) {
        b->jobs.resize(N);
    }
    if (b->orient || b->gray) b->index.resize(N);
    b->arena_dev_used = dev_used;
    b->arena_host_used = host_used;
    return b;
}

// What a context made by batch_create_in took from the front of the caller's arenas: the rest is the caller's.
void lp::batch_arena_used(const lp_batch* b, size_t* dev_bytes, size_t* host_bytes) {
    *dev_bytes = b->arena_dev_used;
    *host_bytes = b->arena_host_used;
}

extern "C" void lp_batch_destroy(lp_batch* b) {
    if (!b) return;
    DeviceGuard dev_guard(b->cfg.device);
    cudaDeviceSynchronize();
    batch_free(b);
}

static int table_set_lookup(lp_batch* b, const JpegHeader& h);
static int table_set_for(lp_batch* b, const JpegHeader& h) {
    // nearly every file of a batch carries the tables of the previous one: compare before building a key
    if (b->last_table_idx >= 0 && !memcmp(h.huff_present, b->last_present, sizeof(h.huff_present)) &&
        !memcmp(h.huff_bits, b->last_bits, sizeof(h.huff_bits)) && !memcmp(h.huff_vals, b->last_vals, sizeof(h.huff_vals)))
        return b->last_table_idx;
    const int found = table_set_lookup(b, h);
    if (found >= 0) {
        memcpy(b->last_present, h.huff_present, sizeof(h.huff_present));
        memcpy(b->last_bits, h.huff_bits, sizeof(h.huff_bits));
        memcpy(b->last_vals, h.huff_vals, sizeof(h.huff_vals));
        b->last_table_idx = found;
    }
    return found;
}

static int table_set_lookup(lp_batch* b, const JpegHeader& h) {
    std::string key;
    for (int tc = 0; tc < 2; tc++)
        for (int th = 0; th < 4; th++) {
            key.push_back((char)h.huff_present[tc][th]);
            if (h.huff_present[tc][th]) {
                key.append((const char*)h.huff_bits[tc][th], 17);
                key.append((const char*)h.huff_vals[tc][th], 256);
            }
        }
    auto it = b->table_index.find(key);
    if (it != b->table_index.end()) return it->second;
    if ((int)b->tables.size() >= b->max_tables) return -1;
    JpegHuffSet hs;
    jpeg_build_huff_set(h, &hs);
    b->tables.push_back(hs);
    int idx = (int)b->tables.size() - 1;
    b->table_index[key] = idx;
    return idx;
}

static void batch_begin(lp_batch* b, int n) {
    b->n = n;
    b->tables.clear();
    b->table_index.clear();
    b->last_table_idx = -1;
    b->tables_uploaded = 0;
    b->scans.clear();
    b->scans_uploaded = 0;
    b->dev_off = b->clean_off = b->state_off = 0;
    for (auto& kv : b->chunk_layout)
        if (kv.second.d_rst_work) cudaFreeAsync(kv.second.d_rst_work, b->st);
    b->chunk_layout.clear();
}

// Host: where the files of images [i0, i0+cnt) go in the device scan buffer (no header parsing, so the
// bytes can start crossing PCIe before the headers are looked at).
static int batch_layout_chunk(lp_batch* b, const uint8_t* const* in, const size_t* in_len, int i0, int cnt) {
    // input files go to HBM as they are (contiguous runs of pointers = one transfer)
    int i = i0;
    while (i < i0 + cnt) {
        int j = i;
        size_t run = in_len[i];
        while (j + 1 < i0 + cnt && in[j + 1] == in[j] + in_len[j]) { j++; run += in_len[j]; }
        if (b->dev_off + run > b->cfg.max_in_bytes + 16 * (size_t)b->cfg.max_images) return LP_ERR_BUF_TOO_SMALL;
        size_t o = b->dev_off;
        for (int k = i; k <= j; k++) { b->file_dev_off[k] = o; o += in_len[k]; }
        b->dev_off = round_up(b->dev_off + run, (size_t)16);
        i = j + 1;
    }
    return LP_OK;
}

// Host: parse the headers of images [i0, i0+cnt), lay out their device scratch.  Pass 1 (a few threads) reads
// the headers; pass 2 lays the chunk's scratch out for the densest sampling layout that occurs IN THIS CHUNK, so a
// batch may mix 4:2:0 / 4:2:2 / 4:4:4 files in any order (the per-chunk scratch is sized for 4:4:4 anyway).
static int batch_parse_chunk(lp_batch* b, const uint8_t* const* in, const size_t* in_len, int i0, int cnt, int ordinal) {
    std::vector<JpegHeader> hdr((size_t)cnt);
    std::vector<uint32_t> blocks_of((size_t)cnt, 0), tiles_of((size_t)cnt, 0), total_of((size_t)cnt, 0);
    std::vector<uint8_t> class_of((size_t)cnt, 0);  // sub-class (top of the file): orientation class, + 3 for gray
    // multi-scan files: their scans (table_set numbering the file's own sets) and the Huffman tables of each set
    std::vector<std::vector<JpegScanDesc>> ms_scans((size_t)cnt);
    std::vector<std::vector<JpegHeader>> ms_sets((size_t)cnt);
    auto pass1 = [&](int k0, int k1) {
        for (int k = k0; k < k1; k++) {
            JpegHeader& h = hdr[k - i0];
            int rc = jpeg_parse_header(in[k], in_len[k], &h);
            const bool ms = !rc && !h.supported && h.multiscan && b->multiscan;
            if (!rc && !h.supported && !ms) rc = LP_ERR_UNSUPPORTED;
            if (!rc && (h.width != b->W || h.height != b->H)) rc = LP_ERR_BAD_ARGUMENT;
            // EXIF values outside 2..8 (0, 9, 300 ... the reader passes them through, like the reference's) are no-ops
            // for OrientationTransform, so they are class 0
            const int o = h.orientation;
            const int cls = o >= 2 && o <= 8 ? (o >= 5 ? 2 : 1) : 0;
            if (!rc && cls && !b->orient) rc = LP_ERR_UNSUPPORTED;
            if (!rc && h.ncomp != 3 && !(h.ncomp == 1 && b->gray)) rc = LP_ERR_UNSUPPORTED;
            class_of[k - i0] = (uint8_t)(cls + (h.ncomp == 1 ? 3 : 0));
            if (!rc && ms) {
                // what the per-image decoder refuses when it reads the scans (damage, over the work budget), lp_transform
                // reports as a failed decode
                std::vector<JpegScanDesc>& sc = ms_scans[k - i0];
                std::vector<JpegHeader>& sets = ms_sets[k - i0];
                sc.resize(kMultiscanMaxScans);
                sets.resize(kMultiscanMaxSets);
                int nscans = 0, nsets = 0;
                rc = jpeg_parse_scans(in[k], in_len[k], h, sc.data(), (int)sc.size(), &nscans, sets.data(), (int)sets.size(), &nsets);
                if (rc || jpeg_multiscan_visits(h, sc.data(), nscans) > kMultiscanMaxVisits) rc = LP_ERR_DECODING_FAILED;
                sc.resize(rc ? 0 : (size_t)nscans);
                sets.resize(rc ? 0 : (size_t)nsets);
            }
            JpegDecodeItem& it = b->items[k];
            memset(&it, 0, sizeof(it));
            if (!rc) {
                it.scan_len = (uint32_t)(ms ? in_len[k] : h.scan_length);  // multi-scan: the whole file
                it.restart_interval = ms ? 0 : h.restart_interval;
                const uint32_t total_blocks = jpeg_decode_item(h, &it);
                // decode only what Fit will read: the crop window (+ the chroma-upsampling margin); a rotated item's
                // crop is in its oriented frame, and the window is that crop's pre-image in the source
                int x0 = b->crop_x, y0 = b->crop_y, x1 = b->crop_x + b->crop_w, y1 = b->crop_y + b->crop_h;
                if (cls) {
                    const int cx = cls == 1 ? b->crop_x : b->crop2_x, cy = cls == 1 ? b->crop_y : b->crop2_y;
                    const int cw = cls == 1 ? b->crop_w : b->crop2_w, ch = cls == 1 ? b->crop_h : b->crop2_h;
                    int ax, ay, bx, by;  // opposite corners
                    orient_source_pixel(o, b->W, b->H, cx, cy, &ax, &ay);
                    orient_source_pixel(o, b->W, b->H, cx + cw - 1, cy + ch - 1, &bx, &by);
                    x0 = std::min(ax, bx); x1 = std::max(ax, bx) + 1;
                    y0 = std::min(ay, by); y1 = std::max(ay, by) + 1;
                }
                uint32_t tiles = 0;
                const uint32_t blocks = jpeg_item_set_window(&it, x0, y0, x1, y1, true, &tiles);
                blocks_of[k - i0] = blocks;
                tiles_of[k - i0] = tiles;
                total_of[k - i0] = total_blocks;
                if (blocks > b->max_blocks_alloc || total_blocks > b->max_blocks_alloc)
                    rc = LP_ERR_UNSUPPORTED;  // beyond what the context was created for
            }
            b->parse_status[k] = rc;
            it.status = rc ? -1 : 0;
        }
    };
    const int nthreads = cnt >= 256 ? 4 : 1;
    if (nthreads == 1) {
        pass1(i0, i0 + cnt);
    } else {
        std::vector<std::thread> pool;
        const int per = ceil_div(cnt, nthreads);
        for (int t = 1; t < nthreads; t++)
            pool.emplace_back(pass1, std::min(i0 + cnt, i0 + t * per), std::min(i0 + cnt, i0 + (t + 1) * per));
        pass1(i0, std::min(i0 + cnt, i0 + per));
        for (auto& th : pool) th.join();
    }
    lp_batch::ChunkLayout lay;
    lay.ordinal = ordinal;
    size_t rotated_window_bytes = 0;
    for (int k = i0; k < i0 + cnt; k++) {
        if (b->parse_status[k]) continue;
        const JpegDecodeItem& it = b->items[k];
        lay.blocks = std::max(lay.blocks, blocks_of[k - i0]);
        lay.tiles = std::max(lay.tiles, tiles_of[k - i0]);
        lay.total_blocks = std::max(lay.total_blocks, total_of[k - i0]);
        if (class_of[k - i0] % 3) rotated_window_bytes = std::max(rotated_window_bytes, (size_t)it.win_stride * it.win_h);
        if (!b->layout_known) {  // class 0's decoded window depends on the geometry only, which the context fixes
            JpegDecodeItem a = it;
            jpeg_item_set_window(&a, b->crop_x, b->crop_y, b->crop_x + b->crop_w, b->crop_y + b->crop_h, true, nullptr);
            b->win_w = a.win_w;
            b->win_h = a.win_h;
            b->win_x0 = a.win_x0;
            b->frame_bytes = (size_t)jpeg_window_row_bytes(a.win_x0, a.win_w, a.width, 3) * a.win_h;
            b->gray_row_bytes = jpeg_window_row_bytes(a.win_x0, a.win_w, a.width, 1);
            b->layout_known = true;
        }
    }
    // slots hold class 0's window, or the chunk's largest rotated window when that is larger
    lay.frame_stride = rotated_window_bytes > b->frame_bytes ? round_up(rotated_window_bytes, (size_t)256) : b->frame_bytes;
    b->blocks = std::max(b->blocks, lay.blocks);
    b->total_blocks = std::max(b->total_blocks, lay.total_blocks);
    b->chunk_layout[i0] = lay;
    for (int k = i0; k < i0 + cnt; k++) {
        if (b->parse_status[k]) continue;
        JpegDecodeItem& it = b->items[k];
        const int slot = k - i0;  // position inside its chunk: the per-chunk scratch is indexed from the chunk's first image
        if (!ms_scans[slot].empty()) {
            // multi-scan: its scans go to the pool with their sets' indices in the batch's table-set store; its nonzero
            // masks take the slot layout of the DC differences
            const std::vector<JpegScanDesc>& sc = ms_scans[slot];
            const std::vector<JpegHeader>& sets = ms_sets[slot];
            std::vector<int> global(sets.size(), -1);
            bool fits = b->scans.size() + sc.size() <= b->max_scans;
            for (size_t q = 0; q < sets.size() && fits; q++) fits = (global[q] = table_set_for(b, sets[q])) >= 0;
            if (!fits) {
                b->parse_status[k] = LP_ERR_UNSUPPORTED;
                it.status = -1;
                continue;
            }
            it.table_set = (uint32_t)b->scans.size();
            it.nscans = (uint32_t)sc.size();
            for (JpegScanDesc d : sc) {
                d.table_set = global[d.table_set];
                b->scans.push_back(d);
            }
            it.scan_off = b->file_dev_off[k];
            it.coef_off = (uint64_t)slot * lay.blocks * 64;
            it.frame_off = (uint64_t)slot * lay.frame_stride;
            it.dcdiff_off = (uint64_t)slot * lay.total_blocks;
            b->chunk_layout[i0].n_multiscan++;
            continue;
        }
        const int ts = table_set_for(b, hdr[k - i0]);
        if (ts < 0) {
            b->parse_status[k] = LP_ERR_UNSUPPORTED;
            it.status = -1;
            continue;
        }
        it.table_set = (uint32_t)ts;
        size_t state_need = 2 * huff_nsub(it.scan_len);
        if (it.restart_interval) {
            // RSTn streams: one thread per restart interval (jpeg_rst_*): the marker offsets live where the
            // self-synchronising decoder keeps its slot counts, clean_len carries the number of intervals
            const uint32_t mcus = (uint32_t)it.mcus_x * it.mcus_y;
            const uint32_t nint = (mcus + (uint32_t)it.restart_interval - 1) / (uint32_t)it.restart_interval;
            it.clean_len = nint;
            state_need = std::max(state_need, (size_t)nint + 2);
            if (b->state_off + state_need > b->state_cap) {  // (a restart interval of a few MCUs over a huge batch)
                b->parse_status[k] = LP_ERR_UNSUPPORTED;
                it.status = -1;
                continue;
            }
            for (uint32_t q = 0; q < nint; q++) b->chunk_layout[i0].rst_work.push_back(make_uint2((unsigned)slot, q));
        }
        it.scan_off = b->file_dev_off[k] + hdr[k - i0].scan_offset;
        it.coef_off = (uint64_t)slot * lay.blocks * 64;
        it.frame_off = (uint64_t)slot * lay.frame_stride;
        it.dcdiff_off = (uint64_t)slot * lay.total_blocks;
        it.clean_off = b->clean_off;
        it.state_off = b->state_off;
        b->clean_off += huff_clean_bytes(it.scan_len);
        b->state_off += state_need;
    }
    if (!b->index.empty()) {
        // the chunk's slots by sub-class (the resize / encode image maps), and the oriented crops of the rotated items in
        // that order; an item refused above is a colour item of class 0 whatever it is
        lp_batch::ChunkLayout& cl = b->chunk_layout[i0];
        int* idx = b->index.data() + i0;
        int at = 0, rotated = 0;
        for (int s = 0; s < 6; s++) {
            const int c = s % 3;
            for (int k = i0; k < i0 + cnt; k++) {
                const int cls = b->parse_status[k] ? 0 : class_of[k - i0];
                if (cls != s) continue;
                idx[at++] = k - i0;
                cl.n_class[s]++;
                if (!c) continue;
                const JpegDecodeItem& it = b->items[k];
                OrientJob& j = b->jobs[i0 + rotated++];
                j.src_off = it.frame_off;
                j.dst_off = (uint64_t)(k - i0) * b->oriented_bytes;
                j.src_stride = it.win_stride;
                j.o = hdr[k - i0].orientation;
                j.cx = c == 1 ? b->crop_x : b->crop2_x;
                j.cy = c == 1 ? b->crop_y : b->crop2_y;
                j.cw = c == 1 ? b->crop_w : b->crop2_w;
                j.ch = c == 1 ? b->crop_h : b->crop2_h;
                j.win_x0 = it.win_x0;
                j.win_y0 = it.win_y0;
            }
        }
    }
    return LP_OK;
}

// H2D: the chunk's files.
static int batch_upload_files(lp_batch* b, const uint8_t* const* in, const size_t* in_len, int i0, int cnt,
                              cudaStream_t st) {
    int i = i0;
    while (i < i0 + cnt) {
        int j = i;
        size_t run = in_len[i];
        while (j + 1 < i0 + cnt && in[j + 1] == in[j] + in_len[j]) { j++; run += in_len[j]; }
        LP_CUDA_OK(cudaMemcpyAsync(b->d_scan + b->file_dev_off[i], in[i], run, cudaMemcpyHostToDevice, st));
        i = j + 1;
    }
    return LP_OK;
}

// H2D: the chunk's items and any Huffman table sets not yet on the device.
static int batch_upload_items(lp_batch* b, int i0, int cnt, cudaStream_t st) {
    LP_CUDA_OK(cudaMemcpyAsync(b->d_items + i0, b->items.data() + i0, (size_t)cnt * sizeof(JpegDecodeItem),
                               cudaMemcpyHostToDevice, st));
    const auto lay = b->chunk_layout.find(i0);
    if (lay != b->chunk_layout.end()) {
        const int* nc = lay->second.n_class;
        const int rotated = nc[1] + nc[2] + nc[4] + nc[5];
        if (lay->second.mapped(cnt))
            LP_CUDA_OK(cudaMemcpyAsync(b->d_index + i0, b->index.data() + i0, (size_t)cnt * sizeof(int), cudaMemcpyHostToDevice, st));
        if (rotated)
            LP_CUDA_OK(cudaMemcpyAsync(b->d_jobs + i0, b->jobs.data() + i0, (size_t)rotated * sizeof(OrientJob),
                                       cudaMemcpyHostToDevice, st));
    }
    if (b->tables.size() > b->tables_uploaded) {
        LP_CUDA_OK(cudaMemcpyAsync(b->d_tables + b->tables_uploaded, b->tables.data() + b->tables_uploaded,
                                   (b->tables.size() - b->tables_uploaded) * sizeof(JpegHuffSet),
                                   cudaMemcpyHostToDevice, st));
        b->tables_uploaded = b->tables.size();
    }
    if (b->scans.size() > b->scans_uploaded) {
        LP_CUDA_OK(cudaMemcpyAsync(b->d_scans + b->scans_uploaded, b->scans.data() + b->scans_uploaded,
                                   (b->scans.size() - b->scans_uploaded) * sizeof(JpegScanDesc), cudaMemcpyHostToDevice,
                                   st));
        b->scans_uploaded = b->scans.size();
    }
    return LP_OK;
}

// Every kernel of the path for images [i0, i0+cnt) on stream st; ev = 6 timing events or null.
static int batch_launch_chunk(lp_batch* b, int i0, int cnt, cudaStream_t st, cudaEvent_t* ev) {
    if (!b->layout_known) {
        // no image up to and including this chunk had a usable header (every item carries its parse error):
        // there is no geometry to launch with and nothing to decode
        if (ev)
            for (int k = 0; k < 6; k++) LP_CUDA_OK(cudaEventRecord(ev[k], st));
        if (!b->resize_only) LP_CUDA_OK(cudaMemsetAsync(b->d_out_len + i0, 0, (size_t)cnt * sizeof(uint32_t), st));
        return LP_OK;
    }
    lp_batch::ChunkLayout none;
    lp_batch::ChunkLayout& lay = b->chunk_layout.count(i0) ? b->chunk_layout[i0] : none;
    if (ev) LP_CUDA_OK(cudaEventRecord(ev[0], st));
    JpegDecodeBatch d;
    if (!lay.rst_work.empty()) {
        if (!lay.d_rst_work) LP_CUDA_OK(cudaMallocAsync(&lay.d_rst_work, lay.rst_work.size() * sizeof(uint2), st));
        LP_CUDA_OK(cudaMemcpyAsync(lay.d_rst_work, lay.rst_work.data(), lay.rst_work.size() * sizeof(uint2), cudaMemcpyHostToDevice, st));
        d.rst_work = lay.d_rst_work;
        d.n_rst_work = (int)lay.rst_work.size();
    }
    d.items = b->d_items + i0;
    d.tables = b->d_tables;
    d.scan = b->d_scan;
    d.coef = b->d_coef;
    d.frames = b->d_frames;
    d.n = cnt;
    d.max_tiles_per_image = (int)lay.tiles;
    d.dcdiff = b->d_dcdiff;
    d.clean = b->d_clean;
    d.states = b->d_states;
    d.nslots = b->d_nslots;
    d.n_multiscan = lay.n_multiscan;
    d.scans = b->d_scans;
    d.masks = b->d_masks;
    int rc = jpeg_decode_launch(d, st, ev ? ev[1] : nullptr);
    if (rc) return rc;
    if (ev) LP_CUDA_OK(cudaEventRecord(ev[2], st));
    // items per sub-class as launched: a chunk that needs no image map is one sub-class in slot order
    const bool mapped = lay.mapped(cnt);
    int count[6];
    for (int s = 0; s < 6; s++) count[s] = mapped ? lay.n_class[s] : 0;
    if (!mapped) count[lay.n_class[3] == cnt ? 3 : 0] = cnt;
    const int* index = b->d_index + i0;
    for (int g = 0, job0 = 0; g < 2; g++) {  // the rotated items' oriented crops: colour, then gray
        const int n1 = lay.n_class[3 * g + 1], n2 = lay.n_class[3 * g + 2];
        if (n1 + n2) {
            rc = orient_crop_launch(b->d_jobs + i0 + job0, n1 + n2, b->d_frames, b->d_oriented, b->W, b->H, g ? 1 : 3,
                                    std::max(n1 ? b->crop_w : 0, n2 ? b->crop2_w : 0),
                                    std::max(n1 ? b->crop_h : 0, n2 ? b->crop2_h : 0), st);
            if (rc) return rc;
        }
        job0 += n1 + n2;
    }
    if (!b->geoms.empty()) {  // several outputs: the chunk's windows go into each before the next chunk reuses them
        for (size_t g = 0; g < b->geoms.size(); g++) {
            const BatchGeom& o = b->geoms[g];
            const size_t os = (size_t)o.out_w * o.out_h * 3;
            ResizeArgs r;
            r.src = b->d_frames;
            r.src_img_stride = lay.frame_stride;
            r.src_row_stride = b->frame_bytes / (size_t)b->win_h;
            r.channels = 3;
            r.crop_x = o.crop_x - b->win_x0;
            r.crop_y = o.crop_y - b->crop_y;  // (the window's top row is the union's)
            r.crop_w = o.crop_w;
            r.crop_h = o.crop_h;
            r.dst = b->d_resized + b->geom_off[g] + (size_t)i0 * os;
            r.dst_img_stride = os;
            r.dst_row_stride = (size_t)o.out_w * 3;
            r.dst_w = o.out_w;
            r.dst_h = o.out_h;
            r.n = cnt;
            r.interpolation = 3;
            rc = resize_launch(r, st);
            if (rc) return rc;
        }
        if (ev)
            for (int k = 3; k < 6; k++) LP_CUDA_OK(cudaEventRecord(ev[k], st));
        return LP_OK;
    }
    uint8_t* const resized = b->d_resized + (size_t)i0 * b->resized_bytes;
    for (int s = 0, at = 0; s < 6; at += count[s++]) {
        if (!count[s]) continue;
        const int c = s % 3, ch = s < 3 ? 3 : 1;
        ResizeArgs r;
        r.channels = ch;
        if (c == 0) {  // from the decoded windows (rows a 16-byte multiple)
            r.src = b->d_frames;
            r.src_img_stride = lay.frame_stride;
            r.src_row_stride = ch == 3 ? b->frame_bytes / (size_t)b->win_h : b->gray_row_bytes;
            r.crop_x = b->crop_x - b->win_x0;
        } else {  // the rotated classes, from their packed oriented crops
            r.src = b->d_oriented;
            r.src_img_stride = b->oriented_bytes;
            r.src_row_stride = (size_t)(c == 1 ? b->crop_w : b->crop2_w) * ch;
            r.crop_x = 0;
        }
        r.crop_y = 0;
        r.crop_w = c == 2 ? b->crop2_w : b->crop_w;
        r.crop_h = c == 2 ? b->crop2_h : b->crop_h;
        r.dst = resized;
        r.dst_img_stride = b->resized_bytes;
        r.dst_w = c == 2 ? b->out_w2 : b->out_w;
        r.dst_h = c == 2 ? b->out_h2 : b->out_h;
        r.dst_row_stride = (size_t)r.dst_w * ch;
        r.n = count[s];
        r.interpolation = 3;
        r.index = mapped ? index + at : nullptr;
        rc = resize_launch(r, st);
        if (rc) return rc;
    }
    if (ev) LP_CUDA_OK(cudaEventRecord(ev[3], st));
    if (b->resize_only) {  // (the encode stages take no time)
        if (ev) {
            LP_CUDA_OK(cudaEventRecord(ev[4], st));
            LP_CUDA_OK(cudaEventRecord(ev[5], st));
        }
        return LP_OK;
    }
    JpegEncodeBatch e;
    e.frames = resized;
    e.frame_img_stride = b->resized_bytes;
    e.quality = b->cfg.jpeg_quality;
    e.out = b->d_out + (size_t)i0 * b->cfg.out_cap;
    e.out_cap = b->cfg.out_cap;
    e.out_len = b->d_out_len + i0;
    e.scratch = b->d_enc_scratch;
    e.progressive = b->progressive;
    // one encode per (channel count, output size) present: class 2 has its own launch when its size differs.  A chunk
    // of one channel count and one size is encoded in slot order, without the image map.
    const bool two_sizes = b->out_w2 != b->out_w || b->out_h2 != b->out_h;
    std::vector<JpegEncodeBatch> enc;
    for (int g = 0, at = 0; g < 2; g++) {
        const int n01 = count[3 * g] + count[3 * g + 1], n2 = count[3 * g + 2];
        const bool split = n2 && two_sizes;
        const bool whole_chunk = n01 + n2 == cnt && !split;
        e.channels = g ? 1 : 3;
        for (int part = 0; part < 2; part++) {
            e.n = split ? (part ? n2 : n01) : (part ? 0 : n01 + n2);
            e.index = whole_chunk ? nullptr : index + at;
            at += e.n;
            e.width = split && part ? b->out_w2 : b->out_w;
            e.height = split && part ? b->out_h2 : b->out_h;
            e.frame_row_stride = (size_t)e.width * e.channels;
            if (e.n) enc.push_back(e);
        }
    }
    for (size_t k = 0; k < enc.size(); k++) {
        rc = jpeg_encode_launch(enc[k], st, ev && k + 1 == enc.size() ? ev[4] : nullptr);
        if (rc) return rc;
    }
    // the encoded bytes leave packed: slots are out_cap (64 KB) apart but hold a few KB each, so a compaction
    // kernel writes them back to back straight into the pinned, device-mapped host buffer (no D2H of the slots)
    rc = compact_launch(e.out, b->cfg.out_cap, e.out_len, (uint32_t)b->cfg.out_cap, cnt, b->h_out + (size_t)i0 * b->cfg.out_cap,
                        b->h_off + i0 + lay.ordinal, st);
    if (rc) return rc;
    if (ev) LP_CUDA_OK(cudaEventRecord(ev[5], st));
    return LP_OK;
}

static int batch_download_chunk(lp_batch* b, int i0, int cnt, cudaStream_t st) {
    const size_t cap = b->cfg.out_cap;
    LP_CUDA_OK(cudaMemcpyAsync(b->h_out_len + i0, b->d_out_len + i0, (size_t)cnt * 4, cudaMemcpyDeviceToHost, st));
    LP_CUDA_OK(cudaMemcpyAsync(b->h_items_back + i0, b->d_items + i0, (size_t)cnt * sizeof(JpegDecodeItem),
                               cudaMemcpyDeviceToHost, st));
    (void)cap;  // the encoded bytes are already in h_out: the compaction kernel wrote them there
    return LP_OK;
}

static void batch_finish_chunk(lp_batch* b, int i0, int cnt, uint8_t* const* out, size_t* out_len, int* status) {
    const size_t cap = b->cfg.out_cap;
    const int ordinal = b->chunk_layout.count(i0) ? b->chunk_layout[i0].ordinal : 0;
    const unsigned long long* off = b->h_off + i0 + ordinal;
    const uint8_t* packed = b->h_out + (size_t)i0 * cap;
    for (int i = i0; i < i0 + cnt; i++) {
        int st = b->parse_status[i];
        if (!st && b->h_items_back[i].status != 0) st = LP_ERR_DECODING_FAILED;
        // (a length above the slot size cannot come from the encoder kernel; it must never reach the memcpy below)
        if (!st && (b->h_out_len[i] == 0 || b->h_out_len[i] > cap)) st = LP_ERR_BUF_TOO_SMALL;
        if (status) status[i] = st;
        out_len[i] = 0;
        if (st) continue;
        if (off[i - i0] + b->h_out_len[i] > (unsigned long long)cnt * cap) {  // (cannot come from the scan kernel)
            if (status) status[i] = LP_ERR_CUDA;
            continue;
        }
        memcpy(out[i], packed + off[i - i0], b->h_out_len[i]);
        out_len[i] = b->h_out_len[i];
    }
}

extern "C" int lp_batch_stage(lp_batch* b, const uint8_t* const* in, const size_t* in_len, int n,
                              int* status) {
    if (!b || (n > 0 && (!in || !in_len)) || n < 0 || n > b->cfg.max_images) return LP_ERR_BAD_ARGUMENT;
    DeviceGuard dev_guard(b->cfg.device);
    if (!dev_guard.ok) return LP_ERR_CUDA;
    batch_begin(b, n);
    for (int i0 = 0; i0 < n; i0 += b->chunk) {
        const int cnt = std::min(b->chunk, n - i0);
        int rc = batch_layout_chunk(b, in, in_len, i0, cnt);
        if (!rc) rc = batch_upload_files(b, in, in_len, i0, cnt, b->st);
        if (!rc) rc = batch_parse_chunk(b, in, in_len, i0, cnt, i0 / b->chunk);
        if (rc) return rc;
        rc = batch_upload_items(b, i0, cnt, b->st);
        if (rc) return rc;
    }
    LP_CUDA_OK(cudaStreamSynchronize(b->st));
    if (status)
        for (int k = 0; k < n; k++) status[k] = b->parse_status[k];
    return LP_OK;
}

extern "C" int lp_batch_run(lp_batch* b, float* stage_ms) {
    if (!b) return LP_ERR_BAD_ARGUMENT;
    DeviceGuard dev_guard(b->cfg.device);
    if (!dev_guard.ok) return LP_ERR_CUDA;
    const long launches0 = g_launches;
    const int nchunks = ceil_div(b->n, b->chunk);
    for (int c = 0; c < nchunks; c++) {
        const int i0 = c * b->chunk, cnt = std::min(b->chunk, b->n - i0);
        int rc = batch_launch_chunk(b, i0, cnt, b->st, &b->ev[(size_t)c * 6]);
        if (rc) return rc;
    }
    LP_CUDA_OK(cudaStreamSynchronize(b->st));
    b->last_launches = (int)(g_launches - launches0);
    if (stage_ms) {
        for (int s = 0; s < LP_STAGE_COUNT; s++) stage_ms[s] = 0.f;
        if (nchunks == 0) return LP_OK;
        for (int c = 0; c < nchunks; c++) {
            cudaEvent_t* ev = &b->ev[(size_t)c * 6];
            float t;
            LP_CUDA_OK(cudaEventElapsedTime(&t, ev[0], ev[1])); stage_ms[LP_STAGE_HUFF_DECODE] += t;
            LP_CUDA_OK(cudaEventElapsedTime(&t, ev[1], ev[2])); stage_ms[LP_STAGE_IDCT_COLOR] += t;
            LP_CUDA_OK(cudaEventElapsedTime(&t, ev[2], ev[3])); stage_ms[LP_STAGE_RESIZE] += t;
            LP_CUDA_OK(cudaEventElapsedTime(&t, ev[3], ev[4])); stage_ms[LP_STAGE_ENC_TRANSFORM] += t;
            LP_CUDA_OK(cudaEventElapsedTime(&t, ev[4], ev[5])); stage_ms[LP_STAGE_ENC_ENTROPY] += t;
        }
        float t;
        LP_CUDA_OK(cudaEventElapsedTime(&t, b->ev[0], b->ev[(size_t)(nchunks - 1) * 6 + 5]));
        stage_ms[LP_STAGE_TOTAL] = t;  // first launch of the first chunk -> end of the last chunk
    }
    return LP_OK;
}

extern "C" int lp_batch_fetch(lp_batch* b, uint8_t* const* out, size_t* out_len, int* status) {
    if (!b || b->resize_only || (b->n > 0 && (!out || !out_len))) return LP_ERR_BAD_ARGUMENT;
    DeviceGuard dev_guard(b->cfg.device);
    if (!dev_guard.ok) return LP_ERR_CUDA;
    if (b->n == 0) return LP_OK;
    int rc = batch_download_chunk(b, 0, b->n, b->st);
    if (rc) return rc;
    LP_CUDA_OK(cudaStreamSynchronize(b->st));
    for (int i0 = 0; i0 < b->n; i0 += b->chunk)  // the chunks lp_batch_stage / lp_batch_run used
        batch_finish_chunk(b, i0, std::min(b->chunk, b->n - i0), out, out_len, status);
    return LP_OK;
}

// The reference-facing call: host buffers in, host buffers out.  Chunks are pipelined over three
// streams: while chunk c is in the kernels, chunk c+1's headers are parsed and its bytes cross PCIe,
// and chunk c-1's encoded bytes come back.
extern "C" int lp_batch_transform(lp_batch* b, const uint8_t* const* in, const size_t* in_len, int n,
                                  uint8_t* const* out, size_t* out_len, int* status) {
    if (!b || b->resize_only || n < 0 || n > b->cfg.max_images || (n > 0 && (!in || !in_len || !out || !out_len)))
        return LP_ERR_BAD_ARGUMENT;
    DeviceGuard dev_guard(b->cfg.device);
    if (!dev_guard.ok) return LP_ERR_CUDA;
    batch_begin(b, n);
    const long launches0 = g_launches;
    // Chunk schedule: nothing can run before the first chunk's headers are parsed and its bytes have
    // crossed PCIe, so the pipeline opens with a SMALL chunk (one full wave of Huffman CTAs instead of
    // three) and continues with full ones.
    std::vector<std::pair<int, int>> sched;
    {
        int i0 = 0;
        if (n > b->pipe_chunk && b->first_chunk >= 1 && b->first_chunk < b->pipe_chunk) {
            // ramp: a third of a wave (one Huffman CTA per SM), then a wave, then full chunks -- what is exposed at
            // the start is the upload + header parse of the FIRST chunk only
            const int third = b->first_chunk / 3;
            if (third >= 32 && n > third + b->first_chunk) {
                sched.push_back({0, third});
                i0 = third;
            }
            sched.push_back({i0, b->first_chunk});
            i0 += b->first_chunk;
        }
        // ... and closes with one wave again: behind the last entropy launch nothing overlaps the IDCT -> colour ->
        // resize -> encode -> D2H tail of the last chunk, so that chunk is kept small
        const bool ramp_down = b->first_chunk >= 1 && b->first_chunk < b->pipe_chunk;
        while (i0 < n) {
            const int left = n - i0;
            int cnt = std::min(b->pipe_chunk, left);
            if (ramp_down && left > b->first_chunk && left <= b->pipe_chunk + b->first_chunk) cnt = left - b->first_chunk;
            sched.push_back({i0, cnt});
            i0 += cnt;
        }
    }
    const int nchunks = (int)sched.size();
    int finished = 0;
    for (int c = 0; c < nchunks; c++) {
        const int i0 = sched[c].first, cnt = sched[c].second;
        // the bytes start crossing PCIe first; the headers are parsed while they travel
        int rc = batch_layout_chunk(b, in, in_len, i0, cnt);
        if (!rc) rc = batch_upload_files(b, in, in_len, i0, cnt, b->st_h2d);
        if (!rc) rc = batch_parse_chunk(b, in, in_len, i0, cnt, c);
        if (!rc) rc = batch_upload_items(b, i0, cnt, b->st_h2d);
        if (rc) return rc;
        LP_CUDA_OK(cudaEventRecord(b->ev_h2d[c], b->st_h2d));
        LP_CUDA_OK(cudaStreamWaitEvent(b->st, b->ev_h2d[c], 0));
        rc = batch_launch_chunk(b, i0, cnt, b->st, nullptr);
        if (rc) return rc;
        LP_CUDA_OK(cudaEventRecord(b->ev[(size_t)c * 6], b->st));
        LP_CUDA_OK(cudaStreamWaitEvent(b->st_d2h, b->ev[(size_t)c * 6], 0));
        rc = batch_download_chunk(b, i0, cnt, b->st_d2h);
        if (rc) return rc;
        LP_CUDA_OK(cudaEventRecord(b->ev_d2h[c], b->st_d2h));
        // hand back chunks whose bytes have already landed
        while (finished < c && cudaEventQuery(b->ev_d2h[finished]) == cudaSuccess) {
            batch_finish_chunk(b, sched[finished].first, sched[finished].second, out, out_len, status);
            finished++;
        }
    }
    for (; finished < nchunks; finished++) {
        LP_CUDA_OK(cudaEventSynchronize(b->ev_d2h[finished]));
        batch_finish_chunk(b, sched[finished].first, sched[finished].second, out, out_len, status);
    }
    b->last_launches = (int)(g_launches - launches0);
    return LP_OK;
}

// A resize-only context after lp_batch_stage + lp_batch_run: the status of every image (its parse error, or
// LP_ERR_DECODING_FAILED when the device decode refused it); the frames of the LP_OK ones are at lp_batch_resized_dev.
int lp::batch_resized_status(lp_batch* b, int* status) {
    if (!b || !b->resize_only) return LP_ERR_BAD_ARGUMENT;
    DeviceGuard dev_guard(b->cfg.device);
    if (!dev_guard.ok) return LP_ERR_CUDA;
    if (b->n == 0) return LP_OK;
    LP_CUDA_OK(cudaMemcpyAsync(b->h_items_back, b->d_items, (size_t)b->n * sizeof(JpegDecodeItem), cudaMemcpyDeviceToHost, b->st));
    LP_CUDA_OK(cudaStreamSynchronize(b->st));
    for (int i = 0; i < b->n; i++) {
        status[i] = b->parse_status[i];
        if (!status[i] && b->h_items_back[i].status != 0) status[i] = LP_ERR_DECODING_FAILED;
    }
    return LP_OK;
}

extern "C" int lp_batch_last_launches(const lp_batch* b) { return b ? b->last_launches : 0; }
// bytes per image that come back besides the encoded file: length, packed offset, the item mirror (status, diagnostics)
extern "C" size_t lp_batch_d2h_overhead_per_image(void) { return 4 + 8 + sizeof(JpegDecodeItem); }
extern "C" int lp_batch_chunk(const lp_batch* b) { return b ? b->chunk : 0; }
extern "C" int lp_batch_item_channels(const lp_batch* b, int i) {
    if (!b || i < 0 || i >= b->n || b->parse_status[i]) return 0;
    return b->items[i].frame_channels;
}
// Diagnostics after lp_batch_fetch / lp_batch_transform: Huffman synchronisation rounds per image.
extern "C" void lp_batch_sync_rounds(const lp_batch* b, double* mean, int* max) {
    double sum = 0;
    int mx = 0, cnt = 0;
    for (int i = 0; i < b->n; i++) {
        if (b->parse_status[i] || b->items[i].restart_interval || b->items[i].nscans) continue;
        const int r = (int)b->h_items_back[i].pad_;
        sum += r;
        mx = std::max(mx, r);
        cnt++;
    }
    if (mean) *mean = cnt ? sum / cnt : 0;
    if (max) *max = mx;
}
// Diagnostics: SM cycles per phase of the JPEG entropy kernels since the last reset (current device).
extern "C" int lp_huff_phase_clocks(unsigned long long* out8, int reset) { return lp::jpeg_huff_phase_clocks(out8, reset); }
extern "C" const uint8_t* lp_batch_decoded_dev(const lp_batch* b, size_t* image_stride) {
    const size_t last = b->chunk_layout.empty() ? 0 : b->chunk_layout.rbegin()->second.frame_stride;
    if (image_stride) *image_stride = last ? last : b->frame_bytes;
    return b->d_frames;
}
extern "C" const uint8_t* lp_batch_resized_dev(const lp_batch* b, size_t* image_stride) {
    if (image_stride) *image_stride = b->resized_bytes;
    return b->d_resized;
}
// A context made with several geometries: the resized frames of geometry g
const uint8_t* lp::batch_resized_geom(const lp_batch* b, int g, size_t* image_stride) {
    const BatchGeom& o = b->geoms[(size_t)g];
    *image_stride = (size_t)o.out_w * o.out_h * 3;
    return b->d_resized + b->geom_off[(size_t)g];
}

// ---- device helpers + single stages ---------------------------------------------------------

extern "C" void* lp_dev_alloc(size_t bytes) {
    if (ensure_device()) return nullptr;
    void* p = nullptr;
    if (cudaMalloc(&p, bytes + 256) != cudaSuccess) return nullptr;
    return p;
}
extern "C" void lp_dev_free(void* p) { cudaFree(p); }
extern "C" void* lp_host_alloc_pinned(size_t bytes) {
    if (ensure_device()) return nullptr;
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
    return p;
}
extern "C" void lp_host_free_pinned(void* p) { cudaFreeHost(p); }
extern "C" int lp_memcpy_h2d(void* dst, const void* src, size_t bytes) {
    LP_CUDA_OK(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
    return LP_OK;
}
extern "C" int lp_memcpy_d2h(void* dst, const void* src, size_t bytes) {
    LP_CUDA_OK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    return LP_OK;
}
extern "C" int lp_dev_synchronize(void) {
    LP_CUDA_OK(cudaDeviceSynchronize());
    return LP_OK;
}
extern "C" int lp_set_device(int device) {
    if (ensure_device()) return LP_ERR_CUDA;
    LP_CUDA_OK(cudaSetDevice(device));
    return LP_OK;
}

extern "C" int lp_resize_area_dev(const uint8_t* src, size_t src_image_stride, size_t src_row_stride,
                                  int channels, int crop_x, int crop_y, int crop_w, int crop_h,
                                  uint8_t* dst, size_t dst_image_stride, size_t dst_row_stride,
                                  int dst_w, int dst_h, int n, void* stream) {
    if (ensure_device()) return LP_ERR_CUDA;
    ResizeArgs a{src, src_image_stride, src_row_stride, channels, crop_x, crop_y, crop_w, crop_h,
                 dst, dst_image_stride, dst_row_stride, dst_w, dst_h, n, 3};
    return resize_launch(a, static_cast<cudaStream_t>(stream));
}

extern "C" int lp_resize_area_time_dev(const uint8_t* src, size_t src_image_stride,
                                       size_t src_row_stride, int channels, int crop_x, int crop_y,
                                       int crop_w, int crop_h, uint8_t* dst, size_t dst_image_stride,
                                       size_t dst_row_stride, int dst_w, int dst_h, int n, int iters,
                                       float* ms_per_iter) {
    if (ensure_device()) return LP_ERR_CUDA;
    cudaStream_t st = thread_stream();
    cudaEvent_t e0, e1;
    LP_CUDA_OK(cudaEventCreate(&e0));
    LP_CUDA_OK(cudaEventCreate(&e1));
    ResizeArgs a{src, src_image_stride, src_row_stride, channels, crop_x, crop_y, crop_w, crop_h,
                 dst, dst_image_stride, dst_row_stride, dst_w, dst_h, n, 3};
    int rc = resize_launch(a, st);  // warm-up (also builds the tap tables)
    if (rc) return rc;
    LP_CUDA_OK(cudaStreamSynchronize(st));
    LP_CUDA_OK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; i++) {
        rc = resize_launch(a, st);
        if (rc) return rc;
    }
    LP_CUDA_OK(cudaEventRecord(e1, st));
    LP_CUDA_OK(cudaEventSynchronize(e1));
    float ms = 0;
    LP_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
    if (ms_per_iter) *ms_per_iter = ms / iters;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return LP_OK;
}

// Encode `n` packed device frames (shared geometry) to baseline JPEG in device memory.
// out: n * out_cap bytes, out_len: n uint32 (0 = did not fit).  Used by bench.py to build the
// synthetic corpus and by tests; same kernels as opencv_encoder_write.
extern "C" int lp_jpeg_encode_dev(const uint8_t* frames, size_t frame_img_stride, size_t frame_row_stride,
                                  int width, int height, int channels, int quality, int n, uint8_t* out,
                                  size_t out_cap, uint32_t* out_len, void* stream) {
    if (ensure_device()) return LP_ERR_CUDA;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    void* scratch = nullptr;
    LP_CUDA_OK(cudaMallocAsync(&scratch, jpeg_encode_scratch_bytes(width, height, channels, n, out_cap), st));
    JpegEncodeBatch e;
    e.frames = frames;
    e.frame_img_stride = frame_img_stride;
    e.frame_row_stride = frame_row_stride;
    e.width = width; e.height = height; e.channels = channels;
    e.quality = quality;
    e.n = n;
    e.out = out;
    e.out_cap = out_cap;
    e.out_len = out_len;
    e.scratch = scratch;
    int rc = jpeg_encode_launch(e, st, nullptr);
    cudaFreeAsync(scratch, st);
    if (rc) return rc;
    LP_CUDA_OK(cudaStreamSynchronize(st));
    return LP_OK;
}
