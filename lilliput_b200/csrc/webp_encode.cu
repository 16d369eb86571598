// webp_encode.cu -- lilliput's WebP encoder surface (include/lp_webp.h = ref webp.hpp:56-73) on
// sm_90a.  Replaces webp_encoder_* (ref webp.cpp:388-783), i.e. libwebp's WebPEncodeBGR(A) /
// WebPEncodeLosslessBGR(A) for the first frame, WebPAnimEncoder for animations, and libwebpmux's
// assembly (VP8X / ICCP / ANIM / ANMF / ALPH chunks).
//
//   lossless (quality > 100, ref webp.cpp:466-470): vp8l_enc_core.h -- residual histograms of every
//     frame in one launch, prefix codes on the host (a few hundred symbols), then every pixel of every
//     frame packed in parallel behind its frame's head.  Exact by construction.  One code path,
//     webp_encode_lossless_batch, for N frames of one geometry: webp_encoder_write calls it with N = 1.
//   lossy: vp8_enc_core.h -- parallel BGR -> YUV 4:2:0, then one WARP per frame walks the
//     macroblocks (mode choice incl. the 16x16-versus-4x4 trial, transforms, quantisation,
//     reconstruction: the work inside a macroblock spread over the lanes) and codes the first partition
//     and up to eight token partitions on a lane each.  A valid VP8 stream at libwebp's quality ->
//     quantiser mapping, PSNR and size; NOT libwebp's own choices, so the bytes differ from the
//     reference's by design (DESIGN.md s.1 row R8 says what is and is not claimed).  One code path,
//     webp_encode_lossy_batch, for N frames of one geometry: webp_encoder_write calls it with N = 1.
//   alpha of a lossy frame: an ALPH chunk holding a VP8L-coded plane (vp8l_enc_core.h; histograms on
//     the device, prefix codes on the host, one CTA per plane packs the pixels).
//   animation: every frame a full-canvas ANMF (no blending, no disposal), durations = the delays
//     handed to webp_encoder_write.  (The reference's WebPAnimEncoder also searches sub-rectangles
//     and key-frame placement; that is a size optimisation, not a semantic one.)
#include <algorithm>
#include <chrono>
#include <cstring>
#include <thread>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"
#include "lp_webp.h"

#define LP_VP8_FN static __device__
#define LP_VP8_INL static __device__ __forceinline__
#define LP_VP8_HD static __host__ __device__
#define LP_VP8_TABLE static __device__ const
#include "vp8_enc_core.h"

#define LP_L_HD static __host__ __device__ __forceinline__
#include "vp8l_enc_core.h"

namespace lp {

int mat_device_view(void* mat, int* cols, int* rows, int* type, const uint8_t** dev, size_t* step);

// ------------------------------------------------------------------ lossless encode
// N frames of one geometry per call: the batch ABI (xbatch.cu) passes every frame of a run, webp_encoder_write one.
// Every frame is cut into the same tiles of kVp8lTile pixels and a launch covers the tiles of all frames (CTA t works on
// tile t % tiles_per_frame of frame t / tiles_per_frame), so one launch spreads a single 16383 x 16383 frame over the
// whole GPU as well as it spreads thousands of emoji frames.
//   1. histograms: a CTA per tile keeps 4 x 256 bins of residual_at in shared memory and adds them once into its frame's
//      histograms;
//   2. heads on the host: write_stream_head per frame builds the prefix codes, and the frame's exact length is then
//      head bits + sum over the four alphabets of count x code length, so the packed output is laid out before any pixel
//      is packed (frames at 4-byte boundaries: no word is shared by two frames);
//   3. pack: the bits of every tile, an exclusive scan of the tile sums within each frame, then every pixel's bits OR-ed
//      into the zeroed output behind its frame's head (a pixel's <= 60 bits touch up to three words);
//   4. the packed payloads home in one copy.
// Residuals are recomputed where they are needed (four neighbour loads per pixel): nothing is stored per pixel.

constexpr int kVp8lThreads = 256, kVp8lPixPerThread = 8, kVp8lTile = kVp8lThreads * kVp8lPixPerThread;
// packed output of one part of a call: a call whose payloads would pass it is packed in parts (same bytes)
constexpr size_t kVp8lPartBytes = (size_t)1 << 30;

struct Vp8lFrameInfo {
    unsigned long long out_word;  // the frame's first output word, relative to its part
    uint32_t head_bits;           // the head's length in bits; the pixels follow it
    uint32_t head_word;           // the head's first word in the staged head area
    uint32_t head_words;
    uint32_t pad_;
};

__device__ __forceinline__ void vp8l_load_table(vp8lenc::CodeTable* dst, const vp8lenc::CodeTable* src) {
    const uint32_t* s = reinterpret_cast<const uint32_t*>(src);
    uint32_t* d = reinterpret_cast<uint32_t*>(dst);
    for (int i = threadIdx.x; i < (int)(sizeof(vp8lenc::CodeTable) / 4); i += blockDim.x) d[i] = s[i];
}

// residual histograms (green, red, blue, alpha) of every frame.  A warp whose live lanes share a symbol (flat art,
// constant alpha) adds it once.
__global__ void __launch_bounds__(kVp8lThreads)
    vp8l_hist_batch_kernel(const uint8_t* frames, size_t img_stride, size_t step, int channels, int width, uint32_t npix,
                           int tiles_per_frame, uint32_t* hist /* n x 4 x 256 */) {
    __shared__ uint32_t sh[4 * 256];
    for (int i = threadIdx.x; i < 4 * 256; i += kVp8lThreads) sh[i] = 0;
    __syncthreads();
    const int f = blockIdx.x / tiles_per_frame;
    const uint32_t p0 = (uint32_t)(blockIdx.x % tiles_per_frame) * kVp8lTile;
    const uint8_t* frame = frames + (size_t)f * img_stride;
    const int lane = threadIdx.x & 31;
    for (int k = 0; k < kVp8lPixPerThread; k++) {
        const uint32_t p = p0 + (uint32_t)(k * kVp8lThreads + threadIdx.x);
        const bool valid = p < npix;
        const unsigned live = __ballot_sync(0xffffffffu, valid);
        if (!live) break;
        const uint32_t r = valid ? vp8lenc::residual_at(frame, step, channels, (int)(p % (uint32_t)width), (int)(p / (uint32_t)width)) : 0;
        const int leader = __ffs((int)live) - 1;
        const uint32_t r0 = __shfl_sync(0xffffffffu, r, leader);
        const uint32_t sym[4] = {(r >> 8) & 255, (r >> 16) & 255, r & 255, r >> 24};
        const uint32_t sym0[4] = {(r0 >> 8) & 255, (r0 >> 16) & 255, r0 & 255, r0 >> 24};
#pragma unroll
        for (int c = 0; c < 4; c++) {
            if (__all_sync(0xffffffffu, !valid || sym[c] == sym0[c])) {
                if (lane == leader) atomicAdd(&sh[c * 256 + sym0[c]], (uint32_t)__popc(live));
            } else if (valid) {
                atomicAdd(&sh[c * 256 + sym[c]], 1u);
            }
        }
    }
    __syncthreads();
    uint32_t* h = hist + (size_t)f * 1024;
    for (int i = threadIdx.x; i < 4 * 256; i += kVp8lThreads)
        if (sh[i]) atomicAdd(&h[i], sh[i]);
}

// bits of every tile under its frame's codes
__global__ void __launch_bounds__(kVp8lThreads)
    vp8l_tile_bits_kernel(const uint8_t* frames, size_t img_stride, size_t step, int channels, int width, uint32_t npix,
                          int tiles_per_frame, const vp8lenc::CodeTable* tables, uint32_t* tile_bits) {
    __shared__ vp8lenc::CodeTable t;
    __shared__ uint32_t warp_sums[kVp8lThreads / 32];
    const int f = blockIdx.x / tiles_per_frame;
    const uint32_t p0 = (uint32_t)(blockIdx.x % tiles_per_frame) * kVp8lTile;
    const uint8_t* frame = frames + (size_t)f * img_stride;
    vp8l_load_table(&t, tables + f);
    __syncthreads();
    uint32_t s = 0;
    for (int k = 0; k < kVp8lPixPerThread; k++) {
        const uint32_t p = p0 + (uint32_t)(k * kVp8lThreads + threadIdx.x);
        if (p >= npix) break;
        const uint32_t r = vp8lenc::residual_at(frame, step, channels, (int)(p % (uint32_t)width), (int)(p / (uint32_t)width));
        uint64_t bits;
        int nb;
        vp8lenc::pixel_bits(r, t, &bits, &nb);
        s += (uint32_t)nb;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t tot = 0;
        for (int w = 0; w < kVp8lThreads / 32; w++) tot += warp_sums[w];
        tile_bits[blockIdx.x] = tot;
    }
}

// exclusive scan of the tile sums within each frame: a CTA per frame, each thread a run of consecutive tiles
__global__ void vp8l_tile_scan_kernel(const uint32_t* tile_bits, int tiles_per_frame, unsigned long long* tile_off) {
    __shared__ unsigned long long warp_sums[32];
    const size_t base = (size_t)blockIdx.x * tiles_per_frame;
    const int per = (tiles_per_frame + (int)blockDim.x - 1) / (int)blockDim.x;
    const int j0 = min((int)threadIdx.x * per, tiles_per_frame), j1 = min(j0 + per, tiles_per_frame);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long s = 0;
    for (int j = j0; j < j1; j++) s += tile_bits[base + j];
    unsigned long long inc = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long v = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += v;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        unsigned long long w = lane < (int)(blockDim.x >> 5) ? warp_sums[lane] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long v = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += v;
        }
        warp_sums[lane] = w;
    }
    __syncthreads();
    unsigned long long at = (wid ? warp_sums[wid - 1] : 0) + inc - s;
    for (int j = j0; j < j1; j++) {
        tile_off[base + j] = at;
        at += tile_bits[base + j];
    }
}

// every pixel of tiles [f_first * tiles_per_frame, ...) into the zeroed output of their part; a thread packs
// kVp8lPixPerThread consecutive pixels.  The tile at the start of a frame also ORs the frame's head in: its last byte's
// unused high bits are zero, the pixels' bits land above them.
__global__ void __launch_bounds__(kVp8lThreads)
    vp8l_pack_batch_kernel(const uint8_t* frames, size_t img_stride, size_t step, int channels, int width, uint32_t npix,
                           int tiles_per_frame, int f_first, const vp8lenc::CodeTable* tables, const Vp8lFrameInfo* info,
                           const uint32_t* heads, const unsigned long long* tile_off, uint32_t* out) {
    __shared__ vp8lenc::CodeTable t;
    __shared__ uint32_t warp_sums[kVp8lThreads / 32];
    const int f = f_first + (int)(blockIdx.x / tiles_per_frame), j = (int)(blockIdx.x % tiles_per_frame);
    const uint8_t* frame = frames + (size_t)f * img_stride;
    const Vp8lFrameInfo fi = info[f];
    uint32_t* o = out + fi.out_word;
    vp8l_load_table(&t, tables + f);
    if (j == 0)
        for (uint32_t i = threadIdx.x; i < fi.head_words; i += kVp8lThreads) atomicOr(&o[i], heads[fi.head_word + i]);
    __syncthreads();
    const uint32_t q0 = (uint32_t)j * kVp8lTile + threadIdx.x * kVp8lPixPerThread;
    uint64_t bits[kVp8lPixPerThread];
    int nb[kVp8lPixPerThread];
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < kVp8lPixPerThread; k++) {
        const uint32_t p = q0 + k;
        bits[k] = 0;
        nb[k] = 0;
        if (p < npix) {
            const uint32_t r = vp8lenc::residual_at(frame, step, channels, (int)(p % (uint32_t)width), (int)(p / (uint32_t)width));
            vp8lenc::pixel_bits(r, t, &bits[k], &nb[k]);
        }
        s += (uint32_t)nb[k];
    }
    // block exclusive scan of the threads' bit counts
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += v;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        uint32_t w = lane < kVp8lThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += v;
        }
        if (lane < kVp8lThreads / 32) warp_sums[lane] = w;
    }
    __syncthreads();
    unsigned long long at = (unsigned long long)fi.head_bits + tile_off[blockIdx.x + (size_t)f_first * tiles_per_frame] +
                            (wid ? warp_sums[wid - 1] : 0) + inc - s;
#pragma unroll
    for (int k = 0; k < kVp8lPixPerThread; k++) {
        if (nb[k]) {
            const size_t w = (size_t)(at >> 5);
            const int sh = (int)(at & 31);
            const uint64_t lo = bits[k] << sh;
            const uint64_t hi = sh ? bits[k] >> (64 - sh) : 0;
            if ((uint32_t)lo) atomicOr(&o[w], (uint32_t)lo);
            if ((uint32_t)(lo >> 32)) atomicOr(&o[w + 1], (uint32_t)(lo >> 32));
            if ((uint32_t)hi) atomicOr(&o[w + 2], (uint32_t)hi);
        }
        at += (unsigned long long)nb[k];
    }
}

// fn(i) for i in [0, n) on a few host threads when n is large (the heads of a task's frames)
template <class F>
static void host_parallel(int n, F&& fn) {
    const int threads = n < 256 ? 1 : (int)std::min(8u, std::max(1u, std::thread::hardware_concurrency()));
    if (threads == 1) {
        for (int i = 0; i < n; i++) fn(i);
        return;
    }
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; t++)
        pool.emplace_back([&, t]() {
            for (int i = t; i < n; i += threads) fn(i);
        });
    for (auto& th : pool) th.join();
}

int webp_encode_lossless_batch(const uint8_t* d_frames, size_t img_stride, size_t row_step, int width, int height,
                               int channels, int n, std::vector<WebpEncodedFrame>* out, cudaStream_t st, size_t part_bytes) {
    out->assign(n > 0 ? (size_t)n : 0, WebpEncodedFrame());
    if (n <= 0) return LP_OK;
    if (width < 1 || height < 1 || width > 16383 || height > 16383 || (channels != 3 && channels != 4)) return LP_ERR_INVALID_IMAGE;
    if (!part_bytes) part_bytes = kVp8lPartBytes;
    const bool dbg = getenv("LP_DEBUG") != nullptr;
    const auto t0 = std::chrono::steady_clock::now();
    const uint32_t npix = (uint32_t)width * (uint32_t)height;
    const int tpf = (int)ceil_div(npix, (uint32_t)kVp8lTile);
    const size_t tiles = (size_t)n * tpf;
    if (tiles > (size_t)INT32_MAX) return LP_ERR_INVALID_IMAGE;  // (one grid dimension holds every tile)
    const size_t hist_b = round_up((size_t)n * 4096, (size_t)256), tbits_b = round_up(tiles * 4, (size_t)256);
    uint8_t* scratch = nullptr;
    if (cudaMallocAsync(&scratch, hist_b + tbits_b + tiles * 8, st) != cudaSuccess) {
        fprintf(stderr, "[lilliput_b200] webp_encode_lossless_batch: cudaMallocAsync(%zu) failed\n", hist_b + tbits_b + tiles * 8);
        cudaGetLastError();
        return LP_ERR_CUDA;
    }
    uint32_t* d_hist = reinterpret_cast<uint32_t*>(scratch);
    uint32_t* d_tile_bits = reinterpret_cast<uint32_t*>(scratch + hist_b);
    auto* d_tile_off = reinterpret_cast<unsigned long long*>(scratch + hist_b + tbits_b);
    uint8_t* staged = nullptr;
    int rc = LP_OK;
    do {
        // 1. histograms
        cudaMemsetAsync(d_hist, 0, (size_t)n * 4096, st);
        vp8l_hist_batch_kernel<<<(unsigned)tiles, kVp8lThreads, 0, st>>>(d_frames, img_stride, row_step, channels, width, npix, tpf,
                                                                         d_hist);
        g_launches++;
        std::vector<uint32_t> hist((size_t)n * 1024);
        if (cudaMemcpyAsync(hist.data(), d_hist, (size_t)n * 4096, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess) {
            rc = LP_ERR_CUDA;
            break;
        }
        const auto t1 = std::chrono::steady_clock::now();
        // 2. heads, codes and exact lengths
        std::vector<vp8lenc::BitWriter> heads((size_t)n);
        std::vector<vp8lenc::CodeTable> tables((size_t)n);
        std::vector<unsigned long long> bytes((size_t)n);
        std::vector<uint32_t> head_bits((size_t)n);
        host_parallel(n, [&](int i) {
            const uint32_t* h = hist.data() + (size_t)i * 1024;
            vp8lenc::BitWriter& bw = heads[i];
            vp8lenc::write_stream_head(bw, width, height, channels == 4, true, true, h, &tables[i]);
            head_bits[i] = (uint32_t)bw.nbits;
            bw.flush();
            unsigned long long bits = bw.nbits;
            for (int k = 0; k < 4; k++)
                for (int s = 0; s < 256; s++) bits += (unsigned long long)h[k * 256 + s] * tables[i].len[k][s];
            bytes[i] = (bits + 7) / 8;
        });
        const auto t2 = std::chrono::steady_clock::now();
        // parts of at most part_bytes of packed output (at least one frame each); frames at word boundaries
        std::vector<int> part_first{0};
        std::vector<Vp8lFrameInfo> info((size_t)n);
        std::vector<uint32_t> head_words;
        unsigned long long part_words = 0, max_part_words = 0;
        for (int i = 0; i < n; i++) {
            const unsigned long long words = (bytes[i] + 3) / 4;
            if (i > part_first.back() && (part_words + words) * 4 > part_bytes) {
                part_first.push_back(i);
                part_words = 0;
            }
            info[i].out_word = part_words;
            info[i].head_bits = head_bits[i];
            info[i].head_word = (uint32_t)head_words.size();
            info[i].head_words = (uint32_t)((heads[i].bytes.size() + 3) / 4);
            info[i].pad_ = 0;
            head_words.resize(head_words.size() + info[i].head_words, 0);
            memcpy(head_words.data() + info[i].head_word, heads[i].bytes.data(), heads[i].bytes.size());
            part_words += words;
            max_part_words = std::max(max_part_words, part_words);
        }
        part_first.push_back(n);
        // 3. codes, frame layout and heads in one upload; bits per tile, their offsets, then the parts
        const size_t tables_b = (size_t)n * sizeof(vp8lenc::CodeTable), info_b = round_up((size_t)n * sizeof(Vp8lFrameInfo), (size_t)256);
        const size_t heads_b = round_up(head_words.size() * 4, (size_t)256), out_b = (size_t)max_part_words * 4 + 256;
        if (cudaMallocAsync(&staged, tables_b + info_b + heads_b + out_b, st) != cudaSuccess) {
            fprintf(stderr, "[lilliput_b200] webp_encode_lossless_batch: cudaMallocAsync(%zu) failed\n", tables_b + info_b + heads_b + out_b);
            cudaGetLastError();
            staged = nullptr;
            rc = LP_ERR_CUDA;
            break;
        }
        std::vector<uint8_t> up(tables_b + info_b + head_words.size() * 4);
        memcpy(up.data(), tables.data(), tables_b);
        memcpy(up.data() + tables_b, info.data(), (size_t)n * sizeof(Vp8lFrameInfo));
        memcpy(up.data() + tables_b + info_b, head_words.data(), head_words.size() * 4);
        auto* d_tables = reinterpret_cast<const vp8lenc::CodeTable*>(staged);
        auto* d_info = reinterpret_cast<const Vp8lFrameInfo*>(staged + tables_b);
        auto* d_heads = reinterpret_cast<const uint32_t*>(staged + tables_b + info_b);
        uint32_t* d_out = reinterpret_cast<uint32_t*>(staged + tables_b + info_b + heads_b);
        cudaMemcpyAsync(staged, up.data(), up.size(), cudaMemcpyHostToDevice, st);
        vp8l_tile_bits_kernel<<<(unsigned)tiles, kVp8lThreads, 0, st>>>(d_frames, img_stride, row_step, channels, width, npix, tpf,
                                                                        d_tables, d_tile_bits);
        vp8l_tile_scan_kernel<<<n, tpf <= 32 ? 32 : 256, 0, st>>>(d_tile_bits, tpf, d_tile_off);
        g_launches += 2;
        std::vector<uint8_t> home;
        for (size_t p = 0; p + 1 < part_first.size() && !rc; p++) {
            const int f0 = part_first[p], f1 = part_first[p + 1];
            const size_t used = (size_t)(info[f1 - 1].out_word * 4 + bytes[f1 - 1]);
            cudaMemsetAsync(d_out, 0, round_up(used, (size_t)4), st);
            vp8l_pack_batch_kernel<<<(unsigned)((size_t)(f1 - f0) * tpf), kVp8lThreads, 0, st>>>(
                d_frames, img_stride, row_step, channels, width, npix, tpf, f0, d_tables, d_info, d_heads, d_tile_off, d_out);
            g_launches++;
            // 4. home
            home.resize(used);
            if (cudaMemcpyAsync(home.data(), d_out, used, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                cudaStreamSynchronize(st) != cudaSuccess) {
                rc = LP_ERR_CUDA;
                break;
            }
            for (int i = f0; i < f1; i++) {
                WebpEncodedFrame& f = (*out)[i];
                f.width = width;
                f.height = height;
                f.lossless = true;
                f.has_alpha = channels == 4;
                const uint8_t* b = home.data() + info[i].out_word * 4;
                f.image.assign(b, b + bytes[i]);
            }
        }
        if (dbg && !rc) {
            const auto t3 = std::chrono::steady_clock::now();
            auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
                return std::chrono::duration<double, std::milli>(b - a).count();
            };
            fprintf(stderr, "[lilliput_b200] vp8l batch: n=%d %dx%dx%d parts=%zu: heads (host) %.3f ms, device + copies %.3f ms\n", n,
                    width, height, channels, part_first.size() - 1, ms(t1, t2), ms(t0, t1) + ms(t2, t3));
        }
    } while (0);
    if (rc) {
        cudaGetLastError();
        for (WebpEncodedFrame& f : *out) f.image.clear();
    }
    if (staged) cudaFreeAsync(staged, st);
    cudaFreeAsync(scratch, st);
    return rc;
}

// n packed device frames -> their "VP8L" payloads back to back in `payloads` (frame i at offsets[i], lengths[i] bytes),
// as lp_xbatch's lossless WebP sink encodes them; part_bytes: the packed-output bound of one part (0 = the library's)
extern "C" int lp_webp_lossless_encode_batch_dev(const uint8_t* d_frames, size_t img_stride, size_t row_step, int width, int height,
                                                 int channels, int n, size_t part_bytes, uint8_t* payloads, size_t payloads_cap,
                                                 size_t* offsets, size_t* lengths) {
    if (ensure_device()) return LP_ERR_CUDA;
    std::vector<WebpEncodedFrame> frames;
    const int rc = webp_encode_lossless_batch(d_frames, img_stride, row_step, width, height, channels, n, &frames, thread_stream(),
                                              part_bytes);
    if (rc) return rc;
    size_t at = 0;
    for (int i = 0; i < n; i++) {
        const std::vector<uint8_t>& b = frames[i].image;
        if (at + b.size() > payloads_cap) return LP_ERR_BUF_TOO_SMALL;
        memcpy(payloads + at, b.data(), b.size());
        offsets[i] = at;
        lengths[i] = b.size();
        at += b.size();
    }
    return LP_OK;
}

// ------------------------------------------------------------------ lossy kernels

// ---- macroblock analysis, one WARP per frame --------------------------------------------------
// vp8enc::analyse_and_reconstruct (vp8_enc_core.h) walks the macroblocks on one lane; that chain (4 + 4 mode trials
// over 384 pixels, 24 forward and 24 inverse 4x4 transforms per macroblock) was the longest stage of the animated
// WebP path.  The macroblocks stay in raster order (each needs its left and top neighbours' reconstruction) but the
// work INSIDE one is spread over the warp: prediction errors 8 luma / 4 chroma pixels per lane + a shuffle
// reduction, one 4x4 block per lane for transform, quantisation and reconstruction.  Same arithmetic, same
// decisions (ties keep the lower mode number), so the stream is byte-identical to the serial walk's.

struct Vp8WarpBuf {
    uint8_t yb[vp8::YB_SIZE], ub[vp8::CB_SIZE], vb[vp8::CB_SIZE];
    int16_t coeffs[25 * 16];
    // the 4x4-prediction trial (vp8enc::analyse_i4 spread over the warp)
    uint8_t yb4[vp8::YB_SIZE];   // the macroblock predicted block by block, same borders as yb
    uint8_t edge[16];            // the 13 edge samples of the 4x4 block being tried
    int16_t lv4[16 * 16];
};

__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// prediction of pixel (x, y) of a size x size block whose borders are in place around dst (mode as vp8::pred_block)
__device__ __forceinline__ int vp8_pred_px(const uint8_t* dst, int bps, int size, int mode, int dc, int x, int y) {
    if (mode == vp8::DC_PRED) return dc;
    if (mode == vp8::TM_PRED) return vp8::clip8(dst[x - bps] + dst[y * bps - 1] - dst[-1 - bps]);
    if (mode == vp8::V_PRED) return dst[x - bps];
    return dst[y * bps - 1];
}
__device__ __forceinline__ int vp8_dc_value(const uint8_t* dst, int bps, int size, bool have_top, bool have_left, int lane) {
    // every lane takes (at most) one border sample pair; vp8::pred_block's three edge cases
    const int sh = size == 16 ? 4 : 3;
    int s = 0;
    if (lane < size) s = (have_top ? dst[lane - bps] : 0) + (have_left ? dst[lane * bps - 1] : 0);
    s = warp_sum_i(s);
    if (have_top && have_left) return (s + size) >> (sh + 1);
    if (have_top || have_left) return (s + (size >> 1)) >> sh;
    return 0x80;
}

// ---- one 4x4 block on 16 lanes (lane L = 4 * row + column; lanes 16..31 run along on zeros) ---------------------------
// The same integer arithmetic as vp8enc::fdct4x4 / quantize_block / vp8::inverse_dct_add / vp8enc::cost_coeffs, with the
// block's rows and columns exchanged by shuffles instead of a tmp[16] on one lane.
__device__ __forceinline__ int fdct4x4_lanes(int diff, int L) {  // residual sample -> coefficient `L` (raster)
    constexpr unsigned FULL = 0xffffffffu;
    const int r0 = L & 12, c = L & 3, r = (L >> 2) & 3;
    const int d0 = __shfl_sync(FULL, diff, r0), d1 = __shfl_sync(FULL, diff, r0 + 1), d2 = __shfl_sync(FULL, diff, r0 + 2),
              d3 = __shfl_sync(FULL, diff, r0 + 3);
    int a0 = d0 + d3, a1 = d1 + d2, a2 = d1 - d2, a3 = d0 - d3;
    const int tmp = c == 0 ? (a0 + a1) * 8 : c == 1 ? (a2 * 2217 + a3 * 5352 + 1812) >> 9 : c == 2 ? (a0 - a1) * 8 : (a3 * 2217 - a2 * 5352 + 937) >> 9;
    const int t0 = __shfl_sync(FULL, tmp, c), t1 = __shfl_sync(FULL, tmp, 4 + c), t2 = __shfl_sync(FULL, tmp, 8 + c),
              t3 = __shfl_sync(FULL, tmp, 12 + c);
    a0 = t0 + t3, a1 = t1 + t2, a2 = t1 - t2, a3 = t0 - t3;
    const int out = r == 0 ? (a0 + a1 + 7) >> 4 : r == 1 ? ((a2 * 2217 + a3 * 5352 + 12000) >> 16) + (a3 != 0) : r == 2 ? (a0 - a1 + 7) >> 4
                                                                                                                   : (a3 * 2217 - a2 * 5352 + 51000) >> 16;
    return (int)(int16_t)out;
}
// dequantised coefficient `L` (raster) -> the residual the decoder adds at pixel L
__device__ __forceinline__ int idct4x4_lanes(int coef, int L) {
    constexpr unsigned FULL = 0xffffffffu;
    {
        const int i = (L >> 2) & 3, k = L & 3;  // vertical pass: this lane makes tmp[4 * i + k] from column i
        const int i0 = __shfl_sync(FULL, coef, i), i4 = __shfl_sync(FULL, coef, 4 + i), i8 = __shfl_sync(FULL, coef, 8 + i),
                  i12 = __shfl_sync(FULL, coef, 12 + i);
        const int a = i0 + i8, b = i0 - i8, c = vp8::mul2(i4) - vp8::mul1(i12), d = vp8::mul1(i4) + vp8::mul2(i12);
        coef = k == 0 ? a + d : k == 1 ? b + c : k == 2 ? b - c : a - d;
    }
    const int i = (L >> 2) & 3, k = L & 3;  // horizontal pass: pixel (row i, column k) from tmp[i], tmp[4 + i], ...
    const int t0 = __shfl_sync(FULL, coef, i), t4 = __shfl_sync(FULL, coef, 4 + i), t8 = __shfl_sync(FULL, coef, 8 + i),
              t12 = __shfl_sync(FULL, coef, 12 + i);
    const int dc = t0 + 4, a = dc + t8, b = dc - t8, c = vp8::mul2(t4) - vp8::mul1(t12), d = vp8::mul1(t4) + vp8::mul2(t12);
    return (k == 0 ? a + d : k == 1 ? b + c : k == 2 ? b - c : a - d) >> 3;
}

__device__ void vp8_analyse_warp(const vp8enc::Params& P, const vp8enc::Buffers& B, Vp8WarpBuf& wb) {
    using namespace vp8enc;
    const int lane = threadIdx.x & 31;
    const int ys = P.mb_w * 16, cs = P.mb_w * 8;
    vp8::QuantMat qm;
    qm.y1[0] = kVp8DcTable[P.q];
    qm.y1[1] = kVp8AcTable[P.q];
    qm.y2[0] = kVp8DcTable[P.q] * 2;
    qm.y2[1] = (kVp8AcTable[P.q] * 101581) >> 16;
    if (qm.y2[1] < 8) qm.y2[1] = 8;
    qm.uv[0] = kVp8DcTable[P.q > 117 ? 117 : P.q];
    qm.uv[1] = kVp8AcTable[P.q];
    uint8_t* yd = wb.yb + BPS + 8;
    uint8_t* ud = wb.ub + BPS + 8;
    uint8_t* vd = wb.vb + BPS + 8;
    int16_t* coeffs = wb.coeffs;
    for (int mb_y = 0; mb_y < P.mb_h; mb_y++)
        for (int mb_x = 0; mb_x < P.mb_w; mb_x++) {
            const uint8_t* sy = B.sy + (size_t)mb_y * 16 * ys + mb_x * 16;
            const uint8_t* su = B.su + (size_t)mb_y * 8 * cs + mb_x * 8;
            const uint8_t* sv = B.sv + (size_t)mb_y * 8 * cs + mb_x * 8;
            uint8_t* py = B.ry + (size_t)mb_y * 16 * ys + mb_x * 16;
            uint8_t* pu = B.ru + (size_t)mb_y * 8 * cs + mb_x * 8;
            uint8_t* pv = B.rv + (size_t)mb_y * 8 * cs + mb_x * 8;
            const bool have_top = mb_y > 0, have_left = mb_x > 0;
            // prediction borders from the reconstruction, as the decoder will see them (s.12.2)
            if (lane < 16) yd[lane * BPS - 1] = have_left ? py[lane * ys - 1] : 129;
            if (lane < 8) {
                ud[lane * BPS - 1] = have_left ? pu[lane * cs - 1] : 129;
                vd[lane * BPS - 1] = have_left ? pv[lane * cs - 1] : 129;
            }
            if (lane < 17) {
                const int i = lane - 1;
                yd[i - BPS] = have_top ? ((i < 0 && mb_x == 0) ? 129 : py[i - ys]) : 127;
            }
            if (lane < 9) {
                const int i = lane - 1;
                ud[i - BPS] = have_top ? ((i < 0 && mb_x == 0) ? 129 : pu[i - cs]) : 127;
                vd[i - BPS] = have_top ? ((i < 0 && mb_x == 0) ? 129 : pv[i - cs]) : 127;
            }
            __syncwarp();
            // luma 16x16 mode: least squared prediction error; lane = (row, half row)
            const int ydc = vp8_dc_value(yd, BPS, 16, have_top, have_left, lane);
            int ymode = 0;
            {
                const int r = lane >> 1, c0 = (lane & 1) * 8;
                uint32_t best = 0xffffffffu;
                for (int m = 0; m < 4; m++) {
                    int e = 0;
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        const int d = (int)sy[r * ys + c0 + k] - vp8_pred_px(yd, BPS, 16, m, ydc, c0 + k, r);
                        e += d * d;
                    }
                    const uint32_t tot = (uint32_t)warp_sum_i(e);
                    if (tot < best) {
                        best = tot;
                        ymode = m;
                    }
                }
            }
            // chroma mode: both planes together; lane = (plane, row, half row)
            const int udc = vp8_dc_value(ud, BPS, 8, have_top, have_left, lane);
            const int vdc = vp8_dc_value(vd, BPS, 8, have_top, have_left, lane);
            int uvmode = 0;
            {
                const int pl = lane >> 4, r = (lane >> 1) & 7, c0 = (lane & 1) * 4;
                const uint8_t* src = pl ? sv : su;
                const uint8_t* dd = pl ? vd : ud;
                const int dc = pl ? vdc : udc;
                uint32_t best = 0xffffffffu;
                for (int m = 0; m < 4; m++) {
                    int e = 0;
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const int d = (int)src[r * cs + c0 + k] - vp8_pred_px(dd, BPS, 8, m, dc, c0 + k, r);
                        e += d * d;
                    }
                    const uint32_t tot = (uint32_t)warp_sum_i(e);
                    if (tot < best) {
                        best = tot;
                        uvmode = m;
                    }
                }
            }
            // the chosen predictions into the work buffers (the borders they read are outside the written area)
            {
                const int r = lane >> 1, c0 = (lane & 1) * 8;
                uint8_t pv8[8];
#pragma unroll
                for (int k = 0; k < 8; k++) pv8[k] = (uint8_t)vp8_pred_px(yd, BPS, 16, ymode, ydc, c0 + k, r);
                const int pl = lane >> 4, cr = (lane >> 1) & 7, cc0 = (lane & 1) * 4;
                uint8_t* dd = pl ? vd : ud;
                uint8_t pc4[4];
#pragma unroll
                for (int k = 0; k < 4; k++) pc4[k] = (uint8_t)vp8_pred_px(dd, BPS, 8, uvmode, pl ? vdc : udc, cc0 + k, cr);
                __syncwarp();
#pragma unroll
                for (int k = 0; k < 8; k++) yd[r * BPS + c0 + k] = pv8[k];
#pragma unroll
                for (int k = 0; k < 4; k++) dd[cr * BPS + cc0 + k] = pc4[k];
            }
            __syncwarp();
            // residual transforms: one 4x4 block per lane (0..15 Y, 16..19 U, 20..23 V)
            int16_t* lv = B.levels + ((size_t)mb_y * P.mb_w + mb_x) * 25 * 16;
            if (lane < 16) {
                fdct4x4(sy + (lane >> 2) * 4 * ys + (lane & 3) * 4, ys, yd + (lane >> 2) * 4 * BPS + (lane & 3) * 4, BPS, coeffs + lane * 16);
            } else if (lane < 24) {
                const int n = (lane - 16) & 3;
                const bool isv = lane >= 20;
                fdct4x4((isv ? sv : su) + (n >> 1) * 4 * cs + (n & 1) * 4, cs, (isv ? vd : ud) + (n >> 1) * 4 * BPS + (n & 1) * 4, BPS,
                        coeffs + lane * 16);
            }
            __syncwarp();
            if (lane == 0) {
                fwht(coeffs, coeffs + 24 * 16);
                quantize_block(coeffs + 24 * 16, lv + 24 * 16, qm.y2, 0, 96, 108);
                vp8::inverse_wht(coeffs + 24 * 16, coeffs);  // plants the dequantised DCs
            }
            __syncwarp();
            if (lane < 16) {
                quantize_block(coeffs + lane * 16, lv + lane * 16, qm.y1, 1, 96, 110);
                vp8::inverse_dct_add(coeffs + lane * 16, yd + (lane >> 2) * 4 * BPS + (lane & 3) * 4, BPS);
            } else if (lane < 24) {
                const int n = (lane - 16) & 3;
                quantize_block(coeffs + lane * 16, lv + lane * 16, qm.uv, 0, 110, 115);
                vp8::inverse_dct_add(coeffs + lane * 16, (lane >= 20 ? vd : ud) + (n >> 1) * 4 * BPS + (n & 1) * 4, BPS);
            }
            __syncwarp();
            // ---- 16x16 or sixteen 4x4 predictions (vp8enc::analyse_and_reconstruct's decision, same arithmetic): the
            //      candidate modes of a 4x4 block are tried by ten lanes at once, the winner's lane transforms,
            //      quantises and reconstructs it (the next block predicts from that), the rate estimates of the sixteen
            //      16x16-mode blocks run one per lane
            uint8_t* md = B.modes + ((size_t)mb_y * P.mb_w + mb_x) * kModeStride;
            bool use_i4 = false;
            unsigned long long modes4 = 0;
            // (flat macroblocks -- no AC level survives the 16x16 candidate's quantisation -- skip the trial, as the
            // serial walk does)
            const uint32_t nzm = __ballot_sync(0xffffffffu, lane < 16 && block_nz(lv + lane * 16, 1) != 0);
            if (P.try_i4 && nzm != 0) {
                uint32_t tm = 0, lm = 0;  // the neighbours' sub-block modes, one nibble each
                for (int i = 0; i < 4; i++) {
                    tm |= (uint32_t)(have_top ? (md - (size_t)P.mb_w * kModeStride)[2 + 12 + i] : (uint8_t)vp8::B_DC) << (4 * i);
                    lm |= (uint32_t)(have_left ? (md - kModeStride)[2 + 4 * i + 3] : (uint8_t)vp8::B_DC) << (4 * i);
                }
                uint32_t d16, r16;
                {
                    const int r = lane >> 1, c0 = (lane & 1) * 8;
                    int e = 0;
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        const int d = (int)sy[r * ys + c0 + k] - (int)yd[r * BPS + c0 + k];
                        e += d * d;
                    }
                    d16 = (uint32_t)warp_sum_i(e);
                    // rate of the 16x16 candidate: Y2 + sixteen luma blocks, two blocks per step, a scan position per lane
                    // (vp8enc::cost_pos summed over positions = vp8enc::cost_coeffs)
                    int c = 0;
                    const int pos = lane & 15;
                    const int zz = (int)((0xFEB7ADC963258410ull >> (4 * pos)) & 15ull);  // zig-zag: scan -> raster
                    for (int it = 0; it < 9; it++) {
                        const int blk = it < 8 ? 2 * it + (lane >> 4) : 24;       // the last step: Y2 on the lower half
                        const bool on = it < 8 || lane < 16;
                        const int first = it < 8 ? 1 : 0, type = it < 8 ? 0 : 1;
                        const int lvv = on ? (int)lv[blk * 16 + zz] : 0;
                        const int v = lvv < 0 ? -lvv : lvv;
                        int vprev = __shfl_up_sync(0xffffffffu, v, 1);
                        if (pos == 0) vprev = 0;
                        const uint32_t nzb = __ballot_sync(0xffffffffu, on && v != 0 && pos >= first);
                        const uint32_t mine = (nzb >> (lane & 16)) & 0xffffu;
                        const int last = mine ? 31 - __clz((int)mine) : -1;
                        const int ctx = it < 8 ? (((blk & 3) ? (int)((nzm >> (blk - 1)) & 1u) : 0) + ((blk >> 2) ? (int)((nzm >> (blk - 4)) & 1u) : 0)) : 0;
                        const uint8_t* tp = &kVp8CoeffProba0[0][0][0][0] + type * (8 * 3 * 11);
                        if (on && pos >= first) c += cost_pos(tp, ctx, first, last, v, vprev, pos);
                    }
                    r16 = (uint32_t)warp_sum_i(c) + (uint32_t)bit_cost(1, 145) + 512u;
                }
                // the trial buffer: yb's borders + the above-right samples (the decoder's rule, s.12.3)
                uint8_t* yd4 = wb.yb4 + BPS + 8;
                if (lane < 17) yd4[lane - 1 - BPS] = yd[lane - 1 - BPS];
                if (lane < 16) yd4[lane * BPS - 1] = yd[lane * BPS - 1];
                if (lane < 16) {
                    const int i = 16 + (lane & 3), r = lane >> 2;
                    const uint8_t v = have_top ? (mb_x < P.mb_w - 1 ? py[i - ys] : py[15 - ys]) : (uint8_t)127;
                    yd4[(r ? 4 * r - 1 : -1) * BPS + i] = v;
                }
                __syncwarp();
                const int q = qm.y1[1];
                const int lambda4 = (3 * q * q) >> 7;
                uint32_t d4 = 0, r4 = (uint32_t)bit_cost(0, 145), tnzb = 0, lnzb = 0;
                const unsigned long long lam = (unsigned long long)((q * q) >> 7);
                const unsigned long long s16 = (unsigned long long)d16 * 256 + (unsigned long long)r16 * lam;
                for (int n = 0; n < 16; n++) {
                    // distortion and rate only grow: once the blocks tried so far cost what the 16x16 candidate costs in
                    // total, the trial is lost -- the serial walk, which always finishes it, decides the same
                    if ((unsigned long long)d4 * 256 + (unsigned long long)r4 * lam >= s16) break;
                    const int bx = n & 3, by = n >> 2;
                    uint8_t* d = yd4 + by * 4 * BPS + bx * 4;
                    const uint8_t* src = sy + by * 4 * ys + bx * 4;
                    const int ctx_top = (int)((tm >> (4 * bx)) & 15u), ctx_left = (int)((lm >> (4 * by)) & 15u);
                    // the block's 13 edge samples {L, K, J, I, X, A..H} where every lane can index them
                    if (lane < 13)
                        wb.edge[lane] = lane < 4 ? d[(3 - lane) * BPS - 1] : lane == 4 ? d[-BPS - 1] : d[-BPS + (lane - 5)];
                    __syncwarp();
                    const uint8_t* e = wb.edge;
                    const int dc = (e[5] + e[6] + e[7] + e[8] + e[0] + e[1] + e[2] + e[3] + 4) >> 3;
                    // all ten modes without a divergent switch (vp8enc::pred4_px): lane = (pixel, half); the lower half of the
                    // warp tries modes 0..4 of its pixel, the upper half modes 5..9; squared errors summed over 16 lanes
                    const int L = lane & 15, pr = L >> 2, pc = L & 3, half = lane >> 4;
                    const int sp = (int)src[pr * ys + pc];
                    uint32_t sse5[5];
#pragma unroll
                    for (int t = 0; t < 5; t++) {
                        const int dd = sp - pred4_px(half * 5 + t, L, e, dc);
                        int v = dd * dd;
#pragma unroll
                        for (int o = 8; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                        sse5[t] = (uint32_t)v;
                    }
                    // lane -> the mode it speaks for: m = 5 * half + (L % 5); score = distortion + lambda * mode bits
                    const int t5 = L % 5, m = half * 5 + t5;
                    const uint32_t my_sse = t5 == 0 ? sse5[0] : t5 == 1 ? sse5[1] : t5 == 2 ? sse5[2] : t5 == 3 ? sse5[3] : sse5[4];
                    const uint32_t score = my_sse * 256u + (uint32_t)(i4_mode_cost_ctx(ctx_top, ctx_left, m) * lambda4);
                    uint32_t mn = score;
#pragma unroll
                    for (int o = 16; o; o >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
                    uint32_t wm = score == mn ? (uint32_t)m : 15u;  // ties: the lower mode number, as the serial walk keeps it
#pragma unroll
                    for (int o = 16; o; o >>= 1) wm = min(wm, __shfl_xor_sync(0xffffffffu, wm, o));
                    const int w = (int)wm;
                    // the winner's prediction, transform, quantisation, reconstruction, distortion and rate of the block on
                    // lanes 0..15 (lane = 4 * row + column; the upper half runs along)
                    const bool act = lane < 16;
                    const int pp = pred4_px(w, L, e, dc);
                    const int coefq = fdct4x4_lanes(sp - pp, L);
                    const int step = qm.y1[L > 0];
                    int lvl;
                    {
                        const int a = coefq < 0 ? -coefq : coefq;
                        int q_ = (a + (((L > 0 ? 110 : 96) * step) >> 8)) / step;
                        if (q_ > 2047) q_ = 2047;
                        lvl = coefq < 0 ? -q_ : q_;
                    }
                    if (act) wb.lv4[n * 16 + L] = (int16_t)lvl;
                    const int rec = vp8::clip8(pp + idct4x4_lanes((int)(int16_t)(lvl * step), L));
                    if (act) d[pr * BPS + pc] = (uint8_t)rec;
                    const uint32_t my_d_all = (uint32_t)warp_sum_i(act ? (sp - rec) * (sp - rec) : 0);
                    // rate: scan position `lane` (vp8enc::cost_pos summed over the positions)
                    uint32_t blk_bits;
                    int blk_nz;
                    {
                        const int zz = lane < 16 ? (int)((0xFEB7ADC963258410ull >> (4 * lane)) & 15ull) : 0;  // zig-zag: scan -> raster
                        const int mag = lvl < 0 ? -lvl : lvl;
                        const int v = __shfl_sync(0xffffffffu, mag, zz);
                        int vprev = __shfl_up_sync(0xffffffffu, v, 1);
                        if (lane == 0) vprev = 0;
                        const uint32_t nzm = __ballot_sync(0xffffffffu, act && v != 0);
                        const int last = nzm ? 31 - __clz((int)nzm) : -1;
                        const uint8_t* tp = &kVp8CoeffProba0[0][0][0][0] + 3 * (8 * 3 * 11);
                        const int ctx0 = (int)((tnzb >> bx) & 1u) + (int)((lnzb >> by) & 1u);
                        const int cp = act ? cost_pos(tp, ctx0, 0, last, v, vprev, lane) : 0;
                        blk_bits = (uint32_t)warp_sum_i(cp) + (uint32_t)i4_mode_cost_ctx(ctx_top, ctx_left, w);
                        blk_nz = last >= 0;
                    }
                    d4 += my_d_all;
                    r4 += blk_bits;
                    const uint32_t nz = (uint32_t)blk_nz;
                    tnzb = (tnzb & ~(1u << bx)) | (nz << bx);
                    lnzb = (lnzb & ~(1u << by)) | (nz << by);
                    tm = (tm & ~(15u << (4 * bx))) | ((uint32_t)w << (4 * bx));
                    lm = (lm & ~(15u << (4 * by))) | ((uint32_t)w << (4 * by));
                    modes4 |= (unsigned long long)w << (4 * n);
                    __syncwarp();
                }
                const unsigned long long s4 = (unsigned long long)d4 * 256 + (unsigned long long)r4 * lam;
                use_i4 = s4 < s16;
                if (use_i4) {
#pragma unroll
                    for (int k = 0; k < 8; k++) lv[lane * 8 + k] = wb.lv4[lane * 8 + k];
                    if (lane < 16) lv[24 * 16 + lane] = 0;
                    const int r = lane >> 1, c0 = (lane & 1) * 8;
#pragma unroll
                    for (int k = 0; k < 8; k++) yd[r * BPS + c0 + k] = yd4[r * BPS + c0 + k];
                }
                __syncwarp();
            }
            if (lane < 16) md[2 + lane] = use_i4 ? (uint8_t)((modes4 >> (4 * lane)) & 15u) : (uint8_t)ymode;
            {
                // which of the 25 blocks kept a non-zero level: one block per lane, once, for the three bitstream walks
                const uint32_t mask = __ballot_sync(0xffffffffu, lane < 25 && block_nz(lv + lane * 16, 0) != 0);
                if (lane == 0) mb_set_nz_mask(md, mask);
            }
            // reconstruction out to the planes: 8 luma pixels and 4 chroma pixels per lane
            {
                const int r = lane >> 1, c0 = (lane & 1) * 8;
#pragma unroll
                for (int k = 0; k < 8; k++) py[r * ys + c0 + k] = yd[r * BPS + c0 + k];
                const int pl = lane >> 4, cr = (lane >> 1) & 7, cc0 = (lane & 1) * 4;
                uint8_t* pc = pl ? pv : pu;
                const uint8_t* dd = pl ? vd : ud;
#pragma unroll
                for (int k = 0; k < 4; k++) pc[cr * cs + cc0 + k] = dd[cr * BPS + cc0 + k];
            }
            if (lane == 0) {
                md[0] = use_i4 ? (uint8_t)kI4 : (uint8_t)ymode;
                md[1] = (uint8_t)uvmode;
            }
            __syncwarp();
            __threadfence_block();  // the next macroblock's borders read what other lanes just wrote to global memory
        }
}

// The bitstream pass on a warp: lanes 0..nparts-1 first count the token-tree branches of their partition (the statistics
// the frame's probabilities are decided from), all 32 lanes settle the 1056 probabilities, then lane q codes token
// partition q and lane `nparts` the first partition, and all lanes copy the pieces into place.  Same bytes as
// vp8enc::write_bitstream (the serial composition of the same pieces).
__device__ size_t vp8_write_bitstream_warp(const vp8enc::Params& P, const vp8enc::Buffers& B, uint8_t* part0, size_t part0_cap,
                                           uint8_t* tokens, size_t tokens_cap, uint8_t* aux, uint8_t* out, size_t out_cap) {
    constexpr unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int nparts = 1 << vp8enc::log2_partitions(P);
    if (vp8enc::partition_scratch_off(P, nparts - 1, nparts) + vp8enc::partition_scratch_cap(P, nparts - 1, nparts) > tokens_cap)
        return 0;
    for (size_t i = lane; i < vp8enc::kAuxBytes / 4; i += 32) reinterpret_cast<uint32_t*>(aux)[i] = 0;
    __syncwarp();
    if (lane < nparts && vp8enc::stats_partition(lane, nparts)) vp8enc::walk_partition<false>(P, B, lane, nparts, aux, nullptr, 0);
    __syncwarp();
    vp8enc::finish_statistics(aux, lane, 32);
    __syncwarp();
    unsigned long long mine = 0;
    if (lane < nparts)
        mine = vp8enc::walk_partition<true>(P, B, lane, nparts, aux, tokens + vp8enc::partition_scratch_off(P, lane, nparts),
                                            vp8enc::partition_scratch_cap(P, lane, nparts));
    else if (lane == nparts)
        mine = vp8enc::write_part0(P, B, aux, part0, part0_cap);
    __syncwarp();
    const size_t part0_len = (size_t)__shfl_sync(FULL, mine, nparts);
    if (!part0_len) return vp8enc::kPart0TooLarge;
    size_t sizes[8];
#pragma unroll
    for (int q = 0; q < 8; q++) sizes[q] = (size_t)__shfl_sync(FULL, mine, q);
    size_t total = 0;
    if (lane == 0) total = vp8enc::write_frame_header(P, part0_len, sizes, nparts, out, out_cap);
    total = (size_t)__shfl_sync(FULL, (unsigned long long)total, 0);
    if (!total) return 0;
    for (size_t i = lane; i < part0_len; i += 32) out[10 + i] = part0[i];
    size_t at = 10 + part0_len + (size_t)3 * (nparts - 1);
#pragma unroll
    for (int q = 0; q < 8; q++) {
        if (q < nparts) {
            const uint8_t* src = tokens + vp8enc::partition_scratch_off(P, q, nparts);
            for (size_t i = lane; i < sizes[q]; i += 32) out[at + i] = src[i];
            at += sizes[q];
        }
    }
    return total;
}

// vp8enc::kTryI4 unless LP_WEBP_I4=0 / 1 says otherwise (measurements; the tests compare against the host build, which
// follows kTryI4)
static int vp8_try_i4() {
    static const int v = getenv("LP_WEBP_I4") ? atoi(getenv("LP_WEBP_I4")) != 0 : vp8enc::kTryI4;
    return v;
}

// ------------------------------------------------------------------ lossy encode
// N frames of one geometry per launch: the batch ABI (xbatch.cu) passes many, webp_encoder_write one.  One frame per
// warp (the macroblock walk and the boolean coder are a serial dependency chain per frame, so the parallelism is
// across frames), alpha planes through one CTA per frame.

// BGR(A) -> padded Y / U / V planes (edge replication up to the macroblock grid); one chroma sample = 2x2 luma.
__global__ void vp8_planes_batch_kernel(const uint8_t* frames, size_t img_stride, size_t step, int channels, int width,
                                        int height, int ys, int yh, uint8_t* planes, size_t planes_stride) {
    const int cx = blockIdx.x * blockDim.x + threadIdx.x, cy = blockIdx.y;
    if (cx >= ys / 2) return;
    const uint8_t* frame = frames + (size_t)blockIdx.z * img_stride;
    uint8_t* sy = planes + (size_t)blockIdx.z * planes_stride;
    const size_t ypl = (size_t)ys * yh;
    uint8_t* su = sy + ypl;
    uint8_t* sv = su + ypl / 4;
    int r = 0, g = 0, b = 0;
    for (int dy = 0; dy < 2; dy++)
        for (int dx = 0; dx < 2; dx++) {
            const int x = min(2 * cx + dx, width - 1), y = min(2 * cy + dy, height - 1);
            const uint8_t* p = frame + (size_t)y * step + (size_t)x * channels;
            sy[(size_t)(2 * cy + dy) * ys + 2 * cx + dx] = (uint8_t)vp8enc::rgb_to_y(p[2], p[1], p[0]);
            b += p[0];
            g += p[1];
            r += p[2];
        }
    su[(size_t)cy * (ys / 2) + cx] = (uint8_t)vp8enc::rgb_to_u(r, g, b);
    sv[(size_t)cy * (ys / 2) + cx] = (uint8_t)vp8enc::rgb_to_v(r, g, b);
}

struct Vp8EncBatch {
    vp8enc::Params P;       // shared geometry / quantiser
    uint8_t* scratch;       // per-frame regions, `stride` apart
    size_t stride;
    size_t off_src, off_rec, off_levels, off_modes, off_part0, off_tokens, off_aux;
    size_t part0_cap, tokens_cap;
    uint8_t* out;           // n * out_cap
    size_t out_cap;
    uint32_t* out_len;      // n (0 = did not fit, (uint32_t)kPart0TooLarge = first partition beyond the format's limit)
    int n;
};

constexpr int kVp8EncWarps = 4;
__global__ void __launch_bounds__(kVp8EncWarps * 32) vp8_encode_batch_kernel(Vp8EncBatch b) {
    __shared__ Vp8WarpBuf wbs[kVp8EncWarps];
    const int f = blockIdx.x * kVp8EncWarps + (threadIdx.x >> 5);
    if (f >= b.n) return;
    vp8enc::Params P = b.P;
    if (P.filter_level < 0) P.filter_level = vp8enc::filter_level_for_q(P.q);
    uint8_t* base = b.scratch + (size_t)f * b.stride;
    const size_t ypl = (size_t)P.mb_w * 16 * P.mb_h * 16;
    vp8enc::Buffers B;
    B.sy = base + b.off_src;
    B.su = B.sy + ypl;
    B.sv = B.su + ypl / 4;
    B.ry = base + b.off_rec;
    B.ru = B.ry + ypl;
    B.rv = B.ru + ypl / 4;
    B.levels = reinterpret_cast<int16_t*>(base + b.off_levels);
    B.modes = base + b.off_modes;
    vp8_analyse_warp(P, B, wbs[threadIdx.x >> 5]);
    const size_t n = vp8_write_bitstream_warp(P, B, base + b.off_part0, b.part0_cap, base + b.off_tokens, b.tokens_cap,
                                              base + b.off_aux, b.out + (size_t)f * b.out_cap, b.out_cap);
    if ((threadIdx.x & 31) == 0) b.out_len[f] = (uint32_t)n;
}

// alpha plane of every frame + "does the frame have any non-opaque pixel" (libwebp drops the ALPH chunk of an
// opaque picture: WebPEncode -> WebPPictureHasTransparency)
__global__ void extract_alpha_batch_kernel(const uint8_t* frames, size_t img_stride, size_t step, int width, int height,
                                           uint8_t* planes, uint32_t* transparent) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    uint8_t a = 255;
    if (x < width) {
        a = frames[(size_t)blockIdx.z * img_stride + (size_t)y * step + (size_t)x * 4 + 3];
        planes[((size_t)blockIdx.z * height + y) * width + x] = a;
    }
    if (__syncthreads_or(a != 255) && threadIdx.x == 0) atomicOr(&transparent[blockIdx.z], 1u);
}

__global__ void vp8l_hist_plane_batch_kernel(const uint8_t* planes, int width, int height, uint32_t* hist /* n x 4 x 256 */) {
    __shared__ uint32_t sh[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    const uint8_t* plane = planes + (size_t)blockIdx.z * width * height;
    if (x < width) {
        const uint32_t r = vp8lenc::residual_at(plane, (size_t)width, 1, x, y);
        atomicAdd(&sh[(r >> 8) & 255], 1u);
    }
    __syncthreads();
    // a lone plane travels in green; red / blue residuals are 0 and alpha's is 0 except at (0,0) -- the
    // host adds those three constant histograms itself
    uint32_t* h = hist + (size_t)blockIdx.z * 1024;
    for (int i = threadIdx.x; i < 256; i += blockDim.x)
        if (sh[i]) atomicAdd(&h[i], sh[i]);
}

// One CTA per frame: bit length of every pixel, running prefix sum, bits OR-ed into the (zeroed) output
// behind the head the host wrote.  total_bits[f] = head bits + pixel bits.
constexpr int kPackThreads = 512;
__global__ void __launch_bounds__(kPackThreads)
    vp8l_pack_plane_batch_kernel(const uint8_t* planes, int width, int height, const vp8lenc::CodeTable* tables,
                                 const uint32_t* head_bits, const uint32_t* transparent, uint32_t* out, size_t out_words,
                                 uint32_t* total_bits) {
    __shared__ uint32_t warp_sums[kPackThreads / 32];
    const int f = blockIdx.x;
    if (!transparent[f]) return;
    const vp8lenc::CodeTable& t = tables[f];
    const uint8_t* plane = planes + (size_t)f * width * height;
    uint32_t* o = out + (size_t)f * out_words;
    const uint32_t npix = (uint32_t)width * height;
    uint32_t base = head_bits[f];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint32_t p0 = 0; p0 < npix; p0 += kPackThreads) {
        const uint32_t p = p0 + threadIdx.x;
        uint64_t bits = 0;
        int nb = 0;
        if (p < npix) {
            const uint32_t r = vp8lenc::residual_at(plane, (size_t)width, 1, (int)(p % width), (int)(p / width));
            vp8lenc::pixel_bits(r, t, &bits, &nb);
        }
        // block exclusive scan of nb
        uint32_t inc = (uint32_t)nb;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += v;
        }
        if (lane == 31) warp_sums[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            uint32_t s = lane < kPackThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t v = __shfl_up_sync(0xffffffffu, s, d);
                if (lane >= d) s += v;
            }
            if (lane < kPackThreads / 32) warp_sums[lane] = s;
        }
        __syncthreads();
        const uint32_t at = base + (wid ? warp_sums[wid - 1] : 0) + inc - (uint32_t)nb;
        base += warp_sums[kPackThreads / 32 - 1];
        if (nb) {
            const size_t w = at >> 5;
            const int sh = (int)(at & 31);
            const uint64_t lo = bits << sh;
            const uint64_t hi = sh ? bits >> (64 - sh) : 0;
            if ((uint32_t)lo) atomicOr(&o[w], (uint32_t)lo);
            if ((uint32_t)(lo >> 32)) atomicOr(&o[w + 1], (uint32_t)(lo >> 32));
            if ((uint32_t)hi) atomicOr(&o[w + 2], (uint32_t)hi);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) total_bits[f] = base;
}

// The one scratch allocation of a batch: frame regions, output slots, then the length and alpha arrays
struct LossyLayout {
    size_t lens_b, aplane_b, hist_b, tables_b, aout_b, alph_words, total;
};

// Geometry, per-frame scratch layout and output slot of a batch of n frames (b->P's size fields, the offsets, stride,
// out_cap), and the sizes of the allocation lossy_batch makes for them
static LossyLayout lossy_layout(int width, int height, int channels, int n, Vp8EncBatch* out) {
    Vp8EncBatch& b = *out;
    b.P.width = width;
    b.P.height = height;
    b.P.mb_w = (width + 15) >> 4;
    b.P.mb_h = (height + 15) >> 4;
    b.n = n;
    const int ys = b.P.mb_w * 16, yh = b.P.mb_h * 16;
    const size_t ypl = (size_t)ys * yh, nmb = (size_t)b.P.mb_w * b.P.mb_h;
    const size_t planes_b = round_up(ypl * 3 / 2, (size_t)256);
    const size_t levels_b = round_up(nmb * 25 * 16 * 2, (size_t)256), modes_b = round_up(nmb * vp8enc::kModeStride, (size_t)256);
    b.part0_cap = vp8enc::part0_scratch_bytes(b.P);  // the sizes the host build of the core encodes with, too
    b.tokens_cap = vp8enc::token_scratch_bytes(b.P);
    const size_t aux_b = vp8enc::kAuxBytes;  // statistics + probabilities of the bitstream pass (vp8_enc_core.h)
    b.off_src = 0;
    b.off_rec = planes_b;
    b.off_levels = 2 * planes_b;
    b.off_modes = b.off_levels + levels_b;
    b.off_part0 = b.off_modes + modes_b;
    b.off_tokens = b.off_part0 + round_up(b.part0_cap, (size_t)256);
    b.off_aux = b.off_tokens + round_up(b.tokens_cap, (size_t)256);
    b.stride = b.off_aux + aux_b;
    // the stream is the two partitions back to back: a slot that holds what they can hold never overflows;
    // real frames use a few per cent of it, so the slots are compacted on the device before they cross PCIe
    b.out_cap = round_up((size_t)16 + b.part0_cap + b.tokens_cap, (size_t)256);
    const bool alpha = channels == 4;
    const size_t npix = (size_t)width * height;
    LossyLayout L;
    L.alph_words = (npix * 2 + 4096 + 3) / 4;  // one <=15-bit green code per pixel + the head
    L.lens_b = round_up((size_t)n * 4, (size_t)256);
    L.aplane_b = alpha ? round_up((size_t)n * npix, (size_t)256) : 0;
    L.hist_b = alpha ? round_up((size_t)n * 1024 * 4, (size_t)256) : 0;
    L.tables_b = alpha ? round_up((size_t)n * sizeof(vp8lenc::CodeTable), (size_t)256) : 0;
    L.aout_b = alpha ? round_up((size_t)n * L.alph_words * 4, (size_t)256) : 0;
    L.total = (size_t)n * b.stride + (size_t)n * b.out_cap + 4 * L.lens_b + L.aplane_b + L.hist_b + L.tables_b + L.aout_b;
    return L;
}

size_t webp_encode_lossy_scratch_bytes(int width, int height, int channels, int n) {
    Vp8EncBatch b{};
    return lossy_layout(width, height, channels, n, &b).total;
}

// `too_large[i]` = 1 when frame i failed only because its first partition outgrew the format's limit
static int lossy_batch(const uint8_t* d_frames, size_t img_stride, size_t row_step, int width, int height, int channels,
                       int n, int quality, int try_i4, std::vector<WebpEncodedFrame>* out, std::vector<uint8_t>* too_large,
                       cudaStream_t st) {
    out->assign((size_t)n, WebpEncodedFrame());
    too_large->assign((size_t)n, 0);
    if (n <= 0) return LP_OK;
    if (width > 16383 || height > 16383 || (channels != 3 && channels != 4)) return LP_ERR_INVALID_IMAGE;
    Vp8EncBatch b;
    const LossyLayout lay = lossy_layout(width, height, channels, n, &b);
    b.P.q = vp8enc::quality_to_q(quality);
    b.P.filter_level = -1;
    b.P.try_i4 = try_i4;
    const int ys = b.P.mb_w * 16, yh = b.P.mb_h * 16;
    const bool alpha = channels == 4;
    const size_t npix = (size_t)width * height;
    const size_t alph_words = lay.alph_words, lens_b = lay.lens_b, aplane_b = lay.aplane_b, hist_b = lay.hist_b,
                 tables_b = lay.tables_b, total = lay.total;
    uint8_t* scratch = nullptr;
    if (cudaMallocAsync(&scratch, total, st) != cudaSuccess) {
        fprintf(stderr, "[lilliput_b200] webp_encode_lossy_batch: cudaMallocAsync(%zu) failed\n", total);
        cudaGetLastError();
        return LP_ERR_CUDA;
    }
    uint8_t* p = scratch;
    b.scratch = p; p += (size_t)n * b.stride;
    b.out = p; p += (size_t)n * b.out_cap;
    b.out_len = reinterpret_cast<uint32_t*>(p); p += lens_b;
    uint32_t* d_transp = reinterpret_cast<uint32_t*>(p); p += lens_b;
    uint32_t* d_head_bits = reinterpret_cast<uint32_t*>(p); p += lens_b;
    uint32_t* d_total_bits = reinterpret_cast<uint32_t*>(p); p += lens_b;
    uint8_t* d_aplanes = p; p += aplane_b;
    uint32_t* d_hist = reinterpret_cast<uint32_t*>(p); p += hist_b;
    auto* d_tables = reinterpret_cast<vp8lenc::CodeTable*>(p); p += tables_b;
    uint32_t* d_aout = reinterpret_cast<uint32_t*>(p);
    int rc = LP_OK;
    std::vector<uint32_t> lens((size_t)n), transp((size_t)n, 0), total_bits((size_t)n, 0);
    do {
        {
            dim3 grid(ceil_div(ys / 2, 128), yh / 2, n);
            vp8_planes_batch_kernel<<<grid, 128, 0, st>>>(d_frames, img_stride, row_step, channels, width, height, ys, yh,
                                                          b.scratch + b.off_src, b.stride);
            vp8_encode_batch_kernel<<<ceil_div(n, kVp8EncWarps), kVp8EncWarps * 32, 0, st>>>(b);
            g_launches += 2;
        }
        std::vector<uint32_t> hist;
        if (alpha) {
            cudaMemsetAsync(d_transp, 0, (size_t)n * 4, st);
            cudaMemsetAsync(d_hist, 0, (size_t)n * 1024 * 4, st);
            dim3 grid(ceil_div(width, 256), height, n);
            extract_alpha_batch_kernel<<<grid, 256, 0, st>>>(d_frames, img_stride, row_step, width, height, d_aplanes, d_transp);
            vp8l_hist_plane_batch_kernel<<<grid, 256, 0, st>>>(d_aplanes, width, height, d_hist);
            g_launches += 2;
            hist.resize((size_t)n * 1024);
            cudaMemcpyAsync(transp.data(), d_transp, (size_t)n * 4, cudaMemcpyDeviceToHost, st);
            cudaMemcpyAsync(hist.data(), d_hist, (size_t)n * 1024 * 4, cudaMemcpyDeviceToHost, st);
        }
        cudaMemcpyAsync(lens.data(), b.out_len, (size_t)n * 4, cudaMemcpyDeviceToHost, st);
        if (cudaStreamSynchronize(st) != cudaSuccess) { rc = LP_ERR_CUDA; break; }
        // alpha planes of the frames that have transparency: prefix codes on the host, packing on the device
        std::vector<vp8lenc::BitWriter> heads;
        bool any_alpha = false;
        if (alpha) {
            heads.resize((size_t)n);
            std::vector<vp8lenc::CodeTable> tables((size_t)n);
            std::vector<uint32_t> head_bits((size_t)n, 0);
            for (int i = 0; i < n; i++) {
                if (!transp[i]) continue;
                any_alpha = true;
                uint32_t* h = hist.data() + (size_t)i * 1024;
                h[256 + 0] = (uint32_t)npix;    // red residuals: all 0
                h[512 + 0] = (uint32_t)npix;    // blue
                h[768 + 0] = (uint32_t)npix;    // alpha: 0xff - 0xff = 0 everywhere (the first pixel predicts 0xff000000)
                vp8lenc::BitWriter& bw = heads[i];
                bw.put(1, 8);  // ALPH header byte: VP8L-compressed, no filter, no pre-processing
                vp8lenc::write_stream_head(bw, width, height, false, false, false, h, &tables[i]);
                head_bits[i] = (uint32_t)bw.nbits;
                bw.flush();
                if (bw.bytes.size() + 8 > alph_words * 4) { rc = LP_ERR_CUDA; break; }
            }
            if (rc) break;
            if (any_alpha) {
                cudaMemsetAsync(d_aout, 0, (size_t)n * alph_words * 4, st);
                cudaMemcpyAsync(d_tables, tables.data(), (size_t)n * sizeof(vp8lenc::CodeTable), cudaMemcpyHostToDevice, st);
                cudaMemcpyAsync(d_head_bits, head_bits.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st);
                for (int i = 0; i < n; i++)
                    if (transp[i])
                        cudaMemcpyAsync(reinterpret_cast<uint8_t*>(d_aout) + (size_t)i * alph_words * 4, heads[i].bytes.data(),
                                        heads[i].bytes.size(), cudaMemcpyHostToDevice, st);
                vp8l_pack_plane_batch_kernel<<<n, kPackThreads, 0, st>>>(d_aplanes, width, height, d_tables, d_head_bits, d_transp,
                                                                         d_aout, alph_words, d_total_bits);
                g_launches++;
                cudaMemcpyAsync(total_bits.data(), d_total_bits, (size_t)n * 4, cudaMemcpyDeviceToHost, st);
                if (cudaStreamSynchronize(st) != cudaSuccess) { rc = LP_ERR_CUDA; break; }  // (tables / heads stay alive until here)
            }
        }
        // results home: the bytes actually used, packed on the device and fetched with ONE copy per kind (a copy per
        // frame -- 16 K of them for a task of 128-frame animations -- cost more than the encoder)
        std::vector<unsigned long long> off((size_t)n + 1, 0), aoff((size_t)n + 1, 0);
        std::vector<uint32_t> alen((size_t)n, 0);
        for (int i = 0; i < n; i++) {
            const uint32_t l = lens[i] > b.out_cap ? 0u : lens[i];
            off[(size_t)i + 1] = off[i] + (((unsigned long long)l + 15ull) & ~15ull);
            if (alpha && transp[i]) {
                const size_t bytes = ((size_t)total_bits[i] + 7) / 8;
                alen[i] = bytes > alph_words * 4 ? 0u : (uint32_t)bytes;
            }
            aoff[(size_t)i + 1] = aoff[i] + (((unsigned long long)alen[i] + 15ull) & ~15ull);
        }
        const size_t img_total = (size_t)off[n], alph_total = (size_t)aoff[n];
        uint8_t* d_pack = nullptr;
        const size_t offs_b = round_up(((size_t)n + 1) * 8, (size_t)256);
        if (cudaMallocAsync(&d_pack, offs_b + img_total + alph_total + 256, st) != cudaSuccess) {
            cudaGetLastError();
            rc = LP_ERR_CUDA;
            break;
        }
        std::vector<uint8_t> home(img_total + alph_total);
        auto* d_off = reinterpret_cast<unsigned long long*>(d_pack);
        rc = compact_launch(b.out, b.out_cap, b.out_len, (uint32_t)b.out_cap, n, d_pack + offs_b, d_off, st);
        if (!rc && img_total) cudaMemcpyAsync(home.data(), d_pack + offs_b, img_total, cudaMemcpyDeviceToHost, st);
        if (!rc && alph_total) {
            // (the packed alpha streams reuse d_head_bits for their byte lengths and the offset table: stream order
            // puts both behind the kernels that read them)
            cudaMemcpyAsync(d_head_bits, alen.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st);
            rc = compact_launch(reinterpret_cast<const uint8_t*>(d_aout), alph_words * 4, d_head_bits, (uint32_t)(alph_words * 4), n,
                                d_pack + offs_b + img_total, d_off, st);
            if (!rc) cudaMemcpyAsync(home.data() + img_total, d_pack + offs_b + img_total, alph_total, cudaMemcpyDeviceToHost, st);
        }
        if (cudaStreamSynchronize(st) != cudaSuccess) rc = LP_ERR_CUDA;
        cudaFreeAsync(d_pack, st);
        for (int i = 0; i < n && !rc; i++) {
            WebpEncodedFrame& f = (*out)[i];
            f.width = width;
            f.height = height;
            f.lossless = false;
            f.has_alpha = alpha && transp[i];
            (*too_large)[i] = lens[i] == (uint32_t)vp8enc::kPart0TooLarge;
            if (lens[i] == 0 || lens[i] > b.out_cap) { f.image.clear(); continue; }  // caller reports the item
            f.image.assign(home.data() + off[i], home.data() + off[i] + lens[i]);
            if (f.has_alpha) {
                if (alen[i] == 0) { f.image.clear(); continue; }
                f.alph.assign(home.data() + img_total + aoff[i], home.data() + img_total + aoff[i] + alen[i]);
            }
        }
    } while (0);
    cudaFreeAsync(scratch, st);
    return rc;
}

int webp_encode_lossy_batch(const uint8_t* d_frames, size_t img_stride, size_t row_step, int width, int height,
                            int channels, int n, int quality, std::vector<WebpEncodedFrame>* out, cudaStream_t st) {
    const int try_i4 = vp8_try_i4();
    std::vector<uint8_t> too_large;
    int rc = lossy_batch(d_frames, img_stride, row_step, width, height, channels, n, quality, try_i4, out, &too_large, st);
    // a frame whose first partition outgrew the format's limit (vp8enc::kPart0TooLarge): once more, alone, with 16x16
    // prediction only.  Rare (large frames of fine detail), so one launch per such frame.
    for (int i = 0; rc == LP_OK && try_i4 && i < n; i++) {
        if (!too_large[i]) continue;
        std::vector<WebpEncodedFrame> one;
        std::vector<uint8_t> again;
        rc = lossy_batch(d_frames + (size_t)i * img_stride, 0, row_step, width, height, channels, 1, quality, 0, &one, &again, st);
        if (rc == LP_OK) (*out)[i] = std::move(one[0]);
    }
    return rc;
}

// ------------------------------------------------------------------ RIFF assembly (host)

static void put_le32(std::vector<uint8_t>& v, uint32_t x) {
    for (int i = 0; i < 4; i++) v.push_back((uint8_t)(x >> (8 * i)));
}
static void put_le24(std::vector<uint8_t>& v, uint32_t x) {
    for (int i = 0; i < 3; i++) v.push_back((uint8_t)(x >> (8 * i)));
}
static void put_chunk(std::vector<uint8_t>& v, const char* tag, const uint8_t* p, size_t n) {
    v.insert(v.end(), tag, tag + 4);
    put_le32(v, (uint32_t)n);
    v.insert(v.end(), p, p + n);
    if (n & 1) v.push_back(0);
}

using EncodedFrame = WebpEncodedFrame;

static void put_image_chunks(std::vector<uint8_t>& v, const EncodedFrame& f) {
    if (!f.alph.empty()) put_chunk(v, "ALPH", f.alph.data(), f.alph.size());
    put_chunk(v, f.lossless ? "VP8L" : "VP8 ", f.image.data(), f.image.size());
}


// RIFF file of one still (n == 1) or an animation: VP8X / ICCP / ANIM / ANMF / ALPH / VP8(L) as libwebpmux
// lays them out (ref webp.cpp:511-560 WebPMuxAssemble).
void webp_assemble(const WebpEncodedFrame* frames, int n, const uint8_t* icc, size_t icc_len, uint32_t bgcolor,
                   uint32_t loop_count, std::vector<uint8_t>* file_out) {
    std::vector<uint8_t> body;
    const bool anim = n > 1;
    bool any_alpha = false;
    for (int i = 0; i < n; i++) any_alpha |= frames[i].has_alpha;
    const WebpEncodedFrame& f0 = frames[0];
    const bool need_vp8x = anim || icc_len != 0 || !f0.alph.empty();
    if (need_vp8x) {
        std::vector<uint8_t> x;
        x.push_back((uint8_t)((anim ? 0x02 : 0) | (any_alpha ? 0x10 : 0) | (icc_len ? 0x20 : 0)));
        x.insert(x.end(), 3, 0);
        put_le24(x, (uint32_t)f0.width - 1);
        put_le24(x, (uint32_t)f0.height - 1);
        put_chunk(body, "VP8X", x.data(), x.size());
        if (icc_len) put_chunk(body, "ICCP", icc, icc_len);
    }
    if (anim) {
        std::vector<uint8_t> a;
        put_le32(a, bgcolor);
        a.push_back((uint8_t)(loop_count & 0xff));
        a.push_back((uint8_t)((loop_count >> 8) & 0xff));
        put_chunk(body, "ANIM", a.data(), a.size());
        for (int i = 0; i < n; i++) {
            const WebpEncodedFrame& f = frames[i];
            std::vector<uint8_t> m;
            put_le24(m, 0);
            put_le24(m, 0);
            put_le24(m, (uint32_t)f.width - 1);
            put_le24(m, (uint32_t)f.height - 1);
            put_le24(m, (uint32_t)(f.duration < 0 ? 0 : f.duration > 0xffffff ? 0xffffff : f.duration));
            m.push_back(0x02);  // do not blend, do not dispose: every frame is a full canvas
            put_image_chunks(m, f);
            put_chunk(body, "ANMF", m.data(), m.size());
        }
    } else {
        put_image_chunks(body, f0);
    }
    std::vector<uint8_t>& file = *file_out;
    file.clear();
    file.insert(file.end(), {'R', 'I', 'F', 'F'});
    put_le32(file, (uint32_t)(4 + body.size()));
    file.insert(file.end(), {'W', 'E', 'B', 'P'});
    file.insert(file.end(), body.begin(), body.end());
}

}  // namespace lp

using namespace lp;

struct webp_encoder_struct {
    uint8_t* dst = nullptr;
    size_t dst_len = 0;
    std::vector<uint8_t> icc;
    uint32_t bgcolor = 0, loop_count = 0;
    int frame_count = 1;  // ref webp.cpp:401: counts from 1
    int first_frame_delay = 0;
    std::vector<EncodedFrame> frames;
};

extern "C" {

// ref webp.cpp:388-421
webp_encoder webp_encoder_create(void* buf, size_t buf_len, const void* icc, size_t icc_len, uint32_t bgcolor, int loop_count) {
    auto* e = new webp_encoder_struct;
    e->dst = static_cast<uint8_t*>(buf);
    e->dst_len = buf_len;
    if (icc_len) e->icc.assign(static_cast<const uint8_t*>(icc), static_cast<const uint8_t*>(icc) + icc_len);
    e->bgcolor = bgcolor;
    e->loop_count = (uint32_t)loop_count;
    return e;
}

// ref webp.cpp:423-560 (finalisation), 562-760 (frames)
size_t webp_encoder_write(webp_encoder e, const opencv_mat src, const int* opt, size_t opt_len, int delay, int, int, int,
                          int) {
    if (!e) return 0;
    // options (ref webp.cpp:451-498): only quality / lossless change what this encoder does
    float quality = 100.0f;
    bool lossless = false;
    for (size_t i = 0; opt && i + 1 < opt_len; i += 2) {
        if (opt[i] == CV_IMWRITE_WEBP_QUALITY) {
            const float q = opt[i + 1] < 1 ? 1.0f : (float)opt[i + 1];
            quality = q > 100.0f ? 100.0f : q;
            lossless = q > 100.0f;
        }
    }
    if (!src) {  // finalise
        if (e->frame_count == 1 || e->frames.empty()) return 0;
        std::vector<uint8_t> file;
        webp_assemble(e->frames.data(), (int)e->frames.size(), e->icc.data(), e->icc.size(), e->bgcolor, e->loop_count, &file);
        if (file.size() > e->dst_len) {
            fprintf(stderr, "Error: Final encoded size (%zu) exceeds buffer size (%zu)\n", file.size(), e->dst_len);
            return 0;
        }
        memcpy(e->dst, file.data(), file.size());
        return file.size();
    }
    int cols = 0, rows = 0, type = 0;
    const uint8_t* dev = nullptr;
    size_t step = 0;
    if (mat_device_view(src, &cols, &rows, &type, &dev, &step)) return 0;
    if (type != CV_8UC3 && type != CV_8UC4) {
        // (the reference converts 1-channel input to BGR first, ref webp.cpp:576-585; not on this path yet)
        fprintf(stderr, "[lilliput_b200] WebP encoder needs a BGR or BGRA frame\n");
        return 0;
    }
    if (cols > 16383 || rows > 16383) return 0;  // WebP's 14-bit dimensions
    if (!e->frames.empty() && (cols != e->frames[0].width || rows != e->frames[0].height)) {
        fprintf(stderr, "[lilliput_b200] WebP animation frames must share the canvas size\n");
        return 0;
    }
    const int channels = type == CV_8UC4 ? 4 : 3;
    cudaStream_t st = thread_stream();
    EncodedFrame f;
    if (lossless) {
        std::vector<WebpEncodedFrame> one;
        if (webp_encode_lossless_batch(dev, 0, step, cols, rows, channels, 1, &one, st)) return 0;
        f = std::move(one[0]);
    } else {
        std::vector<WebpEncodedFrame> one;
        if (webp_encode_lossy_batch(dev, 0, step, cols, rows, channels, 1, (int)quality, &one, st) || one[0].image.empty())
            return 0;
        f = std::move(one[0]);
    }
    f.lossless = lossless;
    f.duration = delay;
    if (e->frames.empty()) e->first_frame_delay = delay;
    const size_t size = f.image.size() + f.alph.size();
    e->frames.push_back(std::move(f));
    e->frame_count++;
    return size;
}

void webp_encoder_release(webp_encoder e) { delete e; }

size_t webp_encoder_flush(webp_encoder e) { return webp_encoder_write(e, nullptr, nullptr, 0, 0, 0, 0, 0, 0); }

}  // extern "C"
