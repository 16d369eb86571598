// png_encode.cu -- PNG encode on sm_90a: scanline filtering + DEFLATE (hash-chain LZ77 whose search effort follows
// PngCompression, per-chunk dynamic Huffman codes, independent 32 KB chunks joined by sync-flush blocks:
// deflate_enc_core.h) + checksums and container, all on the device, for N frames of one geometry per launch.
//
// Replaces: opencv_encoder_write for ".png" (ref opencv.cpp:185-194 -> cv::ImageEncoder::write ->
// OpenCV grfmt_png -> libpng 1.6.47 + zlib-ng 2.3.3).  PNG is lossless and the contract for this
// path is DECODED-PIXEL equality with identical IHDR policy (BGR -> colour type 2, BGRA -> 6,
// Gray -> 0, 8-bit, non-interlaced, no ancillary chunks), not byte-identical files: reproducing
// zlib-ng's match finder bit for bit is neither possible nor useful (SURVEY.md section 7).
// Filter policy follows what OpenCV asks libpng for: with IMWRITE_PNG_COMPRESSION given, libpng's
// adaptive minimum-sum-of-absolute-differences heuristic over None/Sub/Up/Average/Paeth; without
// it, Sub on every row.  Level 0 emits stored blocks.
//
// Kernels, each ONE launch over all N frames (png_encode_batch; the per-image encoder is that launcher with N = 1):
//   png_filter_kernel    warp per (image, scanline): the five candidate sums, pick, write [type][bytes].
//   png_deflate_kernel   warp per (image, 32 KB chunk): lane 0 runs defenc::write_chunk (LZ77 tokens into global scratch,
//                        symbol statistics -> length-limited dynamic Huffman codes in shared memory, or fixed
//                        codes / a stored block when smaller); every chunk ends byte-aligned with an empty stored
//                        block, so chunks are independent and concatenate by memcpy.  All lanes compute the chunk's
//                        Adler-32 partial sums and, once lane 0 has written it, the CRC-32 of the compressed chunk
//                        (a slice per lane, joined by the rule of crc32_core.h).
//   png_pack_kernel      CTA per image: prefix sum of chunk sizes, the chunks copied into the image's file slot behind
//                        signature / IHDR / IDAT header, Adler-32 and the IDAT CRC-32 folded from the chunk partials,
//                        zlib header and final block, IHDR CRC, IEND.  A file that does not fit its slot gets length 0.
// The host does nothing per file but copy it.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"
#include "lp_opencv.h"

#define LP_DEF_FN static __device__
#define LP_DEF_TABLE static __device__ const
#include "deflate_enc_core.h"
#define LP_CRC_FN static __device__
#include "crc32_core.h"

namespace lp {

constexpr int kChunk = defenc::kChunk;        // uncompressed bytes per DEFLATE chunk
constexpr int kChunkOut = defenc::kChunkOut;  // worst case: stored fallback
constexpr int kDefWarps = 2;                  // (defenc::Work is ~15 KB of shared memory per chunk in flight)
constexpr int kPackThreads = 256;
// A file: signature 8 | IHDR chunk 25 | IDAT length + type 8 | zlib header 2 | DEFLATE chunks | final block 2 |
// Adler-32 4 | IDAT CRC 4 | IEND chunk 12
constexpr uint32_t kChunksAt = 8 + 25 + 8 + 2;
constexpr uint32_t kFileOverhead = kChunksAt + 2 + 4 + 4 + 12;

// ------------------------------------------------------------------ filtering

__device__ __forceinline__ int paeth_pred(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// Sample k of pixel x in PNG order (RGB[A] / Gray) from a packed BGR[A] / Gray frame row.
__device__ __forceinline__ int png_sample(const uint8_t* row, int x, int k, int C) {
    if (x < 0 || !row) return 0;
    const int c = (C >= 3 && k < 3) ? 2 - k : k;  // swap B and R
    return row[(size_t)x * C + c];
}

// image i: frame at frames + i * img_stride, filtered scanlines at filt + i * filt_stride
__global__ void __launch_bounds__(128)
    png_filter_kernel(const uint8_t* frames, size_t img_stride, size_t row_stride, int W, int H, int C, int n, int adaptive,
                      uint8_t* filt, size_t filt_stride) {
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= (long long)n * H) return;
    const int img = (int)(warp / H), y = (int)(warp % H);
    const uint8_t* frame = frames + (size_t)img * img_stride;
    const uint8_t* cur = frame + (size_t)y * row_stride;
    const uint8_t* up = y > 0 ? frame + (size_t)(y - 1) * row_stride : nullptr;
    const int nbytes = W * C;
    int best = 1;  // Sub (OpenCV's no-parameter default)
    if (adaptive) {
        uint32_t sum[5] = {0, 0, 0, 0, 0};
        for (int i = lane; i < nbytes; i += 32) {
            const int x = i / C, k = i % C;
            const int v = png_sample(cur, x, k, C), a = png_sample(cur, x - 1, k, C);
            const int b = png_sample(up, x, k, C), c = png_sample(up, x - 1, k, C);
            const int f[5] = {v, v - a, v - b, v - ((a + b) >> 1), v - paeth_pred(a, b, c)};
#pragma unroll
            for (int t = 0; t < 5; t++) {
                const int u = f[t] & 0xff;
                sum[t] += u < 128 ? u : 256 - u;  // libpng: |signed byte|
            }
        }
#pragma unroll
        for (int t = 0; t < 5; t++)
#pragma unroll
            for (int o = 16; o; o >>= 1) sum[t] += __shfl_xor_sync(0xffffffffu, sum[t], o);
        best = 0;
#pragma unroll
        for (int t = 1; t < 5; t++)
            if (sum[t] < sum[best]) best = t;  // strict <: the earliest filter wins ties, as in libpng
    }
    uint8_t* out = filt + (size_t)img * filt_stride + (size_t)y * (nbytes + 1);
    if (lane == 0) out[0] = (uint8_t)best;
    for (int i = lane; i < nbytes; i += 32) {
        const int x = i / C, k = i % C;
        const int v = png_sample(cur, x, k, C), a = png_sample(cur, x - 1, k, C);
        const int b = png_sample(up, x, k, C), c = png_sample(up, x - 1, k, C);
        const int p = best == 0 ? 0 : best == 1 ? a : best == 2 ? b : best == 3 ? ((a + b) >> 1) : paeth_pred(a, b, c);
        out[1 + i] = (uint8_t)(v - p);
    }
}

// ------------------------------------------------------------------ checksums of one chunk (a warp)

// Adler-32 partials of p[0, n): A = sum b_i, B = sum (n - i) b_i, both mod 65521 (every lane returns them)
__device__ __forceinline__ uint2 warp_adler_partials(const uint8_t* p, int n, int lane) {
    uint64_t A = 0, B = 0;
    for (int i = lane; i < n; i += 32) {
        A += p[i];
        B += (uint64_t)(n - i) * p[i];
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        A += __shfl_xor_sync(0xffffffffu, A, o);
        B += __shfl_xor_sync(0xffffffffu, B, o);
    }
    return make_uint2((uint32_t)(A % crc32core::kAdlerMod), (uint32_t)(B % crc32core::kAdlerMod));
}

// CRC-32 of p[0, n): lane l takes bytes [l * s, (l + 1) * s) with s = ceil(n / 32) (the last slices may be short or
// empty), then neighbouring runs of slices are joined pairwise, crc(A || B) = crc(A) * x^(8 |B|) xor crc(B).  The
// result is lane 0's.
__device__ __forceinline__ uint32_t warp_crc32(const uint8_t* p, uint32_t n, int lane) {
    const uint32_t s = (n + 31) / 32;
    const uint32_t beg = min(n, (uint32_t)lane * s), end = min(n, beg + s);
    uint32_t len = end - beg;
    uint32_t c = crc32core::update(0, p + beg, len);
#pragma unroll 1
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t c_hi = __shfl_down_sync(0xffffffffu, c, o), l_hi = __shfl_down_sync(0xffffffffu, len, o);
        if (lane + o < 32) {
            c = crc32core::combine(c, c_hi, l_hi);
            len += l_hi;
        }
    }
    return c;
}

// ------------------------------------------------------------------ DEFLATE

// Chunk j of image i is job i * nchunks + j.  chunk_len[job] = compressed bytes (each job owns kChunkOut bytes of
// `comp`), chunk_crc[job] their CRC-32, adler[job] = the Adler-32 partials of the chunk's filtered bytes.
// scratch: per job kChunk uint16 of hash-chain links + defenc::kTokCap uint16 of tokens.
__global__ void __launch_bounds__(kDefWarps * 32)
    png_deflate_kernel(const uint8_t* filt, size_t filt_stride, size_t raw, int nchunks, int njobs, int level, uint8_t* comp,
                       uint32_t* chunk_len, uint32_t* chunk_crc, uint2* adler, uint16_t* scratch) {
    __shared__ defenc::Work work[kDefWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int job = blockIdx.x * kDefWarps + warp;
    if (job >= njobs) return;
    const int img = job / nchunks, chunk = job % nchunks;
    const uint8_t* src = filt + (size_t)img * filt_stride + (size_t)chunk * kChunk;
    const int n = (int)min((size_t)kChunk, raw - (size_t)chunk * kChunk);
    uint8_t* dst = comp + (size_t)job * kChunkOut;
    const uint2 ad = warp_adler_partials(src, n, lane);
    uint32_t len = 0;
    if (lane == 0) {
        uint16_t* prev = scratch + (size_t)job * (kChunk + defenc::kTokCap);
        len = (uint32_t)defenc::write_chunk(src, n, level, work[warp], prev, prev + kChunk, dst);
    }
    __syncwarp();  // lane 0's bytes are visible to the other lanes from here
    len = __shfl_sync(0xffffffffu, len, 0);
    const uint32_t crc = warp_crc32(dst, len, lane);
    if (lane == 0) {
        adler[job] = ad;
        chunk_len[job] = len;
        chunk_crc[job] = crc;
    }
}

// ------------------------------------------------------------------ pack

__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t x) {
    p[0] = (uint8_t)(x >> 24);
    p[1] = (uint8_t)(x >> 16);
    p[2] = (uint8_t)(x >> 8);
    p[3] = (uint8_t)x;
}

// Block-wide (kPackThreads): the CRC-32 of the concatenation of `nchunks` pieces (piece c: `len[c]` bytes at offset
// `off[c]` of `total`, CRC `crc[c]`) and the Adler-32 of the `raw` bytes the pieces' partials `adler[c]` cover (piece c
// = bytes [c * kChunk, ...)), by the rules of crc32_core.h: every thread folds a strided share of the pieces, then the
// shares are xor-ed / summed.  Thread 0 returns the results.
__device__ void fold_checksums(const uint32_t* len, const uint32_t* off, const uint32_t* crc, const uint2* adler, int nchunks,
                               uint32_t total, size_t raw, uint32_t* out_crc, uint32_t* out_adler) {
    __shared__ uint32_t s_crc[kPackThreads / 32];
    __shared__ unsigned long long s_s1[kPackThreads / 32], s_s2[kPackThreads / 32];
    uint32_t x = 0;
    unsigned long long s1 = 0, s2 = 0;
    for (int c = threadIdx.x; c < nchunks; c += kPackThreads) {
        x ^= crc32core::mulmod(crc[c], crc32core::xpow8(total - (off[c] + len[c])));
        const size_t p = (size_t)c * kChunk, n = min((size_t)kChunk, raw - p);
        s1 += adler[c].x;
        s2 += crc32core::adler_s2_term(raw, p, n, adler[c].x, adler[c].y);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        x ^= __shfl_xor_sync(0xffffffffu, x, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if ((threadIdx.x & 31) == 0) {
        s_crc[threadIdx.x >> 5] = x;
        s_s1[threadIdx.x >> 5] = s1;
        s_s2[threadIdx.x >> 5] = s2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kPackThreads / 32; w++) {
            x ^= s_crc[w];
            s1 += s_s1[w];
            s2 += s_s2[w];
        }
        s1 = (1 + s1) % crc32core::kAdlerMod;
        s2 = (raw % crc32core::kAdlerMod + s2) % crc32core::kAdlerMod;
        *out_crc = x;
        *out_adler = (uint32_t)((s2 << 16) | s1);
    }
}

// Exclusive prefix sum of len[0, n) into off[0, n) (block-wide); every thread returns the total.
__device__ uint32_t block_offsets(const uint32_t* len, int n, uint32_t* off) {
    __shared__ uint32_t s_warp[kPackThreads / 32], s_carry;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += kPackThreads) {
        const int c = base + threadIdx.x;
        const uint32_t v = c < n ? len[c] : 0;
        uint32_t inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += t;
        }
        if (lane == 31) s_warp[wid] = inc;
        __syncthreads();
        uint32_t before = s_carry;
        for (int w = 0; w < wid; w++) before += s_warp[w];
        if (c < n) off[c] = before + inc - v;
        __syncthreads();
        if (threadIdx.x == kPackThreads - 1) s_carry = before + inc;
        __syncthreads();
    }
    return s_carry;
}

// One image per CTA: its chunks -> a complete file in files + image * slot; file_len[image] = 0 when it does not fit.
__global__ void __launch_bounds__(kPackThreads)
    png_pack_kernel(const uint8_t* comp, const uint32_t* chunk_len, const uint32_t* chunk_crc, const uint2* adler,
                    uint32_t* chunk_off, int nchunks, size_t raw, int W, int H, int C, uint8_t* files, size_t slot,
                    uint32_t* file_len) {
    const size_t job0 = (size_t)blockIdx.x * nchunks;
    comp += job0 * kChunkOut;
    chunk_len += job0;
    chunk_crc += job0;
    adler += job0;
    chunk_off += job0;
    uint8_t* file = files + (size_t)blockIdx.x * slot;
    const uint32_t total = block_offsets(chunk_len, nchunks, chunk_off);
    if ((size_t)total + kFileOverhead > slot) {
        if (threadIdx.x == 0) file_len[blockIdx.x] = 0;
        return;
    }
    __syncthreads();  // the offsets, written by other threads, are read below
    for (int c = threadIdx.x >> 5; c < nchunks; c += kPackThreads / 32) {
        const uint8_t* s = comp + (size_t)c * kChunkOut;
        uint8_t* d = file + kChunksAt + chunk_off[c];
        const uint32_t len = chunk_len[c];
        for (uint32_t i = threadIdx.x & 31; i < len; i += 32) d[i] = s[i];
    }
    uint32_t crc_chunks = 0, adler32 = 0;
    fold_checksums(chunk_len, chunk_off, chunk_crc, adler, nchunks, total, raw, &crc_chunks, &adler32);
    if (threadIdx.x != 0) return;
    const uint8_t sig[8] = {0x89, 0x50, 0x4E, 0x47, 0x0D, 0x0A, 0x1A, 0x0A};
    for (int i = 0; i < 8; i++) file[i] = sig[i];
    uint8_t* p = file + 8;
    put_be32(p, 13);
    p[4] = 'I'; p[5] = 'H'; p[6] = 'D'; p[7] = 'R';
    put_be32(p + 8, (uint32_t)W);
    put_be32(p + 12, (uint32_t)H);
    p[16] = 8;
    p[17] = C == 1 ? 0 : C == 3 ? 2 : 6;
    p[18] = p[19] = p[20] = 0;
    put_be32(p + 21, crc32core::update(0, p + 4, 17));
    p += 25;
    put_be32(p, total + 2 + 2 + 4);  // zlib header, chunks, final block, Adler-32
    p[4] = 'I'; p[5] = 'D'; p[6] = 'A'; p[7] = 'T';
    p[8] = 0x78;
    p[9] = 0x01;
    uint32_t crc = crc32core::combine(crc32core::update(0, p + 4, 6), crc_chunks, total);
    p = file + kChunksAt + total;
    p[0] = 0x03;  // BFINAL = 1, BTYPE = 01, EOB (7 zero bits)
    p[1] = 0x00;
    put_be32(p + 2, adler32);
    crc = crc32core::update(crc, p, 6);
    put_be32(p + 6, crc);
    put_be32(p + 10, 0);
    p[14] = 'I'; p[15] = 'E'; p[16] = 'N'; p[17] = 'D';
    put_be32(p + 18, crc32core::update(0, p + 14, 4));
    file_len[blockIdx.x] = total + kFileOverhead;
}

// ------------------------------------------------------------------ host side

void png_encode_policy(const int* opt, size_t opt_len, int* level, bool* adaptive) {
    *level = 1;
    *adaptive = false;
    for (size_t i = 0; i + 1 < opt_len; i += 2)
        if (opt[i] == CV_IMWRITE_PNG_COMPRESSION) {
            *level = std::min(std::max(opt[i + 1], 0), 9);
            *adaptive = true;
        }
}

namespace {
struct PngScratch {  // byte offsets into the caller's scratch, for n frames of one geometry
    size_t raw, filt_stride, njobs;
    int nchunks;
    size_t comp, len, off, crc, adler, lz, bytes;
};
PngScratch png_scratch(int W, int H, int C, int n, int level) {
    PngScratch s;
    s.raw = ((size_t)W * C + 1) * H;
    s.filt_stride = round_up(s.raw, (size_t)16);
    s.nchunks = (int)ceil_div(s.raw, (size_t)kChunk);
    s.njobs = (size_t)n * s.nchunks;
    s.comp = round_up((size_t)n * s.filt_stride, (size_t)256);
    s.len = s.comp + round_up(s.njobs * kChunkOut, (size_t)256);
    s.off = s.len + round_up(s.njobs * 4, (size_t)256);
    s.crc = s.off + round_up(s.njobs * 4, (size_t)256);
    s.adler = s.crc + round_up(s.njobs * 4, (size_t)256);
    s.lz = s.adler + round_up(s.njobs * 8, (size_t)256);
    s.bytes = s.lz + (level == 0 ? 0 : s.njobs * (kChunk + defenc::kTokCap) * sizeof(uint16_t));
    return s;
}
}  // namespace

size_t png_encode_max_file_bytes(int W, int H, int C) {
    return ceil_div(((size_t)W * C + 1) * H, (size_t)kChunk) * kChunkOut + kFileOverhead;
}

size_t png_encode_batch_scratch_bytes(int W, int H, int C, int n, int level) { return png_scratch(W, H, C, n, level).bytes; }

int png_encode_batch(const uint8_t* d_frames, size_t img_stride, size_t row_stride, int W, int H, int C, int n, int level,
                     bool adaptive, uint8_t* d_files, size_t slot, uint32_t* d_len, void* scratch, cudaStream_t st) {
    if (W < 1 || H < 1 || (C != 1 && C != 3 && C != 4) || n < 1 || !d_frames || !d_files || !d_len || !scratch)
        return LP_ERR_BAD_ARGUMENT;
    const int lvl = level < 0 ? 1 : level > 9 ? 9 : level;  // zlib's range; OpenCV's own default is 1
    const PngScratch s = png_scratch(W, H, C, n, lvl);
    if (s.njobs > (size_t)INT32_MAX || (size_t)n * H > (size_t)INT32_MAX * 4) return LP_ERR_BAD_ARGUMENT;
    uint8_t* buf = static_cast<uint8_t*>(scratch);
    uint32_t* chunk_len = reinterpret_cast<uint32_t*>(buf + s.len);
    uint32_t* chunk_off = reinterpret_cast<uint32_t*>(buf + s.off);
    uint32_t* chunk_crc = reinterpret_cast<uint32_t*>(buf + s.crc);
    uint2* adler = reinterpret_cast<uint2*>(buf + s.adler);
    png_filter_kernel<<<(unsigned)ceil_div((long long)n * H * 32, 128LL), 128, 0, st>>>(d_frames, img_stride, row_stride, W, H, C, n,
                                                                                      adaptive ? 1 : 0, buf, s.filt_stride);
    png_deflate_kernel<<<(unsigned)ceil_div(s.njobs, (size_t)kDefWarps), kDefWarps * 32, 0, st>>>(
        buf, s.filt_stride, s.raw, s.nchunks, (int)s.njobs, lvl, buf + s.comp, chunk_len, chunk_crc, adler,
        reinterpret_cast<uint16_t*>(buf + s.lz));
    png_pack_kernel<<<n, kPackThreads, 0, st>>>(buf + s.comp, chunk_len, chunk_crc, adler, chunk_off, s.nchunks, s.raw, W, H, C,
                                               d_files, slot, d_len);
    g_launches += 3;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

// Encodes one packed device frame to a PNG file in `out` (host): a batch of one.  Returns LP_OK / error.
int png_encode_frame(const uint8_t* frame, size_t row_stride, int W, int H, int C, int level, bool adaptive,
                     std::vector<uint8_t>* out, cudaStream_t st) {
    if (W < 1 || H < 1 || (C != 1 && C != 3 && C != 4)) return LP_ERR_BAD_ARGUMENT;
    const size_t slot = round_up(png_encode_max_file_bytes(W, H, C), (size_t)256);  // every chunk stored: always fits
    const size_t scratch_bytes = round_up(png_encode_batch_scratch_bytes(W, H, C, 1, level), (size_t)256);
    uint8_t* buf = nullptr;
    LP_CUDA_OK(cudaMallocAsync(&buf, scratch_bytes + slot + 256, st));
    uint8_t* d_file = buf + scratch_bytes;
    uint32_t* d_len = reinterpret_cast<uint32_t*>(d_file + slot);
    uint32_t len = 0;
    int rc = png_encode_batch(frame, 0, row_stride, W, H, C, 1, level, adaptive, d_file, slot, d_len, buf, st);
    if (!rc && (cudaMemcpyAsync(&len, d_len, 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess ||
                len == 0 || len > slot))
        rc = LP_ERR_CUDA;
    if (!rc) {
        out->resize(len);
        if (cudaMemcpyAsync(out->data(), d_file, len, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess)
            rc = LP_ERR_CUDA;
    }
    cudaFreeAsync(buf, st);
    return rc;
}

// ------------------------------------------------------------------ test entry points

// CRC-32 and Adler-32 of a device buffer the way the encoder computes them: a warp per 32 KB piece (warp_crc32,
// warp_adler_partials), the pieces folded by fold_checksums.  work: 3 uint32 per piece.
__global__ void __launch_bounds__(kPackThreads)
    png_checksum_kernel(const uint8_t* data, size_t n, int npieces, uint32_t* work, uint2* adler, uint32_t* out2) {
    uint32_t *len = work, *off = work + npieces, *crc = work + 2 * (size_t)npieces;
    for (int c = threadIdx.x >> 5; c < npieces; c += kPackThreads / 32) {
        const size_t p = (size_t)c * kChunk;
        const uint32_t l = (uint32_t)min((size_t)kChunk, n - p);
        const uint2 ad = warp_adler_partials(data + p, (int)l, threadIdx.x & 31);
        const uint32_t x = warp_crc32(data + p, l, threadIdx.x & 31);
        if ((threadIdx.x & 31) == 0) {
            len[c] = l;
            off[c] = (uint32_t)p;
            crc[c] = x;
            adler[c] = ad;
        }
    }
    __syncthreads();
    fold_checksums(len, off, crc, adler, npieces, (uint32_t)n, n, &out2[0], &out2[1]);
}

}  // namespace lp

using namespace lp;

extern "C" int lp_png_checksums_dev(const uint8_t* d_data, size_t n, uint32_t* crc32, uint32_t* adler32) {
    if (ensure_device()) return LP_ERR_CUDA;
    if (!crc32 || !adler32 || (n && !d_data) || n > 0xFFFFFFFFull) return LP_ERR_BAD_ARGUMENT;
    cudaStream_t st = thread_stream();
    const int npieces = (int)ceil_div(n, (size_t)kChunk);
    // pieces' {len, off, crc} | their Adler partials | the two results
    const size_t adler_at = round_up((size_t)npieces * 12, (size_t)256), out_at = adler_at + round_up((size_t)npieces * 8, (size_t)256);
    uint8_t* buf = nullptr;
    LP_CUDA_OK(cudaMallocAsync(&buf, out_at + 256, st));
    uint32_t* d_out = reinterpret_cast<uint32_t*>(buf + out_at);
    png_checksum_kernel<<<1, kPackThreads, 0, st>>>(d_data, n, npieces, reinterpret_cast<uint32_t*>(buf),
                                                    reinterpret_cast<uint2*>(buf + adler_at), d_out);
    g_launches++;
    uint32_t h[2] = {0, 0};
    const bool ok = cudaGetLastError() == cudaSuccess &&
                    cudaMemcpyAsync(h, d_out, 8, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
                    cudaStreamSynchronize(st) == cudaSuccess;
    cudaFreeAsync(buf, st);
    if (!ok) return LP_ERR_CUDA;
    *crc32 = h[0];
    *adler32 = h[1];
    return LP_OK;
}

// n packed device frames of one geometry -> n PNG files in device slots (d_len[i] = 0: did not fit), as lp_xbatch's
// PNG sink calls the encoder.
extern "C" int lp_png_encode_batch_dev(const uint8_t* d_frames, size_t img_stride, size_t row_stride, int width, int height,
                                       int channels, int n, int level, int adaptive, uint8_t* d_files, size_t slot,
                                       uint32_t* d_len) {
    if (ensure_device()) return LP_ERR_CUDA;
    cudaStream_t st = thread_stream();
    void* scratch = nullptr;
    LP_CUDA_OK(cudaMallocAsync(&scratch, png_encode_batch_scratch_bytes(width, height, channels, n, level) + 256, st));
    const int rc = png_encode_batch(d_frames, img_stride, row_stride, width, height, channels, n, level, adaptive != 0, d_files,
                                    slot, d_len, scratch, st);
    cudaFreeAsync(scratch, st);
    if (rc) return rc;
    LP_CUDA_OK(cudaStreamSynchronize(st));
    return LP_OK;
}
