// png_decode.cu -- PNG pixel decode on sm_90a: zlib inflate -> scanline defilter -> packed
// Gray / BGR / BGRA u8, as cv::ImageDecoder::readData produces it for lilliput's 8-bit Framebuffer.
//
// Replaces: opencv_decoder_read_data for PNG inputs (ref opencv.cpp:166-171 -> OpenCV grfmt_png ->
// libpng 1.6.47 + zlib-ng 2.3.3).  Lossless: the result is bit-identical to the reference
// (tests/test_gpu_png.py).  Transform set (SURVEY.md Appendix D/E.4): 16-bit -> high byte,
// palette -> BGR (+A with tRNS), gray 1/2/4 -> 8 by replication, gray+alpha -> B=G=R,A, RGB(A) -> BGR(A).
//
// A DEFLATE stream is one serial bit string with back-references, so the unit of parallelism is the
// image: one warp per image.
//   png_inflate_kernel   lane 0 walks the Huffman symbols (10-bit lookahead tables in shared memory);
//                        LZ77 copies and stored blocks are done by all 32 lanes.
//   png_defilter_kernel  32 scanlines at a time, lane r one scanline, skewed by one pixel per lane so
//                        that "up" comes from lane r-1 by shuffle and "left"/"upper-left" stay in
//                        registers (Sub/Up/Average/Paeth, modulo 256), in place.
//   png_convert_kernel   one thread per output pixel.
#include <cstring>

#include "common.cuh"
#include "kernels.cuh"
#include "inflate_core.h"

namespace lp {

constexpr int kPngWarps = 2;  // warps (= images) per CTA: 2 x ~17 KB of shared memory, 6 CTAs = 12 images per SM

// One warp per image; the decoder itself is inflate_core.h (speculative per-lane subsequence decoding,
// shared-memory output ring, 16-byte flushes).  Dynamic shared memory: one WarpShared per warp.
__global__ void __launch_bounds__(kPngWarps * 32)
    png_inflate_kernel(PngDecodeItem* items, const uint8_t* zall, uint8_t* rawall, lpinf::Match* mlists, int n) {
    extern __shared__ __align__(16) uint8_t inflate_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int img = blockIdx.x * kPngWarps + warp;
    if (img >= n) return;
    PngDecodeItem& it = items[img];
    if (it.status != 0) return;
    lpinf::WarpShared& ws = reinterpret_cast<lpinf::WarpShared*>(inflate_smem)[warp];
    lpinf::Stream s;
    s.z = zall + it.z_off;
    s.z_len = it.z_len;
    s.out = rawall + it.raw_off;
    s.cap = it.raw_total;
    s.mlist = mlists + (size_t)img * lpinf::kMaxMatches;
    uint32_t produced = 0;
    int status = lpinf::inflate_stream(ws, s, &produced);
    if (lane == 0) {
        if (!status && produced < it.raw_total) status = -3;  // fewer scanline bytes than the header promises
        it.status = status;
        it.produced = produced;
    }
}

// ------------------------------------------------------------------ defilter

__device__ __forceinline__ int paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// BPP = bytes per complete pixel (1,2,3,4,6,8).  Lane r owns scanline y0 + r and, at step t, pixel
// t - r: the pixel above it was produced by lane r-1 one step earlier.
template <int BPP>
__device__ void defilter_image(uint8_t* raw, uint32_t row_bytes, int height) {
    const int lane = threadIdx.x & 31;
    const uint32_t pitch = row_bytes + 1;
    const int npx = (int)((row_bytes + BPP - 1) / BPP);
    for (int y0 = 0; y0 < height; y0 += 32) {
        const int y = y0 + lane;
        const bool live = y < height;
        uint8_t* row = raw + (size_t)(live ? y : 0) * pitch;
        const int ft = live ? row[0] : 0;
        const uint8_t* above = (y0 > 0) ? raw + (size_t)(y0 - 1) * pitch + 1 : nullptr;  // lane 0's "up"
        uint8_t left[BPP], up[BPP], upleft[BPP], cur[BPP];
#pragma unroll
        for (int k = 0; k < BPP; k++) left[k] = up[k] = upleft[k] = cur[k] = 0;
        for (int t = 0; t < npx + 31; t++) {
            // what lane r-1 produced in the previous step is the pixel above this lane's pixel
            uint32_t lo = 0, hi = 0;
#pragma unroll
            for (int k = 0; k < BPP; k++) {
                if (k < 4) lo |= (uint32_t)cur[k] << (8 * k);
                else hi |= (uint32_t)cur[k] << (8 * (k - 4));
            }
            uint32_t ulo = __shfl_up_sync(0xffffffffu, lo, 1), uhi = BPP > 4 ? __shfl_up_sync(0xffffffffu, hi, 1) : 0;
            const int x = t - lane;
            const bool act = live && x >= 0 && x < npx;
#pragma unroll
            for (int k = 0; k < BPP; k++) {
                upleft[k] = up[k];
                if (lane == 0) {
                    const uint32_t bi = (uint32_t)x * BPP + k;
                    up[k] = (above && act && bi < row_bytes) ? above[bi] : 0;
                } else {
                    up[k] = (uint8_t)((k < 4 ? ulo >> (8 * k) : uhi >> (8 * (k - 4))) & 0xff);
                }
            }
            if (act) {
#pragma unroll
                for (int k = 0; k < BPP; k++) {
                    const uint32_t bi = (uint32_t)x * BPP + k;
                    if (bi < row_bytes) {
                        int v = row[1 + bi];
                        const int a = left[k], b = up[k], c = upleft[k];
                        v += ft == 1 ? a : ft == 2 ? b : ft == 3 ? ((a + b) >> 1) : ft == 4 ? paeth(a, b, c) : 0;
                        cur[k] = (uint8_t)v;
                        row[1 + bi] = (uint8_t)v;
                    }
                }
#pragma unroll
                for (int k = 0; k < BPP; k++) left[k] = cur[k];
            } else if (x < 0) {
#pragma unroll
                for (int k = 0; k < BPP; k++) up[k] = 0;  // not started: nothing above-left yet
            }
        }
        __syncwarp();
        __threadfence_block();
    }
}

// ---- fused path: 8-bit truecolour (colour type 2 without tRNS, or 6), not interlaced -------------------------
// Defilter + RGB(A) -> BGR(A) in one pass: the filtered scanlines are only READ (so they stay in L1; the in-place
// version above invalidates the very line it reads next with each store) and the packed frame is only written.
// Lane r owns scanline y0 + r; per iteration it takes FOUR pixels, one chunk behind lane r-1, whose four output
// pixels of the previous iteration are exactly the pixels above it (shuffled as one word per pixel).  The raw
// bytes of the next chunk are fetched (aligned words + funnel shift) before the current one is worked on.

__device__ __forceinline__ bool png_fused_ok(const PngDecodeItem& it) {
    return it.bit_depth == 8 && !it.interlace && ((it.color_type == 2 && it.out_channels == 3) || it.color_type == 6);
}

// NW 32-bit words starting at (possibly unaligned) p
template <int NW>
__device__ __forceinline__ void load_words_unaligned(const uint8_t* p, uint32_t* out) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(a & 3) * 8;
    uint32_t w[NW + 1];
#pragma unroll
    for (int k = 0; k <= NW; k++) w[k] = q[k];
#pragma unroll
    for (int k = 0; k < NW; k++) out[k] = __funnelshift_r(w[k], w[k + 1], sh);
}

__device__ __forceinline__ uint32_t png_unfilter_px(uint32_t x, uint32_t a, uint32_t b, uint32_t c, int ft, int nbytes) {
    uint32_t r = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (k < nbytes) {
            const int xv = (x >> (8 * k)) & 255, av = (a >> (8 * k)) & 255, bv = (b >> (8 * k)) & 255, cv = (c >> (8 * k)) & 255;
            int pred;
            if (ft == 1) pred = av;
            else if (ft == 2) pred = bv;
            else if (ft == 3) pred = (av + bv) >> 1;
            else if (ft == 4) pred = paeth(av, bv, cv);
            else pred = 0;
            r |= (uint32_t)((xv + pred) & 255) << (8 * k);
        }
    }
    return r;
}

template <int BPP>  // 3 or 4
__device__ void defilter_to_frame(const uint8_t* raw, uint32_t row_bytes, int width, int height, uint8_t* frame,
                                  uint32_t frame_stride) {
    const int lane = threadIdx.x & 31;
    const uint32_t pitch = row_bytes + 1;
    const int nchunks = (width + 3) >> 2;
    constexpr int NW = BPP;  // words per 4-pixel chunk of raw bytes (4 * BPP bytes)
    for (int y0 = 0; y0 < height; y0 += 32) {
        const int y = y0 + lane;
        const bool live = y < height;
        const uint8_t* row = raw + (size_t)(live ? y : 0) * pitch;
        const int ft = live ? row[0] : 0;
        const uint8_t* rp = row + 1;
        uint8_t* fp = frame + (size_t)(live ? y : 0) * frame_stride;
        const uint8_t* above = y0 > 0 ? frame + (size_t)(y0 - 1) * frame_stride : nullptr;  // lane 0's "up": already BGR(A)
        const bool fp_aligned = (reinterpret_cast<uintptr_t>(fp) & 3) == 0;
        uint32_t nxt[NW], cur_raw[NW];
        uint32_t out[4] = {0, 0, 0, 0};       // this lane's pixels of the previous iteration (raw channel order, one word each)
        uint32_t left = 0, upleft = 0;
#pragma unroll
        for (int k = 0; k < NW; k++) nxt[k] = 0;
        if (live && nchunks > 0) load_words_unaligned<NW>(rp, nxt);
        for (int t = 0; t < nchunks + 31; t++) {
            // pixels above: lane r-1's outputs of the previous iteration (its chunk t-1-(r-1) = this lane's chunk)
            uint32_t up[4];
#pragma unroll
            for (int p = 0; p < 4; p++) up[p] = __shfl_up_sync(0xffffffffu, out[p], 1);
            const int c = t - lane;
            const bool act = live && c >= 0 && c < nchunks;
            if (act) {
#pragma unroll
                for (int k = 0; k < NW; k++) cur_raw[k] = nxt[k];
                if (c + 1 < nchunks) load_words_unaligned<NW>(rp + (size_t)(c + 1) * 4 * BPP, nxt);
                if (lane == 0) {
                    if (above) {
                        // read the frame row back and undo the channel swap
                        uint32_t f[NW];
                        load_words_unaligned<NW>(above + (size_t)c * 4 * BPP, f);
                        if (BPP == 4) {
#pragma unroll
                            for (int p = 0; p < 4; p++) up[p] = __byte_perm(f[p], 0, 0x3012);
                        } else {
                            const uint32_t q0 = f[0] & 0xFFFFFFu, q1 = (f[0] >> 24) | ((f[1] & 0xFFFFu) << 8),
                                           q2 = (f[1] >> 16) | ((f[2] & 0xFFu) << 16), q3 = f[2] >> 8;
                            up[0] = __byte_perm(q0, 0, 0x4012); up[1] = __byte_perm(q1, 0, 0x4012);
                            up[2] = __byte_perm(q2, 0, 0x4012); up[3] = __byte_perm(q3, 0, 0x4012);
                        }
                    } else {
                        up[0] = up[1] = up[2] = up[3] = 0;
                    }
                }
                // the four pixels' filtered bytes, one word per pixel
                uint32_t x[4];
                if (BPP == 4) {
#pragma unroll
                    for (int p = 0; p < 4; p++) x[p] = cur_raw[p];
                } else {
                    x[0] = cur_raw[0] & 0xFFFFFFu;
                    x[1] = (cur_raw[0] >> 24) | ((cur_raw[1] & 0xFFFFu) << 8);
                    x[2] = (cur_raw[1] >> 16) | ((cur_raw[2] & 0xFFu) << 16);
                    x[3] = cur_raw[2] >> 8;
                }
                uint32_t sw[4];
#pragma unroll
                for (int p = 0; p < 4; p++) {
                    const uint32_t v = png_unfilter_px(x[p], left, up[p], upleft, ft, BPP);
                    left = v;
                    upleft = up[p];
                    out[p] = v;
                    sw[p] = BPP == 4 ? __byte_perm(v, 0, 0x3012) : __byte_perm(v, 0, 0x4012);  // R,G,B(,A) -> B,G,R(,A)
                }
                const int npx = min(4, width - 4 * c);
                uint8_t* d = fp + (size_t)c * 4 * BPP;
                if (npx == 4 && fp_aligned) {
                    if (BPP == 4) {
                        if ((reinterpret_cast<uintptr_t>(d) & 15) == 0) *reinterpret_cast<uint4*>(d) = make_uint4(sw[0], sw[1], sw[2], sw[3]);
                        else {
#pragma unroll
                            for (int p = 0; p < 4; p++) reinterpret_cast<uint32_t*>(d)[p] = sw[p];
                        }
                    } else {
                        reinterpret_cast<uint32_t*>(d)[0] = sw[0] | (sw[1] << 24);
                        reinterpret_cast<uint32_t*>(d)[1] = (sw[1] >> 8) | (sw[2] << 16);
                        reinterpret_cast<uint32_t*>(d)[2] = (sw[2] >> 16) | (sw[3] << 8);
                    }
                } else {
                    for (int p = 0; p < npx; p++)
#pragma unroll
                        for (int k = 0; k < BPP; k++) d[p * BPP + k] = (uint8_t)(sw[p] >> (8 * k));
                }
            } else if (c < 0) {
                left = upleft = 0;
                out[0] = out[1] = out[2] = out[3] = 0;
            }
        }
        __syncwarp();
        __threadfence_block();
    }
}

__global__ void __launch_bounds__(kPngWarps * 32)
    png_defilter_kernel(PngDecodeItem* items, uint8_t* rawall, uint8_t* frames, int n) {
    const int warp = threadIdx.x >> 5;
    const int img = blockIdx.x * kPngWarps + warp;
    if (img >= n) return;
    PngDecodeItem& it = items[img];
    if (it.status != 0) return;
    if (frames && png_fused_ok(it)) {  // the common case: straight to the packed frame, no convert pass
        const uint8_t* raw = rawall + it.raw_off;
        uint8_t* frame = frames + it.frame_off;
        if (it.bpp == 4) defilter_to_frame<4>(raw, it.row_bytes, it.width, it.height, frame, it.frame_stride);
        else defilter_to_frame<3>(raw, it.row_bytes, it.width, it.height, frame, it.frame_stride);
        return;
    }
    for (int ps = 0; ps < it.npass; ps++) {  // Adam7: every reduced image is filtered on its own
        if (it.pass_w[ps] == 0 || it.pass_h[ps] == 0) continue;
        uint8_t* raw = rawall + it.raw_off + it.pass_off[ps];
        const uint32_t rb = it.pass_rb[ps];
        const int ph = it.pass_h[ps];
        switch (it.bpp) {
            case 1: defilter_image<1>(raw, rb, ph); break;
            case 2: defilter_image<2>(raw, rb, ph); break;
            case 3: defilter_image<3>(raw, rb, ph); break;
            case 4: defilter_image<4>(raw, rb, ph); break;
            case 6: defilter_image<6>(raw, rb, ph); break;
            default: defilter_image<8>(raw, rb, ph); break;
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------ convert

__global__ void png_convert_kernel(const PngDecodeItem* items, const uint8_t* rawall, uint8_t* frames) {
    const PngDecodeItem& it = items[blockIdx.z];
    if (it.status != 0 || png_fused_ok(it)) return;  // (fused: the defilter pass wrote the frame itself)
    const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y;
    if (ox >= it.width || oy >= it.height) return;
    int x = ox, y = oy, ps = 0;
    if (it.interlace) {  // which reduced image holds (ox, oy), and where
        int x0, y0, sx, sy;
        if (oy & 1) { ps = 6; x0 = 0; y0 = 1; sx = 0; sy = 1; }
        else if (ox & 1) { ps = 5; x0 = 1; y0 = 0; sx = 1; sy = 1; }
        else if ((oy & 3) == 2) { ps = 4; x0 = 0; y0 = 2; sx = 1; sy = 2; }
        else if ((ox & 3) == 2) { ps = 3; x0 = 2; y0 = 0; sx = 2; sy = 2; }
        else if ((oy & 7) == 4) { ps = 2; x0 = 0; y0 = 4; sx = 2; sy = 3; }
        else if ((ox & 7) == 4) { ps = 1; x0 = 4; y0 = 0; sx = 3; sy = 3; }
        else { ps = 0; x0 = 0; y0 = 0; sx = 3; sy = 3; }
        x = (ox - x0) >> sx;
        y = (oy - y0) >> sy;
    }
    const uint8_t* c = rawall + it.raw_off + it.pass_off[ps] + (size_t)y * (it.pass_rb[ps] + 1) + 1;
    uint8_t* o = frames + it.frame_off + (size_t)oy * it.frame_stride + (size_t)ox * it.out_channels;
    const int bd = it.bit_depth, sc = it.src_channels, ct = it.color_type, och = it.out_channels;
    uint32_t s[4] = {0, 0, 0, 0};
    for (int k = 0; k < sc; k++) {
        const size_t bit = ((size_t)x * sc + k) * bd;
        if (bd == 16) s[k] = ((uint32_t)c[bit >> 3] << 8) | c[(bit >> 3) + 1];
        else if (bd == 8) s[k] = c[bit >> 3];
        else s[k] = (c[bit >> 3] >> (8 - bd - (bit & 7))) & ((1u << bd) - 1);
    }
    if (ct == 3) {
        const bool ok = s[0] < (uint32_t)it.npal;
        o[0] = ok ? it.palette[s[0] * 3 + 2] : 0;
        o[1] = ok ? it.palette[s[0] * 3 + 1] : 0;
        o[2] = ok ? it.palette[s[0] * 3 + 0] : 0;
        if (och == 4) o[3] = s[0] < (uint32_t)it.ntrns ? it.trns[s[0]] : 255;
    } else if (ct == 0) {
        o[0] = bd == 16 ? (uint8_t)(s[0] >> 8) : bd == 8 ? (uint8_t)s[0] : (uint8_t)(s[0] * (255u / ((1u << bd) - 1)));
    } else if (ct == 4) {
        const uint8_t g = bd == 16 ? (uint8_t)(s[0] >> 8) : (uint8_t)s[0];
        o[0] = o[1] = o[2] = g;
        o[3] = bd == 16 ? (uint8_t)(s[1] >> 8) : (uint8_t)s[1];
    } else {
        const int sh = bd == 16 ? 8 : 0;
        o[0] = (uint8_t)(s[2] >> sh);
        o[1] = (uint8_t)(s[1] >> sh);
        o[2] = (uint8_t)(s[0] >> sh);
        if (ct == 6) o[3] = (uint8_t)(s[3] >> sh);
        else if (och == 4)
            o[3] = (s[0] == it.trns_rgb[0] && s[1] == it.trns_rgb[1] && s[2] == it.trns_rgb[2]) ? 0 : 255;
    }
}

#ifdef LP_INF_STATS
// profiling build only (make EXTRA=-DLP_INF_STATS): the counters / per-phase clocks of inflate_core.h
extern "C" void lp_png_inflate_stats(unsigned long long* out16, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out16, lpinf::g_stats, 16 * sizeof(unsigned long long));
    if (reset) {
        unsigned long long z[16] = {0};
        cudaMemcpyToSymbol(lpinf::g_stats, z, sizeof(z));
    }
}
#endif

void png_decode_item(const PngHeader& h, uint32_t frame_stride, PngDecodeItem* it) {
    memset(it, 0, sizeof(*it));
    it->z_len = (uint32_t)h.idat_total;
    it->width = h.width;
    it->height = h.height;
    it->bit_depth = h.bit_depth;
    it->color_type = h.color_type;
    it->src_channels = h.src_channels;
    it->out_channels = h.out_channels;
    it->bpp = h.bpp;
    it->row_bytes = (uint32_t)h.row_bytes;
    it->frame_stride = frame_stride;
    it->npal = h.npal;
    it->ntrns = h.ntrns;
    it->has_trns = h.has_trns;
    memcpy(it->trns_rgb, h.trns_rgb, sizeof(it->trns_rgb));
    memcpy(it->palette, h.palette, sizeof(it->palette));
    memcpy(it->trns, h.trns, sizeof(it->trns));
    it->interlace = h.interlace ? 1 : 0;
    static const int X0[7] = {0, 4, 0, 2, 0, 1, 0}, Y0[7] = {0, 0, 4, 0, 2, 0, 1};
    static const int DX[7] = {8, 8, 4, 4, 2, 2, 1}, DY[7] = {8, 8, 8, 4, 4, 2, 2};
    const size_t bits = (size_t)it->src_channels * it->bit_depth;
    it->npass = it->interlace ? 7 : 1;
    uint32_t off = 0;
    for (int ps = 0; ps < it->npass; ps++) {
        const int x0 = it->interlace ? X0[ps] : 0, y0 = it->interlace ? Y0[ps] : 0;
        const int dx = it->interlace ? DX[ps] : 1, dy = it->interlace ? DY[ps] : 1;
        const int pw = it->width > x0 ? (it->width - x0 + dx - 1) / dx : 0;
        const int ph = it->height > y0 ? (it->height - y0 + dy - 1) / dy : 0;
        it->pass_w[ps] = pw;
        it->pass_h[ps] = ph;
        it->pass_off[ps] = off;
        it->pass_rb[ps] = (uint32_t)(((size_t)pw * bits + 7) / 8);
        if (pw && ph) off += (it->pass_rb[ps] + 1) * (uint32_t)ph;
    }
    it->raw_total = off;
}

// inflate only: every stream of the batch in one launch (the long pole -- it wants as many streams in flight as fit)
int png_inflate_launch(const PngDecodeBatch& b, cudaStream_t st) {
    if (b.n <= 0) return LP_OK;
    const int ctas = ceil_div(b.n, kPngWarps);
    static bool attr_set = false;
    const size_t smem = sizeof(lpinf::WarpShared) * kPngWarps;
    if (!attr_set) {
        LP_CUDA_OK(cudaFuncSetAttribute(png_inflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        // all of the SM's L1 / shared memory as shared memory: the kernel lives in it
        LP_CUDA_OK(cudaFuncSetAttribute(png_inflate_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
        int per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, png_inflate_kernel, kPngWarps * 32, smem);
        if (getenv("LP_DEBUG")) fprintf(stderr, "[lilliput_b200] png_inflate_kernel: %zu B shared memory per CTA, %d CTAs per SM\n", smem, per_sm);
        attr_set = true;
    }
    lpinf::Match* mlists = nullptr;  // per-image match list of the window being written
    LP_CUDA_OK(cudaMallocAsync(&mlists, (size_t)b.n * lpinf::kMaxMatches * sizeof(lpinf::Match), st));
    png_inflate_kernel<<<ctas, kPngWarps * 32, smem, st>>>(b.items, b.z, b.raw, mlists, b.n);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    cudaFreeAsync(mlists, st);
    return LP_OK;
}

// defilter (+ convert) of items [first, first + count): their frame_off point into b.frames, which may be a buffer
// that is reused from one sub-range to the next (the inflated scanlines of all items stay in b.raw)
int png_unfilter_launch(const PngDecodeBatch& b, int first, int count, cudaStream_t st) {
    if (count <= 0) return LP_OK;
    const int ctas = ceil_div(count, kPngWarps);
    png_defilter_kernel<<<ctas, kPngWarps * 32, 0, st>>>(b.items + first, b.raw, b.frames, count);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    dim3 grid(ceil_div(b.max_width, 128), b.max_height, count);
    png_convert_kernel<<<grid, 128, 0, st>>>(b.items + first, b.raw, b.frames);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

int png_decode_launch(const PngDecodeBatch& b, cudaStream_t st) {
    int rc = png_inflate_launch(b, st);
    if (rc) return rc;
    return png_unfilter_launch(b, 0, b.n, st);
}

}  // namespace lp
