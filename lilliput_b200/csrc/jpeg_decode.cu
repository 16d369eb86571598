// jpeg_decode.cu -- baseline JPEG decode on sm_90a: Huffman scan -> dequant + 8x8 IDCT ->
// fancy chroma upsampling + YCbCr->BGR into a packed device frame.
//
// Replaces: opencv_decoder_read_data (ref opencv.cpp:166-171), i.e. what
// cv::ImageDecoder::readData asks of libjpeg-turbo 3.1.0 with its defaults (ISLOW IDCT,
// fancy upsampling, JCS_EXT_BGR).  Arithmetic contract: SURVEY.md Appendix E.2; results are
// bit-identical to the reference on baseline streams (tests/test_jpeg_decode_gpu.py).
//
// Kernels (each one grid launch over the whole batch):
//   jpeg_rst_*_kernel         lp_batch's scans with restart markers: one thread per restart interval.
//   jpeg_multiscan_kernel     progressive / one-scan-per-component files, and per image a baseline scan with restart
//                             markers: one warp per item clears its blocks, one thread walks its scans
//                             (jpeg_scan_core.h).
//   jpeg_idct_color_kernel    one CTA per tile of MCU rows x columns: dequantise + IDCT (one thread
//                             per 8x8 block, two 1-D passes in registers) into shared-memory
//                             component rows, then triangle upsampling + fixed-point colour
//                             conversion from there into the packed BGR frame.
// Scans without restart markers go to the self-synchronising decoder (jpeg_huff_parallel.cu).  Every entropy decoder
// writes quantised coefficients (int16, natural order) in scan order and clears the blocks it writes.
#include "common.cuh"
#include "kernels.cuh"
#include "jpeg_scan_core.h"

namespace lp {

__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ------------------------------------------------------------------ tile layout (host and device)

// Dynamic shared memory of one jpeg_idct_color_kernel CTA: a 4:2:0 span of up to 36 MCU columns (576 px).  Five
// CTAs of 128 threads per SM (the register limit at 96 registers) then fit in shared memory as well.  On an H100
// that beat a 46 KB budget (one span at the headline's 70-column ROI, four CTAs per SM) by 4 % in kernel time.
constexpr uint32_t kTileSmemBytes = 24 * 1024;

// libjpeg-turbo's fancy upsamplers (jdsample.c) read neighbouring samples: h2v2 and h1v2 the rows above and
// below, h2v2 and h2v1 the columns left and right.  Every other ratio replicates.
__host__ __device__ __forceinline__ bool fancy_rows(int hr, int vr) { return vr == 2 && hr <= 2; }
__host__ __device__ __forceinline__ bool fancy_cols(int hr, int vr) { return hr == 2 && vr <= 2; }

struct TileLayout {
    uint32_t off[3], stride[3];  // component c's rows in shared memory: byte offset, row pitch
    uint32_t bytes;
};

// Shared memory of a tile `cols` MCU columns wide.  Each component keeps rows of cols + 2 MCU columns (a halo
// column on each side).  Components upsampled with rows above and below keep three MCU rows (a ring), the
// others one.
__host__ __device__ inline TileLayout tile_layout(const JpegDecodeItem& it, int cols) {
    int maxh = 1, maxv = 1;
    for (int c = 0; c < it.ncomp; c++) {
        maxh = it.h[c] > maxh ? it.h[c] : maxh;
        maxv = it.v[c] > maxv ? it.v[c] : maxv;
    }
    TileLayout L{};
    for (int c = 0; c < it.ncomp; c++) {
        const int rows = (fancy_rows(maxh / it.h[c], maxv / it.v[c]) ? 3 : 1) * 8 * it.v[c];
        L.stride[c] = (uint32_t)(((cols + 2) * 8 * it.h[c] + 15) & ~15);
        L.off[c] = L.bytes;
        L.bytes += L.stride[c] * (uint32_t)rows;
    }
    return L;
}

// ------------------------------------------------------------------ ROI layout (host)

uint32_t jpeg_item_set_window(JpegDecodeItem* it, int x0, int y0, int x1, int y1, bool align16,
                              uint32_t* tiles_out) {
    int maxh = 1, maxv = 1;
    for (int c = 0; c < it->ncomp; c++) {
        maxh = it->h[c] > maxh ? it->h[c] : maxh;
        maxv = it->v[c] > maxv ? it->v[c] : maxv;
    }
    x0 = x0 < 0 ? 0 : x0;
    y0 = y0 < 0 ? 0 : y0;
    x1 = x1 > it->width ? it->width : x1;
    y1 = y1 > it->height ? it->height : y1;
    if (align16) {
        x0 &= ~15;
        x1 = (x1 + 15) & ~15;
        if (x1 > it->width) x1 = it->width;
    }
    it->win_x0 = x0;
    it->win_y0 = y0;
    it->win_w = x1 - x0;
    it->win_h = y1 - y0;
    it->win_stride = jpeg_window_row_bytes(x0, it->win_w, it->width, it->ncomp == 1 ? 1 : 3);
    // fancy upsampling reads one chroma sample beyond the window on every side = 2 luma pixels at 2x
    const int mw = 8 * maxh, mh = 8 * maxv;
    int px0 = x0 - 2 * maxh, px1 = x1 - 1 + 2 * maxh, py0 = y0 - 2 * maxv, py1 = y1 - 1 + 2 * maxv;
    px0 = px0 < 0 ? 0 : px0;
    py0 = py0 < 0 ? 0 : py0;
    px1 = px1 > it->width - 1 ? it->width - 1 : px1;
    py1 = py1 > it->height - 1 ? it->height - 1 : py1;
    it->roi_mx0 = px0 / mw;
    it->roi_my0 = py0 / mh;
    it->roi_mcx = px1 / mw - it->roi_mx0 + 1;
    it->roi_mcy = py1 / mh - it->roi_my0 + 1;
    uint32_t blocks = 0;
    for (int c = 0; c < it->ncomp; c++) blocks += (uint32_t)(it->roi_mcx * it->h[c]) * (uint32_t)(it->roi_mcy * it->v[c]);
    // Tiles: spans as wide as the shared-memory budget allows, evened out over the ROI width, and four bands of
    // MCU rows so that an image gives several CTAs.
    const int mcx = it->roi_mcx > 0 ? it->roi_mcx : 1, mcy = it->roi_mcy > 0 ? it->roi_mcy : 1;
    int span = mcx;
    while (span > 1 && tile_layout(*it, span).bytes > kTileSmemBytes) span--;
    it->tile_mcx = (mcx + (mcx + span - 1) / span - 1) / ((mcx + span - 1) / span);
    it->tiles_x = (mcx + it->tile_mcx - 1) / it->tile_mcx;
    it->tile_mcy = (mcy + 3) / 4;
    if (tiles_out) *tiles_out = (uint32_t)(it->tiles_x * ((mcy + it->tile_mcy - 1) / it->tile_mcy));
    return blocks;
}

// ------------------------------------------------------------------ restart-interval-parallel decode
// A scan with restart markers (DRI) is a sequence of independently decodable intervals: every RSTn marker is
// byte aligned, the DC predictors restart at 0 behind it (T.81 E.1.4, F.2.2.x; libjpeg-turbo jdhuff.c
// process_restart).  So: one pass finds the markers of every image (jpeg_rst_scan_kernel), then ONE THREAD PER
// INTERVAL decodes its MCUs (jpeg_rst_decode_kernel) -- with DRI = one MCU row a 1080p batch of 4096 images is
// 278 528 independent streams.  Coefficients go to the same scan-order layout the self-synchronising decoder of
// non-DRI streams writes ([roi MCU][block in MCU], DC values final), so both kinds share one IDCT launch.

// positions (byte offsets behind the marker) of the RSTn markers of one image, in order; rst_off[0] = 0
__global__ void __launch_bounds__(256) jpeg_rst_scan_kernel(JpegDecodeItem* items, const uint8_t* scan, uint32_t* rst_all) {
    __shared__ uint32_t warp_sums[8];
    __shared__ uint32_t s_carry;
    JpegDecodeItem& it = items[blockIdx.x];
    if (it.status != 0 || it.restart_interval == 0) return;
    const uint8_t* s = scan + it.scan_off;
    const uint32_t len = it.scan_len;
    uint32_t* out = rst_all + it.state_off;  // (state_off doubles as the interval table offset of DRI images)
    const uint32_t cap = it.clean_len;       // intervals expected (set by the host); out has cap + 1 slots
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    __shared__ uint32_t s_end;
    if (tid == 0) {
        s_carry = 1;
        out[0] = 0;
        s_end = len;
    }
    __syncthreads();
    // The entropy-coded segment ends at the first marker that is not RSTn (EOI): bytes after it -- an appended preview
    // or second frame with restart markers of its own -- are not part of this scan, as libjpeg-turbo reads it.  The
    // tile that holds that marker drops the RSTn behind it and is the last one.
    for (uint32_t base = 0; base < len; base += 256 * 16) {
        // 16 consecutive bytes per thread; marker = FF followed by D0..D7, end = FF followed by anything but 00, FF, RSTn
        const uint32_t b0 = base + (uint32_t)tid * 16;
        uint32_t found = 0, my_end = 0xFFFFFFFFu;
        for (uint32_t k = 0; k < 16; k++) {
            const uint32_t i = b0 + k;
            if (i + 1 < len && s[i] == 0xFF) {
                const uint32_t m = s[i + 1];
                if ((m & 0xF8) == 0xD0) found |= 1u << k;
                else if (m != 0x00 && m != 0xFF) my_end = min(my_end, i);
            }
        }
        if (__syncthreads_or(my_end != 0xFFFFFFFFu)) {
            if (my_end != 0xFFFFFFFFu) atomicMin(&s_end, my_end);
            __syncthreads();
            const uint32_t e = s_end;
            found &= e <= b0 ? 0u : (e - b0 >= 16 ? 0xFFFFu : (1u << (e - b0)) - 1u);
        }
        const uint32_t cnt = __popc(found);
        uint32_t inc = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += t;
        }
        if (lane == 31) warp_sums[wid] = inc;
        __syncthreads();
        uint32_t before = s_carry;
        for (int w = 0; w < wid; w++) before += warp_sums[w];
        uint32_t at = before + inc - cnt;
        for (uint32_t k = 0; k < 16; k++)
            if (found & (1u << k)) {
                if (at <= cap) out[at] = b0 + k + 2;
                at++;
            }
        __syncthreads();
        if (tid == 255) s_carry = before + inc;
        __syncthreads();
        if (s_end < len) break;  // (uniform: s_end last changed before the barriers above)
    }
    if (tid == 0) it.pad_ = s_carry;  // intervals found (markers + 1)
}

__global__ void __launch_bounds__(128)
    jpeg_rst_decode_kernel(JpegDecodeItem* items, const JpegHuffSet* tables, const uint8_t* scan, const uint32_t* rst_all,
                           const uint2* work /* (image, interval) */, int nwork, int16_t* coef) {
    __shared__ uint8_t zz[64];
    for (int k = threadIdx.x; k < 64; k += blockDim.x) zz[k] = c_zigzag[k];
    __syncthreads();
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwork) return;
    JpegDecodeItem& it = items[work[w].x];
    if (it.status != 0) return;
    const uint32_t k = work[w].y, nint = it.clean_len;
    if (it.pad_ != nint) {  // fewer or more markers than intervals: damaged stream (the per-image path resynchronises as libjpeg does)
        if (k == 0) it.status = -3;
        return;
    }
    const uint32_t* off = rst_all + it.state_off;
    const JpegHuffSet* hs = tables + it.table_set;
    const uint8_t* base = scan + it.scan_off;
    const uint32_t begin = off[k], end = k + 1 < nint ? off[k + 1] - 2 : it.scan_len;
    if (k > 0 && (base[begin - 1] & 7u) != ((k - 1) & 7u)) {  // RSTn must count modulo 8
        it.status = -3;
        return;
    }
    BitReader b{base + begin, base + end, 0, 0, false};
    int nb = 0;
    for (int c = 0; c < it.ncomp; c++) nb += it.h[c] * it.v[c];
    const uint32_t total_mcus = (uint32_t)it.mcus_x * it.mcus_y;
    uint32_t mcu = k * (uint32_t)it.restart_interval;
    const uint32_t mcu_end = min(total_mcus, mcu + (uint32_t)it.restart_interval);
    int pred[3] = {0, 0, 0};
    int status = 0;
    int16_t* coef_base = coef + it.coef_off;
    for (; mcu < mcu_end && !status; mcu++) {
        const int mx = (int)(mcu % (uint32_t)it.mcus_x), my = (int)(mcu / (uint32_t)it.mcus_x);
        const int rx = mx - it.roi_mx0, ry = my - it.roi_my0;
        const bool inside = (unsigned)rx < (unsigned)it.roi_mcx && (unsigned)ry < (unsigned)it.roi_mcy;
        int16_t* blk = coef_base + ((size_t)ry * it.roi_mcx + rx) * ((size_t)nb * 64);
        for (int c = 0; c < it.ncomp && !status; c++) {
            const int td = it.td[c], ta = 4 + it.ta[c];
            for (int j = 0; j < it.h[c] * it.v[c]; j++, blk += 64) {
                if (inside) {  // this thread owns the whole block: clear it here instead of memsetting the array
                    uint4* const z = reinterpret_cast<uint4*>(blk);
#pragma unroll
                    for (int i = 0; i < 8; i++) z[i] = make_uint4(0, 0, 0, 0);
                }
                int s = huff_symbol(b, hs, td);
                if (s < 0 || s > 15) { status = -3; break; }
                if (s) pred[c] += receive_extend(b, s);
                if (inside) blk[0] = (int16_t)pred[c];
                for (int q = 1; q < 64;) {
                    const int rs = huff_symbol(b, hs, ta);
                    if (rs < 0) { status = -3; break; }
                    const int r = rs >> 4, sz = rs & 15;
                    if (sz == 0) {
                        if (r != 15) break;
                        q += 16;
                        continue;
                    }
                    q += r;
                    if (q > 63) { status = -3; break; }
                    const int val = receive_extend(b, sz);
                    if (inside) blk[zz[q]] = (int16_t)val;
                    q++;
                }
                if (status) break;
            }
        }
    }
    if (status) it.status = status;
}

int jpeg_rst_launch(JpegDecodeItem* items, const JpegHuffSet* tables, const uint8_t* scan, uint32_t* rst_all, const uint2* d_work,
                    int nwork, int n_images, int16_t* coef, cudaStream_t st) {
    if (nwork <= 0) return LP_OK;
    jpeg_rst_scan_kernel<<<n_images, 256, 0, st>>>(items, scan, rst_all);
    jpeg_rst_decode_kernel<<<ceil_div(nwork, 128), 128, 0, st>>>(items, tables, scan, rst_all, d_work, nwork, coef);
    g_launches += 2;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

// ------------------------------------------------------------------ multi-scan files (serial per image)
// Per image, a baseline scan with restart markers runs here too, as one sequential scan: the walk takes the next RSTn
// whatever its number, where jpeg_rst_decode_kernel refuses markers out of sequence.
// One CTA of one warp per item; items that are not multi-scan return at once.  The warp clears the item's ROI
// blocks (and, for a window smaller than the frame, its nonzero masks), then lane 0 walks every scan
// (jpeg_scan_core.h).  Refinement scans carry no restart-free synchronisation point the way a baseline scan does
// (a refinement bit needs the block's history, the history needs the block's position), so the parallelism is
// across images: a chunk's multi-scan files decode side by side in one launch.

constexpr int kMultiscanThreads = 32;

__global__ void __launch_bounds__(kMultiscanThreads)
    jpeg_multiscan_kernel(JpegDecodeItem* items, const JpegScanDesc* scans, const JpegHuffSet* sets,
                          const uint8_t* files, int16_t* coef, uint64_t* masks) {
    __shared__ uint8_t zz[64];
    JpegDecodeItem& it = items[blockIdx.x];
    if (it.nscans == 0 || it.status != 0) return;
    for (int k = threadIdx.x; k < 64; k += blockDim.x) zz[k] = c_zigzag[k];
    const ScanOrder so = scan_order(it);
    uint4* const z = reinterpret_cast<uint4*>(coef + it.coef_off);
    const size_t nz = (size_t)roi_blocks(it, so) * 8;  // 16-byte words
    for (size_t k = threadIdx.x; k < nz; k += blockDim.x) z[k] = make_uint4(0, 0, 0, 0);
    if (masks && !roi_is_frame(it)) {
        uint64_t* const m = masks + it.dcdiff_off;
        for (uint32_t k = threadIdx.x; k < so.total; k += blockDim.x) m[k] = 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) it.status = multiscan_decode(it, scans, sets, files, coef, masks, zz);
}

// ------------------------------------------------------------------ dequant + ISLOW IDCT

#define LP_FIX_0_298631336 2446
#define LP_FIX_0_390180644 3196
#define LP_FIX_0_541196100 4433
#define LP_FIX_0_765366865 6270
#define LP_FIX_0_899976223 7373
#define LP_FIX_1_175875602 9633
#define LP_FIX_1_501321110 12299
#define LP_FIX_1_847759065 15137
#define LP_FIX_1_961570560 16069
#define LP_FIX_2_053119869 16819
#define LP_FIX_2_562915447 20995
#define LP_FIX_3_072711026 25172

__device__ __forceinline__ int sat_s16(int v) {
    int r;
    asm("cvt.sat.s16.s32 %0, %1;" : "=r"(r) : "r"(v));
    return r;
}

template <int SHIFT, bool SAT16>
__device__ __forceinline__ void idct8(int& v0, int& v1, int& v2, int& v3, int& v4, int& v5, int& v6,
                                      int& v7) {
    // even part
    int z1 = (v2 + v6) * LP_FIX_0_541196100;
    const int tmp2 = z1 - v6 * LP_FIX_1_847759065;
    const int tmp3 = z1 + v2 * LP_FIX_0_765366865;
    const int tmp0 = (v0 + v4) << 13;
    const int tmp1 = (v0 - v4) << 13;
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    // odd part
    int t0 = v7, t1 = v5, t2 = v3, t3 = v1;
    z1 = t0 + t3;
    int z2 = t1 + t2, z3 = t0 + t2, z4 = t1 + t3;
    const int z5 = (z3 + z4) * LP_FIX_1_175875602;
    t0 *= LP_FIX_0_298631336;
    t1 *= LP_FIX_2_053119869;
    t2 *= LP_FIX_3_072711026;
    t3 *= LP_FIX_1_501321110;
    z1 *= -LP_FIX_0_899976223;
    z2 *= -LP_FIX_2_562915447;
    z3 = z3 * -LP_FIX_1_961570560 + z5;
    z4 = z4 * -LP_FIX_0_390180644 + z5;
    t0 += z1 + z3;
    t1 += z2 + z4;
    t2 += z2 + z3;
    t3 += z1 + z4;
    constexpr int R = 1 << (SHIFT - 1);
    v0 = (tmp10 + t3 + R) >> SHIFT;
    v7 = (tmp10 - t3 + R) >> SHIFT;
    v1 = (tmp11 + t2 + R) >> SHIFT;
    v6 = (tmp11 - t2 + R) >> SHIFT;
    v2 = (tmp12 + t1 + R) >> SHIFT;
    v5 = (tmp12 - t1 + R) >> SHIFT;
    v3 = (tmp13 + t0 + R) >> SHIFT;
    v4 = (tmp13 - t0 + R) >> SHIFT;
    if (SAT16) {  // int16 saturation between the passes (what the SIMD IDCT's packssdw does): one cvt.sat each
        v0 = sat_s16(v0); v1 = sat_s16(v1); v2 = sat_s16(v2); v3 = sat_s16(v3);
        v4 = sat_s16(v4); v5 = sat_s16(v5); v6 = sat_s16(v6); v7 = sat_s16(v7);
    }
}

// Four samples: clamp to [-128, 127], + 128, pack.  cvt.pack.sat.s8.s32 saturates and packs two values
// per instruction; the level shift is an XOR of the sign bits.
__device__ __forceinline__ uint32_t pack_px(int a, int b, int c, int d) {
    uint32_t hi, w;
    asm("cvt.pack.sat.s8.s32.b32 %0, %1, %2, %3;" : "=r"(hi) : "r"(d), "r"(c), "r"(0));
    asm("cvt.pack.sat.s8.s32.b32 %0, %1, %2, %3;" : "=r"(w) : "r"(b), "r"(a), "r"(hi));
    return w ^ 0x80808080u;
}

// ------------------------------------------------------------------ fused dequant + IDCT + upsample + colour
//
// jpeg_idct_color_kernel runs one CTA per tile of an image: a band of ROI MCU rows x a span of ROI MCU columns
// (jpeg_item_set_window sizes them).  The CTA walks its band top to bottom.  For each MCU row it dequantises and
// IDCTs the row's blocks into shared-memory component rows, then upsamples and converts those rows straight into
// the frame window.  Only the coefficients are read from HBM and only the window is written.
//
// Components that fancy upsampling reads vertically keep a ring of three MCU rows (m - 1, m, m + 1) and are
// IDCT'd one MCU row ahead.  Fancy upsampling reads one sample beyond the window on every side.  At the ROI edge
// that sample lies inside the ROI (jpeg_item_set_window adds the margin).  At an inner tile edge the CTA IDCTs the
// neighbouring MCU row or column itself.

constexpr int kIdctColorThreads = 128;

// Per-component geometry of one tile, in shared memory.
struct TileCtx {
    int off[3], stride[3];  // shared-memory rows (TileLayout)
    int h[3], v[3];         // sampling factors
    int ring[3];            // 1: three MCU rows kept, IDCT'd one row ahead
    int row0[3];            // full-image component row of ROI row 0
    int col0[3];            // full-image component column of shared-memory column 0
    int xb0[3];             // ROI block column of shared-memory column 0
    int ca[3], nc[3];       // ROI MCU columns IDCT'd: [ca, ca + nc)
    int kfirst[3];          // first block of the component inside a scan-order MCU
    int nb;                 // blocks per MCU
};

// Offset in the tile of full-image component row cy, column 0 (add the column).
__device__ __forceinline__ int tile_row(const TileCtx& t, int c, int cy) {
    const int rows = 8 * t.v[c];
    const int ry = cy - t.row0[c];
    const int mr = ry / rows;
    const int slot = t.ring[c] ? mr % 3 : 0;
    return t.off[c] + (slot * rows + ry - mr * rows) * t.stride[c] - t.col0[c];
}

// Dequantise + IDCT ROI MCU row m_ring of the ring components and m_flat of the others (-1: none) over the
// tile's columns into shared memory, one thread per block.  The entropy decoders store blocks in scan order
// (jpeg_huff_parallel.cu): block (X % h, Y % v) of component c inside ROI MCU (X / h, Y / v).
__device__ __forceinline__ void idct_phase(const JpegDecodeItem& it, const TileCtx& t, const int16_t* coef,
                                           const uint16_t (*qt)[64], uint8_t* tile, int m_flat, int m_ring) {
    int end[3];
    int total = 0;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const int m = t.ring[c] ? m_ring : m_flat;
        if (c < it.ncomp && m >= 0) total += t.nc[c] * t.h[c] * t.v[c];
        end[c] = total;
    }
    for (int j = threadIdx.x; j < total; j += blockDim.x) {
        const int c = j < end[0] ? 0 : (j < end[1] ? 1 : 2);
        const int k = j - (c == 0 ? 0 : (c == 1 ? end[0] : end[1]));
        const int h = t.h[c], vs = t.v[c];
        const int m = t.ring[c] ? m_ring : m_flat;
        const int per = t.nc[c] * h;  // blocks per block row
        const int by = k / per, bx = k - by * per;
        const int X = t.ca[c] * h + bx;  // ROI block column
        const size_t sblk = ((size_t)m * it.roi_mcx + X / h) * t.nb + t.kfirst[c] + by * h + X % h;
        const uint4* src = reinterpret_cast<const uint4*>(coef + it.coef_off + sblk * 64);
        const uint4* q4 = reinterpret_cast<const uint4*>(qt[c]);
        int v[64];
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const uint4 u = __ldg(src + r);
            const uint4 qq = q4[r];
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
            const uint32_t qw[4] = {qq.x, qq.y, qq.z, qq.w};
#pragma unroll
            for (int q = 0; q < 4; q++) {
                // 16-bit wrapping multiply (pmullw), as libjpeg-turbo's SIMD dequantisation does
                const int lo = (int16_t)(w[q] & 0xffff), hi = (int16_t)(w[q] >> 16);
                v[r * 8 + 2 * q] = (int16_t)(lo * (int)(qw[q] & 0xffff));
                v[r * 8 + 2 * q + 1] = (int16_t)(hi * (int)(qw[q] >> 16));
            }
        }
#pragma unroll
        for (int x = 0; x < 8; x++)
            idct8<11, true>(v[x], v[8 + x], v[16 + x], v[24 + x], v[32 + x], v[40 + x], v[48 + x], v[56 + x]);
        const int stride = t.stride[c];
        uint8_t* dst = tile + t.off[c] + ((t.ring[c] ? m % 3 : 0) * 8 * vs + by * 8) * stride + (X - t.xb0[c]) * 8;
#pragma unroll
        for (int r = 0; r < 8; r++) {
            idct8<18, false>(v[r * 8], v[r * 8 + 1], v[r * 8 + 2], v[r * 8 + 3], v[r * 8 + 4], v[r * 8 + 5],
                             v[r * 8 + 6], v[r * 8 + 7]);
            uint2 o;
            o.x = pack_px(v[r * 8], v[r * 8 + 1], v[r * 8 + 2], v[r * 8 + 3]);
            o.y = pack_px(v[r * 8 + 4], v[r * 8 + 5], v[r * 8 + 6], v[r * 8 + 7]);
            *reinterpret_cast<uint2*>(dst + r * stride) = o;
        }
    }
}

// Value of component c at full-resolution pixel (x, y): libjpeg-turbo jdsample.c.  jinit_upsampler picks the
// h2v1 / h2v2 triangle filters only for components more than two samples wide; narrower ones are replicated.
__device__ __forceinline__ int upsampled(const JpegDecodeItem& it, const TileCtx& t, const uint8_t* tile, int c,
                                         int maxh, int maxv, int x, int y) {
    const int hr = maxh / t.h[c], vr = maxv / t.v[c];
    const int cw = it.dw[c], ch = it.dh[c];
    if (hr == 1 && vr == 1) return tile[tile_row(t, c, y) + x];
    if (hr == 2 && vr == 2 && cw > 2) {
        const int cy = y >> 1, i = x >> 1;
        const int fy = min(max((y & 1) ? cy + 1 : cy - 1, 0), ch - 1);
        const uint8_t* s0 = tile + tile_row(t, c, cy);
        const uint8_t* s1 = tile + tile_row(t, c, fy);
        const int cs = 3 * s0[i] + s1[i];
        if (x & 1) {
            if (i == cw - 1) return (cs * 4 + 7) >> 4;
            return (cs * 3 + 3 * s0[i + 1] + s1[i + 1] + 7) >> 4;
        }
        if (i == 0) return (cs * 4 + 8) >> 4;
        return (cs * 3 + 3 * s0[i - 1] + s1[i - 1] + 8) >> 4;
    }
    if (hr == 2 && vr == 1 && cw > 2) {
        const uint8_t* s = tile + tile_row(t, c, y);
        const int i = x >> 1;
        if (x & 1) return (i == cw - 1) ? s[i] : (3 * s[i] + s[i + 1] + 2) >> 2;
        return (i == 0) ? s[0] : (3 * s[i] + s[i - 1] + 1) >> 2;
    }
    if (hr == 1 && vr == 2) {
        const int cy = y >> 1;
        const int fy = min(max((y & 1) ? cy + 1 : cy - 1, 0), ch - 1);
        return (3 * tile[tile_row(t, c, cy) + x] + tile[tile_row(t, c, fy) + x] + ((y & 1) ? 2 : 1)) >> 2;
    }
    return tile[tile_row(t, c, y / vr) + x / hr];  // int_upsample / h2v1_upsample / h2v2_upsample (replication)
}

// 4:2:0, 16-byte aligned: 16 consecutive pixels of row y from x0 (one 16-byte Y load, four 8-byte chroma loads,
// three 16-byte stores).
__device__ __forceinline__ void color16_420(const JpegDecodeItem& it, const TileCtx& t, const uint8_t* tile,
                                            uint8_t* out, int x0, int y) {
    const uint4 yv = *reinterpret_cast<const uint4*>(tile + t.off[0] + ((y - t.row0[0]) & 15) * t.stride[0] +
                                                     (x0 - t.col0[0]));
    const uint32_t yw[4] = {yv.x, yv.y, yv.z, yv.w};
    const int cw = it.dw[1], chh = it.dh[1];
    const int cy = y >> 1;
    const int fy = min(max((y & 1) ? cy + 1 : cy - 1, 0), chh - 1);
    const int i0 = x0 >> 1;
    const int il = max(i0 - 1, 0), ir = min(i0 + 8, cw - 1);
    int cs[2][10];  // 3*near + far for chroma columns i0-1 .. i0+8, Cb and Cr
#pragma unroll
    for (int c = 0; c < 2; c++) {
        // the chroma ring: MCU row r of the ROI sits in slot r % 3
        const int rn = cy - t.row0[1 + c], rf = fy - t.row0[1 + c];
        const uint8_t* pn = tile + t.off[1 + c] + (((rn >> 3) % 3) * 8 + (rn & 7)) * t.stride[1 + c] - t.col0[1 + c];
        const uint8_t* pf = tile + t.off[1 + c] + (((rf >> 3) % 3) * 8 + (rf & 7)) * t.stride[1 + c] - t.col0[1 + c];
        const uint2 n8 = *reinterpret_cast<const uint2*>(pn + i0);
        const uint2 f8 = *reinterpret_cast<const uint2*>(pf + i0);
        cs[c][0] = 3 * pn[il] + pf[il];
        cs[c][9] = 3 * pn[ir] + pf[ir];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            cs[c][1 + k] = 3 * (int)((n8.x >> (8 * k)) & 0xff) + (int)((f8.x >> (8 * k)) & 0xff);
            cs[c][5 + k] = 3 * (int)((n8.y >> (8 * k)) & 0xff) + (int)((f8.y >> (8 * k)) & 0xff);
        }
    }
    // 3 * (3*near + far) per chroma column once, so a pixel's chroma is add + add + shift; the -128 of
    // Cb / Cr is folded into the colour-conversion constants; clamps are one VIMNMX.RELU each; bytes are
    // assembled with PRMT (3 per output word) instead of shift + or per byte.
    int c3[2][10];
#pragma unroll
    for (int c = 0; c < 2; c++)
#pragma unroll
        for (int j = 1; j < 9; j++) c3[c][j] = 3 * cs[c][j];
    uint32_t ow[12];
#pragma unroll
    for (int q = 0; q < 4; q++) {  // 4 pixels -> 3 output words
        uint32_t B[4], G[4], R[4];
#pragma unroll
        for (int p = 0; p < 4; p++) {
            const int k = 4 * q + p;
            const int j = 1 + (k >> 1);
            int cb, cr;
            if (k & 1) {
                cb = (c3[0][j] + cs[0][j + 1] + 7) >> 4;
                cr = (c3[1][j] + cs[1][j + 1] + 7) >> 4;
            } else {
                cb = (c3[0][j] + cs[0][j - 1] + 8) >> 4;
                cr = (c3[1][j] + cs[1][j - 1] + 8) >> 4;
            }
            const int Y = (int)__byte_perm(yw[q], 0, 0x4440 + p);  // byte p of the word, zero-extended
            // (c * (x - 128) + 32768) >> 16 with the -128 folded into the addend
            R[p] = (uint32_t)__vimin_s32_relu(Y + ((91881 * cr + (32768 - 91881 * 128)) >> 16), 255);
            G[p] = (uint32_t)__vimin_s32_relu(Y + ((-22554 * cb - 46802 * cr + (32768 + (22554 + 46802) * 128)) >> 16), 255);
            B[p] = (uint32_t)__vimin_s32_relu(Y + ((116130 * cb + (32768 - 116130 * 128)) >> 16), 255);
        }
        // bytes: B0 G0 R0 B1 | G1 R1 B2 G2 | R2 B3 G3 R3
        ow[3 * q + 0] = __byte_perm(__byte_perm(B[0], G[0], 0x0040), __byte_perm(R[0], B[1], 0x0040), 0x5410);
        ow[3 * q + 1] = __byte_perm(__byte_perm(G[1], R[1], 0x0040), __byte_perm(B[2], G[2], 0x0040), 0x5410);
        ow[3 * q + 2] = __byte_perm(__byte_perm(R[2], B[3], 0x0040), __byte_perm(G[3], R[3], 0x0040), 0x5410);
    }
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)(x0 - it.win_x0) * 3);
    dst[0] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    dst[1] = make_uint4(ow[4], ow[5], ow[6], ow[7]);
    dst[2] = make_uint4(ow[8], ow[9], ow[10], ow[11]);
}

// Grayscale: the window pixels [xa, xb) x [ya, yb) of an MCU row are a copy of the tile.  One thread moves one
// 16-pixel segment of a row; segments are cut at multiples of 16 from the window's left edge, whatever MCU column the
// span starts at.  When the window's rows are 16-byte aligned in the frame (`aligned`; the windows of batch.cu are) a
// whole segment is one 16-byte store, fed by two 8-byte shared-memory loads: the halo column of a one-block MCU is 8
// pixels, so tile columns are 8-byte aligned only.  Ragged segments and unaligned frames go byte by byte.
__device__ __forceinline__ void gray_phase(const JpegDecodeItem& it, const TileCtx& t, const uint8_t* tile, uint8_t* frames,
                                        int xa, int xb, int ya, int yb, bool aligned) {
    const int base = aligned ? it.win_x0 + ((xa - it.win_x0) & ~15) : xa;
    const int segs = (xb - base + 15) >> 4;
    const int n = (yb - ya) * segs;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const int r = j / segs;
        const int y = ya + r, x0 = base + (j - r * segs) * 16;
        uint8_t* out = frames + it.frame_off + (size_t)(y - it.win_y0) * it.win_stride - it.win_x0;
        const uint8_t* in = tile + tile_row(t, 0, y);
        if (aligned && x0 >= xa && x0 + 16 <= xb) {
            const uint2 lo = *reinterpret_cast<const uint2*>(in + x0), hi = *reinterpret_cast<const uint2*>(in + x0 + 8);
            *reinterpret_cast<uint4*>(out + x0) = make_uint4(lo.x, lo.y, hi.x, hi.y);
        } else {
            for (int x = max(x0, xa); x < min(x0 + 16, xb); x++) out[x] = in[x];
        }
    }
}

// Upsample + colour the window pixels of ROI MCU row m inside the span [c0, c1), one thread per 16 consecutive
// pixels of a row.  4:2:0 frames whose rows are 16-byte aligned take color16_420; everything else (other
// samplings, odd widths) goes pixel by pixel through upsampled(); grayscale is a copy (gray_phase).
__device__ __forceinline__ void color_phase(const JpegDecodeItem& it, const TileCtx& t, const uint8_t* tile,
                                            uint8_t* frames, int m, int c0, int c1, int maxh, int maxv, bool fast) {
    const int mh = 8 * maxv, mw = 8 * maxh;
    const int ya = max(it.win_y0, (it.roi_my0 + m) * mh), yb = min(it.win_y0 + it.win_h, (it.roi_my0 + m + 1) * mh);
    const int xa = max(it.win_x0, (it.roi_mx0 + c0) * mw), xb = min(it.win_x0 + it.win_w, (it.roi_mx0 + c1) * mw);
    if (ya >= yb || xa >= xb) return;
    if (it.ncomp == 1) {
        gray_phase(it, t, tile, frames, xa, xb, ya, yb,
                   (it.win_x0 & 15) == 0 && (it.win_stride & 15) == 0 && (it.frame_off & 15) == 0);
        return;
    }
    const int segs = (xb - xa + 15) >> 4;
    const int n = (yb - ya) * segs;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const int r = j / segs;
        const int y = ya + r, x0 = xa + (j - r * segs) * 16;
        uint8_t* out = frames + it.frame_off + (size_t)(y - it.win_y0) * it.win_stride;
        if (fast) {
            color16_420(it, t, tile, out, x0, y);
        } else {
            for (int x = x0; x < min(x0 + 16, xb); x++) {
                const int Y = upsampled(it, t, tile, 0, maxh, maxv, x, y);
                const int cb = upsampled(it, t, tile, 1, maxh, maxv, x, y) - 128;
                const int cr = upsampled(it, t, tile, 2, maxh, maxv, x, y) - 128;
                const int r = Y + ((91881 * cr + 32768) >> 16);
                const int g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
                const int b = Y + ((116130 * cb + 32768) >> 16);
                uint8_t* o = out + (size_t)(x - it.win_x0) * 3;
                o[0] = (uint8_t)min(max(b, 0), 255);
                o[1] = (uint8_t)min(max(g, 0), 255);
                o[2] = (uint8_t)min(max(r, 0), 255);
            }
        }
    }
}

__global__ void __launch_bounds__(kIdctColorThreads, 5)
    jpeg_idct_color_kernel(const JpegDecodeItem* items, const int16_t* coef, uint8_t* frames) {
    const JpegDecodeItem& it = items[blockIdx.y];
    if (it.status != 0) return;
    const int band = (int)blockIdx.x / it.tiles_x, span = (int)blockIdx.x - band * it.tiles_x;
    const int m0 = band * it.tile_mcy, m1 = min(m0 + it.tile_mcy, it.roi_mcy);
    const int c0 = span * it.tile_mcx, c1 = min(c0 + it.tile_mcx, it.roi_mcx);
    if (m0 >= m1 || c0 >= c1) return;
    __shared__ __align__(16) uint16_t s_qt[3][64];
    __shared__ TileCtx s_t;
    extern __shared__ __align__(16) uint8_t s_tile[];
    for (int i = threadIdx.x; i < 3 * 64; i += blockDim.x) s_qt[i >> 6][i & 63] = it.qt[i >> 6][i & 63];
    int maxh = 1, maxv = 1;
    for (int c = 0; c < it.ncomp; c++) {
        maxh = max(maxh, it.h[c]);
        maxv = max(maxv, it.v[c]);
    }
    if (threadIdx.x == 0) {
        const TileLayout L = tile_layout(it, c1 - c0);
        int nb = 0;
        for (int c = 0; c < it.ncomp; c++) {
            const int hr = maxh / it.h[c], vr = maxv / it.v[c];
            const bool halo = fancy_cols(hr, vr);
            s_t.off[c] = (int)L.off[c];
            s_t.stride[c] = (int)L.stride[c];
            s_t.h[c] = it.h[c];
            s_t.v[c] = it.v[c];
            s_t.ring[c] = fancy_rows(hr, vr);
            s_t.row0[c] = it.roi_my0 * 8 * it.v[c];
            s_t.xb0[c] = (c0 - 1) * it.h[c];
            s_t.col0[c] = (it.roi_mx0 * it.h[c] + s_t.xb0[c]) * 8;
            s_t.ca[c] = halo && c0 > 0 ? c0 - 1 : c0;
            s_t.nc[c] = (halo && c1 < it.roi_mcx ? c1 + 1 : c1) - s_t.ca[c];
            s_t.kfirst[c] = nb;
            nb += it.h[c] * it.v[c];
        }
        s_t.nb = nb;
    }
    __syncthreads();
    const TileCtx& t = s_t;
    const bool fast = it.ncomp == 3 && it.h[0] == 2 && it.v[0] == 2 && it.h[1] == 1 && it.v[1] == 1 &&
                      it.h[2] == 1 && it.v[2] == 1 && (it.width & 15) == 0 && (it.win_x0 & 15) == 0 &&
                      (it.win_w & 15) == 0 && (it.win_stride & 15) == 0 && (it.frame_off & 15) == 0;
    // the ring's rows above the band and the band's first row
    if (m0 > 0) idct_phase(it, t, coef, s_qt, s_tile, -1, m0 - 1);
    idct_phase(it, t, coef, s_qt, s_tile, -1, m0);
    for (int m = m0; m < m1; m++) {
        idct_phase(it, t, coef, s_qt, s_tile, m, m + 1 < it.roi_mcy ? m + 1 : -1);
        __syncthreads();
        color_phase(it, t, s_tile, frames, m, c0, c1, maxh, maxv, fast);
        __syncthreads();
    }
}

// ------------------------------------------------------------------ launcher

int jpeg_decode_launch(const JpegDecodeBatch& b, cudaStream_t st, cudaEvent_t ev_after_huff) {
    if (b.n <= 0) return LP_OK;
    // Every decoder clears the blocks of the region of interest itself as it opens them, so the coefficient array is
    // not cleared: at 4096 1080p images a memset alone would write 15 GB per batch.  Blocks of an image that fails
    // are not read.
    if (b.n_multiscan < b.n) {  // the self-synchronising and restart-interval decoders skip multi-scan items
        JpegHuffParallelArgs a{b.items, b.tables, b.scan, b.clean, b.states, b.nslots, b.coef, b.dcdiff, b.n};
        int rc = jpeg_huff_parallel_launch(a, st);  // skips the images that carry restart markers
        if (rc) return rc;
        rc = jpeg_rst_launch(b.items, b.tables, b.scan, b.nslots, b.rst_work, b.n_rst_work, b.n, b.coef, st);
        if (rc) return rc;
    }
    if (b.n_multiscan > 0) {
        jpeg_multiscan_kernel<<<b.n, kMultiscanThreads, 0, st>>>(b.items, b.scans, b.tables, b.scan, b.coef, b.masks);
        g_launches++;
        LP_CUDA_OK(cudaGetLastError());
    }
    if (ev_after_huff) LP_CUDA_OK(cudaEventRecord(ev_after_huff, st));
    if (b.max_tiles_per_image > 0) {
        const dim3 grid((unsigned)b.max_tiles_per_image, b.n);
        jpeg_idct_color_kernel<<<grid, kIdctColorThreads, kTileSmemBytes, st>>>(b.items, b.coef, b.frames);
        g_launches++;
        LP_CUDA_OK(cudaGetLastError());
    }
    return LP_OK;
}

}  // namespace lp
