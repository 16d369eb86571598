// jpeg_encode.cu -- JPEG encode on sm_90a: BGR->YCbCr + 4:2:0 downsample + ISLOW FDCT
// + quantisation, then Huffman coding with a per-image prefix sum over MCU bit lengths,
// bit packing and 0xFF byte stuffing.  Baseline, or progressive (T.81 Annex G) when asked.
//
// Replaces: opencv_encoder_write for ".jpeg"/".jpg" (ref opencv.cpp:185-194), i.e. what
// cv::ImageEncoder::write asks of libjpeg-turbo 3.1.0 defaults.  Arithmetic and bitstream
// contract: SURVEY.md Appendix E.3; output is BYTE-IDENTICAL to the reference's
// (tests/test_jpeg_encode_gpu.py).
//
// Kernels:
//   jpeg_fdct_quant_kernel   one thread per 8x8 block (4 Y + Cb + Cr per MCU): colour convert
//                            (+ 2x2 box with alternating bias for chroma), FDCT, quantise,
//                            store int16 coefficients in zig-zag order.
//   jpeg_entropy_kernel      one CTA per image: per-MCU bit counts -> block scan -> packed
//                            bitstream (atomicOr at MCU boundaries) -> stuffed bytes + header/EOI.
//   jpeg_prog_entropy_kernel one CTA per image, progressive output: the scans of jpeg_simple_progression's
//                            script in turn, each with its own optimal Huffman tables (jpeg_prog_core.h).
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "jpeg_prog_core.h"
#include "kernels.cuh"

namespace lp {

// T.81 Annex K tables
static const uint8_t kStdLumaQ[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                      14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                      18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                      49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
static const uint8_t kStdChromaQ[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                                        24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
                                        99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                        99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
#include "jpeg_std_tables.h"  // kDcLBits / kDcCBits / kDcVals / kAcLBits / kAcLVals / kAcCBits / kAcCVals
static const uint8_t kZigzagH[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                     12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                     35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                     58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Everything the kernels need that depends only on (width, height, gray, quality).
struct EncConst {
    uint16_t q[2][64];        // natural order
    uint32_t huff[4][256];    // [dcL, acL, dcC, acC][symbol] = (size << 16) | code
    uint8_t zigzag[64];       // zigzag position -> natural index
    uint8_t header[640];
    int header_len;
};

static void build_huff(const uint8_t* bits, const uint8_t* vals, uint32_t* out) {
    memset(out, 0, 256 * sizeof(uint32_t));
    unsigned code = 0;
    int k = 0;
    for (int len = 1; len <= 16; len++) {
        for (int i = 0; i < bits[len]; i++, k++) out[vals[k]] = ((uint32_t)len << 16) | code++;
        code <<= 1;
    }
}

static uint8_t* put_marker(uint8_t* p, int m, int len) {
    *p++ = 0xFF;
    *p++ = (uint8_t)m;
    *p++ = (uint8_t)(len >> 8);
    *p++ = (uint8_t)len;
    return p;
}
static uint8_t* put_dht(uint8_t* p, int tc_th, const uint8_t* bits, const uint8_t* vals) {
    int total = 0;
    for (int i = 1; i <= 16; i++) total += bits[i];
    p = put_marker(p, 0xC4, 3 + 16 + total);
    *p++ = (uint8_t)tc_th;
    memcpy(p, bits + 1, 16);
    p += 16;
    memcpy(p, vals, total);
    return p + total;
}

static void build_enc_const(int W, int H, bool gray, int quality, EncConst* c) {
    memset(c, 0, sizeof(*c));
    if (quality <= 0) quality = 1;
    if (quality > 100) quality = 100;
    const int scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
    for (int i = 0; i < 64; i++) {
        long a = ((long)kStdLumaQ[i] * scale + 50) / 100, b = ((long)kStdChromaQ[i] * scale + 50) / 100;
        c->q[0][i] = (uint16_t)(a < 1 ? 1 : a > 255 ? 255 : a);
        c->q[1][i] = (uint16_t)(b < 1 ? 1 : b > 255 ? 255 : b);
    }
    build_huff(kDcLBits, kDcVals, c->huff[0]);
    build_huff(kAcLBits, kAcLVals, c->huff[1]);
    build_huff(kDcCBits, kDcVals, c->huff[2]);
    build_huff(kAcCBits, kAcCVals, c->huff[3]);
    memcpy(c->zigzag, kZigzagH, 64);
    uint8_t* p = c->header;
    *p++ = 0xFF;
    *p++ = 0xD8;
    p = put_marker(p, 0xE0, 16);
    memcpy(p, "JFIF\0\1\1\0\0\1\0\1\0\0", 14);
    p += 14;
    for (int t = 0; t < (gray ? 1 : 2); t++) {
        p = put_marker(p, 0xDB, 67);
        *p++ = (uint8_t)t;
        for (int i = 0; i < 64; i++) *p++ = (uint8_t)c->q[t][kZigzagH[i]];
    }
    p = put_marker(p, 0xC0, 8 + 3 * (gray ? 1 : 3));
    *p++ = 8;
    *p++ = (uint8_t)(H >> 8);
    *p++ = (uint8_t)H;
    *p++ = (uint8_t)(W >> 8);
    *p++ = (uint8_t)W;
    *p++ = (uint8_t)(gray ? 1 : 3);
    if (gray) {
        *p++ = 1; *p++ = 0x11; *p++ = 0;
    } else {
        *p++ = 1; *p++ = 0x22; *p++ = 0;
        *p++ = 2; *p++ = 0x11; *p++ = 1;
        *p++ = 3; *p++ = 0x11; *p++ = 1;
    }
    p = put_dht(p, 0x00, kDcLBits, kDcVals);
    p = put_dht(p, 0x10, kAcLBits, kAcLVals);
    if (!gray) {
        p = put_dht(p, 0x01, kDcCBits, kDcVals);
        p = put_dht(p, 0x11, kAcCBits, kAcCVals);
    }
    p = put_marker(p, 0xDA, 6 + 2 * (gray ? 1 : 3));
    *p++ = (uint8_t)(gray ? 1 : 3);
    *p++ = 1;
    *p++ = 0x00;
    if (!gray) {
        *p++ = 2; *p++ = 0x11;
        *p++ = 3; *p++ = 0x11;
    }
    *p++ = 0;
    *p++ = 63;
    *p++ = 0;
    c->header_len = (int)(p - c->header);
}

static std::mutex g_enc_mu;
static std::map<std::tuple<int, int, int, int, int>, EncConst*> g_enc_consts;  // (dev,W,H,gray,q)

// Cached per (device, size, gray, quality) up to a bound; past it (a service encoding to arbitrary sizes would
// otherwise grow the cache by sizeof(EncConst) per new key for as long as it lives) the constants are built per call
// and live in stream order around the two launches that read them (*transient: the caller frees them on `st`).
static int get_enc_const(int W, int H, bool gray, int quality, cudaStream_t st, EncConst** dev, int* header_len,
                         bool* transient) {
    static const size_t cap = getenv("LP_JPEG_ENC_CONST_CAP") ? (size_t)atol(getenv("LP_JPEG_ENC_CONST_CAP")) : 4096;
    *transient = false;
    int d = 0;
    LP_CUDA_OK(cudaGetDevice(&d));
    std::lock_guard<std::mutex> lk(g_enc_mu);
    auto key = std::make_tuple(d, W, H, (int)gray, quality);
    auto it = g_enc_consts.find(key);
    static std::map<std::tuple<int, int, int, int, int>, int> lens;
    if (it != g_enc_consts.end()) {
        *dev = it->second;
        *header_len = lens[key];
        return LP_OK;
    }
    EncConst h;
    build_enc_const(W, H, gray, quality, &h);
    EncConst* p = nullptr;
    *header_len = h.header_len;
    if (g_enc_consts.size() < cap) {
        LP_CUDA_OK(cudaMalloc(&p, sizeof(EncConst)));
        LP_CUDA_OK(cudaMemcpy(p, &h, sizeof(EncConst), cudaMemcpyHostToDevice));
        g_enc_consts[key] = p;
        lens[key] = h.header_len;
    } else {
        LP_CUDA_OK(cudaMallocAsync(&p, sizeof(EncConst), st));
        // (pageable source: cudaMemcpyAsync has read it by the time it returns)
        LP_CUDA_OK(cudaMemcpyAsync(p, &h, sizeof(EncConst), cudaMemcpyHostToDevice, st));
        *transient = true;
    }
    *dev = p;
    return LP_OK;
}

// ------------------------------------------------------------------ FDCT + quantisation

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

template <bool ROWS>
__device__ __forceinline__ void fdct8(int& d0, int& d1, int& d2, int& d3, int& d4, int& d5, int& d6,
                                      int& d7) {
    const int tmp0 = d0 + d7, tmp7 = d0 - d7, tmp1 = d1 + d6, tmp6 = d1 - d6;
    const int tmp2 = d2 + d5, tmp5 = d2 - d5, tmp3 = d3 + d4, tmp4 = d3 - d4;
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    constexpr int SH = ROWS ? 11 : 15;
    constexpr int R = 1 << (SH - 1);
    int z1 = (tmp12 + tmp13) * LP_FIX_0_541196100;
    if (ROWS) {
        d0 = (tmp10 + tmp11) << 2;
        d4 = (tmp10 - tmp11) << 2;
    } else {
        d0 = (tmp10 + tmp11 + 2) >> 2;
        d4 = (tmp10 - tmp11 + 2) >> 2;
    }
    d2 = (z1 + tmp13 * LP_FIX_0_765366865 + R) >> SH;
    d6 = (z1 - tmp12 * LP_FIX_1_847759065 + R) >> SH;
    z1 = tmp4 + tmp7;
    int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
    const int z5 = (z3 + z4) * LP_FIX_1_175875602;
    const int t4 = tmp4 * LP_FIX_0_298631336, t5 = tmp5 * LP_FIX_2_053119869;
    const int t6 = tmp6 * LP_FIX_3_072711026, t7 = tmp7 * LP_FIX_1_501321110;
    z1 *= -LP_FIX_0_899976223;
    z2 *= -LP_FIX_2_562915447;
    z3 = z3 * -LP_FIX_1_961570560 + z5;
    z4 = z4 * -LP_FIX_0_390180644 + z5;
    d7 = (t4 + z1 + z3 + R) >> SH;
    d5 = (t5 + z2 + z4 + R) >> SH;
    d3 = (t6 + z2 + z3 + R) >> SH;
    d1 = (t7 + z1 + z4 + R) >> SH;
}

struct EncGeom {
    int W, H, C;           // frame size, channels (1, 3, 4)
    int mcus_x, mcus_y;    // MCU grid
    int blocks_per_mcu;    // 6 (colour) or 1 (gray)
    int ybw, ybh;          // real luma blocks
    int cdh;               // true downsampled chroma height
};

// Coefficient layout: [image][mcu][block-in-mcu][64] int16 in ZIG-ZAG order (the order the
// entropy coder walks).  Dummy luma blocks are stored as all-zero with a flag in slot 1..63 = 0
// and their DC resolved by the entropy kernel (jccoefct.c dummy-block rule).
__global__ void __launch_bounds__(128)
    jpeg_fdct_quant_kernel(const uint8_t* frames, size_t img_stride, size_t row_stride, EncGeom g,
                           const EncConst* ec, int16_t* coef, int n, const int* index) {
    __shared__ uint16_t sq[2][64];
    __shared__ float sqr[2][64];  // 1 / (8 * Q)
    if (threadIdx.x < 64) {
        sq[0][threadIdx.x] = ec->q[0][threadIdx.x];
        sq[1][threadIdx.x] = ec->q[1][threadIdx.x];
        sqr[0][threadIdx.x] = 1.0f / (float)((int)ec->q[0][threadIdx.x] << 3);
        sqr[1][threadIdx.x] = 1.0f / (float)((int)ec->q[1][threadIdx.x] << 3);
    }
    __syncthreads();
    const int nmcu = g.mcus_x * g.mcus_y;
    const int blocks_per_img = nmcu * g.blocks_per_mcu;
    const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long)blocks_per_img * n) return;
    // Role-major thread order: all luma blocks of the launch, then all Cb, then all Cr, so that a warp
    // runs ONE of the two very different gather paths below instead of both (the coefficient layout
    // [image][mcu][block] is unchanged).
    int img, mcu, k;
    if (g.blocks_per_mcu == 1) {
        img = (int)(gid / nmcu);
        mcu = (int)(gid % nmcu);
        k = 0;
    } else {
        const long ny = (long)n * nmcu * 4;
        if (gid < ny) {
            img = (int)(gid / (nmcu * 4));
            const int r = (int)(gid % (nmcu * 4));
            mcu = r >> 2;
            k = r & 3;
        } else {
            const long c = gid - ny;
            k = c >= (long)n * nmcu ? 5 : 4;
            const long cc = c % ((long)n * nmcu);
            img = (int)(cc / nmcu);
            mcu = (int)(cc % nmcu);
        }
    }
    const int mx = mcu % g.mcus_x, my = mcu / g.mcus_x;
    const uint8_t* f = frames + (size_t)(index ? __ldg(index + img) : img) * img_stride;
    int16_t* out = coef + (((size_t)img * nmcu + mcu) * g.blocks_per_mcu + k) * 64;
    int d[64];
    int qsel = 0;
    if (g.blocks_per_mcu == 1 || k < 4) {
        const int X = g.blocks_per_mcu == 1 ? mx : mx * 2 + (k & 1);
        const int Y = g.blocks_per_mcu == 1 ? my : my * 2 + (k >> 1);
        if (X >= g.ybw || Y >= g.ybh) {  // dummy block
            uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int i = 0; i < 8; i++) reinterpret_cast<uint4*>(out)[i] = z;
            return;
        }
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const int y = min(Y * 8 + r, g.H - 1);
            const uint8_t* row = f + (size_t)y * row_stride;
#pragma unroll
            for (int x8 = 0; x8 < 8; x8++) {
                const int x = min(X * 8 + x8, g.W - 1);
                int v;
                if (g.C == 1) {
                    v = row[x];
                } else {
                    const uint8_t* px = row + (size_t)x * g.C;
                    v = (19595 * px[2] + 38470 * px[1] + 7471 * px[0] + 32768) >> 16;
                }
                d[r * 8 + x8] = v - 128;
            }
        }
    } else {
        qsel = 1;
        const bool is_cr = (k == 5);
#pragma unroll
        for (int r = 0; r < 8; r++) {
            // chroma row: clamp at the DOWNSAMPLED level (the last real row is replicated), then
            // the two full-resolution rows clamp to H-1 (jcprepct.c expand_bottom_edge)
            const int yc = min(my * 8 + r, g.cdh - 1);
            const int y0 = min(2 * yc, g.H - 1), y1 = min(2 * yc + 1, g.H - 1);
            const uint8_t* r0 = f + (size_t)y0 * row_stride;
            const uint8_t* r1 = f + (size_t)y1 * row_stride;
#pragma unroll
            for (int x8 = 0; x8 < 8; x8++) {
                const int xc = mx * 8 + x8;
                const int x0 = min(2 * xc, g.W - 1), x1 = min(2 * xc + 1, g.W - 1);
                int s = 0;
                const uint8_t* p4[4] = {r0 + (size_t)x0 * g.C, r0 + (size_t)x1 * g.C, r1 + (size_t)x0 * g.C,
                                        r1 + (size_t)x1 * g.C};
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int B = p4[q][0], G = p4[q][1], R = p4[q][2];
                    s += is_cr ? ((32768 * R - 27439 * G - 5329 * B + (128 << 16) + 32767) >> 16)
                               : ((-11059 * R - 21709 * G + 32768 * B + (128 << 16) + 32767) >> 16);
                }
                d[r * 8 + x8] = ((s + 1 + (xc & 1)) >> 2) - 128;
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 8; r++)
        fdct8<true>(d[r * 8], d[r * 8 + 1], d[r * 8 + 2], d[r * 8 + 3], d[r * 8 + 4], d[r * 8 + 5], d[r * 8 + 6],
                    d[r * 8 + 7]);
#pragma unroll
    for (int x = 0; x < 8; x++)
        fdct8<false>(d[x], d[8 + x], d[16 + x], d[24 + x], d[32 + x], d[40 + x], d[48 + x], d[56 + x]);
    // quantise (jcdctmgr.c, islow: divisor = 8*Q, round half away from zero)
#pragma unroll
    for (int i = 0; i < 64; i++) {
        const int q8 = (int)sq[qsel][i] << 3;
        const int c = d[i];
        int a = c < 0 ? -c : c;
        a += q8 >> 1;
        // exact a / q8 without the ~20-instruction integer divide: float estimate (a < 2^24 is exact in
        // fp32) and a +-1 correction from the remainder
        int qt = (int)((float)a * sqr[qsel][i]);
        const int rem = a - qt * q8;
        qt += rem >= q8 ? 1 : (rem < 0 ? -1 : 0);
        d[i] = c < 0 ? -qt : qt;
    }
    // natural -> zig-zag with compile-time indices (keeps d[] in registers)
    constexpr int kZZ[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                             12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                             35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                             58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
#pragma unroll
    for (int i = 0; i < 8; i++) {
        uint4 u;
        u.x = (uint16_t)d[kZZ[i * 8 + 0]] | ((uint32_t)(uint16_t)d[kZZ[i * 8 + 1]] << 16);
        u.y = (uint16_t)d[kZZ[i * 8 + 2]] | ((uint32_t)(uint16_t)d[kZZ[i * 8 + 3]] << 16);
        u.z = (uint16_t)d[kZZ[i * 8 + 4]] | ((uint32_t)(uint16_t)d[kZZ[i * 8 + 5]] << 16);
        u.w = (uint16_t)d[kZZ[i * 8 + 6]] | ((uint32_t)(uint16_t)d[kZZ[i * 8 + 7]] << 16);
        reinterpret_cast<uint4*>(out)[i] = u;
    }
}

// ------------------------------------------------------------------ entropy coding

constexpr int kEntThreads = 256;

__device__ __forceinline__ int nbits_of(int v) { return 32 - __clz(v); }  // v >= 0

// Is block k of MCU (mx,my) a dummy luma block (outside the real block grid)?
__device__ __forceinline__ bool is_dummy(const EncGeom& g, int mx, int my, int k) {
    if (g.blocks_per_mcu == 1 || k >= 4) return false;
    return (mx * 2 + (k & 1)) >= g.ybw || (my * 2 + (k >> 1)) >= g.ybh;
}
// Quantised DC of block k of MCU m, applying jccoefct.c's dummy-block rule (a dummy block
// carries the DC of the block before it in the MCU).
__device__ __forceinline__ int dc_value(const int16_t* coef, const EncGeom& g, int m, int k) {
    const int mx = m % g.mcus_x, my = m / g.mcus_x;
    while (k > 0 && is_dummy(g, mx, my, k)) k--;
    return coef[((size_t)m * g.blocks_per_mcu + k) * 64];
}
__device__ __forceinline__ int dc_pred(const int16_t* coef, const EncGeom& g, int m, int k) {
    if (g.blocks_per_mcu == 1) return m > 0 ? coef[(size_t)(m - 1) * 64] : 0;
    if (k >= 4) return m > 0 ? coef[((size_t)(m - 1) * 6 + k) * 64] : 0;
    if (k > 0) return dc_value(coef, g, m, k - 1);
    return m > 0 ? dc_value(coef, g, m - 1, 3) : 0;
}

// Walks one block's symbols, calling emit(code, size) for every Huffman code / extra-bits group.
template <class Emit>
__device__ __forceinline__ void code_block(const int16_t* blk, bool dummy, int dc, int pred,
                                           const uint32_t* hdc, const uint32_t* hac, Emit&& emit) {
    int diff = dc - pred;
    int t = diff < 0 ? -diff : diff, t2 = diff < 0 ? diff - 1 : diff;
    int n = nbits_of(t);
    uint32_t e = hdc[n];
    emit(e & 0xffff, e >> 16);
    if (n) emit((uint32_t)t2 & ((1u << n) - 1), n);
    if (dummy) {
        e = hac[0];
        emit(e & 0xffff, e >> 16);
        return;
    }
    int r = 0;
    const uint4* b4 = reinterpret_cast<const uint4*>(blk);
#pragma unroll 1
    for (int i = 0; i < 8; i++) {
        const uint4 u = b4[i];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if (i == 0 && j == 0) continue;
            const int v = (int16_t)(j & 1 ? w[j >> 1] >> 16 : w[j >> 1] & 0xffff);
            if (v == 0) {
                r++;
                continue;
            }
            while (r > 15) {
                e = hac[0xF0];
                emit(e & 0xffff, e >> 16);
                r -= 16;
            }
            t = v < 0 ? -v : v;
            t2 = v < 0 ? v - 1 : v;
            n = nbits_of(t);
            e = hac[(r << 4) + n];
            emit(e & 0xffff, e >> 16);
            emit((uint32_t)t2 & ((1u << n) - 1), n);
            r = 0;
        }
    }
    if (r > 0) {
        e = hac[0];
        emit(e & 0xffff, e >> 16);
    }
}

template <class Emit>
__device__ __forceinline__ void code_mcu(const int16_t* coef, const EncGeom& g, int m,
                                         const uint32_t (*huff)[256], Emit&& emit) {
    const int mx = m % g.mcus_x, my = m / g.mcus_x;
    for (int k = 0; k < g.blocks_per_mcu; k++) {
        const bool chroma = k >= 4;
        const bool dummy = is_dummy(g, mx, my, k);
        const int dc = dc_value(coef, g, m, k);
        const int pred = dc_pred(coef, g, m, k);
        code_block(coef + ((size_t)m * g.blocks_per_mcu + k) * 64, dummy, dc, pred,
                   huff[chroma ? 2 : 0], huff[chroma ? 3 : 1], emit);
    }
}

// Block-wide exclusive scan of one value per thread; returns the exclusive prefix and the
// block total through *total.  kEntThreads threads.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* total, uint32_t* warp_sums) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        uint32_t s = lane < kEntThreads / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        if (lane < kEntThreads / 32) warp_sums[lane] = s;
    }
    __syncthreads();
    const uint32_t base = wid ? warp_sums[wid - 1] : 0;
    *total = warp_sums[kEntThreads / 32 - 1];
    __syncthreads();
    return base + inc - v;
}

// 0xFF byte stuffing (T.81 F.1.2.3) of nbytes packed big-endian bytes from words into body; each thread owns 16 bytes
// per round.  Returns the stuffed length, or -1 where it does not fit in room.  kEntThreads threads; s_carry (shared)
// is 0 on entry.  This is phase 4 of jpeg_entropy_kernel, which keeps its own copy so that the baseline kernel's code
// is unchanged by the progressive path.
__device__ __forceinline__ long long stuff_bytes(const uint32_t* words, uint32_t nbytes, uint8_t* body, size_t room,
                                                uint32_t* warp_sums, uint32_t& s_carry) {
    const int tid = threadIdx.x;
    bool overflow = false;
    for (uint32_t base = 0; base < nbytes; base += kEntThreads * 16) {
        const uint32_t b0 = base + tid * 16;
        uint32_t w[4] = {0, 0, 0, 0};
        uint32_t cnt = 0, have = 0;
        if (b0 < nbytes) {
            have = min(16u, nbytes - b0);
#pragma unroll
            for (int i = 0; i < 4; i++) w[i] = words[(b0 >> 2) + i];  // reads <= nwords (zeroed slack)
            for (uint32_t i = 0; i < have; i++)
                cnt += ((w[i >> 2] >> (24 - 8 * (i & 3))) & 0xff) == 0xff;
        }
        uint32_t total;
        const uint32_t ex = block_exclusive_scan(cnt, &total, warp_sums);
        size_t o = (size_t)b0 + s_carry + ex;
        if (b0 < nbytes) {
            if (o + have + cnt > room) {
                overflow = true;
            } else {
                for (uint32_t i = 0; i < have; i++) {
                    const uint8_t v = (w[i >> 2] >> (24 - 8 * (i & 3))) & 0xff;
                    body[o++] = v;
                    if (v == 0xff) body[o++] = 0;
                }
            }
        }
        __syncthreads();
        if (tid == 0) s_carry += total;
        __syncthreads();
    }
    if (__syncthreads_or(overflow)) return -1;
    return (long long)nbytes + s_carry;
}

__global__ void __launch_bounds__(kEntThreads)
    jpeg_entropy_kernel(const int16_t* coef_all, EncGeom g, const EncConst* ec, uint32_t* mcu_bits_all,
                        uint32_t* words_all, size_t words_per_img, uint8_t* out_all, size_t out_cap,
                        uint32_t* out_len, int header_len, const int* index) {
    __shared__ uint32_t huff[4][256];
    __shared__ uint32_t warp_sums[kEntThreads / 32];
    __shared__ uint32_t s_carry;
    const int img = blockIdx.x;
    const int tid = threadIdx.x;
    const int nmcu = g.mcus_x * g.mcus_y;
    const int16_t* coef = coef_all + (size_t)img * nmcu * g.blocks_per_mcu * 64;
    uint32_t* mcu_bits = mcu_bits_all + (size_t)img * nmcu;
    uint32_t* words = words_all + (size_t)img * words_per_img;
    const int slot = index ? __ldg(index + img) : img;
    uint8_t* out = out_all + (size_t)slot * out_cap;
    for (int i = tid; i < 1024; i += kEntThreads) huff[i >> 8][i & 255] = ec->huff[i >> 8][i & 255];
    if (tid == 0) s_carry = 0;
    __syncthreads();

    // phase 1+2: per-MCU bit counts, exclusive scan in chunks of kEntThreads MCUs
    for (int base = 0; base < nmcu; base += kEntThreads) {
        const int m = base + tid;
        uint32_t bits = 0;
        if (m < nmcu) code_mcu(coef, g, m, huff, [&](uint32_t, uint32_t size) { bits += size; });
        uint32_t total;
        const uint32_t ex = block_exclusive_scan(bits, &total, warp_sums);
        if (m < nmcu) mcu_bits[m] = s_carry + ex;
        __syncthreads();
        if (tid == 0) s_carry += total;
        __syncthreads();
    }
    const uint32_t total_bits = s_carry;
    const uint32_t nbytes = (total_bits + 7) >> 3;
    const uint32_t nwords = (nbytes + 3) >> 2;
    const size_t room = out_cap > (size_t)header_len + 2 ? out_cap - header_len - 2 : 0;
    if ((size_t)nbytes > room || nwords + 1 > words_per_img) {  // cannot fit even unstuffed
        if (tid == 0) out_len[slot] = 0;
        return;
    }
    // phase 3: zero the word buffer, then every MCU writes its bits (big-endian bit order)
    for (uint32_t i = tid; i <= nwords; i += kEntThreads) words[i] = 0;
    __syncthreads();
    for (int m = tid; m < nmcu; m += kEntThreads) {
        const uint32_t off = mcu_bits[m];
        uint32_t widx = off >> 5;
        uint64_t acc = 0;
        int nacc = off & 31;  // leading bits of the first word belong to the previous MCU
        bool first = true;
        code_mcu(coef, g, m, huff, [&](uint32_t code, uint32_t size) {
            acc = (acc << size) | code;
            nacc += size;
            if (nacc >= 32) {
                const uint32_t w = (uint32_t)(acc >> (nacc - 32));
                if (first) {
                    atomicOr(&words[widx], w);
                    first = false;
                } else {
                    words[widx] = w;
                }
                widx++;
                nacc -= 32;
                acc &= (1ull << nacc) - 1;
            }
        });
        if (nacc > 0) atomicOr(&words[widx], (uint32_t)(acc << (32 - nacc)));
    }
    __syncthreads();
    if (tid == 0 && (total_bits & 7)) {  // pad the last byte with 1-bits
        const uint32_t padn = 8 - (total_bits & 7);
        const uint32_t pos = total_bits & 31;  // bit position inside the word
        atomicOr(&words[total_bits >> 5], ((1u << padn) - 1) << (32 - pos - padn));
    }
    if (tid == 0) s_carry = 0;
    __syncthreads();
    // phase 4: 0xFF byte stuffing.  Each thread owns 16 bytes per round.
    uint8_t* body = out + header_len;
    bool overflow = false;
    for (uint32_t base = 0; base < nbytes; base += kEntThreads * 16) {
        const uint32_t b0 = base + tid * 16;
        uint32_t w[4] = {0, 0, 0, 0};
        uint32_t cnt = 0, have = 0;
        if (b0 < nbytes) {
            have = min(16u, nbytes - b0);
#pragma unroll
            for (int i = 0; i < 4; i++) w[i] = words[(b0 >> 2) + i];  // reads <= nwords (zeroed slack)
            for (uint32_t i = 0; i < have; i++)
                cnt += ((w[i >> 2] >> (24 - 8 * (i & 3))) & 0xff) == 0xff;
        }
        uint32_t total;
        const uint32_t ex = block_exclusive_scan(cnt, &total, warp_sums);
        size_t o = (size_t)b0 + s_carry + ex;
        if (b0 < nbytes) {
            if (o + have + cnt > room) {
                overflow = true;
            } else {
                for (uint32_t i = 0; i < have; i++) {
                    const uint8_t v = (w[i >> 2] >> (24 - 8 * (i & 3))) & 0xff;
                    body[o++] = v;
                    if (v == 0xff) body[o++] = 0;
                }
            }
        }
        __syncthreads();
        if (tid == 0) s_carry += total;
        __syncthreads();
    }
    const int any_overflow = __syncthreads_or(overflow);
    if (any_overflow) {
        if (tid == 0) out_len[slot] = 0;
        return;
    }
    for (int i = tid; i < header_len; i += kEntThreads) out[i] = ec->header[i];
    if (tid == 0) {
        const size_t end = (size_t)header_len + nbytes + s_carry;
        out[end] = 0xFF;
        out[end + 1] = 0xD9;
        out_len[slot] = (uint32_t)(end + 2);
    }
}

// ------------------------------------------------------------------ progressive entropy coding

// jpeg_prog_core.h's table builder on one warp
struct WarpLanes {
    __device__ int lane() const { return threadIdx.x & 31; }
    __device__ int lanes() const { return 32; }
    __device__ void sync() const { __syncwarp(); }
    __device__ uint64_t min(uint64_t v) const {
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const uint64_t t = __shfl_xor_sync(0xffffffffu, v, o);
            v = t < v ? t : v;
        }
        return v;
    }
};
struct SharedCounts {
    uint32_t (*hist)[257];
    __device__ void sym(int t, int s) { atomicAdd(&hist[t][s], 1u); }
    __device__ void bits(uint32_t, int) {}
};
struct AtomicOrWord {
    __device__ void operator()(uint32_t* w, uint32_t v) const { atomicOr(w, v); }
};

// One CTA per image writes the whole progressive file: the baseline frame header with SOF2, then each scan of the
// script in turn -- symbol counts over the scan's blocks, EOB runs resolved by one thread, optimal tables built by
// warp 0, per-block bit counts and a block scan for offsets, bits packed as in jpeg_entropy_kernel, 1-padding and
// stuffing straight after the scan's DHT/SOS -- then EOI.  summ / runs: per-block scratch, reused by every scan.
__global__ void __launch_bounds__(kEntThreads)
    jpeg_prog_entropy_kernel(const int16_t* coef_all, EncGeom g, const EncConst* ec, uint32_t* summ_all,
                             uint32_t* runs_all, uint32_t* words_all, size_t words_per_img, uint8_t* out_all,
                             size_t out_cap, uint32_t* out_len, const int* index) {
    __shared__ uint32_t hist[2][257];
    __shared__ uint32_t huff[2][256];
    __shared__ int tbl_work[2][257];
    __shared__ uint8_t bits[2][17], vals[2][256];
    __shared__ uint32_t warp_sums[kEntThreads / 32];
    __shared__ uint32_t s_carry;
    __shared__ int s_fail;
    const int img = blockIdx.x;
    const int tid = threadIdx.x;
    const bool gray = g.blocks_per_mcu == 1;
    const jprog::Geom pg{g.mcus_x, g.mcus_y, g.blocks_per_mcu, g.ybw, g.ybh};
    const size_t nblk = (size_t)g.mcus_x * g.mcus_y * g.blocks_per_mcu;
    const int16_t* coef = coef_all + (size_t)img * nblk * 64;
    uint32_t* summ = summ_all + (size_t)img * nblk;
    uint32_t* runs = runs_all + (size_t)img * nblk;
    uint32_t* words = words_all + (size_t)img * words_per_img;
    const int slot = index ? __ldg(index + img) : img;
    uint8_t* out = out_all + (size_t)slot * out_cap;
    const int flen = jprog::frame_len(gray);
    if (out_cap < (size_t)flen + 2) {
        if (tid == 0) out_len[slot] = 0;
        return;
    }
    const int sof = jprog::sof_type_at(gray);
    for (int i = tid; i < flen; i += kEntThreads) out[i] = i == sof ? 0xC2 : ec->header[i];
    if (tid == 0) s_fail = 0;
    size_t pos = flen;
    const int nscans = gray ? jprog::kGrayScans : jprog::kColorScans;
    for (int si = 0; si < nscans; si++) {
        const jprog::Scan s = jprog::scan_of(gray, si);
        const int nb = jprog::scan_blocks(pg, s);
        const int nt = jprog::scan_tables(gray, s);
        for (int i = tid; i < 2 * 257; i += kEntThreads) hist[i / 257][i % 257] = 0;
        __syncthreads();
        SharedCounts cnt{hist};
        for (int i = tid; i < nb; i += kEntThreads) {
            summ[i] = jprog::code_block(coef, pg, s, i, 0, cnt);
            runs[i] = 0;
        }
        __syncthreads();
        if (s.Ss && tid == 0)
            jprog::resolve_runs(summ, nb, [&](int start, int run) {
                runs[start] = (uint32_t)run;
                hist[0][(jprog::nbits((unsigned)run) - 1) << 4]++;
            });
        __syncthreads();
        if (tid < 32) {
            for (int t = 0; t < nt; t++) {
                const int n = jprog::gen_optimal_table(WarpLanes{}, hist[t], tbl_work[0], tbl_work[1], bits[t], vals[t]);
                if (tid == 0) {
                    if (n < 0) s_fail = 1;
                    jprog::make_codes(bits[t], vals[t], huff[t]);
                }
                __syncwarp();
            }
            if (tid == 0) {
                const int hl = jprog::scan_header_len(gray, s, bits);
                if (pos + hl + 2 > out_cap) {
                    s_fail = 1;
                } else {
                    jprog::put_scan_header(out + pos, gray, s, bits, vals);
                    s_carry = (uint32_t)hl;
                }
            }
        }
        __syncthreads();
        if (s_fail) {
            if (tid == 0) out_len[slot] = 0;
            return;
        }
        pos += s_carry;
        __syncthreads();
        if (tid == 0) s_carry = 0;
        __syncthreads();
        // bit offset of every block
        for (int base = 0; base < nb; base += kEntThreads) {
            const int i = base + tid;
            jprog::CountBits c{huff[0], huff[1], 0};
            if (i < nb) jprog::code_block(coef, pg, s, i, (int)runs[i], c);
            uint32_t total;
            const uint32_t ex = block_exclusive_scan(c.total, &total, warp_sums);
            if (i < nb) summ[i] = s_carry + ex;
            __syncthreads();
            if (tid == 0) s_carry += total;
            __syncthreads();
        }
        const uint32_t total_bits = s_carry;
        const uint32_t nbytes = (total_bits + 7) >> 3;
        const uint32_t nwords = (nbytes + 3) >> 2;
        const size_t room = out_cap - pos - 2;
        if ((size_t)nbytes > room || nwords + 1 > words_per_img) {  // cannot fit even unstuffed
            if (tid == 0) out_len[slot] = 0;
            return;
        }
        for (uint32_t i = tid; i <= nwords; i += kEntThreads) words[i] = 0;
        __syncthreads();
        for (int i = tid; i < nb; i += kEntThreads) {
            jprog::BitPacker<AtomicOrWord> p(words, summ[i], AtomicOrWord{});
            jprog::WriteBits<jprog::BitPacker<AtomicOrWord>> e{huff[0], huff[1], &p};
            jprog::code_block(coef, pg, s, i, (int)runs[i], e);
            p.finish();
        }
        __syncthreads();
        if (tid == 0 && (total_bits & 7)) {  // pad the last byte with 1-bits
            const uint32_t padn = 8 - (total_bits & 7);
            const uint32_t at = total_bits & 31;
            atomicOr(&words[total_bits >> 5], ((1u << padn) - 1) << (32 - at - padn));
        }
        if (tid == 0) s_carry = 0;
        __syncthreads();
        const long long stuffed = stuff_bytes(words, nbytes, out + pos, room, warp_sums, s_carry);
        if (stuffed < 0) {
            if (tid == 0) out_len[slot] = 0;
            return;
        }
        pos += (size_t)stuffed;
        __syncthreads();
    }
    if (tid == 0) {
        out[pos] = 0xFF;
        out[pos + 1] = 0xD9;
        out_len[slot] = (uint32_t)(pos + 2);
    }
}

// ------------------------------------------------------------------ launcher

static EncGeom make_geom(int W, int H, int C) {
    EncGeom g;
    g.W = W;
    g.H = H;
    g.C = C;
    const bool gray = C == 1;
    const int hs = gray ? 1 : 2;
    g.mcus_x = (W + 8 * hs - 1) / (8 * hs);
    g.mcus_y = (H + 8 * hs - 1) / (8 * hs);
    g.blocks_per_mcu = gray ? 1 : 6;
    g.ybw = (W + 7) / 8;
    g.ybh = (H + 7) / 8;
    g.cdh = (H + 1) / 2;
    return g;
}

static size_t words_per_image(size_t out_cap) { return (out_cap + 3) / 4 + 8; }

// progressive output: per-block summaries / offsets and EOB run starts, one uint32 each
static size_t prog_block_bytes(const EncGeom& g) {
    return round_up((size_t)g.mcus_x * g.mcus_y * g.blocks_per_mcu * sizeof(uint32_t), (size_t)256);
}

size_t jpeg_encode_scratch_bytes(int W, int H, int C, int n, size_t out_cap, bool progressive) {
    EncGeom g = make_geom(W, H, C);
    const size_t nmcu = (size_t)g.mcus_x * g.mcus_y;
    size_t coef = nmcu * g.blocks_per_mcu * 64 * sizeof(int16_t);
    size_t bits = round_up(nmcu * sizeof(uint32_t), (size_t)256);
    size_t words = round_up(words_per_image(out_cap) * sizeof(uint32_t), (size_t)256);
    size_t prog = progressive ? 2 * prog_block_bytes(g) : 0;
    return (size_t)n * (round_up(coef, (size_t)256) + bits + words + prog);
}

int jpeg_encode_launch(const JpegEncodeBatch& b, cudaStream_t st, cudaEvent_t ev_after_transform) {
    if (b.n <= 0) return LP_OK;
    if (b.width < 1 || b.height < 1 || b.width > 65535 || b.height > 65535) return LP_ERR_BAD_ARGUMENT;
    if (b.channels != 1 && b.channels != 3 && b.channels != 4) return LP_ERR_BAD_ARGUMENT;
    EncGeom g = make_geom(b.width, b.height, b.channels);
    EncConst* ec = nullptr;
    int header_len = 0;
    bool ec_transient = false;
    int rc = get_enc_const(b.width, b.height, b.channels == 1, b.quality, st, &ec, &header_len, &ec_transient);
    if (rc) return rc;
    struct Release {  // constants that are not in the cache go back in stream order, i.e. after the launches below
        EncConst* p;
        bool on;
        cudaStream_t st;
        ~Release() {
            if (on) cudaFreeAsync(p, st);
        }
    } release{ec, ec_transient, st};
    const size_t nmcu = (size_t)g.mcus_x * g.mcus_y;
    const size_t coef_bytes = round_up(nmcu * g.blocks_per_mcu * 64 * sizeof(int16_t), (size_t)256);
    const size_t bits_bytes = round_up(nmcu * sizeof(uint32_t), (size_t)256);
    const size_t wpi = words_per_image(b.out_cap);
    uint8_t* s = static_cast<uint8_t*>(b.scratch);
    int16_t* coef = reinterpret_cast<int16_t*>(s);
    uint32_t* mcu_bits = reinterpret_cast<uint32_t*>(s + (size_t)b.n * coef_bytes);
    uint32_t* words = reinterpret_cast<uint32_t*>(s + (size_t)b.n * (coef_bytes + bits_bytes));
    // NOTE: coef is laid out densely ([n][nmcu*bpm][64]); coef_bytes padding only sizes the region
    const long total_blocks = (long)nmcu * g.blocks_per_mcu * b.n;
    jpeg_fdct_quant_kernel<<<(unsigned)ceil_div(total_blocks, 128L), 128, 0, st>>>(
        b.frames, b.frame_img_stride, b.frame_row_stride, g, ec, coef, b.n, b.index);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    if (ev_after_transform) LP_CUDA_OK(cudaEventRecord(ev_after_transform, st));
    if (b.progressive) {
        const size_t words_bytes = round_up(wpi * sizeof(uint32_t), (size_t)256);
        uint32_t* summ = reinterpret_cast<uint32_t*>(s + (size_t)b.n * (coef_bytes + bits_bytes + words_bytes));
        uint32_t* runs = summ + (size_t)b.n * prog_block_bytes(g) / sizeof(uint32_t);
        jpeg_prog_entropy_kernel<<<b.n, kEntThreads, 0, st>>>(coef, g, ec, summ, runs, words, wpi, b.out, b.out_cap,
                                                             b.out_len, b.index);
    } else {
        jpeg_entropy_kernel<<<b.n, kEntThreads, 0, st>>>(coef, g, ec, mcu_bits, words, wpi, b.out, b.out_cap,
                                                        b.out_len, header_len, b.index);
    }
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

}  // namespace lp
