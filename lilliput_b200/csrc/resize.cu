// resize.cu -- crop + cv::resize for packed u8 frames on sm_90a.
//
// Replaces: opencv_mat_resize on an opencv_mat_crop view (ref opencv.cpp:196-215),
// i.e. Framebuffer.Fit / ResizeTo (ref opencv.go:294-374) and the INTER_LINEAR
// resize inside opencv_copy_to_region* (ref opencv.cpp:585, 710).
//
// Arithmetic contract (bit-exact to the OpenCV 4.11 the reference links;
// SURVEY.md Appendix E.1 / E.5):
//   both scales integer -> box sum; 2x2: (s+2)>>2, else RNE(float(s) * (1.f/area))
//   both scales >= 1    -> per source row a sequential fp32 FMA chain over the x taps,
//                          then per output row `beta*buf` followed by FMA over the y taps,
//                          RNE + clamp.  One thread owns each chain, so no reassociation.
//   otherwise / LINEAR  -> 11-bit fixed-point bilinear.
//
// The general area kernel is the HBM-bound one (BASELINE config 2 reads 3.5 MB and writes
// 0.2 MB per image).  Source row segments are staged into a shared-memory ring by a producer
// warp with 1-D bulk async copies (cp.async.bulk -> UBLKCP, the TMA engine) signalled through
// mbarriers; eight consumer warps turn each staged row into one fp32 partial per output sample
// and keep the vertical sums in registers.  No data is exchanged between CTAs.
#include <algorithm>
#include <cmath>
#include <cfloat>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"

namespace lp {

// ------------------------------------------------------------------ tap tables (host)

// OpenCV computeResizeAreaTab for one axis, grouped per destination index.
struct AreaTabHost {
    int maxt = 0;
    std::vector<int> first, count;
    std::vector<float> w;  // [dsize][maxt], zero padded
};

static AreaTabHost make_area_tab(int ssize, int dsize) {
    double scale = (double)ssize / dsize;
    std::vector<std::vector<float>> rows(dsize);
    AreaTabHost t;
    t.first.resize(dsize);
    t.count.resize(dsize);
    for (int d = 0; d < dsize; d++) {
        double f1 = d * scale, f2 = f1 + scale;
        double cell = std::min(scale, (double)ssize - f1);
        int s1 = (int)std::ceil(f1), s2 = std::min((int)std::floor(f2), ssize - 1);
        s1 = std::min(s1, s2);
        int start = -1;
        auto push = [&](int s, double wv) {
            if (start < 0) start = s;
            rows[d].push_back((float)wv);
        };
        if (s1 - f1 > 1e-3) push(s1 - 1, (s1 - f1) / cell);
        for (int s = s1; s < s2; s++) push(s, 1.0 / cell);
        if (f2 - s2 > 1e-3) push(s2, std::min(std::min(f2 - s2, 1.0), cell) / cell);
        t.first[d] = start < 0 ? 0 : start;
        t.count[d] = (int)rows[d].size();
        t.maxt = std::max(t.maxt, t.count[d]);
    }
    t.w.assign((size_t)dsize * t.maxt, 0.f);
    for (int d = 0; d < dsize; d++)
        for (size_t k = 0; k < rows[d].size(); k++) t.w[(size_t)d * t.maxt + k] = rows[d][k];
    return t;
}

struct AreaTabDev {
    int maxt = 0, padt = 0;  // padt = weights per entry as laid out on the device
    int* first = nullptr;
    int* count = nullptr;
    int* perm = nullptr;  // per 256-px tile: destination indices ordered by tap count (short chains first)
    float* w = nullptr;
    std::vector<int> h_first, h_count;
};

static std::mutex g_tab_mu;
static std::map<std::tuple<int, int, int>, AreaTabDev> g_tabs;  // (device, ssize, dsize)

static int pad_taps(int maxt) {
    const int opts[] = {2, 3, 4, 6, 8, 12, 16};
    for (int o : opts)
        if (maxt <= o) return o;
    return maxt;
}

// The cache is bounded: a service that resizes to arbitrary sizes would otherwise grow it (a few KB of HBM per
// (source, destination) size pair) for as long as it lives.  Past the bound a table is built per call, allocated
// and freed in stream order around the launch that uses it.
static size_t tab_cache_cap() {
    static const size_t cap = getenv("LP_RESIZE_TAB_CAP") ? (size_t)atol(getenv("LP_RESIZE_TAB_CAP")) : 4096;
    return cap;
}

static void free_area_tab(const AreaTabDev& d, cudaStream_t st) {
    cudaFreeAsync(d.first, st);
    cudaFreeAsync(d.count, st);
    cudaFreeAsync(d.perm, st);
    cudaFreeAsync(d.w, st);
}

// Device-resident tap table for (ssize -> dsize), cached per device.  *transient = the table is not in the cache
// (it is full): the caller hands it to free_area_tab on `st` after the launch that reads it.
static int get_area_tab(int ssize, int dsize, cudaStream_t st, AreaTabDev* out, bool* transient) {
    *transient = false;
    int dev = 0;
    LP_CUDA_OK(cudaGetDevice(&dev));
    const auto key = std::make_tuple(dev, ssize, dsize);
    {
        std::lock_guard<std::mutex> lk(g_tab_mu);
        auto it = g_tabs.find(key);
        if (it != g_tabs.end()) {
            *out = it->second;
            return LP_OK;
        }
    }
    // miss: the table is built outside the lock (pure host work)
    AreaTabHost h = make_area_tab(ssize, dsize);
    AreaTabDev d;
    d.maxt = h.maxt;
    d.padt = pad_taps(h.maxt);
    std::vector<float> w((size_t)dsize * d.padt, 0.f);
    for (int i = 0; i < dsize; i++)
        memcpy(&w[(size_t)i * d.padt], &h.w[(size_t)i * h.maxt], sizeof(float) * h.maxt);
    // Within each 256-pixel tile, order destination pixels by tap count so that whole warps share a
    // chain length and the shorter ones skip the zero-weight tail tap.
    std::vector<int> perm(dsize);
    for (int x0 = 0; x0 < dsize; x0 += 256) {
        const int x1 = std::min(x0 + 256, dsize);
        for (int i = x0; i < x1; i++) perm[i] = i;
        std::stable_sort(perm.begin() + x0, perm.begin() + x1,
                         [&](int a, int b) { return h.count[a] < h.count[b]; });
    }
    d.h_first = h.first;
    d.h_count = h.count;
    const size_t ib = sizeof(int) * (size_t)dsize, wb = sizeof(float) * w.size();
    {
        std::lock_guard<std::mutex> lk(g_tab_mu);
        auto it = g_tabs.find(key);  // another thread may have built it meanwhile
        if (it != g_tabs.end()) {
            *out = it->second;
            return LP_OK;
        }
        if (g_tabs.size() < tab_cache_cap()) {
            LP_CUDA_OK(cudaMalloc(&d.first, ib));
            LP_CUDA_OK(cudaMalloc(&d.count, ib));
            LP_CUDA_OK(cudaMalloc(&d.perm, ib));
            LP_CUDA_OK(cudaMalloc(&d.w, wb));
            LP_CUDA_OK(cudaMemcpy(d.first, h.first.data(), ib, cudaMemcpyHostToDevice));
            LP_CUDA_OK(cudaMemcpy(d.count, h.count.data(), ib, cudaMemcpyHostToDevice));
            LP_CUDA_OK(cudaMemcpy(d.perm, perm.data(), ib, cudaMemcpyHostToDevice));
            LP_CUDA_OK(cudaMemcpy(d.w, w.data(), wb, cudaMemcpyHostToDevice));
            g_tabs[key] = d;
            *out = d;
            return LP_OK;
        }
    }
    // cache full: stream-ordered, one launch long.  (The sources are pageable host memory: cudaMemcpyAsync has
    // read them by the time it returns.)
    LP_CUDA_OK(cudaMallocAsync(&d.first, ib, st));
    LP_CUDA_OK(cudaMallocAsync(&d.count, ib, st));
    LP_CUDA_OK(cudaMallocAsync(&d.perm, ib, st));
    LP_CUDA_OK(cudaMallocAsync(&d.w, wb, st));
    LP_CUDA_OK(cudaMemcpyAsync(d.first, h.first.data(), ib, cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(d.count, h.count.data(), ib, cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(d.perm, perm.data(), ib, cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(d.w, w.data(), wb, cudaMemcpyHostToDevice, st));
    *transient = true;
    *out = d;
    return LP_OK;
}

// ------------------------------------------------------------------ device helpers

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
// Blocking wait on a phase.  The suspend-time hint lets the hardware park the warp until the phase
// completes instead of re-polling: a spinning consumer steals issue slots from the warps that are
// doing the arithmetic (13 % of all issued instructions before the hint was added).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "LP_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
        "@p bra LP_DONE;\n"
        "bra LP_WAIT;\n"
        "LP_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity), "r"(0x989680u)  // up to 10 ms per attempt; wakes as soon as the phase flips
        : "memory");
}
// 1-D bulk async copy global -> shared (TMA engine, no tensor map): 16-byte aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
            "r"(smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ uint8_t sat_rne_u8(float v) {
    uint32_t r;  // round-to-nearest-even, saturating to [0,255] (NaN -> 0): one F2I
    asm("cvt.rni.u8.f32 %0, %1;" : "=r"(r) : "f"(v));
    return (uint8_t)r;
}

// ------------------------------------------------------------------ general INTER_AREA kernel

struct AreaParams {
    const uint8_t* src;
    size_t src_img_stride, src_row_stride;
    uint8_t* dst;
    size_t dst_img_stride, dst_row_stride;
    int crop_x, crop_y;
    int dw, dh;
    const int* xfirst;
    const int* xcount;
    const int* xperm;  // thread slot -> destination x (tap-count sorted within each tile)
    const float* xw;   // [dw][MAXT]
    const int* yfirst;
    const int* ycount;
    const float* yw;  // [dh][ypad]
    int ypad;
    int rows_per_band;
    int slot_bytes;
    const int* index = nullptr;  // ResizeArgs::index
};

constexpr int kAreaTile = 256;    // destination pixels per CTA
constexpr int kAreaSlots = 4;     // ring depth (power of two)
constexpr int kAreaMaxBand = 16;  // destination rows per CTA
constexpr int kAreaMaxYTaps = 16;

// u8 -> fp32, exactly.  Two routes so the work can be split across pipes: I2F.U8 runs on the XU
// pipe (16 lanes/clk/SM, the limiter when used for every byte); PRMT + FADD builds 2^23 + b and
// subtracts 2^23 on the ALU and FMA pipes.
template <bool XU_PIPE>
__device__ __forceinline__ float u8_to_f32(uint32_t word, int byte) {
    if (XU_PIPE) return (float)((word >> (8 * byte)) & 0xffu);
    return __uint_as_float(__byte_perm(word, 0x4B000000u, 0x7650u + (uint32_t)byte)) - 8388608.0f;
}

// C channels, MAXT unrolled taps (zero-weight padded), XU = taps converted on the XU pipe,
// PPT = destination pixels per consumer thread.
// One pixel's horizontal pass over NT taps: bytes o.. of the staged row -> C fp32 partials.
template <int C, int NT, int XU>
__device__ __forceinline__ void area_hpass(uint32_t slot, uint32_t o, const float* wx, float* buf) {
    constexpr int NA = (C * NT + 3) / 4;  // aligned words holding the taps
    const uint32_t addr = slot + (o & ~3u);
    const uint32_t sh = (o & 3u) * 8u;
    uint32_t w[NA + 1];
#pragma unroll
    for (int i = 0; i <= NA; i++) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w[i]) : "r"(addr + 4u * i));
    uint32_t a[NA];
#pragma unroll
    for (int i = 0; i < NA; i++) a[i] = __funnelshift_r(w[i], w[i + 1], sh);
#pragma unroll
    for (int c = 0; c < C; c++) buf[c] = 0.f;
#pragma unroll
    for (int t = 0; t < NT; t++) {
#pragma unroll
        for (int c = 0; c < C; c++) {
            const int i = t * C + c;
            const float v = (t < XU) ? u8_to_f32<true>(a[i >> 2], i & 3) : u8_to_f32<false>(a[i >> 2], i & 3);
            buf[c] = __fmaf_rn(v, wx[t], buf[c]);
        }
    }
}

template <int C, int MAXT, int XU, int PPT, bool SORT>
__global__ void __launch_bounds__(kAreaTile / PPT + 32)
    resize_area_kernel(const AreaParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int S = kAreaSlots;
    constexpr int NT = kAreaTile / PPT;  // consumer threads
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);
    uint64_t* empty = full + S;
    int* s_yf = reinterpret_cast<int*>(smem + 64);            // [kAreaMaxBand]
    int* s_yc = s_yf + kAreaMaxBand;                          // [kAreaMaxBand]
    float* s_yw = reinterpret_cast<float*>(smem + 256);       // [kAreaMaxBand][kAreaMaxYTaps]
    uint8_t* ring = smem + 256 + kAreaMaxBand * kAreaMaxYTaps * 4;

    const int tid = threadIdx.x;
    const int img = p.index ? __ldg(p.index + blockIdx.z) : blockIdx.z;
    const int dx0 = blockIdx.x * kAreaTile;
    const int dx1 = min(dx0 + kAreaTile, p.dw);
    const int dy0 = blockIdx.y * p.rows_per_band;
    const int dy1 = min(dy0 + p.rows_per_band, p.dh);

    const int x_begin = __ldg(p.xfirst + dx0);
    const int x_end = __ldg(p.xfirst + dx1 - 1) + __ldg(p.xcount + dx1 - 1);
    const int sy_begin = __ldg(p.yfirst + dy0);
    const int sy_end = __ldg(p.yfirst + dy1 - 1) + __ldg(p.ycount + dy1 - 1);  // exclusive
    const int nrows = sy_end - sy_begin;
    const uint32_t span = (uint32_t)(x_end - x_begin) * C;

    const uint8_t* seg0 = p.src + (size_t)img * p.src_img_stride +
                          (size_t)(p.crop_y + sy_begin) * p.src_row_stride +
                          (size_t)(p.crop_x + x_begin) * C;

    if (tid == 0) {
        for (int s = 0; s < S; s++) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], NT / 32);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // the band's vertical tap table
    for (int k = tid; k < (dy1 - dy0) * kAreaMaxYTaps; k += blockDim.x) {
        const int row = k / kAreaMaxYTaps, j = k % kAreaMaxYTaps;
        s_yw[k] = j < p.ypad ? __ldg(p.yw + (size_t)(dy0 + row) * p.ypad + j) : 0.f;
        if (j == 0) {
            s_yf[row] = __ldg(p.yfirst + dy0 + row) - sy_begin;
            s_yc[row] = __ldg(p.ycount + dy0 + row);
        }
    }
    __syncthreads();

    if (tid >= NT) {
        // ---------------- producer warp: one elected lane feeds the ring ----------------
        if (tid == NT) {
            for (int r = 0; r < nrows; r++) {
                const int s = r & (S - 1);
                if (r >= S) mbar_wait(&empty[s], ((r / S) - 1) & 1);
                const uint8_t* g = seg0 + (size_t)r * p.src_row_stride;
                const uint32_t delta = (uint32_t)((uintptr_t)g & 15);
                const uint32_t bytes = (delta + span + 15u) & ~15u;
                mbar_expect_tx(&full[s], bytes);
                bulk_g2s(ring + (size_t)s * p.slot_bytes, g - delta, bytes, &full[s]);
            }
        }
        return;
    }

    // ---------------- consumers: thread = PPT destination pixels (C chains each) ----------------
    const int lane = tid & 31;
    float wx[PPT][MAXT];
    uint32_t rel[PPT];
    int dxs[PPT];
    bool short_chain[PPT];  // warp-uniform: every lane's pixel has < MAXT taps
#pragma unroll
    for (int q = 0; q < PPT; q++) {
        const int slot = dx0 + tid + q * NT;
        const int dx = slot < dx1 ? (SORT ? __ldg(p.xperm + slot) : slot) : p.dw;
        dxs[q] = dx;
        const int cnt = dx < dx1 ? __ldg(p.xcount + dx) : 0;
        short_chain[q] = SORT && MAXT > 1 && __all_sync(0xffffffffu, cnt < MAXT);
        if (dx < dx1) {
            rel[q] = (uint32_t)(__ldg(p.xfirst + dx) - x_begin) * C;
#pragma unroll
            for (int t = 0; t < MAXT; t++) wx[q][t] = __ldg(p.xw + (size_t)dx * MAXT + t);
        } else {  // zero weights: reads valid ring bytes, contributes nothing, never stored
            rel[q] = 0;
#pragma unroll
            for (int t = 0; t < MAXT; t++) wx[q][t] = 0.f;
        }
    }
    const uint32_t seg_lo = (uint32_t)((uintptr_t)seg0 & 15);
    const uint32_t stride_lo = (uint32_t)(p.src_row_stride & 15);
    const uint32_t ring_base = smem_u32(ring);

    float buf[PPT][C];
    float sum[PPT][C];
#pragma unroll
    for (int q = 0; q < PPT; q++)
#pragma unroll
        for (int c = 0; c < C; c++) buf[q][c] = sum[q][c] = 0.f;

    uint8_t* dptr[PPT];  // this thread's destination pixels in row dy0
#pragma unroll
    for (int q = 0; q < PPT; q++)
        dptr[q] = p.dst + (size_t)img * p.dst_img_stride + (size_t)dy0 * p.dst_row_stride +
                  (size_t)min(dxs[q], p.dw - 1) * C;
    int next_row = 0;  // next ring entry to consume
    for (int dy = dy0; dy < dy1; dy++) {
        const int yf = s_yf[dy - dy0], yc = s_yc[dy - dy0];
        const float* yw = s_yw + (dy - dy0) * kAreaMaxYTaps;
#pragma unroll
        for (int q = 0; q < PPT; q++)
#pragma unroll
            for (int c = 0; c < C; c++) sum[q][c] = 0.f;
        for (int j = 0; j < yc; j++) {
            if (yf + j == next_row) {  // otherwise the row is the one already in buf (shared boundary row)
                const int r = next_row++;
                const int s = r & (S - 1);
                mbar_wait(&full[s], (r / S) & 1);
                const uint32_t delta = (seg_lo + (uint32_t)r * stride_lo) & 15u;
                const uint32_t slot = ring_base + (uint32_t)s * (uint32_t)p.slot_bytes;
#pragma unroll
                for (int q = 0; q < PPT; q++) {
                    const uint32_t o = delta + rel[q];
                    if (short_chain[q])
                        area_hpass<C, (MAXT > 1 ? MAXT - 1 : 1), (XU < MAXT - 1 ? XU : (MAXT > 1 ? MAXT - 1 : 1))>(slot, o, wx[q], buf[q]);
                    else
                        area_hpass<C, MAXT, XU>(slot, o, wx[q], buf[q]);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);
            }
            // first tap: fma(beta, buf, 0) == beta*buf exactly (all operands >= 0)
            const float beta = yw[j];
#pragma unroll
            for (int q = 0; q < PPT; q++)
#pragma unroll
                for (int c = 0; c < C; c++) sum[q][c] = __fmaf_rn(beta, buf[q][c], sum[q][c]);
        }
#pragma unroll
        for (int q = 0; q < PPT; q++) {
            if (dxs[q] < dx1) {
#pragma unroll
                for (int c = 0; c < C; c++) dptr[q][c] = sat_rne_u8(sum[q][c]);
            }
            dptr[q] += p.dst_row_stride;
        }
    }
    // release ring entries the band never consumed (cannot happen with contiguous taps)
    while (next_row < nrows) {
        const int s = next_row & (S - 1);
        mbar_wait(&full[s], (next_row / S) & 1);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
        next_row++;
    }
}

// Fallback for tap counts beyond the unrolled variants (scale > 16): same arithmetic,
// runtime loops, direct global loads.  One thread per destination sample.
__global__ void resize_area_generic_kernel(const AreaParams p, int C, int xpad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int img = p.index ? __ldg(p.index + blockIdx.z) : blockIdx.z;
    if (i >= p.dw * C) return;
    const int dx = i / C, c = i % C;
    const int dy = blockIdx.y;
    const int xf = p.xfirst[dx], xc = p.xcount[dx];
    const int yf = p.yfirst[dy], yc = p.ycount[dy];
    float sum = 0.f;
    for (int j = 0; j < yc; j++) {
        const uint8_t* row = p.src + (size_t)img * p.src_img_stride +
                             (size_t)(p.crop_y + yf + j) * p.src_row_stride +
                             (size_t)(p.crop_x + xf) * C + c;
        float b = 0.f;
        for (int k = 0; k < xc; k++) b = __fmaf_rn((float)row[(size_t)k * C], p.xw[(size_t)dx * xpad + k], b);
        const float beta = p.yw[(size_t)dy * p.ypad + j];
        sum = (j == 0) ? __fmul_rn(beta, b) : __fmaf_rn(beta, b, sum);
    }
    p.dst[(size_t)img * p.dst_img_stride + (size_t)dy * p.dst_row_stride + i] = sat_rne_u8(sum);
}

// ------------------------------------------------------------------ integer-scale box kernel

struct BoxParams {
    const uint8_t* src;
    size_t src_img_stride, src_row_stride;
    uint8_t* dst;
    size_t dst_img_stride, dst_row_stride;
    int crop_x, crop_y, dw, dh, kx, ky, C;
    const int* index = nullptr;  // ResizeArgs::index
};

__global__ void resize_box_kernel(const BoxParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // sample index within the dst row
    if (i >= p.dw * p.C) return;
    const int dy = blockIdx.y, img = p.index ? __ldg(p.index + blockIdx.z) : blockIdx.z;
    const int dx = i / p.C, c = i % p.C;
    const uint8_t* s = p.src + (size_t)img * p.src_img_stride +
                       (size_t)(p.crop_y + dy * p.ky) * p.src_row_stride +
                       (size_t)(p.crop_x + dx * p.kx) * p.C + c;
    int acc = 0;
    for (int y = 0; y < p.ky; y++)
        for (int x = 0; x < p.kx; x++) acc += s[(size_t)y * p.src_row_stride + (size_t)x * p.C];
    uint8_t v;
    if (p.kx == 2 && p.ky == 2)
        v = (uint8_t)((acc + 2) >> 2);
    else
        v = sat_rne_u8(__fmul_rn((float)acc, 1.f / (float)(p.kx * p.ky)));
    p.dst[(size_t)img * p.dst_img_stride + (size_t)dy * p.dst_row_stride + i] = v;
}

// ------------------------------------------------------------------ fixed-point bilinear kernel

struct LinearParams {
    const uint8_t* src;
    size_t src_img_stride, src_row_stride;
    uint8_t* dst;
    size_t dst_img_stride, dst_row_stride;
    int crop_x, crop_y, sw, sh, dw, dh, C;
    const int* xofs;
    const short* xa;  // [dw][2]
    const int* yofs;
    const short* yb;  // [dh][2]
    const int* index = nullptr;  // ResizeArgs::index
};

__global__ void resize_linear_kernel(const LinearParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.dw * p.C) return;
    const int dy = blockIdx.y, img = p.index ? __ldg(p.index + blockIdx.z) : blockIdx.z;
    const int dx = i / p.C, c = i % p.C;
    const int sx = p.xofs[dx], a0 = p.xa[2 * dx], a1 = p.xa[2 * dx + 1];
    const int sx1 = min(sx + 1, p.sw - 1);
    const int sy = p.yofs[dy], b0 = p.yb[2 * dy], b1 = p.yb[2 * dy + 1];
    const int r0 = min(max(sy, 0), p.sh - 1), r1 = min(max(sy + 1, 0), p.sh - 1);
    const uint8_t* base = p.src + (size_t)img * p.src_img_stride + (size_t)p.crop_x * p.C + c;
    const uint8_t* S0 = base + (size_t)(p.crop_y + r0) * p.src_row_stride;
    const uint8_t* S1 = base + (size_t)(p.crop_y + r1) * p.src_row_stride;
    const int t0 = S0[(size_t)sx * p.C] * a0 + S0[(size_t)sx1 * p.C] * a1;
    const int t1 = S1[(size_t)sx * p.C] * a0 + S1[(size_t)sx1 * p.C] * a1;
    const int v = (((b0 * (t0 >> 4)) >> 16) + ((b1 * (t1 >> 4)) >> 16) + 2) >> 2;
    p.dst[(size_t)img * p.dst_img_stride + (size_t)dy * p.dst_row_stride + i] =
        (uint8_t)min(max(v, 0), 255);
}

// Bilinear coefficient tables (OpenCV resize(): plain or INTER_AREA "area mode"), host side.
static void linear_tab(int ssize, int dsize, bool area_mode, bool clamp_ofs, std::vector<int>* ofs,
                       std::vector<short>* coef) {
    double inv = (double)dsize / ssize, scale = 1.0 / inv;
    ofs->resize(dsize);
    coef->resize(2 * (size_t)dsize);
    for (int d = 0; d < dsize; d++) {
        int s;
        float f;
        if (!area_mode) {
            f = (float)((d + 0.5) * scale - 0.5);
            s = (int)std::floor(f);
            f -= s;
        } else {
            s = (int)std::floor(d * scale);
            f = (float)((d + 1) - (s + 1) * inv);
            f = f <= 0 ? 0.f : f - std::floor(f);
        }
        if (clamp_ofs) {  // horizontal only; vertically the two rows are clamped instead
            if (s < 0) { f = 0; s = 0; }
            if (s >= ssize - 1) { f = 0; s = ssize - 1; }
        }
        (*ofs)[d] = s;
        (*coef)[2 * d] = (short)lrintf((1.f - f) * 2048.f);
        (*coef)[2 * d + 1] = (short)lrintf(f * 2048.f);
    }
}


// ------------------------------------------------------------------ bicubic (INTER_CUBIC)
//
// cv::resize(INTER_CUBIC) as the reference's build answers it (ref opencv.cpp:20 exports the constant,
// opencv.cpp:196-208 passes it through): the vendored IPP takes every u8 source of at least 4 x 4 and
// returns the a = -0.75 kernel evaluated exactly (matched here in fp64: rows first, then columns,
// replicated borders, round-half-even; equal to the binary to within 1 LSB on ~1e-5 of the samples, see
// tests); smaller sources fall through to OpenCV's fixed-point code (11-bit coefficients, the first
// width/16*16 samples of a row through the AVX2 fp32 form of the vertical pass), restated bit for bit.

struct CubicParams {
    const uint8_t* src;
    size_t src_img_stride, src_row_stride;
    uint8_t* dst;
    size_t dst_img_stride, dst_row_stride;
    int crop_x, crop_y, sw, sh, dw, dh, C;
    const int* xofs;
    const int* yofs;
    const double* xa;  // [dw][4]   (exact form)
    const double* yb;  // [dh][4]
    const short* xs;   // [dw][4]   (fixed-point form)
    const short* ys;   // [dh][4]
    int fixed, nvec;
};

__global__ void resize_cubic_kernel(const CubicParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.dw * p.C) return;
    const int dy = blockIdx.y, img = blockIdx.z;
    const int dx = i / p.C, c = i % p.C;
    const int sx = p.xofs[dx], sy = p.yofs[dy];
    const uint8_t* base = p.src + (size_t)img * p.src_img_stride + (size_t)p.crop_x * p.C + c;
    int col[4];
    const uint8_t* R[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        col[k] = min(max(sx - 1 + k, 0), p.sw - 1) * p.C;
        R[k] = base + (size_t)(p.crop_y + min(max(sy - 1 + k, 0), p.sh - 1)) * p.src_row_stride;
    }
    uint8_t out;
    if (!p.fixed) {
        double sum = 0.0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            double h = 0.0;
#pragma unroll
            for (int j = 0; j < 4; j++) h = fma((double)R[k][col[j]], p.xa[4 * dx + j], h);
            sum = fma(h, p.yb[4 * dy + k], sum);
        }
        const double r = rint(sum);
        out = (uint8_t)(r < 0.0 ? 0.0 : r > 255.0 ? 255.0 : r);
    } else {
        int h[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            h[k] = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) h[k] += (int)R[k][col[j]] * (int)p.xs[4 * dx + j];
        }
        const short* b = p.ys + 4 * dy;
        if (i < p.nvec) {
            const float scale = 1.f / (2048.f * 2048.f);
            float a = __fmul_rn((float)h[3], __fmul_rn((float)b[3], scale));
            a = __fmaf_rn((float)h[2], __fmul_rn((float)b[2], scale), a);
            a = __fmaf_rn((float)h[1], __fmul_rn((float)b[1], scale), a);
            a = __fmaf_rn((float)h[0], __fmul_rn((float)b[0], scale), a);
            out = sat_rne_u8(a);
        } else {
            const int v = (h[0] * b[0] + h[1] * b[1] + h[2] * b[2] + h[3] * b[3] + (1 << 21)) >> 22;
            out = (uint8_t)min(max(v, 0), 255);
        }
    }
    p.dst[(size_t)img * p.dst_img_stride + (size_t)dy * p.dst_row_stride + i] = out;
}

static void cubic_tab(int ssize, int dsize, std::vector<int>* ofs, std::vector<double>* cd, std::vector<short>* cs) {
    const double scale = 1.0 / ((double)dsize / ssize);
    ofs->resize(dsize);
    cd->resize(4 * (size_t)dsize);
    cs->resize(4 * (size_t)dsize);
    for (int d = 0; d < dsize; d++) {
        const double fd = (d + 0.5) * scale - 0.5;
        {
            const double A = -0.75, x = fd - std::floor(fd);
            double* c = cd->data() + 4 * (size_t)d;
            c[0] = ((A * (x + 1) - 5 * A) * (x + 1) + 8 * A) * (x + 1) - 4 * A;
            c[1] = ((A + 2) * x - (A + 3)) * x * x + 1;
            c[2] = ((A + 2) * (1 - x) - (A + 3)) * (1 - x) * (1 - x) + 1;
            c[3] = 1.0 - c[0] - c[1] - c[2];
        }
        float f = (float)fd;
        const int s = (int)std::floor(f);
        f -= s;
        (*ofs)[d] = s;  // floor of the fp32 position (OpenCV) == floor of the double one except on a rounding edge, where the weights carry it
        {
            // interpolateCubic in fp32 with the multiply-adds fused as the vendored build compiled them
            const float A = -0.75f, x = f, t = x + 1.f, u = 1.f - x;
            float c[4];
            c[0] = fmaf(fmaf(fmaf(A, t, -5 * A), t, 8 * A), t, -4 * A);
            c[1] = fmaf(fmaf(A + 2, x, -(A + 3)) * x, x, 1.f);
            c[2] = fmaf(fmaf(A + 2, u, -(A + 3)) * u, u, 1.f);
            c[3] = 1.f - c[0] - c[1] - c[2];
            for (int k = 0; k < 4; k++)
                (*cs)[4 * (size_t)d + k] = (short)std::min(std::max((int)lrintf(c[k] * 2048.f), -32768), 32767);
        }
    }
}

static int resize_cubic_launch(const ResizeArgs& a, cudaStream_t st) {
    const int C = a.channels;
    const bool fixed = a.crop_w < 4 || a.crop_h < 4;
    std::vector<int> xo, yo;
    std::vector<double> xd, yd;
    std::vector<short> xs, ys;
    cubic_tab(a.crop_w, a.dst_w, &xo, &xd, &xs);
    cubic_tab(a.crop_h, a.dst_h, &yo, &yd, &ys);
    if (!fixed) {  // the exact form takes its offsets from the double position
        const double sxd = 1.0 / ((double)a.dst_w / a.crop_w), syd = 1.0 / ((double)a.dst_h / a.crop_h);
        for (int d = 0; d < a.dst_w; d++) xo[d] = (int)std::floor((d + 0.5) * sxd - 0.5);
        for (int d = 0; d < a.dst_h; d++) yo[d] = (int)std::floor((d + 0.5) * syd - 0.5);
    }
    const size_t nx = (size_t)a.dst_w, ny = (size_t)a.dst_h;
    const size_t bytes = (nx + ny) * (sizeof(int) + 4 * sizeof(double) + 4 * sizeof(short));
    uint8_t* dtab = nullptr;
    LP_CUDA_OK(cudaMallocAsync(&dtab, bytes + 64, st));
    std::vector<uint8_t> host(bytes);
    size_t o = 0;
    auto put = [&](const void* ptr, size_t n) {
        memcpy(host.data() + o, ptr, n);
        const size_t at = o;
        o += n;
        return at;
    };
    const size_t o_xa = put(xd.data(), 4 * nx * sizeof(double)), o_yb = put(yd.data(), 4 * ny * sizeof(double));
    const size_t o_xo = put(xo.data(), nx * sizeof(int)), o_yo = put(yo.data(), ny * sizeof(int));
    const size_t o_xs = put(xs.data(), 4 * nx * sizeof(short)), o_ys = put(ys.data(), 4 * ny * sizeof(short));
    LP_CUDA_OK(cudaMemcpyAsync(dtab, host.data(), bytes, cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaStreamSynchronize(st));  // `host` goes out of scope below
    CubicParams p{a.src, a.src_img_stride, a.src_row_stride, a.dst, a.dst_img_stride, a.dst_row_stride,
                  a.crop_x, a.crop_y, a.crop_w, a.crop_h, a.dst_w, a.dst_h, C,
                  reinterpret_cast<const int*>(dtab + o_xo), reinterpret_cast<const int*>(dtab + o_yo),
                  reinterpret_cast<const double*>(dtab + o_xa), reinterpret_cast<const double*>(dtab + o_yb),
                  reinterpret_cast<const short*>(dtab + o_xs), reinterpret_cast<const short*>(dtab + o_ys),
                  fixed ? 1 : 0, a.dst_w * C / 16 * 16};
    dim3 grid(ceil_div(a.dst_w * C, 256), a.dst_h, a.n);
    resize_cubic_kernel<<<grid, 256, 0, st>>>(p);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    LP_CUDA_OK(cudaFreeAsync(dtab, st));
    return LP_OK;
}

// ------------------------------------------------------------------ launcher

static size_t area_smem_bytes(int slot_bytes) {
    return 256 + (size_t)kAreaMaxBand * kAreaMaxYTaps * 4 + (size_t)kAreaSlots * slot_bytes;
}

template <int C, int MAXT, int XU, int PPT, bool SORT = false>
static int launch_area(const AreaParams& p, int n, cudaStream_t st) {
    auto kern = resize_area_kernel<C, MAXT, XU, PPT, SORT>;
    const size_t smem = area_smem_bytes(p.slot_bytes);
    if (smem > 48 * 1024)
        LP_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid(ceil_div(p.dw, kAreaTile), ceil_div(p.dh, p.rows_per_band), n);
    kern<<<grid, kAreaTile / PPT + 32, smem, st>>>(p);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

// LP_RESIZE_VARIANT=<xu><ppt> (e.g. "21": 2 taps on the XU pipe, 1 pixel per thread) selects a
// tuning variant of the 3-channel 6-tap kernel for A/B timing; unset = the tuned default.
static int area_variant() {
    static int v = [] {
        const char* e = getenv("LP_RESIZE_VARIANT");
        return e ? atoi(e) : -1;
    }();
    return v;
}

template <int C>
static int dispatch_area(int padt, const AreaParams& p, int n, cudaStream_t st) {
    if (C == 3 && padt == 6) {
        switch (area_variant()) {
            case 1: return launch_area<3, 6, 0, 1>(p, n, st);
            case 21: return launch_area<3, 6, 2, 1>(p, n, st);
            case 61: return launch_area<3, 6, 6, 1>(p, n, st);
            case 2: return launch_area<3, 6, 0, 2>(p, n, st);
            case 22: return launch_area<3, 6, 2, 2>(p, n, st);
            case 32: return launch_area<3, 6, 3, 2>(p, n, st);
            case 62: return launch_area<3, 6, 6, 2>(p, n, st);
            case 24: return launch_area<3, 6, 2, 4>(p, n, st);
            case 122: return launch_area<3, 6, 2, 2, true>(p, n, st);
            case 112: return launch_area<3, 6, 1, 2, true>(p, n, st);
            case 132: return launch_area<3, 6, 3, 2, true>(p, n, st);
            case 124: return launch_area<3, 6, 2, 4, true>(p, n, st);
            case 121: return launch_area<3, 6, 2, 1, true>(p, n, st);
            default: return launch_area<3, 6, 2, 2, true>(p, n, st);
        }
    }
    switch (padt) {
        case 2: return launch_area<C, 2, 1, 1>(p, n, st);
        case 3: return launch_area<C, 3, 1, 1>(p, n, st);
        case 4: return launch_area<C, 4, 1, 1>(p, n, st);
        case 6: return launch_area<C, 6, 2, 1>(p, n, st);
        case 8: return launch_area<C, 8, 2, 1>(p, n, st);
        case 12: return launch_area<C, 12, 4, 1>(p, n, st);
        case 16: return launch_area<C, 16, 5, 1>(p, n, st);
    }
    return LP_ERR_BAD_ARGUMENT;
}

int resize_launch(const ResizeArgs& a, cudaStream_t st) {
    if (a.n <= 0) return LP_OK;
    if (a.crop_w < 1 || a.crop_h < 1 || a.dst_w < 1 || a.dst_h < 1) return LP_ERR_BAD_ARGUMENT;
    if (a.channels != 1 && a.channels != 3 && a.channels != 4) return LP_ERR_BAD_ARGUMENT;
    if (a.interpolation != 1 && a.interpolation != 2 && a.interpolation != 3) return LP_ERR_UNSUPPORTED;
    if (a.index && a.interpolation == 2) return LP_ERR_UNSUPPORTED;  // (no caller maps images through INTER_CUBIC)
    // Every kernel below takes the image from blockIdx.z, and gridDim.z is at most 65535: a larger batch (the frames of
    // a GIF task in lp_xbatch can exceed it) goes in slices of that many images.
    constexpr int kMaxImagesPerLaunch = 65535;
    if (a.n > kMaxImagesPerLaunch) {
        for (int i0 = 0; i0 < a.n; i0 += kMaxImagesPerLaunch) {
            ResizeArgs s = a;
            if (a.index) {
                s.index += i0;
            } else {
                s.src += (size_t)i0 * a.src_img_stride;
                s.dst += (size_t)i0 * a.dst_img_stride;
            }
            s.n = std::min(kMaxImagesPerLaunch, a.n - i0);
            const int rc = resize_launch(s, st);
            if (rc) return rc;
        }
        return LP_OK;
    }
    const int C = a.channels;
    if (a.crop_w == a.dst_w && a.crop_h == a.dst_h && a.index) {
        // cv::resize: same size is a copy; with an image map that is the box kernel with 1 x 1 boxes (exact)
        BoxParams p{a.src, a.src_img_stride, a.src_row_stride, a.dst, a.dst_img_stride,
                    a.dst_row_stride, a.crop_x, a.crop_y, a.dst_w, a.dst_h, 1, 1, C, a.index};
        dim3 grid(ceil_div(a.dst_w * C, 256), a.dst_h, a.n);
        resize_box_kernel<<<grid, 256, 0, st>>>(p);
        g_launches++;
        LP_CUDA_OK(cudaGetLastError());
        return LP_OK;
    }
    if (a.crop_w == a.dst_w && a.crop_h == a.dst_h) {  // cv::resize: same size is a copy
        LP_CUDA_OK(cudaMemcpy2DAsync(a.dst, a.dst_row_stride,
                                     a.src + (size_t)a.crop_y * a.src_row_stride + (size_t)a.crop_x * C,
                                     a.src_row_stride, (size_t)a.dst_w * C, a.dst_h,
                                     cudaMemcpyDeviceToDevice, st));
        for (int i = 1; i < a.n; i++)
            LP_CUDA_OK(cudaMemcpy2DAsync(
                a.dst + (size_t)i * a.dst_img_stride, a.dst_row_stride,
                a.src + (size_t)i * a.src_img_stride + (size_t)a.crop_y * a.src_row_stride + (size_t)a.crop_x * C,
                a.src_row_stride, (size_t)a.dst_w * C, a.dst_h, cudaMemcpyDeviceToDevice, st));
        return LP_OK;
    }
    if (a.interpolation == 2) return resize_cubic_launch(a, st);
    double scale_x = 1.0 / ((double)a.dst_w / a.crop_w), scale_y = 1.0 / ((double)a.dst_h / a.crop_h);
    int ix = (int)lrint(scale_x), iy = (int)lrint(scale_y);
    bool is_area_fast = std::fabs(scale_x - ix) < DBL_EPSILON && std::fabs(scale_y - iy) < DBL_EPSILON;
    int interp = a.interpolation;
    if (interp == 1 && is_area_fast && ix == 2 && iy == 2) interp = 3;

    if (interp == 3 && scale_x >= 1 && scale_y >= 1) {
        if (is_area_fast) {
            BoxParams p{a.src, a.src_img_stride, a.src_row_stride, a.dst, a.dst_img_stride,
                        a.dst_row_stride, a.crop_x, a.crop_y, a.dst_w, a.dst_h, ix, iy, C, a.index};
            dim3 grid(ceil_div(a.dst_w * C, 256), a.dst_h, a.n);
            resize_box_kernel<<<grid, 256, 0, st>>>(p);
            g_launches++;
            LP_CUDA_OK(cudaGetLastError());
            return LP_OK;
        }
        AreaTabDev tx, ty;
        bool tx_tmp = false, ty_tmp = false;
        int rc = get_area_tab(a.crop_w, a.dst_w, st, &tx, &tx_tmp);
        if (rc) return rc;
        rc = get_area_tab(a.crop_h, a.dst_h, st, &ty, &ty_tmp);
        if (rc) {
            if (tx_tmp) free_area_tab(tx, st);
            return rc;
        }
        struct Release {  // tables that are not in the cache go back in stream order, i.e. after the launch below
            const AreaTabDev &x, &y;
            bool fx, fy;
            cudaStream_t st;
            ~Release() {
                if (fx) free_area_tab(x, st);
                if (fy) free_area_tab(y, st);
            }
        } release{tx, ty, tx_tmp, ty_tmp, st};
        AreaParams p;
        p.src = a.src; p.src_img_stride = a.src_img_stride; p.src_row_stride = a.src_row_stride;
        p.dst = a.dst; p.dst_img_stride = a.dst_img_stride; p.dst_row_stride = a.dst_row_stride;
        p.crop_x = a.crop_x; p.crop_y = a.crop_y; p.dw = a.dst_w; p.dh = a.dst_h;
        p.xfirst = tx.first; p.xcount = tx.count; p.xperm = tx.perm; p.xw = tx.w;
        p.yfirst = ty.first; p.ycount = ty.count; p.yw = ty.w; p.ypad = ty.padt;
        p.index = a.index;
        if (tx.padt > 16) {
            dim3 grid(ceil_div(a.dst_w * C, 128), a.dst_h, a.n);
            resize_area_generic_kernel<<<grid, 128, 0, st>>>(p, C, tx.padt);
            g_launches++;
            LP_CUDA_OK(cudaGetLastError());
            return LP_OK;
        }
        // widest source span of any x tile (+ alignment slack + unrolled over-read slack)
        int span = 0;
        for (int x0 = 0; x0 < a.dst_w; x0 += kAreaTile) {
            int x1 = std::min(x0 + kAreaTile, a.dst_w) - 1;
            span = std::max(span, tx.h_first[x1] + tx.h_count[x1] - tx.h_first[x0]);
        }
        p.slot_bytes = round_up(span * C + 16 + tx.padt * C + 8, 128);
        // bands: keep >= ~4 CTAs per SM in flight when the batch is small
        long ctas_per_row_group = (long)ceil_div(a.dst_w, kAreaTile) * a.n;
        static const int rpb_env = getenv("LP_RESIZE_RPB") ? atoi(getenv("LP_RESIZE_RPB")) : 0;
        int rpb = rpb_env > 0 ? std::min(rpb_env, kAreaMaxBand) : 16;
        while (rpb > 1 && ctas_per_row_group * ceil_div(a.dst_h, rpb) < 4L * kNumSMs) rpb >>= 1;
        p.rows_per_band = rpb;
        if (area_smem_bytes(p.slot_bytes) > 200 * 1024 || ty.padt > kAreaMaxYTaps) {
            dim3 grid(ceil_div(a.dst_w * C, 128), a.dst_h, a.n);
            resize_area_generic_kernel<<<grid, 128, 0, st>>>(p, C, tx.padt);
            g_launches++;
            LP_CUDA_OK(cudaGetLastError());
            return LP_OK;
        }
        switch (C) {
            case 1: return dispatch_area<1>(tx.padt, p, a.n, st);
            case 3: return dispatch_area<3>(tx.padt, p, a.n, st);
            default: return dispatch_area<4>(tx.padt, p, a.n, st);
        }
    }

    // fixed-point bilinear: INTER_LINEAR, or INTER_AREA when an axis is not a downscale
    bool area_mode = interp == 3;
    std::vector<int> xo, yo;
    std::vector<short> xa, yb;
    linear_tab(a.crop_w, a.dst_w, area_mode, true, &xo, &xa);
    linear_tab(a.crop_h, a.dst_h, area_mode, false, &yo, &yb);
    int *dxo = nullptr, *dyo = nullptr;
    short *dxa = nullptr, *dyb = nullptr;
    LP_CUDA_OK(cudaMallocAsync(&dxo, sizeof(int) * xo.size(), st));
    LP_CUDA_OK(cudaMallocAsync(&dyo, sizeof(int) * yo.size(), st));
    LP_CUDA_OK(cudaMallocAsync(&dxa, sizeof(short) * xa.size(), st));
    LP_CUDA_OK(cudaMallocAsync(&dyb, sizeof(short) * yb.size(), st));
    LP_CUDA_OK(cudaMemcpyAsync(dxo, xo.data(), sizeof(int) * xo.size(), cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(dyo, yo.data(), sizeof(int) * yo.size(), cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(dxa, xa.data(), sizeof(short) * xa.size(), cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(dyb, yb.data(), sizeof(short) * yb.size(), cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaStreamSynchronize(st));  // host vectors go out of scope below
    LinearParams p{a.src, a.src_img_stride, a.src_row_stride, a.dst, a.dst_img_stride,
                   a.dst_row_stride, a.crop_x, a.crop_y, a.crop_w, a.crop_h, a.dst_w, a.dst_h, C,
                   dxo, dxa, dyo, dyb, a.index};
    dim3 grid(ceil_div(a.dst_w * C, 256), a.dst_h, a.n);
    resize_linear_kernel<<<grid, 256, 0, st>>>(p);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    LP_CUDA_OK(cudaFreeAsync(dxo, st));
    LP_CUDA_OK(cudaFreeAsync(dyo, st));
    LP_CUDA_OK(cudaFreeAsync(dxa, st));
    LP_CUDA_OK(cudaFreeAsync(dyb, st));
    return LP_OK;
}

}  // namespace lp
