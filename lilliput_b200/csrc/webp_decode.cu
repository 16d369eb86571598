// webp_decode.cu -- lilliput's WebP decoder surface (include/lp_webp.h = ref webp.hpp:35-51,74-75)
// on sm_90a: host RIFF walk, device VP8 / VP8L / ALPH decode, device upsample + colour conversion.
//
// Replaces: webp_decoder_* (ref webp.cpp:61-370), i.e. libwebpmux's chunk walk
// (WebPMuxCreate / GetFeatures / GetFrame / GetCanvasSize / GetAnimationParams / GetChunk "ICCP")
// and libwebp's WebPDecodeBGRInto / WebPDecodeBGRAInto.  The VP8 decoding logic lives in
// vp8_core.h (shared with the CPU test harness); this file holds the kernels and the ABI.
//
// VP8 on a GPU: one frame's mode bits and coefficient tokens are two serial arithmetic-coded
// streams whose contexts chain through the picture, so the unit of parallelism is the frame: one
// warp per frame.  Lane 0 walks the bitstream and reconstructs macroblocks into the frame's YUV
// planes in HBM; the loop filter then runs warp-wide (32 lanes = the 16 luma + 8 + 8 chroma sample
// positions of one macroblock edge); the compositor (webp_compose_kernel), fully parallel, does libwebp's
// "fancy" chroma upsampling and the fixed-point YUV->BGR(A) conversion per output pixel.  The per-image
// decoder runs each frame through the same launches as the batch (webp_decode_batch with one file).
#include <algorithm>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"
#include "lp_webp.h"
#include "pixel_blend.cuh"

#define LP_VP8_FN static __device__
#define LP_VP8_INL static __device__ __forceinline__
#define LP_VP8_HD static __host__ __device__
#define LP_VP8_TABLE static __device__ const
#include "vp8_core.h"
#include "vp8l_core.h"

namespace lp {

// ------------------------------------------------------------------ kernels

struct Vp8Item {
    const uint8_t* data;  // VP8 payload (frame tag onwards), device
    uint32_t size;
    uint8_t* work;        // vp8::work_bytes(mb_w, mb_h)
    int* status;          // 0 ok
    int mb_w, mb_h;       // from the host's look at the 10-byte frame header
};

// One macroblock's edges, warp-wide.  Lanes 0..15 take the luma sample positions of an edge,
// 16..23 the U and 24..31 the V positions.  Order of edges follows RFC 6386 s.15.
__device__ void filter_macroblock_warp(const vp8::FrameHdr& h, vp8::Work& w, int mb_x, int mb_y, int lane) {
    const uint32_t fi = w.finfo[mb_y * h.mb_w + mb_x];
    const int limit = fi & 255, ilevel = (fi >> 8) & 255, hev_t = (fi >> 16) & 255, inner = fi >> 24;
    if (limit == 0) return;
    const int ys = h.mb_w * 16, cs = h.mb_w * 8;
    const int simple = h.filter_type == 1;
    const bool luma = lane < 16;
    uint8_t* base;
    int stride, pos;
    if (luma) {
        base = w.y + (size_t)mb_y * 16 * ys + mb_x * 16;
        stride = ys;
        pos = lane;
    } else {
        base = (lane < 24 ? w.u : w.v) + (size_t)mb_y * 8 * cs + mb_x * 8;
        stride = cs;
        pos = lane & 7;
    }
    const bool active = luma || !simple;
    // vertical edges (filter crosses columns): sample position = row `pos`
    if (mb_x > 0) {
        if (active) {
            uint8_t* p = base + (size_t)pos * stride;
            if (simple) vp8::filter_pos_simple(p, 1, limit + 4);
            else vp8::filter_pos_normal(p, 1, limit + 4, ilevel, hev_t, 1);
        }
        __syncwarp();
    }
    if (inner) {
        for (int k = 4; k < 16; k += 4) {
            if (active && (luma || k == 4)) {
                uint8_t* p = base + (size_t)pos * stride + k;
                if (simple) vp8::filter_pos_simple(p, 1, limit);
                else vp8::filter_pos_normal(p, 1, limit, ilevel, hev_t, 0);
            }
            __syncwarp();
        }
    }
    // horizontal edges (filter crosses rows): sample position = column `pos`
    if (mb_y > 0) {
        if (active) {
            uint8_t* p = base + pos;
            if (simple) vp8::filter_pos_simple(p, stride, limit + 4);
            else vp8::filter_pos_normal(p, stride, limit + 4, ilevel, hev_t, 1);
        }
        __syncwarp();
    }
    if (inner) {
        for (int k = 4; k < 16; k += 4) {
            if (active && (luma || k == 4)) {
                uint8_t* p = base + (size_t)k * stride + pos;
                if (simple) vp8::filter_pos_simple(p, stride, limit);
                else vp8::filter_pos_normal(p, stride, limit, ilevel, hev_t, 0);
            }
            __syncwarp();
        }
    }
}

constexpr int kVp8WarpsPerBlock = 4;

// Per-warp shared state of the decode kernel.
struct Vp8WarpSmem {
    vp8::FrameHdr hdr;
    vp8::MbInfo mb;
    alignas(16) int16_t coeffs[25 * 16];
    alignas(16) uint8_t yb[vp8::YB_SIZE];
    alignas(16) uint8_t ub[vp8::CB_SIZE];
    alignas(16) uint8_t vb[vp8::CB_SIZE];
};

// 16x16 / 8x8 prediction spread over lanes: `dst` block of `size`, this lane fills `n` pixels
// starting at (row, col).  The DC sum arrives pre-reduced.
__device__ __forceinline__ void pred_span(uint8_t* dst, int size, int mode, int row, int col, int n, int dc) {
    uint8_t* d = dst + row * vp8::BPS + col;
    if (mode == vp8::DC_PRED) {
        for (int i = 0; i < n; i++) d[i] = (uint8_t)dc;
    } else if (mode == vp8::TM_PRED) {
        const uint8_t* top = dst - vp8::BPS;
        const int l = dst[row * vp8::BPS - 1] - top[-1];
        for (int i = 0; i < n; i++) d[i] = vp8::clip8(top[col + i] + l);
    } else if (mode == vp8::V_PRED) {
        const uint8_t* top = dst - vp8::BPS;
        for (int i = 0; i < n; i++) d[i] = top[col + i];
    } else {
        const uint8_t l = dst[row * vp8::BPS - 1];
        for (int i = 0; i < n; i++) d[i] = l;
    }
}

// Sum over a group of `width` consecutive lanes (width = 16 or 32), result in every lane of it.
__device__ __forceinline__ int group_sum(int v, int width) {
    for (int o = width >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Reconstructs one parsed macroblock with the whole warp (same arithmetic as vp8::reconstruct_mb).
__device__ void reconstruct_mb_warp(Vp8WarpSmem& sm, vp8::Work& w, int mb_x, int mb_y, int lane) {
    using namespace vp8;
    const FrameHdr& h = sm.hdr;
    const MbInfo& mb = sm.mb;
    const int mb_w = h.mb_w, ys = mb_w * 16, cs = mb_w * 8;
    uint8_t* yd = sm.yb + BPS + 8;
    uint8_t* ud = sm.ub + BPS + 8;
    uint8_t* vd = sm.vb + BPS + 8;
    uint8_t* py = w.y + (size_t)mb_y * 16 * ys + mb_x * 16;
    uint8_t* pu = w.u + (size_t)mb_y * 8 * cs + mb_x * 8;
    uint8_t* pv = w.v + (size_t)mb_y * 8 * cs + mb_x * 8;
    const bool have_top = mb_y > 0, have_left = mb_x > 0;
    // ---- borders (s.12.2) ----
    if (lane < 16) {
        yd[lane * BPS - 1] = have_left ? py[lane * ys - 1] : 129;
    } else {
        const int j = lane & 7;
        uint8_t* cd = lane < 24 ? ud : vd;
        const uint8_t* pc = lane < 24 ? pu : pv;
        cd[j * BPS - 1] = have_left ? pc[j * cs - 1] : 129;
    }
    if (lane < 21) {  // luma: top-left, 16 above, 4 above-right
        const int i = lane - 1;
        uint8_t v = 127;
        if (have_top) {
            if (i < 0) v = have_left ? py[-1 - ys] : 129;
            else if (i < 16 || mb_x < mb_w - 1) v = py[i - ys];
            else v = py[15 - ys];
        }
        yd[i - BPS] = v;
    }
    {
        const int i = (lane & 15) - 1;  // chroma: top-left + 8 above, U on lanes 0..8, V on 16..24
        if (i < 8) {
            uint8_t* cd = lane < 16 ? ud : vd;
            const uint8_t* pc = lane < 16 ? pu : pv;
            uint8_t v = 127;
            if (have_top) v = i < 0 ? (have_left ? pc[-1 - cs] : 129) : pc[i - cs];
            cd[i - BPS] = v;
        }
    }
    __syncwarp();
    // ---- luma prediction ----
    if (!mb.is_i4x4) {
        int dc = 0x80;
        if (mb.ymode == DC_PRED) {
            int v = 0;
            if (lane < 16) v = have_top ? yd[lane - BPS] : 0;
            else v = have_left ? yd[(lane - 16) * BPS - 1] : 0;
            const int s = group_sum(v, 32);
            if (have_top && have_left) dc = (s + 16) >> 5;
            else if (have_top || have_left) dc = (s + 8) >> 4;
        }
        pred_span(yd, 16, mb.ymode, lane >> 1, (lane & 1) * 8, 8, dc);
    } else if (lane == 0) {
        for (int r = 1; r < 4; r++)
            for (int i = 16; i < 20; i++) yd[(4 * r - 1) * BPS + i] = yd[i - BPS];
        for (int n = 0; n < 16; n++) {
            uint8_t* d = yd + (n >> 2) * 4 * BPS + (n & 3) * 4;
            pred_4x4(d, BPS, mb.modes[n]);
            transform_add((mb.tr_y >> 2 * n) & 3, sm.coeffs + n * 16, d, BPS);
        }
    }
    // ---- chroma prediction: U on lanes 0..15, V on 16..31, 4 pixels each ----
    {
        uint8_t* cd = lane < 16 ? ud : vd;
        const int l = lane & 15;
        int dc = 0x80;
        if (mb.uvmode == DC_PRED) {
            int v = 0;
            if (l < 8) v = have_top ? cd[l - BPS] : 0;
            else v = have_left ? cd[(l - 8) * BPS - 1] : 0;
            const int s = group_sum(v, 16);
            if (have_top && have_left) dc = (s + 8) >> 4;
            else if (have_top || have_left) dc = (s + 4) >> 3;
        }
        pred_span(cd, 8, mb.uvmode, l >> 1, (l & 1) * 4, 4, dc);
    }
    __syncwarp();
    // ---- residuals: one 4x4 block per lane (i4x4 luma was added in order above) ----
    if (lane < 24 && !(mb.is_i4x4 && lane < 16)) {
        const int cls = lane < 16 ? (mb.tr_y >> 2 * lane) & 3 : uv_transform(mb.tr_uv, lane - 16);
        uint8_t* d;
        if (lane < 16) d = yd + (lane >> 2) * 4 * BPS + (lane & 3) * 4;
        else {
            const int n = lane & 3;
            d = (lane < 20 ? ud : vd) + (n >> 1) * 4 * BPS + (n & 1) * 4;
        }
        transform_add(cls, sm.coeffs + lane * 16, d, BPS);
    }
    __syncwarp();
    // ---- store: luma row per lane 0..15, chroma row per lane 16..31 ----
    if (lane < 16) {
        const uint2 a = *reinterpret_cast<const uint2*>(yd + lane * BPS);
        const uint2 b = *reinterpret_cast<const uint2*>(yd + lane * BPS + 8);
        *reinterpret_cast<uint4*>(py + (size_t)lane * ys) = make_uint4(a.x, a.y, b.x, b.y);
    } else {
        const int j = lane & 7;
        const uint8_t* cd = lane < 24 ? ud : vd;
        uint8_t* pc = lane < 24 ? pu : pv;
        *reinterpret_cast<uint2*>(pc + (size_t)j * cs) = *reinterpret_cast<const uint2*>(cd + j * BPS);
    }
    __syncwarp();
}

__global__ void __launch_bounds__(kVp8WarpsPerBlock * 32) vp8_decode_kernel(const Vp8Item* items, int n) {
    __shared__ Vp8WarpSmem s_warp[kVp8WarpsPerBlock];
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int idx = blockIdx.x * kVp8WarpsPerBlock + wid;
    if (idx >= n) return;
    const Vp8Item it = items[idx];
    Vp8WarpSmem& sm = s_warp[wid];
    vp8::FrameHdr& h = sm.hdr;
    vp8::Work w;
    vp8::work_carve(it.work, it.mb_w, it.mb_h, w);
    int st = 0;
    vp8::BoolDec br;        // first partition (lane 0)
    vp8::BoolDec parts[8];  // token partitions (lane 0)
    if (lane == 0) {
        st = vp8::parse_frame_header(it.data, it.size, h, br, w.proba);
        if (!st && (h.mb_w != it.mb_w || h.mb_h != it.mb_h)) st = vp8::VP8_BAD;
        if (!st)
            for (int p = 0; p < h.num_parts; p++) vp8::bd_init(parts[p], it.data + h.part_off[p], h.part_len[p]);
        if (st) *it.status = st;  // zeroed by the launcher; an ALPH error must survive
    }
    st = __shfl_sync(0xffffffffu, st, 0);
    __syncwarp();
    if (st) return;
    const int mb_w = h.mb_w, mb_h = h.mb_h;
    for (int i = lane; i < mb_w * 4; i += 32) w.top_modes[i] = vp8::B_DC;
    for (int i = lane; i < mb_w * 9; i += 32) w.top_nz[i] = 0;
    __syncwarp();
    uint32_t* cz = reinterpret_cast<uint32_t*>(sm.coeffs);
    for (int mb_y = 0; mb_y < mb_h; mb_y++) {
        vp8::RowCtx rc;
        vp8::BoolDec tbr;
        if (lane == 0) {
            vp8::row_ctx_reset(rc);
            tbr = parts[mb_y & (h.num_parts - 1)];
        }
        for (int mb_x = 0; mb_x < mb_w; mb_x++) {
            for (int i = lane; i < 25 * 8; i += 32) cz[i] = 0;
            __syncwarp();
            if (lane == 0) {
                const int skip = vp8::parse_mb_modes(h, br, w.top_modes + mb_x * 4, rc, sm.mb);
                vp8::parse_mb_residuals(h, tbr, w.proba, w.top_nz + mb_x * 9, rc, skip, sm.mb, sm.coeffs);
                w.finfo[mb_y * mb_w + mb_x] = sm.mb.finfo;
            }
            __syncwarp();
            reconstruct_mb_warp(sm, w, mb_x, mb_y, lane);
        }
        if (lane == 0) parts[mb_y & (h.num_parts - 1)] = tbr;
    }
    if (lane == 0 && vp8::frame_truncated(h, br, parts)) *it.status = vp8::VP8_BAD;
    __syncwarp();
    if (h.filter_type == 0) return;
    for (int mb_y = 0; mb_y < mb_h; mb_y++)
        for (int mb_x = 0; mb_x < mb_w; mb_x++) filter_macroblock_warp(h, w, mb_x, mb_y, lane);
}

// VP8L (lossless) frames and ALPH planes: an LZ77 + prefix-coded stream is one serial chain, so
// lane 0 of one warp per stream walks it (vp8l_core.h) inside its own slice of a bump arena in HBM.
// The colour-order conversion onto the canvas is the compositor's.
struct Vp8lItem {
    const uint8_t* data;   // "VP8L" chunk payload, or "ALPH" chunk payload
    uint32_t size;
    int width, height;
    uint8_t* arena;
    size_t arena_cap;
    int is_alph;
    uint8_t* alpha_out;    // is_alph: width*height plane
    uint32_t* argb_out;    // !is_alph: where the warp copies the final ARGB pixels (the arena is reused by the next wave)
    int* status;
};

constexpr int kVp8lWarpsPerBlock = 4;

__global__ void __launch_bounds__(kVp8lWarpsPerBlock * 32) vp8l_decode_kernel(const Vp8lItem* items, int n) {
    const int idx = blockIdx.x * kVp8lWarpsPerBlock + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (idx >= n) return;
    const Vp8lItem& it = items[idx];
    int rc = 0;
    uint32_t* px = nullptr;
    if (lane == 0) {
        vp8l::Arena a{it.arena, it.arena_cap, 0};
        if (it.is_alph) {
            rc = vp8l::decode_alph(it.data, it.size, it.width, it.height, a, it.alpha_out);
        } else {
            rc = vp8l::decode_vp8l(it.data, it.size, it.width, it.height, a, &px);
        }
        if (rc) *it.status = rc;
    }
    if (it.is_alph) return;
    rc = __shfl_sync(0xffffffffu, rc, 0);
    px = reinterpret_cast<uint32_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(px), 0));
    if (rc || !px) return;
    // One warp copies the frame, so it keeps eight 16-byte loads in flight per lane (arena allocations and scratch slots
    // are 16-byte aligned).  The pixels were written in this launch: plain loads, not the read-only path.
    const size_t npix = (size_t)it.width * it.height, nvec = npix / 4;
    const uint4* src = reinterpret_cast<const uint4*>(px);
    uint4* dst = reinterpret_cast<uint4*>(it.argb_out);
    size_t i = lane;
    for (; i + 7 * 32 < nvec; i += 8 * 32) {
        uint4 v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u] = src[i + u * 32];
#pragma unroll
        for (int u = 0; u < 8; u++) dst[i + u * 32] = v[u];
    }
    for (; i < nvec; i += 32) dst[i] = src[i];
    for (size_t j = nvec * 4 + lane; j < npix; j += 32) it.argb_out[j] = px[j];
}

static int vp8l_decode_launch(const Vp8lItem* d_items, int n, cudaStream_t st) {
    if (n <= 0) return LP_OK;
    vp8l_decode_kernel<<<ceil_div(n, kVp8lWarpsPerBlock), kVp8lWarpsPerBlock * 32, 0, st>>>(d_items, n);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

// ------------------------------------------------------------------ frame compositor (batch path)
// Every frame of every animation (a still is one frame, copied) straight from the decoders' output onto its canvas:
// one thread per canvas pixel walks the frame sequence with the pixel's state in registers, exactly the per-image
// region-op sequence of ImageOps (ref ops.go:170-238, 552-582): blend or copy the frame's pixel -> store the composited
// canvas -> clear the pixel if the frame disposes to background.  Every step is a function of one pixel.
struct WebpFrameJob {
    uint64_t work_off;   // lossy: VP8 work area, from the scratch base
    uint64_t px_off;     // lossless: ARGB words; lossy: ALPH plane (~0: none, alpha 255)
    int32_t x, y, w, h;
    int32_t lossless, blend, dispose, mb_w, mb_h;
    int32_t canvas;  // canvas of its file the composited frame is stored at; -1: composited, not stored
};
struct WebpAnimJob {
    uint64_t canvas_off, canvas_stride;
    int32_t first_frame, nframes, width, height, channels, pad_;
};

__global__ void webp_compose_kernel(const WebpAnimJob* anims, const WebpFrameJob* jobs, const uint8_t* base, uint8_t* canvases) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    const WebpAnimJob a = anims[blockIdx.z];
    if (x >= a.width || y >= a.height) return;
    const int ch = a.channels;
    uint8_t px[4] = {0, 0, 0, 0};  // the composite buffer starts transparent (ClearToTransparent of the whole canvas)
    uint8_t* out = canvases + a.canvas_off + ((size_t)y * a.width + x) * ch;
    for (int k = 0; k < a.nframes; k++) {
        const WebpFrameJob& f = jobs[a.first_frame + k];
        const int fx = x - f.x, fy = y - f.y;
        const bool inside = fx >= 0 && fx < f.w && fy >= 0 && fy < f.h;
        if (inside) {
            uint8_t s[4];
            const size_t at = (size_t)fy * f.w + fx;
            if (f.lossless) {
                const uint32_t v = reinterpret_cast<const uint32_t*>(base + f.px_off)[at];
                s[0] = (uint8_t)v;
                s[1] = (uint8_t)(v >> 8);
                s[2] = (uint8_t)(v >> 16);
                s[3] = (uint8_t)(v >> 24);
            } else {
                vp8::Work w;
                vp8::work_carve(const_cast<uint8_t*>(base) + f.work_off, f.mb_w, f.mb_h, w);
                const int u = vp8::upsample_at(w.u, f.mb_w * 8, f.w, f.h, fx, fy);
                const int v = vp8::upsample_at(w.v, f.mb_w * 8, f.w, f.h, fx, fy);
                vp8::yuv_to_bgr(w.y[(size_t)fy * (f.mb_w * 16) + fx], u, v, s);
                s[3] = f.px_off != ~0ull ? base[f.px_off + at] : 255;
            }
            if (f.blend) {  // NoBlend: copyTo, equal channel counts
                for (int c = 0; c < ch; c++) px[c] = s[c];
            } else {
                blend_px(s, ch, px, ch);
            }
        }
        if (f.canvas >= 0) {
            uint8_t* d = out + (size_t)f.canvas * a.canvas_stride;
            for (int c = 0; c < ch; c++) d[c] = px[c];
        }
        if (inside && f.dispose) px[0] = px[1] = px[2] = px[3] = 0;
    }
}

// ------------------------------------------------------------------ container walk (host)
// RIFF layout per the WebP container specification; checks follow what WebPMuxCreate /
// MuxValidate reject (ref webp.cpp:65-69 treats a NULL mux as "not a WebP").

static inline uint32_t le16(const uint8_t* p) { return p[0] | (p[1] << 8); }
static inline uint32_t le24(const uint8_t* p) { return p[0] | (p[1] << 8) | ((uint32_t)p[2] << 16); }
static inline uint32_t le32(const uint8_t* p) { return le24(p) | ((uint32_t)p[3] << 24); }

enum { kFlagAnim = 0x02, kFlagXmp = 0x04, kFlagExif = 0x08, kFlagAlpha = 0x10, kFlagIcc = 0x20 };
constexpr uint32_t kMaxChunkPayload = ~0u - 8 - 1;

struct WebpFrame {
    size_t img_off = 0, img_len = 0;  // VP8 / VP8L payload
    bool lossless = false;
    size_t alph_off = 0, alph_len = 0;
    bool has_alph = false;
    int x_off = 0, y_off = 0, width = 0, height = 0;
    int duration = 0, dispose = 0, blend = 0;
    bool has_alpha = false;  // ALPH chunk, or VP8L header alpha bit
};

struct WebpContainer {
    int canvas_w = 0, canvas_h = 0;
    uint32_t flags = 0;
    bool has_vp8x = false, has_anim_chunk = false;
    uint32_t bgcolor = 0xFFFFFFFFu, loop_count = 0;
    size_t icc_off = 0, icc_len = 0;
    bool has_icc = false, has_exif = false, has_xmp = false;
    std::vector<WebpFrame> frames;
};

// Validates an image payload and fills the frame's size (VP8GetInfo / VP8LGetInfo equivalents).
static bool image_info(const uint8_t* p, size_t n, bool lossless, WebpFrame* f) {
    if (!lossless) {
        if (n < 10) return false;
        const uint32_t tag = le24(p);
        if (tag & 1) return false;                       // not a key frame
        if (((tag >> 1) & 7) > 3) return false;          // unknown profile
        if (!((tag >> 4) & 1)) return false;             // invisible frame
        if ((tag >> 5) >= n) return false;               // partition_length beyond the chunk
        if (p[3] != 0x9d || p[4] != 0x01 || p[5] != 0x2a) return false;
        f->width = le16(p + 6) & 0x3fff;
        f->height = le16(p + 8) & 0x3fff;
        return f->width > 0 && f->height > 0;
    }
    if (n < 5 || p[0] != 0x2f) return false;
    const uint32_t bits = le32(p + 1);
    f->width = (int)(bits & 0x3fff) + 1;
    f->height = (int)((bits >> 14) & 0x3fff) + 1;
    f->has_alpha = (bits >> 28) & 1;
    return ((bits >> 29) & 7) == 0;  // version
}

// The bytes an image payload of `n` bytes is decoded from, `avail` bytes being left in its container: the
// chunk and its padding byte when there is one.  libwebp's decoders read on to the end of their input, so a
// stream cut short can still draw its last bits from the padding byte, and frames are accepted or refused
// as libwebp accepts or refuses them only if ours do too.  (The header checks use the chunk size.)
static size_t image_span(size_t n, size_t avail) {
    const size_t padded = n + (n & 1);
    return padded < avail ? padded : avail;
}

// Walks the sub-chunks that make up one image (ALPH? then VP8 / VP8L) in [pos, end).
static bool parse_image_chunks(const uint8_t* b, size_t pos, size_t end, WebpFrame* f, bool* got_image) {
    *got_image = false;
    while (pos + 8 <= end) {
        const uint32_t n = le32(b + pos + 4);
        if (n > kMaxChunkPayload) return false;
        const size_t padded = 8 + (((size_t)n + 1) & ~(size_t)1);
        if (pos + padded > end && pos + 8 + n > end) return false;
        const uint8_t* tag = b + pos;
        if (!memcmp(tag, "ALPH", 4)) {
            if (f->has_alph || *got_image) return false;
            f->has_alph = true;
            f->alph_off = pos + 8;
            f->alph_len = n;
        } else if (!memcmp(tag, "VP8 ", 4) || !memcmp(tag, "VP8L", 4)) {
            if (*got_image) return false;
            f->lossless = tag[3] == 'L';
            f->img_off = pos + 8;
            if (!image_info(b + f->img_off, n, f->lossless, f)) return false;
            f->img_len = image_span(n, end - f->img_off);
            if (f->has_alph && !f->lossless) f->has_alpha = true;
            *got_image = true;
        }
        pos += padded;
    }
    return true;
}

static bool webp_parse(const uint8_t* b, size_t size, WebpContainer* c) {
    if (size < 20 || memcmp(b, "RIFF", 4) || memcmp(b + 8, "WEBP", 4)) return false;
    uint32_t riff = le32(b + 4);
    if (riff > kMaxChunkPayload) return false;
    riff = (riff + 1) & ~1u;
    if (riff < 8 || riff > size) return false;
    if (size > (size_t)riff + 8) size = (size_t)riff + 8;
    size_t pos = 12;
    WebpFrame still;       // image chunks at the top level (non-animated file)
    bool still_open = false, still_done = false;
    while (pos + 8 <= size) {
        const uint8_t* tag = b + pos;
        const uint32_t n = le32(b + pos + 4);
        if (n > kMaxChunkPayload) return false;
        const size_t padded = 8 + (((size_t)n + 1) & ~(size_t)1);
        if (padded > (size_t)riff) return false;
        if (pos + padded > size) return false;  // truncated chunk
        const uint8_t* d = b + pos + 8;
        if (!memcmp(tag, "VP8X", 4)) {
            if (c->has_vp8x || n < 10) return false;
            c->has_vp8x = true;
            c->flags = d[0];
            c->canvas_w = (int)le24(d + 4) + 1;
            c->canvas_h = (int)le24(d + 7) + 1;
        } else if (!memcmp(tag, "ICCP", 4)) {
            if (c->has_icc) return false;
            c->has_icc = true;
            c->icc_off = pos + 8;
            c->icc_len = n;
        } else if (!memcmp(tag, "EXIF", 4)) {
            if (c->has_exif) return false;
            c->has_exif = true;
        } else if (!memcmp(tag, "XMP ", 4)) {
            if (c->has_xmp) return false;
            c->has_xmp = true;
        } else if (!memcmp(tag, "ANIM", 4)) {
            if (c->has_anim_chunk || n < 6) return false;
            c->has_anim_chunk = true;
            c->bgcolor = le32(d);
            c->loop_count = le16(d + 4);
        } else if (!memcmp(tag, "ANMF", 4)) {
            if (still_open || n < 16) return false;
            WebpFrame f;
            f.x_off = 2 * (int)le24(d);
            f.y_off = 2 * (int)le24(d + 3);
            const int fw = (int)le24(d + 6) + 1, fh = (int)le24(d + 9) + 1;
            f.duration = (int)le24(d + 12);
            f.dispose = d[15] & 1;          // 1 = dispose to background
            f.blend = (d[15] >> 1) & 1;     // 1 = do not blend
            bool got = false;
            if (!parse_image_chunks(b, pos + 8 + 16, pos + 8 + n, &f, &got) || !got) return false;
            if (f.width != fw || f.height != fh) return false;
            c->frames.push_back(f);
        } else if (!memcmp(tag, "ALPH", 4)) {
            if (still_open || still_done) return false;
            still_open = true;
            still.has_alph = true;
            still.alph_off = pos + 8;
            still.alph_len = n;
        } else if (!memcmp(tag, "VP8 ", 4) || !memcmp(tag, "VP8L", 4)) {
            if (still_done) return false;
            still.lossless = tag[3] == 'L';
            still.img_off = pos + 8;
            if (!image_info(d, n, still.lossless, &still)) return false;
            still.img_len = image_span(n, size - still.img_off);
            if (still.has_alph && !still.lossless) still.has_alpha = true;
            still_open = false;
            still_done = true;
        } else {
            if (still_open) return false;  // an ALPH chunk must be followed by its image
        }
        pos += padded;
    }
    if (still_open) return false;
    if (still_done) {
        if (!c->frames.empty()) return false;  // ANMF frames and a bare image do not mix
        still.duration = 1;                    // what WebPMuxGetFrame reports for a non-animated image
        c->frames.push_back(still);
    }
    if (c->frames.empty()) return false;
    // MuxValidate: feature flags and chunks must agree
    const bool anim = c->flags & kFlagAnim;
    if (!c->has_vp8x) {
        if (c->frames.size() != 1 || c->frames[0].has_alph || c->has_icc || c->has_anim_chunk || c->has_exif ||
            c->has_xmp)
            return false;
        c->canvas_w = c->frames[0].width;
        c->canvas_h = c->frames[0].height;
        c->flags = c->frames[0].has_alpha ? kFlagAlpha : 0;
    } else {
        if (((c->flags & kFlagIcc) != 0) != c->has_icc) return false;
        if (((c->flags & kFlagExif) != 0) != c->has_exif) return false;
        if (((c->flags & kFlagXmp) != 0) != c->has_xmp) return false;
        if (anim != c->has_anim_chunk) return false;
        if (!anim && (c->frames.size() != 1 || !still_done)) return false;
        if (anim && still_done) return false;
        bool any_alpha = false;
        for (const WebpFrame& f : c->frames) any_alpha |= f.has_alpha;
        if (any_alpha && !(c->flags & kFlagAlpha)) return false;
        for (const WebpFrame& f : c->frames)
            if (f.x_off + f.width > c->canvas_w || f.y_off + f.height > c->canvas_h) return false;
    }
    return true;
}

// ------------------------------------------------------------------ batch helpers (xbatch.cu)

// The per-image decoder's view of a file (webp_decoder_create / _decode / _get_prev_frame_*), from the same walk.
bool webp_plan_parse(const uint8_t* data, size_t len, WebpPlan* out) {
    WebpContainer c;
    if (!webp_parse(data, len, &c)) return false;
    out->width = c.canvas_w;
    out->height = c.canvas_h;
    out->channels = (c.flags & kFlagAlpha) ? 4 : 3;  // webp_decoder_get_pixel_type
    out->animated = (c.flags & kFlagAnim) != 0;
    out->bgcolor = out->animated ? c.bgcolor : 0xFFFFFFFFu;
    out->loop_count = out->animated ? c.loop_count : 0;
    out->icc_off = c.has_icc ? c.icc_off : 0;
    out->icc_len = c.has_icc ? c.icc_len : 0;
    out->frames.clear();
    for (const WebpFrame& f : c.frames) {
        WebpFramePlan p;
        p.img_off = f.img_off;
        p.img_len = f.img_len;
        p.alph_off = f.alph_off;
        p.alph_len = f.alph_len;
        p.lossless = f.lossless;
        p.has_alph = f.has_alph;
        p.x = f.x_off;
        p.y = f.y_off;
        p.width = f.width;
        p.height = f.height;
        p.duration = f.duration;
        p.dispose = f.dispose;
        p.blend = f.blend;
        p.has_alpha = f.has_alpha;
        out->frames.push_back(p);
    }
    return true;
}

size_t webp_plan_cut(WebpPlan* p, int last) {
    p->frames.resize((size_t)last + 1);
    const WebpFramePlan& f = p->frames[(size_t)last];
    return std::max(f.img_off + f.img_len, f.has_alph ? f.alph_off + f.alph_len : 0);
}

// the VP8L arena bound, per stream
static size_t vp8l_slice_bytes(const WebpFramePlan& f) { return round_up((size_t)f.width * f.height * 12 + (16u << 20), (size_t)256); }
// the ALPH plane is decoded only onto a 4-channel canvas (3 channels drop it)
static bool frame_needs_alph(const WebpPlan& p, const WebpFramePlan& f) { return f.has_alph && !f.lossless && p.channels == 4; }
static size_t file_slot_bytes(size_t file_len) { return round_up(file_len + 4096, (size_t)256); }
// VP8 work area, lossless ARGB words or the ALPH plane of one frame
static size_t frame_slot_bytes(const WebpPlan& p, const WebpFramePlan& f) {
    const size_t npix = (size_t)f.width * f.height;
    if (f.lossless) return round_up(npix * 4, (size_t)256);
    return round_up(vp8::work_bytes((f.width + 15) >> 4, (f.height + 15) >> 4), (size_t)256) +
           (frame_needs_alph(p, f) ? round_up(npix, (size_t)256) : 0);
}
static constexpr size_t kFrameRecordBytes = sizeof(WebpFrameJob) + sizeof(Vp8Item) + sizeof(Vp8lItem) + 4;

size_t webp_plan_device_bytes(const WebpPlan& p, size_t file_len) {
    size_t b = file_slot_bytes(file_len) + sizeof(WebpAnimJob) + 5 * 256;
    for (const WebpFramePlan& f : p.frames) b += frame_slot_bytes(p, f) + kFrameRecordBytes;
    return b;
}

size_t webp_plan_arena_bytes(const WebpPlan& p) {
    size_t b = 0;
    for (const WebpFramePlan& f : p.frames)
        if (f.lossless || frame_needs_alph(p, f)) b += vp8l_slice_bytes(f);
    return b;
}

// Uploads the files, then: ONE vp8_decode_kernel launch over every lossy frame (one warp per frame), the VP8L / ALPH
// streams in waves of one launch each (one warp per stream, each with its own arena slice), and ONE compositor launch
// over every canvas pixel of every file (per run of equal canvas size).
int webp_decode_batch(const WebpPlan* const* plans, const uint8_t* const* files, const size_t* file_len, int n,
                      uint8_t* d_scratch, size_t scratch_bytes, uint8_t* d_arena, size_t arena_bytes, uint8_t* d_canvases,
                      const uint64_t* canvas_off, int* h_status, cudaEvent_t ev_uploaded, cudaStream_t st,
                      const int* canvas_of) {
    if (n <= 0) return LP_OK;
    int nf = 0;
    for (int a = 0; a < n; a++) nf += (int)plans[a]->frames.size();
    // records first, then the files, then the per-frame slots
    size_t used = 0;
    auto take = [&](size_t bytes) {
        const size_t at = used;
        used += round_up(bytes, (size_t)256);
        return at;
    };
    const size_t anims_at = take((size_t)n * sizeof(WebpAnimJob)), jobs_at = take((size_t)nf * sizeof(WebpFrameJob));
    const size_t vp8_at = take((size_t)nf * sizeof(Vp8Item)), vp8l_at = take((size_t)nf * sizeof(Vp8lItem));
    const size_t status_at = take((size_t)nf * 4);
    std::vector<size_t> file_at((size_t)n);
    for (int a = 0; a < n; a++) file_at[a] = take(file_slot_bytes(file_len[a]));
    std::vector<WebpAnimJob> anims((size_t)n);
    std::vector<WebpFrameJob> jobs((size_t)nf);
    std::vector<Vp8Item> vp8;
    std::vector<Vp8lItem> vp8l;
    std::vector<size_t> slice;  // arena bytes of every VP8L / ALPH stream
    int* d_status = reinterpret_cast<int*>(d_scratch + status_at);
    for (int a = 0, k = 0; a < n; a++) {
        const WebpPlan& p = *plans[a];
        WebpAnimJob& aj = anims[a];
        memset(&aj, 0, sizeof(aj));
        aj.canvas_off = canvas_off[a];
        aj.canvas_stride = round_up((size_t)p.width * p.height * p.channels, (size_t)256);
        aj.first_frame = k;
        aj.nframes = (int)p.frames.size();
        aj.width = p.width;
        aj.height = p.height;
        aj.channels = p.channels;
        const uint8_t* d_file = d_scratch + file_at[a];
        for (const WebpFramePlan& f : p.frames) {
            WebpFrameJob& j = jobs[k];
            memset(&j, 0, sizeof(j));
            j.x = f.x;
            j.y = f.y;
            j.w = f.width;
            j.h = f.height;
            j.lossless = f.lossless;
            j.blend = f.blend;
            j.dispose = f.dispose;
            j.mb_w = (f.width + 15) >> 4;
            j.mb_h = (f.height + 15) >> 4;
            j.px_off = ~0ull;
            j.canvas = canvas_of ? canvas_of[k] : k - aj.first_frame;
            const size_t npix = (size_t)f.width * f.height;
            if (f.lossless) {
                j.px_off = take(npix * 4);
                vp8l.push_back(Vp8lItem{d_file + f.img_off, (uint32_t)f.img_len, f.width, f.height, nullptr, 0, 0, nullptr,
                                        reinterpret_cast<uint32_t*>(d_scratch + j.px_off), d_status + k});
                slice.push_back(vp8l_slice_bytes(f));
            } else {
                j.work_off = take(vp8::work_bytes(j.mb_w, j.mb_h));
                vp8.push_back(Vp8Item{d_file + f.img_off, (uint32_t)f.img_len, d_scratch + j.work_off, d_status + k, j.mb_w, j.mb_h});
                if (frame_needs_alph(p, f)) {
                    j.px_off = take(npix);
                    vp8l.push_back(Vp8lItem{d_file + f.alph_off, (uint32_t)f.alph_len, f.width, f.height, nullptr, 0, 1,
                                            d_scratch + j.px_off, nullptr, d_status + k});
                    slice.push_back(vp8l_slice_bytes(f));
                }
            }
            k++;
        }
    }
    if (used > scratch_bytes) return LP_ERR_BUF_TOO_SMALL;
    // VP8L / ALPH waves: consecutive streams while their slices fit the arena (a stream larger than the whole arena
    // gets all of it: arena exhaustion is a clean decode error, and its file goes to the caller's fallback)
    std::vector<int> wave_first;
    for (size_t s = 0, fill = 0; s < vp8l.size(); s++) {
        const size_t need = std::min(slice[s], arena_bytes);
        if (s == 0 || fill + need > arena_bytes) {
            wave_first.push_back((int)s);
            fill = 0;
        }
        vp8l[s].arena = d_arena + fill;
        vp8l[s].arena_cap = need;
        fill += need;
    }
    wave_first.push_back((int)vp8l.size());
    if (!vp8l.empty() && (!d_arena || arena_bytes == 0)) return LP_ERR_BUF_TOO_SMALL;
    int rc = LP_OK;
    auto up = [&](size_t at, const void* src, size_t bytes) {
        if (!rc && bytes && cudaMemcpyAsync(d_scratch + at, src, bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) rc = LP_ERR_CUDA;
    };
    for (int a = 0; a < n; a++) up(file_at[a], files[a], file_len[a]);
    up(anims_at, anims.data(), anims.size() * sizeof(WebpAnimJob));
    up(jobs_at, jobs.data(), jobs.size() * sizeof(WebpFrameJob));
    up(vp8_at, vp8.data(), vp8.size() * sizeof(Vp8Item));
    up(vp8l_at, vp8l.data(), vp8l.size() * sizeof(Vp8lItem));
    if (!rc && cudaMemsetAsync(d_status, 0, (size_t)nf * 4, st) != cudaSuccess) rc = LP_ERR_CUDA;
    if (ev_uploaded) cudaEventRecord(ev_uploaded, st);
    if (!rc && !vp8.empty()) {
        const int m = (int)vp8.size();
        vp8_decode_kernel<<<ceil_div(m, kVp8WarpsPerBlock), kVp8WarpsPerBlock * 32, 0, st>>>(
            reinterpret_cast<const Vp8Item*>(d_scratch + vp8_at), m);
        g_launches++;
        if (cudaGetLastError() != cudaSuccess) rc = LP_ERR_CUDA;
    }
    const Vp8lItem* d_vp8l = reinterpret_cast<const Vp8lItem*>(d_scratch + vp8l_at);
    for (size_t w = 0; !rc && w + 1 < wave_first.size(); w++)
        rc = vp8l_decode_launch(d_vp8l + wave_first[w], wave_first[w + 1] - wave_first[w], st);
    // one compositor launch per run of equal canvas size (the caller keeps equal sizes adjacent), <= 65535 files each
    for (int a0 = 0; !rc && a0 < n;) {
        int a1 = a0 + 1;
        while (a1 < n && a1 - a0 < 65535 && plans[a1]->width == plans[a0]->width && plans[a1]->height == plans[a0]->height) a1++;
        webp_compose_kernel<<<dim3(ceil_div(plans[a0]->width, 128), plans[a0]->height, a1 - a0), 128, 0, st>>>(
            reinterpret_cast<const WebpAnimJob*>(d_scratch + anims_at) + a0, reinterpret_cast<const WebpFrameJob*>(d_scratch + jobs_at),
            d_scratch, d_canvases);
        g_launches++;
        if (cudaGetLastError() != cudaSuccess) rc = LP_ERR_CUDA;
        a0 = a1;
    }
    std::vector<int> fst((size_t)nf, 0);
    if (!rc && (cudaMemcpyAsync(fst.data(), d_status, (size_t)nf * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                cudaStreamSynchronize(st) != cudaSuccess))  // (also keeps the host records alive until the copies are done)
        rc = LP_ERR_CUDA;
    if (rc) return rc;
    for (int a = 0; a < n; a++) {
        h_status[a] = 0;
        for (int k = anims[a].first_frame; k < anims[a].first_frame + anims[a].nframes; k++)
            if (fst[k]) h_status[a] = fst[k];
    }
    return LP_OK;
}

// The mat handle is defined in abi_opencv.cu.
const uint8_t* mat_host_bytes(const void* mat, size_t* len);
int mat_bind_device_frame(void* mat, int cols, int rows, int type, uint8_t** dev, size_t* step);
void mat_mark_device_written(void* mat);

}  // namespace lp

using namespace lp;

struct webp_decoder_struct {
    const uint8_t* bytes = nullptr;
    WebpPlan plan;
    int total_duration = 0;
    int current_frame_index = 1;
    int prev_delay = 0, prev_x = 0, prev_y = 0, prev_dispose = 0, prev_blend = 0;
    bool prev_has_alpha = false;
    // device scratch of webp_decode_batch (webp_plan_device_bytes) and its VP8L / ALPH arena, grown on demand
    uint8_t* d_scratch = nullptr;
    uint8_t* d_arena = nullptr;
    size_t scratch_cap = 0, arena_cap = 0;
};

extern "C" {

// ref webp.cpp:61-139
webp_decoder webp_decoder_create(const opencv_mat buf) {
    if (!buf) return nullptr;
    size_t len = 0;
    const uint8_t* bytes = mat_host_bytes(buf, &len);
    if (!bytes) return nullptr;
    auto* d = new webp_decoder_struct;
    d->bytes = bytes;
    if (!webp_plan_parse(bytes, len, &d->plan)) {
        delete d;
        return nullptr;
    }
    if (d->plan.animated)
        for (const WebpFramePlan& f : d->plan.frames) d->total_duration += f.duration;
    return d;
}

int webp_decoder_get_width(const webp_decoder d) { return d->plan.width; }
int webp_decoder_get_height(const webp_decoder d) { return d->plan.height; }
int webp_decoder_get_pixel_type(const webp_decoder d) { return d->plan.channels == 4 ? CV_8UC4 : CV_8UC3; }
int webp_decoder_get_num_frames(const webp_decoder d) { return d ? (int)d->plan.frames.size() : 0; }
int webp_decoder_get_total_duration(const webp_decoder d) { return d ? d->total_duration : 0; }
int webp_decoder_get_prev_frame_delay(const webp_decoder d) { return d->prev_delay; }
int webp_decoder_get_prev_frame_dispose(const webp_decoder d) { return d->prev_dispose; }
int webp_decoder_get_prev_frame_blend(const webp_decoder d) { return d->prev_blend; }
int webp_decoder_get_prev_frame_x_offset(const webp_decoder d) { return d->prev_x; }
int webp_decoder_get_prev_frame_y_offset(const webp_decoder d) { return d->prev_y; }
bool webp_decoder_get_prev_frame_has_alpha(const webp_decoder d) { return d->prev_has_alpha; }
uint32_t webp_decoder_get_bg_color(const webp_decoder d) { return d->plan.bgcolor; }
uint32_t webp_decoder_get_loop_count(const webp_decoder d) { return d->plan.loop_count; }

// ref webp.cpp:251-262
size_t webp_decoder_get_icc(const webp_decoder d, void* dst, size_t dst_len) {
    if (d->plan.icc_len == 0 || d->plan.icc_len > dst_len) return 0;
    memcpy(dst, d->bytes + d->plan.icc_off, d->plan.icc_len);
    return d->plan.icc_len;
}

// ref webp.cpp:269-281
int webp_decoder_has_more_frames(webp_decoder d) { return d->current_frame_index < (int)d->plan.frames.size(); }
void webp_decoder_advance_frame(webp_decoder d) { d->current_frame_index++; }

void webp_decoder_release(webp_decoder d) {
    if (!d) return;
    cudaStream_t st = thread_stream();
    if (d->d_scratch) cudaFreeAsync(d->d_scratch, st);
    if (d->d_arena) cudaFreeAsync(d->d_arena, st);
    cudaStreamSynchronize(st);
    delete d;
}

// ref webp.cpp:291-359
bool webp_decoder_decode(const webp_decoder d, opencv_mat mat) {
    if (!d || !mat) return false;
    if (d->current_frame_index < 1 || d->current_frame_index > (int)d->plan.frames.size()) return false;
    const WebpFramePlan& f = d->plan.frames[d->current_frame_index - 1];
    const int type = webp_decoder_get_pixel_type(d);
    uint8_t* frame_dev = nullptr;
    size_t frame_step = 0;
    if (mat_bind_device_frame(mat, f.width, f.height, type, &frame_dev, &frame_step) != 0) return false;
    d->prev_delay = f.duration;
    d->prev_x = f.x;
    d->prev_y = f.y;
    d->prev_dispose = f.dispose;
    d->prev_blend = f.blend;
    d->prev_has_alpha = f.has_alpha;
    // the compositor writes packed rows, as a freshly bound mat has them
    if (frame_step != (size_t)f.width * d->plan.channels) return false;
    // The frame alone, as the batch decodes a still: a canvas of the frame's size with the frame copied at its origin.
    // Only the frame's own chunks go up (an ALPH chunk precedes its image), with offsets from the first of them.
    const size_t begin = f.has_alph ? f.alph_off : f.img_off;
    WebpPlan one;
    one.width = f.width;
    one.height = f.height;
    one.channels = d->plan.channels;
    one.frames.push_back(f);
    WebpFramePlan& g = one.frames[0];
    g.img_off -= begin;
    g.alph_off = 0;
    g.x = g.y = 0;
    g.blend = 1;
    g.dispose = 0;
    const uint8_t* file = d->bytes + begin;
    const size_t span = f.img_off + f.img_len - begin;
    cudaStream_t st = thread_stream();
    auto grow = [&](uint8_t** p, size_t* cap, size_t need) -> bool {
        if (need <= *cap) return true;
        if (*p) cudaFreeAsync(*p, st);
        *cap = 0;
        if (cudaMallocAsync(p, need, st) != cudaSuccess) {
            *p = nullptr;
            return false;
        }
        *cap = need;
        return true;
    };
    if (!grow(&d->d_scratch, &d->scratch_cap, webp_plan_device_bytes(one, span))) return false;
    if (!grow(&d->d_arena, &d->arena_cap, webp_plan_arena_bytes(one))) return false;
    const WebpPlan* plans[1] = {&one};
    const uint64_t canvas_off = 0;
    int status = 0;
    if (webp_decode_batch(plans, &file, &span, 1, d->d_scratch, d->scratch_cap, d->d_arena, d->arena_cap, frame_dev,
                          &canvas_off, &status, nullptr, st) != LP_OK || status != 0)
        return false;
    mat_mark_device_written(mat);
    return true;
}

}  // extern "C"
