// pixel_ops.cu -- orientation, region copy, alpha blend, clear/fill on packed u8 frames.
//
// Replaces: cv::OrientationTransform (ref opencv.cpp:217-221), opencv_copy_to_region
// (ref opencv.cpp:680-752), opencv_copy_to_region_with_alpha (ref opencv.cpp:556-667),
// opencv_mat_clear_to_transparent / reset / set_color (ref opencv.cpp:466-543).
// All are byte moves except the blend, which is fp32 with every OpenCV Mat expression
// rounded on its own (explicit __f*_rn intrinsics: no FMA contraction), RNE to u8.
#include "common.cuh"
#include "kernels.cuh"
#include "pixel_blend.cuh"

namespace lp {

// EXIF orientation: destination pixel (x, y) <- source pixel, golden table SURVEY.md 8a R4.
__global__ void orient_kernel(const uint8_t* __restrict__ src, int w, int h, int C, int o,
                              uint8_t* __restrict__ dst, int W, int H) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= W || y >= H) return;
    int sx, sy;
    orient_source_pixel(o, w, h, x, y, &sx, &sy);
    const uint8_t* s = src + ((size_t)sy * w + sx) * C;
    uint8_t* d = dst + ((size_t)y * W + x) * C;
    for (int c = 0; c < C; c++) d[c] = s[c];
}

int orient_launch(const uint8_t* src, int w, int h, int C, int o, uint8_t* dst, cudaStream_t st) {
    const bool swap = o >= 5 && o <= 8;
    const int W = swap ? h : w, H = swap ? w : h;
    dim3 grid(ceil_div(W, 128), H);
    orient_kernel<<<grid, 128, 0, st>>>(src, w, h, C, o, dst, W, H);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

// Oriented crops of decoded windows (batch.cu): one CTA per 32 x 32 tile of a job's crop.  Under every orientation the
// tile's source pixels form a rectangle of the window of at most 32 x 32; it is read row by row into shared memory (a
// pixel of C = 3 (BGR) or 1 (gray) bytes per 32-bit word, rows padded to 33 words so that a column is conflict-free) and
// the tile is written row by row of the crop, so both sides move runs of consecutive pixels even when the orientation
// transposes.
template <int C>
__global__ void __launch_bounds__(256)
    orient_crop_kernel(const OrientJob* __restrict__ jobs, const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                       int w, int h) {
    __shared__ uint32_t tile[32][33];
    const OrientJob j = jobs[blockIdx.z];
    const int x0 = blockIdx.x * 32, y0 = blockIdx.y * 32;
    if (x0 >= j.cw || y0 >= j.ch) return;  // (uniform over the CTA)
    const int x1 = min(x0 + 32, j.cw) - 1, y1 = min(y0 + 32, j.ch) - 1;
    int ax, ay, bx, by;  // pre-images of the tile's first and last pixel: opposite corners of its source rectangle
    orient_source_pixel(j.o, w, h, j.cx + x0, j.cy + y0, &ax, &ay);
    orient_source_pixel(j.o, w, h, j.cx + x1, j.cy + y1, &bx, &by);
    const int sx0 = min(ax, bx), sy0 = min(ay, by);
    const int sw = abs(bx - ax) + 1, sh = abs(by - ay) + 1;
    const uint8_t* s = src + j.src_off + (size_t)(sy0 - j.win_y0) * j.src_stride + (size_t)(sx0 - j.win_x0) * C;
    for (int r = threadIdx.y; r < sh; r += blockDim.y) {
        if ((int)threadIdx.x < sw) {
            const uint8_t* p = s + (size_t)r * j.src_stride + threadIdx.x * C;
            tile[r][threadIdx.x] = C == 1 ? (uint32_t)p[0] : (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16);
        }
    }
    __syncthreads();
    const int x = x0 + (int)threadIdx.x;
    if (x > x1) return;
    for (int y = y0 + (int)threadIdx.y; y <= y1; y += blockDim.y) {
        int sx, sy;
        orient_source_pixel(j.o, w, h, j.cx + x, j.cy + y, &sx, &sy);
        const uint32_t v = tile[sy - sy0][sx - sx0];
        uint8_t* q = dst + j.dst_off + ((size_t)y * j.cw + x) * C;
        q[0] = (uint8_t)v;
        if (C == 3) {
            q[1] = (uint8_t)(v >> 8);
            q[2] = (uint8_t)(v >> 16);
        }
    }
}

int orient_crop_launch(const OrientJob* d_jobs, int n, const uint8_t* src, uint8_t* dst, int w, int h, int channels,
                       int max_cw, int max_ch, cudaStream_t st) {
    if (channels != 1 && channels != 3) return LP_ERR_BAD_ARGUMENT;
    constexpr int kMaxJobsPerLaunch = 65535;  // gridDim.z
    for (int j0 = 0; j0 < n; j0 += kMaxJobsPerLaunch) {
        dim3 grid(ceil_div(max_cw, 32), ceil_div(max_ch, 32), std::min(kMaxJobsPerLaunch, n - j0));
        if (channels == 1)
            orient_crop_kernel<1><<<grid, dim3(32, 8), 0, st>>>(d_jobs + j0, src, dst, w, h);
        else
            orient_crop_kernel<3><<<grid, dim3(32, 8), 0, st>>>(d_jobs + j0, src, dst, w, h);
        g_launches++;
        LP_CUDA_OK(cudaGetLastError());
    }
    return LP_OK;
}

// copyTo with cvtColor channel adaptation: 3->4 (A=255), 4->3 (drop A), 1->3/4 (replicate, A=255).
__global__ void copy_region_kernel(const uint8_t* __restrict__ src, size_t sstep, int sc,
                                   uint8_t* __restrict__ dst, size_t dstep, int dc, int w, int h) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= w || y >= h) return;
    const uint8_t* s = src + (size_t)y * sstep + (size_t)x * sc;
    uint8_t* d = dst + (size_t)y * dstep + (size_t)x * dc;
    if (sc == dc) {
        for (int c = 0; c < dc; c++) d[c] = s[c];
    } else if (sc == 1) {
        d[0] = d[1] = d[2] = s[0];
        if (dc == 4) d[3] = 255;
    } else {
        d[0] = s[0]; d[1] = s[1]; d[2] = s[2];
        if (dc == 4) d[3] = 255;
    }
}

int copy_region_launch(const uint8_t* src, size_t sstep, int sc, uint8_t* dst, size_t dstep, int dc,
                       int w, int h, cudaStream_t st) {
    dim3 grid(ceil_div(w, 128), h);
    copy_region_kernel<<<grid, 128, 0, st>>>(src, sstep, sc, dst, dstep, dc, w, h);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

// "over" compositing exactly as the reference spells it with cv::Mat expressions (pixel_blend.cuh).
__global__ void blend_region_kernel(const uint8_t* __restrict__ src, size_t sstep, int sc,
                                    uint8_t* __restrict__ dst, size_t dstep, int dc, int w, int h) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= w || y >= h) return;
    blend_px(src + (size_t)y * sstep + (size_t)x * sc, sc, dst + (size_t)y * dstep + (size_t)x * dc, dc);
}

int blend_region_launch(const uint8_t* src, size_t sstep, int sc, uint8_t* dst, size_t dstep, int dc,
                        int w, int h, cudaStream_t st) {
    dim3 grid(ceil_div(w, 128), h);
    blend_region_kernel<<<grid, 128, 0, st>>>(src, sstep, sc, dst, dstep, dc, w, h);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

__global__ void fill_kernel(uint8_t* dst, size_t step, int C, int w, int h, uchar4 color) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= w || y >= h) return;
    uint8_t* d = dst + (size_t)y * step + (size_t)x * C;
    const uint8_t v[4] = {color.x, color.y, color.z, color.w};
    for (int c = 0; c < C; c++) d[c] = v[c];
}

int fill_launch(uint8_t* dst, size_t step, int C, int w, int h, int b, int g, int r, int a,
                cudaStream_t st) {
    dim3 grid(ceil_div(w, 128), h);
    fill_kernel<<<grid, 128, 0, st>>>(dst, step, C, w, h, make_uchar4(b, g, r, a));
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

}  // namespace lp

// ------------------------------------------------------------------ slot compaction
// n variable-length byte strings in fixed-size slots (string i = len[i] bytes at src + i*stride) -> one
// contiguous buffer (each string at a 16-byte aligned offset), so a batch's encoded outputs cross PCIe as
// one copy of the bytes actually used instead of n whole slots.  off[i] = start of string i, off[n] = total.
namespace lp {

__global__ void __launch_bounds__(1024) compact_scan_kernel(const uint32_t* len, uint32_t cap, int n, unsigned long long* off) {
    __shared__ unsigned long long warp_sums[32];
    __shared__ unsigned long long carry;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + tid;
        uint32_t l = i < n ? len[i] : 0;
        if (l > cap) l = 0;  // a slot cannot hold more than its capacity: treat as failed (length 0)
        unsigned long long v = ((unsigned long long)l + 15ull) & ~15ull, inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += t;
        }
        if (lane == 31) warp_sums[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            unsigned long long s = warp_sums[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned long long t = __shfl_up_sync(0xffffffffu, s, d);
                if (lane >= d) s += t;
            }
            warp_sums[lane] = s;
        }
        __syncthreads();
        const unsigned long long ex = carry + (wid ? warp_sums[wid - 1] : 0) + inc - v;
        if (i < n) off[i] = ex;
        __syncthreads();
        if (tid == 1023) carry = ex + v;
        __syncthreads();
    }
    if (tid == 0) off[n] = carry;
}

__global__ void compact_copy_kernel(const uint8_t* src, size_t stride, const uint32_t* len, uint32_t cap,
                                    const unsigned long long* off, uint8_t* dst) {
    const int i = blockIdx.x;
    uint32_t l = len[i];
    if (l > cap) l = 0;
    const uint8_t* s = src + (size_t)i * stride;
    uint8_t* d = dst + off[i];
    if ((reinterpret_cast<uintptr_t>(s) & 15) == 0) {
        const uint32_t nv = (l + 15) / 16;  // slots are padded: reading the last vector whole stays inside the slot
        for (uint32_t k = threadIdx.x; k < nv; k += blockDim.x)
            reinterpret_cast<uint4*>(d)[k] = reinterpret_cast<const uint4*>(s)[k];
    } else {
        for (uint32_t k = threadIdx.x; k < l; k += blockDim.x) d[k] = s[k];
    }
}

int compact_launch(const uint8_t* src, size_t stride, const uint32_t* len, uint32_t cap, int n, uint8_t* dst,
                   unsigned long long* off, cudaStream_t st) {
    if (n <= 0) return LP_OK;
    compact_scan_kernel<<<1, 1024, 0, st>>>(len, cap, n, off);
    compact_copy_kernel<<<n, 128, 0, st>>>(src, stride, len, cap, off, dst);
    g_launches += 2;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

// `n` byte ranges copied inside one device buffer (PNG files whose IDAT payload is split over many chunks:
// the zlib stream is gathered on the device instead of on the host)
__global__ void seg_copy_kernel(const SegCopy* segs, uint8_t* base) {
    const SegCopy sg = segs[blockIdx.x];
    const uint8_t* s = base + sg.src;
    uint8_t* d = base + sg.dst;
    for (uint32_t k = threadIdx.x; k < sg.len; k += blockDim.x) d[k] = s[k];
}
int seg_copy_launch(const SegCopy* d_segs, int n, uint8_t* base, cudaStream_t st) {
    if (n <= 0) return LP_OK;
    seg_copy_kernel<<<n, 256, 0, st>>>(d_segs, base);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

}  // namespace lp
