// frames_pack.cu -- resized u8 frames into a caller's device tensor (lp_xbatch_decode_frames), and a caller's tensor
// back into packed u8 frames (lp_xbatch_encode_frames: frames_unpack_kernel, below).
//
// Every frame is packed BGR / BGRA / gray (1, 3 or 4 bytes per pixel, rows `step` apart).  Its slice of the tensor holds
// H x W x C elements (NHWC) or C planes of H x W (NCHW) of one dtype; the frame sits at the slice's top-left and every
// other element of the slice is zero.  Output channel c takes:
//   c == 3            the frame's alpha, or 255 when it has none
//   c < 3, gray       the gray sample (replicated)
//   c < 3, colour     B, G, R in that order, or R, G, B when rgb is set
// Float dtypes store fmaf(sample, scale[c], bias[c]) rounded to nearest; U8 stores the sample.
//
// One thread per 16 bytes of the tensor: the slice is walked in output order, so NHWC and NCHW both write whole 16-byte
// vectors (one st.global.v4 each) and differ only in which source byte each element gathers.  The 16-byte pieces are
// taken in absolute address space, so any element-aligned base works; the (at most two) pieces a slice shares with its
// neighbours or the tensor's ends are written element by element, and only the elements that belong to the slice.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.cuh"

namespace lp {

// The way back (lp_xbatch_encode_frames): fmaf(x, scale, bias) in fp32, rounded half to even and clamped to [0, 255].
// NaN gives 0 (fmaxf returns its number operand), +-inf and out-of-range values the nearer end.
__device__ __forceinline__ uint8_t unpack_u8(float v) { return (uint8_t)__float2uint_rn(fminf(fmaxf(v, 0.f), 255.f)); }

template <int DT>
struct PackElem;
template <>
struct PackElem<LP_DTYPE_U8> {
    using T = uint8_t;
    static __device__ T from(int v, float, float) { return (uint8_t)v; }
    static __device__ uint8_t to(T x, float, float) { return x; }
};
template <>
struct PackElem<LP_DTYPE_F16> {
    using T = __half;
    static __device__ T from(int v, float s, float b) { return __float2half_rn(fmaf((float)v, s, b)); }
    static __device__ uint8_t to(T x, float s, float b) { return unpack_u8(fmaf(__half2float(x), s, b)); }
};
template <>
struct PackElem<LP_DTYPE_BF16> {
    using T = __nv_bfloat16;
    static __device__ T from(int v, float s, float b) { return __float2bfloat16_rn(fmaf((float)v, s, b)); }
    static __device__ uint8_t to(T x, float s, float b) { return unpack_u8(fmaf(__bfloat162float(x), s, b)); }
};
template <>
struct PackElem<LP_DTYPE_F32> {
    using T = float;
    static __device__ T from(int v, float s, float b) { return fmaf((float)v, s, b); }
    static __device__ uint8_t to(T x, float s, float b) { return unpack_u8(fmaf(x, s, b)); }
};

// Position of one element of a slice, advanced in output order
struct PackPos {
    int c, y, x;
};

__device__ __forceinline__ PackPos pack_pos(uint64_t r, const FramePackLayout& t) {
    PackPos p;
    if (t.nchw) {
        const uint64_t plane = (uint64_t)t.H * t.W;
        p.c = (int)(r / plane);
        const uint64_t q = r - (uint64_t)p.c * plane;
        p.y = (int)(q / (uint64_t)t.W);
        p.x = (int)(q - (uint64_t)p.y * t.W);
    } else {
        const uint64_t pix = r / (uint64_t)t.C;
        p.c = (int)(r - pix * t.C);
        p.y = (int)(pix / (uint64_t)t.W);
        p.x = (int)(pix - (uint64_t)p.y * t.W);
    }
    return p;
}

__device__ __forceinline__ void pack_next(PackPos& p, const FramePackLayout& t) {
    if (t.nchw) {
        if (++p.x == t.W) {
            p.x = 0;
            if (++p.y == t.H) {
                p.y = 0;
                p.c++;
            }
        }
    } else if (++p.c == t.C) {
        p.c = 0;
        if (++p.x == t.W) {
            p.x = 0;
            p.y++;
        }
    }
}

template <int DT>
__device__ __forceinline__ typename PackElem<DT>::T pack_value(const FramePackItem& it, const FramePackLayout& t, PackPos p) {
    using E = PackElem<DT>;
    if (p.x >= it.w || p.y >= it.h) return typename E::T(0.f);
    const uint8_t* s = it.src + (size_t)p.y * it.step + (size_t)p.x * it.ch;
    int v;
    if (p.c == 3) v = it.ch == 4 ? s[3] : 255;
    else v = s[it.ch == 1 ? 0 : (t.rgb ? 2 - p.c : p.c)];
    // (selected, not indexed: a kernel parameter indexed at run time is copied to local memory)
    const float sc = p.c == 0 ? t.scale[0] : p.c == 1 ? t.scale[1] : p.c == 2 ? t.scale[2] : t.scale[3];
    const float bi = p.c == 0 ? t.bias[0] : p.c == 1 ? t.bias[1] : p.c == 2 ? t.bias[2] : t.bias[3];
    return E::from(v, sc, bi);
}

// blockIdx.y: the item (items[y], or `one` when items is null); x: 16-byte pieces of its slice
template <int DT>
__global__ void __launch_bounds__(256)
    frames_pack_kernel(const FramePackItem* __restrict__ items, FramePackItem one, FramePackLayout t, uint64_t slice_elems,
                       uint64_t pieces, int off) {
    using T = typename PackElem<DT>::T;
    constexpr int kVec = 16 / (int)sizeof(T);
    const FramePackItem it = items ? items[blockIdx.y] : one;
    T* const base = static_cast<T*>(t.data);
    const uint64_t e0 = (uint64_t)it.slice * slice_elems, e1 = e0 + slice_elems;
    const uint64_t q0 = (e0 + off) / kVec;  // the first piece that touches the slice
    for (uint64_t q = q0 + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; q < q0 + pieces; q += (uint64_t)gridDim.x * blockDim.x) {
        const int64_t first = (int64_t)(q * kVec) - off;  // element index of the piece's first lane
        if (first >= (int64_t)e1) break;
        if (first >= (int64_t)e0 && first + kVec <= (int64_t)e1) {
            PackPos p = pack_pos((uint64_t)first - e0, t);
            union {
                uint4 v;
                T e[kVec];
            } u;
#pragma unroll
            for (int k = 0; k < kVec; k++) {
                u.e[k] = pack_value<DT>(it, t, p);
                pack_next(p, t);
            }
            *reinterpret_cast<uint4*>(base + first) = u.v;
        } else {
            for (int k = 0; k < kVec; k++) {
                const int64_t e = first + k;
                if (e >= (int64_t)e0 && e < (int64_t)e1) base[e] = pack_value<DT>(it, t, pack_pos((uint64_t)e - e0, t));
            }
        }
    }
}

// One byte of a packed frame: output channel p.c (B, G, R, A) of pixel (p.x, p.y), from tensor channel 3 (alpha), or
// 2 - p.c when the tensor is RGB.  plane: H x W, the distance between NCHW channel planes.
template <int DT>
__device__ __forceinline__ uint8_t unpack_value(const typename PackElem<DT>::T* __restrict__ s, const FramePackLayout& t, uint64_t plane,
                                                PackPos p) {
    const int c = p.c == 3 || !t.rgb ? p.c : 2 - p.c;
    const uint64_t e = t.nchw ? (uint64_t)c * plane + (uint64_t)p.y * t.W + p.x : ((uint64_t)p.y * t.W + p.x) * t.C + c;
    // (selected, not indexed, as in pack_value)
    const float sc = c == 0 ? t.scale[0] : c == 1 ? t.scale[1] : c == 2 ? t.scale[2] : t.scale[3];
    const float bi = c == 0 ? t.bias[0] : c == 1 ? t.bias[1] : c == 2 ? t.bias[2] : t.bias[3];
    return PackElem<DT>::to(s[e], sc, bi);
}

// The inverse of frames_pack_kernel.  blockIdx.y: the item (items[y], or `one` when items is null); x: 16-byte pieces of
// its packed frame (w x h x C bytes from it.dst, which is 16-byte aligned), each written with one 128-bit store, the
// frame's last partial piece byte by byte.  The walk runs in output order, so consecutive threads read consecutive
// elements of an NHWC slice and of each plane of an NCHW one.
template <int DT>
__global__ void __launch_bounds__(256)
    frames_unpack_kernel(const FrameUnpackItem* __restrict__ items, FrameUnpackItem one, FramePackLayout t, uint64_t slice_elems) {
    using T = typename PackElem<DT>::T;
    const FrameUnpackItem it = items ? items[blockIdx.y] : one;
    const T* const src = static_cast<const T*>(t.data) + (uint64_t)it.slice * slice_elems;
    FramePackLayout f = t;  // the packed frame: w x h x C, NHWC
    f.H = it.h;
    f.W = it.w;
    f.nchw = 0;
    const uint64_t plane = (uint64_t)t.H * t.W, bytes = (uint64_t)it.w * it.h * t.C;
    for (uint64_t o = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) * 16; o < bytes; o += (uint64_t)gridDim.x * blockDim.x * 16) {
        PackPos p = pack_pos(o, f);
        if (o + 16 <= bytes) {
            union {
                uint4 v;
                uint8_t b[16];
            } u;
#pragma unroll
            for (int k = 0; k < 16; k++) {
                u.b[k] = unpack_value<DT>(src, t, plane, p);
                pack_next(p, f);
            }
            *reinterpret_cast<uint4*>(it.dst + o) = u.v;
        } else {
            for (uint64_t e = o; e < bytes; e++) {
                it.dst[e] = unpack_value<DT>(src, t, plane, p);
                pack_next(p, f);
            }
        }
    }
}

int frames_unpack_launch(const FrameUnpackItem* d_items, const FrameUnpackItem* one, int n, uint64_t max_frame_bytes,
                         const FramePackLayout& t, cudaStream_t st) {
    const size_t es = frames_dtype_bytes(t.dtype);
    if (n < 1 || !es || (!d_items && (!one || n != 1 || (uintptr_t)one->dst % 16)) || (uintptr_t)t.data % es) return LP_ERR_BAD_ARGUMENT;
    if (!max_frame_bytes) return LP_OK;
    const uint64_t slice_elems = (uint64_t)t.H * t.W * t.C;
    const unsigned bx = (unsigned)std::min<uint64_t>(ceil_div<uint64_t>(ceil_div<uint64_t>(max_frame_bytes, 16), 256), 1u << 16);
    const FrameUnpackItem none{};
    for (int i0 = 0; i0 < n; i0 += 65535) {
        const dim3 grid(bx, (unsigned)std::min(n - i0, 65535));
        const FrameUnpackItem* tab = d_items ? d_items + i0 : nullptr;
        const FrameUnpackItem& single = d_items ? none : *one;
        switch (t.dtype) {
            case LP_DTYPE_U8: frames_unpack_kernel<LP_DTYPE_U8><<<grid, 256, 0, st>>>(tab, single, t, slice_elems); break;
            case LP_DTYPE_F16: frames_unpack_kernel<LP_DTYPE_F16><<<grid, 256, 0, st>>>(tab, single, t, slice_elems); break;
            case LP_DTYPE_BF16: frames_unpack_kernel<LP_DTYPE_BF16><<<grid, 256, 0, st>>>(tab, single, t, slice_elems); break;
            default: frames_unpack_kernel<LP_DTYPE_F32><<<grid, 256, 0, st>>>(tab, single, t, slice_elems); break;
        }
        g_launches++;
        LP_CUDA_OK(cudaGetLastError());
    }
    return LP_OK;
}

size_t frames_dtype_bytes(int dtype) {
    switch (dtype) {
        case LP_DTYPE_U8: return 1;
        case LP_DTYPE_F16:
        case LP_DTYPE_BF16: return 2;
        case LP_DTYPE_F32: return 4;
        default: return 0;
    }
}

int frames_pack_launch(const FramePackItem* d_items, const FramePackItem* one, int n, const FramePackLayout& t, cudaStream_t st) {
    const size_t es = frames_dtype_bytes(t.dtype);
    if (n < 1 || !es || (!d_items && (!one || n != 1)) || (uintptr_t)t.data % es) return LP_ERR_BAD_ARGUMENT;
    const uint64_t slice_elems = (uint64_t)t.H * t.W * t.C;
    const int vec = 16 / (int)es, off = (int)(((uintptr_t)t.data % 16) / es);
    const uint64_t pieces = slice_elems / vec + 2;  // (a slice that starts and ends inside a piece spans two more)
    const unsigned bx = (unsigned)std::min<uint64_t>(ceil_div<uint64_t>(pieces, 256), 1u << 16);
    const FramePackItem none{};
    for (int i0 = 0; i0 < n; i0 += 65535) {
        const dim3 grid(bx, (unsigned)std::min(n - i0, 65535));
        const FramePackItem* tab = d_items ? d_items + i0 : nullptr;
        const FramePackItem& single = d_items ? none : *one;
        switch (t.dtype) {
            case LP_DTYPE_U8: frames_pack_kernel<LP_DTYPE_U8><<<grid, 256, 0, st>>>(tab, single, t, slice_elems, pieces, off); break;
            case LP_DTYPE_F16: frames_pack_kernel<LP_DTYPE_F16><<<grid, 256, 0, st>>>(tab, single, t, slice_elems, pieces, off); break;
            case LP_DTYPE_BF16: frames_pack_kernel<LP_DTYPE_BF16><<<grid, 256, 0, st>>>(tab, single, t, slice_elems, pieces, off); break;
            default: frames_pack_kernel<LP_DTYPE_F32><<<grid, 256, 0, st>>>(tab, single, t, slice_elems, pieces, off); break;
        }
        g_launches++;
        LP_CUDA_OK(cudaGetLastError());
    }
    return LP_OK;
}

}  // namespace lp
