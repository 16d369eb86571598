// frames_pack.cu -- resized u8 frames into a caller's device tensor (lp_xbatch_decode_frames).
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

template <int DT>
struct PackElem;
template <>
struct PackElem<LP_DTYPE_U8> {
    using T = uint8_t;
    static __device__ T from(int v, float, float) { return (uint8_t)v; }
};
template <>
struct PackElem<LP_DTYPE_F16> {
    using T = __half;
    static __device__ T from(int v, float s, float b) { return __float2half_rn(fmaf((float)v, s, b)); }
};
template <>
struct PackElem<LP_DTYPE_BF16> {
    using T = __nv_bfloat16;
    static __device__ T from(int v, float s, float b) { return __float2bfloat16_rn(fmaf((float)v, s, b)); }
};
template <>
struct PackElem<LP_DTYPE_F32> {
    using T = float;
    static __device__ T from(int v, float s, float b) { return fmaf((float)v, s, b); }
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
