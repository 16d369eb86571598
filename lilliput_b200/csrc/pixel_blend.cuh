// pixel_blend.cuh -- the per-pixel "over" blend of opencv_copy_to_region_with_alpha (ref opencv.cpp:556-667), shared by
// blend_region_kernel (pixel_ops.cu) and the WebP frame compositor (webp_decode.cu) so both give the same bytes.
// fp32 with every OpenCV Mat expression rounded on its own (explicit __f*_rn intrinsics: no FMA contraction), RNE to u8.
#pragma once
#include <cstdint>

namespace lp {

__device__ __forceinline__ uint8_t sat_rne(float f) {
    if (f != f) return 0;  // 0/0 -> NaN -> cvtss2si gives INT_MIN -> saturates to 0
    const int v = __float2int_rn(f);
    return (uint8_t)min(max(v, 0), 255);
}

// s: source pixel of sc channels (1, 3 or 4); d: destination pixel of dc channels (3 or 4), blended in place.
__device__ __forceinline__ void blend_px(const uint8_t* s, int sc, uint8_t* d, int dc) {
    const float k = (float)(1.0 / 255.0);
    const int g = sc == 1;  // grayscale source is expanded to BGR first
    const float sa = __fmul_rn((float)(sc == 4 ? s[3] : 255), k);
    const float da = __fmul_rn((float)(dc == 4 ? d[3] : 255), k);
    const float oma = __fsub_rn(1.0f, sa);
    const float oa = __fadd_rn(sa, __fmul_rn(da, oma));
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float scf = __fmul_rn((float)s[g ? 0 : c], k), dcf = __fmul_rn((float)d[c], k);
        const float num = __fadd_rn(__fmul_rn(scf, sa), __fmul_rn(__fmul_rn(dcf, da), oma));
        d[c] = sat_rne(__fmul_rn(__fdiv_rn(num, oa), 255.0f));
    }
    if (dc == 4) d[3] = sat_rne(__fmul_rn(oa, 255.0f));
}

}  // namespace lp
