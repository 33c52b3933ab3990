// Pillow's fixed-point BILINEAR resample of one output pixel (src/libImaging/Resample.c ImagingResample): shared by
// frame_preprocess_kernel (input_pipe.cu) and the loader's staging kernel (loader.cu), so the two stay bit-identical.
// Integer coefficients with IP_BITS fractional bits, accumulator 2^(IP_BITS-1) + sum(pixel * coeff), clip8(acc >> IP_BITS),
// horizontal pass first with an 8-bit intermediate, then the vertical pass.  Tables: input_pipeline.resample_tables.
#pragma once
#include "lf_common.cuh"

namespace lf {

constexpr int IP_BITS = 22;

__device__ __forceinline__ int ip_clip8(int acc) {
    const int v = acc >> IP_BITS;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// Output pixel (sx, oy) of one RGB frame: `img` points at the first cropped row (uint8 [rows][Win][3]).  Returns the three
// 8-bit channel values.
__device__ __forceinline__ void ip_bilinear_rgb(const uint8_t* __restrict__ img, int Win, const int* __restrict__ xb,
                                                const int* __restrict__ xk, int kx, const int* __restrict__ yb,
                                                const int* __restrict__ yk, int ky, int sx, int oy, int& c0, int& c1, int& c2) {
    const int xmin = __ldg(xb + 2 * sx), nx = __ldg(xb + 2 * sx + 1);
    const int ymin = __ldg(yb + 2 * oy), ny = __ldg(yb + 2 * oy + 1);
    int av0 = 1 << (IP_BITS - 1), av1 = av0, av2 = av0;
    for (int j = 0; j < ny; ++j) {
        const uint8_t* row = img + ((size_t)(ymin + j) * Win + xmin) * 3;
        int a0 = 1 << (IP_BITS - 1), a1 = a0, a2 = a0;
        for (int i = 0; i < nx; ++i) {
            const int k = __ldg(xk + sx * kx + i);
            a0 += (int)row[3 * i] * k;
            a1 += (int)row[3 * i + 1] * k;
            a2 += (int)row[3 * i + 2] * k;
        }
        const int kyv = __ldg(yk + oy * ky + j);
        av0 += ip_clip8(a0) * kyv;
        av1 += ip_clip8(a1) * kyv;
        av2 += ip_clip8(a2) * kyv;
    }
    c0 = ip_clip8(av0);
    c1 = ip_clip8(av1);
    c2 = ip_clip8(av2);
}

// The loader's label-map class rules (Load_Data_new.py:160-175) on one output pixel: `v` is the map value at the output
// position (mirrored when `fl`), `v0` the unflipped value at the same position.  nclasses < 3 turns 3 and 4 into 0; a flip
// swaps 1 <-> 2 and then -- the reference's masks being taken before the flip -- every pixel whose UNFLIPPED value was
// 3 / 4 becomes 4 / 3.
__device__ __forceinline__ int ip_label_rules(int v, int v0, bool fl, int nclasses) {
    if (nclasses < 3 && (v == 3 || v == 4)) v = 0;
    if (fl) {
        v = v == 1 ? 2 : (v == 2 ? 1 : v);
        v = v0 == 3 ? 4 : (v0 == 4 ? 3 : v);
    }
    return v;
}

}  // namespace lf
