// GPU side of the loader's image path (SURVEY.md 8f-3; BP/Dataloader/Load_Data_new.py:127-131,166-167,178-181):
// decoded RGB frame (uint8 HWC) -> crop the bottom rows -> PIL-BILINEAR resize to (R, 2R) -> optional horizontal
// flip -> ToTensor().float() (uint8 / 255), written in the layout the network consumes.
//
// The resize is Pillow's ImagingResample (src/libImaging/Resample.c; Pillow is a dependency of the reference, not part
// of it): a separable triangle filter widened by the down-scale factor, evaluated in FIXED POINT -- integer coefficients
// (22 fractional bits), accumulator 2^21 + sum(pixel * coeff), clip8(acc >> 22), horizontal pass first with an 8-bit
// intermediate, then the vertical pass.  The coefficient tables depend on the sizes only and are built once on the host
// (input_pipeline.py, float64 like Pillow); the kernel does the integer arithmetic, so the result is bit-identical to
// PIL's (tests: tests/test_input_pipeline_*.py).  One thread = one output pixel (3 channels); the horizontal value of a
// source row is recomputed by the ~2.5 output rows that use it (integer MACs on L1/L2-resident bytes; the kernel reads
// each frame byte from HBM once: 2.4 MB per 1280x640 crop).
#include "lf_common.cuh"

namespace lf {

constexpr int IP_BITS = 22;

__device__ __forceinline__ int ip_clip8(int acc) {
    const int v = acc >> IP_BITS;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

__global__ void __launch_bounds__(256) frame_preprocess_kernel(const uint8_t* __restrict__ frames, int N, int Hin, int Win, int y0,
                                                               const int* __restrict__ xb, const int* __restrict__ xk, int kx,
                                                               const int* __restrict__ yb, const int* __restrict__ yk, int ky,
                                                               int Ho, int Wo, const uint8_t* __restrict__ flip, int layout,
                                                               float* __restrict__ out) {
    pdl_entry();
    const long long total = (long long)N * Ho * Wo;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(idx % Wo);
        const int oy = (int)((idx / Wo) % Ho);
        const int n = (int)(idx / ((long long)Wo * Ho));
        const int sx = (flip && flip[n]) ? Wo - 1 - ox : ox;        // F.hflip of the resized image
        const int xmin = __ldg(xb + 2 * sx), nx = __ldg(xb + 2 * sx + 1);
        const int ymin = __ldg(yb + 2 * oy), ny = __ldg(yb + 2 * oy + 1);
        int av0 = 1 << (IP_BITS - 1), av1 = av0, av2 = av0;
        for (int j = 0; j < ny; ++j) {
            const uint8_t* row = frames + ((size_t)((size_t)n * Hin + y0 + ymin + j) * Win + xmin) * 3;
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
        const float r = __fdiv_rn((float)ip_clip8(av0), 255.f), g = __fdiv_rn((float)ip_clip8(av1), 255.f),
                    b = __fdiv_rn((float)ip_clip8(av2), 255.f);
        if (layout == 1) {   // NHWC, 3 channels padded to 4 (what the stem convolution reads)
            reinterpret_cast<float4*>(out)[idx] = make_float4(r, g, b, 0.f);
        } else {             // NCHW (what the reference's loader returns)
            const size_t plane = (size_t)Ho * Wo;
            float* o = out + (size_t)n * 3 * plane + (size_t)oy * Wo + ox;
            o[0] = r;
            o[plane] = g;
            o[2 * plane] = b;
        }
    }
}

}  // namespace lf

using namespace lf;

extern "C" int lf_frame_preprocess(const unsigned char* frames, int N, int Hin, int Win, int crop_y0, int crop_rows, const int* xb,
                                   const int* xk, int kx, const int* yb, const int* yk, int ky, int Ho, int Wo,
                                   const unsigned char* flip, int layout, float* out, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(frames && xb && xk && yb && yk && out && N >= 1 && Ho >= 1 && Wo >= 1 && kx >= 1 && ky >= 1);
    LF_REQUIRE(crop_y0 >= 0 && crop_rows >= 1 && crop_y0 + crop_rows <= Hin && (layout == 0 || layout == 1));
    const long long total = (long long)N * Ho * Wo;
    const long long cap = (long long)device_sms() * 16;
    const int grid = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
    lf_launch(frame_preprocess_kernel, grid, 256, 0, stream, (const uint8_t*)frames, N, Hin, Win, crop_y0, xb, xk, kx, yb, yk, ky, Ho, Wo,
              (const uint8_t*)flip, layout, out);
    return check_launch();
}
