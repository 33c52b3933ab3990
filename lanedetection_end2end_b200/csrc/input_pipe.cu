// GPU side of the loader's image path (SURVEY.md 8f-3; BP/Dataloader/Load_Data_new.py:127-131,166-167,178-181):
// decoded RGB frame (uint8 HWC) -> crop the bottom rows -> PIL-BILINEAR resize to (R, 2R) -> optional horizontal
// flip -> ToTensor().float() (uint8 / 255), written in the layout the network consumes.
//
// The resize is Pillow's ImagingResample (src/libImaging/Resample.c; Pillow is a dependency of the reference, not part
// of it): a separable triangle filter widened by the down-scale factor, evaluated in FIXED POINT -- integer coefficients
// (22 fractional bits), accumulator 2^21 + sum(pixel * coeff), clip8(acc >> 22), horizontal pass first with an 8-bit
// intermediate, then the vertical pass.  The coefficient tables depend on the sizes only and are built once on the host
// (input_pipeline.py, float64 like Pillow); the kernel does the integer arithmetic (resample.cuh, shared with the loader's
// staging kernel in loader.cu), so the result is bit-identical to
// PIL's (tests: tests/test_input_pipeline_*.py).  One thread = one output pixel (3 channels); the horizontal value of a
// source row is recomputed by the ~2.5 output rows that use it (integer MACs on L1/L2-resident bytes; the kernel reads
// each frame byte from HBM once: 2.4 MB per 1280x640 crop).
#include "resample.cuh"

namespace lf {

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
        int c0, c1, c2;
        ip_bilinear_rgb(frames + ((size_t)n * Hin + y0) * Win * 3, Win, xb, xk, kx, yb, yk, ky, sx, oy, c0, c1, c2);
        const float r = __fdiv_rn((float)c0, 255.f), g = __fdiv_rn((float)c1, 255.f), b = __fdiv_rn((float)c2, 255.f);
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

// Label map of the loader (Load_Data_new.py:129,131,160-184): crop + Pillow NEAREST resize through the index tables,
// nclasses < 3 zeroes 3 and 4, a flip mirrors and swaps 1 <-> 2, and then -- the reference's masks being taken before the
// flip -- every pixel whose UNFLIPPED value was 3 / 4 becomes 4 / 3.  One thread = one output pixel.
__global__ void __launch_bounds__(256) label_preprocess_kernel(const uint8_t* __restrict__ maps, int N, int Hin, int Win, int y0,
                                                               const int* __restrict__ xs, const int* __restrict__ ys, int Ho,
                                                               int Wo, int nclasses, const uint8_t* __restrict__ flip,
                                                               long long* __restrict__ out) {
    pdl_entry();
    const long long total = (long long)N * Ho * Wo;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(idx % Wo);
        const int oy = (int)((idx / Wo) % Ho);
        const int n = (int)(idx / ((long long)Wo * Ho));
        const uint8_t* row = maps + ((size_t)n * Hin + y0 + __ldg(ys + oy)) * Win;
        const int v0 = row[__ldg(xs + ox)];
        const bool fl = flip && flip[n];
        const int v = fl ? row[__ldg(xs + Wo - 1 - ox)] : v0;
        out[idx] = ip_label_rules(v, v0, fl, nclasses);
    }
}

}  // namespace lf

using namespace lf;

extern "C" int lf_label_preprocess(const unsigned char* maps, int N, int Hin, int Win, int crop_y0, const int* xs, const int* ys, int Ho,
                                   int Wo, int nclasses, const unsigned char* flip, long long* out, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(maps && xs && ys && out && N >= 1 && Hin >= 1 && Win >= 1 && Ho >= 1 && Wo >= 1 && crop_y0 >= 0 && crop_y0 < Hin);
    const long long total = (long long)N * Ho * Wo;
    const long long cap = (long long)device_sms() * 16;
    const int grid = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
    lf_launch(label_preprocess_kernel, grid, 256, 0, stream, (const uint8_t*)maps, N, Hin, Win, crop_y0, xs, ys, Ho, Wo, nclasses,
              (const uint8_t*)flip, out);
    return check_launch();
}

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
