// The TuSimple loader's device cache (lanedetection_end2end_b200/Dataloader/Load_Data_new.py; replaces the per-sample
// work of BP/Dataloader/Load_Data_new.py:110-197 after decoding).
//
// lf_loader_stage: decoded frames / label maps of a batch -> crop + resize into slot-addressed uint8 buffers, UNFLIPPED
//   (the reference flips after the resize, so a resized sample is the same every epoch and can be cached).  One thread =
//   one output pixel: Pillow's BILINEAR on the frame (resample.cuh, the arithmetic of frame_preprocess_kernel) and Pillow's
//   NEAREST on the map (the tables of label_preprocess_kernel).
// lf_loader_assemble: the collated batch from the slots and per-sample (slot, table row, flip): image = u8 / 255 (ToTensor,
//   flipped after the resize), gt = the class rules and flip quirk of label_preprocess_kernel on the cached map, and the
//   label elements gathered from per-row tables the host built once in float64 (both flip states).  One thread = one
//   output pixel; the first threads also write the label elements.
// lf_loader_label_rows / lf_loader_assemble_bev: the same cache for the bird's-eye-view loader (bev/Dataloader/
//   Load_Data_new.py; BEV/Dataloader/Load_Data_new.py:62-117): the first labelled row of each newly staged map, recorded
//   once, and the BEV batch (3 / 4 zeroed, 1 <-> 2 on a flip, curve parameters and line classes from tables, horizon from
//   the recorded row).
#include <climits>

#include "resample.cuh"

namespace lf {

__global__ void __launch_bounds__(256) loader_stage_kernel(const uint8_t* __restrict__ frames, const uint8_t* __restrict__ maps, int N,
                                                           int Hin, int Win, int y0, const int* __restrict__ xb,
                                                           const int* __restrict__ xk, int kx, const int* __restrict__ yb,
                                                           const int* __restrict__ yk, int ky, const int* __restrict__ xs,
                                                           const int* __restrict__ ys, int Ho, int Wo, const int* __restrict__ slots,
                                                           uint8_t* __restrict__ cache_frames, uint8_t* __restrict__ cache_maps) {
    pdl_entry();
    const long long total = (long long)N * Ho * Wo;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(idx % Wo);
        const int oy = (int)((idx / Wo) % Ho);
        const int n = (int)(idx / ((long long)Wo * Ho));
        const size_t dst = ((size_t)__ldg(slots + n) * Ho + oy) * Wo + ox;
        int c0, c1, c2;
        ip_bilinear_rgb(frames + ((size_t)n * Hin + y0) * Win * 3, Win, xb, xk, kx, yb, yk, ky, ox, oy, c0, c1, c2);
        uint8_t* f = cache_frames + dst * 3;
        f[0] = (uint8_t)c0;
        f[1] = (uint8_t)c1;
        f[2] = (uint8_t)c2;
        if (maps) cache_maps[dst] = maps[((size_t)n * Hin + y0 + __ldg(ys + oy)) * Win + __ldg(xs + ox)];
    }
}

// ToTensor of one cached RGB pixel `p` into the three planes of the output pixel `o`: u8 / 255 with the division rounded
// as torch rounds it.  The caller picks the mirrored source pixel (the flip comes after the resize).  Shared by both
// assembly kernels so their images stay bit-identical.
__device__ __forceinline__ void loader_image_pixel(const uint8_t* __restrict__ p, float* __restrict__ o, size_t plane) {
    o[0] = __fdiv_rn((float)p[0], 255.f);
    o[plane] = __fdiv_rn((float)p[1], 255.f);
    o[2 * plane] = __fdiv_rn((float)p[2], 255.f);
}

__global__ void __launch_bounds__(256) loader_assemble_kernel(const uint8_t* __restrict__ cache_frames, const uint8_t* __restrict__ cache_maps,
                                                              int N, int Ho, int Wo, int nclasses, const int* __restrict__ sample,
                                                              int nrows, const double* __restrict__ lanes_tab,
                                                              const double* __restrict__ valid_tab, const int* __restrict__ horizon_tab,
                                                              const float* __restrict__ line_tab, float* __restrict__ image,
                                                              long long* __restrict__ gt, double* __restrict__ lanes,
                                                              double* __restrict__ valid, float* __restrict__ horizon,
                                                              float* __restrict__ line) {
    pdl_entry();
    constexpr int LP = LF_LOADER_LANES * LF_LOADER_POINTS;
    const long long total = (long long)N * Ho * Wo;
    const size_t plane = (size_t)Ho * Wo;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(idx % Wo);
        const int oy = (int)((idx / Wo) % Ho);
        const int n = (int)(idx / ((long long)Wo * Ho));
        const int slot = __ldg(sample + 3 * n), fl = __ldg(sample + 3 * n + 2) != 0;
        const size_t src = (size_t)slot * plane + (size_t)oy * Wo;
        const int sx = fl ? Wo - 1 - ox : ox;                        // F.hflip / np.flip after the resize
        if (image) loader_image_pixel(cache_frames + (src + sx) * 3, image + (size_t)n * 3 * plane + (size_t)oy * Wo + ox, plane);
        if (gt) gt[idx] = ip_label_rules(cache_maps[src + sx], cache_maps[src + ox], fl, nclasses);
        // label elements: idx < N * LP (lanes, valid points), < N * Ho (horizon), < N * lanes (line types); N * Ho * Wo
        // covers them all (Wo >= 2, Ho * Wo >= LP)
        if (idx < (long long)N * LP) {
            const int m = (int)(idx / LP), e = (int)(idx % LP);
            const int row = __ldg(sample + 3 * m + 1), f = __ldg(sample + 3 * m + 2) != 0;
            if (lanes) lanes[idx] = __ldg(lanes_tab + ((size_t)f * nrows + row) * LP + e);
            if (valid) valid[idx] = __ldg(valid_tab + (size_t)row * LP + e);
        }
        if (horizon && idx < (long long)N * Ho) {
            const int m = (int)(idx / Ho), y = (int)(idx % Ho);
            horizon[idx] = y < __ldg(horizon_tab + __ldg(sample + 3 * m + 1)) ? 1.f : 0.f;
        }
        if (line && idx < (long long)N * LF_LOADER_LANES) {
            const int m = (int)(idx / LF_LOADER_LANES), e = (int)(idx % LF_LOADER_LANES);
            const int row = __ldg(sample + 3 * m + 1), f = __ldg(sample + 3 * m + 2) != 0;
            line[idx] = __ldg(line_tab + ((size_t)f * nrows + row) * LF_LOADER_LANES + e);
        }
    }
}

// One CTA per staged label map: the first row holding a value outside {0, 3, 4}, or -1.  The bird's-eye-view loader zeroes
// classes 3 and 4 and takes its horizon from the first labelled row; a flip does not move rows, so one value serves both
// flip states.  The CTA scans 8 rows at a time and stops after the first group that holds a hit.
__global__ void __launch_bounds__(256) loader_label_rows_kernel(const uint8_t* __restrict__ cache_maps, int Ho, int Wo,
                                                                const int* __restrict__ slots, const int* __restrict__ positions,
                                                                int* __restrict__ first_row) {
    pdl_entry();
    __shared__ int found;
    if (threadIdx.x == 0) found = INT_MAX;
    __syncthreads();
    const uint8_t* m = cache_maps + (size_t)__ldg(slots + blockIdx.x) * Ho * Wo;
    for (int y0 = 0; y0 < Ho; y0 += 8) {
        const int end = (y0 + 8 < Ho ? y0 + 8 : Ho) * Wo;
        int mine = INT_MAX;
        for (int i = y0 * Wo + threadIdx.x; i < end; i += blockDim.x) {   // ascending: the first hit is this thread's lowest row
            const int v = m[i];
            if (v != 0 && v != 3 && v != 4) {
                mine = i / Wo;
                break;
            }
        }
        if (mine != INT_MAX) atomicMin(&found, mine);
        if (__syncthreads_or(mine != INT_MAX)) break;
    }
    if (threadIdx.x == 0) first_row[__ldg(positions + blockIdx.x)] = found == INT_MAX ? -1 : found;
}

// The bird's-eye-view batch: image as loader_assemble_kernel; gt = the cached map with 3 / 4 -> 0, mirrored with 1 <-> 2 on a
// flip; params / line gathered from per-row tables of both flip states; horizon = y < first_row[row].  One thread = one output
// pixel; the first threads also write the label elements.
__global__ void __launch_bounds__(256) loader_assemble_bev_kernel(const uint8_t* __restrict__ cache_frames,
                                                                  const uint8_t* __restrict__ cache_maps, int N, int Ho, int Wo,
                                                                  const int* __restrict__ sample, int nrows,
                                                                  const float* __restrict__ params_tab,
                                                                  const long long* __restrict__ line_tab,
                                                                  const int* __restrict__ first_row, float* __restrict__ image,
                                                                  long long* __restrict__ gt, float* __restrict__ params,
                                                                  long long* __restrict__ line, float* __restrict__ horizon) {
    pdl_entry();
    constexpr int LC = LF_LOADER_LANES * LF_LOADER_BEV_COEFFS;
    const long long total = (long long)N * Ho * Wo;
    const size_t plane = (size_t)Ho * Wo;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int ox = (int)(idx % Wo);
        const int oy = (int)((idx / Wo) % Ho);
        const int n = (int)(idx / ((long long)Wo * Ho));
        const int slot = __ldg(sample + 3 * n), fl = __ldg(sample + 3 * n + 2) != 0;
        const size_t src = (size_t)slot * plane + (size_t)oy * Wo;
        const int sx = fl ? Wo - 1 - ox : ox;
        loader_image_pixel(cache_frames + (src + sx) * 3, image + (size_t)n * 3 * plane + (size_t)oy * Wo + ox, plane);
        int v = cache_maps[src + sx];
        if (v == 3 || v == 4) v = 0;
        if (fl) v = v == 1 ? 2 : (v == 2 ? 1 : v);
        gt[idx] = v;
        // label elements: idx < N * 12 (params), < N * Ho (horizon), < N * 4 (line); N * Ho * Wo covers them all (Ho * Wo >= 12)
        if (idx < (long long)N * LC) {
            const int m = (int)(idx / LC), e = (int)(idx % LC);
            const int row = __ldg(sample + 3 * m + 1), f = __ldg(sample + 3 * m + 2) != 0;
            params[idx] = __ldg(params_tab + ((size_t)f * nrows + row) * LC + e);
        }
        if (idx < (long long)N * Ho) {
            const int m = (int)(idx / Ho), y = (int)(idx % Ho);
            horizon[idx] = y < __ldg(first_row + __ldg(sample + 3 * m + 1)) ? 1.f : 0.f;
        }
        if (idx < (long long)N * LF_LOADER_LANES) {
            const int m = (int)(idx / LF_LOADER_LANES), e = (int)(idx % LF_LOADER_LANES);
            const int row = __ldg(sample + 3 * m + 1), f = __ldg(sample + 3 * m + 2) != 0;
            line[idx] = __ldg(line_tab + ((size_t)f * nrows + row) * LF_LOADER_LANES + e);
        }
    }
}

inline int loader_grid(long long total) {
    const long long cap = (long long)device_sms() * 16;
    return (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
}

}  // namespace lf

using namespace lf;

extern "C" int lf_loader_stage(const unsigned char* frames, const unsigned char* maps, int N, int Hin, int Win, int crop_y0, int crop_rows,
                               const int* xb, const int* xk, int kx, const int* yb, const int* yk, int ky, const int* xs, const int* ys,
                               int Ho, int Wo, const int* slots, unsigned char* cache_frames, unsigned char* cache_maps,
                               lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(frames && xb && xk && yb && yk && slots && cache_frames && N >= 1 && Ho >= 1 && Wo >= 2 && kx >= 1 && ky >= 1);
    LF_REQUIRE(crop_y0 >= 0 && crop_rows >= 1 && crop_y0 + crop_rows <= Hin && Win >= 1);
    LF_REQUIRE(!maps || (xs && ys && cache_maps));
    lf_launch(loader_stage_kernel, loader_grid((long long)N * Ho * Wo), 256, 0, stream, (const uint8_t*)frames, (const uint8_t*)maps, N,
              Hin, Win, crop_y0, xb, xk, kx, yb, yk, ky, xs, ys, Ho, Wo, slots, (uint8_t*)cache_frames, (uint8_t*)cache_maps);
    return check_launch();
}

extern "C" int lf_loader_assemble(const unsigned char* cache_frames, const unsigned char* cache_maps, int N, int Ho, int Wo, int nclasses,
                                  const int* sample, int nrows, const double* lanes_tab, const double* valid_tab, const int* horizon_tab,
                                  const float* line_tab, float* image, long long* gt, double* lanes, double* valid, float* horizon,
                                  float* line, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(sample && N >= 1 && Ho >= 1 && Wo >= 2 && nrows >= 0 && (long long)Ho * Wo >= LF_LOADER_LANES * LF_LOADER_POINTS);
    LF_REQUIRE((!image || cache_frames) && (!gt || cache_maps) && (!lanes || lanes_tab) && (!valid || valid_tab));
    LF_REQUIRE((!horizon || horizon_tab) && (!line || line_tab));
    LF_REQUIRE(!(lanes || valid || horizon || line) || nrows >= 1);
    lf_launch(loader_assemble_kernel, loader_grid((long long)N * Ho * Wo), 256, 0, stream, (const uint8_t*)cache_frames,
              (const uint8_t*)cache_maps, N, Ho, Wo, nclasses, sample, nrows, lanes_tab, valid_tab, horizon_tab, line_tab, image, gt,
              lanes, valid, horizon, line);
    return check_launch();
}

extern "C" int lf_loader_label_rows(const unsigned char* cache_maps, int N, int Ho, int Wo, const int* slots, const int* positions,
                                    int* first_row, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(cache_maps && slots && positions && first_row && N >= 1 && Ho >= 1 && Wo >= 1);
    lf_launch(loader_label_rows_kernel, N, 256, 0, stream, (const uint8_t*)cache_maps, Ho, Wo, slots, positions, first_row);
    return check_launch();
}

extern "C" int lf_loader_assemble_bev(const unsigned char* cache_frames, const unsigned char* cache_maps, int N, int Ho, int Wo,
                                      const int* sample, int nrows, const float* params_tab, const long long* line_tab,
                                      const int* first_row, float* image, long long* gt, float* params, long long* line, float* horizon,
                                      lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(cache_frames && cache_maps && sample && params_tab && line_tab && first_row && image && gt && params && line && horizon);
    LF_REQUIRE(N >= 1 && Ho >= 1 && Wo >= 2 && nrows >= 1 && (long long)Ho * Wo >= LF_LOADER_LANES * LF_LOADER_BEV_COEFFS);
    lf_launch(loader_assemble_bev_kernel, loader_grid((long long)N * Ho * Wo), 256, 0, stream, (const uint8_t*)cache_frames,
              (const uint8_t*)cache_maps, N, Ho, Wo, sample, nrows, params_tab, line_tab, first_row, image, gt, params, line, horizon);
    return check_launch();
}
