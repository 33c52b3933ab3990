// Segmentation-pretraining branch of the reference (`--end_to_end False`; SURVEY.md 8f-4):
//  * lf_seg_lane_maps  -- BP/Networks/LSQ_layer.py:279-293,301: argmax over the L+1 class planes of the decoder output,
//    one map per lane holding the label value where that lane wins (left = label * (label == 1), ...), top rows zeroed;
//    the maps then go through the same LSQ kernel as the end-to-end path (no gradient on this branch).
//    lf_seg_lane_maps_line adds the gt_line substitution of :308-311 in the same launch, so it needs no host read of gt_line.
//  * lf_ce2d_*         -- the weighted pixel-wise nn.CrossEntropyLoss(weights) of BP/Loss_crit.py:64-65 on the planar
//    [B, C, H, W] logits (BP/main.py:258,307): loss = sum_i w[t_i] (lse_i - x_{t_i}) / sum_i w[t_i], and its gradient
//    w[t_i] (softmax_c - [c == t_i]) / sum w, recomputed from the logits (nothing saved but the two sums).
// Bound: HBM -- each kernel reads the C planes once (the gradient kernel also writes them); fp32 per pixel, fp64 across
// pixels, deterministic two-stage sums.
#include "lf_common.cuh"

namespace lf {

constexpr int SEG_MAXC = 8;
constexpr int SEG_THREADS = 256;

__device__ __forceinline__ int seg_argmax(const float* __restrict__ o, int C, long long HW) {
    float best = o[0];
    int arg = 0;
    for (int c = 1; c < C; ++c) {
        const float v = o[(size_t)c * HW];
        if (v > best) {   // first maximum wins
            best = v;
            arg = c;
        }
    }
    return arg;
}

// gt_line (NULL or [B][nl]): where gt_line[b][k] != 0, map (b, k) is image 0 / lane 0's map instead (LSQ_layer.py:308-311).
// The replacement is read from the logits, not from `maps`, so it is the map before any replacement, as the reference's
// right-hand side masked[0, 0] is evaluated before its boolean assignment.
__global__ void __launch_bounds__(SEG_THREADS) seg_lane_maps_kernel(const float* __restrict__ out, int B, int C, long long HW, int W,
                                                                    int nl, int mask_rows, const float* __restrict__ gt_line,
                                                                    float* __restrict__ maps) {
    pdl_entry();
    const long long total = (long long)B * HW;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / HW, p = i - b * HW;
        const int arg = seg_argmax(out + (size_t)b * C * HW + p, C, HW);
        const bool masked = (int)(p / W) < mask_rows;
        int arg0 = -1;    // image 0's winner at p, computed once if a lane of image b is replaced
        for (int k = 0; k < nl; ++k) {
            float v = (!masked && arg == k + 1) ? (float)(k + 1) : 0.f;
            if (gt_line && gt_line[b * nl + k] != 0.f) {
                if (arg0 < 0) arg0 = seg_argmax(out + p, C, HW);
                v = (!masked && arg0 == 1) ? 1.f : 0.f;
            }
            maps[((size_t)b * nl + k) * HW + p] = v;
        }
    }
}

template <bool GRAD>
__global__ void __launch_bounds__(SEG_THREADS) ce2d_kernel(const float* __restrict__ x, const long long* __restrict__ target,
                                                           const float* __restrict__ weight, int B, int C, long long HW,
                                                           double* __restrict__ partial, const double* __restrict__ sums,
                                                           const double* __restrict__ gout, float* __restrict__ dx) {
    pdl_entry();
    __shared__ double red[2][SEG_THREADS / 32];
    double num = 0.0, den = 0.0;
    float gscale = 0.f;
    if (GRAD) gscale = (float)((gout ? gout[0] : 1.0) / sums[1]);
    const long long total = (long long)B * HW;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / HW, p = i - b * HW;
        const float* xi = x + (size_t)b * C * HW + p;
        float v[SEG_MAXC];
        float m = -INFINITY;
#pragma unroll
        for (int c = 0; c < SEG_MAXC; ++c)
            if (c < C) {
                v[c] = xi[(size_t)c * HW];
                m = fmaxf(m, v[c]);
            }
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < SEG_MAXC; ++c)
            if (c < C) s += expf(v[c] - m);
        const long long tl = target[i];
        const bool counted = tl >= 0 && tl < C;          // anything else (e.g. torch's ignore_index = -100) contributes nothing
        const int t = counted ? (int)tl : 0;
        const float w = counted ? (weight ? __ldg(weight + t) : 1.f) : 0.f;
        if (!GRAD) {
            float xt = 0.f;
#pragma unroll
            for (int c = 0; c < SEG_MAXC; ++c)
                if (c == t) xt = v[c];
            num += (double)(w * ((m + logf(s)) - xt));
            den += (double)w;
        } else {
            const float inv = 1.f / s;
            float* di = dx + (size_t)b * C * HW + p;
#pragma unroll
            for (int c = 0; c < SEG_MAXC; ++c)
                if (c < C) di[(size_t)c * HW] = gscale * w * (expf(v[c] - m) * inv - ((counted && c == t) ? 1.f : 0.f));
        }
    }
    if (!GRAD) {
        num = warp_sum(num);
        den = warp_sum(den);
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        if (lane == 0) {
            red[0][warp] = num;
            red[1][warp] = den;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            double a = 0.0, d = 0.0;
            for (int k = 0; k < SEG_THREADS / 32; ++k) {
                a += red[0][k];
                d += red[1][k];
            }
            partial[2 * blockIdx.x] = a;
            partial[2 * blockIdx.x + 1] = d;
        }
    }
}

__global__ void ce2d_finalize_kernel(const double* __restrict__ partial, int nblk, double* __restrict__ sums, double* __restrict__ loss) {
    pdl_entry();
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double a = 0.0, d = 0.0;
        for (int k = 0; k < nblk; ++k) {
            a += partial[2 * k];
            d += partial[2 * k + 1];
        }
        sums[0] = a;
        sums[1] = d;
        loss[0] = a / d;
    }
}

// Confusion counts of the proxy segmentation branch (validation metrics): counts[t * C + pred] += 1 for every pixel whose
// target t is in [0, C); pred is seg_argmax's winner.  Each CTA counts into a shared-memory histogram (lanes of a warp
// that hit the same bin add once, through their leader), then adds each nonzero bin to `counts` with one 64-bit integer
// atomic: the result is exact and independent of the order.  A nonzero *status (the LSQ status word of the batch)
// makes the launch count nothing.  The loop's trip count is uniform over the CTA, so every lane reaches __match_any_sync.
__global__ void __launch_bounds__(SEG_THREADS) seg_confusion_kernel(const float* __restrict__ x, const long long* __restrict__ target,
                                                                    int B, int C, long long HW, const int* __restrict__ status,
                                                                    unsigned long long* __restrict__ counts) {
    pdl_entry();
    if (status && *status) return;
    __shared__ unsigned long long hist[SEG_MAXC * SEG_MAXC];
    for (int k = threadIdx.x; k < C * C; k += blockDim.x) hist[k] = 0ull;
    __syncthreads();
    const long long total = (long long)B * HW;
    for (long long base = (long long)blockIdx.x * blockDim.x; base < total; base += (long long)gridDim.x * blockDim.x) {
        const long long i = base + threadIdx.x;
        int bin = -1;
        if (i < total) {
            const long long t = target[i];
            if (t >= 0 && t < C) {
                const long long b = i / HW, p = i - b * HW;
                bin = (int)t * C + seg_argmax(x + (size_t)b * C * HW + p, C, HW);
            }
        }
        const unsigned same = __match_any_sync(0xffffffffu, bin);
        if (bin >= 0 && (threadIdx.x & 31) == __ffs(same) - 1) atomicAdd(&hist[bin], (unsigned long long)__popc(same));
    }
    __syncthreads();
    for (int k = threadIdx.x; k < C * C; k += blockDim.x)
        if (hist[k]) atomicAdd(counts + k, hist[k]);
}

static int seg_blocks(long long total) {
    const long long b = (total + SEG_THREADS - 1) / SEG_THREADS;
    const long long cap = (long long)device_sms() * 8;
    return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

}  // namespace lf

using namespace lf;

extern "C" int lf_seg_lane_maps_line(const float* out, int B, int C, int H, int W, int nl, int mask_rows, const float* gt_line,
                                     float* maps, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(out && maps && B >= 1 && C >= 2 && H >= 1 && W >= 1 && nl >= 1 && nl < C && mask_rows >= 0);
    const long long HW = (long long)H * W;
    lf_launch(seg_lane_maps_kernel, seg_blocks(B * HW), SEG_THREADS, 0, stream, out, B, C, HW, W, nl, mask_rows, gt_line, maps);
    return check_launch();
}

extern "C" int lf_seg_lane_maps(const float* out, int B, int C, int H, int W, int nl, int mask_rows, float* maps, lf_stream_t stream_) {
    return lf_seg_lane_maps_line(out, B, C, H, W, nl, mask_rows, nullptr, maps, stream_);
}

extern "C" int lf_ce2d_blocks(int B, int H, int W) { return seg_blocks((long long)B * H * W); }

// partial: 2 * lf_ce2d_blocks(B,H,W) doubles of scratch; sums: 2 doubles kept for the backward; loss: 1 double
extern "C" int lf_ce2d_fwd(const float* x, const long long* target, const float* weight, int B, int C, int H, int W, double* partial,
                           double* sums, double* loss, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(x && target && partial && sums && loss && B >= 1 && C >= 1 && C <= SEG_MAXC && H >= 1 && W >= 1);
    const long long HW = (long long)H * W;
    const int nblk = seg_blocks(B * HW);
    lf_launch(ce2d_kernel<false>, nblk, SEG_THREADS, 0, stream, x, target, weight, B, C, HW, partial, (const double*)nullptr,
              (const double*)nullptr, (float*)nullptr);
    lf_launch(ce2d_finalize_kernel, 1, 32, 0, stream, (const double*)partial, nblk, sums, loss);
    return check_launch();
}

// dx = gout * d loss / d x  (gout: device scalar, NULL = 1)
extern "C" int lf_ce2d_bwd(const float* x, const long long* target, const float* weight, int B, int C, int H, int W, const double* sums,
                           const double* gout, float* dx, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(x && target && sums && dx && B >= 1 && C >= 1 && C <= SEG_MAXC && H >= 1 && W >= 1);
    const long long HW = (long long)H * W;
    lf_launch(ce2d_kernel<true>, seg_blocks(B * HW), SEG_THREADS, 0, stream, x, target, weight, B, C, HW, (double*)nullptr, sums, gout, dx);
    return check_launch();
}

// counts [C*C] int64, zeroed by the caller and accumulated over launches; status NULL or the batch's status word
extern "C" int lf_seg_confusion(const float* logits, const long long* target, int B, int C, int H, int W, const int* status,
                                long long* counts, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(logits && target && counts && B >= 1 && C >= 2 && C <= SEG_MAXC && H >= 1 && W >= 1);
    const long long HW = (long long)H * W;
    lf_launch(seg_confusion_kernel, seg_blocks(B * HW), SEG_THREADS, 0, stream, logits, target, B, C, HW, status,
              reinterpret_cast<unsigned long long*>(counts));
    return check_launch();
}
