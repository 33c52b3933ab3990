// Fully connected layers of the Classification heads (BP/Networks/LSQ_layer.py:188-192,203-206: nn.Linear
// 32768->128 (+ReLU), 128->4 for the line-type head; 2048->256 for the horizon head), forward and both gradients.
//
//     y[b][o] = bias[o] + sum_k x[b][k] * W[o][k]          W in nn.Linear's own [O][K] layout (no repacking)
//
// Bound: HBM, on W.  The 32768->128 layer streams a 16.8 MB weight matrix against a 4 MB activation; at batch 32 that
// is 16 FLOP per weight byte, an order of magnitude under the ridge of any tensor-core formulation, so these are
// fp32 FFMA kernels (fp32-exact, the mode every parity gate accepts) organised around reading W exactly once with
// fully coalesced 128-byte rows:
//   forward       CTA = one K chunk (256 columns): x[:, chunk] staged in shared memory; a warp owns output rows o,
//                 lanes stride the chunk, BT accumulators per lane (one per batch row), warp-shuffle reduction,
//                 per-chunk partials [chunk][b][o]; a finish kernel sums the chunks in fixed order (+bias, ReLU).
//   input grad    CTA = one K chunk, thread = one column k: dx[b][k] = sum_o dy[b][o] W[o][k], dy transposed in
//                 shared memory and read as float4 over the batch (broadcast), W column-coalesced across the CTA.
//   weight grad   CTA = one K chunk, thread = one column k holding x[:, k] in registers:
//                 dW[o][k] = sum_b dy[b][o] x[b][k]; written coalesced, no cross-CTA reduction.  db = column sums of dy.
// Deterministic (no atomics).  Batch rows beyond BT = 64 are processed in further passes over W.
#include "lf_common.cuh"

namespace lf {

constexpr int LIN_KC = 256;        // K columns per CTA
constexpr int LIN_THREADS = 256;

template <int BT>
__global__ void __launch_bounds__(LIN_THREADS) linear_fwd_kernel(const float* __restrict__ x, const float* __restrict__ W,
                                                                 int B, int b0, int K, int O, float* __restrict__ partial) {
    pdl_entry();
    extern __shared__ __align__(16) float xs_raw[];   // [BT][LIN_KC]
    float (*xs)[LIN_KC] = reinterpret_cast<float (*)[LIN_KC]>(xs_raw);
    const int k0 = blockIdx.x * LIN_KC;
    const int kc = min(LIN_KC, K - k0);
    for (int i = threadIdx.x; i < BT * LIN_KC; i += LIN_THREADS) {
        const int b = i / LIN_KC, k = i - b * LIN_KC;
        xs[b][k] = (b0 + b < B && k < kc) ? __ldg(x + (size_t)(b0 + b) * K + k0 + k) : 0.f;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int o = warp; o < O; o += LIN_THREADS / 32) {
        float w[LIN_KC / 32];
#pragma unroll
        for (int j = 0; j < LIN_KC / 32; ++j) {
            const int k = lane + 32 * j;
            w[j] = k < kc ? ld_stream_f1(W + (size_t)o * K + k0 + k) : 0.f;
        }
        float acc[BT];
#pragma unroll
        for (int b = 0; b < BT; ++b) {
            float s = 0.f;
#pragma unroll
            for (int j = 0; j < LIN_KC / 32; ++j) s = fmaf(w[j], xs[b][lane + 32 * j], s);
            acc[b] = s;
        }
        // BT values x 32 lanes -> lane b holds the total of batch row b (+32: second half): transpose-reduce
#pragma unroll
        for (int b = 0; b < BT; ++b) acc[b] = warp_sum(acc[b]);
        if (lane == 0) {
#pragma unroll
            for (int b = 0; b < BT; ++b)
                if (b0 + b < B) partial[((size_t)blockIdx.x * B + b0 + b) * O + o] = acc[b];
        }
    }
}

__global__ void linear_finish_kernel(const float* __restrict__ partial, int nchunks, int B, int O, const float* __restrict__ bias,
                                     int relu, float* __restrict__ y) {
    pdl_entry();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * O) return;
    float s = bias ? __ldg(bias + i % O) : 0.f;
    for (int c = 0; c < nchunks; ++c) s += partial[(size_t)c * B * O + i];
    y[i] = relu ? fmaxf(s, 0.f) : s;
}

// dy [B][O] (optionally gated by relu_out > 0) -> shared memory, transposed [o][BT] and zero padded
template <int BT>
__device__ __forceinline__ void lin_stage_dy(float* dys, const float* __restrict__ dy, const float* __restrict__ relu_out, int B,
                                             int b0, int O) {
    for (int i = threadIdx.x; i < O * BT; i += LIN_THREADS) {
        const int o = i / BT, b = i - o * BT;
        float v = 0.f;
        if (b0 + b < B) {
            v = __ldg(dy + (size_t)(b0 + b) * O + o);
            if (relu_out && !(__ldg(relu_out + (size_t)(b0 + b) * O + o) > 0.f)) v = 0.f;
        }
        dys[i] = v;
    }
}

template <int BT>
__global__ void __launch_bounds__(LIN_THREADS) linear_bwd_data_kernel(const float* __restrict__ dy, const float* __restrict__ relu_out,
                                                                      const float* __restrict__ W, int B, int b0, int K, int O,
                                                                      float* __restrict__ dx) {
    pdl_entry();
    extern __shared__ __align__(16) float dys[];   // [O][BT]
    lin_stage_dy<BT>(dys, dy, relu_out, B, b0, O);
    __syncthreads();
    const int k = blockIdx.x * LIN_KC + threadIdx.x;
    if (k >= K) return;
    float acc[BT];
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[b] = 0.f;
    for (int o = 0; o < O; ++o) {
        const float w = ld_stream_f1(W + (size_t)o * K + k);
        const float4* d4 = reinterpret_cast<const float4*>(dys + o * BT);
#pragma unroll
        for (int q = 0; q < BT / 4; ++q) {
            const float4 d = d4[q];
            acc[4 * q] = fmaf(d.x, w, acc[4 * q]);
            acc[4 * q + 1] = fmaf(d.y, w, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(d.z, w, acc[4 * q + 2]);
            acc[4 * q + 3] = fmaf(d.w, w, acc[4 * q + 3]);
        }
    }
#pragma unroll
    for (int b = 0; b < BT; ++b)
        if (b0 + b < B) dx[(size_t)(b0 + b) * K + k] = acc[b];
}

template <int BT>
__global__ void __launch_bounds__(LIN_THREADS) linear_bwd_weight_kernel(const float* __restrict__ dy, const float* __restrict__ relu_out,
                                                                        const float* __restrict__ x, int B, int b0, int K, int O,
                                                                        int accumulate, float* __restrict__ dW, float* __restrict__ db) {
    pdl_entry();
    extern __shared__ __align__(16) float dys[];   // [O][BT]
    lin_stage_dy<BT>(dys, dy, relu_out, B, b0, O);
    __syncthreads();
    if (db && blockIdx.x == 0) {
        for (int o = threadIdx.x; o < O; o += LIN_THREADS) {
            float s = accumulate ? db[o] : 0.f;
#pragma unroll
            for (int b = 0; b < BT; ++b) s += dys[o * BT + b];
            db[o] = s;
        }
    }
    const int k = blockIdx.x * LIN_KC + threadIdx.x;
    if (k >= K) return;
    float xr[BT];
#pragma unroll
    for (int b = 0; b < BT; ++b) xr[b] = (b0 + b < B) ? __ldg(x + (size_t)(b0 + b) * K + k) : 0.f;
    for (int o = 0; o < O; ++o) {
        const float4* d4 = reinterpret_cast<const float4*>(dys + o * BT);
        float s = accumulate ? dW[(size_t)o * K + k] : 0.f;
#pragma unroll
        for (int q = 0; q < BT / 4; ++q) {
            const float4 d = d4[q];
            s = fmaf(d.x, xr[4 * q], s);
            s = fmaf(d.y, xr[4 * q + 1], s);
            s = fmaf(d.z, xr[4 * q + 2], s);
            s = fmaf(d.w, xr[4 * q + 3], s);
        }
        dW[(size_t)o * K + k] = s;
    }
}

// AvgPool2d((1, W)) of the horizon head (BP/Networks/LSQ_layer.py:184,198) on an NHWC map, written in the order the
// reference's NCHW x.view(B, -1) produces: out[b][c*H + h] = mean_w x[b][h][w][c]; one CTA per (b, h) row.
__global__ void __launch_bounds__(256) rowmean_fwd_kernel(const float* __restrict__ x, int H, int W, int C, float* __restrict__ out) {
    pdl_entry();
    __shared__ float red[256];
    const int bh = blockIdx.x, b = bh / H, h = bh - b * H;
    const float* row = x + (size_t)bh * W * C;
    const int lanes_per_c = 256 / C > 0 ? 256 / C : 1;     // C <= 256
    const int c = threadIdx.x % C, part = threadIdx.x / C;
    float s = 0.f;
    if (part < lanes_per_c)
        for (int w = part; w < W; w += lanes_per_c) s += row[(size_t)w * C + c];
    red[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x < C) {
        float t = 0.f;
        for (int p = 0; p < lanes_per_c; ++p) t += red[p * C + threadIdx.x];
        out[(size_t)b * C * H + (size_t)threadIdx.x * H + h] = t / (float)W;
    }
}
__global__ void __launch_bounds__(256) rowmean_bwd_kernel(const float* __restrict__ dout, int H, int W, int C, long long total,
                                                          float* __restrict__ dx) {
    pdl_entry();
    const float inv = 1.f / (float)W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long long bh = i / ((long long)W * C);
        const int h = (int)(bh % H);
        const long long b = bh / H;
        dx[i] = __ldg(dout + (size_t)b * C * H + (size_t)c * H + h) * inv;
    }
}

static int lin_bt(int B) { return B <= 8 ? 8 : B <= 16 ? 16 : B <= 32 ? 32 : 64; }

}  // namespace lf

using namespace lf;

extern "C" int lf_linear_chunks(int K) { return K > 0 ? (K + LIN_KC - 1) / LIN_KC : 0; }

// partial: [lf_linear_chunks(K)][B][O] floats of caller-owned scratch
extern "C" int lf_linear_fwd(const float* x, const float* W, const float* bias, int B, int K, int O, int relu, float* partial,
                             float* y, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(x && W && partial && y && B >= 1 && K >= 1 && O >= 1);
    const int nch = lf_linear_chunks(K);
    for (int b0 = 0; b0 < B; b0 += 64) {
        const int bt = lin_bt(B - b0);
        const size_t smem = (size_t)bt * LIN_KC * 4;
#define LF_LIN_F(BT_)                                                                                                     \
    do {                                                                                                                  \
        cudaError_t e = cudaFuncSetAttribute(linear_fwd_kernel<BT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024); \
        if (e != cudaSuccess) { set_last_cuda_error(e); return LF_ERR_CUDA; }                                             \
        lf_launch(linear_fwd_kernel<BT_>, nch, LIN_THREADS, smem, stream, x, W, B, b0, K, O, partial);                    \
    } while (0)
        switch (bt) {
            case 8: LF_LIN_F(8); break;
            case 16: LF_LIN_F(16); break;
            case 32: LF_LIN_F(32); break;
            default: LF_LIN_F(64);
        }
#undef LF_LIN_F
    }
    lf_launch(linear_finish_kernel, (B * O + 255) / 256, 256, 0, stream, (const float*)partial, nch, B, O, bias, relu, y);
    return check_launch();
}

// dx[b][k] = sum_o g[b][o] W[o][k],  g = dy (* (relu_out > 0) when relu_out is given: the layer's own ReLU output)
extern "C" int lf_linear_bwd_data(const float* dy, const float* relu_out, const float* W, int B, int K, int O, float* dx,
                                  lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(dy && W && dx && B >= 1 && K >= 1 && O >= 1);
    const int nch = lf_linear_chunks(K);
    for (int b0 = 0; b0 < B; b0 += 64) {
        const int bt = lin_bt(B - b0);
        const size_t smem = (size_t)O * bt * 4;
        LF_REQUIRE(smem <= 96 * 1024);
#define LF_LIN_BD(BT_)                                                                                                      \
    do {                                                                                                                    \
        cudaError_t e = cudaFuncSetAttribute(linear_bwd_data_kernel<BT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024); \
        if (e != cudaSuccess) { set_last_cuda_error(e); return LF_ERR_CUDA; }                                               \
        lf_launch(linear_bwd_data_kernel<BT_>, nch, LIN_THREADS, smem, stream, dy, relu_out, W, B, b0, K, O, dx);           \
    } while (0)
        switch (bt) {
            case 8: LF_LIN_BD(8); break;
            case 16: LF_LIN_BD(16); break;
            case 32: LF_LIN_BD(32); break;
            default: LF_LIN_BD(64);
        }
#undef LF_LIN_BD
    }
    return check_launch();
}

// dW[o][k] = sum_b g[b][o] x[b][k],  db[o] = sum_b g[b][o]
extern "C" int lf_linear_bwd_weight(const float* dy, const float* relu_out, const float* x, int B, int K, int O, float* dW, float* db,
                                    lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(dy && x && dW && B >= 1 && K >= 1 && O >= 1);
    const int nch = lf_linear_chunks(K);
    for (int b0 = 0; b0 < B; b0 += 64) {
        const int bt = lin_bt(B - b0);
        const size_t smem = (size_t)O * bt * 4;
        LF_REQUIRE(smem <= 96 * 1024);
        const int acc = b0 > 0 ? 1 : 0;
#define LF_LIN_BW(BT_)                                                                                                        \
    do {                                                                                                                      \
        cudaError_t e = cudaFuncSetAttribute(linear_bwd_weight_kernel<BT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024); \
        if (e != cudaSuccess) { set_last_cuda_error(e); return LF_ERR_CUDA; }                                                 \
        lf_launch(linear_bwd_weight_kernel<BT_>, nch, LIN_THREADS, smem, stream, dy, relu_out, x, B, b0, K, O, acc, dW, db);  \
    } while (0)
        switch (bt) {
            case 8: LF_LIN_BW(8); break;
            case 16: LF_LIN_BW(16); break;
            case 32: LF_LIN_BW(32); break;
            default: LF_LIN_BW(64);
        }
#undef LF_LIN_BW
    }
    return check_launch();
}

extern "C" int lf_rowmean_fwd(const float* x, int B, int H, int W, int C, float* out, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(x && out && B >= 1 && H >= 1 && W >= 1 && C >= 1 && C <= 256);
    lf_launch(rowmean_fwd_kernel, B * H, 256, 0, stream, x, H, W, C, out);
    return check_launch();
}

extern "C" int lf_rowmean_bwd(const float* dout, int B, int H, int W, int C, float* dx, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(dout && dx && B >= 1 && H >= 1 && W >= 1 && C >= 1);
    const long long total = (long long)B * H * W * C;
    const long long cap = (long long)device_sms() * 8;
    const int grid = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
    lf_launch(rowmean_bwd_kernel, grid, 256, 0, stream, dout, H, W, C, total, dx);
    return check_launch();
}
