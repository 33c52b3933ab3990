// Bandwidth-bound ERFNet pieces for sm_90a: BatchNorm2d (training statistics, apply,
// backward), 2x2 max pooling into a channel slice, the 16->L output ConvTranspose2d and the
// module-boundary layout changes.  All NHWC fp32, 128-bit accesses, deterministic two-stage
// reductions (fp64 partials, fixed summation order).
// Reference: BP/Networks/ERFNet.py:16-22 (pool/cat/bn/relu), :33,39,48-58 (bn, dropout,
// residual), :102-107, :124,152 (output_conv).
#include "lf_common.cuh"

namespace lf {

constexpr int BN_THREADS = 256;
static inline int bn_max_blocks() { return device_sms() * 4; }
constexpr int BN_MIN_PIX_PER_BLOCK = 128;

__device__ __forceinline__ float gate(float v, float m) { return m > 0.f ? v : 0.f; }

// ------------------------------------------------------------------------------------------
// Column statistics.  Thread -> (pixel lane, float4 of channels).  C % 4 == 0, C <= 1024.
// MODE 0: sum x, sum x^2.   MODE 1: sum g, sum g*xhat  with g = dy*(ymask>0)*drop.
// ------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(BN_THREADS) bn_reduce_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                               const float* __restrict__ ymask, const float* __restrict__ drop,
                                                               long long npix, int C, int pix_per_image,
                                                               const float* __restrict__ mean, const float* __restrict__ invstd,
                                                               double* __restrict__ partial) {
    pdl_entry();
    extern __shared__ double sred[];  // [lanes][2][C]
    const int C4 = C >> 2;
    const int lanes = BN_THREADS / C4;
    const int c4 = threadIdx.x % C4, pl = threadIdx.x / C4;
    const long long per = (npix + gridDim.x - 1) / gridDim.x;
    const long long p0 = (long long)blockIdx.x * per;
    const long long p1 = min(npix, p0 + per);
    float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1;
    float4 mu = s1, is = s1;
    if (MODE == 1 && pl < lanes) {
        mu = __ldg(reinterpret_cast<const float4*>(mean) + c4);
        is = __ldg(reinterpret_cast<const float4*>(invstd) + c4);
    }
    if (pl < lanes) {
        for (long long p = p0 + pl; p < p1; p += lanes) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(x + (size_t)p * C) + c4);
            if (MODE == 0) {
                s1.x += v.x; s1.y += v.y; s1.z += v.z; s1.w += v.w;
                s2.x = fmaf(v.x, v.x, s2.x); s2.y = fmaf(v.y, v.y, s2.y);
                s2.z = fmaf(v.z, v.z, s2.z); s2.w = fmaf(v.w, v.w, s2.w);
            } else {
                float4 g = __ldg(reinterpret_cast<const float4*>(dy + (size_t)p * C) + c4);
                if (ymask) {
                    const float4 m = __ldg(reinterpret_cast<const float4*>(ymask + (size_t)p * C) + c4);
                    g.x = gate(g.x, m.x); g.y = gate(g.y, m.y); g.z = gate(g.z, m.z); g.w = gate(g.w, m.w);
                }
                if (drop) {
                    const float4 d = __ldg(reinterpret_cast<const float4*>(drop + (size_t)(p / pix_per_image) * C) + c4);
                    g.x *= d.x; g.y *= d.y; g.z *= d.z; g.w *= d.w;
                }
                s1.x += g.x; s1.y += g.y; s1.z += g.z; s1.w += g.w;
                s2.x = fmaf(g.x, (v.x - mu.x) * is.x, s2.x); s2.y = fmaf(g.y, (v.y - mu.y) * is.y, s2.y);
                s2.z = fmaf(g.z, (v.z - mu.z) * is.z, s2.z); s2.w = fmaf(g.w, (v.w - mu.w) * is.w, s2.w);
            }
        }
        double* r = sred + (size_t)pl * 2 * C;
        r[4 * c4 + 0] = s1.x; r[4 * c4 + 1] = s1.y; r[4 * c4 + 2] = s1.z; r[4 * c4 + 3] = s1.w;
        r[C + 4 * c4 + 0] = s2.x; r[C + 4 * c4 + 1] = s2.y; r[C + 4 * c4 + 2] = s2.z; r[C + 4 * c4 + 3] = s2.w;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 2 * C; k += BN_THREADS) {
        double t = 0.0;
        for (int l = 0; l < lanes; ++l) t += sred[(size_t)l * 2 * C + k];
        partial[(size_t)blockIdx.x * 2 * C + k] = t;
    }
}

// Sum partial[b][2][C] over b for channel c with one warp: lane i takes blocks i, i+32, ... in order,
// then a fixed-shape xor tree -> deterministic, and ~32x less serial latency than one thread.
__device__ __forceinline__ void bn_sum_partials(const double* __restrict__ partial, int nblk, int C, int c, double& s1,
                                                double& s2) {
    const int lane = threadIdx.x & 31;
    // 4 rows per lane in flight (8 independent loads): the strided partial reads are pure latency, and a
    // one-load-at-a-time loop made these finalize kernels 8-11 us each.  Fixed summation order -> deterministic.
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0, b0 = 0.0, b1 = 0.0, b2 = 0.0, b3 = 0.0;
    int k = lane;
    for (; k + 96 < nblk; k += 128) {
        const double x0 = partial[(size_t)k * 2 * C + c], y0 = partial[(size_t)k * 2 * C + C + c];
        const double x1 = partial[(size_t)(k + 32) * 2 * C + c], y1 = partial[(size_t)(k + 32) * 2 * C + C + c];
        const double x2 = partial[(size_t)(k + 64) * 2 * C + c], y2 = partial[(size_t)(k + 64) * 2 * C + C + c];
        const double x3 = partial[(size_t)(k + 96) * 2 * C + c], y3 = partial[(size_t)(k + 96) * 2 * C + C + c];
        a0 += x0; b0 += y0; a1 += x1; b1 += y1; a2 += x2; b2 += y2; a3 += x3; b3 += y3;
    }
    for (; k < nblk; k += 32) {
        a0 += partial[(size_t)k * 2 * C + c];
        b0 += partial[(size_t)k * 2 * C + C + c];
    }
    s1 = warp_sum((a0 + a1) + (a2 + a3));
    s2 = warp_sum((b0 + b1) + (b2 + b3));
}

// Column groups f*C + c (f < fold) of a [nblk][2][C*fold] partial that map to channel c (fold > 1: super-pixel layers),
// each summed by bn_sum_partials, then added in group order
__device__ __forceinline__ void bn_sum_folded(const double* __restrict__ partial, int nblk, int C, int fold, int c, double& s1,
                                              double& s2) {
    s1 = 0.0;
    s2 = 0.0;
    for (int f = 0; f < fold; ++f) {
        double a, b;
        bn_sum_partials(partial, nblk, C * fold, f * C + c, a, b);
        s1 += a;
        s2 += b;
    }
}

// Per-channel finalize arithmetic, shared by the kernels that sum partials themselves and the ones that read totals
// (SyncBatchNorm: totals all-reduced over the ranks), so that both give the same bits from the same sums.
__device__ __forceinline__ void bn_finalize_channel(int c, double s1, double s2, double n, const float* __restrict__ gamma,
                                                    const float* __restrict__ beta, float eps, float momentum,
                                                    float* running_mean, float* running_var, float* mean, float* invstd,
                                                    float* scale, float* shift) {
    const double m = s1 / n;
    double var = s2 / n - m * m;
    if (var < 0.0) var = 0.0;
    const double is = 1.0 / sqrt(var + (double)eps);
    mean[c] = (float)m;
    invstd[c] = (float)is;
    const float sc = gamma[c] * (float)is;
    scale[c] = sc;
    shift[c] = beta[c] - (float)m * sc;
    if (running_mean) {
        const double unb = (n > 1.0) ? var * n / (n - 1.0) : var;
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)m;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unb;
    }
}

// Backward constants from (s1, s2) = (sum g, sum g*xhat): dgamma / dbeta from this rank's sums (l), c1 / c2 from the sums
// over every rank (g) and the global count n.  Single process: l == g.
__device__ __forceinline__ void bn_bwd_finalize_channel(int c, double s1l, double s2l, double s1g, double s2g, double n,
                                                        float* dgamma, float* dbeta, float* c1, float* c2) {
    dbeta[c] = (float)s1l;
    dgamma[c] = (float)s2l;
    c1[c] = (float)(s1g / n);
    c2[c] = (float)(s2g / n);
}

// The same from (s1, s2) = (sum g, sum g*x) of the conv epilogue: sum g*xhat = invstd*(sum g*x - mean*sum g), linear in the
// sums, so converting the all-reduced sums with the (global) mean is exact
__device__ __forceinline__ void bn_bwd_finalize_sx_channel(int c, double s1l, double s2l, double s1g, double s2g, double n,
                                                           const float* __restrict__ mean, const float* __restrict__ invstd,
                                                           float* dgamma, float* dbeta, float* c1, float* c2) {
    const double dgl = (double)invstd[c] * (s2l - (double)mean[c] * s1l);
    const double dgg = (double)invstd[c] * (s2g - (double)mean[c] * s1g);
    dbeta[c] = (float)s1l;
    dgamma[c] = (float)dgl;
    c1[c] = (float)(s1g / n);
    c2[c] = (float)(dgg / n);
}

__global__ void bn_finalize_kernel(const double* __restrict__ partial, int nblk, long long npix, int C,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum,
                                   float* running_mean, float* running_var, float* mean, float* invstd, float* scale,
                                   float* shift) {
    pdl_entry();
    const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // one warp per channel
    if (c >= C) return;
    double s1, s2;
    bn_sum_partials(partial, nblk, C, c, s1, s2);
    if ((threadIdx.x & 31) != 0) return;
    bn_finalize_channel(c, s1, s2, (double)npix, gamma, beta, eps, momentum, running_mean, running_var, mean, invstd, scale,
                        shift);
}

// SyncBatchNorm, step 1: partial[nblk][2][C*fold] -> totals[2C+1] = (sum a [C], sum b [C], npix), summed exactly as the
// finalize kernels sum them (fold == 1: bn_sum_partials, else bn_sum_folded).  local (optional): a second copy, kept
// while `totals` is all-reduced (the backward's dgamma / dbeta are this rank's sums).
__global__ void bn_collapse_kernel(const double* __restrict__ partial, int nblk, int C, int fold, long long npix,
                                   double* __restrict__ totals, double* __restrict__ local) {
    pdl_entry();
    const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // one warp per channel
    if (c >= C) return;
    double s1, s2;
    if (fold == 1) bn_sum_partials(partial, nblk, C, c, s1, s2);
    else bn_sum_folded(partial, nblk, C, fold, c, s1, s2);
    if ((threadIdx.x & 31) != 0) return;
    totals[c] = s1;
    totals[C + c] = s2;
    if (c == 0) totals[2 * C] = (double)npix;
    if (local) {
        local[c] = s1;
        local[C + c] = s2;
        if (c == 0) local[2 * C] = (double)npix;
    }
}

// SyncBatchNorm, step 2 (after the all-reduce of totals): the forward finalize from the global sums and count
__global__ void bn_finalize_tot_kernel(const double* __restrict__ totals, int C, const float* __restrict__ gamma,
                                       const float* __restrict__ beta, float eps, float momentum, float* running_mean,
                                       float* running_var, float* mean, float* invstd, float* scale, float* shift) {
    pdl_entry();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    bn_finalize_channel(c, totals[c], totals[C + c], totals[2 * C], gamma, beta, eps, momentum, running_mean, running_var, mean,
                        invstd, scale, shift);
}

// SX: totals hold (sum g, sum g*x) of the conv epilogue (lf_bn_bwd_finalize_sx), else (sum g, sum g*xhat)
template <bool SX>
__global__ void bn_bwd_finalize_tot_kernel(const double* __restrict__ local, const double* __restrict__ global,
                                           const double* __restrict__ count, int C, const float* __restrict__ mean,
                                           const float* __restrict__ invstd, float* dgamma, float* dbeta, float* c1, float* c2) {
    pdl_entry();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    if (SX)
        bn_bwd_finalize_sx_channel(c, local[c], local[C + c], global[c], global[C + c], *count, mean, invstd, dgamma, dbeta,
                                   c1, c2);
    else
        bn_bwd_finalize_channel(c, local[c], local[C + c], global[c], global[C + c], *count, dgamma, dbeta, c1, c2);
}

__global__ void bn_eval_prepare_kernel(int C, const float* gamma, const float* beta, float eps, const float* rm,
                                       const float* rv, float* scale, float* shift) {
    pdl_entry();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const float is = 1.f / sqrtf(rv[c] + eps);
    const float sc = gamma[c] * is;
    scale[c] = sc;
    shift[c] = beta[c] - rm[c] * sc;
}

__global__ void bn_bwd_finalize_kernel(const double* __restrict__ partial, int nblk, long long npix, int C, float* dgamma,
                                       float* dbeta, float* c1, float* c2) {
    pdl_entry();
    const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // one warp per channel
    if (c >= C) return;
    double s1, s2;
    bn_sum_partials(partial, nblk, C, c, s1, s2);
    if ((threadIdx.x & 31) != 0) return;
    bn_bwd_finalize_channel(c, s1, s2, s1, s2, (double)npix, dgamma, dbeta, c1, c2);
}

// Statistics from the conv epilogue (lf_conv1d_tc[_x3] with mask_scale): [0] = sum g, [1] = sum g*x  ->  sum g*xhat =
// invstd*(sum g*x - mean*sum g), in fp64 (no division by the BatchNorm weight: exact for any gamma, including 0)
__global__ void bn_bwd_finalize_sx_kernel(const double* __restrict__ partial, int nblk, long long npix, int C, int fold,
                                          const float* __restrict__ mean, const float* __restrict__ invstd, float* dgamma,
                                          float* dbeta, float* c1, float* c2) {
    pdl_entry();
    const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // one warp per channel
    if (c >= C) return;
    double s1, s2;
    bn_sum_folded(partial, nblk, C, fold, c, s1, s2);
    if ((threadIdx.x & 31) != 0) return;
    bn_bwd_finalize_sx_channel(c, s1, s2, s1, s2, (double)npix, mean, invstd, dgamma, dbeta, c1, c2);
}

// y = relu?( (x*scale+shift) * drop? + res? )
// BFY: y is bf16, rounded to nearest even
template <bool BFY>
__global__ void __launch_bounds__(256) bn_apply_kernel(const float* __restrict__ x, long long n4, int C4, int pix_per_image,
                                                       const float* __restrict__ scale, const float* __restrict__ shift,
                                                       const float* __restrict__ drop, const float* __restrict__ res, int relu,
                                                       void* __restrict__ y) {
    pdl_entry();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        const long long p = i / C4;
        const float4 v = ld_stream_f4(reinterpret_cast<const float4*>(x) + i);
        const float4 sc = __ldg(reinterpret_cast<const float4*>(scale) + c4);
        const float4 sh = __ldg(reinterpret_cast<const float4*>(shift) + c4);
        float4 o = make_float4(fmaf(v.x, sc.x, sh.x), fmaf(v.y, sc.y, sh.y), fmaf(v.z, sc.z, sh.z), fmaf(v.w, sc.w, sh.w));
        if (drop) {
            const float4 d = __ldg(reinterpret_cast<const float4*>(drop) + (p / pix_per_image) * C4 + c4);
            o.x *= d.x; o.y *= d.y; o.z *= d.z; o.w *= d.w;
        }
        if (res) {
            const float4 r = __ldg(reinterpret_cast<const float4*>(res) + i);
            o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
        }
        if (relu) {
            o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
        }
        if (BFY) reinterpret_cast<uint2*>(y)[i] = f4_to_bf16x4(o);
        else reinterpret_cast<float4*>(y)[i] = o;
    }
}

// dx = gamma*invstd*(g - c1 - xhat*c2),  g = dy*(ymask>0)*drop
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const float* __restrict__ dy, const float* __restrict__ ymask,
                                                           const float* __restrict__ drop, const float* __restrict__ x,
                                                           long long n4, int C4, int pix_per_image,
                                                           const float* __restrict__ mean, const float* __restrict__ invstd,
                                                           const float* __restrict__ gamma, const float* __restrict__ c1,
                                                           const float* __restrict__ c2, float* __restrict__ dx,
                                                           float* __restrict__ gated_out) {
    pdl_entry();
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        const long long p = i / C4;
        float4 g = ld_stream_f4(reinterpret_cast<const float4*>(dy) + i);
        if (ymask) {
            const float4 m = __ldg(reinterpret_cast<const float4*>(ymask) + i);
            g.x = gate(g.x, m.x); g.y = gate(g.y, m.y); g.z = gate(g.z, m.z); g.w = gate(g.w, m.w);
        }
        if (gated_out) reinterpret_cast<float4*>(gated_out)[i] = g;   // dy * (ymask > 0): the residual branch's gradient
        if (drop) {
            const float4 d = __ldg(reinterpret_cast<const float4*>(drop) + (p / pix_per_image) * C4 + c4);
            g.x *= d.x; g.y *= d.y; g.z *= d.z; g.w *= d.w;
        }
        const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
        const float4 mu = __ldg(reinterpret_cast<const float4*>(mean) + c4);
        const float4 is = __ldg(reinterpret_cast<const float4*>(invstd) + c4);
        const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma) + c4);
        const float4 a1 = __ldg(reinterpret_cast<const float4*>(c1) + c4);
        const float4 a2 = __ldg(reinterpret_cast<const float4*>(c2) + c4);
        float4 o;
        o.x = ga.x * is.x * (g.x - a1.x - (v.x - mu.x) * is.x * a2.x);
        o.y = ga.y * is.y * (g.y - a1.y - (v.y - mu.y) * is.y * a2.y);
        o.z = ga.z * is.z * (g.z - a1.z - (v.z - mu.z) * is.z * a2.z);
        o.w = ga.w * is.w * (g.w - a1.w - (v.w - mu.w) * is.w * a2.w);
        reinterpret_cast<float4*>(dx)[i] = o;
    }
}

// ------------------------------------------------------------------------------------------
// 2x2 stride-2 max pooling into a channel slice, and its gradient.
// ------------------------------------------------------------------------------------------
__global__ void maxpool2_fwd_kernel(const float* __restrict__ in, int N, int Hin, int Win, int C, int in_cstride,
                                    float* __restrict__ out, int out_cstride, int out_coff, const float* __restrict__ scale,
                                    const float* __restrict__ shift) {
    pdl_entry();
    const int Ho = Hin >> 1, Wo = Win >> 1;
    const long long total = (long long)N * Ho * Wo * C;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        long long p = idx / C;
        const int ox = (int)(p % Wo);
        p /= Wo;
        const int oy = (int)(p % Ho);
        const int n = (int)(p / Ho);
        const float* b = in + ((size_t)(n * Hin + 2 * oy) * Win + 2 * ox) * in_cstride + c;
        const float v00 = b[0], v01 = b[in_cstride], v10 = b[(size_t)Win * in_cstride], v11 = b[(size_t)(Win + 1) * in_cstride];
        float m = fmaxf(fmaxf(v00, v01), fmaxf(v10, v11));
        if (scale) m = fmaxf(fmaf(m, __ldg(scale + out_coff + c), __ldg(shift + out_coff + c)), 0.f);   // eval: relu(bn(pool))
        out[((size_t)(n * Ho + oy) * Wo + ox) * out_cstride + out_coff + c] = m;
    }
}

__global__ void maxpool2_bwd_kernel(const float* __restrict__ in, int N, int Hin, int Win, int C, int in_cstride,
                                    const float* __restrict__ d_out, int out_cstride, int out_coff, float* __restrict__ d_in,
                                    int din_cstride, int accumulate) {
    pdl_entry();
    const int Ho = Hin >> 1, Wo = Win >> 1;
    const long long total = (long long)N * Ho * Wo * C;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % C);
        long long p = idx / C;
        const int ox = (int)(p % Wo);
        p /= Wo;
        const int oy = (int)(p % Ho);
        const int n = (int)(p / Ho);
        const size_t base = ((size_t)(n * Hin + 2 * oy) * Win + 2 * ox);
        const float* b = in + base * in_cstride + c;
        const float v[4] = {b[0], b[in_cstride], b[(size_t)Win * in_cstride], b[(size_t)(Win + 1) * in_cstride]};
        int arg = 0;
        float best = v[0];
#pragma unroll
        for (int k = 1; k < 4; ++k)
            if (v[k] > best) {  // first maximum wins (ATen max_pool2d)
                best = v[k];
                arg = k;
            }
        const float g = d_out[((size_t)(n * Ho + oy) * Wo + ox) * out_cstride + out_coff + c];
        float* d = d_in + base * din_cstride + c;
        const size_t offs[4] = {0, (size_t)din_cstride, (size_t)Win * din_cstride, (size_t)(Win + 1) * din_cstride};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float gv = (k == arg) ? g : 0.f;
            if (accumulate)
                d[offs[k]] += gv;
            else
                d[offs[k]] = gv;
        }
    }
}

// ------------------------------------------------------------------------------------------
// Decoder.output_conv: ConvTranspose2d(Cin=16 -> L, k=2, s=2):
//   out[n,l,2j+a,2i+b] = bias[l] + sum_ci x[n,j,i,ci] * w[ci][l][a][b]
// ------------------------------------------------------------------------------------------
constexpr int OC_MAXCIN = 16;
constexpr int OC_MAXL = 8;

__global__ void __launch_bounds__(256) outconv_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                          const float* __restrict__ bias, int N, int H, int W, int Cin, int L,
                                                          float* __restrict__ out) {
    pdl_entry();
    __shared__ __align__(16) float ws[OC_MAXCIN * OC_MAXL * 4];
    __shared__ float bs[OC_MAXL];
    for (int k = threadIdx.x; k < Cin * L * 4; k += blockDim.x) ws[k] = w[k];
    if (threadIdx.x < L) bs[threadIdx.x] = bias ? bias[threadIdx.x] : 0.f;
    __syncthreads();
    const long long npix = (long long)N * H * W;
    const int Ho = 2 * H, Wo = 2 * W;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(p % W);
        const int j = (int)((p / W) % H);
        const int n = (int)(p / ((long long)W * H));
        float xv[OC_MAXCIN];
#pragma unroll
        for (int q = 0; q < OC_MAXCIN / 4; ++q) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(x + (size_t)p * Cin) + q);
            xv[4 * q] = v.x; xv[4 * q + 1] = v.y; xv[4 * q + 2] = v.z; xv[4 * q + 3] = v.w;
        }
        for (int l = 0; l < L; ++l) {
            float o[4] = {bs[l], bs[l], bs[l], bs[l]};
#pragma unroll
            for (int ci = 0; ci < OC_MAXCIN; ++ci) {
                const float4 wv = *reinterpret_cast<const float4*>(&ws[(ci * L + l) * 4]);
                o[0] = fmaf(xv[ci], wv.x, o[0]); o[1] = fmaf(xv[ci], wv.y, o[1]);
                o[2] = fmaf(xv[ci], wv.z, o[2]); o[3] = fmaf(xv[ci], wv.w, o[3]);
            }
            float* dst = out + (((size_t)n * L + l) * Ho + 2 * j) * Wo + 2 * i;
            *reinterpret_cast<float2*>(dst) = make_float2(o[0], o[1]);
            *reinterpret_cast<float2*>(dst + Wo) = make_float2(o[2], o[3]);
        }
    }
}

__global__ void __launch_bounds__(256) outconv_bwd_data_kernel(const float* __restrict__ d_out, const float* __restrict__ w,
                                                               int N, int H, int W, int Cin, int L, float* __restrict__ d_x) {
    pdl_entry();
    __shared__ __align__(16) float ws[OC_MAXCIN * OC_MAXL * 4];
    for (int k = threadIdx.x; k < Cin * L * 4; k += blockDim.x) ws[k] = w[k];
    __syncthreads();
    const long long npix = (long long)N * H * W;
    const int Ho = 2 * H, Wo = 2 * W;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(p % W);
        const int j = (int)((p / W) % H);
        const int n = (int)(p / ((long long)W * H));
        float acc[OC_MAXCIN];
#pragma unroll
        for (int ci = 0; ci < OC_MAXCIN; ++ci) acc[ci] = 0.f;
        for (int l = 0; l < L; ++l) {
            const float* src = d_out + (((size_t)n * L + l) * Ho + 2 * j) * Wo + 2 * i;
            const float2 g0 = __ldg(reinterpret_cast<const float2*>(src));
            const float2 g1 = __ldg(reinterpret_cast<const float2*>(src + Wo));
#pragma unroll
            for (int ci = 0; ci < OC_MAXCIN; ++ci) {
                const float4 wv = *reinterpret_cast<const float4*>(&ws[(ci * L + l) * 4]);
                acc[ci] += g0.x * wv.x + g0.y * wv.y + g1.x * wv.z + g1.y * wv.w;
            }
        }
#pragma unroll
        for (int q = 0; q < OC_MAXCIN / 4; ++q)
            *(reinterpret_cast<float4*>(d_x + (size_t)p * Cin) + q) =
                make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
    }
}

constexpr int OCW_PIX_PER_BLOCK = 4096;

// one block = a pixel range; grid.y = lane l.  partial[blk][Cin*L*4 + L]
__global__ void __launch_bounds__(256) outconv_bwd_weight_kernel(const float* __restrict__ x, const float* __restrict__ d_out,
                                                                 int N, int H, int W, int Cin, int L, float* __restrict__ partial) {
    pdl_entry();
    __shared__ float red[8][OC_MAXCIN * 4 + 1];
    const int l = blockIdx.y;
    const long long npix = (long long)N * H * W;
    const long long p0 = (long long)blockIdx.x * OCW_PIX_PER_BLOCK;
    const long long p1 = min(npix, p0 + OCW_PIX_PER_BLOCK);
    const int Ho = 2 * H, Wo = 2 * W;
    float acc[OC_MAXCIN][4];
#pragma unroll
    for (int ci = 0; ci < OC_MAXCIN; ++ci) acc[ci][0] = acc[ci][1] = acc[ci][2] = acc[ci][3] = 0.f;
    float bsum = 0.f;
    for (long long p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
        const int i = (int)(p % W);
        const int j = (int)((p / W) % H);
        const int n = (int)(p / ((long long)W * H));
        const float* src = d_out + (((size_t)n * L + l) * Ho + 2 * j) * Wo + 2 * i;
        const float2 g0 = __ldg(reinterpret_cast<const float2*>(src));
        const float2 g1 = __ldg(reinterpret_cast<const float2*>(src + Wo));
        bsum += (g0.x + g0.y) + (g1.x + g1.y);
#pragma unroll
        for (int q = 0; q < OC_MAXCIN / 4; ++q) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(x + (size_t)p * Cin) + q);
            const float xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                acc[4 * q + e][0] = fmaf(xv[e], g0.x, acc[4 * q + e][0]);
                acc[4 * q + e][1] = fmaf(xv[e], g0.y, acc[4 * q + e][1]);
                acc[4 * q + e][2] = fmaf(xv[e], g1.x, acc[4 * q + e][2]);
                acc[4 * q + e][3] = fmaf(xv[e], g1.y, acc[4 * q + e][3]);
            }
        }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int ci = 0; ci < OC_MAXCIN; ++ci)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float s = warp_sum(acc[ci][e]);
            if (lane == 0) red[warp][ci * 4 + e] = s;
        }
    {
        const float s = warp_sum(bsum);
        if (lane == 0) red[warp][OC_MAXCIN * 4] = s;
    }
    __syncthreads();
    float* dst = partial + (size_t)blockIdx.x * (Cin * L * 4 + L);
    for (int k = threadIdx.x; k < OC_MAXCIN * 4 + 1; k += blockDim.x) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += red[w][k];
        if (k < OC_MAXCIN * 4) {
            const int ci = k >> 2, e = k & 3;
            dst[(ci * L + l) * 4 + e] = s;
        } else {
            dst[Cin * L * 4 + l] = s;
        }
    }
}

// ------------------------------------------------------------------------------------------
// Layout changes at the module boundary (tiled transposes through shared memory).
// ------------------------------------------------------------------------------------------
__global__ void nchw_to_nhwc_pad_kernel(const float* __restrict__ in, int N, int C, int HW, int Cpad, float* __restrict__ out) {
    pdl_entry();
    // thread per output pixel; C is tiny (3) -> each plane read is coalesced across the warp
    const long long total = (long long)N * HW;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(p / HW);
        const int hw = (int)(p % HW);
        for (int c = 0; c < Cpad; ++c) out[(size_t)p * Cpad + c] = (c < C) ? in[((size_t)n * C + c) * HW + hw] : 0.f;
    }
}

// generic [R][S] -> [S][R] per batch item, 32x32 tiles
__global__ void batched_transpose_kernel(const float* __restrict__ in, int R, int S, float* __restrict__ out) {
    pdl_entry();
    __shared__ float tile[32][33];
    const size_t boff = (size_t)blockIdx.z * R * S;
    const int s0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int r = r0 + k, s = s0 + threadIdx.x;
        if (r < R && s < S) tile[k][threadIdx.x] = in[boff + (size_t)r * S + s];
    }
    __syncthreads();
    for (int k = threadIdx.y; k < 32; k += blockDim.y) {
        const int s = s0 + k, r = r0 + threadIdx.x;
        if (r < R && s < S) out[boff + (size_t)s * R + r] = tile[threadIdx.x][k];
    }
}

// Per-image max |x| (the activation scale of an fp8 convolution whose input is not another fp8 convolution's output):
// grid (blocks per image, N); 16-byte loads, a warp max, one atomicMax on the float bits per warp.
template <bool BF>
__global__ void __launch_bounds__(256) amax_per_image_kernel(const void* __restrict__ x, long long per_image, float* amax) {
    pdl_entry();
    const int n = blockIdx.y;
    const long long nvec = per_image / 8;   // 8 elements per step: two float4 or one uint4 of bf16
    float m = 0.f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
        float4 u, v;
        if (BF) {
            const uint4 r = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint16_t*>(x) + (size_t)n * per_image) + i);
            u = bf16x4_to_f4(make_uint2(r.x, r.y));
            v = bf16x4_to_f4(make_uint2(r.z, r.w));
        } else {
            const float4* p = reinterpret_cast<const float4*>(static_cast<const float*>(x) + (size_t)n * per_image) + 2 * i;
            u = __ldg(p);
            v = __ldg(p + 1);
        }
        m = fmaxf(m, fmaxf(fmaxf(fmaxf(fabsf(u.x), fabsf(u.y)), fmaxf(fabsf(u.z), fabsf(u.w))),
                           fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)))));
    }
    const uint32_t w = __reduce_max_sync(0xffffffffu, __float_as_uint(m));   // |x| >= 0: ordered as uint
    if ((threadIdx.x & 31) == 0 && w) atomicMax(reinterpret_cast<unsigned int*>(amax) + n, w);
}

static inline int grid_for(long long n, int threads, int maxblocks = 0) {
    if (maxblocks <= 0) maxblocks = device_sms() * 16;
    long long b = (n + threads - 1) / threads;
    if (b > maxblocks) b = maxblocks;
    if (b < 1) b = 1;
    return (int)b;
}

}  // namespace lf

using namespace lf;
#define STREAM cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_)

extern "C" int lf_bn_blocks(long long npix, int C) {
    (void)C;
    long long b = (npix + BN_MIN_PIX_PER_BLOCK - 1) / BN_MIN_PIX_PER_BLOCK;
    if (b > bn_max_blocks()) b = bn_max_blocks();
    return (int)(b < 1 ? 1 : b);
}

static int bn_check(long long npix, int C) {
    LF_REQUIRE(npix > 0 && C >= 4 && C % 4 == 0 && C <= 1024);
    return LF_OK;
}

extern "C" int lf_bn_stats(const float* x, long long npix, int C, double* partial, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(x && partial);
    int rc = bn_check(npix, C);
    if (rc) return rc;
    const int lanes = BN_THREADS / (C / 4);
    const size_t smem = (size_t)lanes * 2 * C * sizeof(double);
    lf_launch(bn_reduce_kernel<0>, lf_bn_blocks(npix, C), BN_THREADS, smem, stream, x, nullptr, nullptr, nullptr, npix, C, 1, nullptr,
                                                                            nullptr, partial);
    return check_launch();
}

extern "C" int lf_bn_finalize(const double* partial, int nblk, long long npix, int C, const float* gamma, const float* beta,
                              float eps, float momentum, float* running_mean, float* running_var, float* mean, float* invstd,
                              float* scale, float* shift, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(partial && gamma && beta && mean && invstd && scale && shift && nblk >= 1);
    LF_REQUIRE((running_mean == nullptr) == (running_var == nullptr));
    int rc = bn_check(npix, C);   // the kernel divides by npix and the grid is sized from C
    if (rc) return rc;
    lf_launch(bn_finalize_kernel, (C * 32 + 255) / 256, 256, 0, stream, partial, nblk, npix, C, gamma, beta, eps, momentum, running_mean,
                                                            running_var, mean, invstd, scale, shift);
    return check_launch();
}

extern "C" int lf_bn_collapse(const double* partial, int nblk, int C, int fold, long long npix, double* totals, double* local,
                              lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(partial && totals && nblk >= 1 && C >= 1 && fold >= 1 && npix > 0);
    lf_launch(bn_collapse_kernel, (C * 32 + 255) / 256, 256, 0, stream, partial, nblk, C, fold, npix, totals, local);
    return check_launch();
}

extern "C" int lf_bn_finalize_tot(const double* totals, int C, const float* gamma, const float* beta, float eps, float momentum,
                                  float* running_mean, float* running_var, float* mean, float* invstd, float* scale, float* shift,
                                  lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(totals && gamma && beta && mean && invstd && scale && shift && C >= 1);
    LF_REQUIRE((running_mean == nullptr) == (running_var == nullptr));
    lf_launch(bn_finalize_tot_kernel, (C + 127) / 128, 128, 0, stream, totals, C, gamma, beta, eps, momentum, running_mean,
              running_var, mean, invstd, scale, shift);
    return check_launch();
}

extern "C" int lf_bn_bwd_finalize_tot(const double* local, const double* global, const double* count, int C, float* dgamma,
                                      float* dbeta, float* c1, float* c2, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(local && global && count && dgamma && dbeta && c1 && c2 && C >= 1);
    lf_launch(bn_bwd_finalize_tot_kernel<false>, (C + 127) / 128, 128, 0, stream, local, global, count, C, (const float*)nullptr,
              (const float*)nullptr, dgamma, dbeta, c1, c2);
    return check_launch();
}

extern "C" int lf_bn_bwd_finalize_sx_tot(const double* local, const double* global, const double* count, int C, const float* mean,
                                         const float* invstd, float* dgamma, float* dbeta, float* c1, float* c2,
                                         lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(local && global && count && mean && invstd && dgamma && dbeta && c1 && c2 && C >= 1);
    lf_launch(bn_bwd_finalize_tot_kernel<true>, (C + 127) / 128, 128, 0, stream, local, global, count, C, mean, invstd, dgamma,
              dbeta, c1, c2);
    return check_launch();
}

extern "C" int lf_bn_eval_prepare(int C, const float* gamma, const float* beta, float eps, const float* running_mean,
                                  const float* running_var, float* scale, float* shift, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(gamma && beta && running_mean && running_var && scale && shift && C >= 1);
    lf_launch(bn_eval_prepare_kernel, (C + 127) / 128, 128, 0, stream, C, gamma, beta, eps, running_mean, running_var, scale, shift);
    return check_launch();
}

template <bool BFY>
static int bn_apply_run(const float* x, long long npix, int C, int pix_per_image, const float* scale, const float* shift,
                        const float* drop, const float* res, int relu, void* y, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(x && scale && shift && y && pix_per_image > 0);
    int rc = bn_check(npix, C);
    if (rc) return rc;
    const long long n4 = npix * (C / 4);
    lf_launch(bn_apply_kernel<BFY>, grid_for(n4, 256), 256, 0, stream, x, n4, C / 4, pix_per_image, scale, shift, drop, res, relu, y);
    return check_launch();
}

extern "C" int lf_bn_apply(const float* x, long long npix, int C, int pix_per_image, const float* scale, const float* shift,
                           const float* drop, const float* res, int relu, float* y, lf_stream_t stream_) {
    return bn_apply_run<false>(x, npix, C, pix_per_image, scale, shift, drop, res, relu, y, stream_);
}

extern "C" int lf_bn_apply_bf16(const float* x, long long npix, int C, int pix_per_image, const float* scale, const float* shift,
                                const float* drop, const float* res, int relu, void* y, lf_stream_t stream_) {
    return bn_apply_run<true>(x, npix, C, pix_per_image, scale, shift, drop, res, relu, y, stream_);
}

extern "C" int lf_bn_bwd_reduce(const float* dy, const float* ymask, const float* drop, const float* x, long long npix, int C,
                                int pix_per_image, const float* mean, const float* invstd, double* partial,
                                lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(dy && x && mean && invstd && partial && pix_per_image > 0);
    int rc = bn_check(npix, C);
    if (rc) return rc;
    const int lanes = BN_THREADS / (C / 4);
    const size_t smem = (size_t)lanes * 2 * C * sizeof(double);
    lf_launch(bn_reduce_kernel<1>, lf_bn_blocks(npix, C), BN_THREADS, smem, stream, x, dy, ymask, drop, npix, C, pix_per_image, mean,
                                                                            invstd, partial);
    return check_launch();
}

extern "C" int lf_bn_bwd_finalize(const double* partial, int nblk, long long npix, int C, float* dgamma, float* dbeta,
                                  float* c1, float* c2, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(partial && dgamma && dbeta && c1 && c2 && nblk >= 1);
    int rc = bn_check(npix, C);
    if (rc) return rc;
    lf_launch(bn_bwd_finalize_kernel, (C * 32 + 255) / 256, 256, 0, stream, partial, nblk, npix, C, dgamma, dbeta, c1, c2);
    return check_launch();
}

extern "C" int lf_bn_bwd_finalize_sx(const double* partial, int nblk, long long npix, int C, int fold, const float* mean,
                                     const float* invstd, float* dgamma, float* dbeta, float* c1, float* c2, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(partial && mean && invstd && dgamma && dbeta && c1 && c2 && nblk >= 1 && fold >= 1 && C >= 1);
    lf_launch(bn_bwd_finalize_sx_kernel, (C * 32 + 255) / 256, 256, 0, stream, partial, nblk, npix, C, fold, mean, invstd, dgamma, dbeta,
                                                                       c1, c2);
    return check_launch();
}

extern "C" int lf_bn_bwd_apply(const float* dy, const float* ymask, const float* drop, const float* x, long long npix, int C,
                               int pix_per_image, const float* mean, const float* invstd, const float* gamma, const float* c1,
                               const float* c2, float* dx, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(dy && x && mean && invstd && gamma && c1 && c2 && dx && pix_per_image > 0);
    int rc = bn_check(npix, C);
    if (rc) return rc;
    const long long n4 = npix * (C / 4);
    lf_launch(bn_bwd_apply_kernel, grid_for(n4, 256), 256, 0, stream, dy, ymask, drop, x, n4, C / 4, pix_per_image, mean, invstd,
                                                              gamma, c1, c2, dx, (float*)nullptr);
    return check_launch();
}

// Same, and also stores gated = dy * (ymask > 0) (before the dropout factor): in a residual block that is the gradient of
// the skip connection, which the block's last input-gradient conv then adds as ONE pre-masked operand instead of reading
// dy and the mask tensor again in its epilogue (the two-operand residual epilogue was the slowest conv flavour).
extern "C" int lf_bn_bwd_apply_gated(const float* dy, const float* ymask, const float* drop, const float* x, long long npix, int C,
                                     int pix_per_image, const float* mean, const float* invstd, const float* gamma, const float* c1,
                                     const float* c2, float* dx, float* gated, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(dy && x && mean && invstd && gamma && c1 && c2 && dx && gated && pix_per_image > 0);
    int rc = bn_check(npix, C);
    if (rc) return rc;
    const long long n4 = npix * (C / 4);
    lf_launch(bn_bwd_apply_kernel, grid_for(n4, 256), 256, 0, stream, dy, ymask, drop, x, n4, C / 4, pix_per_image, mean, invstd,
                                                              gamma, c1, c2, dx, gated);
    return check_launch();
}

extern "C" int lf_maxpool2_fwd(const float* in, int N, int Hin, int Win, int C, int in_cstride, float* out, int out_cstride,
                               int out_coff, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(in && out && N > 0 && Hin > 1 && Win > 1 && C > 0 && Hin % 2 == 0 && Win % 2 == 0);
    const long long total = (long long)N * (Hin / 2) * (Win / 2) * C;
    lf_launch(maxpool2_fwd_kernel, grid_for(total, 256), 256, 0, stream, in, N, Hin, Win, C, in_cstride, out, out_cstride, out_coff,
              (const float*)nullptr, (const float*)nullptr);
    return check_launch();
}

// eval-mode DownsamplerBlock: the pooled half of relu(bn(cat[conv, pool])) with the BatchNorm as a per-channel affine
// (scale / shift indexed by the OUTPUT channel out_coff + c), so no BatchNorm pass over the concatenated tensor is needed
extern "C" int lf_maxpool2_affine_relu(const float* in, int N, int Hin, int Win, int C, int in_cstride, const float* scale,
                                       const float* shift, float* out, int out_cstride, int out_coff, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(in && out && scale && shift && N > 0 && Hin > 1 && Win > 1 && C > 0 && Hin % 2 == 0 && Win % 2 == 0);
    const long long total = (long long)N * (Hin / 2) * (Win / 2) * C;
    lf_launch(maxpool2_fwd_kernel, grid_for(total, 256), 256, 0, stream, in, N, Hin, Win, C, in_cstride, out, out_cstride, out_coff,
              scale, shift);
    return check_launch();
}

extern "C" int lf_maxpool2_bwd(const float* in, int N, int Hin, int Win, int C, int in_cstride, const float* d_out,
                               int out_cstride, int out_coff, float* d_in, int din_cstride, int accumulate,
                               lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(in && d_out && d_in && N > 0 && Hin > 1 && Win > 1 && C > 0 && Hin % 2 == 0 && Win % 2 == 0);
    const long long total = (long long)N * (Hin / 2) * (Win / 2) * C;
    lf_launch(maxpool2_bwd_kernel, grid_for(total, 256), 256, 0, stream, in, N, Hin, Win, C, in_cstride, d_out, out_cstride, out_coff,
                                                                 d_in, din_cstride, accumulate);
    return check_launch();
}

extern "C" int lf_outconv_fwd(const float* x, const float* w, const float* bias, int N, int H, int W, int Cin, int L,
                              float* out, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(x && w && out && N > 0 && H > 0 && W > 0);
    if (Cin != OC_MAXCIN || L < 1 || L > OC_MAXL) return LF_ERR_UNSUPPORTED;
    lf_launch(outconv_fwd_kernel, grid_for((long long)N * H * W, 256), 256, 0, stream, x, w, bias, N, H, W, Cin, L, out);
    return check_launch();
}

extern "C" int lf_outconv_bwd_data(const float* d_out, const float* w, int N, int H, int W, int Cin, int L, float* d_x,
                                   lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(d_out && w && d_x && N > 0 && H > 0 && W > 0);
    if (Cin != OC_MAXCIN || L < 1 || L > OC_MAXL) return LF_ERR_UNSUPPORTED;
    lf_launch(outconv_bwd_data_kernel, grid_for((long long)N * H * W, 256), 256, 0, stream, d_out, w, N, H, W, Cin, L, d_x);
    return check_launch();
}

extern "C" int lf_outconv_wgrad_blocks(long long npix) { return (int)((npix + OCW_PIX_PER_BLOCK - 1) / OCW_PIX_PER_BLOCK); }

extern "C" int lf_outconv_bwd_weight(const float* x, const float* d_out, int N, int H, int W, int Cin, int L, float* partial,
                                     lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(x && d_out && partial && N > 0 && H > 0 && W > 0);
    if (Cin != OC_MAXCIN || L < 1 || L > OC_MAXL) return LF_ERR_UNSUPPORTED;
    dim3 grid(lf_outconv_wgrad_blocks((long long)N * H * W), L);
    lf_launch(outconv_bwd_weight_kernel, grid, 256, 0, stream, x, d_out, N, H, W, Cin, L, partial);
    return check_launch();
}

// ------------------------------------------------------------------------------------------
// Batched weight packing: every layer's GEMM-layout weight operand (forward, input-gradient, super-pixel ...)
// is a gather of the reference-layout parameter (index -1 = structural zero).  One launch per training step
// serves all ~130 operands (blockIdx.y = job) instead of ~250 small permute / copy / fill launches.
// ------------------------------------------------------------------------------------------
struct PackJob {
    const float* src;
    void* dst;
    const int* idx;
    long long n;
    int dst_dtype;   // LF_F32, or LF_BF16: the operand of the bf16 convolution mode, rounded to nearest even
    int pad;
};
static_assert(sizeof(PackJob) == 40, "LfPackJob layout");

__global__ void __launch_bounds__(256) pack_gather_kernel(const PackJob* __restrict__ jobs) {
    pdl_entry();
    const PackJob j = jobs[blockIdx.y];
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < j.n; k += (long long)gridDim.x * blockDim.x) {
        const int i = __ldg(j.idx + k);
        float v = i >= 0 ? __ldg(j.src + (i & LF_PACK_INDEX_MASK)) : 0.f;
        if (i >= 0 && (i & (LF_PACK_TF32_HI | LF_PACK_TF32_LO))) {
            // 3xTF32 operand split (conv_tc.cu): hi = TF32 round-to-nearest of v, lo = TF32 rounding of v - hi; both
            // have their 13 low mantissa bits cleared, so the tensor core's own fp32 -> TF32 conversion is the identity
            const float hi = __uint_as_float((__float_as_uint(v) + 0x1000u) & 0xffffe000u);
            v = (i & LF_PACK_TF32_HI) ? hi : __uint_as_float((__float_as_uint(v - hi) + 0x1000u) & 0xffffe000u);
        }
        if (j.dst_dtype == LF_BF16) static_cast<__nv_bfloat16*>(j.dst)[k] = __float2bfloat16_rn(v);
        else static_cast<float*>(j.dst)[k] = v;
    }
}

extern "C" int lf_pack_gather(const LfPackJob* jobs_dev, int njobs, int blocks_per_job, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(jobs_dev && njobs > 0 && njobs <= 65535 && blocks_per_job > 0);
    dim3 grid(blocks_per_job, njobs);
    lf_launch(pack_gather_kernel, grid, 256, 0, stream, reinterpret_cast<const PackJob*>(jobs_dev));
    return check_launch();
}

extern "C" int lf_nchw_to_nhwc_pad(const float* in, int N, int C, int H, int W, int Cpad, float* out, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(in && out && N > 0 && C > 0 && Cpad >= C);
    lf_launch(nchw_to_nhwc_pad_kernel, grid_for((long long)N * H * W, 256), 256, 0, stream, in, N, C, H * W, Cpad, out);
    return check_launch();
}

extern "C" int lf_nhwc_to_nchw(const float* in, int N, int H, int W, int C, float* out, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(in && out && N > 0 && N <= 65535);
    const int R = H * W, S = C;  // [HW][C] -> [C][HW]
    dim3 grid((S + 31) / 32, (R + 31) / 32, N), block(32, 8);
    LF_REQUIRE((R + 31) / 32 <= 65535);
    lf_launch(batched_transpose_kernel, grid, block, 0, stream, in, R, S, out);
    return check_launch();
}

extern "C" int lf_nchw_to_nhwc(const float* in, int N, int C, int H, int W, float* out, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(in && out && N > 0 && N <= 65535);
    const int R = C, S = H * W;  // [C][HW] -> [HW][C]
    dim3 grid((S + 31) / 32, (R + 31) / 32, N), block(32, 8);
    lf_launch(batched_transpose_kernel, grid, block, 0, stream, in, R, S, out);
    return check_launch();
}

extern "C" int lf_amax_per_image(const void* x, int dtype, long long per_image, int N, float* amax, lf_stream_t stream_) {
    STREAM;
    LF_REQUIRE(x && amax && N > 0 && N <= 65535 && per_image > 0 && per_image % 8 == 0);
    LF_REQUIRE(dtype == LF_F32 || dtype == LF_BF16);
    int bx = (device_sms() * 4 + N - 1) / N;   // about four CTAs per SM over the whole batch
    const long long need = (per_image / 8 + 255) / 256;
    if (bx > need) bx = (int)need;
    dim3 grid(bx < 1 ? 1 : bx, N);
    if (dtype == LF_BF16) lf_launch(amax_per_image_kernel<true>, grid, 256, 0, stream, x, per_image, amax);
    else lf_launch(amax_per_image_kernel<false>, grid, 256, 0, stream, x, per_image, amax);
    return check_launch();
}
