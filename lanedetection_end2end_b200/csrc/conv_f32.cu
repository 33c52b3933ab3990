// Generic NHWC fp32 implicit-GEMM convolution on CUDA cores ("parity mode": fp32-exact,
// used for every layer shape; the tensor-core kernels in conv_tc.cu take over the dense
// 1-D convolutions in fast mode).
//
// One launch computes, for an output sub-grid ("phase") enumerated as (n, j < Hs, i < Ws):
//     out[n, j*osy+oy0, i*osx+ox0, coff + co] =
//         epi( sum_{t < ntaps} sum_{ci} in[n, j*isy+dy[t], i*isx+dx[t], ci] * Wmat[wtap[t]][ci][co] )
// with zero fill outside the input.  This single form covers
//   - Conv2d forward, any stride / padding / dilation   (BP/Networks/ERFNet.py:15,29-37)
//   - its input gradient for stride 1 (taps negated, weights transposed)
//   - ConvTranspose2d forward / the input gradient of a stride-2 conv, as 4 phases
//     (ERFNet.py:101; the gather form of a transposed conv)
//   - the input gradient of ConvTranspose2d (a stride-2 conv over the output gradient)
// Epilogue: + bias[co], ReLU, * (mask_src > 0) (ReLU backward), + add_src * (add_mask > 0)
// (residual gradient), all optional.
#include "lf_common.cuh"

namespace lf {

constexpr int CONV_BM = 128;
constexpr int CONV_BK = 16;
constexpr int CONV_THREADS = 256;
constexpr int CONV_APAD = 4;

template <int BN>
struct ConvTile {
    // 16-channel layers are bandwidth-bound: a 256-pixel tile doubles the FMAs per shared-memory load
    static constexpr int BM = (BN == 16) ? 256 : CONV_BM;
    static constexpr int AH = BM / 64;            // float4 A loads per thread and K step
    static constexpr int TN = (BN >= 128) ? 8 : 4;
    static constexpr int TX = BN / TN;            // threads along N
    static constexpr int TY = CONV_THREADS / TX;  // threads along M
    static constexpr int TM = BM / TY;
    static_assert(TM * TY == BM, "tile");
    static constexpr int B_F4 = CONV_BK * BN / 4;  // float4 per B tile
    static constexpr int B_PER_THREAD = (B_F4 + CONV_THREADS - 1) / CONV_THREADS;
};

template <int BN>
__global__ void __launch_bounds__(CONV_THREADS) conv_igemm_f32_kernel(const ConvArgs a) {
    pdl_entry();
    using T = ConvTile<BN>;
    constexpr int TM = T::TM, TN = T::TN;
    constexpr int BM = T::BM, AH = T::AH;
    __shared__ __align__(16) float As[2][CONV_BK][BM + CONV_APAD];
    __shared__ __align__(16) float Bs[2][CONV_BK][BN];

    const int tid = threadIdx.x;
    const int tx = tid % T::TX, ty = tid / T::TX;
    const int m_tile = blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int M = a.N * a.Hs * a.Ws;
    const int K = a.ntaps * a.Cin;
    const int nk = (K + CONV_BK - 1) / CONV_BK;

    // --- A loader bookkeeping: this thread loads float4 (4 k's) for pixels m_a[0], m_a[1]
    const int kq = tid & 3;
    int a_n[AH], a_iy0[AH], a_ix0[AH];
    bool a_valid[AH];
#pragma unroll
    for (int h = 0; h < AH; ++h) {
        const int m = m_tile + (tid >> 2) + 64 * h;
        a_valid[h] = m < M;
        const int mm = a_valid[h] ? m : 0;
        const int n = mm / (a.Hs * a.Ws);
        const int rem = mm - n * (a.Hs * a.Ws);
        const int j = rem / a.Ws;
        const int i = rem - j * a.Ws;
        a_n[h] = n;
        a_iy0[h] = j * a.isy;
        a_ix0[h] = i * a.isx;
    }
    float4 ra[AH];
    float4 rb[T::B_PER_THREAD];

    auto load_tiles = [&](int kt) {
        const int kg = kt * CONV_BK + 4 * kq;
        const int t = kg / a.Cin;
        const int ci = kg - t * a.Cin;
        const bool kok = kg < K;
        const int dy = kok ? a.dy[t] : 0, dx = kok ? a.dx[t] : 0;
#pragma unroll
        for (int h = 0; h < AH; ++h) {
            const int iy = a_iy0[h] + dy, ix = a_ix0[h] + dx;
            const bool ok = kok && a_valid[h] && iy >= 0 && iy < a.Hin && ix >= 0 && ix < a.Win;
            if (ok) {
                const float* p = a.in + ((size_t)(a_n[h] * a.Hin + iy) * a.Win + ix) * a.in_cstride + ci;
                ra[h] = __ldg(reinterpret_cast<const float4*>(p));
            } else {
                ra[h] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
#pragma unroll
        for (int q = 0; q < T::B_PER_THREAD; ++q) {
            const int f = tid + q * CONV_THREADS;
            if (f < T::B_F4) {
                const int kr = f / (BN / 4), c4 = f % (BN / 4);
                const int kgb = kt * CONV_BK + kr;
                if (kgb < K) {
                    const int tb = kgb / a.Cin;
                    const int cib = kgb - tb * a.Cin;
                    const float* p = a.wmat + ((size_t)(a.wtap[tb] * a.Cin + cib)) * a.CoutPad + n0 + 4 * c4;
                    rb[q] = __ldg(reinterpret_cast<const float4*>(p));
                } else {
                    rb[q] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
        }
    };
    auto store_tiles = [&](int buf) {
#pragma unroll
        for (int h = 0; h < AH; ++h) {
            const int m = (tid >> 2) + 64 * h;
            As[buf][4 * kq + 0][m] = ra[h].x;
            As[buf][4 * kq + 1][m] = ra[h].y;
            As[buf][4 * kq + 2][m] = ra[h].z;
            As[buf][4 * kq + 3][m] = ra[h].w;
        }
#pragma unroll
        for (int q = 0; q < T::B_PER_THREAD; ++q) {
            const int f = tid + q * CONV_THREADS;
            if (f < T::B_F4) {
                const int kr = f / (BN / 4), c4 = f % (BN / 4);
                *reinterpret_cast<float4*>(&Bs[buf][kr][4 * c4]) = rb[q];
            }
        }
    };

    float acc[TM][TN];
#pragma unroll
    for (int r = 0; r < TM; ++r)
#pragma unroll
        for (int c = 0; c < TN; ++c) acc[r][c] = 0.f;

    load_tiles(0);
    store_tiles(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) load_tiles(kt + 1);
#pragma unroll
        for (int k = 0; k < CONV_BK; ++k) {
            float av[TM], bv[TN];
#pragma unroll
            for (int r = 0; r < TM; r += (TM >= 4 ? 4 : TM)) {
                if (TM >= 4) {
                    const float4 v = *reinterpret_cast<const float4*>(&As[buf][k][ty * TM + r]);
                    av[r] = v.x; av[r + 1] = v.y; av[r + 2] = v.z; av[r + 3] = v.w;
                } else {
                    const float2 v = *reinterpret_cast<const float2*>(&As[buf][k][ty * TM + r]);
                    av[r] = v.x; av[r + 1] = v.y;
                }
            }
#pragma unroll
            for (int c = 0; c < TN; c += 4) {
                const float4 v = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * TN + c]);
                bv[c] = v.x; bv[c + 1] = v.y; bv[c + 2] = v.z; bv[c + 3] = v.w;
            }
#pragma unroll
            for (int r = 0; r < TM; ++r)
#pragma unroll
                for (int c = 0; c < TN; ++c) acc[r][c] = fmaf(av[r], bv[c], acc[r][c]);
        }
        if (kt + 1 < nk) store_tiles(buf ^ 1);
        __syncthreads();
    }

    // --- epilogue
    const int co0 = n0 + tx * TN;
    if (co0 >= a.Cout) return;
    float bias[TN];
#pragma unroll
    for (int c = 0; c < TN; ++c) bias[c] = (a.bias && co0 + c < a.Cout) ? __ldg(a.bias + co0 + c) : 0.f;
#pragma unroll
    for (int r = 0; r < TM; ++r) {
        const int m = m_tile + ty * TM + r;
        if (m >= M) continue;
        const int n = m / (a.Hs * a.Ws);
        const int rem = m - n * (a.Hs * a.Ws);
        const int j = rem / a.Ws;
        const int i = rem - j * a.Ws;
        const size_t pix = ((size_t)(n * a.Hout + j * a.osy + a.oy0) * a.Wout + i * a.osx + a.ox0);
        const size_t off = pix * a.out_cstride + a.out_coff + co0;
        float v[TN];
#pragma unroll
        for (int c = 0; c < TN; ++c) {
            v[c] = acc[r][c] + bias[c];
            if (a.relu) v[c] = fmaxf(v[c], 0.f);
        }
        const bool full = (co0 + TN <= a.Cout);
        if (full) {
#pragma unroll
            for (int c = 0; c < TN; c += 4) {
                float4 o = make_float4(v[c], v[c + 1], v[c + 2], v[c + 3]);
                if (a.mask_src) {
                    const float4 mk = __ldg(reinterpret_cast<const float4*>(a.mask_src + off + c));
                    o.x = mk.x > 0.f ? o.x : 0.f; o.y = mk.y > 0.f ? o.y : 0.f;
                    o.z = mk.z > 0.f ? o.z : 0.f; o.w = mk.w > 0.f ? o.w : 0.f;
                }
                if (a.add_src) {
                    float4 ad = __ldg(reinterpret_cast<const float4*>(a.add_src + off + c));
                    if (a.add_mask) {
                        const float4 mk = __ldg(reinterpret_cast<const float4*>(a.add_mask + off + c));
                        ad.x = mk.x > 0.f ? ad.x : 0.f; ad.y = mk.y > 0.f ? ad.y : 0.f;
                        ad.z = mk.z > 0.f ? ad.z : 0.f; ad.w = mk.w > 0.f ? ad.w : 0.f;
                    }
                    o.x += ad.x; o.y += ad.y; o.z += ad.z; o.w += ad.w;
                }
                *reinterpret_cast<float4*>(a.out + off + c) = o;
            }
        } else {
            for (int c = 0; c < TN && co0 + c < a.Cout; ++c) {
                float o = v[c];
                if (a.mask_src) o = a.mask_src[off + c] > 0.f ? o : 0.f;
                if (a.add_src) {
                    float ad = a.add_src[off + c];
                    if (a.add_mask) ad = a.add_mask[off + c] > 0.f ? ad : 0.f;
                    o += ad;
                }
                a.out[off + c] = o;
            }
        }
    }
}

}  // namespace lf

using namespace lf;

extern "C" int lf_conv_f32(const LfConvArgs* args, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!args) return LF_ERR_INVALID_ARGUMENT;
    const ConvArgs& a = *args;
    LF_REQUIRE(a.in && a.wmat && a.out);
    LF_REQUIRE(a.N > 0 && a.Hs > 0 && a.Ws > 0 && a.Cin > 0 && a.Cout > 0);
    LF_REQUIRE(a.ntaps >= 1 && a.ntaps <= LF_MAX_TAPS);
    LF_REQUIRE(a.Cin % 4 == 0 && a.in_cstride % 4 == 0 && a.out_cstride % 4 == 0 && a.out_coff % 4 == 0);
    LF_REQUIRE(a.CoutPad % 16 == 0 && a.CoutPad >= a.Cout);
    const long long M = (long long)a.N * a.Hs * a.Ws;
    LF_REQUIRE(M < (1ll << 31));
    int BN = 16;
    if (a.CoutPad % 128 == 0) BN = 128;
    else if (a.CoutPad % 64 == 0) BN = 64;
    else if (a.CoutPad % 32 == 0) BN = 32;
    const int BMsel = (BN == 16) ? 256 : CONV_BM;
    dim3 grid((unsigned)((M + BMsel - 1) / BMsel), a.CoutPad / BN);
    switch (BN) {
        case 128: lf_launch(conv_igemm_f32_kernel<128>, grid, CONV_THREADS, 0, stream, a); break;
        case 64: lf_launch(conv_igemm_f32_kernel<64>, grid, CONV_THREADS, 0, stream, a); break;
        case 32: lf_launch(conv_igemm_f32_kernel<32>, grid, CONV_THREADS, 0, stream, a); break;
        default: lf_launch(conv_igemm_f32_kernel<16>, grid, CONV_THREADS, 0, stream, a); break;
    }
    return check_launch();
}
