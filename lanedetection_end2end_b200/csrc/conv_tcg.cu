// Hopper (sm_90a) wgmma "gather-GEMM" convolution for ERFNet's resolution-changing layers: the 3x3 stride-2 Conv2d of
// DownsamplerBlock (BP/Networks/ERFNet.py:15,19-22), the 3x3 stride-2 ConvTranspose2d of UpsamplerBlock
// (:66-73) and the input gradients of both.  fp32 NHWC storage, fp32 accumulate.
//
//   out[n, oy*oy_mul + oy0, ox, c] = bias[c] + sum_{t<ntaps} sum_{k<Kc} A_{map[t]}[n, oy+dy[t], ox+dx[t], k] * Wg[c][t*Kc + k]
//
// over the iteration domain (n, oy, ox) in [N] x [Hs] x [Ws].  The host (ops_net.py) turns the four layer
// forms into this one by viewing two horizontally adjacent pixels as one "pair pixel" with twice the
// channels (a free view of NHWC memory) and the even / odd input rows as two strided views (A_0, A_1), so
// that a stride-2 access pattern becomes unit-stride taps over pair pixels:
//   * stride-2 conv (Down forward, Up input-gradient): 6 taps = 3 kernel rows x pair offsets {-1, 0},
//     Kc = 2*Cin, weights zero where a (pair offset, half) combination is not a kernel column;
//   * stride-2 transposed conv (Up forward, Down input-gradient): one launch per output row parity
//     (2 or 4 taps over the un-strided input), Ng = 2*Cout = both output columns of the pair.
// One TMA box [128 px x 32 ch] per tap and 32-channel chunk (OOB zero fill = conv padding) and the weight chunk
// [Ng x 32] next to it stream through an mbarrier ring (the weight matrices of these layers, up to 393 KB, do not fit in
// shared memory); Ng is a run-time multiple of 16 (<= 128), covered by wgmma m64n16k8 column blocks.
// Two consumer warpgroups own 64 pixel rows each (A fragments loaded from the swizzled box into registers, B through a
// shared-memory descriptor), accumulate in registers and store the tile with bias / ReLU; warp 8 is the TMA producer.
// precision 1 (3xTF32, template X3; arithmetic in tc_ptx.cuh): the weight chunk is the pre-split pair [W_hi rows | W_lo
// rows] (one TMA box of 2*Ng rows); a_hi*w_hi accumulates apart from a_hi*w_lo + a_lo*w_hi and the two are added at the end.
#include <cuda.h>

#include "lf_common.cuh"
#include "tc_ptx.cuh"

namespace lf {

constexpr int TG_THREADS = 288;
constexpr int TG_BM = 128;
constexpr int TG_A_BYTES = TG_BM * 128;  // 16 KB
constexpr int TG_MAX_STAGES = 8;
constexpr int TG_MAXT = LF_TCG_MAX_TAPS;
constexpr int TG_SMEM_LIMIT = 227 * 1024;
constexpr int TG_NB = 8;                 // column blocks of 16 (Ng <= 128)

struct TgArgs {
    float* out;
    const float* bias;
    long long osn, osy, osx;
    int oy_mul, oy0;
    int relu;
    int N, Hs, Ws;
    int bx, by;
    int kchunks, Ng, ntaps;
    int map[TG_MAXT], dy[TG_MAXT], dx[TG_MAXT];
    int stages, stage_bytes;
    int total_tiles;
};

template <bool X3>
__global__ void __launch_bounds__(TG_THREADS, 1)
conv_tcg_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                const __grid_constant__ CUtensorMap tmB, const TgArgs a) {
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)a.stages * a.stage_bytes);
    uint64_t* empty = full + TG_MAX_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_x = a.Ws / a.bx, tiles_y = a.Hs / a.by;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA0);
        tma_prefetch_desc(&tmA1);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < a.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);   // one arrive per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();   // everything above overlapped the previous kernel's tail; global memory is touched only from here on

    if (warp == 8) {
        // ================= TMA producer (converged warp, elected lane issues) =================
        const bool leader = elect_one();
        int stage = 0;
        uint32_t phase = 0;
        for (int mt = blockIdx.x; mt < a.total_tiles; mt += gridDim.x) {
            const int tx = mt % tiles_x;
            const int ty = (mt / tiles_x) % tiles_y;
            const int n = mt / (tiles_x * tiles_y);
            for (int t = 0; t < a.ntaps; ++t) {
                const CUtensorMap* tm = a.map[t] ? &tmA1 : &tmA0;
                const int x0 = tx * a.bx + a.dx[t], y0 = ty * a.by + a.dy[t];
                for (int cb = 0; cb < a.kchunks; ++cb) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    if (leader) {
                        uint8_t* st = smem + (size_t)stage * a.stage_bytes;
                        mbar_arrive_expect_tx(&full[stage], a.stage_bytes);
                        tma_load_5d(tm, &full[stage], st, 0, cb, x0, y0, n);
                        tma_load_2d(&tmB, &full[stage], st + TG_A_BYTES, (t * a.kchunks + cb) * 32, 0);   // X3: 2*Ng rows (hi | lo)
                    }
                    if (++stage == a.stages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
        return;
    }

    // ================= consumers: warpgroup wg owns pixel rows [64 wg, 64 wg + 64) =================
    const int wg = warp >> 2, wl = warp & 3;
    const int g = lane >> 2, t4 = lane & 3;
    const int ra = 64 * wg + 16 * wl + g;   // fragment rows ra, ra + 8
    const int nblk = a.Ng >> 4;
    const int ksteps = a.ntaps * a.kchunks;
    int stage = 0;
    uint32_t phase = 0;
    for (int mt = blockIdx.x; mt < a.total_tiles; mt += gridDim.x) {
        float acc[TG_NB][8], acs[TG_NB][8];
#pragma unroll
        for (int j = 0; j < TG_NB; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[j][i] = acs[j][i] = 0.f;
        for (int ks = 0; ks < ksteps; ++ks) {
            mbar_wait(&full[stage], phase);
            const uint8_t* st = smem + (size_t)stage * a.stage_bytes;
            uint32_t ah[4][4], al[4][4];
#pragma unroll
            for (int k8 = 0; k8 < 4; ++k8) {
                const int c = 8 * k8 + t4;
                const float v[4] = {*reinterpret_cast<const float*>(st + sw128_off(ra, c)),
                                    *reinterpret_cast<const float*>(st + sw128_off(ra + 8, c)),
                                    *reinterpret_cast<const float*>(st + sw128_off(ra, c + 4)),
                                    *reinterpret_cast<const float*>(st + sw128_off(ra + 8, c + 4))};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (X3) {
                        tf32_split(v[q], ah[k8][q], al[k8][q]);
                    } else {
                        ah[k8][q] = tf32_rna(v[q]);
                    }
                }
            }
            const uint64_t bd = wgmma_desc_sw128(smem_u32(st + TG_A_BYTES));
            const uint64_t lo_rows = (uint64_t)(a.Ng * 128) >> 4;   // W_lo rows follow the Ng W_hi rows
            // One column block at a time: its 32 products are summed by the tensor core from zero and added to the running
            // fp32 sum with a rounded FADD (the tensor core's own accumulation does not round like IEEE adds, see conv_tc.cu).
#pragma unroll
            for (int j = 0; j < TG_NB; ++j) {
                if (j < nblk) {
                    const uint64_t bj = bd + (uint64_t)((j * 16 * 128) >> 4);
                    float part[8];
                    wgmma_fence();
#pragma unroll
                    for (int k8 = 0; k8 < 4; ++k8) {
                        wgmma_m64n16k8_tf32(part, ah[k8], bj + 2 * k8, k8);   // k8 = 0: part = product
                        if (X3) {
                            wgmma_m64n16k8_tf32(acs[j], ah[k8], bj + lo_rows + 2 * k8, 1);   // a_hi * w_lo
                            wgmma_m64n16k8_tf32(acs[j], al[k8], bj + 2 * k8, 1);             // a_lo * w_hi
                        }
                    }
                    wgmma_commit();
                    wgmma_wait0();
                    reg_fence(part);
                    if (X3) reg_fence(acs[j]);
#pragma unroll
                    for (int i = 0; i < 8; ++i) acc[j][i] += part[i];
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == a.stages) {
                stage = 0;
                phase ^= 1;
            }
        }
        // epilogue: this thread holds rows ra, ra + 8 and columns 16 j + 8 h + 2 t4 (+1)
        const int tx = mt % tiles_x;
        const int ty = (mt / tiles_x) % tiles_y;
        const int n = mt / (tiles_x * tiles_y);
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
            const int m = ra + 8 * rh;
            const int yy = m / a.bx, xx = m - yy * a.bx;
            float* orow = a.out + (size_t)n * a.osn + (size_t)((ty * a.by + yy) * a.oy_mul + a.oy0) * a.osy +
                          (size_t)(tx * a.bx + xx) * a.osx;
#pragma unroll
            for (int j = 0; j < TG_NB; ++j) {
                if (j < nblk) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int i = 4 * h + 2 * rh;
                        const int c = 16 * j + 8 * h + 2 * t4;
                        float2 o = X3 ? make_float2(acs[j][i] + acc[j][i], acs[j][i + 1] + acc[j][i + 1])
                                      : make_float2(acc[j][i], acc[j][i + 1]);
                        if (a.bias) {
                            const float2 b = __ldg(reinterpret_cast<const float2*>(a.bias + c));
                            o.x += b.x; o.y += b.y;
                        }
                        if (a.relu) {
                            o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f);
                        }
                        *reinterpret_cast<float2*>(orow + c) = o;
                    }
                }
            }
        }
    }
}

static bool tg_pick_patch(int Hs, int Ws, int* bx, int* by) {
    for (int x = 128; x >= 1; x >>= 1) {
        const int y = 128 / x;
        if (x <= 256 && y <= 256 && Ws % x == 0 && Hs % y == 0) {
            *bx = x;
            *by = y;
            return true;
        }
    }
    return false;
}

static bool tg_encode_view(TcEncodeTiledFn enc, CUtensorMap* tm, const LfTcgView& v, int N, int Kc, int bx, int by) {
    // (ci:32, cblk:Kc/32, x, y, n) with the view's element strides
    cuuint64_t dims[5] = {32, (cuuint64_t)(Kc / 32), (cuuint64_t)v.W, (cuuint64_t)v.H, (cuuint64_t)N};
    cuuint64_t strides[4] = {128, (cuuint64_t)v.sx * 4, (cuuint64_t)v.sy * 4, (cuuint64_t)v.sn * 4};
    cuuint32_t box[5] = {32, 1, (cuuint32_t)bx, (cuuint32_t)by, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(v.ptr), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace lf

using namespace lf;

extern "C" int lf_conv_tcg_supported(int N, int Hs, int Ws, int Kc, int Ng) {
    int bx, by;
    if (N <= 0 || Kc < 32 || Kc % 32 != 0 || Kc > 256 || Ng < 16 || Ng % 16 != 0 || Ng > 128) return 0;
    if (!tg_pick_patch(Hs, Ws, &bx, &by)) return 0;
    return tc_get_encode_fn() != nullptr ? 1 : 0;
}

extern "C" int lf_conv_tcg(const LfConvTcgArgs* args, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!args) return LF_ERR_INVALID_ARGUMENT;
    const LfConvTcgArgs& p = *args;
    LF_REQUIRE(p.a[0].ptr && p.wg && p.out && p.ntaps >= 1 && p.ntaps <= TG_MAXT);
    if (!lf_conv_tcg_supported(p.N, p.Hs, p.Ws, p.Kc, p.Ng)) return LF_ERR_UNSUPPORTED;
    LF_REQUIRE(p.osx % 4 == 0 && p.osy % 4 == 0 && p.osn % 4 == 0);
    TcEncodeTiledFn enc = tc_get_encode_fn();
    TgArgs a{};
    tg_pick_patch(p.Hs, p.Ws, &a.bx, &a.by);
    a.out = p.out; a.bias = p.bias; a.relu = p.relu;
    a.osn = p.osn; a.osy = p.osy; a.osx = p.osx; a.oy_mul = p.oy_mul; a.oy0 = p.oy0;
    a.N = p.N; a.Hs = p.Hs; a.Ws = p.Ws;
    a.kchunks = p.Kc / 32; a.Ng = p.Ng; a.ntaps = p.ntaps;
    bool two = false;
    for (int t = 0; t < p.ntaps; ++t) {
        LF_REQUIRE(p.map[t] == 0 || p.map[t] == 1);
        a.map[t] = p.map[t]; a.dy[t] = p.dy[t]; a.dx[t] = p.dx[t];
        two = two || p.map[t] == 1;
    }
    LF_REQUIRE(!two || p.a[1].ptr);
    LF_REQUIRE(p.precision == 0 || p.precision == 1);
    const bool x3 = p.precision == 1;
    const int nb = x3 ? 2 * p.Ng : p.Ng;   // rows of the weight chunk: W, or W_hi | W_lo
    a.stage_bytes = TG_A_BYTES + nb * 128;
    int stages = (TG_SMEM_LIMIT - 1024 - 256) / a.stage_bytes;
    if (stages > TG_MAX_STAGES) stages = TG_MAX_STAGES;
    a.stages = stages;
    a.total_tiles = p.N * (p.Hs / a.by) * (p.Ws / a.bx);

    CUtensorMap tmA0, tmA1, tmB;
    if (!tg_encode_view(enc, &tmA0, p.a[0], p.N, p.Kc, a.bx, a.by)) return LF_ERR_CUDA;
    if (!tg_encode_view(enc, &tmA1, two ? p.a[1] : p.a[0], p.N, p.Kc, a.bx, a.by)) return LF_ERR_CUDA;
    {
        // weights [Ng][ntaps*Kc] (K contiguous); 3xTF32: [2][Ng][ntaps*Kc] = hi rows, then lo rows, one box of 2*Ng rows
        const int K = p.ntaps * p.Kc;
        cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)nb};
        cuuint64_t strides[1] = {(cuuint64_t)K * 4};
        cuuint32_t box[2] = {32, (cuuint32_t)nb};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(p.wg), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return LF_ERR_CUDA;
    }
    const int sms = device_sms();
    const int grid = a.total_tiles < sms ? a.total_tiles : sms;
    const int smem_bytes = 1024 + a.stages * a.stage_bytes + 256;
    cudaError_t e = x3 ? cudaFuncSetAttribute(conv_tcg_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TG_SMEM_LIMIT)
                       : cudaFuncSetAttribute(conv_tcg_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TG_SMEM_LIMIT);
    if (e != cudaSuccess) { set_last_cuda_error(e); return LF_ERR_CUDA; }
    if (x3) lf_launch(conv_tcg_kernel<true>, grid, TG_THREADS, smem_bytes, stream, tmA0, tmA1, tmB, a);
    else lf_launch(conv_tcg_kernel<false>, grid, TG_THREADS, smem_bytes, stream, tmA0, tmA1, tmB, a);
    return check_launch();
}
