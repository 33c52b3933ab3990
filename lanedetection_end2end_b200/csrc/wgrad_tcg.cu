// Tensor-core weight gradients (Hopper, sm_90a), one kernel for every convolution of the network:
//
//     D[blk*32 + c][n] = sum_{img,y,x} A_{map[blk]}(img, y + dy[blk], x + dx[blk], cblk[blk]*32 + c) * B(img, y, x, n)
//
// i.e. one 32-channel block of one tap per `blk` (up to 24 blocks), n < Nn (multiple of 32, <= 128), over strided NHWC
// views.  Its callers:
//  * lf_wgrad_tcg: the resolution-changing layers (3x3 stride-2 Conv2d of DownsamplerBlock, 3x3 stride-2 ConvTranspose2d
//    of UpsamplerBlock; BP/Networks/ERFNet.py:15,101) on the pair-pixel / row-parity views of conv_tcg.cu;
//  * lf_wgrad3_tc / lf_wgrad3_tc_x3: the factorised 3-tap convolutions (C in {64,128}), dW[t][ci][co] = block t*C/32 + cb
//    of X shifted by tap t against dY -- the partial layout [3][C][C] is the block layout above.
// The K dimension of these GEMMs is the pixel index, so both operands lie MN-major in the NHWC boxes.  wgmma reads TF32
// operands from shared memory only K-major, so the fragments are loaded by the threads from the swizzled TMA boxes and
// multiplied with mma.sync m16n8k8.
//
// One CTA = one pixel range (split K; blockIdx.x) x one group of four blocks (128 rows of D; blockIdx.y).  Stage =
// [B boxes: Nn/32 x (32 px x 32 ch)][A boxes of the group], 128B-swizzled, TMA zero-fills out-of-image pixels (conv
// padding); an mbarrier ring feeds 8 MMA warps (warp w: block w & 3, output columns half w >> 2), warp 8 is the TMA
// producer.  Every CTA writes its slice [128 rows][Nn] of one partial; lf_wgrad_reduce sums the partials in fixed order.
// precision 1 (3xTF32; tc_ptx.cuh): both operands split into hi / lo in registers, every product is
// a_hi*b_hi + (a_hi*b_lo + a_lo*b_hi), the correction terms accumulated apart and added at the end.
#include <cuda.h>

#include "lf_common.cuh"
#include "tc_ptx.cuh"

namespace lf {

constexpr int WG_THREADS = 288;
constexpr int WG_KP = 32;                    // pixels per stage
constexpr int WG_BOX = WG_KP * 128;          // one [32 px x 32 ch] box = 4 KB
constexpr int WG_MAXB = LF_WGRAD_TCG_MAX_BLOCKS;
constexpr int WG_MAX_STAGES = 6;
constexpr int WG_SMEM_LIMIT = 227 * 1024;

struct WgtArgs {
    float* partial;  // [nsplit][nblocks*32][Nn]
    int N, Hs, Ws;
    int bx, by;
    int nblocks, nb_b, Nn;   // A blocks, B blocks (Nn/32), B channels
    int map[WG_MAXB], dy[WG_MAXB], dx[WG_MAXB], cblk[WG_MAXB];
    int stages, stage_bytes;
    int total_patches;
};

template <bool X3>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_tcg_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                 const __grid_constant__ CUtensorMap tmB, const WgtArgs a) {
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)a.stages * a.stage_bytes);
    uint64_t* empty = full + WG_MAX_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int per = (a.total_patches + gridDim.x - 1) / gridDim.x;
    const int p_begin = blockIdx.x * per;
    const int p_end = min(a.total_patches, p_begin + per);
    const int tiles_x = a.Ws / a.bx, tiles_y = a.Hs / a.by;
    const int blk0 = 4 * blockIdx.y;                  // first block of this CTA's group
    const int na = min(4, a.nblocks - blk0);          // blocks in the group

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA0);
        tma_prefetch_desc(&tmA1);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < a.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);   // one arrive per MMA warp
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();   // everything above overlapped the previous kernel's tail; global memory is touched only from here on

    if (warp == 8) {
        // TMA producer: converged warp, elected lane issues
        const bool leader = elect_one();
        int stage = 0;
        uint32_t phase = 0;
        for (int p = p_begin; p < p_end; ++p) {
            const int tx = p % tiles_x;
            const int ty = (p / tiles_x) % tiles_y;
            const int n = p / (tiles_x * tiles_y);
            const int x0 = tx * a.bx, y0 = ty * a.by;
            mbar_wait(&empty[stage], phase ^ 1);
            if (leader) {
                uint8_t* st = smem + (size_t)stage * a.stage_bytes;
                mbar_arrive_expect_tx(&full[stage], (a.nb_b + na) * WG_BOX);
                for (int cb = 0; cb < a.nb_b; ++cb) tma_load_5d(&tmB, &full[stage], st + cb * WG_BOX, 0, cb, x0, y0, n);
                for (int i = 0; i < na; ++i) {
                    const int b = blk0 + i;
                    tma_load_5d(a.map[b] ? &tmA1 : &tmA0, &full[stage], st + (a.nb_b + i) * WG_BOX, 0, a.cblk[b], x0 + a.dx[b],
                                y0 + a.dy[b], n);
                }
            }
            if (++stage == a.stages) {
                stage = 0;
                phase ^= 1;
            }
        }
        return;
    }

    // MMA warps: block bi of the group (32 rows = two m16 tiles), columns [nh * Nn/2, (nh + 1) * Nn/2) = nt n8 tiles
    const int bi = warp & 3, nh = warp >> 2;
    const int g = lane >> 2, t4 = lane & 3;
    const int nt = a.Nn >> 4;
    const int n_base = nh * (a.Nn >> 1);
    const bool active = bi < na;
    float acc[2][8][4], acs[2][8][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[mi][j][q] = acs[mi][j][q] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int p = p_begin; p < p_end; ++p) {
        mbar_wait(&full[stage], phase);
        const uint8_t* st = smem + (size_t)stage * a.stage_bytes;
        if (active) {
            const uint8_t* abox = st + (a.nb_b + bi) * WG_BOX;
#pragma unroll
            for (int k8 = 0; k8 < WG_KP / 8; ++k8) {
                const int k0 = 8 * k8 + t4;   // pixel rows k0, k0 + 4
                uint32_t ah[2][4], al[2][4];
#pragma unroll
                for (int mi = 0; mi < 2; ++mi) {
                    const int r = 16 * mi + g;
                    const float v[4] = {*reinterpret_cast<const float*>(abox + sw128_off(k0, r)),
                                        *reinterpret_cast<const float*>(abox + sw128_off(k0, r + 8)),
                                        *reinterpret_cast<const float*>(abox + sw128_off(k0 + 4, r)),
                                        *reinterpret_cast<const float*>(abox + sw128_off(k0 + 4, r + 8))};
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        if (X3) {
                            tf32_split(v[q], ah[mi][q], al[mi][q]);
                        } else {
                            ah[mi][q] = tf32_rna(v[q]);
                        }
                    }
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (j < nt) {
                        const int nn = n_base + 8 * j + g;
                        const uint8_t* bbox = st + (nn >> 5) * WG_BOX;
                        const float w0 = *reinterpret_cast<const float*>(bbox + sw128_off(k0, nn & 31));
                        const float w1 = *reinterpret_cast<const float*>(bbox + sw128_off(k0 + 4, nn & 31));
                        uint32_t bh[2], bl[2];
                        if (X3) {
                            tf32_split(w0, bh[0], bl[0]);
                            tf32_split(w1, bh[1], bl[1]);
                        } else {
                            bh[0] = tf32_rna(w0); bh[1] = tf32_rna(w1);
                        }
#pragma unroll
                        for (int mi = 0; mi < 2; ++mi) {
                            mma_m16n8k8_tf32(acc[mi][j], ah[mi], bh);
                            if (X3) {
                                mma_m16n8k8_tf32(acs[mi][j], ah[mi], bl);
                                mma_m16n8k8_tf32(acs[mi][j], al[mi], bh);
                            }
                        }
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        if (++stage == a.stages) {
            stage = 0;
            phase ^= 1;
        }
    }
    if (!active) return;
    float* dst = a.partial + ((size_t)blockIdx.x * a.nblocks * 32 + (size_t)(blk0 + bi) * 32) * a.Nn;
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j < nt) {
                const int c = n_base + 8 * j + 2 * t4;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = 16 * mi + g + 8 * h;
                    const float2 o = X3 ? make_float2(acs[mi][j][2 * h] + acc[mi][j][2 * h], acs[mi][j][2 * h + 1] + acc[mi][j][2 * h + 1])
                                        : make_float2(acc[mi][j][2 * h], acc[mi][j][2 * h + 1]);
                    *reinterpret_cast<float2*>(dst + (size_t)r * a.Nn + c) = o;
                }
            }
        }
}

static bool wgt_pick_patch(int Hs, int Ws, int* bx, int* by) {
    for (int x = WG_KP; x >= 1; x >>= 1) {
        const int y = WG_KP / x;
        if (Ws % x == 0 && Hs % y == 0) {
            *bx = x;
            *by = y;
            return true;
        }
    }
    return false;
}

static bool wgt_encode(TcEncodeTiledFn enc, CUtensorMap* tm, const LfTcgView& v, int N, int C, int bx, int by) {
    return tc_encode_view(enc, tm, v.ptr, N, v.H, v.W, C, v.sx, v.sy, v.sn, bx, by);
}

// split-K slices for `patches` pixel patches: at least `min_per` patches per slice, at most one slice per SM
static int wgt_split(long long patches, int min_per) {
    long long s = patches / min_per;
    const int sms = device_sms();
    if (s > sms) s = sms;
    return (int)(s < 1 ? 1 : s);
}

static int wgt_ctas(int N, int Hs, int Ws, int Ka, int Nn, int nblocks) {
    int bx, by;
    if (N <= 0 || Ka % 32 != 0 || Ka < 32 || Nn % 32 != 0 || Nn < 32 || Nn > 128 || nblocks < 1 || nblocks > WG_MAXB) return 0;
    if (!wgt_pick_patch(Hs, Ws, &bx, &by)) return 0;
    if (!tc_get_encode_fn()) return 0;
    return wgt_split((long long)N * (Hs / by) * (Ws / bx), 4);
}

// a: A views and their block table, b: the B view; the launch of the generic kernel
static int wgt_run(const LfTcgView* av, const LfTcgView& bv, int N, int Hs, int Ws, int Ka, int Nn, int nblocks, const int* map,
                   const int* dy, const int* dx, const int* cblk, float* partial, int nsplit, bool x3, cudaStream_t stream) {
    TcEncodeTiledFn enc = tc_get_encode_fn();
    if (!enc) return LF_ERR_UNSUPPORTED;
    WgtArgs a{};
    if (!wgt_pick_patch(Hs, Ws, &a.bx, &a.by)) return LF_ERR_UNSUPPORTED;
    a.partial = partial; a.N = N; a.Hs = Hs; a.Ws = Ws;
    a.nblocks = nblocks; a.Nn = Nn; a.nb_b = Nn / 32;
    bool two = false;
    for (int b = 0; b < nblocks; ++b) {
        LF_REQUIRE((map[b] == 0 || map[b] == 1) && cblk[b] >= 0 && cblk[b] < Ka / 32);
        a.map[b] = map[b]; a.dy[b] = dy[b]; a.dx[b] = dx[b]; a.cblk[b] = cblk[b];
        two = two || map[b] == 1;
    }
    LF_REQUIRE(!two || av[1].ptr);
    a.stage_bytes = (a.nb_b + 4) * WG_BOX;
    int stages = (WG_SMEM_LIMIT - 1024 - 256) / a.stage_bytes;
    if (stages > WG_MAX_STAGES) stages = WG_MAX_STAGES;
    a.stages = stages;
    a.total_patches = N * (Hs / a.by) * (Ws / a.bx);

    CUtensorMap tmA0, tmA1, tmB;
    if (!wgt_encode(enc, &tmA0, av[0], N, Ka, a.bx, a.by)) return LF_ERR_CUDA;
    if (!wgt_encode(enc, &tmA1, two ? av[1] : av[0], N, Ka, a.bx, a.by)) return LF_ERR_CUDA;
    if (!wgt_encode(enc, &tmB, bv, N, Nn, a.bx, a.by)) return LF_ERR_CUDA;
    const int smem_bytes = 1024 + a.stages * a.stage_bytes + 256;
    const dim3 grid(nsplit, (nblocks + 3) / 4);
    cudaError_t e = x3 ? cudaFuncSetAttribute(wgrad_tcg_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes)
                       : cudaFuncSetAttribute(wgrad_tcg_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e != cudaSuccess) { set_last_cuda_error(e); return LF_ERR_CUDA; }
    if (x3) lf_launch(wgrad_tcg_kernel<true>, grid, WG_THREADS, smem_bytes, stream, tmA0, tmA1, tmB, a);
    else lf_launch(wgrad_tcg_kernel<false>, grid, WG_THREADS, smem_bytes, stream, tmA0, tmA1, tmB, a);
    return check_launch();
}

}  // namespace lf

using namespace lf;

// number of split-K slices (= partials) lf_wgrad_tcg will use, 0 = unsupported
extern "C" int lf_wgrad_tcg_ctas(int N, int Hs, int Ws, int Ka, int Nn, int nblocks) { return wgt_ctas(N, Hs, Ws, Ka, Nn, nblocks); }
extern "C" int lf_wgrad_tcg_ctas_x3(int N, int Hs, int Ws, int Ka, int Nn, int nblocks) { return wgt_ctas(N, Hs, Ws, Ka, Nn, nblocks); }

extern "C" int lf_wgrad_tcg(const LfWgradTcgArgs* args, lf_stream_t stream_) {
    if (!args) return LF_ERR_INVALID_ARGUMENT;
    const LfWgradTcgArgs& p = *args;
    LF_REQUIRE(p.a[0].ptr && p.b.ptr && p.partial && p.nctas >= 1);
    LF_REQUIRE(p.precision == 0 || p.precision == 1);
    if (!wgt_ctas(p.N, p.Hs, p.Ws, p.Ka, p.Nn, p.nblocks)) return LF_ERR_UNSUPPORTED;
    return wgt_run(p.a, p.b, p.N, p.Hs, p.Ws, p.Ka, p.Nn, p.nblocks, p.map, p.dy, p.dx, p.cblk, p.partial, p.nctas, p.precision == 1,
                   reinterpret_cast<cudaStream_t>(stream_));
}

// ---- factorised 3-tap convolutions: partial[cta][t][ci][co] = blocks t*C/32 + cb of X shifted by tap t against dY
static int wgrad3_ctas(int N, int H, int W, int C, int min_per) {
    int bx, by;
    if (!(C == 64 || C == 128) || N <= 0) return 0;
    if (!wgt_pick_patch(H, W, &bx, &by)) return 0;
    if (!tc_get_encode_fn()) return 0;
    return wgt_split((long long)N * (H / by) * (W / bx), min_per);
}

static int wgrad3_run(const float* x, const float* dy, int N, int H, int W, int C, const int* tap_dy, const int* tap_dx,
                      float* partial, int nctas, bool x3, lf_stream_t stream_) {
    LF_REQUIRE(x && dy && partial && tap_dy && tap_dx && nctas >= 1);
    if (!(C == 64 || C == 128)) return LF_ERR_UNSUPPORTED;
    const LfTcgView xv{x, H, W, (long long)H * W * C, (long long)W * C, C};
    const LfTcgView gv{dy, H, W, (long long)H * W * C, (long long)W * C, C};
    const LfTcgView av[2] = {xv, xv};
    const int cbs = C / 32;
    int map[12], bdy[12], bdx[12], cblk[12];
    for (int t = 0; t < 3; ++t)
        for (int cb = 0; cb < cbs; ++cb) {
            const int b = t * cbs + cb;
            map[b] = 0; bdy[b] = tap_dy[t]; bdx[b] = tap_dx[t]; cblk[b] = cb;
        }
    return wgt_run(av, gv, N, H, W, C, C, 3 * cbs, map, bdy, bdx, cblk, partial, nctas, x3, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_wgrad3_tc_ctas(int N, int H, int W, int C) { return wgrad3_ctas(N, H, W, C, 4); }
extern "C" int lf_wgrad3_tc_x3_ctas(int N, int H, int W, int C) { return wgrad3_ctas(N, H, W, C, 8); }
extern "C" int lf_wgrad3_tc(const float* x, const float* dy, int N, int H, int W, int C, const int* tap_dy, const int* tap_dx,
                            float* partial, int nctas, lf_stream_t stream) {
    return wgrad3_run(x, dy, N, H, W, C, tap_dy, tap_dx, partial, nctas, false, stream);
}
extern "C" int lf_wgrad3_tc_x3(const float* x, const float* dy, int N, int H, int W, int C, const int* tap_dy, const int* tap_dx,
                               float* partial, int nctas, lf_stream_t stream) {
    return wgrad3_run(x, dy, N, H, W, C, tap_dy, tap_dx, partial, nctas, true, stream);
}
