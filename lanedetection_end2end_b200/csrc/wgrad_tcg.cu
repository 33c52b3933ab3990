// Tensor-core weight gradients (Hopper, sm_90a), one wgmma kernel for every convolution of the network:
//
//     D[blk*32 + c][n] = sum_{img,y,x} A_{map[blk]}(img, y + dy[blk], x + dx[blk], cblk[blk]*32 + c) * B(img, y, x, n)
//
// i.e. one 32-channel block of one tap per `blk` (up to 24 blocks), n < Nn (multiple of 32, <= 128), over strided NHWC
// views.  Its one entry point, lf_wgrad_tcg, takes the block table from the host (ops_net.run_wgrad_tcg) for
//  * the resolution-changing layers (3x3 stride-2 Conv2d of DownsamplerBlock, 3x3 stride-2 ConvTranspose2d of
//    UpsamplerBlock; BP/Networks/ERFNet.py:15,101) on the pair-pixel / row-parity views of conv_tcg.cu, and the
//    Classification heads;
//  * the factorised 3-tap convolutions (C in {64,128}; C = 16 on the super-pixel view), dW[t][ci][co] = block
//    t*C/32 + cb of X shifted by tap t against dY -- the partial layout [3][C][C] is the block layout above.
// The K dimension of these GEMMs is the pixel index, so both operands lie MN-major in the NHWC boxes TMA loads.  wgmma
// takes A (rows = x-channels, k = pixels) from registers, which the threads load from the swizzled box like any other
// fragment; it reads TF32 B only K-major from shared memory, so the dY boxes are transposed in shared memory first.
//
// One CTA = one pixel range (split K; blockIdx.x) x one pair of blocks (64 rows of D = one m64 tile; blockIdx.y), so
// every block list, odd ones included, keeps all MMA warps busy.  Stage = [B boxes: Nn/32 x (32 px x 32 ch)][the two A
// boxes of the pair], 128B-swizzled; TMA zero-fills out-of-image pixels (conv padding).  Warp 8 is the TMA producer;
// warps 0-7 form two consumer warpgroups of NW = wgt_cols(Nn) output columns each.  Nn <= 64: both own all columns and
// take alternate stages (one wgmma of N = Nn per k8 instead of two of Nn/2: the kernel is bound by wgmma issue, not by
// tensor-core FLOPs), and warpgroup 1 hands its sums to warpgroup 0 at the end (fixed order).  Nn = 96 / 128: each owns
// half the columns and takes every stage.  Per stage, a warpgroup
//  * transposes its columns of the stage's dY boxes into a K-major, 128B-swizzled [NW x 32 px] tile (the layout TMA
//    would write for K-major data; 3xTF32: a hi tile and a lo tile, every element split once per CTA), double-buffered
//    so that one stage's stores never meet the previous stage's wgmma reads;
//  * loads the m64k8 A fragments of the pair (the rows of warp w come from block w/2) and issues wgmma m64nNWk8.  Each
//    stage's 32 pixels of the large term are summed by the tensor core from zero and added to the fp32 register sum
//    with FADD (the tensor core's accumulation drifts further than an FFMA chain over 10^4+ pixels); 3xTF32
//    (tc_ptx.cuh): every product is a_hi*b_hi + (a_hi*b_lo + a_lo*b_hi), the correction terms accumulated on the tensor
//    core and added in the epilogue.
// BF16 (precision 2): an m64k16 A register packs two pixels of one channel (two LDS from two box rows); the transposition
// writes bf16 pixel pairs into a 64B-swizzled K-major [NW x 32 px] tile, one 32-bit store each after lane pairs swap half
// their columns.  BF16 wgmma could read B MN-major (imm-trans-b = 1) and skip the transposition, but the K-major tile
// keeps one B layout and descriptor (wgmma_desc_sw64) for all three tensor-core kernels; double-buffering and the proxy
// fence are unchanged.  Two wgmma m64nNWk16 per stage.
// BF16 with a bf16 A view (template ABF, LfWgradTcgArgs.a_dtype = LF_BF16): the A boxes are [32 px x 32 ch] bf16,
// 64-byte rows, 64B-swizzled (half the bytes), and an A register is two 16-bit LDS of the ready values -- the bits the
// fp32 path packs from an fp32 copy of the same values, so the same results.  B stays fp32 and keeps its transposition.
// The next stage's fragments are not loaded while a stage's wgmma runs: ptxas then reuses the A registers the running
// wgmma still reads.  Every CTA writes its slice [64 rows][Nn] of one partial; lf_wgrad_reduce sums them in fixed order.
#include <cuda.h>

#include "lf_common.cuh"
#include "tc_ptx.cuh"

namespace lf {

constexpr int WG_THREADS = 288;              // two consumer warpgroups + the TMA warp
constexpr int WG_KP = 32;                    // pixels per stage
constexpr int WG_BOX = WG_KP * 128;          // one [32 px x 32 ch] box = 4 KB
constexpr int WG_MAXB = LF_WGRAD_TCG_MAX_BLOCKS;
constexpr int WG_MAX_STAGES = 8;
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

// B columns per consumer warpgroup for Nn B columns: Nn itself (the warpgroups take alternate stages) up to 64; above,
// three m64nNn accumulator sets would not fit the 168 registers a thread has here (each warpgroup takes half the columns)
constexpr int wgt_cols(int nn) { return nn <= 64 ? nn : nn / 2; }
// shared memory of one warpgroup's transposed B tiles: [2 buffers][hi (, lo)] x [cols x 32 px].  bf16 tiles are half the
// size, but the region keeps the TF32 size: warpgroup 1 hands its cols/2 fp32 sums per thread over through it at the end.
constexpr int wgt_wg_bytes(int nn, int prec) { return 2 * (prec == TC_X3 ? 2 : 1) * wgt_cols(nn) * 128; }
constexpr int wgt_bt_bytes(int nn, int prec) { return 2 * wgt_wg_bytes(nn, prec); }
// bytes of one A box: fp32, or bf16 (ABF)
constexpr int wgt_a_box(bool abf) { return abf ? WG_BOX / 2 : WG_BOX; }

template <int NN, int P, bool ABF>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_tcg_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                 const __grid_constant__ CUtensorMap tmB, const WgtArgs a) {
    static_assert(!ABF || P == TC_BF16, "a bf16 A view needs the BF16 kernel");
    constexpr bool X3 = P == TC_X3, BF = P == TC_BF16;
    constexpr int A_BOX = wgt_a_box(ABF);
    constexpr int NW = wgt_cols(NN);                    // B columns per warpgroup = wgmma N
    constexpr bool KSPLIT = NW == NN;                   // warpgroups split the stages, not the columns
    constexpr int BT_TILE = NW * (BF ? 64 : 128);       // one K-major [NW x 32 px] tile (TF32: 1024-, bf16: 512-byte multiple)
    constexpr int BT_SET = (X3 ? 2 : 1) * BT_TILE;      // hi tile, then lo tile
    constexpr int BT_WG = wgt_wg_bytes(NN, P);          // one warpgroup's region (two sets, or the final hand-over)
    pdl_trigger();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* bt = smem + (size_t)a.stages * a.stage_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(bt + wgt_bt_bytes(NN, P));
    uint64_t* empty = full + WG_MAX_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int per = (a.total_patches + gridDim.x - 1) / gridDim.x;
    const int p_begin = blockIdx.x * per;
    const int p_end = min(a.total_patches, p_begin + per);
    const int tiles_x = a.Ws / a.bx, tiles_y = a.Hs / a.by;
    const int blk0 = 2 * blockIdx.y;                  // first block of this CTA's pair
    const int na = min(2, a.nblocks - blk0);          // blocks in the pair

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA0);
        tma_prefetch_desc(&tmA1);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < a.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], KSPLIT ? 4 : 8);   // one arrive per MMA warp that reads the stage
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
                mbar_arrive_expect_tx(&full[stage], a.nb_b * WG_BOX + na * A_BOX);
                for (int cb = 0; cb < a.nb_b; ++cb) tma_load_5d(&tmB, &full[stage], st + cb * WG_BOX, 0, cb, x0, y0, n);
                for (int i = 0; i < na; ++i) {
                    const int b = blk0 + i;
                    tma_load_5d(a.map[b] ? &tmA1 : &tmA0, &full[stage], st + a.nb_b * WG_BOX + i * A_BOX, 0, a.cblk[b], x0 + a.dx[b],
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

    // consumer warpgroup wg, warp wl: D rows 16*wl + g (+8) = channel 16*(wl & 1) + g (+8) of block blk0 + (wl >> 1),
    // columns [c0, c0 + NW); KSPLIT: warpgroup wg takes the stages p_begin + wg, p_begin + wg + 2, ...
    const int wg = warp >> 2, wl = warp & 3;
    const int g = lane >> 2, t4 = lane & 3;
    const bool rows_ok = (wl >> 1) < na;   // false: the second block of an odd list's last pair (A = 0, not stored)
    const int arow = 16 * (wl & 1) + g;
    const int c0 = KSPLIT ? 0 : wg * NW;
    const uint32_t bt_wg = smem_u32(bt) + wg * BT_WG;
    float acc[NW / 2], part[NW / 2], acs[NW / 2];   // running sum; one stage's large term; 3xTF32 correction terms
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[i] = part[i] = acs[i] = 0.f;
    uint32_t buf = 0;
    for (int p = p_begin + (KSPLIT ? wg : 0); p < p_end; p += (KSPLIT ? 2 : 1)) {
        const int j = p - p_begin;
        const int stage = j % a.stages;
        mbar_wait(&full[stage], (j / a.stages) & 1);
        const uint32_t st = smem_u32(smem) + stage * a.stage_bytes;
        // A fragments (a[0..3] = A[arow][k0], A[arow + 8][k0], A[arow][k0 + 4], A[arow + 8][k0 + 4], A[c][k] = X[px k][ch c])
        // bf16 (m64k16): register q of step kk holds pixels k0, k0 + 1 (k0 = 16 kk + 2 t4, + 8 for q >= 2) of channel
        // arow (+ 8 for odd q) = two LDS from two box rows; av[kk][q] / av[kk][4 + q] are the low / high halves
        float av[WG_KP / 8][4];
        uint32_t ah[WG_KP / 8][4], al[WG_KP / 8][4];
        const uint32_t abox = st + a.nb_b * WG_BOX + (wl >> 1) * A_BOX;
        if constexpr (ABF) {
#pragma unroll
            for (int kk = 0; kk < WG_KP / 16; ++kk)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int k0 = 16 * kk + 2 * t4 + 8 * (q >> 1), r = arow + 8 * (q & 1);
                    ah[kk][q] = rows_ok ? lds_u16(abox + sw64_off(k0, r)) | (lds_u16(abox + sw64_off(k0 + 1, r)) << 16) : 0u;
                }
        } else if constexpr (BF) {
#pragma unroll
            for (int kk = 0; kk < WG_KP / 16; ++kk)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int k0 = 16 * kk + 2 * t4 + 8 * (q >> 1), r = arow + 8 * (q & 1);
                    av[2 * kk][q] = rows_ok ? lds_f32(abox + sw128_off(k0, r)) : 0.f;
                    av[2 * kk + 1][q] = rows_ok ? lds_f32(abox + sw128_off(k0 + 1, r)) : 0.f;
                }
        } else {
#pragma unroll
            for (int k8 = 0; k8 < WG_KP / 8; ++k8) {
                const int k0 = 8 * k8 + t4;
                av[k8][0] = rows_ok ? lds_f32(abox + sw128_off(k0, arow)) : 0.f;
                av[k8][1] = rows_ok ? lds_f32(abox + sw128_off(k0, arow + 8)) : 0.f;
                av[k8][2] = rows_ok ? lds_f32(abox + sw128_off(k0 + 4, arow)) : 0.f;
                av[k8][3] = rows_ok ? lds_f32(abox + sw128_off(k0 + 4, arow + 8)) : 0.f;
            }
        }
        // transpose: warp wl takes the 4-column chunks q = wl + 4i of this warpgroup's columns, lane = pixel.  Reads are
        // one 16-byte chunk per lane, writes one column (32 pixels = one swizzled 128-byte row): both conflict-free.
        const uint32_t bhi = bt_wg + buf * BT_SET;
#pragma unroll
        for (int i = 0; i < NW / 16; ++i) {
            const int q = wl + 4 * i;
            const int n = c0 + 4 * q;   // first B column of the chunk
            const float4 v4 = lds_f32x4(st + (n >> 5) * WG_BOX + sw128_off(lane, n & 31));
            const float v[4] = {v4.x, v4.y, v4.z, v4.w};
            if constexpr (BF) {
                // a bf16 pair of pixels (2m, 2m + 1) per 32-bit store: lane pairs swap half their columns, the even lane
                // then stores columns 0, 1 of the chunk and the odd lane columns 2, 3, at pixel pair m = lane / 2
                const bool odd = lane & 1;
                const float r0 = __shfl_xor_sync(0xffffffffu, odd ? v[0] : v[2], 1);
                const float r1 = __shfl_xor_sync(0xffffffffu, odd ? v[1] : v[3], 1);
                const int e0 = odd ? 2 : 0;
                sts_u32(bhi + sw64_off(4 * q + e0, lane & ~1), odd ? pack_bf16x2(r0, v[2]) : pack_bf16x2(v[0], r0));
                sts_u32(bhi + sw64_off(4 * q + e0 + 1, lane & ~1), odd ? pack_bf16x2(r1, v[3]) : pack_bf16x2(v[1], r1));
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const uint32_t off = sw128_off(4 * q + e, lane);
                    if (X3) {
                        uint32_t hi, lo;
                        tf32_split(v[e], hi, lo);
                        sts_u32(bhi + off, hi);
                        sts_u32(bhi + BT_TILE + off, lo);
                    } else {
                        sts_u32(bhi + off, tf32_rna(v[e]));
                    }
                }
            }
        }
#pragma unroll
        for (int k8 = 0; k8 < WG_KP / 8; ++k8)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (BF) {
                    if (!ABF && k8 < WG_KP / 16) ah[k8][q] = pack_bf16x2(av[2 * k8][q], av[2 * k8 + 1][q]);
                } else if (X3) {
                    tf32_split(av[k8][q], ah[k8][q], al[k8][q]);
                } else {
                    ah[k8][q] = tf32_rna(av[k8][q]);
                }
            }
        fence_proxy_async_smem();
        named_bar_sync(1 + wg, 128);   // the warpgroup's B tiles are complete
        const uint64_t bd = BF ? wgmma_desc_sw64(bhi) : wgmma_desc_sw128(bhi);
        wgmma_fence();
        if constexpr (BF) {
#pragma unroll
            for (int kk = 0; kk < WG_KP / 16; ++kk) wgmma_m64k16_bf16<NW>(part, ah[kk], bd + 2 * kk, kk);
        } else {
#pragma unroll
            for (int k8 = 0; k8 < WG_KP / 8; ++k8) {
                wgmma_m64k8_tf32<NW>(part, ah[k8], bd + 2 * k8, k8);   // k8 = 0: part = product (previous stage dropped)
                if (X3) {
                    wgmma_m64k8_tf32<NW>(acs, ah[k8], bd + (BT_TILE >> 4) + 2 * k8, 1);   // a_hi * b_lo
                    wgmma_m64k8_tf32<NW>(acs, al[k8], bd + 2 * k8, 1);                    // a_lo * b_hi
                }
            }
        }
        wgmma_commit();
        // the stage's boxes have been read into registers and B tiles: hand them back to the producer
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        wgmma_wait0();
        reg_fence(part);
        if (X3) reg_fence(acs);
#pragma unroll
        for (int i = 0; i < NW / 2; ++i) acc[i] += part[i];
        buf ^= 1;
    }
#pragma unroll
    for (int i = 0; i < NW / 2; ++i)
        if (X3) acc[i] = acs[i] + acc[i];   // small terms first
    if (KSPLIT) {
        // warpgroup 1 hands its sums to warpgroup 0 through its own (now idle) B buffers, same fragment order; the two
        // halves are added in a fixed order
        float* xfer = reinterpret_cast<float*>(bt + BT_WG) + (threadIdx.x & 127) * (NW / 2);
        if (wg == 1) {
#pragma unroll
            for (int i = 0; i < NW / 2; i += 2) *reinterpret_cast<float2*>(xfer + i) = make_float2(acc[i], acc[i + 1]);
        }
        named_bar_sync(3, 256);
        if (wg == 1) return;
#pragma unroll
        for (int i = 0; i < NW / 2; i += 2) {
            const float2 o = *reinterpret_cast<const float2*>(xfer + i);
            acc[i] += o.x;
            acc[i + 1] += o.y;
        }
    }
    if (!rows_ok) return;
    float* dst = a.partial + ((size_t)blockIdx.x * a.nblocks * 32 + (size_t)blk0 * 32) * a.Nn + c0;
#pragma unroll
    for (int i = 0; i < NW / 2; i += 2) {
        const int r = 16 * wl + g + 8 * ((i >> 1) & 1);
        const int c = 8 * (i >> 2) + 2 * t4;
        *reinterpret_cast<float2*>(dst + (size_t)r * a.Nn + c) = make_float2(acc[i], acc[i + 1]);
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

static bool wgt_encode(TcEncodeTiledFn enc, CUtensorMap* tm, const LfTcgView& v, int N, int C, int bx, int by, bool bf16 = false) {
    return tc_encode_view(enc, tm, v.ptr, N, v.H, v.W, C, v.sx, v.sy, v.sn, bx, by, bf16);
}

// split-K slices for `patches` pixel patches and `nblocks` blocks: at least `min_per` patches per slice, and at most as
// many slices as fill the SMs once with one CTA per (slice, pair of blocks)
static int wgt_split(long long patches, int min_per, int nblocks) {
    long long s = patches / min_per;
    long long cap = device_sms() / ((nblocks + 1) / 2);
    if (cap < 1) cap = 1;
    if (s > cap) s = cap;
    return (int)(s < 1 ? 1 : s);
}

static int wgt_ctas(int N, int Hs, int Ws, int Ka, int Nn, int nblocks, int min_patches) {
    int bx, by;
    if (N <= 0 || Ka % 32 != 0 || Ka < 32 || Nn % 32 != 0 || Nn < 32 || Nn > 128 || nblocks < 1 || nblocks > WG_MAXB) return 0;
    if (min_patches < 1 || !wgt_pick_patch(Hs, Ws, &bx, &by)) return 0;
    if (!tc_get_encode_fn()) return 0;
    return wgt_split((long long)N * (Hs / by) * (Ws / bx), min_patches, nblocks);
}

template <int NN, int P, bool ABF = false>
static cudaError_t wgt_launch(dim3 grid, int smem_bytes, cudaStream_t stream, const CUtensorMap& tmA0, const CUtensorMap& tmA1,
                              const CUtensorMap& tmB, const WgtArgs& a) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_tcg_kernel<NN, P, ABF>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e != cudaSuccess) return e;
    return lf_launch(wgrad_tcg_kernel<NN, P, ABF>, grid, WG_THREADS, smem_bytes, stream, tmA0, tmA1, tmB, a);
}

template <int P>
static cudaError_t wgt_launch_nn(dim3 grid, int smem_bytes, cudaStream_t stream, const CUtensorMap& tmA0, const CUtensorMap& tmA1,
                                 const CUtensorMap& tmB, const WgtArgs& a) {
    switch (a.Nn) {
        case 32: return wgt_launch<32, P>(grid, smem_bytes, stream, tmA0, tmA1, tmB, a);
        case 64: return wgt_launch<64, P>(grid, smem_bytes, stream, tmA0, tmA1, tmB, a);
        case 96: return wgt_launch<96, P>(grid, smem_bytes, stream, tmA0, tmA1, tmB, a);
        default: return wgt_launch<128, P>(grid, smem_bytes, stream, tmA0, tmA1, tmB, a);
    }
}

// a: A views and their block table, b: the B view; the launch of the generic kernel
static int wgt_run(const LfTcgView* av, const LfTcgView& bv, int N, int Hs, int Ws, int Ka, int Nn, int nblocks, const int* map,
                   const int* dy, const int* dx, const int* cblk, float* partial, int nsplit, int prec, cudaStream_t stream,
                   bool abf) {
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
    // a bf16 A view: the 3-tap weight gradients of the bf16 mode (Nn = C)
    if (abf && (prec != TC_BF16 || !(Nn == 64 || Nn == 128))) return LF_ERR_UNSUPPORTED;
    const int fixed = 1024 + wgt_bt_bytes(Nn, prec) + 256;   // alignment slack + transposed B tiles + barriers
    a.stage_bytes = a.nb_b * WG_BOX + 2 * wgt_a_box(abf);   // a multiple of 4 KB: every stage keeps the 1024-byte swizzle phase
    int stages = (WG_SMEM_LIMIT - fixed) / a.stage_bytes;
    if (stages > WG_MAX_STAGES) stages = WG_MAX_STAGES;
    a.stages = stages;
    a.total_patches = N * (Hs / a.by) * (Ws / a.bx);

    CUtensorMap tmA0, tmA1, tmB;
    if (!wgt_encode(enc, &tmA0, av[0], N, Ka, a.bx, a.by, abf)) return LF_ERR_CUDA;
    if (!wgt_encode(enc, &tmA1, two ? av[1] : av[0], N, Ka, a.bx, a.by, abf)) return LF_ERR_CUDA;
    if (!wgt_encode(enc, &tmB, bv, N, Nn, a.bx, a.by)) return LF_ERR_CUDA;
    const int smem_bytes = fixed + a.stages * a.stage_bytes;
    const dim3 grid(nsplit, (nblocks + 1) / 2);
    const cudaError_t e = abf               ? (Nn == 64 ? wgt_launch<64, TC_BF16, true>(grid, smem_bytes, stream, tmA0, tmA1, tmB, a)
                                                        : wgt_launch<128, TC_BF16, true>(grid, smem_bytes, stream, tmA0, tmA1, tmB, a))
                          : prec == TC_X3   ? wgt_launch_nn<TC_X3>(grid, smem_bytes, stream, tmA0, tmA1, tmB, a)
                          : prec == TC_BF16 ? wgt_launch_nn<TC_BF16>(grid, smem_bytes, stream, tmA0, tmA1, tmB, a)
                                            : wgt_launch_nn<TC_TF32>(grid, smem_bytes, stream, tmA0, tmA1, tmB, a);
    if (e != cudaSuccess) { set_last_cuda_error(e); return LF_ERR_CUDA; }
    return check_launch();
}

}  // namespace lf

using namespace lf;

// number of split-K slices (= partials) lf_wgrad_tcg will use, 0 = unsupported
extern "C" int lf_wgrad_tcg_ctas(int N, int Hs, int Ws, int Ka, int Nn, int nblocks, int min_patches) {
    return wgt_ctas(N, Hs, Ws, Ka, Nn, nblocks, min_patches);
}

extern "C" int lf_wgrad_tcg(const LfWgradTcgArgs* args, lf_stream_t stream_) {
    if (!args) return LF_ERR_INVALID_ARGUMENT;
    const LfWgradTcgArgs& p = *args;
    LF_REQUIRE(p.a[0].ptr && p.b.ptr && p.partial && p.nctas >= 1);
    LF_REQUIRE(p.precision == TC_TF32 || p.precision == TC_X3 || p.precision == TC_BF16);
    LF_REQUIRE(p.a_dtype == LF_F32 || p.a_dtype == LF_BF16);
    if (!wgt_ctas(p.N, p.Hs, p.Ws, p.Ka, p.Nn, p.nblocks, 1)) return LF_ERR_UNSUPPORTED;
    return wgt_run(p.a, p.b, p.N, p.Hs, p.Ws, p.Ka, p.Nn, p.nblocks, p.map, p.dy, p.dx, p.cblk, p.partial, p.nctas, p.precision,
                   reinterpret_cast<cudaStream_t>(stream_), p.a_dtype == LF_BF16);
}
