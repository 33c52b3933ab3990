// Hopper (sm_90a) wgmma implicit-GEMM kernel for ERFNet's factorised 3-tap convolutions
// (non_bottleneck_1d: conv3x1 / conv1x3 with dilation, BP/Networks/ERFNet.py:29-37,44-53) and their input gradients,
// C in {64, 128}, NHWC fp32 activations, fp32 accumulate.  Three operand precisions (template P, tc_ptx.cuh TcPrec):
//  * TF32 (lf_conv1d_tc): operands rounded to TF32 (the arithmetic cuDNN uses for the reference's fp32 convs on
//    Ampere and later), one product per multiply;
//  * 3xTF32 (lf_conv1d_tc_x3, the library default): every fp32 operand is split a = a_hi + a_lo (tc_ptx.cuh) and each
//    product is a_hi*w_hi + (a_hi*w_lo + a_lo*w_hi) with fp32 accumulation -- as accurate as an fp32 FFMA chain.  The
//    weights arrive pre-split from the packer ([2][Cout][3C]: hi rows, then lo rows; both exact TF32 values).
//  * BF16 (lf_conv1d_tc_bf16): both operands rounded to bf16 (nearest even) -- the activations while their k16 fragments
//    are formed (pairs of adjacent channels, one 8-byte load each), the weights by the packer ([Cout][3C] bf16, 64-byte
//    rows, 64B-swizzled tiles of half the TF32 size: resident wherever the TF32 tiles are); products exact in fp32.
//    The activations may also arrive as bf16 (template ABF, LfConvTcArgs.in_dtype): the slab is then a bf16 TMA box of
//    64-byte rows, 64B-swizzled, and each fragment register is one 32-bit load of a ready channel pair -- the same
//    operand bits as rounding the fp32 copy, so the same results.  The BF16 epilogue can also store `out` as bf16
//    (nearest even, = torch's .to(torch.bfloat16); column sums / statistics are of the fp32 values) and read a bf16
//    `mask_src`: the ReLU outputs a non_bottleneck_1d block keeps only as convolution inputs and ReLU masks.
//  * FP8 (lf_conv1d_tc_fp8, inference only): e4m3 operands with fp32 scales.  The weights arrive quantised per output
//    channel ([Cout][3C] e4m3, 32-byte rows, 32B-swizzled [64 x 32] tiles of a quarter of the TF32 size) with their
//    dequantisation factors w_scale[co]; the activations are quantised per image while their k32 fragments are formed:
//    q = e4m3(v * inv[n]), inv[n] = 448 / x_amax[n] (4 adjacent channels per register: one 16-byte load from the fp32
//    slab or 8 bytes from the bf16 slab, two cvt.rn.satfinite.e4m3x2).  One k32 MMA per tap and 32-channel chunk.  The
//    epilogue computes, in this fp32 order, y = acc * (s_x[n] * w_scale[co]) + bias with s_x[n] = x_amax[n] / 448,
//    then the usual ReLU / residual steps, and reduces the per-image max |stored value| into out_amax[n] (a warp max,
//    one shared-memory atomicMax per warp, one global atomicMax per CTA and tile).  Every tile lies within one image.
//
//   out[n,y,x,co] = epi( sum_{t<3} sum_{ci} in[n, (y,x) + o_t, ci] * Wp[co][t*C + ci] )
//
// GEMM view per CTA tile: M = 128 pixels = TA positions along the conv axis x TB across it, N = 64 output channels
// (C = 128: two CTAs per tile, one per 64-channel half), K = 3*C.
//  * A, halo slab (default): ONE TMA box per 32-channel chunk, [(TA+2d) x TB pixels] x 32 channels, 128B-swizzled, cross
//    axis fastest.  The three taps are three views of the same slab, d*TB rows apart (a multiple of 8 rows, so every view
//    keeps the swizzle phase): the input crosses L2 -> SM (TA+2d)/TA times instead of 3 times.  Image borders (the conv
//    zero padding, any dilation) are TMA out-of-bounds fill.
//  * A, per tap (lf_conv1d_tc_set_variant(1), and any TF32 call the slab does not serve): one [128 px x 32 ch] box per
//    tap and chunk at the tap's offset; same kernel, the three views are three boxes.
//  * B: the weights of this CTA's 64 output channels, K-major 128B-swizzled [64 x 32] tiles (hi and lo tiles for 3xTF32).
//    Resident in shared memory for the whole persistent CTA when they leave room for two slab stages, else streamed
//    next to the slab of their 32-channel chunk.
//  * MMA: wgmma m64n64k8 TF32.  Two consumer warpgroups own 64 pixel rows each and take A and B from shared memory
//    through descriptors.  Once a stage has landed, the 256 consumer threads make one elementwise pass over its slab:
//    each word becomes its TF32 rounding in place and, for 3xTF32, the rounded remainder goes to the same offset of a
//    lo buffer outside the ring (two when shared memory allows, else one; else one laid over the staging tile), so
//    every tap view is a descriptor into the slab, 1024-byte aligned like the B tiles.  (BF16 keeps register A.)
//    Accumulators stay in registers: each tap's products are summed by the tensor core from zero and added to the
//    running fp32 sum with a rounded FADD (the tensor core's own accumulation does not round like IEEE adds); 3xTF32
//    keeps the sum of the two small correction terms apart and adds it in the epilogue (small terms first).
//  * Epilogue (both warpgroups): accumulators -> padded shared-memory staging tile -> warpgroup g walks 32-channel half g
//    row-major, 8 consecutive threads per pixel's 32 channels, so bias, ReLU, ReLU-backward mask (optionally formed
//    from the BatchNorm input x as fma(x, scale, shift) > 0), residual-gradient add, column sums / sums of squares (bias
//    gradient, BatchNorm statistics) and the output stores are coalesced 128-bit accesses.  The mask / residual operands
//    of a tile are loaded before its MMAs, so their latency hides behind them.
// Warps 0-7: consumers; warp 8: TMA producer (whole warp converged, one elected lane issues).
#include "lf_common.cuh"
#include "tc_ptx.cuh"

namespace lf {

constexpr int TC_BN = 64;                         // output channels per CTA
constexpr int TC_KCH = 32;                        // fp32 elements per 128-byte swizzle row
constexpr int TC_MAX_STAGES = 8;
constexpr int TC_THREADS = 288;
constexpr int TC_STG_LD = 32 + 4;                 // staging row stride in floats: a 32-channel half + bank spread
constexpr int TC_STG_BYTES = 128 * TC_STG_LD * 4; // 18 KB per half
constexpr int TC_ATOM = TC_BN * 128;              // one [64 out x 32 in] weight tile, 8 KB
constexpr int TC_SMEM_LIMIT = 227 * 1024;
constexpr int TC_FIXED_SMEM = 1024 + 2 * TC_STG_BYTES + 256;   // alignment slack + staging + barriers
// bytes of one [64 out x 32 in] weight tile in precision P: TF32, TF32 hi + lo, bf16 (64-byte rows, 64B-swizzled) or
// e4m3 (32-byte rows, 32B-swizzled)
constexpr int tc_w_atom(int P) {
    return P == TC_X3 ? 2 * TC_ATOM : P == TC_BF16 ? TC_ATOM / 2 : P == TC_FP8 ? TC_ATOM / 4 : TC_ATOM;
}
// the precisions whose kernels read bf16 activations / write bf16 outputs
constexpr bool tc_takes_bf16(int P) { return P == TC_BF16 || P == TC_FP8; }

static int g_tc_variant = 2;  // 2 = halo slab, 1 = one box per tap

struct TcArgs {
    float* out;
    const float* bias;
    const float* mask_src;
    const float* add_src;
    const float* add_mask;
    float* colsum_partial;    // [gridDim.x / n_halves][Ctot] per-CTA column sums of the output, or NULL
    double* stats_partial;    // [gridDim.x / n_halves][2][Ctot] per-CTA sum and sum of squares (BatchNorm), or NULL
    const float* mask_scale;  // non-NULL (with mask_shift): mask_src is a PRE-activation x; the ReLU mask bit is
    const float* mask_shift;  // fma(x, scale[c], shift[c]) > 0 and the second statistic = sum out*x  (BatchNorm backward)
    int N, H, W, Ctot;
    int vertical;             // pixel order of a tile: 1 = along-axis is y (TB pixels along x fastest), 0 = along-axis is x
    int TA, TB, tb_shift;     // tile extent along / across the conv axis (TA*TB = 128), log2(TB)
    int tiles_a, tiles_b;
    int nloads, load_rows;    // TMA boxes per stage (1 slab or 3 tap boxes) and rows of each
    int load_a[3], load_b[3]; // box origin relative to the tile origin (along, across)
    int tap_row[3];           // first stage row of the view used by weight slot t
    int relu;                 // bit 0: ReLU on conv + bias (before mask / add); bit 1: ReLU after the residual add
    int n_halves, total_m_tiles;
    int stages, stage_bytes, a_bytes;   // a stage = a_bytes of activations [+ the three weight tiles of its chunk]
    // 3xTF32: n_lo (1 or 2) lo slab buffers in the lo_bytes after the ring, or (lo_stg = 1) one that ends where the
    // staging tile ends: it overlaps the staging tile and whatever it needs beyond it is the lo_bytes before it
    int n_lo, lo_stg, lo_bytes;
    int out_bf16, mask_bf16;  // BF16 and FP8 kernels only: `out` / `mask_src` hold bf16
    const float* x_amax;      // FP8 only: [N] per-image max |in|, [Ctot] per-channel weight scales, [N] per-image max
    const float* w_scale;     //   |out| (atomicMax on the float bits: zeroed by the caller)
    float* out_amax;
};

// bytes of one activation slab row (32 channels): fp32, or bf16 (ABF)
constexpr int tc_a_row(bool abf) { return abf ? 64 : 128; }

template <int C, int P, bool RES, bool ABF>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv1d_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcArgs a) {
    pdl_trigger();
    static_assert(!ABF || tc_takes_bf16(P), "bf16 activations need the BF16 or FP8 kernel");
    constexpr bool X3 = P == TC_X3;
    constexpr bool FP8 = P == TC_FP8;
    constexpr int A_ROW = tc_a_row(ABF);
    constexpr int NCB = C / TC_KCH;
    constexpr int W_ATOM = tc_w_atom(P);   // 3xTF32: hi tile, then lo tile; bf16: half-size tile
    constexpr int B_RES_BYTES = RES ? 3 * NCB * W_ATOM : 0;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sB = smem;
    uint8_t* sA = smem + B_RES_BYTES;
    uint8_t* sLo = sA + (size_t)a.stages * a.stage_bytes;
    float* stg = reinterpret_cast<float*>(sLo + a.lo_bytes);
    uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stg) + 2 * TC_STG_BYTES);
    uint64_t* empty = full + TC_MAX_STAGES;
    uint64_t* bfull = empty + TC_MAX_STAGES;
    uint32_t* amax_slot = reinterpret_cast<uint32_t*>(bfull + 1);   // FP8: this CTA's per-tile max |out|, two tiles deep

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_half = blockIdx.x % a.n_halves;
    const int cta_m = blockIdx.x / a.n_halves;
    const int m_stride = gridDim.x / a.n_halves;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < a.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);   // one arrive per consumer warp
        }
        mbar_init(bfull, 1);
        amax_slot[0] = amax_slot[1] = 0u;
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();   // everything above overlapped the previous kernel's tail; global memory is touched only from here on

    if (warp == 8) {
        // ================= TMA producer =================
        const bool leader = elect_one();
        auto load_w = [&](uint64_t* bar, uint8_t* dst, int t, int cb) {
            tma_load_2d(&tmB, bar, dst, t * C + cb * TC_KCH, n_half * TC_BN);
            if (X3) tma_load_2d(&tmB, bar, dst + TC_ATOM, t * C + cb * TC_KCH, a.Ctot + n_half * TC_BN);   // lo rows
        };
        if (RES && leader) {
            mbar_arrive_expect_tx(bfull, B_RES_BYTES);
            for (int t = 0; t < 3; ++t)
                for (int cb = 0; cb < NCB; ++cb) load_w(bfull, sB + (t * NCB + cb) * W_ATOM, t, cb);
        }
        int stage = 0;
        uint32_t phase = 0;
        for (int mt = cta_m; mt < a.total_m_tiles; mt += m_stride) {
            const int ta = mt % a.tiles_a;
            const int tb = (mt / a.tiles_a) % a.tiles_b;
            const int n = mt / (a.tiles_a * a.tiles_b);
            for (int cb = 0; cb < NCB; ++cb) {
                mbar_wait(&empty[stage], phase ^ 1);
                if (leader) {
                    uint8_t* st = sA + (size_t)stage * a.stage_bytes;
                    mbar_arrive_expect_tx(&full[stage], a.stage_bytes);
                    // tensor map dims: (ci, cblk, across, along, n)
                    for (int l = 0; l < a.nloads; ++l)
                        tma_load_5d(&tmA, &full[stage], st + l * a.load_rows * A_ROW, 0, cb, tb * a.TB + a.load_b[l],
                                    ta * a.TA + a.load_a[l], n);
                    if (!RES)
                        for (int t = 0; t < 3; ++t) load_w(&full[stage], st + a.a_bytes + t * W_ATOM, t, cb);
                }
                if (++stage == a.stages) {
                    stage = 0;
                    phase ^= 1;
                }
            }
        }
        return;
    }

    // ================= consumers: warpgroup wg owns pixel rows [64 wg, 64 wg + 64) of every tile =================
    const int wg = warp >> 2, wl = warp & 3;
    const int g = lane >> 2, t4 = lane & 3;
    const int et = threadIdx.x & 127;       // phase 2: thread within the warpgroup, which walks channel half wg
    const int c4 = et & 7;                  // phase 2: float4 column inside the half (fixed)
    const int r0 = et >> 3;                 // phase 2: first of this thread's 8 rows (r0, r0+16, ...)
    const int ch0 = n_half * TC_BN + 32 * wg + 4 * c4;
    float* stg_h = stg + wg * (TC_STG_BYTES / 4);
    const bool pre_mask = a.mask_src != nullptr;
    const bool pre_add = (a.add_src != nullptr) && !pre_mask;  // both given: add_src is read in the loop
    const bool affine_mask = a.mask_scale != nullptr;
    const bool out_bf = tc_takes_bf16(P) && a.out_bf16, mask_bf = tc_takes_bf16(P) && a.mask_bf16;
    float4 csum = make_float4(0.f, 0.f, 0.f, 0.f), csq = csum;
    const int ra = 64 * wg + 16 * wl + g;   // this thread's fragment rows ra, ra + 8
    if (RES) mbar_wait(bfull, 0);
    int stage = 0;
    uint32_t phase = 0, chunk = 0, tile_par = 0;
    const int tiles_img = a.tiles_a * a.tiles_b;
    // FP8: max |in| of the next tile's image, loaded one tile ahead (its latency would stall the first fragment)
    float ax_next = FP8 && cta_m < a.total_m_tiles ? __ldg(a.x_amax + cta_m / tiles_img) : 0.f;
    for (int mt = cta_m; mt < a.total_m_tiles; mt += m_stride) {
        const int ta = mt % a.tiles_a;
        const int tb = (mt / a.tiles_a) % a.tiles_b;
        const int n = mt / tiles_img;   // the tile's image (a tile never crosses one: host plan)
        // FP8: the image's activation quantisation factor, 448 / max |in| (0 for an all-zero image: every q = 0)
        float inv = 0.f, ax = 0.f;
        if (FP8) {
            ax = ax_next;
            inv = ax > 0.f ? __fdiv_rn(448.f, ax) : 0.f;
            if (mt + m_stride < a.total_m_tiles) ax_next = __ldg(a.x_amax + (mt + m_stride) / tiles_img);
        }
        // element offset of phase-2 row r0 + 16 j: formed again in the epilogue, not held through the main loop
        auto roff = [&](int j) {
            const int r = r0 + 16 * j;
            const int ap = r >> a.tb_shift, bp = r & (a.TB - 1);
            const int pa = ta * a.TA + ap, pb = tb * a.TB + bp;
            const int y = a.vertical ? pa : pb, x = a.vertical ? pb : pa;
            return ((size_t)(n * a.H + y) * a.W + x) * a.Ctot + ch0;
        };
        float4 pre[8];
        if (pre_mask || pre_add) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const size_t off = roff(j);
                if (pre_mask && mask_bf) {   // the raw bf16 bits, widened in the epilogue: converting here would wait for the load
                    const uint2 u = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const uint16_t*>(a.mask_src) + off));
                    pre[j] = make_float4(__uint_as_float(u.x), __uint_as_float(u.y), 0.f, 0.f);
                } else if (pre_mask) {
                    pre[j] = __ldg(reinterpret_cast<const float4*>(a.mask_src + off));
                } else {
                    float4 ad = __ldg(reinterpret_cast<const float4*>(a.add_src + off));
                    if (a.add_mask) {
                        const float4 mk = __ldg(reinterpret_cast<const float4*>(a.add_mask + off));
                        ad.x = mk.x > 0.f ? ad.x : 0.f; ad.y = mk.y > 0.f ? ad.y : 0.f;
                        ad.z = mk.z > 0.f ? ad.z : 0.f; ad.w = mk.w > 0.f ? ad.w : 0.f;
                    }
                    pre[j] = ad;
                }
            }
        }

        float acc[32], acs[32], part[32];   // large term; 3xTF32 correction terms; one tap's large term
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = acs[i] = part[i] = 0.f;
        for (int cb = 0; cb < NCB; ++cb) {
            mbar_wait(&full[stage], phase);
            uint8_t* st = sA + (size_t)stage * a.stage_bytes;
            const uint32_t wbase = RES ? smem_u32(sB + cb * W_ATOM) : smem_u32(st + a.a_bytes);
            uint8_t* lo = nullptr;   // 3xTF32: this chunk's lo buffer
            if (X3)
                lo = a.lo_stg ? reinterpret_cast<uint8_t*>(stg) + 2 * TC_STG_BYTES - a.a_bytes
                              : sLo + (size_t)(chunk & (a.n_lo - 1)) * a.a_bytes;
            if constexpr (P == TC_TF32 || P == TC_X3) {
                // The slab as the tensor core reads it, one elementwise pass over the swizzled bytes: each word v -> hi =
                // tf32_rna(v) in place and (3xTF32) lo = tf32_rna(v - hi) at the same offset of the lo buffer.  A single
                // lo buffer may still be read by the other warpgroup's MMAs of the previous chunk; with two, the barrier
                // below of the previous chunk already waited for the MMAs that read this one.
                if (X3 && a.n_lo != 2) named_bar_sync(1, 256);
                const uint32_t s_st = smem_u32(st), s_lo = X3 ? smem_u32(lo) : 0;
                for (uint32_t o = 16 * threadIdx.x; o < (uint32_t)a.a_bytes; o += 16 * 256) {
                    const float4 v = lds_f32x4(s_st + o);
                    const uint4 h = make_uint4(tf32_rna(v.x), tf32_rna(v.y), tf32_rna(v.z), tf32_rna(v.w));
                    sts_u32x4(s_st + o, h);
                    if (X3)
                        sts_u32x4(s_lo + o, make_uint4(tf32_rna(v.x - __uint_as_float(h.x)), tf32_rna(v.y - __uint_as_float(h.y)),
                                                       tf32_rna(v.z - __uint_as_float(h.z)), tf32_rna(v.w - __uint_as_float(h.w))));
                }
                fence_proxy_async_smem();   // the generic stores above, before the wgmma (async proxy) reads
                named_bar_sync(1, 256);     // the two warpgroups' tap views overlap in the halo rows
            }
            ++chunk;
            constexpr int W_TAP = RES ? NCB * W_ATOM : W_ATOM;   // distance between the weight tiles of two taps
#pragma unroll
            for (int t = 0; t < 3; ++t) {
                // 8 rows of the swizzle period apart (1024 / 512 bytes): the swizzle phase is the view's row
                const uint8_t* view = st + a.tap_row[t] * A_ROW;
                if constexpr (FP8) {
                    // k32 fragment: four adjacent channels per register = one 16-byte load (fp32 slab) or one 8-byte
                    // load (bf16 slab); q = e4m3(v * inv), the product rounded to nearest in fp32 first
                    uint32_t aq[4];
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        const int row = ra + 8 * (r & 1), c = 4 * t4 + 16 * (r >> 1);
                        float4 v;
                        if constexpr (ABF) v = bf16x4_to_f4(*reinterpret_cast<const uint2*>(view + sw64_off(row, c)));
                        else v = *reinterpret_cast<const float4*>(view + sw128_off(row, c));
                        aq[r] = pack_e4m3x4(__fmul_rn(v.x, inv), __fmul_rn(v.y, inv), __fmul_rn(v.z, inv), __fmul_rn(v.w, inv));
                    }
                    wgmma_fence();
                    wgmma_m64n64k32_e4m3(part, aq, wgmma_desc_sw32(wbase + t * W_TAP), 0);
                    wgmma_commit();
                    wgmma_wait0();
                    reg_fence(part);
#pragma unroll
                    for (int i = 0; i < 32; ++i) acc[i] += part[i];
                } else if constexpr (P == TC_BF16) {
                    // k16 fragments: two adjacent channels per register = one 8-byte load inside a 16-byte chunk (fp32
                    // slab), or one 4-byte load of the ready pair (bf16 slab)
                    uint32_t ab[2][4];
#pragma unroll
                    for (int kk = 0; kk < 2; ++kk) {
                        const int c = 16 * kk + 2 * t4;
                        if constexpr (ABF) {
                            ab[kk][0] = *reinterpret_cast<const uint32_t*>(view + sw64_off(ra, c));
                            ab[kk][1] = *reinterpret_cast<const uint32_t*>(view + sw64_off(ra + 8, c));
                            ab[kk][2] = *reinterpret_cast<const uint32_t*>(view + sw64_off(ra, c + 8));
                            ab[kk][3] = *reinterpret_cast<const uint32_t*>(view + sw64_off(ra + 8, c + 8));
                        } else {
                            const float2 v0 = *reinterpret_cast<const float2*>(view + sw128_off(ra, c));
                            const float2 v1 = *reinterpret_cast<const float2*>(view + sw128_off(ra + 8, c));
                            const float2 v2 = *reinterpret_cast<const float2*>(view + sw128_off(ra, c + 8));
                            const float2 v3 = *reinterpret_cast<const float2*>(view + sw128_off(ra + 8, c + 8));
                            ab[kk][0] = pack_bf16x2(v0.x, v0.y);
                            ab[kk][1] = pack_bf16x2(v1.x, v1.y);
                            ab[kk][2] = pack_bf16x2(v2.x, v2.y);
                            ab[kk][3] = pack_bf16x2(v3.x, v3.y);
                        }
                    }
                    const uint64_t bd = wgmma_desc_sw64(wbase + t * W_TAP);
                    wgmma_fence();
#pragma unroll
                    for (int kk = 0; kk < 2; ++kk) wgmma_m64n64k16_bf16(part, ab[kk], bd + 2 * kk, kk);
                    wgmma_commit();
                    wgmma_wait0();
                    reg_fence(part);
#pragma unroll
                    for (int i = 0; i < 32; ++i) acc[i] += part[i];
                } else {
                    // this warpgroup's 64 rows of the view (hi) and of the same rows of the lo buffer; k8 = 32 bytes along K
                    // (descriptors formed at each MMA from 32-bit addresses: fewer live registers than 64-bit descriptors)
                    const uint32_t va = smem_u32(view) + 64 * wg * 128;
                    const uint32_t vl = X3 ? va - smem_u32(st) + smem_u32(lo) : 0;
                    const uint32_t vb = wbase + t * W_TAP;
                    wgmma_fence();
#pragma unroll
                    for (int k8 = 0; k8 < 4; ++k8) {
                        const uint32_t k = 32 * k8;
                        // k8 = 0: part = product (previous tap dropped)
                        wgmma_m64n64k8_tf32_ss(part, wgmma_desc_sw128(va + k), wgmma_desc_sw128(vb + k), k8);
                        if (X3) {
                            wgmma_m64n64k8_tf32_ss(acs, wgmma_desc_sw128(va + k), wgmma_desc_sw128(vb + TC_ATOM + k), 1);   // a_hi * w_lo
                            wgmma_m64n64k8_tf32_ss(acs, wgmma_desc_sw128(vl + k), wgmma_desc_sw128(vb + k), 1);             // a_lo * w_hi
                        }
                    }
                    wgmma_commit();
                    wgmma_wait0();
                    reg_fence(part);
                    if (X3) reg_fence(acs);
                    // The tensor core adds into its accumulator without IEEE rounding; a chain over all 3*C products drifts
                    // several times further from the exact sum than an fp32 FFMA chain does.  Each tap's 32 products are
                    // summed there from zero and added to the running sum here, rounded to nearest.
#pragma unroll
                    for (int i = 0; i < 32; ++i) acc[i] += part[i];
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == a.stages) {
                stage = 0;
                phase ^= 1;
            }
        }

        // phase-2 channel vectors: loaded per tile (cache hits), not held through the main loop
        float4 bsv = make_float4(0.f, 0.f, 0.f, 0.f), msc = bsv, msh = bsv;
        if (a.bias) bsv = __ldg(reinterpret_cast<const float4*>(a.bias + ch0));
        float4 dqs = make_float4(0.f, 0.f, 0.f, 0.f);   // FP8: dequantisation factors s_x[n] * w_scale[co]
        if (FP8) {
            const float sx = __fdiv_rn(ax, 448.f);
            const float4 ws = __ldg(reinterpret_cast<const float4*>(a.w_scale + ch0));
            dqs = make_float4(__fmul_rn(sx, ws.x), __fmul_rn(sx, ws.y), __fmul_rn(sx, ws.z), __fmul_rn(sx, ws.w));
        }
        float amax = 0.f;                                 // FP8: max |stored value| of this thread's part of the tile
        if (affine_mask) {
            msc = __ldg(reinterpret_cast<const float4*>(a.mask_scale + ch0));
            msh = __ldg(reinterpret_cast<const float4*>(a.mask_shift + ch0));
        }
        // ---- phase 1: accumulator fragments -> staging tile (both halves)
        if (X3 && a.lo_stg) named_bar_sync(1, 256);   // the other warpgroup's last MMAs may still read the lo buffer there
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            const int row = ra + 8 * ((i >> 1) & 1);
            const int col = 8 * (i >> 2) + 2 * t4;
            const float2 v = X3 ? make_float2(acs[i] + acc[i], acs[i + 1] + acc[i + 1]) : make_float2(acc[i], acc[i + 1]);
            *reinterpret_cast<float2*>(&stg[(col >> 5) * (TC_STG_BYTES / 4) + row * TC_STG_LD + (col & 31)]) = v;
        }
        named_bar_sync(1, 256);   // staging complete
        // ---- phase 2: row-major walk of half wg, 8 consecutive threads = one pixel's 32 channels (128 B)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int r = r0 + 16 * j;
            const size_t off = roff(j);
            if (mask_bf) pre[j] = bf16x4_to_f4(make_uint2(__float_as_uint(pre[j].x), __float_as_uint(pre[j].y)));
            float4 o = *reinterpret_cast<const float4*>(&stg_h[r * TC_STG_LD + 4 * c4]);
            if (FP8) {   // acc * (s_x * s_w), rounded, then + bias (never contracted into an FMA)
                o.x = __fmul_rn(o.x, dqs.x); o.y = __fmul_rn(o.y, dqs.y); o.z = __fmul_rn(o.z, dqs.z); o.w = __fmul_rn(o.w, dqs.w);
            }
            o.x += bsv.x; o.y += bsv.y; o.z += bsv.z; o.w += bsv.w;
            if (a.relu & 1) {
                o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
            }
            if (pre_mask) {
                float4 mk = pre[j];
                if (affine_mask) {   // the same fma the forward BatchNorm-apply performed before its ReLU: bit-identical mask
                    mk.x = fmaf(mk.x, msc.x, msh.x); mk.y = fmaf(mk.y, msc.y, msh.y);
                    mk.z = fmaf(mk.z, msc.z, msh.z); mk.w = fmaf(mk.w, msc.w, msh.w);
                }
                o.x = mk.x > 0.f ? o.x : 0.f; o.y = mk.y > 0.f ? o.y : 0.f;
                o.z = mk.z > 0.f ? o.z : 0.f; o.w = mk.w > 0.f ? o.w : 0.f;
            }
            if (pre_add) {
                o.x += pre[j].x; o.y += pre[j].y; o.z += pre[j].z; o.w += pre[j].w;
            } else if (a.add_src) {
                float4 ad = __ldg(reinterpret_cast<const float4*>(a.add_src + off));
                if (a.add_mask) {
                    const float4 mk = __ldg(reinterpret_cast<const float4*>(a.add_mask + off));
                    ad.x = mk.x > 0.f ? ad.x : 0.f; ad.y = mk.y > 0.f ? ad.y : 0.f;
                    ad.z = mk.z > 0.f ? ad.z : 0.f; ad.w = mk.w > 0.f ? ad.w : 0.f;
                }
                o.x += ad.x; o.y += ad.y; o.z += ad.z; o.w += ad.w;
            }
            if (a.relu & 2) {   // ReLU AFTER the residual add: the closing relu(conv + x) of an eval-mode (BN-folded) block
                o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
            }
            if (out_bf) *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(a.out) + off) = f4_to_bf16x4(o);
            else *reinterpret_cast<float4*>(a.out + off) = o;
            if (FP8) amax = fmaxf(amax, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
            csum.x += o.x; csum.y += o.y; csum.z += o.z; csum.w += o.w;
            if (affine_mask) {   // pre[j] is the BatchNorm input x
                csq.x = fmaf(o.x, pre[j].x, csq.x); csq.y = fmaf(o.y, pre[j].y, csq.y);
                csq.z = fmaf(o.z, pre[j].z, csq.z); csq.w = fmaf(o.w, pre[j].w, csq.w);
            } else {
                csq.x = fmaf(o.x, o.x, csq.x); csq.y = fmaf(o.y, o.y, csq.y);
                csq.z = fmaf(o.z, o.z, csq.z); csq.w = fmaf(o.w, o.w, csq.w);
            }
        }
        if (FP8) {
            // a bf16 `out` stores the rounded values: rounding to nearest is monotonic, so their max is the rounded max
            if (out_bf) amax = __uint_as_float(f4_to_bf16x4(make_float4(amax, 0.f, 0.f, 0.f)).x << 16);
            const uint32_t wmax = __reduce_max_sync(0xffffffffu, __float_as_uint(amax));   // |v| >= 0: ordered as uint
            if (lane == 0) atomicMax(&amax_slot[tile_par], wmax);
        }
        named_bar_sync(1, 256);   // staging tile may be overwritten (FP8: and the tile's max is complete)
        if (FP8) {
            if (threadIdx.x == 0) {   // the tile's image: one global atomic per CTA and tile; the slot is free again
                const uint32_t m = amax_slot[tile_par];
                if (m) atomicMax(reinterpret_cast<unsigned int*>(a.out_amax) + n, m);
                amax_slot[tile_par] = 0u;
            }
            tile_par ^= 1u;
        }
    }
    if (a.colsum_partial || a.stats_partial) {
        // 16 threads share each float4 column of the half: combine them through the (now free) staging half
        *reinterpret_cast<float4*>(&stg_h[r0 * TC_STG_LD + 4 * c4]) = csum;
        *reinterpret_cast<float4*>(&stg_h[(32 + r0) * TC_STG_LD + 4 * c4]) = csq;
        named_bar_sync(2 + wg, 128);
        if (et < 32) {
            const int ch = n_half * TC_BN + 32 * wg + et;
            double tot = 0.0, tsq = 0.0;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                tot += (double)stg_h[k * TC_STG_LD + et];
                tsq += (double)stg_h[(32 + k) * TC_STG_LD + et];
            }
            if (a.colsum_partial) a.colsum_partial[(size_t)cta_m * a.Ctot + ch] = (float)tot;
            if (a.stats_partial) {
                double* sp = a.stats_partial + (size_t)cta_m * 2 * a.Ctot + ch;
                sp[0] = tot;
                sp[a.Ctot] = tsq;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
struct TcPlan {
    TcArgs geo;     // the geometry fields of the kernel arguments
    bool res;
    int smem_bytes, m_ctas;
};

static int tc_m_ctas(int N, int C, int tiles_per_image) {
    const int n_halves = C / TC_BN;
    const long long tiles = (long long)N * tiles_per_image;
    long long m_ctas = device_sms() / n_halves;
    if (m_ctas > tiles) m_ctas = tiles;
    return (int)(m_ctas < 1 ? 1 : m_ctas);
}

// Shared memory: resident weights when they leave room for two stages, else streamed per stage.  3xTF32 also needs lo
// buffers of one slab each, outside the ring: two when two stages still fit next to them, else one, else one laid over
// the staging tile (idle during the main loop; slabs larger than it reach back into the space before it).
static bool tc_fit(int C, int prec, bool abf, TcPlan* p) {
    const int w_atom = tc_w_atom(prec);
    const int b_res = 3 * (C / TC_KCH) * w_atom;
    TcArgs& g = p->geo;
    g.a_bytes = g.nloads * g.load_rows * tc_a_row(abf);
    p->res = TC_FIXED_SMEM + b_res + 2 * g.a_bytes <= TC_SMEM_LIMIT;
    g.stage_bytes = g.a_bytes + (p->res ? 0 : 3 * w_atom);
    const int avail = TC_SMEM_LIMIT - TC_FIXED_SMEM - (p->res ? b_res : 0);
    g.n_lo = g.lo_stg = g.lo_bytes = 0;
    if (prec == TC_X3) {
        g.n_lo = 2;
        while (g.n_lo > 0 && avail - g.n_lo * g.a_bytes < 2 * g.stage_bytes) --g.n_lo;
        g.lo_bytes = g.n_lo * g.a_bytes;
        if (g.n_lo == 0) {
            g.n_lo = g.lo_stg = 1;
            g.lo_bytes = g.a_bytes > 2 * TC_STG_BYTES ? g.a_bytes - 2 * TC_STG_BYTES : 0;
        }
    }
    int stages = (avail - g.lo_bytes) / g.stage_bytes;
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    if (stages < 1) return false;
    g.stages = stages;
    p->smem_bytes = TC_FIXED_SMEM + (p->res ? b_res : 0) + stages * g.stage_bytes + g.lo_bytes;
    return true;
}

// Halo-slab plan: taps {-d, 0, +d} (forward) or {+d, 0, -d} (input gradient) along one axis.  TA x TB = 128 pixels with
// TB a power of two such that the tap shift d*TB is a multiple of the 8-row swizzle period; the slab with the fewest
// rows wins (tall tiles for the large dilations: halo 2d / TA).
static bool tc_plan_slab(int N, int H, int W, int C, const int* dy, const int* dx, int prec, TcPlan* p, bool abf = false) {
    if (!(C == 64 || C == 128) || N <= 0) return false;
    const bool vert = dy[0] != 0 || dy[2] != 0;
    const int* o = vert ? dy : dx;
    const int* z = vert ? dx : dy;
    if (z[0] || z[1] || z[2] || o[1] != 0 || o[0] != -o[2] || o[0] == 0) return false;
    const int dil = o[0] < 0 ? -o[0] : o[0];
    const bool fwd_order = o[0] < 0;   // weight slot t reads offset (t-1)*d
    const int ext_a = vert ? H : W, ext_b = vert ? W : H;
    TcArgs& g = p->geo;
    int best_rows = 1 << 30;
    for (int sh = 0; sh <= 4; ++sh) {
        const int TB = 1 << sh, TA = 128 >> sh;
        if (ext_a % TA || ext_b % TB || (dil * TB) % 8 || TA + 2 * dil > 256) continue;
        const int rows = (TA + 2 * dil) * TB;
        if (rows < best_rows) {
            best_rows = rows;
            g.TA = TA;
            g.TB = TB;
            g.tb_shift = sh;
        }
    }
    if (best_rows == (1 << 30)) return false;
    g.vertical = vert ? 1 : 0;
    g.tiles_a = ext_a / g.TA;
    g.tiles_b = ext_b / g.TB;
    g.nloads = 1;
    g.load_rows = best_rows;
    g.load_a[0] = -dil;
    g.load_b[0] = 0;
    for (int t = 0; t < 3; ++t) g.tap_row[t] = (fwd_order ? t : 2 - t) * dil * g.TB;
    if (!tc_fit(C, prec, abf, p)) return false;
    p->m_ctas = tc_m_ctas(N, C, g.tiles_a * g.tiles_b);
    return tc_get_encode_fn() != nullptr;
}

// Per-tap plan: any three taps; a bx x by = 128 pixel patch with bx | W, by | H (wide patches preferred).
static bool tc_plan_taps(int N, int H, int W, int C, const int* dy, const int* dx, int prec, TcPlan* p, bool abf = false) {
    if (!(C == 64 || C == 128) || N <= 0) return false;
    TcArgs& g = p->geo;
    int sh = 7;
    while (sh >= 0 && (W % (1 << sh) || H % (128 >> sh))) --sh;
    if (sh < 0) return false;
    g.vertical = 1;
    g.TB = 1 << sh;
    g.TA = 128 >> sh;
    g.tb_shift = sh;
    g.tiles_a = H / g.TA;
    g.tiles_b = W / g.TB;
    g.nloads = 3;
    g.load_rows = 128;
    for (int t = 0; t < 3; ++t) {
        g.load_a[t] = dy ? dy[t] : 0;
        g.load_b[t] = dx ? dx[t] : 0;
        g.tap_row[t] = t * 128;
    }
    if (!tc_fit(C, prec, abf, p)) return false;
    p->m_ctas = tc_m_ctas(N, C, g.tiles_a * g.tiles_b);
    return tc_get_encode_fn() != nullptr;
}

template <int C, int P, bool RES, bool ABF>
static cudaError_t tc_launch(int grid, int smem_bytes, cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB,
                             const TcArgs& a) {
    cudaError_t e = cudaFuncSetAttribute(conv1d_tc_kernel<C, P, RES, ABF>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT);
    if (e != cudaSuccess) return e;
    return lf_launch(conv1d_tc_kernel<C, P, RES, ABF>, grid, TC_THREADS, smem_bytes, stream, tmA, tmB, a);
}

template <int P, bool ABF = false>
static cudaError_t tc_launch_p(bool res, int C, int grid, int smem_bytes, cudaStream_t stream, const CUtensorMap& tmA,
                               const CUtensorMap& tmB, const TcArgs& a) {
    if (C == 128) return res ? tc_launch<128, P, true, ABF>(grid, smem_bytes, stream, tmA, tmB, a) : tc_launch<128, P, false, ABF>(grid, smem_bytes, stream, tmA, tmB, a);
    return res ? tc_launch<64, P, true, ABF>(grid, smem_bytes, stream, tmA, tmB, a) : tc_launch<64, P, false, ABF>(grid, smem_bytes, stream, tmA, tmB, a);
}

static int tc_run(const LfConvTcArgs* args, lf_stream_t stream_, int prec, const LfConvTcFp8Args* f8 = nullptr) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!args) return LF_ERR_INVALID_ARGUMENT;
    const LfConvTcArgs& p = *args;
    LF_REQUIRE(p.in && p.wpack && p.out);
    LF_REQUIRE(!p.mask_scale || (p.mask_shift && p.mask_src && p.stats_partial));
    LF_REQUIRE((p.in_dtype == LF_F32 || p.in_dtype == LF_BF16) && (p.out_dtype == LF_F32 || p.out_dtype == LF_BF16) &&
               (p.mask_dtype == LF_F32 || p.mask_dtype == LF_BF16));
    if (!tc_takes_bf16(prec) && (p.in_dtype | p.out_dtype | p.mask_dtype) != LF_F32) return LF_ERR_UNSUPPORTED;
    const bool fp8 = prec == TC_FP8;
    // FP8 is an inference epilogue: scales in, per-image max out, no gradient-side outputs
    if (fp8) LF_REQUIRE(f8 && f8->x_amax && f8->w_scale && f8->out_amax && !p.colsum_partial && !p.stats_partial && !p.mask_scale);
    const bool x3 = prec == TC_X3;
    const bool abf = p.in_dtype == LF_BF16;
    TcPlan pl{};
    // bf16 and fp8 take the slab exactly where TF32 does (their smaller weight tiles and bf16 slabs fit wherever the
    // TF32 ones do), so that lf_conv1d_tc_supported / lf_conv1d_tc_slab_ok answer for all three
    const bool slab = (x3 || g_tc_variant != 1) &&
                      (!tc_takes_bf16(prec) || tc_plan_slab(p.N, p.H, p.W, p.C, p.dy, p.dx, TC_TF32, &pl)) &&
                      tc_plan_slab(p.N, p.H, p.W, p.C, p.dy, p.dx, prec, &pl, abf);
    if (!slab && (x3 || !tc_plan_taps(p.N, p.H, p.W, p.C, p.dy, p.dx, prec, &pl, abf))) return LF_ERR_UNSUPPORTED;
    TcArgs a = pl.geo;
    // FP8 scales and maxima are per image: every tile must lie within one image (tiles cover each image exactly)
    if (fp8 && (a.tiles_a * a.TA != (a.vertical ? p.H : p.W) || a.tiles_b * a.TB != (a.vertical ? p.W : p.H)))
        return LF_ERR_UNSUPPORTED;
    a.x_amax = fp8 ? f8->x_amax : nullptr;
    a.w_scale = fp8 ? f8->w_scale : nullptr;
    a.out_amax = fp8 ? f8->out_amax : nullptr;
    a.out = p.out; a.bias = p.bias; a.mask_src = p.mask_src; a.add_src = p.add_src; a.add_mask = p.add_mask;
    a.colsum_partial = p.colsum_partial;
    a.stats_partial = p.stats_partial;
    a.mask_scale = p.mask_scale;
    a.mask_shift = p.mask_shift;
    a.N = p.N; a.H = p.H; a.W = p.W; a.Ctot = p.C; a.relu = p.relu;
    a.n_halves = p.C / TC_BN;
    a.out_bf16 = p.out_dtype == LF_BF16;
    a.mask_bf16 = p.mask_dtype == LF_BF16;
    a.total_m_tiles = p.N * a.tiles_a * a.tiles_b;

    TcEncodeTiledFn enc = tc_get_encode_fn();
    CUtensorMap tmA, tmB;
    {
        // activations [N,H,W,C] viewed as (ci:32, cblk:C/32, across, along, n); one box = the slab or one tap's patch;
        // bf16: rows of 64 bytes, 64B-swizzled
        const cuuint64_t esz = abf ? 2 : 4;
        const cuuint64_t sx = (cuuint64_t)p.C * esz, sy = (cuuint64_t)p.W * p.C * esz;
        cuuint64_t dims[5] = {32, (cuuint64_t)(p.C / 32), (cuuint64_t)(a.vertical ? p.W : p.H),
                              (cuuint64_t)(a.vertical ? p.H : p.W), (cuuint64_t)p.N};
        cuuint64_t strides[4] = {32 * esz, a.vertical ? sx : sy, a.vertical ? sy : sx, (cuuint64_t)p.H * p.W * p.C * esz};
        cuuint32_t box[5] = {32, 1, (cuuint32_t)a.TB, (cuuint32_t)(a.load_rows / a.TB), 1};
        cuuint32_t estr[5] = {1, 1, 1, 1, 1};
        CUresult r = enc(&tmA, abf ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5,
                         const_cast<float*>(p.in), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         abf ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return LF_ERR_CUDA;
    }
    {
        // packed weights [Cout][3*C] (K contiguous); 3xTF32: [2][Cout][3*C] (hi, lo) as one [2*Cout][3*C] matrix;
        // bf16: [Cout][3*C] bf16, [64 x 32] boxes of 64-byte rows, 64B-swizzled; fp8: [Cout][3*C] e4m3 bytes, boxes of
        // 32-byte rows, 32B-swizzled
        const bool bf = prec == TC_BF16;
        const int esz = fp8 ? 1 : bf ? 2 : 4;
        cuuint64_t dims[2] = {(cuuint64_t)(3 * p.C), (cuuint64_t)((x3 ? 2 : 1) * p.C)};
        cuuint64_t strides[1] = {(cuuint64_t)(3 * p.C) * esz};
        cuuint32_t box[2] = {32, TC_BN};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&tmB, fp8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : bf ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                         const_cast<float*>(p.wpack), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         fp8 ? CU_TENSOR_MAP_SWIZZLE_32B : bf ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return LF_ERR_CUDA;
    }
    const int grid = pl.m_ctas * a.n_halves;
    const int s = pl.smem_bytes;
    cudaError_t e;
    if (prec == TC_X3) e = tc_launch_p<TC_X3>(pl.res, p.C, grid, s, stream, tmA, tmB, a);
    else if (prec == TC_BF16 && abf) e = tc_launch_p<TC_BF16, true>(pl.res, p.C, grid, s, stream, tmA, tmB, a);
    else if (prec == TC_BF16) e = tc_launch_p<TC_BF16>(pl.res, p.C, grid, s, stream, tmA, tmB, a);
    else if (fp8 && abf) e = tc_launch_p<TC_FP8, true>(pl.res, p.C, grid, s, stream, tmA, tmB, a);
    else if (fp8) e = tc_launch_p<TC_FP8>(pl.res, p.C, grid, s, stream, tmA, tmB, a);
    else e = tc_launch_p<TC_TF32>(pl.res, p.C, grid, s, stream, tmA, tmB, a);
    if (e != cudaSuccess) { set_last_cuda_error(e); return LF_ERR_CUDA; }
    return check_launch();
}

}  // namespace lf

using namespace lf;

extern "C" void lf_conv1d_tc_set_variant(int v) { g_tc_variant = (v == 1) ? 1 : 2; }

// 0 if the shape is unsupported, else the number of rows of the optional colsum_partial / stats_partial outputs.  Every
// shape the slab plan takes is also taken by the per-tap plan (same number of CTAs), which serves the TF32 and bf16
// calls the slab does not fit.  The bf16 entry serves exactly the shapes and slab cases of the TF32 one.
extern "C" int lf_conv1d_tc_supported(int N, int H, int W, int C) {
    TcPlan pl{};
    return tc_plan_taps(N, H, W, C, nullptr, nullptr, TC_TF32, &pl) ? pl.m_ctas : 0;
}

// 1 if a TF32 (or bf16) call with these taps runs on the halo-slab path
extern "C" int lf_conv1d_tc_slab_ok(int N, int H, int W, int C, int vertical, int dil) {
    if (g_tc_variant == 1 || dil < 1) return 0;
    TcPlan pl{};
    const int zero[3] = {0, 0, 0}, off[3] = {-dil, 0, dil};
    return tc_plan_slab(N, H, W, C, vertical ? off : zero, vertical ? zero : off, TC_TF32, &pl) ? 1 : 0;
}

// rows of colsum_partial / stats_partial (= CTAs per 64-channel half), 0 if a 3xTF32 call with these taps is not served
extern "C" int lf_conv1d_tc_x3_rows(int N, int H, int W, int C, int vertical, int dil) {
    if (dil < 1) return 0;
    TcPlan pl{};
    const int zero[3] = {0, 0, 0}, off[3] = {-dil, 0, dil};
    return tc_plan_slab(N, H, W, C, vertical ? off : zero, vertical ? zero : off, TC_X3, &pl) ? pl.m_ctas : 0;
}

extern "C" int lf_conv1d_tc(const LfConvTcArgs* args, lf_stream_t stream) { return tc_run(args, stream, TC_TF32); }
extern "C" int lf_conv1d_tc_x3(const LfConvTcArgs* args, lf_stream_t stream) { return tc_run(args, stream, TC_X3); }
extern "C" int lf_conv1d_tc_bf16(const LfConvTcArgs* args, lf_stream_t stream) { return tc_run(args, stream, TC_BF16); }
extern "C" int lf_conv1d_tc_fp8(const LfConvTcFp8Args* args, lf_stream_t stream) {
    return args ? tc_run(&args->conv, stream, TC_FP8, args) : LF_ERR_INVALID_ARGUMENT;
}
