// Hopper (sm_90a) wgmma implicit-GEMM kernel for ERFNet's factorised 3-tap convolutions
// (non_bottleneck_1d: conv3x1 / conv1x3 with dilation, BP/Networks/ERFNet.py:29-37,44-53) and their input gradients,
// C in {64, 128}, NHWC fp32 activations, fp32 accumulate.  Two precisions (template X3):
//  * TF32 (lf_conv1d_tc): operands rounded to TF32 (the arithmetic cuDNN uses for the reference's fp32 convs on
//    Ampere and later), one product per multiply;
//  * 3xTF32 (lf_conv1d_tc_x3, the library default): every fp32 operand is split a = a_hi + a_lo (tc_ptx.cuh) and each
//    product is a_hi*w_hi + (a_hi*w_lo + a_lo*w_hi) with fp32 accumulation -- as accurate as an fp32 FFMA chain.  The
//    weights arrive pre-split from the packer ([2][Cout][3C]: hi rows, then lo rows; both exact TF32 values).
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
//  * MMA: wgmma m64n64k8 TF32.  Two consumer warpgroups own 64 pixel rows each; they load their A fragments from the
//    swizzled slab (split into hi / lo in registers for 3xTF32) and take B from shared memory through a descriptor.
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
};

template <int C, bool X3, bool RES>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv1d_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcArgs a) {
    pdl_trigger();
    constexpr int NCB = C / TC_KCH;
    constexpr int W_ATOM = X3 ? 2 * TC_ATOM : TC_ATOM;   // 3xTF32: hi tile, then lo tile
    constexpr int B_RES_BYTES = RES ? 3 * NCB * W_ATOM : 0;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sB = smem;
    uint8_t* sA = smem + B_RES_BYTES;
    float* stg = reinterpret_cast<float*>(sA + (size_t)a.stages * a.stage_bytes);
    uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(stg) + 2 * TC_STG_BYTES);
    uint64_t* empty = full + TC_MAX_STAGES;
    uint64_t* bfull = empty + TC_MAX_STAGES;

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
                        tma_load_5d(&tmA, &full[stage], st + l * a.load_rows * 128, 0, cb, tb * a.TB + a.load_b[l],
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
    float4 csum = make_float4(0.f, 0.f, 0.f, 0.f), csq = csum, msc = csum, msh = csum, bsv = csum;
    if (a.bias) bsv = __ldg(reinterpret_cast<const float4*>(a.bias + ch0));
    if (affine_mask) {
        msc = __ldg(reinterpret_cast<const float4*>(a.mask_scale + ch0));
        msh = __ldg(reinterpret_cast<const float4*>(a.mask_shift + ch0));
    }
    const int ra = 64 * wg + 16 * wl + g;   // this thread's fragment rows ra, ra + 8
    if (RES) mbar_wait(bfull, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int mt = cta_m; mt < a.total_m_tiles; mt += m_stride) {
        const int ta = mt % a.tiles_a;
        const int tb = (mt / a.tiles_a) % a.tiles_b;
        const int n = mt / (a.tiles_a * a.tiles_b);
        size_t roff[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int r = r0 + 16 * j;
            const int ap = r >> a.tb_shift, bp = r & (a.TB - 1);
            const int pa = ta * a.TA + ap, pb = tb * a.TB + bp;
            const int y = a.vertical ? pa : pb, x = a.vertical ? pb : pa;
            roff[j] = ((size_t)(n * a.H + y) * a.W + x) * a.Ctot + ch0;
        }
        float4 pre[8];
        if (pre_mask || pre_add) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (pre_mask) {
                    pre[j] = __ldg(reinterpret_cast<const float4*>(a.mask_src + roff[j]));
                } else {
                    float4 ad = __ldg(reinterpret_cast<const float4*>(a.add_src + roff[j]));
                    if (a.add_mask) {
                        const float4 mk = __ldg(reinterpret_cast<const float4*>(a.add_mask + roff[j]));
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
            const uint8_t* st = sA + (size_t)stage * a.stage_bytes;
            const uint32_t wbase = RES ? smem_u32(sB + cb * W_ATOM) : smem_u32(st + a.a_bytes);
            constexpr int W_TAP = RES ? NCB * W_ATOM : W_ATOM;   // distance between the weight tiles of two taps
#pragma unroll
            for (int t = 0; t < 3; ++t) {
                const uint8_t* view = st + a.tap_row[t] * 128;   // 1024-byte aligned: the swizzle phase is the view's row
                uint32_t ah[4][4], al[4][4];
#pragma unroll
                for (int k8 = 0; k8 < 4; ++k8) {
                    const int c = 8 * k8 + t4;
                    const float v[4] = {*reinterpret_cast<const float*>(view + sw128_off(ra, c)),
                                        *reinterpret_cast<const float*>(view + sw128_off(ra + 8, c)),
                                        *reinterpret_cast<const float*>(view + sw128_off(ra, c + 4)),
                                        *reinterpret_cast<const float*>(view + sw128_off(ra + 8, c + 4))};
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        if (X3) {
                            tf32_split(v[q], ah[k8][q], al[k8][q]);
                        } else {
                            ah[k8][q] = tf32_rna(v[q]);
                        }
                    }
                }
                const uint64_t bd = wgmma_desc_sw128(wbase + t * W_TAP);
                wgmma_fence();
#pragma unroll
                for (int k8 = 0; k8 < 4; ++k8) {
                    wgmma_m64n64k8_tf32(part, ah[k8], bd + 2 * k8, k8);   // k8 = 0: part = product (previous tap dropped)
                    if (X3) {
                        wgmma_m64n64k8_tf32(acs, ah[k8], bd + (TC_ATOM >> 4) + 2 * k8, 1);   // a_hi * w_lo
                        wgmma_m64n64k8_tf32(acs, al[k8], bd + 2 * k8, 1);                    // a_lo * w_hi
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
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == a.stages) {
                stage = 0;
                phase ^= 1;
            }
        }

        // ---- phase 1: accumulator fragments -> staging tile (both halves)
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
            const size_t off = roff[j];
            float4 o = *reinterpret_cast<const float4*>(&stg_h[r * TC_STG_LD + 4 * c4]);
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
            *reinterpret_cast<float4*>(a.out + off) = o;
            csum.x += o.x; csum.y += o.y; csum.z += o.z; csum.w += o.w;
            if (affine_mask) {   // pre[j] is the BatchNorm input x
                csq.x = fmaf(o.x, pre[j].x, csq.x); csq.y = fmaf(o.y, pre[j].y, csq.y);
                csq.z = fmaf(o.z, pre[j].z, csq.z); csq.w = fmaf(o.w, pre[j].w, csq.w);
            } else {
                csq.x = fmaf(o.x, o.x, csq.x); csq.y = fmaf(o.y, o.y, csq.y);
                csq.z = fmaf(o.z, o.z, csq.z); csq.w = fmaf(o.w, o.w, csq.w);
            }
        }
        named_bar_sync(1, 256);   // staging tile may be overwritten
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

// Shared memory: resident weights when they leave room for two stages, else streamed per stage.
static bool tc_fit(int C, bool x3, TcPlan* p) {
    const int w_atom = (x3 ? 2 : 1) * TC_ATOM;
    const int b_res = 3 * (C / TC_KCH) * w_atom;
    TcArgs& g = p->geo;
    g.a_bytes = g.nloads * g.load_rows * 128;
    p->res = TC_FIXED_SMEM + b_res + 2 * g.a_bytes <= TC_SMEM_LIMIT;
    g.stage_bytes = g.a_bytes + (p->res ? 0 : 3 * w_atom);
    const int avail = TC_SMEM_LIMIT - TC_FIXED_SMEM - (p->res ? b_res : 0);
    int stages = avail / g.stage_bytes;
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    if (stages < 1) return false;
    g.stages = stages;
    p->smem_bytes = TC_FIXED_SMEM + (p->res ? b_res : 0) + stages * g.stage_bytes;
    return true;
}

// Halo-slab plan: taps {-d, 0, +d} (forward) or {+d, 0, -d} (input gradient) along one axis.  TA x TB = 128 pixels with
// TB a power of two such that the tap shift d*TB is a multiple of the 8-row swizzle period; the slab with the fewest
// rows wins (tall tiles for the large dilations: halo 2d / TA).
static bool tc_plan_slab(int N, int H, int W, int C, const int* dy, const int* dx, bool x3, TcPlan* p) {
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
    if (!tc_fit(C, x3, p)) return false;
    p->m_ctas = tc_m_ctas(N, C, g.tiles_a * g.tiles_b);
    return tc_get_encode_fn() != nullptr;
}

// Per-tap plan: any three taps; a bx x by = 128 pixel patch with bx | W, by | H (wide patches preferred).
static bool tc_plan_taps(int N, int H, int W, int C, const int* dy, const int* dx, TcPlan* p) {
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
    if (!tc_fit(C, false, p)) return false;
    p->m_ctas = tc_m_ctas(N, C, g.tiles_a * g.tiles_b);
    return tc_get_encode_fn() != nullptr;
}

template <int C, bool X3, bool RES>
static cudaError_t tc_launch(int grid, int smem_bytes, cudaStream_t stream, const CUtensorMap& tmA, const CUtensorMap& tmB,
                             const TcArgs& a) {
    cudaError_t e = cudaFuncSetAttribute(conv1d_tc_kernel<C, X3, RES>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT);
    if (e != cudaSuccess) return e;
    return lf_launch(conv1d_tc_kernel<C, X3, RES>, grid, TC_THREADS, smem_bytes, stream, tmA, tmB, a);
}

static int tc_run(const LfConvTcArgs* args, lf_stream_t stream_, bool x3) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!args) return LF_ERR_INVALID_ARGUMENT;
    const LfConvTcArgs& p = *args;
    LF_REQUIRE(p.in && p.wpack && p.out);
    LF_REQUIRE(!p.mask_scale || (p.mask_shift && p.mask_src && p.stats_partial));
    TcPlan pl{};
    const bool slab = (x3 || g_tc_variant != 1) && tc_plan_slab(p.N, p.H, p.W, p.C, p.dy, p.dx, x3, &pl);
    if (!slab && (x3 || !tc_plan_taps(p.N, p.H, p.W, p.C, p.dy, p.dx, &pl))) return LF_ERR_UNSUPPORTED;
    TcArgs a = pl.geo;
    a.out = p.out; a.bias = p.bias; a.mask_src = p.mask_src; a.add_src = p.add_src; a.add_mask = p.add_mask;
    a.colsum_partial = p.colsum_partial;
    a.stats_partial = p.stats_partial;
    a.mask_scale = p.mask_scale;
    a.mask_shift = p.mask_shift;
    a.N = p.N; a.H = p.H; a.W = p.W; a.Ctot = p.C; a.relu = p.relu;
    a.n_halves = p.C / TC_BN;
    a.total_m_tiles = p.N * a.tiles_a * a.tiles_b;

    TcEncodeTiledFn enc = tc_get_encode_fn();
    CUtensorMap tmA, tmB;
    {
        // activations [N,H,W,C] viewed as (ci:32, cblk:C/32, across, along, n); one box = the slab or one tap's patch
        const cuuint64_t sx = (cuuint64_t)p.C * 4, sy = (cuuint64_t)p.W * p.C * 4;
        cuuint64_t dims[5] = {32, (cuuint64_t)(p.C / 32), (cuuint64_t)(a.vertical ? p.W : p.H),
                              (cuuint64_t)(a.vertical ? p.H : p.W), (cuuint64_t)p.N};
        cuuint64_t strides[4] = {128, a.vertical ? sx : sy, a.vertical ? sy : sx, (cuuint64_t)p.H * p.W * p.C * 4};
        cuuint32_t box[5] = {32, 1, (cuuint32_t)a.TB, (cuuint32_t)(a.load_rows / a.TB), 1};
        cuuint32_t estr[5] = {1, 1, 1, 1, 1};
        CUresult r = enc(&tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(p.in), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return LF_ERR_CUDA;
    }
    {
        // packed weights [Cout][3*C] (K contiguous); 3xTF32: [2][Cout][3*C] (hi, lo) as one [2*Cout][3*C] matrix
        cuuint64_t dims[2] = {(cuuint64_t)(3 * p.C), (cuuint64_t)((x3 ? 2 : 1) * p.C)};
        cuuint64_t strides[1] = {(cuuint64_t)(3 * p.C) * 4};
        cuuint32_t box[2] = {32, TC_BN};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(p.wpack), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return LF_ERR_CUDA;
    }
    const int grid = pl.m_ctas * a.n_halves;
    const int s = pl.smem_bytes;
    cudaError_t e;
    if (p.C == 128) {
        if (x3) e = pl.res ? tc_launch<128, true, true>(grid, s, stream, tmA, tmB, a) : tc_launch<128, true, false>(grid, s, stream, tmA, tmB, a);
        else e = pl.res ? tc_launch<128, false, true>(grid, s, stream, tmA, tmB, a) : tc_launch<128, false, false>(grid, s, stream, tmA, tmB, a);
    } else {
        if (x3) e = pl.res ? tc_launch<64, true, true>(grid, s, stream, tmA, tmB, a) : tc_launch<64, true, false>(grid, s, stream, tmA, tmB, a);
        else e = pl.res ? tc_launch<64, false, true>(grid, s, stream, tmA, tmB, a) : tc_launch<64, false, false>(grid, s, stream, tmA, tmB, a);
    }
    if (e != cudaSuccess) { set_last_cuda_error(e); return LF_ERR_CUDA; }
    return check_launch();
}

}  // namespace lf

using namespace lf;

extern "C" void lf_conv1d_tc_set_variant(int v) { g_tc_variant = (v == 1) ? 1 : 2; }

// 0 if the shape is unsupported, else the number of rows of the optional colsum_partial / stats_partial outputs.  Every
// shape the slab plan takes is also taken by the per-tap plan (same number of CTAs), which serves the TF32 calls the slab
// does not fit.
extern "C" int lf_conv1d_tc_supported(int N, int H, int W, int C) {
    TcPlan pl{};
    return tc_plan_taps(N, H, W, C, nullptr, nullptr, &pl) ? pl.m_ctas : 0;
}

// 1 if a TF32 call with these taps runs on the halo-slab path
extern "C" int lf_conv1d_tc_slab_ok(int N, int H, int W, int C, int vertical, int dil) {
    if (g_tc_variant == 1 || dil < 1) return 0;
    TcPlan pl{};
    const int zero[3] = {0, 0, 0}, off[3] = {-dil, 0, dil};
    return tc_plan_slab(N, H, W, C, vertical ? off : zero, vertical ? zero : off, false, &pl) ? 1 : 0;
}

// rows of colsum_partial / stats_partial (= CTAs per 64-channel half), 0 if a 3xTF32 call with these taps is not served
extern "C" int lf_conv1d_tc_x3_rows(int N, int H, int W, int C, int vertical, int dil) {
    if (dil < 1) return 0;
    TcPlan pl{};
    const int zero[3] = {0, 0, 0}, off[3] = {-dil, 0, dil};
    return tc_plan_slab(N, H, W, C, vertical ? off : zero, vertical ? zero : off, true, &pl) ? pl.m_ctas : 0;
}

extern "C" int lf_conv1d_tc(const LfConvTcArgs* args, lf_stream_t stream) { return tc_run(args, stream, false); }
extern "C" int lf_conv1d_tc_x3(const LfConvTcArgs* args, lf_stream_t stream) { return tc_run(args, stream, true); }
