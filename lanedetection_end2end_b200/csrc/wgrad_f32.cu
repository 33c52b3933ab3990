// Weight gradients as a split-K GEMM over pixels (fp32 CUDA cores, parity mode) plus the
// deterministic split reductions.  See LfWgradArgs in include/lanefit_b200.h.
// Replaces autograd's convolution_backward weight/bias paths for every Conv2d /
// ConvTranspose2d of BP/Networks/ERFNet.py (:15,29-37,101).
#include "lf_common.cuh"

namespace lf {

constexpr int WG_TILE = 64;       // padding granularity of the partial buffers
constexpr int WG_THREADS = 256;

// CTA tile TP x TQ of the weight gradient; every thread owns a 4x4 micro-tile.  When the tile needs
// fewer than 256 threads (small channel counts: stem, C=16 blocks, 64->16 upsampler) the CTA splits
// its pixels over G = 256 / ((TP/4)*(TQ/4)) thread groups and reduces them through shared memory at
// the end, so no FMA is spent on zero padding.
template <int TP, int TQ>
struct WgCfg {
    static constexpr int TPG = (TP / 4) * (TQ / 4);   // threads per pixel group
    static constexpr int G = WG_THREADS / TPG;        // pixel groups
    static constexpr int PXG = (TP == 16 && TQ == 16) ? 8 : 16;  // pixels per group and step
    static constexpr int PXS = PXG * G;               // pixels per step
    static constexpr int PF4 = PXS * TP / 4, QF4 = PXS * TQ / 4;  // float4 per tile
    static constexpr int PL = (PF4 + WG_THREADS - 1) / WG_THREADS, QL = (QF4 + WG_THREADS - 1) / WG_THREADS;
    static constexpr int SMEM_FLOATS = 2 * PXS * (TP + TQ);
    static_assert(TPG * G == WG_THREADS, "tile");
    static_assert(SMEM_FLOATS * 4 <= 48 * 1024, "smem");
    static_assert(G == 1 || G * TP * TQ <= SMEM_FLOATS, "group reduction reuses the tile buffers");
};

template <int TP, int TQ>
__global__ void __launch_bounds__(WG_THREADS) wgrad_f32_kernel(const WgradArgs a) {
    pdl_entry();
    using Cfg = WgCfg<TP, TQ>;
    __shared__ __align__(16) float smem[Cfg::SMEM_FLOATS];
    float(*Ps)[Cfg::PXS][TP] = reinterpret_cast<float(*)[Cfg::PXS][TP]>(smem);
    float(*Qs)[Cfg::PXS][TQ] = reinterpret_cast<float(*)[Cfg::PXS][TQ]>(smem + 2 * Cfg::PXS * TP);
    const int tid = threadIdx.x;
    // 16-wide tiles cover the (<= 16) real channels of a 64-padded buffer with ONE tile (host agrees)
    const int tilesQ = (TQ == 16) ? 1 : a.CqPad / TQ, tilesP = (TP == 16) ? 1 : a.CpPad / TP;
    const int tq = blockIdx.x % tilesQ;
    const int tp = (blockIdx.x / tilesQ) % tilesP;
    const int t = blockIdx.x / (tilesQ * tilesP);
    const int split = blockIdx.y;
    // 32-bit pixel arithmetic (the host guarantees N*Hs*Ws < 2^31): the index math is on the critical path
    const int M = a.N * a.Hs * a.Ws;
    int per = (M + a.nsplit - 1) / a.nsplit;
    per = ((per + Cfg::PXS - 1) / Cfg::PXS) * Cfg::PXS;
    const int m_begin = min(M, split * per);
    const int m_end = min(M, m_begin + per);
    const int HW = a.Hs * a.Ws;

    const int g = tid / Cfg::TPG, r = tid % Cfg::TPG;
    const int tx = r % (TQ / 4), ty = r / (TQ / 4);
    const int pdy = a.pdy[t], pdx = a.pdx[t], qdy = a.qdy[t], qdx = a.qdx[t];
    const bool do_qsum = (a.qsum_partial != nullptr) && t == 0 && tp == 0 && ty == 0;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[i][c] = 0.f;
    float qs[4] = {0.f, 0.f, 0.f, 0.f};

    float4 rp[Cfg::PL], rq[Cfg::QL];
    auto load = [&](int m0) {
#pragma unroll
        for (int q = 0; q < Cfg::PL; ++q) {
            rp[q] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int f = tid + q * WG_THREADS;
            if (f < Cfg::PF4) {
                const int lp = f / (TP / 4), c4 = f % (TP / 4);
                const int m = m0 + lp;
                const int cp0 = tp * TP + 4 * c4;
                if (m < m_end && cp0 < a.Cp) {
                    const int n = m / HW;
                    const int rem = m - n * HW;
                    const int j = rem / a.Ws, i = rem - j * a.Ws;
                    const int py = j * a.psy + pdy, px = i * a.psx + pdx;
                    if (py >= 0 && py < a.Hp && px >= 0 && px < a.Wp)
                        rp[q] = __ldg(reinterpret_cast<const float4*>(
                            a.P + ((size_t)(n * a.Hp + py) * a.Wp + px) * a.p_cstride + a.p_coff + cp0));
                }
            }
        }
#pragma unroll
        for (int q = 0; q < Cfg::QL; ++q) {
            rq[q] = make_float4(0.f, 0.f, 0.f, 0.f);
            const int f = tid + q * WG_THREADS;
            if (f < Cfg::QF4) {
                const int lp = f / (TQ / 4), c4 = f % (TQ / 4);
                const int m = m0 + lp;
                const int cq0 = tq * TQ + 4 * c4;
                if (m < m_end && cq0 < a.Cq) {
                    const int n = m / HW;
                    const int rem = m - n * HW;
                    const int j = rem / a.Ws, i = rem - j * a.Ws;
                    const int qy = j * a.qsy + qdy, qx = i * a.qsx + qdx;
                    if (qy >= 0 && qy < a.Hq && qx >= 0 && qx < a.Wq)
                        rq[q] = __ldg(reinterpret_cast<const float4*>(
                            a.Q + ((size_t)(n * a.Hq + qy) * a.Wq + qx) * a.q_cstride + a.q_coff + cq0));
                }
            }
        }
    };
    auto store = [&](int buf) {
#pragma unroll
        for (int q = 0; q < Cfg::PL; ++q) {
            const int f = tid + q * WG_THREADS;
            if (f < Cfg::PF4) *reinterpret_cast<float4*>(&Ps[buf][f / (TP / 4)][4 * (f % (TP / 4))]) = rp[q];
        }
#pragma unroll
        for (int q = 0; q < Cfg::QL; ++q) {
            const int f = tid + q * WG_THREADS;
            if (f < Cfg::QF4) *reinterpret_cast<float4*>(&Qs[buf][f / (TQ / 4)][4 * (f % (TQ / 4))]) = rq[q];
        }
    };

    if (m_begin < m_end) {
        load(m_begin);
        store(0);
    }
    __syncthreads();
    int it = 0;
    for (int m0 = m_begin; m0 < m_end; m0 += Cfg::PXS, ++it) {
        const int buf = it & 1;
        const bool more = (m0 + Cfg::PXS) < m_end;
        if (more) load(m0 + Cfg::PXS);
#pragma unroll
        for (int pp = 0; pp < Cfg::PXG; ++pp) {
            const int p = pp * Cfg::G + g;  // groups interleave the pixels of a step
            const float4 av = *reinterpret_cast<const float4*>(&Ps[buf][p][4 * ty]);
            const float4 bv = *reinterpret_cast<const float4*>(&Qs[buf][p][4 * tx]);
            const float aa[4] = {av.x, av.y, av.z, av.w};
            const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[i][c] = fmaf(aa[i], bb[c], acc[i][c]);
            if (do_qsum) {
                qs[0] += bb[0]; qs[1] += bb[1]; qs[2] += bb[2]; qs[3] += bb[3];
            }
        }
        if (more) store(buf ^ 1);
        __syncthreads();
    }
    float* dst = a.partial + (((size_t)split * a.ntaps + t) * a.CpPad + tp * TP) * a.CqPad + tq * TQ;
    float* qdst = a.qsum_partial ? a.qsum_partial + (size_t)split * a.CqPad + tq * TQ : nullptr;
    if (Cfg::G == 1) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
            *reinterpret_cast<float4*>(dst + (size_t)(4 * ty + i) * a.CqPad + 4 * tx) =
                make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        if (do_qsum) *reinterpret_cast<float4*>(qdst + 4 * tx) = make_float4(qs[0], qs[1], qs[2], qs[3]);
    } else {
        // fixed-order reduction over the G pixel groups through shared memory (tiles are free now)
        float* red = smem;  // [G][TP][TQ]
#pragma unroll
        for (int i = 0; i < 4; ++i)
            *reinterpret_cast<float4*>(&red[((size_t)g * TP + 4 * ty + i) * TQ + 4 * tx]) =
                make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        __syncthreads();
        for (int e = tid; e < TP * TQ; e += WG_THREADS) {
            float sum = 0.f;
#pragma unroll
            for (int gg = 0; gg < Cfg::G; ++gg) sum += red[(size_t)gg * TP * TQ + e];
            dst[(size_t)(e / TQ) * a.CqPad + (e % TQ)] = sum;
        }
        if (a.qsum_partial != nullptr && t == 0 && tp == 0) {
            __syncthreads();
            if (ty == 0) *reinterpret_cast<float4*>(&red[g * TQ + 4 * tx]) = make_float4(qs[0], qs[1], qs[2], qs[3]);
            __syncthreads();
            for (int e = tid; e < TQ; e += WG_THREADS) {
                float sum = 0.f;
#pragma unroll
                for (int gg = 0; gg < Cfg::G; ++gg) sum += red[gg * TQ + e];
                qdst[e] = sum;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// Small-channel weight gradient (stem 3->13, 16->48 downsampler, 64->16 upsampler): all taps in one CTA.
// Per pixel m the gradient is an outer product U^T V with
//   taps on P (Conv2d):          U = concat_t P[m*s + tap_t] (ntaps*Cp values),  V = Q[m] (Cq values)
//   taps on Q (ConvTranspose2d): U = P[m] (Cp values),  V = concat_t Q[m*s + tap_t] (ntaps*Cq values).
// A thread owns a 4 (U) x 16 (V) register tile: 5 shared-memory loads per 64 FMAs, no zero padding of the
// channel dimensions to 64, and Q / P are staged once for all taps.  (LU/4)*(LV/16) threads cover one
// pixel; the CTA runs G such pixel groups side by side and sums them in fixed order at the end.
// The generic tile kernel above spent 316-443 us per launch on these layers; this one is FMA/HBM-bound.
// ------------------------------------------------------------------------------------------
struct WsPlan {
    int LU, LV, TPG, G, PXG, PXS, threads, taps_on_p, smem_bytes, ppp, passes;
};

static bool ws_make_plan(const WgradArgs& a, WsPlan* p) {
    bool p_same = true, q_same = true;
    for (int t = 1; t < a.ntaps; ++t) {
        p_same = p_same && a.pdy[t] == a.pdy[0] && a.pdx[t] == a.pdx[0];
        q_same = q_same && a.qdy[t] == a.qdy[0] && a.qdx[t] == a.qdx[0];
    }
    if (a.ntaps > 1 && p_same == q_same) return false;  // exactly one side may be gathered per tap
    if (a.Cp > 16 && a.Cq > 16) return false;            // the 64x64 tile kernel serves the wide layers
    p->taps_on_p = (a.ntaps == 1) || !p_same;
    if (!p->taps_on_p && (a.qsum_partial || a.Cq % 16 != 0)) return false;
    p->LU = p->taps_on_p ? a.ntaps * a.Cp : a.Cp;
    p->LV = p->taps_on_p ? a.Cq : a.ntaps * a.Cq;
    if (p->LU % 4 != 0 || p->LV % 16 != 0) return false;
    p->TPG = (p->LU / 4) * (p->LV / 16);
    if (p->TPG > 256 || p->TPG < 1) return false;
    p->G = 256 / p->TPG;
    p->threads = ((p->G * p->TPG + 31) / 32) * 32;
    p->PXG = p->G >= 8 ? 4 : (p->G >= 2 ? 16 : 32);
    p->PXS = p->PXG * p->G;
    const int per_px4 = (p->LU + p->LV) / 4;
    if (per_px4 > p->threads) return false;
    p->ppp = p->threads / per_px4;                       // pixels fetched per pass (one float4 per thread)
    p->passes = (p->PXS + p->ppp - 1) / p->ppp;
    const int tile_floats = 2 * p->PXS * (p->LU + p->LV);
    if (p->G > 1 && p->LU * p->LV + p->LV > tile_floats) return false;  // group reduction reuses the tiles
    p->smem_bytes = tile_floats * 4;
    return p->smem_bytes <= 96 * 1024;
}

__device__ __forceinline__ void ws_cp_async16(float* smem_dst, const float* gsrc, bool valid) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    const int bytes = valid ? 16 : 0;  // 0 -> the 16 destination bytes are zero-filled, nothing is read
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(bytes) : "memory");
}

__global__ void __launch_bounds__(256, 2) wgrad_small_kernel(const WgradArgs a, const WsPlan pl) {
    pdl_entry();
    extern __shared__ __align__(16) float ws_smem[];
    const int LU = pl.LU, LV = pl.LV, PXS = pl.PXS, G = pl.G;
    float* sU = ws_smem;                  // [2][PXS][LU]
    float* sV = ws_smem + 2 * PXS * LU;   // [2][PXS][LV]
    const int tid = threadIdx.x;
    const int split = blockIdx.x;
    const int M = a.N * a.Hs * a.Ws;
    int per = (M + a.nsplit - 1) / a.nsplit;
    per = ((per + PXS - 1) / PXS) * PXS;
    const int m_begin = min(M, split * per);
    const int m_end = min(M, m_begin + per);
    const int HW = a.Hs * a.Ws;

    // ---- fetch role: this thread always fetches float4 number `e` of a pixel's (U | V) vector, for pixel
    // lp0, lp0 + ppp, ... of the step (cp.async straight into shared memory, zero fill outside the image)
    const int nU4 = LU / 4, per_px4 = (LU + LV) / 4;
    const int lp0 = tid / per_px4, e = tid - lp0 * per_px4;
    const bool fetcher = lp0 < pl.ppp;
    const bool is_u = e < nU4;
    int f_dy, f_dx, f_goff, f_soff;
    if (is_u) {
        const int u = 4 * e;
        const int t = pl.taps_on_p ? u / a.Cp : 0;
        f_goff = a.p_coff + (pl.taps_on_p ? u - t * a.Cp : u);
        f_dy = a.pdy[t]; f_dx = a.pdx[t]; f_soff = u;
    } else {
        const int v = 4 * (e - nU4);
        const int t = pl.taps_on_p ? 0 : v / a.Cq;
        f_goff = a.q_coff + (pl.taps_on_p ? v : v - t * a.Cq);
        f_dy = a.qdy[t]; f_dx = a.qdx[t]; f_soff = v;
    }
    const float* f_base = is_u ? a.P : a.Q;
    const int f_H = is_u ? a.Hp : a.Hq, f_W = is_u ? a.Wp : a.Wq, f_cs = is_u ? a.p_cstride : a.q_cstride;
    const int f_sy = is_u ? a.psy : a.qsy, f_sx = is_u ? a.psx : a.qsx;
    const int f_L = is_u ? LU : LV;
    auto fetch = [&](int m0, int buf) {
        if (!fetcher) return;
        float* sdst = (is_u ? sU + buf * PXS * LU : sV + buf * PXS * LV) + f_soff;
        // decode the first pixel once, then step by ppp pixels with carries (no division per pixel)
        int m = m0 + lp0;
        int n = m / HW;
        int rem = m - n * HW;
        int j = rem / a.Ws, i = rem - j * a.Ws;
        for (int k = 0, lp = lp0; k < pl.passes; ++k, lp += pl.ppp, m += pl.ppp) {
            if (lp < PXS) {
                const int y = j * f_sy + f_dy, x = i * f_sx + f_dx;
                const bool ok = m < m_end && y >= 0 && y < f_H && x >= 0 && x < f_W;
                const float* src = ok ? f_base + ((size_t)(n * f_H + y) * f_W + x) * f_cs + f_goff : f_base;
                ws_cp_async16(sdst + lp * f_L, src, ok);
            }
            i += pl.ppp;
            while (i >= a.Ws) { i -= a.Ws; ++j; }
            while (j >= a.Hs) { j -= a.Hs; ++n; }
        }
    };

    // ---- compute role
    const bool active = tid < G * pl.TPG;
    const int g = tid / pl.TPG, r = tid - g * pl.TPG;
    // U index fastest inside a warp: a quarter-warp reads 8 consecutive float4s of U (conflict-free) and ONE
    // broadcast address of V.  (V fastest made every V load a 4-way bank conflict: 64-byte stride.)
    const int nug = LU / 4;
    const int vg = r / nug, ug = r - vg * nug;
    const bool do_qsum = active && a.qsum_partial != nullptr && ug == 0;
    float acc[4][16];
    float qs[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        qs[c] = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i][c] = 0.f;
    }

    if (m_begin < m_end) fetch(m_begin, 0);
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    int it = 0;
    for (int m0 = m_begin; m0 < m_end; m0 += PXS, ++it) {
        const int buf = it & 1;
        if (m0 + PXS < m_end) fetch(m0 + PXS, buf ^ 1);
        asm volatile("cp.async.commit_group;" ::: "memory");
        if (active) {
            const float* bu = sU + buf * PXS * LU + 4 * ug;
            const float* bv = sV + buf * PXS * LV + 16 * vg;
#pragma unroll 2
            for (int pp = 0; pp < pl.PXG; ++pp) {
                const int p = pp * G + g;  // groups interleave the pixels of a step
                const float4 u4 = *reinterpret_cast<const float4*>(bu + p * LU);
                const float uu[4] = {u4.x, u4.y, u4.z, u4.w};
                float vv[16];
#pragma unroll
                for (int c4 = 0; c4 < 4; ++c4) {
                    const float4 v4 = *reinterpret_cast<const float4*>(bv + p * LV + 4 * c4);
                    vv[4 * c4] = v4.x; vv[4 * c4 + 1] = v4.y; vv[4 * c4 + 2] = v4.z; vv[4 * c4 + 3] = v4.w;
                }
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int c = 0; c < 16; ++c) acc[i][c] = fmaf(uu[i], vv[c], acc[i][c]);
                if (do_qsum) {
#pragma unroll
                    for (int c = 0; c < 16; ++c) qs[c] += vv[c];
                }
            }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
    }

    // ---- write [t][cp][cq] partials (fixed-order sum over the G pixel groups through shared memory)
    float* dst = a.partial + (size_t)split * a.ntaps * a.CpPad * a.CqPad;
    auto out_index = [&](int u, int v) -> size_t {
        int t, cp, cq;
        if (pl.taps_on_p) {
            t = u / a.Cp; cp = u - t * a.Cp; cq = v;
        } else {
            t = v / a.Cq; cq = v - t * a.Cq; cp = u;
        }
        return ((size_t)t * a.CpPad + cp) * a.CqPad + cq;
    };
    if (G == 1) {
        if (active) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int c4 = 0; c4 < 4; ++c4)
                    *reinterpret_cast<float4*>(dst + out_index(4 * ug + i, 16 * vg + 4 * c4)) =
                        make_float4(acc[i][4 * c4], acc[i][4 * c4 + 1], acc[i][4 * c4 + 2], acc[i][4 * c4 + 3]);
            if (do_qsum) {
#pragma unroll
                for (int c = 0; c < 16; ++c) a.qsum_partial[(size_t)split * a.CqPad + 16 * vg + c] = qs[c];
            }
        }
        return;
    }
    float* red = ws_smem;         // [LU][LV] then [LV] for the bias sums
    float* redq = ws_smem + LU * LV;
    for (int gg = 0; gg < G; ++gg) {
        if (active && g == gg) {
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int c = 0; c < 16; ++c) {
                    float* ep = red + (4 * ug + i) * LV + 16 * vg + c;
                    *ep = (gg == 0) ? acc[i][c] : *ep + acc[i][c];
                }
            if (do_qsum) {
#pragma unroll
                for (int c = 0; c < 16; ++c) {
                    float* ep = redq + 16 * vg + c;
                    *ep = (gg == 0) ? qs[c] : *ep + qs[c];
                }
            }
        }
        __syncthreads();
    }
    for (int o = tid; o < LU * LV; o += blockDim.x) dst[out_index(o / LV, o % LV)] = red[o];
    if (a.qsum_partial != nullptr)
        for (int o = tid; o < LV; o += blockDim.x) a.qsum_partial[(size_t)split * a.CqPad + o] = redq[o];
}

// dst[t*st + cp*sp + cq*sq] = sum_k partial[k][t][cp][cq], fixed order.  One thread = 4 consecutive cq
// (float4 loads) x one of 8 split lanes (k = lane, lane+8, ...); the 8 lanes are combined through
// shared memory in lane order -> deterministic, 8x shorter dependent chains than one thread per output.
constexpr int WR_LANES = 8;
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float* __restrict__ partial, int nsplit, int ntaps, int Cp,
                                                            int Cq, int CpPad, int CqPad, float* __restrict__ dst, int st, int sp,
                                                            int sq) {
    pdl_entry();
    __shared__ float4 red[256];
    const int Cq4 = (Cq + 3) >> 2;
    const int total4 = ntaps * Cp * Cq4;
    // thread = (output float4 `o`, split lane): a WARP covers 32 consecutive outputs of one split lane, so each load
    // instruction reads 512 contiguous bytes of one partial (the previous (o, lane) = (tid / 8, tid % 8) mapping read eight
    // 64-byte pieces 100s of KB apart: 36 % of the DRAM roof in the round-2 ncu capture); same per-lane k sequence and
    // the same lane-ordered combine, so the result is bit-identical
    const int o = blockIdx.x * (256 / WR_LANES) + (threadIdx.x & 31);
    const int lane = threadIdx.x >> 5;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int cq = 0, cp = 0, t = 0;
    if (o < total4) {
        cq = (o % Cq4) * 4;
        cp = (o / Cq4) % Cp;
        t = o / (Cq4 * Cp);
        const size_t stride = (size_t)ntaps * CpPad * CqPad;
        const float* p = partial + ((size_t)t * CpPad + cp) * CqPad + cq;   // CqPad % 64 == 0 -> 16B aligned
        int k = lane;
        for (; k + 3 * WR_LANES < nsplit; k += 4 * WR_LANES) {   // 4 loads in flight per lane, fixed order
            const float4 v0 = __ldg(reinterpret_cast<const float4*>(p + (size_t)k * stride));
            const float4 v1 = __ldg(reinterpret_cast<const float4*>(p + (size_t)(k + WR_LANES) * stride));
            const float4 v2 = __ldg(reinterpret_cast<const float4*>(p + (size_t)(k + 2 * WR_LANES) * stride));
            const float4 v3 = __ldg(reinterpret_cast<const float4*>(p + (size_t)(k + 3 * WR_LANES) * stride));
            acc.x += (v0.x + v1.x) + (v2.x + v3.x); acc.y += (v0.y + v1.y) + (v2.y + v3.y);
            acc.z += (v0.z + v1.z) + (v2.z + v3.z); acc.w += (v0.w + v1.w) + (v2.w + v3.w);
        }
        for (; k < nsplit; k += WR_LANES) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(p + (size_t)k * stride));
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    if (lane == 0 && o < total4) {
        float4 s4 = red[threadIdx.x];
#pragma unroll
        for (int l = 1; l < WR_LANES; ++l) {
            const float4 v = red[threadIdx.x + 32 * l];
            s4.x += v.x; s4.y += v.y; s4.z += v.z; s4.w += v.w;
        }
        const float vals[4] = {s4.x, s4.y, s4.z, s4.w};
        for (int e = 0; e < 4 && cq + e < Cq; ++e) dst[(size_t)t * st + (size_t)cp * sp + (size_t)(cq + e) * sq] = vals[e];
    }
}

// Several split reductions in one launch (blockIdx.y = job): the four weight gradients and two bias gradients
// of a non_bottleneck_1d block are ~12 us latency-bound launches each when reduced one by one.
struct ReduceJobs {
    LfReduceJob job[LF_REDUCE_MAX_JOBS];
    int njobs;
};
__global__ void __launch_bounds__(256) reduce_multi_kernel(const ReduceJobs js) {
    pdl_entry();
    __shared__ float4 red[256];
    const LfReduceJob& j = js.job[blockIdx.y];
    const int Cq4 = (j.Cq + 3) >> 2;
    const int total4 = j.ntaps * j.Cp * Cq4;
    if ((int)(blockIdx.x * (256 / WR_LANES)) >= total4) return;   // whole block beyond this job (uniform)
    const int o = blockIdx.x * (256 / WR_LANES) + (threadIdx.x & 31);   // warp = 32 consecutive outputs of one split lane
    const int lane = threadIdx.x >> 5;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int cq = 0, cp = 0, t = 0;
    if (o < total4) {
        cq = (o % Cq4) * 4;
        cp = (o / Cq4) % j.Cp;
        t = o / (Cq4 * j.Cp);
        const size_t stride = (size_t)j.ntaps * j.CpPad * j.CqPad;
        const float* p = j.partial + ((size_t)t * j.CpPad + cp) * j.CqPad + cq;
        int k = lane;
        for (; k + 3 * WR_LANES < j.nsplit; k += 4 * WR_LANES) {   // 4 loads in flight per lane, fixed order
            const float4 v0 = __ldg(reinterpret_cast<const float4*>(p + (size_t)k * stride));
            const float4 v1 = __ldg(reinterpret_cast<const float4*>(p + (size_t)(k + WR_LANES) * stride));
            const float4 v2 = __ldg(reinterpret_cast<const float4*>(p + (size_t)(k + 2 * WR_LANES) * stride));
            const float4 v3 = __ldg(reinterpret_cast<const float4*>(p + (size_t)(k + 3 * WR_LANES) * stride));
            acc.x += (v0.x + v1.x) + (v2.x + v3.x); acc.y += (v0.y + v1.y) + (v2.y + v3.y);
            acc.z += (v0.z + v1.z) + (v2.z + v3.z); acc.w += (v0.w + v1.w) + (v2.w + v3.w);
        }
        for (; k < j.nsplit; k += WR_LANES) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(p + (size_t)k * stride));
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    if (lane == 0 && o < total4) {
        float4 s4 = red[threadIdx.x];
#pragma unroll
        for (int l = 1; l < WR_LANES; ++l) {
            const float4 v = red[threadIdx.x + 32 * l];
            s4.x += v.x; s4.y += v.y; s4.z += v.z; s4.w += v.w;
        }
        const float vals[4] = {s4.x, s4.y, s4.z, s4.w};
        for (int e = 0; e < 4 && cq + e < j.Cq; ++e)
            j.dst[(size_t)t * j.st + (size_t)cp * j.sp + (size_t)(cq + e) * j.sq] = vals[e];
    }
}

__global__ void vec_reduce_kernel(const float* __restrict__ partial, int nsplit, int C, int Cpad, float* __restrict__ dst) {
    pdl_entry();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float s = 0.f;
    for (int k = 0; k < nsplit; ++k) s += partial[(size_t)k * Cpad + c];
    dst[c] = s;
}

constexpr int COLSUM_THREADS = 256;
static inline int colsum_max_blocks() { return device_sms() * 4; }
constexpr int COLSUM_MIN_PIX = 128;

// partial[blk][c] = sum over the block's pixel range of src[p*cstride + coff + c].
// Thread -> (pixel lane, channel); channels fastest so a warp reads contiguous memory.
__global__ void __launch_bounds__(COLSUM_THREADS) colsum_kernel(const float* __restrict__ src, long long npix, int C,
                                                                 int cstride, int coff, float* __restrict__ partial, int Cpad) {
    pdl_entry();
    __shared__ float red[COLSUM_THREADS];
    const int tid = threadIdx.x;
    const long long per = (npix + gridDim.x - 1) / gridDim.x;
    const long long p0 = (long long)blockIdx.x * per;
    const long long p1 = min(npix, p0 + per);
    for (int cbase = 0; cbase < C; cbase += COLSUM_THREADS) {
        const int cw = min(C - cbase, COLSUM_THREADS);
        const int lanes = COLSUM_THREADS / cw;
        const int c = tid % cw, pl = tid / cw;
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;   // 4 independent chains hide the load latency
        if (pl < lanes) {
            long long p = p0 + pl;
            for (; p + 3LL * lanes < p1; p += 4LL * lanes) {
                s0 += src[(size_t)p * cstride + coff + cbase + c];
                s1 += src[(size_t)(p + lanes) * cstride + coff + cbase + c];
                s2 += src[(size_t)(p + 2LL * lanes) * cstride + coff + cbase + c];
                s3 += src[(size_t)(p + 3LL * lanes) * cstride + coff + cbase + c];
            }
            for (; p < p1; p += lanes) s0 += src[(size_t)p * cstride + coff + cbase + c];
        }
        red[tid] = (pl < lanes) ? (s0 + s1) + (s2 + s3) : 0.f;
        __syncthreads();
        if (tid < cw) {
            float tot = 0.f;
            for (int l = 0; l < lanes; ++l) tot += red[l * cw + tid];
            partial[(size_t)blockIdx.x * Cpad + cbase + tid] = tot;
        }
        __syncthreads();
    }
}

}  // namespace lf

using namespace lf;

extern "C" int lf_wgrad_f32(const LfWgradArgs* args, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!args) return LF_ERR_INVALID_ARGUMENT;
    const WgradArgs& a = *args;
    LF_REQUIRE(a.P && a.Q && a.partial);
    LF_REQUIRE(a.N > 0 && a.Hs > 0 && a.Ws > 0 && a.ntaps >= 1 && a.ntaps <= LF_MAX_TAPS && a.nsplit >= 1);
    LF_REQUIRE(a.Cp % 4 == 0 && a.Cq % 4 == 0 && a.p_cstride % 4 == 0 && a.q_cstride % 4 == 0);
    LF_REQUIRE(a.p_coff % 4 == 0 && a.q_coff % 4 == 0);
    LF_REQUIRE(a.CpPad % WG_TILE == 0 && a.CqPad % WG_TILE == 0 && a.CpPad >= a.Cp && a.CqPad >= a.Cq);
    LF_REQUIRE((long long)a.N * a.Hs * a.Ws + 4096 < (1ll << 31));
    WsPlan wsp;
    if (ws_make_plan(a, &wsp)) {
        cudaError_t e = cudaFuncSetAttribute(wgrad_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
        if (e != cudaSuccess) { set_last_cuda_error(e); return LF_ERR_CUDA; }
        lf_launch(wgrad_small_kernel, a.nsplit, wsp.threads, wsp.smem_bytes, stream, a, wsp);
        return check_launch();
    }
    const bool smallP = a.Cp <= 16, smallQ = a.Cq <= 16;
    const int TP = smallP ? 16 : 64, TQ = smallQ ? 16 : 64;
    // small tiles only cover the first 16 channels of the 64-padded buffers: one tile in that dimension
    const int tilesP = smallP ? 1 : a.CpPad / 64, tilesQ = smallQ ? 1 : a.CqPad / 64;
    const WgradArgs& b = a;
    dim3 grid(tilesP * tilesQ * a.ntaps, a.nsplit);
    if (smallP && smallQ)
        lf_launch(wgrad_f32_kernel<16, 16>, grid, WG_THREADS, 0, stream, b);
    else if (smallP)
        lf_launch(wgrad_f32_kernel<16, 64>, grid, WG_THREADS, 0, stream, b);
    else if (smallQ)
        lf_launch(wgrad_f32_kernel<64, 16>, grid, WG_THREADS, 0, stream, b);
    else
        lf_launch(wgrad_f32_kernel<64, 64>, grid, WG_THREADS, 0, stream, b);
    return check_launch();
}

// Split count the small-channel kernel wants for these arguments (its grid IS the split count: two CTAs per
// SM), or 0 when the generic tile kernel will run and the caller's own choice stands.
extern "C" int lf_wgrad_f32_nsplit(const LfWgradArgs* args) {
    if (!args) return 0;
    WsPlan wsp;
    if (!ws_make_plan(*args, &wsp)) return 0;
    const int sms = device_sms();
    const long long M = (long long)args->N * args->Hs * args->Ws;
    long long n = 2LL * sms;
    const long long max_split = (M + 4LL * wsp.PXS - 1) / (4LL * wsp.PXS);   // at least 4 steps per CTA
    if (n > max_split) n = max_split;
    return (int)(n < 1 ? 1 : n);
}

extern "C" int lf_wgrad_reduce(const float* partial, int nsplit, int ntaps, int Cp, int Cq, int CpPad, int CqPad,
                               float* dst, int st, int sp, int sq, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(partial && dst && nsplit >= 1 && ntaps >= 1 && Cp >= 1 && Cq >= 1);
    LF_REQUIRE(CqPad % 4 == 0);
    const int total4 = ntaps * Cp * ((Cq + 3) / 4);
    const int per_block = 256 / WR_LANES;
    lf_launch(wgrad_reduce_kernel, (total4 + per_block - 1) / per_block, 256, 0, stream, partial, nsplit, ntaps, Cp, Cq, CpPad, CqPad,
                                                                                   dst, st, sp, sq);
    return check_launch();
}

extern "C" int lf_reduce_multi(const LfReduceJob* jobs, int njobs, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(jobs && njobs >= 1 && njobs <= LF_REDUCE_MAX_JOBS);
    ReduceJobs js{};
    js.njobs = njobs;
    int max_blocks = 1;
    const int per_block = 256 / WR_LANES;
    for (int i = 0; i < njobs; ++i) {
        const LfReduceJob& j = jobs[i];
        LF_REQUIRE(j.partial && j.dst && j.nsplit >= 1 && j.ntaps >= 1 && j.Cp >= 1 && j.Cq >= 1 && j.CqPad % 4 == 0);
        js.job[i] = j;
        const int total4 = j.ntaps * j.Cp * ((j.Cq + 3) / 4);
        const int nb = (total4 + per_block - 1) / per_block;
        if (nb > max_blocks) max_blocks = nb;
    }
    lf_launch(reduce_multi_kernel, dim3(max_blocks, njobs), 256, 0, stream, js);
    return check_launch();
}

extern "C" int lf_vec_reduce(const float* partial, int nsplit, int C, int Cpad, float* dst, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(partial && dst && nsplit >= 1 && C >= 1 && Cpad >= C);
    lf_launch(vec_reduce_kernel, (C + 127) / 128, 128, 0, stream, partial, nsplit, C, Cpad, dst);
    return check_launch();
}

extern "C" int lf_colsum_blocks(long long npix) {
    long long b = (npix + COLSUM_MIN_PIX - 1) / COLSUM_MIN_PIX;
    if (b > colsum_max_blocks()) b = colsum_max_blocks();
    return (int)(b < 1 ? 1 : b);
}

extern "C" int lf_colsum(const float* src, long long npix, int C, int cstride, int coff, float* partial, int Cpad,
                         lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(src && partial && npix > 0 && C >= 1 && Cpad >= C);
    lf_launch(colsum_kernel, lf_colsum_blocks(npix), COLSUM_THREADS, 0, stream, src, npix, C, cstride, coff, partial, Cpad);
    return check_launch();
}
