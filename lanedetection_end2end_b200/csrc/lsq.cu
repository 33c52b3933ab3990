// Fused weighted least-squares layer for sm_90a:  activation -> row mask ->
// moments of (m*a(o))^2 over the BEV meshgrid -> (order+1)x(order+1) solve, and its
// closed-form backward.  Replaces BP/Networks/LSQ_layer.py:19-20,27-47,85-154,237-238,
// 295,301 and BP/Networks/gels.py:9-25 of the reference (see include/lanefit_b200.h).
//
// Design (DESIGN.md section "K5/K6"):
//  * HBM-bound: each map element is read exactly once (fwd) / read once + written once
//    (bwd); masked rows are never read.
//  * Row-separable fast path: for every homography the reference builds, y depends on
//    the row only, so  S_k = sum_r y_r^k A_r,  T_k = sum_r y_r^k B_r  with
//    A_r = sum_c w^2, B_r = sum_c w^2 x.  Per pixel only 2 fp32 accumulations; the
//    3d+2 moments are accumulated in fp64 once per row by one lane each ("lane k owns
//    moment k"), which keeps the kernel far from the fp64 pipe limit.
//  * x table reads (L2-resident, batch-invariant) are amortised over the lanes of an
//    image: one CTA handles (row chunk, image, up to 4 lanes).
//  * Cross-CTA reduction is deterministic: per-chunk partials in a workspace, the last
//    CTA to arrive (ticket atomic) sums them in fixed order and one thread per system
//    solves it in fp64 registers (LU with partial pivoting == torch.inverse, or
//    Cholesky == GELS).  No cuBLAS/cuSOLVER batched call, no host sync.
#include "lf_common.cuh"

namespace lf {

constexpr int LSQ_THREADS = 256;
constexpr int LSQ_WARPS = LSQ_THREADS / 32;
constexpr int LSQ_MAXL = 4;    // lanes handled by one CTA
constexpr int LSQ_MAXNM = 16;  // >= 3*LF_MAX_ORDER+2 = 14
constexpr int LSQ_ACT_RUNTIME = -1;

struct LsqArgs {
    const void* o;
    const float* xtab;
    const float* ytab;
    const float* yrow;
    int B, L, H, W, order, mask_rows, act, solver, rows_per_cta, nchunks;
    double reg_ls;
    double* beta;
    double* zinv;
    float* masked;
    int* status;
    double* partials;
    int* tickets;
    // backward only
    const double* gbeta;
    void* d_o;
};

// ---------------------------------------------------------------------------------
// activation and its derivative (BP/Networks/LSQ_layer.py:27-47)
// ---------------------------------------------------------------------------------
template <int ACT_T>
__device__ __forceinline__ float act_fn(float o, int act_rt) {
    const int act = (ACT_T == LSQ_ACT_RUNTIME) ? act_rt : ACT_T;
    switch (act) {
        case LF_ACT_SQUARE: return o * o;
        case LF_ACT_ABS: return fabsf(o);
        case LF_ACT_RELU: return fmaxf(o, 0.f);
        case LF_ACT_SIGMOID: return 1.f / (1.f + expf(-o));
        case LF_ACT_SOFTPLUS: return (o > 20.f) ? o : log1pf(expf(o));  // nn.Softplus threshold 20
        default: return o;
    }
}
// returns act'(o) * act(o)  (the product the backward needs), given a = act(o)
template <int ACT_T>
__device__ __forceinline__ float dact_times_act(float o, int act_rt) {
    const int act = (ACT_T == LSQ_ACT_RUNTIME) ? act_rt : ACT_T;
    switch (act) {
        case LF_ACT_SQUARE: return 2.f * o * o * o;
        case LF_ACT_ABS: return o;  // sign(o)*|o|
        case LF_ACT_RELU: return fmaxf(o, 0.f);
        case LF_ACT_SIGMOID: {
            float s = 1.f / (1.f + expf(-o));
            return s * (1.f - s) * s;
        }
        case LF_ACT_SOFTPLUS: {
            if (o > 20.f) return o;
            float e = expf(o);
            return (e / (1.f + e)) * log1pf(e);
        }
        default: return o;
    }
}

template <bool BF16>
__device__ __forceinline__ float4 load_map4(const void* base, size_t elem_off) {
    if (BF16) {
        const uint2* p = reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(base) + elem_off);
        return bf16x4_to_f4(ld_stream_u2(p));
    } else {
        return ld_stream_f4(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem_off));
    }
}
// V consecutive map elements per lane and load: 4 fp32 (16 B) or 8 bf16 (16 B)
template <bool BF16>
struct MapVec {
    static constexpr int V = BF16 ? 8 : 4;
};
template <bool BF16>
__device__ __forceinline__ void load_mapv(const void* base, size_t elem_off, float (&v)[MapVec<BF16>::V]) {
    if constexpr (BF16) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(base) + elem_off));
        const float4 a = bf16x4_to_f4(make_uint2(u.x, u.y)), b = bf16x4_to_f4(make_uint2(u.z, u.w));
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
        const float4 a = ld_stream_f4(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem_off));
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    }
}
template <bool BF16>
__device__ __forceinline__ void store_mapv(void* base, size_t elem_off, const float (&v)[MapVec<BF16>::V]) {
    if constexpr (BF16) {
        const uint2 a = f4_to_bf16x4(make_float4(v[0], v[1], v[2], v[3]));
        const uint2 b = f4_to_bf16x4(make_float4(v[4], v[5], v[6], v[7]));
        *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(base) + elem_off) = make_uint4(a.x, a.y, b.x, b.y);
    } else {
        st_stream_f4(reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + elem_off), make_float4(v[0], v[1], v[2], v[3]));
    }
}
template <int V>
__device__ __forceinline__ void load_xv(const float* xrow, int cv, float (&x)[V]) {
#pragma unroll
    for (int q = 0; q < V / 4; ++q) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(xrow) + cv * (V / 4) + q);
        x[4 * q] = t.x; x[4 * q + 1] = t.y; x[4 * q + 2] = t.z; x[4 * q + 3] = t.w;
    }
}

template <bool BF16>
__device__ __forceinline__ float load_map1(const void* base, size_t elem_off) {
    if (BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[elem_off]);
    return reinterpret_cast<const float*>(base)[elem_off];
}
template <bool BF16>
__device__ __forceinline__ void store_map4(void* base, size_t elem_off, float4 v) {
    if (BF16) {
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(base) + elem_off) = f4_to_bf16x4(v);
    } else {
        st_stream_f4(reinterpret_cast<float4*>(reinterpret_cast<float*>(base) + elem_off), v);
    }
}
template <bool BF16>
__device__ __forceinline__ void store_map1(void* base, size_t elem_off, float v) {
    if (BF16)
        reinterpret_cast<__nv_bfloat16*>(base)[elem_off] = __float2bfloat16(v);
    else
        reinterpret_cast<float*>(base)[elem_off] = v;
}

// ---------------------------------------------------------------------------------
// (order+1)x(order+1) solve in fp64, one thread per system.
//   Z_ij = S_{2d-i-j} + lambda*delta_ij,  X_i = T_{d-i}   (SURVEY.md Appendix C)
// ---------------------------------------------------------------------------------
template <int N>
__device__ int lsq_solve(const double* S, const double* T, double lambda, int solver, double* beta, double* zinv) {
    constexpr int d = N - 1;
    double Z[N][N], Inv[N][N], X[N];
    int st = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
#pragma unroll
        for (int j = 0; j < N; ++j) {
            Z[i][j] = S[2 * d - i - j] + (i == j ? lambda : 0.0);
            Inv[i][j] = (i == j) ? 1.0 : 0.0;
        }
        X[i] = T[d - i];
    }
    for (int k = 0; k <= 2 * d; ++k)
        if (!isfinite(S[k])) st |= LF_STATUS_NONFINITE;
    for (int k = 0; k <= d; ++k)
        if (!isfinite(T[k])) st |= LF_STATUS_NONFINITE;

    if (solver == LF_SOLVER_CHOLESKY) {
        // Z = U^T U (upper), as torch.cholesky(., upper=True) in gels.py:12
        double U[N][N];
        for (int i = 0; i < N; ++i)
            for (int j = 0; j < N; ++j) U[i][j] = 0.0;
        for (int j = 0; j < N; ++j) {
            double s = Z[j][j];
            for (int k = 0; k < j; ++k) s -= U[k][j] * U[k][j];
            if (!(s > 0.0)) {
                st |= LF_STATUS_NOT_POSDEF;
                s = 1.0;
            }
            const double ujj = sqrt(s);
            U[j][j] = ujj;
            for (int i = j + 1; i < N; ++i) {
                double v = Z[j][i];
                for (int k = 0; k < j; ++k) v -= U[k][j] * U[k][i];
                U[j][i] = v / ujj;
            }
        }
        // Inv = (U^T U)^-1 : solve U^T y = e_c, U x = y for every column c
        for (int c = 0; c < N; ++c) {
            double yv[N];
            for (int i = 0; i < N; ++i) {
                double v = (i == c) ? 1.0 : 0.0;
                for (int k = 0; k < i; ++k) v -= U[k][i] * yv[k];
                yv[i] = v / U[i][i];
            }
            for (int i = N - 1; i >= 0; --i) {
                double v = yv[i];
                for (int k = i + 1; k < N; ++k) v -= U[i][k] * Inv[k][c];
                Inv[i][c] = v / U[i][i];
            }
        }
    } else {
        // Gauss-Jordan with partial pivoting on [Z | I]  (torch.inverse, LSQ_layer.py:114)
        for (int col = 0; col < N; ++col) {
            int piv = col;
            double best = fabs(Z[col][col]);
            for (int r = col + 1; r < N; ++r) {
                double v = fabs(Z[r][col]);
                if (v > best) {
                    best = v;
                    piv = r;
                }
            }
            if (!(best > 0.0)) {
                st |= LF_STATUS_SINGULAR;
                break;
            }
            if (piv != col) {
                for (int j = 0; j < N; ++j) {
                    double t0 = Z[col][j];
                    Z[col][j] = Z[piv][j];
                    Z[piv][j] = t0;
                    double t1 = Inv[col][j];
                    Inv[col][j] = Inv[piv][j];
                    Inv[piv][j] = t1;
                }
            }
            const double ip = 1.0 / Z[col][col];
            for (int j = 0; j < N; ++j) {
                Z[col][j] *= ip;
                Inv[col][j] *= ip;
            }
            for (int r = 0; r < N; ++r) {
                if (r == col) continue;
                const double f = Z[r][col];
                for (int j = 0; j < N; ++j) {
                    Z[r][j] -= f * Z[col][j];
                    Inv[r][j] -= f * Inv[col][j];
                }
            }
        }
    }
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);
    for (int i = 0; i < N; ++i) {
        double b = 0.0;
        for (int j = 0; j < N; ++j) b += Inv[i][j] * X[j];  // beta = Z^-1 X  (:116)
        if (st & (LF_STATUS_SINGULAR | LF_STATUS_NOT_POSDEF)) b = qnan;
        if (!isfinite(b)) st |= LF_STATUS_NONFINITE;
        beta[i] = b;
        for (int j = 0; j < N; ++j) zinv[i * N + j] = Inv[i][j];
    }
    return st;
}

// Last-arriving CTA of a (image, lane-group): fixed-order sum of the per-chunk partials
// and the solves.  `mom` is shared memory [LSQ_MAXL][LSQ_MAXNM].
__device__ __noinline__ void lsq_finalize(const LsqArgs& a, int b, int l0, int nl, double (*mom)[LSQ_MAXNM], int ticket_idx) {
    const int t = threadIdx.x;
    const int d = a.order, NM = 3 * d + 2, n = d + 1;
    if (t < LSQ_MAXL * LSQ_MAXNM) {
        const int l = t / LSQ_MAXNM, k = t % LSQ_MAXNM;
        if (l < nl && k < NM) {
            const double* p = a.partials + ((size_t)(b * a.L + l0 + l) * a.nchunks) * NM + k;
            double s = 0.0;
            for (int c = 0; c < a.nchunks; ++c) s += __ldcg(p + (size_t)c * NM);
            mom[l][k] = s;
        }
    }
    __syncthreads();
    if (t < nl) {
        const int bl = b * a.L + l0 + t;
        const double* S = mom[t];
        const double* T = mom[t] + (2 * d + 1);
        double* beta = a.beta + (size_t)bl * n;
        double* zinv = a.zinv + (size_t)bl * n * n;
        int st = 0;
        switch (d) {
            case 0: st = lsq_solve<1>(S, T, a.reg_ls, a.solver, beta, zinv); break;
            case 1: st = lsq_solve<2>(S, T, a.reg_ls, a.solver, beta, zinv); break;
            case 2: st = lsq_solve<3>(S, T, a.reg_ls, a.solver, beta, zinv); break;
            case 3: st = lsq_solve<4>(S, T, a.reg_ls, a.solver, beta, zinv); break;
            default: st = lsq_solve<5>(S, T, a.reg_ls, a.solver, beta, zinv); break;
        }
        if (st) atomicOr(a.status, st);
    }
    if (t == 0) a.tickets[ticket_idx] = 0;  // leave the workspace reusable
}

// Resident CTAs per SM the row-separable kernels are compiled for (register cap 128 / 64 per thread): the forward keeps
// NL * RU * UNR 16-byte loads per thread in flight and needs the registers; memory-level parallelism comes from the
// batched loads, not from occupancy.
constexpr int LSQ_FWD_CTAS_PER_SM = 2;
constexpr int LSQ_BWD_CTAS_PER_SM = 4;

// Rows of chunk c.  The unmasked rows [mask_rows, H) and the masked rows [0, mask_rows) are BOTH split evenly over the
// chunks of a system: masked rows cost nothing (forward without `masked`) or a zero fill, so chunks of consecutive
// rows would leave the CTAs of the top of the image idle (round 1: 25 % of the CTAs had no work, 0.5 of the HBM roof).
__device__ __forceinline__ void lsq_chunk_rows(const LsqArgs& a, int chunk, int& m0, int& m1, int& r0, int& r1) {
    const long long n = a.nchunks, ha = a.H - a.mask_rows;
    m0 = (int)(chunk * (long long)a.mask_rows / n);
    m1 = (int)((chunk + 1) * (long long)a.mask_rows / n);
    r0 = a.mask_rows + (int)(chunk * ha / n);
    r1 = a.mask_rows + (int)((chunk + 1) * ha / n);
}

// Block-level tail shared by both forward kernels: red[warp][l][k] holds per-warp
// moment sums; write this chunk's partial, take a ticket, finalize if last.
__device__ void lsq_chunk_tail(const LsqArgs& a, double (*red)[LSQ_MAXL][LSQ_MAXNM], double (*mom)[LSQ_MAXNM], int chunk,
                               int b, int lg, int l0, int nl) {
    const int t = threadIdx.x;
    const int NM = 3 * a.order + 2;
    __syncthreads();
    if (t < LSQ_MAXL * LSQ_MAXNM) {
        const int l = t / LSQ_MAXNM, k = t % LSQ_MAXNM;
        if (l < nl && k < NM) {
            double s = 0.0;
#pragma unroll
            for (int w = 0; w < LSQ_WARPS; ++w) s += red[w][l][k];
            a.partials[((size_t)(b * a.L + l0 + l) * a.nchunks + chunk) * NM + k] = s;
        }
        __threadfence();  // writers only: publish this chunk's partial before the ticket is taken
    }
    __syncthreads();
    __shared__ int is_last;
    const int ticket_idx = b * gridDim.z + lg;
    if (t == 0) {
        const int tk = atomicAdd(&a.tickets[ticket_idx], 1);
        is_last = (tk == a.nchunks - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    lsq_finalize(a, b, l0, nl, mom, ticket_idx);
}

// Warp reduction of NV (2, 4 or 8) per-thread values at once: each butterfly step also halves the number of values a
// lane carries, so the whole reduction takes NV/2 + NV/4 + .. + 1 + (5 - log2 NV) shuffles instead of 5 * NV.
// Returns, in every lane, the warp total of ONE value: value i ends up in the lanes packed_holder<NV>(i) + {0 .. 32/NV - 1}.
template <int NV>
__device__ __forceinline__ float warp_sum_packed(float (&v)[NV], int lane) {
    int m = 16;
#pragma unroll
    for (int n = NV; n > 1; n >>= 1, m >>= 1) {
        const bool up = (lane & m) != 0;
#pragma unroll
        for (int i = 0; i < n / 2; ++i) {
            const float send = up ? v[i] : v[i + n / 2];
            const float keep = up ? v[i + n / 2] : v[i];
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
        }
    }
    float r = v[0];
#pragma unroll
    for (; m > 0; m >>= 1) r += __shfl_xor_sync(0xffffffffu, r, m);
    return r;
}
// first lane that holds the total of value i after warp_sum_packed<NV>: step s (mask 16 >> s) keeps the upper half of the
// remaining values in the lanes whose bit (4 - s) is set, i.e. lane bit (4 - s) = bit (log2 NV - 1 - s) of i
template <int NV>
__device__ __forceinline__ int packed_holder(int i) {
    constexpr int LOG = NV == 8 ? 3 : NV == 4 ? 2 : 1;
    int lane = 0;
#pragma unroll
    for (int s = 0; s < LOG; ++s)
        if ((i >> (LOG - 1 - s)) & 1) lane |= 16 >> s;
    return lane;
}

// ---------------------------------------------------------------------------------
// Forward, row-separable fast path.  grid = (nchunks, B, ceil(L/4)), 256 threads.
// ---------------------------------------------------------------------------------
// NL = lanes per CTA (compile time, so the loads of all lanes and column steps of a row are in flight
// together: the kernel is latency-bound otherwise -- long-scoreboard stalls).
template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_FWD_CTAS_PER_SM) lsq_fwd_rowsep_kernel(const LsqArgs a) {
    pdl_entry();
    __shared__ double red[LSQ_WARPS][LSQ_MAXL][LSQ_MAXNM];
    __shared__ double mom[LSQ_MAXL][LSQ_MAXNM];
    const int chunk = blockIdx.x, b = blockIdx.y, lg = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int l0 = lg * NL;
    const int nl = min(NL, a.L - l0);
    constexpr int UNR = (NL <= 2) ? 4 : 2;
    constexpr int NLP = NL <= 1 ? 1 : NL <= 2 ? 2 : 4;   // lanes padded to a power of two
    constexpr int NV = 2 * NLP;                          // values per packed warp reduction
    const int d = a.order, NM = 3 * d + 2;
    constexpr int V = MapVec<BF16>::V;
    const int WV = a.W / V;
    // lane k owns moment k:  k <= 2d -> S_k (power k of y, times A);  else T_{k-2d-1} (times B)
    const bool useB = lane > 2 * d;
    const int ek = useB ? lane - (2 * d + 1) : lane;

    double acc[NL];
#pragma unroll
    for (int l = 0; l < NL; ++l) acc[l] = 0.0;

    int m_begin, m_end, r_begin, r_end;
    lsq_chunk_rows(a, chunk, m_begin, m_end, r_begin, r_end);
    if (a.masked) {
        for (int r = m_begin + warp; r < m_end; r += LSQ_WARPS)
            for (int l = 0; l < nl; ++l) {
                float* m = a.masked + ((size_t)(b * a.L + l0 + l) * a.H + r) * a.W;
                for (int c4 = lane; c4 < (a.W >> 2); c4 += 32)
                    st_stream_f4(reinterpret_cast<float4*>(m) + c4, make_float4(0.f, 0.f, 0.f, 0.f));
            }
    }
    // Hot loop.  No run-time lane-count test around the loads: a partial lane group re-reads its last lane (map_base is
    // clamped) and simply drops the duplicates afterwards -- with `if (l < nl)` around each load the compiler kept the
    // loads of a row in separate basic blocks and every one of them was waited for on its own (ncu r01: 65 % of the
    // stall samples on the first use of each float4, 30 % of the DRAM roof).  RU rows per warp iteration (2 for bf16
    // maps, whose rows are only two 16-byte loads per lane) put NL * RU * UNR loads in flight per thread.
    constexpr int RU = BF16 ? 2 : 1;
    size_t map_base[NL];
#pragma unroll
    for (int l = 0; l < NL; ++l) map_base[l] = ((size_t)(b * a.L + min(l0 + l, a.L - 1)) * a.H) * a.W;
    for (int r = r_begin + warp * RU; r < r_end; r += LSQ_WARPS * RU) {
        float A[RU][NL], Bx[RU][NL];
        size_t rowoff[RU];
        bool rvalid[RU];
#pragma unroll
        for (int u = 0; u < RU; ++u) {
            rvalid[u] = r + u < r_end;
            rowoff[u] = (size_t)(rvalid[u] ? r + u : r) * a.W;
#pragma unroll
            for (int l = 0; l < NL; ++l) A[u][l] = Bx[u][l] = 0.f;
        }
#pragma unroll UNR
        for (int cv = lane; cv < WV; cv += 32) {
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                float x[V];
                load_xv<V>(a.xtab + rowoff[u], cv, x);
#pragma unroll
                for (int l = 0; l < NL; ++l) {
                    const size_t off = map_base[l] + rowoff[u] + (size_t)V * cv;
                    float o[V];
                    load_mapv<BF16>(a.o, off, o);
                    float sa = 0.f, sb = 0.f;
                    // (the backward kernel writes its math with the f2_* pair helpers of lf_common.cuh; on sm_90a they are
                    // two scalar ops each, rounded identically)
#pragma unroll
                    for (int e = 0; e < V; ++e) {
                        o[e] = act_fn<ACT_T>(o[e], a.act);
                        const float w = o[e] * o[e];
                        sa += w;
                        sb = fmaf(w, x[e], sb);
                    }
                    if (a.masked && l < nl && rvalid[u]) {
#pragma unroll
                        for (int q = 0; q < V / 4; ++q)
                            st_stream_f4(reinterpret_cast<float4*>(a.masked + off) + q,
                                         make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]));
                    }
                    A[u][l] += sa;
                    Bx[u][l] += sb;
                }
            }
        }
#pragma unroll
        for (int u = 0; u < RU; ++u) {
            if (!rvalid[u]) continue;                 // warp-uniform
            const double y = (double)__ldg(a.yrow + r + u);
            double pw = 1.0;
            for (int i = 0; i < ek && i < 2 * LF_MAX_ORDER; ++i) pw *= y;
            // The 2*NL row sums (A_l, B_l) are reduced over the warp TOGETHER, in fp32: NV/2 + NV/4 + .. shuffles instead of
            // 2*NL full fp64 butterflies (80 64-bit shuffles per row at NL = 4, the kernel's issue bound: a row is only 2-8 KB
            // of map data).  The per-thread partials are fp32 sums of 16-32 products already; five more fp32 additions do
            // not change the error class, and the sum over rows -- where the cancellation lives -- stays fp64.
            float v[NV];
#pragma unroll
            for (int l = 0; l < NLP; ++l) {
                v[l] = l < NL ? A[u][l] : 0.f;
                v[NLP + l] = l < NL ? Bx[u][l] : 0.f;
            }
            const float tot = warp_sum_packed<NV>(v, lane);
#pragma unroll
            for (int l = 0; l < NL; ++l) {
                const float s = __shfl_sync(0xffffffffu, tot, packed_holder<NV>((useB ? NLP : 0) + l));
                acc[l] = fma(pw, (double)s, acc[l]);
            }
        }
    }
    if (lane < LSQ_MAXNM) {
#pragma unroll
        for (int l = 0; l < NL; ++l) red[warp][l][lane] = (lane < NM && l < nl) ? acc[l] : 0.0;
    }
    lsq_chunk_tail(a, red, mom, chunk, b, lg, l0, nl);
}

// ---------------------------------------------------------------------------------
// Forward, general grid (y varies inside a row): per-pixel fp64 accumulation of all
// 3d+2 moments.  grid = (nchunks, B, L), one lane per CTA.  Slow path, any W.
// ---------------------------------------------------------------------------------
template <int ACT_T, bool BF16>
__global__ void __launch_bounds__(LSQ_THREADS) lsq_fwd_general_kernel(const LsqArgs a) {
    pdl_entry();
    __shared__ double red[LSQ_WARPS][LSQ_MAXL][LSQ_MAXNM];
    __shared__ double mom[LSQ_MAXL][LSQ_MAXNM];
    const int chunk = blockIdx.x, b = blockIdx.y, l = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int d = a.order;
    double S[2 * LF_MAX_ORDER + 1], T[LF_MAX_ORDER + 1];
#pragma unroll
    for (int k = 0; k <= 2 * LF_MAX_ORDER; ++k) S[k] = 0.0;
#pragma unroll
    for (int k = 0; k <= LF_MAX_ORDER; ++k) T[k] = 0.0;
    const size_t map_off = ((size_t)(b * a.L + l) * a.H) * a.W;
    int m_begin, m_end, r_begin, r_end;
    lsq_chunk_rows(a, chunk, m_begin, m_end, r_begin, r_end);
    if (a.masked)
        for (size_t p = (size_t)m_begin * a.W + threadIdx.x; p < (size_t)m_end * a.W; p += LSQ_THREADS) a.masked[map_off + p] = 0.f;
    const size_t p_begin = (size_t)r_begin * a.W, p_end = (size_t)r_end * a.W;
    for (size_t p = p_begin + threadIdx.x; p < p_end; p += LSQ_THREADS) {
        const float v = act_fn<ACT_T>(load_map1<BF16>(a.o, map_off + p), a.act);
        if (a.masked) a.masked[map_off + p] = v;
        const double w = (double)(v * v);
        const double y = (double)__ldg(a.ytab + p);
        const double wx = w * (double)__ldg(a.xtab + p);
        double py = 1.0;
#pragma unroll
        for (int k = 0; k <= 2 * LF_MAX_ORDER; ++k) {
            if (k <= 2 * d) S[k] = fma(w, py, S[k]);
            if (k <= d) T[k] = fma(wx, py, T[k]);
            py *= y;
        }
    }
#pragma unroll
    for (int k = 0; k <= 2 * LF_MAX_ORDER; ++k) {
        const double s = warp_sum(S[k]);
        if (lane == 0 && k <= 2 * d) red[warp][0][k] = s;
    }
#pragma unroll
    for (int k = 0; k <= LF_MAX_ORDER; ++k) {
        const double s = warp_sum(T[k]);
        if (lane == 0 && k <= d) red[warp][0][2 * d + 1 + k] = s;
    }
    lsq_chunk_tail(a, red, mom, chunk, b, l, l, 1);
}

// ---------------------------------------------------------------------------------
// Backward.  d_o = m * a'(o) * 2 a(o) * (x - phi^T beta) * (phi^T z),  z = Z^-1 g.
// ---------------------------------------------------------------------------------
__device__ __forceinline__ void lsq_bwd_load_coeffs(const LsqArgs& a, int b, int l0, int nl, double (*bs)[LF_MAX_ORDER + 1],
                                                    double (*zs)[LF_MAX_ORDER + 1]) {
    const int n = a.order + 1;
    const int t = threadIdx.x;
    if (t < LSQ_MAXL * (LF_MAX_ORDER + 1)) {
        const int l = t / (LF_MAX_ORDER + 1), i = t % (LF_MAX_ORDER + 1);
        if (l < nl && i < n) {
            const size_t bl = (size_t)(b * a.L + l0 + l);
            bs[l][i] = a.beta[bl * n + i];
            double s = 0.0;
            for (int j = 0; j < n; ++j) s += a.zinv[bl * n * n + i * n + j] * a.gbeta[bl * n + j];
            zs[l][i] = 2.0 * s;  // fold the factor 2
        }
    }
    __syncthreads();
}

template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, 4) lsq_bwd_rowsep_kernel(const LsqArgs a) {
    pdl_entry();
    __shared__ double bs[LSQ_MAXL][LF_MAX_ORDER + 1], zs[LSQ_MAXL][LF_MAX_ORDER + 1];
    const int chunk = blockIdx.x, b = blockIdx.y, lg = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int l0 = lg * NL;
    const int nl = min(NL, a.L - l0);
    constexpr int UNR = (NL <= 2) ? 4 : 2;
    const int d = a.order;
    constexpr int V = MapVec<BF16>::V;
    const int WV = a.W / V;
    lsq_bwd_load_coeffs(a, b, l0, nl, bs, zs);
    int m_begin, m_end, r_begin, r_end;
    lsq_chunk_rows(a, chunk, m_begin, m_end, r_begin, r_end);
    for (int r = m_begin + warp; r < m_end; r += LSQ_WARPS) {   // masked rows: zero gradient
        float z[V];
#pragma unroll
        for (int e = 0; e < V; ++e) z[e] = 0.f;
        for (int l = 0; l < nl; ++l) {
            const size_t off = ((size_t)(b * a.L + l0 + l) * a.H + r) * a.W;
            for (int cv = lane; cv < WV; cv += 32) store_mapv<BF16>(a.d_o, off + (size_t)V * cv, z);
        }
    }
    for (int r = r_begin + warp; r < r_end; r += LSQ_WARPS) {
        const size_t rowoff = (size_t)r * a.W;
        const double y = (double)__ldg(a.yrow + r);
        float qh[NL], ql[NL], sf[NL];
#pragma unroll
        for (int l = 0; l < NL; ++l) {
            qh[l] = ql[l] = sf[l] = 0.f;
            if (l < nl) {
                double q = bs[l][0], s = zs[l][0];
                for (int i = 1; i <= d; ++i) {
                    q = fma(q, y, bs[l][i]);
                    s = fma(s, y, zs[l][i]);
                }
                qh[l] = (float)q;
                ql[l] = (float)(q - (double)qh[l]);
                sf[l] = (float)s;
            }
        }
#pragma unroll UNR
        for (int cv = lane; cv < WV; cv += 32) {
            float x[V];
            load_xv<V>(a.xtab + rowoff, cv, x);
#pragma unroll
            for (int l = 0; l < NL; ++l) {
                // unconditional load from a clamped lane (see the forward kernel); only the store is predicated
                const size_t off = ((size_t)(b * a.L + min(l0 + l, a.L - 1)) * a.H) * a.W + rowoff + (size_t)V * cv;
                float o[V], g[V];
                load_mapv<BF16>(a.o, off, o);
                if constexpr (ACT_T == LF_ACT_SQUARE) {
                    // two pixels per instruction (see the forward kernel): g = o^3 * (((x - q_hi) - q_lo) * (2 s))
                    const f32x2_t nqh = f2_pack(-qh[l], -qh[l]), nql = f2_pack(-ql[l], -ql[l]), s2 = f2_pack(2.f * sf[l], 2.f * sf[l]);
#pragma unroll
                    for (int e = 0; e < V; e += 2) {
                        const f32x2_t o2 = f2_pack(o[e], o[e + 1]);
                        const f32x2_t o3 = f2_mul(f2_mul(o2, o2), o2);
                        const f32x2_t t = f2_mul(f2_add(f2_add(f2_pack(x[e], x[e + 1]), nqh), nql), s2);
                        f2_unpack(f2_mul(o3, t), g[e], g[e + 1]);
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < V; ++e)
                        g[e] = dact_times_act<ACT_T>(o[e], a.act) * (((x[e] - qh[l]) - ql[l]) * sf[l]);
                }
                if (l < nl) store_mapv<BF16>(a.d_o, off, g);
            }
        }
    }
}

template <int ACT_T, bool BF16>
__global__ void __launch_bounds__(LSQ_THREADS) lsq_bwd_general_kernel(const LsqArgs a) {
    pdl_entry();
    __shared__ double bs[LSQ_MAXL][LF_MAX_ORDER + 1], zs[LSQ_MAXL][LF_MAX_ORDER + 1];
    const int chunk = blockIdx.x, b = blockIdx.y, l = blockIdx.z;
    const int d = a.order;
    lsq_bwd_load_coeffs(a, b, l, 1, bs, zs);
    const size_t map_off = ((size_t)(b * a.L + l) * a.H) * a.W;
    int m_begin, m_end, r_begin, r_end;
    lsq_chunk_rows(a, chunk, m_begin, m_end, r_begin, r_end);
    for (size_t p = (size_t)m_begin * a.W + threadIdx.x; p < (size_t)m_end * a.W; p += LSQ_THREADS)
        store_map1<BF16>(a.d_o, map_off + p, 0.f);
    const size_t p_begin = (size_t)r_begin * a.W, p_end = (size_t)r_end * a.W;
    for (size_t p = p_begin + threadIdx.x; p < p_end; p += LSQ_THREADS) {
        const float o = load_map1<BF16>(a.o, map_off + p);
        const double y = (double)__ldg(a.ytab + p);
        double q = bs[0][0], s = zs[0][0];
        for (int i = 1; i <= d; ++i) {
            q = fma(q, y, bs[0][i]);
            s = fma(s, y, zs[0][i]);
        }
        const float g = (float)((double)dact_times_act<ACT_T>(o, a.act) * ((double)__ldg(a.xtab + p) - q) * s);
        store_map1<BF16>(a.d_o, map_off + p, g);
    }
}

// Chunks per system (image x lane group).  Every chunk gets an equal share of the unmasked rows (and of the masked
// rows), so all CTAs carry the same work; the count is chosen so that the CTAs fill whole waves of the resident CTAs
// per SM (the tail wave of a 1.7-wave grid cost 15 % in round 1), at least one row per warp and chunk, and few enough
// chunks that the per-CTA tail (block reduction, fence, ticket) stays small.
static int pick_nchunks(int B, int groups, int H, int mask_rows, int ctas_per_sm) {
    const int sms = device_sms();
    const long long slots = (long long)sms * ctas_per_sm, units = (long long)B * groups;
    const int ha = H - mask_rows > 0 ? H - mask_rows : 1;
    const int n_max = ha / LSQ_WARPS > 1 ? ha / LSQ_WARPS : 1;          // >= 8 unmasked rows per chunk
    const int n_cap = (H + LSQ_WARPS - 1) / LSQ_WARPS;                  // what lf_lsq_workspace_bytes provides
    int best = 1;
    double best_score = -1.0;
    for (int n = 1; n <= n_max && n <= n_cap; ++n) {
        const long long ctas = units * n;
        const long long waves = (ctas + slots - 1) / slots;
        const double fill = (double)ctas / (double)(waves * slots);      // how full the waves are
        const double rows = (double)ha / n;
        const double tail = rows / (rows + 6.0);                         // fixed per-CTA cost ~ 6 rows' worth
        const double score = fill * tail;
        if (score > best_score + 1e-9) {
            best_score = score;
            best = n;
        }
    }
    return best;
}

static int validate(const LsqArgs& a, int o_dtype) {
    LF_REQUIRE(a.o && a.xtab && (a.ytab || a.yrow));
    LF_REQUIRE(a.B > 0 && a.L > 0 && a.H > 0 && a.W > 0);
    LF_REQUIRE(a.order >= 0 && a.order <= LF_MAX_ORDER);
    LF_REQUIRE(a.mask_rows >= 0 && a.mask_rows <= a.H);
    LF_REQUIRE(a.act >= LF_ACT_NONE && a.act <= LF_ACT_SOFTPLUS);
    LF_REQUIRE(o_dtype == LF_F32 || o_dtype == LF_BF16);
    LF_REQUIRE(a.B <= 65535 && a.L <= 65535);
    return LF_OK;
}

}  // namespace lf

using namespace lf;

// Workspace = [ticket region: LSQ_TICKET_BYTES, fixed so that tickets never alias partials of a call
// with another shape] [partials].  Tickets are left at zero by every launch.
constexpr size_t LSQ_TICKET_BYTES = 64 * 1024;

extern "C" size_t lf_lsq_workspace_bytes(int B, int L, int H, int W, int order) {
    (void)W;
    if (B <= 0 || L <= 0 || H <= 0 || order < 0 || order > LF_MAX_ORDER) return 0;
    if ((size_t)B * L * sizeof(int) > LSQ_TICKET_BYTES) return 0;
    // worst case: rows_per_cta = 8 -> nchunks = ceil(H/8)
    const size_t nchunks = (size_t)(H + LSQ_WARPS - 1) / LSQ_WARPS;
    return LSQ_TICKET_BYTES + (size_t)B * L * nchunks * (3 * order + 2) * sizeof(double);
}

#define LSQ_DISPATCH(KERNEL, grid, args)                                                   \
    do {                                                                                   \
        if (args.act == LF_ACT_SQUARE) {                                                   \
            if (o_dtype == LF_BF16)                                                        \
                lf_launch(KERNEL<LF_ACT_SQUARE, true>, grid, LSQ_THREADS, 0, stream, args);       \
            else                                                                           \
                lf_launch(KERNEL<LF_ACT_SQUARE, false>, grid, LSQ_THREADS, 0, stream, args);      \
        } else {                                                                           \
            if (o_dtype == LF_BF16)                                                        \
                lf_launch(KERNEL<LSQ_ACT_RUNTIME, true>, grid, LSQ_THREADS, 0, stream, args);     \
            else                                                                           \
                lf_launch(KERNEL<LSQ_ACT_RUNTIME, false>, grid, LSQ_THREADS, 0, stream, args);    \
        }                                                                                  \
    } while (0)

#define LSQ_DISPATCH_NL2(KERNEL, NL, grid, args)                                               \
    do {                                                                                       \
        if (args.act == LF_ACT_SQUARE) {                                                       \
            if (o_dtype == LF_BF16)                                                            \
                lf_launch(KERNEL<LF_ACT_SQUARE, true, NL>, grid, LSQ_THREADS, 0, stream, args);       \
            else                                                                               \
                lf_launch(KERNEL<LF_ACT_SQUARE, false, NL>, grid, LSQ_THREADS, 0, stream, args);      \
        } else {                                                                               \
            if (o_dtype == LF_BF16)                                                            \
                lf_launch(KERNEL<LSQ_ACT_RUNTIME, true, NL>, grid, LSQ_THREADS, 0, stream, args);     \
            else                                                                               \
                lf_launch(KERNEL<LSQ_ACT_RUNTIME, false, NL>, grid, LSQ_THREADS, 0, stream, args);    \
        }                                                                                      \
    } while (0)

#define LSQ_DISPATCH_NL(KERNEL, nlg, grid, args)                       \
    do {                                                               \
        switch (nlg) {                                                 \
            case 1: LSQ_DISPATCH_NL2(KERNEL, 1, grid, args); break;    \
            case 2: LSQ_DISPATCH_NL2(KERNEL, 2, grid, args); break;    \
            case 3: LSQ_DISPATCH_NL2(KERNEL, 3, grid, args); break;    \
            default: LSQ_DISPATCH_NL2(KERNEL, 4, grid, args); break;   \
        }                                                              \
    } while (0)

// lanes per CTA: balanced groups of at most LSQ_MAXL (L=6 -> 2 groups of 3, not 4+2)
static void lsq_lane_groups(int L, int* groups, int* nlg) {
    *groups = (L + LSQ_MAXL - 1) / LSQ_MAXL;
    *nlg = (L + *groups - 1) / *groups;
}

extern "C" int lf_lsq_fwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow, int B,
                          int L, int H, int W, int order, int mask_rows, int act, double reg_ls, int solver,
                          double* beta, double* zinv, float* masked, int* status, void* workspace,
                          size_t workspace_bytes, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LsqArgs a{};
    a.o = o; a.xtab = xtab; a.ytab = ytab; a.yrow = yrow;
    a.B = B; a.L = L; a.H = H; a.W = W; a.order = order; a.mask_rows = mask_rows; a.act = act; a.solver = solver;
    a.reg_ls = reg_ls; a.beta = beta; a.zinv = zinv; a.masked = masked; a.status = status;
    int rc = validate(a, o_dtype);
    if (rc != LF_OK) return rc;
    LF_REQUIRE(beta && zinv && status && workspace);
    LF_REQUIRE(solver == LF_SOLVER_INVERSE || solver == LF_SOLVER_CHOLESKY);
    const size_t need = lf_lsq_workspace_bytes(B, L, H, W, order);
    if (need == 0) return LF_ERR_UNSUPPORTED;
    if (workspace_bytes < need) return LF_ERR_WORKSPACE_TOO_SMALL;
    const bool rowsep = (yrow != nullptr) && (W % (o_dtype == LF_BF16 ? 8 : 4) == 0);
    if (!rowsep && !ytab) return LF_ERR_INVALID_ARGUMENT;
    int groups = L, nlg = 1;
    if (rowsep) lsq_lane_groups(L, &groups, &nlg);
    a.nchunks = pick_nchunks(B, groups, H, mask_rows, rowsep ? LSQ_FWD_CTAS_PER_SM : 4);
    a.rows_per_cta = 0;
    a.tickets = reinterpret_cast<int*>(workspace);
    a.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + LSQ_TICKET_BYTES);
    dim3 grid(a.nchunks, B, groups);
    if (rowsep)
        LSQ_DISPATCH_NL(lsq_fwd_rowsep_kernel, nlg, grid, a);
    else
        LSQ_DISPATCH(lsq_fwd_general_kernel, grid, a);
    return check_launch();
}

extern "C" int lf_lsq_bwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow, int B,
                          int L, int H, int W, int order, int mask_rows, int act, const double* beta,
                          const double* zinv, const double* gbeta, void* d_o, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LsqArgs a{};
    a.o = o; a.xtab = xtab; a.ytab = ytab; a.yrow = yrow;
    a.B = B; a.L = L; a.H = H; a.W = W; a.order = order; a.mask_rows = mask_rows; a.act = act;
    a.beta = const_cast<double*>(beta); a.zinv = const_cast<double*>(zinv); a.gbeta = gbeta; a.d_o = d_o;
    int rc = validate(a, o_dtype);
    if (rc != LF_OK) return rc;
    LF_REQUIRE(beta && zinv && gbeta && d_o);
    const bool rowsep = (yrow != nullptr) && (W % (o_dtype == LF_BF16 ? 8 : 4) == 0);
    if (!rowsep && !ytab) return LF_ERR_INVALID_ARGUMENT;
    int groups = L, nlg = 1;
    if (rowsep) lsq_lane_groups(L, &groups, &nlg);
    a.nchunks = pick_nchunks(B, groups, H, mask_rows, LSQ_BWD_CTAS_PER_SM);
    a.rows_per_cta = 0;
    dim3 grid(a.nchunks, B, groups);
    if (rowsep)
        LSQ_DISPATCH_NL(lsq_bwd_rowsep_kernel, nlg, grid, a);
    else
        LSQ_DISPATCH(lsq_bwd_general_kernel, grid, a);
    return check_launch();
}
