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
//  * Per-pixel keep map (the *_keep entry points, KEEP template flag): an optional uint8 [H, W] map shared by every
//    image and lane zeroes act(o) where it is 0, before the square -- the reference's trapezium mask.  Its 16-byte
//    rows are read with the x table's (L2-resident); the KEEP = false instantiations compile to the same code as
//    before the flag existed.
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

// keep bytes of V consecutive pixels (4 or 8 bytes, aligned with the map vector); byte e is pixel e
template <int V>
__device__ __forceinline__ void load_keepv(const uint8_t* krow, int cv, uint32_t (&k)[V / 4]) {
    if constexpr (V == 8) {
        const uint2 t = __ldg(reinterpret_cast<const uint2*>(krow) + cv);
        k[0] = t.x;
        k[1] = t.y;
    } else {
        k[0] = __ldg(reinterpret_cast<const unsigned int*>(krow) + cv);
    }
}
template <int V>
__device__ __forceinline__ bool kept(const uint32_t (&k)[V / 4], int e) {
    return ((k[e >> 2] >> (8 * (e & 3))) & 0xffu) != 0u;
}
// v, or +0.0 where the pixel is masked: a bitwise AND in inline PTX, so the compiler cannot fold the mask into the
// square and the row sums after it (whatever v holds at a masked pixel, NaN and Inf included, the result is +0.0).
template <int V>
__device__ __forceinline__ float keep_or_zero(const uint32_t (&k)[V / 4], int e, float v) {
    uint32_t r;
    asm("and.b32 %0, %1, %2;" : "=r"(r) : "r"(__float_as_uint(v)), "r"(kept<V>(k, e) ? 0xffffffffu : 0u));
    return __uint_as_float(r);
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
// ROWSUMS: also accumulate C_r = sum_c w c and store (A_r, B_r, C_r) of every unmasked row in rowsums [B][L][H][3] --
// what the gradient with respect to a learned homography's tables needs (lsq_grid_grad_kernel).  `rowsums` is a kernel
// parameter of its own, not an LsqArgs field, so the other kernels' argument block stays as it was.
// KEEP: act(o) is zeroed where keep [H][W] (uint8, a kernel parameter of its own like rowsums) is 0, so w, the
// moments, the row sums and `masked` see a zero there.
template <int ACT_T, bool BF16, int NL, bool ROWSUMS, bool KEEP>
__device__ __forceinline__ void lsq_fwd_rowsep_body(const LsqArgs& a, float* rowsums, const uint8_t* keep) {
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
        float A[RU][NL], Bx[RU][NL], Cx[RU][NL];
        size_t rowoff[RU];
        bool rvalid[RU];
#pragma unroll
        for (int u = 0; u < RU; ++u) {
            rvalid[u] = r + u < r_end;
            rowoff[u] = (size_t)(rvalid[u] ? r + u : r) * a.W;
#pragma unroll
            for (int l = 0; l < NL; ++l) A[u][l] = Bx[u][l] = Cx[u][l] = 0.f;
        }
#pragma unroll UNR
        for (int cv = lane; cv < WV; cv += 32) {
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                float x[V];
                load_xv<V>(a.xtab + rowoff[u], cv, x);
                uint32_t kw[V / 4];
                if constexpr (KEEP) load_keepv<V>(keep + rowoff[u], cv, kw);
#pragma unroll
                for (int l = 0; l < NL; ++l) {
                    const size_t off = map_base[l] + rowoff[u] + (size_t)V * cv;
                    float o[V];
                    load_mapv<BF16>(a.o, off, o);
                    float sa = 0.f, sb = 0.f, sc = 0.f;
                    // (the backward kernel writes its math with the f2_* pair helpers of lf_common.cuh; on sm_90a they are
                    // two scalar ops each, rounded identically)
#pragma unroll
                    for (int e = 0; e < V; ++e) {
                        o[e] = act_fn<ACT_T>(o[e], a.act);
                        if constexpr (KEEP) o[e] = keep_or_zero<V>(kw, e, o[e]);
                        const float w = o[e] * o[e];
                        sa += w;
                        sb = fmaf(w, x[e], sb);
                        if constexpr (ROWSUMS) sc = fmaf(w, (float)(V * cv + e), sc);
                    }
                    if (a.masked && l < nl && rvalid[u]) {
#pragma unroll
                        for (int q = 0; q < V / 4; ++q)
                            st_stream_f4(reinterpret_cast<float4*>(a.masked + off) + q,
                                         make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]));
                    }
                    A[u][l] += sa;
                    Bx[u][l] += sb;
                    if constexpr (ROWSUMS) Cx[u][l] += sc;
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
            if constexpr (ROWSUMS) {
#pragma unroll
                for (int l = 0; l < NL; ++l) {
                    const float sa = __shfl_sync(0xffffffffu, tot, packed_holder<NV>(l));
                    const float sb = __shfl_sync(0xffffffffu, tot, packed_holder<NV>(NLP + l));
                    const float sc = warp_sum(Cx[u][l]);
                    if (lane == 0 && l < nl) {
                        float* rs = rowsums + ((size_t)(b * a.L + l0 + l) * a.H + r + u) * 3;
                        rs[0] = sa;
                        rs[1] = sb;
                        rs[2] = sc;
                    }
                }
            }
        }
    }
    if (lane < LSQ_MAXNM) {
#pragma unroll
        for (int l = 0; l < NL; ++l) red[warp][l][lane] = (lane < NM && l < nl) ? acc[l] : 0.0;
    }
    lsq_chunk_tail(a, red, mom, chunk, b, lg, l0, nl);
}

template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_FWD_CTAS_PER_SM) lsq_fwd_rowsep_kernel(const LsqArgs a) {
    lsq_fwd_rowsep_body<ACT_T, BF16, NL, false, false>(a, nullptr, nullptr);
}

template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_FWD_CTAS_PER_SM) lsq_fwd_rowsums_kernel(const LsqArgs a, float* rowsums) {
    lsq_fwd_rowsep_body<ACT_T, BF16, NL, true, false>(a, rowsums, nullptr);
}

template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_FWD_CTAS_PER_SM) lsq_fwd_rowsep_keep_kernel(const LsqArgs a,
                                                                                               const uint8_t* keep) {
    lsq_fwd_rowsep_body<ACT_T, BF16, NL, false, true>(a, nullptr, keep);
}

template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_FWD_CTAS_PER_SM) lsq_fwd_rowsums_keep_kernel(const LsqArgs a,
                                                                                                float* rowsums,
                                                                                                const uint8_t* keep) {
    lsq_fwd_rowsep_body<ACT_T, BF16, NL, true, true>(a, rowsums, keep);
}

// Per-image tables (a predicted homography, lf_lsq_fwd_per_image / lf_lsq_bwd_per_image): a.xtab is [B][H][W] and
// a.yrow [B][H]; the CTAs of image b run the shared-table body on b's slice, so the arithmetic is the shared-table
// kernel's and the existing kernels are untouched.
__device__ __forceinline__ LsqArgs lsq_image_args(const LsqArgs& a, int b) {
    LsqArgs ai = a;
    ai.xtab = a.xtab + (size_t)b * a.H * a.W;
    ai.yrow = a.yrow + (size_t)b * a.H;
    return ai;
}

// ROWSUMS / KEEP as above; rowsums and keep may be unused
template <int ACT_T, bool BF16, int NL, bool ROWSUMS, bool KEEP>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_FWD_CTAS_PER_SM) lsq_fwd_rowsep_pi_kernel(const LsqArgs a,
                                                                                             float* rowsums,
                                                                                             const uint8_t* keep) {
    lsq_fwd_rowsep_body<ACT_T, BF16, NL, ROWSUMS, KEEP>(lsq_image_args(a, blockIdx.y), rowsums, keep);
}

// ---------------------------------------------------------------------------------
// Gradient of the loss with respect to the row-separable tables x_{r,c} = alpha_r c + gamma_r, y_r = const - y'_r,
// from the forward's row sums (DESIGN.md "Learned homography"), summed over images and lanes in a fixed order:
//   dL/dgamma_r = (phi_r.z) A_r ,  dL/dalpha_r = (phi_r.z) C_r ,
//   dL/dy_r     = (phi'_r.z)(B_r - (phi_r.beta) A_r) - (phi_r.z)(phi'_r.beta) A_r ,   dL/dy'_r = -dL/dy_r
// with phi_r = [y^d .. y 1], z = Z^-1 g.  One thread per row; masked rows get 0.  g_rowp [H][3] = (alpha, gamma, y').
// ---------------------------------------------------------------------------------
constexpr int LSQ_GG_THREADS = 128;

// row r of g_rowp, summed over the systems bl0 .. bl0 + nbl - 1 in order
__device__ __forceinline__ void lsq_grid_grad_row(const float* __restrict__ rowsums, const float* __restrict__ yrow,
                                                  const double* __restrict__ beta, const double* __restrict__ zinv,
                                                  const double* __restrict__ gbeta, int bl0, int nbl, int H, int order,
                                                  int mask_rows, int r, double* __restrict__ g_rowp) {
    const int n = order + 1;
    double ga = 0.0, gg = 0.0, gy = 0.0;
    if (r >= mask_rows) {
        const double y = (double)yrow[r];
        double phi[LF_MAX_ORDER + 1], dphi[LF_MAX_ORDER + 1];   // index i: power d - i
        double pw = 1.0, pwm = 0.0;                                 // y^k, k y^(k-1)
        for (int i = order; i >= 0; --i) {
            phi[i] = pw;
            dphi[i] = pwm;
            pwm = pwm * y + pw;
            pw *= y;
        }
        for (int bl = bl0; bl < bl0 + nbl; ++bl) {
            const double* bt = beta + (size_t)bl * n;
            const double* zi = zinv + (size_t)bl * n * n;
            const double* g = gbeta + (size_t)bl * n;
            double pz = 0.0, dz = 0.0, pb = 0.0, db = 0.0;
            for (int i = 0; i < n; ++i) {
                double z = 0.0;
                for (int j = 0; j < n; ++j) z += zi[i * n + j] * g[j];
                pz += phi[i] * z;
                dz += dphi[i] * z;
                pb += phi[i] * bt[i];
                db += dphi[i] * bt[i];
            }
            const float* rs = rowsums + ((size_t)bl * H + r) * 3;
            const double A = rs[0], Bs = rs[1], C = rs[2];
            gg += pz * A;
            ga += pz * C;
            gy += dz * (Bs - pb * A) - pz * db * A;
        }
    }
    g_rowp[(size_t)r * 3 + 0] = ga;
    g_rowp[(size_t)r * 3 + 1] = gg;
    g_rowp[(size_t)r * 3 + 2] = -gy;
}

__global__ void __launch_bounds__(LSQ_GG_THREADS) lsq_grid_grad_kernel(const float* __restrict__ rowsums,
                                                                        const float* __restrict__ yrow,
                                                                        const double* __restrict__ beta,
                                                                        const double* __restrict__ zinv,
                                                                        const double* __restrict__ gbeta, int B, int L,
                                                                        int H, int order, int mask_rows,
                                                                        double* __restrict__ g_rowp) {
    pdl_entry();
    const int r = blockIdx.x * LSQ_GG_THREADS + threadIdx.x;
    if (r >= H) return;
    lsq_grid_grad_row(rowsums, yrow, beta, zinv, gbeta, 0, B * L, H, order, mask_rows, r, g_rowp);
}

// per-image tables: grid (rows, B), image b's g_rowp [H][3] summed over its lanes only, from its yrow [H]
__global__ void __launch_bounds__(LSQ_GG_THREADS) lsq_grid_grad_pi_kernel(const float* __restrict__ rowsums,
                                                                           const float* __restrict__ yrow,
                                                                           const double* __restrict__ beta,
                                                                           const double* __restrict__ zinv,
                                                                           const double* __restrict__ gbeta, int L, int H,
                                                                           int order, int mask_rows,
                                                                           double* __restrict__ g_rowp) {
    pdl_entry();
    const int r = blockIdx.x * LSQ_GG_THREADS + threadIdx.x, b = blockIdx.y;
    if (r >= H) return;
    // image b's systems are bl = b L .. b L + L - 1; rowsums is indexed by bl, so only yrow and g_rowp move
    lsq_grid_grad_row(rowsums, yrow + (size_t)b * H, beta, zinv, gbeta, b * L, L, H, order, mask_rows, r,
                      g_rowp + (size_t)b * H * 3);
}

// ---------------------------------------------------------------------------------
// Forward, general grid (y varies inside a row): per-pixel fp64 accumulation of all
// 3d+2 moments.  grid = (nchunks, B, L), one lane per CTA.  Slow path, any W.
// ---------------------------------------------------------------------------------
template <int ACT_T, bool BF16, bool KEEP>
__device__ __forceinline__ void lsq_fwd_general_body(const LsqArgs& a, const uint8_t* keep) {
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
        float v = act_fn<ACT_T>(load_map1<BF16>(a.o, map_off + p), a.act);
        if constexpr (KEEP) v = __ldg(keep + p) ? v : 0.f;
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

template <int ACT_T, bool BF16>
__global__ void __launch_bounds__(LSQ_THREADS) lsq_fwd_general_kernel(const LsqArgs a) {
    lsq_fwd_general_body<ACT_T, BF16, false>(a, nullptr);
}

template <int ACT_T, bool BF16>
__global__ void __launch_bounds__(LSQ_THREADS) lsq_fwd_general_keep_kernel(const LsqArgs a, const uint8_t* keep) {
    lsq_fwd_general_body<ACT_T, BF16, true>(a, keep);
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

template <int ACT_T, bool BF16, int NL, bool KEEP>
__device__ __forceinline__ void lsq_bwd_rowsep_body(const LsqArgs& a, const uint8_t* keep) {
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
            uint32_t kw[V / 4];
            if constexpr (KEEP) load_keepv<V>(keep + rowoff, cv, kw);
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
                if constexpr (KEEP) {
#pragma unroll
                    for (int e = 0; e < V; ++e) g[e] = kept<V>(kw, e) ? g[e] : 0.f;
                }
                if (l < nl) store_mapv<BF16>(a.d_o, off, g);
            }
        }
    }
}

template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_BWD_CTAS_PER_SM) lsq_bwd_rowsep_kernel(const LsqArgs a) {
    lsq_bwd_rowsep_body<ACT_T, BF16, NL, false>(a, nullptr);
}

template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_BWD_CTAS_PER_SM) lsq_bwd_rowsep_keep_kernel(const LsqArgs a,
                                                                                               const uint8_t* keep) {
    lsq_bwd_rowsep_body<ACT_T, BF16, NL, true>(a, keep);
}

// per-image tables (lf_lsq_bwd_per_image)
template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_BWD_CTAS_PER_SM) lsq_bwd_rowsep_pi_kernel(const LsqArgs a,
                                                                                             const uint8_t* keep) {
    lsq_bwd_rowsep_body<ACT_T, BF16, NL, false>(lsq_image_args(a, blockIdx.y), keep);
}

template <int ACT_T, bool BF16, int NL>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_BWD_CTAS_PER_SM) lsq_bwd_rowsep_pi_keep_kernel(const LsqArgs a,
                                                                                                  const uint8_t* keep) {
    lsq_bwd_rowsep_body<ACT_T, BF16, NL, true>(lsq_image_args(a, blockIdx.y), keep);
}

template <int ACT_T, bool BF16, bool KEEP>
__device__ __forceinline__ void lsq_bwd_general_body(const LsqArgs& a, const uint8_t* keep) {
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
        float g = (float)((double)dact_times_act<ACT_T>(o, a.act) * ((double)__ldg(a.xtab + p) - q) * s);
        if constexpr (KEEP) g = __ldg(keep + p) ? g : 0.f;
        store_map1<BF16>(a.d_o, map_off + p, g);
    }
}

template <int ACT_T, bool BF16>
__global__ void __launch_bounds__(LSQ_THREADS) lsq_bwd_general_kernel(const LsqArgs a) {
    lsq_bwd_general_body<ACT_T, BF16, false>(a, nullptr);
}

template <int ACT_T, bool BF16>
__global__ void __launch_bounds__(LSQ_THREADS) lsq_bwd_general_keep_kernel(const LsqArgs a, const uint8_t* keep) {
    lsq_bwd_general_body<ACT_T, BF16, true>(a, keep);
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

// ---------------------------------------------------------------------------------
// Prefix fits (the *_lanes entry points, a lane curriculum): lanes [0, L) of maps with Lmap >= L channels, o and d_o
// [B][Lmap][H][W].  The bodies index a map as (b * L + l) * H * W; moving o and d_o of image b by b * (Lmap - L) maps
// turns that into (b * Lmap + l) * H * W, so the fitted lanes run the plain kernels' bodies unchanged and every plain
// kernel keeps its code.  masked, beta, zinv, rowsums and the workspace stay compact, sized by L.  per_image: the
// per-image tables of lsq_image_args as well.
// ---------------------------------------------------------------------------------
template <bool BF16>
__device__ __forceinline__ LsqArgs lsq_lanes_args(const LsqArgs& a, int b, int Lmap, int per_image) {
    LsqArgs ai = per_image ? lsq_image_args(a, b) : a;
    const size_t shift = (size_t)b * (Lmap - a.L) * a.H * a.W * (BF16 ? 2 : 4);     // bytes
    ai.o = reinterpret_cast<const char*>(a.o) + shift;
    if (a.d_o) ai.d_o = reinterpret_cast<char*>(a.d_o) + shift;
    return ai;
}

template <int ACT_T, bool BF16, int NL, bool ROWSUMS, bool KEEP>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_FWD_CTAS_PER_SM) lsq_fwd_rowsep_lanes_kernel(const LsqArgs a,
                                                                                                float* rowsums,
                                                                                                const uint8_t* keep,
                                                                                                int Lmap, int per_image) {
    lsq_fwd_rowsep_body<ACT_T, BF16, NL, ROWSUMS, KEEP>(lsq_lanes_args<BF16>(a, blockIdx.y, Lmap, per_image), rowsums,
                                                        keep);
}

template <int ACT_T, bool BF16, bool KEEP>
__global__ void __launch_bounds__(LSQ_THREADS) lsq_fwd_general_lanes_kernel(const LsqArgs a, const uint8_t* keep,
                                                                             int Lmap) {
    lsq_fwd_general_body<ACT_T, BF16, KEEP>(lsq_lanes_args<BF16>(a, blockIdx.y, Lmap, 0), keep);
}

// d_o of the unfitted lanes [L, Lmap) of image b is +0.0: the CTAs of lane group 0 store zeros over their chunk's rows,
// after the fitted lanes' pass (so after the body's PDL wait), in the same launch.
template <bool BF16>
__device__ __forceinline__ void lsq_bwd_zero_unfitted(const LsqArgs& a, int b, int chunk, int Lmap) {
    int m_begin, m_end, r_begin, r_end;
    lsq_chunk_rows(a, chunk, m_begin, m_end, r_begin, r_end);
    const int nm = m_end - m_begin, nrows = nm + (r_end - r_begin);
    for (int l = a.L; l < Lmap; ++l)
        for (int i = 0; i < nrows; ++i) {
            const int r = i < nm ? m_begin + i : r_begin + (i - nm);
            const size_t row = ((size_t)(b * Lmap + l) * a.H + r) * a.W;
            for (int c = threadIdx.x; c < a.W; c += LSQ_THREADS) store_map1<BF16>(a.d_o, row + c, 0.f);
        }
}

template <int ACT_T, bool BF16, int NL, bool KEEP>
__global__ void __launch_bounds__(LSQ_THREADS, LSQ_BWD_CTAS_PER_SM) lsq_bwd_rowsep_lanes_kernel(const LsqArgs a,
                                                                                                const uint8_t* keep,
                                                                                                int Lmap, int per_image) {
    lsq_bwd_rowsep_body<ACT_T, BF16, NL, KEEP>(lsq_lanes_args<BF16>(a, blockIdx.y, Lmap, per_image), keep);
    if (blockIdx.z == 0) lsq_bwd_zero_unfitted<BF16>(a, blockIdx.y, blockIdx.x, Lmap);
}

template <int ACT_T, bool BF16, bool KEEP>
__global__ void __launch_bounds__(LSQ_THREADS) lsq_bwd_general_lanes_kernel(const LsqArgs a, const uint8_t* keep,
                                                                             int Lmap) {
    lsq_bwd_general_body<ACT_T, BF16, KEEP>(lsq_lanes_args<BF16>(a, blockIdx.y, Lmap, 0), keep);
    if (blockIdx.z == 0) lsq_bwd_zero_unfitted<BF16>(a, blockIdx.y, blockIdx.x, Lmap);
}

}  // namespace lf

using namespace lf;

// Workspace = [ticket region: LSQ_TICKET_BYTES, fixed so that tickets never alias partials of a call
// with another shape] [partials].  Tickets are left at zero by every launch.
constexpr size_t LSQ_TICKET_BYTES = 64 * 1024;

// lanes per CTA: balanced groups of at most LSQ_MAXL (L=6 -> 2 groups of 3, not 4+2)
static void lsq_lane_groups(int L, int* groups, int* nlg) {
    *groups = (L + LSQ_MAXL - 1) / LSQ_MAXL;
    *nlg = (L + *groups - 1) / *groups;
}

// What one lf_lsq_fwd (bwd = 0) or lf_lsq_bwd (bwd = 1) call launches: the kernel, the activation template, the lanes
// per CTA and the chunks per system.  Both entry points and lf_lsq_plan take their decisions here, so the query cannot
// drift from the launch.
struct LsqPlan {
    int rowsep, act_t, nl, groups, nchunks, ctas_per_sm, align;
};

static int lsq_plan(int bwd, int o_dtype, int has_yrow, int has_ytab, int B, int L, int H, int W, int order, int mask_rows,
                    int act, LsqPlan* p) {
    LF_REQUIRE(B > 0 && L > 0 && H > 0 && W > 0);
    LF_REQUIRE(order >= 0 && order <= LF_MAX_ORDER);
    LF_REQUIRE(mask_rows >= 0 && mask_rows <= H);
    LF_REQUIRE(act >= LF_ACT_NONE && act <= LF_ACT_SOFTPLUS);
    LF_REQUIRE(o_dtype == LF_F32 || o_dtype == LF_BF16);
    LF_REQUIRE(B <= 65535 && L <= 65535);
    if (!bwd && lf_lsq_workspace_bytes(B, L, H, W, order) == 0) return LF_ERR_UNSUPPORTED;   // ticket region full
    // the row-separable kernels move 16 bytes per load and store: 4 fp32 or 8 bf16 map elements
    p->rowsep = has_yrow && W % (o_dtype == LF_BF16 ? 8 : 4) == 0;
    if (!p->rowsep && !has_ytab) return LF_ERR_INVALID_ARGUMENT;
    p->act_t = act == LF_ACT_SQUARE ? LF_ACT_SQUARE : LSQ_ACT_RUNTIME;
    p->groups = L;
    p->nl = 1;
    if (p->rowsep) lsq_lane_groups(L, &p->groups, &p->nl);
    p->ctas_per_sm = bwd ? LSQ_BWD_CTAS_PER_SM : (p->rowsep ? LSQ_FWD_CTAS_PER_SM : 4);
    p->nchunks = pick_nchunks(B, p->groups, H, mask_rows, p->ctas_per_sm);
    p->align = p->rowsep ? 16 : 0;
    return LF_OK;
}

static bool aligned16(const void* ptr) { return ptr == nullptr || (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

extern "C" int lf_lsq_plan(int bwd, int o_dtype, int has_yrow, int has_ytab, int B, int L, int H, int W, int order,
                           int mask_rows, int act, int* info) {
    LF_REQUIRE(info && (bwd == 0 || bwd == 1));
    LsqPlan p{};
    const int rc = lsq_plan(bwd, o_dtype, has_yrow != 0, has_ytab != 0, B, L, H, W, order, mask_rows, act, &p);
    if (rc != LF_OK) return rc;
    const int v[LF_LSQ_PLAN_INFO] = {p.rowsep, p.act_t, p.nl, p.groups, p.nchunks, p.ctas_per_sm, p.align};
    for (int i = 0; i < LF_LSQ_PLAN_INFO; ++i) info[i] = v[i];
    return LF_OK;
}

extern "C" size_t lf_lsq_workspace_bytes(int B, int L, int H, int W, int order) {
    (void)W;
    if (B <= 0 || L <= 0 || H <= 0 || order < 0 || order > LF_MAX_ORDER) return 0;
    if ((size_t)B * L * sizeof(int) > LSQ_TICKET_BYTES) return 0;
    // worst case: 8 rows per chunk -> nchunks = ceil(H/8)
    const size_t nchunks = (size_t)(H + LSQ_WARPS - 1) / LSQ_WARPS;
    return LSQ_TICKET_BYTES + (size_t)B * L * nchunks * (3 * order + 2) * sizeof(double);
}

// Launch KERNEL<activation template, bf16 map[, NL]> with the kernel arguments that follow `grid` (LsqArgs `a` first).
#define LSQ_DISPATCH(KERNEL, grid, ...)                                                            \
    do {                                                                                           \
        if (a.act == LF_ACT_SQUARE) {                                                              \
            if (o_dtype == LF_BF16)                                                                \
                lf_launch(KERNEL<LF_ACT_SQUARE, true>, grid, LSQ_THREADS, 0, stream, __VA_ARGS__);    \
            else                                                                                   \
                lf_launch(KERNEL<LF_ACT_SQUARE, false>, grid, LSQ_THREADS, 0, stream, __VA_ARGS__);   \
        } else {                                                                                   \
            if (o_dtype == LF_BF16)                                                                \
                lf_launch(KERNEL<LSQ_ACT_RUNTIME, true>, grid, LSQ_THREADS, 0, stream, __VA_ARGS__);  \
            else                                                                                   \
                lf_launch(KERNEL<LSQ_ACT_RUNTIME, false>, grid, LSQ_THREADS, 0, stream, __VA_ARGS__); \
        }                                                                                          \
    } while (0)

#define LSQ_DISPATCH_NL2(KERNEL, NL, grid, ...)                                                        \
    do {                                                                                               \
        if (a.act == LF_ACT_SQUARE) {                                                                  \
            if (o_dtype == LF_BF16)                                                                    \
                lf_launch(KERNEL<LF_ACT_SQUARE, true, NL>, grid, LSQ_THREADS, 0, stream, __VA_ARGS__);    \
            else                                                                                       \
                lf_launch(KERNEL<LF_ACT_SQUARE, false, NL>, grid, LSQ_THREADS, 0, stream, __VA_ARGS__);   \
        } else {                                                                                       \
            if (o_dtype == LF_BF16)                                                                    \
                lf_launch(KERNEL<LSQ_ACT_RUNTIME, true, NL>, grid, LSQ_THREADS, 0, stream, __VA_ARGS__);  \
            else                                                                                       \
                lf_launch(KERNEL<LSQ_ACT_RUNTIME, false, NL>, grid, LSQ_THREADS, 0, stream, __VA_ARGS__); \
        }                                                                                              \
    } while (0)

#define LSQ_DISPATCH_NL(KERNEL, nlg, grid, ...)                               \
    do {                                                                      \
        switch (nlg) {                                                        \
            case 1: LSQ_DISPATCH_NL2(KERNEL, 1, grid, __VA_ARGS__); break;    \
            case 2: LSQ_DISPATCH_NL2(KERNEL, 2, grid, __VA_ARGS__); break;    \
            case 3: LSQ_DISPATCH_NL2(KERNEL, 3, grid, __VA_ARGS__); break;    \
            default: LSQ_DISPATCH_NL2(KERNEL, 4, grid, __VA_ARGS__); break;   \
        }                                                                     \
    } while (0)

// The *_lanes kernels, used when Lmap > L (a prefix fit): rowsums / keep NULL select the instantiation as for the
// per-image kernels, per_image the per-image tables.
template <int ACT_T, bool BF16, int NL>
static void launch_lanes_nl(int bwd, dim3 grid, cudaStream_t stream, const LsqArgs& a, float* rowsums, const uint8_t* keep,
                            int Lmap, int pi) {
    if (bwd) {
        if (keep)
            lf_launch(lsq_bwd_rowsep_lanes_kernel<ACT_T, BF16, NL, true>, grid, LSQ_THREADS, 0, stream, a, keep, Lmap, pi);
        else
            lf_launch(lsq_bwd_rowsep_lanes_kernel<ACT_T, BF16, NL, false>, grid, LSQ_THREADS, 0, stream, a, keep, Lmap, pi);
    } else if (rowsums) {
        if (keep)
            lf_launch(lsq_fwd_rowsep_lanes_kernel<ACT_T, BF16, NL, true, true>, grid, LSQ_THREADS, 0, stream, a, rowsums,
                      keep, Lmap, pi);
        else
            lf_launch(lsq_fwd_rowsep_lanes_kernel<ACT_T, BF16, NL, true, false>, grid, LSQ_THREADS, 0, stream, a, rowsums,
                      keep, Lmap, pi);
    } else {
        if (keep)
            lf_launch(lsq_fwd_rowsep_lanes_kernel<ACT_T, BF16, NL, false, true>, grid, LSQ_THREADS, 0, stream, a, rowsums,
                      keep, Lmap, pi);
        else
            lf_launch(lsq_fwd_rowsep_lanes_kernel<ACT_T, BF16, NL, false, false>, grid, LSQ_THREADS, 0, stream, a, rowsums,
                      keep, Lmap, pi);
    }
}

template <int ACT_T, bool BF16>
static void launch_lanes_t(int rowsep, int nl, int bwd, dim3 grid, cudaStream_t stream, const LsqArgs& a, float* rowsums,
                           const uint8_t* keep, int Lmap, int pi) {
    if (!rowsep) {
        if (bwd)
            keep ? lf_launch(lsq_bwd_general_lanes_kernel<ACT_T, BF16, true>, grid, LSQ_THREADS, 0, stream, a, keep, Lmap)
                 : lf_launch(lsq_bwd_general_lanes_kernel<ACT_T, BF16, false>, grid, LSQ_THREADS, 0, stream, a, keep, Lmap);
        else
            keep ? lf_launch(lsq_fwd_general_lanes_kernel<ACT_T, BF16, true>, grid, LSQ_THREADS, 0, stream, a, keep, Lmap)
                 : lf_launch(lsq_fwd_general_lanes_kernel<ACT_T, BF16, false>, grid, LSQ_THREADS, 0, stream, a, keep, Lmap);
        return;
    }
    switch (nl) {
        case 1: launch_lanes_nl<ACT_T, BF16, 1>(bwd, grid, stream, a, rowsums, keep, Lmap, pi); break;
        case 2: launch_lanes_nl<ACT_T, BF16, 2>(bwd, grid, stream, a, rowsums, keep, Lmap, pi); break;
        case 3: launch_lanes_nl<ACT_T, BF16, 3>(bwd, grid, stream, a, rowsums, keep, Lmap, pi); break;
        default: launch_lanes_nl<ACT_T, BF16, 4>(bwd, grid, stream, a, rowsums, keep, Lmap, pi); break;
    }
}

static int launch_lanes(const LsqPlan& p, int bwd, int o_dtype, dim3 grid, cudaStream_t stream, const LsqArgs& a,
                        float* rowsums, const uint8_t* keep, int Lmap, int pi) {
    if (a.act == LF_ACT_SQUARE)
        o_dtype == LF_BF16 ? launch_lanes_t<LF_ACT_SQUARE, true>(p.rowsep, p.nl, bwd, grid, stream, a, rowsums, keep, Lmap, pi)
                           : launch_lanes_t<LF_ACT_SQUARE, false>(p.rowsep, p.nl, bwd, grid, stream, a, rowsums, keep, Lmap, pi);
    else
        o_dtype == LF_BF16 ? launch_lanes_t<LSQ_ACT_RUNTIME, true>(p.rowsep, p.nl, bwd, grid, stream, a, rowsums, keep, Lmap, pi)
                           : launch_lanes_t<LSQ_ACT_RUNTIME, false>(p.rowsep, p.nl, bwd, grid, stream, a, rowsums, keep, Lmap, pi);
    return check_launch();
}

// lf_lsq_fwd and lf_lsq_fwd_keep (keep = NULL: the KEEP = false kernels, exactly as before the keep map existed)
static int lsq_fwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
                   const uint8_t* keep, int B, int L, int Lmap, int H, int W, int order, int mask_rows, int act,
                   double reg_ls, int solver, double* beta, double* zinv, float* masked, int* status, void* workspace,
                   size_t workspace_bytes, cudaStream_t stream) {
    LF_REQUIRE(o && xtab && (ytab || yrow) && beta && zinv && status && workspace);
    LF_REQUIRE(Lmap >= L && Lmap <= 65535);
    LF_REQUIRE(solver == LF_SOLVER_INVERSE || solver == LF_SOLVER_CHOLESKY);
    LsqPlan p{};
    const int rc = lsq_plan(0, o_dtype, yrow != nullptr, ytab != nullptr, B, L, H, W, order, mask_rows, act, &p);
    if (rc != LF_OK) return rc;
    if (workspace_bytes < lf_lsq_workspace_bytes(B, L, H, W, order)) return LF_ERR_WORKSPACE_TOO_SMALL;
    if (p.rowsep) LF_REQUIRE(aligned16(o) && aligned16(xtab) && aligned16(masked) && aligned16(keep));
    LsqArgs a{};
    a.o = o; a.xtab = xtab; a.ytab = ytab; a.yrow = yrow;
    a.B = B; a.L = L; a.H = H; a.W = W; a.order = order; a.mask_rows = mask_rows; a.act = act; a.solver = solver;
    a.reg_ls = reg_ls; a.beta = beta; a.zinv = zinv; a.masked = masked; a.status = status;
    a.nchunks = p.nchunks;
    a.tickets = reinterpret_cast<int*>(workspace);
    a.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + LSQ_TICKET_BYTES);
    dim3 grid(a.nchunks, B, p.groups);
    if (Lmap > L) return launch_lanes(p, 0, o_dtype, grid, stream, a, nullptr, keep, Lmap, 0);
    if (p.rowsep) {
        if (keep)
            LSQ_DISPATCH_NL(lsq_fwd_rowsep_keep_kernel, p.nl, grid, a, keep);
        else
            LSQ_DISPATCH_NL(lsq_fwd_rowsep_kernel, p.nl, grid, a);
    } else {
        if (keep)
            LSQ_DISPATCH(lsq_fwd_general_keep_kernel, grid, a, keep);
        else
            LSQ_DISPATCH(lsq_fwd_general_kernel, grid, a);
    }
    return check_launch();
}

extern "C" int lf_lsq_fwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow, int B,
                          int L, int H, int W, int order, int mask_rows, int act, double reg_ls, int solver,
                          double* beta, double* zinv, float* masked, int* status, void* workspace,
                          size_t workspace_bytes, lf_stream_t stream_) {
    return lsq_fwd(o, o_dtype, xtab, ytab, yrow, nullptr, B, L, L, H, W, order, mask_rows, act, reg_ls, solver, beta, zinv,
                   masked, status, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_fwd_keep(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
                               const uint8_t* keep, int B, int L, int H, int W, int order, int mask_rows, int act,
                               double reg_ls, int solver, double* beta, double* zinv, float* masked, int* status,
                               void* workspace, size_t workspace_bytes, lf_stream_t stream_) {
    LF_REQUIRE(keep);
    return lsq_fwd(o, o_dtype, xtab, ytab, yrow, keep, B, L, L, H, W, order, mask_rows, act, reg_ls, solver, beta, zinv,
                   masked, status, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

template <int ACT_T, bool BF16, int NL>
static void launch_rowsums_nl(dim3 grid, cudaStream_t stream, const LsqArgs& a, float* rowsums, const uint8_t* keep) {
    if (keep)
        lf_launch(lsq_fwd_rowsums_keep_kernel<ACT_T, BF16, NL>, grid, LSQ_THREADS, 0, stream, a, rowsums, keep);
    else
        lf_launch(lsq_fwd_rowsums_kernel<ACT_T, BF16, NL>, grid, LSQ_THREADS, 0, stream, a, rowsums);
}

template <int ACT_T, bool BF16>
static void launch_rowsums(int nl, dim3 grid, cudaStream_t stream, const LsqArgs& a, float* rowsums, const uint8_t* keep) {
    switch (nl) {
        case 1: launch_rowsums_nl<ACT_T, BF16, 1>(grid, stream, a, rowsums, keep); break;
        case 2: launch_rowsums_nl<ACT_T, BF16, 2>(grid, stream, a, rowsums, keep); break;
        case 3: launch_rowsums_nl<ACT_T, BF16, 3>(grid, stream, a, rowsums, keep); break;
        default: launch_rowsums_nl<ACT_T, BF16, 4>(grid, stream, a, rowsums, keep); break;
    }
}

// lf_lsq_fwd on the row-separable kernel that also stores the row sums: same arguments and plan, yrow required,
// rowsums [B][L][H][3] float32 (rows >= mask_rows written).  keep as in lsq_fwd.
static int lsq_fwd_rowsums(const void* o, int o_dtype, const float* xtab, const float* yrow, const uint8_t* keep, int B,
                           int L, int Lmap, int H, int W, int order, int mask_rows, int act, double reg_ls, int solver,
                           double* beta, double* zinv, float* masked, int* status, float* rowsums, void* workspace,
                           size_t workspace_bytes, cudaStream_t stream) {
    LF_REQUIRE(o && xtab && yrow && beta && zinv && status && rowsums && workspace);
    LF_REQUIRE(Lmap >= L && Lmap <= 65535);
    LF_REQUIRE(solver == LF_SOLVER_INVERSE || solver == LF_SOLVER_CHOLESKY);
    LsqPlan p{};
    const int rc = lsq_plan(0, o_dtype, 1, 0, B, L, H, W, order, mask_rows, act, &p);
    if (rc != LF_OK) return rc;
    if (workspace_bytes < lf_lsq_workspace_bytes(B, L, H, W, order)) return LF_ERR_WORKSPACE_TOO_SMALL;
    LF_REQUIRE(aligned16(o) && aligned16(xtab) && aligned16(masked) && aligned16(keep));
    LsqArgs a{};
    a.o = o; a.xtab = xtab; a.yrow = yrow;
    a.B = B; a.L = L; a.H = H; a.W = W; a.order = order; a.mask_rows = mask_rows; a.act = act; a.solver = solver;
    a.reg_ls = reg_ls; a.beta = beta; a.zinv = zinv; a.masked = masked; a.status = status;
    a.nchunks = p.nchunks;
    a.tickets = reinterpret_cast<int*>(workspace);
    a.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + LSQ_TICKET_BYTES);
    dim3 grid(a.nchunks, B, p.groups);
    if (Lmap > L) return launch_lanes(p, 0, o_dtype, grid, stream, a, rowsums, keep, Lmap, 0);
    if (act == LF_ACT_SQUARE)
        o_dtype == LF_BF16 ? launch_rowsums<LF_ACT_SQUARE, true>(p.nl, grid, stream, a, rowsums, keep)
                           : launch_rowsums<LF_ACT_SQUARE, false>(p.nl, grid, stream, a, rowsums, keep);
    else
        o_dtype == LF_BF16 ? launch_rowsums<LSQ_ACT_RUNTIME, true>(p.nl, grid, stream, a, rowsums, keep)
                           : launch_rowsums<LSQ_ACT_RUNTIME, false>(p.nl, grid, stream, a, rowsums, keep);
    return check_launch();
}

extern "C" int lf_lsq_fwd_rowsums(const void* o, int o_dtype, const float* xtab, const float* yrow, int B, int L, int H,
                                  int W, int order, int mask_rows, int act, double reg_ls, int solver, double* beta,
                                  double* zinv, float* masked, int* status, float* rowsums, void* workspace,
                                  size_t workspace_bytes, lf_stream_t stream_) {
    return lsq_fwd_rowsums(o, o_dtype, xtab, yrow, nullptr, B, L, L, H, W, order, mask_rows, act, reg_ls, solver, beta, zinv,
                           masked, status, rowsums, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_fwd_rowsums_keep(const void* o, int o_dtype, const float* xtab, const float* yrow,
                                       const uint8_t* keep, int B, int L, int H, int W, int order, int mask_rows,
                                       int act, double reg_ls, int solver, double* beta, double* zinv, float* masked,
                                       int* status, float* rowsums, void* workspace, size_t workspace_bytes,
                                       lf_stream_t stream_) {
    LF_REQUIRE(keep);
    return lsq_fwd_rowsums(o, o_dtype, xtab, yrow, keep, B, L, L, H, W, order, mask_rows, act, reg_ls, solver, beta, zinv,
                           masked, status, rowsums, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_grid_grad(const float* rowsums, const float* yrow, const double* beta, const double* zinv,
                                const double* gbeta, int B, int L, int H, int order, int mask_rows, double* g_rowp,
                                lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(rowsums && yrow && beta && zinv && gbeta && g_rowp);
    LF_REQUIRE(B > 0 && L > 0 && H > 0 && order >= 0 && order <= LF_MAX_ORDER && mask_rows >= 0 && mask_rows <= H);
    lf_launch(lsq_grid_grad_kernel, (H + LSQ_GG_THREADS - 1) / LSQ_GG_THREADS, LSQ_GG_THREADS, 0, stream, rowsums, yrow,
              beta, zinv, gbeta, B, L, H, order, mask_rows, g_rowp);
    return check_launch();
}

// lf_lsq_bwd and lf_lsq_bwd_keep (keep = NULL: the KEEP = false kernels)
static int lsq_bwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
                   const uint8_t* keep, int B, int L, int Lmap, int H, int W, int order, int mask_rows, int act,
                   const double* beta, const double* zinv, const double* gbeta, void* d_o, cudaStream_t stream) {
    LF_REQUIRE(o && xtab && (ytab || yrow) && beta && zinv && gbeta && d_o);
    LF_REQUIRE(Lmap >= L && Lmap <= 65535);
    LsqPlan p{};
    const int rc = lsq_plan(1, o_dtype, yrow != nullptr, ytab != nullptr, B, L, H, W, order, mask_rows, act, &p);
    if (rc != LF_OK) return rc;
    if (p.rowsep) LF_REQUIRE(aligned16(o) && aligned16(xtab) && aligned16(d_o) && aligned16(keep));
    LsqArgs a{};
    a.o = o; a.xtab = xtab; a.ytab = ytab; a.yrow = yrow;
    a.B = B; a.L = L; a.H = H; a.W = W; a.order = order; a.mask_rows = mask_rows; a.act = act;
    a.beta = const_cast<double*>(beta); a.zinv = const_cast<double*>(zinv); a.gbeta = gbeta; a.d_o = d_o;
    a.nchunks = p.nchunks;
    dim3 grid(a.nchunks, B, p.groups);
    if (Lmap > L) return launch_lanes(p, 1, o_dtype, grid, stream, a, nullptr, keep, Lmap, 0);
    if (p.rowsep) {
        if (keep)
            LSQ_DISPATCH_NL(lsq_bwd_rowsep_keep_kernel, p.nl, grid, a, keep);
        else
            LSQ_DISPATCH_NL(lsq_bwd_rowsep_kernel, p.nl, grid, a);
    } else {
        if (keep)
            LSQ_DISPATCH(lsq_bwd_general_keep_kernel, grid, a, keep);
        else
            LSQ_DISPATCH(lsq_bwd_general_kernel, grid, a);
    }
    return check_launch();
}

extern "C" int lf_lsq_bwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow, int B,
                          int L, int H, int W, int order, int mask_rows, int act, const double* beta,
                          const double* zinv, const double* gbeta, void* d_o, lf_stream_t stream_) {
    return lsq_bwd(o, o_dtype, xtab, ytab, yrow, nullptr, B, L, L, H, W, order, mask_rows, act, beta, zinv, gbeta, d_o,
                   reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_bwd_keep(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
                               const uint8_t* keep, int B, int L, int H, int W, int order, int mask_rows, int act,
                               const double* beta, const double* zinv, const double* gbeta, void* d_o,
                               lf_stream_t stream_) {
    LF_REQUIRE(keep);
    return lsq_bwd(o, o_dtype, xtab, ytab, yrow, keep, B, L, L, H, W, order, mask_rows, act, beta, zinv, gbeta, d_o,
                   reinterpret_cast<cudaStream_t>(stream_));
}

// ---------------------------------------------------------------------------------------------------------------------
// Per-image tables (a predicted homography, --predict_homography): xtab [B][H][W] and yrow [B][H], image b fitted on its
// own slice, on the row-separable kernels only (yrow is required and W must suit the 16-byte loads).  Same plan, checks,
// workspace and outputs as the shared-table entry points; rowsums (NULL: none, as lf_lsq_fwd) and keep (NULL: no map)
// select the instantiation, exactly as lf_lsq_fwd_rowsums / the *_keep entry points do.
template <int ACT_T, bool BF16, int NL>
static void launch_fwd_pi_nl(dim3 grid, cudaStream_t stream, const LsqArgs& a, float* rowsums, const uint8_t* keep) {
    if (rowsums) {
        if (keep)
            lf_launch(lsq_fwd_rowsep_pi_kernel<ACT_T, BF16, NL, true, true>, grid, LSQ_THREADS, 0, stream, a, rowsums, keep);
        else
            lf_launch(lsq_fwd_rowsep_pi_kernel<ACT_T, BF16, NL, true, false>, grid, LSQ_THREADS, 0, stream, a, rowsums, keep);
    } else {
        if (keep)
            lf_launch(lsq_fwd_rowsep_pi_kernel<ACT_T, BF16, NL, false, true>, grid, LSQ_THREADS, 0, stream, a, rowsums, keep);
        else
            lf_launch(lsq_fwd_rowsep_pi_kernel<ACT_T, BF16, NL, false, false>, grid, LSQ_THREADS, 0, stream, a, rowsums, keep);
    }
}

template <int ACT_T, bool BF16>
static void launch_fwd_pi(int nl, dim3 grid, cudaStream_t stream, const LsqArgs& a, float* rowsums, const uint8_t* keep) {
    switch (nl) {
        case 1: launch_fwd_pi_nl<ACT_T, BF16, 1>(grid, stream, a, rowsums, keep); break;
        case 2: launch_fwd_pi_nl<ACT_T, BF16, 2>(grid, stream, a, rowsums, keep); break;
        case 3: launch_fwd_pi_nl<ACT_T, BF16, 3>(grid, stream, a, rowsums, keep); break;
        default: launch_fwd_pi_nl<ACT_T, BF16, 4>(grid, stream, a, rowsums, keep); break;
    }
}

static int lsq_fwd_per_image(const void* o, int o_dtype, const float* xtab, const float* yrow, const uint8_t* keep, int B,
                             int L, int Lmap, int H, int W, int order, int mask_rows, int act, double reg_ls, int solver,
                             double* beta, double* zinv, float* masked, int* status, float* rowsums, void* workspace,
                             size_t workspace_bytes, cudaStream_t stream) {
    LF_REQUIRE(o && xtab && yrow && beta && zinv && status && workspace);
    LF_REQUIRE(Lmap >= L && Lmap <= 65535);
    LF_REQUIRE(solver == LF_SOLVER_INVERSE || solver == LF_SOLVER_CHOLESKY);
    LsqPlan p{};
    const int rc = lsq_plan(0, o_dtype, 1, 0, B, L, H, W, order, mask_rows, act, &p);
    if (rc != LF_OK) return rc;
    if (!p.rowsep) return LF_ERR_INVALID_ARGUMENT;
    if (workspace_bytes < lf_lsq_workspace_bytes(B, L, H, W, order)) return LF_ERR_WORKSPACE_TOO_SMALL;
    LF_REQUIRE(aligned16(o) && aligned16(xtab) && aligned16(masked) && aligned16(keep));
    LsqArgs a{};
    a.o = o; a.xtab = xtab; a.yrow = yrow;
    a.B = B; a.L = L; a.H = H; a.W = W; a.order = order; a.mask_rows = mask_rows; a.act = act; a.solver = solver;
    a.reg_ls = reg_ls; a.beta = beta; a.zinv = zinv; a.masked = masked; a.status = status;
    a.nchunks = p.nchunks;
    a.tickets = reinterpret_cast<int*>(workspace);
    a.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + LSQ_TICKET_BYTES);
    dim3 grid(a.nchunks, B, p.groups);
    if (Lmap > L) return launch_lanes(p, 0, o_dtype, grid, stream, a, rowsums, keep, Lmap, 1);
    if (act == LF_ACT_SQUARE)
        o_dtype == LF_BF16 ? launch_fwd_pi<LF_ACT_SQUARE, true>(p.nl, grid, stream, a, rowsums, keep)
                           : launch_fwd_pi<LF_ACT_SQUARE, false>(p.nl, grid, stream, a, rowsums, keep);
    else
        o_dtype == LF_BF16 ? launch_fwd_pi<LSQ_ACT_RUNTIME, true>(p.nl, grid, stream, a, rowsums, keep)
                           : launch_fwd_pi<LSQ_ACT_RUNTIME, false>(p.nl, grid, stream, a, rowsums, keep);
    return check_launch();
}

static int lsq_bwd_per_image(const void* o, int o_dtype, const float* xtab, const float* yrow, const uint8_t* keep, int B,
                             int L, int Lmap, int H, int W, int order, int mask_rows, int act, const double* beta,
                             const double* zinv, const double* gbeta, void* d_o, cudaStream_t stream) {
    LF_REQUIRE(o && xtab && yrow && beta && zinv && gbeta && d_o);
    LF_REQUIRE(Lmap >= L && Lmap <= 65535);
    LsqPlan p{};
    const int rc = lsq_plan(1, o_dtype, 1, 0, B, L, H, W, order, mask_rows, act, &p);
    if (rc != LF_OK) return rc;
    if (!p.rowsep) return LF_ERR_INVALID_ARGUMENT;
    LF_REQUIRE(aligned16(o) && aligned16(xtab) && aligned16(d_o) && aligned16(keep));
    LsqArgs a{};
    a.o = o; a.xtab = xtab; a.yrow = yrow;
    a.B = B; a.L = L; a.H = H; a.W = W; a.order = order; a.mask_rows = mask_rows; a.act = act;
    a.beta = const_cast<double*>(beta); a.zinv = const_cast<double*>(zinv); a.gbeta = gbeta; a.d_o = d_o;
    a.nchunks = p.nchunks;
    dim3 grid(a.nchunks, B, p.groups);
    if (Lmap > L) return launch_lanes(p, 1, o_dtype, grid, stream, a, nullptr, keep, Lmap, 1);
    if (keep)
        LSQ_DISPATCH_NL(lsq_bwd_rowsep_pi_keep_kernel, p.nl, grid, a, keep);
    else
        LSQ_DISPATCH_NL(lsq_bwd_rowsep_pi_kernel, p.nl, grid, a, keep);
    return check_launch();
}

extern "C" int lf_lsq_fwd_per_image(const void* o, int o_dtype, const float* xtab, const float* yrow, const uint8_t* keep,
                                    int B, int L, int H, int W, int order, int mask_rows, int act, double reg_ls,
                                    int solver, double* beta, double* zinv, float* masked, int* status, float* rowsums,
                                    void* workspace, size_t workspace_bytes, lf_stream_t stream_) {
    return lsq_fwd_per_image(o, o_dtype, xtab, yrow, keep, B, L, L, H, W, order, mask_rows, act, reg_ls, solver, beta, zinv,
                             masked, status, rowsums, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_bwd_per_image(const void* o, int o_dtype, const float* xtab, const float* yrow, const uint8_t* keep,
                                    int B, int L, int H, int W, int order, int mask_rows, int act, const double* beta,
                                    const double* zinv, const double* gbeta, void* d_o, lf_stream_t stream_) {
    return lsq_bwd_per_image(o, o_dtype, xtab, yrow, keep, B, L, L, H, W, order, mask_rows, act, beta, zinv, gbeta, d_o,
                             reinterpret_cast<cudaStream_t>(stream_));
}

// ---------------------------------------------------------------------------------------------------------------------
// Prefix fits (a lane curriculum): the entry points above with the maps' channel count Lmap >= L after L.  Lanes [0, L)
// of o [B][Lmap][H][W] are fitted exactly as the plain entry point fits o[:, :L]; masked is [B][L][H][W]; d_o is
// [B][Lmap][H][W] with lanes [L, Lmap) zero (written by the backward's own launch).  Lmap = L runs the plain kernels.
extern "C" int lf_lsq_fwd_lanes(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow, int B,
                                int L, int Lmap, int H, int W, int order, int mask_rows, int act, double reg_ls, int solver,
                                double* beta, double* zinv, float* masked, int* status, void* workspace,
                                size_t workspace_bytes, lf_stream_t stream_) {
    return lsq_fwd(o, o_dtype, xtab, ytab, yrow, nullptr, B, L, Lmap, H, W, order, mask_rows, act, reg_ls, solver, beta,
                   zinv, masked, status, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_fwd_keep_lanes(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
                                     const uint8_t* keep, int B, int L, int Lmap, int H, int W, int order, int mask_rows,
                                     int act, double reg_ls, int solver, double* beta, double* zinv, float* masked,
                                     int* status, void* workspace, size_t workspace_bytes, lf_stream_t stream_) {
    LF_REQUIRE(keep);
    return lsq_fwd(o, o_dtype, xtab, ytab, yrow, keep, B, L, Lmap, H, W, order, mask_rows, act, reg_ls, solver, beta, zinv,
                   masked, status, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_fwd_rowsums_lanes(const void* o, int o_dtype, const float* xtab, const float* yrow, int B, int L,
                                        int Lmap, int H, int W, int order, int mask_rows, int act, double reg_ls,
                                        int solver, double* beta, double* zinv, float* masked, int* status,
                                        float* rowsums, void* workspace, size_t workspace_bytes, lf_stream_t stream_) {
    return lsq_fwd_rowsums(o, o_dtype, xtab, yrow, nullptr, B, L, Lmap, H, W, order, mask_rows, act, reg_ls, solver, beta,
                           zinv, masked, status, rowsums, workspace, workspace_bytes,
                           reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_fwd_rowsums_keep_lanes(const void* o, int o_dtype, const float* xtab, const float* yrow,
                                             const uint8_t* keep, int B, int L, int Lmap, int H, int W, int order,
                                             int mask_rows, int act, double reg_ls, int solver, double* beta,
                                             double* zinv, float* masked, int* status, float* rowsums, void* workspace,
                                             size_t workspace_bytes, lf_stream_t stream_) {
    LF_REQUIRE(keep);
    return lsq_fwd_rowsums(o, o_dtype, xtab, yrow, keep, B, L, Lmap, H, W, order, mask_rows, act, reg_ls, solver, beta,
                           zinv, masked, status, rowsums, workspace, workspace_bytes,
                           reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_bwd_lanes(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow, int B,
                                int L, int Lmap, int H, int W, int order, int mask_rows, int act, const double* beta,
                                const double* zinv, const double* gbeta, void* d_o, lf_stream_t stream_) {
    return lsq_bwd(o, o_dtype, xtab, ytab, yrow, nullptr, B, L, Lmap, H, W, order, mask_rows, act, beta, zinv, gbeta, d_o,
                   reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_bwd_keep_lanes(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
                                     const uint8_t* keep, int B, int L, int Lmap, int H, int W, int order, int mask_rows,
                                     int act, const double* beta, const double* zinv, const double* gbeta, void* d_o,
                                     lf_stream_t stream_) {
    LF_REQUIRE(keep);
    return lsq_bwd(o, o_dtype, xtab, ytab, yrow, keep, B, L, Lmap, H, W, order, mask_rows, act, beta, zinv, gbeta, d_o,
                   reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_fwd_per_image_lanes(const void* o, int o_dtype, const float* xtab, const float* yrow,
                                          const uint8_t* keep, int B, int L, int Lmap, int H, int W, int order,
                                          int mask_rows, int act, double reg_ls, int solver, double* beta, double* zinv,
                                          float* masked, int* status, float* rowsums, void* workspace,
                                          size_t workspace_bytes, lf_stream_t stream_) {
    return lsq_fwd_per_image(o, o_dtype, xtab, yrow, keep, B, L, Lmap, H, W, order, mask_rows, act, reg_ls, solver, beta,
                             zinv, masked, status, rowsums, workspace, workspace_bytes,
                             reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int lf_lsq_bwd_per_image_lanes(const void* o, int o_dtype, const float* xtab, const float* yrow,
                                          const uint8_t* keep, int B, int L, int Lmap, int H, int W, int order,
                                          int mask_rows, int act, const double* beta, const double* zinv,
                                          const double* gbeta, void* d_o, lf_stream_t stream_) {
    return lsq_bwd_per_image(o, o_dtype, xtab, yrow, keep, B, L, Lmap, H, W, order, mask_rows, act, beta, zinv, gbeta, d_o,
                             reinterpret_cast<cudaStream_t>(stream_));
}

// g_rowp [B][H][3] f64: image b's table gradient, summed over its lanes (rowsums, beta, zinv, gbeta as lf_lsq_grid_grad,
// yrow [B][H]) -- DEVICE.
extern "C" int lf_lsq_grid_grad_per_image(const float* rowsums, const float* yrow, const double* beta, const double* zinv,
                                          const double* gbeta, int B, int L, int H, int order, int mask_rows,
                                          double* g_rowp, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(rowsums && yrow && beta && zinv && gbeta && g_rowp);
    LF_REQUIRE(B > 0 && B <= 65535 && L > 0 && H > 0 && order >= 0 && order <= LF_MAX_ORDER && mask_rows >= 0 &&
               mask_rows <= H);
    lf_launch(lsq_grid_grad_pi_kernel, dim3((H + LSQ_GG_THREADS - 1) / LSQ_GG_THREADS, B), LSQ_GG_THREADS, 0, stream,
              rowsums, yrow, beta, zinv, gbeta, L, H, order, mask_rows, g_rowp);
    return check_launch();
}
