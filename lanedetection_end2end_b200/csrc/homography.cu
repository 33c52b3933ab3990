// Learned bird's-eye-view homography (DESIGN.md "Learned homography"): the warp of get_homography(resize) with its source
// corners shifted by theta [5] (float32), its tables for the least-squares layer and the back-projection loss built on the
// device every forward, and the gradient of the loss with respect to theta.
//
//   source corners (x0, yt) (x1, yt) (x2, yb) (x3, yb):  x_i = base_i + theta_i * 2R,  yt = base_top + theta_4 * R
//   destination corners fixed;  M maps source to destination, M^-1 destination to source.
//
// Both warps keep the two corner rows level, so they are row-preserving: M = [[a,b,c],[0,e,f],[0,g,1]] in closed form
// (row_preserving() below), no 8x8 solve.  Row v of the network image then maps to one bird's-eye-view row:
//   den_v = g v + 1,  alpha_v = a / den_v,  gamma_v = (b v + c) / den_v,  y'_v = (e v + f) / den_v
//   xtab[v][u] = alpha_v u + gamma_v,  yrow[v] = y_const - y'_v          (BP/Networks/LSQ_layer.py:93-94)
// The backward runs the same closed form on dual numbers with one tangent per entry of theta (forward-mode
// differentiation: exact, a few hundred fp64 operations per thread) and sums the chain rule over the rows, the 56 sample
// rows of the loss and M^-1 in a fixed order.  Everything is fp64; no host synchronisation.
#include "lf_common.cuh"

namespace lf {

constexpr int HG_THREADS = 128;
constexpr int HG_BWD_THREADS = 256;
constexpr int HG_NT = 5;          // entries of theta
constexpr int HG_SAMPLES = 56;    // the loss's sample rows (h_samples 160..710 step 10)

template <int N>
struct Dual {
    double v, d[N];
    __host__ __device__ Dual(double x = 0.0) : v(x) {
        for (int i = 0; i < N; ++i) d[i] = 0.0;
    }
};
template <int N>
__host__ __device__ inline Dual<N> operator+(const Dual<N>& a, const Dual<N>& b) {
    Dual<N> r(a.v + b.v);
    for (int i = 0; i < N; ++i) r.d[i] = a.d[i] + b.d[i];
    return r;
}
template <int N>
__host__ __device__ inline Dual<N> operator-(const Dual<N>& a, const Dual<N>& b) {
    Dual<N> r(a.v - b.v);
    for (int i = 0; i < N; ++i) r.d[i] = a.d[i] - b.d[i];
    return r;
}
template <int N>
__host__ __device__ inline Dual<N> operator*(const Dual<N>& a, const Dual<N>& b) {
    Dual<N> r(a.v * b.v);
    for (int i = 0; i < N; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i];
    return r;
}
template <int N>
__host__ __device__ inline Dual<N> operator/(const Dual<N>& a, const Dual<N>& b) {
    const double q = a.v / b.v;
    Dual<N> r(q);
    for (int i = 0; i < N; ++i) r.d[i] = (a.d[i] - q * b.d[i]) / b.v;
    return r;
}

// Row-preserving homography mapping (sx0, yt), (sx1, yt), (sx2, yb), (sx3, yb) to (dx0, Yt), (dx1, Yt), (dx2, Yb),
// (dx3, Yb), normalised to m[8] = 1 (as cv2.getPerspectiveTransform).  Per row r the map is affine in x with scale
// s_r = a / (g y_r + 1) and offset o_r; s_t (g yt + 1) = s_b (g yb + 1) gives g, then (b, c) and (e, f) are 2x2 solves.
template <class T>
__host__ __device__ inline void row_preserving(const T* sx, T yt, T yb, const T* dx, T Yt, T Yb, T* m) {
    const T st = (dx[1] - dx[0]) / (sx[1] - sx[0]), sb = (dx[3] - dx[2]) / (sx[3] - sx[2]);
    const T ot = dx[0] - st * sx[0], ob = dx[2] - sb * sx[2];
    const T one(1.0);
    const T g = (sb - st) / (st * yt - sb * yb);
    const T kt = g * yt + one, kb = g * yb + one;
    const T b = (ot * kt - ob * kb) / (yt - yb);
    const T e = (Yt * kt - Yb * kb) / (yt - yb);
    m[0] = st * kt;
    m[1] = b;
    m[2] = ot * kt - b * yt;
    m[3] = T(0.0);
    m[4] = e;
    m[5] = Yt * kt - e * yt;
    m[6] = T(0.0);
    m[7] = g;
    m[8] = one;
}

// The corners get_homography(resize) hands cv2 (float32, BP/Networks/utils.py:104-121), shifted by theta.
template <class T>
__host__ __device__ inline void warp_corners(const float* theta, int R, T* sx, T& yt, T& yb, T* dx, T& Yt, T& Yb) {
    const double w = 2.0 * R;
    const double bx[4] = {(double)(float)(0.45 * w), (double)(float)(0.55 * w), (double)(float)(0.02 * w),
                          (double)(float)(0.97 * w)};
    const double dxb[4] = {(double)(float)(0.45 * w), (double)(float)(0.55 * w), (double)(float)(0.45 * w),
                           (double)(float)(0.55 * w)};
    const double top = (double)(float)(0.20 * R), bottom = (double)(float)(R - 1);
    for (int i = 0; i < 4; ++i) {
        sx[i] = T(bx[i]) + T((double)theta[i]) * T(w);
        dx[i] = T(dxb[i]);
    }
    yt = T(top) + T((double)theta[4]) * T((double)R);
    yb = T(bottom);
    Yt = T(top);
    Yb = T(bottom);
}

// M (m[0..8]) and M^-1 (m[9..17]) of theta
template <class T>
__host__ __device__ inline void warp_pair(const float* theta, int R, T* m) {
    T sx[4], dx[4], yt, yb, Yt, Yb;
    warp_corners<T>(theta, R, sx, yt, yb, dx, Yt, Yb);
    row_preserving<T>(sx, yt, yb, dx, Yt, Yb, m);
    row_preserving<T>(dx, Yt, Yb, sx, yt, yb, m + 9);
}
// the same on dual numbers, seeded so that tangent j is d/dtheta_j
__host__ __device__ inline void warp_pair_dual(const float* theta, int R, Dual<HG_NT>* m) {
    const double w = 2.0 * R;
    Dual<HG_NT> sx[4], dx[4], yt, yb, Yt, Yb;
    warp_corners<Dual<HG_NT>>(theta, R, sx, yt, yb, dx, Yt, Yb);
    for (int i = 0; i < 4; ++i) sx[i].d[i] = w;
    yt.d[4] = (double)R;
    row_preserving(sx, yt, yb, dx, Yt, Yb, m);
    row_preserving(dx, Yt, Yb, sx, yt, yb, m + 9);
}

// image row of the loss's sample s (BP/Loss_crit.py:173; the reference divides by 2.5 whatever --resize is)
__host__ __device__ inline double sample_row(int s) { return (double)(160 + 10 * s - 80) / 2.5; }

// alpha, gamma, y' of image row v
template <class T>
__host__ __device__ inline void row_params(const T* m, double v, T* p) {
    const T vv(v);
    const T den = m[7] * vv + m[8];
    p[0] = m[0] / den;
    p[1] = (m[1] * vv + m[2]) / den;
    p[2] = (m[4] * vv + m[5]) / den;
}

__global__ void __launch_bounds__(HG_THREADS) homography_tables_kernel(const float* __restrict__ theta, int R, int mask_rows,
                                                                        double y_const, double* __restrict__ M,
                                                                        double* __restrict__ Minv,
                                                                        double* __restrict__ rowp, float* __restrict__ xtab,
                                                                        float* __restrict__ yrow, double* __restrict__ yk,
                                                                        int* __restrict__ status) {
    pdl_entry();
    const int v = blockIdx.x, t = threadIdx.x, W = 2 * R;
    float th[HG_NT];
    for (int j = 0; j < HG_NT; ++j) th[j] = theta[j];
    double m[18];
    warp_pair<double>(th, R, m);
    double p[3];
    row_params<double>(m, (double)v, p);
    const bool guarded = v >= mask_rows;
    bool bad = false;
    for (int u = t; u < W; u += HG_THREADS) {
        const float x = (float)(p[0] * u + p[1]);
        xtab[(size_t)v * W + u] = x;
        bad |= !isfinite(x);
    }
    if (t == 0) {
        // with m22 = 1 the rows below the vanishing line have den < 0: a usable row has the bottom row's sign of den
        const double den = (m[7] * v + m[8]) * (m[7] * (R - 1) + m[8]);
        const float y = (float)(y_const - p[2]);
        rowp[(size_t)v * 3 + 0] = p[0];
        rowp[(size_t)v * 3 + 1] = p[1];
        rowp[(size_t)v * 3 + 2] = p[2];
        yrow[v] = y;
        bad |= !(den > 0.0) || !isfinite(p[0]) || !isfinite(p[1]) || !isfinite(y);
    }
    // an unmasked row at or above the vanishing line: the batch is skipped like a singular system
    if (guarded && bad) atomicOr(status, LF_STATUS_NONFINITE);
    if (v == 0) {
        if (t < 9) M[t] = m[t];
        if (t >= 9 && t < 18) Minv[t - 9] = m[t];
        if (t < HG_SAMPLES) {
            const double y = sample_row(t);
            yk[t] = (m[4] * y + m[5]) / (m[7] * y + m[8]);
        }
    }
}

// One thread's share of dL/dtheta (N tangents): rows t, t + T, ... (unmasked rows only), sample t < 56, and M^-1 on
// thread 0.
template <int N>
__host__ __device__ inline void homography_bwd_partial(const Dual<N>* m, int t, int nthreads, int R, int mask_rows,
                                                       const double* g_rowp, const double* g_minv, const double* g_yk,
                                                       double* acc) {
    for (int j = 0; j < N; ++j) acc[j] = 0.0;
    if (g_rowp)
        for (int v = mask_rows + t; v < R; v += nthreads) {
            Dual<N> p[3];
            row_params(m, (double)v, p);
            for (int k = 0; k < 3; ++k) {
                const double g = g_rowp[(size_t)v * 3 + k];
                for (int j = 0; j < N; ++j) acc[j] += g * p[k].d[j];
            }
        }
    if (g_yk && t < HG_SAMPLES) {
        const Dual<N> y(sample_row(t));
        const Dual<N> q = (m[4] * y + m[5]) / (m[7] * y + m[8]);
        for (int j = 0; j < N; ++j) acc[j] += g_yk[t] * q.d[j];
    }
    if (g_minv && t == 0)
        for (int i = 0; i < 9; ++i)
            for (int j = 0; j < N; ++j) acc[j] += g_minv[i] * m[9 + i].d[j];
}

__global__ void __launch_bounds__(HG_BWD_THREADS) homography_bwd_kernel(const float* __restrict__ theta, int R, int mask_rows,
                                                                         const double* __restrict__ g_rowp,
                                                                         const double* __restrict__ g_minv,
                                                                         const double* __restrict__ g_yk,
                                                                         float* __restrict__ g_theta) {
    pdl_entry();
    __shared__ double red[HG_NT][HG_BWD_THREADS];
    const int t = threadIdx.x;
    float th[HG_NT];
    for (int j = 0; j < HG_NT; ++j) th[j] = theta[j];
    Dual<HG_NT> m[18];
    warp_pair_dual(th, R, m);
    double acc[HG_NT];
    homography_bwd_partial<HG_NT>(m, t, HG_BWD_THREADS, R, mask_rows, g_rowp, g_minv, g_yk, acc);
    for (int j = 0; j < HG_NT; ++j) red[j][t] = acc[j];
    __syncthreads();
    for (int w = HG_BWD_THREADS / 2; w > 0; w >>= 1) {   // fixed tree
        if (t < w)
            for (int j = 0; j < HG_NT; ++j) red[j][t] += red[j][t + w];
        __syncthreads();
    }
    if (t < HG_NT) g_theta[t] = (float)red[t][0];
}

// ---------------------------------------------------------------------------------------------------------------------
// Predicted homography (--predict_homography, DESIGN.md "Predicted homography"): one warp per image from the branch's
// output z [B][NZ], in one of two parametrisations of get_homography(resize)'s corners (--predict_homography_corners).
// Both keep the corner rows level, so both warps stay row-preserving and the closed form above applies (no 6x6 or 8x8
// solve).
//
//   destination (the reference DLT's): delta = tanh(z) / 16 [3] moves the DESTINATION corners -- the left column by
//     delta_0 * 2R, the right column by delta_1 * 2R, the top row by delta_2 * R -- with the source corners and the bottom
//     row fixed.  Any two such warps differ by an affine change of the bird's-eye-view coordinates, which the fit and
//     the back-projection undo: the loss does not see this warp (NOTES.md).
//   source (--learn_homography's, per image): theta = tanh(z) / 64 [5], rounded to float32, moves the SOURCE corners as
//     warp_corners does; each image's tables are lf_homography_tables(theta_b).
constexpr int PH_NZ = 3;

template <class T>
__host__ __device__ inline void predicted_pair(const T* delta, int R, T* m) {
    const double w = 2.0 * R;
    const float zero5[HG_NT] = {0.f, 0.f, 0.f, 0.f, 0.f};
    T sx[4], dx[4], yt, yb, Yt, Yb;
    warp_corners<T>(zero5, R, sx, yt, yb, dx, Yt, Yb);
    dx[0] = dx[0] + delta[0] * T(w);
    dx[2] = dx[2] + delta[0] * T(w);
    dx[1] = dx[1] + delta[1] * T(w);
    dx[3] = dx[3] + delta[1] * T(w);
    Yt = Yt + delta[2] * T((double)R);
    row_preserving<T>(sx, yt, yb, dx, Yt, Yb, m);
    row_preserving<T>(dx, Yt, Yb, sx, yt, yb, m + 9);
}

// delta_j = tanh(z_j) / 16 in fp64, with tangent j seeded as d delta_j / d z_j = (1 - tanh^2) / 16
__host__ __device__ inline void predicted_delta(const float* z, double* delta, Dual<PH_NZ>* dd) {
    for (int j = 0; j < PH_NZ; ++j) {
        const double t = tanh((double)z[j]);
        delta[j] = t / 16.0;
        if (dd) {
            dd[j] = Dual<PH_NZ>(delta[j]);
            dd[j].d[j] = (1.0 - t * t) / 16.0;
        }
    }
}

// The parametrisations as policies of the kernels and host hooks below.  NZ: entries of z per image; Param: the type of
// the per-image parameters the tables kernel writes (delta f64, theta f32); warp(): those parameters and the pair
// (M, M^-1); warp_dual(): the pair on dual numbers; dz(): dL/dz_j from the tree's sum of tangent j.
struct DestinationCorners {
    static constexpr int NZ = PH_NZ;
    using Param = double;
    __host__ __device__ static void warp(const float* z, int R, double* delta, double* m) {
        predicted_delta(z, delta, nullptr);
        predicted_pair<double>(delta, R, m);
    }
    // tangent j is d/dz_j (seeded in predicted_delta), so the sum is dL/dz_j
    __host__ __device__ static void warp_dual(const float* z, int R, Dual<NZ>* m) {
        double dl[NZ];
        Dual<NZ> dd[NZ];
        predicted_delta(z, dl, dd);
        predicted_pair<Dual<NZ>>(dd, R, m);
    }
    __host__ __device__ static double dz(const float*, int, double g) { return g; }
};

struct SourceCorners {
    static constexpr int NZ = HG_NT;
    using Param = float;
    // theta_j = tanh(z_j) / 64 rounded to float32: the theta of --learn_homography, so warp_pair gives its bits
    __host__ __device__ static void theta_of(const float* z, float* theta) {
        for (int j = 0; j < NZ; ++j) theta[j] = (float)(tanh((double)z[j]) / 64.0);
    }
    __host__ __device__ static void warp(const float* z, int R, float* theta, double* m) {
        theta_of(z, theta);
        warp_pair<double>(theta, R, m);
    }
    // tangent j is d/dtheta_j (warp_pair_dual's seeds 2R, R): the tree reduces dL/dtheta_b exactly as
    // homography_bwd_kernel reduces dL/dtheta, and dz() applies d theta_j / d z_j = (1 - tanh^2 z_j) / 64 once, after it
    __host__ __device__ static void warp_dual(const float* z, int R, Dual<NZ>* m) {
        float th[NZ];
        theta_of(z, th);
        warp_pair_dual(th, R, m);
    }
    __host__ __device__ static double dz(const float* z, int j, double g) {
        const double t = tanh((double)z[j]);
        return g * ((1.0 - t * t) / 64.0);
    }
};

// grid (R, B): image b's row v, as homography_tables_kernel on image b's warp.  Per-image outputs are contiguous slices:
// param [B][NZ], M / Minv [B][9], rowp [B][R][3], xtab [B][R][2R], yrow [B][R], yk [B][56].
template <class P>
__global__ void __launch_bounds__(HG_THREADS) predicted_tables_kernel(const float* __restrict__ z, int R, int mask_rows,
                                                                       double y_const, typename P::Param* __restrict__ param,
                                                                       double* __restrict__ M, double* __restrict__ Minv,
                                                                       double* __restrict__ rowp, float* __restrict__ xtab,
                                                                       float* __restrict__ yrow, double* __restrict__ yk,
                                                                       int* __restrict__ status) {
    pdl_entry();
    const int v = blockIdx.x, b = blockIdx.y, t = threadIdx.x, W = 2 * R;
    float zb[P::NZ];
    for (int j = 0; j < P::NZ; ++j) zb[j] = z[(size_t)b * P::NZ + j];
    typename P::Param q[P::NZ];
    double m[18];
    P::warp(zb, R, q, m);
    double p[3];
    row_params<double>(m, (double)v, p);
    const bool guarded = v >= mask_rows;
    bool bad = false;
    float* xrow = xtab + ((size_t)b * R + v) * W;
    for (int u = t; u < W; u += HG_THREADS) {
        const float x = (float)(p[0] * u + p[1]);
        xrow[u] = x;
        bad |= !isfinite(x);
    }
    if (t == 0) {
        const double den = (m[7] * v + m[8]) * (m[7] * (R - 1) + m[8]);
        const float y = (float)(y_const - p[2]);
        double* rp = rowp + ((size_t)b * R + v) * 3;
        rp[0] = p[0];
        rp[1] = p[1];
        rp[2] = p[2];
        yrow[(size_t)b * R + v] = y;
        bad |= !(den > 0.0) || !isfinite(p[0]) || !isfinite(p[1]) || !isfinite(y);
    }
    // any image's unmasked row at or above its vanishing line: the whole batch is skipped like a singular system
    if (guarded && bad) atomicOr(status, LF_STATUS_NONFINITE);
    if (v == 0) {
        if (t < P::NZ) param[(size_t)b * P::NZ + t] = q[t];
        if (t < 9) M[(size_t)b * 9 + t] = m[t];
        if (t >= 9 && t < 18) Minv[(size_t)b * 9 + t - 9] = m[t];
        if (t < HG_SAMPLES) {
            const double y = sample_row(t);
            yk[(size_t)b * HG_SAMPLES + t] = (m[4] * y + m[5]) / (m[7] * y + m[8]);
        }
    }
}

// grid B: dL/dz of image b from its dL/drowp [R][3], dL/dMinv [9], dL/dyk [56]; the fixed tree of homography_bwd_kernel.
// g_sum [B][NZ] (f64, may be NULL): the tree's sums themselves (source corners: dL/dtheta_b).
template <class P>
__global__ void __launch_bounds__(HG_BWD_THREADS) predicted_bwd_kernel(const float* __restrict__ z, int R, int mask_rows,
                                                                        const double* __restrict__ g_rowp,
                                                                        const double* __restrict__ g_minv,
                                                                        const double* __restrict__ g_yk,
                                                                        float* __restrict__ g_z, double* __restrict__ g_sum) {
    pdl_entry();
    __shared__ double red[P::NZ][HG_BWD_THREADS];
    const int t = threadIdx.x, b = blockIdx.x;
    float zb[P::NZ];
    for (int j = 0; j < P::NZ; ++j) zb[j] = z[(size_t)b * P::NZ + j];
    Dual<P::NZ> m[18];
    P::warp_dual(zb, R, m);
    double acc[P::NZ];
    homography_bwd_partial<P::NZ>(m, t, HG_BWD_THREADS, R, mask_rows, g_rowp ? g_rowp + (size_t)b * R * 3 : nullptr,
                                  g_minv ? g_minv + (size_t)b * 9 : nullptr,
                                  g_yk ? g_yk + (size_t)b * HG_SAMPLES : nullptr, acc);
    for (int j = 0; j < P::NZ; ++j) red[j][t] = acc[j];
    __syncthreads();
    for (int w = HG_BWD_THREADS / 2; w > 0; w >>= 1) {
        if (t < w)
            for (int j = 0; j < P::NZ; ++j) red[j][t] += red[j][t + w];
        __syncthreads();
    }
    if (t < P::NZ) {
        g_z[(size_t)b * P::NZ + t] = (float)P::dz(zb, t, red[t][0]);
        if (g_sum) g_sum[(size_t)b * P::NZ + t] = red[t][0];
    }
}

// the same on the host for one image (the test hooks): the kernel's partials and tree
template <class P>
static void predicted_bwd_host(const float* z, int R, int mask_rows, const double* g_rowp, const double* g_minv,
                               const double* g_yk, double* g_z, double* g_sum) {
    Dual<P::NZ> m[18];
    P::warp_dual(z, R, m);
    double red[P::NZ][HG_BWD_THREADS];
    for (int t = 0; t < HG_BWD_THREADS; ++t) {
        double acc[P::NZ];
        homography_bwd_partial<P::NZ>(m, t, HG_BWD_THREADS, R, mask_rows, g_rowp, g_minv, g_yk, acc);
        for (int j = 0; j < P::NZ; ++j) red[j][t] = acc[j];
    }
    for (int w = HG_BWD_THREADS / 2; w > 0; w >>= 1)
        for (int t = 0; t < w; ++t)
            for (int j = 0; j < P::NZ; ++j) red[j][t] += red[j][t + w];
    for (int j = 0; j < P::NZ; ++j) {
        g_z[j] = P::dz(z, j, red[j][0]);
        if (g_sum) g_sum[j] = red[j][0];
    }
}

}  // namespace lf

using namespace lf;

// theta [5] f32, M [9], M^-1 [9] (row-major), rowp [R][3] f64 (alpha, gamma, y'), xtab [R][2R] f32, yrow [R] f32,
// yk [56] f64, status: one int OR-ed with LF_STATUS_NONFINITE -- all DEVICE.
extern "C" int lf_homography_tables(const float* theta, int resize, int mask_rows, double y_const, double* M,
                                    double* Minv, double* rowp, float* xtab, float* yrow, double* yk, int* status, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(theta && M && Minv && rowp && xtab && yrow && yk && status);
    LF_REQUIRE(resize >= 2 && resize <= 65535 && mask_rows >= 0 && mask_rows <= resize);
    lf_launch(homography_tables_kernel, resize, HG_THREADS, 0, stream, theta, resize, mask_rows, y_const, M, Minv, rowp, xtab,
              yrow, yk, status);
    return check_launch();
}

// dL/dtheta [5] f32 from dL/d(alpha, gamma, y') [R][3], dL/dM^-1 [9] and dL/dy'_k [56] (each f64, may be NULL) -- DEVICE.
extern "C" int lf_homography_bwd(const float* theta, int resize, int mask_rows, const double* g_rowp, const double* g_minv,
                                 const double* g_yk, float* g_theta, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(theta && g_theta && resize >= 2 && mask_rows >= 0 && mask_rows <= resize);
    lf_launch(homography_bwd_kernel, 1, HG_BWD_THREADS, 0, stream, theta, resize, mask_rows, g_rowp, g_minv, g_yk, g_theta);
    return check_launch();
}

// TEST HOOKS: the same code on HOST arrays; never called by the package.  lf_homography_host: Mpair [18], and with
// rowp != NULL the (alpha, gamma, y') of every row and with yk != NULL the 56 sample rows' y'.
extern "C" int lf_homography_host(const float* theta, int resize, double* Mpair, double* rowp, double* yk) {
    if (!(theta && Mpair && resize >= 2)) return LF_ERR_INVALID_ARGUMENT;
    warp_pair<double>(theta, resize, Mpair);
    if (rowp)
        for (int v = 0; v < resize; ++v) row_params<double>(Mpair, (double)v, rowp + (size_t)v * 3);
    if (yk)
        for (int s = 0; s < HG_SAMPLES; ++s) {
            const double y = sample_row(s);
            yk[s] = (Mpair[4] * y + Mpair[5]) / (Mpair[7] * y + Mpair[8]);
        }
    return LF_OK;
}

extern "C" int lf_homography_bwd_host(const float* theta, int resize, int mask_rows, const double* g_rowp,
                                      const double* g_minv, const double* g_yk, double* g_theta) {
    if (!(theta && g_theta && resize >= 2 && mask_rows >= 0 && mask_rows <= resize)) return LF_ERR_INVALID_ARGUMENT;
    Dual<HG_NT> m[18];
    warp_pair_dual(theta, resize, m);
    double red[HG_NT][HG_BWD_THREADS];
    for (int t = 0; t < HG_BWD_THREADS; ++t) {
        double acc[HG_NT];
        homography_bwd_partial<HG_NT>(m, t, HG_BWD_THREADS, resize, mask_rows, g_rowp, g_minv, g_yk, acc);
        for (int j = 0; j < HG_NT; ++j) red[j][t] = acc[j];
    }
    for (int w = HG_BWD_THREADS / 2; w > 0; w >>= 1)
        for (int t = 0; t < w; ++t)
            for (int j = 0; j < HG_NT; ++j) red[j][t] += red[j][t + w];
    for (int j = 0; j < HG_NT; ++j) g_theta[j] = red[j][0];
    return LF_OK;
}

template <class P>
static int predicted_tables_run(const float* z, int B, int resize, int mask_rows, double y_const,
                                typename P::Param* param, double* M, double* Minv, double* rowp, float* xtab, float* yrow,
                                double* yk, int* status, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(z && param && M && Minv && rowp && xtab && yrow && yk && status);
    LF_REQUIRE(B > 0 && B <= 65535 && resize >= 2 && resize <= 65535 && mask_rows >= 0 && mask_rows <= resize);
    lf_launch(predicted_tables_kernel<P>, dim3(resize, B), HG_THREADS, 0, stream, z, resize, mask_rows, y_const, param, M,
              Minv, rowp, xtab, yrow, yk, status);
    return check_launch();
}

template <class P>
static int predicted_bwd_run(const float* z, int B, int resize, int mask_rows, const double* g_rowp, const double* g_minv,
                             const double* g_yk, float* g_z, double* g_sum, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(z && g_z && B > 0 && resize >= 2 && mask_rows >= 0 && mask_rows <= resize);
    lf_launch(predicted_bwd_kernel<P>, B, HG_BWD_THREADS, 0, stream, z, resize, mask_rows, g_rowp, g_minv, g_yk, g_z, g_sum);
    return check_launch();
}

// z [B][3] f32 -> delta [B][3], M [B][9], Minv [B][9], rowp [B][R][3], yk [B][56] (f64), xtab [B][R][2R], yrow [B][R]
// (f32); status as lf_homography_tables, OR-ed once for the batch -- all DEVICE.
extern "C" int lf_predicted_homography_tables(const float* z, int B, int resize, int mask_rows, double y_const,
                                              double* delta, double* M, double* Minv, double* rowp, float* xtab,
                                              float* yrow, double* yk, int* status, lf_stream_t stream_) {
    return predicted_tables_run<DestinationCorners>(z, B, resize, mask_rows, y_const, delta, M, Minv, rowp, xtab, yrow, yk,
                                                    status, stream_);
}

// dL/dz [B][3] f32 from dL/drowp [B][R][3], dL/dMinv [B][9], dL/dyk [B][56] (each f64, may be NULL) -- DEVICE.
extern "C" int lf_predicted_homography_bwd(const float* z, int B, int resize, int mask_rows, const double* g_rowp,
                                           const double* g_minv, const double* g_yk, float* g_z, lf_stream_t stream_) {
    return predicted_bwd_run<DestinationCorners>(z, B, resize, mask_rows, g_rowp, g_minv, g_yk, g_z, nullptr, stream_);
}

// The source-corner parametrisation: z [B][5] f32 -> theta [B][5] f32 (tanh(z) / 64 rounded), and the tables of
// lf_predicted_homography_tables, image b's bit for bit lf_homography_tables(theta_b) -- all DEVICE.
extern "C" int lf_predicted_homography_source_tables(const float* z, int B, int resize, int mask_rows, double y_const,
                                                     float* theta, double* M, double* Minv, double* rowp, float* xtab,
                                                     float* yrow, double* yk, int* status, lf_stream_t stream_) {
    return predicted_tables_run<SourceCorners>(z, B, resize, mask_rows, y_const, theta, M, Minv, rowp, xtab, yrow, yk,
                                               status, stream_);
}

// dL/dz [B][5] f32 and, when g_theta is not NULL, dL/dtheta [B][5] f64 (image b's as lf_homography_bwd reduces it) from
// dL/drowp [B][R][3], dL/dMinv [B][9], dL/dyk [B][56] (each f64, may be NULL) -- DEVICE.
extern "C" int lf_predicted_homography_source_bwd(const float* z, int B, int resize, int mask_rows, const double* g_rowp,
                                                  const double* g_minv, const double* g_yk, float* g_z, double* g_theta,
                                                  lf_stream_t stream_) {
    return predicted_bwd_run<SourceCorners>(z, B, resize, mask_rows, g_rowp, g_minv, g_yk, g_z, g_theta, stream_);
}

// TEST HOOKS (host arrays, one image; never called by the package).  lf_predicted_homography_host: Mpair [18] (M, M^-1)
// of delta [3] given directly (inside the tanh box [-1/16, 1/16]^3), rowp [R][3] and yk [56] when not NULL.
// lf_predicted_homography_bwd_host: dL/dz [3] (f64) of z [3], the kernel's partials and tree.
extern "C" int lf_predicted_homography_host(const double* delta, int resize, double* Mpair, double* rowp, double* yk) {
    if (!(delta && Mpair && resize >= 2)) return LF_ERR_INVALID_ARGUMENT;
    predicted_pair<double>(delta, resize, Mpair);
    if (rowp)
        for (int v = 0; v < resize; ++v) row_params<double>(Mpair, (double)v, rowp + (size_t)v * 3);
    if (yk)
        for (int s = 0; s < HG_SAMPLES; ++s) {
            const double y = sample_row(s);
            yk[s] = (Mpair[4] * y + Mpair[5]) / (Mpair[7] * y + Mpair[8]);
        }
    return LF_OK;
}

extern "C" int lf_predicted_homography_bwd_host(const float* z, int resize, int mask_rows, const double* g_rowp,
                                                const double* g_minv, const double* g_yk, double* g_z) {
    if (!(z && g_z && resize >= 2 && mask_rows >= 0 && mask_rows <= resize)) return LF_ERR_INVALID_ARGUMENT;
    predicted_bwd_host<DestinationCorners>(z, resize, mask_rows, g_rowp, g_minv, g_yk, g_z, nullptr);
    return LF_OK;
}

// lf_predicted_homography_source_host: theta [5] (when not NULL) and Mpair [18] of z [5], then as lf_homography_host.
// lf_predicted_homography_source_bwd_host: dL/dz [5] and, when not NULL, dL/dtheta [5] (f64), the kernel's partials
// and tree.
extern "C" int lf_predicted_homography_source_host(const float* z, int resize, float* theta, double* Mpair, double* rowp,
                                                   double* yk) {
    if (!(z && Mpair && resize >= 2)) return LF_ERR_INVALID_ARGUMENT;
    float th[HG_NT];
    SourceCorners::theta_of(z, th);
    if (theta)
        for (int j = 0; j < HG_NT; ++j) theta[j] = th[j];
    return lf_homography_host(th, resize, Mpair, rowp, yk);
}

extern "C" int lf_predicted_homography_source_bwd_host(const float* z, int resize, int mask_rows, const double* g_rowp,
                                                       const double* g_minv, const double* g_yk, double* g_z,
                                                       double* g_theta) {
    if (!(z && g_z && resize >= 2 && mask_rows >= 0 && mask_rows <= resize)) return LF_ERR_INVALID_ARGUMENT;
    predicted_bwd_host<SourceCorners>(z, resize, mask_rows, g_rowp, g_minv, g_yk, g_z, g_theta);
    return LF_OK;
}
