// Fused back-projection loss over all lanes, forward + gradient in one launch (SURVEY.md 8f-1):
// BP/Loss_crit.py:161-218 (`backprojection_loss.forward`) applied per lane and averaged as BP/main.py:297-305 does.
//
//   x'      = Y56 . beta                    (curve sampled at the 56 TuSimple rows, BEV space; Y56 = [y^d .. y 1])
//   x_cal   = (Mi00 x' + Mi01 y' + Mi02) / (Mi20 x' + Mi21 y' + Mi22)            (back-projection with M^-1)
//   loss_l  = sum_{b,s} ((x_gt - x_cal) valid)^2 / sum_{b,s} valid               (0 when nothing is valid)
//   loss    = (1/L) sum_l loss_l ,   dloss/dbeta[b,l,:] alongside (closed form)
//
// Everything is float64 like the reference; one CTA per lane, fixed-order reductions (deterministic), no host sync
// (the reference's `if valid.sum() == 0` becomes a select).  The per-point arithmetic lives in `bp_point()` which is
// __host__ __device__: `lf_backproj_loss_host` runs the same code on the CPU so the CPU test suite can pin the math
// against the oracle (a test hook -- nothing in the product calls it).
//
// This is the training loss of every back-projection step (Loss_crit.fused_backprojection_loss, which
// engine.GraphedTrainStep and engine.train_epoch call); tests/test_net_gpu.py checks it on the GPU against the
// per-lane calls of Loss_crit.backprojection_loss.
#include "lf_common.cuh"

namespace lf {

constexpr int BP_S = 56;        // sample rows (h_samples 160..710 step 10)
constexpr int BP_MAXN = 5;      // order + 1 <= 5
constexpr int BP_THREADS = 256;

struct BpConst {
    double Y[BP_S][BP_MAXN];    // design matrix rows (highest power first)
    double yp[BP_S];            // y' of the sample rows
    double Mi[9];               // M^-1 row-major
};

// one (image, sample) point: squared masked error and d(err^2)/dx' (before the 1/nvalid, 1/L factors)
__host__ __device__ inline void bp_point(const BpConst& c, const double* beta, int n, int s, double xgt, double valid,
                                         double* xcal_out, double* sq_out, double* dsq_dxp_out) {
    double xp = 0.0;
    for (int k = 0; k < n; ++k) xp += c.Y[s][k] * beta[k];
    const double num = c.Mi[0] * xp + (c.Mi[1] * c.yp[s] + c.Mi[2]);
    const double den = c.Mi[6] * xp + (c.Mi[7] * c.yp[s] + c.Mi[8]);
    const double xcal = num / den;
    const double err = (xgt - xcal) * valid;
    *xcal_out = xcal * valid;
    *sq_out = err * err;
    // d err / d xcal = -valid ; d xcal / d xp = (Mi00 den - Mi20 num) / den^2
    const double dxcal_dxp = (c.Mi[0] * den - c.Mi[6] * num) / (den * den);
    *dsq_dxp_out = 2.0 * err * (-valid) * dxcal_dxp;
}

// beta [B][L][n], x_gt / valid [B][L][56]  ->  lane_loss[L], loss[1], dbeta [B][L][n] (gradient of loss), xcal [B][L][56]
__global__ void __launch_bounds__(BP_THREADS) backproj_loss_kernel(const BpConst c, const double* __restrict__ beta,
                                                                    const double* __restrict__ x_gt,
                                                                    const double* __restrict__ valid, int B, int L, int n,
                                                                    double* __restrict__ lane_loss, double* __restrict__ dbeta,
                                                                    double* __restrict__ xcal, unsigned int* ticket,
                                                                    double* __restrict__ loss) {
    pdl_entry();
    __shared__ double red_sq[BP_THREADS], red_nv[BP_THREADS];
    __shared__ double s_scale;
    const int l = blockIdx.x;
    const int tid = threadIdx.x;
    // pass 1: sum of squared errors and of valid over (b, s), fixed assignment of points to threads
    double sq = 0.0, nv = 0.0;
    for (int i = tid; i < B * BP_S; i += BP_THREADS) {
        const int b = i / BP_S, s = i - b * BP_S;
        const size_t o = ((size_t)b * L + l) * BP_S + s;
        double xc, q, dq;
        bp_point(c, beta + ((size_t)b * L + l) * n, n, s, x_gt[o], valid[o], &xc, &q, &dq);
        if (xcal) xcal[o] = xc;
        sq += q;
        nv += valid[o];
    }
    red_sq[tid] = sq;
    red_nv[tid] = nv;
    __syncthreads();
    for (int w = BP_THREADS / 2; w > 0; w >>= 1) {   // fixed tree
        if (tid < w) {
            red_sq[tid] += red_sq[tid + w];
            red_nv[tid] += red_nv[tid + w];
        }
        __syncthreads();
    }
    if (tid == 0) {
        const double nvl = red_nv[0];
        const double denom = nvl == 0.0 ? 1.0 : nvl;
        lane_loss[l] = red_sq[0] / denom;              // 0 when nothing is valid (sum of squares is 0 then)
        s_scale = 1.0 / (denom * (double)L);
    }
    __syncthreads();
    const double scale = s_scale;
    // pass 2: dloss/dbeta[b,l,k] = scale * sum_s dsq/dxp(b,s) * Y[s][k]   (one thread per (b, k))
    if (dbeta) {
        for (int i = tid; i < B * n; i += BP_THREADS) {
            const int b = i / n, k = i - b * n;
            const double* bt = beta + ((size_t)b * L + l) * n;
            double g = 0.0;
            for (int s = 0; s < BP_S; ++s) {
                const size_t o = ((size_t)b * L + l) * BP_S + s;
                double xc, q, dq;
                bp_point(c, bt, n, s, x_gt[o], valid[o], &xc, &q, &dq);
                g += dq * c.Y[s][k];
            }
            dbeta[((size_t)b * L + l) * n + k] = g * scale;
        }
    }
    // last lane CTA to finish sums the lane losses in lane order
    __threadfence();
    __shared__ bool last;
    if (tid == 0) {
        const unsigned int t = atomicAdd(ticket, 1u);
        last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (last && tid == 0) {
        __threadfence();
        double tot = 0.0;
        for (int j = 0; j < L; ++j) tot += ((volatile double*)lane_loss)[j];
        *loss = tot / (double)L;
        *ticket = 0u;   // self-cleaning: ready for the next launch / graph replay
    }
}

static int bp_fill_const(const double* Y56, const double* yprime, const double* Minv, int n, BpConst* c) {
    if (n < 1 || n > BP_MAXN) return LF_ERR_INVALID_ARGUMENT;
    for (int s = 0; s < BP_S; ++s) {
        for (int k = 0; k < BP_MAXN; ++k) c->Y[s][k] = k < n ? Y56[s * n + k] : 0.0;
        c->yp[s] = yprime[s];
    }
    for (int i = 0; i < 9; ++i) c->Mi[i] = Minv[i];
    return LF_OK;
}

}  // namespace lf

using namespace lf;

// Y56 [56][n], yprime [56], Minv [9]: HOST arrays (constants of the loss object, passed by value into the launch).
// beta [B][L][n], x_gt, valid [B][L][56], lane_loss [L], loss [1], dbeta [B][L][n] or NULL, xcal [B][L][56] or NULL,
// ticket: one zero-initialised unsigned int -- all DEVICE.
extern "C" int lf_backproj_loss(const double* Y56, const double* yprime, const double* Minv, const double* beta,
                                const double* x_gt, const double* valid, int B, int L, int n, double* lane_loss, double* loss,
                                double* dbeta, double* xcal, unsigned int* ticket, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(Y56 && yprime && Minv && beta && x_gt && valid && lane_loss && loss && ticket && B > 0 && L > 0 && L <= 65535);
    BpConst c;
    int rc = bp_fill_const(Y56, yprime, Minv, n, &c);
    if (rc) return rc;
    lf_launch(backproj_loss_kernel, L, BP_THREADS, 0, stream, c, beta, x_gt, valid, B, L, n, lane_loss, dbeta, xcal, ticket, loss);
    return check_launch();
}

// TEST HOOK: the same arithmetic (bp_point) on the host, all pointers HOST memory.  Lets `pytest -m "not gpu"` pin the
// kernel's math against the oracle without a GPU; never called by the package.
extern "C" int lf_backproj_loss_host(const double* Y56, const double* yprime, const double* Minv, const double* beta,
                                     const double* x_gt, const double* valid, int B, int L, int n, double* lane_loss,
                                     double* loss, double* dbeta, double* xcal) {
    if (!(Y56 && yprime && Minv && beta && x_gt && valid && lane_loss && loss && B > 0 && L > 0)) return LF_ERR_INVALID_ARGUMENT;
    BpConst c;
    int rc = bp_fill_const(Y56, yprime, Minv, n, &c);
    if (rc) return rc;
    double tot = 0.0;
    for (int l = 0; l < L; ++l) {
        double sq = 0.0, nv = 0.0;
        for (int b = 0; b < B; ++b)
            for (int s = 0; s < BP_S; ++s) {
                const size_t o = ((size_t)b * L + l) * BP_S + s;
                double xc, q, dq;
                bp_point(c, beta + ((size_t)b * L + l) * n, n, s, x_gt[o], valid[o], &xc, &q, &dq);
                if (xcal) xcal[o] = xc;
                sq += q;
                nv += valid[o];
            }
        const double denom = nv == 0.0 ? 1.0 : nv;
        lane_loss[l] = sq / denom;
        tot += lane_loss[l];
        if (dbeta) {
            const double scale = 1.0 / (denom * (double)L);
            for (int b = 0; b < B; ++b)
                for (int k = 0; k < n; ++k) {
                    double g = 0.0;
                    for (int s = 0; s < BP_S; ++s) {
                        const size_t o = ((size_t)b * L + l) * BP_S + s;
                        double xc, q, dq;
                        bp_point(c, beta + ((size_t)b * L + l) * n, n, s, x_gt[o], valid[o], &xc, &q, &dq);
                        g += dq * c.Y[s][k];
                    }
                    dbeta[((size_t)b * L + l) * n + k] = g * scale;
                }
        }
    }
    *loss = tot / (double)L;
    return LF_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// The same loss with its warp constants on the DEVICE (a learned homography, csrc/homography.cu): y'_k of the 56 sample
// rows and M^-1 are read at run time, so a captured graph follows the warp, and the kernel also emits the loss's gradient
// with respect to them: g_const [65] = dloss/dM^-1 (9, row-major) then dloss/dy'_k (56).  Y56 is built from y'_k as the
// reference builds it (rows [y^d .. y 1], y = 255 - y'_k, BP/Loss_crit.py:175-188), so y'_k reaches the loss both
// through the back-projection and through the curve's sample points.
namespace lf {

constexpr int BP_NG = 9 + BP_S;

// row s of the constants from y'_s (and, for s < 9, entry s of M^-1)
__host__ __device__ inline void bp_const_row(const double* yk, const double* Minv, int n, int s, BpConst* c) {
    c->yp[s] = yk[s];
    const double y = 255.0 - yk[s];
    double pw = 1.0;
    for (int k = BP_MAXN - 1; k >= 0; --k) {
        c->Y[s][k] = k < n ? pw : 0.0;
        if (k < n) pw *= y;
    }
    if (s < 9) c->Mi[s] = Minv[s];
}

// one (image, sample) point: adds d(err^2)/dM^-1 to gmi[9] and returns d(err^2)/dy'_s (before the 1/nvalid, 1/L factors)
__host__ __device__ inline double bp_point_const_grad(const BpConst& c, const double* beta, int n, int s, double xgt,
                                                      double valid, double* gmi) {
    double xp = 0.0;
    for (int k = 0; k < n; ++k) xp += c.Y[s][k] * beta[k];
    const double yk = c.yp[s];
    const double num = c.Mi[0] * xp + (c.Mi[1] * yk + c.Mi[2]);
    const double den = c.Mi[6] * xp + (c.Mi[7] * yk + c.Mi[8]);
    const double xcal = num / den;
    const double err = (xgt - xcal) * valid;
    const double id = -2.0 * err * valid / den;      // d(err^2)/dxcal / den
    gmi[0] += id * xp;
    gmi[1] += id * yk;
    gmi[2] += id;
    gmi[6] -= id * xcal * xp;
    gmi[7] -= id * xcal * yk;
    gmi[8] -= id * xcal;
    // dx'/dy of the sampled curve, y = 255 - y'
    const double y = 255.0 - yk;
    double dxp = 0.0, pw = 1.0;
    for (int k = n - 2; k >= 0; --k) {
        dxp += beta[k] * (double)(n - 1 - k) * pw;
        pw *= y;
    }
    return id * ((c.Mi[1] - c.Mi[7] * xcal) - (c.Mi[0] - c.Mi[6] * xcal) * dxp);
}

__global__ void __launch_bounds__(BP_THREADS) backproj_loss_dev_kernel(const double* __restrict__ yk,
                                                                        const double* __restrict__ Minv,
                                                                        const double* __restrict__ beta,
                                                                        const double* __restrict__ x_gt,
                                                                        const double* __restrict__ valid, int B, int L, int n,
                                                                        double* __restrict__ lane_loss,
                                                                        double* __restrict__ dbeta, double* __restrict__ xcal,
                                                                        double* __restrict__ g_part, unsigned int* ticket,
                                                                        double* __restrict__ loss, double* __restrict__ g_const) {
    pdl_entry();
    __shared__ BpConst c;
    __shared__ double red_sq[BP_THREADS], red_nv[BP_THREADS];
    __shared__ double gm[9][BP_S];
    __shared__ double s_scale;
    const int l = blockIdx.x;
    const int tid = threadIdx.x;
    if (tid < BP_S) bp_const_row(yk, Minv, n, tid, &c);
    __syncthreads();
    // pass 1: sum of squared errors and of valid over (b, s), as backproj_loss_kernel
    double sq = 0.0, nv = 0.0;
    for (int i = tid; i < B * BP_S; i += BP_THREADS) {
        const int b = i / BP_S, s = i - b * BP_S;
        const size_t o = ((size_t)b * L + l) * BP_S + s;
        double xc, q, dq;
        bp_point(c, beta + ((size_t)b * L + l) * n, n, s, x_gt[o], valid[o], &xc, &q, &dq);
        if (xcal) xcal[o] = xc;
        sq += q;
        nv += valid[o];
    }
    red_sq[tid] = sq;
    red_nv[tid] = nv;
    __syncthreads();
    for (int w = BP_THREADS / 2; w > 0; w >>= 1) {
        if (tid < w) {
            red_sq[tid] += red_sq[tid + w];
            red_nv[tid] += red_nv[tid + w];
        }
        __syncthreads();
    }
    if (tid == 0) {
        const double denom = red_nv[0] == 0.0 ? 1.0 : red_nv[0];
        lane_loss[l] = red_sq[0] / denom;
        s_scale = 1.0 / (denom * (double)L);
    }
    __syncthreads();
    const double scale = s_scale;
    // pass 2: dloss/dbeta, one thread per (b, k)
    for (int i = tid; i < B * n; i += BP_THREADS) {
        const int b = i / n, k = i - b * n;
        const double* bt = beta + ((size_t)b * L + l) * n;
        double g = 0.0;
        for (int s = 0; s < BP_S; ++s) {
            const size_t o = ((size_t)b * L + l) * BP_S + s;
            double xc, q, dq;
            bp_point(c, bt, n, s, x_gt[o], valid[o], &xc, &q, &dq);
            g += dq * c.Y[s][k];
        }
        dbeta[((size_t)b * L + l) * n + k] = g * scale;
    }
    // pass 3: dloss/dy'_s (thread s, images in order) and dloss/dM^-1 (per-sample partials, summed in sample order)
    if (tid < BP_S) {
        double gmi[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        double gy = 0.0;
        for (int b = 0; b < B; ++b) {
            const size_t o = ((size_t)b * L + l) * BP_S + tid;
            gy += bp_point_const_grad(c, beta + ((size_t)b * L + l) * n, n, tid, x_gt[o], valid[o], gmi);
        }
        g_part[(size_t)l * BP_NG + 9 + tid] = gy * scale;
        for (int i = 0; i < 9; ++i) gm[i][tid] = gmi[i];
    }
    __syncthreads();
    if (tid < 9) {
        double g = 0.0;
        for (int s = 0; s < BP_S; ++s) g += gm[tid][s];
        g_part[(size_t)l * BP_NG + tid] = g * scale;
    }
    // the last lane CTA sums the lane losses and the lanes' constant gradients in lane order
    __threadfence();
    __syncthreads();
    __shared__ bool last;
    if (tid == 0) last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (tid < BP_NG) {
        double g = 0.0;
        for (int j = 0; j < L; ++j) g += __ldcg(g_part + (size_t)j * BP_NG + tid);
        g_const[tid] = g;
    }
    if (tid == 0) {
        double tot = 0.0;
        for (int j = 0; j < L; ++j) tot += __ldcg(lane_loss + j);
        *loss = tot / (double)L;
        *ticket = 0u;
    }
}


// The same loss with one warp per image (a predicted homography, --predict_homography): yk [B][56], Minv [B][9].  Each
// lane CTA first builds the B images' constants into its own slice of `consts` (global scratch, [L][B]); passes 1 and 2
// then run backproj_loss_dev_kernel's thread assignment and per-point code on image b's constants, so with every image
// given the same warp the loss, dbeta and xcal are that kernel's bits.  Pass 3 keeps the constants' gradient per image:
// g_part [L][B][65], and the last CTA sums it over the lanes in lane order into g_const [B][65].
__global__ void __launch_bounds__(BP_THREADS) backproj_loss_pi_kernel(const double* __restrict__ yk,
                                                                       const double* __restrict__ Minv,
                                                                       const double* __restrict__ beta,
                                                                       const double* __restrict__ x_gt,
                                                                       const double* __restrict__ valid, int B, int L, int n,
                                                                       double* __restrict__ lane_loss,
                                                                       double* __restrict__ dbeta, double* __restrict__ xcal,
                                                                       BpConst* __restrict__ consts,
                                                                       double* __restrict__ g_part, unsigned int* ticket,
                                                                       double* __restrict__ loss, double* __restrict__ g_const) {
    pdl_entry();
    __shared__ double red_sq[BP_THREADS], red_nv[BP_THREADS];
    __shared__ double gm[9][BP_S];
    __shared__ double s_scale;
    const int l = blockIdx.x;
    const int tid = threadIdx.x;
    BpConst* cs = consts + (size_t)l * B;
    for (int i = tid; i < B * BP_S; i += BP_THREADS) {
        const int b = i / BP_S, s = i - b * BP_S;
        bp_const_row(yk + (size_t)b * BP_S, Minv + (size_t)b * 9, n, s, cs + b);
    }
    __syncthreads();
    double sq = 0.0, nv = 0.0;
    for (int i = tid; i < B * BP_S; i += BP_THREADS) {
        const int b = i / BP_S, s = i - b * BP_S;
        const size_t o = ((size_t)b * L + l) * BP_S + s;
        double xc, q, dq;
        bp_point(cs[b], beta + ((size_t)b * L + l) * n, n, s, x_gt[o], valid[o], &xc, &q, &dq);
        if (xcal) xcal[o] = xc;
        sq += q;
        nv += valid[o];
    }
    red_sq[tid] = sq;
    red_nv[tid] = nv;
    __syncthreads();
    for (int w = BP_THREADS / 2; w > 0; w >>= 1) {
        if (tid < w) {
            red_sq[tid] += red_sq[tid + w];
            red_nv[tid] += red_nv[tid + w];
        }
        __syncthreads();
    }
    if (tid == 0) {
        const double denom = red_nv[0] == 0.0 ? 1.0 : red_nv[0];
        lane_loss[l] = red_sq[0] / denom;
        s_scale = 1.0 / (denom * (double)L);
    }
    __syncthreads();
    const double scale = s_scale;
    for (int i = tid; i < B * n; i += BP_THREADS) {
        const int b = i / n, k = i - b * n;
        const double* bt = beta + ((size_t)b * L + l) * n;
        double g = 0.0;
        for (int s = 0; s < BP_S; ++s) {
            const size_t o = ((size_t)b * L + l) * BP_S + s;
            double xc, q, dq;
            bp_point(cs[b], bt, n, s, x_gt[o], valid[o], &xc, &q, &dq);
            g += dq * cs[b].Y[s][k];
        }
        dbeta[((size_t)b * L + l) * n + k] = g * scale;
    }
    // pass 3, image by image: dloss/dy'_s on thread s, dloss/dM^-1 summed over the samples in order
    for (int b = 0; b < B; ++b) {
        double* gp = g_part + ((size_t)l * B + b) * BP_NG;
        if (tid < BP_S) {
            double gmi[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
            const size_t o = ((size_t)b * L + l) * BP_S + tid;
            const double gy = bp_point_const_grad(cs[b], beta + ((size_t)b * L + l) * n, n, tid, x_gt[o], valid[o], gmi);
            gp[9 + tid] = gy * scale;
            for (int i = 0; i < 9; ++i) gm[i][tid] = gmi[i];
        }
        __syncthreads();
        if (tid < 9) {
            double g = 0.0;
            for (int s = 0; s < BP_S; ++s) g += gm[tid][s];
            gp[tid] = g * scale;
        }
        __syncthreads();
    }
    __threadfence();
    __syncthreads();
    __shared__ bool last;
    if (tid == 0) last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    for (int i = tid; i < B * BP_NG; i += BP_THREADS) {
        double g = 0.0;
        for (int j = 0; j < L; ++j) g += __ldcg(g_part + (size_t)j * B * BP_NG + i);
        g_const[i] = g;
    }
    if (tid == 0) {
        double tot = 0.0;
        for (int j = 0; j < L; ++j) tot += __ldcg(lane_loss + j);
        *loss = tot / (double)L;
        *ticket = 0u;
    }
}

}  // namespace lf

// yk [56], Minv [9]: DEVICE constants; beta, x_gt, valid, lane_loss, loss, dbeta, xcal (or NULL), ticket as
// lf_backproj_loss; g_part [L][65] scratch (the per-lane gradients, scaled like dbeta), g_const [65] -- all DEVICE.
extern "C" int lf_backproj_loss_dev(const double* yk, const double* Minv, const double* beta, const double* x_gt,
                                    const double* valid, int B, int L, int n, double* lane_loss, double* loss, double* dbeta,
                                    double* xcal, double* g_part, double* g_const, unsigned int* ticket, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(yk && Minv && beta && x_gt && valid && lane_loss && loss && dbeta && g_part && g_const && ticket);
    LF_REQUIRE(B > 0 && L > 0 && L <= 65535 && n >= 1 && n <= BP_MAXN);
    lf_launch(backproj_loss_dev_kernel, L, BP_THREADS, 0, stream, yk, Minv, beta, x_gt, valid, B, L, n, lane_loss, dbeta, xcal,
              g_part, ticket, loss, g_const);
    return check_launch();
}

// Scratch doubles lf_backproj_loss_per_image needs for B images and L lanes: the per-lane constants and gradients.
extern "C" size_t lf_backproj_loss_per_image_scratch(int B, int L) {
    if (B <= 0 || L <= 0) return 0;
    return (size_t)L * B * (sizeof(BpConst) / sizeof(double) + BP_NG);
}

// lf_backproj_loss_dev with one warp per image: yk [B][56], Minv [B][9]; g_const [B][65] = each image's dloss/dM^-1 (9)
// then dloss/dy'_k (56); scratch: lf_backproj_loss_per_image_scratch(B, L) doubles -- all DEVICE.
extern "C" int lf_backproj_loss_per_image(const double* yk, const double* Minv, const double* beta, const double* x_gt,
                                          const double* valid, int B, int L, int n, double* lane_loss, double* loss,
                                          double* dbeta, double* xcal, double* scratch, double* g_const,
                                          unsigned int* ticket, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(yk && Minv && beta && x_gt && valid && lane_loss && loss && dbeta && scratch && g_const && ticket);
    LF_REQUIRE(B > 0 && L > 0 && L <= 65535 && n >= 1 && n <= BP_MAXN);
    LF_REQUIRE((reinterpret_cast<uintptr_t>(scratch) & 7) == 0);
    BpConst* consts = reinterpret_cast<BpConst*>(scratch);
    double* g_part = scratch + (size_t)L * B * (sizeof(BpConst) / sizeof(double));
    lf_launch(backproj_loss_pi_kernel, L, BP_THREADS, 0, stream, yk, Minv, beta, x_gt, valid, B, L, n, lane_loss, dbeta,
              xcal, consts, g_part, ticket, loss, g_const);
    return check_launch();
}

// TEST HOOK: lf_backproj_loss_dev's arithmetic on HOST arrays (g_const [65] may be NULL); never called by the package.
extern "C" int lf_backproj_loss_dev_host(const double* yk, const double* Minv, const double* beta, const double* x_gt,
                                         const double* valid, int B, int L, int n, double* lane_loss, double* loss,
                                         double* dbeta, double* xcal, double* g_const) {
    if (!(yk && Minv && beta && x_gt && valid && lane_loss && loss && B > 0 && L > 0 && n >= 1 && n <= BP_MAXN))
        return LF_ERR_INVALID_ARGUMENT;
    BpConst c;
    for (int s = 0; s < BP_S; ++s) bp_const_row(yk, Minv, n, s, &c);
    double Y56[BP_S * BP_MAXN];
    for (int s = 0; s < BP_S; ++s)
        for (int k = 0; k < n; ++k) Y56[s * n + k] = c.Y[s][k];
    const int rc = lf_backproj_loss_host(Y56, c.yp, c.Mi, beta, x_gt, valid, B, L, n, lane_loss, loss, dbeta, xcal);
    if (rc || !g_const) return rc;
    for (int i = 0; i < BP_NG; ++i) g_const[i] = 0.0;
    for (int l = 0; l < L; ++l) {
        double nv = 0.0;
        for (int b = 0; b < B; ++b)
            for (int s = 0; s < BP_S; ++s) nv += valid[((size_t)b * L + l) * BP_S + s];
        const double scale = 1.0 / ((nv == 0.0 ? 1.0 : nv) * (double)L);
        double gm[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int s = 0; s < BP_S; ++s) {
            double gy = 0.0;
            for (int b = 0; b < B; ++b) {
                const size_t o = ((size_t)b * L + l) * BP_S + s;
                gy += bp_point_const_grad(c, beta + ((size_t)b * L + l) * n, n, s, x_gt[o], valid[o], gm);
            }
            g_const[9 + s] += gy * scale;
        }
        for (int i = 0; i < 9; ++i) g_const[i] += gm[i] * scale;
    }
    return LF_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Area loss of the bird's-eye-view experiment over all lanes, its gradient and the exact-area metric in one launch:
// Birds_Eye_View_Loss/Loss_crit.py:98-134 (`Area_Loss`, order 2) summed over the lanes as BEV/main.py:223,237 does, and
// `polynomial.trapezoidal` (:12-35) as BEV/main.py:273-280 / :436-442 evaluates it.
//
//   d       = beta[b][l] - params[b][l]                    (a, b, c in float64 from the float32 inputs)
//   f(d)    = int_0^0.7 W(y) (a y^2 + b y + c)^2 dy = sum_ij Q_ij d_i d_j,   Q_ij = int_0^0.7 W(y) y^(p_i + p_j) dy
//   loss    = sum_l (1 / n_l) sum_{b present in l} f(d)    (n_l images whose three ground-truth coefficients are non-zero;
//                                                            a lane with none contributes 0)
//   dbeta   = present ? 2 (Q d) / n_l : 0
//   exact_b = (trap(beta_0, gt_0) + trap(beta_1, gt_1)) / 2 in the reference's float32 arithmetic, op for op
//
// The quadratic form holds the reference's three closed forms (none, linear, quadratic) term by term.  float64 terms,
// sums in a fixed order (thread t takes images t, t + T, ...; then a fixed tree), one rounding to float32 at the end.
// `lf_area_loss_host` replays the same per-image code and the same summation order on host arrays (a test hook); the
// explicit round-to-nearest intrinsics keep nvcc from contracting a multiply and an add into one FMA, which the host
// code does not do, so both give the same bits.
namespace lf {

constexpr int AREA_THREADS = 128;
constexpr int AREA_STEPS = 100;     // polynomial(..., n=100)
constexpr int AREA_MAXL = 4;

struct AreaConst {
    double Q[3][3];                 // moments of the weight function (a, b, c order: powers 2, 1, 0)
    float x[AREA_STEPS + 1];        // float32(x_i), x_i = i * h as Python computes it; x_100 = 0.7 (self.b)
    float x2[AREA_STEPS + 1];       // float32(x_i ** 2)
    float h;                        // float32(0.7 / 100)
};

__host__ __device__ inline float area_fmul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}

__host__ __device__ inline float area_fadd(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

__host__ __device__ inline double area_dmul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

__host__ __device__ inline double area_dadd(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

__host__ __device__ inline float area_fsub(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}

// polynomial.calc_pol: (a1 * x**2 + b1 * x) + c1, every op rounded to float32
__host__ __device__ inline float area_pol(const float* p, float x2, float x) {
    return area_fadd(area_fadd(area_fmul(p[0], x2), area_fmul(p[1], x)), p[2]);
}

// polynomial(pred).trapezoidal(polynomial(gt)) of one image
__host__ __device__ inline float area_trap(const AreaConst& c, const float* pred, const float* gt) {
    float s = fabsf(area_fsub(area_fmul(area_pol(pred, c.x2[0], c.x[0]), 0.5f), area_fmul(area_pol(gt, c.x2[0], c.x[0]), 0.5f)));
    for (int i = 1; i < AREA_STEPS; ++i)
        s = area_fadd(s, fabsf(area_fsub(area_pol(pred, c.x2[i], c.x[i]), area_pol(gt, c.x2[i], c.x[i]))));
    const int e = AREA_STEPS;
    s = area_fadd(s, fabsf(area_fsub(area_fmul(area_pol(pred, c.x2[e], c.x[e]), 0.5f), area_fmul(area_pol(gt, c.x2[e], c.x[e]), 0.5f))));
    return area_fmul(s, c.h);
}

// one (image, lane): present flag, f(d) and Q d
__host__ __device__ inline bool area_term(const AreaConst& c, const float* beta, const float* gt, double* f, double qd[3]) {
    const double d[3] = {(double)beta[0] - (double)gt[0], (double)beta[1] - (double)gt[1], (double)beta[2] - (double)gt[2]};
    double s = 0.0;
    for (int i = 0; i < 3; ++i) {
        qd[i] = area_dadd(area_dadd(area_dmul(c.Q[i][0], d[0]), area_dmul(c.Q[i][1], d[1])), area_dmul(c.Q[i][2], d[2]));
        s = area_dadd(s, area_dmul(d[i], qd[i]));
    }
    *f = s;
    return gt[0] != 0.0f && gt[1] != 0.0f && gt[2] != 0.0f;
}

// per-"thread" partial sums of one image: lane sums, lane counts, exact value (slot 2 * AREA_MAXL)
__host__ __device__ inline void area_accumulate(const AreaConst& c, const float* beta, const float* params, int b, int L,
                                                bool want_exact, double acc[2 * AREA_MAXL + 1], float* exact) {
#pragma unroll
    for (int l = 0; l < AREA_MAXL; ++l) {      // constant indices: acc stays in registers
        double f, qd[3];
        if (l < L && area_term(c, beta + ((size_t)b * L + l) * 3, params + ((size_t)b * 4 + l) * 3, &f, qd)) {
            acc[l] += f;
            acc[AREA_MAXL + l] += 1.0;
        }
    }
    if (want_exact) {
        const float tl = area_trap(c, beta + (size_t)b * L * 3, params + (size_t)b * 12);
        const float tr = area_trap(c, beta + ((size_t)b * L + 1) * 3, params + ((size_t)b * 4 + 1) * 3);
        const float e = area_fmul(area_fadd(tl, tr), 0.5f);
        if (exact) exact[b] = e;
        acc[2 * AREA_MAXL] += (double)e;
    }
}

__host__ __device__ inline void area_gradient(const AreaConst& c, const float* beta, const float* params, int b, int L,
                                              const double* inv_n, float* dbeta) {
#pragma unroll
    for (int l = 0; l < AREA_MAXL; ++l) {
        if (l >= L) break;
        double f, qd[3];
        const bool present = area_term(c, beta + ((size_t)b * L + l) * 3, params + ((size_t)b * 4 + l) * 3, &f, qd);
        for (int k = 0; k < 3; ++k) dbeta[((size_t)b * L + l) * 3 + k] = present ? (float)area_dmul(area_dmul(2.0, qd[k]), inv_n[l]) : 0.0f;
    }
}

// loss from the reduced sums; fills inv_n (0 for a lane without images)
__host__ __device__ inline float area_finish(const double* acc, int L, double* inv_n) {
    double loss = 0.0;
#pragma unroll
    for (int l = 0; l < AREA_MAXL; ++l) {
        if (l >= L) {
            inv_n[l] = 0.0;
            continue;
        }
        const double n = acc[AREA_MAXL + l];
        inv_n[l] = n == 0.0 ? 0.0 : 1.0 / n;
        loss = area_dadd(loss, area_dmul(acc[l], inv_n[l]));
    }
    return (float)loss;
}

__global__ void __launch_bounds__(AREA_THREADS) area_loss_kernel(const AreaConst c, const float* __restrict__ beta,
                                                                  const float* __restrict__ params, int B, int L,
                                                                  float* __restrict__ loss, float* __restrict__ dbeta,
                                                                  float* __restrict__ exact, float* __restrict__ exact_mean) {
    pdl_entry();
    constexpr int NA = 2 * AREA_MAXL + 1;
    __shared__ double red[NA][AREA_THREADS];
    __shared__ double s_inv_n[AREA_MAXL];
    const int tid = threadIdx.x;
    const bool want_exact = exact || exact_mean;
    double acc[NA];
#pragma unroll
    for (int j = 0; j < NA; ++j) acc[j] = 0.0;
    for (int b = tid; b < B; b += AREA_THREADS) area_accumulate(c, beta, params, b, L, want_exact, acc, exact);
#pragma unroll
    for (int j = 0; j < NA; ++j) red[j][tid] = acc[j];
    __syncthreads();
    for (int w = AREA_THREADS / 2; w > 0; w >>= 1) {     // fixed tree
        if (tid < w) {
#pragma unroll
            for (int j = 0; j < NA; ++j) red[j][tid] += red[j][tid + w];
        }
        __syncthreads();
    }
    if (tid == 0) {
        double tot[NA], inv_n[AREA_MAXL];
#pragma unroll
        for (int j = 0; j < NA; ++j) tot[j] = red[j][0];
        const float l = area_finish(tot, L, inv_n);
        if (loss) *loss = l;
        if (exact_mean) *exact_mean = (float)(tot[2 * AREA_MAXL] / (double)B);
#pragma unroll
        for (int j = 0; j < AREA_MAXL; ++j) s_inv_n[j] = inv_n[j];
    }
    __syncthreads();
    if (dbeta)
        for (int b = tid; b < B; b += AREA_THREADS) area_gradient(c, beta, params, b, L, s_inv_n, dbeta);
}

static int area_fill_const(int weight, AreaConst* c) {
    // moments M_k = int_0^t W(y) y^k dy, t = 0.7, of W = 1 (0), 1 - y (1), 1 - sqrt(y) (2)
    const double t = 0.7;
    double M[5];
    for (int k = 0; k <= 4; ++k) {
        M[k] = pow(t, k + 1.0) / (k + 1.0);
        if (weight == 1) M[k] -= pow(t, k + 2.0) / (k + 2.0);
        else if (weight == 2) M[k] -= pow(t, k + 1.5) / (k + 1.5);
        else if (weight != 0) return LF_ERR_INVALID_ARGUMENT;
    }
    const int p[3] = {2, 1, 0};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c->Q[i][j] = M[p[i] + p[j]];
    // polynomial(..., a=0, b=0.7, n=100): h = 0.7 / 100, x_i = 0 + i*h in Python doubles, x ** 2 through libm's pow as
    // Python's float power does; torch rounds each Python scalar to float32 against a float32 tensor
    const double h = 0.7 / AREA_STEPS;
    for (int i = 0; i <= AREA_STEPS; ++i) {
        const double x = i == AREA_STEPS ? 0.7 : (double)i * h;
        c->x[i] = (float)x;
        c->x2[i] = (float)pow(x, 2.0);
    }
    c->h = (float)h;
    return LF_OK;
}

}  // namespace lf

// beta [B][L][3], params [B][4][3] float32: DEVICE; weight 0 none / 1 linear / 2 quadratic; outputs DEVICE, each optional.
extern "C" int lf_area_loss(const float* beta, const float* params, int B, int L, int weight, float* loss, float* dbeta,
                            float* exact, float* exact_mean, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(beta && params && B > 0 && (L == 2 || L == 4));
    AreaConst c;
    int rc = area_fill_const(weight, &c);
    if (rc) return rc;
    lf_launch(area_loss_kernel, 1, AREA_THREADS, 0, stream, c, beta, params, B, L, loss, dbeta, exact, exact_mean);
    return check_launch();
}

// TEST HOOK: the kernel's per-image code and summation order on HOST arrays; never called by the package.
extern "C" int lf_area_loss_host(const float* beta, const float* params, int B, int L, int weight, float* loss, float* dbeta,
                                 float* exact, float* exact_mean) {
    if (!(beta && params && B > 0 && (L == 2 || L == 4))) return LF_ERR_INVALID_ARGUMENT;
    AreaConst c;
    int rc = area_fill_const(weight, &c);
    if (rc) return rc;
    constexpr int NA = 2 * AREA_MAXL + 1;
    static thread_local double red[NA][AREA_THREADS];
    const bool want_exact = exact || exact_mean;
    for (int t = 0; t < AREA_THREADS; ++t) {
        double acc[NA] = {0.0};
        for (int b = t; b < B; b += AREA_THREADS) area_accumulate(c, beta, params, b, L, want_exact, acc, exact);
        for (int j = 0; j < NA; ++j) red[j][t] = acc[j];
    }
    for (int w = AREA_THREADS / 2; w > 0; w >>= 1)
        for (int t = 0; t < w; ++t)
            for (int j = 0; j < NA; ++j) red[j][t] += red[j][t + w];
    double tot[NA], inv_n[AREA_MAXL];
    for (int j = 0; j < NA; ++j) tot[j] = red[j][0];
    const float l = area_finish(tot, L, inv_n);
    if (loss) *loss = l;
    if (exact_mean) *exact_mean = (float)(tot[2 * AREA_MAXL] / (double)B);
    if (dbeta)
        for (int b = 0; b < B; ++b) area_gradient(c, beta, params, b, L, inv_n, dbeta);
    return LF_OK;
}
