/*
 * lanefit_b200.h -- C ABI of the H100-native (sm_90a) hot path of
 * wvangansbeke/LaneDetection_End2End.
 *
 * The reference is pure Python/PyTorch and has NO FFI of its own (SURVEY.md 8b);
 * the entry points below are what a binding for its hot path would bind.  Each
 * one names the reference code it replaces (paths relative to the reference
 * root, BP = Backprojection_Loss).  INTEGRATION.md shows the ctypes stub a
 * maintainer would add on the reference side.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless noted; the caller owns all memory,
 *     the library never allocates or frees user-visible buffers;
 *   - every call is asynchronous on `stream` and never synchronises it;
 *   - return value: 0 = LF_OK, negative = LF_ERR_* (argument / launch errors,
 *     detected on the host before or at launch);
 *   - numerical failures (singular normal equations) are reported through a
 *     device-side `status` word the caller reads when it chooses to;
 *   - feature maps are NHWC ("channels_last") fp32 unless a dtype argument says
 *     otherwise; lane weight maps are planar [B, L, H, W].
 */
#ifndef LANEFIT_B200_H
#define LANEFIT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* lf_stream_t; /* == cudaStream_t */

#define LF_OK 0
#define LF_ERR_INVALID_ARGUMENT (-1)
#define LF_ERR_UNSUPPORTED (-2)
#define LF_ERR_WORKSPACE_TOO_SMALL (-3)
#define LF_ERR_CUDA (-4)

/* element types */
#define LF_F32 0
#define LF_BF16 1

/* activation applied to the decoder output before the fit (BP/Networks/LSQ_layer.py:27-47) */
#define LF_ACT_NONE 0
#define LF_ACT_SQUARE 1
#define LF_ACT_ABS 2
#define LF_ACT_RELU 3
#define LF_ACT_SIGMOID 4
#define LF_ACT_SOFTPLUS 5

/* normal-equation solver (BP/Networks/LSQ_layer.py:112-118) */
#define LF_SOLVER_INVERSE 0  /* torch.inverse + bmm  (:114-116): LU, partial pivoting  */
#define LF_SOLVER_CHOLESKY 1 /* GELS                 (BP/Networks/gels.py:11-15)       */

/* bits of the device status word written by lf_lsq_fwd */
#define LF_STATUS_SINGULAR 1    /* zero pivot: torch.inverse would raise (BP/main.py:289-292) */
#define LF_STATUS_NONFINITE 2   /* NaN/Inf in the moments or in beta                         */
#define LF_STATUS_NOT_POSDEF 4  /* Cholesky pivot <= 0: torch.cholesky would raise           */

#define LF_MAX_ORDER 4

int lf_version(void);
/* Programmatic dependent launch of the library's kernels (default off; LANEFIT_PDL=1 or lf_set_pdl(1) enables): each kernel
 * may then be scheduled while its predecessor in the stream drains, and waits (griddepcontrol.wait) before touching global
 * memory.  Measured neutral on the graph-replayed training step (DESIGN.md). */
void lf_set_pdl(int on);
int lf_get_pdl(void);
const char* lf_error_string(int code);
/* last CUDA error string seen by the library on this thread (host pointer) */
const char* lf_last_cuda_error(void);

/* ------------------------------------------------------------------------- *
 * Weighted least-squares layer, forward.
 * Replaces, fused into one launch: square_tensor / activation_layer
 * (BP/Networks/LSQ_layer.py:19-20,27-47,295), the row mask index_fill (:237-238,301)
 * and Weighted_least_squares.forward (:85-154), incl. the GELS variant
 * (BP/Networks/gels.py:11-15); BEV variant: Birds_Eye_View_Loss/Networks/LSQ_layer.py:90-167.
 *
 *   o        [B,L,H,W]  raw decoder output (o_dtype LF_F32 | LF_BF16)
 *   xtab     [H*W] f32  grid[:,0]                      (BEV x coordinate of every pixel)
 *   ytab     [H*W] f32  const - grid[:,1]              (:94, const = 255 BP / 1 BEV)
 *   yrow     [H]   f32  ytab of each row if ytab is constant along rows (true for every
 *                       homography the reference builds), else NULL -> general kernel
 *   mask_rows           rows [0,mask_rows) get weight zero and are never read
 *   beta     [B,L,order+1] f64 out, highest power first (:100-104)
 *   zinv     [B,L,(order+1)^2] f64 out: (Y^T W^2 Y + reg I)^-1, consumed by lf_lsq_bwd
 *   masked   [B,L,H,W] f32 out or NULL: activation(o) with masked rows zeroed (output #5
 *            of Net.forward, :315)
 *   status   int32 out: OR of LF_STATUS_* over all B*L systems (caller zeroes it)
 *   workspace: lf_lsq_workspace_bytes() bytes, ZEROED once before first use; the
 *            library leaves it reusable (tickets reset) after every launch.
 * ------------------------------------------------------------------------- */
size_t lf_lsq_workspace_bytes(int B, int L, int H, int W, int order);
int lf_lsq_fwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
               int B, int L, int H, int W, int order, int mask_rows, int act, double reg_ls, int solver,
               double* beta, double* zinv, float* masked, int* status,
               void* workspace, size_t workspace_bytes, lf_stream_t stream);

/* Backward of the above: d_o = dL/d o given gbeta = dL/d beta [B,L,order+1] f64.
 * Replaces autograd through mul/bmm/inverse (BP/Networks/LSQ_layer.py:111-116) ==
 * GELS.backward (BP/Networks/gels.py:18-25) composed with the activation and mask:
 *   z = Z^-1 g ;  d_o = mask * act'(o) * 2 act(o) * (x - phi^T beta) * (phi^T z).
 * d_o has the dtype of o. */
int lf_lsq_bwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
               int B, int L, int H, int W, int order, int mask_rows, int act,
               const double* beta, const double* zinv, const double* gbeta,
               void* d_o, lf_stream_t stream);

/* ========================================================================= *
 * ERFNet encoder/decoder building blocks (BP/Networks/ERFNet.py:11-176).
 * Feature maps are NHWC fp32: element (n,y,x,c) at ((n*H+y)*W+x)*cstride + coff + c.
 * The reference modules are assembled from these calls by
 * lanedetection_end2end_b200/ops_net.py (one autograd Function per reference block).
 * ========================================================================= */
#define LF_MAX_TAPS 9

/* Generic implicit-GEMM convolution, one output phase per call:
 *   out[n, j*osy+oy0, i*osx+ox0, out_coff+co] =
 *     epi( sum_t sum_ci in[n, j*isy+dy[t], i*isx+dx[t], ci] * wmat[(wtap[t]*Cin+ci)*CoutPad + co] )
 * for n<N, j<Hs, i<Ws, co<Cout, zero outside the input.  Covers Conv2d forward (any stride,
 * padding, dilation: ERFNet.py:15,29-37), ConvTranspose2d forward as 4 phases (:101), and both
 * input gradients.  epi: +bias, ReLU, *(mask_src>0), +add_src*(add_mask>0); mask/add tensors
 * share the output layout. */
typedef struct LfConvArgs {
    const float* in;
    const float* wmat;      /* [ntap_slots][Cin][CoutPad] packed GEMM weights */
    const float* bias;      /* [Cout] or NULL */
    float* out;
    const float* mask_src;  /* NULL or forward activation whose sign gates the result */
    const float* add_src;   /* NULL or tensor added to the result ... */
    const float* add_mask;  /* ... gated by (add_mask > 0) when non-NULL */
    int N, Hin, Win, Cin, in_cstride;
    int Hout, Wout, out_cstride, out_coff, Cout, CoutPad;
    int Hs, Ws, osy, osx, oy0, ox0, isy, isx;
    int ntaps;
    int dy[LF_MAX_TAPS], dx[LF_MAX_TAPS], wtap[LF_MAX_TAPS];
    int relu;
} LfConvArgs;
int lf_conv_f32(const LfConvArgs* args, lf_stream_t stream);

/* Tensor-core (wgmma; TF32 in, fp32 accumulate) implementation of the factorised 3-tap convolutions of
 * non_bottleneck_1d (BP/Networks/ERFNet.py:29-37) and their input gradients, for dense NHWC fp32
 * tensors with C in {64,128} channels in and out:
 *   out[n,y,x,co] = epi( sum_{t<3} sum_ci in[n, y+dy[t], x+dx[t], ci] * wpack[co*3*C + t*C + ci] )
 * epi as in LfConvArgs.  Requires a bx*by = 128 pixel patch with bx | W, by | H
 * (lf_conv1d_tc_supported tells).  Same results as lf_conv_f32 up to TF32 rounding of the operands. */
typedef struct LfConvTcArgs {
    const float* in;
    const float* wpack;    /* [C][3*C], K contiguous */
    const float* bias;     /* [C] or NULL */
    float* out;
    const float* mask_src;
    const float* add_src;
    const float* add_mask;
    float* colsum_partial; /* NULL, or [lf_conv1d_tc_supported(...)][C]: per-CTA column sums of `out`
                              (the bias gradient when `out` is an output gradient); reduce with lf_vec_reduce */
    double* stats_partial; /* NULL, or [lf_conv1d_tc_supported(...)][2][C]: per-CTA sum and sum of squares of `out`
                              = the `partial` input of lf_bn_finalize (replaces an lf_bn_stats pass over `out`);
                              LF_ERR_UNSUPPORTED when the launch has to use the per-tap variant */
    const float* mask_scale; /* NULL, or [C] together with mask_shift [C] (needs mask_src and stats_partial): mask_src is then
                              a PRE-activation x, the ReLU-backward mask bit is fma(x, mask_scale[c], mask_shift[c]) > 0
                              (bit-identical to the forward's relu(bn(x)) when scale / shift are lf_bn_finalize's), and the
                              second statistic becomes sum(out * x) instead of sum(out^2): the launch that produces the
                              gradient w.r.t. relu(bn(x)) also delivers BatchNorm backward's two reductions
                              (lf_bn_bwd_finalize_sx) without a pass over (g, x) -- and without reading relu(bn(x)). */
    const float* mask_shift;
    int N, H, W, C;
    int dy[3], dx[3];
    int relu;                /* bit 0: ReLU on conv + bias (before mask / add_src); bit 1: ReLU after add_src -- the closing
                                relu(conv + x) of an eval-mode block whose BatchNorm is folded into the weights */
    int in_dtype, out_dtype, mask_dtype; /* element types of `in`, `out` and `mask_src`: LF_F32 (0, every pointer above
                                typed float), or LF_BF16 -- lf_conv1d_tc_bf16 only, else LF_ERR_UNSUPPORTED.  A bf16 `in`
                                gives the same results as its fp32 copy (the kernel rounds fp32 activations to bf16 itself);
                                a bf16 `out` is the fp32 result rounded to nearest even (colsum / stats are of the fp32
                                values); a bf16 `mask_src` gates like its fp32 copy.  Same shapes and slab cases as fp32. */
} LfConvTcArgs;
/* Arguments of lf_conv1d_tc_fp8: the LfConvTcArgs of the launch (unchanged layout) followed by the fp8 scales. */
typedef struct LfConvTcFp8Args {
    LfConvTcArgs conv;
    const float* x_amax;     /* [N] per-image max |in| over the stored input values (the activation scale) */
    const float* w_scale;    /* [C] per-output-channel dequantisation factors of the e4m3 `wpack` (a_w / 448) */
    float* out_amax;         /* [N] per-image max |out| of the stored values, reduced with atomicMax on the float bits:
                                the caller zeroes it; it is the `x_amax` of the next convolution */
} LfConvTcFp8Args;
/* 0 = unsupported shape, else the number of CTA rows of colsum_partial */
int lf_conv1d_tc_supported(int N, int H, int W, int C);
/* 3xTF32 variant (csrc/conv_tc.cu): same arguments and epilogue, but `wpack` is the pre-split operand
 * [2][C][3*C] (TF32 hi parts, then lo parts: LF_PACK_TF32_HI / _LO) and every product is formed as
 * a_hi*w_hi + (a_hi*w_lo + a_lo*w_hi) with fp32 accumulation -- results agree with lf_conv_f32 to fp32 round-off
 * (the arithmetic the reference's fp32 Conv2d performs, BP/Networks/ERFNet.py:29-37) while running on tensor cores.
 * lf_conv1d_tc_x3_rows: 0 if a call with taps {-dil,0,+dil} along y (vertical) or x is not served, else the number of
 * rows of colsum_partial / stats_partial.  Unsupported shapes return LF_ERR_UNSUPPORTED (no fallback inside). */
int lf_conv1d_tc_x3_rows(int N, int H, int W, int C, int vertical, int dil);
int lf_conv1d_tc_x3(const LfConvTcArgs* args, lf_stream_t stream);
int lf_conv1d_tc(const LfConvTcArgs* args, lf_stream_t stream);
/* BF16 variant: same arguments and epilogue, but `wpack` points at a [C][3*C] bf16 operand (LfPackJob.dst_dtype =
 * LF_BF16) and the activations are rounded to bf16 (nearest even) in the kernel; products are exact in fp32, fp32
 * accumulate.  It serves exactly the shapes of lf_conv1d_tc and runs on the slab kernel exactly where lf_conv1d_tc does,
 * so lf_conv1d_tc_supported and lf_conv1d_tc_slab_ok answer for it. */
int lf_conv1d_tc_bf16(const LfConvTcArgs* args, lf_stream_t stream);
/* FP8 variant (inference only): conv.wpack is a [C][3*C] e4m3 operand quantised per output channel (w_scale), the
 * activations (fp32, or bf16 with in_dtype = LF_BF16) are quantised per image in the kernel: q = e4m3(v * (448 /
 * x_amax[n])), round to nearest even with saturation (0 when x_amax[n] = 0).  Each tap's products of one 32-channel
 * chunk are summed from zero by the tensor core and added to the fp32 sum; then
 *   out = epi( acc * ((x_amax[n] / 448) * w_scale[co]) + bias )     (each operation rounded to nearest in fp32)
 * and out_amax[n] receives the per-image max |stored out|.  x_amax, w_scale and out_amax are required; colsum_partial,
 * stats_partial and mask_scale are not taken.  Same shapes and slab cases as lf_conv1d_tc. */
int lf_conv1d_tc_fp8(const LfConvTcFp8Args* args, lf_stream_t stream);
/* amax[n] = max(amax[n], max |x[n, ...]|) over the `per_image` elements of each of the N images of x (fp32, or bf16
 * with dtype = LF_BF16), by atomicMax on the float bits: zero amax first for the plain per-image max. */
int lf_amax_per_image(const void* x, int dtype, long long per_image, int N, float* amax, lf_stream_t stream);
/* 2 (default) = halo-slab kernel (one TMA slab per 32-channel chunk shared by the three taps);
 * 1 = first version (one TMA box per tap).  Same results; process-wide switch for A/B measurements. */
void lf_conv1d_tc_set_variant(int variant);
/* 1 if a call with taps {-dil,0,+dil} along y (vertical) or x runs on the slab kernel, i.e. may ask for stats_partial */
int lf_conv1d_tc_slab_ok(int N, int H, int W, int C, int vertical, int dil);

/* Tensor-core weight gradient of the same 3-tap convolutions:
 *   partial[cta][t][ci][co] = sum over this CTA's pixel range of x[n,y+dy[t],x+dx[t],ci] * dy[n,y,x,co]
 * nctas = lf_wgrad3_tc_ctas(...) (0 = unsupported shape); finish with
 * lf_wgrad_reduce(partial, nctas, 3, C, C, C, C, dst, st, sp, sq). */
int lf_wgrad3_tc_ctas(int N, int H, int W, int C);
int lf_wgrad3_tc(const float* x, const float* dy, int N, int H, int W, int C, const int* tap_dy, const int* tap_dx,
                 float* partial, int nctas, lf_stream_t stream);
/* 3xTF32 variant (csrc/wgrad_tcg.cu): same arguments and partial layout; both operands are split into TF32 hi / lo
 * parts on the fly and every product is x_hi*g_hi + (x_hi*g_lo + x_lo*g_hi), fp32 accumulate -- results agree with
 * lf_wgrad_f32 to fp32 round-off (the weight gradient the reference's autograd forms in fp32). */
int lf_wgrad3_tc_x3_ctas(int N, int H, int W, int C);
int lf_wgrad3_tc_x3(const float* x, const float* dy, int N, int H, int W, int C, const int* tap_dy, const int* tap_dx,
                    float* partial, int nctas, lf_stream_t stream);
/* BF16 variant: same arguments and partial layout; both operands rounded to bf16 (nearest even) in the kernel, fp32
 * accumulate. */
int lf_wgrad3_tc_bf16_ctas(int N, int H, int W, int C);
int lf_wgrad3_tc_bf16(const float* x, const float* dy, int N, int H, int W, int C, const int* tap_dy, const int* tap_dx,
                      float* partial, int nctas, lf_stream_t stream);
/* lf_wgrad3_tc_bf16 with the layer input x stored as bf16 [N,H,W,C] (dy stays fp32): same results as lf_wgrad3_tc_bf16
 * on the fp32 copy of x, same arguments, nctas (lf_wgrad3_tc_bf16_ctas) and partial layout. */
int lf_wgrad3_tc_bf16a(const void* x, const float* dy, int N, int H, int W, int C, const int* tap_dy, const int* tap_dx,
                       float* partial, int nctas, lf_stream_t stream);

/* Weight gradient as a split-K GEMM over pixels:
 *   partial[s][t][cp][cq] = sum_{(n,j,i) in split s} P[n, j*psy+pdy[t], i*psx+pdx[t], cp]
 *                                                  * Q[n, j*qsy+qdy[t], i*qsx+qdx[t], cq]
 * Conv2d: P = layer input (gathered), Q = output gradient (dense); ConvTranspose2d: P = layer
 * input (dense), Q = output gradient (gathered).  qsum_partial (optional) receives the column
 * sums of Q over the domain (bias gradient when Q is dense).  lf_wgrad_reduce sums the splits in
 * fixed order into dst[t*st + cp*sp + cq*sq] (any weight layout). */
typedef struct LfWgradArgs {
    const float* P;
    const float* Q;
    float* partial;       /* [nsplit][ntaps][CpPad][CqPad] */
    float* qsum_partial;  /* [nsplit][CqPad] or NULL */
    int N, Hs, Ws;
    int Hp, Wp, Cp, p_cstride, p_coff, psy, psx;
    int Hq, Wq, Cq, q_cstride, q_coff, qsy, qsx;
    int ntaps;
    int pdy[LF_MAX_TAPS], pdx[LF_MAX_TAPS], qdy[LF_MAX_TAPS], qdx[LF_MAX_TAPS];
    int CpPad, CqPad; /* multiples of 64 */
    int nsplit;
} LfWgradArgs;
int lf_wgrad_f32(const LfWgradArgs* args, lf_stream_t stream);
/* split count lf_wgrad_f32 prefers for these arguments (nsplit field ignored), 0 = no preference */
int lf_wgrad_f32_nsplit(const LfWgradArgs* args);
int lf_wgrad_reduce(const float* partial, int nsplit, int ntaps, int Cp, int Cq, int CpPad, int CqPad,
                    float* dst, int st, int sp, int sq, lf_stream_t stream);
/* up to LF_REDUCE_MAX_JOBS such reductions in one launch (a bias-gradient reduction is the job ntaps = Cp = CpPad = 1,
 * sq = 1): the per-block weight and bias gradients of non_bottleneck_1d (host array, copied into the launch) */
#define LF_REDUCE_MAX_JOBS 8
typedef struct LfReduceJob {
    const float* partial;
    float* dst;
    int nsplit, ntaps, Cp, Cq, CpPad, CqPad, st, sp, sq;
} LfReduceJob;
int lf_reduce_multi(const LfReduceJob* jobs, int njobs, lf_stream_t stream);
/* dst[c] = sum over splits of partial[s][c]  (bias gradients) */
int lf_vec_reduce(const float* partial, int nsplit, int C, int Cpad, float* dst, lf_stream_t stream);
/* partial[blk][c] = sum over a pixel range of src[pix*cstride + coff + c]; nblk returned by the query */
int lf_colsum_blocks(long long npix);
int lf_colsum(const float* src, long long npix, int C, int cstride, int coff, float* partial, int Cpad,
              lf_stream_t stream);

/* 2x2/stride-2 max pooling into a channel slice (DownsamplerBlock, ERFNet.py:16,20) and its
 * gradient (first maximum wins, like ATen); accumulate != 0 adds into d_in. */
int lf_maxpool2_fwd(const float* in, int N, int Hin, int Win, int C, int in_cstride, float* out,
                    int out_cstride, int out_coff, lf_stream_t stream);
/* eval mode: out = relu(pool * scale[out_coff + c] + shift[out_coff + c]) -- the pooled half of relu(bn(cat[conv, pool]))
 * with the BatchNorm reduced to its running-statistics affine (lf_bn_eval_prepare) */
int lf_maxpool2_affine_relu(const float* in, int N, int Hin, int Win, int C, int in_cstride, const float* scale,
                            const float* shift, float* out, int out_cstride, int out_coff, lf_stream_t stream);
int lf_maxpool2_bwd(const float* in, int N, int Hin, int Win, int C, int in_cstride, const float* d_out,
                    int out_cstride, int out_coff, float* d_in, int din_cstride, int accumulate,
                    lf_stream_t stream);

/* BatchNorm2d, training mode, eps as given (1e-3 in ERFNet.py:17,33,39,102), dense [npix][C].
 *  stats   : per-block fp64 partial sums of x and x^2      -> partial[nblk][2][C]
 *  finalize: mean, invstd, scale = gamma*invstd, shift = beta - mean*scale; running stats
 *            updated with `momentum` (unbiased variance) when running_mean != NULL
 *  apply   : y = relu?( (x*scale+shift) * drop[n][c]? + res? )
 *  bwd     : g = dy * (ymask>0)? * drop? ;  s1 = sum g, s2 = sum g*xhat  (dgamma = s2, dbeta = s1)
 *            dx = scale * (g - s1/npix - xhat*s2/npix)                                        */
int lf_bn_blocks(long long npix, int C);
int lf_bn_stats(const float* x, long long npix, int C, double* partial, lf_stream_t stream);
int lf_bn_finalize(const double* partial, int nblk, long long npix, int C, const float* gamma,
                   const float* beta, float eps, float momentum, float* running_mean, float* running_var,
                   float* mean, float* invstd, float* scale, float* shift, lf_stream_t stream);
int lf_bn_eval_prepare(int C, const float* gamma, const float* beta, float eps, const float* running_mean,
                       const float* running_var, float* scale, float* shift, lf_stream_t stream);
int lf_bn_apply(const float* x, long long npix, int C, int pix_per_image, const float* scale,
                const float* shift, const float* drop, const float* res, int relu, float* y,
                lf_stream_t stream);
/* lf_bn_apply storing y as bf16, each element of the fp32 result rounded to nearest even (= torch's .to(torch.bfloat16)) */
int lf_bn_apply_bf16(const float* x, long long npix, int C, int pix_per_image, const float* scale,
                     const float* shift, const float* drop, const float* res, int relu, void* y,
                     lf_stream_t stream);
int lf_bn_bwd_reduce(const float* dy, const float* ymask, const float* drop, const float* x, long long npix,
                     int C, int pix_per_image, const float* mean, const float* invstd, double* partial,
                     lf_stream_t stream);
int lf_bn_bwd_finalize(const double* partial, int nblk, long long npix, int C, float* dgamma, float* dbeta,
                       float* c1, float* c2, lf_stream_t stream);
/* Finalize for statistics gathered by lf_conv1d_tc[_x3] with mask_scale: partial[nblk][2][C*fold] holds per-CTA
 * s1 = sum g and s2 = sum g*x (g = the masked gradient, x = the BatchNorm input) of `fold` column groups that map to
 * the same channel (fold > 1: super-pixel layers).  dbeta = s1, dgamma = invstd*(s2 - mean*s1) (fp64),
 * c1 = dbeta/npix, c2 = dgamma/npix = the per-channel constants lf_bn_bwd_apply takes. */
int lf_bn_bwd_finalize_sx(const double* partial, int nblk, long long npix, int C, int fold, const float* mean,
                          const float* invstd, float* dgamma, float* dbeta, float* c1, float* c2, lf_stream_t stream);
/* SyncBatchNorm (nn.SyncBatchNorm containers): the statistics of every rank, with the all-reduce between two launches.
 *  collapse : partial[nblk][2][C*fold] (of lf_bn_stats, the conv epilogue's stats_partial or lf_bn_bwd_reduce) ->
 *             totals[2C+1] = (sum a [C], sum b [C], npix), each sum in the order the finalize kernels above use
 *             (fold > 1 as lf_bn_bwd_finalize_sx); local (optional) receives a copy.  All-reduce (SUM) `totals`.
 *  finalize_tot        : lf_bn_finalize from the summed totals (count = totals[2C], as fp64).
 *  bwd_finalize_tot    : lf_bn_bwd_finalize; dgamma / dbeta from `local` (this rank's sums), c1 / c2 from `global` and *count
 *                        (the forward's global count).
 *  bwd_finalize_sx_tot : the same for lf_bn_bwd_finalize_sx's (sum g, sum g*x), with mean / invstd of the forward.
 * Each shares its per-channel arithmetic with the kernel it mirrors: totals of one process give the same bits. */
int lf_bn_collapse(const double* partial, int nblk, int C, int fold, long long npix, double* totals, double* local,
                   lf_stream_t stream);
int lf_bn_finalize_tot(const double* totals, int C, const float* gamma, const float* beta, float eps, float momentum,
                       float* running_mean, float* running_var, float* mean, float* invstd, float* scale, float* shift,
                       lf_stream_t stream);
int lf_bn_bwd_finalize_tot(const double* local, const double* global, const double* count, int C, float* dgamma,
                           float* dbeta, float* c1, float* c2, lf_stream_t stream);
int lf_bn_bwd_finalize_sx_tot(const double* local, const double* global, const double* count, int C, const float* mean,
                              const float* invstd, float* dgamma, float* dbeta, float* c1, float* c2, lf_stream_t stream);
int lf_bn_bwd_apply(const float* dy, const float* ymask, const float* drop, const float* x, long long npix,
                    int C, int pix_per_image, const float* mean, const float* invstd, const float* gamma,
                    const float* c1, const float* c2, float* dx, lf_stream_t stream);
/* lf_bn_bwd_apply that also stores gated = dy * (ymask > 0): the skip connection's gradient of a residual block, added by
 * the block's last input-gradient conv as one pre-masked operand (LfConvTcArgs.add_src without add_mask) */
int lf_bn_bwd_apply_gated(const float* dy, const float* ymask, const float* drop, const float* x, long long npix, int C,
                          int pix_per_image, const float* mean, const float* invstd, const float* gamma, const float* c1,
                          const float* c2, float* dx, float* gated, lf_stream_t stream);

/* Decoder.output_conv: ConvTranspose2d(16 -> L, 2, stride 2) (ERFNet.py:124,152).
 * x NHWC [N,H,W,Cin] -> out planar [N,L,2H,2W] (the layout the LSQ layer reads).
 * w is the reference layout [Cin][L][2][2]. */
int lf_outconv_fwd(const float* x, const float* w, const float* bias, int N, int H, int W, int Cin, int L,
                   float* out, lf_stream_t stream);
int lf_outconv_bwd_data(const float* d_out, const float* w, int N, int H, int W, int Cin, int L, float* d_x,
                        lf_stream_t stream);
int lf_outconv_wgrad_blocks(long long npix);
/* partial[blk][Cin*L*4 + L]: weight gradient (reference layout) then bias gradient */
int lf_outconv_bwd_weight(const float* x, const float* d_out, int N, int H, int W, int Cin, int L,
                          float* partial, lf_stream_t stream);

/* NCHW fp32 image [N,C,H,W] -> NHWC padded to Cpad channels (zeros), the stem's input layout */
int lf_nchw_to_nhwc_pad(const float* in, int N, int C, int H, int W, int Cpad, float* out, lf_stream_t stream);
/* wgmma gather-GEMM convolution for the resolution-changing layers (csrc/conv_tcg.cu): the 3x3 stride-2
 * Conv2d of DownsamplerBlock (BP/Networks/ERFNet.py:15,19-22), the 3x3 stride-2 ConvTranspose2d of UpsamplerBlock
 * (:66-73) and their input gradients, TF32 multiply / fp32 accumulate:
 *   out[n*osn + (oy*oy_mul + oy0)*osy + ox*osx + c] =
 *       bias[c] + sum_{t<ntaps} sum_{k<Kc} A_{map[t]}(n, oy+dy[t], ox+dx[t], k) * wg[c*ntaps*Kc + t*Kc + k]
 * for (n, oy, ox) in [N]x[Hs]x[Ws], c < Ng; A_i(n,y,x,k) = a[i].ptr[n*sn + y*sy + x*sx + k], zero outside
 * [0,H)x[0,W).  Kc: multiple of 32 (<= 256); Ng: multiple of 16 (<= 128); all strides multiples of 4 elements.
 * ops_net.py (tcg_* packers) maps the four layer forms onto this through pair-pixel / row-parity views. */
#define LF_TCG_MAX_TAPS 9   /* 6 for the stride-2 layers; 9 = a dense 3x3 stride-1 conv (Classification heads) */
typedef struct LfTcgView {
    const float* ptr;
    int H, W;
    long long sn, sy, sx;   /* element strides of image, row, pixel */
} LfTcgView;
typedef struct LfConvTcgArgs {
    LfTcgView a[2];
    const float* wg;        /* [Ng][ntaps*Kc] */
    const float* bias;      /* [Ng] or NULL */
    float* out;
    long long osn, osy, osx;
    int oy_mul, oy0;
    int N, Hs, Ws;
    int Kc, Ng, ntaps;
    int map[LF_TCG_MAX_TAPS], dy[LF_TCG_MAX_TAPS], dx[LF_TCG_MAX_TAPS];
    int precision;          /* 0 = TF32 multiply; 1 = 3xTF32 (fp32-grade): wg is [2][Ng][ntaps*Kc], the TF32 hi parts then
                               the lo parts (LF_PACK_TF32_HI / _LO), activations are split in shared memory;
                               2 = BF16 multiply: wg is [Ng][ntaps*Kc] bf16, activations rounded to bf16 in the kernel */
    int relu;               /* ReLU on conv + bias (eval-mode layers with the BatchNorm folded into wg / bias) */
} LfConvTcgArgs;
int lf_conv_tcg_supported(int N, int Hs, int Ws, int Kc, int Ng);
int lf_conv_tcg(const LfConvTcgArgs* args, lf_stream_t stream);

/* Weight gradients of the same layers on tensor cores (csrc/wgrad_tcg.cu), over the same views:
 *   D[blk*32 + c][n] = sum_{img,y,x} A_{map[blk]}(img, y+dy[blk], x+dx[blk], cblk[blk]*32 + c) * B(img, y, x, n)
 * for blk < nblocks (<= LF_WGRAD_TCG_MAX_BLOCKS), c < 32, n < Nn (multiple of 32, <= 128; ceil(nblocks/4)*Nn <= 512).
 * partial: [nctas][nblocks*32][Nn] per-CTA partial sums (nctas from lf_wgrad_tcg_ctas); reduce with lf_wgrad_reduce
 * (ntaps = 1, Cp = nblocks*32, Cq = Nn), then gather into [Co,Ci,3,3] (ops_net.wgrad_tcg_*). */
#define LF_WGRAD_TCG_MAX_BLOCKS 24
typedef struct LfWgradTcgArgs {
    LfTcgView a[2];
    LfTcgView b;
    float* partial;
    int N, Hs, Ws;
    int Ka, Nn, nblocks;
    int map[LF_WGRAD_TCG_MAX_BLOCKS], dy[LF_WGRAD_TCG_MAX_BLOCKS], dx[LF_WGRAD_TCG_MAX_BLOCKS], cblk[LF_WGRAD_TCG_MAX_BLOCKS];
    int nctas;
    int precision;          /* 0 = TF32 multiply; 1 = 3xTF32 (both operands split in shared memory, fp32-grade);
                               2 = BF16 multiply (both operands rounded to bf16 in the kernel) */
} LfWgradTcgArgs;
int lf_wgrad_tcg_ctas(int N, int Hs, int Ws, int Ka, int Nn, int nblocks);
int lf_wgrad_tcg_ctas_x3(int N, int Hs, int Ws, int Ka, int Nn, int nblocks);     /* same, for precision 1 */
int lf_wgrad_tcg_ctas_bf16(int N, int Hs, int Ws, int Ka, int Nn, int nblocks);   /* same, for precision 2 */
int lf_wgrad_tcg(const LfWgradTcgArgs* args, lf_stream_t stream);

/* Batched weight packing (host side: ops_net.WeightPackCache).  The reference keeps Conv2d / ConvTranspose2d
 * weights as [Co,Ci,kh,kw] (Networks/ERFNet.py:18-55 builds them with nn.Conv2d); every kernel above wants a
 * GEMM layout.  Each job gathers dst[k] = idx[k] >= 0 ? src[idx[k]] : 0 for k < n; one launch runs all jobs.
 * jobs_dev: DEVICE array of njobs records. */
/* Gather index flags: idx >= 0 selects src[idx & LF_PACK_INDEX_MASK]; with LF_PACK_TF32_HI / _LO the element written is
 * the TF32 "hi" part of that value (round to nearest, low 13 mantissa bits cleared) or the TF32 rounding of the
 * remainder value - hi: the pre-split weight operand of lf_conv1d_tc_x3 / lf_conv_tcg (precision 1). */
#define LF_PACK_INDEX_MASK 0x1fffffff
#define LF_PACK_TF32_HI 0x20000000
#define LF_PACK_TF32_LO 0x40000000
typedef struct LfPackJob {
    const float* src;   /* parameter in the reference layout (device) */
    void* dst;          /* packed operand (device), of dtype dst_dtype */
    const int* idx;     /* n gather indices into src, -1 = zero (device) */
    long long n;
    int dst_dtype;      /* LF_F32, or LF_BF16: every element rounded to bf16 (nearest even; = torch's .to(torch.bfloat16)),
                           the weight operand of lf_conv1d_tc_bf16 / lf_conv_tcg (precision 2).  Not combined with the
                           TF32 flags. */
    int pad;
} LfPackJob;
int lf_pack_gather(const LfPackJob* jobs_dev, int njobs, int blocks_per_job, lf_stream_t stream);

/* NHWC [N,H,W,C] <-> NCHW [N,C,H,W] (module-boundary layout changes) */
int lf_nhwc_to_nchw(const float* in, int N, int H, int W, int C, float* out, lf_stream_t stream);
int lf_nchw_to_nhwc(const float* in, int N, int C, int H, int W, float* out, lf_stream_t stream);

/* Back-projection loss over all lanes, forward and gradient in one launch (SURVEY.md 8f-1; replaces
 * BP/Loss_crit.py:161-218 applied per lane and averaged as BP/main.py:297-305): float64 throughout.
 *   Y56 [56][n], yprime [56], Minv [9] (row-major M^-1): HOST constants of the loss object (travel inside the launch);
 *   beta [B][L][n], x_gt / valid [B][L][56]: DEVICE inputs;  lane_loss [L], loss [1]: DEVICE outputs,
 *   loss = mean_l sum((x_gt - x_cal) valid)^2 / sum(valid)  (a lane with no valid sample contributes 0);
 *   dbeta [B][L][n] = d loss / d beta (or NULL), xcal [B][L][56] = x_cal * valid (or NULL);
 *   ticket: one zero-initialised device word (self-resetting).  No host synchronisation.
 * lf_backproj_loss_host runs the SAME per-point code on host arrays: a test hook for the CPU suite, not a fallback. */
int lf_backproj_loss(const double* Y56, const double* yprime, const double* Minv, const double* beta, const double* x_gt,
                     const double* valid, int B, int L, int n, double* lane_loss, double* loss, double* dbeta, double* xcal,
                     unsigned int* ticket, lf_stream_t stream);
int lf_backproj_loss_host(const double* Y56, const double* yprime, const double* Minv, const double* beta, const double* x_gt,
                          const double* valid, int B, int L, int n, double* lane_loss, double* loss, double* dbeta,
                          double* xcal);

/* Fully connected layers of the Classification heads (csrc/linear.cu; replaces nn.Linear at
 * BP/Networks/LSQ_layer.py:188-192,203-206): y[b][o] = bias[o] + sum_k x[b][k] W[o][k], W in nn.Linear's [O][K] layout,
 * fp32, deterministic.  partial: caller-owned scratch of lf_linear_chunks(K)*B*O floats.  relu: apply ReLU to y.
 * Backward: g = dy, or dy * (relu_out > 0) when relu_out (the forward's ReLU output) is given;
 *   lf_linear_bwd_data:   dx[b][k] = sum_o g[b][o] W[o][k]
 *   lf_linear_bwd_weight: dW[o][k] = sum_b g[b][o] x[b][k],  db[o] = sum_b g[b][o]  (db may be NULL). */
int lf_linear_chunks(int K);
/* AvgPool2d((1,W)) of the horizon head on an NHWC map, flattened as the reference's NCHW view does:
 * out[b][c*H + h] = mean_w x[b][h][w][c] (C <= 256); and its gradient dx[b][h][w][c] = dout[b][c*H + h] / W. */
int lf_rowmean_fwd(const float* x, int B, int H, int W, int C, float* out, lf_stream_t stream);
int lf_rowmean_bwd(const float* dout, int B, int H, int W, int C, float* dx, lf_stream_t stream);
int lf_linear_fwd(const float* x, const float* W, const float* bias, int B, int K, int O, int relu, float* partial, float* y,
                  lf_stream_t stream);
int lf_linear_bwd_data(const float* dy, const float* relu_out, const float* W, int B, int K, int O, float* dx, lf_stream_t stream);
int lf_linear_bwd_weight(const float* dy, const float* relu_out, const float* x, int B, int K, int O, float* dW, float* db,
                         lf_stream_t stream);

/* Segmentation-pretraining branch (csrc/seg.cu).  lf_seg_lane_maps replaces BP/Networks/LSQ_layer.py:279-293,301:
 * out [B][C][H][W] class planes (C = nl + 1) -> maps [B][nl][H][W], maps[b][k] = (argmax == k+1) ? k+1 : 0, rows < mask_rows
 * zeroed.  lf_ce2d_fwd / _bwd replace nn.CrossEntropyLoss(weight) on the planar logits (BP/Loss_crit.py:64-65,
 * BP/main.py:258,307): target [B][H][W] int64, weight [C] or NULL; partial = 2*lf_ce2d_blocks() doubles of scratch, sums = 2
 * doubles (weighted loss sum, weight sum) kept for the backward, loss = 1 double; dx = gout * dloss/dx (gout NULL = 1). */
int lf_seg_lane_maps(const float* out, int B, int C, int H, int W, int nl, int mask_rows, float* maps, lf_stream_t stream);
int lf_ce2d_blocks(int B, int H, int W);
int lf_ce2d_fwd(const float* x, const long long* target, const float* weight, int B, int C, int H, int W, double* partial, double* sums,
                double* loss, lf_stream_t stream);
int lf_ce2d_bwd(const float* x, const long long* target, const float* weight, int B, int C, int H, int W, const double* sums,
                const double* gout, float* dx, lf_stream_t stream);

/* Loader image path on the GPU (csrc/input_pipe.cu; replaces BP/Dataloader/Load_Data_new.py:127-131,166-167,178-181):
 * frames uint8 [N][Hin][Win][3] (decoded RGB) -> rows [crop_y0, crop_y0+crop_rows) -> PIL-BILINEAR resize to [Ho][Wo]
 * (Pillow's fixed-point two-pass resample, bit-identical) -> per-image horizontal flip (flip[n] != 0; NULL = none) ->
 * float32 / 255.  xb/yb: [Wo][2] / [Ho][2] (first source index, tap count) and xk/yk: [Wo][kx] / [Ho][ky] integer
 * coefficients (22 fractional bits) of the two axes, built by input_pipeline.resample_tables (the vertical axis over the
 * crop_rows rows).  layout 0: out [N][3][Ho][Wo]; 1: out [N][Ho][Wo][4] (NHWC, channel 3 = 0). */
int lf_frame_preprocess(const unsigned char* frames, int N, int Hin, int Win, int crop_y0, int crop_rows, const int* xb, const int* xk,
                        int kx, const int* yb, const int* yk, int ky, int Ho, int Wo, const unsigned char* flip, int layout,
                        float* out, lf_stream_t stream);

/* Optimizer update (csrc/optim.cu; replaces the torch.optim.Adam / SGD / RMSprop that BP/Networks/utils.py define_optim
 * builds, stepped at BP/main.py:262,340): one multi-tensor launch updates every parameter listed in `segs`, in place.
 * Each tensor stays where it is; the launch splits every segment into chunks of LF_OPTIM_CHUNK elements (the last one
 * shorter) and maps chunks to CTAs.  A chunk uses 16-byte accesses when all of its pointers are 16-byte aligned, scalar
 * accesses otherwise, so gradients may be views at any offset into a flat buffer.
 * Scalars are formed in fp64 from `hyper` and the step counter, then rounded to fp32; the elementwise arithmetic is fp32
 * in torch's order, each operation an explicit round-to-nearest intrinsic (nothing left for the compiler to contract);
 * a term a + s*b is one fused multiply-add exactly where torch's CUDA kernels form it as one (add_ with alpha, lerp_,
 * addcmul_, addcdiv_).  g = grad + wd*p in every algorithm:
 *   LF_OPTIM_ADAM    state0 = exp_avg, state1 = exp_avg_sq (amsgrad off, L2 weight decay, not AdamW):
 *                    m = m + (1-b1)(g-m);  v = b2 v + (1-b2) g g;  t += 1;
 *                    p -= (lr / (1-b1^t)) * m / (sqrt(v) / sqrt(1-b2^t) + eps)
 *   LF_OPTIM_SGD     state0 = momentum_buffer, state1 unused (NULL; dampening 0, no Nesterov):
 *                    buf = g on the first step (t = 0 before it), else momentum*buf + g;  p -= lr*buf
 *   LF_OPTIM_RMSPROP state0 = square_avg, state1 = momentum_buffer (not centred; hyper.beta2 is alpha):
 *                    sq = alpha sq + (1-alpha) g g;  buf = momentum*buf + g / (sqrt(sq) + eps);  p -= lr*buf
 * `state->step` is advanced once per launch, by the last CTA to finish (ticket).  `status`: NULL, or a device word
 * (lf_lsq_fwd's status); when it is nonzero the launch changes no parameter, state tensor or step counter and only
 * increments `state->skipped` -- the reference skips the batch of a singular system (BP/main.py:289-292) without a host
 * round trip.  `segs`, `hyper` and `state` are DEVICE pointers; `state` is zeroed once before first use and the ticket is
 * left at zero by every launch.  Never synchronises; graph-capturable (a replay reads the current `hyper`). */
#define LF_OPTIM_ADAM 0
#define LF_OPTIM_SGD 1
#define LF_OPTIM_RMSPROP 2
#define LF_OPTIM_CHUNK 2048
typedef struct LfOptimSeg {
    float* param;
    const float* grad;
    float* state0;
    float* state1;
    long long numel;
    long long chunk0;       /* index of this segment's first chunk: sum of ceil(numel / LF_OPTIM_CHUNK) over the rows before */
} LfOptimSeg;
typedef struct LfOptimHyper {
    double lr, beta1, beta2, eps, weight_decay, momentum;    /* beta2 = alpha for RMSprop; unused fields ignored */
} LfOptimHyper;
typedef struct LfOptimState {
    long long step;         /* updates applied (torch's per-parameter `step`, shared by every parameter) */
    long long skipped;      /* launches skipped by a nonzero status word */
    unsigned long long ticket;
} LfOptimState;
/* nchunks = total chunks over all rows (the chunk0 of a row one past the last) */
int lf_optim_step(int algo, const LfOptimSeg* segs, int nsegs, long long nchunks, const LfOptimHyper* hyper,
                  LfOptimState* state, const int* status, lf_stream_t stream);

/* Baseline JPEG decode (csrc/jpeg.cu; replaces Image.open(f).convert('RGB') of BP/Dataloader/Load_Data_new.py:118-119):
 * a batch of same-size baseline (SOF0 / 8-bit SOF1, Huffman) single-scan JPEGs, YCbCr 4:4:4 / 4:2:2 / 4:2:0 or grayscale,
 * with or without restart markers -> uint8 RGB [N][H][W][3], bit-identical to Pillow (libjpeg-turbo: ISLOW IDCT, fancy
 * upsampling, fixed-point YCbCr->RGB).  The markers are parsed on the host (lanedetection_end2end_b200/jpeg.py), which
 * fills one LfJpegImage per image; the entropy-coded bytes are unstuffed and decoded on the device.
 * The device blob is LfJpegImage[N] followed by the compressed bytes (ecs_off counts from the blob start).
 * lf_jpeg_workspace_bytes (HOST): checks the descriptors, fills their layout fields (in place) and returns the scratch
 *   bytes `workspace` needs (0 = invalid descriptors); *coef_bytes receives the size of the coefficient buffer, which the
 *   caller zeroes once before first use and which every launch leaves zeroed.
 * lf_jpeg_decode: three launches (entropy decode, dequantise + IDCT, upsample + colour); corrupt entropy data ORs
 *   LF_STATUS_JPEG_CORRUPT into *status.  Calls sharing `coef` / `workspace` must be ordered by the caller. */
#define LF_STATUS_JPEG_CORRUPT 8
#define LF_JPEG_PIECE_BYTES 128   /* size of one piece of the unstuffed bitstream a thread decodes */
#define LF_JPEG_MAX_BPM 6         /* blocks per MCU (4:2:0) */
typedef struct LfJpegHuff {
    unsigned short look[512];     /* 9-bit lookahead: (code length << 8) | symbol, 0 = longer code */
    int maxcode[18];              /* largest code of each length 1..16, -1 if none; [17] sentinel */
    int valoff[18];               /* symbol index - code, per length */
    unsigned char val[256];
} LfJpegHuff;
typedef struct LfJpegImage {
    long long ecs_off;            /* entropy-coded segment: blob offset and length in bytes */
    int ecs_len;
    int W, H, ncomp;              /* ncomp 1 (grayscale) or 3 (YCbCr) */
    int mcux, mcuy, bpm;          /* MCUs per row / column, blocks per MCU */
    int restart, nint;            /* restart interval in MCUs (0 = none), number of intervals */
    int hs[3], vs[3];             /* sampling factors; comp_w / comp_h: component size in samples */
    int comp_w[3], comp_h[3];
    int qtab[3];                  /* quantisation table of each component */
    int blk_comp[LF_JPEG_MAX_BPM], blk_dx[LF_JPEG_MAX_BPM], blk_dy[LF_JPEG_MAX_BPM];
    int blk_dc[LF_JPEG_MAX_BPM], blk_ac[LF_JPEG_MAX_BPM]; /* Huffman tables of each block of the MCU (0..3 each) */
    /* layout, filled by lf_jpeg_workspace_bytes: byte offsets into workspace, block offset into coef */
    long long stream_off, x_off, b_off, us_off, pb_off, plane_off[3], block_off;
    int plane_stride[3], npieces_max;
    unsigned short qt[4][64];     /* quantisation tables, natural order */
    LfJpegHuff dc[4], ac[4];
} LfJpegImage;
size_t lf_jpeg_workspace_bytes(LfJpegImage* images, int N, size_t* coef_bytes);
int lf_jpeg_decode(const void* blob, int N, int W, int H, unsigned char* out, int* status, void* coef, size_t coef_bytes,
                   void* workspace, size_t workspace_bytes, lf_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LANEFIT_B200_H */
