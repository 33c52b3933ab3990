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
 *   mask_rows           rows [0,mask_rows) get weight zero and are never read: NaN or Inf
 *                       in those rows of o, xtab, ytab or yrow changes no output bit
 *   beta     [B,L,order+1] f64 out, highest power first (:100-104); NaN for a system
 *            whose solve sets SINGULAR or NOT_POSDEF
 *   zinv     [B,L,(order+1)^2] f64 out, row-major: (Y^T W^2 Y + reg I)^-1, consumed by
 *            lf_lsq_bwd.  Z_ij = S_{2d-i-j} + reg_ls*delta_ij, X_i = T_{d-i} with
 *            S_k = sum w y^k, T_k = sum w x y^k, w = act(o)^2 over the unmasked rows
 *   solver   LF_SOLVER_INVERSE (Gauss-Jordan, partial pivoting) or LF_SOLVER_CHOLESKY
 *   masked   [B,L,H,W] f32 out or NULL: activation(o) with masked rows zeroed (output #5
 *            of Net.forward, :315); the masked rows are +0.0
 *   status   int32 out: OR of LF_STATUS_* over all B*L systems (caller zeroes it; bits
 *            already set stay set)
 *   workspace: lf_lsq_workspace_bytes() bytes, ZEROED once before first use; the
 *            library leaves it reusable (tickets reset) after every launch, by any
 *            later call of any shape.  Calls sharing a workspace must be stream-ordered.
 * Row-separable kernel (yrow given, W % 4 == 0 for f32 o, W % 8 == 0 for bf16 o): 16-byte
 * loads and stores, so o, xtab and masked (d_o in the backward) must be 16-byte aligned;
 * a misaligned pointer is refused with LF_ERR_INVALID_ARGUMENT.  Otherwise the general
 * kernel runs (ytab required, any alignment of the element type).
 * lf_lsq_fwd returns LF_ERR_UNSUPPORTED for B*L > 16384 (the workspace's ticket region);
 * lf_lsq_bwd uses no workspace and has no such limit.
 * ------------------------------------------------------------------------- */
size_t lf_lsq_workspace_bytes(int B, int L, int H, int W, int order);
/* The plan lf_lsq_fwd (bwd = 0) or lf_lsq_bwd (bwd = 1) selects for these arguments (has_yrow / has_ytab: whether
 * that pointer is non-NULL); no device needed (132 SMs assumed without one).  LF_OK and info[LF_LSQ_PLAN_INFO] =
 * {row-separable kernel (1) or general (0), activation template (LF_ACT_SQUARE, or -1 = run-time activation), lanes
 * per CTA NL, lane groups (= grid z), chunks per system (= grid x), resident CTAs per SM the chunk count is fitted to,
 * byte alignment required of o / xtab / masked / d_o (16, or 0 = element alignment)}; otherwise the code the entry
 * point returns for the same arguments (pointer and solver checks aside).  Chunk c of a system covers the masked rows
 * [c*m/n, (c+1)*m/n) and the unmasked rows mask_rows + [c*h/n, (c+1)*h/n), m = mask_rows, h = H - m, n = chunks. */
#define LF_LSQ_PLAN_INFO 7
int lf_lsq_plan(int bwd, int o_dtype, int has_yrow, int has_ytab, int B, int L, int H, int W, int order, int mask_rows,
                int act, int* info);
int lf_lsq_fwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
               int B, int L, int H, int W, int order, int mask_rows, int act, double reg_ls, int solver,
               double* beta, double* zinv, float* masked, int* status,
               void* workspace, size_t workspace_bytes, lf_stream_t stream);

/* lf_lsq_fwd on the row-separable kernel (yrow required, no ytab) that also stores, per (image, lane, unmasked row r),
 * rowsums[b][l][r] = (A_r, B_r, C_r) = sum_c (w, w x, w c), w = (mask * act(o))^2, float32 [B][L][H][3]: what
 * lf_lsq_grid_grad needs.  Same plan, checks and outputs as lf_lsq_fwd. */
int lf_lsq_fwd_rowsums(const void* o, int o_dtype, const float* xtab, const float* yrow, int B, int L, int H, int W,
                       int order, int mask_rows, int act, double reg_ls, int solver, double* beta, double* zinv,
                       float* masked, int* status, float* rowsums, void* workspace, size_t workspace_bytes,
                       lf_stream_t stream);
/* Gradient with respect to row-separable tables x[r][c] = alpha_r c + gamma_r, y_r = const - y'_r (a learned
 * homography), summed over images and lanes in a fixed order, from lf_lsq_fwd_rowsums' row sums and beta, Z^-1 and
 * gbeta = dL/dbeta:  dL/dgamma_r = (phi.z) A_r,  dL/dalpha_r = (phi.z) C_r,
 * dL/dy'_r = -[(phi'.z)(B_r - (phi.beta) A_r) - (phi.z)(phi'.beta) A_r],  z = Z^-1 gbeta, phi = [y^d .. y 1].
 * g_rowp [H][3] f64 = (alpha, gamma, y'); 0 for the masked rows. */
int lf_lsq_grid_grad(const float* rowsums, const float* yrow, const double* beta, const double* zinv, const double* gbeta,
                     int B, int L, int H, int order, int mask_rows, double* g_rowp, lf_stream_t stream);

/* Backward of the above: d_o = dL/d o given gbeta = dL/d beta [B,L,order+1] f64.
 * Replaces autograd through mul/bmm/inverse (BP/Networks/LSQ_layer.py:111-116) ==
 * GELS.backward (BP/Networks/gels.py:18-25) composed with the activation and mask:
 *   z = Z^-1 g ;  d_o = mask * act'(o) * 2 act(o) * (x - phi^T beta) * (phi^T z).
 * d_o has the dtype of o. */
int lf_lsq_bwd(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
               int B, int L, int H, int W, int order, int mask_rows, int act,
               const double* beta, const double* zinv, const double* gbeta,
               void* d_o, lf_stream_t stream);

/* Per-pixel keep map (the reference's trapezium mask, --trapezium_mask): lf_lsq_fwd, lf_lsq_fwd_rowsums and lf_lsq_bwd
 * with one more operand,
 *   keep     [H,W] uint8, shared by every image and lane: where keep is 0 the activated map act(o) is replaced by
 *            +0.0 before it is squared, so the pixel adds nothing to S_k, T_k (or the row sums), `masked` holds +0.0
 *            there and d_o is +0.0 there (o is still read; NaN or Inf there changes no output bit).  Any nonzero
 *            byte keeps the pixel.  Required (NULL is LF_ERR_INVALID_ARGUMENT); on the row-separable kernel it must
 *            be 16-byte aligned like o.
 * Rows [0, mask_rows) are handled as without the map.  The plan is lf_lsq_plan's for the same arguments: the map
 * changes neither the kernel choice, the lanes per CTA nor the chunks.  An all-ones map gives the bits of the entry
 * point without it for act = LF_ACT_SQUARE, for lf_lsq_bwd_keep and on the general kernel; the row-separable forward
 * with a run-time activation may differ from them in the last bits of its fp32 row sums. */
int lf_lsq_fwd_keep(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
                    const uint8_t* keep, int B, int L, int H, int W, int order, int mask_rows, int act, double reg_ls,
                    int solver, double* beta, double* zinv, float* masked, int* status, void* workspace,
                    size_t workspace_bytes, lf_stream_t stream);
int lf_lsq_fwd_rowsums_keep(const void* o, int o_dtype, const float* xtab, const float* yrow, const uint8_t* keep,
                            int B, int L, int H, int W, int order, int mask_rows, int act, double reg_ls, int solver,
                            double* beta, double* zinv, float* masked, int* status, float* rowsums, void* workspace,
                            size_t workspace_bytes, lf_stream_t stream);
int lf_lsq_bwd_keep(const void* o, int o_dtype, const float* xtab, const float* ytab, const float* yrow,
                    const uint8_t* keep, int B, int L, int H, int W, int order, int mask_rows, int act,
                    const double* beta, const double* zinv, const double* gbeta, void* d_o, lf_stream_t stream);

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
 * (lf_conv1d_tc_supported tells).  Same results as lf_conv_f32 up to the TF32 form of the operands: the kernel rounds
 * the activations to TF32 (nearest, ties away from zero), while `wpack` reaches the tensor core as its fp32 bits, which
 * wgmma .tf32 truncates (low 13 mantissa bits ignored); pass TF32-rounded weights for rounded ones. */
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
                              the slab and the per-tap variants fill it alike */
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
/* 1 if a call with taps {-dil,0,+dil} along y (vertical) or x runs on the slab kernel */
int lf_conv1d_tc_slab_ok(int N, int H, int W, int C, int vertical, int dil);
/* The plan lf_conv1d_tc (prec 0), _x3 (1), _bf16 (2) or _fp8 (3) selects for these arguments (in_dtype: of `in`), with
 * the variant set now; no device needed.  LF_OK and info[LF_TC_PLAN_INFO] = {slab (1) or one box per tap (0), weights
 * resident (1) or streamed per stage (0), pipeline stages, 3xTF32 lo buffers (0 otherwise), lo buffer over the staging
 * tile (1), lo bytes outside the ring, tile extent along the conv axis TA, across it TB (pixels), vertical, CTAs per
 * 64-channel half (= rows of colsum_partial / stats_partial), dynamic shared memory bytes, activation bytes per stage};
 * LF_ERR_UNSUPPORTED where the launch would return it, LF_ERR_INVALID_ARGUMENT for N, H, W < 1 or a bad prec / dtype.
 * Tile m = (image * tiles across + tile across) * tiles along + tile along runs on CTA row m % CTAs. */
#define LF_TC_PLAN_INFO 12
int lf_conv1d_tc_plan(int prec, int in_dtype, int N, int H, int W, int C, const int* dy, const int* dx, int* info);

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

/* Weight gradients on tensor cores (csrc/wgrad_tcg.cu), over the views above -- of these layers, of the Classification
 * heads' stride-1 convolutions and of the factorised 3-tap convolutions of non_bottleneck_1d:
 *   D[blk*32 + c][n] = sum_{img,y,x} A_{map[blk]}(img, y+dy[blk], x+dx[blk], cblk[blk]*32 + c) * B(img, y, x, n)
 * for blk < nblocks (<= LF_WGRAD_TCG_MAX_BLOCKS, any Nn: a CTA takes one pair of blocks), c < 32, n < Nn (multiple of
 * 32, <= 128).
 * partial: [nctas][nblocks*32][Nn] per-CTA partial sums; reduce with lf_wgrad_reduce (ntaps = 1, Cp = nblocks*32, Cq = Nn),
 * then gather into [Co,Ci,3,3] (ops_net.wgrad_tcg_*), or for a 3-tap convolution with blk = t*C/32 + cb
 * (ntaps = 3, Cp = Cq = C) straight into the weight layout.
 * nctas = lf_wgrad_tcg_ctas(..., min_patches): split-K slices of at least min_patches 32-pixel patches each, at most one
 * wave of CTAs (0 = unsupported shape).  The split count fixes the order in which the partials are summed. */
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
    int a_dtype;            /* element type of the A views: LF_F32, or LF_BF16 (the bf16-stored layer inputs of the bf16
                               mode: same results as their fp32 copy) -- precision 2 and Nn in {64, 128} only, else
                               LF_ERR_UNSUPPORTED; B stays fp32 */
} LfWgradTcgArgs;
int lf_wgrad_tcg_ctas(int N, int Hs, int Ws, int Ka, int Nn, int nblocks, int min_patches);
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
/* lf_backproj_loss with the warp constants on the DEVICE (a learned homography): yk [56] = y' of the sample rows, Minv [9];
 * Y56 is built from yk in the kernel.  Also emits g_const [65] = dloss/dM^-1 (9) then dloss/dy'_k (56); g_part [L][65]
 * is scratch (per-lane gradients).  dbeta is required.  lf_backproj_loss_dev_host: the same arithmetic on host arrays
 * (test hook). */
int lf_backproj_loss_dev(const double* yk, const double* Minv, const double* beta, const double* x_gt, const double* valid,
                         int B, int L, int n, double* lane_loss, double* loss, double* dbeta, double* xcal, double* g_part,
                         double* g_const, unsigned int* ticket, lf_stream_t stream);
int lf_backproj_loss_dev_host(const double* yk, const double* Minv, const double* beta, const double* x_gt,
                              const double* valid, int B, int L, int n, double* lane_loss, double* loss, double* dbeta,
                              double* xcal, double* g_const);

/* Learned bird's-eye-view homography (csrc/homography.cu): get_homography(resize)'s source corners shifted by theta [5]
 * float32 (theta_0..3: x of the four corners in units of 2*resize; theta_4: row of the two top corners in units of
 * resize).  The warp stays row-preserving, M and M^-1 come in closed form.
 * lf_homography_tables: M [9] and Minv [9] (row-major), rowp [resize][3] f64 (alpha_v, gamma_v, y'_v), xtab
 * [resize][2*resize] f32 = alpha_v u + gamma_v, yrow [resize] f32 = y_const - y'_v, yk [56] f64 (y' of the loss's sample
 * rows); an unmasked row (v >= mask_rows) on the vanishing line or beyond it (den_v = m21 v + m22 zero or of the
 * other sign than the bottom row's) or with a non-finite table entry ORs LF_STATUS_NONFINITE into
 * *status.  lf_homography_bwd: g_theta [5] f32 = dL/dtheta from dL/drowp [resize][3], dL/dMinv [9], dL/dyk [56] (f64,
 * each may be NULL).  All DEVICE.  The _host variants are test hooks on host arrays (g_theta f64 there). */
int lf_homography_tables(const float* theta, int resize, int mask_rows, double y_const, double* M, double* Minv,
                         double* rowp, float* xtab, float* yrow, double* yk, int* status, lf_stream_t stream);
int lf_homography_bwd(const float* theta, int resize, int mask_rows, const double* g_rowp, const double* g_minv,
                      const double* g_yk, float* g_theta, lf_stream_t stream);
int lf_homography_host(const float* theta, int resize, double* Mpair, double* rowp, double* yk);
int lf_homography_bwd_host(const float* theta, int resize, int mask_rows, const double* g_rowp, const double* g_minv,
                           const double* g_yk, double* g_theta);

/* Predicted bird's-eye-view homography (csrc/homography.cu, --predict_homography): one warp per image from z [B][3]
 * float32, the output of the spatial-transformer branch.  delta = tanh(z) / 16 (f64) moves get_homography(resize)'s
 * DESTINATION corners: the left column by delta_0 * 2*resize, the right column by delta_1 * 2*resize, the top row by
 * delta_2 * resize; source corners and the bottom row stay fixed, so every warp is row-preserving (closed form).
 * lf_predicted_homography_tables: delta [B][3], M / Minv [B][9], rowp [B][resize][3], yk [B][56] (f64), xtab
 * [B][resize][2*resize], yrow [B][resize] (f32), each image's slice as lf_homography_tables computes it; the guard of
 * lf_homography_tables on every image, OR-ed once into *status.  lf_predicted_homography_bwd: g_z [B][3] f32 from dL/drowp
 * [B][resize][3], dL/dMinv [B][9], dL/dyk [B][56] (f64, each may be NULL), forward-mode dual numbers through tanh / 16,
 * one fixed-order tree per image.  All DEVICE.  Test hooks on host arrays for one image: _host takes delta [3] (f64)
 * directly and returns Mpair [18] (M, Minv), rowp [resize][3] and yk [56] when not NULL; _bwd_host returns g_z [3] f64. */
int lf_predicted_homography_tables(const float* z, int B, int resize, int mask_rows, double y_const, double* delta,
                                   double* M, double* Minv, double* rowp, float* xtab, float* yrow, double* yk,
                                   int* status, lf_stream_t stream);
int lf_predicted_homography_bwd(const float* z, int B, int resize, int mask_rows, const double* g_rowp,
                                const double* g_minv, const double* g_yk, float* g_z, lf_stream_t stream);
int lf_predicted_homography_host(const double* delta, int resize, double* Mpair, double* rowp, double* yk);
int lf_predicted_homography_bwd_host(const float* z, int resize, int mask_rows, const double* g_rowp,
                                     const double* g_minv, const double* g_yk, double* g_z);

/* The same per-image warp in the source-corner parametrisation (--predict_homography_corners source): z [B][5] float32,
 * theta = tanh(z) / 64 rounded to float32 is lf_homography_tables' theta for each image (source corners moved,
 * destination corners and bottom row fixed).  lf_predicted_homography_source_tables: theta [B][5] f32 and the tables of
 * lf_predicted_homography_tables, image b's slice bit for bit lf_homography_tables(theta_b); the same guard.
 * lf_predicted_homography_source_bwd: g_z [B][5] f32 and, when g_theta is not NULL, g_theta [B][5] f64 = dL/dtheta_b as
 * lf_homography_bwd's tree sums it for one warp, from dL/drowp [B][resize][3], dL/dMinv [B][9], dL/dyk [B][56] (f64,
 * each may be NULL); g_z = g_theta (1 - tanh^2 z) / 64.  All DEVICE.  Test hooks on host arrays for one image:
 * _source_host takes z [5] and returns theta [5] (when not NULL), then as lf_homography_host; _source_bwd_host returns
 * g_z [5] and g_theta [5] (when not NULL) in f64. */
int lf_predicted_homography_source_tables(const float* z, int B, int resize, int mask_rows, double y_const, float* theta,
                                          double* M, double* Minv, double* rowp, float* xtab, float* yrow, double* yk,
                                          int* status, lf_stream_t stream);
int lf_predicted_homography_source_bwd(const float* z, int B, int resize, int mask_rows, const double* g_rowp,
                                       const double* g_minv, const double* g_yk, float* g_z, double* g_theta,
                                       lf_stream_t stream);
int lf_predicted_homography_source_host(const float* z, int resize, float* theta, double* Mpair, double* rowp,
                                        double* yk);
int lf_predicted_homography_source_bwd_host(const float* z, int resize, int mask_rows, const double* g_rowp,
                                            const double* g_minv, const double* g_yk, double* g_z, double* g_theta);

/* Per-image least-squares tables (a predicted homography): xtab [B][H][W] and yrow [B][H], image b fitted on its own
 * slice, on the row-separable plan only (LF_ERR_INVALID_ARGUMENT when lf_lsq_plan would not pick it).
 * lf_lsq_fwd_per_image: lf_lsq_fwd (rowsums = NULL) or lf_lsq_fwd_rowsums (rowsums [B][L][H][3]); keep as the *_keep
 * entry points, or NULL for none.  lf_lsq_bwd_per_image: lf_lsq_bwd / lf_lsq_bwd_keep likewise.  Each image's outputs
 * are a single-image call's bits on that image's tables.  lf_lsq_grid_grad_per_image: g_rowp [B][H][3], image b's
 * lf_lsq_grid_grad summed over its own lanes only.  All DEVICE. */
int lf_lsq_fwd_per_image(const void* o, int o_dtype, const float* xtab, const float* yrow, const uint8_t* keep, int B,
                         int L, int H, int W, int order, int mask_rows, int act, double reg_ls, int solver, double* beta,
                         double* zinv, float* masked, int* status, float* rowsums, void* workspace,
                         size_t workspace_bytes, lf_stream_t stream);
int lf_lsq_bwd_per_image(const void* o, int o_dtype, const float* xtab, const float* yrow, const uint8_t* keep, int B,
                         int L, int H, int W, int order, int mask_rows, int act, const double* beta, const double* zinv,
                         const double* gbeta, void* d_o, lf_stream_t stream);
int lf_lsq_grid_grad_per_image(const float* rowsums, const float* yrow, const double* beta, const double* zinv,
                               const double* gbeta, int B, int L, int H, int order, int mask_rows, double* g_rowp,
                               lf_stream_t stream);

/* lf_backproj_loss_dev with one warp per image: yk [B][56], Minv [B][9]; g_const [B][65] holds each image's gradient
 * (dloss/dMinv, then dloss/dyk); scratch: lf_backproj_loss_per_image_scratch(B, L) doubles.  With every image given
 * the same warp, loss, dbeta and xcal are lf_backproj_loss_dev's bits.  All DEVICE. */
size_t lf_backproj_loss_per_image_scratch(int B, int L);
int lf_backproj_loss_per_image(const double* yk, const double* Minv, const double* beta, const double* x_gt,
                               const double* valid, int B, int L, int n, double* lane_loss, double* loss, double* dbeta,
                               double* xcal, double* scratch, double* g_const, unsigned int* ticket, lf_stream_t stream);


/* Area loss of the bird's-eye-view experiment over all lanes, its gradient and the exact-area metric in one launch
 * (csrc/loss.cu; replaces Birds_Eye_View_Loss/Loss_crit.py:98-134 summed over the lanes as BEV/main.py:223,237 does, and
 * the `polynomial.trapezoidal` metric of BEV/main.py:273-280,436-442).  Order 2 only.
 *   beta [B][L][3], params [B][4][3] (the loader's ground-truth coefficients): float32 DEVICE inputs; L is 2 or 4, B >= 1;
 *   weight: 0 none (W = 1), 1 linear (W = 1 - y), 2 quadratic (W = 1 - sqrt y); anything else LF_ERR_INVALID_ARGUMENT.
 *   loss [1] = sum_l mean over the images whose three params[b][l] are all non-zero of int_0^0.7 W (beta - params)^2 dy
 *     (0 for a lane without such an image): float64 terms, fixed-order sums, one rounding to float32;
 *   dbeta [B][L][3] = d loss / d beta, same arithmetic;
 *   exact [B] = (trap(lane 0) + trap(lane 1)) / 2, trap the reference's float32 trapezium rule (101 points on [0, 0.7]),
 *     bit-identical to polynomial(beta).trapezoidal(polynomial(params)) on the CPU;  exact_mean [1] = its batch mean.
 *   Every output may be NULL.  One CTA, no atomics, deterministic; no host synchronisation (capturable).
 * lf_area_loss_host runs the SAME per-image code and summation order on host arrays: a test hook, not a fallback. */
int lf_area_loss(const float* beta, const float* params, int B, int L, int weight, float* loss, float* dbeta, float* exact,
                 float* exact_mean, lf_stream_t stream);
int lf_area_loss_host(const float* beta, const float* params, int B, int L, int weight, float* loss, float* dbeta,
                      float* exact, float* exact_mean);

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
/* lf_seg_lane_maps plus the gt_line substitution of BP/Networks/LSQ_layer.py:308-311 (`masked[gt_mask] = masked[0, 0]...`):
 * gt_line [B][nl] float on the device, or NULL (then the output is lf_seg_lane_maps'); where gt_line[b][k] != 0, maps[b][k] is
 * image 0 / lane 0's map as lf_seg_lane_maps computes it. */
int lf_seg_lane_maps_line(const float* out, int B, int C, int H, int W, int nl, int mask_rows, const float* gt_line, float* maps,
                          lf_stream_t stream);
int lf_ce2d_blocks(int B, int H, int W);
int lf_ce2d_fwd(const float* x, const long long* target, const float* weight, int B, int C, int H, int W, double* partial, double* sums,
                double* loss, lf_stream_t stream);
int lf_ce2d_bwd(const float* x, const long long* target, const float* weight, int B, int C, int H, int W, const double* sums,
                const double* gout, float* dx, lf_stream_t stream);
/* Confusion counts of a segmentation output (the proxy branch's validation metrics): logits [B][C][H][W] float, target
 * [B][H][W] int64; for every pixel with 0 <= target < C, counts[target * C + pred] += 1, pred the segmentation branch's
 * argmax (the first maximum wins; a NaN logit in class c >= 1 never wins; a NaN in class 0 keeps class 0, since no
 * comparison with it succeeds).  counts [C*C] int64 is zeroed by the caller and accumulated; exact and independent of
 * the launch order.  status: NULL, or a device int whose nonzero value makes the launch count nothing (the LSQ status
 * word of a skipped batch).  Capturable, never synchronises.  2 <= C <= 8 and positive sizes, else
 * LF_ERR_INVALID_ARGUMENT. */
int lf_seg_confusion(const float* logits, const long long* target, int B, int C, int H, int W, const int* status,
                     long long* counts, lf_stream_t stream);

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

/* The same update with one step count per parameter, as torch.optim keeps it: a parameter that misses an update (no
 * gradient, e.g. the heads while only the segmentation output is trained, BP/main.py:32-43,255-282) keeps its count, and
 * a parameter that joins later starts at step 1.  Row r of `segs` updates the parameter whose count is steps[slot].
 * `steps` (DEVICE, nparams counts, zeroed once before first use) outlives the tables built over it, so a parameter that
 * drops out of a table keeps its count.  `slots` (HOST, nsegs entries) repeats the rows' slots for the argument checks:
 * every slot in [0, nparams), no slot in two rows; the rows in `segs` must carry the same values.
 * Two launches on `stream`:
 *   1. one thread per row: with `status` NULL or zero, forms the row's scalars from steps[slot] (fp64 bias corrections
 *      rounded to fp32, as lf_optim_step; for SGD `first` is steps[slot] == 0), stores them in `scalars` and increments
 *      steps[slot]; with a nonzero status it changes nothing and increments *skipped once;
 *   2. lf_optim_step's chunk loop, each chunk with its row's scalars; nothing when the status is nonzero.
 * The elementwise arithmetic is lf_optim_step's, one code.  `scalars`: DEVICE workspace of
 * nsegs * LF_OPTIM_PP_SCALAR_BYTES bytes, 16-byte aligned.  Never synchronises; graph-capturable. */
#define LF_OPTIM_PP_SCALAR_BYTES 48
typedef struct LfOptimSegPP {
    LfOptimSeg seg;
    int slot;               /* index into `steps` */
    int reserved;
} LfOptimSegPP;
int lf_optim_step_pp(int algo, const LfOptimSegPP* segs, const int* slots, int nsegs, long long nchunks,
                     const LfOptimHyper* hyper, long long* steps, int nparams, void* scalars, long long* skipped,
                     const int* status, lf_stream_t stream);

/* Gradient clipping by the global L2 norm, torch.nn.utils.clip_grad_norm_(params, max_norm) before the update, inside the
 * captured step.  `clip` is a DEVICE LfGradClip, zeroed once before first use, then max_norm set (> 0, finite; a
 * replay reads its current value, so a new threshold needs no recapture).
 * lf_grad_norm (lf_grad_norm_pp over an LfOptimSegPP table): one launch over the rows' gradients, chunked as the update
 *   chunks them.  Each fp32 element is squared exactly in fp64 and summed in fp64, one partial per chunk into
 *   `workspace` (DEVICE, lf_grad_norm_workspace_bytes(nchunks) bytes, 8-byte aligned); the last CTA (ticket, left at
 *   zero) sums the partials in a fixed order.  Every order is set by the table alone, so the result is bit-identical
 *   from run to run and does not depend on the grid size or on a gradient's alignment.  It writes
 *     total_norm = fp32(sqrt(sum)), the sqrt in fp64 and rounded once;
 *     clip_coef  = min(fl(fl(1 / fl(total_norm + fl(1e-6))) * max_norm), 1) in fp32, torch's op order (`max_norm /
 *                  (total_norm + 1e-6)` is reciprocal() * max_norm), a NaN kept as torch.clamp keeps it;
 *     nonfinite  = 1 exactly when some element is NaN or +-Inf, else 0.  The squares are non-negative and fp64 cannot
 *                  overflow on their sum (each is below 2^256), so the sum is non-finite only through such an element.
 *   The norm is more exact than torch's fp32 per-tensor norms and may differ from them in the last bits.
 * lf_optim_step_clip / lf_optim_step_pp_clip: the update of lf_optim_step / lf_optim_step_pp with every gradient element
 *   first multiplied by clip_coef (one fp32 rounding, torch's _foreach_mul_(grads, clip_coef)), then the same
 *   arithmetic.  The gradients themselves are not rewritten.  The launch is skipped -- no parameter, state tensor or step
 *   count changes -- when the status word is nonzero or `nonfinite` is set; each skipped launch increments the skipped
 *   count, and one skipped by `nonfinite` alone (status NULL or zero) also increments clip->nonfinite_skipped.
 * Never synchronise; graph-capturable.  Calls sharing `clip` or `workspace` must be ordered by the caller. */
typedef struct LfGradClip {
    float max_norm;                 /* in */
    float total_norm;               /* out of the norm launch */
    float clip_coef;                /* out of the norm launch */
    int nonfinite;                  /* out of the norm launch */
    long long nonfinite_skipped;    /* updates skipped by `nonfinite` alone */
    unsigned long long ticket;
} LfGradClip;
size_t lf_grad_norm_workspace_bytes(long long nchunks);     /* HOST; 0 for nchunks <= 0 */
int lf_grad_norm(const LfOptimSeg* segs, int nsegs, long long nchunks, LfGradClip* clip, void* workspace,
                 size_t workspace_bytes, lf_stream_t stream);
int lf_grad_norm_pp(const LfOptimSegPP* segs, int nsegs, long long nchunks, LfGradClip* clip, void* workspace,
                    size_t workspace_bytes, lf_stream_t stream);
int lf_optim_step_clip(int algo, const LfOptimSeg* segs, int nsegs, long long nchunks, const LfOptimHyper* hyper,
                       LfOptimState* state, const int* status, LfGradClip* clip, lf_stream_t stream);
int lf_optim_step_pp_clip(int algo, const LfOptimSegPP* segs, const int* slots, int nsegs, long long nchunks,
                          const LfOptimHyper* hyper, long long* steps, int nparams, void* scalars, long long* skipped,
                          const int* status, LfGradClip* clip, lf_stream_t stream);

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

/* Baseline JPEG encode (csrc/jpeg_enc.cu): a batch of N same-size frames, uint8 RGB [N][H][W][3] (ncomp 3) or grayscale
 * [N][H][W] (ncomp 1) -> one JPEG file per frame, byte-identical to Pillow's
 * Image.fromarray(a).save(buf, "JPEG", quality=q, subsampling=s) (libjpeg-turbo: fixed-point YCbCr, h2v2 downsampling,
 * ISLOW forward DCT, its reciprocal quantisation, standard Huffman tables, no restart markers).
 *   sampling: 2 = 4:2:0 (Pillow's default), 0 = 4:4:4.  A grayscale file codes the same bytes either way; Pillow's header
 *   records 2x2 for its component under 4:2:0, and so does this one.  W, H in 1..65535.
 *   qtables: HOST uint16 [ncomp == 3 ? 2 : 1][64], natural order, each entry 1..255 (lf_jpeg_quality_tables fills them).
 *   out: device bytes, image n's file at out + n * out_cap; out_cap >= lf_jpeg_encode_bound(W, H, ncomp, sampling).
 *   out_len: device int64 [N], each file's length.  workspace: lf_jpeg_encode_workspace_bytes(N, W, H, ncomp, sampling).
 * Four launches (block transform, bit-offset scan, bit packing, byte stuffing); never synchronises, graph-capturable.
 * Calls sharing `workspace` must be ordered by the caller.  Bad shapes, sampling, tables or capacity return
 * LF_ERR_INVALID_ARGUMENT. */
int lf_jpeg_quality_tables(int quality, int ncomp, unsigned short* qtables);  /* HOST: jpeg_set_quality(q, TRUE), q 1..100 */
long long lf_jpeg_encode_bound(int W, int H, int ncomp, int sampling);        /* HOST: worst-case file bytes, 0 = invalid */
size_t lf_jpeg_encode_workspace_bytes(int N, int W, int H, int ncomp, int sampling);   /* HOST: 0 = invalid */
int lf_jpeg_encode(const unsigned char* frames, int N, int W, int H, int ncomp, int sampling, const unsigned short* qtables,
                   unsigned char* out, long long out_cap, long long* out_len, void* workspace, lf_stream_t stream);

/* PNG decode of label maps (csrc/png.cu; replaces Image.open(f).convert('P') of BP/Dataloader/Load_Data_new.py:120-121):
 * a batch of same-size non-interlaced PNGs, 8-bit grayscale or 1/2/4/8-bit palette -> uint8 [N][H][W] holding the gray
 * values or palette indices, bit-identical to Pillow.  The chunks are walked on the host (lanedetection_end2end_b200/png.py),
 * which checks the 2-byte zlib header and fills one LfPngImage per image; the DEFLATE data is inflated, unfiltered and
 * unpacked on the device.  The device blob is LfPngImage[N] followed by each image's zlib stream (its IDAT payloads
 * concatenated; zoff counts from the blob start).
 * lf_png_workspace_bytes (HOST): checks the descriptors, fills rowbytes and raw_off (in place) and returns the scratch
 *   bytes `workspace` needs (0 = invalid descriptors).
 * lf_png_decode: two launches (inflate; unfilter + unpack); a corrupt stream (invalid code or code-length set, distance
 *   before the start of the output, output longer or shorter than H * (1 + rowbytes), stream ending before its final block,
 *   Adler-32 mismatch, filter type above 4) ORs LF_STATUS_PNG_CORRUPT into *status; that image's frame is undefined.
 *   Calls sharing `workspace` must be ordered by the caller. */
#define LF_STATUS_PNG_CORRUPT 16
typedef struct LfPngImage {
    long long zoff;               /* zlib stream (2-byte header, DEFLATE data, Adler-32): blob offset and length */
    int zlen;
    int W, H;
    int depth;                    /* bits per sample: 8 (grayscale or palette) or 1, 2, 4 (palette) */
    /* layout, filled by lf_png_workspace_bytes */
    int rowbytes;                 /* (W * depth + 7) / 8: a scanline is one filter-type byte + rowbytes */
    int reserved;
    long long raw_off;            /* workspace offset of the H * (1 + rowbytes) inflated (still filtered) bytes */
} LfPngImage;
size_t lf_png_workspace_bytes(LfPngImage* images, int N);
int lf_png_decode(const void* blob, int N, int W, int H, unsigned char* out, int* status, void* workspace, size_t workspace_bytes,
                  lf_stream_t stream);

/* Label-map transform of the reference loader (csrc/input_pipe.cu; BP/Dataloader/Load_Data_new.py:129,131,160-184): uint8
 * maps [N][Hin][Win] -> int64 [N][1][Ho][Wo] = the collated `gt`.  Row oy of the output reads source row crop_y0 + ys[oy],
 * column ox reads xs[ox] (Pillow's NEAREST resize, tables from input_pipeline.nearest_table).  nclasses < 3 turns 3 and 4
 * into 0.  A flipped image (flip[n] != 0; flip may be NULL) is mirrored with 1 and 2 swapped, and then every pixel where the
 * UNFLIPPED resized map held 3 / 4 is set to 4 / 3, as the reference does (its masks are taken before the flip). */
int lf_label_preprocess(const unsigned char* maps, int N, int Hin, int Win, int crop_y0, const int* xs, const int* ys, int Ho,
                        int Wo, int nclasses, const unsigned char* flip, long long* out, lf_stream_t stream);

/* TuSimple test-set scoring of one batch (csrc/tusimple.cu; replaces the lane gating of BP/test.py:66-89 and
 * LaneEval.bench of BP/eval_lane.py:27-57): one launch, no host synchronisation, graph-capturable.
 *   x_cal [B][P][S] f64: Projections.compute_all's output (1280-wide pixels); line_pred [B][4] f32: the rounded sigmoid in the
 *   head's order (the launch applies the reference's [1, 2, 0, 3] permutation; needs P == 4), or NULL; horizon_pred [B] int32
 *   (720p rows), or NULL.
 *   Ground-truth table of the whole file (N rows, table width G <= LF_TUSIMPLE_MAX_GT lanes): gt_x [N][G][S] int32,
 *   gt_lanes [N] (lanes per row), thresh [N][G] f64 (20 / cos(arctan(k)) of each lane, LaneEval.get_angle's value).
 *   pos: device int32, the file row of slot 0.  Rows pos .. min(pos + B, N) - 1 are scored; *pos += B afterwards.
 *   lanes [N][P][S] int32: the gated, rounded lanes the reference writes into its JSON (-2 = no point; a NaN becomes -2);
 *   per_image [N][3] f64: (accuracy, fp, fn) of each row as LaneEval.bench returns them, bit-identical. */
#define LF_TUSIMPLE_MAX_GT 8
#define LF_TUSIMPLE_MAX_S 64
int lf_tusimple_score(const double* x_cal, const float* line_pred, const int* horizon_pred, int B, int P, int S, const int* gt_x,
                      const int* gt_lanes, const double* thresh, int N, int G, int* pos, int* lanes, double* per_image,
                      lf_stream_t stream);

/* The bird's-eye-view validation score of one batch (csrc/tusimple.cu; write_lsq_results(..., all_branches_ready=False,
 * horizon_on=False) of BEV/Dataloader/Load_Data_new.py:335-410 and LaneEval.bench of BEV/eval_lane.py, as
 * BEV/main.py:445-488 run them): one launch, no host synchronisation, graph-capturable.
 *   beta [B][4][3] f32: each image's fitted coefficients (a, b, c) per lane; rows [B] int64: each image's validation row;
 *   status: device int32, the batch's LSQ status word; pos: device int64, the visit slot of image 0 (image b's results go
 *   to slot *pos + b; slots >= V are not written; *pos is not changed).  warp: HOST [18] f64, M then M^-1 row-major (cv2's
 *   getPerspectiveTransform of the normalised trapezoid, as write_lsq_results builds them); no_ortho != 0 samples the
 *   curve in the image plane instead.
 *   Ground-truth table of the validation file (N rows, table width G lanes, 4 <= G <= LF_TUSIMPLE_MAX_GT; every row has at
 *   least 4 lanes): gt_S [N] samples per row (<= LF_TUSIMPLE_MAX_S), h_samples [N][LF_TUSIMPLE_MAX_S] int32, gt_x
 *   [N][G][LF_TUSIMPLE_MAX_S] int32, gt_lanes [N], thresh [N][G] f64 (LaneEval.get_angle's threshold of each lane).
 *   Per visit slot (V slots): lanes [V][4][LF_TUSIMPLE_MAX_S] int64: the sampled columns write_lsq_results writes
 *   (np.int_(np.round(x * 1279)), -2 outside a lane's labelled rows, every float64 step in the host formula's order without
 *   FMA contraction; NaN and values beyond int64 give INT64_MIN as numpy does on x86-64); per_row [V][3] f64:
 *   LaneEval.bench's (accuracy, fp, fn) of the slot's row, bit-identical; scored [V] int32: 1 when the status word was 0,
 *   else 0. */
int lf_bev_lane_score(const float* beta, const long long* rows, const int* status, const long long* pos, int B, int no_ortho,
                      const double* warp, const int* gt_S, const int* h_samples, const int* gt_x, const int* gt_lanes,
                      const double* thresh, int N, int G, long long V, long long* lanes, double* per_row, int* scored,
                      lf_stream_t stream);

/* The predicted points drawn onto the test frames (csrc/tusimple.cu; the cv2.circle loop of BP/test.py:115-119):
 * frames uint8 [N][H][W][3] in place; lanes [N][L][S] int32 (-2 = no point) at rows h_samples [N][S] int32; colors: HOST
 * uint8 [L][3], the colour of each lane.  Every point is stamped with cv2.circle(img, (x, y), radius, color, thickness=-1)'s
 * pixels (LINE_8, shift 0; the stamp's spans are computed on the host), clipped at the frame borders; where stamps overlap
 * the pixel takes the colour of the last one in the reference's order (lane by lane, point by point).  One launch. */
#define LF_DRAW_MAX_LANES 8
#define LF_DRAW_MAX_RADIUS 16
int lf_draw_lane_points(unsigned char* frames, int N, int H, int W, const int* lanes, int L, int S, const int* h_samples,
                        const unsigned char* colors, int radius, lf_stream_t stream);

/* The TuSimple loader's device cache (csrc/loader.cu; Dataloader/Load_Data_new.py of this package, replacing the per-sample
 * work of BP/Dataloader/Load_Data_new.py:110-197 after decoding).  A cache is two slot-addressed uint8 buffers of resized,
 * UNFLIPPED samples: frames [S][Ho][Wo][3] and label maps [S][Ho][Wo].
 * lf_loader_stage: frames uint8 [N][Hin][Win][3] (decoded RGB) and maps uint8 [N][Hin][Win] (decoded label maps; NULL =
 *   frames only, for a test set) -> rows [crop_y0, crop_y0+crop_rows) -> frame n into cache_frames[slots[n]] by Pillow's
 *   BILINEAR (xb/xk/yb/yk as lf_frame_preprocess takes them) and map n into cache_maps[slots[n]] by Pillow's NEAREST (xs/ys
 *   as lf_label_preprocess takes them).  slots: device int32 [N].  One launch; bit-identical to what lf_frame_preprocess /
 *   lf_label_preprocess read before their flip.
 * lf_loader_assemble: one collated batch, one launch.  sample: device int32 [N][3] = (slot, table row, flip).
 *   image [N][3][Ho][Wo] f32 = cache_frames / 255 (__fdiv_rn, ToTensor's value), mirrored when flip != 0;
 *   gt [N][1][Ho][Wo] int64 = the class rules of lf_label_preprocess (nclasses, flip, the 3 / 4 quirk) on the cached map;
 *   per-row tables over nrows rows, flip state f = (flip != 0):
 *     lanes [N][4][56] f64 = lanes_tab[f][row]   (lanes_tab [2][nrows][4][56])
 *     valid [N][4][56] f64 = valid_tab[row]      (valid_tab [nrows][4][56]: not flipped, as the reference leaves it)
 *     horizon [N][Ho] f32 = 1 for y < horizon_tab[row], else 0 (horizon_tab [nrows] int32)
 *     line [N][4] f32 = line_tab[f][row]         (line_tab [2][nrows][4])
 *   Every output may be NULL (not written); the tables and caches an output needs must not be.  Needs Ho * Wo >= 224. */
#define LF_LOADER_LANES 4
#define LF_LOADER_POINTS 56
int lf_loader_stage(const unsigned char* frames, const unsigned char* maps, int N, int Hin, int Win, int crop_y0, int crop_rows,
                    const int* xb, const int* xk, int kx, const int* yb, const int* yk, int ky, const int* xs, const int* ys, int Ho,
                    int Wo, const int* slots, unsigned char* cache_frames, unsigned char* cache_maps, lf_stream_t stream);
int lf_loader_assemble(const unsigned char* cache_frames, const unsigned char* cache_maps, int N, int Ho, int Wo, int nclasses,
                       const int* sample, int nrows, const double* lanes_tab, const double* valid_tab, const int* horizon_tab,
                       const float* line_tab, float* image, long long* gt, double* lanes, double* valid, float* horizon, float* line,
                       lf_stream_t stream);

/* The bird's-eye-view loader on the same cache (csrc/loader.cu; bev/Dataloader/Load_Data_new.py of this package, replacing
 * the per-sample work of BEV/Dataloader/Load_Data_new.py:77-112 after decoding).
 * lf_loader_label_rows: for each of N staged maps, cache_maps[slots[n]] -> first_row[positions[n]] = the first row holding a
 *   value outside {0, 3, 4}, or -1 if there is none (the horizon of the reference's gt.nonzero()[0, 1]; a flip does not move
 *   rows).  slots, positions: device int32 [N]; first_row: device int32 indexed by table row.  One CTA per map.
 * lf_loader_assemble_bev: one collated batch, one launch.  sample: device int32 [N][3] = (slot, table row, flip).
 *   image [N][3][Ho][Wo] f32 as lf_loader_assemble;
 *   gt [N][1][Ho][Wo] int64 = the cached map (mirrored when flip != 0) with 3 and 4 -> 0, then 1 <-> 2 when flip != 0;
 *   per-row tables over nrows rows, flip state f = (flip != 0):
 *     params [N][4][3] f32 = params_tab[f][row]  (params_tab [2][nrows][4][3])
 *     line [N][4] int64 = line_tab[f][row]       (line_tab [2][nrows][4])
 *     horizon [N][Ho] f32 = 1 for y < first_row[row], else 0
 *   Every pointer is required.  Needs Ho * Wo >= 12. */
#define LF_LOADER_BEV_COEFFS 3
int lf_loader_label_rows(const unsigned char* cache_maps, int N, int Ho, int Wo, const int* slots, const int* positions, int* first_row,
                         lf_stream_t stream);
int lf_loader_assemble_bev(const unsigned char* cache_frames, const unsigned char* cache_maps, int N, int Ho, int Wo,
                           const int* sample, int nrows, const float* params_tab, const long long* line_tab, const int* first_row,
                           float* image, long long* gt, float* params, long long* line, float* horizon, lf_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LANEFIT_B200_H */
