// Multi-tensor optimizer update (Adam / SGD / RMSprop with torch.optim's semantics) in one launch
// (include/lanefit_b200.h: lf_optim_step).
//
//  * Work unit = a chunk of LF_OPTIM_CHUNK elements of one segment (parameter tensor); CTAs stride over the chunks, and a
//    chunk finds its segment by binary search over the rows' chunk0.  Chunks partition every segment, so each element is
//    read and written by exactly one thread.
//  * The update is memory bound (Adam: 28 B per element), so a chunk whose four pointers are 16-byte aligned moves float4s;
//    any other chunk (a gradient view at an odd offset into the flat all-reduce buffer) runs the same arithmetic on
//    scalars.  The elementwise arithmetic is identical in both paths.
//  * Thread 0 forms the scalars (bias corrections, fp64 like torch's host code, then rounded to fp32) once per CTA from
//    the device hyperparameter block and step counter, so a CUDA graph replay picks up a new learning rate without a
//    recapture.  The step counter is advanced by the last CTA to arrive (ticket, as in lsq.cu): every CTA reads it before
//    taking its ticket, so no CTA can see the advanced value.
//  * lf_optim_step_pp keeps one step count per parameter (torch's per-parameter `step`): a first launch with one thread
//    per row forms that row's scalars from its own count and advances the count, a second runs the same chunk loop with
//    each chunk's row scalars.  opt_scalars / opt_elem / opt_chunk are shared, so the arithmetic is the same code.
//  * Gradient clipping by the global L2 norm (lf_grad_norm, then lf_optim_step_clip / lf_optim_step_pp_clip): the norm
//    launch runs over the same table and chunks, one fp64 partial per chunk, summed by the last CTA in a fixed order, so
//    the norm is bit-identical from run to run whatever the grid size or the load path.  The clipped update is the same
//    template with CLIP set: one __fmul_rn by the coefficient before opt_elem's arithmetic, and the non-finite flag
//    skips the launch as the status word does.
#include <vector>

#include "lf_common.cuh"

namespace lf {

constexpr int OPT_THREADS = 256;

// fp32 scalars of one launch.  a = beta2 (Adam) or alpha (RMSprop), c = 1 - a, w = 1 - beta1 (Adam's lerp weight),
// lr = lr / (1 - beta1^t) for Adam (torch's step_size), bc2 = sqrt(1 - beta2^t), mu = momentum.
struct OptScalars {
    float lr, a, c, w, bc2, eps, wd, mu;
    int first;                          // SGD: no momentum buffer yet
    int lerp_small;                     // Adam: |w| < 0.5 selects ATen's first lerp formula
};

__device__ __noinline__ void opt_scalars(int algo, const LfOptimHyper* h, long long step, OptScalars* s) {
    const double t = (double)(step + 1);
    s->wd = (float)h->weight_decay;
    s->eps = (float)h->eps;
    s->mu = (float)h->momentum;
    s->a = (float)h->beta2;
    s->c = (float)(1.0 - h->beta2);
    s->first = step == 0;
    const double w = 1.0 - h->beta1;
    s->w = (float)w;
    s->lerp_small = fabs(w) < 0.5;
    s->lr = algo == LF_OPTIM_ADAM ? (float)(h->lr / (1.0 - pow(h->beta1, t))) : (float)h->lr;
    s->bc2 = (float)sqrt(1.0 - pow(h->beta2, t));
}

// Every operation is an explicit round-to-nearest intrinsic, so nvcc cannot contract or reorder anything.  A fused
// multiply-add appears exactly where torch's CUDA kernels form `a + s*b` as one: the alpha forms of add_ (weight decay,
// the parameter update), lerp_, and addcmul_ / addcdiv_ (ATen's pointwise_op_impl calls fma explicitly).
template <int ALGO, bool CLIP>
__device__ __forceinline__ void opt_elem(float& p, float g, float& s0, float& s1, const OptScalars& s, float coef) {
    if (CLIP) g = __fmul_rn(g, coef);                                             // torch._foreach_mul_(grads, clip_coef)
    if (s.wd != 0.f) g = __fmaf_rn(s.wd, p, g);                                   // grad.add(p, alpha=wd)
    if (ALGO == LF_OPTIM_ADAM) {
        // exp_avg.lerp_(g, 1-b1): self + w (end - self) for |w| < 0.5, else end - (end - self)(1 - w)
        s0 = s.lerp_small ? __fmaf_rn(s.w, __fsub_rn(g, s0), s0) : __fmaf_rn(-__fsub_rn(g, s0), __fsub_rn(1.f, s.w), g);
        s1 = __fmaf_rn(s.c, __fmul_rn(g, g), __fmul_rn(s1, s.a));               // mul_(b2).addcmul_(g, g, 1-b2)
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(s1), s.bc2), s.eps);
        p = __fmaf_rn(-s.lr, __fdiv_rn(s0, denom), p);                           // addcdiv_(m, denom, -step_size)
    } else if (ALGO == LF_OPTIM_SGD) {
        s0 = s.first ? g : __fadd_rn(__fmul_rn(s0, s.mu), g);                   // mul_(mu).add_(g)
        p = __fmaf_rn(-s.lr, s0, p);                                             // add_(buf, alpha=-lr)
    } else {
        s0 = __fmaf_rn(s.c, __fmul_rn(g, g), __fmul_rn(s0, s.a));               // mul_(alpha).addcmul_(g, g, 1-alpha)
        const float avg = __fadd_rn(__fsqrt_rn(s0), s.eps);
        s1 = __fadd_rn(__fmul_rn(s1, s.mu), __fdiv_rn(g, avg));                 // mul_(mu).addcdiv_(g, avg): value 1
        p = __fmaf_rn(-s.lr, s1, p);                                             // add_(buf, alpha=-lr)
    }
}

template <int ALGO, bool CLIP>
__device__ __forceinline__ void opt_chunk(const LfOptimSeg& sg, long long base, int n, const OptScalars& s, float coef) {
    float* p = sg.param + base;
    const float* g = sg.grad + base;
    float* s0 = sg.state0 + base;
    float* s1 = ALGO == LF_OPTIM_SGD ? nullptr : sg.state1 + base;
    const uintptr_t align = reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(s0) |
                            reinterpret_cast<uintptr_t>(s1);
    int i0 = 0;
    if ((align & 15) == 0) {
        const int n4 = n >> 2;
        for (int i = threadIdx.x; i < n4; i += OPT_THREADS) {
            float4 vp = reinterpret_cast<float4*>(p)[i];
            const float4 vg = __ldg(reinterpret_cast<const float4*>(g) + i);
            float4 v0 = reinterpret_cast<float4*>(s0)[i];
            float4 v1 = ALGO == LF_OPTIM_SGD ? make_float4(0.f, 0.f, 0.f, 0.f) : reinterpret_cast<float4*>(s1)[i];
            opt_elem<ALGO, CLIP>(vp.x, vg.x, v0.x, v1.x, s, coef);
            opt_elem<ALGO, CLIP>(vp.y, vg.y, v0.y, v1.y, s, coef);
            opt_elem<ALGO, CLIP>(vp.z, vg.z, v0.z, v1.z, s, coef);
            opt_elem<ALGO, CLIP>(vp.w, vg.w, v0.w, v1.w, s, coef);
            reinterpret_cast<float4*>(p)[i] = vp;
            reinterpret_cast<float4*>(s0)[i] = v0;
            if (ALGO != LF_OPTIM_SGD) reinterpret_cast<float4*>(s1)[i] = v1;
        }
        i0 = n4 << 2;
    }
    for (int i = i0 + threadIdx.x; i < n; i += OPT_THREADS) {
        float vp = p[i], v0 = s0[i], v1 = ALGO == LF_OPTIM_SGD ? 0.f : s1[i];
        opt_elem<ALGO, CLIP>(vp, __ldg(g + i), v0, v1, s, coef);
        p[i] = vp;
        s0[i] = v0;
        if (ALGO != LF_OPTIM_SGD) s1[i] = v1;
    }
}

__device__ __forceinline__ const LfOptimSeg& row_seg(const LfOptimSeg& r) { return r; }
__device__ __forceinline__ const LfOptimSeg& row_seg(const LfOptimSegPP& r) { return r.seg; }

// the last row with chunk0 <= c
template <typename Row>
__device__ __forceinline__ int find_row(const Row* segs, int nsegs, long long c) {
    int lo = 0, hi = nsegs - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(&row_seg(segs[mid]).chunk0) <= c) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// CLIP: every gradient element is first scaled by clip->clip_coef (lf_grad_norm's), and a set clip->nonfinite skips
// the launch as a nonzero status does.  Without it the launch is the unclipped one, bit for bit.
template <int ALGO, bool CLIP>
__global__ void __launch_bounds__(OPT_THREADS) optim_kernel(const LfOptimSeg* __restrict__ segs, int nsegs, long long nchunks,
                                                            const LfOptimHyper* __restrict__ hyper, LfOptimState* state,
                                                            const int* __restrict__ status, LfGradClip* clip) {
    pdl_entry();
    __shared__ OptScalars sc;
    __shared__ long long step_read;
    __shared__ float coef;
    __shared__ int skip;
    if (threadIdx.x == 0) {
        const int bad = status != nullptr && *status != 0;
        skip = bad || (CLIP && clip->nonfinite != 0);
        if (!skip) {
            step_read = state->step;
            opt_scalars(ALGO, hyper, step_read, &sc);
            coef = CLIP ? clip->clip_coef : 1.f;
        } else if (blockIdx.x == 0) {
            state->skipped += 1;
            if (CLIP && !bad) clip->nonfinite_skipped += 1;
        }
    }
    __syncthreads();
    if (skip) return;    // every CTA reads the same words: none takes a ticket, the counter stays
    const OptScalars s = sc;
    const float k = coef;
    for (long long c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const LfOptimSeg sg = segs[find_row(segs, nsegs, c)];
        const long long base = (c - sg.chunk0) * LF_OPTIM_CHUNK;
        const long long rem = sg.numel - base;
        if (rem > 0) opt_chunk<ALGO, CLIP>(sg, base, rem < LF_OPTIM_CHUNK ? (int)rem : LF_OPTIM_CHUNK, s, k);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long tk = atomicAdd(&state->ticket, 1ull);
        if (tk == gridDim.x - 1) {
            state->ticket = 0;                // leave the block reusable
            state->step = step_read + 1;
        }
    }
}

// ---- per-parameter step counts (lf_optim_step_pp) -------------------------------------------------------------------
static_assert(sizeof(OptScalars) <= LF_OPTIM_PP_SCALAR_BYTES, "LF_OPTIM_PP_SCALAR_BYTES too small");
constexpr int OPT_PP_SCALAR_THREADS = 128;

// launch 1: row r's scalars from its own count, then the count advances.  Rows name distinct slots (checked on the
// host), so no two threads touch one count.  `clip` NULL: unclipped; else a set clip->nonfinite skips as the status does.
__global__ void __launch_bounds__(OPT_PP_SCALAR_THREADS) optim_pp_scalars_kernel(
    int algo, const LfOptimSegPP* __restrict__ segs, int nsegs, const LfOptimHyper* __restrict__ hyper, long long* steps,
    OptScalars* __restrict__ scal, long long* skipped, const int* __restrict__ status, LfGradClip* clip) {
    pdl_entry();
    const int r = blockIdx.x * OPT_PP_SCALAR_THREADS + threadIdx.x;
    if (r >= nsegs) return;
    const int bad = status != nullptr && *status != 0;
    if (bad || (clip != nullptr && clip->nonfinite != 0)) {
        if (r == 0) {
            *skipped += 1;
            if (!bad) clip->nonfinite_skipped += 1;
        }
        return;
    }
    const int slot = segs[r].slot;
    const long long t = steps[slot];
    opt_scalars(algo, hyper, t, scal + r);
    steps[slot] = t + 1;
}

// launch 2: optim_kernel's chunk loop with each chunk's row scalars; no ticket, no count
template <int ALGO, bool CLIP>
__device__ __forceinline__ void optim_pp_chunks(const LfOptimSegPP* __restrict__ segs, int nsegs, long long nchunks,
                                                const OptScalars* __restrict__ scal, const int* __restrict__ status,
                                                const LfGradClip* clip) {
    if (status != nullptr && *status != 0) return;     // every thread reads the words launch 1 read
    if (CLIP && clip->nonfinite != 0) return;
    const float k = CLIP ? clip->clip_coef : 1.f;
    for (long long c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const int lo = find_row(segs, nsegs, c);
        const LfOptimSeg sg = segs[lo].seg;
        const OptScalars s = scal[lo];
        const long long base = (c - sg.chunk0) * LF_OPTIM_CHUNK;
        const long long rem = sg.numel - base;
        if (rem > 0) opt_chunk<ALGO, CLIP>(sg, base, rem < LF_OPTIM_CHUNK ? (int)rem : LF_OPTIM_CHUNK, s, k);
    }
}

template <int ALGO>
__global__ void __launch_bounds__(OPT_THREADS) optim_pp_kernel(const LfOptimSegPP* __restrict__ segs, int nsegs,
                                                               long long nchunks, const OptScalars* __restrict__ scal,
                                                               const int* __restrict__ status) {
    pdl_entry();
    optim_pp_chunks<ALGO, false>(segs, nsegs, nchunks, scal, status, nullptr);
}

template <int ALGO>
__global__ void __launch_bounds__(OPT_THREADS) optim_pp_clip_kernel(const LfOptimSegPP* __restrict__ segs, int nsegs,
                                                                    long long nchunks, const OptScalars* __restrict__ scal,
                                                                    const int* __restrict__ status, const LfGradClip* clip) {
    pdl_entry();
    optim_pp_chunks<ALGO, true>(segs, nsegs, nchunks, scal, status, clip);
}

// ---- global L2 norm of the gradients (lf_grad_norm) -----------------------------------------------------------------
constexpr int NORM_GROUPS = LF_OPTIM_CHUNK / (4 * OPT_THREADS);     // groups of four elements per thread and chunk
static_assert(LF_OPTIM_CHUNK % (4 * OPT_THREADS) == 0, "a chunk is a whole number of float4 groups per thread");

// Sum over the CTA of one fp64 value per thread, in a fixed order (xor butterfly in each warp, then the warps in order);
// the result is valid in thread 0.  red: OPT_THREADS / 32 entries of shared memory, reusable when this returns.
__device__ __forceinline__ double cta_sum_fixed(double v, double* red) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 0; w < OPT_THREADS / 32; ++w) t = __dadd_rn(t, red[w]);
    }
    __syncthreads();
    return t;
}

// Sum of squares of one chunk's n gradient elements in an order set by the chunk alone: thread t takes the groups
// q = t + j * OPT_THREADS (j ascending) of four consecutive elements, each group's elements in order, and the CTA sum is
// fixed.  A group that lies inside the chunk is one float4 load when the gradient is 16-byte aligned and four scalar
// loads otherwise; missing elements of the chunk's last group count as 0 (adding +0 changes no sum), so both paths sum
// the same values in the same order.  Each square of an fp32 value is exact in fp64.
__device__ __forceinline__ double chunk_sumsq(const float* g, int n, bool vec, double* red) {
    float v[NORM_GROUPS][4];
#pragma unroll
    for (int j = 0; j < NORM_GROUPS; ++j) {
        const int e = 4 * (threadIdx.x + j * OPT_THREADS);
        if (vec && e + 4 <= n) {
            const float4 x = __ldg(reinterpret_cast<const float4*>(g + e));
            v[j][0] = x.x;
            v[j][1] = x.y;
            v[j][2] = x.z;
            v[j][3] = x.w;
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) v[j][i] = e + i < n ? __ldg(g + e + i) : 0.f;
        }
    }
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < NORM_GROUPS; ++j) {
#pragma unroll
        for (int i = 0; i < 4; ++i) acc = __fma_rn((double)v[j][i], (double)v[j][i], acc);
    }
    return cta_sum_fixed(acc, red);
}

// One fp64 partial per chunk into `partial`; the last CTA to arrive (ticket) sums the partials in a fixed order and
// writes the norm, the clip coefficient and the non-finite flag.  Every sum's order is set by the table alone, so the
// result does not depend on the grid size.
template <typename Row>
__global__ void __launch_bounds__(OPT_THREADS) grad_norm_kernel(const Row* __restrict__ segs, int nsegs, long long nchunks,
                                                                LfGradClip* clip, double* partial) {
    pdl_entry();
    __shared__ double red[OPT_THREADS / 32];
    __shared__ int last;
    for (long long c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const LfOptimSeg sg = row_seg(segs[find_row(segs, nsegs, c)]);
        const long long base = (c - sg.chunk0) * LF_OPTIM_CHUNK;
        const long long rem = sg.numel - base;
        const float* g = sg.grad + base;
        const double s = chunk_sumsq(g, rem <= 0 ? 0 : rem < LF_OPTIM_CHUNK ? (int)rem : LF_OPTIM_CHUNK,
                                     (reinterpret_cast<uintptr_t>(g) & 15) == 0, red);
        if (threadIdx.x == 0) partial[c] = s;
    }
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long tk = atomicAdd(&clip->ticket, 1ull);
        last = tk == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    double acc = 0.0;
    for (long long c = threadIdx.x; c < nchunks; c += OPT_THREADS) acc = __dadd_rn(acc, __ldcg(partial + c));
    const double tot = cta_sum_fixed(acc, red);
    if (threadIdx.x == 0) {
        const float norm = __double2float_rn(__dsqrt_rn(tot));
        // torch.clamp(max_norm / (total_norm + 1e-6), max=1.0) in fp32, where `float / Tensor` is reciprocal() * float
        // and clamp keeps a NaN
        const float coef = __fmul_rn(__fdiv_rn(1.f, __fadd_rn(norm, 1e-6f)), clip->max_norm);
        clip->total_norm = norm;
        clip->clip_coef = coef <= 1.f || coef != coef ? coef : 1.f;
        // the squares are finite and non-negative and fp64 cannot overflow on their sum (below 2^63 * 2^256), so the sum
        // is non-finite exactly when some element is NaN or +-Inf
        clip->nonfinite = !isfinite(tot);
        clip->ticket = 0;                     // leave the block reusable
    }
}

// one wave of resident CTAs (the register count sets how many fit per SM), and no more CTAs than chunks, so every CTA has
// at least one chunk
template <typename... KArgs>
dim3 one_wave(void (*kernel)(KArgs...), long long nchunks) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, OPT_THREADS, 0) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        per_sm = 1;
    }
    const long long cap = (long long)device_sms() * per_sm;
    return dim3((unsigned)(nchunks < cap ? nchunks : cap));
}

template <bool CLIP>
int optim_step(int algo, const LfOptimSeg* segs, int nsegs, long long nchunks, const LfOptimHyper* hyper,
               LfOptimState* state, const int* status, LfGradClip* clip, cudaStream_t stream) {
    LF_REQUIRE(segs && nsegs > 0 && nchunks > 0 && hyper && state && (clip || !CLIP));
    LF_REQUIRE(algo == LF_OPTIM_ADAM || algo == LF_OPTIM_SGD || algo == LF_OPTIM_RMSPROP);
    void (*kernel)(const LfOptimSeg*, int, long long, const LfOptimHyper*, LfOptimState*, const int*, LfGradClip*) =
        algo == LF_OPTIM_ADAM ? optim_kernel<LF_OPTIM_ADAM, CLIP> : algo == LF_OPTIM_SGD ? optim_kernel<LF_OPTIM_SGD, CLIP>
                                                                                      : optim_kernel<LF_OPTIM_RMSPROP, CLIP>;
    lf_launch(kernel, one_wave(kernel, nchunks), OPT_THREADS, 0, stream, segs, nsegs, nchunks, hyper, state, status, clip);
    return check_launch();
}

template <bool CLIP>
int optim_step_pp(int algo, const LfOptimSegPP* segs, const int* slots, int nsegs, long long nchunks,
                  const LfOptimHyper* hyper, long long* steps, int nparams, void* scalars, long long* skipped,
                  const int* status, LfGradClip* clip, cudaStream_t stream) {
    LF_REQUIRE(segs && slots && nsegs > 0 && nchunks > 0 && hyper && steps && nparams > 0 && scalars && skipped &&
               (clip || !CLIP));
    LF_REQUIRE(algo == LF_OPTIM_ADAM || algo == LF_OPTIM_SGD || algo == LF_OPTIM_RMSPROP);
    LF_REQUIRE((reinterpret_cast<uintptr_t>(scalars) & 15) == 0);
    std::vector<char> used(nparams, 0);
    for (int r = 0; r < nsegs; ++r) {
        LF_REQUIRE(slots[r] >= 0 && slots[r] < nparams && !used[slots[r]]);
        used[slots[r]] = 1;
    }
    OptScalars* scal = static_cast<OptScalars*>(scalars);
    lf_launch(optim_pp_scalars_kernel, dim3((nsegs + OPT_PP_SCALAR_THREADS - 1) / OPT_PP_SCALAR_THREADS),
              OPT_PP_SCALAR_THREADS, 0, stream, algo, segs, nsegs, hyper, steps, scal, skipped, status, CLIP ? clip : nullptr);
    const int rc = check_launch();
    if (rc != LF_OK) return rc;
    if (CLIP) {
        void (*kernel)(const LfOptimSegPP*, int, long long, const OptScalars*, const int*, const LfGradClip*) =
            algo == LF_OPTIM_ADAM ? optim_pp_clip_kernel<LF_OPTIM_ADAM>
                                  : algo == LF_OPTIM_SGD ? optim_pp_clip_kernel<LF_OPTIM_SGD> : optim_pp_clip_kernel<LF_OPTIM_RMSPROP>;
        lf_launch(kernel, one_wave(kernel, nchunks), OPT_THREADS, 0, stream, segs, nsegs, nchunks, (const OptScalars*)scal,
                  status, (const LfGradClip*)clip);
    } else {
        void (*kernel)(const LfOptimSegPP*, int, long long, const OptScalars*, const int*) =
            algo == LF_OPTIM_ADAM ? optim_pp_kernel<LF_OPTIM_ADAM>
                                  : algo == LF_OPTIM_SGD ? optim_pp_kernel<LF_OPTIM_SGD> : optim_pp_kernel<LF_OPTIM_RMSPROP>;
        lf_launch(kernel, one_wave(kernel, nchunks), OPT_THREADS, 0, stream, segs, nsegs, nchunks, (const OptScalars*)scal,
                  status);
    }
    return check_launch();
}

template <typename Row>
int grad_norm(const Row* segs, int nsegs, long long nchunks, LfGradClip* clip, void* workspace, size_t workspace_bytes,
              cudaStream_t stream) {
    LF_REQUIRE(segs && nsegs > 0 && nchunks > 0 && clip && workspace);
    LF_REQUIRE(workspace_bytes >= lf_grad_norm_workspace_bytes(nchunks) && (reinterpret_cast<uintptr_t>(workspace) & 7) == 0);
    void (*kernel)(const Row*, int, long long, LfGradClip*, double*) = grad_norm_kernel<Row>;
    lf_launch(kernel, one_wave(kernel, nchunks), OPT_THREADS, 0, stream, segs, nsegs, nchunks, clip,
              static_cast<double*>(workspace));
    return check_launch();
}

}  // namespace lf

using namespace lf;

extern "C" int lf_optim_step(int algo, const LfOptimSeg* segs, int nsegs, long long nchunks, const LfOptimHyper* hyper,
                             LfOptimState* state, const int* status, lf_stream_t stream) {
    return optim_step<false>(algo, segs, nsegs, nchunks, hyper, state, status, nullptr,
                             reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int lf_optim_step_pp(int algo, const LfOptimSegPP* segs, const int* slots, int nsegs, long long nchunks,
                                const LfOptimHyper* hyper, long long* steps, int nparams, void* scalars, long long* skipped,
                                const int* status, lf_stream_t stream) {
    return optim_step_pp<false>(algo, segs, slots, nsegs, nchunks, hyper, steps, nparams, scalars, skipped, status, nullptr,
                                reinterpret_cast<cudaStream_t>(stream));
}

extern "C" size_t lf_grad_norm_workspace_bytes(long long nchunks) {
    return nchunks > 0 ? (size_t)nchunks * sizeof(double) : 0;
}

extern "C" int lf_grad_norm(const LfOptimSeg* segs, int nsegs, long long nchunks, LfGradClip* clip, void* workspace,
                            size_t workspace_bytes, lf_stream_t stream) {
    return grad_norm(segs, nsegs, nchunks, clip, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int lf_grad_norm_pp(const LfOptimSegPP* segs, int nsegs, long long nchunks, LfGradClip* clip, void* workspace,
                               size_t workspace_bytes, lf_stream_t stream) {
    return grad_norm(segs, nsegs, nchunks, clip, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int lf_optim_step_clip(int algo, const LfOptimSeg* segs, int nsegs, long long nchunks, const LfOptimHyper* hyper,
                                  LfOptimState* state, const int* status, LfGradClip* clip, lf_stream_t stream) {
    return optim_step<true>(algo, segs, nsegs, nchunks, hyper, state, status, clip, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int lf_optim_step_pp_clip(int algo, const LfOptimSegPP* segs, const int* slots, int nsegs, long long nchunks,
                                     const LfOptimHyper* hyper, long long* steps, int nparams, void* scalars,
                                     long long* skipped, const int* status, LfGradClip* clip, lf_stream_t stream) {
    return optim_step_pp<true>(algo, segs, slots, nsegs, nchunks, hyper, steps, nparams, scalars, skipped, status, clip,
                               reinterpret_cast<cudaStream_t>(stream));
}
