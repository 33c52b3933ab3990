// TuSimple test-set scoring of one batch in one launch (replaces BP/test.py:66-99 and LaneEval.bench of
// BP/eval_lane.py:27-57 for the rows of that batch):
//
//   gate   lane j -> -2 when 1 - line_pred[perm[j]] != 0 (perm = [1, 2, 0, 3]); the first max(int((h - 160) / 10), 0)
//          samples -> -2; values > 1279 or < 0 -> -2 (before rounding); the rest rounded half to even (np.round)
//   score  per ground-truth lane g: max over predictions p of the line accuracy (#samples with |p' - g'| < thresh[g]) / S,
//          where a negative sample counts as -100; matched when >= 0.85.  (a, fp, fn) as LaneEval.bench forms them, the
//          lane sum sequential in lane order, float64.
//
// The ground-truth angle thresholds depend on the ground truth alone and come in precomputed (inference.TuSimpleScorer,
// bit-identical to LaneEval.get_angle); everything here is integer counting, compares and a few float64 additions and
// divisions, so the result equals LaneEval's bit for bit.  One CTA per launch, one warp per image: a latency-bound launch.
// The batch covers file rows pos .. pos + B - 1; rows >= N are not scored, and the launch advances *pos by B so a
// captured graph can be replayed once per batch.
//
// lf_draw_lane_points stamps the predicted points onto the test frames as BP/test.py:115-119 does with cv2.circle(...,
// thickness=-1): one CTA per frame; each (point, stamp pixel) pair writes its lane's colour unless a later point in the
// drawing order (lane by lane, point by point) also covers the pixel, so every pixel is written at most once and the last
// stamp wins without ordering the writes.
#include <climits>

#include "lf_common.cuh"

namespace lf {

constexpr int TS_WARPS = 8;
constexpr int TS_MAXP = 4;      // predicted lanes (the reference's 4-lane --clas model)

// LaneEval.bench of one row (eval_lane.py:27-57), called by a whole warp: one thread per (ground-truth lane, prediction)
// pair counts the samples with |p' - g'| < thresh[g] (a negative value counts as -100; the difference and its absolute
// value wrap as numpy's int64 do), then lane 0 forms (accuracy, fp, fn) with LaneEval's float64 operations in its order.
// pred [P][S] (the warp's gated lanes), gx [g_n][gs] (the row's ground-truth columns, lane stride gs), th [g_n].
template <typename T>
__device__ void lane_eval_row(const T* pred, int P, int S, const int* __restrict__ gx, int gs, const double* __restrict__ th,
                              int g_n, double* s_acc, int lane, double* r) {
    const bool early = g_n + 2 < P;           // LaneEval's early return (0, 0, 1)
    if (!early && lane < g_n * P) {
        const int g = lane / P, p = lane - g * P;
        const int* gl = gx + (size_t)g * gs;
        const double t = th[g];
        int cnt = 0;
        for (int s = 0; s < S; ++s) {
            const long long pv = pred[p * S + s] >= 0 ? (long long)pred[p * S + s] : -100;
            const long long gv = gl[s] >= 0 ? gl[s] : -100;
            const unsigned long long d = (unsigned long long)pv - (unsigned long long)gv;
            const long long ad = (long long)((long long)d < 0 ? 0ull - d : d);
            cnt += (double)ad < t ? 1 : 0;
        }
        s_acc[lane] = (double)cnt / (double)S;
    }
    __syncwarp();
    if (lane == 0) {
        if (early) {
            r[0] = 0.0;
            r[1] = 0.0;
            r[2] = 1.0;
        } else {
            double sum = 0.0, mn = 0.0, fn = 0.0, matched = 0.0;
            for (int g = 0; g < g_n; ++g) {
                double m = s_acc[g * P];
                for (int p = 1; p < P; ++p) m = s_acc[g * P + p] > m ? s_acc[g * P + p] : m;
                if (m < 0.85) fn += 1.0;
                else matched += 1.0;
                sum += m;
                mn = (g == 0 || m < mn) ? m : mn;
            }
            const double fp = (double)P - matched;
            if (g_n > 4 && fn > 0.0) fn -= 1.0;
            if (g_n > 4) sum -= mn;
            const double den = fmax(fmin(4.0, (double)g_n), 1.0);
            r[0] = sum / den;
            r[1] = fp / (double)P;
            r[2] = fn / den;
        }
    }
}

__global__ void __launch_bounds__(TS_WARPS * 32) tusimple_score_kernel(
    const double* __restrict__ x_cal, const float* __restrict__ line_pred, const int* __restrict__ horizon_pred, int B, int P,
    int S, const int* __restrict__ gt_x, const int* __restrict__ gt_lanes, const double* __restrict__ thresh, int N, int G,
    int* pos, int* __restrict__ lanes, double* __restrict__ per_image) {
    pdl_entry();
    __shared__ int s_pred[TS_WARPS][TS_MAXP * LF_TUSIMPLE_MAX_S];
    __shared__ double s_acc[TS_WARPS][LF_TUSIMPLE_MAX_GT * TS_MAXP];
    __shared__ long long s_pos;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) s_pos = *pos;
    __syncthreads();
    const long long p0 = s_pos;
    for (int b = warp; b < B; b += TS_WARPS) {
        const long long row = p0 + b;
        if (row < 0 || row >= N) continue;
        // ---- gating (lanes_from_predictions): the same compares on the same float32 / float64 values
        int cut = 0;
        if (horizon_pred) {
            const float bound = (float)(horizon_pred[b] - 160) / 10.0f;     // torch true division of an int32 tensor
            cut = bound >= (float)S ? S : (bound >= 1.0f ? (int)bound : 0);  // max(int(bound), 0), capped by the slice
        }
        unsigned off = 0;       // bit p: lane p switched off by the line-type head
        if (line_pred) {
            const int perm[TS_MAXP] = {1, 2, 0, 3};
#pragma unroll
            for (int p = 0; p < TS_MAXP; ++p)
                if (1.0f - line_pred[(size_t)b * TS_MAXP + perm[p]] != 0.0f) off |= 1u << p;
        }
        int* out = lanes + (size_t)row * P * S;
        for (int i = lane; i < P * S; i += 32) {
            const int p = i / S, s = i - p * S;
            double v = x_cal[(size_t)b * P * S + i];
            if (((off >> p) & 1u) || s < cut) v = -2.0;
            // > 1279 or < 0 -> -2; NaN (a singular fit, reported through the LSQ status word) -> -2 as well
            const int q = (v >= 0.0 && v <= 1279.0) ? __double2int_rn(v) : -2;
            out[i] = q;
            s_pred[warp][i] = q;
        }
        __syncwarp();
        lane_eval_row(s_pred[warp], P, S, gt_x + (size_t)row * G * S, S, thresh + (size_t)row * G,
                      min(max(gt_lanes[row], 0), G), s_acc[warp], lane, per_image + (size_t)row * 3);
        __syncwarp();
    }
    __syncthreads();
    if (threadIdx.x == 0) *pos = (int)(p0 + B);
}

struct BevWarp {
    double m11, m12, m21, m22;                   // M: the rows that map a normalised y into the bird's-eye view
    double i00, i01, i02, i20, i21, i22;         // M^-1: the rows that give x and the homogeneous w back in the image
};

// numpy's np.int_ of a rounded float64 on x86-64: NaN and values outside int64 become INT64_MIN
__device__ __forceinline__ long long np_int64_rn(double v) {
    return fabs(v) < 9223372036854775808.0 ? __double2ll_rn(v) : LLONG_MIN;
}

// The validation pass's lane sampling and score (BEV/main.py:445-488): write_lsq_results with all_branches_ready = False
// and horizon_on = False, then LaneEval.bench, for the batch's validation rows.  One warp per image; image b's results go
// to visit slot *pos + b (the caller advances *pos after the launch, so a captured graph can be replayed per batch).
// Every float64 operation is the host formula's, in its order, as an explicit _rn intrinsic so that nothing contracts
// into an FMA.
__global__ void __launch_bounds__(TS_WARPS * 32) bev_lane_score_kernel(
    const float* __restrict__ beta, const long long* __restrict__ rows, const int* __restrict__ status,
    const long long* __restrict__ pos, int B, int no_ortho, const __grid_constant__ BevWarp Wp, const int* __restrict__ gt_S,
    const int* __restrict__ h_samples, const int* __restrict__ gt_x, const int* __restrict__ gt_lanes,
    const double* __restrict__ thresh, int N, int G, long long V, long long* __restrict__ lanes, double* __restrict__ per_row,
    int* __restrict__ scored) {
    pdl_entry();
    constexpr int MS = LF_TUSIMPLE_MAX_S;
    __shared__ long long s_pred[TS_WARPS][TS_MAXP * MS];
    __shared__ double s_acc[TS_WARPS][LF_TUSIMPLE_MAX_GT * TS_MAXP];
    __shared__ int s_lo[TS_WARPS][TS_MAXP], s_hi[TS_WARPS][TS_MAXP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * TS_WARPS + warp;
    if (b >= B) return;
    const long long row = rows[b], slot = *pos + b;
    if (row < 0 || row >= N || slot < 0 || slot >= V) return;
    const int S = gt_S[row];
    const int* hs = h_samples + (size_t)row * MS;
    const int* gx = gt_x + (size_t)row * G * MS;
    // the labelled rows of each lane: points from max(210, min y) to max y are kept; a lane without one stays -2
    if (lane < TS_MAXP) {
        int lo = INT_MAX, hi = INT_MIN;
        for (int s = 0; s < S; ++s)
            if (gx[(size_t)lane * MS + s] != -2) {
                lo = min(lo, hs[s]);
                hi = max(hi, hs[s]);
            }
        s_lo[warp][lane] = hi == INT_MIN ? 1 : max(210, lo);
        s_hi[warp][lane] = hi == INT_MIN ? 0 : hi;
    }
    __syncwarp();
    long long* out = lanes + (size_t)slot * TS_MAXP * MS;
    for (int i = lane; i < TS_MAXP * S; i += 32) {
        const int p = i / S, s = i - p * S;
        const int y = hs[s];
        long long q = -2;
        if (s_lo[warp][p] <= y && y <= s_hi[warp][p]) {
            const double a = beta[((size_t)b * TS_MAXP + p) * 3], bb = beta[((size_t)b * TS_MAXP + p) * 3 + 1],
                         c = beta[((size_t)b * TS_MAXP + p) * 3 + 2];
            const double yd = __ddiv_rn((double)(y - 80), 639.0);
            double x;
            if (no_ortho) {
                const double u = __dadd_rn(1.0, -yd);
                x = __dadd_rn(__dadd_rn(__dmul_rn(a, __dmul_rn(u, u)), __dmul_rn(bb, u)), c);
            } else {
                const double yp = __ddiv_rn(__dadd_rn(__dmul_rn(Wp.m11, yd), Wp.m12), __dadd_rn(__dmul_rn(Wp.m21, yd), Wp.m22));
                const double ye = __dadd_rn(1.0, -yp);
                const double xb = __dadd_rn(__dadd_rn(__dmul_rn(a, __dmul_rn(ye, ye)), __dmul_rn(bb, ye)), c);
                const double tx = __dadd_rn(__dadd_rn(__dmul_rn(Wp.i00, xb), __dmul_rn(Wp.i01, yp)), Wp.i02);
                const double tw = __dadd_rn(__dadd_rn(__dmul_rn(Wp.i20, xb), __dmul_rn(Wp.i21, yp)), Wp.i22);
                x = __ddiv_rn(tx, tw);
            }
            q = np_int64_rn(__dmul_rn(x, 1279.0));
        }
        out[p * MS + s] = q;
        s_pred[warp][p * S + s] = q;
    }
    __syncwarp();
    lane_eval_row(s_pred[warp], TS_MAXP, S, gx, MS, thresh + (size_t)row * G, min(max(gt_lanes[row], 0), G), s_acc[warp],
                  lane, per_row + (size_t)slot * 3);
    if (lane == 0) scored[slot] = *status == 0 ? 1 : 0;
}

struct DrawParams {
    int hw[LF_DRAW_MAX_RADIUS + 1];              // stamp half-width on rows 0..radius from the centre
    unsigned char rgb[LF_DRAW_MAX_LANES][3];
};

constexpr int DRAW_OFF = INT_MIN;                // no point, or a point whose stamp misses the frame

__global__ void __launch_bounds__(256) draw_lane_points_kernel(uint8_t* __restrict__ frames, int H, int W, const int* __restrict__ lanes,
                                                               int L, int S, const int* __restrict__ h_samples, int R,
                                                               const __grid_constant__ DrawParams D) {
    pdl_entry();
    __shared__ int s_x[LF_DRAW_MAX_LANES * LF_TUSIMPLE_MAX_S], s_y[LF_DRAW_MAX_LANES * LF_TUSIMPLE_MAX_S];
    const int n = blockIdx.x, np = L * S;
    for (int p = threadIdx.x; p < np; p += blockDim.x) {
        const int x = lanes[(size_t)n * np + p], y = h_samples[(size_t)n * S + p % S];
        const bool off = x == -2 || x < -R || x >= W + R || y < -R || y >= H + R;
        s_x[p] = off ? DRAW_OFF : x;
        s_y[p] = y;
    }
    __syncthreads();
    const int side = 2 * R + 1, box = side * side;
    uint8_t* img = frames + (size_t)n * H * W * 3;
    for (int it = threadIdx.x; it < np * box; it += blockDim.x) {
        const int p = it / box, j = it - p * box;
        if (s_x[p] == DRAW_OFF) continue;
        const int dy = j / side - R, dx = j % side - R;
        if (abs(dx) > D.hw[abs(dy)]) continue;
        const int px = s_x[p] + dx, py = s_y[p] + dy;
        if (px < 0 || px >= W || py < 0 || py >= H) continue;
        bool later = false;
        for (int q = p + 1; q < np && !later; ++q) {
            const int ey = py - s_y[q];
            later = s_x[q] != DRAW_OFF && abs(ey) <= R && abs(px - s_x[q]) <= D.hw[abs(ey)];
        }
        if (later) continue;
        uint8_t* o = img + ((size_t)py * W + px) * 3;
        const unsigned char* c = D.rgb[p / S];
        o[0] = c[0];
        o[1] = c[1];
        o[2] = c[2];
    }
}

}  // namespace lf

using namespace lf;

// Half-widths of cv2's filled integer circle (drawing.cpp Circle with fill, LINE_8, shift 0): the midpoint loop emits
// spans on rows cy -+ dy (x within dx) and cy -+ dx (x within dy); the stamp is their union.
static void circle_halfwidths(int R, int* hw) {
    for (int i = 0; i <= R; ++i) hw[i] = -1;
    int err = 0, dx = R, dy = 0, plus = 1, minus = (R << 1) - 1;
    while (dx >= dy) {
        hw[dy] = hw[dy] > dx ? hw[dy] : dx;
        hw[dx] = hw[dx] > dy ? hw[dx] : dy;
        ++dy;
        err += plus;
        plus += 2;
        const int mask = (err <= 0) - 1;
        err -= minus & mask;
        dx += mask;
        minus -= mask & 2;
    }
}

extern "C" int lf_draw_lane_points(unsigned char* frames, int N, int H, int W, const int* lanes, int L, int S, const int* h_samples,
                                   const unsigned char* colors, int radius, lf_stream_t stream_) {
    LF_REQUIRE(frames && lanes && h_samples && colors && N >= 1 && H >= 1 && W >= 1);
    LF_REQUIRE(L >= 1 && L <= LF_DRAW_MAX_LANES && S >= 1 && S <= LF_TUSIMPLE_MAX_S && radius >= 0 && radius <= LF_DRAW_MAX_RADIUS);
    DrawParams D;
    circle_halfwidths(radius, D.hw);
    for (int l = 0; l < L; ++l)
        for (int k = 0; k < 3; ++k) D.rgb[l][k] = colors[l * 3 + k];
    lf_launch(draw_lane_points_kernel, dim3(N), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream_), frames, H, W, lanes, L, S,
              h_samples, radius, D);
    return check_launch();
}

extern "C" int lf_tusimple_score(const double* x_cal, const float* line_pred, const int* horizon_pred, int B, int P, int S,
                                 const int* gt_x, const int* gt_lanes, const double* thresh, int N, int G, int* pos, int* lanes,
                                 double* per_image, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(x_cal && gt_x && gt_lanes && thresh && pos && lanes && per_image);
    LF_REQUIRE(B > 0 && P >= 1 && P <= TS_MAXP && S >= 1 && S <= LF_TUSIMPLE_MAX_S && N > 0 && G >= 1 && G <= LF_TUSIMPLE_MAX_GT);
    LF_REQUIRE(!line_pred || P == TS_MAXP);
    lf_launch(tusimple_score_kernel, 1, TS_WARPS * 32, 0, stream, x_cal, line_pred, horizon_pred, B, P, S, gt_x, gt_lanes, thresh,
              N, G, pos, lanes, per_image);
    return check_launch();
}

extern "C" int lf_bev_lane_score(const float* beta, const long long* rows, const int* status, const long long* pos, int B,
                                 int no_ortho, const double* warp, const int* gt_S, const int* h_samples, const int* gt_x,
                                 const int* gt_lanes, const double* thresh, int N, int G, long long V, long long* lanes,
                                 double* per_row, int* scored, lf_stream_t stream_) {
    LF_REQUIRE(beta && rows && status && pos && warp && gt_S && h_samples && gt_x && gt_lanes && thresh && lanes && per_row &&
               scored);
    LF_REQUIRE(B > 0 && N > 0 && V > 0 && G >= TS_MAXP && G <= LF_TUSIMPLE_MAX_GT);
    BevWarp Wp;
    Wp.m11 = warp[4], Wp.m12 = warp[5], Wp.m21 = warp[7], Wp.m22 = warp[8];
    Wp.i00 = warp[9], Wp.i01 = warp[10], Wp.i02 = warp[11], Wp.i20 = warp[15], Wp.i21 = warp[16], Wp.i22 = warp[17];
    lf_launch(bev_lane_score_kernel, dim3((B + TS_WARPS - 1) / TS_WARPS), dim3(TS_WARPS * 32), 0,
              reinterpret_cast<cudaStream_t>(stream_), beta, rows, status, pos, B, no_ortho, Wp, gt_S, h_samples, gt_x, gt_lanes,
              thresh, N, G, V, lanes, per_row, scored);
    return check_launch();
}
