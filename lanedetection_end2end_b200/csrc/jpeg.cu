// Baseline JPEG decode on the GPU (replaces Image.open(f).convert('RGB') of BP/Dataloader/Load_Data_new.py:118-119),
// bit-identical to Pillow, which decodes through libjpeg-turbo with the ISLOW integer IDCT, "fancy" chroma upsampling and
// fixed-point YCbCr->RGB.  All three are exact integer arithmetic and are restated exactly below.
//
// Launch 1, jpeg_entropy_kernel (one CTA of 1024 threads per image):
//   a. unstuff: drop the FF00 stuffing bytes and the RSTn markers of the entropy-coded segment; every restart interval
//      starts at a multiple of LF_JPEG_PIECE_BYTES in the unstuffed stream, so no piece straddles a restart boundary;
//   b. self-synchronising decode (Weissenberger & Schmidt): the stream is cut into pieces of PBITS bits; a thread decodes
//      its pieces from a guessed state (bit position = piece start, first block of the MCU, zig-zag index 0) and records
//      the exit state (bit position, block of the MCU, zig-zag index, blocks started).  Huffman codes resynchronise,
//      so most exits are already exact; rounds re-decode each thread's first piece from its predecessor's exit until no
//      exit changes.  The fixed point is the sequential decode whatever the guesses; only the number of rounds depends
//      on them.  The first piece of every restart interval starts from its true state (forced sync point);
//   c. a segmented exclusive scan of the blocks started per piece gives each piece its first block index;
//   d. a final pass re-decodes every piece from its true entry and scatters natural-order int16 coefficients;
//   e. a segmented inclusive scan per component, reset at every restart interval, turns DC differences into DC values.
// Launch 2, jpeg_idct_kernel: dequantise + jpeg_idct_islow (jidctint.c) incl. its range-limit table and 10-bit mask,
//   one uint8 plane per component at the component's padded block resolution; clears the coefficients it read.
// Launch 3, jpeg_color_kernel: jdsample.c h2v1 / h2v2 fancy upsampling (plain replication when the chroma component is at
//   most 2 samples wide, as jinit_upsampler chooses) + jdcolor.c ycc_rgb_convert, cropped to W x H.
#include "lf_common.cuh"

namespace lf {

constexpr int JPB = LF_JPEG_PIECE_BYTES;
constexpr unsigned JPBITS = JPB * 8;
constexpr int JT = 1024;   // threads of the entropy kernel

__constant__ unsigned char c_natural[80] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
    6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
    39, 46, 53, 60, 61, 54, 47, 55, 62, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};

// ---- CTA-wide scans (blockDim.x == JT; cta_excl_sum is in lf_common.cuh) ----------------------------------------------
// segmented sum: (f, v) with f = "a segment starts inside"; returns the carry into this thread (sum since the last start)
__device__ __forceinline__ void seg_comb(int& f, int& v, int pf, int pv) {
    if (!f) v += pv;
    f |= pf;
}
__device__ int cta_excl_segsum(int f, int v, int2* sh) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int pf = __shfl_up_sync(0xffffffffu, f, o), pv = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) seg_comb(f, v, pf, pv);
    }
    if (lane == 31) sh[w] = make_int2(f, v);
    __syncthreads();
    if (w == 0) {
        int tf = sh[lane].x, tv = sh[lane].y;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int pf = __shfl_up_sync(0xffffffffu, tf, o), pv = __shfl_up_sync(0xffffffffu, tv, o);
            if (lane >= o) seg_comb(tf, tv, pf, pv);
        }
        sh[lane] = make_int2(tf, tv);
    }
    __syncthreads();
    int ef = __shfl_up_sync(0xffffffffu, f, 1), ev = __shfl_up_sync(0xffffffffu, v, 1);
    if (lane == 0) ef = ev = 0;
    if (w > 0) seg_comb(ef, ev, sh[w - 1].x, sh[w - 1].y);
    __syncthreads();
    return ev;
}

// ---- piece state: bit position [0,32), zig-zag index [32,39), block of the MCU [39,43), error [43], blocks started [44,64)
__device__ __forceinline__ unsigned long long st_pack(unsigned p, int z, int cb, int err, int n) {
    return (unsigned long long)p | ((unsigned long long)z << 32) | ((unsigned long long)cb << 39) |
           ((unsigned long long)err << 43) | ((unsigned long long)n << 44);
}
__device__ __forceinline__ unsigned st_p(unsigned long long s) { return (unsigned)s; }
__device__ __forceinline__ int st_z(unsigned long long s) { return (int)(s >> 32) & 127; }
__device__ __forceinline__ int st_cb(unsigned long long s) { return (int)(s >> 39) & 15; }
__device__ __forceinline__ int st_n(unsigned long long s) { return (int)(s >> 44); }

struct JSmem {
    LfJpegHuff h[8];   // DC tables 0..3, AC tables 4..7
    int dc[LF_JPEG_MAX_BPM], ac[LF_JPEG_MAX_BPM];
    int bpm;
};

__device__ __forceinline__ unsigned bswap32(unsigned x) { return __byte_perm(x, 0, 0x0123); }

// 32 stream bits starting at bit p, most significant first
__device__ __forceinline__ unsigned peek32(const unsigned* __restrict__ words, unsigned p) {
    const unsigned w0 = bswap32(words[p >> 5]), w1 = bswap32(words[(p >> 5) + 1]);
    return __funnelshift_l(w1, w0, p & 31);
}

// one Huffman symbol from the window; returns the code length (0 = invalid code) and the symbol
__device__ __forceinline__ int huff_decode(const LfJpegHuff& t, unsigned win, int& sym) {
    const unsigned look = t.look[win >> 23];
    if (look) {
        sym = look & 0xff;
        return (int)(look >> 8);
    }
    for (int l = 10; l <= 16; ++l) {
        const int code = (int)(win >> (32 - l));
        if (code <= t.maxcode[l]) {
            sym = t.val[(code + t.valoff[l]) & 255];
            return l;
        }
    }
    sym = 0;
    return 0;
}

// Decode from state `st` while the bit position is below min(pend, dend).  Returns the exit state.  WRITE: scatter the
// coefficients of blocks cur in [0, blk_end) (cur = index of the block in progress at entry, relative to the image) into
// coef; an invalid code inside a real block sets *bad.
template <bool WRITE>
__device__ unsigned long long decode_piece(const unsigned* __restrict__ words, unsigned long long st, unsigned pend, unsigned dend,
                                           const JSmem& sm, int16_t* __restrict__ coef, int cur, int blk_end, int* bad) {
    unsigned p = st_p(st);
    int z = st_z(st), cb = st_cb(st), n = 0;
    const unsigned lim = pend < dend ? pend : dend;
    while (p < lim) {
        const unsigned win = peek32(words, p);
        int sym;
        const int len = huff_decode(sm.h[z == 0 ? sm.dc[cb] : sm.ac[cb]], win, sym);
        if (len == 0) {
            if (WRITE && cur + (z == 0) < blk_end) *bad = 1;
            return st_pack(p > pend ? p : pend, z, cb, 1, n);
        }
        const int s = sym & 15;
        int v = 0;
        if (s) {
            const int r = (int)((win << len) >> (32 - s));
            v = r < (1 << (s - 1)) ? r - (1 << s) + 1 : r;
        }
        p += (unsigned)(len + s);
        if (z == 0) {           // DC difference (the category is the whole symbol: DC tables hold 0..15 only)
            ++n;
            ++cur;
            if (WRITE && cur < blk_end) coef[(size_t)cur * 64] = (int16_t)v;
            z = 1;
        } else if (s) {
            z += sym >> 4;
            if (WRITE && cur < blk_end) coef[(size_t)cur * 64 + c_natural[z]] = (int16_t)v;
            ++z;
        } else if ((sym >> 4) == 15) {
            z += 16;            // ZRL
        } else {
            z = 64;             // EOB
        }
        if (z >= 64) {
            z = 0;
            cb = cb + 1 == sm.bpm ? 0 : cb + 1;
        }
    }
    return st_pack(p, z, cb, 0, n);
}

// 0 = dropped, 1 = data byte, 2 + n = first byte of marker RSTn (the second byte is dropped)
__device__ __forceinline__ int ecs_class(const uint8_t* __restrict__ e, int i, int L) {
    const int b = e[i];
    if (b == 0xFF) {
        if (i + 1 < L) {
            const int nx = e[i + 1];
            if (nx == 0) return 1;
            if (nx >= 0xD0 && nx <= 0xD7) return 2 + (nx - 0xD0);
        }
        return 0;   // fill byte, or a trailing FF
    }
    if (i > 0 && e[i - 1] == 0xFF && (b == 0 || (b >= 0xD0 && b <= 0xD7))) return 0;
    return 1;
}

// largest k < nint with pbase[k] <= pos
__device__ __forceinline__ int find_interval(const int* pbase, int nint, int pos) {
    int lo = 0, hi = nint - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (pbase[mid] <= pos) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(JT, 1) jpeg_entropy_kernel(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws,
                                                             int16_t* __restrict__ coef_all, int* __restrict__ status) {
    pdl_entry();
    __shared__ JSmem sm;
    __shared__ unsigned long long sh_scan[32];
    __shared__ int2 sh_seg[32];
    __shared__ int sh_bad;
    const int tid = threadIdx.x;
    const LfJpegImage& im = reinterpret_cast<const LfJpegImage*>(blob)[blockIdx.x];
    {
        const int* src = reinterpret_cast<const int*>(&im.dc[0]);   // dc[4] and ac[4] are contiguous
        int* dst = reinterpret_cast<int*>(&sm.h[0]);
        for (int i = tid; i < (int)(sizeof(LfJpegHuff) * 8 / 4); i += JT) dst[i] = src[i];
        if (tid < LF_JPEG_MAX_BPM) {
            sm.dc[tid] = im.blk_dc[tid] & 3;
            sm.ac[tid] = 4 + (im.blk_ac[tid] & 3);
        }
        if (tid == 0) {
            sm.bpm = im.bpm;
            sh_bad = 0;
        }
    }
    const uint8_t* ecs = blob + im.ecs_off;
    const int L = im.ecs_len, nint = im.nint, bpm = im.bpm, R = im.restart;
    const int nmcu = im.mcux * im.mcuy;
    uint8_t* stream = ws + im.stream_off;
    int* ustart = reinterpret_cast<int*>(ws + im.us_off);
    int* pbase = reinterpret_cast<int*>(ws + im.pb_off);
    unsigned long long* X = reinterpret_cast<unsigned long long*>(ws + im.x_off);
    int* Bs = reinterpret_cast<int*>(ws + im.b_off);
    int16_t* coef = coef_all + (size_t)im.block_off * 64;

    // ---- a. unstuff -------------------------------------------------------------------------------------------------
    const int chunk = (L + JT - 1) / JT;
    const int i0 = min(L, tid * chunk), i1 = min(L, i0 + chunk);
    unsigned long long agg = 0;
    for (int i = i0; i < i1; ++i) {
        const int c = ecs_class(ecs, i, L);
        agg += c == 1 ? 1ull : (c >= 2 ? (1ull << 32) : 0ull);
    }
    unsigned long long tot;
    const unsigned long long pre = cta_excl_sum(agg, sh_scan, tot);
    const int total = (int)(tot & 0xffffffffu), nrst = (int)(tot >> 32);
    if (tid == 0) {
        ustart[0] = 0;
        ustart[nint] = total;
        if (nrst != nint - 1) sh_bad = 1;
    }
    {
        int u = (int)(pre & 0xffffffffu), k = (int)(pre >> 32);
        for (int i = i0; i < i1; ++i) {
            const int c = ecs_class(ecs, i, L);
            if (c == 1) {
                ++u;
            } else if (c >= 2) {
                if (c - 2 != (k & 7)) sh_bad = 1;
                ++k;
                if (k < nint) ustart[k] = u;
            }
        }
    }
    for (int k = nrst + 1 + tid; k < nint; k += JT) ustart[k] = total;   // missing markers (flagged): empty intervals
    __syncthreads();
    const int kc = (nint + JT - 1) / JT;
    const int k0 = min(nint, tid * kc), k1 = min(nint, k0 + kc);
    agg = 0;
    for (int k = k0; k < k1; ++k) agg += (unsigned)((ustart[k + 1] - ustart[k] + JPB - 1) / JPB * JPB);
    const unsigned long long ppre = cta_excl_sum(agg, sh_scan, tot);
    const int ptot = (int)tot;
    {
        int run = (int)ppre;
        for (int k = k0; k < k1; ++k) {
            pbase[k] = run;
            run += (ustart[k + 1] - ustart[k] + JPB - 1) / JPB * JPB;
        }
    }
    if (tid == 0) pbase[nint] = ptot;
    __syncthreads();
    {
        int u = (int)(pre & 0xffffffffu), k = (int)(pre >> 32);
        for (int i = i0; i < i1; ++i) {
            const int c = ecs_class(ecs, i, L);
            if (c == 1) {
                const int kk = k < nint - 1 ? k : nint - 1;
                stream[pbase[kk] + u - ustart[kk]] = ecs[i];
                ++u;
            } else if (c >= 2) {
                ++k;
            }
        }
        for (int k = k0; k < k1; ++k)
            for (int b = pbase[k] + ustart[k + 1] - ustart[k]; b < pbase[k + 1]; ++b) stream[b] = 0;
        if (tid < 8) stream[ptot + tid] = 0;
    }
    __syncthreads();

    // ---- b. self-synchronising decode of the pieces ---------------------------------------------------------------------
    const unsigned* words = reinterpret_cast<const unsigned*>(stream);
    const int np = ptot / JPB;
    const int pc = max(2, (np + JT - 1) / JT);
    const int s0 = min(np, tid * pc), s1 = min(np, s0 + pc);
    const int kfirst = s0 < s1 ? find_interval(pbase, nint, s0 * JPB) : 0;
    if (s0 < s1) {
        unsigned long long prev = 0;
        int k = kfirst;
        for (int s = s0; s < s1; ++s) {
            while (k + 1 < nint && pbase[k + 1] <= s * JPB) ++k;
            const bool first = pbase[k] == s * JPB;
            const unsigned long long entry = first ? st_pack((unsigned)pbase[k] * 8u, 0, 0, 0, 0)
                                                   : (s == s0 ? st_pack((unsigned)s * JPBITS, 0, 0, 0, 0) : prev);
            const unsigned dend = (unsigned)(pbase[k] + ustart[k + 1] - ustart[k]) * 8u;
            prev = decode_piece<false>(words, entry, (unsigned)(s + 1) * JPBITS, dend, sm, nullptr, 0, 0, nullptr);
            X[s] = prev;
        }
    }
    __syncthreads();
    for (;;) {
        int changed = 0;
        if (s0 < s1 && pbase[kfirst] != s0 * JPB) {
            unsigned long long entry = *reinterpret_cast<volatile unsigned long long*>(X + s0 - 1);
            int k = kfirst;
            for (int s = s0; s < s1; ++s) {
                while (k + 1 < nint && pbase[k + 1] <= s * JPB) ++k;
                if (pbase[k] == s * JPB) break;   // a forced sync point: the rest of the chain is exact
                const unsigned dend = (unsigned)(pbase[k] + ustart[k + 1] - ustart[k]) * 8u;
                const unsigned long long e = decode_piece<false>(words, entry & ~(0xfffffull << 44), (unsigned)(s + 1) * JPBITS,
                                                                 dend, sm, nullptr, 0, 0, nullptr);
                if (e == X[s]) break;
                *reinterpret_cast<volatile unsigned long long*>(X + s) = e;
                changed = 1;
                entry = e;
            }
        }
        if (!__syncthreads_or(changed)) break;
    }

    // ---- c. first block of every piece: segmented (per interval) exclusive scan of the blocks started ---------------
    {
        int f = 0, v = 0, k = kfirst;
        for (int s = s0; s < s1; ++s) {
            while (k + 1 < nint && pbase[k + 1] <= s * JPB) ++k;
            if (pbase[k] == s * JPB) {
                f = 1;
                v = 0;
            }
            v += st_n(X[s]);
        }
        int run = cta_excl_segsum(f, v, sh_seg);
        k = kfirst;
        for (int s = s0; s < s1; ++s) {
            while (k + 1 < nint && pbase[k + 1] <= s * JPB) ++k;
            if (pbase[k] == s * JPB) run = 0;
            Bs[s] = (R ? k * R : 0) * bpm + run;
            run += st_n(X[s]);
        }
    }
    __syncthreads();

    // ---- d. final pass: coefficients; e. truncation check per interval ------------------------------------------------
    {
        int bad = 0, k = kfirst;
        for (int s = s0; s < s1; ++s) {
            while (k + 1 < nint && pbase[k + 1] <= s * JPB) ++k;
            const bool first = pbase[k] == s * JPB;
            const unsigned long long entry = first ? st_pack((unsigned)pbase[k] * 8u, 0, 0, 0, 0) : (X[s - 1] & ~(0xfffffull << 44));
            const unsigned dend = (unsigned)(pbase[k] + ustart[k + 1] - ustart[k]) * 8u;
            const int blk_end = (R ? min((k + 1) * R, nmcu) : nmcu) * bpm;
            decode_piece<true>(words, entry, (unsigned)(s + 1) * JPBITS, dend, sm, coef, Bs[s] - 1, blk_end, &bad);
        }
        for (int kk = k0; kk < k1; ++kk) {
            const int ibase = (R ? kk * R : 0) * bpm, iend = (R ? min((kk + 1) * R, nmcu) : nmcu) * bpm;
            if (pbase[kk + 1] == pbase[kk]) {
                bad |= iend > ibase;
                continue;
            }
            const int sl = pbase[kk + 1] / JPB - 1;
            const int started = Bs[sl] + st_n(X[sl]);
            bad |= started < iend || (started == iend && st_z(X[sl]) != 0);
        }
        if (bad) sh_bad = 1;
    }
    __syncthreads();

    // ---- e. DC differences -> DC values, per component, reset at every restart interval --------------------------------
    const int ncomp = im.ncomp;
    for (int c = 0; c < ncomp; ++c) {
        int cb0 = 0;
        while (cb0 < bpm && im.blk_comp[cb0] != c) ++cb0;
        const int nb = ncomp == 1 ? 1 : im.hs[c] * im.vs[c];
        const int n = nmcu * nb, seg = R ? R * nb : n;
        const int tc = (n + JT - 1) / JT;
        const int t0 = min(n, tid * tc), t1 = min(n, t0 + tc);
        int f = 0, v = 0;
        for (int t = t0; t < t1; ++t) {
            if (t % seg == 0) {
                f = 1;
                v = 0;
            }
            v += coef[(size_t)((t / nb) * bpm + cb0 + t % nb) * 64];
        }
        int run = cta_excl_segsum(f, v, sh_seg);
        for (int t = t0; t < t1; ++t) {
            if (t % seg == 0) run = 0;
            int16_t* d = coef + (size_t)((t / nb) * bpm + cb0 + t % nb) * 64;
            run += *d;
            *d = (int16_t)run;
        }
        __syncthreads();
    }
    if (tid == 0 && sh_bad) atomicOr(status, LF_STATUS_JPEG_CORRUPT);
}

// ---- launch 2: dequantise + ISLOW IDCT (jidctint.c: CONST_BITS 13, PASS1_BITS 2) -----------------------------------
constexpr int F_0_298 = 2446, F_0_390 = 3196, F_0_541 = 4433, F_0_765 = 6270, F_0_899 = 7373, F_1_175 = 9633,
              F_1_501 = 12299, F_1_847 = 15137, F_1_961 = 16069, F_2_053 = 16819, F_2_562 = 20995, F_3_072 = 25172;

// one 1-D pass over 8 values d0..d7 (even / odd parts of jpeg_idct_islow); o[i] = un-descaled outputs
__device__ __forceinline__ void islow_1d(const int* d, int* o) {
    int z2 = d[2], z3 = d[6];
    int z1 = (z2 + z3) * F_0_541;
    const int t2 = z1 + z3 * -F_1_847, t3 = z1 + z2 * F_0_765;
    int t0 = (d[0] + d[4]) * (1 << 13), t1 = (d[0] - d[4]) * (1 << 13);
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    int a0 = d[7], a1 = d[5], a2 = d[3], a3 = d[1];
    z1 = a0 + a3;
    z2 = a1 + a2;
    z3 = a0 + a2;
    int z4 = a1 + a3;
    const int z5 = (z3 + z4) * F_1_175;
    a0 *= F_0_298;
    a1 *= F_2_053;
    a2 *= F_3_072;
    a3 *= F_1_501;
    z1 *= -F_0_899;
    z2 *= -F_2_562;
    z3 = z3 * -F_1_961 + z5;
    z4 = z4 * -F_0_390 + z5;
    a0 += z1 + z3;
    a1 += z2 + z4;
    a2 += z2 + z3;
    a3 += z1 + z4;
    o[0] = t10 + a3; o[7] = t10 - a3;
    o[1] = t11 + a2; o[6] = t11 - a2;
    o[2] = t12 + a1; o[5] = t12 - a1;
    o[3] = t13 + a0; o[4] = t13 - a0;
}

// range_limit[(x >> n) & 1023] of jdmaster.c prepare_range_limit_table, with the +128 centring of the IDCT output
__device__ __forceinline__ unsigned idct_out(int x) {
    const int m = ((x + (1 << 17)) >> 18) & 1023;
    const int t = (m < 512 ? m : m - 1024) + 128;
    return (unsigned)(t < 0 ? 0 : (t > 255 ? 255 : t));
}

__global__ void __launch_bounds__(256) jpeg_idct_kernel(const uint8_t* __restrict__ blob, int16_t* __restrict__ coef_all,
                                                        uint8_t* __restrict__ ws) {
    pdl_entry();
    __shared__ int sh_ws[32][64];
    const LfJpegImage& im = reinterpret_cast<const LfJpegImage*>(blob)[blockIdx.y];
    const int lb = threadIdx.x >> 3, r = threadIdx.x & 7;
    const int gb = blockIdx.x * 32 + lb;
    const int bpm = im.bpm, nblk = im.mcux * im.mcuy * bpm;
    const bool live = gb < nblk;
    int c = 0;
    if (live) {
        const int m = gb / bpm, cb = gb - m * bpm;
        c = im.blk_comp[cb];
        int16_t* cf = coef_all + ((size_t)im.block_off + gb) * 64;
        const unsigned short* q = im.qt[im.qtab[c] & 3];
        int d[8], o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            d[i] = (int)cf[i * 8 + r] * (int)(short)q[i * 8 + r];   // ISLOW_MULT_TYPE is a 16-bit multiplier
            cf[i * 8 + r] = 0;                                     // leave the coefficient buffer zeroed
        }
        islow_1d(d, o);
#pragma unroll
        for (int i = 0; i < 8; ++i) sh_ws[lb][i * 8 + r] = (o[i] + (1 << 10)) >> 11;   // DESCALE(, CONST_BITS - PASS1_BITS)
    }
    __syncthreads();
    if (live) {
        const int m = gb / bpm, cb = gb - m * bpm;
        const int h = im.ncomp == 1 ? 1 : im.hs[c], v = im.ncomp == 1 ? 1 : im.vs[c];
        const int bx = (m % im.mcux) * h + im.blk_dx[cb], by = (m / im.mcux) * v + im.blk_dy[cb];
        int d[8], o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = sh_ws[lb][r * 8 + i];
        islow_1d(d, o);
        uint2 pk;
        pk.x = idct_out(o[0]) | (idct_out(o[1]) << 8) | (idct_out(o[2]) << 16) | (idct_out(o[3]) << 24);
        pk.y = idct_out(o[4]) | (idct_out(o[5]) << 8) | (idct_out(o[6]) << 16) | (idct_out(o[7]) << 24);
        uint8_t* dst = ws + im.plane_off[c] + (size_t)(by * 8 + r) * im.plane_stride[c] + bx * 8;
        *reinterpret_cast<uint2*>(dst) = pk;
    }
}

// ---- launch 3: fancy upsampling (jdsample.c) + YCbCr -> RGB (jdcolor.c, SCALEBITS 16) --------------------------------
__device__ __forceinline__ int fancy_sample(const uint8_t* __restrict__ pl, int stride, int dw, int dh, int hup, int vup, int x,
                                            int y) {
    if (!hup) return pl[(size_t)y * stride + x];
    const int j = x >> 1;
    // jinit_upsampler takes the fancy filters only for downsampled_width > 2; narrower components are replicated
    // (h2v1_upsample / h2v2_upsample)
    if (dw <= 2) return pl[(size_t)(vup ? y >> 1 : y) * stride + j];
    if (!vup) {   // h2v1_fancy_upsample
        const uint8_t* row = pl + (size_t)y * stride;
        const int c = row[j] * 3;
        if ((x & 1) == 0) return j == 0 ? row[0] : (c + row[j - 1] + 1) >> 2;
        return j == dw - 1 ? row[j] : (c + row[j + 1] + 2) >> 2;
    }
    // h2v2_fancy_upsample: column sums 3 * nearer row + further row (first / last row replicated)
    const int i = y >> 1;
    const int i1 = (y & 1) ? (i + 1 < dh ? i + 1 : dh - 1) : (i > 0 ? i - 1 : 0);
    const uint8_t* r0 = pl + (size_t)i * stride;
    const uint8_t* r1 = pl + (size_t)i1 * stride;
    const int cs = r0[j] * 3 + r1[j];
    if ((x & 1) == 0) return j == 0 ? (cs * 4 + 8) >> 4 : (cs * 3 + r0[j - 1] * 3 + r1[j - 1] + 8) >> 4;
    return j == dw - 1 ? (cs * 4 + 7) >> 4 : (cs * 3 + r0[j + 1] * 3 + r1[j + 1] + 7) >> 4;
}

__device__ __forceinline__ uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

__global__ void __launch_bounds__(256) jpeg_color_kernel(const uint8_t* __restrict__ blob, const uint8_t* __restrict__ ws, int W, int H,
                                                         uint8_t* __restrict__ out) {
    pdl_entry();
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, n = blockIdx.z;
    if (x >= W) return;
    const LfJpegImage& im = reinterpret_cast<const LfJpegImage*>(blob)[n];
    uint8_t* o = out + (((size_t)n * H + y) * W + x) * 3;
    const int Y = ws[im.plane_off[0] + (size_t)y * im.plane_stride[0] + x];
    if (im.ncomp == 1) {
        o[0] = o[1] = o[2] = (uint8_t)Y;
        return;
    }
    const int hup = im.hs[0] > im.hs[1], vup = im.vs[0] > im.vs[1];
    const int cb = fancy_sample(ws + im.plane_off[1], im.plane_stride[1], im.comp_w[1], im.comp_h[1], hup, vup, x, y) - 128;
    const int cr = fancy_sample(ws + im.plane_off[2], im.plane_stride[2], im.comp_w[2], im.comp_h[2], hup, vup, x, y) - 128;
    o[0] = clamp255(Y + ((91881 * cr + 32768) >> 16));
    o[1] = clamp255(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
    o[2] = clamp255(Y + ((116130 * cb + 32768) >> 16));
}

}  // namespace lf

using namespace lf;

static long long align16(long long x) { return (x + 15) & ~15ll; }

extern "C" size_t lf_jpeg_workspace_bytes(LfJpegImage* images, int N, size_t* coef_bytes) {
    if (!images || N < 1 || !coef_bytes) return 0;
    long long ws = 0, blocks = 0;
    for (int n = 0; n < N; ++n) {
        LfJpegImage& im = images[n];
        if (im.W != images[0].W || im.H != images[0].H || im.W < 1 || im.H < 1 || im.ecs_len < 0 || im.ecs_off < 0) return 0;
        if (!(im.ncomp == 1 || im.ncomp == 3) || im.bpm < 1 || im.bpm > LF_JPEG_MAX_BPM || im.mcux < 1 || im.mcuy < 1) return 0;
        if (im.restart < 0 || im.nint < 1) return 0;
        const long long nmcu = (long long)im.mcux * im.mcuy;
        if (im.nint != (im.restart ? (nmcu + im.restart - 1) / im.restart : 1)) return 0;
        if (nmcu * im.bpm >= (1 << 30)) return 0;
        im.npieces_max = (int)((im.ecs_len + JPB - 1) / JPB + im.nint + 1);
        im.stream_off = ws;
        ws = align16(ws + (long long)im.npieces_max * JPB + 16);
        im.x_off = ws;
        ws = align16(ws + 8ll * im.npieces_max);
        im.b_off = ws;
        ws = align16(ws + 4ll * im.npieces_max);
        im.us_off = ws;
        ws = align16(ws + 4ll * (im.nint + 1));
        im.pb_off = ws;
        ws = align16(ws + 4ll * (im.nint + 1));
        for (int c = 0; c < 3; ++c) {
            if (c >= im.ncomp) {
                im.plane_off[c] = im.plane_off[0];
                im.plane_stride[c] = im.plane_stride[0];
                continue;
            }
            const int h = im.ncomp == 1 ? 1 : im.hs[c], v = im.ncomp == 1 ? 1 : im.vs[c];
            im.plane_off[c] = ws;
            im.plane_stride[c] = im.mcux * h * 8;
            ws = align16(ws + (long long)im.plane_stride[c] * im.mcuy * v * 8);
        }
        im.block_off = blocks;
        blocks += nmcu * im.bpm;
    }
    *coef_bytes = (size_t)blocks * 128;
    return (size_t)ws;
}

extern "C" int lf_jpeg_decode(const void* blob, int N, int W, int H, unsigned char* out, int* status, void* coef, size_t coef_bytes,
                              void* workspace, size_t workspace_bytes, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(blob && out && status && coef && workspace && N >= 1 && W >= 1 && H >= 1 && coef_bytes > 0 && workspace_bytes > 0);
    const uint8_t* b = static_cast<const uint8_t*>(blob);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    int16_t* cf = static_cast<int16_t*>(coef);
    cudaError_t e = lf_launch(jpeg_entropy_kernel, dim3(N), dim3(JT), 0, stream, b, ws, cf, status);
    if (e == cudaSuccess) {
        const long long maxblk = 12ll * ((W + 15) / 16) * ((H + 15) / 16);
        e = lf_launch(jpeg_idct_kernel, dim3((unsigned)((maxblk + 31) / 32), N), dim3(256), 0, stream, b, cf, ws);
    }
    if (e == cudaSuccess) e = lf_launch(jpeg_color_kernel, dim3((W + 127) / 128, H, N), dim3(128), 0, stream, b, (const uint8_t*)ws, W, H, out);
    if (e != cudaSuccess) {
        set_last_cuda_error(e);
        return LF_ERR_CUDA;
    }
    return check_launch();
}
