// PNG decode of the loader's label maps on the GPU (replaces Image.open(f).convert('P') of
// BP/Dataloader/Load_Data_new.py:120-121), bit-identical to Pillow: the gray values or palette indices of a non-interlaced
// 8-bit grayscale or 1/2/4/8-bit palette PNG.  The host (png.py) walks the chunks and concatenates the IDAT payloads.
//
// Launch 1, png_inflate_kernel (one warp per image): RFC 1951 inflate of the zlib stream into the filtered scanlines
//   (H x (1 + rowbytes) bytes in the workspace).  Lane 0 reads the block headers and decodes the symbols serially, with
//   the Huffman tables in shared memory (a 9-bit LSB-first lookahead, canonical bit-by-bit decode for longer codes, as
//   zlib's puff.c); the tables of each block are built by the whole warp.  Literals are stored by lane 0 as they are
//   decoded; matches and stored blocks go to a queue that the warp then copies in order, 32 bytes per step.  A match of
//   distance d is copied as out[p + i] = out[p - d + i mod d], which reads only bytes before p, so overlapping matches
//   (distance 1, length 258 is the commonest symbol of a label map) need no step-by-step ordering.  Every check of zlib's
//   inflate on a well-formed stream is made: invalid codes and code-length sets, distances before the start, output
//   longer or shorter than the image, a stream ending before its final block.  The expected Adler-32 is read after the
//   final block and left in the image's meta word.
// Launch 2, png_unfilter_kernel (one warp per image): PNG filters None / Sub / Up / Average / Paeth with a 1-byte filter
//   unit, then unpacking of 1/2/4-bit samples (most significant bits first) into the uint8 frame.  Average and Paeth are
//   serial along a row and depend on the row above, so the warp runs a wavefront over 32 rows at a time: lane i
//   unfilters row r + i one 4-byte chunk per step, one chunk behind lane i - 1, whose result it receives by a shuffle.
//   The last row of each group is written back in place for the next group's first lane.  The lanes sum the Adler-32
//   of the bytes they read and the warp checks it against the stream's.
#include "lf_common.cuh"

namespace lf {

constexpr int PNG_LOOK = 9;      // lookahead bits of the Huffman tables
constexpr int PNG_QUEUE = 64;    // copies queued by lane 0 before the warp executes them
constexpr unsigned FULL = 0xffffffffu;
constexpr unsigned ADLER_MOD = 65521u;

__constant__ unsigned short c_len_base[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                              31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ unsigned char c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ unsigned short c_dist_base[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,    65,    97,    129,
                                               193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ unsigned char c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ unsigned char c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct PngHuff {
    unsigned short look[1 << PNG_LOOK];   // next PNG_LOOK bits (LSB first) -> (length << 9) | symbol; 0 = longer or no code
    unsigned short count[16];             // number of codes of each length
    unsigned short offs[16];              // index in sym of the first code of each length
    unsigned short sym[288];              // symbols ordered by (length, value)
};

// Bit reader of lane 0: LSB-first bits of the stream, zeros past its end (overrun() tells when those were consumed).
struct PngBits {
    const uint8_t* p;
    long long n, pos;
    unsigned long long buf;
    int cnt;
    __device__ __forceinline__ void refill() {        // at least 32 bits in buf afterwards
        if (cnt < 32) {
            unsigned w = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) w |= (unsigned)(pos + k < n ? p[pos + k] : 0) << (8 * k);
            buf |= (unsigned long long)w << cnt;
            cnt += 32;
            pos += 4;
        }
    }
    __device__ __forceinline__ unsigned get(int k) {
        const unsigned v = (unsigned)(buf & ((1ull << k) - 1));
        buf >>= k;
        cnt -= k;
        return v;
    }
    __device__ __forceinline__ bool overrun() const { return pos * 8 - cnt > n * 8; }
    __device__ __forceinline__ long long byte_pos() const { return pos - (cnt >> 3); }   // after align()
    __device__ __forceinline__ void align() { get(cnt & 7); }
};

// canonical decode bit by bit for codes longer than the lookahead (zlib's puff.c decode()); -1 = no such code
__device__ int huff_slow(const PngHuff& h, PngBits& br) {
    int code = 0, first = 0, index = 0;
    for (int len = 1; len <= 15; ++len) {
        code |= (int)((br.buf >> (len - 1)) & 1);
        const int count = h.count[len];
        if (code - count < first) {
            br.get(len);
            return h.sym[index + (code - first)];
        }
        index += count;
        first += count;
        first <<= 1;
        code <<= 1;
    }
    return -1;
}

__device__ __forceinline__ int huff_decode(const PngHuff& h, PngBits& br) {
    const unsigned e = h.look[br.buf & ((1u << PNG_LOOK) - 1)];
    if (e) {
        br.get((int)(e >> 9));
        return (int)(e & 511);
    }
    return huff_slow(h, br);
}

// count / offs / sym of a code (lane 0, serial); false for an over-subscribed set, or an incomplete one unless it is a
// single code of length 1 (or no code at all) and `single_ok` -- zlib's inflate_table rules
__device__ bool huff_counts(PngHuff& h, const unsigned char* lens, int nsym, bool single_ok) {
    for (int l = 0; l < 16; ++l) h.count[l] = 0;
    for (int s = 0; s < nsym; ++s) ++h.count[lens[s]];
    int left = 1, maxlen = 0;
    for (int l = 1; l < 16; ++l) {
        left = (left << 1) - h.count[l];
        if (left < 0) return false;
        if (h.count[l]) maxlen = l;
    }
    if (maxlen == 0) {
        h.count[0] = 0;
        return single_ok;
    }
    if (left > 0 && !(single_ok && maxlen == 1)) return false;
    h.offs[1] = 0;
    for (int l = 1; l < 15; ++l) h.offs[l + 1] = h.offs[l] + h.count[l];
    unsigned short next[16];
    for (int l = 1; l < 16; ++l) next[l] = h.offs[l];
    for (int s = 0; s < nsym; ++s)
        if (lens[s]) h.sym[next[lens[s]]++] = (unsigned short)s;
    h.count[0] = 0;
    return true;
}

// lookahead table of a code whose count / offs / sym are set (whole warp)
__device__ void huff_look(PngHuff& h, int lane) {
    for (int i = lane; i < (1 << PNG_LOOK); i += 32) h.look[i] = 0;
    __syncwarp();
    int total = 0, first[16];
    int code = 0;
    for (int l = 1; l < 16; ++l) {
        first[l] = code;
        code = (code + h.count[l]) << 1;
        total += h.count[l];
    }
    for (int j = lane; j < total; j += 32) {
        int l = 1;
        while (l < 15 && j >= h.offs[l] + h.count[l]) ++l;
        if (l > PNG_LOOK) continue;
        const unsigned c = (unsigned)(first[l] + j - h.offs[l]);
        const unsigned rev = __brev(c) >> (32 - l);
        const unsigned short e = (unsigned short)((l << 9) | h.sym[j]);
        for (unsigned k = rev; k < (1u << PNG_LOOK); k += 1u << l) h.look[k] = e;
    }
}

enum { ST_HDR = 0, ST_BUILD = 1, ST_DATA = 2, ST_END = 3, ST_BAD = 4 };

// one block header (lane 0): a stored block is queued as one copy, fixed / dynamic code lengths go to lens
__device__ int png_block_header(PngBits& br, PngHuff& scratch, unsigned char* lens, int* nlit, int* ndist, int* final_,
                                int4* queue, int* nq, int* pos, int total) {
    br.refill();
    *final_ = (int)br.get(1);
    const int type = (int)br.get(2);
    if (type == 0) {
        br.align();
        br.refill();
        const unsigned len = br.get(16), nlen = br.get(16);
        if (len != (~nlen & 0xffffu)) return ST_BAD;
        const long long bp = br.byte_pos();
        if (bp + len > br.n || (int)len > total - *pos) return ST_BAD;
        queue[0] = make_int4(*pos, (int)len, 0, (int)bp);
        *nq = 1;
        *pos += (int)len;
        br.pos = bp + len;
        br.buf = 0;
        br.cnt = 0;
        return *final_ ? ST_END : ST_HDR;
    }
    if (type == 1) {
        for (int s = 0; s < 288; ++s) lens[s] = s < 144 ? 8 : (s < 256 ? 9 : (s < 280 ? 7 : 8));
        for (int s = 0; s < 32; ++s) lens[288 + s] = 5;   // 30 and 31 complete the code; decoding them is an error
        *nlit = 288;
        *ndist = 32;
        return ST_BUILD;
    }
    if (type == 3) return ST_BAD;
    const int hlit = (int)br.get(5) + 257, hdist = (int)br.get(5) + 1, hclen = (int)br.get(4) + 4;
    if (hlit > 286 || hdist > 30) return ST_BAD;
    unsigned char clens[19];
    for (int k = 0; k < 19; ++k) clens[k] = 0;
    for (int k = 0; k < hclen; ++k) {
        br.refill();
        clens[c_clen_order[k]] = (unsigned char)br.get(3);
    }
    if (!huff_counts(scratch, clens, 19, false)) return ST_BAD;
    const int n = hlit + hdist;
    int idx = 0;
    while (idx < n) {
        br.refill();
        const int sym = huff_slow(scratch, br);
        if (sym < 0) return ST_BAD;
        if (sym < 16) {
            lens[idx++] = (unsigned char)sym;
            continue;
        }
        int rep, val = 0;
        if (sym == 16) {
            if (idx == 0) return ST_BAD;
            val = lens[idx - 1];
            rep = 3 + (int)br.get(2);
        } else if (sym == 17) {
            rep = 3 + (int)br.get(3);
        } else {
            rep = 11 + (int)br.get(7);
        }
        if (idx + rep > n) return ST_BAD;
        while (rep--) lens[idx++] = (unsigned char)val;
    }
    if (lens[256] == 0) return ST_BAD;
    // the literal/length and distance lengths lie back to back; the distance table reads them from lens + 288
    for (int k = hdist - 1; k >= 0; --k) lens[288 + k] = lens[hlit + k];
    *nlit = hlit;
    *ndist = hdist;
    return br.overrun() ? ST_BAD : ST_BUILD;
}

__global__ void __launch_bounds__(32) png_inflate_kernel(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws, int* status) {
    pdl_entry();
    __shared__ PngHuff s_lit, s_dist;
    __shared__ unsigned char s_lens[288 + 32];
    __shared__ int4 s_queue[PNG_QUEUE];
    __shared__ int s_state, s_nq, s_nlit, s_ndist, s_final;
    const int lane = threadIdx.x;
    const LfPngImage im = reinterpret_cast<const LfPngImage*>(blob)[blockIdx.x];
    const uint8_t* zs = blob + im.zoff;
    uint8_t* raw = ws + im.raw_off;
    int4* meta = reinterpret_cast<int4*>(ws) + blockIdx.x;   // x: corrupt, y: Adler-32 of the stream
    const int total = im.H * (1 + im.rowbytes);
    PngBits br;
    int pos = 0;
    if (lane == 0) {
        br.p = zs;
        br.n = im.zlen;
        br.pos = 2;                                            // the zlib header was checked on the host
        br.buf = 0;
        br.cnt = 0;
        s_state = ST_HDR;
        s_nq = 0;
        s_final = 0;
    }
    for (;;) {
        __syncwarp();
        if (lane == 0 && s_state == ST_HDR) {
            int nq = 0, nlit = 0, ndist = 0, fin = 0;
            s_state = png_block_header(br, s_dist, s_lens, &nlit, &ndist, &fin, s_queue, &nq, &pos, total);
            s_nq = nq;
            s_nlit = nlit;
            s_ndist = ndist;
            s_final = fin;
        }
        __syncwarp();
        if (s_state == ST_BUILD) {
            bool ok = true;
            if (lane == 0) ok = huff_counts(s_lit, s_lens, s_nlit, true) && huff_counts(s_dist, s_lens + 288, s_ndist, true);
            ok = __shfl_sync(FULL, ok, 0);
            __syncwarp();
            if (ok) {
                huff_look(s_lit, lane);
                huff_look(s_dist, lane);
            }
            __syncwarp();
            if (lane == 0) s_state = ok ? ST_DATA : ST_BAD;
            __syncwarp();
        }
        if (lane == 0 && s_state == ST_DATA) {
            int nq = 0, st = ST_DATA;
            while (nq < PNG_QUEUE) {
                br.refill();
                const int s = huff_decode(s_lit, br);
                if (s < 256) {
                    if (s < 0 || pos >= total) {
                        st = ST_BAD;
                        break;
                    }
                    raw[pos++] = (uint8_t)s;
                } else if (s == 256) {
                    st = s_final ? ST_END : ST_HDR;
                    break;
                } else {
                    if (s > 285) {
                        st = ST_BAD;
                        break;
                    }
                    const int len = c_len_base[s - 257] + (int)br.get(c_len_extra[s - 257]);
                    br.refill();
                    const int d = huff_decode(s_dist, br);
                    if (d < 0 || d > 29) {
                        st = ST_BAD;
                        break;
                    }
                    const int dist = c_dist_base[d] + (int)br.get(c_dist_extra[d]);
                    if (dist > pos || len > total - pos) {
                        st = ST_BAD;
                        break;
                    }
                    s_queue[nq++] = make_int4(pos, len, dist, 0);
                    pos += len;
                }
                if (br.overrun()) {
                    st = ST_BAD;
                    break;
                }
            }
            s_nq = nq;
            s_state = st;
        }
        __syncwarp();
        const int nq = s_nq;
        for (int k = 0; k < nq; ++k) {
            const int4 e = s_queue[k];                         // (output position, length, distance or 0, stored source)
            if (e.z == 0) {
                for (int i = lane; i < e.y; i += 32) raw[e.x + i] = zs[e.w + i];
            } else {
                const uint8_t* src = raw + e.x - e.z;
                const int step = 32 % e.z;
                int j = lane % e.z;
                for (int i = lane; i < e.y; i += 32) {
                    raw[e.x + i] = src[j];
                    j += step;
                    if (j >= e.z) j -= e.z;
                }
            }
            __syncwarp();
        }
        if (lane == 0) s_nq = 0;
        const int st = s_state;
        if (st == ST_END || st == ST_BAD) break;
    }
    if (lane == 0) {
        bool bad = s_state == ST_BAD || pos != total;
        unsigned adler = 0;
        if (!bad) {
            br.align();
            br.refill();
            for (int k = 0; k < 4; ++k) adler = (adler << 8) | br.get(8);
            bad = br.overrun();
        }
        *meta = make_int4(bad ? 1 : 0, (int)adler, 0, 0);
        if (bad) atomicOr(status, LF_STATUS_PNG_CORRUPT);
    }
}

__device__ __forceinline__ unsigned png_paeth(unsigned a, unsigned b, unsigned c) {
    const int p = (int)a + (int)b - (int)c;
    const int pa = abs(p - (int)a), pb = abs(p - (int)b), pc = abs(p - (int)c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__global__ void __launch_bounds__(32) png_unfilter_kernel(const uint8_t* __restrict__ blob, uint8_t* __restrict__ ws,
                                                          uint8_t* __restrict__ out, int* status) {
    pdl_entry();
    const LfPngImage im = reinterpret_cast<const LfPngImage*>(blob)[blockIdx.x];
    const int4 meta = reinterpret_cast<const int4*>(ws)[blockIdx.x];
    if (meta.x) return;                                        // the inflate already reported this image
    const int lane = threadIdx.x;
    uint8_t* raw = ws + im.raw_off;
    const int W = im.W, H = im.H, rb = im.rowbytes, stride = rb + 1, depth = im.depth;
    const int ppb = 8 / depth;                                 // pixels per byte
    const unsigned smask = (1u << depth) - 1;
    uint8_t* frame = out + (size_t)blockIdx.x * H * W;
    const int nch = (rb + 3) >> 2;
    unsigned long long s1 = 0, s2 = 0;                         // sum of bytes, sum of index * byte (Adler-32)
    bool bad = false;
    for (int r0 = 0; r0 < H; r0 += 32) {
        const int y = r0 + lane;
        const bool act = y < H;
        const long long rowoff = (long long)y * stride;
        unsigned ft = 0;
        if (act) {
            ft = raw[rowoff];
            s1 += ft;
            s2 += (unsigned long long)rowoff * ft;
        }
        if (__any_sync(FULL, ft > 4)) {
            bad = true;
            break;
        }
        const uint8_t* above = r0 > 0 ? raw + (long long)(r0 - 1) * stride + 1 : nullptr;   // unfiltered, for lane 0
        uint8_t* row = raw + rowoff + 1;
        uint8_t* orow = frame + (size_t)y * W;
        unsigned last = 0, upprev = 0, left = 0;
        for (int t = 0; t < nch + 31; ++t) {
            const int c = t - lane;
            unsigned up = __shfl_up_sync(FULL, last, 1);
            if (act && c >= 0 && c < nch) {
                const int nb = min(4, rb - 4 * c);
                if (lane == 0) {
                    up = 0;
                    if (above)
                        for (int k = 0; k < nb; ++k) up |= (unsigned)above[4 * c + k] << (8 * k);
                }
                unsigned x4 = 0;
                for (int k = 0; k < nb; ++k) x4 |= (unsigned)row[4 * c + k] << (8 * k);
                unsigned a = left, ul = c > 0 ? upprev >> 24 : 0, cur = 0;
                for (int k = 0; k < nb; ++k) {
                    const unsigned x = (x4 >> (8 * k)) & 255u, b = (up >> (8 * k)) & 255u;
                    s1 += x;
                    s2 += (unsigned long long)(rowoff + 1 + 4 * c + k) * x;
                    unsigned v = x;
                    if (ft == 1) v += a;
                    else if (ft == 2) v += b;
                    else if (ft == 3) v += (a + b) >> 1;
                    else if (ft == 4) v += png_paeth(a, b, ul);
                    v &= 255u;
                    cur |= v << (8 * k);
                    ul = b;
                    a = v;
                    if (depth == 8) {
                        orow[4 * c + k] = (uint8_t)v;
                    } else {
                        const int px0 = (4 * c + k) * ppb;
                        for (int q = 0; q < ppb && px0 + q < W; ++q) orow[px0 + q] = (uint8_t)((v >> (8 - depth * (q + 1))) & smask);
                    }
                }
                if (lane == 31)
                    for (int k = 0; k < nb; ++k) row[4 * c + k] = (uint8_t)(cur >> (8 * k));
                left = a;
                upprev = up;
                last = cur;
            }
        }
        __syncwarp();
    }
    s1 %= ADLER_MOD;
    s2 %= ADLER_MOD;
    for (int o = 16; o > 0; o >>= 1) {
        s1 += __shfl_xor_sync(FULL, s1, o);
        s2 += __shfl_xor_sync(FULL, s2, o);
    }
    if (lane == 0) {
        // Adler-32 of n bytes d_i: A = 1 + sum d_i, B = n + sum (n - i) d_i = n (1 + sum d_i) - sum i d_i   (mod 65521)
        const unsigned long long n = (unsigned long long)H * stride % ADLER_MOD;
        const unsigned long long A = (1 + s1) % ADLER_MOD;
        const unsigned long long B = (n * A + ADLER_MOD - s2 % ADLER_MOD) % ADLER_MOD;
        if (bad || (unsigned)((B << 16) | A) != (unsigned)meta.y) atomicOr(status, LF_STATUS_PNG_CORRUPT);
    }
}

}  // namespace lf

using namespace lf;

static long long png_align16(long long x) { return (x + 15) & ~15ll; }

extern "C" size_t lf_png_workspace_bytes(LfPngImage* images, int N) {
    if (!images || N < 1) return 0;
    long long ws = png_align16(16ll * N);                      // one int4 meta word per image
    for (int n = 0; n < N; ++n) {
        LfPngImage& im = images[n];
        if (im.W != images[0].W || im.H != images[0].H || im.W < 1 || im.H < 1 || im.zoff < 0 || im.zlen < 2) return 0;
        if (!(im.depth == 1 || im.depth == 2 || im.depth == 4 || im.depth == 8)) return 0;
        const long long rb = ((long long)im.W * im.depth + 7) / 8;
        if ((long long)im.H * (rb + 1) > (1ll << 28)) return 0;    // keeps the Adler-32 sums exact in 64 bits
        im.rowbytes = (int)rb;
        im.raw_off = ws;
        ws = png_align16(ws + (long long)im.H * (rb + 1));
    }
    return (size_t)ws;
}

extern "C" int lf_png_decode(const void* blob, int N, int W, int H, unsigned char* out, int* status, void* workspace,
                             size_t workspace_bytes, lf_stream_t stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    LF_REQUIRE(blob && out && status && workspace && N >= 1 && W >= 1 && H >= 1 && workspace_bytes > 0);
    const uint8_t* b = static_cast<const uint8_t*>(blob);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    cudaError_t e = lf_launch(png_inflate_kernel, dim3(N), dim3(32), 0, stream, b, ws, status);
    if (e == cudaSuccess) e = lf_launch(png_unfilter_kernel, dim3(N), dim3(32), 0, stream, b, ws, out, status);
    if (e != cudaSuccess) {
        set_last_cuda_error(e);
        return LF_ERR_CUDA;
    }
    return check_launch();
}
