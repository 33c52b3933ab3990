// Baseline JPEG encode on the GPU, byte-identical to Image.fromarray(a).save(buf, "JPEG", quality=q, subsampling=s) of
// Pillow, which encodes through libjpeg-turbo: fixed-point RGB->YCbCr (jccolor.c), edge replication and h2v2 downsampling
// (jcprepct.c, jcsample.c), the ISLOW integer forward DCT (jfdctint.c), reciprocal quantisation (jcdctmgr.c), DC-only
// dummy blocks in partial 4:2:0 MCUs (jccoefct.c) and the standard Huffman tables without optimisation (jchuff.c).  All
// of it is exact integer arithmetic; oracle/jpeg_enc_oracle.py restates it in numpy.
//
// Launch 1, enc_block_kernel (8 threads per 8x8 block, blocks in MCU order): samples (colour conversion, replication,
//   downsampling), DCT, quantisation; stores the zig-zag coefficients, the block's nonzero mask and the bits of its AC
//   symbols (code + magnitude bits, ZRLs, EOB).
// Launch 2, enc_scan_kernel (one CTA of 1024 threads per image): DC differences in MCU order per component (a dummy block
//   takes its neighbour's DC), every block's bit count, an exclusive scan into bit offsets; zeroes the bit-packing words.
// Launch 3, enc_pack_kernel (one thread per block): writes the block's codes into its disjoint bit range [off, off + bits)
//   with a 64-bit accumulator; the two words it may share with its neighbours are combined with atomicOr.
// Launch 4, enc_stuff_kernel (one CTA per image): headers, the 1-padded scan bytes with 0xFF -> 0xFF 0x00 stuffing
//   (per-tile count of 0xFF bytes, CTA scan, compaction into place), EOI, and the file's length.
#include <algorithm>
#include <cstring>

#include "lf_common.cuh"

namespace lf {
namespace {

constexpr int ET = 1024;         // threads of the per-image kernels
constexpr int HDR_MAX = 640;     // RGB headers are 623 bytes
constexpr int BLOCK_BITS = 1664; // bound on one block's bits: 22 (DC) + 63 * 26 (AC)

// ITU-T T.81 Annex K.1 (natural order) and K.3 (16 code counts, then the symbols)
const unsigned char STD_Q[2][64] = {
    {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,  14, 13, 16, 24, 40,  57,  69,  56,
     14, 17, 22, 29, 51,  87,  80,  62,  18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
    {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
const unsigned char DC_LUMA[] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const unsigned char DC_CHROMA[] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const unsigned char AC_LUMA[] = {
    0,    2,    1,    3,    3,    2,    4,    3,    5,    5,    4,    4,    0,    0,    1,    0x7d, 0x01, 0x02, 0x03, 0x00, 0x04, 0x11,
    0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1,
    0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a,
    0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59,
    0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2,
    0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6,
    0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa};
const unsigned char AC_CHROMA[] = {
    0,    2,    1,    2,    4,    4,    3,    4,    7,    5,    4,    4,    0,    1,    2,    0x77, 0x00, 0x01, 0x02, 0x03, 0x11, 0x04,
    0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09,
    0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28,
    0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58,
    0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85,
    0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
    0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4,
    0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa};

const unsigned char ZIGZAG[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                  41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                  30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ unsigned char c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                           41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                           30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Everything a launch needs besides the pointers, passed by value (kernel parameter space): no host-to-device copy, so a
// call never synchronises and can be captured into a CUDA graph.
struct EncParams {
    int W, H, ncomp, sub420;       // sub420: 4:2:0 interleaved MCUs (RGB only; a grayscale scan is one block per MCU)
    int mcux, mcuy, bpm, nblk;     // MCU grid, blocks per MCU, blocks per image
    int wb, hb;                    // luma blocks per row / column that hold image data (4:2:0 dummies lie beyond)
    int hdr_len;
    long long cap, ws_img;         // output bytes and workspace bytes per image
    long long coef_off, mask_off, bits_off, diff_off, boff_off, words_off, total_off;   // workspace offsets in an image
    unsigned short rec[2][64], cor[2][64];   // jcdctmgr.c compute_reciprocal of q * 8, natural order
    unsigned char shift[2][64];
    unsigned short dc_code[2][16], ac_code[2][256];   // [0] luma, [1] chroma
    unsigned char dc_size[2][16], ac_size[2][256];
    unsigned char hdr[HDR_MAX];
};

__device__ __forceinline__ int ycc(int r, int g, int b, int c) {   // jccolor.c rgb_ycc_convert, SCALEBITS 16
    if (c == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
    if (c == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
    return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

__device__ __forceinline__ int pixel_comp(const uint8_t* __restrict__ img, int W, int ncomp, int x, int y, int c) {
    const uint8_t* p = img + ((size_t)y * W + x) * ncomp;
    return ncomp == 1 ? p[0] : ycc(p[0], p[1], p[2], c);
}

// one sample of component c at (x, y) of its padded plane, as libjpeg's preprocessing hands it to the DCT
__device__ __forceinline__ int sample(const uint8_t* __restrict__ img, const EncParams& P, int c, int x, int y) {
    if (c == 0 || !P.sub420) return pixel_comp(img, P.W, P.ncomp, min(x, P.W - 1), min(y, P.H - 1), c);
    // h2v2: the row pair 2cy, 2cy + 1 (an odd last row replicated), the last downsampled row replicated below; columns
    // replicated right of the image; bias 1, 2, 1, 2 along the row
    const int cy = min(y, (P.H + 1) / 2 - 1);
    const int r0 = 2 * cy, r1 = min(2 * cy + 1, P.H - 1), x0 = min(2 * x, P.W - 1), x1 = min(2 * x + 1, P.W - 1);
    const int s = pixel_comp(img, P.W, 3, x0, r0, c) + pixel_comp(img, P.W, 3, x1, r0, c) + pixel_comp(img, P.W, 3, x0, r1, c) +
                  pixel_comp(img, P.W, 3, x1, r1, c);
    return (s + 1 + (x & 1)) >> 2;
}

constexpr int F_0_298 = 2446, F_0_390 = 3196, F_0_541 = 4433, F_0_765 = 6270, F_0_899 = 7373, F_1_175 = 9633,
              F_1_501 = 12299, F_1_847 = 15137, F_1_961 = 16069, F_2_053 = 16819, F_2_562 = 20995, F_3_072 = 25172;

// one pass of jpeg_fdct_islow over d[0..7]; FIRST: the row pass (outputs scaled up by PASS1_BITS), else the column pass
template <bool FIRST>
__device__ __forceinline__ void fdct_1d(const int* d, int* o) {
    constexpr int n = FIRST ? 11 : 15;   // CONST_BITS -+ PASS1_BITS
    auto ds = [](int x) { return (x + (1 << (n - 1))) >> n; };
    const int t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
    const int t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    o[0] = FIRST ? (t10 + t11) * 4 : (t10 + t11 + 2) >> 2;
    o[4] = FIRST ? (t10 - t11) * 4 : (t10 - t11 + 2) >> 2;
    const int z1 = (t12 + t13) * F_0_541;
    o[2] = ds(z1 + t13 * F_0_765);
    o[6] = ds(z1 - t12 * F_1_847);
    const int z5 = (t4 + t6 + t5 + t7) * F_1_175;
    const int y1 = (t4 + t7) * -F_0_899, y2 = (t5 + t6) * -F_2_562;
    const int y3 = (t4 + t6) * -F_1_961 + z5, y4 = (t5 + t7) * -F_0_390 + z5;
    o[7] = ds(t4 * F_0_298 + y1 + y3);
    o[5] = ds(t5 * F_2_053 + y2 + y4);
    o[3] = ds(t6 * F_3_072 + y2 + y3);
    o[1] = ds(t7 * F_1_501 + y1 + y4);
}

__device__ __forceinline__ int nbits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }

// component, block column and block row (in the component's plane) of MCU block cb of MCU m
__device__ __forceinline__ void block_coords(const EncParams& P, int m, int cb, int& c, int& bx, int& by) {
    const int mx = m % P.mcux, my = m / P.mcux;
    if (P.sub420 && cb < 4) {
        c = 0;
        bx = 2 * mx + (cb & 1);
        by = 2 * my + (cb >> 1);
    } else {
        c = P.sub420 ? cb - 3 : cb;
        bx = mx;
        by = my;
    }
}

__global__ void __launch_bounds__(256) enc_block_kernel(const uint8_t* __restrict__ frames, const __grid_constant__ EncParams P,
                                                        uint8_t* __restrict__ ws) {
    pdl_entry();
    __shared__ int sh[32][64];
    const int lb = threadIdx.x >> 3, r = threadIdx.x & 7, n = blockIdx.y;
    const int g = blockIdx.x * 32 + lb;
    const bool live = g < P.nblk;
    const uint8_t* img = frames + (size_t)n * P.H * P.W * P.ncomp;
    uint8_t* w = ws + (size_t)n * P.ws_img;
    int c = 0, bx = 0, by = 0;
    bool dummy = false;
    if (live) {
        block_coords(P, g / P.bpm, g % P.bpm, c, bx, by);
        dummy = c == 0 && P.sub420 && (bx >= P.wb || by >= P.hb);
        int d[8], o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = dummy ? 0 : sample(img, P, c, bx * 8 + i, by * 8 + r) - 128;
        fdct_1d<true>(d, o);
#pragma unroll
        for (int i = 0; i < 8; ++i) sh[lb][r * 8 + i] = o[i];
    }
    __syncthreads();
    const int t = c ? 1 : 0;
    if (live) {   // column r; quantise (jcdctmgr.c quantize with the reciprocal, correction and shift of q * 8)
        int d[8], o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = sh[lb][i * 8 + r];
        fdct_1d<false>(d, o);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int k = i * 8 + r;
            const unsigned a = (unsigned)abs(o[i]);
            const int q = (int)(((a + P.cor[t][k]) * (unsigned)P.rec[t][k]) >> (P.shift[t][k] + 16));
            o[i] = o[i] < 0 ? -q : q;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) sh[lb][i * 8 + r] = dummy ? 0 : o[i];
    }
    __syncthreads();
    // zig-zag entries r*8 .. r*8+7: store, nonzero mask, bits of the AC symbols (a run counts from the last nonzero entry)
    unsigned long long m = 0;
    int16_t z[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        z[i] = (int16_t)(live ? sh[lb][c_zigzag[r * 8 + i]] : 0);
        if (z[i]) m |= 1ull << (r * 8 + i);
    }
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) m |= __shfl_xor_sync(0xffffffffu, m, o);
    const unsigned long long mr = m | 1ull;   // the DC entry starts the first run
    int bits = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int k = r * 8 + i;
        if (k > 0 && z[i]) {
            const int prev = 63 - __clzll(mr & ((1ull << k) - 1));
            const int run = k - prev - 1, s = nbits(z[i]);
            bits += (run >> 4) * P.ac_size[t][0xF0] + P.ac_size[t][((run & 15) << 4) | s] + s;
        }
    }
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) bits += __shfl_xor_sync(0xffffffffu, bits, o);
    if (!live) return;
    uint4 pk;
    pk.x = (uint16_t)z[0] | ((unsigned)(uint16_t)z[1] << 16);
    pk.y = (uint16_t)z[2] | ((unsigned)(uint16_t)z[3] << 16);
    pk.z = (uint16_t)z[4] | ((unsigned)(uint16_t)z[5] << 16);
    pk.w = (uint16_t)z[6] | ((unsigned)(uint16_t)z[7] << 16);
    reinterpret_cast<uint4*>(w + P.coef_off)[(size_t)g * 8 + r] = pk;
    if (r == 0) {
        if (63 - __clzll(mr) < 63) bits += P.ac_size[t][0];   // EOB
        reinterpret_cast<unsigned long long*>(w + P.mask_off)[g] = m;
        reinterpret_cast<int*>(w + P.bits_off)[g] = bits;
    }
}

// the block whose DC a block codes: itself, or for a dummy luma block of a partial 4:2:0 MCU the block jccoefct.c copies
// it from (right edge: the block to its left; bottom row: block 1 of the MCU, itself possibly a right-edge dummy)
__device__ __forceinline__ int dc_source(const EncParams& P, int g) {
    if (!P.sub420) return g;
    const int m = g / 6, cb = g % 6;
    if (cb >= 4) return g;
    const int mx = m % P.mcux, my = m / P.mcux;
    int s = cb;
    if (2 * my + (cb >> 1) >= P.hb) s = 1;
    if (2 * mx + (s & 1) >= P.wb) s -= 1;
    return m * 6 + s;
}

// the previous block of the same component in MCU order, or -1
__device__ __forceinline__ int dc_prev(const EncParams& P, int g) {
    if (!P.sub420) return g - P.bpm;
    const int cb = g % 6;
    if (cb == 1 || cb == 2 || cb == 3) return g - 1;
    return g - (cb == 0 ? 3 : 6);
}

__global__ void __launch_bounds__(ET, 1) enc_scan_kernel(const __grid_constant__ EncParams P, uint8_t* __restrict__ ws) {
    pdl_entry();
    __shared__ unsigned long long sh_scan[32];
    uint8_t* w = ws + (size_t)blockIdx.x * P.ws_img;
    const int16_t* coef = reinterpret_cast<const int16_t*>(w + P.coef_off);
    int* bits = reinterpret_cast<int*>(w + P.bits_off);
    int* diff = reinterpret_cast<int*>(w + P.diff_off);
    unsigned long long* boff = reinterpret_cast<unsigned long long*>(w + P.boff_off);
    const int chunk = (P.nblk + ET - 1) / ET;
    const int g0 = min(P.nblk, (int)threadIdx.x * chunk), g1 = min(P.nblk, g0 + chunk);
    unsigned long long sum = 0;
    for (int g = g0; g < g1; ++g) {
        int c, bx, by;
        block_coords(P, g / P.bpm, g % P.bpm, c, bx, by);
        const int p = dc_prev(P, g);
        const int dv = coef[(size_t)dc_source(P, g) * 64] - (p >= 0 ? coef[(size_t)dc_source(P, p) * 64] : 0);
        const int s = nbits(dv), b = bits[g] + P.dc_size[c ? 1 : 0][s] + s;
        diff[g] = dv;
        bits[g] = b;
        sum += (unsigned)b;
    }
    unsigned long long total;
    unsigned long long run = cta_excl_sum(sum, sh_scan, total);
    for (int g = g0; g < g1; ++g) {
        boff[g] = run;
        run += (unsigned)bits[g];
    }
    if (threadIdx.x == 0) *reinterpret_cast<unsigned long long*>(w + P.total_off) = total;
    unsigned* words = reinterpret_cast<unsigned*>(w + P.words_off);
    const long long nw = (long long)(total >> 5) + 1;
    for (long long i = threadIdx.x; i < nw; i += ET) words[i] = 0;
}

// MSB-first bit writer over big-endian-ordered 32-bit words; acc holds the pending bits left-aligned
struct BitWriter {
    unsigned* words;
    long long w;
    unsigned long long acc;
    int nacc;
    __device__ BitWriter(unsigned* words_, unsigned long long pos) : words(words_), w((long long)(pos >> 5)), acc(0), nacc((int)(pos & 31)) {}
    __device__ __forceinline__ void put(unsigned v, int len) {   // len <= 27
        acc |= (unsigned long long)v << (64 - nacc - len);
        nacc += len;
        if (nacc >= 32) {
            atomicOr(words + w, (unsigned)(acc >> 32));
            ++w;
            acc <<= 32;
            nacc -= 32;
        }
    }
    __device__ __forceinline__ void flush() {
        if (nacc > 0 && (acc >> 32)) atomicOr(words + w, (unsigned)(acc >> 32));
    }
};

__global__ void __launch_bounds__(256) enc_pack_kernel(const __grid_constant__ EncParams P, uint8_t* __restrict__ ws) {
    pdl_entry();
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= P.nblk) return;
    uint8_t* w = ws + (size_t)blockIdx.y * P.ws_img;
    const int16_t* z = reinterpret_cast<const int16_t*>(w + P.coef_off) + (size_t)g * 64;
    const unsigned long long m = reinterpret_cast<const unsigned long long*>(w + P.mask_off)[g];
    int c, bx, by;
    block_coords(P, g / P.bpm, g % P.bpm, c, bx, by);
    const int t = c ? 1 : 0;
    BitWriter bw(reinterpret_cast<unsigned*>(w + P.words_off), reinterpret_cast<const unsigned long long*>(w + P.boff_off)[g]);
    const int dv = reinterpret_cast<const int*>(w + P.diff_off)[g];
    int s = nbits(dv);
    bw.put(((unsigned)P.dc_code[t][s] << s) | ((unsigned)(dv < 0 ? dv - 1 : dv) & ((1u << s) - 1)), P.dc_size[t][s] + s);
    unsigned long long rest = m & ~1ull;
    int prev = 0;
    while (rest) {
        const int k = __ffsll((long long)rest) - 1;
        rest &= rest - 1;
        int run = k - prev - 1;
        for (; run > 15; run -= 16) bw.put(P.ac_code[t][0xF0], P.ac_size[t][0xF0]);
        const int v = z[k];
        s = nbits(v);
        const int sym = (run << 4) | s;
        bw.put(((unsigned)P.ac_code[t][sym] << s) | ((unsigned)(v < 0 ? v - 1 : v) & ((1u << s) - 1)), P.ac_size[t][sym] + s);
        prev = k;
    }
    if (prev < 63) bw.put(P.ac_code[t][0], P.ac_size[t][0]);
    bw.flush();
}

constexpr int SB = 16;   // scan bytes per thread per tile of the stuffing kernel

__global__ void __launch_bounds__(ET, 1) enc_stuff_kernel(const __grid_constant__ EncParams P, const uint8_t* __restrict__ ws, uint8_t* __restrict__ out,
                                                          long long* __restrict__ out_len) {
    pdl_entry();
    __shared__ unsigned long long sh_scan[32];
    const int n = blockIdx.x;
    const uint8_t* w = ws + (size_t)n * P.ws_img;
    uint8_t* o = out + (size_t)n * P.cap;
    const unsigned long long total = *reinterpret_cast<const unsigned long long*>(w + P.total_off);
    const long long nbytes = (long long)((total + 7) >> 3);
    const unsigned* words = reinterpret_cast<const unsigned*>(w + P.words_off);
    const unsigned pad = (total & 7) ? 0xFFu >> (total & 7) : 0u;   // 1-bits up to the byte boundary
    for (int i = threadIdx.x; i < P.hdr_len; i += ET) o[i] = P.hdr[i];
    long long carry = P.hdr_len;   // output position of the tile's first byte
    for (long long t0 = 0; t0 < nbytes; t0 += (long long)ET * SB) {
        const long long b0 = t0 + (long long)threadIdx.x * SB;
        uint8_t by[SB];
        unsigned ff = 0;
#pragma unroll
        for (int i = 0; i < SB; ++i) {
            const long long b = b0 + i;
            unsigned v = 0;
            if (b < nbytes) {
                v = (words[b >> 2] >> (24 - 8 * (b & 3))) & 0xFFu;
                if (b == nbytes - 1) v |= pad;
            }
            by[i] = (uint8_t)v;
            ff += b < nbytes && v == 0xFFu;
        }
        unsigned long long tile_ff;
        const long long pre = (long long)cta_excl_sum(ff, sh_scan, tile_ff);
        long long q = carry + b0 - t0 + pre;
#pragma unroll
        for (int i = 0; i < SB; ++i) {
            if (b0 + i >= nbytes) break;
            o[q++] = by[i];
            if (by[i] == 0xFF) o[q++] = 0;
        }
        carry += min((long long)ET * SB, nbytes - t0) + (long long)tile_ff;
    }
    if (threadIdx.x == 0) {
        o[carry] = 0xFF;
        o[carry + 1] = 0xD9;
        out_len[n] = carry + 2;
    }
}

// ---- host ------------------------------------------------------------------------------------------------------------
void derive_huffman(const unsigned char* spec, int nsym_max, unsigned short* code, unsigned char* size) {
    std::memset(code, 0, sizeof(unsigned short) * nsym_max);
    std::memset(size, 0, nsym_max);
    const unsigned char* vals = spec + 16;
    int c = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        for (int i = 0; i < spec[l - 1]; ++i, ++k, ++c) {
            code[vals[k]] = (unsigned short)c;
            size[vals[k]] = (unsigned char)l;
        }
        c <<= 1;
    }
}

int spec_len(const unsigned char* spec) {
    int n = 16;
    for (int l = 0; l < 16; ++l) n += spec[l];
    return n;
}

struct Geometry {
    int ncomp, sub420, mcux, mcuy, bpm, nblk;
};

bool geometry(int W, int H, int ncomp, int sampling, Geometry& g) {
    if (W < 1 || H < 1 || W > 65535 || H > 65535 || !(ncomp == 1 || ncomp == 3) || !(sampling == 0 || sampling == 2)) return false;
    g.ncomp = ncomp;
    g.sub420 = ncomp == 3 && sampling == 2;
    const int mw = g.sub420 ? 16 : 8;
    g.mcux = (W + mw - 1) / mw;
    g.mcuy = (H + mw - 1) / mw;
    g.bpm = g.sub420 ? 6 : ncomp;
    g.nblk = g.mcux * g.mcuy * g.bpm;
    return g.nblk < (1 << 28);
}

long long header_bytes(int ncomp) { return ncomp == 3 ? 623 : 321; }

long long bound_bytes(const Geometry& g) {
    return header_bytes(g.ncomp) + 2 * ((long long)g.nblk * (BLOCK_BITS / 8) + 1) + 2;
}

long long align256(long long x) { return (x + 255) & ~255ll; }

// workspace layout of one image; returns its size
long long layout(const Geometry& g, EncParams* P) {
    long long off = 0;
    const long long nb = g.nblk;
    auto take = [&](long long bytes) {
        const long long o = off;
        off = align256(off + bytes);
        return o;
    };
    const long long coef = take(nb * 128), mask = take(nb * 8), bits = take(nb * 4), diff = take(nb * 4), boff = take(nb * 8);
    const long long words = take((nb * BLOCK_BITS / 32 + 2) * 4), total = take(8);
    if (P) {
        P->coef_off = coef;
        P->mask_off = mask;
        P->bits_off = bits;
        P->diff_off = diff;
        P->boff_off = boff;
        P->words_off = words;
        P->total_off = total;
        P->ws_img = off;
    }
    return off;
}

void put16(unsigned char*& p, int v) {
    *p++ = (unsigned char)(v >> 8);
    *p++ = (unsigned char)v;
}

// SOI, APP0 JFIF 1.01, DQT per table, SOF0, DHT (DC and AC per table), SOS, as Pillow's libjpeg-turbo writes them
int build_headers(unsigned char* h, int W, int H, int ncomp, int sampling, const unsigned short* qt) {
    unsigned char* p = h;
    static const unsigned char soi_app0[] = {0xFF, 0xD8, 0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
    std::memcpy(p, soi_app0, sizeof(soi_app0));
    p += sizeof(soi_app0);
    const int nt = ncomp == 3 ? 2 : 1;
    for (int t = 0; t < nt; ++t) {
        *p++ = 0xFF;
        *p++ = 0xDB;
        put16(p, 67);
        *p++ = (unsigned char)t;
        for (int k = 0; k < 64; ++k) *p++ = (unsigned char)qt[t * 64 + ZIGZAG[k]];
    }
    *p++ = 0xFF;
    *p++ = 0xC0;
    put16(p, 8 + 3 * ncomp);
    *p++ = 8;
    put16(p, H);
    put16(p, W);
    *p++ = (unsigned char)ncomp;
    for (int c = 0; c < ncomp; ++c) {   // Pillow sets 2x2 on the first component for 4:2:0, grayscale included
        *p++ = (unsigned char)(c + 1);
        *p++ = c == 0 && sampling == 2 ? 0x22 : 0x11;
        *p++ = c ? 1 : 0;
    }
    const unsigned char* specs[4] = {DC_LUMA, AC_LUMA, DC_CHROMA, AC_CHROMA};
    for (int i = 0; i < 2 * nt; ++i) {
        const int len = spec_len(specs[i]);
        *p++ = 0xFF;
        *p++ = 0xC4;
        put16(p, len + 3);
        *p++ = (unsigned char)(((i & 1) << 4) | (i >> 1));
        std::memcpy(p, specs[i], len);
        p += len;
    }
    *p++ = 0xFF;
    *p++ = 0xDA;
    put16(p, 6 + 2 * ncomp);
    *p++ = (unsigned char)ncomp;
    for (int c = 0; c < ncomp; ++c) {
        *p++ = (unsigned char)(c + 1);
        *p++ = c ? 0x11 : 0x00;
    }
    *p++ = 0;
    *p++ = 63;
    *p++ = 0;
    return (int)(p - h);
}

}  // namespace
}  // namespace lf

using namespace lf;

extern "C" int lf_jpeg_quality_tables(int quality, int ncomp, unsigned short* qtables) {
    LF_REQUIRE(qtables && quality >= 1 && quality <= 100 && (ncomp == 1 || ncomp == 3));
    const int scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
    for (int t = 0; t < (ncomp == 3 ? 2 : 1); ++t)
        for (int k = 0; k < 64; ++k) qtables[t * 64 + k] = (unsigned short)std::min(255, std::max(1, (STD_Q[t][k] * scale + 50) / 100));
    return LF_OK;
}

extern "C" long long lf_jpeg_encode_bound(int W, int H, int ncomp, int sampling) {
    Geometry g;
    return geometry(W, H, ncomp, sampling, g) ? bound_bytes(g) : 0;
}

extern "C" size_t lf_jpeg_encode_workspace_bytes(int N, int W, int H, int ncomp, int sampling) {
    Geometry g;
    if (N < 1 || !geometry(W, H, ncomp, sampling, g)) return 0;
    return (size_t)N * (size_t)layout(g, nullptr);
}

extern "C" int lf_jpeg_encode(const unsigned char* frames, int N, int W, int H, int ncomp, int sampling, const unsigned short* qtables,
                              unsigned char* out, long long out_cap, long long* out_len, void* workspace, lf_stream_t stream_) {
    Geometry g;
    LF_REQUIRE(frames && qtables && out && out_len && workspace && N >= 1 && geometry(W, H, ncomp, sampling, g));
    LF_REQUIRE(out_cap >= bound_bytes(g));
    const int nt = ncomp == 3 ? 2 : 1;
    for (int i = 0; i < 64 * nt; ++i) LF_REQUIRE(qtables[i] >= 1 && qtables[i] <= 255);   // baseline: 8-bit tables
    static const EncParams* tables = [] {
        static EncParams t;
        derive_huffman(DC_LUMA, 16, t.dc_code[0], t.dc_size[0]);
        derive_huffman(DC_CHROMA, 16, t.dc_code[1], t.dc_size[1]);
        derive_huffman(AC_LUMA, 256, t.ac_code[0], t.ac_size[0]);
        derive_huffman(AC_CHROMA, 256, t.ac_code[1], t.ac_size[1]);
        return &t;
    }();
    EncParams prm = *tables;
    EncParams* p = &prm;
    p->W = W;
    p->H = H;
    p->ncomp = ncomp;
    p->sub420 = g.sub420;
    p->mcux = g.mcux;
    p->mcuy = g.mcuy;
    p->bpm = g.bpm;
    p->nblk = g.nblk;
    p->wb = (W + 7) / 8;
    p->hb = (H + 7) / 8;
    p->cap = out_cap;
    layout(g, p);
    for (int t = 0; t < 2; ++t)
        for (int k = 0; k < 64; ++k) {   // jcdctmgr.c compute_reciprocal(q << 3) with a 16-bit DCTELEM
            const unsigned d = (unsigned)qtables[std::min(t, nt - 1) * 64 + k] << 3;
            int b = 31 - __builtin_clz(d), r = 16 + b;
            unsigned fq = (1u << r) / d, fr = (1u << r) % d, c = d / 2;
            if (fr == 0) {
                fq >>= 1;
                --r;
            } else if (fr <= d / 2) {
                ++c;
            } else {
                ++fq;
            }
            p->rec[t][k] = (unsigned short)fq;
            p->cor[t][k] = (unsigned short)c;
            p->shift[t][k] = (unsigned char)(r - 16);
        }
    p->hdr_len = build_headers(p->hdr, W, H, ncomp, sampling, qtables);
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    cudaError_t e = lf_launch(enc_block_kernel, dim3((unsigned)((g.nblk + 31) / 32), N), dim3(256), 0, stream, frames, *p, ws);
    if (e == cudaSuccess) e = lf_launch(enc_scan_kernel, dim3(N), dim3(ET), 0, stream, *p, ws);
    if (e == cudaSuccess) e = lf_launch(enc_pack_kernel, dim3((unsigned)((g.nblk + 255) / 256), N), dim3(256), 0, stream, *p, ws);
    if (e == cudaSuccess) e = lf_launch(enc_stuff_kernel, dim3(N), dim3(ET), 0, stream, *p, (const uint8_t*)ws, out, out_len);
    if (e != cudaSuccess) {
        set_last_cuda_error(e);
        return LF_ERR_CUDA;
    }
    return check_launch();
}
