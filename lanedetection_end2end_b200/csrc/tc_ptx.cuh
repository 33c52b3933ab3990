// Shared Hopper (sm_90a) tensor-core PTX wrappers: TMA, mbarrier, wgmma (TF32 and BF16), shared-memory accesses, TF32
// operand splitting, bf16 packing and the tensor-map helpers.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace lf {

constexpr uint32_t TC_SPIN_LIMIT = 1u << 22;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0, spins = 0;
    while (true) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) break;
        if (++spins > TC_SPIN_LIMIT) __trap();  // a protocol bug ends the kernel with an error instead of hanging the GPU
    }
}
// One lane of a converged warp: the TMA issuing warp runs its loop with all 32 lanes so that coordinates and barrier
// addresses stay warp-uniform; only the issuing instruction is predicated on the elected lane.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* tm, uint64_t* bar, void* dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* tm, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3,
                                            int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], "
        "[%2];" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ------------------------------------------------------------------------------------------
// TF32 operands.  Every product the tensor core forms here takes operands that are exact TF32 values (low 13 mantissa
// bits zero), so the result does not depend on how the hardware would round an fp32 bit pattern.
// 3xTF32: a = hi + lo with hi = tf32_rna(a) and lo = tf32_rna(a - hi) (a - hi is exact); a*w = hi*w_hi + (hi*w_lo +
// lo*w_hi) up to O(2^-22 |a||w|), below the fp32 rounding of the sum.
// ------------------------------------------------------------------------------------------
// round-to-nearest (ties away) to TF32 with the dropped bits cleared
__device__ __forceinline__ uint32_t tf32_rna(float a) { return (__float_as_uint(a) + 0x1000u) & 0xffffe000u; }
__device__ __forceinline__ void tf32_split(float a, uint32_t& hi, uint32_t& lo) {
    hi = tf32_rna(a);
    lo = tf32_rna(a - __uint_as_float(hi));
}

// Element (row r, column c < 32) of a [rows x 32] fp32 tile that TMA wrote with CU_TENSOR_MAP_SWIZZLE_128B: rows of 128
// bytes, the 16-byte chunk index XORed with r & 7.  Byte offset from the tile base.
__device__ __forceinline__ uint32_t sw128_off(int r, int c) { return (uint32_t)(r * 128 + ((((c >> 2) ^ r) & 7) << 4) + ((c & 3) << 2)); }

// ------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA).  B operand: K-major, 128B-swizzled tile in shared memory (rows of 32 fp32 = 128 bytes, 8-row
// groups 1024 bytes apart) = exactly what TMA writes with CU_TENSOR_MAP_SWIZZLE_128B.  Descriptor: start >> 4 (bits 0-13),
// LBO >> 4 (16-29; unused for swizzled K-major), SBO >> 4 (32-45), layout 1 = SWIZZLE_128B (bits 62-63).  The tile base
// must be 1024-byte aligned; the k-th group of 8 TF32 along K starts 32*k bytes later (+2 in the start field).
// A operand: registers (or shared memory, wgmma_m64n64k8_tf32_ss), the m64k8 TF32 fragment of this thread:
//   a[0] = A[16w + g][t], a[1] = A[16w + g + 8][t], a[2] = A[16w + g][t + 4], a[3] = A[16w + g + 8][t + 4]
// (w = warp within the warpgroup, g = lane / 4, t = lane % 4).  Accumulator fragment of m64nN, register i:
//   row 16w + g + 8 * ((i >> 1) & 1), column 8 * (i >> 2) + 2t + (i & 1).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from touching accumulator registers across an asynchronous wgmma
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 64] (+)= A[64 x 8] * B[64 x 8]^T, TF32 in, fp32 accumulate
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// The same with A from shared memory: adesc describes a K-major, 128B-swizzled [64 x 32] fp32 tile exactly like B (rows =
// the 64 M rows; wgmma_desc_sw128 of a 1024-byte aligned base, +2 per k8).  The words must already be TF32 values.
__device__ __forceinline__ void wgmma_m64n64k8_tf32_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// D[64 x 48] (+)= A[64 x 8] * B[48 x 8]^T
__device__ __forceinline__ void wgmma_m64n48k8_tf32(float (&d)[24], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
        "{%24, %25, %26, %27}, %28, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// D[64 x 32] (+)= A[64 x 8] * B[32 x 8]^T
__device__ __forceinline__ void wgmma_m64n32k8_tf32(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// D[64 x 16] (+)= A[64 x 8] * B[16 x 8]^T
__device__ __forceinline__ void wgmma_m64n16k8_tf32(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T for N in {16, 32, 48, 64}
template <int N>
__device__ __forceinline__ void wgmma_m64k8_tf32(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    static_assert(N == 16 || N == 32 || N == 48 || N == 64, "wgmma_m64k8_tf32: N");
    if constexpr (N == 16) wgmma_m64n16k8_tf32(d, a, bdesc, accumulate);
    else if constexpr (N == 32) wgmma_m64n32k8_tf32(d, a, bdesc, accumulate);
    else if constexpr (N == 48) wgmma_m64n48k8_tf32(d, a, bdesc, accumulate);
    else wgmma_m64n64k8_tf32(d, a, bdesc, accumulate);
}

// ------------------------------------------------------------------------------------------
// BF16 operands (the "bf16" convolution mode): both operands rounded to bf16 (round to nearest even), products exact in
// fp32, fp32 accumulate.  Operand precision of the tensor-core kernel templates (= the `precision` fields of the C ABI):
// ------------------------------------------------------------------------------------------
enum TcPrec : int { TC_TF32 = 0, TC_X3 = 1, TC_BF16 = 2 };

// bf16x2 of (lo, hi), round to nearest even: `lo` in bits 0-15 (the lower K index of a fragment register)
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

// B operand: K-major, 64B-swizzled bf16 tile in shared memory (rows of 32 bf16 = 64 bytes, 8-row groups 512 bytes
// apart) = what TMA writes for a [rows x 32] bf16 box with CU_TENSOR_MAP_SWIZZLE_64B: the 16-byte chunk index within a
// row is XORed with (r >> 1) & 3.  Descriptor: layout 2 = SWIZZLE_64B, SBO = 512; the tile base must be 512-byte
// aligned; the k-th group of 16 bf16 along K starts 32*k bytes later (+2 in the start field).
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t smem_addr) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)(512 >> 4) << 32) | (2ull << 62);
}
// Byte offset of bf16 element (row r, k < 32) of such a tile
__device__ __forceinline__ uint32_t sw64_off(int r, int k) { return (uint32_t)(r * 64 + ((((k >> 3) ^ (r >> 1)) & 3) << 4) + ((k & 7) << 1)); }

// A operand: registers, the m64k16 BF16 fragment of this thread (PTX ISA, "Register fragment for matrix A" of
// wgmma .m64nNk16), two bf16 per register, the lower K index in the low half:
//   a[0] = A[16w + g][2t, 2t+1],     a[1] = A[16w + g + 8][2t, 2t+1],
//   a[2] = A[16w + g][2t+8, 2t+9],   a[3] = A[16w + g + 8][2t+8, 2t+9]
// (w, g, t as for TF32).  The accumulator fragment is the one of the TF32 instructions.  B K-major: imm-trans-b = 0.
// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, BF16 in, fp32 accumulate
__device__ __forceinline__ void wgmma_m64n64k16_bf16(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// D[64 x 48] (+)= A[64 x 16] * B[48 x 16]^T
__device__ __forceinline__ void wgmma_m64n48k16_bf16(float (&d)[24], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
        "{%24, %25, %26, %27}, %28, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// D[64 x 32] (+)= A[64 x 16] * B[32 x 16]^T
__device__ __forceinline__ void wgmma_m64n32k16_bf16(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// D[64 x 16] (+)= A[64 x 16] * B[16 x 16]^T
__device__ __forceinline__ void wgmma_m64n16k16_bf16(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T for N in {16, 32, 48, 64}
template <int N>
__device__ __forceinline__ void wgmma_m64k16_bf16(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    static_assert(N == 16 || N == 32 || N == 48 || N == 64, "wgmma_m64k16_bf16: N");
    if constexpr (N == 16) wgmma_m64n16k16_bf16(d, a, bdesc, accumulate);
    else if constexpr (N == 32) wgmma_m64n32k16_bf16(d, a, bdesc, accumulate);
    else if constexpr (N == 48) wgmma_m64n48k16_bf16(d, a, bdesc, accumulate);
    else wgmma_m64n64k16_bf16(d, a, bdesc, accumulate);
}

// Shared-state-space accesses (addresses from smem_u32): LDS / STS without generic-address translation.
__device__ __forceinline__ float lds_f32(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {   // zero-extended
    uint32_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ float4 lds_f32x4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void sts_u32x4(uint32_t addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// orders this thread's generic-proxy shared-memory stores before later async-proxy (wgmma, TMA) accesses
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------
// host: cuTensorMapEncodeTiled through the runtime's driver entry point (no libcuda link)
// ------------------------------------------------------------------------------------------
typedef CUresult (*TcEncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline TcEncodeTiledFn tc_get_encode_fn() {
    static TcEncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<TcEncodeTiledFn>(p);
    }
    return fn;
}

// Strided fp32 view (element strides sx, sy, sn; channels contiguous) as (ci:32, cblk:C/32, x:W, y:H, n:N); one box =
// [bx*by pixels] x [32 channels] = rows of 128 bytes, 128B-swizzled; out-of-bounds -> zeros.  bf16: a bf16 view, rows of
// 64 bytes, 64B-swizzled.
inline bool tc_encode_view(TcEncodeTiledFn enc, CUtensorMap* tm, const float* base, int N, int H, int W, int C, long long sx,
                           long long sy, long long sn, int bx, int by, bool bf16 = false) {
    const cuuint64_t esz = bf16 ? 2 : 4;
    cuuint64_t dims[5] = {32, (cuuint64_t)(C / 32), (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[4] = {32 * esz, (cuuint64_t)sx * esz, (cuuint64_t)sy * esz, (cuuint64_t)sn * esz};
    cuuint32_t box[5] = {32, 1, (cuuint32_t)bx, (cuuint32_t)by, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    return enc(tm, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(base), dims,
               strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, bf16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}


}  // namespace lf
