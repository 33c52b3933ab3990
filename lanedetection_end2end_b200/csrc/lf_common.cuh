// Shared helpers for the lanefit_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include "../../include/lanefit_b200.h"

namespace lf {

using ConvArgs = LfConvArgs;      // internal names of the public argument structs
using WgradArgs = LfWgradArgs;

void set_last_cuda_error(cudaError_t e);

inline int check_launch() {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_last_cuda_error(e);
        return LF_ERR_CUDA;
    }
    return LF_OK;
}

// ---------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  Every kernel of the library is launched through lf_launch(); with the switch on
// (lf_set_pdl(1) / LANEFIT_PDL=1; DEFAULT OFF: the whole step already replays as one CUDA graph, and a tensor-core kernel's CTA (up to 227 KB of shared
// memory) cannot become resident next to its predecessor's, so there is little prologue to overlap; the gain with it on
// is not measured on the H100)
// the launch carries cudaLaunchAttributeProgrammaticStreamSerialization, so the
// grid may be scheduled while its predecessor in the stream is still draining: its launch latency and on-chip prologue
// (barrier init, descriptor prefetch) overlap the predecessor's tail instead of following it.  The
// contract every kernel keeps: pdl_trigger() first (dependents may be scheduled once ALL CTAs of this grid are
// resident -- so a waiting dependent can never starve CTAs of this grid that have not started), and pdl_wait() before
// the first global-memory access (reads of the predecessor's results AND writes: the allocator may hand a buffer the
// predecessor still reads to this kernel as output).  griddepcontrol.wait returns when the prerequisite grid has
// COMPLETED and flushed, so completion stays transitive along the stream exactly as without PDL.  Both instructions are
// no-ops for a launch without the attribute.  A step of ~470 launches of 10-60 us each has ~2-3 us of launch gap per
// kernel otherwise (CUDA graph replay included).
// ---------------------------------------------------------------------------------
bool pdl_enabled();

// SMs of the current device; launch sizes follow it (132 on an H100 SXM).  The fallback serves host-side sizing queries
// on a machine without a device, where nothing is launched.
inline int device_sms() {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        sms <= 0) {
        cudaGetLastError();
        return 132;
    }
    return sms;
}

__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_entry() {
    pdl_trigger();
    pdl_wait();
}

template <typename... KArgs, typename... Args>
inline cudaError_t lf_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

#define LF_REQUIRE(cond)                            \
    do {                                            \
        if (!(cond)) return LF_ERR_INVALID_ARGUMENT; \
    } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Packed fp32 pairs: two IEEE fp32 lanes in one 64-bit value, each lane rounded exactly like the scalar op (lsq.cu).
typedef unsigned long long f32x2_t;
__device__ __forceinline__ f32x2_t f2_pack(float lo, float hi) {
    f32x2_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void f2_unpack(f32x2_t v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ f32x2_t f2_mul(f32x2_t a, f32x2_t b) {
    float a0, a1, b0, b1;
    f2_unpack(a, a0, a1);
    f2_unpack(b, b0, b1);
    return f2_pack(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ f32x2_t f2_add(f32x2_t a, f32x2_t b) {
    float a0, a1, b0, b1;
    f2_unpack(a, a0, a1);
    f2_unpack(b, b0, b1);
    return f2_pack(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ f32x2_t f2_fma(f32x2_t a, f32x2_t b, f32x2_t c) {
    float a0, a1, b0, b1, c0, c1;
    f2_unpack(a, a0, a1);
    f2_unpack(b, b0, b1);
    f2_unpack(c, c0, c1);
    return f2_pack(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

// streaming 128-bit load (read once, do not pollute L1)
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ float ld_stream_f1(const float* p) {
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream_f4(float4* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ uint2 ld_stream_u2(const uint2* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ float4 bf16x4_to_f4(uint2 u) {
    float4 r;
    r.x = __uint_as_float(u.x << 16);
    r.y = __uint_as_float(u.x & 0xffff0000u);
    r.z = __uint_as_float(u.y << 16);
    r.w = __uint_as_float(u.y & 0xffff0000u);
    return r;
}
__device__ __forceinline__ uint2 f4_to_bf16x4(float4 v) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y);
    __nv_bfloat162 b = __floats2bfloat162_rn(v.z, v.w);
    uint2 r;
    r.x = *reinterpret_cast<uint32_t*>(&a);
    r.y = *reinterpret_cast<uint32_t*>(&b);
    return r;
}

}  // namespace lf
