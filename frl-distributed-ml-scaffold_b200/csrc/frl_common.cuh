// Shared device/host helpers for the frl_b200 kernels (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#include "frl_b200.h"

namespace frl {

// ---- error / launch bookkeeping (defined in api.cu) -----------------------------------------
void        set_error(const char* fmt, ...);
int         after_launch(const char* what);    // bumps the launch counter, returns cudaGetLastError()
int         sm_count();                        // cached SM count of the current device

#define FRL_REQUIRE(cond, code, ...)                  \
    do {                                              \
        if (!(cond)) {                                \
            frl::set_error(__VA_ARGS__);              \
            return (code);                            \
        }                                             \
    } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- 128-bit streaming loads / stores -------------------------------------------------------
// The arena is far larger than L2 and every element is touched once per step, so loads skip L1
// allocation and stores are marked streaming.
struct __align__(16) f32x4 { float x, y, z, w; };
struct __align__(16) bf16x8 { uint32_t a, b, c, d; };
struct __align__(8)  bf16x4 { uint32_t a, b; };

__device__ __forceinline__ f32x4 ld_stream(const f32x4* p) {
    f32x4 r;
    asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ f32x4 ld_stream_ro(const f32x4* p) {
    f32x4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ bf16x8 ld_stream_ro(const bf16x8* p) {
    bf16x8 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.a), "=r"(r.b), "=r"(r.c), "=r"(r.d) : "l"(p));
    return r;
}
__device__ __forceinline__ bf16x4 ld_stream_ro(const bf16x4* p) {
    bf16x4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];"
                 : "=r"(r.a), "=r"(r.b) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream(f32x4* p, const f32x4& v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void st_stream(bf16x4* p, const bf16x4& v) {
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};"
                 :: "l"(p), "r"(v.a), "r"(v.b) : "memory");
}
__device__ __forceinline__ void st_stream(bf16x8* p, const bf16x8& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.a), "r"(v.b), "r"(v.c), "r"(v.d) : "memory");
}

// ---- bf16 pack / unpack ---------------------------------------------------------------------
__device__ __forceinline__ float bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    // round-to-nearest-even, same rounding torch's float->bfloat16 copy uses
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_to_f32(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// ---- warp / block reductions ----------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// Sum over the block; result valid in thread 0. `smem` holds >= 32 floats. Fixed order.
__device__ __forceinline__ float block_sum(float v, float* smem) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();                 // smem may still be read from a previous call
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    const int nwarp = (blockDim.x + 31) >> 5;
    v = (threadIdx.x < nwarp) ? smem[threadIdx.x] : 0.f;
    if (warp == 0) v = warp_sum(v);
    return v;
}

}  // namespace frl
