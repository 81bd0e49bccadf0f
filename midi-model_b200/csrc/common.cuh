// Common device/host helpers for the sm_90a kernels of the MIDIModel hot path.
// Everything here is plain CUDA C++ + inline PTX (no CUTLASS / no torch types).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

typedef __nv_bfloat16 bf16;
typedef __nv_bfloat162 bf162;

// ---------------------------------------------------------------------------
// error reporting: every C-ABI entry returns 0 or a negative code; the message
// is kept per thread and read back with b200_last_error().
// ---------------------------------------------------------------------------
extern "C" const char* b200_last_error(void);
void b200_set_error(const char* fmt, ...);

#define B200_OK 0
#define B200_ERR_ARG (-1)
#define B200_ERR_CUDA (-2)
#define B200_ERR_UNSUPPORTED (-3)

#define B200_CHECK_ARG(cond, ...)                \
    do {                                         \
        if (!(cond)) {                           \
            b200_set_error(__VA_ARGS__);         \
            return B200_ERR_ARG;                 \
        }                                        \
    } while (0)

// every kernel launch of this library is counted (bench.py reports `gpu_launches` from it)
void b200_count_launches(int n);
#define B200_COUNT_EXTRA(n) b200_count_launches(n)

#define B200_CHECK_LAUNCH(name)                                                       \
    do {                                                                              \
        b200_count_launches(1);                                                       \
        cudaError_t e__ = cudaGetLastError();                                         \
        if (e__ != cudaSuccess) {                                                     \
            b200_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));   \
            return B200_ERR_CUDA;                                                     \
        }                                                                             \
    } while (0)

#define B200_CUDA(call, name)                                                         \
    do {                                                                              \
        cudaError_t e__ = (call);                                                     \
        if (e__ != cudaSuccess) {                                                     \
            b200_set_error("%s: %s", name, cudaGetErrorString(e__));                  \
            return B200_ERR_CUDA;                                                     \
        }                                                                             \
    } while (0)

int b200_num_sms();

// Programmatic dependent launch (PDL).  Kernels that run right before a tensor-core GEMM execute
// `griddepcontrol.launch_dependents` first thing: a GEMM launched with the programmatic-serialization attribute may then be
// scheduled onto SMs as they drain and run its prologue (barrier init, tensor-map prefetch) under this
// kernel's tail; it touches no memory before its own `griddepcontrol.wait`, which returns only once this grid has completed
// and flushed.  Without the launch attribute on the next kernel both instructions are no-ops.
#define B200_PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")
#define B200_PDL_WAIT() asm volatile("griddepcontrol.wait;" ::: "memory")

// ---------------------------------------------------------------------------
// small device helpers
// ---------------------------------------------------------------------------
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

// round-to-nearest-even fp32 -> bf16 -> fp32 (a "rounding point" of the reference's eager bf16 path)
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// silu(x) = x * sigmoid(x) with the SFU approximations (ex2.approx, rcp.approx: relative error ~2^-22, far below the bf16
// rounding that follows).  ONE definition for every kernel that forms SwiGLU (stand-alone kernels, GEMM epilogue, decode
// projections), so that fused and unfused paths stay bit-identical to each other.
__device__ __forceinline__ float sigmoid_f(float x) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-x * 1.4426950408889634f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.f + e));
    return r;
}
__device__ __forceinline__ float silu_f(float x) { return x * sigmoid_f(x); }

struct __align__(16) bf16x8 {
    bf162 v[4];
};

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    const bf162* p = reinterpret_cast<const bf162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        float2 t = __bfloat1622float2(p[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
    uint4 u;
    bf162* p = reinterpret_cast<bf162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; i++) p[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    return u;
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    bf162 t = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
}

__device__ __forceinline__ uint4 ld_nc16(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
