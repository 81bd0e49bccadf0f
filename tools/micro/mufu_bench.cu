// Micro-benchmark of the exponential path of the attention softmax on one SM sub-partition: cycles per warp-level
// MUFU.EX2 as a function of warps per sub-partition and of the instruction mix around it (the softmax inner loop issues,
// per element, 1 FFMA (scale), 1 MUFU.EX2, 1 FADD (row sum) and 1/2 F2FP (bf16 pack)).  Also: packed half-precision
// exponentials, and a degree-3 polynomial 2^x on the FMA pipe.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o mufu_bench mufu_bench.cu && ./mufu_bench
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ float ex2(float x) {
    float y;
    asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t ex2_h2(uint32_t x) {
    uint32_t y;
    asm volatile("ex2.approx.f16x2 %0, %1;" : "=r"(y) : "r"(x));
    return y;
}
__device__ __forceinline__ uint32_t ex2_bf2(uint32_t x) {
    uint32_t y;
    asm volatile("ex2.approx.ftz.bf16x2 %0, %1;" : "=r"(y) : "r"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_bf2(float a, float b) {
    uint32_t y;
    asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(y) : "f"(b), "f"(a));
    return y;
}
// 2^x for x <= 0 on the FMA pipe: round-to-nearest split x = n + f, |f| <= 0.5, degree-3 minimax of 2^f, exponent add
__device__ __forceinline__ float ex2_poly(float x) {
    x = fmaxf(x, -125.f);
    const float r = x + 12582912.f;              // 1.5 * 2^23: the integer part lands in the low mantissa bits
    const float n = r - 12582912.f;
    const float f = x - n;
    float p = fmaf(f, 0.0555041f, 0.2402265f);
    p = fmaf(p, f, 0.6931472f);
    p = fmaf(p, f, 1.0f);
    return __int_as_float(__float_as_int(p) + (__float_as_int(r) << 23));
}

// MODE 0: MUFU only   1: FFMA + MUFU + FADD + pack (the softmax mix)   2: f16x2 exponentials   3: bf16x2 exponentials
// MODE 4: the mix with every 4th exponential on the FMA pipe          5: polynomial only
template <int MODE>
__global__ void bench(float* out, long long* cycles, int iters, float seed) {
    float x[16];
#pragma unroll
    for (int i = 0; i < 16; i++) x[i] = seed * (float)(i + 1 + (threadIdx.x & 7));
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    uint32_t keep = 0;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        if (MODE == 0) {
#pragma unroll
            for (int i = 0; i < 16; i++) x[i] = ex2(x[i]) - 1.0f;
        } else if (MODE == 1 || MODE == 4) {
#pragma unroll
            for (int i = 0; i < 16; i += 2) {
                const float a = fmaf(x[i], 0.18f, -seed), b = fmaf(x[i + 1], 0.18f, -seed);
                const float p0 = ex2(a);
                const float p1 = (MODE == 4 && (i & 2)) ? ex2_poly(b) : ex2(b);
                acc[(i >> 1) & 3] += p0 + p1;
                keep ^= pack_bf2(p0, p1);
                x[i] = p0 - 1.0f; x[i + 1] = p1 - 1.0f;
            }
        } else if (MODE == 2 || MODE == 3) {
#pragma unroll
            for (int i = 0; i < 16; i++) {
                uint32_t u = __float_as_uint(x[i]);
                u = (MODE == 2) ? ex2_h2(u) : ex2_bf2(u);
                x[i] = __uint_as_float(u & 0x3c003c00u);
            }
        } else {
#pragma unroll
            for (int i = 0; i < 16; i++) x[i] = ex2_poly(x[i] * 0.18f - seed) - 1.0f;
        }
    }
    const long long t1 = clock64();
    float s = acc[0] + acc[1] + acc[2] + acc[3] + __uint_as_float(keep & 0x3f800000u);
#pragma unroll
    for (int i = 0; i < 16; i++) s += x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int MODE>
void run(const char* name, int exps_per_iter_per_thread) {
    float* out; long long* cyc;
    cudaMalloc(&out, 132 * 1024 * sizeof(float));
    cudaMalloc(&cyc, 132 * sizeof(long long));
    const int iters = 2000;
    for (int wps = 1; wps <= 4; wps *= 2) {       // warps per sub-partition
        const int threads = 128 * wps;
        bench<MODE><<<132, threads>>>(out, cyc, 10, 0.25f);
        bench<MODE><<<132, threads>>>(out, cyc, iters, 0.25f);
        cudaDeviceSynchronize();
        long long h[132];
        cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
        double avg = 0;
        for (int i = 0; i < 132; i++) avg += (double)h[i];
        avg /= 132;
        // warp-level exponential instructions issued per sub-partition = wps * iters * exps_per_iter
        printf("%-44s warps/SMSP %d : %7.2f cycles per warp-exponential per SMSP  (%s)\n", name, wps,
               avg / ((double)wps * iters * exps_per_iter_per_thread), cudaGetErrorString(cudaGetLastError()));
    }
    cudaFree(out); cudaFree(cyc);
}

int main() {
    run<0>("MUFU.EX2 only (16 independent chains)", 16);
    run<1>("softmax mix: FFMA + MUFU + FADD + pack", 16);
    run<4>("softmax mix, every 4th 2^x on the FMA pipe", 16);
    run<5>("polynomial 2^x only", 16);
    run<2>("ex2.approx.f16x2 (2 results per instruction)", 16);
    run<3>("ex2.approx.ftz.bf16x2", 16);
    return 0;
}
