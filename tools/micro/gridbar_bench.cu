// Micro-benchmark of grid-wide barrier variants on one CTA per SM (cooperative launch): cycles per barrier, measured by
// CTA 0, with and without a burst of weight-like global loads issued by the other warps right before the barrier.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o gridbar_bench gridbar_bench.cu && ./gridbar_bench
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

template <int VARIANT>
__device__ __forceinline__ void grid_sync(unsigned* ctr, unsigned& target, unsigned n) {
    __syncthreads();
    target += n;
    if (threadIdx.x == 0) {
        if (VARIANT == 0) {            // cooperative-groups style: fence + atomic + acquire polling + fence
            __threadfence();
            atomicAdd(ctr, 1u);
            while (ld_acquire(ctr) < target) {}
            __threadfence();
        } else if (VARIANT == 1) {     // release reduction + relaxed polling
            asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
            while (ld_relaxed(ctr) < target) {}
        } else if (VARIANT == 2) {     // + back-off between polls
            asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
            while (ld_relaxed(ctr) < target) { __nanosleep(64); }
        } else if (VARIANT == 3) {     // last arriver flips a flag in a separate line; everyone polls the flag
            unsigned* flag = ctr + 32;
            const unsigned gen = target / n;
            __threadfence();
            const unsigned old = atomicAdd(ctr, 1u);
            if (old + 1 == target) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flag), "r"(gen) : "memory"); }
            else while (ld_relaxed(flag) < gen) {}
        }
    }
    __syncthreads();
}

template <int VARIANT>
__global__ void __launch_bounds__(512, 1) bench(unsigned* ctr, const uint4* w, size_t w_elems, int iters, int burst, long long* out,
                                                 uint4* sink) {
    unsigned target = 0;
    const unsigned n = gridDim.x;
    uint4 acc = make_uint4(0, 0, 0, 0);
    long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
        if (burst && threadIdx.x >= 32) {     // 15 warps x 32 lanes x 8 x 16 B = 61 KB per CTA, like one projection's prefetch
            const size_t base = ((size_t)it * gridDim.x + blockIdx.x) * 512 * 8 + threadIdx.x;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                uint4 v;
                const uint4* p = w + (base + (size_t)k * 512) % w_elems;
                asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
                if (burst == 2) { acc.x ^= v.x; acc.y ^= v.y; acc.z ^= v.z; acc.w ^= v.w; }   // burst == 2: consume before the barrier
                else { acc.x += (v.x & 0); }                                                  // burst == 1: value needed only at the end
            }
        }
        grid_sync<VARIANT>(ctr, target, n);
    }
    long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) out[0] = (t1 - t0) / iters;
    if (acc.x == 0x12345678u) sink[blockIdx.x * 512 + threadIdx.x] = acc;
}

template <int V>
void run(const char* name, unsigned* ctr, uint4* w, size_t w_elems, long long* out, uint4* sink, int sms) {
    for (int burst = 0; burst < 3; burst++) {
        cudaMemset(ctr, 0, 256);
        int iters = 2000;
        void* args[] = {&ctr, &w, &w_elems, &iters, &burst, &out, &sink};
        cudaLaunchCooperativeKernel((void*)bench<V>, dim3(sms), dim3(512), args, 0, 0);
        cudaError_t e = cudaDeviceSynchronize();
        long long h = 0;
        cudaMemcpy(&h, out, 8, cudaMemcpyDeviceToHost);
        printf("%-44s burst=%d : %6lld cycles / barrier  (%s)\n", name, burst, h, cudaGetErrorString(e));
    }
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    unsigned* ctr;
    long long* out;
    uint4 *w, *sink;
    const size_t w_elems = (size_t)512 << 20 >> 4;      // 512 MB of "weights"
    cudaMalloc(&ctr, 256);
    cudaMalloc(&out, 64);
    cudaMalloc(&w, w_elems * 16);
    cudaMalloc(&sink, (size_t)sms * 512 * 16);
    cudaMemset(w, 1, w_elems * 16);
    printf("SMs %d\n", sms);
    run<0>("fence+atomicAdd, acquire polling, fence", ctr, w, w_elems, out, sink, sms);
    run<1>("red.release, relaxed polling", ctr, w, w_elems, out, sink, sms);
    run<2>("red.release, relaxed polling + nanosleep(64)", ctr, w, w_elems, out, sink, sms);
    run<3>("atomicAdd ticket, last arriver sets flag", ctr, w, w_elems, out, sink, sms);
    return 0;
}
