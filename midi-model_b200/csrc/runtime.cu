// Error channel and device queries shared by all C-ABI entry points.
#include <stdarg.h>

#include "common.cuh"

static thread_local char g_err[512] = {0};

void b200_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char* b200_last_error(void) { return g_err; }

#include <atomic>
static std::atomic<long long> g_launches{0};
void b200_count_launches(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
extern "C" long long b200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int b200_num_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    }
    return sms;
}

extern "C" int b200_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    B200_CUDA(cudaGetDevice(&dev), "device_info");
    B200_CUDA(cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev), "device_info");
    B200_CUDA(cudaDeviceGetAttribute(cc_major, cudaDevAttrComputeCapabilityMajor, dev), "device_info");
    B200_CUDA(cudaDeviceGetAttribute(cc_minor, cudaDevAttrComputeCapabilityMinor, dev), "device_info");
    return B200_OK;
}

extern "C" int b200_abi_version(void) { return 1; }
