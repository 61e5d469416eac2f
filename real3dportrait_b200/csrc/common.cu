// Error plumbing and device queries of libr3dp_b200.
#include "common.cuh"
#include <string.h>

namespace r3dp {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

static unsigned long long g_launches = 0;
void count_launches(int n) { __atomic_fetch_add(&g_launches, (unsigned long long)n, __ATOMIC_RELAXED); }

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

}  // namespace r3dp

extern "C" int r3dp_abi_version(void) { return R3DP_ABI_VERSION; }

extern "C" const char* r3dp_last_error(void) { return r3dp::g_err; }

extern "C" int r3dp_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    R3DP_CUDA(cudaGetDevice(&dev));
    int sms = 0, major = 0, minor = 0;
    R3DP_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    R3DP_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    R3DP_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (sm_count) *sm_count = sms;
    if (cc_major) *cc_major = major;
    if (cc_minor) *cc_minor = minor;
    R3DP_REQUIRE(major == 9 && minor == 0, "libr3dp_b200 is built for sm_90a only; current device is sm_%d%d", major, minor);
    return 0;
}

extern "C" unsigned long long r3dp_launch_count(void) { return __atomic_load_n(&r3dp::g_launches, __ATOMIC_RELAXED); }

extern "C" int r3dp_peer_copy(void* dst, int dst_device, const void* src, int src_device, size_t bytes, r3dp_stream_t stream) {
    R3DP_REQUIRE(dst && src && dst_device >= 0 && src_device >= 0, "peer_copy: bad arguments");
    if (bytes == 0) return 0;
    if (dst_device == src_device) { R3DP_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, r3dp::as_stream(stream))); return 0; }
    int can = 0;
    R3DP_CUDA(cudaDeviceCanAccessPeer(&can, src_device, dst_device));
    if (can) {                                       // direct NVLink path; without it the driver stages the copy through the host
        cudaError_t e = cudaDeviceEnablePeerAccess(dst_device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { R3DP_CUDA(e); }
        (void)cudaGetLastError();
    }
    R3DP_CUDA(cudaMemcpyPeerAsync(dst, dst_device, src, src_device, bytes, r3dp::as_stream(stream)));
    return 0;
}
