// Host-side runtime of libstmgcn_b200.so: the thread-local error string, the launch counter, the SM count and the
// per-(kernel, device) dynamic shared memory attribute (declared in common.cuh), and the ABI's four getters.
#include "common.cuh"

#include <atomic>
#include <mutex>

namespace stmgcn {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int32_t fail(int32_t code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
int32_t check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail((int32_t)e, "%s: %s", what, cudaGetErrorString(e));
    return 0;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
// SMs of the current device.  If the device query fails, the H100 SXM's 132: only grid sizes depend on it, and the
// launch that follows reports the device error itself.
int sm_count() {
    constexpr int kFallback = 132;
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return kFallback;
    if (cached[dev] == 0) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = kFallback;
        cached[dev] = v;
    }
    return cached[dev];
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute: remember (kernel, device) pairs, not a
// process-wide flag, so a model moved to another GPU of the same process still launches; mutex: the forward thread and
// the autograd thread may both get here first.  The library registers 37 kernels: 12 lstm16 forward / backward variants,
// 3 in proj_tc.cu, 18 tall_gemm_kernel and 4 reduce_gemm_kernel instances; a kernel past the table would set the
// attribute on every launch.
int32_t ensure_dyn_smem(const void* kernel, size_t bytes) {
    constexpr int kMaxKernels = 64, kMaxDev = 64;
    static std::mutex mu;
    static const void* kernels[kMaxKernels] = {};
    static bool done[kMaxKernels][kMaxDev] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) dev = -1;
    std::lock_guard<std::mutex> lock(mu);
    int slot = -1;
    for (int i = 0; i < kMaxKernels; ++i) {
        if (kernels[i] == kernel) { slot = i; break; }
        if (kernels[i] == nullptr) { kernels[i] = kernel; slot = i; break; }
    }
    if (slot >= 0 && dev >= 0 && dev < kMaxDev && done[slot][dev]) return 0;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return fail((int32_t)e, "cudaFuncSetAttribute(MaxDynamicSharedMemorySize=%zu) failed: %s", bytes, cudaGetErrorString(e));
    if (slot >= 0 && dev >= 0 && dev < kMaxDev) done[slot][dev] = true;
    return 0;
}

}  // namespace stmgcn

extern "C" {

int32_t stmgcn_abi_version(void) { return STMGCN_ABI_VERSION; }
const char* stmgcn_last_error(void) { return stmgcn::g_err; }
int32_t stmgcn_sm_count(void) { return stmgcn::sm_count(); }
int64_t stmgcn_launch_count(void) { return stmgcn::g_launches.load(); }

}  // extern "C"
