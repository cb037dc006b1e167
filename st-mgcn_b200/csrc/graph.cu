// Graph handles: the constant operand of GCN.forward (reference GCN.py:24-36 receives dense (K+1,N,N)
// supports; the hot path keeps supports[1] -- the rescaled Laplacian -- as CSR and CSR^T on the device).
// One-time setup code: cub (CUDA toolkit, header-only) is used for the scans and the transpose sort.
#include "common.cuh"
#include <mutex>

#include <cub/cub.cuh>
#include <atomic>
#include <string.h>
#include <stdlib.h>

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

using namespace stmgcn;

struct stmgcn_graph {
    int64_t n = 0, nnz = 0;
    int device = 0;
    int32_t* rowptr = nullptr;
    int32_t* colidx = nullptr;
    float* vals = nullptr;
    bool has_t = false;
    int32_t* t_rowptr = nullptr;
    int32_t* t_colidx = nullptr;
    float* t_vals = nullptr;
};

namespace {

// one warp per row: count entries != 0
__global__ void count_row_nnz_kernel(const float* __restrict__ dense, int64_t n, int64_t ld,
                                     int32_t* __restrict__ counts) {
    int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= n) return;
    const float* p = dense + row * ld;
    int c = 0;
    for (int64_t j = lane; j < n; j += 32) c += (p[j] != 0.0f);
    c = (int)warp_sum((float)c);   // counts < 2^24: exact in fp32
    if (lane == 0) counts[row] = c;
}

// one warp per row: ordered compaction (columns ascending)
__global__ void fill_rows_kernel(const float* __restrict__ dense, int64_t n, int64_t ld,
                                 const int32_t* __restrict__ rowptr, int32_t* __restrict__ colidx,
                                 float* __restrict__ vals) {
    int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= n) return;
    const float* p = dense + row * ld;
    int32_t base = rowptr[row];
    for (int64_t j0 = 0; j0 < n; j0 += 32) {
        int64_t j = j0 + lane;
        float v = (j < n) ? p[j] : 0.0f;
        unsigned m = __ballot_sync(0xffffffffu, v != 0.0f);
        if (v != 0.0f) {
            int pos = base + __popc(m & ((1u << lane) - 1u));
            colidx[pos] = (int32_t)j;
            vals[pos] = v;
        }
        base += __popc(m);
    }
}

__global__ void make_keys_kernel(int64_t n, const int32_t* __restrict__ rowptr,
                                 const int32_t* __restrict__ colidx, uint64_t* __restrict__ keys,
                                 int32_t* __restrict__ col_counts) {
    // one warp per row
    int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int lane = threadIdx.x & 31;
    if (row >= n) return;
    for (int32_t i = rowptr[row] + lane; i < rowptr[row + 1]; i += 32) {
        int32_t c = colidx[i];
        keys[i] = ((uint64_t)(uint32_t)c << 32) | (uint64_t)(uint32_t)row;
        atomicAdd(&col_counts[c], 1);
    }
}

__global__ void unpack_keys_kernel(int64_t nnz, const uint64_t* __restrict__ keys,
                                   int32_t* __restrict__ t_colidx) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nnz) t_colidx[i] = (int32_t)(uint32_t)(keys[i] & 0xffffffffull);
}

int32_t exclusive_scan(const int32_t* in, int32_t* out, int64_t count, cudaStream_t st) {
    size_t bytes = 0;
    STMGCN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int)count, st));
    void* tmp = nullptr;
    STMGCN_CUDA(cudaMalloc(&tmp, bytes ? bytes : 16));
    cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, (int)count, st);
    count_launch(2);
    cudaError_t e2 = cudaStreamSynchronize(st);
    cudaFree(tmp);
    if (e != cudaSuccess) return fail((int32_t)e, "cub scan: %s", cudaGetErrorString(e));
    if (e2 != cudaSuccess) return fail((int32_t)e2, "cub scan sync: %s", cudaGetErrorString(e2));
    return 0;
}

int32_t build_transpose(stmgcn_graph* g, cudaStream_t st) {
    const int64_t n = g->n, nnz = g->nnz;
    STMGCN_CUDA(cudaMalloc(&g->t_rowptr, (n + 1) * sizeof(int32_t)));
    STMGCN_CUDA(cudaMalloc(&g->t_colidx, (nnz ? nnz : 1) * sizeof(int32_t)));
    STMGCN_CUDA(cudaMalloc(&g->t_vals, (nnz ? nnz : 1) * sizeof(float)));
    int32_t* counts = nullptr;
    uint64_t *keys_in = nullptr, *keys_out = nullptr;
    void* tmp = nullptr;
    int32_t rc = 0;
    do {
        if ((rc = cudaMalloc(&counts, (n + 1) * sizeof(int32_t)))) break;
        if ((rc = cudaMemsetAsync(counts, 0, (n + 1) * sizeof(int32_t), st))) break;
        if (nnz > 0) {
            if ((rc = cudaMalloc(&keys_in, nnz * sizeof(uint64_t)))) break;
            if ((rc = cudaMalloc(&keys_out, nnz * sizeof(uint64_t)))) break;
            make_keys_kernel<<<(unsigned)ceil_div(n, 8), 256, 0, st>>>(n, g->rowptr, g->colidx, keys_in, counts);
            count_launch();
            size_t bytes = 0;
            if ((rc = cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys_in, keys_out, g->vals, g->t_vals,
                                                      (int)nnz, 0, 64, st))) break;
            if ((rc = cudaMalloc(&tmp, bytes ? bytes : 16))) break;
            if ((rc = cub::DeviceRadixSort::SortPairs(tmp, bytes, keys_in, keys_out, g->vals, g->t_vals,
                                                      (int)nnz, 0, 64, st))) break;
            count_launch(8);
            unpack_keys_kernel<<<(unsigned)ceil_div(nnz, 256), 256, 0, st>>>(nnz, keys_out, g->t_colidx);
            count_launch();
        }
        rc = exclusive_scan(counts, g->t_rowptr, n + 1, st);
    } while (0);
    cudaStreamSynchronize(st);
    cudaFree(counts);
    cudaFree(keys_in);
    cudaFree(keys_out);
    cudaFree(tmp);
    if (rc > 0) return fail(rc, "transpose build: %s", cudaGetErrorString((cudaError_t)rc));
    if (rc < 0) return rc;
    g->has_t = true;
    return check_launch("transpose build");
}


void free_graph(stmgcn_graph* g) {
    if (!g) return;
    cudaFree(g->rowptr);
    cudaFree(g->colidx);
    cudaFree(g->vals);
    cudaFree(g->t_rowptr);
    cudaFree(g->t_colidx);
    cudaFree(g->t_vals);
    delete g;
}

}  // namespace

extern "C" {

int32_t stmgcn_abi_version(void) { return STMGCN_ABI_VERSION; }
const char* stmgcn_last_error(void) { return stmgcn::g_err; }
int32_t stmgcn_sm_count(void) { return stmgcn::sm_count(); }
int64_t stmgcn_launch_count(void) { return stmgcn::g_launches.load(); }

int32_t stmgcn_graph_from_dense(stmgcn_graph_t** out, const float* dense, int64_t n, int64_t ld,
                                int32_t build_t, void* stream) {
    STMGCN_REQUIRE(out && dense, STMGCN_ERR_ARG, "graph_from_dense: null pointer");
    STMGCN_REQUIRE(n > 0 && ld >= n && n < (1ll << 30), STMGCN_ERR_SHAPE, "graph_from_dense: n=%lld ld=%lld",
                   (long long)n, (long long)ld);
    cudaStream_t st = (cudaStream_t)stream;
    stmgcn_graph* g = new stmgcn_graph();
    g->n = n;
    cudaGetDevice(&g->device);
    int32_t* counts = nullptr;
    int32_t rc = 0;
    do {
        if ((rc = cudaMalloc(&counts, (n + 1) * sizeof(int32_t)))) break;
        if ((rc = cudaMemsetAsync(counts, 0, (n + 1) * sizeof(int32_t), st))) break;
        if ((rc = cudaMalloc(&g->rowptr, (n + 1) * sizeof(int32_t)))) break;
        count_row_nnz_kernel<<<(unsigned)ceil_div(n, 8), 256, 0, st>>>(dense, n, ld, counts);
        count_launch();
        if ((rc = exclusive_scan(counts, g->rowptr, n + 1, st))) break;
        int32_t total = 0;
        if ((rc = cudaMemcpyAsync(&total, g->rowptr + n, sizeof(int32_t), cudaMemcpyDeviceToHost, st))) break;
        if ((rc = cudaStreamSynchronize(st))) break;
        g->nnz = total;
        if ((rc = cudaMalloc(&g->colidx, (total ? total : 1) * sizeof(int32_t)))) break;
        if ((rc = cudaMalloc(&g->vals, (total ? total : 1) * sizeof(float)))) break;
        fill_rows_kernel<<<(unsigned)ceil_div(n, 8), 256, 0, st>>>(dense, n, ld, g->rowptr, g->colidx, g->vals);
        count_launch();
        if ((rc = check_launch("graph_from_dense"))) break;
        if (build_t) rc = build_transpose(g, st);
    } while (0);
    cudaFree(counts);
    if (rc != 0) {
        free_graph(g);
        if (rc > 0) return fail(rc, "graph_from_dense: %s", cudaGetErrorString((cudaError_t)rc));
        return rc;
    }
    *out = g;
    return 0;
}

int32_t stmgcn_graph_from_csr(stmgcn_graph_t** out, int64_t n, int64_t nnz, const int32_t* rowptr,
                              const int32_t* colidx, const float* vals, int32_t build_t, void* stream) {
    STMGCN_REQUIRE(out && rowptr && (nnz == 0 || (colidx && vals)), STMGCN_ERR_ARG, "graph_from_csr: null pointer");
    STMGCN_REQUIRE(n > 0 && nnz >= 0 && n < (1ll << 30) && nnz < (1ll << 31), STMGCN_ERR_SHAPE,
                   "graph_from_csr: n=%lld nnz=%lld", (long long)n, (long long)nnz);
    cudaStream_t st = (cudaStream_t)stream;
    stmgcn_graph* g = new stmgcn_graph();
    g->n = n;
    g->nnz = nnz;
    cudaGetDevice(&g->device);
    int32_t rc = 0;
    do {
        if ((rc = cudaMalloc(&g->rowptr, (n + 1) * sizeof(int32_t)))) break;
        if ((rc = cudaMalloc(&g->colidx, (nnz ? nnz : 1) * sizeof(int32_t)))) break;
        if ((rc = cudaMalloc(&g->vals, (nnz ? nnz : 1) * sizeof(float)))) break;
        if ((rc = cudaMemcpyAsync(g->rowptr, rowptr, (n + 1) * sizeof(int32_t), cudaMemcpyDeviceToDevice, st))) break;
        if (nnz) {
            if ((rc = cudaMemcpyAsync(g->colidx, colidx, nnz * sizeof(int32_t), cudaMemcpyDeviceToDevice, st))) break;
            if ((rc = cudaMemcpyAsync(g->vals, vals, nnz * sizeof(float), cudaMemcpyDeviceToDevice, st))) break;
        }
        if ((rc = cudaStreamSynchronize(st))) break;
        if (build_t) rc = build_transpose(g, st);
    } while (0);
    if (rc != 0) {
        free_graph(g);
        if (rc > 0) return fail(rc, "graph_from_csr: %s", cudaGetErrorString((cudaError_t)rc));
        return rc;
    }
    *out = g;
    return 0;
}

int32_t stmgcn_graph_destroy(stmgcn_graph_t* g) {
    free_graph(g);
    return 0;
}
int64_t stmgcn_graph_n(const stmgcn_graph_t* g) { return g ? g->n : -1; }
int64_t stmgcn_graph_nnz(const stmgcn_graph_t* g) { return g ? g->nnz : -1; }

int32_t stmgcn_graph_export(const stmgcn_graph_t* g, int32_t transpose, int32_t* rowptr, int32_t* colidx,
                            float* vals, void* stream) {
    STMGCN_REQUIRE(g && rowptr && colidx && vals, STMGCN_ERR_ARG, "graph_export: null pointer");
    STMGCN_REQUIRE(!transpose || g->has_t, STMGCN_ERR_STATE, "graph_export: handle has no transpose");
    cudaStream_t st = (cudaStream_t)stream;
    const int32_t* rp = transpose ? g->t_rowptr : g->rowptr;
    const int32_t* ci = transpose ? g->t_colidx : g->colidx;
    const float* va = transpose ? g->t_vals : g->vals;
    STMGCN_CUDA(cudaMemcpyAsync(rowptr, rp, (g->n + 1) * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (g->nnz) {
        STMGCN_CUDA(cudaMemcpyAsync(colidx, ci, g->nnz * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
        STMGCN_CUDA(cudaMemcpyAsync(vals, va, g->nnz * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    return 0;
}

}  // extern "C"

// accessor used by spmm.cu (same shared object)
namespace stmgcn {
void graph_view(const stmgcn_graph* g, bool transpose, int64_t* n, int64_t* nnz, const int32_t** rowptr,
                const int32_t** colidx, const float** vals, bool* ok) {
    *n = g->n;
    *nnz = g->nnz;
    *ok = !transpose || g->has_t;
    *rowptr = transpose ? g->t_rowptr : g->rowptr;
    *colidx = transpose ? g->t_colidx : g->colidx;
    *vals = transpose ? g->t_vals : g->vals;
}
}  // namespace stmgcn
