// Weight gradient of the stacked-K projection on the Hopper tensor cores (wgmma, register accumulators, 3xTF32 -- see
// tc_common.cuh):  dW[kd x 64] += [T_kX | T_{k+1}X]^T . dZ  per 128-row block of W (reference: the autograd of GCN.py:39).
// (The shared LSTM's own weight gradient is fused into lstm16_bwd_kernel, lstm16.cu; this kernel keeps the generic
// two-segment form.)
#include "tc_pipeline.cuh"
#include <stdlib.h>
#include <string.h>

using namespace stmgcn;
using namespace stmgcn::tc;

namespace {

// =====================================================================================================
// dW[kd x N] += sum over rows r of [seg0 | seg1][r, :]^T . da[r, :]
// M = kd index (padded to 128; warpgroup w owns kd rows 64w .. 64w+63), N = 64, K = rows, 32 rows per k-block.  Both
// operands are row-major in HBM (K is the slow dimension) and tf32 wgmma reads K-major operands only, so the loaders
// transpose on their way to shared memory: element (row r, m) lands at sw128_offset(m, r) of a [m][32 k] tile.  The
// accumulators live for the whole launch and are flushed with atomics once.
// =====================================================================================================
constexpr int kWgRows = 32;                                        // K per k-block
constexpr int kWgThreads = 256;
template <int N> struct WgCfg {
    static constexpr int kBBytes = N * kWgRows * 4;                // [N][32 k] K-major
    static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;
    static constexpr size_t kSmem = 1024 + (size_t)kStageBytes;
};

struct WgParams {
    const float* seg0;       // h_below tape base for this layer: (T, rows, 64) or nullptr (layer 0)
    const float* seg1;       // this layer's h tape base (T, rows, 64): read shifted by one step
    const float* h0;         // (rows, 64) value of h_{-1} or nullptr (zeros)
    const float* da;         // (T, rows, N)
    float* dwp;              // (kd, N) +=
    int shift1;              // 1: seg1 is read one step back (LSTM h_{t-1}); 0: same step (projection)
    int kd;                  // 128 or 64 (layer 0: only seg1)
    int t_len;
    int64_t rows;
    int64_t chunks_per_t;    // ceil(rows / 32)
    int64_t total_chunks;
};

template <int N>
__global__ void __launch_bounds__(kWgThreads, 1) lstm_wgrad_tc_kernel(const __grid_constant__ WgParams p) {
    using Cfg = WgCfg<N>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* st = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // keeps the __shared__ address space
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int wg = tid >> 7;
    constexpr int kNA = 1024 / kWgThreads, kNB = (kWgRows * N / 4) / kWgThreads;
    static_assert(kNB >= 1, "loader mapping");
    const uint32_t s_u = smem_u32(st);
    const uint32_t a_hi = s_u + (uint32_t)wg * 64u * 128u, a_lo = a_hi + kABytes;
    const uint32_t b_hi = s_u + 2 * kABytes, b_lo = b_hi + Cfg::kBBytes;
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    bool first = true;

    for (int64_t chunk = blockIdx.x; chunk < p.total_chunks; chunk += gridDim.x) {
        const int t = (int)(chunk / p.chunks_per_t);
        const int64_t r0 = (chunk % p.chunks_per_t) * kWgRows;
        const float* s0 = p.seg0 ? p.seg0 + (int64_t)t * p.rows * kHid : nullptr;
        const float* s1 = p.shift1 ? ((t > 0) ? p.seg1 + (int64_t)(t - 1) * p.rows * kHid : p.h0)
                                    : p.seg1 + (int64_t)t * p.rows * kHid;
        const float* dt = p.da + (int64_t)t * p.rows * N;
        float4 va[kNA], vb[kNB];
#pragma unroll
        for (int i = 0; i < kNA; ++i) {                   // A': 32 rows x 32 float4 (128 kd values), coalesced
            const int idx = tid + i * kWgThreads;
            const int row = idx >> 5, q = idx & 31;
            const int64_t r = r0 + row;
            // kd = 128: m 0..63 from seg0 (h_below), 64..127 from seg1 (h_prev); kd = 64: m 0..63 from seg1
            const float* src = (p.kd == 128) ? (q < 16 ? s0 : s1) : (q < 16 ? s1 : nullptr);
            va[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (src != nullptr && r < p.rows) va[i] = *reinterpret_cast<const float4*>(src + r * kHid + (q & 15) * 4);
        }
#pragma unroll
        for (int i = 0; i < kNB; ++i) {                   // B': 32 rows x N/4 float4, coalesced
            const int idx = tid + i * kWgThreads;
            const int row = idx / (N / 4), q = idx % (N / 4);
            const int64_t r = r0 + row;
            vb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < p.rows) vb[i] = *reinterpret_cast<const float4*>(dt + r * N + q * 4);
        }
        wg_wait<0>();
        __syncthreads();                                  // both warpgroups are done with the stage
#pragma unroll
        for (int i = 0; i < kNA; ++i) {
            const int idx = tid + i * kWgThreads;
            split_store_t(st, st + kABytes, (idx & 31) * 4, idx >> 5, va[i]);
        }
#pragma unroll
        for (int i = 0; i < kNB; ++i) {
            const int idx = tid + i * kWgThreads;
            split_store_t(st + 2 * kABytes, st + 2 * kABytes + Cfg::kBBytes, (idx % (N / 4)) * 4, idx / (N / 4), vb[i]);
        }
        fence_proxy_async_smem();
        __syncthreads();
        wg_fence_regs(acc);
        wg_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {
            const uint64_t da = smem_desc_k_sw128(pass == 1 ? a_lo : a_hi);
            const uint64_t db = smem_desc_k_sw128(pass == 2 ? b_lo : b_hi);
#pragma unroll
            for (int k = 0; k < kWgRows / 8; ++k)
                wgmma_tf32_n64(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (!first || pass > 0 || k > 0) ? 1u : 0u);
        }
        wg_commit();
        first = false;
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    if (first) return;                                    // no chunk: nothing accumulated
    // ===================== accumulator fragment (rows = kd index) -> atomics into dWp =====================
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = r0 + 8 * h;
        if (m >= p.kd) continue;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
            atomicAdd(p.dwp + (int64_t)m * N + 8 * j + c0, acc[4 * j + 2 * h]);
            atomicAdd(p.dwp + (int64_t)m * N + 8 * j + c0 + 1, acc[4 * j + 2 * h + 1]);
        }
    }
}


}  // namespace

namespace stmgcn {

// Weight-gradient reduction on the tensor cores for the projection (n = 64, shift1 = 0, t_len = 1): called from
// stmgcn_proj_bwd, once per 128-row block of dW.
int32_t launch_wgrad_tc(const float* seg0, const float* seg1, const float* h0, int shift1, const float* da, int n,
                        float* dwp, int kd, int t_len, int64_t rows, cudaStream_t st) {
    WgParams p;
    p.seg0 = seg0;
    p.seg1 = seg1;
    p.h0 = h0;
    p.da = da;
    p.dwp = dwp;
    p.shift1 = shift1;
    p.kd = kd;
    p.t_len = t_len;
    p.rows = rows;
    p.chunks_per_t = ceil_div(rows, kWgRows);
    p.total_chunks = p.chunks_per_t * t_len;
    const int64_t grid = p.total_chunks < sm_count() ? p.total_chunks : sm_count();
    STMGCN_REQUIRE(n == 64, STMGCN_ERR_SHAPE, "wgrad_tc: n=%d (only the projection's N = 64 is instantiated)", n);
    if (int32_t rc = ensure_dyn_smem((const void*)lstm_wgrad_tc_kernel<64>, WgCfg<64>::kSmem)) return rc;
    lstm_wgrad_tc_kernel<64><<<(int)grid, kWgThreads, WgCfg<64>::kSmem, st>>>(p);
    count_launch();
    return check_launch("wgrad_tc");
}

}  // namespace stmgcn
