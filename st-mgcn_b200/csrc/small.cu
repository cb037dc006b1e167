// Small memory-bound kernels around the three hot kernels: the training windows gathered from a resident series
// (Data_Container.py:114-146), layout change of the observations, the context gate's tiny FC (STMGCN.py:42-43) and the
// fusion over graphs + output FC (STMGCN.py:116-118).
#include "common.cuh"

using namespace stmgcn;

namespace {

// obs (B,T,N,C) -> xo (N,B,T,C), xt (N,B,T) = sum_c      (STMGCN.py:36, :39, :47)
__global__ void obs_to_node_major_kernel(const float* __restrict__ obs, float* __restrict__ xo,
                                         float* __restrict__ xt, int64_t b_sz, int64_t t_len, int64_t n,
                                         int64_t c_in) {
    // one thread per (n, b, t); consecutive threads walk t then b (coalesced writes, strided reads;
    // the whole tensor is ~13 MB at 4096 regions x 64 windows x 12 steps).
    const int64_t total = n * b_sz * t_len;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = i % t_len;
        const int64_t b = (i / t_len) % b_sz;
        const int64_t nn = i / (t_len * b_sz);
        const float* src = obs + ((b * t_len + t) * n + nn) * c_in;
        float sum = 0.f;
        for (int64_t c = 0; c < c_in; ++c) {
            const float v = src[c];
            sum += v;
            if (xo != nullptr) xo[i * c_in + c] = v;
        }
        xt[i] = sum;
    }
}

// adjoint of obs_to_node_major: d_obs[b,t,n,c] = d_xo[n,b,t,c] + d_xt[n,b,t]   (either input may be NULL)
__global__ void obs_grad_kernel(const float* __restrict__ d_xo, const float* __restrict__ d_xt, float* __restrict__ d_obs,
                                int64_t b_sz, int64_t t_len, int64_t n, int64_t c_in) {
    // one thread per (b, t, n); consecutive threads walk n (coalesced writes, strided reads)
    const int64_t total = b_sz * t_len * n;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t nn = i % n;
        const int64_t bt = i / n;                           // = b * t_len + t
        const int64_t j = nn * b_sz * t_len + bt;           // (n, b, t) node-major
        const float g = d_xt != nullptr ? d_xt[j] : 0.f;
        for (int64_t c = 0; c < c_in; ++c) d_obs[i * c_in + c] = (d_xo != nullptr ? d_xo[j * c_in + c] : 0.f) + g;
    }
}

// ---- context gate ----------------------------------------------------------------------------------
// one limit for both directions: the backward keeps 4*T floats in (default, 48 KB) dynamic shared memory
constexpr int kMaxGateSteps = 2048;

// one CTA per window b; T threads-worth of work looped over blockDim
__global__ void gate_fwd_kernel(const float* __restrict__ pool, int t_len, float inv_n,
                                const float* __restrict__ fcw, const float* __restrict__ fcb,
                                float* __restrict__ z, float* __restrict__ a1, float* __restrict__ s) {
    extern __shared__ float sm[];            // z[T], r1[T]
    float* zs = sm;
    float* rs = sm + t_len;
    const int64_t b = blockIdx.x;
    for (int j = threadIdx.x; j < t_len; j += blockDim.x) {
        const float v = pool[b * t_len + j] * inv_n;
        zs[j] = v;
        z[b * t_len + j] = v;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < t_len; j += blockDim.x) {
        float acc = fcb[j];
        for (int i = 0; i < t_len; ++i) acc = fmaf(fcw[j * t_len + i], zs[i], acc);
        a1[b * t_len + j] = acc;
        rs[j] = relu_(acc);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < t_len; j += blockDim.x) {
        float acc = fcb[j];
        for (int i = 0; i < t_len; ++i) acc = fmaf(fcw[j * t_len + i], rs[i], acc);
        s[b * t_len + j] = sigmoidf_(acc);
    }
}

__global__ void gate_bwd_kernel(const float* __restrict__ d_s, const float* __restrict__ z,
                                const float* __restrict__ a1, const float* __restrict__ s, int t_len,
                                const float* __restrict__ fcw, float* __restrict__ d_fcw,
                                float* __restrict__ d_fcb, float* __restrict__ d_z) {
    extern __shared__ float sm[];            // da2[T], da1[T], r1[T], z[T]
    float* da2 = sm;
    float* da1 = sm + t_len;
    float* r1 = sm + 2 * t_len;
    float* zs = sm + 3 * t_len;
    const int64_t b = blockIdx.x;
    for (int j = threadIdx.x; j < t_len; j += blockDim.x) {
        const float sv = s[b * t_len + j];
        da2[j] = d_s[b * t_len + j] * sv * (1.f - sv);
        r1[j] = relu_(a1[b * t_len + j]);
        zs[j] = z[b * t_len + j];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < t_len; i += blockDim.x) {
        float acc = 0.f;                                     // d r1[i] = sum_j da2[j] fcw[j,i]
        for (int j = 0; j < t_len; ++j) acc = fmaf(da2[j], fcw[j * t_len + i], acc);
        da1[i] = (a1[b * t_len + i] <= 0.f) ? 0.f : acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < t_len; i += blockDim.x) {
        float acc = 0.f;                                     // d z[i] = sum_j da1[j] fcw[j,i]
        for (int j = 0; j < t_len; ++j) acc = fmaf(da1[j], fcw[j * t_len + i], acc);
        d_z[b * t_len + i] = acc;
        if (d_fcb != nullptr) atomicAdd(&d_fcb[i], da2[i] + da1[i]);
    }
    if (d_fcw == nullptr) return;                            // d_z only (d_fcw and d_fcb go together)
    for (int e = threadIdx.x; e < t_len * t_len; e += blockDim.x) {
        const int j = e / t_len, i = e % t_len;              // fc used twice: both uses accumulate
        atomicAdd(&d_fcw[e], da2[j] * r1[i] + da1[j] * zs[i]);
    }
}

// ---- fusion over graphs + output FC -------------------------------------------------------------------
constexpr int kMaxGraphs = 8;
// C*G + C floats: the backward's shared-memory accumulator (48 KB); the forward takes the same limit, so no shape runs its
// forward and is then refused by its backward
constexpr int kMaxFuseFloats = 48 * 1024 / 4;
struct GraphPtrs {
    const float* g[kMaxGraphs];
};

// one warp per node-major row r = n*B + b
__global__ void fuse_out_fwd_kernel(GraphPtrs gp, int m, int64_t n, int64_t b_sz, int gdim, int c_out,
                                    const float* __restrict__ fcw, const float* __restrict__ fcb,
                                    float* __restrict__ feat, float* __restrict__ y) {
    const int lane = threadIdx.x & 31;
    const int64_t rows = n * b_sz;
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows;
         r += (int64_t)gridDim.x * (blockDim.x >> 5)) {
        const int64_t nn = r / b_sz, b = r % b_sz;
        for (int c = 0; c < c_out; ++c) {
            float dot = 0.f;
            for (int g = lane; g < gdim; g += 32) {
                float v = 0.f;
                for (int k = 0; k < m; ++k) v += gp.g[k][r * gdim + g];
                if (c == 0) feat[r * gdim + g] = v;
                dot = fmaf(v, fcw[c * gdim + g], dot);
            }
            dot = warp_sum(dot);
            if (lane == 0) y[(b * n + nn) * c_out + c] = dot + fcb[c];
        }
    }
}

__global__ void fuse_out_bwd_kernel(const float* __restrict__ d_y, const float* __restrict__ feat, int64_t n,
                                    int64_t b_sz, int gdim, int c_out, const float* __restrict__ fcw,
                                    float* __restrict__ d_feat, float* __restrict__ d_fcw,
                                    float* __restrict__ d_fcb) {
    extern __shared__ float sacc[];          // c_out*gdim + c_out
    const int lane = threadIdx.x & 31;
    const bool wgrad = d_fcw != nullptr;     // else d_feat only (d_fcw and d_fcb go together)
    const int n_acc = c_out * gdim + c_out;
    for (int e = threadIdx.x; e < n_acc; e += blockDim.x) sacc[e] = 0.f;
    __syncthreads();
    const int64_t rows = n * b_sz;
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows;
         r += (int64_t)gridDim.x * (blockDim.x >> 5)) {
        const int64_t nn = r / b_sz, b = r % b_sz;
        const float* dyr = d_y + (b * n + nn) * c_out;
        for (int g = lane; g < gdim; g += 32) {
            const float fv = feat[r * gdim + g];
            float acc = 0.f;
            for (int c = 0; c < c_out; ++c) {
                const float dv = dyr[c];
                acc = fmaf(dv, fcw[c * gdim + g], acc);
                if (wgrad) atomicAdd(&sacc[c * gdim + g], dv * fv);
            }
            d_feat[r * gdim + g] = acc;
        }
        if (!wgrad) continue;
        if (lane < c_out) atomicAdd(&sacc[c_out * gdim + lane], dyr[lane]);
        for (int c = 32 + lane; c < c_out; c += 32) atomicAdd(&sacc[c_out * gdim + c], dyr[c]);
    }
    if (!wgrad) return;
    __syncthreads();
    for (int e = threadIdx.x; e < c_out * gdim; e += blockDim.x) atomicAdd(&d_fcw[e], sacc[e]);
    for (int e = threadIdx.x; e < c_out; e += blockDim.x) atomicAdd(&d_fcb[e], sacc[c_out * gdim + e]);
}

// ---- training windows gathered from a resident series ---------------------------------------------------
// One limit with the context gate: T <= 2048.  The lags travel by value in the kernel's parameter block (8 KB at the
// limit, above the classic 4 KB: CUDA >= 12.1 on sm_70+), read from the constant bank through __grid_constant__.
constexpr int kMaxGatherSteps = 2048;
struct GatherLags {
    int32_t v[kMaxGatherSteps];
};
constexpr int kGatherThreads = 256;
constexpr int kGatherUnroll = 4;                        // elements per thread per tile: loads issued before stores
constexpr int64_t kGatherTile = kGatherThreads * kGatherUnroll;

// A tile is one destination row (an obs row (k, t) or the target row k) times one span of kGatherTile elements of V
// (float4 or float).  Slot j < t_len of window k reads series row wrap(first + k - lags[j]), slot t_len reads first + k.
// A plain copy: loads and stores only, so output bits are input bits.
template <typename V>
__global__ void __launch_bounds__(kGatherThreads)
window_gather_kernel(const V* __restrict__ series, int64_t s_len, int64_t row, const __grid_constant__ GatherLags lags,
                     int t_len, int64_t first, int64_t b, V* __restrict__ obs, V* __restrict__ y) {
    const int64_t spans = (row + kGatherTile - 1) / kGatherTile;
    const int64_t tiles = b * (t_len + 1) * spans;
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t slot = tile / spans;
        const int64_t c0 = (tile - slot * spans) * kGatherTile + threadIdx.x;
        const int64_t k = slot / (t_len + 1);
        const int j = (int)(slot - k * (t_len + 1));
        int64_t src_row = first + k;
        V* dst = y + k * row;
        if (j < t_len) {
            src_row -= lags.v[j];
            if (src_row < 0) src_row += s_len;             // numpy's negative index (checked >= -s_len at enqueue)
            dst = obs + (k * t_len + j) * row;
        }
        const V* src = series + src_row * row;
        V v[kGatherUnroll];
#pragma unroll
        for (int u = 0; u < kGatherUnroll; ++u) {
            const int64_t c = c0 + u * kGatherThreads;
            if (c < row) v[u] = src[c];
        }
#pragma unroll
        for (int u = 0; u < kGatherUnroll; ++u) {
            const int64_t c = c0 + u * kGatherThreads;
            if (c < row) dst[c] = v[u];
        }
    }
}

}  // namespace

extern "C" {

int32_t stmgcn_window_gather(const float* series, int64_t s_len, int64_t row, const int32_t* lags, int32_t t_len,
                             int64_t first, int64_t b, float* obs, float* y, void* stream) {
    STMGCN_REQUIRE(series && lags && obs && y, STMGCN_ERR_ARG, "window_gather: null pointer");
    STMGCN_REQUIRE(s_len > 0 && row > 0 && b > 0 && t_len > 0, STMGCN_ERR_SHAPE,
                   "window_gather: bad shape (s_len=%lld row=%lld b=%lld t_len=%d)", (long long)s_len, (long long)row,
                   (long long)b, (int)t_len);
    STMGCN_REQUIRE(t_len <= kMaxGatherSteps, STMGCN_ERR_SHAPE, "window_gather: T=%d (max %d)", (int)t_len, kMaxGatherSteps);
    // byte counts below must fit in int64: series s_len*row floats, obs b*t_len*row floats (b <= s_len by the next check)
    STMGCN_REQUIRE(row <= INT64_MAX / 4 / s_len / (kMaxGatherSteps + 1), STMGCN_ERR_SHAPE,
                   "window_gather: s_len=%lld x row=%lld too large", (long long)s_len, (long long)row);
    STMGCN_REQUIRE(first >= 0 && first <= s_len && b <= s_len - first, STMGCN_ERR_SHAPE,
                   "window_gather: windows [%lld, %lld) run past the series (s_len=%lld)", (long long)first,
                   (long long)first + (long long)b, (long long)s_len);
    GatherLags lv;
    for (int t = 0; t < t_len; ++t) {
        STMGCN_REQUIRE(lags[t] >= 0, STMGCN_ERR_ARG, "window_gather: lags[%d]=%d is negative", t, (int)lags[t]);
        STMGCN_REQUIRE(first - lags[t] >= -s_len, STMGCN_ERR_SHAPE,
                       "window_gather: lags[%d]=%d reaches row %lld, before -s_len=%lld", t, (int)lags[t],
                       (long long)(first - lags[t]), (long long)-s_len);
        lv.v[t] = lags[t];
    }
    const int64_t s_bytes = s_len * row * 4, obs_bytes = b * t_len * row * 4, y_bytes = b * row * 4;
    STMGCN_REQUIRE(!overlaps(obs, obs_bytes, series, s_bytes) && !overlaps(y, y_bytes, series, s_bytes), STMGCN_ERR_ARG,
                   "window_gather: obs / y overlap the series");
    STMGCN_REQUIRE(!overlaps(obs, obs_bytes, y, y_bytes), STMGCN_ERR_ARG, "window_gather: obs and y overlap");
    const bool vec4 = row % 4 == 0 && aligned16(series) && aligned16(obs) && aligned16(y);
    const int64_t row_v = vec4 ? row / 4 : row;
    const int64_t tiles = b * (t_len + 1) * ceil_div(row_v, kGatherTile);
    const int64_t cap = (int64_t)sm_count() * 8;
    const unsigned grid = (unsigned)(tiles < cap ? tiles : cap);
    cudaStream_t st = (cudaStream_t)stream;
    if (vec4)
        window_gather_kernel<float4><<<grid, kGatherThreads, 0, st>>>((const float4*)series, s_len, row_v, lv, t_len, first,
                                                                      b, (float4*)obs, (float4*)y);
    else
        window_gather_kernel<float><<<grid, kGatherThreads, 0, st>>>(series, s_len, row_v, lv, t_len, first, b, obs, y);
    count_launch();
    return check_launch("window_gather");
}

int32_t stmgcn_obs_to_node_major(const float* obs, float* xo, float* xt, int64_t b, int64_t t, int64_t n,
                                 int64_t c, void* stream) {
    STMGCN_REQUIRE(obs && xt, STMGCN_ERR_ARG, "obs_to_node_major: null pointer");
    STMGCN_REQUIRE(b > 0 && t > 0 && n > 0 && c > 0, STMGCN_ERR_SHAPE, "obs_to_node_major: bad shape");
    STMGCN_REQUIRE(xo != nullptr || c == 1, STMGCN_ERR_ARG, "obs_to_node_major: xo required when C > 1");
    const int64_t total = n * b * t;
    const int64_t blocks = ceil_div(total, 256);
    const int64_t cap = (int64_t)sm_count() * 16;
    obs_to_node_major_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, (cudaStream_t)stream>>>(
        obs, xo, xt, b, t, n, c);
    count_launch();
    return check_launch("obs_to_node_major");
}

int32_t stmgcn_obs_grad(const float* d_xo, const float* d_xt, float* d_obs, int64_t b, int64_t t, int64_t n, int64_t c,
                        void* stream) {
    STMGCN_REQUIRE(d_obs, STMGCN_ERR_ARG, "obs_grad: null pointer");
    STMGCN_REQUIRE(b > 0 && t > 0 && n > 0 && c > 0, STMGCN_ERR_SHAPE, "obs_grad: bad shape");
    const int64_t total = n * b * t;
    const int64_t blocks = ceil_div(total, 256);
    const int64_t cap = (int64_t)sm_count() * 16;
    obs_grad_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, (cudaStream_t)stream>>>(d_xo, d_xt, d_obs, b, t, n, c);
    count_launch();
    return check_launch("obs_grad");
}

int32_t stmgcn_gate_fwd(const float* pool, int64_t b, int32_t t, int64_t n_regions, const float* fcw,
                        const float* fcb, float* z, float* a1, float* s, void* stream) {
    STMGCN_REQUIRE(pool && fcw && fcb && z && a1 && s, STMGCN_ERR_ARG, "gate_fwd: null pointer");
    STMGCN_REQUIRE(b > 0 && t > 0 && n_regions > 0, STMGCN_ERR_SHAPE, "gate_fwd: bad shape");
    STMGCN_REQUIRE(t <= kMaxGateSteps, STMGCN_ERR_SHAPE, "gate_fwd: T=%d (max %d)", t, kMaxGateSteps);
    const int threads = t <= 32 ? 32 : (t <= 128 ? 128 : 256);
    gate_fwd_kernel<<<(unsigned)b, threads, 2 * t * sizeof(float), (cudaStream_t)stream>>>(
        pool, t, 1.0f / (float)n_regions, fcw, fcb, z, a1, s);
    count_launch();
    return check_launch("gate_fwd");
}

int32_t stmgcn_gate_bwd(const float* d_s, const float* z, const float* a1, const float* s, int64_t b,
                        int32_t t, const float* fcw, float* d_fcw, float* d_fcb, float* d_z, void* stream) {
    STMGCN_REQUIRE(d_s && z && a1 && s && fcw && d_z, STMGCN_ERR_ARG, "gate_bwd: null pointer");
    STMGCN_REQUIRE((d_fcw == nullptr) == (d_fcb == nullptr), STMGCN_ERR_ARG, "gate_bwd: d_fcw and d_fcb go together");
    STMGCN_REQUIRE(b > 0 && t > 0, STMGCN_ERR_SHAPE, "gate_bwd: bad shape");
    STMGCN_REQUIRE(t <= kMaxGateSteps, STMGCN_ERR_SHAPE, "gate_bwd: T=%d (max %d)", t, kMaxGateSteps);
    const int threads = t <= 32 ? 32 : (t <= 128 ? 128 : 256);
    gate_bwd_kernel<<<(unsigned)b, threads, 4 * t * sizeof(float), (cudaStream_t)stream>>>(
        d_s, z, a1, s, t, fcw, d_fcw, d_fcb, d_z);
    count_launch();
    return check_launch("gate_bwd");
}

int32_t stmgcn_fuse_out_fwd(const float* const* g, int32_t m, int64_t n, int64_t b, int32_t gdim, int32_t c,
                            const float* fcw, const float* fcb, float* feat, float* y, void* stream) {
    STMGCN_REQUIRE(g && fcw && fcb && feat && y, STMGCN_ERR_ARG, "fuse_out_fwd: null pointer");
    STMGCN_REQUIRE(m >= 1 && m <= kMaxGraphs, STMGCN_ERR_SHAPE, "fuse_out_fwd: M=%d (max %d)", m, kMaxGraphs);
    STMGCN_REQUIRE(n > 0 && b > 0 && gdim > 0 && c > 0, STMGCN_ERR_SHAPE, "fuse_out_fwd: bad shape");
    STMGCN_REQUIRE((int64_t)c * gdim + c <= kMaxFuseFloats, STMGCN_ERR_SHAPE, "fuse_out_fwd: C*G=%lld too large (C*G + C "
                   "<= %d)", (long long)c * gdim, kMaxFuseFloats);
    GraphPtrs gp;
    for (int k = 0; k < kMaxGraphs; ++k) gp.g[k] = k < m ? g[k] : nullptr;
    for (int k = 0; k < m; ++k) STMGCN_REQUIRE(gp.g[k], STMGCN_ERR_ARG, "fuse_out_fwd: g[%d] null", k);
    const int64_t rows = n * b;
    const int64_t blocks = ceil_div(rows, 8);
    const int64_t cap = (int64_t)sm_count() * 8;
    fuse_out_fwd_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, (cudaStream_t)stream>>>(
        gp, m, n, b, gdim, c, fcw, fcb, feat, y);
    count_launch();
    return check_launch("fuse_out_fwd");
}

int32_t stmgcn_fuse_out_bwd(const float* d_y, const float* feat, int64_t n, int64_t b, int32_t gdim,
                            int32_t c, const float* fcw, float* d_feat, float* d_fcw, float* d_fcb,
                            void* stream) {
    STMGCN_REQUIRE(d_y && feat && fcw && d_feat, STMGCN_ERR_ARG, "fuse_out_bwd: null pointer");
    STMGCN_REQUIRE((d_fcw == nullptr) == (d_fcb == nullptr), STMGCN_ERR_ARG, "fuse_out_bwd: d_fcw and d_fcb go together");
    STMGCN_REQUIRE(n > 0 && b > 0 && gdim > 0 && c > 0, STMGCN_ERR_SHAPE, "fuse_out_bwd: bad shape");
    STMGCN_REQUIRE((int64_t)c * gdim + c <= kMaxFuseFloats, STMGCN_ERR_SHAPE, "fuse_out_bwd: C*G=%lld too large (C*G + C "
                   "<= %d)", (long long)c * gdim, kMaxFuseFloats);
    const size_t smem = ((size_t)c * gdim + c) * sizeof(float);
    const int64_t rows = n * b;
    const int64_t blocks = ceil_div(rows, 8);
    const int64_t cap = (int64_t)sm_count() * 4;
    fuse_out_bwd_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, smem, (cudaStream_t)stream>>>(
        d_y, feat, n, b, gdim, c, fcw, d_feat, d_fcw, d_fcb);
    count_launch();
    return check_launch("fuse_out_bwd");
}

}  // extern "C"
