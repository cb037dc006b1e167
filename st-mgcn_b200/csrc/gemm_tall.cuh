// Tall-skinny fp32 GEMM building blocks (CUDA-core FFMA, exact-fp32 path).
//
// Every dense contraction on the hot path has a huge row count (R = regions x windows, 10^5..10^6) and
// small inner/outer dimensions (<= 256):
//   forward :  C[R x Nc]  = A[R x Kd] . B[Kd x Nc]          (tall_gemm_kernel, fused epilogue functor)
//   reduce  :  G[Kd x Nc] += sum_r A[r,:]^T D[r,:]           (reduce_gemm_kernel, weight gradients)
// A is the concatenation along K of up to 8 equal-width row-major segments (the stacked-K projection reads
// T_0X..T_KX without materialising the reference's torch.cat, GCN.py:37; the LSTM reads [h_below | h_prev]).
//
// CTA = 512 threads, thread tile 8 x 8, k-chunks of 16 staged with cp.async (2 stages).
#pragma once
#include "common.cuh"

namespace stmgcn {

constexpr int kGemmThreads = 512;
constexpr int kKC = 16;            // k-chunk (forward) / row-chunk (reduce)
constexpr int kAPad = 4;
constexpr int kMaxSegs = 8;

struct ASegs {
    const float* seg[kMaxSegs];    // nullptr => zeros
    int nseg;
    int segw;                      // width of every segment (floats)
    int64_t lda;                   // row stride of every segment (floats)
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem, bool valid) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    int sz = valid ? 4 : 0;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(s), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

template <int TN>
struct TallCfg {
    static constexpr int NT = TN / 8;                  // threads along n
    static constexpr int MG = kGemmThreads / NT;       // row groups
    static constexpr int TM = MG * 8;                  // rows per CTA tile
    static constexpr int A_STRIDE = kKC + kAPad;       // floats
    static constexpr int A_STAGE = TM * A_STRIDE;      // floats
    static constexpr int B_STAGE = kKC * TN;
    static constexpr size_t SMEM = 2 * (size_t)(A_STAGE + B_STAGE) * sizeof(float);
};

// ----------------------------------------------------------------------------------------------------
// forward: C tile [TM x TN] at rows [row0, row0+TM), columns [col0, col0+TN)
// Epi::operator()(acc, tile, rows, nc) consumes the 8x8 register tile: acc[i][j] is row tile.row(i), column tile.col(j).
// The columns of a thread are two float4 groups TN/2 apart, the two float4 each k step reads from the staged B row.
// ----------------------------------------------------------------------------------------------------
template <int TN>
struct TallTile {
    int64_t row0;
    int mg, col0, tn;
    __device__ __forceinline__ int64_t row(int i) const { return row0 + mg + (int64_t)i * TallCfg<TN>::MG; }
    __device__ __forceinline__ int col(int j) const { return col0 + 4 * tn + (j & 3) + (j >> 2) * (TN / 2); }
};

template <int TN, bool VEC, class Epi>
__global__ void __launch_bounds__(kGemmThreads, 1)
tall_gemm_kernel(ASegs a, int64_t rows, int kd, const float* __restrict__ bmat, int ldb, int nc, Epi epi) {
    using Cfg = TallCfg<TN>;
    extern __shared__ __align__(16) float smem[];
    float* a_s = smem;                                // [2][TM][A_STRIDE]
    float* b_s = smem + 2 * Cfg::A_STAGE;             // [2][kKC][TN]
    const int tid = threadIdx.x;
    const int tn = tid % Cfg::NT;
    const int mg = tid / Cfg::NT;
    const int64_t row0 = (int64_t)blockIdx.x * Cfg::TM;
    const int col0 = blockIdx.y * TN;

    auto issue = [&](int chunk, int stage) {
        const int k0 = chunk * kKC;
        float* as = a_s + stage * Cfg::A_STAGE;
        float* bs = b_s + stage * Cfg::B_STAGE;
        if (VEC) {
            constexpr int A_ELEMS = Cfg::TM * (kKC / 4);
            for (int idx = tid; idx < A_ELEMS; idx += kGemmThreads) {
                const int m = idx / (kKC / 4), kq = idx % (kKC / 4);
                const int k = k0 + kq * 4;
                const int64_t r = row0 + m;
                const int sg = k / a.segw;
                const float* base = (k < kd) ? a.seg[sg < kMaxSegs ? sg : 0] : nullptr;
                const bool ok = (r < rows) && (k < kd) && (base != nullptr);
                const float* src = ok ? base + r * a.lda + (k - sg * a.segw) : bmat;
                cp_async16(as + m * Cfg::A_STRIDE + kq * 4, src, ok);
            }
            constexpr int B_ELEMS = kKC * (TN / 4);
            for (int idx = tid; idx < B_ELEMS; idx += kGemmThreads) {
                const int kk = idx / (TN / 4), nq = idx % (TN / 4);
                const int k = k0 + kk, n = col0 + nq * 4;
                const bool ok = (k < kd) && (n < nc);
                const float* src = ok ? bmat + (int64_t)k * ldb + n : bmat;
                cp_async16(bs + kk * TN + nq * 4, src, ok);
            }
        } else {
            constexpr int A_ELEMS = Cfg::TM * kKC;
            for (int idx = tid; idx < A_ELEMS; idx += kGemmThreads) {
                const int m = idx / kKC, kk = idx % kKC;
                const int k = k0 + kk;
                const int64_t r = row0 + m;
                const int sg = k / a.segw;
                const float* base = (k < kd) ? a.seg[sg < kMaxSegs ? sg : 0] : nullptr;
                const bool ok = (r < rows) && (k < kd) && (base != nullptr);
                const float* src = ok ? base + r * a.lda + (k - sg * a.segw) : bmat;
                cp_async4(as + m * Cfg::A_STRIDE + kk, src, ok);
            }
            constexpr int B_ELEMS = kKC * TN;
            for (int idx = tid; idx < B_ELEMS; idx += kGemmThreads) {
                const int kk = idx / TN, nn = idx % TN;
                const int k = k0 + kk, n = col0 + nn;
                const bool ok = (k < kd) && (n < nc);
                const float* src = ok ? bmat + (int64_t)k * ldb + n : bmat;
                cp_async4(bs + kk * TN + nn, src, ok);
            }
        }
        cp_async_commit();
    };

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    const int nchunks = (kd + kKC - 1) / kKC;
    issue(0, 0);
    for (int c = 0; c < nchunks; ++c) {
        if (c + 1 < nchunks) {
            issue(c + 1, (c + 1) & 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float* as = a_s + (c & 1) * Cfg::A_STAGE + mg * Cfg::A_STRIDE;
        const float* bs = b_s + (c & 1) * Cfg::B_STAGE + 4 * tn;
#pragma unroll
        for (int k4 = 0; k4 < kKC / 4; ++k4) {
            float4 av[8];
#pragma unroll
            for (int i = 0; i < 8; ++i)
                av[i] = *reinterpret_cast<const float4*>(as + (i * Cfg::MG) * Cfg::A_STRIDE + k4 * 4);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const float4 b0 = *reinterpret_cast<const float4*>(bs + (k4 * 4 + kk) * TN);
                const float4 b1 = *reinterpret_cast<const float4*>(bs + (k4 * 4 + kk) * TN + TN / 2);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float ai = kk == 0 ? av[i].x : (kk == 1 ? av[i].y : (kk == 2 ? av[i].z : av[i].w));
                    acc[i][0] = fmaf(ai, b0.x, acc[i][0]);
                    acc[i][1] = fmaf(ai, b0.y, acc[i][1]);
                    acc[i][2] = fmaf(ai, b0.z, acc[i][2]);
                    acc[i][3] = fmaf(ai, b0.w, acc[i][3]);
                    acc[i][4] = fmaf(ai, b1.x, acc[i][4]);
                    acc[i][5] = fmaf(ai, b1.y, acc[i][5]);
                    acc[i][6] = fmaf(ai, b1.z, acc[i][6]);
                    acc[i][7] = fmaf(ai, b1.w, acc[i][7]);
                }
            }
        }
        __syncthreads();
    }
    epi(acc, TallTile<TN>{row0, mg, col0, tn}, rows, nc);
}

// ----------------------------------------------------------------------------------------------------
// reduce: G[Kd x Nc] += sum over (t, r) of A_t[r,:]^T D_t[r,:]
// Time loop inside the kernel so each CTA flushes its register tile with atomics exactly once.
// A_t segment s  = a.seg[s] + t * a_tstride[s]   (segment pointer nullptr => zeros;  t_first_zero[s]: the
//                  segment is zeros at t == 0, and shifted by one step otherwise -- the LSTM's h_{t-1})
// D_t            = d + t * d_tstride, row stride ldd.
// ----------------------------------------------------------------------------------------------------
struct ReduceTime {
    int n_t;
    int64_t a_tstride[kMaxSegs];
    int a_shift[kMaxSegs];         // 1: segment at time t reads (t-1), zeros (or a_t0[s]) at t == 0
    const float* a_t0[kMaxSegs];   // value at t == 0 for shifted segments (nullptr => zeros)
    int64_t d_tstride;
};

template <int TN>
struct ReduceCfg {
    static constexpr int NT = TN / 8;
    static constexpr int MG = kGemmThreads / NT;
    static constexpr int TMK = MG * 8;                 // kd values per CTA tile
    static constexpr int A_STAGE = kKC * TMK;          // [rc][TMK]
    static constexpr int D_STAGE = kKC * TN;           // [rc][TN]
    static constexpr size_t SMEM = 2 * (size_t)(A_STAGE + D_STAGE) * sizeof(float);
};

template <int TN, bool VEC>
__global__ void __launch_bounds__(kGemmThreads, 1)
reduce_gemm_kernel(ASegs a, ReduceTime tm, int64_t rows, int kd, const float* __restrict__ d, int64_t ldd,
                   int nc, float* __restrict__ gout, int ldg) {
    using Cfg = ReduceCfg<TN>;
    extern __shared__ __align__(16) float smem[];
    float* a_s = smem;
    float* d_s = smem + 2 * Cfg::A_STAGE;
    const int tid = threadIdx.x;
    const int tn = tid % Cfg::NT;
    const int mg = tid / Cfg::NT;
    const int kd0 = blockIdx.y * Cfg::TMK;
    const int col0 = blockIdx.z * TN;
    const int64_t chunks_per_t = (rows + kKC - 1) / kKC;
    const int64_t total_chunks = chunks_per_t * tm.n_t;

    auto issue = [&](int64_t chunk, int stage) {
        const int t = (int)(chunk / chunks_per_t);
        const int64_t r0 = (chunk % chunks_per_t) * kKC;
        float* as = a_s + stage * Cfg::A_STAGE;
        float* ds = d_s + stage * Cfg::D_STAGE;
        const float* dt = d + (int64_t)t * tm.d_tstride;
        if (VEC) {
            constexpr int A_ELEMS = kKC * (Cfg::TMK / 4);
            for (int idx = tid; idx < A_ELEMS; idx += kGemmThreads) {
                const int rr = idx / (Cfg::TMK / 4), kq = idx % (Cfg::TMK / 4);
                const int k = kd0 + kq * 4;
                const int64_t r = r0 + rr;
                const int sg = (k < kd) ? k / a.segw : 0;
                const float* base = a.seg[sg];
                if (tm.a_shift[sg]) base = (t == 0) ? tm.a_t0[sg] : (base ? base + (int64_t)(t - 1) * tm.a_tstride[sg] : nullptr);
                else if (base) base += (int64_t)t * tm.a_tstride[sg];
                const bool ok = (r < rows) && (k < kd) && (base != nullptr);
                const float* src = ok ? base + r * a.lda + (k - sg * a.segw) : d;
                cp_async16(as + rr * Cfg::TMK + kq * 4, src, ok);
            }
            constexpr int D_ELEMS = kKC * (TN / 4);
            for (int idx = tid; idx < D_ELEMS; idx += kGemmThreads) {
                const int rr = idx / (TN / 4), nq = idx % (TN / 4);
                const int n = col0 + nq * 4;
                const int64_t r = r0 + rr;
                const bool ok = (r < rows) && (n < nc);
                const float* src = ok ? dt + r * ldd + n : d;
                cp_async16(ds + rr * TN + nq * 4, src, ok);
            }
        } else {
            constexpr int A_ELEMS = kKC * Cfg::TMK;
            for (int idx = tid; idx < A_ELEMS; idx += kGemmThreads) {
                const int rr = idx / Cfg::TMK, kk = idx % Cfg::TMK;
                const int k = kd0 + kk;
                const int64_t r = r0 + rr;
                const int sg = (k < kd) ? k / a.segw : 0;
                const float* base = a.seg[sg];
                if (tm.a_shift[sg]) base = (t == 0) ? tm.a_t0[sg] : (base ? base + (int64_t)(t - 1) * tm.a_tstride[sg] : nullptr);
                else if (base) base += (int64_t)t * tm.a_tstride[sg];
                const bool ok = (r < rows) && (k < kd) && (base != nullptr);
                const float* src = ok ? base + r * a.lda + (k - sg * a.segw) : d;
                cp_async4(as + rr * Cfg::TMK + kk, src, ok);
            }
            constexpr int D_ELEMS = kKC * TN;
            for (int idx = tid; idx < D_ELEMS; idx += kGemmThreads) {
                const int rr = idx / TN, nn = idx % TN;
                const int n = col0 + nn;
                const int64_t r = r0 + rr;
                const bool ok = (r < rows) && (n < nc);
                const float* src = ok ? dt + r * ldd + n : d;
                cp_async4(ds + rr * TN + nn, src, ok);
            }
        }
        cp_async_commit();
    };

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    // grid-stride over row chunks: CTA x takes chunks x, x+gridDim.x, ...
    int64_t c = blockIdx.x;
    int stage = 0;
    if (c < total_chunks) issue(c, 0);
    for (; c < total_chunks; c += gridDim.x, stage ^= 1) {
        const int64_t nxt = c + gridDim.x;
        if (nxt < total_chunks) {
            issue(nxt, stage ^ 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float* as = a_s + stage * Cfg::A_STAGE + 8 * mg;
        const float* ds = d_s + stage * Cfg::D_STAGE + 4 * tn;
#pragma unroll
        for (int rr = 0; rr < kKC; ++rr) {
            const float4 a0 = *reinterpret_cast<const float4*>(as + rr * Cfg::TMK);
            const float4 a1 = *reinterpret_cast<const float4*>(as + rr * Cfg::TMK + 4);
            const float4 b0 = *reinterpret_cast<const float4*>(ds + rr * TN);
            const float4 b1 = *reinterpret_cast<const float4*>(ds + rr * TN + TN / 2);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                acc[i][0] = fmaf(av[i], b0.x, acc[i][0]);
                acc[i][1] = fmaf(av[i], b0.y, acc[i][1]);
                acc[i][2] = fmaf(av[i], b0.z, acc[i][2]);
                acc[i][3] = fmaf(av[i], b0.w, acc[i][3]);
                acc[i][4] = fmaf(av[i], b1.x, acc[i][4]);
                acc[i][5] = fmaf(av[i], b1.y, acc[i][5]);
                acc[i][6] = fmaf(av[i], b1.z, acc[i][6]);
                acc[i][7] = fmaf(av[i], b1.w, acc[i][7]);
            }
        }
        __syncthreads();
    }
    // flush: G[kd0 + 8*mg + i][col] += acc
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int k = kd0 + 8 * mg + i;
        if (k >= kd) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = col0 + (j < 4 ? 4 * tn + j : TN / 2 + 4 * tn + (j - 4));
            if (n < nc) atomicAdd(gout + (int64_t)k * ldg + n, acc[i][j]);
        }
    }
}

// host-side launch helpers -----------------------------------------------------------------------------
// The VEC kernels stage A, B and D with 16-byte cp.async: every 4-float group must lie inside one segment and one row,
// and start 16-byte aligned.  Loaders of both variants feed the same FMA order, so the choice never changes results.
inline bool vec_ok(const ASegs& a, const float* b, int64_t ldb, int nc) {
    if (a.segw % 4 || a.lda % 4 || ldb % 4 || nc % 4 || !aligned16(b)) return false;
    for (int s = 0; s < a.nseg; ++s)
        if (a.seg[s] && !aligned16(a.seg[s])) return false;
    return true;
}

inline bool reduce_vec_ok(const ASegs& a, const ReduceTime& tm, const float* d, int64_t ldd, int nc) {
    if (!vec_ok(a, d, ldd, nc) || tm.d_tstride % 4) return false;
    for (int s = 0; s < a.nseg; ++s)
        if (tm.a_tstride[s] % 4 || (tm.a_t0[s] && !aligned16(tm.a_t0[s]))) return false;
    return true;
}

template <int TN, class Epi>
inline int32_t launch_tall(const ASegs& a, int64_t rows, int kd, const float* bmat, int ldb, int nc,
                           const Epi& epi, cudaStream_t st, const char* what) {
    using Cfg = TallCfg<TN>;
    auto kern = vec_ok(a, bmat, ldb, nc) ? tall_gemm_kernel<TN, true, Epi> : tall_gemm_kernel<TN, false, Epi>;
    if (int32_t rc = ensure_dyn_smem((const void*)kern, Cfg::SMEM)) return rc;
    dim3 grid((unsigned)ceil_div(rows, Cfg::TM), (unsigned)ceil_div(nc, TN));
    kern<<<grid, kGemmThreads, Cfg::SMEM, st>>>(a, rows, kd, bmat, ldb, nc, epi);
    count_launch();
    return check_launch(what);
}

template <int TN>
inline int32_t launch_reduce(const ASegs& a, const ReduceTime& tm, int64_t rows, int kd, const float* d,
                             int64_t ldd, int nc, float* gout, int ldg, cudaStream_t st, const char* what) {
    using Cfg = ReduceCfg<TN>;
    auto kern = reduce_vec_ok(a, tm, d, ldd, nc) ? reduce_gemm_kernel<TN, true> : reduce_gemm_kernel<TN, false>;
    if (int32_t rc = ensure_dyn_smem((const void*)kern, Cfg::SMEM)) return rc;
    const int64_t total_chunks = ceil_div(rows, kKC) * tm.n_t;
    const int panels = (int)(ceil_div(kd, Cfg::TMK) * ceil_div(nc, TN));
    int64_t gx = (int64_t)sm_count() / (panels > 0 ? panels : 1);
    if (gx < 1) gx = 1;
    if (gx > total_chunks) gx = total_chunks;
    dim3 grid((unsigned)gx, (unsigned)ceil_div(kd, Cfg::TMK), (unsigned)ceil_div(nc, TN));
    kern<<<grid, kGemmThreads, Cfg::SMEM, st>>>(a, tm, rows, kd, d, ldd, nc, gout, ldg);
    count_launch();
    return check_launch(what);
}

}  // namespace stmgcn
