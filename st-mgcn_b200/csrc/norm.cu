// K1c: the supports of a learnable adjacency on a fixed sparsity pattern, and their backward (d w).
//
// The pattern is the adjacency's stored entries plus the diagonal slots a kind needs, as CSR (rowptr, colidx) and
// CSR^T (rowptr_t, colidx_t, perm_t: CSR^T position p holds CSR entry perm_t[p]).  widx maps each pattern entry to its
// weight (or -1: a slot that holds the diagonal term only).  From the weights w the forward forms the stored values of
// the matrices Adj_Preprocessor.process_sparse builds (GCN.py:99-111):
//   chebyshev  v[e] = -s * ((a_i * w) * a_j) + (i == j) (s - 1),   a = D^-1/2, D the row sums of the stored weights
//   localpool  v[e] =       (a_i * w) * a_j  + (i == j)
//   diffusion  P_b^T (CSR order)   v[e] = w * inv(d_in)[j]
//              P_f^T (CSR^T order) v[p] = w * inv(d_out)[i],   inv(d) = 0 where 1/d is infinite (GCN.py:100-104)
// One warp owns one row (or one column of the transpose); its lanes take the segment's entries strided by 32 and a fixed
// xor tree sums them: every sum has one owner and one order, no float atomics, two runs agree bit for bit.
// When the adjacency is multiplied dense, pattern_scatter writes the values into the dense matrix and pattern_gather reads
// the matrix's gradient back into the values' order for the backward (one warp per row as well).
#include "common.cuh"
#include <math.h>

using namespace stmgcn;

namespace {

constexpr int kWarps = 8;
enum Kind { kChebyshev = 0, kLocalpool = 1, kDiffusion = 2 };

__device__ __forceinline__ int32_t weight_of(const int32_t* widx, int64_t e) {
    return widx == nullptr ? (int32_t)e : __ldg(widx + e);
}

// deg^-1/2 as torch's pow(deg, -0.5): +inf at +-0, NaN below 0 and at NaN, 0 at +inf (IEEE sqrt and division)
__device__ __forceinline__ float rsqrt_deg(float d) { return d == 0.f ? __int_as_float(0x7f800000) : 1.f / sqrtf(d); }
// the random walk's inverse degree: 1/d, 0 where that is infinite
__device__ __forceinline__ float inv_deg(float r) { return isinf(r) ? 0.f : r; }

// stored row sum of CSR row k
__device__ __forceinline__ float row_sum(const int32_t* rowptr, const int32_t* widx, const float* w, int64_t k, int lane) {
    float s = 0.f;
    for (int32_t e = rowptr[k] + lane; e < rowptr[k + 1]; e += 32) {
        const int32_t wi = weight_of(widx, e);
        if (wi >= 0) s += __ldg(w + wi);
    }
    return warp_sum(s);
}

// pass 1 (both directions): the degree terms.  Symmetric kinds: work[k] = a_k; diffusion: work[k] = 1/d_out,
// work[n + k] = 1/d_in (the raw reciprocals: the backward needs to know where they are infinite)
template <bool DIFF>
__global__ void __launch_bounds__(kWarps * 32)
norm_degrees_kernel(int64_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ rowptr_t,
                    const int32_t* __restrict__ perm_t, const int32_t* __restrict__ widx, const float* __restrict__ w,
                    float* __restrict__ work) {
    const int lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (k >= n) return;
    const float dout = row_sum(rowptr, widx, w, k, lane);
    if (!DIFF) {
        if (lane == 0) work[k] = rsqrt_deg(dout);
        return;
    }
    float din = 0.f;
    for (int32_t p = rowptr_t[k] + lane; p < rowptr_t[k + 1]; p += 32) {
        const int32_t wi = weight_of(widx, __ldg(perm_t + p));
        if (wi >= 0) din += __ldg(w + wi);
    }
    din = warp_sum(din);
    if (lane == 0) {
        work[k] = 1.f / dout;
        work[n + k] = 1.f / din;
    }
}

// forward pass 2: the values of row k (and, diffusion, of column k of the transpose)
template <bool DIFF>
__global__ void __launch_bounds__(kWarps * 32)
norm_values_kernel(int64_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                   const int32_t* __restrict__ rowptr_t, const int32_t* __restrict__ colidx_t,
                   const int32_t* __restrict__ perm_t, const int32_t* __restrict__ widx, const float* __restrict__ w,
                   float coef, float diag, const float* __restrict__ work, float* __restrict__ vals,
                   float* __restrict__ vals_t) {
    const int lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (k >= n) return;
    if (!DIFF) {
        const float ai = work[k];
        for (int32_t e = rowptr[k] + lane; e < rowptr[k + 1]; e += 32) {
            const int32_t j = __ldg(colidx + e), wi = weight_of(widx, e);
            float v = wi >= 0 ? coef * ((ai * __ldg(w + wi)) * work[j]) : 0.f;
            if (j == k && diag != 0.f) v = wi >= 0 ? v + diag : diag;
            vals[e] = v;
        }
        return;
    }
    for (int32_t e = rowptr[k] + lane; e < rowptr[k + 1]; e += 32) {          // P_b^T[k, j] = w / d_in(j)
        const int32_t j = __ldg(colidx + e), wi = weight_of(widx, e);
        vals[e] = wi >= 0 ? __ldg(w + wi) * inv_deg(work[n + j]) : 0.f;
    }
    for (int32_t p = rowptr_t[k] + lane; p < rowptr_t[k + 1]; p += 32) {      // P_f^T[k, i] = w / d_out(i)
        const int32_t i = __ldg(colidx_t + p), wi = weight_of(widx, __ldg(perm_t + p));
        vals_t[p] = wi >= 0 ? __ldg(w + wi) * inv_deg(work[i]) : 0.f;
    }
}

// backward pass 2: the column sums, over CSR^T.  Symmetric kinds: work[2n + k] = sum_{col k} (g c a_i) w, the adjoint of
// a_k through its column uses.  Diffusion: work[2n + k] = d L / d d_in(k), and g_f scattered into CSR order at work[3n:].
template <bool DIFF>
__global__ void __launch_bounds__(kWarps * 32)
norm_grad_cols_kernel(int64_t n, const int32_t* __restrict__ rowptr_t, const int32_t* __restrict__ colidx_t,
                      const int32_t* __restrict__ perm_t, const int32_t* __restrict__ widx, const float* __restrict__ w,
                      float coef, const float* __restrict__ g, const float* __restrict__ g_t, float* __restrict__ work) {
    const int lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (k >= n) return;
    float s = 0.f;
    for (int32_t p = rowptr_t[k] + lane; p < rowptr_t[k + 1]; p += 32) {
        const int32_t e = __ldg(perm_t + p), wi = weight_of(widx, e);
        if (DIFF) work[3 * n + e] = __ldg(g_t + p);
        if (wi < 0) continue;
        if (DIFF)
            s += __ldg(g + e) * __ldg(w + wi);
        else
            s += ((__ldg(g + e) * coef) * work[__ldg(colidx_t + p)]) * __ldg(w + wi);
    }
    s = warp_sum(s);
    if (lane == 0) {
        if (DIFF) {
            const float r = work[n + k];
            // torch's chain: the masked reciprocal passes 0, and pow's backward multiplies it by -d^-2 = -inf at a zero
            // degree: NaN wherever a zero-sum column has stored entries, as in the fp64 restatement
            s = (isinf(r) ? 0.f : s) * -(r * r);
        }
        work[2 * n + k] = s;
    }
}

// backward pass 3: row k's degree term, then d w of row k's stored entries
template <bool DIFF>
__global__ void __launch_bounds__(kWarps * 32)
norm_grad_rows_kernel(int64_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                      const int32_t* __restrict__ widx, const float* __restrict__ w, float coef,
                      const float* __restrict__ g, const float* __restrict__ work, float* __restrict__ dw) {
    const int lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (k >= n) return;
    const int32_t beg = rowptr[k], end = rowptr[k + 1];
    float s = 0.f;
    for (int32_t e = beg + lane; e < end; e += 32) {
        const int32_t wi = weight_of(widx, e);
        if (wi < 0) continue;
        if (DIFF)
            s += work[3 * n + e] * __ldg(w + wi);
        else
            s += ((__ldg(g + e) * coef) * work[__ldg(colidx + e)]) * __ldg(w + wi);
    }
    s = warp_sum(s);
    float gdeg;                                           // d L / d D_kk (the row sum of the stored weights)
    if (DIFF) {
        const float r = work[k];
        gdeg = (isinf(r) ? 0.f : s) * -(r * r);            // as the column term: NaN at a zero-sum row
    } else {
        const float a = work[k];
        gdeg = (s + work[2 * n + k]) * (-0.5f * (a * a * a));       // d(D^-1/2)/dD = -1/2 D^-3/2
    }
    for (int32_t e = beg + lane; e < end; e += 32) {
        const int32_t wi = weight_of(widx, e);
        if (wi < 0) continue;
        const int32_t j = __ldg(colidx + e);
        float d;
        if (DIFF)
            d = (__ldg(g + e) * inv_deg(work[n + j]) + work[3 * n + e] * inv_deg(work[k])) + (gdeg + work[2 * n + j]);
        else
            d = ((__ldg(g + e) * coef) * work[j]) * work[k] + gdeg;
        dw[wi] = d;
    }
}

// pattern -> dense: row k of the n x n matrix is zeroed, then its segment's values are added in entry order.  A chunk of
// 32 entries at a time: lanes holding the same column (a repeated entry) form a group whose lowest lane adds the
// group's values to the element one by one in lane order, so every element is ((0 + v_e0) + v_e1) + ... over its
// entries e0 < e1 < ..., whatever the repeats; each element has one writer per chunk and the chunks run in order.
__global__ void __launch_bounds__(kWarps * 32)
pattern_scatter_kernel(int64_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                       const float* __restrict__ vals, float* __restrict__ dense) {
    const int lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (k >= n) return;
    float* row = dense + k * n;
    for (int64_t j = lane; j < n; j += 32) row[j] = 0.f;
    __syncwarp();
    const int32_t beg = rowptr[k], end = rowptr[k + 1];
    for (int32_t base = beg; base < end; base += 32) {
        const int32_t e = base + lane;
        const bool in = e < end;
        const int32_t j = in ? __ldg(colidx + e) : -1 - lane;        // lanes past the segment: a column of their own
        const float v = in ? __ldg(vals + e) : 0.f;
        const unsigned grp = __match_any_sync(0xffffffffu, j);
        const bool leader = in && lane == __ffs(grp) - 1;
        float s = leader ? row[j] : 0.f;
        if (__all_sync(0xffffffffu, __popc(grp) == 1)) {
            s += v;
        } else {
#pragma unroll 1
            for (int r = 0; r < 32; ++r) {
                const float vr = __shfl_sync(0xffffffffu, v, r);
                if ((grp >> r) & 1u) s += vr;
            }
        }
        if (leader) row[j] = s;
        __syncwarp();
    }
}

// dense -> pattern: d vals[e] = dense[k][colidx[e]] for row k's entries (a repeated entry gets the element at each)
__global__ void __launch_bounds__(kWarps * 32)
pattern_gather_kernel(int64_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                      const float* __restrict__ dense, float* __restrict__ dvals) {
    const int lane = threadIdx.x & 31;
    const int64_t k = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (k >= n) return;
    const float* row = dense + k * n;
    for (int32_t e = rowptr[k] + lane; e < rowptr[k + 1]; e += 32) dvals[e] = __ldg(row + __ldg(colidx + e));
}

struct Range {
    const void* p;
    int64_t bytes;
};

bool overlaps(const Range& x, const Range& y) { return stmgcn::overlaps(x.p, x.bytes, y.p, y.bytes); }

// the checks both directions share; returns 0 or the error already reported.  outs: the ranges the call writes, ins: the
// ranges it reads
int32_t check_call(const char* what, int32_t kind, int64_t n, const int32_t* rowptr, const int32_t* colidx,
                   const int32_t* rowptr_t, const int32_t* colidx_t, const int32_t* perm_t, int64_t nnz,
                   const int32_t* widx, const float* w, int64_t nnz_w, float scale, const float* work, int64_t work_count,
                   int64_t work_need, const Range* outs, int nouts, const Range* ins, int nins) {
    STMGCN_REQUIRE(n > 0 && n < ((int64_t)1 << 30) && nnz >= 0 && nnz < ((int64_t)1 << 31), STMGCN_ERR_SHAPE,
                   "%s: n=%lld nnz=%lld", what, (long long)n, (long long)nnz);
    STMGCN_REQUIRE(nnz_w >= 0 && nnz_w <= nnz && (widx != nullptr || nnz_w == nnz), STMGCN_ERR_SHAPE,
                   "%s: nnz_w=%lld must be in [0, nnz=%lld], and equal to it without widx", what, (long long)nnz_w,
                   (long long)nnz);
    STMGCN_REQUIRE(rowptr && rowptr_t, STMGCN_ERR_ARG, "%s: null rowptr / rowptr_t", what);
    STMGCN_REQUIRE(nnz == 0 || (colidx && colidx_t && perm_t), STMGCN_ERR_ARG, "%s: null colidx / colidx_t / perm_t", what);
    STMGCN_REQUIRE(nnz_w == 0 || w, STMGCN_ERR_ARG, "%s: null w", what);
    STMGCN_REQUIRE(kind != kChebyshev || isfinite(scale), STMGCN_ERR_ARG, "%s: scale=%g must be finite", what,
                   (double)scale);
    STMGCN_REQUIRE(work && work_count >= work_need, STMGCN_ERR_ARG,
                   "%s: a workspace of %lld floats is needed (work_count=%lld)", what, (long long)work_need,
                   (long long)work_count);
    for (int i = 0; i < nouts; ++i) {
        for (int j = 0; j < nins; ++j)
            STMGCN_REQUIRE(!overlaps(outs[i], ins[j]), STMGCN_ERR_ARG, "%s: output %d overlaps input %d", what, i, j);
        for (int j = 0; j < i; ++j)
            STMGCN_REQUIRE(!overlaps(outs[i], outs[j]), STMGCN_ERR_ARG, "%s: outputs %d and %d overlap", what, j, i);
    }
    return 0;
}

}  // namespace

extern "C" int32_t stmgcn_adj_norm_fwd(int32_t kind, int64_t n, const int32_t* rowptr, const int32_t* colidx,
                                       const int32_t* rowptr_t, const int32_t* colidx_t, const int32_t* perm_t,
                                       int64_t nnz, const int32_t* widx, const float* w, int64_t nnz_w, float scale,
                                       float* work, int64_t work_count, float* vals, float* vals_t, void* stream) {
    STMGCN_REQUIRE(kind >= kChebyshev && kind <= kDiffusion, STMGCN_ERR_ARG, "adj_norm_fwd: kind=%d (0..2)", (int)kind);
    const bool diff = kind == kDiffusion;
    STMGCN_REQUIRE(nnz == 0 || (vals && (!diff || vals_t)), STMGCN_ERR_ARG, "adj_norm_fwd: null vals / vals_t");
    STMGCN_REQUIRE(diff || vals_t == nullptr, STMGCN_ERR_ARG, "adj_norm_fwd: vals_t is for the diffusion kind only");
    const int64_t i4 = 4;
    const Range ins[] = {{rowptr, (n + 1) * i4}, {colidx, nnz * i4}, {rowptr_t, (n + 1) * i4}, {colidx_t, nnz * i4},
                         {perm_t, nnz * i4}, {widx, widx ? nnz * i4 : 0}, {w, nnz_w * i4}};
    const Range outs[] = {{work, work_count * i4}, {vals, nnz * i4}, {vals_t, diff ? nnz * i4 : 0}};
    int32_t rc = check_call("adj_norm_fwd", kind, n, rowptr, colidx, rowptr_t, colidx_t, perm_t, nnz, widx, w, nnz_w,
                            scale, work, work_count, 2 * n, outs, 3, ins, 7);
    if (rc != 0) return rc;
    if (nnz == 0) return 0;            // no entry, no value: nothing is enqueued
    const float coef = kind == kChebyshev ? -scale : 1.f;
    const float diag = kind == kChebyshev ? scale - 1.f : kind == kLocalpool ? 1.f : 0.f;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = (unsigned)ceil_div(n, kWarps);
    if (diff)
        norm_degrees_kernel<true><<<grid, kWarps * 32, 0, st>>>(n, rowptr, rowptr_t, perm_t, widx, w, work);
    else
        norm_degrees_kernel<false><<<grid, kWarps * 32, 0, st>>>(n, rowptr, rowptr_t, perm_t, widx, w, work);
    count_launch();
    if (diff)
        norm_values_kernel<true><<<grid, kWarps * 32, 0, st>>>(n, rowptr, colidx, rowptr_t, colidx_t, perm_t, widx, w, coef, diag, work, vals, vals_t);
    else
        norm_values_kernel<false><<<grid, kWarps * 32, 0, st>>>(n, rowptr, colidx, rowptr_t, colidx_t, perm_t, widx, w, coef, diag, work, vals, vals_t);
    count_launch();
    return check_launch("adj_norm_fwd");
}

extern "C" int32_t stmgcn_adj_norm_bwd(int32_t kind, int64_t n, const int32_t* rowptr, const int32_t* colidx,
                                       const int32_t* rowptr_t, const int32_t* colidx_t, const int32_t* perm_t,
                                       int64_t nnz, const int32_t* widx, const float* w, int64_t nnz_w, float scale,
                                       const float* dvals, const float* dvals_t, float* work, int64_t work_count,
                                       float* dw, void* stream) {
    STMGCN_REQUIRE(kind >= kChebyshev && kind <= kDiffusion, STMGCN_ERR_ARG, "adj_norm_bwd: kind=%d (0..2)", (int)kind);
    const bool diff = kind == kDiffusion;
    STMGCN_REQUIRE(nnz_w == 0 || (dvals && dw && (!diff || dvals_t)), STMGCN_ERR_ARG,
                   "adj_norm_bwd: null dvals / dvals_t / dw");
    STMGCN_REQUIRE(diff || dvals_t == nullptr, STMGCN_ERR_ARG, "adj_norm_bwd: dvals_t is for the diffusion kind only");
    const int64_t i4 = 4;
    const Range ins[] = {{rowptr, (n + 1) * i4}, {colidx, nnz * i4}, {rowptr_t, (n + 1) * i4}, {colidx_t, nnz * i4},
                         {perm_t, nnz * i4}, {widx, widx ? nnz * i4 : 0}, {w, nnz_w * i4}, {dvals, nnz * i4},
                         {dvals_t, diff ? nnz * i4 : 0}};
    const Range outs[] = {{work, work_count * i4}, {dw, nnz_w * i4}};
    int32_t rc = check_call("adj_norm_bwd", kind, n, rowptr, colidx, rowptr_t, colidx_t, perm_t, nnz, widx, w, nnz_w,
                            scale, work, work_count, 3 * n + nnz, outs, 2, ins, 9);
    if (rc != 0) return rc;
    if (nnz_w == 0) return 0;          // no weight, no gradient: nothing is enqueued
    const float coef = kind == kChebyshev ? -scale : 1.f;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = (unsigned)ceil_div(n, kWarps);
    if (diff)
        norm_degrees_kernel<true><<<grid, kWarps * 32, 0, st>>>(n, rowptr, rowptr_t, perm_t, widx, w, work);
    else
        norm_degrees_kernel<false><<<grid, kWarps * 32, 0, st>>>(n, rowptr, rowptr_t, perm_t, widx, w, work);
    count_launch();
    if (diff)
        norm_grad_cols_kernel<true><<<grid, kWarps * 32, 0, st>>>(n, rowptr_t, colidx_t, perm_t, widx, w, coef, dvals, dvals_t, work);
    else
        norm_grad_cols_kernel<false><<<grid, kWarps * 32, 0, st>>>(n, rowptr_t, colidx_t, perm_t, widx, w, coef, dvals, dvals_t, work);
    count_launch();
    if (diff)
        norm_grad_rows_kernel<true><<<grid, kWarps * 32, 0, st>>>(n, rowptr, colidx, widx, w, coef, dvals, work, dw);
    else
        norm_grad_rows_kernel<false><<<grid, kWarps * 32, 0, st>>>(n, rowptr, colidx, widx, w, coef, dvals, work, dw);
    count_launch();
    return check_launch("adj_norm_bwd");
}

// the checks the pattern <-> dense entry points share: `in` (n x n, or nnz values) is read, `out` (nnz values, or n x n)
// written, and the output shares no byte with the inputs
static int32_t check_pattern_dense(const char* what, int64_t n, const int32_t* rowptr, const int32_t* colidx, int64_t nnz,
                                   const void* in, int64_t in_count, const void* out, int64_t out_count) {
    STMGCN_REQUIRE(n > 0 && n < ((int64_t)1 << 24) && nnz >= 0 && nnz < ((int64_t)1 << 31), STMGCN_ERR_SHAPE,
                   "%s: n=%lld must be in [1, 2^24) and nnz=%lld in [0, 2^31)", what, (long long)n, (long long)nnz);
    STMGCN_REQUIRE(rowptr, STMGCN_ERR_ARG, "%s: null rowptr", what);
    STMGCN_REQUIRE((in || in_count == 0) && (out || out_count == 0) && (colidx || nnz == 0), STMGCN_ERR_ARG,
                   "%s: null colidx / input / output", what);
    const int64_t i4 = 4;
    const Range o = {out, out_count * i4};
    const Range ins[] = {{rowptr, (n + 1) * i4}, {colidx, nnz * i4}, {in, in_count * i4}};
    for (const Range& r : ins)
        STMGCN_REQUIRE(!overlaps(o, r), STMGCN_ERR_ARG, "%s: the output overlaps an input", what);
    return 0;
}

extern "C" int32_t stmgcn_pattern_scatter(int64_t n, const int32_t* rowptr, const int32_t* colidx, int64_t nnz,
                                          const float* vals, float* dense, void* stream) {
    if (int32_t rc = check_pattern_dense("pattern_scatter", n, rowptr, colidx, nnz, vals, nnz, dense, n * n)) return rc;
    pattern_scatter_kernel<<<(unsigned)ceil_div(n, kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(n, rowptr, colidx,
                                                                                                  vals, dense);
    count_launch();
    return check_launch("pattern_scatter");
}

extern "C" int32_t stmgcn_pattern_gather(int64_t n, const int32_t* rowptr, const int32_t* colidx, int64_t nnz,
                                         const float* dense, float* dvals, void* stream) {
    if (int32_t rc = check_pattern_dense("pattern_gather", n, rowptr, colidx, nnz, dense, n * n, dvals, nnz)) return rc;
    if (nnz == 0) return 0;            // no entry, no gradient: nothing is enqueued
    pattern_gather_kernel<<<(unsigned)ceil_div(n, kWarps), kWarps * 32, 0, (cudaStream_t)stream>>>(n, rowptr, colidx,
                                                                                                 dense, dvals);
    count_launch();
    return check_launch("pattern_gather");
}
