// K1: one Chebyshev recurrence step on node-major features (replaces the dense einsum GCN.py:35 and the
// matrix-matrix recurrence GCN.py:125-135):   Y = alpha * op(A) X + beta * Z + gamma * U.
//
// One warp owns one output row x one 128-float column tile; lanes hold a float4 each, so every non-zero drives one
// fully coalesced 512 B gather of the neighbour's feature run.  The grid is column-tile-major (blockIdx.y = column tile)
// so the CTAs resident at any moment share one column tile of X (N x 512 B = 2 MB at N=4096): gathers are served by
// L2/L1, HBM sees X, Z, U once and Y once.
// The kernel's time is its gather volume nnz*F*4 B (2.87 GB per launch at BASELINE configs[2]) divided by what the
// on-chip levels can serve for RANDOM row gathers, not its algorithmic HBM bytes (bench.py reports both).
#include "common.cuh"
#include <stdlib.h>

using namespace stmgcn;

namespace {

constexpr int kRowsPerCta = 32;
constexpr int kWarpsPerCta = 8;

template <int VEC>
struct VecT;
template <>
struct VecT<4> {
    using type = float4;
};
template <>
struct VecT<1> {
    using type = float;
};

__device__ __forceinline__ void fma_vec(float4& a, float s, const float4& x) {
    a.x = fmaf(s, x.x, a.x);
    a.y = fmaf(s, x.y, a.y);
    a.z = fmaf(s, x.z, a.z);
    a.w = fmaf(s, x.w, a.w);
}
__device__ __forceinline__ void fma_vec(float& a, float s, const float& x) { a = fmaf(s, x, a); }
__device__ __forceinline__ float4 zero_vec(float4*) { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float zero_vec(float*) { return 0.f; }
__device__ __forceinline__ float4 axpbypcz(float a, const float4& x, float b, const float4& y, float c,
                                           const float4& z) {
    return make_float4(a * x.x + b * y.x + c * z.x, a * x.y + b * y.y + c * z.y, a * x.z + b * y.z + c * z.z,
                       a * x.w + b * y.w + c * z.w);
}
__device__ __forceinline__ float axpbypcz(float a, float x, float b, float y, float c, float z) {
    return a * x + b * y + c * z;
}

template <int VEC>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
spmm_row_gather_kernel(int64_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                       const float* __restrict__ vals, float alpha, const float* __restrict__ x, float beta,
                       const float* __restrict__ z, float gamma, const float* __restrict__ u,
                       float* __restrict__ y, int64_t f_total) {
    using V = typename VecT<VEC>::type;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int64_t f = ((int64_t)blockIdx.y * 32 + lane) * VEC;      // first feature of this lane
    const bool live = f < f_total;
    const int64_t row0 = (int64_t)blockIdx.x * kRowsPerCta;
    for (int r = warp; r < kRowsPerCta; r += kWarpsPerCta) {
        const int64_t row = row0 + r;
        if (row >= n) break;
        const int32_t beg = rowptr[row], end = rowptr[row + 1];
        V acc0 = zero_vec((V*)nullptr), acc1 = zero_vec((V*)nullptr);
        int32_t i = beg;
        if (live) {
            for (; i + 4 <= end; i += 4) {
                const int32_t c0 = __ldg(colidx + i), c1 = __ldg(colidx + i + 1);
                const int32_t c2 = __ldg(colidx + i + 2), c3 = __ldg(colidx + i + 3);
                const float v0 = __ldg(vals + i), v1 = __ldg(vals + i + 1);
                const float v2 = __ldg(vals + i + 2), v3 = __ldg(vals + i + 3);
                const V x0 = *reinterpret_cast<const V*>(x + (int64_t)c0 * f_total + f);
                const V x1 = *reinterpret_cast<const V*>(x + (int64_t)c1 * f_total + f);
                const V x2 = *reinterpret_cast<const V*>(x + (int64_t)c2 * f_total + f);
                const V x3 = *reinterpret_cast<const V*>(x + (int64_t)c3 * f_total + f);
                fma_vec(acc0, v0, x0);
                fma_vec(acc1, v1, x1);
                fma_vec(acc0, v2, x2);
                fma_vec(acc1, v3, x3);
            }
            for (; i < end; ++i) {
                const int32_t c0 = __ldg(colidx + i);
                const float v0 = __ldg(vals + i);
                const V x0 = *reinterpret_cast<const V*>(x + (int64_t)c0 * f_total + f);
                fma_vec(acc0, v0, x0);
            }
            V acc = axpbypcz(1.f, acc0, 1.f, acc1, 0.f, acc0);
            const int64_t off = row * f_total + f;
            V zz = zero_vec((V*)nullptr), uu = zero_vec((V*)nullptr);
            if (z != nullptr) zz = *reinterpret_cast<const V*>(z + off);
            if (u != nullptr) uu = *reinterpret_cast<const V*>(u + off);
            *reinterpret_cast<V*>(y + off) = axpbypcz(alpha, acc, beta, zz, gamma, uu);
        }
    }
}

// ---- bf16 gather source (the bf16-arithmetic mode of the bf16-quoted configurations) ---------------------------------
// The kernel's time is its gather volume, so the GATHERED operand is read from a bf16 shadow copy (half the bytes per
// neighbour); the recurrence's own-row operands z, u and the result y stay fp32 (they are read / written once), and the
// kernel writes the bf16 shadow of y for the next step.  A lane holds 8 bf16 = 16 bytes: one non-zero is still one fully
// coalesced 512-byte gather per warp, now covering 256 features.
__device__ __forceinline__ void fma_bf16x8(float (&acc)[8], float s, const uint4& v) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        acc[2 * j] = fmaf(s, __uint_as_float(w[j] << 16), acc[2 * j]);
        acc[2 * j + 1] = fmaf(s, __uint_as_float(w[j] & 0xffff0000u), acc[2 * j + 1]);
    }
}
__device__ __forceinline__ uint32_t pack2_bf16(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}

__global__ void __launch_bounds__(kWarpsPerCta * 32)
spmm_row_gather16_kernel(int64_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                         const float* __restrict__ vals, float alpha, const uint16_t* __restrict__ x16, float beta,
                         const float* z, float gamma, const float* u, float* y,      // (u may alias y: no __restrict__)
                         uint16_t* __restrict__ y16, int64_t f_total) {
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int64_t f = ((int64_t)blockIdx.y * 32 + lane) * 8;       // first feature of this lane
    if (f >= f_total) return;
    const int64_t row0 = (int64_t)blockIdx.x * kRowsPerCta;
    for (int r = warp; r < kRowsPerCta; r += kWarpsPerCta) {
        const int64_t row = row0 + r;
        if (row >= n) break;
        const int32_t beg = rowptr[row], end = rowptr[row + 1];
        float a0[8], a1[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) a0[j] = a1[j] = 0.f;
        int32_t i = beg;
        for (; i + 4 <= end; i += 4) {
            const int32_t c0 = __ldg(colidx + i), c1 = __ldg(colidx + i + 1);
            const int32_t c2 = __ldg(colidx + i + 2), c3 = __ldg(colidx + i + 3);
            const float v0 = __ldg(vals + i), v1 = __ldg(vals + i + 1);
            const float v2 = __ldg(vals + i + 2), v3 = __ldg(vals + i + 3);
            const uint4 x0 = *reinterpret_cast<const uint4*>(x16 + (int64_t)c0 * f_total + f);
            const uint4 x1 = *reinterpret_cast<const uint4*>(x16 + (int64_t)c1 * f_total + f);
            const uint4 x2 = *reinterpret_cast<const uint4*>(x16 + (int64_t)c2 * f_total + f);
            const uint4 x3 = *reinterpret_cast<const uint4*>(x16 + (int64_t)c3 * f_total + f);
            fma_bf16x8(a0, v0, x0);
            fma_bf16x8(a1, v1, x1);
            fma_bf16x8(a0, v2, x2);
            fma_bf16x8(a1, v3, x3);
        }
        for (; i < end; ++i) {
            const int32_t c0 = __ldg(colidx + i);
            const float v0 = __ldg(vals + i);
            const uint4 x0 = *reinterpret_cast<const uint4*>(x16 + (int64_t)c0 * f_total + f);
            fma_bf16x8(a0, v0, x0);
        }
        const int64_t off = row * f_total + f;
        float res[8];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float4 zz = make_float4(0.f, 0.f, 0.f, 0.f), uu = zz;
            if (z != nullptr) zz = *reinterpret_cast<const float4*>(z + off + 4 * h);
            if (u != nullptr) uu = *reinterpret_cast<const float4*>(u + off + 4 * h);
            res[4 * h + 0] = alpha * (a0[4 * h + 0] + a1[4 * h + 0]) + beta * zz.x + gamma * uu.x;
            res[4 * h + 1] = alpha * (a0[4 * h + 1] + a1[4 * h + 1]) + beta * zz.y + gamma * uu.y;
            res[4 * h + 2] = alpha * (a0[4 * h + 2] + a1[4 * h + 2]) + beta * zz.z + gamma * uu.z;
            res[4 * h + 3] = alpha * (a0[4 * h + 3] + a1[4 * h + 3]) + beta * zz.w + gamma * uu.w;
            *reinterpret_cast<float4*>(y + off + 4 * h) = make_float4(res[4 * h], res[4 * h + 1], res[4 * h + 2], res[4 * h + 3]);
        }
        if (y16 != nullptr)
            *reinterpret_cast<uint4*>(y16 + off) = make_uint4(pack2_bf16(res[0], res[1]), pack2_bf16(res[2], res[3]),
                                                              pack2_bf16(res[4], res[5]), pack2_bf16(res[6], res[7]));
    }
}

// ---- K1b: CSR SDDMM, the gradient of a support's stored values ---------------------------------------------------
//   dvals[e] += sum_t coef[t] * < A_t[row(e), :], B_t[colidx[e], :] >
// The SpMM's gather, transposed: one warp owns one row x one column tile; lanes hold the row's own A_t run in registers
// (one vector per term) and every entry gathers B_t[colidx[e]]'s run (one coalesced 512 B read per warp, as the forward's
// X), then a fixed xor-tree warp sum.  Same column-tile-major grid as the SpMM (the resident CTAs share one column strip
// of every B_t in L2).  Each (entry, tile) partial has one owner; with more than one tile the partials go to the caller's
// workspace [tile][e] and a second pass adds them in tile order: no float atomics, two runs agree bit for bit.
constexpr int kMaxSddmmTerms = 8;
struct SddmmTerms {
    const float* a[kMaxSddmmTerms];
    const float* b[kMaxSddmmTerms];
    float coef[kMaxSddmmTerms];
};

__device__ __forceinline__ float round_bf16(float v) {
    return __uint_as_float(pack2_bf16(v, 0.f) << 16);
}
__device__ __forceinline__ float dot_vec(const float4& a, float4 b, bool rnd) {
    if (rnd) {
        b.x = round_bf16(b.x);
        b.y = round_bf16(b.y);
        b.z = round_bf16(b.z);
        b.w = round_bf16(b.w);
    }
    return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)));
}
__device__ __forceinline__ float dot_vec(float a, float b, bool rnd) { return a * (rnd ? round_bf16(b) : b); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// out[e] = partial of entry e over this CTA's column tile (accumulate: out[e] += it, the single-tile case)
template <int VEC, bool ROUND>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
sddmm_row_gather_kernel(int64_t n, const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, int nterms,
                        const SddmmTerms terms, int64_t f_total, float* __restrict__ out, int64_t tile_stride,
                        bool accumulate) {
    using V = typename VecT<VEC>::type;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int64_t f = ((int64_t)blockIdx.y * 32 + lane) * VEC;
    const bool live = f < f_total;
    float* __restrict__ dst = out + (int64_t)blockIdx.y * tile_stride;
    const int64_t row0 = (int64_t)blockIdx.x * kRowsPerCta;
    for (int r = warp; r < kRowsPerCta; r += kWarpsPerCta) {
        const int64_t row = row0 + r;
        if (row >= n) break;
        const int32_t beg = rowptr[row], end = rowptr[row + 1];
        if (beg == end) continue;
        V a[kMaxSddmmTerms];
#pragma unroll
        for (int t = 0; t < kMaxSddmmTerms; ++t) {
            a[t] = zero_vec((V*)nullptr);
            if (t < nterms && live) a[t] = *reinterpret_cast<const V*>(terms.a[t] + row * f_total + f);
        }
        int32_t i = beg;
        for (; i + 4 <= end; i += 4) {
            const int64_t c0 = __ldg(colidx + i), c1 = __ldg(colidx + i + 1);
            const int64_t c2 = __ldg(colidx + i + 2), c3 = __ldg(colidx + i + 3);
            float p0 = 0.f, p1 = 0.f, p2 = 0.f, p3 = 0.f;
            if (live) {
#pragma unroll
                for (int t = 0; t < kMaxSddmmTerms; ++t) {
                    if (t >= nterms) break;
                    const float* __restrict__ b = terms.b[t] + f;
                    const V b0 = *reinterpret_cast<const V*>(b + c0 * f_total);
                    const V b1 = *reinterpret_cast<const V*>(b + c1 * f_total);
                    const V b2 = *reinterpret_cast<const V*>(b + c2 * f_total);
                    const V b3 = *reinterpret_cast<const V*>(b + c3 * f_total);
                    const float cf = terms.coef[t];
                    p0 = fmaf(cf, dot_vec(a[t], b0, ROUND), p0);
                    p1 = fmaf(cf, dot_vec(a[t], b1, ROUND), p1);
                    p2 = fmaf(cf, dot_vec(a[t], b2, ROUND), p2);
                    p3 = fmaf(cf, dot_vec(a[t], b3, ROUND), p3);
                }
            }
            p0 = warp_sum(p0);
            p1 = warp_sum(p1);
            p2 = warp_sum(p2);
            p3 = warp_sum(p3);
            if (lane == 0) {
                if (accumulate) {
                    dst[i] += p0;
                    dst[i + 1] += p1;
                    dst[i + 2] += p2;
                    dst[i + 3] += p3;
                } else {
                    dst[i] = p0;
                    dst[i + 1] = p1;
                    dst[i + 2] = p2;
                    dst[i + 3] = p3;
                }
            }
        }
        for (; i < end; ++i) {
            const int64_t c0 = __ldg(colidx + i);
            float p0 = 0.f;
            if (live) {
#pragma unroll
                for (int t = 0; t < kMaxSddmmTerms; ++t) {
                    if (t >= nterms) break;
                    const V b0 = *reinterpret_cast<const V*>(terms.b[t] + c0 * f_total + f);
                    p0 = fmaf(terms.coef[t], dot_vec(a[t], b0, ROUND), p0);
                }
            }
            p0 = warp_sum(p0);
            if (lane == 0) {
                if (accumulate)
                    dst[i] += p0;
                else
                    dst[i] = p0;
            }
        }
    }
}

// second pass: dvals[e] += sum over tiles, in tile order
__global__ void sddmm_tiles_sum_kernel(const float* __restrict__ work, int64_t tiles, int64_t nnz,
                                       float* __restrict__ dvals) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        float s = work[e];
        for (int64_t t = 1; t < tiles; ++t) s += work[t * nnz + e];
        dvals[e] += s;
    }
}

__global__ void to_bf16_kernel(const float* __restrict__ x, uint16_t* __restrict__ y, int64_t n8) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 a = *reinterpret_cast<const float4*>(x + 8 * i), b = *reinterpret_cast<const float4*>(x + 8 * i + 4);
        *reinterpret_cast<uint4*>(y + 8 * i) = make_uint4(pack2_bf16(a.x, a.y), pack2_bf16(a.z, a.w), pack2_bf16(b.x, b.y), pack2_bf16(b.z, b.w));
    }
}

}  // namespace

extern "C" int32_t stmgcn_to_bf16(const float* x, void* y16, int64_t count, void* stream) {
    STMGCN_REQUIRE(x && y16, STMGCN_ERR_ARG, "to_bf16: null pointer");
    STMGCN_REQUIRE(count > 0 && count % 8 == 0 && aligned16(x) && aligned16(y16), STMGCN_ERR_SHAPE,
                   "to_bf16: count=%lld must be a positive multiple of 8, pointers 16-byte aligned", (long long)count);
    const int64_t n8 = count / 8;
    const int64_t cap = (int64_t)sm_count() * 16;
    const int blocks = (int)(n8 / 256 + 1 < cap ? n8 / 256 + 1 : cap);
    to_bf16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, (uint16_t*)y16, n8);
    count_launch();
    return check_launch("to_bf16");
}

extern "C" int32_t stmgcn_cheb_spmm_step16(int64_t n, const int32_t* rowptr, const int32_t* colidx, const float* vals,
                                           float alpha, const void* x16, float beta, const float* z, float gamma,
                                           const float* u, float* y, void* y16, int64_t f_total, void* stream) {
    STMGCN_REQUIRE(rowptr && x16 && y, STMGCN_ERR_ARG, "cheb_spmm_step16: null pointer");
    STMGCN_REQUIRE(n > 0, STMGCN_ERR_SHAPE, "cheb_spmm_step16: n=%lld", (long long)n);
    STMGCN_REQUIRE(x16 != y16, STMGCN_ERR_ARG, "cheb_spmm_step16: y16 must not alias x16");
    STMGCN_REQUIRE(f_total > 0 && f_total % 8 == 0 && aligned16(x16) && aligned16(y) && (!y16 || aligned16(y16)) &&
                       (!z || aligned16(z)) && (!u || aligned16(u)),
                   STMGCN_ERR_SHAPE, "cheb_spmm_step16: f_total=%lld must be a multiple of 8, pointers 16-byte aligned",
                   (long long)f_total);
    const int64_t col_tiles = ceil_div(f_total, 32 * 8);
    STMGCN_REQUIRE(col_tiles <= 65535, STMGCN_ERR_SHAPE, "cheb_spmm_step16: f_total=%lld too wide", (long long)f_total);
    dim3 grid((unsigned)ceil_div(n, kRowsPerCta), (unsigned)col_tiles);
    spmm_row_gather16_kernel<<<grid, kWarpsPerCta * 32, 0, (cudaStream_t)stream>>>(n, rowptr, colidx, vals, alpha, (const uint16_t*)x16,
                                                                                beta, z, gamma, u, y, (uint16_t*)y16, f_total);
    count_launch();
    return check_launch("cheb_spmm_step16");
}

extern "C" int32_t stmgcn_csr_sddmm(int64_t n, const int32_t* rowptr, const int32_t* colidx, int64_t nnz, int32_t nterms,
                                    const float* const* a, const float* const* b, const float* coef,
                                    int32_t round_b_bf16, int64_t f_total, float* work, int64_t work_count,
                                    float* dvals, void* stream) {
    STMGCN_REQUIRE(rowptr && a && b && coef, STMGCN_ERR_ARG, "csr_sddmm: null pointer");
    STMGCN_REQUIRE(n > 0 && nnz >= 0 && nnz < ((int64_t)1 << 31), STMGCN_ERR_SHAPE, "csr_sddmm: n=%lld nnz=%lld",
                   (long long)n, (long long)nnz);
    STMGCN_REQUIRE(nnz == 0 || (colidx && dvals), STMGCN_ERR_ARG, "csr_sddmm: colidx / dvals null with nnz=%lld",
                   (long long)nnz);
    STMGCN_REQUIRE(nterms >= 1 && nterms <= kMaxSddmmTerms, STMGCN_ERR_SHAPE, "csr_sddmm: nterms=%d (1..%d)", (int)nterms,
                   kMaxSddmmTerms);
    STMGCN_REQUIRE(f_total > 0, STMGCN_ERR_SHAPE, "csr_sddmm: f_total=%lld", (long long)f_total);
    STMGCN_REQUIRE(round_b_bf16 == 0 || round_b_bf16 == 1, STMGCN_ERR_ARG, "csr_sddmm: round_b_bf16=%d", (int)round_b_bf16);
    const bool vec4 = f_total % 4 == 0;
    SddmmTerms terms{};
    for (int t = 0; t < nterms; ++t) {
        STMGCN_REQUIRE(a[t] && b[t], STMGCN_ERR_ARG, "csr_sddmm: null operand of term %d", t);
        STMGCN_REQUIRE(!vec4 || (aligned16(a[t]) && aligned16(b[t])), STMGCN_ERR_ALIGN,
                       "csr_sddmm: f_total=%lld is a multiple of 4: the operands of term %d must be 16-byte aligned",
                       (long long)f_total, t);
        const int64_t op_bytes = n * f_total * 4;
        STMGCN_REQUIRE(!overlaps(a[t], op_bytes, dvals, nnz * 4) && !overlaps(b[t], op_bytes, dvals, nnz * 4) &&
                           !overlaps(a[t], op_bytes, work, work_count * 4) && !overlaps(b[t], op_bytes, work, work_count * 4),
                       STMGCN_ERR_ARG, "csr_sddmm: dvals / work must not overlap the operands of term %d", t);
        terms.a[t] = a[t];
        terms.b[t] = b[t];
        terms.coef[t] = coef[t];
    }
    const int64_t tiles = ceil_div(f_total, 32 * (vec4 ? 4 : 1));
    STMGCN_REQUIRE(tiles <= 65535, STMGCN_ERR_SHAPE, "csr_sddmm: f_total=%lld too wide", (long long)f_total);
    STMGCN_REQUIRE(tiles == 1 || nnz == 0 || (work && work_count >= tiles * nnz && !overlaps(work, work_count * 4, dvals, nnz * 4)),
                   STMGCN_ERR_ARG,
                   "csr_sddmm: %lld column tiles need a workspace of %lld floats distinct from dvals (work_count=%lld)",
                   (long long)tiles, (long long)(tiles * nnz), (long long)work_count);
    if (nnz == 0) return 0;             // no entry, nothing to add: nothing is enqueued
    cudaStream_t st = (cudaStream_t)stream;
    const bool one = tiles == 1;
    float* out = one ? dvals : work;
    const int64_t stride = one ? 0 : nnz;
    dim3 grid((unsigned)ceil_div(n, kRowsPerCta), (unsigned)tiles);
    const int blk = kWarpsPerCta * 32;
    if (vec4) {
        if (round_b_bf16)
            sddmm_row_gather_kernel<4, true><<<grid, blk, 0, st>>>(n, rowptr, colidx, nterms, terms, f_total, out, stride, one);
        else
            sddmm_row_gather_kernel<4, false><<<grid, blk, 0, st>>>(n, rowptr, colidx, nterms, terms, f_total, out, stride, one);
    } else {
        if (round_b_bf16)
            sddmm_row_gather_kernel<1, true><<<grid, blk, 0, st>>>(n, rowptr, colidx, nterms, terms, f_total, out, stride, one);
        else
            sddmm_row_gather_kernel<1, false><<<grid, blk, 0, st>>>(n, rowptr, colidx, nterms, terms, f_total, out, stride, one);
    }
    count_launch();
    if (!one) {
        int32_t rc = check_launch("csr_sddmm");
        if (rc != 0) return rc;
        const int64_t cap = (int64_t)sm_count() * 8;
        const int blocks = (int)(ceil_div(nnz, 256) < cap ? ceil_div(nnz, 256) : cap);
        sddmm_tiles_sum_kernel<<<blocks, 256, 0, st>>>(work, tiles, nnz, dvals);
        count_launch();
    }
    return check_launch("csr_sddmm");
}

extern "C" int32_t stmgcn_cheb_spmm_step(int64_t n, const int32_t* rowptr, const int32_t* colidx, const float* vals,
                                         float alpha, const float* x, float beta, const float* z, float gamma,
                                         const float* u, float* y, int64_t f_total, void* stream) {
    STMGCN_REQUIRE(rowptr && x && y, STMGCN_ERR_ARG, "cheb_spmm_step: null pointer");
    STMGCN_REQUIRE(n > 0, STMGCN_ERR_SHAPE, "cheb_spmm_step: n=%lld", (long long)n);
    STMGCN_REQUIRE(x != y, STMGCN_ERR_ARG, "cheb_spmm_step: y must not alias x");
    STMGCN_REQUIRE(f_total > 0, STMGCN_ERR_SHAPE, "cheb_spmm_step: f_total=%lld", (long long)f_total);
    cudaStream_t st = (cudaStream_t)stream;
    const bool vec4 = (f_total % 4 == 0) && aligned16(x) && aligned16(y) && (!z || aligned16(z)) &&
                      (!u || aligned16(u));
    const int vec = vec4 ? 4 : 1;
    const int64_t col_tiles = ceil_div(f_total, 32 * vec);
    STMGCN_REQUIRE(col_tiles <= 65535, STMGCN_ERR_SHAPE, "cheb_spmm_step: f_total=%lld too wide", (long long)f_total);
    dim3 grid((unsigned)ceil_div(n, kRowsPerCta), (unsigned)col_tiles);
    if (vec4)
        spmm_row_gather_kernel<4><<<grid, kWarpsPerCta * 32, 0, st>>>(n, rowptr, colidx, vals, alpha, x, beta, z, gamma, u, y, f_total);
    else
        spmm_row_gather_kernel<1><<<grid, kWarpsPerCta * 32, 0, st>>>(n, rowptr, colidx, vals, alpha, x, beta, z, gamma, u, y, f_total);
    count_launch();
    return check_launch("cheb_spmm_step");
}
