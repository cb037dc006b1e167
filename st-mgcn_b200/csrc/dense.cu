// K1e: one recurrence step with a DENSE support matrix on the tensor cores -- the primitive of K1 for a matrix too dense
// to gather (GCN.py:35 is a dense einsum):   Y = alpha * op(A) X + beta * Z + gamma * U,   A fp32 n x n (leading
// dimension lda), op(A) = A or A^T, X / Z / U / Y fp32 (n, F) row-major.
//
// wgmma computes Y's tile [128 rows i][BN columns f] as M = i, N = f, K = j (the contraction over A's columns).  tf32
// wgmma reads K-major operands only, so:
//   * A (op = A) is K-major as stored: row i, 32 consecutive j per k-block, float4 loads, split and stored swizzled as
//     the projection's A operand (proj_tc.cu);
//   * A (op = A^T) and X are MN-major (the contraction index is their row): each thread loads a 4 x 4 block (4 rows k,
//     4 consecutive mn) with four coalesced float4 loads, transposes it in registers and stores four 16-byte chunks,
//     one per mn row of the K-major tile.  Within a warp's 32 (mn) x 16 (k) unit, lane bit 0 and bits 3-4 pick the mn
//     quad and bits 1-2 the k quad, so each quarter-warp's stores land in 8 distinct swizzled chunks (no bank conflict)
//     and each load instruction reads four 128-byte rows.
// 3xTF32 (tc_common.cuh): A = A_hi + A_lo, X = X_hi + X_lo, split in registers on the way to shared memory (rounded,
// see put4); Ahi.Xhi + Alo.Xhi + Ahi.Xlo.  Each k-block's 32-term product is accumulated by the tensor cores alone and
// then added into an fp32 register total (IEEE adds): the tensor cores' own fp32 accumulation loses the low bits of
// small terms added to a large running sum, and a dense support matrix is exactly that -- a dense similarity graph's
// L~ x is ~70x smaller than its diagonal term, and accumulated over all 4096 terms in the tensor cores it came out
// 2.8e-4 off fp64 at cfg3's output (measured; the CSR step: 7e-6).  The bf16 twin multiplies the bf16 copy x16 (exact in tf32): Ahi.X + Alo.X, and writes
// the bf16 copy of Y for the next step.
// Two shared-memory stages: the global loads of k-block kb + 1 and their split stores into the other stage run under the
// wgmma of kb, whose product is then added to the total; one barrier per k-block.  Persistent grid over (row tile, column tile), column tiles fastest; the column-tile width BN (128 or
// 96: the register total doubles the accumulator) is the one whose schedule fills the SMs best (F = 768 at N = 4096:
// 256 tiles of 96 on 132 SMs, not 192 of 128).
// Every output element has one owner and a fixed k order (no split-K, no atomics): reruns are bit-identical.
#include "tc_common.cuh"
#include "wgmma.cuh"

using namespace stmgcn;
using namespace stmgcn::tc;

namespace {

constexpr int kTM = 128;                       // output rows per tile: warpgroup w owns rows 64w .. 64w+63
constexpr int kKB = 32;                        // k-block: one 128-byte swizzle row of fp32
constexpr int kThreads = 256;
constexpr int kABytes = kTM * kKB * 4;         // 16 KB: the hi or the lo A tile

template <int BN>
struct DmmCfg {
    static constexpr int kBBytes = BN * kKB * 4;
    static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;     // [A hi | A lo | X hi | X lo]
    static constexpr size_t kSmem = 1024 + 2 * (size_t)kStageBytes;
    static constexpr int kXUnits = BN / 32 * 2;                       // 32 (mn) x 16 (k) units of the X tile
    static constexpr int kXPer = (kXUnits + 7) / 8;                   // per warp
};

struct DmmParams {
    const float* a;
    int64_t lda;
    const float* x;          // fp32 operand (step) or nullptr
    const uint16_t* x16;     // bf16 operand (step16) or nullptr
    const float* z;          // nullable
    const float* u;          // nullable, may be y
    float* y;
    uint16_t* y16;           // nullable (step16 only)
    float alpha, beta, gamma;
    int64_t n, f;
    int64_t n_ct, n_tiles;
    int nkb;
};

// 4 consecutive floats of row `row` from column `col` of a row-major matrix (leading dimension ld), zeros past
// `rows` x `cols`.  VEC: one float4 (cols % 4 == 0, 16-byte aligned rows).
template <bool VEC>
__device__ __forceinline__ float4 ld4(const float* m, int64_t ld, int64_t row, int64_t col, int64_t rows, int64_t cols) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row >= rows || col >= cols) return v;
    const float* src = m + row * ld + col;
    if (VEC) return *reinterpret_cast<const float4*>(src);
    v.x = src[0];
    if (col + 1 < cols) v.y = src[1];
    if (col + 2 < cols) v.z = src[2];
    if (col + 3 < cols) v.w = src[3];
    return v;
}
// the same from a bf16 matrix, widened exactly (cols % 8 == 0: a quad is all in or all out)
__device__ __forceinline__ float4 ld4_bf16(const uint16_t* m, int64_t ld, int64_t row, int64_t col, int64_t rows,
                                           int64_t cols) {
    if (row >= rows || col >= cols) return make_float4(0.f, 0.f, 0.f, 0.f);
    const uint2 w = *reinterpret_cast<const uint2*>(m + row * ld + col);
    return make_float4(__uint_as_float(w.x << 16), __uint_as_float(w.x & 0xffff0000u), __uint_as_float(w.y << 16),
                       __uint_as_float(w.y & 0xffff0000u));
}
// the 4 x 4 block rows k0 .. k0+3, columns mn0 .. mn0+3 transposed: o[m] = the 4 k of column mn0 + m
template <bool VEC, bool B16>
__device__ __forceinline__ void ld4x4_t(float4 (&o)[4], const float* m, const uint16_t* m16, int64_t ld, int64_t k0,
                                        int64_t mn0, int64_t rows, int64_t cols) {
    float4 r[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) r[i] = B16 ? ld4_bf16(m16, ld, k0 + i, mn0, rows, cols) : ld4<VEC>(m, ld, k0 + i, mn0, rows, cols);
    o[0] = make_float4(r[0].x, r[1].x, r[2].x, r[3].x);
    o[1] = make_float4(r[0].y, r[1].y, r[2].y, r[3].y);
    o[2] = make_float4(r[0].z, r[1].z, r[2].z, r[3].z);
    o[3] = make_float4(r[0].w, r[1].w, r[2].w, r[3].w);
}

// 16-byte chunk k4 (k = 4 k4 .. 4 k4 + 3) of row mn of a K-major [rows][32] tile with the 128-byte swizzle
// (sw128<4>(mn, 4 k4)); SPLIT: tf32 hi at t, lo at t + lo_off; else v as it is (a bf16 value is exact in tf32).
// The split ROUNDS (hi = rna(v), lo = rna(v - hi): |v - hi - lo| <= 2^-24 |v|, errors of either sign) where K1d and K2
// truncate (2^-22, always towards zero): the products of a dense support matrix cancel (see the top), and the biased
// truncation error doubled cfg3's output error (measured).  (A finite value within half a tf32 ulp of FLT_MAX rounds
// to Inf, and then gives NaN as an Inf does.)
template <bool SPLIT>
__device__ __forceinline__ void put4(uint8_t* t, uint32_t lo_off, int mn, int k4, const float4& v) {
    const uint32_t off = (uint32_t)mn * 128u + ((((uint32_t)k4 ^ (uint32_t)mn) & 7u) << 4);
    if (!SPLIT) {
        *reinterpret_cast<float4*>(t + off) = v;
        return;
    }
    float4 hi, lo;
    hi.x = tf32_rna(v.x); hi.y = tf32_rna(v.y); hi.z = tf32_rna(v.z); hi.w = tf32_rna(v.w);
    lo.x = tf32_rna(v.x - hi.x); lo.y = tf32_rna(v.y - hi.y); lo.z = tf32_rna(v.z - hi.z); lo.w = tf32_rna(v.w - hi.w);
    *reinterpret_cast<float4*>(t + off) = hi;
    *reinterpret_cast<float4*>(t + lo_off + off) = lo;
}

// acc = A[64 x 32] . X[32 x BN]: Ahi.Xhi + Alo.Xhi (+ Ahi.Xlo with X_LO), four k8 steps each
template <int BN, bool X_LO>
__device__ __forceinline__ void dmm_mma(float (&acc)[BN / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
#pragma unroll
    for (int pass = 0; pass < (X_LO ? 3 : 2); ++pass) {
        const uint64_t da = smem_desc_k_sw128(pass == 1 ? a_lo : a_hi);
        const uint64_t db = smem_desc_k_sw128(pass == 2 ? b_lo : b_hi);
#pragma unroll
        for (int k = 0; k < kKB / 8; ++k) {
            const uint32_t sc = (pass > 0 || k > 0) ? 1u : 0u;
            if constexpr (BN == 128) wgmma_tf32_n128(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), sc);
            else wgmma_tf32_n96(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), sc);
        }
    }
}

__device__ __forceinline__ uint32_t pack2_bf16(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}

// VEC: 16-byte A loads (n % 4 == 0, lda % 4 == 0, A 16-byte aligned) and, fp32 operand, 16-byte X loads and 8-byte
// Y / Z / U accesses (F % 4 == 0, all 16-byte aligned); X16 always has them (F % 8 == 0, checked by the entry point)
template <int BN, bool TRANS, bool VEC, bool X16>
__global__ void __launch_bounds__(kThreads, 1) dense_mm_kernel(const __grid_constant__ DmmParams p) {
    using Cfg = DmmCfg<BN>;
    constexpr bool kVecOut = VEC || X16;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* st0 = smem_raw + smem_pad1024(smem_raw);
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int wg = tid >> 7;
    const int c = tid & 7, rsub = tid >> 3;                              // K-major A: chunk c of rows rsub + 32 i
    const int q = (lane & 1) | ((lane >> 3) << 1), kq = (lane >> 1) & 3;  // MN-major units: mn quad, k quad
    float acc[BN / 2], tot[BN / 2];
    float4 va[4];
    float4 vb[Cfg::kXPer][4];

    for (int64_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const int64_t ct = tile % p.n_ct, rt = tile / p.n_ct;
        const int64_t i0 = rt * kTM, f0 = ct * BN;
        auto load = [&](int kb) {
            const int64_t k0 = (int64_t)kb * kKB;
            if (!TRANS) {
#pragma unroll
                for (int i = 0; i < 4; ++i) va[i] = ld4<VEC>(p.a, p.lda, i0 + rsub + 32 * i, k0 + c * 4, p.n, p.n);
            } else {    // op(A)[i][j] = A[j][i]: warp w loads mn 32 (w & 3) .., k 16 (w >> 2) ..
                ld4x4_t<VEC, false>(va, p.a, nullptr, p.lda, k0 + 16 * (warp >> 2) + 4 * kq, i0 + 32 * (warp & 3) + 4 * q,
                                    p.n, p.n);
            }
#pragma unroll
            for (int s = 0; s < Cfg::kXPer; ++s) {
                const int unit = warp + 8 * s;
                if (unit < Cfg::kXUnits)
                    ld4x4_t<VEC, X16>(vb[s], p.x, p.x16, p.f, k0 + 16 * (unit & 1) + 4 * kq, f0 + 32 * (unit >> 1) + 4 * q,
                                      p.n, p.f);
            }
        };
        auto store = [&](int stage) {
            uint8_t* st = st0 + (size_t)stage * Cfg::kStageBytes;
            if (!TRANS) {
#pragma unroll
                for (int i = 0; i < 4; ++i) put4<true>(st, kABytes, rsub + 32 * i, c, va[i]);
            } else {
#pragma unroll
                for (int m = 0; m < 4; ++m) put4<true>(st, kABytes, 32 * (warp & 3) + 4 * q + m, 4 * (warp >> 2) + kq, va[m]);
            }
            uint8_t* sb = st + 2 * kABytes;
#pragma unroll
            for (int s = 0; s < Cfg::kXPer; ++s) {
                const int unit = warp + 8 * s;
                if (unit < Cfg::kXUnits) {
#pragma unroll
                    for (int m = 0; m < 4; ++m)
                        put4<!X16>(sb, Cfg::kBBytes, 32 * (unit >> 1) + 4 * q + m, 4 * (unit & 1) + kq, vb[s][m]);
                }
            }
        };
        load(0);
        __syncthreads();                                     // both warpgroups are done with the previous tile's stages
        store(0);
        fence_proxy_async_smem();
        __syncthreads();
        for (int kb = 0; kb < p.nkb; ++kb) {
            const uint32_t s_u = smem_u32(st0) + (uint32_t)(kb & 1) * (uint32_t)Cfg::kStageBytes;
            const uint32_t a_hi = s_u + (uint32_t)wg * 64u * 128u, a_lo = a_hi + kABytes;
            const uint32_t b_hi = s_u + 2 * kABytes, b_lo = b_hi + Cfg::kBBytes;
            wg_fence_regs(acc);
            wg_fence();
            dmm_mma<BN, !X16>(acc, a_hi, a_lo, b_hi, b_lo);
            wg_commit();
            if (kb + 1 < p.nkb) {
                // under this block's MMAs: the next block's loads and split stores into the other stage, whose last
                // reader, k-block kb - 1's MMAs, both warpgroups waited for before the barrier that ended that iteration
                load(kb + 1);
                store((kb + 1) & 1);
                fence_proxy_async_smem();
            }
            wg_wait<0>();
            wg_fence_regs(acc);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) tot[i] = kb == 0 ? acc[i] : tot[i] + acc[i];
            if (kb + 1 < p.nkb) __syncthreads();             // both stages' writes and reads of this block are done
        }
        // ===================== accumulator fragment -> y = alpha acc + beta z + gamma u =====================
        // (u may be y: each element is read and then written by the same thread)
        const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t i = i0 + r0 + 8 * h;
            if (i >= p.n) continue;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int64_t col = f0 + 8 * j + c0;
                if (col >= p.f) continue;
                const int64_t off = i * p.f + col;
                const float a0 = tot[4 * j + 2 * h], a1 = tot[4 * j + 2 * h + 1];
                if (kVecOut) {                                   // f even: col + 1 < f
                    float2 zz = make_float2(0.f, 0.f), uu = zz;
                    if (p.z != nullptr) zz = *reinterpret_cast<const float2*>(p.z + off);
                    if (p.u != nullptr) uu = *reinterpret_cast<const float2*>(p.u + off);
                    const float2 o = make_float2(p.alpha * a0 + p.beta * zz.x + p.gamma * uu.x,
                                                 p.alpha * a1 + p.beta * zz.y + p.gamma * uu.y);
                    *reinterpret_cast<float2*>(p.y + off) = o;
                    if (X16 && p.y16 != nullptr) *reinterpret_cast<uint32_t*>(p.y16 + off) = pack2_bf16(o.x, o.y);
                } else {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        if (col + e >= p.f) break;
                        const float zz = p.z != nullptr ? p.z[off + e] : 0.f;
                        const float uu = p.u != nullptr ? p.u[off + e] : 0.f;
                        p.y[off + e] = p.alpha * (e ? a1 : a0) + p.beta * zz + p.gamma * uu;
                    }
                }
            }
        }
    }
}

template <int BN, bool X16>
int32_t launch_bn(const DmmParams& p, bool trans, bool vec, cudaStream_t st) {
    auto kern = trans ? (vec ? dense_mm_kernel<BN, true, true, X16> : dense_mm_kernel<BN, true, false, X16>)
                      : (vec ? dense_mm_kernel<BN, false, true, X16> : dense_mm_kernel<BN, false, false, X16>);
    if (int32_t rc = ensure_dyn_smem((const void*)kern, DmmCfg<BN>::kSmem)) return rc;
    kern<<<persistent_grid(p.n_tiles), kThreads, DmmCfg<BN>::kSmem, st>>>(p);
    count_launch();
    return check_launch("dense_mm_step");
}

// Column-tile width: the one whose persistent schedule ends first, costing a round of tiles as its MMA width plus 64
// for the A tile's loads and split, which every tile pays whatever its width.
int column_tile(int64_t n, int64_t f) {
    const int64_t rt = ceil_div(n, kTM), sms = sm_count();
    const int64_t c128 = ceil_div(rt * ceil_div(f, 128), sms) * (128 + 64);
    const int64_t c96 = ceil_div(rt * ceil_div(f, 96), sms) * (96 + 64);
    return c96 < c128 ? 96 : 128;
}

// the checks both entry points share; y and x (x16: 2-byte elements) must not overlap, u must be y or apart from it
int32_t check_common(const char* what, int64_t n, const float* a, int64_t lda, int32_t transpose, const void* x,
                     int64_t x_elem, const float* z, const float* u, const float* y, int64_t f_total) {
    STMGCN_REQUIRE(a && x && y, STMGCN_ERR_ARG, "%s: null pointer", what);
    STMGCN_REQUIRE(transpose == 0 || transpose == 1, STMGCN_ERR_ARG, "%s: transpose=%d (0 or 1)", what, (int)transpose);
    STMGCN_REQUIRE(n >= 1 && n < (1 << 24), STMGCN_ERR_SHAPE, "%s: n=%lld must be in [1, 2^24)", what, (long long)n);
    STMGCN_REQUIRE(lda >= n && lda < ((int64_t)1 << 31), STMGCN_ERR_SHAPE, "%s: lda=%lld must be in [n, 2^31)", what,
                   (long long)lda);
    STMGCN_REQUIRE(f_total >= 1 && f_total < ((int64_t)1 << 31) && n * f_total < ((int64_t)1 << 48), STMGCN_ERR_SHAPE,
                   "%s: f_total=%lld must be in [1, 2^31) with n * f_total below 2^48", what, (long long)f_total);
    const int64_t op = n * f_total * 4, a_bytes = ((n - 1) * lda + n) * 4;
    STMGCN_REQUIRE(!overlaps(y, op, x, n * f_total * x_elem) && !overlaps(y, op, z, op) && !overlaps(y, op, a, a_bytes),
                   STMGCN_ERR_ARG, "%s: y must not overlap x, z or a", what);
    STMGCN_REQUIRE(u == y || !overlaps(y, op, u, op), STMGCN_ERR_ARG, "%s: u must be y or not overlap it", what);
    return 0;
}

DmmParams make_params(int64_t n, const float* a, int64_t lda, float alpha, float beta, const float* z, float gamma,
                      const float* u, float* y, int64_t f_total, int bn) {
    DmmParams p{};
    p.a = a;
    p.lda = lda;
    p.z = z;
    p.u = u;
    p.y = y;
    p.alpha = alpha;
    p.beta = beta;
    p.gamma = gamma;
    p.n = n;
    p.f = f_total;
    p.n_ct = ceil_div(f_total, bn);
    p.n_tiles = ceil_div(n, kTM) * p.n_ct;
    p.nkb = (int)ceil_div(n, kKB);
    return p;
}

}  // namespace

extern "C" int32_t stmgcn_dense_mm_step(int64_t n, const float* a, int64_t lda, int32_t transpose, float alpha,
                                        const float* x, float beta, const float* z, float gamma, const float* u, float* y,
                                        int64_t f_total, void* stream) {
    if (int32_t rc = check_common("dense_mm_step", n, a, lda, transpose, x, 4, z, u, y, f_total)) return rc;
    const int bn = column_tile(n, f_total);
    DmmParams p = make_params(n, a, lda, alpha, beta, z, gamma, u, y, f_total, bn);
    p.x = x;
    const bool vec = n % 4 == 0 && lda % 4 == 0 && aligned16(a) && f_total % 4 == 0 && aligned16(x) && aligned16(y) &&
                     (!z || aligned16(z)) && (!u || aligned16(u));
    cudaStream_t st = (cudaStream_t)stream;
    return bn == 128 ? launch_bn<128, false>(p, transpose, vec, st) : launch_bn<96, false>(p, transpose, vec, st);
}

extern "C" int32_t stmgcn_dense_mm_step16(int64_t n, const float* a, int64_t lda, int32_t transpose, float alpha,
                                          const void* x16, float beta, const float* z, float gamma, const float* u,
                                          float* y, void* y16, int64_t f_total, void* stream) {
    if (int32_t rc = check_common("dense_mm_step16", n, a, lda, transpose, x16, 2, z, u, y, f_total)) return rc;
    STMGCN_REQUIRE(f_total % 8 == 0 && aligned16(x16) && aligned16(y) && (!y16 || aligned16(y16)) && (!z || aligned16(z)) &&
                       (!u || aligned16(u)),
                   STMGCN_ERR_SHAPE, "dense_mm_step16: f_total=%lld must be a multiple of 8, pointers 16-byte aligned",
                   (long long)f_total);
    const int64_t op = n * f_total * 4, op16 = n * f_total * 2, a_bytes = ((n - 1) * lda + n) * 4;
    STMGCN_REQUIRE(!overlaps(y16, op16, x16, op16) && !overlaps(y16, op16, y, op) && !overlaps(y16, op16, z, op) &&
                       !overlaps(y16, op16, u, op) && !overlaps(y16, op16, a, a_bytes),
                   STMGCN_ERR_ARG, "dense_mm_step16: y16 must not overlap x16, y, z, u or a");
    const int bn = column_tile(n, f_total);
    DmmParams p = make_params(n, a, lda, alpha, beta, z, gamma, u, y, f_total, bn);
    p.x16 = (const uint16_t*)x16;
    p.y16 = (uint16_t*)y16;
    const bool vec = n % 4 == 0 && lda % 4 == 0 && aligned16(a);
    cudaStream_t st = (cudaStream_t)stream;
    return bn == 128 ? launch_bn<128, true>(p, transpose, vec, st) : launch_bn<96, true>(p, transpose, vec, st);
}
