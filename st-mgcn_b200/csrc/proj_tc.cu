// K2 on the Hopper tensor cores (p = q = 64, the reference's lstm_hidden_dim / gcn_hidden_dim, Main.py:62-63):
//   forward : out[128 x 64]  = act( [T_0X | T_1X | ... | T_KX][128 x Ks*64] . W[Ks*64 x 64] + b )   (GCN.py:37-42)
//             -- the A operand is read segment by segment straight from the Chebyshev stack the SpMM steps wrote
//             (no torch.cat), split to tf32 hi/lo on its way to shared memory, accumulated in registers by wgmma
//             (3xTF32, tc_common.cuh)
//   backward: dZ = dOut (.) [!(out <= 0)] is formed in the loader (and written out for the weight-gradient kernel, with
//             the bias gradient as a by-product);  U[128 x Ks*64] = dZ[128 x 64] . W^T  -> U_k segments;
//             dW[kd x 64] += [T_kX | T_{k+1}X]^T . dZ per pair of supports (proj_wgrad_tc_kernel)
// CTA = two warpgroups, one 128-row tile at a time (persistent over tiles); warpgroup w owns rows 64w .. 64w+63 of the
// tile.  Per 32-wide k-block every thread loads its share of A (and the pre-packed weight image), the block stores both
// into one shared-memory stage, and each warpgroup issues 3 x 4 wgmma (k8) into its accumulator; the global loads of
// the next k-block are in flight while those run.
#include "tc_common.cuh"
#include "wgmma.cuh"

using namespace stmgcn;
using namespace stmgcn::tc;

namespace {

constexpr int kTileM = 128;
constexpr int kKB = 32;                              // k-block: one 128-byte swizzle row of fp32
constexpr int kABytes = kTileM * kKB * 4;            // 16 KB per hi or lo A tile of 128 rows
constexpr int kPThreads = 256;
constexpr int kPWarps = kPThreads / 32;
constexpr int kMaxSeg = 8;

// hi at st + off, lo at st + kLo + off (the tile pair's lo half starts kLo bytes after its hi half)
template <uint32_t kLo = kABytes>
__device__ __forceinline__ void split_store(uint8_t* st, uint32_t off, const float4& v) {
    float4 hi, lo;
    hi.x = tf32_hi(v.x); hi.y = tf32_hi(v.y); hi.z = tf32_hi(v.z); hi.w = tf32_hi(v.w);
    lo.x = tf32_lo(v.x, hi.x); lo.y = tf32_lo(v.y, hi.y); lo.z = tf32_lo(v.z, hi.z); lo.w = tf32_lo(v.w, hi.w);
    *reinterpret_cast<float4*>(st + off) = hi;
    *reinterpret_cast<float4*>(st + kLo + off) = lo;
}

// transpose-store one float4 (4 consecutive M/N indices mn..mn+3 of row k) into a K-major swizzled tile pair
__device__ __forceinline__ void split_store_t(uint8_t* hi_tile, uint8_t* lo_tile, int mn, int k, const float4& v) {
    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t off = sw128<4>((uint32_t)(mn + j), (uint32_t)k);
        const float hi = tf32_hi(vv[j]);
        *reinterpret_cast<float*>(hi_tile + off) = hi;
        *reinterpret_cast<float*>(lo_tile + off) = tf32_lo(vv[j], hi);
    }
}

// K-major hi/lo image of a logical B[n][k] = src[n*rs + k*cs]: per 32-wide k-block [hi | lo], each an [n_rows][32] fp32
// tile with the 128-byte swizzle.
__global__ void pack_image_kernel(const float* __restrict__ src, int n_rows, int k_cols, int64_t rs, int64_t cs,
                                  float* __restrict__ img, int tile_rows) {
    const int total = n_rows * k_cols;
    const int tile_floats = tile_rows * kKB;      // tile_rows >= n_rows: extra rows keep what the caller put there (zeros)
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
        const int n = e / k_cols, k = e % k_cols;
        const float v = src[(int64_t)n * rs + (int64_t)k * cs];
        const float hi = tf32_hi(v);
        const float lo = tf32_lo(v, hi);
        const int kb = k / kKB, kk = k % kKB;
        const uint32_t off = sw128<4>((uint32_t)n, (uint32_t)kk) / 4;
        float* base = img + (size_t)kb * (2 * tile_floats);
        base[off] = hi;
        base[tile_floats + off] = lo;
    }
}

template <int N>
struct PCfg {
    static constexpr int kBBytes = N * kKB * 4;
    static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;
};

struct PTail {
    float bias[64];
    float s_db[kPWarps][64];
};
template <int N>
constexpr size_t psmem() { return 1024 + (size_t)PCfg<N>::kStageBytes + sizeof(PTail); }

struct PParams {
    const float* seg[kMaxSeg];   // forward: A segments (rows x 64)
    int nkb;                     // k-blocks (2 per 64-wide segment)
    // backward (dz mode): A = d_out (.) [!(out <= 0)]
    const float* d_out;          // (rows, 64) or nullptr
    const float* out_act;        // (rows, 64) forward output (mask source)
    int act;
    float* dz_out;               // (rows, 64) or nullptr (second pass of a > 4-support backward: dZ is already stored)
    float* dbias;                // (64) += or nullptr
    const float* wimg;
    const float* bias;           // forward epilogue
    float* out;                  // forward: (rows, 64)
    float* u;                    // backward: U_k = u + k*stride_u, (rows, 64) each
    int64_t stride_u;
    int ks_out;                  // backward: number of valid U segments (<= 4)
    int64_t rows;
    int n_tiles;
};

// acc (+)= A[64 x 32] . B[32 x N] in 3xTF32: Ahi.Bhi + Alo.Bhi + Ahi.Blo, four k8 steps each; `first` overwrites acc
template <int N>
__device__ __forceinline__ void proj_mma(float (&acc)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                         bool first) {
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {
        const uint64_t da = smem_desc_k_sw128(pass == 1 ? a_lo : a_hi);
        const uint64_t db = smem_desc_k_sw128(pass == 2 ? b_lo : b_hi);
#pragma unroll
        for (int k = 0; k < kKB / 8; ++k) {
            const uint32_t sc = (!first || pass > 0 || k > 0) ? 1u : 0u;
            if constexpr (N == 64) wgmma_tf32_n64(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), sc);
            else if constexpr (N == 128) wgmma_tf32_n128(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), sc);
            else wgmma_tf32_n256(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), sc);
        }
    }
}

template <int N, bool DZ>
__global__ void __launch_bounds__(kPThreads, 1) proj_rows_tc_kernel(const __grid_constant__ PParams p) {
    using Cfg = PCfg<N>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* st = smem_raw + smem_pad1024(smem_raw);
    PTail* tail = (PTail*)(st + (size_t)Cfg::kStageBytes);
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int wg = tid >> 7;                             // warpgroup: rows 64 wg .. 64 wg + 63 of the tile

    for (int i = tid; i < 64; i += kPThreads) tail->bias[i] = (!DZ && p.bias) ? p.bias[i] : 0.f;
    for (int i = tid; i < kPWarps * 64; i += kPThreads) (&tail->s_db[0][0])[i] = 0.f;
    __syncthreads();

    constexpr int kPer = 1024 / kPThreads;               // float4 of the 128 x 32 A block per thread
    constexpr int kBVec = 2 * Cfg::kBBytes / 16 / kPThreads;
    const int c = tid & 7, rsub = tid >> 3;
    const uint32_t s_u = smem_u32(st);
    const uint32_t a_hi = s_u + (uint32_t)wg * 64u * 128u, a_lo = a_hi + kABytes;
    const uint32_t b_hi = s_u + 2 * kABytes, b_lo = b_hi + Cfg::kBBytes;
    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;

    for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        for (int kb = 0; kb < p.nkb; ++kb) {
            const int koff = (kb & 1) * kKB + c * 4;
            float4 v[kPer];
            if (DZ) {
                float4 sb = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int i = 0; i < kPer; ++i) {
                    const int64_t r = (int64_t)tile * kTileM + rsub + 32 * i;
                    float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (r < p.rows) {
                        d = *reinterpret_cast<const float4*>(p.d_out + r * 64 + koff);
                        if (p.act == STMGCN_ACT_RELU) {
                            const float4 m = *reinterpret_cast<const float4*>(p.out_act + r * 64 + koff);
                            if (m.x <= 0.f) d.x = 0.f;
                            if (m.y <= 0.f) d.y = 0.f;
                            if (m.z <= 0.f) d.z = 0.f;
                            if (m.w <= 0.f) d.w = 0.f;
                        }
                    }
                    v[i] = d;
                    sb.x += d.x; sb.y += d.y; sb.z += d.z; sb.w += d.w;
                }
#pragma unroll
                for (int o = 8; o <= 16; o <<= 1) {
                    sb.x += __shfl_xor_sync(0xffffffffu, sb.x, o); sb.y += __shfl_xor_sync(0xffffffffu, sb.y, o);
                    sb.z += __shfl_xor_sync(0xffffffffu, sb.z, o); sb.w += __shfl_xor_sync(0xffffffffu, sb.w, o);
                }
                if (lane < 8) {
                    float4* a = reinterpret_cast<float4*>(&tail->s_db[warp][koff]);
                    float4 t = *a;
                    t.x += sb.x; t.y += sb.y; t.z += sb.z; t.w += sb.w;
                    *a = t;
                }
            } else {
                const float* seg = p.seg[kb >> 1];
#pragma unroll
                for (int i = 0; i < kPer; ++i) {
                    const int64_t r = (int64_t)tile * kTileM + rsub + 32 * i;
                    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (seg != nullptr && r < p.rows) v[i] = *reinterpret_cast<const float4*>(seg + r * 64 + koff);
                }
            }
            const uint4* wsrc = reinterpret_cast<const uint4*>(p.wimg + (size_t)kb * (2 * Cfg::kBBytes / 4));
            uint4 wv[kBVec];
#pragma unroll
            for (int i = 0; i < kBVec; ++i) wv[i] = wsrc[tid + i * kPThreads];
            wg_wait<0>();                                     // this warpgroup's MMAs of the previous k-block are done
            __syncthreads();                                  // ... and the other warpgroup's: the stage may be overwritten
#pragma unroll
            for (int i = 0; i < kPer; ++i) {
                const int row = rsub + 32 * i;
                // sw128<16>(row, c) without its final & 7, which would keep the swizzle from being hoisted out of i
                split_store(st, (uint32_t)row * 128u + (uint32_t)((c ^ (row & 7)) << 4), v[i]);
            }
#pragma unroll
            for (int i = 0; i < kBVec; ++i) reinterpret_cast<uint4*>(st + 2 * kABytes)[tid + i * kPThreads] = wv[i];
            fence_proxy_async_smem();
            __syncthreads();
            wg_fence_regs(acc);
            wg_fence();
            proj_mma<N>(acc, a_hi, a_lo, b_hi, b_lo, kb == 0);
            wg_commit();
            if (DZ && p.dz_out != nullptr) {   // dZ tape for the weight-gradient kernel
#pragma unroll
                for (int i = 0; i < kPer; ++i) {
                    const int64_t r = (int64_t)tile * kTileM + rsub + 32 * i;
                    if (r < p.rows) *reinterpret_cast<float4*>(p.dz_out + r * 64 + koff) = v[i];
                }
            }
        }
        wg_wait<0>();
        wg_fence_regs(acc);
        // ===================== epilogue: accumulator fragment -> global =====================
        const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t r = (int64_t)tile * kTileM + r0 + 8 * h;
            if (r >= p.rows) continue;
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int col = 8 * j + c0;
                float2 o = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                if (N == 64) {
                    o.x += tail->bias[col];
                    o.y += tail->bias[col + 1];
                    if (p.act == STMGCN_ACT_RELU) { o.x = relu_(o.x); o.y = relu_(o.y); }
                    *reinterpret_cast<float2*>(p.out + r * 64 + col) = o;
                } else {
                    if ((col >> 6) >= p.ks_out) continue;      // U_k, k = col / 64
                    *reinterpret_cast<float2*>(p.u + (int64_t)(col >> 6) * p.stride_u + r * 64 + (col & 63)) = o;
                }
            }
        }
    }
    __syncthreads();
    if (DZ && p.dbias != nullptr) {
        for (int i = tid; i < 64; i += kPThreads) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < kPWarps; ++w) v += tail->s_db[w][i];
            atomicAdd(&p.dbias[i], v);
        }
    }
}

// =====================================================================================================
// dW[kd x 64] += sum over rows r of [S_k | S_{k+1}][r, :]^T . dZ[r, :]   (kd = 128; kd = 64: S_k alone)
// M = kd index (warpgroup w owns kd rows 64w .. 64w+63), N = 64, K = rows, 32 rows per k-block.  Both operands are
// row-major in HBM (K is the slow dimension) and tf32 wgmma reads K-major operands only, so the loaders transpose on
// their way to shared memory: element (row r, m) lands at sw128<4>(m, r) of a [m][32 k] tile.  The accumulators live
// for the whole launch and are flushed with atomics once.
// =====================================================================================================
constexpr int kWgBBytes = 64 * kKB * 4;                            // dZ: [64][32 k] K-major
constexpr size_t kWgSmem = 1024 + 2 * (size_t)kABytes + 2 * (size_t)kWgBBytes;

struct WgParams {
    const float* s;          // S_k: (rows, 64)
    int64_t stride_k;        // S_{k+1} = s + stride_k (kd = 128)
    const float* dz;         // (rows, 64)
    float* dw;               // (kd, 64) +=
    int kd;                  // 128 or 64
    int64_t rows;
    int64_t n_chunks;        // ceil(rows / 32)
};

__global__ void __launch_bounds__(kPThreads, 1) proj_wgrad_tc_kernel(const __grid_constant__ WgParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* st = smem_raw + smem_pad1024(smem_raw);
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int wg = tid >> 7;
    constexpr int kNA = 1024 / kPThreads, kNB = (kKB * 64 / 4) / kPThreads;
    const uint32_t s_u = smem_u32(st);
    const uint32_t a_hi = s_u + (uint32_t)wg * 64u * 128u, a_lo = a_hi + kABytes;
    const uint32_t b_hi = s_u + 2 * kABytes, b_lo = b_hi + kWgBBytes;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    bool first = true;

    for (int64_t chunk = blockIdx.x; chunk < p.n_chunks; chunk += gridDim.x) {
        const int64_t r0 = chunk * kKB;
        float4 va[kNA], vb[kNB];
#pragma unroll
        for (int i = 0; i < kNA; ++i) {                   // A': 32 rows x 32 float4 (128 kd values), coalesced
            const int idx = tid + i * kPThreads;
            const int row = idx >> 5, q = idx & 31;
            const int64_t r = r0 + row;
            // m 0..63 from S_k, 64..127 from S_{k+1}
            const float* src = q < 16 ? p.s : (p.kd == 128 ? p.s + p.stride_k : nullptr);
            va[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (src != nullptr && r < p.rows) va[i] = *reinterpret_cast<const float4*>(src + r * 64 + (q & 15) * 4);
        }
#pragma unroll
        for (int i = 0; i < kNB; ++i) {                   // B': 32 rows x 16 float4, coalesced
            const int idx = tid + i * kPThreads;
            const int row = idx >> 4, q = idx & 15;
            const int64_t r = r0 + row;
            vb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < p.rows) vb[i] = *reinterpret_cast<const float4*>(p.dz + r * 64 + q * 4);
        }
        wg_wait<0>();
        __syncthreads();                                  // both warpgroups are done with the stage
#pragma unroll
        for (int i = 0; i < kNA; ++i) {
            const int idx = tid + i * kPThreads;
            split_store_t(st, st + kABytes, (idx & 31) * 4, idx >> 5, va[i]);
        }
#pragma unroll
        for (int i = 0; i < kNB; ++i) {
            const int idx = tid + i * kPThreads;
            split_store_t(st + 2 * kABytes, st + 2 * kABytes + kWgBBytes, (idx & 15) * 4, idx >> 4, vb[i]);
        }
        fence_proxy_async_smem();
        __syncthreads();
        wg_fence_regs(acc);
        wg_fence();
        proj_mma<64>(acc, a_hi, a_lo, b_hi, b_lo, first);
        wg_commit();
        first = false;
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    if (first) return;                                    // no chunk: nothing accumulated
    // ===================== accumulator fragment (rows = kd index) -> atomics into dW =====================
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = r0 + 8 * h;
        if (m >= p.kd) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            atomicAdd(p.dw + (int64_t)m * 64 + 8 * j + c0, acc[4 * j + 2 * h]);
            atomicAdd(p.dw + (int64_t)m * 64 + 8 * j + c0 + 1, acc[4 * j + 2 * h + 1]);
        }
    }
}

// =====================================================================================================
// Dense support gradient: da[k][i][j] = sum_f U_k[i][f] . x[j][f]   (dA_k = U_k x^T, GCN.py:35 differentiated in A)
// Both operands are row-major (n, f) with f contiguous, i.e. K-major as they sit in HBM: every k-block of 32 f is
// loaded row by row (float4 when f % 4 == 0 and the pointers are 16-byte aligned, scalars otherwise; rows past n and
// columns past f read as zeros), split to tf32 hi/lo and stored swizzled, exactly as the projection's A operand.
// Output tile 128 (i) x 256 (j): warpgroup w owns rows 64w .. 64w+63 against all 256 columns (wgmma m64n256k8, the
// projection backward's shape).  Two shared-memory stages: the wgmma of k-block kb run while the loads of kb + 1 are in
// flight and their split stores fill the other stage.  Persistent over (k, row tile, column tile), column tiles
// fastest; every output element has one owner and a fixed k order (no split-K, no atomics).
//
// Dense chain gradient (the same tile loop with a term loop): out[i][j] = sum_t coef_t sum_f A_t[i][f] . B_t[j][f], the
// gradient of a dense Chebyshev recurrence matrix X (A_t = G_k, B_t = T_{k-1}, coef 1 for k = 1 and 2 after).  The k
// blocks of all terms run as one sequence, term-major.  Its products cancel as K1e's do (a dense similarity graph's
// T_k carry a large diagonal part), so it takes K1e's scheme: the split ROUNDS (tf32_rna) and each k-block's product,
// accumulated by the tensor cores alone, is added times coef_t into an fp32 register total.  The total doubles the
// accumulator, so the tile is 128 x 128 (m64n128k8); the next block's loads and split stores run under the current
// block's wgmma.  round_b16: every B element rounded to bf16 (to nearest even) on load, the operand the bf16 forward
// multiplied.
// =====================================================================================================
constexpr int kDsgN = 256;
using DsgCfg = PCfg<kDsgN>;
constexpr size_t kDsgSmem = 1024 + 2 * (size_t)DsgCfg::kStageBytes;
constexpr int kDcgN = 128;
using DcgCfg = PCfg<kDcgN>;
constexpr size_t kDcgSmem = 1024 + 2 * (size_t)DcgCfg::kStageBytes;
constexpr int kMaxTerms = 8;

struct DsgParams {
    const float* u;          // U_k = u + k * u_stride, (n, f) each
    int64_t u_stride;
    const float* x;          // (n, f)
    float* da;               // (ks, n, n), overwritten
    int64_t n, f;
    int64_t n_rt, n_ct;      // row tiles of 128, column tiles of 256
    int64_t n_tiles;         // ks * n_rt * n_ct
    int nkb;                 // k-blocks: ceil(f / 32)
    bool pair_store;         // n even and da 8-byte aligned: float2 stores
};

struct DcgParams {
    const float* a[kMaxTerms];   // A_t (n, f)
    const float* b[kMaxTerms];   // B_t (n, f)
    float coef[kMaxTerms];
    float* out;                  // (n, n), overwritten
    int64_t n, f;
    int64_t n_rt, n_ct;          // row tiles of 128, column tiles of 128
    int64_t n_tiles;             // n_rt * n_ct
    int nkb;                     // k-blocks per term: ceil(f / 32)
    int nterms;
    bool pair_store;             // n even and out 8-byte aligned: float2 stores
    bool round_b16;
};

// 4 consecutive f of row `row` of a row-major (n, f) matrix, zeros past its edges
template <bool VEC>
__device__ __forceinline__ float4 dsg_load(const float* m, int64_t row, int64_t col, int64_t n, int64_t f) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row >= n || col >= f) return v;
    const float* src = m + row * f + col;
    if (VEC) return *reinterpret_cast<const float4*>(src);
    v.x = src[0];
    if (col + 1 < f) v.y = src[1];
    if (col + 2 < f) v.z = src[2];
    if (col + 3 < f) v.w = src[3];
    return v;
}

// v rounded to bf16 (to nearest even), widened back exactly
__device__ __forceinline__ float round_bf16(float v) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(0.f), "f"(v));
    return __uint_as_float(r << 16);
}

// the rounded split of split_store: hi at st + off, lo at st + kLo + off
template <uint32_t kLo>
__device__ __forceinline__ void split_store_rna(uint8_t* st, uint32_t off, const float4& v) {
    float4 hi, lo;
    hi.x = tf32_rna(v.x); hi.y = tf32_rna(v.y); hi.z = tf32_rna(v.z); hi.w = tf32_rna(v.w);
    lo.x = tf32_rna(v.x - hi.x); lo.y = tf32_rna(v.y - hi.y); lo.z = tf32_rna(v.z - hi.z); lo.w = tf32_rna(v.w - hi.w);
    *reinterpret_cast<float4*>(st + off) = hi;
    *reinterpret_cast<float4*>(st + kLo + off) = lo;
}

// the tile loop both kernels run; CHAIN: the chain gradient (DcgParams), else K1d (DsgParams)
template <bool VEC, bool CHAIN, class P>
__device__ __forceinline__ void dsg_tiles(const P& p) {
    constexpr int BN = CHAIN ? kDcgN : kDsgN;
    using Cfg = PCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* st0 = smem_raw + smem_pad1024(smem_raw);
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int wg = tid >> 7;
    const int c = tid & 7, rsub = tid >> 3;                  // float4 column of the k-block, first row
    constexpr int kNA = kTileM / 32, kNB = BN / 32;          // float4 per thread of the A / B block
    float acc[BN / 2];
    float tot[CHAIN ? BN / 2 : 1];

    for (int64_t tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        const int64_t ct = tile % p.n_ct, rest = tile / p.n_ct;
        const int64_t rt = rest % p.n_rt, k = rest / p.n_rt;
        const float* uk;
        const float* xk;
        if constexpr (CHAIN) {
            uk = p.a[0];
            xk = p.b[0];
        } else {
            uk = p.u + k * p.u_stride;
            xk = p.x;
        }
        const int64_t i0 = rt * kTileM, j0 = ct * BN;
        float4 va[kNA], vb[kNB];
        // k-block q: term q / nkb (CHAIN), columns 32 (q % nkb) ..
        auto load = [&](int q) {
            const float* ma = uk;
            const float* mb = xk;
            int kb = q;
            if constexpr (CHAIN) {
                const int t = q / p.nkb;
                kb = q - t * p.nkb;
                ma = p.a[t];
                mb = p.b[t];
            }
            const int64_t col = (int64_t)kb * kKB + c * 4;
#pragma unroll
            for (int i = 0; i < kNA; ++i) va[i] = dsg_load<VEC>(ma, i0 + rsub + 32 * i, col, p.n, p.f);
#pragma unroll
            for (int i = 0; i < kNB; ++i) vb[i] = dsg_load<VEC>(mb, j0 + rsub + 32 * i, col, p.n, p.f);
            if constexpr (CHAIN) {
                if (p.round_b16) {
#pragma unroll
                    for (int i = 0; i < kNB; ++i)
                        vb[i] = make_float4(round_bf16(vb[i].x), round_bf16(vb[i].y), round_bf16(vb[i].z), round_bf16(vb[i].w));
                }
            }
        };
        auto store = [&](int stage) {
            uint8_t* st = st0 + (size_t)stage * Cfg::kStageBytes;
#pragma unroll
            for (int i = 0; i < kNA; ++i) {
                const int row = rsub + 32 * i;
                const uint32_t off = (uint32_t)row * 128u + (uint32_t)((c ^ (row & 7)) << 4);
                if constexpr (CHAIN) split_store_rna<kABytes>(st, off, va[i]);
                else split_store(st, off, va[i]);
            }
#pragma unroll
            for (int i = 0; i < kNB; ++i) {
                const int row = rsub + 32 * i;
                const uint32_t off = (uint32_t)row * 128u + (uint32_t)((c ^ (row & 7)) << 4);
                if constexpr (CHAIN) split_store_rna<Cfg::kBBytes>(st + 2 * kABytes, off, vb[i]);
                else split_store<Cfg::kBBytes>(st + 2 * kABytes, off, vb[i]);
            }
        };
        load(0);
        __syncthreads();                                     // both warpgroups are done with the previous tile's stages
        store(0);
        fence_proxy_async_smem();
        __syncthreads();
        if constexpr (!CHAIN) {
            for (int kb = 0; kb < p.nkb; ++kb) {
                const uint32_t s_u = smem_u32(st0) + (uint32_t)(kb & 1) * (uint32_t)Cfg::kStageBytes;
                const uint32_t a_hi = s_u + (uint32_t)wg * 64u * 128u, a_lo = a_hi + kABytes;
                const uint32_t b_hi = s_u + 2 * kABytes, b_lo = b_hi + Cfg::kBBytes;
                wg_fence_regs(acc);
                wg_fence();
                proj_mma<BN>(acc, a_hi, a_lo, b_hi, b_lo, kb == 0);
                wg_commit();
                if (kb + 1 < p.nkb) {
                    load(kb + 1);
                    wg_wait<1>();                            // this warpgroup's MMAs of k-block kb - 1 are done
                    __syncthreads();                         // ... and the other's: their stage may be overwritten
                    store((kb + 1) & 1);
                    fence_proxy_async_smem();
                    __syncthreads();
                }
            }
            wg_wait<0>();
            wg_fence_regs(acc);
        } else {
            const int nq = p.nterms * p.nkb;
            for (int q = 0; q < nq; ++q) {
                const uint32_t s_u = smem_u32(st0) + (uint32_t)(q & 1) * (uint32_t)Cfg::kStageBytes;
                const uint32_t a_hi = s_u + (uint32_t)wg * 64u * 128u, a_lo = a_hi + kABytes;
                const uint32_t b_hi = s_u + 2 * kABytes, b_lo = b_hi + Cfg::kBBytes;
                wg_fence_regs(acc);
                wg_fence();
                proj_mma<BN>(acc, a_hi, a_lo, b_hi, b_lo, true);
                wg_commit();
                if (q + 1 < nq) {
                    // under this block's MMAs: the next block's loads and split stores into the other stage, whose last
                    // reader, block q - 1's MMAs, both warpgroups waited for before the barrier that ended that iteration
                    load(q + 1);
                    store((q + 1) & 1);
                    fence_proxy_async_smem();
                }
                wg_wait<0>();
                wg_fence_regs(acc);
                const float cf = p.coef[q / p.nkb];
#pragma unroll
                for (int i = 0; i < BN / 2; ++i) tot[i] = q == 0 ? cf * acc[i] : tot[i] + cf * acc[i];
                if (q + 1 < nq) __syncthreads();             // both stages' writes and reads of this block are done
            }
        }
        // ===================== accumulator fragment -> da[k] / out =====================
        float* dak;
        if constexpr (CHAIN) dak = p.out;
        else dak = p.da + k * p.n * p.n;
        const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int64_t i = i0 + r0 + 8 * h;
            if (i >= p.n) continue;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int64_t col = j0 + 8 * j + c0;
                float lo, hi;
                if constexpr (CHAIN) {
                    lo = tot[4 * j + 2 * h];
                    hi = tot[4 * j + 2 * h + 1];
                } else {
                    lo = acc[4 * j + 2 * h];
                    hi = acc[4 * j + 2 * h + 1];
                }
                if (p.pair_store) {
                    if (col < p.n) *reinterpret_cast<float2*>(dak + i * p.n + col) = make_float2(lo, hi);
                } else {
                    if (col < p.n) dak[i * p.n + col] = lo;
                    if (col + 1 < p.n) dak[i * p.n + col + 1] = hi;
                }
            }
        }
    }
}

template <bool VEC>
__global__ void __launch_bounds__(kPThreads, 1) dense_support_grad_kernel(const __grid_constant__ DsgParams p) {
    dsg_tiles<VEC, false>(p);
}

template <bool VEC>
__global__ void __launch_bounds__(kPThreads, 1) dense_chain_grad_kernel(const __grid_constant__ DcgParams p) {
    dsg_tiles<VEC, true>(p);
}

int32_t launch_pack_image(const float* src, int n_rows, int k_cols, int64_t rs, int64_t cs, float* img, int tile_rows,
                          cudaStream_t st) {
    pack_image_kernel<<<(n_rows * k_cols + 255) / 256, 256, 0, st>>>(src, n_rows, k_cols, rs, cs, img, tile_rows);
    count_launch();
    return check_launch("pack_image");
}

// dZ = d_out (.) mask (written to dz_out unless null, bias gradient accumulated unless null), U_k = dZ W_k^T for
// ks <= 4 supports; wimg_t = image of B[n = k*64+i][k' = j] = W[n][j]  (2 k-blocks of [hi|lo] [256][32])
int32_t launch_rows_bwd(const float* d_out, const float* out_act, int act, int64_t rows, int ks, const float* wimg_t,
                        float* dz_out, float* dbias, float* u, int64_t stride_u, cudaStream_t st) {
    auto kern = proj_rows_tc_kernel<256, true>;
    if (int32_t rc = ensure_dyn_smem((const void*)kern, psmem<256>())) return rc;
    PParams p{};
    p.nkb = 2;
    p.ks_out = ks;
    p.d_out = d_out;
    p.out_act = out_act;
    p.act = act;
    p.dz_out = dz_out;
    p.dbias = dbias;
    p.wimg = wimg_t;
    p.u = u;
    p.stride_u = stride_u;
    p.rows = rows;
    p.n_tiles = (int)ceil_div(rows, kTileM);
    kern<<<persistent_grid(p.n_tiles), kPThreads, psmem<256>(), st>>>(p);
    count_launch();
    return check_launch("proj_bwd_tc");
}

int32_t launch_wgrad(const float* s, int64_t stride_k, int kd, const float* dz, int64_t rows, float* dw, cudaStream_t st) {
    if (int32_t rc = ensure_dyn_smem((const void*)proj_wgrad_tc_kernel, kWgSmem)) return rc;
    WgParams p;
    p.s = s;
    p.stride_k = stride_k;
    p.dz = dz;
    p.dw = dw;
    p.kd = kd;
    p.rows = rows;
    p.n_chunks = ceil_div(rows, kKB);
    proj_wgrad_tc_kernel<<<persistent_grid(p.n_chunks), kPThreads, kWgSmem, st>>>(p);
    count_launch();
    return check_launch("proj_wgrad_tc");
}

}  // namespace

namespace stmgcn {

bool proj_tc_applicable(int ks, int p, int q, const void* a, const void* b, const void* c) {
    return p == 64 && q == 64 && ks >= 1 && ks <= 8 && aligned16(a) && aligned16(b) && (!c || aligned16(c));
}

// forward: out = act(sum_k S_k W_k + bias); wimg = image of B[n][k] = W[k][n] (2*ks k-blocks of [hi|lo] [64][32])
int32_t launch_proj_fwd_tc(const float* s, int64_t stride_k, int ks, int64_t rows, const float* wimg, const float* bias,
                           int act, float* out, cudaStream_t st) {
    auto kern = proj_rows_tc_kernel<64, false>;
    if (int32_t rc = ensure_dyn_smem((const void*)kern, psmem<64>())) return rc;
    PParams p{};
    for (int k = 0; k < ks; ++k) p.seg[k] = s + (int64_t)k * stride_k;
    p.nkb = 2 * ks;
    p.wimg = wimg;
    p.bias = bias;
    p.act = act;
    p.out = out;
    p.rows = rows;
    p.n_tiles = (int)ceil_div(rows, kTileM);
    kern<<<persistent_grid(p.n_tiles), kPThreads, psmem<64>(), st>>>(p);
    count_launch();
    return check_launch("proj_fwd_tc");
}

// backward: dZ + bias gradient + U in one row-kernel launch per group of 4 supports (the second one re-forms dZ in its
// loader but neither stores it nor accumulates the bias gradient again), then dW_k = S_k^T dZ, one launch per pair of
// supports (none when dw is NULL); wimg_t: stmgcn_proj_pack_tc's backward image
int32_t launch_proj_bwd_tc(const float* s, int64_t stride_k, int ks, int64_t rows, const float* d_out, const float* out_act,
                           int act, const float* wimg_t, float* dz, float* dbias, float* u, int64_t stride_u, float* dw,
                           cudaStream_t st) {
    if (int32_t rc = launch_rows_bwd(d_out, out_act, act, rows, ks < 4 ? ks : 4, wimg_t, dz, dbias, u, stride_u, st)) return rc;
    if (ks > 4)
        if (int32_t rc = launch_rows_bwd(d_out, out_act, act, rows, ks - 4, wimg_t + 2 * 2 * 256 * 32, nullptr, nullptr,
                                         u + 4 * stride_u, stride_u, st))
            return rc;
    for (int k0 = 0; k0 < ks && dw != nullptr; k0 += 2)
        if (int32_t rc = launch_wgrad(s + (int64_t)k0 * stride_k, stride_k, k0 + 1 < ks ? 128 : 64, dz, rows,
                                      dw + (int64_t)k0 * 64 * 64, st))
            return rc;
    return 0;
}

}  // namespace stmgcn

extern "C" int32_t stmgcn_proj_pack_tc(const float* w, int32_t ks, float* img_fwd, float* img_bwd, void* stream) {
    STMGCN_REQUIRE(w && img_fwd, STMGCN_ERR_ARG, "proj_pack_tc: null pointer");
    STMGCN_REQUIRE(ks >= 1 && ks <= 8, STMGCN_ERR_SHAPE, "proj_pack_tc: ks=%d (tensor-core path supports 1..8 supports)", ks);
    cudaStream_t st = (cudaStream_t)stream;
    // forward operand B[n = out col][k = ks*64 index] = W[k][n]
    if (int32_t rc = launch_pack_image(w, 64, ks * 64, 1, 64, img_fwd, 64, st)) return rc;
    // backward operand B[n = k*64+i][k' = out col] = W[n][k'], one 256-row image per group of 4 supports (caller
    // zero-fills img_bwd: rows beyond the last support stay zero)
    if (img_bwd) {
        const int k0 = ks < 4 ? ks : 4;
        if (int32_t rc = launch_pack_image(w, k0 * 64, 64, 64, 1, img_bwd, 256, st)) return rc;
        if (ks > 4) return launch_pack_image(w + (int64_t)256 * 64, (ks - 4) * 64, 64, 64, 1, img_bwd + 2 * 2 * 256 * 32, 256, st);
    }
    return 0;
}

extern "C" int32_t stmgcn_dense_support_grad(int64_t n, int64_t f_total, int32_t ks, const float* u, int64_t u_stride,
                                             const float* x, float* da, void* stream) {
    STMGCN_REQUIRE(u && x && da, STMGCN_ERR_ARG, "dense_support_grad: null pointer");
    STMGCN_REQUIRE(ks >= 1 && ks <= 8, STMGCN_ERR_SHAPE, "dense_support_grad: ks=%d (1..8 supports)", ks);
    STMGCN_REQUIRE(n >= 1 && n < (1 << 24), STMGCN_ERR_SHAPE, "dense_support_grad: n=%lld must be in [1, 2^24)", (long long)n);
    STMGCN_REQUIRE(f_total >= 1 && f_total < ((int64_t)1 << 31) && n * f_total < ((int64_t)1 << 48), STMGCN_ERR_SHAPE,
                   "dense_support_grad: f_total=%lld must be in [1, 2^31) with n * f_total below 2^48", (long long)f_total);
    STMGCN_REQUIRE(u_stride >= 0 && u_stride < ((int64_t)1 << 48), STMGCN_ERR_ARG, "dense_support_grad: u_stride=%lld",
                   (long long)u_stride);
    const int64_t op_bytes = n * f_total * 4, u_bytes = ((int64_t)(ks - 1) * u_stride + n * f_total) * 4;
    const int64_t da_bytes = (int64_t)ks * n * n * 4;
    STMGCN_REQUIRE(!overlaps(da, da_bytes, u, u_bytes) && !overlaps(da, da_bytes, x, op_bytes), STMGCN_ERR_ARG,
                   "dense_support_grad: da must not overlap u or x");
    DsgParams p;
    p.u = u;
    p.u_stride = u_stride;
    p.x = x;
    p.da = da;
    p.n = n;
    p.f = f_total;
    p.n_rt = ceil_div(n, kTileM);
    p.n_ct = ceil_div(n, kDsgN);
    p.n_tiles = (int64_t)ks * p.n_rt * p.n_ct;
    p.nkb = (int)ceil_div(f_total, kKB);
    p.pair_store = n % 2 == 0 && (reinterpret_cast<uintptr_t>(da) & 7u) == 0;
    const bool vec = f_total % 4 == 0 && aligned16(u) && aligned16(x) && (ks == 1 || u_stride % 4 == 0);
    auto kern = vec ? dense_support_grad_kernel<true> : dense_support_grad_kernel<false>;
    if (int32_t rc = ensure_dyn_smem((const void*)kern, kDsgSmem)) return rc;
    kern<<<persistent_grid(p.n_tiles), kPThreads, kDsgSmem, (cudaStream_t)stream>>>(p);
    count_launch();
    return check_launch("dense_support_grad");
}

extern "C" int32_t stmgcn_dense_chain_grad(int64_t n, int64_t f_total, int32_t nterms, const float* const* a,
                                           const float* const* b, const float* coef, int32_t round_b16, float* out,
                                           void* stream) {
    STMGCN_REQUIRE(nterms >= 1 && nterms <= kMaxTerms, STMGCN_ERR_SHAPE, "dense_chain_grad: nterms=%d (1..%d)", nterms,
                   kMaxTerms);
    STMGCN_REQUIRE(a && b && coef && out, STMGCN_ERR_ARG, "dense_chain_grad: null pointer");
    STMGCN_REQUIRE(round_b16 == 0 || round_b16 == 1, STMGCN_ERR_ARG, "dense_chain_grad: round_b16=%d (0 or 1)", round_b16);
    STMGCN_REQUIRE(n >= 1 && n < (1 << 24), STMGCN_ERR_SHAPE, "dense_chain_grad: n=%lld must be in [1, 2^24)", (long long)n);
    STMGCN_REQUIRE(f_total >= 1 && f_total < ((int64_t)1 << 31) && n * f_total < ((int64_t)1 << 48), STMGCN_ERR_SHAPE,
                   "dense_chain_grad: f_total=%lld must be in [1, 2^31) with n * f_total below 2^48", (long long)f_total);
    const int64_t op_bytes = n * f_total * 4, out_bytes = n * n * 4;
    bool vec = f_total % 4 == 0;
    for (int t = 0; t < nterms; ++t) {
        STMGCN_REQUIRE(a[t] && b[t], STMGCN_ERR_ARG, "dense_chain_grad: null A / B of term %d", t);
        STMGCN_REQUIRE(!overlaps(out, out_bytes, a[t], op_bytes) && !overlaps(out, out_bytes, b[t], op_bytes),
                       STMGCN_ERR_ARG, "dense_chain_grad: out must not overlap A / B of term %d", t);
        vec = vec && aligned16(a[t]) && aligned16(b[t]);
    }
    DcgParams p;
    for (int t = 0; t < kMaxTerms; ++t) {
        p.a[t] = t < nterms ? a[t] : nullptr;
        p.b[t] = t < nterms ? b[t] : nullptr;
        p.coef[t] = t < nterms ? coef[t] : 0.f;
    }
    p.out = out;
    p.n = n;
    p.f = f_total;
    p.n_rt = ceil_div(n, kTileM);
    p.n_ct = ceil_div(n, kDcgN);
    p.n_tiles = p.n_rt * p.n_ct;
    p.nkb = (int)ceil_div(f_total, kKB);
    p.nterms = nterms;
    p.pair_store = n % 2 == 0 && (reinterpret_cast<uintptr_t>(out) & 7u) == 0;
    p.round_b16 = round_b16 != 0;
    auto kern = vec ? dense_chain_grad_kernel<true> : dense_chain_grad_kernel<false>;
    if (int32_t rc = ensure_dyn_smem((const void*)kern, kDcgSmem)) return rc;
    kern<<<persistent_grid(p.n_tiles), kPThreads, kDcgSmem, (cudaStream_t)stream>>>(p);
    count_launch();
    return check_launch("dense_chain_grad");
}
