// K2 on the Hopper tensor cores (p = q = 64, the reference's lstm_hidden_dim / gcn_hidden_dim, Main.py:62-63):
//   forward : out[128 x 64]  = act( [T_0X | T_1X | ... | T_KX][128 x Ks*64] . W[Ks*64 x 64] + b )   (GCN.py:37-42)
//             -- the A operand is read segment by segment straight from the Chebyshev stack the SpMM steps wrote
//             (no torch.cat), split to tf32 hi/lo on its way to shared memory, accumulated in registers by wgmma
//             (3xTF32, tc_common.cuh)
//   backward: dZ = dOut (.) [out > 0] is formed in the loader (and written out for the weight-gradient kernel, with
//             the bias gradient as a by-product);  U[128 x Ks*64] = dZ[128 x 64] . W^T  -> U_k segments
// CTA = two warpgroups, one 128-row tile at a time (persistent over tiles); warpgroup w owns rows 64w .. 64w+63 of the
// tile.  Per 32-wide k-block every thread loads its share of A (and the pre-packed weight image), the block stores both
// into one shared-memory stage, and each warpgroup issues 3 x 4 wgmma (k8) into its accumulator; the global loads of
// the next k-block are in flight while those run.
#include "tc_pipeline.cuh"

using namespace stmgcn;
using namespace stmgcn::tc;

namespace {

constexpr int kPThreads = 256;
constexpr int kPWarps = kPThreads / 32;
constexpr int kMaxSeg = 8;

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
    // backward (dz mode): A = d_out (.) [out > 0]
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
            else wgmma_tf32_n256(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), sc);
        }
    }
}

template <int N, bool DZ>
__global__ void __launch_bounds__(kPThreads, 1) proj_rows_tc_kernel(const __grid_constant__ PParams p) {
    using Cfg = PCfg<N>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* st = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // keeps the __shared__ address space
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
                            if (!(m.x > 0.f)) d.x = 0.f;
                            if (!(m.y > 0.f)) d.y = 0.f;
                            if (!(m.z > 0.f)) d.z = 0.f;
                            if (!(m.w > 0.f)) d.w = 0.f;
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
                    if (p.act == STMGCN_ACT_RELU) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
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
    const int grid = p.n_tiles < sm_count() ? p.n_tiles : sm_count();
    kern<<<grid, kPThreads, psmem<64>(), st>>>(p);
    count_launch();
    return check_launch("proj_fwd_tc");
}

// backward data: dZ = d_out (.) mask (written to dz_out, bias gradient accumulated), U_k = dZ W_k^T (if u != nullptr);
// wimg_t = image of B[n = k*64+i][k' = j] = W[n][j]  (2 k-blocks of [hi|lo] [ks*64][32])
int32_t launch_proj_bwd_tc(const float* d_out, const float* out_act, int act, int64_t rows, int ks, const float* wimg_t,
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
    const int grid = p.n_tiles < sm_count() ? p.n_tiles : sm_count();
    kern<<<grid, kPThreads, psmem<256>(), st>>>(p);
    count_launch();
    return check_launch("proj_bwd_tc");
}

int32_t launch_pack_image(const float* src, int n_rows, int k_cols, int64_t rs, int64_t cs, float* img, int tile_rows,
                          cudaStream_t st) {
    pack_image_kernel<<<(n_rows * k_cols + 255) / 256, 256, 0, st>>>(src, n_rows, k_cols, rs, cs, img, tile_rows);
    count_launch();
    return check_launch("pack_image");
}

}  // namespace stmgcn
