// K3b, second generation (H = 64): the shared LSTM of CG_LSTM (reference STMGCN.py:21-22, :47-50; nn.LSTM semantics)
// on the Hopper tensor cores (wgmma) with bf16 hi/lo PLANES ("3xBF16", see tc16.cuh) and NO gate tape.
//
// Tape written by the forward (all the backward needs; it recomputes the gates from it):
//   hp : (L, T, P, rows, 64) bf16  -- the hidden state of every layer-step as P planes (P = 2: hi | lo, fp32-grade
//        arithmetic; P = 1: hi only, the bf16 mode).  A 128-row x 64-column piece of a plane IS a K-major, 128-byte
//        swizzled wgmma operand tile once a TMA tensor load has put it into shared memory.
//   cs : (L, T, rows_pad, 64) fp32, tile-blocked ([tile][unit/4][128 rows][4 units], see below).
// 4 + 4 bytes per (row, unit, layer-step) instead of 4 + 4 + 16 with a gate tape.
//
// forward kernel (one launch per layer-step, persistent, one CTA per SM):
//   producer warp : loads the layer's weight image ONCE (resident for the whole launch: [256 gate cols][64 k] bf16 tiles,
//                   hi and lo, per K segment = 128 KB) and streams the A planes of every tile through a ring of 16 KB
//                   stages with TMA tensor loads (h_below hi, h_below lo, h_prev hi, h_prev lo)
//   2 warpgroups  : per tile and warpgroup (64 rows) 8 (P = 1) or 24 (P = 2) wgmma m64n256k16 into registers:
//                   Ahi.Whi + Ahi.Wlo + Alo.Whi, then bias (+ layer 0: x*s . W_ih in exact fp32) -> gates -> c, h ->
//                   h split into bf16 planes -> global stores.  Nothing of the gates leaves the SM.
#include "tc16.cuh"
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

using namespace stmgcn;
using namespace stmgcn::tc;

namespace stmgcn {
bool make_plane_map(CUtensorMap* map, const void* base, int64_t rows, int64_t slices);
}

namespace {

constexpr int kTileM = 128;
constexpr int kHid = 64;
constexpr int kGateCols = 256;
constexpr int kMaxC = 4;
constexpr int kWTileBytes = kGateCols * 128;          // [256 gate cols][64 k] bf16 = 32 KB
constexpr int kATileBytes = kTile16Bytes;             // [128 rows][64 k] bf16 = 16 KB

// element (row r, unit u) of a tile-blocked (rows_pad x 64) fp32 workspace lives at
//   (((r >> 7) * 16 + (unit >> 2)) * 128 + (r & 127)) * 4 + (unit & 3)        (host side: ops.to_blocked / from_blocked)

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 :: "r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// ---- LSTM cell with 8 MUFU operations instead of 10 ------------------------------------------------------------
// sigmoid(v) = 1 / (1 + e^-v), tanh(v) = (1 - e^-2v) / (1 + e^-2v).  Five exponentials per cell are unavoidable (i, f, g, o,
// tanh(c)); the five reciprocals are not: reciprocals of PRODUCTS of two (1 + e) terms serve two activations at once.
// The exponentials are capped at e^30 (the capped activations differ from the exact ones by < 1e-13) so that a
// product of two (1 + e^30) terms stays far below the fp32 overflow threshold.  The cell epilogue is MUFU-bound
// (16 MUFU results per clock and SM), so this is 20 % off its critical resource.
// (one-sided: only a large NEGATIVE argument makes e^-v large; for large positive v the exponential underflows to 0, which is exact)
// The kernels keep bias and W_ih PRE-SCALED by the exponent factor of their gate (kGateScale: -log2(e) for i, f, o and
// -2 log2(e) for g), so "accumulator + bias, times -log2(e)" is ONE fma per gate: arg = fma(acc, scale, bias_scaled).
__device__ __forceinline__ float gate_scale(int col) { return (col & 3) == 2 ? -2.8853900817779268f : -1.4426950408889634f; }
__device__ __forceinline__ float exp_arg_(float a) { return ex2_ftz_(fminf(a, 43.28f)); }      // e^(-v) or e^(-2v), <= e^30
// forward: exponent arguments of (i, f, g, o) and c_{t-1} -> c_t, h_t
__device__ __forceinline__ void lstm_cell_fwd8(float ai, float af, float ag, float ao, float cp, float& c, float& h) {
    const float ei = exp_arg_(ai), ef = exp_arg_(af), eg = exp_arg_(ag), eo = exp_arg_(ao);
    const float ig = (1.f - eg) * rcp_ftz_((1.f + ei) * (1.f + eg));          // sigmoid(pi) * tanh(pg)
    c = fmaf(rcp_ftz_(1.f + ef), cp, ig);
    const float ec = exp_arg_(-2.8853900817779268f * c);
    h = (1.f - ec) * rcp_ftz_((1.f + eo) * (1.f + ec));                      // sigmoid(po) * tanh(c)
}
// backward recompute: all four gate activations, c_t and tanh(c_t)
__device__ __forceinline__ void lstm_cell_gates8(float ai, float af, float ag, float ao, float cp, float& gi, float& gf,
                                                 float& gg, float& go, float& tc) {
    const float ei = 1.f + exp_arg_(ai), ef = 1.f + exp_arg_(af), eo = 1.f + exp_arg_(ao);
    const float eg = exp_arg_(ag);
    const float r1 = rcp_ftz_(ei * (1.f + eg));
    const float r2 = rcp_ftz_(ef * eo);
    gi = r1 * (1.f + eg);
    gg = (1.f - eg) * (r1 * ei);
    gf = r2 * eo;
    go = r2 * ef;
    const float ec = exp_arg_(-2.8853900817779268f * fmaf(gf, cp, gi * gg));
    tc = (1.f - ec) * rcp_ftz_(1.f + ec);
}

// =====================================================================================================
// forward
// =====================================================================================================
// CTA = two consumer warpgroups + one producer warp, persistent over 128-row tiles.  Warpgroup w owns rows 64w .. 64w+63
// of a tile and accumulates its [64 x 256] gate pre-activations in registers (wgmma m64n256k16).  Accumulator fragment
// (wgmma.cuh): thread holds columns 8j + 2(lane%4) + {0,1} of rows r0 and r0 + 8; with gate-interleaved columns
// n = 4 unit + gate that is gates (i, f) (lane%4 even) or (g, o) (odd) of unit 2j + (lane%4)/2.  Partner lanes (lane ^ 1)
// swap one row's pair, after which the even lane owns the cell (r0, unit) and the odd lane the cell (r0 + 8, unit).
constexpr int kFWarpgroups = 2;
constexpr int kFThreads = kFWarpgroups * 128 + 32;     // + producer warp
constexpr int kFStages = 5;

struct F16Tail {
    float bias[kGateCols];
    float wih[kMaxC * kGateCols];
    uint64_t full[kFStages];
    uint64_t empty[kFStages];
    uint64_t w_full;
};
constexpr size_t kFSmem = 1024 + 4 * (size_t)kWTileBytes + (size_t)kFStages * kATileBytes + sizeof(F16Tail);
static_assert(kFSmem <= 232448, "lstm16 forward kernel exceeds the 227 KB shared-memory limit");

struct Fwd16Params {
    alignas(64) CUtensorMap amap[2];   // per K segment: (64, rows, slices) bf16 view of a plane tensor, box 64 x 128 x 1, 128B swizzle
    int aslice[2];                     // slice of the segment's hi plane (lo plane = +1)
    int nseg;                          // K segments present: layer 0: h_prev; layers > 0: h_below, h_prev (absent at t = 0 without h0)
    const uint8_t* wimg;               // tiles [(seg*2 + plane)] of 32 KB
    const float* bias;                 // (256) gate-interleaved b_ih + b_hh
    const float* wih;                  // layer 0: (C, 256) gate-interleaved W_ih^T; else nullptr
    const float* xo;                   // (rows, T, C)
    const float* sg;                   // (B, T)
    int c_in, t, t_len;
    int64_t b_inner;
    const float* c_prev;               // tile-blocked or nullptr (zeros)
    float* c_out;                      // tile-blocked
    uint16_t* h_hi;                    // (rows, 64) bf16 plane
    uint16_t* h_lo;                    // (rows, 64) bf16 plane (PLANES = 2)
    float* h_f32;                      // (rows, 64) fp32 copy of h or nullptr
    int64_t rows;
    int n_tiles;
};

__device__ __forceinline__ uint16_t bf16_bits(float v) {
    return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}

// CIN: 0 = not layer 0; 1 = layer 0 with one input channel (the reference's input_dim, compile-time: no predicated-off
// W_ih FMAs / loads in the cell loop); kMaxC = layer 0 with a runtime channel count <= kMaxC
template <int PLANES, int CIN>
__global__ void __launch_bounds__(kFThreads, 1) lstm16_fwd_kernel(const __grid_constant__ Fwd16Params p) {
    constexpr bool L0 = CIN > 0;
    constexpr int kC = (CIN == 1) ? 1 : kMaxC;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* wsm = smem;                                           // resident weight tiles
    uint8_t* stages = smem + 4 * (size_t)kWTileBytes;
    F16Tail* tail = (F16Tail*)(stages + (size_t)kFStages * kATileBytes);
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    constexpr int kProdWarp = kFWarpgroups * 4;

    if (tid == 0) {
        for (int s = 0; s < kFStages; ++s) {
            mbar_init(&tail->full[s], 1);
            mbar_init(&tail->empty[s], kFWarpgroups);          // one arrival per consumer warpgroup
        }
        mbar_init(&tail->w_full, 1);
        fence_barrier_init();
    }
    for (int i = tid; i < kGateCols; i += kFThreads) tail->bias[i] = p.bias[i] * gate_scale(i);
    if (L0)
        for (int i = tid; i < p.c_in * kGateCols; i += kFThreads) tail->wih[i] = p.wih[i] * gate_scale(i);
    __syncthreads();
    const int my_tiles = (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

    if (warp == kProdWarp) {
        // ===================== producer: resident weights once, then the A planes of every tile =====================
        const bool leader = elect_one_sync();
        if (leader && p.nseg > 0) {
            mbar_arrive_expect_tx(&tail->w_full, (uint32_t)(p.nseg * PLANES * kWTileBytes));
            for (int s = 0; s < p.nseg; ++s)
                for (int pl = 0; pl < PLANES; ++pl)
                    bulk_g2s(wsm + (size_t)(s * 2 + pl) * kWTileBytes, p.wimg + (size_t)(s * 2 + pl) * kWTileBytes, kWTileBytes,
                             &tail->w_full);
            uint32_t it = 0;
            for (int i = 0; i < my_tiles; ++i) {
                const int tile = blockIdx.x + i * gridDim.x;
                if (p.c_prev != nullptr && i + 2 < my_tiles)     // c_{t-1} of the tile after next -> L2 (a tile is contiguous)
                    prefetch_l2(p.c_prev + (int64_t)(tile + 2 * (int)gridDim.x) * kTileM * kHid, kTileM * kHid * 4);
                for (int s = 0; s < p.nseg; ++s)
                    for (int pl = 0; pl < PLANES; ++pl, ++it) {
                        const int stg = it % kFStages;
                        const uint32_t ph = (it / kFStages) & 1;
                        mbar_wait_p(&tail->empty[stg], ph ^ 1, 0);
                        mbar_arrive_expect_tx(&tail->full[stg], kATileBytes);
                        tma_load_3d(stages + (size_t)stg * kATileBytes, &p.amap[s], 0, tile * kTileM, p.aslice[s] + pl,
                                    &tail->full[stg]);
                    }
            }
        }
        return;
    }
    // ===================== consumers: gate GEMM (wgmma) + LSTM cell =====================
    const int wg = tid >> 7;
    const int q = lane & 3;
    const bool odd = (q & 1) != 0;
    const uint32_t row_in_tile = (uint32_t)(64 * wg + 16 * (warp & 3) + (lane >> 2) + (odd ? 8 : 0));
    const uint32_t rows32 = (uint32_t)p.rows;
    const uint32_t w_u = smem_u32(wsm), a_u = smem_u32(stages) + (uint32_t)wg * 64u * 128u;
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    if (p.nseg > 0) mbar_wait(&tail->w_full, 0, 0);
    uint32_t it = 0;
    for (int i = 0; i < my_tiles; ++i) {
        const int tile = (int)blockIdx.x + i * (int)gridDim.x;
        const uint32_t r = (uint32_t)tile * kTileM + row_in_tile;
        const bool valid = r < rows32;
        // layer 0: x * s of this thread's row (loaded before the MMAs: the latency hides behind them)
        float xs[kMaxC];
        if (L0) {
            const float sv = valid ? p.sg[(r % (uint32_t)p.b_inner) * (uint32_t)p.t_len + (uint32_t)p.t] : 0.f;
#pragma unroll
            for (int c = 0; c < kMaxC; ++c)
                xs[c] = (c < kC && valid && (CIN == 1 || c < p.c_in)) ? p.xo[((int64_t)r * p.t_len + p.t) * p.c_in + c] * sv : 0.f;
        }
        wg_fence_regs(acc);
        for (int s = 0; s < p.nseg; ++s) {
            const uint64_t w_hi = desc16_k(w_u + (uint32_t)(s * 2) * kWTileBytes);
            const uint64_t w_lo = desc16_k(w_u + (uint32_t)(s * 2 + 1) * kWTileBytes);
#pragma unroll
            for (int pl = 0; pl < PLANES; ++pl, ++it) {
                const int stg = it % kFStages;
                mbar_wait(&tail->full[stg], (it / kFStages) & 1, 1);
                const uint64_t a_d = desc16_k(a_u + (uint32_t)stg * kATileBytes);
                wg_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    // hi plane: A_hi . W_hi (+ A_hi . W_lo); lo plane: A_lo . W_hi
                    wgmma_bf16_n256_t00(acc, a_d + (uint64_t)(2 * kk), w_hi + (uint64_t)(2 * kk), (s > 0 || pl > 0 || kk > 0) ? 1u : 0u);
                    if (PLANES == 2 && pl == 0) wgmma_bf16_n256_t00(acc, a_d + (uint64_t)(2 * kk), w_lo + (uint64_t)(2 * kk), 1u);
                }
                wg_commit();
                wg_wait<0>();
                wg_fence_regs(acc);
                // the stage has been read: one arrival per warpgroup
                asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
                if ((tid & 127) == 0) mbar_arrive(&tail->empty[stg]);
            }
        }
        if (p.nseg == 0) {
#pragma unroll
            for (int k = 0; k < 128; ++k) acc[k] = 0.f;
        }
        // ---- LSTM cell: 32 cells per thread, row row_in_tile, units 2j + q/2 ----
        const uint32_t cbase = (uint32_t)tile * 8192u + row_in_tile * 4u;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const float s0 = odd ? acc[4 * j + 0] : acc[4 * j + 2];
            const float s1 = odd ? acc[4 * j + 1] : acc[4 * j + 3];
            const float o0 = __shfl_xor_sync(0xffffffffu, s0, 1);
            const float o1 = __shfl_xor_sync(0xffffffffu, s1, 1);
            const float vi = odd ? o0 : acc[4 * j + 0], vf = odd ? o1 : acc[4 * j + 1];
            const float vg = odd ? acc[4 * j + 2] : o0, vo = odd ? acc[4 * j + 3] : o1;
            const int unit = 2 * j + (q >> 1);
            const int col = 4 * unit;
            const float4 bv = *reinterpret_cast<const float4*>(&tail->bias[col]);      // pre-scaled (gate_scale)
            float pi = fmaf(vi, -1.4426950408889634f, bv.x);
            float pf = fmaf(vf, -1.4426950408889634f, bv.y);
            float pg = fmaf(vg, -2.8853900817779268f, bv.z);
            float po = fmaf(vo, -1.4426950408889634f, bv.w);
            if (L0) {
#pragma unroll
                for (int c = 0; c < kC; ++c)
                    if (CIN == 1 || c < p.c_in) {
                        const float4 wv = *reinterpret_cast<const float4*>(&tail->wih[c * kGateCols + col]);
                        pi = fmaf(xs[c], wv.x, pi); pf = fmaf(xs[c], wv.y, pf);
                        pg = fmaf(xs[c], wv.z, pg); po = fmaf(xs[c], wv.w, po);
                    }
            }
            const uint32_t co = cbase + (uint32_t)(unit >> 2) * 512u + (uint32_t)(unit & 3);
            const float cp = (p.c_prev != nullptr && valid) ? p.c_prev[co] : 0.f;
            float cn, hn;
            lstm_cell_fwd8(pi, pf, pg, po, cp, cn, hn);
            if (valid) {
                p.c_out[co] = cn;
                const uint32_t ho = r * (uint32_t)kHid + (uint32_t)unit;
                const __nv_bfloat16 hb = __float2bfloat16_rn(hn);
                p.h_hi[ho] = __bfloat16_as_ushort(hb);
                if (PLANES == 2) p.h_lo[ho] = bf16_bits(hn - __bfloat162float(hb));
                if (p.h_f32 != nullptr) p.h_f32[ho] = hn;
            }
        }
    }
}

// ---- weight image packer: nn.LSTM parameters of one layer -> resident operand tiles + interleaved bias / W_ih^T ----
// tile (seg, plane): [256 rows n = 4*unit + gate][64 k] bf16, 128-byte swizzle; seg 0 = W_ih (layers > 0) or W_hh (layer 0),
// seg 1 = W_hh (layers > 0).  Native row of gate-interleaved column n: (n & 3) * 64 + (n >> 2)  (gate order i, f, g, o).
__global__ void lstm16_pack_kernel(const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                                   const float* __restrict__ b_ih, const float* __restrict__ b_hh, int layer, int c_in,
                                   uint8_t* __restrict__ wimg, float* __restrict__ bias, float* __restrict__ wih_t) {
    const int nseg = layer == 0 ? 1 : 2;
    const int total = nseg * kGateCols * kHid;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
        const int s = e / (kGateCols * kHid), n = (e / kHid) % kGateCols, k = e % kHid;
        const int nat = (n & 3) * kHid + (n >> 2);
        const float* src = (layer > 0 && s == 0) ? w_ih : w_hh;
        const float v = src[(int64_t)nat * kHid + k];
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        const __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
        const uint32_t off = sw128_off16((uint32_t)n, (uint32_t)k);
        *reinterpret_cast<__nv_bfloat16*>(wimg + (size_t)(s * 2) * kWTileBytes + off) = h;
        *reinterpret_cast<__nv_bfloat16*>(wimg + (size_t)(s * 2 + 1) * kWTileBytes + off) = l;
    }
    for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < kGateCols; n += gridDim.x * blockDim.x) {
        const int nat = (n & 3) * kHid + (n >> 2);
        bias[n] = b_ih[nat] + b_hh[nat];
        if (layer == 0 && wih_t != nullptr)
            for (int c = 0; c < c_in; ++c) wih_t[c * kGateCols + n] = w_ih[(int64_t)nat * c_in + c];
    }
}


// =====================================================================================================
// backward: gate recompute + BPTT pointwise + data gradient + weight gradient in ONE kernel, time-fused per layer
// (a launch = one layer x a run of timesteps, see Bwd16Params; "item" below = one (step, tile) work item)
// =====================================================================================================
// CTA = two consumer warpgroups (warpgroup w: rows 64w .. 64w+63 of a tile) + one producer warp.  The layer's weight image
// stays resident in shared memory; the producer streams the A planes ([h_below | h_prev], hi and lo) of each item with
// TMA.  Per item the 256 gate columns are processed as four chunks of 64 (16 units x i,f,g,o):
//   R_c : recompute  G_c[64 x 64] = [h_below | h_prev] . Wp[:, chunk]                      (registers, m64n64)
//   P_c : gates -> c_t, tanh(c_t) -> BPTT pointwise -> dA_c (fp32) -> bf16 hi/lo planes in a 128-byte-swizzled
//         shared-memory tile; dc in place
//   W_c : weight gradient  dWp[kd, chunk] = A^T . dA_c, warpgroup w: kd rows 64w .. (both operands: MN-major views of
//         tiles already in shared memory), added into this CTA's own slice of a scratch buffer with vector reductions
//   B_c : bias gradient    db[chunk] += ones . dA_c (warpgroup 0, A = a register fragment of ones), summed in shared memory
//   D_c : data gradient    [dx_below | dh_prev] += dA_c . Wp[:, chunk]^T  (B: MN-major view of the resident weights;
//         accumulated in registers over the four chunks, stored at the end of the item)
// dA never leaves the SM; the gates are never stored.  stmgcn_lstm16_wgrad_reduce sums the slices once per layer and
// writes nn.LSTM-native gradients.
constexpr int kBWarpgroups = 2;
constexpr int kBThreads = kBWarpgroups * 128 + 32;      // + producer warp
constexpr int kBATiles = 4;                             // (seg0 | seg1) x (hi | lo); layer 0: seg 1 = the auxiliary [x*s] tile

struct B16Tail {
    float db[kGateCols];
    uint64_t a_full, a_empty, w_full;
};
constexpr size_t kBSmem = 1024 + 4 * (size_t)kWTileBytes + kBATiles * (size_t)kATileBytes + 2 * (size_t)kATileBytes + sizeof(B16Tail);
static_assert(kBSmem <= 232448, "lstm16 backward kernel exceeds the 227 KB shared-memory limit");

// One launch = one LAYER, a run of timesteps from T-1 down (the tiles of a CTA are its own through time: rows never mix).
// A step of a tile needs what the SAME CTA produced for that tile one step later (dh_rec, dc: global, in place), so nothing
// but the launch order of the layers (top down) synchronises.
constexpr int kBMaxSteps = 64;
struct Bwd16Step {
    int32_t slice[2];          // plane slice of K segment s in its tensor map (hi plane; lo = + 1)
    int8_t src[2];             // 0: maps[0] (hp), 1: maps[1] (h0p), 2: zeros (h_prev at t = 0 without an initial state)
    int8_t first;              // t == T-1: incoming dh_rec / dc are zero and not read
    int8_t store_dh;           // write dh_prev (t > 0 or an initial state exists)
    int32_t t;
    const float* c_prev;       // blocked or nullptr (zeros)
    const float* dh_in;        // blocked or nullptr: gradient from the layer above at this step (top layer: d_top at T-1)
    float* dx_out;             // blocked or nullptr (layer 0)
};
struct Bwd16Params {
    alignas(64) CUtensorMap maps[2];
    const uint8_t* zero_tile;  // 16 KB of zeros
    const uint8_t* wimg;
    const float* bias;
    const float* wih;          // layer 0: (C,256) gate-interleaved
    const float* xo;           // (rows, T, C)
    const float* sg;           // (B, T)
    float* d_s;                // (B, T) +=   (layer 0)
    int c_in, t_len, n_steps;
    int64_t b_inner;
    float* dh_rec;             // blocked, in (unless first) / out, in place through the steps
    float* dc;                 // blocked, in (unless first) / out, in place through the steps
    float* dbp;                // (256) +=  gate-interleaved bias gradient
    float* dw_slice;           // gridDim.x slices of 128 x 256 floats (row-major [kd][gate column]), +=
    int64_t rows;
    int n_tiles;
    Bwd16Step steps[kBMaxSteps];   // in execution order: steps[0] is t = T-1
};
static_assert(sizeof(Bwd16Params) <= 4096, "kernel parameter block exceeds 4 KB");

__device__ __forceinline__ void cons_sync(int n_threads) { asm volatile("bar.sync 1, %0;" ::"r"(n_threads) : "memory"); }

template <int PLANES, int CIN>                                  // CIN: see lstm16_fwd_kernel
__global__ void __launch_bounds__(kBThreads, 1) lstm16_bwd_kernel(const __grid_constant__ Bwd16Params p) {
    constexpr bool L0 = CIN > 0;
    constexpr int kC = (CIN == 1) ? 1 : kMaxC;
    constexpr int kNseg = L0 ? 1 : 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* w_sm = smem;                                          // resident weights: tiles (seg*2 + plane) of 32 KB
    uint8_t* a_sm = w_sm + 4 * (size_t)kWTileBytes;                // A planes: tiles (seg*2 + plane) of 16 KB
    uint8_t* da_sm = a_sm + kBATiles * (size_t)kATileBytes;        // dA chunk: hi tile | lo tile
    B16Tail* tail = (B16Tail*)(da_sm + 2 * (size_t)kATileBytes);
    // layer 0 has one weight segment: the pre-scaled W_ih^T lives in the unused seg-1 weight slot
    float* wih_s = reinterpret_cast<float*>(w_sm + 2 * (size_t)kWTileBytes);
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    constexpr int kProdWarp = kBWarpgroups * 4;
    constexpr int kCons = kBWarpgroups * 128;

    if (tid == 0) {
        mbar_init(&tail->a_full, 1);
        mbar_init(&tail->a_empty, kBWarpgroups);
        mbar_init(&tail->w_full, 1);
        fence_barrier_init();
    }
    for (int i = tid; i < kGateCols; i += kBThreads) tail->db[i] = 0.f;
    if (L0) {
        for (int i = tid; i < p.c_in * kGateCols; i += kBThreads) wih_s[i] = p.wih[i] * gate_scale(i);
        // auxiliary tiles (seg-1 slots): zero once; columns 0..C-1 are rewritten per item
        for (int i = tid; i < 2 * kATileBytes / 16; i += kBThreads)
            reinterpret_cast<uint4*>(a_sm + 2 * (size_t)kATileBytes)[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    fence_proxy_async_smem();
    __syncthreads();
    const int my_tiles = (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int n_items = my_tiles * p.n_steps;                      // work items (step, tile), step-major

    if (warp == kProdWarp) {
        // ===================== producer =====================
        const bool leader = elect_one_sync();
        if (leader && n_items > 0) {
            mbar_arrive_expect_tx(&tail->w_full, (uint32_t)(kNseg * PLANES * kWTileBytes));
            for (int sg = 0; sg < kNseg; ++sg)
                for (int pl = 0; pl < PLANES; ++pl)
                    bulk_g2s(w_sm + (size_t)(sg * 2 + pl) * kWTileBytes, p.wimg + (size_t)(sg * 2 + pl) * kWTileBytes, kWTileBytes,
                             &tail->w_full);
            for (int w = 0; w < n_items; ++w) {
                const int st = w / my_tiles, tile = (int)blockIdx.x + (w - st * my_tiles) * (int)gridDim.x;
                const Bwd16Step& sp = p.steps[st];
                mbar_wait_p(&tail->a_empty, (uint32_t)(w & 1) ^ 1u, 0);
                mbar_arrive_expect_tx(&tail->a_full, (uint32_t)(kNseg * PLANES * kATileBytes));
                for (int sg = 0; sg < kNseg; ++sg)
                    for (int pl = 0; pl < PLANES; ++pl) {
                        uint8_t* dst = a_sm + (size_t)(sg * 2 + pl) * kATileBytes;
                        if (sp.src[sg] == 2) bulk_g2s(dst, p.zero_tile, kATileBytes, &tail->a_full);
                        else tma_load_3d(dst, &p.maps[sp.src[sg]], 0, tile * kTileM, sp.slice[sg] + pl, &tail->a_full);
                    }
                // the per-row inputs of this item -> L2 (a tile is one contiguous 32 KB run in every workspace)
                const int64_t o = (int64_t)tile * kTileM * kHid;
                constexpr uint32_t kB = kTileM * kHid * 4;
                if (sp.c_prev) prefetch_l2(sp.c_prev + o, kB);
                if (sp.dh_in) prefetch_l2(sp.dh_in + o, kB);
            }
        }
        return;
    }

    // ===================== consumers =====================
    const int wg = tid >> 7;
    const int q = lane & 3;
    const bool odd = (q & 1) != 0;
    const uint32_t rw0 = (uint32_t)(64 * wg + 16 * (warp & 3) + (lane >> 2));   // fragment row (and rw0 + 8)
    const uint32_t row_in_tile = rw0 + (odd ? 8u : 0u);                          // this thread's cell row
    const uint32_t rows32 = (uint32_t)p.rows;
    const uint32_t w_u = smem_u32(w_sm), a_u = smem_u32(a_sm), da_u = smem_u32(da_sm);
    const uint32_t a_rows = (uint32_t)wg * 64u * 128u;             // this warpgroup's rows inside a 128-row tile
    constexpr uint32_t kStepMN = 2048;                             // MN-major k16 step: 16 rows of 128 bytes
    // layer 0: when b_inner divides the tile height, a thread's row belongs to the same window b in every tile: its share of
    // d_s is summed in a register and added once per step
    const bool ds_fixed = L0 && (kTileM % (uint32_t)p.b_inner) == 0u;
    float ds_acc = 0.f;
    float* slice = p.dw_slice + (size_t)blockIdx.x * (kTileM * kGateCols);
    uint32_t ones[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) ones[k] = 0x3f803f80u;                // bf16 pair (1, 1)
    mbar_wait(&tail->w_full, 0, 0);

    for (int w = 0; w < n_items; ++w) {
        const int st = w / my_tiles, tile = (int)blockIdx.x + (w - st * my_tiles) * (int)gridDim.x;
        const Bwd16Step& sp = p.steps[st];
        const uint32_t r = (uint32_t)tile * kTileM + row_in_tile;
        const bool valid = r < rows32;
        const bool last_of_step = (w - st * my_tiles) == my_tiles - 1;
        float xs[kMaxC], xraw[kMaxC], dxs[kMaxC];
        if (L0) {
            const float sv = valid ? p.sg[(r % (uint32_t)p.b_inner) * (uint32_t)p.t_len + (uint32_t)sp.t] : 0.f;
#pragma unroll
            for (int c = 0; c < kMaxC; ++c) {
                xraw[c] = (c < kC && valid && (CIN == 1 || c < p.c_in)) ? p.xo[((int64_t)r * p.t_len + sp.t) * p.c_in + c] : 0.f;
                xs[c] = xraw[c] * sv;
                dxs[c] = 0.f;
            }
        }
        // the previous item's stores (dh_rec, dc of other threads' cells) and its reads of the shared tiles are complete
        cons_sync(kCons);
        if (L0 && (q >> 1) == 0) {
            // auxiliary weight-gradient operand (seg-1 slots): row = this thread's row, columns 0..C-1 = x*s (hi / lo split)
            uint32_t hi[2], lo[2];
            split_bf16x2(xs[0], xs[1], hi[0], lo[0]);
            split_bf16x2(xs[2], xs[3], hi[1], lo[1]);
            const uint32_t off = row_in_tile * 128u + ((0u ^ (row_in_tile & 7u)) << 4);
            *reinterpret_cast<uint2*>(a_sm + 2 * (size_t)kATileBytes + off) = make_uint2(hi[0], hi[1]);
            *reinterpret_cast<uint2*>(a_sm + 3 * (size_t)kATileBytes + off) = make_uint2(lo[0], lo[1]);
        }
        mbar_wait(&tail->a_full, (uint32_t)w & 1u, 1);
        float dacc[32 * kNseg];                                    // [dx_below | dh_prev] (layer 0: [dh_prev])
#pragma unroll
        for (int k = 0; k < 32 * kNseg; ++k) dacc[k] = 0.f;
        for (int c = 0; c < 4; ++c) {
            // ---- R_c ----
            float g[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) g[k] = 0.f;
            wg_fence_regs(g);
            wg_fence();
#pragma unroll
            for (int s = 0; s < kNseg; ++s) {
                const uint64_t a_hi = desc16_k(a_u + (uint32_t)(s * 2) * kATileBytes + a_rows);
                const uint64_t a_lo = desc16_k(a_u + (uint32_t)(s * 2 + 1) * kATileBytes + a_rows);
                const uint64_t b_hi = desc16_k(w_u + (uint32_t)(s * 2) * kWTileBytes + (uint32_t)c * 8192u);
                const uint64_t b_lo = desc16_k(w_u + (uint32_t)(s * 2 + 1) * kWTileBytes + (uint32_t)c * 8192u);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    wgmma_bf16_n64_t00(g, a_hi + 2 * kk, b_hi + 2 * kk, (s > 0 || kk > 0) ? 1u : 0u);
                    if (PLANES == 2) {
                        wgmma_bf16_n64_t00(g, a_hi + 2 * kk, b_lo + 2 * kk, 1u);
                        wgmma_bf16_n64_t00(g, a_lo + 2 * kk, b_hi + 2 * kk, 1u);
                    }
                }
            }
            wg_commit();
            wg_wait<0>();
            wg_fence_regs(g);
            // ---- P_c: 8 cells per thread (row row_in_tile, units 16c + 2j + q/2) ----
            uint32_t dhi[8], dlo[8];
            const uint32_t bo = (uint32_t)tile * 8192u + row_in_tile * 4u;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float s0 = odd ? g[4 * j + 0] : g[4 * j + 2];
                const float s1 = odd ? g[4 * j + 1] : g[4 * j + 3];
                const float o0 = __shfl_xor_sync(0xffffffffu, s0, 1);
                const float o1 = __shfl_xor_sync(0xffffffffu, s1, 1);
                const float vi = odd ? o0 : g[4 * j + 0], vf = odd ? o1 : g[4 * j + 1];
                const float vg = odd ? g[4 * j + 2] : o0, vo = odd ? g[4 * j + 3] : o1;
                const int unit = 16 * c + 2 * j + (q >> 1);
                const int col = 4 * unit;
                const float4 bv = *reinterpret_cast<const float4*>(p.bias + col);
                float pi = fmaf(vi, -1.4426950408889634f, bv.x * -1.4426950408889634f);
                float pf = fmaf(vf, -1.4426950408889634f, bv.y * -1.4426950408889634f);
                float pg = fmaf(vg, -2.8853900817779268f, bv.z * -2.8853900817779268f);
                float po = fmaf(vo, -1.4426950408889634f, bv.w * -1.4426950408889634f);
                if (L0) {
#pragma unroll
                    for (int cc = 0; cc < kC; ++cc)
                        if (CIN == 1 || cc < p.c_in) {
                            const float4 wv = *reinterpret_cast<const float4*>(&wih_s[cc * kGateCols + col]);
                            pi = fmaf(xs[cc], wv.x, pi); pf = fmaf(xs[cc], wv.y, pf);
                            pg = fmaf(xs[cc], wv.z, pg); po = fmaf(xs[cc], wv.w, po);
                        }
                }
                const uint32_t o = bo + (uint32_t)(unit >> 2) * 512u + (uint32_t)(unit & 3);
                float cp = 0.f, dh = 0.f, dci = 0.f;
                if (valid) {
                    if (sp.c_prev) cp = sp.c_prev[o];
                    if (sp.dh_in) dh = sp.dh_in[o];
                    if (!sp.first) {
                        dh += p.dh_rec[o];
                        dci = p.dc[o];
                    }
                }
                float gi, gf, gg, go, tc_;
                lstm_cell_gates8(pi, pf, pg, po, cp, gi, gf, gg, go, tc_);
                // rows past the end: dh = dci = 0, so dA = 0
                const float dcv = fmaf(dh * go, 1.f - tc_ * tc_, dci);
                const float da0 = dcv * gg * gi * (1.f - gi);
                const float da1 = dcv * cp * gf * (1.f - gf);
                const float da2 = dcv * gi * (1.f - gg * gg);
                const float da3 = dh * tc_ * go * (1.f - go);
                if (valid) p.dc[o] = dcv * gf;
                if (L0) {
#pragma unroll
                    for (int cc = 0; cc < kC; ++cc)
                        if (CIN == 1 || cc < p.c_in) {
                            // W_ih is stored pre-scaled: undo -log2(e) (and the g gate's extra factor 2)
                            const float4 wv = *reinterpret_cast<const float4*>(&wih_s[cc * kGateCols + col]);
                            dxs[cc] = fmaf(da0 * wv.x + da1 * wv.y + 0.5f * (da2 * wv.z) + da3 * wv.w, -0.6931471805599453f, dxs[cc]);
                        }
                }
                split_bf16x2(da0, da1, dhi[j], dlo[j]);
                uint32_t h2, l2;
                split_bf16x2(da2, da3, h2, l2);
                const uint32_t off = row_in_tile * 128u + ((((uint32_t)j) ^ (row_in_tile & 7u)) << 4) + (uint32_t)(q >> 1) * 8u;
                if (j == 0) cons_sync(kCons);                      // W / D / B of the previous chunk have read the dA tile
                *reinterpret_cast<uint2*>(da_sm + off) = make_uint2(dhi[j], h2);
                *reinterpret_cast<uint2*>(da_sm + kATileBytes + off) = make_uint2(dlo[j], l2);
            }
            fence_proxy_async_smem();
            cons_sync(kCons);                                      // the dA tile (both row halves) is complete
            // ---- W_c: dWp[kd rows 64 wg .., chunk] = A^T . dA_c ----
            float wgr[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) wgr[k] = 0.f;
            float bgr[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) bgr[k] = 0.f;
            wg_fence_regs(wgr);
            wg_fence_regs(bgr);
            wg_fence_regs(dacc);
            wg_fence();
            {
                const uint32_t wa_hi = a_u + (uint32_t)(wg * 2) * kATileBytes, wa_lo = wa_hi + kATileBytes;
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) {
                    const uint64_t ah = desc16_mn(wa_hi + ks * kStepMN, kATileBytes);
                    const uint64_t al = desc16_mn(wa_lo + ks * kStepMN, kATileBytes);
                    const uint64_t bh = desc16_mn(da_u + ks * kStepMN, kATileBytes);
                    const uint64_t bl = desc16_mn(da_u + kATileBytes + ks * kStepMN, kATileBytes);
                    // dA always has its lo plane; in the single-plane mode only the STORED operands are rounded to bf16
                    wgmma_bf16_n64_t11(wgr, ah, bh, ks > 0 ? 1u : 0u);
                    wgmma_bf16_n64_t11(wgr, ah, bl, 1u);
                    if (PLANES == 2) wgmma_bf16_n64_t11(wgr, al, bh, 1u);
                    // (both warpgroups issue it -- only warpgroup 0's result is used -- so that no wgmma sits on a
                    // warpgroup-dependent branch, which would make ptxas serialise every wgmma of the kernel)
                    wgmma_bf16_n64_rs_t1(bgr, ones, bh, ks > 0 ? 1u : 0u);
                    wgmma_bf16_n64_rs_t1(bgr, ones, bl, 1u);
                }
            }
            // ---- D_c: [dx_below | dh_prev] += dA_c . Wp[:, chunk]^T ----
            {
                const uint64_t ah = desc16_k(da_u + a_rows), al = desc16_k(da_u + kATileBytes + a_rows);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) {
                    const uint32_t wb = w_u + (uint32_t)c * 8192u + (uint32_t)kk * kStepMN;
                    const uint64_t bh = desc16_mn(wb, 2 * kWTileBytes), bl = desc16_mn(wb + kWTileBytes, 2 * kWTileBytes);
                    if constexpr (kNseg == 2) {
                        wgmma_bf16_n128_t01(dacc, ah + 2 * kk, bh, 1u);
                        if (PLANES == 2) wgmma_bf16_n128_t01(dacc, ah + 2 * kk, bl, 1u);
                        wgmma_bf16_n128_t01(dacc, al + 2 * kk, bh, 1u);
                    } else {
                        wgmma_bf16_n64_t01(dacc, ah + 2 * kk, bh, 1u);
                        if (PLANES == 2) wgmma_bf16_n64_t01(dacc, ah + 2 * kk, bl, 1u);
                        wgmma_bf16_n64_t01(dacc, al + 2 * kk, bh, 1u);
                    }
                }
            }
            wg_commit();
            wg_wait<0>();
            wg_fence_regs(wgr);
            wg_fence_regs(bgr);
            wg_fence_regs(dacc);
            // weight-gradient fragment -> this CTA's slice (row-major [kd][256]); bias sums: row 0 of warpgroup 0
            {
                const uint32_t m0 = rw0;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const uint32_t n = (uint32_t)(64 * c + 8 * j + 2 * q);
                    red_add_f32x2(slice + (size_t)m0 * kGateCols + n, wgr[4 * j], wgr[4 * j + 1]);
                    red_add_f32x2(slice + (size_t)(m0 + 8) * kGateCols + n, wgr[4 * j + 2], wgr[4 * j + 3]);
                }
                if (wg == 0 && m0 == 0) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        tail->db[64 * c + 8 * j + 2 * q] += bgr[4 * j];
                        tail->db[64 * c + 8 * j + 2 * q + 1] += bgr[4 * j + 1];
                    }
                }
            }
        }
        // the A planes of this item have been read by every MMA: one arrival per warpgroup
        asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
        if ((tid & 127) == 0) mbar_arrive(&tail->a_empty);
        // ---- [dx_below | dh_prev] fragment -> tile-blocked workspaces ----
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t rr = rw0 + 8u * h;
            if ((uint32_t)tile * kTileM + rr >= rows32) continue;
#pragma unroll
            for (int j = 0; j < 8 * kNseg; ++j) {
                const int col = 8 * j + 2 * q;
                // layers > 0: columns [0,64) = dx_below, [64,128) = dh_prev; layer 0: [0,64) = dh_prev
                const bool is_dx = !L0 && col < 64;
                float* base = is_dx ? sp.dx_out : p.dh_rec;
                if (base == nullptr || !(is_dx || sp.store_dh)) continue;
                const int unit = col & 63;
                *reinterpret_cast<float2*>(base + (uint32_t)tile * 8192u + (uint32_t)(unit >> 2) * 512u + rr * 4u + (uint32_t)(unit & 3)) =
                    make_float2(dacc[4 * j + 2 * h], dacc[4 * j + 2 * h + 1]);
            }
        }
        if (L0) {
            // gate adjoint: d s[b, t] += sum_c dxmod[r, c] * xo[r, t, c]   (STMGCN.py:44); this thread has half the row's units
            float contrib = 0.f;
#pragma unroll
            for (int cc = 0; cc < kC; ++cc) contrib += dxs[cc] * xraw[cc];
            contrib += __shfl_xor_sync(0xffffffffu, contrib, 2);
            if ((q >> 1) == 0 && valid) {
                if (ds_fixed) ds_acc += contrib;
                else atomicAdd(&p.d_s[(int64_t)(r % (uint32_t)p.b_inner) * p.t_len + sp.t], contrib);
            }
            if (ds_fixed && last_of_step) {
                if ((q >> 1) == 0 && ds_acc != 0.f)
                    atomicAdd(&p.d_s[(int64_t)(row_in_tile % (uint32_t)p.b_inner) * p.t_len + sp.t], ds_acc);
                ds_acc = 0.f;
            }
        }
    }
    cons_sync(kCons);
    for (int i = tid; i < kGateCols; i += kCons)
        if (n_items > 0) atomicAdd(&p.dbp[i], tail->db[i]);
}

// Sum the per-CTA weight-gradient slices of one layer and write nn.LSTM-native gradients:
//   d_w_ih (256, in), d_w_hh (256, 64), d_b_ih = d_b_hh (256); native row of gate-interleaved column n: (n & 3) * 64 + (n >> 2).
// Slice row m = kd index: layers > 0: m < 64 -> W_ih[:, m], m >= 64 -> W_hh[:, m - 64]; layer 0: m < 64 -> W_hh[:, m],
// m = 64 + c -> W_ih[:, c].
__global__ void lstm16_wgrad_reduce_kernel(const float* __restrict__ slices, int n_slices, int layer, int c_in,
                                           const float* __restrict__ dbp, float* __restrict__ d_w_ih,
                                           float* __restrict__ d_w_hh, float* __restrict__ d_b_ih, float* __restrict__ d_b_hh) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;           // index in the slice layout
    if (e < kTileM * kGateCols) {
        float s = 0.f;
        for (int i = 0; i < n_slices; ++i) s += slices[(size_t)i * (kTileM * kGateCols) + e];
        const int m = e / kGateCols, n = e % kGateCols;
        const int nat = (n & 3) * kHid + (n >> 2);
        if (layer > 0) {
            if (m < 64) d_w_ih[(size_t)nat * kHid + m] = s;
            else d_w_hh[(size_t)nat * kHid + (m - 64)] = s;
        } else {
            if (m < 64) d_w_hh[(size_t)nat * kHid + m] = s;
            else if (m - 64 < c_in) d_w_ih[(size_t)nat * c_in + (m - 64)] = s;
        }
    }
    if (e < kGateCols) {
        const int nat = (e & 3) * kHid + (e >> 2);
        d_b_ih[nat] = dbp[e];
        d_b_hh[nat] = dbp[e];
    }
}

}  // namespace

namespace stmgcn {

typedef CUresult (*EncodeTiledFn16)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn16 encode_fn16() {
    static EncodeTiledFn16 fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn16)sym;
    }
    return fn;
}
// (slices, rows, 64) bf16 plane tensor, box = 1 x 128 x 64, 128-byte swizzle (rows past the end read as zeros)
bool make_plane_map(CUtensorMap* map, const void* base, int64_t rows, int64_t slices) {
    EncodeTiledFn16 fn = encode_fn16();
    if (fn == nullptr) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)kHid, (cuuint64_t)rows, (cuuint64_t)slices};
    const cuuint64_t strides[2] = {(cuuint64_t)kHid * 2, (cuuint64_t)rows * kHid * 2};
    const cuuint32_t box[3] = {(cuuint32_t)kHid, (cuuint32_t)kTileM, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int32_t set_smem_attr(const void* fn, size_t bytes) { return ensure_dyn_smem(fn, bytes); }

// kernel variant for (planes, cin): cin = 0 (not layer 0), 1 (layer 0, one input channel), kMaxC (layer 0, runtime count)
using FwdFn = void (*)(const Fwd16Params);
using BwdFn = void (*)(const Bwd16Params);
static FwdFn fwd_kernel_for(int planes, int cin) {
    if (planes == 2) return cin == 0 ? lstm16_fwd_kernel<2, 0> : (cin == 1 ? lstm16_fwd_kernel<2, 1> : lstm16_fwd_kernel<2, kMaxC>);
    return cin == 0 ? lstm16_fwd_kernel<1, 0> : (cin == 1 ? lstm16_fwd_kernel<1, 1> : lstm16_fwd_kernel<1, kMaxC>);
}
static BwdFn bwd_kernel_for(int planes, int cin) {
    if (planes == 2) return cin == 0 ? lstm16_bwd_kernel<2, 0> : (cin == 1 ? lstm16_bwd_kernel<2, 1> : lstm16_bwd_kernel<2, kMaxC>);
    return cin == 0 ? lstm16_bwd_kernel<1, 0> : (cin == 1 ? lstm16_bwd_kernel<1, 1> : lstm16_bwd_kernel<1, kMaxC>);
}

}  // namespace stmgcn

extern "C" int32_t stmgcn_lstm16_pack(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                      int32_t layer, int32_t c_in, void* wimg, float* bias, float* wih_t, void* stream) {
    STMGCN_REQUIRE(w_ih && w_hh && b_ih && b_hh && wimg && bias, STMGCN_ERR_ARG, "lstm16_pack: null pointer");
    STMGCN_REQUIRE(layer >= 0 && c_in >= 1 && c_in <= kMaxC, STMGCN_ERR_SHAPE, "lstm16_pack: layer=%d c_in=%d", layer, c_in);
    STMGCN_REQUIRE(layer > 0 || wih_t != nullptr, STMGCN_ERR_ARG, "lstm16_pack: layer 0 needs wih_t");
    lstm16_pack_kernel<<<64, 256, 0, (cudaStream_t)stream>>>(w_ih, w_hh, b_ih, b_hh, layer, c_in, (uint8_t*)wimg, bias, wih_t);
    count_launch();
    return check_launch("lstm16_pack");
}

extern "C" int32_t stmgcn_lstm16_step_fwd(int32_t t, int32_t t_len, int32_t n_layers, int64_t rows, int32_t c_in,
                                          int64_t b_inner, int32_t planes, const float* xo, const float* s_gate,
                                          const void* const* wimg, const float* const* bias, const float* wih_t,
                                          const void* h0p, const float* c0, void* hp, float* cs, float* h_top,
                                          float* h_n, void* stream) {
    STMGCN_REQUIRE(xo && s_gate && wimg && bias && wih_t && hp && cs, STMGCN_ERR_ARG, "lstm16_step_fwd: null pointer");
    STMGCN_REQUIRE(planes == 1 || planes == 2, STMGCN_ERR_ARG, "lstm16_step_fwd: planes=%d", planes);
    STMGCN_REQUIRE(t >= 0 && t < t_len && n_layers >= 1 && n_layers <= 8 && rows > 0 && c_in >= 1 && c_in <= kMaxC && b_inner > 0,
                   STMGCN_ERR_SHAPE, "lstm16_step_fwd: t=%d T=%d L=%d rows=%lld C=%d", t, t_len, n_layers, (long long)rows, c_in);
    STMGCN_REQUIRE(rows <= (1LL << 25), STMGCN_ERR_SHAPE, "lstm16_step_fwd: rows=%lld too large (32-bit element offsets)", (long long)rows);
    STMGCN_REQUIRE((h0p == nullptr) == (c0 == nullptr), STMGCN_ERR_ARG, "lstm16_step_fwd: h0p and c0 go together");
    cudaStream_t st = (cudaStream_t)stream;
    const int n_tiles = (int)ceil_div(rows, kTileM);
    const int64_t rows_pad = (int64_t)n_tiles * kTileM;
    const int64_t plane_elems = rows * kHid;                       // bf16 elements per plane
    const int64_t cslice = rows_pad * kHid;
    const FwdFn fn0 = fwd_kernel_for(planes, c_in == 1 ? 1 : kMaxC), fn1 = fwd_kernel_for(planes, 0);
    if (int32_t rc = set_smem_attr((const void*)fn0, kFSmem)) return rc;
    if (int32_t rc = set_smem_attr((const void*)fn1, kFSmem)) return rc;
    CUtensorMap hp_map, h0_map;
    STMGCN_REQUIRE(make_plane_map(&hp_map, hp, rows, (int64_t)n_layers * t_len * planes), STMGCN_ERR_STATE,
                   "lstm16_step_fwd: cuTensorMapEncodeTiled failed (hp)");
    if (h0p != nullptr)
        STMGCN_REQUIRE(make_plane_map(&h0_map, h0p, rows, (int64_t)n_layers * planes), STMGCN_ERR_STATE,
                       "lstm16_step_fwd: cuTensorMapEncodeTiled failed (h0p)");
    const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
    for (int l = 0; l < n_layers; ++l) {
        STMGCN_REQUIRE(wimg[l] && bias[l], STMGCN_ERR_ARG, "lstm16_step_fwd: wimg/bias[%d] null", l);
        Fwd16Params p;
        memset(&p, 0, sizeof(p));
        int ns = 0;
        if (l > 0) {                                               // segment: h of the layer below at this step
            p.amap[ns] = hp_map;
            p.aslice[ns] = ((l - 1) * t_len + t) * planes;
            ++ns;
        }
        if (t > 0) {                                               // segment: this layer's h of the previous step
            p.amap[ns] = hp_map;
            p.aslice[ns] = (l * t_len + t - 1) * planes;
            ++ns;
        } else if (h0p != nullptr) {
            p.amap[ns] = h0_map;
            p.aslice[ns] = l * planes;
            ++ns;
        }
        p.nseg = ns;
        // the weight image holds [seg0 hi | seg0 lo | seg1 hi | seg1 lo]; at t = 0 without h0 the h_prev segment is absent:
        // layers > 0 then use only seg 0 (W_ih), layer 0 has no MMA at all
        p.wimg = (const uint8_t*)wimg[l];
        p.bias = bias[l];
        p.wih = (l == 0) ? wih_t : nullptr;
        p.xo = xo;
        p.sg = s_gate;
        p.c_in = c_in;
        p.t = t;
        p.t_len = t_len;
        p.b_inner = b_inner;
        p.c_prev = t > 0 ? cs + (int64_t)(l * t_len + t - 1) * cslice : (c0 ? c0 + (int64_t)l * cslice : nullptr);
        p.c_out = cs + (int64_t)(l * t_len + t) * cslice;
        uint16_t* hbase = (uint16_t*)hp + (int64_t)(l * t_len + t) * planes * plane_elems;
        p.h_hi = hbase;
        p.h_lo = planes == 2 ? hbase + plane_elems : nullptr;
        p.h_f32 = nullptr;
        if (t == t_len - 1) {
            if (h_n != nullptr) p.h_f32 = h_n + (int64_t)l * rows * kHid;
            else if (l == n_layers - 1) p.h_f32 = h_top;
        }
        p.rows = rows;
        p.n_tiles = n_tiles;
        (l == 0 ? fn0 : fn1)<<<grid, kFThreads, kFSmem, st>>>(p);
        count_launch();
        if (int32_t rc = check_launch("lstm16_fwd")) return rc;
    }
    return 0;
}

extern "C" int32_t stmgcn_lstm16_grid(int64_t rows) {
    const int64_t n_tiles = ceil_div(rows, kTileM);
    return (int32_t)(n_tiles < sm_count() ? n_tiles : sm_count());
}

extern "C" int32_t stmgcn_lstm16_layer_bwd(int32_t layer, int32_t t_len, int32_t n_layers, int64_t rows, int32_t c_in,
                                           int64_t b_inner, int32_t planes, const float* xo, const float* s_gate,
                                           const void* wimg, const float* bias, const float* wih_t, const void* h0p,
                                           const float* c0, const void* hp, const float* cs, const float* dh_in,
                                           float* dx_out, float* dh_rec, float* dc, float* d_s, float* dbp,
                                           float* dw_scratch, const void* zero_tile, void* stream) {
    STMGCN_REQUIRE(xo && s_gate && wimg && bias && hp && cs && dh_in && dh_rec && dc && d_s && dbp && dw_scratch && zero_tile,
                   STMGCN_ERR_ARG, "lstm16_layer_bwd: null pointer");
    STMGCN_REQUIRE(planes == 1 || planes == 2, STMGCN_ERR_ARG, "lstm16_layer_bwd: planes=%d", planes);
    STMGCN_REQUIRE(layer >= 0 && layer < n_layers && n_layers <= 8 && t_len >= 1 && t_len <= kBMaxSteps && rows > 0 && c_in >= 1 &&
                       c_in <= kMaxC && b_inner > 0,
                   STMGCN_ERR_SHAPE, "lstm16_layer_bwd: layer=%d L=%d T=%d (max %d) rows=%lld C=%d", layer, n_layers, t_len,
                   kBMaxSteps, (long long)rows, c_in);
    STMGCN_REQUIRE(rows <= (1LL << 25), STMGCN_ERR_SHAPE, "lstm16_layer_bwd: rows=%lld too large (32-bit element offsets)", (long long)rows);
    STMGCN_REQUIRE((h0p == nullptr) == (c0 == nullptr), STMGCN_ERR_ARG, "lstm16_layer_bwd: h0p and c0 go together");
    STMGCN_REQUIRE((layer == 0) == (dx_out == nullptr), STMGCN_ERR_ARG, "lstm16_layer_bwd: dx_out is for layers > 0 only");
    STMGCN_REQUIRE(layer > 0 || wih_t != nullptr, STMGCN_ERR_ARG, "lstm16_layer_bwd: wih_t null");
    cudaStream_t st = (cudaStream_t)stream;
    const int n_tiles = (int)ceil_div(rows, kTileM);
    const int64_t cslice = (int64_t)n_tiles * kTileM * kHid;
    const int l = layer;
    const BwdFn fn = bwd_kernel_for(planes, l == 0 ? (c_in == 1 ? 1 : kMaxC) : 0);
    if (int32_t rc = set_smem_attr((const void*)fn, kBSmem)) return rc;
    Bwd16Params p;
    memset(&p, 0, sizeof(p));
    STMGCN_REQUIRE(make_plane_map(&p.maps[0], hp, rows, (int64_t)n_layers * t_len * planes), STMGCN_ERR_STATE,
                   "lstm16_layer_bwd: cuTensorMapEncodeTiled failed (hp)");
    if (h0p != nullptr)
        STMGCN_REQUIRE(make_plane_map(&p.maps[1], h0p, rows, (int64_t)n_layers * planes), STMGCN_ERR_STATE,
                       "lstm16_layer_bwd: cuTensorMapEncodeTiled failed (h0p)");
    const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
    const bool top = (l == n_layers - 1);
    p.zero_tile = (const uint8_t*)zero_tile;
    p.wimg = (const uint8_t*)wimg;
    p.bias = bias;
    p.wih = (l == 0) ? wih_t : nullptr;
    p.xo = xo;
    p.sg = s_gate;
    p.d_s = d_s;
    p.c_in = c_in;
    p.t_len = t_len;
    p.b_inner = b_inner;
    p.dh_rec = dh_rec;
    p.dc = dc;
    p.dbp = dbp;
    p.dw_slice = dw_scratch;
    p.rows = rows;
    // every CTA adds into its own slice: start from zero
    STMGCN_CUDA(cudaMemsetAsync(dw_scratch, 0, (size_t)grid * kTileM * kGateCols * sizeof(float), st));
    p.n_tiles = n_tiles;
    // one launch covers all timesteps of the layer (t_len <= kBMaxSteps); the weight-gradient partials of every chunk are
    // added into fp32 memory, so the length of the run does not lengthen any tensor-core accumulation chain
    const int steps_per_launch = t_len;
    for (int s0 = 0; s0 < t_len; s0 += steps_per_launch) {
        const int ns_launch = (t_len - s0 < steps_per_launch) ? (t_len - s0) : steps_per_launch;
        p.n_steps = ns_launch;
        for (int sj = 0; sj < ns_launch; ++sj) {
            const int si = s0 + sj;
            const int t = t_len - 1 - si;
            Bwd16Step& sp = p.steps[sj];
            int ns = 0;
            if (l > 0) {                                               // K segment: h of the layer below at this step
                sp.src[ns] = 0;
                sp.slice[ns] = ((l - 1) * t_len + t) * planes;
                ++ns;
            }
            if (t > 0) {                                               // K segment: this layer's h of the previous step
                sp.src[ns] = 0;
                sp.slice[ns] = (l * t_len + t - 1) * planes;
            } else if (h0p != nullptr) {
                sp.src[ns] = 1;
                sp.slice[ns] = l * planes;
            } else {
                sp.src[ns] = 2;                                        // zeros (STMGCN.py:53-57)
                sp.slice[ns] = 0;
            }
            sp.t = t;
            sp.first = (t == t_len - 1) ? 1 : 0;
            sp.store_dh = (t > 0 || h0p != nullptr) ? 1 : 0;
            sp.c_prev = t > 0 ? cs + (int64_t)(l * t_len + t - 1) * cslice : (c0 ? c0 + (int64_t)l * cslice : nullptr);
            sp.dh_in = top ? (t == t_len - 1 ? dh_in : nullptr) : dh_in + (int64_t)t * cslice;
            sp.dx_out = l > 0 ? dx_out + (int64_t)t * cslice : nullptr;
        }
        fn<<<grid, kBThreads, kBSmem, st>>>(p);
        count_launch();
        if (int32_t rc = check_launch("lstm16_layer_bwd")) return rc;
    }
    return 0;
}

extern "C" int32_t stmgcn_lstm16_wgrad_reduce(int32_t layer, int32_t c_in, int32_t n_slices, const float* slices,
                                              const float* dbp, float* d_w_ih, float* d_w_hh, float* d_b_ih,
                                              float* d_b_hh, void* stream) {
    STMGCN_REQUIRE(slices && dbp && d_w_ih && d_w_hh && d_b_ih && d_b_hh, STMGCN_ERR_ARG, "lstm16_wgrad_reduce: null pointer");
    STMGCN_REQUIRE(layer >= 0 && n_slices >= 1 && c_in >= 1 && c_in <= kMaxC, STMGCN_ERR_SHAPE, "lstm16_wgrad_reduce: bad sizes");
    lstm16_wgrad_reduce_kernel<<<(kTileM * kGateCols) / 256, 256, 0, (cudaStream_t)stream>>>(slices, n_slices, layer, c_in, dbp,
                                                                                        d_w_ih, d_w_hh, d_b_ih, d_b_hh);
    count_launch();
    return check_launch("lstm16_wgrad_reduce");
}
