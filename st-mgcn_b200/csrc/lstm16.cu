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
// forward kernel (one launch per layer covering all T steps, persistent, one CTA per SM):
//   producer warp : loads the layer's weight image ONCE (resident for the whole launch: [256 gate cols][64 k] bf16 tiles,
//                   hi and lo, per K segment = 128 KB); layers > 0: streams h_below (hp of the layer below) of every
//                   (tile, step) into one stage per warpgroup with TMA tensor loads
//   2 warpgroups  : each walks its 64 rows of a tile through t = 0 .. T-1; per step 8 (P = 1) or 24 (P = 2) wgmma
//                   m64n256k16 into registers: Ahi.Whi + Ahi.Wlo + Alo.Whi, then bias (+ layer 0: x*s . W_ih in exact
//                   fp32) -> gates -> c, h -> h split into bf16 planes in shared memory, which is both the h_prev operand
//                   of the next step and the source of a TMA tensor store of the tape; c stays in shared memory too
//                   (and is stored to the cs tape).  Nothing of the gates leaves the SM.
#include "tc16.cuh"
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

using namespace stmgcn;
using namespace stmgcn::tc;

namespace {

constexpr int kTileM = 128;
constexpr int kHid = 64;
constexpr int kGateCols = 256;
constexpr int kMaxC = 4;
constexpr int kWTileBytes = kGateCols * 128;          // [256 gate cols][64 k] bf16 = 32 KB
constexpr int kATileBytes = kTile16Bytes;             // [128 rows][64 k] bf16 = 16 KB

// Tile-blocked (rows_pad x 64) fp32 workspaces (cs, c0, dh, dc, dx): [tile][unit / 4][128 rows][4 units], a tile one 32 KB
// run.  Offset of (row of tile, unit), and the size of a (layer, step) slice.  Host side: ops.to_blocked / from_blocked.
__host__ __device__ __forceinline__ uint32_t blocked_off(uint32_t tile, uint32_t row, uint32_t unit) {
    return tile * 8192u + (unit >> 2) * 512u + row * 4u + (unit & 3u);
}
__host__ __device__ __forceinline__ int64_t blocked_slice(int n_tiles) { return (int64_t)n_tiles * kTileM * kHid; }

// ---- LSTM cell with 8 MUFU operations instead of 10 ------------------------------------------------------------
// sigmoid(v) = 1 / (1 + e^-v), tanh(v) = (1 - e^-2v) / (1 + e^-2v).  Five exponentials per cell are unavoidable (i, f, g, o,
// tanh(c)); the five reciprocals are not: reciprocals of PRODUCTS of two (1 + e) terms serve two activations at once.
// The exponentials are capped at e^30 (the capped activations differ from the exact ones by < 1e-13) so that a
// product of two (1 + e^30) terms stays far below the fp32 overflow threshold.  The cell epilogue is MUFU-bound
// (16 MUFU results per clock and SM), so this is 20 % off its critical resource.
// (one-sided: only a large NEGATIVE argument makes e^-v large; for large positive v the exponential underflows to 0, which is exact)
// The kernels keep bias and W_ih PRE-SCALED by the exponent factor of their gate (gate_scale: kNegLog2e for i, f, o and
// kNeg2Log2e for g), so "accumulator + bias, times -log2(e)" is ONE fma per gate: arg = fma(acc, scale, bias_scaled).
__device__ __forceinline__ float gate_scale(int col) { return (col & 3) == 2 ? kNeg2Log2e : kNegLog2e; }
// min.NaN keeps a NaN argument (fminf(NaN, c) would return the cap, a saturated gate), so a NaN gate stays NaN.
__device__ __forceinline__ float exp_arg_(float a) {                                          // e^(-v) or e^(-2v), <= e^30
    float m;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(m) : "f"(a), "f"(43.28f));
    return ex2_ftz_(m);
}
// forward: exponent arguments of (i, f, g, o) and c_{t-1} -> c_t, h_t
__device__ __forceinline__ void lstm_cell_fwd8(float ai, float af, float ag, float ao, float cp, float& c, float& h) {
    const float ei = exp_arg_(ai), ef = exp_arg_(af), eg = exp_arg_(ag), eo = exp_arg_(ao);
    const float ig = (1.f - eg) * rcp_ftz_((1.f + ei) * (1.f + eg));          // sigmoid(pi) * tanh(pg)
    c = fmaf(rcp_ftz_(1.f + ef), cp, ig);
    const float ec = exp_arg_(kNeg2Log2e * c);
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
    const float ec = exp_arg_(kNeg2Log2e * fmaf(gf, cp, gi * gg));
    tc = (1.f - ec) * rcp_ftz_(1.f + ec);
}

// ---- pieces of the cell epilogue shared by the forward and the backward kernel ----------------------------------
// Accumulator values d[4j .. 4j+3] (gate-interleaved columns, see the forward kernel) -> pre-activations (i, f, g, o) of
// this thread's cell: partner lanes (lane ^ 1) swap one row's pair.
template <int R>
__device__ __forceinline__ float4 frag_to_gates(const float (&d)[R], int j, bool odd) {
    const float s0 = odd ? d[4 * j + 0] : d[4 * j + 2];
    const float s1 = odd ? d[4 * j + 1] : d[4 * j + 3];
    const float o0 = __shfl_xor_sync(0xffffffffu, s0, 1);
    const float o1 = __shfl_xor_sync(0xffffffffu, s1, 1);
    return make_float4(odd ? o0 : d[4 * j + 0], odd ? o1 : d[4 * j + 1], odd ? d[4 * j + 2] : o0, odd ? d[4 * j + 3] : o1);
}
// exponent arguments of (i, f, g, o): pre-activation times the gate's exponent factor plus the scaled bias b, and on
// layer 0 plus x*s . W_ih (wih: the scaled, gate-interleaved (C, 256) W_ih^T in shared memory)
template <int CIN>
__device__ __forceinline__ float4 gate_args(float4 v, float4 b, const float (&xs)[kMaxC], const float* wih, int col, int c_in) {
    constexpr int kC = (CIN == 1) ? 1 : kMaxC;
    float4 a = make_float4(fmaf(v.x, kNegLog2e, b.x), fmaf(v.y, kNegLog2e, b.y), fmaf(v.z, kNeg2Log2e, b.z),
                           fmaf(v.w, kNegLog2e, b.w));
    if (CIN > 0) {
#pragma unroll
        for (int c = 0; c < kC; ++c)
            if (CIN == 1 || c < c_in) {
                const float4 wv = *reinterpret_cast<const float4*>(&wih[c * kGateCols + col]);
                a.x = fmaf(xs[c], wv.x, a.x); a.y = fmaf(xs[c], wv.y, a.y);
                a.z = fmaf(xs[c], wv.z, a.z); a.w = fmaf(xs[c], wv.w, a.w);
            }
    }
    return a;
}

// producer: the layer's resident weight image p.wimg (tiles seg * 2 + plane of kWTileBytes) -> shared memory, on bar
template <int NSEG, int PLANES, class Params>
__device__ __forceinline__ void load_weights(uint8_t* w_sm, const Params& p, uint64_t* bar) {
    mbar_arrive_expect_tx(bar, (uint32_t)(NSEG * PLANES * kWTileBytes));
    for (int s = 0; s < NSEG; ++s)
        for (int pl = 0; pl < PLANES; ++pl)
            bulk_g2s(w_sm + (size_t)(s * 2 + pl) * kWTileBytes, p.wimg + (size_t)(s * 2 + pl) * kWTileBytes, kWTileBytes, bar);
}

// =====================================================================================================
// forward: one launch per LAYER over all its timesteps (a tile's rows never mix with other tiles', so a CTA walks its
// own tiles through time, as the backward does)
// =====================================================================================================
// CTA = two consumer warpgroups + one producer warp, persistent over 128-row tiles.  Warpgroup w owns rows 64w .. 64w+63
// of a tile, walks them through t = 0 .. T-1 and accumulates their [64 x 256] gate pre-activations in registers (wgmma
// m64n256k16).  The warpgroups share nothing but the resident weights, so they run out of phase: one's wgmma overlaps
// the other's MUFU-bound cell epilogue.
//   h_prev : never leaves the SM.  The epilogue of step t writes h_t as bf16 planes into the warpgroup's own [64][64]
//            128-byte-swizzled tiles (one per plane): the K-major A operand of step t + 1, and the source of the TMA
//            tensor store of hp[l, t].  At t = 0 the tiles are loaded from h0p, or the segment is absent (zeros).
//   h_below: layers > 0: hp[l - 1, t], written by the previous launch, streamed by the producer into one stage per
//            warpgroup; released as soon as the step's wgmma have completed, so the next load overlaps the epilogue.
//   c      : never read back from global memory.  c_{t-1} of a cell is private to the thread that computes c_t, so each
//            warpgroup keeps its rows' c in a private fp32 tile in shared memory (filled from c0, or zeros, at the start
//            of a tile); c_t goes to it and, fire-and-forget, to the tile-blocked cs tape for the backward.  (Read back
//            from the tape, every cell waited one L2 round trip: the load cannot pass the previous cell's tape store.)
// Accumulator fragment (wgmma.cuh): thread holds columns 8j + 2(lane%4) + {0,1} of rows r0 and r0 + 8; with
// gate-interleaved columns n = 4 unit + gate that is gates (i, f) (lane%4 even) or (g, o) (odd) of unit 2j + (lane%4)/2.
// Partner lanes (lane ^ 1) swap one row's pair, after which the even lane owns the cell (r0, unit) and the odd lane the
// cell (r0 + 8, unit).
constexpr int kFWarpgroups = 2;
constexpr int kFThreads = kFWarpgroups * 128 + 32;     // + producer warp
constexpr uint32_t kFBarWg = 1;                        // named barrier kFBarWg + w: warpgroup w (128 threads)
constexpr int kHTileBytes = 64 * 128;                  // one plane of a warpgroup's rows: [64 rows][64] bf16 = 8 KB
constexpr int kFWgBytes = 4 * kHTileBytes;             // per warpgroup: h_prev hi | lo, h_below stage hi | lo
constexpr int kFCBytes = 64 * kHid * 4;                // per warpgroup: fp32 c of its rows, [32 cells j][128 threads]
constexpr int kFCellBatch = 8;                         // cells per batch of the cell epilogue (of a thread's 32)

struct F16Tail {
    float bias[kGateCols];
    uint64_t full[kFWarpgroups];       // h_below stage of warpgroup w loaded
    uint64_t empty[kFWarpgroups];      // ... and consumed
    uint64_t h0_full[kFWarpgroups];    // h_prev tiles of warpgroup w loaded from h0p
    uint64_t w_full;
};
constexpr size_t kFSmem =
    1024 + 4 * (size_t)kWTileBytes + kFWarpgroups * ((size_t)kFWgBytes + kFCBytes) + sizeof(F16Tail);
static_assert(kFSmem <= 232448, "lstm16 forward kernel exceeds the 227 KB shared-memory limit");

struct Fwd16Params {
    alignas(64) CUtensorMap hp_map;    // (64, rows, L*T*P) bf16 view of hp, box 64 x 64 x 1, 128B swizzle
    alignas(64) CUtensorMap h0_map;    // (64, rows, L*P) view of h0p, same box (has_h0)
    const uint8_t* wimg;               // this layer's tiles [(seg*2 + plane)] of 32 KB
    const float* bias;                 // (256) gate-interleaved b_ih + b_hh
    const float* wih;                  // layer 0: (C, 256) gate-interleaved W_ih^T; else nullptr
    const float* xo;                   // (rows, T, C)
    const float* sg;                   // (B, T)
    int layer, c_in, t_len;
    int has_h0;                        // h0_map and c0 are set
    int64_t b_inner;
    const float* c0;                   // this layer's initial cell state, tile-blocked, or nullptr (zeros)
    float* cs;                         // this layer's cell-state tape (T, rows_pad, 64), tile-blocked
    float* h_f32;                      // (rows, 64) fp32 copy of h at t = T-1, or nullptr
    int64_t rows;
    int n_tiles;
};

// One K segment of the gate GEMM: A = the PLANES [64][64] tiles at a_u (hi | lo, kHTileBytes apart), W = the segment's
// resident [256][64] tiles at w_u (hi | lo).  Issue order per plane: hi: Ahi.Whi, Ahi.Wlo per k-step; lo: Alo.Whi.
template <int PLANES>
__device__ __forceinline__ void fwd_segment_mma(float (&acc)[128], uint32_t a_u, uint32_t w_u, bool first) {
    const uint64_t w_hi = desc16_k(w_u), w_lo = desc16_k(w_u + kWTileBytes);
#pragma unroll
    for (int pl = 0; pl < PLANES; ++pl) {
        const uint64_t a_d = desc16_k(a_u + (uint32_t)pl * kHTileBytes);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            wgmma_bf16_n256_t00(acc, a_d + (uint64_t)(2 * kk), w_hi + (uint64_t)(2 * kk), (!first || pl > 0 || kk > 0) ? 1u : 0u);
            if (PLANES == 2 && pl == 0) wgmma_bf16_n256_t00(acc, a_d + (uint64_t)(2 * kk), w_lo + (uint64_t)(2 * kk), 1u);
        }
    }
}

// CIN: 0 = not layer 0; 1 = layer 0 with one input channel (the reference's input_dim, compile-time: no predicated-off
// W_ih FMAs / loads in the cell loop); kMaxC = layer 0 with a runtime channel count <= kMaxC
template <int PLANES, int CIN>
__global__ void __launch_bounds__(kFThreads, 1) lstm16_fwd_kernel(const __grid_constant__ Fwd16Params p) {
    constexpr bool L0 = CIN > 0;
    constexpr int kC = (CIN == 1) ? 1 : kMaxC;
    constexpr int kNseg = L0 ? 1 : 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
    uint8_t* wsm = smem;                                           // resident weight tiles (seg*2 + plane)
    uint8_t* hsm = smem + 4 * (size_t)kWTileBytes;                 // per warpgroup: kFWgBytes
    uint8_t* csm = hsm + kFWarpgroups * (size_t)kFWgBytes;         // per warpgroup: kFCBytes
    F16Tail* tail = (F16Tail*)(csm + kFWarpgroups * (size_t)kFCBytes);
    // layer 0 has one weight segment: the pre-scaled W_ih^T lives in the unused seg-1 weight slot
    float* wih_s = reinterpret_cast<float*>(wsm + 2 * (size_t)kWTileBytes);
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    constexpr int kProdWarp = kFWarpgroups * 4;

    if (tid == 0) {
        for (int w = 0; w < kFWarpgroups; ++w) {
            mbar_init(&tail->full[w], 1);
            mbar_init(&tail->empty[w], 1);
            mbar_init(&tail->h0_full[w], 1);
        }
        mbar_init(&tail->w_full, 1);
        fence_barrier_init();
    }
    for (int i = tid; i < kGateCols; i += kFThreads) tail->bias[i] = p.bias[i] * gate_scale(i);
    // rows c_in .. kC-1 of W_ih^T are zeros, so that the cells add all kC channels without a predicate per channel
    // (x * s of those channels is zero too; the extra fma(0, 0, a) turns at most a -0 into +0, and ex2 of either is 1)
    if (L0)
        for (int i = tid; i < kC * kGateCols; i += kFThreads) wih_s[i] = i < p.c_in * kGateCols ? p.wih[i] * gate_scale(i) : 0.f;
    __syncthreads();
    const int my_tiles = cta_tiles(p.n_tiles);

    if (warp == kProdWarp) {
        // ===================== producer: resident weights once, then h_below of every (tile, step) =====================
        const bool leader = elect_one_sync();
        if (leader && my_tiles > 0) {
            load_weights<kNseg, PLANES>(wsm, p, &tail->w_full);
            if (!L0) {
                // the warpgroups drift apart: serve whichever has released its stage instead of alternating
                const int n_loads = my_tiles * p.t_len;
                int done[kFWarpgroups] = {0, 0};
                uint32_t idle = 0;
                while (done[0] < n_loads || done[1] < n_loads) {
                    bool issued = false;
#pragma unroll
                    for (int w = 0; w < kFWarpgroups; ++w) {
                        const int n = done[w];
                        if (n < n_loads && mbar_try_wait(&tail->empty[w], (uint32_t)(n & 1) ^ 1u)) {
                            const int i = n / p.t_len, t = n - i * p.t_len;
                            const int row0 = cta_tile(i) * kTileM + 64 * w;
                            uint8_t* stage = hsm + (size_t)w * kFWgBytes + 2 * (size_t)kHTileBytes;
                            mbar_arrive_expect_tx(&tail->full[w], (uint32_t)(PLANES * kHTileBytes));
                            for (int pl = 0; pl < PLANES; ++pl)
                                tma_load_3d(stage + (size_t)pl * kHTileBytes, &p.hp_map, 0, row0,
                                            ((p.layer - 1) * p.t_len + t) * PLANES + pl, &tail->full[w]);
                            done[w] = n + 1;
                            issued = true;
                        }
                    }
                    if (issued) {
                        idle = 0;
                    } else {
                        if (++idle == (1u << 28)) __trap();            // ~20 s without progress: a protocol bug
                        __nanosleep(40);
                    }
                }
            }
        }
        return;
    }
    // ===================== consumers: gate GEMM (wgmma) + LSTM cell, step after step =====================
    const int wg = tid >> 7;
    const int q = lane & 3;
    const bool odd = (q & 1) != 0;
    const bool issuer = (tid & 127) == 0;                          // the warpgroup's TMA / mbarrier thread
    const uint32_t row_in_wg = (uint32_t)(16 * (warp & 3) + (lane >> 2) + (odd ? 8 : 0));
    const uint32_t row_in_tile = 64u * (uint32_t)wg + row_in_wg;
    const uint32_t rows32 = (uint32_t)p.rows;
    uint8_t* h_sm = hsm + (size_t)wg * kFWgBytes;                  // h_prev: hi | lo
    // c of this thread's 32 cells: element 128 j (thread-major: conflict free; only the owning thread touches it)
    float* c_sm = reinterpret_cast<float*>(csm + (size_t)wg * kFCBytes) + (tid & 127);
    const uint32_t w_u = smem_u32(wsm), h_u = smem_u32(h_sm), b_u = h_u + 2u * kHTileBytes;
    const int64_t cslice = blocked_slice(p.n_tiles);
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    mbar_wait_raw(&tail->w_full, 0);
    uint32_t n_below = 0;                                          // h_below stages consumed
    for (int i = 0; i < my_tiles; ++i) {
        const int tile = cta_tile(i);
        const int row0 = tile * kTileM + 64 * wg;                  // first row of this warpgroup
        const uint32_t r = (uint32_t)tile * kTileM + row_in_tile;
        const bool valid = r < rows32;
        const uint32_t cbase = blocked_off(tile, row_in_tile, 0);    // this thread's row; unit u is + blocked_off(0, 0, u)
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const int unit = 2 * j + (q >> 1);
            c_sm[128 * j] = (p.c0 != nullptr && valid) ? p.c0[cbase + blocked_off(0, 0, unit)] : 0.f;
        }
        if (p.has_h0) {
            if (issuer) {
                bulk_wait_group_read0();                           // the previous tile's last store has read the tiles
                mbar_arrive_expect_tx(&tail->h0_full[wg], (uint32_t)(PLANES * kHTileBytes));
                for (int pl = 0; pl < PLANES; ++pl)
                    tma_load_3d(h_sm + (size_t)pl * kHTileBytes, &p.h0_map, 0, row0, p.layer * PLANES + pl, &tail->h0_full[wg]);
            }
            mbar_wait_raw(&tail->h0_full[wg], (uint32_t)i & 1u);
        }
        for (int t = 0; t < p.t_len; ++t) {
            // layer 0: x * s of this thread's row (loaded before the MMAs: the latency hides behind them)
            float xs[kMaxC];
            if (L0) {
                const float sv = valid ? p.sg[(r % (uint32_t)p.b_inner) * (uint32_t)p.t_len + (uint32_t)t] : 0.f;
#pragma unroll
                for (int c = 0; c < kMaxC; ++c)
                    xs[c] = (c < kC && valid && (CIN == 1 || c < p.c_in)) ? p.xo[((int64_t)r * p.t_len + t) * p.c_in + c] * sv : 0.f;
            }
            // K segments: h_below (layers > 0), then h_prev (absent at t = 0 without an initial state)
            // (each branch a complete fence .. wait sequence: a segment count known only at run time makes ptxas
            // serialise every wgmma of the kernel)
            const int nseg = (L0 ? 0 : 1) + ((t > 0 || p.has_h0) ? 1 : 0);
            if (nseg > 0) {
                wg_fence_regs(acc);
                if (!L0) mbar_wait_raw(&tail->full[wg], n_below & 1u);
                if (!L0 && nseg == 2) {
                    wg_fence();
                    fwd_segment_mma<PLANES>(acc, b_u, w_u, true);
                    fwd_segment_mma<PLANES>(acc, h_u, w_u + 2u * kWTileBytes, false);
                    wg_commit();
                    wg_wait<0>();
                } else {
                    wg_fence();
                    fwd_segment_mma<PLANES>(acc, L0 ? h_u : b_u, w_u, true);
                    wg_commit();
                    wg_wait<0>();
                }
                wg_fence_regs(acc);
            } else {
#pragma unroll
                for (int k = 0; k < 128; ++k) acc[k] = 0.f;
            }
            // every warp's wgmma have read the operands, and the store of h_{t-1} has read the h_prev tiles: the stage
            // goes back to the producer, and the tiles may be overwritten
            if (issuer) bulk_wait_group_read0();
            bar_sync(kFBarWg + wg, 128);
            if (!L0) {
                if (issuer) mbar_arrive(&tail->empty[wg]);
                ++n_below;
            }
            // ---- LSTM cell: 32 cells per thread, row row_in_tile, units 2j + q/2 ----
            // In batches of kFCellBatch independent cells: the batch's shuffles, then its shared-memory loads, then the
            // cells' arithmetic, then its stores.  A cell's loads cannot pass an earlier cell's stores (they may alias,
            // as far as the compiler knows), so cells written one after another run their MUFU chains strictly in
            // sequence, with nothing to hide the latency.  The stores are predicated: a branch around a cell's stores
            // is a scheduling barrier as well.
            // c_row / h_row: this thread's row of the cs slice and of h_f32; cell j sits at a constant offset from it
            float* c_row = p.cs + (int64_t)t * cslice + cbase + blocked_off(0, 0, q >> 1);
            const bool store_h = valid && t == p.t_len - 1 && p.h_f32 != nullptr;    // h_f32 only at t = T-1
            float* h_row = p.h_f32 + (store_h ? r * (uint32_t)kHid + (uint32_t)(q >> 1) : 0u);
#pragma unroll
            for (int j0 = 0; j0 < 32; j0 += kFCellBatch) {
                float4 v[kFCellBatch], bv[kFCellBatch];
                float cp[kFCellBatch], cn[kFCellBatch], hn[kFCellBatch];
#pragma unroll
                for (int k = 0; k < kFCellBatch; ++k) v[k] = frag_to_gates(acc, j0 + k, odd);
#pragma unroll
                for (int k = 0; k < kFCellBatch; ++k) {
                    const int col = 4 * (2 * (j0 + k) + (q >> 1));
                    bv[k] = *reinterpret_cast<const float4*>(&tail->bias[col]);         // pre-scaled (gate_scale)
                    cp[k] = c_sm[128 * (j0 + k)];
                }
#pragma unroll
                for (int k = 0; k < kFCellBatch; ++k) {
                    const int col = 4 * (2 * (j0 + k) + (q >> 1));
                    const float4 a = gate_args<CIN>(v[k], bv[k], xs, wih_s, col, kC);
                    lstm_cell_fwd8(a.x, a.y, a.z, a.w, cp[k], cn[k], hn[k]);
                }
#pragma unroll
                for (int k = 0; k < kFCellBatch; ++k) {
                    const int unit = 2 * (j0 + k) + (q >> 1);
                    c_sm[128 * (j0 + k)] = cn[k];
                    if (valid) c_row[blocked_off(0, 0, 2 * (j0 + k))] = cn[k];
                    if (store_h) h_row[2 * (j0 + k)] = hn[k];
                    // rows past the end are computed too (a row's gates depend on that row alone) and dropped by the store
                    const uint32_t off = sw128<2>(row_in_wg, (uint32_t)unit);
                    const __nv_bfloat16 hb = __float2bfloat16_rn(hn[k]);
                    *reinterpret_cast<__nv_bfloat16*>(h_sm + off) = hb;
                    if (PLANES == 2) *reinterpret_cast<__nv_bfloat16*>(h_sm + kHTileBytes + off) = __float2bfloat16_rn(hn[k] - __bfloat162float(hb));
                }
            }
            // h_t -> the async proxy (the store below, the next step's wgmma)
            fence_proxy_async_smem();
            bar_sync(kFBarWg + wg, 128);
            if (issuer) {
                for (int pl = 0; pl < PLANES; ++pl)
                    tma_store_3d(&p.hp_map, h_sm + (size_t)pl * kHTileBytes, 0, row0, (p.layer * p.t_len + t) * PLANES + pl);
                bulk_commit_group();
            }
        }
    }
    if (issuer) bulk_wait_group_read0();                           // shared memory outlives the stores' reads
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
        const uint32_t off = sw128<2>((uint32_t)n, (uint32_t)k);
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
// (a launch = one layer x all its timesteps, see Bwd16Params; "item" below = one (step, tile) work item)
// =====================================================================================================
// CTA = two consumer warpgroups (warpgroup w: rows 64w .. 64w+63 of a tile) + one producer warpgroup, warp-specialised:
// the producer drops to kBProdRegs registers so that the consumers can hold the accumulators of two chunks at once.
// The layer's weight image stays resident in shared memory; one producer thread streams the A planes ([h_below |
// h_prev], hi and lo) of each item with TMA and prefetches the next item's into L2.  Per item the 256 gate columns are
// processed as four chunks of 64 (16 units x i,f,g,o):
//   R_c : recompute  G_c[64 x 64] = [h_below | h_prev] . Wp[:, chunk]                      (registers, m64n64)
//   P_c : gates -> c_t, tanh(c_t) -> BPTT pointwise -> dA_c (fp32) -> bf16 hi/lo planes in a 128-byte-swizzled
//         shared-memory tile; dc in place
//   B_c : bias gradient    db[chunk] += column sums of dA_c = hi + lo, read back from the shared tile by two producer
//         warps (kBDbWarps) while the consumers go on with the next chunk; fp32 sums in their registers for the
//         whole launch, one global atomic per column and warp at the end
//   W_c : weight gradient  dWp[kd, chunk] = A^T . dA_c, warpgroup w: kd rows 64w .. (both operands: MN-major views of
//         tiles already in shared memory), added into this CTA's own slice of a scratch buffer with vector reductions
//   D_c : data gradient    [dx_below | dh_prev] += dA_c . Wp[:, chunk]^T  (B: MN-major view of the resident weights;
//         accumulated in registers over the four chunks, stored at the end of the item)
// Schedule of a warpgroup (one dA tile shared by both warpgroups and the B_c warps, so they stay in step at its two
// barriers per chunk):
//   c = 0      : R_0; wait; P_0; barrier; dA_0 -> tile; barrier                                   (then B_0)
//   c = 1 .. 3 : R_c | W_{c-1} + D_{c-1} (two commit groups); wait for R_c only; P_c (dA_c kept in registers)
//                while the tensor pipe runs W / D; wait; red.add W_{c-1}; barrier; dA_c -> tile; barrier (then B_c)
//   item end   : W_3 | D_3; wait for W_3; A planes released to the producer; red.add W_3; wait for D_3; store
// The wgmma operands and the accumulation order of every accumulator are those of the unpipelined schedule.
// dA never leaves the SM; the gates are never stored.  lstm16_wgrad_reduce_kernel sums the slices after each layer's
// launch and writes nn.LSTM-native gradients.
constexpr int kBWarpgroups = 2;
constexpr int kBThreads = kBWarpgroups * 128 + 128;     // + producer warpgroup (one thread of it issues the loads)
constexpr int kBCons = kBWarpgroups * 128;              // consumer threads
constexpr uint32_t kBBarCons = 1;                       // named barrier of the consumer warpgroups (kBCons threads)
constexpr uint32_t kBBarWg = 2;                         // named barrier kBBarWg + w: consumer warpgroup w (128 threads)
constexpr int kBDbWarps = 2;                            // producer warps 1 .. kBDbWarps: the bias gradient (B_c)
constexpr uint32_t kBBarDa = 4;                         // named barrier of the dA tile: consumers + the B_c warps
constexpr uint32_t kBDaThreads = kBCons + 32 * kBDbWarps;
// registers per thread after setmaxnreg: 256 * 240 + 128 * 24 = 64 512 of the SM's 65 536 (launched at 384 * 168)
constexpr uint32_t kBConsRegs = 240, kBProdRegs = 24;
constexpr int kBATiles = 4;                             // (seg0 | seg1) x (hi | lo); layer 0: seg 1 = the auxiliary [x*s] tile

struct B16Tail {
    float bias[kGateCols];             // gate-interleaved bias, pre-scaled (gate_scale) as the forward's
    uint64_t a_full, a_empty, w_full;
};
constexpr size_t kBSmem = 1024 + 4 * (size_t)kWTileBytes + kBATiles * (size_t)kATileBytes + 2 * (size_t)kATileBytes + sizeof(B16Tail);
static_assert(kBSmem <= 232448, "lstm16 backward kernel exceeds the 227 KB shared-memory limit");

// One launch = one LAYER, its timesteps from T-1 down (the tiles of a CTA are its own through time: rows never mix).
// A step of a tile needs what the SAME CTA produced for that tile one step later (dh_rec, dc: global, in place), so nothing
// but the launch order of the layers (top down) synchronises.  Items are tile-major: a CTA walks one tile through all
// T steps before the next, so dh_rec / dc are read back one item after they were written (64 KB per CTA, ~8.4 MB for
// 132 CTAs, L2-resident) instead of after a whole step of every tile had gone through the 50 MB L2.
constexpr int kBMaxSteps = 64;
struct Bwd16Step {
    int32_t slice[2];          // plane slice of K segment s in its tensor map (hi plane; lo = + 1)
    int8_t src[2];             // 0: maps[0] (hp), 1: maps[1] (h0p), 2: zeros (h_prev at t = 0 without an initial state)
    int8_t first;              // t == T-1 without seeds: incoming dh_rec / dc are zero and not read
    int8_t store_dh;           // write dh_prev (t > 0, an initial state exists, or its gradient is wanted)
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
    float* d_xo;               // (rows, T, C) overwritten, or nullptr   (layer 0)
    int c_in, t_len, n_steps;
    int64_t b_inner;
    float* dh_rec;             // blocked, in (unless first) / out, in place through the steps
    float* dc;                 // blocked, in (unless first) / out, in place through the steps
    float* dbp;                // (256) +=  gate-interleaved bias gradient
    float* dw_slice;           // gridDim.x slices of 128 x 256 floats (fragment order, see bwd_wgrad_red), +=
    int64_t rows;
    int n_tiles;
    Bwd16Step steps[kBMaxSteps];   // in execution order: steps[0] is t = T-1
};
static_assert(sizeof(Bwd16Params) <= 4096, "kernel parameter block exceeds 4 KB");

// R_c: g = [h_below | h_prev] . Wp[:, chunk c] of this warpgroup's 64 rows
template <int PLANES, int NSEG>
__device__ __forceinline__ void bwd_recompute_mma(float (&g)[32], uint32_t a_u, uint32_t a_rows, uint32_t w_u, int c) {
#pragma unroll
    for (int s = 0; s < NSEG; ++s) {
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
}

constexpr uint32_t kStepMN = 2048;                             // MN-major k16 step: 16 rows of 128 bytes

// W_c: wgr = A^T . dA_c, kd rows 64 wg .. 64 wg + 63 (wa_hi: this warpgroup's A tile, hi plane; its lo plane follows)
template <int PLANES, bool L0>
__device__ __forceinline__ void bwd_wgrad_mma(float (&wgr)[32], uint32_t wa_hi, uint32_t da_u) {
    const uint32_t wa_lo = wa_hi + kATileBytes;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
        const uint64_t ah = desc16_mn(wa_hi + ks * kStepMN, kATileBytes);
        const uint64_t al = desc16_mn(wa_lo + ks * kStepMN, kATileBytes);
        const uint64_t bh = desc16_mn(da_u + ks * kStepMN, kATileBytes);
        const uint64_t bl = desc16_mn(da_u + kATileBytes + ks * kStepMN, kATileBytes);
        // dA always has its lo plane; in the single-plane mode only the STORED operands are rounded to bf16.
        // Layer 0's warpgroup 1 multiplies the auxiliary x*s tile, which is not stored: it keeps its lo plane in
        // both modes, as the forward's fp32 FMAs do (warpgroup 0's lo slot is zero then, and adds nothing; both
        // warpgroups issue the pass so that no wgmma sits on a warpgroup-dependent branch, which would make
        // ptxas serialise every wgmma of the kernel)
        wgmma_bf16_n64_t11(wgr, ah, bh, ks > 0 ? 1u : 0u);
        wgmma_bf16_n64_t11(wgr, ah, bl, 1u);
        if (PLANES == 2 || L0) wgmma_bf16_n64_t11(wgr, al, bh, 1u);
    }
}

// D_c: [dx_below | dh_prev] += dA_c . Wp[:, chunk c]^T
template <int PLANES, int NSEG>
__device__ __forceinline__ void bwd_dgrad_mma(float (&dacc)[32 * NSEG], uint32_t da_u, uint32_t a_rows, uint32_t w_u, int c) {
    const uint64_t ah = desc16_k(da_u + a_rows), al = desc16_k(da_u + kATileBytes + a_rows);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        const uint32_t wb = w_u + (uint32_t)c * 8192u + (uint32_t)kk * kStepMN;
        const uint64_t bh = desc16_mn(wb, 2 * kWTileBytes), bl = desc16_mn(wb + kWTileBytes, 2 * kWTileBytes);
        if constexpr (NSEG == 2) {
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

// The per-CTA weight-gradient slice is kept in FRAGMENT order: float4 (c, j, consumer thread) holds wgr[4j .. 4j+3] of
// chunk c, i.e. the four accumulator values a consumer thread owns for every item of the launch, at float offset
// ((8c + j) * kBCons + thread) * 4.  A warp's flush of one j is then one red.v4 over 512 contiguous bytes, four whole
// L2 lines; row-major [kd][256], the same adds took two red.v2 that each touched eight lines.
// lstm16_wgrad_reduce_kernel maps it back (wgrad_slice_row_col).
constexpr int kWgrSliceFloats = kTileM * kGateCols;
__device__ __forceinline__ void wgrad_slice_row_col(int e, int& m, int& n) {
    const int v = e & 3, thr = (e >> 2) % kBCons, cj = (e >> 2) / kBCons;
    const int lane = thr & 31, q = lane & 3;
    m = 64 * (thr >> 7) + 16 * ((thr >> 5) & 3) + (lane >> 2) + 8 * (v >> 1);      // fragment rows rw0, rw0 + 8
    n = 8 * cj + 2 * q + (v & 1);                                                     // 64 c + 8 j + 2 q + {0, 1}
}
// weight-gradient fragment of chunk c -> this CTA's slice; slice_t: the slice + 4 * (this consumer thread)
__device__ __forceinline__ void bwd_wgrad_red(float* slice_t, const float (&wgr)[32], int c) {
    float* dst = slice_t + (size_t)c * (8 * 4 * kBCons);
#pragma unroll
    for (int j = 0; j < 8; ++j)
        red_add_f32x4(dst + j * (4 * kBCons), wgr[4 * j], wgr[4 * j + 1], wgr[4 * j + 2], wgr[4 * j + 3]);
}

// CIN: see lstm16_fwd_kernel.  WGRAD = false: the variant for a caller that wants no weight gradients -- the schedule
// above with the W_c wgmma, their red.add flushes and the B_c warps compiled out (everything else in the same order:
// the W_3 commit group stays, empty, so the A planes are still released after the item's last wait for it; the dA tile
// is released by the D_c waits alone).  p.dbp and p.dw_slice are not used.
template <int PLANES, int CIN, bool WGRAD>
__global__ void __launch_bounds__(kBThreads, 1) lstm16_bwd_kernel(const __grid_constant__ Bwd16Params p) {
    constexpr bool L0 = CIN > 0;
    // threads of the dA tile's named barrier: the consumers, and the B_c warps when they sum the bias gradient
    constexpr uint32_t kDaThreads = WGRAD ? kBDaThreads : (uint32_t)kBCons;
    constexpr int kC = (CIN == 1) ? 1 : kMaxC;
    constexpr int kNseg = L0 ? 1 : 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + smem_pad1024(smem_raw);
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

    if (tid == 0) {
        mbar_init(&tail->a_full, 1);
        mbar_init(&tail->a_empty, kBWarpgroups);
        mbar_init(&tail->w_full, 1);
        fence_barrier_init();
    }
    for (int i = tid; i < kGateCols; i += kBThreads) tail->bias[i] = p.bias[i] * gate_scale(i);
    if (L0) {
        for (int i = tid; i < p.c_in * kGateCols; i += kBThreads) wih_s[i] = p.wih[i] * gate_scale(i);
        // auxiliary tiles (seg-1 slots): zero once; columns 0..C-1 are rewritten per item.  One plane: the h_prev lo slot is
        // never loaded; zeroed, it lets both warpgroups issue the lo-plane weight-gradient pass (see W_c)
        for (int i = tid; i < 2 * kATileBytes / 16; i += kBThreads)
            reinterpret_cast<uint4*>(a_sm + 2 * (size_t)kATileBytes)[i] = make_uint4(0u, 0u, 0u, 0u);
        if (PLANES == 1)
            for (int i = tid; i < kATileBytes / 16; i += kBThreads)
                reinterpret_cast<uint4*>(a_sm + (size_t)kATileBytes)[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    fence_proxy_async_smem();
    __syncthreads();
    const int my_tiles = cta_tiles(p.n_tiles);
    const int n_items = my_tiles * p.n_steps;                      // work items (step, tile), tile-major

    if (warp >= kProdWarp) {
        // ===================== producer =====================
        setmaxnreg_dec<kBProdRegs>();
        const bool leader = warp == kProdWarp && elect_one_sync();
        if (leader && n_items > 0) {
            load_weights<kNseg, PLANES>(w_sm, p, &tail->w_full);
            const uint64_t once = l2_evict_first();          // the A planes; dh_rec / dc and the slices keep their L2 place
            for (int w = 0; w < n_items; ++w) {
                const int ti = w / p.n_steps, st = w - ti * p.n_steps, tile = cta_tile(ti);
                const Bwd16Step& sp = p.steps[st];
                mbar_wait_polite(&tail->a_empty, (uint32_t)(w & 1) ^ 1u);
                mbar_arrive_expect_tx(&tail->a_full, (uint32_t)(kNseg * PLANES * kATileBytes));
                for (int sg = 0; sg < kNseg; ++sg)
                    for (int pl = 0; pl < PLANES; ++pl) {
                        uint8_t* dst = a_sm + (size_t)(sg * 2 + pl) * kATileBytes;
                        if (sp.src[sg] == 2) bulk_g2s(dst, p.zero_tile, kATileBytes, &tail->a_full);
                        else tma_load_3d_hint(dst, &p.maps[sp.src[sg]], 0, tile * kTileM, sp.slice[sg] + pl, &tail->a_full, once);
                    }
                // the per-row inputs of this item -> L2 (a tile is one contiguous 32 KB run in every workspace)
                const int64_t o = (int64_t)tile * kTileM * kHid;
                constexpr uint32_t kB = kTileM * kHid * 4;
                if (sp.c_prev) prefetch_l2(sp.c_prev + o, kB);
                if (sp.dh_in) prefetch_l2(sp.dh_in + o, kB);
                // the next item's A planes -> L2, a whole item ahead of the load that waits for them
                if (w + 1 < n_items) {
                    const int ti1 = (w + 1) / p.n_steps, tile1 = cta_tile(ti1);
                    const Bwd16Step& sp1 = p.steps[w + 1 - ti1 * p.n_steps];
                    for (int sg = 0; sg < kNseg; ++sg)
                        for (int pl = 0; pl < PLANES; ++pl)
                            if (sp1.src[sg] != 2) tma_prefetch_3d(&p.maps[sp1.src[sg]], 0, tile1 * kTileM, sp1.slice[sg] + pl);
                }
            }
        } else if (WGRAD && warp > kProdWarp && warp <= kProdWarp + kBDbWarps && n_items > 0) {
            // ---- B_c: bias gradient, column sums of every dA_c tile (hi + lo; rows past the end carry dA = 0) ----
            // Warp kProdWarp + 1 + h sums rows 64h .. 64h + 63, lane l the columns 2l, 2l + 1 of each chunk: a warp reads one
            // 128-byte tile row per load, conflict free.  The tile is read between store_da's second barrier (complete)
            // and the first of the next store_da (free to be overwritten), which the consumers reach a whole chunk later.
            // All of it fits the producer's kBProdRegs registers: 8 sums for the launch, 8 loaded words in flight.
            // (rows: this warp's first row, a multiple of 8, so a row's swizzle phase is its index in the warp's half & 7)
            const uint8_t* rows = da_sm + (size_t)(warp - kProdWarp - 1) * 64u * 128u;
            float db[4][2] = {};
            for (int w = 0; w < n_items; ++w) {
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    bar_sync(kBBarDa, kBDaThreads);                // store_da: the tile is free
                    bar_sync(kBBarDa, kBDaThreads);                // store_da: dA_c is complete
#pragma unroll 1
                    for (uint32_t r4 = 0; r4 < 64u; r4 += 4u) {
#pragma unroll
                        for (uint32_t k = 0; k < 4; ++k) {
                            const uint32_t off = sw128<2>(r4 + k, 2u * (uint32_t)lane);
                            const uint32_t hi = *reinterpret_cast<const uint32_t*>(rows + off);
                            const uint32_t lo = *reinterpret_cast<const uint32_t*>(rows + kATileBytes + off);
                            db[c][0] += bf16_lo_as_f32(hi) + bf16_lo_as_f32(lo);
                            db[c][1] += bf16_hi_as_f32(hi) + bf16_hi_as_f32(lo);
                        }
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                atomicAdd(&p.dbp[64 * c + 2 * lane], db[c][0]);
                atomicAdd(&p.dbp[64 * c + 2 * lane + 1], db[c][1]);
            }
        }
        return;
    }

    // ===================== consumers =====================
    setmaxnreg_inc<kBConsRegs>();
    const int wg = tid >> 7;
    const int q = lane & 3;
    const bool odd = (q & 1) != 0;
    const uint32_t rw0 = (uint32_t)(64 * wg + 16 * (warp & 3) + (lane >> 2));   // fragment row (and rw0 + 8)
    const uint32_t row_in_tile = rw0 + (odd ? 8u : 0u);                          // this thread's cell row
    const uint32_t rows32 = (uint32_t)p.rows;
    const uint32_t w_u = smem_u32(w_sm), a_u = smem_u32(a_sm), da_u = smem_u32(da_sm);
    const uint32_t a_rows = (uint32_t)wg * 64u * 128u;             // this warpgroup's rows inside a 128-row tile
    const uint32_t wa_u = a_u + (uint32_t)(wg * 2) * kATileBytes;  // W_c's A operand: this warpgroup's kd rows
    float* slice_t = WGRAD ? p.dw_slice + (size_t)blockIdx.x * kWgrSliceFloats + 4 * tid : nullptr;
    mbar_wait_raw(&tail->w_full, 0);

    for (int w = 0; w < n_items; ++w) {
        const int ti = w / p.n_steps, st = w - ti * p.n_steps, tile = cta_tile(ti);
        const Bwd16Step& sp = p.steps[st];
        const uint32_t r = (uint32_t)tile * kTileM + row_in_tile;
        const bool valid = r < rows32;
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
        bar_sync(kBBarCons, kBCons);
        if (WGRAD && L0 && (q >> 1) == 0) {
            // auxiliary weight-gradient operand (seg-1 slots): row = this thread's row, columns 0..C-1 = x*s (hi / lo split)
            uint32_t hi[2], lo[2];
            split_bf16x2(xs[0], xs[1], hi[0], lo[0]);
            split_bf16x2(xs[2], xs[3], hi[1], lo[1]);
            const uint32_t off = sw128<2>(row_in_tile, 0);
            *reinterpret_cast<uint2*>(a_sm + 2 * (size_t)kATileBytes + off) = make_uint2(hi[0], hi[1]);
            *reinterpret_cast<uint2*>(a_sm + 3 * (size_t)kATileBytes + off) = make_uint2(lo[0], lo[1]);
        }
        mbar_wait_raw(&tail->a_full, (uint32_t)w & 1u);
        float dacc[32 * kNseg];                                    // [dx_below | dh_prev] (layer 0: [dh_prev])
#pragma unroll
        for (int k = 0; k < 32 * kNseg; ++k) dacc[k] = 0.f;
        float wgr[32];                                             // W of the previous chunk, in flight during P_c
        const uint32_t bo = blocked_off(tile, row_in_tile, 0);     // this thread's row; unit u is + blocked_off(0, 0, u)
        float cpv[8], dhv[8], dciv[8];
        // the cells' global inputs of chunk c, all issued while the tensor pipe runs: each cell loading its own after
        // the previous cell's dc store (which they may alias, as far as the compiler knows) waited one memory round
        // trip per cell.  dh_in and dh_rec are added once all loads are issued, so that no load waits on an add.
        // c_prev and dh_in are read once per launch: streaming loads (evict-first).
        auto load_cells = [&](int c) {
            float dhr[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int unit = 16 * c + 2 * j + (q >> 1);
                const uint32_t o = bo + blocked_off(0, 0, unit);
                const bool rec = valid && !sp.first;
                cpv[j] = (valid && sp.c_prev) ? __ldcs(sp.c_prev + o) : 0.f;
                dhv[j] = (valid && sp.dh_in) ? __ldcs(sp.dh_in + o) : 0.f;
                dhr[j] = rec ? p.dh_rec[o] : 0.f;
                dciv[j] = rec ? p.dc[o] : 0.f;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) dhv[j] += dhr[j];
        };
        uint32_t dpk[32];                                          // dA_c as bf16 planes: [4j, 4j+1] hi, [4j+2, 4j+3] lo
        // ---- P_c: 8 cells per thread (row row_in_tile, units 16c + 2j + q/2) -> dpk, dc ----
        auto cell_epilogue = [&](int c, const float (&g)[32]) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float4 v = frag_to_gates(g, j, odd);
                const int unit = 16 * c + 2 * j + (q >> 1);
                const int col = 4 * unit;
                const float4 bv = *reinterpret_cast<const float4*>(&tail->bias[col]);      // pre-scaled (gate_scale)
                const float4 a = gate_args<CIN>(v, bv, xs, wih_s, col, p.c_in);
                const uint32_t o = bo + blocked_off(0, 0, unit);
                const float cp = cpv[j], dh = dhv[j], dci = dciv[j];
                float gi, gf, gg, go, tc_;
                lstm_cell_gates8(a.x, a.y, a.z, a.w, cp, gi, gf, gg, go, tc_);
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
                            // W_ih is stored pre-scaled: undo kNegLog2e (and the g gate's extra factor 2)
                            const float4 wv = *reinterpret_cast<const float4*>(&wih_s[cc * kGateCols + col]);
                            dxs[cc] = fmaf(da0 * wv.x + da1 * wv.y + 0.5f * (da2 * wv.z) + da3 * wv.w, -kLn2, dxs[cc]);
                        }
                }
                split_bf16x2(da0, da1, dpk[4 * j], dpk[4 * j + 2]);
                split_bf16x2(da2, da3, dpk[4 * j + 1], dpk[4 * j + 3]);
            }
        };
        // dpk -> the shared dA tile, once both warpgroups' W / D and the B warps of the previous chunk have read it
        auto store_da = [&]() {
            bar_sync(kBBarDa, kDaThreads);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint32_t off = sw128<2>(row_in_tile, 4 * (2 * j + (q >> 1)));   // gates of unit 16c + 2j + q/2
                *reinterpret_cast<uint2*>(da_sm + off) = make_uint2(dpk[4 * j], dpk[4 * j + 1]);
                *reinterpret_cast<uint2*>(da_sm + kATileBytes + off) = make_uint2(dpk[4 * j + 2], dpk[4 * j + 3]);
            }
            fence_proxy_async_smem();
            bar_sync(kBBarDa, kDaThreads);                         // the dA tile (both row halves) is complete
        };
        // ---- chunk 0: R_0 alone ----
        {
            float g[32];                                           // (the first wgmma of R overwrites: scale-d 0)
            wg_fence_regs(g);
            wg_fence();
            bwd_recompute_mma<PLANES, kNseg>(g, a_u, a_rows, w_u, 0);
            wg_commit();
            load_cells(0);
            wg_wait<0>();
            wg_fence_regs(g);
            cell_epilogue(0, g);
            store_da();
        }
        // ---- chunks 1..3, software-pipelined: R_c and W_{c-1} + D_{c-1} are committed as two groups; waiting for the
        // first retires R_c only, so P_c runs on the CUDA cores while the tensor pipe still works on chunk c - 1.  The dA
        // tile holds dA_{c-1} until W / D of both warpgroups have read it, so dA_c waits in registers (dpk) until then.
        // (The loop is not unrolled, and no wgmma is behind a branch: either makes ptxas serialise the wgmma.)
#pragma unroll 1
        for (int c = 1; c < 4; ++c) {
            // the operand addresses, opaque to the compiler once per chunk: the wgmma descriptors derived from them are
            // then rebuilt in the uniform datapath at each issue instead of being hoisted out of the loop, where their
            // 64-bit values outlived P_c and were spilled to local memory
            uint32_t a_c = a_u, w_c = w_u, wa_c = wa_u, da_c = da_u;
            asm volatile("" : "+r"(a_c), "+r"(w_c), "+r"(wa_c), "+r"(da_c));
            float g[32];
            wg_fence_regs(g);
            if constexpr (WGRAD) wg_fence_regs(wgr);
            wg_fence_regs(dacc);
            wg_fence();
            bwd_recompute_mma<PLANES, kNseg>(g, a_c, a_rows, w_c, c);
            wg_commit();
            if constexpr (WGRAD) bwd_wgrad_mma<PLANES, L0>(wgr, wa_c, da_c);
            bwd_dgrad_mma<PLANES, kNseg>(dacc, da_c, a_rows, w_c, c - 1);
            wg_commit();
            load_cells(c);
            wg_wait<1>();
            wg_fence_regs(g);
            cell_epilogue(c, g);
            wg_wait<0>();
            if constexpr (WGRAD) wg_fence_regs(wgr);
            wg_fence_regs(dacc);
            if constexpr (WGRAD) bwd_wgrad_red(slice_t, wgr, c - 1);
            store_da();
        }
        // ---- chunk 3's gradients: W_3 alone first, so that the A planes go back to the producer before D_3 is done ----
        if constexpr (WGRAD) wg_fence_regs(wgr);
        wg_fence_regs(dacc);
        wg_fence();
        if constexpr (WGRAD) bwd_wgrad_mma<PLANES, L0>(wgr, wa_u, da_u);
        wg_commit();
        bwd_dgrad_mma<PLANES, kNseg>(dacc, da_u, a_rows, w_u, 3);
        wg_commit();
        wg_wait<1>();
        if constexpr (WGRAD) wg_fence_regs(wgr);
        // the A planes of this item have been read by every MMA: one arrival per warpgroup
        bar_sync(kBBarWg + wg, 128);
        if ((tid & 127) == 0) mbar_arrive(&tail->a_empty);
        if constexpr (WGRAD) bwd_wgrad_red(slice_t, wgr, 3);
        wg_wait<0>();
        wg_fence_regs(dacc);
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
                // = blocked_off(tile, rr, unit), added to the pointer term by term (one 32-bit sum compiles differently)
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
            if ((q >> 1) == 0 && valid) atomicAdd(&p.d_s[(int64_t)(r % (uint32_t)p.b_inner) * p.t_len + sp.t], contrib);
            if (p.d_xo != nullptr) {
                // input gradient: d xo[r, t, c] = dxmod[r, c] * s[b, t]; the lane pair (q, q ^ 2) holds the row's two halves
                float* dst = p.d_xo + ((int64_t)r * p.t_len + sp.t) * p.c_in;
                const float sv = valid ? p.sg[(r % (uint32_t)p.b_inner) * (uint32_t)p.t_len + (uint32_t)sp.t] : 0.f;
#pragma unroll
                for (int cc = 0; cc < kC; ++cc) {
                    const float dx = dxs[cc] + __shfl_xor_sync(0xffffffffu, dxs[cc], 2);
                    if ((q >> 1) == 0 && valid && (CIN == 1 || cc < p.c_in)) dst[cc] = dx * sv;
                }
            }
        }
    }
}

// Sum the per-CTA weight-gradient slices of one layer and write nn.LSTM-native gradients:
//   d_w_ih (256, in), d_w_hh (256, 64), d_b_ih = d_b_hh (256); native row of gate-interleaved column n: (n & 3) * 64 + (n >> 2).
// Slice element e holds kd row m, gate column n (wgrad_slice_row_col): layers > 0: m < 64 -> W_ih[:, m], m >= 64 ->
// W_hh[:, m - 64]; layer 0: m < 64 -> W_hh[:, m], m = 64 + c -> W_ih[:, c].
__global__ void lstm16_wgrad_reduce_kernel(const float* __restrict__ slices, int n_slices, int layer, int c_in,
                                           const float* __restrict__ dbp, float* __restrict__ d_w_ih,
                                           float* __restrict__ d_w_hh, float* __restrict__ d_b_ih, float* __restrict__ d_b_hh) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;           // index in the slice layout
    if (e < kWgrSliceFloats) {
        float s = 0.f;
        for (int i = 0; i < n_slices; ++i) s += slices[(size_t)i * kWgrSliceFloats + e];
        int m, n;
        wgrad_slice_row_col(e, m, n);
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
// (slices, rows, 64) bf16 plane tensor, box = 1 x box_rows x 64, 128-byte swizzle (rows past the end read as zeros;
// stores drop them)
static bool make_plane_map(CUtensorMap* map, const void* base, int64_t rows, int64_t slices, int box_rows) {
    EncodeTiledFn16 fn = encode_fn16();
    if (fn == nullptr) return false;
    const cuuint64_t dims[3] = {(cuuint64_t)kHid, (cuuint64_t)rows, (cuuint64_t)slices};
    const cuuint64_t strides[2] = {(cuuint64_t)kHid * 2, (cuuint64_t)rows * kHid * 2};
    const cuuint32_t box[3] = {(cuuint32_t)kHid, (cuuint32_t)box_rows, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// the maps of hp (L, T, P, R, 64) and, if given, h0p (L, P, R, 64)
static int32_t make_plane_maps(const char* who, CUtensorMap* hp_map, CUtensorMap* h0_map, const void* hp, const void* h0p,
                               int64_t rows, int n_layers, int t_len, int planes, int box_rows) {
    STMGCN_REQUIRE(make_plane_map(hp_map, hp, rows, (int64_t)n_layers * t_len * planes, box_rows), STMGCN_ERR_STATE,
                   "%s: cuTensorMapEncodeTiled failed (hp)", who);
    if (h0p != nullptr)
        STMGCN_REQUIRE(make_plane_map(h0_map, h0p, rows, (int64_t)n_layers * planes, box_rows), STMGCN_ERR_STATE,
                       "%s: cuTensorMapEncodeTiled failed (h0p)", who);
    return 0;
}

static int32_t check_dims16(const char* who, int32_t t_len, int32_t n_layers, int64_t rows, int32_t c_in, int64_t b_inner,
                            int32_t planes, const float* wih_t, const void* h0p, const float* c0) {
    STMGCN_REQUIRE(planes == 1 || planes == 2, STMGCN_ERR_ARG, "%s: planes=%d", who, planes);
    STMGCN_REQUIRE(n_layers >= 1 && n_layers <= 8 && t_len >= 1 && rows > 0 && c_in >= 1 && c_in <= kMaxC && b_inner > 0,
                   STMGCN_ERR_SHAPE, "%s: L=%d T=%d rows=%lld C=%d", who, n_layers, t_len, (long long)rows, c_in);
    STMGCN_REQUIRE(rows <= (1LL << 25), STMGCN_ERR_SHAPE, "%s: rows=%lld too large (32-bit element offsets)", who, (long long)rows);
    STMGCN_REQUIRE((h0p == nullptr) == (c0 == nullptr), STMGCN_ERR_ARG, "%s: h0p and c0 go together", who);
    STMGCN_REQUIRE(wih_t != nullptr, STMGCN_ERR_ARG, "%s: wih_t null", who);
    return 0;
}

// start of layer l's image in the flat wimg: layer 0 has one K segment (64 KB), every other layer two (128 KB)
static int64_t wimg_off(int l) { return (int64_t)2 * kWTileBytes * (l == 0 ? 0 : 2 * l - 1); }

// kernel(Int<PLANES>, Int<CIN>) for (planes, layer): CIN = 0 (not layer 0), 1 (layer 0, one input channel), else kMaxC
template <int N> struct Int { static constexpr int value = N; };
template <class Kernel>
static auto kernel_for(Kernel kernel, int planes, int l, int c_in) {
    const int cin = l == 0 ? (c_in == 1 ? 1 : kMaxC) : 0;
    if (planes == 2) return cin == 1 ? kernel(Int<2>{}, Int<1>{}) : (cin == kMaxC ? kernel(Int<2>{}, Int<kMaxC>{}) : kernel(Int<2>{}, Int<0>{}));
    return cin == 1 ? kernel(Int<1>{}, Int<1>{}) : (cin == kMaxC ? kernel(Int<1>{}, Int<kMaxC>{}) : kernel(Int<1>{}, Int<0>{}));
}

}  // namespace stmgcn

extern "C" int32_t stmgcn_lstm16_pack(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                      int32_t layer, int32_t c_in, void* wimg, float* bias, float* wih_t, void* stream) {
    STMGCN_REQUIRE(w_ih && w_hh && b_ih && b_hh && wimg && bias, STMGCN_ERR_ARG, "lstm16_pack: null pointer");
    STMGCN_REQUIRE(layer >= 0 && c_in >= 1 && c_in <= kMaxC, STMGCN_ERR_SHAPE, "lstm16_pack: layer=%d c_in=%d", layer, c_in);
    STMGCN_REQUIRE(layer > 0 || wih_t != nullptr, STMGCN_ERR_ARG, "lstm16_pack: layer 0 needs wih_t");
    lstm16_pack_kernel<<<64, 256, 0, (cudaStream_t)stream>>>(w_ih, w_hh, b_ih, b_hh, layer, c_in, (uint8_t*)wimg + wimg_off(layer),
                                                              bias + (int64_t)layer * kGateCols, wih_t);
    count_launch();
    return check_launch("lstm16_pack");
}

extern "C" int32_t stmgcn_lstm16_fwd(int32_t t_len, int32_t n_layers, int64_t rows, int32_t c_in, int64_t b_inner,
                                     int32_t planes, const float* xo, const float* s_gate, const void* wimg,
                                     const float* bias, const float* wih_t, const void* h0p, const float* c0, void* hp,
                                     float* cs, float* h_top, float* h_n, void* stream) {
    STMGCN_REQUIRE(xo && s_gate && wimg && bias && hp && cs, STMGCN_ERR_ARG, "lstm16_fwd: null pointer");
    if (int32_t rc = check_dims16("lstm16_fwd", t_len, n_layers, rows, c_in, b_inner, planes, wih_t, h0p, c0)) return rc;
    STMGCN_REQUIRE(h_n != nullptr || h_top != nullptr, STMGCN_ERR_ARG, "lstm16_fwd: h_top null");
    cudaStream_t st = (cudaStream_t)stream;
    const int n_tiles = (int)ceil_div(rows, kTileM);
    const int64_t cslice = blocked_slice(n_tiles);
    const int grid = persistent_grid(n_tiles);
    Fwd16Params p;
    memset(&p, 0, sizeof(p));
    // a warpgroup's 64 rows are one box: its h_below loads, h0 loads and tape stores
    if (int32_t rc = make_plane_maps("lstm16_fwd", &p.hp_map, &p.h0_map, hp, h0p, rows, n_layers, t_len, planes, 64)) return rc;
    p.xo = xo;
    p.sg = s_gate;
    p.c_in = c_in;
    p.t_len = t_len;
    p.has_h0 = h0p != nullptr ? 1 : 0;
    p.b_inner = b_inner;
    p.rows = rows;
    p.n_tiles = n_tiles;
    // bottom-up: layer l reads the hp planes of layer l - 1
    for (int l = 0; l < n_layers; ++l) {
        const auto fn = kernel_for([](auto P, auto C) { return lstm16_fwd_kernel<P.value, C.value>; }, planes, l, c_in);
        if (int32_t rc = ensure_dyn_smem((const void*)fn, kFSmem)) return rc;
        p.wimg = (const uint8_t*)wimg + wimg_off(l);
        p.bias = bias + (int64_t)l * kGateCols;
        p.wih = l == 0 ? wih_t : nullptr;
        p.layer = l;
        p.c0 = c0 != nullptr ? c0 + (int64_t)l * cslice : nullptr;
        p.cs = cs + (int64_t)l * t_len * cslice;
        p.h_f32 = h_n != nullptr ? h_n + (int64_t)l * rows * kHid : (l == n_layers - 1 ? h_top : nullptr);
        fn<<<grid, kFThreads, kFSmem, st>>>(p);
        count_launch();
        if (int32_t rc = check_launch("lstm16_fwd")) return rc;
    }
    return 0;
}

extern "C" int32_t stmgcn_lstm16_grid(int64_t rows) { return persistent_grid(ceil_div(rows, kTileM)); }

extern "C" int32_t stmgcn_lstm16_bwd_ex(int32_t t_len, int32_t n_layers, int64_t rows, int32_t c_in, int64_t b_inner,
                                        int32_t planes, const float* xo, const float* s_gate, const void* wimg,
                                        const float* bias, const float* wih_t, const void* h0p, const float* c0,
                                        const void* hp, const float* cs, const float* d_top, float* dh_rec, float* dc,
                                        float* dx_work, float* dw_scratch, float* dbp, const void* zero_tile, float* d_s,
                                        float* grads, const float* dh_n, const float* dc_n, float* dh0, float* dc0,
                                        float* d_xo, void* stream) {
    // grads NULL: no weight or bias gradients (dw_scratch and dbp are then unused and may be NULL too)
    const bool wgrad = grads != nullptr;
    STMGCN_REQUIRE(xo && s_gate && wimg && bias && hp && cs && d_top && dh_rec && dc && zero_tile && d_s &&
                       (!wgrad || (dw_scratch && dbp)),
                   STMGCN_ERR_ARG, "lstm16_bwd: null pointer");
    if (int32_t rc = check_dims16("lstm16_bwd", t_len, n_layers, rows, c_in, b_inner, planes, wih_t, h0p, c0)) return rc;
    STMGCN_REQUIRE(t_len <= kBMaxSteps, STMGCN_ERR_SHAPE, "lstm16_bwd: T=%d (max %d)", t_len, kBMaxSteps);
    STMGCN_REQUIRE(n_layers == 1 || dx_work != nullptr, STMGCN_ERR_ARG, "lstm16_bwd: dx_work null with L=%d", n_layers);
    cudaStream_t st = (cudaStream_t)stream;
    const int n_tiles = (int)ceil_div(rows, kTileM);
    const int64_t cslice = blocked_slice(n_tiles);
    const int grid = persistent_grid(n_tiles);
    Bwd16Params p;
    memset(&p, 0, sizeof(p));
    if (int32_t rc = make_plane_maps("lstm16_bwd", &p.maps[0], &p.maps[1], hp, h0p, rows, n_layers, t_len, planes, kTileM))
        return rc;
    p.zero_tile = (const uint8_t*)zero_tile;
    p.xo = xo;
    p.sg = s_gate;
    p.d_s = d_s;
    p.c_in = c_in;
    p.t_len = t_len;
    p.b_inner = b_inner;
    const bool seeded = dh_n != nullptr || dc_n != nullptr;
    const size_t slice_bytes = (size_t)blocked_slice(n_tiles) * sizeof(float);
    p.dh_rec = dh_rec;
    p.dc = dc;
    p.dw_slice = dw_scratch;
    p.rows = rows;
    p.n_tiles = n_tiles;
    // one launch covers all timesteps of a layer (t_len <= kBMaxSteps); the weight-gradient partials of every chunk are
    // added into fp32 memory, so the length of the run does not lengthen any tensor-core accumulation chain
    p.n_steps = t_len;
    if (wgrad) STMGCN_CUDA(cudaMemsetAsync(dbp, 0, (size_t)n_layers * kGateCols * sizeof(float), st));
    // top-down: layer l reads the dx that layer l + 1 wrote into one half of dx_work and writes its own into the other
    const float* dh_in = d_top;
    for (int l = n_layers - 1; l >= 0; --l) {
        const auto fn = kernel_for([wgrad](auto P, auto C) {
            return wgrad ? lstm16_bwd_kernel<P.value, C.value, true> : lstm16_bwd_kernel<P.value, C.value, false>;
        }, planes, l, c_in);
        if (int32_t rc = ensure_dyn_smem((const void*)fn, kBSmem)) return rc;
        float* dx_out = l > 0 ? dx_work + (int64_t)((n_layers - 1 - l) % 2) * t_len * cslice : nullptr;
        p.wimg = (const uint8_t*)wimg + wimg_off(l);
        p.bias = bias + (int64_t)l * kGateCols;
        p.wih = l == 0 ? wih_t : nullptr;
        p.dbp = wgrad ? dbp + (int64_t)l * kGateCols : nullptr;
        p.d_xo = l == 0 ? d_xo : nullptr;
        if (seeded) {
            // the gradients of h_n[l] / c_n[l] are what the step at T-1 reads as the incoming dh_rec / dc
            if (dh_n != nullptr) STMGCN_CUDA(cudaMemcpyAsync(dh_rec, dh_n + (int64_t)l * cslice, slice_bytes, cudaMemcpyDeviceToDevice, st));
            else STMGCN_CUDA(cudaMemsetAsync(dh_rec, 0, slice_bytes, st));
            if (dc_n != nullptr) STMGCN_CUDA(cudaMemcpyAsync(dc, dc_n + (int64_t)l * cslice, slice_bytes, cudaMemcpyDeviceToDevice, st));
            else STMGCN_CUDA(cudaMemsetAsync(dc, 0, slice_bytes, st));
        }
        for (int si = 0; si < t_len; ++si) {
            const int t = t_len - 1 - si;
            Bwd16Step& sp = p.steps[si];
            sp = Bwd16Step{};
            // the K segments in the order of the weight image's: layers > 0 first read h of the layer below at step t;
            // then h_prev: hp at t - 1, at t = 0 the initial state h0p if there is one, else the zero tile (STMGCN.py:53-57)
            const int s = l > 0 ? 1 : 0;
            if (l > 0) sp.slice[0] = ((l - 1) * t_len + t) * planes;
            if (t > 0) {
                sp.slice[s] = (l * t_len + t - 1) * planes;
            } else if (h0p != nullptr) {
                sp.src[s] = 1;
                sp.slice[s] = l * planes;
            } else {
                sp.src[s] = 2;
            }
            sp.t = t;
            sp.first = (t == t_len - 1 && !seeded) ? 1 : 0;
            // the gradient at a zero initial state is well defined: dh0 wants it stored too
            sp.store_dh = (t > 0 || h0p != nullptr || dh0 != nullptr) ? 1 : 0;
            sp.c_prev = t > 0 ? cs + (int64_t)(l * t_len + t - 1) * cslice : (c0 ? c0 + (int64_t)l * cslice : nullptr);
            sp.dh_in = l == n_layers - 1 ? (t == t_len - 1 ? d_top : nullptr) : dh_in + (int64_t)t * cslice;
            sp.dx_out = l > 0 ? dx_out + (int64_t)t * cslice : nullptr;
        }
        // every CTA adds into its own slice: start from zero
        if (wgrad) STMGCN_CUDA(cudaMemsetAsync(dw_scratch, 0, (size_t)grid * kWgrSliceFloats * sizeof(float), st));
        fn<<<grid, kBThreads, kBSmem, st>>>(p);
        count_launch();
        if (int32_t rc = check_launch("lstm16_bwd")) return rc;
        // after the step at t = 0, dh_rec / dc hold the gradients of h0[l] / c0[l]: out before the next layer reuses them
        if (dh0 != nullptr) STMGCN_CUDA(cudaMemcpyAsync(dh0 + (int64_t)l * cslice, dh_rec, slice_bytes, cudaMemcpyDeviceToDevice, st));
        if (dc0 != nullptr) STMGCN_CUDA(cudaMemcpyAsync(dc0 + (int64_t)l * cslice, dc, slice_bytes, cudaMemcpyDeviceToDevice, st));
        dh_in = dx_out;
        if (!wgrad) continue;
        // the slices -> this layer's d_w_ih (256, in_l) | d_w_hh (256, 64) | d_b_ih | d_b_hh, before the next layer
        // reuses dw_scratch
        const int in_l = l == 0 ? c_in : kHid;
        float* g = grads + (l == 0 ? 0 : (int64_t)kGateCols * (c_in + kHid + 2 + (l - 1) * (2 * kHid + 2)));
        lstm16_wgrad_reduce_kernel<<<kWgrSliceFloats / 256, 256, 0, st>>>(dw_scratch, grid, l, c_in, p.dbp, g, g + kGateCols * in_l,
                                                                          g + kGateCols * (in_l + kHid),
                                                                          g + kGateCols * (in_l + kHid + 1));
        count_launch();
        if (int32_t rc = check_launch("lstm16_wgrad_reduce")) return rc;
    }
    return 0;
}

extern "C" int32_t stmgcn_lstm16_bwd(int32_t t_len, int32_t n_layers, int64_t rows, int32_t c_in, int64_t b_inner,
                                     int32_t planes, const float* xo, const float* s_gate, const void* wimg,
                                     const float* bias, const float* wih_t, const void* h0p, const float* c0,
                                     const void* hp, const float* cs, const float* d_top, float* dh_rec, float* dc,
                                     float* dx_work, float* dw_scratch, float* dbp, const void* zero_tile, float* d_s,
                                     float* grads, void* stream) {
    return stmgcn_lstm16_bwd_ex(t_len, n_layers, rows, c_in, b_inner, planes, xo, s_gate, wimg, bias, wih_t, h0p, c0, hp, cs,
                                d_top, dh_rec, dc, dx_work, dw_scratch, dbp, zero_tile, d_s, grads, nullptr, nullptr, nullptr,
                                nullptr, nullptr, stream);
}
