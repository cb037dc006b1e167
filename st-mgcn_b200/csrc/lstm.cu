// K3b: the shared-weight LSTM of CG_LSTM (reference STMGCN.py:21-22, :44, :47-50; nn.LSTM semantics: gate
// order i,f,g,o, b_ih + b_hh, zero initial state STMGCN.py:53-57), exact-fp32 CUDA-core path: the shapes the
// tensor-core kernels of lstm16.cu do not cover (H != 64, T > 64) within this file's own limits -- H a multiple of 4
// and <= 128, C <= 4, L <= 8 (check_dims; larger shapes return STMGCN_ERR_SHAPE, they do not run) -- and the on-device
// reference the parity tests compare those kernels with.  Own tape: hs, cs (L,T,R,H) and post-activation gates
// (L,T,R,4H), fp32 row-major.
//
// Rows r = n*B + b (node-major) so the top layer's last hidden state IS the (N,B,H) operand of the spatial
// Chebyshev GCN (STMGCN.py:114) with no permute.  The context-gate modulation obs * s[b,t] (STMGCN.py:44)
// is folded into the layer-0 input read.  Weights arrive packed (see include/stmgcn_b200.h):
//   wx  (C, 4H)      = W_ih_l0^T, columns gate-interleaved (col = 4*unit + gate)
//   wp_l (kd_l, 4H)  = [W_ih_l^T ; W_hh_l^T] (l > 0) or W_hh_0^T (l = 0), same column order
//   wpt_l (4H, kd_l) = wp_l^T                (backward data GEMM operand)
//   bp (L, 4H)       = b_ih + b_hh, same column order
// wp_l and wpt_l are layer l's blocks of the flat wp / wpt buffers, at layer_off(l).
// stmgcn_lstm_fwd enqueues one tall GEMM per (t, l), t outer; stmgcn_lstm_bwd enqueues, for t = T-1 .. 0 and within a
// step l = L-1 .. 0, the pointwise kernel and the data GEMM -- layers interleaved within a step, so dx between layers
// needs one (R, H) buffer -- and then one reduce GEMM per layer for the weight gradients.
#include "gemm_tall.cuh"

using namespace stmgcn;


namespace {

constexpr int kMaxLayers = 8;
constexpr int kMaxC = 4;
constexpr int kMaxUnitsPerLane = 4;      // hid <= 128

// ---- forward cell epilogue -----------------------------------------------------------------------------
struct LstmCellEpi {
    const float* bias;       // (4H) interleaved
    const float* wx;         // (C,4H) interleaved or nullptr (layers > 0)
    const float* xo;         // (R,T,C)
    const float* sg;         // (B,T)
    int c_in, t, t_len;
    int64_t b_inner;
    const float* c_prev;     // (R,H) or nullptr
    float* h_out;            // (R,H)
    float* c_out;            // (R,H)
    float* gates_out;        // (R,4H) or nullptr
    int hid;

    template <int TN>
    __device__ __forceinline__ void operator()(float (&acc)[8][8], const TallTile<TN>& tile, int64_t rows, int nc) const {
        const int h4 = 4 * hid;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int64_t r = tile.row(i);
            if (r >= rows) continue;
            float xs[kMaxC];
            if (wx != nullptr) {
                const float sv = sg[(r % b_inner) * t_len + t];
#pragma unroll
                for (int c = 0; c < kMaxC; ++c)
                    xs[c] = (c < c_in) ? xo[(r * t_len + t) * c_in + c] * sv : 0.f;
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int unit = (int)((unsigned)tile.col(4 * u) / 4u);   // columns are >= 0: no sign fix-up
                if (unit >= hid) continue;
                const float4 bv = *reinterpret_cast<const float4*>(bias + 4 * unit);
                float pi = acc[i][4 * u + 0] + bv.x, pf = acc[i][4 * u + 1] + bv.y;
                float pg = acc[i][4 * u + 2] + bv.z, po = acc[i][4 * u + 3] + bv.w;
                if (wx != nullptr) {
#pragma unroll
                    for (int c = 0; c < kMaxC; ++c) {
                        if (c < c_in) {
                            const float4 wv = *reinterpret_cast<const float4*>(wx + (int64_t)c * h4 + 4 * unit);
                            pi = fmaf(xs[c], wv.x, pi);
                            pf = fmaf(xs[c], wv.y, pf);
                            pg = fmaf(xs[c], wv.z, pg);
                            po = fmaf(xs[c], wv.w, po);
                        }
                    }
                }
                const float gi = sigmoidf_(pi), gf = sigmoidf_(pf), gg = tanhf_(pg), go = sigmoidf_(po);
                const float cp = c_prev ? c_prev[r * hid + unit] : 0.f;
                const float cn = fmaf(gf, cp, gi * gg);
                const float hn = go * tanhf_(cn);
                c_out[r * hid + unit] = cn;
                h_out[r * hid + unit] = hn;
                if (gates_out) *reinterpret_cast<float4*>(gates_out + r * h4 + 4 * unit) = make_float4(gi, gf, gg, go);
            }
        }
    }
};

// ---- backward data epilogue: columns [0,w0) -> dst0, [w0, nc) -> dst1 ----------------------------------
struct StoreSplitEpi {
    float* dst0;
    int64_t ld0;
    int w0;
    float* dst1;
    int64_t ld1;

    template <int TN>
    __device__ __forceinline__ void operator()(float (&acc)[8][8], const TallTile<TN>& tile, int64_t rows, int nc) const {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int64_t r = tile.row(i);
            if (r >= rows) continue;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int n = tile.col(j);
                if (n >= nc) continue;
                if (n < w0) dst0[r * ld0 + n] = acc[i][j];
                else dst1[r * ld1 + (n - w0)] = acc[i][j];
            }
        }
    }
};

// ---- backward pointwise: gates (post-activation) -> dA (pre-activation gradient), in place ----------------
// one warp per row; lane owns units lane, lane+32, ...
__global__ void __launch_bounds__(256)
lstm_bwd_pointwise_kernel(int64_t rows, int hid, float* __restrict__ gates, const float* __restrict__ c_t,
                          const float* __restrict__ c_prev, const float* __restrict__ dh_in,
                          const float* __restrict__ dh_rec, float* __restrict__ dc,
                          float* __restrict__ dbp,            // (4H) +=, or nullptr: no bias / dwx gradients
                          // layer-0 extras (wx == nullptr otherwise)
                          const float* __restrict__ wx, float* __restrict__ dwx, const float* __restrict__ xo,
                          const float* __restrict__ sg, float* __restrict__ d_s, int c_in, int t, int t_len,
                          int64_t b_inner, float* __restrict__ d_xo, int seeded) {
    // the incoming dh_rec / dc are zero at the last time step unless the caller seeded them with dh_n / dc_n
    const bool first = (t == t_len - 1) && !seeded;
    extern __shared__ float sm[];            // [4H] dbias | [C*4H] dwx | [b_inner] ds (if it fits)
    const int h4 = 4 * hid;
    float* s_db = sm;
    float* s_dwx = sm + h4;
    float* s_ds = s_dwx + (wx ? c_in * h4 : 0);
    const bool ds_in_smem = (wx != nullptr) && (b_inner <= 2048);
    for (int e = threadIdx.x; e < h4 * (1 + (wx ? c_in : 0)); e += blockDim.x) sm[e] = 0.f;
    if (ds_in_smem)
        for (int e = threadIdx.x; e < b_inner; e += blockDim.x) s_ds[e] = 0.f;
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const int ul = (hid + 31) / 32;
    float4 acc_b[kMaxUnitsPerLane];
    float4 acc_x[kMaxC][kMaxUnitsPerLane];
#pragma unroll
    for (int u = 0; u < kMaxUnitsPerLane; ++u) {
        acc_b[u] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int c = 0; c < kMaxC; ++c) acc_x[c][u] = make_float4(0.f, 0.f, 0.f, 0.f);
    }

    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows;
         r += (int64_t)gridDim.x * (blockDim.x >> 5)) {
        float xs[kMaxC];
        float dxs[kMaxC];
        float sv = 0.f;
        if (wx != nullptr) {
            sv = sg[(r % b_inner) * t_len + t];
#pragma unroll
            for (int c = 0; c < kMaxC; ++c) {
                xs[c] = (c < c_in) ? xo[(r * t_len + t) * c_in + c] * sv : 0.f;
                dxs[c] = 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < kMaxUnitsPerLane; ++u) {
            const int unit = lane + 32 * u;
            if (u >= ul || unit >= hid) continue;
            const int64_t e = r * hid + unit;
            const float4 g = *reinterpret_cast<const float4*>(gates + r * h4 + 4 * unit);   // i,f,g,o
            float dh = first ? 0.f : dh_rec[e];
            if (dh_in) dh += dh_in[e];
            const float tc = tanhf_(c_t[e]);
            const float cp = c_prev ? c_prev[e] : 0.f;
            const float dcv = (first ? 0.f : dc[e]) + dh * g.w * (1.f - tc * tc);
            float4 da;
            da.x = dcv * g.z * g.x * (1.f - g.x);
            da.y = dcv * cp * g.y * (1.f - g.y);
            da.z = dcv * g.x * (1.f - g.z * g.z);
            da.w = dh * tc * g.w * (1.f - g.w);
            dc[e] = dcv * g.y;
            *reinterpret_cast<float4*>(gates + r * h4 + 4 * unit) = da;
            acc_b[u].x += da.x; acc_b[u].y += da.y; acc_b[u].z += da.z; acc_b[u].w += da.w;
            if (wx != nullptr) {
#pragma unroll
                for (int c = 0; c < kMaxC; ++c) {
                    if (c < c_in) {
                        acc_x[c][u].x = fmaf(xs[c], da.x, acc_x[c][u].x);
                        acc_x[c][u].y = fmaf(xs[c], da.y, acc_x[c][u].y);
                        acc_x[c][u].z = fmaf(xs[c], da.z, acc_x[c][u].z);
                        acc_x[c][u].w = fmaf(xs[c], da.w, acc_x[c][u].w);
                        const float4 wv = *reinterpret_cast<const float4*>(wx + (int64_t)c * h4 + 4 * unit);
                        dxs[c] += da.x * wv.x + da.y * wv.y + da.z * wv.z + da.w * wv.w;
                    }
                }
            }
        }
        if (wx != nullptr) {
            // d s[b,t] += sum_c dxmod[r,c] * xo[r,t,c]   (xs = xo*s  =>  xo = xs/s is avoided: reload xo)
            float contrib = 0.f;
#pragma unroll
            for (int c = 0; c < kMaxC; ++c) {
                if (c < c_in) {
                    const float dx = warp_sum(dxs[c]);
                    contrib = fmaf(dx, xo[(r * t_len + t) * c_in + c], contrib);
                    if (d_xo != nullptr && lane == 0) d_xo[(r * t_len + t) * c_in + c] = dx * sv;   // input gradient
                }
            }
            if (lane == 0) {
                const int64_t b = r % b_inner;
                if (ds_in_smem) atomicAdd(&s_ds[b], contrib);
                else atomicAdd(&d_s[b * t_len + t], contrib);
            }
        }
    }
    // CTA reduction of the bias / wx gradients through shared memory, then one global atomic per entry
    const bool wgrad = dbp != nullptr;
#pragma unroll
    for (int u = 0; u < kMaxUnitsPerLane; ++u) {
        const int unit = lane + 32 * u;
        if (!wgrad || u >= ul || unit >= hid) continue;
        atomicAdd(&s_db[4 * unit + 0], acc_b[u].x);
        atomicAdd(&s_db[4 * unit + 1], acc_b[u].y);
        atomicAdd(&s_db[4 * unit + 2], acc_b[u].z);
        atomicAdd(&s_db[4 * unit + 3], acc_b[u].w);
        if (wx != nullptr) {
#pragma unroll
            for (int c = 0; c < kMaxC; ++c) {
                if (c < c_in) {
                    atomicAdd(&s_dwx[c * h4 + 4 * unit + 0], acc_x[c][u].x);
                    atomicAdd(&s_dwx[c * h4 + 4 * unit + 1], acc_x[c][u].y);
                    atomicAdd(&s_dwx[c * h4 + 4 * unit + 2], acc_x[c][u].z);
                    atomicAdd(&s_dwx[c * h4 + 4 * unit + 3], acc_x[c][u].w);
                }
            }
        }
    }
    __syncthreads();
    if (wgrad) for (int e = threadIdx.x; e < h4; e += blockDim.x) atomicAdd(&dbp[e], s_db[e]);
    if (wx != nullptr) {
        if (wgrad) for (int e = threadIdx.x; e < c_in * h4; e += blockDim.x) atomicAdd(&dwx[e], s_dwx[e]);
        if (ds_in_smem)
            for (int e = threadIdx.x; e < b_inner; e += blockDim.x) atomicAdd(&d_s[(int64_t)e * t_len + t], s_ds[e]);
    }
}

int32_t check_dims(const char* who, int32_t t_len, int32_t n_layers, int64_t rows, int32_t hid, int32_t c_in,
                   int64_t b_inner) {
    STMGCN_REQUIRE(t_len >= 1, STMGCN_ERR_SHAPE, "%s: t_len=%d", who, t_len);
    STMGCN_REQUIRE(n_layers >= 1 && n_layers <= kMaxLayers, STMGCN_ERR_SHAPE, "%s: layers=%d (max %d)", who,
                   n_layers, kMaxLayers);
    STMGCN_REQUIRE(rows > 0 && b_inner > 0 && rows % b_inner == 0, STMGCN_ERR_SHAPE, "%s: rows=%lld b=%lld", who,
                   (long long)rows, (long long)b_inner);
    STMGCN_REQUIRE(hid > 0 && hid % 4 == 0 && hid <= 32 * kMaxUnitsPerLane, STMGCN_ERR_SHAPE,
                   "%s: lstm hidden=%d unsupported (need multiple of 4, <= %d)", who, hid, 32 * kMaxUnitsPerLane);
    STMGCN_REQUIRE(c_in >= 1 && c_in <= kMaxC, STMGCN_ERR_SHAPE, "%s: input_dim=%d unsupported (max %d)", who,
                   c_in, kMaxC);
    return 0;
}

// start of layer l's (kd_l, 4H) block in the flat wp / dwp buffers and of its (4H, kd_l) block in wpt: kd_0 = H and
// kd_l = 2H for l > 0, stored back to back
int64_t layer_off(int l, int hid) { return (int64_t)4 * hid * hid * (l == 0 ? 0 : 2 * l - 1); }

}  // namespace

extern "C" {

int32_t stmgcn_lstm_fwd(int32_t t_len, int32_t n_layers, int64_t rows, int32_t hid, int32_t c_in, int64_t b_inner,
                        const float* xo, const float* s_gate, const float* wx, const float* wp, const float* bp,
                        const float* h0, const float* c0, float* hs, float* cs, float* gates, void* stream) {
    STMGCN_REQUIRE(xo && s_gate && wx && wp && bp && hs && cs, STMGCN_ERR_ARG, "lstm_fwd: null pointer");
    if (int32_t rc = check_dims("lstm_fwd", t_len, n_layers, rows, hid, c_in, b_inner)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t rh = rows * hid;
    const int h4 = 4 * hid;
    for (int t = 0; t < t_len; ++t) {
        for (int l = 0; l < n_layers; ++l) {
            const float* h_prev = t > 0 ? hs + ((int64_t)(l * t_len + t - 1)) * rh : (h0 ? h0 + (int64_t)l * rh : nullptr);
            const float* c_prev = t > 0 ? cs + ((int64_t)(l * t_len + t - 1)) * rh : (c0 ? c0 + (int64_t)l * rh : nullptr);
            ASegs a{};
            a.segw = hid;
            a.lda = hid;
            if (l == 0) {
                a.nseg = 1;
                a.seg[0] = h_prev;
            } else {
                a.nseg = 2;
                a.seg[0] = hs + ((int64_t)((l - 1) * t_len + t)) * rh;
                a.seg[1] = h_prev;
            }
            LstmCellEpi epi;
            epi.bias = bp + (int64_t)l * h4;
            epi.wx = (l == 0) ? wx : nullptr;
            epi.xo = xo;
            epi.sg = s_gate;
            epi.c_in = c_in;
            epi.t = t;
            epi.t_len = t_len;
            epi.b_inner = b_inner;
            epi.c_prev = c_prev;
            epi.h_out = hs + ((int64_t)(l * t_len + t)) * rh;
            epi.c_out = cs + ((int64_t)(l * t_len + t)) * rh;
            epi.gates_out = gates ? gates + ((int64_t)(l * t_len + t)) * rows * h4 : nullptr;
            epi.hid = hid;
            if (int32_t rc = launch_tall<256>(a, rows, a.nseg * hid, wp + layer_off(l, hid), h4, h4, epi, st, "lstm_fwd"))
                return rc;
        }
    }
    return 0;
}

int32_t stmgcn_lstm_bwd_ex(int32_t t_len, int32_t n_layers, int64_t rows, int32_t hid, int32_t c_in, int64_t b_inner,
                           const float* xo, const float* s_gate, const float* wx, const float* wpt, const float* h0,
                           const float* c0, const float* cs, const float* hs, float* gates, const float* d_top,
                           float* dh_rec, float* dc, float* dx_work, float* d_s, float* dwx, float* dwp, float* dbp,
                           const float* dh_n, const float* dc_n, float* dh0, float* dc0, float* d_xo, void* stream) {
    STMGCN_REQUIRE(xo && s_gate && wx && wpt && cs && hs && gates && dh_rec && dc && dx_work && d_s, STMGCN_ERR_ARG,
                   "lstm_bwd: null pointer");
    // dwx, dwp and dbp all NULL: no weight or bias gradients (no reduce GEMMs, no bias sums)
    const bool wgrad = dwx != nullptr;
    STMGCN_REQUIRE((dwp != nullptr) == wgrad && (dbp != nullptr) == wgrad, STMGCN_ERR_ARG,
                   "lstm_bwd: dwx, dwp and dbp go together");
    if (int32_t rc = check_dims("lstm_bwd", t_len, n_layers, rows, hid, c_in, b_inner)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t rh = rows * hid;
    const int h4 = 4 * hid;
    const size_t state_bytes = (size_t)n_layers * rh * sizeof(float);
    const int seeded = (dh_n != nullptr || dc_n != nullptr) ? 1 : 0;
    if (seeded) {
        // the gradients of h_n / c_n are what the step at T-1 reads as the incoming dh_rec / dc
        if (dh_n != nullptr) STMGCN_CUDA(cudaMemcpyAsync(dh_rec, dh_n, state_bytes, cudaMemcpyDeviceToDevice, st));
        else STMGCN_CUDA(cudaMemsetAsync(dh_rec, 0, state_bytes, st));
        if (dc_n != nullptr) STMGCN_CUDA(cudaMemcpyAsync(dc, dc_n, state_bytes, cudaMemcpyDeviceToDevice, st));
        else STMGCN_CUDA(cudaMemsetAsync(dc, 0, state_bytes, st));
    }
    const int grid_pw = (int)((ceil_div(rows, 8) < (int64_t)sm_count() * 4) ? ceil_div(rows, 8) : (int64_t)sm_count() * 4);
    for (int t = t_len - 1; t >= 0; --t) {
        for (int l = n_layers - 1; l >= 0; --l) {
            float* g_lt = gates + ((int64_t)(l * t_len + t)) * rows * h4;
            const float* c_t = cs + ((int64_t)(l * t_len + t)) * rh;
            const float* c_prev = t > 0 ? cs + ((int64_t)(l * t_len + t - 1)) * rh : (c0 ? c0 + (int64_t)l * rh : nullptr);
            const float* dh_in = (l == n_layers - 1) ? ((t == t_len - 1) ? d_top : nullptr) : dx_work;
            const bool l0 = (l == 0);
            size_t smem = (size_t)h4 * (1 + (l0 ? c_in : 0)) * sizeof(float);
            if (l0 && b_inner <= 2048) smem += (size_t)b_inner * sizeof(float);
            lstm_bwd_pointwise_kernel<<<grid_pw, 256, smem, st>>>(
                rows, hid, g_lt, c_t, c_prev, dh_in, dh_rec + (int64_t)l * rh, dc + (int64_t)l * rh,
                wgrad ? dbp + (int64_t)l * h4 : nullptr, l0 ? wx : nullptr, l0 ? dwx : nullptr, xo, s_gate, d_s, c_in, t,
                t_len, b_inner, l0 ? d_xo : nullptr, seeded);
            count_launch();
            if (int32_t rc = check_launch("lstm_bwd_pointwise")) return rc;
            // data gradients: [dx_below | dh_rec] = dA . wpt_l      (dA: rows x 4H, wpt_l: 4H x kd_l)
            ASegs a{};
            a.nseg = 1;
            a.segw = h4;
            a.lda = h4;
            a.seg[0] = g_lt;
            StoreSplitEpi epi;
            epi.dst0 = l0 ? nullptr : dx_work;
            epi.ld0 = hid;
            epi.w0 = l0 ? 0 : hid;
            epi.dst1 = dh_rec + (int64_t)l * rh;
            epi.ld1 = hid;
            const int nc = l0 ? hid : 2 * hid;
            const float* wpt_l = wpt + layer_off(l, hid);
            const int32_t rc = nc > 64 ? launch_tall<128>(a, rows, h4, wpt_l, nc, nc, epi, st, "lstm_bwd_data")
                                       : launch_tall<64>(a, rows, h4, wpt_l, nc, nc, epi, st, "lstm_bwd_data");
            if (rc) return rc;
        }
    }
    // after the step at t = 0, dh_rec / dc hold the gradients of h0 / c0 (also of a zero initial state)
    if (dh0 != nullptr) STMGCN_CUDA(cudaMemcpyAsync(dh0, dh_rec, state_bytes, cudaMemcpyDeviceToDevice, st));
    if (dc0 != nullptr) STMGCN_CUDA(cudaMemcpyAsync(dc0, dc, state_bytes, cudaMemcpyDeviceToDevice, st));
    // weight gradients: dwp_l (kd_l, 4H) += [h_below_t | h_{t-1}]^T dA summed over all (t, r)
    for (int l = 0; l < n_layers && wgrad; ++l) {
        ASegs a{};
        ReduceTime tm{};
        a.segw = hid;
        a.lda = hid;
        tm.n_t = t_len;
        tm.d_tstride = rows * h4;
        int s = 0;
        if (l > 0) {                           // input from the layer below, same step
            a.seg[s] = hs + ((int64_t)(l - 1) * t_len) * rh;
            tm.a_tstride[s] = rh;
            tm.a_shift[s] = 0;
            tm.a_t0[s] = nullptr;
            ++s;
        }
        a.seg[s] = hs + ((int64_t)l * t_len) * rh;          // h_{t-1} of this layer
        tm.a_tstride[s] = rh;
        tm.a_shift[s] = 1;
        tm.a_t0[s] = h0 ? h0 + (int64_t)l * rh : nullptr;
        ++s;
        a.nseg = s;
        const float* d = gates + ((int64_t)l * t_len) * rows * h4;
        if (int32_t rc = launch_reduce<256>(a, tm, rows, s * hid, d, h4, h4, dwp + layer_off(l, hid), h4, st, "lstm_wgrad"))
            return rc;
    }
    return 0;
}

int32_t stmgcn_lstm_bwd(int32_t t_len, int32_t n_layers, int64_t rows, int32_t hid, int32_t c_in, int64_t b_inner,
                        const float* xo, const float* s_gate, const float* wx, const float* wpt, const float* h0,
                        const float* c0, const float* cs, const float* hs, float* gates, const float* d_top,
                        float* dh_rec, float* dc, float* dx_work, float* d_s, float* dwx, float* dwp, float* dbp,
                        void* stream) {
    return stmgcn_lstm_bwd_ex(t_len, n_layers, rows, hid, c_in, b_inner, xo, s_gate, wx, wpt, h0, c0, cs, hs, gates, d_top,
                              dh_rec, dc, dx_work, d_s, dwx, dwp, dbp, nullptr, nullptr, nullptr, nullptr, nullptr, stream);
}

}  // extern "C"
