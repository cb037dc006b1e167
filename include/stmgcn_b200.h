/*
 * stmgcn_b200.h -- C ABI of libstmgcn_b200.so: the H100 (sm_90a) ST-MGCN hot path.
 *
 * The reference (underdoc-wang/ST-MGCN) has NO plugin / FFI / operator interface: its boundary is the
 * Python nn.Module surface (GCN.py:7-46, STMGCN.py:7-119).  This header is therefore the boundary a
 * binding for that surface calls into; each entry point names the reference lines whose arithmetic it
 * replaces.  The Python mirror of the reference modules (repo-root GCN.py / STMGCN.py) binds these with
 * ctypes (st-mgcn_b200/stmgcn_b200/_lib.py); INTEGRATION.md shows the stub.
 *
 * Conventions (SURVEY.md section 8(b)):
 *   - plain C types only: device pointers as void* / const float*, sizes as int64_t, flags as int32_t,
 *     the CUDA stream as void* (a cudaStream_t; NULL = legacy default stream).
 *   - every entry returns int32_t: 0 ok, >0 a cudaError_t, <0 an argument / shape / alignment error.
 *     stmgcn_last_error() returns a thread-local message for the last non-zero return.
 *   - a negative return means nothing was enqueued: the call checks all its arguments before its first launch.
 *   - the library never allocates, never frees and owns no memory; all tensors and workspaces are
 *     caller-owned device buffers.
 *   - entries enqueue on the given stream and return; no device synchronisation inside.
 *   - all feature tensors are fp32, "node-major": rows r = n * B + b (region n outer, window b inner),
 *     features contiguous.  (N, B, p) row-major == (N, B*p) row-major == (N*B, p) row-major.
 *   - non-finite values propagate as torch's IEEE arithmetic does: a NaN or +-Inf in data, weights or supports reaches
 *     every result that depends on it and no other.  ReLU is torch's (relu(NaN) = NaN; its backward masks with
 *     out <= 0, so it passes the gradient at NaN), and the tensor-core LSTM's capped exponential keeps a NaN argument.
 *     Three deviations from a dense torch restatement, by design:
 *       spmm_stored_entries_only -- the SpMM multiplies stored entries only, so a NaN in X reaches the rows with a
 *         stored entry in its column, not every row (a dense product forms 0 * NaN);
 *       inf_through_split_operands -- the 3xTF32 / 3xBF16 operand splits form lo = Inf - Inf = NaN, so an Inf operand
 *         of a tensor-core product gives NaN where torch gives +-Inf (relu(-Inf) = 0 becomes NaN): still non-finite;
 *       products_skipped_with_a_zero_initial_state -- without h0 the tensor-core LSTM skips W_hh . 0 at t = 0, so a
 *         NaN W_hh leaves step 0 finite (the exact-fp32 LSTM forms the product, as torch does).
 */
#ifndef STMGCN_B200_H_
#define STMGCN_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define STMGCN_ABI_VERSION 8

/* error codes < 0 */
#define STMGCN_ERR_ARG      (-1)   /* null pointer / bad enum */
#define STMGCN_ERR_SHAPE    (-2)   /* size out of the supported range */
#define STMGCN_ERR_ALIGN    (-3)   /* pointer or leading dimension not aligned as required */
#define STMGCN_ERR_STATE    (-4)   /* the call could not set up what it needs (e.g. a TMA descriptor) */

/* activation of the projection epilogue (GCN.py:42; the reference passes nn.ReLU or None) */
#define STMGCN_ACT_NONE 0
#define STMGCN_ACT_RELU 1

int32_t     stmgcn_abi_version(void);
const char* stmgcn_last_error(void);
/* number of SMs of the current device (grid sizing is done inside; exposed for bench.py's records) */
int32_t     stmgcn_sm_count(void);
/* how many kernels this library has launched in this process (bench.py "gpu_launches") */
int64_t     stmgcn_launch_count(void);

/* ---- K1: one Chebyshev recurrence step on the features --------------------------------------------
 * Y = alpha * op(A) X + beta * Z + gamma * U,   X/Z/U/Y: (N, f_total) fp32 row-major.
 * op(A) is the N x N sparse support GCN.forward receives as A[k] (GCN.py:24-36), given as the caller's device CSR:
 * rowptr (n+1 int32, non-decreasing from 0), colidx (int32 column indices) and vals (fp32), nnz = rowptr[n] entries.
 * colidx and vals may be NULL only when the matrix has no entries.  Passing the CSR of A^T makes op(A) = A^T.
 * Z and U may be NULL (their terms vanish).  Forward step k (replaces the dense einsum GCN.py:35 and the
 * matrix recurrence GCN.py:134): op(A) = L~, alpha=2 (1 for k=1), beta=-1, Z=T_{k-2}X.  Backward (adjoint Clenshaw,
 * SURVEY.md section 8(a)): op(A) = L~^T, U = U_k.  Y must not alias X. */
int32_t stmgcn_cheb_spmm_step(int64_t n, const int32_t* rowptr, const int32_t* colidx, const float* vals, float alpha,
                              const float* x, float beta, const float* z, float gamma, const float* u, float* y,
                              int64_t f_total, void* stream);

/* The same step with the GATHERED operand read from a bf16 copy (the bf16-arithmetic mode of the bf16-quoted
 * configurations: the kernel's time is its gather volume): x16 (N, f_total) bf16; z, u, y stay fp32; y16 (nullable) receives
 * the bf16 copy of y for the next step.  f_total must be a multiple of 8.  stmgcn_to_bf16 makes the first copy
 * (count elements, a multiple of 8). */
int32_t stmgcn_cheb_spmm_step16(int64_t n, const int32_t* rowptr, const int32_t* colidx, const float* vals,
                                float alpha, const void* x16, float beta, const float* z, float gamma, const float* u,
                                float* y, void* y16, int64_t f_total, void* stream);
int32_t stmgcn_to_bf16(const float* x, void* y16, int64_t count, void* stream);

/* ---- K1b: gradient of a support's stored values (CSR SDDMM) ------------------------------------------
 *   dvals[e] += sum_t coef[t] * < A_t[i, :], B_t[j, :] >   for every stored entry e = (i, j) of the CSR (rowptr, colidx),
 * i the row that owns e and j = colidx[e]; nnz = rowptr[n] entries, dvals in the CSR's storage order (a repeated (i, j)
 * gets the same value at each of its entries).  A_t, B_t: (N, f_total) fp32 row-major, nterms = 1..8 term pairs given as
 * host arrays a[nterms], b[nterms] of device pointers and coef[nterms] of host floats.  Chebyshev chain X with
 * T_1 = X T_0, T_k = 2 X T_{k-1} - T_{k-2}: A_t = G_k (the total adjoint dL/dT_k), B_t = T_{k-1}, coef 1 for k = 1 and 2
 * otherwise; a generic support S = A x: one term, A_0 = dL/dS, B_0 = x.  round_b_bf16 = 1 rounds every B element to bf16
 * (to nearest even) before the product: the operand stmgcn_cheb_spmm_step16 multiplied by.
 * f_total % 4 == 0 takes the float4 kernel (every A_t and B_t 16-byte aligned, else STMGCN_ERR_ALIGN), any other width
 * the scalar one.  Column tiles: tiles = ceil(f_total / 128) (float4) or ceil(f_total / 32) (scalar); with tiles > 1,
 * work (tiles * nnz floats, work_count >= that) receives one partial per tile and entry and a second launch adds them
 * to dvals in tile order; with tiles == 1 work may be NULL.  Every sum has one owner in a fixed order: two calls with
 * the same inputs give bit-identical dvals.  A_t and B_t may alias one another.  dvals (nnz floats) and work (work_count
 * floats) share no byte with any A_t / B_t (n * f_total floats each) or with each other: the byte ranges are checked.
 * nnz == 0 enqueues nothing (colidx and dvals may then be NULL). */
int32_t stmgcn_csr_sddmm(int64_t n, const int32_t* rowptr, const int32_t* colidx, int64_t nnz, int32_t nterms,
                         const float* const* a, const float* const* b, const float* coef, int32_t round_b_bf16,
                         int64_t f_total, float* work, int64_t work_count, float* dvals, void* stream);

/* ---- K1d: gradient of dense support slices (GCN.py:35 differentiated in A[k]) ---------------------------------------
 *   da[k][i][j] = sum_f U_k[i][f] * x[j][f]     (dA_k = U_k x^T),   k < ks, i, j < n, f < f_total
 * U_k = u + k * u_stride and x are (n, f_total) fp32 row-major: U_k = dL/dS_k, the gradient of the slice's product
 * S_k = A_k x (stmgcn_proj_bwd's u, taken before the adjoint Clenshaw overwrites it), x the features it multiplied.
 * da: (ks, n, n) row-major, OVERWRITTEN (not accumulated).  1 <= ks <= 8, 1 <= n < 2^24, 1 <= f_total < 2^31,
 * u_stride >= 0; segments of u may overlap one another, but da shares no byte with u (its ks segments) or x (checked).
 * 3xTF32 on the tensor cores (fp32-grade, as the projection); 16-byte loads when f_total % 4 == 0 and u, x (and, ks > 1,
 * u_stride % 4 == 0) allow them, scalar loads otherwise; any n and f_total.  One launch.  Every element has one owner
 * and a fixed summation order: two calls with the same inputs give bit-identical da.  A NaN in row i of U_k makes row i
 * of dA_k NaN, a NaN in row j of x column j of every dA_k; an Inf gives NaN (inf_through_split_operands). */
int32_t stmgcn_dense_support_grad(int64_t n, int64_t f_total, int32_t ks, const float* u, int64_t u_stride,
                                  const float* x, float* da, void* stream);

/* ---- K1f: gradient of a DENSE Chebyshev recurrence matrix (a learnable adjacency multiplied dense) ------------------
 *   out[i][j] = sum_t coef[t] * sum_f A_t[i][f] * B_t[j][f]      (out = sum_t coef_t A_t B_t^T),   i, j < n, f < f_total
 * stmgcn_csr_sddmm's sum over every n x n entry: chain X with T_1 = X T_0, T_k = 2 X T_{k-1} - T_{k-2} gives
 * dX = sum_k c_k G_k T_{k-1}^T with A_t = G_k (the total adjoint dL/dT_k), B_t = T_{k-1}, coef 1 for k = 1 and 2 after.
 * A_t, B_t: (n, f_total) fp32 row-major, nterms = 1..8 pairs as host arrays a[nterms], b[nterms] of device pointers and
 * coef[nterms] of host floats, read at enqueue.  round_b16 = 1 rounds every B element to bf16 (to nearest even) before
 * the product: the operand stmgcn_dense_mm_step16 multiplied by.  out: (n, n) row-major, OVERWRITTEN.
 * 1 <= n < 2^24, 1 <= f_total < 2^31; A_t and B_t may alias one another, out shares no byte with any (checked).
 * 3xTF32 on the tensor cores with K1e's rounded split, each 32-term block's product added times coef_t into an fp32
 * register total (fp32-grade where the products cancel); 16-byte loads when f_total % 4 == 0 and every A_t, B_t is
 * 16-byte aligned, scalar loads otherwise.  One launch.  Every element has one owner and a fixed summation order (the
 * terms in order, each over f in order): two calls with the same inputs give bit-identical out.  A NaN in row i of an
 * A_t makes row i of out NaN, a NaN in row j of a B_t column j; an Inf gives NaN (inf_through_split_operands). */
int32_t stmgcn_dense_chain_grad(int64_t n, int64_t f_total, int32_t nterms, const float* const* a, const float* const* b,
                                const float* coef, int32_t round_b16, float* out, void* stream);

/* ---- K1e: the recurrence step with a DENSE support matrix (GCN.py:35 as the reference computes it) ------------------
 *   Y = alpha * op(A) X + beta * Z + gamma * U      on (n, f_total) fp32 row-major X, Z, U, Y
 * stmgcn_cheb_spmm_step's step for a matrix held dense: a (n x n) fp32 row-major with leading dimension lda >= n;
 * op(A) = A (transpose = 0) or A^T (transpose = 1).  Z and U may be NULL (their terms vanish).  Y may BE U (the adjoint
 * Clenshaw's y = u[k], gamma = 1) but shares no other byte with U, and none with X, Z or a (checked).
 * 1 <= n < 2^24, lda < 2^31, 1 <= f_total < 2^31.  3xTF32 on the tensor cores with a rounded split, each 32-term block
 * added into an fp32 register total (fp32-grade, also where the products cancel); 16-byte loads when n, lda and
 * f_total are multiples of 4 and every pointer is 16-byte aligned, scalar loads otherwise.  One launch.  Every element has
 * one owner and a fixed summation order: two calls with the same inputs give bit-identical y.
 * Non-finite values: the product is dense, as the reference's einsum, so it forms 0 * NaN: a NaN in row j of X reaches
 * every row of Y in its columns (spmm_stored_entries_only does not apply); an Inf operand gives NaN
 * (inf_through_split_operands). */
int32_t stmgcn_dense_mm_step(int64_t n, const float* a, int64_t lda, int32_t transpose, float alpha, const float* x,
                             float beta, const float* z, float gamma, const float* u, float* y, int64_t f_total,
                             void* stream);

/* The same step multiplying the bf16 copy x16 (n, f_total) bf16 (the bf16-arithmetic mode, as stmgcn_cheb_spmm_step16):
 * a bf16 value is exact in tf32, so two tensor-core passes A_hi x16 + A_lo x16; z, u, y stay fp32, and y16 (nullable)
 * receives the bf16 copy of y (round to nearest even, as stmgcn_to_bf16).  f_total must be a multiple of 8 and x16, y,
 * y16, z, u 16-byte aligned; y16 shares no byte with x16, y, z, u or a. */
int32_t stmgcn_dense_mm_step16(int64_t n, const float* a, int64_t lda, int32_t transpose, float alpha, const void* x16,
                               float beta, const float* z, float gamma, const float* u, float* y, void* y16,
                               int64_t f_total, void* stream);

/* ---- K1c: the supports of a learnable adjacency on a fixed sparsity pattern ----------------------------------------
 * The pattern is an n x n CSR (rowptr, colidx; nnz = rowptr[n] entries, no repeated (i, j)) and its transpose's structure
 * rowptr_t, colidx_t with perm_t: CSR^T position p holds CSR entry perm_t[p].  widx (int32 per pattern entry) gives the
 * entry's index in w, or -1 for a slot with no weight of its own (a diagonal slot that holds only the diagonal term);
 * it maps onto [0, nnz_w) one to one.  widx NULL: the pattern's entries are w's, in order (nnz_w == nnz).  w (fp32): the
 * edge weights; D below sums them per row (d_out) or per column (d_in), over the entries that have one.  kind:
 *   STMGCN_NORM_CHEBYSHEV  vals[e] = -scale * D^-1/2 A D^-1/2 + (scale - 1) I     (scale = 2 / lambda_max, finite)
 *   STMGCN_NORM_LOCALPOOL  vals[e] =  I + D^-1/2 A D^-1/2
 *   STMGCN_NORM_DIFFUSION  vals[e]   = P_b^T = w * d_in^-1[col]   (CSR order)
 *                          vals_t[p] = P_f^T = w * d_out^-1[row]  (CSR^T order), an infinite d^-1 taken as 0 (GCN.py:100-104)
 * D^-1/2 is torch's pow(D, -0.5): +inf at a zero sum, NaN at a negative one.  The backward is torch autograd's chain
 * through these formulas, non-finite values included: at a zero sum the degree term is NaN (0 * -inf for DIFFUSION, whose
 * masked reciprocal passes 0 into pow(D, -1)'s -D^-2), so a row or column of stored entries that sum to zero (stored
 * zeros, say) gets NaN in dw; an empty row or column has no entry to pass it to.  The diagonal terms go into the pattern's
 * diagonal slot of each row (added to a stored self-loop); the caller's pattern has one in every row for the symmetric
 * kinds (unless scale == 1 for CHEBYSHEV).  vals_t / dvals_t are for DIFFUSION only (NULL otherwise).
 * Every sum has one owner and a fixed order (no float atomics): two calls give bit-identical results.  Nothing is
 * allocated and nothing synchronises; the workspace (work_count floats) needs no initialisation: 2n floats forward,
 * 3n + nnz backward.  Outputs (work, vals, vals_t, dw) share no byte with any input or with one another (checked).  The
 * forward enqueues 2 launches (none when nnz == 0), the backward 3 (none when nnz_w == 0). */
#define STMGCN_NORM_CHEBYSHEV 0
#define STMGCN_NORM_LOCALPOOL 1
#define STMGCN_NORM_DIFFUSION 2
int32_t stmgcn_adj_norm_fwd(int32_t kind, int64_t n, const int32_t* rowptr, const int32_t* colidx, const int32_t* rowptr_t,
                            const int32_t* colidx_t, const int32_t* perm_t, int64_t nnz, const int32_t* widx, const float* w,
                            int64_t nnz_w, float scale, float* work, int64_t work_count, float* vals, float* vals_t,
                            void* stream);
/* The backward: dw (nnz_w, overwritten) from the values' gradients dvals (CSR order) and, DIFFUSION, dvals_t (CSR^T
 * order): the direct term plus the degree terms (a row segment sum over the CSR, a column segment sum over the CSR^T,
 * then one pass over the entries).  Same pattern, w and scale as the forward. */
int32_t stmgcn_adj_norm_bwd(int32_t kind, int64_t n, const int32_t* rowptr, const int32_t* colidx, const int32_t* rowptr_t,
                            const int32_t* colidx_t, const int32_t* perm_t, int64_t nnz, const int32_t* widx, const float* w,
                            int64_t nnz_w, float scale, const float* dvals, const float* dvals_t, float* work,
                            int64_t work_count, float* dw, void* stream);

/* A pattern's values <-> the dense matrix they form (a learnable adjacency multiplied dense).  The pattern: CSR rowptr
 * (n + 1) and colidx (nnz) int32 -- a learnable adjacency's CSR, or its CSR^T (rowptr_t, colidx_t) for the values in
 * CSR^T order (diffusion's P_f^T).  Columns may be unsorted within a row and entries repeated.
 * scatter: dense (n x n fp32 row-major) OVERWRITTEN with the matrix: zeros, plus each entry's value added at (i, j) in
 *   entry order (repeats add up as CSR applies them: ((0 + v_e0) + v_e1) + ...).  One launch, also when nnz == 0.
 * gather: dvals[e] = dense[i][colidx[e]] for every entry e = (i, j), OVERWRITTEN: the values' gradient from the
 *   matrix's.  One launch; none when nnz == 0.
 * 1 <= n < 2^24, 0 <= nnz < 2^31; column indices in [0, n) (not checked: the caller's pattern, as for the SpMM).  The
 * output shares no byte with the pattern or the input (checked).  Plain fp32 adds and copies: NaN and Inf pass as
 * they are, and a stored zero is an entry like any other. */
int32_t stmgcn_pattern_scatter(int64_t n, const int32_t* rowptr, const int32_t* colidx, int64_t nnz, const float* vals,
                               float* dense, void* stream);
int32_t stmgcn_pattern_gather(int64_t n, const int32_t* rowptr, const int32_t* colidx, int64_t nnz, const float* dense,
                              float* dvals, void* stream);

/* ---- input pipeline: training windows gathered from a device-resident series (Data_Container.py:114-146) ----------
 *   obs[k, t, :] = series[wrap(first + k - lags[t]), :],   y[k, :] = series[first + k, :]      (k < b, t < t_len)
 * A row is `row` = N*C fp32 values; series is (s_len, row) row-major; obs is (b, t_len, row); y is (b, row).
 * wrap(r) = r + s_len for -s_len <= r < 0 (numpy's negative indexing, which the reference's periodic windows hit).
 * lags: host array of t_len int32 values, read at enqueue.  A plain copy: output bits equal input bits (NaN payloads, -0).
 * Requires s_len, row, b > 0, 0 < t_len <= 2048, 0 <= first, first + b <= s_len, every lags[t] >= 0 and
 * first - lags[t] >= -s_len; obs and y share no byte with the series or with each other.  One launch: 16-byte loads and
 * stores when row % 4 == 0 and series, obs and y are 16-byte aligned, scalar ones otherwise. */
int32_t stmgcn_window_gather(const float* series, int64_t s_len, int64_t row, const int32_t* lags, int32_t t_len,
                             int64_t first, int64_t b, float* obs, float* y, void* stream);

/* ---- layout: obs (B,T,N,C) -> node-major (STMGCN.py:36,39 sum over C + permute; :47 row order) ----
 * xo: (N,B,T,C) copy of obs;  xt: (N,B,T) = sum_c obs.  xo may be NULL when C == 1 (xt is then xo). */
int32_t stmgcn_obs_to_node_major(const float* obs, float* xo, float* xt, int64_t b, int64_t t,
                                 int64_t n, int64_t c, void* stream);
/* Its adjoint (the gradient w.r.t. obs): d_obs[b,t,n,c] = d_xo[n,b,t,c] + d_xt[n,b,t], d_obs (B,T,N,C) overwritten.
 * d_xo (N,B,T,C) and d_xt (N,B,T) may each be NULL (that term vanishes). */
int32_t stmgcn_obs_grad(const float* d_xo, const float* d_xt, float* d_obs, int64_t b, int64_t t, int64_t n, int64_t c,
                        void* stream);

/* ---- K2: stacked-K projection (GCN.py:37-42) --------------------------------------------------------
 * out[r,:] = act( sum_k S_k[r,:] W[k*p:(k+1)*p, :] + bias ),  r in [0, rows), S_k = s + k*stride_k
 * (rows x p, row-major), W: (ks*p, q) row-major, bias: q or NULL.  ks <= 8 and q <= 8192 in both directions.
 * Optional gate pooling (STMGCN.py:41-42), requires q == p: pool[(r % b_inner)*q + j] +=
 * S_0[r,j] + out[r,j]  (caller zeroes pool; sum over regions of x_hat, not yet divided by N). */
int32_t stmgcn_proj_fwd(const float* s, int64_t stride_k, int32_t ks, int64_t rows, int32_t p,
                        const float* w, const float* bias, int32_t q, int32_t act, float* out,
                        float* pool, int64_t b_inner, const float* wimg, void* stream);
/* Tensor-core operand images of W (ks*64, 64) for p = q = 64, ks <= 8 (3xTF32: every fp32 operand split into tf32 hi + lo, three wgmma passes):
 * img_fwd: ks*64*64*2 floats; img_bwd (may be NULL): one 2*2*256*32-float image per group of 4 supports (two images
 * when ks > 4), ZERO-FILLED by the caller (rows beyond ks*64 stay zero).  Passing wimg / wimg_t != NULL to stmgcn_proj_fwd / _bwd selects the wgmma kernels when
 * p = q = 64 (and, for the backward, a full d_out and u are given); otherwise the exact-FFMA kernels run. */
int32_t stmgcn_proj_pack_tc(const float* w, int32_t ks, float* img_fwd, float* img_bwd, void* stream);
/* backward of the projection.  dZ = dOut (.) [out > 0] (act = RELU) with dOut either a full (rows, q)
 * tensor (d_out) or, when d_out_bcast != NULL, the broadcast dOut[r,:] = d_out_bcast[(r % b_inner), :] *
 * bcast_scale (the mean-pool adjoint dz/N, STMGCN.py:42).  dz_work: (rows, q) workspace receiving dZ.
 * Accumulates (+=) dw (ks*p, q) and dbias (q, may be NULL) -- caller zeroes them -- and, if u != NULL,
 * writes U_k = dZ W_k^T into u + k*stride_u (rows x p); wt is then W^T, (q, ks*p) row-major.
 * dw may be NULL (a frozen W): no dW launch on either path (neither proj_wgrad_tc_kernel nor the FFMA dW); dz_work and u
 * are written as before.  dw, dbias and u all NULL is STMGCN_ERR_ARG. */
int32_t stmgcn_proj_bwd(const float* s, int64_t stride_k, int32_t ks, int64_t rows, int32_t p,
                        const float* wt, int32_t q, int32_t act, const float* out, const float* d_out,
                        const float* d_out_bcast, float bcast_scale, int64_t b_inner, float* dz_work,
                        float* dw, float* dbias, float* u, int64_t stride_u, const float* wimg_t,
                        void* stream);

/* ---- K3a: context gate (STMGCN.py:42-43) -----------------------------------------------------------
 * z = pool / n_regions; a1 = z fcw^T + fcb; s = sigmoid(relu(a1) fcw^T + fcb).  All (B, T); fcw (T,T).
 * Both directions take T <= 2048 (the backward's shared memory); beyond it STMGCN_ERR_SHAPE. */
int32_t stmgcn_gate_fwd(const float* pool, int64_t b, int32_t t, int64_t n_regions, const float* fcw,
                        const float* fcb, float* z, float* a1, float* s, void* stream);
/* d_s -> d_fcw (+=), d_fcb (+=), d_z (B,T).  d_fcw and d_fcb may be NULL together (a frozen fc): d_z only.  One of
 * them NULL without the other is STMGCN_ERR_ARG. */
int32_t stmgcn_gate_bwd(const float* d_s, const float* z, const float* a1, const float* s, int64_t b,
                        int32_t t, const float* fcw, float* d_fcw, float* d_fcb, float* d_z, void* stream);

/* ---- K3b (exact fp32, any H <= 128): shared-weight LSTM over the whole sequence (STMGCN.py:44, :47-50) ---------------
 * The CUDA-core path for every shape the tensor-core kernels below do not cover (H != 64, C > 4 or T > 64), and the
 * on-device reference the parity tests compare them with.  Weights are passed packed, H = hid, columns gate-interleaved
 * col = 4*unit + gate (gate order i,f,g,o):
 *   wx   : (C, 4H)      = W_ih_l0^T                      (layer-0 input weights)
 *   wp   : flat, layer l's block wp_l (kd_l, 4H) = W_hh_0^T (l = 0, kd_0 = H) or [W_ih_l^T ; W_hh_l^T] (l > 0,
 *          kd_l = 2H); the blocks lie back to back, so wp_l starts 4H*H*(l == 0 ? 0 : 2l - 1) floats in
 *   wpt  : flat, layer l's block (4H, kd_l) = wp_l^T at the same offset (backward data operand)
 *   bp   : (L, 4H)      = b_ih_l + b_hh_l
 * State / tape tensors, rows r = n*B + b, fp32 row-major:
 *   hs, cs: (L, T, R, H);  gates: (L, T, R, 4H) post-activation, gate-interleaved (NULL in inference);
 * xo: (R, T, C) node-major observations, s_gate: (B, T) context gate (the modulation xo * s is fused into the layer-0
 * input read, STMGCN.py:44).  h0/c0: (L, R, H) or NULL (zeros, STMGCN.py:53-57).
 * Limits: H % 4 == 0, H <= 128, C <= 4, L <= 8. */
int32_t stmgcn_lstm_fwd(int32_t t_len, int32_t n_layers, int64_t rows, int32_t hid, int32_t c_in, int64_t b_inner,
                        const float* xo, const float* s_gate, const float* wx, const float* wp, const float* bp,
                        const float* h0, const float* c0, float* hs, float* cs, float* gates, void* stream);
/* BPTT over all timesteps, then the weight gradients.  d_top: (R, H) gradient of hs[L-1][T-1].
 * Workspaces: dh_rec, dc: (L, R, H); dx_work: (R, H).  No initialisation is needed: the step t = T-1 treats the incoming
 * dh_rec / dc as zero without reading them (ST_MGCN discards h_n / c_n, STMGCN.py:113); stmgcn_lstm_bwd_ex seeds them.
 * gates is overwritten IN PLACE with the pre-activation gradients dA, so it serves one backward only.
 * Accumulates (+=; caller zeroes): d_s (B,T) = sum_{n,c} dxmod * xo (gate adjoint, STMGCN.py:44), dwx (C,4H),
 * dwp (laid out like wp) += [h_below_t | h_{t-1}]^T dA summed over all (t, r), dbp (L, 4H).
 * dwx, dwp and dbp may be NULL together (frozen LSTM weights): the per-layer reduce GEMMs and the bias / dwx sums are
 * skipped, everything else is as with them.  A mix of NULL and non-NULL is STMGCN_ERR_ARG. */
int32_t stmgcn_lstm_bwd(int32_t t_len, int32_t n_layers, int64_t rows, int32_t hid, int32_t c_in, int64_t b_inner,
                        const float* xo, const float* s_gate, const float* wx, const float* wpt, const float* h0,
                        const float* c0, const float* cs, const float* hs, float* gates, const float* d_top,
                        float* dh_rec, float* dc, float* dx_work, float* d_s, float* dwx, float* dwp, float* dbp,
                        void* stream);
/* stmgcn_lstm_bwd with the gradients at the model's inputs and recurrent state (nn.LSTM semantics).  All (L, R, H)
 * row-major, each NULL when unused:
 *   dh_n, dc_n: incoming gradients of the final state h_n = hs[:, T-1] / c_n = cs[:, T-1] (dh_n[L-1] adds to d_top);
 *   dh0, dc0  : overwritten with the gradients of h0 / c0 (of the zero initial state when h0 / c0 are NULL).
 * d_xo: (R, T, C) overwritten with the gradient of xo (d xo = dxmod * s[b, t]), or NULL.
 * With every extra NULL this is stmgcn_lstm_bwd, launch for launch; dwx, dwp, dbp may be NULL together as there. */
int32_t stmgcn_lstm_bwd_ex(int32_t t_len, int32_t n_layers, int64_t rows, int32_t hid, int32_t c_in, int64_t b_inner,
                           const float* xo, const float* s_gate, const float* wx, const float* wpt, const float* h0,
                           const float* c0, const float* cs, const float* hs, float* gates, const float* d_top,
                           float* dh_rec, float* dc, float* dx_work, float* d_s, float* dwx, float* dwp, float* dbp,
                           const float* dh_n, const float* dc_n, float* dh0, float* dc0, float* d_xo, void* stream);

/* ---- K3b on the tensor cores (H = 64, C <= 4): bf16-plane LSTM without a gate tape -----------------------------
 * Same arithmetic contract as stmgcn_lstm_fwd/_bwd (STMGCN.py:44, :47-50; nn.LSTM semantics, fp32 state and
 * accumulation), different tape:
 *   hp : (L, T, P, R, 64) bf16 -- every hidden state as P planes; P = 2: hi = bf16(h), lo = bf16(h - hi) (3-pass
 *        "3xBF16" products, ~2^-18 operand error: fp32-grade, the 1e-4 parity bar holds with >10x margin);
 *        P = 1: hi only, single-pass bf16 products (the arithmetic of the bf16-quoted BASELINE configs).
 *   cs : (L, T, ceil(R/128)*128, 64) fp32, tile-blocked (element (r,u) at (((r/128)*16 + u/4)*128 + r%128)*4 + u%4).
 *        Of every tile-blocked tensor only the first R rows mean anything; the padding rows of the tile-blocked inputs
 *        c0 and d_top are never read.
 * No gate tape: the backward recomputes the gates from hp (which it needs anyway for the weight gradients).
 * Weights are passed as flat operand images:
 *   wimg : layer l's resident image (tiles [(segment, plane)] of [256 gate-interleaved columns][64 k] bf16, 128-byte
 *          swizzled; layer 0: 64 KB, layers > 0: 128 KB), back to back, so layer l starts 65536*(l == 0 ? 0 : 2l - 1)
 *          bytes in;
 *   bias : (L, 256) = b_ih_l + b_hh_l gate-interleaved (col = 4*unit + gate);
 *   wih_t: (C, 256) = W_ih_l0^T gate-interleaved.
 * h0p: (L, P, R, 64) bf16 planes of the initial hidden state and c0: (L, R_pad, 64) fp32 tile-blocked, or both NULL
 * (zeros, STMGCN.py:53-57).  C <= 4, L <= 8.
 * stmgcn_lstm16_pack turns layer `layer`'s nn.LSTM parameters (native layout: w_ih (256, in), w_hh (256, 64), b_ih,
 * b_hh (256), gate order i,f,g,o) into that layer's slot of wimg and bias and, for layer 0, into wih_t. */
int32_t stmgcn_lstm16_pack(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, int32_t layer,
                           int32_t c_in, void* wimg, float* bias, float* wih_t, void* stream);
/* Forward through all layers and timesteps: one launch per layer, bottom-up (layer l reads the hp planes of layer
 * l - 1).  A tile's rows never mix with other tiles', so each CTA walks its own tiles through time inside a layer's
 * launch, keeping h_{t-1} in shared memory.  At t = T-1 the fp32 hidden state is also written: into h_n (L, R, 64) when
 * h_n != NULL, else for the top layer into h_top (R, 64) -- the (N,B,H) operand of the spatial GCN (STMGCN.py:50, :114). */
int32_t stmgcn_lstm16_fwd(int32_t t_len, int32_t n_layers, int64_t rows, int32_t c_in, int64_t b_inner, int32_t planes,
                          const float* xo, const float* s_gate, const void* wimg, const float* bias, const float* wih_t,
                          const void* h0p, const float* c0, void* hp, float* cs, float* h_top, float* h_n,
                          void* stream);

/* grid (CTAs) the lstm16 kernels use for `rows` rows: the number of weight-gradient scratch slices */
int32_t stmgcn_lstm16_grid(int64_t rows);
/* BPTT through all layers and timesteps, T <= 64.  Per layer, top-down: one launch over T-1 .. 0 that recomputes the
 * gates from hp, forms dA, accumulates the weight and bias gradients and propagates [dx_below | dh_prev]; then one
 * launch that sums the layer's weight-gradient slices.  d_top: (R_pad, 64) tile-blocked gradient of the top layer's
 * last hidden state.
 * Workspaces (tile-blocked, R_pad = ceil(R/128)*128 rows; none needs initialisation):
 *   dh_rec, dc: (R_pad, 64);   dx_work: (min(2, L-1), T, R_pad, 64), the dx one layer hands to the layer below (may be
 *   NULL when L = 1);   dw_scratch: (stmgcn_lstm16_grid(rows), 128*256);   dbp: (L, 256);
 *   zero_tile: 16 KB of zeros (the h_prev operand at t = 0 without an initial state).
 * Accumulates (+=; caller zeroes) d_s (B,T) = sum_{n,c} dxmod * xo (gate adjoint, STMGCN.py:44).  Overwrites grads: one
 * flat buffer in nn.LSTM parameter order, per layer d_w_ih (256, in_l) | d_w_hh (256, 64) | d_b_ih (256) | d_b_hh (256).
 * grads may be NULL (frozen LSTM weights), and dw_scratch and dbp with it: no weight or bias gradients for any layer --
 * each layer's launch runs the kernel variant without the weight-gradient stage and the slice-sum launch is skipped.
 * Every other output is bit-identical to the call with grads. */
int32_t stmgcn_lstm16_bwd(int32_t t_len, int32_t n_layers, int64_t rows, int32_t c_in, int64_t b_inner, int32_t planes,
                          const float* xo, const float* s_gate, const void* wimg, const float* bias, const float* wih_t,
                          const void* h0p, const float* c0, const void* hp, const float* cs, const float* d_top,
                          float* dh_rec, float* dc, float* dx_work, float* dw_scratch, float* dbp, const void* zero_tile,
                          float* d_s, float* grads, void* stream);
/* stmgcn_lstm16_bwd with the gradients at the model's inputs and recurrent state.  dh_n, dc_n, dh0, dc0: (L, R_pad, 64)
 * fp32 tile-blocked like c0, each NULL when unused; the padding rows of dh_n / dc_n are never used, those of dh0 / dc0
 * are unspecified.
 *   dh_n, dc_n: incoming gradients of the final state (dh_n[L-1] adds to d_top), copied into dh_rec / dc before each
 *               layer's launch (the other one zeroed when only one is given);
 *   dh0, dc0  : overwritten with the gradients of the initial state (of the zero state when h0p / c0 are NULL);
 *   d_xo      : (R, T, C) overwritten with the gradient of xo, or NULL.
 * With every extra NULL this is stmgcn_lstm16_bwd, launch for launch; grads (with dw_scratch, dbp) may be NULL as there. */
int32_t stmgcn_lstm16_bwd_ex(int32_t t_len, int32_t n_layers, int64_t rows, int32_t c_in, int64_t b_inner, int32_t planes,
                             const float* xo, const float* s_gate, const void* wimg, const float* bias, const float* wih_t,
                             const void* h0p, const float* c0, const void* hp, const float* cs, const float* d_top,
                             float* dh_rec, float* dc, float* dx_work, float* dw_scratch, float* dbp, const void* zero_tile,
                             float* d_s, float* grads, const float* dh_n, const float* dc_n, float* dh0, float* dc0,
                             float* d_xo, void* stream);

/* ---- fusion over graphs + output FC (STMGCN.py:116-118) ------------------------------------------
 * feat = sum_m g[m] (each (R, G) node-major); y[b, n, c] = feat[n*B+b, :] . fcw[c, :] + fcb[c].
 * M <= 8.  Both directions take C*G + C <= 12288 (the backward's 48 KB shared-memory accumulator). */
int32_t stmgcn_fuse_out_fwd(const float* const* g, int32_t m, int64_t n, int64_t b, int32_t gdim,
                            int32_t c, const float* fcw, const float* fcb, float* feat, float* y,
                            void* stream);
/* d_y (B,N,C) -> d_feat (R,G), d_fcw (C,G) +=, d_fcb (C) +=.  d_fcw and d_fcb may be NULL together (a frozen output fc):
 * d_feat only.  One of them NULL without the other is STMGCN_ERR_ARG. */
int32_t stmgcn_fuse_out_bwd(const float* d_y, const float* feat, int64_t n, int64_t b, int32_t gdim,
                            int32_t c, const float* fcw, float* d_feat, float* d_fcw, float* d_fcb,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STMGCN_B200_H_ */
