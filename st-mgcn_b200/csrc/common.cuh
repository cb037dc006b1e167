// Shared host/device helpers for libstmgcn_b200.so (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/stmgcn_b200.h"

namespace stmgcn {

// ---- error reporting across the C boundary (no exceptions; thread-local message) -------------------
void set_error(const char* fmt, ...);
int32_t fail(int32_t code, const char* fmt, ...);
int32_t check_launch(const char* what);        // cudaGetLastError() only -- never synchronises
void count_launch(int n = 1);
int sm_count();
int32_t ensure_dyn_smem(const void* kernel, size_t bytes);   // per-(kernel, device) cudaFuncAttributeMaxDynamicSharedMemorySize

#define STMGCN_REQUIRE(cond, code, ...)                                   \
    do {                                                                  \
        if (!(cond)) return ::stmgcn::fail((code), __VA_ARGS__);          \
    } while (0)

#define STMGCN_CUDA(expr)                                                                     \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess)                                                                \
            return ::stmgcn::fail((int32_t)_e, "%s failed: %s", #expr, cudaGetErrorString(_e)); \
    } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
// whether the byte ranges [p, p + pb) and [q, q + qb) share a byte (a NULL or empty range shares none): the entry points'
// check that an output does not alias an input
static inline bool overlaps(const void* p, int64_t pb, const void* q, int64_t qb) {
    if (p == nullptr || q == nullptr || pb <= 0 || qb <= 0) return false;
    const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = reinterpret_cast<uintptr_t>(q);
    return a < b + (uintptr_t)qb && b < a + (uintptr_t)pb;
}

// ---- persistent schedule: `work` tiles dealt round-robin over at most one CTA per SM; this CTA's count and i-th tile --
static inline int persistent_grid(int64_t work) { return (int)(work < sm_count() ? work : sm_count()); }
__device__ __forceinline__ int cta_tiles(int n_tiles) { return (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x; }
__device__ __forceinline__ int cta_tile(int i) { return (int)blockIdx.x + i * (int)gridDim.x; }

// ---- device helpers ---------------------------------------------------------------------------------
// exponent factors of the activations, e^-v = 2^(kNegLog2e v) and e^-2v = 2^(kNeg2Log2e v), and ln 2, which undoes them
constexpr float kNegLog2e = -1.4426950408889634f;
constexpr float kNeg2Log2e = -2.8853900817779268f;
constexpr float kLn2 = 0.6931471805599453f;
// sigmoid / tanh on the MUFU pipe: ex2.approx + rcp.approx (~2 ulp each); absolute error < 1e-6, far inside
// the 1e-4 parity budget, and 2 MUFU + 3 FP32 ops per value instead of an IEEE division sequence.
// Written with the .ftz MUFU forms directly: __expf / __fdividef wrap the same instructions in denormal-range fix-ups
// (FSETP + two predicated FMUL per ex2, a range test per division) that the saturating activations do not need --
// e^-v below 1e-38 contributes nothing to 1 + e^-v, and rcp(inf) = 0 is the correct limit.  4 / 5 instructions per value.
__device__ __forceinline__ float ex2_ftz_(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_ftz_(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float sigmoidf_(float v) { return rcp_ftz_(1.0f + ex2_ftz_(kNegLog2e * v)); }
__device__ __forceinline__ float tanhf_(float v) { return fmaf(2.0f, rcp_ftz_(1.0f + ex2_ftz_(kNeg2Log2e * v)), -1.0f); }

// ReLU as torch defines it: NaN stays NaN (fmaxf(NaN, 0) would be 0).  max.NaN is one FMNMX.NAN, as cheap as fmaxf.
// Its backward masks with out <= 0, which passes the gradient at a NaN output, as torch's does.
__device__ __forceinline__ float relu_(float v) {
    float y;
    asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(y) : "f"(v));
    return y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace stmgcn
