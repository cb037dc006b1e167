// 16-bit (bf16) operand helpers for the wgmma kernels: the 128-byte-swizzled tile layout shared by K-major and MN-major
// operands, its descriptors, and the bf16 hi/lo split.
//
// Precision scheme "3xBF16": every fp32 operand v is stored as TWO bf16 planes, hi = bf16(v) (round to nearest) and
// lo = bf16(v - hi); v = hi + lo up to 2^-18 relative.  A.B is accumulated in fp32 registers as Ahi.Bhi + Alo.Bhi + Ahi.Blo
// (the dropped Alo.Blo term is ~2^-18 relative), inside the 1e-4 parity bar (BASELINE.json) at half the tensor-pipe time
// and half the shared-memory / L2 operand bytes of 3xTF32; the planes cost the same 4 bytes per value in HBM as the fp32
// number they replace.  A single pass over the hi planes is the bf16 arithmetic mode of the bf16-quoted configurations
// (BASELINE.json configs[1], [3], [4]).
//
// One tile layout for everything: a [rows][64 bf16] tile, 128 bytes per row, 8-row groups of 1024 bytes, 16-byte
// chunk index XORed with (row & 7) -- the TMA SWIZZLE_128B pattern.  Read with a K-major descriptor it is an operand
// whose K runs along the 64 columns (M/N = rows); read with an MN-major descriptor (canonical layout ((64,n),(8,k)),
// tc_common.cuh) it is the TRANSPOSED operand: M/N runs along the 64 columns (one 64-element atom; further atoms LBO
// bytes apart), K along the rows (8-row atoms, SBO = 1024 bytes apart).  So the same shared-memory image of
// [h_below | h_prev] feeds the gate GEMM (K-major A) and the weight-gradient GEMM (MN-major A), and one image of dA
// feeds the data-gradient GEMM (K-major A) and the weight-gradient GEMM (MN-major B).
#pragma once
#include "tc_common.cuh"
#include "wgmma.cuh"
#include <cuda_bf16.h>

namespace stmgcn {
namespace tc {

constexpr int kTile16Cols = 64;                       // bf16 per 128-byte row
constexpr int kTile16Bytes = 128 * 128;               // [128 rows][64 bf16] = 16 KB

// byte offset of element (row, col) in a [rows][64 bf16] 128B-swizzled tile
__host__ __device__ __forceinline__ uint32_t sw128_off16(uint32_t row, uint32_t col) {
    return row * 128u + ((((col >> 3) ^ (row & 7u)) & 7u) << 4) + ((col & 7u) << 1);
}

// K-major 128B-swizzled tile: rows of 128 B, 8-row groups 1024 B apart; one k16 MMA consumes 32 bytes of the row:
// advance the start address by 32 B (+2 in the encoded field) per k-step.
__device__ __forceinline__ uint64_t desc16_k(uint32_t smem_addr) { return smem_desc_k_sw128(smem_addr); }
// MN-major view of the same tile: K = 16 rows per MMA = two 8-row atoms (SBO = 1024 B); advance by 2048 B per k-step.
// lbo_bytes: distance between 64-element atoms along M/N (unused when the operand is 64 wide).
__device__ __forceinline__ uint64_t desc16_mn(uint32_t smem_addr, uint32_t lbo_bytes) {
    return smem_desc_mn_sw128(smem_addr, lbo_bytes, 1024u);
}

// ---- bf16 hi / lo split ------------------------------------------------------------------------------------
// two fp32 -> packed bf16x2 (round to nearest even); low half = a, high half = b
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}
__device__ __forceinline__ float bf16_lo_as_f32(uint32_t packed) { return __uint_as_float(packed << 16); }
__device__ __forceinline__ float bf16_hi_as_f32(uint32_t packed) { return __uint_as_float(packed & 0xffff0000u); }
// (a, b) -> hi plane pair and lo plane pair
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
    hi = pack_bf16x2(a, b);
    lo = pack_bf16x2(a - bf16_lo_as_f32(hi), b - bf16_hi_as_f32(hi));
}

}  // namespace tc
}  // namespace stmgcn
