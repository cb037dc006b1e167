// Shared pieces of the 3xTF32 wgmma kernels: tile constants, the tf32 hi/lo split + swizzled store helpers and the
// weight-image packer.  Included by proj_tc.cu and wgrad_tc.cu.
#pragma once
#include "tc_common.cuh"
#include "wgmma.cuh"

namespace stmgcn {
namespace tc {

constexpr int kTileM = 128;
constexpr int kKB = 32;              // k-block: one 128-byte swizzle row of fp32
constexpr int kHid = 64;
constexpr int kGateCols = 256;       // 4H
constexpr int kABytes = kTileM * kKB * 4;            // 16 KB per hi or lo A tile of 128 rows

__device__ __forceinline__ void split_store(uint8_t* st, uint32_t off, const float4& v) {
    float4 hi, lo;
    hi.x = tf32_hi(v.x); hi.y = tf32_hi(v.y); hi.z = tf32_hi(v.z); hi.w = tf32_hi(v.w);
    lo.x = tf32_lo(v.x, hi.x); lo.y = tf32_lo(v.y, hi.y); lo.z = tf32_lo(v.z, hi.z); lo.w = tf32_lo(v.w, hi.w);
    *reinterpret_cast<float4*>(st + off) = hi;
    *reinterpret_cast<float4*>(st + kABytes + off) = lo;
}


// transpose-store one float4 (4 consecutive M/N indices mn..mn+3 of row k) into a K-major swizzled tile pair
__device__ __forceinline__ void split_store_t(uint8_t* hi_tile, uint8_t* lo_tile, int mn, int k, const float4& v) {
    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t off = sw128_offset((uint32_t)(mn + j), (uint32_t)k);
        const float hi = tf32_hi(vv[j]);
        *reinterpret_cast<float*>(hi_tile + off) = hi;
        *reinterpret_cast<float*>(lo_tile + off) = tf32_lo(vv[j], hi);
    }
}

// Generic K-major hi/lo image of a logical B[n][k] = src[n*rs + k*cs]: per 32-wide k-block [hi | lo], each an
// [n_rows][32] fp32 tile with the 128-byte swizzle.
static __global__ void pack_image_kernel(const float* __restrict__ src, int n_rows, int k_cols, int64_t rs, int64_t cs,
                                         float* __restrict__ img, int tile_rows) {
    const int total = n_rows * k_cols;
    const int tile_floats = tile_rows * kKB;      // tile_rows >= n_rows: extra rows keep what the caller put there (zeros)
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
        const int n = e / k_cols, k = e % k_cols;
        const float v = src[(int64_t)n * rs + (int64_t)k * cs];
        const float hi = tf32_hi(v);
        const float lo = tf32_lo(v, hi);
        const int kb = k / kKB, kk = k % kKB;
        const uint32_t off = sw128_offset((uint32_t)n, (uint32_t)kk) / 4;
        float* base = img + (size_t)kb * (2 * tile_floats);
        base[off] = hi;
        base[tile_floats + off] = lo;
    }
}

}  // namespace tc
}  // namespace stmgcn
