// Hopper (sm_90a) primitives used by the tensor-core kernels: barriers, register budgets, bulk and TMA tensor copies, L2
// policies, the 128-byte swizzle and wgmma shared-memory matrix descriptors (the instructions themselves: wgmma.cuh).
//
// Precision scheme "3xTF32": every fp32 operand v is split into hi = v with the low 13 mantissa bits cleared
// (exactly representable in tf32, so the tensor core's own fp32->tf32 conversion cannot change it) and
// lo = v - hi (exact in fp32; <= 13 significant bits, again masked to tf32).  A.B is accumulated in fp32
// registers as Ahi.Bhi + Alo.Bhi + Ahi.Blo; the dropped Alo.Blo term is ~2^-22 relative, well inside the 1e-4
// parity bar that rules out single-pass TF32 (SURVEY.md section 0.5).
#pragma once
#include "common.cuh"

namespace stmgcn {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// bytes from the dynamic shared memory to its first 1024-byte boundary, where swizzled tiles may start (launches request
// 1024 bytes more than they use); kernels offset the __shared__ array itself by it, which keeps its address space
__device__ __forceinline__ uint32_t smem_pad1024(const void* smem_raw) { return (1024u - (smem_u32(smem_raw) & 1023u)) & 1023u; }

// named barrier `id` (0 is __syncthreads') over n_threads threads, a multiple of 32
__device__ __forceinline__ void bar_sync(uint32_t id, uint32_t n_threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory");
}
// a warpgroup's per-thread register budget (every warp of the warpgroup executes the same instruction)
template <uint32_t N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// ---- tf32 split ---------------------------------------------------------------------------------------
__device__ __forceinline__ float tf32_hi(float v) { return __uint_as_float(__float_as_uint(v) & 0xffffe000u); }
__device__ __forceinline__ float tf32_lo(float v, float hi) {
    return __uint_as_float(__float_as_uint(v - hi) & 0xffffe000u);
}
// v rounded to the nearest tf32 value (ties away from zero), exact in tf32: the rounded split hi = rna(v),
// lo = rna(v - hi) of the kernels whose products cancel (K1e, the chain gradient), |v - hi - lo| <= 2^-24 |v|
__device__ __forceinline__ float tf32_rna(float v) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
}

// ---- mbarrier -----------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded waits: a protocol bug traps (the launch fails with an error) instead of hanging the GPU; ~20 s before the trap,
// so profiler / sanitizer slow-downs of 100x do not kill the context.
// mbar_wait_raw spins (fast polls first, then a nanosleep back-off): for the consumer warpgroups, whose wait ends the
// moment the data lands.  mbar_wait_polite backs off ~40 ns between polls: for the single-thread roles (TMA producer),
// whose spinning warp would compete for issue slots with the warps doing the arithmetic on the same SM sub-partition
// (a quarter of all executed instructions were try_wait / branch pairs).
__device__ __forceinline__ void mbar_wait_raw(uint64_t* bar, uint32_t parity) {
    for (uint32_t it = 0; it < (1u << 16); ++it)
        if (mbar_try_wait(bar, parity)) return;
    for (uint32_t it = 0; it < (1u << 26); ++it) {
        if (mbar_try_wait(bar, parity)) return;
        __nanosleep(256);
    }
    __trap();
}
__device__ __forceinline__ void mbar_wait_polite(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    for (uint32_t it = 0; it < (1u << 28); ++it) {
        __nanosleep(40);
        if (mbar_try_wait(bar, parity)) return;
    }
    __trap();
}

// generic-proxy smem writes -> visible to the async proxy (wgmma / bulk copies read smem through it)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- 1-D bulk async copy global -> shared, completion on an mbarrier (TMA unit; SASS: UBLKCP) -----------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---- TMA tensor copies through a CUtensorMap: a load completes on an mbarrier; a store drops the rows past the tensor's
// end, and its completion is tracked per issuing thread in bulk async-groups ------------------------------------------
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 :: "r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_3d_hint(void* smem_dst, const void* tmap, int c0, int c1, int c2, uint64_t* bar,
                                                 uint64_t pol) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
                 " [%0], [%1, {%3, %4, %5}], [%2], %6;"
                 :: "r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(pol) : "memory");
}
__device__ __forceinline__ void tma_prefetch_3d(const void* tmap, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];"
                 :: "l"(tmap), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const void* tmap, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 :: "l"(tmap), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the issuing thread's bulk groups have finished READING shared memory (the source tile may be overwritten)
__device__ __forceinline__ void bulk_wait_group_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// One elected lane of a fully converged warp, for the single-thread TMA / mbarrier instructions (ptxas can prove that
// elect.sync selects one thread; a `lane == 0` guard gets wrapped in a serialisation loop).
__device__ __forceinline__ bool elect_one_sync() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}
// fire-and-forget 16-byte reduction into global memory (the add happens in L2, nothing returns); dst 16-byte aligned
__device__ __forceinline__ void red_add_f32x4(float* dst, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
// L2 prefetch of a contiguous global range (no registers, no shared memory)
__device__ __forceinline__ void prefetch_l2(const void* gmem, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem), "r"(bytes) : "memory");
}
// L2 policy for data a launch reads exactly once: evicted first, so that the lines read again keep their place in L2
__device__ __forceinline__ uint64_t l2_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

// ---- wgmma shared-memory matrix descriptors (sm_90: start >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46),
// layout type [62,64) with 1 = 128-byte swizzle).  Tiles are 1024-byte aligned, so the base-offset field stays 0.
// K-major operand, 128-byte swizzle: rows of 128 B along K, 8-row groups 1024 B apart (SBO); LBO is unused.
// A k-step inside the 128-byte row is an add on the start address (32 B = +2 encoded for k16 bf16 / k8 tf32).
__device__ __forceinline__ uint64_t smem_desc_k_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// MN-major operand (16-bit types only), 128-byte swizzle: canonical layout ((64, n), (8, k)) in elements -- an atom of
// 1024 B holds 64 consecutive M/N elements (one 128-byte row) for each of 8 consecutive K; LBO = byte distance between
// atoms along M/N, SBO = between atoms along K.
__device__ __forceinline__ uint64_t smem_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// ---- 128-byte swizzle (TMA SWIZZLE_128B): 128-byte rows, 8-row groups of 1024 bytes, a byte's 16-byte chunk index XORed
// with (row & 7).  Byte offset of element e of a row of BYTES-byte elements (sw128<1>: byte e; <2>: bf16; <4>: fp32):
template <uint32_t BYTES>
__host__ __device__ __forceinline__ uint32_t sw128(uint32_t row, uint32_t e) {
    constexpr uint32_t kPerChunk = 16u / BYTES;
    return row * 128u + ((((e / kPerChunk) ^ (row & 7u)) & 7u) << 4) + ((e % kPerChunk) * BYTES);
}

}  // namespace tc
}  // namespace stmgcn
