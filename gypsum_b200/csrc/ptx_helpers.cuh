// Device-only helpers shared by the kernels: mbarrier + 1-D TMA bulk copy (global -> shared), named barriers,
// cp.async, warp reductions.
#pragma once
#include <stdint.h>

#include "gb_common.cuh"

namespace gb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void pair_barrier(int pair) { asm volatile("bar.sync %0, 64;" ::"r"(pair + 1) : "memory"); }


__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8(void* dst, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// Hint: bring [src, src + bytes) into L2 (TMA bulk prefetch; src and bytes multiples of 16).
__device__ __forceinline__ void prefetch_l2_bulk(const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Warp-level merge of per-thread peaks: REDUX for (max, first index, count), shuffles for the float64 sum.
// Profile values are >= 0 (an excluded slot holds -1), so their IEEE bit patterns order like signed ints.
__device__ __forceinline__ void warp_reduce_peak(Peak& p) {
    const int bits = __float_as_int(p.mx);
    const int mb = __reduce_max_sync(0xffffffffu, bits);
    const bool is = bits == mb;
    p.idx = __reduce_min_sync(0xffffffffu, is ? p.idx : 0x7fffffff);
    p.cnt = __reduce_add_sync(0xffffffffu, is ? p.cnt : 0);
    p.mx = __int_as_float(mb);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) p.sum += __shfl_xor_sync(0xffffffffu, p.sum, off);
}
// Warp sum of a coherent probe value: only the lane holding the probed lag contributes a non-zero value.
__device__ __forceinline__ void warp_reduce_probe(float& re, float& im) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        re += __shfl_xor_sync(0xffffffffu, re, off);
        im += __shfl_xor_sync(0xffffffffu, im, off);
    }
}

}  // namespace gb
