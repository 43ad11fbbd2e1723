// Primitives shared by the tensor-core (wgmma) kernels of the nets, sm_90a: the conv kernels (tcx_first.cuh, tcx_conv.cuh) and the 8x8
// head GEMMs (tc_head.cuh).  Shared-memory addresses, mbarriers, bulk global -> shared copies, named barriers, the matrix descriptor
// of the no-swizzle K-major layout, and the source of the fused first conv layer.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace ag {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// try_wait carries a suspend-time hint, so a waiting warp sleeps in hardware until the phase completes (or the hint expires)
// instead of re-issuing try_wait + branch
#ifndef AG_MBAR_HINT_NS
#define AG_MBAR_HINT_NS 200000
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#if AG_MBAR_HINT_NS > 0
    asm volatile(
        "{\n .reg .pred P;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 P, [%0], %1, %2;\n @P bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}\n" ::"r"(smem_u32(bar)),
        "r"(parity), "r"((uint32_t)AG_MBAR_HINT_NS)
        : "memory");
#else
    asm volatile(
        "{\n .reg .pred P;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 P, [%0], %1;\n @P bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
#endif
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// named barrier of `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// Shared-memory matrix descriptor of the no-swizzle K-major layout: core matrices of 8 rows x 16 bytes, rows 16 bytes apart, 8-row
// groups SBO = 128 bytes apart (hi word), the two 16-byte K halves of a K = 16 step LBO bytes apart.  The lo word (start address and LBO
// in 16-byte units) is what the issuing loops compute; the hi word is the constant SBO.
constexpr uint32_t DESC_HI = 0x0008u;
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr, uint32_t lbo_bytes) { return ((saddr >> 4) & 0x3FFFu) | ((lbo_bytes >> 4) << 16); }
__device__ __forceinline__ uint64_t desc64(uint32_t lo) { return ((uint64_t)DESC_HI << 32) | lo; }

// Source of the fused first layer (tcx_first_kernel): either materialised patches [n,32,32] fp32, or the pyramid + keypoints
// (the affine bilinear sampler of LAF.py:313-372 runs inside the kernel; patches never touch HBM).
struct PyrGeomTC {
    int n_octaves, n_levels;
    int h[AG_MAX_OCTAVES], w[AG_MAX_OCTAVES];
    long long off[AG_MAX_OCTAVES][AG_MAX_LEVELS];
};
struct FirstSrc {
    const float* patches;   // if non-NULL: [n][32][32]
    const float* pyr;       // else: pyramid base, rows (b, i) = (pi / cap, pi % cap)
    const float* lafs;      // [B*cap][2][3] normalised
    const int* oct;
    const int* lvl;
    int cap;
    const float* w1;        // [9][C1] fp32 (BatchNorm folded)
    float w1_scale, w1_inv; // tensor-core layer 1: weights are used times w1_scale (a power of two), accumulators times w1_inv
    const float* b1;        // [C1]
    PyrGeomTC geom;
};

}  // namespace tc
}  // namespace ag
