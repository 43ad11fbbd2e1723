// HardNet 8x8 head on tensor cores: conv8x8(128->128, no bias) == GEMM [n, 8192] x [8192, 128], then BatchNorm and
// L2 normalisation (HardNet.py:86-101, 12-19).  A = trunk features in the L_HEAD layout (tcx_conv.cuh) written by the last conv layer
// ([patch/128][k/8][patch%128][8] fp16: 128 patches are the M rows of one tile), B = head weights [k/8][cout][8] fp16.
// One CTA per 128-patch tile streams K in 64-wide stages (A 16 KiB + B 16 KiB per stage, bulk copies, 6-stage ring); two
// consumer warpgroups hold the 64 x 128 fp32 accumulators of their half of the tile in registers, and the quad of threads that
// owns a row does BN + sum of squares + scale.
#pragma once
#include "tc_common.cuh"

namespace ag {
namespace tc {

constexpr int HEAD_K = 8192, HEAD_N = 128, HEAD_KS = 64, HEAD_STAGES = 6;
constexpr uint32_t HEAD_STAGE_A = (HEAD_KS / 8) * 128 * 16, HEAD_STAGE_B = (HEAD_KS / 8) * HEAD_N * 16;
constexpr size_t HEAD_SMEM = 1024 + (size_t)HEAD_STAGES * (HEAD_STAGE_A + HEAD_STAGE_B);

template <int BF>
__global__ void __launch_bounds__(288, 1) tc_head_kernel(const __half* __restrict__ feat, const __half* __restrict__ wh,
                                                          const float* __restrict__ bn /*scale[128], shift[128]*/, float* __restrict__ out,
                                                          int n, int group, const int* __restrict__ count) {
    extern __shared__ __align__(1024) unsigned char smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);
    uint64_t* empty = full + HEAD_STAGES;
    unsigned char* sA = smem + 1024;
    unsigned char* sB = sA + (size_t)HEAD_STAGES * HEAD_STAGE_A;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x;
    constexpr int NK = HEAD_K / HEAD_KS;  // 128 stages

    if (threadIdx.x == 0) {
        for (int s = 0; s < HEAD_STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            const unsigned char* ga = reinterpret_cast<const unsigned char*>(feat) + (size_t)tile * (HEAD_K / 8) * 128 * 16;
            const unsigned char* gb = reinterpret_cast<const unsigned char*>(wh);
            for (int k = 0; k < NK; k++) {
                const int s = k % HEAD_STAGES;
                mbar_wait(&empty[s], ((k / HEAD_STAGES) & 1) ^ 1);
                mbar_expect_tx(&full[s], HEAD_STAGE_A + HEAD_STAGE_B);
                bulk_g2s(sA + (size_t)s * HEAD_STAGE_A, ga + (size_t)k * HEAD_STAGE_A, HEAD_STAGE_A, &full[s]);
                bulk_g2s(sB + (size_t)s * HEAD_STAGE_B, gb + (size_t)k * HEAD_STAGE_B, HEAD_STAGE_B, &full[s]);
            }
        }
    } else {
        const int wg = warp >> 2, wq = warp & 3;
        float d[HEAD_N / 2];
        // stage k's MMAs are issued before stage k-1's are waited for: the tensor core always has the next stage queued
        for (int k = 0; k < NK; k++) {
            const int s = k % HEAD_STAGES;
            mbar_wait(&full[s], (k / HEAD_STAGES) & 1);
            const uint32_t a0 = smem_u32(sA + (size_t)s * HEAD_STAGE_A) + wg * 64 * 16, b0 = smem_u32(sB + (size_t)s * HEAD_STAGE_B);
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < HEAD_KS / 16; j++)
                Wgmma<HEAD_N, BF>::mma(d, desc64(desc_lo(a0 + (uint32_t)(2 * j) * 128u * 16u, 128u * 16u)),
                                       desc64(desc_lo(b0 + (uint32_t)(2 * j) * HEAD_N * 16u, HEAD_N * 16u)), (k | j) != 0);
            wgmma_commit();
            if (k > 0) {
                wgmma_wait<1>();
                bar_sync(3 + wg, 128);
                if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[(k - 1) % HEAD_STAGES]);
            }
        }
        wgmma_wait<0>();
        wgmma_reg_fence<HEAD_N / 2>(d);
        // rows r0 = 16 wq + lane/4 (h = 0) and r0 + 8 (h = 1) of this warpgroup's 64; columns 8 j + 2 (lane % 4) + e
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int pi = tile * 128 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
            const bool ok = pi < n && (count == nullptr || (pi % group) < count[pi / group]);
            float ss = 0.f;
#pragma unroll
            for (int j = 0; j < HEAD_N / 8; j++) {
                const int c = j * 8 + 2 * (lane & 3);
                const float v0 = fmaf(d[4 * j + 2 * h], __ldg(bn + c), __ldg(bn + 128 + c));
                const float v1 = fmaf(d[4 * j + 2 * h + 1], __ldg(bn + c + 1), __ldg(bn + 128 + c + 1));
                ss = fmaf(v0, v0, ss);
                ss = fmaf(v1, v1, ss);
            }
            ss += __shfl_xor_sync(0xffffffffu, ss, 1);
            ss += __shfl_xor_sync(0xffffffffu, ss, 2);
            const float inv = 1.0f / sqrtf(ss + 1e-8f);
            if (ok) {
#pragma unroll
                for (int j = 0; j < HEAD_N / 8; j++) {
                    const int c = j * 8 + 2 * (lane & 3);
                    float2 v;
                    v.x = fmaf(d[4 * j + 2 * h], __ldg(bn + c), __ldg(bn + 128 + c)) * inv;
                    v.y = fmaf(d[4 * j + 2 * h + 1], __ldg(bn + c + 1), __ldg(bn + 128 + c + 1)) * inv;
                    *reinterpret_cast<float2*>(out + (size_t)pi * 128 + c) = v;
                }
            }
        }
    }
}

// ---- AffNet / OriNet heads on tensor cores -------------------------------------------------------------------------------
// conv8x8(64 -> 3) resp. the padded conv8x8(64 -> 2) seen as 18 shifted dot products (nets_simt.cu) == GEMM [n, 4096] x
// [4096, 32] with fp32-grade operands: the last conv layer writes its output as fp16 hi + lo planes in the L_HEAD layout (tcx_conv.cuh), the head
// weights are stored as [k/8][W_hi rows 0..31 | W_lo rows 32..63][8], and per K step the issuer runs A_hi x [W_hi ; W_lo]
// (N = 64) and A_lo x W_hi (N = 32); the epilogue adds the two accumulator halves and applies the reference's post-processing
// (architectures.py:57-59,76-82,228-230; LAF.py:276-291).  One CTA per 128-patch tile, K streamed in 64-wide stages.
// The tensor core adds into its fp32 accumulator with truncation, and the error grows with the length of the running sum (one
// accumulator over all 512 MMAs costs about 2e-4 rad of OriNet angle against 2.6e-5 with an fp32 FMA chain).  Every K stage therefore
// starts a fresh accumulator, and the stage sums are added in fp32 registers.
constexpr int HX_K = 4096, HX_NP = 32, HX_KS = 64, HX_STAGES = 5;
constexpr uint32_t HX_STAGE_A = (HX_KS / 8) * 128 * 16, HX_STAGE_B = (HX_KS / 8) * (2 * HX_NP) * 16;
constexpr size_t HX_SMEM = 1024 + (size_t)HX_STAGES * (2 * HX_STAGE_A + HX_STAGE_B);
constexpr size_t HX_PLANE_TILE = (size_t)(HX_K / 8) * 128 * 16;   // bytes of one 128-patch tile in one plane

template <int KIND /* 0 AffNet, 1 OriNet */>
__global__ void __launch_bounds__(288, 1) tc_headx_kernel(const __half* __restrict__ feat, const __half* __restrict__ wh, const float* __restrict__ bias,
                                                           const float inv_scale, float* __restrict__ out, float* __restrict__ angle_out, float* __restrict__ raw_out, int n, int group,
                                                           const int* __restrict__ count) {
    extern __shared__ __align__(1024) unsigned char smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);
    uint64_t* empty = full + HX_STAGES;
    unsigned char* sA = smem + 1024;                                    // [stage][hi | lo]
    unsigned char* sB = sA + (size_t)HX_STAGES * 2 * HX_STAGE_A;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x, tiles = gridDim.x;
    constexpr int NK = HX_K / HX_KS;

    {   // a tile without a single live patch has nothing to do (rows beyond count[] of every image it touches)
        int live = 0;
        if (threadIdx.x < 128) {
            const int pi = tile * 128 + threadIdx.x;
            live = pi < n && (count == nullptr || (pi % group) < count[pi / group]);
        }
        if (!__syncthreads_or(live)) return;
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < HX_STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            const unsigned char* ga = reinterpret_cast<const unsigned char*>(feat) + (size_t)tile * HX_PLANE_TILE;
            const unsigned char* gl = ga + (size_t)tiles * HX_PLANE_TILE;
            const unsigned char* gb = reinterpret_cast<const unsigned char*>(wh);
            for (int k = 0; k < NK; k++) {
                const int s = k % HX_STAGES;
                mbar_wait(&empty[s], ((k / HX_STAGES) & 1) ^ 1);
                mbar_expect_tx(&full[s], 2 * HX_STAGE_A + HX_STAGE_B);
                bulk_g2s(sA + (size_t)s * 2 * HX_STAGE_A, ga + (size_t)k * HX_STAGE_A, HX_STAGE_A, &full[s]);
                bulk_g2s(sA + (size_t)s * 2 * HX_STAGE_A + HX_STAGE_A, gl + (size_t)k * HX_STAGE_A, HX_STAGE_A, &full[s]);
                bulk_g2s(sB + (size_t)s * HX_STAGE_B, gb + (size_t)k * HX_STAGE_B, HX_STAGE_B, &full[s]);
            }
        }
    } else {
        const int wg = warp >> 2, wq = warp & 3;
        float tot[HX_NP], d[HX_NP];   // fragment of the N = 64 accumulator: columns [0, 32) = A_hi W_hi + A_lo W_hi, [32, 64) = A_hi W_lo
#pragma unroll
        for (int i = 0; i < HX_NP; i++) tot[i] = 0.f;
        for (int k = 0; k < NK; k++) {
            const int s = k % HX_STAGES;
            mbar_wait(&full[s], (k / HX_STAGES) & 1);
            const uint32_t a0 = smem_u32(sA + (size_t)s * 2 * HX_STAGE_A) + wg * 64 * 16, b0 = smem_u32(sB + (size_t)s * HX_STAGE_B);
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < HX_KS / 16; j++) {
                const uint64_t da = desc64(desc_lo(a0 + (uint32_t)(2 * j) * 128u * 16u, 128u * 16u));
                const uint64_t dl = desc64(desc_lo(a0 + HX_STAGE_A + (uint32_t)(2 * j) * 128u * 16u, 128u * 16u));
                const uint64_t db = desc64(desc_lo(b0 + (uint32_t)(2 * j) * (2 * HX_NP) * 16u, (2 * HX_NP) * 16u));
                Wgmma<2 * HX_NP, 0>::mma(d, da, db, j != 0);   // A_hi x [W_hi ; W_lo]
                Wgmma<HX_NP, 0>::mma(d, dl, db, 1);            // A_lo x W_hi -> hi columns
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_reg_fence<HX_NP>(d);
            bar_sync(3 + wg, 128);
            if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);
#pragma unroll
            for (int i = 0; i < HX_NP; i++) tot[i] += d[i];
        }
        constexpr int NO = KIND == 0 ? 3 : 18;
        // the quad of lanes that shares a row gathers the NO head outputs of that row: column o lives in lane 4 (lane / 4) + (o % 8) / 2,
        // register 4 (o / 8) + 2 h + o % 2, its A_hi W_lo part 16 registers further (column o + 32)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            float acc[NO];
#pragma unroll
            for (int o = 0; o < NO; o++) {
                const int src_lane = (lane & ~3) | ((o & 7) >> 1), reg = 4 * (o >> 3) + 2 * h + (o & 1);
                acc[o] = __shfl_sync(0xffffffffu, tot[reg] + tot[reg + 16], src_lane);
            }
            const int pi = tile * 128 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
            const bool ok = (lane & 3) == 0 && pi < n && (count == nullptr || (pi % group) < count[pi / group]);
            if (!ok) continue;
            if (KIND == 0) {
                const float s0 = acc[0] * inv_scale, s1 = acc[1] * inv_scale, s2 = acc[2 % NO] * inv_scale;
                const float a00 = 1.0f + tanhf(s0 + bias[0]), a10 = tanhf(s1 + bias[1]), a11 = 1.0f + tanhf(s2 + bias[2]);
                if (raw_out) { raw_out[(size_t)pi * 3] = a00; raw_out[(size_t)pi * 3 + 1] = a10; raw_out[(size_t)pi * 3 + 2] = a11; }   // convertJIT/AffNetJIT.pt: xy + [1, 0, 1]
                if (out) rectify_up_is_up(a00, 0.f, a10, a11, out + (size_t)pi * 4);
            } else {
                float m0 = 0.f, m1 = 0.f;
#pragma unroll
                for (int o = 0; o < 9; o++) {
                    m0 += tanhf(acc[o % NO] * inv_scale + bias[0]);
                    m1 += tanhf(acc[(9 + o) % NO] * inv_scale + bias[1]);
                }
                m0 /= 9.0f; m1 /= 9.0f;
                if (raw_out) { raw_out[(size_t)pi * 2] = m0; raw_out[(size_t)pi * 2 + 1] = m1; }   // convertJIT/OriNetJIT.pt: the mean of tanh over the 3x3 map
                const float ang = atan2f(m0 + 1e-8f, m1 + 1e-8f);
                if (angle_out) angle_out[pi] = ang;
                if (out) {
                    const float c = cosf(ang), sn = sinf(ang);
                    float* o = out + (size_t)pi * 4;
                    o[0] = c; o[1] = sn; o[2] = -sn; o[3] = c;
                }
            }
        }
    }
}

}  // namespace tc
}  // namespace ag
