// Tensor-core (wgmma) 3x3 convolution engine for the AffNet / OriNet / HardNet trunks (sm_90a).
//
// Formulation: shifted-window implicit GEMM.  The fp16 activations of one patch live in the canonical no-swizzle K-major layout
// [C/8][NPIX][8]  (8 channels = one 16-byte core-matrix row, pixel slots contiguous), over a zero-padded pixel plane.  For tap
// (dy,dx) the A operand of the M=64 block starting at output row m0 is the SAME buffer with its descriptor start address advanced
// by (m0 + off(dy,dx)) * 16 bytes - no im2col copy.  Stride-2 layers read a phase-split plane (4 parity planes) so that they are
// shifted-window GEMMs too.
//   D[64 x N] (fp32, registers) += A[64 x 16] (smem desc) * W[N x 16]^T (smem desc)      9 * C/16 MMAs per block
// One persistent CTA keeps the layer's (BatchNorm-folded) weights resident in shared memory and loops over patches:
//   warps 0-7: two consumer warpgroups - warpgroup g takes the M=64 blocks g, g+2, ... of a patch: wgmma, then bias + ReLU,
//              fp16 pack, stores straight into the NEXT layer's canonical layout (or fp32 NCHW for the last trunk layer), plus the
//              zero border of that layout
//   warp 8   : loader - one cp.async.bulk per channel group and patch (global -> smem stage), mbarrier complete_tx
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace ag {
namespace tc {

enum LayoutKind { PLAIN = 0, PHASE = 1, FINAL = 2, HEADL = 3 };  // HEADL: fp16 [patch/128][pixel*C/8 + c/8][patch%128][8], the A operand of the 8x8-head GEMM

// Pixel-slot geometry of an activation buffer that is the INPUT of a layer with `stride` on an HxH map.
template <int H, int STRIDE>
struct InLay {
    static constexpr int HOUT = H / STRIDE;
    static constexpr int PITCH = (STRIDE == 1) ? H + 2 : H / 2 + 1;          // row pitch of the output-row index space
    static constexpr int ROWS = (HOUT - 1) * PITCH + HOUT;                    // output rows m = y*PITCH + x
    static constexpr int BLOCKS = (ROWS + 63) / 64;                           // M = 64 blocks of output rows
    static constexpr int PLANE = (STRIDE == 1) ? 0 : ((PITCH * PITCH + 7) / 8) * 8;   // parity-plane stride (slots)
    static constexpr int MAXOFF = (STRIDE == 1) ? 2 * PITCH + 2 : 3 * PLANE + PITCH + 1;
    static constexpr int NPIX = ((64 * BLOCKS + MAXOFF + 1 + 7) / 8) * 8;     // slots per channel group incl. slack
    // slots that hold data (padded plane / four parity planes); the slack behind them only feeds accumulator rows that are never
    // stored, so loaders copy just this prefix of every channel group and leave whatever is in shared memory behind it
    static constexpr int USED = (STRIDE == 1) ? (H + 2) * (H + 2) : 3 * PLANE + PITCH * PITCH;
    __host__ __device__ static constexpr int tap_off(int dy, int dx) {
        return (STRIDE == 1) ? dy * PITCH + dx : ((dy & 1) * 2 + (dx & 1)) * PLANE + (dy >> 1) * PITCH + (dx >> 1);
    }
    // slot of padded coordinate (Y,X) in [0,H+1]^2
    __host__ __device__ static constexpr int slot(int Y, int X) {
        return (STRIDE == 1) ? Y * PITCH + X : ((Y & 1) * 2 + (X & 1)) * PLANE + (Y >> 1) * PITCH + (X >> 1);
    }
};

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

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

// Source of the fused first layer (FIRST = 1): either materialised patches [n,32,32] fp32, or the pyramid + keypoints
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

struct ConvArgs {
    const __half* in;     // [n][CIN/8][NPIX_IN][8]
    void* out;            // next layer's canonical fp16 buffer, or fp32 [n][COUT][HOUT][HOUT]
    const __half* wpk;    // [NSPLIT][9][CIN/8][hi rows | lo rows][8]: (1+SW)*COUT/NSPLIT rows per K chunk
    const float* bias;    // [COUT]
    float inv_scale;      // wpk holds the weights times a power of two (fp16 residuals stay normal); accumulators are multiplied by its inverse
    int n, group;
    const int* count;
};

// CIN, COUT: channels; H: input map edge; STRIDE 1|2; NSPLIT: CTAs sharing one patch along COUT; STAGES: smem stages;
// OUT: layout of the output buffer (PLAIN / PHASE for the next conv, FINAL = fp32 NCHW).
// Split precision (fp32-grade results from fp16 tensor cores): SA = the input carries hi and lo fp16 planes
// (x = hi + lo, channel groups [0,KC) hi then [KC,2KC) lo), SW = the weights carry hi and lo copies, OSA = write the
// output as hi/lo planes.  D = A_hi W_hi (+ A_lo W_hi if SA) (+ A_hi W_lo if SW); the lo*lo term (2^-22) is dropped.
// FIRST = 1: layer 1 (sampler + input_norm + conv3x3(1 -> CIN) + ReLU, fp32 on CUDA cores) runs in eight producer warps and
// fills the stages of this layer.
template <int CIN, int COUT, int H, int STRIDE, int NSPLIT, int STAGES, int OUT, int SA = 0, int SW = 0, int OSA = 0, int FIRST = 0>
struct ConvCfg {
    using In = InLay<H, STRIDE>;
    static constexpr int HOUT = H / STRIDE;
    static constexpr int KC = CIN / 8;                  // 16-byte channel groups
    static constexpr int NT = COUT / NSPLIT;            // MMA N
    // With split weights the B operand stacks W_hi and W_lo along N (rows [0,NT) hi, [NT,2NT) lo of every K chunk): ONE MMA of
    // N = 2*NT yields A*W_hi and A*W_lo side by side and the epilogue adds the two halves.
    static constexpr int ACCW = NT * (1 + SW);                      // accumulator width (columns)
    static constexpr uint32_t IN_BYTES = (uint32_t)KC * (1 + SA) * In::NPIX * 16;     // one patch
    static constexpr uint32_t W_HALF = 9u * KC * NT * 16;
    static constexpr uint32_t W_BYTES = W_HALF * (1 + SW);
    static constexpr int THREADS = FIRST ? 544 : 288;   // 2 consumer warpgroups + loader (+ 8 producer warps for FIRST)
    static constexpr size_t FIRST_BYTES = FIRST ? (size_t)(2 * 34 * 36 + 9 * CIN + CIN + 64) * 4 : 0;
    static constexpr size_t SMEM = 1024 + (size_t)W_BYTES + (size_t)STAGES * IN_BYTES + FIRST_BYTES;
    // output buffer geometry
    using OutP = InLay<HOUT, 1>;   // if the consumer has stride 1
    using OutS = InLay<HOUT, 2>;   // if the consumer has stride 2
    static constexpr int OUT_NPIX = (OUT == PLAIN) ? OutP::NPIX : (OUT == PHASE) ? OutS::NPIX : 0;
    static constexpr size_t OUT_BYTES = (OUT == FINAL) ? (size_t)COUT * HOUT * HOUT * 4
                                        : (OUT == HEADL) ? (size_t)COUT * HOUT * HOUT * 2
                                                         : (size_t)(COUT / 8) * (1 + OSA) * OUT_NPIX * 16;
    static_assert(CIN % 16 == 0 && NT % 16 == 0 && NT <= 128 && ACCW <= 256, "wgmma shape / bias staging");
    static_assert(2 * STAGES + 1 <= 60, "barrier area");
    static_assert(SMEM <= 232448, "shared memory budget");
};

template <int CIN, int COUT, int H, int STRIDE, int NSPLIT, int STAGES, int OUT, int SA, int SW, int OSA, int FIRST>
__global__ void __launch_bounds__(FIRST ? 544 : 288, 1) tc_conv_kernel(const ConvArgs a, const FirstSrc src) {
    using Cfg = ConvCfg<CIN, COUT, H, STRIDE, NSPLIT, STAGES, OUT, SA, SW, OSA, FIRST>;
    using In = typename Cfg::In;
    constexpr int KC = Cfg::KC, NT = Cfg::NT, ACCW = Cfg::ACCW, BLOCKS = In::BLOCKS, HOUT = Cfg::HOUT;
    extern __shared__ __align__(1024) unsigned char smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);  // [STAGES]
    uint64_t* empty = full + STAGES;                       // [STAGES]
    uint64_t* wbar = empty + STAGES;
    float* s_bias = reinterpret_cast<float*>(smem + 512);  // [NT] (NT <= 128)
    unsigned char* sW = smem + 1024;
    unsigned char* sIn = sW + Cfg::W_BYTES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int split = blockIdx.y;

    if (threadIdx.x < NT) s_bias[threadIdx.x] = a.bias[split * NT + threadIdx.x];
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; s++) { mbar_init(&full[s], FIRST ? 256 : 1); mbar_init(&empty[s], 2); }
        mbar_init(wbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    auto valid = [&](int pi) -> bool { return a.count == nullptr || (pi % a.group) < a.count[pi / a.group]; };

    if (warp == 8) {
        // ===== loader =====
        if (lane == 0) {
            mbar_expect_tx(wbar, Cfg::W_BYTES);
            bulk_g2s(sW, reinterpret_cast<const unsigned char*>(a.wpk) + (size_t)split * Cfg::W_BYTES, Cfg::W_BYTES, wbar);
            int it = 0;
            for (int pi = blockIdx.x; pi < a.n && !FIRST; pi += gridDim.x) {
                if (!valid(pi)) continue;
                const int s = it % STAGES;
                mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
                constexpr int G = KC * (1 + SA);
                mbar_expect_tx(&full[s], (uint32_t)G * In::USED * 16u);
                const unsigned char* gsrc = reinterpret_cast<const unsigned char*>(a.in) + (size_t)pi * Cfg::IN_BYTES;
#pragma unroll
                for (int g = 0; g < G; g++)
                    bulk_g2s(sIn + (size_t)s * Cfg::IN_BYTES + (size_t)g * In::NPIX * 16, gsrc + (size_t)g * In::NPIX * 16, In::USED * 16u, &full[s]);
                it++;
            }
        }
    } else if (warp < 8) {
        // ===== consumers: warpgroup wg takes the M = 64 blocks wg, wg + 2, ... of every patch =====
        const int wg = warp >> 2, wq = warp & 3;
        const int et = threadIdx.x;   // 0..255
        mbar_wait(wbar, 0);
        const uint32_t w_lo = desc_lo(smem_u32(sW), ACCW * 16u);
        int it = 0;
        for (int pi = blockIdx.x; pi < a.n; pi += gridDim.x) {
            if (!valid(pi)) continue;
            const int s = it % STAGES;
            unsigned char* outp = reinterpret_cast<unsigned char*>(a.out) + (size_t)pi * Cfg::OUT_BYTES;
            // zero border of the consumer's padded plane (each split its own channel groups)
            if (OUT == PLAIN || OUT == PHASE) {
                constexpr int HB = HOUT + 1;  // border cells: 4*HB
                for (int i = et; i < 4 * HB; i += 256) {
                    const int side = i / HB, k = i - side * HB;
                    int Y, X;
                    if (side == 0) { Y = 0; X = k; } else if (side == 1) { Y = HOUT + 1; X = k + 1; }
                    else if (side == 2) { Y = k + 1; X = 0; } else { Y = k; X = HOUT + 1; }
                    const int slot = (OUT == PLAIN) ? Cfg::OutP::slot(Y, X) : Cfg::OutS::slot(Y, X);
#pragma unroll
                    for (int g = 0; g < NT / 8; g++) {
                        const int cg = split * (NT / 8) + g;
                        *reinterpret_cast<uint4*>(outp + ((size_t)cg * Cfg::OUT_NPIX + slot) * 16) = make_uint4(0, 0, 0, 0);
                        if (OSA) *reinterpret_cast<uint4*>(outp + ((size_t)(COUT / 8 + cg) * Cfg::OUT_NPIX + slot) * 16) = make_uint4(0, 0, 0, 0);
                    }
                }
            }
            mbar_wait(&full[s], (it / STAGES) & 1);
            const uint32_t in_lo = desc_lo(smem_u32(sIn + (size_t)s * Cfg::IN_BYTES), In::NPIX * 16u);
#pragma unroll 1
            for (int b = wg; b < BLOCKS; b += 2) {
                float d[ACCW / 2];
                const uint32_t a_t = in_lo + (uint32_t)(b * 64);  // 16-byte units
                wgmma_fence();
#pragma unroll
                for (int tap = 0; tap < 9; tap++) {
#pragma unroll
                    for (int j = 0; j < KC / 2; j++) {
                        const uint32_t alo = a_t + (uint32_t)(In::tap_off(tap / 3, tap % 3) + 2 * j * In::NPIX);
                        const uint32_t blo = w_lo + (uint32_t)((tap * KC + 2 * j) * ACCW);
                        Wgmma<ACCW, 0>::mma(d, desc64(alo), desc64(blo), (tap | j) != 0);                           // A_hi * [W_hi ; W_lo]
                        if (SA) Wgmma<NT, 0>::mma(d, desc64(alo + (uint32_t)(KC * In::NPIX)), desc64(blo), 1);     // A_lo * W_hi -> hi columns
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_reg_fence<ACCW / 2>(d);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int m = b * 64 + wq * 16 + (lane >> 2) + 8 * h;
                    const int y = m / In::PITCH, x = m - y * In::PITCH;
                    if (y >= HOUT || x >= HOUT) continue;
#pragma unroll
                    for (int j = 0; j < NT / 8; j++) {
                        const int c = j * 8 + 2 * (lane & 3);    // this thread's channel pair of the block
                        const int ch = split * NT + c;
                        float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
                        if (SW) { v0 += d[4 * (j + NT / 8) + 2 * h]; v1 += d[4 * (j + NT / 8) + 2 * h + 1]; }
                        v0 = fmaxf(fmaf(v0, a.inv_scale, s_bias[c]), 0.f);
                        v1 = fmaxf(fmaf(v1, a.inv_scale, s_bias[c + 1]), 0.f);
                        const uint32_t hi = pack_h2(v0, v1);
                        const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
                        const uint32_t lo = pack_h2(v0 - hf.x, v1 - hf.y);   // residual plane: lo = fp16(v - fp16(v))
                        if (OUT == FINAL) {
                            float* o = reinterpret_cast<float*>(outp);
                            o[(size_t)ch * HOUT * HOUT + y * HOUT + x] = v0;
                            o[(size_t)(ch + 1) * HOUT * HOUT + y * HOUT + x] = v1;
                        } else if (OUT == HEADL) {
                            const size_t kch = (size_t)(y * HOUT + x) * (COUT / 8) + ch / 8;
                            unsigned char* hb = reinterpret_cast<unsigned char*>(a.out);
                            const size_t off = (((size_t)(pi >> 7) * (HOUT * HOUT * COUT / 8) + kch) * 128 + (pi & 127)) * 16 + (ch & 7) * 2;
                            *reinterpret_cast<uint32_t*>(hb + off) = hi;
                            if (OSA) *reinterpret_cast<uint32_t*>(hb + (size_t)((a.n + 127) >> 7) * (HOUT * HOUT * COUT / 8) * 128 * 16 + off) = lo;   // behind the hi plane of all tiles
                        } else {
                            const int slot = (OUT == PLAIN) ? Cfg::OutP::slot(y + 1, x + 1) : Cfg::OutS::slot(y + 1, x + 1);
                            *reinterpret_cast<uint32_t*>(outp + ((size_t)(ch / 8) * Cfg::OUT_NPIX + slot) * 16 + (ch & 7) * 2) = hi;
                            if (OSA) *reinterpret_cast<uint32_t*>(outp + ((size_t)(COUT / 8 + ch / 8) * Cfg::OUT_NPIX + slot) * 16 + (ch & 7) * 2) = lo;
                        }
                    }
                }
            }
            bar_sync(3 + wg, 128);   // every warp of the warpgroup has finished its MMAs on this stage
            if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);
            it++;
        }
    } else if (FIRST) {
        // ===== fused first layer (warps 9-16): sampler (or patch load) -> input_norm -> conv3x3(1 -> CIN) + ReLU -> fp16 stage =====
        static_assert(!FIRST || (H == 32 && STRIDE == 1), "the first conv layer feeds a stride-1 32x32 layer");
        float* s_patch = reinterpret_cast<float*>(sIn + (size_t)STAGES * Cfg::IN_BYTES);  // [2][34][36]
        float* s_w1 = s_patch + 2 * 34 * 36;                                               // [9][CIN]
        float* s_b1 = s_w1 + 9 * CIN;                                                      // [CIN]
        float* s_red = s_b1 + CIN;                                                         // [8][2] (+pad)
        const int pt = threadIdx.x - 288;  // 0..255
        const int pw = warp - 9;
        for (int i = pt; i < 9 * CIN; i += 256) s_w1[i] = src.w1[i];
        if (pt < CIN) s_b1[pt] = src.b1[pt];
        for (int i = pt; i < 2 * 34 * 36; i += 256) s_patch[i] = 0.f;
        // the zero border / slack of the stages is written once: conv1 only ever writes interior slots
        for (int i = pt; i < (int)(STAGES * Cfg::IN_BYTES / 16); i += 256) reinterpret_cast<uint4*>(sIn)[i] = make_uint4(0, 0, 0, 0);
        bar_sync(1, 256);
        // raw bilinear taps of the NEXT patch are requested before the conv of the current one so that their latency hides
        // behind compute (software prefetch): 16 values + the two fractional weights per pixel.
        float tp[4][4], fx[4], fy[4];
        auto issue_fetch = [&](int pi) {
            if (src.patches != nullptr) {
                const float* pp = src.patches + (size_t)pi * 1024;
#pragma unroll
                for (int k = 0; k < 4; k++) { tp[k][0] = pp[pt + k * 256]; tp[k][1] = tp[k][2] = tp[k][3] = 0.f; fx[k] = 0.f; fy[k] = 0.f; }
            } else {
                const int b = pi / src.cap;
                const int o = min(max(src.oct[pi], 0), src.geom.n_octaves - 1), l = min(max(src.lvl[pi], 0), src.geom.n_levels - 1);
                const int h = src.geom.h[o], w = src.geom.w[o];
                const float* img = src.pyr + src.geom.off[o][l] + (size_t)b * h * w;
                const float* Lf = src.lafs + (size_t)pi * 6;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int p = pt + k * 256;
                    float px, py;
                    laf_sample_xy(Lf, h, w, p >> 5, p & 31, 1.0f / 32.0f, px, py);
                    bilinear_taps(img, h, w, px, py, tp[k], fx[k], fy[k]);
                }
            }
        };
        int pi = blockIdx.x;
        while (pi < a.n && !valid(pi)) pi += gridDim.x;
        if (pi < a.n) issue_fetch(pi);
        int it = 0;
        while (pi < a.n) {
            const int s = it % STAGES;
            float* sp = s_patch + (it & 1) * 34 * 36;
            float v4[4];
#pragma unroll
            for (int k = 0; k < 4; k++) v4[k] = bilinear_combine(tp[k], fx[k], fy[k]);
            int pn = pi + gridDim.x;
            while (pn < a.n && !valid(pn)) pn += gridDim.x;
            if (pn < a.n) issue_fetch(pn);
            // 2. input_norm statistics over the 256 producer threads
            float sm = (v4[0] + v4[1]) + (v4[2] + v4[3]);
            for (int o = 16; o > 0; o >>= 1) sm += __shfl_xor_sync(0xffffffffu, sm, o);
            if (lane == 0) s_red[pw * 2 + (it & 1) * 16] = sm;
            bar_sync(1, 256);
            sm = 0.f;
#pragma unroll
            for (int i = 0; i < 8; i++) sm += s_red[i * 2 + (it & 1) * 16];
            const float mean = sm / 1024.f;
            float q = 0.f;
#pragma unroll
            for (int k = 0; k < 4; k++) { const float d = v4[k] - mean; q = fmaf(d, d, q); }
            for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
            if (lane == 0) s_red[pw * 2 + 1 + (it & 1) * 16] = q;
#pragma unroll
            for (int k = 0; k < 4; k++) { const int p = pt + k * 256; sp[((p >> 5) + 1) * 36 + (p & 31) + 1] = v4[k] - mean; }
            bar_sync(1, 256);
            q = 0.f;
#pragma unroll
            for (int i = 0; i < 8; i++) q += s_red[i * 2 + 1 + (it & 1) * 16];
            const float inv = 1.f / (sqrtf(q / 1023.f) + 1e-7f);
            // 3. conv1 + ReLU -> fp16 canonical stage (wait until the MMAs of the previous use of this stage are done)
            mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
            unsigned char* st = sIn + (size_t)s * Cfg::IN_BYTES;
#pragma unroll 1
            for (int k2 = 0; k2 < 2; k2++) {  // two pixels at a time: weights are read once for both
                const int p0 = pt + (2 * k2) * 256, p1 = p0 + 256;
                const int y0 = p0 >> 5, x0 = p0 & 31, y1 = p1 >> 5, x1 = p1 & 31;
                float acc0[CIN], acc1[CIN];
#pragma unroll
                for (int c = 0; c < CIN; c++) { acc0[c] = s_b1[c]; acc1[c] = acc0[c]; }
#pragma unroll
                for (int tap = 0; tap < 9; tap++) {
                    const float av0 = sp[(y0 + tap / 3) * 36 + x0 + tap % 3] * inv, av1 = sp[(y1 + tap / 3) * 36 + x1 + tap % 3] * inv;
#pragma unroll
                    for (int c4 = 0; c4 < CIN / 4; c4++) {
                        const float4 wv = *reinterpret_cast<const float4*>(s_w1 + tap * CIN + c4 * 4);
                        acc0[c4 * 4 + 0] = fmaf(av0, wv.x, acc0[c4 * 4 + 0]); acc1[c4 * 4 + 0] = fmaf(av1, wv.x, acc1[c4 * 4 + 0]);
                        acc0[c4 * 4 + 1] = fmaf(av0, wv.y, acc0[c4 * 4 + 1]); acc1[c4 * 4 + 1] = fmaf(av1, wv.y, acc1[c4 * 4 + 1]);
                        acc0[c4 * 4 + 2] = fmaf(av0, wv.z, acc0[c4 * 4 + 2]); acc1[c4 * 4 + 2] = fmaf(av1, wv.z, acc1[c4 * 4 + 2]);
                        acc0[c4 * 4 + 3] = fmaf(av0, wv.w, acc0[c4 * 4 + 3]); acc1[c4 * 4 + 3] = fmaf(av1, wv.w, acc1[c4 * 4 + 3]);
                    }
                }
#pragma unroll
                for (int half = 0; half < 2; half++) {
                    const float* acc = half ? acc1 : acc0;
                    const int slot = half ? In::slot(y1 + 1, x1 + 1) : In::slot(y0 + 1, x0 + 1);
#pragma unroll
                    for (int g = 0; g < CIN / 8; g++) {
                        float v[8];
#pragma unroll
                        for (int e = 0; e < 8; e++) v[e] = fmaxf(acc[g * 8 + e], 0.f);
                        uint4 pk;
                        pk.x = pack_h2(v[0], v[1]); pk.y = pack_h2(v[2], v[3]); pk.z = pack_h2(v[4], v[5]); pk.w = pack_h2(v[6], v[7]);
                        *reinterpret_cast<uint4*>(st + ((size_t)g * In::NPIX + slot) * 16) = pk;
                        if (SA) {
                            float lo[8];
#pragma unroll
                            for (int e = 0; e < 8; e++) lo[e] = v[e] - __half2float(__float2half_rn(v[e]));
                            pk.x = pack_h2(lo[0], lo[1]); pk.y = pack_h2(lo[2], lo[3]); pk.z = pack_h2(lo[4], lo[5]); pk.w = pack_h2(lo[6], lo[7]);
                            *reinterpret_cast<uint4*>(st + ((size_t)(CIN / 8 + g) * In::NPIX + slot) * 16) = pk;
                        }
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to the tensor core
            mbar_arrive(&full[s]);
            it++;
            pi = pn;
        }
    }
}

}  // namespace tc
}  // namespace ag
