// First two conv layers of AffNet / OriNet / HardNet in ONE kernel (AffNet / OriNet: three, L3 below), second-generation formulation
// (see tcx_conv.cuh):
//
//   sampler (LAF.py:313-372) -> input_norm (architectures.py:231-235) -> conv3x3(1 -> C1)+BN+ReLU -> conv3x3(C1 -> COUT)+BN+ReLU
//
// 32x32 patches and the layer-1 activations never exist in HBM.  M = 64 blocks are 64 consecutive pixels = 2 image rows of 32 (16
// blocks per patch, no padded columns; each half row of 16 pixels in the neighbour-paired order of tcx_conv.cuh, even x first, which
// the P planes set and every later stage keeps).  Layer 1 (K = 9): the sliding-window plane P[y*32 + x] = {4 pixels of padded row y from
// column x | 4 pixels of padded row y+1} makes one K = 16 MMA cover kernel rows 0 and 1, the same plane two rows further (descriptor
// leading-byte offset) kernel row 2.  Layer 2: for kernel row dy one MMA over the layer-1 stage advanced by dy rows with the three
// taps of that row stacked along N (N = 3*COUT); the epilogue shifts the dx = 0 / dx = 2 blocks by one pixel with warp shuffles, and
// through shared memory where an image row continues in the next warp (a warp holds 16 accumulator rows, half an image row).
// Split precision: the input and layer-1 weights always carry fp16 residual planes; SA / SW / OSA as in tcx_conv.cuh.
// L3 = 1 (AffNet / OriNet): layer 3 (stride 2, 32x32 -> 16x16) runs in the same kernel.  Layer 2's epilogue then writes its hi / lo
// values into shared memory, in the parity planes a stride-2 tcx_conv_kernel would load (a zero row, then 256 data slots per plane),
// instead of to HBM, and once both warpgroups are done each runs layer 3's blocks wg, wg + 2 with tcx_conv_kernel's own block functions
// (xconv_block_issue / xconv_block_epilogue), writing L_S1_16 hi + lo planes to HBM.  The 64 KiB per patch of layer 2's output never
// leave the SM.  To make room, the layer-1 stage is single-buffered (see the consumer loop).
//
// Warp roles (16 warps): 0-7 sampler + input_norm + P planes (two halves with their own barriers, so that the producers build one
// half while the MMAs read the other) | 8-15 two consumer warpgroups: layer 1 of a patch (MMA, then bias/ReLU -> fp16 stage in shared
// memory), then its layer 2 (MMA, then x shifts -> bias/ReLU -> fp16 -> global, stride-2 consumer layout; L3: -> shared memory, then
// layer 3); warpgroup g takes the blocks g, g + 2, ... of each layer.
// Within a layer each consumer warpgroup keeps two blocks in flight: it issues and commits the MMAs of its next block, waits until only
// that group is pending (wgmma_wait<1>) and runs the epilogue of the previous one, so the tensor core works through one block while
// the warpgroup's epilogue of the other runs.  The second accumulator set is what the producers' registers pay for (setmaxnreg:
// producers 96, consumers 160 per thread).
#pragma once
#include "tcx_conv.cuh"

// AG_FIRST_TIMELINE (developer builds, scripts/first_kernel_timeline.py): every warp of CTAs 0 .. TL_CTAS - 1 adds up the SM cycles
// (clock64) it spends in each TL_* state and stores the sums per launch in g_first_tl; ag_first_timeline_read copies them out.
#ifdef AG_FIRST_TIMELINE
#define AG_TL(state, ...) do { const long long t_ = clock64(); __VA_ARGS__; tl[state] += (unsigned long long)(clock64() - t_); } while (0)
#else
#define AG_TL(state, ...) do { __VA_ARGS__; } while (0)
#endif

namespace ag {
namespace tcx {

// timeline states: consumers  TOTAL | wait p_full | issue MMAs | wgmma_wait | warpgroup barrier | barrier of both warpgroups
//                  producers  TOTAL | wait p_empty | -          | -          | barrier 1 (input_norm) | - | build the P planes
enum { TL_TOTAL, TL_WAIT_P, TL_ISSUE, TL_MMA_WAIT, TL_WG_BAR, TL_STAGE_BAR, TL_PBUILD, TL_STATES };
#ifdef AG_FIRST_TIMELINE
constexpr int TL_CTAS = 4, TL_LAUNCHES = 8;
__device__ unsigned long long g_first_tl[TL_LAUNCHES][TL_CTAS][16][TL_STATES];
__device__ int g_first_tl_launch[TL_CTAS];
#endif

// Four 8x8 16-bit matrices to shared memory in one instruction.  r0 .. r3: the thread's packed accumulator-fragment word of each
// (row lane/4, columns 2 (lane%4) and + 1); row: the 16-byte address of row lane%8 of matrix lane/8 that this lane supplies.
__device__ __forceinline__ void stmatrix_x4(const void* row, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(smem_u32(row)), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
                 : "memory");
}

template <int C1, int COUT, int SA, int SW, int OSA, int L3 = 0>
struct XFirstCfg {
    using X3 = XCfg<COUT, 2 * COUT, 32, 2, 1, 1, L_S1_16, 1, 1, 1>;   // layer 3 (L3 = 1): its input planes as ONE stage in shared memory
    static constexpr int KC = C1 / 8, NT = COUT;
    static constexpr int BLOCKS = 16;                          // M = 64 blocks of a patch
    static constexpr int NPIXP = 18 * 32;                      // slots of one HALF P plane: 18 window rows (16 image rows of outputs + 2 rows of look-ahead)
    static constexpr int SX = 1200;                            // floats of one padded fp32 patch buffer: 34*34 + zero tail (windows of row 33 look one row further)
    static constexpr int S1 = (C1 == 16) ? 1 : 0;              // layer 1: x_hi * [w_hi ; w_lo] as one N = 2*C1 MMA
    static constexpr int ACC1 = 32;                            // layer-1 accumulator columns (2*16 stacked, or 32)
    static constexpr int ACCW = 3 * NT;
    static constexpr int G = KC * (1 + SA);
    static constexpr int SLOT_STAGE = 1024 + 32;               // zero row + 32 data rows; the zero row below is the next stage's / the trailing one
    static constexpr int NSTAGE = L3 ? 1 : 2;                  // layer-1 stages (L3: single-buffered)
    static constexpr int GS = NSTAGE * SLOT_STAGE + 32;
    static constexpr int NR = (1 + SW) * 3 * NT;               // weight rows per K group of a (dy, k step) block
    static constexpr uint32_t W_BYTES = 9u * C1 * NT * 2u * (1 + SW);
    static constexpr uint32_t IN_BYTES = (uint32_t)G * GS * 16u;
    static constexpr uint32_t W1_BYTES = 2u * 2u * C1 * 16;    // [K chunk 0|1][hi rows | lo rows][8]
    static constexpr uint32_t P_BYTES = 2u * 2u * NPIXP * 16;   // [half][hi | lo][NPIXP]: the halves are built and consumed alternately
    static constexpr uint32_t XCH_BYTES = 2u * 2u * 4u * 2u * NT * 4u;   // [warpgroup][block parity][warp][left | right][NT] row-boundary values
    static constexpr uint32_t W3_BYTES = L3 ? X3::W_BYTES : 0u;     // layer-3 weights
    static constexpr uint32_t IN3_BYTES = L3 ? X3::IN_BYTES : 0u;   // layer-3 input planes = layer 2's output
    static constexpr size_t SMEM = 1024 + (size_t)W_BYTES + W3_BYTES + IN_BYTES + IN3_BYTES + P_BYTES + W1_BYTES + 2 * SX * 4 + 256 + XCH_BYTES;
    static constexpr size_t HI_OUT_BYTES = (size_t)(COUT / 8) * 1024 * 16;
    static constexpr size_t UNIT_OUT_BYTES = HI_OUT_BYTES * (1 + OSA);
    static constexpr int THREADS = 512;
    static constexpr int REG_PRODUCER = 96, REG_CONSUMER = 160;   // setmaxnreg: 256 threads of each role share the 64 Ki registers
    static_assert(256 * (REG_PRODUCER + REG_CONSUMER) <= 65536 && REG_PRODUCER % 8 == 0 && REG_CONSUMER % 8 == 0, "register split");
    static_assert(BLOCKS % 4 == 0 && (!L3 || X3::BLOCKS == 4), "two blocks in flight per warpgroup: an even count of blocks each");
    static_assert(C1 % 16 == 0 && NT % 16 == 0 && ACCW <= 256, "shape");
    static_assert(SA <= 1 && SW <= 1 && OSA <= 1, "split-precision switches are 0 | 1");
    static_assert(!L3 || (OSA == 1 && X3::NT <= 32), "layer 3 reads hi + lo planes; its bias fits smem[640, 768)");
    static_assert(C1 == 16 || C1 == 32, "layer-1 accumulator width");
    static_assert(SA || KC % 2 == 0, "layer-1 epilogue: one stmatrix.x4 per channel group (hi + lo) or per two (hi only)");
    static_assert(SMEM <= 232448, "shared memory budget");
};

// a: layer 2 (L3 = 0: a.out receives its output), a3: layer 3 (L3 = 1 only; a3.in unused)
template <int C1, int COUT, int SA, int SW, int OSA, int BF = 0, int L3 = 0>
__global__ void __launch_bounds__(512, 1) tcx_first_kernel(const XArgs a, const FirstSrc src, const XArgs a3) {
    using Cfg = XFirstCfg<C1, COUT, SA, SW, OSA, L3>;
    using X3 = typename Cfg::X3;
    constexpr int KC = Cfg::KC, NT = Cfg::NT, ACCW = Cfg::ACCW, NPIXP = Cfg::NPIXP, SX = Cfg::SX, GS = Cfg::GS;
    extern __shared__ __align__(1024) unsigned char smem[];
    uint64_t* wbar = reinterpret_cast<uint64_t*>(smem);
    uint64_t* p_full = wbar + 1;                            // [2] half P plane written (256 producer threads)
    uint64_t* p_empty = p_full + 2;                         // [2] layer-1 MMAs done with the half (2 warpgroups)
    float* s_bias1 = reinterpret_cast<float*>(smem + 384);  // [C1]
    float* s_bias = reinterpret_cast<float*>(smem + 512);   // [NT]
    float* s_bias3 = reinterpret_cast<float*>(smem + 640);  // [X3::NT] (L3)
    unsigned char* sW = smem + 1024;
    unsigned char* sW3 = sW + Cfg::W_BYTES;                 // layer-3 weights (L3)
    unsigned char* sIn = sW3 + Cfg::W3_BYTES;               // [G][NSTAGE stages][zero row | 32 data rows] + trailing zero row
    unsigned char* sIn3 = sIn + Cfg::IN_BYTES;              // (L3) [X3::G][4 parity planes][zero row | 256 data slots]
    unsigned char* sP = sIn3 + Cfg::IN3_BYTES;              // [half][hi|lo][NPIXP][8] fp16
    unsigned char* sW1 = sP + Cfg::P_BYTES;                 // [chunk][hi|lo][C1][8] fp16
    float* s_x = reinterpret_cast<float*>(sW1 + Cfg::W1_BYTES);   // [2][SX]
    float* s_red = s_x + 2 * SX;                            // [2][8][2]
    float* s_xch = s_red + 64;                              // [2][2][4][2][NT]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    auto valid = [&](int pi) -> bool { return a.count == nullptr || (pi % a.group) < a.count[pi / a.group]; };
    auto next_valid = [&](int pi) -> int {
        while (pi < a.n && !valid(pi)) pi += gridDim.x;
        return pi;
    };

    // ---- one-time setup by all threads ----
    if (threadIdx.x < NT) s_bias[threadIdx.x] = a.bias[threadIdx.x];
    if (threadIdx.x < C1) s_bias1[threadIdx.x] = src.b1[threadIdx.x];
    if (L3 && threadIdx.x < X3::NT) s_bias3[threadIdx.x] = a3.bias[threadIdx.x];
    if (threadIdx.x == 0) {
        mbar_init(wbar, 1);
        for (int hh = 0; hh < 2; hh++) { mbar_init(&p_full[hh], 256); mbar_init(&p_empty[hh], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
#ifdef AG_FIRST_TIMELINE
    int* s_tl_slot = reinterpret_cast<int*>(smem + 128);    // this launch's slot in g_first_tl (TL_LAUNCHES: not recorded)
    if (threadIdx.x == 0) *s_tl_slot = blockIdx.x < TL_CTAS ? min(atomicAdd(&g_first_tl_launch[blockIdx.x], 1), TL_LAUNCHES) : TL_LAUNCHES;
    unsigned long long tl[TL_STATES] = {};
#endif
    for (int i = threadIdx.x; i < 2 * 2 * C1 * 8; i += blockDim.x) {   // W1[chunk][hi rows | lo rows][e]: chunk 0 = kernel rows 0 (e 0..2), 1 (e 4..6); chunk 1 = kernel row 2
        const int e = i & 7, co = (i >> 3) % C1, part = (i / (8 * C1)) & 1, ch = i / (8 * C1 * 2);
        const int dy = ch == 0 ? (e >> 2) : 2, dx = e & 3;
        float v = 0.f;
        if (dx < 3 && (ch == 0 || e < 4)) {
            const float wv = src.w1[(dy * 3 + dx) * C1 + co] * src.w1_scale;   // power-of-two scale, undone in the epilogue
            const float hi = unpack2<BF>(pack2<BF>(wv, 0.f)).x;      // wv rounded to the operand format
            v = part == 0 ? hi : wv - hi;
        }
        reinterpret_cast<unsigned short*>(sW1)[i] = (unsigned short)(pack2<BF>(v, 0.f) & 0xFFFFu);
    }
    // zero rows of the stages and of the layer-3 planes: written once, the epilogues only ever write data slots
    for (int i = threadIdx.x; i < (int)((Cfg::IN_BYTES + Cfg::IN3_BYTES + Cfg::P_BYTES) / 16); i += blockDim.x) reinterpret_cast<uint4*>(sIn)[i] = make_uint4(0, 0, 0, 0);
    for (int i = threadIdx.x; i < 2 * SX; i += blockDim.x) s_x[i] = 0.f;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
#ifdef AG_FIRST_TIMELINE
    const long long tl_start = clock64();
#endif

    if (warp >= 8) {
        // ===== consumers =====
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::REG_CONSUMER));
        const int wg = (warp - 8) >> 2, wq = warp & 3;
        if (threadIdx.x == 256) {
            mbar_expect_tx(wbar, Cfg::W_BYTES + Cfg::W3_BYTES);
            bulk_g2s(sW, a.wpk, Cfg::W_BYTES, wbar);
            if (L3) bulk_g2s(sW3, a3.wpk, Cfg::W3_BYTES, wbar);
        }
        mbar_wait(wbar, 0);
        const uint32_t w_base = smem_u32(sW) >> 4, in_base = smem_u32(sIn) >> 4;
        const uint32_t w3_base = smem_u32(sW3) >> 4, in3_base = smem_u32(sIn3) >> 4;
        const uint32_t w1_lo = desc_lo(smem_u32(sW1), 2 * C1 * 16u);       // K chunks are 2*C1 rows apart (hi rows, then lo rows)
        const uint32_t p_lo = desc_lo(smem_u32(sP), 2 * 32 * 16u);          // leading-byte offset = two image rows
        constexpr uint32_t LBO_A = ((uint32_t)GS) << 16;
        // layer 1 of block b (of half plane hh): issue and commit its MMAs into d1
        auto l1_issue = [&](float* d1, int hh, int b) {
            const uint32_t alo = p_lo + (uint32_t)(hh * 2 * NPIXP + (b & 7) * 64);
            wgmma_fence();
            if (Cfg::S1) {   // x_hi * [w_hi ; w_lo] in one MMA, then x_lo * w_hi
                Wgmma<2 * C1, BF>::mma(d1, desc64(alo), desc64(w1_lo), 0);
                Wgmma<C1, BF>::mma(d1, desc64(alo + (uint32_t)NPIXP), desc64(w1_lo), 1);
            } else {
                Wgmma<C1, BF>::mma(d1, desc64(alo), desc64(w1_lo), 0);
                Wgmma<C1, BF>::mma(d1, desc64(alo + (uint32_t)NPIXP), desc64(w1_lo), 1);             // x_lo * w_hi
                Wgmma<C1, BF>::mma(d1, desc64(alo), desc64(w1_lo + (uint32_t)C1), 1);                 // x_hi * w_lo (lo rows follow the hi rows)
            }
            wgmma_commit();
        };
        // its epilogue, once the MMAs have completed: bias / ReLU -> fp16 (hi [+lo]) into stage st of layer 2
        // (M row = stage slot: the P planes are built in the stage's neighbour-paired order)
        auto l1_epilogue = [&](float* d1, unsigned char* st, int b) {
            wgmma_reg_fence<Cfg::ACC1 / 2>(d1);
            uint32_t hi[KC][2], lo[KC][2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
#pragma unroll
                for (int j = 0; j < KC; j++) {
                    const int c = j * 8 + 2 * (lane & 3);
                    float v0 = d1[4 * j + 2 * h], v1 = d1[4 * j + 2 * h + 1];
                    if (Cfg::S1) { v0 += d1[4 * (j + 2) + 2 * h]; v1 += d1[4 * (j + 2) + 2 * h + 1]; }   // [x*w_hi | x_hi*w_lo] side by side
                    v0 = fmaxf(fmaf(v0, src.w1_inv, s_bias1[c]), 0.f);
                    v1 = fmaxf(fmaf(v1, src.w1_inv, s_bias1[c + 1]), 0.f);
                    split_pack2<SA, BF>(v0, v1, hi[j][h], lo[j][h]);
                }
            }
            // matrix mx = lane / 8: rows h = mx % 2 of channel group j (SA: of the hi plane for mx < 2, else the lo plane; without
            // SA: of group j + mx / 2)
            const int mx = lane >> 3;
            const int slot = b * 64 + wq * 16 + (lane & 7) + 8 * (mx & 1) + 32;     // pixel m sits one (zero) row into the stage
#pragma unroll
            for (int j = 0; j < KC; j += SA ? 1 : 2) {
                if constexpr (SA) stmatrix_x4(st + ((size_t)((mx >> 1) * KC + j) * GS + slot) * 16, hi[j][0], hi[j][1], lo[j][0], lo[j][1]);
                else stmatrix_x4(st + ((size_t)(j + (mx >> 1)) * GS + slot) * 16, hi[j][0], hi[j][1], hi[j + 1][0], hi[j + 1][1]);
            }
        };
        // block k = 0 .. 7 of this warpgroup's layer-1 blocks: half plane k / 4, block 8 (k / 4) + wg + 2 (k % 4)
        auto l1_block = [&](int k) -> int { return (k >> 2) * 8 + wg + 2 * (k & 3); };
        int it = 0, nblk = 0;
        for (int pi = next_valid(blockIdx.x); pi < a.n; pi = next_valid(pi + gridDim.x), it++) {
            // L3: one stage.  Layer 1 of the next patch overwrites it only after the barrier between layers 2 and 3 below, which
            // both warpgroups reach after their last layer-2 MMAs have completed (the layer-2 loop ends in wgmma_wait<0>): nobody
            // still reads it.
            const int s = L3 ? 0 : (it & 1);
            unsigned char* st = sIn + (size_t)s * Cfg::SLOT_STAGE * 16;
            // ---- layer 1, half plane by half plane -> fp16 (hi [+lo]) stage of layer 2; block k + 1's MMAs run during block k's
            // epilogue (the second half plane is waited for before its first block is issued) ----
            float d1[2][Cfg::ACC1 / 2];
            AG_TL(TL_WAIT_P, mbar_wait(&p_full[0], it & 1));
            AG_TL(TL_ISSUE, l1_issue(d1[0], 0, l1_block(0)));
#pragma unroll
            for (int k = 0; k < 8; k++) {
                if (k < 7) {
                    if (k == 3) AG_TL(TL_WAIT_P, mbar_wait(&p_full[1], it & 1));
                    AG_TL(TL_ISSUE, l1_issue(d1[(k + 1) & 1], (k + 1) >> 2, l1_block(k + 1)));
                    AG_TL(TL_MMA_WAIT, wgmma_wait<1>());
                } else {
                    AG_TL(TL_MMA_WAIT, wgmma_wait<0>());
                }
                l1_epilogue(d1[k & 1], st, l1_block(k));
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> visible to the tensor core
            AG_TL(TL_STAGE_BAR, bar_sync(2, 256));   // the whole stage is written (both warpgroups)
            // p_empty means "the layer-1 MMAs of both warpgroups have completed on the half", not merely been issued: every consumer
            // thread passed its wgmma_wait<0> above before the barrier.  Both halves are released here, the producers build the
            // next patch's planes during this patch's layer 2.
            if ((threadIdx.x & 127) == 0) { mbar_arrive(&p_empty[0]); mbar_arrive(&p_empty[1]); }
            // ---- layer 2: block k + 1's MMAs run during block k's epilogue ----
            unsigned char* outp = L3 ? nullptr : reinterpret_cast<unsigned char*>(a.out) + (size_t)pi * Cfg::UNIT_OUT_BYTES;
            const uint32_t st_base = in_base + (uint32_t)(s * Cfg::SLOT_STAGE);
            auto l2_issue = [&](float* d, int b) {
                const uint32_t a_t = st_base + (uint32_t)(b * 64);
                wgmma_fence();
#pragma unroll
                for (int dy = 0; dy < 3; dy++) {
#pragma unroll
                    for (int j = 0; j < KC / 2; j++) {
                        const uint32_t ahi = ((a_t + (uint32_t)(dy * 32 + 2 * j * GS)) & 0x3FFFu) | LBO_A;
                        const uint32_t alo = ((a_t + (uint32_t)(dy * 32 + (KC + 2 * j) * GS)) & 0x3FFFu) | LBO_A;
                        const uint32_t blk = w_base + (uint32_t)((dy * (KC / 2) + j) * 2 * Cfg::NR);
                        const uint32_t bhi = (blk & 0x3FFFu) | ((uint32_t)Cfg::NR << 16), blo = ((blk + 3 * NT) & 0x3FFFu) | ((uint32_t)Cfg::NR << 16);
                        Wgmma<3 * NT, BF>::mma(d, desc64(ahi), desc64(bhi), (dy | j) != 0);
                        if (SW) Wgmma<3 * NT, BF>::mma(d, desc64(ahi), desc64(blo), 1);
                        if (SA) Wgmma<3 * NT, BF>::mma(d, desc64(alo), desc64(bhi), 1);
                    }
                }
                wgmma_commit();
            };
            // epilogue of block b, the warpgroup's nb-th layer-2 block, once its MMAs have completed
            auto l2_epilogue = [&](float* d, int b, int nb) {
                wgmma_reg_fence<ACCW / 2>(d);
                // rows r = 16 wq + lane/4 + 8 h of the block: image row y = (64 b + 16 wq) / 32, x = 16 (wq % 2) + 2 (lane/4) + h
                // (neighbour-paired half rows).  Warps 2k and 2k+1 share an image row: x = 15 (lanes 28-31, h = 1, of the even warp) and
                // x = 16 (lanes 0-3, h = 0, of the odd one) exchange their dx = 0 / dx = 2 values through shared memory.
                // The exchange is double-buffered by block parity and a warpgroup runs its epilogues one at a time in block order (the
                // second block in flight is in MMAs, not in an epilogue): a warp rewrites a buffer only after every warp of the warpgroup
                // has passed the barrier of the following block, so after it read the buffer.
                float* xw = s_xch + (size_t)((wg * 2 + (nb & 1)) * 4) * 2 * NT;
                if (lane >= 28) {
#pragma unroll
                    for (int j = 0; j < NT / 8; j++) {
                        const int c = j * 8 + 2 * (lane & 3);
                        xw[(wq * 2 + 0) * NT + c] = d[4 * j + 2]; xw[(wq * 2 + 0) * NT + c + 1] = d[4 * j + 3];   // row 15, dx = 0
                    }
                }
                if (lane < 4) {
#pragma unroll
                    for (int j = 0; j < NT / 8; j++) {
                        const int c = j * 8 + 2 * (lane & 3);
                        xw[(wq * 2 + 1) * NT + c] = d[4 * (j + 2 * NT / 8)]; xw[(wq * 2 + 1) * NT + c + 1] = d[4 * (j + 2 * NT / 8) + 1];   // row 0, dx = 2
                    }
                }
                AG_TL(TL_WG_BAR, bar_sync(3 + wg, 128));
                const int y0 = (b * 64 + wq * 16) >> 5;
                const int x0 = (wq & 1) * 16 + 2 * (lane >> 2);         // h = 0 (even pixel); h = 1 is x0 + 1
                // Each pixel keeps the rounding it had when row i + 8 h of a warp was pixel 16 (wq % 2) + i + 8 h: the first 8 pixels
                // of a half row (lanes 0-15 now) l + (r + c), with the left neighbour masked at x = 0, the last 8 (lanes 16-31)
                // r + (l + c), with the right one masked at x = 31.  sum = fmaf(outer, mask, inner + c).
                const bool first8 = lane < 16;
                const float m0 = (first8 && x0 == 0) ? 0.f : 1.f, m1 = (!first8 && x0 + 1 == 31) ? 0.f : 1.f;
                const bool from_prev = (wq & 1) && lane < 4, from_next = !(wq & 1) && lane >= 28;
                // L3: the shared-memory row of the layer-3 planes that this lane supplies to stmatrix: row lane % 8 of matrix
                // mx = lane / 8 = rows h = mx % 2 of the hi (mx < 2) or lo plane
                size_t s3 = 0;
                if (L3) {
                    using In3 = typename X3::In;
                    const int mx = lane >> 3;
                    const int slot = layout_slot(L_S2_16, y0, (wq & 1) * 16 + 2 * (lane & 7) + (mx & 1), 0);
                    s3 = (size_t)(mx >> 1) * X3::KC * X3::GS + (size_t)(slot / In3::DATA) * In3::PLANE + In3::RW + slot % In3::DATA;
                }
#pragma unroll
                for (int j = 0; j < NT / 8; j++) {
                    const int c = j * 8 + 2 * (lane & 3);
                    // neighbours (tcx_conv.cuh, frag_left_even) of both columns: x0 - 1 from lane - 4, x0 + 2 from lane + 4, or across
                    // the two warps of the image row from shared memory (one 8-byte load each)
                    float2 l0 = make_float2(frag_left_even(d[4 * j + 2], lane), frag_left_even(d[4 * j + 3], lane));
                    float2 r1 = make_float2(frag_right_odd(d[4 * (j + 2 * NT / 8)], lane), frag_right_odd(d[4 * (j + 2 * NT / 8) + 1], lane));
                    if (from_prev) l0 = *reinterpret_cast<const float2*>(xw + ((wq - 1) * 2 + 0) * NT + c);
                    if (from_next) r1 = *reinterpret_cast<const float2*>(xw + ((wq + 1) * 2 + 1) * NT + c);
                    float v[2][2];
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const float l1 = d[4 * j + e], c10 = d[4 * (j + NT / 8) + e], c11 = d[4 * (j + NT / 8) + 2 + e], r0 = d[4 * (j + 2 * NT / 8) + 2 + e];
                        const float le = e ? l0.y : l0.x, re = e ? r1.y : r1.x;
                        // 0/1 masks: zero padding outside the row (x = 0: h = 0 of even warps' lanes 0-3, x = 31: h = 1 of odd warps' lanes 28-31)
                        const float acc0 = fmaf(first8 ? le : r0, m0, (first8 ? r0 : le) + c10);
                        const float acc1 = fmaf(first8 ? l1 : re, m1, (first8 ? re : l1) + c11);
                        v[0][e] = fmaxf(fmaf(acc0, a.inv_scale, s_bias[c + e]), 0.f);
                        v[1][e] = fmaxf(fmaf(acc1, a.inv_scale, s_bias[c + e]), 0.f);
                    }
                    uint32_t hi[2], lo[2];
#pragma unroll
                    for (int h = 0; h < 2; h++) split_pack2<OSA, BF>(v[h][0], v[h][1], hi[h], lo[h]);
                    if (L3) {   // rows h = 0 / 1 lie in the even-x / odd-x parity plane
                        stmatrix_x4(sIn3 + ((size_t)j * X3::GS + s3) * 16, hi[0], hi[1], lo[0], lo[1]);
                    } else {
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const int slot = layout_slot(L_S2_16, y0, x0 + h, 0);
                            const size_t goff = (size_t)(c / 8) * 1024 * 16;
                            *reinterpret_cast<uint32_t*>(outp + goff + (size_t)slot * 16 + (c & 7) * 2) = hi[h];
                            if (OSA) *reinterpret_cast<uint32_t*>(outp + (size_t)(COUT / 8) * 1024 * 16 + goff + (size_t)slot * 16 + (c & 7) * 2) = lo[h];
                        }
                    }
                }
            };
            // this warpgroup's blocks wg + 2 k, k = 0 .. 7: d[k & 1].  Unrolled: with MMAs in flight across a loop's back edge ptxas
            // serialises the wgmma pipeline.
            float d[2][ACCW / 2];
            AG_TL(TL_ISSUE, l2_issue(d[0], wg));
#pragma unroll
            for (int k = 0; k < Cfg::BLOCKS / 2; k++) {
                if (k + 1 < Cfg::BLOCKS / 2) {
                    AG_TL(TL_ISSUE, l2_issue(d[(k + 1) & 1], wg + 2 * (k + 1)));
                    AG_TL(TL_MMA_WAIT, wgmma_wait<1>());
                } else {
                    // the last layer-2 MMAs on the stage have completed: the barrier below (L3) or the next patch's "stage written"
                    // barrier releases the stage to the next layer-1 epilogue that writes it
                    AG_TL(TL_MMA_WAIT, wgmma_wait<0>());
                }
                l2_epilogue(d[k & 1], wg + 2 * k, nblk + k);
            }
            nblk += Cfg::BLOCKS / 2;
            if (L3) {
                // ---- layer 3: both warpgroups' layer-2 planes are written (and their layer-2 MMAs are done with the stage) ----
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                AG_TL(TL_STAGE_BAR, bar_sync(2, 256));
                // both of the warpgroup's blocks (wg, wg + 2) in flight, the second one's MMAs run during the first one's epilogue
                float d3[2][X3::ACCW / 2];
                AG_TL(TL_ISSUE, xconv_block_issue<X3, BF>(d3[0], in3_base + (uint32_t)(wg * 64), w3_base));
                AG_TL(TL_ISSUE, xconv_block_issue<X3, BF>(d3[1], in3_base + (uint32_t)((wg + 2) * 64), w3_base));
                AG_TL(TL_MMA_WAIT, wgmma_wait<1>());
                wgmma_reg_fence<X3::ACCW / 2>(d3[0]);
                xconv_block_epilogue<X3, BF>(d3[0], a3, s_bias3, pi, wg, 0, wq, lane);
                AG_TL(TL_MMA_WAIT, wgmma_wait<0>());
                wgmma_reg_fence<X3::ACCW / 2>(d3[1]);
                xconv_block_epilogue<X3, BF>(d3[1], a3, s_bias3, pi, wg + 2, 0, wq, lane);
                // sIn3 is rewritten by the next patch's layer-2 epilogue only after that patch's "stage written" barrier, which the
                // other warpgroup reaches after its layer-3 MMAs here have completed (wgmma_wait<0> above)
            }
        }
    } else {
        // ===== producers (8 warps): sampler (or patch load) -> input_norm -> sliding-window planes P_hi / P_lo =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::REG_PRODUCER));
        const int pw = warp;                                 // 0..7
        const int pt = pw * 32 + lane;                       // 0..255
        float tp[4][4], fx[4], fy[4];
        // pixel k of this thread: warp pw owns image rows 4pw .. 4pw+3; k = 8-column block, lane = (row, column) inside the 4x8 block
        auto pix_of = [&](int k) -> int { return (pw * 4 + (lane >> 3)) * 32 + k * 8 + (lane & 7); };
        auto issue_fetch = [&](int pi) {
            if (src.patches != nullptr) {
                const float* pp = src.patches + (size_t)pi * 1024;
#pragma unroll
                for (int k = 0; k < 4; k++) { tp[k][0] = pp[pix_of(k)]; tp[k][1] = tp[k][2] = tp[k][3] = 0.f; fx[k] = 0.f; fy[k] = 0.f; }
            } else {
                const int b = pi / src.cap;
                const int o = min(max(src.oct[pi], 0), src.geom.n_octaves - 1), l = min(max(src.lvl[pi], 0), src.geom.n_levels - 1);
                const int h = src.geom.h[o], w = src.geom.w[o];
                const float* img = src.pyr + src.geom.off[o][l] + (size_t)b * h * w;
                const float* Lf = src.lafs + (size_t)pi * 6;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const int p = pix_of(k);
                    float px, py;
                    laf_sample_xy(Lf, h, w, p >> 5, p & 31, 1.0f / 32.0f, px, py);
                    bilinear_taps(img, h, w, px, py, tp[k], fx[k], fy[k]);
                }
            }
        };
        int pi = next_valid(blockIdx.x);
        if (pi < a.n) issue_fetch(pi);
        int it = 0;
        while (pi < a.n) {
            float* sx = s_x + (it & 1) * SX;
            float* red = s_red + (it & 1) * 16;
            float v[4];
#pragma unroll
            for (int k = 0; k < 4; k++) v[k] = bilinear_combine(tp[k], fx[k], fy[k]);
            const int pn = next_valid(pi + gridDim.x);
            if (pn < a.n) issue_fetch(pn);
            // input_norm: mean, unbiased std + 1e-7 (two passes, as the reference)
            float sm = (v[0] + v[1]) + (v[2] + v[3]);
            for (int o = 16; o > 0; o >>= 1) sm += __shfl_xor_sync(0xffffffffu, sm, o);
            if (lane == 0) red[pw * 2] = sm;
            AG_TL(TL_WG_BAR, asm volatile("bar.sync 1, 256;" ::: "memory"));
            const float mean = (((red[0] + red[2]) + (red[4] + red[6])) + ((red[8] + red[10]) + (red[12] + red[14]))) / 1024.f;
            float qs = 0.f;
#pragma unroll
            for (int k = 0; k < 4; k++) { const float d = v[k] - mean; qs = fmaf(d, d, qs); }
            for (int o = 16; o > 0; o >>= 1) qs += __shfl_xor_sync(0xffffffffu, qs, o);
            if (lane == 0) red[pw * 2 + 1] = qs;
            AG_TL(TL_WG_BAR, asm volatile("bar.sync 1, 256;" ::: "memory"));
            const float inv = 1.f / (sqrtf((((red[1] + red[3]) + (red[5] + red[7])) + ((red[9] + red[11]) + (red[13] + red[15]))) / 1023.f) + 1e-7f);
#pragma unroll
            for (int k = 0; k < 4; k++) { const int p = pix_of(k); sx[((p >> 5) + 1) * 34 + (p & 31) + 1] = (v[k] - mean) * inv; }
            AG_TL(TL_WG_BAR, asm volatile("bar.sync 1, 256;" ::: "memory"));
            // P planes, half by half
#pragma unroll 1
            for (int hh = 0; hh < 2; hh++) {
                AG_TL(TL_WAIT_P, mbar_wait(&p_empty[hh], (it & 1) ^ 1));   // layer-1 MMAs of the previous patch have completed on this half
#ifdef AG_FIRST_TIMELINE
                const long long tb = clock64();
#endif
                unsigned char* ph = sP + (size_t)hh * 2 * NPIXP * 16;
                // one 16-byte window per thread and step: slot s0 holds the window of the pixel that M row s0 stands for (each half row
                // of 16 in the neighbour-paired order, tcx_conv.cuh), so a warp reads the 32 pixels of one row and writes consecutive
                // slots (no bank conflicts; the shared-memory pipe is this kernel's busiest unit)
#pragma unroll 1
                for (int s0 = pt; s0 < NPIXP; s0 += 256) {
                    const float* rowp = sx + (hh * 16 + (s0 >> 5)) * 34 + (s0 & 16) + 2 * (s0 & 7) + ((s0 >> 3) & 1);   // x with rpos(x & 15) = s0 & 15
                    float xv[8];
#pragma unroll
                    for (int e = 0; e < 4; e++) { xv[e] = rowp[e]; xv[4 + e] = rowp[34 + e]; }
                    uint4 hi, lo;
                    split_pack8<1, BF>(xv, hi, lo);
                    *reinterpret_cast<uint4*>(ph + (size_t)s0 * 16) = hi;
                    *reinterpret_cast<uint4*>(ph + (size_t)(NPIXP + s0) * 16) = lo;
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                mbar_arrive(&p_full[hh]);
#ifdef AG_FIRST_TIMELINE
                tl[TL_PBUILD] += (unsigned long long)(clock64() - tb);
#endif
            }
            it++;
            pi = pn;
        }
    }
#ifdef AG_FIRST_TIMELINE
    tl[TL_TOTAL] = (unsigned long long)(clock64() - tl_start);
    if (lane == 0 && *s_tl_slot < TL_LAUNCHES)
        for (int i = 0; i < TL_STATES; i++) g_first_tl[*s_tl_slot][blockIdx.x][warp][i] = tl[i];
#endif
}

}  // namespace tcx
}  // namespace ag
