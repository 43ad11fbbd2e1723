// Second-generation tensor-core (wgmma) 3x3 convolution engine (sm_90a): row tiles without x padding, taps of one kernel row
// stacked along N.
//
// An MMA with a small N (16 .. 64) spends most of its time reading its A operand from shared memory, so the three taps of a kernel
// ROW share one MMA:
//
//   pixel planes are stored WITHOUT x padding, so that an M = 64 block is 64 consecutive pixels = whole image rows (2 rows of 32,
//   4 rows of 16, or 4 rows of 8 of TWO patches interleaved row by row), and every warp's 16 accumulator rows are whole image rows
//   (or, at 32 pixels per row, half of one);
//   for kernel row dy the A operand is the input plane advanced by dy rows (descriptor start address; a zero row above and below
//   the plane in shared memory gives the y padding) and the B operand stacks the three taps of that row along N:
//        D[q, (dx, c)] += sum_ci  in[q + (dy-1) W, ci] * w[dy][dx][ci][c]             one MMA per (dy, 16 input channels), N = 3 C
//   the x shift moves to the epilogue:   out[p, c] = D[p-1, (0,c)] + D[p, (1,c)] + D[p+1, (2,c)]   (warp shuffles inside an image
//   row; the neighbour outside the row is the zero padding).
// Stride-2 layers read four parity planes; the taps dx = 0 and dx = 2 share the odd-x plane (N = 2 C), dx = 1 reads the even-x
// plane (N = C):   out[x] = Dodd[x-1, dx0] + Dodd[x, dx2] + Deven[x, dx1].
// Split precision: x = hi + lo fp16 planes (SA), w = hi + lo fp16 copies (SW), D = A_hi W_hi + A_hi W_lo + A_lo W_hi, each
// product its own MMA into the SAME accumulator registers.
//
// Activations between layers (HBM): fp16, 16-byte slots of 8 channels, [unit][channel group (hi groups, then lo groups)][plane][slot],
// data rows only (the consumer's loader places them between zero rows in shared memory):
//   L_S2_16  stride-2 consumer on a 32x32 map   unit = patch   4 parity planes x 256 slots  slot = (y/2)*16 + rpos(x/2), plane = (y&1)*2 + (x&1)
//   L_S1_16  stride-1 consumer on a 16x16 map   unit = patch   256 slots                    slot = y*16 + rpos(x)
//   L_S2_8P  stride-2 consumer on a 16x16 map   unit = PAIR    4 parity planes x 128 slots  slot = (y/2)*16 + ppos(x/2, p)
//   L_S1_8P  stride-1 consumer on an 8x8 map    unit = PAIR    128 slots                    slot = y*16 + ppos(x, p)       (p = patch & 1)
//   L_HEAD   the 8x8 head GEMM's A operand (tc_head.cuh): [patch/128][pixel*C/8 + c/8][patch%128][8] (+ a residual plane behind it)
// Neighbour-paired order inside every 16-slot row group (one row of 16 pixels, or the 8 pixels of patch 0 and of patch 1 of one row):
// the even-x pixels first, then the odd-x pixels, so that M row i < 8 of a warp's 16 rows holds an even pixel and row i + 8 its right
// neighbour, and a thread (rows lane/4 and lane/4 + 8) holds both:
//   rpos(x) = (x&1)*8 + x/2                  x = 0 .. 15
//   ppos(x, p) = (x&1)*8 + p*4 + x/2         x = 0 .. 7: rows 0-3 patch 0 at x = 0, 2, 4, 6, rows 4-7 patch 1, rows 8-15 the odd x
// Whole rows stay whole rows, so the dy shift (one row further), the zero rows and the M = 64 blocks are those of the natural order.
// The 32x32 layer-1 stage of tcx_first_kernel orders each half row of 16 pixels the same way.
//
// Warp roles: 0-7 two consumer warpgroups (warpgroup g takes the M = 64 blocks g, g + 2, ... of a unit: wgmma into registers, then the
// epilogue from the accumulator fragment) | 8 loader (cp.async.bulk per channel group and plane).  The MMAs and the epilogue of one
// block are xconv_block_issue + wgmma_wait / xconv_block_epilogue, which tcx_first_kernel also runs for layer 3 of AffNet / OriNet.
//
// Ping-pong (template switch PPS, set per launch in nets_tcx.cu; used at 8x8 outputs, BLOCKS = 2: one block per warpgroup and unit,
// where the MMAs are a large share of the time): the two warpgroups issue their blocks' MMAs in strict turns,
// ordered by a pair of named barriers (warpgroup 0 unit k, warpgroup 1 unit k, warpgroup 0 unit k + 1, ...).  A warpgroup's MMAs are
// then queued behind its partner's, and its epilogue runs while the tensor core works through the partner's block; without the order
// both warpgroups issue together, wait together and leave the tensor core idle through both epilogues.  Each warp releases the stage
// as soon as its MMAs on it have completed, before its epilogue, so the loader can refill it during the epilogue.  Both warpgroups
// still share each unit: owning whole units would need a stage per warpgroup plus one to load into, and the 8x8 layers fit only two
// (226 KB of shared memory at HardNet / AffNet layer 6).  The other launches keep the plain schedule (both warpgroups issue at once and
// release the stage after their epilogues), and so does every launch in a build with AG_CONV_PINGPONG = 0 (A/B runs).
#pragma once
#include <cuda_bf16.h>

#include "tc_common.cuh"

#ifndef AG_CONV_PINGPONG
#define AG_CONV_PINGPONG 1
#endif

namespace ag {
namespace tcx {

using namespace ag::tc;

constexpr int XORDER = 5;    // ping-pong: named barrier XORDER + g lets warpgroup g issue its next block's MMAs (3, 4: the warpgroups)

// AG_CONV_TIMELINE (developer builds, scripts/conv_kernel_timeline.py): every warp of the split-0 CTAs 0 .. CT_CTAS - 1 adds up the SM
// cycles (clock64) it spends in each CT_* state and stores the sums per launch in g_conv_tl; warp 0 of each consumer warpgroup of CTA 0
// also logs, per block, when its MMA issue starts, when its MMAs have completed and when its epilogue ends (g_conv_ev), from which the
// script derives how much of the epilogues overlap and how long no MMA was in flight.  ag_conv_timeline_read copies both out.
// States: consumers  TOTAL | wait full | wait for the turn (ping-pong) | issue MMAs | wgmma_wait | epilogue | warpgroup barrier | - | other
//         loader     TOTAL | -         | -                              | -          | -          | -        | -                 | wait empty | other
enum { CT_TOTAL, CT_WAIT_FULL, CT_TURN, CT_ISSUE, CT_MMA_WAIT, CT_EPILOGUE, CT_WG_BAR, CT_WAIT_EMPTY, CT_OTHER, CT_STATES };
#ifdef AG_CONV_TIMELINE
constexpr int CT_CTAS = 4, CT_LAUNCHES = 16, CT_EVENTS = 2048;
__device__ unsigned long long g_conv_tl[CT_LAUNCHES][CT_CTAS][9][CT_STATES];
__device__ unsigned long long g_conv_ev[CT_LAUNCHES][2][CT_EVENTS][3];
__device__ int g_conv_tl_launch[CT_CTAS];
struct ConvTimeline {
    unsigned long long t[CT_STATES];
    long long start, mark;
    int slot, warp, n_ev;   // slot CT_LAUNCHES: not recorded
    // thread 0, before the block-wide barrier: this launch's slot in g_conv_tl, published in shared memory
    __device__ static void claim(int* s_slot) {
        if (threadIdx.x == 0)
            *s_slot = (blockIdx.y == 0 && blockIdx.x < CT_CTAS) ? min(atomicAdd(&g_conv_tl_launch[blockIdx.x], 1), CT_LAUNCHES) : CT_LAUNCHES;
    }
    __device__ void init(const int* s_slot) {
        for (int i = 0; i < CT_STATES; i++) t[i] = 0;
        slot = *s_slot; warp = threadIdx.x >> 5; n_ev = 0;
        start = mark = clock64();
    }
    // the cycles since the previous lap go to `state`
    __device__ void lap(int state) { const long long now = clock64(); t[state] += (unsigned long long)(now - mark); mark = now; }
    // event k of the current block (0 issue start, 1 MMAs done, 2 epilogue end) at the last lap's time
    __device__ void event(int k) {
        if (blockIdx.x == 0 && slot < CT_LAUNCHES && (threadIdx.x & 127) == 0 && n_ev < CT_EVENTS) g_conv_ev[slot][warp >> 2][n_ev][k] = (unsigned long long)mark;
        if (k == 2) n_ev++;
    }
    __device__ void finish() {
        t[CT_TOTAL] = (unsigned long long)(clock64() - start);
        if ((threadIdx.x & 31) == 0 && slot < CT_LAUNCHES)
            for (int i = 0; i < CT_STATES; i++) g_conv_tl[slot][blockIdx.x][warp][i] = t[i];
    }
};
#else
struct ConvTimeline {
    __device__ static void claim(int*) {}
    __device__ void init(const int*) {}
    __device__ void lap(int) {}
    __device__ void event(int) {}
    __device__ void finish() {}
};
#endif

enum XLayout { L_S2_16 = 0, L_S1_16 = 1, L_S2_8P = 2, L_S1_8P = 3, L_HEAD = 4 };

// Cluster multicast (the two CTAs that split a layer's output channels read the SAME input unit): a bulk copy lands at the same
// shared-memory offset of every CTA in the mask and completes bytes on the mbarrier at the same offset of each; a commit arrives on the
// barrier at the same offset of each.
__device__ __forceinline__ void bulk_g2s_mc(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint16_t mask) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask)
                 : "memory");
}
// arrive on the barrier at the same shared-memory offset of CTA `cta` of the cluster.  Release at CTA scope (the default semantics):
// the consumers' arrivals on `empty` only have to follow their own completed wgmma reads of the stage (wgmma_wait), not their global
// stores.  A cluster-scope release compiles to MEMBAR.ALL.GPU before the arrival, which waits for every store the warp still has in
// flight (the previous block's epilogue) and stalled the consumers of the multicast layer for about a fifth of their cycles.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
    asm volatile("{\n .reg .b32 ra;\n mapa.shared::cluster.u32 ra, %0, %1;\n mbarrier.arrive.release.cta.shared::cluster.b64 _, [ra];\n}\n" ::"r"(smem_u32(bar)), "r"(cta)
                 : "memory");
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Operand type of an engine instance: BF = 0 fp16, BF = 1 bf16 (BASELINE.json configs[4]: "bf16 HardNet tensor-core path").
template <int BF>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
    if (BF) { const __nv_bfloat162 h = __floats2bfloat162_rn(a, b); return *reinterpret_cast<const uint32_t*>(&h); }
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
template <int BF>
__device__ __forceinline__ float2 unpack2(uint32_t u) {
    if (BF) return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xFFFF0000u));
    return __half22float2(*reinterpret_cast<const __half2*>(&u));
}
// 8 fp32 values -> 8 16-bit floats (hi) and, when LO, the residuals v - hi rounded to the same format; the residual is taken from the
// packed hi (one F2FP per pair)
template <int LO, int BF = 0>
__device__ __forceinline__ void split_pack8(const float* v, uint4& hi, uint4& lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        h[i] = pack2<BF>(v[2 * i], v[2 * i + 1]);
        if (LO) {
            const float2 f = unpack2<BF>(h[i]);
            l[i] = pack2<BF>(v[2 * i] - f.x, v[2 * i + 1] - f.y);
        } else l[i] = 0;
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// the same for one pair of values (one 32-bit word of each plane)
template <int LO, int BF = 0>
__device__ __forceinline__ void split_pack2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
    hi = pack2<BF>(v0, v1);
    if (LO) {
        const float2 f = unpack2<BF>(hi);
        lo = pack2<BF>(v0 - f.x, v1 - f.y);
    } else lo = 0;
}

// slots per channel group and unit of an HBM activation layout, and patches per unit
__host__ __device__ constexpr int layout_slots(int lay) { return lay == L_S2_16 ? 1024 : lay == L_S1_16 ? 256 : lay == L_S2_8P ? 512 : 128; }
__host__ __device__ constexpr int layout_pair(int lay) { return (lay == L_S2_8P || lay == L_S1_8P) ? 1 : 0; }
// position of pixel x inside a 16-slot row group (neighbour-paired order, see the top of this file): a row of 16 pixels, or of two
// patches' 8 pixels each (p = patch parity)
__host__ __device__ constexpr int rpos(int x) { return (x & 1) * 8 + (x >> 1); }
__host__ __device__ constexpr int ppos(int x, int p) { return (x & 1) * 8 + p * 4 + (x >> 1); }
// slot of pixel (y, x) of patch parity p in a layout
__host__ __device__ constexpr int layout_slot(int lay, int y, int x, int p) {
    return lay == L_S2_16 ? ((y & 1) * 2 + (x & 1)) * 256 + (y >> 1) * 16 + rpos(x >> 1)
         : lay == L_S1_16 ? y * 16 + rpos(x)
         : lay == L_S2_8P ? ((y & 1) * 2 + (x & 1)) * 128 + (y >> 1) * 16 + ppos(x >> 1, p)
                          : y * 16 + ppos(x, p);
}

// Geometry of a layer's input in shared memory.  H: input map edge, STRIDE 1 | 2.
template <int H, int STRIDE>
struct XIn {
    static constexpr int HOUT = H / STRIDE;
    static constexpr int PAIR = (HOUT == 8) ? 1 : 0;              // two patches per tile, interleaved row by row
    static constexpr int W = HOUT;                                // pixels of one patch per image row
    static constexpr int RW = W * (1 + PAIR);                     // slots per (interleaved) row
    static constexpr int TILES = HOUT * RW / 128;                 // 8 | 2 | 1
    static constexpr int NPLANES = (STRIDE == 1) ? 1 : 4;
    static constexpr int DATA = HOUT * RW;                        // data slots per plane
    static constexpr int PLANE = DATA + RW;                       // + one zero row above
    static constexpr int SLOT_STAGE = NPLANES * PLANE;            // stride 1: the zero row BELOW a stage is the next stage's (or the group's trailing) zero row
    static constexpr int LAYOUT = (STRIDE == 2) ? (PAIR ? L_S2_8P : L_S2_16) : (PAIR ? L_S1_8P : L_S1_16);
    static_assert(HOUT == 8 || HOUT == 16 || HOUT == 32, "map sizes of the three nets");
    static_assert(!(STRIDE == 1 && H == 32), "the 32x32 stride-1 layer lives in tcx_first.cuh");
};

struct XArgs {
    const __half* in;     // HBM activation buffer in the layer's input layout
    void* out;            // next layer's buffer
    const __half* wpk;    // packed weights (tcx_pack_layer)
    const float* bias;    // [COUT]
    float inv_scale;      // 1 / (power-of-two scale of wpk)
    int n, group;         // patches, patches per image
    const int* count;     // valid patches per image (NULL: all)
};

// SA: input hi/lo planes; SW: weight hi/lo copies; OSA: write hi/lo planes.  OUT: layout of the output buffer.
template <int CIN, int COUT, int H, int STRIDE, int NSPLIT, int STAGES, int OUT, int SA, int SW, int OSA>
struct XCfg {
    using In = XIn<H, STRIDE>;
    static constexpr int CO = COUT, STRD = STRIDE, OUTL = OUT, SPLIT_A = SA, SPLIT_W = SW, SPLIT_O = OSA;   // for the block functions below
    static constexpr int KC = CIN / 8, NT = COUT / NSPLIT, HOUT = In::HOUT;
    static constexpr int G = KC * (1 + SA);                                   // channel groups of one unit (in shared memory)
    static constexpr int GS = STAGES * In::SLOT_STAGE + (STRIDE == 1 ? In::RW : 0);   // slots per channel group in shared memory
    static constexpr int ACCW = 3 * NT;                                        // accumulator columns of one block
    static constexpr int BLOCKS = 2 * In::TILES;                               // M = 64 blocks of one unit
    static constexpr uint32_t W_BYTES = 9u * CIN * NT * 2u * (1 + SW);         // per split
    static constexpr uint32_t IN_BYTES = (uint32_t)G * GS * 16u;               // all stages
    static constexpr uint32_t HI_IN_BYTES = (uint32_t)KC * In::NPLANES * In::DATA * 16u;
    static constexpr uint32_t UNIT_IN_BYTES = HI_IN_BYTES * (1 + SA);        // one unit in HBM
    static constexpr int THREADS = 288;
    static constexpr size_t SMEM = 1024 + (size_t)W_BYTES + IN_BYTES;
    static constexpr size_t HI_OUT_BYTES = (size_t)(COUT / 8) * layout_slots(OUT) * 16;
    static constexpr size_t UNIT_OUT_BYTES = (OUT == L_HEAD) ? 0 : HI_OUT_BYTES * (1 + OSA);
    // weight rows per K group of one (dy, k step) block
    static constexpr int NR1 = (1 + SW) * 3 * NT;                              // stride 1: [hi: dx0 dx1 dx2][lo: dx0 dx1 dx2]
    static constexpr int NRO = (1 + SW) * 2 * NT, NRE = (1 + SW) * NT;         // stride 2: odd-x plane [hi: dx0 dx2][lo: ...], even-x plane [hi: dx1][lo: dx1]
    static_assert(CIN % 16 == 0 && NT % 16 == 0 && ACCW <= 256, "wgmma shape");
    static_assert(In::W == 8 || In::W == 16, "a warp's 16 accumulator rows hold whole image rows");
    static_assert(SA <= 1 && SW <= 1 && OSA <= 1, "split-precision switches are 0 | 1");
    static_assert(2 * STAGES + 1 <= 60, "barrier area");
    static_assert(SMEM <= 232448, "shared memory budget");
    static_assert(GS < 16384, "leading-byte offset field");
    static_assert(OUT == L_HEAD || layout_pair(OUT) || !In::PAIR, "a pair layer writes pair layouts or the head operand");
};

// Neighbours along x of an accumulator fragment in the neighbour-paired order: a thread holds rows i = lane/4 (h = 0, an even pixel)
// and i + 8 (h = 1, the odd pixel to its right) of its warp's 16 rows.  The even pixel's right neighbour and the odd pixel's left one
// are the thread's own other value; the even pixel's left neighbour is the odd pixel of row i - 1 (lane - 4, its h = 1 value) and the
// odd pixel's right neighbour the even pixel of row i + 1 (lane + 4, its h = 0 value).
// A neighbour outside the image row is garbage that callers must drop by a select, never by multiplying with 0: in the pair layouts it
// is the other patch of the unit, whose input rows are stale workspace when that patch is skipped (beyond a count, or the tail of an
// odd n).  NaN * 0 = NaN, and the ReLU's fmaxf(NaN, 0) = 0 then silently zeroes the valid patch's border pixel.
__device__ __forceinline__ float frag_left_even(float v1, int lane) { return __shfl_sync(0xffffffffu, v1, (lane + 28) & 31); }
__device__ __forceinline__ float frag_right_odd(float v0, int lane) { return __shfl_sync(0xffffffffu, v0, (lane + 4) & 31); }

__device__ __forceinline__ bool xpatch_valid(const XArgs& a, int pi) { return pi < a.n && (a.count == nullptr || (pi % a.group) < a.count[pi / a.group]); }

// The MMAs of one M = 64 block of a layer (Cfg: XCfg) into d[ACCW / 2]: a_t = the block's first slot in shared memory, w_base = the
// layer's packed weights (both in 16-byte units).  The input's channel groups are Cfg::GS slots apart.  Issues and commits them as one
// wgmma group and returns at once: the caller waits (wgmma_wait, wgmma_reg_fence) before it reads d.
template <class Cfg, int BF>
__device__ __forceinline__ void xconv_block_issue(float* d, uint32_t a_t, uint32_t w_base) {
    using In = typename Cfg::In;
    constexpr int KC = Cfg::KC, NT = Cfg::NT, GS = Cfg::GS, RW = In::RW, SA = Cfg::SPLIT_A, SW = Cfg::SPLIT_W;
    constexpr uint32_t LBO_A = ((uint32_t)GS) << 16;      // (bytes >> 4) << 16
    wgmma_fence();
    if (Cfg::STRD == 1) {
#pragma unroll
        for (int dy = 0; dy < 3; dy++) {
#pragma unroll
            for (int j = 0; j < KC / 2; j++) {
                const uint32_t ahi = ((a_t + (uint32_t)(dy * RW + 2 * j * GS)) & 0x3FFFu) | LBO_A;
                const uint32_t alo = ((a_t + (uint32_t)(dy * RW + (KC + 2 * j) * GS)) & 0x3FFFu) | LBO_A;
                const uint32_t blk = w_base + (uint32_t)((dy * (KC / 2) + j) * 2 * Cfg::NR1);
                const uint32_t bhi = (blk & 0x3FFFu) | ((uint32_t)Cfg::NR1 << 16), blo = ((blk + 3 * NT) & 0x3FFFu) | ((uint32_t)Cfg::NR1 << 16);
                Wgmma<3 * NT, BF>::mma(d, desc64(ahi), desc64(bhi), (dy | j) != 0);
                if (SW) Wgmma<3 * NT, BF>::mma(d, desc64(ahi), desc64(blo), 1);
                if (SA) Wgmma<3 * NT, BF>::mma(d, desc64(alo), desc64(bhi), 1);
            }
        }
    } else {
#pragma unroll
        for (int dy = 0; dy < 3; dy++) {
            constexpr int PL = In::PLANE;
            const int py = (dy == 1) ? 0 : 1, ro = (dy == 0) ? 0 : 1;
#pragma unroll
            for (int j = 0; j < KC / 2; j++) {
                const uint32_t blk = w_base + (uint32_t)((dy * (KC / 2) + j) * 2 * (Cfg::NRO + Cfg::NRE));
                const uint32_t bo_hi = (blk & 0x3FFFu) | ((uint32_t)Cfg::NRO << 16), bo_lo = ((blk + 2 * NT) & 0x3FFFu) | ((uint32_t)Cfg::NRO << 16);
                const uint32_t be = blk + 2 * Cfg::NRO;
                const uint32_t be_hi = (be & 0x3FFFu) | ((uint32_t)Cfg::NRE << 16), be_lo = ((be + NT) & 0x3FFFu) | ((uint32_t)Cfg::NRE << 16);
                // odd-x plane (px = 1): taps dx = 0 and dx = 2 -> columns [0, 2 NT)
                const uint32_t ao = a_t + (uint32_t)((py * 2 + 1) * PL + ro * RW);
                const uint32_t ao_hi = ((ao + (uint32_t)(2 * j * GS)) & 0x3FFFu) | LBO_A, ao_lo = ((ao + (uint32_t)((KC + 2 * j) * GS)) & 0x3FFFu) | LBO_A;
                Wgmma<2 * NT, BF>::mma(d, desc64(ao_hi), desc64(bo_hi), (dy | j) != 0);
                if (SW) Wgmma<2 * NT, BF>::mma(d, desc64(ao_hi), desc64(bo_lo), 1);
                if (SA) Wgmma<2 * NT, BF>::mma(d, desc64(ao_lo), desc64(bo_hi), 1);
                // even-x plane (px = 0): tap dx = 1 -> columns [2 NT, 3 NT) = fragment registers from NT on
                const uint32_t ae = a_t + (uint32_t)((py * 2 + 0) * PL + ro * RW);
                const uint32_t ae_hi = ((ae + (uint32_t)(2 * j * GS)) & 0x3FFFu) | LBO_A, ae_lo = ((ae + (uint32_t)((KC + 2 * j) * GS)) & 0x3FFFu) | LBO_A;
                Wgmma<NT, BF>::mma(d + NT, desc64(ae_hi), desc64(be_hi), (dy | j) != 0);
                if (SW) Wgmma<NT, BF>::mma(d + NT, desc64(ae_hi), desc64(be_lo), 1);
                if (SA) Wgmma<NT, BF>::mma(d + NT, desc64(ae_lo), desc64(be_hi), 1);
            }
        }
    }
    wgmma_commit();
}
// Epilogue of one block from the accumulator fragment d (xconv_block_issue, completed) of warp wq of a warpgroup: x shifts, bias, ReLU, fp16 hi [+ lo]
// into a.out in the layout Cfg::OUTL.  Rows r = 64 b + 16 wq + lane/4 + 8 h of unit u, columns 8 j + 2 (lane % 4) + e of each NT block;
// output channels from split * NT on.
template <class Cfg, int BF>
__device__ __forceinline__ void xconv_block_epilogue(const float* d, const XArgs& a, const float* s_bias, int u, int b, int split, int wq, int lane) {
    using In = typename Cfg::In;
    constexpr int NT = Cfg::NT, HOUT = Cfg::HOUT, W = In::W, PAIR = In::PAIR, COUT = Cfg::CO, OUT = Cfg::OUTL, OSA = Cfg::SPLIT_O;
    unsigned char* obase[2];
    bool ok[2];
    size_t lo_off = 0;
    // row group position i = lane/4: pixel x = 2i + h (PAIR: x = 2 (i % 4) + h of patch 2u + i / 4); only the even pixel's left
    // neighbour (x = 0) and the odd pixel's right neighbour (x = W - 1) can fall outside the image row (else: zero padding)
    const int i = lane >> 2, xi = PAIR ? (i & 3) : i;
    const bool has_l0 = xi > 0, has_r1 = xi < W / 2 - 1;
    static_assert(W == 16 || PAIR, "neighbour-paired row groups: 16 pixels, or 8 of each patch of a pair");
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const int y = b * 4 + wq, x = 2 * xi + h, pi = PAIR ? 2 * u + (i >> 2) : u;   // a warp's 16 rows are image row y
        ok[h] = !PAIR || xpatch_valid(a, pi);   // a single-patch unit: the callers only run valid ones
        if (OUT == L_HEAD) {
            obase[h] = reinterpret_cast<unsigned char*>(a.out) + (((size_t)(pi >> 7) * (HOUT * HOUT * COUT / 8) + (size_t)(y * HOUT + x) * (COUT / 8)) * 128 + (pi & 127)) * 16;
            lo_off = (size_t)((a.n + 127) >> 7) * (HOUT * HOUT * COUT / 8) * 128 * 16;
        } else {
            const int ou = layout_pair(OUT) ? (pi >> 1) : pi;
            obase[h] = reinterpret_cast<unsigned char*>(a.out) + (size_t)ou * Cfg::UNIT_OUT_BYTES + (size_t)layout_slot(OUT, y, x, pi & 1) * 16;
            lo_off = (size_t)(COUT / 8) * layout_slots(OUT) * 16;
        }
    }
#pragma unroll
    for (int j = 0; j < NT / 8; j++) {
        const int c = j * 8 + 2 * (lane & 3);
        float v[2][2];
#pragma unroll
        for (int e = 0; e < 2; e++) {
            // stride 1: blocks dx0 | dx1 | dx2;  stride 2: odd dx0 | odd dx2 | even dx1
            const float c00 = d[4 * j + e], c01 = d[4 * j + 2 + e];                                   // block 0, rows h = 0 / 1
            const float c10 = d[4 * (j + NT / 8) + e], c11 = d[4 * (j + NT / 8) + 2 + e];             // block 1
            const float c20 = d[4 * (j + 2 * NT / 8) + e], c21 = d[4 * (j + 2 * NT / 8) + 2 + e];     // block 2
            // left neighbours: even pixel from lane - 4, odd pixel c00 (stride 2: both in the odd-x plane, x - 1)
            const float l0 = frag_left_even(c01, lane);
            // zero padding by selects: the same roundings as adding the neighbour (fmaf(l, 1, t) == l + t), and a NaN of a
            // skipped pair partner stays out of the valid patch.  Every pixel: l + (r + centre)
            float acc0, acc1;
            if (Cfg::STRD == 1) {
                const float r1 = frag_right_odd(c20, lane);     // right neighbours: even pixel c21, odd pixel from lane + 4
                const float t0 = c21 + c10, t1 = has_r1 ? r1 + c11 : c11;
                acc0 = has_l0 ? l0 + t0 : t0;
                acc1 = c00 + t1;
            } else {
                const float t0 = c10 + c20, t1 = c11 + c21;
                acc0 = has_l0 ? l0 + t0 : t0;
                acc1 = c00 + t1;
            }
            v[0][e] = fmaxf(fmaf(acc0, a.inv_scale, s_bias[c + e]), 0.f);
            v[1][e] = fmaxf(fmaf(acc1, a.inv_scale, s_bias[c + e]), 0.f);
        }
        const int ch = split * NT + c;       // output channel of the pair
        const size_t goff = ((OUT == L_HEAD) ? (size_t)(ch / 8) * 128 * 16 : (size_t)(ch / 8) * layout_slots(OUT) * 16) + (ch & 7) * 2;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            if (!ok[h]) continue;
            uint32_t hi, lo;
            split_pack2<OSA, BF>(v[h][0], v[h][1], hi, lo);
            *reinterpret_cast<uint32_t*>(obase[h] + goff) = hi;
            if (OSA) *reinterpret_cast<uint32_t*>(obase[h] + lo_off + goff) = lo;
        }
    }
}

// MC = 1 (NSPLIT = 2 only): the two CTAs of a unit form a thread-block cluster (1 x 2); each loader fetches half of the unit's planes and
// multicasts them to both, so the input crosses the L2 -> SM fabric once instead of twice.
template <int CIN, int COUT, int H, int STRIDE, int NSPLIT, int STAGES, int OUT, int SA, int SW, int OSA, int BF = 0, int MC = 0, int PPS = 0>
__global__ void __launch_bounds__(288, 1) tcx_conv_kernel(const XArgs a) {
    static_assert(MC == 0 || NSPLIT == 2, "multicast pairs the two channel-split CTAs");
    using Cfg = XCfg<CIN, COUT, H, STRIDE, NSPLIT, STAGES, OUT, SA, SW, OSA>;
    using In = typename Cfg::In;
    constexpr int ACCW = Cfg::ACCW, BLOCKS = Cfg::BLOCKS, GS = Cfg::GS, RW = In::RW;
    constexpr int PAIR = In::PAIR;
    constexpr bool PP = AG_CONV_PINGPONG && PPS;   // PPS: this launch runs the ping-pong schedule
    extern __shared__ __align__(1024) unsigned char smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);  // [STAGES]
    uint64_t* empty = full + STAGES;                       // [STAGES]
    uint64_t* wbar = empty + STAGES;
    float* s_bias = reinterpret_cast<float*>(smem + 512);  // [NT]
    unsigned char* sW = smem + 1024;
    unsigned char* sIn = sW + Cfg::W_BYTES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int split = blockIdx.y;
    const int n_units = PAIR ? (a.n + 1) >> 1 : a.n;

    int* s_tl_slot = reinterpret_cast<int*>(smem + 496);    // AG_CONV_TIMELINE: after the barriers (2 STAGES + 1 <= 60 of them)

    if (threadIdx.x < Cfg::NT) s_bias[threadIdx.x] = a.bias[split * Cfg::NT + threadIdx.x];
    if (threadIdx.x == 0) {
        // empty, MC: arrivals of both CTAs, the stage holds planes multicast by both loaders
        //   ping-pong: one arrival per consumer warp, when its last MMAs on the stage have completed
        //   otherwise: one per consumer warpgroup, after its epilogues
        for (int s = 0; s < STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], (PP ? 8 : 2) * (1 + MC)); }
        mbar_init(wbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    ConvTimeline::claim(s_tl_slot);
    // zero rows of every stage: written once, the loader only ever writes data rows
    for (int i = threadIdx.x; i < (int)(Cfg::IN_BYTES / 16); i += blockDim.x) reinterpret_cast<uint4*>(sIn)[i] = make_uint4(0, 0, 0, 0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (MC) cluster_sync();      // the peer's barriers are initialised before anything is multicast into this CTA
    ConvTimeline tl;
    tl.init(s_tl_slot);
    // one consumer warp's arrival(s) on `empty`
    auto release = [&](uint64_t* e) {
        if (MC) { mbar_arrive_cluster(e, 0); mbar_arrive_cluster(e, 1); }
        else mbar_arrive(e);
    };

    auto uvalid = [&](int u) -> bool { return PAIR ? (xpatch_valid(a, 2 * u) || xpatch_valid(a, 2 * u + 1)) : xpatch_valid(a, u); };

    if (warp == 8) {
        // ===== loader =====
        if (lane == 0) {
            mbar_expect_tx(wbar, Cfg::W_BYTES);
            bulk_g2s(sW, reinterpret_cast<const unsigned char*>(a.wpk) + (size_t)split * Cfg::W_BYTES, Cfg::W_BYTES, wbar);
            int it = 0;
            for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
                if (!uvalid(u)) continue;
                const int s = it % STAGES;
                tl.lap(CT_OTHER);
                mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
                tl.lap(CT_WAIT_EMPTY);
                mbar_expect_tx(&full[s], Cfg::UNIT_IN_BYTES);
                const unsigned char* gsrc = reinterpret_cast<const unsigned char*>(a.in) + (size_t)u * Cfg::UNIT_IN_BYTES;
#pragma unroll 1
                for (int g = 0; g < Cfg::G; g++)
#pragma unroll
                    for (int pl = 0; pl < In::NPLANES; pl++) {
                        unsigned char* dst = sIn + ((size_t)g * GS + (size_t)s * In::SLOT_STAGE + (size_t)pl * In::PLANE + RW) * 16;
                        const unsigned char* srcp = gsrc + ((size_t)g * In::NPLANES + pl) * In::DATA * 16;
                        if (MC) { if (((g * In::NPLANES + pl) & 1) == split) bulk_g2s_mc(dst, srcp, In::DATA * 16u, &full[s], (uint16_t)3); }
                        else bulk_g2s(dst, srcp, In::DATA * 16u, &full[s]);
                    }
                it++;
            }
            tl.lap(CT_OTHER);
            if (MC) {   // drain: the peer's last arrivals on this CTA's `empty` barriers must have landed before the CTA may exit
                for (int k = 0; k < STAGES && k < it; k++) { const int j = it - 1 - k; mbar_wait(&empty[j % STAGES], (j / STAGES) & 1); }
            }
            tl.lap(CT_WAIT_EMPTY);
        }
    } else if (warp < 8) {
        // ===== consumers: warpgroup wg takes the M = 64 blocks wg, wg + 2, ... of every unit =====
        const int wg = warp >> 2, wq = warp & 3;
        mbar_wait(wbar, 0);
        const uint32_t w_base = smem_u32(sW) >> 4;           // 16-byte units
        const uint32_t in_base = smem_u32(sIn) >> 4;
        int it = 0;
        for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
            if (!uvalid(u)) continue;
            const int s = it % STAGES;
            tl.lap(CT_OTHER);
            mbar_wait(&full[s], (it / STAGES) & 1);
            tl.lap(CT_WAIT_FULL);
            const uint32_t st_base = in_base + (uint32_t)(s * In::SLOT_STAGE);
#pragma unroll 1
            for (int b = wg; b < BLOCKS; b += 2) {
                float d[ACCW / 2];
                // ping-pong: the turns alternate over the whole run, as both warpgroups take BLOCKS / 2 blocks of every unit.
                // Warpgroup 0's first block is the only one not preceded by a partner block.
                if (PP && (wg == 1 || it > 0 || b > 0)) bar_sync(XORDER + wg, 256);
                tl.lap(CT_TURN);
                tl.event(0);
                xconv_block_issue<Cfg, BF>(d, st_base + (uint32_t)(b * 64), w_base);
                if (PP) asm volatile("bar.arrive %0, 256;" ::"r"(XORDER + (wg ^ 1)) : "memory");   // the partner's turn
                tl.lap(CT_ISSUE);
                wgmma_wait<0>();
                wgmma_reg_fence<ACCW / 2>(d);
                tl.lap(CT_MMA_WAIT);
                tl.event(1);
                // ping-pong: this warp's last MMAs on the stage have completed; the epilogue reads registers only
                if (PP && b + 2 >= BLOCKS && lane == 0) release(&empty[s]);
                xconv_block_epilogue<Cfg, BF>(d, a, s_bias, u, b, split, wq, lane);
                tl.lap(CT_EPILOGUE);
                tl.event(2);
            }
            if (!PP) {
                bar_sync(3 + wg, 128);   // every warp of the warpgroup has finished its MMAs on this stage
                tl.lap(CT_WG_BAR);
                if ((threadIdx.x & 127) == 0) release(&empty[s]);
            }
            it++;
        }
        if (PP && wg == 0 && it > 0) bar_sync(XORDER, 256);   // warpgroup 1's arrival after its last block
        tl.lap(CT_OTHER);
    }
    tl.finish();
    __syncthreads();
    if (MC) cluster_sync();      // neither CTA leaves while the other may still signal its barriers
}

}  // namespace tcx
}  // namespace ag
