// Second-generation tensor-core engine of AffNet / OriNet / HardNet (tcx_first.cuh, tcx_conv.cuh): row tiles without x padding, the
// three taps of a kernel row stacked along N, x shifts by warp shuffles in the epilogue.  Replaces the conv stacks of
// architectures.py:207-235 / 36-82 and HardNet.py:67-101 (BatchNorm folded, ReLU fused); the 8x8 heads are the GEMM kernels of
// tc_head.cuh over the trunk's last output.  Per net:  AffNet / OriNet  tcx_first_kernel (sampler + input_norm + conv1 + conv2 + conv3)
// ->  tcx_conv_kernel x3;  HardNet  tcx_first_kernel (sampler + input_norm + conv1 + conv2)  ->  tcx_conv_kernel x4.
// Numerics: AffNet / OriNet with fp16 residual planes of weights and activations in every layer (three MMAs per K step, fp32-grade);
// HardNet fp16 activations, weights with their fp16 residual in layers 2 and 3 (emulation on the 2000 graf patches: plain fp16 weights give a
// descriptor error of 1.1e-3, dominated by the weight rounding of the early layers; with the residuals of layers 2-3 the parity tests hold
// the descriptors to 6e-4; adding layer 4's residual buys about 0.5e-4).
#include <stdlib.h>
#include <string.h>

#include <vector>

#include <cuda_bf16.h>

#include "net_impl.cuh"
#include "tc_head.cuh"
#include "tcx_conv.cuh"
#include "tcx_first.cuh"

namespace ag {
namespace tcx {

static int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

template <int CIN, int COUT, int H, int STRIDE, int NSPLIT, int STAGES, int OUT, int SA, int SW, int OSA, int BF = 0, int MC = 0, int PPS = 0>
static int launch_conv(const void* in, void* out, const __half* w, const float* b, float inv_scale, int n, int group, const int* count, cudaStream_t st) {
    using Cfg = XCfg<CIN, COUT, H, STRIDE, NSPLIT, STAGES, OUT, SA, SW, OSA>;
    auto kern = tcx_conv_kernel<CIN, COUT, H, STRIDE, NSPLIT, STAGES, OUT, SA, SW, OSA, BF, MC, PPS>;
    static SmemAttrOnce attr_once;
    int rc = attr_once.ensure(kern, Cfg::SMEM, "tcx_conv smem attr");
    if (rc != AG_OK) return rc;
    XArgs a;
    a.in = (const __half*)in; a.out = out; a.wpk = w; a.bias = b; a.inv_scale = inv_scale; a.n = n; a.group = group; a.count = count;
    const int units = Cfg::In::PAIR ? (n + 1) / 2 : n;
    int gx = num_sms() / NSPLIT;
    if (gx > units) gx = units;
    if (gx < 1) gx = 1;
    if (MC) {   // the two channel-split CTAs of a unit as one thread-block cluster (1 x 2)
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = dim3(gx, NSPLIT); cfg.blockDim = dim3(Cfg::THREADS); cfg.dynamicSmemBytes = Cfg::SMEM; cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = 2; attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        rc = check_cuda(cudaLaunchKernelEx(&cfg, kern, a), "tcx_conv cluster launch");
        if (rc != AG_OK) return rc;
    } else
        kern<<<dim3(gx, NSPLIT), Cfg::THREADS, Cfg::SMEM, st>>>(a);
    AG_CHECK_LAUNCH("tcx_conv_kernel");
    return AG_OK;
}

// L3 = 1: layer 3 as well, with weights w3 / bias b3, into out3 (out is then unused)
template <int C1, int COUT, int SA, int SW, int OSA, int BF = 0, int L3 = 0>
static int launch_first(void* out, const __half* w, const float* b, float inv_scale, int n, int group, const int* count, cudaStream_t st, const FirstSrc& src,
                        void* out3 = nullptr, const __half* w3 = nullptr, const float* b3 = nullptr, float inv_scale3 = 0.f) {
    using Cfg = XFirstCfg<C1, COUT, SA, SW, OSA, L3>;
    auto kern = tcx_first_kernel<C1, COUT, SA, SW, OSA, BF, L3>;
    static SmemAttrOnce attr_once;
    int rc = attr_once.ensure(kern, Cfg::SMEM, "tcx_first smem attr");
    if (rc != AG_OK) return rc;
    XArgs a;
    a.in = nullptr; a.out = out; a.wpk = w; a.bias = b; a.inv_scale = inv_scale; a.n = n; a.group = group; a.count = count;
    XArgs a3 = a;
    a3.out = out3; a3.wpk = w3; a3.bias = b3; a3.inv_scale = inv_scale3;
    int gx = num_sms();
    if (gx > n) gx = n;
    if (gx < 1) gx = 1;
    kern<<<gx, Cfg::THREADS, Cfg::SMEM, st>>>(a, src, a3);
    AG_CHECK_LAUNCH("tcx_first_kernel");
    return AG_OK;
}

// debug / test helper: an activation buffer in one of the HBM layouts (L_HEAD included) -> fp32 [n][C][H][H] (hi + lo planes added;
// bf: 16-bit bf16 values)
__global__ void tcx_decode_kernel(const __half* __restrict__ buf, int layout, int C, int osa, int H, int n, int bf, float* __restrict__ out) {
    const size_t total = (size_t)n * C * H * H;
    auto val = [&](size_t k) -> float { return bf ? __uint_as_float((uint32_t)__half_as_ushort(buf[k]) << 16) : __half2float(buf[k]); };
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % H), y = (int)((i / H) % H), c = (int)((i / ((size_t)H * H)) % C), pi = (int)(i / ((size_t)H * H * C));
        size_t hi, lo;
        if (layout == L_HEAD) {   // [patch/128][pixel*C/8 + c/8][patch%128][8], the residual plane behind all tiles
            const size_t tile = (size_t)H * H * (C / 8) * 128 * 8;
            hi = (size_t)(pi >> 7) * tile + ((((size_t)(y * H + x) * (C / 8) + c / 8) * 128 + (pi & 127)) * 8 + (c & 7));
            lo = hi + (size_t)((n + 127) >> 7) * tile;
        } else {
            const int slots = layout_slots(layout);
            const size_t unit_halfs = (size_t)(C / 8) * slots * 8 * (osa ? 2 : 1);
            const int unit = layout_pair(layout) ? (pi >> 1) : pi;
            const int slot = layout_slot(layout, y, x, pi & 1);
            hi = (size_t)unit * unit_halfs + ((size_t)(c / 8) * slots + slot) * 8 + (c & 7);
            lo = hi + (size_t)(C / 8) * slots * 8;
        }
        float v = val(hi);
        if (osa) v += val(lo);
        out[i] = v;
    }
}

}  // namespace tcx

tc::FirstSrc tc_src_patches(const float* patches) {
    tc::FirstSrc s;
    memset(&s, 0, sizeof(s));
    s.patches = patches;
    s.cap = 1;
    return s;
}

tc::FirstSrc tc_src_pyramid(const ag_pyramid_plan_t* p, const float* pyr, const float* lafs, const int* oct, const int* lvl, int cap) {
    tc::FirstSrc s;
    memset(&s, 0, sizeof(s));
    s.pyr = pyr; s.lafs = lafs; s.oct = oct; s.lvl = lvl; s.cap = cap;
    s.geom.n_octaves = p->n_octaves; s.geom.n_levels = p->n_levels;
    for (int o = 0; o < AG_MAX_OCTAVES; o++) {
        s.geom.h[o] = p->h[o]; s.geom.w[o] = p->w[o];
        for (int l = 0; l < AG_MAX_LEVELS; l++) s.geom.off[o][l] = p->level_offset[o][l];
    }
    return s;
}

// ---- weight packing (host) --------------------------------------------------------------------------------------------------------
// wf: fp32 [tap = dy*3+dx][ci][co] (BatchNorm folded), scale: power of two.  Blocks per (split, dy, 16 input channels):
//   stride 1: [K group (2)][part hi|lo][dx 0,1,2][co][8]
//   stride 2: odd-x plane [K group][part][dx 0,2][co][8], then even-x plane [K group][part][dx 1][co][8]
static __half bf16_bits_as_half(float v) {   // bf16(v) stored in a 16-bit slot of the (type-agnostic) weight buffer
    const __nv_bfloat16 b = __float2bfloat16_rn(v);
    __half h;
    memcpy(&h, &b, 2);
    return h;
}
static float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

void tcx_pack_layer(const float* wf, int ci, int co, int stride, int nsplit, int sw, float scale, std::vector<__half>& out, int bf16) {
    const int nt = co / nsplit;
    auto put = [&](int dy, int dx, int cin, int c, int part) {
        const float v = scale * wf[((size_t)(dy * 3 + dx) * ci + cin) * co + c];
        if (bf16) {
            const float hi = bf16_round(v);
            out.push_back(bf16_bits_as_half(part == 0 ? hi : v - hi));
        } else {
            const __half hi = __float2half_rn(v);
            out.push_back(part == 0 ? hi : __float2half_rn(v - __half2float(hi)));
        }
    };
    for (int sp = 0; sp < nsplit; sp++)
        for (int dy = 0; dy < 3; dy++)
            for (int j = 0; j < ci / 16; j++) {
                if (stride == 1) {
                    for (int kg = 0; kg < 2; kg++)
                        for (int part = 0; part <= sw; part++)
                            for (int dx = 0; dx < 3; dx++)
                                for (int c = 0; c < nt; c++)
                                    for (int e = 0; e < 8; e++) put(dy, dx, (2 * j + kg) * 8 + e, sp * nt + c, part);
                } else {
                    for (int kg = 0; kg < 2; kg++)
                        for (int part = 0; part <= sw; part++)
                            for (int dx = 0; dx < 3; dx += 2)
                                for (int c = 0; c < nt; c++)
                                    for (int e = 0; e < 8; e++) put(dy, dx, (2 * j + kg) * 8 + e, sp * nt + c, part);
                    for (int kg = 0; kg < 2; kg++)
                        for (int part = 0; part <= sw; part++)
                            for (int c = 0; c < nt; c++)
                                for (int e = 0; e < 8; e++) put(dy, 1, (2 * j + kg) * 8 + e, sp * nt + c, part);
                }
            }
}

int tcx_nsplit(int kind, int layer) { return (kind == AG_NET_HARDNET && layer >= 4) ? 2 : 1; }
// weight residual copies: AffNet / OriNet every layer; HardNet layers 2-3 (layer index 1..2; see the A/B switches)
#ifndef AG_HARD_SW2
#define AG_HARD_SW2 1
#endif
#ifndef AG_HARD_SW3
#define AG_HARD_SW3 1   // HardNet layer 3 / layer 4 weight residuals (A/B switches for the accuracy / time trade, see DESIGN.md)
#endif
#ifndef AG_HARD_SW4
#define AG_HARD_SW4 0   // worst descriptor error over the parity configurations about 4.9e-4 without it, 4.4e-4 with it
#endif
int tcx_split_w(int kind, int layer) { return kind == AG_NET_HARDNET ? (layer == 1 ? AG_HARD_SW2 : layer == 2 ? AG_HARD_SW3 : layer == 3 ? AG_HARD_SW4 : 0) : 1; }
int tcx_stride(int layer) { return (layer == 2 || layer == 4) ? 2 : 1; }

// bytes of each of the two ping-pong activation buffers for n patches (largest layer output: 64 KiB per patch; pair layouts round n up)
size_t tcx_act_bytes(int n) { return (size_t)(n + 1) * 65536; }

// ---- trunks -------------------------------------------------------------------------------------------------------------------------
// AffNet / OriNet (same shapes, own weights): features as fp16 hi + lo planes in the head-GEMM layout.  upto: stop after conv layer
// `upto` (2..6; for the debug decode), 6 = whole trunk.
// cluster-multicast input of HardNet's channel-split layers (the two CTAs of a patch read its input once from L2)
#ifndef AG_HARD_MC5
#define AG_HARD_MC5 1
#endif
#ifndef AG_HARD_MC6
#define AG_HARD_MC6 0
#endif
// tcx_conv_kernel's last template argument selects the ping-pong schedule (tcx_conv.cuh) for the layers it makes faster: AffNet / OriNet
// layer 6 and HardNet layers 5 and 6 (H100, DESIGN.md section 4).  The 16x16-output layers and AffNet / OriNet layer 5 are close to their
// HBM floor and were no faster with it (AffNet layer 5 3-5 % slower).
// Layers 1-3 run in one kernel (layer 2's 32x32 output stays in shared memory).  upto = 2 runs the layers 1-2 kernel instead, which
// writes layer 2's output to bufB for the debug decode.
int tcx_trunk_affori(const ag_net* net, const tc::FirstSrc& src0, int n, int group, const int* count, void* bufA, void* bufB, void* feat,
                     cudaStream_t st, int upto) {
    using namespace tcx;
    tc::FirstSrc src = src0;
    src.w1 = net->d_w1; src.b1 = net->d_b[0]; src.w1_inv = net->w_inv_scale[0]; src.w1_scale = 1.0f / net->w_inv_scale[0];
    int rc;
    if (upto <= 2) return launch_first<16, 16, 1, 1, 1>(bufB, net->d_wx[1], net->d_b[1], net->w_inv_scale[1], n, group, count, st, src);
    if ((rc = launch_first<16, 16, 1, 1, 1, 0, 1>(nullptr, net->d_wx[1], net->d_b[1], net->w_inv_scale[1], n, group, count, st, src,
                                                   bufA, net->d_wx[2], net->d_b[2], net->w_inv_scale[2]))) return rc;
    if (upto <= 3) return AG_OK;
    if ((rc = launch_conv<32, 32, 16, 1, 1, 4, L_S2_8P, 1, 1, 1>(bufA, bufB, net->d_wx[3], net->d_b[3], net->w_inv_scale[3], n, group, count, st))) return rc;
    if (upto <= 4) return AG_OK;
    if ((rc = launch_conv<32, 64, 16, 2, 1, 2, L_S1_8P, 1, 1, 1>(bufB, bufA, net->d_wx[4], net->d_b[4], net->w_inv_scale[4], n, group, count, st))) return rc;
    if (upto <= 5) return AG_OK;
    return launch_conv<64, 64, 8, 1, 1, 2, L_HEAD, 1, 1, 1, 0, 0, 1>(bufA, feat, net->d_wx[5], net->d_b[5], net->w_inv_scale[5], n, group, count, st);
}

template <int BF>
static int trunk_hardnet_t(const ag_net* net, const tc::FirstSrc& src0, int n, int group, const int* count, void* bufA, void* bufB, void* headbuf,
                           cudaStream_t st, int upto) {
    using namespace tcx;
    tc::FirstSrc src = src0;
    src.w1 = net->d_w1; src.b1 = net->d_b[0]; src.w1_inv = net->w_inv_scale[0]; src.w1_scale = 1.0f / net->w_inv_scale[0];
    __half* const* wx = BF ? net->d_wx_bf : net->d_wx;
    int rc;
    if ((rc = launch_first<32, 32, 0, AG_HARD_SW2, 0, BF>(bufB, wx[1], net->d_b[1], net->w_inv_scale[1], n, group, count, st, src))) return rc;
    if (upto <= 2) return AG_OK;
    if ((rc = launch_conv<32, 64, 32, 2, 1, 2, L_S1_16, 0, AG_HARD_SW3, 0, BF>(bufB, bufA, wx[2], net->d_b[2], net->w_inv_scale[2], n, group, count, st))) return rc;
    if (upto <= 3) return AG_OK;
    if ((rc = launch_conv<64, 64, 16, 1, 1, 2, L_S2_8P, 0, AG_HARD_SW4, 0, BF>(bufA, bufB, wx[3], net->d_b[3], net->w_inv_scale[3], n, group, count, st))) return rc;
    if (upto <= 4) return AG_OK;
    if ((rc = launch_conv<64, 128, 16, 2, 2, 2, L_S1_8P, 0, 0, 0, BF, AG_HARD_MC5, 1>(bufB, bufA, wx[4], net->d_b[4], net->w_inv_scale[4], n, group, count, st))) return rc;
    if (upto <= 5) return AG_OK;
    return launch_conv<128, 128, 8, 1, 2, 2, L_HEAD, 0, 0, 0, BF, AG_HARD_MC6, 1>(bufA, headbuf, wx[5], net->d_b[5], net->w_inv_scale[5], n, group, count, st);
}

int tcx_trunk_hardnet(const ag_net* net, const tc::FirstSrc& src0, int n, int group, const int* count, void* bufA, void* bufB, void* headbuf,
                      cudaStream_t st, int upto, int bf16) {
    return bf16 ? trunk_hardnet_t<1>(net, src0, n, group, count, bufA, bufB, headbuf, st, upto)
                : trunk_hardnet_t<0>(net, src0, n, group, count, bufA, bufB, headbuf, st, upto);
}

// ---- heads ---------------------------------------------------------------------------------------------------------------------------
// HardNet 8x8 head GEMM + BatchNorm + L2 norm over the head operand a trunk left in `headbuf`
int tc_hardnet_head(const ag_net* net, const void* headbuf, int n, int group, const int* count, float* out, cudaStream_t st, int bf16) {
    using namespace tc;
    static SmemAttrOnce once0, once1;
    {
        int rc = once0.ensure(tc_head_kernel<0>, HEAD_SMEM, "tc_head smem attr");
        if (rc == AG_OK) rc = once1.ensure(tc_head_kernel<1>, HEAD_SMEM, "tc_head smem attr");
        if (rc != AG_OK) return rc;
    }
    if (bf16) tc_head_kernel<1><<<(n + 127) / 128, 288, HEAD_SMEM, st>>>((const __half*)headbuf, net->d_headh_bf, net->d_head_b, out, n, group, count);
    else tc_head_kernel<0><<<(n + 127) / 128, 288, HEAD_SMEM, st>>>((const __half*)headbuf, net->d_headh, net->d_head_bx, out, n, group, count);
    AG_CHECK_LAUNCH("tc_head_kernel");
    return AG_OK;
}

// AffNet / OriNet head on tensor cores over the hi/lo feature planes tcx_trunk_affori leaves in `feat`
int tc_headx_forward(const ag_net* net, const void* feat, int n, int group, const int* count, float* out, float* angle, cudaStream_t st, float* raw) {
    using namespace tc;
    static SmemAttrOnce once0, once1;
    {
        int rc = once0.ensure(tc_headx_kernel<0>, HX_SMEM, "tc_headx smem attr");
        if (rc == AG_OK) rc = once1.ensure(tc_headx_kernel<1>, HX_SMEM, "tc_headx smem attr");
        if (rc != AG_OK) return rc;
    }
    const int tiles = (n + 127) / 128;
    if (net->kind == AG_NET_AFFNET) tc_headx_kernel<0><<<tiles, 288, HX_SMEM, st>>>((const __half*)feat, net->d_headh, net->d_head_b, net->head_inv_scale, out, nullptr, raw, n, group, count);
    else tc_headx_kernel<1><<<tiles, 288, HX_SMEM, st>>>((const __half*)feat, net->d_headh, net->d_head_b, net->head_inv_scale, out, angle, raw, n, group, count);
    AG_CHECK_LAUNCH("tc_headx_kernel");
    return AG_OK;
}

// bytes of the head-GEMM operand of n patches (hi + lo planes, padded to whole 128-patch tiles)
size_t tc_headx_bytes(int n) { return (size_t)((n + 127) / 128) * 2 * tc::HX_PLANE_TILE; }

}  // namespace ag

using namespace ag;

extern "C" {

// Developer diagnostic (tests/test_gpu_tcx.py, tests/test_gpu_net_bounds.py, tests/test_gpu_simt_exact.py): run the trunk of `net` with
// the handle's engine on materialised patches [n,32,32] up to conv layer `upto` and return that layer's output as fp32 [n][C][H][H].
// ENGINE_SIMT: the fp32 trunk (upto 1..6), its output copied as it is.  Otherwise the second-generation trunk (ENGINE_TC2_BF16: the bf16
// HardNet trunk; any other engine: the fp16 one; upto 2..6), that layer's output decoded from its fp16 / bf16 hi [+ lo] planes in its HBM
// layout (layer 6: the head operand).  d_ws: ag_net_workspace_bytes().
int ag_debug_tcx_layer(const ag_net_t* net, const float* d_patches, int n, int upto, float* d_out, void* d_ws, size_t ws_bytes, void* stream) {
    AG_REQUIRE(net && d_patches && d_out && d_ws, "NULL argument");
    const bool simt = net->engine == AG_ENGINE_SIMT;
    AG_REQUIRE(upto >= (simt ? 1 : 2) && upto <= 6 && n >= 1, "layer out of range");
    if (simt) return simt_trunk_layer(net, d_patches, n, upto, d_out, d_ws, ws_bytes, (cudaStream_t)stream);
    const size_t act = align_up(tcx_act_bytes(n), 256);
    AG_REQUIRE(ws_bytes >= ag_net_workspace_bytes(net->kind, n), "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    char* base = (char*)d_ws;
    const tc::FirstSrc src = tc_src_patches(d_patches);
    const bool hard = net->kind == AG_NET_HARDNET;
    const int bf = hard && net->engine == AG_ENGINE_TC2_BF16;
    int rc = hard ? tcx_trunk_hardnet(net, src, n, n, nullptr, base, base + act, base + 2 * act, st, upto, bf)
                  : tcx_trunk_affori(net, src, n, n, nullptr, base, base + act, base + 2 * act, st, upto);
    if (rc) return rc;
    // layer l writes: 2 -> bufB (L_S2_16, 32x32), 3 -> bufA (L_S1_16, 16x16), 4 -> bufB (L_S2_8P, 16x16), 5 -> bufA (L_S1_8P, 8x8),
    // 6 -> the head operand behind both buffers (L_HEAD, 8x8)
    const int lay = upto == 2 ? tcx::L_S2_16 : upto == 3 ? tcx::L_S1_16 : upto == 4 ? tcx::L_S2_8P : upto == 5 ? tcx::L_S1_8P : tcx::L_HEAD;
    const int H = upto == 2 ? 32 : (upto <= 4 ? 16 : 8);
    const int Cb = hard ? 32 : 16;
    const int C = upto == 2 ? Cb : (upto <= 4 ? 2 * Cb : 4 * Cb);
    const void* buf = upto == 6 ? base + 2 * act : (upto == 2 || upto == 4) ? base + act : base;
    const int osa = hard ? 0 : 1;
    tcx::tcx_decode_kernel<<<296, 256, 0, st>>>((const __half*)buf, lay, C, osa, H, n, bf, d_out);
    AG_CHECK_LAUNCH("tcx_decode_kernel");
    return AG_OK;
}

#ifdef AG_FIRST_TIMELINE
// Developer builds with -DAG_FIRST_TIMELINE only (scripts/first_kernel_timeline.py): copy the per-warp state cycle sums of
// tcx_first_kernel, uint64 [TL_LAUNCHES][TL_CTAS][16 warps][TL_STATES] in launch order since the last reset, to `host`; reset != 0
// then clears them.  dims (may be NULL) receives TL_LAUNCHES, TL_CTAS, TL_STATES.
int ag_first_timeline_read(unsigned long long* host, int* dims, int reset) {
    constexpr size_t n = (size_t)tcx::TL_LAUNCHES * tcx::TL_CTAS * 16 * tcx::TL_STATES;
    if (dims) { dims[0] = tcx::TL_LAUNCHES; dims[1] = tcx::TL_CTAS; dims[2] = tcx::TL_STATES; }
    cudaDeviceSynchronize();
    if (host) {
        const int rc = check_cuda(cudaMemcpyFromSymbol(host, tcx::g_first_tl, n * 8), "timeline read");
        if (rc != AG_OK) return rc;
    }
    if (reset) {
        static unsigned long long zeros[n];
        static int zl[tcx::TL_CTAS];
        int rc = check_cuda(cudaMemcpyToSymbol(tcx::g_first_tl, zeros, sizeof(zeros)), "timeline reset");
        if (rc == AG_OK) rc = check_cuda(cudaMemcpyToSymbol(tcx::g_first_tl_launch, zl, sizeof(zl)), "timeline reset");
        return rc;
    }
    return AG_OK;
}
#endif

#ifdef AG_CONV_TIMELINE
// Developer builds with -DAG_CONV_TIMELINE only (scripts/conv_kernel_timeline.py): copy the per-warp state cycle sums of
// tcx_conv_kernel, uint64 [CT_LAUNCHES][CT_CTAS][9 warps][CT_STATES], and CTA 0's block events, uint64 [CT_LAUNCHES][2 warpgroups]
// [CT_EVENTS][issue start | MMAs done | epilogue end] (0: no such block), in launch order since the last reset, to `sums` / `events`
// (either may be NULL); reset != 0 then clears them.  dims (may be NULL) receives CT_LAUNCHES, CT_CTAS, CT_STATES, CT_EVENTS.
int ag_conv_timeline_read(unsigned long long* sums, unsigned long long* events, int* dims, int reset) {
    using namespace tcx;
    if (dims) { dims[0] = CT_LAUNCHES; dims[1] = CT_CTAS; dims[2] = CT_STATES; dims[3] = CT_EVENTS; }
    int rc = check_cuda(cudaDeviceSynchronize(), "timeline read");
    if (rc == AG_OK && sums) rc = check_cuda(cudaMemcpyFromSymbol(sums, g_conv_tl, sizeof(g_conv_tl)), "timeline read");
    if (rc == AG_OK && events) rc = check_cuda(cudaMemcpyFromSymbol(events, g_conv_ev, sizeof(g_conv_ev)), "timeline read");
    if (rc == AG_OK && reset) {
        void* p = nullptr;
        const int zl[CT_CTAS] = {};
        if (rc == AG_OK) rc = check_cuda(cudaGetSymbolAddress(&p, g_conv_tl), "timeline reset");
        if (rc == AG_OK) rc = check_cuda(cudaMemset(p, 0, sizeof(g_conv_tl)), "timeline reset");
        if (rc == AG_OK) rc = check_cuda(cudaGetSymbolAddress(&p, g_conv_ev), "timeline reset");
        if (rc == AG_OK) rc = check_cuda(cudaMemset(p, 0, sizeof(g_conv_ev)), "timeline reset");
        if (rc == AG_OK) rc = check_cuda(cudaMemcpyToSymbol(g_conv_tl_launch, zl, sizeof(zl)), "timeline reset");
        if (rc == AG_OK) rc = check_cuda(cudaDeviceSynchronize(), "timeline reset");
    }
    return rc;
}
#endif

}  // extern "C"
