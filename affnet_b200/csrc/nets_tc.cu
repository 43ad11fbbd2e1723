// Tensor-core engine of AffNet / OriNet / HardNet (replaces the conv stacks and heads of architectures.py:207-235 / 36-82 and
// HardNet.py:67-101; BatchNorm folded, ReLU fused).  Per net:
//   tc_conv_kernel<first>  sampler + input_norm + conv1 (fp32, CUDA cores) + conv2 (tensor cores); patches and layer-1
//                          activations stay on the SM
//   tc_conv_kernel         conv3 .. conv6 as shifted-window implicit GEMMs (tc_conv.cuh); HardNet's 128-channel layers as two
//                          CTAs per patch, each computing half of the output channels
//   tc_head_kernel / tc_headx_kernel   the 8x8 heads as GEMMs over 128-patch tiles (tc_head.cuh)
// Numerics: fp16 operands with fp16 residual planes where a net needs them, fp32 accumulation (DESIGN.md section 4).
#include <vector>

#include "net_impl.cuh"
#include "tc_conv.cuh"
#include "tc_head.cuh"
#include <stdlib.h>
#include <string.h>

namespace ag {
namespace tc {

static int g_num_sms = 0;
static int num_sms() {
    if (g_num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
        if (g_num_sms <= 0) g_num_sms = 132;
    }
    return g_num_sms;
}

template <int CIN, int COUT, int H, int STRIDE, int NSPLIT, int STAGES, int OUT, int SA = 0, int SW = 0, int OSA = 0, int FIRST = 0>
static int launch_tc(const __half* in, void* out, const __half* w, const float* b, float inv_scale, int n, int group, const int* count, cudaStream_t st,
                     const FirstSrc* src = nullptr) {
    using Cfg = ConvCfg<CIN, COUT, H, STRIDE, NSPLIT, STAGES, OUT, SA, SW, OSA, FIRST>;
    auto kern = tc_conv_kernel<CIN, COUT, H, STRIDE, NSPLIT, STAGES, OUT, SA, SW, OSA, FIRST>;
    static SmemAttrOnce attr_once;
    {
        int rc = attr_once.ensure(kern, Cfg::SMEM, "tc_conv smem attr");
        if (rc != AG_OK) return rc;
    }
    ConvArgs a;
    a.in = in; a.out = out; a.wpk = w; a.bias = b; a.inv_scale = inv_scale; a.n = n; a.group = group; a.count = count;
    int gx = num_sms() / NSPLIT;
    if (gx > n) gx = n;
    if (gx < 1) gx = 1;
    FirstSrc fs;
    if (src) fs = *src; else memset(&fs, 0, sizeof(fs));
    kern<<<dim3(gx, NSPLIT), Cfg::THREADS, Cfg::SMEM, st>>>(a, fs);
    AG_CHECK_LAUNCH(FIRST ? "tc_conv_kernel<first>" : "tc_conv_kernel");
    return AG_OK;
}

}  // namespace tc

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

// bytes per patch of each of the two ping-pong fp16 activation buffers (largest layer output)
size_t tc_act_bytes(int kind) {
    using namespace tc;
    if (kind == AG_NET_HARDNET) return ConvCfg<32, 32, 32, 1, 1, 2, PHASE>::OUT_BYTES;        // 82,944 B (L2 out)
    if (kind == AG_NET_ORINET) return ConvCfg<16, 16, 32, 1, 1, 2, PHASE, 1, 1, 1>::OUT_BYTES;  // hi+lo planes
    return ConvCfg<16, 16, 32, 1, 1, 2, PHASE, 0, 1, 0>::OUT_BYTES;
}

// HardNet: trunk (fp16 operands) + tensor-core head -> L2-normalised descriptors [n,128] in `out`.
// `headbuf` holds the last layer's output in the HEADL layout for ceil(n/128)*128 patches (16 KiB each).
int tc_hardnet_forward(const ag_net* net, const tc::FirstSrc& src0, int n, int group, const int* count, void* bufA, void* bufB, void* headbuf,
                       float* out, cudaStream_t st) {
    using namespace tc;
    __half* A = (__half*)bufA;
    __half* B = (__half*)bufB;
    FirstSrc src = src0;
    src.w1 = net->d_w1; src.b1 = net->d_b[0]; src.w1_inv = net->w_inv_scale[0]; src.w1_scale = 1.0f / net->w_inv_scale[0];
    int rc;
    if ((rc = launch_tc<32, 32, 32, 1, 1, 2, PHASE, 0, 0, 0, 1>(nullptr, B, net->d_wh[1], net->d_b[1], net->w_inv_scale[1], n, group, count, st, &src))) return rc;
    if ((rc = launch_tc<32, 64, 32, 2, 1, 2, PLAIN>(B, A, net->d_wh[2], net->d_b[2], net->w_inv_scale[2], n, group, count, st))) return rc;
    if ((rc = launch_tc<64, 64, 16, 1, 1, 2, PHASE>(A, B, net->d_wh[3], net->d_b[3], net->w_inv_scale[3], n, group, count, st))) return rc;
    if ((rc = launch_tc<64, 128, 16, 2, 2, 2, PLAIN>(B, A, net->d_wh[4], net->d_b[4], net->w_inv_scale[4], n, group, count, st))) return rc;
    if ((rc = launch_tc<128, 128, 8, 1, 2, 2, HEADL>(A, headbuf, net->d_wh[5], net->d_b[5], net->w_inv_scale[5], n, group, count, st))) return rc;
    return tc_hardnet_head(net, headbuf, n, group, count, out, st);
}

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

// AffNet trunk -> features as fp16 hi + lo planes in the head-GEMM layout (tc_head.cuh).  Weights split hi/lo (A error 1.8e-4; plain fp16 weights give 1.8e-3).
int tc_trunk_affnet(const ag_net* net, const tc::FirstSrc& src0, int n, int group, const int* count, void* bufA, void* bufB, void* feat,
                    cudaStream_t st) {
    using namespace tc;
    __half* A = (__half*)bufA;
    __half* B = (__half*)bufB;
    FirstSrc src = src0;
    src.w1 = net->d_w1; src.b1 = net->d_b[0]; src.w1_inv = net->w_inv_scale[0]; src.w1_scale = 1.0f / net->w_inv_scale[0];
    int rc;
    rc = launch_tc<16, 16, 32, 1, 1, 2, PHASE, 0, 1, 0, 1>(nullptr, B, net->d_wh[1], net->d_b[1], net->w_inv_scale[1], n, group, count, st, &src);
    if (rc) return rc;
    if ((rc = launch_tc<16, 32, 32, 2, 1, 4, PLAIN, 0, 1, 0>(B, A, net->d_wh[2], net->d_b[2], net->w_inv_scale[2], n, group, count, st))) return rc;
    if ((rc = launch_tc<32, 32, 16, 1, 1, 6, PHASE, 0, 1, 0>(A, B, net->d_wh[3], net->d_b[3], net->w_inv_scale[3], n, group, count, st))) return rc;
    if ((rc = launch_tc<32, 64, 16, 2, 1, 5, PLAIN, 0, 1, 0>(B, A, net->d_wh[4], net->d_b[4], net->w_inv_scale[4], n, group, count, st))) return rc;
    if ((rc = launch_tc<64, 64, 8, 1, 1, 4, HEADL, 0, 1, 1>(A, feat, net->d_wh[5], net->d_b[5], net->w_inv_scale[5], n, group, count, st))) return rc;
    return AG_OK;
}

// OriNet trunk (and AffNet under the exact engine) -> features as fp16 hi + lo planes in the head-GEMM layout, or fp32 [n,64,8,8].  The angle is ill-conditioned in the features (fp16 activations give 8e-3 rad),
// so both operands are split: three MMAs per K step, fp32-grade result (1.6e-5 rad in emulation).
int tc_trunk_orinet(const ag_net* net, const tc::FirstSrc& src0, int n, int group, const int* count, void* bufA, void* bufB, void* feat,
                    cudaStream_t st) {
    using namespace tc;
    __half* A = (__half*)bufA;
    __half* B = (__half*)bufB;
    FirstSrc src = src0;
    src.w1 = net->d_w1; src.b1 = net->d_b[0]; src.w1_inv = net->w_inv_scale[0]; src.w1_scale = 1.0f / net->w_inv_scale[0];
    int rc;
    rc = launch_tc<16, 16, 32, 1, 1, 2, PHASE, 1, 1, 1, 1>(nullptr, B, net->d_wh[1], net->d_b[1], net->w_inv_scale[1], n, group, count, st, &src);
    if (rc) return rc;
    if ((rc = launch_tc<16, 32, 32, 2, 1, 2, PLAIN, 1, 1, 1>(B, A, net->d_wh[2], net->d_b[2], net->w_inv_scale[2], n, group, count, st))) return rc;
    if ((rc = launch_tc<32, 32, 16, 1, 1, 3, PHASE, 1, 1, 1>(A, B, net->d_wh[3], net->d_b[3], net->w_inv_scale[3], n, group, count, st))) return rc;
    if ((rc = launch_tc<32, 64, 16, 2, 1, 2, PLAIN, 1, 1, 1>(B, A, net->d_wh[4], net->d_b[4], net->w_inv_scale[4], n, group, count, st))) return rc;
    // default engine: hi/lo head-GEMM operand; exact engine: fp32 NCHW features for the fp32 FMA-chain heads of nets_simt.cu
    if (net->engine == AG_ENGINE_TC_EXACT) return launch_tc<64, 64, 8, 1, 1, 2, FINAL, 1, 1, 0>(A, feat, net->d_wh[5], net->d_b[5], net->w_inv_scale[5], n, group, count, st);
    return launch_tc<64, 64, 8, 1, 1, 2, HEADL, 1, 1, 1>(A, feat, net->d_wh[5], net->d_b[5], net->w_inv_scale[5], n, group, count, st);
}

// AffNet / OriNet head on tensor cores over the hi/lo feature planes the trunks above leave in `feat`
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

int tc_nsplit(int kind, int layer) { return (kind == AG_NET_HARDNET && layer >= 4) ? 2 : 1; }
int tc_split_w(int kind) { return kind == AG_NET_HARDNET ? 0 : 1; }

}  // namespace ag
