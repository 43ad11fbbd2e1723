// Hand-crafted orientation and affine shape (SURVEY.md §8(f) rows 1 and 2): the estimators the reference uses when no OriNet /
// AffNet is given.  Replaces OrientationDetector.forward (HandCraftedModules.py:168-192) and AffineShapeEstimator.forward
// (HandCraftedModules.py:94-132).  One warp per patch; the patch (PS x PS, PS <= 41) is staged in shared memory, either loaded from
// materialised patches (ag_orientation_hist / ag_baumberg_shape) or sampled from the pyramid (orientation_hist_pyr / baumberg_pyr, the
// batched pipeline).  Both kinds of kernel call the same per-warp estimator bodies.
#include <math.h>

#include "common.cuh"

namespace ag {

constexpr int HC_MAXPS = 41, HC_WARPS = 2;

__device__ __forceinline__ float warp_sum_f(float v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// OrientationDetector.forward on the PS x PS patch `p` (shared memory) of one warp; s_w [PS*PS], s_b [PS*PS], s_h [40] are the warp's
// scratch.  Returns the angle on every lane.  A non-finite weight (a NaN or infinite pixel, or gx^2 + gy^2 overflowing) gives bin 0, the
// angle pi: the reference multiplies it by the 0 of every other bin's mask, so every smoothed bin is NaN and torch's max returns index 0.
__device__ __forceinline__ float orientation_hist_warp(const float* p, int PS, const float* gk, float* s_w, unsigned char* s_b, float* s_h,
                                                       int lane) {
    const int NP = PS * PS;
    const float PI_F = 3.14159265358979323846f;
    bool nonfinite = false;
    for (int i = lane; i < NP; i += 32) {
        float gx, gy;
        grad_at(p, PS, i / PS, i % PS, 0.5f, -0.5f, gx, gy);   // weights (0.5, 0, -0.5): 0.5*x[j-1] - 0.5*x[j+1]
        const float mag = __fmul_rn(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), 1e-10f)), gk[i]);
        const float ori = atan2f(gy, gx);
        const float o_big = __fdiv_rn(__fmul_rn(36.0f, __fadd_rn(ori, PI_F)), 2.0f * PI_F);
        float bo0 = floorf(o_big);
        const float wo1 = __fsub_rn(o_big, bo0);
        bo0 = fmodf(bo0, 36.0f);
        s_b[i] = (unsigned char)(int)bo0;
        const float w = __fmul_rn(__fsub_rn(1.0f, wo1), mag);   // only the lower-bin weight is accumulated (as the reference does)
        s_w[i] = w;
        nonfinite |= !isfinite(w);
    }
    nonfinite = __any_sync(0xffffffffu, nonfinite);
    __syncwarp();
    // deterministic histogram: lane b sums bin b (and b+32) over all pixels in raster order
    for (int b = lane; b < 36; b += 32) {
        float acc = 0.f;
        for (int i = 0; i < NP; i++)
            if (s_b[i] == b) acc += s_w[i];
        s_h[b + 1] = acc / (float)NP;   // adaptive_avg_pool2d -> mean
    }
    if (lane == 0) { s_h[0] = 0.f; s_h[37] = 0.f; }   // conv1d zero padding
    __syncwarp();
    float best = -INFINITY;
    int bidx = 0;
    for (int b = lane; b < 36; b += 32) {
        const float v = fmaf(0.33f, s_h[b + 2], fmaf(0.34f, s_h[b + 1], 0.33f * s_h[b]));
        if (v > best) { best = v; bidx = b; }
    }
    // first maximum wins (torch.max on CPU)
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
        if (ov > best || (ov == best && oi < bidx)) { best = ov; bidx = oi; }
    }
    if (nonfinite) bidx = 0;
    return -__fsub_rn(__fdiv_rn(__fmul_rn(2.0f * PI_F, (float)bidx), 36.0f), PI_F);
}

// AffineShapeEstimator.forward on the PS x PS patch `p` (shared memory) of one warp -> up-is-up rectified A, on every lane.
// Every fp32 operation is rounded on its own, in the left-to-right order of the reference's torch expressions (no fused multiply-adds),
// so the result is a function of the patch alone: tests/handcrafted_restated.py states the same arithmetic.  The moments are summed
// per lane over i = lane, lane + 32, ... and then by the xor butterfly of warp_sum_f.  A flat patch, a ramp along one axis or a
// non-finite pixel gives NaN in all four entries, as in the reference (A[0,1] is 0 * det there).
__device__ __forceinline__ void baumberg_warp(const float* p, int PS, const float* gk, int lane, float (&A)[4]) {
    const int NP = PS * PS;
    float a = 0.f, b = 0.f, c = 0.f;
    for (int i = lane; i < NP; i += 32) {
        float gx, gy;
        grad_at(p, PS, i / PS, i % PS, -1.0f, 1.0f, gx, gy);   // weights (-1, 0, 1)
        const float g = gk[i];
        a = __fadd_rn(a, __fmul_rn(__fmul_rn(gx, gx), g));
        b = __fadd_rn(b, __fmul_rn(__fmul_rn(gx, gy), g));
        c = __fadd_rn(c, __fmul_rn(__fmul_rn(gy, gy), g));
    }
    a = __fdiv_rn(warp_sum_f(a), (float)NP); b = __fdiv_rn(warp_sum_f(b), (float)NP); c = __fdiv_rn(warp_sum_f(c), (float)NP);
    // invSqrt (HandCraftedModules.py:94-117)
    const float eps = 1e-12f;
    const float mask = (b != 0.f) ? 1.f : 0.f;
    const float r1 = __fdiv_rn(__fmul_rn(mask, __fsub_rn(c, a)), __fadd_rn(__fmul_rn(2.f, b), eps));
    const float sgn = (r1 > 0.f) ? 1.f : ((r1 < 0.f) ? -1.f : 0.f);   // torch.sign: 0 for +-0 and NaN
    const float t1 = __fdiv_rn(sgn, __fadd_rn(fabsf(r1), __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(r1, r1)))));
    float r = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(t1, t1))));
    float t = __fmul_rn(t1, r);
    r = __fadd_rn(__fmul_rn(r, mask), __fsub_rn(1.f, mask));   // r * mask + 1.0 * (1.0 - mask); 1.0 * y == y
    t = __fmul_rn(t, mask);
    const float rr = __fmul_rn(r, r), tt = __fmul_rn(t, t), rt2 = __fmul_rn(__fmul_rn(2.f, r), t);
    float x = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fsub_rn(__fmul_rn(rr, a), __fmul_rn(rt2, b)), __fmul_rn(tt, c))));
    float z = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(tt, a), __fmul_rn(rt2, b)), __fmul_rn(rr, c))));
    const float d = __fsqrt_rn(__fmul_rn(x, z));
    x = __fdiv_rn(x, d); z = __fdiv_rn(z, d);
    const float na = __fadd_rn(__fmul_rn(rr, x), __fmul_rn(tt, z));
    const float nb = __fadd_rn(__fmul_rn(__fmul_rn(-r, t), x), __fmul_rn(__fmul_rn(t, r), z));
    const float nc = __fadd_rn(__fmul_rn(tt, x), __fmul_rn(rr, z));
    // abc2A + rectifyAffineTransformationUpIsUp (LAF.py:285-291)
    const float a00 = na, a01 = nb, a10 = nb, a11 = nc;
    const float det = __fsqrt_rn(fabsf(__fadd_rn(__fsub_rn(__fmul_rn(a00, a11), __fmul_rn(a10, a01)), 1e-10f)));
    const float b2a2 = __fsqrt_rn(__fadd_rn(__fmul_rn(a01, a01), __fmul_rn(a00, a00)));
    A[0] = __fdiv_rn(b2a2, det); A[1] = __fmul_rn(0.f, det);
    A[2] = __fdiv_rn(__fadd_rn(__fmul_rn(a11, a01), __fmul_rn(a10, a00)), __fmul_rn(b2a2, det)); A[3] = __fdiv_rn(det, b2a2);
}

__global__ void __launch_bounds__(HC_WARPS * 32) orientation_hist_kernel(const float* __restrict__ patches, int n, int PS, const float* __restrict__ gk,
                                                                        float* __restrict__ angle) {
    __shared__ float s_p[HC_WARPS][HC_MAXPS * HC_MAXPS];
    __shared__ float s_w[HC_WARPS][HC_MAXPS * HC_MAXPS];
    __shared__ unsigned char s_b[HC_WARPS][HC_MAXPS * HC_MAXPS];
    __shared__ float s_h[HC_WARPS][40];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pi = blockIdx.x * HC_WARPS + warp;
    if (pi >= n) return;
    const int NP = PS * PS;
    float* p = s_p[warp];
    for (int i = lane; i < NP; i += 32) p[i] = patches[(size_t)pi * NP + i];
    __syncwarp();
    const float ang = orientation_hist_warp(p, PS, gk, s_w[warp], s_b[warp], s_h[warp], lane);
    if (lane == 0) angle[pi] = ang;
}

__global__ void __launch_bounds__(HC_WARPS * 32) baumberg_kernel(const float* __restrict__ patches, int n, int PS, const float* __restrict__ gk,
                                                                float* __restrict__ A) {
    __shared__ float s_p[HC_WARPS][HC_MAXPS * HC_MAXPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pi = blockIdx.x * HC_WARPS + warp;
    if (pi >= n) return;
    const int NP = PS * PS;
    float* p = s_p[warp];
    for (int i = lane; i < NP; i += 32) p[i] = patches[(size_t)pi * NP + i];
    __syncwarp();
    float a[4];
    baumberg_warp(p, PS, gk, lane, a);
    if (lane != 0) return;
    float* o = A + (size_t)pi * 4;
    o[0] = a[0]; o[1] = a[1]; o[2] = a[2]; o[3] = a[3];
}

// ---- the estimators sampling the pyramid directly (batched pipeline) ----------------------------------------------------------------
// One warp per keypoint (b, i), i < count[b]; the PS x PS patch is sampled from pyr[oct][lvl] into shared memory with the arithmetic of
// extract_patches_pyr_kernel (laf_sample_xy + bilinear_zero), so the estimators see the bits ag_extract_patches_pyr would write to HBM.
constexpr int HC_PYR_WARPS = 4;

struct HcPyrParams {
    PyrGeom G;
    const float* pyr;
    const float* lafs;   // [B,cap,2,3] normalised
    const int* oct;
    const int* lvl;
    const int* count;    // [B]
    int cap, PS, iters;
    float* out;          // [B,cap,2,2]
    float gk[HC_MAXPS * HC_MAXPS];
};

// floats of shared memory per warp: patch + weights + histogram (40) + bin bytes (orientation) or the patch alone (Baumberg)
__host__ __device__ inline int hc_ori_warp_floats(int PS) { return 2 * PS * PS + 40 + (PS * PS + 3) / 4; }
__host__ __device__ inline int hc_baum_warp_floats(int PS) { return PS * PS; }

// the row of warp `warp` in this block, or -1 when it is at or beyond the image's count (a count of -1 = overflow: nothing to do)
__device__ __forceinline__ long long hc_pyr_row(const HcPyrParams& P, int warp) {
    const int b = blockIdx.y, i = blockIdx.x * HC_PYR_WARPS + warp;
    if (i >= P.cap || i >= P.count[b]) return -1;
    return (long long)b * P.cap + i;
}

__device__ __forceinline__ void sample_patch_warp(const HcPyrParams& P, long long row, const float* L, float* p, int lane) {
    const int o = clampi(P.oct[row], 0, P.G.n_octaves - 1), l = clampi(P.lvl[row], 0, P.G.n_levels - 1);
    const int h = P.G.h[o], w = P.G.w[o];
    const float* img = P.pyr + P.G.off[o][l] + (size_t)blockIdx.y * h * w;
    const int PS = P.PS, NP = PS * PS;
    for (int t = lane; t < NP; t += 32) {
        const int i = t / PS, j = t - i * PS;
        float px, py;
        laf_sample_xy(L, h, w, i, j, 1.0f / (float)PS, px, py);
        p[t] = bilinear_zero(img, h, w, px, py);
    }
    __syncwarp();
}

__global__ void __launch_bounds__(HC_PYR_WARPS * 32) orientation_hist_pyr_kernel(const __grid_constant__ HcPyrParams P) {
    extern __shared__ float hc_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = hc_pyr_row(P, warp);
    if (row < 0) return;
    const int NP = P.PS * P.PS;
    float* p = hc_smem + (size_t)warp * hc_ori_warp_floats(P.PS);
    float* s_w = p + NP;
    float* s_h = s_w + NP;
    unsigned char* s_b = (unsigned char*)(s_h + 40);
    sample_patch_warp(P, row, P.lafs + row * 6, p, lane);
    const float ang = orientation_hist_warp(p, P.PS, P.gk, s_w, s_b, s_h, lane);
    if (lane == 0) {   // angles2A (LAF.py:306-311)
        const float c = cosf(ang), s = sinf(ang);
        float* o = P.out + row * 4;
        o[0] = c; o[1] = s; o[2] = -s; o[3] = c;
    }
}

// getAffineShape's loop (SparseImgRepresenter.py:127-141) with AffineShapeEstimator, all iterations in one launch: sample at the working
// LAF, Baumberg step A, base_A <- A base_A (the first iteration takes A as is), working LAF <- [base_A LAF_A | t] if another follows.
__global__ void __launch_bounds__(HC_PYR_WARPS * 32) baumberg_pyr_kernel(const __grid_constant__ HcPyrParams P) {
    extern __shared__ float hc_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row = hc_pyr_row(P, warp);
    if (row < 0) return;
    float* p = hc_smem + (size_t)warp * hc_baum_warp_floats(P.PS);
    float L0[6], cur[6], base[4];
#pragma unroll
    for (int q = 0; q < 6; q++) L0[q] = cur[q] = P.lafs[row * 6 + q];
    for (int it = 0; it < P.iters; it++) {
        sample_patch_warp(P, row, cur, p, lane);
        float A[4];
        baumberg_warp(p, P.PS, P.gk, lane, A);
        if (it == 0) {
#pragma unroll
            for (int q = 0; q < 4; q++) base[q] = A[q];
        } else {
            float nb[4];
            mat2_mul(A, base, nb);
#pragma unroll
            for (int q = 0; q < 4; q++) base[q] = nb[q];
        }
        if (it != P.iters - 1) laf_left_mul(base, L0, cur);
        __syncwarp();   // every lane is done with this patch before the next one overwrites it
    }
    if (lane == 0) {
        float* o = P.out + row * 4;
        o[0] = base[0]; o[1] = base[1]; o[2] = base[2]; o[3] = base[3];
    }
}

static int launch_hc_pyr(bool ori, const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                         const int* d_count, int cap, int PS, int iters, const float* gk, float* d_out, cudaStream_t st) {
    AG_REQUIRE(plan && d_pyr && d_lafs && d_oct && d_lvl && d_count && gk && d_out, "NULL argument");
    AG_REQUIRE(PS >= 3 && PS <= HC_MAXPS, "patch size out of range (3..41)");
    AG_REQUIRE(cap >= 1 && plan->B >= 1 && plan->B <= 65535 && iters >= 1, "bad sizes");
    HcPyrParams P;
    P.G = make_geom(plan);
    P.pyr = d_pyr; P.lafs = d_lafs; P.oct = d_oct; P.lvl = d_lvl; P.count = d_count;
    P.cap = cap; P.PS = PS; P.iters = iters; P.out = d_out;
    memcpy(P.gk, gk, sizeof(float) * PS * PS);
    const size_t smem = sizeof(float) * HC_PYR_WARPS * (size_t)(ori ? hc_ori_warp_floats(PS) : hc_baum_warp_floats(PS));   // <= 59 KiB at PS 41
    static SmemAttrOnce attr_ori, attr_baum;
    if (smem > 48 * 1024) {
        const int rc = ori ? attr_ori.ensure(orientation_hist_pyr_kernel, smem, "orientation_hist_pyr smem attr")
                           : attr_baum.ensure(baumberg_pyr_kernel, smem, "baumberg_pyr smem attr");
        if (rc != AG_OK) return rc;
    }
    const dim3 grid(cdiv(cap, HC_PYR_WARPS), plan->B);
    if (ori) {
        orientation_hist_pyr_kernel<<<grid, HC_PYR_WARPS * 32, smem, st>>>(P);
        AG_CHECK_LAUNCH("orientation_hist_pyr_kernel");
    } else {
        baumberg_pyr_kernel<<<grid, HC_PYR_WARPS * 32, smem, st>>>(P);
        AG_CHECK_LAUNCH("baumberg_pyr_kernel");
    }
    return AG_OK;
}

int orientation_hist_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                         const int* d_count, int cap, int PS, const float* gk, float* d_R, void* stream) {
    return launch_hc_pyr(true, plan, d_pyr, d_lafs, d_oct, d_lvl, d_count, cap, PS, 1, gk, d_R, (cudaStream_t)stream);
}

int baumberg_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                 const int* d_count, int cap, int PS, int iters, const float* gk, float* d_A, void* stream) {
    return launch_hc_pyr(false, plan, d_pyr, d_lafs, d_oct, d_lvl, d_count, cap, PS, iters, gk, d_A, (cudaStream_t)stream);
}

// The device libm calls of the estimators, one element per thread, compiled with this file's flags (ag_debug_libm).
__global__ void libm_probe_kernel(const float* __restrict__ y, const float* __restrict__ x, int n, float* __restrict__ at,
                                  float* __restrict__ co, float* __restrict__ si) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    at[i] = atan2f(y[i], x[i]);
    co[i] = cosf(x[i]);
    si[i] = sinf(x[i]);
}

}  // namespace ag

using namespace ag;

extern "C" {

int ag_circular_gauss_kernel(int kernlen, double sigma, float* h_out) {
    AG_REQUIRE(h_out && kernlen >= 1, "bad arguments");
    // CircularGaussKernel(kernlen, sigma, circ_zeros=False, norm=True) under python3 (Utils.py:92-114)
    const double half = kernlen / 2.0, r2 = half * half;
    const double sigma2 = (sigma > 0.0) ? 2.0 * sigma * sigma : 0.9 * r2;
    const double step = (kernlen > 1) ? (2.0 * half) / (kernlen - 1) : 0.0;
    double sum = 0.0;
    for (int i = 0; i < kernlen; i++)
        for (int j = 0; j < kernlen; j++) {
            const double y = (i == kernlen - 1) ? half : -half + i * step, x = (j == kernlen - 1) ? half : -half + j * step;
            sum += exp(-(x * x + y * y) / sigma2);
        }
    for (int i = 0; i < kernlen; i++)
        for (int j = 0; j < kernlen; j++) {
            const double y = (i == kernlen - 1) ? half : -half + i * step, x = (j == kernlen - 1) ? half : -half + j * step;
            h_out[i * kernlen + j] = (float)(exp(-(x * x + y * y) / sigma2) / sum);
        }
    return AG_OK;
}

int ag_orientation_hist(const float* d_patches, int n, int PS, const float* d_gk, float* d_angle, void* stream) {
    AG_REQUIRE(d_patches && d_gk && d_angle, "NULL argument");
    AG_REQUIRE(PS >= 3 && PS <= HC_MAXPS, "patch size out of range (3..41)");
    if (n <= 0) return AG_OK;
    orientation_hist_kernel<<<cdiv(n, HC_WARPS), HC_WARPS * 32, 0, (cudaStream_t)stream>>>(d_patches, n, PS, d_gk, d_angle);
    AG_CHECK_LAUNCH("orientation_hist_kernel");
    return AG_OK;
}

int ag_baumberg_shape(const float* d_patches, int n, int PS, const float* d_gk, float* d_A, void* stream) {
    AG_REQUIRE(d_patches && d_gk && d_A, "NULL argument");
    AG_REQUIRE(PS >= 3 && PS <= HC_MAXPS, "patch size out of range (3..41)");
    if (n <= 0) return AG_OK;
    baumberg_kernel<<<cdiv(n, HC_WARPS), HC_WARPS * 32, 0, (cudaStream_t)stream>>>(d_patches, n, PS, d_gk, d_A);
    AG_CHECK_LAUNCH("baumberg_kernel");
    return AG_OK;
}

int ag_debug_libm(const float* d_y, const float* d_x, int n, float* d_atan2, float* d_cos, float* d_sin, void* stream) {
    AG_REQUIRE(d_y && d_x && d_atan2 && d_cos && d_sin, "NULL argument");
    if (n <= 0) return AG_OK;
    libm_probe_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(d_y, d_x, n, d_atan2, d_cos, d_sin);
    AG_CHECK_LAUNCH("libm_probe_kernel");
    return AG_OK;
}

int ag_debug_orientation_hist_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                                  const int* d_count, int cap, int PS, const float* h_gk, float* d_R, void* stream) {
    return launch_hc_pyr(true, plan, d_pyr, d_lafs, d_oct, d_lvl, d_count, cap, PS, 1, h_gk, d_R, (cudaStream_t)stream);
}

int ag_debug_baumberg_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                          const int* d_count, int cap, int PS, int iters, const float* h_gk, float* d_A, void* stream) {
    return launch_hc_pyr(false, plan, d_pyr, d_lafs, d_oct, d_lvl, d_count, cap, PS, iters, h_gk, d_A, (cudaStream_t)stream);
}

}  // extern "C"
