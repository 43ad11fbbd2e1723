// Shared helpers for the affnet_b200 CUDA library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/affnet_b200.h"

namespace ag {

void set_error(const char* fmt, ...);
extern thread_local int g_launches;  // kernels launched since last reset (host-side counter)

inline int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return AG_OK;
    set_error("%s: %s", what, cudaGetErrorString(e));
    return (e == cudaErrorNoKernelImageForDevice || e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver)
               ? AG_ERR_NO_DEVICE
               : AG_ERR_CUDA;
}

void prof_mark(const char* name);  // records an event after a launch when profiling is on (see ag_prof_begin)

#define AG_CHECK_LAUNCH(name)                                        \
    do {                                                             \
        ::ag::g_launches++;                                          \
        int _rc = ::ag::check_cuda(cudaGetLastError(), name);        \
        if (_rc != AG_OK) return _rc;                                \
        ::ag::prof_mark(name);                                       \
    } while (0)

#define AG_REQUIRE(cond, msg)                                        \
    do {                                                             \
        if (!(cond)) {                                               \
            ::ag::set_error("%s: %s", __func__, msg);                \
            return AG_ERR_INVALID;                                   \
        }                                                            \
    } while (0)

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute: remember per device what was set (a process may drive several GPUs)
struct SmemAttrOnce {
    size_t set[64] = {};
    template <typename K>
    int ensure(K kernel, size_t bytes, const char* what) {
        int dev = 0;
        cudaGetDevice(&dev);
        dev &= 63;
        if (bytes <= set[dev]) return AG_OK;
        int rc = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes), what);
        if (rc == AG_OK) set[dev] = bytes;
        return rc;
    }
};

inline int cdiv(int a, int b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Order-preserving float -> uint32 (larger float => larger uint), total order incl. negatives.
__host__ __device__ inline uint32_t float_to_ordered(float f) {
    uint32_t u;
#ifdef __CUDA_ARCH__
    u = __float_as_uint(f);
#else
    memcpy(&u, &f, 4);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Exclusive prefix sum of one int per thread over a block of NT threads (a multiple of 32, at most 1024); `total` receives the block's
// sum.  s_warp holds NT / 32 ints of shared memory.  Starts and ends with a barrier, so it may be called in a loop on the same s_warp.
template <int NT>
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int& total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    __syncthreads();
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    int before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; w++) {
        const int t = s_warp[w];
        before += (w < wid) ? t : 0;
        sum += t;
    }
    total = sum;
    __syncthreads();
    return before + incl - v;
}

// Block-wide bitonic sort (descending) of n = 2^k 64-bit keys in shared memory, optionally with an int payload.  Every thread owns whole
// compare-exchange PAIRS (pair p -> elements i = p with a 0 bit inserted at log2(j), i | j), so no thread idles on the "ixj > i" half:
// half the loop trips of the textbook form.
template <bool HAS_IDX>
__device__ __forceinline__ void bitonic_sort_desc(unsigned long long* key, int* idx, int n) {
    for (int k2 = 2; k2 <= n; k2 <<= 1)
        for (int j = k2 >> 1; j > 0; j >>= 1) {
            for (int p = threadIdx.x; p < (n >> 1); p += blockDim.x) {
                const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1)), l = i | j;
                const unsigned long long a = key[i], c = key[l];
                const bool desc = (i & k2) == 0;
                if (desc ? (a < c) : (a > c)) {
                    key[i] = c; key[l] = a;
                    if (HAS_IDX) { const int t = idx[i]; idx[i] = idx[l]; idx[l] = t; }
                }
            }
            __syncthreads();
        }
}

// Bilinear tap with zeros outside the image (F.grid_sample, padding_mode='zeros').  Explicit rounding steps so that the
// standalone sampler and the sampler fused into the first CNN layer produce identical bits.
// The integer corner is converted from the floor clamped to [-2, w] x [-2, h]: every tap outside the image stays outside, and a
// sample point beyond the int32 range cannot saturate to INT_MAX, whose x0 + 1 would wrap into the "inside" test.
__device__ __forceinline__ float bilinear_zero(const float* __restrict__ img, int h, int w, float px, float py) {
    const float fx0 = floorf(px), fy0 = floorf(py);
    const int x0 = (int)fminf(fmaxf(fx0, -2.f), (float)w), y0 = (int)fminf(fmaxf(fy0, -2.f), (float)h);
    const float ax = __fsub_rn(px, fx0), ay = __fsub_rn(py, fy0);
    const float bx = __fsub_rn(1.f, ax), by = __fsub_rn(1.f, ay);
    const bool xin0 = (x0 >= 0) & (x0 < w), xin1 = (x0 + 1 >= 0) & (x0 + 1 < w);
    const bool yin0 = (y0 >= 0) & (y0 < h), yin1 = (y0 + 1 >= 0) & (y0 + 1 < h);
    const float v00 = (xin0 & yin0) ? __ldg(img + (size_t)y0 * w + x0) : 0.f;
    const float v01 = (xin1 & yin0) ? __ldg(img + (size_t)y0 * w + x0 + 1) : 0.f;
    const float v10 = (xin0 & yin1) ? __ldg(img + (size_t)(y0 + 1) * w + x0) : 0.f;
    const float v11 = (xin1 & yin1) ? __ldg(img + (size_t)(y0 + 1) * w + x0 + 1) : 0.f;
    const float top = __fmaf_rn(v01, ax, __fmul_rn(v00, bx)), bot = __fmaf_rn(v11, ax, __fmul_rn(v10, bx));
    return __fmaf_rn(bot, ay, __fmul_rn(top, by));
}

// The same tap in two phases (issue the four loads early, combine later); bit-identical to bilinear_zero.
__device__ __forceinline__ void bilinear_taps(const float* __restrict__ img, int h, int w, float px, float py, float (&t)[4], float& ax, float& ay) {
    const float fx0 = floorf(px), fy0 = floorf(py);
    const int x0 = (int)fminf(fmaxf(fx0, -2.f), (float)w), y0 = (int)fminf(fmaxf(fy0, -2.f), (float)h);   // as bilinear_zero
    ax = __fsub_rn(px, fx0); ay = __fsub_rn(py, fy0);
    const bool xin0 = (x0 >= 0) & (x0 < w), xin1 = (x0 + 1 >= 0) & (x0 + 1 < w);
    const bool yin0 = (y0 >= 0) & (y0 < h), yin1 = (y0 + 1 >= 0) & (y0 + 1 < h);
    t[0] = (xin0 & yin0) ? __ldg(img + (size_t)y0 * w + x0) : 0.f;
    t[1] = (xin1 & yin0) ? __ldg(img + (size_t)y0 * w + x0 + 1) : 0.f;
    t[2] = (xin0 & yin1) ? __ldg(img + (size_t)(y0 + 1) * w + x0) : 0.f;
    t[3] = (xin1 & yin1) ? __ldg(img + (size_t)(y0 + 1) * w + x0 + 1) : 0.f;
}
__device__ __forceinline__ float bilinear_combine(const float (&t)[4], float ax, float ay) {
    const float bx = __fsub_rn(1.f, ax), by = __fsub_rn(1.f, ay);
    const float top = __fmaf_rn(t[1], ax, __fmul_rn(t[0], bx)), bot = __fmaf_rn(t[3], ax, __fmul_rn(t[2], bx));
    return __fmaf_rn(bot, ay, __fmul_rn(top, by));
}

// Patch-grid coordinate of sample (i,j) of a PSxPS patch under a normalised LAF on an h x w image (LAF.py:313-324).
__device__ __forceinline__ void laf_sample_xy(const float* __restrict__ L, int h, int w, int i, int j, float inv_ps, float& px, float& py) {
    const float ms = (float)min(h, w);
    const float a11 = __fmul_rn(L[0], ms), a12 = __fmul_rn(L[1], ms), tx = __fmul_rn(L[2], (float)w);
    const float a21 = __fmul_rn(L[3], ms), a22 = __fmul_rn(L[4], ms), ty = __fmul_rn(L[5], (float)h);
    const float xj = __fsub_rn(__fmul_rn(__fmaf_rn(2.f, (float)j, 1.f), inv_ps), 1.f), yi = __fsub_rn(__fmul_rn(__fmaf_rn(2.f, (float)i, 1.f), inv_ps), 1.f);
    px = __fsub_rn(__fmaf_rn(a11, xj, __fmaf_rn(a12, yi, tx)), 0.5f);
    py = __fsub_rn(__fmaf_rn(a21, xj, __fmaf_rn(a22, yi, ty)), 0.5f);
}

// Gradient of a PS x PS patch with replicate padding; (wm, wp) = (w_minus, w_plus) of the (1x3) / (3x1) cross-correlation.  Used by the
// hand-crafted estimators (handcrafted.cu) and the SIFT descriptor (sift.cu).
__device__ __forceinline__ void grad_at(const float* p, int PS, int i, int j, float wm, float wp, float& gx, float& gy) {
    const int jm = max(j - 1, 0), jp = min(j + 1, PS - 1), im = max(i - 1, 0), ip = min(i + 1, PS - 1);
    gx = __fadd_rn(__fmul_rn(wm, p[i * PS + jm]), __fmul_rn(wp, p[i * PS + jp]));
    gy = __fadd_rn(__fmul_rn(wm, p[im * PS + j]), __fmul_rn(wp, p[ip * PS + j]));
}

// Pyramid geometry passed by value to the kernels that sample pyr[oct][lvl] directly.
struct PyrGeom {
    int n_octaves, n_levels, B;
    int h[AG_MAX_OCTAVES], w[AG_MAX_OCTAVES];
    long long off[AG_MAX_OCTAVES][AG_MAX_LEVELS];
};

inline PyrGeom make_geom(const ag_pyramid_plan_t* p) {
    PyrGeom g;
    g.n_octaves = p->n_octaves; g.n_levels = p->n_levels; g.B = p->B;
    for (int o = 0; o < AG_MAX_OCTAVES; o++) {
        g.h[o] = p->h[o]; g.w[o] = p->w[o];
        for (int l = 0; l < AG_MAX_LEVELS; l++) g.off[o][l] = p->level_offset[o][l];
    }
    return g;
}

// Hand-crafted estimators sampling the pyramid (handcrafted.cu), used by the batched pipeline.  `gk` is the module's Gaussian window
// (PS x PS, host memory: copied into the launch parameters).  Rows at or beyond d_count[b] are neither read nor written.
//   orientation_hist_pyr: d_R [B,cap,2,2] = [[cos, sin], [-sin, cos]] of the gradient-histogram angle at pyr[oct][lvl]
//   baumberg_pyr:         d_A [B,cap,2,2] = base_A after `iters` Baumberg iterations (SparseImgRepresenter.py:127-141)
int orientation_hist_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                         const int* d_count, int cap, int PS, const float* gk, float* d_R, void* stream);
int baumberg_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                 const int* d_count, int cap, int PS, int iters, const float* gk, float* d_A, void* stream);

// SIFT descriptor (sift.cu).  sift_geometry: false unless 16 <= PS <= 65 and the pooling grid is 4 x 4, else k and s of
// get_bin_weight_kernel_size_and_stride.  sift_windows: SIFTNet's Gaussian window gk [PS,PS] and pooling kernel pk [k,k] (host).
// sift_pyr: ag_sift_describe_pyr with the windows given (the pipeline computes them once at create time).
constexpr int SIFT_MIN_PS = 16, SIFT_MAX_PS = 65, SIFT_MAX_K = 25;
bool sift_geometry(int PS, int* k, int* s);
void sift_windows(int PS, int k, float* gk, float* pk);
int sift_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl, const int* d_count,
             int cap, int PS, int k, int s, const float* gk, const float* pk, float clipval, float* d_out, void* stream);

// 2x2 products in torch.bmm's fp32 CPU arithmetic: each entry rounds both products and then adds them, fl(fl(a*b) + fl(c*d)) (no fused
// multiply-add: it differs in about a quarter of the entries), into an accumulator that starts at +0 (two -0 products give +0).  Used by the Baumberg chain (mat2_compose_kernel /
// lafs_left_multiply_kernel, baumberg_pyr_kernel in handcrafted.cu) and by the shape filter's compose and the orientation compose
// (geometry.cu); tests/geometry_restated.py states the same arithmetic.
__device__ __forceinline__ float dot2_rn(float a, float b, float c, float d) {
    return __fadd_rn(__fadd_rn(0.f, __fmul_rn(a, b)), __fmul_rn(c, d));
}
// out = A * B   (base_A <- A base_A, SparseImgRepresenter.py:133)
__device__ __forceinline__ void mat2_mul(const float (&a)[4], const float (&b)[4], float (&o)[4]) {
    o[0] = dot2_rn(a[0], b[0], a[1], b[2]); o[1] = dot2_rn(a[0], b[1], a[1], b[3]);
    o[2] = dot2_rn(a[2], b[0], a[3], b[2]); o[3] = dot2_rn(a[2], b[1], a[3], b[3]);
}
// out = [A * L[:, :2] | L[:, 2]]   (the working LAF of the next Baumberg iteration, SparseImgRepresenter.py:134-135)
__device__ __forceinline__ void laf_left_mul(const float (&a)[4], const float (&l)[6], float (&o)[6]) {
    o[0] = dot2_rn(a[0], l[0], a[1], l[3]); o[1] = dot2_rn(a[0], l[1], a[1], l[4]); o[2] = l[2];
    o[3] = dot2_rn(a[2], l[0], a[3], l[3]); o[4] = dot2_rn(a[2], l[1], a[3], l[4]); o[5] = l[5];
}
// rectifyAffineTransformationUpIsUp (LAF.py:285-291) of [[a00, a01], [a10, a11]] -> A[4], each torch operation one fp32 operation in
// the expression's left-to-right order (no contraction); A[0,1] = 0 * det as in the reference (NaN when det is).  Shared by the
// Baumberg estimator and the AffNet heads, and restated by tests/handcrafted_restated.py and tests/nets_restated.py.
__device__ __forceinline__ void rectify_up_is_up(float a00, float a01, float a10, float a11, float* A) {
    const float det = __fsqrt_rn(fabsf(__fadd_rn(__fsub_rn(__fmul_rn(a00, a11), __fmul_rn(a10, a01)), 1e-10f)));
    const float b2a2 = __fsqrt_rn(__fadd_rn(__fmul_rn(a01, a01), __fmul_rn(a00, a00)));
    A[0] = __fdiv_rn(b2a2, det); A[1] = __fmul_rn(0.f, det);
    A[2] = __fdiv_rn(__fadd_rn(__fmul_rn(a11, a01), __fmul_rn(a10, a00)), __fmul_rn(b2a2, det)); A[3] = __fdiv_rn(det, b2a2);
}

}  // namespace ag
