// SIFT descriptor (SIFTNet.forward, pytorch_sift.py:69-94): 8 angle bins x 4 x 4 spatial cells of gradient magnitude, weighted by the
// module's circular Gaussian window, pooled per angle bin by a k x k tent kernel with stride s, L2-normalised, clipped at `clipval` and
// L2-normalised again.  One block per patch; the patch (PS x PS, 16 <= PS <= 65) is staged in shared memory, either loaded from
// materialised patches (ag_sift_describe) or sampled from the pyramid (ag_sift_describe_pyr, the batched pipeline).  Both kernels call the
// same per-block body, so the fused kernel gives the bits of ag_extract_patches_pyr followed by ag_sift_describe.
#include <math.h>

#include "common.cuh"

namespace ag {

constexpr int SIFT_THREADS = 128;   // one thread per output value: 8 angle bins x 16 cells

struct SiftParams {
    PyrGeom G;
    const float* patches;   // [n,PS,PS] (ag_sift_describe)
    const float* pyr;       // the pyramid (ag_sift_describe_pyr)
    const float* lafs;      // [B,cap,2,3] normalised
    const int* oct;
    const int* lvl;
    const int* count;       // [B] or NULL (every row valid)
    int cap, PS, k, s;
    float clip;
    float* out;             // [rows,128]
    float gk[SIFT_MAX_PS * SIFT_MAX_PS];
    float pk[SIFT_MAX_K * SIFT_MAX_K];
};

// shared memory per block: the patch, the two bin weights per pixel and the lower bin index per pixel
__host__ __device__ inline size_t sift_smem_bytes(int PS) { return (size_t)PS * PS * (3 * sizeof(float) + 1) + 4 * sizeof(float); }

__device__ __forceinline__ float block_sum_128(float v, float* s_red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();   // s_red may still be read by the previous call
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    return (s_red[0] + s_red[1]) + (s_red[2] + s_red[3]);   // a fixed order: every thread gets the same bits
}

// SIFTNet.forward on the PS x PS patch `p` (shared memory, complete on entry) -> out[0..127] in [bin][cy][cx] order.  A non-finite bin
// weight (a NaN or infinite pixel, or gx^2 + gy^2 overflowing) at a pixel the pooling reads makes all 128 outputs NaN, as in the
// reference: it multiplies that weight by the 0 of every other bin's mask, and the NaN reaches every output through the L2 norms.
__device__ __forceinline__ void sift_block(const SiftParams& P, float* p, float* out) {
    const int PS = P.PS, NP = PS * PS;
    float* s_w0 = p + NP;
    float* s_w1 = s_w0 + NP;
    float* s_red = s_w1 + NP;
    unsigned char* s_b = (unsigned char*)(s_red + 4);
    const float TWO_PI_F = 6.28318530717958647692f;
    const int pooled = 3 * P.s + P.k;   // the four windows of a row / column cover [0, 3 s + k)
    int nonfinite = 0;
    for (int t = threadIdx.x; t < NP; t += SIFT_THREADS) {
        float gx, gy;
        const int ti = t / PS, tj = t % PS;
        grad_at(p, PS, ti, tj, -1.0f, 1.0f, gx, gy);   // weights (-1, 0, 1), replicate padding
        const float mag = __fmul_rn(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), 1e-10f)), P.gk[t]);
        const float ori = atan2f(gy, __fadd_rn(gx, 1e-8f));
        const float o_big = __fmul_rn(__fdiv_rn(__fadd_rn(ori, TWO_PI_F), TWO_PI_F), 8.0f);
        const float bo0 = floorf(o_big);
        const float wo1 = __fsub_rn(o_big, bo0);
        s_b[t] = (unsigned char)((int)bo0 & 7);                 // floor(o) % 8; the upper bin is (bo0 + 1) % 8
        const float w0 = __fmul_rn(__fsub_rn(1.0f, wo1), mag), w1 = __fmul_rn(wo1, mag);
        s_w0[t] = w0;
        s_w1[t] = w1;
        nonfinite |= (ti < pooled) & (tj < pooled) & !(isfinite(w0) & isfinite(w1));
    }
    nonfinite = __syncthreads_or(nonfinite);
    // the k x k pooling of angle bin `bin` over the window of cell (cy, cx), stride s, no padding
    const int bin = threadIdx.x & 7, cell = threadIdx.x >> 3, cy = cell >> 2, cx = cell & 3;
    const int k = P.k, base = cy * P.s * PS + cx * P.s;
    float acc = 0.f;
    for (int dy = 0; dy < k; dy++) {
        const int r = base + dy * PS;
        for (int dx = 0; dx < k; dx++) {
            const int b0 = s_b[r + dx];
            const float v = (b0 == bin) ? s_w0[r + dx] : (((b0 + 1) & 7) == bin ? s_w1[r + dx] : 0.f);
            acc = __fmaf_rn(P.pk[dy * k + dx], v, acc);
        }
    }
    // L2Norm, clamp(0, clipval), L2Norm
    float x = __fdiv_rn(acc, __fsqrt_rn(__fadd_rn(fabsf(block_sum_128(__fmul_rn(acc, acc), s_red)), 1e-10f)));
    x = fminf(fmaxf(x, 0.f), P.clip);
    x = __fdiv_rn(x, __fsqrt_rn(__fadd_rn(fabsf(block_sum_128(__fmul_rn(x, x), s_red)), 1e-10f)));
    out[bin * 16 + cell] = nonfinite ? __int_as_float(0x7fffffff) : x;
}

__global__ void __launch_bounds__(SIFT_THREADS) sift_kernel(const __grid_constant__ SiftParams P) {
    extern __shared__ float sift_smem[];
    const int NP = P.PS * P.PS;
    const size_t row = blockIdx.x;
    for (int t = threadIdx.x; t < NP; t += SIFT_THREADS) sift_smem[t] = P.patches[row * NP + t];
    __syncthreads();
    sift_block(P, sift_smem, P.out + row * 128);
}

// One block per keypoint (b, i), i < count[b]; the patch is sampled from pyr[oct][lvl] with the arithmetic of extract_patches_pyr_kernel
// (laf_sample_xy + bilinear_zero).
__global__ void __launch_bounds__(SIFT_THREADS) sift_pyr_kernel(const __grid_constant__ SiftParams P) {
    extern __shared__ float sift_smem[];
    const int b = blockIdx.y, i = blockIdx.x;
    if (P.count != nullptr && i >= P.count[b]) return;   // a count of -1 (overflow): nothing to do
    const long long row = (long long)b * P.cap + i;
    const int o = clampi(P.oct[row], 0, P.G.n_octaves - 1), l = clampi(P.lvl[row], 0, P.G.n_levels - 1);
    const int h = P.G.h[o], w = P.G.w[o];
    const float* img = P.pyr + P.G.off[o][l] + (size_t)b * h * w;
    const float* L = P.lafs + row * 6;
    const int PS = P.PS, NP = PS * PS;
    for (int t = threadIdx.x; t < NP; t += SIFT_THREADS) {
        const int pi = t / PS, pj = t - pi * PS;
        float px, py;
        laf_sample_xy(L, h, w, pi, pj, 1.0f / (float)PS, px, py);
        sift_smem[t] = bilinear_zero(img, h, w, px, py);
    }
    __syncthreads();
    sift_block(P, sift_smem, P.out + row * 128);
}

bool sift_geometry(int PS, int* k, int* s) {
    if (PS < SIFT_MIN_PS || PS > SIFT_MAX_PS) return false;
    // get_bin_weight_kernel_size_and_stride (pytorch_sift.py:26-29) with 4 spatial bins; 2 floor(PS/2) / 5 is never a tie of round()
    const int st = (int)nearbyint(2.0 * (double)(PS / 2) / 5.0), ks = 2 * st - 1;
    if ((PS - ks) / st + 1 != 4) return false;   // the pooling grid must come out 4 x 4
    if (k) *k = ks;
    if (s) *s = st;
    return true;
}

void sift_windows(int PS, int k, float* gk, float* pk) {
    // SIFTNet.CircularGaussKernel (pytorch_sift.py:31-44): centre kernlen / 2 (a float: 32.5 at PS 65), sigma^2 = 0.9 r^2, 0 outside
    // the circle, not normalised; float64, then rounded to fp32
    const double half = PS / 2.0, r2 = half * half, sigma2 = 0.9 * r2;
    for (int y = 0; y < PS; y++)
        for (int x = 0; x < PS; x++) {
            const double dy = y - half, dx = x - half;
            const double dy2 = dy * dy, dx2 = dx * dx, disq = dy2 + dx2;
            gk[y * PS + x] = disq < r2 ? (float)exp(-disq / sigma2) : 0.f;
        }
    // getPoolingKernel (pytorch_sift.py:19-25): np.arange(step / 2, 1, step) filled as numpy does (start + i * delta, delta = the
    // rounded second element minus the first), mirrored around a 1, outer product, float64, then rounded to fp32
    double xc[SIFT_MAX_K];
    const double step = 1.0 / (double)(k / 2), start = step / 2.0;
    const int n = (int)ceil((1.0 - start) / step);
    const double second = start + step, delta = second - start;
    for (int i = 0; i < n; i++) {
        const double v = i == 0 ? start : (i == 1 ? second : start + (double)i * delta);
        xc[i] = v;
        xc[2 * n - i] = v;
    }
    xc[n] = 1.0;
    for (int i = 0; i < k; i++)
        for (int j = 0; j < k; j++) {
            const double v = xc[i] * xc[j];
            pk[i * k + j] = (float)(v > 0.0 ? v : 0.0);
        }
}

static int launch_sift(bool pyr, const ag_pyramid_plan_t* plan, const float* d_src, const float* d_lafs, const int* d_oct,
                       const int* d_lvl, const int* d_count, int rows, int PS, int k, int s, const float* gk, const float* pk, float clipval,
                       float* d_out, cudaStream_t st) {
    SiftParams P;
    memset(&P, 0, sizeof(P));
    if (pyr) {
        P.G = make_geom(plan);
        P.pyr = d_src; P.lafs = d_lafs; P.oct = d_oct; P.lvl = d_lvl; P.count = d_count;
    } else {
        P.patches = d_src;
    }
    P.cap = rows; P.PS = PS; P.k = k; P.s = s; P.clip = clipval; P.out = d_out;
    memcpy(P.gk, gk, sizeof(float) * PS * PS);
    memcpy(P.pk, pk, sizeof(float) * k * k);
    const size_t smem = sift_smem_bytes(PS);   // <= 54.9 KB at PS 65
    static SmemAttrOnce attr_plain, attr_pyr;
    if (smem > 48 * 1024) {
        const int rc = pyr ? attr_pyr.ensure(sift_pyr_kernel, smem, "sift_pyr smem attr") : attr_plain.ensure(sift_kernel, smem, "sift smem attr");
        if (rc != AG_OK) return rc;
    }
    if (pyr) {
        sift_pyr_kernel<<<dim3(rows, plan->B), SIFT_THREADS, smem, st>>>(P);
        AG_CHECK_LAUNCH("sift_pyr_kernel");
    } else {
        sift_kernel<<<rows, SIFT_THREADS, smem, st>>>(P);
        AG_CHECK_LAUNCH("sift_kernel");
    }
    return AG_OK;
}

int sift_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl, const int* d_count,
             int cap, int PS, int k, int s, const float* gk, const float* pk, float clipval, float* d_out, void* stream) {
    return launch_sift(true, plan, d_pyr, d_lafs, d_oct, d_lvl, d_count, cap, PS, k, s, gk, pk, clipval, d_out,
                       (cudaStream_t)stream);
}

}  // namespace ag

using namespace ag;

extern "C" {

int ag_sift_windows(int PS, float* h_gk, float* h_pk, int* k, int* stride) {
    int ks, st;
    AG_REQUIRE(sift_geometry(PS, &ks, &st), "unsupported patch size: 16..65 with a 4 x 4 pooling grid (not 17, 18, 23, 28, 38, 48, 58)");
    float gk[SIFT_MAX_PS * SIFT_MAX_PS], pk[SIFT_MAX_K * SIFT_MAX_K];
    sift_windows(PS, ks, gk, pk);
    if (h_gk) memcpy(h_gk, gk, sizeof(float) * PS * PS);
    if (h_pk) memcpy(h_pk, pk, sizeof(float) * ks * ks);
    if (k) *k = ks;
    if (stride) *stride = st;
    return AG_OK;
}

int ag_sift_describe(const float* d_patches, int n, int PS, float clipval, float* d_out, void* stream) {
    int k, s;
    AG_REQUIRE(d_patches && d_out, "NULL argument");
    AG_REQUIRE(sift_geometry(PS, &k, &s), "unsupported patch size: 16..65 with a 4 x 4 pooling grid (not 17, 18, 23, 28, 38, 48, 58)");
    AG_REQUIRE(isfinite(clipval) && clipval > 0.f, "clipval must be finite and positive");
    AG_REQUIRE(n >= 0, "bad sizes");
    if (n == 0) return AG_OK;
    float gk[SIFT_MAX_PS * SIFT_MAX_PS], pk[SIFT_MAX_K * SIFT_MAX_K];
    sift_windows(PS, k, gk, pk);
    return launch_sift(false, nullptr, d_patches, nullptr, nullptr, nullptr, nullptr, n, PS, k, s, gk, pk, clipval, d_out,
                       (cudaStream_t)stream);
}

int ag_sift_describe_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                         const int* d_count, int cap, int PS, float clipval, float* d_out, void* stream) {
    int k, s;
    AG_REQUIRE(plan && d_pyr && d_lafs && d_oct && d_lvl && d_out, "NULL argument");
    AG_REQUIRE(sift_geometry(PS, &k, &s), "unsupported patch size: 16..65 with a 4 x 4 pooling grid (not 17, 18, 23, 28, 38, 48, 58)");
    AG_REQUIRE(isfinite(clipval) && clipval > 0.f, "clipval must be finite and positive");
    AG_REQUIRE(cap >= 1 && plan->B >= 1 && plan->B <= 65535, "bad sizes");
    float gk[SIFT_MAX_PS * SIFT_MAX_PS], pk[SIFT_MAX_K * SIFT_MAX_K];
    sift_windows(PS, k, gk, pk);
    return sift_pyr(plan, d_pyr, d_lafs, d_oct, d_lvl, d_count, cap, PS, k, s, gk, pk, clipval, d_out, stream);
}

}  // extern "C"
