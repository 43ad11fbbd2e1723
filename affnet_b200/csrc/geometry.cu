// Per-keypoint geometry: affine-shape filter, orientation compose, LAF (de)normalisation
// (SURVEY.md §8a rows a10 (partly), a11, a13, a14).
//
// Replaces the tail of getAffineShape (SparseImgRepresenter.py:136-162) with batch_eig2x2 (Utils.py:168-175)
// and checkTouchBoundary (LAF.py:98-104), the compose step of getOrientation (SparseImgRepresenter.py:175)
// and denormalizeLAFs / normalizeLAFs (LAF.py:407-429).
// Decisions (eigen-ratio test, boundary test) use the reference's fp32 operation order with non-contracted
// intrinsics so that identical A matrices give the identical survivor set.
#include "common.cuh"
#include "topk.cuh"

namespace ag {

constexpr int GNT = 1024;

struct ShapeParams {
    const float* A;      // [B,cap,2,2]
    const float* resp;   // [B,cap]
    const float* lafs;   // [B,cap,2,3]
    const int* oct;
    const int* lvl;
    const int* count_in;
    int cap, num_features, out_cap, sort_cap;
    float* resp_out;
    float* lafs_out;
    int* oct_out;
    int* lvl_out;
    int* count_out;
};

__device__ __forceinline__ bool shape_ok(const float* A, const float* NL) {
    // batch_eig2x2 (Utils.py:168-175)
    const float trace = __fadd_rn(A[0], A[3]);
    const float det = __fsub_rn(__fmul_rn(A[0], A[3]), __fmul_rn(A[2], A[1]));
    const float delta1 = __fsub_rn(__fmul_rn(trace, trace), __fmul_rn(4.0f, det));
    float l1, l2;
    if (delta1 > 0.f) {
        const float delta = __fsqrt_rn(fabsf(delta1));
        l1 = __fdiv_rn(__fadd_rn(trace, delta), 2.0f);
        l2 = __fdiv_rn(__fsub_rn(trace, delta), 2.0f);
    } else {
        l1 = 1000.0f; l2 = 0.0001f;
    }
    const float ratio = fabsf(__fdiv_rn(l1, __fadd_rn(l2, 1e-8f)));
    bool ok = (ratio < 6.0f) && (ratio > (float)(1.0 / 6.0));  // SparseImgRepresenter.py:149
    // checkTouchBoundary (LAF.py:98-104): corners (+-1,+-1) through the normalised LAF must lie in [0,1] (Q5)
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const float x = (c & 2) ? 1.f : -1.f, y = (c & 1) ? 1.f : -1.f;
        // (h0*x + h1*y) + h2, as the reference's matmul sums it (h1*y + h2 first can put a corner on the other side of 0 or 1)
        const float ox = __fadd_rn(__fadd_rn(__fmul_rn(NL[0], x), __fmul_rn(NL[1], y)), NL[2]);
        const float oy = __fadd_rn(__fadd_rn(__fmul_rn(NL[3], x), __fmul_rn(NL[4], y)), NL[5]);
        ok = ok && !(ox > 1.0f || ox < 0.0f || oy > 1.0f || oy < 0.0f);
    }
    return ok;
}

__device__ __forceinline__ void compose_laf(const float* A, const float* L, float* NL) {
    // new_LAF = [bmm(A, LAF[:, :, 0:2]), LAF[:, :, 2:]]   SparseImgRepresenter.py:138 (laf_left_mul: both products rounded, as bmm)
    const float a[4] = {A[0], A[1], A[2], A[3]};
    const float l[6] = {L[0], L[1], L[2], L[3], L[4], L[5]};
    float o[6];
    laf_left_mul(a, l, o);
#pragma unroll
    for (int q = 0; q < 6; q++) NL[q] = o[q];
}

__global__ void __launch_bounds__(GNT) shape_filter_kernel(const ShapeParams P) {
    extern __shared__ unsigned long long s_key[];
    __shared__ int s_surv;
    const int b = blockIdx.x;
    const int n = max(0, min(P.count_in[b], P.cap));
    const float* A = P.A + (size_t)b * P.cap * 4;
    const float* L = P.lafs + (size_t)b * P.cap * 6;
    const float* R = P.resp + (size_t)b * P.cap;
    if (threadIdx.x == 0) s_surv = 0;
    __syncthreads();
    // pass 1: count survivors
    int local = 0;
    for (int i = threadIdx.x; i < n; i += GNT) {
        float NL[6];
        compose_laf(A + i * 4, L + i * 6, NL);
        local += shape_ok(A + i * 4, NL) ? 1 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(&s_surv, local);
    __syncthreads();
    const int S = s_surv;
    const bool sorted = (P.num_features > 0) && (S > P.num_features);  // SparseImgRepresenter.py:151
    int m = sorted ? P.num_features : S;
    if (m > P.out_cap) m = P.out_cap;
    // pass 2: keys
    for (int i = threadIdx.x; i < P.sort_cap; i += GNT) {
        unsigned long long k = 0ull;
        if (i < n) {
            float NL[6];
            compose_laf(A + i * 4, L + i * 6, NL);
            const bool ok = shape_ok(A + i * 4, NL);
            // sorted: the key is resp * mask (rejected rows as zeros, ahead of negative survivors), -0 made +0 so that it ties by index
            const unsigned hi = sorted ? float_to_ordered(__fadd_rn(__fmul_rn(R[i], ok ? 1.f : 0.f), 0.f)) : (ok ? 1u : 0u);
            k = ((unsigned long long)hi << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i);
        }
        s_key[i] = k;
    }
    __syncthreads();
    bitonic_sort_desc<false>(s_key, nullptr, P.sort_cap);
    for (int r = threadIdx.x; r < m; r += GNT) {
        const int i = (int)(0xFFFFFFFFu - (unsigned)(s_key[r] & 0xFFFFFFFFull));
        const size_t o = (size_t)b * P.out_cap + r;
        float NL[6];
        compose_laf(A + i * 4, L + i * 6, NL);
        // sorted: topk's value, resp * mask (a rejected row that makes the cut comes out as the reference's zero); else resp
        P.resp_out[o] = sorted ? __fmul_rn(R[i], shape_ok(A + i * 4, NL) ? 1.f : 0.f) : R[i];
#pragma unroll
        for (int q = 0; q < 6; q++) P.lafs_out[o * 6 + q] = NL[q];
        P.oct_out[o] = P.oct[(size_t)b * P.cap + i];
        P.lvl_out[o] = P.lvl[(size_t)b * P.cap + i];
    }
    if (threadIdx.x == 0) P.count_out[b] = (P.count_in[b] < 0) ? -1 : m;   // -1 = upstream capacity overflow, propagated
}

// getAffineShape's num_features <= 0 branch (SparseImgRepresenter.py:151-156): every survivor in index order with its response unchanged,
// at any cap.  One CTA per image walks the rows in chunks of GNT * FA_RPT; a block scan of the survivor flags gives each survivor its output
// row.  Same compose_laf / shape_ok as shape_filter_kernel, so the rows equal its num_features = 0 answer bit for bit.
constexpr int FA_RPT = 4;   // consecutive rows per thread and chunk

__global__ void __launch_bounds__(GNT) shape_filter_all_kernel(const ShapeParams P) {
    __shared__ int s_warp[GNT / 32];
    const int b = blockIdx.x;
    const int cin = P.count_in[b];
    const int n = max(0, min(cin, P.cap));
    const size_t rb = (size_t)b * P.cap;
    const float* A = P.A + rb * 4;
    const float* L = P.lafs + rb * 6;
    int base = 0;
    for (int r0 = 0; r0 < n; r0 += GNT * FA_RPT) {
        const int i0 = r0 + threadIdx.x * FA_RPT;
        float NL[FA_RPT][6];
        bool ok[FA_RPT];
        int c = 0;
#pragma unroll
        for (int k = 0; k < FA_RPT; k++) {
            const int i = i0 + k;
            ok[k] = false;
            if (i < n) {
                compose_laf(A + (size_t)i * 4, L + (size_t)i * 6, NL[k]);
                ok[k] = shape_ok(A + (size_t)i * 4, NL[k]);
            }
            c += ok[k] ? 1 : 0;
        }
        int total;
        int dst = base + block_exclusive_scan<GNT>(c, s_warp, total);
#pragma unroll
        for (int k = 0; k < FA_RPT; k++) {
            if (!ok[k]) continue;
            const size_t i = rb + i0 + k, o = rb + dst++;
            P.resp_out[o] = P.resp[i];
#pragma unroll
            for (int q = 0; q < 6; q++) P.lafs_out[o * 6 + q] = NL[k][q];
            P.oct_out[o] = P.oct[i];
            P.lvl_out[o] = P.lvl[i];
        }
        base += total;
    }
    if (threadIdx.x == 0) P.count_out[b] = (cin < 0) ? -1 : base;   // -1 = upstream capacity overflow, propagated
}

// ---- top-K filter at any cap (ag_affine_shape_filter_topk above TOPK_SMEM_MAX rows) -----------------------------------------------------
// shape_filter_kernel's rule on the global-memory top-m primitive (topk.cuh).  One pass over the rows writes each row's keep flag, its
// sorted-mode key resp * keep (-0 made +0) and the survivor count; the key source then reads them, and the writer recomputes the row with the
// same compose_laf / shape_ok.
constexpr int SK_NT = 256;

__global__ void __launch_bounds__(SK_NT) shape_keys_kernel(const ShapeParams P, uint32_t* __restrict__ ord, unsigned char* __restrict__ keep,
                                                           int* __restrict__ surv) {
    const int b = blockIdx.y, i = blockIdx.x * SK_NT + threadIdx.x;
    const int n = max(0, min(P.count_in[b], P.cap));
    bool ok = false;
    if (i < n) {
        const size_t r = (size_t)b * P.cap + i;
        float NL[6];
        compose_laf(P.A + r * 4, P.lafs + r * 6, NL);
        ok = shape_ok(P.A + r * 4, NL);
        ord[r] = float_to_ordered(__fadd_rn(__fmul_rn(P.resp[r], ok ? 1.f : 0.f), 0.f));
        keep[r] = ok ? 1 : 0;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&surv[b], __popc(bal));
}

struct ShapeTopkSrc {
    const uint32_t* ord;
    const unsigned char* keep;
    const int* surv;
    const int* count_in;
    int cap, num_features, out_cap;

    __device__ TopkSetup setup(int b) const {
        const int S = surv[b];
        const bool sorted = (num_features > 0) && (S > num_features);  // SparseImgRepresenter.py:151
        int m = sorted ? num_features : S;
        if (m > out_cap) m = out_cap;
        TopkSetup t;
        t.n = max(0, min(count_in[b], cap)); t.m = m; t.sorted = sorted; t.radix = 1; t.fail = count_in[b] < 0; t.ctx = 0;
        return t;
    }
    // shape_filter_kernel's key: sorted, (resp * keep, row ascending); else (keep, row ascending)
    __device__ unsigned long long key(int b, int i, const TopkSetup& t) const {
        const size_t r = (size_t)b * cap + i;
        const unsigned hi = t.sorted ? ord[r] : (unsigned)keep[r];
        return ((unsigned long long)hi << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i);
    }
};

__global__ void __launch_bounds__(SK_NT) shape_topk_write_kernel(const ShapeParams P, const int* __restrict__ idx, const TopkImage* __restrict__ img,
                                                                 int rows) {
    const int b = blockIdx.y, r = blockIdx.x * SK_NT + threadIdx.x;
    const TopkImage im = img[b];
    if (r == 0) P.count_out[b] = im.count;   // -1 = upstream capacity overflow, propagated
    if (r >= im.count) return;
    const int i = idx[(size_t)b * rows + r];
    const size_t ri = (size_t)b * P.cap + i, o = (size_t)b * P.out_cap + r;
    float NL[6];
    compose_laf(P.A + ri * 4, P.lafs + ri * 6, NL);
    P.resp_out[o] = im.sorted ? __fmul_rn(P.resp[ri], shape_ok(P.A + ri * 4, NL) ? 1.f : 0.f) : P.resp[ri];
#pragma unroll
    for (int q = 0; q < 6; q++) P.lafs_out[o * 6 + q] = NL[q];
    P.oct_out[o] = P.oct[ri];
    P.lvl_out[o] = P.lvl[ri];
}

__global__ void lafs_rotate_kernel(float* __restrict__ lafs, const float* __restrict__ R, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float* L = lafs + (size_t)i * 6;
    const float* r = R + (size_t)i * 4;
    const float l[4] = {L[0], L[1], L[3], L[4]}, rr[4] = {r[0], r[1], r[2], r[3]};
    float o[4];
    mat2_mul(l, rr, o);   // bmm(LAF[:, :, :2], R), SparseImgRepresenter.py:175
    L[0] = o[0]; L[1] = o[1]; L[3] = o[2]; L[4] = o[3];
}

__global__ void lafs_scale_kernel(const float* __restrict__ in, float* __restrict__ out, int n, float ac, float xc, float yc) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* L = in + (size_t)i * 6;
    float* O = out + (size_t)i * 6;
    O[0] = __fmul_rn(L[0], ac); O[1] = __fmul_rn(L[1], ac); O[2] = __fmul_rn(L[2], xc);
    O[3] = __fmul_rn(L[3], ac); O[4] = __fmul_rn(L[4], ac); O[5] = __fmul_rn(L[5], yc);
}

// LAFs2ellT (LAF.py:35-51) with the closed-form 2x2 SVD of bsvd2x2 (LAF.py:106-144): one thread per keypoint.  Only U and
// the singular values of A / scale enter the result: ell = (x, y, M00, M01, M11), M = U diag(1 / (scale^2 s_i^2)) U^T.
__global__ void lafs_to_ell_kernel(const float* __restrict__ lafs, float* __restrict__ ell, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* L = lafs + (size_t)i * 6;
    const float scale = sqrtf(__fadd_rn(__fsub_rn(__fmul_rn(L[0], L[4]), __fmul_rn(L[1], L[3])), 1e-10f));   // not contracted
    const float a00 = L[0] / scale, a01 = L[1] / scale, a10 = L[3] / scale, a11 = L[4] / scale;
    // Su = A A^T
    const float s00 = a00 * a00 + a01 * a01, s01 = a00 * a10 + a01 * a11, s11 = a10 * a10 + a11 * a11;
    const float phi = 0.5f * atan2f(s01 + s01 + 1e-12f, s00 - s11 + 1e-12f);
    const float c = cosf(phi), sn = sinf(phi);   // U = [[c, -s], [s, c]]
    const float sum = s00 + s11;
    const float dif = sqrtf((s00 - s11) * (s00 - s11) + 4.0f * s01 * s01 + 1e-12f);
    const float sig0 = sqrtf((sum + dif) / 2.0f), sig1 = sqrtf((sum - dif) / 2.0f);
    const float w0 = 1.0f / (scale * scale * sig0 * sig0), w1 = 1.0f / (scale * scale * sig1 * sig1);
    float* o = ell + (size_t)i * 5;
    o[0] = L[2]; o[1] = L[5];
    o[2] = c * w0 * c + sn * w1 * sn;          // (U W U^T)[0][0]
    o[3] = c * w0 * sn - sn * w1 * c;          // [0][1]
    o[4] = sn * w0 * sn + c * w1 * c;          // [1][1]
}

// ells2LAFsT (LAF.py:76-89) with invSqrtTorch (:52-74): one thread per ellipse, each torch operation one rounded fp32 operation in the
// expression's left-to-right order (tests/given_restated.py states the same).  torch.sign is (x > 0) - (x < 0): 0 for +-0 and NaN.
__global__ void ells_to_lafs_kernel(const float* __restrict__ ell, float* __restrict__ lafs, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float* E = ell + (size_t)i * 5;
    const float a = E[2], b = E[3], c = E[4];
    const float sc = __fsqrt_rn(__fsqrt_rn(__fadd_rn(__fsub_rn(__fmul_rn(a, c), __fmul_rn(b, b)), 1e-12f)));
    // invSqrtTorch
    const float mask = (b != 0.f) ? 1.f : 0.f;
    const float r1 = __fdiv_rn(__fmul_rn(mask, __fsub_rn(c, a)), __fadd_rn(__fmul_rn(2.f, b), 1e-12f));
    const float sg = (r1 > 0.f) ? 1.f : ((r1 < 0.f) ? -1.f : 0.f);
    const float t1 = __fdiv_rn(sg, __fadd_rn(fabsf(r1), __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(r1, r1)))));
    float r = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(t1, t1))));
    float t = __fmul_rn(t1, r);
    r = __fadd_rn(__fmul_rn(r, mask), __fmul_rn(1.f, __fsub_rn(1.f, mask)));
    t = __fmul_rn(t, mask);
    const float rr = __fmul_rn(r, r), tt = __fmul_rn(t, t), rt2 = __fmul_rn(__fmul_rn(2.f, r), t);
    float x = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fsub_rn(__fmul_rn(rr, a), __fmul_rn(rt2, b)), __fmul_rn(tt, c))));
    float z = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(tt, a), __fmul_rn(rt2, b)), __fmul_rn(rr, c))));
    const float d = __fsqrt_rn(__fmul_rn(x, z));
    x = __fdiv_rn(x, d);
    z = __fdiv_rn(z, d);
    const float ia = __fadd_rn(__fmul_rn(rr, x), __fmul_rn(tt, z));
    const float ib = __fadd_rn(__fmul_rn(__fmul_rn(-r, t), x), __fmul_rn(__fmul_rn(t, r), z));
    const float ic = __fadd_rn(__fmul_rn(tt, x), __fmul_rn(rr, z));
    // A = [[ia, ib], [ib, ic]] / sc; its scale; rectifyAffineTransformationUpIsUp(A / scale) * scale
    const float a00 = __fdiv_rn(ia, sc), a01 = __fdiv_rn(ib, sc), a11 = __fdiv_rn(ic, sc);
    const float s = __fsqrt_rn(fabsf(__fsub_rn(__fmul_rn(a00, a11), __fmul_rn(a01, a01))));
    float R[4];
    rectify_up_is_up(__fdiv_rn(a00, s), __fdiv_rn(a01, s), __fdiv_rn(a01, s), __fdiv_rn(a11, s), R);
    float* L = lafs + (size_t)i * 6;
    L[0] = __fmul_rn(R[0], s); L[1] = __fmul_rn(R[1], s); L[2] = E[0];
    L[3] = __fmul_rn(R[2], s); L[4] = __fmul_rn(R[3], s); L[5] = E[1];
}

}  // namespace ag

using namespace ag;

namespace ag {
// out = A * B for [n,2,2] batches (mat2_mul, common.cuh): the Baumberg chain base_A <- A base_A of SparseImgRepresenter.py:133
__global__ void mat2_compose_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float a[4] = {A[i * 4], A[i * 4 + 1], A[i * 4 + 2], A[i * 4 + 3]};
    const float b[4] = {B[i * 4], B[i * 4 + 1], B[i * 4 + 2], B[i * 4 + 3]};
    float o[4];
    mat2_mul(a, b, o);
#pragma unroll
    for (int q = 0; q < 4; q++) out[i * 4 + q] = o[q];
}
// out = [A * L[:, :, :2] | L[:, :, 2]] (laf_left_mul, common.cuh): the working LAF of the next Baumberg iteration (SparseImgRepresenter.py:134-135)
__global__ void lafs_left_multiply_kernel(const float* __restrict__ A, const float* __restrict__ Lf, float* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float a[4] = {A[i * 4], A[i * 4 + 1], A[i * 4 + 2], A[i * 4 + 3]};
    float l[6], o[6];
#pragma unroll
    for (int q = 0; q < 6; q++) l[q] = Lf[i * 6 + q];
    laf_left_mul(a, l, o);
#pragma unroll
    for (int q = 0; q < 6; q++) out[i * 6 + q] = o[q];
}
}  // namespace ag

extern "C" {

int ag_affine_shape_filter(const float* d_A, const float* d_resp, const float* d_lafs, const int* d_oct, const int* d_lvl,
                           const int* d_count_in, int B, int cap, int num_features, int out_cap, float* d_resp_out,
                           float* d_lafs_out, int* d_oct_out, int* d_lvl_out, int* d_count_out, void* stream) {
    AG_REQUIRE(d_A && d_resp && d_lafs && d_oct && d_lvl && d_count_in && d_resp_out && d_lafs_out && d_oct_out &&
                   d_lvl_out && d_count_out, "NULL argument");
    AG_REQUIRE(B >= 1 && cap >= 1 && out_cap >= 1, "bad sizes");
    int sort_cap = 32;
    while (sort_cap < cap) sort_cap <<= 1;
    const size_t smem = (size_t)sort_cap * sizeof(unsigned long long);
    if (smem > 200 * 1024) {
        set_error("ag_affine_shape_filter: cap %d needs %zu B of shared memory (max 200 KiB)", cap, smem);
        return AG_ERR_CAPACITY;
    }
    static SmemAttrOnce attr_once;
    if (smem > 32 * 1024) {  // static + dynamic must stay under the 48 KiB default
        int rc = attr_once.ensure(shape_filter_kernel, smem, "shape smem attr");
        if (rc != AG_OK) return rc;
    }
    ShapeParams P;
    P.A = d_A; P.resp = d_resp; P.lafs = d_lafs; P.oct = d_oct; P.lvl = d_lvl; P.count_in = d_count_in;
    P.cap = cap; P.num_features = num_features; P.out_cap = out_cap; P.sort_cap = sort_cap;
    P.resp_out = d_resp_out; P.lafs_out = d_lafs_out; P.oct_out = d_oct_out; P.lvl_out = d_lvl_out; P.count_out = d_count_out;
    shape_filter_kernel<<<B, GNT, smem, (cudaStream_t)stream>>>(P);
    AG_CHECK_LAUNCH("shape_filter_kernel");
    return AG_OK;
}

int ag_affine_shape_filter_all(const float* d_A, const float* d_resp, const float* d_lafs, const int* d_oct, const int* d_lvl,
                               const int* d_count_in, int B, int cap, float* d_resp_out, float* d_lafs_out, int* d_oct_out, int* d_lvl_out,
                               int* d_count_out, void* stream) {
    AG_REQUIRE(d_A && d_resp && d_lafs && d_oct && d_lvl && d_count_in && d_resp_out && d_lafs_out && d_oct_out &&
                   d_lvl_out && d_count_out, "NULL argument");
    AG_REQUIRE(B >= 1 && cap >= 1, "bad sizes");
    ShapeParams P;
    P.A = d_A; P.resp = d_resp; P.lafs = d_lafs; P.oct = d_oct; P.lvl = d_lvl; P.count_in = d_count_in;
    P.cap = cap; P.num_features = 0; P.out_cap = cap; P.sort_cap = 0;
    P.resp_out = d_resp_out; P.lafs_out = d_lafs_out; P.oct_out = d_oct_out; P.lvl_out = d_lvl_out; P.count_out = d_count_out;
    shape_filter_all_kernel<<<B, GNT, 0, (cudaStream_t)stream>>>(P);
    AG_CHECK_LAUNCH("shape_filter_all_kernel");
    return AG_OK;
}

size_t ag_affine_shape_filter_topk_workspace_bytes(int B, int cap) {
    if (B < 1 || cap <= TOPK_SMEM_MAX) return 0;
    const size_t nb = B, nc = cap;
    return topk_scratch_bytes(nb, nc) + align_up(nb * nc * sizeof(uint32_t), 256) + align_up(nb * nc, 256) + align_up(nb * sizeof(int), 256);
}

int ag_affine_shape_filter_topk(const float* d_A, const float* d_resp, const float* d_lafs, const int* d_oct, const int* d_lvl,
                                const int* d_count_in, int B, int cap, int num_features, int out_cap, void* d_scratch, size_t scratch_bytes,
                                float* d_resp_out, float* d_lafs_out, int* d_oct_out, int* d_lvl_out, int* d_count_out, void* stream) {
    AG_REQUIRE(d_A && d_resp && d_lafs && d_oct && d_lvl && d_count_in && d_resp_out && d_lafs_out && d_oct_out && d_lvl_out && d_count_out &&
                   (d_scratch || scratch_bytes == 0), "NULL argument");
    AG_REQUIRE(B >= 1 && cap >= 1 && out_cap >= 1, "bad sizes");
    if (cap <= TOPK_SMEM_MAX)   // the shared-memory kernel holds it: bit-identical by construction
        return ag_affine_shape_filter(d_A, d_resp, d_lafs, d_oct, d_lvl, d_count_in, B, cap, num_features, out_cap, d_resp_out, d_lafs_out,
                                      d_oct_out, d_lvl_out, d_count_out, stream);
    const size_t nb = ag_affine_shape_filter_topk_workspace_bytes(B, cap);
    if (scratch_bytes < nb) {
        set_error("ag_affine_shape_filter_topk: scratch of %zu bytes needed, %zu given", nb, scratch_bytes);
        return AG_ERR_CAPACITY;
    }
    TopkBufs T;
    unsigned char* c = topk_carve((unsigned char*)d_scratch, B, cap, T);
    uint32_t* ord = (uint32_t*)c; c += align_up((size_t)B * cap * sizeof(uint32_t), 256);
    unsigned char* keep = c; c += align_up((size_t)B * cap, 256);
    int* surv = (int*)c;
    ShapeParams P;
    P.A = d_A; P.resp = d_resp; P.lafs = d_lafs; P.oct = d_oct; P.lvl = d_lvl; P.count_in = d_count_in;
    P.cap = cap; P.num_features = num_features; P.out_cap = out_cap; P.sort_cap = 0;
    P.resp_out = d_resp_out; P.lafs_out = d_lafs_out; P.oct_out = d_oct_out; P.lvl_out = d_lvl_out; P.count_out = d_count_out;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_cuda(cudaMemsetAsync(surv, 0, (size_t)B * sizeof(int), st), "memset survivor counts");
    if (rc != AG_OK) return rc;
    shape_keys_kernel<<<dim3(cdiv(cap, SK_NT), B), SK_NT, 0, st>>>(P, ord, keep, surv);
    AG_CHECK_LAUNCH("shape_keys_kernel");
    ShapeTopkSrc S;
    S.ord = ord; S.keep = keep; S.surv = surv; S.count_in = d_count_in; S.cap = cap; S.num_features = num_features; S.out_cap = out_cap;
    int need = out_cap < cap ? out_cap : cap;   // the most rows the rule can select
    if (num_features > 0 && num_features < need) need = num_features;
    int fin = 0;
    if ((rc = topk_run(S, T, B, need, st, &fin)) != AG_OK) return rc;
    shape_topk_write_kernel<<<dim3(cdiv(need, SK_NT), B), SK_NT, 0, st>>>(P, T.idx[fin], T.img, T.rows);
    AG_CHECK_LAUNCH("shape_topk_write_kernel");
    return AG_OK;
}

int ag_lafs_apply_rotation(float* d_lafs, const float* d_R, int n, void* stream) {
    AG_REQUIRE(d_lafs && d_R, "NULL argument");
    if (n <= 0) return AG_OK;
    lafs_rotate_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(d_lafs, d_R, n);
    AG_CHECK_LAUNCH("lafs_rotate_kernel");
    return AG_OK;
}

int ag_mat2_compose(const float* d_A, const float* d_B, float* d_out, int n, void* stream) {
    AG_REQUIRE(d_A && d_B && d_out, "NULL argument");
    if (n <= 0) return AG_OK;
    mat2_compose_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(d_A, d_B, d_out, n);
    AG_CHECK_LAUNCH("mat2_compose_kernel");
    return AG_OK;
}

int ag_lafs_left_multiply(const float* d_A, const float* d_lafs, float* d_out, int n, void* stream) {
    AG_REQUIRE(d_A && d_lafs && d_out, "NULL argument");
    if (n <= 0) return AG_OK;
    lafs_left_multiply_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(d_A, d_lafs, d_out, n);
    AG_CHECK_LAUNCH("lafs_left_multiply_kernel");
    return AG_OK;
}

int ag_lafs_scale(const float* d_in, float* d_out, int n, float a_coef, float x_coef, float y_coef, void* stream) {
    AG_REQUIRE(d_in && d_out, "NULL argument");
    if (n <= 0) return AG_OK;
    lafs_scale_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(d_in, d_out, n, a_coef, x_coef, y_coef);
    AG_CHECK_LAUNCH("lafs_scale_kernel");
    return AG_OK;
}

int ag_lafs_to_ell(const float* d_lafs, int n, float* d_ell, void* stream) {
    AG_REQUIRE(d_lafs && d_ell, "NULL argument");
    if (n <= 0) return AG_OK;
    lafs_to_ell_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(d_lafs, d_ell, n);
    AG_CHECK_LAUNCH("lafs_to_ell_kernel");
    return AG_OK;
}

int ag_ells_to_lafs(const float* d_ell, int n, float* d_lafs, void* stream) {
    AG_REQUIRE(d_ell && d_lafs, "NULL argument");
    if (n <= 0) return AG_OK;
    ells_to_lafs_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(d_ell, d_lafs, n);
    AG_CHECK_LAUNCH("ells_to_lafs_kernel");
    return AG_OK;
}

}  // extern "C"
