// Geometric verification of the batched matcher's tentatives (after ag_match_pairs), one CTA per pair:
//   ag_homography_ransac         homography RANSAC (the notebook's ransac_validate: findHomography(src, dst, 2.0, 0.99, 50000))
//   ag_homography_ransac_affine  the same from 2 affine correspondences per sample, with frame-consistent inliers
//   ag_fundamental_ransac        fundamental-matrix RANSAC (the notebook's commented-out findFundamentalMatrix(src, dst, 0.5))
//   ag_fundamental_degensac      the same with DEGENSAC's degeneracy test, plane-and-parallax and local optimisation (pydegensac's family)
//   ag_gt_correspondences_pairs  ReprojectionStuff.get_GT_correspondence_indexes (the reference's "true matches" count), per pair
//   ag_gt_frobenius_pairs / _sets  get_GT_correspondence_indexes_Fro(_and_center): affine-shape ground truth on tentatives or whole sets
//   ag_reproject_lafs            ReprojectionStuff.reprojectLAFs
//
// The RANSACs are deterministic and restated line by line in numpy by tests/oracle_ransac.py, tests/oracle_ac_ransac.py,
// tests/oracle_fransac.py and tests/oracle_degensac.py, so their
// decisions (samples, degeneracy, inlier counts, the stopping point) are reproduced exactly.  For that reason all their arithmetic is
// fp64, with + - * / sqrt only where a decision depends on it, and this file is compiled with
// -fmad=false (build.sh): numpy rounds every product and sum separately, so fused multiply-adds here would move near-threshold decisions.
// The block reductions of the refit run in a fixed order (strided per-thread sums, an xor butterfly per warp, warps in ascending order)
// that the restatement repeats.
//
// Each RANSAC kernel (ransac_kernel, fransac_kernel<DEGEN>, ac_ransac_kernel) keeps its own search loop: sample, solver, scoring over
// the tile, chunk key and stopping rule.  The steps they share are one device function each: verify_pair (the pair's rows, or -1),
// draw_sample (the first K distinct draws), block_max_key (the chunk's winner), hartley (normalisation statistics), denormalise_h /
// denormalise_f, refit_rounds and finish_ransac (the refits and the result).
#include "common.cuh"

namespace ag {

constexpr int VT = 256;              // threads per CTA = hypotheses per chunk: the stopping rule is checked after each chunk
constexpr int VTILE = 2048;          // tentative centres per shared-memory tile (32 KB)
constexpr int MAX_DRAWS = 64;        // draws per hypothesis before it is counted as degenerate (fewer than 4 distinct indices)
constexpr double COLLINEAR_EPS = 1e-6;   // |cross(b - a, c - a)| <= eps * (|dx1| + |dy1|) * (|dx2| + |dy2|): collinear
constexpr int JACOBI_SWEEPS = 10;
constexpr int REFIT_ROUNDS = 3;
constexpr int F_REFIT_MIN = 8;       // inliers needed by the fundamental matrix's 8-point refit
constexpr int MAX_TCAP = 4194240;    // ag_match_pairs' cap1 limit

__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// Index of draw d of hypothesis h in [0, n): splitmix64(splitmix64((h << 32) | d) ^ seed), high 32 bits scaled by n.
__device__ __forceinline__ int draw_index(uint64_t seed, int h, int d, int n) {
    const uint64_t r = splitmix64(splitmix64(((uint64_t)(uint32_t)h << 32) | (uint32_t)d) ^ seed);
    return (int)(((r >> 32) * (uint64_t)(uint32_t)n) >> 32);
}

// The sample of hypothesis h: its first K distinct draws, in draw order.  False when MAX_DRAWS draws give fewer (a degenerate sample).
template <int K>
__device__ __forceinline__ bool draw_sample(uint64_t seed, int h, int n, int (&idx)[K]) {
    int got = 0;
    for (int d = 0; d < MAX_DRAWS && got < K; d++) {
        const int v = draw_index(seed, h, d, n);
        bool dup = false;
        for (int q = 0; q < got; q++) dup |= idx[q] == v;
        if (!dup) idx[got++] = v;
    }
    return got == K;
}

// Pair p = (i, j) -> n tentatives, or -1 when the pair cannot be verified (an image index out of range, ntent outside 0..tcap).
__device__ __forceinline__ int pair_tentatives(const int* __restrict__ pairs, int p, int S1, int S2, const int* __restrict__ ntent, int tcap,
                                               int& i, int& j) {
    i = pairs ? pairs[2 * (size_t)p] : p;
    j = pairs ? pairs[2 * (size_t)p + 1] : p;
    const int n = ntent[p];
    if (i < 0 || i >= S1 || j < 0 || j >= S2 || n < 0 || n > tcap) return -1;
    return n;
}

// Block-wide over NT threads: true when every tentative row of the pair indexes a row inside its set's cap (nothing is read otherwise).
template <int NT = VT>
__device__ bool rows_in_range(const int* __restrict__ tent, int n, int cap1, int cap2) {
    bool bad = false;
    for (int t = threadIdx.x; t < n; t += NT) {
        const int r1 = tent[2 * (size_t)t], r2 = tent[2 * (size_t)t + 1];
        bad |= r1 < 0 || r1 >= cap1 || r2 < 0 || r2 >= cap2;
    }
    return !__syncthreads_or(bad);
}

// Pair blockIdx.x of a one-CTA-per-pair kernel: its n tentatives `tent` and the LAF sets L1, L2 they index.  False, after thread 0
// has written -1 to flag[pair], when the pair cannot be verified (pair_tentatives, rows_in_range).  Block-wide.
__device__ __forceinline__ bool verify_pair(const float* __restrict__ lafs1, int S1, int cap1, const float* __restrict__ lafs2, int S2,
                                           int cap2, const int* __restrict__ pairs, const int* __restrict__ tent_all,
                                           const int* __restrict__ ntent, int tcap, int* __restrict__ flag, int& n, const int*& tent,
                                           const float*& L1, const float*& L2) {
    const int p = blockIdx.x;
    int i, j;
    n = pair_tentatives(pairs, p, S1, S2, ntent, tcap, i, j);
    tent = tent_all + (size_t)p * tcap * 2;
    if (n < 0 || !rows_in_range(tent, n, cap1, cap2)) {
        if (threadIdx.x == 0) flag[p] = -1;
        return false;
    }
    L1 = lafs1 + (size_t)i * cap1 * 6;
    L2 = lafs2 + (size_t)j * cap2 * 6;
    return true;
}

// Ordered compaction of one block of VT rows: every thread whose row t is kept writes t to out[base + run + its rank among the kept
// rows]; returns run plus the block's count.  Block-wide; wsum is VT / 32 shared ints, free again on return.
__device__ __forceinline__ int compact_rows(bool keep, int t, int* __restrict__ out, size_t base, int run, int* wsum) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned b = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) wsum[warp] = __popc(b);
    __syncthreads();
    int off = run, tot = 0;
#pragma unroll
    for (int w = 0; w < VT / 32; w++) {
        off += w < warp ? wsum[w] : 0;
        tot += wsum[w];
    }
    if (keep) out[base + off + __popc(b & ((1u << lane) - 1u))] = t;
    __syncthreads();   // wsum is rewritten by the next row block
    return run + tot;
}

// Centres of tentative t: (x1, y1) in image 1, (x2, y2) in image 2 (the LAF's third column).
__device__ __forceinline__ float4 tent_centres(const float* __restrict__ L1, const float* __restrict__ L2, const int* __restrict__ tent, int t) {
    const float* a = L1 + (size_t)tent[2 * (size_t)t] * 6;
    const float* b = L2 + (size_t)tent[2 * (size_t)t + 1] * 6;
    return make_float4(a[2], a[5], b[2], b[5]);
}

// Tentative t as an affine correspondence: its centres c (as tent_centres) and the 2x2 parts (a00, a01, a10, a11) of both frames.
struct AcRow {
    float4 c, a1, a2;
};
__device__ __forceinline__ AcRow tent_ac(const float* __restrict__ L1, const float* __restrict__ L2, const int* __restrict__ tent, int t) {
    const float* a = L1 + (size_t)tent[2 * (size_t)t] * 6;
    const float* b = L2 + (size_t)tent[2 * (size_t)t + 1] * 6;
    return {make_float4(a[2], a[5], b[2], b[5]), make_float4(a[0], a[1], a[3], a[4]), make_float4(b[0], b[1], b[3], b[4])};
}

__device__ __forceinline__ bool finite4(float4 c) { return isfinite(c.x) && isfinite(c.y) && isfinite(c.z) && isfinite(c.w); }

// ---- fp64 3x3 helpers (row-major), in the restatement's operation order ------------------------------------------------------------
__device__ __forceinline__ void adj3(const double* m, double* o) {
    o[0] = m[4] * m[8] - m[5] * m[7]; o[1] = m[2] * m[7] - m[1] * m[8]; o[2] = m[1] * m[5] - m[2] * m[4];
    o[3] = m[5] * m[6] - m[3] * m[8]; o[4] = m[0] * m[8] - m[2] * m[6]; o[5] = m[2] * m[3] - m[0] * m[5];
    o[6] = m[3] * m[7] - m[4] * m[6]; o[7] = m[1] * m[6] - m[0] * m[7]; o[8] = m[0] * m[4] - m[1] * m[3];
}
__device__ __forceinline__ void mul3(const double* a, const double* b, double* o) {
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) o[3 * r + c] = a[3 * r] * b[c] + a[3 * r + 1] * b[3 + c] + a[3 * r + 2] * b[6 + c];
}
// H /= H[2][2]; false when that is zero or the result is not finite.
__device__ __forceinline__ bool normalise_h(double* H) {
    const double s = H[8];
    bool ok = s != 0.0;
#pragma unroll
    for (int k = 0; k < 9; k++) {
        H[k] = H[k] / s;
        ok &= isfinite(H[k]);
    }
    return ok;
}

// Hartley normalisation x -> T x, T = [s 0 -s cx; 0 s -s cy; 0 0 1], of both images.
struct Hartley {
    double c1x, c1y, s1, c2x, c2y, s2;
};

// H = T2^-1 Hn T1, normalised by normalise_h.
__device__ __forceinline__ bool denormalise_h(const Hartley& T, const double* Hn, double* H) {
    const double T1[9] = {T.s1, 0.0, -(T.s1 * T.c1x), 0.0, T.s1, -(T.s1 * T.c1y), 0.0, 0.0, 1.0};
    const double T2i[9] = {1.0 / T.s2, 0.0, T.c2x, 0.0, 1.0 / T.s2, T.c2y, 0.0, 0.0, 1.0};
    double tmp[9];
    mul3(T2i, Hn, tmp);
    mul3(tmp, T1, H);
    return normalise_h(H);
}

// Inlier test: positive denominator and squared forward error <= th2.
__device__ __forceinline__ bool is_inlier(const double* H, float4 c, double th2) {
    const double x = c.x, y = c.y;
    const double w = H[6] * x + H[7] * y + H[8];
    if (!(w > 0.0)) return false;
    const double u = (H[0] * x + H[1] * y + H[2]) / w - (double)c.z;
    const double v = (H[3] * x + H[4] * y + H[5]) / w - (double)c.w;
    return u * u + v * v <= th2;
}

__device__ __forceinline__ double cross3(double ax, double ay, double bx, double by, double cx, double cy, bool& collinear) {
    const double dx1 = bx - ax, dy1 = by - ay, dx2 = cx - ax, dy2 = cy - ay;
    const double cr = dx1 * dy2 - dx2 * dy1;
    collinear |= fabs(cr) <= COLLINEAR_EPS * ((fabs(dx1) + fabs(dy1)) * (fabs(dx2) + fabs(dy2)));
    return cr;
}

// Basis map of 4 points: M = [p0 p1 p2] diag(adj([p0 p1 p2]) p3), p = (x, y, 1).
__device__ __forceinline__ void basis_map(const double* x, const double* y, double* M) {
    const double P[9] = {x[0], x[1], x[2], y[0], y[1], y[2], 1.0, 1.0, 1.0};
    double A[9];
    adj3(P, A);
    double l[3];
#pragma unroll
    for (int r = 0; r < 3; r++) l[r] = A[3 * r] * x[3] + A[3 * r + 1] * y[3] + A[3 * r + 2];
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
        for (int c = 0; c < 3; c++) M[3 * r + c] = P[3 * r + c] * l[c];
}

// Hypothesis from 4 correspondences; false for a degenerate sample (collinear triplet in either image, a mixed orientation of the four
// triplets between the images, or H[2][2] zero / non-finite).
__device__ bool minimal_homography(const float4 (&c)[4], double* H) {
    double x1[4], y1[4], x2[4], y2[4];
#pragma unroll
    for (int k = 0; k < 4; k++) { x1[k] = c[k].x; y1[k] = c[k].y; x2[k] = c[k].z; y2[k] = c[k].w; }
    constexpr int tt[4][3] = {{0, 1, 2}, {1, 2, 3}, {0, 2, 3}, {0, 1, 3}};
    bool col = false;
    int neg = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int a = tt[k][0], b = tt[k][1], d = tt[k][2];
        const double c1 = cross3(x1[a], y1[a], x1[b], y1[b], x1[d], y1[d], col);
        const double c2 = cross3(x2[a], y2[a], x2[b], y2[b], x2[d], y2[d], col);
        neg += (c1 * c2 < 0.0) ? 1 : 0;
    }
    if (col || (neg != 0 && neg != 4)) return false;
    double M1[9], M2[9], A1[9];
    basis_map(x1, y1, M1);
    basis_map(x2, y2, M2);
    adj3(M1, A1);
    mul3(M2, A1, H);
    return normalise_h(H);
}

// Sum of K doubles over the block in the fixed order described at the top, into out[0..K) (shared), valid for every thread on return.
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double (*red)[K], double* out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; k++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] = v[k] + __shfl_xor_sync(0xffffffffu, v[k], o);
    }
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < K; k++) red[warp][k] = v[k];
    __syncthreads();
    if (threadIdx.x < K) {
        double s = red[0][threadIdx.x];
        for (int w = 1; w < VT / 32; w++) s = s + red[w][threadIdx.x];
        out[threadIdx.x] = s;
    }
    __syncthreads();
}

// The largest of the threads' keys (0: none), valid for every thread: an xor butterfly per warp, one key per warp in red (VT / 32
// shared entries), a barrier, then the maximum over the warps.  red may be written again only after the caller's next barrier.
__device__ __forceinline__ unsigned long long block_max_key(unsigned long long key, unsigned long long* red) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long k2 = __shfl_xor_sync(0xffffffffu, key, o);
        key = k2 > key ? k2 : key;
    }
    if (lane == 0) red[warp] = key;
    __syncthreads();
    unsigned long long bk = 0;
#pragma unroll
    for (int w = 0; w < VT / 32; w++) bk = red[w] > bk ? red[w] : bk;
    return bk;
}

struct RansacShared {
    float4 tile[VTILE];
    double H[9], Hr[9];
    double red[VT / 32][45];
    double sums[45];
    double A[81], V[81];
    unsigned long long key[VT / 32];
    int count[VT / 32];
    int bad;
};

// Jacobi rotation (p, q) of the symmetric N x N A (row-major), accumulated into V, for row / column k: the column step, then (after
// the caller's barrier) the row step.  Each element is one rounded product pair, in the restatement's order.
struct JacobiRot {
    double cs, sn;
    bool skip;
};
__device__ __forceinline__ JacobiRot jacobi_rot(double app, double aqq, double apq) {
    if (apq == 0.0) return {1.0, 0.0, true};
    const double theta = (aqq - app) / (2.0 * apq);
    const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
    const double cs = 1.0 / sqrt(t * t + 1.0);
    return {cs, t * cs, false};
}
template <int N>
__device__ __forceinline__ void jacobi_cols(double* A, int p, int q, int k, JacobiRot r) {
    const double akp = A[N * k + p], akq = A[N * k + q];
    A[N * k + p] = r.cs * akp - r.sn * akq;
    A[N * k + q] = r.sn * akp + r.cs * akq;
}
template <int N>
__device__ __forceinline__ void jacobi_rows(double* A, double* V, int p, int q, int k, JacobiRot r) {
    const double apk = A[N * p + k], aqk = A[N * q + k];
    A[N * p + k] = r.cs * apk - r.sn * aqk;
    A[N * q + k] = r.sn * apk + r.cs * aqk;
    const double vkp = V[N * k + p], vkq = V[N * k + q];
    V[N * k + p] = r.cs * vkp - r.sn * vkq;
    V[N * k + q] = r.sn * vkp + r.cs * vkq;
}

// Cyclic Jacobi of the symmetric 9x9 s.A with s.V = I, on warp 0 (lane k < 9 owns row / column k): JACOBI_SWEEPS sweeps of the pairs
// (p, q), p < q, in row order.  Block-wide; on return s.A is (nearly) diagonal and s.V holds the eigenvectors in its columns.
__device__ void jacobi9_warp(double* A, double* V) {
    if (threadIdx.x < 32) {
        const int k = threadIdx.x;
        for (int sweep = 0; sweep < JACOBI_SWEEPS; sweep++)
            for (int p = 0; p < 8; p++)
                for (int q = p + 1; q < 9; q++) {
                    const JacobiRot r = jacobi_rot(A[9 * p + p], A[9 * q + q], A[9 * p + q]);
                    __syncwarp();
                    if (r.skip) continue;
                    if (k < 9) jacobi_cols<9>(A, p, q, k, r);
                    __syncwarp();
                    if (k < 9) jacobi_rows<9>(A, V, p, q, k, r);
                    __syncwarp();
                }
    }
    __syncthreads();
}

// The same sweeps on one thread, for a 3x3.
__device__ __forceinline__ void jacobi3(double* A, double* V) {
    for (int sweep = 0; sweep < JACOBI_SWEEPS; sweep++)
        for (int p = 0; p < 2; p++)
            for (int q = p + 1; q < 3; q++) {
                const JacobiRot r = jacobi_rot(A[3 * p + p], A[3 * q + q], A[3 * p + q]);
                if (r.skip) continue;
                for (int k = 0; k < 3; k++) jacobi_cols<3>(A, p, q, k, r);
                for (int k = 0; k < 3; k++) jacobi_rows<3>(A, V, p, q, k, r);
            }
}

// Index of the smallest diagonal entry (the lowest on ties).
template <int N>
__device__ __forceinline__ int smallest_diag(const double* A) {
    int m = 0;
    for (int e = 1; e < N; e++)
        if (A[N * e + e] < A[N * m + m]) m = e;
    return m;
}

// v = the eigenvector of the smallest eigenvalue of the symmetric 3x3 G (jacobi3, which overwrites G).
__device__ __forceinline__ void smallest_eigvec3(double* G, double (&v)[3]) {
    double V[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0};
    jacobi3(G, V);
    const int m = smallest_diag<3>(G);
    v[0] = V[m]; v[1] = V[3 + m]; v[2] = V[6 + m];
}

// s.A = the symmetric 9x9 whose upper triangle is s.sums (row by row), s.V = I, then jacobi9_warp.  Block-wide.
__device__ void normal_matrix_eigen(RansacShared& s) {
    if (threadIdx.x < 81) {
        const int r = threadIdx.x / 9, c = threadIdx.x % 9, lo = min(r, c), hi = max(r, c);
        s.A[threadIdx.x] = s.sums[lo * 9 - lo * (lo - 1) / 2 + (hi - lo)];
        s.V[threadIdx.x] = r == c ? 1.0 : 0.0;
    }
    __syncthreads();
    jacobi9_warp(s.A, s.V);
}

__device__ __forceinline__ bool is_inlier_f(const double* F, float4 c, double th2);
__device__ __forceinline__ bool is_inlier_ac(const double* H, const double* G, const AcRow& r, double th2, double laf_th);

// Inliers of H (a homography, or a fundamental matrix when FUND; with AFF a homography whose inliers must also pass the frame test at
// laf_th) over all n tentatives (thread t handles rows t, t + VT, ...); writes the mask when `inl` is not NULL.  Block total.
template <bool FUND = false, bool AFF = false>
__device__ int score_rows(const double* H, const float* L1, const float* L2, const int* tent, int n, double th2, unsigned char* inl,
                          RansacShared& s, double laf_th = 0.0) {
    double G[9];
    if (AFF) adj3(H, G);
    int cnt = 0;
    for (int t = threadIdx.x; t < n; t += VT) {
        bool in;
        if (AFF) in = is_inlier_ac(H, G, tent_ac(L1, L2, tent, t), th2, laf_th);
        else {
            const float4 c = tent_centres(L1, L2, tent, t);
            in = FUND ? is_inlier_f(H, c, th2) : is_inlier(H, c, th2);
        }
        cnt += in;
        if (inl) inl[t] = in;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) s.count[warp] = cnt;
    __syncthreads();
    int tot = 0;
#pragma unroll
    for (int w = 0; w < VT / 32; w++) tot += s.count[w];
    __syncthreads();
    return tot;
}

// Hartley normalisation of the rows in the mask `inl`, or, without a mask, of the rows whose four coordinates are finite: per image
// the centroid c and s = sqrt(2 / var), var the mean squared distance to c.  The sums of x, y, x^2, y^2 per image and the row count
// (exact: at most MAX_TCAP) go through one block_sum, which reduces each of them on its own; the count into *nrows when given.
// Block-wide; false, on every thread, unless var > 0 in both images.
__device__ __forceinline__ bool hartley(const float* L1, const float* L2, const int* tent, int n, const unsigned char* inl, RansacShared& s,
                                        Hartley& T, double* nrows = nullptr) {
    double st[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int t = threadIdx.x; t < n; t += VT) {
        const float4 c = tent_centres(L1, L2, tent, t);
        const bool in = inl ? inl[t] != 0 : finite4(c);
        const double x1 = in ? (double)c.x : 0.0, y1 = in ? (double)c.y : 0.0, x2 = in ? (double)c.z : 0.0, y2 = in ? (double)c.w : 0.0;
        st[0] = st[0] + x1; st[1] = st[1] + y1; st[2] = st[2] + x1 * x1; st[3] = st[3] + y1 * y1;
        st[4] = st[4] + x2; st[5] = st[5] + y2; st[6] = st[6] + x2 * x2; st[7] = st[7] + y2 * y2;
        st[8] = st[8] + (in ? 1.0 : 0.0);
    }
    block_sum<9>(st, reinterpret_cast<double(*)[9]>(&s.red[0][0]), s.sums);
    const double nd = s.sums[8];
    if (nrows) *nrows = nd;
    T.c1x = s.sums[0] / nd; T.c1y = s.sums[1] / nd; T.c2x = s.sums[4] / nd; T.c2y = s.sums[5] / nd;
    const double var1 = (s.sums[2] + s.sums[3]) / nd - (T.c1x * T.c1x + T.c1y * T.c1y);
    const double var2 = (s.sums[6] + s.sums[7]) / nd - (T.c2x * T.c2x + T.c2y * T.c2y);
    T.s1 = sqrt(2.0 / var1);
    T.s2 = sqrt(2.0 / var2);
    return var1 > 0.0 && var2 > 0.0;
}

// Normalised-DLT least squares on the rows of the mask `inl` (Hartley normalisation, 9x9 normal matrix, smallest eigenvector by
// cyclic Jacobi on warp 0).  Writes s.Hr; false when the inliers do not determine a finite homography.
__device__ bool refit(const float* L1, const float* L2, const int* tent, int n, const unsigned char* inl, RansacShared& s) {
    Hartley T;
    if (!hartley(L1, L2, tent, n, inl, s, T)) return false;   // uniform across the block: every thread returns
    // normal matrix: upper triangle, row by row
    double nm[45];
#pragma unroll
    for (int k = 0; k < 45; k++) nm[k] = 0.0;
    for (int t = threadIdx.x; t < n; t += VT) {
        const float4 c = tent_centres(L1, L2, tent, t);
        const bool in = inl[t];
        const double u = (c.x - T.c1x) * T.s1, v = (c.y - T.c1y) * T.s1, up = (c.z - T.c2x) * T.s2, vp = (c.w - T.c2y) * T.s2;
        const double a1[9] = {-u, -v, -1.0, 0.0, 0.0, 0.0, up * u, up * v, up};
        const double a2[9] = {0.0, 0.0, 0.0, -u, -v, -1.0, vp * u, vp * v, vp};
        int e = 0;
#pragma unroll
        for (int k = 0; k < 9; k++)
#pragma unroll
            for (int l = k; l < 9; l++, e++) nm[e] = nm[e] + (in ? a1[k] * a1[l] + a2[k] * a2[l] : 0.0);
    }
    block_sum<45>(nm, s.red, s.sums);
    normal_matrix_eigen(s);
    if (threadIdx.x == 0) {
        const int m = smallest_diag<9>(s.A);
        double Hn[9];
        for (int e = 0; e < 9; e++) Hn[e] = s.V[9 * e + m];
        s.bad = !denormalise_h(T, Hn, s.Hr);
    }
    __syncthreads();
    return !s.bad;
}

__device__ bool refit_f(const float* L1, const float* L2, const int* tent, int n, const unsigned char* inl, RansacShared& s);

// Up to REFIT_ROUNDS least-squares refits of the model M (shared; a homography, or a fundamental matrix when FUND) on its inliers at
// th2, each kept only if the inlier count does not drop: the rounds that end every RANSAC kernel, for DEGENSAC's plane H and its local
// optimisation, and (AFF: the inliers also pass the frame test at laf_th; the refit is the same point DLT) for the affine homography
// RANSAC's.  Block-wide; on return M is the last kept model and `inl` its mask (rows < n).
// Returns its inlier count.
template <bool FUND, bool AFF = false>
__device__ __forceinline__ int refit_rounds(const float* L1, const float* L2, const int* tent, int n, double th2, unsigned char* inl,
                                            double* M, RansacShared& s, double laf_th = 0.0) {
    int cnt = score_rows<FUND, AFF>(M, L1, L2, tent, n, th2, inl, s, laf_th);
    for (int r = 0; r < REFIT_ROUNDS && cnt >= (FUND ? F_REFIT_MIN : 4); r++) {
        if (!(FUND ? refit_f(L1, L2, tent, n, inl, s) : refit(L1, L2, tent, n, inl, s))) break;
        const int c2 = score_rows<FUND, AFF>(s.Hr, L1, L2, tent, n, th2, nullptr, s, laf_th);
        if (c2 < cnt) break;
        cnt = c2;
        if (threadIdx.x < 9) M[threadIdx.x] = s.Hr[threadIdx.x];
        __syncthreads();
        score_rows<FUND, AFF>(M, L1, L2, tent, n, th2, inl, s, laf_th);
    }
    return cnt;
}

// The end of a RANSAC kernel for pair blockIdx.x: the refit rounds on the search's winner s.H when it has `best` > 0 inliers (else an
// all-zero mask), then the model (zero when nothing was found), its inlier count and the number of hypotheses evaluated.  Block-wide.
template <bool FUND, bool AFF = false>
__device__ __forceinline__ void finish_ransac(const float* L1, const float* L2, const int* tent, int n, double th2, int best, int h_done,
                                              unsigned char* inl, RansacShared& s, float* __restrict__ Mout, int* __restrict__ ninl,
                                              int* __restrict__ iters, double laf_th = 0.0) {
    const int p = blockIdx.x, tid = threadIdx.x;
    if (best > 0) best = refit_rounds<FUND, AFF>(L1, L2, tent, n, th2, inl, s.H, s, laf_th);
    else
        for (int t = tid; t < n; t += VT) inl[t] = 0;
    if (tid < 9) Mout[(size_t)p * 9 + tid] = best > 0 ? (float)s.H[tid] : 0.f;
    if (tid == 0) {
        ninl[p] = best;
        if (iters) iters[p] = h_done;
    }
}

__global__ void __launch_bounds__(VT) ransac_kernel(const float* __restrict__ lafs1, int S1, int cap1, const float* __restrict__ lafs2, int S2,
                                                    int cap2, const int* __restrict__ pairs, const int* __restrict__ tent_all,
                                                    const int* __restrict__ ntent, int tcap, double th2, double log1mconf, int max_iters,
                                                    uint64_t seed, float* __restrict__ Hout, unsigned char* __restrict__ inl_all,
                                                    int* __restrict__ ninl, int* __restrict__ iters) {
    __shared__ RansacShared s;
    const int tid = threadIdx.x;
    const int* tent;
    const float *L1, *L2;
    int n;
    if (!verify_pair(lafs1, S1, cap1, lafs2, S2, cap2, pairs, tent_all, ntent, tcap, ninl, n, tent, L1, L2)) return;
    unsigned char* inl = inl_all + (size_t)blockIdx.x * tcap;
    int best = 0, h_done = 0;
    if (n >= 4) {
        const int ntiles = (n + VTILE - 1) / VTILE;
        for (int h0 = 0;; h0 += VT) {
            const int h = h0 + tid;
            double H[9];
            int idx[4];
            bool ok = h < max_iters && draw_sample(seed, h, n, idx);
            if (ok) {
                float4 c[4];
#pragma unroll
                for (int q = 0; q < 4; q++) c[q] = tent_centres(L1, L2, tent, idx[q]);
                ok = minimal_homography(c, H);
            }
            int cnt = 0;
            for (int tb = 0; tb < ntiles; tb++) {
                const int t0 = tb * VTILE, m = min(VTILE, n - t0);
                if (ntiles > 1 || h0 == 0) {
                    __syncthreads();
                    for (int t = tid; t < m; t += VT) s.tile[t] = tent_centres(L1, L2, tent, t0 + t);
                    __syncthreads();
                }
                if (ok)
                    for (int t = 0; t < m; t++) cnt += is_inlier(H, s.tile[t], th2);
            }
            // best of the chunk: highest count, then lowest h
            const unsigned long long mine = ok ? ((unsigned long long)cnt << 32) | (unsigned)~(unsigned)h : 0ull;
            const unsigned long long bk = block_max_key(mine, s.key);
            const int bc = (int)(bk >> 32);
            if (bk != 0 && bc > best) {
                if (mine == bk) {
#pragma unroll
                    for (int k = 0; k < 9; k++) s.H[k] = H[k];
                }
                best = bc;
            }
            h_done = min(h0 + VT, max_iters);
            double need;   // adaptive number of hypotheses for `confidence`
            const double pr = (double)best / (double)n, p4 = pr * pr * pr * pr;
            if (p4 >= 1.0) need = 0.0;
            else if (p4 <= 0.0) need = INFINITY;
            else need = ceil(log1mconf / log(1.0 - p4));
            __syncthreads();
            if ((double)h_done >= fmin(need, (double)max_iters)) break;
        }
    }
    finish_ransac<false>(L1, L2, tent, n, th2, best, h_done, inl, s, Hout, ninl, iters);
}

// ---- ground-truth check (ReprojectionStuff.py:126-137) ----------------------------------------------------------------------------
constexpr int GT_TILE = 2048;

// H1to2^-1 = adj(H) / det(H) of the fp32 H, in fp64.
__device__ __forceinline__ void inverse_h(const float* __restrict__ H1to2, double* Hi) {
    double H[9], A[9];
    for (int k = 0; k < 9; k++) H[k] = H1to2[k];
    adj3(H, A);
    const double det = H[0] * A[0] + H[1] * A[3] + H[2] * A[6];
    for (int k = 0; k < 9; k++) Hi[k] = A[k] / det;
}

// Distance between the centre (ax, ay), na = |a|^2, and q = (x, y, |p|^2, -): sqrt(|(|p|^2 + |a|^2) - 2 a.p + 1e-12|), the rounding
// steps of ReprojectionStuff.distance_matrix_vector.
__device__ __forceinline__ float centre_dist(float ax, float ay, float na, float4 q) {
    const float dot = __fmaf_rn(ay, q.y, __fmul_rn(ax, q.x));
    return sqrtf(fabsf(__fadd_rn(__fsub_rn(__fadd_rn(q.z, na), __fmul_rn(2.f, dot)), 1e-12f)));
}

__global__ void __launch_bounds__(VT) gt_kernel(const float* __restrict__ lafs1, int S1, int cap1, const float* __restrict__ lafs2, int S2,
                                                int cap2, const int* __restrict__ pairs, const int* __restrict__ tent_all,
                                                const int* __restrict__ ntent, int tcap, const float* __restrict__ H1to2, float th,
                                                float* __restrict__ min_dist, int* __restrict__ idx2, int* __restrict__ true_all,
                                                int* __restrict__ ntrue) {
    __shared__ float4 tile[GT_TILE];   // (x, y, |x|^2, -) of the image-2 centres mapped into image 1
    __shared__ double Hi[9];
    __shared__ int wsum[VT / 32];
    const int p = blockIdx.x, tid = threadIdx.x;
    const int* tent;
    const float *L1, *L2;
    int n;
    if (!verify_pair(lafs1, S1, cap1, lafs2, S2, cap2, pairs, tent_all, ntent, tcap, ntrue, n, tent, L1, L2)) return;
    if (tid == 0) inverse_h(H1to2 + (size_t)p * 9, Hi);
    __syncthreads();
    const size_t base = (size_t)p * tcap;
    int run = 0;
    for (int r0 = 0; r0 < n; r0 += VT) {
        const int t = r0 + tid;
        float ax = 0.f, ay = 0.f, na = 0.f, best = INFINITY;
        int bi = 0;
        if (t < n) {
            const float4 c = tent_centres(L1, L2, tent, t);
            ax = c.x; ay = c.y;
            na = __fadd_rn(__fmul_rn(ax, ax), __fmul_rn(ay, ay));
        }
        for (int u0 = 0; u0 < n; u0 += GT_TILE) {
            const int m = min(GT_TILE, n - u0);
            __syncthreads();
            for (int u = tid; u < m; u += VT) {
                const float4 c = tent_centres(L1, L2, tent, u0 + u);
                const double x = c.z, y = c.w, w = Hi[6] * x + Hi[7] * y + Hi[8];
                const float px = (float)((Hi[0] * x + Hi[1] * y + Hi[2]) / w), py = (float)((Hi[3] * x + Hi[4] * y + Hi[5]) / w);
                tile[u] = make_float4(px, py, __fadd_rn(__fmul_rn(px, px), __fmul_rn(py, py)), 0.f);
            }
            __syncthreads();
            if (t < n)
                for (int u = 0; u < m; u++) {
                    const float v = centre_dist(ax, ay, na, tile[u]);
                    if (v < best) { best = v; bi = u0 + u; }   // ascending u: the lowest index among the minima
                }
        }
        const bool keep = t < n && best <= th;
        if (t < n) { min_dist[base + t] = best; idx2[base + t] = bi; }
        run = compact_rows(keep, t, true_all, base, run, wsum);
    }
    if (tid == 0) ntrue[p] = run;
}

// ---- Frobenius ground truth (ReprojectionStuff.py:139-203): affine-shape consistency of every row of side 1 against side 2 ----------
// Per-row and per-column operands are derived in fp64 from the fp32 LAFs and rounded once to fp32; the (row, column) loop is fp32 in
// the order below, and tests/frobenius_restated.py restates all of it.  CUDA cores only: the loop ends in a min / argmin and a
// threshold decision, so a reduced-precision product would move rows across the threshold and change which column wins.
constexpr int FRO_NT = 64;       // side-1 rows per CTA, one per thread: many CTAs per pair, so one large pair still fills the GPU
constexpr int FRO_TILE = 512;    // side-2 columns per shared-memory tile (18 KB): 12 CTAs per SM

// s = sqrt|det A| in fp64, rounded once; with up_is_up the 2x2 part becomes rectify_up_is_up(A / s) * s in fp32 (LAF.py:285-291,
// ReprojectionStuff.py:162-169).  s is that of A as given.
__device__ __forceinline__ float frame_2x2(float (&a)[4], bool up_is_up) {
    const float s = (float)sqrt(fabs((double)a[0] * a[3] - (double)a[1] * a[2]));
    if (up_is_up) {
        float r[4];
        rectify_up_is_up(__fdiv_rn(a[0], s), __fdiv_rn(a[1], s), __fdiv_rn(a[2], s), __fdiv_rn(a[3], s), r);
        for (int k = 0; k < 4; k++) a[k] = __fmul_rn(r[k], s);
    }
    return s;
}

// reprojectLAFs (ReprojectionStuff.py:9-40) of the LAF l = [[a00, a01, x], [a10, a11, y]] through G, in fp64: the centre
// (u, v, w) = G (x, y, 1) / w and the 2x2 part linH(G, x, y) A; A' (row-major) and t' rounded once.
// linH (ReprojectionStuff.py:9-21): the Jacobian j (row-major) of x -> G x at (x, y), with (n1, n2, w) = G (x, y, 1).  It does not
// depend on G's scale.
__device__ __forceinline__ void lin_h(const double* G, double x, double y, double (&j)[4], double& n1, double& n2, double& w) {
    w = G[6] * x + G[7] * y + G[8];
    n1 = G[0] * x + G[1] * y + G[2];
    n2 = G[3] * x + G[4] * y + G[5];
    const double q1 = n1 / (w * w), q2 = n2 / (w * w);
    j[0] = G[0] / w - q1 * G[6]; j[1] = G[1] / w - q1 * G[7]; j[2] = G[3] / w - q2 * G[6]; j[3] = G[4] / w - q2 * G[7];
}

__device__ __forceinline__ void reproject_laf(const double* G, const float* __restrict__ l, float (&A)[4], float (&t)[2]) {
    double j[4], n1, n2, w;
    lin_h(G, l[2], l[5], j, n1, n2, w);
    const double j00 = j[0], j01 = j[1], j10 = j[2], j11 = j[3];
    const double a00 = l[0], a01 = l[1], a10 = l[3], a11 = l[4];
    A[0] = (float)(j00 * a00 + j01 * a10); A[1] = (float)(j00 * a01 + j01 * a11);
    A[2] = (float)(j10 * a00 + j11 * a10); A[3] = (float)(j10 * a01 + j11 * a11);
    t[0] = (float)(n1 / w); t[1] = (float)(n2 / w);
}

// Row i of side 1.  inv_to_eye: m = (B, c) with B = A^-1 and c = -B t (fp64 from A's fp64 inverse), all NaN when the frame is
// non-finite or singular (det == 0) or B, c do not fit fp32, so none of the row's distances is below anything.  Otherwise m is the
// LHF's entries (a00, a01, tx, a10, a11, ty) and nl its squared norm (the LHF's 9 entries, or the 2x2 part's 4 with skip_center).
struct FroRow {
    float m[6], nl, x, y, na, s1e;
};

__device__ __forceinline__ void frob_row(const float* __restrict__ l, const ag_frobenius_params_t& prm, FroRow& r) {
    float a[4] = {l[0], l[1], l[3], l[4]};
    const float s = frame_2x2(a, prm.do_up_is_up != 0);
    r.x = l[2]; r.y = l[5];
    r.na = __fadd_rn(__fmul_rn(r.x, r.x), __fmul_rn(r.y, r.y));
    r.s1e = __fadd_rn(s, 1e-12f);
    r.nl = 0.f;
    if (prm.inv_to_eye) {
        const double det = (double)a[0] * a[3] - (double)a[1] * a[2];
        const double b0 = a[3] / det, b1 = -(double)a[1] / det, b2 = -(double)a[2] / det, b3 = a[0] / det;
        const double tx = r.x, ty = r.y;
        r.m[0] = (float)b0; r.m[1] = (float)b1; r.m[2] = (float)b2; r.m[3] = (float)b3;
        r.m[4] = (float)(-(b0 * tx + b1 * ty)); r.m[5] = (float)(-(b2 * tx + b3 * ty));
        bool ok = det != 0.0;
        for (int k = 0; k < 4; k++) ok &= isfinite(a[k]);
        for (int k = 0; k < 6; k++) ok &= isfinite(r.m[k]);
        if (!ok)
            for (int k = 0; k < 6; k++) r.m[k] = __int_as_float(0x7fc00000);
    } else {
        r.m[0] = a[0]; r.m[1] = a[1]; r.m[2] = r.x; r.m[3] = a[2]; r.m[4] = a[3]; r.m[5] = r.y;
        double q = (double)a[0] * a[0] + (double)a[1] * a[1] + (double)a[2] * a[2] + (double)a[3] * a[3];
        if (!prm.skip_center) q = q + (double)r.x * r.x + (double)r.y * r.y + 1.0;
        r.nl = (float)q;
    }
}

// Column j of side 2 mapped into image 1 -> tile entries: ta = A' (rectified with up_is_up), tt = (x', y', |t'|^2, s'), tn = |LHF'|^2
// (only read when inv_to_eye is 0).
__device__ __forceinline__ void frob_col(const double* G, const float* __restrict__ l, const ag_frobenius_params_t& prm, float4& ta, float4& tt,
                                         float& tn) {
    float A[4], t[2];
    reproject_laf(G, l, A, t);
    const float s = frame_2x2(A, prm.do_up_is_up != 0);
    ta = make_float4(A[0], A[1], A[2], A[3]);
    tt = make_float4(t[0], t[1], __fadd_rn(__fmul_rn(t[0], t[0]), __fmul_rn(t[1], t[1])), s);
    double q = (double)A[0] * A[0] + (double)A[1] * A[1] + (double)A[2] * A[2] + (double)A[3] * A[3];
    if (!prm.skip_center) q = q + (double)t[0] * t[0] + (double)t[1] * t[1] + 1.0;
    tn = (float)q;
}

__device__ __forceinline__ float dot2f(float a, float b, float c, float d) { return __fadd_rn(__fmul_rn(a, b), __fmul_rn(c, d)); }
__device__ __forceinline__ float sqf(float a) { return __fmul_rn(a, a); }

// One row against m columns of a tile.  The distance D, in this order of fp32 operations:
//   INV:  M = B A' (each entry fl(fl(b a) + fl(b a))), D = ((fl(M00 - 1)^2 + M01^2) + M10^2) + fl(M11 - 1)^2, and without SKIP
//         D = D + (r0^2 + r1^2), r = fl(fl(B t') + c) with (B t')_k = fl(fl(b_k0 x') + fl(b_k1 y'));
//   !INV: dot = the products of the LHFs' entries summed left to right (a00, a01, [tx,] a10, a11[, ty, then + 1]),
//         D = sqrt(|fl(fl(|LHF'|^2 + |LHF|^2) - fl(2 dot)) + 1e-12|).
// GATE: D + 1000 (1 - scale_ok + centre_far) with centre_far = centre_dist >= cth and scale_ok = |1 - s' / fl(s + 1e-12)| <= coef
// (always true when coef <= 0).  That sum is never below D, so it is only formed when D < best.
template <bool INV, bool SKIP, bool GATE>
__device__ __forceinline__ void frob_scan(const FroRow& r, const float4* __restrict__ ta, const float4* __restrict__ tt,
                                          const float* __restrict__ tn, int m, int u0, const ag_frobenius_params_t& prm, float& best, int& bi) {
    const bool sgate = prm.scale_diff_coef > 0.f;
    for (int u = 0; u < m; u++) {
        const float4 a = ta[u], t = tt[u];
        float d;
        if (INV) {
            const float m00 = dot2f(r.m[0], a.x, r.m[1], a.z), m01 = dot2f(r.m[0], a.y, r.m[1], a.w);
            const float m10 = dot2f(r.m[2], a.x, r.m[3], a.z), m11 = dot2f(r.m[2], a.y, r.m[3], a.w);
            d = __fadd_rn(__fadd_rn(__fadd_rn(sqf(__fsub_rn(m00, 1.f)), sqf(m01)), sqf(m10)), sqf(__fsub_rn(m11, 1.f)));
            if (!SKIP) {
                const float r0 = __fadd_rn(dot2f(r.m[0], t.x, r.m[1], t.y), r.m[4]);
                const float r1 = __fadd_rn(dot2f(r.m[2], t.x, r.m[3], t.y), r.m[5]);
                d = __fadd_rn(d, __fadd_rn(sqf(r0), sqf(r1)));
            }
        } else {
            float dot;
            if (SKIP) {
                dot = __fadd_rn(__fadd_rn(dot2f(r.m[0], a.x, r.m[1], a.y), __fmul_rn(r.m[3], a.z)), __fmul_rn(r.m[4], a.w));
            } else {
                dot = __fadd_rn(dot2f(r.m[0], a.x, r.m[1], a.y), __fmul_rn(r.m[2], t.x));
                dot = __fadd_rn(__fadd_rn(__fadd_rn(dot, __fmul_rn(r.m[3], a.z)), __fmul_rn(r.m[4], a.w)), __fmul_rn(r.m[5], t.y));
                dot = __fadd_rn(dot, 1.f);
            }
            d = sqrtf(fabsf(__fadd_rn(__fsub_rn(__fadd_rn(tn[u], r.nl), __fmul_rn(2.f, dot)), 1e-12f)));
        }
        if (!(d < best)) continue;
        if (GATE) {
            const bool far = centre_dist(r.x, r.y, r.na, t) >= prm.center_dist_th;
            const bool ok = !sgate || fabsf(__fsub_rn(1.f, __fdiv_rn(t.w, r.s1e))) <= prm.scale_diff_coef;
            d = __fadd_rn(__fmul_rn(__fadd_rn(__fsub_rn(1.f, ok ? 1.f : 0.f), far ? 1.f : 0.f), 1000.f), d);
            if (!(d < best)) continue;
        }
        best = d; bi = u0 + u;   // ascending u: the lowest index among the minima; NaN never wins
    }
}

// Pair p -> (i, j) and the row / column counts n1, n2 (tentative mode: n1 = n2 = ntent[p]), or false when the pair cannot be checked:
// an image index out of range, a count outside 0..cap.  The tentative rows' range is checked by the caller (block-wide).
template <bool TENT>
__device__ __forceinline__ bool frob_pair(const int* __restrict__ pairs, int p, int S1, int cap1, int S2, int cap2, const int* __restrict__ cnt1,
                                          const int* __restrict__ cnt2, int tcap, int& i, int& j, int& n1, int& n2) {
    if (TENT) {
        n1 = n2 = pair_tentatives(pairs, p, S1, S2, cnt1, tcap, i, j);
        return n1 >= 0;
    }
    i = pairs ? pairs[2 * (size_t)p] : p;
    j = pairs ? pairs[2 * (size_t)p + 1] : p;
    if (i < 0 || i >= S1 || j < 0 || j >= S2) return false;
    n1 = cnt1[i]; n2 = cnt2[j];
    return n1 >= 0 && n1 <= cap1 && n2 >= 0 && n2 <= cap2;
}

// Grid (P, rcap / FRO_NT): thread t of CTA y owns row y FRO_NT + t of pair p; the CTA streams the pair's reprojected columns through
// shared memory and writes the row's (min_dist, idx2).  TENT: rows and columns are the tentatives' rows of lafs1 / lafs2, cnt1 = ntent;
// otherwise rows 0..cnt1[i]-1 of set i against rows 0..cnt2[j]-1 of set j.
template <bool TENT>
__global__ void __launch_bounds__(FRO_NT) frob_pass_kernel(const float* __restrict__ lafs1, int S1, int cap1, const float* __restrict__ lafs2,
                                                           int S2, int cap2, const int* __restrict__ pairs, const int* __restrict__ tent_all,
                                                           const int* __restrict__ cnt1, const int* __restrict__ cnt2, int rcap,
                                                           const float* __restrict__ H1to2, const ag_frobenius_params_t prm,
                                                           float* __restrict__ min_dist, int* __restrict__ idx2) {
    __shared__ float4 ta[FRO_TILE], tt[FRO_TILE];
    __shared__ float tn[FRO_TILE];
    __shared__ double G[9];
    const int p = blockIdx.x, tid = threadIdx.x, t = blockIdx.y * FRO_NT + tid;
    int i, j, n1, n2;
    if (!frob_pair<TENT>(pairs, p, S1, cap1, S2, cap2, cnt1, cnt2, rcap, i, j, n1, n2) || (int)blockIdx.y * FRO_NT >= n1) return;
    const int* tent = TENT ? tent_all + (size_t)p * rcap * 2 : nullptr;
    if (TENT && !rows_in_range<FRO_NT>(tent, n1, cap1, cap2)) return;
    const float* L1 = lafs1 + (size_t)i * cap1 * 6;
    const float* L2 = lafs2 + (size_t)j * cap2 * 6;
    if (tid == 0) inverse_h(H1to2 + (size_t)p * 9, G);
    FroRow r;
    if (t < n1) frob_row(L1 + (size_t)(TENT ? tent[2 * (size_t)t] : t) * 6, prm, r);
    float best = INFINITY;
    int bi = 0;
    const int variant = (prm.inv_to_eye ? 4 : 0) + (prm.skip_center ? 2 : 0) + (prm.center_gate ? 1 : 0);
    for (int u0 = 0; u0 < n2; u0 += FRO_TILE) {
        const int m = min(FRO_TILE, n2 - u0);
        __syncthreads();
        for (int u = tid; u < m; u += FRO_NT)
            frob_col(G, L2 + (size_t)(TENT ? tent[2 * (size_t)(u0 + u) + 1] : u0 + u) * 6, prm, ta[u], tt[u], tn[u]);
        __syncthreads();
        if (t >= n1) continue;
        switch (variant) {
            case 0: frob_scan<false, false, false>(r, ta, tt, tn, m, u0, prm, best, bi); break;
            case 1: frob_scan<false, false, true>(r, ta, tt, tn, m, u0, prm, best, bi); break;
            case 2: frob_scan<false, true, false>(r, ta, tt, tn, m, u0, prm, best, bi); break;
            case 3: frob_scan<false, true, true>(r, ta, tt, tn, m, u0, prm, best, bi); break;
            case 4: frob_scan<true, false, false>(r, ta, tt, tn, m, u0, prm, best, bi); break;
            case 5: frob_scan<true, false, true>(r, ta, tt, tn, m, u0, prm, best, bi); break;
            case 6: frob_scan<true, true, false>(r, ta, tt, tn, m, u0, prm, best, bi); break;
            default: frob_scan<true, true, true>(r, ta, tt, tn, m, u0, prm, best, bi); break;
        }
    }
    if (t < n1) {
        min_dist[(size_t)p * rcap + t] = best;
        idx2[(size_t)p * rcap + t] = bi;
    }
}

// One CTA per pair: the rows with min_dist <= dist_threshold in ascending order into true / ntrue (-1 for a pair that cannot be checked).
template <bool TENT>
__global__ void __launch_bounds__(VT) frob_compact_kernel(int S1, int cap1, int S2, int cap2, const int* __restrict__ pairs,
                                                          const int* __restrict__ tent_all, const int* __restrict__ cnt1,
                                                          const int* __restrict__ cnt2, int rcap, float th, const float* __restrict__ min_dist,
                                                          int* __restrict__ true_all, int* __restrict__ ntrue) {
    __shared__ int wsum[VT / 32];
    const int p = blockIdx.x, tid = threadIdx.x;
    int i, j, n1, n2;
    bool ok = frob_pair<TENT>(pairs, p, S1, cap1, S2, cap2, cnt1, cnt2, rcap, i, j, n1, n2);
    if (TENT && ok) ok = rows_in_range(tent_all + (size_t)p * rcap * 2, n1, cap1, cap2);
    if (!ok) {
        if (tid == 0) ntrue[p] = -1;
        return;
    }
    const size_t base = (size_t)p * rcap;
    int run = 0;
    for (int r0 = 0; r0 < n1; r0 += VT) {
        const int t = r0 + tid;
        const bool keep = t < n1 && min_dist[base + t] <= th;
        run = compact_rows(keep, t, true_all, base, run, wsum);
    }
    if (tid == 0) ntrue[p] = run;
}

// reprojectLAFs for S sets of cap rows, one H per set (G = H, or H^-1 with invert), the 2x2 part rectified with up_is_up.
__global__ void reproject_lafs_kernel(const float* __restrict__ lafs, int cap, const float* __restrict__ H, int invert, int up_is_up,
                                      float* __restrict__ out) {
    const int s = blockIdx.y, r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= cap) return;
    double G[9];
    if (invert) inverse_h(H + (size_t)s * 9, G);
    else
        for (int k = 0; k < 9; k++) G[k] = H[(size_t)s * 9 + k];
    const size_t o = ((size_t)s * cap + r) * 6;
    float A[4], t[2];
    reproject_laf(G, lafs + o, A, t);
    frame_2x2(A, up_is_up != 0);
    out[o] = A[0]; out[o + 1] = A[1]; out[o + 2] = t[0];
    out[o + 3] = A[2]; out[o + 4] = A[3]; out[o + 5] = t[1];
}

// ---- fundamental-matrix RANSAC (the notebook's alternative line, findFundamentalMatrix(src, dst, 0.5)) ----------------------------
constexpr int F_SAMPLE = 7;            // correspondences per hypothesis
constexpr double PIVOT_EPS = 1e-9;     // 7-point elimination: a column whose largest candidate |pivot| <= PIVOT_EPS * max|A| is free
constexpr int BISECT_STEPS = 1100;     // bisection cap per bracketed cubic root: enough to close any bracket in the double range

// Sampson test in pixels, division-free: (x2' F x1)^2 <= th^2 ((F x1)_0^2 + (F x1)_1^2 + (F' x2)_0^2 + (F' x2)_1^2), the right-hand
// side positive.  A NaN anywhere fails both comparisons.
__device__ __forceinline__ bool is_inlier_f(const double* F, float4 c, double th2) {
    const double x = c.x, y = c.y, x2 = c.z, y2 = c.w;
    const double a = F[0] * x + F[1] * y + F[2], b = F[3] * x + F[4] * y + F[5], d = F[6] * x + F[7] * y + F[8];
    const double g = F[0] * x2 + F[3] * y2 + F[6], k = F[1] * x2 + F[4] * y2 + F[7];
    const double e = x2 * a + y2 * b + d;
    const double den = a * a + b * b + g * g + k * k;
    return den > 0.0 && e * e <= th2 * den;
}

// F /= +-|F|_F, the sign making the largest-magnitude entry (the lowest index on ties) positive; false when F is zero or not finite.
__device__ __forceinline__ bool normalise_f(double* F) {
    double ss = 0.0;
    int m = 0;
    for (int k = 0; k < 9; k++) {
        ss = ss + F[k] * F[k];
        if (fabs(F[k]) > fabs(F[m])) m = k;
    }
    if (!(ss > 0.0) || !isfinite(ss)) return false;
    const double nr = F[m] < 0.0 ? -sqrt(ss) : sqrt(ss);
    for (int k = 0; k < 9; k++) F[k] = F[k] / nr;
    return true;
}

// F = T2' Fn T1, normalised by normalise_f.
__device__ __forceinline__ bool denormalise_f(const Hartley& T, const double* Fn, double* F) {
    const double T1[9] = {T.s1, 0.0, -(T.s1 * T.c1x), 0.0, T.s1, -(T.s1 * T.c1y), 0.0, 0.0, 1.0};
    const double T2t[9] = {T.s2, 0.0, 0.0, 0.0, T.s2, 0.0, -(T.s2 * T.c2x), -(T.s2 * T.c2y), 1.0};
    double tmp[9];
    mul3(T2t, Fn, tmp);
    mul3(tmp, T1, F);
    return normalise_f(F);
}

// Real roots of a3 x^3 + a2 x^2 + a1 x + a0 in ascending order, with + - * / sqrt only (no libm transcendentals, so every platform gets
// the same bits).  a3 == 0 drops to the quadratic (numerically stable form) or linear case.  Otherwise, on the monic form, the
// critical points c1 < c2 (when the derivative has two real roots) split [-R, R], R = 1 + max|b_k| the Cauchy bound, into monotone
// pieces; each piece whose end values change sign (a zero at its right end counts) is bisected, keeping the end with the left
// value's strict sign as `lo`, until the midpoint equals an end (at most BISECT_STEPS times), and gives its `hi`.  Values are
// evaluated from the original coefficients (Horner): a tiny a3 makes the monic ones huge and cancel at the finite roots.  Non-finite coefficients give no roots.
__device__ __forceinline__ int cubic_roots(double a3, double a2, double a1, double a0, double* r) {
    if (!isfinite(a3) || !isfinite(a2) || !isfinite(a1) || !isfinite(a0)) return 0;
    if (a3 == 0.0) {
        if (a2 == 0.0) {
            if (a1 == 0.0) return 0;
            r[0] = -a0 / a1;
            return 1;
        }
        const double disc = a1 * a1 - 4.0 * a2 * a0;
        if (disc < 0.0) return 0;
        if (disc == 0.0) {
            r[0] = -a1 / (2.0 * a2);
            return 1;
        }
        const double sq = sqrt(disc);
        const double q = a1 >= 0.0 ? -0.5 * (a1 + sq) : -0.5 * (a1 - sq);
        const double x1 = q / a2, x2 = a0 / q;
        r[0] = x1 < x2 ? x1 : x2;
        r[1] = x1 < x2 ? x2 : x1;
        return 2;
    }
    const double b2 = a2 / a3, b1 = a1 / a3, b0 = a0 / a3;
    double m = fabs(b2);
    if (fabs(b1) > m) m = fabs(b1);
    if (fabs(b0) > m) m = fabs(b0);
    const double R = 1.0 + m;
    if (!isfinite(R)) return 0;
    double x[4];
    int np = 2;
    x[0] = -R;
    const double d = b2 * b2 - 3.0 * b1;
    if (d > 0.0) {
        const double sq = sqrt(d);
        x[1] = (-b2 - sq) / 3.0;
        x[2] = (-b2 + sq) / 3.0;
        np = 4;
    }
    x[np - 1] = R;
    int nr = 0;
    for (int i = 0; i + 1 < np; i++) {
        double lo = x[i], hi = x[i + 1];
        const double fl = ((a3 * lo + a2) * lo + a1) * lo + a0, fh = ((a3 * hi + a2) * hi + a1) * hi + a0;
        if (!((fl < 0.0 && fh >= 0.0) || (fl > 0.0 && fh <= 0.0))) continue;
        for (int it = 0; it < BISECT_STEPS; it++) {
            const double mid = 0.5 * (lo + hi);
            if (mid == lo || mid == hi) break;   // the bracket is two adjacent doubles
            const double fm = ((a3 * mid + a2) * mid + a1) * mid + a0;
            if (fl < 0.0 ? fm < 0.0 : fm > 0.0) lo = mid;
            else hi = mid;
        }
        r[nr++] = hi;
    }
    return nr;
}

// det(F2 + l D) = a3 l^3 + a2 l^2 + a1 l + a0: a0 = det F2, a1 = tr(adj(F2) D), a2 = tr(adj(D) F2), a3 = det D (first-row cofactor
// expansions; traces summed over the 9 products in row-major order of the adjugate).
__device__ __forceinline__ void det_cubic(const double* F2, const double* D, double* a) {
    double A2[9], AD[9];
    adj3(F2, A2);
    adj3(D, AD);
    a[0] = F2[0] * A2[0] + F2[1] * A2[3] + F2[2] * A2[6];
    a[3] = D[0] * AD[0] + D[1] * AD[3] + D[2] * AD[6];
    double t1 = 0.0, t2 = 0.0;
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) {
            t1 = t1 + A2[3 * r + c] * D[3 * c + r];
            t2 = t2 + AD[3 * r + c] * F2[3 * c + r];
        }
    a[1] = t1;
    a[2] = t2;
}

// 7-point solver on normalised correspondences u[k] = (u1, v1, u2, v2): row k of the 7x9 constraint matrix is
// (u2 u1, u2 v1, u2, v2 u1, v2 v1, v2, u1, v1, 1), so row k . vec(F) = x2' F x1.  Gauss-Jordan elimination column by column with
// partial pivoting (largest |A[r][c]| over the rows not yet pivots, the lowest row on ties; a column is free when that is
// <= PIVOT_EPS * max|A|); a rank below 7 is a degenerate sample (0 models).  The two free columns f1 < f2 give the null vectors F1, F2
// (1 at their own free column, 0 at the other, -A[i][f] / A[i][pivot_i] at pivot column i); every real root l of det(F2 + l (F1 - F2))
// (l of the form l F1 + (1 - l) F2) gives a model Fn = F2 + l D, in ascending l.  Returns the number of models (<= 3).
__device__ __forceinline__ int seven_point(const double (&u)[F_SAMPLE][4], double (&Fn)[3][9]) {
    double A[F_SAMPLE][9];
    double mx = 0.0;
    for (int k = 0; k < F_SAMPLE; k++) {
        const double u1 = u[k][0], v1 = u[k][1], u2 = u[k][2], v2 = u[k][3];
        const double row[9] = {u2 * u1, u2 * v1, u2, v2 * u1, v2 * v1, v2, u1, v1, 1.0};
        for (int c = 0; c < 9; c++) {
            A[k][c] = row[c];
            if (fabs(row[c]) > mx) mx = fabs(row[c]);
        }
    }
    const double tol = PIVOT_EPS * mx;
    int pc[F_SAMPLE], rank = 0;
    unsigned freemask = 0;
    for (int c = 0; c < 9; c++) {
        if (rank == F_SAMPLE) {
            freemask |= 1u << c;
            continue;
        }
        int pr = rank;
        double pa = fabs(A[rank][c]);
        for (int r = rank + 1; r < F_SAMPLE; r++)
            if (fabs(A[r][c]) > pa) { pa = fabs(A[r][c]); pr = r; }
        if (!(pa > tol)) {
            freemask |= 1u << c;
            continue;
        }
        if (pr != rank)
            for (int k = 0; k < 9; k++) {
                const double t = A[rank][k];
                A[rank][k] = A[pr][k];
                A[pr][k] = t;
            }
        for (int r = 0; r < F_SAMPLE; r++) {
            if (r == rank) continue;
            const double f = A[r][c] / A[rank][c];
            for (int k = 0; k < 9; k++) A[r][k] = k == c ? 0.0 : A[r][k] - f * A[rank][k];
        }
        pc[rank++] = c;
    }
    if (rank < F_SAMPLE) return 0;
    int f1 = -1, f2 = -1;
    for (int c = 0; c < 9; c++)
        if ((freemask >> c) & 1u) {
            if (f1 < 0) f1 = c;
            else if (f2 < 0) f2 = c;
        }
    double F1[9], F2[9], D[9];
    for (int k = 0; k < 9; k++) { F1[k] = 0.0; F2[k] = 0.0; }
    F1[f1] = 1.0;
    F2[f2] = 1.0;
    for (int i = 0; i < F_SAMPLE; i++) {
        F1[pc[i]] = -(A[i][f1] / A[i][pc[i]]);
        F2[pc[i]] = -(A[i][f2] / A[i][pc[i]]);
    }
    // Scale both null vectors to unit norm: in normalised coordinates the true F's constant entry is ~0, so the vector with its 1
    // there is huge, all roots then bunch near l = 1 and the cubic's coefficients cancel.
    double n1 = 0.0, n2 = 0.0;
    for (int k = 0; k < 9; k++) {
        n1 = n1 + F1[k] * F1[k];
        n2 = n2 + F2[k] * F2[k];
    }
    n1 = sqrt(n1);
    n2 = sqrt(n2);
    for (int k = 0; k < 9; k++) {
        F1[k] = F1[k] / n1;
        F2[k] = F2[k] / n2;
    }
    for (int k = 0; k < 9; k++) D[k] = F1[k] - F2[k];
    double a[4], l[3];
    det_cubic(F2, D, a);
    const int nl = cubic_roots(a[3], a[2], a[1], a[0], l);
    for (int m = 0; m < nl; m++)
        for (int k = 0; k < 9; k++) Fn[m][k] = F2[k] + l[m] * D[k];
    return nl;
}

// Rank-2 fundamental matrix from the normalised 9x9 normal matrix in s.A / s.V (after normal_matrix_eigen): Fn = the eigenvector of
// the smallest eigenvalue, then Fn <- Fn (I - v v'), v the eigenvector of the smallest eigenvalue of Fn'Fn (jacobi3), then
// denormalised.  Thread 0.
__device__ bool rank2_refit_f(const RansacShared& s, const Hartley& T, double* F) {
    const int m = smallest_diag<9>(s.A);
    double Fn[9], G[9], v[3], P[9], Fr[9];
    for (int e = 0; e < 9; e++) Fn[e] = s.V[9 * e + m];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) G[3 * r + c] = Fn[r] * Fn[c] + Fn[3 + r] * Fn[3 + c] + Fn[6 + r] * Fn[6 + c];
    smallest_eigvec3(G, v);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) P[3 * r + c] = (r == c ? 1.0 : 0.0) - v[r] * v[c];
    mul3(Fn, P, Fr);
    return denormalise_f(T, Fr, F);
}

// Normalised 8-point least squares on the rows of the mask `inl` (Hartley normalisation of those rows, the 9x9 normal matrix of the
// constraint rows reduced in the fixed order, its smallest eigenvector, rank 2).  Writes s.Hr; false when the inliers do not give a
// finite non-zero F.
__device__ bool refit_f(const float* L1, const float* L2, const int* tent, int n, const unsigned char* inl, RansacShared& s) {
    Hartley T;
    if (!hartley(L1, L2, tent, n, inl, s, T)) return false;   // uniform across the block: every thread returns
    double nm[45];
#pragma unroll
    for (int k = 0; k < 45; k++) nm[k] = 0.0;
    for (int t = threadIdx.x; t < n; t += VT) {
        const float4 c = tent_centres(L1, L2, tent, t);
        const bool in = inl[t];
        const double u = (c.x - T.c1x) * T.s1, v = (c.y - T.c1y) * T.s1, up = (c.z - T.c2x) * T.s2, vp = (c.w - T.c2y) * T.s2;
        const double a[9] = {up * u, up * v, up, vp * u, vp * v, vp, u, v, 1.0};
        int e = 0;
#pragma unroll
        for (int k = 0; k < 9; k++)
#pragma unroll
            for (int l = k; l < 9; l++, e++) nm[e] = nm[e] + (in ? a[k] * a[l] : 0.0);
    }
    block_sum<45>(nm, s.red, s.sums);
    normal_matrix_eigen(s);
    if (threadIdx.x == 0) s.bad = !rank2_refit_f(s, T, s.Hr);
    __syncthreads();
    return !s.bad;
}

// ---- DEGENSAC (Chum, Werner and Matas, CVPR 2005): degeneracy test, plane-and-parallax, local optimisation ------------------------
constexpr double DEG_H_TH_FACTOR = 4.0;   // DEG_H_TH = DEG_H_TH_FACTOR * inl_th: a point agrees with a plane H within it (transfer, px)
constexpr int DEG_MIN_AGREE = 5;          // a 7-point sample is H-degenerate when some triplet's H agrees with this many of its points
constexpr uint64_t DEG_SEED_TAG = 0xD5A61266F0C9392Cull;   // the plane-and-parallax sampler's stream: seed ^ DEG_SEED_TAG
constexpr uint32_t DEG_H_BASE = 0x80000000u;   // its hypotheses: DEG_H_BASE + k VT + thread (k: degeneracy tests so far), above any h
__constant__ int deg_triplets[5][3] = {{0, 1, 2}, {3, 4, 5}, {0, 1, 6}, {3, 4, 6}, {2, 5, 6}};

// (a x b) into o.
__device__ __forceinline__ void cross_v(const double* a, const double* b, double* o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}
// O = [e]x M: column c of O is e x (column c of M).
__device__ __forceinline__ void skew_mul(const double* e, const double* M, double* O) {
    for (int c = 0; c < 3; c++) {
        const double m[3] = {M[c], M[3 + c], M[6 + c]};
        double o[3];
        cross_v(e, m, o);
        O[c] = o[0]; O[3 + c] = o[1]; O[6 + c] = o[2];
    }
}

// The homography of the plane through the three correspondences c[0..2] compatible with F (Hartley and Zisserman, result 13.6):
// H = A - e' (M^-1 b)', A = [e']x F, M the image-1 points as rows, b_m = (x'_m x A x_m).(x'_m x e') / |x'_m x e'|^2, normalised by
// normalise_h.  False when M is singular or H / H[2][2] is not finite.
__device__ bool triplet_homography(const double* A, const double* e, const float4* c, double* H) {
    double b[3], M[9];
    for (int m = 0; m < 3; m++) {
        const double x = c[m].x, y = c[m].y;
        const double ax[3] = {A[0] * x + A[1] * y + A[2], A[3] * x + A[4] * y + A[5], A[6] * x + A[7] * y + A[8]};
        const double xp[3] = {(double)c[m].z, (double)c[m].w, 1.0};
        double pp[3], q[3];
        cross_v(xp, ax, pp);
        cross_v(xp, e, q);
        b[m] = (pp[0] * q[0] + pp[1] * q[1] + pp[2] * q[2]) / (q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
        M[3 * m] = x; M[3 * m + 1] = y; M[3 * m + 2] = 1.0;
    }
    double Ad[9];
    adj3(M, Ad);
    const double det = M[0] * Ad[0] + M[1] * Ad[3] + M[2] * Ad[6];
    if (det == 0.0) return false;
    double v[3];
    for (int k = 0; k < 9; k++) Ad[k] = Ad[k] / det;
    for (int r = 0; r < 3; r++) v[r] = Ad[3 * r] * b[0] + Ad[3 * r + 1] * b[1] + Ad[3 * r + 2] * b[2];
    for (int r = 0; r < 3; r++)
        for (int k = 0; k < 3; k++) H[3 * r + k] = A[3 * r + k] - e[r] * v[k];
    return normalise_h(H);
}

// Degeneracy test of the 7-point sample c with its model F: e' the left epipole (F' e' = 0, the smallest eigenvector of F F' by jacobi3),
// and for each of the five triplets of Chum et al. the H of triplet_homography.  Returns the most sample points that one H agrees with
// (is_inlier at thd2), that H (the lowest triplet on ties) in Hd.  One thread.
__device__ int degeneracy_test(const double* F, const float4 (&c)[F_SAMPLE], double thd2, double* Hd) {
    double G[9], e[3];
    for (int r = 0; r < 3; r++)
        for (int k = 0; k < 3; k++) G[3 * r + k] = F[3 * r] * F[3 * k] + F[3 * r + 1] * F[3 * k + 1] + F[3 * r + 2] * F[3 * k + 2];
    smallest_eigvec3(G, e);
    double A[9];
    skew_mul(e, F, A);
    int best = 0;
    for (int t = 0; t < 5; t++) {
        const float4 ct[3] = {c[deg_triplets[t][0]], c[deg_triplets[t][1]], c[deg_triplets[t][2]]};
        double H[9];
        if (!triplet_homography(A, e, ct, H)) continue;
        int k = 0;
        for (int q = 0; q < F_SAMPLE; q++) k += is_inlier(H, c[q], thd2);
        if (k > best) {
            best = k;
            for (int i = 0; i < 9; i++) Hd[i] = H[i];
        }
    }
    return best;
}

// Shared state of the DEGENSAC steps (apart from RansacShared).
struct DegenShared {
    double Hd[9];
    unsigned long long key[VT / 32];
    int agree;
};

// The DEGENSAC steps after a chunk's winner (sample h, model s.H, `best` inliers) has raised the so-far-best count: the degeneracy test
// of its sample; for an H-degenerate sample, H refitted on its inliers at DEG_H_TH (the homography RANSAC's rounds) and
// plane-and-parallax, thread t drawing two rows that are not inliers of H from hypothesis DEG_H_BASE + k VT + t of the stream
// seed ^ DEG_SEED_TAG, F = [e']x H with e' = (H x_a x x'_a) x (H x_b x x'_b), the best (most inliers, then lowest thread) replacing
// s.H when it has more inliers; then the refit rounds on s.H.  `inl` is scratch.  Block-wide; returns the new so-far-best count.
__device__ __noinline__ int degensac_step(const float* L1, const float* L2, const int* tent, int n, int ntiles, double th2, uint64_t seed,
                                          int h, int k, unsigned char* inl, int best, RansacShared& s) {
    __shared__ DegenShared d;
    const int tid = threadIdx.x;
    const double thd2 = (DEG_H_TH_FACTOR * DEG_H_TH_FACTOR) * th2;
    if (tid == 0) {
        int idx[F_SAMPLE];
        draw_sample(seed, h, n, idx);   // the winner's sample: complete, since it gave a model
        float4 c[F_SAMPLE];
        for (int q = 0; q < F_SAMPLE; q++) c[q] = tent_centres(L1, L2, tent, idx[q]);
        d.agree = degeneracy_test(s.H, c, thd2, d.Hd);
    }
    __syncthreads();
    if (d.agree >= DEG_MIN_AGREE) {
        refit_rounds<false>(L1, L2, tent, n, thd2, inl, d.Hd, s);   // inl: the inliers of d.Hd
        double F[9];
        bool ok;
        {
            const uint32_t hh = DEG_H_BASE + (uint32_t)k * VT + (uint32_t)tid;
            int idx[2], got = 0;
            for (int dr = 0; dr < MAX_DRAWS && got < 2; dr++) {
                const int v = draw_index(seed ^ DEG_SEED_TAG, (int)hh, dr, n);
                if (!inl[v] && (got == 0 || v != idx[0])) idx[got++] = v;
            }
            ok = got == 2;
            if (ok) {
                double l[2][3];
                for (int q = 0; q < 2; q++) {
                    const float4 c = tent_centres(L1, L2, tent, idx[q]);
                    const double x = c.x, y = c.y;
                    const double hx[3] = {d.Hd[0] * x + d.Hd[1] * y + d.Hd[2], d.Hd[3] * x + d.Hd[4] * y + d.Hd[5],
                                          d.Hd[6] * x + d.Hd[7] * y + d.Hd[8]};
                    const double xp[3] = {(double)c.z, (double)c.w, 1.0};
                    cross_v(hx, xp, l[q]);
                }
                double e[3];
                cross_v(l[0], l[1], e);
                skew_mul(e, d.Hd, F);
                ok = normalise_f(F);
            }
        }
        int cnt = 0;
        for (int tb = 0; tb < ntiles; tb++) {
            const int t0 = tb * VTILE, m = min(VTILE, n - t0);
            if (ntiles > 1) {   // one tile stays loaded from the first chunk
                __syncthreads();
                for (int t = tid; t < m; t += VT) s.tile[t] = tent_centres(L1, L2, tent, t0 + t);
                __syncthreads();
            }
            if (ok)
                for (int t = 0; t < m; t++) cnt += is_inlier_f(F, s.tile[t], th2);
        }
        const unsigned long long mine = ok ? ((unsigned long long)cnt << 32) | (unsigned)~(unsigned)tid : 0ull;
        const unsigned long long bk = block_max_key(mine, d.key);
        const int bc = (int)(bk >> 32);
        if (bk != 0 && bc > best) {
            if (mine == bk)
                for (int q = 0; q < 9; q++) s.H[q] = F[q];
            best = bc;
        }
        __syncthreads();
    }
    return refit_rounds<true>(L1, L2, tent, n, th2, inl, s.H, s);
}

// DEGEN: ag_fundamental_degensac (degensac_step whenever a chunk's winner raises the so-far-best count); otherwise ag_fundamental_ransac.
template <bool DEGEN>
__global__ void __launch_bounds__(VT) fransac_kernel(const float* __restrict__ lafs1, int S1, int cap1, const float* __restrict__ lafs2, int S2,
                                                     int cap2, const int* __restrict__ pairs, const int* __restrict__ tent_all,
                                                     const int* __restrict__ ntent, int tcap, double th2, double log1mconf, int max_iters,
                                                     uint64_t seed, float* __restrict__ Fout, unsigned char* __restrict__ inl_all,
                                                     int* __restrict__ ninl, int* __restrict__ iters) {
    __shared__ RansacShared s;
    const int tid = threadIdx.x;
    const int* tent;
    const float *L1, *L2;
    int n;
    if (!verify_pair(lafs1, S1, cap1, lafs2, S2, cap2, pairs, tent_all, ntent, tcap, ninl, n, tent, L1, L2)) return;
    unsigned char* inl = inl_all + (size_t)blockIdx.x * tcap;
    int best = 0, h_done = 0;
    if (n >= F_SAMPLE) {
        // Hartley normalisation of the rows whose four coordinates are finite
        Hartley T;
        double nd;
        const bool spread = hartley(L1, L2, tent, n, nullptr, s, T, &nd);
        // fewer than 7 finite rows, or all of them on one point in an image: no hypothesis is drawn (iters = 0)
        const bool search = nd >= (double)F_SAMPLE && spread;
        const int ntiles = (n + VTILE - 1) / VTILE;
        int ntests = 0;   // DEGEN: degeneracy tests so far
        for (int h0 = 0; search; h0 += VT) {
            const int h = h0 + tid;
            double Fm[3][9];
            bool okm[3] = {false, false, false};   // model r (root r in ascending order) exists
            int idx[F_SAMPLE];
            if (h < max_iters && draw_sample(seed, h, n, idx)) {
                double u[F_SAMPLE][4];
                bool fin = true;
                for (int q = 0; q < F_SAMPLE; q++) {
                    const float4 c = tent_centres(L1, L2, tent, idx[q]);
                    fin &= finite4(c);
                    u[q][0] = (c.x - T.c1x) * T.s1; u[q][1] = (c.y - T.c1y) * T.s1;
                    u[q][2] = (c.z - T.c2x) * T.s2; u[q][3] = (c.w - T.c2y) * T.s2;
                }
                double Fn[3][9];
                const int nl = fin ? seven_point(u, Fn) : 0;
#pragma unroll
                for (int r = 0; r < 3; r++)
                    if (r < nl) okm[r] = denormalise_f(T, Fn[r], Fm[r]);
            }
            const bool any = okm[0] || okm[1] || okm[2];
            int cnt[3] = {0, 0, 0};
            for (int tb = 0; tb < ntiles; tb++) {
                const int t0 = tb * VTILE, m = min(VTILE, n - t0);
                if (ntiles > 1 || h0 == 0) {
                    __syncthreads();
                    for (int t = tid; t < m; t += VT) s.tile[t] = tent_centres(L1, L2, tent, t0 + t);
                    __syncthreads();
                }
                if (any)
                    for (int t = 0; t < m; t++) {
                        const float4 c = s.tile[t];
#pragma unroll
                        for (int r = 0; r < 3; r++)
                            if (okm[r]) cnt[r] += is_inlier_f(Fm[r], c, th2);
                    }
            }
            // best of the chunk: highest count, then lowest h, then lowest root
            int rb = -1, cb = -1;
#pragma unroll
            for (int r = 0; r < 3; r++)
                if (okm[r] && cnt[r] > cb) { cb = cnt[r]; rb = r; }
            const unsigned long long mine =
                any ? ((unsigned long long)cb << 34) | ((unsigned long long)(0x7fffffff - h) << 2) | (unsigned long long)(3 - rb) : 0ull;
            const unsigned long long bk = block_max_key(mine, s.key);
            const int bc = (int)(bk >> 34);
            if (bk != 0 && bc > best) {
                if (mine == bk) {
#pragma unroll
                    for (int r = 0; r < 3; r++)
                        if (r == rb)
#pragma unroll
                            for (int k = 0; k < 9; k++) s.H[k] = Fm[r][k];
                }
                best = bc;
                if constexpr (DEGEN) {
                    __syncthreads();
                    best = degensac_step(L1, L2, tent, n, ntiles, th2, seed, 0x7fffffff - (int)((bk >> 2) & 0xffffffffull), ntests++, inl,
                                         best, s);
                }
            }
            h_done = min(h0 + VT, max_iters);
            double need;   // adaptive number of samples for `confidence`
            const double pr = (double)best / (double)n, p7 = pr * pr * pr * pr * pr * pr * pr;
            if (p7 >= 1.0) need = 0.0;
            else if (p7 <= 0.0 || 1.0 - p7 == 1.0) need = INFINITY;   // log(1 - p7) would be 0: no sample count reaches confidence
            else need = ceil(log1mconf / log(1.0 - p7));
            __syncthreads();
            if ((double)h_done >= fmin(need, (double)max_iters)) break;
        }
    }
    finish_ransac<true>(L1, L2, tent, n, th2, best, h_done, inl, s, Fout, ninl, iters);
}

// ---- homography RANSAC from two affine correspondences (ag_homography_ransac_affine) -------------------------------------------------
// A tentative of two LAFs gives the centre pair and the local affinity A2 A1^-1, which is the Jacobian a homography has at that point:
// two of them determine H, where points need four, and a row whose frames disagree with H is not an inlier.
constexpr int ATILE = sizeof(RansacShared::tile) / sizeof(AcRow);   // 682 rows of 48 B in RansacShared's tile (32 KB)
constexpr double CHOL_EPS = 1e-10;   // 2-AC normal equations: a Cholesky pivot <= CHOL_EPS times its diagonal entry is a degenerate sample
// LO-RANSAC's iterative local optimisation (Chum, Matas and Kittler, 2003): point DLT on the inliers at LO_FACTOR times both thresholds
// (centre and frame), then at half that, ... down to 1 times.  A 2-AC hypothesis from two true matches with noisy frames fits near its
// sample only: it may have fewer than 4 inliers at the strict thresholds, where the refit rounds cannot start.
constexpr double LO_FACTOR = 16.0;
constexpr int LO_STEPS = 5;          // factors 16, 8, 4, 2, 1

// The frame distance of row r under the homography whose adjugate is G (H^-1 up to scale): D = |A1^-1 J A2 - I|_F^2 with J = linH(G) at
// the image-2 centre, the reference's skip-centre Frobenius distance (get_GT_correspondence_indexes_Fro with skip_center_in_Fro) of the
// row's own pair, in fp64.  False when either frame is not finite or singular.
__device__ __forceinline__ bool frame_distance(const double* G, const AcRow& r, double& D) {
    if (!finite4(r.a1) || !finite4(r.a2)) return false;
    const double a00 = r.a1.x, a01 = r.a1.y, a10 = r.a1.z, a11 = r.a1.w;
    const double b00 = r.a2.x, b01 = r.a2.y, b10 = r.a2.z, b11 = r.a2.w;
    const double det1 = a00 * a11 - a01 * a10, det2 = b00 * b11 - b01 * b10;
    if (det1 == 0.0 || det2 == 0.0) return false;
    double j[4], n1, n2, w;
    lin_h(G, r.c.z, r.c.w, j, n1, n2, w);
    const double e00 = j[0] * b00 + j[1] * b10, e01 = j[0] * b01 + j[1] * b11, e10 = j[2] * b00 + j[3] * b10, e11 = j[2] * b01 + j[3] * b11;
    const double i00 = a11 / det1, i01 = -a01 / det1, i10 = -a10 / det1, i11 = a00 / det1;
    const double d00 = (i00 * e00 + i01 * e10) - 1.0, m01 = i00 * e01 + i01 * e11, m10 = i10 * e00 + i11 * e10;
    const double d11 = (i10 * e01 + i11 * e11) - 1.0;
    D = ((d00 * d00 + m01 * m01) + m10 * m10) + d11 * d11;
    return true;
}

// Affine inlier: is_inlier(H) at the centres, finite non-singular frames and D <= laf_th (G = adj(H)).
__device__ __forceinline__ bool is_inlier_ac(const double* H, const double* G, const AcRow& r, double th2, double laf_th) {
    if (!is_inlier(H, r.c, th2)) return false;
    double D;
    return frame_distance(G, r, D) && D <= laf_th;
}

// Hypothesis from 2 affine correspondences, fp64 in this order; false for a degenerate sample.
//  - Degenerate: a non-finite centre or frame, coincident centres in either image, det A1 or det A2 = 0, det(A2 A1^-1) of different
//    signs for the two ACs (the counterpart of the 4-point mixed-orientation rule), a Cholesky pivot <= CHOL_EPS times its diagonal entry,
//    or a non-finite H.
//  - Each image's two centres are Hartley-normalised: midpoint c and scale s = sqrt(2 / var), var = (d / 2)^2 (refit's, for two points).
//  - In normalised coordinates AC k gives A_n = (s2 / s1) A2 A1^-1 and 6 equations linear in (h11 .. h32) with h33 = 1: the 2 point
//    equations and the 4 of dx'/dx = A_n, e.g. h11 - (u' + a11 u) h31 - a11 v h32 = a11.  Fixing h33 = 1 is safe: Hn[2][2] is the w of H
//    at the image-1 midpoint, and w > 0 at both sample points (both visible under H) makes it positive at their midpoint.
//  - The 12 x 8 system is solved by least squares: normal equations (upper triangle, accumulated row by row), Cholesky, forward and back
//    substitution; then H = T2^-1 Hn T1 and normalise_h.
__device__ bool ac_homography(const AcRow (&a)[2], double* H) {
    double d1[2], d2[2];
#pragma unroll
    for (int k = 0; k < 2; k++) {
        if (!finite4(a[k].c) || !finite4(a[k].a1) || !finite4(a[k].a2)) return false;
        d1[k] = (double)a[k].a1.x * a[k].a1.w - (double)a[k].a1.y * a[k].a1.z;
        d2[k] = (double)a[k].a2.x * a[k].a2.w - (double)a[k].a2.y * a[k].a2.z;
        if (d1[k] == 0.0 || d2[k] == 0.0) return false;
    }
    if (((d1[0] > 0.0) == (d2[0] > 0.0)) != ((d1[1] > 0.0) == (d2[1] > 0.0))) return false;
    const double c1x = ((double)a[0].c.x + a[1].c.x) * 0.5, c1y = ((double)a[0].c.y + a[1].c.y) * 0.5;
    const double c2x = ((double)a[0].c.z + a[1].c.z) * 0.5, c2y = ((double)a[0].c.w + a[1].c.w) * 0.5;
    const double h1x = ((double)a[1].c.x - a[0].c.x) * 0.5, h1y = ((double)a[1].c.y - a[0].c.y) * 0.5;
    const double h2x = ((double)a[1].c.z - a[0].c.z) * 0.5, h2y = ((double)a[1].c.w - a[0].c.w) * 0.5;
    const double var1 = h1x * h1x + h1y * h1y, var2 = h2x * h2x + h2y * h2y;
    if (!(var1 > 0.0) || !(var2 > 0.0)) return false;
    const double s1 = sqrt(2.0 / var1), s2 = sqrt(2.0 / var2), rs = s2 / s1;
    double N[8][8], b[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        b[k] = 0.0;
#pragma unroll
        for (int l = 0; l < 8; l++) N[k][l] = 0.0;
    }
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const double u = (a[k].c.x - c1x) * s1, v = (a[k].c.y - c1y) * s1, up = (a[k].c.z - c2x) * s2, vp = (a[k].c.w - c2y) * s2;
        const double p00 = a[k].a1.x, p01 = a[k].a1.y, p10 = a[k].a1.z, p11 = a[k].a1.w;
        const double q00 = a[k].a2.x, q01 = a[k].a2.y, q10 = a[k].a2.z, q11 = a[k].a2.w;
        const double i00 = p11 / d1[k], i01 = -p01 / d1[k], i10 = -p10 / d1[k], i11 = p00 / d1[k];
        const double n00 = (q00 * i00 + q01 * i10) * rs, n01 = (q00 * i01 + q01 * i11) * rs;
        const double n10 = (q10 * i00 + q11 * i10) * rs, n11 = (q10 * i01 + q11 * i11) * rs;
        const double rows[6][9] = {{u, v, 1.0, 0.0, 0.0, 0.0, -(up * u), -(up * v), up},
                                   {0.0, 0.0, 0.0, u, v, 1.0, -(vp * u), -(vp * v), vp},
                                   {1.0, 0.0, 0.0, 0.0, 0.0, 0.0, -(up + n00 * u), -(n00 * v), n00},
                                   {0.0, 1.0, 0.0, 0.0, 0.0, 0.0, -(n01 * u), -(up + n01 * v), n01},
                                   {0.0, 0.0, 0.0, 1.0, 0.0, 0.0, -(vp + n10 * u), -(n10 * v), n10},
                                   {0.0, 0.0, 0.0, 0.0, 1.0, 0.0, -(n11 * u), -(vp + n11 * v), n11}};
#pragma unroll
        for (int e = 0; e < 6; e++)
#pragma unroll
            for (int i = 0; i < 8; i++) {
                b[i] = b[i] + rows[e][i] * rows[e][8];
#pragma unroll
                for (int l = i; l < 8; l++) N[i][l] = N[i][l] + rows[e][i] * rows[e][l];
            }
    }
    // Cholesky N = L L' (L in the lower triangle of N; N's upper triangle stays), then L z = b and L' h = z
    double dg[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        double d = N[j][j];
#pragma unroll
        for (int k = 0; k < j; k++) d = d - N[j][k] * N[j][k];
        if (!(d > CHOL_EPS * N[j][j])) return false;
        dg[j] = sqrt(d);
#pragma unroll
        for (int i = j + 1; i < 8; i++) {
            double t = N[j][i];
#pragma unroll
            for (int k = 0; k < j; k++) t = t - N[i][k] * N[j][k];
            N[i][j] = t / dg[j];
        }
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        double t = b[i];
#pragma unroll
        for (int k = 0; k < i; k++) t = t - N[i][k] * b[k];
        b[i] = t / dg[i];
    }
#pragma unroll
    for (int i = 7; i >= 0; i--) {
        double t = b[i];
#pragma unroll
        for (int k = i + 1; k < 8; k++) t = t - N[k][i] * b[k];
        b[i] = t / dg[i];
    }
    const double Hn[9] = {b[0], b[1], b[2], b[3], b[4], b[5], b[6], b[7], 1.0};
    return denormalise_h({c1x, c1y, s1, c2x, c2y, s2}, Hn, H);
}

// The local optimisation of a chunk's winner (in s.H and Hl, shared) that raised the so-far-best count: the refit rounds on s.H, and
// from Hl the shrinking-threshold refits (LO_FACTOR, LO_STEPS; stopping at fewer than 4 inliers or a failed refit) followed by the refit
// rounds.  s.H ends as the second result when its count is higher, else the first.  `inl` is scratch.  Block-wide; returns the count.
__device__ int ac_local_opt(const float* L1, const float* L2, const int* tent, int n, double th2, double laf_th, unsigned char* inl,
                            double* Hl, RansacShared& s) {
    const int c0 = refit_rounds<false, true>(L1, L2, tent, n, th2, inl, s.H, s, laf_th);
    double f = LO_FACTOR;
    for (int k = 0; k < LO_STEPS; k++) {
        const int c = score_rows<false, true>(Hl, L1, L2, tent, n, th2 * (f * f), inl, s, laf_th * f);
        if (c < 4 || !refit(L1, L2, tent, n, inl, s)) break;   // c is the block total: uniform
        if (threadIdx.x < 9) Hl[threadIdx.x] = s.Hr[threadIdx.x];
        __syncthreads();
        f = f * 0.5;
    }
    const int c1 = refit_rounds<false, true>(L1, L2, tent, n, th2, inl, Hl, s, laf_th);
    if (c1 <= c0) return c0;
    if (threadIdx.x < 9) s.H[threadIdx.x] = Hl[threadIdx.x];
    __syncthreads();
    return c1;
}

// ransac_kernel's search with 2-AC samples and the affine inlier test, and ac_local_opt each time a chunk's winner raises the
// so-far-best count.  Rows go through RansacShared's tile as AcRow, ATILE at a time.
__global__ void __launch_bounds__(VT) ac_ransac_kernel(const float* __restrict__ lafs1, int S1, int cap1, const float* __restrict__ lafs2,
                                                       int S2, int cap2, const int* __restrict__ pairs, const int* __restrict__ tent_all,
                                                       const int* __restrict__ ntent, int tcap, double th2, double laf_th, double log1mconf,
                                                       int max_iters, uint64_t seed, float* __restrict__ Hout, unsigned char* __restrict__ inl_all,
                                                       int* __restrict__ ninl, int* __restrict__ iters) {
    __shared__ RansacShared s;
    __shared__ double Hl[9];   // ac_local_opt's second model
    AcRow* tile = reinterpret_cast<AcRow*>(s.tile);
    const int tid = threadIdx.x;
    const int* tent;
    const float *L1, *L2;
    int n;
    if (!verify_pair(lafs1, S1, cap1, lafs2, S2, cap2, pairs, tent_all, ntent, tcap, ninl, n, tent, L1, L2)) return;
    unsigned char* inl = inl_all + (size_t)blockIdx.x * tcap;
    int best = 0, h_done = 0;
    if (n >= 2) {
        const int ntiles = (n + ATILE - 1) / ATILE;
        for (int h0 = 0;; h0 += VT) {
            const int h = h0 + tid;
            double H[9], G[9];
            int idx[2];
            bool ok = h < max_iters && draw_sample(seed, h, n, idx);
            if (ok) {
                const AcRow a[2] = {tent_ac(L1, L2, tent, idx[0]), tent_ac(L1, L2, tent, idx[1])};
                ok = ac_homography(a, H);
            }
            if (ok) adj3(H, G);
            int cnt = 0;
            for (int tb = 0; tb < ntiles; tb++) {
                const int t0 = tb * ATILE, m = min(ATILE, n - t0);
                if (ntiles > 1 || h0 == 0) {
                    __syncthreads();
                    for (int t = tid; t < m; t += VT) tile[t] = tent_ac(L1, L2, tent, t0 + t);
                    __syncthreads();
                }
                if (ok)
                    for (int t = 0; t < m; t++) cnt += is_inlier_ac(H, G, tile[t], th2, laf_th);
            }
            // best of the chunk: highest count, then lowest h
            const unsigned long long mine = ok ? ((unsigned long long)cnt << 32) | (unsigned)~(unsigned)h : 0ull;
            const unsigned long long bk = block_max_key(mine, s.key);
            const int bc = (int)(bk >> 32);
            if (bk != 0 && bc > best) {
                if (mine == bk) {
#pragma unroll
                    for (int k = 0; k < 9; k++) s.H[k] = Hl[k] = H[k];
                }
                __syncthreads();
                // local optimisation: a 2-AC hypothesis is noisier than a 4-point one; the point-DLT refits bring it to their accuracy
                best = ac_local_opt(L1, L2, tent, n, th2, laf_th, inl, Hl, s);
            }
            h_done = min(h0 + VT, max_iters);
            double need;   // adaptive number of samples for `confidence`
            const double pr = (double)best / (double)n, p2 = pr * pr;
            if (p2 >= 1.0) need = 0.0;
            else if (p2 <= 0.0) need = INFINITY;
            else need = ceil(log1mconf / log(1.0 - p2));
            __syncthreads();
            if ((double)h_done >= fmin(need, (double)max_iters)) break;
        }
    }
    finish_ransac<false, true>(L1, L2, tent, n, th2, best, h_done, inl, s, Hout, ninl, iters, laf_th);
}

int verify_args(const char* fn, const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                const int* d_tent, const int* d_ntent, int tcap) {
    const char* msg = nullptr;
    if (!d_lafs1 || !d_lafs2 || !d_tent || !d_ntent) msg = "NULL LAFs or tentatives";
    else if (S1 < 1 || S2 < 1 || cap1 < 1 || cap2 < 1 || P < 1) msg = "S1, S2, cap1, cap2 and P must be >= 1";
    else if (!d_pairs && (S1 != S2 || P != S1)) msg = "d_pairs == NULL (pair p = (p, p)) needs S1 == S2 == P";
    else if (tcap < 1 || tcap > MAX_TCAP) msg = "tcap must be in 1..4194240";
    if (!msg) return AG_OK;
    set_error("%s: %s", fn, msg);
    return AG_ERR_INVALID;
}

// The RANSAC entry points' outputs and search parameters (M: the model output, H or F).
int ransac_args(const char* fn, const float* d_M, const unsigned char* d_inl, const int* d_ninl, float inl_th, float confidence,
                int max_iters) {
    const char* msg = nullptr;
    if (!d_M || !d_inl || !d_ninl) msg = "NULL output";
    else if (!(inl_th > 0.f && isfinite(inl_th))) msg = "inl_th must be finite and > 0";
    else if (!(confidence > 0.f && confidence < 1.f)) msg = "confidence must be in (0, 1)";
    else if (!(max_iters >= 1 && max_iters <= 0x7fffffff - VT)) msg = "max_iters must be >= 1";
    if (!msg) return AG_OK;
    set_error("%s: %s", fn, msg);
    return AG_ERR_INVALID;
}

// ag_fundamental_ransac (DEGEN false) and ag_fundamental_degensac, named fn.
template <bool DEGEN>
int fundamental_ransac(const char* fn, const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                       const int* d_tent, const int* d_ntent, int tcap, float inl_th, float confidence, int max_iters, unsigned long long seed,
                       float* d_F, unsigned char* d_inl, int* d_ninl, int* d_iters, void* stream) {
    int rc = verify_args(fn, d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, P, d_tent, d_ntent, tcap);
    if (rc || (rc = ransac_args(fn, d_F, d_inl, d_ninl, inl_th, confidence, max_iters))) return rc;
    const double th = inl_th;
    fransac_kernel<DEGEN><<<P, VT, 0, (cudaStream_t)stream>>>(d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, d_tent, d_ntent, tcap, th * th,
                                                              log(1.0 - (double)confidence), max_iters, (uint64_t)seed, d_F, d_inl, d_ninl,
                                                              d_iters);
    AG_CHECK_LAUNCH(DEGEN ? "fransac_kernel<DEGEN>" : "fransac_kernel");
    return AG_OK;
}

}  // namespace ag

using namespace ag;

extern "C" {

int ag_homography_ransac(const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                         const int* d_tent, const int* d_ntent, int tcap, float inl_th, float confidence, int max_iters, unsigned long long seed,
                         float* d_H, unsigned char* d_inl, int* d_ninl, int* d_iters, void* stream) {
    const char* fn = "ag_homography_ransac";
    int rc = verify_args(fn, d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, P, d_tent, d_ntent, tcap);
    if (rc || (rc = ransac_args(fn, d_H, d_inl, d_ninl, inl_th, confidence, max_iters))) return rc;
    const double th = inl_th;
    ransac_kernel<<<P, VT, 0, (cudaStream_t)stream>>>(d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, d_tent, d_ntent, tcap, th * th,
                                                      log(1.0 - (double)confidence), max_iters, (uint64_t)seed, d_H, d_inl, d_ninl, d_iters);
    AG_CHECK_LAUNCH("ransac_kernel");
    return AG_OK;
}

int ag_homography_ransac_affine(const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                                const int* d_tent, const int* d_ntent, int tcap, float inl_th, float laf_th, float confidence, int max_iters,
                                unsigned long long seed, float* d_H, unsigned char* d_inl, int* d_ninl, int* d_iters, void* stream) {
    const char* fn = "ag_homography_ransac_affine";
    int rc = verify_args(fn, d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, P, d_tent, d_ntent, tcap);
    if (rc || (rc = ransac_args(fn, d_H, d_inl, d_ninl, inl_th, confidence, max_iters))) return rc;
    AG_REQUIRE(laf_th > 0.f, "laf_th must be > 0 (and not NaN)");
    const double th = inl_th;
    ac_ransac_kernel<<<P, VT, 0, (cudaStream_t)stream>>>(d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, d_tent, d_ntent, tcap, th * th,
                                                         (double)laf_th, log(1.0 - (double)confidence), max_iters, (uint64_t)seed, d_H, d_inl,
                                                         d_ninl, d_iters);
    AG_CHECK_LAUNCH("ac_ransac_kernel");
    return AG_OK;
}

int ag_fundamental_ransac(const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                          const int* d_tent, const int* d_ntent, int tcap, float inl_th, float confidence, int max_iters, unsigned long long seed,
                          float* d_F, unsigned char* d_inl, int* d_ninl, int* d_iters, void* stream) {
    return fundamental_ransac<false>("ag_fundamental_ransac", d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, P, d_tent, d_ntent, tcap, inl_th,
                                     confidence, max_iters, seed, d_F, d_inl, d_ninl, d_iters, stream);
}

int ag_fundamental_degensac(const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                            const int* d_tent, const int* d_ntent, int tcap, float inl_th, float confidence, int max_iters, unsigned long long seed,
                            float* d_F, unsigned char* d_inl, int* d_ninl, int* d_iters, void* stream) {
    return fundamental_ransac<true>("ag_fundamental_degensac", d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, P, d_tent, d_ntent, tcap, inl_th,
                                    confidence, max_iters, seed, d_F, d_inl, d_ninl, d_iters, stream);
}

int ag_gt_correspondences_pairs(const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                                const int* d_tent, const int* d_ntent, int tcap, const float* d_H1to2, float dist_threshold,
                                float* d_min_dist, int* d_idx2, int* d_true, int* d_ntrue, void* stream) {
    int rc = verify_args("ag_gt_correspondences_pairs", d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, P, d_tent, d_ntent, tcap);
    if (rc) return rc;
    AG_REQUIRE(d_H1to2 && d_min_dist && d_idx2 && d_true && d_ntrue, "NULL homography or output");
    AG_REQUIRE(dist_threshold >= 0.f, "dist_threshold must be >= 0 (and not NaN)");
    gt_kernel<<<P, VT, 0, (cudaStream_t)stream>>>(d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, d_tent, d_ntent, tcap, d_H1to2, dist_threshold,
                                                  d_min_dist, d_idx2, d_true, d_ntrue);
    AG_CHECK_LAUNCH("gt_kernel");
    return AG_OK;
}

static int frobenius_params(const ag_frobenius_params_t* prm) {
    AG_REQUIRE(prm, "NULL parameters");
    AG_REQUIRE(prm->dist_threshold >= 0.f, "dist_threshold must be >= 0 (and not NaN)");
    AG_REQUIRE(prm->center_dist_th >= 0.f, "center_dist_th must be >= 0 (and not NaN)");
    AG_REQUIRE(prm->scale_diff_coef == prm->scale_diff_coef, "scale_diff_coef must not be NaN");
    return AG_OK;
}

int ag_gt_frobenius_pairs(const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                          const int* d_tent, const int* d_ntent, int tcap, const float* d_H1to2, const ag_frobenius_params_t* prm,
                          float* d_min_dist, int* d_idx2, int* d_true, int* d_ntrue, void* stream) {
    int rc = verify_args("ag_gt_frobenius_pairs", d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, P, d_tent, d_ntent, tcap);
    if (rc) return rc;
    AG_REQUIRE(d_H1to2 && d_min_dist && d_idx2 && d_true && d_ntrue, "NULL homography or output");
    if ((rc = frobenius_params(prm))) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    frob_pass_kernel<true><<<dim3(P, cdiv(tcap, FRO_NT)), FRO_NT, 0, st>>>(d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, d_tent, d_ntent,
                                                                          nullptr, tcap, d_H1to2, *prm, d_min_dist, d_idx2);
    AG_CHECK_LAUNCH("frob_pass_kernel");
    frob_compact_kernel<true><<<P, VT, 0, st>>>(S1, cap1, S2, cap2, d_pairs, d_tent, d_ntent, nullptr, tcap, prm->dist_threshold, d_min_dist,
                                                d_true, d_ntrue);
    AG_CHECK_LAUNCH("frob_compact_kernel");
    return AG_OK;
}

int ag_gt_frobenius_sets(const float* d_lafs1, int S1, int cap1, const int* d_count1, const float* d_lafs2, int S2, int cap2,
                         const int* d_count2, const int* d_pairs, int P, const float* d_H1to2, const ag_frobenius_params_t* prm,
                         float* d_min_dist, int* d_idx2, int* d_true, int* d_ntrue, void* stream) {
    AG_REQUIRE(d_lafs1 && d_lafs2 && d_count1 && d_count2, "NULL LAFs or counts");
    AG_REQUIRE(S1 >= 1 && S2 >= 1 && cap1 >= 1 && cap2 >= 1 && P >= 1, "S1, S2, cap1, cap2 and P must be >= 1");
    AG_REQUIRE(d_pairs || (S1 == S2 && P == S1), "d_pairs == NULL (pair p = (p, p)) needs S1 == S2 == P");
    AG_REQUIRE(cap1 <= MAX_TCAP, "cap1 must be <= 4194240");
    AG_REQUIRE(d_H1to2 && d_min_dist && d_idx2 && d_true && d_ntrue, "NULL homography or output");
    int rc = frobenius_params(prm);
    if (rc) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    frob_pass_kernel<false><<<dim3(P, cdiv(cap1, FRO_NT)), FRO_NT, 0, st>>>(d_lafs1, S1, cap1, d_lafs2, S2, cap2, d_pairs, nullptr, d_count1,
                                                                           d_count2, cap1, d_H1to2, *prm, d_min_dist, d_idx2);
    AG_CHECK_LAUNCH("frob_pass_kernel");
    frob_compact_kernel<false><<<P, VT, 0, st>>>(S1, cap1, S2, cap2, d_pairs, nullptr, d_count1, d_count2, cap1, prm->dist_threshold,
                                                 d_min_dist, d_true, d_ntrue);
    AG_CHECK_LAUNCH("frob_compact_kernel");
    return AG_OK;
}

int ag_reproject_lafs(const float* d_lafs, int S, int cap, const float* d_H, int invert, int up_is_up, float* d_out, void* stream) {
    AG_REQUIRE(d_lafs && d_H && d_out, "NULL LAFs, homography or output");
    AG_REQUIRE(S >= 1 && S <= 65535 && cap >= 1, "S must be in 1..65535 and cap >= 1");
    reproject_lafs_kernel<<<dim3(cdiv(cap, VT), S), VT, 0, (cudaStream_t)stream>>>(d_lafs, cap, d_H, invert, up_is_up, d_out);
    AG_CHECK_LAUNCH("reproject_lafs_kernel");
    return AG_OK;
}

}  // extern "C"
