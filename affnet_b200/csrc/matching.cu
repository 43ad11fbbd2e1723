// Descriptor matching right after the hot path (SURVEY.md §8(f) row 3): distance_matrix_vector (Losses.py:5-13) and the
// second-nearest-neighbour ratio test of train_AffNet_test_on_graffity.py:292-298, including its quirk: before the second
// minimum is taken, EVERY column that is the nearest neighbour of ANY row is set to 100000 (`dist_matrix[:, idxs_in_2] = 100000`).
// fp32 FFMA throughout: the ratio test is a decision, and fp16 / bf16 / TF32 operand rounding would move distances at near-ties.
//
// The matcher (ag_match_pairs, and ag_match_snn as its one-pair case) never stores the n1 x n2 distance matrix: two passes recompute
// the distance tiles, the first for the nearest neighbour and the column mask, the second for the masked second minimum.
#include "common.cuh"

namespace ag {

constexpr int MT = 64, MK = 16;

// The one per-element distance of the library: sqrt((|a|^2 + |b|^2 - 2 a.b) + 1e-6) with non-contracted rounding steps.  Both
// dist_matrix_kernel and the matcher's passes call it, so ag_distance_matrix and the matcher agree bit for bit by construction.
__device__ __forceinline__ float snn_dist(float na, float nb, float acc) {
    return sqrtf(__fadd_rn(__fsub_rn(__fadd_rn(na, nb), __fmul_rn(2.0f, acc)), 1e-6f));
}

// dist[i][j] = sqrt((|a_i|^2 + |b_j|^2 - 2 a_i.b_j) + 1e-6)
__global__ void __launch_bounds__(256) dist_matrix_kernel(const float* __restrict__ a, int n1, const float* __restrict__ b, int n2, int D,
                                                           float* __restrict__ out) {
    __shared__ float sa[MK][MT + 1], sb[MK][MT + 1];
    const int i0 = blockIdx.y * MT, j0 = blockIdx.x * MT;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;   // 16 x 16 threads, 4 x 4 outputs each
    float acc[4][4] = {}, na[4] = {}, nb[4] = {};
    for (int k0 = 0; k0 < D; k0 += MK) {
        for (int t = threadIdx.x; t < MT * MK; t += 256) {
            const int r = t / MK, k = t - r * MK;
            sa[k][r] = (i0 + r < n1 && k0 + k < D) ? a[(size_t)(i0 + r) * D + k0 + k] : 0.f;
            sb[k][r] = (j0 + r < n2 && k0 + k < D) ? b[(size_t)(j0 + r) * D + k0 + k] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < MK; k++) {
            float va[4], vb[4];
#pragma unroll
            for (int q = 0; q < 4; q++) { va[q] = sa[k][ty * 4 + q]; vb[q] = sb[k][tx * 4 + q]; }
#pragma unroll
            for (int q = 0; q < 4; q++) {
                na[q] = fmaf(va[q], va[q], na[q]); nb[q] = fmaf(vb[q], vb[q], nb[q]);
#pragma unroll
                for (int p = 0; p < 4; p++) acc[q][p] = fmaf(va[q], vb[p], acc[q][p]);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < 4; q++)
#pragma unroll
        for (int p = 0; p < 4; p++) {
            const int i = i0 + ty * 4 + q, j = j0 + tx * 4 + p;
            if (i < n1 && j < n2) out[(size_t)i * n2 + j] = snn_dist(na[q], nb[p], acc[q][p]);
        }
}

// ---- batched SNN matcher ------------------------------------------------------------------------------------------------------------
// Pair p = (image i of set 1, image j of set 2) -> its row counts.  Returns -1 for a pair the caller cannot match (an index out of range,
// a count of -1 from the pipeline's candidate overflow or any other count outside 0..cap), 0 when either image has no rows, else n1.
__device__ __forceinline__ int pair_rows(const int* __restrict__ pairs, int p, const int* __restrict__ c1, int S1, int cap1,
                                         const int* __restrict__ c2, int S2, int cap2, int& i, int& j, int& n1, int& n2) {
    i = pairs ? pairs[2 * (size_t)p] : p;
    j = pairs ? pairs[2 * (size_t)p + 1] : p;
    if (i < 0 || i >= S1 || j < 0 || j >= S2) return -1;
    n1 = c1 ? c1[i] : cap1;
    n2 = c2 ? c2[j] : cap2;
    if (n1 < 0 || n1 > cap1 || n2 < 0 || n2 > cap2) return -1;
    return (n1 == 0 || n2 == 0) ? 0 : n1;
}

// |x|^2 of every valid descriptor row of both sets: the fmaf chain over k ascending from +0 that dist_matrix_kernel runs (its zero
// padding of k adds exact zeros).  Rows at or beyond their image's count are skipped.
__global__ void __launch_bounds__(256) row_norms_kernel(const float* __restrict__ d1, const int* __restrict__ c1, int cap1, long long rows1,
                                                         const float* __restrict__ d2, const int* __restrict__ c2, int cap2, long long rows2,
                                                         int D, float* __restrict__ norm1, float* __restrict__ norm2) {
    long long r = blockIdx.x * 256ll + threadIdx.x;
    const float* d = d1;
    const int* c = c1;
    int cap = cap1;
    float* out = norm1;
    if (r >= rows1) {
        r -= rows1;
        if (r >= rows2) return;
        d = d2; c = c2; cap = cap2; out = norm2;
    }
    const long long s = r / cap;
    if (c && r - s * cap >= c[s]) return;
    const float* x = d + r * D;
    float acc = 0.f;
    for (int k = 0; k < D; k++) acc = fmaf(x[k], x[k], acc);
    out[r] = acc;
}

constexpr int BM = 64, BN = 64, BK = 16, SPAD = 4;   // CTA tile: 64 set-1 rows x 64 set-2 columns, k in chunks of 16

__device__ __forceinline__ void cp_async4(float* smem, const float* gmem, bool pred) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem), "r"(pred ? 4 : 0)
                 : "memory");
}

// One pass over the distance tiles of every pair.  Grid (pair, row tile): a CTA holds 64 rows of image i of set 1 and streams the
// column tiles of image j of set 2 through shared memory (cp.async, double-buffered); 16 x 16 threads, 4 x 4 distances each.
//   PASS 1: running (min, lowest arg-min) per row, NaN ignored; writes d_min / d_idx2 and marks the arg-min column in the pair's mask.
//   PASS 2: fminf over the columns of (masked ? 100000 : dist); writes d_second and d_keep.
template <int PASS>
__global__ void __launch_bounds__(256) snn_pass_kernel(const float* __restrict__ d1, const int* __restrict__ c1, int S1, int cap1,
                                                        const float* __restrict__ d2, const int* __restrict__ c2, int S2, int cap2, int D,
                                                        const int* __restrict__ pairs, const float* __restrict__ norm1,
                                                        const float* __restrict__ norm2, unsigned char* __restrict__ colmask, float ratio,
                                                        int* __restrict__ idx2, float* __restrict__ mn, float* __restrict__ second,
                                                        unsigned char* __restrict__ keep) {
    __shared__ __align__(16) float sa[2][BK][BM + SPAD], sb[2][BK][BN + SPAD];
    const int p = blockIdx.x;
    int i, j, n1, n2;
    if (pair_rows(pairs, p, c1, S1, cap1, c2, S2, cap2, i, j, n1, n2) <= 0) return;
    const int r0 = blockIdx.y * BM;
    if (r0 >= n1) return;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const float* A = d1 + ((size_t)i * cap1 + r0) * D;
    const float* B = d2 + (size_t)j * cap2 * D;
    unsigned char* mask = colmask + (size_t)p * cap2;
    const int nk = (D + BK - 1) / BK, ns = (n2 + BN - 1) / BN * nk, arows = min(BM, n1 - r0);

    auto load = [&](int s, int buf) {
        const int t = s / nk, k0 = (s - t * nk) * BK, c0 = t * BN;
#pragma unroll
        for (int u = 0; u < (BM * BK) / 256; u++) {
            const int e = threadIdx.x + 256 * u, r = e / BK, k = e % BK;
            const bool kin = k0 + k < D, pa = kin && r < arows, pb = kin && c0 + r < n2;
            cp_async4(&sa[buf][k][r], pa ? A + (size_t)r * D + k0 + k : A, pa);
            cp_async4(&sb[buf][k][r], pb ? B + (size_t)(c0 + r) * D + k0 + k : B, pb);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    float na[4], best[4], acc[4][4];
    int bj[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const int r = r0 + ty * 4 + q;
        na[q] = r < n1 ? norm1[(size_t)i * cap1 + r] : 0.f;
        best[q] = INFINITY;
        bj[q] = 0x7fffffff;   // stays so only when the row saw nothing below +inf (e.g. a row of NaNs): resolved to column 0 below
#pragma unroll
        for (int c = 0; c < 4; c++) acc[q][c] = 0.f;
    }
    load(0, 0);
    for (int s = 0; s < ns; s++) {
        const int buf = s & 1;
        if (s + 1 < ns) {
            load(s + 1, buf ^ 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; k++) {
            const float4 va = *reinterpret_cast<const float4*>(&sa[buf][k][ty * 4]);
            const float4 vb = *reinterpret_cast<const float4*>(&sb[buf][k][tx * 4]);
            const float a4[4] = {va.x, va.y, va.z, va.w}, b4[4] = {vb.x, vb.y, vb.z, vb.w};
#pragma unroll
            for (int q = 0; q < 4; q++)
#pragma unroll
                for (int c = 0; c < 4; c++) acc[q][c] = fmaf(a4[q], b4[c], acc[q][c]);
        }
        __syncthreads();   // buffer `buf` is refilled by the load issued in the next iteration
        if ((s + 1) % nk == 0) {   // the tile's k loop is complete: fold its distances into the row state
            const int c0 = (s / nk) * BN + tx * 4;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int jc = c0 + c;
                if (jc < n2) {
                    const float nb = norm2[(size_t)j * cap2 + jc];
                    const bool marked = PASS == 2 && mask[jc];
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        const float v = snn_dist(na[q], nb, acc[q][c]);
                        if (PASS == 1) {
                            if (v < best[q]) { best[q] = v; bj[q] = jc; }   // columns arrive in ascending order: the first minimum stays
                        } else {
                            best[q] = fminf(best[q], marked ? 100000.0f : v);
                        }
                    }
                }
#pragma unroll
                for (int q = 0; q < 4; q++) acc[q][c] = 0.f;
            }
        }
    }
    // the 16 threads of a row are 16 consecutive lanes of one half-warp
#pragma unroll
    for (int q = 0; q < 4; q++) {
        for (int o = 8; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best[q], o);
            if (PASS == 1) {
                const int oj = __shfl_xor_sync(0xffffffffu, bj[q], o);
                if (ov < best[q] || (ov == best[q] && oj < bj[q])) { best[q] = ov; bj[q] = oj; }
            } else {
                best[q] = fminf(best[q], ov);
            }
        }
        const int r = r0 + ty * 4 + q;
        if (tx == 0 && r < n1) {
            const size_t o = (size_t)p * cap1 + r;
            if (PASS == 1) {
                const int col = (bj[q] < 0 || bj[q] >= n2) ? 0 : bj[q];
                mn[o] = best[q]; idx2[o] = col;
                mask[col] = 1;   // every CTA of the pair that marks a column stores the same value: no atomics needed
            } else {
                second[o] = best[q];
                keep[o] = (__fdiv_rn(mn[o], __fadd_rn(best[q], 1e-8f)) <= ratio) ? 1 : 0;
            }
        }
    }
}

// One CTA per pair: ordered compaction of the kept rows into (row, idx2[row]) and their number; -1 / 0 for invalid / empty pairs.
__global__ void __launch_bounds__(256) snn_compact_kernel(const int* __restrict__ pairs, const int* __restrict__ c1, int S1, int cap1,
                                                           const int* __restrict__ c2, int S2, int cap2, const unsigned char* __restrict__ keep,
                                                           const int* __restrict__ idx2, int* __restrict__ tent, int* __restrict__ ntent) {
    __shared__ int wsum[8];
    const int p = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int i, j, n1, n2;
    const int v = pair_rows(pairs, p, c1, S1, cap1, c2, S2, cap2, i, j, n1, n2);
    if (v <= 0) {
        if (threadIdx.x == 0 && ntent) ntent[p] = v;
        return;
    }
    const size_t base = (size_t)p * cap1;
    int run = 0;
    for (int r0 = 0; r0 < n1; r0 += 256) {
        const int r = r0 + threadIdx.x;
        const bool k = r < n1 && keep[base + r];
        const unsigned b = __ballot_sync(0xffffffffu, k);
        if (lane == 0) wsum[warp] = __popc(b);
        __syncthreads();
        int off = run, tot = 0;
#pragma unroll
        for (int w = 0; w < 8; w++) {
            off += w < warp ? wsum[w] : 0;
            tot += wsum[w];
        }
        if (k && tent) {
            const size_t o = base + off + __popc(b & ((1u << lane) - 1u));
            tent[2 * o] = r;
            tent[2 * o + 1] = idx2[base + r];
        }
        run += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0 && ntent) ntent[p] = run;
}

}  // namespace ag

using namespace ag;

extern "C" {

int ag_distance_matrix(const float* d_a, int n1, const float* d_b, int n2, int dim, float* d_out, void* stream) {
    AG_REQUIRE(d_a && d_b && d_out && n1 >= 1 && n2 >= 1 && dim >= 1, "bad arguments");
    dist_matrix_kernel<<<dim3(cdiv(n2, MT), cdiv(n1, MT)), 256, 0, (cudaStream_t)stream>>>(d_a, n1, d_b, n2, dim, d_out);
    AG_CHECK_LAUNCH("dist_matrix_kernel");
    return AG_OK;
}

size_t ag_match_pairs_workspace_bytes(int S1, int cap1, int S2, int cap2, int P) {
    if (S1 < 1 || cap1 < 1 || S2 < 1 || cap2 < 1 || P < 1) return 0;
    return align_up((size_t)S1 * cap1 * sizeof(float), 256) + align_up((size_t)S2 * cap2 * sizeof(float), 256) + align_up((size_t)P * cap2, 256);
}

int ag_match_pairs(const float* d_desc1, const int* d_count1, int S1, int cap1, const float* d_desc2, const int* d_count2, int S2, int cap2,
                   int dim, const int* d_pairs, int P, float ratio, void* d_ws, size_t ws_bytes, int* d_idx2, float* d_min, float* d_second,
                   unsigned char* d_keep, int* d_tent, int* d_ntent, void* stream) {
    AG_REQUIRE(d_desc1 && d_desc2 && d_ws && d_idx2 && d_min && d_second && d_keep, "NULL descriptors, workspace or output");
    AG_REQUIRE(dim >= 1 && S1 >= 1 && S2 >= 1 && cap1 >= 1 && cap2 >= 1 && P >= 1, "dim, S1, S2, cap1, cap2 and P must be >= 1");
    AG_REQUIRE(d_pairs || (S1 == S2 && P == S1), "d_pairs == NULL (pair p = (p, p)) needs S1 == S2 == P");
    AG_REQUIRE(cdiv(cap1, BM) <= 65535, "cap1 above 4194240 rows");
    const size_t need = ag_match_pairs_workspace_bytes(S1, cap1, S2, cap2, P);
    if (ws_bytes < need) {
        set_error("ag_match_pairs: workspace too small (%zu bytes, needs %zu)", ws_bytes, need);
        return AG_ERR_CAPACITY;
    }
    cudaStream_t st = (cudaStream_t)stream;
    float* norm1 = (float*)d_ws;
    float* norm2 = (float*)((char*)d_ws + align_up((size_t)S1 * cap1 * sizeof(float), 256));
    unsigned char* colmask = (unsigned char*)norm2 + align_up((size_t)S2 * cap2 * sizeof(float), 256);
    int rc = check_cuda(cudaMemsetAsync(colmask, 0, (size_t)P * cap2, st), "ag_match_pairs: memset column masks");
    if (rc) return rc;
    const long long rows1 = (long long)S1 * cap1, rows2 = (long long)S2 * cap2;
    row_norms_kernel<<<(unsigned)((rows1 + rows2 + 255) / 256), 256, 0, st>>>(d_desc1, d_count1, cap1, rows1, d_desc2, d_count2, cap2, rows2, dim,
                                                                              norm1, norm2);
    AG_CHECK_LAUNCH("row_norms_kernel");
    const dim3 grid(P, cdiv(cap1, BM));   // pairs on x (up to 2^31 - 1); CTAs beyond a pair's count exit at once
    snn_pass_kernel<1><<<grid, 256, 0, st>>>(d_desc1, d_count1, S1, cap1, d_desc2, d_count2, S2, cap2, dim, d_pairs, norm1, norm2, colmask, ratio,
                                             d_idx2, d_min, d_second, d_keep);
    AG_CHECK_LAUNCH("snn_pass1_kernel");
    snn_pass_kernel<2><<<grid, 256, 0, st>>>(d_desc1, d_count1, S1, cap1, d_desc2, d_count2, S2, cap2, dim, d_pairs, norm1, norm2, colmask, ratio,
                                             d_idx2, d_min, d_second, d_keep);
    AG_CHECK_LAUNCH("snn_pass2_kernel");
    if (d_tent || d_ntent) {
        snn_compact_kernel<<<P, 256, 0, st>>>(d_pairs, d_count1, S1, cap1, d_count2, S2, cap2, d_keep, d_idx2, d_tent, d_ntent);
        AG_CHECK_LAUNCH("snn_compact_kernel");
    }
    return AG_OK;
}

size_t ag_match_snn_workspace_bytes(int n1, int n2) { return ag_match_pairs_workspace_bytes(1, n1, 1, n2, 1); }

int ag_match_snn(const float* d_desc1, int n1, const float* d_desc2, int n2, int dim, float ratio, void* d_ws, size_t ws_bytes, int* d_idx2,
                 float* d_min, float* d_second, unsigned char* d_keep, void* stream) {
    AG_REQUIRE(d_desc1 && d_desc2 && d_ws && d_idx2 && d_min && d_second && d_keep, "NULL argument");
    AG_REQUIRE(n1 >= 1 && n2 >= 1 && dim >= 1, "bad sizes");
    if (ws_bytes < ag_match_snn_workspace_bytes(n1, n2)) { set_error("ag_match_snn: workspace too small"); return AG_ERR_CAPACITY; }
    return ag_match_pairs(d_desc1, nullptr, 1, n1, d_desc2, nullptr, 1, n2, dim, nullptr, 1, ratio, d_ws, ws_bytes, d_idx2, d_min, d_second,
                          d_keep, nullptr, nullptr, stream);
}

}  // extern "C"
