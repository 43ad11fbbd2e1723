// Top-m of unique 64-bit keys at any m, in global memory: the large-count path of the keypoint selection (detect.cu) and of the affine
// shape filter (geometry.cu).  Their shared-memory kernels (select_kernel, shape_filter_kernel) sort at most 16384 keys per image; this
// primitive has no such limit.  Per image:
//   1. topk_select_kernel<Src>: a cluster of TK_CL CTAs runs the radix select of the m-th largest key (8 bits per pass from the top, the
//      per-CTA histograms merged by rank 0 through distributed shared memory, as select_kernel does) and copies every key >= it, with its
//      source index, to the image's key buffer.  Keys are unique, so exactly m survive; the append order does not matter.
//   2. topk_tile_sort_kernel: TK_TILE-key tiles sorted descending in shared memory (bitonic_sort_desc).
//   3. topk_merge_kernel, once per doubling of the sorted run length: every key's row in the merged run is its row in its own run plus the
//      number of keys of the partner run above it (a binary search; keys are unique, so there are no ties to break).
// The tile-sort and merge kernels have internal linkage: every .cu that includes this header owns its copy.
// The caller's writer then reads rows 0 .. count-1 of the final buffer.  The number of launches is fixed on the host from the largest m the
// call can select, and every launch reads m from the device, so the whole sequence is CUDA-graph capturable without a host synchronisation.
//
// A key source Src provides, per image b:
//   TopkSetup setup(int b) const                         (one thread: candidate count, m, mode)
//   unsigned long long key(int b, int i, const TopkSetup&) const   (key of source row i < n; 0 = never selected)
#pragma once
#include "common.cuh"

namespace ag {

constexpr int TOPK_SMEM_MAX = 16384;   // keys the shared-memory top-K kernels sort per image; above it the primitive below runs
constexpr int TK_CL = 8;               // CTAs per image in the radix select (one thread-block cluster)
constexpr int TK_NT = 1024;            // threads per CTA of the select and tile-sort kernels
constexpr int TK_TILE = 8192;          // keys per shared-memory tile sort (96 KiB of keys and indices)
constexpr int TK_MNT = 256;            // threads per CTA of the merge passes

__device__ __forceinline__ uint32_t dsmem_addr(const void* p, int rank) {
    uint32_t a = (uint32_t)__cvta_generic_to_shared(p), r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
    return r;
}
__device__ __forceinline__ int dsmem_ld_i32(uint32_t a) { int v; asm volatile("ld.shared::cluster.s32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ unsigned long long dsmem_ld_u64(uint32_t a) { unsigned long long v; asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ void dsmem_st_i32(uint32_t a, int v) { asm volatile("st.shared::cluster.s32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void dsmem_st_u64(uint32_t a, unsigned long long v) { asm volatile("st.shared::cluster.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ int dsmem_atomic_add(uint32_t a, int v) { int o; asm volatile("atom.shared::cluster.add.s32 %0, [%1], %2;" : "=r"(o) : "r"(a), "r"(v) : "memory"); return o; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

struct TopkSetup {
    int n;          // source rows of the image
    int m;          // keys to select
    int sorted;     // passed on to the writer
    int radix;      // 0: every non-zero key is selected (no radix select needed)
    int fail;       // the image reports count -1 and nothing of it is written
    unsigned ctx;   // source-specific (the selection's accepted-slot mask)
};

struct TopkImage {  // per image, written by topk_select_kernel
    int m_out;      // keys in the buffer
    int count;      // rows the writer writes (m_out), or -1
    int sorted;
    int pad;
};

struct TopkBufs {
    unsigned long long* key[2];   // [B, rows] ping-pong key buffers
    int* idx[2];                  // [B, rows] source rows of the keys
    TopkImage* img;               // [B]
    int rows;                     // rows per image of each buffer (the largest m)
};

// Scratch layout: two key buffers, two index buffers, the per-image records; `extra` bytes for the source follow (256-B aligned).
inline size_t topk_scratch_bytes(size_t B, size_t rows) {
    return 2 * align_up(B * rows * sizeof(unsigned long long), 256) + 2 * align_up(B * rows * sizeof(int), 256) +
           align_up(B * sizeof(TopkImage), 256);
}
inline unsigned char* topk_carve(unsigned char* c, int B, int rows, TopkBufs& T) {
    const size_t kb = align_up((size_t)B * rows * sizeof(unsigned long long), 256), ib = align_up((size_t)B * rows * sizeof(int), 256);
    T.key[0] = (unsigned long long*)c; c += kb;
    T.key[1] = (unsigned long long*)c; c += kb;
    T.idx[0] = (int*)c; c += ib;
    T.idx[1] = (int*)c; c += ib;
    T.img = (TopkImage*)c; c += align_up((size_t)B * sizeof(TopkImage), 256);
    T.rows = rows;
    return c;
}
// merge passes after the tile sort for at most `need` keys per image
inline int topk_merge_passes(int need) {
    int p = 0;
    for (long long w = TK_TILE; w < need; w <<= 1) p++;
    return p;
}

template <class Src>
__global__ void __launch_bounds__(TK_NT) topk_select_kernel(const Src S, const TopkBufs T) {
    __shared__ int s_hist[256];
    __shared__ TopkSetup s_set;
    __shared__ int s_fill;                     // rank 0: keys appended
    __shared__ unsigned long long s_prefix;    // rank 0 publishes the radix prefix here
    __shared__ int s_ctl[2];                   // rank 0: [0] remaining, [1] done
    unsigned rank;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    const int b = blockIdx.x / TK_CL;
    if (threadIdx.x == 0) {   // every CTA of the cluster derives the same parameters
        s_set = S.setup(b);
        s_fill = 0;
        s_prefix = 0ull;
        s_ctl[0] = s_set.m; s_ctl[1] = 0;
    }
    __syncthreads();
    const TopkSetup st = s_set;
    const int n = st.n, m = st.m;
    const uint32_t r0_prefix = dsmem_addr(&s_prefix, 0), r0_ctl = dsmem_addr(s_ctl, 0), r0_fill = dsmem_addr(&s_fill, 0);

    unsigned long long kth = 1ull;   // no radix select: every non-zero key is taken
    if (m > 0 && st.radix) {
        unsigned long long prefix = 0ull;
        for (int pass = 7; pass >= 0; pass--) {
            for (int i = threadIdx.x; i < 256; i += TK_NT) s_hist[i] = 0;
            __syncthreads();
            const int shift = pass * 8;
            const unsigned long long hi_mask = (pass == 7) ? 0ull : (~0ull << (shift + 8));
            for (int i = (int)rank * TK_NT + threadIdx.x; i < n; i += TK_CL * TK_NT) {
                const unsigned long long k = S.key(b, i, st);
                if ((k & hi_mask) == prefix) atomicAdd(&s_hist[(int)((k >> shift) & 0xFF)], 1);
            }
            cluster_sync_all();                      // all local histograms complete
            if (rank == 0) {
                if (threadIdx.x < 256) {             // merge the other CTAs' histograms into this one
                    int t = s_hist[threadIdx.x];
                    for (int r = 1; r < TK_CL; r++) t += dsmem_ld_i32(dsmem_addr(&s_hist[threadIdx.x], r));
                    s_hist[threadIdx.x] = t;
                }
                __syncthreads();
                if (threadIdx.x < 32) {              // warp 0: the digit d with count(> d) < remaining <= count(>= d), 8 bins per lane
                    const int lane = threadIdx.x;
                    int loc[8], tot = 0;
#pragma unroll
                    for (int j = 0; j < 8; j++) { loc[j] = s_hist[lane * 8 + j]; tot += loc[j]; }
                    int above = tot;
                    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_down_sync(0xffffffffu, above, o); if (lane + o < 32) above += t; }
                    above -= tot;
                    const int remaining = s_ctl[0];
                    int cum = above, dsel = -1, need = 0, cnt = 0;
#pragma unroll
                    for (int j = 7; j >= 0; j--) {
                        if (dsel < 0 && cum < remaining && cum + loc[j] >= remaining) { dsel = lane * 8 + j; need = remaining - cum; cnt = loc[j]; }
                        cum += loc[j];
                    }
                    const unsigned hit = __ballot_sync(0xffffffffu, dsel >= 0);
                    if (hit == 0) { if (lane == 0) s_ctl[1] = 1; }             // fewer keys than requested: stop
                    else if (lane == (int)(31 - __clz(hit))) {
                        s_prefix = prefix | ((unsigned long long)dsel << shift);
                        s_ctl[0] = need;
                        s_ctl[1] = (need == cnt) ? 1 : 0;                       // the whole bucket is needed
                    }
                }
            }
            cluster_sync_all();                      // rank 0 has published prefix / remaining / done
            prefix = dsmem_ld_u64(r0_prefix);
            const int done = dsmem_ld_i32(r0_ctl + 4);
            if (done) break;
        }
        kth = prefix;
    }
    cluster_sync_all();                              // rank 0's fill counter is initialised before any CTA appends to it
    if (m > 0) {
        unsigned long long* K = T.key[0] + (size_t)b * T.rows;
        int* I = T.idx[0] + (size_t)b * T.rows;
        for (int i = (int)rank * TK_NT + threadIdx.x; i < n; i += TK_CL * TK_NT) {
            const unsigned long long k = S.key(b, i, st);
            if (k >= kth && k != 0ull) {
                const int pos = dsmem_atomic_add(r0_fill, 1);
                if (pos < T.rows) { K[pos] = k; I[pos] = i; }
            }
        }
    }
    cluster_sync_all();                              // every append is done
    if (rank == 0 && threadIdx.x == 0) {
        const int mo = m > 0 ? min(min(s_fill, m), T.rows) : 0;
        TopkImage r;
        r.m_out = mo; r.count = st.fail ? -1 : mo; r.sorted = st.sorted; r.pad = 0;
        T.img[b] = r;
    }
}

// Tiles of TK_TILE keys of buffer 0, sorted descending in place.
template <int TILE>
static __global__ void __launch_bounds__(TK_NT) topk_tile_sort_kernel(const TopkBufs T) {
    extern __shared__ __align__(16) unsigned char tk_smem[];
    unsigned long long* s_key = reinterpret_cast<unsigned long long*>(tk_smem);
    int* s_idx = reinterpret_cast<int*>(tk_smem + sizeof(unsigned long long) * TILE);
    const int b = blockIdx.y, t0 = blockIdx.x * TILE;
    const int m = T.img[b].m_out;
    if (t0 >= m) return;
    const int len = min(TILE, m - t0);
    unsigned long long* K = T.key[0] + (size_t)b * T.rows + t0;
    int* I = T.idx[0] + (size_t)b * T.rows + t0;
    for (int i = threadIdx.x; i < TILE; i += TK_NT) {
        s_key[i] = i < len ? K[i] : 0ull;   // selected keys are non-zero: the padding sorts last
        s_idx[i] = i < len ? I[i] : -1;
    }
    __syncthreads();
    bitonic_sort_desc<true>(s_key, s_idx, TILE);
    for (int i = threadIdx.x; i < len; i += TK_NT) { K[i] = s_key[i]; I[i] = s_idx[i]; }
}

// One merge pass: sorted runs of w keys (Ki, Ii) -> runs of 2 w (Ko, Io).
template <int NT>
static __global__ void __launch_bounds__(NT) topk_merge_kernel(const unsigned long long* __restrict__ Ki, const int* __restrict__ Ii,
                                                               unsigned long long* __restrict__ Ko, int* __restrict__ Io,
                                                               const TopkImage* __restrict__ img, int rows, int w) {
    const int b = blockIdx.y;
    const int p = blockIdx.x * NT + threadIdx.x;
    const int m = img[b].m_out;
    if (p >= m) return;
    const size_t base = (size_t)b * rows;
    const unsigned long long* K = Ki + base;
    const int r = p / w, i = p - r * w;
    const int ps = (r ^ 1) * w;
    const int len = max(0, min(w, m - ps));
    const unsigned long long k = K[p];
    int lo = 0, hi = len;   // partner keys above k (the partner run is descending)
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (K[ps + mid] > k) lo = mid + 1;
        else hi = mid;
    }
    const size_t o = base + (size_t)((r & ~1) * w + i + lo);
    Ko[o] = k;
    Io[o] = Ii[base + p];
}

// Enqueues steps 1-3 for B images; -> the buffer that holds the sorted keys (0 or 1) through *final, or an AG_ERR_* code.
template <class Src>
static int topk_run(const Src& S, const TopkBufs& T, int B, int need, cudaStream_t st, int* final) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(B * TK_CL); cfg.blockDim = dim3(TK_NT); cfg.dynamicSmemBytes = 0; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = TK_CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    int rc = check_cuda(cudaLaunchKernelEx(&cfg, topk_select_kernel<Src>, S, T), "topk_select_kernel launch");
    if (rc != AG_OK) return rc;
    AG_CHECK_LAUNCH("topk_select_kernel");
    constexpr size_t smem = (size_t)TK_TILE * (sizeof(unsigned long long) + sizeof(int));
    static SmemAttrOnce attr_once;
    if ((rc = attr_once.ensure(topk_tile_sort_kernel<TK_TILE>, smem, "topk tile sort smem attr")) != AG_OK) return rc;
    topk_tile_sort_kernel<TK_TILE><<<dim3(cdiv(need, TK_TILE), B), TK_NT, smem, st>>>(T);
    AG_CHECK_LAUNCH("topk_tile_sort_kernel");
    const int passes = topk_merge_passes(need);
    int src = 0;
    for (int q = 0, w = TK_TILE; q < passes; q++, w <<= 1, src ^= 1) {
        topk_merge_kernel<TK_MNT><<<dim3(cdiv(need, TK_MNT), B), TK_MNT, 0, st>>>(T.key[src], T.idx[src], T.key[src ^ 1], T.idx[src ^ 1], T.img, T.rows, w);
        AG_CHECK_LAUNCH("topk_merge_kernel");
    }
    *final = src;
    return AG_OK;
}

}  // namespace ag
