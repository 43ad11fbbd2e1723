// Batched end-to-end pipeline: ScaleSpaceAffinePatchExtractor.forward (SparseImgRepresenter.py:189-209) with any shape estimator
// (AffNet or Baumberg, any number of iterations, or none) and orientation estimator (OriNet, gradient histogram or none)
// + extract_patches_from_pyr (:181-188) + HardNet.forward or SIFTNet.forward for B images of one size, as a
// fixed sequence of kernel launches on one stream with fixed-capacity buffers and device-side counters
// (no host synchronisation, CUDA-graph capturable).  The reference processes one image at a time with
// several .item()/nonzero host round trips (SURVEY.md §3); this is the on-device replacement.  ag_pipeline_create_given runs the same
// estimator and descriptor steps on caller-supplied keypoints instead of detected ones (getAffineShape / getOrientation /
// extract_patches_from_pyr on arbitrary LAFs, as the reference's SIFT-AffNet-HardNet notebook composes them).
#include <math.h>

#include <vector>

#include "common.cuh"

struct ag_pipeline {
    ag_pipeline_config_t cfg;
    ag_pipeline_estimators_t est;
    ag_pipeline_descriptor_t desc;
    std::vector<float> shape_gk, ori_gk;
    std::vector<float> sift_gk, sift_pk;   // SIFTNet's Gaussian window and pooling kernel (ag_sift_windows), host copies
    int sift_k, sift_s;   // the hand-crafted estimators' Gaussian windows (HandCraftedModules._gauss_window), host copies
    ag_pyramid_plan_t plan;
    const ag_net_t* aff;
    const ag_net_t* ori;
    const ag_net_t* hard;
    int M;          // prefilter keypoints per image = int(1.5 K) with a shape step, K without; C in threshold mode
    int cand_cap;
    bool th_mode;   // ag_pipeline_create_th: detector threshold th, keep-all selection and shape filter
    bool topk;      // ag_pipeline_create_topk: the top-K steps at any count (ag_select_topk_keypoints, ag_affine_shape_filter_topk)
    bool given;     // ag_pipeline_create_given: caller-supplied keypoints, no detector and no selection
    float th;
    // workspace layout (byte offsets)
    size_t off_pyr, off_det, off_resp1, off_lafs1, off_oct1, off_lvl1, off_cnt1, off_patches, off_A, off_lafs2, off_oct2,
        off_lvl2, off_nlafs, off_oct3, off_lvl3, off_net, net_bytes, off_A2, off_base2, off_lafsw, off_sel, sel_bytes, total;
    size_t off_src, off_dl;   // given keypoints: the shape filter's source rows (fp32), the output LAFs before the count-bounded copy
    int launches;
};

using namespace ag;

// ag_pipeline_create, ag_pipeline_create_ex, ag_pipeline_create_desc, ag_pipeline_create_th and ag_pipeline_create_topk: `fn` names the entry point the caller called in the error texts
#define PIPE_REQUIRE(cond, msg)                         \
    do {                                                \
        if (!(cond)) {                                  \
            set_error("%s: %s", fn, msg);               \
            return AG_ERR_INVALID;                      \
        }                                               \
    } while (0)

static int pipeline_create(const char* fn, const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est,
                           const ag_pipeline_descriptor_t* desc, const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet,
                           bool th_mode, float th, bool topk, bool given, ag_pipeline_t** out) {
    PIPE_REQUIRE(cfg && est && desc && out, "NULL argument");
    PIPE_REQUIRE(isfinite(th), "th must be finite");
    PIPE_REQUIRE(desc->kind == AG_DESC_HARDNET || desc->kind == AG_DESC_SIFT, "unknown descriptor kind");
    const bool sift = desc->kind == AG_DESC_SIFT;
    PIPE_REQUIRE(sift || hardnet, "NULL argument: AG_DESC_HARDNET needs a HardNet");
    PIPE_REQUIRE(sift || desc->ps == 32, "AG_DESC_HARDNET needs ps = 32");
    int sift_k = 0, sift_s = 0;
    PIPE_REQUIRE(!sift || sift_geometry(desc->ps, &sift_k, &sift_s),
                 "AG_DESC_SIFT: unsupported ps (16..65 with a 4 x 4 pooling grid, not 17, 18, 23, 28, 38, 48, 58)");
    PIPE_REQUIRE(!sift || (isfinite(desc->clipval) && desc->clipval > 0.f), "AG_DESC_SIFT: clipval must be finite and positive");
    PIPE_REQUIRE(est->shape == AG_SHAPE_NONE || est->shape == AG_SHAPE_AFFNET || est->shape == AG_SHAPE_BAUMBERG, "unknown shape estimator");
    PIPE_REQUIRE(est->ori == AG_ORI_NONE || est->ori == AG_ORI_ORINET || est->ori == AG_ORI_HISTOGRAM, "unknown orientation estimator");
    PIPE_REQUIRE(est->shape != AG_SHAPE_AFFNET || affnet, "AG_SHAPE_AFFNET needs an AffNet");
    PIPE_REQUIRE(est->ori != AG_ORI_ORINET || orinet, "AG_ORI_ORINET needs an OriNet");
    PIPE_REQUIRE(est->shape == AG_SHAPE_NONE || est->num_baum_iters >= 1, "num_baum_iters must be at least 1 with a shape estimator");
    PIPE_REQUIRE(est->shape != AG_SHAPE_BAUMBERG || (est->shape_ps >= 3 && est->shape_ps <= 41), "shape_ps out of range (3..41)");
    PIPE_REQUIRE(est->ori != AG_ORI_HISTOGRAM || (est->ori_ps >= 3 && est->ori_ps <= 41), "ori_ps out of range (3..41)");
    PIPE_REQUIRE((cfg->do_ori != 0) == (est->ori != AG_ORI_NONE), "cfg->do_ori disagrees with est->ori");
    PIPE_REQUIRE(cfg->num_features >= 1, "num_features must be positive");
    // given keypoints: the row index travels through the keep-all filter as an fp32 response, exact up to 2^24
    PIPE_REQUIRE(!given || cfg->num_features <= (1 << 24), "num_features above 2^24 rows per image");
    PIPE_REQUIRE(!given || (cfg->B >= 1 && cfg->B <= 65535 && (long long)cfg->B * cfg->num_features <= 0x7fffffffLL),
                 "B outside 1..65535 or B x num_features rows above 2^31 - 1");
    const bool shape = est->shape != AG_SHAPE_NONE;
    ag_pipeline* p = new ag_pipeline();
    p->cfg = *cfg; p->est = *est; p->desc = *desc;
    p->aff = est->shape == AG_SHAPE_AFFNET ? affnet : nullptr;
    p->ori = est->ori == AG_ORI_ORINET ? orinet : nullptr;
    p->hard = sift ? nullptr : hardnet;
    int rc = ag_pyramid_plan(cfg->B, cfg->H, cfg->W, cfg->nlevels, cfg->init_sigma, cfg->border, &p->plan);
    if (rc != AG_OK) { delete p; return rc; }
    // the top-K selection kernels sort in shared memory (ag_select_keypoints / ag_affine_shape_filter): fail here, not at run time.
    // Threshold mode keeps everything without a sort and has no such limit, and the top-K entry points sort in global memory above it.
    if (!given && !th_mode && !topk && shape && (int)(1.5 * cfg->num_features) > 16384) {
        set_error("%s: num_features %d needs a prefilter of int(1.5 K) = %d keypoints; the shared-memory selection holds 16384 (K <= 10923)",
                  fn, cfg->num_features, (int)(1.5 * cfg->num_features));
        delete p;
        return AG_ERR_CAPACITY;
    }
    if (!given && !th_mode && !topk && !shape && cfg->num_features > 16384) {
        set_error("%s: num_features %d without a shape estimator: the shared-memory selection holds 16384 (K <= 16384)", fn,
                  cfg->num_features);
        delete p;
        return AG_ERR_CAPACITY;
    }
    // Gaussian windows of HandCraftedModules._gauss_window: CircularGaussKernel(PS, sigma = PS/6) for Baumberg, 10x the default for the
    // histogram, rounded to fp32 exactly as torch multiplies the fp32 kernel by the Python scale
    if (est->shape == AG_SHAPE_BAUMBERG) {
        const int ps = est->shape_ps;
        p->shape_gk.resize((size_t)ps * ps);
        ag_circular_gauss_kernel(ps, (ps / 2.0) / 3.0, p->shape_gk.data());
    }
    if (est->ori == AG_ORI_HISTOGRAM) {
        const int ps = est->ori_ps;
        p->ori_gk.resize((size_t)ps * ps);
        ag_circular_gauss_kernel(ps, 0.0, p->ori_gk.data());
        for (float& v : p->ori_gk) v = v * 10.0f;
    }
    if (sift) {
        p->sift_k = sift_k; p->sift_s = sift_s;
        p->sift_gk.resize((size_t)desc->ps * desc->ps);
        p->sift_pk.resize((size_t)sift_k * sift_k);
        sift_windows(desc->ps, sift_k, p->sift_gk.data(), p->sift_pk.data());
    }
    p->th_mode = th_mode;
    p->topk = topk && !th_mode;
    p->th = th_mode ? th : 0.f;
    p->given = given;
    p->launches = 0;
    if (given) {
        // rows of C per image: the normalised input, its level and the sanitised counts (with a shape step; without one they go straight
        // to the post-shape buffers), the estimators' A, the post-shape rows, the output LAFs before the copy, the descriptor's level
        const size_t B = cfg->B, C = cfg->num_features, S = shape ? C : 0;
        const bool any_step = shape || est->ori != AG_ORI_NONE;
        const bool aff_chain = est->shape == AG_SHAPE_AFFNET && est->num_baum_iters > 1;
        p->M = cfg->num_features;
        p->cand_cap = 0;
        size_t o = 0;
        auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 256); return r; };
        p->off_pyr = take(sizeof(float) * (size_t)p->plan.total_floats);
        p->off_det = p->off_resp1 = p->off_sel = p->sel_bytes = p->off_patches = 0;
        p->off_src = take(sizeof(float) * B * S * 2);   // the filter's input rows 0..C-1 and its output, as fp32
        p->off_lafs1 = take(sizeof(float) * B * S * 6);
        p->off_oct1 = take(sizeof(int) * B * S);
        p->off_lvl1 = take(sizeof(int) * B * S);
        p->off_cnt1 = take(shape ? sizeof(int) * B : 0);
        p->off_A = take(any_step ? sizeof(float) * B * C * 4 : 0);
        p->off_lafs2 = take(any_step ? sizeof(float) * B * C * 6 : 0);
        p->off_oct2 = take(any_step ? sizeof(int) * B * C : 0);
        p->off_lvl2 = take(any_step ? sizeof(int) * B * C : 0);
        p->off_dl = take(any_step ? sizeof(float) * B * C * 6 : 0);
        p->off_nlafs = take(sizeof(float) * B * C * 6);
        p->off_oct3 = take(sizeof(int) * B * C);
        p->off_lvl3 = take(sizeof(int) * B * C);
        size_t nb = 0;
        if (est->shape == AG_SHAPE_AFFNET) nb = ag_net_workspace_bytes(AG_NET_AFFNET, (int)(B * C));
        if (est->ori == AG_ORI_ORINET) {
            const size_t ob = ag_net_workspace_bytes(AG_NET_ORINET, (int)(B * C));
            if (ob > nb) nb = ob;
        }
        const size_t hb = sift ? 0 : ag_net_workspace_bytes(AG_NET_HARDNET, (int)(B * C));
        p->net_bytes = nb > hb ? nb : hb;
        p->off_net = take(p->net_bytes);
        p->off_A2 = take(aff_chain ? sizeof(float) * B * C * 4 : 0);
        p->off_base2 = take(aff_chain ? sizeof(float) * B * C * 4 : 0);
        p->off_lafsw = take(aff_chain ? sizeof(float) * B * C * 6 : 0);
        p->total = o;
        *out = p;
        return AG_OK;
    }
    // SparseImgRepresenter.py:192-194; threshold mode keeps every candidate, so the prefilter is the capacity C itself
    p->M = (shape && !th_mode) ? (int)(1.5 * cfg->num_features) : cfg->num_features;
    p->cand_cap = cfg->cand_cap > 0 ? cfg->cand_cap : (cfg->H * cfg->W) / 8;
    if (p->cand_cap < p->M) p->cand_cap = p->M;
    const size_t B = cfg->B, M = shape ? p->M : 0, K = cfg->num_features;
    const bool aff_chain = est->shape == AG_SHAPE_AFFNET && est->num_baum_iters > 1;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 256); return r; };
    p->off_pyr = take(sizeof(float) * (size_t)p->plan.total_floats);
    p->off_det = take(ag_detect_ws_bytes(&p->plan, p->cand_cap));
    p->off_resp1 = take(sizeof(float) * B * M);   // prefilter rows: only with a shape step
    p->off_lafs1 = take(sizeof(float) * B * M * 6);
    p->off_oct1 = take(sizeof(int) * B * M);
    p->off_lvl1 = take(sizeof(int) * B * M);
    p->off_cnt1 = take(shape ? sizeof(int) * B : 0);
    p->off_patches = 0;  // patches are never materialised: the samplers are fused into the first tensor-core layer / the hand-crafted estimators
    p->off_A = take(sizeof(float) * B * (shape ? M : K) * 4);
    p->off_lafs2 = take(sizeof(float) * B * K * 6);
    p->off_oct2 = take(sizeof(int) * B * K);
    p->off_lvl2 = take(sizeof(int) * B * K);
    p->off_nlafs = take(sizeof(float) * B * K * 6);
    p->off_oct3 = take(sizeof(int) * B * K);
    p->off_lvl3 = take(sizeof(int) * B * K);
    size_t nb = 0;
    if (est->shape == AG_SHAPE_AFFNET) nb = ag_net_workspace_bytes(AG_NET_AFFNET, (int)(B * M));
    if (est->ori == AG_ORI_ORINET) {
        const size_t ob = ag_net_workspace_bytes(AG_NET_ORINET, (int)(B * K));
        if (ob > nb) nb = ob;
    }
    const size_t hb = sift ? 0 : ag_net_workspace_bytes(AG_NET_HARDNET, (int)(B * K));
    p->net_bytes = nb > hb ? nb : hb;
    p->off_net = take(p->net_bytes);
    // AffNet with several iterations: the net's A of the current iteration, the other base_A buffer, the working LAFs
    p->off_A2 = take(aff_chain ? sizeof(float) * B * M * 4 : 0);
    p->off_base2 = take(aff_chain ? sizeof(float) * B * M * 4 : 0);
    p->off_lafsw = take(aff_chain ? sizeof(float) * B * M * 6 : 0);
    p->sel_bytes = th_mode ? ag_select_all_workspace_bytes(&p->plan, p->cand_cap) : 0;
    if (p->topk) {   // one scratch for both top-K steps, which run one after the other; 0 while both fit the shared-memory kernels
        const size_t sb = ag_select_topk_workspace_bytes(&p->plan, p->cand_cap, shape ? p->M : cfg->num_features);
        const size_t fb = shape ? ag_affine_shape_filter_topk_workspace_bytes(cfg->B, p->M) : 0;
        p->sel_bytes = sb > fb ? sb : fb;
    }
    p->off_sel = take(p->sel_bytes);
    p->total = o;
    p->launches = 0;
    *out = p;
    return AG_OK;
}
#undef PIPE_REQUIRE

// getAffineShape's iterations (SparseImgRepresenter.py:127-141) over M rows per image: base_A into A.  Shared by ag_pipeline_run and
// ag_pipeline_run_given.
static int shape_iterations(const ag_pipeline* p, char* ws, const float* pyr, const float* lafs1, const int* oct1, const int* lvl1,
                            const int* cnt1, int M, float* A, void* stream) {
    const ag_pipeline_estimators_t& e = p->est;
    void* netws = ws + p->off_net;
    int rc;
    if (e.shape == AG_SHAPE_BAUMBERG) {
        if ((rc = baumberg_pyr(&p->plan, pyr, lafs1, oct1, lvl1, cnt1, M, e.shape_ps, e.num_baum_iters, p->shape_gk.data(), A, stream)))
            return rc;
    } else if (e.num_baum_iters == 1) {
        if ((rc = ag_net_forward_pyr(p->aff, &p->plan, pyr, lafs1, oct1, lvl1, cnt1, M, A, netws, p->net_bytes, stream))) return rc;
    } else {
        // the mirror's order (SparseImgRepresenter.getAffineShape): A_i of the working LAFs, base_A <- A_i base_A, working LAFs <-
        // [base_A LAF_A | t]; base_A ping-pongs between A and base2 so that it ends in A.  The 2x2 products run over all B*M rows, so
        // they also combine the (unwritten) rows at or beyond cnt1: those results are never read - the net and the shape filter stop
        // at the count - and computing them keeps the step one count-free elementwise launch each.
        float* A_i = (float*)(ws + p->off_A2);
        float* lafsw = (float*)(ws + p->off_lafsw);
        float* bufs[2] = {A, (float*)(ws + p->off_base2)};
        const int n = p->cfg.B * M, it_n = e.num_baum_iters;
        float* base = bufs[(it_n - 1) & 1];   // the first iteration's A, in the buffer that makes the last product land in A
        for (int it = 0; it < it_n; it++) {
            const float* cur = it == 0 ? lafs1 : lafsw;
            float* dst = it == 0 ? base : A_i;
            if ((rc = ag_net_forward_pyr(p->aff, &p->plan, pyr, cur, oct1, lvl1, cnt1, M, dst, netws, p->net_bytes, stream))) return rc;
            if (it > 0) {
                float* nbase = bufs[(it_n - 1 - it) & 1];
                if ((rc = ag_mat2_compose(A_i, base, nbase, n, stream))) return rc;
                base = nbase;
            }
            if (it != it_n - 1 && (rc = ag_lafs_left_multiply(base, lafs1, lafsw, n, stream))) return rc;
        }
    }
    return AG_OK;
}

// getOrientation (SparseImgRepresenter.py:167-180) over K rows per image: lafs2 <- lafs2 R, with A as the rotations' scratch
static int orientation_step(const ag_pipeline* p, char* ws, const float* pyr, float* lafs2, const int* oct2, const int* lvl2,
                            const int* count, int K, float* A, void* stream) {
    const ag_pipeline_estimators_t& e = p->est;
    const int n = p->cfg.B * K;
    int rc;
    if (e.ori == AG_ORI_ORINET) {
        if ((rc = ag_net_forward_pyr(p->ori, &p->plan, pyr, lafs2, oct2, lvl2, count, K, A, ws + p->off_net, p->net_bytes, stream))) return rc;
        if ((rc = ag_lafs_apply_rotation(lafs2, A, n, stream))) return rc;
    } else if (e.ori == AG_ORI_HISTOGRAM) {
        if ((rc = orientation_hist_pyr(&p->plan, pyr, lafs2, oct2, lvl2, count, K, e.ori_ps, p->ori_gk.data(), A, stream))) return rc;
        if ((rc = ag_lafs_apply_rotation(lafs2, A, n, stream))) return rc;
    }
    return AG_OK;
}

// extract_patches_from_pyr(dLAFs, desc.ps) (SparseImgRepresenter.py:181-188) and the descriptor: level choice on the pixel LAFs d_lafs,
// normalizeLAFs (LAF.py:419-429), then SIFT or HardNet on the first count[b] rows of each image
static int describe_step(const ag_pipeline* p, char* ws, const float* pyr, const float* d_lafs, const int* count, int K, float* d_desc,
                         void* stream) {
    const ag_pipeline_config_t& c = p->cfg;
    const int n = c.B * K, dps = p->desc.ps;
    const float ms = (float)(c.H < c.W ? c.H : c.W);
    float* nlafs = (float*)(ws + p->off_nlafs); int* oct3 = (int*)(ws + p->off_oct3); int* lvl3 = (int*)(ws + p->off_lvl3);
    int rc;
    if ((rc = ag_pyramid_level_for_lafs(&p->plan, d_lafs, n, dps, oct3, lvl3, stream))) return rc;
    if ((rc = ag_lafs_scale(d_lafs, nlafs, n, 1.0f / ms, (float)(1.0 / (double)c.W), (float)(1.0 / (double)c.H), stream))) return rc;
    if (p->desc.kind == AG_DESC_SIFT)
        return sift_pyr(&p->plan, pyr, nlafs, oct3, lvl3, count, K, dps, p->sift_k, p->sift_s, p->sift_gk.data(), p->sift_pk.data(),
                        p->desc.clipval, d_desc, stream);
    return ag_net_forward_pyr(p->hard, &p->plan, pyr, nlafs, oct3, lvl3, count, K, d_desc, ws + p->off_net, p->net_bytes, stream);
}

namespace ag {
// ag_pipeline_run_given, before any other step: count[b] = count_in[b] where it lies in 0..C, else -1 (nothing of the image is written);
// with a shape step, rows i < count of src are the row indices i as fp32 - the keep-all shape filter passes a response through unchanged,
// so its response output is the source row of each survivor (exact up to 2^24).
__global__ void given_counts_kernel(const int* __restrict__ count_in, int C, int* __restrict__ count, float* __restrict__ src) {
    const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
    const int c = count_in[b];
    const bool ok = c >= 0 && c <= C;
    if (i == 0) count[b] = ok ? c : -1;
    if (src && ok && i < c) src[(size_t)b * C + i] = (float)i;
}

// ag_pipeline_run_given, last: rows j < count[b] of the output LAFs and source indices (src_f NULL: no shape step, row j is input row j).
// The count-bounded copy keeps every row at or beyond the count unwritten.
__global__ void given_finish_kernel(const float* __restrict__ dl, const float* __restrict__ src_f, const int* __restrict__ count, int C,
                                    float* lafs, int* __restrict__ src) {
    const int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count[b]) return;
    const size_t r = (size_t)b * C + j;
#pragma unroll
    for (int q = 0; q < 6; q++) lafs[r * 6 + q] = dl[r * 6 + q];
    src[r] = src_f ? (int)src_f[r] : j;
}
}  // namespace ag

static const ag_pipeline_descriptor_t HARDNET_DESC = {AG_DESC_HARDNET, 32, 0.2f};

extern "C" {

int ag_pipeline_create(const ag_pipeline_config_t* cfg, const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet,
                       ag_pipeline_t** out) {
    AG_REQUIRE(cfg && affnet && hardnet && out, "NULL argument");
    AG_REQUIRE(!cfg->do_ori || orinet, "do_ori needs an OriNet");
    const ag_pipeline_estimators_t est = {AG_SHAPE_AFFNET, 1, 0, cfg->do_ori ? AG_ORI_ORINET : AG_ORI_NONE, 0};
    return pipeline_create(__func__, cfg, &est, &HARDNET_DESC, affnet, orinet, hardnet, false, 0.f, false, false, out);
}

int ag_pipeline_create_ex(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_net_t* affnet,
                          const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out) {
    return pipeline_create(__func__, cfg, est, &HARDNET_DESC, affnet, orinet, hardnet, false, 0.f, false, false, out);
}

int ag_pipeline_create_desc(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_pipeline_descriptor_t* desc,
                            const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out) {
    return pipeline_create(__func__, cfg, est, desc, affnet, orinet, hardnet, false, 0.f, false, false, out);
}

int ag_pipeline_create_th(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_pipeline_descriptor_t* desc,
                          float th, const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out) {
    return pipeline_create(__func__, cfg, est, desc, affnet, orinet, hardnet, true, th, false, false, out);
}

int ag_pipeline_create_given(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_pipeline_descriptor_t* desc,
                             const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out) {
    return pipeline_create(__func__, cfg, est, desc, affnet, orinet, hardnet, false, 0.f, false, true, out);
}

int ag_pipeline_create_topk(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_pipeline_descriptor_t* desc,
                            const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out) {
    return pipeline_create(__func__, cfg, est, desc, affnet, orinet, hardnet, false, 0.f, true, false, out);
}

void ag_pipeline_destroy(ag_pipeline_t* p) { delete p; }
size_t ag_pipeline_workspace_bytes(const ag_pipeline_t* p) { return p ? p->total : 0; }
const ag_pyramid_plan_t* ag_pipeline_plan(const ag_pipeline_t* p) { return p ? &p->plan : nullptr; }
int ag_pipeline_launch_count(const ag_pipeline_t* p) { return p ? p->launches : 0; }

int ag_pipeline_run(ag_pipeline_t* p, const float* d_img, void* d_ws, size_t ws_bytes, float* d_lafs, float* d_resp,
                    float* d_desc, int* d_count, void* stream) {
    AG_REQUIRE(p && d_img && d_ws && d_lafs && d_resp && d_desc && d_count, "NULL argument");
    AG_REQUIRE(!p->given, "a given-keypoints pipeline runs with ag_pipeline_run_given");
    if (ws_bytes < p->total) {
        set_error("ag_pipeline_run: workspace of %zu bytes needed, %zu given", p->total, ws_bytes);
        return AG_ERR_CAPACITY;
    }
    char* ws = (char*)d_ws;
    const ag_pipeline_config_t& c = p->cfg;
    const int B = c.B, M = p->M, K = c.num_features;
    float* pyr = (float*)(ws + p->off_pyr);
    float* resp1 = (float*)(ws + p->off_resp1); float* lafs1 = (float*)(ws + p->off_lafs1);
    int* oct1 = (int*)(ws + p->off_oct1); int* lvl1 = (int*)(ws + p->off_lvl1); int* cnt1 = (int*)(ws + p->off_cnt1);
    float* A = (float*)(ws + p->off_A);
    float* lafs2 = (float*)(ws + p->off_lafs2); int* oct2 = (int*)(ws + p->off_oct2); int* lvl2 = (int*)(ws + p->off_lvl2);
    const int launches0 = g_launches;
    int rc;
    ag_detect_ws_t det;
    if ((rc = ag_detect_ws_carve(&p->plan, p->cand_cap, ws + p->off_det, &det))) return rc;
    if ((rc = ag_pyramid_build(&p->plan, d_img, pyr, stream))) return rc;
    if ((rc = ag_detect(&p->plan, pyr, p->th, (int)c.mrSize, &det, stream))) return rc;
    const ag_pipeline_estimators_t& e = p->est;
    void* sel = ws + p->off_sel;
    if (e.shape == AG_SHAPE_NONE) {
        // num_Baum_iters = 0: K keypoints straight from the detector, no shape filter (SparseImgRepresenter.py:192-200)
        if (p->th_mode) {
            if ((rc = ag_select_all_keypoints(&p->plan, &det, (float)c.mrSize, K, sel, p->sel_bytes, d_resp, lafs2, oct2, lvl2, d_count, stream)))
                return rc;
        } else if (p->topk) {
            if ((rc = ag_select_topk_keypoints(&p->plan, &det, K, (float)c.mrSize, K, sel, p->sel_bytes, d_resp, lafs2, oct2, lvl2, d_count, stream)))
                return rc;
        } else if ((rc = ag_select_keypoints(&p->plan, &det, K, (float)c.mrSize, K, d_resp, lafs2, oct2, lvl2, d_count, stream))) {
            return rc;
        }
    } else {
        if (p->th_mode) {
            if ((rc = ag_select_all_keypoints(&p->plan, &det, (float)c.mrSize, M, sel, p->sel_bytes, resp1, lafs1, oct1, lvl1, cnt1, stream)))
                return rc;
        } else if (p->topk) {
            if ((rc = ag_select_topk_keypoints(&p->plan, &det, M, (float)c.mrSize, M, sel, p->sel_bytes, resp1, lafs1, oct1, lvl1, cnt1, stream)))
                return rc;
        } else if ((rc = ag_select_keypoints(&p->plan, &det, M, (float)c.mrSize, M, resp1, lafs1, oct1, lvl1, cnt1, stream))) {
            return rc;
        }
        if ((rc = shape_iterations(p, ws, pyr, lafs1, oct1, lvl1, cnt1, M, A, stream))) return rc;
        if (p->th_mode) {
            // num_features <= 0: every survivor in order (SparseImgRepresenter.py:151-156); M = K = C
            if ((rc = ag_affine_shape_filter_all(A, resp1, lafs1, oct1, lvl1, cnt1, B, M, d_resp, lafs2, oct2, lvl2, d_count, stream))) return rc;
        } else if (p->topk) {
            if ((rc = ag_affine_shape_filter_topk(A, resp1, lafs1, oct1, lvl1, cnt1, B, M, K, K, sel, p->sel_bytes, d_resp, lafs2, oct2, lvl2, d_count,
                                                  stream)))
                return rc;
        } else if ((rc = ag_affine_shape_filter(A, resp1, lafs1, oct1, lvl1, cnt1, B, M, K, K, d_resp, lafs2, oct2, lvl2, d_count, stream))) {
            return rc;
        }
    }
    if ((rc = orientation_step(p, ws, pyr, lafs2, oct2, lvl2, d_count, K, A, stream))) return rc;
    // denormalizeLAFs (LAF.py:407-417), then descriptor patches: level choice + normalizeLAFs (LAF.py:419-429)
    const float ms = (float)(c.H < c.W ? c.H : c.W);
    if ((rc = ag_lafs_scale(lafs2, d_lafs, B * K, ms, (float)c.W, (float)c.H, stream))) return rc;
    if ((rc = describe_step(p, ws, pyr, d_lafs, d_count, K, d_desc, stream))) return rc;
    p->launches = g_launches - launches0;
    return AG_OK;
}

int ag_pipeline_run_given(ag_pipeline_t* p, const float* d_img, const float* d_lafs_in, const int* d_count_in, void* d_ws, size_t ws_bytes,
                          float* d_lafs, int* d_src, float* d_desc, int* d_count, void* stream) {
    AG_REQUIRE(p && d_img && d_lafs_in && d_count_in && d_ws && d_lafs && d_src && d_desc && d_count, "NULL argument");
    AG_REQUIRE(p->given, "only a pipeline of ag_pipeline_create_given runs with ag_pipeline_run_given");
    if (ws_bytes < p->total) {
        set_error("ag_pipeline_run_given: workspace of %zu bytes needed, %zu given", p->total, ws_bytes);
        return AG_ERR_CAPACITY;
    }
    char* ws = (char*)d_ws;
    const ag_pipeline_config_t& c = p->cfg;
    const ag_pipeline_estimators_t& e = p->est;
    const int B = c.B, C = c.num_features, n = B * C;
    const bool shape = e.shape != AG_SHAPE_NONE, any_step = shape || e.ori != AG_ORI_NONE;
    float* pyr = (float*)(ws + p->off_pyr);
    float* src_in = (float*)(ws + p->off_src); float* src_out = src_in + (size_t)B * C * (shape ? 1 : 0);
    float* lafs1 = (float*)(ws + p->off_lafs1); int* oct1 = (int*)(ws + p->off_oct1); int* lvl1 = (int*)(ws + p->off_lvl1);
    int* cnt1 = (int*)(ws + p->off_cnt1);
    float* A = (float*)(ws + p->off_A);
    float* lafs2 = (float*)(ws + p->off_lafs2); int* oct2 = (int*)(ws + p->off_oct2); int* lvl2 = (int*)(ws + p->off_lvl2);
    const float ms = (float)(c.H < c.W ? c.H : c.W);
    cudaStream_t st = (cudaStream_t)stream;
    const int launches0 = g_launches;
    int rc;
    given_counts_kernel<<<dim3(shape ? cdiv(C, 256) : 1, B), 256, 0, st>>>(d_count_in, C, shape ? cnt1 : d_count, shape ? src_in : nullptr);
    AG_CHECK_LAUNCH("given_counts_kernel");
    if ((rc = ag_pyramid_build(&p->plan, d_img, pyr, stream))) return rc;
    const float* dl = d_lafs_in;   // the pixel LAFs to describe: the input itself when no step changes them
    if (any_step) {
        // the estimators' level, get_pyramid_and_level_index_for_LAFs(dLAFs, PS = 32), and normalizeLAFs, into the rows of the first step
        float* L0 = shape ? lafs1 : lafs2;
        if ((rc = ag_pyramid_level_for_lafs(&p->plan, d_lafs_in, n, 32, shape ? oct1 : oct2, shape ? lvl1 : lvl2, stream))) return rc;
        if ((rc = ag_lafs_scale(d_lafs_in, L0, n, 1.0f / ms, (float)(1.0 / (double)c.W), (float)(1.0 / (double)c.H), stream))) return rc;
        if (shape) {
            if ((rc = shape_iterations(p, ws, pyr, lafs1, oct1, lvl1, cnt1, C, A, stream))) return rc;
            // getAffineShape(num_features = 0): every survivor in input order, its row index in src_out
            if ((rc = ag_affine_shape_filter_all(A, src_in, lafs1, oct1, lvl1, cnt1, B, C, src_out, lafs2, oct2, lvl2, d_count, stream))) return rc;
        }
        if ((rc = orientation_step(p, ws, pyr, lafs2, oct2, lvl2, d_count, C, A, stream))) return rc;
        float* dlw = (float*)(ws + p->off_dl);
        if ((rc = ag_lafs_scale(lafs2, dlw, n, ms, (float)c.W, (float)c.H, stream))) return rc;   // denormalizeLAFs
        dl = dlw;
    }
    if ((rc = describe_step(p, ws, pyr, dl, d_count, C, d_desc, stream))) return rc;
    given_finish_kernel<<<dim3(cdiv(C, 256), B), 256, 0, st>>>(dl, shape ? src_out : nullptr, d_count, C, d_lafs, d_src);
    AG_CHECK_LAUNCH("given_finish_kernel");
    p->launches = g_launches - launches0;
    return AG_OK;
}

}  // extern "C"
