// Batched end-to-end pipeline: ScaleSpaceAffinePatchExtractor.forward (SparseImgRepresenter.py:189-209) with any shape estimator
// (AffNet or Baumberg, any number of iterations, or none) and orientation estimator (OriNet, gradient histogram or none)
// + extract_patches_from_pyr (:181-188) + HardNet.forward for B images of one size, as a
// fixed sequence of kernel launches on one stream with fixed-capacity buffers and device-side counters
// (no host synchronisation, CUDA-graph capturable).  The reference processes one image at a time with
// several .item()/nonzero host round trips (SURVEY.md §3); this is the on-device replacement.
#include <vector>

#include "common.cuh"

struct ag_pipeline {
    ag_pipeline_config_t cfg;
    ag_pipeline_estimators_t est;
    std::vector<float> shape_gk, ori_gk;   // the hand-crafted estimators' Gaussian windows (HandCraftedModules._gauss_window), host copies
    ag_pyramid_plan_t plan;
    const ag_net_t* aff;
    const ag_net_t* ori;
    const ag_net_t* hard;
    int M;          // prefilter keypoints per image = int(1.5 K) with a shape step, K without
    int cand_cap;
    // workspace layout (byte offsets)
    size_t off_pyr, off_det, off_resp1, off_lafs1, off_oct1, off_lvl1, off_cnt1, off_patches, off_A, off_lafs2, off_oct2,
        off_lvl2, off_nlafs, off_oct3, off_lvl3, off_net, net_bytes, off_A2, off_base2, off_lafsw, total;
    int launches;
};

using namespace ag;

// ag_pipeline_create and ag_pipeline_create_ex: `fn` names the entry point the caller called in the error texts
#define PIPE_REQUIRE(cond, msg)                         \
    do {                                                \
        if (!(cond)) {                                  \
            set_error("%s: %s", fn, msg);               \
            return AG_ERR_INVALID;                      \
        }                                               \
    } while (0)

static int pipeline_create(const char* fn, const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_net_t* affnet,
                           const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out) {
    PIPE_REQUIRE(cfg && est && hardnet && out, "NULL argument");
    PIPE_REQUIRE(est->shape == AG_SHAPE_NONE || est->shape == AG_SHAPE_AFFNET || est->shape == AG_SHAPE_BAUMBERG, "unknown shape estimator");
    PIPE_REQUIRE(est->ori == AG_ORI_NONE || est->ori == AG_ORI_ORINET || est->ori == AG_ORI_HISTOGRAM, "unknown orientation estimator");
    PIPE_REQUIRE(est->shape != AG_SHAPE_AFFNET || affnet, "AG_SHAPE_AFFNET needs an AffNet");
    PIPE_REQUIRE(est->ori != AG_ORI_ORINET || orinet, "AG_ORI_ORINET needs an OriNet");
    PIPE_REQUIRE(est->shape == AG_SHAPE_NONE || est->num_baum_iters >= 1, "num_baum_iters must be at least 1 with a shape estimator");
    PIPE_REQUIRE(est->shape != AG_SHAPE_BAUMBERG || (est->shape_ps >= 3 && est->shape_ps <= 41), "shape_ps out of range (3..41)");
    PIPE_REQUIRE(est->ori != AG_ORI_HISTOGRAM || (est->ori_ps >= 3 && est->ori_ps <= 41), "ori_ps out of range (3..41)");
    PIPE_REQUIRE((cfg->do_ori != 0) == (est->ori != AG_ORI_NONE), "cfg->do_ori disagrees with est->ori");
    PIPE_REQUIRE(cfg->num_features >= 1, "num_features must be positive");
    const bool shape = est->shape != AG_SHAPE_NONE;
    ag_pipeline* p = new ag_pipeline();
    p->cfg = *cfg; p->est = *est;
    p->aff = est->shape == AG_SHAPE_AFFNET ? affnet : nullptr;
    p->ori = est->ori == AG_ORI_ORINET ? orinet : nullptr;
    p->hard = hardnet;
    int rc = ag_pyramid_plan(cfg->B, cfg->H, cfg->W, cfg->nlevels, cfg->init_sigma, cfg->border, &p->plan);
    if (rc != AG_OK) { delete p; return rc; }
    // the selection kernels sort in shared memory (ag_select_keypoints / ag_affine_shape_filter): fail here, not at run time
    if (shape && (int)(1.5 * cfg->num_features) > 16384) {
        set_error("%s: num_features %d needs a prefilter of int(1.5 K) = %d keypoints; the shared-memory selection holds 16384 (K <= 10923)",
                  fn, cfg->num_features, (int)(1.5 * cfg->num_features));
        delete p;
        return AG_ERR_CAPACITY;
    }
    if (!shape && cfg->num_features > 16384) {
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
    p->M = shape ? (int)(1.5 * cfg->num_features) : cfg->num_features;  // SparseImgRepresenter.py:192-194
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
    size_t hb = ag_net_workspace_bytes(AG_NET_HARDNET, (int)(B * K));
    p->net_bytes = nb > hb ? nb : hb;
    p->off_net = take(p->net_bytes);
    // AffNet with several iterations: the net's A of the current iteration, the other base_A buffer, the working LAFs
    p->off_A2 = take(aff_chain ? sizeof(float) * B * M * 4 : 0);
    p->off_base2 = take(aff_chain ? sizeof(float) * B * M * 4 : 0);
    p->off_lafsw = take(aff_chain ? sizeof(float) * B * M * 6 : 0);
    p->total = o;
    p->launches = 0;
    *out = p;
    return AG_OK;
}
#undef PIPE_REQUIRE

extern "C" {

int ag_pipeline_create(const ag_pipeline_config_t* cfg, const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet,
                       ag_pipeline_t** out) {
    AG_REQUIRE(cfg && affnet && hardnet && out, "NULL argument");
    AG_REQUIRE(!cfg->do_ori || orinet, "do_ori needs an OriNet");
    const ag_pipeline_estimators_t est = {AG_SHAPE_AFFNET, 1, 0, cfg->do_ori ? AG_ORI_ORINET : AG_ORI_NONE, 0};
    return pipeline_create(__func__, cfg, &est, affnet, orinet, hardnet, out);
}

int ag_pipeline_create_ex(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_net_t* affnet,
                          const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out) {
    return pipeline_create(__func__, cfg, est, affnet, orinet, hardnet, out);
}

void ag_pipeline_destroy(ag_pipeline_t* p) { delete p; }
size_t ag_pipeline_workspace_bytes(const ag_pipeline_t* p) { return p ? p->total : 0; }
const ag_pyramid_plan_t* ag_pipeline_plan(const ag_pipeline_t* p) { return p ? &p->plan : nullptr; }
int ag_pipeline_launch_count(const ag_pipeline_t* p) { return p ? p->launches : 0; }

int ag_pipeline_run(ag_pipeline_t* p, const float* d_img, void* d_ws, size_t ws_bytes, float* d_lafs, float* d_resp,
                    float* d_desc, int* d_count, void* stream) {
    AG_REQUIRE(p && d_img && d_ws && d_lafs && d_resp && d_desc && d_count, "NULL argument");
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
    float* nlafs = (float*)(ws + p->off_nlafs); int* oct3 = (int*)(ws + p->off_oct3); int* lvl3 = (int*)(ws + p->off_lvl3);
    void* netws = ws + p->off_net;
    const int launches0 = g_launches;
    int rc;
    ag_detect_ws_t det;
    if ((rc = ag_detect_ws_carve(&p->plan, p->cand_cap, ws + p->off_det, &det))) return rc;
    if ((rc = ag_pyramid_build(&p->plan, d_img, pyr, stream))) return rc;
    if ((rc = ag_detect(&p->plan, pyr, 0.f, (int)c.mrSize, &det, stream))) return rc;
    const ag_pipeline_estimators_t& e = p->est;
    if (e.shape == AG_SHAPE_NONE) {
        // num_Baum_iters = 0: K keypoints straight from the detector, no shape filter (SparseImgRepresenter.py:192-200)
        if ((rc = ag_select_keypoints(&p->plan, &det, K, (float)c.mrSize, K, d_resp, lafs2, oct2, lvl2, d_count, stream))) return rc;
    } else {
        if ((rc = ag_select_keypoints(&p->plan, &det, M, (float)c.mrSize, M, resp1, lafs1, oct1, lvl1, cnt1, stream))) return rc;
        // affine shape: base_A of getAffineShape's loop (SparseImgRepresenter.py:127-141) into A
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
            const int n = B * M, it_n = e.num_baum_iters;
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
        if ((rc = ag_affine_shape_filter(A, resp1, lafs1, oct1, lvl1, cnt1, B, M, K, K, d_resp, lafs2, oct2, lvl2, d_count, stream))) return rc;
    }
    if (e.ori == AG_ORI_ORINET) {
        if ((rc = ag_net_forward_pyr(p->ori, &p->plan, pyr, lafs2, oct2, lvl2, d_count, K, A, netws, p->net_bytes, stream))) return rc;
        if ((rc = ag_lafs_apply_rotation(lafs2, A, B * K, stream))) return rc;
    } else if (e.ori == AG_ORI_HISTOGRAM) {
        if ((rc = orientation_hist_pyr(&p->plan, pyr, lafs2, oct2, lvl2, d_count, K, e.ori_ps, p->ori_gk.data(), A, stream))) return rc;
        if ((rc = ag_lafs_apply_rotation(lafs2, A, B * K, stream))) return rc;
    }
    // denormalizeLAFs (LAF.py:407-417), then descriptor patches: level choice + normalizeLAFs (LAF.py:419-429)
    const float ms = (float)(c.H < c.W ? c.H : c.W);
    if ((rc = ag_lafs_scale(lafs2, d_lafs, B * K, ms, (float)c.W, (float)c.H, stream))) return rc;
    if ((rc = ag_pyramid_level_for_lafs(&p->plan, d_lafs, B * K, 32, oct3, lvl3, stream))) return rc;
    if ((rc = ag_lafs_scale(d_lafs, nlafs, B * K, 1.0f / ms, (float)(1.0 / (double)c.W), (float)(1.0 / (double)c.H), stream))) return rc;
    if ((rc = ag_net_forward_pyr(p->hard, &p->plan, pyr, nlafs, oct3, lvl3, d_count, K, d_desc, netws, p->net_bytes, stream))) return rc;
    p->launches = g_launches - launches0;
    return AG_OK;
}

}  // extern "C"
