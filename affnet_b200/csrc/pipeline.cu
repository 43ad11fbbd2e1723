// Batched end-to-end pipeline: ScaleSpaceAffinePatchExtractor.forward (SparseImgRepresenter.py:189-209,
// num_Baum_iters=1) + extract_patches_from_pyr (:181-188) + HardNet.forward for B images of one size, as a
// fixed sequence of kernel launches on one stream with fixed-capacity buffers and device-side counters
// (no host synchronisation, CUDA-graph capturable).  The reference processes one image at a time with
// several .item()/nonzero host round trips (SURVEY.md §3); this is the on-device replacement.
#include "common.cuh"

struct ag_pipeline {
    ag_pipeline_config_t cfg;
    ag_pyramid_plan_t plan;
    const ag_net_t* aff;
    const ag_net_t* ori;
    const ag_net_t* hard;
    int M;          // prefilter keypoints per image = int(1.5 K)
    int cand_cap;
    // workspace layout (byte offsets)
    size_t off_pyr, off_det, off_resp1, off_lafs1, off_oct1, off_lvl1, off_cnt1, off_patches, off_A, off_lafs2, off_oct2,
        off_lvl2, off_nlafs, off_oct3, off_lvl3, off_net, net_bytes, total;
    int launches;
};

using namespace ag;

extern "C" {

int ag_pipeline_create(const ag_pipeline_config_t* cfg, const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet,
                       ag_pipeline_t** out) {
    AG_REQUIRE(cfg && affnet && hardnet && out, "NULL argument");
    AG_REQUIRE(!cfg->do_ori || orinet, "do_ori needs an OriNet");
    AG_REQUIRE(cfg->num_features >= 1, "num_features must be positive");
    ag_pipeline* p = new ag_pipeline();
    p->cfg = *cfg; p->aff = affnet; p->ori = orinet; p->hard = hardnet;
    int rc = ag_pyramid_plan(cfg->B, cfg->H, cfg->W, cfg->nlevels, cfg->init_sigma, cfg->border, &p->plan);
    if (rc != AG_OK) { delete p; return rc; }
    p->M = (int)(1.5 * cfg->num_features);  // SparseImgRepresenter.py:194
    if (p->M > 16384) {   // the selection kernels sort in shared memory (ag_select_keypoints / ag_affine_shape_filter): fail here, not at run time
        set_error("ag_pipeline_create: num_features %d needs a prefilter of int(1.5 K) = %d keypoints; the shared-memory selection holds 16384 (K <= 10922)",
                  cfg->num_features, p->M);
        delete p;
        return AG_ERR_CAPACITY;
    }
    p->cand_cap = cfg->cand_cap > 0 ? cfg->cand_cap : (cfg->H * cfg->W) / 8;
    if (p->cand_cap < p->M) p->cand_cap = p->M;
    const size_t B = cfg->B, M = p->M, K = cfg->num_features;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o += align_up(bytes, 256); return r; };
    p->off_pyr = take(sizeof(float) * (size_t)p->plan.total_floats);
    p->off_det = take(ag_detect_ws_bytes(&p->plan, p->cand_cap));
    p->off_resp1 = take(sizeof(float) * B * M);
    p->off_lafs1 = take(sizeof(float) * B * M * 6);
    p->off_oct1 = take(sizeof(int) * B * M);
    p->off_lvl1 = take(sizeof(int) * B * M);
    p->off_cnt1 = take(sizeof(int) * B);
    p->off_patches = 0;  // 32x32 patches are never materialised: the sampler is fused into the first tensor-core layer
    p->off_A = take(sizeof(float) * B * M * 4);
    p->off_lafs2 = take(sizeof(float) * B * K * 6);
    p->off_oct2 = take(sizeof(int) * B * K);
    p->off_lvl2 = take(sizeof(int) * B * K);
    p->off_nlafs = take(sizeof(float) * B * K * 6);
    p->off_oct3 = take(sizeof(int) * B * K);
    p->off_lvl3 = take(sizeof(int) * B * K);
    size_t nb = ag_net_workspace_bytes(AG_NET_AFFNET, (int)(B * M));
    size_t hb = ag_net_workspace_bytes(AG_NET_HARDNET, (int)(B * K));
    p->net_bytes = nb > hb ? nb : hb;
    p->off_net = take(p->net_bytes);
    p->total = o;
    p->launches = 0;
    *out = p;
    return AG_OK;
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
    if ((rc = ag_select_keypoints(&p->plan, &det, M, (float)c.mrSize, M, resp1, lafs1, oct1, lvl1, cnt1, stream))) return rc;
    // affine shape (one AffNet iteration)
    if ((rc = ag_net_forward_pyr(p->aff, &p->plan, pyr, lafs1, oct1, lvl1, cnt1, M, A, netws, p->net_bytes, stream))) return rc;
    if ((rc = ag_affine_shape_filter(A, resp1, lafs1, oct1, lvl1, cnt1, B, M, K, K, d_resp, lafs2, oct2, lvl2, d_count, stream))) return rc;
    if (c.do_ori) {
        if ((rc = ag_net_forward_pyr(p->ori, &p->plan, pyr, lafs2, oct2, lvl2, d_count, K, A, netws, p->net_bytes, stream))) return rc;
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
