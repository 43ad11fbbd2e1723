/*
 * affnet_b200 C ABI  --  the drop-in boundary of the H100-native HesAffNet + HardNet hot path.
 *
 * The reference (ducha-aiki/affnet) has no FFI: its boundary is the Python module API
 * (SURVEY.md §8b).  The thin Python mirror in `affnet_b200/` keeps those names and calls ONLY the
 * entry points below (ctypes).  Each entry point cites the reference code it replaces.
 *
 * Conventions
 *   - plain pointers and sizes only; every `d_*` pointer is DEVICE memory owned by the caller,
 *     every `h_*` pointer is HOST memory.  The library never allocates result buffers and never
 *     synchronises the stream (except the two `*_create` functions, which upload weights).
 *   - `stream` is a `cudaStream_t` passed as `void*`; all work is enqueued on it.
 *   - return value: 0 on success, negative `AG_ERR_*` otherwise; `ag_last_error()` gives a message.
 *   - images / pyramid levels are float32 `[B, h, w]` (single channel, batch-major), 0..255 scale.
 *   - LAFs are float32 `[n, 2, 3]` = [[a11 a12 x], [a21 a22 y]]; "normalised" means A in units of
 *     min(h,w) and (x,y) in units of (w,h)  (LAF.py:407-429).
 *   - fixed-capacity outputs: rows >= count are unspecified; counts live in device int32 arrays.
 */
#ifndef AFFNET_B200_H
#define AFFNET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AG_OK 0
#define AG_ERR_INVALID -1   /* bad argument */
#define AG_ERR_CUDA -2      /* a CUDA runtime call failed */
#define AG_ERR_CAPACITY -3  /* a fixed-capacity buffer is too small */
#define AG_ERR_NO_DEVICE -4 /* no sm_90 device / kernel image not loadable */

#define AG_MAX_OCTAVES 16
#define AG_MAX_LEVELS 8 /* nlevels + 2 */

const char* ag_last_error(void);
/* ABI version of this header; bumps when a signature changes. */
int ag_abi_version(void);

/* Per-launch CUDA-event profiler (used by bench.py for the roofline leg; new, no reference counterpart).
 * Between ag_prof_begin(stream) and ag_prof_end() every kernel the library launches is followed by an event
 * record on `stream`; ag_prof_end() synchronises and returns the number of launches (or <0), ag_prof_get(i)
 * the name and duration in ms of launch i. */
int ag_prof_begin(void* stream);
int ag_prof_end(void);
int ag_prof_get(int i, const char** name, float* ms);

/* ------------------------------------------------------------------------------------------
 * Scale pyramid                   replaces ScalePyramid.forward  (HandCraftedModules.py:13-56)
 *                                 and GaussianBlur               (Utils.py:92-114,150-166)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    int B, H, W;
    int n_octaves;
    int n_levels;                                        /* nlevels + 2 maps per octave */
    int h[AG_MAX_OCTAVES], w[AG_MAX_OCTAVES];            /* ceil-halved sizes (Q6) */
    long long level_offset[AG_MAX_OCTAVES][AG_MAX_LEVELS]; /* in floats from the pyramid base; each level is [B,h,w] */
    long long total_floats;
    double sigma[AG_MAX_OCTAVES][AG_MAX_LEVELS];         /* sigmas[o][l] of the reference (python floats) */
    double blur_sigma[AG_MAX_OCTAVES][AG_MAX_LEVELS];    /* sigma of the blur that produces level l (0: decimation) */
    double pix_dist[AG_MAX_OCTAVES];                     /* 2^o */
} ag_pyramid_plan_t;

/* Host-only: sizes, sigmas and buffer offsets (HandCraftedModules.py:15-22, 23-56 loop logic). */
int ag_pyramid_plan(int B, int H, int W, int nlevels, double init_sigma, int border, ag_pyramid_plan_t* plan);

/* d_img [B,H,W] -> d_pyr (plan->total_floats floats). */
int ag_pyramid_build(const ag_pyramid_plan_t* plan, const float* d_img, float* d_pyr, void* stream);

/* One Gaussian blur exactly as GaussianBlur(sigma)(x): k=int(6 sigma+1)|1 taps at linspace(-k/2,k/2,k),
 * replicate padding (Utils.py:150-166).  d_in/d_out [B,h,w]. */
int ag_gaussian_blur(const float* d_in, float* d_out, int B, int h, int w, double sigma, void* stream);

/* ------------------------------------------------------------------------------------------
 * Hessian response                replaces HessianResp.forward   (HandCraftedModules.py:58-78)
 * out = max(|gxx*gyy - gxy^2| * sigma^4 - th, 0)   (clamp: SparseImgRepresenter.py:77-84)
 * ------------------------------------------------------------------------------------------ */
int ag_hessian_response(const float* d_in, float* d_out, int B, int h, int w, double sigma, float th, void* stream);

/* ------------------------------------------------------------------------------------------
 * Detector: 3x3x3 NMS + border + octave map + soft-argmax + compaction
 *                                 replaces NMS3dAndComposeA.forward (HandCraftedModules.py:222-291)
 *                                 and the loop of multiScaleDetector (SparseImgRepresenter.py:53-111)
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    int B;
    int cand_cap;              /* capacity of the candidate list per image */
    int n_level_slots;         /* n_octaves * (n_levels-2) detection levels */
    /* device buffers, caller-allocated (sizes in elements) */
    float* d_cand_val;         /* [B, cand_cap]   response after octave-map masking (may be negative, Q4) */
    uint32_t* d_cand_seq;      /* [B, cand_cap]   (level_slot << 27) | flat pixel index; 0xFFFFFFFF = dropped */
    float* d_cand_scyx;        /* [B, cand_cap, 3] normalised (scale, y, x) */
    float* d_cand_aux;         /* [B, cand_cap, 2] raw NMS value of the same pixel at the octave's detection levels 1 and 2 */
    int* d_cand_count;         /* [B]             number appended (may exceed cand_cap -> overflow) */
    int* d_level_pos;          /* [B, n_level_slots] count of responses > 0 at each detection level */
    int* d_level_emit;         /* [B, n_level_slots] count of non-zero responses at each level */
    int* d_variants;           /* [B, n_octaves, 16] acceptance-hypothesis counters of the fused detector */
    uint8_t* d_octave_maps;    /* [4 * B * sum_o h_o*w_o] scratch for the octave maps (uint8, Q4 semantics) */
} ag_detect_ws_t;

/* Bytes needed for each workspace member are fixed by the struct comments; helper for callers: */
size_t ag_detect_ws_bytes(const ag_pyramid_plan_t* plan, int cand_cap);
/* Carves `d_ws` (ag_detect_ws_bytes bytes, 256-B aligned) into the struct's pointers. */
int ag_detect_ws_carve(const ag_pyramid_plan_t* plan, int cand_cap, void* d_ws, ag_detect_ws_t* ws);

/* All octaves/levels, Hessian fused (responses never touch HBM).  mr_border = int(mrSize). */
int ag_detect(const ag_pyramid_plan_t* plan, const float* d_pyr, float th, int mr_border, ag_detect_ws_t* ws, void* stream);

/* One detection level from precomputed response maps (B=1), for stage-isolated parity:
 * d_low/d_cur/d_high [h,w]; d_omap_in / d_omap_out uint8 [h,w] (in may be NULL = zeros).
 * Appends to ws (level slot `slot`), exactly like NMS3dAndComposeA given the same maps. */
int ag_detect_level_from_responses(const float* d_low, const float* d_cur, const float* d_high, int h, int w,
                                   const double scales[3], int mr_border, const uint8_t* d_omap_in,
                                   uint8_t* d_omap_out, int slot, ag_detect_ws_t* ws, void* stream);

/* Global selection (SparseImgRepresenter.py:100-111 + per-level rule HandCraftedModules.py:252-263):
 * levels with <=1 positive response are dropped; if more than num_features candidates remain the
 * top num_features by (response desc, seq asc) are returned sorted, otherwise all in
 * (octave, level, raster) order.  num_features <= 0 returns everything (capacity permitting).
 * out_cap bounds the rows written: when it is below the number the rule above selects, the first out_cap rows of that answer
 * are returned in the same order (the out_cap highest by (response desc, seq asc) when sorted, else the out_cap first in
 * (octave, level, raster) order), deterministically.  min(num_features, out_cap) (out_cap when num_features <= 0) may not
 * exceed 16384 (shared-memory sort): larger requests return AG_ERR_CAPACITY and write nothing (ag_select_topk_keypoints has no limit).
 * a_scale multiplies the A part of the LAF (mrSize; SparseImgRepresenter.py:198).
 * Outputs [B, out_cap(,..)]: resp, LAFs (normalised), octave idx, level idx (= detection level-1); d_count[b] = -1 if the
 * candidate list of image b overflowed ws->cand_cap (the caller should retry with a larger capacity). */
int ag_select_keypoints(const ag_pyramid_plan_t* plan, const ag_detect_ws_t* ws, int num_features, float a_scale,
                        int out_cap, float* d_resp, float* d_lafs, int* d_oct, int* d_lvl, int* d_count,
                        void* stream);

/* Ordered keep-all selection at any count (threshold mode, SparseImgRepresenter.py:104-110 with num = -1): for each image, every candidate of
 * the accepted levels (more than one positive response) in (octave, level, raster) order, the A part of the LAF scaled by a_scale.  The
 * rows equal ag_select_keypoints(num_features <= 0, out_cap >= their number) bit for bit, and there is no 16384 limit: a bitmap over the
 * detection levels' pixels and per-word popcount prefixes give each candidate its row, without a sort.
 * d_count[b] = -1 when image b's candidate list overflowed ws->cand_cap or when it has more than out_cap keypoints; nothing of such an
 * image is written.  Rows at or beyond d_count[b] are never written.
 * d_scratch: ag_select_all_workspace_bytes(plan, ws->cand_cap) bytes, 256-B aligned, any content (about B * 8 bytes per 32 pixels of
 * every detection level: the size is set by the pyramid, cand_cap only has to be positive).  A memset and four launches, deterministic,
 * no host synchronisation (CUDA-graph capturable).  AG_ERR_CAPACITY for a smaller scratch, before any CUDA call. */
size_t ag_select_all_workspace_bytes(const ag_pyramid_plan_t* plan, int cand_cap);
int ag_select_all_keypoints(const ag_pyramid_plan_t* plan, const ag_detect_ws_t* ws, float a_scale, int out_cap,
                            void* d_scratch, size_t scratch_bytes, float* d_resp, float* d_lafs, int* d_oct, int* d_lvl,
                            int* d_count, void* stream);

/* Top-K selection at any count: the rule, order, out_cap truncation and outputs of ag_select_keypoints without its 16384 limit.  When
 * min(num_features, out_cap) (out_cap when num_features <= 0) is at most 16384 it runs ag_select_keypoints itself (bit-identical by
 * construction; no scratch is needed).  Above that a cluster radix select of the cut key, a compaction and a global-memory sort (shared-memory
 * tiles, then merge passes) produce the same answer: the number of launches is fixed on the host from out_cap and num_features, and each
 * launch reads the device counts (no host synchronisation, CUDA-graph capturable).  In that regime an image whose candidate list overflowed
 * ws->cand_cap gets d_count[b] = -1 and nothing of it is written.
 * d_scratch: ag_select_topk_workspace_bytes(plan, ws->cand_cap, out_cap) bytes, 256-B aligned, any content (0 when out_cap <= 16384, else
 * about B * out_cap * 24 bytes); d_scratch may be NULL when scratch_bytes is 0.  AG_ERR_CAPACITY for a smaller scratch, before any CUDA call. */
size_t ag_select_topk_workspace_bytes(const ag_pyramid_plan_t* plan, int cand_cap, int out_cap);
int ag_select_topk_keypoints(const ag_pyramid_plan_t* plan, const ag_detect_ws_t* ws, int num_features, float a_scale, int out_cap,
                             void* d_scratch, size_t scratch_bytes, float* d_resp, float* d_lafs, int* d_oct, int* d_lvl, int* d_count,
                             void* stream);

/* ------------------------------------------------------------------------------------------
 * Affine bilinear sampler          replaces extract_patches / generate_patch_grid_from_normalized_LAFs
 *                                  (LAF.py:313-372) and extract_patches_from_pyramid_with_inv_index
 *                                  (LAF.py:376-404)
 * out[n,c,i,j] = bilinear(img, p-0.5), p = A*min(h,w)*(xj,yi) + (x*w, y*h), xj=(2j+1)/PS-1, zeros outside
 * ------------------------------------------------------------------------------------------ */
/* Single image [C,h,w] (or per-patch images [n,C,h,w] when per_patch_img != 0), LAFs [n,2,3] normalised. */
int ag_extract_patches(const float* d_img, int C, int h, int w, int per_patch_img, const float* d_lafs, int n,
                       int PS, float* d_out, void* stream);

/* From the pyramid: image b of the batch, LAF i sampled at pyr[oct[i]][lvl[i]].  d_lafs [B,cap,2,3],
 * d_oct/d_lvl [B,cap], d_count [B] (NULL => all `cap` rows valid), d_out [B,cap,PS,PS]. */
int ag_extract_patches_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct,
                           const int* d_lvl, const int* d_count, int cap, int PS, float* d_out, void* stream);

/* get_pyramid_and_level_index_for_LAFs (LAF.py:450-472): float64 argmin of |sigma_l*2^o - sqrt(|det A|+1e-12)/PS|.
 * d_dlafs [n,2,3] in pixel units. */
int ag_pyramid_level_for_lafs(const ag_pyramid_plan_t* plan, const float* d_dlafs, int n, int PS, int* d_oct,
                              int* d_lvl, void* stream);

/* ------------------------------------------------------------------------------------------
 * The three CNNs                    replaces AffNetFast.forward (architectures.py:204-252),
 *                                   OriNetFast.forward (architectures.py:33-82), HardNet.forward (HardNet.py:61-101)
 * ------------------------------------------------------------------------------------------ */
#define AG_NET_AFFNET 0
#define AG_NET_ORINET 1
#define AG_NET_HARDNET 2

typedef struct ag_net ag_net_t;

/* h_blob: the checkpoint tensors flattened in state_dict order without num_batches_tracked:
 * for each of the 6 conv layers: weight[Cout,Cin,3,3], running_mean[Cout], running_var[Cout];
 * then features.19.weight[Cout,Cin,8,8]; then bias[Cout] (AffNet, OriNet) or running_mean, running_var (HardNet).
 * BatchNorm (affine=False, eps 1e-5) is folded into the conv weights at upload. */
int ag_net_create(int kind, const float* h_blob, size_t n_floats, ag_net_t** out);
void ag_net_destroy(ag_net_t* net);
size_t ag_net_blob_floats(int kind);
/* Compute engine: 0 = exact fp32 SIMT (needs materialised patches);
 * 4 = tensor-core engine, THE DEFAULT for all three nets: fp16 operands, fp32 accumulation, all six conv layers and the 8x8 heads as
 * MMAs; AffNet and OriNet carry fp16 residual planes of weights AND activations in every layer (fp32-grade - OriNet's atan2 amplifies
 * an error of AffNet's A about 15x, so the 1e-3 LAF contract needs A to 5e-5), HardNet fp16 operands with fp16 residuals of its
 * layer 2-3 weights (descriptors 4e-4); 64-pixel row tiles without x padding, the three taps of a kernel row stacked along N of one
 * MMA, x shifts by warp shuffles in the epilogue;
 * 5 = engine 4 with bf16 operands (HardNet only; BASELINE.json configs[4] "bf16 HardNet tensor-core path"; descriptors ~4e-3).
 * Any other value is refused with AG_ERR_INVALID and leaves the engine as it was. */
int ag_net_set_engine(ag_net_t* net, int engine);
int ag_net_get_engine(const ag_net_t* net);
/* Developer diagnostic: run the trunk with the handle's engine on materialised patches [n,32,32] up to conv layer `upto` and return that
 * layer's activations as fp32 [n,C,H,H].  ENGINE_SIMT: the exact-fp32 trunk, upto 1..6, its fp32 output as it is.  Any other engine: the
 * second-generation trunk (ENGINE_TC2_BF16: bf16 operands, HardNet; otherwise fp16), upto 2..6, its hi [+ lo] planes in the engine's HBM
 * layout (layer 6: the 8x8 head's operand) decoded.  d_ws: ag_net_workspace_bytes(). */
int ag_debug_tcx_layer(const ag_net_t* net, const float* d_patches, int n, int upto, float* d_out, void* d_ws, size_t ws_bytes, void* stream);
/* Developer diagnostic: d_y[i] = tanhf(d_x[i]) for i < n, compiled with the flags of the exact-fp32 engine's AffNet and OriNet heads.
 * Lets a test restate those heads bit for bit (tests/nets_simt_restated.py); not used by the pipeline. */
int ag_debug_tanhf(const float* d_x, int n, float* d_y, void* stream);
/* Developer diagnostic: the device libm calls of the hand-crafted estimators, compiled with their flags, one element per thread:
 * d_atan2[i] = atan2f(d_y[i], d_x[i]), d_cos[i] = cosf(d_x[i]), d_sin[i] = sinf(d_x[i]) for i < n.  Lets a test restate the estimators
 * bit for bit (tests/handcrafted_restated.py); not used by the pipeline. */
int ag_debug_libm(const float* d_y, const float* d_x, int n, float* d_atan2, float* d_cos, float* d_sin, void* stream);
/* Developer diagnostic: the batched pipeline's fused hand-crafted estimators called directly (same layout as ag_extract_patches_pyr;
 * d_count [B] required; h_gk [PS,PS] in host memory, 3 <= PS <= 41).  Rows at or beyond d_count[b] are not written.
 *   ag_debug_orientation_hist_pyr  d_R [B,cap,2,2] = [[cos, sin], [-sin, cos]] of the gradient-histogram angle of each sampled patch
 *   ag_debug_baumberg_pyr          d_A [B,cap,2,2] = base_A after `iters` >= 1 Baumberg iterations (SparseImgRepresenter.py:127-141) */
int ag_debug_orientation_hist_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                                  const int* d_count, int cap, int PS, const float* h_gk, float* d_R, void* stream);
int ag_debug_baumberg_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                          const int* d_count, int cap, int PS, int iters, const float* h_gk, float* d_A, void* stream);
/* Scratch bytes for a forward over n patches. */
size_t ag_net_workspace_bytes(int kind, int n);

/* d_patches [n,1,32,32] (any scale: per-patch mean/std normalisation is part of forward).
 * Row validity: rows are grouped in groups of `group` rows (group <= 0 => one group of n rows); if d_count is
 * not NULL, only the first d_count[g] rows of group g are computed (device int32 array), else all rows.  Rows beyond `d_count` are
 * not written (d_out / d_angle keep what the caller left there), and every engine gives a valid row the same bits whatever the other
 * rows hold and whatever the workspace held before the call (tests/test_gpu_rows.py).
 * AffNet -> d_out [n,2,2] rectified A.   OriNet -> d_out [n,2,2] rotation (and/or d_angle [n]; either may be NULL).
 * HardNet -> d_out [n,128] L2-normalised. */
int ag_affnet_forward(const ag_net_t* net, const float* d_patches, int n, const int* d_count, int group, float* d_out,
                      void* d_ws, size_t ws_bytes, void* stream);
int ag_orinet_forward(const ag_net_t* net, const float* d_patches, int n, const int* d_count, int group, float* d_out,
                      float* d_angle, void* d_ws, size_t ws_bytes, void* stream);
int ag_hardnet_forward(const ag_net_t* net, const float* d_patches, int n, const int* d_count, int group, float* d_out,
                       void* d_ws, size_t ws_bytes, void* stream);

/* f4: the TorchScript exports' contract (convertJIT/AffNetJIT.pt, OriNetJIT.pt; convert_OriNet_and_AffNet_to_JIT.ipynb): the RAW head
 * outputs.  AffNet: xy + [1, 0, 1] = (1 + x0, x1, 1 + x2) -> d_raw [n,3] (architectures.py:228-230 before rectification);
 * OriNet: the mean over the 3x3 map of tanh(conv8x8) -> d_raw [n,2] = (sin-like, cos-like) (architectures.py:57-59,76).
 * Tensor-core engine (4) only. */
int ag_affnet_forward_raw(const ag_net_t* net, const float* d_patches, int n, float* d_raw, void* d_ws, size_t ws_bytes, void* stream);
int ag_orinet_forward_raw(const ag_net_t* net, const float* d_patches, int n, float* d_raw, void* d_ws, size_t ws_bytes, void* stream);
/* Fused sampler + net (tensor-core engine): LAF i of image b is sampled at pyr[oct][lvl] INSIDE the first tensor-core
 * layer (32x32 patches never touch HBM), then the net runs as above.  Layout as ag_extract_patches_pyr: d_lafs
 * [B,cap,2,3] normalised, d_oct/d_lvl [B,cap], d_count [B] or NULL (rows beyond d_count[b] of image b are not written).
 * d_out: [B*cap,2,2] (AffNet, OriNet) or [B*cap,128].  The fp32 SIMT engine (0) is refused with AG_ERR_INVALID. */
int ag_net_forward_pyr(const ag_net_t* net, const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct,
                       const int* d_lvl, const int* d_count, int cap, float* d_out, void* d_ws, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Keypoint geometry                 replaces getAffineShape's filter (SparseImgRepresenter.py:136-162,
 *                                   Utils.py:168-175, LAF.py:98-104), getOrientation's compose (:175),
 *                                   denormalizeLAFs / normalizeLAFs (LAF.py:407-429)
 * ------------------------------------------------------------------------------------------ */
/* Per image b (B images, `cap` rows each, d_count_in[b] valid):  new_LAF = [A*LAF_A, t]; keep where
 * 1/6 < |l1/(l2+1e-8)| < 6 and the LAF does not touch the boundary; if survivors > num_features keep the
 * top num_features by resp * keep (desc; ties by index, -0 equal to +0) else all survivors in order.  In the first case the response
 * written is resp * keep, so a rejected row that makes the cut (when survivors have negative responses) comes out as 0, as
 * torch.topk returns it in the reference.  All arithmetic is the reference's fp32 CPU arithmetic, without fused multiply-adds
 * (tests/test_gpu_geometry.py pins it bit for bit).
 * Outputs are compacted: d_resp_out/d_lafs_out/d_oct_out/d_lvl_out [B,out_cap..], d_count_out [B]; only the first d_count_out[b] rows
 * of image b are written, and d_count_out[b] = -1 where d_count_in[b] < 0.  cap above 16384 returns AG_ERR_CAPACITY and writes nothing
 * (ag_affine_shape_filter_topk has no limit). */
int ag_affine_shape_filter(const float* d_A, const float* d_resp, const float* d_lafs, const int* d_oct,
                           const int* d_lvl, const int* d_count_in, int B, int cap, int num_features, int out_cap,
                           float* d_resp_out, float* d_lafs_out, int* d_oct_out, int* d_lvl_out, int* d_count_out,
                           void* stream);
/* Keep-all shape filter at any cap (getAffineShape's num_features <= 0 branch, SparseImgRepresenter.py:151-156): every survivor of image b
 * in index order with its response unchanged, written to rows 0 .. d_count_out[b]-1 of [B,cap..] outputs.  Bit-identical to
 * ag_affine_shape_filter(num_features = 0, out_cap = cap) wherever that accepts the call (same device arithmetic), with no cap limit and
 * no workspace.  d_count_out[b] = -1 where d_count_in[b] < 0; a count above cap is read as cap.  One launch. */
int ag_affine_shape_filter_all(const float* d_A, const float* d_resp, const float* d_lafs, const int* d_oct, const int* d_lvl,
                               const int* d_count_in, int B, int cap, float* d_resp_out, float* d_lafs_out, int* d_oct_out,
                               int* d_lvl_out, int* d_count_out, void* stream);
/* Top-K shape filter at any cap: the rule, order, responses and counts of ag_affine_shape_filter without its 16384 limit.  At cap <= 16384
 * it runs ag_affine_shape_filter itself (bit-identical by construction; no scratch is needed).  Above, one pass writes every row's keep flag
 * and key, then the global-memory top-K of ag_select_topk_keypoints picks and sorts the rows, and the writer recomputes them with the same
 * device arithmetic.  A memset and a number of launches fixed on the host from cap, num_features and out_cap; CUDA-graph capturable.
 * d_scratch: ag_affine_shape_filter_topk_workspace_bytes(B, cap) bytes, 256-B aligned, any content (0 when cap <= 16384, else about
 * B * cap * 29 bytes); d_scratch may be NULL when scratch_bytes is 0.  AG_ERR_CAPACITY for a smaller scratch, before any CUDA call. */
size_t ag_affine_shape_filter_topk_workspace_bytes(int B, int cap);
int ag_affine_shape_filter_topk(const float* d_A, const float* d_resp, const float* d_lafs, const int* d_oct, const int* d_lvl,
                                const int* d_count_in, int B, int cap, int num_features, int out_cap, void* d_scratch, size_t scratch_bytes,
                                float* d_resp_out, float* d_lafs_out, int* d_oct_out, int* d_lvl_out, int* d_count_out, void* stream);

/* LAF_A <- LAF_A * R  then (optionally) denormalise to pixels of a WxH image.  d_lafs [n,2,3] in/out. */
int ag_lafs_apply_rotation(float* d_lafs, const float* d_R, int n, void* stream);
int ag_lafs_scale(const float* d_in, float* d_out, int n, float a_coef, float x_coef, float y_coef, void* stream);
/* The 2x2 chain of the Baumberg iterations (SparseImgRepresenter.py:127-141, torch.bmm there): d_out [n,2,2] = d_A * d_B;
 * d_out [n,2,3] = [d_A * d_lafs[:, :, :2] | d_lafs[:, :, 2]]. */
int ag_mat2_compose(const float* d_A, const float* d_B, float* d_out, int n, void* stream);
int ag_lafs_left_multiply(const float* d_A, const float* d_lafs, float* d_out, int n, void* stream);
/* Output format of the reference's writers (hesaffBaum.py:46-48): replaces LAFs2ellT (LAF.py:35-51, bsvd2x2 :106-144).
 * d_lafs [n,2,3] in pixels -> d_ell [n,5] = (x, y, a, b, c) with a u^2 + 2 b u v + c v^2 = 1.  A LAF with a negative
 * determinant gives NaN, as in the reference. */
int ag_lafs_to_ell(const float* d_lafs, int n, float* d_ell, void* stream);
/* The reference's reader of that format: replaces ells2LAFsT (LAF.py:76-89, invSqrtTorch :52-74, rectifyAffineTransformationUpIsUp
 * :285-291).  d_ell [n,5] = (x, y, a, b, c) -> d_lafs [n,2,3] in pixels, upright (A[0][1] = 0).  Each torch operation of the reference is
 * one fp32 operation in its order (IEEE division and square root, no fused multiply-add), so the rows equal the reference's fp32 CPU
 * result bit for bit, including the b == 0 branch and the NaN of an ellipse that is not positive definite.  One launch. */
int ag_ells_to_lafs(const float* d_ell, int n, float* d_lafs, void* stream);

/* ------------------------------------------------------------------------------------------
 * Hand-crafted estimators (SURVEY.md §8f "next" rows): what the reference uses when OriNet / AffNet are None.
 *   ag_orientation_hist  replaces OrientationDetector.forward   (HandCraftedModules.py:133-192): 36-bin gradient histogram,
 *                        (0.33,0.34,0.33) smoothing, arg-max -> angle [n]
 *   ag_baumberg_shape    replaces AffineShapeEstimator.forward  (HandCraftedModules.py:81-132): second-moment matrix ->
 *                        inverse square root -> up-is-up rectified A [n,2,2]
 * d_patches [n,PS,PS] (3 <= PS <= 41); d_gk [PS,PS] = the module's Gaussian window: ag_circular_gauss_kernel(PS, sigma, h_out)
 * reproduces CircularGaussKernel (Utils.py:92-114; sigma <= 0 selects the default sigma^2 = 0.9 (PS/2)^2 / 2); the orientation
 * window is 10x that kernel, the Baumberg window uses sigma = (PS/2)/3.
 * ------------------------------------------------------------------------------------------ */
int ag_circular_gauss_kernel(int kernlen, double sigma, float* h_out);
int ag_orientation_hist(const float* d_patches, int n, int PS, const float* d_gk, float* d_angle, void* stream);
int ag_baumberg_shape(const float* d_patches, int n, int PS, const float* d_gk, float* d_A, void* stream);

/* SIFT descriptor: replaces SIFTNet.forward (pytorch_sift.py:69-94) with 8 angle bins and 4 x 4 spatial bins -> [n,128] in
 * [bin][cy][cx] order: (-1, 0, 1) gradients with replicate borders, magnitude times the module's Gaussian window, angle bins
 * interpolated linearly, a k x k tent pooling with stride s per angle bin, L2 normalisation, clamp(0, clipval), L2 normalisation.
 * Supported patch sizes: 16..65 where the pooling grid comes out 4 x 4 (all but 17, 18, 23, 28, 38, 48, 58); AG_ERR_INVALID otherwise.
 *   ag_sift_windows       host only: SIFTNet.CircularGaussKernel h_gk [PS,PS] (centre PS/2, not normalised) and getPoolingKernel
 *                         h_pk [k,k], with k = 2 s - 1 and s = round(2 floor(PS/2) / 5), as SIFTNet.__init__ builds them in float64 and
 *                         rounds to fp32.  Any output may be NULL.
 *   ag_sift_describe      d_patches [n,PS,PS] -> d_out [n,128].  clipval finite and positive (the reference's 0.2).
 *   ag_sift_describe_pyr  samples each keypoint's patch from the pyramid as ag_extract_patches_pyr does (same layout, d_count [B] or
 *                         NULL) and describes it without writing the patch: d_out [B,cap,128], bit-identical to ag_extract_patches_pyr
 *                         followed by ag_sift_describe.  Rows at or beyond d_count[b] (all of them for a count of -1) are not written.
 * Deterministic: a row's bits do not depend on the launch or the other rows.  One launch; no allocation. */
int ag_sift_windows(int PS, float* h_gk, float* h_pk, int* k, int* stride);
int ag_sift_describe(const float* d_patches, int n, int PS, float clipval, float* d_out, void* stream);
int ag_sift_describe_pyr(const ag_pyramid_plan_t* plan, const float* d_pyr, const float* d_lafs, const int* d_oct, const int* d_lvl,
                         const int* d_count, int cap, int PS, float clipval, float* d_out, void* stream);

/* Descriptor matching (SURVEY.md §8f row 3).
 *   ag_distance_matrix replaces distance_matrix_vector (Losses.py:5-13): out[n1,n2] = sqrt(|a|^2 + |b|^2 - 2 a.b + 1e-6)
 *   ag_match_snn       replaces the SNN-ratio block of train_AffNet_test_on_graffity.py:292-298: nearest neighbour, then
 *                      `dist[:, idxs_in_2] = 100000` (all columns that are anybody's nearest neighbour), second minimum,
 *                      keep[i] = min/(second + 1e-8) <= ratio.   Outputs [n1]: d_idx2, d_min, d_second, d_keep (uint8).
 *   ag_distance_matrix refuses n1 above 4194240 rows (65535 tiles of 64), as ag_match_pairs refuses such a cap1, before any CUDA call. */
int ag_distance_matrix(const float* d_a, int n1, const float* d_b, int n2, int dim, float* d_out, void* stream);
size_t ag_match_snn_workspace_bytes(int n1, int n2);
int ag_match_snn(const float* d_desc1, int n1, const float* d_desc2, int n2, int dim, float ratio, void* d_ws, size_t ws_bytes, int* d_idx2,
                 float* d_min, float* d_second, unsigned char* d_keep, void* stream);

/* Batched SNN matcher (new; the reference matches one pair at a time): ag_match_snn's rule for every pair p = (i, j) of a list, between
 * image i of set 1 (d_desc1 [S1,cap1,dim], d_count1 [S1]) and image j of set 2 (d_desc2 [S2,cap2,dim], d_count2 [S2]), on
 * d_desc1[i, :count1[i]] and d_desc2[j, :count2[j]].  Set 2 may be set 1.  A NULL count array means every image has cap rows;
 * d_pairs [P,2] int32, or NULL for pair p = (p, p) (then S1 == S2 == P).  Counts and pair indices are read on the device.
 * Per pair: nearest neighbour (min, lowest column among the minima, NaN ignored, (+inf, 0) for a row with nothing below +inf), the
 * columns that are the nearest neighbour of any row of the pair set to 100000, the second minimum (fminf), keep = min/(second+1e-8) <=
 * ratio, and the kept rows compacted in ascending order: d_tent[p, t] = (row, idx2[row]) for t < d_ntent[p].
 *   d_idx2, d_min, d_second, d_keep [P,cap1]; d_tent [P,cap1,2] and d_ntent [P] (both may be NULL: no compaction).
 *   d_ntent[p] = -1 for a pair with an index out of range or a count outside 0..cap (the pipeline's -1 overflow count), 0 when either
 *   image has no rows; nothing else of such a pair is written.  Rows at or beyond count1[i] and tentative rows at or beyond d_ntent[p]
 *   are not written.  The distance matrix is never stored: d_ws holds the row norms and a column mask per pair.
 * Enqueues 4 or 5 launches and a memset whatever P is; no allocation, no synchronisation (CUDA-graph capturable).
 * AG_ERR_INVALID: NULL descriptors, workspace or outputs, dim / S / cap / P < 1, d_pairs == NULL with S1 != S2 or P != S1, cap1 above
 * 4194240.  AG_ERR_CAPACITY: ws_bytes below ag_match_pairs_workspace_bytes().  Both are checked before any CUDA call. */
size_t ag_match_pairs_workspace_bytes(int S1, int cap1, int S2, int cap2, int P);
int ag_match_pairs(const float* d_desc1, const int* d_count1, int S1, int cap1, const float* d_desc2, const int* d_count2, int S2, int cap2,
                   int dim, const int* d_pairs, int P, float ratio, void* d_ws, size_t ws_bytes, int* d_idx2, float* d_min, float* d_second,
                   unsigned char* d_keep, int* d_tent, int* d_ntent, void* stream);

/* Geometric verification of the batched matcher's tentatives (new; the reference verifies one pair at a time on the CPU).  Both take
 * ag_match_pairs' outputs as they are: LAFs of set 1 d_lafs1 [S1,cap1,2,3] and set 2 d_lafs2 [S2,cap2,2,3] (pixel LAFs of the pipeline),
 * d_pairs [P,2] (NULL: pair p = (p, p), then S1 == S2 == P), d_tent [P,tcap,2] and d_ntent [P].  Tentative t of pair p = (i, j) joins the
 * centre lafs1[i, tent[p,t,0], :, 2] with lafs2[j, tent[p,t,1], :, 2].  Everything is read on the device; one launch whatever P is, no
 * allocation, no synchronisation (CUDA-graph capturable), no workspace.
 * A pair with ntent outside 0..tcap, an image index out of range or a tentative row outside 0..cap-1 gets -1 in its count (d_ninl /
 * d_ntrue) and nothing else of it is written.  Rows at or beyond ntent[p] are not written.
 * AG_ERR_INVALID, before any CUDA call: NULL inputs or outputs, S / cap / P < 1, d_pairs == NULL with S1 != S2 or P != S1, tcap outside
 * 1..4194240, and the parameter ranges given below.
 *
 * ag_homography_ransac: homography RANSAC per pair (the notebook's ransac_validate, findHomography(src, dst, 2.0, 0.99, 50000)),
 * deterministic for a given seed and independent of P and of the pair's position in the list.  Hypothesis h draws 4 distinct indices
 * from splitmix64(splitmix64((h << 32) | draw) ^ seed) (at most 64 draws), rejects samples with a collinear triplet in either image or a
 * triplet orientation that differs between the images for some but not all triplets, and solves H = M2 adj(M1) in fp64 (M maps the
 * projective basis onto the 4 points).  Inlier: h20 x + h21 y + h22 > 0 and |H x1 - x2|^2 <= inl_th^2 in fp64.  Best: most inliers,
 * ties to the lowest h.  Hypotheses are evaluated in chunks of 256; after each chunk the search stops once the number evaluated reaches
 * min(N, max_iters), N = ceil(log(1 - confidence) / log(1 - (best/n)^4)).  Then up to 3 rounds of normalised-DLT least squares on the
 * inliers, each kept only if the inlier count does not drop.
 *   d_H [P,3,3] (H[2][2] = 1), d_inl [P,tcap] u8, d_ninl [P], d_iters [P] (hypotheses evaluated; may be NULL).  n < 4 tentatives or no
 *   hypothesis with an inlier: ninl = 0, H = 0, mask rows < n = 0.
 *   AG_ERR_INVALID also for inl_th not finite and > 0, confidence outside (0, 1), max_iters < 1.
 * ag_fundamental_ransac: fundamental-matrix RANSAC per pair (the notebook's alternative, findFundamentalMatrix(src, dst, 0.5)), for
 * scenes with depth, which one homography does not explain; the arguments, refusals and -1 rule of ag_homography_ransac.  Everything is
 * fp64 in a fixed operation order.  The centres of the rows whose four coordinates are finite are Hartley-normalised (centroid, scale
 * sqrt(2) / RMS radius) once per pair.  Hypothesis h draws 7 distinct indices with the homography's sampler; its 7x9 constraint matrix
 * is reduced by Gauss-Jordan elimination with partial pivoting (a column whose best pivot is <= 1e-9 max|A| is free; rank < 7, or a
 * non-finite centre, is a degenerate sample).  The two null vectors F1, F2, each scaled to unit norm, give the cubic
 * det(l F1 + (1 - l) F2), whose real roots are found with + - * / sqrt only (critical points by the quadratic formula, sign changes on
 * [-R, c1, c2, R] with R the Cauchy bound, each bracket bisected until it is two adjacent doubles, at most 1100 times); each root is a
 * model, denormalised as F = T2' Fn T1 (at most 3 per sample).  Inlier, in pixels and without
 * division: (x2' F x1)^2 <= inl_th^2 ((F x1)_0^2 + (F x1)_1^2 + (F' x2)_0^2 + (F' x2)_1^2) with a positive right-hand side (the Sampson
 * distance; a NaN row is never an inlier).  Best: most inliers, then lowest h, then lowest root.  Samples are evaluated in chunks of
 * 256; after each chunk the search stops once the samples evaluated reach min(N, max_iters), N = ceil(log(1 - confidence) /
 * log(1 - (best/n)^7)), infinite when 1 - (best/n)^7 rounds to 1 (inlier ratios below ~0.5 %).  Then up to 3 rounds of normalised 8-point least squares on the inliers (at least 8): the smallest eigenvector
 * of the 9x9 normal matrix, rank 2 enforced as F (I - v v') with v the smallest eigenvector of F'F, each round kept only if the inlier
 * count does not drop.
 *   d_F [P,3,3]: unit Frobenius norm, its largest-magnitude entry (the lowest index on ties) positive; d_inl [P,tcap] the mask of that
 *   F; d_ninl [P], d_iters [P] (samples evaluated; may be NULL).  n < 7 tentatives, fewer than 7 finite ones, all of them on one point
 *   of an image (iters = 0), or no model with an inlier: ninl = 0, F = 0, mask rows < n = 0.
 *   AG_ERR_INVALID also for inl_th not finite and > 0, confidence outside (0, 1), max_iters < 1.
 * ag_gt_correspondences_pairs: get_GT_correspondence_indexes (ReprojectionStuff.py:126-137) per pair with d_H1to2 [P,3,3]: the image-2
 * centres of all the pair's tentatives are mapped through H^-1 into image 1, and tentative t is true when ANY of them lies within
 * dist_threshold of its image-1 centre, by the fp32 distance sqrt(|(|p|^2 + |a|^2) - 2 a.p + 1e-12|) (nearest: the lowest index among the
 * minima, NaN ignored).  d_min_dist, d_idx2 [P,tcap]; d_true [P,tcap] the true t in ascending order, d_ntrue [P] their number.
 *   AG_ERR_INVALID also for dist_threshold < 0 or NaN. */
int ag_homography_ransac(const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                         const int* d_tent, const int* d_ntent, int tcap, float inl_th, float confidence, int max_iters, unsigned long long seed,
                         float* d_H, unsigned char* d_inl, int* d_ninl, int* d_iters, void* stream);
int ag_fundamental_ransac(const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                          const int* d_tent, const int* d_ntent, int tcap, float inl_th, float confidence, int max_iters, unsigned long long seed,
                          float* d_F, unsigned char* d_inl, int* d_ninl, int* d_iters, void* stream);
int ag_gt_correspondences_pairs(const float* d_lafs1, int S1, int cap1, const float* d_lafs2, int S2, int cap2, const int* d_pairs, int P,
                                const int* d_tent, const int* d_ntent, int tcap, const float* d_H1to2, float dist_threshold,
                                float* d_min_dist, int* d_idx2, int* d_true, int* d_ntrue, void* stream);

/* ------------------------------------------------------------------------------------------
 * Batched end-to-end pipeline (new; the reference processes one image at a time):
 * pyramid -> detect -> select(1.5K) -> sample -> AffNet -> filter(K) -> [sample -> OriNet -> rotate]
 * -> denormalise -> level select -> sample -> HardNet (ag_pipeline_create; ag_pipeline_create_ex selects the other
 * estimators: Baumberg or no shape step, gradient-histogram orientation).    = ScaleSpaceAffinePatchExtractor.forward
 * + extract_patches_from_pyr + HardNet.forward (train_AffNet_test_on_graffity.py:255-260) for B images.
 * ------------------------------------------------------------------------------------------ */
typedef struct ag_pipeline ag_pipeline_t;

typedef struct {
    int B, H, W;
    int num_features;   /* K */
    int nlevels;        /* 3 */
    int border;         /* 5 */
    double init_sigma;  /* 1.6 */
    double mrSize;      /* 5.192 */
    int do_ori;         /* 1: OriNet orientation */
    int cand_cap;       /* candidate capacity per image (0 => H*W/8); on overflow the image's count is reported as -1 */
} ag_pipeline_config_t;

/* Nets are borrowed (must outlive the pipeline).  The pipeline owns no device memory: the caller passes one
 * workspace of ag_pipeline_workspace_bytes() bytes.  = ag_pipeline_create_ex with {AG_SHAPE_AFFNET, 1, -, do_ori ? AG_ORI_ORINET : AG_ORI_NONE, -}. */
int ag_pipeline_create(const ag_pipeline_config_t* cfg, const ag_net_t* affnet, const ag_net_t* orinet,
                       const ag_net_t* hardnet, ag_pipeline_t** out);

/* Estimators of the pipeline (ScaleSpaceAffinePatchExtractor's AffNet / OriNet / num_Baum_iters, SparseImgRepresenter.py:26-49):
 *   shape  AG_SHAPE_NONE      num_Baum_iters = 0: K keypoints straight from the detector, no prefilter and no shape filter;
 *          AG_SHAPE_AFFNET    num_baum_iters AffNet iterations (affnet), then the shape filter;
 *          AG_SHAPE_BAUMBERG  num_baum_iters iterations of AffineShapeEstimator(patch_size = shape_ps) (HandCraftedModules.py:81-132),
 *                             all in one launch that samples the pyramid directly, then the shape filter;
 *   ori    AG_ORI_NONE, AG_ORI_ORINET (orinet), AG_ORI_HISTOGRAM: OrientationDetector(patch_size = ori_ps) (HandCraftedModules.py:133-192)
 *          sampling the pyramid directly.
 * The hand-crafted estimators' patches never reach memory; their Gaussian windows are computed at create time. */
#define AG_SHAPE_NONE 0
#define AG_SHAPE_AFFNET 1
#define AG_SHAPE_BAUMBERG 2
#define AG_ORI_NONE 0
#define AG_ORI_ORINET 1
#define AG_ORI_HISTOGRAM 2
typedef struct {
    int shape;           /* AG_SHAPE_* */
    int num_baum_iters;  /* >= 1 with a shape estimator; ignored with AG_SHAPE_NONE */
    int shape_ps;        /* AG_SHAPE_BAUMBERG patch size, 3..41 (the reference's 19) */
    int ori;             /* AG_ORI_*; must agree with cfg->do_ori */
    int ori_ps;          /* AG_ORI_HISTOGRAM patch size, 3..41 (the reference's 19) */
} ag_pipeline_estimators_t;
/* Nets the mode does not use may be NULL and are ignored.  AG_ERR_INVALID: a missing net for the chosen mode, num_baum_iters < 1 with
 * a shape estimator, a patch size outside 3..41, cfg->do_ori inconsistent with est->ori.  AG_ERR_CAPACITY: a prefilter of
 * int(1.5 K) > 16384 keypoints with a shape estimator (K > 10923), K > 16384 without (ag_pipeline_create_topk has no such limit). */
int ag_pipeline_create_ex(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_net_t* affnet,
                          const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out);

/* Descriptor of the pipeline (get_geometry_and_descriptors(img, det, desc)'s `desc`):
 *   AG_DESC_HARDNET  HardNet (hardnet) on 32 x 32 patches; ps must be 32, clipval is ignored.
 *   AG_DESC_SIFT     SIFTNet(patch_size = ps, clipval) (ag_sift_describe_pyr) in one launch that samples the pyramid directly; hardnet
 *                    may be NULL.  The descriptor's pyramid level is chosen for ps (ag_pyramid_level_for_lafs).  The workspace holds no
 *                    HardNet buffers, and no net buffers at all without AG_SHAPE_AFFNET and AG_ORI_ORINET.
 * ag_pipeline_create_ex is ag_pipeline_create_desc with {AG_DESC_HARDNET, 32, -}.  AG_ERR_INVALID (before any CUDA call) additionally
 * for an unknown kind, HardNet with ps != 32 or without a net, SIFT with an unsupported ps or a clipval that is not finite and positive. */
#define AG_DESC_HARDNET 0
#define AG_DESC_SIFT 1
typedef struct {
    int kind;       /* AG_DESC_* */
    int ps;         /* descriptor patch size: 32 for HardNet; a supported ag_sift_windows size for SIFT (the reference's 65 by default) */
    float clipval;  /* SIFT: the clip between the two L2 normalisations (the reference's 0.2) */
} ag_pipeline_descriptor_t;
int ag_pipeline_create_desc(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_pipeline_descriptor_t* desc,
                            const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out);
/* Threshold mode (ScaleSpaceAffinePatchExtractor(th = th), SparseImgRepresenter.py:33-37; the reference's hesaffnet.py runs th = -1, its
 * HessianAffine default is 28.41): the detector subtracts th from the Hessian response, every candidate of the accepted levels is kept
 * in (octave, level, raster) order (ag_select_all_keypoints), and with a shape step every survivor of the shape filter in that order
 * (ag_affine_shape_filter_all): there is no top-K.  cfg->num_features is the per-image keypoint capacity C (>= 1, no 16384 limit): the
 * prefilter and the outputs hold C rows, and an image with more than C accepted candidates gets count -1, as a candidate-list overflow
 * does.  Estimators and descriptor as ag_pipeline_create_desc.  The workspace is that formula with M = K = C plus the selection's scratch:
 * the net share grows by about 256 KB per HardNet row, so B x C decides the cost (2 x 32768 rows: about 16 GB).
 * AG_ERR_INVALID (before any CUDA call) for th NaN or infinite and for everything ag_pipeline_create_desc refuses except its K limits. */
int ag_pipeline_create_th(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_pipeline_descriptor_t* desc,
                          float th, const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out);
/* ag_pipeline_create_desc without its K limits: the selection and the shape filter run ag_select_topk_keypoints and
 * ag_affine_shape_filter_topk, so any K is accepted.  The kernels are chosen by size: while the prefilter (int(1.5 K) with a shape step, K
 * without) is at most 16384 the pipeline is ag_pipeline_create_desc's - the same workspace bytes, launch count and outputs.  Above, the
 * workspace adds one scratch region shared by the two steps. */
int ag_pipeline_create_topk(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_pipeline_descriptor_t* desc,
                            const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out);
void ag_pipeline_destroy(ag_pipeline_t* p);
size_t ag_pipeline_workspace_bytes(const ag_pipeline_t* p);
const ag_pyramid_plan_t* ag_pipeline_plan(const ag_pipeline_t* p);
/* d_img [B,H,W] -> d_lafs [B,K,2,3] (pixel units), d_resp [B,K], d_desc [B,K,128], d_count [B].
 * Enqueues kernels only (CUDA-graph capturable). */
int ag_pipeline_run(ag_pipeline_t* p, const float* d_img, void* d_ws, size_t ws_bytes, float* d_lafs, float* d_resp,
                    float* d_desc, int* d_count, void* stream);
/* Number of kernel launches the last ag_pipeline_run / ag_pipeline_run_given enqueued (for bench.py's gpu_launches). */
int ag_pipeline_launch_count(const ag_pipeline_t* p);

/* Given keypoints (new; the reference composes these steps by hand, e.g. its SIFT-AffNet-HardNet notebook): describe caller-supplied
 * pixel LAFs with the pipeline's estimators and descriptor, nothing detected and nothing sorted.  cfg->num_features is the per-image
 * capacity C of the input and output rows (1 .. 2^24, no 16384 limit); cfg->cand_cap and cfg->mrSize are ignored; est and desc as
 * ag_pipeline_create_desc, with its refusals (AG_ERR_INVALID before any CUDA call).  Per image b, rows i < d_count_in[b]:
 *   1. the ScalePyramid of image b (the plan of ag_pipeline_create);
 *   2. (oct, lvl) = get_pyramid_and_level_index_for_LAFs(dLAF, PS = 32) (LAF.py:453-472), the level every estimator samples, as
 *      getAffineShape and getOrientation reuse one level (SparseImgRepresenter.py:113-180);
 *   3. normalizeLAFs with the coefficients of ag_pipeline_run;
 *   4. with a shape estimator, num_baum_iters iterations of it, then getAffineShape's keep-all branch (num_features <= 0, :151-156): every
 *      survivor of the eigenvalue-ratio and boundary tests in input order; d_src[b,j] is the input row of output row j.  Without one
 *      every row survives and d_src[b,j] = j;
 *   5. the orientation estimator, if any (getOrientation), at the same (oct, lvl);
 *   6. denormalizeLAFs into d_lafs, then extract_patches_from_pyr(·, desc->ps) and the descriptor into d_desc.  With neither a shape nor
 *      an orientation step the LAFs are not touched: d_lafs[b,j] equals the input row bit for bit (no normalise / denormalise round trip).
 * d_img [B,H,W]; d_lafs_in [B,C,2,3] pixel LAFs; d_count_in [B].  Outputs d_lafs [B,C,2,3], d_src [B,C] int32, d_desc [B,C,128],
 * d_count [B] = the survivors.  A count_in[b] outside 0..C gives d_count[b] = -1 and nothing else of image b is written (the pipeline's
 * overflow count travels through the matcher this way); rows at or beyond d_count[b] of every output are never written.  Launches are
 * fixed on the host and counts read on the device: no host synchronisation, CUDA-graph capturable.  The workspace holds the pyramid, the
 * per-row buffers of C rows and the net scratch, no detector or selection regions.  ag_pipeline_run refuses a given-keypoints pipeline
 * and ag_pipeline_run_given every other kind, with AG_ERR_INVALID before any CUDA call. */
int ag_pipeline_create_given(const ag_pipeline_config_t* cfg, const ag_pipeline_estimators_t* est, const ag_pipeline_descriptor_t* desc,
                             const ag_net_t* affnet, const ag_net_t* orinet, const ag_net_t* hardnet, ag_pipeline_t** out);
int ag_pipeline_run_given(ag_pipeline_t* p, const float* d_img, const float* d_lafs_in, const int* d_count_in, void* d_ws, size_t ws_bytes,
                          float* d_lafs, int* d_src, float* d_desc, int* d_count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AFFNET_B200_H */
