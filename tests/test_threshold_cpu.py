"""CPU tests (-m "not gpu") of the threshold mode: the oracle's restatement (tests/oracle_threshold.py) against the unmodified reference's
own threshold-mode output (tests/golden/threshold.npz, tests/golden/make_golden_threshold.py), ag_pipeline_create_th's refusals, which
come before any CUDA call, and the size of ag_select_all_keypoints' scratch."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

import oracle_threshold as OT
from helpers import gold, gray_from_rgb, load_weights, match_keypoints

AG_ERR_INVALID, AG_ERR_CAPACITY = -1, -3


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


@pytest.mark.parametrize("case", ["graf-th28.41", "crop-th-1"])
def test_oracle_threshold_mode_vs_reference_golden(case):
    """hesaffnet.py's configuration (AffNet x 1, border 5, mrSize 5.192, no orientation) with th set: the reference keeps every
    keypoint above th and every survivor of the shape filter.  The restatement finds the same keypoints; its responses are the
    reference's bit for bit (same detector ops), and its LAFs agree to the oracle's AffNet tolerance."""
    W = load_weights()
    z = gold("threshold.npz")
    if case == "graf-th28.41":
        img, th, key = gray_from_rgb(gold("graf_full.npz")["rgb"]), 28.41, "th28"
    else:
        img, th, key = gray_from_rgb(gold("graf_crop.npz")["rgb"]), -1.0, "thm1"
    torch.set_num_threads(min(16, torch.get_num_threads()))
    dL, resp, _ = OT.detect(img, th, "affnet", 1, W["affnet"])
    gL, gr = torch.from_numpy(z[key + "_dLAFs"]), torch.from_numpy(z[key + "_resp"])
    ia, ib = match_keypoints(gL, dL)
    print("\n%s: reference %d keypoints, restatement %d, matched %d" % (case, gL.shape[0], dL.shape[0], len(ia)))
    assert abs(dL.shape[0] - gL.shape[0]) <= max(2, 0.002 * gL.shape[0])
    assert len(ia) >= 0.995 * gL.shape[0]
    assert torch.equal(resp[ib], gr[ia])
    s = (gL[ia][:, 0, 0] * gL[ia][:, 1, 1] - gL[ia][:, 0, 1] * gL[ia][:, 1, 0]).abs().sqrt()
    err = (gL[ia] - dL[ib]).abs().amax(dim=(1, 2)) / s
    assert float((err < 1e-3).float().mean()) >= 0.995, err.max()
    if dL.shape[0] == gL.shape[0] and len(ia) == gL.shape[0]:
        assert torch.equal(resp, gr)                              # same order: (octave, level, raster), survivors in index order


def configs(L, C_=300, B=2, H=240, W=320, shape=None, ori=None, desc=None):
    cfg = L.PipelineConfig(B, H, W, C_, 3, 5, 1.6, 5.192, 0 if ori is None else 1, 0)
    est = shape or L.PipelineEstimators(L.SHAPE_BAUMBERG, 16, 19, L.ORI_NONE if ori is None else ori, 19)
    return cfg, est, desc or L.PipelineDescriptor(L.DESC_SIFT, 32, 0.2)


def create_th(L, cfg, est, desc, th, nets=(None, None, None)):
    h = C.c_void_p()
    rc = L.lib().ag_pipeline_create_th(C.byref(cfg), C.byref(est), C.byref(desc), th, nets[0], nets[1], nets[2], C.byref(h))
    if rc == 0:
        ws = L.lib().ag_pipeline_workspace_bytes(h)
        L.lib().ag_pipeline_destroy(h)
        return rc, ws
    return rc, L.lib().ag_last_error().decode()


def test_pipeline_create_th_refusals(L):
    """AG_ERR_INVALID for NaN or infinite th, a capacity below 1 and the existing mode refusals; no 16384 / 10923 limit on C.  The modes
    used here need no net, so every call runs on the host only (the library has no device to touch)."""
    cfg, est, desc = configs(L)
    for th in (float("nan"), float("inf"), -float("inf")):
        rc, msg = create_th(L, cfg, est, desc, th)
        assert rc == AG_ERR_INVALID and "ag_pipeline_create_th: th must be finite" in msg, (th, rc, msg)
    for c in (0, -5):
        rc, msg = create_th(L, configs(L, C_=c)[0], est, desc, 28.41)
        assert rc == AG_ERR_INVALID and "num_features must be positive" in msg, (c, rc, msg)
    bad = [
        (L.PipelineEstimators(7, 1, 0, L.ORI_NONE, 0), desc, "unknown shape estimator"),
        (L.PipelineEstimators(L.SHAPE_AFFNET, 1, 0, L.ORI_NONE, 0), desc, "AG_SHAPE_AFFNET needs an AffNet"),
        (L.PipelineEstimators(L.SHAPE_BAUMBERG, 0, 19, L.ORI_NONE, 0), desc, "num_baum_iters must be at least 1"),
        (L.PipelineEstimators(L.SHAPE_BAUMBERG, 1, 2, L.ORI_NONE, 0), desc, "shape_ps out of range"),
        (est, L.PipelineDescriptor(L.DESC_SIFT, 17, 0.2), "unsupported ps"),
        (est, L.PipelineDescriptor(L.DESC_SIFT, 32, float("nan")), "clipval"),
        (est, L.PipelineDescriptor(L.DESC_HARDNET, 32, 0.2), "needs a HardNet"),
    ]
    for e, d, text in bad:
        rc, msg = create_th(L, cfg, e, d, -1.0)
        assert rc == AG_ERR_INVALID and text in msg, (text, rc, msg)
    rc, msg = create_th(L, cfg, L.PipelineEstimators(L.SHAPE_NONE, 0, 0, L.ORI_HISTOGRAM, 19), desc, -1.0)
    assert rc == AG_ERR_INVALID and "cfg->do_ori disagrees" in msg, msg
    # capacities the top-K modes refuse
    for shape in (L.PipelineEstimators(L.SHAPE_BAUMBERG, 16, 19, L.ORI_NONE, 0), L.PipelineEstimators(L.SHAPE_NONE, 0, 0, L.ORI_NONE, 0)):
        big = configs(L, C_=40000, shape=shape)
        rc, ws = create_th(L, *big, 28.41)
        assert rc == 0 and ws > 0, (rc, ws)
        h = C.c_void_p()
        assert L.lib().ag_pipeline_create_desc(C.byref(big[0]), C.byref(big[1]), C.byref(big[2]), None, None, None, C.byref(h)) == AG_ERR_CAPACITY


def test_pipeline_th_workspace_is_the_top_k_formula_with_m_equal_k(L):
    """Threshold mode's workspace is the existing layout with M = K = C plus the selection's scratch: without a shape step (M = K in both
    modes) exactly that scratch more than ag_pipeline_create_desc at the same K."""
    cfg, _, desc = configs(L, C_=1000)
    est = L.PipelineEstimators(L.SHAPE_NONE, 0, 0, L.ORI_HISTOGRAM, 19)
    cfg.do_ori = 1
    rc, ws_th = create_th(L, cfg, est, desc, 28.41)
    assert rc == 0
    h = C.c_void_p()
    assert L.lib().ag_pipeline_create_desc(C.byref(cfg), C.byref(est), C.byref(desc), None, None, None, C.byref(h)) == 0
    ws_top = L.lib().ag_pipeline_workspace_bytes(h)
    L.lib().ag_pipeline_destroy(h)
    plan = L.make_plan(cfg.B, cfg.H, cfg.W)
    sel = L.lib().ag_select_all_workspace_bytes(C.byref(plan), cfg.H * cfg.W // 8)
    assert ws_th == ws_top + sel, (ws_th, ws_top, sel)


def test_select_all_workspace_bytes(L):
    """The scratch holds a bitmap and a prefix word per 32 pixels of every detection level, for every image: it grows with B and the image
    size, is independent of cand_cap, and a non-positive cand_cap gives 0."""
    lib = L.lib()
    sizes = {}
    for B in (1, 2, 4):
        for (H, W) in ((240, 320), (768, 1024), (1080, 1920)):
            plan = L.make_plan(B, H, W)
            n = lib.ag_select_all_workspace_bytes(C.byref(plan), 4096)
            px = sum(plan.h[o] * plan.w[o] for o in range(plan.n_octaves)) * (plan.n_levels - 2)
            assert n >= B * 8 * math.ceil(px / 32), (B, H, W, n)
            assert n == lib.ag_select_all_workspace_bytes(C.byref(plan), 10 ** 6)
            assert lib.ag_select_all_workspace_bytes(C.byref(plan), 0) == 0
            sizes[(B, H, W)] = n
    for (B, H, W), n in sizes.items():
        if B < 4:
            assert sizes[(2 * B, H, W)] > n
    assert sizes[(1, 240, 320)] < sizes[(1, 768, 1024)] < sizes[(1, 1080, 1920)]
    assert lib.ag_select_all_workspace_bytes(None, 4096) == 0
