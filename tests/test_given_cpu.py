"""CPU tests (-m "not gpu") of the given-keypoints mode: the ells2LAFsT restatement (tests/given_restated.py, the arithmetic of
ag_ells_to_lafs) and the oracle's composition on caller-supplied keypoints against the unmodified reference (tests/golden/given.npz,
tests/golden/make_golden_given.py), and ag_pipeline_create_given / ag_pipeline_run_given refusals, which come before any CUDA call."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import given_restated as G
from helpers import TOL, gold, gray_from_rgb, load_weights

AG_ERR_INVALID, AG_ERR_CAPACITY = -1, -3


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


def ulps(a, b):
    """|a - b| in units in the last place of float32 (0 where both are NaN)."""
    ia, ib = a.astype(np.float32).view(np.int32).astype(np.int64), b.astype(np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    return np.where(np.isnan(a) & np.isnan(b), 0, d)


def test_ells_to_lafs_restatement_vs_reference_golden():
    """ells2LAFsT's operations one for one in IEEE fp32.  The reference's torch.sqrt on the CPU is MKL's vector square root, which is not
    correctly rounded for about 0.7% of inputs, so the restatement (correctly rounded, as the device's __fsqrt_rn) equals the reference bit
    for bit on the rows where that rounding does not enter and stays within a few ulp elsewhere.  NaN (an ellipse that is not positive
    definite) and the b == 0 branch come out where the reference has them."""
    z = gold("given.npz")
    r, g = G.ells_to_lafs(z["ell_in"]), z["ell_lafs"]
    assert np.array_equal(np.isnan(r), np.isnan(g))
    assert np.isnan(g).any(axis=(1, 2)).sum() >= 3
    u = ulps(r, g)
    exact = (u == 0).all(axis=(1, 2))
    print("\n%d ellipses: %d rows bit-identical, max %d ulp" % (len(r), exact.sum(), u.max()))
    fin = ~np.isnan(g).any(axis=(1, 2))
    sc = np.sqrt(np.abs(g[fin, 0, 0] * g[fin, 1, 1] - g[fin, 0, 1] * g[fin, 1, 0]))
    rel = (np.abs(r[fin] - g[fin]).max(axis=(1, 2)) / sc).max()
    print("largest difference %.2e of the LAF scale" % rel)
    assert exact.mean() >= 0.9 and u.max() <= 32 and rel < 1e-6
    assert np.array_equal(r[:, :, 2], g[:, :, 2]) and (r[:, 0, 1][~np.isnan(r[:, 0, 1])] == 0).all()


def test_ells_to_lafs_inverts_lafs_to_ell():
    """ell.npz holds LAFs2ellT of the graf crop's LAFs: reading them back gives an upright LAF of the same ellipse, A A^T = the inverse of
    [[a, b], [b, c]] to float32 rounding (amplified by the ellipse's elongation)."""
    z = gold("ell.npz")
    ell = z["ell"].astype(np.float64)
    lafs = G.ells_to_lafs(z["ell"]).astype(np.float64)
    A = lafs[:, :, :2]
    M = np.linalg.inv(np.stack([ell[:, 2], ell[:, 3], ell[:, 3], ell[:, 4]], 1).reshape(-1, 2, 2))
    AAt = A @ A.transpose(0, 2, 1)
    ok = ~np.isnan(AAt).any(axis=(1, 2))
    assert ok.mean() > 0.99
    err = np.abs(AAt[ok] - M[ok]).max(axis=(1, 2)) / np.abs(M[ok]).max(axis=(1, 2))
    assert np.quantile(err, 0.95) < 1e-5 and err.max() < 1e-2, (np.quantile(err, 0.95), err.max())   # the worst: strongly elongated ellipses
    assert np.array_equal(lafs[:, :, 2], ell[:, :2])


def test_oracle_given_composition_vs_reference_golden():
    """The reference's notebook chain on the graf crop's upright detections plus hand-placed keypoints near and across the border:
    get_pyramid_and_level_index_for_LAFs(., 32), getAffineShape(num_features = 0) with AffNet x 1, OriNet, HardNet.  The oracle keeps
    the reference's survivors in the reference's order, except rows on the eigenvalue test's knife edge; LAFs and descriptors agree to
    the end-to-end tolerance."""
    W = load_weights()
    z = gold("given.npz")
    torch.set_num_threads(min(16, torch.get_num_threads()))
    img = gray_from_rgb(gold("graf_crop.npz")["rgb"])
    dL = torch.from_numpy(z["in_dLAFs"])
    out, src, desc, st = G.describe_given(img, dL, "affnet", 1, W["affnet"], "orinet", W["orinet"], W["hardnet"])
    gsrc = torch.from_numpy(z["src"])
    edge = G.knife_edge(st["debug"]["aff"]["base_A"])
    diff = set(src.tolist()) ^ set(gsrc.tolist())
    print("\n%d keypoints in, reference %d survivors, oracle %d; disagreements %s, knife-edge rows %d" % (
        dL.size(0), gsrc.numel(), src.numel(), sorted(diff), int(edge.sum())))
    assert all(bool(edge[i]) for i in diff) and len(diff) <= 2
    n_in = dL.size(0)
    hand = set(range(int(z["n_plain"]), n_in))
    assert hand - set(gsrc.tolist()) and hand & set(gsrc.tolist())   # the border keypoints: some dropped, some kept
    common = sorted(set(src.tolist()) & set(gsrc.tolist()))
    io = torch.tensor([src.tolist().index(i) for i in common])
    ig = torch.tensor([gsrc.tolist().index(i) for i in common])
    gL = torch.from_numpy(z["out_dLAFs"])[ig]
    s = (gL[:, 0, 0] * gL[:, 1, 1] - gL[:, 0, 1] * gL[:, 1, 0]).abs().sqrt()
    eL = ((gL - out[io]).abs().amax(dim=(1, 2)) / s).max().item()
    dd = (torch.from_numpy(z["desc"])[ig] - desc[io]).abs().max().item()
    print("LAF error %.2e (relative to the scale), descriptors %.2e" % (eL, dd))
    assert eL < TOL and dd < TOL


def cfg_of(L, C_=300, B=2, H=240, W=320, ori=False):
    return L.PipelineConfig(B, H, W, C_, 3, 5, 1.6, 5.192, 1 if ori else 0, 0)


def create_given(L, cfg, est, desc, nets=(None, None, None)):
    h = C.c_void_p()
    rc = L.lib().ag_pipeline_create_given(C.byref(cfg), C.byref(est), C.byref(desc), nets[0], nets[1], nets[2], C.byref(h))
    if rc == 0:
        return rc, h
    return rc, L.lib().ag_last_error().decode()


def test_pipeline_create_given_refusals(L):
    """AG_ERR_INVALID for NULL arguments, mode / net mismatches, a capacity below 1 or above 2^24, and the descriptor refusals of
    ag_pipeline_create_desc; no 16384 limit.  The modes here need no net, so every call runs on the host only."""
    lib = L.lib()
    est = L.PipelineEstimators(L.SHAPE_BAUMBERG, 16, 19, L.ORI_NONE, 19)
    desc = L.PipelineDescriptor(L.DESC_SIFT, 32, 0.2)
    cfg = cfg_of(L)
    h = C.c_void_p()
    assert lib.ag_pipeline_create_given(None, C.byref(est), C.byref(desc), None, None, None, C.byref(h)) == AG_ERR_INVALID
    assert lib.ag_pipeline_create_given(C.byref(cfg), None, C.byref(desc), None, None, None, C.byref(h)) == AG_ERR_INVALID
    assert lib.ag_pipeline_create_given(C.byref(cfg), C.byref(est), None, None, None, None, C.byref(h)) == AG_ERR_INVALID
    assert lib.ag_pipeline_create_given(C.byref(cfg), C.byref(est), C.byref(desc), None, None, None, None) == AG_ERR_INVALID
    assert b"ag_pipeline_create_given: NULL argument" in lib.ag_last_error()
    for c in (0, -1, (1 << 24) + 1):
        rc, msg = create_given(L, cfg_of(L, C_=c), est, desc)
        assert rc == AG_ERR_INVALID and "num_features" in msg, (c, rc, msg)
    bad = [
        (L.PipelineEstimators(7, 1, 0, L.ORI_NONE, 0), desc, "unknown shape estimator"),
        (L.PipelineEstimators(L.SHAPE_AFFNET, 1, 0, L.ORI_NONE, 0), desc, "AG_SHAPE_AFFNET needs an AffNet"),
        (L.PipelineEstimators(L.SHAPE_BAUMBERG, 0, 19, L.ORI_NONE, 0), desc, "num_baum_iters must be at least 1"),
        (L.PipelineEstimators(L.SHAPE_BAUMBERG, 1, 2, L.ORI_NONE, 0), desc, "shape_ps out of range"),
        (L.PipelineEstimators(L.SHAPE_NONE, 0, 0, L.ORI_HISTOGRAM, 19), desc, "cfg->do_ori disagrees"),
        (est, L.PipelineDescriptor(L.DESC_SIFT, 17, 0.2), "unsupported ps"),
        (est, L.PipelineDescriptor(L.DESC_SIFT, 32, float("nan")), "clipval"),
        (est, L.PipelineDescriptor(L.DESC_HARDNET, 32, 0.2), "needs a HardNet"),
    ]
    for e, d, text in bad:
        rc, msg = create_given(L, cfg, e, d)
        assert rc == AG_ERR_INVALID and text in msg and "ag_pipeline_create_given" in msg, (text, rc, msg)
    rc, msg = create_given(L, cfg_of(L, ori=True), L.PipelineEstimators(L.SHAPE_NONE, 0, 0, L.ORI_ORINET, 0), desc)
    assert rc == AG_ERR_INVALID and "AG_ORI_ORINET needs an OriNet" in msg, msg
    # above the top-K modes' sort limit
    rc, h = create_given(L, cfg_of(L, C_=40000), est, desc)
    assert rc == 0 and lib.ag_pipeline_workspace_bytes(h) > 0
    lib.ag_pipeline_destroy(h)


def test_run_refuses_the_other_kind_before_any_cuda_call(L):
    """ag_pipeline_run on a given-keypoints pipeline and ag_pipeline_run_given on a detecting one return AG_ERR_INVALID without touching
    the (dummy, never dereferenced) device pointers."""
    lib = L.lib()
    est = L.PipelineEstimators(L.SHAPE_BAUMBERG, 1, 19, L.ORI_HISTOGRAM, 19)
    desc = L.PipelineDescriptor(L.DESC_SIFT, 32, 0.2)
    cfg = cfg_of(L, ori=True)
    rc, g = create_given(L, cfg, est, desc)
    assert rc == 0
    d = C.c_void_p(0x1000)
    ws = lib.ag_pipeline_workspace_bytes(g)
    assert lib.ag_pipeline_run(g, d, d, ws, d, d, d, d, None) == AG_ERR_INVALID
    assert b"ag_pipeline_run_given" in lib.ag_last_error()
    h = C.c_void_p()
    assert lib.ag_pipeline_create_desc(C.byref(cfg), C.byref(est), C.byref(desc), None, None, None, C.byref(h)) == 0
    assert lib.ag_pipeline_run_given(h, d, d, d, d, lib.ag_pipeline_workspace_bytes(h), d, d, d, d, None) == AG_ERR_INVALID
    assert b"ag_pipeline_create_given" in lib.ag_last_error()
    assert lib.ag_pipeline_run_given(g, d, None, d, d, ws, d, d, d, d, None) == AG_ERR_INVALID
    assert lib.ag_pipeline_run_given(g, d, d, d, d, ws - 1, d, d, d, d, None) == AG_ERR_CAPACITY
    lib.ag_pipeline_destroy(g)
    lib.ag_pipeline_destroy(h)


def test_given_workspace_has_no_detector_or_selection(L):
    """The given pipeline's workspace holds the pyramid, the per-row buffers and the net share: less than the detecting pipeline's at the
    same K, and it grows linearly with C."""
    lib = L.lib()
    est = L.PipelineEstimators(L.SHAPE_BAUMBERG, 1, 19, L.ORI_HISTOGRAM, 19)
    desc = L.PipelineDescriptor(L.DESC_SIFT, 32, 0.2)
    sizes = []
    for c in (1000, 2000, 4000):
        cfg = cfg_of(L, C_=c, ori=True)
        rc, g = create_given(L, cfg, est, desc)
        assert rc == 0
        sizes.append(lib.ag_pipeline_workspace_bytes(g))
        lib.ag_pipeline_destroy(g)
        h = C.c_void_p()
        assert lib.ag_pipeline_create_desc(C.byref(cfg), C.byref(est), C.byref(desc), None, None, None, C.byref(h)) == 0
        assert sizes[-1] < lib.ag_pipeline_workspace_bytes(h)
        lib.ag_pipeline_destroy(h)
    assert abs((sizes[2] - sizes[1]) - 2 * (sizes[1] - sizes[0])) <= 4096
