"""CPU tests of the pipeline's estimator modes: the oracle's restated getAffineShape loop (tests/oracle_estimators.py) against the
pinned AffNet x 1 stage and the reference default detector's golden output, ag_pipeline_create_ex's refusals and error texts, and
DetectDescribePipeline's mapping of the mirror's constructor arguments onto the modes.  No device code runs: create_ex does host
work only (pyramid plan, Gaussian windows, workspace layout)."""
import ctypes as C
import os

import pytest
import torch

import affnet_oracle as O
import oracle_estimators as OE
from helpers import gold, gray_from_rgb, load_weights, match_keypoints

W = load_weights()


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


def crop_img():
    return gray_from_rgb(gold("graf_crop.npz")["rgb"])


def test_restated_loop_at_affnet_x1_is_get_affine_shape():
    """num_iters = 1 with AffNet: the same stage as affnet_oracle.get_affine_shape, tensor for tensor."""
    x = crop_img()
    K, mr = 300, 5.192
    pyr, sigmas, _ = O.scale_pyramid(x, 3, 1.6, 5)
    resp, LAFs, pidx, lidx = O.multi_scale_detector(pyr, sigmas, int(1.5 * K), mr)
    LAFs = LAFs.clone()
    LAFs[:, 0:2, 0:2] = mr * LAFs[:, :, 0:2]
    a = O.get_affine_shape(pyr, resp, LAFs, pidx, lidx, K, W["affnet"])
    b = OE.get_affine_shape_iter(pyr, resp, LAFs, pidx, lidx, K, lambda P: O.affnet_forward(P, W["affnet"]), 1, 32)
    for u, v in zip(a[:4], b[:4]):
        assert torch.equal(u, v)
    assert a[0].numel() == K
    # and end to end: detect with the default arguments is affnet_oracle.detect
    dA, rA, _ = O.detect(x, W["affnet"], W["orinet"], K, do_ori=True)
    dB, rB, _ = OE.detect(x, "affnet", 1, W["affnet"], "orinet", W["orinet"], K)
    assert torch.equal(dA, dB) and torch.equal(rA, rB)


def test_no_shape_step_with_histogram_reproduces_the_reference_default_detector():
    """num_Baum_iters = 0 + OrientationDetector(19): the reference's default ScaleSpaceAffinePatchExtractor on the graf crop, K = 300
    (golden default_dLAFs), with the matching rule of the GPU test of the single-image API (test_gpu_parity.py::test_handcrafted_estimators_8f)."""
    z = gold("handcrafted.npz")
    dL, r, _ = OE.detect(crop_img(), None, 0, None, "histogram", None, 300)
    gL = torch.from_numpy(z["default_dLAFs"])
    assert dL.shape[0] == gL.shape[0] == 300
    assert torch.equal(r, torch.from_numpy(z["default_resp"]))
    ia, ib = match_keypoints(gL, dL, tol_px=0.05)
    same = ((gL[ia] - dL[ib]).abs().amax(dim=(1, 2)) < 1e-2).float().mean().item()
    print("\noracle, no shape step + histogram orientation: matched %d/%d, identical LAF %.3f" % (len(ia), gL.shape[0], same))
    assert len(ia) >= gL.shape[0] - 3 and same >= 0.97


def test_restated_loop_iterates_baumberg():
    """Baumberg iterations: iteration i samples at [base_A LAF_A | t] of the previous ones; with one iteration base_A is the module's A."""
    x = crop_img()
    pyr, sigmas, _ = O.scale_pyramid(x, 3, 1.6, 5)
    resp, LAFs, pidx, lidx = O.multi_scale_detector(pyr, sigmas, 150, 5.192)
    LAFs = LAFs.clone()
    LAFs[:, 0:2, 0:2] = 5.192 * LAFs[:, :, 0:2]
    one = OE.get_affine_shape_iter(pyr, resp, LAFs, pidx, lidx, 100, O.baumberg_shape, 1, 19)[4]
    assert torch.equal(one["base_A"], O.baumberg_shape(O.extract_patches_from_pyramid(pyr, pidx, lidx, LAFs, 19)))
    two = OE.get_affine_shape_iter(pyr, resp, LAFs, pidx, lidx, 100, O.baumberg_shape, 2, 19)[4]
    cur = torch.cat([torch.bmm(one["base_A"], LAFs[:, :, :2]), LAFs[:, :, 2:]], dim=2)
    A2 = O.baumberg_shape(O.extract_patches_from_pyramid(pyr, pidx, lidx, cur, 19))
    assert torch.equal(two["base_A"], torch.bmm(A2, one["base_A"]))


def test_baumberg_x16_conditioning_is_selective():
    """oracle_estimators.shape_spread, the conditioning criterion the GPU comparison of Baumberg x16 accounts keypoints with: on graf img1
    at 1024x768, K = 2000, the oracle's own loop keeps base_A within 1e-4 under every fp32-level perturbation at 1 and 2 iterations, and at
    16 iterations moves a few percent of the keypoints by 1e-4 or more (up to more than 1) while the median moves by less than 1e-5."""
    import cv2
    torch.set_num_threads(min(16, torch.get_num_threads()))
    img = gray_from_rgb(cv2.resize(gold("graf_full.npz")["rgb"], (1024, 768), interpolation=cv2.INTER_LINEAR))
    pyr, _, _ = O.scale_pyramid(img, 3, 1.6, 5)
    g = torch.Generator().manual_seed(3)
    L = torch.rand(256, 2, 3, generator=g) * 0.02
    L[:, 0, 2] = torch.rand(256, generator=g); L[:, 1, 2] = torch.rand(256, generator=g)
    d = (OE.extract_patches_fp32(pyr[0][1], L, 19) - O.extract_patches(pyr[0][1], L, 19)).abs().max().item()
    assert 0 < d < 0.05, d                            # the fp32 sampler is a perturbation at the fp32 level of 0..255 coordinates
    for it in (1, 2, 16):
        _, _, st = OE.detect(img, "baumberg", it, None, "histogram", None, 2000)
        sp = OE.shape_spread(st, 2000, it)[st["debug"]["aff"]["idxs"]]
        ill = int((sp >= 1e-4).sum())
        print("\nBaumberg x%d: %d of %d keypoints move by 1e-4 or more (median %.1e, max %.1e)" % (it, ill, sp.numel(), sp.median(), sp.max()))
        assert sp.median() < 1e-5
        if it < 16:
            assert ill == 0
        else:
            assert 0.01 * sp.numel() <= ill <= 0.1 * sp.numel() and sp.max() > 1e-2


# ---- ag_pipeline_create_ex -------------------------------------------------------------------------------------------------------------
class FakeNets:
    """Non-NULL net handles: create_ex stores the borrowed pointers and never dereferences them at create time."""

    def __init__(self):
        self._buf = (C.c_char * 64)()
        self.h = C.c_void_p(C.addressof(self._buf))


def cfg_of(L, K=300, do_ori=1, B=2, H=240, Wd=320):
    return L.PipelineConfig(B, H, Wd, K, 3, 5, 1.6, 5.192, do_ori, 0)


def create_ex(L, cfg, est, aff, ori, hard):
    h = C.c_void_p()
    rc = L.lib().ag_pipeline_create_ex(C.byref(cfg), C.byref(est), aff, ori, hard, C.byref(h))
    nbytes = L.lib().ag_pipeline_workspace_bytes(h) if rc == 0 else 0
    if rc == 0:
        L.lib().ag_pipeline_destroy(h)
    return rc, L.lib().ag_last_error().decode() if rc else "", nbytes


def test_create_ex_refusals_and_error_texts(L):
    f = FakeNets().h
    E = L.PipelineEstimators
    cases = [
        (cfg_of(L), E(L.SHAPE_AFFNET, 1, 0, L.ORI_ORINET, 0), None, f, f, -1, "AG_SHAPE_AFFNET needs an AffNet"),
        (cfg_of(L), E(L.SHAPE_AFFNET, 1, 0, L.ORI_ORINET, 0), f, None, f, -1, "AG_ORI_ORINET needs an OriNet"),
        (cfg_of(L, do_ori=1), E(L.SHAPE_NONE, 0, 0, L.ORI_ORINET, 0), f, None, f, -1, "AG_ORI_ORINET needs an OriNet"),
        (cfg_of(L), E(L.SHAPE_AFFNET, 1, 0, L.ORI_ORINET, 0), f, f, None, -1, "NULL argument"),
        (cfg_of(L), E(L.SHAPE_AFFNET, 0, 0, L.ORI_ORINET, 0), f, f, f, -1, "num_baum_iters must be at least 1"),
        (cfg_of(L), E(L.SHAPE_BAUMBERG, -2, 19, L.ORI_ORINET, 0), f, f, f, -1, "num_baum_iters must be at least 1"),
        (cfg_of(L), E(L.SHAPE_BAUMBERG, 1, 2, L.ORI_ORINET, 0), f, f, f, -1, "shape_ps out of range (3..41)"),
        (cfg_of(L), E(L.SHAPE_BAUMBERG, 1, 42, L.ORI_ORINET, 0), f, f, f, -1, "shape_ps out of range (3..41)"),
        (cfg_of(L), E(L.SHAPE_AFFNET, 1, 0, L.ORI_HISTOGRAM, 2), f, f, f, -1, "ori_ps out of range (3..41)"),
        (cfg_of(L), E(L.SHAPE_AFFNET, 1, 0, L.ORI_HISTOGRAM, 42), f, f, f, -1, "ori_ps out of range (3..41)"),
        (cfg_of(L, do_ori=0), E(L.SHAPE_AFFNET, 1, 0, L.ORI_HISTOGRAM, 19), f, f, f, -1, "cfg->do_ori disagrees with est->ori"),
        (cfg_of(L, do_ori=1), E(L.SHAPE_AFFNET, 1, 0, L.ORI_NONE, 0), f, f, f, -1, "cfg->do_ori disagrees with est->ori"),
        (cfg_of(L), E(3, 1, 0, L.ORI_ORINET, 0), f, f, f, -1, "unknown shape estimator"),
        (cfg_of(L), E(L.SHAPE_AFFNET, 1, 0, 3, 0), f, f, f, -1, "unknown orientation estimator"),
        (cfg_of(L, K=10924), E(L.SHAPE_BAUMBERG, 1, 19, L.ORI_ORINET, 0), f, f, f, -3, "int(1.5 K) = 16386"),
        (cfg_of(L, K=10924), E(L.SHAPE_AFFNET, 2, 0, L.ORI_ORINET, 0), f, f, f, -3, "int(1.5 K) = 16386"),
        (cfg_of(L, K=16385), E(L.SHAPE_NONE, 0, 0, L.ORI_ORINET, 0), f, f, f, -3, "K <= 16384"),
        (cfg_of(L, K=0), E(L.SHAPE_NONE, 0, 0, L.ORI_ORINET, 0), f, f, f, -1, "num_features must be positive"),
    ]
    for cfg, est, a, o, h, rc_want, text in cases:
        rc, msg, _ = create_ex(L, cfg, est, a, o, h)
        assert rc == rc_want and text in msg and msg.startswith("ag_pipeline_create_ex: "), (rc, msg, text)
    # the limits themselves are accepted (int(1.5 * 10923) = 16384)
    for cfg, est in ((cfg_of(L, K=10923), E(L.SHAPE_BAUMBERG, 16, 19, L.ORI_HISTOGRAM, 19)),
                     (cfg_of(L, K=16384), E(L.SHAPE_NONE, 0, 0, L.ORI_HISTOGRAM, 41)),
                     (cfg_of(L, K=300), E(L.SHAPE_BAUMBERG, 1, 3, L.ORI_HISTOGRAM, 3))):
        assert create_ex(L, cfg, est, f, f, f)[0] == 0, L.lib().ag_last_error()
    # nets the mode does not use may be NULL
    assert create_ex(L, cfg_of(L, do_ori=0), E(L.SHAPE_NONE, 0, 0, L.ORI_NONE, 0), None, None, f)[0] == 0
    assert create_ex(L, cfg_of(L), E(L.SHAPE_BAUMBERG, 4, 19, L.ORI_HISTOGRAM, 19), None, None, f)[0] == 0
    # ag_pipeline_create keeps its own checks and texts
    h = C.c_void_p()
    assert L.lib().ag_pipeline_create(C.byref(cfg_of(L)), f, None, f, C.byref(h)) == -1
    assert L.lib().ag_last_error() == b"ag_pipeline_create: do_ori needs an OriNet"
    assert L.lib().ag_pipeline_create(C.byref(cfg_of(L, K=10924)), f, f, f, C.byref(h)) == -3
    assert L.lib().ag_last_error().decode().startswith("ag_pipeline_create: num_features 10924") and b"(K <= 10923)" in L.lib().ag_last_error()
    assert L.lib().ag_pipeline_create(C.byref(cfg_of(L, K=0)), f, f, f, C.byref(h)) == -1
    assert L.lib().ag_last_error() == b"ag_pipeline_create: num_features must be positive"


def test_workspace_covers_only_the_nets_the_mode_uses(L):
    f = FakeNets().h
    E = L.PipelineEstimators
    lib = L.lib()
    B, K = 2, 300
    cfg = cfg_of(L, K=K, B=B)
    h = C.c_void_p()
    assert lib.ag_pipeline_create(C.byref(cfg), f, f, f, C.byref(h)) == 0
    legacy = lib.ag_pipeline_workspace_bytes(h)
    lib.ag_pipeline_destroy(h)
    _, _, default = create_ex(L, cfg, E(L.SHAPE_AFFNET, 1, 0, L.ORI_ORINET, 0), f, f, f)
    assert default == legacy                     # ag_pipeline_create is create_ex with these estimators: same layout
    _, _, hist = create_ex(L, cfg, E(L.SHAPE_AFFNET, 1, 0, L.ORI_HISTOGRAM, 19), f, None, f)
    assert hist == legacy                        # AffNet's workspace (1.5 K rows) already covers OriNet's (K rows)
    _, _, chain = create_ex(L, cfg, E(L.SHAPE_AFFNET, 3, 0, L.ORI_HISTOGRAM, 19), f, None, f)
    M = int(1.5 * K)
    al = lambda n: (n + 255) // 256 * 256  # noqa: E731
    assert chain == legacy + 2 * al(B * M * 16) + al(B * M * 24)     # net output, second base_A buffer, working LAFs
    _, _, baum = create_ex(L, cfg, E(L.SHAPE_BAUMBERG, 16, 19, L.ORI_HISTOGRAM, 19), None, None, f)
    _, _, none = create_ex(L, cfg_of(L, K=K, B=B, do_ori=0), E(L.SHAPE_NONE, 0, 0, L.ORI_NONE, 0), None, None, f)
    hb = lib.ag_net_workspace_bytes(L.NET_HARDNET, B * K)
    ab = lib.ag_net_workspace_bytes(L.NET_AFFNET, B * M)
    ob = lib.ag_net_workspace_bytes(L.NET_ORINET, B * K)
    assert none < baum <= legacy
    assert baum == legacy - al(max(ab, ob, hb)) + al(hb)      # the nets share one region, sized for the largest net the mode runs


def test_pipeline_arguments_select_the_mirrors_estimators(L):
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HandCraftedModules import AffineShapeEstimator, OrientationDetector
    from affnet_b200.pipeline import estimators
    a, o = AffNetFast(PS=32), OriNetFast(PS=32)
    ae, od = AffineShapeEstimator(patch_size=15), OrientationDetector(patch_size=41)

    def m(*args):
        e, aff, ori = estimators(*args)
        return (e.shape, e.num_baum_iters, e.shape_ps, e.ori, e.ori_ps), aff, ori

    assert m(a, o, True, 1) == ((L.SHAPE_AFFNET, 1, 0, L.ORI_ORINET, 0), a, o)          # today's default
    assert m(a, o, False, 1) == ((L.SHAPE_AFFNET, 1, 0, L.ORI_NONE, 0), a, None)        # unused OriNet is ignored
    assert m(a, None, True, 1) == ((L.SHAPE_AFFNET, 1, 0, L.ORI_HISTOGRAM, 19), a, None)
    assert m(a, od, True, 3) == ((L.SHAPE_AFFNET, 3, 0, L.ORI_HISTOGRAM, 41), a, None)
    assert m(None, None, True, 16) == ((L.SHAPE_BAUMBERG, 16, 19, L.ORI_HISTOGRAM, 19), None, None)
    assert m(ae, o, True, 2) == ((L.SHAPE_BAUMBERG, 2, 15, L.ORI_ORINET, 0), None, o)
    assert m(a, o, True, 0) == ((L.SHAPE_NONE, 0, 0, L.ORI_ORINET, 0), None, o)          # num_Baum_iters = 0: AffNet unused
    assert m(None, None, False, 0) == ((L.SHAPE_NONE, 0, 0, L.ORI_NONE, 0), None, None)
    with pytest.raises(L.AffnetB200Error):
        estimators(o, None, True, 1)
    with pytest.raises(L.AffnetB200Error):
        estimators(a, a, True, 1)
