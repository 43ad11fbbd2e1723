"""GPU tests (-m gpu) of the batched pipeline's estimator modes (ag_pipeline_create_ex): AffNet or Baumberg iterations or no shape
step, OriNet, gradient-histogram or no orientation.  (i) Bit for bit against the single-image API (ScaleSpaceAffinePatchExtractor, which
materialises the patches and runs the stand-alone estimator kernels) and under CUDA-graph replay; (ii) the reference's application check
(graf 1<->6, AffNet + histogram) through one B = 2 batch; (iii) against the CPU oracle (tests/oracle_estimators.py) at 1024x768, K = 2000."""
import ctypes as C

import pytest
import torch

import affnet_oracle as O
import oracle_estimators as OE
from helpers import SENTINEL, TOL, gold, gray_from_rgb, load_weights, match_keypoints, orientation_boundary_shares

pytestmark = pytest.mark.gpu

DEV = "cuda"
W = load_weights()


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


@pytest.fixture(scope="module")
def nets():
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    return a.eval().to(DEV), o.eval().to(DEV), h.eval().to(DEV)


def crop_img():
    return gray_from_rgb(gold("graf_crop.npz")["rgb"])


def _graf_1024():
    import cv2
    return gray_from_rgb(cv2.resize(gold("graf_full.npz")["rgb"], (1024, 768), interpolation=cv2.INTER_LINEAR))


def mode_args(mode, nets):
    """mode -> (AffNet, num_Baum_iters, OriNet, do_ori): the constructor arguments of ScaleSpaceAffinePatchExtractor / DetectDescribePipeline."""
    from affnet_b200.HandCraftedModules import AffineShapeEstimator, OrientationDetector
    aff, ori, _ = nets
    return {
        "affnet1-histogram": (aff, 1, None, True),
        "affnet2-orinet": (aff, 2, ori, True),
        "baumberg16-histogram": (None, 16, None, True),
        "baumberg1-none": (None, 1, None, False),
        "none-histogram": (None, 0, None, True),
        "none-orinet": (None, 0, ori, True),
        "none-none": (None, 0, None, False),
        "baumberg2ps15-histogram15": (AffineShapeEstimator(patch_size=15), 2, OrientationDetector(patch_size=15), True),
        "baumberg2ps41-histogram41": (AffineShapeEstimator(patch_size=41), 2, OrientationDetector(patch_size=41), True),
    }[mode]


def differing_rows(a, b):
    return (a != b).flatten(1).any(dim=1).nonzero().view(-1).tolist()


@pytest.mark.parametrize("mode", ["affnet1-histogram", "affnet2-orinet", "baumberg16-histogram", "baumberg1-none", "none-histogram",
                                  "none-orinet", "none-none", "baumberg2ps15-histogram15", "baumberg2ps41-histogram41"])
def test_pipeline_modes_equal_single_image_api(L, nets, mode):
    """Every mode over a workspace of 0xFF bytes, with the four images of test_pipeline_batched_equals_single_image_api (graf crop, a
    constant image with no keypoints, the flipped crop, a synthetic image) at K = 300 and 301: counts, responses, LAFs and descriptors
    equal to the single-image API's bit for bit, CUDA-graph replay equal to the run, and response / descriptor rows beyond the counts
    untouched.  A LAF row that differs is named with its angle (the histogram's cosf / sinf against torch's cos / sin)."""
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    hn = nets[2]
    AffNet, iters, OriNet, do_ori = mode_args(mode, nets)
    img = crop_img()
    imgs = torch.cat([img, torch.full_like(img, 77.0), img.flip(3), O.synthetic_image(img.size(2), img.size(3), 5)]).to(DEV)
    B, H, Wd = imgs.size(0), img.size(2), img.size(3)
    for K in (300, 301):
        out = (torch.full((B, K, 2, 3), SENTINEL, device=DEV), torch.full((B, K, 128), SENTINEL, device=DEV),
               torch.full((B,), -7, dtype=torch.int32, device=DEV))
        pipe = DetectDescribePipeline(B, H, Wd, AffNet, hn, OriNet, num_features=K, do_ori=do_ori, outputs=[out], num_Baum_iters=iters)
        pipe.ws.fill_(0xFF)
        pipe.resp.fill_(SENTINEL)
        lafs, resp, desc, cnt = pipe.run(imgs)
        torch.cuda.synchronize()
        lafs, resp, desc, cnt = lafs.clone(), resp.clone(), desc.clone(), cnt.clone()
        assert int(cnt[1]) == 0 and bool((cnt >= 0).all()) and bool((cnt <= K).all()), cnt
        det = ScaleSpaceAffinePatchExtractor(mrSize=5.192, num_features=K, border=5, num_Baum_iters=iters, AffNet=AffNet, OriNet=OriNet)
        for b in range(B):
            n = int(cnt[b])
            assert bool((resp[b, n:] == SENTINEL).all()) and bool((desc[b, n:] == SENTINEL).all()), (mode, K, b, "rows beyond the count written")
            dL, r = det(imgs[b:b + 1], do_ori=do_ori)
            assert n == dL.size(0), (mode, K, b, n, dL.size(0))
            if n == 0:
                continue
            assert bool(torch.isfinite(lafs[b, :n]).all()) and bool(torch.isfinite(desc[b, :n]).all()), (mode, K, b)
            d = hn(det.extract_patches_from_pyr(dL, PS=32))
            assert torch.equal(resp[b, :n], r), (mode, K, b, differing_rows(resp[b, :n], r))
            rows = differing_rows(lafs[b, :n], dL)
            assert not rows, (mode, K, b, "LAF rows differ from the single-image API", [(i, lafs[b, i].tolist(), dL[i].tolist()) for i in rows[:8]])
            assert torch.equal(desc[b, :n], d), (mode, K, b, differing_rows(desc[b, :n], d))
        launches = pipe.launches
        assert launches > 20
        pipe.capture()
        l2, r2, d2, c2 = pipe.replay(imgs)
        torch.cuda.synchronize()
        assert torch.equal(c2, cnt) and pipe.launches == launches
        for b in range(B):
            n = int(cnt[b])
            assert torch.equal(l2[b, :n], lafs[b, :n]) and torch.equal(r2[b, :n], resp[b, :n]) and torch.equal(d2[b, :n], desc[b, :n]), (mode, K, b)


def test_default_mode_keeps_its_launch_sequence(L, nets):
    """ag_pipeline_create is create_ex with {AFFNET, 1, -, ORINET, -}: the same launches, the same bits; the hand-crafted modes add
    exactly their own launches (one fused kernel for all Baumberg iterations, one for the histogram)."""
    import affnet_b200._lib as lib
    from affnet_b200.pipeline import DetectDescribePipeline
    aff, ori, hn = nets
    img = _graf_1024()
    H, Wd = img.shape[2:]
    imgs = torch.cat([img, img.flip(3)]).to(DEV)
    base = DetectDescribePipeline(2, H, Wd, aff, hn, ori, num_features=2000)
    cfg = lib.PipelineConfig(2, H, Wd, 2000, 3, 5, 1.6, 5.192, 1, 0)
    h = C.c_void_p()
    L.check(L.lib().ag_pipeline_create(C.byref(cfg), aff.handle(), ori.handle(), hn.handle(), C.byref(h)))
    try:
        assert L.lib().ag_pipeline_workspace_bytes(h) == base.ws_bytes
        lafs, resp, desc, cnt = [t.clone() for t in base.run(imgs)]
        o = (torch.empty_like(lafs), torch.empty_like(resp), torch.empty_like(desc), torch.empty_like(cnt))
        L.check(L.lib().ag_pipeline_run(h, L.ptr(imgs), L.ptr(base.ws), base.ws_bytes, L.ptr(o[0]), L.ptr(o[1]), L.ptr(o[2]), L.ptr(o[3]),
                                        L.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(o[3], cnt)
        for b in range(2):
            n = int(cnt[b])
            assert torch.equal(o[0][b, :n], lafs[b, :n]) and torch.equal(o[1][b, :n], resp[b, :n]) and torch.equal(o[2][b, :n], desc[b, :n])
        assert L.lib().ag_pipeline_launch_count(h) == base.launches
    finally:
        L.lib().ag_pipeline_destroy(h)
    names = lambda p: [n for n, _ in lib.profile(lambda: p.run(imgs))]  # noqa: E731
    ref = names(base)
    hist = names(DetectDescribePipeline(2, H, Wd, aff, hn, None, num_features=2000))
    baum = names(DetectDescribePipeline(2, H, Wd, None, hn, None, num_features=2000, num_Baum_iters=16))
    print("\nlaunches: default %d, AffNet + histogram %d, Baumberg x16 + histogram %d" % (len(ref), len(hist), len(baum)))
    assert hist.count("orientation_hist_pyr_kernel") == 1 and baum.count("baumberg_pyr_kernel") == 1
    assert "orientation_hist_pyr_kernel" not in ref and "baumberg_pyr_kernel" not in ref


def test_refusals(L, nets):
    """OriNet mode without a net, and K above the selection's limits, are refused at construction."""
    import affnet_b200._lib as lib
    from affnet_b200.pipeline import DetectDescribePipeline
    aff, ori, hn = nets
    cfg = lib.PipelineConfig(1, 240, 320, 300, 3, 5, 1.6, 5.192, 1, 0)
    h = C.c_void_p()
    est = lib.PipelineEstimators(lib.SHAPE_AFFNET, 1, 0, lib.ORI_ORINET, 0)
    assert L.lib().ag_pipeline_create_ex(C.byref(cfg), C.byref(est), aff.handle(), None, hn.handle(), C.byref(h)) == -1
    assert b"AG_ORI_ORINET needs an OriNet" in L.lib().ag_last_error()
    with pytest.raises(lib.AffnetB200Error, match="K <= 10923"):
        DetectDescribePipeline(1, 240, 320, None, hn, None, num_features=10924, num_Baum_iters=16)
    with pytest.raises(lib.AffnetB200Error, match="K <= 16384"):
        DetectDescribePipeline(1, 240, 320, None, hn, None, num_features=16385, num_Baum_iters=0)
    p = DetectDescribePipeline(1, 240, 320, None, hn, None, num_features=16384, num_Baum_iters=0)
    assert p.ws_bytes > 0


def test_graf_1_to_6_application_counts_batched(L, nets):
    """The reference's own end-to-end check (train_AffNet_test_on_graffity.py:262-300, AffNet + gradient-histogram orientation, K = 3000)
    with graf img1 and img6 as ONE B = 2 batch of the pipeline: SNN matcher on the device, reprojection check by the oracle, the tolerances
    and per-keypoint near-tie accounting of test_gpu_parity.py::test_graf_1_to_6_application_counts[hcori]."""
    from affnet_b200.Losses import match_snn
    from affnet_b200.pipeline import DetectDescribePipeline
    aff, ori, hn = nets
    z, f = gold("graf_match.npz"), gold("graf_full.npz")
    x1, x6 = gray_from_rgb(f["rgb"]), gray_from_rgb(z["rgb6"])
    assert x1.shape == x6.shape
    H, Wd = x1.shape[2:]
    pipe = DetectDescribePipeline(2, H, Wd, aff, hn, None, num_features=3000, do_ori=True)
    lafs, _, desc, cnt = pipe.run(torch.cat([x1, x6]).to(DEV))
    pipe.check()
    n1, n2 = int(cnt[0]), int(cnt[1])
    assert n1 == int(z["hcori_n1"]) and n2 == int(z["hcori_n2"]), (n1, n2)
    L1, d1, L2, d2 = lafs[0, :n1], desc[0, :n1], lafs[1, :n2], desc[1, :n2]
    i1, i2, _, _ = match_snn(d1, d2, float(z["snn"]))
    _, keep, _ = O.gt_correspondences(L1[i1].cpu(), L2[i2].cpu(), torch.from_numpy(z["H1to6"]), float(z["px"]))
    tent, true = int(i1.numel()), int(keep.numel())
    print("\ngraf 1<->6 batched, AffNet + histogram: %d tentatives / %d true (reference %d / %d)" % (tent, true, int(z["hcori_tent"]), int(z["hcori_true"])))
    assert abs(tent - int(z["hcori_tent"])) <= max(4, 0.03 * int(z["hcori_tent"]))
    assert abs(true - int(z["hcori_true"])) <= max(6, 0.08 * int(z["hcori_true"]))
    oL, _, st = O.detect(x1, W["affnet"], None, 3000, do_ori=True, debug=True)
    margin, share = orientation_boundary_shares(st["debug"]["ori"]["patches"])
    ia, ib = match_keypoints(oL, L1.cpu())
    eA = ((oL[ia][:, :, :2] - L1.cpu()[ib][:, :, :2]).abs().amax(dim=(1, 2)) / (oL[ia][:, 0, 0] * oL[ia][:, 1, 1] - oL[ia][:, 0, 1] * oL[ia][:, 1, 0]).abs().sqrt())
    flipped = (eA > 1e-2).nonzero().view(-1)
    print("img1: %d of %d matched keypoints take another orientation bin than the oracle; their top-2 bin margins (oracle): %s" % (
        flipped.numel(), len(ia), ["%.1e" % margin[ia[i]].item() for i in flipped.tolist()]))
    assert len(ia) >= 0.995 * oL.shape[0] and flipped.numel() <= 0.005 * len(ia)
    assert all(margin[ia[i]].item() < 5e-3 or share[ia[i]].item() > margin[ia[i]].item() for i in flipped.tolist())


ILL_CONDITIONED = 1e-4   # oracle_estimators.shape_spread at or above a tenth of the bound: base_A moves under an fp32-level perturbation


def accounted_rows(oL, odesc, dL, dd, st, tag, spread=None):
    """Match the oracle's keypoints (oL, odesc, state st of oracle_estimators.detect) with ours (dL, dd) and return (ia, ib, outside,
    unaccounted): `outside` are the matched pairs (indices into ia) with a LAF (relative to its scale) or descriptor error of 1e-3 or more,
    `unaccounted` those of them that are none of: an orientation near-tie (top-2 bin margin below 5e-3, or a pixel on a bin boundary that
    outweighs the margin), a keypoint whose base_A has an eigen ratio within 1e-3 of 6 or 1/6, or - when `spread` (the oracle's
    oracle_estimators.shape_spread per prefilter row) is given - a keypoint whose base_A the oracle's own loop moves by ILL_CONDITIONED or
    more under an fp32-level perturbation."""
    ia, ib = match_keypoints(oL, dL)
    A, B = oL[ia].double(), dL[ib].double()
    s = (A[:, 0, 0] * A[:, 1, 1] - A[:, 0, 1] * A[:, 1, 0]).abs().sqrt()
    eA = (A[:, :, :2] - B[:, :, :2]).abs().amax(dim=(1, 2)) / s
    ec = (A[:, :, 2] - B[:, :, 2]).abs().amax(dim=1) / s
    ed = (odesc[ia] - dd[ib]).abs().amax(dim=1).double()
    outside = ((eA >= TOL) | (ec >= TOL) | (ed >= TOL)).nonzero().view(-1).tolist()
    margin, share = orientation_boundary_shares(st["debug"]["ori"]["patches"])
    aff_dbg = st["debug"]["aff"]
    l1, l2 = O.batch_eig2x2(aff_dbg["base_A"][aff_dbg["idxs"]])
    ratio = (l1 / (l2 + 1e-8)).abs()
    near6 = ((ratio - 6.0).abs() < 1e-3) | ((ratio - 1.0 / 6.0).abs() < 1e-3)
    ill = torch.zeros(oL.shape[0], dtype=torch.bool) if spread is None else spread[aff_dbg["idxs"]] >= ILL_CONDITIONED
    tie = lambda k: margin[k].item() < 5e-3 or share[k].item() > margin[k].item()  # noqa: E731
    unaccounted = [i for i in outside if not (tie(ia[i]) or bool(near6[ia[i]]) or bool(ill[ia[i]]))]
    inside = sorted(set(range(len(ia))) - set(outside))
    print("\n%s: ours %d, oracle %d, matched %d; within the bound: max |dA|/s %.2e |dc|/s %.2e |ddesc| %.2e; %d outside (%d near-ties, %d "
          "ill-conditioned), %d unaccounted: %s" % (
              tag, dL.shape[0], oL.shape[0], len(ia), eA[inside].max().item(), ec[inside].max().item(), ed[inside].max().item(), len(outside),
              sum(tie(ia[i]) for i in outside), sum(bool(ill[ia[i]]) for i in outside), len(unaccounted),
              [(int(ia[i]), "%.1e" % eA[i].item(), "%.1e" % ed[i].item()) for i in unaccounted[:12]]))
    return ia, ib, outside, unaccounted, ill


@pytest.mark.parametrize("mode", ["affnet1-histogram", "baumberg16-histogram"])
def test_modes_vs_oracle_graf_1024(L, nets, mode):
    """graf img1 at 1024x768, K = 2000, against the oracle's restated loop: >= 99.5 % of the keypoints matched, and every matched keypoint
    with a LAF (relative to its scale) or descriptor error of 1e-3 or more accounted for individually (accounted_rows): an orientation
    near-tie, or an eigen ratio of base_A within 1e-3 of 6 or 1/6, or (Baumberg) an ill-conditioned shape.

    Sixteen Baumberg iterations amplify fp32-level differences for a few percent of the keypoints: the oracle's OWN loop moves their base_A
    by 1e-4 to more than 1 when its float64 sampler is replaced by the kernel's fp32 sampler arithmetic, its Baumberg step is evaluated in
    float64, or its input LAFs move by one ulp (oracle_estimators.shape_spread; median change 1.5e-6, none at 1 or 2 iterations: CPU
    test_baumberg_x16_conditioning_is_selective).  The kernels differ from the oracle by more than such a perturbation in every step (fp32
    sampler, other summation order), so those keypoints are accounted as ill-conditioned; the test requires them to stay a small minority,
    and every well-conditioned keypoint to be within the bound."""
    from affnet_b200.pipeline import DetectDescribePipeline
    aff, ori, hn = nets
    AffNet, iters, OriNet, do_ori = mode_args(mode, nets)
    img = _graf_1024()
    H, Wd = img.shape[2:]
    K = 2000
    pipe = DetectDescribePipeline(1, H, Wd, AffNet, hn, OriNet, num_features=K, do_ori=do_ori, num_Baum_iters=iters)
    lafs, _, desc, cnt = pipe.run(img.to(DEV))
    pipe.check()
    n = int(cnt[0])
    dL, dd = lafs[0, :n].cpu(), desc[0, :n].cpu()
    torch.set_num_threads(min(16, torch.get_num_threads()))
    shape = "affnet" if AffNet is aff else "baumberg"
    oL, _, st = OE.detect(img, shape, iters, W["affnet"], "histogram", None, K)
    odesc, _, _ = O.describe(oL, st, W["hardnet"])
    spread = OE.shape_spread(st, K, iters) if shape == "baumberg" else None
    ia, ib, outside, unaccounted, ill = accounted_rows(oL, odesc, dL, dd, st, mode + " vs oracle", spread)
    assert abs(n - oL.shape[0]) <= 0.005 * K and len(ia) >= 0.995 * oL.shape[0]
    assert not unaccounted, (mode, len(outside), unaccounted)
    if shape == "affnet":
        assert len(outside) <= 0.005 * len(ia), (mode, len(outside))
    else:
        assert int(ill.sum()) <= 0.1 * oL.shape[0], (mode, int(ill.sum()))
