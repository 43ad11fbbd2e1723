"""GPU tests (-m gpu) of the SIFT descriptor: SIFTNet against the oracle on the golden patch sets, the fused pyramid kernel against
ag_extract_patches_pyr + ag_sift_describe over ragged counts, the batched pipeline with SIFT in place of HardNet (same geometry as the
HardNet pipeline, the single-image mirror's descriptors, graph replay, launches), the oracle at 1024x768 and the graf 1<->6 check."""
import ctypes as C

import pytest
import torch

import affnet_oracle as O
import oracle_estimators as OE
import oracle_sift as OS
from helpers import SENTINEL, gold, gray_from_rgb, load_weights
from test_gpu_pipeline_estimators import _graf_1024, accounted_rows

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


@pytest.mark.parametrize("PS", [16, 32, 41, 65])
def test_siftnet_vs_oracle_on_golden_patches(L, PS):
    """SIFT is continuous in its inputs (interpolated bins, a continuous clip), so the bound holds without near-tie exceptions."""
    from affnet_b200.pytorch_sift import SIFTNet
    z = gold("sift.npz")
    sift = SIFTNet(PS)
    for name in ("random", "graf", "constructed"):
        P = OS.golden_patches(z, name, PS)
        d = sift(P.to(DEV)).cpu()
        err = max((d - OS.sift_describe(P)).abs().max().item(), (d - torch.from_numpy(z["%s_desc_%d" % (name, PS)])).abs().max().item())
        print("\nPS %d %s: max |SIFTNet - oracle / reference| = %.2e" % (PS, name, err))
        assert bool(torch.isfinite(d).all()) and err <= 1e-5, (PS, name, err)


def _pyramid_and_lafs(L, B, cap, seed):
    """A B-image pyramid (graf crop, flipped crop, synthetic images) and random normalised LAFs [B,cap,2,3] with octave / level indices,
    some of them reaching past the image border."""
    from affnet_b200.HandCraftedModules import ScalePyramid
    img = gray_from_rgb(gold("graf_crop.npz")["rgb"])
    H, Wd = img.shape[2:]
    imgs = [img, img.flip(3)] + [O.synthetic_image(H, Wd, seed + b) for b in range(B - 2)]
    plan, pyr = ScalePyramid().build(torch.cat(imgs).to(DEV))
    g = torch.Generator().manual_seed(seed)
    ang = torch.rand(B, cap, generator=g) * 6.3
    sc = 0.02 + 0.15 * torch.rand(B, cap, generator=g)
    an = 0.6 + 0.8 * torch.rand(B, cap, generator=g)
    lafs = torch.zeros(B, cap, 2, 3)
    lafs[..., 0, 0], lafs[..., 0, 1] = sc * an * torch.cos(ang), -sc * torch.sin(ang)
    lafs[..., 1, 0], lafs[..., 1, 1] = sc * an * torch.sin(ang), sc * torch.cos(ang)
    lafs[..., 0, 2], lafs[..., 1, 2] = torch.rand(B, cap, generator=g) * 1.1 - 0.05, torch.rand(B, cap, generator=g) * 1.1 - 0.05
    oct_ = torch.randint(0, plan.n_octaves, (B, cap), generator=g, dtype=torch.int32)
    lvl = torch.randint(0, plan.n_levels, (B, cap), generator=g, dtype=torch.int32)
    return plan, pyr, lafs.to(DEV).contiguous(), oct_.to(DEV), lvl.to(DEV)


@pytest.mark.parametrize("PS", [32, 65])
def test_describe_pyr_equals_extract_then_describe(L, PS):
    """ag_sift_describe_pyr == ag_extract_patches_pyr + ag_sift_describe bit for bit, over ragged counts (0, 1, odd, a full odd cap,
    -1) into a sentinel-filled output; rows beyond the counts are untouched.  Also with no count array (every row valid)."""
    B, cap = 6, 37
    plan, pyr, lafs, oct_, lvl = _pyramid_and_lafs(L, B, cap, 3)
    counts = torch.tensor([0, 1, 7, cap, -1, 20], dtype=torch.int32, device=DEV)
    patches = torch.zeros(B, cap, PS, PS, device=DEV)
    L.check(L.lib().ag_extract_patches_pyr(C.byref(plan), L.ptr(pyr), L.ptr(lafs), L.ptr(oct_), L.ptr(lvl), None, cap, PS, L.ptr(patches),
                                           L.stream_ptr()))
    want = torch.full((B, cap, 128), SENTINEL, device=DEV)
    L.check(L.lib().ag_sift_describe(L.ptr(patches), B * cap, PS, 0.2, L.ptr(want), L.stream_ptr()))
    for cnt in (counts, None):
        out = torch.full((B, cap, 128), SENTINEL, device=DEV)
        L.check(L.lib().ag_sift_describe_pyr(C.byref(plan), L.ptr(pyr), L.ptr(lafs), L.ptr(oct_), L.ptr(lvl), L.ptr(cnt), cap, PS, 0.2,
                                             L.ptr(out), L.stream_ptr()))
        torch.cuda.synchronize()
        for b in range(B):
            n = cap if cnt is None else max(int(counts[b]), 0)
            assert torch.equal(out[b, :n], want[b, :n]), (PS, b, n)
            assert bool((out[b, n:] == SENTINEL).all()), (PS, b, "rows beyond the count written")
    assert bool(torch.isfinite(want).all())


def mode_args(mode, nets):
    aff, ori, _ = nets
    return {
        "affnet1-orinet": (aff, 1, ori, True),
        "affnet1-histogram": (aff, 1, None, True),
        "baumberg16-histogram": (None, 16, None, True),
        "none-histogram": (None, 0, None, True),
        "none-none": (None, 0, None, False),
    }[mode]


@pytest.mark.parametrize("mode,PS", [("affnet1-orinet", 32), ("affnet1-histogram", 32), ("baumberg16-histogram", 32),
                                     ("none-histogram", 41), ("none-none", 65)])
def test_pipeline_with_sift(L, nets, mode, PS):
    """Four images (graf crop, a constant image, the flipped crop, a synthetic image), K = 301, over a 0xFF workspace: LAFs, responses and
    counts equal to the HardNet pipeline of the same mode, descriptors equal to the single-image mirror (det, extract_patches_from_pyr(dL,
    PS), SIFTNet(PS)) bit for bit, graph replay equal to the run, and HardNet's launches replaced by one."""
    import affnet_b200._lib as lib
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.pytorch_sift import SIFTNet
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    hn = nets[2]
    AffNet, iters, OriNet, do_ori = mode_args(mode, nets)
    img = gray_from_rgb(gold("graf_crop.npz")["rgb"])
    imgs = torch.cat([img, torch.full_like(img, 77.0), img.flip(3), O.synthetic_image(img.size(2), img.size(3), 5)]).to(DEV)
    B, H, Wd = imgs.size(0), img.size(2), img.size(3)
    K = 301
    sift = SIFTNet(PS)
    res = {}
    for kind, desc_mod in (("hardnet", hn), ("sift", sift)):
        out = (torch.full((B, K, 2, 3), SENTINEL, device=DEV), torch.full((B, K, 128), SENTINEL, device=DEV),
               torch.full((B,), -7, dtype=torch.int32, device=DEV))
        pipe = DetectDescribePipeline(B, H, Wd, AffNet, desc_mod, OriNet, num_features=K, do_ori=do_ori, outputs=[out], num_Baum_iters=iters)
        pipe.ws.fill_(0xFF)
        pipe.resp.fill_(SENTINEL)
        r = [t.clone() for t in pipe.run(imgs)]
        torch.cuda.synchronize()
        res[kind] = (pipe, r, [n for n, _ in lib.profile(lambda: pipe.run(imgs))])
    (hp, (hl, hr, _, hc), hnames), (sp, (sl, sr, sd, sc), snames) = res["hardnet"], res["sift"]
    assert sp._used[2] is None and sp.ws_bytes <= hp.ws_bytes
    assert torch.equal(sc, hc) and int(sc[1]) == 0, (sc, hc)
    det = ScaleSpaceAffinePatchExtractor(mrSize=5.192, num_features=K, border=5, num_Baum_iters=iters, AffNet=AffNet, OriNet=OriNet)
    for b in range(B):
        n = int(sc[b])
        assert torch.equal(sl[b, :n], hl[b, :n]) and torch.equal(sr[b, :n], hr[b, :n]), (mode, b, "geometry differs from the HardNet pipeline")
        assert bool((sd[b, n:] == SENTINEL).all()), (mode, b, "rows beyond the count written")
        if n == 0:
            continue
        dL, _ = det(imgs[b:b + 1], do_ori=do_ori)
        assert torch.equal(dL, sl[b, :n]), (mode, b)
        d = sift(det.extract_patches_from_pyr(dL, PS=PS))
        assert torch.equal(sd[b, :n], d), (mode, b, (sd[b, :n] - d).abs().max().item())
    # launches: HardNet's (the trailing stage) replaced by the one fused SIFT kernel
    print("\n%s: launches HardNet %d, SIFT(%d) %d" % (mode, len(hnames), PS, len(snames)))
    assert snames[-1] == "sift_pyr_kernel" and snames[:-1] == hnames[:len(snames) - 1] and "sift_pyr_kernel" not in hnames
    assert sp.launches == len(snames) and hp.launches == len(hnames)
    n_hard = len(hnames) - (len(snames) - 1)
    assert n_hard >= 2 and len(snames) == len(hnames) - n_hard + 1
    sp.capture()
    l2, r2, d2, c2 = sp.replay(imgs)
    torch.cuda.synchronize()
    assert torch.equal(c2, sc)
    for b in range(B):
        n = int(sc[b])
        assert torch.equal(l2[b, :n], sl[b, :n]) and torch.equal(r2[b, :n], sr[b, :n]) and torch.equal(d2[b, :n], sd[b, :n]), (mode, b)


def test_pipeline_sift_needs_no_hardnet_handle(L):
    """create_desc with AG_DESC_SIFT and hardnet = NULL in a hand-crafted mode: no net at all, and a run works."""
    import affnet_b200._lib as lib
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.pytorch_sift import SIFTNet
    img = gray_from_rgb(gold("graf_crop.npz")["rgb"]).to(DEV)
    pipe = DetectDescribePipeline(1, img.size(2), img.size(3), None, SIFTNet(32), None, num_features=200, do_ori=True, num_Baum_iters=16)
    assert pipe._used == (None, None, None)
    lafs, _, desc, cnt = pipe.run(img)
    pipe.check()
    n = int(cnt[0])
    assert n > 100 and bool(torch.isfinite(desc[0, :n]).all())
    assert torch.allclose(desc[0, :n].norm(dim=1), torch.ones(n, device=DEV), atol=1e-5)
    cfg = lib.PipelineConfig(1, img.size(2), img.size(3), 200, 3, 5, 1.6, 5.192, 1, 0)
    est = lib.PipelineEstimators(lib.SHAPE_BAUMBERG, 16, 19, lib.ORI_HISTOGRAM, 19)
    h = C.c_void_p()
    L.check(L.lib().ag_pipeline_create_desc(C.byref(cfg), C.byref(est), C.byref(lib.PipelineDescriptor(lib.DESC_SIFT, 32, 0.2)), None, None,
                                            None, C.byref(h)))
    L.lib().ag_pipeline_destroy(h)


def test_sift_pipeline_vs_oracle_graf_1024(L, nets):
    """graf img1 at 1024x768, K = 2000, AffNet + histogram + SIFT(32) against the oracle: >= 99.5 % of the keypoints matched, descriptors
    within 1e-3, and every exception accounted for by the orientation near-tie rule of test_gpu_pipeline_estimators.py."""
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.pytorch_sift import SIFTNet
    aff = nets[0]
    img = _graf_1024()
    H, Wd = img.shape[2:]
    K = 2000
    pipe = DetectDescribePipeline(1, H, Wd, aff, SIFTNet(32), None, num_features=K, do_ori=True)
    lafs, _, desc, cnt = pipe.run(img.to(DEV))
    pipe.check()
    n = int(cnt[0])
    dL, dd = lafs[0, :n].cpu(), desc[0, :n].cpu()
    torch.set_num_threads(min(16, torch.get_num_threads()))
    oL, _, st = OE.detect(img, "affnet", 1, W["affnet"], "histogram", None, K)
    odesc, _, _ = OS.describe_sift(oL, st, 32)
    ia, ib, outside, unaccounted, _ = accounted_rows(oL, odesc, dL, dd, st, "AffNet + histogram + SIFT(32) vs oracle")
    assert abs(n - oL.shape[0]) <= 0.005 * K and len(ia) >= 0.995 * oL.shape[0]
    assert not unaccounted, (len(outside), unaccounted)
    assert len(outside) <= 0.005 * len(ia), len(outside)


def test_graf_1_to_6_application_counts_sift_batched(L, nets):
    """The reference's application check with SIFTNet(32) in place of HardNet (AffNet + histogram, K = 3000): graf img1 and img6 as one
    B = 2 batch, match_snn_pairs on the device, the oracle's 6 px reprojection check; within the slack of the batched HardNet test of the
    reference's SIFT counts."""
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.pytorch_sift import SIFTNet
    aff = nets[0]
    z, f, s = gold("graf_match.npz"), gold("graf_full.npz"), gold("sift.npz")
    x1, x6 = gray_from_rgb(f["rgb"]), gray_from_rgb(z["rgb6"])
    H, Wd = x1.shape[2:]
    pipe = DetectDescribePipeline(2, H, Wd, aff, SIFTNet(32), None, num_features=int(s["K"]), do_ori=True)
    lafs, _, desc, cnt = pipe.run(torch.cat([x1, x6]).to(DEV))
    pipe.check()
    n1, n2 = int(cnt[0]), int(cnt[1])
    assert n1 == int(s["hcori_n1"]) and n2 == int(s["hcori_n2"]), (n1, n2)
    pairs = torch.tensor([[0, 1]], dtype=torch.int32, device=DEV)
    tent, ntent, _, _ = match_snn_pairs(desc, cnt, desc, cnt, pairs, float(s["snn"]))
    nt = int(ntent[0])
    t = tent[0, :nt].long().cpu()
    _, keep, _ = O.gt_correspondences(lafs[0, :n1].cpu()[t[:, 0]], lafs[1, :n2].cpu()[t[:, 1]], torch.from_numpy(z["H1to6"]), float(s["px"]))
    true = int(keep.numel())
    gt, gtrue = int(s["hcori_tent"]), int(s["hcori_true"])
    print("\ngraf 1<->6 batched, AffNet + histogram + SIFT(32): %d tentatives / %d true (reference %d / %d)" % (nt, true, gt, gtrue))
    assert abs(nt - gt) <= max(4, 0.03 * gt) and abs(true - gtrue) <= max(6, 0.08 * gtrue)
