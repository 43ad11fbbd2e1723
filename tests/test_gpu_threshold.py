"""GPU tests (-m gpu) of the threshold mode: ag_select_all_keypoints (ordered keep-all selection), ag_affine_shape_filter_all (keep-all
shape filter), the single-image API with th set above the 16384 keypoints the top-K kernels sort, and the batched pipeline's
ag_pipeline_create_th against that API.  Outputs, workspaces and scratch start poisoned, and rows at or beyond a count must keep their
sentinel."""
import ctypes as C

import numpy as np
import pytest
import torch

import affnet_oracle as O
import geometry_cases as K
import geometry_restated as G
import oracle_threshold as OT
from helpers import SENTINEL, TOL, gold, gray_from_rgb, load_weights, match_keypoints, synthetic_image

pytestmark = pytest.mark.gpu

DEV = "cuda"
MR = 5.192
ISENT = int(SENTINEL)
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


def graf_1024():
    import cv2
    return gray_from_rgb(cv2.resize(gold("graf_full.npz")["rgb"], (1024, 768), interpolation=cv2.INTER_LINEAR))


def crop_img():
    return gray_from_rgb(gold("graf_crop.npz")["rgb"])


def pyramids(L, imgs, border=5):
    from affnet_b200.HandCraftedModules import ScalePyramid
    plan, buf = ScalePyramid(3, 1.6, border).build(imgs.to(DEV).contiguous())
    views, _, _ = ScalePyramid.views(plan, buf)
    pyrs = [[[lv[b:b + 1].cpu() for lv in octave] for octave in views] for b in range(plan.B)]
    return plan, buf, pyrs


class Detection:
    """ag_detect with th over a 0xFF workspace of `cap` candidates per image; both selections into sentinel-filled outputs."""

    def __init__(self, L, plan, buf, th, cap=None):
        self.L, self.lib, self.plan = L, L.lib(), plan
        self.cap = cap or max(plan.H * plan.W // 4, 4096)
        self.ws_buf = torch.full((self.lib.ag_detect_ws_bytes(C.byref(plan), self.cap),), 0xFF, dtype=torch.uint8, device=DEV)
        self.ws = L.DetectWs()
        L.check(self.lib.ag_detect_ws_carve(C.byref(plan), self.cap, L.ptr(self.ws_buf), C.byref(self.ws)))
        L.check(self.lib.ag_detect(C.byref(plan), L.ptr(buf), float(th), int(MR), C.byref(self.ws), L.stream_ptr()))

    def cand_counts(self):
        off = self.ws.d_cand_count - self.ws_buf.data_ptr()
        return self.ws_buf[off:off + 4 * self.plan.B].view(torch.int32).cpu()

    def outputs(self, out_cap):
        B = self.plan.B
        return (torch.full((B, out_cap), SENTINEL, device=DEV), torch.full((B, out_cap, 2, 3), SENTINEL, device=DEV),
                torch.full((B, out_cap), ISENT, dtype=torch.int32, device=DEV), torch.full((B, out_cap), ISENT, dtype=torch.int32, device=DEV),
                torch.full((B,), ISENT, dtype=torch.int32, device=DEV))

    def select_topk(self, out_cap):
        out = self.outputs(out_cap)
        self.L.check(self.lib.ag_select_keypoints(C.byref(self.plan), C.byref(self.ws), 0, 1.0, out_cap, *[self.L.ptr(t) for t in out],
                                                  self.L.stream_ptr()))
        torch.cuda.synchronize()
        return [t.cpu() for t in out]

    def select_all(self, out_cap, a_scale=1.0):
        out = self.outputs(out_cap)
        n = self.lib.ag_select_all_workspace_bytes(C.byref(self.plan), self.cap)
        scratch = torch.full((n,), 0xFF, dtype=torch.uint8, device=DEV)
        self.L.check(self.lib.ag_select_all_keypoints(C.byref(self.plan), C.byref(self.ws), float(a_scale), out_cap, self.L.ptr(scratch), n,
                                                      *[self.L.ptr(t) for t in out], self.L.stream_ptr()))
        torch.cuda.synchronize()
        return [t.cpu() for t in out]


def assert_unwritten(out, b, n, tag):
    resp, lafs, oc, lv, _ = out
    assert bool((resp[b, n:] == SENTINEL).all()) and bool((lafs[b, n:] == SENTINEL).all()), (tag, b, "rows beyond the count written")
    assert bool((oc[b, n:] == ISENT).all()) and bool((lv[b, n:] == ISENT).all()), (tag, b, "rows beyond the count written")


# ---- ag_select_all_keypoints ------------------------------------------------------------------------------------------------------------
def small_batches():
    crop = crop_img()
    h, w = crop.shape[2:]
    const = torch.full_like(crop, 77.0)
    yield "crop", crop
    yield "crop+const", torch.cat([crop, const])
    yield "crop,const,flip", torch.cat([crop, const, crop.flip(3)])
    yield "4 mixed", torch.cat([crop, synthetic_image(h, w, 5), const, synthetic_image(h, w, 6)])
    yield "97x131 x3", torch.cat([synthetic_image(97, 131, s) for s in (1, 2, 3)])


@pytest.mark.parametrize("th", [0.0, 5.0, 28.41, -1.0])
def test_select_all_equals_select_keypoints(L, th):
    """At 16384 keypoints and below: ag_select_all_keypoints equals ag_select_keypoints(num_features = 0, out_cap = total) bit for bit,
    rows beyond the count included (both leave them unwritten), for B = 1..4 with a constant image among them."""
    for tag, imgs in small_batches():
        plan, buf, _ = pyramids(L, imgs)
        det = Detection(L, plan, buf, th)
        ref0 = det.select_topk(16384)
        total = max(int(ref0[4].max()), 1)
        assert total <= 16384
        for out_cap in sorted({total, total + 7}):
            ref, got = det.select_topk(out_cap), det.select_all(out_cap)
            for b in range(plan.B):
                if int(ref[4][b]) < 0:
                    # candidate overflow: ag_select_keypoints reports -1 after writing rows, the keep-all selection writes none
                    assert int(got[4][b]) == -1, (th, tag, b)
                    assert_unwritten(got, b, 0, (th, tag))
                    continue
                for x, y in zip(ref[:4], got[:4]):
                    assert torch.equal(x[b], y[b]), (th, tag, out_cap, b)
                assert int(ref[4][b]) == int(got[4][b])
        if "const" in tag:
            # a constant image has no keypoint at th >= 0; at th = -1 its response is exactly 1 everywhere, every pixel of the first
            # detection level is a maximum, and the candidate list overflows
            assert int(got[4][1]) == (-1 if th < 0 else 0), (th, tag)
        print("\nth %g %s: counts %s" % (th, tag, got[4].tolist()))


@pytest.mark.parametrize("shape", [(768, 1024), (1080, 1920)])
def test_select_all_above_16384_identical_to_oracle(L, shape):
    """th = 28.41 on the bench workload's first image and on 1080p (about 28.5k and 76k keypoints): the oracle's order, responses, octave and
    level indices bit for bit and its LAFs within 1e-6, given the same pyramid."""
    H, Wd = shape
    plan, buf, pyrs = pyramids(L, synthetic_image(H, Wd, 1234))
    det = Detection(L, plan, buf, 28.41)
    sig = [[plan.sigma[o][l] for l in range(plan.n_levels)] for o in range(plan.n_octaves)]
    r_o, L_o, p_o, l_o = O.multi_scale_detector(pyrs[0], sig, -1, MR, th=28.41)
    n = r_o.numel()
    assert n > 16384, n
    out = det.select_all(n + 100)
    resp, lafs, oc, lv, cnt = out
    print("\n%dx%d th 28.41: %d keypoints" % (Wd, H, n))
    assert int(cnt[0]) == n
    assert torch.equal(resp[0, :n], r_o) and torch.equal(oc[0, :n].float(), p_o) and torch.equal(lv[0, :n].float(), l_o)
    assert (lafs[0, :n] - L_o).abs().max().item() < 1e-6
    assert_unwritten(out, 0, n, shape)


def test_select_all_overflow_is_per_image(L):
    """out_cap one below an image's total, and a candidate list that overflows its capacity, give -1 for that image only, and nothing of
    it is written."""
    crop = crop_img()
    imgs = torch.cat([crop, crop[:, :, :, :160].repeat(1, 1, 1, 2)])
    plan, buf, _ = pyramids(L, imgs)
    det = Detection(L, plan, buf, 5.0)
    full = det.select_all(16384)
    tot = [int(c) for c in full[4]]
    big = int(np.argmax(tot))
    assert tot[big] > tot[1 - big] > 0, tot
    out = det.select_all(tot[big] - 1)
    assert int(out[4][big]) == -1 and int(out[4][1 - big]) == tot[1 - big], out[4]
    assert_unwritten(out, big, 0, "out_cap")
    n = tot[1 - big]
    for a, b in zip(out[:4], full[:4]):
        assert torch.equal(a[1 - big, :n], b[1 - big, :n])
    assert_unwritten(out, 1 - big, n, "out_cap")
    cands = [int(c) for c in det.cand_counts()]
    cap = (cands[0] + cands[1]) // 2
    assert min(cands) <= cap < max(cands), cands
    small = Detection(L, plan, buf, 5.0, cap=cap)
    out = small.select_all(16384)
    hi = int(np.argmax(cands))
    assert int(out[4][hi]) == -1 and int(out[4][1 - hi]) == tot[1 - hi], (cands, out[4])
    assert_unwritten(out, hi, 0, "cand_cap")
    for a, b in zip(out[:4], full[:4]):
        assert torch.equal(a[1 - hi, :tot[1 - hi]], b[1 - hi, :tot[1 - hi]])


# ---- ag_affine_shape_filter_all ---------------------------------------------------------------------------------------------------------
def run_filter(L, fn, A, Lf, resp, octs, lvls, counts, cap):
    B = len(counts)
    d = [torch.from_numpy(np.ascontiguousarray(x)).to(DEV) for x in (A, resp, Lf, octs, lvls)]
    outs = (torch.full((B, cap), SENTINEL, device=DEV), torch.full((B, cap, 2, 3), SENTINEL, device=DEV),
            torch.full((B, cap), ISENT, dtype=torch.int32, device=DEV), torch.full((B, cap), ISENT, dtype=torch.int32, device=DEV),
            torch.full((B,), ISENT, dtype=torch.int32, device=DEV))
    ci = torch.tensor(counts, dtype=torch.int32, device=DEV)
    args = [L.ptr(t) for t in d] + [L.ptr(ci), B, cap]
    if fn == "all":
        rc = L.lib().ag_affine_shape_filter_all(*args, *[L.ptr(t) for t in outs], L.stream_ptr())
    else:
        rc = L.lib().ag_affine_shape_filter(*args, 0, cap, *[L.ptr(t) for t in outs], L.stream_ptr())
    L.check(rc)
    torch.cuda.synchronize()
    return [t.cpu() for t in outs]


def same_bits(a, b):
    """Bit-identical fp32; any NaN equals any NaN (the device's NaN payload is canonical, numpy propagates the operand's)."""
    a = np.ascontiguousarray(a.numpy() if isinstance(a, torch.Tensor) else a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and bool(((a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))).all())


def filter_inputs(cap, B, seed):
    rows = [K.shape_rows(cap, seed + 13 * b) for b in range(B)]
    A = np.stack([r[0] for r in rows]); Lf = np.stack([r[1] for r in rows]); resp = np.stack([r[2] for r in rows])
    octs = np.arange(B * cap, dtype=np.int32).reshape(B, cap) % 7
    lvls = (np.arange(B * cap, dtype=np.int32).reshape(B, cap) * 3 + 1) % 5
    return A, Lf, resp, octs, lvls


@pytest.mark.parametrize("cap", [1, 33, 1025, 4097, 16384])
def test_shape_filter_all_equals_top_k_filter(L, cap):
    """Where ag_affine_shape_filter accepts the call, the keep-all filter equals its num_features = 0 answer bit for bit (ragged counts:
    full, 0, -1, above cap, two thirds)."""
    counts = [cap, 0, -1, cap + 5, max(1, 2 * cap // 3)]
    inp = filter_inputs(cap, len(counts), cap)
    a, b = run_filter(L, "all", *inp, counts, cap), run_filter(L, "topk", *inp, counts, cap)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), cap      # bit for bit, NaN rows included


@pytest.mark.parametrize("cap", [16385, 40000, 100000])
def test_shape_filter_all_above_16384_equals_restatement(L, cap):
    """Caps the shared-memory filter refuses: every survivor in order, bit for bit against tests/geometry_restated.py, counts 0, -1, above
    cap and the full cap; rows beyond the counts unwritten."""
    counts = [cap, 0, -1, cap + 3]
    A, Lf, resp, octs, lvls = filter_inputs(cap, len(counts), cap)
    out = run_filter(L, "all", A, Lf, resp, octs, lvls, counts, cap)
    ro, lo, oo, vo, co = out
    for b, c in enumerate(counts):
        n = max(0, min(c, cap))
        rows, vals, lafs = G.shape_filter(A[b, :n], resp[b, :n], Lf[b, :n], 0)
        m = len(rows)
        assert int(co[b]) == (-1 if c < 0 else m), (cap, b)
        assert same_bits(ro[b, :m], vals) and same_bits(lo[b, :m], lafs), (cap, b)
        assert np.array_equal(oo[b, :m].numpy(), octs[b, rows]) and np.array_equal(vo[b, :m].numpy(), lvls[b, rows]), (cap, b)
        assert_unwritten(out, b, m, cap)
    print("\ncap %d: %d survivors" % (cap, int(co[0])))


# ---- the single-image API ---------------------------------------------------------------------------------------------------------------
def test_mirror_threshold_mode_above_16384(L, nets):
    """ScaleSpaceAffinePatchExtractor(th=28.41, num_Baum_iters=1, AffNet) on the bench workload's first image (about 28.5k keypoints, which
    the top-K shape filter refuses): the detector's output is the oracle's given the same pyramid, and forward runs to the end with every
    survivor of the shape filter in order."""
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    img = synthetic_image(768, 1024, 1234)
    det = ScaleSpaceAffinePatchExtractor(mrSize=MR, num_features=2000, border=5, num_Baum_iters=1, th=28.41, AffNet=nets[0])
    r, la, oc, lv = det.multiScaleDetector(img.to(DEV), det.num)
    sig = det.sigmas
    pyr_g = [[t.cpu() for t in o] for o in det.scale_pyr]
    r_o, L_o, p_o, l_o = O.multi_scale_detector(pyr_g, sig, -1, MR, th=28.41)
    assert r_o.numel() > 16384
    assert r.numel() == r_o.numel() and torch.equal(r.cpu(), r_o) and torch.equal(oc.cpu(), p_o) and torch.equal(lv.cpu(), l_o)
    assert (la.cpu() - L_o).abs().max() < 1e-6
    dL, resp = det(img.to(DEV))
    assert 0 < dL.size(0) <= r_o.numel() and bool(torch.isfinite(dL).all())
    print("\nmirror th 28.41 on 1024x768 synthetic: %d detected, %d after the shape filter" % (r_o.numel(), dL.size(0)))


def test_mirror_threshold_mode_vs_oracle_graf_1024(L, nets):
    """graf img1 at 1024x768, th = 28.41, AffNet x 1 + HardNet, no orientation (hesaffnet.py's configuration) against the threshold-mode
    restatement: at least 99.5 % of the keypoints matched, and at least 99.5 % of them with LAF (relative to the scale) and descriptor errors
    below 1e-3."""
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    aff, _, hn = nets
    img = graf_1024()
    det = ScaleSpaceAffinePatchExtractor(mrSize=MR, num_features=2000, border=5, num_Baum_iters=1, th=28.41, AffNet=aff)
    dL, _ = det(img.to(DEV))
    dd = hn(det.extract_patches_from_pyr(dL, PS=32)).cpu()
    dL = dL.cpu()
    torch.set_num_threads(min(16, torch.get_num_threads()))
    oL, _, st = OT.detect(img, 28.41, "affnet", 1, W["affnet"])
    odesc, _, _ = O.describe(oL, st, W["hardnet"])
    ia, ib = match_keypoints(oL, dL)
    A, Bm = oL[ia].double(), dL[ib].double()
    s = (A[:, 0, 0] * A[:, 1, 1] - A[:, 0, 1] * A[:, 1, 0]).abs().sqrt()
    e = torch.maximum((A - Bm).abs().amax(dim=(1, 2)) / s, (odesc[ia] - dd[ib]).abs().amax(dim=1).double())
    print("\ngraf 1024x768 th 28.41: ours %d, oracle %d, matched %d, within 1e-3 %d, worst %.2e" % (
        dL.shape[0], oL.shape[0], len(ia), int((e < TOL).sum()), e.max().item()))
    assert len(ia) >= 0.995 * oL.shape[0] and abs(dL.shape[0] - oL.shape[0]) <= 0.005 * oL.shape[0]
    assert float((e < TOL).double().mean()) >= 0.995


# ---- the batched pipeline ---------------------------------------------------------------------------------------------------------------
def mode_args(mode, nets):
    """-> (AffNet, num_Baum_iters, OriNet, do_ori, descriptor module)."""
    from affnet_b200.pytorch_sift import SIFTNet
    aff, ori, hn = nets
    return {
        "affnet1-none": (aff, 1, None, False, hn),
        "affnet1-orinet": (aff, 1, ori, True, hn),
        "baumberg16-histogram": (None, 16, None, True, hn),
        "none-histogram": (None, 0, None, True, hn),
        "affnet1-none-sift32": (aff, 1, None, False, SIFTNet(32)),
    }[mode]


def compare_with_mirror(pipe, imgs, out, mode_a, th, tag):
    """Each image of a pipeline run against ScaleSpaceAffinePatchExtractor(th) + extract_patches_from_pyr + the descriptor, bit for bit."""
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    AffNet, iters, OriNet, do_ori, D = mode_a
    lafs, resp, desc, cnt = out
    det = ScaleSpaceAffinePatchExtractor(mrSize=MR, num_features=100, border=5, num_Baum_iters=iters, th=th, AffNet=AffNet, OriNet=OriNet)
    for b in range(imgs.size(0)):
        n = max(int(cnt[b]), 0)
        assert bool((resp[b, n:] == SENTINEL).all()) and bool((desc[b, n:] == SENTINEL).all()), (tag, b, "rows beyond the count written")
        if int(cnt[b]) < 0:
            continue
        dL, r = det(imgs[b:b + 1], do_ori=do_ori)
        assert n == dL.size(0), (tag, b, n, dL.size(0))
        if n == 0:
            continue
        d = D(det.extract_patches_from_pyr(dL, PS=32))
        assert torch.equal(resp[b, :n], r), (tag, b)
        assert torch.equal(lafs[b, :n], dL), (tag, b)
        assert torch.equal(desc[b, :n], d.view(n, -1)), (tag, b)


def run_pipe(pipe, imgs):
    pipe.ws.fill_(0xFF)
    pipe.resp.fill_(SENTINEL); pipe.lafs.fill_(SENTINEL); pipe.desc.fill_(SENTINEL); pipe.count.fill_(ISENT)
    out = [t.clone() for t in pipe.run(imgs)]
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("th", [28.41, -1.0])
@pytest.mark.parametrize("mode", ["affnet1-none", "affnet1-orinet", "baumberg16-histogram", "none-histogram", "affnet1-none-sift32"])
def test_pipeline_threshold_mode_equals_single_image_api(L, nets, mode, th):
    """B = 3 (graf crop, a synthetic image, a constant image) through ag_pipeline_create_th: every image equals the single-image API with
    the same th bit for bit; CUDA-graph replay equals the run with the same launch count.  The constant image has no keypoint at th =
    28.41; at th = -1 every pixel of its first detection level is a maximum of response exactly 1, its candidate list overflows, and its
    count is -1 with nothing written."""
    from affnet_b200.pipeline import DetectDescribePipeline
    m = mode_args(mode, nets)
    crop = crop_img()
    h, w = crop.shape[2:]
    imgs = torch.cat([crop, synthetic_image(h, w, 9), torch.full_like(crop, 77.0)]).to(DEV)
    Cap = 12000
    pipe = DetectDescribePipeline(3, h, w, m[0], m[4], m[2], num_features=Cap, do_ori=m[3], num_Baum_iters=m[1], th=th)
    out = run_pipe(pipe, imgs)
    cnt = out[3]
    assert int(cnt[2]) == (-1 if th < 0 else 0) and bool((cnt > 0)[:2].all()), cnt
    compare_with_mirror(pipe, imgs, out, m, th, (mode, th))
    launches = pipe.launches
    pipe.capture()
    l2, r2, d2, c2 = pipe.replay(imgs)
    torch.cuda.synchronize()
    assert torch.equal(c2, cnt) and pipe.launches == launches
    for b in range(3):
        n = max(int(cnt[b]), 0)
        assert torch.equal(l2[b, :n], out[0][b, :n]) and torch.equal(r2[b, :n], out[1][b, :n]) and torch.equal(d2[b, :n], out[2][b, :n])
    print("\n%s th %g: counts %s, %d launches" % (mode, th, cnt.tolist(), launches))


def test_pipeline_threshold_mode_above_16384(L, nets):
    """C = 32768 > 16384 on the bench workload's first image at th = 28.41 (AffNet x 1, no orientation): equal to the single-image API."""
    from affnet_b200.pipeline import DetectDescribePipeline
    m = mode_args("affnet1-none", nets)
    imgs = synthetic_image(768, 1024, 1234).to(DEV)
    pipe = DetectDescribePipeline(1, 768, 1024, m[0], m[4], m[2], num_features=32768, do_ori=False, num_Baum_iters=1, th=28.41)
    out = run_pipe(pipe, imgs)
    pipe.check()
    assert int(out[3][0]) > 16384, out[3]
    compare_with_mirror(pipe, imgs, out, m, 28.41, "C 32768")
    print("\nC 32768: %d keypoints, workspace %.2f GB" % (int(out[3][0]), pipe.ws_bytes / 1e9))


def test_pipeline_threshold_capacity_is_per_image(L, nets):
    """C one below an image's number of accepted candidates gives that image count -1 (and check() names both causes); the other images are
    unchanged."""
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200 import _lib
    m = mode_args("affnet1-none", nets)
    crop = crop_img()
    h, w = crop.shape[2:]
    imgs = torch.cat([crop, synthetic_image(h, w, 9), torch.full_like(crop, 77.0)]).to(DEV)
    plan, buf, _ = pyramids(L, imgs)
    det = Detection(L, plan, buf, 28.41)
    tot = [int(c) for c in det.select_all(16384)[4]]
    big = int(np.argmax(tot))
    full = run_pipe(DetectDescribePipeline(3, h, w, m[0], m[4], None, num_features=max(tot), do_ori=False, th=28.41), imgs)
    pipe = DetectDescribePipeline(3, h, w, m[0], m[4], None, num_features=tot[big] - 1, do_ori=False, th=28.41)
    out = run_pipe(pipe, imgs)
    cnt = out[3]
    assert int(cnt[big]) == -1, (tot, cnt)
    assert bool((out[1][big] == SENTINEL).all()) and bool((out[2][big] == SENTINEL).all())
    for b in range(3):
        if b != big:
            n = int(cnt[b])
            assert n == int(full[3][b])
            assert torch.equal(out[0][b, :n], full[0][b, :n]) and torch.equal(out[2][b, :n], full[2][b, :n])
    with pytest.raises(_lib.AffnetB200Error, match="more keypoints above th than num_features"):
        pipe.check()
