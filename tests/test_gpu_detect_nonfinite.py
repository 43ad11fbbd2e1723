"""GPU tests (-m gpu): the detector on NaN, +inf and -inf values and on images that overflow fp32, against the oracle (pinned to the
unmodified reference by tests/test_detect_nonfinite_cpu.py) under its one deviation: a NaN survivor of the NMS is no keypoint.

- ag_hessian_response bit for bit against the oracle (NaN at the same positions) on the golden images, on 1xN, Nx1 and 1x1 images
  and at B = 3 with a NaN tile on a 32-pixel tile seam.
- ag_detect_level_from_responses on the golden NMS cases (a NaN beside a maximum, an inf centre, NaN survivors on a nonzero octave
  map, a level dropped by a NaN).
- The detector (the rows kernel at nlevels = 3, detect_level_kernel at other level counts) with NaN and
  +-inf in the image and in single pyramid levels on the 30-column strip seams, the 48-row band seams and the edges, at border 0 and
  5, for nlevels 1, 3 and 6; on images scaled by 2^k across the Hessian's overflow; a batch of 16 holding one NaN image.  Per image:
  the count, responses, octave and level identical to the oracle, LAFs bit for bit the restatement of the kernel's order (NaN
  positions included, the float64 bound where the sums are finite), no NaN response, rows beyond the count untouched.
- Selection through ag_select_keypoints, ag_select_topk_keypoints above 16384 keys and ag_select_all_keypoints at th = 28.41.
- DetectDescribePipeline (AffNet + OriNet, Baumberg + histogram) on a batch holding a NaN image, against the single-image API."""
import ctypes as C

import numpy as np
import pytest
import torch

import affnet_oracle as O
from detect_restated import Restated, bits, bound_ratio, same_bits, softargmax32
from helpers import (SENTINEL, Detector, OracleCandidates, flat_pyramid, gold, gpu_pyramids, load_weights, plan_sigmas,
                     synthetic_image)

pytestmark = pytest.mark.gpu

DEV = "cuda"
MR = 5.192
ISENT = int(SENTINEL)
Z = gold("nonfinite.npz")
NAN, INF = float("nan"), float("inf")
SEAMS = [(47, 29, NAN), (48, 30, INF), (20, 59, -INF), (48, 60, NAN), (0, 40, NAN), (96, 130, INF), (50, 0, NAN), (0, 0, -INF),
         (96, 89, NAN), (10, 130, NAN)]        # (y, x, value) on 97x131: strip seams x = 29|30, 59|60, band seam y = 47|48, edges


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


def order_of(plan):
    return "rows" if plan.n_levels - 2 == 3 else "taps"


def poke(img, spots):
    img = img.clone()
    for (y, x, v) in spots:
        if y < img.size(-2) and x < img.size(-1):
            img[..., y, x] = v
    return img


def assert_image(out, b, c, R, nf, tag, out_cap=None):
    """Image b of a select output against the oracle's candidates c and the restated rows R; -> rows compared."""
    resp, lafs, oc, lv, cnt = out
    idx = torch.from_numpy(np.ascontiguousarray(c.order(nf)[0])).long()
    if out_cap is not None:
        idx = idx[:out_cap]
    n = idx.numel()
    assert int(cnt[b]) == n, (tag, b, int(cnt[b]), n)
    assert not bool(torch.isnan(resp[b, :n]).any()), (tag, b, "NaN response emitted")
    assert torch.equal(resp[b, :n], c.resp[idx]), (tag, b)
    assert torch.equal(oc[b, :n].float(), c.oct[idx]) and torch.equal(lv[b, :n].float(), c.lvl[idx]), (tag, b)
    assert same_bits(lafs[b, :n], R.lafs32[idx]), (tag, b, "LAFs differ from the restated soft-argmax")
    fin = R.finite[idx]
    assert bound_ratio(lafs[b, :n][fin], R.lafs64[idx][fin], R.bound[idx][fin]) <= 1.0, (tag, b)
    assert bool((resp[b, n:] == SENTINEL).all()) and bool((lafs[b, n:] == SENTINEL).all()), (tag, b, "rows beyond the count")
    assert bool((oc[b, n:] == ISENT).all()) and bool((lv[b, n:] == ISENT).all()), (tag, b, "rows beyond the count")
    return n


def check(L, plan, pyrs, nfs, tag, buf=None, th=0.0, mr=MR, order=None):
    det = Detector(L, plan, flat_pyramid(plan, pyrs) if buf is None else buf, th=th, mr=mr)
    cands = [OracleCandidates(p, plan_sigmas(plan), mr, th) for p in pyrs]
    Rs = [Restated(c.pyr, c.sigmas, c.seq, order or order_of(plan), th=th) for c in cands]
    assert int(det.cand_counts().max()) <= det.cap
    rows = 0
    for nf in nfs:
        out = det.checked_select(nf, nf)
        rows += sum(assert_image(out, b, c, R, nf, (tag, nf)) for b, (c, R) in enumerate(zip(cands, Rs)))
    out = det.select_all(max([c.total for c in cands] + [1]))
    rows += sum(assert_image(out, b, c, R, 0, (tag, "all")) for b, (c, R) in enumerate(zip(cands, Rs)))
    return det, cands, rows


# ---- Hessian response maps -----------------------------------------------------------------------------------------------------
def test_hessian_response_bit_for_bit_with_nonfinite_pixels(L):
    from affnet_b200.HandCraftedModules import HessianResp
    imgs = [torch.from_numpy(Z[k]) for k in sorted(Z.files) if k.startswith("img_")]
    g = torch.Generator().manual_seed(5)
    for (h, w) in ((1, 37), (37, 1), (1, 1), (2, 2), (33, 65)):
        x = torch.rand(1, 1, h, w, generator=g) * 255
        imgs += [x, poke(x, [(0, 0, NAN)]), poke(x, [(h - 1, w - 1, INF)]), poke(x, [(h // 2, w // 2, -INF)])]
    x = torch.rand(3, 1, 70, 100, generator=g) * 255
    x[1, 0, 28:36, 60:68] = NAN                      # a NaN tile across the 32-pixel tile seams of the kernel
    x[2, 0, 31, 32] = INF
    imgs.append(x)
    n = 0
    for x in imgs:
        for s in (1.6, 3.2):
            got = HessianResp()(x.to(DEV).contiguous(), s).cpu()
            assert same_bits(got, O.hessian_response(x, s)), (tuple(x.shape), s)
            n += int((~torch.isfinite(got)).sum())
    print("\nag_hessian_response: %d maps bit for bit, %d non-finite responses" % (2 * len(imgs), n))
    assert n > 0


# ---- response-map entry point: the golden NMS cases ------------------------------------------------------------------------------
@pytest.mark.parametrize("mr", [5, 0])
def test_level_from_responses_on_golden_nms_cases(L, mr):
    lib = L.lib()
    names = sorted(k[4:-5] for k in Z.files if k.startswith("nms_") and k.endswith("_none"))
    scales = list(Z["nms_scales"])
    for name in names:
        arr = {k: Z["nms_%s_%s" % (name, k)] for k in ("low", "cur", "high", "omap")}
        h, w = arr["cur"].shape
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).float().view(1, 1, h, w)  # noqa: E731
        r_o, A_o, om_o, idx_o = O.nms3d_and_compose(t(arr["low"]), t(arr["cur"]), t(arr["high"]), 0, arr["omap"].copy(), scales, float(mr))
        plan = L.make_plan(1, h, w, 3, 1.6, 0)
        cap = h * w
        ws_buf = torch.full((lib.ag_detect_ws_bytes(C.byref(plan), cap),), 0xFF, dtype=torch.uint8, device=DEV)
        ws = L.DetectWs()
        L.check(lib.ag_detect_ws_carve(C.byref(plan), cap, L.ptr(ws_buf), C.byref(ws)))
        off = ws.d_cand_count - ws_buf.data_ptr()
        ws_buf[off:off + 4 * (1 + 2 * ws.n_level_slots)].zero_()
        d = [t(arr[k]).to(DEV).contiguous() for k in ("low", "cur", "high")]
        om_in = torch.from_numpy(arr["omap"]).to(DEV).contiguous()
        om_out = torch.full_like(om_in, 0xAB)
        L.check(lib.ag_detect_level_from_responses(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), h, w, (C.c_double * 3)(*scales), mr,
                                                   L.ptr(om_in), L.ptr(om_out), 0, C.byref(ws), L.stream_ptr()))
        torch.cuda.synchronize()
        lp = ws_buf[off + 4:off + 8].view(torch.int32).item()
        maps3 = torch.cat([t(arr[k])[0] for k in ("low", "cur", "high")])
        nm = O.nms3d_mask(t(arr["low"]), t(arr["cur"]), t(arr["high"]))
        if mr < w and mr < h:
            nm[..., :mr, :] = 0; nm[..., h - mr:, :] = 0; nm[..., :, :mr] = 0; nm[..., :, w - mr:] = 0
        nm = nm * (1.0 - torch.from_numpy(arr["omap"].astype(np.float32)))
        assert lp == int((nm > 0).sum()), (name, mr, lp)
        assert np.array_equal(om_out.cpu().numpy(), O.float_to_u8_cpu((torch.from_numpy(arr["omap"].astype(np.float32)) + nm[0, 0]).numpy())), (name, mr)
        if r_o is None:
            assert lp <= 1, (name, mr)
            continue
        n = r_o.numel()
        out = [torch.full((n,), SENTINEL, device=DEV), torch.full((n, 2, 3), SENTINEL, device=DEV)] + \
              [torch.full((n,), ISENT, dtype=torch.int32, device=DEV) for _ in range(2)] + [torch.empty(1, dtype=torch.int32, device=DEV)]
        L.check(lib.ag_select_keypoints(C.byref(plan), C.byref(ws), 0, 1.0, n, *[L.ptr(x) for x in out], L.stream_ptr()))
        torch.cuda.synchronize()
        resp, lafs, cnt = out[0].cpu(), out[1].cpu(), int(out[4].item())
        assert cnt == n and torch.equal(resp, r_o), (name, mr, cnt, n)
        assert torch.equal(bits(lafs), bits(softargmax32(maps3, scales, idx_o, "taps"))), (name, mr)


# ---- the detector ----------------------------------------------------------------------------------------------------------------
def seam_batch(h=97, w=131, seed=31):
    """A clean image, the image with NaN / +-inf pixels on the seams and edges, and a second textured image with one NaN in the middle."""
    a = synthetic_image(h, w, seed)
    return torch.cat([a, poke(a, SEAMS), poke(synthetic_image(h, w, seed + 1), [(h // 2, w // 2, NAN)])])


def level_pokes(pyrs, n_levels):
    """Single NaN / inf values written into one pyramid level (not spread by the blur), on seams and edges of octave 0."""
    out = []
    for b, pyr in enumerate(pyrs):
        p = [[lv.clone() for lv in octave] for octave in pyr]
        for i, (y, x, v) in enumerate(SEAMS):
            lv = p[0][(i + b) % n_levels]
            if y < lv.size(-2) and x < lv.size(-1):
                lv[..., y, x] = v
        out.append(p)
    return out


@pytest.mark.parametrize("nlevels", [3, 1, 6])
@pytest.mark.parametrize("border", [5, 0])
def test_detector_nonfinite_pixels_on_seams_and_edges(L, nlevels, border):
    imgs = seam_batch()
    if nlevels == 1:        # the GPU blur refuses sigma 5.54: the oracle's dense blur builds the pyramid
        plan, buf = L.make_plan(3, 97, 131, 1, 1.6, 5), None
        pyrs = [O.scale_pyramid(imgs[b:b + 1], 1, 1.6, 5)[0] for b in range(3)]
    else:
        plan, buf, pyrs = gpu_pyramids(L, imgs, nlevels)
    _, cands, rows = check(L, plan, pyrs, [1, 40], "image, nlevels %d border %d" % (nlevels, border), buf=buf, mr=float(border))
    assert cands[0].total > 0 and cands[2].total > 0
    poked = level_pokes(pyrs, nlevels + 2)
    _, cands2, rows2 = check(L, plan, poked, [1, 40], "levels, nlevels %d border %d" % (nlevels, border), mr=float(border))
    print("\nnon-finite pixels, nlevels %d, border %d: %d + %d rows identical to the oracle" % (nlevels, border, rows, rows2))


def test_detector_images_scaled_across_the_overflow(L):
    a = synthetic_image(97, 131, 41)
    ks = (54, 57, 58, 60, 61, 63)
    plan, buf, pyrs = gpu_pyramids(L, torch.cat([a * 2.0 ** k for k in ks]), 3)
    det, cands, rows = check(L, plan, pyrs, [1, 50], "scaled", buf=buf)
    nonfin = [int((~torch.isfinite(Restated(c.pyr, c.sigmas, c.seq, "rows").lafs32)).sum()) for c in cands]
    print("\nimages x 2^%s: %d rows, non-finite LAF entries per image %s, keypoints %s" % (ks, rows, nonfin, [c.total for c in cands]))


def test_batch_of_16_with_one_nan_image(L):
    h, w = 97, 131
    clean = torch.cat([synthetic_image(h, w, 700 + b) for b in range(16)])
    dirty = clean.clone()
    dirty[5, 0, 40, 60] = NAN
    plan, buf, pyrs = gpu_pyramids(L, clean, 3)
    plan_d, buf_d, pyrs_d = gpu_pyramids(L, dirty, 3)
    for b in range(16):
        if b != 5:
            assert all(torch.equal(x, y) for o in range(plan.n_octaves) for x, y in zip(pyrs[b][o], pyrs_d[b][o]))
    det_c, det_d = Detector(L, plan, buf), Detector(L, plan_d, buf_d)
    c5 = OracleCandidates(pyrs_d[5], plan_sigmas(plan_d), MR)
    R5 = Restated(c5.pyr, c5.sigmas, c5.seq, "rows")
    for nf, cap in ((50, 50), (0, 4096)):
        oc, od = (det_c.checked_select(nf, cap), det_d.checked_select(nf, cap)) if nf else (det_c.select_all(cap), det_d.select_all(cap))
        keep = torch.arange(16) != 5
        for x, y in zip(oc, od):
            assert torch.equal(bits(x[keep]) if x.is_floating_point() else x[keep], bits(y[keep]) if y.is_floating_point() else y[keep]), nf
        assert_image(od, 5, c5, R5, nf, ("B16 nan image", nf))


# ---- selection -------------------------------------------------------------------------------------------------------------------
def test_select_topk_above_16384_and_threshold_keep_all(L):
    img = synthetic_image(1080, 1920, 77)
    spots = [(y, x, NAN if (y + x) % 3 else INF) for y in range(47, 1080, 96) for x in range(29, 1920, 120)]
    imgs = torch.cat([poke(img, spots), img])
    plan, buf, pyrs = gpu_pyramids(L, imgs, 3)
    det = Detector(L, plan, buf)
    cands = [OracleCandidates(p, plan_sigmas(plan), MR) for p in pyrs]
    Rs = [Restated(c.pyr, c.sigmas, c.seq, "rows", device=DEV) for c in cands]
    nf = 20000
    lib = L.lib()
    n = lib.ag_select_topk_workspace_bytes(C.byref(plan), det.cap, nf)
    scratch = torch.full((max(n, 1),), 0xFF, dtype=torch.uint8, device=DEV)
    out = det._outputs(nf)
    L.check(lib.ag_select_topk_keypoints(C.byref(plan), C.byref(det.ws), nf, 1.0, nf, L.ptr(scratch), n, *[L.ptr(t) for t in out], L.stream_ptr()))
    torch.cuda.synchronize()
    out = tuple(t.cpu() for t in out)
    rows = sum(assert_image(out, b, c, R, nf, "topk 20000") for b, (c, R) in enumerate(zip(cands, Rs)))
    assert min(c.total for c in cands) > 16384
    # threshold mode: keep-all at th = 28.41
    pyr_t = pyrs
    det_t = Detector(L, plan, buf, th=28.41)
    ct = [OracleCandidates(p, plan_sigmas(plan), MR, 28.41) for p in pyr_t]
    Rt = [Restated(c.pyr, c.sigmas, c.seq, "rows", th=28.41, device=DEV) for c in ct]
    out = det_t.select_all(max(c.total for c in ct))
    rows_t = sum(assert_image(out, b, c, R, 0, "th 28.41 all") for b, (c, R) in enumerate(zip(ct, Rt)))
    print("\n1080x1920 with %d NaN / inf pixels: top-20000 %d rows, th 28.41 keep-all %d rows" % (len(spots), rows, rows_t))


# ---- the batched pipeline --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["affnet1-orinet", "baumberg16-histogram"])
def test_pipeline_batch_holding_a_nan_image(L, mode):
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    W = load_weights()
    a, o, hn = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); hn.load_state_dict(W["hardnet"])
    a, o, hn = a.eval().to(DEV), o.eval().to(DEV), hn.eval().to(DEV)
    aff, iters, ori, do_ori = {"affnet1-orinet": (a, 1, o, True), "baumberg16-histogram": (None, 16, None, True)}[mode]
    h, w, K = 200, 328, 300
    clean = torch.cat([synthetic_image(h, w, 90), synthetic_image(h, w, 91), synthetic_image(h, w, 92)])
    dirty = clean.clone()
    dirty[1, 0, 100, 150] = NAN
    dirty[1, 0, 47, 29] = INF
    outs = []
    for imgs in (clean, dirty):
        pipe = DetectDescribePipeline(3, h, w, aff, hn, ori, num_features=K, do_ori=do_ori, num_Baum_iters=iters)
        pipe.ws.fill_(0xFF)
        pipe.resp.fill_(SENTINEL); pipe.lafs.fill_(SENTINEL); pipe.desc.fill_(SENTINEL); pipe.count.fill_(ISENT)
        outs.append([t.clone().cpu() for t in pipe.run(imgs.to(DEV))])
        torch.cuda.synchronize()
    lafs, resp, desc, cnt = outs[1]
    for b in (0, 2):
        for x, y in zip(outs[0], outs[1]):
            assert torch.equal(bits(x[b]) if x.is_floating_point() else x[b], bits(y[b]) if y.is_floating_point() else y[b]), (mode, b)
    det = ScaleSpaceAffinePatchExtractor(mrSize=MR, num_features=K, border=5, num_Baum_iters=iters, AffNet=aff, OriNet=ori)
    n = int(cnt[1])
    assert n > 0
    dL, r = det(dirty[1:2].to(DEV), do_ori=do_ori)
    d = hn(det.extract_patches_from_pyr(dL, PS=32)).view(dL.size(0), -1)
    assert n == dL.size(0) and not bool(torch.isnan(resp[1, :n]).any())
    assert torch.equal(resp[1, :n], r.cpu()) and same_bits(lafs[1, :n], dL.cpu()) and same_bits(desc[1, :n], d.cpu()), mode
    assert bool((resp[1, n:] == SENTINEL).all()) and bool((desc[1, n:] == SENTINEL).all()), mode
    print("\npipeline %s: NaN image %d keypoints equal to the single-image API, %d descriptors with NaN; other images bit-identical"
          % (mode, n, int(torch.isnan(desc[1, :n]).any(1).sum())))
