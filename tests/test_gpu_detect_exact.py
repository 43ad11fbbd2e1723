"""GPU tests (-m gpu): every keypoint LAF the detector writes, bit for bit against the soft-argmax restatement
(tests/detect_restated.py) in the order of the kernel that produced it, and within the float64 bound.

The register kernel (detect_rows_kernel, at nlevels = 3) sums the window by rows; detect_level_kernel (other level counts, and
the response-map entry point) tap by tap.  The two orders differ in the last bits on most candidates, so only a bit-exact comparison tells
which ran.  Counts, responses, octave and level indices are the oracle's (tests/helpers.py::OracleCandidates) as in
test_gpu_detect.py, and rows beyond the count keep their sentinel.  The cases put candidates on the strip and band seams, on the
image edges at border 0 and 1, and at low contrast (pyramids scaled by 2^-k), where every positive pixel is a candidate, den is
dominated by its 1e-8 and the responses are fp32 subnormals."""
import ctypes as C

import numpy as np
import pytest
import torch

import affnet_oracle as O
import detect_cases as DC
from detect_restated import Restated, bits, bound_ratio, softargmax32, softargmax64
from helpers import (SENTINEL, Detector, OracleCandidates, adversarial_pyramid, flat_pyramid, gold, gpu_pyramids, gray_from_rgb,
                     mixed_batch, plan_sigmas, synthetic_image)

pytestmark = pytest.mark.gpu

DEV = "cuda"
MR = 5.192
ISENT = int(SENTINEL)
WORST = {}


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


def restated(cands, order, a_scale=1.0):
    return [Restated(c.pyr, c.sigmas, c.seq, order, a_scale=a_scale, th=c.th, device=DEV if c.total > 20000 else None) for c in cands]


def assert_exact(out, b, c, R, nf, tag, out_cap=None):
    """Image b of a select output: the oracle's count, responses, octave and level indices, the restated LAF bits and the float64
    bound, and the sentinel beyond the count.  -> rows compared."""
    resp, lafs, oc, lv, cnt = out
    idx = torch.from_numpy(np.ascontiguousarray(c.order(nf)[0])).long()
    if out_cap is not None:
        idx = idx[:out_cap]
    n = idx.numel()
    assert int(cnt[b]) == n, (tag, b, int(cnt[b]), n)
    assert torch.equal(resp[b, :n], c.resp[idx]), (tag, b)
    assert torch.equal(oc[b, :n].float(), c.oct[idx]) and torch.equal(lv[b, :n].float(), c.lvl[idx]), (tag, b)
    got, want = lafs[b, :n], R.lafs32[idx]
    bad = (bits(got) != bits(want)).any(2).any(1)
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError("%s image %d: %d of %d LAF rows differ from the restatement; first row %d (seq %#x): got %s want %s"
                             % (tag, b, int(bad.sum()), n, i, int(c.seq[idx[i]]), got[i].tolist(), want[i].tolist()))
    ratio = bound_ratio(got, R.lafs64[idx], R.bound[idx])
    assert ratio <= 1.0, (tag, b, ratio)
    key = tag[0] if isinstance(tag, tuple) else tag
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    assert bool((resp[b, n:] == SENTINEL).all()) and bool((lafs[b, n:] == SENTINEL).all()), (tag, b, "rows beyond the count")
    assert bool((oc[b, n:] == ISENT).all()) and bool((lv[b, n:] == ISENT).all()), (tag, b, "rows beyond the count")
    return n


def run_case(L, plan, pyrs, order, nfs, tag, buf=None, th=0.0, mr=MR, cap=None, select_all=True, a_scales=(1.0,)):
    det = Detector(L, plan, flat_pyramid(plan, pyrs) if buf is None else buf, th=th, mr=mr, cap=cap)
    cands = [OracleCandidates(p, plan_sigmas(plan), mr, th) for p in pyrs]
    assert int(det.cand_counts().max()) <= det.cap
    rows = 0
    for a in a_scales:
        Rs = restated(cands, order, a)
        for nf in nfs:
            out = det.checked_select(nf, None, a)
            rows += sum(assert_exact(out, b, c, R, nf, (tag, nf, a)) for b, (c, R) in enumerate(zip(cands, Rs)))
        if select_all:
            cap_all = max([c.total for c in cands] + [1])
            out = det.select_all(cap_all, a)
            rows += sum(assert_exact(out, b, c, R, -1, (tag, "all", a)) for b, (c, R) in enumerate(zip(cands, Rs)))
    print("\n%s (%s order): %d images, %d LAF rows bit-exact, worst error / bound %.3f" % (tag, order, plan.B, rows, WORST.get(tag, 0.0)))
    return det, cands


def _graf_1024():
    import cv2
    rgb = cv2.resize(gold("graf_full.npz")["rgb"], (1024, 768), interpolation=cv2.INTER_LINEAR)
    return gray_from_rgb(rgb)


# ---- default build ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["2x768x1024", "graf1024", "1080x1920"])
def test_rows_order_at_bench_shapes(L, case):
    imgs = {"2x768x1024": lambda: torch.cat([synthetic_image(768, 1024, 1234), synthetic_image(768, 1024, 1235)]),
            "graf1024": _graf_1024, "1080x1920": lambda: synthetic_image(1080, 1920, 77)}[case]()
    plan, buf, pyrs = gpu_pyramids(L, imgs, 3, 5)
    run_case(L, plan, pyrs, "rows", [3000, 16384], case, buf=buf, select_all=False)


def test_rows_order_odd_shapes_and_batches(L):
    for (h, w) in [(97, 131), (64, 29), (64, 30), (64, 31), (64, 61), (47, 70), (48, 70), (49, 70), (97, 70), (14, 50)]:
        plan, buf, pyrs = gpu_pyramids(L, mixed_batch(h, w, h * 1000 + w), 3)
        run_case(L, plan, pyrs, "rows", [1, 50], "odd B3", buf=buf)
    plan, buf, pyrs = gpu_pyramids(L, synthetic_image(97, 131, 9), 3)
    run_case(L, plan, pyrs, "rows", [100], "odd B1", buf=buf)
    imgs = torch.cat([synthetic_image(97, 131, 500 + b) if b % 5 else torch.full((1, 1, 97, 131), float(b)) for b in range(16)])
    plan, buf, pyrs = gpu_pyramids(L, imgs, 3)
    run_case(L, plan, pyrs, "rows", [50], "odd B16", buf=buf)


@pytest.mark.parametrize("nlevels", [1, 2, 4, 5, 6])
def test_taps_order_other_level_counts(L, nlevels):
    for (h, w) in [(97, 131), (64, 61), (49, 70)]:
        imgs = mixed_batch(h, w, h * 1000 + w)
        if nlevels == 1:        # the GPU blur refuses sigma 5.54: the oracle's dense blur builds the pyramid
            plan, buf = L.make_plan(3, h, w, 1, 1.6, 5), None
            pyrs = [O.scale_pyramid(imgs[b:b + 1], 1, 1.6, 5)[0] for b in range(3)]
        else:
            plan, buf, pyrs = gpu_pyramids(L, imgs, nlevels)
        run_case(L, plan, pyrs, "taps", [1, 50], "nlevels %d" % nlevels, buf=buf)
    plan8 = L.make_plan(8, 40, 40, nlevels, 1.6, 5)
    run_case(L, plan8, [adversarial_pyramid(s, nlevels) for s in range(8)], "taps", [1, 40], "nlevels %d adv" % nlevels)


def test_taps_order_from_response_maps(L):
    """ag_detect_level_from_responses: the nms_q4 golden maps and random ones, border 0, 1 and 5, with octave maps."""
    lib = L.lib()
    z = gold("nms_q4.npz")
    cases = [(z["low"], z["cur"], z["high"], z["omap"], list(z["scales"]))]
    g = torch.Generator().manual_seed(11)
    for (h, w) in ((37, 45), (64, 96), (12, 13)):
        maps = [O.gaussian_blur(torch.rand(1, 1, h, w, generator=g) * 500, 0.9)[0, 0].numpy() for _ in range(3)]
        om = (torch.rand(h, w, generator=g) * 3.2).byte().numpy()
        om[:, : w // 2] = 0
        cases.append((maps[0], maps[1], maps[2], om, [1.6, 2.0158736798317967, 2.5398416831491195]))
    rows, worst = 0, 0.0
    for mr in (5, 1, 0):
        for low, cur, high, om, scales in cases:
            h, w = cur.shape
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).view(1, 1, h, w)  # noqa: E731
            r_o, A_o, om_o, idx_o = O.nms3d_and_compose(t(low), t(cur), t(high), 0, om.copy(), scales, float(mr))
            plan = L.make_plan(1, h, w, 3, 1.6, 0)
            cap = h * w
            ws_buf = torch.zeros(lib.ag_detect_ws_bytes(C.byref(plan), cap), dtype=torch.uint8, device=DEV)
            ws = L.DetectWs()
            L.check(lib.ag_detect_ws_carve(C.byref(plan), cap, L.ptr(ws_buf), C.byref(ws)))
            d = [t(a).to(DEV).contiguous() for a in (low, cur, high)]
            om_in = torch.from_numpy(om).to(DEV).contiguous()
            om_out = torch.zeros_like(om_in)
            L.check(lib.ag_detect_level_from_responses(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), h, w, (C.c_double * 3)(*scales), mr,
                                                       L.ptr(om_in), L.ptr(om_out), 0, C.byref(ws), L.stream_ptr()))
            if r_o is None:
                continue
            n = r_o.numel()
            lafs = torch.full((n, 2, 3), SENTINEL, device=DEV)
            resp = torch.empty(n, device=DEV)
            oc, lv, cnt = (torch.empty(n, dtype=torch.int32, device=DEV), torch.empty(n, dtype=torch.int32, device=DEV),
                           torch.empty(1, dtype=torch.int32, device=DEV))
            L.check(lib.ag_select_keypoints(C.byref(plan), C.byref(ws), 0, 1.0, n, L.ptr(resp), L.ptr(lafs), L.ptr(oc), L.ptr(lv),
                                            L.ptr(cnt), L.stream_ptr()))
            torch.cuda.synchronize()
            assert int(cnt.item()) == n and torch.equal(resp.cpu(), r_o)
            maps3 = torch.stack([torch.from_numpy(np.ascontiguousarray(a)) for a in (low, cur, high)])
            want = softargmax32(maps3, scales, idx_o, "taps")
            assert torch.equal(bits(lafs.cpu()), bits(want)), (h, w, mr)
            L64, B64 = softargmax64(maps3, scales, idx_o)
            worst = max(worst, bound_ratio(lafs.cpu(), L64, B64), bound_ratio(A_o, L64, B64))
            rows += n
    print("\nresponse-map entry point (taps order): %d LAF rows bit-exact, worst error / bound %.3f (GPU and oracle)" % (rows, worst))
    assert worst <= 1.0


def test_rows_order_threshold_mode(L):
    plan, buf, pyrs = gpu_pyramids(L, mixed_batch(200, 328, 8), 3)
    run_case(L, plan, pyrs, "rows", [1, 300], "th 5", buf=buf, th=5.0)


def test_a_scale_through_both_selections(L):
    plan, buf, pyrs = gpu_pyramids(L, mixed_batch(200, 328, 61), 3)
    run_case(L, plan, pyrs, "rows", [300], "a_scale", buf=buf, a_scales=(1.0, 3.0, 5.192, 0.125))


# ---- seams and edges ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("border", [0, 1])
def test_seams_and_edges(L, border):
    """Blobs on the strip and band seams, the corners and the edges (tests/detect_cases.py::seam_pyramid), batched with a shifted
    copy; at border 0 candidates sit on all four image edges, so the zero padding of the window is read."""
    plan = L.make_plan(2, *DC.SEAM_SHAPE, 3, 1.6, 5)
    sizes, sig, pyr = DC.seam_case()
    assert [(plan.h[o], plan.w[o]) for o in range(plan.n_octaves)] == sizes and plan_sigmas(plan) == sig
    other = DC.seam_pyramid(sizes, 3, 4)
    run_case(L, plan, [pyr, other], "rows", [1, 200], "seams border %d" % border, mr=float(border))


# ---- low contrast ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def low_base(L):
    plan, buf, pyrs = gpu_pyramids(L, torch.cat([_graf_1024(), synthetic_image(768, 1024, 5)]), 3, 5)
    return plan, pyrs


@pytest.mark.parametrize("k", DC.LOW_K)
def test_low_contrast(L, low_base, k):
    """The graf 1024x768 pyramid and a synthetic one times 2^-k: at k >= 14 every positive pixel inside the border is a maximum,
    ~3 million candidates per image, selected by top-k at 2000 and 16384 (ties at the cut by seq) and all by
    ag_select_all_keypoints.  cand_cap holds every positive pixel; one below an image's raw count gives -1 for that image only."""
    plan, base = low_base
    pyrs = [DC.scaled(p, k) for p in base]
    cap = 3 * sum(plan.h[o] * plan.w[o] for o in range(plan.n_octaves))
    det, cands = run_case(L, plan, pyrs, "rows", [2000, 16384], "low contrast", cap=cap)
    n_c = det.cand_counts()
    print("low contrast k %d: raw candidates %s, totals %s" % (k, n_c.tolist(), [c.total for c in cands]))
    if k in (16, 66):
        big = int(n_c.argmax())
        small = Detector(L, plan, flat_pyramid(plan, pyrs), mr=MR, cap=int(n_c[big]) - 1)
        if int(n_c.min()) < int(n_c[big]):
            out = small.checked_select(2000)
            ref = det.checked_select(2000)
            assert int(out[4][big]) == -1
            for b in range(plan.B):
                if b != big:
                    for x, y in zip(out, ref):
                        assert torch.equal(x[b], y[b]), (k, b)
