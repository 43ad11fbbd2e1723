"""GPU tests (-m gpu) of the top-K steps at any count: ag_select_topk_keypoints and ag_affine_shape_filter_topk above the 16384 keys the
shared-memory kernels sort (radix select, compaction and global-memory sort of csrc/topk.cuh), their identity with the old entry points
below it, and DetectDescribePipeline(large_k=True) against the single-image API and the CPU oracle.  Outputs and scratch start poisoned;
rows at or beyond a count must keep their sentinel.  Every large case asserts that its count really exceeds 16384."""
import ctypes as C

import numpy as np
import pytest
import torch

import affnet_oracle as O
import detect_cases as DC
import geometry_cases as K
import geometry_restated as G
from helpers import (SENTINEL, TOL, Detector, OracleCandidates, flat_pyramid, gold, gpu_pyramids, gray_from_rgb, load_weights,
                     match_keypoints, plan_sigmas, synthetic_image)

pytestmark = pytest.mark.gpu

DEV = "cuda"
MR = 5.192
ISENT = int(SENTINEL)
LIMIT = 16384
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


def outputs(B, cap):
    return (torch.full((B, cap), SENTINEL, device=DEV), torch.full((B, cap, 2, 3), SENTINEL, device=DEV),
            torch.full((B, cap), ISENT, dtype=torch.int32, device=DEV), torch.full((B, cap), ISENT, dtype=torch.int32, device=DEV),
            torch.full((B,), ISENT, dtype=torch.int32, device=DEV))


def select_topk(L, det, nf, out_cap=None):
    """ag_select_topk_keypoints over a 0xFF scratch -> outputs on the CPU."""
    lib, plan = L.lib(), det.plan
    out_cap = out_cap or nf
    n = lib.ag_select_topk_workspace_bytes(C.byref(plan), det.cap, out_cap)
    scratch = torch.full((max(n, 1),), 0xFF, dtype=torch.uint8, device=DEV)
    out = outputs(plan.B, out_cap)
    L.check(lib.ag_select_topk_keypoints(C.byref(plan), C.byref(det.ws), int(nf), 1.0, out_cap, L.ptr(scratch), n, *[L.ptr(t) for t in out],
                                         L.stream_ptr()))
    torch.cuda.synchronize()
    return tuple(t.cpu() for t in out)


def assert_unwritten(out, b, n, tag):
    resp, lafs, oc, lv, _ = out
    assert bool((resp[b, n:] == SENTINEL).all()) and bool((lafs[b, n:] == SENTINEL).all()), (tag, b, "rows beyond the count written")
    assert bool((oc[b, n:] == ISENT).all()) and bool((lv[b, n:] == ISENT).all()), (tag, b, "rows beyond the count written")


def assert_rule(out, every, b, c, nf, out_cap, tag):
    """Image b of a top-K output against the restated rule (OracleCandidates.order): responses, octave and level indices of the oracle's
    candidates, and LAFs bit for bit those of the keep-all selection (every candidate in seq order, pinned elsewhere) at the same rows."""
    idx = np.ascontiguousarray(c.order(nf)[0][:out_cap])
    n = len(idx)
    ti = torch.from_numpy(idx).long()
    resp, lafs, oc, lv, cnt = out
    assert int(cnt[b]) == n, (tag, b, int(cnt[b]), n)
    assert torch.equal(resp[b, :n], c.resp[ti]), (tag, b)
    assert torch.equal(oc[b, :n].float(), c.oct[ti]) and torch.equal(lv[b, :n].float(), c.lvl[ti]), (tag, b)
    assert torch.equal(resp[b, :n], every[0][b, ti]) and torch.equal(lafs[b, :n].view(-1, 6).view(torch.int32),
                                                                     every[1][b, ti].view(-1, 6).view(torch.int32)), (tag, b)
    assert_unwritten(out, b, n, tag)
    return n


def detection(L, imgs, cap=None):
    plan, buf, pyrs = gpu_pyramids(L, imgs)
    det = Detector(L, plan, buf, mr=MR, cap=cap)
    cands = [OracleCandidates(p, plan_sigmas(plan), MR) for p in pyrs]
    assert int(det.cand_counts().max()) <= det.cap
    every = det.select_all(max(c.total for c in cands))
    return plan, buf, pyrs, det, cands, every


@pytest.fixture(scope="module")
def hd(L):
    return detection(L, torch.cat([synthetic_image(1080, 1920, 31), synthetic_image(1080, 1920, 32)]))


def test_select_above_16384_bit_for_bit(L, hd):
    """B = 2 synthetic 1080p images: num_features 16385, 20000, total - 1, total, total + 1 (of either image) and out_cap below
    num_features, against the restated rule."""
    plan, buf, pyrs, det, cands, every = hd
    totals = [c.total for c in cands]
    print("\n1080p totals %s" % totals)
    assert min(totals) > 20001, totals
    nfs = sorted({16385, 20000} | {t + d for t in totals for d in (-1, 0, 1)})
    for nf in nfs:
        for out_cap in (nf, 16385 + 7, max(16385, nf - 1000)):
            out = select_topk(L, det, nf, out_cap)
            rows = [assert_rule(out, every, b, c, nf, out_cap, (nf, out_cap)) for b, c in enumerate(cands)]
            assert max(rows) > LIMIT, (nf, out_cap, rows)


def test_select_4k(L):
    plan, buf, pyrs, det, cands, every = detection(L, synthetic_image(2160, 3840, 77))
    total = cands[0].total
    print("\n4K total %d" % total)
    assert total > 40001
    for nf in (40000, total - 1, total + 1):
        out = select_topk(L, det, nf)
        assert assert_rule(out, every, 0, cands[0], nf, nf, ("4K", nf)) > LIMIT


def test_select_low_contrast_ties_at_the_cut(L):
    """The graf 1024x768 pyramid and a synthetic one times 2^-16: every positive pixel is a candidate (about 3 M), responses are fp32
    subnormals with many ties; num_features about 100000, chosen so that the cut splits a group of equal responses (broken by seq)."""
    import cv2
    img = gray_from_rgb(cv2.resize(gold("graf_full.npz")["rgb"], (1024, 768), interpolation=cv2.INTER_LINEAR))
    plan, _, base = gpu_pyramids(L, torch.cat([img, synthetic_image(768, 1024, 5)]))
    pyrs = [DC.scaled(p, 16) for p in base]
    cap = 3 * sum(plan.h[o] * plan.w[o] for o in range(plan.n_octaves))
    det = Detector(L, plan, flat_pyramid(plan, pyrs), mr=MR, cap=cap)
    cands = [OracleCandidates(p, plan_sigmas(plan), MR) for p in pyrs]
    every = det.select_all(max(c.total for c in cands))
    # from 100000 on, the first cut of image 0 that splits a group of equal responses
    v = np.sort(cands[0].resp.numpy())[::-1]
    nf = 100000
    while v[nf - 1] != v[nf]:
        nf += 1
    out = select_topk(L, det, nf)
    straddling = []
    for b, c in enumerate(cands):
        vals = c.resp[torch.from_numpy(np.ascontiguousarray(c.order(nf)[0])).long()]
        cut = float(vals[-1])
        straddling.append(int((c.resp == cut).sum()) - int((vals == cut).sum()))
        assert assert_rule(out, every, b, c, nf, nf, ("low", b)) == nf
    assert straddling[0] > 0
    print("\nlow contrast: raw candidates %s, nf %d, candidates tied with the cut left out %s" % (det.cand_counts().tolist(), nf, straddling))


def test_select_overflow_writes_nothing(L, hd):
    plan, buf, pyrs, det, cands, every = hd
    n_c = [int(x) for x in det.cand_counts()]
    big = int(np.argmax(n_c))
    assert min(n_c) < n_c[big]
    small = Detector(L, plan, buf, mr=MR, cap=n_c[big] - 1)
    out = select_topk(L, small, 20000)
    assert int(out[4][big]) == -1
    assert_unwritten(out, big, 0, "overflow")
    assert assert_rule(out, every, 1 - big, cands[1 - big], 20000, 20000, "other image") == 20000


def test_select_below_the_limit_is_the_old_entry_point(L, hd):
    plan, buf, pyrs, det, cands, every = hd
    for nf in (1, 2000, LIMIT):
        for out_cap in (nf, nf + 100000):
            a = det.select(nf, out_cap)[1]
            b = select_topk(L, det, nf, out_cap)
            for x, y in zip(a, b):
                assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (nf, out_cap)


# ---- ag_affine_shape_filter_topk ----------------------------------------------------------------------------------------------------------
def filter_inputs(cap, B, seed):
    rows = [K.shape_rows(cap, seed + 13 * b) for b in range(B)]
    A = np.stack([r[0] for r in rows]); Lf = np.stack([r[1] for r in rows]); resp = np.stack([r[2] for r in rows])
    octs = np.arange(B * cap, dtype=np.int32).reshape(B, cap) % 7
    lvls = (np.arange(B * cap, dtype=np.int32).reshape(B, cap) * 3 + 1) % 5
    return A, Lf, resp, octs, lvls


def run_filter(L, fn, inp, counts, cap, nf, out_cap):
    A, Lf, resp, octs, lvls = inp
    B = len(counts)
    d = [torch.from_numpy(np.ascontiguousarray(x)).to(DEV) for x in (A, resp, Lf, octs, lvls)]
    out = outputs(B, out_cap)
    ci = torch.tensor(counts, dtype=torch.int32, device=DEV)
    args = [L.ptr(t) for t in d] + [L.ptr(ci), B, cap, nf, out_cap]
    lib = L.lib()
    if fn == "old":
        rc = lib.ag_affine_shape_filter(*args, *[L.ptr(t) for t in out], L.stream_ptr())
    else:
        n = lib.ag_affine_shape_filter_topk_workspace_bytes(B, cap)
        scratch = torch.full((max(n, 1),), 0xFF, dtype=torch.uint8, device=DEV)
        rc = lib.ag_affine_shape_filter_topk(*args, L.ptr(scratch), n, *[L.ptr(t) for t in out], L.stream_ptr())
    L.check(rc)
    torch.cuda.synchronize()
    return [t.cpu() for t in out]


def same_bits(a, b):
    a = np.ascontiguousarray(a.numpy() if isinstance(a, torch.Tensor) else a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and bool(((a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))).all())


@pytest.mark.parametrize("cap", [16385, 40000, 100000])
def test_filter_above_16384_bit_for_bit(L, cap):
    """Responses with ties, zeros, negatives and -0: num_features below, at and above the survivors, so that rejected rows (key 0) make the
    cut ahead of negative survivors; counts full, 0, -1 and above cap; out_cap below the answer."""
    counts = [cap, 0, -1, cap + 3]
    inp = filter_inputs(cap, len(counts), cap)
    A, Lf, resp, octs, lvls = inp
    mask = G.shape_mask(A[0], Lf[0])
    S = int(mask.sum())
    assert 1 < S < cap and bool((resp[0][mask] < 0).any()) and bool((np.signbit(resp[0]) & (resp[0] == 0)).any())
    print("\ncap %d: %d survivors" % (cap, S))
    for nf, out_cap in ((LIMIT + 1, cap), (S - 1, cap), (S, cap), (S + 1, cap), (cap - 5, cap), (0, cap), (S - 1, LIMIT + 2)):
        out = run_filter(L, "topk", inp, counts, cap, nf, out_cap)
        ro, lo, oo, vo, co = out
        for b, c in enumerate(counts):
            n = max(0, min(c, cap))
            rows, vals, lafs = G.shape_filter(A[b, :n], resp[b, :n], Lf[b, :n], nf, out_cap)
            m = len(rows)
            assert int(co[b]) == (-1 if c < 0 else m), (cap, nf, b, int(co[b]), m)
            assert same_bits(ro[b, :m], vals) and same_bits(lo[b, :m], lafs), (cap, nf, b)
            assert np.array_equal(oo[b, :m].numpy(), octs[b, rows]) and np.array_equal(vo[b, :m].numpy(), lvls[b, rows]), (cap, nf, b)
            assert_unwritten(out, b, m, (cap, nf))
        if nf == S - 1:   # survivors with negative responses miss the cut: rejected rows (resp * keep = 0) rank above them
            assert not mask[G.shape_filter(A[0], resp[0], Lf[0], nf)[0]].all()


@pytest.mark.parametrize("cap", [1, 1025, LIMIT])
def test_filter_below_the_limit_is_the_old_entry_point(L, cap):
    counts = [cap, 0, -1, cap + 5, max(1, 2 * cap // 3)]
    inp = filter_inputs(cap, len(counts), cap + 1)
    for nf in (0, 1, cap // 2, cap):
        a, b = run_filter(L, "old", inp, counts, cap, nf, cap), run_filter(L, "topk", inp, counts, cap, nf, cap)
        for x, y in zip(a, b):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (cap, nf)


# ---- DetectDescribePipeline(large_k=True) -------------------------------------------------------------------------------------------------
def mode_args(mode, nets):
    """-> (AffNet, num_Baum_iters, OriNet, do_ori, descriptor module)."""
    from affnet_b200.pytorch_sift import SIFTNet
    aff, ori, hn = nets
    return {
        "affnet1-orinet": (aff, 1, ori, True, hn),
        "baumberg16-histogram": (None, 16, None, True, hn),
        "none-none": (None, 0, None, False, hn),
        "affnet1-none-sift32": (aff, 1, None, False, SIFTNet(32)),
    }[mode]


def run_pipe(pipe, imgs):
    pipe.ws.fill_(0xFF)
    pipe.resp.fill_(SENTINEL); pipe.lafs.fill_(SENTINEL); pipe.desc.fill_(SENTINEL); pipe.count.fill_(ISENT)
    out = [t.clone() for t in pipe.run(imgs)]
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("mode,Kf", [("affnet1-orinet", 20000), ("baumberg16-histogram", 20000), ("none-none", 40000),
                                     ("affnet1-none-sift32", 20000)])
def test_pipeline_large_k_equals_single_image_api(L, nets, mode, Kf):
    """B = 2 synthetic 1080p images through DetectDescribePipeline(large_k=True): every image's LAFs, responses and descriptors equal the
    single-image API's at the same K bit for bit, and a CUDA-graph replay equals the run."""
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.SparseImgRepresenter import ScaleSpaceAffinePatchExtractor
    AffNet, iters, OriNet, do_ori, D = mode_args(mode, nets)
    imgs = torch.cat([synthetic_image(1080, 1920, 41), synthetic_image(1080, 1920, 42)]).to(DEV)
    pipe = DetectDescribePipeline(2, 1080, 1920, AffNet, D, OriNet, num_features=Kf, do_ori=do_ori, num_Baum_iters=iters, large_k=True)
    out = run_pipe(pipe, imgs)
    pipe.check()
    lafs, resp, desc, cnt = out
    assert int(cnt.max()) > LIMIT, cnt
    det = ScaleSpaceAffinePatchExtractor(mrSize=MR, num_features=Kf, border=5, num_Baum_iters=iters, AffNet=AffNet, OriNet=OriNet)
    for b in range(2):
        n = int(cnt[b])
        assert bool((resp[b, n:] == SENTINEL).all()) and bool((desc[b, n:] == SENTINEL).all()), (mode, b, "rows beyond the count written")
        dL, r = det(imgs[b:b + 1], do_ori=do_ori)
        assert n == dL.size(0) and n > 0, (mode, b, n, dL.size(0))
        d = D(det.extract_patches_from_pyr(dL, PS=32))
        assert torch.equal(resp[b, :n], r), (mode, b)
        assert torch.equal(lafs[b, :n], dL), (mode, b)
        assert torch.equal(desc[b, :n], d.view(n, -1)), (mode, b)
    launches = pipe.launches
    pipe.capture()
    l2, r2, d2, c2 = pipe.replay(imgs)
    torch.cuda.synchronize()
    assert torch.equal(c2, cnt) and pipe.launches == launches
    for b in range(2):
        n = int(cnt[b])
        assert torch.equal(l2[b, :n], lafs[b, :n]) and torch.equal(r2[b, :n], resp[b, :n]) and torch.equal(d2[b, :n], desc[b, :n])
    print("\n%s K %d: counts %s, %d launches" % (mode, Kf, cnt.tolist(), launches))


def test_pipeline_large_k_within_the_limit_is_the_default(L, nets):
    """K = 2000: large_k=True builds the same pipeline - workspace, launch count and bits."""
    from affnet_b200.pipeline import DetectDescribePipeline
    aff, ori, hn = nets
    imgs = torch.cat([synthetic_image(1080, 1920, 41), synthetic_image(1080, 1920, 42)]).to(DEV)
    a = DetectDescribePipeline(2, 1080, 1920, aff, hn, ori, num_features=2000)
    b = DetectDescribePipeline(2, 1080, 1920, aff, hn, ori, num_features=2000, large_k=True)
    oa, ob = run_pipe(a, imgs), run_pipe(b, imgs)
    assert a.ws_bytes == b.ws_bytes and a.launches == b.launches
    for x, y in zip(oa, ob):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_pipeline_large_k_vs_oracle(L, nets):
    """One synthetic 1024x768 image at K = 20000 (a prefilter of 30000), AffNet x 1, OriNet and HardNet, against the CPU oracle: the
    end-to-end parity contract (SURVEY.md §8a-Q7: at least 99.5 % of the keypoints matched, matched LAFs and descriptors within 1e-3)."""
    from affnet_b200.pipeline import DetectDescribePipeline
    aff, ori, hn = nets
    Kf = 20000
    img = synthetic_image(768, 1024, 1234)
    pipe = DetectDescribePipeline(1, 768, 1024, aff, hn, ori, num_features=Kf, large_k=True)
    lafs, resp, desc, cnt = pipe.run(img.to(DEV))
    pipe.check()
    n = int(cnt[0])
    torch.set_num_threads(min(16, torch.get_num_threads()))
    oL, _, st = O.detect(img, W["affnet"], W["orinet"], Kf, do_ori=True)
    odesc, _, _ = O.describe(oL, st, W["hardnet"])
    dL, dd = lafs[0, :n].cpu(), desc[0, :n].cpu()
    ia, ib = match_keypoints(oL, dL)
    A, Bm = oL[ia].double(), dL[ib].double()
    s = (A[:, 0, 0] * A[:, 1, 1] - A[:, 0, 1] * A[:, 1, 0]).abs().sqrt()
    e = torch.maximum((A - Bm).abs().amax(dim=(1, 2)) / s, (odesc[ia] - dd[ib]).abs().amax(dim=1).double())
    print("\nK 20000 on 1024x768: ours %d, oracle %d, matched %d, within 1e-3 %d, worst %.2e" % (
        n, oL.shape[0], len(ia), int((e < TOL).sum()), e.max().item()))
    assert n > LIMIT and abs(n - oL.shape[0]) <= 0.005 * oL.shape[0]
    assert len(ia) >= 0.995 * oL.shape[0] and float((e < TOL).double().mean()) >= 0.995
