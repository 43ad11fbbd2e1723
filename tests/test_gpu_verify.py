"""GPU tests (-m gpu) of the device verification: ag_homography_ransac against its numpy restatement (tests/oracle_ransac.py) on
constructed pairs, ag_gt_correspondences_pairs against the oracle's gt_correspondences, both on seeded warped pipeline pairs and graf
1<->6, and both captured with the pipeline and the matcher in one CUDA graph.  Outputs are prefilled with sentinels, so rows and pairs
that must not be written are checked too."""
import numpy as np
import pytest
import torch

import affnet_oracle as O
import oracle_ransac as R
from helpers import SENTINEL, gold, gray_from_rgb, load_weights, synthetic_image
from verify_cases import corner_error, correspondences, project, random_homography

pytestmark = pytest.mark.gpu

DEV = "cuda"
INL_SENTINEL = 0xAB
CAP = 16384


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


@pytest.fixture(scope="module")
def nets():
    from affnet_b200.architectures import AffNetFast, OriNetFast
    from affnet_b200.HardNet import HardNet
    W = load_weights()
    a, o, h = AffNetFast(PS=32), OriNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); o.load_state_dict(W["orinet"]); h.load_state_dict(W["hardnet"])
    return a.eval().to(DEV), o.eval().to(DEV), h.eval().to(DEV)


def run_ransac(L, lafs1, lafs2, pairs, tent, ntent, th=2.0, conf=0.99, iters=50000, seed=0):
    """ag_homography_ransac over sentinel-filled outputs -> dict (H, inl, ninl, iters) on the host."""
    P, tcap = tent.shape[:2]
    o = dict(H=torch.full((P, 3, 3), SENTINEL, device=DEV), inl=torch.full((P, tcap), INL_SENTINEL, dtype=torch.uint8, device=DEV),
             ninl=torch.full((P,), -9, dtype=torch.int32, device=DEV), iters=torch.full((P,), -9, dtype=torch.int32, device=DEV))
    L.check(L.lib().ag_homography_ransac(L.ptr(lafs1), lafs1.size(0), lafs1.size(1), L.ptr(lafs2), lafs2.size(0), lafs2.size(1), L.ptr(pairs), P,
                                         L.ptr(tent), L.ptr(ntent), tcap, th, conf, iters, seed, L.ptr(o["H"]), L.ptr(o["inl"]), L.ptr(o["ninl"]),
                                         L.ptr(o["iters"]), L.stream_ptr()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


def run_gt(L, lafs1, lafs2, pairs, tent, ntent, H, th=6.0):
    P, tcap = tent.shape[:2]
    o = dict(min=torch.full((P, tcap), SENTINEL, device=DEV), idx2=torch.full((P, tcap), -7, dtype=torch.int32, device=DEV),
             true=torch.full((P, tcap), -7, dtype=torch.int32, device=DEV), ntrue=torch.full((P,), -9, dtype=torch.int32, device=DEV))
    L.check(L.lib().ag_gt_correspondences_pairs(L.ptr(lafs1), lafs1.size(0), lafs1.size(1), L.ptr(lafs2), lafs2.size(0), lafs2.size(1), L.ptr(pairs),
                                                P, L.ptr(tent), L.ptr(ntent), tcap, L.ptr(H), th, L.ptr(o["min"]), L.ptr(o["idx2"]), L.ptr(o["true"]),
                                                L.ptr(o["ntrue"]), L.stream_ptr()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


def constructed_cases():
    """name -> (pts [n,4] float32, H1to2 used to make them or None).  Image s of both LAF sets holds case s."""
    Hm = random_homography(7)
    cases = {}
    for n in (0, 3, 4, 5, 1000, 16384):
        pts, _ = correspondences(100 + n, n, Hm, outliers=0.0 if n <= 5 else 0.4, sigma=0.0 if n <= 5 else 0.3)
        cases["n%d" % n] = (pts, Hm)
    x = np.arange(50, dtype=np.float32) * 7.0
    cases["collinear"] = (np.stack([x, 2 * x + 3, x + 1, np.full_like(x, 9.0)], 1), None)          # collinear in both images
    cases["duplicated"] = (np.tile(np.array([[100.0, 200.0, 110.0, 190.0]], np.float32), (30, 1)), None)
    pts, _ = correspondences(9, 300, Hm)
    pts[::3] = pts[0]                                                                                 # every third row is row 0
    cases["some_duplicated"] = (pts, Hm)
    return cases, Hm


def build_sets(cases, seed=0):
    """LAF sets [S,CAP,2,3] whose image s holds case s's centres at permuted rows; tent [S,CAP,2] pointing at them, ntent [S]."""
    g = torch.Generator().manual_seed(seed)
    S = len(cases)
    l1, l2 = torch.zeros(S, CAP, 2, 3), torch.zeros(S, CAP, 2, 3)
    l1[..., 0, 0] = l1[..., 1, 1] = l2[..., 0, 0] = l2[..., 1, 1] = 3.0
    tent = torch.full((S, CAP, 2), -5, dtype=torch.int32)
    ntent = torch.zeros(S, dtype=torch.int32)
    for s, (pts, _) in enumerate(cases.values()):
        n = len(pts)
        r1, r2 = torch.randperm(CAP, generator=g)[:n], torch.randperm(CAP, generator=g)[:n]
        p = torch.from_numpy(pts)
        l1[s, r1, 0, 2], l1[s, r1, 1, 2], l2[s, r2, 0, 2], l2[s, r2, 1, 2] = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
        tent[s, :n, 0], tent[s, :n, 1], ntent[s] = r1.int(), r2.int(), n
    return l1.to(DEV), l2.to(DEV), tent.to(DEV), ntent.to(DEV)


def check_ransac_pair(o, p, pts, tag, th=2.0, max_iters=50000):
    """Pair p of the GPU outputs against the restatement: ninl and iters exactly, masks except near-threshold points, H to 1e-4."""
    H, m, n, it = R.ransac(pts, th, 0.99, max_iters, 0)
    k = len(pts)
    assert int(o["ninl"][p]) == n and int(o["iters"][p]) == it, (tag, int(o["ninl"][p]), n, int(o["iters"][p]), it)
    gm = o["inl"][p, :k].numpy()
    assert set(np.unique(gm).tolist()) <= {0, 1}, tag
    if n > 0:
        Hd = H.astype(np.float64).reshape(9)
        x, y = pts[:, 0].astype(np.float64), pts[:, 1].astype(np.float64)
        w = Hd[6] * x + Hd[7] * y + Hd[8]
        err = ((Hd[0] * x + Hd[1] * y + Hd[2]) / w - pts[:, 2]) ** 2 + ((Hd[3] * x + Hd[4] * y + Hd[5]) / w - pts[:, 3]) ** 2
        border = np.abs(err - th * th) <= 1e-6 * th * th
        assert np.array_equal(gm.astype(bool)[~border], m[~border]), tag
        assert np.linalg.norm(o["H"][p].numpy() - H) <= 1e-4 * np.linalg.norm(H), (tag, o["H"][p], H)
        assert float(o["H"][p, 2, 2]) == 1.0
    else:
        assert not gm.any() and not o["H"][p].any(), tag
    assert bool((o["inl"][p, k:] == INL_SENTINEL).all()), (tag, "mask rows beyond ntent written")
    return n, it


def test_constructed_pairs_against_the_restatement(L):
    cases, Hm = constructed_cases()
    names = list(cases)
    l1, l2, tent, ntent = build_sets(cases)
    S = len(names)
    # self pairs, then pairs that cannot be verified: ntent -1, ntent > tcap, image indices out of range, a row index out of range
    pl = [(s, s) for s in range(S)] + [(0, 0), (0, 0), (S, 0), (0, -1), (names.index("n1000"),) * 2, (names.index("n1000"),) * 2]
    P = len(pl)
    t = torch.cat([tent, tent[:1].repeat(4, 1, 1), tent[names.index("n1000")][None].repeat(2, 1, 1)]).contiguous()
    nt = torch.cat([ntent, torch.tensor([-1, CAP + 1, 4, 4, 1000, 1000], dtype=torch.int32, device=DEV)]).contiguous()
    t[S + 4, 500, 0] = CAP          # row index == cap: out of range
    t[S + 5, 999, 1] = -1
    pairs = torch.tensor(pl, dtype=torch.int32, device=DEV)
    o = run_ransac(L, l1, l2, pairs, t, nt)
    for s, name in enumerate(names):
        pts = cases[name][0]
        n, it = check_ransac_pair(o, s, pts, name)
        err = corner_error(o["H"][s].numpy(), Hm) if n > 0 else float("nan")
        print("\n%-16s n=%5d: %5d inliers, %5d iterations, corner error %.4f px" % (name, len(pts), n, it, err), end="")
        if name in ("n0", "n3", "collinear", "duplicated"):
            assert n == 0 and not o["H"][s].any()
        if name in ("collinear", "duplicated"):
            assert it == 50000
        if name in ("n4", "n5"):
            assert n == len(pts) and err < 1e-2
        if name in ("n1000", "n16384", "some_duplicated"):
            assert err < 1.0
    print()
    for p in range(S, P):
        assert int(o["ninl"][p]) == -1, (p, pl[p])
        assert bool((o["H"][p] == SENTINEL).all()) and bool((o["inl"][p] == INL_SENTINEL).all()) and int(o["iters"][p]) == -9, p
    # the same through the wrapper (iters included)
    from affnet_b200.ReprojectionStuff import find_homography_pairs
    H, inl, ninl, iters = find_homography_pairs(l1, t, nt, l2, pairs)
    torch.cuda.synchronize()
    assert torch.equal(ninl.cpu(), o["ninl"]) and torch.equal(iters.cpu()[:S], o["iters"][:S]) and torch.equal(H.cpu()[:S], o["H"][:S])


def test_determinism_and_independence(L):
    """Two runs give identical bits; a pair alone gives the bits it gives at a shuffled position of a list of 64."""
    cases, _ = constructed_cases()
    l1, l2, tent, ntent = build_sets(cases, seed=3)
    S = len(cases)
    k = list(cases).index("n1000")
    g = torch.Generator().manual_seed(4)
    pl = torch.randint(0, S, (64,), generator=g)
    pl[17] = k
    pairs = torch.stack([pl, pl], 1).int().to(DEV)
    t, nt = tent[pl.to(DEV)].contiguous(), ntent[pl.to(DEV)].contiguous()
    a = run_ransac(L, l1, l2, pairs, t, nt)
    b = run_ransac(L, l1, l2, pairs, t, nt)
    for key in a:
        assert torch.equal(a[key].view(torch.uint8) if a[key].is_floating_point() else a[key],
                           b[key].view(torch.uint8) if b[key].is_floating_point() else b[key]), key
    one = run_ransac(L, l1, l2, pairs[17:18].contiguous(), t[17:18].contiguous(), nt[17:18].contiguous())
    n = int(nt[17])
    assert torch.equal(one["H"][0].view(torch.int32), a["H"][17].view(torch.int32))
    assert torch.equal(one["inl"][0, :n], a["inl"][17, :n]) and one["ninl"][0] == a["ninl"][17] and one["iters"][0] == a["iters"][17]
    g1 = run_gt(L, l1, l2, pairs, t, nt, torch.eye(3, device=DEV).expand(64, 3, 3).contiguous())
    g2 = run_gt(L, l1, l2, pairs, t, nt, torch.eye(3, device=DEV).expand(64, 3, 3).contiguous())
    assert all(torch.equal(g1[key], g2[key]) for key in g1)


def gt_oracle(pts, Hm, th):
    """O.gt_correspondences on the tentatives' centres -> (kept rows, min_dist of every row)."""
    n = len(pts)
    if n == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.float32)
    LA, LB = torch.zeros(n, 2, 3), torch.zeros(n, 2, 3)
    LA[:, :, 2], LB[:, :, 2] = torch.from_numpy(pts[:, :2]), torch.from_numpy(pts[:, 2:])
    H = torch.from_numpy(np.asarray(Hm, np.float32))
    _, keep, _ = O.gt_correspondences(LA, LB, H, th)
    mn, _, _ = O.gt_correspondences(LA, LB, H, float("inf"))
    return keep.numpy(), mn.numpy()


def check_gt_pair(o, p, pts, Hm, th, tag):
    """The kept set equals the oracle's except rows within 0.1 px of the threshold; min_dist within 0.05 px, or min_dist^2 within 1 px^2.
    The reference's formula subtracts fp32 terms of up to ~3e6 px^2 (ulp 0.25), so its value carries rounding noise of ~1 px^2 that
    depends on the order of the operations: ~0.08 px at the 6 px threshold, more at small distances."""
    n = len(pts)
    keep, mn = gt_oracle(pts, Hm, th)
    ntrue = int(o["ntrue"][p])
    got = o["true"][p, :ntrue].numpy()
    assert np.all(np.diff(got) > 0), tag
    gm = o["min"][p, :n].numpy().astype(np.float64)
    near = np.abs(mn - th) <= 0.1
    assert set(got[~near[got]].tolist()) == set(keep[~near[keep]].tolist()), tag
    ok = (np.abs(gm - mn) <= 0.05) | (np.abs(gm * gm - mn.astype(np.float64) ** 2) <= 1.0)
    assert ok.all(), (tag, np.flatnonzero(~ok)[:5], gm[~ok][:5], mn[~ok][:5])
    assert bool((o["true"][p, ntrue:] == -7).all()) and bool((o["min"][p, n:] == SENTINEL).all()), (tag, "rows beyond ntent written")
    return ntrue, len(keep)


def test_gt_check_against_the_oracle(L):
    from affnet_b200.ReprojectionStuff import get_GT_correspondence_indexes, gt_correspondences_pairs
    cases, Hm = constructed_cases()
    names = ["n0", "n3", "n5", "n1000", "n16384", "some_duplicated"]
    sub = {k: cases[k] for k in names}
    l1, l2, tent, ntent = build_sets(sub, seed=5)
    P = len(names)
    Ht = torch.from_numpy(np.asarray(Hm, np.float32)).to(DEV).expand(P, 3, 3).contiguous()
    o = run_gt(L, l1, l2, None, tent, ntent, Ht, 6.0)
    for p, name in enumerate(names):
        nt, nk = check_gt_pair(o, p, sub[name][0], Hm, 6.0, name)
        print("\nGT %-16s: %d true of %d (oracle %d)" % (name, nt, len(sub[name][0]), nk), end="")
    print()
    # an out-of-range row and a -1 count give -1, and nothing else is written
    t2, n2 = tent.clone(), ntent.clone()
    t2[3, 10, 1] = CAP
    n2[0] = -1
    o2 = run_gt(L, l1, l2, None, t2, n2, Ht, 6.0)
    assert int(o2["ntrue"][0]) == -1 and int(o2["ntrue"][3]) == -1 and bool((o2["min"][3] == SENTINEL).all())
    assert torch.equal(o2["ntrue"][1:3], o["ntrue"][1:3])
    # the wrapper and the drop-in (P = 1)
    true, ntrue, mn, idx2 = gt_correspondences_pairs(l1, tent, ntent, Ht, l2)
    assert torch.equal(ntrue.cpu(), o["ntrue"])
    k = names.index("n1000")
    n = int(ntent[k])
    LA = l1[k][tent[k, :n, 0].long()]
    LB = l2[k][tent[k, :n, 1].long()]
    dmin, i1, i2 = get_GT_correspondence_indexes(LA, LB, Ht[k], 6.0)
    m = int(o["ntrue"][k])
    assert torch.equal(i1.cpu(), o["true"][k, :m].long()) and torch.equal(dmin.cpu(), o["min"][k][o["true"][k, :m].long()])
    assert torch.equal(i2.cpu(), o["idx2"][k][o["true"][k, :m].long()].long())


def warp(img, Hm):
    """img [1,1,H,W] warped by Hm (pixel-index coordinates): out(x) = img(Hm^-1 x), bilinear, zeros outside."""
    H, W = img.shape[2:]
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    src = project(np.linalg.inv(Hm), np.stack([xs.reshape(-1).numpy(), ys.reshape(-1).numpy()], 1))
    grid = torch.from_numpy(np.stack([2 * src[:, 0] / (W - 1) - 1, 2 * src[:, 1] / (H - 1) - 1], 1)).float().view(1, H, W, 2)
    return torch.nn.functional.grid_sample(img, grid, mode="bilinear", padding_mode="zeros", align_corners=True)


def test_synthetic_warped_pairs(L, nets):
    """8 seeded 768x1024 images, each with its own warp (rotation <= 20 deg, scale 0.8-1.1, perspective ~1e-4), as one B = 16 pipeline
    batch (AffNet + histogram orientation, K = 2000): at least 95 % of the tentatives are GT-true at 6 px, every estimate lies within the
    2 px inlier threshold of the true homography at all its inliers, and maps the frame's corners within 2 px.  On an H100 the corner
    errors were 0.08 to 1.37 px: where the warp moves a corner out of view there are no keypoints, and the estimate is extrapolated."""
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import find_homography_pairs, gt_correspondences_pairs
    aff, _, hn = nets
    Hh, Ww, K = 768, 1024, 2000
    Hs = [random_homography(500 + k, Hh, Ww) for k in range(8)]
    imgs = []
    for k in range(8):
        x = synthetic_image(Hh, Ww, 900 + k)
        imgs += [x, warp(x, Hs[k])]
    pipe = DetectDescribePipeline(16, Hh, Ww, aff, hn, None, num_features=K, do_ori=True)
    lafs, _, desc, cnt = pipe.run(torch.cat(imgs).to(DEV))
    pairs = torch.tensor([(2 * k, 2 * k + 1) for k in range(8)], device=DEV)
    tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=pairs)
    H, inl, ninl, iters = find_homography_pairs(lafs, tent, ntent, pairs=pairs)
    Ht = torch.from_numpy(np.stack(Hs).astype(np.float32)).to(DEV)
    true, ntrue, _, _ = gt_correspondences_pairs(lafs, tent, ntent, Ht, pairs=pairs)
    pipe.check()
    nt, nti, nin, it = ntent.tolist(), ntrue.tolist(), ninl.tolist(), iters.tolist()
    print()
    for k in range(8):
        He = H[k].cpu().numpy().astype(np.float64)
        err = corner_error(He, Hs[k], Hh, Ww)
        xy = lafs[2 * k, tent[k, :nt[k], 0].long(), :, 2].cpu().numpy().astype(np.float64)[inl[k, :nt[k]].cpu().numpy().astype(bool)]
        at_inl = float(np.linalg.norm(project(He, xy) - project(Hs[k], xy), axis=1).max())
        print("warped pair %d: %4d tentatives, %4d GT-true (>= %.0f), %4d inliers, %5d iterations, largest error at the inliers %.3f px (<= 2), "
              "corner error %.3f px (< 2)" % (k, nt[k], nti[k], 0.95 * nt[k], nin[k], it[k], at_inl, err))
        assert nt[k] > 100 and nti[k] >= 0.95 * nt[k] and at_inl <= 2.0 and err < 2.0, k
        # the restatement on the same tentatives gives the same counts
        t = tent[k, :nt[k]].long()
        pts = torch.cat([lafs[2 * k, t[:, 0], :, 2], lafs[2 * k + 1, t[:, 1], :, 2]], 1).cpu().numpy()
        _, _, n_r, it_r = R.ransac(pts)
        assert (n_r, it_r) == (nin[k], it[k]), k


def test_graf_1_to_6(L, nets):
    """graf img1 and img6 as one B = 2 batch (AffNet + histogram, K = 3000): the GT check gives the golden 91 true matches within 2, and
    RANSAC at 2 px finds >= 35 inliers, at each of which the estimate lies within 5 px of H1to6.  The inliers cover part of the frame
    only, and graf 1<->6 is a strong perspective change, so the error at the frame's corners is an extrapolation: it is printed, not
    asserted (the restatement on the oracle's 282 tentatives gives 46 inliers and 9.9 px there, cv2's RANSAC 42 and 6.0 px)."""
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import find_homography_pairs, gt_correspondences_pairs
    aff, _, hn = nets
    z, f = gold("graf_match.npz"), gold("graf_full.npz")
    x1, x6 = gray_from_rgb(f["rgb"]), gray_from_rgb(z["rgb6"])
    Hh, Ww = x1.shape[2:]
    pipe = DetectDescribePipeline(2, Hh, Ww, aff, hn, None, num_features=3000, do_ori=True)
    lafs, _, desc, cnt = pipe.run(torch.cat([x1, x6]).to(DEV))
    pairs = torch.tensor([[0, 1]], device=DEV)
    tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=pairs, SNN_threshold=float(z["snn"]))
    H16 = torch.from_numpy(z["H1to6"].astype(np.float32)).to(DEV)
    true, ntrue, _, _ = gt_correspondences_pairs(lafs, tent, ntent, H16, pairs=pairs, dist_threshold=float(z["px"]))
    H, inl, ninl, iters = find_homography_pairs(lafs, tent, ntent, pairs=pairs)
    pipe.check()
    n = int(ntent[0])
    He = H[0].cpu().numpy().astype(np.float64)
    xy = lafs[0, tent[0, :n, 0].long(), :, 2].cpu().numpy().astype(np.float64)[inl[0, :n].cpu().numpy().astype(bool)]
    at_inl = float(np.linalg.norm(project(He, xy) - project(z["H1to6"], xy), axis=1).max())
    err = corner_error(He, z["H1to6"], Hh, Ww)
    print("\ngraf 1<->6: %d tentatives, %d GT-true (golden %d, within 2), RANSAC %d inliers (>= 35) in %d iterations, largest error at the "
          "inliers %.2f px (<= 5), corner error %.2f px" % (n, int(ntrue[0]), int(z["hcori_true"]), int(ninl[0]), int(iters[0]), at_inl, err))
    assert abs(int(ntrue[0]) - int(z["hcori_true"])) <= 2
    assert int(ninl[0]) >= 35 and at_inl <= 5.0


def test_one_graph_with_the_pipeline_and_matcher(L, nets):
    """pipe.run + match_snn_pairs + find_homography_pairs + gt_correspondences_pairs in ONE CUDA graph over all 240 ordered pairs of 16
    images; a replay on other images equals the eager run, and each verification call is one launch for 1 pair and for 240."""
    import affnet_b200._lib as lib
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import find_homography_pairs, gt_correspondences_pairs
    aff, _, hn = nets
    B, Hh, Ww, K = 16, 768, 1024, 2000
    mk = lambda s: torch.cat([synthetic_image(Hh, Ww, s + i) for i in range(B)]).to(DEV)  # noqa: E731
    imgs, imgs2 = mk(1234), mk(777)
    pairs = torch.tensor([(i, j) for i in range(B) for j in range(B) if i != j], device=DEV)
    Hid = torch.eye(3, device=DEV).expand(pairs.size(0), 3, 3).contiguous()
    pipe = DetectDescribePipeline(B, Hh, Ww, aff, hn, None, num_features=K, do_ori=True)

    def step(x):
        lafs, _, d, c = pipe.run(x)
        tent, ntent, _, _ = match_snn_pairs(d, c, pairs=pairs)
        return (ntent,) + find_homography_pairs(lafs, tent, ntent, pairs=pairs) + gt_correspondences_pairs(lafs, tent, ntent, Hid, pairs=pairs)

    lafs, _, d, c = pipe.run(imgs)
    tent, ntent, _, _ = match_snn_pairs(d, c, pairs=pairs)
    for fn in (lambda q: find_homography_pairs(lafs, tent[q], ntent[q], pairs=pairs[q]),
               lambda q: gt_correspondences_pairs(lafs, tent[q], ntent[q], Hid[q], pairs=pairs[q])):
        n_one = len(lib.profile(lambda: fn(slice(0, 1))))
        n_all = len(lib.profile(lambda: fn(slice(None))))
        assert n_one == n_all == 1, (n_one, n_all)

    static_in = imgs.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(static_in)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = step(static_in)
    static_in.copy_(imgs2)
    g.replay()
    torch.cuda.synchronize()
    got = [t.clone() for t in res]
    ref = step(imgs2)
    torch.cuda.synchronize()
    nt, ninl, ntrue = ref[0].tolist(), ref[3].tolist(), ref[6].tolist()
    # (ntent, H, inl, ninl, iters, true, ntrue, min_dist, idx2)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[3], ref[3]) and torch.equal(got[4], ref[4]) and torch.equal(got[6], ref[6])
    for p in range(pairs.size(0)):
        n = max(nt[p], 0)
        assert torch.equal(got[2][p, :n], ref[2][p, :n]) and torch.equal(got[7][p, :n], ref[7][p, :n]), p
        assert torch.equal(got[5][p, :max(ntrue[p], 0)], ref[5][p, :max(ntrue[p], 0)]), p
        if ninl[p] >= 0:
            assert torch.equal(got[1][p], ref[1][p]), p
    print("\n240 pairs in one graph: tentatives %d..%d, inliers %d..%d" % (min(nt), max(nt), min(ninl), max(ninl)))
