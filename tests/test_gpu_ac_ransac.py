"""GPU tests (-m gpu) of the affine homography RANSAC (ag_homography_ransac_affine, find_homography_pairs(affine=True)): bit for bit
against its numpy restatement (tests/oracle_ac_ransac.py) on constructed scenes with frames, ragged and invalid counts, degenerate sets and
laf_th = inf; determinism and pair independence; the warped pipeline pairs and graf 1->6 next to the 4-point RANSAC; and one CUDA graph
with the pipeline and the matcher.  Outputs are prefilled with sentinels, so rows and pairs that must not be written are checked too."""
import math

import numpy as np
import pytest
import torch

import affine_cases as AC
import oracle_ac_ransac as A
import oracle_ransac as R
from helpers import SENTINEL, gold, gray_from_rgb, load_weights, synthetic_image
from test_gpu_verify import INL_SENTINEL, warp
from verify_cases import corner_error, project, random_homography

pytestmark = pytest.mark.gpu

DEV = "cuda"
CAP = 4096


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


def default_laf_th():
    from affnet_b200.ReprojectionStuff import AFFINE_LAF_TH
    return AFFINE_LAF_TH


def run_ac(L, lafs1, lafs2, pairs, tent, ntent, th=2.0, lth=None, conf=0.99, iters=50000, seed=0):
    """ag_homography_ransac_affine over sentinel-filled outputs -> dict (H, inl, ninl, iters) on the host."""
    P, tcap = tent.shape[:2]
    lth = default_laf_th() if lth is None else lth
    o = dict(H=torch.full((P, 3, 3), SENTINEL, device=DEV), inl=torch.full((P, tcap), INL_SENTINEL, dtype=torch.uint8, device=DEV),
             ninl=torch.full((P,), -9, dtype=torch.int32, device=DEV), iters=torch.full((P,), -9, dtype=torch.int32, device=DEV))
    L.check(L.lib().ag_homography_ransac_affine(L.ptr(lafs1), lafs1.size(0), lafs1.size(1), L.ptr(lafs2), lafs2.size(0), lafs2.size(1),
                                                L.ptr(pairs), P, L.ptr(tent), L.ptr(ntent), tcap, th, lth, conf, iters, seed, L.ptr(o["H"]),
                                                L.ptr(o["inl"]), L.ptr(o["ninl"]), L.ptr(o["iters"]), L.stream_ptr()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


def constructed_cases():
    """name -> (lafs1 [n,2,3], lafs2 [n,2,3], H or None).  Image s of both LAF sets holds case s."""
    cases = {}
    for n in (0, 1, 2, 3, 5):
        l1, l2, Hm, _ = AC.scene(200 + n, n, outliers=0.0, eps=0.0, sigma=0.0)
        cases["exact_n%d" % n] = (l1, l2, Hm)
    for name, n, out, fo in (("n1000_40", 1000, 0.4, 0.05), ("n1000_70", 1000, 0.7, 0.05), ("n1000_85", 1000, 0.85, 0.05),
                             ("n3000_multitile", 3000, 0.5, 0.1), ("n300_frame_outliers", 300, 0.2, 0.4)):
        l1, l2, Hm, _ = AC.scene(300 + n + int(100 * out), n, outliers=out, frame_outliers=fo)
        cases[name] = (l1, l2, Hm)
    l1, l2, Hm, _ = AC.scene(7, 400, outliers=0.3)
    l1[::4, 0, 0] = np.nan                                               # NaN frames on a quarter of the rows
    l2[1::7, 1, 1] = np.inf
    cases["nan_frames"] = (l1, l2, Hm)
    l1, l2, Hm, _ = AC.scene(8, 200, outliers=0.3)
    l1[:, 1, :2] = 0.0                                                   # every image-1 frame singular: every sample degenerate
    cases["all_degenerate"] = (l1, l2, None)
    l1, l2, Hm, _ = AC.scene(9, 60, outliers=0.0)
    l1[:, :, 2] = l1[0, :, 2]                                            # one centre in image 1
    cases["coincident"] = (l1, l2, None)
    l1, l2 = AC.pivot_scene(11, 64)                                      # every sample rejected by the relative Cholesky pivot rule
    cases["pivot"] = (l1, l2, None)
    return cases


def build_sets(cases, seed=0):
    """LAF sets [S,CAP,2,3] whose image s holds case s's frames at permuted rows; tent [S,CAP,2] pointing at them, ntent [S]."""
    g = torch.Generator().manual_seed(seed)
    S = len(cases)
    l1, l2 = torch.zeros(S, CAP, 2, 3), torch.zeros(S, CAP, 2, 3)
    l1[..., 0, 0] = l1[..., 1, 1] = l2[..., 0, 0] = l2[..., 1, 1] = 3.0
    tent = torch.full((S, CAP, 2), -5, dtype=torch.int32)
    ntent = torch.zeros(S, dtype=torch.int32)
    for s, (a, b, _) in enumerate(cases.values()):
        n = len(a)
        r1, r2 = torch.randperm(CAP, generator=g)[:n], torch.randperm(CAP, generator=g)[:n]
        l1[s, r1], l2[s, r2] = torch.from_numpy(a), torch.from_numpy(b)
        tent[s, :n, 0], tent[s, :n, 1], ntent[s] = r1.int(), r2.int(), n
    return l1.to(DEV), l2.to(DEV), tent.to(DEV), ntent.to(DEV)


def check_pair(o, p, ac, tag, lth, th=2.0):
    """Pair p of the GPU outputs against the restatement: ninl, iters, the whole inlier mask and the bits of H equal."""
    H, m, n, it = A.ransac_ac(ac, th, lth)
    k = len(ac)
    assert int(o["ninl"][p]) == n and int(o["iters"][p]) == it, (tag, int(o["ninl"][p]), n, int(o["iters"][p]), it)
    assert np.array_equal(o["inl"][p, :k].numpy(), m.astype(np.uint8)), (tag, int((o["inl"][p, :k].numpy() != m).sum()))
    assert np.array_equal(o["H"][p].numpy().view(np.int32), H.view(np.int32)), (tag, o["H"][p], H)
    if n > 0:
        assert float(o["H"][p, 2, 2]) == 1.0
    else:
        assert not o["H"][p].any(), tag
    assert bool((o["inl"][p, k:] == INL_SENTINEL).all()), (tag, "mask rows beyond ntent written")
    return n, it


@pytest.mark.parametrize("lth", ["default", math.inf])
def test_constructed_pairs_against_the_restatement(L, lth):
    lth = default_laf_th() if lth == "default" else lth
    cases = constructed_cases()
    names = list(cases)
    l1, l2, tent, ntent = build_sets(cases)
    S = len(names)
    k = names.index("n1000_40")
    # self pairs, then pairs that cannot be verified: ntent -1, ntent > tcap, image indices out of range, a row index out of range
    pl = [(s, s) for s in range(S)] + [(0, 0), (0, 0), (S, 0), (0, -1), (k, k), (k, k)]
    P = len(pl)
    t = torch.cat([tent, tent[:1].repeat(4, 1, 1), tent[k][None].repeat(2, 1, 1)]).contiguous()
    nt = torch.cat([ntent, torch.tensor([-1, CAP + 1, 4, 4, 1000, 1000], dtype=torch.int32, device=DEV)]).contiguous()
    t[S + 4, 500, 0] = CAP          # row index == cap: out of range
    t[S + 5, 999, 1] = -1
    pairs = torch.tensor(pl, dtype=torch.int32, device=DEV)
    o = run_ac(L, l1, l2, pairs, t, nt, lth=lth)
    print()
    for s, name in enumerate(names):
        a, b, Hm = cases[name]
        n, it = check_pair(o, s, A.ac_rows(a, b), name, lth)
        err = corner_error(o["H"][s].numpy(), Hm) if n > 0 and Hm is not None else float("nan")
        print("laf_th %g %-20s n=%5d: %5d inliers, %5d samples, corner error %.4f px" % (lth, name, len(a), n, it, err))
        if name in ("exact_n0", "exact_n1", "all_degenerate", "coincident", "pivot"):
            assert n == 0 and not o["H"][s].any()
        if name in ("all_degenerate", "coincident", "pivot"):
            assert it == 50000
        if name in ("exact_n2", "exact_n3", "exact_n5"):
            assert n == len(a) and err < 1e-2
        if name.startswith("n1000") or name.startswith("n3000") or name == "nan_frames":
            assert err < 1.0
    for p in range(S, P):
        assert int(o["ninl"][p]) == -1, (p, pl[p])
        assert bool((o["H"][p] == SENTINEL).all()) and bool((o["inl"][p] == INL_SENTINEL).all()) and int(o["iters"][p]) == -9, p
    # the same through the wrapper
    from affnet_b200.ReprojectionStuff import find_homography_pairs
    H, inl, ninl, iters = find_homography_pairs(l1, t, nt, l2, pairs, affine=True, laf_th=lth)
    torch.cuda.synchronize()
    assert torch.equal(ninl.cpu(), o["ninl"]) and torch.equal(iters.cpu()[:S], o["iters"][:S]) and torch.equal(H.cpu()[:S], o["H"][:S])


def test_determinism_and_independence(L):
    """Two runs give identical bits; a pair alone gives the bits it gives at a shuffled position of a list of 64."""
    cases = constructed_cases()
    l1, l2, tent, ntent = build_sets(cases, seed=3)
    S = len(cases)
    k = list(cases).index("n1000_70")
    g = torch.Generator().manual_seed(4)
    pl = torch.randint(0, S, (64,), generator=g)
    pl[17] = k
    pairs = torch.stack([pl, pl], 1).int().to(DEV)
    t, nt = tent[pl.to(DEV)].contiguous(), ntent[pl.to(DEV)].contiguous()
    a = run_ac(L, l1, l2, pairs, t, nt)
    b = run_ac(L, l1, l2, pairs, t, nt)
    for key in a:
        assert torch.equal(a[key].view(torch.uint8) if a[key].is_floating_point() else a[key],
                           b[key].view(torch.uint8) if b[key].is_floating_point() else b[key]), key
    one = run_ac(L, l1, l2, pairs[17:18].contiguous(), t[17:18].contiguous(), nt[17:18].contiguous())
    n = int(nt[17])
    assert torch.equal(one["H"][0].view(torch.int32), a["H"][17].view(torch.int32))
    assert torch.equal(one["inl"][0, :n], a["inl"][17, :n]) and one["ninl"][0] == a["ninl"][17] and one["iters"][0] == a["iters"][17]


def warped_pairs(nets):
    """The 8 warped pairs of test_gpu_verify.test_synthetic_warped_pairs (AffNet + histogram orientation, K = 2000) -> (lafs, tent,
    ntent, pairs, the true homographies, Hh, Ww)."""
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
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
    pipe.check()
    return lafs.clone(), tent, ntent, pairs, Hs, Hh, Ww


def graf_pair(nets):
    """graf img1 and img6 as in test_gpu_verify.test_graf_1_to_6 -> (lafs, tent, ntent, pairs, H1to6, the golden file, Hh, Ww)."""
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    aff, _, hn = nets
    z, f = gold("graf_match.npz"), gold("graf_full.npz")
    x1, x6 = gray_from_rgb(f["rgb"]), gray_from_rgb(z["rgb6"])
    Hh, Ww = x1.shape[2:]
    pipe = DetectDescribePipeline(2, Hh, Ww, aff, hn, None, num_features=3000, do_ori=True)
    lafs, _, desc, cnt = pipe.run(torch.cat([x1, x6]).to(DEV))
    pairs = torch.tensor([[0, 1]], device=DEV)
    tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=pairs, SNN_threshold=float(z["snn"]))
    pipe.check()
    return lafs.clone(), tent, ntent, pairs, z["H1to6"], z, Hh, Ww


def pair_rows(lafs, tent, ntent, pairs, p):
    """AC rows [n,12] float32 of pair p's tentatives."""
    n = int(ntent[p])
    i, j = (int(v) for v in pairs[p])
    t = tent[p, :n].long()
    return A.ac_rows(lafs[i, t[:, 0]].cpu().numpy(), lafs[j, t[:, 1]].cpu().numpy())


def test_synthetic_warped_pairs(L, nets):
    """The 8 warped pipeline pairs pass the 4-point test's bars (error <= 2 px at every inlier, corner error < 2 px), equal the
    restatement bit for bit, and use no more samples than the 4-point call on any pair."""
    from affnet_b200.ReprojectionStuff import find_homography_pairs
    lafs, tent, ntent, pairs, Hs, Hh, Ww = warped_pairs(nets)
    H4, inl4, ninl4, it4 = find_homography_pairs(lafs, tent, ntent, pairs=pairs)
    H, inl, ninl, iters = find_homography_pairs(lafs, tent, ntent, pairs=pairs, affine=True)
    nt, nin, it, nin4, i4 = ntent.tolist(), ninl.tolist(), iters.tolist(), ninl4.tolist(), it4.tolist()
    print()
    for k in range(8):
        He = H[k].cpu().numpy().astype(np.float64)
        err = corner_error(He, Hs[k], Hh, Ww)
        ac = pair_rows(lafs, tent, ntent, pairs, k)
        m = inl[k, :nt[k]].cpu().numpy().astype(bool)
        xy = ac[:, :2].astype(np.float64)[m]
        at_inl = float(np.linalg.norm(project(He, xy) - project(Hs[k], xy), axis=1).max())
        print("warped pair %d: %4d tentatives; 2-AC %4d inliers in %5d samples; 4-point %4d inliers in %5d samples; largest error at the "
              "inliers %.3f px (<= 2), corner error %.3f px (< 2)" % (k, nt[k], nin[k], it[k], nin4[k], i4[k], at_inl, err))
        assert at_inl <= 2.0 and err < 2.0 and it[k] <= i4[k], k
        H_r, m_r, n_r, it_r = A.ransac_ac(ac, 2.0, default_laf_th())
        assert (n_r, it_r) == (nin[k], it[k]), k
        assert np.array_equal(m, m_r) and np.array_equal(H[k].cpu().numpy().view(np.int32), H_r.view(np.int32)), k


def test_graf_1_to_6(L, nets):
    """graf 1->6 (AffNet + histogram orientation, K = 3000): the 4-point test's bar, >= 35 inliers each within 5 px of H1to6, at the
    default laf_th; the outputs equal the restatement.  graf's frames are noisy at this viewpoint change, and only 34 tentatives pass both
    the 2 px centre test and D <= 0.5 under H1to6 itself: the 2-AC hypotheses fit near their samples only, and it is the shrinking-threshold
    local optimisation (ac_local_opt) that lifts them to the model.  The counts at the other candidate thresholds are printed."""
    from affnet_b200.ReprojectionStuff import find_homography_pairs
    lafs, tent, ntent, pairs, H16, z, Hh, Ww = graf_pair(nets)
    _, _, ninl4, it4 = find_homography_pairs(lafs, tent, ntent, pairs=pairs)
    H, inl, ninl, iters = find_homography_pairs(lafs, tent, ntent, pairs=pairs, affine=True)
    n = int(ntent[0])
    He = H[0].cpu().numpy().astype(np.float64)
    ac = pair_rows(lafs, tent, ntent, pairs, 0)
    m = inl[0, :n].cpu().numpy().astype(bool)
    xy = ac[:, :2].astype(np.float64)[m]
    at_inl = float(np.linalg.norm(project(He, xy) - project(H16, xy), axis=1).max())
    print("\ngraf 1->6: %d tentatives; 2-AC %d inliers (>= 35) in %d samples, largest error at the inliers %.2f px (<= 5), corner error "
          "%.2f px; 4-point %d inliers in %d samples" % (n, int(ninl[0]), int(iters[0]), at_inl, corner_error(He, H16, Hh, Ww),
                                                         int(ninl4[0]), int(it4[0])))
    for lth in (0.5, 1.0, 2.0, 4.0, math.inf):
        Hc, ic, nc, tc = find_homography_pairs(lafs, tent, ntent, pairs=pairs, affine=True, laf_th=lth)
        xc = ac[:, :2].astype(np.float64)[ic[0, :n].cpu().numpy().astype(bool)]
        ec = float(np.linalg.norm(project(Hc[0].cpu().numpy().astype(np.float64), xc) - project(H16, xc), axis=1).max()) if len(xc) else 0.0
        print("  laf_th %g: %d inliers in %d samples, largest error at the inliers %.2f px" % (lth, int(nc[0]), int(tc[0]), ec))
    assert int(ninl[0]) >= 35 and at_inl <= 5.0
    H_r, m_r, n_r, it_r = A.ransac_ac(ac, 2.0, default_laf_th())
    assert (n_r, it_r) == (int(ninl[0]), int(iters[0])) and np.array_equal(m, m_r)


def test_one_graph_with_the_pipeline_and_matcher(L, nets):
    """pipe.run + match_snn_pairs + find_homography_pairs(affine=True) in ONE CUDA graph over all 240 ordered pairs of 16 images; a
    replay on other images equals the eager run, and the call is one launch for 1 pair and for 240."""
    import affnet_b200._lib as lib
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import find_homography_pairs
    aff, _, hn = nets
    B, Hh, Ww, K = 16, 768, 1024, 2000
    mk = lambda s: torch.cat([synthetic_image(Hh, Ww, s + i) for i in range(B)]).to(DEV)  # noqa: E731
    imgs, imgs2 = mk(1234), mk(777)
    pairs = torch.tensor([(i, j) for i in range(B) for j in range(B) if i != j], device=DEV)
    pipe = DetectDescribePipeline(B, Hh, Ww, aff, hn, None, num_features=K, do_ori=True)

    def step(x):
        lafs, _, d, c = pipe.run(x)
        tent, ntent, _, _ = match_snn_pairs(d, c, pairs=pairs)
        return (ntent,) + find_homography_pairs(lafs, tent, ntent, pairs=pairs, affine=True)

    lafs, _, d, c = pipe.run(imgs)
    tent, ntent, _, _ = match_snn_pairs(d, c, pairs=pairs)
    fn = lambda q: find_homography_pairs(lafs, tent[q], ntent[q], pairs=pairs[q], affine=True)  # noqa: E731
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
    nt, ninl = ref[0].tolist(), ref[3].tolist()
    # (ntent, H, inl, ninl, iters)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[3], ref[3]) and torch.equal(got[4], ref[4])
    for p in range(pairs.size(0)):
        n = max(nt[p], 0)
        assert torch.equal(got[2][p, :n], ref[2][p, :n]), p
        if ninl[p] >= 0:
            assert torch.equal(got[1][p], ref[1][p]), p
    print("\n240 pairs in one graph: tentatives %d..%d, affine inliers %d..%d" % (min(nt), max(nt), min(ninl), max(ninl)))
