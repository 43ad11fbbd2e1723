"""GPU tests (-m gpu) of ag_fundamental_ransac / find_fundamental_pairs: constructed pairs against the numpy restatement
(tests/oracle_fransac.py) bit for bit, determinism and independence of the pair's position, two-plane scenes through the whole chain
(pipeline -> match_snn_pairs -> fundamental and homography RANSAC), and one CUDA graph with the pipeline and the matcher.  Outputs are
prefilled with sentinels, so rows and pairs that must not be written are checked too."""
import numpy as np
import pytest
import torch

import fundamental_cases as FC
import oracle_fransac as FR
import oracle_ransac as R
from helpers import SENTINEL, load_weights, synthetic_image
from test_gpu_verify import CAP, INL_SENTINEL, build_sets, warp

pytestmark = pytest.mark.gpu

DEV = "cuda"
TH = 0.5


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


@pytest.fixture(scope="module")
def nets():
    from affnet_b200.architectures import AffNetFast
    from affnet_b200.HardNet import HardNet
    W = load_weights()
    a, h = AffNetFast(PS=32), HardNet()
    a.load_state_dict(W["affnet"]); h.load_state_dict(W["hardnet"])
    return a.eval().to(DEV), h.eval().to(DEV)


def run_fransac(L, lafs1, lafs2, pairs, tent, ntent, th=TH, conf=0.99, iters=50000, seed=0):
    """ag_fundamental_ransac over sentinel-filled outputs -> dict (F, inl, ninl, iters) on the host."""
    P, tcap = tent.shape[:2]
    o = dict(F=torch.full((P, 3, 3), SENTINEL, device=DEV), inl=torch.full((P, tcap), INL_SENTINEL, dtype=torch.uint8, device=DEV),
             ninl=torch.full((P,), -9, dtype=torch.int32, device=DEV), iters=torch.full((P,), -9, dtype=torch.int32, device=DEV))
    L.check(L.lib().ag_fundamental_ransac(L.ptr(lafs1), lafs1.size(0), lafs1.size(1), L.ptr(lafs2), lafs2.size(0), lafs2.size(1), L.ptr(pairs),
                                          P, L.ptr(tent), L.ptr(ntent), tcap, th, conf, iters, seed, L.ptr(o["F"]), L.ptr(o["inl"]),
                                          L.ptr(o["ninl"]), L.ptr(o["iters"]), L.stream_ptr()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


def constructed_cases():
    """name -> pts [n,4] float32.  Image s of both LAF sets holds case s."""
    cases = {}
    for n in (0, 6, 7, 8, 1000, 16384):
        pts, _, _ = FC.scene(200 + n, n, outliers=0.0 if n <= 8 else 0.4, sigma=0.0 if n <= 8 else 0.3)
        cases["n%d" % n] = pts
    x = np.arange(50, dtype=np.float32) * 7.0
    cases["collinear"] = np.stack([x, 2 * x + 3, x + 1, np.full_like(x, 9.0)], 1)
    cases["duplicated"] = np.tile(np.array([[100.0, 200.0, 110.0, 190.0]], np.float32), (30, 1))
    pts, _, _ = FC.scene(9, 300)
    pts[::3] = pts[0]
    cases["some_duplicated"] = pts
    cases["planar"], _, _ = FC.plane_scene(11, 500)
    pts, _, _ = FC.scene(13, 400)
    pts[::17, 0] = np.nan
    pts[5::23, 3] = np.nan
    cases["nan_centres"] = pts
    return cases


def check_pair(o, p, pts, tag, th=TH, max_iters=50000):
    """Pair p of the GPU outputs against the restatement: ninl, iters, the whole inlier mask and the bits of F equal."""
    F, m, n, it = FR.ransac_f(pts, th, 0.99, max_iters, 0)
    k = len(pts)
    assert int(o["ninl"][p]) == n and int(o["iters"][p]) == it, (tag, int(o["ninl"][p]), n, int(o["iters"][p]), it)
    assert np.array_equal(o["inl"][p, :k].numpy(), m.astype(np.uint8)), (tag, int((o["inl"][p, :k].numpy() != m).sum()))
    assert np.array_equal(o["F"][p].numpy().view(np.int32), F.view(np.int32)), (tag, o["F"][p], F)
    if n > 0:
        assert abs(float(o["F"][p].norm()) - 1.0) < 1e-6
    else:
        assert not o["F"][p].any(), tag
    assert bool((o["inl"][p, k:] == INL_SENTINEL).all()), (tag, "mask rows beyond ntent written")
    return n, it


def test_constructed_pairs_against_the_restatement(L):
    cases = constructed_cases()
    names = list(cases)
    l1, l2, tent, ntent = build_sets({k: (v, None) for k, v in cases.items()})
    S = len(names)
    k1000 = names.index("n1000")
    # self pairs, then pairs that cannot be verified: ntent -1, ntent > tcap, image indices out of range, a row index out of range
    pl = [(s, s) for s in range(S)] + [(0, 0), (0, 0), (S, 0), (0, -1), (k1000, k1000), (k1000, k1000)]
    P = len(pl)
    t = torch.cat([tent, tent[:1].repeat(4, 1, 1), tent[k1000][None].repeat(2, 1, 1)]).contiguous()
    nt = torch.cat([ntent, torch.tensor([-1, CAP + 1, 4, 4, 1000, 1000], dtype=torch.int32, device=DEV)]).contiguous()
    t[S + 4, 500, 0] = CAP
    t[S + 5, 999, 1] = -1
    pairs = torch.tensor(pl, dtype=torch.int32, device=DEV)
    o = run_fransac(L, l1, l2, pairs, t, nt)
    print()
    for s, name in enumerate(names):
        pts = cases[name]
        n, it = check_pair(o, s, pts, name)
        print("%-16s n=%5d: %5d inliers, %5d samples" % (name, len(pts), n, it))
        if name in ("n0", "n6", "collinear", "duplicated"):
            assert n == 0 and not o["F"][s].any()
        if name == "collinear":
            assert it == 50000
        if name in ("n7", "n8"):
            assert n == len(pts)
        if name == "nan_centres":
            assert not o["inl"][s, :len(pts)][torch.from_numpy(~np.isfinite(pts).all(1))].any()
    for p in range(S, P):
        assert int(o["ninl"][p]) == -1, (p, pl[p])
        assert bool((o["F"][p] == SENTINEL).all()) and bool((o["inl"][p] == INL_SENTINEL).all()) and int(o["iters"][p]) == -9, p
    from affnet_b200.ReprojectionStuff import find_fundamental_pairs
    F, inl, ninl, iters = find_fundamental_pairs(l1, t, nt, l2, pairs)
    torch.cuda.synchronize()
    assert torch.equal(ninl.cpu(), o["ninl"]) and torch.equal(iters.cpu()[:S], o["iters"][:S]) and torch.equal(F.cpu()[:S], o["F"][:S])


def test_determinism_and_independence(L):
    """Two runs give identical bits; a pair alone gives the bits it gives at position 17 of a shuffled list of 64."""
    cases = constructed_cases()
    l1, l2, tent, ntent = build_sets({k: (v, None) for k, v in cases.items()}, seed=3)
    S = len(cases)
    k = list(cases).index("n1000")
    g = torch.Generator().manual_seed(4)
    pl = torch.randint(0, S, (64,), generator=g)
    pl[17] = k
    pairs = torch.stack([pl, pl], 1).int().to(DEV)
    t, nt = tent[pl.to(DEV)].contiguous(), ntent[pl.to(DEV)].contiguous()
    a = run_fransac(L, l1, l2, pairs, t, nt)
    b = run_fransac(L, l1, l2, pairs, t, nt)
    for key in a:
        assert torch.equal(a[key].view(torch.uint8) if a[key].is_floating_point() else a[key],
                           b[key].view(torch.uint8) if b[key].is_floating_point() else b[key]), key
    one = run_fransac(L, l1, l2, pairs[17:18].contiguous(), t[17:18].contiguous(), nt[17:18].contiguous())
    n = int(nt[17])
    assert torch.equal(one["F"][0].view(torch.int32), a["F"][17].view(torch.int32))
    assert torch.equal(one["inl"][0, :n], a["inl"][17, :n]) and one["ninl"][0] == a["ninl"][17] and one["iters"][0] == a["iters"][17]


def test_tiny_inlier_ratio_runs_to_max_iters(L):
    """16384 uniform random correspondences at inl_th = 0.25: 1 - (best/n)^7 rounds to 1, so no sample count reaches the confidence and
    the search runs to max_iters (1024 here), bit for bit as the restatement.  (At 0.5 the final ratio, 80 / 16384, is just above the
    rounding threshold.)"""
    rng = np.random.default_rng(1)
    n = 16384
    pts = np.stack([rng.uniform(0, 1024, n), rng.uniform(0, 768, n), rng.uniform(0, 1024, n), rng.uniform(0, 768, n)], 1).astype(np.float32)
    l1, l2, tent, ntent = build_sets({"uniform": (pts, None)})
    o = run_fransac(L, l1, l2, None, tent, ntent, th=0.25, iters=1024)
    k, it = check_pair(o, 0, pts, "uniform", th=0.25, max_iters=1024)
    pr = k / n
    assert k > 0 and it == 1024 and 1.0 - pr * pr * pr * pr * pr * pr * pr == 1.0, (k, it)


def two_plane_pairs(Hh, Ww, k_pairs=8):
    """k seeded image pairs: image 2 is image 1 warped by the homographies that one camera motion induces for two fronto-parallel
    planes (depths 3 and 6), its left half by the first and its right half by the second -> (images [2k,1,H,W], true F per pair)."""
    imgs, Fs = [], []
    for k in range(k_pairs):
        rng = np.random.default_rng(700 + k)
        K = FC.intrinsics(800.0, Hh, Ww)
        R = FC.rotation(rng, 3.0)
        t = np.array([rng.choice([-1, 1]) * rng.uniform(0.25, 0.35), rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05)])
        Ha, Hb = (FC.plane_homography(K, R, t, np.array([0.0, 0.0, 1.0]), d) for d in (3.0, 6.0))   # the planes z = 3 and z = 6
        x = synthetic_image(Hh, Ww, 950 + k)
        wa, wb = warp(x, Ha / Ha[2, 2]), warp(x, Hb / Hb[2, 2])
        y = torch.cat([wa[..., :Ww // 2], wb[..., Ww // 2:]], 3)
        imgs += [x, y]
        Fs.append(FC.true_f(K, R, t))
    return torch.cat(imgs), Fs


def test_two_plane_scenes_through_the_chain(L, nets):
    """8 seeded two-plane pairs as one B = 16 pipeline batch (AffNet, HardNet, K = 2000), match_snn_pairs, then find_fundamental_pairs
    and find_homography_pairs on the same tentatives: >= 95 % of the F-inliers lie within 2 inl_th (Sampson) of the true F, F keeps
    >= 1.3 x the homography's inliers, and both equal their restatements bit for bit."""
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import find_fundamental_pairs, find_homography_pairs
    aff, hn = nets
    Hh, Ww, K = 768, 1024, 2000
    imgs, Fs = two_plane_pairs(Hh, Ww)
    pipe = DetectDescribePipeline(16, Hh, Ww, aff, hn, None, num_features=K, do_ori=True)
    lafs, _, desc, cnt = pipe.run(imgs.to(DEV))
    pairs = torch.tensor([(2 * k, 2 * k + 1) for k in range(8)], device=DEV)
    tent, ntent, _, _ = match_snn_pairs(desc, cnt, pairs=pairs)
    F, inl, ninl, iters = find_fundamental_pairs(lafs, tent, ntent, pairs=pairs)
    H, hinl, hninl, hiters = find_homography_pairs(lafs, tent, ntent, pairs=pairs)
    pipe.check()
    nt, nf, nh, it = ntent.tolist(), ninl.tolist(), hninl.tolist(), iters.tolist()
    print()
    for k in range(8):
        t = tent[k, :nt[k]].long()
        pts = torch.cat([lafs[2 * k, t[:, 0], :, 2], lafs[2 * k + 1, t[:, 1], :, 2]], 1).cpu().numpy()
        m = inl[k, :nt[k]].cpu().numpy().astype(bool)
        d = FR.sampson(Fs[k], pts[m])
        close = float((d <= 2 * TH).mean()) if m.any() else 0.0
        print("two-plane pair %d: %4d tentatives, F %4d inliers in %5d samples (%.3f within %.1f px of the true F), homography %4d inliers"
              % (k, nt[k], nf[k], it[k], close, 2 * TH, nh[k]))
        assert nt[k] > 100 and close >= 0.95 and nf[k] >= 1.3 * nh[k], k
        F_r, m_r, n_r, it_r = FR.ransac_f(pts)
        assert (n_r, it_r) == (nf[k], it[k]), k
        assert np.array_equal(m.astype(np.uint8), m_r.astype(np.uint8)), k
        assert np.array_equal(F[k].cpu().numpy().view(np.int32), F_r.view(np.int32)), k
        H_r, hm_r, hn_r, hit_r = R.ransac(pts)
        assert (hn_r, hit_r) == (nh[k], int(hiters[k])) and np.array_equal(H[k].cpu().numpy().view(np.int32), H_r.view(np.int32)), k


def test_one_graph_with_the_pipeline_and_matcher(L, nets):
    """pipe.run + match_snn_pairs + find_fundamental_pairs in ONE CUDA graph over all 240 ordered pairs of 16 images; a replay on other
    images equals the eager run, and the call is one launch for 1 pair and for 240."""
    import affnet_b200._lib as lib
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import find_fundamental_pairs
    aff, hn = nets
    B, Hh, Ww, K = 16, 768, 1024, 2000
    mk = lambda s: torch.cat([synthetic_image(Hh, Ww, s + i) for i in range(B)]).to(DEV)  # noqa: E731
    imgs, imgs2 = mk(1234), mk(777)
    pairs = torch.tensor([(i, j) for i in range(B) for j in range(B) if i != j], device=DEV)
    pipe = DetectDescribePipeline(B, Hh, Ww, aff, hn, None, num_features=K, do_ori=True)

    def step(x):
        lafs, _, d, c = pipe.run(x)
        tent, ntent, _, _ = match_snn_pairs(d, c, pairs=pairs)
        return (ntent,) + find_fundamental_pairs(lafs, tent, ntent, pairs=pairs)

    lafs, _, d, c = pipe.run(imgs)
    tent, ntent, _, _ = match_snn_pairs(d, c, pairs=pairs)
    fn = lambda q: find_fundamental_pairs(lafs, tent[q], ntent[q], pairs=pairs[q])  # noqa: E731
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
    # (ntent, F, inl, ninl, iters)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[3], ref[3]) and torch.equal(got[4], ref[4])
    for p in range(pairs.size(0)):
        n = max(nt[p], 0)
        assert torch.equal(got[2][p, :n], ref[2][p, :n]), p
        if ninl[p] >= 0:
            assert torch.equal(got[1][p], ref[1][p]), p
    print("\n240 pairs in one graph: tentatives %d..%d, F inliers %d..%d" % (min(nt), max(nt), min(ninl), max(ninl)))
