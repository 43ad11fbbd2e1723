"""GPU tests (-m gpu) of ag_fundamental_degensac / find_fundamental_pairs(degensac=True): the constructed pairs of
test_gpu_fundamental.py and dominant-plane pairs against the numpy restatement (tests/oracle_degensac.py) bit for bit, determinism and
independence of P and of the pair's position, degensac=False keeping ag_fundamental_ransac's bits, and two-plane image pairs through
pipeline -> match_snn_pairs -> DEGENSAC in one CUDA graph.  Outputs are prefilled with sentinels."""
import numpy as np
import pytest
import torch

import degensac_cases as DC
import oracle_degensac as DG
import oracle_fransac as FR
from helpers import SENTINEL, load_weights
from test_gpu_fundamental import constructed_cases, run_fransac, two_plane_pairs
from test_gpu_verify import INL_SENTINEL, build_sets

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


def run_degensac(L, lafs1, lafs2, pairs, tent, ntent, th=TH, conf=0.99, iters=50000, seed=0):
    """ag_fundamental_degensac over sentinel-filled outputs -> dict (F, inl, ninl, iters) on the host."""
    P, tcap = tent.shape[:2]
    o = dict(F=torch.full((P, 3, 3), SENTINEL, device=DEV), inl=torch.full((P, tcap), INL_SENTINEL, dtype=torch.uint8, device=DEV),
             ninl=torch.full((P,), -9, dtype=torch.int32, device=DEV), iters=torch.full((P,), -9, dtype=torch.int32, device=DEV))
    L.check(L.lib().ag_fundamental_degensac(L.ptr(lafs1), lafs1.size(0), lafs1.size(1), L.ptr(lafs2), lafs2.size(0), lafs2.size(1),
                                            L.ptr(pairs), P, L.ptr(tent), L.ptr(ntent), tcap, th, conf, iters, seed, L.ptr(o["F"]),
                                            L.ptr(o["inl"]), L.ptr(o["ninl"]), L.ptr(o["iters"]), L.stream_ptr()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


def cases():
    """The constructed pairs of the plain RANSAC's GPU test, a tiny-inlier-ratio pair and the dominant-plane seeds 0-5."""
    c = {k: (v, TH, 50000) for k, v in constructed_cases().items()}
    rng = np.random.default_rng(1)
    n = 16384
    c["uniform"] = (np.stack([rng.uniform(0, 1024, n), rng.uniform(0, 768, n), rng.uniform(0, 1024, n), rng.uniform(0, 768, n)],
                             1).astype(np.float32), 0.25, 1024)
    for s in range(6):
        c["dominant%d" % s] = (DC.dominant_plane(s, 600)[0], TH, 50000)
    return c


def check_pair(o, p, pts, tag, th=TH, max_iters=50000):
    F, m, n, it = DG.degensac_f(pts, th, 0.99, max_iters, 0)
    k = len(pts)
    assert int(o["ninl"][p]) == n and int(o["iters"][p]) == it, (tag, int(o["ninl"][p]), n, int(o["iters"][p]), it)
    assert np.array_equal(o["inl"][p, :k].numpy(), m.astype(np.uint8)), (tag, int((o["inl"][p, :k].numpy() != m).sum()))
    assert np.array_equal(o["F"][p].numpy().view(np.int32), F.view(np.int32)), (tag, o["F"][p], F)
    if n == 0:
        assert not o["F"][p].any(), tag
    assert bool((o["inl"][p, k:] == INL_SENTINEL).all()), (tag, "mask rows beyond ntent written")
    return n, it, m


def test_constructed_pairs_against_the_restatement(L):
    """Every case, one launch per (inl_th, max_iters) group, bit for bit; pairs that cannot be verified get -1 and nothing else."""
    cs = cases()
    print()
    for key in sorted({(th, it) for _, th, it in cs.values()}):
        names = [k for k, v in cs.items() if (v[1], v[2]) == key]
        l1, l2, tent, ntent = build_sets({k: (cs[k][0], None) for k in names})
        S = len(names)
        pl = [(s, s) for s in range(S)] + [(S, 0)]
        t = torch.cat([tent, tent[:1]]).contiguous()
        nt = torch.cat([ntent, ntent[:1]]).contiguous()
        o = run_degensac(L, l1, l2, torch.tensor(pl, dtype=torch.int32, device=DEV), t, nt, th=key[0], iters=key[1])
        for s, name in enumerate(names):
            pts = cs[name][0]
            n, it, m = check_pair(o, s, pts, name, th=key[0], max_iters=key[1])
            extra = ""
            if name.startswith("dominant"):
                _, out, _, offp = DC.dominant_plane(int(name[-1]), 600)
                frac = float(m[~out & offp].mean())
                extra = ", %.3f of the off-plane matches" % frac
                assert frac >= 0.8, name
            print("%-16s n=%5d: %5d inliers, %5d samples%s" % (name, len(pts), n, it, extra))
        assert int(o["ninl"][S]) == -1 and bool((o["F"][S] == SENTINEL).all()) and int(o["iters"][S]) == -9


def test_determinism_and_independence(L):
    """Two runs give identical bits; a pair alone gives the bits it gives at position 17 of a shuffled list of 64."""
    cs = {k: v[0] for k, v in cases().items() if v[1] == TH}
    l1, l2, tent, ntent = build_sets({k: (v, None) for k, v in cs.items()}, seed=3)
    S = len(cs)
    k = list(cs).index("dominant3")
    g = torch.Generator().manual_seed(4)
    pl = torch.randint(0, S, (64,), generator=g)
    pl[17] = k
    pairs = torch.stack([pl, pl], 1).int().to(DEV)
    t, nt = tent[pl.to(DEV)].contiguous(), ntent[pl.to(DEV)].contiguous()
    a = run_degensac(L, l1, l2, pairs, t, nt)
    b = run_degensac(L, l1, l2, pairs, t, nt)
    for key in a:
        assert torch.equal(a[key].view(torch.uint8) if a[key].is_floating_point() else a[key],
                           b[key].view(torch.uint8) if b[key].is_floating_point() else b[key]), key
    one = run_degensac(L, l1, l2, pairs[17:18].contiguous(), t[17:18].contiguous(), nt[17:18].contiguous())
    n = int(nt[17])
    assert torch.equal(one["F"][0].view(torch.int32), a["F"][17].view(torch.int32))
    assert torch.equal(one["inl"][0, :n], a["inl"][17, :n]) and one["ninl"][0] == a["ninl"][17] and one["iters"][0] == a["iters"][17]


def test_degensac_false_keeps_the_plain_bits(L):
    """find_fundamental_pairs(degensac=False) and the default give ag_fundamental_ransac's bits; degensac=True those of the new entry."""
    from affnet_b200.ReprojectionStuff import find_fundamental_pairs
    cs = {k: v[0] for k, v in cases().items() if v[1] == TH}
    l1, l2, tent, ntent = build_sets({k: (v, None) for k, v in cs.items()})
    pairs = torch.tensor([(s, s) for s in range(len(cs))], dtype=torch.int32, device=DEV)
    plain = run_fransac(L, l1, l2, pairs, tent, ntent)
    deg = run_degensac(L, l1, l2, pairs, tent, ntent)
    for flag, ref in ((None, plain), (False, plain), (True, deg)):
        kw = {} if flag is None else dict(degensac=flag)
        F, inl, ninl, iters = find_fundamental_pairs(l1, tent, ntent, l2, pairs, **kw)
        torch.cuda.synchronize()
        assert torch.equal(ninl.cpu(), ref["ninl"]) and torch.equal(iters.cpu(), ref["iters"]), flag
        assert torch.equal(F.cpu().view(torch.int32), ref["F"].view(torch.int32)), flag
        for p, n in enumerate(ntent.tolist()):
            assert torch.equal(inl.cpu()[p, :n], ref["inl"][p, :n]), (flag, p)


def test_two_plane_scenes_in_one_graph(L, nets):
    """The 8 two-plane pairs of test_gpu_fundamental.py: pipeline (B = 16, AffNet, HardNet, K = 2000) + match_snn_pairs +
    find_fundamental_pairs(degensac=True) captured in ONE CUDA graph and replayed; the replay equals the eager call and the restatement
    bit for bit, keeps >= 99 % of the plain call's inliers, and >= 95 % of its inliers lie within 1 px (Sampson) of the true F.  (Not
    always all of them: the local optimisation moves the search to another model and stopping point, and on pair 1 DEGENSAC ends with
    1095 inliers where the plain call has 1097, all of both within 1 px of the true F.)"""
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import find_fundamental_pairs
    aff, hn = nets
    Hh, Ww, K = 768, 1024, 2000
    imgs, Fs = two_plane_pairs(Hh, Ww)
    imgs = imgs.to(DEV)
    pairs = torch.tensor([(2 * k, 2 * k + 1) for k in range(8)], device=DEV)
    pipe = DetectDescribePipeline(16, Hh, Ww, aff, hn, None, num_features=K, do_ori=True)

    def step(x):
        lafs, _, d, c = pipe.run(x)
        tent, ntent, _, _ = match_snn_pairs(d, c, pairs=pairs)
        return (lafs, tent, ntent) + find_fundamental_pairs(lafs, tent, ntent, pairs=pairs, degensac=True)

    static_in = torch.zeros_like(imgs)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step(static_in)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = step(static_in)
    static_in.copy_(imgs)
    g.replay()
    torch.cuda.synchronize()
    lafs, tent, ntent, F, inl, ninl, iters = [t.clone() for t in res]
    pipe.check()
    ref = step(imgs)
    _, _, nplain, _ = find_fundamental_pairs(lafs, tent, ntent, pairs=pairs)
    torch.cuda.synchronize()
    assert torch.equal(ref[5], ninl) and torch.equal(ref[6], iters) and torch.equal(ref[3].view(torch.int32), F.view(torch.int32))
    nt, nf, npl, it = ntent.tolist(), ninl.tolist(), nplain.tolist(), iters.tolist()
    print()
    for k in range(8):
        t = tent[k, :nt[k]].long()
        pts = torch.cat([lafs[2 * k, t[:, 0], :, 2], lafs[2 * k + 1, t[:, 1], :, 2]], 1).cpu().numpy()
        m = inl[k, :nt[k]].cpu().numpy().astype(bool)
        d = FR.sampson(Fs[k], pts[m])
        close = float((d <= 2 * TH).mean()) if m.any() else 0.0
        print("two-plane pair %d: %4d tentatives, DEGENSAC %4d inliers in %5d samples (%.3f within %.1f px of the true F), plain %4d"
              % (k, nt[k], nf[k], it[k], close, 2 * TH, npl[k]))
        assert nt[k] > 100 and close >= 0.95 and nf[k] >= 0.99 * npl[k], k
        F_r, m_r, n_r, it_r = DG.degensac_f(pts)
        assert (n_r, it_r) == (nf[k], it[k]) and np.array_equal(m.astype(np.uint8), m_r.astype(np.uint8)), k
        assert np.array_equal(F[k].cpu().numpy().view(np.int32), F_r.view(np.int32)), k
