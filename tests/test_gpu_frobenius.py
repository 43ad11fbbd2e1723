"""GPU tests of the Frobenius ground truth (ag_gt_frobenius_pairs / _sets, ag_reproject_lafs): bit for bit against the restatement
(tests/frobenius_restated.py) on every flag combination in both modes, with ragged, empty and out-of-range counts, out-of-range
tentative rows, ties, NaN and singular frames; the golden graf cases with the agreement rule of the CPU tests; pair independence; one
16384 x 16384 pair; the drop-ins; and the whole chain captured in one CUDA graph."""
import numpy as np
import pytest
import torch

import frobenius_restated as FR
import test_frobenius_cpu as CPU
from helpers import gold, load_weights, synthetic_image

pytestmark = pytest.mark.gpu

DEV = "cuda"
CASES = dict(CPU.CASES, fc_noscale=dict(center_dist_th=2.0, scale_diff_coef=0.0), fro_up_noinv=dict(do_up_is_up=True, inv_to_eye=False),
             fc_tight=dict(dist_threshold=0.05, center_dist_th=0.5, scale_diff_coef=0.05))


def prm_of(kw):
    kw = dict(kw)
    return FR.Params(kw.pop("dist_threshold", 4.0), **kw), kw


def random_homography(g):
    H = np.eye(3) + g.normal(0, [[0.05, 0.05, 5.0], [0.05, 0.05, 5.0], [2e-4, 2e-4, 0]])
    return H.astype(np.float32)


def random_lafs(g, n):
    s = np.exp(g.uniform(0.5, 3.0, n))
    ang, sk = g.uniform(0, 2 * np.pi, n), g.uniform(-0.5, 0.5, n)
    c, si = np.cos(ang), np.sin(ang)
    a = np.stack([np.stack([s * c, s * (sk * c - si)], 1), np.stack([s * si, s * (sk * si + c)], 1)], 1)
    t = g.uniform(0, 300, (n, 2, 1))
    return np.concatenate([a, t], 2).astype(np.float32)


def side2_of(g, l1, H):
    """Side 2: side 1 mapped into image 2 (so its frames come back close to side 1's), jittered and permuted."""
    l2 = FR.reproject_lafs(l1, H, False, False)
    l2 = l2 + g.normal(0, 1, l2.shape).astype(np.float32) * np.array([[0.05, 0.05, 0.7], [0.05, 0.05, 0.7]], np.float32) * np.abs(l2).clip(1, 3)
    return l2[g.permutation(len(l2))].astype(np.float32)


def special_rows(l1, l2):
    """NaN and singular side-1 frames, a NaN and an infinite side-2 frame, and two identical side-2 frames (a tie)."""
    l1[3, 0, 1] = np.nan
    l1[4, :, :2] = [[1.0, 2.0], [2.0, 4.0]]
    l1[5, 1, 2] = np.inf
    l2[2, 1, 0] = np.nan
    l2[5, 0, 2] = np.inf
    l2[7] = l2[6]


def batch(seed, S=5, cap=300):
    g = np.random.default_rng(seed)
    Hs = np.stack([random_homography(g) for _ in range(S)])
    l1 = np.stack([random_lafs(g, cap) for _ in range(S)])
    l2 = np.stack([side2_of(g, l1[s], Hs[s]) for s in range(S)])
    for s in range(S):
        special_rows(l1[s], l2[s])
    return l1, l2, Hs


def same_bits(a, b):
    """Equal bit for bit, any NaN equal to any NaN (the device's and numpy's NaN payloads differ)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(((a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))).all())


def check_pair(mn, idx, true, ntrue, want):
    wm, wi, wt = want
    n = len(wm)
    assert np.array_equal(mn[:n].view(np.int32), wm.view(np.int32))
    assert np.array_equal(idx[:n], wi)
    assert ntrue == len(wt) and np.array_equal(true[:ntrue], wt)


@pytest.mark.parametrize("case", list(CASES))
def test_sets_equal_the_restatement(case):
    from affnet_b200.ReprojectionStuff import frobenius_gt_sets
    prm, kw = prm_of(CASES[case])
    l1, l2, Hs = batch(11)
    S, cap = l1.shape[:2]
    count1 = np.array([300, 217, 0, 1, 299], np.int32)
    count2 = np.array([256, 300, 40, -1, 301], np.int32)
    pairs = np.array([(0, 0), (1, 1), (2, 2), (3, 1), (0, 3), (4, 0), (1, 4), (0, 2), (5, 0), (1, -1), (4, 1)], np.int32)
    Hp = np.stack([Hs[min(max(j, 0), S - 1)] for _, j in pairs])
    out = frobenius_gt_sets(torch.from_numpy(l1).to(DEV), torch.from_numpy(count1).to(DEV), torch.from_numpy(Hp).to(DEV),
                            torch.from_numpy(l2).to(DEV), torch.from_numpy(count2).to(DEV), torch.from_numpy(pairs).to(DEV),
                            dist_threshold=float(prm.th), **kw)
    true, ntrue, mn, idx = (t.cpu().numpy() for t in out)
    for p, (i, j) in enumerate(pairs.tolist()):
        if not (0 <= i < S and 0 <= j < S and 0 <= count1[i] <= cap and 0 <= count2[j] <= cap):
            assert ntrue[p] == -1, p
            continue
        want = FR.frobenius(l1[i, :count1[i]], l2[j, :count2[j]], Hp[p], prm)
        check_pair(mn[p], idx[p], true[p], ntrue[p], want)
    if case != "fc_tight":
        assert (ntrue[[0, 1]] > 0).all()


@pytest.mark.parametrize("case", list(CASES))
def test_pairs_equal_the_restatement(case):
    from affnet_b200.ReprojectionStuff import frobenius_gt_pairs
    prm, kw = prm_of(CASES[case])
    l1, l2, Hs = batch(12, S=4, cap=200)
    g = np.random.default_rng(5)
    P, tcap = 7, 180
    pairs = np.array([(0, 0), (1, 1), (2, 2), (3, 3), (0, 1), (1, 0), (2, 3)], np.int32)
    ntent = np.array([180, 97, 0, -1, 181, 120, 60], np.int32)
    tent = np.full((P, tcap, 2), 10 ** 6, np.int32)                     # rows at or beyond ntent: never read
    for p in range(P):
        n = min(max(ntent[p], 0), tcap)
        tent[p, :n, 0] = g.integers(0, 200, n)
        tent[p, :n, 1] = g.integers(0, 200, n)
        tent[p, :min(n, 10), 1] = np.arange(min(n, 10))                  # the special side-2 frames 0..9
    tent[0, 1, 1] = tent[0, 2, 1]                                       # a repeated column: a tie
    tent[5, 7, 0] = 200                                                 # out of range: pair 5 cannot be checked
    Hp = Hs[pairs[:, 1]]
    out = frobenius_gt_pairs(torch.from_numpy(l1).to(DEV), torch.from_numpy(tent).to(DEV), torch.from_numpy(ntent).to(DEV),
                             torch.from_numpy(Hp).to(DEV), torch.from_numpy(l2).to(DEV), torch.from_numpy(pairs).to(DEV),
                             dist_threshold=float(prm.th), **kw)
    true, ntrue, mn, idx = (t.cpu().numpy() for t in out)
    for p, (i, j) in enumerate(pairs.tolist()):
        if p in (3, 4, 5):
            assert ntrue[p] == -1, p
            continue
        want = FR.frobenius_tent(l1[i], l2[j], tent[p, :ntent[p]], Hp[p], prm)
        check_pair(mn[p], idx[p], true[p], ntrue[p], want)


def test_a_pair_alone_equals_its_result_in_the_batch():
    from affnet_b200.ReprojectionStuff import frobenius_gt_sets
    l1, l2, Hs = batch(13)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    c1, c2 = d(np.array([300, 250, 120, 7, 1], np.int32)), d(np.array([280, 300, 1, 77, 300], np.int32))
    pairs = np.array([(i, j) for i in range(5) for j in range(5)], np.int32)
    Hp = Hs[pairs[:, 1]]
    kw = dict(center_dist_th=2.0)
    allp = frobenius_gt_sets(d(l1), c1, d(Hp), d(l2), c2, d(pairs), **kw)
    nt = allp[1].tolist()
    for p in range(len(pairs)):
        one = frobenius_gt_sets(d(l1), c1, d(Hp[p:p + 1]), d(l2), c2, d(pairs[p:p + 1]), **kw)
        n1 = int(c1[pairs[p, 0]])
        assert one[1].item() == nt[p]
        assert torch.equal(one[0][0, :nt[p]], allp[0][p, :nt[p]])
        assert torch.equal(one[2][0, :n1], allp[2][p, :n1]) and torch.equal(one[3][0, :n1], allp[3][p, :n1])


@pytest.mark.parametrize("mode", ["set", "tent"])
@pytest.mark.parametrize("case", list(CPU.CASES))
def test_graf_golden(mode, case):
    """The reference detector's graf 1 -> 6 LAFs: the device equals the restatement bit for bit, and so agrees with the reference's
    outputs by the CPU tests' rule (the same rows differ, each within rounding of a decision)."""
    from affnet_b200.ReprojectionStuff import frobenius_gt_pairs, frobenius_gt_sets
    z, m = gold("frobenius.npz"), gold("graf_match.npz")
    prm, kw = prm_of(CASES[case])
    H = torch.from_numpy(z["H1to6"]).to(DEV)
    if mode == "set":
        l1, l2 = torch.from_numpy(z["lafs1"]).to(DEV)[None], torch.from_numpy(z["lafs6"]).to(DEV)[None]
        c1 = torch.tensor([l1.size(1)], dtype=torch.int32, device=DEV)
        c2 = torch.tensor([l2.size(1)], dtype=torch.int32, device=DEV)
        out = frobenius_gt_sets(l1, c1, H, l2, c2, **kw)
        want = FR.frobenius(z["lafs1"], z["lafs6"], z["H1to6"], prm)
    else:
        tent = torch.from_numpy(np.stack([m["noori_t1"], m["noori_t2"]], 1)).to(DEV)[None]
        ntent = torch.tensor([tent.size(1)], dtype=torch.int32, device=DEV)
        out = frobenius_gt_pairs(torch.from_numpy(z["lafs1"]).to(DEV)[None], tent, ntent, H, torch.from_numpy(z["lafs6"]).to(DEV)[None], **kw)
        want = FR.frobenius_tent(z["lafs1"], z["lafs6"], tent[0].cpu().numpy(), z["H1to6"], prm)
    true, ntrue, mn, idx = (t.cpu().numpy() for t in out)
    check_pair(mn[0], idx[0], true[0], ntrue[0], want)
    l1n, l2n, Hn = CPU.graf_case(mode)
    differ, missing = CPU.agreement(l1n, l2n, Hn, CASES[case], z["%s_%s_min" % (mode, case)], z["%s_%s_i1" % (mode, case)],
                                    z["%s_%s_i2" % (mode, case)])
    assert differ == CPU.EXEMPT.get((mode, case), set()) and missing == []
    print("\ngraf 1->6 %s %s: %d of %d rows true at 4" % (mode, case, int(ntrue[0]), len(want[0])))


def test_one_large_pair_on_sampled_rows():
    from affnet_b200.ReprojectionStuff import frobenius_gt_sets
    g = np.random.default_rng(21)
    n = 16384
    H = random_homography(g)
    l1 = random_lafs(g, n)
    l1[:, :, 2] *= 10.0
    l2 = side2_of(g, l1, H)
    c = torch.tensor([n], dtype=torch.int32, device=DEV)
    for kw in ({}, dict(center_dist_th=2.0)):
        prm, _ = prm_of(kw)
        true, ntrue, mn, idx = frobenius_gt_sets(torch.from_numpy(l1).to(DEV)[None], c, torch.from_numpy(H).to(DEV),
                                                 torch.from_numpy(l2).to(DEV)[None], c, **kw)
        rows = np.sort(np.concatenate([g.choice(n, 60, replace=False), [0, n - 1]]))
        r, cl = FR.rows(l1[rows], prm), FR.cols(l2, H, prm)
        wm, wi, _ = FR.reduce_rows(FR.distances(r, cl, prm), np.inf)
        gm, gi = mn[0].cpu().numpy()[rows], idx[0].cpu().numpy()[rows]
        assert np.array_equal(gm.view(np.int32), wm.view(np.int32)) and np.array_equal(gi, wi)
        tr = set(true[0, :int(ntrue[0])].tolist())
        assert {int(x) for x in rows[wm <= prm.th]} == tr & set(rows.tolist())
        assert len(tr) > 0


def test_drop_ins_equal_the_batched_calls():
    import affnet_b200.ReprojectionStuff as RS
    l1, l2, Hs = batch(14, S=1, cap=250)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    L1, L2, H = d(l1[0]), d(l2[0, :230]), d(Hs[0])
    c1, c2 = torch.tensor([250], dtype=torch.int32, device=DEV), torch.tensor([230], dtype=torch.int32, device=DEV)
    for name, kw, bkw in [("get_GT_correspondence_indexes_Fro", {}, {}),
                          ("get_GT_correspondence_indexes_Fro", dict(skip_center_in_Fro=True), dict(skip_center=True)),
                          ("get_GT_correspondence_indexes_Fro_and_center", {}, dict(center_dist_th=2.0)),
                          ("get_GT_correspondence_indexes_Fro_and_center", dict(do_up_is_up=True, inv_to_eye=False, return_LAF2_in_1=True),
                           dict(center_dist_th=2.0, do_up_is_up=True, inv_to_eye=False))]:
        got = getattr(RS, name)(L1, L2, H, **kw)
        true, ntrue, mn, idx = RS.frobenius_gt_sets(L1[None], c1, H, L2[None], c2, **bkw)
        keep = true[0, :int(ntrue[0])].long()
        assert torch.equal(got[1], keep) and torch.equal(got[0], mn[0][keep]) and torch.equal(got[2], idx[0][keep].long())
        if kw.get("return_LAF2_in_1"):
            want = FR.reproject_lafs(l2[0, :230], Hs[0], True, True)
            assert same_bits(got[3].cpu().numpy(), want)
    got = RS.reprojectLAFs(L1, H)
    assert same_bits(got.cpu().numpy(), FR.reproject_lafs(l1[0], Hs[0], False, False))
    lhf = RS.reprojectLAFs(L1, H, return_LHFs=True)
    assert lhf.shape == (250, 3, 3) and same_bits(lhf[:, :2].cpu().numpy(), got.cpu().numpy())
    assert torch.equal(lhf[:, 2], torch.tensor([0.0, 0.0, 1.0], device=DEV).expand(250, 3))
    e = RS.get_GT_correspondence_indexes_Fro(L1[:0], L2, H)
    assert all(t.numel() == 0 for t in e)


def test_one_graph_with_the_pipeline_and_matcher():
    """pipe.run + match_snn_pairs + frobenius_gt_pairs + frobenius_gt_sets in ONE CUDA graph over the 12 ordered pairs of 4 images; a
    replay on other images equals the eager run, and each Frobenius call is two launches for 1 pair and for 12."""
    import affnet_b200._lib as lib
    from affnet_b200.architectures import AffNetFast
    from affnet_b200.HardNet import HardNet
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    from affnet_b200.ReprojectionStuff import frobenius_gt_pairs, frobenius_gt_sets
    W = load_weights()
    aff, hn = AffNetFast(PS=32), HardNet()
    aff.load_state_dict(W["affnet"]); hn.load_state_dict(W["hardnet"])
    aff, hn = aff.eval().to(DEV), hn.eval().to(DEV)
    B, Hh, Ww, K = 4, 480, 640, 1000
    mk = lambda s: torch.cat([synthetic_image(Hh, Ww, s + i) for i in range(B)]).to(DEV)  # noqa: E731
    imgs, imgs2 = mk(31), mk(57)
    pairs = torch.tensor([(i, j) for i in range(B) for j in range(B) if i != j], device=DEV)
    Hid = torch.eye(3, device=DEV).expand(pairs.size(0), 3, 3).contiguous()
    pipe = DetectDescribePipeline(B, Hh, Ww, aff, hn, None, num_features=K, do_ori=False)

    def step(x):
        lafs, _, dsc, c = pipe.run(x)
        tent, ntent, _, _ = match_snn_pairs(dsc, c, pairs=pairs)
        return ((ntent, c) + frobenius_gt_pairs(lafs, tent, ntent, Hid, pairs=pairs, center_dist_th=2.0)
                + frobenius_gt_sets(lafs, c, Hid, pairs=pairs, dist_threshold=50.0))

    lafs, _, dsc, c = pipe.run(imgs)
    tent, ntent, _, _ = match_snn_pairs(dsc, c, pairs=pairs)
    for fn in (lambda q: frobenius_gt_pairs(lafs, tent[q], ntent[q], Hid[q], pairs=pairs[q]),
               lambda q: frobenius_gt_sets(lafs, c, Hid[q], pairs=pairs[q])):
        assert len(lib.profile(lambda: fn(slice(0, 1)))) == len(lib.profile(lambda: fn(slice(None)))) == 2

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
    # (ntent, count, then true, ntrue, min_dist, idx2 of the tentatives, then those of the sets)
    nt, cnt = ref[0].tolist(), ref[1].tolist()
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]) and torch.equal(got[3], ref[3]) and torch.equal(got[7], ref[7])
    for p, (i, _) in enumerate(pairs.tolist()):
        n, k, n1, k1 = nt[p], int(ref[3][p]), cnt[i], int(ref[7][p])
        assert torch.equal(got[2][p, :k], ref[2][p, :k]) and torch.equal(got[4][p, :n], ref[4][p, :n]) and torch.equal(got[5][p, :n], ref[5][p, :n])
        assert torch.equal(got[6][p, :k1], ref[6][p, :k1]) and torch.equal(got[8][p, :n1], ref[8][p, :n1]) and torch.equal(got[9][p, :n1], ref[9][p, :n1])
    print("\n12 pairs in one graph: tentatives %d..%d, Frobenius-true %d..%d, set rows true %d..%d"
          % (min(nt), max(nt), int(ref[3].min()), int(ref[3].max()), int(ref[7].min()), int(ref[7].max())))
