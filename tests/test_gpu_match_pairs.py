"""GPU tests (-m gpu) of the batched SNN matcher (ag_match_pairs, Losses.match_snn_pairs).  The expected values are computed without the
matcher's kernels: ag_distance_matrix (distance_matrix_vector) on the count-sliced descriptors of each pair, then the torch reductions of
snn_rule.snn_expected.  Every output is prefilled with a sentinel, so rows the matcher must not write are checked as well."""
import pytest
import torch

from helpers import SENTINEL, gold, gray_from_rgb, load_weights, synthetic_image
from snn_rule import snn_expected

pytestmark = pytest.mark.gpu

DEV = "cuda"
KEEP_SENTINEL = 0xAB


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


def run_pairs(L, d1, c1, d2, c2, pairs, ratio=0.8):
    """ag_match_pairs over sentinel-filled outputs -> dict of all of them (idx2, min, second, keep, tent, ntent)."""
    S1, cap1, D = d1.shape
    S2, cap2 = d2.shape[:2]
    P = S1 if pairs is None else pairs.size(0)
    o = dict(idx2=torch.full((P, cap1), -7, dtype=torch.int32, device=DEV), min=torch.full((P, cap1), SENTINEL, device=DEV),
             second=torch.full((P, cap1), SENTINEL, device=DEV), keep=torch.full((P, cap1), KEEP_SENTINEL, dtype=torch.uint8, device=DEV),
             tent=torch.full((P, cap1, 2), -7, dtype=torch.int32, device=DEV), ntent=torch.full((P,), -9, dtype=torch.int32, device=DEV))
    nb = L.lib().ag_match_pairs_workspace_bytes(S1, cap1, S2, cap2, P)
    ws = torch.full((nb,), 0xFF, dtype=torch.uint8, device=DEV)   # a dirty workspace: the column masks must be cleared by the call
    L.check(L.lib().ag_match_pairs(L.ptr(d1), L.ptr(c1), S1, cap1, L.ptr(d2), L.ptr(c2), S2, cap2, D, L.ptr(pairs), P, float(ratio), L.ptr(ws), nb,
                                   L.ptr(o["idx2"]), L.ptr(o["min"]), L.ptr(o["second"]), L.ptr(o["keep"]), L.ptr(o["tent"]), L.ptr(o["ntent"]),
                                   L.stream_ptr()))
    torch.cuda.synchronize()
    return o


def pair_list(pairs, S):
    return [(p, p) for p in range(S)] if pairs is None else [tuple(x) for x in pairs.tolist()]


def check_against_expected(o, d1, c1, d2, c2, pairs, ratio=0.8, tag=""):
    """Valid pairs: idx2, min, second and keep bit-identical to snn_expected, tent[:ntent] = (arange[keep], idx2[keep]), rows beyond n1 and
    tentative rows beyond ntent untouched.  Pairs with an index out of range or a count outside 0..cap: ntent -1; with an empty image: 0;
    nothing else written.  Returns the per-pair tentative counts."""
    from affnet_b200.Losses import distance_matrix_vector
    S1, cap1 = d1.shape[:2]
    S2, cap2 = d2.shape[:2]
    cnt1 = [cap1] * S1 if c1 is None else c1.tolist()
    cnt2 = [cap2] * S2 if c2 is None else c2.tolist()
    ntent = o["ntent"].tolist()
    out = []
    for p, (i, j) in enumerate(pair_list(pairs, S1)):
        what = (tag, p, i, j)
        valid = 0 <= i < S1 and 0 <= j < S2 and 0 <= cnt1[i] <= cap1 and 0 <= cnt2[j] <= cap2
        n1 = cnt1[i] if valid else 0
        if not valid or n1 == 0 or cnt2[j] == 0:
            assert ntent[p] == (0 if valid else -1), what
            n1 = 0
        else:
            n2 = cnt2[j]
            idx2, mn, sec, keep, tent = snn_expected(distance_matrix_vector(d1[i, :n1], d2[j, :n2]), ratio)
            assert torch.equal(o["idx2"][p, :n1].long(), idx2), what
            assert torch.equal(o["min"][p, :n1], mn), what
            assert torch.equal(o["second"][p, :n1], sec), what
            assert torch.equal(o["keep"][p, :n1].bool(), keep) and bool((o["keep"][p, :n1] <= 1).all()), what
            assert ntent[p] == tent.size(0), what
            assert torch.equal(o["tent"][p, :ntent[p]].long(), tent), what
        t = max(ntent[p], 0)
        assert bool((o["tent"][p, t:] == -7).all()), (what, "tentative rows beyond ntent written")
        assert bool((o["idx2"][p, n1:] == -7).all()) and bool((o["min"][p, n1:] == SENTINEL).all()), (what, "rows beyond n1 written")
        assert bool((o["second"][p, n1:] == SENTINEL).all()) and bool((o["keep"][p, n1:] == KEEP_SENTINEL).all()), (what, "rows beyond n1 written")
        out.append(ntent[p])
    return out


def related_sets(S, cap, D, seed, noise=0.3):
    """S sets of unit descriptors that share a common base (so the ratio test keeps a fair share of rows)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(cap, D, generator=g)
    perm = lambda: torch.randperm(cap, generator=g)  # noqa: E731
    d = torch.stack([torch.nn.functional.normalize(base[perm()] + noise * torch.randn(cap, D, generator=g), dim=1) for _ in range(S)])
    return d.to(DEV)


def test_ragged_sets(L):
    """S = 6, cap 700, counts [700, 1, 0, 333, 699, -1]: self pairs, both directions, a repeated pair, n1 = 1, n2 = 1 (every second is
    100000), n1 = 0, n2 = 0, the -1 count on either side, indices out of range; the wrapper gives the same outputs."""
    from affnet_b200.Losses import match_snn_pairs
    d = related_sets(6, 700, 128, 3)
    cnt = torch.tensor([700, 1, 0, 333, 699, -1], dtype=torch.int32, device=DEV)
    pl = [(0, 0), (3, 3), (4, 4), (0, 3), (3, 0), (0, 4), (0, 4), (4, 0), (0, 1), (3, 1), (1, 0), (1, 1), (2, 0), (0, 2), (2, 2),
          (5, 0), (0, 5), (6, 0), (0, 6), (-1, 0), (0, -1), (3, 4), (4, 3)]
    pairs = torch.tensor(pl, dtype=torch.int32, device=DEV)
    o = run_pairs(L, d, cnt, d, cnt, pairs)
    nt = check_against_expected(o, d, cnt, d, cnt, pairs, tag="ragged")
    print("\nragged: tentatives per pair %s" % nt)
    assert nt[pl.index((0, 0))] == 700 and nt[pl.index((0, 1))] == 700       # n2 = 1: second is 100000 for every row
    assert bool((o["second"][pl.index((0, 1)), :700] == 100000).all())
    assert nt[pl.index((2, 0))] == 0 and nt[pl.index((0, 2))] == 0 and nt[pl.index((5, 0))] == -1 and nt[pl.index((0, -1))] == -1
    assert 0 < nt[pl.index((0, 3))] < 333 + 700 and nt[5] == nt[6]
    tent, ntent, mn, sec = match_snn_pairs(d, cnt, pairs=pairs.long())
    torch.cuda.synchronize()
    assert torch.equal(ntent, o["ntent"])
    for p, t in enumerate(nt):
        i = pl[p][0]
        n1 = int(cnt[i]) if t > 0 else 0
        assert torch.equal(tent[p, :max(t, 0)], o["tent"][p, :max(t, 0)])
        assert torch.equal(mn[p, :n1], o["min"][p, :n1]) and torch.equal(sec[p, :n1], o["second"][p, :n1])


def test_two_sets_different_caps(L):
    """Set 1 [4,500,128], set 2 [4,300,128] with counts, pairs=None (pair p = (p, p)), then an explicit list across S1 = 4, S2 = 3."""
    from affnet_b200.Losses import match_snn_pairs
    d1 = related_sets(4, 500, 128, 11)
    d2 = (d1[:, :300] * 0.5 + 0.5 * related_sets(4, 300, 128, 12)).contiguous()
    c1 = torch.tensor([500, 17, 250, 0], dtype=torch.int32, device=DEV)
    c2 = torch.tensor([300, 299, 1, 5], dtype=torch.int32, device=DEV)
    o = run_pairs(L, d1, c1, d2, c2, None)
    check_against_expected(o, d1, c1, d2, c2, None, tag="pairs=None")
    o = run_pairs(L, d1, None, d2, None, None)
    check_against_expected(o, d1, None, d2, None, None, tag="pairs=None, no counts")
    d3, c3 = d2[:3].contiguous(), c2[:3].contiguous()
    pairs = torch.tensor([[0, 0], [1, 2], [3, 1], [2, 1], [0, 2], [3, 3]], dtype=torch.int32, device=DEV)
    o = run_pairs(L, d1, c1, d3, c3, pairs)
    check_against_expected(o, d1, c1, d3, c3, pairs, tag="S1 = 4, S2 = 3")
    tent, ntent, _, _ = match_snn_pairs(d1, c1, d3, c3, pairs)
    assert torch.equal(ntent, o["ntent"]) and ntent.tolist()[-1] == -1


@pytest.mark.parametrize("D", [128, 40, 1])
def test_constructed_cases(L, D):
    """Duplicate columns (the lowest index must win), NaN rows in either set, and a row whose second-nearest column is another row's
    nearest, so that the 100000 mask changes its second distance."""
    g = torch.Generator().manual_seed(5 + D)
    n1, n2 = 150, 130
    a = torch.nn.functional.normalize(torch.randn(n1, D, generator=g), dim=1)
    b = torch.nn.functional.normalize(torch.randn(n2, D, generator=g), dim=1)
    b[7] = b[3]; b[100] = b[3]; b[64] = b[3]            # equal columns on both sides of a column-tile edge
    a[0] = b[3]; a[1] = b[3] * 0.999                     # rows whose nearest column is one of the duplicates
    a[5] = float("nan")                                   # a NaN row: (+inf, column 0)
    b[20] = float("nan")                                  # a NaN column: ignored
    # row 10's nearest is column 50 and its second-nearest column 51, which is row 11's nearest: masked to 100000
    b[50] = a[10]; b[51] = torch.nn.functional.normalize(a[10] + 0.05 * torch.randn(D, generator=g), dim=0); a[11] = b[51]
    d1, d2 = a.view(1, n1, D).to(DEV), b.view(1, n2, D).to(DEV)
    o = run_pairs(L, d1, None, d2, None, None)
    check_against_expected(o, d1, None, d2, None, None, tag="constructed D=%d" % D)
    idx2 = o["idx2"][0].tolist()
    assert idx2[5] == 0 and o["min"][0, 5].item() == float("inf")
    if D > 1:
        assert idx2[0] == 3 and idx2[1] == 3 and idx2[10] == 50 and idx2[11] == 51 and 20 not in idx2
        from affnet_b200.Losses import distance_matrix_vector
        dm = distance_matrix_vector(d1[0], d2[0])
        unmasked = torch.where(torch.isnan(dm[10]), float("inf"), dm[10]).sort().values[1]
        assert o["second"][0, 10].item() != unmasked.item()
    # the same rows twice, as set 1 and set 2 of one tensor (self matching)
    o = run_pairs(L, d1, None, d1, None, None)
    check_against_expected(o, d1, None, d1, None, None, tag="self D=%d" % D)


def test_single_pair_matcher_is_the_batched_one(L):
    """Losses.match_snn (ag_match_snn) = pair (0, 0) of the batched call, on the test_snn_matcher_8f fixture."""
    from affnet_b200.Losses import match_snn, match_snn_pairs
    g = torch.Generator().manual_seed(21)
    d1 = torch.nn.functional.normalize(torch.randn(700, 128, generator=g), dim=1)
    d2 = torch.cat([torch.nn.functional.normalize(d1[:400] + 0.25 * torch.randn(400, 128, generator=g), dim=1),
                    torch.nn.functional.normalize(torch.randn(333, 128, generator=g), dim=1)])
    d1, d2 = d1.to(DEV), d2.to(DEV)
    i1, i2, mn, sec = match_snn(d1, d2, 0.8)
    tent, ntent, mn2, sec2 = match_snn_pairs(d1[None], None, d2[None], None)
    n = int(ntent[0])
    assert n == i1.numel() and torch.equal(tent[0, :n, 0].long(), i1) and torch.equal(tent[0, :n, 1].long(), i2)
    assert torch.equal(mn2[0], mn) and torch.equal(sec2[0], sec)


def test_pipeline_outputs_all_ordered_pairs_and_graph(L, nets):
    """16 x 1024x768 synthetic images (one constant: count 0), K = 2000: all 240 ordered pairs i != j in one call against the expected
    values; pipe.run and match_snn_pairs captured in ONE CUDA graph, replayed on other images, equal to the eager run; the launch count
    does not depend on the number of pairs."""
    import affnet_b200._lib as lib
    from affnet_b200.Losses import match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    aff, ori, hn = nets
    B, H, Wd, K = 16, 768, 1024, 2000
    mk = lambda s: torch.cat([synthetic_image(H, Wd, s + i) if i != 6 else torch.full((1, 1, H, Wd), 90.0) for i in range(B)]).to(DEV)  # noqa: E731
    imgs, imgs2 = mk(1234), mk(777)
    pairs = torch.tensor([(i, j) for i in range(B) for j in range(B) if i != j], device=DEV)
    pipe = DetectDescribePipeline(B, H, Wd, aff, hn, ori, num_features=K)
    _, _, desc, cnt = pipe.run(imgs)
    pipe.check()
    assert int(cnt[6]) == 0 and bool((cnt[:6] > 1000).all())
    o = run_pairs(L, desc, cnt, desc, cnt, pairs.int().contiguous())
    nt = check_against_expected(o, desc, cnt, desc, cnt, pairs, tag="pipeline")
    print("\npipeline 240 pairs: tentatives min %d max %d" % (min(t for t in nt if t > 0), max(nt)))
    assert sum(1 for t in nt if t == 0) >= 30 and all(t >= 0 for t in nt)
    n_one = len(lib.profile(lambda: match_snn_pairs(desc, cnt, pairs=pairs[:1])))
    n_all = len(lib.profile(lambda: match_snn_pairs(desc, cnt, pairs=pairs)))
    assert n_one == n_all == 4, (n_one, n_all)

    static_in = imgs.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _, _, dd, cc = pipe.run(static_in)
        match_snn_pairs(dd, cc, pairs=pairs)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _, _, dd, cc = pipe.run(static_in)
        res = match_snn_pairs(dd, cc, pairs=pairs)
    static_in.copy_(imgs2)
    g.replay()
    torch.cuda.synchronize()
    got = [t.clone() for t in res]
    gcnt = cc.clone()
    _, _, desc2, cnt2 = pipe.run(imgs2)
    ref = match_snn_pairs(desc2, cnt2, pairs=pairs)
    torch.cuda.synchronize()
    assert torch.equal(gcnt, cnt2) and torch.equal(got[1], ref[1])
    cl = cnt2.tolist()
    for p, (i, j) in enumerate(pair_list(pairs, B)):
        t = max(int(ref[1][p]), 0)
        assert torch.equal(got[0][p, :t], ref[0][p, :t]), p
        n1 = cl[i] if cl[j] > 0 else 0   # an empty image 2: the pair's rows are not written
        assert torch.equal(got[2][p, :n1], ref[2][p, :n1]) and torch.equal(got[3][p, :n1], ref[3][p, :n1]), p
    assert not torch.equal(got[1], o["ntent"])   # the replay really ran on the other images


def test_graf_1_to_6_as_a_batch(L, nets):
    """graf img1 and img6 as one B = 2 batch of the pipeline (AffNet + histogram, K = 3000): pair (0, 1) gives the tentatives of
    Losses.match_snn on the count-sliced descriptors."""
    from affnet_b200.Losses import match_snn, match_snn_pairs
    from affnet_b200.pipeline import DetectDescribePipeline
    aff, ori, hn = nets
    z, f = gold("graf_match.npz"), gold("graf_full.npz")
    x1, x6 = gray_from_rgb(f["rgb"]), gray_from_rgb(z["rgb6"])
    H, Wd = x1.shape[2:]
    pipe = DetectDescribePipeline(2, H, Wd, aff, hn, None, num_features=3000, do_ori=True)
    _, _, desc, cnt = pipe.run(torch.cat([x1, x6]).to(DEV))
    tent, ntent, mn, sec = match_snn_pairs(desc, cnt, pairs=torch.tensor([[0, 1]], device=DEV), SNN_threshold=float(z["snn"]))
    pipe.check()
    n1, n2 = int(cnt[0]), int(cnt[1])
    i1, i2, omn, osec = match_snn(desc[0, :n1], desc[1, :n2], float(z["snn"]))
    t = int(ntent[0])
    print("\ngraf 1<->6 as a batch: %d tentatives" % t)
    assert t == i1.numel() > 0 and torch.equal(tent[0, :t, 0].long(), i1) and torch.equal(tent[0, :t, 1].long(), i2)
    assert torch.equal(mn[0, :n1], omn) and torch.equal(sec[0, :n1], osec)


def test_one_large_pair(L):
    """16384 x 12000 rows: the workspace is the norms and one column mask (no 750 MiB matrix), and every output matches."""
    d1 = related_sets(1, 16384, 128, 31)
    d2 = torch.nn.functional.normalize(d1[:, :12000] + 0.03 * torch.randn(1, 12000, 128, device=DEV, generator=torch.Generator(DEV).manual_seed(3)), dim=2)
    nb = L.lib().ag_match_pairs_workspace_bytes(1, 16384, 1, 12000, 1)
    assert nb < 256 * 1024, nb
    o = run_pairs(L, d1, None, d2.contiguous(), None, None)
    nt = check_against_expected(o, d1, None, d2.contiguous(), None, None, tag="large")
    print("\n16384 x 12000: %d tentatives, workspace %d bytes" % (nt[0], nb))
    assert nt[0] > 1000
