"""GPU tests (-m gpu): the SNN matcher, ag_distance_matrix and the ground-truth check bit for bit against their exact restatements
(tests/matching_restated.py), and RANSAC bit for bit against tests/oracle_ransac.py, on the constructed cases of tests/matching_cases.py;
the distances also within their float64 bounds.  Outputs start as a sentinel, so a missing or stray write is seen.
tests/test_matching_restated_cpu.py shows on the CPU that these cases separate the restatements from plausible wrong kernels."""
import numpy as np
import pytest
import torch

import matching_cases as K
import matching_restated as M
import oracle_ransac as R
from helpers import SENTINEL

pytestmark = pytest.mark.gpu

DEV = "cuda"
KEEP_SENTINEL = 0xAB
WORST = {}


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    lib.lib()
    return lib


def same_bits(a, b):
    """Bit-identical fp32 (any NaN equals any NaN: the device's NaN payload is canonical)."""
    a, b = a.detach().cpu().float().contiguous(), b.detach().cpu().float().contiguous()
    return a.shape == b.shape and bool(((a.view(torch.int32) == b.view(torch.int32)) | (torch.isnan(a) & torch.isnan(b))).all())


def note(key, v):
    WORST[key] = max(WORST.get(key, 0.0), v)


def bound_ratio(d, a, b):
    """Worst |d^2 - D^2| / bound over d's finite entries (NaN only where the exact value is within the bound of zero)."""
    val, Mg = M.dist_sq64(a, b)
    bound = M.dist_sq_bound(val, Mg, a.shape[1])
    d = d.double()
    fin = torch.isfinite(Mg)
    assert bool(((torch.isnan(d) & fin) <= (val <= bound)).all())
    ok = fin & torch.isfinite(d)
    r = ((d * d - val).abs() / bound)[ok]
    return float(r.max()) if r.numel() else 0.0


@pytest.mark.parametrize("D", K.SNN_DIMS)
def test_distance_matrix_bit_exact(L, D):
    """ag_distance_matrix at n1, n2 across the 64-row / 64-column tile edges, into a sentinel-filled buffer twice as long."""
    a, b = K.snn_sets(D)
    ref = M.distances(a, b)
    for n1, n2 in ((1, 1), (1, 129), (63, 65), (64, 64), (65, 63), (129, 129)):
        out = torch.full((2 * n1 * n2 + 64,), SENTINEL, device=DEV)
        da, db = a[:n1].to(DEV).contiguous(), b[:n2].to(DEV).contiguous()
        L.check(L.lib().ag_distance_matrix(L.ptr(da), n1, L.ptr(db), n2, D, L.ptr(out), L.stream_ptr()))
        torch.cuda.synchronize()
        got = out[:n1 * n2].view(n1, n2).cpu()
        assert same_bits(got, ref[:n1, :n2]), (D, n1, n2, int((got != ref[:n1, :n2]).sum()))
        assert bool((out[n1 * n2:] == SENTINEL).all()), (D, n1, n2, "written past n1 * n2")
        note("distance", bound_ratio(got, a[:n1], b[:n2]))


def run_pairs(L, d1, c1, d2, c2, pairs, ratio):
    S1, cap1, D = d1.shape
    S2, cap2 = d2.shape[:2]
    P = pairs.size(0)
    o = dict(idx2=torch.full((P, cap1), -7, dtype=torch.int32, device=DEV), min=torch.full((P, cap1), SENTINEL, device=DEV),
             second=torch.full((P, cap1), SENTINEL, device=DEV), keep=torch.full((P, cap1), KEEP_SENTINEL, dtype=torch.uint8, device=DEV),
             tent=torch.full((P, cap1, 2), -7, dtype=torch.int32, device=DEV), ntent=torch.full((P,), -9, dtype=torch.int32, device=DEV))
    nb = L.lib().ag_match_pairs_workspace_bytes(S1, cap1, S2, cap2, P)
    ws = torch.full((nb,), 0xFF, dtype=torch.uint8, device=DEV)
    L.check(L.lib().ag_match_pairs(L.ptr(d1), L.ptr(c1), S1, cap1, L.ptr(d2), L.ptr(c2), S2, cap2, D, L.ptr(pairs), P, float(ratio), L.ptr(ws), nb,
                                   L.ptr(o["idx2"]), L.ptr(o["min"]), L.ptr(o["second"]), L.ptr(o["keep"]), L.ptr(o["tent"]), L.ptr(o["ntent"]),
                                   L.stream_ptr()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


@pytest.mark.parametrize("D", K.SNN_DIMS)
def test_match_pairs_bit_exact(L, D):
    """One ragged batch: set 1 holds the case's rows at counts 1, 63, 64, 65, 129 (one image each), set 2 likewise; all 25 pairs and
    a pair with a count of -1.  idx2, min, second, keep, tent and ntent equal the restatement bit for bit at ratio 0.8, at one row's
    exact quotient and at the next fp32 value toward 0; rows beyond n1 and tentatives beyond ntent keep their sentinels."""
    a, b = K.snn_sets(D)
    dist = M.distances(a, b)
    S = len(K.SNN_COUNTS)
    d1 = a[None].expand(S + 1, -1, -1).contiguous().to(DEV)
    d2 = b[None].expand(S + 1, -1, -1).contiguous().to(DEV)
    cnt = torch.tensor(list(K.SNN_COUNTS) + [-1], dtype=torch.int32, device=DEV)
    pl = [(i, j) for i in range(S) for j in range(S)] + [(S, 0), (0, S)]
    pairs = torch.tensor(pl, dtype=torch.int32, device=DEV)
    q = M.ratio_quotients(dist)
    qr = float(q[K.ratio_edge_row(q)])
    for ratio in (0.8, qr, float(np.nextafter(np.float32(qr), np.float32(0)))):
        o = run_pairs(L, d1, cnt, d2, cnt, pairs, ratio)
        for p, (i, j) in enumerate(pl):
            what = (D, ratio, p, i, j)
            if i == S or j == S:
                assert int(o["ntent"][p]) == -1 and bool((o["idx2"][p] == -7).all()), what
                continue
            n1, n2 = K.SNN_COUNTS[i], K.SNN_COUNTS[j]
            idx2, mn, sec, keep, tent = M.snn_rows(dist[:n1, :n2], ratio)
            assert torch.equal(o["idx2"][p, :n1].long(), idx2), what
            assert same_bits(o["min"][p, :n1], mn) and same_bits(o["second"][p, :n1], sec), what
            assert torch.equal(o["keep"][p, :n1], keep.to(torch.uint8)), what
            nt = int(o["ntent"][p])
            assert nt == tent.size(0) and torch.equal(o["tent"][p, :nt].long(), tent), what
            assert bool((o["tent"][p, nt:] == -7).all()) and bool((o["min"][p, n1:] == SENTINEL).all()), what
            assert bool((o["keep"][p, n1:] == KEEP_SENTINEL).all()) and bool((o["idx2"][p, n1:] == -7).all()), what
    # the one-pair entry point is the batched one
    from affnet_b200.Losses import match_snn
    i1, i2, mn, sec = match_snn(a.to(DEV), b.to(DEV), qr)
    idx2, rmn, rsec, keep, tent = M.snn_rows(dist, qr)
    assert torch.equal(i1.cpu(), tent[:, 0]) and torch.equal(i2.cpu(), tent[:, 1]) and same_bits(mn, rmn) and same_bits(sec, rsec)


# ---- ground-truth check ----------------------------------------------------------------------------------------------------------------
def gt_call(L, pts_list, Hs, th):
    """ag_gt_correspondences_pairs, pair p holding case p's centres at permuted LAF rows (tcap = the largest n + 3)."""
    P = len(pts_list)
    cap = max(len(p) for p in pts_list) + 3
    g = torch.Generator().manual_seed(P)
    l1, l2 = torch.zeros(P, cap, 2, 3), torch.zeros(P, cap, 2, 3)
    tent = torch.full((P, cap, 2), -5, dtype=torch.int32)
    for s, pts in enumerate(pts_list):
        n = len(pts)
        r1, r2 = torch.randperm(cap, generator=g)[:n], torch.randperm(cap, generator=g)[:n]
        p = torch.from_numpy(pts)
        l1[s, r1, 0, 2], l1[s, r1, 1, 2], l2[s, r2, 0, 2], l2[s, r2, 1, 2] = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
        tent[s, :n, 0], tent[s, :n, 1] = r1.int(), r2.int()
    ntent = torch.tensor([len(p) for p in pts_list], dtype=torch.int32, device=DEV)
    H = torch.from_numpy(np.stack([np.asarray(h, np.float32) for h in Hs])).to(DEV).contiguous()
    l1, l2, tent = l1.to(DEV), l2.to(DEV), tent.to(DEV)
    o = dict(min=torch.full((P, cap), SENTINEL, device=DEV), idx2=torch.full((P, cap), -7, dtype=torch.int32, device=DEV),
             true=torch.full((P, cap), -7, dtype=torch.int32, device=DEV), ntrue=torch.full((P,), -9, dtype=torch.int32, device=DEV))
    L.check(L.lib().ag_gt_correspondences_pairs(L.ptr(l1), P, cap, L.ptr(l2), P, cap, None, P, L.ptr(tent), L.ptr(ntent), cap, L.ptr(H),
                                                float(th), L.ptr(o["min"]), L.ptr(o["idx2"]), L.ptr(o["true"]), L.ptr(o["ntrue"]), L.stream_ptr()))
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


def check_gt(o, p, pts, H, th, tag):
    n = len(pts)
    mn, idx2, true = M.gt_check(pts, H, th, DEV)
    assert same_bits(o["min"][p, :n], mn), (tag, int((o["min"][p, :n] != mn).sum()))
    assert torch.equal(o["idx2"][p, :n].long(), idx2), tag
    nt = int(o["ntrue"][p])
    assert nt == true.numel() and torch.equal(o["true"][p, :nt].long(), true), tag
    assert bool((o["min"][p, n:] == SENTINEL).all()) and bool((o["true"][p, nt:] == -7).all()), tag
    if np.isfinite(pts).all() and np.isfinite(M.gt_inverse(H)).all() and n <= 2100:
        D2, bound = M.gt_sq64(pts, H)
        D2 = np.where(np.isfinite(D2), D2, np.inf)               # centres mapped to w = 0 are never a minimum
        j = np.argmin(D2, 1)
        ok = np.isfinite(D2[np.arange(n), j])
        r = (np.abs(mn.numpy().astype(np.float64) ** 2 - D2[np.arange(n), j]) / bound[np.arange(n), j])[ok]
        assert (r <= 1).all(), (tag, r.max())
        note("gt", float(r.max()))
    return nt


def test_gt_bit_exact(L):
    """Every GT case alone (its own threshold), then the threshold-6 cases as one batch of pairs."""
    cases = K.gt_cases()
    for name, (pts, H, th) in cases.items():
        o = gt_call(L, [pts], [H], th)
        check_gt(o, 0, pts, H, th, name)
    names = [k for k, v in cases.items() if v[2] == 6.0]
    o = gt_call(L, [cases[k][0] for k in names], [cases[k][1] for k in names], 6.0)
    for p, k in enumerate(names):
        check_gt(o, p, cases[k][0], cases[k][1], 6.0, "batch " + k)


# ---- RANSAC -----------------------------------------------------------------------------------------------------------------------------
def test_ransac_bit_exact(L):
    """Each RANSAC case (grouped into one batch per max_iters, seed and threshold): H bit for bit, the whole inlier mask, ninl and
    iters equal the restatement."""
    from test_gpu_verify import build_sets, run_ransac
    cases = K.ransac_cases()
    groups = {}
    for name, (pts, it, seed, th) in cases.items():
        groups.setdefault((it, seed, th), []).append(name)
    for (it, seed, th), names in groups.items():
        sub = {k: (cases[k][0], None) for k in names}
        l1, l2, tent, ntent = build_sets(sub, seed=len(names))
        o = run_ransac(L, l1, l2, None, tent, ntent, th=th, iters=it, seed=seed)
        for p, k in enumerate(names):
            pts = cases[k][0]
            H, m, n, iters = R.ransac(pts, th, 0.99, it, seed)
            assert int(o["ninl"][p]) == n and int(o["iters"][p]) == iters, (k, int(o["ninl"][p]), n, int(o["iters"][p]), iters)
            assert np.array_equal(o["inl"][p, :len(pts)].numpy(), m.astype(np.uint8)), k
            assert np.array_equal(o["H"][p].numpy().view(np.int32), H.view(np.int32)), (k, o["H"][p], H)
            print("\nRANSAC %-18s n=%5d: %4d inliers, %5d iterations" % (k, len(pts), n, iters), end="")
    print()


def test_report_worst_bounds():
    """The worst float64 errors seen above, as fractions of their derived bounds."""
    print("\nworst |d^2 - D^2| / bound: distances %.3f, GT min_dist %.3f" % (WORST.get("distance", float("nan")), WORST.get("gt", float("nan"))))
    assert all(v <= 1.0 for v in WORST.values())
