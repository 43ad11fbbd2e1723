"""CPU tests of the matcher and ground-truth restatements (tests/matching_restated.py) and of the RANSAC restatement's solver
(tests/oracle_ransac.py): the restatements lie within their float64 bounds together with the reference, the constructed cases
(tests/matching_cases.py) reach the edges the GPU tests are meant to see, and those cases tell the restatements apart from plausible
wrong kernels, so tests/test_gpu_matching_exact.py can fail."""
import numpy as np
import torch

import affnet_oracle as O
import matching_cases as K
import matching_restated as M
import oracle_ransac as R
from helpers import gold
from snn_rule import snn_expected


def same_bits(a, b):
    """Bit-identical fp32 tensors, where any NaN equals any NaN."""
    a, b = a.contiguous(), b.contiguous()
    return a.shape == b.shape and bool(((a.view(torch.int32) == b.view(torch.int32)) | (torch.isnan(a) & torch.isnan(b))).all())


def within_bound(d, a, b):
    """Worst |d^2 - D^2| / bound over the finite entries of d, after checking that d is NaN only where D^2 <= bound (the exact sum
    under the sqrt may be cancelled below zero there) and finite wherever the inputs are."""
    val, Mg = M.dist_sq64(a, b)
    bound = M.dist_sq_bound(val, Mg, a.shape[1])
    fin = torch.isfinite(Mg)
    d = d.double()
    assert bool((torch.isnan(d) & fin <= (val <= bound)).all()), "NaN where the exact value is clear of zero"
    ok = fin & torch.isfinite(d)
    assert bool((ok == (fin & ~torch.isnan(d))).all())
    r = ((d * d - val).abs() / bound)[ok]
    assert bool((r <= 1).all()), float(r.max())
    return float(r.max()) if r.numel() else 0.0


def test_distances_within_the_float64_bound_with_the_reference():
    """The restated distances and the reference's (the golden of the unmodified Losses.distance_matrix_vector, and the oracle's on
    every constructed set) both lie within the derived bound of the float64 value."""
    z = gold("distance_matrix.npz")
    g = torch.Generator().manual_seed(5)
    a, b = torch.randn(50, 128, generator=g), torch.randn(70, 128, generator=g)
    assert a.double().sum().item() == float(z["a_sum"]) and b.double().sum().item() == float(z["b_sum"])
    worst = [within_bound(M.distances(a, b), a, b), within_bound(torch.from_numpy(z["dm"]), a, b)]
    nan = 0
    for D in K.SNN_DIMS:
        a, b = K.snn_sets(D)
        d = M.distances(a, b)
        worst += [within_bound(d, a, b), within_bound(O.distance_matrix_vector(a, b), a, b)]
        nan += int(torch.isnan(d).sum())
    print("\ndistances: worst |d^2 - D^2| %.3f of the bound (restatement and reference); %d NaN entries" % (max(worst), nan))


def test_cases_reach_the_matcher_edges():
    nan_entries = dup = tie_rows = edge_rows = 0
    for D in K.SNN_DIMS:
        a, b = K.snn_sets(D)
        d = M.distances(a, b)
        nan_entries += int(torch.isnan(d[10:18, 10:18].diagonal()).sum())
        dup += int((d[[18, 19], [18, 19]] == np.float32(np.sqrt(np.float32(1e-6)))).sum())
        if D > 1:
            row = d[4]
            assert bool((row[list(K.TIE_COLS)] == row[K.TIE_COLS[0]]).all()), D      # one minimum in three column tiles
            idx2, mn, _, _, _ = M.snn_rows(d)
            assert int(idx2[4]) == K.TIE_COLS[0] and int(idx2[70]) == K.TIE_COLS[0] and mn[4] == row[4]
            tie_rows += 2
            assert int(idx2[40]) == 40 and int(idx2[41]) == 41      # row 40's second-nearest column is masked
        q = M.ratio_quotients(d)
        r = K.ratio_edge_row(q)
        ratio = float(q[r])
        keep_at = M.snn_rows(d, ratio)[3]
        keep_below = M.snn_rows(d, float(np.nextafter(np.float32(ratio), np.float32(0))))[3]
        assert bool(keep_at[r]) and not bool(keep_below[r])
        edge_rows += 1
    print("\nmatcher cases: %d NaN distances of near-duplicates, %d exact duplicates at sqrt(1e-6), %d rows tied across tiles, "
          "%d ratio-edge rows" % (nan_entries, dup, tie_rows, edge_rows))
    assert nan_entries >= 10 and dup == 2 * len(K.SNN_DIMS) and edge_rows == len(K.SNN_DIMS)


def test_snn_rule_on_restated_distances():
    """snn_rows is snn_expected on the same distances, bit for bit (NaN and +-0 included); on NaN-free unit descriptors the
    decisions equal the oracle's match_snn wherever the nearest two columns and the ratio are clear of the distance bound."""
    for D in K.SNN_DIMS:
        a, b = K.snn_sets(D)
        d = M.distances(a, b)
        for ratio in (0.8, 1.0):
            got, exp = M.snn_rows(d, ratio), snn_expected(d, ratio)
            assert torch.equal(got[0], exp[0]) and same_bits(got[1], exp[1]) and same_bits(got[2], exp[2]), D
            assert torch.equal(got[3], exp[3]) and torch.equal(got[4], exp[4]), D
    g = torch.Generator().manual_seed(21)
    a = torch.nn.functional.normalize(torch.randn(700, 128, generator=g), dim=1)
    b = torch.cat([torch.nn.functional.normalize(a[:400] + 0.25 * torch.randn(400, 128, generator=g), dim=1),
                   torch.nn.functional.normalize(torch.randn(333, 128, generator=g), dim=1)])
    d = M.distances(a, b)
    idx2, mn, sec, keep, _ = M.snn_rows(d)
    o1, o2, omn, osec = O.match_snn(a, b)
    okeep = torch.zeros(700, dtype=torch.bool)
    okeep[o1] = True
    val, Mg = M.dist_sq64(a, b)
    slack = (M.dist_sq_bound(val, Mg, 128).max() / (2 * d.double().min() ** 2)).item()     # relative error of one distance
    top2 = d.double().sort(1).values[:, :2]
    clear = (top2[:, 1] - top2[:, 0] > 4 * slack * top2[:, 0]) & ((mn.double() / sec.double() - 0.8).abs() > 4 * slack)
    assert clear.sum() >= 650
    oidx2 = O.distance_matrix_vector(a, b).min(1).indices
    assert torch.equal(idx2[clear], oidx2[clear]) and torch.equal(keep[clear], okeep[clear])
    assert torch.equal(keep[clear][okeep[clear]], torch.ones(int(okeep[clear].sum()), dtype=torch.bool))


def test_cases_separate_the_matcher_mutations():
    """Each wrong kernel changes some output on the cases: a split-K (blocked) or pairwise distance sum, `<` in the ratio test, the
    highest column among equal minima, a NaN-propagating minimum."""
    caught = dict(kblocked=0, pairwise=0, ratio_lt=0, highest=0, nan_min=0)
    for D in K.SNN_DIMS:
        a, b = K.snn_sets(D)
        d = M.distances(a, b)
        if D > 16:
            caught["kblocked"] += int(not same_bits(M.distances(a, b, M.kblocked_dots), d))
        if D > 2:
            caught["pairwise"] += int(not same_bits(M.distances(a, b, M.pairwise_dots), d))
        q = M.ratio_quotients(d)
        ratio = float(q[K.ratio_edge_row(q)])
        caught["ratio_lt"] += int(not torch.equal(M.snn_rows(d, ratio)[3], M.snn_rows(d, ratio, le=False)[3]))
        caught["highest"] += int(not torch.equal(M.snn_rows(d)[0], M.snn_rows(d, lowest=False)[0]))
        ref, mut = M.snn_rows(d), M.snn_rows(d, nan_ignored=False)
        caught["nan_min"] += int(not (same_bits(ref[1], mut[1]) and torch.equal(ref[0], mut[0])))
    print("\nmatcher mutations caught (of %d dims): %s" % (len(K.SNN_DIMS), caught))
    assert caught["kblocked"] == sum(D > 16 for D in K.SNN_DIMS) and caught["pairwise"] == sum(D > 2 for D in K.SNN_DIMS)
    assert caught["ratio_lt"] == caught["highest"] == caught["nan_min"] == len(K.SNN_DIMS)


# ---- ground-truth check -----------------------------------------------------------------------------------------------------------------
def gt_oracle(c1, c2, H):
    """O.gt_correspondences of image-1 centres c1 [n,2] against image-2 centres c2 [m,2] at threshold +inf -> min_dist [n] of the
    reference's fp32 torch arithmetic."""
    LA, LB = torch.zeros(len(c1), 2, 3), torch.zeros(len(c2), 2, 3)
    LA[:, :, 2], LB[:, :, 2] = torch.from_numpy(np.ascontiguousarray(c1)), torch.from_numpy(np.ascontiguousarray(c2))
    mn, _, _ = O.gt_correspondences(LA, LB, torch.from_numpy(np.asarray(H, np.float32)), float("inf"))
    return mn.numpy().astype(np.float64)


def test_gt_restatement_and_reference_within_the_float64_bound():
    """Per row, min_dist^2 of the restatement (tight bound: the kernel maps in float64) and of the reference (its fp32 inverse and
    product widen the bound) against the float64 minimum; the true / not-true decisions of both agree with float64 wherever the
    float64 margin to the threshold exceeds the bound.  Rows with a NaN centre, and the singular H, are left out of the comparison
    with the reference (it propagates NaN through torch.min; the kernel ignores NaN)."""
    worst_k = worst_r = 0.0
    decided = 0
    for name, (pts, H, th) in K.gt_cases().items():
        if len(pts) > 2100 or name == "singular":
            continue                        # n = 4097 takes 2049's code path (checked on the device); no inverse to compare with
        mn, idx2, true = M.gt_check(pts, H, th)
        D2, bound = M.gt_sq64(pts, H)
        rows = np.isfinite(pts[:, :2]).all(1)
        cols = np.isfinite(pts[:, 2:]).all(1)
        rows &= np.isfinite(D2[:, cols]).all(1)
        if not rows.any():
            continue
        j = np.argmin(np.where(cols[None], D2, np.inf), 1)
        d2min, bmin = D2[np.arange(len(pts)), j], bound[np.arange(len(pts)), j]
        got = mn.numpy().astype(np.float64)
        rk = np.abs(got ** 2 - d2min)[rows] / bmin[rows]
        assert (rk <= 1).all(), (name, rk.max())
        worst_k = max(worst_k, float(rk.max()))
        _, bref = M.gt_sq64(pts, H, fp32_inverse=True)
        brmin = bref[np.arange(len(pts)), j]
        ref = np.full(len(pts), np.nan)
        ref[rows] = gt_oracle(pts[rows, :2], pts[cols, 2:], H)
        rr = np.abs(ref ** 2 - d2min)[rows] / brmin[rows]
        assert (rr <= 1).all(), (name, rr.max())
        worst_r = max(worst_r, float(rr.max()))
        th2 = float(np.float32(th)) ** 2
        sure = rows & (np.abs(d2min - th2) > np.maximum(bmin, brmin))
        kept = np.zeros(len(pts), bool)
        kept[true.numpy()] = True
        assert np.array_equal(kept[sure], (d2min <= th2)[sure]), name
        assert np.array_equal((ref <= np.float32(th))[sure], (d2min <= th2)[sure]), name
        decided += int(sure.sum())
    print("\nGT: worst |min_dist^2 - D^2| %.3f of the bound (restatement), %.3f (reference); %d decisions compared" % (worst_k, worst_r, decided))
    assert decided > 5000


def test_cases_reach_the_gt_edges():
    cases = K.gt_cases()
    kept, mn = {}, {}
    for name in ("at5", "at5_th_below", "at5_th_above", "th0", "nearer", "nearer_th_below", "farther"):
        m, idx2, true = M.gt_check(*cases["identity_" + name])
        kept[name], mn[name] = 0 in true.tolist(), float(m[0])
        assert int(idx2[0]) == 0
    f5 = float(np.float32(5))
    assert mn["at5"] == f5 and mn["nearer"] < f5 < mn["farther"]            # one ulp of the centre moves the distance
    assert kept["at5"] and not kept["at5_th_below"] and kept["at5_th_above"] and not kept["th0"]
    assert kept["nearer"] and kept["nearer_th_below"] and not kept["farther"]
    pts, H, th = cases["n2049"]
    mn, idx2, _ = M.gt_check(pts, H, th)
    assert idx2[100] == idx2[7] == 7 or idx2[100] == idx2[7]      # rows 7 and 100-102 are one row: one answer
    d = M.gt_dist(pts, H)
    assert int((d[7] == d[7, 7]).sum()) >= 4                        # duplicate image-2 centres: a tie among 4 columns
    assert mn[60] == np.inf and idx2[60] == 0                       # a NaN centre in image 1: (+inf, 0)
    mn, idx2, true = M.gt_check(*cases["singular"])
    assert bool(torch.isinf(mn).all()) and not bool(idx2.any()) and true.numel() == 0
    pts, H, th = cases["horizon"]
    px, _ = M.gt_mapped(pts, H)
    assert not np.isfinite(px[:2]).any() and np.isfinite(px[2:]).all()     # w = 0 at x = -64; w < 0 further left maps finitely
    pts, H, th = cases["large"]
    D2, bound = M.gt_sq64(pts, H)
    print("\nGT cases: exact-threshold rows reached; large-coordinate bound median %.2f px^2" % float(np.median(bound.min(1))))
    assert np.median(bound.min(1)) > 0.5


def test_cases_separate_the_gt_mutations():
    """An unfused dot, the other fused operand order, `<` for `<=`, the highest index among equal minima and a NaN-propagating
    minimum each change the output of some case."""
    cases = K.gt_cases()
    pts, H, th = cases["large"]
    d = M.gt_dist(pts, H)
    nu = int((M.gt_dist(pts, H, fused=False) != d).sum())
    ns = int((M.gt_dist(pts, H, swap=True) != d).sum())
    pts5, I, _ = cases["identity_at5"]
    d5 = M.gt_dist(pts5, I)
    lt = not torch.equal(M.gt_rows(d5, 5.0)[2], M.gt_rows(d5, 5.0, le=False)[2])
    p, Hn, thn = cases["n2049"]
    dn = M.gt_dist(p, Hn)
    hi = not torch.equal(M.gt_rows(dn, thn)[1], M.gt_rows(dn, thn, lowest=False)[1])
    nanp = not same_bits(M.gt_rows(dn, thn)[0], M.gt_rows(dn, thn, nan_ignored=False)[0])
    print("\nGT mutations: unfused dot changes %d distances, the other operand order %d; <: %s, highest index: %s, NaN-propagating: %s"
          % (nu, ns, lt, hi, nanp))
    assert nu > 1000 and ns > 1000 and lt and hi and nanp


# ---- RANSAC -----------------------------------------------------------------------------------------------------------------------------
def run_cases(**kw):
    out = {}
    for name, (pts, it, seed, th) in K.ransac_cases().items():
        tr = {}
        out[name] = R.ransac(pts, th, 0.99, it, seed, trace=tr, **kw) + (tr,)
    return out


def test_cases_reach_the_ransac_edges():
    res = run_cases()
    pts, at, beyond = K.translation_edge()
    tr = res["translation_edge"][4]
    H0 = tr["H0"]
    assert np.array_equal(H0, np.array([1, 0, K.TRANSLATION[0], 0, 1, K.TRANSLATION[1], 0, 0, 1.0]))
    p = pts.astype(np.float64)
    err = (p[:, 0] + H0[2] - p[:, 2]) ** 2 + (p[:, 1] + H0[5] - p[:, 3]) ** 2
    assert np.all(err[at] == K.EDGE_TH ** 2) and np.all(err[beyond] > K.EDGE_TH ** 2)
    assert R.inliers(H0, p, K.EDGE_TH ** 2)[0][at].all() and not R.inliers(H0, p, K.EDGE_TH ** 2)[0][beyond].any()
    hp, behind = K.horizon_pairs()
    assert behind.sum() > 20 and not res["horizon"][1][behind].any()
    c = res["refit_break"][4]["counts"]
    assert any(c[i + 1] < c[i] for i in range(len(c) - 1)), c
    assert [res["iters%d" % k][3] for k in (1, 255, 256, 257)] == [1, 255, 256, 257]
    assert not np.array_equal(res["seed_max_iters257"][1], res["iters257"][1])      # the seed changes the draws
    print("\nRANSAC cases: %d rows at err == th^2, a refit round lowering %s, %d rows beyond the horizon" % (len(at), c, behind.sum()))


def test_cases_separate_the_ransac_mutation(monkeypatch):
    """`<` for `<=` in the inlier test changes the translation case's result."""
    pts, it, seed, th = K.ransac_cases()["translation_edge"]
    H, m, n, _ = R.ransac(pts, th, 0.99, it, seed)
    strict = R.inliers

    def lt(H, pts, th2):
        return strict(H, pts, np.nextafter(th2, 0.0))
    monkeypatch.setattr(R, "inliers", lt)
    H2, m2, n2, _ = R.ransac(pts, th, 0.99, it, seed)
    print("\nRANSAC with <: %d inliers instead of %d" % (n2, n))
    assert n2 != n or not np.array_equal(m2, m) or not np.array_equal(H2, H)


def test_ransac_refits_against_float64():
    """Every refit the cases reach: the Jacobi off-diagonal norm after JACOBI_SWEEPS is below 1e-14 of |A|, the chosen eigenvector is
    eigh's smallest within its Davis-Kahan bound, and where that bound is below 1e-9 the homography maps the frame's corners within
    1e-6 px of the float64 SVD of the same normalised DLT."""
    from verify_cases import correspondences, random_homography
    res = run_cases()
    extra = [correspondences(200 + s, 1000, random_homography(300 + s), outliers=0.4)[0] for s in range(4)]
    for k, p in enumerate(extra):
        tr = {}
        res["synthetic%d" % k] = R.ransac(p, trace=tr) + (tr,)
    cases = K.ransac_cases()
    w_off = w_sin = w_err = 0.0
    n = 0
    for name, r in res.items():
        pts = (cases[name][0] if name in cases else extra[int(name[9:])]).astype(np.float64)
        for t in r[4].get("refits", []):
            off, sin, bound, err = M.refit_report(t, pts)
            assert off <= 1e-14 and sin <= bound, (name, off, sin, bound)
            w_off, w_sin = max(w_off, off), max(w_sin, sin)
            if bound <= 1e-9:
                assert err <= 1e-6, (name, err)
                w_err = max(w_err, err)
            n += 1
    print("\nRANSAC refits (%d) against float64: worst Jacobi residual %.1e of |A|, eigenvector error %.1e, DLT corner error %.1e px"
          % (n, w_off, w_sin, w_err))
    assert n >= 30
