"""CPU tests (-m "not gpu") of the affine homography RANSAC (ag_homography_ransac_affine, find_homography_pairs(affine=True)) and its
numpy restatement tests/oracle_ac_ransac.py: the prototype and the refusals, the 2-AC solver on exact correspondences, every degeneracy
rule, the frame distance against the Frobenius restatement pinned to the reference, and the search on constructed scenes."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

import affine_cases as AC
import frobenius_restated as FR
import oracle_ac_ransac as A
import oracle_ransac as R
from verify_cases import corner_error, project

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "ag_homography_ransac_affine"


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


def test_prototype_matches_the_header(L):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "affnet_b200.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+%s\s*\(([^;]*)\)\s*;" % NAME, hdr)
    assert m
    args = [a.strip() for a in m.group(1).split(",") if a.strip()]
    proto = L.PROTOTYPES[NAME][1]
    assert len(proto) == len(args)
    assert args[15].startswith("unsigned long long") and proto[15] is C.c_uint64   # the 64-bit seed
    assert args[12] == "float laf_th" and proto[12] is C.c_float
    # ag_homography_ransac's arguments with laf_th after inl_th
    assert proto[:12] + proto[13:] == L.PROTOTYPES["ag_homography_ransac"][1]


def test_refusals_before_any_cuda_call(L):
    """ag_homography_ransac's refusals, named after this entry point, and laf_th NaN or <= 0; the pointers are never dereferenced."""
    lib = L.lib()
    f = C.c_void_p(256)

    def call(l1=f, S1=2, cap1=10, l2=f, S2=2, cap2=10, pairs=None, P=2, tent=f, ntent=f, tcap=10, th=2.0, lth=2.0, conf=0.99, it=50000,
             outs=(f, f, f)):
        return lib.ag_homography_ransac_affine(l1, S1, cap1, l2, S2, cap2, pairs, P, tent, ntent, tcap, th, lth, conf, it, 0, *outs, None,
                                               None)

    def refused(rc, text):
        msg = lib.ag_last_error().decode()
        assert rc == -1 and msg.startswith(NAME) and text in msg, (rc, msg)

    for kw in (dict(l1=None), dict(l2=None), dict(tent=None), dict(ntent=None)):
        refused(call(**kw), "NULL")
    for kw in (dict(S1=0), dict(S2=0), dict(cap1=0), dict(cap2=-1), dict(P=0)):
        refused(call(**kw), "must be >= 1")
    refused(call(P=3), "S1 == S2 == P")
    for tcap in (0, 4194241):
        refused(call(tcap=tcap), "tcap must be in 1..4194240")
    for th in (0.0, float("nan"), float("inf")):
        refused(call(th=th), "inl_th")
    for lth in (0.0, -1.0, float("nan"), float("-inf")):
        refused(call(lth=lth), "laf_th")
    for conf in (0.0, 1.0):
        refused(call(conf=conf), "confidence")
    for it in (0, 0x7fffffff):
        refused(call(it=it), "max_iters")
    for k in range(3):
        refused(call(outs=tuple(None if q == k else f for q in range(3))), "NULL output")


def test_wrapper_refusals(L):
    from affnet_b200.ReprojectionStuff import AFFINE_LAF_TH, find_homography_pairs as fn
    lafs = torch.zeros(2, 5, 2, 3)
    tent = torch.zeros(2, 5, 2, dtype=torch.int32)
    nt = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(L.AffnetB200Error, match="needs affine=True"):
        fn(lafs, tent, nt, laf_th=2.0)
    for lth in (0.0, -1.0, float("nan")):
        with pytest.raises(L.AffnetB200Error, match="laf_th must be > 0"):
            fn(lafs, tent, nt, affine=True, laf_th=lth)
    with pytest.raises(L.AffnetB200Error, match="inl_th"):
        fn(lafs, tent, nt, inl_th=0.0, affine=True)
    for kw in (dict(affine=True), dict(affine=True, laf_th=float("inf"))):
        with pytest.raises(L.AffnetB200Error, match="must be a CUDA tensor"):
            fn(lafs, tent, nt, **kw)
    assert AFFINE_LAF_TH in (0.5, 1.0, 2.0, 4.0)


def exact_acs(seed, c1):
    """Two (or more) exact float64 ACs of a seeded homography at the image-1 centres c1 -> (s [1,k,12], Hm)."""
    Hm = AC.random_homography(seed)
    A1 = AC.random_frames(np.random.default_rng(seed), len(c1))
    A2 = AC.jacobian(Hm, c1) @ A1
    return np.concatenate([c1, project(Hm, c1), A1.reshape(-1, 4), A2.reshape(-1, 4)], 1)[None], Hm


@pytest.mark.parametrize("seed", range(8))
def test_solver_recovers_h_from_two_exact_acs(seed):
    r = np.random.default_rng(100 + seed)
    s, Hm = exact_acs(seed, np.stack([r.uniform(0, 1024, 2), r.uniform(0, 768, 2)], 1))
    H, ok = A.ac_homographies(s)
    assert ok[0]
    assert np.abs(H[0] - Hm.reshape(9)).max() <= 1e-9 * np.abs(Hm).max(), np.abs(H[0] - Hm.reshape(9)).max()


def base_sample():
    s, _ = exact_acs(3, np.array([[100.0, 200.0], [700.0, 500.0]]))
    return s.astype(np.float32).astype(np.float64)


@pytest.mark.parametrize("rule", ["centre_nan", "frame_inf", "coincident_1", "coincident_2", "det_a1", "det_a2", "mixed_sign", "pivot",
                                  "h_not_finite"])
def test_each_degeneracy_rule_fires(rule):
    s = base_sample()
    assert A.ac_homographies(s)[1][0]
    if rule == "centre_nan":
        s[0, 1, 2] = np.nan
    elif rule == "frame_inf":
        s[0, 0, 9] = np.inf
    elif rule == "coincident_1":
        s[0, 1, 0:2] = s[0, 0, 0:2]
    elif rule == "coincident_2":
        s[0, 1, 2:4] = s[0, 0, 2:4]
    elif rule == "det_a1":
        s[0, 1, 4:8] = (2.0, 4.0, 1.0, 2.0)
    elif rule == "det_a2":
        s[0, 0, 8:12] = (3.0, 6.0, 1.0, 2.0)
    elif rule == "mixed_sign":
        s[0, 1, 8:12] = s[0, 1, [9, 8, 11, 10]]             # A2's columns swapped: det(A2 A1^-1) changes sign for AC 1 only
    elif rule == "pivot":
        # both ACs: a nearly singular A1 and A2 = I, so A_n is huge and the h31 and h32 columns are nearly parallel
        a1 = np.float32([1, 1, 1, 1.0000001]).astype(np.float64)
        s[0, :, 4:8] = a1
        s[0, :, 8:12] = (1.0, 0.0, 0.0, 1.0)
        old = A.CHOL_EPS
        try:
            A.CHOL_EPS = 0.0
            assert A.ac_homographies(s)[1][0]                   # only the relative pivot threshold rejects it
        finally:
            A.CHOL_EPS = old
    elif rule == "h_not_finite":
        s[0, :, 0:4] = (1e200, 0.0, 0.0, 0.0), (-1e200, 1.0, 1.0, 1.0)   # finite float64, overflowing products
    assert not A.ac_homographies(s)[1][0], rule


def test_frame_distance_equals_the_frobenius_restatement():
    """D of the restatement (fp64) against frobenius_restated's skip-centre distance (fp32, pinned to the reference's golden) on the
    paired rows of constructed scenes: within that file's fp32 bound, and a singular or non-finite frame is never an inlier."""
    prm = FR.Params(skip_center=True)
    for seed, fo in ((0, 0.0), (1, 0.2), (2, 0.5)):
        l1, l2, Hm, kind = AC.scene(seed, 400, outliers=0.3, frame_outliers=fo)
        Hf = np.asarray(Hm, np.float32)
        ac = A.ac_rows(l1, l2).astype(np.float64)
        D, ok = A.frame_distance(Hf.astype(np.float64).reshape(9), ac)
        r, c = FR.rows(l1, prm), FR.cols(l2, Hf, prm)
        Df = np.diagonal(FR.distances(r, c, prm)).astype(np.float64)
        bound = np.diagonal(FR.d_bound(FR.distances(r, c, prm), r, c, prm))
        assert ok[0].all()
        err = np.abs(D[0] - Df)
        assert np.all(err <= bound + 1e-6 * (1.0 + D[0])), (seed, float(np.max(err - bound)))
        assert np.all(D[0][kind == AC.FRAME_OUTLIER] > 4.0)
    l1[3, :, :2] = 0.0
    l2[5, 0, 0] = np.nan
    D, ok = A.frame_distance(Hf.astype(np.float64).reshape(9), A.ac_rows(l1, l2).astype(np.float64))
    assert not ok[0, 3] and not ok[0, 5] and ok[0, 4]
    assert not A.inliers_ac(Hf.astype(np.float64).reshape(9), A.ac_rows(l1, l2).astype(np.float64), 4.0, math.inf)[0, [3, 5]].any()


@pytest.mark.parametrize("seed,outliers", [(20, 0.4), (21, 0.7), (22, 0.85)])
def test_restatement_finds_h_and_drops_the_frame_outliers(seed, outliers):
    """On constructed scenes with 5 % frame outliers: corner error < 1 px; every frame outlier is out of the affine mask at every
    admissible default, and the 4-point RANSAC keeps them."""
    l1, l2, Hm, kind = AC.scene(seed, 1000, outliers=outliers, frame_outliers=0.05)
    ac = A.ac_rows(l1, l2)
    fo = kind == AC.FRAME_OUTLIER
    _, m4, _, _ = R.ransac(ac[:, :4])
    assert m4[fo].mean() > 0.9
    for lth in (0.5, 1.0, 2.0, 4.0):
        H, m, n, it = A.ransac_ac(ac, laf_th=lth)
        assert corner_error(H, Hm) < 1.0 and not m[fo].any(), (lth, corner_error(H, Hm), int(m[fo].sum()))
        assert n >= 0.95 * (kind == AC.INLIER).sum()
    H, m, n, it = A.ransac_ac(ac, laf_th=math.inf)       # no frame threshold: only the finite frames are tested
    assert corner_error(H, Hm) < 1.0 and m[fo].mean() > 0.9


def test_fewer_samples_than_four_points_at_85_percent_outliers():
    l1, l2, Hm, kind = AC.scene(30, 1000, outliers=0.85)
    ac = A.ac_rows(l1, l2)
    _, _, n4, it4 = R.ransac(ac[:, :4])
    H, m, n, it = A.ransac_ac(ac)
    print("\n85 %% outliers: 2-AC %d inliers in %d samples, 4-point %d in %d" % (n, it, n4, it4))
    assert it < it4 and corner_error(H, Hm) < 1.0


def test_restatement_edge_cases():
    l1, l2, _, _ = AC.scene(5, 10, outliers=0.0)
    ac = A.ac_rows(l1, l2)
    for k in (0, 1):
        H, m, n, it = A.ransac_ac(ac[:k])
        assert n == 0 and it == 0 and not H.any() and len(m) == k
    l1, l2, _, _ = AC.scene(5, 2, outliers=0.0, eps=0.0, sigma=0.0)
    H, m, n, it = A.ransac_ac(A.ac_rows(l1, l2))          # two exact ACs: one hypothesis, too few inliers for a refit
    assert n == 2 and it == 256 and m.all()
    bad = ac.copy()
    bad[:, 4:8] = np.nan                                   # every sample degenerate: all max_iters hypotheses evaluated, nothing found
    H, m, n, it = A.ransac_ac(bad, max_iters=1000)
    assert n == 0 and it == 1000 and not m.any() and not H.any()


def test_pivot_scene_is_rejected_by_the_pivot_rule_only():
    """tests/affine_cases.pivot_scene (a GPU bits case): every sample of its first chunks is degenerate although no rule before the
    Cholesky applies, and with the relative pivot threshold at 0 a large share of them solves (the rest have a pivot <= 0)."""
    l1, l2 = AC.pivot_scene(11, 64)
    ac = A.ac_rows(l1, l2).astype(np.float64)
    idx, ok = A.samples2(0, np.arange(1024), len(ac))
    assert ok.all() and np.isfinite(ac).all()
    s = ac[idx]
    d1 = s[..., 4] * s[..., 7] - s[..., 5] * s[..., 6]
    d2 = s[..., 8] * s[..., 11] - s[..., 9] * s[..., 10]
    assert (d1 > 0).all() and (d2 > 0).all() and ((s[:, 0, 0:2] != s[:, 1, 0:2]).any(1) & (s[:, 0, 2:4] != s[:, 1, 2:4]).any(1)).all()
    assert not A.ac_homographies(s)[1].any()
    old = A.CHOL_EPS
    try:
        A.CHOL_EPS = 0.0
        assert A.ac_homographies(s)[1].mean() > 0.3
    finally:
        A.CHOL_EPS = old
    H, m, n, it = A.ransac_ac(A.ac_rows(l1, l2), max_iters=2000)
    assert n == 0 and it == 2000


def test_local_optimisation_lifts_a_noisy_winner():
    """On a constructed scene the shrinking-threshold refits start from the chunk's winner and never end below the refit rounds."""
    l1, l2, Hm, kind = AC.scene(40, 600, outliers=0.6, eps=0.15)
    ac = A.ac_rows(l1, l2).astype(np.float64)
    idx, ok = A.samples2(0, np.arange(256), len(ac))
    Hs, okh = A.ac_homographies(ac[idx])
    th2 = 4.0
    for k in np.nonzero(ok & okh)[0][:40]:
        _, _, c0 = A.local_opt(Hs[k], ac, th2, 0.5)
        _, _, c = A.search_lo(Hs[k], ac, th2, 0.5)
        assert c >= c0
