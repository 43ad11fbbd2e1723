"""CPU tests (-m "not gpu") of DEGENSAC (ag_fundamental_degensac and its numpy restatement tests/oracle_degensac.py): the prototype and
the host-side refusals, the degeneracy test and plane-and-parallax on exact correspondences, and the restatement on dominant-plane
scenes (against OpenCV's USAC_DEFAULT where cv2 imports), general scenes and the edge cases of the plain fundamental-matrix RANSAC."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import degensac_cases as DC
import fundamental_cases as FC
import oracle_degensac as DG
import oracle_fransac as FR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "ag_fundamental_degensac"


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
    assert len(L.PROTOTYPES[NAME][1]) == len([a for a in m.group(1).split(",") if a.strip()])
    assert L.PROTOTYPES[NAME] == L.PROTOTYPES["ag_fundamental_ransac"]


def test_refusals_before_any_cuda_call(L):
    """The refusals of ag_fundamental_ransac, named after this entry point; the pointers are never dereferenced."""
    lib = L.lib()
    f = C.c_void_p(256)

    def call(l1=f, S1=2, cap1=10, l2=f, S2=2, cap2=10, pairs=None, P=2, tent=f, ntent=f, tcap=10, th=0.5, conf=0.99, it=50000,
             outs=(f, f, f)):
        return lib.ag_fundamental_degensac(l1, S1, cap1, l2, S2, cap2, pairs, P, tent, ntent, tcap, th, conf, it, 0, *outs, None, None)

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
    for conf in (0.0, 1.0):
        refused(call(conf=conf), "confidence")
    for it in (0, 0x7fffffff):
        refused(call(it=it), "max_iters")
    for k in range(3):
        refused(call(outs=tuple(None if q == k else f for q in range(3))), "NULL output")


def test_wrapper_refusals(L):
    from affnet_b200.ReprojectionStuff import find_fundamental_pairs as fn
    lafs = torch.zeros(2, 5, 2, 3)
    tent = torch.zeros(2, 5, 2, dtype=torch.int32)
    nt = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(L.AffnetB200Error, match="inl_th"):
        fn(lafs, tent, nt, inl_th=0.0, degensac=True)
    with pytest.raises(L.AffnetB200Error, match="must be a CUDA tensor"):
        fn(lafs, tent, nt, degensac=True)


def exact_pair(seed, n_plane, n_off, d=6.0):
    """Noise-free float64 correspondences: n_plane points on the plane z = d, then n_off at depths 2.5-20 -> (pts [n,4], F, H true)."""
    rng = np.random.default_rng(seed)
    K, R, t = FC.motion(seed + 1000)
    n = n_plane + n_off
    x1 = np.stack([rng.uniform(0, FC.W_IMG, n), rng.uniform(0, FC.H_IMG, n)], 1)
    z = np.concatenate([np.full(n_plane, d), rng.uniform(2.5, 20.0, n_off)])
    X = np.concatenate([x1, np.ones((n, 1))], 1) @ np.linalg.inv(K).T * z[:, None]
    p = (X @ R.T + t) @ K.T
    return np.concatenate([x1, p[:, :2] / p[:, 2:3]], 1), FC.true_f(K, R, t).reshape(9), FC.plane_homography(K, R, t, np.array([0, 0, 1.0]), d)


def test_triplet_homography_maps_its_points():
    """The H from the true F and any 3 exact correspondences (on a plane or not: three points always span one) maps them to within
    1e-8 px (F's own rounding, at pixel coordinates and a nearly sideways baseline, puts the worst of 60 at a few 1e-9 px), and for 3
    points of the scene plane it is that plane's homography."""
    worst = 0.0
    for seed in range(20):
        pts, F, Ht = exact_pair(seed, 4, 4)
        e = DG.left_epipole(F)
        A = DG.skew_mul(e, F)
        for tri in ((0, 1, 2), (4, 5, 6), (1, 3, 7)):
            H = DG.triplet_homography(A, e, pts[list(tri)])
            assert H is not None
            q = pts[list(tri)]
            w = H[6] * q[:, 0] + H[7] * q[:, 1] + H[8]
            err = np.hypot((H[0] * q[:, 0] + H[1] * q[:, 1] + H[2]) / w - q[:, 2], (H[3] * q[:, 0] + H[4] * q[:, 1] + H[5]) / w - q[:, 3])
            worst = max(worst, float(err.max()))
            assert err.max() < 1e-8, (seed, tri, err)
            if tri == (0, 1, 2):
                assert np.abs(H - (Ht / Ht[2, 2]).reshape(9)).max() < 1e-9 * np.abs(H).max(), seed
    print("\ntriplet H on exact points: worst transfer error %.1e px" % worst)


def test_degeneracy_flags_five_coplanar_points():
    """A 7-point sample with 5 exact points on one plane (indices 0-4, so triplet {0,1,2} spans it) is H-degenerate; a sample of 7
    points at random depths is not."""
    thd2 = (DG.DEG_H_TH_FACTOR * 0.5) ** 2
    for seed in range(20):
        pts, F, _ = exact_pair(seed, 5, 2)
        H, k = DG.degenerate_h(F, pts, thd2)
        assert k >= DG.DEG_MIN_AGREE, (seed, k)
        assert FR.inliers_f(F, pts, 1e-12)[0].all()
        pts, F, _ = exact_pair(seed, 0, 7)
        H, k = DG.degenerate_h(F, pts, thd2)
        assert k < DG.DEG_MIN_AGREE, (seed, k)


def test_plane_and_parallax_on_exact_data():
    """Plane points and two off-plane points, the plane's H: F = [e']x H from the two equals the true F to 1e-9."""
    for seed in range(20):
        pts, Ft, Ht = exact_pair(seed, 20, 2)
        H = (Ht / Ht[2, 2]).reshape(9)
        F, ok = DG.plane_and_parallax(H, pts, np.array([20]), np.array([21]), np.array([True]))
        assert ok[0] and np.abs(F[0] - Ft).max() < 1e-9, (seed, np.abs(F[0] - Ft).max())


@pytest.mark.parametrize("seed", range(6))
def test_dominant_plane_recovers_the_off_plane_matches(seed):
    """600 correspondences, 30 % outliers, 0.3 px noise, 15 % of the true matches off the plane at depth 6: DEGENSAC marks >= 0.8 of
    the off-plane true matches and <= 2 % of the outliers, median Sampson error of the true matches < 0.5 px; not more than 0.1 below
    cv2's USAC_DEFAULT (degeneracy test and LO) where cv2 imports.  The plain RANSAC finds 3-32 % of them on these seeds."""
    pts, out, Ft, offp = DC.dominant_plane(seed, 600)
    tin = ~out
    F, m, k, it = DG.degensac_f(pts, 0.5, 0.99, 50000, 0)
    med = float(np.median(FR.sampson(F, pts[tin])))
    frac = float(m[tin & offp].mean())
    _, mp, _, _ = FR.ransac_f(pts, 0.5, 0.99, 50000, 0)
    print("\ndominant plane seed %d: %d inliers (%d true, %d off-plane), %d samples, %.3f of the off-plane matches (plain RANSAC %.3f), "
          "%.4f of the outliers, median Sampson %.3f px" % (seed, k, tin.sum(), (tin & offp).sum(), it, frac, mp[tin & offp].mean(),
                                                              m[out].mean(), med))
    assert k == m.sum() and frac >= 0.8 and m[out].mean() <= 0.02 and med < 0.5
    assert abs(np.linalg.norm(F) - 1.0) < 1e-6 and F.flat[np.argmax(np.abs(F))] > 0
    try:
        import cv2
    except ImportError:
        pytest.skip("cv2 not importable: the USAC comparison is skipped")
    Fc, mc = cv2.findFundamentalMat(pts[:, :2], pts[:, 2:], cv2.USAC_DEFAULT, 0.5, 0.99, 50000)
    mc = mc.ravel().astype(bool)
    print("cv2 USAC_DEFAULT: %d inliers, %.3f of the off-plane matches" % (mc.sum(), mc[tin & offp].mean()))
    assert frac >= mc[tin & offp].mean() - 0.1


@pytest.mark.parametrize("n", [200, 2000])
def test_restatement_recovers_a_scene(n):
    """The bounds of the plain RANSAC's general-scene test: >= 95 % of the true inliers, <= 2 % of the outliers, median Sampson < 0.5."""
    pts, out, Ft = FC.scene(7 + n, n)
    F, m, k, it = DG.degensac_f(pts, 1.0, 0.99, 50000, 0)
    tin = ~out
    med = float(np.median(FR.sampson(F, pts[tin])))
    print("\nDEGENSAC n=%d: %d inliers (%d true), %d samples, %.3f of the true inliers, %.4f of the outliers, median Sampson %.3f px"
          % (n, k, tin.sum(), it, m[tin].mean(), m[out].mean(), med))
    assert k == m.sum() and m[tin].mean() >= 0.95 and m[out].mean() <= 0.02 and med < 0.5 and it < 50000


def test_restatement_edge_cases():
    F, m, k, it = DG.degensac_f(np.zeros((6, 4), np.float32))
    assert k == 0 and it == 0 and not m.any() and not F.any()
    F, m, k, it = DG.degensac_f(np.tile(np.array([[1.0, 2.0, 3.0, 4.0]], np.float32), (20, 1)))
    assert k == 0 and it == 0 and not F.any()
    x = np.arange(40, dtype=np.float32) * 10
    F, m, k, it = DG.degensac_f(np.stack([x, 2 * x + 5, x + 3, np.full_like(x, 7.0)], 1), max_iters=1000)
    assert k == 0 and it == 1000 and not m.any() and not F.any()
    pts, out, _ = FC.scene(5, 300, outliers=0.0)
    pts[::10, 1] = np.nan
    F, m, k, it = DG.degensac_f(pts, 1.0)
    assert not m[::10].any() and k >= 0.95 * 270
    # a planar scene: every sample is degenerate, plane-and-parallax runs and the result is still a model of the plane's inliers
    pts, out, _ = FC.plane_scene(11, 500)
    tr = []
    F, m, k, it = DG.degensac_f(pts, trace=tr)
    assert tr and tr[0]["degenerate"] and k >= 0.9 * (~out).sum() and m[out].mean() <= 0.02
