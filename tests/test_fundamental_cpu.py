"""CPU tests (-m "not gpu") of the fundamental-matrix RANSAC: the prototype of ag_fundamental_ransac and its host-side refusals (returned
before any CUDA call), the wrapper's refusals, the restated cubic root finder against numpy.roots, the 7-point solver on exact
correspondences, and the numpy restatement (tests/oracle_fransac.py) on seeded 3D scenes, against OpenCV's RANSAC where cv2 imports."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import fundamental_cases as FC
import oracle_fransac as FR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "ag_fundamental_ransac"


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
    assert L.PROTOTYPES[NAME][1][14] is C.c_uint64   # the seed is 64-bit
    assert L.PROTOTYPES[NAME] == L.PROTOTYPES["ag_homography_ransac"]


def test_refusals_before_any_cuda_call(L):
    """The pointers are never dereferenced: every refusal returns before a launch and names the entry point."""
    lib = L.lib()
    f = C.c_void_p(256)

    def call(l1=f, S1=2, cap1=10, l2=f, S2=2, cap2=10, pairs=None, P=2, tent=f, ntent=f, tcap=10, th=0.5, conf=0.99, it=50000,
             outs=(f, f, f)):
        return lib.ag_fundamental_ransac(l1, S1, cap1, l2, S2, cap2, pairs, P, tent, ntent, tcap, th, conf, it, 0, *outs, None, None)

    def refused(rc, text):
        msg = lib.ag_last_error().decode()
        assert rc == -1 and msg.startswith(NAME) and text in msg, (rc, msg)

    for kw in (dict(l1=None), dict(l2=None), dict(tent=None), dict(ntent=None)):
        refused(call(**kw), "NULL")
    for kw in (dict(S1=0), dict(S2=0), dict(cap1=0), dict(cap2=-1), dict(P=0), dict(pairs=f, P=-3)):
        refused(call(**kw), "must be >= 1")
    refused(call(S1=3, P=3), "S1 == S2 == P")
    refused(call(P=3), "S1 == S2 == P")
    for tcap in (0, -1, 4194241):
        refused(call(tcap=tcap), "tcap must be in 1..4194240")
    assert call(tcap=4194240, l1=None) == -1
    nan = float("nan")
    for th in (0.0, -1.0, nan, float("inf")):
        refused(call(th=th), "inl_th")
    for conf in (0.0, 1.0, -0.5, 1.5, nan):
        refused(call(conf=conf), "confidence")
    for it in (0, -5, 0x7fffffff):
        refused(call(it=it), "max_iters")
    for k in range(3):
        refused(call(outs=tuple(None if q == k else f for q in range(3))), "NULL output")


def test_wrapper_refusals(L):
    from affnet_b200.ReprojectionStuff import find_fundamental_pairs as fn
    lafs = torch.zeros(2, 5, 2, 3)
    tent = torch.zeros(2, 5, 2, dtype=torch.int32)
    nt = torch.zeros(2, dtype=torch.int32)
    cases = [
        (dict(lafs1=torch.zeros(2, 5, 6), tent=tent, ntent=nt), r"lafs1 must be \[S,cap,2,3\]"),
        (dict(lafs1=lafs, tent=tent, ntent=nt, lafs2=torch.zeros(5, 2, 3)), r"lafs2 must be \[S,cap,2,3\]"),
        (dict(lafs1=lafs, tent=tent[..., :1], ntent=nt), r"tent must be an integer tensor \[P,tcap,2\]"),
        (dict(lafs1=lafs, tent=tent.float(), ntent=nt), r"tent must be an integer tensor"),
        (dict(lafs1=lafs, tent=tent, ntent=nt[:1]), r"ntent must be an integer tensor \[2\]"),
        (dict(lafs1=lafs, tent=tent[:1], ntent=nt[:1]), "needs S1 == S2 == P"),
        (dict(lafs1=lafs, tent=tent, ntent=nt, pairs=torch.zeros(2, 3, dtype=torch.int32)), r"pairs must be an integer"),
        (dict(lafs1=lafs, tent=tent, ntent=nt, inl_th=0.0), "inl_th"),
        (dict(lafs1=lafs, tent=tent, ntent=nt, inl_th=float("inf")), "inl_th"),
        (dict(lafs1=lafs, tent=tent, ntent=nt, confidence=1.0), "confidence"),
        (dict(lafs1=lafs, tent=tent, ntent=nt, max_iters=0), "max_iters"),
        (dict(lafs1=lafs, tent=torch.zeros(2, 0, 2, dtype=torch.int32), ntent=nt), "tcap must be in 1..4194240"),
        (dict(lafs1=lafs, tent=tent, ntent=nt), "must be a CUDA tensor"),
    ]
    for kw, text in cases:
        with pytest.raises(L.AffnetB200Error, match=text) as e:
            fn(**kw)
        assert "must be a CUDA tensor" in text or str(e.value).startswith("find_fundamental_pairs: "), str(e.value)


def _real_numpy_roots(c):
    r = np.roots(c)
    return np.sort(r[np.abs(r.imag) <= 1e-7 * np.maximum(1.0, np.abs(r))].real)


def test_cubic_roots_against_numpy():
    rng = np.random.default_rng(0)
    seen = {1: 0, 3: 0}
    for _ in range(400):
        c = rng.normal(size=4) * 10.0 ** rng.uniform(-3, 3, 4)
        got = FR.cubic_roots(*c)
        ref = _real_numpy_roots(c)
        assert got == sorted(got)
        assert len(got) == len(ref), (c, got, ref)
        assert np.allclose(got, ref, rtol=1e-9, atol=1e-12 * max(1.0, float(np.max(np.abs(ref))))), (c, got, ref)
        seen[len(got)] += 1
    assert seen[1] > 50 and seen[3] > 20, seen
    # three known real roots, scaled
    for r in ([-3.0, 0.5, 7.0], [-1e-3, 2e-3, 5.0], [10.0, 20.0, 30.0]):
        c = 2.5 * np.poly(r)
        assert np.allclose(FR.cubic_roots(*c), r, rtol=1e-12, atol=1e-12)
    # a double root (x - 1)^2 (x + 2), at a critical point: -2 and 1, each once (a double root is found to ~sqrt(eps) only)
    got = FR.cubic_roots(1.0, 0.0, -3.0, 2.0)
    assert len(got) == 2 and abs(got[0] + 2.0) < 1e-12 and abs(got[1] - 1.0) < 1e-7, got
    # a triple root: one root
    assert np.allclose(FR.cubic_roots(1.0, -3.0, 3.0, -1.0), [1.0], atol=1e-5)
    # a zero leading coefficient: quadratic, linear, none
    assert np.allclose(FR.cubic_roots(0.0, 2.0, -2.0, -12.0), [-2.0, 3.0], rtol=1e-15)
    assert FR.cubic_roots(0.0, 1.0, 0.0, 1.0) == []
    assert FR.cubic_roots(0.0, 1.0, -2.0, 1.0) == [1.0]
    assert FR.cubic_roots(0.0, 0.0, 4.0, -2.0) == [0.5]
    assert FR.cubic_roots(0.0, 0.0, 0.0, 1.0) == []
    assert FR.cubic_roots(1.0, float("nan"), 0.0, 0.0) == []


def _normalised(pts):
    """Hartley normalisation of pts [n,4] fp64 as the restatement computes it -> (u [n,4], T)."""
    c1, c2 = pts[:, :2].mean(0), pts[:, 2:].mean(0)
    s1 = np.sqrt(2.0 / np.mean(np.sum((pts[:, :2] - c1) ** 2, 1)))
    s2 = np.sqrt(2.0 / np.mean(np.sum((pts[:, 2:] - c2) ** 2, 1)))
    u = np.concatenate([(pts[:, :2] - c1) * s1, (pts[:, 2:] - c2) * s2], 1)
    return u, (c1[0], c1[1], s1, c2[0], c2[1], s2)


def test_seven_point_on_exact_correspondences():
    """Noise-free float64 correspondences of 200 seeded 3D scenes: one model equals the true F up to scale, in the solver's normalised
    coordinates, to 1e-9 of its norm, and every model meets the 7 epipolar constraints and has det ~ 0."""
    errs = []
    for seed in range(200):
        rng = np.random.default_rng(seed)
        K, R, t = FC.motion(seed + 1050)
        x1 = np.stack([rng.uniform(0, 1024, 7), rng.uniform(0, 768, 7)], 1)
        X = np.concatenate([x1, np.ones((7, 1))], 1) @ np.linalg.inv(K).T * rng.uniform(4, 12, 7)[:, None]
        p = (X @ R.T + t) @ K.T
        pts = np.concatenate([x1, p[:, :2] / p[:, 2:3]], 1)
        Ft = FC.true_f(K, R, t)
        u, T = _normalised(pts)
        Fn, ok = FR.seven_point(u[None])
        models = Fn[0][ok[0]]
        assert len(models), seed
        assert FR.denormalise_f(T, models)[1].all()
        T1, T2t = FR.hartley_mats(T)
        Ftn = (np.linalg.inv(T2t.reshape(3, 3)) @ Ft @ np.linalg.inv(T1.reshape(3, 3))).reshape(9)
        Ftn /= np.linalg.norm(Ftn)
        e = min(min(np.abs(F / np.linalg.norm(F) - Ftn).max(), np.abs(F / np.linalg.norm(F) + Ftn).max()) for F in models)
        errs.append(e)
        assert e < 1e-9, (seed, e)
        for F in models:
            res = [u[i, 2] * (F[0] * u[i, 0] + F[1] * u[i, 1] + F[2]) + u[i, 3] * (F[3] * u[i, 0] + F[4] * u[i, 1] + F[5])
                   + F[6] * u[i, 0] + F[7] * u[i, 1] + F[8] for i in range(7)]
            assert np.max(np.abs(res)) < 1e-12 * np.linalg.norm(F), (seed, res)
            assert abs(np.linalg.det(F.reshape(3, 3))) < 1e-11 * np.linalg.norm(F) ** 3, seed
    print("\n7-point on 200 exact scenes: largest error of the true model %.1e (median %.1e)" % (max(errs), float(np.median(errs))))


def test_seven_point_degenerate_samples():
    """Duplicated and collinear samples have rank < 7: no model."""
    u = np.tile(np.array([[0.1, 0.2, 0.3, 0.4]]), (7, 1))
    assert not FR.seven_point(u[None])[1].any()
    x = np.linspace(-1, 1, 7)
    u = np.stack([x, 2 * x + 0.1, 0.5 * x - 0.2, -x], 1)
    assert not FR.seven_point(u[None])[1].any()


@pytest.mark.parametrize("n", [200, 2000])
def test_restatement_recovers_a_scene(n):
    """40 % uniform outliers, 0.3 px noise, inl_th = 1 px: >= 95 % of the true inliers and <= 2 % of the outliers marked, median Sampson
    error of the true inliers under the estimate < 0.5 px; cv2's RANSAC on the same scene is printed when cv2 imports."""
    pts, out, Ft = FC.scene(7 + n, n)
    F, m, k, it = FR.ransac_f(pts, 1.0, 0.99, 50000, 0)
    tin = ~out
    med = float(np.median(FR.sampson(F, pts[tin])))
    print("\nrestatement n=%d: %d inliers (%d true), %d samples, %.3f of the true inliers, %.4f of the outliers, median Sampson %.3f px"
          % (n, k, tin.sum(), it, m[tin].mean(), m[out].mean(), med))
    assert k == m.sum() and m[tin].mean() >= 0.95 and m[out].mean() <= 0.02 and med < 0.5 and it < 50000
    assert abs(np.linalg.norm(F) - 1.0) < 1e-6 and F.flat[np.argmax(np.abs(F))] > 0
    try:
        import cv2
    except ImportError:
        pytest.skip("cv2 not importable: the OpenCV comparison is skipped")
    Fc, mc = cv2.findFundamentalMat(pts[:, :2], pts[:, 2:], cv2.FM_RANSAC, 1.0, 0.99, 50000)
    mc = mc.ravel().astype(bool)
    print("cv2.findFundamentalMat(FM_RANSAC, 1.0): %d inliers, %.3f of the true inliers, median Sampson %.3f px"
          % (mc.sum(), mc[tin].mean(), float(np.median(FR.sampson(Fc[:3], pts[tin])))))


def test_restatement_edge_cases():
    F, m, k, it = FR.ransac_f(np.zeros((6, 4), np.float32))
    assert k == 0 and it == 0 and not m.any() and not F.any()
    # every row on one point: no normalisation, no sample drawn
    F, m, k, it = FR.ransac_f(np.tile(np.array([[1.0, 2.0, 3.0, 4.0]], np.float32), (20, 1)))
    assert k == 0 and it == 0 and not F.any()
    # all points on one line in both images: every sample is degenerate, all max_iters samples are evaluated
    x = np.arange(40, dtype=np.float32) * 10
    F, m, k, it = FR.ransac_f(np.stack([x, 2 * x + 5, x + 3, np.full_like(x, 7.0)], 1), max_iters=1000)
    assert k == 0 and it == 1000 and not m.any() and not F.any()
    # NaN rows are never inliers, and do not stop the others being found
    pts, out, _ = FC.scene(5, 300, outliers=0.0)
    pts[::10, 1] = np.nan
    F, m, k, it = FR.ransac_f(pts, 1.0)
    assert not m[::10].any() and k >= 0.95 * 270


def test_restatement_stopping_rule_at_a_tiny_inlier_ratio():
    """12000 uniform random correspondences: (best/n)^7 < 2^-54, so 1 - (best/n)^7 rounds to 1 and log(1 - (best/n)^7) would be 0.  No
    sample count then reaches the confidence: the search runs to max_iters."""
    rng = np.random.default_rng(1)
    n = 12000
    pts = np.stack([rng.uniform(0, 1024, n), rng.uniform(0, 768, n), rng.uniform(0, 1024, n), rng.uniform(0, 768, n)], 1).astype(np.float32)
    F, m, k, it = FR.ransac_f(pts, 0.5, 0.99, 1024, 0)
    pr = k / n
    assert 0 < k and 1.0 - pr * pr * pr * pr * pr * pr * pr == 1.0 and it == 1024, (k, it)
