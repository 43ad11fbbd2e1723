"""CPU tests (-m "not gpu") of the device verification: the host-side refusals of ag_homography_ransac and ag_gt_correspondences_pairs
(returned before any CUDA call) and of their Python wrappers, known answers of the restated sampler, and the numpy restatement
(tests/oracle_ransac.py) recovering a homography, against OpenCV's RANSAC where cv2 imports."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

import oracle_ransac as R
from verify_cases import corner_error, correspondences, random_homography

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("ag_homography_ransac", "ag_gt_correspondences_pairs")


@pytest.fixture(scope="module")
def L():
    import affnet_b200._lib as lib
    if not os.path.isfile(lib.LIB_PATH):
        lib.build()
    lib.lib()
    return lib


def test_new_prototypes_match_the_header(L):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "affnet_b200.h")).read(), flags=re.S)
    for name in NEW:
        m = re.search(r"\bint\s+%s\s*\(([^;]*)\)\s*;" % name, hdr)
        assert m, name
        nargs = len([a for a in m.group(1).split(",") if a.strip()])
        assert len(L.PROTOTYPES[name][1]) == nargs, name
    assert L.PROTOTYPES["ag_homography_ransac"][1][14] is C.c_uint64   # the seed is 64-bit


def test_refusals_before_any_cuda_call(L):
    """The pointers are never dereferenced: every refusal returns before a launch and names the entry point."""
    lib = L.lib()
    f = C.c_void_p(256)

    def ransac(l1=f, S1=2, cap1=10, l2=f, S2=2, cap2=10, pairs=None, P=2, tent=f, ntent=f, tcap=10, th=2.0, conf=0.99, it=50000,
               outs=(f, f, f)):
        return lib.ag_homography_ransac(l1, S1, cap1, l2, S2, cap2, pairs, P, tent, ntent, tcap, th, conf, it, 0, *outs, None, None)

    def gt(l1=f, S1=2, cap1=10, l2=f, S2=2, cap2=10, pairs=None, P=2, tent=f, ntent=f, tcap=10, H=f, th=6.0, outs=(f, f, f, f)):
        return lib.ag_gt_correspondences_pairs(l1, S1, cap1, l2, S2, cap2, pairs, P, tent, ntent, tcap, H, th, *outs, None)

    def refused(rc, name, text):
        msg = lib.ag_last_error().decode()
        assert rc == -1 and msg.startswith(name) and text in msg, (rc, msg)

    for fn, name in ((ransac, NEW[0]), (gt, NEW[1])):
        for kw in (dict(l1=None), dict(l2=None), dict(tent=None), dict(ntent=None)):
            refused(fn(**kw), name, "NULL")
        for kw in (dict(S1=0), dict(S2=0), dict(cap1=0), dict(cap2=-1), dict(P=0), dict(pairs=f, P=-3)):
            refused(fn(**kw), name, "must be >= 1")
        refused(fn(S1=3, P=3), name, "S1 == S2 == P")
        refused(fn(P=3), name, "S1 == S2 == P")
        for tcap in (0, -1, 4194241):
            refused(fn(tcap=tcap), name, "tcap must be in 1..4194240")
        assert fn(tcap=4194240, l1=None) == -1    # the largest tcap passes that check (the NULL is refused instead)
    nan = float("nan")
    for th in (0.0, -1.0, nan, float("inf")):
        refused(ransac(th=th), NEW[0], "inl_th")
    for conf in (0.0, 1.0, -0.5, 1.5, nan):
        refused(ransac(conf=conf), NEW[0], "confidence")
    for it in (0, -5):
        refused(ransac(it=it), NEW[0], "max_iters")
    for k in range(3):
        refused(ransac(outs=tuple(None if q == k else f for q in range(3))), NEW[0], "NULL output")
    for th in (-0.5, nan):
        refused(gt(th=th), NEW[1], "dist_threshold")
    refused(gt(H=None), NEW[1], "NULL")
    for k in range(4):
        refused(gt(outs=tuple(None if q == k else f for q in range(4))), NEW[1], "NULL")


def test_wrapper_refusals(L):
    from affnet_b200.ReprojectionStuff import find_homography_pairs, get_GT_correspondence_indexes, gt_correspondences_pairs
    lafs = torch.zeros(2, 5, 2, 3)
    tent = torch.zeros(2, 5, 2, dtype=torch.int32)
    nt = torch.zeros(2, dtype=torch.int32)
    cases = [
        (find_homography_pairs, dict(lafs1=torch.zeros(2, 5, 6), tent=tent, ntent=nt), r"lafs1 must be \[S,cap,2,3\]"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, lafs2=torch.zeros(5, 2, 3)), r"lafs2 must be \[S,cap,2,3\]"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent[..., :1], ntent=nt), r"tent must be an integer tensor \[P,tcap,2\]"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent.float(), ntent=nt), r"tent must be an integer tensor"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent, ntent=nt[:1]), r"ntent must be an integer tensor \[2\]"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent[:1], ntent=nt[:1]), "needs S1 == S2 == P"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, pairs=torch.zeros(2, 3, dtype=torch.int32)), r"pairs must be an integer"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, inl_th=0.0), "inl_th"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, confidence=1.0), "confidence"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, max_iters=0), "max_iters"),
        (find_homography_pairs, dict(lafs1=lafs, tent=torch.zeros(2, 0, 2, dtype=torch.int32), ntent=nt), "tcap must be in 1..4194240"),
        (find_homography_pairs, dict(lafs1=lafs, tent=tent, ntent=nt), "must be a CUDA tensor"),
        (gt_correspondences_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=torch.eye(3)[None]), r"H1to2 must be \[P,3,3\] or \[3,3\]"),
        (gt_correspondences_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=torch.eye(3), dist_threshold=float("nan")), "dist_threshold"),
        (gt_correspondences_pairs, dict(lafs1=lafs, tent=tent, ntent=nt, H1to2=torch.eye(3)), "must be a CUDA tensor"),
        (get_GT_correspondence_indexes, dict(LAFs1=torch.zeros(3, 2, 3), LAFs2=torch.zeros(4, 2, 3), H1to2=torch.eye(3)), "same number of rows"),
        (get_GT_correspondence_indexes, dict(LAFs1=torch.zeros(3, 6), LAFs2=torch.zeros(3, 2, 3), H1to2=torch.eye(3)), r"LAFs1 must be \[n,2,3\]"),
        (get_GT_correspondence_indexes, dict(LAFs1=torch.zeros(3, 2, 3), LAFs2=torch.zeros(3, 2, 3), H1to2=torch.eye(3)), "must be a CUDA tensor"),
    ]
    for fn, kw, text in cases:
        with pytest.raises(L.AffnetB200Error, match=text):
            fn(**kw)


def test_sampler_known_answers():
    # splitmix64's published first outputs from state 0 (state advances by the golden gamma)
    assert R.splitmix64(0) == 0xE220A8397B1DCDAF
    assert R.splitmix64(0x9E3779B97F4A7C15) == 0x6E789E6AA1B965F4
    x = np.array([0, 1, 0x9E3779B97F4A7C15, (7 << 32) | 3, (1 << 64) - 1], dtype=np.uint64)
    assert [int(v) for v in R.splitmix64(x)] == [R.splitmix64(int(v)) for v in x]
    # draw d of hypothesis h: high 32 bits of splitmix64(splitmix64((h << 32) | d) ^ seed) scaled by n
    for seed, h, n in ((0, 0, 1000), (12345, 77, 4), (2 ** 64 - 1, 49999, 4194240)):
        dr = R.draw_indices(seed, [h], n)[0]
        for d in (0, 1, 63):
            r = R.splitmix64(R.splitmix64((h << 32) | d) ^ seed)
            assert int(dr[d]) == ((r >> 32) * n) >> 32
    idx, ok = R.samples(0, np.arange(1024), 1000)
    assert ok.all() and (idx >= 0).all() and (idx < 1000).all()
    assert all(len(set(r)) == 4 for r in idx.tolist())
    assert idx[:2].tolist() == [[int(v) for v in R.draw_indices(0, [h], 1000)[0][:4]] for h in (0, 1)]   # no repeats there
    # n = 4: every sample is a permutation of 0..3; the seed changes the draws
    idx, ok = R.samples(5, np.arange(256), 4)
    assert ok.all() and all(sorted(r) == [0, 1, 2, 3] for r in idx.tolist())
    assert not np.array_equal(R.draw_indices(1, np.arange(8), 1000), R.draw_indices(2, np.arange(8), 1000))


def test_block_sum_order_is_a_sum():
    x = np.random.default_rng(0).normal(size=(1000, 3))
    assert np.allclose(R.block_sum(x), x.sum(0), rtol=1e-12, atol=1e-12)


def test_restatement_edge_cases():
    H, m, n, it = R.ransac(np.zeros((3, 4), np.float32))
    assert n == 0 and it == 0 and not m.any() and not H.any()
    # all points on one line: every sample is degenerate, all max_iters hypotheses are evaluated
    x = np.arange(40, dtype=np.float32) * 10
    pts = np.stack([x, np.full_like(x, 5.0), x + 3, np.full_like(x, 7.0)], 1)
    H, m, n, it = R.ransac(pts, max_iters=1000)
    assert n == 0 and it == 1000 and not m.any() and not H.any()
    # exact correspondences: everything is an inlier and the search stops after the first chunk
    Hm = random_homography(3)
    pts, _ = correspondences(4, 200, Hm, outliers=0.0, sigma=0.0)
    H, m, n, it = R.ransac(pts)
    assert n == 200 and it == 256 and corner_error(H, Hm) < 1e-2


def test_restatement_recovers_a_warped_pair():
    """40 % uniform outliers around a seeded homography with 0.3 px noise; cv2's RANSAC at 2 px, when it imports, finds as many inliers
    within 5 %."""
    Hm = random_homography(11)
    pts, out = correspondences(12, 1000, Hm)
    H, m, n, it = R.ransac(pts, 2.0, 0.99, 50000, 0)
    err = corner_error(H, Hm)
    print("\nrestatement: %d inliers of 1000 (%d true inliers), %d iterations, corner error %.3f px" % (n, (~out).sum(), it, err))
    assert err < 1.0 and n == m.sum() and n >= 0.95 * (~out).sum() and it < 50000
    assert (m & out).sum() < 0.02 * out.sum()
    try:
        import cv2
    except ImportError:
        pytest.skip("cv2 not importable: the OpenCV comparison is skipped")
    Hc, mc = cv2.findHomography(pts[:, :2], pts[:, 2:], cv2.RANSAC, 2.0, maxIters=50000, confidence=0.99)
    nc = int(mc.sum())
    print("cv2.findHomography(RANSAC, 2.0): %d inliers, corner error %.3f px" % (nc, corner_error(Hc, Hm)))
    assert abs(n - nc) <= 0.05 * nc
