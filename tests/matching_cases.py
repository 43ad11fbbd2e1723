"""Constructed cases for the SNN matcher, the ground-truth check and RANSAC, aimed at the edges where their kernels could go wrong
unseen: tile and thread boundaries, ties, NaN / inf / signed zeros, cancellation, and decisions exactly on their thresholds.  Shared
by tests/test_matching_restated_cpu.py (which shows that the cases reach those edges) and tests/test_gpu_matching_exact.py."""
import numpy as np
import torch

import oracle_ransac as R
from verify_cases import correspondences, project, random_homography

SNN_DIMS = (1, 3, 15, 16, 17, 127, 128, 129, 256)
SNN_COUNTS = (1, 63, 64, 65, 129)           # n1 and n2: one row / column tile, its edge, and three tiles
SNN_CAP = max(SNN_COUNTS)
GT_SIZES = (1, 255, 256, 257, 2047, 2048, 2049, 4097)
TIE_COLS = (4, 9, 67, 128)                  # one descriptor in different threads and in column tiles 0, 1 and 2
BIG = 1000.0                                # norm of the near-duplicate rows: cancellation far below -1e-6


def snn_sets(D, seed=0):
    """(a, b): [SNN_CAP, D] fp32 tensors with the edges at fixed rows / columns; a count n uses the first n rows.
      rows / columns 0-3   ordinary unit descriptors
      4, 9, 67, 128 of b   one descriptor t (equal minima across threads and column tiles); a[4] is t slightly perturbed
      10-17                a[r] = BIG * v_r, b[r] = a[r] + 1e-4 noise: near-duplicates whose cancelled sum is NaN under the sqrt
      18-19                exact duplicates b[r] = a[r]: distance sqrt(1e-6f)
      30 / 31              a +0 row and a -0 row (b[30] = +0)
      32                   a[32] holds +inf, b[32] -inf
      33                   a[33] is NaN, b[33] has a NaN
      40-41                b[40] = a[40], b[41] near a[40], a[41] = b[41]: row 40's second-nearest column is masked
      70 (row)             equal to a[4]: ties for a row in the second row tile"""
    g = torch.Generator().manual_seed(1000 * D + seed)
    nrm = lambda x: torch.nn.functional.normalize(x, dim=-1)  # noqa: E731
    a, b = nrm(torch.randn(SNN_CAP, D, generator=g)), nrm(torch.randn(SNN_CAP, D, generator=g))
    t = nrm(torch.randn(D, generator=g))
    for c in TIE_COLS:
        b[c] = t
    a[4] = nrm(t + 1e-3 * torch.randn(D, generator=g))
    a[70] = a[4]
    for r in range(10, 18):
        a[r] = BIG * nrm(torch.randn(D, generator=g))
        b[r] = a[r] + 1e-4 * torch.randn(D, generator=g)
    b[18], b[19] = a[18], a[19]
    a[30], a[31], b[30] = 0.0, -0.0, 0.0
    a[32, 0], b[32, -1] = float("inf"), float("-inf")
    a[33], b[33, 0] = float("nan"), float("nan")
    b[40] = a[40]
    b[41] = nrm(a[40] + 0.05 * torch.randn(D, generator=g))
    a[41] = b[41]
    return a.contiguous(), b.contiguous()


def ratio_edge_row(q):
    """The row whose fp32 quotient min / (second + 1e-8) is finite and closest to 0.8: the ratio is then set to that quotient and to
    the next fp32 value toward 0, so one row's decision sits exactly on the edge."""
    qq = torch.where(torch.isfinite(q) & (q > 0), q, torch.full_like(q, float("inf")))
    return int(torch.argmin((qq - 0.8).abs()))


# ---- ground-truth check ----------------------------------------------------------------------------------------------------------------
def _mapped_pairs(n, Hm, seed, W=1024, H=768, noise=4.0):
    """n correspondences: image-1 centres uniform in the frame, image-2 centres Hm x + N(0, noise): about half within 6 px."""
    r = np.random.default_rng(seed)
    x1 = np.stack([r.uniform(0, W, n), r.uniform(0, H, n)], 1)
    x2 = project(Hm, x1) + r.normal(0, noise, (n, 2))
    return np.concatenate([x1, x2], 1).astype(np.float32)


def threshold_pts(dy):
    """Under identity H: row 0 maps (0, 0) to (3, 4 + dy), 5 px away when dy = 0 (3-4-5: near the origin every fp32 step is exact,
    so a dy of one ulp of 4 moves the distance by an ulp), then 40 rows in the frame, far from it."""
    row = np.array([[0, 0, 3, np.float32(4) + np.float32(dy)]], np.float32)
    return np.concatenate([row, _mapped_pairs(40, np.eye(3), 3) + np.float32(100)]).astype(np.float32)


def gt_cases():
    """name -> (pts [n,4] fp32 (x1, y1, x2, y2), H1to2 [3,3] fp32, threshold)."""
    cases = {}
    Hm = random_homography(41).astype(np.float32)
    I = np.eye(3, dtype=np.float32)
    for n in GT_SIZES:
        pts = _mapped_pairs(n, Hm.astype(np.float64), 50 + n)
        if n >= 255:
            pts[100:103] = pts[7]                     # duplicate image-2 centres (and rows): ties
            pts[200, 2:] = pts[5, 2:]
            pts[60, 0] = np.nan                       # a NaN centre in image 1 and one in image 2
            pts[61, 3] = np.nan
        cases["n%d" % n] = (pts, Hm, 6.0)
    f = np.float32
    ulp4 = float(np.nextafter(f(4), f(8)) - f(4))
    below5, above5 = float(np.nextafter(f(5), f(0))), float(np.nextafter(f(5), f(8)))
    for name, dy, th in (("at5", 0.0, 5.0), ("at5_th_below", 0.0, below5), ("at5_th_above", 0.0, above5), ("th0", 0.0, 0.0),
                         ("nearer", -ulp4, 5.0), ("nearer_th_below", -ulp4, below5), ("farther", ulp4, 5.0)):
        cases["identity_" + name] = (threshold_pts(dy), I, th)
    # H1to2^-1 = [[1,0,0],[0,1,0],[1/64,0,1]]: w = x/64 + 1 is 0 at x = -64 and negative left of it
    Hw = np.array([[1, 0, 0], [0, 1, 0], [-1 / 64, 0, 1]], np.float32)
    r = np.random.default_rng(9)
    pw = np.stack([r.uniform(-300, 300, 300), r.uniform(-200, 200, 300)], 1)
    pw[:4, 0] = (-64.0, -64.0, -100.0, -1000.0)
    pts = np.concatenate([pw + r.normal(0, 3, pw.shape), pw], 1).astype(np.float32)
    cases["horizon"] = (pts, Hw, 6.0)
    cases["singular"] = (_mapped_pairs(300, np.eye(3), 4), np.array([[1, 2, 3], [2, 4, 6], [0, 0, 1]], np.float32), 6.0)
    # large coordinates: |a|^2 ~ 1e8, so the fp32 cancellation is ~1 px^2
    Hl = random_homography(43, 6000, 8000).astype(np.float32)
    cases["large"] = (_mapped_pairs(2000, Hl.astype(np.float64), 44, W=8000, H=6000, noise=3.0), Hl, 6.0)
    return cases


# ---- RANSAC -----------------------------------------------------------------------------------------------------------------------------
GRID = 64.0                                  # spacing of the translation case's grid: a power of two keeps its arithmetic exact
TRANSLATION = (3 * GRID, 5 * GRID)
EDGE_TH = 2.0


def translation_edge(seed=0):
    """Image-1 centres on the grid GRID * (0..15) (in units of GRID the minimal solver's fp64 products are integers below 2^53, so a
    sample of exact rows gives the exact translation), image-2 centres translated by TRANSLATION: 100 exact rows, 6 rows EDGE_TH off in x (err == th^2,
    inliers by <=), 6 rows one fp32 ulp beyond that, 10 outliers.  Hypotheses with an edge row in their sample bend a little and can
    take in more rows, so the case runs with max_iters = 1 and its rows are ordered so that hypothesis 0 samples exact rows.  -> (pts, rows at th^2, rows one ulp beyond)."""
    r = np.random.default_rng(seed)
    grid = np.array([(x, y) for x in range(16) for y in range(16)], np.float32) * np.float32(GRID)
    p1 = grid[r.permutation(len(grid))[:122]]
    p2 = p1 + np.array(TRANSLATION, np.float32)
    p2[100:106, 0] += EDGE_TH
    p2[106:112, 0] = np.nextafter(p2[106:112, 0] + EDGE_TH, np.float32(np.inf))
    p2[112:] = r.uniform(0, 16 * GRID, (10, 2)).astype(np.float32)
    pts = np.concatenate([p1, p2], 1).astype(np.float32)
    order = r.permutation(len(pts))
    first = R.samples(0, [0], len(pts))[0][0]               # hypothesis 0 of seed 0 draws exact rows: it is the translation
    for k, pos in enumerate(first):
        if order[pos] >= 100:
            other = next(q for q in range(len(order)) if order[q] < 100 and q not in first)
            order[pos], order[other] = order[other], order[pos]
    inv = np.argsort(order)
    return pts[order], inv[100:106], inv[106:112]


def horizon_pairs(n=300, seed=12):
    """A homography whose horizon x = -256 crosses the frame: rows left of it map with w < 0 and are never inliers."""
    Hm = np.array([[1.0, 0.05, 10], [0.02, 1.0, -7], [1 / 256, 0, 1]])
    r = np.random.default_rng(seed)
    x1 = np.stack([r.uniform(-600, 600, n), r.uniform(-400, 400, n)], 1)
    p = np.concatenate([x1, np.ones((n, 1))], 1) @ Hm.T
    x2 = p[:, :2] / p[:, 2:3] + r.normal(0, 0.3, (n, 2))
    return np.concatenate([x1, x2], 1).astype(np.float32), p[:, 2] <= 0


def near_degenerate(n=60, seed=13):
    """Centres on a line up to 1e-4 px in both images: the collinearity test decides near its epsilon."""
    r = np.random.default_rng(seed)
    x = r.uniform(0, 500, n)
    y = 0.5 * x + 20 + r.normal(0, 1e-4, n)
    return np.stack([x, y, 1.1 * x + 3, 0.7 * y - 2 + r.normal(0, 1e-4, n)], 1).astype(np.float32)


REFIT_BREAK_SEED = 3     # correspondences(REFIT_BREAK_SEED, 400, ..., sigma=1.2): a refit round lowers the inlier count


def ransac_cases():
    """name -> (pts [n,4] fp32, max_iters, seed, inl_th)."""
    Hm = random_homography(61)
    cases = {"translation_edge": (translation_edge()[0], 1, 0, EDGE_TH)}
    cases["horizon"] = (horizon_pairs()[0], 50000, 0, 2.0)
    for n in (2047, 2048, 2049):
        cases["n%d" % n] = (correspondences(70 + n, n, Hm, outliers=0.5)[0], 50000, 0, 2.0)
    hard = correspondences(71, 500, Hm, outliers=0.8)[0]
    for it in (1, 255, 256, 257):
        cases["iters%d" % it] = (hard, it, 0, 2.0)
    cases["seed_max"] = (hard, 50000, 2 ** 64 - 1, 2.0)
    cases["seed_max_iters257"] = (hard, 257, 2 ** 64 - 1, 2.0)
    cases["refit_break"] = (correspondences(REFIT_BREAK_SEED, 400, Hm, outliers=0.3, sigma=1.2)[0], 50000, 0, 2.0)
    cases["near_degenerate"] = (near_degenerate(), 5000, 0, 2.0)
    return cases
