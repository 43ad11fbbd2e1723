"""Constructed scenes with frames for the affine homography RANSAC (ag_homography_ransac_affine, tests/oracle_ac_ransac.py): affine
correspondences around a seeded homography (verify_cases.random_homography), outliers with random centres and frames, and frame outliers
whose centres agree with H but whose frames do not."""
import numpy as np

from verify_cases import project, random_homography

INLIER, OUTLIER, FRAME_OUTLIER = 0, 1, 2


def jacobian(Hm, xy):
    """[n,2,2] Jacobians of x -> Hm x at the points xy [n,2]."""
    p = np.concatenate([xy, np.ones((len(xy), 1))], 1) @ Hm.T
    w = p[:, 2]
    x2 = p[:, :2] / w[:, None]
    return (Hm[None, :2, :2] - x2[:, :, None] * Hm[None, 2:3, :2]) / w[:, None, None]


def rotation(a):
    c, s = np.cos(a), np.sin(a)
    return np.stack([np.stack([c, -s], -1), np.stack([s, c], -1)], -2)


def random_frames(r, n):
    """[n,2,2]: scale 5-40 px x rotation x anisotropy 1-3 (determinant scale^2)."""
    s = r.uniform(5.0, 40.0, n)
    k = r.uniform(1.0, 3.0, n)
    D = np.zeros((n, 2, 2))
    D[:, 0, 0], D[:, 1, 1] = np.sqrt(k), 1.0 / np.sqrt(k)
    return s[:, None, None] * rotation(r.uniform(-np.pi, np.pi, n)) @ D


def scene(seed, n, outliers=0.4, frame_outliers=0.0, eps=0.03, sigma=0.3, Hm=None, H=768, W=1024):
    """n affine correspondences -> (lafs1 [n,2,3] float32, lafs2 [n,2,3] float32, Hm, kind [n]).  Inliers: c2 = Hm(c1) + N(0, sigma),
    A2 = J_Hm(c1) A1 (I + E), E ~ N(0, eps).  A fraction `outliers` gets a random image-2 centre and an unrelated random frame; a fraction
    `frame_outliers` keeps the centre and gets A2 = J A1 R(100..180 deg) or J A1 diag(k, 1/k), k in 3..5, so that D > 4."""
    r = np.random.default_rng(seed)
    Hm = random_homography(seed) if Hm is None else Hm
    c1 = np.stack([r.uniform(40, W - 40, n), r.uniform(40, H - 40, n)], 1)
    c2 = project(Hm, c1) + r.normal(0, sigma, (n, 2))
    A1 = random_frames(r, n)
    J = jacobian(Hm, c1)
    A2 = J @ A1 @ (np.eye(2)[None] + r.normal(0, eps, (n, 2, 2)))
    u = r.random(n)
    kind = np.where(u < outliers, OUTLIER, np.where(u < outliers + frame_outliers, FRAME_OUTLIER, INLIER))
    o = kind == OUTLIER
    c2[o] = np.stack([r.uniform(0, W, o.sum()), r.uniform(0, H, o.sum())], 1)
    A2[o] = random_frames(r, int(o.sum()))
    f = np.nonzero(kind == FRAME_OUTLIER)[0]
    rot = r.random(len(f)) < 0.5
    k = r.uniform(3.0, 5.0, len(f))
    B = np.zeros((len(f), 2, 2))
    B[:, 0, 0], B[:, 1, 1] = k, 1.0 / k
    B[rot] = rotation(np.deg2rad(r.uniform(100.0, 180.0, int(rot.sum()))) * r.choice([-1.0, 1.0], int(rot.sum())))
    A2[f] = J[f] @ A1[f] @ B
    l1 = np.concatenate([A1, c1[:, :, None]], 2).astype(np.float32)
    l2 = np.concatenate([A2, c2[:, :, None]], 2).astype(np.float32)
    return l1, l2, Hm, kind


def pivot_scene(seed, n, H=768, W=1024):
    """n rows with distinct random centres, every image-1 frame the same nearly singular [[1, 1], [1, 1.0000001]] (float32) and every
    image-2 frame 100 I -> (lafs1, lafs2).  Each 2-AC sample then has a huge A_n, so the h31 and h32 columns of its system are nearly
    parallel: the solver's relative Cholesky pivot rule rejects it, and no other degeneracy rule applies (finite, non-singular frames of
    one orientation, distinct centres)."""
    r = np.random.default_rng(seed)
    l1, l2 = np.zeros((n, 2, 3), np.float32), np.zeros((n, 2, 3), np.float32)
    l1[:, :, :2] = np.float32([[1.0, 1.0], [1.0, 1.0000001]])
    l2[:, :, :2] = 100.0 * np.eye(2, dtype=np.float32)
    l1[:, :, 2] = np.stack([r.uniform(0, W, n), r.uniform(0, H, n)], 1)
    l2[:, :, 2] = np.stack([r.uniform(0, W, n), r.uniform(0, H, n)], 1)
    return l1, l2
