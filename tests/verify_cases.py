"""Fixtures shared by the CPU and GPU tests of the device verification (ag_homography_ransac, ag_gt_correspondences_pairs): seeded
homographies, correspondences around them, and the corner error used to judge an estimate."""
import numpy as np


def random_homography(seed, H=768, W=1024, max_deg=20.0, scale=(0.8, 1.1), persp=1e-4):
    """A homography about the image centre: rotation up to max_deg, isotropic scale in `scale`, perspective terms ~persp."""
    r = np.random.default_rng(seed)
    a = np.deg2rad(r.uniform(-max_deg, max_deg))
    s = r.uniform(*scale)
    c = np.array([[1, 0, W / 2], [0, 1, H / 2], [0, 0, 1.0]])
    ci = np.array([[1, 0, -W / 2], [0, 1, -H / 2], [0, 0, 1.0]])
    R = np.array([[s * np.cos(a), -s * np.sin(a), r.uniform(-20, 20)], [s * np.sin(a), s * np.cos(a), r.uniform(-20, 20)],
                  [r.uniform(-persp, persp), r.uniform(-persp, persp), 1.0]])
    Hm = c @ R @ ci
    return Hm / Hm[2, 2]


def project(Hm, xy):
    p = np.concatenate([xy, np.ones((len(xy), 1))], 1) @ Hm.T
    return p[:, :2] / p[:, 2:3]


def correspondences(seed, n, Hm, outliers=0.4, sigma=0.3, H=768, W=1024):
    """[n,4] float32 (x1, y1, x2, y2): image-1 points uniform in the frame, mapped by Hm with N(0, sigma) noise; a fraction `outliers`
    of the rows gets a uniform image-2 point instead.  Also returns the outlier mask."""
    r = np.random.default_rng(seed)
    x1 = np.stack([r.uniform(0, W, n), r.uniform(0, H, n)], 1)
    x2 = project(Hm, x1) + r.normal(0, sigma, (n, 2))
    out = r.random(n) < outliers
    x2[out] = np.stack([r.uniform(0, W, out.sum()), r.uniform(0, H, out.sum())], 1)
    return np.concatenate([x1, x2], 1).astype(np.float32), out


def corner_error(Ha, Hb, H=768, W=1024):
    """Largest distance between the images of the frame's corners under Ha and Hb (px)."""
    c = np.array([[0, 0], [W, 0], [W, H], [0, H]], dtype=np.float64)
    return float(np.max(np.linalg.norm(project(np.asarray(Ha, np.float64), c) - project(np.asarray(Hb, np.float64), c), axis=1)))
