"""Seeded dominant-plane scenes for DEGENSAC (ag_fundamental_degensac and its restatement tests/oracle_degensac.py), built on the
cameras and finishing step of tests/fundamental_cases.py: most true matches on one fronto-parallel plane, a few off it, uniform
outliers and pixel noise, with the true F (pixel coordinates, unit Frobenius norm) and the off-plane rows."""
import numpy as np

from fundamental_cases import H_IMG, W_IMG, _finish, motion


def dominant_plane(seed, n, off=0.15, outliers=0.3, sigma=0.3, d=6.0, depths=(2.5, 20.0), H=H_IMG, W=W_IMG):
    """As fundamental_cases.scene(), with most points on the fronto-parallel plane at depth d and a fraction `off` of the rows at
    depths uniform in `depths` (a facade or a floor with a few points off it) -> (pts, outlier mask, F true, off-plane mask).  A
    7-point sample drawn from the plane is degenerate: every [e']x H explains the plane, whatever the epipole."""
    rng = np.random.default_rng(seed)
    K, R, t = motion(seed + 1000)
    x1 = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1)
    offp = rng.random(n) < off
    z = np.where(offp, rng.uniform(*depths, n), d)
    X = np.concatenate([x1, np.ones((n, 1))], 1) @ np.linalg.inv(K).T * z[:, None]
    pts, out, F = _finish(rng, x1, X, K, R, t, n, outliers, sigma, H, W)
    return pts, out, F, offp
