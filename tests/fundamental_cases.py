"""Seeded two-view scenes for the fundamental-matrix RANSAC (ag_fundamental_ransac and its restatement tests/oracle_fransac.py): 3D
points in front of two pinhole cameras (K, R, t) with pixel noise and uniform outliers, a planar scene and a two-plane scene, each with
its true F (pixel coordinates, unit Frobenius norm)."""
import numpy as np

H_IMG, W_IMG = 768, 1024


def intrinsics(f=800.0, H=H_IMG, W=W_IMG):
    return np.array([[f, 0.0, W / 2], [0.0, f, H / 2], [0.0, 0.0, 1.0]])


def rotation(rng, max_deg):
    """A rotation about a random axis by up to max_deg."""
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    a = np.deg2rad(rng.uniform(-max_deg, max_deg))
    Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx


def motion(seed, max_deg=8.0, baseline=0.5):
    """(K, R, t) of camera 2 relative to camera 1 (X2 = R X1 + t): a seeded rotation and a mostly sideways baseline."""
    rng = np.random.default_rng(seed)
    R = rotation(rng, max_deg)
    t = np.array([rng.uniform(0.6, 1.0) * rng.choice([-1, 1]), rng.uniform(-0.3, 0.3), rng.uniform(-0.2, 0.2)])
    return intrinsics(), R, baseline * t / np.linalg.norm(t)


def true_f(K, R, t):
    """F = K^-T [t]x R K^-1, unit Frobenius norm, its largest-magnitude entry positive."""
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    Ki = np.linalg.inv(K)
    F = Ki.T @ tx @ R @ Ki
    F /= np.linalg.norm(F)
    return F if F.flat[np.argmax(np.abs(F))] > 0 else -F


def plane_homography(K, R, t, n, d):
    """Homography image 1 -> image 2 induced by the plane n.X = d (camera-1 frame): K (R + t n^T / d) K^-1."""
    return K @ (R + np.outer(t, n) / d) @ np.linalg.inv(K)


def _project(K, X):
    p = X @ K.T
    return p[:, :2] / p[:, 2:3]


def _finish(rng, x1, X, K, R, t, n, outliers, sigma, H, W):
    x2 = _project(K, X @ R.T + t) + rng.normal(0, sigma, (n, 2))
    x1 = x1 + rng.normal(0, sigma, (n, 2))
    out = rng.random(n) < outliers
    x2[out] = np.stack([rng.uniform(0, W, out.sum()), rng.uniform(0, H, out.sum())], 1)
    return np.concatenate([x1, x2], 1).astype(np.float32), out, true_f(K, R, t)


def scene(seed, n, outliers=0.4, sigma=0.3, depth=(4.0, 12.0), H=H_IMG, W=W_IMG):
    """-> (pts [n,4] float32 (x1, y1, x2, y2), outlier mask, F true): image-1 pixels uniform in the frame at depths uniform in `depth`,
    seen by both cameras; N(0, sigma) noise in both images; a fraction `outliers` of the rows gets a uniform image-2 point."""
    rng = np.random.default_rng(seed)
    K, R, t = motion(seed + 1000)
    x1 = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1)
    z = rng.uniform(*depth, n)
    X = np.concatenate([x1, np.ones((n, 1))], 1) @ np.linalg.inv(K).T * z[:, None]
    return _finish(rng, x1, X, K, R, t, n, outliers, sigma, H, W)


def plane_scene(seed, n, depths=(6.0,), outliers=0.4, sigma=0.3, H=H_IMG, W=W_IMG):
    """As scene(), with every point on a fronto-parallel plane: one depth (a planar scene, where F is not determined by the points) or
    two (left half of image 1 on the first plane, right half on the second)."""
    rng = np.random.default_rng(seed)
    K, R, t = motion(seed + 1000)
    x1 = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1)
    z = np.where(x1[:, 0] < W / 2, depths[0], depths[-1])
    X = np.concatenate([x1, np.ones((n, 1))], 1) @ np.linalg.inv(K).T * z[:, None]
    return _finish(rng, x1, X, K, R, t, n, outliers, sigma, H, W)
