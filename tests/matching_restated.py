"""Exact restatements of the SNN matcher (affnet_b200/csrc/matching.cu) and of the ground-truth reprojection check (gt_kernel in
affnet_b200/csrc/verify.cu), operation by operation (test infrastructure, not product).

Every fp32 step is one float64 tensor operation whose result is rounded to fp32; float64 holds each fp32 sum, difference, product,
quotient and square root exactly enough for that rounding to be the correctly rounded fp32 result.  The fused multiply-adds are
`scale_space_restated.fmaf32`.  So the functions here run on the CPU or, for large cases, in float64 on the device, and a kernel that
differs from them in one bit is wrong.  No library kernel is called.

Next to them are float64 statements of the same formulas and per-element bounds, derived from the fp32 chains, on the squared
distance: the kernels and the reference (whose summation order depends on its BLAS and on the sizes) both lie within them."""
import math

import numpy as np
import torch

import oracle_ransac as R
from scale_space_restated import fmaf32

U32 = 2.0 ** -24                           # unit roundoff of fp32
U64 = 2.0 ** -53
EPS_SNN = float(np.float32(1e-6))          # the 1e-6 of distance_matrix_vector (Losses.py), an fp32 constant
EPS_RATIO = float(np.float32(1e-8))
EPS_GT = float(np.float32(1e-12))          # the 1e-12 of ReprojectionStuff.distance_matrix_vector
MASKED = 100000.0
INF = float("inf")


def _d(x):
    return x.to(torch.float64)


def _f(x):
    """Round float64 values to fp32: one fp32 operation's rounding."""
    return x.to(torch.float32)


def _t32(x, device=None):
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x))
    return x.to(device=device, dtype=torch.float32)


# ---- the matcher's distances --------------------------------------------------------------------------------------------------------
def fma_norms(x):
    """|x|^2 per row of x [n,D] fp32: acc = fmaf(x[k], x[k], acc) over k ascending from +0 (row_norms_kernel, dist_matrix_kernel)."""
    acc = torch.zeros(x.size(0), dtype=torch.float32, device=x.device)
    for k in range(x.size(1)):
        acc = fmaf32(x[:, k], x[:, k], acc)
    return acc


def fma_dots(a, b):
    """a.b for a [n1,D], b [n2,D] fp32 -> [n1,n2]: acc = fmaf(a[k], b[k], acc) over k ascending from +0.  The kernels' zero padding of
    k adds fmaf(0, 0, acc) = acc (acc is never -0), so it is left out."""
    acc = torch.zeros(a.size(0), b.size(0), dtype=torch.float32, device=a.device)
    for k in range(a.size(1)):
        acc = fmaf32(a[:, k:k + 1], b[None, :, k], acc)
    return acc


def snn_dist(na, nb, acc):
    """snn_dist: sqrtf(((na + nb) - 2 acc) + 1e-6f), each step rounded to fp32 (2 acc is rounded too: it overflows to inf)."""
    t = _f(_d(na)[:, None] + _d(nb)[None, :])
    t = _f(_d(t) - _d(_f(2.0 * _d(acc))))
    t = _f(_d(t) + EPS_SNN)
    return _f(torch.sqrt(_d(t)))


def distances(a, b, dots=fma_dots):
    """ag_distance_matrix / the matcher's per-element distance of a [n1,D] and b [n2,D] (tensors or arrays) -> fp32 [n1,n2].
    `dots` replaces the dot products (the tests pass other summation orders to show that the cases see them)."""
    a, b = _t32(a), _t32(b)
    b = b.to(a.device)
    return snn_dist(fma_norms(a), fma_norms(b), dots(a, b))


def distances_blocked(a, b, dev=None, rows=1024):
    """distances() in row blocks, on `dev` (float64 on the device for the large cases)."""
    a, b = _t32(a, dev), _t32(b, dev)
    nb = fma_norms(b)
    out = []
    for r0 in range(0, a.size(0), rows):
        x = a[r0:r0 + rows]
        out.append(snn_dist(fma_norms(x), nb, fma_dots(x, b)))
    return torch.cat(out)


def kblocked_dots(a, b, kb=16):
    """A split-K rewrite: an fmaf chain per k block of `kb`, the block partials added in order (a mutation, not the kernels)."""
    tot = None
    for k0 in range(0, a.size(1), kb):
        part = fma_dots(a[:, k0:k0 + kb], b[:, k0:k0 + kb])
        tot = part if tot is None else _f(_d(tot) + _d(part))
    return tot


def pairwise_dots(a, b):
    """Rounded products summed as a binary tree (a mutation, not the kernels)."""
    terms = [_f(_d(a[:, k:k + 1]) * _d(b[None, :, k])) for k in range(a.size(1))]
    while len(terms) > 1:
        nxt = [_f(_d(terms[i]) + _d(terms[i + 1])) for i in range(0, len(terms) - 1, 2)]
        terms = nxt + ([terms[-1]] if len(terms) % 2 else [])
    return terms[0]


# ---- the matcher's reductions -------------------------------------------------------------------------------------------------------
def snn_rows(dist, ratio=0.8, lowest=True, nan_ignored=True, le=True):
    """snn_pass_kernel's two passes and snn_compact_kernel on one pair's distances dist [n1,n2] fp32 ->
    (idx2 int64, min, second, keep bool, tent [ntent,2] int64).

    Pass 1: the minimum below +inf with NaN ignored and the lowest column among equal minima; min is the distance at that column;
    (+inf, column 0) for a row with nothing below +inf.  Every row's idx2 column is masked, column 0 included for such rows.  Pass 2:
    fminf over (masked ? 100000 : dist), NaN ignored, +inf when nothing is left.  keep = fl(min / fl(second + 1e-8f)) <= ratio (fp32).
    The keyword arguments select mutations: the highest column among equal minima, a NaN-propagating minimum, `<` for `<=`."""
    n1, n2 = dist.shape
    dev = dist.device
    nan = torch.isnan(dist)
    lt = torch.where(nan, INF, dist) if nan_ignored else dist
    mval = lt.min(1).values
    cols = torch.arange(n2, device=dev).expand(n1, n2)
    hit = (lt == mval[:, None]) & (lt < INF)
    if lowest:
        pick = torch.where(hit, cols, n2).min(1).values
    else:
        pick = torch.where(hit, cols, -1).max(1).values
    has = hit.any(1)
    idx2 = torch.where(has, pick, torch.zeros_like(pick))
    mn = torch.where(has, dist.gather(1, idx2[:, None])[:, 0], torch.full_like(mval, INF))
    if not nan_ignored:
        mn = torch.where(torch.isnan(mval), mval, mn)
    mask = torch.zeros(n2, dtype=torch.bool, device=dev)
    mask[idx2] = True
    sec = torch.where(mask[None, :], torch.full_like(dist, MASKED), dist)
    sec = torch.where(torch.isnan(sec), INF, sec).min(1).values
    q = _f(_d(mn) / _d(_f(_d(sec) + EPS_RATIO)))
    r = torch.tensor(float(np.float32(ratio)), dtype=torch.float32, device=dev)
    keep = (q <= r) if le else (q < r)
    rows = torch.arange(n1, device=dev)
    return idx2, mn, sec, keep, torch.stack([rows[keep], idx2[keep]], 1)


def ratio_quotients(dist):
    """fl(min / fl(second + 1e-8f)) per row: the value the ratio decision compares."""
    _, mn, sec, _, _ = snn_rows(dist)
    return _f(_d(mn) / _d(_f(_d(sec) + EPS_RATIO)))


# ---- float64 statement and bound of the matcher's distance ---------------------------------------------------------------------------
def dist_sq64(a, b):
    """(|a|^2 + |b|^2 - 2 a.b) + 1e-6f in float64 for a [n1,D], b [n2,D] -> (value [n1,n2], M [n1,n2] = sum a^2 + sum b^2 + 2 sum |ab|,
    the magnitude the fp32 chain's rounding errors scale with)."""
    a, b = _d(_t32(a)), _d(_t32(b))
    b = b.to(a.device)
    na, nb = (a * a).sum(1), (b * b).sum(1)
    val = (na[:, None] + nb[None, :] - 2.0 * (a @ b.t())) + EPS_SNN
    M = na[:, None] + nb[None, :] + 2.0 * (a.abs() @ b.abs().t())
    return val, M


def dist_sq_bound(val, M, D):
    """|d^2 - val| for the fp32 distance d of any summation order of the three sums (fused or not): each sum of D terms is within
    gamma_D of its exact value, the three adds and the sqrt round once each (the sqrt's relative u doubles in the square).
    bound = (D + 4) u M + 3 u |val|, with gamma_D <= 1.01 D u folded in, plus the float64 statement's own D 2^-53 M."""
    return (1.01 * (D + 4) * U32 + D * U64) * M + 3.0 * U32 * val.abs()


# ---- ground-truth check ---------------------------------------------------------------------------------------------------------------
def gt_inverse(H):
    """H1to2^-1 = adj(H) / det(H) of the fp32 H in float64, in adj3's order and without fused multiply-adds."""
    H = np.asarray(H, np.float32).astype(np.float64).reshape(1, 9)
    A = R.adj3(H)[0]
    with np.errstate(all="ignore"):
        det = H[0, 0] * A[0] + H[0, 1] * A[3] + H[0, 2] * A[6]
        return A / det


def gt_mapped(pts, H):
    """The image-2 centres pts[:, 2:4] mapped into image 1 in float64 and cast to fp32 -> (px, py) float32 arrays."""
    Hi = gt_inverse(H)
    x, y = pts[:, 2].astype(np.float32).astype(np.float64), pts[:, 3].astype(np.float32).astype(np.float64)
    with np.errstate(all="ignore"):
        w = Hi[6] * x + Hi[7] * y + Hi[8]
        px = ((Hi[0] * x + Hi[1] * y + Hi[2]) / w).astype(np.float32)
        py = ((Hi[3] * x + Hi[4] * y + Hi[5]) / w).astype(np.float32)
    return px, py


def _sq32(x, y):
    return _f(_d(_f(x * x)) + _d(_f(y * y)))


def gt_dist(pts, H, dev=None, fused=True, swap=False, rows=1024):
    """gt_kernel's distances [n,n]: row t is centre t of image 1, column u the mapped image-2 centre u:
    sqrtf(fabsf(((|p|^2 + |a|^2) - 2 dot) + 1e-12f)), dot = fmaf(ay, qy, ax qx).  `fused=False` (an unfused dot) and `swap=True`
    (fmaf(ax, qx, ay qy)) are mutations."""
    px, py = gt_mapped(pts, H)
    qx, qy = torch.from_numpy(px).to(dev), torch.from_numpy(py).to(dev)
    ax_all = torch.from_numpy(np.ascontiguousarray(pts[:, 0], np.float32)).to(dev)
    ay_all = torch.from_numpy(np.ascontiguousarray(pts[:, 1], np.float32)).to(dev)
    nq = _sq32(_d(qx), _d(qy))
    out = []
    for r0 in range(0, len(pts), rows):
        ax, ay = ax_all[r0:r0 + rows, None], ay_all[r0:r0 + rows, None]
        na = _sq32(_d(ax), _d(ay))
        if not fused:
            dot = _f(_d(_f(_d(ax) * _d(qx)[None])) + _d(_f(_d(ay) * _d(qy)[None])))
        elif swap:
            dot = fmaf32(ax, qx[None], _f(_d(ay) * _d(qy)[None]))
        else:
            dot = fmaf32(ay, qy[None], _f(_d(ax) * _d(qx)[None]))
        t = _f(_d(nq)[None] + _d(na))
        t = _f(_d(t) - _d(_f(2.0 * _d(dot))))
        t = _f(_d(t) + EPS_GT)
        out.append(_f(torch.sqrt(_d(t).abs())))
    return torch.cat(out) if out else torch.zeros(0, 0, dtype=torch.float32, device=dev)


def gt_rows(dist, th, lowest=True, nan_ignored=True, le=True):
    """gt_kernel's reduction of dist [n,n] -> (min_dist fp32, idx2 int64, true int64 ascending): the minimum below +inf with NaN
    ignored and the lowest index, (+inf, 0) when there is none; a row is true when min_dist <= th (fp32).  The keywords are mutations."""
    n = dist.size(0)
    if n == 0:
        z = torch.zeros(0, dtype=torch.int64)
        return torch.zeros(0, dtype=torch.float32), z, z
    lt = torch.where(torch.isnan(dist), INF, dist) if nan_ignored else dist
    mval = lt.min(1).values
    cols = torch.arange(n, device=dist.device).expand(n, n)
    hit = (lt == mval[:, None]) & (lt < INF)
    pick = torch.where(hit, cols, n).min(1).values if lowest else torch.where(hit, cols, -1).max(1).values
    has = hit.any(1)
    idx2 = torch.where(has, pick, torch.zeros_like(pick))
    mn = torch.where(has, dist.gather(1, idx2[:, None])[:, 0], torch.full_like(mval, INF))
    if not nan_ignored:
        mn = torch.where(torch.isnan(mval), mval, mn)
    t32 = torch.tensor(float(np.float32(th)), dtype=torch.float32, device=dist.device)
    keep = (mn <= t32) if le else (mn < t32)
    return mn, idx2, torch.arange(n, device=dist.device)[keep]


def gt_check(pts, H, th, dev=None):
    """ag_gt_correspondences_pairs for one pair -> (min_dist, idx2, true) as CPU tensors."""
    mn, idx2, true = gt_rows(gt_dist(pts, H, dev), th)
    return mn.cpu(), idx2.cpu(), true.cpu()


# ---- float64 statement and bound of the ground-truth distance ------------------------------------------------------------------------
def gt_sq64(pts, H, fp32_inverse=False):
    """Squared distances [n,n] between the image-1 centres and the exactly mapped image-2 centres (float64, H^-1 by np.linalg.inv),
    and the bound on |d^2 - D^2| of an fp32 distance d computed by the reference's formula from mapped centres p':

        6 u (|a| + |p|)^2           the two norms, the 2-term dot (fused or not, any order) and the three adds
        + 3 u D^2 + 2e-12           the sqrt's rounding and the 1e-12
        + 2 D |e| + |e|^2            the mapped centres' error e (2-norm) moves the distance by at most |e|

    e is bounded per component as (G_r + |p_r| G_w) / |w| with G = c (|H^-1| |H| |H^-1| + |H^-1|) |c2| (componentwise): the
    kernel maps in float64 (c = 16 * 2^-53) and casts to fp32 (u |p_r| more); the reference inverts and multiplies in fp32
    (c = 16 u, and the cast is exact).  -> (D2 [n,n], bound [n,n]) as float64 arrays; rows or columns with non-finite terms are NaN."""
    H64 = np.asarray(H, np.float32).astype(np.float64)
    Hi = np.linalg.inv(H64)
    c2 = np.stack([pts[:, 2].astype(np.float64), pts[:, 3].astype(np.float64), np.ones(len(pts))], 1)
    hom = c2 @ Hi.T
    w = hom[:, 2]
    with np.errstate(all="ignore"):
        p = hom[:, :2] / w[:, None]
        K = np.abs(Hi) @ np.abs(H64) @ np.abs(Hi) + np.abs(Hi)
        G = np.abs(c2) @ K.T * (16.0 * (U32 if fp32_inverse else U64))
        e = (G[:, :2] + np.abs(p) * G[:, 2:3]) / np.abs(w)[:, None]
        if not fp32_inverse:
            e = e + U32 * np.abs(p)
        en = np.hypot(e[:, 0], e[:, 1])
        a = pts[:, :2].astype(np.float64)
        D2 = ((a[:, None, :] - p[None, :, :]) ** 2).sum(2)
        ra, rp = np.hypot(a[:, 0], a[:, 1]), np.hypot(p[:, 0], p[:, 1])
        bound = 6 * U32 * (ra[:, None] + rp[None, :]) ** 2 + 3 * U32 * D2 + 2e-12 + 2 * np.sqrt(D2) * en[None] + en[None] ** 2
    return D2, bound


# ---- RANSAC against float64 -----------------------------------------------------------------------------------------------------------
def dlt_svd(pts, mask):
    """The normalised DLT of the rows of `mask` solved by a float64 SVD of the 2n x 9 design matrix (not the normal matrix), with
    the Hartley normalisation recomputed by numpy -> H [3,3] with H[2,2] = 1."""
    p = pts[mask].astype(np.float64)
    c1, c2 = p[:, :2].mean(0), p[:, 2:].mean(0)
    s1 = math.sqrt(2.0 / ((p[:, :2] - c1) ** 2).sum(1).mean())
    s2 = math.sqrt(2.0 / ((p[:, 2:] - c2) ** 2).sum(1).mean())
    u, v = (p[:, 0] - c1[0]) * s1, (p[:, 1] - c1[1]) * s1
    up, vp = (p[:, 2] - c2[0]) * s2, (p[:, 3] - c2[1]) * s2
    z, one = np.zeros_like(u), np.ones_like(u)
    A = np.concatenate([np.stack([-u, -v, -one, z, z, z, up * u, up * v, up], 1), np.stack([z, z, z, -u, -v, -one, vp * u, vp * v, vp], 1)])
    h = np.linalg.svd(A)[2][-1].reshape(3, 3)
    T1 = np.array([[s1, 0, -s1 * c1[0]], [0, s1, -s1 * c1[1]], [0, 0, 1.0]])
    T2i = np.array([[1 / s2, 0, c2[0]], [0, 1 / s2, c2[1]], [0, 0, 1.0]])
    H = T2i @ h @ T1
    return H / H[2, 2]


def refit_report(tr, pts):
    """One traced refit of oracle_ransac.refit against float64 -> (Jacobi off-diagonal norm / |A|, sin of the angle between the
    chosen eigenvector and eigh's smallest, its bound, corner error (px) of H against dlt_svd on the same rows).

    The bound is Davis-Kahan's: sin <= (|off(A_J)|_F + 64 * 9 * 2^-53 |A|_F) / (lambda_2 - lambda_1), the rotations' own rounding
    taken as 64 unit roundoffs per entry."""
    from verify_cases import corner_error
    A0, Aj, V, mi = tr["A0"], tr["A"], tr["V"], tr["mi"]
    nA = np.linalg.norm(A0)
    off = np.linalg.norm(Aj - np.diag(np.diag(Aj)))
    lam, W = np.linalg.eigh(A0)
    v, w = V[:, mi] / np.linalg.norm(V[:, mi]), W[:, 0] / np.linalg.norm(W[:, 0])
    sin = float(np.linalg.norm(v - (v @ w) * w))
    bound = (off + 64 * 9 * U64 * nA) / (lam[1] - lam[0])
    err = corner_error(tr["H"].reshape(3, 3), dlt_svd(pts, tr["mask"])) if tr["H"] is not None else float("nan")
    return off / nA, sin, bound, err
