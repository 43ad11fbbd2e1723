"""numpy restatement of ag_fundamental_degensac (affnet_b200/csrc/verify.cu), operation for operation, on top of oracle_fransac: the
7-point search of ag_fundamental_ransac with, whenever a chunk's winner raises the so-far-best count, DEGENSAC's degeneracy test of the
winning sample (the left epipole by the 3x3 Jacobi, the homographies of five point triplets, their transfer errors), plane-and-parallax
for an H-degenerate sample (two-point samples by rejection over the splitmix64 sampler, F = [e']x H, the Sampson count) and the refit
rounds as local optimisation.  numpy and Python round every product and sum separately, as verify.cu does (it is built without fused
multiply-adds), so the two agree on every decision and on the bits of F."""
import math

import numpy as np

from oracle_fransac import (F_REFIT_MIN, F_SAMPLE, REFIT_ROUNDS, VT, _stats, block_sum, count_inliers, denormalise_f, draw_indices,
                            inliers_f, jacobi, normalise_f, refit_f, samples, seven_point, smallest_diag)
from oracle_ransac import adj3, inliers, normalise_h, refit

DEG_H_TH_FACTOR = 4.0                 # DEG_H_TH = DEG_H_TH_FACTOR * inl_th: a point agrees with a plane H within it (transfer error, px)
DEG_MIN_AGREE = 5                     # a sample is H-degenerate when some triplet's H agrees with this many of its 7 points
DEG_TRIPLETS = ((0, 1, 2), (3, 4, 5), (0, 1, 6), (3, 4, 6), (2, 5, 6))   # Chum, Werner and Matas, CVPR 2005
DEG_SEED_TAG = 0xD5A61266F0C9392C     # the plane-and-parallax sampler's stream: seed ^ DEG_SEED_TAG
DEG_H_BASE = 1 << 31                  # its hypotheses: DEG_H_BASE + k * VT + thread, k the degeneracy tests so far
M64 = (1 << 64) - 1


def cross(a, b):
    """a x b of [..., 3] (or sequences of 3), verify.cu's order."""
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def skew_mul(e, M):
    """[e]x M for e (3 values) and M [..., 9] row-major: column c of the product is e x (column c of M)."""
    o = np.empty(np.broadcast_shapes(np.shape(M), np.shape(e[0]) + (9,)), dtype=np.float64)
    for c in range(3):
        r = cross(e, (M[..., c], M[..., 3 + c], M[..., 6 + c]))
        o[..., c], o[..., 3 + c], o[..., 6 + c] = r
    return o


def left_epipole(F):
    """e' with F' e' = 0: the eigenvector of the smallest eigenvalue of F F' (verify.cu's jacobi3)."""
    G = np.empty((3, 3))
    for r in range(3):
        for c in range(3):
            G[r, c] = F[3 * r] * F[3 * c] + F[3 * r + 1] * F[3 * c + 1] + F[3 * r + 2] * F[3 * c + 2]
    V = np.eye(3)
    jacobi(G, V)
    m = smallest_diag(G)
    return (float(V[0, m]), float(V[1, m]), float(V[2, m]))


def triplet_homography(A, e, c):
    """H = A - e' (M^-1 b)' of the three correspondences c [3,4] (Hartley and Zisserman, result 13.6) with A = [e']x F, or None when M
    (the image-1 points as rows) is singular or H / H[2][2] is not finite.  Normalised as the homography RANSAC's hypotheses are."""
    b = []
    for m in range(3):
        x, y, x2, y2 = (float(v) for v in c[m])
        ax = (A[0] * x + A[1] * y + A[2], A[3] * x + A[4] * y + A[5], A[6] * x + A[7] * y + A[8])
        xp = (x2, y2, 1.0)
        p = cross(xp, ax)
        q = cross(xp, e)
        with np.errstate(all="ignore"):
            b.append(np.float64(p[0] * q[0] + p[1] * q[1] + p[2] * q[2]) / np.float64(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]))
    M = np.array([c[0][0], c[0][1], 1.0, c[1][0], c[1][1], 1.0, c[2][0], c[2][1], 1.0], dtype=np.float64)
    Ad = adj3(M)
    det = M[0] * Ad[0] + M[1] * Ad[3] + M[2] * Ad[6]
    if det == 0.0:
        return None
    with np.errstate(all="ignore"):
        Mi = Ad / det
        v = [Mi[3 * r] * b[0] + Mi[3 * r + 1] * b[1] + Mi[3 * r + 2] * b[2] for r in range(3)]
        H = np.array([A[3 * r + k] - e[r] * v[k] for r in range(3) for k in range(3)])
    H, ok = normalise_h(H)
    return H if ok else None


def degenerate_h(F, c, thd2):
    """The degeneracy test of a 7-point sample c [7,4] with its model F [9] -> (H [9] agreeing with the most sample points, the lowest
    triplet on ties, and that number), or (None, 0) when no triplet gives a finite H."""
    e = left_epipole(F)
    A = skew_mul(e, np.asarray(F, np.float64))
    best, bH = 0, None
    for t in DEG_TRIPLETS:
        H = triplet_homography(A, e, c[list(t)])
        if H is None:
            continue
        k = int(inliers(H, c, thd2).sum())
        if k > best:
            best, bH = k, H
    return bH, best


def pp_draws(seed, k, n, hin):
    """Two-point samples of plane-and-parallax test k: thread i draws from hypothesis DEG_H_BASE + k VT + i of the stream
    seed ^ DEG_SEED_TAG, rejecting rows that are inliers of H (hin [n]) and the first index again -> (a, b, ok) of [VT]."""
    h = DEG_H_BASE + k * VT + np.arange(VT)
    dr = draw_indices((seed ^ DEG_SEED_TAG) & M64, h, n).astype(np.int64)   # [VT, MAX_DRAWS]
    acc = ~hin[dr]
    ar = np.arange(VT)
    pa = np.argmax(acc, axis=1)
    a = dr[ar, pa]
    acc2 = acc & (dr != a[:, None])
    pb = np.argmax(acc2, axis=1)
    return a, dr[ar, pb], acc.any(axis=1) & acc2.any(axis=1)


def plane_and_parallax(H, pts, a, b, ok):
    """F = [e']x H, e' = (H x_a x x'_a) x (H x_b x x'_b), normalised -> (F [VT,9], ok [VT])."""
    def line(i):
        x, y, x2, y2 = pts[i, 0], pts[i, 1], pts[i, 2], pts[i, 3]
        hx = (H[0] * x + H[1] * y + H[2], H[3] * x + H[4] * y + H[5], H[6] * x + H[7] * y + H[8])
        return cross(hx, (x2, y2, np.ones_like(x2)))
    with np.errstate(all="ignore"):
        e = cross(line(a), line(b))
        F = skew_mul(e, np.broadcast_to(H, (len(a), 9)))
        F, okf = normalise_f(F)
    return F, ok & okf


def refine_h(H, pts, thd2):
    """The homography RANSAC's refit rounds (normalised DLT) on the plane H at DEG_H_TH -> (H, its inlier mask over all rows)."""
    mask = inliers(H, pts, thd2)[0]
    cnt = int(mask.sum())
    for _ in range(REFIT_ROUNDS):
        if cnt < 4:
            break
        Hr = refit(pts, mask)
        if Hr is None:
            break
        mr = inliers(Hr, pts, thd2)[0]
        if int(mr.sum()) < cnt:
            break
        H, mask, cnt = Hr, mr, int(mr.sum())
    return H, mask


def local_opt(F, pts, th2):
    """The refit rounds of ag_fundamental_ransac's end on F -> (F, mask, count)."""
    mask = inliers_f(F, pts, th2)[0]
    cnt = int(mask.sum())
    for _ in range(REFIT_ROUNDS):
        if cnt < F_REFIT_MIN:
            break
        Fr = refit_f(pts, mask)
        if Fr is None:
            break
        mr = inliers_f(Fr, pts, th2)[0]
        if int(mr.sum()) < cnt:
            break
        F, mask, cnt = Fr, mr, int(mr.sum())
    return F, mask, cnt


def degensac_f(pts, inl_th=0.5, confidence=0.99, max_iters=50000, seed=0, trace=None):
    """pts [n,4] float32 (x1, y1, x2, y2) -> (F [3,3] float32, mask [n] bool, ninl, iters) as ag_fundamental_degensac computes them.
    A list `trace` receives one dict per degeneracy test: the sample's h, whether it was H-degenerate, the agreeing points, the best
    plane-and-parallax count (or None) and the count after the local optimisation."""
    pts = np.asarray(pts, dtype=np.float32).astype(np.float64)
    n = len(pts)
    th = float(np.float32(inl_th))
    th2 = th * th
    thd2 = (DEG_H_TH_FACTOR * DEG_H_TH_FACTOR) * th2
    log1mconf = math.log(1.0 - float(np.float32(confidence)))
    best, best_F, h_done, ntests = 0, None, 0, 0
    if n >= F_SAMPLE:
        fin = np.isfinite(pts).all(axis=1)
        x1, y1, x2, y2 = [np.where(fin, pts[:, k], 0.0) for k in range(4)]
        with np.errstate(all="ignore"):
            st = np.stack([x1, y1, x1 * x1, y1 * y1, x2, y2, x2 * x2, y2 * y2, np.where(fin, 1.0, 0.0)], axis=1)
            nd = float(block_sum(st)[8])
            c1x, c1y, c2x, c2y, var1, var2 = _stats(st, nd)
        search = nd >= F_SAMPLE and var1 > 0.0 and var2 > 0.0
        if search:
            T = (c1x, c1y, math.sqrt(2.0 / var1), c2x, c2y, math.sqrt(2.0 / var2))
        h0 = 0
        while search:
            h = np.arange(h0, h0 + VT)
            idx, ok = samples(seed, h, n)
            ok &= h < max_iters
            c = pts[idx]                                                    # [VT,7,4]
            ok &= np.isfinite(c).all(axis=(1, 2))
            with np.errstate(all="ignore"):
                u = np.stack([(c[..., 0] - T[0]) * T[2], (c[..., 1] - T[1]) * T[2], (c[..., 2] - T[3]) * T[5], (c[..., 3] - T[4]) * T[5]], 2)
            cnt = np.full(VT * 3, -1, dtype=np.int64)
            Fall = np.zeros((VT * 3, 9))
            hv = np.nonzero(ok)[0]
            if len(hv):
                Fn, okm = seven_point(u[hv])
                Fd, okd = denormalise_f(T, Fn.reshape(-1, 9))
                okd &= okm.reshape(-1)
                rows = (hv[:, None] * 3 + np.arange(3)[None, :]).reshape(-1)[okd]
                Fall[rows] = Fd[okd]
                cnt[rows] = count_inliers(Fd[okd], pts, th2)
            k = int(np.argmax(cnt))                                         # the first maximum: lowest h, then lowest root
            if cnt[k] > best:
                best, best_F = int(cnt[k]), Fall[k]
                rec = dict(h=h0 + k // 3)
                # 1. degeneracy test of the winning sample
                Hd, agree = degenerate_h(best_F, c[k // 3], thd2)
                rec.update(degenerate=agree >= DEG_MIN_AGREE, agree=agree, pp=None)
                # 2. plane-and-parallax
                if agree >= DEG_MIN_AGREE:
                    Hd, hin = refine_h(Hd, pts, thd2)
                    a, b, okp = pp_draws(seed, ntests, n, hin)
                    Fp, okp = plane_and_parallax(Hd, pts, a, b, okp)
                    cp = np.full(VT, -1, dtype=np.int64)
                    if okp.any():
                        cp[okp] = count_inliers(Fp[okp], pts, th2)
                    kp = int(np.argmax(cp))                                 # the first maximum: the lowest thread
                    rec["pp"] = int(cp[kp])
                    if cp[kp] > best:
                        best, best_F = int(cp[kp]), Fp[kp]
                ntests += 1
                # 3. local optimisation of the so-far-best model
                best_F, _, best = local_opt(best_F, pts, th2)
                rec["lo"] = best
                if trace is not None:
                    trace.append(rec)
            h_done = min(h0 + VT, max_iters)
            pr = best / n
            p7 = pr * pr * pr * pr * pr * pr * pr
            need = 0.0 if p7 >= 1.0 else (math.inf if p7 <= 0.0 or 1.0 - p7 == 1.0 else math.ceil(log1mconf / math.log(1.0 - p7)))
            if h_done >= min(need, float(max_iters)):
                break
            h0 += VT
    if best == 0:
        return np.zeros((3, 3), np.float32), np.zeros(n, bool), 0, h_done
    F, mask, cnt = local_opt(best_F, pts, th2)
    return F.reshape(3, 3).astype(np.float32), mask, cnt, h_done
