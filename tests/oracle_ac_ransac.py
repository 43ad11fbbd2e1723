"""numpy restatement of ag_homography_ransac_affine (affnet_b200/csrc/verify.cu), operation for operation, on top of oracle_ransac: the
splitmix64 sampler's first 2 distinct draws, the degeneracy rules, the fp64 2-AC solver (Hartley similarity of the two centres, the 12 x 8
least squares through its normal equations by Cholesky), the affine inlier test (the centre test and the skip-centre Frobenius distance of
the row's own frames under H), the local optimisation whenever a chunk's winner raises the best count (the refit rounds, and
LO-RANSAC's shrinking-threshold refits), and the chunked adaptive stop with sample size 2.  numpy and Python round every product and sum
separately, as verify.cu does (it is built without fused multiply-adds), so the two agree on every decision and on the bits of H.

An affine correspondence (AC) is a row of 12 values: the centres (x1, y1, x2, y2), then the 2x2 parts (a00, a01, a10, a11) of the
image-1 and the image-2 frame."""
import math

import numpy as np

from oracle_ransac import REFIT_ROUNDS, VT, adj3, inliers, mul3, normalise_h, refit, samples

CHOL_EPS = 1e-10      # a Cholesky pivot <= CHOL_EPS times its diagonal entry is a degenerate sample
LO_FACTOR = 16.0           # shrinking_lo's first threshold factor (halved at each refit)
LO_STEPS = 5               # its refits: factors 16, 8, 4, 2, 1


def ac_rows(lafs1, lafs2):
    """Paired LAFs [n,2,3] (image 1, image 2) -> AC rows [n,12] float32."""
    l1 = np.asarray(lafs1, np.float32).reshape(-1, 6)
    l2 = np.asarray(lafs2, np.float32).reshape(-1, 6)
    return np.concatenate([l1[:, [2, 5]], l2[:, [2, 5]], l1[:, [0, 1, 3, 4]], l2[:, [0, 1, 3, 4]]], 1)


def ac_homographies(s):
    """s [K,2,12] fp64 (two ACs per hypothesis) -> (H [K,9] normalised, ok [K]): ac_homography of verify.cu."""
    K = len(s)
    c, a1, a2 = s[..., 0:4], s[..., 4:8], s[..., 8:12]
    ok = np.isfinite(s).all(axis=(1, 2))
    with np.errstate(all="ignore"):
        d1 = a1[..., 0] * a1[..., 3] - a1[..., 1] * a1[..., 2]                         # [K,2]
        d2 = a2[..., 0] * a2[..., 3] - a2[..., 1] * a2[..., 2]
        ok &= (d1 != 0.0).all(1) & (d2 != 0.0).all(1)
        ok &= ((d1[:, 0] > 0.0) == (d2[:, 0] > 0.0)) == ((d1[:, 1] > 0.0) == (d2[:, 1] > 0.0))
        c1x, c1y = (c[:, 0, 0] + c[:, 1, 0]) * 0.5, (c[:, 0, 1] + c[:, 1, 1]) * 0.5
        c2x, c2y = (c[:, 0, 2] + c[:, 1, 2]) * 0.5, (c[:, 0, 3] + c[:, 1, 3]) * 0.5
        h1x, h1y = (c[:, 1, 0] - c[:, 0, 0]) * 0.5, (c[:, 1, 1] - c[:, 0, 1]) * 0.5
        h2x, h2y = (c[:, 1, 2] - c[:, 0, 2]) * 0.5, (c[:, 1, 3] - c[:, 0, 3]) * 0.5
        var1, var2 = h1x * h1x + h1y * h1y, h2x * h2x + h2y * h2y
        ok &= (var1 > 0.0) & (var2 > 0.0)
        s1, s2 = np.sqrt(2.0 / var1), np.sqrt(2.0 / var2)
        rs = s2 / s1
        N = np.zeros((K, 8, 8))
        b = np.zeros((K, 8))
        z, one = np.zeros(K), np.ones(K)
        for k in range(2):
            u, v = (c[:, k, 0] - c1x) * s1, (c[:, k, 1] - c1y) * s1
            up, vp = (c[:, k, 2] - c2x) * s2, (c[:, k, 3] - c2y) * s2
            p00, p01, p10, p11 = (a1[:, k, q] for q in range(4))
            q00, q01, q10, q11 = (a2[:, k, q] for q in range(4))
            i00, i01, i10, i11 = p11 / d1[:, k], -p01 / d1[:, k], -p10 / d1[:, k], p00 / d1[:, k]
            n00, n01 = (q00 * i00 + q01 * i10) * rs, (q00 * i01 + q01 * i11) * rs
            n10, n11 = (q10 * i00 + q11 * i10) * rs, (q10 * i01 + q11 * i11) * rs
            rows = [[u, v, one, z, z, z, -(up * u), -(up * v), up],
                    [z, z, z, u, v, one, -(vp * u), -(vp * v), vp],
                    [one, z, z, z, z, z, -(up + n00 * u), -(n00 * v), n00],
                    [z, one, z, z, z, z, -(n01 * u), -(up + n01 * v), n01],
                    [z, z, z, one, z, z, -(vp + n10 * u), -(n10 * v), n10],
                    [z, z, z, z, one, z, -(n11 * u), -(vp + n11 * v), n11]]
            for r in rows:
                for i in range(8):
                    b[:, i] = b[:, i] + r[i] * r[8]
                    for l in range(i, 8):
                        N[:, i, l] = N[:, i, l] + r[i] * r[l]
        # Cholesky into the lower triangle, then the two triangular solves
        dg = np.zeros((K, 8))
        for j in range(8):
            d = N[:, j, j].copy()
            for k in range(j):
                d = d - N[:, j, k] * N[:, j, k]
            ok &= d > CHOL_EPS * N[:, j, j]
            dg[:, j] = np.sqrt(d)
            for i in range(j + 1, 8):
                t = N[:, j, i].copy()
                for k in range(j):
                    t = t - N[:, i, k] * N[:, j, k]
                N[:, i, j] = t / dg[:, j]
        for i in range(8):
            t = b[:, i].copy()
            for k in range(i):
                t = t - N[:, i, k] * b[:, k]
            b[:, i] = t / dg[:, i]
        for i in range(7, -1, -1):
            t = b[:, i].copy()
            for k in range(i + 1, 8):
                t = t - N[:, k, i] * b[:, k]
            b[:, i] = t / dg[:, i]
        Hn = np.concatenate([b, one[:, None]], 1)
        T1 = np.stack([s1, z, -(s1 * c1x), z, s1, -(s1 * c1y), z, z, one], 1)
        T2i = np.stack([1.0 / s2, z, c2x, z, 1.0 / s2, c2y, z, z, one], 1)
        H, okh = normalise_h(mul3(mul3(T2i, Hn), T1))
    return H, ok & okh


def frame_distance(H, ac):
    """H [9] or [K,9], ac [n,12] fp64 -> (D [K,n], ok [K,n]): |A1^-1 J A2 - I|_F^2 with J = linH(adj(H)) at the image-2 centre;
    ok False where a frame is not finite or singular."""
    G = adj3(np.atleast_2d(np.asarray(H, np.float64)))[:, :, None]
    x, y = ac[:, 2], ac[:, 3]
    a00, a01, a10, a11 = (ac[:, 4 + q] for q in range(4))
    b00, b01, b10, b11 = (ac[:, 8 + q] for q in range(4))
    with np.errstate(all="ignore"):
        det1, det2 = a00 * a11 - a01 * a10, b00 * b11 - b01 * b10
        ok = np.isfinite(ac[:, 4:12]).all(1) & (det1 != 0.0) & (det2 != 0.0)
        w = G[:, 6] * x + G[:, 7] * y + G[:, 8]
        n1 = G[:, 0] * x + G[:, 1] * y + G[:, 2]
        n2 = G[:, 3] * x + G[:, 4] * y + G[:, 5]
        q1, q2 = n1 / (w * w), n2 / (w * w)
        j00, j01, j10, j11 = G[:, 0] / w - q1 * G[:, 6], G[:, 1] / w - q1 * G[:, 7], G[:, 3] / w - q2 * G[:, 6], G[:, 4] / w - q2 * G[:, 7]
        e00, e01, e10, e11 = j00 * b00 + j01 * b10, j00 * b01 + j01 * b11, j10 * b00 + j11 * b10, j10 * b01 + j11 * b11
        i00, i01, i10, i11 = a11 / det1, -a01 / det1, -a10 / det1, a00 / det1
        d00, m01, m10 = (i00 * e00 + i01 * e10) - 1.0, i00 * e01 + i01 * e11, i10 * e00 + i11 * e10
        d11 = (i10 * e01 + i11 * e11) - 1.0
        D = ((d00 * d00 + m01 * m01) + m10 * m10) + d11 * d11
    return D, np.broadcast_to(ok, D.shape)


def inliers_ac(H, ac, th2, laf_th):
    """The affine inlier test of H [9] or [K,9] over ac [n,12] fp64 -> bool [K,n]."""
    D, ok = frame_distance(H, ac)
    with np.errstate(invalid="ignore"):
        return inliers(H, ac[:, :4], th2) & ok & (D <= laf_th)


def local_opt(H, ac, th2, laf_th):
    """The refit rounds (point DLT on the inliers, kept while the count under the affine test does not drop) -> (H, mask, count)."""
    mask = inliers_ac(H, ac, th2, laf_th)[0]
    cnt = int(mask.sum())
    for _ in range(REFIT_ROUNDS):
        if cnt < 4:
            break
        Hr = refit(ac[:, :4], mask)
        if Hr is None:
            break
        mr = inliers_ac(Hr, ac, th2, laf_th)[0]
        if int(mr.sum()) < cnt:
            break
        H, mask, cnt = Hr, mr, int(mr.sum())
    return H, mask, cnt


def shrinking_lo(H, ac, th2, laf_th):
    """LO-RANSAC's iterative step (ac_local_opt): point DLT on the inliers at LO_FACTOR times both thresholds (centre and frame), then
    at half that, ... down to 1 times (at most LO_STEPS refits, stopping at fewer than 4 inliers or a failed refit), then the refit rounds
    -> (H, mask, count)."""
    f = LO_FACTOR
    for _ in range(LO_STEPS):
        m = inliers_ac(H, ac, th2 * (f * f), laf_th * f)[0]
        if int(m.sum()) < 4:
            break
        Hr = refit(ac[:, :4], m)
        if Hr is None:
            break
        H = Hr
        f = f * 0.5
    return local_opt(H, ac, th2, laf_th)


def search_lo(H, ac, th2, laf_th):
    """The local optimisation of a chunk's winner that raised the best count: the refit rounds, and shrinking_lo from the same winner;
    the latter when its count is higher -> (H, mask, count)."""
    H0, m0, c0 = local_opt(H, ac, th2, laf_th)
    H1, m1, c1 = shrinking_lo(H, ac, th2, laf_th)
    return (H1, m1, c1) if c1 > c0 else (H0, m0, c0)


def ransac_ac(ac, inl_th=2.0, laf_th=2.0, confidence=0.99, max_iters=50000, seed=0, trace=None):
    """ac [n,12] float32 -> (H [3,3] float32, mask [n] bool, ninl, iters) as ag_homography_ransac_affine computes them.  A list `trace`
    receives (h of the chunk's winner, its count, the count after the local optimisation) each time the best count rises."""
    ac = np.asarray(ac, dtype=np.float32).astype(np.float64).reshape(-1, 12)
    n = len(ac)
    th = float(np.float32(inl_th))
    th2 = th * th
    lth = float(np.float32(laf_th))
    log1mconf = math.log(1.0 - float(np.float32(confidence)))
    best, best_H, h_done = 0, None, 0
    if n >= 2:
        h0 = 0
        while True:
            h = np.arange(h0, h0 + VT)
            idx, ok = samples(seed, h, n, 2)
            ok &= h < max_iters
            Hs, okh = ac_homographies(ac[idx])
            ok &= okh
            cnt = np.full(VT, -1, dtype=np.int64)
            if ok.any():
                cnt[ok] = inliers_ac(Hs[ok], ac, th2, lth).sum(axis=1)
            k = int(np.argmax(cnt))          # the first maximum: the lowest h
            if cnt[k] > best:
                best_H, _, lo = search_lo(Hs[k], ac, th2, lth)
                if trace is not None:
                    trace.append((h0 + k, int(cnt[k]), lo))
                best = lo
            h_done = min(h0 + VT, max_iters)
            pr = best / n
            p2 = pr * pr
            need = 0.0 if p2 >= 1.0 else (math.inf if p2 <= 0.0 else math.ceil(log1mconf / math.log(1.0 - p2)))
            if h_done >= min(need, float(max_iters)):
                break
            h0 += VT
    if best == 0:
        return np.zeros((3, 3), np.float32), np.zeros(n, bool), 0, h_done
    H, mask, cnt = local_opt(best_H, ac, th2, lth)
    return H.reshape(3, 3).astype(np.float32), mask, cnt, h_done
