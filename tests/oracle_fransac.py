"""numpy restatement of ag_fundamental_ransac (affnet_b200/csrc/verify.cu), operation for operation: the Hartley normalisation with
its fixed-order block reduction, the splitmix64 sampler drawing 7 distinct indices, the 7-point solver (Gauss-Jordan elimination with
partial pivoting, the cubic det(F2 + l D) from one fixed expansion, its real roots by bisection with + - * / sqrt only), the
division-free Sampson test, the chunked adaptive stop and the normalised 8-point refit with rank 2 enforced.  numpy and Python round
every product and sum separately, as verify.cu does (it is built without fused multiply-adds), so the two agree on every decision and
on the bits of F."""
import math

import numpy as np

from oracle_ransac import JACOBI_SWEEPS, MAX_DRAWS, REFIT_ROUNDS, VT, adj3, block_sum, draw_indices, mul3, splitmix64  # noqa: F401

F_SAMPLE = 7
F_REFIT_MIN = 8
PIVOT_EPS = 1e-9
BISECT_STEPS = 1100   # enough to close any bracket in the double range; the bisection stops once the midpoint is an end


def samples(seed, h, n, k=F_SAMPLE):
    """-> (idx [len(h),k] int64, ok [len(h)]): the first k distinct draws of each hypothesis (ok False when 64 draws give fewer)."""
    dr = draw_indices(seed, h, n).astype(np.int64)
    eq = dr[:, :, None] == dr[:, None, :]
    first = ~np.tril(eq, -1).any(axis=2)
    rank = np.cumsum(first, axis=1)
    ok = rank[:, -1] >= k
    idx = np.zeros((len(dr), k), dtype=np.int64)
    for q in range(k):
        pos = np.argmax(first & (rank == q + 1), axis=1)
        idx[:, q] = dr[np.arange(len(dr)), pos]
    return idx, ok


def cubic_roots(a3, a2, a1, a0):
    """Real roots of a3 x^3 + a2 x^2 + a1 x + a0 in ascending order, as verify.cu's cubic_roots finds them (Python floats)."""
    a3, a2, a1, a0 = float(a3), float(a2), float(a1), float(a0)
    if not all(math.isfinite(v) for v in (a3, a2, a1, a0)):
        return []
    if a3 == 0.0:
        if a2 == 0.0:
            return [] if a1 == 0.0 else [-a0 / a1]
        disc = a1 * a1 - 4.0 * a2 * a0
        if disc < 0.0:
            return []
        if disc == 0.0:
            return [-a1 / (2.0 * a2)]
        sq = math.sqrt(disc)
        q = -0.5 * (a1 + sq) if a1 >= 0.0 else -0.5 * (a1 - sq)
        x1, x2 = q / a2, a0 / q
        return [x1, x2] if x1 < x2 else [x2, x1]
    b2, b1, b0 = a2 / a3, a1 / a3, a0 / a3
    m = abs(b2)
    if abs(b1) > m:
        m = abs(b1)
    if abs(b0) > m:
        m = abs(b0)
    R = 1.0 + m
    if not math.isfinite(R):
        return []
    d = b2 * b2 - 3.0 * b1
    if d > 0.0:
        sq = math.sqrt(d)
        x = [-R, (-b2 - sq) / 3.0, (-b2 + sq) / 3.0, R]
    else:
        x = [-R, R]

    def f(v):
        return ((a3 * v + a2) * v + a1) * v + a0

    roots = []
    for i in range(len(x) - 1):
        lo, hi = x[i], x[i + 1]
        fl, fh = f(lo), f(hi)
        if not ((fl < 0.0 and fh >= 0.0) or (fl > 0.0 and fh <= 0.0)):
            continue
        for _ in range(BISECT_STEPS):
            mid = 0.5 * (lo + hi)
            if mid == lo or mid == hi:
                break
            fm = f(mid)
            if (fm < 0.0) if fl < 0.0 else (fm > 0.0):
                lo = mid
            else:
                hi = mid
        roots.append(hi)
    return roots


def det_cubic(F2, D):
    """[..., 9] -> (a3, a2, a1, a0) of det(F2 + l D), verify.cu's expansion."""
    A2, AD = adj3(F2), adj3(D)
    a0 = F2[..., 0] * A2[..., 0] + F2[..., 1] * A2[..., 3] + F2[..., 2] * A2[..., 6]
    a3 = D[..., 0] * AD[..., 0] + D[..., 1] * AD[..., 3] + D[..., 2] * AD[..., 6]
    t1 = np.zeros_like(a0)
    t2 = np.zeros_like(a0)
    for r in range(3):
        for c in range(3):
            t1 = t1 + A2[..., 3 * r + c] * D[..., 3 * c + r]
            t2 = t2 + AD[..., 3 * r + c] * F2[..., 3 * c + r]
    return a3, t2, t1, a0


def seven_point(u):
    """u [H,7,4] normalised (u1, v1, u2, v2) -> (Fn [H,3,9], ok [H,3]) models in ascending root order, as verify.cu's seven_point."""
    Hn = len(u)
    u1, v1, u2, v2 = u[:, :, 0], u[:, :, 1], u[:, :, 2], u[:, :, 3]
    with np.errstate(all="ignore"):
        A = np.stack([u2 * u1, u2 * v1, u2, v2 * u1, v2 * v1, v2, u1, v1, np.ones_like(u1)], axis=2)   # [H,7,9]
        mx = np.abs(A).reshape(Hn, -1).max(axis=1) if Hn else np.zeros(0)
        tol = PIVOT_EPS * mx
        ar = np.arange(Hn)
        rows = np.arange(F_SAMPLE)
        rank = np.zeros(Hn, dtype=np.int64)
        free = np.zeros((Hn, 9), dtype=bool)
        pc = np.zeros((Hn, F_SAMPLE), dtype=np.int64)
        for c in range(9):
            full = rank == F_SAMPLE
            free[full, c] = True
            cand = np.where(rows[None, :] >= rank[:, None], np.abs(A[:, :, c]), -1.0)
            pr = np.argmax(cand, axis=1)                       # the first maximum: the lowest row
            pa = cand[ar, pr]
            piv = ~full & (pa > tol)
            free[~full & ~piv, c] = True
            hp, rk, pp = ar[piv], rank[piv], pr[piv]
            tmp = A[hp, rk].copy()
            A[hp, rk] = A[hp, pp]
            A[hp, pp] = tmp
            prow = A[hp, rk].copy()
            for r in range(F_SAMPLE):
                sel = rk != r
                h2 = hp[sel]
                f = A[h2, r, c] / prow[sel, c]
                nr = A[h2, r] - f[:, None] * prow[sel]
                nr[:, c] = 0.0
                A[h2, r] = nr
            pc[hp, rk] = c
            rank[hp] += 1
        Fn = np.zeros((Hn, 3, 9))
        okm = np.zeros((Hn, 3), dtype=bool)
        for h in np.nonzero(rank == F_SAMPLE)[0]:
            fr = np.nonzero(free[h])[0]
            f1, f2 = int(fr[0]), int(fr[1])
            F1, F2 = np.zeros(9), np.zeros(9)
            F1[f1] = 1.0
            F2[f2] = 1.0
            for i in range(F_SAMPLE):
                F1[pc[h, i]] = -(A[h, i, f1] / A[h, i, pc[h, i]])
                F2[pc[h, i]] = -(A[h, i, f2] / A[h, i, pc[h, i]])
            n1, n2 = 0.0, 0.0
            for k in range(9):
                n1 = n1 + F1[k] * F1[k]
                n2 = n2 + F2[k] * F2[k]
            F1, F2 = F1 / math.sqrt(n1), F2 / math.sqrt(n2)
            D = F1 - F2
            a3, a2, a1, a0 = det_cubic(F2, D)
            for m, lam in enumerate(cubic_roots(a3, a2, a1, a0)):
                Fn[h, m] = F2 + lam * D
                okm[h, m] = True
    return Fn, okm


def normalise_f(F):
    """[K,9] -> (F / +-|F|, ok): unit Frobenius norm, the largest-magnitude entry (the lowest index on ties) positive."""
    F = np.atleast_2d(F)
    ss = np.zeros(len(F))
    m = np.zeros(len(F), dtype=np.int64)
    ar = np.arange(len(F))
    with np.errstate(all="ignore"):
        for k in range(9):
            ss = ss + F[:, k] * F[:, k]
            m = np.where(np.abs(F[:, k]) > np.abs(F[ar, m]), k, m)
        ok = (ss > 0.0) & np.isfinite(ss)
        sq = np.sqrt(ss)
        nr = np.where(F[ar, m] < 0.0, -sq, sq)
        return F / nr[:, None], ok


def hartley_mats(T):
    c1x, c1y, s1, c2x, c2y, s2 = T
    T1 = np.array([s1, 0.0, -(s1 * c1x), 0.0, s1, -(s1 * c1y), 0.0, 0.0, 1.0])
    T2t = np.array([s2, 0.0, 0.0, 0.0, s2, 0.0, -(s2 * c2x), -(s2 * c2y), 1.0])
    return T1, T2t


def denormalise_f(T, Fn):
    """Fn [K,9] -> normalise_f(T2' Fn T1)."""
    T1, T2t = hartley_mats(T)
    with np.errstate(all="ignore"):
        return normalise_f(mul3(mul3(T2t, Fn), T1))


def inliers_f(F, pts, th2):
    """F [9] or [K,9], pts [n,4] fp64 -> bool [K,n]: the division-free Sampson test."""
    F = np.atleast_2d(F)[:, :, None]
    x, y, x2, y2 = pts[:, 0], pts[:, 1], pts[:, 2], pts[:, 3]
    with np.errstate(all="ignore"):
        a = F[:, 0] * x + F[:, 1] * y + F[:, 2]
        b = F[:, 3] * x + F[:, 4] * y + F[:, 5]
        d = F[:, 6] * x + F[:, 7] * y + F[:, 8]
        g = F[:, 0] * x2 + F[:, 3] * y2 + F[:, 6]
        k = F[:, 1] * x2 + F[:, 4] * y2 + F[:, 7]
        e = x2 * a + y2 * b + d
        den = a * a + b * b + g * g + k * k
        return (den > 0.0) & (e * e <= th2 * den)


def sampson(F, pts):
    """Sampson distances (px, float64) of the rows of pts [n,4] to F [3,3]."""
    F = np.asarray(F, np.float64).reshape(9)
    pts = np.asarray(pts, np.float64)
    x, y, x2, y2 = pts.T
    a, b, d = F[0] * x + F[1] * y + F[2], F[3] * x + F[4] * y + F[5], F[6] * x + F[7] * y + F[8]
    g, k = F[0] * x2 + F[3] * y2 + F[6], F[1] * x2 + F[4] * y2 + F[7]
    return np.abs(x2 * a + y2 * b + d) / np.sqrt(a * a + b * b + g * g + k * k)


def count_inliers(Fs, pts, th2, block=64):
    out = np.zeros(len(Fs), dtype=np.int64)
    for k0 in range(0, len(Fs), block):
        out[k0:k0 + block] = inliers_f(Fs[k0:k0 + block], pts, th2).sum(axis=1)
    return out


def jacobi(A, V):
    """verify.cu's cyclic Jacobi (jacobi9_warp / jacobi3) of the symmetric A, in place, rotations accumulated into V."""
    N = len(A)
    for _ in range(JACOBI_SWEEPS):
        for p in range(N - 1):
            for q in range(p + 1, N):
                apq, app, aqq = float(A[p, q]), float(A[p, p]), float(A[q, q])
                if apq == 0.0:
                    continue
                theta = (aqq - app) / (2.0 * apq)
                t = (1.0 if theta >= 0.0 else -1.0) / (abs(theta) + math.sqrt(theta * theta + 1.0))
                cs = 1.0 / math.sqrt(t * t + 1.0)
                sn = t * cs
                cp, cq = A[:, p].copy(), A[:, q].copy()
                A[:, p], A[:, q] = cs * cp - sn * cq, sn * cp + cs * cq
                rp, rq = A[p, :].copy(), A[q, :].copy()
                A[p, :], A[q, :] = cs * rp - sn * rq, sn * rp + cs * rq
                vp, vq = V[:, p].copy(), V[:, q].copy()
                V[:, p], V[:, q] = cs * vp - sn * vq, sn * vp + cs * vq


def smallest_diag(A):
    m = 0
    for e in range(1, len(A)):
        if A[e, e] < A[m, m]:
            m = e
    return m


def _stats(contrib, nd):
    st = block_sum(contrib)
    c1x, c1y, c2x, c2y = st[0] / nd, st[1] / nd, st[4] / nd, st[5] / nd
    var1 = (st[2] + st[3]) / nd - (c1x * c1x + c1y * c1y)
    var2 = (st[6] + st[7]) / nd - (c2x * c2x + c2y * c2y)
    return c1x, c1y, c2x, c2y, var1, var2


def refit_f(pts, mask):
    """Normalised 8-point least squares with rank 2 on the rows of `mask` -> F [9] (normalised) or None."""
    x1, y1, x2, y2 = [np.where(mask, pts[:, k], 0.0) for k in range(4)]
    c1x, c1y, c2x, c2y, var1, var2 = _stats(np.stack([x1, y1, x1 * x1, y1 * y1, x2, y2, x2 * x2, y2 * y2], axis=1), float(mask.sum()))
    if not (var1 > 0.0) or not (var2 > 0.0):
        return None
    s1, s2 = math.sqrt(2.0 / var1), math.sqrt(2.0 / var2)
    with np.errstate(all="ignore"):
        u, v = (pts[:, 0] - c1x) * s1, (pts[:, 1] - c1y) * s1
        up, vp = (pts[:, 2] - c2x) * s2, (pts[:, 3] - c2y) * s2
        a = [up * u, up * v, up, vp * u, vp * v, vp, u, v, np.ones_like(u)]
        terms = [np.where(mask, a[k] * a[l], 0.0) for k in range(9) for l in range(k, 9)]
    nm = block_sum(np.stack(terms, axis=1))
    A = np.empty((9, 9))
    e = 0
    for k in range(9):
        for l in range(k, 9):
            A[k, l] = A[l, k] = nm[e]
            e += 1
    V = np.eye(9)
    jacobi(A, V)
    Fn = V[:, smallest_diag(A)].copy()
    G = np.empty((3, 3))
    for r in range(3):
        for c in range(3):
            G[r, c] = Fn[r] * Fn[c] + Fn[3 + r] * Fn[3 + c] + Fn[6 + r] * Fn[6 + c]
    V3 = np.eye(3)
    jacobi(G, V3)
    vv = V3[:, smallest_diag(G)].copy()
    P = np.array([(1.0 if r == c else 0.0) - vv[r] * vv[c] for r in range(3) for c in range(3)])
    F, ok = denormalise_f((c1x, c1y, s1, c2x, c2y, s2), mul3(Fn, P)[None])
    return F[0] if ok[0] else None


def ransac_f(pts, inl_th=0.5, confidence=0.99, max_iters=50000, seed=0):
    """pts [n,4] float32 (x1, y1, x2, y2) -> (F [3,3] float32, mask [n] bool, ninl, iters) as ag_fundamental_ransac computes them."""
    pts = np.asarray(pts, dtype=np.float32).astype(np.float64)
    n = len(pts)
    th = float(np.float32(inl_th))
    th2 = th * th
    log1mconf = math.log(1.0 - float(np.float32(confidence)))
    best, best_F, h_done = 0, None, 0
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
            h_done = min(h0 + VT, max_iters)
            pr = best / n
            p7 = pr * pr * pr * pr * pr * pr * pr
            need = 0.0 if p7 >= 1.0 else (math.inf if p7 <= 0.0 or 1.0 - p7 == 1.0 else math.ceil(log1mconf / math.log(1.0 - p7)))
            if h_done >= min(need, float(max_iters)):
                break
            h0 += VT
    if best == 0:
        return np.zeros((3, 3), np.float32), np.zeros(n, bool), 0, h_done
    F = best_F
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
    return F.reshape(3, 3).astype(np.float32), mask, cnt, h_done
