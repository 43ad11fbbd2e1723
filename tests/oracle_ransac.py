"""numpy restatement of ag_homography_ransac (affnet_b200/csrc/verify.cu), operation for operation: the splitmix64 sampler, the
degeneracy rules, the fp64 closed-form minimal solver, the scoring, the chunked adaptive stop and the normalised-DLT refit with its
fixed-order block reductions and warp-parallel Jacobi.  numpy rounds every product and sum separately, as verify.cu does (it is built
without fused multiply-adds), so the two agree on every decision: samples, inlier counts, iterations and masks."""
import math

import numpy as np

VT = 256              # hypotheses per chunk (threads per CTA)
MAX_DRAWS = 64
COLLINEAR_EPS = 1e-6
JACOBI_SWEEPS = 10
REFIT_ROUNDS = 3
M64 = (1 << 64) - 1


def splitmix64(x):
    """uint64 numpy arrays (wrapping arithmetic) or Python ints."""
    if isinstance(x, int):
        z = (x + 0x9E3779B97F4A7C15) & M64
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        return z ^ (z >> 31)
    z = x + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def draw_indices(seed, h, n):
    """[len(h), MAX_DRAWS] draws in [0, n) of hypotheses h: splitmix64(splitmix64((h << 32) | d) ^ seed), high 32 bits scaled by n."""
    h = np.asarray(h, dtype=np.uint64)[:, None]
    d = np.arange(MAX_DRAWS, dtype=np.uint64)[None, :]
    r = splitmix64(splitmix64((h << np.uint64(32)) | d) ^ np.uint64(seed & M64))
    return ((r >> np.uint64(32)) * np.uint64(n)) >> np.uint64(32)


def samples(seed, h, n):
    """-> (idx [len(h),4] int64, ok [len(h)]): the first 4 distinct draws of each hypothesis (ok False when 64 draws give fewer)."""
    dr = draw_indices(seed, h, n).astype(np.int64)
    eq = dr[:, :, None] == dr[:, None, :]                                   # [H, d, e]
    first = ~np.tril(eq, -1).any(axis=2)                                    # draw d differs from every earlier draw
    rank = np.cumsum(first, axis=1)
    ok = rank[:, -1] >= 4
    idx = np.zeros((len(dr), 4), dtype=np.int64)
    for k in range(4):
        pos = np.argmax(first & (rank == k + 1), axis=1)
        idx[:, k] = dr[np.arange(len(dr)), pos]
    return idx, ok


def adj3(m):
    """Adjugate of [..., 9] row-major matrices, in verify.cu's operation order."""
    o = np.empty_like(m)
    o[..., 0] = m[..., 4] * m[..., 8] - m[..., 5] * m[..., 7]; o[..., 1] = m[..., 2] * m[..., 7] - m[..., 1] * m[..., 8]
    o[..., 2] = m[..., 1] * m[..., 5] - m[..., 2] * m[..., 4]; o[..., 3] = m[..., 5] * m[..., 6] - m[..., 3] * m[..., 8]
    o[..., 4] = m[..., 0] * m[..., 8] - m[..., 2] * m[..., 6]; o[..., 5] = m[..., 2] * m[..., 3] - m[..., 0] * m[..., 5]
    o[..., 6] = m[..., 3] * m[..., 7] - m[..., 4] * m[..., 6]; o[..., 7] = m[..., 1] * m[..., 6] - m[..., 0] * m[..., 7]
    o[..., 8] = m[..., 0] * m[..., 4] - m[..., 1] * m[..., 3]
    return o


def mul3(a, b):
    o = np.empty(np.broadcast_shapes(a.shape, b.shape), dtype=np.float64)
    for r in range(3):
        for c in range(3):
            o[..., 3 * r + c] = a[..., 3 * r] * b[..., c] + a[..., 3 * r + 1] * b[..., 3 + c] + a[..., 3 * r + 2] * b[..., 6 + c]
    return o


def normalise_h(H):
    """H / H[2][2] (rows of [..., 9]) and whether that is finite and H[2][2] != 0."""
    s = H[..., 8:9].copy()
    with np.errstate(divide="ignore", invalid="ignore"):
        Hn = H / s
    return Hn, (s[..., 0] != 0.0) & np.isfinite(Hn).all(axis=-1)


def _cross(ax, ay, bx, by, cx, cy):
    dx1, dy1, dx2, dy2 = bx - ax, by - ay, cx - ax, cy - ay
    cr = dx1 * dy2 - dx2 * dy1
    col = np.abs(cr) <= COLLINEAR_EPS * ((np.abs(dx1) + np.abs(dy1)) * (np.abs(dx2) + np.abs(dy2)))
    return cr, col


def _basis_map(x, y):
    one = np.ones_like(x[:, 0])
    P = np.stack([x[:, 0], x[:, 1], x[:, 2], y[:, 0], y[:, 1], y[:, 2], one, one, one], axis=1)
    A = adj3(P)
    lam = [A[:, 3 * r] * x[:, 3] + A[:, 3 * r + 1] * y[:, 3] + A[:, 3 * r + 2] for r in range(3)]
    return np.stack([P[:, 3 * r + c] * lam[c] for r in range(3) for c in range(3)], axis=1)


def minimal_homographies(c):
    """c [H,4,4] (x1, y1, x2, y2 of the 4 samples, fp64) -> (H [H,9] normalised, ok [H])."""
    x1, y1, x2, y2 = c[:, :, 0], c[:, :, 1], c[:, :, 2], c[:, :, 3]
    col = np.zeros(len(c), dtype=bool)
    neg = np.zeros(len(c), dtype=np.int64)
    for a, b, d in ((0, 1, 2), (1, 2, 3), (0, 2, 3), (0, 1, 3)):
        c1, k1 = _cross(x1[:, a], y1[:, a], x1[:, b], y1[:, b], x1[:, d], y1[:, d])
        c2, k2 = _cross(x2[:, a], y2[:, a], x2[:, b], y2[:, b], x2[:, d], y2[:, d])
        col |= k1 | k2
        neg += (c1 * c2 < 0.0)
    with np.errstate(all="ignore"):
        H = mul3(_basis_map(x2, y2), adj3(_basis_map(x1, y1)))
        H, ok = normalise_h(H)
    return H, ok & ~col & ((neg == 0) | (neg == 4))


def inliers(H, pts, th2):
    """H [9] or [K,9], pts [n,4] -> bool [n] or [K,n]."""
    H = np.atleast_2d(H)[:, :, None]
    x, y, x2, y2 = pts[:, 0], pts[:, 1], pts[:, 2], pts[:, 3]
    with np.errstate(all="ignore"):
        w = H[:, 6] * x + H[:, 7] * y + H[:, 8]
        u = (H[:, 0] * x + H[:, 1] * y + H[:, 2]) / w - x2
        v = (H[:, 3] * x + H[:, 4] * y + H[:, 5]) / w - y2
        m = (w > 0.0) & (u * u + v * v <= th2)
    return m


def block_sum(contrib):
    """contrib [n, K]: the per-row terms, zero rows included; verify.cu's order: thread t sums rows t, t + 256, ... in sequence, an xor
    butterfly within each warp, then warps 0..7 in sequence."""
    n, K = contrib.shape
    R = -(-n // VT)
    X = np.zeros((R * VT, K))
    X[:n] = contrib
    X = X.reshape(R, VT, K)
    acc = np.zeros((VT, K))
    for r in range(R):
        acc = acc + X[r]
    lanes = acc.reshape(VT // 32, 32, K)
    li = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, li ^ o]
    s = lanes[0, 0]
    for w in range(1, VT // 32):
        s = s + lanes[w, 0]
    return s


def refit(pts, mask):
    """Normalised DLT on the rows of `mask` -> H [9] or None."""
    m = mask[:, None]
    x1, y1, x2, y2 = [np.where(mask, pts[:, k], 0.0) for k in range(4)]
    st = block_sum(np.stack([x1, y1, x1 * x1, y1 * y1, x2, y2, x2 * x2, y2 * y2], axis=1))
    nd = float(mask.sum())
    c1x, c1y, c2x, c2y = st[0] / nd, st[1] / nd, st[4] / nd, st[5] / nd
    var1 = (st[2] + st[3]) / nd - (c1x * c1x + c1y * c1y)
    var2 = (st[6] + st[7]) / nd - (c2x * c2x + c2y * c2y)
    if not (var1 > 0.0) or not (var2 > 0.0):
        return None
    s1, s2 = math.sqrt(2.0 / var1), math.sqrt(2.0 / var2)
    u, v = (pts[:, 0] - c1x) * s1, (pts[:, 1] - c1y) * s1
    up, vp = (pts[:, 2] - c2x) * s2, (pts[:, 3] - c2y) * s2
    z, one = np.zeros_like(u), np.ones_like(u)
    a1 = [-u, -v, -one, z, z, z, up * u, up * v, up]
    a2 = [z, z, z, -u, -v, -one, vp * u, vp * v, vp]
    terms = [np.where(mask, a1[k] * a1[l] + a2[k] * a2[l], 0.0) for k in range(9) for l in range(k, 9)]
    nm = block_sum(np.stack(terms, axis=1))
    A = np.empty((9, 9))
    e = 0
    for k in range(9):
        for l in range(k, 9):
            A[k, l] = A[l, k] = nm[e]
            e += 1
    V = np.eye(9)
    for _ in range(JACOBI_SWEEPS):
        for p in range(8):
            for q in range(p + 1, 9):
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
                vp_, vq_ = V[:, p].copy(), V[:, q].copy()
                V[:, p], V[:, q] = cs * vp_ - sn * vq_, sn * vp_ + cs * vq_
    mi = 0
    for e in range(1, 9):
        if A[e, e] < A[mi, mi]:
            mi = e
    Hn = V[:, mi].copy()
    T1 = np.array([s1, 0.0, -(s1 * c1x), 0.0, s1, -(s1 * c1y), 0.0, 0.0, 1.0])
    T2i = np.array([1.0 / s2, 0.0, c2x, 0.0, 1.0 / s2, c2y, 0.0, 0.0, 1.0])
    H, ok = normalise_h(mul3(mul3(T2i, Hn), T1))
    return H if ok else None


def ransac(pts, inl_th=2.0, confidence=0.99, max_iters=50000, seed=0):
    """pts [n,4] float32 (x1, y1, x2, y2) -> (H [3,3] float32, mask [n] bool, ninl, iters) as ag_homography_ransac computes them."""
    pts = np.asarray(pts, dtype=np.float32).astype(np.float64)
    n = len(pts)
    th = float(np.float32(inl_th))
    th2 = th * th
    log1mconf = math.log(1.0 - float(np.float32(confidence)))
    best, best_H, h_done = 0, None, 0
    if n >= 4:
        h0 = 0
        while True:
            h = np.arange(h0, h0 + VT)
            idx, ok = samples(seed, h, n)
            ok &= h < max_iters
            Hs, okh = minimal_homographies(pts[idx])
            ok &= okh
            cnt = np.where(ok, inliers(Hs, pts, th2).sum(axis=1), -1)
            k = int(np.argmax(cnt))          # the first maximum: the lowest h
            if cnt[k] > best:
                best, best_H = int(cnt[k]), Hs[k]
            h_done = min(h0 + VT, max_iters)
            pr = best / n
            p4 = pr * pr * pr * pr
            need = 0.0 if p4 >= 1.0 else (math.inf if p4 <= 0.0 else math.ceil(log1mconf / math.log(1.0 - p4)))
            if h_done >= min(need, float(max_iters)):
                break
            h0 += VT
    if best == 0:
        return np.zeros((3, 3), np.float32), np.zeros(n, bool), 0, h_done
    H = best_H
    mask = inliers(H, pts, th2)[0]
    cnt = int(mask.sum())
    for _ in range(REFIT_ROUNDS):
        if cnt < 4:
            break
        Hr = refit(pts, mask)
        if Hr is None:
            break
        mr = inliers(Hr, pts, th2)[0]
        if int(mr.sum()) < cnt:
            break
        H, mask, cnt = Hr, mr, int(mr.sum())
    return H.reshape(3, 3).astype(np.float32), mask, cnt, h_done
